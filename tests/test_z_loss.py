"""Z-loss in the fused cross-entropy (``z_loss_weight`` on the native models): the fp64 oracle of the ``kZ`` kernels and its
per-element bounds, the margin table of a blockwise fp32 emulator and its mutants, and the op, model and trainer routes.  Runs on
the CPU without the extension; ``test_z_loss_gpu.py`` runs the kernels against the same oracle.

Semantics (PaLM's auxiliary z-loss on top of the, possibly smoothed, cross-entropy; mean over the non-ignored rows)::

    row_loss = ce_row + z lse^2,   lse = log sum_{c<V} exp(x_c)                                  (ignored rows: 0)
    dx_c     = scale (softmax_c (1 + 2 z lse) - (1 - eps) [c = label] - eps / V)          (c < V; padding, ignored rows: 0)
    z_out    = mean over the non-ignored rows of z lse^2

Bounds, on top of those of the smoothed kernels (``test_label_smoothing.ls_ref``; ``E_lse`` the error of the kernel's ``lse``):

* Row term ``(z lse) lse`` and the add to ``ce_row``: ``2 z |lse| E_lse + 2 U z lse^2 + U |row|``; the mean and ``z_out`` add the
  ``ce_reduce`` terms of ``ce_loss_bound`` (the z-terms are summed in the same order as the row losses).
* ``g = 1 + (2 z) lse`` errs by ``E_g = 2 z E_lse + U (|2 z lse| + |g|)``; ``p g`` by ``|g| E_p + p E_g + U |p g|`` with ``E_p`` the
  softmax's bound; then the subtractions and the scale as for smoothing.  Every term is absolute, so ``g`` near 0 (``lse`` near
  ``-1 / 2z``) does not break the bound.

As elsewhere ``E`` is doubled and a bf16 output gets one bf16 ulp on top.  The margin table asserts the emulator stays within half of
every bound and that each mutant (factor 2 missing, ``log2`` for ``ln``, the term on ignored rows, on padding columns, not divided
by the count of valid rows) lands more than 3x outside on some case.  Print it with ``python tests/test_z_loss.py``."""
from __future__ import annotations

import functools
import json
import math
import os
import sys
from typing import Dict, Optional

import pytest
import torch
import torch.nn.functional as F

from test_gemm_oracle import bf16_rn  # noqa: E402
from test_label_smoothing import _block_sum32, host_coeffs, ls_inputs, ls_ref  # noqa: E402
from test_rowwise_oracle import FTZ, U, ce_inputs, ce_loss_bound, e_exp, emulate_ce, f32, out_bound, ratio  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ================================================================================================= fp64 oracle
def formula(x: torch.Tensor, labels: torch.Tensor, eps: float, z: float, ignore_index: int = -100) -> torch.Tensor:
    """The loss as torch autograd sees it: ``F.cross_entropy(label_smoothing=eps) + z mean(logsumexp^2)`` over non-ignored rows."""
    valid = labels != ignore_index
    ce = F.cross_entropy(x, labels, ignore_index=ignore_index, label_smoothing=eps)
    return ce + z * torch.logsumexp(x[valid], -1).square().sum() / max(int(valid.sum()), 1)


def z_ref(logits, labels, V: int, eps: float, z: float, ignore_index: int = -100, scale: Optional[float] = None):
    """fp64 oracle of the ``kZ`` kernels: ``lse`` / ``inv_n`` as the unsmoothed oracle, row losses with the z-term, mean ``loss``,
    mean z-term ``z_out``, and with ``scale`` the d-logits (0 on ignored rows and padding columns).  Bounds included."""
    o = ls_ref(logits, labels, V, eps, ignore_index)
    T, Vp = logits.shape
    x = logits[:, :V].double()
    valid = labels.to(x.device) != ignore_index
    lab = torch.where(valid, labels.to(x.device), torch.zeros_like(labels.to(x.device)))
    lse = torch.logsumexp(x, 1)
    E_lse = torch.where(valid, (o["b_lse"] - FTZ) / 2, torch.zeros_like(lse))
    zt = torch.where(valid, z * lse * lse, torch.zeros_like(lse))
    row = o["row"] + zt
    E_zt = torch.where(valid, 2 * z * lse.abs() * E_lse + 2 * U * zt, torch.zeros_like(lse))
    E_row = o["E_row"] + E_zt + U * row.abs()
    inv = o["inv_n"]
    loss = float(row.sum()) * inv
    z_out = float(zt.sum()) * inv
    res = {"lse": o["lse"], "inv_n": inv, "b_lse": o["b_lse"], "b_inv": o["b_inv"], "loss": loss, "row": row, "E_row": E_row,
           "b_loss": ce_loss_bound(float(E_row.sum()), float(row.abs().sum()), T, loss, inv),
           "z": z_out, "zt": zt, "E_zt": E_zt, "b_z": ce_loss_bound(float(E_zt.sum()), float(zt.sum()), T, z_out, inv)}
    if scale is not None:
        a, b = 1.0 - eps, eps / V
        arg = x - lse[:, None]
        p = torch.exp(arg)
        g = (1 + 2 * z * lse)[:, None]
        oh = torch.zeros_like(p)
        oh.scatter_(1, lab[:, None], 1.0)
        pg = p * g
        q = (pg - a * oh - b) * scale
        E_p = p * (E_lse[:, None] + U * arg.abs() + e_exp(arg))
        E_g = 2 * z * E_lse[:, None] + U * ((g - 1).abs() + g.abs())
        E_pg = g.abs() * E_p + p * E_g + U * pg.abs()
        E_sub = U * (pg - b).abs() + 2 * U * b + oh * (U * (pg - b - a).abs() + U * (eps + a))
        E = 2 * (abs(scale) * (E_pg + E_sub) + U * q.abs())
        grad = torch.zeros(T, Vp, dtype=torch.float64, device=x.device)
        bnd = torch.full((T, Vp), FTZ, dtype=torch.float64, device=x.device)
        grad[:, :V] = torch.where(valid[:, None], q, torch.zeros_like(q))
        bnd[:, :V] = torch.where(valid[:, None], out_bound(q, E, FTZ * (1 + abs(scale) * (1 + g.abs()))), torch.full_like(q, FTZ))
        res.update(grad=grad, b_grad=bnd)
    return res


def z_checks(got, o) -> Dict[str, float]:
    out = {"lse": ratio(got["lse"], o["lse"], o["b_lse"]),
           "loss": abs(float(got["loss"]) - o["loss"]) / o["b_loss"],
           "z": abs(float(got["z"]) - o["z"]) / o["b_z"],
           "inv_n": abs(float(got["inv_n"]) - o["inv_n"]) / max(o["b_inv"], FTZ)}
    if "grad" in got:
        out["grad"] = ratio(got["grad"], o["grad"], o["b_grad"])
    return out


# ================================================================================================= emulator
Z_MUTANTS = ("no_factor_2", "log2", "z_on_ignored", "z_on_padding", "not_divided")


def emulate_z(logits, labels, V: int, eps: float, z: float, ignore_index: int = -100, scale: float = 1.0, mutant=None):
    """fp32 emulator of ``ce_fwd_kernel<kSmooth, true>`` (the unsmoothed emulator's lse; with eps the row sum of x in the kernel's
    order), ``ce_reduce_kernel<true>`` and ``ce_bwd_kernel<kSmooth, true>``."""
    T, Vp = logits.shape
    x = logits.double()
    lse = emulate_ce(logits, labels, V, ignore_index)["lse"]
    valid = labels != ignore_index
    lab = torch.where(valid, labels, torch.zeros_like(labels))
    xl = x.gather(1, lab[:, None])[:, 0]
    if eps:
        a, bV = host_coeffs(eps)
        b = bV(V)
        nvf = V // 8
        K = -(-nvf // 512)
        xv = torch.zeros(T, K * 512 * 8, dtype=torch.float64)
        xv[:, :nvf * 8] = x[:, :nvf * 8]
        xv = xv.view(T, K, 512, 8)
        sx = torch.zeros(T, 512, dtype=torch.float64)
        for k in range(K):
            ax = xv[:, k, :, 0]
            for j in range(1, 8):
                ax = f32(ax + xv[:, k, :, j])
            sx = f32(sx + ax)
        for c in range(nvf * 8, V):
            sx[:, c - nvf * 8] = f32(sx[:, c - nvf * 8] + x[:, c])
        ce = f32(f32(lse - a * xl) - b * _block_sum32(sx))
    else:
        a, b = 1.0, 0.0
        ce = f32(lse - xl)
    lz = lse
    if mutant == "log2":
        lz = f32(lse / math.log(2.0))
    if mutant in ("z_on_ignored", "z_on_padding"):       # lse of every row (ignored ones too) / over the padding columns as well
        lz = f32(torch.logsumexp(torch.nan_to_num(x[:, :Vp if mutant == "z_on_padding" else V], nan=0.0), 1))
        if mutant == "z_on_padding":
            lz = torch.where(valid, lz, torch.zeros_like(lz))
    zt = f32(f32(z * lz) * lz)
    row = torch.where(valid, f32(ce + zt), torch.zeros_like(ce))
    counted = torch.ones_like(valid) if mutant == "z_on_ignored" else valid
    tot = torch.tensor(0.0, dtype=torch.float64)
    zs = torch.tensor(0.0, dtype=torch.float64)
    for i in range(T):
        if counted[i]:
            tot = f32(tot + (row[i] if valid[i] else zt[i]))
            zs = f32(zs + zt[i])
    n = int(valid.sum())
    inv = float(f32(torch.tensor(1.0 / n))) if n else 0.0
    loss = float(f32(tot * inv))
    z_out = float(f32(zs * inv))
    if mutant == "not_divided":               # mean CE + sum of the z-terms: the z-gradient carries n times its weight
        loss = float(f32(f32(f32(tot - zs) * inv) + zs))
        z_out = float(zs)
    zf = f32(z * (n if mutant == "not_divided" else 1) * (1 if mutant == "no_factor_2" else 2) * lz)
    gf = f32(1 + zf)
    cols = torch.arange(Vp)
    live = cols[None, :] < (Vp if mutant == "z_on_padding" else V)
    p = torch.where(live, f32(torch.exp(f32(torch.nan_to_num(x, nan=0.0) - lse[:, None]))), torch.zeros_like(x))
    p = torch.where(live, f32(p * gf[:, None] - b), p)
    if mutant == "z_on_padding":             # padding columns: only the z part of the gradient, 2 z lse softmax
        pad = cols[None, :] >= V
        p = torch.where(pad, f32(f32(torch.exp(f32(torch.nan_to_num(x, nan=0.0) - lse[:, None]))) * zf[:, None]), p)
    lab_row = torch.where(valid, lab, torch.full_like(lab, -1))
    p = torch.where(cols[None, :] == lab_row[:, None], f32(p - a), p)
    grad = bf16_rn(f32(p * scale)).double()
    if mutant != "z_on_ignored":
        grad = torch.where(valid[:, None], grad, torch.zeros_like(grad))
    else:                                     # ignored rows keep the z part of their gradient
        zg = bf16_rn(f32(f32(torch.exp(f32(torch.nan_to_num(x, nan=0.0) - lz[:, None])) * zf[:, None]) * scale)).double()
        zg = torch.where(cols[None, :] < V, zg, torch.zeros_like(zg))
        grad = torch.where(valid[:, None], grad, zg)
    return {"lse": lse, "loss": loss, "z": z_out, "inv_n": inv, "grad": grad}


# ================================================================================================= oracle vs autograd
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("z", [1e-4, 1e-2, 1.0])
@pytest.mark.parametrize("V,Vp", [(37, 40), (40, 40), (1003, 1008)], ids=["ragged-padded", "exact", "ragged-1003"])
def test_oracle_matches_fp64_autograd(eps, z, V, Vp):
    """Ignored rows (every 5th), padding columns and a ragged V, against autograd of the formula in fp64."""
    lg, lab = ce_inputs(12, V, Vp, seed=V, pad_fill=30.0)
    n = int((lab != -100).sum())
    o = z_ref(lg, lab, V, eps, z, scale=2.5 / n)                        # the kernel's scale is dloss * inv_n
    xr = lg[:, :V].double().requires_grad_(True)
    loss = formula(xr, lab, eps, z)
    (loss * 2.5).backward()
    assert abs(o["loss"] - float(loss.detach())) < 1e-12 * max(1.0, abs(o["loss"]))
    torch.testing.assert_close(o["grad"][:, :V], xr.grad, rtol=1e-12, atol=1e-12)
    assert bool((o["grad"][:, V:] == 0).all()) and bool((o["grad"][lab == -100] == 0).all())
    valid = lab != -100
    want_z = z * float(torch.logsumexp(lg[valid, :V].double(), -1).square().mean())
    assert abs(o["z"] - want_z) <= 1e-12 * want_z
    assert abs(o["loss"] - o["z"] - float(F.cross_entropy(lg[:, :V].double(), lab, label_smoothing=eps))) < 1e-12 * abs(o["loss"])


@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_all_ignored_batch_has_zero_loss_and_gradient(eps):
    lg, lab = ce_inputs(8, 50, 56, seed=4)
    lab[:] = -100
    o = z_ref(lg, lab, 50, eps, 1.0, scale=1.0)
    assert o["loss"] == 0.0 and o["z"] == 0.0 and o["inv_n"] == 0.0 and bool((o["grad"] == 0).all())
    e = emulate_z(lg, lab, 50, eps, 1.0)
    assert e["loss"] == 0.0 and e["z"] == 0.0 and e["inv_n"] == 0.0 and bool((e["grad"] == 0).all())


# ================================================================================================= margin table
Z_CASES = [
    # (name, T, V, Vp, eps, z, shift of every logit, padding fill)
    ("z-50257-1e-4", 6, 50257, 50304, 0.0, 1e-4, 0.0, None),
    ("z-50257-1e-4-shift", 6, 50257, 50304, 0.0, 1e-4, 12.0, 30.0),
    ("z-50257-1e-2-e0.1", 6, 50257, 50304, 0.1, 1e-2, 12.0, 30.0),
    ("z-131-1-shift", 12, 131, 136, 0.0, 1.0, 12.0, 30.0),
    ("z-131-1e-2-e0.1", 12, 131, 136, 0.1, 1e-2, 0.0, None),
    ("z-1000-1e-2-neg", 12, 1000, 1008, 0.0, 1e-2, -40.0, 30.0),
    ("z-1003-1-e0.1", 12, 1003, 1008, 0.1, 1.0, 4.0, 20.0),
    ("z-128256-1e-4-e0.1", 6, 128256, 128256, 0.1, 1e-4, 0.0, None),
]


def z_row(name, T, V, Vp, eps, z, shift, pad_fill):
    lg, lab = ls_inputs(T, V, Vp, shift, pad_fill, seed=V)
    o = z_ref(lg, lab, V, eps, z, scale=0.75)
    emu = z_checks(emulate_z(lg, lab, V, eps, z, scale=0.75), o)
    caught = {}
    for m in Z_MUTANTS:
        if m == "z_on_padding" and Vp == V:
            continue
        c = z_checks(emulate_z(lg, lab, V, eps, z, scale=0.75, mutant=m), o)
        caught[m] = max(c.items(), key=lambda kv: kv[1])
    return emu, caught


ROWS = {c[0]: functools.lru_cache(maxsize=None)(lambda c=c: z_row(*c)) for c in Z_CASES}     # both tests read one evaluation


@pytest.mark.parametrize("name", list(ROWS))
def test_margin_table_emulator_within_half(name):
    emu, _ = ROWS[name]()
    for k, r in emu.items():
        assert r < 0.5, (name, "emulator", k, r)


def test_every_mutant_lands_3x_outside_on_some_case():
    best = {m: 0.0 for m in Z_MUTANTS}
    for name, row in ROWS.items():
        _, caught = row()
        for m, (k, r) in caught.items():
            best[m] = max(best[m], r)
    assert all(r > 3.0 for r in best.values()), best


# ================================================================================================= op reference path
def test_op_reference_path_adds_the_term_and_writes_z_out():
    from acco_b200 import ops
    lg, lab = ce_inputs(9, 37, 40, seed=6)
    out = torch.full((1,), -1.0)
    got = ops.softmax_cross_entropy(lg.float(), lab, 37, -100, label_smoothing=0.2, z_loss=1e-2, z_loss_out=out)
    x = lg[:, :37].float()
    valid = lab != -100
    zt = 1e-2 * torch.logsumexp(x[valid], -1).square().mean()
    assert torch.allclose(out, zt.reshape(1), rtol=1e-6, atol=0)
    assert float(got) == pytest.approx(float(F.cross_entropy(x, lab, label_smoothing=0.2) + zt), rel=1e-6)
    plain = ops.softmax_cross_entropy(lg.float(), lab, 37, -100, label_smoothing=0.2)
    assert float(ops.softmax_cross_entropy(lg.float(), lab, 37, -100, label_smoothing=0.2, z_loss=0.0)) == float(plain)
    for bad in (-1e-4, math.nan, math.inf):
        with pytest.raises(ValueError, match="z_loss"):
            ops.softmax_cross_entropy(lg.float(), lab, 37, z_loss=bad)


# ================================================================================================= models
def _tiny_llama():
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    return LlamaForCausalLM(LlamaConfig(vocab_size=90, hidden_size=32, intermediate_size=48, num_hidden_layers=2, num_attention_heads=4,
                                        num_key_value_heads=2, max_position_embeddings=32, pad_vocab_multiple=8))


def _tiny_gpt():
    from acco_b200.models import GPTConfig, GPTForCausalLM
    torch.manual_seed(0)
    return GPTForCausalLM(GPTConfig(vocab_size=90, hidden_size=32, num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=32,
                                    attention_layers=["global", "local"], window_size=8, pad_vocab_multiple=8))


@pytest.mark.parametrize("make", [_tiny_llama, _tiny_gpt], ids=["llama-gqa", "gptneo"])
@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_native_model_matches_the_formula(make, eps):
    """``model.z_loss_weight = z`` with labels gives the loss and gradients of the formula on the model's own logits (fp32)."""
    m = make().float()
    assert m.config.padded_vocab > m.config.vocab_size and m.z_loss_weight == 0.0
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 90, (3, 16), generator=g)
    labels = ids.clone()
    labels[0, 10:] = -100
    labels[2, :] = -100
    m.label_smoothing, m.z_loss_weight = eps, 1e-2
    m.z_loss_out = torch.zeros(1)
    loss = m(input_ids=ids, labels=labels)[0]
    loss.backward()
    got = {k: p.grad.clone() for k, p in m.named_parameters()}
    m.zero_grad()
    m.z_loss_weight = 0.0
    logits = m(input_ids=ids).logits[:, :-1].reshape(-1, 90)
    tgt = labels[:, 1:].reshape(-1)
    ref = formula(logits, tgt, eps, 1e-2)
    ref.backward()
    assert abs(float(loss.detach()) - float(ref.detach())) <= 2e-6 * abs(float(ref.detach()))
    zt = 1e-2 * torch.logsumexp(logits.detach()[tgt != -100], -1).square().mean()
    assert float(m.z_loss_out) == pytest.approx(float(zt), rel=2e-6)
    for k, p in m.named_parameters():
        torch.testing.assert_close(got[k], p.grad, rtol=1e-4, atol=1e-6, msg=k)


# ================================================================================================= trainer
class _ZRef(torch.nn.Module):
    """A non-native model around the same weights whose loss is the formula in plain torch: the reference the trainer is checked
    against (it runs with the key off)."""

    def __init__(self, m, z):
        super().__init__()
        self.m, self.z = m, z

    def forward(self, input_ids=None, labels=None, **kw):
        logits = self.m(input_ids=input_ids, **kw).logits
        V = logits.shape[-1]
        return (formula(logits[:, :-1].reshape(-1, V).float(), labels[:, 1:].reshape(-1), 0.0, self.z),)


def _trainer(model, z, method="acco", **kw):
    from acco_b200 import DecoupledTrainer
    from acco_b200.data import synthetic_pretrain_dataset
    from acco_b200.launch import DistEnv
    from helpers import LOG, base_args
    ds = synthetic_pretrain_dataset(200, 30, 96, 16, seed=3)
    args = base_args(method_name=method, **{"nb_steps_tot": 8, **kw})
    if z is not None:
        args["z_loss_weight"] = z
    return DecoupledTrainer(model=model, train_dataset=ds, eval_dataset=ds, args=args, log=LOG, env=DistEnv(id_run="zl"))


class _Recorder:
    def __init__(self):
        self.logs = []

    def __getattr__(self, name):
        return lambda *a: None

    def on_log(self, trainer, scalars):
        self.logs.append(dict(scalars))


def _trace(t):
    out = []
    while not t.finished():
        t.step()
        out.append((float(t.loss_host), float(t.z_loss_host)))
    return out


def _logged(t):
    rec = _Recorder()
    t.add_callback(rec)
    t.train()
    return [(d["loss"], d.get("z_loss")) for d in rec.logs]


@pytest.mark.parametrize("method,impl", [("acco", "native"), ("dpu", "native"), ("ddp", "native"), ("ddp", "torch")])
def test_trainers_track_the_torch_reference(workdir, method, impl):
    from helpers import tiny_model
    t = _trainer(tiny_model(), 1e-2, method, ddp_impl=impl, log_every=1, nb_steps_tot=16)
    assert t.model.z_loss_weight == 1e-2 and t.model.z_loss_out is t.z_loss_static
    t.is_cuda = True                                       # graphs need a GPU; everything else about the route allows them
    assert t._use_graphs()
    t.is_cuda = False
    ref = _trainer(_ZRef(tiny_model(), 1e-2), None, method, ddp_impl=impl, log_every=1, nb_steps_tot=16)
    a, b = _logged(t), _logged(ref)
    assert len(a) == len(b) >= 4
    for (x, zx), (y, zy) in zip(a, b):
        assert abs(x - y) <= 1e-5 * abs(y), (a, b)
        assert 0.0 < zx < x and zy is None
    plain = _logged(_trainer(tiny_model(), None, method, ddp_impl=impl, log_every=1, nb_steps_tot=16))
    assert max(abs(x - y) for (x, _), (y, _) in zip(a, plain)) > 1e-2       # the term is really on


def test_weight_zero_is_the_run_without_the_key(workdir):
    from helpers import tiny_model
    t0, t1 = _trainer(tiny_model(), 0, "acco"), _trainer(tiny_model(), None, "acco")
    assert t0.model.z_loss_weight == 0.0 and t0.model.z_loss_out is None
    assert _trace(t0) == _trace(t1)
    assert torch.equal(t0.get_weights(), t1.get_weights())


@pytest.mark.parametrize("z", [-1e-4, math.nan, math.inf, -math.inf, True, False, "1e-4"])
def test_trainer_rejects_bad_weight(workdir, z):
    from helpers import tiny_model
    with pytest.raises(ValueError, match="z_loss_weight"):
        _trainer(tiny_model(), z)


def test_trainer_rejects_a_non_native_model(workdir):
    from helpers import tiny_model
    with pytest.raises(ValueError, match="native model"):
        _trainer(_ZRef(tiny_model(), 0.0), 1e-4)
    assert _trainer(_ZRef(tiny_model(), 0.0), 0.0).z_loss_weight == 0.0          # the key off is accepted with any model


def test_eval_loop_returns_the_unregularised_loss(workdir):
    from helpers import tiny_model
    on, off = _trainer(tiny_model(), 1.0, max_eval_batches=3), _trainer(tiny_model(), None, max_eval_batches=3)
    e_on, e_off = on.eval_loop(), off.eval_loop()
    assert float(e_on) == float(e_off)
    assert on.model.z_loss_weight == 1.0 and float(on.z_loss_static) == 0.0       # restored, and eval wrote no z-term
    _trace(on)
    assert float(on.z_loss_static) > 0.0


@pytest.mark.parametrize("z", [None, 1e-2])
def test_z_loss_is_logged_only_with_the_key(workdir, z):
    from helpers import tiny_model
    t = _trainer(tiny_model(), z, tensorboard=True, log_every=2, nb_steps_tot=10)
    rec = _Recorder()
    t.add_callback(rec)
    t.train()
    t.writer.flush()
    assert rec.logs
    rows = [json.loads(line) for line in open(os.path.join(t.writer.logdir, "scalars.jsonl"))]
    tags = {r["tag"] for r in rows}
    if z is None:
        assert all("z_loss" not in d for d in rec.logs) and "z_loss" not in tags
        return
    assert all(0.0 < d["z_loss"] < d["loss"] for d in rec.logs), rec.logs
    assert "z_loss" in tags and sum(r["tag"] == "z_loss" for r in rows) == len(rec.logs)


def test_cli_pretraining_with_z_loss(workdir, monkeypatch):
    sys.path.insert(0, ROOT)
    import main as cli
    from acco_b200 import ops
    seen = []
    orig = ops.softmax_cross_entropy

    def ce(*a, **kw):
        seen.append(kw.get("z_loss"))
        return orig(*a, **kw)
    monkeypatch.setattr(ops, "softmax_cross_entropy", ce)
    stats = cli.main(["train=acco", "model=tiny", "data=synthetic", "train.nb_steps_tot=6", "train.batch_size=2", "train.max_length=32",
                      "train.use_mixed_precision=False", "data.synthetic_docs=200", "data.synthetic_mean_len=12", "train.warmup=0",
                      "run_name=zloss", "train.save=False", "train.z_loss_weight=1e-4", "train.dataloader_num_workers=0"])
    assert stats["count_grad_tot"] >= 6
    assert seen and set(seen) == {1e-4}


if __name__ == "__main__":               # print the margin table: python tests/test_z_loss.py
    for name, row in ROWS.items():
        emu, caught = row()
        print(f"{name:22s} emulator/bound " + " ".join(f"{k}={v:.3f}" for k, v in emu.items()))
        for m, (k, r) in caught.items():
            print(f"{'':22s}   mutant {m:15s} worst {k}: {r:.3g}x")
