"""Label smoothing in the fused cross-entropy (``label_smoothing_factor`` on the native models): the fp64 oracle of the smoothed
kernels and its per-element bounds, the margin table of a blockwise fp32 emulator and its mutants, and the model and trainer
routes.  Runs on the CPU without the extension; ``test_label_smoothing_gpu.py`` runs the kernels against the same oracle.

Semantics (HF ``LabelSmoother`` / ``F.cross_entropy(label_smoothing=eps)`` over the V valid columns, mean over non-ignored rows)::

    row_loss = lse - (1 - eps) x[label] - (eps / V) sum_{c<V} x_c              (ignored rows: 0)
    dx_c     = scale (softmax_c - (1 - eps) [c = label] - eps / V)            (c < V; padding columns and ignored rows: 0)

Bounds, on top of those of the unsmoothed kernels (``test_rowwise_oracle.py``: ``E_lse``, the ``ce_reduce`` sum and ``1 / n``).
``a = 1 - eps`` and ``b = eps / V`` are rounded to fp32 on the host from the fp32 eps: ``|a - (1 - eps)| <= U (eps + a)``,
``|b - eps / V| <= 2 U b``.

* ``sum x``: a thread adds 8 logits in sequence per vector, adds that to its running sum (``n_sw`` sweeps including the ragged
  tail), and the CTA sums 512 partials through two 5-level butterflies, so the row sum errs by at most ``D_SX U sum|x|`` with
  ``D_SX = n_sw + 17``.
* Row loss ``(lse - a xl) - b sx`` (two subtractions, products possibly fused): ``E_lse + |xl| U (eps + a) + U |a xl| +
  b (D_SX U sum|x| + 3 U |sx|) + 2 U (|lse| + |a xl| + |b sx|)``; the mean adds the ``ce_reduce`` terms of ``ce_loss_bound``.
* d-logits ``((p - b) - a [label]) * scale``: ``p`` errs by ``p (E_lse + U |x - lse| + e_exp(x - lse))`` as before; the two
  subtractions add ``U |p - b| + 2 U b`` and, at the label, ``U |p - b - a| + U (eps + a)``; the product ``U |q|``.  Every term is
  absolute, so ``p ~ b`` (a row of equal logits at eps = 1) cancels without breaking the bound.

As for the other row-wise kernels, ``E`` is doubled and a bf16 output gets one bf16 ulp on top (``out_bound``).  The margin table
(``test_margin_table_emulator_within_half``, ``test_every_mutant_lands_3x_outside_on_some_case``) asserts the emulator stays
within half of every bound and that each mutant lands more than 3x outside on some case.  The ``eps / Vp`` mutant moves the loss by ``eps (Vp - V) / V`` times the mean logit, so its cases shift the logits by a
constant; the ``padding in sum x`` mutant is caught where the padding holds large values.  Print the table with
``python tests/test_label_smoothing.py``."""
from __future__ import annotations

import math
from typing import Dict, Optional

import pytest
import torch
import torch.nn.functional as F

from test_gemm_oracle import bf16_rn  # noqa: E402
from test_rowwise_oracle import (FTZ, U, ce_inputs, ce_loss_bound, ce_ref, e_exp, emulate_ce, f32, out_bound,  # noqa: E402
                                 ratio)


# ================================================================================================= fp64 oracle
def host_coeffs(eps: float):
    """``(1 - eps, eps / V)`` as the host computes them: fp32, from the fp32 eps (returned as a function of V)."""
    e32 = torch.tensor(eps, dtype=torch.float32)
    a = float(torch.tensor(1.0, dtype=torch.float32) - e32)
    return a, (lambda V: float(e32 / torch.tensor(float(V), dtype=torch.float32)))


def ls_ref(logits, labels, V: int, eps: float, ignore_index: int = -100, scale: Optional[float] = None):
    """fp64 oracle of the smoothed kernels: ``lse`` / ``inv_n`` (and their bounds) as the unsmoothed oracle, smoothed row losses
    and mean ``loss``, and with ``scale`` the smoothed d-logits (0 on ignored rows and padding columns).  Bounds included."""
    o = ce_ref(logits, labels, V, ignore_index)
    T, Vp = logits.shape
    x = logits[:, :V].double()
    valid = labels.to(x.device) != ignore_index
    lab = torch.where(valid, labels.to(x.device), torch.zeros_like(labels.to(x.device)))
    lse = torch.logsumexp(x, 1)
    xl = x.gather(1, lab[:, None])[:, 0]
    sx = x.sum(1)
    sabs = x.abs().sum(1)
    a, b = 1.0 - eps, eps / V
    row = torch.where(valid, lse - a * xl - b * sx, torch.zeros_like(lse))
    inv = o["inv_n"]
    loss = float(row.sum()) * inv
    E_lse = (o["b_lse"] - FTZ) / 2
    n_sw = -(-(V // 8) // 512) + 1
    D_SX = n_sw + 17
    E_row = E_lse + xl.abs() * U * (eps + a) + U * (a * xl).abs() + b * (D_SX * U * sabs + 3 * U * sx.abs()) \
        + 2 * U * (lse.abs() + (a * xl).abs() + (b * sx).abs())
    E_row = torch.where(valid, E_row, torch.zeros_like(E_row))
    res = {"lse": o["lse"], "inv_n": inv, "b_lse": o["b_lse"], "b_inv": o["b_inv"], "loss": loss, "row": row, "E_row": E_row,
           "b_loss": ce_loss_bound(float(E_row.sum()), float(row.abs().sum()), T, loss, inv)}
    if scale is not None:
        arg = x - lse[:, None]
        p = torch.exp(arg)
        oh = torch.zeros_like(p)
        oh.scatter_(1, lab[:, None], 1.0)
        q = (p - a * oh - b) * scale
        E_p = p * (E_lse[:, None] + U * arg.abs() + e_exp(arg))
        E_sub = U * (p - b).abs() + 2 * U * b + oh * (U * (p - b - a).abs() + U * (eps + a))
        E = 2 * (abs(scale) * (E_p + E_sub) + U * q.abs())
        grad = torch.zeros(T, Vp, dtype=torch.float64, device=x.device)
        bnd = torch.full((T, Vp), FTZ, dtype=torch.float64, device=x.device)
        grad[:, :V] = torch.where(valid[:, None], q, torch.zeros_like(q))
        bnd[:, :V] = torch.where(valid[:, None], out_bound(q, E, FTZ * (1 + abs(scale))), torch.full_like(q, FTZ))
        res.update(grad=grad, b_grad=bnd)
    return res


def ls_checks(got, o) -> Dict[str, float]:
    out = {"lse": ratio(got["lse"], o["lse"], o["b_lse"]),
           "loss": abs(float(got["loss"]) - o["loss"]) / o["b_loss"],
           "inv_n": abs(float(got["inv_n"]) - o["inv_n"]) / max(o["b_inv"], FTZ)}
    if "grad" in got:
        out["grad"] = ratio(got["grad"], o["grad"], o["b_grad"])
    return out


# ================================================================================================= emulator
LS_MUTANTS = ("eps_over_Vp", "pad_in_sum", "no_one_m_eps", "no_eps_v_bwd", "smooth_ignored")


def _block_sum32(part: torch.Tensor) -> torch.Tensor:
    """``block_sum`` over 512 per-thread fp32 values ``[T, 512]``: a 5-level butterfly per warp, then one over the 16 warp sums."""
    T = part.shape[0]
    v = part.view(T, 16, 32)
    for o in (16, 8, 4, 2, 1):
        v = f32(v + v[..., torch.arange(32) ^ o])
    w = torch.zeros(T, 32, dtype=torch.float64)
    w[:, :16] = v[..., 0]
    for o in (16, 8, 4, 2, 1):
        w = f32(w + w[:, torch.arange(32) ^ o])
    return w[:, 0]


def emulate_ls(logits, labels, V: int, eps: float, ignore_index: int = -100, scale: float = 1.0, mutant=None):
    """fp32 emulator of the smoothed ``ce_fwd_kernel`` (the unsmoothed emulator's lse, plus the row sum of x in the kernel's
    order: 8-term vector sums, a running sum over the sweeps and the ragged tail, ``block_sum``), ``ce_reduce_kernel`` and the
    smoothed ``ce_bwd_kernel``."""
    T, Vp = logits.shape
    x = logits.double()
    lse = emulate_ce(logits, labels, V, ignore_index)["lse"]
    a, bV = host_coeffs(eps)
    b = bV(Vp if mutant == "eps_over_Vp" else V)
    Vs = Vp if mutant == "pad_in_sum" else V
    nvf = Vs // 8
    K = -(-nvf // 512)
    xv = torch.zeros(T, K * 512 * 8, dtype=torch.float64)
    xv[:, :nvf * 8] = torch.nan_to_num(x[:, :nvf * 8], nan=0.0)
    xv = xv.view(T, K, 512, 8)
    sx = torch.zeros(T, 512, dtype=torch.float64)
    for k in range(K):
        ax = xv[:, k, :, 0]
        for j in range(1, 8):
            ax = f32(ax + xv[:, k, :, j])
        sx = f32(sx + ax)
    for c in range(nvf * 8, Vs):
        t = c - nvf * 8
        sx[:, t] = f32(sx[:, t] + x[:, c])
    gsx = _block_sum32(sx)
    valid = labels != ignore_index
    lab = torch.where(valid, labels, torch.zeros_like(labels))
    xl = x.gather(1, lab[:, None])[:, 0]
    a_l = 1.0 if mutant == "no_one_m_eps" else a
    lse_all = f32(torch.logsumexp(x[:, :V], 1)) if mutant == "smooth_ignored" else lse
    row = f32(f32(lse_all - a_l * xl) - b * gsx)
    if mutant == "smooth_ignored":        # ignored rows keep the smoothing term eps (lse - mean x) and its gradient
        row = torch.where(valid, row, f32(eps * lse_all - b * gsx))
    else:
        row = torch.where(valid, row, torch.zeros_like(row))
    tot = torch.tensor(0.0, dtype=torch.float64)
    for i in range(T):
        if valid[i] or mutant == "smooth_ignored":
            tot = f32(tot + row[i])
    n = int(valid.sum())
    inv = float(f32(torch.tensor(1.0 / n))) if n else 0.0
    loss = float(f32(tot * inv))
    cols = torch.arange(Vp)
    live = cols[None, :] < V
    p = torch.where(live, ex32(f32(torch.nan_to_num(x, nan=0.0) - lse_all[:, None])), torch.zeros_like(x))
    if mutant != "no_eps_v_bwd":
        p = torch.where(live, f32(p - b), p)
    lab_row = torch.where(valid, lab, torch.full_like(lab, -1))
    p = torch.where(cols[None, :] == lab_row[:, None], f32(p - a_l), p)
    grad = bf16_rn(f32(p * scale)).double()
    if mutant != "smooth_ignored":
        grad = torch.where(valid[:, None], grad, torch.zeros_like(grad))
    return {"lse": lse, "loss": loss, "inv_n": inv, "grad": grad}


def ex32(a):
    return f32(torch.exp(a))


# ================================================================================================= oracle vs autograd
@pytest.mark.parametrize("eps", [0.1, 0.5, 1.0])
def test_oracle_matches_fp64_autograd_and_label_smoother(eps):
    from acco_b200.utils.misc import LabelSmoother
    lg, lab = ce_inputs(12, 37, 40, seed=3)
    n = int((lab != -100).sum())
    o = ls_ref(lg, lab, 37, eps, scale=2.5 / n)                        # the kernel's scale is dloss * inv_n
    xr = lg[:, :37].double().requires_grad_(True)
    loss = F.cross_entropy(xr, lab, ignore_index=-100, label_smoothing=eps)
    (loss * 2.5).backward()
    assert abs(o["loss"] - float(loss.detach())) < 1e-12
    torch.testing.assert_close(o["grad"][:, :37], xr.grad, rtol=1e-12, atol=1e-12)
    assert bool((o["grad"][:, 37:] == 0).all()) and bool((o["grad"][lab == -100] == 0).all())
    # LabelSmoother up-casts to fp32 whatever it is given: agreement to fp32 accuracy
    xs = lg[:, :37].double().requires_grad_(True)
    ls = LabelSmoother(eps)({"logits": xs}, lab)
    (ls * 2.5).backward()
    assert abs(float(ls.detach()) - o["loss"]) <= 1e-5 * abs(o["loss"])
    torch.testing.assert_close(o["grad"][:, :37], xs.grad, rtol=1e-4, atol=1e-7)


def test_all_ignored_batch_has_zero_loss_and_gradient():
    lg, lab = ce_inputs(8, 50, 56, seed=4)
    lab[:] = -100
    o = ls_ref(lg, lab, 50, 0.3, scale=1.0)
    assert o["loss"] == 0.0 and o["inv_n"] == 0.0 and bool((o["grad"] == 0).all())
    e = emulate_ls(lg, lab, 50, 0.3)
    assert e["loss"] == 0.0 and e["inv_n"] == 0.0 and bool((e["grad"] == 0).all())


def test_host_coefficients_are_fp32():
    a, bV = host_coeffs(0.1)
    assert a == float(torch.tensor(0.9, dtype=torch.float32)) or abs(a - 0.9) < 2 ** -24
    assert bV(50257) == float(torch.tensor(0.1, dtype=torch.float32) / 50257)


# ================================================================================================= margin table
LS_CASES = [
    # (name, T, V, Vp, eps, shift of every logit, padding fill)
    ("ls-50257-e0.1", 10, 50257, 50304, 0.1, 0.0, None),
    ("ls-50257-e0.1-shift", 10, 50257, 50304, 0.1, 12.0, 30.0),
    ("ls-131-e0.5-shift", 12, 131, 136, 0.5, 12.0, 30.0),
    ("ls-1000-e1.0-shift", 12, 1000, 1008, 1.0, 12.0, 30.0),
    ("ls-1000-e0.1", 10, 1000, 1000, 0.1, 0.0, None),
    ("ls-128256-e0.1", 6, 128256, 128256, 0.1, 0.0, None),
]


def ls_inputs(T, V, Vp, shift, pad_fill, seed):
    lg, lab = ce_inputs(T, V, Vp, seed=seed)
    if shift:
        lg = (lg.float() + shift).to(torch.bfloat16)
        if T > 3:
            lab[3] = int(lg[3, :V].float().argmax())
    if pad_fill is not None and Vp > V:
        lg[:, V:] = pad_fill
    return lg, lab


def ls_row(name, T, V, Vp, eps, shift, pad_fill):
    lg, lab = ls_inputs(T, V, Vp, shift, pad_fill, seed=V)
    o = ls_ref(lg, lab, V, eps, scale=0.75)
    emu = ls_checks(emulate_ls(lg, lab, V, eps, scale=0.75), o)
    caught = {}
    for m in LS_MUTANTS:
        if m in ("eps_over_Vp", "pad_in_sum") and Vp == V:
            continue
        c = ls_checks(emulate_ls(lg, lab, V, eps, scale=0.75, mutant=m), o)
        caught[m] = max(c.items(), key=lambda kv: kv[1])
    return emu, caught


ROWS = {c[0]: (lambda c=c: ls_row(*c)) for c in LS_CASES}


@pytest.mark.parametrize("name", list(ROWS))
def test_margin_table_emulator_within_half(name):
    emu, _ = ROWS[name]()
    for k, r in emu.items():
        assert r < 0.5, (name, "emulator", k, r)


def test_every_mutant_lands_3x_outside_on_some_case():
    best = {m: 0.0 for m in LS_MUTANTS}
    for name, row in ROWS.items():
        _, caught = row()
        for m, (k, r) in caught.items():
            best[m] = max(best[m], r)
    assert all(r > 3.0 for r in best.values()), best


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


@pytest.mark.parametrize("make", [_tiny_llama, _tiny_gpt], ids=["llama", "gptneo"])
@pytest.mark.parametrize("eps", [0.1, 1.0])
def test_native_model_matches_label_smoother(make, eps):
    """``model.label_smoothing = eps`` with labels gives the loss and gradients of ``LabelSmoother`` on the model's logits (fp32)."""
    from acco_b200.utils.misc import LabelSmoother
    m = make().float()
    assert m.config.padded_vocab > m.config.vocab_size
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 90, (3, 16), generator=g)
    labels = ids.clone()
    labels[0, 10:] = -100
    labels[2, :] = -100
    m.label_smoothing = eps
    loss = m(input_ids=ids, labels=labels)[0]
    loss.backward()
    got = {k: p.grad.clone() for k, p in m.named_parameters()}
    m.zero_grad()
    m.label_smoothing = 0.0
    ref = LabelSmoother(eps)(m(input_ids=ids), labels, shift_labels=True)
    ref.backward()
    assert abs(float(loss.detach()) - float(ref.detach())) <= 2e-6 * abs(float(ref.detach()))
    for k, p in m.named_parameters():
        torch.testing.assert_close(got[k], p.grad, rtol=1e-4, atol=1e-6, msg=k)


def test_default_is_unsmoothed():
    m = _tiny_llama().float()
    assert m.label_smoothing == 0.0 and _tiny_gpt().label_smoothing == 0.0
    ids = torch.randint(0, 90, (2, 16), generator=torch.Generator().manual_seed(2))
    want = F.cross_entropy(m(input_ids=ids).logits[:, :-1].reshape(-1, 90), ids[:, 1:].reshape(-1))
    assert float(m(input_ids=ids, labels=ids)[0]) == pytest.approx(float(want), rel=1e-6)


def test_op_reference_path_smooths():
    from acco_b200 import ops
    lg, lab = ce_inputs(9, 37, 40, seed=6)
    got = ops.softmax_cross_entropy(lg.float(), lab, 37, -100, label_smoothing=0.2)
    want = F.cross_entropy(lg[:, :37].float(), lab, ignore_index=-100, label_smoothing=0.2)
    assert float(got) == float(want)


# ================================================================================================= trainer
class _Wrapped(torch.nn.Module):
    """A non-native model around the same weights: HF-style, logits only, so the trainer smooths it with ``LabelSmoother``."""

    def __init__(self, m):
        super().__init__()
        self.m = m

    def forward(self, input_ids=None, labels=None, attention_mask=None, **kw):
        return {"logits": self.m(input_ids=input_ids).logits}


def _trainer(model, eps, method="acco", sft=True, **kw):
    from acco_b200 import DecoupledTrainer
    from acco_b200.data import ByteTokenizer, synthetic_pretrain_dataset, synthetic_sft_dataset
    from acco_b200.launch import DistEnv
    from helpers import LOG, base_args
    if sft:
        ds = synthetic_sft_dataset(60, 10, 96, 16, seed=1)
        tok = ByteTokenizer()
        tok.pad_token_id = 95
        args = base_args(method_name=method, const_len_batch=False, nb_steps_tot=8, **kw)
    else:
        ds, tok = synthetic_pretrain_dataset(200, 30, 96, 16, seed=3), None
        args = base_args(method_name=method, nb_steps_tot=8, **kw)
    if eps is not None:
        args["label_smoothing_factor"] = eps
    return DecoupledTrainer(model=model, tokenizer=tok, train_dataset=ds, args=args, log=LOG, env=DistEnv(id_run="ls"))


def _trace(t):
    out = []
    while not t.finished():
        t.step()
        out.append(float(t.loss_host))
    return out


@pytest.mark.parametrize("method", ["acco", "dpu", "ddp"])
def test_trainer_fused_route_tracks_label_smoother_route(workdir, method):
    from helpers import tiny_model
    fused = _trainer(tiny_model(), 0.1, method)
    assert fused.label_smoother is None and fused.model.label_smoothing == 0.1
    fused.is_cuda = True                                  # graphs need a GPU; everything else about the route allows them
    assert fused._use_graphs()
    fused.is_cuda = False
    old = _trainer(_Wrapped(tiny_model()), 0.1, method)
    assert old.label_smoother is not None and not getattr(old.model, "label_smoothing", 0.0)
    a, b = _trace(fused), _trace(old)
    assert len(a) == len(b) >= 8
    for x, y in zip(a, b):
        assert abs(x - y) <= 1e-5 * abs(y), (a, b)
    unsmoothed = _trace(_trainer(tiny_model(), None, method))
    assert max(abs(x - y) for x, y in zip(a, unsmoothed)) > 1e-3       # the smoothing is really on


def test_trainer_batches_without_labels_stay_unsmoothed(workdir):
    """Pre-training batches carry no labels: both routes score them on their own tokens without smoothing."""
    from helpers import tiny_model
    t = _trainer(tiny_model(), 0.1, sft=False)
    assert t.label_smoother is None
    a = _trace(t)
    assert t.model.label_smoothing == 0.1
    b = _trace(_trainer(tiny_model(), None, sft=False))
    assert a == b


def test_trainer_eps_zero_is_the_run_without_the_key(workdir):
    from helpers import tiny_model
    t0, t1 = _trainer(tiny_model(), 0, "acco"), _trainer(tiny_model(), None, "acco")
    assert t0.label_smoother is None and t0.model.label_smoothing == 0.0
    assert _trace(t0) == _trace(t1)
    assert torch.equal(t0.get_weights(), t1.get_weights())


@pytest.mark.parametrize("eps", [-0.1, 1.5, math.nan, math.inf, True, "0.1"])
def test_trainer_rejects_bad_factor(workdir, eps):
    from helpers import tiny_model
    with pytest.raises(ValueError, match="label_smoothing_factor"):
        _trainer(tiny_model(), eps)


if __name__ == "__main__":               # print the margin table: python tests/test_label_smoothing.py
    for name, row in ROWS.items():
        emu, caught = row()
        print(f"{name:22s} emulator/bound " + " ".join(f"{k}={v:.3f}" for k, v in emu.items()))
        for m, (k, r) in caught.items():
            print(f"{'':22s}   mutant {m:15s} worst {k}: {r:.3g}x")
