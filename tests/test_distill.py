"""Knowledge distillation from a frozen teacher (``train.distill_teacher`` / ``DecoupledTrainer(teacher=...)``): the fp64 oracle of
the ``kd_*`` kernels and its per-element bounds, the margin table of a blockwise fp32 emulator and its mutants, and the op, model
and trainer routes.  Runs on the CPU without the extension; ``test_distill_gpu.py`` runs the kernels against the same oracle.

Semantics (student logits ``s``, teacher logits ``t``, temperature ``T``, weight ``a``; mean over the rows whose shifted label is
not -100; Hinton's forward KL with the teacher's entropy)::

    row  = (1 - a) (lse(s) - s[y])  +  a T^2 KL(softmax(t/T) || softmax(s/T))                        (ignored rows: 0)
    KL   = sum_c q_c (t_c/T - s_c/T) - lse(t/T) + lse(s/T),   q = softmax(t/T)
    ds_c = scale ((1 - a) (softmax(s)_c - [c = y]) + a T (softmax(s/T)_c - q_c))           (c < V; padding, ignored rows: 0)
    out  = (mean CE, mean KL)

Bounds (``E`` of the unsmoothed CE oracle for each of the three ``lse``, the inputs scaled by ``1/T`` rounded once more):

* ``sum q (u - w)`` as ``K / S``: the running sum ``K`` has the depth of ``S`` plus one product and one difference per term, so
  ``E = (2 rel_S + 3 U) sum q |u - w| + U |K / S|``; the KL adds ``E_lse(t/T) + E_lse(s/T)`` and two roundings.
* The objective: ``(1 - a)`` times the CE mean's bound plus ``a T^2`` times the KL mean's, plus four roundings.
* The gradient: ``(1 - a) E_p + a T (E_ps + E_q)`` with each softmax's bound as in the CE oracle, three roundings of every term,
  then the scale; a bf16 output gets one bf16 ulp on top.  Everything is doubled, as elsewhere.

The margin table asserts the emulator stays within half of every bound and that each mutant (``T^2`` missing, reverse KL,
untempered teacher, padding column included, ignored row counted) lands more than 3x outside on some case.  Print it with
``python tests/test_distill.py``."""
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
from test_rowwise_oracle import E_LG2, FTZ, U, ULP, ce_inputs, ce_loss_bound, e_exp, f32, out_bound, ratio  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ================================================================================================= fp64 oracle
def formula(s: torch.Tensor, t: torch.Tensor, labels: torch.Tensor, a: float, T: float, ignore_index: int = -100) -> torch.Tensor:
    """The objective as torch autograd sees it: ``(1-a) F.cross_entropy + a T^2 F.kl_div(log_softmax(s/T), log_softmax(t/T),
    log_target=True)`` over the non-ignored rows."""
    valid = labels != ignore_index
    ce = F.cross_entropy(s, labels, ignore_index=ignore_index)
    kl = F.kl_div(torch.log_softmax(s[valid] / T, -1), torch.log_softmax(t[valid] / T, -1), reduction="batchmean", log_target=True)
    return (1 - a) * ce + a * T * T * kl


def _lse_bound(x: torch.Tensor, lse: torch.Tensor, V: int, scaled: bool) -> torch.Tensor:
    """Absolute error of the kernel's online ``lse`` over ``x`` [T, V] (``ce_ref``'s terms; ``scaled``: x was rounded once more)."""
    n_sw = -(-(V // 8) // 512) + 1
    R = x.max(1).values - x.min(1).values
    gs = torch.exp(lse - x.max(1).values)
    rel_gs = (10 * n_sw + 12) * U + (n_sw + 2) * e_exp(R)
    E = rel_gs + E_LG2 + 3 * ULP * torch.log(gs).abs() + U * lse.abs()
    if scaled:
        E = E + 2 * U * x.abs().max(1).values
    return E, rel_gs


def kd_ref(s, t, labels, V: int, a: float, T: float, ignore_index: int = -100, scale: Optional[float] = None):
    """fp64 oracle of the ``kd_*`` kernels: the three ``lse`` (0 on ignored rows), row CE and KL, the objective, ``inv_n``, the
    means, and with ``scale`` the d-logits.  Bounds included."""
    Tn, Vp = s.shape
    x = s[:, :V].double()
    y = t[:, :V].double()
    labels = labels.to(x.device)
    valid = labels != ignore_index
    lab = torch.where(valid, labels, torch.zeros_like(labels))
    w, u = x / T, y / T
    lse1, lse2, lset = torch.logsumexp(x, 1), torch.logsumexp(w, 1), torch.logsumexp(u, 1)
    q = torch.exp(u - lset[:, None])
    kq = (q * (u - w)).sum(1)
    z = torch.zeros_like(lse1)
    ce = torch.where(valid, lse1 - x.gather(1, lab[:, None])[:, 0], z)
    kl = torch.where(valid, kq - lset + lse2, z)
    E1, _ = _lse_bound(x, lse1, V, False)
    E2, _ = _lse_bound(w, lse2, V, T != 1)
    Et, rel_t = _lse_bound(u, lset, V, T != 1)
    A = (q * (u - w).abs()).sum(1)
    E_ce = torch.where(valid, E1 + U * ce.abs(), z)
    E_kl = torch.where(valid, (2 * rel_t + 3 * U) * A + U * kq.abs() + Et + E2 + U * ((kq - lset).abs() + kl.abs()), z)
    n = int(valid.sum())
    inv = 1.0 / n if n else 0.0
    ce_m, kl_m = float(ce.sum()) * inv, float(kl.sum()) * inv
    b_ce = ce_loss_bound(float(E_ce.sum()), float(ce.abs().sum()), Tn, ce_m, inv)
    b_kl = ce_loss_bound(float(E_kl.sum()), float(kl.abs().sum()), Tn, kl_m, inv)
    loss = (1 - a) * ce_m + a * T * T * kl_m
    b_loss = (1 - a) * b_ce + a * T * T * b_kl + 8 * U * ((1 - a) * abs(ce_m) + a * T * T * abs(kl_m)) + FTZ
    zr = torch.zeros_like(lse1)
    res = {"lse": torch.stack([torch.where(valid, lse1, zr), torch.where(valid, lse2, zr), torch.where(valid, lset, zr)]),
           "b_lse": torch.stack([2 * torch.where(valid, E1, zr), 2 * torch.where(valid, E2, zr), 2 * torch.where(valid, Et, zr)]) + FTZ,
           "ce_row": ce, "kl_row": kl, "b_kl_row": 2 * E_kl + FTZ, "loss": loss, "b_loss": b_loss, "inv_n": inv,
           "b_inv": 2 * 2.0 ** -22 * inv, "ce": ce_m, "b_ce": b_ce, "kl": kl_m, "b_kl": b_kl}
    if scale is not None:
        p, ps = torch.exp(x - lse1[:, None]), torch.exp(w - lse2[:, None])
        oh = torch.zeros_like(p)
        oh.scatter_(1, lab[:, None], 1.0)
        d0 = (1 - a) * (p - oh) + a * T * (ps - q)
        gq = d0 * scale
        E_p = p * (E1[:, None] + U * (x - lse1[:, None]).abs() + e_exp(x - lse1[:, None]))
        E_ps = ps * (E2[:, None] + U * (w - lse2[:, None]).abs() + e_exp(w - lse2[:, None]) + 2 * U * w.abs())
        E_q = q * (Et[:, None] + U * (u - lset[:, None]).abs() + e_exp(u - lset[:, None]) + 2 * U * u.abs())
        E_d = (1 - a) * E_p + a * T * (E_ps + E_q) + 3 * U * ((1 - a) * (p + oh) + a * T * (ps + q))
        E = 2 * (abs(scale) * E_d + U * gq.abs())
        grad = torch.zeros(Tn, Vp, dtype=torch.float64)
        bnd = torch.full((Tn, Vp), FTZ, dtype=torch.float64)
        grad[:, :V] = torch.where(valid[:, None], gq, torch.zeros_like(gq))
        bnd[:, :V] = torch.where(valid[:, None], out_bound(gq, E, FTZ * (1 + abs(scale) * (1 + a * T))), torch.full_like(gq, FTZ))
        res.update(grad=grad, b_grad=bnd)
    return res


def kd_checks(got, o) -> Dict[str, float]:
    out = {"lse": ratio(got["lse"], o["lse"], o["b_lse"]),
           "loss": abs(float(got["loss"]) - o["loss"]) / o["b_loss"],
           "ce": abs(float(got["ce"]) - o["ce"]) / o["b_ce"],
           "kl": abs(float(got["kl"]) - o["kl"]) / o["b_kl"],
           "inv_n": abs(float(got["inv_n"]) - o["inv_n"]) / max(o["b_inv"], FTZ)}
    if "grad" in got:
        out["grad"] = ratio(got["grad"], o["grad"], o["b_grad"])
    return out


# ================================================================================================= emulator
KD_MUTANTS = ("no_T2", "reverse_kl", "untempered_teacher", "padding_included", "ignored_counted")


def _bsum32(part: torch.Tensor) -> torch.Tensor:
    """``block_sum`` over 512 threads: xor butterflies in each warp, then over the 16 warp sums."""
    Tn = part.shape[0]
    v = part.reshape(Tn, 16, 32)
    for o in (16, 8, 4, 2, 1):
        v = f32(v + v[..., torch.arange(32) ^ o])
    w = torch.zeros(Tn, 32, dtype=torch.float64)
    w[:, :16] = v[..., 0]
    for o in (16, 8, 4, 2, 1):
        w = f32(w + w[:, torch.arange(32) ^ o])
    return w[:, 0]


def _ex(a):
    return f32(torch.exp(a))


def emulate_kd(s, t, labels, V: int, a: float, T: float, ignore_index: int = -100, scale: float = 1.0, mutant=None):
    """fp32 emulator of ``kd_fwd_kernel`` (512 threads, online max / sum of s, s/T and t/T plus the running K over 8-wide vectors,
    scalar ragged tail, block reductions), ``kd_reduce_kernel`` and ``kd_bwd_kernel``."""
    Tn, Vp = s.shape
    Vs = Vp if mutant == "padding_included" else V
    Tt = 1.0 if mutant == "untempered_teacher" else T
    inv_t, inv_tt = float(f32(torch.tensor(1.0 / T))), float(f32(torch.tensor(1.0 / Tt)))
    x, y = s.double(), t.double()
    nvf = Vs // 8
    K = -(-nvf // 512)

    def vec(z):
        zv = torch.full((Tn, K * 512 * 8), -math.inf, dtype=torch.float64)
        zv[:, :nvf * 8] = z[:, :nvf * 8]
        return zv.view(Tn, K, 512, 8)

    xv, yv = vec(x), vec(y)
    st = {k: (torch.full((Tn, 512), -math.inf, dtype=torch.float64), torch.zeros(Tn, 512, dtype=torch.float64)) for k in (1, 2, 3)}
    k3 = torch.zeros(Tn, 512, dtype=torch.float64)

    def online(m, sm, f):                    # f [Tn, 512, 8] -> new (m, s); dead lanes (-inf) keep theirs
        live = torch.isfinite(f[..., 0])
        nm = torch.maximum(m, f.max(-1).values)
        acc = torch.zeros_like(sm)
        for j in range(8):
            acc = f32(acc + _ex(f32(f[..., j] - nm)))
        r = torch.where(torch.isfinite(m), _ex(f32(m - nm)), torch.zeros_like(m))
        return torch.where(live, nm, m), torch.where(live, f32(f32(sm * r) + acc), sm), nm, r, live

    for k in range(K):
        f, g = xv[:, k], yv[:, k]
        st[1] = online(*st[1], f)[:2]
        fs, gs = f32(f * inv_t), f32(g * inv_tt)
        st[2] = online(*st[2], fs)[:2] if T != 1 else st[1]
        m3o = st[3][0]
        m3, s3, nm, r, live = online(*st[3], gs)
        acck = torch.zeros_like(k3)
        for j in range(8):
            e = _ex(f32(gs[..., j] - nm))
            acck = f32(acck + f32(e * torch.nan_to_num(f32(gs[..., j] - fs[..., j]), nan=0.0)))
        k3 = torch.where(live, f32(f32(k3 * r) + acck), k3)
        st[3] = (m3, s3)
        del m3o
    for c in range(nvf * 8, Vs):
        i = c - nvf * 8
        fc, gc = x[:, c], y[:, c]
        fcs, gcs = f32(fc * inv_t), f32(gc * inv_tt)
        for key, val in ((1, fc), (2, fcs), (3, gcs)):
            if key == 2 and T == 1:
                continue
            m, sm = st[key]
            nm = torch.maximum(m[:, i], val)
            r = torch.where(torch.isfinite(m[:, i]), _ex(f32(m[:, i] - nm)), torch.zeros_like(nm))
            e = _ex(f32(val - nm))
            sm[:, i] = f32(f32(sm[:, i] * r) + e)
            if key == 3:
                k3[:, i] = f32(f32(k3[:, i] * r) + f32(e * f32(gcs - fcs)))
            m[:, i] = nm
        if T == 1:
            st[2] = st[1]

    def lse_of(m, sm):
        gm = m.max(1).values
        w = torch.where(torch.isfinite(m), _ex(f32(m - gm[:, None])), torch.zeros_like(m))
        return gm, w, f32(gm + f32(torch.log(_bsum32(f32(sm * w)))))

    lse1 = lse_of(*st[1])[2]
    lse2 = lse_of(*st[2])[2]
    gm3, w3, lset = lse_of(*st[3])
    gs3, gk3 = _bsum32(f32(st[3][1] * w3)), _bsum32(f32(k3 * w3))
    kq = f32(gk3 / gs3)
    kl = f32(f32(kq - lset) + lse2)
    if mutant == "reverse_kl":               # KL(student || teacher) = sum p_s (w - u) - lse(s/T) + lse(t/T), computed in fp64
        wv, uv = f32(x[:, :V] * inv_t), f32(y[:, :V] * inv_t)
        ps = torch.softmax(wv, 1)
        kl = f32((ps * (wv - uv)).sum(1) - torch.logsumexp(wv, 1) + torch.logsumexp(uv, 1))
    valid = labels != ignore_index
    lab = torch.where(valid, labels, torch.zeros_like(labels))
    ce = f32(lse1 - x.gather(1, lab[:, None])[:, 0])
    counted = torch.ones_like(valid) if mutant == "ignored_counted" else valid
    z = torch.zeros_like(ce)
    ce = torch.where(valid, ce, z)
    kl = torch.where(counted, kl, z)
    sc = sk = torch.tensor(0.0, dtype=torch.float64)
    for i in range(Tn):
        if counted[i]:
            sc, sk = f32(sc + ce[i]), f32(sk + kl[i])
    n = int(counted.sum())
    inv = float(f32(torch.tensor(1.0 / n))) if n else 0.0
    ce_m, kl_m = float(f32(sc * inv)), float(f32(sk * inv))
    one_m_a = float(f32(torch.tensor(1.0 - a)))
    a_t2 = float(f32(torch.tensor(a * (1.0 if mutant == "no_T2" else T * T))))
    a_t = float(f32(torch.tensor(a * (1.0 / T if mutant == "no_T2" else T))))
    loss = float(f32(f32(torch.tensor(one_m_a * ce_m)) + f32(torch.tensor(a_t2 * kl_m))))
    zr = torch.zeros_like(lse1)
    lse_out = torch.stack([torch.where(valid, lse1, zr), torch.where(valid, lse2, zr), torch.where(valid, lset, zr)])
    # backward
    cols = torch.arange(Vp)
    live = cols[None, :] < Vs
    xs = torch.nan_to_num(x, nan=0.0)
    p = torch.where(live, _ex(f32(xs - lse1[:, None])), torch.zeros_like(x))
    ps = torch.where(live, _ex(f32(f32(xs * inv_t) - lse2[:, None])), torch.zeros_like(x))
    qv = torch.where(live, _ex(f32(f32(torch.nan_to_num(y, nan=0.0) * inv_tt) - lset[:, None])), torch.zeros_like(x))
    if mutant == "reverse_kl":               # d/dw of T^2 KL(p_s || q) / T = T p_s ((w - lse_s) - (u - lse_t) - KL)
        wv, uv = f32(xs * inv_t), f32(torch.nan_to_num(y, nan=0.0) * inv_t)
        dk = f32(ps * ((wv - lse2[:, None]) - (uv - lset[:, None]) - kl[:, None]))
    else:
        dk = f32(ps - qv)
    d = f32(f32(one_m_a * p) + f32(a_t * dk))
    d = torch.where(cols[None, :] == lab[:, None], f32(d - one_m_a), d)
    d = torch.where(live, d, torch.zeros_like(d))
    grad = bf16_rn(f32(d * scale)).double()
    if mutant == "ignored_counted":          # ignored rows keep the KL part of their gradient
        gk = bf16_rn(f32(f32(a_t * dk) * scale)).double()
        grad = torch.where(valid[:, None], grad, torch.where(live, gk, torch.zeros_like(gk)))
    else:
        grad = torch.where(valid[:, None], grad, torch.zeros_like(grad))
    return {"lse": lse_out, "loss": loss, "ce": ce_m, "kl": kl_m, "inv_n": inv, "grad": grad, "kl_row": kl}


def kd_inputs(Tn: int, V: int, Vp: int, seed: int, pad_fill: Optional[float] = None, same_row: bool = True):
    """Student logits as ``ce_inputs`` (ignored rows, a wide row, a flat row); the teacher a sharper, noisy copy, one row equal to the
    student's; with ``pad_fill`` both padding regions hold that value."""
    s, lab = ce_inputs(Tn, V, Vp, seed=seed, pad_fill=pad_fill)
    g = torch.Generator().manual_seed(seed + 1)
    t = (1.5 * s.float() + torch.randn(Tn, Vp, generator=g)).to(torch.bfloat16)
    if same_row and Tn > 5:
        t[5] = s[5]
    if pad_fill is not None and Vp > V:
        t[:, V:] = pad_fill
    return s, t, lab


# ================================================================================================= oracle vs autograd
@pytest.mark.parametrize("a", [0.25, 1.0])
@pytest.mark.parametrize("T", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("V,Vp", [(37, 40), (40, 40), (1003, 1008)], ids=["ragged-padded", "exact", "ragged-1003"])
def test_oracle_matches_fp64_autograd(a, T, V, Vp):
    """Ignored rows (every 5th), padding columns, a ragged V, against autograd of the torch formula in fp64."""
    s, t, lab = kd_inputs(12, V, Vp, seed=V, pad_fill=30.0)
    n = int((lab != -100).sum())
    o = kd_ref(s, t, lab, V, a, T, scale=2.5 / n)                      # the kernel's scale is dloss * inv_n
    xr = s[:, :V].double().requires_grad_(True)
    loss = formula(xr, t[:, :V].double(), lab, a, T)
    (loss * 2.5).backward()
    assert abs(o["loss"] - float(loss.detach())) < 1e-12 * max(1.0, abs(o["loss"]))
    torch.testing.assert_close(o["grad"][:, :V], xr.grad, rtol=1e-12, atol=1e-12)
    assert bool((o["grad"][:, V:] == 0).all()) and bool((o["grad"][lab == -100] == 0).all())
    assert abs(o["ce"] - float(F.cross_entropy(s[:, :V].double(), lab))) < 1e-12 * o["ce"]
    assert o["kl"] > 0 and bool((o["kl_row"] >= -1e-12).all())


@pytest.mark.parametrize("T", [0.5, 1.0, 2.0])
def test_teacher_equal_to_student_gives_kl_0_and_the_scaled_ce_gradient(T):
    s, _, lab = kd_inputs(10, 131, 136, seed=3)
    o = kd_ref(s, s, lab, 131, 0.25, T, scale=1.0)
    c = kd_ref(s, s, lab, 131, 0.0, T, scale=1.0)                       # a = 0: the plain CE and its gradient
    assert abs(o["kl"]) < 1e-12 and float(o["kl_row"].abs().max()) < 1e-12
    torch.testing.assert_close(o["grad"], 0.75 * c["grad"], rtol=1e-12, atol=1e-15)
    assert o["loss"] == pytest.approx(0.75 * c["ce"], rel=1e-12)
    e = emulate_kd(s, s, lab, 131, 0.25, T)
    assert e["kl"] == 0.0 and bool((e["kl_row"] == 0).all())          # the kernel computes both sides with the same operations
    from acco_b200 import ops
    out = torch.zeros(2)
    ops.distill_cross_entropy(s.float(), s.float(), lab, 131, 0.25, T, out=out)
    assert abs(float(out[1])) < 1e-6


def test_all_ignored_batch_has_zero_loss_and_gradient():
    s, t, lab = kd_inputs(8, 50, 56, seed=4)
    lab[:] = -100
    o = kd_ref(s, t, lab, 50, 0.5, 2.0, scale=1.0)
    assert o["loss"] == 0.0 and o["ce"] == 0.0 and o["kl"] == 0.0 and o["inv_n"] == 0.0 and bool((o["grad"] == 0).all())
    e = emulate_kd(s, t, lab, 50, 0.5, 2.0)
    assert e["loss"] == 0.0 and e["inv_n"] == 0.0 and bool((e["grad"] == 0).all())
    from acco_b200 import ops
    x = s.float().requires_grad_(True)
    loss = ops.distill_cross_entropy(x, t.float(), lab, 50, 0.5, 2.0)
    loss.backward()
    assert float(loss) == 0.0 and bool((x.grad == 0).all())


# ================================================================================================= margin table
KD_CASES = [
    # (name, rows, V, Vp, a, T, padding fill)
    ("kd-50257-T1", 6, 50257, 50304, 0.5, 1.0, None),
    ("kd-50257-T2-pad", 6, 50257, 50304, 0.5, 2.0, 30.0),
    ("kd-131-T0.5-pad", 12, 131, 136, 0.25, 0.5, 30.0),
    ("kd-131-T2-a1", 12, 131, 136, 1.0, 2.0, None),
    ("kd-1003-T2-pad", 12, 1003, 1008, 0.25, 2.0, 20.0),
    ("kd-1000-T1-a1", 12, 1000, 1008, 1.0, 1.0, 30.0),
    ("kd-128256-T2", 6, 128256, 128256, 0.5, 2.0, None),
]


def kd_row(name, Tn, V, Vp, a, T, pad_fill):
    s, t, lab = kd_inputs(Tn, V, Vp, seed=V, pad_fill=pad_fill)
    o = kd_ref(s, t, lab, V, a, T, scale=0.75)
    emu = kd_checks(emulate_kd(s, t, lab, V, a, T, scale=0.75), o)
    caught = {}
    for m in KD_MUTANTS:
        if (m == "padding_included" and Vp == V) or (m in ("no_T2", "untempered_teacher") and T == 1):
            continue
        c = kd_checks(emulate_kd(s, t, lab, V, a, T, scale=0.75, mutant=m), o)
        caught[m] = max(c.items(), key=lambda kv: kv[1])
    return emu, caught


ROWS = {c[0]: functools.lru_cache(maxsize=None)(lambda c=c: kd_row(*c)) for c in KD_CASES}     # both tests read one evaluation


@pytest.mark.parametrize("name", list(ROWS))
def test_margin_table_emulator_within_half(name):
    emu, _ = ROWS[name]()
    for k, r in emu.items():
        assert r < 0.5, (name, "emulator", k, r)


def test_every_mutant_lands_3x_outside_on_some_case():
    best = {m: 0.0 for m in KD_MUTANTS}
    for name, row in ROWS.items():
        _, caught = row()
        for m, (k, r) in caught.items():
            best[m] = max(best[m], r)
    assert all(r > 3.0 for r in best.values()), best


# ================================================================================================= op reference path
def test_op_reference_path_matches_the_formula_and_writes_out():
    from acco_b200 import ops
    s, t, lab = kd_inputs(9, 37, 40, seed=6, pad_fill=5.0)
    out = torch.full((2,), -1.0)
    x = s.float().requires_grad_(True)
    tt = t.float()
    got = ops.distill_cross_entropy(x, tt, lab, 37, 0.25, 2.0, out=out)
    got.backward()
    xr = s[:, :37].float().requires_grad_(True)
    ref = formula(xr, t[:, :37].float(), lab, 0.25, 2.0)
    ref.backward()
    assert float(got) == pytest.approx(float(ref), rel=1e-6)
    torch.testing.assert_close(x.grad[:, :37], xr.grad, rtol=1e-5, atol=1e-7)
    assert bool((x.grad[:, 37:] == 0).all())
    assert float(out[0]) == pytest.approx(float(F.cross_entropy(s[:, :37].float(), lab)), rel=1e-6)
    assert float(got) == pytest.approx(0.75 * float(out[0]) + 0.25 * 4 * float(out[1]), rel=1e-6)
    assert torch.equal(tt, t.float())                                  # the teacher logits are never written
    for bad in (0.0, -0.5, 1.5, math.nan, True):
        with pytest.raises(ValueError, match="alpha"):
            ops.distill_cross_entropy(s.float(), tt, lab, 37, bad, 1.0)
    for bad in (0.0, -1.0, math.inf, math.nan):
        with pytest.raises(ValueError, match="temperature"):
            ops.distill_cross_entropy(s.float(), tt, lab, 37, 0.5, bad)
    with pytest.raises(ValueError, match="teacher_logits"):
        ops.distill_cross_entropy(s.float(), tt[:, :36], lab, 37, 0.5, 1.0)


# ================================================================================================= models
def _tiny_llama(seed=0, layers=2):
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(seed)
    return LlamaForCausalLM(LlamaConfig(vocab_size=90, hidden_size=32, intermediate_size=48, num_hidden_layers=layers, num_attention_heads=4,
                                        num_key_value_heads=2, max_position_embeddings=32, pad_vocab_multiple=8))


def _tiny_gpt(seed=0):
    from acco_b200.models import GPTConfig, GPTForCausalLM
    torch.manual_seed(seed)
    return GPTForCausalLM(GPTConfig(vocab_size=90, hidden_size=32, num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=32,
                                    attention_layers=["global", "local"], window_size=8, pad_vocab_multiple=8))


@pytest.mark.parametrize("make", [_tiny_llama, _tiny_gpt], ids=["llama-gqa", "gptneo"])
@pytest.mark.parametrize("T", [1.0, 2.0])
def test_native_model_matches_the_formula(make, T):
    """``teacher_logits`` (a teacher's padded logits) with labels gives the loss and gradients of the formula on the model's own
    logits (fp32); the teacher gets no gradient."""
    m, teacher = make(0).float(), _tiny_llama(seed=5, layers=1).float()
    teacher.requires_grad_(False)
    assert m.config.padded_vocab > m.config.vocab_size
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 90, (3, 16), generator=g)
    labels = ids.clone()
    labels[0, 10:] = -100
    labels[2, :] = -100
    m.distill_alpha, m.distill_temperature, m.distill_out = 0.25, T, torch.zeros(2)
    with torch.no_grad():
        tl = teacher.padded_logits(ids)
    assert tl.shape == (48, m.config.padded_vocab)
    loss = m(input_ids=ids, labels=labels, teacher_logits=tl)[0]
    loss.backward()
    got = {k: p.grad.clone() for k, p in m.named_parameters()}
    m.zero_grad()
    logits = m(input_ids=ids).logits[:, :-1].reshape(-1, 90)
    tgt = labels[:, 1:].reshape(-1)
    tv = tl.view(3, 16, -1)[:, :-1, :90].reshape(-1, 90)
    ref = formula(logits, tv, tgt, 0.25, T)
    ref.backward()
    assert abs(float(loss.detach()) - float(ref.detach())) <= 2e-6 * abs(float(ref.detach()))
    assert float(m.distill_out[0]) == pytest.approx(float(F.cross_entropy(logits.detach(), tgt)), rel=2e-6)
    for k, p in m.named_parameters():
        torch.testing.assert_close(got[k], p.grad, rtol=1e-4, atol=1e-6, msg=k)
    assert all(p.grad is None for p in teacher.parameters())
    with pytest.raises(ValueError, match="labels"):
        m(input_ids=ids, teacher_logits=tl)


# ================================================================================================= trainer
class _KDRef(torch.nn.Module):
    """A non-native model around the student's weights whose loss is the formula in plain torch, with the teacher outside its
    parameters: the reference the trainer is checked against."""

    def __init__(self, m, teacher, a, T):
        super().__init__()
        self.m, self._t, self.a, self.T = m, [teacher], a, T

    def forward(self, input_ids=None, labels=None, position_ids=None, **kw):
        logits = self.m(input_ids=input_ids, position_ids=position_ids).logits
        with torch.no_grad():
            tl = self._t[0](input_ids=input_ids, position_ids=position_ids).logits
        V = logits.shape[-1]
        tgt = labels[:, 1:].reshape(-1)
        return (formula(logits[:, :-1].reshape(-1, V).float(), tl[:, :-1].reshape(-1, V).float(), tgt, self.a, self.T),)


def _trainer(model, teacher=None, method="acco", **kw):
    from acco_b200 import DecoupledTrainer
    from acco_b200.data import synthetic_pretrain_dataset
    from acco_b200.launch import DistEnv
    from helpers import LOG, base_args
    ds = synthetic_pretrain_dataset(200, 30, 96, 16, seed=3)
    args = base_args(method_name=method, **{"nb_steps_tot": 8, **kw})
    return DecoupledTrainer(model=model, train_dataset=ds, eval_dataset=ds, args=args, log=LOG, env=DistEnv(id_run="kd"), teacher=teacher)


def _teacher(seed=9):
    from helpers import tiny_model
    return tiny_model(seed=seed, layers=1)


class _Recorder:
    def __init__(self):
        self.logs = []

    def __getattr__(self, name):
        return lambda *a: None

    def on_log(self, trainer, scalars):
        self.logs.append(dict(scalars))


def _logged(t):
    rec = _Recorder()
    t.add_callback(rec)
    t.train()
    return rec.logs


@pytest.mark.parametrize("method,impl", [("acco", "native"), ("dpu", "native"), ("ddp", "native"), ("ddp", "torch")])
def test_trainers_track_the_torch_reference(workdir, method, impl):
    from helpers import tiny_model
    kw = dict(ddp_impl=impl, log_every=1, nb_steps_tot=16, distill_alpha=0.5, distill_temperature=2.0)
    t = _trainer(tiny_model(), _teacher(), method, **kw)
    assert t.model.distill_out is t.distill_static and t.model.distill_temperature == 2.0
    t.is_cuda = True                                       # graphs need a GPU; everything else about the route allows them
    assert t._use_graphs()
    t.is_cuda = False
    ref = _trainer(_KDRef(tiny_model(), _teacher(), 0.5, 2.0), None, method, **kw)
    a, b = _logged(t), _logged(ref)
    assert len(a) == len(b) >= 4
    for x, y in zip(a, b):
        assert abs(x["loss"] - y["loss"]) <= 1e-5 * abs(y["loss"]), (a, b)
        assert x["loss"] == pytest.approx(0.5 * x["distill_ce"] + 0.5 * 4 * x["distill_kl"], rel=1e-5)
        assert x["distill_kl"] > 0 and "distill_kl" not in y
    plain = _logged(_trainer(tiny_model(), None, method, ddp_impl=impl, log_every=1, nb_steps_tot=16))
    assert max(abs(x["loss"] - y["loss"]) for x, y in zip(a, plain)) > 1e-2       # the term is really on
    assert all(not p.requires_grad for p in t.teacher.parameters())


def test_packed_rows_use_the_same_positions_for_the_teacher(workdir):
    """A micro-batch with ``position_ids`` (packed or document-masked rows) runs the teacher on the student's positions, so both
    models mask the same documents: the objective equals the formula on both models' logits for those positions."""
    from helpers import tiny_model
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(9)
    teacher = LlamaForCausalLM(LlamaConfig(vocab_size=96, hidden_size=32, intermediate_size=48, num_hidden_layers=1, num_attention_heads=4,
                                           max_position_embeddings=32, pad_vocab_multiple=8, initializer_range=0.5))   # position-sensitive
    t = _trainer(tiny_model(), teacher, "acco", distill_alpha=1.0, distill_temperature=0.5)        # the KL alone
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(0, 96, (2, 16), generator=g)
    pos = torch.cat([torch.arange(7), torch.arange(9)]).repeat(2, 1)            # two documents per row
    labels = ids.clone()
    labels[:, 7] = -100                                                         # the second document's first token is no target
    inputs = {"input_ids": ids, "labels": labels, "position_ids": pos}
    got = float(t._forward_loss(t.model, inputs, t.teacher))
    with torch.no_grad():
        s = t.model(input_ids=ids, position_ids=pos).logits[:, :-1].reshape(-1, 96)
        want = {}
        for name, tp in (("same", pos), ("arange", None)):
            tl = t.teacher(input_ids=ids, position_ids=tp).logits[:, :-1].reshape(-1, 96)
            want[name] = float(formula(s, tl, labels[:, 1:].reshape(-1), 1.0, 0.5))
    assert got == pytest.approx(want["same"], rel=1e-6)
    assert abs(want["arange"] - want["same"]) > 1e-2 * abs(want["same"])       # the positions matter to the teacher


def _worker(rank, world, port, tmp, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(CUDA_VISIBLE_DEVICES="", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    os.chdir(tmp)
    torch.set_num_threads(2)
    from acco_b200 import DecoupledTrainer
    from acco_b200.data import synthetic_pretrain_dataset
    from acco_b200.launch import shutdown_distributed
    from helpers import LOG, base_args, tiny_model
    ds = synthetic_pretrain_dataset(300, 30, 96, 16, seed=7)
    args = base_args(method_name="acco", nb_steps_tot=16, batch_size=2, distill_alpha=0.5, distill_temperature=2.0)
    t = DecoupledTrainer(model=tiny_model(seed=rank), train_dataset=ds, args=args, log=LOG, teacher=tiny_model(seed=9, layers=1))
    kls = []
    while not t.finished():
        t.step()
        kls.append(float(t.distill_host[1]))
    t._drain()
    t._finish("")
    q.put((rank, float(t.params.double().sum()), kls, sum(p.numel() for p in t.teacher.parameters()), t.len_params))
    shutdown_distributed()


def test_two_gloo_ranks_train_with_a_teacher(workdir):
    import tempfile
    import torch.multiprocessing as mp
    from acco_b200.launch import free_port
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    with tempfile.TemporaryDirectory() as tmp:
        procs = [ctx.Process(target=_worker, args=(r, 2, port, tmp, q)) for r in range(2)]
        for p in procs:
            p.start()
        out = sorted(q.get(timeout=240) for _ in procs)
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    (_, w0, k0, nt, n_student), (_, w1, k1, _, _) = out
    assert w0 == w1                                        # the ranks end on the same weights
    assert all(k > 0 for k in k0 + k1)
    from helpers import tiny_model
    assert n_student == sum(p.numel() for p in tiny_model().parameters()) and nt > 0     # the arena holds the student only


def test_the_rejections(workdir):
    from helpers import tiny_model
    from acco_b200.models import GPTConfig, GPTForCausalLM
    with pytest.raises(ValueError, match="not both"):
        _trainer(tiny_model(), _teacher(), distill_teacher="/nonexistent")
    for bad in (0, 0.0, -0.1, 1.5, math.nan, True, "0.5"):
        with pytest.raises(ValueError, match="distill_alpha"):
            _trainer(tiny_model(), _teacher(), distill_alpha=bad)
    for bad in (0, -1.0, math.inf, math.nan, False, "2"):
        with pytest.raises(ValueError, match="distill_temperature"):
            _trainer(tiny_model(), _teacher(), distill_temperature=bad)
    with pytest.raises(ValueError, match="native student"):
        _trainer(_KDRef(tiny_model(), _teacher(), 0.5, 1.0), _teacher())
    with pytest.raises(ValueError, match="native model"):
        _trainer(tiny_model(), _KDRef(_teacher(), _teacher(), 0.5, 1.0))
    with pytest.raises(ValueError, match="vocabularies differ"):
        _trainer(tiny_model(), tiny_model(vocab=90))
    gpt = GPTForCausalLM(GPTConfig(vocab_size=96, hidden_size=32, num_hidden_layers=1, num_attention_heads=4, max_position_embeddings=32,
                                   pad_vocab_multiple=8))
    assert _trainer(tiny_model(), gpt).teacher is gpt                  # any native teacher with the student's vocabulary
    with pytest.raises(ValueError, match="label_smoothing_factor"):
        _trainer(tiny_model(), _teacher(), label_smoothing_factor=0.1)
    with pytest.raises(ValueError, match="z_loss_weight"):
        _trainer(tiny_model(), _teacher(), z_loss_weight=1e-4)
    m = tiny_model()
    with pytest.raises(ValueError, match="separate model"):
        _trainer(m, m)
    assert _trainer(_KDRef(tiny_model(), _teacher(), 0.5, 1.0), None).teacher is None     # off is accepted with any model


def test_eval_is_pure_ce_and_the_teacher_stays_out_of_the_arena_and_checkpoint(workdir):
    from helpers import tiny_model
    from acco_b200.models import from_pretrained
    on, off = _trainer(tiny_model(), _teacher(), max_eval_batches=3), _trainer(tiny_model(), None, max_eval_batches=3)
    assert float(on.eval_loop()) == float(off.eval_loop())
    assert float(on.distill_static.abs().sum()) == 0.0                # eval wrote nothing
    student_ids = {id(p) for p in on.model.parameters()}
    assert not any(id(p) in student_ids for p in on.teacher.parameters())
    assert on.len_params == off.len_params == sum(p.numel() for p in on.model.parameters())
    assert not any(isinstance(mod, type(on.teacher)) and mod is on.teacher for mod in on.model.modules())
    on.train()
    assert float(on.distill_static[1]) > 0.0
    assert set(on.model.state_dict()) == set(off.model.state_dict())
    d = os.path.join(os.getcwd(), "ck")
    on.save_checkpoint(os.path.join(d, "student.pt"))
    saved = torch.load(os.path.join(d, "student.pt"), map_location="cpu", weights_only=False)
    flat = json.dumps(sorted(_keys(saved)))
    assert "teacher" not in flat
    assert sum(v.numel() for v in _tensors(saved)) == sum(v.numel() for v in off.model.state_dict().values())   # the student alone


def _keys(obj, prefix=""):
    if isinstance(obj, dict):
        for k, v in obj.items():
            yield f"{prefix}{k}"
            yield from _keys(v, f"{prefix}{k}.")


def _tensors(obj):
    if isinstance(obj, torch.Tensor):
        yield obj
    elif isinstance(obj, dict):
        for v in obj.values():
            yield from _tensors(v)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            yield from _tensors(v)


@pytest.mark.parametrize("with_teacher", [False, True])
def test_distill_scalars_are_logged_only_with_a_teacher(workdir, with_teacher):
    from helpers import tiny_model
    t = _trainer(tiny_model(), _teacher() if with_teacher else None, tensorboard=True, log_every=2, nb_steps_tot=10)
    logs = _logged(t)
    t.writer.flush()
    assert logs
    rows = [json.loads(line) for line in open(os.path.join(t.writer.logdir, "scalars.jsonl"))]
    tags = {r["tag"] for r in rows}
    if not with_teacher:
        assert all("distill_kl" not in d and "distill_ce" not in d for d in logs) and "distill_kl" not in tags
        return
    for d in logs:
        assert d["distill_kl"] > 0 and d["distill_ce"] > 0
        assert d["loss"] == pytest.approx(0.5 * d["distill_ce"] + 0.5 * d["distill_kl"], rel=1e-5)
    assert {"distill_kl", "distill_ce"} <= tags and sum(r["tag"] == "distill_kl" for r in rows) == len(logs)


def _write_hf_dir(model, d: str) -> None:
    """An HF checkpoint directory (``config.json`` + safetensors) of a native model."""
    from safetensors.torch import save_file
    os.makedirs(d)
    with open(os.path.join(d, "config.json"), "w") as f:
        json.dump(model.config.to_dict(), f)
    save_file({k: v.detach().contiguous().clone() for k, v in model.state_dict().items()}, os.path.join(d, "model.safetensors"))


def test_cli_pretraining_with_a_teacher_checkpoint(workdir, monkeypatch):
    sys.path.insert(0, ROOT)
    import main as cli
    from acco_b200 import ops
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    seen = []
    orig = ops.distill_cross_entropy

    def kd(*a, **kw):
        seen.append((a[4], a[5]))
        return orig(*a, **kw)
    monkeypatch.setattr(ops, "distill_cross_entropy", kd)
    torch.manual_seed(2)
    teacher = LlamaForCausalLM(LlamaConfig(vocab_size=512, hidden_size=32, intermediate_size=48, num_hidden_layers=1,
                                           num_attention_heads=4, max_position_embeddings=64))      # config/model/tiny.yaml's vocabulary
    tdir = os.path.join(os.getcwd(), "teacher")
    _write_hf_dir(teacher, tdir)
    stats = cli.main(["train=acco", "model=tiny", "data=synthetic", "train.nb_steps_tot=6", "train.batch_size=2", "train.max_length=32",
                      "train.use_mixed_precision=False", "data.synthetic_docs=200", "data.synthetic_mean_len=12", "train.warmup=0",
                      "run_name=kd", "train.save=False", f"train.distill_teacher={tdir}", "train.distill_alpha=0.25",
                      "train.distill_temperature=2.0", "train.dataloader_num_workers=0"])
    assert stats["count_grad_tot"] >= 6
    assert seen and set(seen) == {(0.25, 2.0)}


if __name__ == "__main__":               # print the margin table: python tests/test_distill.py
    for name, row in ROWS.items():
        emu, caught = row()
        print(f"{name:18s} emulator/bound " + " ".join(f"{k}={v:.3f}" for k, v in emu.items()))
        for m, (k, r) in caught.items():
            print(f"{'':18s}   mutant {m:20s} worst {k}: {r:.3g}x")
