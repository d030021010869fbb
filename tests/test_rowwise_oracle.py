"""fp64 oracles of the row-wise kernels (norms, RoPE, SwiGLU, GELU-new, cross-entropy), the per-element bounds of their GPU tests
(``test_rowwise_kernels_gpu.py``), and the margin table that shows the bounds are the right size.  Runs on the CPU without the
extension.

The oracles are written from the math in fp64; ``test_oracles_match_fp64_autograd`` checks each once against fp64 torch autograd.

What the binary executes.  ``build_ext.py`` compiles with ``--use_fast_math``, so fp32 subnormals are flushed to zero (FTZ),
divisions are approximate and the transcendentals are MUFU instructions.  The sm_90a SASS of the kernels contains:

==========================================  ==========================================================
kernel                                      approximate instructions
==========================================  ==========================================================
``norm_fwd_kernel`` (every instantiation)   ``MUFU.RSQ`` (rsqrt), ``MUFU.RCP`` (``/ H``)
``norm_bwd_kernel``                         ``MUFU.RCP`` (``/ H``)
``rope_qkv_kernel``, ``rope_pack_bwd``      ``MUFU.RCP`` (integer ``t % S``, ``t / S`` only; no float op)
``swiglu_fwd_kernel``, ``swiglu_bwd``       ``MUFU.EX2`` (``__expf``), ``MUFU.RCP`` (``1 / (1 + e)``)
``gelu_fwd_kernel``, ``gelu_bwd_kernel``    ``MUFU.EX2``, ``MUFU.RCP`` (sigmoid form; before: ``MUFU.TANH``)
``ce_fwd_kernel``                           ``MUFU.EX2``, ``MUFU.LG2`` (``__logf``)
``ce_reduce_kernel``                        ``MUFU.RCP`` (``1 / n``)
``ce_bwd_kernel``                           ``MUFU.EX2``
==========================================  ==========================================================

Documented errors used (CUDA C++ Programming Guide, intrinsic functions; PTX ISA for ``tanh.approx``), ``U = 2^-24`` the fp32 unit
roundoff, one ulp at most ``2^-23`` relative:

* ``rsqrt`` (``E_RSQ``), reciprocal and fast division (``E_RCP``): 2 ulp, ``2^-22`` relative;
* ``__expf(a)``: ``2 + 1.173 |a|`` ulp (``e_exp``; the ``|a|`` term is the rounding of ``a log2 e`` before ``ex2``);
* ``__logf(x)``: ``2^-21.41`` absolute for x in [0.5, 2], 3 ulp otherwise (``E_LG2`` + 3 ulp of the result);
* ``tanh.approx.f32``: ``2^-10.987`` relative (only the former GELU used it).

Bounds.  Every bf16 output ``y`` gets ``|y - y64| <= 2^-7 (|y64| + E) + E + ftz`` where ``E`` is twice a first-order bound of the
kernel's fp32 error and ``2^-7`` is one bf16 ulp (twice the half ulp of rounding to nearest, so an honest kernel stays within half).
fp32 outputs (``mean``, ``rstd``, ``lse``, ``inv_n``, fp32 ``dw | db``) get ``E + ftz`` alone: an ``H - 1`` variance or a misplaced
eps shows up there.  ``ftz`` is ``2^-125`` (twice the flush threshold ``2^-126``) times one (the output itself flushed) plus
the factors a flushed intermediate is multiplied by.  Per kernel:

* Norms.  Row sums: each owner (lane or thread) adds ``8 VPT`` terms in sequence, then a butterfly of 5 levels (warp) or 10
  (warp + CTA), so a row sum errs by at most ``D_ROW U sum|terms|`` with ``D_ROW = 8 VPT + 12``.  LayerNorm mean:
  ``e_mu = D_ROW U mean|h| + (E_RCP + U) |mu|``; the variance about the computed mean is the true one plus ``e_mu^2`` (the cross
  term vanishes), so ``var_err = (D_ROW + 5 + E_RCP/U) U var + e_mu^2 + U eps``; ``e_r = E_RSQ + var_err / (2 (var + eps))``.  This
  is where a LayerNorm row of tiny variance is ill-conditioned: ``e_mu rstd`` grows with ``|mu| / std``.  ``xh`` errs by
  ``e_mu rstd + |xh| (e_r + 2U)``; y by ``|w| xh_err + 3U |xh w| + U |y|``.  Backward: ``c1 = mean(g xh)`` and ``c2 = mean(g)``
  (``g = dy w`` is exact) err by their sums' ``D_ROW`` terms plus ``mean(|g| xh_err)``; ``dh = rstd (g - c2 - xh c1)`` cancels
  when the three terms meet, so its bound is absolute in them: ``rstd (3U (|g| + |c2| + |xh c1|) + e_c2 + |xh| e_c1 + |c1| xh_err)
  + |inner| rstd (e_r + U) + U (|dh| + |dh_extra|)``.  ``dw = sum_rows dy xh`` and ``db = sum_rows dy``: every owner adds its rows in
  sequence (``ceil(T / owners)`` terms), then 8 warps (warp rows), then ``reduce_partials`` (``ceil(grid / 64) + 33`` adds), so
  ``D_T = rows_per_owner + ceil(grid / 64) + 45`` and ``e_dw = D_T U sum|dy xh| + sum |dy| xh_err``.  Into a bf16 ``.grad``: one
  more fp32 add and the bf16 rounding of ``g0 + dw``.
* RoPE: ``x1 c - x2 s`` (contracted or not) errs by ``2U (|x1 c| + |x2 s|)`` before the bf16 rounding.  Tables are inputs.
* SwiGLU: ``sig = rcp(1 + e^-g)`` errs by ``e_sig = E_RCP + U + (1 - sig) e_exp(g)`` relative; the forward by ``e_sig + 2U``.  The
  backward's ``1 + g (1 - sig)`` cancels at ``g ~ -1.278``: its error is absolute, ``|g| sig e_sig + 2U |g| (1 - sig) +
  U (1 + |g (1 - sig)|)``, times ``|d u sig|``, plus ``|dgate| (e_sig + 3U)``.
* GELU-new, evaluated as ``x sig(z)``, ``z = 2 k0 x (1 + k1 x^2)`` (the tanh form cancels in ``1 + t`` for x < -2, where
  the tanh error is tens to thousands of bf16 ulps): ``z`` errs by ``5U |z|``, so ``e_sig = E_RCP + U + (1 - sig) (e_exp(z) + 5U |z|)``;
  forward ``e_sig + U``.  Backward ``sig (1 + x (1 - sig) z')``, ``z' = 2 k0 (1 + 3 k1 x^2)``, has the same absolute treatment of
  the bracket as SwiGLU.  ``ftz``: ``sig`` below ``2^-126`` is flushed, so the bound adds ``2^-125 (1 + |dy| (1 + |x|) (1 + |x| z'))``.
* Cross-entropy: a thread sweeps ``n_sw = ceil(V / 8 / 512) + 1`` vectors, each an 8-term sum and one rescale ``exp(m - m')``, and
  the CTA sums 512 partials: ``rel(gs) = (10 n_sw + 12) U + (n_sw + 2) e_exp(R)`` with ``R`` the row's logit spread;
  ``E_lse = rel(gs) + E_LG2 + 3 * 2^-23 |ln gs| + U |lse|``.  Row loss ``lse - x[label]``; the mean adds
  ``(ceil(T / 1024) + 10) U`` of the absolute row losses and ``E_RCP``.  d-logits ``(exp(x - lse) - onehot) * scale``: ``p`` errs
  by ``p (E_lse + U |x - lse| + e_exp(x - lse))``.

The margin table (``test_margin_table``) runs a blockwise fp32 emulator of each kernel in its own summation order (MUFU results
rounded correctly to fp32) and asserts that it stays within half of every bound, and that each mutant lands more than 3x outside on
at least one check.  Print it with ``python tests/test_rowwise_oracle.py``."""
from __future__ import annotations

import math
from typing import Dict, Optional

import pytest
import torch
import torch.nn.functional as F

from test_gemm_oracle import bf16_rn

U = 2.0 ** -24                 # fp32 unit roundoff
ULP = 2.0 ** -23
B7 = 2.0 ** -7                 # one bf16 ulp, relative
FTZ = 2.0 ** -125             # twice the flush-to-zero threshold 2^-126, as every other term of a bound is doubled
BF16_OVF = (2 - 2.0 ** -8) * 2.0 ** 127      # the smallest magnitude that rounds to inf in bf16
E_RSQ = E_RCP = 2.0 ** -22
E_LG2 = 2.0 ** -21.41
K0, K1 = 0.7978845608028654, 0.044715
KZ = 2 * K0
EPS = 1e-5


def e_exp(a: torch.Tensor) -> torch.Tensor:
    """Relative error of ``__expf(a)``: ``2 + 1.173 |a|`` ulp."""
    return (2.0 + 1.173 * a.abs()) * ULP


def f32(x: torch.Tensor) -> torch.Tensor:
    """Round to fp32 (nearest), returned as fp64."""
    return x.double().float().double()


def out_bound(y64: torch.Tensor, E: torch.Tensor, ftz=FTZ) -> torch.Tensor:
    """Bound of a bf16 output: one bf16 ulp of ``|y64| + E``, plus ``E``, plus the flush-to-zero allowance."""
    return B7 * (y64.abs() + E) + E + ftz


def ratio(got: torch.Tensor, want: torch.Tensor, bnd: torch.Tensor) -> float:
    """Largest ``|got - want| / bound`` (non-finite ``got`` counts as infinitely wrong)."""
    got, want = got.double(), want.double()
    err = (got - want).abs()
    err = torch.where(torch.isfinite(got), err, torch.full_like(err, math.inf))
    overflow = torch.isinf(got) & (want.abs() >= BF16_OVF) & (torch.sign(got) == torch.sign(want))   # rounds to inf in bf16
    err = torch.where(overflow, torch.zeros_like(err), err)
    return float((err / bnd).max()) if err.numel() else 0.0


def finite_bf16() -> torch.Tensor:
    """Every finite bf16 value (both zeros, subnormals), as bf16."""
    x = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    return x[torch.isfinite(x.float())]


# ================================================================================================= norms
def norm_geometry(H: int):
    """(VPT, CTA_ROW, owners of a row) exactly as ``ACCO_NORM_DISPATCH`` / ``cta_geom`` pick them."""
    nvec = H // 8
    if H <= 1024:
        return max(1, -(-nvec // 32)), False, 32
    vpt = 1
    while -(-nvec // vpt) > 512:
        vpt *= 2
    return vpt, True, -(-(-(-nvec // vpt)) // 32) * 32


def norm_grid(T: int, H: int, sms: int, backward: bool) -> int:
    """``acco_norm_grid``."""
    if H <= 1024:
        want, per_sm = -(-T // 8), (2 if backward else 8)
    else:
        want, per_sm = T, 2048 // norm_geometry(H)[2]
        if backward:
            per_sm = min(per_sm, 4)
    return max(1, min(want, sms * per_sm))


def rows_per_owner(T: int, H: int, grid: int) -> int:
    """Most rows one warp (H <= 1024) or CTA walks in the grid-stride loop."""
    step = grid * (1 if H > 1024 else 8)
    return -(-T // step)


def norm_ref(a, w, b=None, r=None, dy=None, extra=None, eps=EPS) -> Dict[str, torch.Tensor]:
    """fp64 oracle from the math.  ``h`` is the stored bf16 residual sum ``bf16_rn(a + r)`` (what the kernel normalises)."""
    layer = b is not None
    h = bf16_rn(a.double() + r.double()).double() if r is not None else a.double()
    H = h.shape[-1]
    mu = h.mean(-1, keepdim=True) if layer else torch.zeros_like(h[:, :1])
    var = ((h - mu) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xh = (h - mu) * rstd
    w64 = w.double()
    out = {"h": h, "mean": mu[:, 0], "rstd": rstd[:, 0], "var": var[:, 0], "xh": xh,
           "y": xh * w64 + (b.double() if layer else 0.0)}
    if dy is not None:
        d = dy.double()
        g = d * w64
        c1 = (g * xh).mean(-1, keepdim=True)
        c2 = g.mean(-1, keepdim=True) if layer else torch.zeros_like(c1)
        inner = g - c2 - xh * c1
        out.update(g=g, c1=c1, c2=c2, inner=inner, dh=rstd * inner + (extra.double() if extra is not None else 0.0),
                   dw=(d * xh).sum(0), db=d.sum(0))
    return out


def norm_bounds(o, w, H: int, T: int, grid: int, layer: bool, dy=None, extra=None, g0w=None, g0b=None, eps=EPS):
    """Per-element / per-row bounds (module docstring) for the outputs of ``norm_ref``; ``g0w`` / ``g0b``: the bf16 ``.grad``
    content dw / db are added to (None: fp32 output)."""
    vpt, cta, _ = norm_geometry(H)
    D_ROW = 8 * vpt + 12
    h, mu, var, rstd, xh = o["h"], o["mean"][:, None], o["var"][:, None], o["rstd"][:, None], o["xh"]
    w64 = w.double().abs()
    e_mu = (D_ROW * U * h.abs().mean(-1, keepdim=True) + (E_RCP + U) * mu.abs()) if layer else torch.zeros_like(mu)
    var_err = (D_ROW + 5 + E_RCP / U) * U * var + e_mu ** 2 + U * eps
    e_r = E_RSQ + var_err / (2 * (var + eps))
    xh_err = e_mu * rstd + xh.abs() * (e_r + 2 * U)
    E_y = 2 * (w64 * xh_err + 3 * U * (xh * w64).abs() + U * o["y"].abs())
    out = {"y": out_bound(o["y"], E_y), "rstd": (2 * e_r * rstd + FTZ)[:, 0]}
    if layer:
        out["mean"] = (2 * e_mu + FTZ)[:, 0]
    if dy is None:
        return out
    g, c1, c2, inner = o["g"], o["c1"], o["c2"], o["inner"]
    d = dy.double().abs()
    e_c1 = (D_ROW + 3) * U * (g * xh).abs().mean(-1, keepdim=True) + (g.abs() * xh_err).mean(-1, keepdim=True) + (E_RCP + U) * c1.abs()
    e_c2 = (D_ROW + 2) * U * g.abs().mean(-1, keepdim=True) + (E_RCP + U) * c2.abs()
    e_in = 3 * U * (g.abs() + c2.abs() + (xh * c1).abs()) + e_c2 + xh.abs() * e_c1 + c1.abs() * xh_err
    ex = extra.double().abs() if extra is not None else 0.0
    E_dh = 2 * (rstd * e_in + inner.abs() * rstd * (e_r + U) + U * (o["dh"].abs() + ex))
    out["dh"] = out_bound(o["dh"], E_dh)
    D_T = rows_per_owner(T, H, grid) + -(-grid // 64) + 45
    E_dw = 2 * (D_T * U * (d * xh.abs()).sum(0) + (d * xh_err).sum(0))
    E_db = 2 * D_T * U * d.sum(0)
    out["E_dw"], out["E_db"] = E_dw, E_db
    for name, E, g0 in (("dw", E_dw, g0w), ("db", E_db, g0b)):
        if name == "db" and not layer:
            continue
        out[name] = param_bound(o[name], E, g0)
    return out


def param_bound(d64: torch.Tensor, E: torch.Tensor, g0=None) -> torch.Tensor:
    """dw / db: fp32 output (``g0`` None), or added to the bf16 ``.grad`` content ``g0`` (one fp32 add and one bf16 rounding)."""
    if g0 is None:
        return E + FTZ
    return out_bound(g0.double() + d64, E + 2 * U * (g0.double().abs() + d64.abs()))


def norm_want(o, g0w=None, g0b=None):
    """The values the kernel must approximate: dw / db added to the bf16 ``.grad`` content when accumulating."""
    want = dict(o)
    if g0w is not None:
        want["dw"] = g0w.double() + o["dw"]
    if g0b is not None:
        want["db"] = g0b.double() + o["db"]
    return want


def _row_sum32(terms: torch.Tensor, H: int) -> torch.Tensor:
    """Row sums of fp64 ``terms [T, H]`` in the kernel's order: every owner adds its ``8 VPT`` terms in sequence (one fp32 rounding
    per add, which also models a contracted ``s += a * b``), then the xor butterfly of ``warp_sum`` (and ``block_sum``'s second
    butterfly over the warps for CTA rows)."""
    vpt, cta, owners = norm_geometry(H)
    T = terms.shape[0]
    x = torch.zeros(T, vpt * owners * 8, dtype=torch.float64)
    x[:, :H] = terms
    x = x.view(T, vpt, owners, 8)
    s = torch.zeros(T, owners, dtype=torch.float64)
    for i in range(vpt):
        for j in range(8):
            s = f32(s + x[:, i, :, j])

    def butterfly(v):                                  # v [T, n, 32]
        for o in (16, 8, 4, 2, 1):
            v = f32(v + v[..., torch.arange(32) ^ o])
        return v[..., 0]

    s = butterfly(s.view(T, owners // 32, 32))         # [T, warps]
    if cta:
        pad = torch.zeros(T, 32, dtype=torch.float64)
        pad[:, :s.shape[1]] = s
        s = butterfly(pad[:, None, :])[:, 0:1]
    return s[:, 0]


def _reduce_partials32(P: torch.Tensor) -> torch.Tensor:
    """``reduce_partials_kernel`` over fp64 partials ``[nparts, W]`` (fp32 values): two interleaved running sums per row of the
    block, then 32 in sequence."""
    nparts, W = P.shape
    sm = torch.zeros(32, W, dtype=torch.float64)
    for ty in range(32):
        s0 = torch.zeros(W, dtype=torch.float64)
        s1 = torch.zeros(W, dtype=torch.float64)
        p = ty
        while p + 32 < nparts:
            s0, s1 = f32(s0 + P[p]), f32(s1 + P[p + 32])
            p += 64
        if p < nparts:
            s0 = f32(s0 + P[p])
        sm[ty] = f32(s0 + s1)
    s = torch.zeros(W, dtype=torch.float64)
    for k in range(32):
        s = f32(s + sm[k])
    return s


NORM_MUTANTS = ("acc_reset", "drop_last_partial", "no_extra_cta", "var_h1", "eps_outside", "no_c2", "fp32_h")


def emulate_norm(a, w, b=None, r=None, dy=None, extra=None, sms: int = 2, eps=EPS, mutant: Optional[str] = None):
    """Blockwise fp32 emulator of ``norm_fwd_kernel`` + ``norm_bwd_kernel`` + ``reduce_partials`` (fp32 dw | db) at ``sms`` SMs."""
    layer = b is not None
    T, H = a.shape
    vpt, cta, owners = norm_geometry(H)
    inv_h = f32(torch.tensor(1.0 / H))
    hf = f32(a.double() + r.double()) if r is not None else a.double()
    h = hf if mutant == "fp32_h" else bf16_rn(hf).double()
    if layer:
        mu = f32(_row_sum32(h, H) * inv_h)[:, None]
        dev = f32(h - mu)
        ss = _row_sum32(dev * dev, H)
    else:
        mu = torch.zeros(T, 1, dtype=torch.float64)
        ss = _row_sum32(h * h, H)
    var = f32(ss / (H - 1)) if mutant == "var_h1" else f32(ss * inv_h)
    if mutant == "eps_outside":
        rstd = f32(f32(1.0 / torch.sqrt(var)) + eps)[:, None]
    else:
        rstd = f32(1.0 / torch.sqrt(f32(var + eps)))[:, None]
    xh = f32(f32(h - mu) * rstd)
    y = bf16_rn(f32(f32(xh * w.double()) + (b.double() if layer else 0.0))).double()
    out = {"h": bf16_rn(hf).double(), "y": y, "rstd": rstd[:, 0], "mean": mu[:, 0]}
    if dy is None:
        return out
    # the backward reads the stored bf16 h and the forward's statistics
    h = bf16_rn(hf).double()
    xh = f32(f32(h - mu) * rstd)
    d = dy.double()
    g = d * w.double()
    c1 = f32(_row_sum32(g * xh, H) * inv_h)[:, None]
    c2 = f32(_row_sum32(g, H) * inv_h)[:, None] if layer and mutant != "no_c2" else torch.zeros_like(c1)
    o = f32(rstd * f32(f32(g - c2) - f32(xh * c1)))
    if extra is not None and not (mutant == "no_extra_cta" and cta):
        o = f32(o + extra.double())
    out["dh"] = bf16_rn(o).double()
    grid = norm_grid(T, H, sms, True)
    per = 1 if cta else 8
    step = grid * per
    parts = []
    for term in ([d * xh, d] if layer else [d * xh]):
        acc = torch.zeros(step, H, dtype=torch.float64)          # one accumulator per (CTA, warp)
        for k in range(0, T, step):
            rows = slice(k, min(T, k + step))
            n = rows.stop - rows.start
            acc[:n] = term[rows] if mutant == "acc_reset" else f32(acc[:n] + term[rows])
        if not cta:                                              # the 8 warps of a CTA, in order, through shared memory
            acc = acc.view(grid, 8, H)
            s = torch.zeros(grid, H, dtype=torch.float64)
            for k in range(8):
                s = f32(s + acc[:, k])
            acc = s
        parts.append(acc)
    P = torch.cat(parts, 1)
    if mutant == "drop_last_partial":
        P = P[:-1]
    dwdb = _reduce_partials32(P)
    out["dw"] = dwdb[:H]
    if layer:
        out["db"] = dwdb[H:]
    return out


def norm_inputs(T: int, H: int, layer: bool, residual: bool, extra: bool, seed: int, device="cpu"):
    """Rows scaled by distinct powers of two (a row mix-up is gross), weights near 1, small bias."""
    g = torch.Generator(device=device).manual_seed(seed)
    rn = lambda *shape: torch.randn(*shape, generator=g, device=device)
    scale = 2.0 ** (torch.arange(T, device=device) % 9 - 4).float()[:, None]
    a = (rn(T, H) * scale).to(torch.bfloat16)
    r = (rn(T, H) * scale).to(torch.bfloat16) if residual else None
    w = (1 + 0.1 * rn(H)).to(torch.bfloat16)
    b = (0.1 * rn(H)).to(torch.bfloat16) if layer else None
    dy = rn(T, H).to(torch.bfloat16)
    ex = rn(T, H).to(torch.bfloat16) if extra else None
    return a, w, b, r, dy, ex


def norm_checks(got, o, bnd, layer: bool, residual: bool) -> Dict[str, float]:
    names = ["y", "rstd", "dh", "dw"] + (["mean", "db"] if layer else [])
    out = {k: ratio(got[k], o[k], bnd[k]) for k in names if k in got}
    if residual:
        out["h"] = 0.0 if torch.equal(got["h"].double(), o["h"]) else math.inf
    return out


# ================================================================================================= RoPE
def rope_tables64(S: int, D: int, theta: float):
    """The fp32 tables of ``ops.rope_tables`` (computed the same way, in fp32), which the kernels take as given inputs."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
    fr = torch.outer(torch.arange(S, dtype=torch.float32), inv_freq)
    return fr.cos().contiguous(), fr.sin().contiguous()


def rope_ref(x, cos, sin, n_rot: int, S: Optional[int] = None, inverse: bool = False, pos=None):
    """fp64 oracle of the rotate-half RoPE on ``x [T, n_total, D]``: heads ``< n_rot`` rotated at position ``t % S`` (or the per-token
    ``pos``), the rest copied.  Returns ``(y64, E)`` with ``E`` the fp32 error bound before the bf16 rounding."""
    T, n, D = x.shape
    half = D // 2
    if pos is None:
        pos = torch.arange(T, device=x.device) % S
    c = cos.double()[pos][:, None, :]
    s = sin.double()[pos][:, None, :] * (-1.0 if inverse else 1.0)
    x64 = x.double()
    x1, x2 = x64[..., :half], x64[..., half:]
    y = x64.clone()
    E = torch.zeros_like(x64)
    rot1, rot2 = x1 * c - x2 * s, x2 * c + x1 * s
    mag = 4 * U * ((x1 * c).abs() + (x2 * s).abs() + (x2 * c).abs() + (x1 * s).abs())
    y[:, :n_rot, :half], y[:, :n_rot, half:] = rot1[:, :n_rot], rot2[:, :n_rot]
    E[:, :n_rot, :half], E[:, :n_rot, half:] = mag[:, :n_rot], mag[:, :n_rot]
    return y, E


ROPE_MUTANTS = ("pos_t", "interleaved", "no_sign_flip", "k_unrotated")


def emulate_rope(x, cos, sin, S: int, n_rot: int, Hq: int, inverse=False, mutant=None):
    T, n, D = x.shape
    half = D // 2
    pos = torch.arange(T) if mutant == "pos_t" else torch.arange(T) % S
    c = cos.double()[pos][:, None, :]
    sg = -1.0 if inverse and mutant != "no_sign_flip" else 1.0
    s = sin.double()[pos][:, None, :] * sg
    x64 = x.double()
    if mutant == "interleaved":
        x1, x2 = x64[..., 0::2], x64[..., 1::2]
    else:
        x1, x2 = x64[..., :half], x64[..., half:]
    o1 = bf16_rn(f32(f32(x1 * c) - f32(x2 * s))).double()
    o2 = bf16_rn(f32(f32(x2 * c) + f32(x1 * s))).double()
    nr = Hq if mutant == "k_unrotated" else n_rot
    y = x64.clone()
    if mutant == "interleaved":
        y[:, :nr, 0::2], y[:, :nr, 1::2] = o1[:, :nr], o2[:, :nr]
    else:
        y[:, :nr, :half], y[:, :nr, half:] = o1[:, :nr], o2[:, :nr]
    return y


# ================================================================================================= SwiGLU / GELU-new
def _sig(z):
    return torch.where(z >= 0, 1.0 / (1.0 + torch.exp(-z)), torch.exp(z) / (1.0 + torch.exp(z)))


def swiglu_ref(g, u, d=None):
    """fp64 ``out = silu(g) u``; with ``d``: ``(dgate, dup)`` and the bounds of all three."""
    g64, u64 = g.double(), u.double()
    sg = _sig(g64)
    out = g64 * sg * u64
    e_sig = E_RCP + U + (1 - sg) * e_exp(g64)
    res = {"out": out, "b_out": out_bound(out, 2 * (e_sig + 2 * U) * out.abs(), FTZ * (1 + (1 + g64.abs()) * u64.abs()))}
    if d is not None:
        d64 = d.double()
        br = 1 + g64 * (1 - sg)
        dg = d64 * u64 * sg * br
        du = d64 * g64 * sg
        e_br = g64.abs() * sg * e_sig + 2 * U * (g64 * (1 - sg)).abs() + U * (1 + (g64 * (1 - sg)).abs())
        E_dg = 2 * ((d64 * u64 * sg).abs() * e_br + dg.abs() * (e_sig + 3 * U))
        ftz = FTZ * (1 + (d64 * u64).abs() * (1 + g64.abs()) ** 2)
        res.update(dgate=dg, dup=du, b_dgate=out_bound(dg, E_dg, ftz),
                   b_dup=out_bound(du, 2 * (e_sig + 2 * U) * du.abs(), FTZ * (1 + (1 + g64.abs()) * d64.abs())))
    return res


def emulate_swiglu(g, u, d, mutant=None):
    g64, u64, d64 = g.double(), u.double(), d.double()
    e = f32(torch.exp(-g64))
    sg = f32(1.0 / f32(1 + e))
    out = bf16_rn(f32(f32(g64 * sg) * u64)).double()
    br = f32(1 + f32(g64 * f32(1 - sg)))
    if mutant == "no_g_term":
        br = torch.ones_like(br)
    dg = bf16_rn(f32(f32(f32(d64 * u64) * sg) * br)).double()
    du = bf16_rn(f32(d64 * f32(g64 * sg))).double()
    return {"out": out, "dgate": dg, "dup": du}


def gelu_ref(x, dy=None):
    """fp64 ``gelu_new(x) = x sig(2 k0 (x + k1 x^3))`` (= ``0.5 x (1 + tanh(.))``) and, with ``dy``, ``dy gelu'(x)``, with bounds."""
    x64 = x.double()
    z = KZ * x64 * (1 + K1 * x64 * x64)
    s = _sig(z)
    y = x64 * s
    e_sig = E_RCP + U + (1 - s) * (e_exp(z) + 5 * U * z.abs())
    res = {"y": y, "b_y": out_bound(y, 2 * (e_sig + U) * y.abs(), FTZ * (2 + x64.abs()))}
    if dy is not None:
        d64 = dy.double()
        zp = KZ * (1 + 3 * K1 * x64 * x64)
        A = x64 * (1 - s) * zp
        gp = s * (1 + A)
        dx = d64 * gp
        e_A = x64.abs() * zp * (e_sig * s + 2 * U * (1 - s)) + 3 * U * A.abs()
        E = 2 * d64.abs() * (s * (e_A + U * (1 + A.abs())) + gp.abs() * (e_sig + 2 * U))
        ftz = FTZ * (1 + d64.abs() * (1 + x64.abs()) * (1 + x64.abs() * zp))
        res.update(dx=dx, b_dx=out_bound(dx, E, ftz))
    return res


def emulate_gelu(x, dy, mutant=None, form: str = "sigmoid"):
    """fp32 emulator of the GELU kernels: the sigmoid form, or ``form="tanh"`` for the former ``0.5 x (1 + tanh(u))`` (tanh rounded
    correctly to fp32, i.e. without the MUFU.TANH error)."""
    x64, d64 = x.double(), dy.double()
    k3 = K1 if mutant == "k1_for_3k1" else 3 * K1
    if form == "tanh":
        u = f32(K0 * f32(x64 + f32(K1 * f32(x64 * f32(x64 * x64)))))
        t = f32(torch.tanh(u))
        y = f32(f32(0.5 * x64) * f32(1 + t))
        gp = f32(f32(0.5 * f32(1 + t)) + f32(f32(f32(0.5 * x64) * f32(1 - f32(t * t))) * f32(K0 * f32(1 + f32(k3 * f32(x64 * x64))))))
    else:
        xc = x64.clamp(-12, 12)
        z = f32(f32(KZ * x64) * f32(1 + f32(K1 * f32(x64 * x64))))
        y = f32(x64 * f32(1.0 / f32(1 + f32(torch.exp(-z)))))
        x2 = f32(xc * xc)
        s = f32(1.0 / f32(1 + f32(torch.exp(-f32(f32(KZ * xc) * f32(1 + f32(K1 * x2)))))))
        gp = f32(s * f32(1 + f32(f32(f32(xc * f32(1 - s)) * KZ) * f32(1 + f32(k3 * x2)))))
    return {"y": bf16_rn(y).double(), "dx": bf16_rn(f32(d64 * gp)).double()}


# ================================================================================================= cross-entropy
def ce_ref(logits, labels, V: int, ignore_index: int = -100, scale: Optional[float] = None):
    """fp64 oracle: ``lse`` (0 on ignored rows), row losses, mean ``loss`` and ``inv_n`` (both 0 when every row is ignored), and
    with ``scale`` the d-logits ``(softmax - onehot) * scale`` (0 on ignored rows and padding columns).  Bounds included."""
    T, Vp = logits.shape
    x = logits[:, :V].double()
    valid = labels != ignore_index
    labels = labels.to(x.device)
    lab = torch.where(valid, labels, torch.zeros_like(labels))
    lse = torch.logsumexp(x, 1)
    xl = x.gather(1, lab[:, None])[:, 0]
    row = torch.where(valid, lse - xl, torch.zeros_like(lse))
    lse = torch.where(valid, lse, torch.zeros_like(lse))
    n = int(valid.sum())
    inv = 1.0 / n if n else 0.0
    loss = float(row.sum()) * inv
    # bounds
    n_sw = -(-(V // 8) // 512) + 1
    R = x.max(1).values - x.min(1).values
    gs = torch.exp(lse - x.max(1).values)
    rel_gs = (10 * n_sw + 12) * U + (n_sw + 2) * e_exp(R)
    E_lse = torch.where(valid, rel_gs + E_LG2 + 3 * ULP * torch.log(gs).abs() + U * lse.abs(), torch.zeros_like(lse))
    E_row = E_lse + U * row.abs()
    res = {"lse": lse, "loss": loss, "inv_n": inv, "row": row, "E_row": E_row, "b_lse": 2 * E_lse + FTZ,
           "b_loss": ce_loss_bound(float(E_row.sum()), float(row.abs().sum()), T, loss, inv), "b_inv": 2 * E_RCP * inv}
    if scale is not None:
        arg = x - lse[:, None]
        p = torch.exp(arg)
        oh = torch.zeros_like(p)
        oh.scatter_(1, lab[:, None], 1.0)
        q = (p - oh) * scale
        E_p = p * (E_lse[:, None] + U * arg.abs() + e_exp(arg))
        E = 2 * (abs(scale) * (E_p + U * (p - oh).abs()) + U * q.abs())
        grad = torch.zeros(T, Vp, dtype=torch.float64, device=x.device)
        bnd = torch.full((T, Vp), FTZ, dtype=torch.float64, device=x.device)
        grad[:, :V] = torch.where(valid[:, None], q, torch.zeros_like(q))
        bnd[:, :V] = torch.where(valid[:, None], out_bound(q, E, FTZ * (1 + abs(scale))), torch.full_like(q, FTZ))
        res.update(grad=grad, b_grad=bnd)
    return res


def ce_loss_bound(sum_E_row: float, sum_abs_row: float, T: int, loss: float, inv: float) -> float:
    """Bound of the mean loss: the row losses' own bounds, ``ce_reduce``'s ``ceil(T / 1024) + 10``-deep fp32 sum and ``1 / n``."""
    D_T = -(-T // 1024) + 10
    return 2 * ((sum_E_row + D_T * U * sum_abs_row) * inv + abs(loss) * (E_RCP + U)) + FTZ


CE_MUTANTS = ("pad_in_softmax", "ignored_counted", "label_shift")


def emulate_ce(logits, labels, V: int, ignore_index: int = -100, scale: float = 1.0, mutant=None):
    """fp32 emulator of ``ce_fwd_kernel`` (512 threads, online max / sum over 8-wide vectors, scalar ragged tail, block max and
    sum), ``ce_reduce_kernel`` and ``ce_bwd_kernel``."""
    T, Vp = logits.shape
    Vs = Vp if mutant == "pad_in_softmax" else V
    x = logits.double()
    nvf = Vs // 8
    K = -(-nvf // 512)
    xv = torch.full((T, K * 512 * 8), -math.inf, dtype=torch.float64)
    xv[:, :nvf * 8] = x[:, :nvf * 8]
    xv = xv.view(T, K, 512, 8)
    m = torch.full((T, 512), -math.inf, dtype=torch.float64)
    s = torch.zeros(T, 512, dtype=torch.float64)

    def ex(a):
        return f32(torch.exp(a))

    for k in range(K):
        f = xv[:, k]
        live = torch.isfinite(f[..., 0])
        nm = torch.maximum(m, f.max(-1).values)
        acc = torch.zeros_like(s)
        for j in range(8):
            acc = f32(acc + ex(f32(f[..., j] - nm)))
        resc = torch.where(torch.isfinite(m), ex(f32(m - nm)), torch.zeros_like(m))
        s = torch.where(live, f32(f32(s * resc) + acc), s)
        m = torch.where(live, nm, m)
    for c in range(nvf * 8, Vs):
        t = c - nvf * 8
        f = x[:, c]
        nm = torch.maximum(m[:, t], f)
        resc = torch.where(torch.isfinite(m[:, t]), ex(f32(m[:, t] - nm)), torch.zeros_like(nm))
        s[:, t] = f32(f32(s[:, t] * resc) + ex(f32(f - nm)))
        m[:, t] = nm
    gm = m.max(1).values
    part = torch.where(torch.isfinite(m), f32(s * ex(f32(m - gm[:, None]))), torch.zeros_like(s))
    v = part.view(T, 16, 32)
    for o in (16, 8, 4, 2, 1):
        v = f32(v + v[..., torch.arange(32) ^ o])
    w = torch.zeros(T, 32, dtype=torch.float64)
    w[:, :16] = v[..., 0]
    for o in (16, 8, 4, 2, 1):
        w = f32(w + w[:, torch.arange(32) ^ o])
    gs = w[:, 0]
    valid = labels != ignore_index
    lab = torch.where(valid, labels, torch.zeros_like(labels))
    lse = f32(gm + f32(torch.log(gs)))
    row = f32(lse - x.gather(1, lab[:, None])[:, 0])
    lse = torch.where(valid, lse, torch.zeros_like(lse))
    row = torch.where(valid, row, torch.zeros_like(row))
    counted = torch.ones_like(valid) if mutant == "ignored_counted" else valid
    # ce_reduce: 1024 threads, each a strided running sum, then the block tree (approximated by a sequential fp32 sum)
    tot = torch.tensor(0.0, dtype=torch.float64)
    for i in range(T):
        if counted[i]:
            tot = f32(tot + row[i])
    n = int(counted.sum())
    inv = float(f32(torch.tensor(1.0 / n))) if n else 0.0
    loss = float(f32(tot * inv))
    cols = torch.arange(Vp)
    p = torch.where(cols[None, :] < Vs, ex(f32(torch.nan_to_num(x, nan=0.0) - lse[:, None])), torch.zeros_like(x))
    tgt = lab + 1 if mutant == "label_shift" else lab
    p = torch.where(cols[None, :] == tgt[:, None], f32(p - 1), p)
    grad = bf16_rn(f32(p * scale)).double()
    grad = torch.where(valid[:, None], grad, torch.zeros_like(grad))
    return {"lse": lse, "loss": loss, "inv_n": inv, "grad": grad}


def ce_inputs(T: int, V: int, Vp: int, seed: int, pad_fill: Optional[float] = None, device="cpu"):
    """Logits ~ 2 N(0, 1), a row of spread +-60, a row of equal logits; labels at 0, at V - 1 (the ragged tail), at the row's argmax,
    random elsewhere, every 5th row ignored."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = 2 * torch.randn(T, Vp, generator=g, device=device)
    if T > 2:
        x[1] = torch.rand(Vp, generator=g, device=device) * 120 - 60
        x[2] = 0.75
    lg = x.to(torch.bfloat16)
    if pad_fill is not None and Vp > V:
        lg[:, V:] = pad_fill
    lab = torch.randint(0, V, (T,), generator=g, device=device)
    lab[0] = 0
    if T > 1:
        lab[1] = V - 1
    if T > 3:
        lab[3] = int(lg[3, :V].float().argmax())
    lab[4::5] = -100
    return lg, lab


def ce_checks(got, o) -> Dict[str, float]:
    out = {"lse": ratio(got["lse"], o["lse"], o["b_lse"]),
           "loss": abs(float(got["loss"]) - o["loss"]) / o["b_loss"],
           "inv_n": abs(float(got["inv_n"]) - o["inv_n"]) / max(o["b_inv"], FTZ)}
    if "grad" in got:
        out["grad"] = ratio(got["grad"], o["grad"], o["b_grad"])
    return out


# ================================================================================================= oracle vs autograd
def test_oracles_match_fp64_autograd():
    g = torch.Generator().manual_seed(0)
    T, H = 6, 40
    a = torch.randn(T, H, generator=g, dtype=torch.float64).to(torch.bfloat16)
    r = torch.randn(T, H, generator=g, dtype=torch.float64).to(torch.bfloat16)
    w = (1 + 0.1 * torch.randn(H, generator=g)).to(torch.bfloat16)
    b = (0.1 * torch.randn(H, generator=g)).to(torch.bfloat16)
    dy = torch.randn(T, H, generator=g).to(torch.bfloat16)
    ex = torch.randn(T, H, generator=g).to(torch.bfloat16)
    close = lambda x, y: torch.testing.assert_close(x, y, rtol=1e-12, atol=1e-12)
    for layer in (False, True):
        o = norm_ref(a, w, b if layer else None, r, dy, ex)
        h = o["h"].clone().requires_grad_(True)
        w64 = w.double().requires_grad_(True)
        b64 = b.double().requires_grad_(True)
        if layer:
            y = F.layer_norm(h, (H,), w64, b64, EPS)
        else:
            y = h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + EPS) * w64
        (y * dy.double()).sum().backward()
        close(o["y"], y.detach())
        close(o["dh"], h.grad + ex.double())
        close(o["dw"], w64.grad)
        if layer:
            close(o["db"], b64.grad)
            close(o["mean"], o["h"].mean(-1))
            close(o["rstd"], 1 / torch.sqrt(o["h"].var(-1, unbiased=False) + EPS))
    # RoPE: the rotate-half pairing, against the complex-number rotation
    x = torch.randn(5, 3, 16, generator=g, dtype=torch.float64).to(torch.bfloat16)
    cos, sin = rope_tables64(4, 16, 500000.0)
    y, _ = rope_ref(x, cos, sin, n_rot=2, S=4)
    z = torch.complex(x.double()[..., :8], x.double()[..., 8:]) * torch.complex(cos.double(), sin.double())[torch.arange(5) % 4][:, None]
    close(y[:, :2], torch.cat([z.real, z.imag], -1)[:, :2])
    assert torch.equal(y[:, 2], x[:, 2].double())
    yi, _ = rope_ref(y, cos, sin, n_rot=2, S=4, inverse=True)
    torch.testing.assert_close(yi, x.double(), rtol=0, atol=1e-6)     # the fp32 tables have cos^2 + sin^2 = 1 to fp32 only
    # SwiGLU and GELU against autograd on silu / gelu(tanh)
    gg = torch.linspace(-20, 20, 4001, dtype=torch.float64).requires_grad_(True)
    uu = torch.linspace(-3, 3, 4001, dtype=torch.float64).requires_grad_(True)
    dd = torch.linspace(2, -2, 4001, dtype=torch.float64)
    s = swiglu_ref(gg.detach(), uu.detach(), dd)
    (F.silu(gg) * uu * dd).sum().backward()
    close(s["out"], F.silu(gg.detach()) * uu.detach())
    close(s["dgate"], gg.grad)
    close(s["dup"], uu.grad)
    xx = torch.linspace(-6, 6, 4001, dtype=torch.float64).requires_grad_(True)
    gr = gelu_ref(xx.detach(), dd)
    (F.gelu(xx, approximate="tanh") * dd).sum().backward()
    # absolute: fp64 autograd evaluates the tanh form, whose 1 + tanh cancels in the negative tail (the oracle's sigmoid form does not)
    torch.testing.assert_close(gr["y"], F.gelu(xx.detach(), approximate="tanh"), rtol=1e-12, atol=1e-13)
    torch.testing.assert_close(gr["dx"], xx.grad, rtol=1e-12, atol=1e-13)
    # cross-entropy, with padding and ignored rows
    lg, lab = ce_inputs(12, 37, 40, seed=3)
    o = ce_ref(lg, lab, 37, scale=2.5 / int((lab != -100).sum()))      # the kernel's scale is dloss * inv_n
    xr = lg[:, :37].double().requires_grad_(True)
    loss = F.cross_entropy(xr, lab, ignore_index=-100)
    (loss * 2.5).backward()
    assert abs(o["loss"] - float(loss.detach())) < 1e-12
    close(o["grad"][:, :37], xr.grad)
    assert bool((o["grad"][:, 37:] == 0).all())
    v = lab != -100
    close(o["lse"][v], torch.logsumexp(lg[:, :37].double(), 1)[v])
    assert o["inv_n"] == 1.0 / int(v.sum())


def test_all_ignored_batch_has_zero_loss_and_gradient():
    """The kernels return loss 0 and inverse count 0 when every row is ignored (HF's mean would be 0 / 0 = NaN); the oracle says
    the same, so a NaN from the kernel fails."""
    lg, lab = ce_inputs(8, 50, 56, seed=4)
    lab[:] = -100
    o = ce_ref(lg, lab, 50, scale=1.0)
    assert o["loss"] == 0.0 and o["inv_n"] == 0.0 and bool((o["lse"] == 0).all()) and bool((o["grad"] == 0).all())
    e = emulate_ce(lg, lab, 50)
    assert e["loss"] == 0.0 and e["inv_n"] == 0.0 and bool((e["grad"] == 0).all())


def test_norm_geometry_matches_dispatch():
    """Warp VPT 1..4 up to H = 1024, CTA VPT 1 / 2 / 4 above; the test widths reach every instantiation."""
    assert [norm_geometry(H)[:2] for H in (64, 256, 264, 512, 520, 768, 776, 1024)] == \
        [(1, False), (1, False), (2, False), (2, False), (3, False), (3, False), (4, False), (4, False)]
    assert [norm_geometry(H) for H in (1032, 4096, 4104, 8192, 8200, 16384)] == \
        [(1, True, 160), (1, True, 512), (2, True, 288), (2, True, 512), (4, True, 288), (4, True, 512)]
    assert norm_grid(8192, 768, 132, True) == 264 and rows_per_owner(8192, 768, 264) == 4


# ================================================================================================= margin table
NORM_CASES = [
    # (name, T, H, layer, residual, extra)
    ("rms-768", 150, 768, False, False, False),
    ("rms-res-2048", 40, 2048, False, True, True),
    ("ln-768", 150, 768, True, False, False),
    ("ln-res-4104", 36, 4104, True, True, True),
]


def norm_mutants(H, layer, residual, extra):
    out = ["acc_reset", "drop_last_partial", "eps_outside"]
    if extra and H > 1024:
        out.append("no_extra_cta")
    if layer:
        out += ["var_h1", "no_c2"]
    if residual:
        out.append("fp32_h")
    return out


def norm_row(name, T, H, layer, residual, extra):
    a, w, b, r, dy, ex = norm_inputs(T, H, layer, residual, extra, seed=T + H)
    sms = 2
    grid = norm_grid(T, H, sms, True)
    assert rows_per_owner(T, H, grid) >= 2
    o = norm_ref(a, w, b, r, dy, ex)
    bnd = norm_bounds(o, w, H, T, grid, layer, dy, ex)
    emu = norm_checks(emulate_norm(a, w, b, r, dy, ex, sms), o, bnd, layer, residual)
    caught = {}
    for m in norm_mutants(H, layer, residual, extra):
        c = norm_checks(emulate_norm(a, w, b, r, dy, ex, sms, mutant=m), o, bnd, layer, residual)
        k = max(c, key=c.get)
        caught[m] = (k, c[k])
    return emu, caught


ROPE_CASES = [("rope-d64", 2, 37, 4, 2, 64), ("rope-d128", 3, 11, 4, 1, 128), ("rope-d16", 2, 9, 2, 2, 16)]


def rope_row(name, B, S, Hq, Hk, D):
    g = torch.Generator().manual_seed(S * D)
    n = Hq + 2 * Hk
    x = torch.randn(B * S, n, D, generator=g).to(torch.bfloat16)
    cos, sin = rope_tables64(B * S, D, 500000.0)       # longer than a row, as for the model's max positions
    checks = {}
    per_mut = {m: {} for m in ROPE_MUTANTS}
    for inv in (False, True):
        y64, E = rope_ref(x, cos, sin, Hq + Hk, S, inverse=inv)
        bnd = out_bound(y64, 2 * E)
        key = "inv" if inv else "fwd"
        checks[key] = ratio(emulate_rope(x, cos, sin, S, Hq + Hk, Hq, inverse=inv), y64, bnd)
        for m in ROPE_MUTANTS:
            per_mut[m][key] = ratio(emulate_rope(x, cos, sin, S, Hq + Hk, Hq, inverse=inv, mutant=m), y64, bnd)
    caught = {m: max(c.items(), key=lambda kv: kv[1]) for m, c in per_mut.items()}
    return checks, caught


def act_row(name):
    """SwiGLU over every finite bf16 gate x three up values (forward) and x two dout values (backward); GELU over every finite bf16
    input with two dy values."""
    xs = finite_bf16()
    if name == "swiglu":
        ups = torch.tensor([1.0, -0.75, 3.5], dtype=torch.bfloat16)
        ds = torch.tensor([1.0, -2.5], dtype=torch.bfloat16)
        g = xs.repeat(len(ups) * len(ds))
        u = ups.repeat_interleave(len(xs)).repeat(len(ds))
        d = ds.repeat_interleave(len(xs) * len(ups))
        o = swiglu_ref(g, u, d)

        def chk(e):
            return {k: ratio(e[k], o[k], o["b_" + k]) for k in ("out", "dgate", "dup")}
        return chk(emulate_swiglu(g, u, d)), {"no_g_term": max(chk(emulate_swiglu(g, u, d, "no_g_term")).items(), key=lambda kv: kv[1])}
    ds = torch.tensor([1.0, -0.375], dtype=torch.bfloat16)
    x = xs.repeat(len(ds))
    d = ds.repeat_interleave(len(xs))
    o = gelu_ref(x, d)

    def chk(e):
        return {"y": ratio(e["y"], o["y"], o["b_y"]), "dx": ratio(e["dx"], o["dx"], o["b_dx"])}
    return chk(emulate_gelu(x, d)), {"k1_for_3k1": max(chk(emulate_gelu(x, d, "k1_for_3k1")).items(), key=lambda kv: kv[1])}


CE_CASES = [("ce-50257", 10, 50257, 50304), ("ce-131", 12, 131, 136), ("ce-1000", 10, 1000, 1000)]


def ce_row(name, T, V, Vp):
    lg, lab = ce_inputs(T, V, Vp, seed=V)
    o = ce_ref(lg, lab, V, scale=0.75)
    emu = ce_checks(emulate_ce(lg, lab, V, scale=0.75), o)
    caught = {}
    for m in CE_MUTANTS:
        if m == "pad_in_softmax" and Vp == V:
            continue
        c = ce_checks(emulate_ce(lg, lab, V, scale=0.75, mutant=m), o)
        caught[m] = max(c.items(), key=lambda kv: kv[1])
    return emu, caught


ROWS = {**{c[0]: (lambda c=c: norm_row(*c)) for c in NORM_CASES}, **{c[0]: (lambda c=c: rope_row(*c)) for c in ROPE_CASES},
        "swiglu": lambda: act_row("swiglu"), "gelu": lambda: act_row("gelu"), **{c[0]: (lambda c=c: ce_row(*c)) for c in CE_CASES}}


@pytest.mark.parametrize("name", list(ROWS))
def test_margin_table(name):
    emu, caught = ROWS[name]()
    for k, r in emu.items():
        assert r < 0.5, (name, "emulator", k, r)
    for m, (k, r) in caught.items():
        assert r > 3.0, (name, m, k, r)


def test_every_norm_mutant_has_a_case():
    assert set().union(*(norm_mutants(*c[2:]) for c in NORM_CASES)) == set(NORM_MUTANTS)


def test_former_gelu_tanh_form_cancels_in_the_negative_tail():
    """The former ``0.5 x (1 + tanh(u))`` evaluated in fp32 with a correctly rounded tanh already loses the negative tail to
    cancellation (bound exceeded), before any MUFU.TANH error; the sigmoid form stays within half of the bound."""
    x = finite_bf16()
    x = x[(x.float() < -2) & (x.float() > -9)]
    d = torch.ones_like(x)
    o = gelu_ref(x, d)
    old = emulate_gelu(x, d, form="tanh")
    new = emulate_gelu(x, d)
    assert ratio(new["y"], o["y"], o["b_y"]) < 0.5 and ratio(new["dx"], o["dx"], o["b_dx"]) < 0.5
    assert ratio(old["y"], o["y"], o["b_y"]) > 3.0


if __name__ == "__main__":               # print the margin table: python tests/test_rowwise_oracle.py
    for name, row in ROWS.items():
        emu, caught = row()
        print(f"{name:14s} emulator/bound " + " ".join(f"{k}={v:.3f}" for k, v in emu.items()))
        print(" " * 15 + "mutants " + "  ".join(f"{m}: {k}={r:.3g}" for m, (k, r) in caught.items()))
