"""fp64 oracle of KERNEL A's local arithmetic (``rs_adam_ag_kernel``: stash, scale, AdamW, commit flags, counters; and
``round_norm_kernel``: the norm pass of ``max_grad_norm``), the per-element bounds of its GPU tests (``test_round_kernels_gpu.py``),
and the margin table that shows the bounds are the right size.  Runs on the CPU without the extension.

The oracle is written from the math in the ``optim.py`` docstring, in fp64, with the bias corrections computed from ``step``;
``test_oracle_matches_torch_adamw_fp64`` checks it over several steps against ``torch.optim.AdamW`` with a second, decay-free
parameter group, and ``test_norm_oracle_matches_clip_grad_norm`` checks the norm pass against ``clip_grad_norm_``.

What the binary executes.  ``build_ext.py`` compiles with ``--use_fast_math``: fp32 subnormals are flushed to zero (FTZ) and
division and square root are approximate.  The PTX of every instantiation (``nvcc -ptx`` of ``csrc/rs_adam_ag.cu`` with the
``build_ext.py`` flags; the local and P2P variants of ``rs_adam_ag_kernel`` and ``round_norm_kernel`` list the same
floating-point instructions, the multimem variants add only the switch-side reduction) contains, per element:

=======================================  ==================================================================================
value                                    instruction(s)
=======================================  ==================================================================================
``1 / max(total, 1)`` (in-kernel count)  ``rcp.approx.ftz.f32``
``lr / bc1`` (once per thread)           ``div.approx.ftz.f32``
``1 - lr * wd`` (once per thread)        ``mul.ftz``, ``sub.ftz``
``acc = g (+ stash)``                    ``add.ftz`` (bf16 gradients: ``cvt.f32.bf16``, exact)
``gj = acc * inv``                       ``mul.ftz``
``m' = m + (1 - b1) (gj - m)``           ``sub.ftz`` (``1 - b1``, exact: Sterbenz), ``sub.ftz``, ``fma.rn.ftz``
``v' = b2 v + (1 - b2) gj gj``           ``mul.ftz`` (``b2 v``), ``mul.ftz`` (``(1 - b2) gj``), ``fma.rn.ftz`` (``gj * . + b2 v``)
``denom = sqrt(v') bc2_rsqrt + eps``     ``sqrt.approx.ftz.f32``, ``fma.rn.ftz``
``upd = (lr / bc1) (m' / denom)``        ``div.approx.ftz.f32``, ``mul.ftz``
``p' = p decay - upd``                   ``mul.ftz``, ``sub.ftz`` (``kNoDecay``: ``p * 1`` is exact)
bf16 output                              ``cvt.rn.bf16x2.f32`` (round to nearest even: checked bit for bit, no bound)
norm pass ``sumsq``                      ``fma.rn.ftz`` chain per thread, ``add.ftz`` (butterfly, warps, CTA partials)
``norm``, ``inv_eff``                    ``rcp.approx``, ``sqrt.approx``, ``mul``, ``add`` (``+ 1e-6``), ``div.approx``, ``mul``
=======================================  ==================================================================================

``docs/sass/mnemonics.json`` lists the SASS of a few of these kernels; it counts ``MUFU.SQRT`` only, the PTX above is the
complete list.  Documented errors (PTX ISA, floating-point instructions), ``U = 2^-24`` the fp32 unit roundoff, one ulp at most
``2^-23`` relative: ``div.approx.f32`` 2 ulp for divisors in ``[2^-126, 2^126]`` (``E_DIV = 2^-22``); ``rcp.approx.f32`` 1 ulp
(``E_RCP = 2^-23``); ``sqrt.approx.f32`` ``2^-23`` relative (``E_SQRT``).  ``fma.rn`` rounds once.

The fp32 scalars.  The binding rounds ``lr, b1, b2, eps, wd`` to fp32 and computes ``bc1 = 1 - b1^t`` and
``bc2_rsqrt = 1 / sqrt(1 - b2^t)`` in double before rounding them; the kernel forms ``1 - b1`` and ``1 - b2`` in fp32 from the
rounded betas.  So the kernel solves a slightly different AdamW, and the bound carries the differences as named terms:
``db1 = |f32(b1) - b1|`` times ``|g - m|``, ``db2`` times ``v + g^2``, ``|f32(eps) - eps|``, ``|f32(lr) - lr| / lr`` on the step size
and ``|f32(lr) f32(wd) - lr wd| + U lr wd`` on the decay.  At ``b2 = 0.9999`` the ``db2`` term is ``1.7e-4`` of ``(1 - b2) g^2``,
which makes a step-1 update ``8.3e-5`` relative smaller than ``torch.optim.AdamW``'s (``test_beta2_representation_term``);
far below one bf16 ulp, and kept in the kernel on purpose (its SASS is as measured).

Bounds (first order, doubled so that an honest kernel stays within half; ``e_g = U [stash add] + E_RCP [in-kernel count] + U``
is the relative error of ``gj``, ``FTZ = 2^-125``):

* ``m'``: ``c1 (|g| e_g + U |g - m|) + db1 |g - m| + U |m'| + FTZ`` (the lerp can cancel, so it is relative to its terms);
* ``v'``: ``U b2 v + db2 (v + g^2) + (1 - b2) g^2 (2 e_g + U) + U v' + FTZ``, relative to ``v'`` (every term is non-negative);
* ``denom``: ``bc2r (ds + E_SQRT sqrt(v')) + s U + |f32(eps) - eps| + U denom`` with ``ds`` the error of ``sqrt(v')`` from
  ``v'`` (``min(E_v / 2 sqrt(v'), sqrt(E_v))``) and ``s = sqrt(v') bc2r``;
* ``upd``: ``step_size (E_m / denom + |q| (E_den / denom + E_DIV)) + |upd| (E_DIV + dlr / lr + 2U)``;
* ``master'``: absolute, because ``p decay - upd`` cancels: ``|p| ddec + U |p decay| + E_upd + U |p'| + FTZ``.

The fp32 output equals ``master'`` and the bf16 output ``bf16_rn(master')`` of the same launch, bit for bit; the stash write
is exactly ``f32(acc)``.  Norm pass: a thread adds ``8 n_k`` squares in one ``fma`` chain (``n_k = ceil(nvec / (grid * 256))``),
then 5 butterfly levels, 8 warps in order and ``grid`` CTA partials in order, so ``sumsq`` errs by ``D U sum(acc^2)`` with
``D = 8 n_k + 13 + grid`` (``+ 2U sum(acc^2)`` when the stash is added).  ``norm = sqrt(sumsq) / total`` and ``inv_eff`` are
bounded from the kernel's own ``sumsq``: ``e_n = E_SQRT + E_RCP + U``; the clip coefficient ``min(1, max_norm / (norm + 1e-6))``
errs by ``c (e_n + E_DIV + 2U + representation of max_norm and 1e-6)``, and by nothing when ``c`` is clearly above 1.

The margin table (``test_margin_table``) runs a blockwise fp32 emulator of both kernels in their own operation order
(approximate instructions rounded correctly, FTZ applied) and asserts that it stays within half of every bound, and that each
mutant lands more than 3x outside on at least one check.  Two mutants are below any bound and are caught by exact checks of
the GPU file instead (``NOT_BOUNDED``).  Print the table with ``python tests/test_round_oracle.py``."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import pytest
import torch

from test_gemm_oracle import bf16_rn

U = 2.0 ** -24
FTZ = 2.0 ** -125
E_DIV = 2.0 ** -22
E_RCP = 2.0 ** -23
E_SQRT = 2.0 ** -23
E_DBL = 2.0 ** -40          # the binding's double-precision bias corrections, before their rounding to fp32
COMMIT_NONE, COMMIT_PARAM, COMMIT_STATE, COMMIT_ALL = 0, 1, 2, 3
NORM_THREADS = 256


def f32s(x: float) -> float:
    """A Python float rounded to fp32 (what the binding passes the kernel)."""
    return float(np.float32(x))


def f32(x: torch.Tensor) -> torch.Tensor:
    """Round to fp32 (nearest) and flush subnormals, as the ``.ftz`` instructions do; returned as fp64."""
    y = x.double().float().double()
    return torch.where(y.abs() < 2.0 ** -126, torch.zeros_like(y), y)


def fma(a, b, c) -> torch.Tensor:
    """``fma.rn.ftz.f32``: the product of two fp32 values is exact in fp64, the sum is rounded once (to fp32)."""
    return f32(a * b + c)


@dataclass
class Hyper:
    lr: float = 1e-3
    b1: float = 0.9
    b2: float = 0.95
    eps: float = 1e-8
    wd: float = 0.1
    step: int = 1


@dataclass
class Round:
    """Flags and counters of one round: the commit mode, the stash use and the count the kernel sees."""
    commit: int = COMMIT_ALL
    add_stash: bool = False
    write_stash: bool = False
    local_count: int = 1
    stash_count: int = 0
    inv: Optional[float] = None       # a device inv_count (adamw_shard, or round_norm's inv_eff); None: the in-kernel count


def round_count(rd: Round) -> Tuple[int, int]:
    """The count rule: ``total = local_count + stash_count [add_stash]``; the stash count after the round is ``total`` when the
    stash is written, 0 when it is consumed, else unchanged."""
    total = rd.local_count + (rd.stash_count if rd.add_stash else 0)
    after = total if rd.write_stash else (0 if rd.add_stash else rd.stash_count)
    return total, after


def keep_mask(S: int, ranges: Optional[Sequence[Tuple[int, int]]], base: int = 0, device="cpu") -> torch.Tensor:
    """Elements of the shard ``[base, base + S)`` inside a no-decay range."""
    keep = torch.zeros(S, dtype=torch.bool, device=device)
    for lo, hi in ranges or ():
        keep[max(lo - base, 0):max(min(hi - base, S), 0)] = True
    return keep


# ================================================================================================= oracle
def round_ref(grad, master, m, v, stash, hp: Hyper, rd: Round, keep=None) -> Dict[str, torch.Tensor]:
    """One AdamW round in fp64 from the math (inputs are the fp32 / bf16 values the kernel reads).  Returns the update
    (``m1, v1, p1``: what the round computes whatever the flags), the state after the commit flags (``master, m, v``), the
    stash after the round, the counts, and the intermediates the bounds use."""
    total, stash_count = round_count(rd)
    inv = (1.0 / max(total, 1)) if rd.inv is None else rd.inv
    acc = grad.double() + (stash.double() if rd.add_stash else 0.0)
    g = acc * inv
    m0, v0, p0 = m.double(), v.double(), master.double()
    m1 = hp.b1 * m0 + (1 - hp.b1) * g
    v1 = hp.b2 * v0 + (1 - hp.b2) * g * g
    bc1 = 1 - hp.b1 ** hp.step
    bc2 = 1 - hp.b2 ** hp.step
    denom = torch.sqrt(v1) / math.sqrt(bc2) + hp.eps
    q = m1 / denom
    upd = hp.lr / bc1 * q
    decay = torch.full_like(p0, 1 - hp.lr * hp.wd)
    if keep is not None:
        decay = torch.where(keep, torch.ones_like(decay), decay)
    pdec = p0 * decay
    p1 = pdec - upd
    return {"acc": acc, "g": g, "m0": m0, "v0": v0, "p0": p0, "m1": m1, "v1": v1, "denom": denom, "q": q, "upd": upd,
            "decay": decay, "pdec": pdec, "p1": p1, "total": total, "stash_count": stash_count, "inv": inv,
            "master": p1 if rd.commit & COMMIT_PARAM else p0,
            "m": m1 if rd.commit & COMMIT_STATE else m0, "v": v1 if rd.commit & COMMIT_STATE else v0,
            "stash": acc if rd.write_stash else stash.double()}


def rep_terms(hp: Hyper) -> Dict[str, float]:
    """How far the kernel's fp32 scalars are from the exact hyperparameters (module docstring)."""
    lr, wd = f32s(hp.lr), f32s(hp.wd)
    return {"db1": abs(f32s(hp.b1) - hp.b1), "db2": abs(f32s(hp.b2) - hp.b2), "deps": abs(f32s(hp.eps) - hp.eps),
            "dlr": abs(lr - hp.lr) / hp.lr if hp.lr else 0.0,
            "ddec": abs(lr * wd - hp.lr * hp.wd) + U * hp.lr * hp.wd + U}


def round_bounds(o, hp: Hyper, rd: Round) -> Dict[str, torch.Tensor]:
    """Per-element bounds (doubled) of ``m1``, ``v1``, ``upd`` and ``p1`` (module docstring)."""
    r = rep_terms(hp)
    e_g = (U if rd.add_stash else 0.0) + (E_RCP if rd.inv is None else 0.0) + U
    g, m0, v0, m1, v1 = o["g"], o["m0"], o["v0"], o["m1"], o["v1"]
    ag, d = g.abs(), (g - m0).abs()
    E_m = (1 - hp.b1) * (ag * e_g + U * d) + r["db1"] * d + U * m1.abs() + FTZ
    E_v = U * hp.b2 * v0 + r["db2"] * (v0 + g * g) + (1 - hp.b2) * g * g * (2 * e_g + U) + U * v1 + FTZ
    bc2r = 1 / math.sqrt(1 - hp.b2 ** hp.step)
    sv = torch.sqrt(v1)
    ds = torch.minimum(E_v / (2 * sv).clamp_min(1e-300), torch.sqrt(E_v))
    denom = o["denom"]
    E_den = bc2r * (ds + E_SQRT * sv) + sv * bc2r * (U + E_DBL) + r["deps"] + U * denom
    ss = hp.lr / (1 - hp.b1 ** hp.step)
    E_q = E_m / denom + o["q"].abs() * (E_den / denom + E_DIV)
    E_upd = ss * E_q + o["upd"].abs() * (E_DIV + r["dlr"] + 2 * U + E_DBL)
    ddec = torch.where(o["decay"] == 1, torch.zeros_like(o["p0"]), torch.full_like(o["p0"], r["ddec"]))
    E_p = o["p0"].abs() * ddec + U * o["pdec"].abs() + E_upd + U * o["p1"].abs() + FTZ
    return {"m": 2 * E_m, "v": 2 * E_v, "upd": 2 * E_upd, "p": 2 * E_p}


def ratio(got: torch.Tensor, want: torch.Tensor, bnd: torch.Tensor) -> float:
    """Largest ``|got - want| / bound``; a non-finite ``got`` counts as infinitely wrong unless ``want`` is the same non-finite."""
    got, want = got.double(), want.double()
    err = (got - want).abs()
    same = (got == want) | (torch.isnan(got) & torch.isnan(want))
    err = torch.where(same, torch.zeros_like(err), torch.where(torch.isfinite(err), err, torch.full_like(err, math.inf)))
    return float((err / bnd).max()) if err.numel() else 0.0


def round_checks(got: Dict[str, torch.Tensor], o, bnd) -> Dict[str, float]:
    """Error / bound of the update; exact checks (stash, counts) as 0 or inf."""
    out = {"m": ratio(got["m1"], o["m1"], bnd["m"]), "v": ratio(got["v1"], o["v1"], bnd["v"]), "p": ratio(got["p1"], o["p1"], bnd["p"])}
    if "stash" in got:
        out["stash"] = 0.0 if torch.equal(got["stash"].double(), f32(o["stash"])) else math.inf
    if "total" in got:
        out["total"] = 0.0 if (got["total"], got["stash_count"]) == (o["total"], o["stash_count"]) else math.inf
    return out


# ================================================================================================= emulator
ROUND_MUTANTS = ("eps_in_bc", "bc_t_minus_1", "bc2_not_sqrt", "decay_after", "decay_scaled", "stash_after_scale",
                 "stash_written_scaled", "stash_count_ignored", "v_unscaled")
# Below any bound: the GPU file catches them with exact checks.
NOT_BOUNDED = {
    "bf16_truncated": "below one bf16 ulp; test_round_kernels_gpu.py::test_round_against_bounds asserts out == bf16_rn(master') "
                      "bit for bit",
    "commit_state_writes_master": "the master is then a correct update; test_round_kernels_gpu.py::test_commit_modes_and_stash "
                                  "asserts the master is untouched under COMMIT_STATE",
}


def emulate_round(grad, master, m, v, stash, hp: Hyper, rd: Round, keep=None, mutant: Optional[str] = None):
    """fp32 emulator of one element pass of ``rs_adam_ag_kernel`` (local mode), in its instruction order."""
    lr, b1, b2, eps, wd = (f32s(x) for x in (hp.lr, hp.b1, hp.b2, hp.eps, hp.wd))
    t = hp.step - 1 if mutant == "bc_t_minus_1" else hp.step
    bc1 = f32s(1 - hp.b1 ** t)
    bc2r = f32s(1 / (1 - hp.b2 ** t)) if mutant == "bc2_not_sqrt" else f32s(1 / math.sqrt(1 - hp.b2 ** t))
    total, stash_count = round_count(rd)
    if mutant == "stash_count_ignored":
        total = rd.local_count
        stash_count = total if rd.write_stash else (0 if rd.add_stash else rd.stash_count)
    inv = f32s(1.0 / max(total, 1)) if rd.inv is None else f32s(rd.inv)
    acc = grad.double()
    s = stash.double()
    if rd.add_stash and mutant != "stash_after_scale":
        acc = f32(acc + s)
    gj = f32(acc * inv)
    if rd.add_stash and mutant == "stash_after_scale":
        gj = f32(gj + s)
    stash_out = s
    if rd.write_stash:
        stash_out = gj if mutant == "stash_written_scaled" else acc
    c1, c2 = f32s(1 - b1), f32s(1 - b2)
    m1 = fma(c1, f32(gj - m.double()), m.double())
    gv = acc if mutant == "v_unscaled" else gj
    v1 = fma(gv, f32(c2 * gv), f32(b2 * v.double()))
    sq = f32(torch.sqrt(v1))
    den = f32(f32(sq + eps) * bc2r) if mutant == "eps_in_bc" else fma(sq, bc2r, eps)
    ss = f32s(lr / bc1)
    dec = f32s(1 - f32s(lr * wd))
    if mutant == "decay_scaled":
        dec = f32s(1 - f32s(ss * wd))
    decay = torch.full_like(master.double(), dec)
    if keep is not None:
        decay = torch.where(keep, torch.ones_like(decay), decay)
    u = f32(ss * f32(m1 / den))
    if mutant == "decay_after":
        p1 = f32(f32(master.double() - u) * decay)
    else:
        p1 = f32(f32(master.double() * decay) - u)
    return {"m1": m1, "v1": v1, "p1": p1, "stash": stash_out, "total": total, "stash_count": stash_count}


# ================================================================================================= norm pass
def norm_ref(grad, stash, add_stash: bool, total: int, max_norm: float) -> Dict[str, float]:
    """fp64 norm pass: ``sumsq`` of the unscaled sum, ``norm = sqrt(sumsq) / max(total, 1)``, ``inv_eff = inv * coef`` with
    ``coef = min(1, max_norm / (norm + 1e-6))``; NaN propagates (as ``torch.clamp(max=1)`` in ``clip_grad_norm_``)."""
    acc = grad.double() + (stash.double() if add_stash else 0.0)
    sumsq = float((acc * acc).sum())
    inv = 1.0 / max(total, 1)
    norm = math.sqrt(sumsq) * inv
    c = max_norm / (norm + 1e-6)
    coef = c if (math.isnan(c) or c < 1) else 1.0
    return {"sumsq": sumsq, "norm": norm, "inv_eff": inv * coef, "coef": coef, "inv": inv}


def norm_depth(S: int, grid: int) -> int:
    """Additions a square passes through in ``round_norm_kernel`` (local mode): the thread's ``fma`` chain, the 5-level warp
    butterfly, the 8 warps and the ``grid`` CTA partials."""
    n_k = -(-(S // 8) // (grid * NORM_THREADS))
    return 8 * n_k + 5 + 8 + grid


def norm_bounds(grad, stash, add_stash: bool, total: int, max_norm: float, grid: int, sumsq_k: float) -> Dict[str, float]:
    """Bounds (doubled) of ``sumsq`` against the exact value, and of ``norm`` and ``inv_eff`` against the oracle evaluated on
    the kernel's own ``sumsq_k`` (returned as ``want_norm`` / ``want_inv_eff``)."""
    acc = grad.double() + (stash.double() if add_stash else 0.0)
    sum2 = float((acc * acc).sum())
    D = norm_depth(acc.numel(), grid)
    E_ss = 2 * (D * U * sum2 + (2 * U * sum2 if add_stash else 0.0)) + FTZ
    inv = 1.0 / max(total, 1)
    norm = math.sqrt(sumsq_k) * inv if sumsq_k >= 0 else math.nan
    e_n = E_SQRT + E_RCP + U
    c = max_norm / (norm + 1e-6)
    e_c = e_n * norm / (norm + 1e-6) + 2 * U + E_DIV + abs(f32s(max_norm) - max_norm) / max_norm + abs(f32s(1e-6) - 1e-6) / (norm + 1e-6)
    coef = c if (math.isnan(c) or c < 1) else 1.0
    E_coef = 0.0 if c * (1 - 2 * e_c) > 1 else 2 * c * e_c
    return {"sumsq": E_ss, "norm": 2 * norm * e_n + FTZ, "inv_eff": inv * E_coef + 2 * inv * coef * (E_RCP + U) + FTZ,
            "want_norm": norm, "want_inv_eff": inv * coef}


def emulate_norm(grad, stash, add_stash: bool, total: int, max_norm: float, grid: int, mutant: Optional[str] = None):
    """fp32 emulator of ``round_norm_kernel<G, 0>``: thread ``t`` of the grid owns vectors ``t, t + grid * 256, ...`` (the
    ``kU = 4`` unroll visits them in that order) and chains ``fma(x, x, ss)`` over their elements; then the xor butterfly, the
    8 warps in order, and the last CTA's sum of the partials in CTA order."""
    acc = grad.double()
    if add_stash:
        acc = f32(acc + stash.double())
    S = acc.numel()
    vs = grid * NORM_THREADS
    K = -(-(S // 8) // vs)
    x = torch.zeros(K * vs * 8, dtype=torch.float64)
    x[:S] = acc
    x = x.view(K, vs, 8)
    ss = torch.zeros(vs, dtype=torch.float64)
    for k in range(K):
        for j in range(8):
            ss = fma(x[k, :, j], x[k, :, j], ss)
    w = ss.view(grid, 8, 32)
    for o in (16, 8, 4, 2, 1):
        w = f32(w + w[..., torch.arange(32) ^ o])
    cta = torch.zeros(grid, dtype=torch.float64)
    for k in range(8):
        cta = f32(cta + w[:, k, 0])
    parts = cta[:-1] if mutant == "drop_last_partial" else cta
    s = torch.tensor(0.0, dtype=torch.float64)
    for p in parts:
        s = f32(s + p)
    sumsq = float(s)
    inv = f32s(1.0 / max(total, 1))
    norm = f32s(f32s(math.sqrt(sumsq)) * inv)
    c = f32s(f32s(max_norm) / f32s(norm + f32s(1e-6)))
    coef = 1.0 if c > 1 else c
    return {"sumsq": sumsq, "norm": norm, "inv_eff": f32s(inv * coef)}


def norm_checks(got, grad, stash, add_stash, total, max_norm, grid) -> Dict[str, float]:
    o = norm_ref(grad, stash, add_stash, total, max_norm)
    b = norm_bounds(grad, stash, add_stash, total, max_norm, grid, got["sumsq"])

    def r(a, want, bound):
        if math.isnan(a) and math.isnan(want):
            return 0.0
        return abs(a - want) / bound if math.isfinite(a) else math.inf
    return {"sumsq": r(got["sumsq"], o["sumsq"], b["sumsq"]), "norm": r(got["norm"], b["want_norm"], b["norm"]),
            "inv_eff": r(got["inv_eff"], b["want_inv_eff"], b["inv_eff"])}


# ================================================================================================= inputs
def round_inputs(S: int, gdtype=torch.float32, seed: int = 0, scale: float = 1.0, eps_dominated: bool = False, device="cpu"):
    """Gradient sum ``~ scale N(0, 1)``, stash of the same size, master ``~ 0.02 N(0, 1)``, ``m ~ 0.1 scale N``, ``v ~ scale^2 U(0, 1)``.
    ``eps_dominated``: every other element has ``|g| ~ 1e-9`` and ``v = 0`` (the denominator is ``eps``)."""
    gen = torch.Generator(device=device).manual_seed(seed)
    rn = lambda: torch.randn(S, generator=gen, device=device)
    grad = (rn() * scale).to(gdtype)
    stash = rn() * scale
    master = rn() * 0.02
    m = rn() * 0.1 * scale
    v = torch.rand(S, generator=gen, device=device) * scale * scale
    if eps_dominated:
        tiny = torch.arange(S, device=device) % 2 == 0
        grad = torch.where(tiny, (rn() * 1e-9).to(gdtype), grad)
        stash = torch.where(tiny, rn() * 1e-9, stash)
        m = torch.where(tiny, torch.zeros_like(m), m)
        v = torch.where(tiny, torch.zeros_like(v), v)
    return grad, master, m, v, stash


# ================================================================================================= oracle vs torch
def test_oracle_matches_torch_adamw_fp64():
    """Five committed steps of the oracle (gradient sums of 4 micro-batches, ``inv = 1/4``) equal ``torch.optim.AdamW`` in fp64
    with the no-decay elements in a second parameter group of ``weight_decay = 0``."""
    S = 40
    gen = torch.Generator().manual_seed(1)
    p0 = torch.randn(S, generator=gen, dtype=torch.float64)
    keep = keep_mask(S, [(3, 9), (17, 18), (38, 45)])
    hp0 = Hyper(lr=3e-3, b1=0.9, b2=0.999, eps=1e-8, wd=0.1)
    pa = torch.nn.Parameter(p0[~keep].clone())
    pb = torch.nn.Parameter(p0[keep].clone())
    opt = torch.optim.AdamW([{"params": [pa]}, {"params": [pb], "weight_decay": 0.0}], lr=hp0.lr, betas=(hp0.b1, hp0.b2),
                            eps=hp0.eps, weight_decay=hp0.wd)
    master, m, v = p0.clone(), torch.zeros(S, dtype=torch.float64), torch.zeros(S, dtype=torch.float64)
    for step in range(1, 6):
        gsum = torch.randn(S, generator=gen, dtype=torch.float64) * 4
        pa.grad, pb.grad = (gsum / 4)[~keep].clone(), (gsum / 4)[keep].clone()
        opt.step()
        hp = Hyper(hp0.lr, hp0.b1, hp0.b2, hp0.eps, hp0.wd, step)
        o = round_ref(gsum, master, m, v, torch.zeros(S), hp, Round(local_count=4), keep)
        master, m, v = o["master"], o["m"], o["v"]
        torch.testing.assert_close(master[~keep], pa.detach(), rtol=1e-13, atol=1e-15)
        torch.testing.assert_close(master[keep], pb.detach(), rtol=1e-13, atol=1e-15)
        torch.testing.assert_close(m[~keep], opt.state[pa]["exp_avg"], rtol=1e-13, atol=1e-15)
        torch.testing.assert_close(v[keep], opt.state[pb]["exp_avg_sq"], rtol=1e-13, atol=1e-18)


def test_commit_flags_stash_and_counts():
    """Commit flags select what the state becomes; the stash is written unscaled; the count rule and its transitions."""
    grad, master, m, v, stash = round_inputs(16, seed=2)
    for commit in (COMMIT_NONE, COMMIT_PARAM, COMMIT_STATE, COMMIT_ALL):
        o = round_ref(grad, master, m, v, stash, Hyper(), Round(commit=commit, local_count=3))
        assert torch.equal(o["master"], o["p1"] if commit & 1 else master.double())
        assert torch.equal(o["m"], o["m1"] if commit & 2 else m.double())
        assert torch.equal(o["v"], o["v1"] if commit & 2 else v.double())
    o = round_ref(grad, master, m, v, stash, Hyper(), Round(write_stash=True, local_count=3))
    assert torch.equal(o["stash"], grad.double()) and o["stash_count"] == 3
    o = round_ref(grad, master, m, v, stash, Hyper(), Round(add_stash=True, local_count=3, stash_count=5))
    assert o["total"] == 8 and o["stash_count"] == 0 and o["inv"] == 1 / 8
    torch.testing.assert_close(o["g"], (grad.double() + stash.double()) / 8, rtol=0, atol=0)
    assert round_count(Round(local_count=2, stash_count=7)) == (2, 7)
    assert round_count(Round(local_count=0)) == (0, 0)
    o = round_ref(grad, master, m, v, stash, Hyper(), Round(local_count=0))
    assert o["inv"] == 1.0 and torch.equal(o["g"], grad.double())           # a round with count 0 scales by 1


def test_norm_oracle_matches_clip_grad_norm():
    """``norm`` and ``inv_eff`` against ``clip_grad_norm_`` in fp64 (clipping and not), and NaN propagation."""
    gen = torch.Generator().manual_seed(3)
    grad, stash = torch.randn(64, generator=gen, dtype=torch.float64), torch.randn(64, generator=gen, dtype=torch.float64)
    for add, total, max_norm in ((False, 4, 0.5), (True, 6, 100.0), (True, 1, 1.0)):
        o = norm_ref(grad, stash, add, total, max_norm)
        p = torch.nn.Parameter(torch.zeros(64, dtype=torch.float64))
        p.grad = (grad + (stash if add else 0)) / total
        want = p.grad.clone()
        n = torch.nn.utils.clip_grad_norm_([p], max_norm)
        assert abs(o["norm"] - float(n)) <= 1e-12 * float(n)
        torch.testing.assert_close(p.grad, want * o["inv_eff"] * total, rtol=1e-13, atol=0)
    bad = grad.clone()
    bad[5] = math.nan
    o = norm_ref(bad, stash, False, 2, 1.0)
    assert math.isnan(o["norm"]) and math.isnan(o["inv_eff"])
    z = norm_ref(torch.zeros(64), stash, False, 2, 1.0)
    assert z["norm"] == 0.0 and z["coef"] == 1.0


def test_beta2_representation_term():
    """At ``b2 = 0.9999``, step 1, ``m = v = 0`` and ``|g| >> eps``, the exact update is ``lr sign(g)``; ``1 - f32(b2)`` is
    ``1.7e-4`` relative off ``1 - b2``, so the kernel's update is ``8.3e-5`` relative smaller.  The bound carries exactly that
    (``db2``), and the emulator's deviation is that term and nothing else."""
    hp = Hyper(lr=1e-3, b1=0.9, b2=0.9999, eps=1e-8, wd=0.0, step=1)
    assert abs((1 - f32s(hp.b2)) / (1 - hp.b2) - 1 - 1.66e-4) < 1e-6
    g = torch.tensor([1.0, -1.0, 3.0, -0.25] * 2)
    z = torch.zeros(8)
    o = round_ref(g, z, z, z, z, hp, Round(local_count=1))
    torch.testing.assert_close(o["upd"], hp.lr * g.double() / (g.double().abs() + hp.eps), rtol=1e-12, atol=0)
    e = emulate_round(g, z, z, z, z, hp, Round(local_count=1))
    rel = (-e["p1"] / o["upd"] - 1)
    predicted = math.sqrt((1 - hp.b2) / (1 - f32s(hp.b2))) * (1 - f32s(hp.b1)) / (1 - hp.b1) - 1
    assert -9.5e-5 < predicted < -7e-5
    assert float((rel - predicted).abs().max()) < 8 * U                   # the term, and rounding
    bnd = round_bounds(o, hp, Round(local_count=1))
    assert ratio(e["p1"], o["p1"], bnd["p"]) < 0.5                       # inside the bound because the bound names it
    hp_exact = Hyper(hp.lr, f32s(hp.b1), f32s(hp.b2), hp.eps, 0.0, 1)    # betas that fp32 represents exactly: no deviation left
    assert rep_terms(hp_exact)["db1"] == rep_terms(hp_exact)["db2"] == 0.0
    e2 = emulate_round(g, z, z, z, z, hp_exact, Round(local_count=1))
    assert float((-e2["p1"] / o["upd"] - 1).abs().max()) < 8 * U


# ================================================================================================= margin table
ROUND_CASES = [
    # (name, S, gdtype, hyper, round, eps_dominated, keep ranges, mutants that must land > 3x out)
    ("bf16-step1-b2=0.95-write", 512, torch.bfloat16, Hyper(step=1), Round(commit=COMMIT_NONE, write_stash=True, local_count=4),
     False, None, ("bc2_not_sqrt", "stash_written_scaled", "v_unscaled")),
    ("fp32-step2-add-incount", 512, torch.float32, Hyper(step=2), Round(add_stash=True, local_count=3, stash_count=5),
     False, None, ("bc_t_minus_1", "bc2_not_sqrt", "decay_after", "decay_scaled", "stash_after_scale", "stash_count_ignored",
                   "v_unscaled")),
    ("fp32-step1-eps", 512, torch.float32, Hyper(step=1), Round(local_count=2, inv=0.5), True, None, ("eps_in_bc", "bc2_not_sqrt")),
    ("bf16-step1000-b2=0.999", 512, torch.bfloat16, Hyper(b2=0.999, step=1000), Round(add_stash=True, local_count=2, stash_count=2),
     False, [(5, 77), (300, 301)], ("bc2_not_sqrt", "stash_after_scale", "stash_count_ignored", "v_unscaled")),
    ("fp32-step1e6-nodecay", 512, torch.float32, Hyper(step=10 ** 6, wd=0.1, lr=3e-4), Round(local_count=8),
     False, [(0, 100), (250, 257)], ("v_unscaled",)),
    ("fp32-step1-b2=0.9999", 512, torch.float32, Hyper(b2=0.9999, step=1), Round(local_count=1), False, None, ("bc2_not_sqrt",)),
]

NORM_CASES = [
    # (name, S, gdtype, add_stash, total, max_norm_factor, grid)
    ("norm-bf16-grid3", 8 * 3 * 256 * 2 + 8 * 5, torch.bfloat16, False, 4, 0.5, 3),
    ("norm-fp32-stash-grid7", 8 * 7 * 256 * 3 - 8, torch.float32, True, 6, 2.0, 7),
    ("norm-fp32-grid1", 8 * 256 * 4 + 8, torch.float32, False, 1, 0.999, 1),
]


def round_row(name, S, gdtype, hp, rd, eps_dom, ranges, mutants):
    grad, master, m, v, stash = round_inputs(S, gdtype, seed=S + hp.step, eps_dominated=eps_dom)
    keep = keep_mask(S, ranges) if ranges else None
    o = round_ref(grad, master, m, v, stash, hp, rd, keep)
    bnd = round_bounds(o, hp, rd)
    emu = round_checks(emulate_round(grad, master, m, v, stash, hp, rd, keep), o, bnd)
    caught = {}
    for mu in mutants:
        c = round_checks(emulate_round(grad, master, m, v, stash, hp, rd, keep, mutant=mu), o, bnd)
        k = max(c, key=c.get)
        caught[mu] = (k, c[k])
    return emu, caught


def norm_row(name, S, gdtype, add, total, factor, grid):
    gen = torch.Generator().manual_seed(S)
    grad = (torch.randn(S, generator=gen) * 3).to(gdtype)
    stash = torch.randn(S, generator=gen)
    max_norm = factor * norm_ref(grad, stash, add, total, 1.0)["norm"]
    args = (grad, stash, add, total, max_norm, grid)
    emu = norm_checks(emulate_norm(*args), *args)
    c = norm_checks(emulate_norm(*args, mutant="drop_last_partial"), *args)
    k = max(c, key=c.get)
    return emu, {"drop_last_partial": (k, c[k])}


ROWS = {**{c[0]: (lambda c=c: round_row(*c)) for c in ROUND_CASES}, **{c[0]: (lambda c=c: norm_row(*c)) for c in NORM_CASES}}


@pytest.mark.parametrize("name", list(ROWS))
def test_margin_table(name):
    emu, caught = ROWS[name]()
    for k, r in emu.items():
        assert r < 0.5, (name, "emulator", k, r)
    for mu, (k, r) in caught.items():
        assert r > 3.0, (name, mu, k, r)


def test_every_mutant_has_a_case():
    assert set().union(*(set(c[-1]) for c in ROUND_CASES)) == set(ROUND_MUTANTS)
    assert set(NOT_BOUNDED) == {"bf16_truncated", "commit_state_writes_master"}


def test_bf16_truncation_is_below_the_bound():
    """Why ``bf16_truncated`` needs the exact check: truncating ``master'`` to bf16 errs by less than one bf16 ulp, while an fp32
    bound cannot see the output's rounding mode at all (the output is bf16 of the same ``master'``)."""
    x = torch.randn(4096, dtype=torch.float64) * 0.02
    x32 = f32(x)
    rn = bf16_rn(x32).double()
    rz = (x32.float().view(torch.int32) & ~0xFFFF).view(torch.float32).double()
    assert float((rn - rz).abs().max()) > 0 and bool(((rz - x32).abs() <= x32.abs() * 2.0 ** -7).all())
    assert int((rn != rz).sum()) > 1000                                    # about half the values: the GPU check sees it


if __name__ == "__main__":               # print the margin table: python tests/test_round_oracle.py
    for name, row in ROWS.items():
        emu, caught = row()
        print(f"{name:28s} emulator/bound " + " ".join(f"{k}={v:.3f}" for k, v in emu.items()))
        print(" " * 29 + "mutants " + "  ".join(f"{m}: {k}={r:.3g}" for m, (k, r) in caught.items()))
    for mu, why in NOT_BOUNDED.items():
        print(f"{mu:28s} not bounded: {why}")
