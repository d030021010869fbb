"""An fp64 oracle of the bf16 wgmma GEMM (``csrc/gemm_wgmma.cu``), the operand generators of its exact tier and the tolerances of its
random-operand tier (``test_gemm_oracle_gpu.py``), with the evidence that they are the right size.

What the kernel computes, per output element of ``D[M, N] (+)= A[M, K] B[N, K]^T (+ bias[N])`` on bf16 operands:

* every split of K (``kb_per_split`` 64-deep k-blocks) sums its products in an fp32 register accumulator, one wgmma k16 step at a
  time (the product of two bf16 numbers is exact in fp32);
* one K split: ``v = acc + bias`` (``+ C``, read back in fp32, when accumulating), rounded once to bf16 (round to nearest even);
* several K splits: every split rounds its partial sum (split 0 with the bias) to bf16 and adds it into D with a TMA bf16
  reduce-add.  D holds C (accumulating GEMM) or zeros (a non-accumulating GEMM split along K: the host zero-fills D first).

Exact tier.  Operands whose every intermediate is an integer that both fp32 and bf16 hold exactly make the result independent of
summation order, truncation and split count, so the kernel must equal ``bf16_rn(exact sum)`` bit for bit:

* dense-exact (``dense_exact``): integer entries in [-2, 2], integer bias and C with ``|.| <= 2^10``.  Every partial sum of a split
  is an integer of magnitude ``<= 4 K + 2^11 < 2^24`` (K <= ``K_DENSE_MAX``), exact in fp32 in any order, and the single rounding
  to bf16 at the end is the only one.  Splits = 1 paths only (split partials would be rounded to bf16).  The entries lean positive
  so that partial sums exceed 256 and a kernel that rounds its accumulator to bf16 on the way shows up.
* sparse-exact (``sparse_exact``), for the split-K (atomic) paths: every row of A has at most 64 nonzeros of +-1, with one at the
  first and at the last k of every K split and the rest spread at random; B is in {-1, 0, 1}; C and bias are integers with
  ``|C| <= 64``, ``|bias| <= 32``.  Every split partial, and every running sum of the bf16 reduce-adds, is an integer of magnitude
  ``<= 64 + 32 + 64 = 160 <= 256``: exact in bf16, in any order.

Random tier: bounds against the fp64 result ``y64 = A B^T (+ bias) (+ C)``, with ``S = |A| |B|^T``, ``u = 2^-23`` and
``nk = ceil(K / 16)``.

* Accumulation.  The tensor core's rounding inside a wgmma is not documented; assume only that one k16 step (16 exact products
  added into the accumulator) errs by at most one fp32 ulp per term it adds, in any direction (alignment truncation included).
  The step's own sum then errs by at most ``16 u S_step``, the addition into the accumulator by ``u S``; over the ``nk`` steps
  ``e_acc <= (nk + 16) u S``.  The epilogue's fp32 additions of bias and C add ``2 u (S + |bias| + |C|)``:
  ``e = (nk + 18) u (S + |bias| + |C|)``.
* One split: a single bf16 rounding, allowed one ulp ``2^-7 |v|`` with ``|v| <= |y64| + e`` (twice the half ulp of rounding to
  nearest, so that an honest kernel stays within half of the bound; the ``share`` statistic below is what pins the rounding to
  nearest): ``|y - y64| <= 2^-7 |y64| + (1 + 2^-7) e + 2^-133`` (the last term: the smallest bf16 subnormal).
* ``s`` splits: ``2 s`` bf16 roundings (each split's partial, then its reduce-add into D), each at most one bf16 ulp (``2^-7``
  relative; the rounding mode of the reduce-add is not assumed) of a value bounded by ``R = S + |bias| + |C| + e``:
  ``|y - y64| <= e + ((1 + 2^-7)^(2 s) - 1) R + 2^-133``.

The per-element bound is rigorous and therefore loose: a kernel that rounds its accumulator to bf16 after every k-block stays
inside it.  Two aggregate statistics are sharp enough to require an fp32 accumulator:

* ``share``: the share of elements that differ from ``bf16_rn(y64)`` (one split only).  An fp32 accumulator moves a value across
  a bf16 rounding boundary rarely; rounding the accumulator to bf16 on the way moves most values.  Tolerance ``share_tol(K)``.
* ``rms``: ``||y - y64||_2 / ||y64||_2``, every path.  Tolerance ``rms_tol(splits)``.

The margin table (``test_margin_table``) runs the kernel's arithmetic (``emulate``: fp32 per k16 step, rounded to nearest or toward
zero, one bf16 rounding per split, bf16 reduce-adds) at small shapes of every epilogue path and asserts that it stays within half of
every tolerance, and that each mutant (accumulator rounded to bf16 per k-block, last k-block of a split dropped, bias added by every
split, C added twice, output shifted by one column at a tile edge) lands more than 3x outside on at least one check.  Print it with
``python tests/test_gemm_oracle.py``."""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import pytest
import torch

BM, BK = 128, 64
U = 2.0 ** -23                 # one fp32 ulp, relative
TINY = 2.0 ** -133             # smallest bf16 subnormal
K_DENSE_MAX = 8192             # largest K the GPU exact tier runs on dense-exact operands
K_SPARSE_MAX = 128256          # largest K of the sparse-exact operands (Llama-3 LM-head dgrad)
SPARSE_NNZ = 64


# ---------------------------------------------------------------------------------------------- rounding
def f32(x: torch.Tensor, mode: str = "rn") -> torch.Tensor:
    """fp64 -> nearest fp32 (``rn``) or fp32 toward zero (``rz``), returned as fp64."""
    f = x.float()
    if mode == "rz":
        over = f.double().abs() > x.abs()
        f = torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f)
    return f.double()


def bf16_rn(x: torch.Tensor) -> torch.Tensor:
    """fp64 -> bf16 rounded to nearest even, correctly (round to odd in fp32 first, so the two steps cannot double-round)."""
    f = f32(x, "rz").float()
    inexact = (f.double() != x).to(torch.int32)
    f = (f.view(torch.int32) | inexact).view(torch.float32)
    return f.to(torch.bfloat16)


def logical(a, b, a_mn=False, b_mn=False) -> Tuple[torch.Tensor, torch.Tensor]:
    """The operands as ``A [M, K]`` and ``B [N, K]`` views, whatever their storage."""
    return (a.t() if a_mn else a), (b.t() if b_mn else b)


def split_geometry(K: int, splits: int) -> Tuple[int, int]:
    """(k-blocks per split, effective splits) exactly as the host computes them: no empty split."""
    nk = -(-K // BK)
    splits = max(1, min(splits, nk))
    kbs = -(-nk // splits)
    return kbs, -(-nk // kbs)


# ---------------------------------------------------------------------------------------------- operand generators
_DENSE_VALUES = (-2, -1, 0, 1, 1, 2, 2, 2)      # mean 5/8: partial sums grow past 256 (bf16 loses integers there)


def dense_exact(rows: int, cols: int, seed: int, device="cpu") -> torch.Tensor:
    """bf16 [rows, cols] of integers in [-2, 2], leaning positive."""
    g = torch.Generator(device=device).manual_seed(seed)
    lut = torch.tensor(_DENSE_VALUES, dtype=torch.bfloat16, device=device)
    return lut[torch.randint(0, len(_DENSE_VALUES), (rows, cols), generator=g, device=device)]


def ints(shape, lim: int, seed: int, device="cpu") -> torch.Tensor:
    """bf16 integers in [-lim, lim]."""
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randint(-lim, lim + 1, shape, generator=g, device=device).to(torch.bfloat16)


def sparse_exact(rows: int, K: int, splits: int, seed: int, device="cpu") -> torch.Tensor:
    """bf16 A [rows, K] with at most ``SPARSE_NNZ`` nonzeros of +-1 per row: one at the first and one at the last k of every K split
    (``splits`` as the host makes them), the rest at random in disjoint strata of K.  No index is written twice in one scatter, so
    the result does not depend on the order of the writes (a CUDA scatter with repeated indices would)."""
    kbs, s_eff = split_geometry(K, splits)
    fixed = sorted({k for s in range(s_eff) for k in (s * kbs * BK, min(K, (s + 1) * kbs * BK) - 1)})
    assert len(fixed) <= SPARSE_NNZ
    R = min(SPARSE_NNZ - len(fixed), K)
    g = torch.Generator(device=device).manual_seed(seed)
    base = torch.arange(R, device=device) * K // R                   # strata [base_j, base_j + K // R) are disjoint
    cols = base + torch.randint(0, max(1, K // R), (rows, R), generator=g, device=device)
    sign = lambda n: (torch.randint(0, 2, (rows, n), generator=g, device=device) * 2 - 1).to(torch.bfloat16)
    a = torch.zeros(rows, K, dtype=torch.bfloat16, device=device)
    a.scatter_(1, cols, sign(R))
    a.scatter_(1, torch.tensor(fixed, device=device).expand(rows, -1), sign(len(fixed)))   # overwrites a stratum pick it meets
    return a


def random_operands(M: int, N: int, K: int, seed: int, bias=False, acc=False, device="cpu"):
    """Random tier: A, B ~ N(0, 1) in bf16; bias ~ N(0, K / 4) and C ~ N(0, K), the scales of the product itself."""
    g = torch.Generator(device=device).manual_seed(seed)
    A = torch.randn(M, K, generator=g, device=device).to(torch.bfloat16)
    B = torch.randn(N, K, generator=g, device=device).to(torch.bfloat16)
    bv = (torch.randn(N, generator=g, device=device) * (0.5 * math.sqrt(K))).to(torch.bfloat16) if bias else None
    C = (torch.randn(M, N, generator=g, device=device) * math.sqrt(K)).to(torch.bfloat16) if acc else None
    return A, B, bv, C


# ---------------------------------------------------------------------------------------------- the oracle
def exact_result(A, B, bias=None, C=None, budget: int = 1 << 26) -> torch.Tensor:
    """``bf16_rn(A B^T + bias + C)`` for exact-tier operands, from fp64 sums (exact: integers below 2^53), in chunks of about
    ``budget`` doubles."""
    M, K = A.shape
    N = B.shape[0]
    rm = max(1, min(M, budget // max(K, N)))
    cn = max(1, min(N, budget // K))
    out = torch.empty(M, N, dtype=torch.bfloat16, device=A.device)
    for c0 in range(0, N, cn):
        b = B[c0:c0 + cn].double()
        for r0 in range(0, M, rm):
            y = A[r0:r0 + rm].double() @ b.t()
            if bias is not None:
                y += bias[c0:c0 + cn].double()
            if C is not None:
                y += C[r0:r0 + rm, c0:c0 + cn].double()
            out[r0:r0 + rm, c0:c0 + cn] = bf16_rn(y)
    return out


def bound(y64: torch.Tensor, mag: torch.Tensor, K: int, splits: int) -> torch.Tensor:
    """Per-element error bound (module docstring); ``mag = S + |bias| + |C|``."""
    e = (-(-K // 16) + 18) * U * mag
    if splits == 1:
        return 2.0 ** -7 * y64.abs() + (1 + 2.0 ** -7) * e + TINY
    return e + ((1 + 2.0 ** -7) ** (2 * splits) - 1) * (mag + e) + TINY


def share_tol(K: int) -> float:
    """Largest share of elements allowed to differ from ``bf16_rn(y64)`` on one-split paths.  The fixed 1 % covers fp32 rounding to
    nearest (the emulator moves about 0.1 % of the elements at every K); the K term covers an accumulator that truncates every k16
    step, whose bias grows with the number of steps (the emulator moves 0.6 % at K = 8192, 3.7 % at 50304, 6.2 % at 128256).  Sized
    by the margin table and ``test_share_tolerance_covers_truncation_at_the_largest_k``."""
    return 0.01 + K * 2.0 ** -19


def rms_tol(splits: int) -> float:
    """Largest ``||y - y64|| / ||y64||``: the bf16 rounding of the result, once per split partial and once per reduce-add."""
    return 2.0 ** -8 * math.sqrt(2 * splits - 1)


def check_random(y, A, B, bias=None, C=None, splits: int = 1, budget: int = 1 << 26) -> Dict[str, float]:
    """The random tier over the full output in fp64 chunks (peak extra memory a few ``budget`` doubles): ``bound`` = the largest
    error / bound ratio, ``share`` = mismatch share / ``share_tol`` (one split only), ``rms`` = relative rms error / ``rms_tol``.
    ``C`` is the output's content before the call."""
    M, K = A.shape
    N = B.shape[0]
    rm = max(1, min(M, budget // K, 4096))
    cn = max(1, min(N, budget // K, 4096))
    worst, mism, sq_err, sq_y = 0.0, 0, 0.0, 0.0
    for r0 in range(0, M, rm):
        a = A[r0:r0 + rm].double()
        aa = a.abs()
        for c0 in range(0, N, cn):
            b = B[c0:c0 + cn].double()
            y64 = a @ b.t()
            mag = aa @ b.abs().t()
            del b
            if bias is not None:
                bb = bias[c0:c0 + cn].double()
                y64 += bb
                mag += bb.abs()
            if C is not None:
                cc = C[r0:r0 + rm, c0:c0 + cn].double()
                y64 += cc
                mag += cc.abs()
                del cc
            got = y[r0:r0 + rm, c0:c0 + cn]
            err = (got.double() - y64).abs()
            worst = max(worst, float((err / bound(y64, mag, K, splits)).max()))
            sq_err += float((err * err).sum())
            sq_y += float((y64 * y64).sum())
            if splits == 1:
                mism += int((got.view(torch.int16) != bf16_rn(y64).view(torch.int16)).sum())
            del y64, mag, err
    out = {"bound": worst, "rms": math.sqrt(sq_err / max(sq_y, 1e-300)) / rms_tol(splits)}
    if splits == 1:
        out["share"] = mism / (M * N) / share_tol(K)
    return out


# ---------------------------------------------------------------------------------------------- the kernel's arithmetic
MUTANTS = ("bf16_per_kblock", "drop_last_kblock", "bias_every_split", "c_twice", "shift")


def emulate(A, B, bias=None, C=None, splits: int = 1, accumulate: bool = False, mode: str = "rn", mutant: Optional[str] = None):
    """Blockwise emulator of the kernel: fp32 accumulator per k16 step (``mode`` rn / rz), bias on split 0, C read back in fp32 with
    one split, bf16 partials and bf16 reduce-adds (split order) with several.  ``mutant`` breaks one step (``MUTANTS``)."""
    M, K = A.shape
    N = B.shape[0]
    kbs, splits = split_geometry(K, splits)
    nk = -(-K // BK)
    A64, B64 = A.double(), B.double()
    c64 = C.double() if C is not None else torch.zeros(M, N, dtype=torch.float64)
    if splits > 1:
        D = c64 * (2 if mutant == "c_twice" else 1) if accumulate else torch.zeros(M, N, dtype=torch.float64)
    for s in range(splits):
        kb0, kb1 = s * kbs, min(nk, (s + 1) * kbs)
        if mutant == "drop_last_kblock":
            kb1 -= 1
        acc = torch.zeros(M, N, dtype=torch.float64)
        for kb in range(kb0, kb1):
            for k in range(kb * BK, min(K, kb * BK + BK), 16):
                acc = f32(acc + A64[:, k:k + 16] @ B64[:, k:k + 16].t(), mode)
            if mutant == "bf16_per_kblock":
                acc = bf16_rn(acc).double()
        v = acc
        if bias is not None and (s == 0 or mutant == "bias_every_split"):
            v = f32(v + bias.double(), mode)
        if splits == 1:
            if accumulate:
                v = f32(v + c64, mode)
                if mutant == "c_twice":
                    v = f32(v + c64, mode)
            out = bf16_rn(v)
        else:
            D = bf16_rn(D + bf16_rn(v).double()).double()
    if splits > 1:
        out = D.to(torch.bfloat16)
    if mutant == "shift":                       # the first column of every 64-wide sub-tile takes its left neighbour's value
        out = out.clone()
        out[:, 64::64] = out[:, 63:-1:64][:, :out[:, 64::64].shape[1]]
    return out


# ---------------------------------------------------------------------------------------------- exactness of the generators
def test_bf16_rn_is_correct_rounding():
    """Against the definition: the nearer of the two bf16 neighbours, ties to even; including values where fp64 -> fp32 -> bf16
    by plain casts would round twice."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(20000, generator=g, dtype=torch.float64) * 10.0 ** torch.randint(-6, 6, (20000,), generator=g)
    tie = torch.tensor([1.0 + 2.0 ** -8 + 2.0 ** -30, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(256.0 + 1.0 + 2.0 ** -40)], dtype=torch.float64)
    x = torch.cat([x, tie])
    r = bf16_rn(x).double()
    lo = torch.where(r <= x, r, torch.nextafter(r.to(torch.bfloat16), torch.full_like(r, -math.inf).to(torch.bfloat16)).double())
    hi = torch.where(r >= x, r, torch.nextafter(r.to(torch.bfloat16), torch.full_like(r, math.inf).to(torch.bfloat16)).double())
    assert bool(((x - lo).abs().minimum((hi - x).abs()) == (r - x).abs()).all())
    assert bf16_rn(tie).double().tolist() == [1.0078125, 1.0, 1.015625, -258.0]


@pytest.mark.parametrize("K", [8, 40, 72, 768, K_DENSE_MAX])
def test_dense_exact_partial_sums_fit_fp32(K):
    a, b = dense_exact(64, K, 1), dense_exact(64, K, 2)
    bias, c = ints((64,), 1024, 3), ints((64, 64), 1024, 4)
    assert set(torch.unique(a.float()).tolist()) <= {-2.0, -1.0, 0.0, 1.0, 2.0}
    worst = float(a.double().abs().max() * b.double().abs().max()) * K + 1024 + 1024
    assert worst <= 4 * K + 2048 < 2 ** 24                                 # every partial sum an exact fp32 integer
    y = a.double() @ b.double().t() + bias.double() + c.double()
    assert torch.equal(y, a.float().double() @ b.float().double().t() + bias.double() + c.double())
    if K >= 768:
        assert float((a.double() @ b.double().t()).abs().median()) > 256   # bf16 would lose the partial sums


@pytest.mark.parametrize("K,splits", [(2048, 4), (50304, 4), (K_SPARSE_MAX, 4), (K_SPARSE_MAX, 2), (8192, 16), (200, 3)])
def test_sparse_exact_every_running_sum_fits_bf16(K, splits):
    kbs, s_eff = split_geometry(K, splits)
    a = sparse_exact(32, K, splits, seed=K + splits)
    assert torch.equal(a, sparse_exact(32, K, splits, seed=K + splits))
    b = ints((48, K), 1, seed=1)
    bias, c = ints((48,), 32, 2), ints((32, 48), 64, 3)
    assert int((a != 0).sum(1).max()) <= SPARSE_NNZ and set(torch.unique(a.float()).tolist()) <= {-1.0, 0.0, 1.0}
    parts = torch.zeros(32, 48, dtype=torch.float64)                        # sum over the splits of |partial|, per element
    for s in range(s_eff):
        k0, k1 = s * kbs * BK, min(K, (s + 1) * kbs * BK)
        assert bool((a[:, k0] != 0).all()) and bool((a[:, k1 - 1] != 0).all())     # every split, including its last k-block, is live
        parts += (a[:, k0:k1].double() @ b[:, k0:k1].double().t()).abs()
    bound_run = float(c.abs().max()) + float(bias.abs().max()) + float(parts.max())
    assert bound_run <= 64 + 32 + 64 <= 256                                 # every partial and running sum: an exact bf16 integer
    # the split-wise bf16 sum in any order equals the exact sum
    y = exact_result(a, b, bias, c)
    assert torch.equal(y, emulate(a, b, bias, c, splits, accumulate=True))
    assert torch.equal(exact_result(a, b, bias), emulate(a, b, bias, None, splits))


# ---------------------------------------------------------------------------------------------- the margin table
# (name, M, N, K, splits, bias, accumulate): one small case per epilogue path of the kernel, and the LM-head dgrad's zero-filled
# split-K at its real K on a few rows
CASES = [
    ("store", 256, 192, 768, 1, False, False),
    ("bias", 256, 192, 768, 1, True, False),
    ("beta1", 256, 192, 768, 1, False, True),
    ("beta1-bias", 192, 128, 1088, 1, True, True),
    ("acc-split3", 256, 192, 1536, 3, True, True),
    ("zerofill-split4", 256, 192, 2048, 4, False, False),
    ("zerofill-split4-bias", 256, 192, 2048, 4, True, False),
    ("lmhead-dgrad-split2", 64, 128, 50304, 2, False, False),
]


def case_mutants(splits, bias, acc):
    out = ["bf16_per_kblock", "drop_last_kblock", "shift"]
    if bias and splits > 1:
        out.append("bias_every_split")
    if acc:
        out.append("c_twice")
    return out


def separable(mutant, K, splits) -> bool:
    """Whether a mutant must be caught.  On the split-K paths the kernel itself rounds every split's partial to bf16, and the exact
    tier keeps every partial exact in bf16 by construction, so rounding the accumulator to bf16 per k-block as well only shows once
    a split spans hundreds of k-blocks (the LM-head dgrad: 393 per split at K = 50304)."""
    return not (mutant == "bf16_per_kblock" and splits > 1 and split_geometry(K, splits)[0] < 256)


def margin_row(name, M, N, K, splits, bias, acc):
    """-> (emulator {check: worst ratio over rn / rz}, {mutant: (random-tier check, ratio, exact-tier mismatches)}).  Ratios are
    statistic / tolerance on the random tier (``bound``, ``share``, ``rms``); ``exact`` counts the elements that differ from the
    exact-tier oracle."""
    A, B, bv, C = random_operands(M, N, K, seed=M + N + K + splits, bias=bias, acc=acc)
    if splits == 1:
        eA, eB = dense_exact(M, K, 11), dense_exact(N, K, 12)
        ebv = ints((N,), 1024, 13) if bias else None
        eC = ints((M, N), 1024, 14) if acc else None
    else:
        eA, eB = sparse_exact(M, K, splits, 11), ints((N, K), 1, 12)
        ebv = ints((N,), 32, 13) if bias else None
        eC = ints((M, N), 64, 14) if acc else None
    want = exact_result(eA, eB, ebv, eC)

    def checks(**kw):
        r = check_random(emulate(A, B, bv, C, splits, acc, **kw), A, B, bv, C, splits)
        return r, int((emulate(eA, eB, ebv, eC, splits, acc, **kw) != want).sum())

    emu = {"exact": 0}
    for mode in ("rn", "rz"):
        r, n_bad = checks(mode=mode)
        for k, v in r.items():
            emu[k] = max(emu.get(k, 0.0), v)
        emu["exact"] += n_bad
    caught = {}
    for mut in case_mutants(splits, bias, acc):
        r, n_bad = checks(mutant=mut)
        k = max(r, key=r.get)
        caught[mut] = (k, r[k], n_bad)
    return emu, caught


@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_margin_table(case):
    emu, caught = margin_row(*case)
    assert emu.pop("exact") == 0, case[0]
    for name, r in emu.items():
        assert r < 0.5, (case[0], "emulator", name, r)
    for mut, (check, r, n_bad) in caught.items():
        if separable(mut, case[3], case[4]):
            assert r > 3.0 or n_bad > 0, (case[0], mut, check, r, n_bad)


def test_every_mutant_is_caught_somewhere():
    need = {m for c in CASES for m in case_mutants(*c[4:]) if separable(m, c[3], c[4])}
    assert need == set(MUTANTS)


def test_share_tolerance_covers_truncation_at_the_largest_k():
    """The one-split paths of the fp64 tier reach K = 128256 (the Llama-3 LM-head dgrad at T >= 1024).  An accumulator that truncates
    every k16 step stays within half of ``share_tol`` there too; one that rounds to bf16 per k-block lands more than 3x outside."""
    K = K_SPARSE_MAX
    A, B, _, _ = random_operands(32, 64, K, seed=5)
    r = check_random(emulate(A, B, mode="rz"), A, B)
    assert r["share"] < 0.5 and r["rms"] < 0.5 and r["bound"] < 0.5, r
    bad = check_random(emulate(A, B, mutant="bf16_per_kblock"), A, B)
    assert bad["share"] > 3.0, bad


if __name__ == "__main__":                  # print the margin table: python tests/test_gemm_oracle.py
    for c in CASES:
        emu, caught = margin_row(*c)
        print(f"{c[0]:22s} emulator/tol " + " ".join(f"{k}={v:.3f}" for k, v in emu.items() if k != "exact") + f"  exact mismatches {emu['exact']}")
        print(" " * 23 + "mutants " + "  ".join(f"{m}: {k}={r:.3g} exact={n}" + ("" if separable(m, c[3], c[4]) else " (not separable)")
                                               for m, (k, r, n) in caught.items()))
