"""An fp64 oracle of the FP8 path (``csrc/fp8.cu`` quantiser, ``gemm_fp8_kernel`` in ``csrc/gemm_wgmma.cu``), the operand generators of
its exact tier and the tolerances of its random tier (``test_fp8_oracle_gpu.py``), with the evidence that they are the right size.

The contract, in fp64.

* Quantiser, per tensor ``t`` (bf16) and format ``f`` (``max_e4m3 = 448 = 1.75 * 2^8``, ``max_e5m2 = 57344 = 1.75 * 2^15``):
  ``amax = max |t|``; ``s = 2^k`` with ``k`` the largest integer such that ``amax * 2^k <= max_f``, capped at 127; ``amax = 0`` gives
  ``s = 1``, a NaN / Inf anywhere gives ``s = NaN``; ``1/s`` exactly (``2^-127`` at the cap, an fp32 subnormal);
  ``q = t * s`` rounded to nearest even on the format's grid (``scale64``, ``cast64``).  ``t * s`` never exceeds ``max_f``, so the
  saturation of ``cvt.rn.satfinite`` is never reached.
* GEMM: ``y = A B^T / (s_a s_b) (+ bias) (+ C)`` on the dequantised operands, rounded to bf16 (``y64``).  One named allowance:
  results with ``|y64| < 2^-126`` may come back as +-0 (the build flushes subnormals to zero): ``FLUSH``.

What the kernel computes.  A k-block is ``BKE = 128`` one-byte elements (four ``k32`` wgmma steps).  Each k-block sums into a fresh
tensor-core accumulator that keeps ``ACC_BITS`` significant bits (modelled as truncation toward zero of the running block sum after
every k32 step), and is then promoted: added to the tile's fp32 sum.  Split-K is the host's (``split_geometry``: no empty split).  The
epilogue is ``fma(acc, 1 / (s_a s_b), bias)`` (bias on split 0), ``+ C`` in fp32 with one split, one bf16 rounding; with several splits
every partial is rounded to bf16 and reduce-added into D (C, or zeros).

Exact tier (bit for bit against ``bf16_rn(y64)``):

* ``dense_fp8``: integers in [-2, 2] leaning positive (as ``dense_exact`` of the bf16 oracle) in e4m3 / e5m2, one K split.  A k32
  step's products are integers ``|.| <= 4``; a block's running sum is an integer ``<= 4 * 128 = 512``: ``EXACT_BITS = 10`` bits, which
  the accumulator must keep (``ACC_BITS >= EXACT_BITS``, asserted by the GPU probe); promoted sums are integers ``<= 4 K < 2^24``.  With
  power-of-two scales, bias and C integers times ``1 / (s_a s_b)`` (``|.| <= 1024``), ``fma`` and ``+ C`` are exact and the bf16 rounding
  is the only one.  ``EXACT_SCALES`` has ``s_a s_b != 1`` and ``s_b != 1``, so a kernel that applies one inverse only fails.
* ``sparse_fp8``: +-1 rows with at most 64 nonzeros, one at the first and last k of every split; B in {-1, 0, 1}; bias ``<= 32`` and
  C ``<= 64`` (times the output scale): every split partial and reduce-add is an integer ``<= 160``, exact in bf16 in any order.

Random tier, against ``y64`` with ``S = |A| |B|^T / (s_a s_b)`` and ``nb = ceil(K / 128)`` k-blocks:

* accumulation: each k32 step truncates a running block sum bounded by the block's ``S`` with relative error below ``2^(1 - ACC_BITS)``;
  four steps per block: ``4 * 2^(1 - ACC_BITS) S``.  Promotion adds ``nb`` fp32 roundings of sums below ``S`` and the epilogue two more
  (``fma``, ``+ C``): ``e = (2^(3 - ACC_BITS) + (nb + 2) 2^-24) S + 2^-23 (|bias| + |C|)``.
* one split: ``|y - y64| <= 2^-7 |y64| + (1 + 2^-7) e + FLUSH`` (one bf16 ulp: twice the half ulp, so that an honest kernel stays within
  half of it); ``s`` splits: ``e + ((1 + 2^-7)^(2 s) - 1) (S + |bias| + |C| + e) + FLUSH``.
* ``share``: the share of elements that differ from ``bf16_rn(y64)`` (one split), below ``share_tol(K)``; ``rms``: ``||y - y64|| /
  ||y64||`` below ``rms_tol(splits)``.  These are the sharp checks: the per-element bound also holds for a kernel that never promotes.
  They catch one from ``K = NO_PROMOTION_MIN_K`` on; below that, and on split-K paths, the GPU accumulator probe does.

The margin table (``python tests/test_fp8_oracle.py``) runs ``emulate`` (the blockwise arithmetic above) at small shapes of every
epilogue and both A formats: it stays within half of every tolerance, and every GEMM mutant lands more than 3x outside on at least one
check (``no_promotion``: where ``separable`` says so).  Quantiser mutants are caught by the GPU probes named in ``QUANT_MUTANTS``; ``test_quantiser_mutants_fail_their_probe`` shows
that each of those probes' inputs separates its mutant from the contract."""
from __future__ import annotations

import math
from typing import Dict, Optional

import pytest
import torch

from test_gemm_oracle import bf16_rn, dense_exact, exact_result, ints

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FMT = {E4M3: dict(e_max=8, mbits=3, emin=-6, max=448.0), E5M2: dict(e_max=15, mbits=2, emin=-14, max=57344.0)}
K_MIN = {E4M3: -120, E5M2: -113}        # k of the largest finite bf16 amax (0x7F7F)
BM, BKE, K32 = 128, 128, 32
ACC_BITS = 14                           # significant bits the FP8 tensor-core accumulator keeps (asserted by the GPU probe)
EXACT_BITS = 10                         # bits a dense_fp8 block sum needs: integers <= 4 * 128
FLUSH = 2.0 ** -126                     # |y64| below this may come back as +-0
SPARSE_NNZ = 64
EXACT_SCALES = ((0, 0), (3, -2), (-4, 1), (7, 5))     # (k_a, k_b): s = 2^k


# ---------------------------------------------------------------------------------------------- quantiser contract
def scale64(amax: float, fmt):
    """(s, 1/s) as Python floats: the largest ``2^k`` with ``amax * 2^k <= max_f`` (k <= 127), from the definition."""
    if amax == 0.0:
        return 1.0, 1.0
    if not math.isfinite(amax):
        return math.nan, math.nan
    mx = FMT[fmt]["max"]
    k = math.floor(math.log2(mx / amax))
    while amax * 2.0 ** k > mx:
        k -= 1
    while amax * 2.0 ** (k + 1) <= mx:
        k += 1
    k = min(k, 127)
    return 2.0 ** k, 2.0 ** -k


def bf16_of_bits(bits) -> torch.Tensor:
    return torch.as_tensor(bits, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)


def cast64(x: torch.Tensor, fmt, mode: str = "rn") -> torch.Tensor:
    """fp64 -> the format's grid, round to nearest even (``rn``) or toward zero (``rz``), as fp64.  |x| <= max_f assumed."""
    f = FMT[fmt]
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -200))).clamp_min(f["emin"])
    ulp = torch.pow(2.0, e - f["mbits"])
    r = x / ulp
    r = torch.round(r) if mode == "rn" else torch.trunc(r)       # torch.round: half to even
    return r * ulp


def quantize64(t: torch.Tensor, fmt, mode="rn"):
    """-> (q as fp64 values, s, 1/s, amax) of the contract."""
    amax = float(t.float().abs().max())
    s, inv = scale64(amax, fmt)
    return cast64(t.double() * s, fmt, mode), s, inv, amax


def amax_ctas(n: int, sms: int) -> int:
    """Twin of ``acco_fp8_amax_ctas``: CTAs of ``fp8_amax_kernel`` for ``n`` elements."""
    g = (n // 8 + 1023) // 1024
    return max(1, min(g, 2 * sms, 1024))


def amax_emulate(t: torch.Tensor, ctas: int, mutant: Optional[str] = None) -> int:
    """bf16 bits of the amax ``fp8_amax_kernel`` finds: vector ``v`` (8 elements) is read by thread ``v % (256 ctas)`` in pass
    ``v // (256 ctas)``.  Mutants: ``amax_last_pass`` skips every thread's last pass, ``amax_high_half`` ignores the high bf16 of each
    32-bit word (the odd elements)."""
    bits = t.contiguous().view(torch.int16).flatten().to(torch.int64) & 0x7FFF
    n8 = bits.numel() // 8
    stride = 256 * ctas
    keep = torch.ones_like(bits, dtype=torch.bool)
    if mutant == "amax_last_pass":
        v = torch.arange(n8)
        thread = v % stride
        last = (n8 - 1 - thread) // stride                 # the last pass of each vector's thread
        keep &= (v // stride != last).repeat_interleave(8)
    if mutant == "amax_high_half":
        keep[1::2] = False
    return int(torch.where(keep, bits, torch.zeros_like(bits)).max())


def scale_rule_mutant(amax_bits: int, fmt, mutant: str):
    """The kernel's rule (``scale_from_amax``) with one change: ``ge_0x60`` (``mant7 >= 0x60``) or ``cap_126``."""
    e_max = FMT[fmt]["e_max"]
    if amax_bits == 0:
        return 1.0
    ex, man = amax_bits >> 7, amax_bits & 0x7F
    if ex == 0:
        lead = man.bit_length() - 1
        e, mant7 = -133 + lead, (man << (7 - lead)) & 0x7F
    else:
        e, mant7 = ex - 127, man
    k = e_max - e - ((mant7 >= 0x60) if mutant == "ge_0x60" else (mant7 > 0x60))
    return 2.0 ** min(k, 126 if mutant == "cap_126" else 127)


def cast_set(fmt, k: int) -> torch.Tensor:
    """bf16 [R, 256] for ``test_cast_every_k``: every non-negative bf16 value whose image under ``s = 2^k`` lies in the format's range,
    with both signs, padded with zeros; its amax makes the rule pick exactly ``k``."""
    mx = FMT[fmt]["max"]
    top = torch.tensor(mx * 2.0 ** -k, dtype=torch.float64).clamp(max=3.3e38).to(torch.float32).to(torch.bfloat16)
    while float(top) * 2.0 ** k > mx:                         # round down onto the bf16 grid
        top = bf16_of_bits(int(top.view(torch.int16)) - 1)
    hi = int(top.view(torch.int16))
    pos = bf16_of_bits(torch.arange(0, hi + 1))
    vals = torch.cat([pos, -pos])
    n = -(-vals.numel() // 4096) * 4096
    out = torch.zeros(n, dtype=torch.bfloat16)
    out[:vals.numel()] = vals
    return out.view(-1, 256)


def cast_ks(fmt):
    return range(K_MIN[fmt], 128)


def planted_positions(n: int, ctas: int):
    """Element indices of the GPU amax probe: each of the 8 lanes of a 16-byte vector at the first vector, at the CTA boundaries
    (vectors 255 / 256), at the grid-stride boundary (256 ctas - 1 / 256 ctas), in the last pass, and the last element."""
    stride = 256 * ctas
    n8 = n // 8
    vecs = sorted({0, 255, 256, stride - 1, stride, n8 - stride, n8 - 1})
    pos = [v * 8 + lane for v in vecs if 0 <= v < n8 for lane in range(8)]
    return sorted(set(pos + [n - 1]))


# Quantiser mutants -> the GPU check that catches each
QUANT_MUTANTS = {
    "ge_0x60": "test_fp8_oracle_gpu.py::test_scale_rule_every_bf16_amax",
    "cap_126": "test_fp8_oracle_gpu.py::test_scale_rule_every_bf16_amax",
    "cast_rz": "test_fp8_oracle_gpu.py::test_cast_every_k_every_value",
    "amax_last_pass": "test_fp8_oracle_gpu.py::test_amax_planted_values",
    "amax_high_half": "test_fp8_oracle_gpu.py::test_amax_planted_values",
}
GEMM_PROBES = {"no_promotion": "test_fp8_oracle_gpu.py::test_accumulator_width (below NO_PROMOTION_MIN_K and on split-K paths)"}
PLANT_SHAPE = (4160, 528)               # 274,560 vectors of 8: 264 CTAs on 132 SMs stride 67,584 vectors, 4.06 passes


# ---------------------------------------------------------------------------------------------- GEMM geometry and generators
def split_geometry(K: int, splits: int):
    """(k-blocks per split, effective splits) as the host computes them for FP8 (128-element k-blocks): no empty split."""
    nk = -(-K // BKE)
    splits = max(1, min(splits, nk))
    kbs = -(-nk // splits)
    return kbs, -(-nk // kbs)


def scales(k: int, device="cpu") -> torch.Tensor:
    """The scale tensor the quantiser writes for ``s = 2^k``: {s, 1/s, amax} (amax unused by the GEMM)."""
    return torch.tensor([2.0 ** k, 2.0 ** -k, 1.0], dtype=torch.float32, device=device)


def dense_fp8(rows, K, seed, fmt, device="cpu"):
    return dense_exact(rows, K, seed, device).to(fmt)


def sparse_fp8(rows, K, splits, seed, fmt, device="cpu"):
    """+-1 rows with at most ``SPARSE_NNZ`` nonzeros, one at the first and the last k of every K split (FP8 geometry), the rest at random
    in disjoint strata; no index written twice."""
    kbs, s_eff = split_geometry(K, splits)
    fixed = sorted({k for s in range(s_eff) for k in (s * kbs * BKE, min(K, (s + 1) * kbs * BKE) - 1)})
    R = min(SPARSE_NNZ - len(fixed), K)
    g = torch.Generator(device=device).manual_seed(seed)
    base = torch.arange(R, device=device) * K // R
    cols = base + torch.randint(0, max(1, K // R), (rows, R), generator=g, device=device)
    sign = lambda n: (torch.randint(0, 2, (rows, n), generator=g, device=device) * 2 - 1).to(torch.bfloat16)
    a = torch.zeros(rows, K, dtype=torch.bfloat16, device=device)
    a.scatter_(1, cols, sign(R))
    a.scatter_(1, torch.tensor(fixed, device=device).expand(rows, -1), sign(len(fixed)))
    return a.to(fmt)


def exact_operands(M, N, K, fmt, splits, bias, acc, ka, kb, seed, device="cpu", shift=(0, 0)):
    """(A, B, s_a, s_b, bias, C) of the exact tier: dense for one split, sparse for several; bias and C on the output's grid.
    ``shift = (j_a, j_b)`` multiplies the A and B entries by ``2^j_a`` and ``2^j_b`` (still exact in their formats for
    ``-8 <= j <= 7``): every sum keeps its significant bits, so the exactness above holds unchanged, and the output grid moves by
    ``2^(j_a + j_b)``.  That keeps bias, C, every split partial and the result normal numbers at scale pairs whose product
    ``1 / (s_a s_b)`` lies outside fp32's normal range."""
    post = 2.0 ** (-ka - kb + shift[0] + shift[1])
    if splits == 1:
        A, B = dense_fp8(M, K, seed, fmt, device), dense_fp8(N, K, seed + 1, E4M3, device)
        bl, cl = 1024, 1024
    else:
        A, B = sparse_fp8(M, K, splits, seed, fmt, device), ints((N, K), 1, seed + 1, device).to(E4M3)
        bl, cl = 32, 64
    if shift != (0, 0):
        A = (A.float() * 2.0 ** shift[0]).to(fmt)
        B = (B.float() * 2.0 ** shift[1]).to(E4M3)
    bv = (ints((N,), bl, seed + 2, device).double() * post).to(torch.bfloat16) if bias else None
    C = (ints((M, N), cl, seed + 3, device).double() * post).to(torch.bfloat16) if acc else None
    return A, B, scales(ka, device), scales(kb, device), bv, C


def exact_fp8(A, B, sa, sb, bias=None, C=None):
    """``bf16_rn(y64)`` for exact-tier operands (fp64 sums of exact products)."""
    return exact_result(A.double() * float(sa[1]), B.double() * float(sb[1]), bias, C)


def random_fp8(M, N, K, fmt, seed, bias=False, acc=False, device="cpu"):
    """Random tier: A = q(N(0, 1)) in ``fmt``, B = q(N(0, 0.05^2)) in e4m3 with the quantiser's scales; bias and C at the product's
    scale (``0.05 sqrt(K)``)."""
    from acco_b200.ops.fp8 import quantize_ref
    g = torch.Generator(device=device).manual_seed(seed)
    a = torch.randn(M, K, generator=g, device=device).to(torch.bfloat16)
    b = (torch.randn(N, K, generator=g, device=device) * 0.05).to(torch.bfloat16)
    A, _, sa = quantize_ref(a, fmt)
    B, _, sb = quantize_ref(b, E4M3)
    sc = 0.05 * math.sqrt(K)
    bv = (torch.randn(N, generator=g, device=device) * 0.5 * sc).to(torch.bfloat16) if bias else None
    C = (torch.randn(M, N, generator=g, device=device) * sc).to(torch.bfloat16) if acc else None
    return A, B, sa, sb, bv, C


# ---------------------------------------------------------------------------------------------- bounds and statistics
def bound(y64, S, mag, K, splits):
    """Per-element bound (module docstring); ``S`` scaled, ``mag = S + |bias| + |C|``."""
    nb = -(-K // BKE)
    e = (2.0 ** (3 - ACC_BITS) + (nb + 2) * 2.0 ** -24) * S + 2.0 ** -23 * (mag - S)
    if splits == 1:
        return 2.0 ** -7 * y64.abs() + (1 + 2.0 ** -7) * e + FLUSH
    return e + ((1 + 2.0 ** -7) ** (2 * splits) - 1) * (mag + e) + FLUSH


def share_tol(K: int) -> float:
    """Largest share of one-split elements that may differ from ``bf16_rn(y64)``.  The promoted accumulator truncated to ``ACC_BITS``
    (``emulate``) moves 4 to 5.5 % of them at every K from 768 to 28672; one that never promotes moves 37 % at K = 2048, 59 % at 4096
    and over 90 % from 14336 on.  The per-block truncation does not grow with K, so neither does the tolerance."""
    return 0.12


def rms_tol(splits: int) -> float:
    """Largest ``||y - y64|| / ||y64||``: bf16 rounding of the result, once per split partial and reduce-add, plus the promoted
    accumulator's truncation, which is well below it."""
    return 2.0 ** -8 * math.sqrt(2 * splits - 1)


def check_random(y, A, B, sa, sb, bias=None, C=None, splits=1, budget=1 << 26) -> Dict[str, float]:
    """Random tier over the full output in fp64 chunks: ``bound`` = largest error / bound, ``share`` = mismatch share / ``share_tol``
    (one split), ``rms`` = relative rms error / ``rms_tol``.  ``C`` is the output's content before the call."""
    M, K = A.shape
    N = B.shape[0]
    ia, ib = float(sa[1]), float(sb[1])
    rm = max(1, min(M, budget // K, 4096))
    cn = max(1, min(N, budget // K, 4096))
    worst, mism, sq_err, sq_y = 0.0, 0, 0.0, 0.0
    for r0 in range(0, M, rm):
        a = A[r0:r0 + rm].double() * ia
        aa = a.abs()
        for c0 in range(0, N, cn):
            b = B[c0:c0 + cn].double() * ib
            y64 = a @ b.t()
            S = aa @ b.abs().t()
            mag = S.clone()
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
            worst = max(worst, float((err / bound(y64, S, mag, K, splits)).max()))
            sq_err += float((err * err).sum())
            sq_y += float((y64 * y64).sum())
            if splits == 1:
                mism += int((got.view(torch.int16) != bf16_rn(y64).view(torch.int16)).sum())
            del y64, S, mag, err
    out = {"bound": worst, "rms": math.sqrt(sq_err / max(sq_y, 1e-300)) / rms_tol(splits)}
    if splits == 1:
        out["share"] = mism / (M * N) / share_tol(K)
    return out


# ---------------------------------------------------------------------------------------------- the kernel's arithmetic
MUTANTS = ("no_promotion", "drop_tail", "one_inverse", "scale_twice", "e5m2_as_e4m3", "bias_every_split", "c_twice", "shift",
           "out_scale_flush")


def trunc_bits(x: torch.Tensor, bits: int) -> torch.Tensor:
    """Truncate toward zero to ``bits`` significant bits (fp64 in, fp64 out)."""
    m, e = torch.frexp(x)
    return torch.ldexp(torch.trunc(torch.ldexp(m, torch.full_like(e, bits))), e - bits)


def f32(x: torch.Tensor) -> torch.Tensor:
    return x.float().double()


def f32_ftz(v: float) -> float:
    """A float as the fast-math build reads it: subnormals are 0."""
    return 0.0 if abs(v) < 2.0 ** -126 else v


def emulate(A, B, sa, sb, bias=None, C=None, splits=1, accumulate=False, bits=ACC_BITS, mutant=None):
    """Blockwise emulator of the FP8 kernel (module docstring).  ``mutant`` breaks one step (``MUTANTS``)."""
    M, K = A.shape
    N = B.shape[0]
    kbs, splits = split_geometry(K, splits)
    nk = -(-K // BKE)
    if mutant == "e5m2_as_e4m3" and A.dtype == E5M2:
        A = A.view(torch.uint8).view(E4M3)
    A64, B64 = A.double(), B.double()
    Klive = (K // BKE) * BKE if mutant == "drop_tail" and K % BKE else K
    ia, ib = float(sa[1]), float(sb[1])
    post = {"one_inverse": ia, "scale_twice": (ia * ib) ** 2}.get(mutant, ia * ib)
    if mutant == "out_scale_flush":
        post = f32_ftz(f32_ftz(ia) * f32_ftz(ib))
    c64 = C.double() if C is not None else torch.zeros(M, N, dtype=torch.float64)
    if splits > 1:
        D = c64 * (2 if mutant == "c_twice" else 1) if accumulate else torch.zeros(M, N, dtype=torch.float64)
    for s in range(splits):
        acc = torch.zeros(M, N, dtype=torch.float64)
        blk = torch.zeros(M, N, dtype=torch.float64)
        for kb in range(s * kbs, min(nk, (s + 1) * kbs)):
            if mutant != "no_promotion":
                blk = torch.zeros(M, N, dtype=torch.float64)
            for k in range(kb * BKE, min(Klive, kb * BKE + BKE), K32):
                blk = trunc_bits(blk + A64[:, k:k + K32] @ B64[:, k:k + K32].t(), bits)
            if mutant != "no_promotion":
                acc = f32(acc + blk)
        if mutant == "no_promotion":
            acc = f32(blk)
        v = acc * post
        if bias is not None and (s == 0 or mutant == "bias_every_split"):
            v = v + bias.double()
        v = f32(v)                                           # fma: one rounding
        if splits == 1:
            if accumulate:
                v = f32(v + c64)
                if mutant == "c_twice":
                    v = f32(v + c64)
            out = bf16_rn(v)
        else:
            D = bf16_rn(D + bf16_rn(v).double()).double()
    if splits > 1:
        out = D.to(torch.bfloat16)
    if mutant == "shift":
        out = out.clone()
        out[:, 64::64] = out[:, 63:-1:64][:, :out[:, 64::64].shape[1]]
    return out


# ---------------------------------------------------------------------------------------------- quantiser contract tests
@pytest.mark.parametrize("fmt", [E4M3, E5M2], ids=["e4m3", "e5m2"])
def test_scale_ref_is_the_definition_at_every_bf16_amax(fmt):
    from acco_b200.ops.fp8 import scale_ref
    bits = torch.arange(0, 0x7F80)
    amax = bf16_of_bits(bits).float()
    s, inv = scale_ref(amax, fmt)
    want = [scale64(float(a), fmt) for a in amax.tolist()]
    assert s.double().tolist() == [w[0] for w in want]
    assert inv.double().tolist() == [w[1] for w in want]
    assert float(inv[1]) == 2.0 ** -127 and float(s[1]) == 2.0 ** 127            # the cap, reached by bf16 subnormals
    assert int(torch.log2(s[-1])) == K_MIN[fmt]


@pytest.mark.parametrize("fmt", [E4M3, E5M2], ids=["e4m3", "e5m2"])
def test_quantize_ref_is_rne_on_the_format_grid(fmt):
    """``quantize_ref`` (torch's float8 casts) against ``cast64``, on every value set the GPU cast test uses, at a third of the k."""
    from acco_b200.ops.fp8 import quantize_ref
    for k in list(cast_ks(fmt))[::3] + [127]:
        t = cast_set(fmt, k)
        q, s, inv, _ = quantize64(t, fmt)
        assert s == 2.0 ** k
        rq, _, rs = quantize_ref(t, fmt)
        assert float(rs[0]) == s and float(rs[1]) == inv
        assert torch.equal(rq.double(), q), k
        assert float(q.abs().max()) <= FMT[fmt]["max"]


def test_quantiser_mutants_fail_their_probe():
    """Every quantiser mutant differs from the contract on the inputs of the GPU probe named for it in ``QUANT_MUTANTS``."""
    assert set(QUANT_MUTANTS) == {"ge_0x60", "cap_126", "cast_rz", "amax_last_pass", "amax_high_half"}
    for fmt in (E4M3, E5M2):
        diff = {m: [b for b in range(0x7F80) if scale_rule_mutant(b, fmt, m) != scale64(float(bf16_of_bits(b)), fmt)[0]]
                for m in ("ge_0x60", "cap_126")}
        assert diff["ge_0x60"] and all(b & 0x7F == 0x60 or (b >> 7 == 0) for b in diff["ge_0x60"])
        assert diff["cap_126"] and all(scale64(float(bf16_of_bits(b)), fmt)[0] == 2.0 ** 127 for b in diff["cap_126"])
        t = cast_set(fmt, 0)
        assert not torch.equal(quantize64(t, fmt, "rz")[0], quantize64(t, fmt)[0])
    n = PLANT_SHAPE[0] * PLANT_SHAPE[1]
    ctas = amax_ctas(n, 132)
    assert n // 8 > 256 * ctas                                 # the grid-stride loop wraps
    base = torch.full((n,), 0.25, dtype=torch.bfloat16)
    missed = {m: 0 for m in ("amax_last_pass", "amax_high_half")}
    for p in planted_positions(n, ctas):
        t = base.clone()
        t[p] = 3.0
        for m in missed:
            missed[m] += amax_emulate(t, ctas, m) != amax_emulate(t, ctas)
        assert amax_emulate(t, ctas) == 0x4040
    assert all(v > 0 for v in missed.values()), missed


# ---------------------------------------------------------------------------------------------- GEMM generators
@pytest.mark.parametrize("K", [16, 112, 784, 1040, 8192])
def test_dense_fp8_is_exact_in_every_accumulator(K):
    A, B = dense_fp8(64, K, 1, E5M2), dense_fp8(48, K, 2, E4M3)
    assert torch.equal(A.double(), dense_exact(64, K, 1).double())      # the integers survive both formats
    assert ACC_BITS >= EXACT_BITS and 4 * BKE <= 2 ** EXACT_BITS and 4 * K < 2 ** 24
    for ka, kb in EXACT_SCALES:
        sa, sb = scales(ka), scales(kb)
        assert torch.equal(emulate(A, B, sa, sb, bits=EXACT_BITS), exact_fp8(A, B, sa, sb))
    assert any(ka + kb != 0 and kb != 0 for ka, kb in EXACT_SCALES)
    if K >= 784:
        assert float((A.double() @ B.double().t()).abs().median()) > 256


@pytest.mark.parametrize("splits", [1, 3])
@pytest.mark.parametrize("shift,scale", [((7, 7), (127, 1)), ((-8, -8), (-60, -70))])
def test_shifted_operands_stay_exact_at_out_of_range_scales(shift, scale, splits):
    """The operand shift of ``exact_operands``: the values are those of the unshifted generator times ``2^j``, the emulator (with its
    exponent-aware scale) still equals the oracle, and bias, C and the result are normal bf16 numbers where they are not zero, though
    ``1 / (s_a s_b)`` (2^-128, 2^130) is outside fp32's normal range."""
    for fmt in (E4M3, E5M2):
        A, B, sa, sb, bv, C = exact_operands(65, 72, 1040, fmt, splits, True, True, *scale, seed=3, shift=shift)
        A0, B0 = exact_operands(65, 72, 1040, fmt, splits, False, False, 0, 0, seed=3)[:2]
        assert torch.equal(A.double(), A0.double() * 2.0 ** shift[0]) and torch.equal(B.double(), B0.double() * 2.0 ** shift[1])
        post = float(sa[1]) * float(sb[1])
        assert not 2.0 ** -126 <= post < 2.0 ** 128
        want = exact_fp8(A, B, sa, sb, bv, C)
        for t in (bv, C, want):
            nz = t.float() != 0
            assert bool((t.float().abs()[nz] >= 2.0 ** -126).all() and torch.isfinite(t.float()).all())
        assert torch.equal(emulate(A, B, sa, sb, bv, C, splits, accumulate=True), want)


@pytest.mark.parametrize("K,splits", [(1040, 3), (4096, 4), (8192, 16), (144, 2)])
def test_sparse_fp8_every_partial_is_exact_in_bf16(K, splits):
    kbs, s_eff = split_geometry(K, splits)
    A = sparse_fp8(32, K, splits, K, E5M2)
    B = ints((40, K), 1, 1).to(E4M3)
    for ka, kb in EXACT_SCALES:
        _, _, sa, sb, bv, C = exact_operands(32, 40, K, E5M2, splits, True, True, ka, kb, seed=K)
        for s in range(s_eff):
            k0, k1 = s * kbs * BKE, min(K, (s + 1) * kbs * BKE)
            assert bool((A[:, k0].float() != 0).all()) and bool((A[:, k1 - 1].float() != 0).all())
        want = exact_fp8(A, B, sa, sb, bv, C)
        assert torch.equal(emulate(A, B, sa, sb, bv, C, splits, accumulate=True), want)
        assert torch.equal(emulate(A, B, sa, sb, bv, None, splits), exact_fp8(A, B, sa, sb, bv))


# ---------------------------------------------------------------------------------------------- the margin table
# (name, M, N, K, A format, splits, bias, accumulate)
CASES = [
    ("store", 192, 136, 784, E4M3, 1, False, False),
    ("bias", 200, 200, 1040, E4M3, 1, True, False),
    ("beta1", 129, 136, 1024, E5M2, 1, False, True),
    ("beta1-bias", 65, 200, 784, E5M2, 1, True, True),
    ("acc-split3", 128, 136, 1552, E5M2, 3, True, True),
    ("zerofill-split2", 128, 136, 1040, E4M3, 2, False, False),
    ("zerofill-split2-bias", 128, 136, 1040, E5M2, 2, True, False),
    ("store-long", 64, 136, 4112, E5M2, 1, False, False),
]
NO_PROMOTION_MIN_K = 4096               # from here on a kernel that never promotes is > 3x outside ``share`` (one split)
EXTREME = (127, 1)                      # (k_a, k_b) of the out_scale_flush probe: 1 / s_a = 2^-127, a subnormal


def case_mutants(fmt, K, splits, bias, acc):
    out = ["no_promotion", "one_inverse", "scale_twice", "shift"]
    if K % BKE:
        out.append("drop_tail")
    if fmt == E5M2:
        out.append("e5m2_as_e4m3")
    if bias and splits > 1:
        out.append("bias_every_split")
    if acc:
        out.append("c_twice")
    return out


def margin_row(name, M, N, K, fmt, splits, bias, acc):
    """-> (emulator {check: ratio}, {mutant: (check, ratio, exact-tier mismatches)})."""
    A, B, sa, sb, bv, C = random_fp8(M, N, K, fmt, seed=M + N + K, bias=bias, acc=acc)
    ka, kb = EXACT_SCALES[(M + K) % len(EXACT_SCALES)]
    if (ka, kb) == (0, 0):
        ka, kb = EXACT_SCALES[1]
    eA, eB, esa, esb, ebv, eC = exact_operands(M, N, K, fmt, splits, bias, acc, ka, kb, seed=11)
    want = exact_fp8(eA, eB, esa, esb, ebv, eC)

    def checks(**kw):
        r = check_random(emulate(A, B, sa, sb, bv, C, splits, acc, **kw), A, B, sa, sb, bv, C, split_geometry(K, splits)[1])
        return r, int((emulate(eA, eB, esa, esb, ebv, eC, splits, acc, **kw) != want).sum())

    r, n_bad = checks()
    emu = dict(r, exact=n_bad)
    caught = {}
    for mut in case_mutants(fmt, K, splits, bias, acc):
        r, n_bad = checks(mutant=mut)
        k = max(r, key=r.get)
        caught[mut] = (k, r[k], n_bad)
    return emu, caught


def extreme_row():
    """The out_scale_flush mutant on the scale-edge probe: 1/s_a = 2^-127 read as 0 by a flushing multiply."""
    A, B = dense_fp8(64, 136, 5, E4M3), dense_fp8(72, 136, 6, E4M3)
    sa, sb = scales(EXTREME[0]), scales(EXTREME[1])
    want = exact_fp8(A, B, sa, sb)
    normal = want.float().abs() >= 2.0 ** -126
    assert int(normal.sum()) > 0.9 * want.numel()
    good = int((emulate(A, B, sa, sb) != want)[normal].sum())
    bad = int((emulate(A, B, sa, sb, mutant="out_scale_flush") != want)[normal].sum())
    return good, bad


@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_margin_table(case):
    emu, caught = margin_row(*case)
    assert emu.pop("exact") == 0, case[0]
    for k, r in emu.items():
        assert r <= 0.5, (case[0], "emulator", k, r)
    for mut, (check, r, n_bad) in caught.items():
        if separable(mut, case[3], case[5]):
            assert r > 3.0 or n_bad > 0, (case[0], mut, check, r, n_bad)


def separable(mutant, K, splits) -> bool:
    """Whether a mutant must be caught by the checks of this file.  A kernel that never promotes keeps every exact-tier block exact
    (``EXACT_BITS <= ACC_BITS``) and, below ``NO_PROMOTION_MIN_K`` or split along K, stays too close to an honest one for the random
    statistics; there ``test_fp8_oracle_gpu.py::test_accumulator_width`` catches it: a small product in the k-block after a large one
    must survive to fp32 precision."""
    return not (mutant == "no_promotion" and (splits > 1 or K < NO_PROMOTION_MIN_K))


def test_extreme_scale_probe_catches_a_flushed_scale():
    good, bad = extreme_row()
    assert good == 0 and bad > 0


# K of the GPU random tier (block linears of llama125m, llama3-1b, llama3-8b: forward / dgrad K = H, I or qkv / 2I rows, wgrad K = T)
RANDOM_TIER_K = (768, 2048, 2304, 3072, 4096, 6144, 8192, 14336, 16384, 28672)


@pytest.mark.parametrize("K", [4096, 8192, 14336, 28672])
def test_no_promotion_is_caught_at_the_gpu_tier_k(K):
    """A kernel that never promotes sums a whole split in the truncated accumulator: more than 3x outside ``share`` or ``rms`` at the
    GPU random tier's K from ``NO_PROMOTION_MIN_K`` on, while the promoting emulator stays within half."""
    assert K in RANDOM_TIER_K and K >= NO_PROMOTION_MIN_K
    A, B, sa, sb, _, _ = random_fp8(64, 96, K, E5M2, seed=K)
    ok = check_random(emulate(A, B, sa, sb), A, B, sa, sb)
    assert max(ok.values()) <= 0.5, ok
    bad = check_random(emulate(A, B, sa, sb, mutant="no_promotion"), A, B, sa, sb)
    assert max(bad["share"], bad["rms"]) > 3.0, bad


def test_every_mutant_is_caught_somewhere():
    need = {m for c in CASES for m in case_mutants(c[4], c[3], *c[5:]) if separable(m, c[3], c[5])} | {"out_scale_flush"}
    assert need == set(MUTANTS)


if __name__ == "__main__":                  # print the margin table: python tests/test_fp8_oracle.py
    import sys
    sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
    for c in CASES:
        emu, caught = margin_row(*c)
        print(f"{c[0]:22s} emulator/tol " + " ".join(f"{k}={v:.3f}" for k, v in emu.items() if k != "exact") + f"  exact mismatches {emu['exact']}")
        print(" " * 23 + "mutants " + "  ".join(f"{m}: {k}={r:.3g} exact={n}" + ("" if separable(m, c[3], c[5]) else " (GPU probe)")
                                               for m, (k, r, n) in caught.items()))
    for K in (768, 2048, 4096, 8192, 14336, 28672):
        A, B, sa, sb, _, _ = random_fp8(64, 96, K, E5M2, seed=K)
        ok = check_random(emulate(A, B, sa, sb), A, B, sa, sb)
        bad = check_random(emulate(A, B, sa, sb, mutant="no_promotion"), A, B, sa, sb)
        print(f"K={K:5d} emulator " + " ".join(f"{k}={v:.3f}" for k, v in ok.items()) + "   no_promotion "
              + " ".join(f"{k}={v:.3g}" for k, v in bad.items()))
    good, bad = extreme_row()
    print(f"extreme scale (k_a, k_b) = {EXTREME}: emulator mismatches {good}, out_scale_flush mismatches {bad}")
    for m, probe in list(GEMM_PROBES.items()) + list(QUANT_MUTANTS.items()):
        print(f"mutant {m:15s} -> {probe}")
