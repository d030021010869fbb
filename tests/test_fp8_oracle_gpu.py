"""The FP8 quantiser and FP8 wgmma GEMM (``csrc/fp8.cu``, ``gemm_fp8_kernel``) against the oracle of ``test_fp8_oracle.py``.

* Exact tier: on exact operands (``dense_fp8`` for one K split, ``sparse_fp8`` for split-K) with power-of-two scales, the full output must
  equal ``bf16_rn(y64)`` bit for bit at every instantiation (BN 64 / 128 x A e4m3 / e5m2) x epilogue x K of its list, ragged M and N,
  with operands and output as strided views inside guard buffers, with a CTA cap down to one CTA, and under forced cluster shapes; a
  probe row shows that the split epilogues do run several splits.
* Scale edges: every pair of scales the quantiser can emit, ``1/s = 2^-127`` included; the output must meet the contract wherever it is a
  normal bf16 number.  Two pairs whose product leaves fp32's normal range also run through every instantiation and epilogue.
* Accumulator width: how many bits of a small product survive next to a large one, within a k32 step, across the steps of a k-block, and
  across k-blocks (the promotion to fp32); printed with ``-s``.
* Random tier: each instantiation and the forward / dgrad / wgrad shapes of the block linears of three Llama presets against the oracle's
  bound and statistics; the largest ratios are printed.
* Quantiser: the scale rule at every finite bf16 amax, the cast at every k on every representable value, planted maxima / NaN / Inf at
  every lane, CTA and grid-stride boundary, and ragged tile shapes, bit for bit.
* The FP8 linear layer on exact operands over two micro-batches on each wgrad branch (with its FP8 launch counts), eagerly and replayed
  from a CUDA graph, and with programmatic dependent launch off.
* Rejected requests raise and write nothing."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_fp8_oracle import (ACC_BITS, E4M3, E5M2, EXACT_SCALES, K_MIN, PLANT_SHAPE, amax_ctas, bf16_of_bits,  # noqa: E402
                             cast_ks, cast_set, check_random, exact_fp8, exact_operands, planted_positions, random_fp8, scales,
                             split_geometry)
from test_gemm_oracle import bf16_rn, exact_result, ints  # noqa: E402
from test_gemm_oracle_gpu import embed, guard_mask  # noqa: E402

DEV = "cuda"
FMTS = {"e4m3": E4M3, "e5m2": E5M2}


def ext():
    from acco_b200.ops import load_ext
    return load_ext(required=True)


def gemm_fp8(*args, **kw):
    from acco_b200.ops.fp8 import gemm_fp8 as _g
    return _g(*args, **kw)


def quantize(*args):
    from acco_b200.ops.fp8 import quantize as _q
    return _q(*args)


def bits16(t):
    return t.view(torch.int16)


def embed8(t: torch.Tensor, seed: int):
    """(big, view): an FP8 matrix copied into rows [1, 1 + r) and columns [16, 16 + c) of a larger byte buffer of random guard bytes;
    row stride a multiple of 16 bytes, view 16-byte aligned."""
    r, c = t.shape
    width = -(-c // 16) * 16 + 48
    g = torch.Generator(device=DEV).manual_seed(seed)
    big = torch.randint(0, 256, (r + 3, width), generator=g, device=DEV, dtype=torch.uint8)
    view = big[1:r + 1, 16:c + 16]
    view.copy_(t.view(torch.uint8))
    view = view.view(t.dtype)
    assert view.data_ptr() % 16 == 0 and view.stride(0) % 16 == 0 and view.stride(0) > c
    return big, view


EPILOGUES = ("store", "bias", "beta1", "acc_split", "zf_split", "zf_split_bias")


def run_exact(fmt, M, N, K, bn=0, epi="store", cap=0, splits=2, scale=(3, -2), seed=0, shift=(0, 0)):
    split = epi in ("acc_split", "zf_split", "zf_split_bias")
    acc = epi in ("beta1", "acc_split")
    bias_on = epi in ("bias", "zf_split_bias")
    s = splits if split else 1
    ka, kb = scale
    A, B, sa, sb, bv, C0 = exact_operands(M, N, K, fmt, s, bias_on, acc, ka, kb, seed, DEV, shift=shift)
    a_big, a = embed8(A, seed + 4)
    b_big, b = embed8(B, seed + 5)
    o_big, out = embed(C0 if acc else torch.zeros(M, N, dtype=torch.bfloat16, device=DEV), seed + 6)
    if not acc:
        out.copy_(ints((M, N), 64, seed + 7, DEV))          # stale content: the store and the zero-fill must replace it
    a_before, b_before, o_before = a_big.clone(), b_big.clone(), o_big.clone()
    y = gemm_fp8(a, b, sa, sb, out=out, bias=bv, accumulate=acc, bn=bn, splits=s, max_ctas=cap)
    assert y.data_ptr() == out.data_ptr()
    want = exact_fp8(A, B, sa, sb, bv, C0)
    bad = bits16(out) != bits16(want)
    assert not bool(bad.any()), f"{int(bad.sum())} of {M * N} elements differ, first at {bad.nonzero()[0].tolist()}"
    mask = guard_mask(o_big, M, N)
    assert torch.equal(o_big[mask], o_before[mask]), "a write outside the output view"
    assert torch.equal(a_big, a_before) and torch.equal(b_big, b_before)
    return out


ONE_SPLIT_K = (16, 112, 144, 784, 1024, 1040)      # part of a k32 step, < 1 k-block, 1 + a tail, deep (dense sums past 256) ragged / not
SPLIT_K = (1040, 1552, 2064)


def _exact_cases():
    """Every instantiation x epilogue x K of its list (``ONE_SPLIT_K`` for the one-split epilogues, ``SPLIT_K`` for the split ones).
    M, the CTA cap and the scale pair rotate with independent offsets, so each takes all its values within every (instantiation,
    epilogue); N is ragged against the tile and 64."""
    Ms = (1, 63, 65, 127, 129, 200)
    caps = (0, 1, 7, 131)
    cases = []
    for ii, (fname, bn) in enumerate((f, b) for f in FMTS for b in (64, 128)):
        for ei, epi in enumerate(EPILOGUES):
            for ki, K in enumerate(SPLIT_K if "split" in epi else ONE_SPLIT_K):
                cases.append((fname, bn, Ms[(ki + ei + 2 * ii) % len(Ms)], 2 * bn + 40 + 8 * ((ki + ei) % 3), K, epi,
                              caps[(ki + ii + ei) % len(caps)], EXACT_SCALES[(ki + 3 * ei + ii) % len(EXACT_SCALES)]))
    for fname in FMTS:
        for bn in (64, 128):
            for epi in EPILOGUES:
                ks = {c[4] for c in cases if c[:2] == (fname, bn) and c[5] == epi}
                assert ks == set(SPLIT_K if "split" in epi else ONE_SPLIT_K)
                assert len({c[2] for c in cases if c[:2] == (fname, bn) and c[5] == epi}) == len(ks)
    return cases


@pytest.mark.parametrize("fname,bn,M,N,K,epi,cap,scale", _exact_cases(), ids=lambda v: str(v).replace(" ", ""))
def test_exact_every_path(fname, bn, M, N, K, epi, cap, scale):
    if os.environ.get("ACCO_GEMM_CLUSTER") and 0 < cap < 8:
        cap = 0                                             # a forced 2 x 2 cluster needs at least 4 CTAs
    run_exact(FMTS[fname], M, N, K, bn, epi, cap, splits=3 if epi != "zf_split" else 2, scale=scale, seed=M + N + K)


def test_exact_split_geometry_matches_the_host():
    """The sparse generator's splits are the host's: 2064 = 16 full k-blocks + a 16-element tail, 3 splits of 6 blocks."""
    assert split_geometry(2064, 3) == (6, 3) and split_geometry(1040, 3) == (3, 3) and split_geometry(144, 4) == (1, 2)


@pytest.mark.parametrize("fname,epi,bn,cap", [("e4m3", "store", 64, 1), ("e5m2", "beta1", 64, 1), ("e4m3", "bias", 128, 1),
                                              ("e5m2", "acc_split", 64, 7), ("e5m2", "zf_split_bias", 128, 1)])
def test_exact_persistent_ctas_run_hundreds_of_units(fname, epi, bn, cap):
    """One CTA (or 7) walks every unit: ring-phase wrap-around, staging-buffer reuse and the C prefetch at BN 64 (one sub-tile)."""
    M, N, K = 2049, 1000 * (bn // 64), 272
    units = -(-M // 128) * -(-N // bn) * (1 if "split" not in epi else split_geometry(K, 3)[1])
    assert units >= 250
    run_exact(FMTS[fname], M, N, K, bn, epi, cap, splits=3, seed=cap + bn)


@pytest.mark.parametrize("epi", ["acc_split", "zf_split", "zf_split_bias"])
@pytest.mark.parametrize("fname,bn", [("e4m3", 64), ("e4m3", 128), ("e5m2", 64), ("e5m2", 128)])
def test_split_epilogues_run_several_splits(fname, bn, epi):
    """The exact split-K operands give the same result split or not; this row does not.  257 ones in the first split and one in the
    second: one split stores bf16(258) = 258, two or more round the first partial to bf16(257) = 256 and then add 1 (256 again)."""
    K, splits = 1040, (2 if epi == "zf_split" else 3)
    kbs, s_eff = split_geometry(K, splits)
    assert s_eff == splits
    A = torch.zeros(8, K)
    A[0, :257] = 1.0
    A[0, kbs * 128 + 5] = 1.0
    A = A.to(DEV).to(FMTS[fname])
    B = torch.ones(16, K, device=DEV).to(E4M3)
    bias = torch.zeros(16, dtype=torch.bfloat16, device=DEV) if epi == "zf_split_bias" else None
    acc = epi == "acc_split"
    one, sc = scales(0, DEV), {}
    for sp in (1, splits):
        out = torch.zeros(8, 16, dtype=torch.bfloat16, device=DEV)
        gemm_fp8(A, B, one, one, out=out, bias=bias, accumulate=acc, bn=bn, splits=sp)
        sc[sp] = out[0].float().unique().tolist()
    assert sc == {1: [258.0], splits: [256.0]}, sc


@pytest.mark.parametrize("scale,shift", [((127, 1), (7, 7)), ((-60, -70), (-8, -8))], ids=["1/s_a=2^-127", "product=2^130"])
@pytest.mark.parametrize("epi", EPILOGUES)
@pytest.mark.parametrize("fname,bn", [("e4m3", 64), ("e4m3", 128), ("e5m2", 64), ("e5m2", 128)])
def test_exact_out_of_range_scale_every_path(fname, bn, epi, scale, shift):
    """Every instantiation and epilogue bit for bit at a scale pair whose product ``1 / (s_a s_b)`` lies outside fp32's normal range
    (the epilogue's exponent-aware path), on operands shifted so that bias, C, the split partials and the result stay normal."""
    run_exact(FMTS[fname], 129, 2 * bn + 40, 1040, bn, epi, 0, splits=3 if epi != "zf_split" else 2, scale=scale, seed=bn + 7,
              shift=shift)


@pytest.mark.parametrize("cluster", ["2,1", "1,2", "2,2"])
def test_exact_under_forced_cluster(cluster):
    """``ACCO_GEMM_CLUSTER`` is read once per process and applies to the FP8 kernels too: the exact tier again in a fresh process."""
    if os.environ.get("ACCO_GEMM_CLUSTER"):
        pytest.skip("already a forced-cluster run")
    env = dict(os.environ, ACCO_GEMM_CLUSTER=cluster)
    py = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    p = subprocess.run(py + ["-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu", f"{os.path.abspath(__file__)}::test_exact_every_path"],
                       env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900,
                       cwd=os.path.dirname(os.path.abspath(__file__)))
    assert p.returncode == 0 and f"{len(_exact_cases())} passed" in p.stdout, p.stdout[-3000:]


# ---------------------------------------------------------------------------------------------- scale edges
EDGE_K = (-120, -60, -1, 0, 1, 60, 100, 126, 127)


@pytest.mark.parametrize("fname", list(FMTS))
def test_scale_edges(fname):
    """Every (k_a, k_b) of the grid (k = -120 is the e4m3 floor; e5m2's is -113): where the contract is a normal bf16 number the output
    equals it bit for bit, where it overflows it is +-Inf, where it is below 2^-126 it is +-0 or exact."""
    fmt = FMTS[fname]
    A = exact_operands(129, 136, 1040, fmt, 1, False, False, 0, 0, seed=1, device=DEV)[0]
    B = exact_operands(136, 136, 1040, E4M3, 1, False, False, 0, 0, seed=2, device=DEV)[0]
    y64 = A.double() @ B.double().t()
    bad = []
    for ka in EDGE_K:
        for kb in EDGE_K:
            ka_ = max(ka, K_MIN[fmt])
            sa, sb = scales(ka_, DEV), scales(kb, DEV)
            assert (float(sa[1]) == 2.0 ** -127) == (ka_ == 127)
            y = gemm_fp8(A, B, sa, sb)
            want64 = y64 * 2.0 ** (-ka_ - kb)
            want = bf16_rn(want64)
            mag = want64.abs()
            normal = (mag >= 2.0 ** -126) & torch.isfinite(want.float())
            over = ~torch.isfinite(want.float())
            tiny = mag < 2.0 ** -126
            ok = torch.where(normal, bits16(y) == bits16(want), torch.ones_like(normal))
            ok &= torch.where(over, y.float() == want.float(), torch.ones_like(ok))
            ok &= torch.where(tiny, (y.float() == 0) | (bits16(y) == bits16(want)), torch.ones_like(ok))
            if not bool(ok.all()):
                bad.append((ka_, kb, int((~ok).sum()), int(normal.sum())))
    assert not bad, f"(k_a, k_b, wrong, normal) {bad}"


# ---------------------------------------------------------------------------------------------- accumulator width
def _width_probe(fmt, bn):
    """Rows of A against 8 identical rows of B (e4m3): +2^8 at k0, a small product 2^(8 - d) at k1, -2^8 at k2; the result is the small
    product exactly iff the accumulator kept it.  Three placements: all in one k32 step; k1 and k2 in the next two steps of the same
    k-block; k1 and k2 in the next two k-blocks (promotion: fp32 keeps 24 bits).  -> {placement: bits kept}."""
    places = {"k32 step": (0, 1, 2), "k-block steps": (0, 32, 64), "k-blocks": (0, 128, 256)}
    K, ds = 384, list(range(1, 27))
    B = torch.zeros(8, K, dtype=torch.float64)
    A = torch.zeros(len(places) * len(ds), K, dtype=torch.float64)
    expect = []
    for pi, (k0, k1, k2) in enumerate(places.values()):
        B[:, [k0, k1, k2]] = 1.0
        B[:, k1 + 3] = 2.0 ** -9                     # small products below 2^-9: a 2^-9 operand in B
        for di, d in enumerate(ds):
            r = pi * len(ds) + di
            A[r, k0], A[r, k2] = 256.0, -256.0
            p = 8 - d
            if p >= -9:
                A[r, k1] = 2.0 ** p
            else:
                A[r, k1 + 3] = 2.0 ** (p + 9)
            expect.append(2.0 ** p)
    y = gemm_fp8(A.float().to(DEV).to(fmt), B.float().to(DEV).to(E4M3), scales(0, DEV), scales(0, DEV), bn=bn).double().cpu()
    got = (y[:, 0] == torch.tensor(expect, dtype=torch.float64)).view(len(places), len(ds))
    assert bool((y == y[:, :1]).all())
    out = {}
    for pi, name in enumerate(places):
        kept = 0
        while kept < len(ds) and bool(got[pi, kept]):
            kept += 1
        out[name] = kept + 1                          # bits from the large product's leading bit to the last surviving one
    return out


@pytest.mark.parametrize("fname,bn", [("e4m3", 64), ("e4m3", 128), ("e5m2", 64), ("e5m2", 128)])
def test_accumulator_width(fname, bn):
    """Characterisation: prints the bits the FP8 accumulator keeps and asserts at least ``ACC_BITS`` inside a k-block (the oracle's
    bound and emulator assume that) and fp32's 24 across k-blocks (the kernel promotes every k-block)."""
    w = _width_probe(FMTS[fname], bn)
    print(f"[fp8 accumulator] A {fname} BN {bn}: bits kept " + ", ".join(f"{k}: {v}" for k, v in w.items()))
    assert w["k32 step"] >= ACC_BITS and w["k-block steps"] >= ACC_BITS, w
    assert w["k-blocks"] >= 24, w


# ---------------------------------------------------------------------------------------------- random tier
PRESETS = {"llama125m": (768, 2304, 2048), "llama3-1b": (2048, 3072, 8192), "llama3-8b": (4096, 6144, 14336)}   # H, qkv rows, I


def preset_gemms(preset, T):
    """(name, M, N, K, A format, accumulate) of the forward, dgrad and wgrad of every block linear."""
    H, QKV, I = PRESETS[preset]
    out = []
    for lin, Nw, Kw in (("qkv", QKV, H), ("o", H, H), ("gate_up", 2 * I, H), ("down", H, I)):
        out += [(lin + ".fwd", T, Nw, Kw, E4M3, False), (lin + ".dgrad", T, Kw, Nw, E5M2, False), (lin + ".wgrad", Nw, Kw, T, E5M2, True)]
    return out


def _random_case(M, N, K, fmt, acc, seed, bn=0, splits=1):
    A, B, sa, sb, _, C0 = random_fp8(M, N, K, fmt, seed, acc=acc, device=DEV)
    sa, sb = sa.to(DEV), sb.to(DEV)
    out = C0.clone() if acc else None
    y = gemm_fp8(A, B, sa, sb, out=out, accumulate=acc, bn=bn, splits=splits)
    r = check_random(y, A, B, sa, sb, None, C0, split_geometry(K, splits)[1])
    del A, B, C0, out, y
    return r


def _assert_rows(rows):
    for row in rows:
        print("[fp8 random] " + " ".join(str(v) for v in row[:-1]) + " " + " ".join(f"{k}={v:.3f}" for k, v in row[-1].items()))
    for row in rows:
        assert all(v <= 1.0 for v in row[-1].values()), row


def test_random_every_instantiation():
    rows = []
    for fname, fmt in FMTS.items():
        for bn in (64, 128):
            for acc, splits in ((False, 1), (True, 1), (True, 4), (False, 2)):
                rows.append((fname, bn, acc, splits, _random_case(1000, 776, 2064, fmt, acc, seed=bn + splits, bn=bn, splits=splits)))
    _assert_rows(rows)


@pytest.mark.parametrize("T", [2048, 8192])
@pytest.mark.parametrize("preset", sorted(PRESETS))
def test_random_block_linears(preset, T):
    """Each GEMM with one K split (all three statistics); the wgrad also split 4 ways into the gradient (bound and rms)."""
    rows = []
    for i, (name, M, N, K, fmt, acc) in enumerate(preset_gemms(preset, T)):
        rows.append((preset, T, name, M, N, K, 1, _random_case(M, N, K, fmt, acc, seed=100 * i + T)))
        if acc:
            rows.append((preset, T, name, M, N, K, 4, _random_case(M, N, K, fmt, acc, seed=100 * i + T + 1, splits=4)))
        torch.cuda.empty_cache()
    _assert_rows(rows)


# ---------------------------------------------------------------------------------------------- quantiser
@pytest.mark.parametrize("fname", list(FMTS))
def test_scale_rule_every_bf16_amax(fname):
    """Every finite non-negative bf16 amax (0x0000 - 0x7F7F), signed and placed anywhere in a 16 x 16 tensor: {s, 1/s, amax} bitwise
    those of ``scale_ref``."""
    from acco_b200.ops.fp8 import scale_ref
    fmt = FMTS[fname]
    bits = torch.arange(0, 0x7F80)
    vals = bf16_of_bits(bits)
    t = torch.zeros(16, 16, dtype=torch.bfloat16, device=DEV)
    got = []
    for i, v in enumerate(vals.to(DEV)):
        t.zero_()
        t[(7 * i) % 16, (3 * i) % 16] = v if i % 2 else -v
        got.append(quantize(t, fmt, True, False)[2][:3])
    got = torch.stack(got).cpu()
    s, inv = scale_ref(vals.float(), fmt)
    assert torch.equal(got[:, 0].view(torch.int32), s.view(torch.int32))
    assert torch.equal(got[:, 1].view(torch.int32), inv.view(torch.int32))
    assert torch.equal(got[:, 2], vals.float())


@pytest.mark.parametrize("fname", list(FMTS))
def test_cast_every_k_every_value(fname):
    """At every k the rule can pick, a tensor of every bf16 value whose scaled image lies in the format's range (ties included), both
    signs: q and qT bit for bit against ``quantize_ref``."""
    from acco_b200.ops.fp8 import quantize_ref
    fmt = FMTS[fname]
    for k in cast_ks(fmt):
        t = cast_set(fmt, k)
        q, qT, s = quantize(t.to(DEV), fmt, True, True)
        rq, _, rs = quantize_ref(t, fmt)
        assert float(rs[0]) == 2.0 ** k and torch.equal(s[:3].cpu(), rs), k
        assert torch.equal(q.view(torch.uint8).cpu(), rq.view(torch.uint8)), k
        assert torch.equal(qT.view(torch.uint8).cpu(), rq.view(torch.uint8).t()), k


def test_amax_planted_values():
    """A dominant element, NaN, +Inf and -Inf at each lane of a 16-byte vector, at the CTA and grid-stride boundaries, in the last pass
    and at the last element, in a tensor whose amax loop wraps."""
    from acco_b200.ops.fp8 import quantize_ref
    R, C = PLANT_SHAPE
    n = R * C
    ctas = amax_ctas(n, ext().num_sms())
    assert n // 8 > 256 * ctas
    g = torch.Generator(device=DEV).manual_seed(3)
    base = ((torch.rand(R, C, generator=g, device=DEV) - 0.5) * 0.4).to(torch.bfloat16)
    flat = base.view(-1)
    positions = planted_positions(n, ctas)
    want_s = {E4M3: 128.0, E5M2: 16384.0}                     # amax 3: the largest 2^k with 3 * 2^k <= 448 / 57344
    assert float(base.abs().max()) < 0.25
    for fmt in (E4M3, E5M2):
        for j, p in enumerate(positions):
            old = flat[p].clone()
            flat[p] = -3.0 if j % 2 else 3.0
            q, _, s = quantize(base, fmt, True, False)
            assert s[:3].tolist() == [want_s[fmt], 1.0 / want_s[fmt], 3.0], (p, s[:3].tolist())
            if j % 7 == 0:
                rq, _, _ = quantize_ref(base.cpu(), fmt)
                assert torch.equal(q.view(torch.uint8).cpu(), rq.view(torch.uint8)), p
            for bad in (float("nan"), float("inf"), -float("inf")):
                flat[p] = bad
                s = quantize(base, fmt, True, False)[2][:2].cpu()
                assert bool(torch.isnan(s).all()), (p, bad)
            flat[p] = old


def test_quantize_ragged_tiles():
    """R % 64 and C % 64 in {0, 16, 32, 48}, every combination: q and qT bit for bit."""
    from acco_b200.ops.fp8 import quantize_ref
    for r in (0, 16, 32, 48):
        for c in (0, 16, 32, 48):
            t = (torch.randn(128 + r, 192 + c, device=DEV) * 3).to(torch.bfloat16)
            for fmt in (E4M3, E5M2):
                q, qT, s = quantize(t, fmt, True, True)
                rq, _, rs = quantize_ref(t.cpu(), fmt)
                assert torch.equal(s[:3].cpu(), rs)
                assert torch.equal(q.view(torch.uint8).cpu(), rq.view(torch.uint8)), (r, c)
                assert torch.equal(qT.view(torch.uint8).cpu(), rq.view(torch.uint8).t()), (r, c)


# ---------------------------------------------------------------------------------------------- FP8 linear, exact
def _linear_operands(T=4096, K=128, N=64):
    """x: one +-1 per row (amax 1: q(x) = 256 x exactly); W in {-1, 0, 1} (amax 1); g integers in [-2, 2] (amax 2: q(g) = 2^14 g);
    bias integers.  Every forward, dgrad (|.| <= 2 N = 128), wgrad (T / K = 32 tokens per column: |.| <= 64 per micro-batch, split
    partials included) and bias sum is an integer that bf16 holds, except the bias sums, which bf16 rounds once."""
    g = torch.Generator(device=DEV).manual_seed(5)
    sign = (torch.randint(0, 2, (T,), generator=g, device=DEV) * 2 - 1).to(torch.bfloat16)
    x = torch.zeros(T, K, dtype=torch.bfloat16, device=DEV)
    x[torch.arange(T, device=DEV), torch.arange(T, device=DEV) * 37 % K] = sign
    w = ints((N, K), 1, 6, DEV)
    w[0, 0] = 1.0
    b = ints((N,), 8, 7, DEV)
    gs = []
    for i in range(2):
        gy = ints((T, N), 2, 8 + i, DEV)
        gy[i, 0] = 2.0
        gs.append(gy)
    return x, w, b, gs


def _linear_oracle(x, w, b, gs, w0, b0):
    y = exact_result(x, w, b)
    dx = [exact_result(gy, w.t()) for gy in gs]
    dw = w0
    db = b0
    for gy in gs:
        dw = exact_result(gy.t(), x.t(), C=dw)
        db = bf16_rn(db.double() + bf16_rn(gy.double().sum(0)).double())
    return y, dx, dw, db


def _linear_run(x, w, b, gs, branch, w0, b0):
    """Two micro-batches of ``ops.linear(fp8=True)``; -> (y, [dx per micro-batch], weight gradient, bias gradient)."""
    from acco_b200 import ops
    xs = x.clone().requires_grad_(True)
    wp = torch.nn.Parameter(w.clone())
    bp = torch.nn.Parameter(b.clone())
    if branch == "arena":
        wp.grad = w0.clone()
    elif branch == "add":
        wp.grad = w0.t().contiguous().t()                     # not an arena view (column-major): .add_
        assert wp.grad.stride(1) != 1
    bp.grad = b0.clone()
    dxs = []
    for gy in gs:
        xs.grad = None
        y = ops.linear(xs, wp, bp, accumulate_into_grad=branch != "returned", fp8=True)
        y.backward(gy)
        dxs.append(xs.grad.clone())
    return y.detach(), dxs, wp.grad, bp.grad


@pytest.mark.parametrize("branch", ["arena", "add", "returned"])
def test_linear_exact_eager_and_graph(branch):
    x, w, b, gs = _linear_operands()
    w0 = ints(w.shape, 16, 9, DEV)
    b0 = ints(b.shape, 16, 10, DEV)
    if branch == "returned":
        w0 = torch.zeros_like(w)
    from acco_b200 import ops
    ops.reset_launch_counts()
    y, dxs, dw, db = _linear_run(x, w, b, gs, branch, w0, b0)
    c = ops.launch_counts()                                   # the FP8 path ran (bf16 would give the same bits on these operands)
    assert (c.get("gemm_fp8"), c.get("fp8_amax"), c.get("fp8_cast"), c.get("gemm", 0)) == (6, 6, 6, 0), c
    wy, wdx, wdw, wdb = _linear_oracle(x, w, b, gs, w0, b0)
    if branch == "returned":                                  # autograd sums the two returned dw in bf16: exact (|.| <= 128)
        wdw = exact_result(gs[1].t(), x.t(), C=exact_result(gs[0].t(), x.t()))
    assert torch.equal(bits16(y), bits16(wy))
    for a, e in zip(dxs, wdx):
        assert torch.equal(bits16(a), bits16(e))
    assert torch.equal(bits16(dw.contiguous()), bits16(wdw)), int((dw != wdw).sum())
    assert torch.equal(bits16(db), bits16(wdb))
    if branch != "arena":
        return
    # the same two micro-batches captured in a CUDA graph and replayed: equal to eager bit for bit
    xs = x.clone().requires_grad_(True)
    wp = torch.nn.Parameter(w.clone())
    bp = torch.nn.Parameter(b.clone())
    wp.grad, bp.grad = w0.clone(), b0.clone()
    gys = [gy.clone() for gy in gs]
    dx_out = [torch.empty_like(x) for _ in gs]

    def step():
        wp.grad.copy_(w0)
        bp.grad.copy_(b0)
        for gy, dxo in zip(gys, dx_out):
            xs.grad = None
            yy = ops.linear(xs, wp, bp, accumulate_into_grad=True, fp8=True)
            yy.backward(gy)
            dxo.copy_(xs.grad)
        return yy.detach()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            y_g = step()
    torch.cuda.current_stream().wait_stream(s)
    wp.grad.fill_(7.0)
    for d in dx_out:
        d.fill_(7.0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits16(y_g), bits16(y))
    for a, e in zip(dx_out, dxs):
        assert torch.equal(bits16(a), bits16(e))
    assert torch.equal(bits16(wp.grad), bits16(dw)) and torch.equal(bits16(bp.grad), bits16(db))


def test_linear_without_programmatic_dependent_launch():
    """``ACCO_GEMM_PDL`` is read once per process: the exact linear (eager and graph) again in a fresh one with PDL off."""
    if os.environ.get("ACCO_GEMM_PDL") == "0":
        pytest.skip("already the PDL-off run")
    env = dict(os.environ, ACCO_GEMM_PDL="0")
    py = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    p = subprocess.run(py + ["-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                             f"{os.path.abspath(__file__)}::test_linear_exact_eager_and_graph"], env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600, cwd=os.path.dirname(os.path.abspath(__file__)))
    assert p.returncode == 0 and "3 passed" in p.stdout, p.stdout[-3000:]


# ---------------------------------------------------------------------------------------------- rejections
def _rejects(fn, out):
    before = out.clone()
    with pytest.raises(RuntimeError):
        fn()
    torch.cuda.synchronize()
    assert torch.equal(out, before), "a rejected request wrote into its output"


def test_requests_the_kernel_cannot_serve_raise():
    A = exact_operands(256, 192, 128, E4M3, 1, False, False, 0, 0, 1, DEV)[0]
    B = exact_operands(192, 192, 128, E4M3, 1, False, False, 0, 0, 2, DEV)[0]
    sa, sb = scales(0, DEV), scales(0, DEV)
    out = torch.full((256, 192), 5.0, dtype=torch.bfloat16, device=DEV)
    _rejects(lambda: gemm_fp8(A, B, sa, sb, out=out, bn=256), out)
    _rejects(lambda: gemm_fp8(A, B, sa, sb, out=out, bn=96), out)
    _rejects(lambda: gemm_fp8(A, B.view(torch.uint8).view(E5M2), sa, sb, out=out), out)              # B e5m2
    _rejects(lambda: ext().gemm_fp8(A.float().bfloat16(), B.float().bfloat16(), sa, sb, out, None, False, 0, 0, 0), out)
    wide = torch.zeros(256, 48, dtype=torch.uint8, device=DEV).view(E4M3)
    wideb = torch.zeros(192, 48, dtype=torch.uint8, device=DEV).view(E4M3)
    _rejects(lambda: gemm_fp8(wide[:, :40], wideb[:, :40], sa, sb, out=out), out)                      # K % 16 != 0
    odd = torch.zeros(256, 40, dtype=torch.uint8, device=DEV).view(E4M3)
    oddb = torch.zeros(192, 40, dtype=torch.uint8, device=DEV).view(E4M3)
    _rejects(lambda: gemm_fp8(odd[:, :32], oddb[:, :32], sa, sb, out=out), out)                        # row stride 40 bytes
    big = torch.full((256, 192 + 16), 5.0, dtype=torch.bfloat16, device=DEV)
    _rejects(lambda: gemm_fp8(A, B, sa, sb, out=big[:, 1:193]), big)                                   # output misaligned
    bias = torch.zeros(193, dtype=torch.bfloat16, device=DEV)
    _rejects(lambda: gemm_fp8(A, B, sa, sb, out=out, bias=bias[1:]), out)                              # bias misaligned
    _rejects(lambda: ext().gemm_fp8(A, B, sa, sb, None, None, True, 0, 0, 0), out)                     # accumulate without out
    _rejects(lambda: gemm_fp8(A, B, sa.cpu(), sb, out=out), out)                                       # scale on the CPU
    for bad in (torch.ones(24, 64, dtype=torch.bfloat16, device=DEV), torch.ones(64, 40, dtype=torch.bfloat16, device=DEV),
                torch.ones(64 * 64 + 8, dtype=torch.bfloat16, device=DEV)[1:1 + 64 * 64].view(64, 64)):
        with pytest.raises(RuntimeError):
            ext().fp8_quantize(bad, False, True, True)
        torch.cuda.synchronize()
        assert bool((bad == 1).all()), "a rejected quantise wrote into its input"
