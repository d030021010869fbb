"""The bf16 wgmma GEMM (``csrc/gemm_wgmma.cu``, called through ``ops.gemm.gemm``) against the oracle of ``test_gemm_oracle.py``.

* Exact tier: on operands whose every intermediate is exact (``dense_exact`` for one K split, ``sparse_exact`` for the split-K
  paths), the full output must equal ``bf16_rn(exact sum)`` bit for bit, for every layout, tile width, cluster shape, epilogue,
  ragged edge and CTA cap, with operands and output as strided views inside larger buffers whose guard cells must not change.
* LM-head shapes: the banded forward (8192 x 50304 x 768) in full, and the zero-filled split-K dgrad at every pick of the heuristic
  that splits, each asserted to take the path it is there for.
* fp64 tier: every GEMM of a training step of four presets at three token counts, with the heuristic's pick, on random operands,
  within the bounds derived in ``test_gemm_oracle.py``; the largest error / bound ratio of each case is printed (``-s``).
* Repeatability: every one-split path is bitwise repeatable on random operands.  The split-K paths add their partials with bf16
  reduce-adds in whatever order the splits finish, so they are only required to repeat on exact operands, where the order cannot
  matter.
* Chains of dependent GEMMs without a host sync, eagerly, captured in a CUDA graph and with programmatic dependent launch off.
* Requests the kernel cannot serve raise and write nothing."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_gemm_oracle import (K_DENSE_MAX, check_random, dense_exact, exact_result, ints, random_operands,  # noqa: E402
                              sparse_exact, split_geometry)

DEV = "cuda"


def ext():
    from acco_b200.ops import load_ext
    return load_ext(required=True)


def gemm(*args, **kw):
    from acco_b200.ops.gemm import gemm as _gemm
    return _gemm(*args, **kw)


# ---------------------------------------------------------------------------------------------- strided views with guard cells
def embed(t: torch.Tensor, seed: int):
    """(big, view): ``t`` copied into rows [1, 1 + r) and columns [8, 8 + c) of a larger buffer of random guard values.  The row
    stride is a multiple of 8 elements and the view starts 16-byte aligned, as a TMA tensor map requires."""
    r, c = t.shape
    width = -(-c // 8) * 8 + 24
    g = torch.Generator(device=DEV).manual_seed(seed)
    big = torch.randn(r + 3, width, generator=g, device=DEV).to(torch.bfloat16)
    view = big[1:r + 1, 8:c + 8]
    view.copy_(t)
    assert view.data_ptr() % 16 == 0 and view.stride(0) % 8 == 0
    return big, view


def guard_mask(big, r, c):
    m = torch.ones_like(big, dtype=torch.bool)
    m[1:r + 1, 8:c + 8] = False
    return m


LAYOUTS = {"tn": (False, False), "nn": (False, True), "tt": (True, True), "a_mn": (True, False)}
EPILOGUES = ("store", "bias", "beta1", "acc_split", "zf_split", "zf_split_bias")


def run_exact(layout, M, N, K, bn=0, pm=0, pn=0, epi="store", max_ctas=0, splits=0, seed=0):
    """One exact-tier case: the full output bit for bit and the guard cells around every view."""
    a_mn, b_mn = LAYOUTS[layout]
    split = epi in ("acc_split", "zf_split", "zf_split_bias")
    acc = epi in ("beta1", "acc_split")
    bias_on = epi in ("bias", "zf_split_bias")
    if split:
        s = splits or 2
        A, B = sparse_exact(M, K, s, seed, DEV), ints((N, K), 1, seed + 1, DEV)
        bias = ints((N,), 32, seed + 2, DEV) if bias_on else None
        C0 = ints((M, N), 64, seed + 3, DEV) if acc else None
    else:
        s = 1
        A, B = dense_exact(M, K, seed, DEV), dense_exact(N, K, seed + 1, DEV)
        bias = ints((N,), 1024, seed + 2, DEV) if bias_on else None
        C0 = ints((M, N), 1024, seed + 3, DEV) if acc else None
    a_big, a = embed(A.t() if a_mn else A, seed + 4)
    b_big, b = embed(B.t() if b_mn else B, seed + 5)
    o_big, out = embed(C0 if acc else torch.zeros(M, N, dtype=torch.bfloat16, device=DEV), seed + 6)
    if not acc:
        out.copy_(ints((M, N), 64, seed + 7, DEV))        # stale content: the store and the zero-fill must replace it
    a_before, b_before, o_before = a_big.clone(), b_big.clone(), o_big.clone()
    y = gemm(a, b, out=out, bias=bias, a_mn=a_mn, b_mn=b_mn, accumulate=acc, bn=bn, splits=s, pm=pm, pn=pn, max_ctas=max_ctas)
    assert y.data_ptr() == out.data_ptr()
    want = exact_result(A, B, bias, C0)
    bad = (out.view(torch.int16) != want.view(torch.int16))
    assert not bool(bad.any()), f"{int(bad.sum())} of {M * N} elements differ, first at {bad.nonzero()[0].tolist()}"
    mask = guard_mask(o_big, M, N)
    assert torch.equal(o_big[mask], o_before[mask]), "a write outside the output view"
    assert torch.equal(a_big, a_before) and torch.equal(b_big, b_before)
    return out


def _exact_cases():
    """Every layout x tile width x epilogue once, with the cluster shape, the ragged M and K and the CTA cap rotating through their
    values; N is ragged against both the tile and 64.  MN-major B cannot split a 64-wide tile between two CTAs (pm = 2, bn = 64):
    that request is a rejection case below."""
    Ms = (1, 63, 64, 65, 127, 129, 200)
    Ks = (8, 40, 72, 136, 520)
    clusters = ((1, 1), (2, 1), (1, 2), (2, 2))
    caps = (0, 1, 7, 131)
    cases, i = [], 0
    for layout in LAYOUTS:
        for bn in (64, 128, 256):
            for epi in EPILOGUES:
                M = Ms[i % len(Ms)]
                N = 2 * bn + 40 + 8 * (i % 3)                  # 3 tiles of bn, the last one ragged; N % 64 != 0
                K = Ks[i % len(Ks)]
                if epi in ("acc_split", "zf_split", "zf_split_bias"):
                    K = (200, 520, 1000)[i % 3]
                pm, pn = clusters[i % 4]
                if LAYOUTS[layout][1] and bn == 64:
                    pm = 1
                cap = caps[(i // 4) % 4]
                if cap and cap < pm * pn:
                    cap = 7
                cases.append((layout, M, N, K, bn, pm, pn, epi, cap))
                i += 1
    return cases


@pytest.mark.parametrize("layout,M,N,K,bn,pm,pn,epi,cap", _exact_cases(),
                         ids=lambda v: str(v) if not isinstance(v, str) else v)
def test_exact_every_path(layout, M, N, K, bn, pm, pn, epi, cap):
    run_exact(layout, M, N, K, bn, pm, pn, epi, cap, splits=3 if epi != "zf_split" else 2, seed=M + N + K)


@pytest.mark.parametrize("layout,epi,bn,cap", [("tn", "store", 64, 1), ("tn", "beta1", 64, 1), ("nn", "bias", 64, 1),
                                               ("tt", "acc_split", 64, 1), ("tn", "zf_split_bias", 128, 7), ("tt", "beta1", 64, 131)])
def test_exact_persistent_ctas_run_hundreds_of_units(layout, epi, bn, cap):
    """One CTA (or 7, or 131) walks every unit: ring-phase wrap-around, staging-buffer reuse and the C prefetch of the next tile."""
    M, N, K = 2049, 1000, 200
    units = -(-M // 128) * -(-N // bn) * (1 if epi in ("store", "bias", "beta1") else split_geometry(K, 3)[1])
    assert units >= 2 * cap and (cap > 1 or units >= 250)
    run_exact(layout, M, N, K, bn, 1, 1, epi, cap, splits=3, seed=cap + bn)


@pytest.mark.parametrize("K", [8, 40, 72, 4104, K_DENSE_MAX])
def test_exact_ragged_k(K):
    for layout in ("tn", "tt"):
        run_exact(layout, 129, 200, K, epi="beta1", seed=K)
        run_exact(layout, 65, 136, K, epi="store", seed=K + 1)


# ---------------------------------------------------------------------------------------------- LM-head shapes
def tile_band(M, K, bn_cols, num_sn, l2):
    """Twin of ``tile_band`` in csrc/gemm_wgmma.cu."""
    if l2 <= 0 or M * K * 2.0 > l2 / 3.0:
        return num_sn
    return max(1, min(num_sn, int(l2 / 8.0 / (bn_cols * K * 2.0))))


def test_lm_head_forward_banded_full_output():
    M, N, K = 8192, 50304, 768
    bn, splits, pm, pn, _ = ext().gemm_choose(M, N, K, False, False, False)
    num_n = -(-N // bn)
    num_sn = -(-num_n // pn)
    band = tile_band(M, K, bn * pn, num_sn, torch.cuda.get_device_properties(0).L2_cache_size)
    assert splits == 1 and band < num_sn and num_sn % band != 0, (bn, band, num_sn)      # banded, with a partial last band
    A, B = dense_exact(M, K, 1, DEV), dense_exact(N, K, 2, DEV)
    y = gemm(A, B)
    want = exact_result(A, B)
    assert torch.equal(y.view(torch.int16), want.view(torch.int16)), int((y != want).sum())
    assert torch.equal(gemm(A, B).view(torch.int16), y.view(torch.int16))


# (hidden, padded vocab, T): the heuristic splits the LM-head dgrad (M = T, N = H, K = vocab) at these picks on 132 SMs
LM_DGRAD_SPLITS = [(768, 50304, T) for T in (256, 512, 1024, 2048, 4096)] + [(2048, 128256, 256), (2048, 128256, 512),
                                                                            (4096, 128256, 256), (4096, 128256, 8192)]


@pytest.mark.parametrize("H,V,T", LM_DGRAD_SPLITS)
def test_lm_head_dgrad_zero_filled_split_k(H, V, T):
    if ext().num_sms() != 132:
        pytest.skip("the picks are those of a 132-SM H100")
    bn, splits, _, _, _ = ext().gemm_choose(T, H, V, False, True, False)
    assert splits > 1, (H, V, T, bn, splits)                   # the zero-fill + reduce-add path
    dy = sparse_exact(T, V, splits, seed=T, device=DEV)
    w = ints((V, H), 1, seed=H, device=DEV)                     # the weight [V, H] as an MN-major B
    out = torch.full((T, H), 7.0, dtype=torch.bfloat16, device=DEV)
    gemm(dy, w, out=out, b_mn=True)
    want = exact_result(dy, w.t())
    assert torch.equal(out.view(torch.int16), want.view(torch.int16)), int((out != want).sum())
    again = gemm(dy, w, b_mn=True)
    assert torch.equal(again.view(torch.int16), out.view(torch.int16))
    del dy, w


# ---------------------------------------------------------------------------------------------- fp64 tier at a training step
PRESETS = {   # hidden, padded vocab, block linears (name, N_w, K_w, bias)
    "llama125m": (768, 50304, [("qkv", 2304, 768, False), ("o", 768, 768, False), ("gate_up", 4096, 768, False), ("down", 768, 2048, False)]),
    "llama3.2-1b": (2048, 128256, [("qkv", 3072, 2048, False), ("o", 2048, 2048, False), ("gate_up", 16384, 2048, False),
                                   ("down", 2048, 8192, False)]),
    "llama3-8b": (4096, 128256, [("qkv", 6144, 4096, False), ("o", 4096, 4096, False), ("gate_up", 28672, 4096, False),
                                 ("down", 4096, 14336, False)]),
    "gptneo125m": (768, 50304, [("qkv", 2304, 768, False), ("out_proj", 768, 768, True), ("c_fc", 3072, 768, True),
                                ("c_proj", 768, 3072, True)]),
}
TOKENS = (256, 2048, 8192)


def step_gemms(preset, T):
    """(name, M, N, K, a_mn, b_mn, accumulate, bias) of every GEMM of one training step: forward, dgrad and wgrad (added into the
    gradient) of every block linear and of the LM head."""
    H, V, lins = PRESETS[preset]
    out = []
    for name, Nw, Kw, bias in lins + [("lm_head", V, H, False)]:
        out.append((name + ".fwd", T, Nw, Kw, False, False, False, bias))
        out.append((name + ".dgrad", T, Kw, Nw, False, True, False, False))
        out.append((name + ".wgrad", Nw, Kw, T, True, True, True, False))
    return out


def mode_of(accumulate, bias, splits):
    if splits > 1:
        return ("acc_split" if accumulate else "zf_split") + ("_bias" if bias else "")
    return "beta1" if accumulate else ("bias" if bias else "store")


def test_step_picks_cover_every_tile_and_epilogue():
    seen_bn, seen_mode = set(), set()
    for preset in PRESETS:
        for T in TOKENS:
            for _, M, N, K, a_mn, b_mn, acc, bias in step_gemms(preset, T):
                bn, splits, *_ = ext().gemm_choose(M, N, K, a_mn, b_mn, acc)
                seen_bn.add(bn)
                seen_mode.add(mode_of(acc, bias, splits))
    assert seen_bn == {64, 128, 256}, seen_bn
    # a bias GEMM is never split: biases sit on forwards, whose K is far below the 128 k-blocks a zero-filled split needs
    assert seen_mode == {"store", "bias", "beta1", "acc_split", "zf_split"}, seen_mode


@pytest.mark.parametrize("T", TOKENS)
@pytest.mark.parametrize("preset", sorted(PRESETS))
def test_fp64_training_step(preset, T):
    rows = []
    for i, (name, M, N, K, a_mn, b_mn, acc, bias) in enumerate(step_gemms(preset, T)):
        bn, splits, *_ = ext().gemm_choose(M, N, K, a_mn, b_mn, acc)
        A, B, bv, C0 = random_operands(M, N, K, seed=1000 * i + T, bias=bias, acc=acc, device=DEV)
        a = A.t().contiguous() if a_mn else A
        b = B.t().contiguous() if b_mn else B
        out = C0.clone() if acc else None
        y = gemm(a, b, out=out, bias=bv, a_mn=a_mn, b_mn=b_mn, accumulate=acc)
        _, s_eff = split_geometry(K, splits)
        r = check_random(y, A, B, bv, C0, s_eff)
        rows.append((name, M, N, K, bn, s_eff, mode_of(acc, bias, s_eff), r))
        del A, B, bv, C0, a, b, out, y
    torch.cuda.empty_cache()
    for name, M, N, K, bn, s, mode, r in rows:
        print(f"[fp64] {preset:11s} T={T:5d} {name:14s} {M:6d}x{N:6d}x{K:6d} bn={bn:3d} splits={s} {mode:9s} "
              + " ".join(f"{k}={v:.3f}" for k, v in r.items()))
    for name, M, N, K, bn, s, mode, r in rows:
        assert r["bound"] <= 1.0 and r["rms"] <= 1.0 and r.get("share", 0.0) <= 1.0, (preset, T, name, r)


# ---------------------------------------------------------------------------------------------- repeatability
@pytest.mark.parametrize("layout,bias,acc,bn,cap", [("tn", False, False, 256, 0), ("tn", True, False, 64, 7), ("nn", False, False, 128, 0),
                                                    ("tt", False, True, 128, 0), ("a_mn", False, True, 64, 131)])
def test_one_split_paths_are_bitwise_repeatable(layout, bias, acc, bn, cap):
    a_mn, b_mn = LAYOUTS[layout]
    A, B, bv, C0 = random_operands(1000, 776, 2048, seed=bn + cap, bias=bias, acc=acc, device=DEV)
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    outs = []
    for _ in range(2):
        out = C0.clone() if acc else None
        outs.append(gemm(a, b, out=out, bias=bv, a_mn=a_mn, b_mn=b_mn, accumulate=acc, bn=bn, splits=1 if acc else 0, max_ctas=cap))
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))


@pytest.mark.parametrize("epi", ["acc_split", "zf_split_bias"])
def test_split_paths_repeat_on_exact_operands(epi):
    y1 = run_exact("tt", 1000, 776, 4096, epi=epi, splits=4, seed=3).clone()
    y2 = run_exact("tt", 1000, 776, 4096, epi=epi, splits=4, seed=3).clone()
    d = y1.view(torch.int16) != y2.view(torch.int16)
    assert not bool(d.any()), (int(d.sum()), d.nonzero()[:4].tolist(), y1[d][:4].tolist(), y2[d][:4].tolist())


# ---------------------------------------------------------------------------------------------- chains, graphs, PDL
def _chain_operands():
    """Exact through the chain: x has one +-1 per row, so y = x w^T is in {-1, 0, 1}; dgrad sums of y w stay below 256 in
    magnitude; the wgrad adds integers <= 256 into an integer gradient; the split dgrad's partials and running sums stay below 256
    and so equal the one-split dgrad bit for bit."""
    T, K, N = 512, 128, 192
    g = torch.Generator(device=DEV).manual_seed(21)
    sign = torch.randint(0, 2, (T,), generator=g, device=DEV) * 2 - 1
    x = torch.zeros(T, K, dtype=torch.bfloat16, device=DEV)
    x[torch.arange(T, device=DEV), torch.arange(T, device=DEV) * 37 % K] = sign.to(torch.bfloat16)
    return x, ints((N, K), 1, 23, DEV), ints((N, K), 64, 24, DEV)


def _chain(x, w, g, y, dx, dx2):
    gemm(x, w, out=y)                                             # forward  y  = x w^T          (TN)
    gemm(y, w, out=dx, b_mn=True)                                 # dgrad    dx = y w            (NN)
    gemm(y, x, out=g, a_mn=True, b_mn=True, accumulate=True)      # wgrad    g += y^T x          (TT, beta = 1)
    gemm(y, w, out=dx2, b_mn=True, splits=2)                      # dgrad again, zero-filled and split along K


def _chain_oracle(x, w, g0):
    y = exact_result(x, w)
    dx = exact_result(y, w.t())
    g = exact_result(y.t(), x.t(), C=g0)
    return y, dx, g


def _check_chain(outs, want):
    y, dx, g, dx2 = outs
    wy, wdx, wg = want
    for got, exp in ((y, wy), (dx, wdx), (g, wg), (dx2, wdx)):
        assert torch.equal(got.view(torch.int16), exp.view(torch.int16)), int((got != exp).sum())


def test_chain_eager_and_graph():
    x, w, g0 = _chain_operands()
    assert float(exact_result(x, w).abs().max()) <= 1 and float(x.abs().sum(1).max()) == 1
    want = _chain_oracle(x, w, g0)
    T, K = x.shape
    N = w.shape[0]
    bufs = [torch.empty(T, N, dtype=torch.bfloat16, device=DEV), torch.empty(T, K, dtype=torch.bfloat16, device=DEV),
            torch.empty(T, K, dtype=torch.bfloat16, device=DEV)]
    g = g0.clone()
    _chain(x, w, g, *bufs)                                          # no host sync between the four launches
    _check_chain((bufs[0], bufs[1], g, bufs[2]), want)
    for t in bufs:
        t.fill_(3.0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        g.copy_(g0)                                                 # warm-up outside capture (tensor maps cached)
        _chain(x, w, g, *bufs)
        with torch.cuda.graph(graph, stream=s):
            g.copy_(g0)
            _chain(x, w, g, *bufs)
    torch.cuda.current_stream().wait_stream(s)
    for t in bufs:
        t.fill_(3.0)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    _check_chain((bufs[0], bufs[1], g, bufs[2]), want)


def test_chain_without_programmatic_dependent_launch():
    """``ACCO_GEMM_PDL`` is read once per process: the chain again in a fresh one with PDL off."""
    if os.environ.get("ACCO_GEMM_PDL") == "0":
        pytest.skip("already the PDL-off run")
    env = dict(os.environ, ACCO_GEMM_PDL="0")
    py = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    p = subprocess.run(py + ["-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                        f"{os.path.abspath(__file__)}::test_chain_eager_and_graph"], env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600, cwd=os.path.dirname(os.path.abspath(__file__)))
    assert p.returncode == 0 and "1 passed" in p.stdout, p.stdout[-3000:]


# ---------------------------------------------------------------------------------------------- rejections
def _rejects(fn, out):
    before = out.clone()
    with pytest.raises(RuntimeError):
        fn()
    torch.cuda.synchronize()
    assert torch.equal(out, before), "a rejected request wrote into its output"


def test_requests_the_kernel_cannot_serve_raise():
    A, B = dense_exact(256, 128, 1, DEV), dense_exact(192, 128, 2, DEV)
    out = torch.full((256, 192), 5.0, dtype=torch.bfloat16, device=DEV)
    _rejects(lambda: gemm(A, B, out=out, bn=96), out)
    _rejects(lambda: gemm(A, B, out=out, pm=3), out)
    _rejects(lambda: gemm(A, B, out=out, msub=2), out)
    _rejects(lambda: gemm(A, B.t().contiguous(), out=out, b_mn=True, bn=64, pm=2), out)      # a 64-wide MN-major B tile split in two
    big = torch.full((256, 192 + 16), 5.0, dtype=torch.bfloat16, device=DEV)
    _rejects(lambda: gemm(A, B, out=big[:, 1:193]), big)                                       # output not 16-byte aligned
    bias = torch.zeros(193, dtype=torch.bfloat16, device=DEV)
    _rejects(lambda: gemm(A, B, out=out, bias=bias[1:]), out)                                  # bias not 16-byte aligned
    _rejects(lambda: ext().gemm(A[:, 1:121], B[:, :120], out, None, False, False, False, 0, 0, 0, 0, 0, 0), out)   # operand misaligned
    out_odd = torch.full((256, 188), 5.0, dtype=torch.bfloat16, device=DEV)
    _rejects(lambda: gemm(A, B[:188], out=out_odd), out_odd)                                   # N % 8 != 0
