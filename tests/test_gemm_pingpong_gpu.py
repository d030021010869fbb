"""The ping-pong schedule of the bf16 wgmma GEMM (``gemm_pingpong_kernel`` in ``csrc/gemm_wgmma.cu``): every forward and dgrad GEMM of
the Llama-125M and Llama-3.2-1B steps, ragged M / N, N < 128, bias on and off, and a call inside a CUDA graph.

Each case first asserts the schedule the call runs on (``acco_gemm_schedule``): ping-pong for the Llama-125M step and the other
shapes here, the cooperative kernel for the Llama-3.2-1B step, whose 256-wide picks at K >= 2048 stay there (``use_pingpong``).  Then
it checks the output two ways:

* bit for bit against the cooperative kernel on the same inputs.  A call that requests a tile width runs on the cooperative kernel,
  so ``bn=128`` (the same 128-wide tiles) and ``bn`` = the heuristic's pick both serve as the reference.  Every output element is the
  same chain of k16 wgmma steps in the same k order in both kernels, so the results must be identical.
* against the fp64 bounds of ``test_gemm_oracle.py`` (``check_random``, imported unchanged)."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_gemm_oracle import check_random, random_operands  # noqa: E402

DEV = "cuda"


def ext():
    from acco_b200.ops import load_ext
    return load_ext(required=True)


def lib():
    L = ctypes.CDLL(ext().__file__)
    L.acco_gemm_schedule.argtypes = [ctypes.c_int] * 7
    L.acco_gemm_schedule.restype = ctypes.c_int
    L.acco_gemm_choose.argtypes = [ctypes.c_int] * 7 + [ctypes.POINTER(ctypes.c_int)]
    L.acco_gemm_choose.restype = None
    return L


def gemm(*args, **kw):
    from acco_b200.ops.gemm import gemm as _gemm
    return _gemm(*args, **kw)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def step_shapes(T, H, I, Nqkv, V):
    """(name, M, N, K, b_mn): the forward (x [T, K] @ w [N, K]^T) and dgrad (dy [T, K] @ w [K, N]) GEMMs of one step"""
    return [("qkv_fwd", T, Nqkv, H, 0), ("o_fwd", T, H, H, 0), ("gateup_fwd", T, 2 * I, H, 0), ("down_fwd", T, H, I, 0),
            ("lmhead_fwd", T, V, H, 0),
            ("qkv_dgrad", T, H, Nqkv, 1), ("o_dgrad", T, H, H, 1), ("gateup_dgrad", T, H, 2 * I, 1), ("down_dgrad", T, I, H, 1),
            ("lmhead_dgrad", T, H, V, 1)]


CASES = ([("llama125m_" + n, M, N, K, b, False) for n, M, N, K, b in step_shapes(8192, 768, 2048, 2304, 50304)] +
         [("llama1b_" + n, M, N, K, b, False) for n, M, N, K, b in step_shapes(4096, 2048, 8192, 3072, 128256)] +
         [   # ragged M and N (the output map clips the last tiles), N < 128, bias on
             ("ragged_tn", 8100, 2296, 776, 0, False), ("ragged_nn", 8100, 2296, 776, 1, False),
             ("narrow_tn", 16384, 96, 768, 0, False), ("narrow_nn", 16300, 72, 200, 1, False),
             ("bias_tn", 8192, 768, 768, 0, True), ("bias_ragged_tn", 8100, 2296, 776, 0, True), ("bias_narrow_tn", 16300, 120, 776, 0, True),
             ("bias_nn", 8192, 2048, 768, 1, True),
         ])


def operands(M, N, K, b_mn, bias, seed):
    A, B, bv, _ = random_operands(M, N, K, seed, bias=bias, device=DEV)
    return A, (B.t().contiguous() if b_mn else B), B, bv


def assert_pingpong(M, N, K, b_mn, expect=1):
    assert lib().acco_gemm_schedule(M, N, K, 0, b_mn, 0, sms()) == expect, (M, N, K, b_mn)


def heuristic_bn(M, N, K, b_mn):
    out = (ctypes.c_int * 5)()
    lib().acco_gemm_choose(M, N, K, 0, b_mn, 0, sms(), out)
    assert out[1] == 1
    return out[0]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_pingpong_matches_cooperative_and_fp64(case):
    name, M, N, K, b_mn, bias = case
    assert_pingpong(M, N, K, b_mn, expect=0 if name.startswith("llama1b_") else 1)
    A, Bop, B, bv = operands(M, N, K, b_mn, bias, seed=CASES.index(case))
    y = gemm(A, Bop, bias=bv, b_mn=bool(b_mn))
    for bn in sorted({128, heuristic_bn(M, N, K, b_mn)}):
        ref = gemm(A, Bop, bias=bv, b_mn=bool(b_mn), bn=bn)      # a tile-width request: cooperative kernel
        torch.cuda.synchronize()
        diff = int((y.view(torch.int16) != ref.view(torch.int16)).sum())
        assert diff == 0, f"{name}: {diff} elements differ from the cooperative kernel at bn={bn}"
        del ref
    r = check_random(y, A, B, bv)
    print(name, r)
    assert r["bound"] <= 1.0 and r["rms"] <= 1.0 and r["share"] <= 1.0, (name, r)


def test_pingpong_repeatable_and_strided_output():
    """Repeated calls are bitwise equal, and a strided output view is written inside its extents only."""
    M, N, K = 8100, 2296, 776
    assert_pingpong(M, N, K, 0)
    A, B, _, bv = operands(M, N, K, 0, True, seed=7)
    y0 = gemm(A, B, bias=bv)
    big = torch.full((M + 3, N + 24), 3.0, dtype=torch.bfloat16, device=DEV)
    view = big[1:M + 1, 8:N + 8]
    gemm(A, B, out=view, bias=bv)
    torch.cuda.synchronize()
    assert torch.equal(view.view(torch.int16), y0.view(torch.int16))
    guard = torch.ones_like(big, dtype=torch.bool)
    guard[1:M + 1, 8:N + 8] = False
    assert bool((big[guard] == 3.0).all())


def test_pingpong_in_cuda_graph():
    """A forward and a dgrad on the ping-pong kernel, captured in a CUDA graph and replayed, give the eager result."""
    T, H, N = 8192, 768, 2304
    assert_pingpong(T, N, H, 0)                                    # y [T, N] = x [T, H] @ w [N, H]^T
    assert_pingpong(T, H, N, 1)                                    # dx [T, H] = dy [T, N] @ w [N, H]
    x, w, _, _ = operands(T, N, H, 0, False, seed=11)
    dy = torch.randn(T, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(13)).to(torch.bfloat16)
    want_y = gemm(x, w)
    want_dx = gemm(dy, w, b_mn=True)
    y = torch.empty_like(want_y)
    dx = torch.empty_like(want_dx)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        gemm(x, w, out=y)                                           # warm-up outside capture (tensor maps cached)
        gemm(dy, w, out=dx, b_mn=True)
        with torch.cuda.graph(graph, stream=s):
            gemm(x, w, out=y)
            gemm(dy, w, out=dx, b_mn=True)
    torch.cuda.current_stream().wait_stream(s)
    y.fill_(3.0)
    dx.fill_(3.0)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(y.view(torch.int16), want_y.view(torch.int16))
    assert torch.equal(dx.view(torch.int16), want_dx.view(torch.int16))
