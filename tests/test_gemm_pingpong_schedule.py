"""Which kernel each GEMM of a training step runs on (`use_pingpong` in csrc/gemm_wgmma.cu, queried through the C entry
`acco_gemm_schedule` on a CPU, like `test_gemm_heuristic.py` queries `acco_gemm_choose`): 1 = the ping-pong kernel, 0 = the cooperative
one.  Pinned for every GEMM of the Llama-125M (8 x 1024 tokens) and Llama-3.2-1B (4 x 1024 tokens) steps on 132 SMs."""
import ctypes
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "acco_b200", "_C.so")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(SO):
        pytest.skip("extension not built")
    try:
        L = ctypes.CDLL(SO)
    except OSError as e:                                   # libcuda / libtorch not loadable on this box
        pytest.skip(f"extension not loadable here: {e}")
    L.acco_gemm_schedule.argtypes = [ctypes.c_int] * 7
    L.acco_gemm_schedule.restype = ctypes.c_int
    L.acco_gemm_choose.argtypes = [ctypes.c_int] * 7 + [ctypes.POINTER(ctypes.c_int)]
    L.acco_gemm_choose.restype = None
    return L


def step(T, H, I, Nqkv, V):
    """name -> (M, N, K, a_mn, b_mn, accumulate) of the 15 GEMMs of one step (forward, dgrad, wgrad of each linear layer)"""
    fwd = {"qkv": (Nqkv, H), "o": (H, H), "gateup": (2 * I, H), "down": (H, I), "lmhead": (V, H)}      # weight [N, K]
    g = {}
    for n, (N, K) in fwd.items():
        g[n + "_fwd"] = (T, N, K, 0, 0, 0)             # y = x w^T
        g[n + "_dgrad"] = (T, K, N, 0, 1, 0)           # dx = dy w
        g[n + "_wgrad"] = (N, K, T, 1, 1, 1)           # dw += dy^T x
    return g


LLAMA125M = step(8192, 768, 2048, 2304, 50304)
LLAMA1B = step(4096, 2048, 8192, 3072, 128256)


def test_llama125m_schedule(lib):
    """Every forward and dgrad GEMM of the Llama-125M step runs on the ping-pong kernel, every wgrad on the cooperative one."""
    for name, (M, N, K, a, b, acc) in LLAMA125M.items():
        want = 0 if name.endswith("_wgrad") else 1
        assert lib.acco_gemm_schedule(M, N, K, a, b, acc, 132) == want, name


def test_llama1b_schedule(lib):
    """The Llama-3.2-1B step stays on the cooperative kernel: its forward and dgrad picks are 256 wide at K >= 2048, where the
    128 x 128 ping-pong unit's extra operand traffic outweighs the hidden epilogue."""
    for name, (M, N, K, a, b, acc) in LLAMA1B.items():
        out = (ctypes.c_int * 5)()
        lib.acco_gemm_choose(M, N, K, a, b, acc, 132, out)
        if not name.endswith("_wgrad"):
            assert out[0] == 256 and K >= 2048, (name, list(out))
        assert lib.acco_gemm_schedule(M, N, K, a, b, acc, 132) == 0, name


def test_schedule_follows_the_pick(lib):
    """Ping-pong exactly for non-accumulating K-major-A calls whose pick is one split and 128 wide, or 256 wide with K <= 1024."""
    import itertools
    for M, N, K in itertools.product((128, 1000, 4096, 8192, 16384), (72, 96, 768, 2304, 50304), (64, 200, 768, 1024, 1088, 4096, 50304)):
        for a, b, acc in ((0, 0, 0), (0, 1, 0), (1, 1, 1), (1, 0, 0)):
            out = (ctypes.c_int * 5)()
            lib.acco_gemm_choose(M, N, K, a, b, acc, 132, out)
            bn, splits = out[0], out[1]
            want = int(not a and not acc and splits == 1 and (bn == 128 or (bn == 256 and K <= 1024)))
            assert lib.acco_gemm_schedule(M, N, K, a, b, acc, 132) == want, (M, N, K, a, b, acc, bn, splits)
