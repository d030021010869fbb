"""The tile / split-K / cluster choice of the wgmma GEMM (`choose_config` in csrc/gemm_wgmma.cu) is host code: it can be queried
on a CPU through the extension's C entry point (`acco_gemm_choose`) without launching anything.  Properties that must hold for every
shape - they are the preconditions of the kernel's operand layouts and epilogue - plus the picks for the Llama-125M step on an
H100's 132 SMs as a regression guard for the cost model."""
import ctypes
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "acco_b200", "_C.so")


@pytest.fixture(scope="module")
def choose():
    if not os.path.exists(SO):
        pytest.skip("extension not built")
    try:
        lib = ctypes.CDLL(SO)
    except OSError as e:                                   # libcuda / libtorch not loadable on this box
        pytest.skip(f"extension not loadable here: {e}")
    fn = lib.acco_gemm_choose
    fn.argtypes = [ctypes.c_int] * 7 + [ctypes.POINTER(ctypes.c_int)]
    fn.restype = None

    def call(M, N, K, a_mn=0, b_mn=0, accumulate=0, sms=132):
        out = (ctypes.c_int * 5)()
        fn(M, N, K, a_mn, b_mn, accumulate, sms, out)
        return dict(bn=out[0], splits=out[1], pm=out[2], pn=out[3], msub=out[4])
    return call


def test_choices_respect_the_kernel_preconditions(choose):
    import itertools
    for M, N, K in itertools.product((8, 128, 1000, 4096, 8192), (8, 72, 768, 2304, 50304), (8, 64, 200, 768, 8192, 50304)):
        for a_mn, b_mn, acc in ((0, 0, 0), (0, 1, 0), (1, 1, 1)):
            c = choose(M, N, K, a_mn, b_mn, acc)
            assert c["bn"] in (64, 128, 256), (M, N, K, c)
            assert c["msub"] == 1 and c["pm"] == 1 and c["pn"] == 1, (M, N, K, c)            # multicast only on request
            if b_mn:
                assert c["bn"] % 64 == 0, (M, N, K, c)                                         # MN-major B: whole 64-n chunks per CTA
            num_k = (K + 63) // 64
            assert 1 <= c["splits"] <= num_k, (M, N, K, c)
            if not acc:
                assert c["splits"] <= 4 and (c["splits"] == 1 or num_k >= 128), (M, N, K, c)    # zero-fill + reduce only when K dwarfs the output
            else:
                assert c["splits"] <= 16


def test_llama125m_step_shapes(choose):
    """One pinned pick per GEMM of the Llama-125M step (8 x 1024 tokens) on 132 SMs."""
    T = 8192
    picks = {   # (M, N, K, a_mn, b_mn, accumulate) -> (bn, splits)
        (T, 2304, 768, 0, 0, 0): (128, 1),      # qkv forward
        (T, 4096, 768, 0, 0, 0): (256, 1),      # gate|up forward
        (T, 768, 2304, 0, 1, 0): (128, 1),      # qkv dgrad
        (T, 2048, 768, 0, 1, 0): (256, 1),      # down dgrad
        (2304, 768, T, 1, 1, 1): (128, 1),      # qkv wgrad
        (4096, 768, T, 1, 1, 1): (128, 2),      # gate|up wgrad
        (768, 2048, T, 1, 1, 1): (128, 1),      # down wgrad
        (768, 768, T, 1, 1, 1): (128, 3),       # o_proj wgrad
        (T, 768, 50304, 0, 1, 0): (128, 1),     # LM-head dgrad: 384 output tiles already fill the GPU, no split-K
        (T, 50304, 768, 0, 0, 0): (256, 1),     # LM-head forward
    }
    for (M, N, K, a, b, acc), (bn, splits) in picks.items():
        c = choose(M, N, K, a, b, acc)
        assert (c["bn"], c["splits"], c["pm"], c["pn"], c["msub"]) == (bn, splits, 1, 1, 1), ((M, N, K, a, b, acc), c)
    # fewer SMs (a caller-imposed cap) never makes the choice invalid
    c = choose(T, 768, 768, 0, 0, 0, sms=64)
    assert c["bn"] in (64, 128, 256)
