"""The weight-gradient (wgrad) GEMM - ``grad [M, N] += dy [T, M]^T x [T, N]``, both operands MN-major - bit for bit against the fp64
oracle of ``test_gemm_oracle.py`` on exact operands.  Its operands are loaded one folded TMA box per stage when their MN-major extents
are whole 64-element chunks, and one box per 64-element chunk otherwise; both are covered here:

* every wgrad shape of the Llama-125M (T = 8192) and Llama-3.2-1B (T = 4096) steps at the heuristic's pick, into a strided view of a
  larger gradient buffer whose guard cells must not change, in bf16 and in fp32 (``grad_accum_dtype=fp32``), the split-K picks
  (o_proj 3 splits, the 125M gate|up 2) included;
* ragged extents (not whole 64-element chunks, and whole chunks but not whole 128-row tiles), operands as strided views, each tile
  width, and 2-CTA clusters that multicast the folded boxes;
* a CUDA graph replaying the call."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_gemm_oracle import dense_exact, exact_result, ints, sparse_exact  # noqa: E402

DEV = "cuda"
# (name, M, N, T): grad [M, N] += dy [T, M]^T x [T, N]
SHAPES = [
    ("125m_qkv", 2304, 768, 8192), ("125m_o", 768, 768, 8192), ("125m_gateup", 4096, 768, 8192), ("125m_down", 768, 2048, 8192),
    ("1b_qkv", 3072, 2048, 4096), ("1b_o", 2048, 2048, 4096), ("1b_gateup", 16384, 2048, 4096), ("1b_down", 2048, 8192, 4096),
]


def ext():
    from acco_b200.ops import load_ext
    return load_ext(required=True)


def pick(M, N, K):
    lib = ctypes.CDLL(ext().__file__)
    lib.acco_gemm_choose.argtypes = [ctypes.c_int] * 7 + [ctypes.POINTER(ctypes.c_int)]
    out = (ctypes.c_int * 5)()
    lib.acco_gemm_choose(M, N, K, 1, 1, 1, torch.cuda.get_device_properties(0).multi_processor_count, out)
    return out[0], out[1]


def mn_major(t: torch.Tensor, pad: int, seed: int):
    """``t`` [rows, K] stored MN-major: a [K, rows] view with row stride rows + pad inside a buffer of random guard values."""
    rows, K = t.shape
    g = torch.Generator(device=DEV).manual_seed(seed)
    big = torch.randn(K, rows + pad + 8, generator=g, device=DEV).to(torch.bfloat16)
    view = big[:, 8:8 + rows]
    view.copy_(t.t())
    return view


def arena_view(C0: torch.Tensor, seed: int):
    """(big, view, guard): ``C0`` in rows [1, 1 + M) and columns [8, 8 + N) of a larger buffer, like a weight's gradient slot."""
    M, N = C0.shape
    g = torch.Generator(device=DEV).manual_seed(seed)
    big = (torch.randn(M + 3, N + 24, generator=g, device=DEV) * 100).to(C0.dtype)
    view = big[1:M + 1, 8:N + 8]
    view.copy_(C0)
    guard = torch.ones_like(big, dtype=torch.bool)
    guard[1:M + 1, 8:N + 8] = False
    return big, view, guard


def operands(M, N, K, splits, seed):
    """Exact-tier logical operands A [M, K], B [N, K] for `splits` K splits, and the starting gradient C0 (bf16 integers)."""
    if splits == 1:
        return dense_exact(M, K, seed, DEV), dense_exact(N, K, seed + 1, DEV), ints((M, N), 1024, seed + 2, DEV)
    return sparse_exact(M, K, splits, seed, DEV), ints((N, K), 1, seed + 1, DEV), ints((M, N), 64, seed + 2, DEV)


def run(M, N, K, f32=False, pad=0, bn=0, splits=0, pm=0, pn=0, seed=0):
    from acco_b200.ops.gemm import gemm, gemm_wgrad_f32
    s = splits or pick(M, N, K)[1]
    A, B, C0 = operands(M, N, K, s, seed)
    dy, x = mn_major(A, pad, seed + 3), mn_major(B, pad, seed + 4)
    big, grad, guard = arena_view(C0.float() if f32 else C0, seed + 5)
    before = big.clone()
    if f32:
        gemm_wgrad_f32(dy, x, grad, bn=bn, splits=splits)
    else:
        gemm(dy, x, out=grad, a_mn=True, b_mn=True, accumulate=True, bn=bn, splits=splits, pm=pm, pn=pn)
    torch.cuda.synchronize()
    if f32:                                                   # integers below 2^24: the fp32 sum is exact
        want = (A.double() @ B.double().t() + C0.double()).float()
        assert torch.equal(grad, want)
    else:
        want = exact_result(A, B, C=C0)
        assert torch.equal(grad.view(torch.int16), want.view(torch.int16))
    assert torch.equal(big[guard], before[guard])


@pytest.mark.parametrize("f32", [False, True], ids=["bf16", "fp32"])
@pytest.mark.parametrize("name,M,N,T", SHAPES, ids=[s[0] for s in SHAPES])
def test_step_shapes_at_the_heuristic_pick(name, M, N, T, f32):
    run(M, N, T, f32=f32, seed=len(name))


def test_split_k_picks_are_covered():
    assert pick(768, 768, 8192) == (128, 3)                  # 125M o_proj
    assert pick(4096, 768, 8192) == (128, 2)                 # 125M gate|up


@pytest.mark.parametrize("f32", [False, True], ids=["bf16", "fp32"])
@pytest.mark.parametrize("M,N,K,bn,splits", [
    (200, 136, 1000, 0, 0),          # neither extent whole 64-element chunks: one 2-D box per chunk
    (320, 136, 1000, 0, 0),          # A folded, B per chunk
    (200, 192, 1000, 0, 0),          # A per chunk, B folded
    (320, 192, 2000, 128, 1),        # whole chunks, half a 128-row tile at the edge
    (384, 320, 3000, 64, 2),
    (448, 512, 4096, 256, 3),
])
def test_ragged_extents_and_tile_widths(M, N, K, bn, splits, f32):
    run(M, N, K, f32=f32, pad=0, bn=bn, splits=splits, seed=M + N)
    run(M, N, K, f32=f32, pad=40, bn=bn, splits=splits, seed=K)


@pytest.mark.parametrize("pm,pn", [(2, 1), (1, 2)])
def test_multicast_clusters(pm, pn):
    run(1024, 1024, 2048, bn=128, splits=1, pm=pm, pn=pn, seed=pm)
    run(1000, 1000, 2048, bn=128, splits=1, pm=pm, pn=pn, seed=pn)


@pytest.mark.parametrize("f32", [False, True], ids=["bf16", "fp32"])
def test_cuda_graph_replay(f32):
    from acco_b200.ops.gemm import gemm_tt_acc
    M, N, K = 768, 768, 8192                                  # the o_proj wgrad: three K splits
    A, B, C0 = operands(M, N, K, pick(M, N, K)[1], 7)
    dy, x = mn_major(A, 8, 8), mn_major(B, 8, 9)
    big, grad, guard = arena_view(C0.float() if f32 else C0, 10)
    before = big.clone()
    gemm_tt_acc(dy, x, grad)                                  # warm-up outside the capture: tensor maps, attributes
    grad.copy_(C0)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gemm_tt_acc(dy, x, grad)
    grad.copy_(C0)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    if f32:
        assert torch.equal(grad, (2 * (A.double() @ B.double().t()) + C0.double()).float())
    else:
        assert torch.equal(grad.view(torch.int16), exact_result(torch.cat([A, A], 1), torch.cat([B, B], 1), C=C0).view(torch.int16))
    assert torch.equal(big[guard], before[guard])
