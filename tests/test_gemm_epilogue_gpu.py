"""The GEMM epilogue (csrc/gemm_wgmma.cu): outputs staged through shared memory and written by TMA stores, beta = 1 with one K split
read through a TMA load and rounded once, split-K partials added by bulk tensor reduce-adds, and the L2-aware tile order."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from acco_b200.ops.gemm import gemm, gemm_tn  # noqa: E402

DEV = "cuda"


def rnd(*s, seed=0, scale=0.5):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*s, device=DEV, generator=g) * scale).to(torch.bfloat16)


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """one bf16 ulp at the magnitude of x (x fp32)"""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def test_single_split_accumulate_into_zero_is_bit_identical_to_store():
    M, N, K = 1000, 776, 4096
    dy, x = rnd(K, M, seed=1), rnd(K, N, seed=2)
    ref = gemm(dy, x, a_mn=True, b_mn=True, splits=1)
    acc = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
    gemm(dy, x, out=acc, a_mn=True, b_mn=True, accumulate=True, splits=1)
    assert torch.equal(ref, acc)


@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("M,N", [(1000, 776), (2304, 768), (136, 72)])
def test_accumulate_into_strided_view_one_rounding(bn, M, N):
    K = 2048
    dy, x = rnd(K, M, seed=3), rnd(K, N, seed=4)
    big = rnd(M + 3, N + 24, seed=5)
    before = big.clone()
    view = big[1:M + 1, 8:N + 8]
    c = view.float().clone()
    gemm(dy, x, out=view, a_mn=True, b_mn=True, accumulate=True, bn=bn, splits=1)
    want = c + dy.float().t() @ x.float()
    err = (view.float() - want).abs()
    assert bool((err <= ulp_bf16(want) * 1.01 + 1e-3).all()), float(err.max())
    mask = torch.ones_like(big, dtype=torch.bool)
    mask[1:M + 1, 8:N + 8] = False
    assert torch.equal(big[mask], before[mask])          # nothing around the view was written


@pytest.mark.parametrize("splits", [2, 3, 8])
def test_split_k_partials(splits):
    M, N, K = 768, 776, 8192
    dy, x = rnd(K, M, seed=6), rnd(K, N, seed=7)
    big = rnd(M, N + 16, seed=8)
    view = big[:, 8:N + 8]
    c = view.float().clone()
    gemm(dy, x, out=view, a_mn=True, b_mn=True, accumulate=True, splits=splits)
    want = c + dy.float().t() @ x.float()
    torch.testing.assert_close(view.float(), want, rtol=2e-2, atol=splits * 0.25)
    assert torch.equal(big[:, :8], rnd(M, N + 16, seed=8)[:, :8])


@pytest.mark.parametrize("bn", [64, 128, 256])
def test_bias_with_ragged_n(bn):
    M, N, K = 333, 200, 768
    x, w, b = rnd(M, K, seed=9), rnd(N, K, seed=10), rnd(N, seed=11)
    y = gemm(x, w, bias=b, bn=bn)
    want = x.float() @ w.float().t() + b.float()
    torch.testing.assert_close(y.float(), want, rtol=2e-2, atol=5e-2)


def test_lm_head_forward_deterministic():
    M, N, K = 8192, 50304, 768
    x, w = rnd(M, K, seed=12), rnd(N, K, seed=13, scale=0.05)
    y1 = gemm_tn(x, w)
    y2 = gemm_tn(x, w)
    assert torch.equal(y1, y2)
    rows = torch.tensor([0, 1, 127, 128, 4095, 8191], device=DEV)
    want = x[rows].float() @ w.float().t()
    torch.testing.assert_close(y1[rows].float(), want, rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("pm,pn", [(2, 1), (1, 2), (2, 2)])
@pytest.mark.parametrize("kind", ["tn", "tt_acc"])
def test_multicast_clusters_match_fp32(pm, pn, kind):
    if kind == "tn":
        M, N, K = 1000, 776, 1024
        a, b = rnd(M, K, seed=14), rnd(N, K, seed=15)
        y = gemm(a, b, pm=pm, pn=pn, bn=128)
        want = a.float() @ b.float().t()
    else:
        M, N, K = 1000, 776, 2048
        a, b = rnd(K, M, seed=16), rnd(K, N, seed=17)
        y = rnd(M, N, seed=18)
        want = y.float() + a.float().t() @ b.float()
        gemm(a, b, out=y, a_mn=True, b_mn=True, accumulate=True, pm=pm, pn=pn, bn=128, splits=1)
    torch.testing.assert_close(y.float(), want, rtol=2e-2, atol=5e-2)
