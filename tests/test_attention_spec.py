"""CPU checks of the flash-attention specification and the glue of the own kernels (csrc/attention_wgmma.cu) - what can be verified
without a GPU:

* the blockwise schedule the kernels implement (``attention_blockwise_ref`` / ``attention_blockwise_bwd_ref``: delayed P V
  accumulation, running-max rescale, bf16 rounding points, dS scaling, GQA accumulation) against the fp32 reference + autograd;
* the block ranges of the forward / backward loops against a brute-force visibility test (causal and sliding window);
* the shared-memory images: what ``st_swz`` / a SWIZZLE_128B TMA box write versus what the wgmma shared-memory descriptors
  (K-major and MN-major views, the LBO / SBO / K-step constants of the kernel) address.  The address model is first checked on the
  two operand configurations that are proven on hardware by the GEMM tests (K-major boxes; MN-major {64, 64} boxes 8 KiB apart)."""
import numpy as np
import pytest
import torch

from acco_b200.ops.attention import (attention_blockwise_bwd_ref, attention_blockwise_ref, bwd_query_blocks, causal_attention_ref,
                                     fwd_key_blocks)


@pytest.mark.parametrize("B,S,Hq,Hk,window,scale", [(1, 256, 2, 1, None, None), (1, 384, 2, 2, 200, 1.0), (2, 256, 4, 2, 128, None)])
def test_blockwise_schedule_matches_reference(B, S, Hq, Hk, window, scale):
    torch.manual_seed(0)
    q, k, v = (torch.randn(B, S, h, 64, requires_grad=True) for h in (Hq, Hk, Hk))
    ref = causal_attention_ref(q, k, v, scale=scale, window=window)
    d_o = torch.randn_like(ref)
    gq, gk, gv = torch.autograd.grad(ref, (q, k, v), d_o)
    with torch.no_grad():
        o, lse = attention_blockwise_ref(q, k, v, scale, window)
        dq, dk, dv = attention_blockwise_bwd_ref(q, k, v, o, d_o, lse, scale, window)
    assert (o - ref).abs().max() < 1e-2
    sc = (64 ** -0.5) if scale is None else scale
    att = (q.detach().transpose(1, 2) @ k.detach().repeat_interleave(Hq // Hk, 2).transpose(1, 2).transpose(-1, -2)) * sc
    i = torch.arange(S)
    vis = (i[None, :] <= i[:, None]) & (i[None, :] > i[:, None] - (window or S))
    assert torch.allclose(lse, att.masked_fill(~vis, float("-inf")).logsumexp(-1), atol=1e-4)
    for got, want in ((dq, gq), (dk, gk), (dv, gv)):
        assert (got - want).abs().max() / want.abs().max() < 1e-2      # P / dS are rounded to bf16 before the gradient products


@pytest.mark.parametrize("S", [128, 512, 1024])
@pytest.mark.parametrize("window", [1, 64, 128, 129, 256, 300, 1024])
def test_block_ranges_cover_exactly_the_visible_pairs(S, window):
    win = min(window, S)
    nb = S // 128
    i = torch.arange(S)
    vis = (i[None, :] <= i[:, None]) & (i[None, :] + win > i[:, None])               # [q, kv]
    blocks = vis.view(nb, 128, nb, 128).any(dim=3).any(dim=1)                        # [q block, kv block]
    want = {(m, n) for m in range(nb) for n in range(nb) if blocks[m, n]}
    fwd = {(m, j) for m in range(nb) for j in fwd_key_blocks(m, S, win)}
    bwd = {(m, n) for n in range(nb) for m in bwd_query_blocks(n, S, win)}
    assert fwd == want and bwd == want


# ---------------------------------------------------------------------------------------------- shared-memory images
TILE = 128 * 128                     # bytes of a {64 bf16, 128 rows} box


def swz(off: int) -> int:
    """SWIZZLE_128B: byte-address bits [4,7) ^= bits [7,10) (tiles are 1024-byte aligned, so offsets behave like addresses)."""
    return off ^ (((off >> 7) & 7) << 4)


def tma_box_image(mat: np.ndarray) -> np.ndarray:
    """Image of a row-major [rows, 64] 2-byte matrix loaded as one SWIZZLE_128B box: row r at r * 128, 16-byte chunk c at c ^ (r & 7)
    - identical to what `st_swz(tile, r, c, v)` writes."""
    rows = mat.shape[0]
    img = np.zeros(rows * 64, dtype=mat.dtype)
    for r in range(rows):
        for c in range(8):
            dst = (r * 128 + ((c ^ (r & 7)) << 4)) // 2
            img[dst:dst + 8] = mat[r, c * 8:(c + 1) * 8]
    return img


def read_kmajor(img, base, row, k, sbo=1024, kstep=32):
    """Element (row, k) of a K-major SWIZZLE_128B operand whose descriptor starts at byte `base`; the MMA issuer advances the start
    address by `kstep` bytes per 16 k (k < 64 per 128-byte row)."""
    assert k < 64
    return img[swz(base + (k // 16) * kstep + (row % 8) * 128 + (row // 8) * sbo + (k % 16) * 2) // 2]


def read_mnmajor(img, base, mn, k, lbo, sbo=1024, kstep=2048):
    """Element (mn, k) of an MN-major SWIZZLE_128B operand: 64 mn contiguous in a 128-byte row, 8-k groups `sbo` apart,
    64-mn chunks `lbo` apart, +`kstep` bytes per 16 k."""
    return img[swz(base + (k // 16) * kstep + (mn % 64) * 2 + (mn // 64) * lbo + (k % 8) * 128 + ((k % 16) // 8) * sbo) // 2]


def test_address_model_reproduces_the_gemm_operands():
    rng = np.random.default_rng(0)
    a = rng.integers(0, 60000, size=(128, 64)).astype(np.uint16)      # K-major A tile: box {64 k, 128 rows}
    img = tma_box_image(a)
    assert all(read_kmajor(img, 0, r, k) == a[r, k] for r in range(0, 128, 7) for k in range(64))
    at = rng.integers(0, 60000, size=(64, 128)).astype(np.uint16)     # MN-major A^T [K=64, M=128]: two {64 m, 64 k} boxes, 8 KiB apart
    img = np.concatenate([tma_box_image(at[:, :64]), tma_box_image(at[:, 64:])])
    assert all(read_mnmajor(img, 0, m, k, lbo=8192) == at[k, m] for m in range(0, 128, 5) for k in range(64))


def test_attention_tiles_match_their_descriptor_views():
    rng = np.random.default_rng(1)
    # V / K / Q / dO tiles: one {64 d, 128 rows} box; MN-major view (N = d, contraction over the 128 rows), 8 K-steps of 2 KiB
    v = rng.integers(0, 60000, size=(128, 64)).astype(np.uint16)
    img = tma_box_image(v)
    assert all(read_mnmajor(img, 0, d, kv, lbo=TILE) == v[kv, d] for d in range(64) for kv in range(0, 128, 3))
    # P / dS tile [128 q, 128 kv] written by the softmax threads: two 64-column halves, 16 KiB apart
    p = rng.integers(0, 60000, size=(128, 128)).astype(np.uint16)
    img = np.concatenate([tma_box_image(p[:, :64]), tma_box_image(p[:, 64:])])
    for q in range(0, 128, 5):
        for kv in range(128):
            # K-major view (P V, dS K): the issuer picks the half with `sP + (k >> 2) * TILE` and steps 32 B inside it
            assert read_kmajor(img, (kv // 64) * TILE, q, kv % 64) == p[q, kv]
            # MN-major view (P^T dO, dS^T Q): M = kv with LBO = 16 KiB between the halves, contraction over q
            assert read_mnmajor(img, 0, kv, q, lbo=TILE) == p[q, kv]


def test_dq_staging_image_matches_an_fp32_box():
    """fp32 dQ staging: [32 rows x 32 floats] halves, 16-byte chunk j (4 floats) of row r at j ^ (r & 7) - the image a
    {32 fp32, 32 rows} SWIZZLE_128B box expects."""
    rng = np.random.default_rng(2)
    dq = rng.standard_normal((32, 32)).astype(np.float32)
    img = np.zeros(32 * 32, dtype=np.float32)
    for r in range(32):
        for j in range(8):
            dst = (r * 128 + ((j ^ (r & 7)) << 4)) // 4
            img[dst:dst + 4] = dq[r, j * 4:(j + 1) * 4]
    for r in range(32):
        for col in range(32):
            assert img[swz(r * 128 + col * 4) // 4] == dq[r, col]


# ---------------------------------------------------------------------------------------------- autograd glue of the opt-in path
class _FakeExt:
    """Stand-in for acco_b200._C on the CPU: the attention entry points backed by the blockwise specification, the RoPE kernels by
    their reference math.  Exercises `_RopeAttentionFn`'s own-kernel branch (ACCO_ATTN=own) end to end - argument order,
    saved tensors, packed d(qkv) layout, inverse rotation - everything except the CUDA kernels themselves."""

    @staticmethod
    def attn_supported(B, S, Hq, Hk, D, scale):
        return D == 64 and S % 128 == 0 and Hq % Hk == 0 and scale > 0

    @staticmethod
    def attn_fwd(qkv, B, S, Hq, Hk, D, sc, window):
        x = qkv.view(B, S, Hq + 2 * Hk, D)
        o, lse = attention_blockwise_ref(x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:], sc, window)
        return o.reshape(B * S, Hq * D), lse

    @staticmethod
    def attn_bwd(qkv, o, d_o, lse, B, S, Hq, Hk, D, sc, window):
        x = qkv.view(B, S, Hq + 2 * Hk, D)
        dq, dk, dv = attention_blockwise_bwd_ref(x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:], o.view(B, S, Hq, D), d_o.view(B, S, Hq, D),
                                                 lse, sc, window)
        return dq.reshape(B * S, Hq * D), dk.reshape(B * S, Hk * D), dv.reshape(B * S, Hk * D)

    @staticmethod
    def rope_qkv_inplace(qkv, cos, sin, B, S, n_rot, n_total, D, inverse):
        from acco_b200.ops.rope import apply_rope_ref
        x = qkv.view(B, S, n_total, D)
        x[:, :, :n_rot] = apply_rope_ref(x[:, :, :n_rot], cos, -sin if inverse else sin)

    @staticmethod
    def rope_pack_bwd(dq, dk, dv, cos, sin):
        from acco_b200.ops.rope import apply_rope_ref
        B, S = dq.shape[:2]
        return torch.cat([apply_rope_ref(dq, cos, -sin), apply_rope_ref(dk, cos, -sin), dv], dim=2).reshape(B * S, -1)


@pytest.mark.parametrize("rope,window,scale", [(True, None, None), (False, 160, 1.0)])
def test_own_attention_autograd_glue(monkeypatch, rope, window, scale):
    from acco_b200 import ops
    from acco_b200.ops import attention as A
    from acco_b200.ops.rope import rope_qkv_ref, rope_tables
    monkeypatch.setenv("ACCO_ATTN", "own")
    monkeypatch.setattr(ops, "load_ext", lambda required=False: _FakeExt)
    B, S, Hq, Hk, D = 2, 256, 4, 2, 64
    torch.manual_seed(1)
    qkv = (torch.randn(B * S, (Hq + 2 * Hk) * D) * 0.5).requires_grad_()
    cos, sin = rope_tables(S, D, 10000.0, "cpu") if rope else A._identity_tables(S, D, "cpu")
    d_o = torch.randn(B * S, Hq * D)
    x = qkv.clone()                                             # the op consumes (rotates) its input in place: differentiate through a clone
    out = A._RopeAttentionFn.apply(x, cos, sin, B, S, Hq, Hk, D, rope, scale, window)
    out.backward(d_o)
    got = qkv.grad.clone()
    # oracle: reference RoPE + fp32 attention, autograd end to end
    q2 = qkv.detach().clone().requires_grad_()
    y = rope_qkv_ref(q2, cos, sin, B, S, Hq, Hk, D) if rope else q2
    y = y.view(B, S, Hq + 2 * Hk, D)
    ref = causal_attention_ref(y[:, :, :Hq], y[:, :, Hq:Hq + Hk], y[:, :, Hq + Hk:], scale=scale, window=window).reshape(B * S, Hq * D)
    ref.backward(d_o)
    assert (out - ref).abs().max() < 2e-2
    assert (got - q2.grad).abs().max() / q2.grad.abs().max() < 2e-2


def test_attn_supported_matrix():
    """Which shapes the kernels claim (host predicate `acco_attn_supported`, callable on a CPU): head_dim 64, S a multiple of the
    128-row tile, grouped-query heads dividing evenly, positive scale.  Everything else must fall back to the library path."""
    import ctypes
    import os
    so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "acco_b200", "_C.so")
    if not os.path.exists(so):
        pytest.skip("extension not built")
    try:
        fn = ctypes.CDLL(so).acco_attn_supported
    except OSError as e:
        pytest.skip(f"extension not loadable here: {e}")
    fn.argtypes = [ctypes.c_int] * 5 + [ctypes.c_float]
    fn.restype = ctypes.c_int
    ok = lambda B, S, Hq, Hk, D, sc=0.125: bool(fn(B, S, Hq, Hk, D, sc))
    assert ok(8, 1024, 12, 12, 64) and ok(2, 8192, 32, 8, 64) and ok(1, 128, 1, 1, 64) and ok(4, 512, 12, 12, 64, 1.0)
    assert not ok(8, 1024, 32, 8, 128)            # Llama-3-8B head_dim
    assert not ok(8, 1000, 12, 12, 64)            # S not a multiple of 128
    assert not ok(8, 1024, 12, 5, 64)             # heads do not group evenly
    assert not ok(8, 1024, 12, 12, 64, 0.0) and not ok(0, 1024, 12, 12, 64)
