"""Causal (optionally sliding-window) self-attention.

Default path: library flash kernels (cuDNN / flash through ``scaled_dot_product_attention``, flash-attn for sliding windows).
The reference uses the HF attention dispatch (`modeling_llama.py:272`) or eager fp32 attention for GPT-Neo
(`modeling_gpt_neo.py:105-130`, including its missing 1/sqrt(d) scale and the 256-token local window on odd layers - both
reproduced through ``scale`` / ``window``).

``ACCO_ATTN=own`` switches the fused-QKV attention block to the repo's own flash-attention kernels
(``csrc/attention_wgmma.cu``: forward + backward on the tensor cores, head_dim 64, S a multiple of 128).  ``tools/attn_check.py``
compares them with the fp32 reference, and :func:`attention_blockwise_ref` / :func:`attention_blockwise_bwd_ref` below give the
reference semantics of their masking and bf16 rounding points (CPU-tested against the fp32 reference)."""
from __future__ import annotations

import math
import os
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

_SDPA_BACKENDS = None


def _sdpa_ctx():
    global _SDPA_BACKENDS
    from torch.nn.attention import SDPBackend, sdpa_kernel
    if _SDPA_BACKENDS is None:
        _SDPA_BACKENDS = [SDPBackend.CUDNN_ATTENTION, SDPBackend.FLASH_ATTENTION, SDPBackend.EFFICIENT_ATTENTION, SDPBackend.MATH]
    try:
        return sdpa_kernel(_SDPA_BACKENDS, set_priority=True)
    except TypeError:  # older signature
        return sdpa_kernel(_SDPA_BACKENDS)


def _window_mask(S: int, window: int, device) -> torch.Tensor:
    i = torch.arange(S, device=device)[:, None]
    j = torch.arange(S, device=device)[None, :]
    return (j <= i) & (j > i - window)


def causal_attention_ref(q, k, v, scale: Optional[float] = None, window: Optional[int] = None):
    """q [B,S,Hq,D], k/v [B,S,Hk,D] -> [B,S,Hq,D]; fp32 math."""
    B, S, Hq, D = q.shape
    Hk = k.shape[2]
    qf, kf, vf = (t.float().transpose(1, 2) for t in (q, k, v))
    if Hk != Hq:
        kf = kf.repeat_interleave(Hq // Hk, dim=1)
        vf = vf.repeat_interleave(Hq // Hk, dim=1)
    sc = (1.0 / math.sqrt(D)) if scale is None else scale
    att = qf @ kf.transpose(-1, -2) * sc
    mask = _window_mask(S, window if window else S, q.device)
    att = att.masked_fill(~mask, float("-inf")).softmax(-1)
    return (att @ vf).transpose(1, 2).to(q.dtype)


def causal_attention(q, k, v, scale: Optional[float] = None, window: Optional[int] = None):
    """q [B,S,Hq,D], k/v [B,S,Hk,D] (strided views allowed) -> [B,S,Hq,D] contiguous."""
    B, S, Hq, D = q.shape
    Hk = k.shape[2]
    if window is not None and window >= S:
        window = None
    if q.is_cuda and window is not None:
        try:
            from flash_attn import flash_attn_func
            return flash_attn_func(q, k, v, softmax_scale=scale, causal=True, window_size=(window - 1, 0))
        except Exception:
            pass
    qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    kw = {}
    if Hk != Hq:
        kw["enable_gqa"] = True
    if window is None:
        if q.is_cuda:
            with _sdpa_ctx():
                o = F.scaled_dot_product_attention(qt, kt, vt, is_causal=True, scale=scale, **kw)
        else:
            o = F.scaled_dot_product_attention(qt, kt, vt, is_causal=True, scale=scale, **kw)
    else:
        mask = _window_mask(S, window, q.device)
        o = F.scaled_dot_product_attention(qt, kt, vt, attn_mask=mask, scale=scale, **kw)
    return o.transpose(1, 2).contiguous()


def own_attention_enabled() -> bool:
    """``ACCO_ATTN=own``: route the fused-QKV attention block through ``csrc/attention_wgmma.cu``."""
    return os.environ.get("ACCO_ATTN", "").lower() == "own"


# ----------------------------------------------------------------------------------------------
# Executable specification of a blockwise flash attention: 128 queries x 128 keys per tile, the order of operations
# (row max of the raw scores -> accumulate the PREVIOUS block's P V -> rescale -> exponentials of this block), the same masking
# rule, the same places where values are rounded to bf16 (P, dS, outputs).  fp32 everywhere else.
# ----------------------------------------------------------------------------------------------
_BLK = 128
_LOG2E = 1.4426950408889634
_LN2 = 0.6931471805599453


def _bf16_round(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16).float()


def _block_mask(q0: int, kv0: int, window: int, device) -> torch.Tensor:
    q = torch.arange(q0, q0 + _BLK, device=device)[:, None]
    kv = torch.arange(kv0, kv0 + _BLK, device=device)[None, :]
    return (kv <= q) & (kv + window > q)


def fwd_key_blocks(qb: int, S: int, window: int) -> range:
    """Key blocks visited by the forward CTA of query block ``qb`` (`attn_fwd_kernel`: ``j_lo .. qb``)."""
    lo = qb * _BLK - window + 1
    return range(lo // _BLK if lo > 0 else 0, qb + 1)


def bwd_query_blocks(n: int, S: int, window: int) -> range:
    """Query blocks visited by the backward CTA of key block ``n`` (`attn_bwd_kernel`: ``n .. m_hi``)."""
    return range(n, min(S // _BLK - 1, (n * _BLK + _BLK - 2 + window) // _BLK) + 1)


def attention_blockwise_ref(q, k, v, scale: Optional[float] = None, window: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """q [B,S,Hq,64], k/v [B,S,Hk,64], S % 128 == 0 -> (o [B,S,Hq,64] in q.dtype, lse [B,Hq,S] fp32 natural log).
    Mirrors ``attn_fwd_kernel`` (one loop body = one CTA's softmax thread group)."""
    B, S, Hq, D = q.shape
    Hk = k.shape[2]
    assert S % _BLK == 0 and Hq % Hk == 0
    sc = (1.0 / math.sqrt(D)) if scale is None else float(scale)
    c = sc * _LOG2E
    win = S if (window is None or window <= 0 or window > S) else int(window)
    o = torch.empty(B, S, Hq, D, dtype=torch.float32, device=q.device)
    lse = torch.empty(B, Hq, S, dtype=torch.float32, device=q.device)
    for b in range(B):
        for h in range(Hq):
            g = h // (Hq // Hk)
            for qb in range(S // _BLK):
                q0 = qb * _BLK
                Q = q[b, q0:q0 + _BLK, h].float()
                m_run = torch.full((_BLK,), -1e30)
                l_run = torch.zeros(_BLK)
                O = torch.zeros(_BLK, D)
                pending = None                                   # P_{i-1} V_{i-1}: issued, read back one iteration later
                for j in fwd_key_blocks(qb, S, win):
                    kv0 = j * _BLK
                    Sraw = Q @ k[b, kv0:kv0 + _BLK, g].float().T
                    vis = _block_mask(q0, kv0, win, q.device)
                    mx = Sraw.masked_fill(~vis, float("-inf")).max(dim=1).values
                    m_new = torch.maximum(m_run, mx * c)
                    alpha = torch.exp2(m_run - m_new)
                    if pending is not None:
                        O = (O + pending) * alpha[:, None]
                    l_run = l_run * alpha
                    m_run = m_new
                    Pm = torch.exp2(Sraw * c - m_new[:, None]).masked_fill(~vis, 0.0)
                    l_run = l_run + Pm.sum(dim=1)
                    pending = _bf16_round(Pm) @ v[b, kv0:kv0 + _BLK, g].float()
                O = (O + pending) / l_run[:, None]
                o[b, q0:q0 + _BLK, h] = O
                lse[b, h, q0:q0 + _BLK] = (m_run + torch.log2(l_run)) * _LN2
    return o.to(q.dtype), lse


def attention_blockwise_bwd_ref(q, k, v, o, d_o, lse, scale: Optional[float] = None, window: Optional[int] = None):
    """Mirrors ``attn_bwd_kernel``: K_n / V_n stationary, loop over (query head of the GQA group, query block m >= n);
    P and dS rounded to bf16 before the three gradient products; dQ accumulated in fp32 across key blocks.
    -> (dq fp32 [B,S,Hq,64], dk, dv in q.dtype [B,S,Hk,64])."""
    B, S, Hq, D = q.shape
    Hk = k.shape[2]
    G = Hq // Hk
    sc = (1.0 / math.sqrt(D)) if scale is None else float(scale)
    c = sc * _LOG2E
    win = S if (window is None or window <= 0 or window > S) else int(window)
    nqb = S // _BLK
    delta = (d_o.float() * o.float()).sum(-1).permute(0, 2, 1)            # [B, Hq, S]
    dq = torch.zeros(B, S, Hq, D, dtype=torch.float32, device=q.device)
    dk = torch.empty(B, S, Hk, D, dtype=torch.float32, device=q.device)
    dv = torch.empty(B, S, Hk, D, dtype=torch.float32, device=q.device)
    for b in range(B):
        for g in range(Hk):
            for n in range(nqb):
                kv0 = n * _BLK
                K = k[b, kv0:kv0 + _BLK, g].float()
                V = v[b, kv0:kv0 + _BLK, g].float()
                dK = torch.zeros(_BLK, D)
                dV = torch.zeros(_BLK, D)
                for gi in range(G):
                    hq = g * G + gi
                    for m in bwd_query_blocks(n, S, win):
                        q0 = m * _BLK
                        Q = q[b, q0:q0 + _BLK, hq].float()
                        dO = d_o[b, q0:q0 + _BLK, hq].float()
                        L2 = lse[b, hq, q0:q0 + _BLK] * _LOG2E
                        dl = delta[b, hq, q0:q0 + _BLK]
                        vis = _block_mask(q0, kv0, win, q.device)
                        Pm = torch.exp2((Q @ K.T) * c - L2[:, None]).masked_fill(~vis, 0.0)
                        dS = Pm * ((dO @ V.T) - dl[:, None]) * sc
                        Pb, dSb = _bf16_round(Pm), _bf16_round(dS)
                        dV += Pb.T @ dO
                        dK += dSb.T @ Q
                        dq[b, q0:q0 + _BLK, hq] += dSb @ K
                dk[b, kv0:kv0 + _BLK, g] = dK
                dv[b, kv0:kv0 + _BLK, g] = dV
    return dq, dk.to(q.dtype), dv.to(q.dtype)


# ----------------------------------------------------------------------------------------------
# Fused attention block for the native Llama: RoPE (in place on the fused QKV buffer) + SDPA, with a
# backward that gathers dq/dk/dv into ONE d(qkv) buffer while applying the inverse rotation
# (``csrc/elementwise.cu: rope_pack_bwd_kernel``).  Autograd's default for three slices of one tensor is
# zero-fill + slice-copy + add per slice (~400 MB of traffic per layer at 8x1024x768); this is one pass.
# ----------------------------------------------------------------------------------------------

def _sdpa(qt, kt, vt, scale, gqa: bool):
    kw = {"enable_gqa": True} if gqa else {}
    if qt.is_cuda:
        with _sdpa_ctx():
            return F.scaled_dot_product_attention(qt, kt, vt, is_causal=True, scale=scale, **kw)
    return F.scaled_dot_product_attention(qt, kt, vt, is_causal=True, scale=scale, **kw)


def _attend(q, k, v, scale, window, gqa: bool):
    """q [B,Hq,S,D] / k, v [B,Hk,S,D] (strided views) -> [B,Hq,S,D]; causal, optional sliding window."""
    S = q.shape[2]
    if window is not None and window < S:
        if q.is_cuda:
            try:
                from flash_attn import flash_attn_func
                o = flash_attn_func(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), softmax_scale=scale, causal=True,
                                    window_size=(window - 1, 0))
                return o.transpose(1, 2)
            except ImportError:
                pass
        kw = {"enable_gqa": True} if gqa else {}
        return F.scaled_dot_product_attention(q, k, v, attn_mask=_window_mask(S, window, q.device), scale=scale, **kw)
    kw = {"enable_gqa": True} if gqa else {}
    if q.is_cuda:
        with _sdpa_ctx():
            return F.scaled_dot_product_attention(q, k, v, is_causal=True, scale=scale, **kw)
    return F.scaled_dot_product_attention(q, k, v, is_causal=True, scale=scale, **kw)


_IDENT_TABLES = {}


def _identity_tables(S: int, D: int, device):
    """cos = 1, sin = 0: turns the RoPE kernels into pure (un)packing kernels for models without rotary embeddings."""
    key = (S, D, str(device))
    if key not in _IDENT_TABLES:
        _IDENT_TABLES[key] = (torch.ones(S, D // 2, device=device, dtype=torch.float32), torch.zeros(S, D // 2, device=device, dtype=torch.float32))
    return _IDENT_TABLES[key]


class _RopeAttentionFn(torch.autograd.Function):
    """Attention block on the fused QKV buffer: optional RoPE in place, attention on strided head views, and a backward that
    gathers dq/dk/dv into ONE packed d(qkv) buffer (with the inverse rotation) instead of autograd's zero-fill + slice-add chain."""

    @staticmethod
    def forward(ctx, qkv, cos, sin, B, S, Hq, Hk, D, rope=True, scale=None, window=None):
        from . import count_launch, load_ext
        C = load_ext(required=True)
        # `qkv` is CONSUMED: rotated in place without telling autograd (no mark_dirty - the inner SDPA graph
        # below saves views of it, and a version bump would invalidate them).  Contract: the caller hands
        # over the fresh output of the QKV GEMM and never reads it again (LinearFn does not save its output).
        if rope:
            C.rope_qkv_inplace(qkv, cos, sin, B, S, Hq + Hk, Hq + 2 * Hk, D, False)
            count_launch("rope_qkv")
        sc = (1.0 / math.sqrt(D)) if scale is None else float(scale)
        if own_attention_enabled() and C.attn_supported(B, S, Hq, Hk, D, sc):
            o, lse = C.attn_fwd(qkv.detach(), B, S, Hq, Hk, D, sc, int(window or 0))
            count_launch("attn_fwd")
            ctx.inner = None
            ctx.own = (qkv.detach(), o, lse, sc, int(window or 0))
            ctx.dims = (B, S, Hq, Hk, D)
            ctx.save_for_backward(cos, sin)
            return o
        ctx.own = None
        x = qkv.detach().view(B, S, Hq + 2 * Hk, D)
        with torch.enable_grad():
            q = x[:, :, :Hq].transpose(1, 2).requires_grad_()
            k = x[:, :, Hq:Hq + Hk].transpose(1, 2).requires_grad_()
            v = x[:, :, Hq + Hk:].transpose(1, 2).requires_grad_()
            out = _attend(q, k, v, scale, window, Hk != Hq)          # [B, Hq, S, D]
        ctx.inner = (out, q, k, v)
        ctx.dims = (B, S, Hq, Hk, D)
        ctx.save_for_backward(cos, sin)
        return out.detach().transpose(1, 2).reshape(B * S, Hq * D)

    @staticmethod
    def backward(ctx, dout):
        from . import count_launch, load_ext
        C = load_ext(required=True)
        cos, sin = ctx.saved_tensors
        B, S, Hq, Hk, D = ctx.dims
        if ctx.own is not None:
            qkv, o, lse, sc, window = ctx.own
            ctx.own = None
            dq, dk, dv = C.attn_bwd(qkv, o, dout.contiguous(), lse, B, S, Hq, Hk, D, sc, window)
            count_launch("attn_bwd", 2)
            dqkv = C.rope_pack_bwd(dq.to(torch.bfloat16).view(B, S, Hq, D), dk.view(B, S, Hk, D), dv.view(B, S, Hk, D), cos, sin)
            count_launch("rope_pack_bwd")
            return (dqkv,) + (None,) * 10
        out, q, k, v = ctx.inner
        ctx.inner = None
        do = dout.reshape(B, S, Hq, D).transpose(1, 2)
        dq, dk, dv = torch.autograd.grad(out, (q, k, v), do)
        dq, dk, dv = (t if t.stride(-1) == 1 else t.contiguous() for t in (dq, dk, dv))
        dqkv = C.rope_pack_bwd(dq.transpose(1, 2), dk.transpose(1, 2), dv.transpose(1, 2), cos, sin)
        count_launch("rope_pack_bwd")
        return (dqkv,) + (None,) * 10


def rope_causal_attention(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, B: int, S: int, Hq: int, Hk: int, D: int) -> torch.Tensor:
    """``qkv [B*S, (Hq+2Hk)*D]`` (output of the fused QKV GEMM; consumed/modified in place on CUDA)
    -> attention output ``[B*S, Hq*D]``."""
    from . import use_kernels
    from .rope import rope_qkv_ref
    if use_kernels(qkv):
        if torch.is_grad_enabled() and qkv.requires_grad:
            return _RopeAttentionFn.apply(qkv, cos, sin, B, S, Hq, Hk, D)
        from . import count_launch, load_ext
        load_ext(required=True).rope_qkv_inplace(qkv, cos, sin, B, S, Hq + Hk, Hq + 2 * Hk, D, False)
        count_launch("rope_qkv")
        x = qkv.view(B, S, Hq + 2 * Hk, D)
        out = _sdpa(x[:, :, :Hq].transpose(1, 2), x[:, :, Hq:Hq + Hk].transpose(1, 2), x[:, :, Hq + Hk:].transpose(1, 2), None, Hk != Hq)
        return out.transpose(1, 2).reshape(B * S, Hq * D)
    x = rope_qkv_ref(qkv, cos, sin, B, S, Hq, Hk, D).view(B, S, Hq + 2 * Hk, D)
    return causal_attention(x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:]).reshape(B * S, Hq * D)


def packed_causal_attention(qkv: torch.Tensor, B: int, S: int, Hq: int, Hk: int, D: int, scale=None, window=None) -> torch.Tensor:
    """Attention on a fused ``qkv [B*S, (Hq+2Hk)*D]`` buffer WITHOUT rotary embeddings (GPT-2 / GPT-Neo: learned positions;
    ``scale`` 1.0 and a 256-token ``window`` on the local layers reproduce `modeling_gpt_neo.py:105-130`) -> ``[B*S, Hq*D]``.
    On CUDA the backward packs dq/dk/dv into one d(qkv) buffer in a single pass (``rope_pack_bwd`` with identity tables)."""
    from . import use_kernels
    if use_kernels(qkv) and D % 16 == 0 and torch.is_grad_enabled() and qkv.requires_grad:
        cos, sin = _identity_tables(S, D, qkv.device)
        return _RopeAttentionFn.apply(qkv, cos, sin, B, S, Hq, Hk, D, False, scale, window)
    x = qkv.view(B, S, Hq + 2 * Hk, D)
    return causal_attention(x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:], scale=scale, window=window).reshape(B * S, Hq * D)
