"""The flash-attention kernels (``csrc/attention_wgmma.cu``: ``attn_fwd_kernel`` / ``attn_bwd_kernel``, plain and document-masked)
and their autograd glue against the fp64 oracle of ``test_attention_oracle.py``, at the shapes, windows and row layouts the models
run: a single tile and GQA 4:1, GPT-Neo (scale 1.0, every window edge), Llama-125M, Llama-3.2-1B rows up to 8192 tokens, and packed
rows with sample boundaries on the warpgroup and CTA edges.  The kernels are called directly, so they run whatever ``ACCO_ATTN`` says.

* dense: O, LSE, dQ, dK, dV within ``TOL`` (the margin table shows an honest bf16 kernel passes with half of it to spare);
* mask-edge probes: a planted key that dominates the softmax, just outside each mask edge (where a leak moves O by about 64 or blows
  up the key's dK / dV rows) and just inside it (where the oracle shows the probe is live);
* exactness: two launches agree bit for bit (dQ, summed by fp32 atomics, to 1e-6), and a sample that fills whole 128-row blocks of a
  packed row gives the unsegmented kernels' bits on the same sample alone;
* the autograd glue (RoPE, packed rows, ``ACCO_ATTN=own``) and the SDPA fallback of packed rows with head_dim 128."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops

from test_attention_oracle import (GPTNEO_WINDOWS, PLANT_V, SEG_KINDS, TOL, check_probes_live, dense_errors, doc_ids, heads_of,
                                   make_qkv, oracle, plant, probe_bwd_ratios, probe_fwd_ratios, probe_slots, probes, row_lengths,
                                   seg_starts_of, split, visibility)

DEV = "cuda"
D = 64


def _ext():
    return ops.load_ext(required=True)


def run_kernels(qkv, d_o, B, S, Hq, Hk, scale, window, seg=None):
    """Both kernels on one input -> the oracle's layout: o [B,S,Hq,D], lse [B,Hq,S], dq [B,S,Hq,D], dk / dv [B,S,Hk,D]."""
    C = _ext()
    extra = () if seg is None else (seg.to(DEV),)
    o, lse = C.attn_fwd(qkv, B, S, Hq, Hk, D, scale, window, *extra)
    out = {"o": o.view(B, S, Hq, D), "lse": lse}
    if d_o is not None:
        dq, dk, dv = C.attn_bwd(qkv, o, d_o, lse, B, S, Hq, Hk, D, scale, window, *extra)
        out.update(dq=dq.view(B, S, Hq, D), dk=dk.view(B, S, Hk, D), dv=dv.view(B, S, Hk, D))
    torch.cuda.synchronize()
    return out


def _report(name, errs):
    print(f"[attn] {name}: " + " ".join(f"{k}={v:.2e}/{TOL[k]:.1e}" for k, v in errs.items()))


def check_dense(name, B, S, Hq, Hk, scale, window, lengths=None, groups=None, seed=0):
    qkv, d_o = (t.to(DEV) for t in make_qkv(B, S, Hq, Hk, seed=seed))
    seg = None if lengths is None else seg_starts_of(lengths, S)
    got = run_kernels(qkv, d_o, B, S, Hq, Hk, scale, window, seg)
    doc = doc_ids(lengths or [[S]] * B, S).to(DEV)
    q, k, v = split(qkv, B, S, Hq, Hk)
    want = oracle(q, k, v, d_o.view(B, S, Hq, D), scale, visibility(doc, window), groups=groups)
    if groups is not None:
        hs = heads_of(groups, Hq, Hk)
        got = {"o": got["o"][:, :, hs], "lse": got["lse"][:, hs], "dq": got["dq"][:, :, hs], "dk": got["dk"][:, :, list(groups)],
               "dv": got["dv"][:, :, list(groups)]}
    errs = dense_errors(got, want)
    _report(name, errs)
    for n, e in errs.items():
        assert e < TOL[n], (name, n, e, TOL[n])


# ---------------------------------------------------------------------------------------------- a. dense comparison
@pytest.mark.parametrize("B,S,Hq,Hk", [(1, 128, 1, 1), (2, 256, 4, 1)])
def test_dense_small_and_gqa(B, S, Hq, Hk):
    check_dense(f"B{B} S{S} {Hq}/{Hk}", B, S, Hq, Hk, 0.125, 0, seed=S)


@pytest.mark.parametrize("window", GPTNEO_WINDOWS)
def test_dense_gptneo_scale1(window):
    check_dense(f"gpt-neo w{window}", 2, 1024, 12, 12, 1.0, window, seed=window)


def test_dense_llama125m():
    check_dense("llama-125m", 8, 1024, 12, 12, 0.125, 0, seed=1)


@pytest.mark.parametrize("S", [2048, 4096, 8192])
def test_dense_llama32_1b_long_rows(S):
    """32 query heads over 8 KV heads; the oracle computes the first and the last KV group."""
    check_dense(f"llama-3.2-1b S{S}", 1, S, 32, 8, 0.125, 0, groups=[0, 7], seed=S)


@pytest.mark.parametrize("scale", [1.0, 0.125])
@pytest.mark.parametrize("window", [0, 256])
@pytest.mark.parametrize("kind", SEG_KINDS)
def test_dense_segmented(kind, window, scale):
    B, S = 2, 1024
    check_dense(f"seg {kind} w{window} s{scale}", B, S, 4, 2, scale, window, lengths=row_lengths(kind, B, S, seed=window + 3),
                seed=window + int(8 * scale))


# ---------------------------------------------------------------------------------------------- b. mask-edge probes
def _probe_cases():
    cs = [(1.0, w, None) for w in GPTNEO_WINDOWS] + [(0.125, 256, None)]
    cs += [(sc, w, kind) for kind in SEG_KINDS for w in (0, 256) for sc in (1.0, 0.125)]
    return cs


@pytest.mark.parametrize("scale,window,kind", _probe_cases(), ids=lambda x: str(x))
def test_mask_edge_probes(scale, window, kind):
    B, S = 2, 1024
    row = None if kind is None else row_lengths(kind, 1, S, seed=window + 5)[0]
    lengths = [row] * B if row is not None else None
    seg = None if row is None else seg_starts_of(lengths, S)
    pl = probes(S, window, row, B)
    H = probe_slots(pl, B)
    vis = visibility(doc_ids(lengths or [[S]] * B, S), window).to(DEV)
    # forward: the planted key carries 64 in every dim; a leak moves O by about 64 and the LSE by about 128 * scale
    fq, _ = make_qkv(B, S, H, H, seed=11)
    placed = plant(fq, None, B, S, H, pl, PLANT_V)
    fq = fq.to(DEV)
    want = oracle(*split(fq, B, S, H, H), None, scale, vis)
    check_probes_live(want, placed)
    got = run_kernels(fq, None, B, S, H, H, scale, window, seg)
    r = probe_fwd_ratios(got, want, placed)
    # backward: a large dO on the queries that must not see the key; a leak there swamps the key's dK / dV rows
    bq, bd = make_qkv(B, S, H, H, seed=12)
    plant(bq, bd, B, S, H, pl, None)
    bq, bd = bq.to(DEV), bd.to(DEV)
    got = run_kernels(bq, bd, B, S, H, H, scale, window, seg)
    want = oracle(*split(bq, B, S, H, H), bd.view(B, S, H, D), scale, vis)
    r.update(probe_bwd_ratios(got, want, placed))
    print(f"[attn] probes s{scale} w{window} {kind} ({len(pl)} probes): " + " ".join(f"{k}={v:.2f}" for k, v in r.items()))
    for k, v in r.items():
        assert v <= 1.0, (k, v, [p["kind"] for p in pl])


# ---------------------------------------------------------------------------------------------- c. exactness
@pytest.mark.parametrize("kind", [None, "edges"])
def test_two_launches_are_bitwise_identical(kind):
    B, S, Hq, Hk, window = 2, 1024, 12, 4, 256
    qkv, d_o = (t.to(DEV) for t in make_qkv(B, S, Hq, Hk, seed=21))
    seg = None if kind is None else seg_starts_of(row_lengths(kind, B, S), S)
    a = run_kernels(qkv, d_o, B, S, Hq, Hk, 1.0, window, seg)
    b = run_kernels(qkv, d_o, B, S, Hq, Hk, 1.0, window, seg)
    for n in ("o", "lse", "dk", "dv"):
        assert torch.equal(a[n], b[n]), n
    torch.testing.assert_close(b["dq"], a["dq"], rtol=1e-6, atol=1e-6 * float(a["dq"].abs().max()))


@pytest.mark.parametrize("window,scale", [(0, 0.125), (256, 1.0), (100, 0.125)])
def test_block_aligned_sample_matches_the_unsegmented_kernels(window, scale):
    """A sample filling rows [256, 640) of packed row 1 (whole 128-row blocks, a = 2, b = 5): the segmented kernels visit the same
    key / query blocks in the same order as the unsegmented kernels on that sample alone in a row of 384, so O, LSE, dK and dV agree
    bit for bit."""
    B, S, Hq, Hk = 2, 1024, 4, 2
    lengths = [[1024], [256, 384, 384]]
    a0, a1 = 1 * S + 256, 1 * S + 640
    qkv, d_o = (t.to(DEV) for t in make_qkv(B, S, Hq, Hk, seed=31))
    packed = run_kernels(qkv, d_o, B, S, Hq, Hk, scale, window, seg_starts_of(lengths, S))
    alone = run_kernels(qkv[a0:a1].contiguous(), d_o[a0:a1].contiguous(), 1, 384, Hq, Hk, scale, window)
    for n in ("o", "dk", "dv", "dq"):
        got = packed[n].reshape(B * S, -1)[a0:a1]
        want = alone[n].reshape(384, -1)
        if n == "dq":
            torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-6 * float(want.abs().max()))
        else:
            assert torch.equal(got, want), n
    assert torch.equal(packed["lse"][1, :, 256:640], alone["lse"][0])


# ---------------------------------------------------------------------------------------------- d. autograd glue
def _rope64(x, pos, theta=500000.0):
    """Rotate-half RoPE in fp64 from positions: x [B,S,H,d], pos [B,S]."""
    d = x.shape[-1]
    inv = theta ** (-torch.arange(0, d, 2, dtype=torch.float64, device=x.device) / d)
    ang = pos.double()[:, :, None, None] * inv
    c, s = torch.cos(ang), torch.sin(ang)
    x1, x2 = x[..., :d // 2], x[..., d // 2:]
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1)


def _glue_oracle(qkv, d_o, B, S, Hq, Hk, d, scale, window, lengths, pos, rope):
    """Oracle of the whole attention block on a fused qkv buffer: (RoPE from positions) -> attention -> d(qkv)."""
    x = qkv.double().view(B, S, Hq + 2 * Hk, d).requires_grad_()
    q, k, v = x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:]
    qr, kr = (_rope64(q, pos), _rope64(k, pos)) if rope else (q, k)
    vis = visibility(doc_ids(lengths, S), window).to(qkv.device)
    w = oracle(qr.detach(), kr.detach(), v.detach(), d_o.view(B, S, Hq, d), scale, vis)
    g = torch.autograd.grad((qr, kr, v), x, (w["dq"], w["dk"], w["dv"]))[0]
    return w["o"].reshape(B * S, Hq * d), g.reshape(B * S, -1)


def _glue_check(name, out, dqkv, want_o, want_g, Hq, Hk, d):
    errs = {"o": float((out.double() - want_o).abs().max())}
    cols = {"dq": slice(0, Hq * d), "dk": slice(Hq * d, (Hq + Hk) * d), "dv": slice((Hq + Hk) * d, None)}
    for n, c in cols.items():
        errs[n] = float((dqkv[:, c].double() - want_g[:, c]).abs().max() / want_g[:, c].abs().max())
    _report(name, errs)
    for n, e in errs.items():
        assert e < TOL[n], (name, n, e)


def _positions(lengths, S):
    pos = torch.zeros(len(lengths), S, dtype=torch.long)
    for b, row in enumerate(lengths):
        pos[b] = torch.cat([torch.arange(n) for n in row])
    return pos.to(DEV)


def _run_glue(fn, qkv, d_o, *args, **kw):
    leaf = qkv.clone().requires_grad_()
    out = fn(leaf.clone(), *args, **kw)        # the attention block rotates its input in place: hand it a copy
    out.backward(d_o)
    torch.cuda.synchronize()
    return out.detach(), leaf.grad


@pytest.mark.parametrize("packed", [True, False])
def test_rope_causal_attention_glue(packed, monkeypatch):
    """Packed rows: per-token RoPE tables (one row of B*S tokens) and the segmented kernels.  Unpacked under ACCO_ATTN=own: [S, D/2]
    tables and the unsegmented kernels."""
    B, S, Hq, Hk = 2, 512, 4, 2
    if not packed:
        monkeypatch.setenv("ACCO_ATTN", "own")
    lengths = row_lengths("edges", B, S) if packed else [[S]] * B
    pos = _positions(lengths, S)
    cos, sin = ops.rope_tables(S, D, 500000.0, DEV)
    qkv, d_o = (t.to(DEV) for t in make_qkv(B, S, Hq, Hk, seed=41))
    ops.reset_launch_counts()
    if packed:
        seg = seg_starts_of(lengths, S).to(DEV)
        idx = pos.reshape(-1)
        out, g = _run_glue(ops.rope_causal_attention, qkv, d_o, cos[idx].contiguous(), sin[idx].contiguous(), B, S, Hq, Hk, D, seg=seg)
    else:
        out, g = _run_glue(ops.rope_causal_attention, qkv, d_o, cos, sin, B, S, Hq, Hk, D)
    counts = ops.launch_counts()
    suffix = "_seg" if packed else ""
    assert counts.get("attn_fwd" + suffix) == 1 and counts.get("attn_bwd" + suffix) == 2, counts
    assert counts.get("rope_qkv") == 1 and counts.get("rope_pack_bwd") == 1, counts
    want_o, want_g = _glue_oracle(qkv, d_o, B, S, Hq, Hk, D, 1 / math.sqrt(D), 0, lengths, pos, rope=True)
    _glue_check(f"rope_causal_attention packed={packed}", out, g, want_o, want_g, Hq, Hk, D)


def test_packed_causal_attention_gptneo_glue():
    B, S, H = 2, 1024, 4
    lengths = row_lengths("random", B, S, seed=2)
    seg = seg_starts_of(lengths, S).to(DEV)
    qkv, d_o = (t.to(DEV) for t in make_qkv(B, S, H, H, seed=43))
    ops.reset_launch_counts()
    out, g = _run_glue(ops.packed_causal_attention, qkv, d_o, B, S, H, H, D, scale=1.0, window=256, seg=seg)
    counts = ops.launch_counts()
    assert counts.get("attn_fwd_seg") == 1 and counts.get("attn_bwd_seg") == 2 and counts.get("rope_pack_bwd") == 1, counts
    want_o, want_g = _glue_oracle(qkv, d_o, B, S, H, H, D, 1.0, 256, lengths, None, rope=False)
    _glue_check("packed_causal_attention gpt-neo", out, g, want_o, want_g, H, H, D)


# ---------------------------------------------------------------------------------------------- e. the SDPA fallback
def test_sdpa_fallback_packed_head_dim_128():
    """Llama-3-8B heads (32 / 8, head_dim 128) on packed rows: the kernels do not cover head_dim 128, so the block takes SDPA with a
    dense document mask (and the kernels' RoPE / d(qkv) packing around it)."""
    B, S, Hq, Hk, d = 2, 512, 32, 8, 128
    lengths = row_lengths("edges", B, S)
    pos = _positions(lengths, S)
    cos, sin = ops.rope_tables(S, d, 500000.0, DEV)
    idx = pos.reshape(-1)
    seg = seg_starts_of(lengths, S).to(DEV)
    qkv, d_o = (t.to(DEV) for t in make_qkv(B, S, Hq, Hk, seed=45, d=d))
    ops.reset_launch_counts()
    out, g = _run_glue(ops.rope_causal_attention, qkv, d_o, cos[idx].contiguous(), sin[idx].contiguous(), B, S, Hq, Hk, d, seg=seg)
    counts = ops.launch_counts()
    assert "attn_fwd_seg" not in counts and counts.get("rope_qkv") == 1 and counts.get("rope_pack_bwd") == 1, counts
    want_o, want_g = _glue_oracle(qkv, d_o, B, S, Hq, Hk, d, 1 / math.sqrt(d), 0, lengths, pos, rope=True)
    _glue_check("sdpa fallback head_dim 128", out, g, want_o, want_g, Hq, Hk, d)
