#!/usr/bin/env python
"""Check of the own flash-attention kernels (csrc/attention_wgmma.cu; single GPU):

    timeout 300 python tools/attn_check.py [--quick] [--no-bwd] [--out attn_check.json]

Per shape: forward (O, LSE) and backward (dQ, dK, dV) of the own kernels against the fp32 PyTorch reference (the same oracle the
CPU spec test uses), then device time per call against the library path (cuDNN / flash SDPA forward + backward on the same
tensors).  Exit code 0 = every shape within tolerance."""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from acco_b200 import ops
from acco_b200.ops.attention import causal_attention_ref

DEV = "cuda"

# (B, S, Hq, Hk, window, scale)   head_dim 64
SHAPES = [
    (1, 128, 1, 1, 0, None),          # one tile, one key block: diagonal masking only
    (1, 256, 2, 1, 0, None),          # two key blocks (delayed P V accumulation), GQA group of 2
    (2, 512, 4, 2, 0, None),
    (1, 512, 2, 2, 256, 1.0),         # GPT-Neo local layer: window 256, scale 1
    (1, 1024, 2, 2, 300, None),       # window not a multiple of the tile
    (8, 1024, 12, 12, 0, None),       # Llama-125M micro-batch
    (2, 1024, 32, 8, 0, None),        # Llama-3.2-1B heads
]


def timed(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="first four shapes only")
    ap.add_argument("--no-bwd", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    C = ops.load_ext(required=True)
    report, ok = [], True
    for (B, S, Hq, Hk, window, scale) in (SHAPES[:4] if a.quick else SHAPES):
        D = 64
        sc = (1.0 / math.sqrt(D)) if scale is None else scale
        torch.manual_seed(S + Hq)
        qkv = (torch.randn(B * S, (Hq + 2 * Hk) * D, device=DEV) * 0.7).to(torch.bfloat16)
        d_o = (torch.randn(B * S, Hq * D, device=DEV) * 0.5).to(torch.bfloat16)
        x = qkv.view(B, S, Hq + 2 * Hk, D)
        q, k, v = (t.float().requires_grad_() for t in (x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:]))
        ref = causal_attention_ref(q, k, v, scale=sc, window=window or None)
        gq, gk, gv = torch.autograd.grad(ref, (q, k, v), d_o.view(B, S, Hq, D).float())
        entry = {"shape": [B, S, Hq, Hk, window, sc]}
        assert C.attn_supported(B, S, Hq, Hk, D, sc)
        o, lse = C.attn_fwd(qkv, B, S, Hq, Hk, D, sc, window)
        torch.cuda.synchronize()
        err_o = float((o.view(B, S, Hq, D).float() - ref.detach()).abs().max())
        entry["fwd_max_abs_err"] = err_o
        good = err_o < 2e-2 and bool(torch.isfinite(lse).all())
        if not a.no_bwd:
            dq, dk, dv = C.attn_bwd(qkv, o, d_o, lse, B, S, Hq, Hk, D, sc, window)
            torch.cuda.synchronize()
            for name, got, want in (("dq", dq.view(B, S, Hq, D), gq), ("dk", dk.view(B, S, Hk, D).float(), gk), ("dv", dv.view(B, S, Hk, D).float(), gv)):
                rel = float((got - want).abs().max() / want.abs().max())
                entry[f"{name}_rel_err"] = rel
                good = good and rel < 3e-2
        # speed vs the library path on the same tensors
        qt, kt, vt = (t.transpose(1, 2).detach().requires_grad_() for t in (x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:]))
        do_t = d_o.view(B, S, Hq, D).transpose(1, 2)
        kw = {"enable_gqa": True} if Hk != Hq else {}
        mask = None
        if window:
            i = torch.arange(S, device=DEV)
            mask = (i[None, :] <= i[:, None]) & (i[None, :] > i[:, None] - window)

        def lib_fwd():
            if mask is None:
                return torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, is_causal=True, scale=sc, **kw)
            return torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, attn_mask=mask, scale=sc, **kw)

        def lib_fwd_bwd():
            out = lib_fwd()
            torch.autograd.grad(out, (qt, kt, vt), do_t)

        entry["own_fwd_ms"] = timed(lambda: C.attn_fwd(qkv, B, S, Hq, Hk, D, sc, window))
        entry["lib_fwd_ms"] = timed(lib_fwd)
        if not a.no_bwd:
            entry["own_bwd_ms"] = timed(lambda: C.attn_bwd(qkv, o, d_o, lse, B, S, Hq, Hk, D, sc, window))
            entry["lib_fwd_bwd_ms"] = timed(lib_fwd_bwd)
        # useful work: 2 MMAs of 2*S*S*D flops per head forward (causal: half of it, windows less), 5 backward
        vis = S * (S + 1) / 2 if not window else sum(min(i + 1, window) for i in range(S))
        fwd_flops = 4.0 * vis * D * Hq * B
        entry["own_fwd_tflops"] = fwd_flops / (entry["own_fwd_ms"] * 1e-3) / 1e12 if entry["own_fwd_ms"] > 0 else None
        if not a.no_bwd:
            entry["own_bwd_tflops"] = 2.5 * fwd_flops / (entry["own_bwd_ms"] * 1e-3) / 1e12 if entry["own_bwd_ms"] > 0 else None
        entry["ok"] = good
        ok = ok and good
        report.append(entry)
        print(json.dumps(entry), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump({"ok": ok, "shapes": report}, open(a.out, "w"), indent=1)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
