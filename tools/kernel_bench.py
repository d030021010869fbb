#!/usr/bin/env python
"""Isolated timing of every hand-written kernel at the Llama-125M shapes (T = 8x1024 tokens), with achieved
HBM bandwidth / tensor throughput against MEASURED_PEAKS.json.  L2 is flushed between timed launches.

    python tools/kernel_bench.py [--only rmsnorm,ce,...] [--iters 20] [--out kernel_bench.json]
Also the target of `ncu --set full -k regex:<kernel>` captures (use --iters 1 --no-flush)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from acco_b200 import ops
from acco_b200.optim import AdamHyper, ShardedAdamW
from acco_b200.ops.gemm import gemm_tn

DEV = "cuda"


def timed(fn, iters, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    buf = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=DEV) if flush else None
    ts = []
    for _ in range(iters):
        if buf is not None:
            buf.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--no-flush", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    only = set(x for x in a.only.split(",") if x)
    peaks = {"hbm_gbs": 6462.4, "bf16_tflops": 1686.0}
    try:
        peaks.update(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))))
    except Exception:
        pass
    C = ops.load_ext(required=True)
    T, H, I, V, Vp, Hq, D, B, S = 8192, 768, 2048, 50257, 50304, 12, 64, 8, 1024
    bf = lambda *s: (torch.randn(*s, device=DEV) * 0.5).to(torch.bfloat16)
    res = {}

    def rec(name, fn, bytes_=None, flops=None):
        if only and not any(name.startswith(o) for o in only):
            return
        ms = timed(fn, a.iters, not a.no_flush)
        r = {"ms": ms}
        if bytes_:
            r["GBps"] = bytes_ / ms / 1e6
            r["frac_of_measured_hbm"] = r["GBps"] / peaks["hbm_gbs"]
        if flops:
            r["TFLOPs"] = flops / ms / 1e9
            r["frac_of_measured_bf16"] = r["TFLOPs"] / peaks["bf16_tflops"]
        res[name] = r
        print(name, json.dumps(r), flush=True)

    x, r_, w = bf(T, H), bf(T, H), torch.ones(H, device=DEV, dtype=torch.bfloat16)
    y, rstd = C.rmsnorm_fwd(x, w, 1e-5)
    rec("rmsnorm_fwd", lambda: C.rmsnorm_fwd(x, w, 1e-5), bytes_=2 * T * H * 2)
    rec("add_rmsnorm_fwd", lambda: C.add_rmsnorm_fwd(x, r_, w, 1e-5), bytes_=4 * T * H * 2)
    dy = bf(T, H)
    wg = torch.zeros(H, device=DEV, dtype=torch.bfloat16)
    rec("rmsnorm_bwd", lambda: C.rmsnorm_bwd(dy, x, w, rstd, wg), bytes_=3 * T * H * 2)
    rec("add_rmsnorm_bwd", lambda: C.add_rmsnorm_bwd(dy, r_, x, w, rstd, wg), bytes_=4 * T * H * 2)
    qkv = bf(T, 3 * Hq * D)
    cos, sin = ops.rope_tables(S, D, 10000.0, DEV)
    rec("rope_qkv", lambda: C.rope_qkv_inplace(qkv, cos, sin, B, S, 2 * Hq, 3 * Hq, D, False), bytes_=2 * T * 2 * Hq * D * 2)
    dq, dk, dv = (bf(B, Hq, S, D).transpose(1, 2) for _ in range(3))
    rec("rope_pack_bwd", lambda: C.rope_pack_bwd(dq, dk, dv, cos, sin), bytes_=2 * T * 3 * Hq * D * 2)
    gu, dout = bf(T, 2 * I), bf(T, I)
    rec("swiglu_fwd", lambda: C.swiglu_fwd(gu), bytes_=3 * T * I * 2)
    rec("swiglu_bwd", lambda: C.swiglu_bwd(dout, gu), bytes_=5 * T * I * 2)
    logits = bf(T, Vp)
    labels = torch.randint(0, V, (T,), device=DEV)
    loss, inv_n, lse = C.ce_fwd(logits, labels, V, -100)
    rec("ce_fwd", lambda: C.ce_fwd(logits, labels, V, -100), bytes_=T * Vp * 2)
    scale = torch.ones(1, device=DEV)
    rec("ce_bwd", lambda: C.ce_bwd_inplace(logits, labels, lse, scale, V, -100), bytes_=2 * T * Vp * 2)
    N = 123_587_328 // 1024 * 1024
    opt = ShardedAdamW(torch.zeros(N, device=DEV), 1e-3)
    g = torch.zeros(N, device=DEV, dtype=torch.bfloat16)
    out = torch.zeros(N, device=DEV, dtype=torch.bfloat16)
    hp = AdamHyper(lr=1e-3, step=2, inv_count=torch.ones(1, device=DEV), commit=3)
    rec("adamw_shard_commit", lambda: ops.fused_adamw_shard(g, opt.master, opt.exp_avg, opt.exp_avg_sq, opt.stash, out, hp), bytes_=N * (2 + 12 + 12 + 2))
    hp2 = AdamHyper(lr=1e-3, step=2, inv_count=torch.ones(1, device=DEV), commit=0, write_stash=True)
    rec("adamw_shard_tentative", lambda: ops.fused_adamw_shard(g, opt.master, opt.exp_avg, opt.exp_avg_sq, opt.stash, out, hp2), bytes_=N * (2 + 12 + 4 + 2))
    for (M, Nn, K) in ((T, 3 * H, H), (T, 2 * I, H), (T, H, I), (T, Vp, H), (8192, 8192, 8192)):
        xa, wb = bf(M, K), bf(Nn, K)
        rec(f"gemm_{M}x{Nn}x{K}", lambda: gemm_tn(xa, wb), flops=2.0 * M * Nn * K)
        rec(f"gemm_cublas_{M}x{Nn}x{K}", lambda: torch.nn.functional.linear(xa, wb), flops=2.0 * M * Nn * K)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump({"peaks": peaks, "shapes": {"T": T, "H": H, "I": I, "Vp": Vp}, "kernels": res}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
