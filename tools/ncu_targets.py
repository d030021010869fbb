#!/usr/bin/env python
"""Tiny drivers for `ncu --set full -k regex:<kernel>` captures (one launch of each hot kernel at model shapes)."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from acco_b200 import ops
from acco_b200.optim import AdamHyper, ShardedAdamW
from acco_b200.ops.gemm import gemm_tn
C = ops.load_ext(required=True)
which = sys.argv[1]
bf = lambda *s: (torch.randn(*s, device="cuda") * 0.5).to(torch.bfloat16)
T, H, V, Vp = 8192, 768, 50257, 50304
if which == "adam":
    N = 123_587_328 // 1024 * 1024
    opt = ShardedAdamW(torch.zeros(N, device="cuda"), 1e-3)
    g = torch.zeros(N, device="cuda", dtype=torch.bfloat16); out = torch.zeros_like(g)
    hp = AdamHyper(lr=1e-3, step=2, inv_count=torch.ones(1, device="cuda"), commit=3)
    for _ in range(3):
        ops.fused_adamw_shard(g, opt.master, opt.exp_avg, opt.exp_avg_sq, opt.stash, out, hp)
elif which == "gemm":
    x, w = bf(T, H), bf(4096, H)
    for _ in range(3):
        gemm_tn(x, w)
    x, w = bf(8192, 8192), bf(8192, 8192)
    for _ in range(2):
        gemm_tn(x, w)
elif which == "ce":
    lg = bf(T, Vp); lb = torch.randint(0, V, (T,), device="cuda")
    for _ in range(3):
        loss, inv_n, lse = C.ce_fwd(lg, lb, V, -100)
        C.ce_bwd_inplace(lg, lb, lse, torch.ones(1, device="cuda"), V, -100)
elif which == "norm":
    x, r, w = bf(T, H), bf(T, H), torch.ones(H, device="cuda", dtype=torch.bfloat16)
    for _ in range(3):
        y, h, _, rstd = C.norm_fwd(x, r, w, None, 1e-5)
        C.norm_bwd(x, r, h, w, None, rstd, None, None)
torch.cuda.synchronize()
