#!/usr/bin/env python
"""Time each of the 15 GEMM calls of one Llama-125M training step (8 x 1024 tokens) in the layouts the trainer uses:

    forward  gemm_tn(x [M, K], w [N, K])                 -> y [M, N]
    dgrad    gemm_nn(dy [M, K], w [K, N])                -> dx [M, N]
    wgrad    gemm_tt_acc(dy [K, M], x [K, N], grad)      grad [M, N] += ..., grad a strided view into a larger bf16 buffer

Per shape: the heuristic's pick (bn, splits), device ms (CUDA events around --iters back-to-back launches after warm-up, median of
--reps), TFLOP/s, the lower bound max(FLOP / 989 TFLOP/s, bytes / 3.35 TB/s) of an H100 SXM (data sheet, dense bf16), and the
library call that ACCO_GEMM=cublas would make, for context.

    python tools/gemm_step_bench.py --out results/gemm_step [--tree DIR]

--tree times the package of another checkout (an older build of the same project) with this script."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12
T, H, I, V = 8192, 768, 2048, 50304

# (name, kind, M, N, K, calls per step): out [M, N], contraction K
SHAPES = [
    ("qkv_fwd", "tn", T, 3 * H, H, 12), ("o_fwd", "tn", T, H, H, 12), ("gateup_fwd", "tn", T, 2 * I, H, 12), ("down_fwd", "tn", T, H, I, 12),
    ("qkv_dgrad", "nn", T, H, 3 * H, 12), ("o_dgrad", "nn", T, H, H, 12), ("gateup_dgrad", "nn", T, H, 2 * I, 12),
    ("down_dgrad", "nn", T, I, H, 12),
    ("qkv_wgrad", "tt_acc", 3 * H, H, T, 12), ("o_wgrad", "tt_acc", H, H, T, 12), ("gateup_wgrad", "tt_acc", 2 * I, H, T, 12),
    ("down_wgrad", "tt_acc", H, I, T, 12),
    ("lmhead_fwd", "tn", T, V, H, 1), ("lmhead_dgrad", "nn", T, H, V, 1), ("lmhead_wgrad", "tt_acc", V, H, T, 1),
]


def gpu_info():
    try:
        p = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           stderr=subprocess.DEVNULL, text=True, timeout=30)
        return p.stdout.strip().splitlines()[0] if p.stdout.strip() else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory (gemm_step_bench.json)")
    ap.add_argument("--tree", default=ROOT, help="checkout whose acco_b200 package is timed")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-cublas", action="store_true")
    a = ap.parse_args()
    tree = os.path.abspath(a.tree)
    sys.path.insert(0, tree)
    import torch
    from acco_b200 import ops
    from acco_b200.ops.gemm import gemm_nn, gemm_tn, gemm_tt_acc
    ext = ops.load_ext(required=True)
    lib = ctypes.CDLL(ext.__file__)
    lib.acco_gemm_choose.argtypes = [ctypes.c_int] * 7 + [ctypes.POINTER(ctypes.c_int)]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: (torch.randn(*s, device=dev, generator=g) * 0.1).to(torch.bfloat16)

    def time_ms(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / a.iters)
        ts.sort()
        return ts[len(ts) // 2], ts[-1] - ts[0]

    rows = []
    for name, kind, M, N, K, calls in SHAPES:
        pick = (ctypes.c_int * 5)()
        a_mn, b_mn, acc = {"tn": (0, 0, 0), "nn": (0, 1, 0), "tt_acc": (1, 1, 1)}[kind]
        lib.acco_gemm_choose(M, N, K, a_mn, b_mn, acc, sms, pick)
        if kind == "tn":
            x, w = rnd(M, K), rnd(N, K)
            ours, lib_call, lib_name = (lambda: gemm_tn(x, w)), (lambda: torch.nn.functional.linear(x, w)), "F.linear(x, w)"
            nbytes = 2 * (M * K + N * K + M * N)
        elif kind == "nn":
            dy, w = rnd(M, K), rnd(K, N)
            ours, lib_call, lib_name = (lambda: gemm_nn(dy, w)), (lambda: dy.matmul(w)), "dy.matmul(w)"
            nbytes = 2 * (M * K + N * K + M * N)
        else:
            dy, x = rnd(K, M), rnd(K, N)
            big = torch.zeros(M + 2, N + 16, device=dev, dtype=torch.bfloat16)
            grad = big[1:M + 1, 8:N + 8]                      # a strided view, like a weight's slot in the gradient arena
            ours, lib_call, lib_name = (lambda: gemm_tt_acc(dy, x, grad)), (lambda: grad.addmm_(dy.t(), x)), "grad.addmm_(dy.t(), x)"
            nbytes = 2 * (M * K + N * K + 2 * M * N)
        flops = 2.0 * M * N * K
        ms, spread = time_ms(ours)
        bound = max(flops / PEAK_FLOPS, nbytes / PEAK_BYTES) * 1e3
        r = {"name": name, "kind": kind, "M": M, "N": N, "K": K, "calls_per_step": calls, "bn": pick[0], "splits": pick[1], "ms": ms,
             "spread_ms": spread, "tflops": flops / ms / 1e9, "bound_ms": bound, "frac_of_bound": bound / ms, "library_call": lib_name}
        if not a.no_cublas:
            r["library_ms"] = time_ms(lib_call)[0]
        rows.append(r)
        print(json.dumps(r), flush=True)
        del ours, lib_call
        torch.cuda.empty_cache()
    total = sum(r["ms"] * r["calls_per_step"] for r in rows)
    out = {"gpu": gpu_info(), "tree": tree, "sms": sms, "iters": a.iters, "reps": a.reps, "shapes": rows, "gemm_ms_per_step": total}
    print(json.dumps({"gpu": out["gpu"], "gemm_ms_per_step": total}), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "gemm_step_bench.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
