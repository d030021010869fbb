#!/usr/bin/env python
"""Where the time of the weight-gradient (wgrad) GEMMs goes: each wgrad shape of the Llama-125M (T = 8192) and Llama-3.2-1B
(T = 4096) steps, timed in variants that isolate one cause each.  The wgrad is ``grad [M, N] += dy [T, M]^T @ x [T, N]``: both
operands MN-major (``gemm_tt_acc``), an adding epilogue into a strided view of the gradient arena.

    shipped       the call the trainer makes (heuristic pick, a = 1, b = 1, accumulate)
    a1b0 / a0b1 / a0b0   the same product with one or both operands K-major (transposed copies made before timing)
    store         accumulate = 0 at the shipped layout, pick and splits (the epilogue stores instead of reading C)
    f32           the fp32-D instantiation (``grad_accum_dtype=fp32``) at the heuristic's pick
    pad           dy and x as views with a leading dimension of rows + 64 (breaks power-of-two row strides)
    bn128 / bn256 forced tile width (the heuristic picks the K splits)
    k768          the same M at K = 768 with N scaled so the FLOPs match, at the shipped tile width and one split
    fwd           controls: the step's forward shapes at a forced 128-wide cooperative tile, and as shipped

Per variant: median device time (CUDA events around --iters back-to-back launches after warm-up, --reps samples), TFLOP/s,
units (tiles x K splits), busy SMs, and the time per k-block of one CTA (``ns_per_kb``: time x busy SMs / (units x k-blocks per
unit)) and per 128 output columns of its tile (``ns_per_kb_128``), which compares tile widths.  The shipped call is also launched
once with ``acco_gemm_set_debug``: CTA 0 of the cooperative kernel stamps %globaltimer at its phases (stamp() in
csrc/gemm_wgmma.cu), giving its mainloop (first full stage -> last load issued) and tail (last load -> last store) times.

    python tools/wgrad_probe.py --out results/wgrad_probe [--tree DIR] [--only 125m|1b]

--tree times the package of another checkout (an older build of the same project) with this script."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BK = 64


def shapes():
    """(preset, name, M, N, T): wgrad out [M, N] += dy [T, M]^T x [T, N]"""
    out = []
    T, H, I, V = 8192, 768, 2048, 50304                       # Llama-125M, 8 x 1024 tokens
    out += [("125m", "qkv", 3 * H, H, T), ("125m", "o", H, H, T), ("125m", "gateup", 2 * I, H, T), ("125m", "down", H, I, T),
            ("125m", "lmhead", V, H, T)]
    T, H, I, KV, V = 4096, 2048, 8192, 512, 128256            # Llama-3.2-1B, 4 x 1024 tokens
    out += [("1b", "qkv", H + 2 * KV, H, T), ("1b", "o", H, H, T), ("1b", "gateup", 2 * I, H, T), ("1b", "down", H, I, T),
            ("1b", "lmhead", V, H, T)]
    return out


def gpu_info():
    try:
        p = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           stderr=subprocess.DEVNULL, text=True, timeout=30)
        return p.stdout.strip().splitlines()[0] if p.stdout.strip() else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory (wgrad_probe[_TAG].json)")
    ap.add_argument("--tree", default=ROOT, help="checkout whose acco_b200 package is timed")
    ap.add_argument("--tag", default="", help="suffix of the output file name")
    ap.add_argument("--only", default="", help="125m or 1b: one preset")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-variants", action="store_true", help="time the shipped calls only")
    a = ap.parse_args()
    tree = os.path.abspath(a.tree)
    sys.path.insert(0, tree)
    import torch
    from acco_b200 import ops
    from acco_b200.ops.gemm import gemm, gemm_tt_acc, gemm_wgrad_f32
    ext = ops.load_ext(required=True)
    lib = ctypes.CDLL(ext.__file__)
    lib.acco_gemm_choose.argtypes = [ctypes.c_int] * 7 + [ctypes.POINTER(ctypes.c_int)]
    lib.acco_gemm_set_debug.argtypes = [ctypes.c_void_p]
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: (torch.randn(*s, device=dev, generator=g) * 0.1).to(torch.bfloat16)

    def pick(M, N, K, a_mn=1, b_mn=1, acc=1):
        p = (ctypes.c_int * 5)()
        lib.acco_gemm_choose(M, N, K, a_mn, b_mn, acc, sms, p)
        return p[0], p[1]

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

    def phases(fn):
        buf = torch.zeros(16, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        lib.acco_gemm_set_debug(ctypes.c_void_p(buf.data_ptr()))
        try:
            fn()
            torch.cuda.synchronize()
        finally:
            lib.acco_gemm_set_debug(None)
        s = buf.tolist()
        if not s[4]:
            return None
        us = lambda i, j: (s[j] - s[i]) / 1e3 if s[i] and s[j] else None
        return {"start_to_first_full_us": us(0, 4), "mainloop_us": us(4, 9), "tail_us": us(9, 7), "total_us": us(0, 10)}

    def record(rows, preset, name, variant, M, N, K, bn, splits, fn, extra=None):
        ms, spread = time_ms(fn)
        flops = 2.0 * M * N * K
        num_k = (K + BK - 1) // BK
        splits = max(1, min(splits, num_k))
        kbs = (num_k + splits - 1) // splits
        splits = (num_k + kbs - 1) // kbs
        units = ((M + 127) // 128) * ((N + bn - 1) // bn) * splits
        busy = min(units, sms)
        r = {"preset": preset, "shape": name, "variant": variant, "M": M, "N": N, "K": K, "bn": bn, "splits": splits, "units": units,
             "busy_sms": busy, "ms": ms, "spread_ms": spread, "tflops": flops / ms / 1e9, "tflops_per_busy_sm_x_sms": flops / ms / 1e9 * sms / busy,
             "ns_per_kb": ms * 1e6 * busy / (units * kbs), "ns_per_kb_128": ms * 1e6 * busy / (units * kbs) * 128 / bn}
        if extra:
            r.update(extra)
        rows.append(r)
        print(json.dumps(r), flush=True)

    rows = []
    for preset, name, M, N, T in shapes():
        if a.only and preset != a.only:
            continue
        dy, x = rnd(T, M), rnd(T, N)
        big = torch.zeros(M + 2, N + 16, device=dev, dtype=torch.bfloat16)
        grad = big[1:M + 1, 8:N + 8]                          # a strided view, like a weight's slot in the gradient arena
        bn, sp = pick(M, N, T)
        shipped = lambda: gemm_tt_acc(dy, x, grad)
        record(rows, preset, name, "shipped", M, N, T, bn, sp, shipped, {"phases": phases(shipped)})
        if a.no_variants:
            continue
        g32 = torch.zeros(M, N, device=dev, dtype=torch.float32)
        record(rows, preset, name, "f32", M, N, T, bn, sp, lambda: gemm_wgrad_f32(dy, x, g32))
        del g32
        if name == "lmhead":
            torch.cuda.empty_cache()
            continue
        dyt, xt = dy.t().contiguous(), x.t().contiguous()     # K-major copies: [M, T], [N, T]
        record(rows, preset, name, "a1b0", M, N, T, bn, sp, lambda: gemm(dy, xt, out=grad, a_mn=True, b_mn=False, accumulate=True))
        record(rows, preset, name, "a0b1", M, N, T, bn, sp, lambda: gemm(dyt, x, out=grad, a_mn=False, b_mn=True, accumulate=True))
        record(rows, preset, name, "a0b0", M, N, T, bn, sp, lambda: gemm(dyt, xt, out=grad, a_mn=False, b_mn=False, accumulate=True))
        del dyt, xt
        if sp == 1:
            record(rows, preset, name, "store", M, N, T, bn, sp, lambda: gemm(dy, x, out=grad, a_mn=True, b_mn=True, bn=bn, splits=1))
        dyp = torch.empty(T, M + 64, device=dev, dtype=torch.bfloat16)[:, :M]
        xp = torch.empty(T, N + 64, device=dev, dtype=torch.bfloat16)[:, :N]
        dyp.copy_(dy)
        xp.copy_(x)
        record(rows, preset, name, "pad", M, N, T, bn, sp, lambda: gemm(dyp, xp, out=grad, a_mn=True, b_mn=True, accumulate=True),
               {"lda": M + 64, "ldb": N + 64})
        del dyp, xp
        for fbn in (128, 256):
            # the splits the heuristic would add at a forced width are not reported: the shipped pick's, else one split
            fsp = sp if fbn == bn else 1
            record(rows, preset, name, f"bn{fbn}", M, N, T, fbn, fsp,
                   lambda: gemm(dy, x, out=grad, a_mn=True, b_mn=True, accumulate=True, bn=fbn, splits=fsp))
        n2 = max(128, (N * T // 768) // 128 * 128)
        dy2, x2 = rnd(768, M), rnd(768, n2)
        g2 = torch.zeros(M, n2, device=dev, dtype=torch.bfloat16)
        record(rows, preset, name, "k768", M, n2, 768, bn, 1, lambda: gemm(dy2, x2, out=g2, a_mn=True, b_mn=True, accumulate=True, bn=bn, splits=1))
        del dy2, x2, g2, dy, x, big, grad
        torch.cuda.empty_cache()
    # controls: the 125M forward shapes (x [T, K] @ w [N, K]^T) on the cooperative kernel at 128-wide tiles, and as shipped
    if not a.no_variants and a.only != "1b":
        T, H, I = 8192, 768, 2048
        for name, N, K in (("qkv_fwd", 3 * H, H), ("o_fwd", H, H), ("gateup_fwd", 2 * I, H), ("down_fwd", H, I)):
            xx, w = rnd(T, K), rnd(N, K)
            record(rows, "125m", name, "fwd_coop_bn128", T, N, K, 128, 1, lambda: gemm(xx, w, bn=128, splits=1))
            fbn, fsp = pick(T, N, K, 0, 0, 0)
            record(rows, "125m", name, "fwd_shipped", T, N, K, 128 if fbn == 128 else fbn, fsp, lambda: gemm(xx, w))
    out = {"gpu": gpu_info(), "device": props.name, "sms": sms, "tree": tree, "iters": a.iters, "reps": a.reps, "rows": rows}
    print(json.dumps({"gpu": out["gpu"], "tree": tree}), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, f"wgrad_probe{('_' + a.tag) if a.tag else ''}.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
