#!/usr/bin/env python
"""FP8 against bf16 on one GPU (train key ``fp8``, ``ops/fp8.py``).  Prints the card name and power limit of the run, then:

  (a) gemms : device-timed (CUDA events) forward / dgrad / wgrad of the block linears of llama125m, llama3-1b and llama3-8b at
              T = 4096 and 8192, bf16 wgmma GEMM against FP8 GEMM, with achieved TFLOP/s; the quantisation kernels (amax + cast of x,
              W and g) are timed on their own and added into the FP8 total.
  (b) steps : trainer tokens/s, bf16 against FP8, llama125m at 8 x 1024 and llama3-1b at 4 x 1024 (CUDA graphs, device-resident
              batches, ACCO on one GPU), three alternated runs of each.
  (c) loss  : ~300 steps of Llama-125M on synthetic_pretrain_dataset (learnable Markov tokens), same seed, bf16 against FP8.

    python tools/fp8_bench.py [--parts gemms,steps,loss] [--out fp8_bench.json]
"""
import argparse
import json
import logging
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

BLOCKS = {   # (H, qkv rows, I) of the Llama presets
    "llama125m": (768, 2304, 2048),
    "llama3-1b": (2048, 3072, 8192),
    "llama3-8b": (4096, 6144, 14336),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, iters=20, warmup=3):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_gemms():
    from acco_b200.ops.fp8 import E4M3, E5M2, gemm_fp8, quantize
    from acco_b200.ops.gemm import gemm
    dev = torch.device("cuda")
    rows = []
    for name, (H, QKV, I) in BLOCKS.items():
        for T in (4096, 8192):
            for lin, N, K in (("qkv", QKV, H), ("o", H, H), ("gate_up", 2 * I, H), ("down", H, I)):
                x = torch.randn(T, K, device=dev).to(torch.bfloat16)
                w = (torch.randn(N, K, device=dev) * 0.02).to(torch.bfloat16)
                g = (torch.randn(T, N, device=dev) * 1e-3).to(torch.bfloat16)
                wg = torch.zeros(N, K, device=dev, dtype=torch.bfloat16)
                qx, qxT, sx = quantize(x, E4M3, True, True)
                qw, qwT, sw = quantize(w, E4M3, True, True)
                qg, qgT, sg = quantize(g, E5M2, True, True)
                fl = 2.0 * T * N * K
                r = {"preset": name, "T": T, "linear": lin, "N": N, "K": K}
                r["bf16_fwd_ms"] = timed(lambda: gemm(x, w))
                r["bf16_dgrad_ms"] = timed(lambda: gemm(g, w, b_mn=True))
                r["bf16_wgrad_ms"] = timed(lambda: gemm(g, x, out=wg, a_mn=True, b_mn=True, accumulate=True))
                r["fp8_fwd_ms"] = timed(lambda: gemm_fp8(qx, qw, sx, sw))
                r["fp8_dgrad_ms"] = timed(lambda: gemm_fp8(qg, qwT, sg, sw))
                r["fp8_wgrad_ms"] = timed(lambda: gemm_fp8(qgT, qxT, sg, sx, out=wg, accumulate=True))
                r["quant_ms"] = (timed(lambda: quantize(x, E4M3, True, True)) + timed(lambda: quantize(w, E4M3, True, True))
                                 + timed(lambda: quantize(g, E5M2, True, True)))
                r["bf16_total_ms"] = r["bf16_fwd_ms"] + r["bf16_dgrad_ms"] + r["bf16_wgrad_ms"]
                r["fp8_total_ms"] = r["fp8_fwd_ms"] + r["fp8_dgrad_ms"] + r["fp8_wgrad_ms"] + r["quant_ms"]
                for k in ("fwd", "dgrad", "wgrad"):
                    r[f"bf16_{k}_tflops"] = fl / r[f"bf16_{k}_ms"] / 1e9
                    r[f"fp8_{k}_tflops"] = fl / r[f"fp8_{k}_ms"] / 1e9
                rows.append(r)
                print(f"{name:10s} T={T:5d} {lin:8s} N={N:6d} K={K:6d} | bf16 fwd/dgrad/wgrad {r['bf16_fwd_tflops']:6.0f} "
                      f"{r['bf16_dgrad_tflops']:6.0f} {r['bf16_wgrad_tflops']:6.0f} TF/s | fp8 {r['fp8_fwd_tflops']:6.0f} "
                      f"{r['fp8_dgrad_tflops']:6.0f} {r['fp8_wgrad_tflops']:6.0f} TF/s | quant {r['quant_ms']:.3f} ms | total "
                      f"{r['bf16_total_ms']:.3f} -> {r['fp8_total_ms']:.3f} ms", flush=True)
                del x, w, g, wg, qx, qxT, qw, qwT, qg, qgT
    return rows


def _trainer(model_name, batch, seq, fp8, ds=None, steps=10 ** 12, method="acco", seed=1234, log_every=10 ** 9):
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import TokenDataset
    from acco_b200.models import preset
    dev = torch.device("cuda")
    torch.manual_seed(seed)
    model = preset(model_name, device=dev, dtype=torch.bfloat16)
    if ds is None:
        g = torch.Generator().manual_seed(7)
        ds = TokenDataset({"input_ids": torch.randint(0, model.config.vocab_size, (64 * batch, seq), generator=g, dtype=torch.long)})
    args = AttrDict(method_name=method, batch_size=batch, n_grad_accumulation=1, max_length=seq, learning_rate=6e-4, weight_decay=0.1,
                    scheduler_name="cosine", warmup=30, nb_steps_tot=steps, use_mixed_precision=True, save=False, tensorboard=False,
                    cuda_graphs=True, seed=seed, log_every=log_every, fp8=fp8)
    log = logging.getLogger("fp8_bench")
    log.setLevel(logging.WARNING)
    return DecoupledTrainer(model=model, train_dataset=ds, args=args, log=log, run_name="fp8_bench")


def bench_steps():
    """Each run in a process of its own (a trainer's CUDA-graph pools stay allocated until its process ends)."""
    out = []
    for model_name, batch in (("llama125m", 8), ("llama3-1b", 4)):
        for rep in range(3):
            for fp8 in (False, True):
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--step-run", f"{model_name},{batch},{int(fp8)}"],
                                   stdout=subprocess.PIPE, text=True)
                line = [x for x in p.stdout.splitlines() if x.startswith("{")]
                assert p.returncode == 0 and line, p.stdout[-2000:]
                r = dict(json.loads(line[-1]), run=rep)
                out.append(r)
                print(json.dumps(r), flush=True)
    return out


def step_run(model_name, batch, fp8, steps=30, warmup=5):
    t = _trainer(model_name, batch, 1024, fp8)
    dev = torch.device("cuda")
    pool = [{"input_ids": torch.randint(0, t.model.config.vocab_size, (batch, 1024), device=dev)} for _ in range(4)]
    it = [0]

    def nxt():
        it[0] += 1
        return pool[it[0] % 4]
    t.input_override = nxt
    flips = 0
    while flips < warmup:
        flips += 1 if t.step() else 0
    torch.cuda.synchronize()
    m0 = t.micro_batches
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    flips = 0
    while flips < steps:
        flips += 1 if t.step() else 0
    e1.record()
    torch.cuda.synchronize()
    tok_s = (t.micro_batches - m0) * batch * 1024 / (e0.elapsed_time(e1) / 1e3)
    t._drain()
    print(json.dumps({"model": model_name, "batch": batch, "seq": 1024, "fp8": fp8, "tokens_per_s": tok_s}), flush=True)


def bench_loss(steps=300):
    from acco_b200.callbacks import TrainerCallback
    from acco_b200.data import synthetic_pretrain_dataset

    class Rec(TrainerCallback):
        def __init__(self):
            self.losses = []

        def on_log(self, trainer, scalars):
            self.losses.append(float(scalars["loss"]))
    res = {}
    ds = synthetic_pretrain_dataset(8 * steps * 2, 1024, 50257, 1024, seed=3)
    for fp8 in (False, True):
        t = _trainer("llama125m", 8, 1024, fp8, ds=ds, steps=steps, method="ddp", seed=0, log_every=1)   # on_log after every step
        cb = Rec()
        t.add_callback(cb)
        t.train()
        res["fp8" if fp8 else "bf16"] = cb.losses
        tail = cb.losses[-50:]
        print(f"loss fp8={fp8}: first {cb.losses[0]:.4f} last-50 mean {sum(tail) / len(tail):.4f} ({len(cb.losses)} steps)", flush=True)
        del t
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="gemms,steps,loss")
    ap.add_argument("--out", default=None)
    ap.add_argument("--step-run", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "fp8_bench measures on the GPU"
    os.environ.setdefault("ACCO_ALLOW_NCCL_FALLBACK", "1")
    from acco_b200 import ops
    ops.load_ext(required=True)
    if a.step_run:
        m, b, f = a.step_run.split(",")
        os.chdir(tempfile.mkdtemp(prefix="fp8_bench_"))
        step_run(m, int(b), bool(int(f)))
        from acco_b200.launch import shutdown_distributed
        shutdown_distributed()
        return
    res = {"card": card()}
    print("card:", res["card"], flush=True)
    cwd = os.getcwd()
    os.chdir(tempfile.mkdtemp(prefix="fp8_bench_"))
    try:
        parts = a.parts.split(",")
        if "gemms" in parts:
            res["gemms"] = bench_gemms()
        if "steps" in parts:
            res["steps"] = bench_steps()
        if "loss" in parts:
            res["loss"] = bench_loss()
    finally:
        os.chdir(cwd)
    from acco_b200.launch import shutdown_distributed
    shutdown_distributed()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
