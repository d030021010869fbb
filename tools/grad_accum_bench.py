#!/usr/bin/env python
"""Cost of fp32 gradient accumulators (train key ``grad_accum_dtype=fp32``) on one GPU, against the bf16 accumulators of the default:

    python tools/grad_accum_bench.py [--out results.json] [--runs 3] [--flips 6]

* wgrad GEMM time (``gemm_tt_acc``) into a bf16 and into an fp32 accumulator, at the four block-linear wgrad shapes of Llama-125M and
  Llama-3.2-1B at T = 8192 tokens: CUDA events around 50 back-to-back launches, the two targets alternated over 7 samples, medians;
* trainer tokens/s and peak allocated memory for Llama-125M at 8 x 1024 and Llama-3.2-1B at 4 x 1024 with n_grad_accumulation 8 (ACCO,
  CUDA graphs, synthetic tokens): the two settings alternated, ``--runs`` runs each, medians.

The card's name, power limit and SM clock limit are read in the same run and printed with the numbers."""
import argparse
import gc
import json
import logging
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

# (model, layer, M = weight rows, N = weight columns): the wgrad writes [M, N] from dy [T, M] and x [T, N]
SHAPES = [("llama125m", "qkv", 2304, 768), ("llama125m", "o", 768, 768), ("llama125m", "gate_up", 4096, 768), ("llama125m", "down", 768, 2048),
          ("llama3-1b", "qkv", 3072, 2048), ("llama3-1b", "o", 2048, 2048), ("llama3-1b", "gate_up", 16384, 2048), ("llama3-1b", "down", 2048, 8192)]


def card() -> dict:
    q = "name,power.limit,clocks.max.sm"
    p = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    name, power, clock = [x.strip() for x in p.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def gemm_times(T: int = 8192, reps: int = 50, samples: int = 7):
    from acco_b200.ops.gemm import gemm_tt_acc
    out = []
    for model, layer, M, N in SHAPES:
        dy = torch.randn(T, M, device="cuda").to(torch.bfloat16)
        x = torch.randn(T, N, device="cuda").to(torch.bfloat16)
        acc = {torch.bfloat16: torch.zeros(M, N, dtype=torch.bfloat16, device="cuda"), torch.float32: torch.zeros(M, N, device="cuda")}
        ms = {dt: [] for dt in acc}
        for dt in acc:                                   # warm-up: module load, tensor maps
            for _ in range(3):
                gemm_tt_acc(dy, x, acc[dt])
        for _ in range(samples):
            for dt, g in acc.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(reps):
                    gemm_tt_acc(dy, x, g)
                e1.record()
                torch.cuda.synchronize()
                ms[dt].append(e0.elapsed_time(e1) / reps)
        b, f = statistics.median(ms[torch.bfloat16]), statistics.median(ms[torch.float32])
        tflops = 2.0 * T * M * N / (f * 1e-3) / 1e12
        out.append({"model": model, "layer": layer, "M": M, "N": N, "T": T, "bf16_us": b * 1e3, "fp32_us": f * 1e3, "fp32_over_bf16": f / b,
                    "fp32_tflops": tflops})
        del dy, x, acc
    return out


def trainer_run(model_name: str, batch: int, seq: int, n_acc: int, fp32: bool, flips: int) -> dict:
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import TokenDataset
    from acco_b200.models import PRESETS, preset
    vocab = PRESETS[model_name][1]["vocab_size"]
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    torch.manual_seed(1234)
    model = preset(model_name, device=torch.device("cuda", 0), dtype=torch.bfloat16)
    g = torch.Generator().manual_seed(7)
    ds = TokenDataset({"input_ids": torch.randint(0, vocab, (64 * batch, seq), generator=g, dtype=torch.long)})
    args = AttrDict(method_name="acco", batch_size=batch, n_grad_accumulation=n_acc, max_length=seq, learning_rate=6e-4, weight_decay=0.1,
                    warmup=1000, nb_steps_tot=10 ** 12, use_mixed_precision=True, const_len_batch=True, eval=False, save=False,
                    tensorboard=False, seed=1234, log_every=10 ** 9, static_accumulation=True,
                    grad_accum_dtype="fp32" if fp32 else None)
    log = logging.getLogger("grad_accum_bench")
    log.setLevel(logging.WARNING)
    cwd = os.getcwd()
    tmp = tempfile.mkdtemp(prefix="acco_ga_bench_")
    os.chdir(tmp)
    try:
        t = DecoupledTrainer(model=model, train_dataset=ds, args=args, log=log, run_name="ga")
        pool = [{"input_ids": torch.randint(0, vocab, (batch, seq), device="cuda")} for _ in range(8)]
        it = [0]

        def from_pool():
            it[0] += 1
            return pool[it[0] % len(pool)]
        t.input_override = from_pool
        for _ in range(3):
            while not t.step():
                pass
        torch.cuda.synchronize()
        m0, t0 = t.micro_batches, time.perf_counter()
        for _ in range(flips):
            while not t.step():
                pass
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        micro = t.micro_batches - m0
        t._drain()
        peak = torch.cuda.max_memory_allocated()
        assert t.arena.grad_dtype == (torch.float32 if fp32 else torch.bfloat16)
    finally:
        os.chdir(cwd)
    del t, model, pool
    gc.collect()
    torch.cuda.empty_cache()
    return {"tokens_per_s": micro * batch * seq / dt, "peak_gb": peak / 1e9}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--flips", type=int, default=6, help="timed trainer steps (rounds of n_grad_accumulation micro-batches) per run")
    ap.add_argument("--skip-trainer", action="store_true")
    a = ap.parse_args(argv)
    assert torch.cuda.is_available(), "grad_accum_bench measures on a GPU"
    os.environ.setdefault("ACCO_ALLOW_NCCL_FALLBACK", "1")
    res = {"card": card(), "gemm": gemm_times()}
    for r in res["gemm"]:
        print(f"{r['model']:10s} {r['layer']:8s} [{r['M']} x {r['N']}] T={r['T']}: bf16 {r['bf16_us']:.1f} us, fp32 {r['fp32_us']:.1f} us "
              f"({r['fp32_over_bf16']:.3f}x)", flush=True)
    if not a.skip_trainer:
        res["trainer"] = []
        for model_name, batch in (("llama125m", 8), ("llama3-1b", 4)):
            runs = {False: [], True: []}
            for _ in range(a.runs):
                for fp32 in (False, True):
                    runs[fp32].append(trainer_run(model_name, batch, 1024, 8, fp32, a.flips))
            row = {"model": model_name, "batch": batch, "seq": 1024, "n_grad_accumulation": 8}
            for fp32, rs in runs.items():
                k = "fp32" if fp32 else "bf16"
                row[f"{k}_tokens_per_s"] = statistics.median(r["tokens_per_s"] for r in rs)
                row[f"{k}_peak_gb"] = statistics.median(r["peak_gb"] for r in rs)
                row[f"{k}_runs"] = rs
            res["trainer"].append(row)
            print(f"{model_name} {batch}x1024 nacc8: bf16 {row['bf16_tokens_per_s']:.0f} tok/s {row['bf16_peak_gb']:.2f} GB, "
                  f"fp32 {row['fp32_tokens_per_s']:.0f} tok/s {row['fp32_peak_gb']:.2f} GB", flush=True)
    print(json.dumps(res["card"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    return res


if __name__ == "__main__":
    main()
