#!/usr/bin/env python
"""Cost of gradient-norm clipping on the headline workload (Llama-125M, 8 x 1024 tokens per micro-batch, ACCO, CUDA graphs, one GPU):
time ``trainer.step()`` with ``max_grad_norm`` unset and 1.0, runs alternated, and report tokens/s, the round time and the GPU.

    python tools/clip_bench.py [--steps 20 --warmup 5 --repeats 3 --out clip_bench.json]

With clipping on, every round first streams the gradient accumulator once more (``round_norm_kernel``) before the fused AdamW
round; the difference between the two arms is that pass plus its launch."""
import argparse
import json
import logging
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run_arm(max_grad_norm, steps, warmup):
    import torch
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import TokenDataset
    from acco_b200.launch import DistEnv
    from acco_b200.models import preset
    from bench import model_kwargs
    dev = torch.device("cuda", 0)
    kw = model_kwargs("llama125m")
    torch.manual_seed(1234)
    model = preset("llama125m", device=dev, dtype=torch.bfloat16)
    B, S = 8, 1024
    ds = TokenDataset({"input_ids": torch.randint(0, kw["vocab_size"], (64 * B, S), generator=torch.Generator().manual_seed(7))})
    args = AttrDict(method_name="acco", batch_size=B, n_grad_accumulation=1, max_length=S, learning_rate=6e-4, weight_decay=0.1,
                    adam_beta1=0.9, adam_beta2=0.95, scheduler_name="cosine", warmup=1000, nb_steps_tot=10 ** 12, use_mixed_precision=True,
                    const_len_batch=True, eval=False, save=False, tensorboard=False, cuda_graphs=True, seed=1234, log_every=10 ** 9,
                    max_grad_norm=max_grad_norm)
    log = logging.getLogger("clip_bench")
    log.setLevel(logging.WARNING)
    cwd = os.getcwd()
    os.chdir(tempfile.mkdtemp(prefix="acco_clip_bench_"))
    try:
        t = DecoupledTrainer(model=model, train_dataset=ds, args=args, log=log, env=DistEnv(id_run="clip_bench"))
        pool = [{"input_ids": torch.randint(0, kw["vocab_size"], (B, S), device=dev)} for _ in range(8)]
        it = [0]

        def from_pool():
            it[0] += 1
            return pool[it[0] % len(pool)]
        t.input_override = from_pool

        def flips(n):
            k = 0
            while k < n:
                k += 1 if t.step() else 0
        flips(warmup)
        torch.cuda.synchronize()
        m0 = t.micro_batches
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        flips(steps)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        res = {"tokens_per_s": (t.micro_batches - m0) * B * S / (ms / 1e3), "ms_per_step": ms / steps,
               "comm_ms_per_round": t.overlap.summary()["comm_ms_mean"], "backend": t.backend.name,
               "last_grad_norm": t.backend.last_grad_norm}
        t._drain()
    finally:
        os.chdir(cwd)
    del t, model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("clip_bench needs a GPU")
    runs = {"off": [], "1.0": []}
    for _ in range(a.repeats):
        runs["off"].append(run_arm(None, a.steps, a.warmup))
        runs["1.0"].append(run_arm(1.0, a.steps, a.warmup))
    med = {k: statistics.median(r["tokens_per_s"] for r in v) for k, v in runs.items()}
    rep = {"gpu": gpu_info(), "workload": "llama125m, 8x1024 tokens, acco, cuda graphs, 1 GPU", "runs": runs,
           "median_tokens_per_s": med, "slowdown_pct": 100.0 * (1.0 - med["1.0"] / med["off"]),
           "spread_pct": {k: 100.0 * (max(r["tokens_per_s"] for r in v) - min(r["tokens_per_s"] for r in v)) / med[k] for k, v in runs.items()}}
    print(json.dumps(rep, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
