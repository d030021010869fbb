#!/usr/bin/env python
"""Per-kernel device time of a few training steps of the headline benchmark configuration (Llama-125M ACCO, bf16, 8 x 1024 tokens,
one GPU), from torch.profiler, grouped by kernel name.  Profiling slows the run down: this is a breakdown, not a timing - take
throughput from bench.py in a separate run.

    python tools/step_profile.py --out results/profile [--steps 3] [--graphs]

Writes step_profile.json (kernels sorted by device time, share of the total, the GEMM share) under --out.  Without --graphs the
steps run eagerly, so every kernel launch is attributed individually."""
import argparse
import json
import logging
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--graphs", action="store_true", help="replay CUDA graphs as bench.py does")
    a = ap.parse_args()
    os.environ.setdefault("ACCO_ALLOW_NCCL_FALLBACK", "1")
    import torch
    from torch.profiler import ProfilerActivity, profile

    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import TokenDataset
    from acco_b200.launch import discover_env, init_distributed, shutdown_distributed
    from acco_b200.models import preset
    from bench import model_kwargs

    env = init_distributed(discover_env())
    dev = torch.device("cuda", env.local_rank)
    kw = model_kwargs("llama125m")
    torch.manual_seed(1234)
    model = preset("llama125m", device=dev, dtype=torch.bfloat16)
    g = torch.Generator().manual_seed(7)
    ds = TokenDataset({"input_ids": torch.randint(0, kw["vocab_size"], (64 * 8, 1024), generator=g, dtype=torch.long)})
    targs = AttrDict(method_name="acco", run_baseline_ddp=False, batch_size=8, n_grad_accumulation=1, max_length=1024, learning_rate=6e-4,
                     weight_decay=0.1, adam_beta1=0.9, adam_beta2=0.95, scheduler_name="cosine", warmup=1000, nb_steps_tot=10 ** 12,
                     n_warmup_steps=0, use_mixed_precision=True, const_len_batch=True, eval=False, save=False, tensorboard=False,
                     comm_backend="auto", cuda_graphs=a.graphs, seed=1234, log_every=10 ** 9, fused_ag_gemm=False, run_expe_slow=False,
                     slow_ranks=[1], slow_factor_ms=0.0)
    log = logging.getLogger("step_profile")
    log.setLevel(logging.WARNING)
    cwd = os.getcwd()
    out_dir = os.path.abspath(a.out)
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            trainer = DecoupledTrainer(model=model, train_dataset=ds, args=targs, log=log, run_name="profile")
            pool = [{"input_ids": torch.randint(0, kw["vocab_size"], (8, 1024), device=dev)} for _ in range(4)]
            it = [0]

            def from_pool():
                it[0] += 1
                return pool[it[0] % len(pool)]
            trainer.input_override = from_pool

            def run(n):
                flips = 0
                while flips < n:
                    flips += 1 if trainer.step() else 0
            run(a.warmup)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run(a.steps)
                torch.cuda.synchronize()
            trainer._drain()
        finally:
            os.chdir(cwd)
    kernels = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        d = kernels.setdefault(e.name, {"name": e.name, "us": 0.0, "count": 0})
        d["us"] += e.device_time
        d["count"] += 1
    rows = sorted(kernels.values(), key=lambda d: -d["us"])
    total = sum(d["us"] for d in rows) or 1.0
    for d in rows:
        d["share"] = d["us"] / total
        d["us_per_step"] = d["us"] / a.steps
    gemm = sum(d["us"] for d in rows if "gemm_kernel" in d["name"])
    res = {"config": "llama125m acco bf16 8x1024, 1 GPU", "steps": a.steps, "cuda_graphs": a.graphs, "device_us_per_step": total / a.steps,
           "gemm_kernel_share": gemm / total, "gemm_kernel_us_per_step": gemm / a.steps, "kernels": rows}
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "step_profile.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "kernels"}))
    for d in rows[:15]:
        print(f"{d['share'] * 100:6.2f} %  {d['us_per_step'] / 1e3:8.3f} ms/step  x{d['count'] // a.steps:<5d} {d['name'][:110]}")
    shutdown_distributed()


if __name__ == "__main__":
    main()
