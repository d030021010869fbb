#!/usr/bin/env python
"""Cost and effect of the z-loss (train key ``z_loss_weight``) on the native models, three ways:

(a) ``kernels``: device time of the cross-entropy forward (``ce_fwd`` + ``ce_reduce``) and in-place backward at z = 0 and z = 1e-4,
    T x Vp = 8192 x 50304 (V = 50257) and 4096 x 128256; CUDA events over many launches, the two arms alternated, medians.  The
    forward reads the logits once, the backward reads and writes them: 6 bytes per logit, reported against HBM3's 3.35 TB/s.
(b) ``trainer``: ACCO tokens/s with CUDA graphs, key off vs on, for Llama-125M at 8 x 1024 and the Llama-3.2-1B preset at 4 x 1024
    (const-len synthetic pre-training rows, one GPU); the arms alternated ``--repeats`` times, medians.
(c) ``effect``: two same-seed ACCO runs of Llama-125M on ``synthetic_pretrain_dataset`` (``--effect-steps`` micro-batches of
    8 x 1024), without and with z = 1e-4.  Over the last 50 micro-batches, each batch is scored before it trains (the round in
    flight drained first, so on the weights it runs on): mean cross-entropy and mean ``lse^2``.  It reports; it asserts nothing.

    python tools/z_loss_bench.py [--only kernels,trainer,effect] [--out z_loss_bench.json]

Prints the card name and power limit with the numbers.  Needs a GPU."""
import argparse
import gc
import json
import logging
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

Z = 1e-4
HBM_TBPS = 3.35
SEQ = 1024


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def bench_kernels(launches, samples):
    import torch
    from acco_b200 import ops
    C = ops.load_ext(required=True)
    out = []
    for T, V, Vp in ((8192, 50257, 50304), (4096, 128256, 128256)):
        g = torch.Generator(device="cuda").manual_seed(0)
        lg = (2 * torch.randn(T, Vp, device="cuda", generator=g)).bfloat16()
        lab = torch.randint(0, V, (T,), device="cuda", generator=g)
        scratch = lg.clone()                     # the backward overwrites its input; its cost does not depend on the values
        z_out = torch.zeros(1, device="cuda")
        res = {"T": T, "V": V, "Vp": Vp}
        arms = {}
        for z in (0.0, Z):
            _, inv_n, lse = C.ce_fwd(lg, lab, V, -100, 0.0, z, z_out)
            fwd = lambda z=z: C.ce_fwd(lg, lab, V, -100, 0.0, z, z_out)
            bwd = lambda z=z, lse=lse, inv_n=inv_n: C.ce_bwd_inplace(scratch, lab, lse, inv_n, V, -100, 0.0, z)
            for _ in range(10):
                fwd(), bwd()
            arms[z] = (fwd, bwd, {"fwd": [], "bwd": []})
        torch.cuda.synchronize()
        for _ in range(samples):
            for z, (fwd, bwd, acc) in arms.items():
                acc["fwd"].append(timed(fwd, launches))
                acc["bwd"].append(timed(bwd, launches))
        for z, (_, _, acc) in arms.items():
            f, b = statistics.median(acc["fwd"]), statistics.median(acc["bwd"])
            tbps = T * Vp * 6 / ((f + b) * 1e-3) / 1e12
            res[f"z={z}"] = {"fwd_us": 1e3 * f, "bwd_us": 1e3 * b, "total_us": 1e3 * (f + b),
                             "fwd_min_max_us": [1e3 * min(acc["fwd"]), 1e3 * max(acc["fwd"])],
                             "bwd_min_max_us": [1e3 * min(acc["bwd"]), 1e3 * max(acc["bwd"])],
                             "TBps": tbps, "share_of_3.35_TBps": tbps / HBM_TBPS}
        res["z_over_plain_pct"] = 100.0 * (res[f"z={Z}"]["total_us"] / res["z=0.0"]["total_us"] - 1.0)
        out.append(res)
        del lg, scratch
        torch.cuda.empty_cache()
    return out


def _trainer(model_name, B, z, ds):
    import torch
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.launch import DistEnv
    from acco_b200.models import preset
    torch.manual_seed(0)
    model = preset(model_name, device="cuda", dtype=torch.bfloat16)
    args = AttrDict(method_name="acco", batch_size=B, n_grad_accumulation=1, max_length=SEQ, learning_rate=6e-4, weight_decay=0.1,
                    adam_beta1=0.9, adam_beta2=0.95, scheduler_name="cosine", warmup=100, nb_steps_tot=10 ** 12, use_mixed_precision=True,
                    const_len_batch=True, eval=False, save=False, tensorboard=False, seed=1, log_every=10 ** 9, z_loss_weight=z)
    log = logging.getLogger("z_loss_bench")
    log.setLevel(logging.WARNING)
    return DecoupledTrainer(model=model, train_dataset=ds, args=args, log=log, env=DistEnv(id_run=f"{model_name}-z{z}"))


def _close(t):
    import torch
    t._drain()
    if t._feeder is not None:
        t._feeder.close()
    del t
    gc.collect()
    torch.cuda.empty_cache()


def run_e2e(model_name, B, z, ds, warmup, micro):
    import torch
    t = _trainer(model_name, B, z, ds)
    while t.micro_batches < warmup:
        t.step()
    torch.cuda.synchronize()
    m0 = t.micro_batches
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    while t.micro_batches < m0 + micro:
        t.step()
    e1.record()
    torch.cuda.synchronize()
    n = t.micro_batches - m0
    ms = e0.elapsed_time(e1) / n
    out = {"ms_per_micro_batch": ms, "tokens_per_s": B * SEQ / (ms * 1e-3), "graphs": t._graphs is not None and not
           getattr(t, "_graphs_disabled", None), "z_loss": float(t.z_loss_host) if z else None}
    _close(t)
    return out


def bench_trainer(repeats, warmup, micro):
    from acco_b200.data import synthetic_pretrain_dataset
    from acco_b200.models import PRESETS
    out = []
    for name, B in (("llama125m", 8), ("llama3-1b", 4)):
        V = PRESETS[name][1]["vocab_size"]
        ds = synthetic_pretrain_dataset(3000, 400, V, SEQ, seed=0)
        res = {"model": name, "batch": B, "seq": SEQ, "runs": {0.0: [], Z: []}}
        for _ in range(repeats):
            for z in (0.0, Z):
                r = run_e2e(name, B, z, ds, warmup, micro)
                res["runs"][z].append(r)
                print(name, z, json.dumps(r), flush=True)
        res["runs"] = {f"z={z}": v for z, v in res["runs"].items()}
        for k, v in res["runs"].items():
            res[f"{k}_median_tokens_per_s"] = statistics.median(r["tokens_per_s"] for r in v)
        res["z_over_plain_pct"] = 100.0 * (res[f"z={Z}_median_tokens_per_s"] / res["z=0.0_median_tokens_per_s"] - 1.0)
        out.append(res)
    return out


def bench_effect(steps, last=50):
    import torch
    import torch.nn.functional as F
    from acco_b200.data import stack_collate, synthetic_pretrain_dataset
    from acco_b200.models import PRESETS
    V = PRESETS["llama125m"][1]["vocab_size"]
    B = 8
    ds = synthetic_pretrain_dataset(2 * (steps + 2) * B * SEQ // 400, 400, V, SEQ, seed=0)     # about twice the rows the run reads
    assert len(ds) >= (steps + 2) * B, len(ds)
    out = {"model": "llama125m", "batch": B, "seq": SEQ, "micro_batches": steps, "last": last}
    for z in (0.0, Z):
        t = _trainer("llama125m", B, z, ds)
        k = [0]

        def nxt():
            i = k[0]
            k[0] += 1
            return {"input_ids": stack_collate([ds[j] for j in range(i * B, (i + 1) * B)])["input_ids"].cuda()}
        batch = [nxt()]
        t.input_override = lambda: batch[0]
        ce, lse2 = [], []
        while t.micro_batches < steps:
            if t.micro_batches >= steps - last:
                t._drain()
                with torch.no_grad():
                    ids = batch[0]["input_ids"]
                    lg = t.model(input_ids=ids).logits[:, :-1].reshape(-1, V).float()
                    ce.append(float(F.cross_entropy(lg, ids[:, 1:].reshape(-1))))
                    lse2.append(float(torch.logsumexp(lg, -1).square().mean()))
                    del lg
            t.step()
            batch[0] = nxt()
        out[f"z={z}"] = {"mean_ce_last": statistics.fmean(ce), "mean_lse2_last": statistics.fmean(lse2), "final_loss": float(t.loss_host)}
        print("effect", z, json.dumps(out[f"z={z}"]), flush=True)
        _close(t)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="kernels,trainer,effect")
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--samples", type=int, default=7)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=20, help="micro-batches before the timed window")
    ap.add_argument("--micro", type=int, default=60, help="micro-batches in the timed window")
    ap.add_argument("--effect-steps", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("z_loss_bench needs a GPU")
    os.environ.setdefault("ACCO_ALLOW_NCCL_FALLBACK", "1")
    parts = a.only.split(",")
    rep = {"gpu": gpu_info(), "z": Z}
    print("GPU:", rep["gpu"], flush=True)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)                            # the trainer writes nothing here with save / tensorboard off; keep the tree clean anyway
        try:
            if "kernels" in parts:
                rep["kernels"] = bench_kernels(a.launches, a.samples)
                print(json.dumps(rep["kernels"], indent=1), flush=True)
            if "trainer" in parts:
                rep["trainer"] = bench_trainer(a.repeats, a.warmup, a.micro)
            if "effect" in parts:
                rep["effect"] = bench_effect(a.effect_steps)
        finally:
            os.chdir(cwd)
    rep["gpu_after"] = gpu_info()
    print(json.dumps(rep))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
