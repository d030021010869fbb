#!/usr/bin/env python
"""Cost of the no-decay table (train key ``no_decay_1d``) in the fused AdamW pass: the local ``adamw_shard`` at the shard sizes of
Llama-125M and Llama-3.2-1B (the whole model, and rank 3's slice of eight), bf16 gradients and weights, without a table and with
the model's real table, arms alternated.

    python tools/no_decay_bench.py [--launches 200 --samples 5 --out no_decay_bench.json]

Per launch the pass reads the gradient (2 B/element) and master, exp_avg, exp_avg_sq (12 B) and writes those three (12 B) and the
bf16 weights (2 B): 28 bytes per element; the GB/s below is that over the CUDA-event time.  Needs a GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BYTES_PER_ELEMENT = 2 + 12 + 12 + 2


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def model_table(name):
    """(numel, no-decay ranges, number of excluded parameters) of a preset, from its shapes alone (meta device)."""
    import torch
    from acco_b200.models import preset
    from acco_b200.parallel.arena import no_decay_ranges, unique_parameters
    params = unique_parameters(preset(name, device=torch.device("meta"), dtype=torch.bfloat16))
    return sum(p.numel() for p in params), no_decay_ranges(params), sum(1 for p in params if p.ndim <= 1 and p.requires_grad)


def cases():
    from acco_b200.parallel.arena import ShardLayout
    out = []
    for name in ("llama125m", "llama3-1b"):
        numel, ranges, n_params = model_table(name)
        for world, rank in ((1, 0), (8, 3)):
            lay = ShardLayout(numel, world, 1024)
            S, base = lay.size_slice, rank * lay.size_slice
            out.append(dict(model=name, world=world, rank=rank, shard=S, base=base, ranges=ranges, excluded_parameters=n_params,
                            excluded_elements=sum(b - a for a, b in ranges),
                            ranges_in_shard=sum(1 for a, b in ranges if a < base + S and b > base)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no_decay_bench needs a GPU")
    from acco_b200 import ops
    from acco_b200.parallel.schedule import COMMIT_ALL
    C = ops.load_ext(required=True)
    dev = torch.device("cuda", 0)
    rep = {"gpu": gpu_info(), "launches_per_sample": a.launches, "bytes_per_element": BYTES_PER_ELEMENT, "cases": []}
    for c in cases():
        S = c["shard"]
        g = (torch.randn(S, device=dev) * 0.01).bfloat16()
        master, m, v, stash = (torch.randn(S, device=dev) * 0.02, torch.zeros(S, device=dev), torch.zeros(S, device=dev), torch.zeros(8, device=dev))
        out = torch.zeros(S, device=dev, dtype=torch.bfloat16)
        inv, scratch = torch.ones(1, device=dev), torch.zeros(4, dtype=torch.int32, device=dev)
        table = torch.tensor(c["ranges"], dtype=torch.int64, device=dev)

        def launch(tab):
            C.adamw_shard(g, master, m, v, stash, out, inv, scratch, 6e-4, 0.9, 0.95, 1e-8, 0.1, 10, COMMIT_ALL, False, False, tab, c["base"])

        def sample(tab):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.launches):
                launch(tab)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / a.launches

        for tab in (None, table):
            for _ in range(20):
                launch(tab)
        torch.cuda.synchronize()
        ms = {"absent": [], "table": []}
        for _ in range(a.samples):
            ms["absent"].append(sample(None))
            ms["table"].append(sample(table))
        res = {k: c[k] for k in c if k != "ranges"}
        res["ranges"] = len(c["ranges"])
        for k, xs in ms.items():
            med = statistics.median(xs)
            res[k] = {"ms_median": med, "ms_min": min(xs), "ms_max": max(xs), "GBps": S * BYTES_PER_ELEMENT / (med * 1e-3) / 1e9}
        res["table_over_absent_pct"] = 100.0 * (res["table"]["ms_median"] / res["absent"]["ms_median"] - 1.0)
        rep["cases"].append(res)
        del g, master, m, v, out
        torch.cuda.empty_cache()
    print(json.dumps(rep, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
