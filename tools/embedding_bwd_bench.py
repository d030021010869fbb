#!/usr/bin/env python
"""The embedding backward at the Llama-3.2-1B shape (V = 128256, H = 2048, T = 4096 tokens) three ways, timed with uniform ids, Zipf
ids, Zipf ids with half the tokens set to one pad id (padded SFT rows), and one id over all T:

* ``index_add``: ``grad.index_add_(0, ids, dy)`` in bf16, the former backward (atomic adds, one bf16 rounding per occurrence);
* ``index_put``: ``grad.index_put_((ids,), dy, accumulate=True)``, PyTorch's sort-based scatter;
* ``kernel``: ``ops.embedding.embedding_bwd`` (stable ``torch.sort`` + ``embedding_bwd_kernel``), the current backward.

For each: device time per call (CUDA events over many calls, the three alternated over several samples; the median is printed), and, on
the Zipf ids with a prior row, the worst error / bound of the rows hit against the fp64 oracle of ``tests/test_step_oracle.py``
(within 0.5 is one rounding of an fp32 sum) and whether two calls give the same bits.

    python tools/embedding_bwd_bench.py [--calls 200] [--samples 5] [--out embedding_bwd_bench.json]

Prints the card name and power limit with the numbers.  Needs a GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

V, H, T = 128256, 2048, 4096


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def variants():
    from acco_b200.ops.embedding import embedding_bwd
    return {
        "index_add": lambda g, i, d: g.index_add_(0, i, d),
        "index_put": lambda g, i, d: g.index_put_((i,), d, accumulate=True),
        "kernel": embedding_bwd,
    }


def timed(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def accuracy():
    import torch
    from test_step_oracle import emb_bound, emb_checks, emb_inputs, emb_ref
    grad0, ids, dy = (t.cuda() for t in emb_inputs(V, V, H, T, "zipf", seed=V + T, prior="small"))
    o = emb_ref(grad0, ids, dy)
    bnd = emb_bound(o)
    out = {}
    for name, fn in variants().items():
        a, b = grad0.clone(), grad0.clone()
        fn(a, ids, dy)
        fn(b, ids, dy)
        c = emb_checks(a, grad0, o, bnd)
        out[name] = {"worst_error_over_bound": round(c["rows"], 3), "untouched_rows_kept": c["untouched"] == 0.0,
                     "repeatable": bool(torch.equal(a.view(torch.int16), b.view(torch.int16)))}
    return out


def timing(calls, samples):
    import torch
    from test_step_oracle import zipf_ids
    g = torch.Generator().manual_seed(0)
    dy = (torch.randn(T, H, generator=g) * 2 ** -10).bfloat16().cuda()
    grad = torch.zeros(V, H, dtype=torch.bfloat16, device="cuda")
    res = {}
    pad_half = zipf_ids(T, V, seed=2)
    pad_half[torch.randperm(T, generator=g)[: T // 2]] = V - 1          # padded SFT rows: half the tokens are the pad id
    dists = (("uniform", torch.randint(0, V, (T,), generator=g)), ("zipf", zipf_ids(T, V, seed=1)), ("pad_half", pad_half),
             ("one_id", torch.full((T,), 17, dtype=torch.long)))
    for dist, ids in dists:
        ids = ids.cuda()
        fns = variants()
        ms = {k: [] for k in fns}
        for k, fn in fns.items():                      # warm-up: module load, sort temporaries
            timed(lambda: fn(grad, ids, dy), 5)
        for _ in range(samples):
            for k, fn in fns.items():
                ms[k].append(timed(lambda: fn(grad, ids, dy), calls))
        res[dist] = {k: {"median_us": round(1e3 * statistics.median(v), 2), "min_us": round(1e3 * min(v), 2)} for k, v in ms.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu": gpu_info(), "shape": {"V": V, "H": H, "T": T}, "accuracy_zipf": accuracy(), "time": timing(a.calls, a.samples)}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
