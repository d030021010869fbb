#!/usr/bin/env python
"""Fine-tuning throughput with and without sample packing (single GPU):

    python tools/sft_packing_bench.py [--models llama125m,llama3-1b] [--repeats 3] [--out DIR]

End to end: the `acco-ft` settings (ACCO, batch 4, n_grad_accumulation 2, max_length 512, bf16, CUDA graphs) on alpaca-shaped
synthetic samples (`synthetic_sft_dataset(n, 180, V, 512)`: lognormal lengths, mean ~160 tokens), three variants:
  * padded  - `PadCollator` (right-padded to the longest sample, multiple of 64), library SDPA attention;
  * own     - the same with ACCO_ATTN=own (own flash-attention kernels, padded to a multiple of 128);
  * packed  - `packing=True`: first-fit-decreasing rows of 512 tokens, document-masked own kernels, one graph shape.
It reports target tokens/s (labels != -100, the tokens that train the model) and ms per micro-batch.  The target count of a
micro-batch is the mean over one epoch of the run's own loader; the time is CUDA events around `trainer.step()` after a warm-up.

Attention only (fwd + bwd, CUDA events): the segmented kernels against the unsegmented ones on single-sample rows (the cost of the
bound), and on packed rows against the dense-mask SDPA fallback and `flash_attn_varlen_func` (with the q/k/v copies it needs).

Variants alternate inside each repeat; the card name and power limit are read in the same run and printed with the numbers."""
import argparse
import gc
import json
import logging
import math
import os
import statistics
import subprocess
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from acco_b200 import AttrDict, ops

VARIANTS = ("padded", "own", "packed")


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [x.strip() for x in q.split(",")]
    except Exception as e:  # noqa: BLE001 - report what could not be read instead of a number
        info["power_limit"] = f"unknown ({type(e).__name__})"
    return info


# ---------------------------------------------------------------------------------------------- end to end
def run_e2e(model_name: str, variant: str, ds, warmup: int, micro: int) -> dict:
    from acco_b200 import DecoupledTrainer
    from acco_b200.launch import DistEnv
    from acco_b200.models import PRESETS, preset
    V = PRESETS[model_name][1]["vocab_size"]
    if variant == "own":
        os.environ["ACCO_ATTN"] = "own"
    else:
        os.environ.pop("ACCO_ATTN", None)
    torch.manual_seed(0)
    model = preset(model_name, device="cuda", dtype=torch.bfloat16)
    tok = types.SimpleNamespace(pad_token_id=V - 1, eos_token_id=V - 1)
    args = AttrDict(method_name="acco", batch_size=4, n_grad_accumulation=2, max_length=512, learning_rate=2e-5, weight_decay=0.0,
                    adam_beta1=0.9, adam_beta2=0.95, scheduler_name="cosine", warmup=0, nb_steps_tot=10 ** 12, use_mixed_precision=True,
                    const_len_batch=False, packing=(variant == "packed"), eval=False, save=False, tensorboard=False, seed=1,
                    log_every=10 ** 9)
    log = logging.getLogger("sft_packing_bench")
    log.setLevel(logging.WARNING)
    t = DecoupledTrainer(model=model, tokenizer=tok, train_dataset=ds, args=args, log=log, env=DistEnv(id_run=f"{model_name}-{variant}"))
    targets = [int((b["labels"] != -100).sum()) for b in t.train_dataloader]
    while t.micro_batches < warmup:
        t.step()
    torch.cuda.synchronize()
    m0, g0 = t.micro_batches, (len(t._graphs._graphs) if t._graphs is not None else 0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    while t.micro_batches < m0 + micro:
        t.step()
    e1.record()
    torch.cuda.synchronize()
    n = t.micro_batches - m0
    ms = e0.elapsed_time(e1) / n
    out = {"model": model_name, "variant": variant, "ms_per_micro_batch": ms, "target_tokens_per_micro_batch": statistics.mean(targets),
           "target_tokens_per_s": statistics.mean(targets) / (ms * 1e-3), "micro_batches_timed": n,
           "graphs_captured_in_window": (len(t._graphs._graphs) if t._graphs is not None else 0) - g0,
           "loss": float(t.loss_host)}
    t._drain()
    if t._feeder is not None:
        t._feeder.close()
    del t, model
    gc.collect()
    torch.cuda.empty_cache()
    os.environ.pop("ACCO_ATTN", None)
    return out


# ---------------------------------------------------------------------------------------------- attention only
def timed(fn, iters=20) -> float:
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def attention_cases(B: int, S: int, Hq: int, Hk: int):
    """-> {variant: fwd+bwd callable} on the same bf16 qkv / dO."""
    import numpy as np
    from acco_b200.data import pack_sft, synthetic_documents
    from acco_b200.ops.attention import _attend
    C = ops.load_ext(required=True)
    D = 64
    sc = 1.0 / math.sqrt(D)
    g = torch.Generator().manual_seed(0)
    qkv = (torch.randn(B * S, (Hq + 2 * Hk) * D, generator=g) * 0.7).to("cuda", torch.bfloat16)
    d_o = (torch.randn(B * S, Hq * D, generator=g) * 0.5).to("cuda", torch.bfloat16)
    packed = pack_sft(synthetic_documents(400, 180, 1000, seed=1, min_len=4, max_len=S), S)
    seg = np.zeros((B, S), dtype=np.int32)
    lens = []
    for b, row in enumerate(packed["doc_lens"][:B]):
        a = 0
        for n in row + [S - sum(row)]:                         # the pad tail is one more segment
            if n:
                seg[b, a:a + n] = a
                lens.append(n)
            a += n
    seg = torch.from_numpy(seg.reshape(-1)).cuda()
    zero = torch.zeros(B * S, dtype=torch.int32, device="cuda")
    cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device="cuda")

    def own(s):
        def f():
            o, lse = C.attn_fwd(qkv, B, S, Hq, Hk, D, sc, 0, *(() if s is None else (s,)))
            C.attn_bwd(qkv, o, d_o, lse, B, S, Hq, Hk, D, sc, 0, *(() if s is None else (s,)))
        return f

    x = qkv.view(B, S, Hq + 2 * Hk, D)
    q, k, v = (t.transpose(1, 2).detach().requires_grad_() for t in (x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:]))
    do_t = d_o.view(B, S, Hq, D).transpose(1, 2)

    def sdpa_mask():
        o = _attend(q, k, v, sc, None, Hk != Hq, seg)
        torch.autograd.grad(o, (q, k, v), do_t)

    def own_fwd(s):
        return lambda: C.attn_fwd(qkv, B, S, Hq, Hk, D, sc, 0, *(() if s is None else (s,)))

    cases = {"own_unsegmented_single_sample": own(None), "own_segmented_single_sample": own(zero), "own_segmented_packed": own(seg),
             "sdpa_dense_mask_packed": sdpa_mask,
             "own_unsegmented_single_sample_fwd_only": own_fwd(None), "own_segmented_single_sample_fwd_only": own_fwd(zero)}
    try:
        from flash_attn import flash_attn_varlen_func
        x2 = qkv.view(B * S, Hq + 2 * Hk, D)
        dof = d_o.view(B * S, Hq, D)
        max_len = max(lens)

        def flash():
            fq, fk, fv = (t.contiguous().requires_grad_() for t in (x2[:, :Hq], x2[:, Hq:Hq + Hk], x2[:, Hq + Hk:]))   # the copies it needs
            o = flash_attn_varlen_func(fq, fk, fv, cu, cu, max_len, max_len, softmax_scale=sc, causal=True)
            torch.autograd.grad(o, (fq, fk, fv), dof)
        cases["flash_attn_varlen_packed"] = flash
    except Exception as e:  # noqa: BLE001
        print(f"flash_attn_varlen_func not available: {type(e).__name__}: {e}", flush=True)
    return cases


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="llama125m,llama3-1b")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=40, help="micro-batches before the timed window")
    ap.add_argument("--micro", type=int, default=60, help="micro-batches in the timed window")
    ap.add_argument("--samples", type=int, default=4000)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--out", default=None, help="directory for sft_packing_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    ops.load_ext(required=True)
    os.environ.setdefault("ACCO_ALLOW_NCCL_FALLBACK", "1")
    report = {"card": card(), "e2e": [], "attention": []}
    print(json.dumps({"card": report["card"]}), flush=True)
    cwd = os.getcwd()
    os.chdir(tempfile.mkdtemp(prefix="sft_packing_bench_"))          # the trainer writes its run files into the working directory
    try:
        from acco_b200.data import synthetic_sft_dataset
        from acco_b200.models import PRESETS
        for name in ([] if a.skip_e2e else a.models.split(",")):
            V = PRESETS[name][1]["vocab_size"]
            ds = synthetic_sft_dataset(a.samples, 180, V - 1, 512, seed=0)
            for r in range(a.repeats):
                for variant in VARIANTS:
                    res = run_e2e(name, variant, ds, a.warmup, a.micro)
                    res["repeat"] = r
                    report["e2e"].append(res)
                    print(json.dumps(res), flush=True)
        for (B, S, Hq, Hk) in ((4, 512, 12, 12), (4, 512, 32, 8)):
            cases = attention_cases(B, S, Hq, Hk)
            times = {k: [] for k in cases}
            for _ in range(a.repeats):
                for k, f in cases.items():
                    times[k].append(timed(f))
            for k, ts in times.items():
                res = {"shape": [B, S, Hq, Hk], "variant": k, "fwd_bwd_ms": ts, "median_ms": statistics.median(ts)}
                report["attention"].append(res)
                print(json.dumps(res), flush=True)
    finally:
        os.chdir(cwd)
    from acco_b200.launch import shutdown_distributed
    shutdown_distributed()
    c = report["card"]
    print(f"\n{c['name']}, power limit {c.get('power_limit')}, max SM clock {c.get('max_sm_clock')}")
    print("| model | variant | target tokens/s (median of runs) | ms / micro-batch | runs |\n|---|---|---|---|---|")
    for name in sorted({e["model"] for e in report["e2e"]}):
        for variant in VARIANTS:
            rs = [e for e in report["e2e"] if e["model"] == name and e["variant"] == variant]
            tps = [e["target_tokens_per_s"] for e in rs]
            print(f"| {name} | {variant} | {statistics.median(tps):,.0f} | {statistics.median(e['ms_per_micro_batch'] for e in rs):.2f} | "
                  f"{', '.join(f'{x:,.0f}' for x in tps)} |")
    print("\n| B, S, Hq, Hk | attention fwd+bwd | median ms | runs |\n|---|---|---|---|")
    for e in report["attention"]:
        print(f"| {e['shape']} | {e['variant']} | {e['median_ms']:.3f} | {', '.join(f'{x:.3f}' for x in e['fwd_bwd_ms'])} |")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(report, open(os.path.join(a.out, "sft_packing_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
