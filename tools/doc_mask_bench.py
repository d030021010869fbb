#!/usr/bin/env python
"""Pre-training throughput with and without document masking (single GPU):

    python tools/doc_mask_bench.py [--models llama125m,llama3-1b] [--repeats 3] [--out DIR]

End to end: ACCO, bf16, CUDA graphs, n_grad_accumulation 1, const-len rows of 1024 tokens packed from openwebtext-shaped synthetic
documents (`synthetic_pretrain_dataset(n, 900, V, 1024)`, mean length ~900 tokens), Llama-125M at batch 8 and the Llama-3.2-1B
shape at batch 4, with `document_mask` off (`stack_collate`, attention through cuDNN SDPA) and on (`DocumentCollator`, the
segmented own kernels).  Every token of a const-len row trains, so the rate is tokens/s = B * S / time per micro-batch, the time
being CUDA events around `trainer.step()` after a warm-up.  The two settings alternate inside each repeat.

Attention only (fwd + bwd per layer, CUDA events) at the same shapes and segmentations: the unmasked SDPA path the key-off runs
take, and the segmented kernels on the rows `DocumentCollator` makes.

The card name and power limit are read in the same run and printed with the numbers."""
import argparse
import gc
import json
import logging
import math
import os
import statistics
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from acco_b200 import AttrDict, ops

from sft_packing_bench import card, timed

SHAPES = {"llama125m": 8, "llama3-1b": 4}         # micro-batch of each model at S = 1024
SEQ = 1024


# ---------------------------------------------------------------------------------------------- end to end
def run_e2e(model_name: str, masked: bool, ds, warmup: int, micro: int) -> dict:
    from acco_b200 import DecoupledTrainer
    from acco_b200.launch import DistEnv
    from acco_b200.models import PRESETS, preset
    V = PRESETS[model_name][1]["vocab_size"]
    B = SHAPES[model_name]
    torch.manual_seed(0)
    model = preset(model_name, device="cuda", dtype=torch.bfloat16)
    tok = types.SimpleNamespace(eos_token_id=V - 1)
    args = AttrDict(method_name="acco", batch_size=B, n_grad_accumulation=1, max_length=SEQ, learning_rate=6e-4, weight_decay=0.1,
                    adam_beta1=0.9, adam_beta2=0.95, scheduler_name="cosine", warmup=0, nb_steps_tot=10 ** 12, use_mixed_precision=True,
                    const_len_batch=True, document_mask=masked, eval=False, save=False, tensorboard=False, seed=1, log_every=10 ** 9)
    log = logging.getLogger("doc_mask_bench")
    log.setLevel(logging.WARNING)
    t = DecoupledTrainer(model=model, tokenizer=tok, train_dataset=ds, args=args, log=log,
                         env=DistEnv(id_run=f"{model_name}-{'masked' if masked else 'plain'}"))
    ops.reset_launch_counts()
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
    counts = ops.launch_counts()
    out = {"model": model_name, "document_mask": masked, "batch": B, "seq": SEQ, "ms_per_micro_batch": ms,
           "tokens_per_s": B * SEQ / (ms * 1e-3), "micro_batches_timed": n,
           "graphs": len(t._graphs._graphs) if t._graphs is not None else 0,
           "graphs_captured_in_window": (len(t._graphs._graphs) if t._graphs is not None else 0) - g0,
           "segmented_attention_launches": counts.get("attn_fwd_seg", 0), "loss": float(t.loss_host)}
    t._drain()
    if t._feeder is not None:
        t._feeder.close()
    del t, model
    gc.collect()
    torch.cuda.empty_cache()
    return out


# ---------------------------------------------------------------------------------------------- attention only
def attention_cases(ds, eos: int, B: int, S: int, Hq: int, Hk: int):
    """-> ({variant: fwd+bwd callable} on the same bf16 qkv / dO, segments per row) for the first B rows of ``ds``."""
    from acco_b200.data import DocumentCollator
    from acco_b200.ops.attention import _sdpa, segment_starts
    C = ops.load_ext(required=True)
    D = 64
    sc = 1.0 / math.sqrt(D)
    g = torch.Generator().manual_seed(0)
    qkv = (torch.randn(B * S, (Hq + 2 * Hk) * D, generator=g) * 0.7).to("cuda", torch.bfloat16)
    d_o = (torch.randn(B * S, Hq * D, generator=g) * 0.5).to("cuda", torch.bfloat16)
    batch = DocumentCollator(eos)([ds[i] for i in range(B)])
    seg = segment_starts(batch["position_ids"]).cuda()
    n_seg = int((batch["position_ids"] == 0).sum()) / B

    def own():
        o, lse = C.attn_fwd(qkv, B, S, Hq, Hk, D, sc, 0, seg)
        C.attn_bwd(qkv, o, d_o, lse, B, S, Hq, Hk, D, sc, 0, seg)

    x = qkv.view(B, S, Hq + 2 * Hk, D)
    q, k, v = (t.transpose(1, 2).detach().requires_grad_() for t in (x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:]))
    do_t = d_o.view(B, S, Hq, D).transpose(1, 2)

    def sdpa():                                         # what the key-off model runs (`rope_causal_attention` without seg)
        o = _sdpa(q, k, v, None, Hk != Hq)
        torch.autograd.grad(o, (q, k, v), do_t)

    return {"sdpa_unmasked": sdpa, "own_segmented": own}, n_seg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="llama125m,llama3-1b")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=20, help="micro-batches before the timed window")
    ap.add_argument("--micro", type=int, default=50, help="micro-batches in the timed window")
    ap.add_argument("--docs", type=int, default=3000)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--out", default=None, help="directory for doc_mask_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    ops.load_ext(required=True)
    os.environ.setdefault("ACCO_ALLOW_NCCL_FALLBACK", "1")
    os.environ.pop("ACCO_ATTN", None)
    report = {"card": card(), "e2e": [], "attention": []}
    print(json.dumps({"card": report["card"]}), flush=True)
    cwd = os.getcwd()
    os.chdir(tempfile.mkdtemp(prefix="doc_mask_bench_"))          # the trainer writes its run files into the working directory
    try:
        from acco_b200.data import synthetic_pretrain_dataset
        from acco_b200.models import PRESETS
        names = a.models.split(",")
        data = {}
        for name in names:
            V = PRESETS[name][1]["vocab_size"]
            data[name] = synthetic_pretrain_dataset(a.docs, 900, V, SEQ, eos_token_id=V - 1, seed=0)
        for name in ([] if a.skip_e2e else names):
            for r in range(a.repeats):
                for masked in (False, True):
                    res = run_e2e(name, masked, data[name], a.warmup, a.micro)
                    res["repeat"] = r
                    report["e2e"].append(res)
                    print(json.dumps(res), flush=True)
        for name in names:
            kw = PRESETS[name][1]
            B, Hq, Hk = SHAPES[name], kw["num_attention_heads"], kw["num_key_value_heads"]
            cases, n_seg = attention_cases(data[name], kw["vocab_size"] - 1, B, SEQ, Hq, Hk)
            times = {k: [] for k in cases}
            for _ in range(a.repeats):
                for k, f in cases.items():
                    times[k].append(timed(f))
            for k, ts in times.items():
                res = {"model": name, "shape": [B, SEQ, Hq, Hk], "segments_per_row": n_seg, "variant": k, "fwd_bwd_ms": ts,
                       "median_ms": statistics.median(ts)}
                report["attention"].append(res)
                print(json.dumps(res), flush=True)
    finally:
        os.chdir(cwd)
    from acco_b200.launch import shutdown_distributed
    shutdown_distributed()
    c = report["card"]
    print(f"\n{c['name']}, power limit {c.get('power_limit')}, max SM clock {c.get('max_sm_clock')}")
    print("| model | B x S | document_mask | tokens/s (median) | ms / micro-batch | runs |\n|---|---|---|---|---|---|")
    for name in sorted({e["model"] for e in report["e2e"]}):
        for masked in (False, True):
            rs = [e for e in report["e2e"] if e["model"] == name and e["document_mask"] == masked]
            tps = [e["tokens_per_s"] for e in rs]
            print(f"| {name} | {rs[0]['batch']} x {rs[0]['seq']} | {masked} | {statistics.median(tps):,.0f} | "
                  f"{statistics.median(e['ms_per_micro_batch'] for e in rs):.2f} | {', '.join(f'{x:,.0f}' for x in tps)} |")
    print("\n| model | B, S, Hq, Hk | segments / row | attention fwd+bwd per layer | median ms | runs |\n|---|---|---|---|---|---|")
    for e in report["attention"]:
        print(f"| {e['model']} | {e['shape']} | {e['segments_per_row']:.2f} | {e['variant']} | {e['median_ms']:.3f} | "
              f"{', '.join(f'{x:.3f}' for x in e['fwd_bwd_ms'])} |")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "doc_mask_bench.json"), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
