#!/usr/bin/env python
"""Per-GPU memory plan of a training configuration (no GPU needed):

    python tools/memory_plan.py --model llama3-1b --gpus 8 --batch 4 --seq 512

Persistent buffers are exact (they follow the arena / optimizer layout: two bf16 parameter sets, two bf16 gradient accumulators and
the fp32 optimizer shard); activations are an estimate of what the native Llama keeps for backward (bf16 tensors saved by the
fused ops + the padded logits).  Budget: an 80 GB H100, of which 92 % is planned."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from acco_b200.models import PRESETS, LlamaConfig
from acco_b200.parallel.arena import ShardLayout

GB = 1e9


def plan(cfg: LlamaConfig, world: int, batch: int, seq: int, method: str = "acco", align: int = 1024) -> dict:
    n = cfg.num_parameters(padded=True)
    lay = ShardLayout(n, world, align)
    two = 2                                                    # bf16
    buffers = {
        "theta x2 (live + shadow parameters, bf16)": 2 * lay.padded * two,
        "gradient accumulators x2 (bf16)": 2 * lay.padded * two,
        "optimizer shard: master, exp_avg, exp_avg_sq, stash (fp32)": 4 * lay.size_slice * 4,
    }
    if method == "ddp":
        buffers["gradient accumulators x2 (bf16)"] = lay.padded * two       # one accumulator is enough without overlap
    T = batch * seq
    H, I, L = cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers
    D, Hq, Hk = cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads
    per_layer = T * two * (
        2 * H                      # inputs of the two add+RMSNorm ops (h)
        + 2 * H                    # normalised activations fed to the qkv / gate|up GEMMs
        + (Hq + 2 * Hk) * D        # rotated qkv (attention backward)
        + Hq * D                   # attention output (o_proj input) 
        + 2 * I                    # gate|up (SwiGLU backward)
        + I                        # SwiGLU output (down_proj input)
    ) + T * 4 * (2 + Hq)           # rstd x2, attention LSE
    acts = L * per_layer + T * two * H + T * two * cfg.padded_vocab          # final norm input + logits (turned into dlogits in place)
    buffers["activations kept for backward (estimate, one micro-batch)"] = acts
    total = sum(buffers.values())
    return {"parameters": n, "size_slice": lay.size_slice, "buffers_gb": {k: v / GB for k, v in buffers.items()}, "total_gb": total / GB,
            "fits_80gb": total < 0.92 * 80e9}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama3-1b", choices=[k for k, (a, _) in PRESETS.items() if a == "llama"])
    ap.add_argument("--gpus", type=int, default=8)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--method", default="acco", choices=["acco", "dpu", "ddp"])
    a = ap.parse_args(argv)
    cfg = LlamaConfig.from_dict(PRESETS[a.model][1])
    out = plan(cfg, a.gpus, a.batch, a.seq, a.method)
    print(json.dumps({"model": a.model, "gpus": a.gpus, "batch": a.batch, "seq": a.seq, **out}, indent=1))
    return out


if __name__ == "__main__":
    main()
