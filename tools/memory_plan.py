#!/usr/bin/env python
"""Per-GPU memory plan of a training configuration (no GPU needed):

    python tools/memory_plan.py --model llama3-1b --gpus 8 --batch 4 --seq 512

Persistent buffers are exact (they follow the arena / optimizer layout: two bf16 parameter sets, two bf16 gradient accumulators and
the fp32 optimizer shard); activations are an estimate of what the native Llama keeps for backward (bf16 tensors saved by the
fused ops + the padded logits).  ``--fp8`` (train key ``fp8``): the block linears keep their GEMM inputs as FP8 copies, 1 byte per
element instead of 2.  ``--grad-accum-dtype fp32`` (train key ``grad_accum_dtype``): the two gradient accumulators are fp32.  Budget: an 80 GB H100, of which 92 % is planned."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from acco_b200.models import PRESETS, LlamaConfig
from acco_b200.parallel.arena import ShardLayout

GB = 1e9


def plan(cfg: LlamaConfig, world: int, batch: int, seq: int, method: str = "acco", align: int = 1024, fp8: bool = False,
         grad_accum_dtype=None) -> dict:
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
    if grad_accum_dtype == "fp32":
        buffers["gradient accumulators x2 (fp32)"] = buffers.pop("gradient accumulators x2 (bf16)") * 2
    T = batch * seq
    H, I, L = cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers
    D, Hq, Hk = cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads
    gemm_in = 1 if fp8 else two                                # FP8: the block GEMMs keep q(x)^T instead of x
    per_layer = T * two * (
        2 * H                      # inputs of the two add+RMSNorm ops (h)
        + (Hq + 2 * Hk) * D        # rotated qkv (attention backward)
        + 2 * I                    # gate|up (SwiGLU backward)
    ) + T * gemm_in * (
        2 * H                      # normalised activations fed to the qkv / gate|up GEMMs
        + Hq * D                   # attention output (o_proj input)
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
    ap.add_argument("--fp8", action="store_true", help="train.fp8: FP8 copies of the block GEMM inputs are kept for backward")
    ap.add_argument("--grad-accum-dtype", dest="grad_accum_dtype", default=None, choices=["fp32"],
                    help="train.grad_accum_dtype: fp32 gradient accumulators")
    a = ap.parse_args(argv)
    cfg = LlamaConfig.from_dict(PRESETS[a.model][1])
    out = plan(cfg, a.gpus, a.batch, a.seq, a.method, fp8=a.fp8, grad_accum_dtype=a.grad_accum_dtype)
    head = {"model": a.model, "gpus": a.gpus, "batch": a.batch, "seq": a.seq, "fp8": a.fp8}
    if a.grad_accum_dtype:
        head["grad_accum_dtype"] = a.grad_accum_dtype
    print(json.dumps({**head, **out}, indent=1))
    return out


if __name__ == "__main__":
    main()
