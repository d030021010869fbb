#!/usr/bin/env python
"""End-to-end check of the fused all-gather + GEMM training path (train.fused_ag_gemm=True) on >= 2 GPUs:
same seed / data with the flag off and on must give the same loss trajectory (up to GEMM rounding) and
bit-identical parameters on all ranks after `_ensure_gathered()`.

    torchrun --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29515 tools/fused_ag_check.py"""
import json
import logging
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.distributed as dist

from acco_b200 import AttrDict, DecoupledTrainer
from acco_b200.data import TokenDataset
from acco_b200.launch import discover_env, init_distributed
from acco_b200.models import LlamaConfig, LlamaForCausalLM


def run(fused: bool, env, steps: int, graphs: bool):
    torch.manual_seed(0)
    cfg = LlamaConfig(vocab_size=4096, hidden_size=768, intermediate_size=2048, num_hidden_layers=3, num_attention_heads=12,
                      num_key_value_heads=4, max_position_embeddings=256, tie_word_embeddings=False)
    model = LlamaForCausalLM(cfg)
    g = torch.Generator().manual_seed(3)
    ds = TokenDataset({"input_ids": torch.randint(0, 4096, (64 * 8 * env.world_size, 256), generator=g)})
    args = AttrDict(method_name="acco", batch_size=8, max_length=256, nb_steps_tot=10 ** 9, warmup=2, learning_rate=1e-3, save=False,
                    tensorboard=False, cuda_graphs=graphs, seed=11, fused_ag_gemm=fused, comm_backend="symm", log_every=10 ** 9)
    log = logging.getLogger("fa")
    log.setLevel(logging.ERROR)
    t = DecoupledTrainer(model=model, train_dataset=ds, args=args, log=log)
    losses = []
    for _ in range(steps):
        t.step()
        losses.append(float(t.loss_host))
    t._drain()
    flat = t.params.detach().clone()
    chk = flat.view(torch.int16).to(torch.int64).sum().reshape(1)
    lo, hi = chk.clone(), chk.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    bad = []
    for name, (off, n) in t.arena.param_slices().items():
        c = flat[off:off + n].view(torch.int16).to(torch.int64).sum().reshape(1)
        a, b = c.clone(), c.clone()
        dist.all_reduce(a, op=dist.ReduceOp.MIN)
        dist.all_reduce(b, op=dist.ReduceOp.MAX)
        if int((b - a).item()) != 0:
            # where inside the tensor?
            full = [torch.empty_like(flat[off:off + n]) for _ in range(env.world_size)]
            dist.all_gather(full, flat[off:off + n].contiguous())
            diff = (full[0].float() - full[1].float()).abs() > 0
            idx = diff.nonzero().flatten()
            bad.append({"name": name, "offset": off, "numel": n, "n_diff": int(diff.sum()), "first": int(idx[0]) if idx.numel() else -1,
                        "last": int(idx[-1]) if idx.numel() else -1, "size_slice": t.size_slice})
    info = {"losses": losses, "rank_divergence": int((hi - lo).item()), "backend": t.backend.name, "bad": bad[:8],
            "fused": getattr(t, "stats_fused_ag", None), "launches": dict(__import__("acco_b200").ops.launch_counts())}
    if t._feeder is not None:
        t._feeder.close()
    return info, flat


def main():
    env = init_distributed(discover_env())
    os.chdir(tempfile.mkdtemp())
    steps = 14
    report = {"world": env.world_size}
    ok = True
    for graphs in (False, True):
        base, p0 = run(False, env, steps, graphs)
        fused, p1 = run(True, env, steps, graphs)
        dl = max(abs(a - b) for a, b in zip(base["losses"], fused["losses"]))
        dp = float((p0.float() - p1.float()).abs().max())
        good = (dl < 5e-2 and fused["rank_divergence"] == 0 and base["rank_divergence"] == 0 and dp < 2e-2
                and fused["launches"].get("gemm_gather", 0) > 0 and fused["losses"][-1] < fused["losses"][0])
        ok = ok and good
        report["graphs" if graphs else "eager"] = {"max_loss_diff": dl, "max_param_diff": dp, "ok": good, "losses_base": base["losses"][-3:],
                                                   "losses_fused": fused["losses"][-3:], "fused": fused["fused"], "backend": fused["backend"],
                                                   "gather_gemm_launches": fused["launches"].get("gemm_gather", 0),
                                                   "rank_divergence": fused["rank_divergence"], "base_rank_divergence": base["rank_divergence"], "bad": fused["bad"]}
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    report["ok"] = bool(flag.item())
    if env.rank == 0:
        print(json.dumps(report, indent=1))
        out = os.path.join(ROOT, "results", "fused_ag_check.json")
        os.makedirs(os.path.dirname(out), exist_ok=True)
        json.dump(report, open(out, "w"), indent=1)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if report["ok"] else 1)


if __name__ == "__main__":
    main()
