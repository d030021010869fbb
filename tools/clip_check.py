#!/usr/bin/env python
"""Multi-GPU check of gradient-norm clipping (run under torchrun, one rank per GPU): for each transport - the fused round over NVLS
multicast, over P2P loads/stores, and the NCCL path - train a tiny Llama for a few ACCO rounds with a binding ``max_grad_norm`` and
check that

* the logged norm of every round is bit-identical on every rank;
* it agrees with an fp64 oracle: the norm of the all-reduced fp64 copy of every rank's bf16 accumulator (+ the stash);
* the parameters are bit-identical on every rank at the end.

    torchrun --nproc-per-node=N tools/clip_check.py"""
import logging
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(transport, rank, world, dev):
    import torch
    import torch.distributed as dist
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import synthetic_pretrain_dataset
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    if transport.startswith("symm-"):
        os.environ["ACCO_SYMM_MODE"] = transport[len("symm-"):]
    torch.manual_seed(0)
    cfg = LlamaConfig(vocab_size=1000, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4, max_position_embeddings=128)
    ds = synthetic_pretrain_dataset(512, 100, 1000, 128, seed=0)
    args = AttrDict(method_name="acco", batch_size=4, n_grad_accumulation=1, max_length=128, nb_steps_tot=12 * world, warmup=0,
                    learning_rate=1e-3, save=False, tensorboard=False, use_mixed_precision=True, static_accumulation=True,
                    comm_backend="nccl" if transport == "nccl" else "symm", max_grad_norm=0.05, seed=1)
    t = DecoupledTrainer(model=LlamaForCausalLM(cfg), train_dataset=ds, args=args, log=logging.getLogger("clip_check"))
    be = t.backend
    if be.name != transport:
        return {"available": False, "backend": be.name}
    launch, finish = be.launch_round, be.finish_round
    expected, got, stash = [], [], [None]

    def launch_round(plan, lr, local_count):
        s = t.arena.acc[plan.read_acc].double()
        cnt = torch.tensor([float(local_count)], dtype=torch.float64, device=dev)
        dist.all_reduce(s)
        dist.all_reduce(cnt)
        if plan.add_stash:
            s, cnt = s + stash[0][0], cnt + stash[0][1]
        if plan.write_stash:
            stash[0] = (s, cnt)
        expected.append(float((s / cnt).norm()))
        launch(plan, lr, local_count)

    def finish_round(plan):
        total = finish(plan)
        got.append(be.last_grad_norm)
        return total

    be.launch_round, be.finish_round = launch_round, finish_round
    t.train()
    norms = torch.tensor(got, dtype=torch.float64, device=dev)
    allg = [torch.empty_like(norms) for _ in range(world)]
    dist.all_gather(allg, norms)
    flat = t.arena.params_flat.float()
    pg = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(pg, flat)
    same_norm = all(torch.equal(x, allg[0]) for x in allg)
    same_params = all(torch.equal(x, pg[0]) for x in pg)
    worst = max(abs(g - e) / e for g, e in zip(got, expected))
    ok = same_norm and same_params and worst < 1e-3 and len(got) >= 4 and min(got) > 0.05
    return {"available": True, "ok": ok, "rounds": len(got), "same_norm_on_all_ranks": same_norm, "same_params_on_all_ranks": same_params,
            "max_rel_err_vs_fp64": worst}


def main():
    import torch
    from acco_b200.launch import discover_env, init_distributed, shutdown_distributed
    env = init_distributed(discover_env())
    dev = torch.device("cuda", env.local_rank)
    torch.cuda.set_device(dev)
    cwd = os.getcwd()
    os.chdir(tempfile.mkdtemp(prefix="acco_clip_check_"))
    res = {}
    try:
        for transport in ("symm-multimem", "symm-p2p", "nccl"):
            res[transport] = run(transport, env.rank, env.world_size, dev)
            if env.rank == 0:
                print(transport, res[transport], flush=True)
    finally:
        os.chdir(cwd)
    shutdown_distributed()
    ran = [r for r in res.values() if r["available"]]
    if not ran or not all(r["ok"] for r in ran):
        sys.exit(1)


if __name__ == "__main__":
    main()
