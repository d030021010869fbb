"""Weight-decay exclusion of norm gains and biases (train key ``no_decay_1d``) on the GPU: the local instantiation of the fused
AdamW round with a no-decay table against the reference update, the boundary probe bit for bit, the trainer against the fp32 CPU
trainer, and (2+ GPUs) the P2P and multimem rounds with a table that straddles the rank boundaries."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops
from acco_b200.optim import AdamHyper, ShardedAdamW, adamw_shard_update_
from acco_b200.parallel.schedule import COMMIT_ALL, COMMIT_NONE, COMMIT_STATE

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tables(S, base):
    """name -> ranges in global indices for a shard [base, base + S)."""
    every_offset = [(base + 64 * (k + 1) + k, base + 64 * (k + 1) + 9 + (3 * k) % 8) for k in range(8)]   # start at offset k of a vector, end at every offset
    singles = [(base + 8 * k + (k % 8), base + 8 * k + (k % 8) + 1) for k in range(100, 108)]
    sixty = [(base + 1000 + 97 * k, base + 1000 + 97 * k + 1 + (k * 7) % 23) for k in range(60)]
    return {
        "offsets": every_offset + singles,
        "edges": [(base, base + 1), (base + 3, base + 5), (base + 5, base + 6), (base + S - 1, base + S)],
        "whole": [(max(base - 11, 0), base + S + 5)],
        "outside": [(0, max(base - 1, 1))] if base > 8 else [(base + S + 3, base + S + 9)],
        "sixty": sixty,
    }


def run_pair(S, base, ranges, gdtype, odtype, commit, add, write, lr=1e-2, wd=0.1, zero=False):
    torch.manual_seed(3)
    p0 = torch.randn(S, device=DEV) + (3.0 if zero else 0.0)
    a, b = ShardedAdamW(p0, lr=lr), ShardedAdamW(p0, lr=lr)
    if not zero:
        for o in (a, b):
            o.exp_avg.copy_(torch.randn(S, device=DEV, generator=torch.Generator(DEV).manual_seed(5)) * 0.1)
            o.exp_avg_sq.copy_(torch.rand(S, device=DEV, generator=torch.Generator(DEV).manual_seed(6)) * 0.1)
            o.stash.copy_(torch.randn(S, device=DEV, generator=torch.Generator(DEV).manual_seed(7)))
    g = (torch.zeros(S, device=DEV) if zero else torch.randn(S, device=DEV)).to(gdtype)
    oa, ob = torch.zeros(S, device=DEV, dtype=odtype), torch.zeros(S, device=DEV, dtype=odtype)
    hp = AdamHyper(lr=lr, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=wd, step=3, inv_count=torch.tensor([0.25], device=DEV),
                   commit=commit, add_stash=add, write_stash=write, no_decay=ranges, shard_base=base)
    adamw_shard_update_(g, a.master, a.exp_avg, a.exp_avg_sq, a.stash, oa, hp)
    ops.fused_adamw_shard(g, b.master, b.exp_avg, b.exp_avg_sq, b.stash, ob, hp)
    return p0, a, b, oa, ob


def wrapping_size():
    """A shard the grid-stride loop of the local instantiation passes over more than once (4 vectors per thread and pass)."""
    C = ops.load_ext(required=True)
    return 8 * (4 * 512 * 4 * int(C.num_sms()) * 2 + 8 * 4099 + 3)


@pytest.mark.parametrize("gdtype,odtype", [(torch.bfloat16, torch.bfloat16), (torch.float32, torch.float32), (torch.float32, torch.bfloat16),
                                           (torch.bfloat16, torch.float32)])
@pytest.mark.parametrize("commit,add,write", [(COMMIT_ALL, False, False), (COMMIT_NONE, False, True), (COMMIT_ALL, True, False),
                                              (COMMIT_STATE, False, False)])
def test_fused_adamw_with_table_matches_reference(gdtype, odtype, commit, add, write):
    S, base = 8 * 4099, 8 * 517
    for name, ranges in tables(S, base).items():
        _, a, b, oa, ob = run_pair(S, base, sorted(ranges), gdtype, odtype, commit, add, write)
        for x, y in ((a.master, b.master), (a.exp_avg, b.exp_avg), (a.exp_avg_sq, b.exp_avg_sq), (a.stash, b.stash)):
            torch.testing.assert_close(y, x, rtol=1e-5, atol=1e-6, msg=lambda m: f"{name}: {m}")
        tol = (1e-2, 1e-2) if odtype == torch.bfloat16 else (1e-5, 1e-6)
        torch.testing.assert_close(ob.float(), oa.float(), rtol=tol[0], atol=tol[1], msg=lambda m: f"{name}: {m}")


@pytest.mark.parametrize("size", ["wraps", "tiny"])
def test_probe_is_bit_exact_at_every_boundary(size):
    """lr * wd = 0.5, zero gradient and moments: elements inside a range keep their bits, every other element halves, over a shard
    the grid-stride loop wraps on and one smaller than a CTA.  The ~80-range table puts boundaries at every offset of a vector, at
    the first and the last element of the shard and beyond its end."""
    base = 8 * 1000
    if size == "wraps":
        S = wrapping_size()
        tab = tables(S, base)
        ranges = sorted(tab["offsets"] + tab["sixty"] + [(base, base + 1), (base + S - 40, base + S - 33), (base + S - 1, base + S + 4)])
    else:
        S = 8 * 37
        ranges = [(base - 3, base + 1), (base + 6, base + 9), (base + 17, base + 18), (base + S - 1, base + S + 4)]
    p0, a, b, oa, ob = run_pair(S, base, ranges, torch.bfloat16, torch.float32, COMMIT_ALL, False, False, lr=0.5, wd=1.0, zero=True)
    inside = torch.zeros(S, dtype=torch.bool, device=DEV)
    for lo, hi in ranges:
        inside[max(lo - base, 0):max(min(hi - base, S), 0)] = True
    want = torch.where(inside, p0, 0.5 * p0)
    assert torch.equal(b.master, want) and torch.equal(ob, want) and torch.equal(a.master, want)
    assert 0 < int(inside.sum()) < S


def test_small_instantiation_with_table():
    """The 256-thread, 64-register local instantiation (ACCO_ROUND_LOCAL_SMALL=1) in a process of its own: the switch is read once."""
    code = f"""
import sys, torch
sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})
import test_no_decay_gpu as T
from acco_b200.parallel.schedule import COMMIT_ALL
S, base = 8 * 40999, 8 * 77
tab = T.tables(S, base)
ranges = sorted(tab["offsets"] + tab["edges"][:1] + tab["edges"][3:] + tab["sixty"])
p0, a, b, oa, ob = T.run_pair(S, base, ranges, torch.bfloat16, torch.float32, COMMIT_ALL, False, False, lr=0.5, wd=1.0, zero=True)
assert torch.equal(b.master, a.master) and torch.equal(ob, oa) and not torch.equal(b.master, 0.5 * p0)
_, a, b, oa, ob = T.run_pair(S, base, ranges, torch.bfloat16, torch.bfloat16, COMMIT_ALL, True, False)
torch.testing.assert_close(b.master, a.master, rtol=1e-5, atol=1e-6)
print("small ok")
"""
    env = dict(os.environ, ACCO_ROUND_LOCAL_SMALL="1")
    p = subprocess.run([sys.executable, "-c", code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert p.returncode == 0 and "small ok" in p.stdout, p.stdout[-3000:]


@pytest.mark.parametrize("table", ["none", "empty"])
def test_absent_table_is_bitwise_the_call_without_the_argument(table):
    C = ops.load_ext(required=True)
    S = 8 * 4099
    torch.manual_seed(0)
    p0, g = torch.randn(S, device=DEV), torch.randn(S, device=DEV).bfloat16()
    res = []
    for with_arg in (False, True):
        o = ShardedAdamW(p0, lr=1e-2)
        o.exp_avg.fill_(0.01)
        out = torch.zeros(S, device=DEV, dtype=torch.bfloat16)
        args = [g, o.master, o.exp_avg, o.exp_avg_sq, o.stash, out, torch.tensor([0.5], device=DEV), torch.zeros(4, dtype=torch.int32, device=DEV),
                1e-2, 0.9, 0.95, 1e-8, 0.1, 2, COMMIT_ALL, False, False]
        if with_arg:
            args += [None if table == "none" else torch.zeros(0, 2, dtype=torch.int64, device=DEV), 64]
        C.adamw_shard(*args)
        res.append((o.master.clone(), o.exp_avg.clone(), o.exp_avg_sq.clone(), out.clone()))
    assert all(torch.equal(x, y) for x, y in zip(*res))


def test_binding_rejects_malformed_tables():
    C = ops.load_ext(required=True)
    S = 64
    z = lambda: torch.zeros(S, device=DEV)
    base = [z().bfloat16(), z(), z(), z(), z(), z().bfloat16(), torch.ones(1, device=DEV), torch.zeros(4, dtype=torch.int32, device=DEV),
            1e-2, 0.9, 0.95, 1e-8, 0.1, 1, COMMIT_ALL, False, False]
    for bad in (torch.tensor([[0, 4]], dtype=torch.int64), torch.tensor([[0, 4]], dtype=torch.int32, device=DEV),
                torch.tensor([0, 4, 8], dtype=torch.int64, device=DEV)):
        with pytest.raises(RuntimeError, match="no_decay_ranges"):
            C.adamw_shard(*base, bad, 0)
    with pytest.raises(ValueError):
        ShardedAdamW(z(), lr=1e-2, no_decay=[(4, 8), (0, 2)])


_TRAINER_SCRIPT = r"""
import logging, sys, torch
sys.path.insert(0, {root!r})
from acco_b200 import AttrDict, DecoupledTrainer, ops
from acco_b200.data import synthetic_pretrain_dataset
from acco_b200.launch import discover_env
from acco_b200.models import LlamaConfig, LlamaForCausalLM
cuda, extra = sys.argv[1] == "cuda", sys.argv[3] == "compose"
cfg = LlamaConfig(vocab_size=512, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                  num_key_value_heads=2, max_position_embeddings=64)
torch.manual_seed(0)
m = LlamaForCausalLM(cfg)
init = {{k: v.detach().float().clone() for k, v in m.state_dict().items()}}
ds = synthetic_pretrain_dataset(400, 80, 512, 64, seed=3)
# weight_decay 5: twelve decayed steps would pull a norm gain from 1 to about 0.94, far outside bf16 training noise
args = AttrDict(method_name="acco", batch_size=4, max_length=64, nb_steps_tot=24, warmup=2, learning_rate=1e-3, save=False, tensorboard=False,
                seed=1, weight_decay=5.0, use_mixed_precision=cuda, no_decay_1d=sys.argv[4] == "on",
                max_grad_norm=1.0 if extra else None, fp8=bool(extra and cuda))
env = discover_env()
env.id_run = "nd"
t = DecoupledTrainer(model=m, train_dataset=ds, args=args, log=logging.getLogger("nd"), env=env)
t.train()
torch.save({{"init": init, "final": {{k: v.detach().float().cpu().clone() for k, v in t.model.state_dict().items()}},
            "counts": (t.sched.count_grad_tot, t.sched.opt_steps), "cuda": t.is_cuda, "graphs": t._graphs is not None,
            "launches": ops.launch_counts() if cuda else {{}}, "ranges": len(t.sharded_optimizer.no_decay or ())}}, sys.argv[2])
"""


def _train(tmp_path, dev, compose, key="on"):
    from acco_b200.launch import free_port
    script = tmp_path / "nd_train.py"
    script.write_text(_TRAINER_SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR")}
    env["MASTER_PORT"] = str(free_port())
    if dev == "cpu":
        env["CUDA_VISIBLE_DEVICES"] = ""
    out = tmp_path / f"{dev}_{compose}_{key}.pt"
    p = subprocess.run([sys.executable, str(script), dev, str(out), compose, key], cwd=tmp_path, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:]
    return torch.load(out, weights_only=False)


@pytest.mark.parametrize("compose", ["plain", "compose"])
def test_trainer_with_graphs_tracks_fp32_cpu_trainer(tmp_path, compose):
    """One GPU, CUDA graphs, bf16 (``compose``: with max_grad_norm = 1 and fp8 as well) against the fp32 CPU trainer with the same
    key: parameters within bf16 training noise, and the norm gains stay where a decayed run would have pulled them away from."""
    gpu, cpu = _train(tmp_path, "cuda", compose), _train(tmp_path, "cpu", compose)
    assert gpu["cuda"] and gpu["graphs"] and not cpu["cuda"]
    assert gpu["counts"] == cpu["counts"] and gpu["ranges"] == cpu["ranges"] == 5
    assert gpu["launches"].get("rs_adam_ag", 0) > 0
    for k, ref in cpu["final"].items():
        moved = (ref - cpu["init"][k]).norm()
        err = (gpu["final"][k] - ref).norm()
        assert float(err) <= (0.5 if compose == "compose" else 0.35) * float(moved) + 2e-2 * float(ref.norm()) + 1e-3, (k, float(err), float(moved))
    decayed = _train(tmp_path, "cpu", compose, key="off")
    for k, v in gpu["final"].items():
        if k.endswith("norm.weight"):
            assert float(v.mean()) > 0.985 and float(decayed["final"][k].mean()) < 0.97, (k, float(v.mean()))


@pytest.mark.multigpu
def test_p2p_and_multimem_rounds_with_a_table_across_rank_boundaries(tmp_path):
    """2+ GPUs: tools/symm_check.py --no-decay, every round of both transports against the exact oracle with the same table."""
    import json
    from acco_b200.launch import free_port
    n = min(torch.cuda.device_count(), 8)
    out = tmp_path / "symm_nd.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.join(ROOT, "tools", "symm_check.py"), "--no-decay", "--numel", "5000011",
           "--bench-numel", "8000000", "--bench-iters", "3", "--out", str(out)]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:]
    rep = json.load(open(out))
    assert rep["no_decay"] and any(v.get("available") and v.get("ok") for v in rep["modes"].values()), rep
