"""Weight-decay exclusion of norm gains and biases (train key ``no_decay_1d``), CPU side: the range table of the flat vector, the
reference update with a table against ``torch.optim.AdamW`` with two parameter groups, and the trainer on the gloo path."""
import os
import sys
import tempfile

import pytest
import torch
import torch.multiprocessing as mp
import torch.nn as nn

from acco_b200 import DecoupledTrainer
from acco_b200.data import synthetic_pretrain_dataset
from acco_b200.launch import DistEnv
from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM
from acco_b200.optim import AdamHyper, ShardedAdamW, adamw_shard_update_, check_no_decay_ranges
from acco_b200.parallel.arena import FlatArena, ShardLayout
from acco_b200.parallel.schedule import COMMIT_ALL, COMMIT_NONE, COMMIT_PARAM, COMMIT_STATE

from helpers import LOG, base_args, tiny_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HP = dict(lr=3e-2, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1)


class Toy(nn.Module):
    """1-D parameters of 1, 3, 7 and 13 elements: first, back to back in the middle, and last.  40 elements, no-decay ranges
    [0, 1), [13, 23), [27, 40): the 2-rank slice boundary (20) and both 3-rank ones (14, 28) cut through a range.  The loss is
    linear with fixed coefficients, so the gradient depends on neither the weights nor the batch."""

    def __init__(self, seed=0):
        super().__init__()
        gen = torch.Generator().manual_seed(seed)
        shapes = dict(b0=(1,), w1=(4, 3), g1=(3,), g2=(7,), w2=(2, 2), b3=(13,))
        for name, shape in shapes.items():
            setattr(self, name, nn.Parameter(torch.randn(shape, generator=gen)))
            self.register_buffer("c_" + name, torch.randn(shape, generator=gen))

    def forward(self, input_ids=None, labels=None, **kw):
        return (sum((p * getattr(self, "c_" + n)).sum() for n, p in self.named_parameters()),)


TOY_RANGES = [(0, 1), (13, 23), (27, 40)]


def ranges_of(model):
    return FlatArena(model, 1, 0, torch.float32, "cpu").no_decay_ranges()


def check_table(model, ranges):
    """Sorted, disjoint, merged, and exactly the elements of the trainable ndim <= 1 parameters."""
    assert check_no_decay_ranges(ranges) == tuple(ranges)
    assert all(a[1] < b[0] for a, b in zip(ranges, ranges[1:]))          # touching ranges would not be merged
    arena = FlatArena(model, 1, 0, torch.float32, "cpu")
    want = torch.zeros(arena.numel, dtype=torch.bool)
    for p, o, n in zip(arena.params, arena.offsets, arena.numels):
        if p.ndim <= 1 and p.requires_grad:
            want[o:o + n] = True
    got = torch.zeros(arena.numel, dtype=torch.bool)
    for lo, hi in ranges:
        got[lo:hi] = True
    assert torch.equal(got, want)


# ------------------------------------------------------------------ range table
def test_toy_ranges_are_merged_and_exact():
    r = ranges_of(Toy())
    assert r == TOY_RANGES
    check_table(Toy(), r)


@pytest.mark.parametrize("tied", [False, True])
def test_llama_ranges(tied):
    m = LlamaForCausalLM(LlamaConfig(vocab_size=96, hidden_size=32, intermediate_size=48, num_hidden_layers=3, num_attention_heads=4,
                                     num_key_value_heads=2, max_position_embeddings=32, tie_word_embeddings=tied))
    r = ranges_of(m)
    check_table(m, r)
    assert len(r) == 2 * 3 + 1                       # two norms per block, never adjacent, and the final norm
    assert sum(hi - lo for lo, hi in r) == 7 * 32


def test_gpt_neo_ranges_merge_runs_of_1d_parameters():
    m = GPTForCausalLM(GPTConfig(vocab_size=96, hidden_size=32, num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=32))
    r = ranges_of(m)
    check_table(m, r)
    n_1d = sum(1 for p in m.parameters() if p.ndim <= 1)
    assert len(r) < n_1d                              # LayerNorm weight + bias (and a bias next to them) share a range


def test_frozen_1d_parameters_stay_out_and_table_ignores_world_size():
    m = Toy()
    m.g2.requires_grad_(False)
    assert ranges_of(m) == [(0, 1), (13, 16), (27, 40)]
    full = ranges_of(Toy())
    for world in (2, 3):
        assert FlatArena(Toy(), world, world - 1, torch.float32, "cpu").no_decay_ranges() == full


@pytest.mark.parametrize("bad", [[(3, 3)], [(5, 2)], [(0, 4), (3, 6)], [(8, 9), (0, 1)], [(-1, 2)]])
def test_malformed_tables_are_rejected(bad):
    with pytest.raises(ValueError):
        check_no_decay_ranges(bad)


def test_empty_table_is_none():
    assert check_no_decay_ranges(None) is None and check_no_decay_ranges([]) is None


# ------------------------------------------------------------------ reference update
def adamw_groups(p0, ranges, dtype):
    """torch.optim.AdamW over the flat vector cut into one tensor per segment, no-decay segments in a group of their own."""
    cuts = sorted({0, p0.numel()} | {x for r in ranges for x in r})
    segs = [(a, b, any(lo <= a and b <= hi for lo, hi in ranges)) for a, b in zip(cuts, cuts[1:])]
    ps = [p0[a:b].to(dtype).clone().requires_grad_(True) for a, b, _ in segs]
    opt = torch.optim.AdamW([dict(params=[p for p, s in zip(ps, segs) if not s[2]]),
                             dict(params=[p for p, s in zip(ps, segs) if s[2]], weight_decay=0.0)],
                            lr=HP["lr"], betas=(HP["beta1"], HP["beta2"]), eps=HP["eps"], weight_decay=HP["weight_decay"])
    return ps, segs, opt


@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_sharded_update_with_table_equals_adamw_with_two_groups(world, dtype):
    torch.manual_seed(world)
    N = 40
    lay = ShardLayout(N, world)
    S = lay.size_slice
    p0 = torch.randn(lay.padded)
    p0[N:] = 0
    ps, segs, opt = adamw_groups(p0[:N], TOY_RANGES, dtype)
    shards = [ShardedAdamW(p0[r * S:(r + 1) * S], no_decay=TOY_RANGES, shard_base=r * S, **{k: HP[k] for k in ("lr", "eps", "weight_decay")},
                           betas=(HP["beta1"], HP["beta2"])) for r in range(world)]
    outs = [torch.zeros(S) for _ in range(world)]
    for step in range(1, 6):
        g_half, g = torch.randn(lay.padded), torch.randn(lay.padded)
        g_half[N:], g[N:] = 0, 0
        for p, (a, b, _) in zip(ps, segs):
            p.grad = ((g_half + g) / 2)[a:b].to(dtype)
        opt.step()
        for r, o in enumerate(shards):
            sl = slice(r * S, (r + 1) * S)
            before = [t.clone() for t in (o.master, o.exp_avg, o.exp_avg_sq)]
            # tentative round: stash the half-batch sum, commit nothing; state-only and parameter-only commits leave the other half
            hp = AdamHyper(step=step, inv_count=1.0, commit=COMMIT_NONE, write_stash=True, no_decay=o.no_decay, shard_base=o.shard_base, **HP)
            adamw_shard_update_(g_half[sl], o.master, o.exp_avg, o.exp_avg_sq, o.stash, outs[r], hp)
            assert all(torch.equal(x, y) for x, y in zip(before, (o.master, o.exp_avg, o.exp_avg_sq)))
            for commit in (COMMIT_PARAM, COMMIT_STATE):
                trial = [t.clone() for t in (o.master, o.exp_avg, o.exp_avg_sq, o.stash)]
                hp = AdamHyper(step=step, inv_count=0.5, commit=commit, add_stash=True, no_decay=o.no_decay, shard_base=o.shard_base, **HP)
                adamw_shard_update_(g[sl], *trial, outs[r], hp)
                assert torch.equal(trial[0], before[0]) == (commit == COMMIT_STATE)
                assert torch.equal(trial[1], before[1]) == (commit == COMMIT_PARAM)
            # the real round, through ShardedAdamW.hyper
            plan = type("Plan", (), dict(commit=COMMIT_ALL, add_stash=True, write_stash=False))
            adamw_shard_update_(g[sl], o.master, o.exp_avg, o.exp_avg_sq, o.stash, outs[r], o.hyper(HP["lr"], plan, 0.5))
            o.after_launch(plan)
        got = torch.cat([o.master for o in shards])[:N]
        want = torch.cat([p.detach() for p in ps]).float()
        torch.testing.assert_close(got, want, rtol=2e-6, atol=2e-7)
        torch.testing.assert_close(torch.cat(outs)[:N], got, rtol=0, atol=0)


def test_update_without_table_is_bitwise_the_plain_update():
    torch.manual_seed(0)
    p0, g = torch.randn(64), torch.randn(64)
    res = []
    for no_decay in (None, [], ()):
        o = ShardedAdamW(p0, lr=HP["lr"], weight_decay=0.1, no_decay=no_decay, shard_base=7)
        out = torch.zeros(64)
        plan = type("Plan", (), dict(commit=COMMIT_ALL, add_stash=False, write_stash=False))
        adamw_shard_update_(g, o.master, o.exp_avg, o.exp_avg_sq, o.stash, out, o.hyper(HP["lr"], plan, 1.0))
        res.append(out)
    o = ShardedAdamW(p0, lr=HP["lr"], weight_decay=0.1)
    want = p0 * (1.0 - HP["lr"] * 0.1)
    hp = AdamHyper(lr=HP["lr"], weight_decay=0.1, step=1, inv_count=1.0)
    out = torch.zeros(64)
    adamw_shard_update_(g, o.master, o.exp_avg, o.exp_avg_sq, o.stash, out, hp)
    assert all(torch.equal(r, out) for r in res) and not torch.equal(out, want)


@pytest.mark.parametrize("base", [0, 5, 24])
def test_probe_excluded_elements_keep_their_bits_and_neighbours_halve(base):
    """lr * wd = 0.5, zero gradient, zero moments: an element inside a range keeps its value bit for bit, the element on either
    side of every range boundary halves.  An off-by-one at either end of a range fails."""
    S = 16
    ranges = [(0, 1), (6, 7), (9, 13), (26, 29), (39, 40)]
    p0 = torch.randn(S, generator=torch.Generator().manual_seed(1)) + 3.0
    out = torch.zeros(S)
    z = torch.zeros(S)
    hp = AdamHyper(lr=0.5, weight_decay=1.0, step=1, inv_count=1.0, commit=COMMIT_ALL, no_decay=ranges, shard_base=base)
    m = p0.clone()
    adamw_shard_update_(z, m, z.clone(), z.clone(), None, out, hp)
    for i in range(S):
        inside = any(lo <= base + i < hi for lo, hi in ranges)
        assert m[i].item() == (p0[i].item() if inside else 0.5 * p0[i].item()), (base, i, inside)
    assert torch.equal(out, m)


# ------------------------------------------------------------------ trainer
@pytest.fixture(autouse=True)
def _cpu_path(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)


def make(method, model, **kw):
    ds = synthetic_pretrain_dataset(200, 30, 96, 16, seed=3)
    args = base_args(method_name=method, learning_rate=HP["lr"], weight_decay=HP["weight_decay"], adam_beta1=HP["beta1"],
                     adam_beta2=HP["beta2"], **kw)
    return DecoupledTrainer(model=model, train_dataset=ds, args=args, log=LOG, env=DistEnv(id_run="nd"))


def toy_adamw(steps, no_decay=True):
    """`steps` AdamW steps on the toy's constant gradient, norm gains and biases in a weight_decay = 0 group."""
    m = Toy()
    excluded = [p for p in m.parameters() if p.ndim <= 1] if no_decay else []
    rest = [p for p in m.parameters() if not any(p is q for q in excluded)]
    opt = torch.optim.AdamW([dict(params=rest), dict(params=excluded, weight_decay=0.0)], lr=HP["lr"], betas=(HP["beta1"], HP["beta2"]),
                            eps=HP["eps"], weight_decay=HP["weight_decay"])
    for _ in range(steps):
        for n, p in m.named_parameters():
            p.grad = getattr(m, "c_" + n).clone()
        opt.step()
    return torch.cat([p.detach().reshape(-1) for p in m.parameters()])


@pytest.mark.parametrize("method", ["acco", "dpu", "ddp"])
def test_trainer_equals_adamw_with_groups(workdir, method):
    t = make(method, Toy(), nb_steps_tot=12, no_decay_1d=True)
    t.train()
    assert t.sharded_optimizer.no_decay == tuple(TOY_RANGES)
    steps = t.sharded_optimizer.step
    assert steps >= 5
    got = t.sharded_optimizer.master[:40]
    torch.testing.assert_close(got, toy_adamw(steps), rtol=2e-6, atol=2e-7)
    assert (got - toy_adamw(steps, no_decay=False)).abs().max() > 1e-3          # decaying everything is measurably different


def test_trainer_torch_ddp_builds_the_two_groups(workdir):
    t = make("ddp", Toy(), nb_steps_tot=6, no_decay_1d=True, ddp_impl="torch")
    t.train()
    groups = t.optimizer.param_groups
    assert [g["weight_decay"] for g in groups] == [HP["weight_decay"], 0.0]
    assert sorted(p.numel() for p in groups[1]["params"]) == [1, 3, 7, 13]
    flat = torch.cat([p.detach().reshape(-1) for p in t.model.parameters()])
    torch.testing.assert_close(flat, toy_adamw(6), rtol=2e-6, atol=2e-7)


@pytest.mark.parametrize("method", ["acco", "ddp"])
def test_key_false_is_bitwise_the_run_without_the_key(workdir, method):
    runs = []
    for kw in ({}, {"no_decay_1d": False}, {"no_decay_1d": True}):
        t = make(method, tiny_model(), nb_steps_tot=12, **kw)
        t.train()
        runs.append(t.sharded_optimizer.master.clone())
    assert torch.equal(runs[0], runs[1]) and not torch.equal(runs[0], runs[2])


@pytest.mark.parametrize("value", [1, 0, "true", None, 0.0])
def test_non_bool_values_are_rejected(workdir, value):
    with pytest.raises(ValueError, match="no_decay_1d"):
        make("acco", Toy(), no_decay_1d=value)


def test_start_up_log_line_counts_parameters_elements_and_ranges(workdir, caplog):
    import logging
    with caplog.at_level(logging.INFO, logger=LOG.name):
        make("acco", Toy(), no_decay_1d=True)
    assert any("no_decay_1d: 4 parameters (24 elements, 3 ranges" in r.getMessage() for r in caplog.records)


# ------------------------------------------------------------------ several ranks, elastic resume
def _worker(rank, world, port, tmp, phase, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(CUDA_VISIBLE_DEVICES="", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), ACCO_RUN_ID="nd")
    os.chdir(tmp)
    torch.set_num_threads(1)
    from acco_b200.launch import shutdown_distributed
    ds = synthetic_pretrain_dataset(300, 30, 96, 16, seed=7)
    ck = os.path.join(tmp, "checkpoints", "nd_ddp_model.pt")
    # synchronous rounds on the toy's constant gradient: the weights after k optimizer steps do not depend on the world size
    kw = dict(method_name="ddp", learning_rate=HP["lr"], weight_decay=HP["weight_decay"], adam_beta1=HP["beta1"], adam_beta2=HP["beta2"],
              no_decay_1d=True)
    if phase == "first":
        args = base_args(nb_steps_tot=6 * world, save=True, save_optimizer=True, **kw)
    else:
        args = base_args(nb_steps_tot=12 + 6 * world, save=False, resume_from=ck, **kw)
    t = DecoupledTrainer(model=Toy(), train_dataset=ds, args=args, log=LOG)
    t.train()
    flat = torch.cat([p.detach().reshape(-1) for p in t.model.parameters()])
    q.put((rank, t.sharded_optimizer.step, flat, t.sharded_optimizer.no_decay, t.sharded_optimizer.shard_base))
    shutdown_distributed()


def _spawn(world, tmp, phase):
    from acco_b200.launch import free_port
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, tmp, phase, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = sorted((q.get(timeout=240) for _ in procs), key=lambda o: o[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return out


def test_two_ranks_save_three_ranks_resume_matches_an_uninterrupted_run():
    with tempfile.TemporaryDirectory() as tmp:
        first = _spawn(2, tmp, "first")
        assert [o[1] for o in first] == [6, 6]
        assert all(torch.equal(o[2], first[0][2]) for o in first)               # identical parameters on every rank
        assert [o[4] for o in first] == [0, 20]                                  # the slices cut through [13, 23)
        torch.testing.assert_close(first[0][2], toy_adamw(6), rtol=2e-6, atol=2e-7)
        second = _spawn(3, tmp, "second")
        assert [o[1] for o in second] == [12, 12, 12]
        assert all(torch.equal(o[2], second[0][2]) for o in second)
        assert all(o[3] == tuple(TOY_RANGES) for o in first + second)           # the table does not depend on the world size
        assert [o[4] for o in second] == [0, 14, 28]
        torch.testing.assert_close(second[0][2], toy_adamw(12), rtol=2e-6, atol=2e-7)
