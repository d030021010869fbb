"""Global gradient-norm clipping (train key ``max_grad_norm``) on the CPU / gloo path: the formula (`optim.clip_scale`) against
``torch.nn.utils.clip_grad_norm_``, validation, ACCO stash semantics, trainer equivalence in fp32, logging, 2- and 3-rank gloo runs."""
import json
import math
import os
import sys
import tempfile

import pytest
import torch
import torch.multiprocessing as mp

from acco_b200 import DecoupledTrainer, ops
from acco_b200.callbacks import TrainerCallback
from acco_b200.data import synthetic_pretrain_dataset
from acco_b200.launch import DistEnv
from acco_b200.optim import check_max_grad_norm, clip_scale
from acco_b200.parallel.schedule import COMMIT_ALL, COMMIT_NONE, RoundPlan

from helpers import LOG, base_args, tiny_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _cpu_path(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)


def make(method="acco", model=None, ds=None, **kw):
    ds = ds if ds is not None else synthetic_pretrain_dataset(200, 30, 96, 16, seed=3)
    return DecoupledTrainer(model=model or tiny_model(), train_dataset=ds, args=base_args(method_name=method, **kw), log=LOG,
                            env=DistEnv(id_run="clip"))


# ---------------------------------------------------------------------------------------------------------- formula
@pytest.mark.parametrize("max_norm", [1e-3, 0.7, 1e6, math.inf])
def test_clip_scale_matches_clip_grad_norm(max_norm):
    g = torch.Generator().manual_seed(0)
    grad_sum = [torch.randn(37, generator=g) * 3, torch.randn(5, 8, generator=g)]   # a sum over 4 micro-batches
    inv = 0.25
    params = [torch.nn.Parameter(torch.zeros_like(s)) for s in grad_sum]
    for p, s in zip(params, grad_sum):
        p.grad = s * inv
    ref_norm = torch.nn.utils.clip_grad_norm_(params, max_norm)
    sumsq = sum(float((s.double() ** 2).sum()) for s in grad_sum)
    norm, inv_eff = clip_scale(torch.tensor([sumsq], dtype=torch.float32), torch.tensor([inv]), max_norm)
    torch.testing.assert_close(norm, ref_norm.reshape(1), rtol=1e-6, atol=0)
    for p, s in zip(params, grad_sum):
        torch.testing.assert_close(s * inv_eff, p.grad, rtol=1e-6, atol=1e-12)
    if max_norm >= float(ref_norm):
        assert float(inv_eff) == inv                                        # coefficient exactly 1: the unclipped update
    else:
        clipped = math.sqrt(sum(float(((s * inv_eff).double() ** 2).sum()) for s in grad_sum))
        assert clipped == pytest.approx(max_norm, rel=1e-5)


def test_clip_scale_propagates_a_nan_norm_like_torch():
    norm, inv_eff = clip_scale(torch.tensor([float("nan")]), 0.5, 1.0)
    assert math.isnan(float(norm)) and math.isnan(float(inv_eff))


@pytest.mark.parametrize("bad", [0, -1.0, float("nan"), "1.0", True, [1.0]])
def test_bad_max_grad_norm_is_rejected(workdir, bad):
    with pytest.raises(ValueError, match="max_grad_norm"):
        check_max_grad_norm(bad)
    with pytest.raises(ValueError, match="max_grad_norm"):
        make("acco", max_grad_norm=bad)


def test_good_max_grad_norm_values():
    assert check_max_grad_norm(None) is None
    assert check_max_grad_norm(1) == 1.0
    assert check_max_grad_norm(math.inf) == math.inf


# ---------------------------------------------------------------------------------------------------------- ACCO stash
def test_real_round_clips_the_norm_of_both_halves_and_the_stash_stays_unclipped(workdir):
    t = make("acco", max_grad_norm=1e-3, nb_steps_tot=10 ** 6)
    be, arena, opt = t.backend, t.arena, t.sharded_optimizer
    S = arena.layout.size_slice
    g = torch.Generator().manual_seed(1)
    a0, a1 = torch.randn(S, generator=g), torch.randn(S, generator=g) * 2
    master0 = opt.master.clone()
    tent = RoundPlan(index=0, kind="tentative", read_acc=0, write_theta=1, commit=COMMIT_NONE, add_stash=False, write_stash=True,
                     lr_step=False, counts_toward_total=False, blocking=False)
    real = RoundPlan(index=1, kind="real", read_acc=1, write_theta=0, commit=COMMIT_ALL, add_stash=True, write_stash=False,
                     lr_step=True, counts_toward_total=True, blocking=False)
    arena.acc[0][:S].copy_(a0)
    be.launch_round(tent, 1e-2, 3)
    assert be.finish_round(tent) == 3
    assert be.last_grad_norm == pytest.approx(float((a0.double() / 3).norm()), rel=1e-5)
    assert torch.equal(opt.stash, a0)                                  # the unclipped half-batch sum
    assert torch.equal(opt.master, master0)                            # tentative: nothing committed
    arena.acc[1][:S].copy_(a1)
    be.launch_round(real, 1e-2, 2)
    assert be.finish_round(real) == 5
    full = (a0.double() + a1.double()) / 5
    assert be.last_grad_norm == pytest.approx(float(full.norm()), rel=1e-5)


# ---------------------------------------------------------------------------------------------------------- trainer equivalence
def test_ddp_with_clipping_equals_a_plain_torch_loop(workdir):
    """Native sharded DDP with clipping == ``DDP`` + ``clip_grad_norm_`` + ``torch.optim.AdamW`` (ddp_impl="torch") on the same
    batches, in fp32; the threshold is low enough that clipping binds at every step."""
    kw = dict(nb_steps_tot=12, learning_rate=1e-2, weight_decay=0.1, max_grad_norm=0.05, tensorboard=False, log_every=1)
    tn = make("ddp", model=tiny_model(seed=4), **kw)
    tt = make("ddp", model=tiny_model(seed=4), ddp_impl="torch", **kw)
    norms_n, norms_t = [], []
    tn.add_callback(_NormRecorder(norms_n))
    tt.add_callback(_NormRecorder(norms_t))
    tn.train()
    tt.train()
    assert len(norms_n) == len(norms_t) >= 6
    assert all(n > 0.05 * 1.5 for n in norms_n)                        # clipping binds
    torch.testing.assert_close(torch.tensor(norms_n), torch.tensor(norms_t), rtol=1e-4, atol=0)
    for pn, pt in zip(tn.model.parameters(), tt.model.parameters()):
        torch.testing.assert_close(pn.detach(), pt.detach(), rtol=1e-4, atol=1e-5)


class _NormRecorder(TrainerCallback):
    def __init__(self, out):
        self.out = out

    def on_log(self, trainer, logs):
        self.out.append(logs["grad_norm"])


def test_acco_with_clipping_equals_large_batch_ddp_when_estimate_is_exact(workdir):
    """The construction of test_acco_equals_large_batch_ddp_when_estimate_is_exact, with clipping binding: a real ACCO round clips
    the norm of (g~ + g) / count, as one DDP step over both micro-batches does."""
    class Lin(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.linspace(-1, 1, 10))

        def forward(self, input_ids=None, labels=None, **kw):
            x = input_ids.float().mean(0)[:10] / 50.0
            return ((self.w * x).sum(),)

    ds = synthetic_pretrain_dataset(100, 30, 96, 16, seed=5)
    ta = make("acco", model=Lin(), ds=ds, nb_steps_tot=8, learning_rate=1e-1, weight_decay=0.1, max_grad_norm=0.1)
    td = make("ddp", model=Lin(), ds=ds, nb_steps_tot=8, learning_rate=1e-1, weight_decay=0.1, n_grad_accumulation=2, max_grad_norm=0.1)
    ta.train()
    td.train()
    assert ta.sched.opt_steps == td.sched.opt_steps == 4
    assert td._grad_norm > 0.1 * 2                                     # clipping binds
    assert ta._grad_norm == td._grad_norm
    assert torch.equal(ta.sharded_optimizer.master, td.sharded_optimizer.master)
    assert torch.equal(ta.model.w.detach(), td.model.w.detach())


# ---------------------------------------------------------------------------------------------------------- logging
def _scalar_tags(workdir):
    tags = set()
    for root, _, files in os.walk(workdir / "tensorboard"):
        if "scalars.jsonl" in files:
            for line in open(os.path.join(root, "scalars.jsonl")):
                tags.add(json.loads(line).get("tag"))
    return tags


def test_default_off_logs_no_grad_norm_and_launches_no_norm_pass(workdir):
    ops.reset_launch_counts()
    logs = []
    t = make("acco", nb_steps_tot=8, tensorboard=True, log_every=1)
    t.add_callback(_LogRecorder(logs))
    t.train()
    assert logs and all("grad_norm" not in d for d in logs)
    assert "grad_norm" not in _scalar_tags(workdir)
    assert t.backend.last_grad_norm is None
    assert "round_norm" not in ops.launch_counts()


def test_grad_norm_is_logged_when_set(workdir, caplog):
    logs = []
    t = make("dpu", nb_steps_tot=8, tensorboard=True, log_every=1, max_grad_norm=math.inf)
    t.add_callback(_LogRecorder(logs))
    with caplog.at_level("INFO", logger=LOG.name):
        t.train()
    assert logs and all(d["grad_norm"] > 0 for d in logs)
    assert "grad_norm" in _scalar_tags(workdir)
    assert "grad_norm" in caplog.text


class _LogRecorder(_NormRecorder):
    def on_log(self, trainer, logs):
        self.out.append(dict(logs))


# ---------------------------------------------------------------------------------------------------------- gloo ranks
def _worker(rank, world, port, tmp, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(CUDA_VISIBLE_DEVICES="", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    os.chdir(tmp)
    torch.set_num_threads(1)
    import torch.distributed as dist
    from acco_b200 import DecoupledTrainer
    from acco_b200.data import synthetic_pretrain_dataset
    from acco_b200.launch import shutdown_distributed
    from helpers import LOG, base_args, tiny_model
    ds = synthetic_pretrain_dataset(300, 30, 96, 16, seed=7)
    out = {}
    for method in ("acco", "dpu", "ddp"):
        t = DecoupledTrainer(model=tiny_model(seed=0, hidden=40), train_dataset=ds,
                             args=base_args(method_name=method, nb_steps_tot=24, learning_rate=5e-3, batch_size=2, max_grad_norm=0.05), log=LOG)
        be = t.backend
        launch, finish = be.launch_round, be.finish_round
        expected, got, stash = [], [], [None]

        def launch_round(plan, lr, local_count, launch=launch, expected=expected, stash=stash, t=t):
            # oracle: the norm of the full averaged gradient, in fp64, from every rank's whole accumulator
            acc = t.arena.acc[plan.read_acc].double().clone()
            cnt = torch.tensor([float(local_count)], dtype=torch.float64)
            dist.all_reduce(acc)
            dist.all_reduce(cnt)
            if plan.add_stash:
                acc, cnt = acc + stash[0][0], cnt + stash[0][1]
            if plan.write_stash:
                stash[0] = (acc, cnt)
            expected.append(float((acc / cnt).norm()))
            launch(plan, lr, local_count)

        def finish_round(plan, finish=finish, got=got, be=be):
            total = finish(plan)
            got.append(be.last_grad_norm)
            return total

        be.launch_round, be.finish_round = launch_round, finish_round
        t.train()
        flat = torch.cat([p.detach().reshape(-1).double() for p in t.model.parameters()])
        out[method] = (float(flat.sum()), expected, got, t.size_slice, t.len_params)
    q.put((rank, out))
    shutdown_distributed()


@pytest.mark.parametrize("world", [2, 3])
def test_multi_rank_gloo_clipping(world):
    from acco_b200.launch import free_port
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    with tempfile.TemporaryDirectory() as tmp:
        procs = [ctx.Process(target=_worker, args=(r, world, port, tmp, q)) for r in range(world)]
        for p in procs:
            p.start()
        res = dict(q.get(timeout=300) for _ in procs)
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    for method in ("acco", "dpu", "ddp"):
        sums = {res[r][method][0] for r in range(world)}
        assert len(sums) == 1, (method, sums)                          # identical parameters on every rank
        expected, got = res[0][method][1], res[0][method][2]
        assert len(got) == len(expected) >= 4
        for r in range(1, world):
            assert res[r][method][2] == got                            # every rank logs the same norm
        for e, g in zip(expected, got):
            assert g == pytest.approx(e, rel=1e-5), method
        assert min(got) > 0.05 * 1.5, method                           # clipping binds
    if world == 3:
        sl, n = res[0]["acco"][3], res[0]["acco"][4]
        assert n % 3 != 0 and sl * 3 >= n                              # ragged last slice
