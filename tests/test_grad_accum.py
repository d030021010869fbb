"""fp32 gradient accumulators under bf16 weights (train key ``grad_accum_dtype``), CPU side: the key, the arena's ``main_grad`` binding,
the torch paths of every op that adds into the arena, and the ACCO / DPU / DDP trainers on gloo CPU ranks."""
import os
import sys
import tempfile

import pytest
import torch
import torch.multiprocessing as mp

from acco_b200 import DecoupledTrainer, TRAIN_DEFAULTS, ops
from acco_b200.data import synthetic_pretrain_dataset
from acco_b200.launch import DistEnv
from acco_b200.models import GPTConfig, GPTForCausalLM
from acco_b200.ops.fp8 import E4M3, E5M2, Fp8LinearFn, quantize_ref
from acco_b200.ops.linear import LinearFn
from acco_b200.parallel.arena import FlatArena

from helpers import LOG, base_args, tiny_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _cpu_path(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)


def _neo(seed=0):
    torch.manual_seed(seed)
    return GPTForCausalLM(GPTConfig(vocab_size=96, hidden_size=32, num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=32,
                                    attention_layers=["global", "local"], window_size=8, pad_vocab_multiple=8))


def make(model, **kw):
    ds = synthetic_pretrain_dataset(200, 30, 96, 16, seed=3)
    kw.setdefault("use_mixed_precision", True)
    return DecoupledTrainer(model=model, train_dataset=ds, args=base_args(**kw), log=LOG, env=DistEnv(id_run="ga"))


def no_own_grads(model) -> bool:
    return all(p.grad is None for p in model.parameters())


# ------------------------------------------------------------------ key handling, arena binding
@pytest.mark.parametrize("mixed,want", [(True, torch.bfloat16), (False, torch.float32)])
def test_null_keeps_the_weights_dtype(workdir, mixed, want):
    t = make(tiny_model(), use_mixed_precision=mixed)
    assert TRAIN_DEFAULTS["grad_accum_dtype"] is None
    assert t.arena.grad_dtype == want and all(a.dtype == want for a in t.arena.acc)
    assert not t.arena.main_grad and all(not hasattr(p, "main_grad") for p in t.model.parameters())
    assert all(p.grad is not None and p.grad.dtype == want for p in t.model.parameters())


def test_fp32_binds_main_grad_and_leaves_grad_none(workdir):
    t = make(tiny_model(), grad_accum_dtype="fp32")
    a = t.arena
    assert a.dtype == torch.bfloat16 and a.grad_dtype == torch.float32 and [x.dtype for x in a.acc] == [torch.float32] * 2
    assert no_own_grads(t.model)
    for idx in (1, 0):
        a.point_grads(idx)
        for p, o, n in zip(a.params, a.offsets, a.numels):
            assert p.main_grad.dtype == torch.float32 and p.main_grad.data_ptr() == a.acc[idx][o:o + n].data_ptr()
        assert no_own_grads(t.model)
    assert t.get_grads().dtype == torch.float32 and t.get_grads().data_ptr() == a.acc[0].data_ptr()


def test_fp32_with_fp32_weights_changes_nothing(workdir):
    t = make(tiny_model(), grad_accum_dtype="fp32", use_mixed_precision=False)
    assert t.arena.grad_dtype == torch.float32 and not t.arena.main_grad
    assert all(p.grad is not None for p in t.model.parameters())


@pytest.mark.parametrize("value", ["fp16", "bf16", "float32", 32, True])
def test_bad_values_are_rejected(workdir, value):
    with pytest.raises(ValueError, match="grad_accum_dtype"):
        make(tiny_model(), grad_accum_dtype=value)


def test_rejects_a_non_native_model(workdir):
    class Wrapped(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.inner = tiny_model()

        def forward(self, **kw):
            return self.inner(**kw)
    with pytest.raises(ValueError, match="native model"):
        make(Wrapped(), grad_accum_dtype="fp32")


def test_rejects_torch_ddp(workdir):
    with pytest.raises(ValueError, match="ddp_impl=torch"):
        make(tiny_model(), grad_accum_dtype="fp32", method_name="ddp", ddp_impl="torch")


def test_train_config_carries_the_key():
    import yaml
    with open(os.path.join(ROOT, "config", "train", "acco.yaml")) as f:
        assert yaml.safe_load(f)["grad_accum_dtype"] is None


# ------------------------------------------------------------------ torch paths add into main_grad
class _Params(torch.nn.Module):
    def __init__(self, shapes, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        for k, s in shapes.items():
            setattr(self, k, torch.nn.Parameter((torch.randn(s, generator=g) * 0.5).to(torch.bfloat16)))


def _arena(m):
    return FlatArena(m, 1, 0, torch.bfloat16, "cpu", grad_dtype=torch.float32)


def _mb(seed, *shape):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed))).to(torch.bfloat16)


def _check_sum(acc, want64):
    # fp32 accumulation of N terms: per element within (N + 1) * 2^-24 * sum|terms| (first order); want64 carries the |terms| sum
    got, exact, mag = acc.double(), want64[0], want64[1]
    assert ((got - exact).abs() <= (want64[2] + 1) * 2.0 ** -24 * mag + 1e-30).all()


@pytest.mark.parametrize("n", [1, 8])
def test_linear_with_bias_adds_into_main_grad(n):
    m = _Params(dict(w=(24, 16), b=(24,)))
    ar = _arena(m)
    exact_w, mag_w = torch.zeros(24, 16, dtype=torch.float64), torch.zeros(24, 16, dtype=torch.float64)
    exact_b, mag_b = torch.zeros(24, dtype=torch.float64), torch.zeros(24, dtype=torch.float64)
    for i in range(n):
        x, gy = _mb(2 * i, 10, 16).requires_grad_(), _mb(2 * i + 1, 10, 24)
        y = LinearFn.apply(x, m.w, m.b, True)
        y.backward(gy)
        assert no_own_grads(m)
        dw = gy.double().t() @ x.detach().double()
        exact_w += dw
        mag_w += (gy.double().abs().t() @ x.detach().double().abs())
        exact_b += gy.double().sum(0)
        mag_b += gy.double().abs().sum(0)
    _check_sum(m.w.main_grad, (exact_w, mag_w, 10 * n))
    _check_sum(m.b.main_grad, (exact_b, mag_b, 10 * n))
    assert ar.acc[0].dtype == torch.float32


@pytest.mark.parametrize("layer", [False, True], ids=["rmsnorm", "layernorm"])
def test_norm_adds_into_main_grad(layer):
    m = _Params(dict(w=(16,), b=(16,)) if layer else dict(w=(16,)))
    _arena(m)
    n, acc_w = 4, torch.zeros(16, dtype=torch.float64)
    for i in range(n):
        x, gy = _mb(3 * i, 6, 16), _mb(3 * i + 1, 6, 16)
        y = ops.layernorm(x, m.w, m.b) if layer else ops.rmsnorm(x, m.w)
        y.backward(gy)
        assert no_own_grads(m)
        xf = x.double()
        if layer:
            xh = (xf - xf.mean(-1, keepdim=True)) / torch.sqrt(xf.var(-1, unbiased=False, keepdim=True) + 1e-5)
        else:
            xh = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5)
        acc_w += (gy.double() * xh).sum(0)
    torch.testing.assert_close(m.w.main_grad.double(), acc_w, rtol=1e-5, atol=1e-5)
    if layer:
        assert m.b.main_grad.abs().sum() > 0


def test_embedding_adds_into_main_grad():
    m = _Params(dict(w=(12, 8)))
    _arena(m)
    want = torch.zeros(12, 8, dtype=torch.float64)
    for i in range(16):
        ids = torch.randint(0, 12, (20,), generator=torch.Generator().manual_seed(i))
        gy = _mb(100 + i, 20, 8)
        ops.embedding(ids, m.w).backward(gy)
        assert no_own_grads(m)
        want.index_add_(0, ids, gy.double())
    torch.testing.assert_close(m.w.main_grad.double(), want, rtol=1e-6, atol=1e-6)


def test_gpt_neo_positions_add_into_main_grad(workdir):
    t = make(_neo(), grad_accum_dtype="fp32", nb_steps_tot=2)
    t.train()
    assert no_own_grads(t.model)
    wpe = t.model.transformer.wpe
    assert wpe.main_grad.dtype == torch.float32


def test_fp8_reference_adds_into_main_grad():
    m = _Params(dict(w=(32, 16)))
    _arena(m)
    want = torch.zeros(32, 16, dtype=torch.float64)
    for i in range(4):
        x, gy = _mb(7 * i, 16, 16).requires_grad_(), _mb(7 * i + 1, 16, 32)
        Fp8LinearFn.apply(x, m.w, None, True).backward(gy)
        assert no_own_grads(m)
        qg, _, sg = quantize_ref(gy, E5M2)
        qx, _, sx = quantize_ref(x.detach(), E4M3)
        want += (qg.double().t() @ qx.double()) * (sg[1].double() * sx[1].double())
    torch.testing.assert_close(m.w.main_grad.double(), want, rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------ trainers
def _run(model, **kw):
    t = make(model, **kw)
    t.train()
    return t


@pytest.mark.parametrize("method", ["acco", "dpu", "ddp"])
@pytest.mark.parametrize("arch", ["llama", "gptneo"])
def test_trainer_matches_the_fp32_trainer(workdir, method, arch):
    mk = (lambda: tiny_model()) if arch == "llama" else _neo
    kw = dict(method_name=method, nb_steps_tot=12, n_grad_accumulation=4, learning_rate=3e-3)
    ref = _run(mk(), use_mixed_precision=False, **kw)
    got = _run(mk(), grad_accum_dtype="fp32", **kw)
    assert no_own_grads(got.model)
    assert got.sharded_optimizer.step == ref.sharded_optimizer.step >= 2
    # what training moved the fp32 masters by, from the bf16 start and from the fp32 start: bf16 weights against fp32 weights change
    # the forward at bf16 resolution, which moves the updates by a small fraction of their size
    moved_got = got.sharded_optimizer.master - _run(mk(), grad_accum_dtype="fp32", **dict(kw, nb_steps_tot=0)).sharded_optimizer.master
    moved_ref = ref.sharded_optimizer.master - _run(mk(), use_mixed_precision=False, **dict(kw, nb_steps_tot=0)).sharded_optimizer.master
    rel = ((moved_got - moved_ref).norm() / moved_ref.norm()).item()
    print(f"{arch} {method}: relative difference of the updates {rel:.3g}")
    assert rel < 0.15


def _worker(rank, world, port, tmp, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(CUDA_VISIBLE_DEVICES="", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), ACCO_RUN_ID="ga")
    os.chdir(tmp)
    torch.set_num_threads(1)
    from acco_b200.launch import shutdown_distributed
    out = []
    for kw in (dict(use_mixed_precision=False), dict(use_mixed_precision=True, grad_accum_dtype="fp32")):
        ds = synthetic_pretrain_dataset(300, 30, 96, 16, seed=7)
        args = base_args(method_name="acco", nb_steps_tot=12, n_grad_accumulation=2, learning_rate=3e-3, static_accumulation=True, **kw)
        t = DecoupledTrainer(model=tiny_model(), train_dataset=ds, args=args, log=LOG)
        t.train()
        out.append((t.sharded_optimizer.step, t.arena.params_flat.float().clone(), no_own_grads(t.model), t.arena.grad_dtype))
    q.put((rank, out))
    shutdown_distributed()


def test_two_gloo_ranks():
    from acco_b200.launch import free_port
    with tempfile.TemporaryDirectory() as tmp:
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        port = free_port()
        procs = [ctx.Process(target=_worker, args=(r, 2, port, tmp, q)) for r in range(2)]
        for p in procs:
            p.start()
        res = sorted((q.get(timeout=300) for _ in procs), key=lambda o: o[0])
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    (_, r0), (_, r1) = res
    for (s0, w0, clean0, dt0), (s1, w1, clean1, dt1) in zip(r0, r1):
        assert s0 == s1 >= 2 and dt0 == dt1
        assert torch.equal(w0, w1)                                  # every rank holds the same weights
    assert r0[1][3] == torch.float32 and r0[1][2] and r1[1][2]      # fp32 accumulators, no parameter holds a .grad of its own
    ref, got = r0[0][1], r0[1][1]
    assert (got - ref).abs().max() < 2e-2
