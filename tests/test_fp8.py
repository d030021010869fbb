"""FP8 linear layers (train key ``fp8``) on the CPU reference path: the quantiser's scale rule and edges, the reference FP8 linear
against the contract written out in fp64, the trainer with ``fp8=True`` on tiny Llama / GPT-Neo models, the rejected combinations,
the train configs, and the SASS summary of the FP8 kernels."""
import json
import os

import pytest
import torch
import yaml

from acco_b200 import DecoupledTrainer, TRAIN_DEFAULTS, ops
from acco_b200.data import synthetic_pretrain_dataset
from acco_b200.launch import DistEnv
from acco_b200.models import GPTConfig, GPTForCausalLM
from acco_b200.ops.fp8 import E4M3, E5M2, FP8_MAX, quantize_ref, scale_ref

from helpers import LOG, base_args, tiny_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FMTS = [E4M3, E5M2]


@pytest.fixture(autouse=True)
def _cpu_path(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)


# ------------------------------------------------------------------------------------------------------------------ quantiser
@pytest.mark.parametrize("fmt", FMTS)
def test_scale_is_the_largest_power_of_two_that_fits(fmt):
    mx = FP8_MAX[fmt]
    g = torch.Generator().manual_seed(0)
    amaxes = torch.cat([torch.rand(200, generator=g) * 10 ** torch.randint(-30, 30, (200,), generator=g).float(),
                        torch.tensor([1.0, 3.0, 448.0, 57344.0, 1e-20, 3e38])]).bfloat16().float()
    for a in amaxes:
        s, inv = scale_ref(a, fmt)
        k = int(torch.log2(s))
        assert float(s) == 2.0 ** k and float(inv) == 2.0 ** -k
        assert float(a) * 2.0 ** k <= mx < float(a) * 2.0 ** (k + 1)


@pytest.mark.parametrize("fmt", FMTS)
def test_scale_edges(fmt):
    mx = FP8_MAX[fmt]
    for k in (-20, -1, 0, 3, 40):
        p = torch.tensor(mx * 2.0 ** k)                       # amax = max_f * 2^k exactly: s = 2^-k, q(amax) = max_f
        assert float(scale_ref(p, fmt)[0]) == 2.0 ** -k
        up = p.bfloat16().float() * (1 + 2 ** -7)              # one bf16 ulp either side of max_f * 2^k
        dn = p.bfloat16().float() * (1 - 2 ** -8)
        assert float(scale_ref(up, fmt)[0]) == 2.0 ** (-k - 1)
        assert float(scale_ref(dn, fmt)[0]) == 2.0 ** -k
    for k in (-9, 0, 7):                                      # amax a power of two: amax * s = the largest power of two <= max_f
        s = float(scale_ref(torch.tensor(2.0 ** k), fmt)[0])
        assert 2.0 ** k * s == (256.0 if fmt == E4M3 else 32768.0)
    assert [float(v) for v in scale_ref(torch.tensor(0.0), fmt)] == [1.0, 1.0]
    for bad in (float("nan"), float("inf"), -float("inf")):
        s, inv = scale_ref(torch.tensor(bad).abs(), fmt)
        assert torch.isnan(s) and torch.isnan(inv)


@pytest.mark.parametrize("fmt", FMTS)
def test_quantize_ref_never_overflows_and_handles_zero_subnormal_nan(fmt):
    g = torch.Generator().manual_seed(1)
    for scale in (1e-6, 1.0, 3e4, 1e30):
        t = (torch.randn(64, 48, generator=g) * scale).bfloat16()
        q, qT, s = quantize_ref(t, fmt, True, True)
        assert torch.isfinite(q.float()).all()
        assert float(q.float().abs().max()) <= FP8_MAX[fmt]
        assert float(s[2]) == float(t.float().abs().max())
        assert torch.equal(qT.view(torch.uint8), q.view(torch.uint8).t())
        # round to nearest: the dequantised value is within half a format ulp of t
        rel = ((q.float() * s[1] - t.float()).abs() / t.float().abs().clamp_min(1e-38))
        big = t.float().abs() * s[0] >= (2.0 ** -6 if fmt == E4M3 else 2.0 ** -14)      # normal range of the format
        assert float(rel[big].max()) <= (2.0 ** -4 if fmt == E4M3 else 2.0 ** -3)
    z = torch.zeros(16, 16).bfloat16()
    q, _, s = quantize_ref(z, fmt)
    assert s.tolist() == [1.0, 1.0, 0.0] and float(q.float().abs().max()) == 0
    sub = torch.full((16, 16), 2.0 ** -130).bfloat16()                                   # bf16 subnormals
    q, _, s = quantize_ref(sub, fmt)
    assert float(s[0]) == 2.0 ** 127                                                     # the cap: the largest fp32 power of two
    assert torch.equal(q.float(), (sub.float() * 2.0 ** 127).to(fmt).float())
    n = torch.ones(16, 16).bfloat16()
    n[3, 4] = float("nan")
    q, _, s = quantize_ref(n, fmt)
    assert torch.isnan(s[0]) and torch.isnan(q.float()).all()


# ------------------------------------------------------------------------------------------------------------------ linear
def _deq(t, fmt):
    q, _, s = quantize_ref(t, fmt)
    return q.double() * float(s[1])


def test_reference_fp8_linear_matches_the_fp64_contract():
    g = torch.Generator().manual_seed(2)
    T, K, N = 64, 48, 32
    x = (torch.randn(T, K, generator=g)).bfloat16().requires_grad_(True)
    w = torch.nn.Parameter((torch.randn(N, K, generator=g) * 0.1).bfloat16())
    b = torch.nn.Parameter((torch.randn(N, generator=g) * 0.1).bfloat16())
    w.grad = torch.zeros_like(w)
    b.grad = torch.zeros_like(b)
    dw = torch.zeros(N, K, dtype=torch.float64)
    bsum = torch.zeros(N, dtype=torch.float64)
    for mb in range(2):                                       # two micro-batches accumulate into the same .grad
        gy = (torch.randn(T, N, generator=g) * 1e-2).bfloat16()
        y = ops.linear(x, w, b, fp8=True)
        y64 = _deq(x.detach(), E4M3) @ _deq(w.detach(), E4M3).t() + b.detach().double()
        assert torch.equal(y, y64.bfloat16())                 # fp32 accumulation of K = 48 products: exact here, one rounding
        x.grad = None
        y.backward(gy)
        dx64 = _deq(gy, E5M2) @ _deq(w.detach(), E4M3)
        assert torch.equal(x.grad, dx64.bfloat16())
        dw = (dw + _deq(gy, E5M2).t() @ _deq(x.detach(), E4M3)).bfloat16().double()   # bf16 gradient, one rounding per add
        bsum += gy.double().sum(0)
        assert torch.equal(w.grad, dw.bfloat16())
    torch.testing.assert_close(b.grad.double(), bsum, rtol=1e-2, atol=1e-3)


def test_fp8_flag_only_affects_grad_enabled_calls_of_supported_shapes():
    x = torch.randn(32, 48).bfloat16()
    w = torch.nn.Parameter((torch.randn(32, 48) * 0.1).bfloat16())
    with torch.no_grad():
        assert torch.equal(ops.linear(x, w, fp8=True), ops.linear(x, w))
    y = ops.linear(x, w, fp8=True)
    assert type(y.grad_fn).__name__ == "Fp8LinearFnBackward"
    w2 = torch.nn.Parameter((torch.randn(40, 48) * 0.1).bfloat16())         # N = 40: not a multiple of 16
    assert type(ops.linear(x, w2, fp8=True).grad_fn).__name__ == "LinearFnBackward"
    assert type(ops.linear(torch.randn(24, 48).bfloat16(), w, fp8=True).grad_fn).__name__ == "LinearFnBackward"   # T = 24


# ------------------------------------------------------------------------------------------------------------------ trainer
def _neo(seed=0):
    torch.manual_seed(seed)
    return GPTForCausalLM(GPTConfig(vocab_size=96, hidden_size=32, num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=32,
                                    attention_layers=["global", "local"], window_size=8, pad_vocab_multiple=8))


def _make(model, **kw):
    ds = synthetic_pretrain_dataset(200, 30, 96, 16, seed=3)
    kw.setdefault("use_mixed_precision", True)
    return DecoupledTrainer(model=model, train_dataset=ds, args=base_args(**kw), log=LOG, env=DistEnv(id_run="fp8"))


def _run(model, **kw):
    from acco_b200.callbacks import TrainerCallback

    class Rec(TrainerCallback):
        losses = []

        def on_log(self, trainer, scalars):
            self.losses.append(float(scalars["loss"]))
    t = _make(model, **kw)
    cb = Rec()
    cb.losses = []
    t.add_callback(cb)
    t.train()
    return t, cb.losses


@pytest.mark.parametrize("make", [lambda: tiny_model(hidden=32), _neo], ids=["llama", "gptneo"])
def test_trainer_fp8_on_the_reference_path(workdir, make):
    t, losses = _run(make(), fp8=True, nb_steps_tot=30, batch_size=4, learning_rate=3e-3)
    assert t.model.fp8 is True
    assert sum(losses[-5:]) / 5 < losses[0]                   # the loss falls
    assert all(p.dtype == torch.bfloat16 for p in t.model.parameters())   # weights stay bf16
    path = str(workdir / "fp8.pt")
    t.save_checkpoint(path)
    sd = torch.load(path, map_location="cpu")
    assert set(sd) == set(t.model.state_dict())                           # the checkpoint format is unchanged: same keys,
    assert all(v.dtype == torch.bfloat16 for v in sd.values())            # bf16 tensors, no FP8 state
    fresh = make()
    fresh.load_state_dict(sd)
    assert fresh.fp8 is False                                              # FP8 is a training setting, not part of the model file


def test_fp8_false_is_bitwise_the_default(workdir):
    a, la = _run(tiny_model(), nb_steps_tot=6, fp8=False)
    b, lb = _run(tiny_model(), nb_steps_tot=6)
    assert la == lb
    for (n, p), (_, q) in zip(a.model.named_parameters(), b.model.named_parameters()):
        assert torch.equal(p, q), n
    assert a.model.fp8 is False and TRAIN_DEFAULTS["fp8"] is False


@pytest.mark.parametrize("kw,match", [
    (dict(use_mixed_precision=False), "use_mixed_precision"),
    (dict(ddp_weights_dtype="fp32"), "ddp_weights_dtype"),
    (dict(fused_ag_gemm=True), "fused_ag_gemm"),
])
def test_fp8_rejects_unsupported_combinations(workdir, kw, match):
    with pytest.raises(ValueError, match=match):
        _make(tiny_model(), fp8=True, **kw)


def test_fp8_rejects_a_non_native_model(workdir):
    class Wrapped(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.inner = tiny_model()

        def forward(self, **kw):
            return self.inner(**kw)
    with pytest.raises(ValueError, match="native model"):
        _make(Wrapped(), fp8=True)


# ------------------------------------------------------------------------------------------------------------------ configs, SASS
def test_train_configs_carry_fp8_false():
    d = os.path.join(ROOT, "config", "train")
    names = sorted(f for f in os.listdir(d) if f.endswith(".yaml"))
    assert len(names) == 6
    for f in names:
        assert yaml.safe_load(open(os.path.join(d, f)))["fp8"] is False, f


def test_sass_summary_of_the_fp8_kernels():
    from acco_b200.ops import ext_path
    if ext_path() is None:
        pytest.skip("extension not built")
    summary = json.load(open(os.path.join(ROOT, "docs", "sass", "mnemonics.json")))
    gemms = [k for k in summary if k.startswith("gemm_fp8")]
    assert len(gemms) >= 2
    for k in gemms:
        e = summary[k]
        # FP8 wgmma.mma_async assembles to QGMMA (the bf16 one to HGMMA); no legacy mma.sync (HMMA)
        assert e.get("QGMMA", 0) > 0 and e["UTMALDG"] > 0 and e["UTMASTG"] > 0 and e["HMMA"] == 0, (k, e)
    assert any(k.startswith("fp8_cast") for k in summary) and any(k.startswith("fp8_amax") for k in summary)
