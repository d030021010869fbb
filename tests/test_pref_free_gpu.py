"""SimPO and ORPO on the GPU: ``ce_fwd`` + ``pref_reduce`` + ``dpo_bwd`` against the fp64 oracle and bounds of ``test_pref_free.py`` on
the vocabulary shapes of the CE tests and at 2 x 4 x 1024 rows x 128256, two launches bitwise equal, the identical-pair identities,
whole native models against TRL's formulas on bf16 weights, the launches of one micro-batch, the trainer with CUDA graphs against the
fp32 CPU trainer (plain, ``fp8``, ``grad_accum_dtype=fp32``, ``max_grad_norm``), and the logged scalars against a recomputation from
the same batch.  Run with ``pytest -m gpu -s`` to see the worst error / bound ratios."""
import math
import os
import subprocess
import sys
from collections import Counter

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops  # noqa: E402
from test_dpo import dpo_grad_ref, shift  # noqa: E402
from test_pref_free import pref_checks, pref_inputs, pref_ref, token_terms, trl_orpo, trl_simpo  # noqa: E402
from test_rowwise_kernels_gpu import CE_SHAPES  # noqa: E402
from test_rowwise_oracle import ratio  # noqa: E402

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LN2 = math.log(2.0)


@pytest.fixture(scope="module")
def C():
    return ops.load_ext(required=True)


@pytest.fixture(autouse=True)
def _free_between_cases():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def run_pref(C, s, lb, P, V, obj, coef, gamma=0.0, dloss=0.75, rows=256):
    """Kernel forward + backward (on a copy) against the fp64 oracle, token terms and gradient in row chunks on the device; returns
    the worst error / bound per output, the oracle and the kernel's outputs."""
    Tn, Vp = s.shape
    S = Tn // (2 * P)
    out = torch.full((3,), math.nan, device=DEV)
    loss, lse, w = C.pref_fwd(s, lb, P, V, -100, obj == "orpo", coef, gamma, out)
    grad = s.clone()
    C.dpo_bwd_inplace(grad, lb, lse, w, torch.tensor([dloss], device=DEV), P, V, -100)
    chunks = [token_terms(s[a:a + rows], lb[a:a + rows], V) for a in range(0, Tn, rows)]
    terms = {k: torch.cat([c[k] for c in chunks]) for k in chunks[0]}
    o = pref_ref(None, None, P, V, obj, coef, gamma, terms=terms)
    got = {"loss": float(loss), "out0": float(out[0]), "out1": float(out[1]), "out2": float(out[2]), "lse": lse.cpu(), "w": w.cpu()}
    worst = pref_checks(got, o)
    row = torch.arange(Tn, device=DEV) // S
    wv, E_w = o["w"].to(DEV), o["E_w"].to(DEV)
    g = 0.0
    for a in range(0, Tn, rows):
        sl = slice(a, a + rows)
        want, bnd = dpo_grad_ref(s[sl], lb[sl], terms["lse"][sl], terms["E_lse"][sl], wv[row[sl]], E_w[row[sl]], V, dloss)
        g = max(g, ratio(grad[sl], want, bnd))
    worst["grad"] = g
    return worst, o, got


def report(name, worst):
    print(f"\n[pref] {name}: " + " ".join(f"{k}={v:.3f}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 1.0, (name, k, v)


ARMS = [("simpo", 2.5, 0.5, 3.0, 0.0), ("simpo", 0.5, 1.4, 40.0, 0.0), ("orpo", 0.1, 0.0, 3.0, 0.0), ("orpo", 1.0, 0.0, 3.0, 12.0),
        ("orpo", 0.1, 0.0, 3.0, 60.0)]
ARM_IDS = ["simpo-b2.5-g0.5", "simpo-b0.5-g1.4-large-z", "orpo-l0.1", "orpo-l1-confident", "orpo-l0.1-clamped"]


@pytest.mark.parametrize("obj,coef,gamma,scale,sharp", ARMS, ids=ARM_IDS)
@pytest.mark.parametrize("V,Vp,pad", [(V, Vp, pad) for V, Vp in CE_SHAPES for pad in ((None, math.nan) if Vp > V else (None,))])
def test_kernels_against_fp64(C, V, Vp, pad, obj, coef, gamma, scale, sharp):
    P, S = (3, 16) if Vp <= 4096 else (2, 8)
    s, lb, _, _ = pref_inputs(P, S, V, Vp, seed=V + S, scale=scale, sharp=sharp, pad_fill=pad)
    worst, o, got = run_pref(C, s.to(DEV), lb.to(DEV), P, V, obj, coef, gamma)
    report(f"{obj} P{P} S{S} V{V} Vp{Vp} coef{coef} gamma{gamma} scale{scale} sharp{sharp} pad{pad}", worst)
    assert o["n"] == P - 1 and math.isfinite(got["loss"])


@pytest.mark.parametrize("obj,coef,gamma", [("simpo", 2.0, 0.5), ("orpo", 0.1, 0.0)])
def test_kernels_llama3_microbatch(C, obj, coef, gamma):
    """2 x 4 x 1024 token rows of the Llama-3 vocabulary (4 pairs of 1024-token rows, padded and prompt-masked)."""
    P, S, V = 4, 1024, 128256
    g = torch.Generator(device=DEV).manual_seed(11)
    s = (3 * torch.randn(2 * P * S, V, generator=g, device=DEV)).to(torch.bfloat16)
    tok = torch.randint(0, V, (2 * P, S), generator=g, device=DEV)
    a = torch.randint(1, S // 2, (2 * P, 1), generator=g, device=DEV)
    e = torch.randint(S // 2 + 1, S + 1, (2 * P, 1), generator=g, device=DEV)
    col = torch.arange(S, device=DEV)[None, :]
    lab = torch.where((col >= a) & (col < e), tok, torch.full_like(tok, -100))
    worst, o, _ = run_pref(C, s, shift(lab), P, V, obj, coef, gamma, rows=128)
    report(f"{obj} P{P} S{S} V{V}", worst)
    assert o["n"] == P


def test_two_launches_are_bitwise_equal_and_identical_pairs_give_the_identities(C):
    P, S, V, Vp = 3, 64, 50257, 50304
    s, lb, _, _ = pref_inputs(P, S, V, Vp, seed=2, sharp=6.0, invalid=False)
    s, lb = s.to(DEV), lb.to(DEV)
    for orpo, coef, gamma in ((False, 2.0, 0.5), (True, 0.1, 0.0)):
        res = []
        for _ in range(2):
            o = torch.zeros(3, device=DEV)
            loss, lse, w = C.pref_fwd(s, lb, P, V, -100, orpo, coef, gamma, o)
            gr = s.clone()
            C.dpo_bwd_inplace(gr, lb, lse, w, torch.ones(1, device=DEV), P, V, -100)
            res.append((loss.clone(), lse.clone(), w.clone(), o.clone(), gr))
        for a, b in zip(*res):
            assert torch.equal(a.view(-1).view(torch.uint8), b.view(-1).view(torch.uint8))
    s2, lb2 = s.clone(), lb.clone()
    s2.view(2 * P, S, Vp)[P:] = s2.view(2 * P, S, Vp)[:P]
    lb2.view(2 * P, S)[P:] = lb2.view(2 * P, S)[:P]
    out = torch.zeros(3, device=DEV)
    loss, _, w = C.pref_fwd(s2, lb2, P, V, -100, False, 2.5, 1.4, out)
    assert abs(float(loss) - math.log1p(math.exp(1.4))) <= 8 * 2.0 ** -24 * 2, float(loss)
    assert torch.equal(w[:P], -w[P:]) and out[2] == 0.0
    out = torch.zeros(3, device=DEV)
    loss, _, w = C.pref_fwd(s2, lb2, P, V, -100, True, 0.5, 0.0, out)
    n_c = float((lb2.view(2 * P, S)[:P] != -100).sum())
    assert out[1] == 0.0 and out[2] == 0.0
    assert abs(float(loss) - (float(out[0]) + 0.5 * LN2)) <= 8 * 2.0 ** -24 * (1 + abs(float(loss)))
    torch.testing.assert_close(w[:P] - 1.0 / n_c, -w[P:], rtol=1e-5, atol=1e-7)


def test_all_invalid_batch_and_bindings_reject_bad_arguments(C):
    P, S, V, Vp = 2, 8, 1000, 1008
    s, lb, _, _ = pref_inputs(P, S, V, Vp, seed=4)
    s, lb = s.to(DEV), lb.to(DEV)
    lb.view(2 * P, S)[P:] = -100
    for orpo, coef, gamma in ((False, 2.0, 0.5), (True, 0.1, 0.0)):
        out = torch.full((3,), -1.0, device=DEV)
        loss, lse, w = C.pref_fwd(s, lb, P, V, -100, orpo, coef, gamma, out)
        gr = s.clone()
        C.dpo_bwd_inplace(gr, lb, lse, w, torch.ones(1, device=DEV), P, V, -100)
        assert float(loss) == 0.0 and bool((out == 0).all()) and bool((w == 0).all()) and bool((gr.float() == 0).all())
    out = torch.zeros(3, device=DEV)
    for bad in (0.0, -1.0, math.inf, math.nan):
        with pytest.raises(RuntimeError, match="beta"):
            C.pref_fwd(s, lb, P, V, -100, False, bad, 0.5, out)
        with pytest.raises(RuntimeError, match="lambda"):
            C.pref_fwd(s, lb, P, V, -100, True, bad, 0.0, out)
    for bad in (-1.0, math.inf, math.nan):
        with pytest.raises(RuntimeError, match="gamma"):
            C.pref_fwd(s, lb, P, V, -100, False, 2.0, bad, out)
    with pytest.raises(RuntimeError, match="gamma"):
        C.pref_fwd(s, lb, P, V, -100, True, 0.1, 0.5, out)
    with pytest.raises(RuntimeError, match="2 P S"):
        C.pref_fwd(s, lb, 3, V, -100, False, 2.0, 0.5, out)
    with pytest.raises(RuntimeError, match="three-element"):
        C.pref_fwd(s, lb, P, V, -100, False, 2.0, 0.5, torch.zeros(2, device=DEV))
    with pytest.raises(RuntimeError, match="multiple of 8"):
        C.pref_fwd(s, lb, P, Vp + 1, -100, False, 2.0, 0.5, out)


# ================================================================================================= whole models
def _policy(which):
    from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    if which == "llama":
        return LlamaForCausalLM(LlamaConfig(vocab_size=50257, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                                            num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=256))
    return GPTForCausalLM(GPTConfig(vocab_size=50257, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                                    max_position_embeddings=256, attention_layers="alternating", window_size=64))


def _pairs_batch(P, S, V, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ids = torch.randint(0, V, (2 * P, S), generator=g, device=DEV)
    col = torch.arange(S, device=DEV)[None, :]
    a = torch.randint(1, S // 2, (2 * P, 1), generator=g, device=DEV)
    e = torch.randint(S // 2 + 1, S + 1, (2 * P, 1), generator=g, device=DEV)
    return ids, torch.where((col >= a) & (col < e), ids, torch.full_like(ids, -100))


def _set(m, obj):
    if obj == "simpo":
        m.simpo_beta, m.simpo_gamma = 2.0, 0.5
    else:
        m.orpo_lambda = 0.1
    m.pref_out = torch.zeros(3, device=DEV)


def _formula(obj, logits, labels, P):
    return trl_simpo(logits, labels, P, 2.0, 0.5) if obj == "simpo" else trl_orpo(logits, labels, P, 0.1)


@pytest.mark.parametrize("obj", ["simpo", "orpo"])
@pytest.mark.parametrize("which", ["llama", "gptneo"])
def test_native_model_matches_trl_formula(which, obj):
    """Same bf16 weights and batch, fwd + bwd with ``preference_pairs=True`` and through TRL's formula in fp32 torch on the logits;
    parameter gradients agree to ``2^-6`` of their norm."""
    m = _policy(which).to(DEV, torch.bfloat16)
    _set(m, obj)
    ids, labels = _pairs_batch(2, 256, 50257, seed=3)
    loss = m(input_ids=ids, labels=labels, preference_pairs=True)[0]
    loss.backward()
    got = {k: p.grad.float().clone() for k, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    want = _formula(obj, m(input_ids=ids).logits.float(), labels, 2)
    want.backward()
    loss, want = float(loss.detach()), float(want.detach())
    assert abs(loss - want) <= 1e-3 * max(abs(want), 1e-2), (loss, want)
    for k, p in m.named_parameters():
        r = p.grad.float()
        assert float((got[k] - r).norm()) <= 2.0 ** -6 * float(r.norm()) + 1e-8, k


@pytest.mark.parametrize("obj", ["simpo", "orpo"])
def test_launches_of_one_micro_batch(obj):
    """One SimPO / ORPO micro-batch = the CE micro-batch with ``ce_reduce`` replaced by ``pref_reduce`` and ``ce_bwd`` by ``dpo_bwd``:
    no reference or teacher forward, no other launch."""
    m = _policy("llama").to(DEV, torch.bfloat16)
    _set(m, obj)
    ids, labels = _pairs_batch(1, 256, 50257, seed=1)

    def counts(fn):
        fn()
        torch.cuda.synchronize()
        ops.reset_launch_counts()
        fn()
        torch.cuda.synchronize()
        return Counter(ops.launch_counts())

    c_plain = counts(lambda: m(input_ids=ids, labels=labels)[0].backward())
    c_pref = counts(lambda: m(input_ids=ids, labels=labels, preference_pairs=True)[0].backward())
    assert c_pref["ce_fwd"] == 1 and c_pref["pref_reduce"] == 1 and c_pref["dpo_bwd"] == 1 and c_pref["ce_bwd"] == 0, c_pref
    assert c_pref["dpo_fwd"] == 0 and c_pref["kd_fwd"] == 0
    want = c_plain + Counter(pref_reduce=1, dpo_bwd=1)
    want.subtract(Counter(ce_fwd=1, ce_bwd=1))
    assert +want == +c_pref, (dict(want), dict(c_pref))


# ================================================================================================= trainer
_TRAINER_SCRIPT = r"""
import logging, sys, torch
sys.path.insert(0, {root!r})
from acco_b200 import AttrDict, DecoupledTrainer, ops
from acco_b200.callbacks import TrainerCallback
from acco_b200.data import ByteTokenizer, synthetic_preference_dataset
from acco_b200.launch import discover_env
from acco_b200.models import LlamaConfig, LlamaForCausalLM
from acco_b200.trainer import PREF_SCALARS
cuda, variant, obj = sys.argv[1] == "cuda", sys.argv[3], sys.argv[4]
cfg = LlamaConfig(vocab_size=1000, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                  num_key_value_heads=2, max_position_embeddings=128)
torch.manual_seed(0)
m = LlamaForCausalLM(cfg)
tok = ByteTokenizer()
tok.pad_token_id = tok.eos_token_id = 999
ds = synthetic_preference_dataset(2000, 100, 999, seed=1)
keys = dict(simpo_beta=2.0, simpo_gamma=0.5) if obj == "simpo" else dict(orpo_lambda=0.1)
args = AttrDict(method_name="acco", batch_size=4, n_grad_accumulation=1, max_length=128, nb_steps_tot=40, warmup=2, learning_rate=1e-3,
                save=False, tensorboard=False, seed=1, const_len_batch=False, pad_to_multiple_of=128, use_mixed_precision=cuda,
                fp8=bool(variant == "fp8" and cuda), grad_accum_dtype="fp32" if variant == "grad_accum_fp32" else None,
                max_grad_norm=0.5 if variant == "max_grad_norm" else None, static_accumulation=True, log_every=1, **keys)
env = discover_env()
env.id_run = "pref"
t = DecoupledTrainer(model=m, tokenizer=tok, train_dataset=ds, args=args, log=logging.getLogger("pref"), env=env)
logs = []
class Rec(TrainerCallback):
    def on_log(self, trainer, scalars):
        logs.append([scalars["loss"]] + [scalars[k] for k in PREF_SCALARS[obj]])
t.add_callback(Rec())
t.train()
torch.save({{"logs": logs, "counts": (t.sched.count_grad_tot, t.sched.opt_steps), "cuda": t.is_cuda,
            "graphs": t._graphs is not None and len(t._graphs._graphs) > 0, "graphs_disabled": bool(getattr(t, "_graphs_disabled", None)),
            "launches": ops.launch_counts() if cuda else {{}}}}, sys.argv[2])
"""


def _train(tmp_path, dev, variant, obj):
    from acco_b200.launch import free_port
    script = tmp_path / "pref_train.py"
    script.write_text(_TRAINER_SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR")}
    env["MASTER_PORT"] = str(free_port())
    if dev == "cpu":
        env["CUDA_VISIBLE_DEVICES"] = ""
    out = tmp_path / f"{dev}_{variant}_{obj}.pt"
    p = subprocess.run([sys.executable, str(script), dev, str(out), variant, obj], cwd=tmp_path, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:]
    return torch.load(out, weights_only=False)


@pytest.mark.parametrize("obj", ["simpo", "orpo"])
@pytest.mark.parametrize("variant", ["plain", "fp8", "grad_accum_fp32", "max_grad_norm"])
def test_trainer_with_graphs_tracks_fp32_cpu_trainer(tmp_path, variant, obj):
    """One GPU, ACCO, CUDA graphs, bf16, against the fp32 CPU trainer.  The GPU run must capture graphs and keep them on and run the
    SimPO / ORPO kernels; its logged loss and scalars must stay within bf16 training noise of the CPU ones, and the loss must fall as
    the policy learns the preference."""
    gpu, cpu = _train(tmp_path, "cuda", variant, obj), _train(tmp_path, "cpu", variant, obj)
    assert gpu["cuda"] and not cpu["cuda"]
    assert gpu["graphs"] and not gpu["graphs_disabled"], gpu
    L = gpu["launches"]
    assert L.get("pref_reduce", 0) > 0 and L.get("dpo_bwd", 0) > 0 and not L.get("dpo_fwd") and not L.get("ce_bwd"), L
    if variant == "fp8":
        assert any(k.startswith("gemm_fp8") for k in L), L
    assert gpu["counts"] == cpu["counts"] and len(gpu["logs"]) == len(cpu["logs"]) >= 10
    a, b = torch.tensor(gpu["logs"]), torch.tensor(cpu["logs"])
    tol = 0.03 if variant == "fp8" else 0.015
    noise = float((a[:, 0] - b[:, 0]).abs().mean())
    assert noise <= tol * float(b[:, 0].abs().mean()), (variant, gpu["logs"], cpu["logs"])
    j = 1 if obj == "simpo" else 2                        # SimPO: the chosen reward; ORPO: the mean log odds ratio
    assert float((a[:, j] - b[:, j]).abs().mean()) <= 0.05 * float(b[:, j].abs().mean()) + 0.02, (variant, gpu["logs"], cpu["logs"])
    assert float(b[-3:, 0].mean()) < float(b[:3, 0].mean()) and float(a[-3:, 0].mean()) < float(a[:3, 0].mean())


@pytest.mark.parametrize("obj", ["simpo", "orpo"])
def test_logged_scalars_match_the_batch(workdir, obj):
    """A fixed device batch through the graphed micro-batch: the scalars the trainer copies to the host are those of that batch under
    the weights it ran on, and the loss is the objective."""
    import logging
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.launch import DistEnv
    m = _policy("llama")
    keys = dict(simpo_beta=2.0, simpo_gamma=0.5) if obj == "simpo" else dict(orpo_lambda=0.1)
    args = AttrDict(method_name="acco", batch_size=2, max_length=256, nb_steps_tot=64, warmup=0, learning_rate=1e-3, save=False,
                    tensorboard=False, const_len_batch=False, **keys)
    t = DecoupledTrainer(model=m, train_dataset=None, args=args, log=logging.getLogger("pref"), env=DistEnv(id_run="pref"))
    ids, labels = _pairs_batch(2, 256, 50257, seed=5)
    batch = {"input_ids": ids, "labels": labels}
    t.input_override = lambda: batch
    for _ in range(3):
        t._drain()
        with torch.no_grad():
            s = t.model(input_ids=ids).logits.float()
        want_out = torch.zeros(3)
        flat = s.reshape(-1, s.shape[-1]).cpu()
        want_loss = float(ops.simpo_loss(flat, shift(labels).cpu(), 2, flat.shape[1], 2.0, 0.5, out=want_out) if obj == "simpo"
                          else ops.orpo_loss(flat, shift(labels).cpu(), 2, flat.shape[1], 0.1, out=want_out))
        assert want_loss == pytest.approx(float(_formula(obj, s, labels, 2)), rel=1e-5)
        t.step()
        torch.cuda.synchronize()
        got = [float(v) for v in t.pref_host]
        assert t._graphs is not None and not getattr(t, "_graphs_disabled", None)
        for k in (0, 1):
            assert abs(got[k] - float(want_out[k])) <= 2e-3 * abs(float(want_out[k])) + 2e-3, (got, want_out)
        assert got[2] == float(want_out[2])
        assert abs(float(t.loss_host) - want_loss) <= 2e-3 * abs(want_loss) + 1e-4, (float(t.loss_host), want_loss)
