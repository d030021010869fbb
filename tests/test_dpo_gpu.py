"""DPO on the GPU: the ``dpo_*`` kernels against the fp64 oracle and bounds of ``test_dpo.py`` on the vocabulary shapes of the CE
tests and at 2 x 4 x 1024 rows x 128256, equal inputs giving ln 2, two launches bitwise equal, whole native models against TRL's
formula on bf16 weights, the launches of one micro-batch, the trainer with CUDA graphs against the fp32 CPU trainer (plain, ``fp8``,
``grad_accum_dtype=fp32``, ``max_grad_norm``), and the logged rewards and accuracy against a recomputation from the same batch.
Run with ``pytest -m gpu -s`` to see the worst error / bound ratios."""
import math
import os
import subprocess
import sys
from collections import Counter

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops  # noqa: E402
from test_dpo import LN2, dpo_checks, dpo_grad_ref, dpo_inputs, dpo_ref, dpo_token_terms, shift, trl_loss  # noqa: E402
from test_rowwise_kernels_gpu import CE_SHAPES  # noqa: E402
from test_rowwise_oracle import FTZ, ratio  # noqa: E402

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def C():
    return ops.load_ext(required=True)


@pytest.fixture(autouse=True)
def _free_between_cases():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def run_dpo(C, s, r, lb, P, V, beta, dloss=0.75, rows=256):
    """DPO kernel forward + backward (on a copy) against the fp64 oracle, token terms and gradient in row chunks on the device;
    returns the worst error / bound per output."""
    Tn, Vp = s.shape
    S = Tn // (2 * P)
    out = torch.full((3,), math.nan, device=DEV)
    r_keep = r.clone()
    loss, lse, w = C.dpo_fwd(s, r, lb, P, V, -100, beta, out)
    grad = s.clone()
    C.dpo_bwd_inplace(grad, lb, lse, w, torch.tensor([dloss], device=DEV), P, V, -100)
    assert torch.equal(r.view(torch.int16), r_keep.view(torch.int16)), "the reference logits must not be written"
    del r_keep
    chunks = [dpo_token_terms(s[a:a + rows], r[a:a + rows], lb[a:a + rows], V) for a in range(0, Tn, rows)]
    terms = {k: torch.cat([c[k] for c in chunks]) for k in chunks[0]}
    o = dpo_ref(None, None, None, P, V, beta, terms=terms)
    got = {"loss": float(loss), "reward_chosen": float(out[0]), "reward_rejected": float(out[1]), "accuracy": float(out[2]),
           "lse": lse.cpu(), "w": w.cpu()}
    worst = dpo_checks(got, o)
    row = torch.arange(Tn, device=DEV) // S
    wv, E_w = o["w"].to(DEV), ((o["b_w"] - FTZ) / 2).to(DEV)                  # b_w = 2 E_w + FTZ
    g = 0.0
    for a in range(0, Tn, rows):
        sl = slice(a, a + rows)
        want, bnd = dpo_grad_ref(s[sl], lb[sl], terms["lse"][sl], terms["E_lse"][sl], wv[row[sl]], E_w[row[sl]], V, dloss)
        g = max(g, ratio(grad[sl], want, bnd))
    worst["grad"] = g
    return worst, o, float(loss), out.cpu()


def report(name, worst):
    print(f"\n[dpo] {name}: " + " ".join(f"{k}={v:.3f}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 1.0, (name, k, v)


def _gpu_inputs(P, S, V, Vp, seed, noise=0.5, pad=None):
    s, r, lb, _, _ = dpo_inputs(P, S, V, Vp, seed=seed, noise=noise, pad_fill=pad)
    return s.to(DEV), r.to(DEV), lb.to(DEV)


@pytest.mark.parametrize("beta,noise", [(0.1, 0.5), (1.0, 0.5), (1.0, 8.0)], ids=["b0.1", "b1", "b1-large-z"])
@pytest.mark.parametrize("V,Vp,pad", [(V, Vp, pad) for V, Vp in CE_SHAPES for pad in ((None, math.nan) if Vp > V else (None,))])
def test_dpo_kernels_against_fp64(C, V, Vp, pad, beta, noise):
    P, S = (3, 16) if Vp <= 4096 else (2, 8)
    s, r, lb = _gpu_inputs(P, S, V, Vp, seed=V + S, noise=noise, pad=pad)
    worst, o, _, _ = run_dpo(C, s, r, lb, P, V, beta)
    report(f"P{P} S{S} V{V} Vp{Vp} beta{beta} noise{noise} pad{pad}", worst)
    assert o["n"] == P - 1


@pytest.mark.parametrize("beta", [0.1, 1.0])
def test_dpo_kernels_llama3_microbatch(C, beta):
    """2 x 4 x 1024 token rows of the Llama-3 vocabulary (4 pairs of 1024-token rows, padded and prompt-masked)."""
    P, S, V = 4, 1024, 128256
    g = torch.Generator(device=DEV).manual_seed(11)
    s = (3 * torch.randn(2 * P * S, V, generator=g, device=DEV)).to(torch.bfloat16)
    r = (s.float() + 0.5 * torch.randn(2 * P * S, V, generator=g, device=DEV)).to(torch.bfloat16)
    tok = torch.randint(0, V, (2 * P, S), generator=g, device=DEV)
    a = torch.randint(1, S // 2, (2 * P, 1), generator=g, device=DEV)
    e = torch.randint(S // 2 + 1, S + 1, (2 * P, 1), generator=g, device=DEV)
    col = torch.arange(S, device=DEV)[None, :]
    lab = torch.where((col >= a) & (col < e), tok, torch.full_like(tok, -100))
    worst, o, _, _ = run_dpo(C, s, r, shift(lab), P, V, beta, rows=128)
    report(f"P{P} S{S} V{V} beta{beta}", worst)
    assert o["n"] == P


def test_equal_inputs_give_ln2_and_two_launches_are_bitwise_equal(C):
    P, S, V, Vp = 3, 64, 50257, 50304
    s, r, lb = _gpu_inputs(P, S, V, Vp, seed=2)
    out = torch.zeros(3, device=DEV)
    loss, lse, w = C.dpo_fwd(s, s, lb, P, V, -100, 0.1, out)
    n = P - 1
    assert abs(float(loss) - LN2) <= 2 * 2.0 ** -24 * 4, float(loss)
    assert out.tolist() == [0.0, 0.0, 0.0]
    want_w = torch.tensor([0.0] + [0.05 / n] * (P - 1) + [0.0] + [-0.05 / n] * (P - 1), dtype=torch.float32)
    torch.testing.assert_close(w.cpu(), want_w, rtol=2e-7, atol=0)
    res = []
    for _ in range(2):
        o = torch.zeros(3, device=DEV)
        l2, lse2, w2 = C.dpo_fwd(s, r, lb, P, V, -100, 0.1, o)
        gr = s.clone()
        C.dpo_bwd_inplace(gr, lb, lse2, w2, torch.ones(1, device=DEV), P, V, -100)
        res.append((l2.clone(), lse2.clone(), w2.clone(), o.clone(), gr))
    for a, b in zip(*res):
        assert torch.equal(a.view(-1).view(torch.uint8), b.view(-1).view(torch.uint8))


def test_all_invalid_batch_and_bindings_reject_bad_arguments(C):
    P, S, V, Vp = 2, 8, 1000, 1008
    s, r, lb = _gpu_inputs(P, S, V, Vp, seed=4)
    lb.view(2 * P, S)[P:] = -100
    out = torch.full((3,), -1.0, device=DEV)
    loss, lse, w = C.dpo_fwd(s, r, lb, P, V, -100, 0.1, out)
    gr = s.clone()
    C.dpo_bwd_inplace(gr, lb, lse, w, torch.ones(1, device=DEV), P, V, -100)
    assert float(loss) == 0.0 and bool((out == 0).all()) and bool((w == 0).all()) and bool((gr.float() == 0).all())
    for bad in (0.0, -1.0, math.inf, math.nan):
        with pytest.raises(RuntimeError, match="beta"):
            C.dpo_fwd(s, r, lb, P, V, -100, bad, out)
    with pytest.raises(RuntimeError, match="ref_logits"):
        C.dpo_fwd(s, r[:-8], lb, P, V, -100, 0.1, out)
    with pytest.raises(RuntimeError, match="2 P S"):
        C.dpo_fwd(s, r, lb, 3, V, -100, 0.1, out)
    with pytest.raises(RuntimeError, match="three-element"):
        C.dpo_fwd(s, r, lb, P, V, -100, 0.1, torch.zeros(2, device=DEV))
    with pytest.raises(RuntimeError, match="multiple of 8"):
        C.dpo_fwd(s, r, lb, P, Vp + 1, -100, 0.1, out)


# ================================================================================================= whole models
def _policy(which):
    from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    if which == "llama":
        return LlamaForCausalLM(LlamaConfig(vocab_size=50257, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                                            num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=256))
    return GPTForCausalLM(GPTConfig(vocab_size=50257, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                                    max_position_embeddings=256, attention_layers="alternating", window_size=64))


def _reference(which):
    m = _policy(which)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.01 * torch.randn_like(p))               # a nearby reference, as after a little SFT
    return m


def _pairs_batch(P, S, V, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ids = torch.randint(0, V, (2 * P, S), generator=g, device=DEV)
    col = torch.arange(S, device=DEV)[None, :]
    a = torch.randint(1, S // 2, (2 * P, 1), generator=g, device=DEV)
    e = torch.randint(S // 2 + 1, S + 1, (2 * P, 1), generator=g, device=DEV)
    return ids, torch.where((col >= a) & (col < e), ids, torch.full_like(ids, -100))


@pytest.mark.parametrize("which", ["llama", "gptneo"])
def test_native_model_matches_trl_formula(which):
    """Same bf16 weights and batch, fwd + bwd with ``reference_logits`` and through TRL's formula in fp32 torch on the logits;
    parameter gradients agree to ``2^-6`` of their norm."""
    m, ref = _policy(which).to(DEV, torch.bfloat16), _reference(which).to(DEV, torch.bfloat16).requires_grad_(False)
    ids, labels = _pairs_batch(2, 256, 50257, seed=3)
    m.dpo_beta, m.dpo_out = 0.5, torch.zeros(3, device=DEV)
    with torch.no_grad():
        rl = ref.padded_logits(ids)
    loss = m(input_ids=ids, labels=labels, reference_logits=rl)[0]
    loss.backward()
    got = {k: p.grad.float().clone() for k, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    want = trl_loss(m(input_ids=ids).logits.float(), rl.view(4, 256, -1)[..., :50257].float(), labels, 2, 0.5)
    want.backward()
    assert abs(float(loss) - float(want)) <= 1e-3 * max(abs(float(want)), 1e-2), (float(loss), float(want))
    for k, p in m.named_parameters():
        r = p.grad.float()
        assert float((got[k] - r).norm()) <= 2.0 ** -6 * float(r.norm()) + 1e-8, k
    assert all(p.grad is None for p in ref.parameters())


def test_launches_of_one_micro_batch():
    """One DPO micro-batch = the policy's CE micro-batch with the CE kernels replaced by one DPO forward + reduce and one DPO
    backward, plus exactly the launches of one no-grad reference forward: no reference backward."""
    m, ref = _policy("llama").to(DEV, torch.bfloat16), _reference("llama").to(DEV, torch.bfloat16).requires_grad_(False)
    ids, labels = _pairs_batch(1, 256, 50257, seed=1)
    m.dpo_out = torch.zeros(3, device=DEV)

    def counts(fn):
        fn()
        torch.cuda.synchronize()
        ops.reset_launch_counts()
        fn()
        torch.cuda.synchronize()
        return Counter(ops.launch_counts())

    def plain():
        m(input_ids=ids, labels=labels)[0].backward()

    def r_fwd():
        with torch.no_grad():
            ref.padded_logits(ids)

    def dpo():
        with torch.no_grad():
            rl = ref.padded_logits(ids)
        m(input_ids=ids, labels=labels, reference_logits=rl)[0].backward()

    c_plain, c_r, c_dpo = counts(plain), counts(r_fwd), counts(dpo)
    assert c_dpo["dpo_fwd"] == 2 and c_dpo["dpo_bwd"] == 1 and c_dpo["ce_fwd"] == 0 and c_dpo["ce_bwd"] == 0, c_dpo
    want = c_plain + c_r + Counter(dpo_fwd=2, dpo_bwd=1)
    want.subtract(Counter(ce_fwd=2, ce_bwd=1))
    assert +want == +c_dpo, (dict(want), dict(c_dpo))


# ================================================================================================= trainer
_TRAINER_SCRIPT = r"""
import logging, sys, torch
sys.path.insert(0, {root!r})
from acco_b200 import AttrDict, DecoupledTrainer, ops
from acco_b200.callbacks import TrainerCallback
from acco_b200.data import ByteTokenizer, synthetic_preference_dataset
from acco_b200.launch import discover_env
from acco_b200.models import LlamaConfig, LlamaForCausalLM
cuda, variant = sys.argv[1] == "cuda", sys.argv[3]
cfg = LlamaConfig(vocab_size=1000, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                  num_key_value_heads=2, max_position_embeddings=128)
torch.manual_seed(0)
m = LlamaForCausalLM(cfg)
torch.manual_seed(0)
ref = LlamaForCausalLM(cfg)
tok = ByteTokenizer()
tok.pad_token_id = tok.eos_token_id = 999
ds = synthetic_preference_dataset(2000, 100, 999, seed=1)
args = AttrDict(method_name="acco", batch_size=4, n_grad_accumulation=1, max_length=128, nb_steps_tot=40, warmup=2, learning_rate=1e-3,
                save=False, tensorboard=False, seed=1, const_len_batch=False, pad_to_multiple_of=128, use_mixed_precision=cuda,
                fp8=bool(variant == "fp8" and cuda), grad_accum_dtype="fp32" if variant == "grad_accum_fp32" else None,
                max_grad_norm=0.5 if variant == "max_grad_norm" else None, dpo_beta=0.5, static_accumulation=True, log_every=1)
env = discover_env()
env.id_run = "dpo"
t = DecoupledTrainer(model=m, tokenizer=tok, train_dataset=ds, args=args, log=logging.getLogger("dpo"), env=env, reference=ref)
logs = []
class Rec(TrainerCallback):
    def on_log(self, trainer, scalars):
        logs.append((scalars["loss"], scalars["dpo_reward_chosen"], scalars["dpo_reward_rejected"], scalars["dpo_accuracy"]))
t.add_callback(Rec())
t.train()
torch.save({{"logs": logs, "counts": (t.sched.count_grad_tot, t.sched.opt_steps), "cuda": t.is_cuda,
            "graphs": t._graphs is not None and len(t._graphs._graphs) > 0, "graphs_disabled": bool(getattr(t, "_graphs_disabled", None)),
            "launches": ops.launch_counts() if cuda else {{}}}}, sys.argv[2])
"""


def _train(tmp_path, dev, variant):
    from acco_b200.launch import free_port
    script = tmp_path / "dpo_train.py"
    script.write_text(_TRAINER_SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR")}
    env["MASTER_PORT"] = str(free_port())
    if dev == "cpu":
        env["CUDA_VISIBLE_DEVICES"] = ""
    out = tmp_path / f"{dev}_{variant}.pt"
    p = subprocess.run([sys.executable, str(script), dev, str(out), variant], cwd=tmp_path, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:]
    return torch.load(out, weights_only=False)


@pytest.mark.parametrize("variant", ["plain", "fp8", "grad_accum_fp32", "max_grad_norm"])
def test_trainer_with_graphs_tracks_fp32_cpu_trainer(tmp_path, variant):
    """One GPU, ACCO, CUDA graphs, bf16, beta 0.5, the reference = the policy's initial weights, against the fp32 CPU trainer.  The
    GPU run must capture graphs and keep them on and run the DPO kernels; its logged loss and rewards must stay within bf16
    training noise of the CPU ones, and the loss must move away from ln 2 as the policy learns the preference."""
    gpu, cpu = _train(tmp_path, "cuda", variant), _train(tmp_path, "cpu", variant)
    assert gpu["cuda"] and not cpu["cuda"]
    assert gpu["graphs"] and not gpu["graphs_disabled"], gpu
    assert gpu["launches"].get("dpo_fwd", 0) > 0 and gpu["launches"].get("dpo_bwd", 0) > 0 and not gpu["launches"].get("ce_fwd")
    if variant == "fp8":
        assert any(k.startswith("gemm_fp8") for k in gpu["launches"]), gpu["launches"]
    assert gpu["counts"] == cpu["counts"] and len(gpu["logs"]) == len(cpu["logs"]) >= 10
    a, b = torch.tensor(gpu["logs"]), torch.tensor(cpu["logs"])
    assert abs(float(a[0, 0]) - LN2) < 0.05 and abs(float(b[0, 0]) - LN2) < 1e-6     # policy == reference on the first micro-batch
    tol = 0.03 if variant == "fp8" else 0.015
    noise = float((a[:, 0] - b[:, 0]).abs().mean())
    assert noise <= tol * float(b[:, 0].abs().mean()), (variant, gpu["logs"], cpu["logs"])
    margin = (a[:, 1] - a[:, 2]) - (b[:, 1] - b[:, 2])
    assert float(margin.abs().mean()) <= 0.1 * float((b[:, 1] - b[:, 2]).abs().mean()) + 0.02, (variant, gpu["logs"], cpu["logs"])
    assert float(b[-3:, 0].mean()) < LN2 - 0.01 and float(a[-3:, 0].mean()) < LN2 - 0.01      # it learns the preference


def test_logged_rewards_and_accuracy_match_the_batch(workdir):
    """A fixed device batch through the graphed micro-batch: the rewards and accuracy the trainer copies to the host are those of
    that batch under the weights it ran on, and the loss is the DPO objective."""
    import logging
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.launch import DistEnv
    m = _policy("llama")
    args = AttrDict(method_name="acco", batch_size=2, max_length=256, nb_steps_tot=64, warmup=0, learning_rate=1e-3, save=False,
                    tensorboard=False, const_len_batch=False, dpo_beta=0.5)
    t = DecoupledTrainer(model=m, train_dataset=None, args=args, log=logging.getLogger("dpo"), env=DistEnv(id_run="dpo"),
                         reference=_reference("llama"))
    ids, labels = _pairs_batch(2, 256, 50257, seed=5)
    batch = {"input_ids": ids, "labels": labels}
    t.input_override = lambda: batch
    for _ in range(3):
        t._drain()
        with torch.no_grad():
            s = t.model(input_ids=ids).logits.float()
            rl = t.reference(input_ids=ids).logits.float()
        lb, mask = labels[:, 1:], labels[:, 1:] != -100
        idx = torch.where(mask, lb, torch.zeros_like(lb))[..., None]
        lp = lambda x: (torch.log_softmax(x[:, :-1], -1).gather(-1, idx)[..., 0] * mask).sum(-1)
        D = lp(s) - lp(rl)
        rc, rr = 0.5 * D[:2], 0.5 * D[2:]
        want_loss = float(trl_loss(s, rl, labels, 2, 0.5))
        t.step()
        torch.cuda.synchronize()
        got = [float(v) for v in t.dpo_host]
        assert t._graphs is not None and not getattr(t, "_graphs_disabled", None)
        assert abs(got[0] - float(rc.mean())) <= 2e-3 * abs(float(rc.mean())) + 2e-3, (got, rc)
        assert abs(got[1] - float(rr.mean())) <= 2e-3 * abs(float(rr.mean())) + 2e-3, (got, rr)
        assert got[2] == float(((rc - rr) > 0).float().mean())
        assert abs(float(t.loss_host) - want_loss) <= 2e-3 * want_loss, (float(t.loss_host), want_loss)
