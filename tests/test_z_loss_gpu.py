"""Z-loss in the fused cross-entropy kernels on the GPU: the ``kZ`` kernels against the fp64 oracle and bounds of
``test_z_loss.py`` at every vocabulary shape of the unsmoothed tests (alone and with label smoothing), z = 0 bitwise the old call
forms, whole native models against the torch formula on bf16 weights, the trainer with CUDA graphs against the fp32 CPU trainer
(plain, ``packing``, ``document_mask``, ``fp8``, ``grad_accum_dtype=fp32``, ``max_grad_norm``), and the logged ``z_loss`` against a
recomputation from the same batch.  Run with ``pytest -m gpu -s`` to see the worst error / bound ratios."""
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops  # noqa: E402
from test_rowwise_kernels_gpu import CE_SHAPES  # noqa: E402
from test_rowwise_oracle import FTZ, ce_inputs, ce_loss_bound, ratio  # noqa: E402
from test_z_loss import formula, z_ref  # noqa: E402

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


def run_z(C, lg, lab, V, eps, z, dloss=1.0, rows=128):
    """``kZ`` kernel forward + backward (on a copy) against the fp64 oracle on row chunks; returns the worst error / bound."""
    T, Vp = lg.shape
    z_out = torch.full((1,), math.nan, device=DEV)
    loss, inv_n, lse = C.ce_fwd(lg, lab, V, -100, eps, z, z_out)
    n = int((lab != -100).sum())
    scale = torch.tensor([dloss], device=DEV) * inv_n
    grad = lg.clone()
    C.ce_bwd_inplace(grad, lab, lse, scale, V, -100, eps, z)
    inv64 = 1.0 / n if n else 0.0
    worst = {"lse": 0.0, "grad": 0.0}
    sums = dict(row=0.0, E=0.0, abs=0.0, z=0.0, Ez=0.0)
    for r0 in range(0, T, rows):
        sl = slice(r0, r0 + rows)
        o = z_ref(lg[sl], lab[sl], V, eps, z, scale=float(scale))
        worst["lse"] = max(worst["lse"], ratio(lse[sl], o["lse"], o["b_lse"]))
        worst["grad"] = max(worst["grad"], ratio(grad[sl], o["grad"], o["b_grad"]))
        if Vp > V:
            assert bool((grad[sl, V:] == 0).all()), "padding columns must get exactly zero gradient"
        assert bool((grad[sl][lab[sl] == -100] == 0).all()), "ignored rows must get exactly zero gradient"
        sums["row"] += float(o["row"].sum())
        sums["abs"] += float(o["row"].abs().sum())
        sums["E"] += float(o["E_row"].sum())
        sums["z"] += float(o["zt"].sum())
        sums["Ez"] += float(o["E_zt"].sum())
        del o
    loss64, z64 = sums["row"] * inv64, sums["z"] * inv64
    worst["loss"] = abs(float(loss) - loss64) / ce_loss_bound(sums["E"], sums["abs"], T, loss64, inv64)
    worst["z"] = abs(float(z_out) - z64) / ce_loss_bound(sums["Ez"], sums["z"], T, z64, inv64)
    worst["inv_n"] = abs(float(inv_n) - inv64) / max(2 * 2.0 ** -22 * inv64, FTZ)
    assert torch.isfinite(lse).all() and math.isfinite(float(loss))
    return worst


def report(name, worst):
    print(f"\n[z-loss] {name}: worst error/bound " + " ".join(f"{k}={v:.3f}" for k, v in worst.items()))


# ================================================================================================= kernels vs fp64
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("z", [1e-4, 1e-2, 1.0])
@pytest.mark.parametrize("V,Vp,pad", [(V, Vp, pad) for V, Vp in CE_SHAPES for pad in ((None, math.nan, math.inf) if Vp > V else (None,))])
def test_z_kernels_against_fp64(C, V, Vp, pad, z, eps):
    """Labels at 0, V - 1 and the argmax (``ce_inputs``); padding random, NaN or +inf: out of the softmax, the z-term and its
    gradient."""
    lg, lab = ce_inputs(64, V, Vp, seed=V, pad_fill=pad, device=DEV)
    worst = run_z(C, lg, lab, V, eps, z, dloss=2.5)
    report(f"V={V}/{Vp} pad={pad} z={z} eps={eps}", worst)
    for k, v in worst.items():
        assert v <= 1.0, (k, v, worst)


@pytest.mark.parametrize("z,eps,shift", [(1e-4, 0.0, 0.0), (1e-4, 0.0, 12.0), (1e-2, 0.1, 12.0), (1.0, 0.1, -20.0)])
def test_z_kernels_llama3_microbatch(C, z, eps, shift):
    """T = 4096 rows of the Llama-3 vocabulary; ``shift`` moves every logit, so ``lse`` (and the z-term) is large."""
    lg, lab = ce_inputs(4096, 128256, 128256, seed=1, device=DEV)
    if shift:
        lg = (lg.float() + shift).to(torch.bfloat16)
        lab[3] = int(lg[3].float().argmax())
    worst = run_z(C, lg, lab, 128256, eps, z, rows=64)
    report(f"T=4096 V=128256 z={z} eps={eps} shift={shift}", worst)
    for k, v in worst.items():
        assert v <= 1.0, (k, v, worst)


def test_z_all_ignored_batch_is_pinned_to_zero(C):
    lg, lab = ce_inputs(40, 1000, 1008, seed=2, pad_fill=math.nan, device=DEV)
    lab[:] = -100
    z_out = torch.full((1,), math.nan, device=DEV)
    loss, inv_n, lse = C.ce_fwd(lg, lab, 1000, -100, 0.1, 1.0, z_out)
    assert float(loss) == 0.0 and float(inv_n) == 0.0 and float(z_out) == 0.0 and bool((lse == 0).all())
    grad = lg.clone()
    C.ce_bwd_inplace(grad, lab, lse, torch.ones(1, device=DEV) * inv_n, 1000, -100, 0.1, 1.0)
    assert bool((grad == 0).all())


@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("V,Vp", [(50257, 50304), (131, 136), (128256, 128256)])
def test_z_zero_is_bitwise_the_old_call_forms(C, V, Vp, eps):
    lg, lab = ce_inputs(96, V, Vp, seed=7, pad_fill=math.nan if Vp > V else None, device=DEV)
    a = C.ce_fwd(lg, lab, V, -100, eps)
    b = C.ce_fwd(lg, lab, V, -100, eps, 0.0)
    c = C.ce_fwd(lg, lab, V, -100, label_smoothing=eps, z_loss=0.0, z_out=torch.full((1,), 7.0, device=DEV))
    assert len(a) == len(b) == len(c) == 3
    for x, y, w in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, w)
    scale = a[1] * 1.5
    ga, gb, gc = lg.clone(), lg.clone(), lg.clone()
    C.ce_bwd_inplace(ga, lab, a[2], scale, V, -100, eps)
    C.ce_bwd_inplace(gb, lab, a[2], scale, V, -100, eps, 0.0)
    C.ce_bwd_inplace(gc, lab, a[2], scale, V, -100, label_smoothing=eps, z_loss=0.0)
    assert torch.equal(ga.view(torch.int16), gb.view(torch.int16)) and torch.equal(ga.view(torch.int16), gc.view(torch.int16))


@pytest.mark.parametrize("z", [-1e-4, math.nan, math.inf, 1e300])
def test_bindings_reject_bad_z(C, z):
    lg, lab = ce_inputs(8, 131, 136, seed=1, device=DEV)
    out = torch.zeros(1, device=DEV)
    with pytest.raises(RuntimeError, match="z_loss"):
        C.ce_fwd(lg, lab, 131, -100, 0.0, z, out)
    loss, inv_n, lse = C.ce_fwd(lg, lab, 131, -100)
    with pytest.raises(RuntimeError, match="z_loss"):
        C.ce_bwd_inplace(lg.clone(), lab, lse, inv_n, 131, -100, 0.0, z)


def test_binding_needs_a_device_z_out(C):
    lg, lab = ce_inputs(8, 131, 136, seed=1, device=DEV)
    for bad in (None, torch.zeros(1), torch.zeros(2, device=DEV), torch.zeros(1, device=DEV, dtype=torch.float64)):
        with pytest.raises(RuntimeError, match="z_out"):
            C.ce_fwd(lg, lab, 131, -100, 0.0, 1e-4, bad)


# ================================================================================================= ops glue
def test_glue_scale_z_out_and_launch_counts():
    """``softmax_cross_entropy(z_loss=z)`` scales the backward by ``dloss * inv_n``, writes the z-term and launches 2 + 1 kernels."""
    V, Vp = 50257, 50304
    lg, lab = ce_inputs(300, V, Vp, seed=5, device=DEV)
    keep = lg.clone()
    x = lg.clone().requires_grad_(True)
    out = torch.zeros(1, device=DEV)
    ops.reset_launch_counts()
    loss = ops.softmax_cross_entropy(x * 1.0, lab, V, -100, z_loss=1e-2, z_loss_out=out)
    (loss * 3.0).backward()
    counts = ops.launch_counts()
    assert counts.get("ce_fwd") == 2 and counts.get("ce_bwd") == 1, counts
    n = int((lab != -100).sum())
    o = z_ref(keep, lab, V, 0.0, 1e-2)
    assert abs(float(loss) - o["loss"]) <= o["b_loss"] and abs(float(out) - o["z"]) <= o["b_z"]
    for r0 in range(0, 300, 100):
        o = z_ref(keep[r0:r0 + 100], lab[r0:r0 + 100], V, 0.0, 1e-2, scale=3.0 / n)
        assert ratio(x.grad[r0:r0 + 100], o["grad"], o["b_grad"]) <= 1.0


# ================================================================================================= whole models
def _models():
    from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    yield "llama", LlamaForCausalLM(LlamaConfig(vocab_size=50257, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                                                num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=256))
    torch.manual_seed(0)
    yield "gptneo", GPTForCausalLM(GPTConfig(vocab_size=50257, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                                             max_position_embeddings=256, attention_layers="alternating", window_size=64))


@pytest.mark.parametrize("which", ["llama", "gptneo"])
def test_native_model_matches_the_torch_formula(which):
    """Same bf16 weights and batch, fwd + bwd through ``model.z_loss_weight`` and through the formula in fp32 torch on the logits.
    Tolerances as for label smoothing (``test_label_smoothing_gpu``): the logits are bitwise the same on both routes, each d-logit
    is the bf16 rounding of the same real number, so parameter gradients agree to ``2^-6`` of their norm."""
    name, m = next((n, m) for n, m in _models() if n == which)
    m = m.to(DEV, torch.bfloat16)
    g = torch.Generator(device=DEV).manual_seed(3)
    ids = torch.randint(0, 50257, (4, 256), generator=g, device=DEV)
    labels = ids.clone()
    labels[1, 100:] = -100
    m.z_loss_weight, m.z_loss_out = 1e-2, torch.zeros(1, device=DEV)
    loss = m(input_ids=ids, labels=labels)[0]
    loss.backward()
    got = {k: p.grad.float().clone() for k, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    m.z_loss_weight = 0.0
    logits = m(input_ids=ids).logits[:, :-1].reshape(-1, 50257).float()
    tgt = labels[:, 1:].reshape(-1)
    ref = formula(logits, tgt, 0.0, 1e-2)
    ref.backward()
    zt = 1e-2 * torch.logsumexp(logits.detach()[tgt != -100], -1).square().mean()
    assert abs(float(loss) - float(ref)) <= 2e-5 * abs(float(ref)), (float(loss), float(ref))
    assert abs(float(m.z_loss_out) - float(zt)) <= 2e-5 * float(zt)
    flat_g = torch.cat([got[k].reshape(-1) for k, _ in m.named_parameters()])
    flat_r = torch.cat([p.grad.float().reshape(-1) for _, p in m.named_parameters()])
    assert float((flat_g - flat_r).norm()) <= 2.0 ** -6 * float(flat_r.norm())
    for k, p in m.named_parameters():
        r = p.grad.float()
        assert float((got[k] - r).norm()) <= 2.0 ** -6 * float(r.norm()) + 1e-8, k


# ================================================================================================= trainer
_TRAINER_SCRIPT = r"""
import logging, sys, torch
sys.path.insert(0, {root!r})
from acco_b200 import AttrDict, DecoupledTrainer, ops
from acco_b200.callbacks import TrainerCallback
from acco_b200.data import ByteTokenizer, synthetic_pretrain_dataset, synthetic_sft_dataset
from acco_b200.launch import discover_env
from acco_b200.models import LlamaConfig, LlamaForCausalLM
cuda, variant, z = sys.argv[1] == "cuda", sys.argv[3], float(sys.argv[4])
packing = variant == "packing"
L = 512 if packing else 128
cfg = LlamaConfig(vocab_size=1000, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                  num_key_value_heads=2, max_position_embeddings=L)
torch.manual_seed(0)
m = LlamaForCausalLM(cfg)
tok = ByteTokenizer()
tok.pad_token_id = tok.eos_token_id = 999
if packing:
    ds = synthetic_sft_dataset(1200, 90, 999, L, seed=1)
else:
    ds = synthetic_pretrain_dataset(4000, 60, 1000, L, eos_token_id=999, seed=1)
args = AttrDict(method_name="acco", batch_size=4, n_grad_accumulation=2 if packing else 1, max_length=L, nb_steps_tot=48 if packing else 32,
                warmup=2, learning_rate=1e-3, save=False, tensorboard=False, seed=1, const_len_batch=not packing, packing=packing,
                document_mask=variant == "document_mask", use_mixed_precision=cuda, fp8=bool(variant == "fp8" and cuda),
                grad_accum_dtype="fp32" if variant == "grad_accum_fp32" else None,
                max_grad_norm=0.5 if variant == "max_grad_norm" else None, z_loss_weight=z, static_accumulation=True, log_every=1)
env = discover_env()
env.id_run = "zl"
t = DecoupledTrainer(model=m, tokenizer=tok, train_dataset=ds, args=args, log=logging.getLogger("zl"), env=env)
logs = []
class Rec(TrainerCallback):
    def on_log(self, trainer, scalars):
        logs.append((scalars["loss"], scalars.get("z_loss")))
t.add_callback(Rec())
t.train()
torch.save({{"logs": logs, "counts": (t.sched.count_grad_tot, t.sched.opt_steps), "cuda": t.is_cuda,
            "graphs": t._graphs is not None and len(t._graphs._graphs) > 0, "graphs_disabled": bool(getattr(t, "_graphs_disabled", None)),
            "z": float(t.model.z_loss_weight), "launches": ops.launch_counts() if cuda else {{}}}}, sys.argv[2])
"""


def _train(tmp_path, dev, variant, z):
    from acco_b200.launch import free_port
    script = tmp_path / "zl_train.py"
    script.write_text(_TRAINER_SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR")}
    env["MASTER_PORT"] = str(free_port())
    if dev == "cpu":
        env["CUDA_VISIBLE_DEVICES"] = ""
    out = tmp_path / f"{dev}_{variant}_{z}.pt"
    p = subprocess.run([sys.executable, str(script), dev, str(out), variant, str(z)], cwd=tmp_path, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:]
    return torch.load(out, weights_only=False)


@pytest.mark.parametrize("variant", ["plain", "packing", "document_mask", "fp8", "grad_accum_fp32", "max_grad_norm"])
def test_trainer_with_graphs_tracks_fp32_cpu_trainer(tmp_path, variant):
    """One GPU, ACCO, CUDA graphs, bf16, z_loss_weight = 1e-2, against the fp32 CPU trainer with the same key.  The GPU run must
    capture graphs and keep them on and run the CE kernels; its logged loss and z_loss must stay within bf16 training noise of the
    CPU ones (``plain``: and the CPU trace must be further from the run without the key than that noise)."""
    z = 1e-2
    gpu, cpu = _train(tmp_path, "cuda", variant, z), _train(tmp_path, "cpu", variant, z)
    assert gpu["cuda"] and not cpu["cuda"]
    assert gpu["graphs"] and not gpu["graphs_disabled"], gpu
    assert gpu["z"] == cpu["z"] == z
    assert gpu["launches"].get("ce_fwd", 0) > 0 and gpu["launches"].get("ce_bwd", 0) > 0
    if variant == "fp8":
        assert any(k.startswith("gemm_fp8") for k in gpu["launches"]), gpu["launches"]
    assert gpu["counts"] == cpu["counts"] and len(gpu["logs"]) == len(cpu["logs"]) >= 10
    a, b = torch.tensor(gpu["logs"]), torch.tensor(cpu["logs"])
    assert bool((a[:, 1] > 0).all()) and bool((a[:, 1] < a[:, 0]).all())
    tol = 0.02 if variant == "fp8" else 0.01
    noise = float((a[:, 0] - b[:, 0]).abs().mean())
    assert noise <= tol * float(b[:, 0].abs().mean()), (variant, gpu["logs"], cpu["logs"])
    znoise = float((a[:, 1] - b[:, 1]).abs().mean())
    assert znoise <= 4 * tol * float(b[:, 1].abs().mean()), (variant, gpu["logs"], cpu["logs"])
    if variant == "plain":
        off = _train(tmp_path, "cpu", variant, 0.0)
        assert all(zl is None for _, zl in off["logs"])
        plain = torch.tensor([x for x, _ in off["logs"]])
        assert float((b[:, 0] - plain).abs().mean()) > 2 * noise, (float((b[:, 0] - plain).abs().mean()), noise)


def test_logged_z_loss_matches_the_batch(workdir):
    """A fixed device batch through the graphed micro-batch: the z_loss the trainer copies to the host is ``z mean lse^2`` of that
    batch's logits under the weights it ran on, and ``loss - z_loss`` its cross-entropy."""
    import logging
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import synthetic_pretrain_dataset
    from acco_b200.launch import DistEnv
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    m = LlamaForCausalLM(LlamaConfig(vocab_size=50257, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                                     num_key_value_heads=2, max_position_embeddings=256))
    ds = synthetic_pretrain_dataset(256, 200, 50257, 256, seed=0)
    args = AttrDict(method_name="acco", batch_size=4, max_length=256, nb_steps_tot=64, warmup=0, learning_rate=1e-3, save=False,
                    tensorboard=False, z_loss_weight=1e-3)
    t = DecoupledTrainer(model=m, train_dataset=ds, args=args, log=logging.getLogger("zl"), env=DistEnv(id_run="zl"))
    g = torch.Generator(device=DEV).manual_seed(5)
    batch = {"input_ids": torch.randint(0, 50257, (4, 256), generator=g, device=DEV)}
    t.input_override = lambda: batch
    for _ in range(3):
        t._drain()                  # nothing in flight: the next micro-batch runs on the weights bound now
        with torch.no_grad():
            logits = t.model(**batch).logits[:, :-1].reshape(-1, 50257).float()
        ce = float(torch.nn.functional.cross_entropy(logits, batch["input_ids"][:, 1:].reshape(-1)))
        want = 1e-3 * float(torch.logsumexp(logits, -1).square().mean())
        t.step()
        torch.cuda.synchronize()
        got = float(t.z_loss_host)
        assert t._graphs is not None and not getattr(t, "_graphs_disabled", None)
        assert abs(got - want) <= 1e-4 * want, (got, want)
        assert abs(float(t.loss_host) - got - ce) <= 1e-4 * ce, (float(t.loss_host), got, ce)
