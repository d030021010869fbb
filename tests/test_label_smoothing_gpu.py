"""Label smoothing in the fused cross-entropy kernels on the GPU: the smoothed kernels against the fp64 oracle and bounds of
``test_label_smoothing.py`` at every vocabulary shape of the unsmoothed tests, eps = 0 bitwise the call without the argument, the
``ops`` glue, whole native models against the ``LabelSmoother`` route, and the trainer with CUDA graphs against the fp32 CPU
trainer (plain, with ``packing`` at the acco-ft shapes, and with ``fp8``).  Run with ``pytest -m gpu -s`` to see the worst
error / bound ratios."""
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops  # noqa: E402
from test_label_smoothing import ls_ref  # noqa: E402
from test_rowwise_kernels_gpu import CE_SHAPES  # noqa: E402
from test_rowwise_oracle import FTZ, ce_inputs, ce_loss_bound, ratio  # noqa: E402

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


def run_ls(C, lg, lab, V, eps, dloss=1.0, rows=128):
    """Smoothed kernel forward + backward (on a copy) against the fp64 oracle on row chunks."""
    T, Vp = lg.shape
    loss, inv_n, lse = C.ce_fwd(lg, lab, V, -100, eps)
    n = int((lab != -100).sum())
    scale = torch.tensor([dloss], device=DEV) * inv_n
    grad = lg.clone()
    C.ce_bwd_inplace(grad, lab, lse, scale, V, -100, eps)
    inv64 = 1.0 / n if n else 0.0
    worst = {"lse": 0.0, "grad": 0.0}
    row_sum = E_sum = abs_sum = 0.0
    for r0 in range(0, T, rows):
        sl = slice(r0, r0 + rows)
        o = ls_ref(lg[sl], lab[sl], V, eps, scale=float(scale))
        worst["lse"] = max(worst["lse"], ratio(lse[sl], o["lse"], o["b_lse"]))
        worst["grad"] = max(worst["grad"], ratio(grad[sl], o["grad"], o["b_grad"]))
        if Vp > V:
            assert bool((grad[sl, V:] == 0).all()), "padding columns must get exactly zero gradient"
        assert bool((grad[sl][lab[sl] == -100] == 0).all()), "ignored rows must get exactly zero gradient"
        row_sum += float(o["row"].sum())
        abs_sum += float(o["row"].abs().sum())
        E_sum += float(o["E_row"].sum())
        del o
    loss64 = row_sum * inv64
    worst["loss"] = abs(float(loss) - loss64) / ce_loss_bound(E_sum, abs_sum, T, loss64, inv64)
    worst["inv_n"] = abs(float(inv_n) - inv64) / max(2 * 2.0 ** -22 * inv64, FTZ)
    assert torch.isfinite(lse).all() and math.isfinite(float(loss))
    return worst


def report(name, worst):
    print(f"\n[label smoothing] {name}: worst error/bound " + " ".join(f"{k}={v:.3f}" for k, v in worst.items()))


# ================================================================================================= kernels vs fp64
@pytest.mark.parametrize("eps", [0.1, 0.5, 1.0])
@pytest.mark.parametrize("V,Vp,pad", [(V, Vp, pad) for V, Vp in CE_SHAPES for pad in ((None, math.nan, math.inf) if Vp > V else (None,))])
def test_smoothed_kernels_against_fp64(C, V, Vp, pad, eps):
    """Labels at 0, V - 1 and the argmax (``ce_inputs``); padding random, NaN or +inf: out of the softmax and of sum x."""
    lg, lab = ce_inputs(64, V, Vp, seed=V, pad_fill=pad, device=DEV)
    worst = run_ls(C, lg, lab, V, eps, dloss=2.5)
    report(f"V={V}/{Vp} pad={pad} eps={eps}", worst)
    for k, v in worst.items():
        assert v <= 1.0, (k, v, worst)


@pytest.mark.parametrize("shift", [0.0, 12.0])
def test_smoothed_kernels_llama3_microbatch(C, shift):
    """T = 4096 rows of the Llama-3 vocabulary; ``shift`` moves every logit so that sum x is large (the eps / V term matters)."""
    lg, lab = ce_inputs(4096, 128256, 128256, seed=1, device=DEV)
    if shift:
        lg = (lg.float() + shift).to(torch.bfloat16)
        lab[3] = int(lg[3].float().argmax())
    worst = run_ls(C, lg, lab, 128256, 0.1, rows=64)
    report(f"T=4096 V=128256 shift={shift}", worst)
    for k, v in worst.items():
        assert v <= 1.0, (k, v, worst)


def test_smoothed_all_ignored_batch_is_pinned_to_zero(C):
    lg, lab = ce_inputs(40, 1000, 1008, seed=2, pad_fill=math.nan, device=DEV)
    lab[:] = -100
    loss, inv_n, lse = C.ce_fwd(lg, lab, 1000, -100, 0.5)
    assert float(loss) == 0.0 and float(inv_n) == 0.0 and bool((lse == 0).all())
    grad = lg.clone()
    C.ce_bwd_inplace(grad, lab, lse, torch.ones(1, device=DEV) * inv_n, 1000, -100, 0.5)
    assert bool((grad == 0).all())


@pytest.mark.parametrize("V,Vp", [(50257, 50304), (131, 136), (128256, 128256)])
def test_eps_zero_is_bitwise_the_call_without_the_argument(C, V, Vp):
    lg, lab = ce_inputs(96, V, Vp, seed=7, pad_fill=math.nan if Vp > V else None, device=DEV)
    a = C.ce_fwd(lg, lab, V, -100)
    b = C.ce_fwd(lg, lab, V, -100, 0.0)
    c = C.ce_fwd(lg, lab, V, -100, label_smoothing=0.0)
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, z)
    scale = a[1] * 1.5
    ga, gb = lg.clone(), lg.clone()
    C.ce_bwd_inplace(ga, lab, a[2], scale, V, -100)
    C.ce_bwd_inplace(gb, lab, a[2], scale, V, -100, 0.0)
    assert torch.equal(ga.view(torch.int16), gb.view(torch.int16))


@pytest.mark.parametrize("eps", [-0.1, 1.0001, math.nan, math.inf])
def test_bindings_reject_bad_eps(C, eps):
    lg, lab = ce_inputs(8, 131, 136, seed=1, device=DEV)
    with pytest.raises(RuntimeError, match="label_smoothing"):
        C.ce_fwd(lg, lab, 131, -100, eps)
    loss, inv_n, lse = C.ce_fwd(lg, lab, 131, -100)
    with pytest.raises(RuntimeError, match="label_smoothing"):
        C.ce_bwd_inplace(lg.clone(), lab, lse, inv_n, 131, -100, eps)


# ================================================================================================= ops glue
def test_glue_scale_and_launch_counts():
    """``softmax_cross_entropy(label_smoothing=eps)`` scales the backward by ``dloss * inv_n`` and launches 2 + 1 kernels."""
    V, Vp = 50257, 50304
    lg, lab = ce_inputs(300, V, Vp, seed=5, device=DEV)
    keep = lg.clone()
    x = lg.clone().requires_grad_(True)
    ops.reset_launch_counts()
    loss = ops.softmax_cross_entropy(x * 1.0, lab, V, -100, label_smoothing=0.1)
    (loss * 3.0).backward()
    counts = ops.launch_counts()
    assert counts.get("ce_fwd") == 2 and counts.get("ce_bwd") == 1, counts
    n = int((lab != -100).sum())
    o = ls_ref(keep, lab, V, 0.1)
    assert abs(float(loss) - o["loss"]) <= o["b_loss"]
    for r0 in range(0, 300, 100):
        o = ls_ref(keep[r0:r0 + 100], lab[r0:r0 + 100], V, 0.1, scale=3.0 / n)
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
def test_native_model_matches_label_smoother_route(which):
    """Same bf16 weights and batch, fwd + bwd through ``model.label_smoothing`` and through ``LabelSmoother`` on the logits.

    The logits are bitwise the same on both routes (same kernels).  The losses differ by the kernel's error (bounded by the
    oracle, below 1e-5 relative at this size) plus ``LabelSmoother``'s fp32 log-softmax (a few fp32 ulps of the row terms):
    ``2e-5`` relative.  Each d-logit is the bf16 rounding of the same real number on both routes, so the two differ by at most one
    bf16 ulp (``2^-8`` relative); the backward is linear in the d-logits and its bf16 GEMMs round both the same way, so each
    parameter's gradient differs by at most ``2^-8`` of the norm the d-logits carry into it, plus one more bf16 rounding of each
    GEMM output: ``||g - g_ref|| <= 2^-6 ||g_ref||`` leaves a factor of two."""
    from acco_b200.utils.misc import LabelSmoother
    name, m = next((n, m) for n, m in _models() if n == which)
    m = m.to(DEV, torch.bfloat16)
    g = torch.Generator(device=DEV).manual_seed(3)
    ids = torch.randint(0, 50257, (4, 256), generator=g, device=DEV)
    labels = ids.clone()
    labels[1, 100:] = -100
    m.label_smoothing = 0.1
    loss = m(input_ids=ids, labels=labels)[0]
    loss.backward()
    got = {k: p.grad.float().clone() for k, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    m.label_smoothing = 0.0
    ref = LabelSmoother(0.1)(m(input_ids=ids), labels, shift_labels=True)
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 2e-5 * abs(float(ref)), (float(loss), float(ref))
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
from acco_b200.data import ByteTokenizer, synthetic_sft_dataset
from acco_b200.launch import discover_env
from acco_b200.models import LlamaConfig, LlamaForCausalLM
cuda, variant, eps = sys.argv[1] == "cuda", sys.argv[3], float(sys.argv[4])
packing = variant == "packing"
L = 512 if packing else 128
cfg = LlamaConfig(vocab_size=1000, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                  num_key_value_heads=2, max_position_embeddings=L)
torch.manual_seed(0)
m = LlamaForCausalLM(cfg)
tok = ByteTokenizer()
tok.pad_token_id = tok.eos_token_id = 999
ds = synthetic_sft_dataset(1200, 90 if packing else 60, 999, L, seed=1)
args = AttrDict(method_name="acco", batch_size=4, n_grad_accumulation=2 if packing else 1, max_length=L, nb_steps_tot=48 if packing else 32, warmup=2,
                learning_rate=1e-3, save=False, tensorboard=False, seed=1, const_len_batch=False, packing=packing,
                use_mixed_precision=cuda, fp8=bool(variant == "fp8" and cuda), label_smoothing_factor=eps, static_accumulation=True)
env = discover_env()
env.id_run = "ls"
t = DecoupledTrainer(model=m, tokenizer=tok, train_dataset=ds, args=args, log=logging.getLogger("ls"), env=env)
losses = []
while not t.finished():
    t.step()
    losses.append(float(t.loss_host))
t._drain()
t._finish("")
torch.save({{"losses": losses, "counts": (t.sched.count_grad_tot, t.sched.opt_steps), "cuda": t.is_cuda,
            "graphs": t._graphs is not None and len(t._graphs._graphs) > 0, "graphs_disabled": bool(getattr(t, "_graphs_disabled", None)),
            "smoother": t.label_smoother is not None, "eps": float(t.model.label_smoothing),
            "launches": ops.launch_counts() if cuda else {{}}}}, sys.argv[2])
"""


def _train(tmp_path, dev, variant, eps):
    from acco_b200.launch import free_port
    script = tmp_path / "ls_train.py"
    script.write_text(_TRAINER_SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR")}
    env["MASTER_PORT"] = str(free_port())
    if dev == "cpu":
        env["CUDA_VISIBLE_DEVICES"] = ""
    out = tmp_path / f"{dev}_{variant}_{eps}.pt"
    p = subprocess.run([sys.executable, str(script), dev, str(out), variant, str(eps)], cwd=tmp_path, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:]
    return torch.load(out, weights_only=False)


@pytest.mark.parametrize("variant", ["plain", "packing", "fp8"])
def test_trainer_with_graphs_tracks_fp32_cpu_trainer(tmp_path, variant):
    """One GPU, ACCO, CUDA graphs, bf16 (``packing``: packed rows at the acco-ft shapes; ``fp8``: FP8 block GEMMs) with
    label_smoothing_factor = 0.3 against the fp32 CPU trainer with the same key.  The GPU run must capture graphs and keep them on,
    take the fused route (no LabelSmoother) and run the smoothed kernels; its loss trace must stay within bf16 training noise of the
    CPU trace, which is further from the unsmoothed CPU trace than that noise."""
    gpu, cpu = _train(tmp_path, "cuda", variant, 0.3), _train(tmp_path, "cpu", variant, 0.3)
    assert gpu["cuda"] and not cpu["cuda"]
    assert gpu["graphs"] and not gpu["graphs_disabled"], gpu
    assert not gpu["smoother"] and not cpu["smoother"] and gpu["eps"] == cpu["eps"] == 0.3
    assert gpu["launches"].get("ce_fwd", 0) > 0 and gpu["launches"].get("ce_bwd", 0) > 0
    if variant == "fp8":
        assert any(k.startswith("gemm_fp8") for k in gpu["launches"]), gpu["launches"]
    assert gpu["counts"] == cpu["counts"] and len(gpu["losses"]) == len(cpu["losses"]) >= 20
    a, b = torch.tensor(gpu["losses"]), torch.tensor(cpu["losses"])
    noise = float((a - b).abs().mean())
    tol = (0.02 if variant == "fp8" else 0.01) * float(b.abs().mean())
    assert noise <= tol, (noise, tol, gpu["losses"], cpu["losses"])
    plain = torch.tensor(_train(tmp_path, "cpu", variant, 0.0)["losses"])
    assert float((b - plain).abs().mean()) > 2 * noise, (float((b - plain).abs().mean()), noise)
