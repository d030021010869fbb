"""Knowledge distillation on the GPU: the ``kd_*`` kernels against the fp64 oracle and bounds of ``test_distill.py`` on the
vocabulary shapes of the CE tests and at 4096 x 128256, two launches bitwise equal, the binding's rejections, whole native models
against the torch formula on bf16 weights, the launches of one micro-batch, the trainer with CUDA graphs against the fp32 CPU
trainer (plain, ``packing``, ``document_mask``, ``fp8``, ``grad_accum_dtype=fp32``, ``max_grad_norm``), and the logged
``distill_kl`` against a recomputation from the same batch.  Run with ``pytest -m gpu -s`` to see the worst error / bound ratios."""
import math
import os
import subprocess
import sys
from collections import Counter

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops  # noqa: E402
from test_distill import formula, kd_inputs, kd_ref  # noqa: E402
from test_rowwise_kernels_gpu import CE_SHAPES  # noqa: E402
from test_rowwise_oracle import FTZ, U, ce_loss_bound, ratio  # noqa: E402

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


def _inputs(Tn, V, Vp, seed, pad=None):
    s, t, lab = kd_inputs(Tn, V, Vp, seed=seed)
    if pad is not None and Vp > V:
        s[:, V:] = pad
        t[:, V:] = pad
    return s.to(DEV), t.to(DEV), lab.to(DEV)


def run_kd(C, s, t, lab, V, a, T, dloss=1.0, rows=128):
    """KD kernel forward + backward (on a copy) against the fp64 oracle on row chunks; returns the worst error / bound."""
    Tn, Vp = s.shape
    out = torch.full((2,), math.nan, device=DEV)
    t_keep = t.clone()
    loss, inv_n, lse3 = C.kd_fwd(s, t, lab, V, -100, a, T, out)
    n = int((lab != -100).sum())
    scale = torch.tensor([dloss], device=DEV) * inv_n
    grad = s.clone()
    C.kd_bwd_inplace(grad, t, lab, lse3, scale, V, -100, a, T)
    assert torch.equal(t.view(torch.int16), t_keep.view(torch.int16)), "the teacher logits must not be written"
    inv64 = 1.0 / n if n else 0.0
    worst = {"lse": 0.0, "grad": 0.0}
    sums = dict(ce=0.0, kl=0.0, Ece=0.0, Ekl=0.0, ace=0.0, akl=0.0)
    for r0 in range(0, Tn, rows):
        sl = slice(r0, r0 + rows)
        o = kd_ref(s[sl].cpu(), t[sl].cpu(), lab[sl].cpu(), V, a, T, scale=float(scale))
        worst["lse"] = max(worst["lse"], ratio(lse3[:, sl].cpu(), o["lse"], o["b_lse"]))
        worst["grad"] = max(worst["grad"], ratio(grad[sl].cpu(), o["grad"], o["b_grad"]))
        if Vp > V:
            assert bool((grad[sl, V:] == 0).all()), "padding columns must get exactly zero gradient"
        assert bool((grad[sl][lab[sl] == -100] == 0).all()), "ignored rows must get exactly zero gradient"
        sums["ce"] += float(o["ce_row"].sum())
        sums["kl"] += float(o["kl_row"].sum())
        sums["ace"] += float(o["ce_row"].abs().sum())
        sums["akl"] += float(o["kl_row"].abs().sum())
        sums["Ece"] += float(((o["b_lse"][0] - FTZ) / 2 + U * o["ce_row"].abs()).sum())
        sums["Ekl"] += float(((o["b_kl_row"] - FTZ) / 2).sum())
        del o
    ce64, kl64 = sums["ce"] * inv64, sums["kl"] * inv64
    b_ce = ce_loss_bound(sums["Ece"], sums["ace"], Tn, ce64, inv64)
    b_kl = ce_loss_bound(sums["Ekl"], sums["akl"], Tn, kl64, inv64)
    loss64 = (1 - a) * ce64 + a * T * T * kl64
    b_loss = (1 - a) * b_ce + a * T * T * b_kl + 8 * U * ((1 - a) * abs(ce64) + a * T * T * abs(kl64)) + FTZ
    worst["loss"] = abs(float(loss) - loss64) / b_loss
    worst["ce"] = abs(float(out[0]) - ce64) / b_ce
    worst["kl"] = abs(float(out[1]) - kl64) / b_kl
    worst["inv_n"] = abs(float(inv_n) - inv64) / max(2 * 2.0 ** -22 * inv64, FTZ)
    assert torch.isfinite(lse3).all() and math.isfinite(float(loss))
    return worst


def report(name, worst):
    print(f"\n[distill] {name}: worst error/bound " + " ".join(f"{k}={v:.3f}" for k, v in worst.items()))


# ================================================================================================= kernels vs fp64
@pytest.mark.parametrize("a,T", [(0.5, 1.0), (0.25, 2.0), (1.0, 0.5)])
@pytest.mark.parametrize("V,Vp,pad", [(V, Vp, pad) for V, Vp in CE_SHAPES for pad in ((None, math.nan) if Vp > V else (None,))])
def test_kd_kernels_against_fp64(C, V, Vp, pad, a, T):
    """Labels at 0, V - 1 and the argmax, a row where the teacher equals the student; padding random or NaN in both tensors: out
    of every softmax and of the KL."""
    s, t, lab = _inputs(64, V, Vp, seed=V, pad=pad)
    worst = run_kd(C, s, t, lab, V, a, T, dloss=2.5)
    report(f"V={V}/{Vp} pad={pad} a={a} T={T}", worst)
    for k, v in worst.items():
        assert v <= 1.0, (k, v, worst)


@pytest.mark.parametrize("a,T", [(0.5, 1.0), (0.5, 2.0)])
def test_kd_kernels_llama3_microbatch(C, a, T):
    """T = 4096 rows of the Llama-3 vocabulary."""
    s, t, lab = _inputs(4096, 128256, 128256, seed=1)
    worst = run_kd(C, s, t, lab, 128256, a, T, rows=64)
    report(f"T=4096 V=128256 a={a} T={T}", worst)
    for k, v in worst.items():
        assert v <= 1.0, (k, v, worst)


@pytest.mark.parametrize("T", [1.0, 2.0])
def test_two_launches_are_bitwise_equal(C, T):
    s, t, lab = _inputs(512, 50257, 50304, seed=3)
    res = []
    for _ in range(2):
        out = torch.zeros(2, device=DEV)
        loss, inv_n, lse3 = C.kd_fwd(s, t, lab, 50257, -100, 0.5, T, out)
        g = s.clone()
        C.kd_bwd_inplace(g, t, lab, lse3, inv_n * 1.5, 50257, -100, 0.5, T)
        res.append((loss, inv_n, lse3, out, g.view(torch.int16)))
    for x, y in zip(*res):
        assert torch.equal(x, y)


def test_teacher_equal_to_student_on_the_gpu(C):
    """t == s: the KL is within its bound of 0 and the gradient is the plain CE gradient scaled by 1 - a, within the bounds."""
    s, _, lab = _inputs(64, 50257, 50304, seed=4)
    for T in (1.0, 2.0):
        worst = run_kd(C, s, s.clone(), lab, 50257, 0.25, T)
        assert max(worst.values()) <= 1.0, worst
        out = torch.zeros(2, device=DEV)
        C.kd_fwd(s, s.clone(), lab, 50257, -100, 0.25, T, out)
        assert abs(float(out[1])) <= 1e-5


def test_all_ignored_batch_is_pinned_to_zero(C):
    s, t, lab = _inputs(40, 1000, 1008, seed=2, pad=math.nan)
    lab[:] = -100
    out = torch.full((2,), math.nan, device=DEV)
    loss, inv_n, lse3 = C.kd_fwd(s, t, lab, 1000, -100, 0.5, 2.0, out)
    assert float(loss) == 0.0 and float(inv_n) == 0.0 and bool((out == 0).all()) and bool((lse3 == 0).all())
    g = s.clone()
    C.kd_bwd_inplace(g, t, lab, lse3, torch.ones(1, device=DEV) * inv_n, 1000, -100, 0.5, 2.0)
    assert bool((g == 0).all())


def test_bindings_reject_bad_arguments(C):
    s, t, lab = _inputs(8, 131, 136, seed=1)
    out = torch.zeros(2, device=DEV)
    for a in (0.0, -0.5, 1.5, math.nan):
        with pytest.raises(RuntimeError, match="alpha"):
            C.kd_fwd(s, t, lab, 131, -100, a, 1.0, out)
    for T in (0.0, -1.0, math.inf, math.nan, 1e300):
        with pytest.raises(RuntimeError, match="temperature"):
            C.kd_fwd(s, t, lab, 131, -100, 0.5, T, out)
    with pytest.raises(RuntimeError, match="teacher_logits"):
        C.kd_fwd(s, t[:4].contiguous(), lab, 131, -100, 0.5, 1.0, out)
    with pytest.raises(RuntimeError, match="padded vocab"):
        C.kd_fwd(s, t, lab, 137, -100, 0.5, 1.0, out)
    with pytest.raises(RuntimeError, match="padded vocab"):
        C.kd_fwd(s[:, :130].contiguous(), t[:, :130].contiguous(), lab, 130, -100, 0.5, 1.0, out)
    for bad in (torch.zeros(1, device=DEV), torch.zeros(2), torch.zeros(2, device=DEV, dtype=torch.float64)):
        with pytest.raises(RuntimeError, match="out"):
            C.kd_fwd(s, t, lab, 131, -100, 0.5, 1.0, bad)
    loss, inv_n, lse3 = C.kd_fwd(s, t, lab, 131, -100, 0.5, 1.0, out)
    with pytest.raises(RuntimeError, match="temperature"):
        C.kd_bwd_inplace(s.clone(), t, lab, lse3, inv_n, 131, -100, 0.5, 0.0)


# ================================================================================================= ops glue
def test_glue_scale_out_and_launch_counts():
    """``distill_cross_entropy`` scales the backward by ``dloss * inv_n``, writes (CE, KL), launches 2 + 1 kernels, and leaves the
    teacher logits as they were."""
    V, Vp = 50257, 50304
    s, t, lab = _inputs(300, V, Vp, seed=5)
    keep, t_keep = s.clone(), t.clone()
    x = s.clone().requires_grad_(True)
    out = torch.zeros(2, device=DEV)
    ops.reset_launch_counts()
    loss = ops.distill_cross_entropy(x * 1.0, t, lab, V, 0.5, 2.0, out=out)
    (loss * 3.0).backward()
    counts = ops.launch_counts()
    assert counts.get("kd_fwd") == 2 and counts.get("kd_bwd") == 1 and "ce_fwd" not in counts, counts
    assert torch.equal(t.view(torch.int16), t_keep.view(torch.int16))
    n = int((lab != -100).sum())
    o = kd_ref(keep.cpu(), t.cpu(), lab.cpu(), V, 0.5, 2.0)
    assert abs(float(loss) - o["loss"]) <= o["b_loss"] and abs(float(out[1]) - o["kl"]) <= o["b_kl"]
    for r0 in range(0, 300, 100):
        o = kd_ref(keep[r0:r0 + 100].cpu(), t[r0:r0 + 100].cpu(), lab[r0:r0 + 100].cpu(), V, 0.5, 2.0, scale=3.0 / n)
        assert ratio(x.grad[r0:r0 + 100].cpu(), o["grad"], o["b_grad"]) <= 1.0


# ================================================================================================= whole models
def _student(which):
    from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    if which == "llama":
        return LlamaForCausalLM(LlamaConfig(vocab_size=50257, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                                            num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=256))
    return GPTForCausalLM(GPTConfig(vocab_size=50257, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                                    max_position_embeddings=256, attention_layers="alternating", window_size=64))


def _teacher():
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(7)
    return LlamaForCausalLM(LlamaConfig(vocab_size=50257, hidden_size=384, intermediate_size=768, num_hidden_layers=2,
                                        num_attention_heads=6, max_position_embeddings=256, initializer_range=0.05))


@pytest.mark.parametrize("which", ["llama", "gptneo"])
def test_native_model_matches_the_torch_formula(which):
    """Same bf16 weights and batch, fwd + bwd with ``teacher_logits`` and through the formula in fp32 torch on the logits; parameter
    gradients agree to ``2^-6`` of their norm (each d-logit is the bf16 rounding of the same real number)."""
    m, teacher = _student(which).to(DEV, torch.bfloat16), _teacher().to(DEV, torch.bfloat16).requires_grad_(False)
    g = torch.Generator(device=DEV).manual_seed(3)
    ids = torch.randint(0, 50257, (4, 256), generator=g, device=DEV)
    labels = ids.clone()
    labels[1, 100:] = -100
    m.distill_alpha, m.distill_temperature, m.distill_out = 0.5, 2.0, torch.zeros(2, device=DEV)
    with torch.no_grad():
        tl = teacher.padded_logits(ids)
    loss = m(input_ids=ids, labels=labels, teacher_logits=tl)[0]
    loss.backward()
    got = {k: p.grad.float().clone() for k, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    logits = m(input_ids=ids).logits[:, :-1].reshape(-1, 50257).float()
    tv = tl.view(4, 256, -1)[:, :-1, :50257].reshape(-1, 50257).float()
    tgt = labels[:, 1:].reshape(-1)
    ref = formula(logits, tv, tgt, 0.5, 2.0)
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 2e-5 * abs(float(ref)), (float(loss), float(ref))
    for k, p in m.named_parameters():
        r = p.grad.float()
        assert float((got[k] - r).norm()) <= 2.0 ** -6 * float(r.norm()) + 1e-8, k
    assert all(p.grad is None for p in teacher.parameters())


def test_launches_of_one_micro_batch():
    """One distillation micro-batch = the student's CE micro-batch with the CE kernels replaced by one KD forward + reduce and one
    KD backward, plus exactly the launches of one no-grad teacher forward: no teacher backward."""
    m, teacher = _student("llama").to(DEV, torch.bfloat16), _teacher().to(DEV, torch.bfloat16).requires_grad_(False)
    ids = torch.randint(0, 50257, (2, 256), device=DEV)
    m.distill_out = torch.zeros(2, device=DEV)

    def counts(fn):
        fn()
        torch.cuda.synchronize()
        ops.reset_launch_counts()
        fn()
        torch.cuda.synchronize()
        return Counter(ops.launch_counts())

    def plain():
        m(input_ids=ids, labels=ids)[0].backward()

    def t_fwd():
        with torch.no_grad():
            teacher.padded_logits(ids)

    def kd():
        with torch.no_grad():
            tl = teacher.padded_logits(ids)
        m(input_ids=ids, labels=ids, teacher_logits=tl)[0].backward()

    c_plain, c_t, c_kd = counts(plain), counts(t_fwd), counts(kd)
    assert c_kd["kd_fwd"] == 2 and c_kd["kd_bwd"] == 1 and c_kd["ce_fwd"] == 0 and c_kd["ce_bwd"] == 0, c_kd
    want = c_plain + c_t + Counter(kd_fwd=2, kd_bwd=1)
    want.subtract(Counter(ce_fwd=2, ce_bwd=1))
    assert +want == +c_kd, (dict(want), dict(c_kd))


# ================================================================================================= trainer
_TRAINER_SCRIPT = r"""
import logging, sys, torch
sys.path.insert(0, {root!r})
from acco_b200 import AttrDict, DecoupledTrainer, ops
from acco_b200.callbacks import TrainerCallback
from acco_b200.data import ByteTokenizer, synthetic_pretrain_dataset, synthetic_sft_dataset
from acco_b200.launch import discover_env
from acco_b200.models import LlamaConfig, LlamaForCausalLM
cuda, variant, kd = sys.argv[1] == "cuda", sys.argv[3], sys.argv[4] == "1"
packing = variant == "packing"
L = 512 if packing else 128
cfg = LlamaConfig(vocab_size=1000, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                  num_key_value_heads=2, max_position_embeddings=L)
torch.manual_seed(0)
m = LlamaForCausalLM(cfg)
torch.manual_seed(5)
teacher = LlamaForCausalLM(LlamaConfig(vocab_size=1000, hidden_size=128, intermediate_size=256, num_hidden_layers=1, num_attention_heads=4,
                                       max_position_embeddings=L, initializer_range=0.1)) if kd else None
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
                max_grad_norm=0.5 if variant == "max_grad_norm" else None, distill_alpha=0.5, distill_temperature=2.0,
                static_accumulation=True, log_every=1)
env = discover_env()
env.id_run = "kd"
t = DecoupledTrainer(model=m, tokenizer=tok, train_dataset=ds, args=args, log=logging.getLogger("kd"), env=env, teacher=teacher)
logs = []
class Rec(TrainerCallback):
    def on_log(self, trainer, scalars):
        logs.append((scalars["loss"], scalars.get("distill_kl", -1.0), scalars.get("distill_ce", -1.0)))
t.add_callback(Rec())
t.train()
torch.save({{"logs": logs, "counts": (t.sched.count_grad_tot, t.sched.opt_steps), "cuda": t.is_cuda,
            "graphs": t._graphs is not None and len(t._graphs._graphs) > 0, "graphs_disabled": bool(getattr(t, "_graphs_disabled", None)),
            "launches": ops.launch_counts() if cuda else {{}}}}, sys.argv[2])
"""


def _train(tmp_path, dev, variant, kd):
    from acco_b200.launch import free_port
    script = tmp_path / "kd_train.py"
    script.write_text(_TRAINER_SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR")}
    env["MASTER_PORT"] = str(free_port())
    if dev == "cpu":
        env["CUDA_VISIBLE_DEVICES"] = ""
    out = tmp_path / f"{dev}_{variant}_{int(kd)}.pt"
    p = subprocess.run([sys.executable, str(script), dev, str(out), variant, "1" if kd else "0"], cwd=tmp_path, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:]
    return torch.load(out, weights_only=False)


@pytest.mark.parametrize("variant", ["plain", "packing", "document_mask", "fp8", "grad_accum_fp32", "max_grad_norm"])
def test_trainer_with_graphs_tracks_fp32_cpu_trainer(tmp_path, variant):
    """One GPU, ACCO, CUDA graphs, bf16, a random-weight teacher (a = 0.5, T = 2), against the fp32 CPU trainer with the same
    teacher.  The GPU run must capture graphs and keep them on and run the KD kernels; its logged loss and distill_kl must stay
    within bf16 training noise of the CPU ones (``plain``: and the CPU trace must be further from the run without a teacher)."""
    gpu, cpu = _train(tmp_path, "cuda", variant, True), _train(tmp_path, "cpu", variant, True)
    assert gpu["cuda"] and not cpu["cuda"]
    assert gpu["graphs"] and not gpu["graphs_disabled"], gpu
    assert gpu["launches"].get("kd_fwd", 0) > 0 and gpu["launches"].get("kd_bwd", 0) > 0 and not gpu["launches"].get("ce_fwd")
    if variant == "fp8":
        assert any(k.startswith("gemm_fp8") for k in gpu["launches"]), gpu["launches"]
    assert gpu["counts"] == cpu["counts"] and len(gpu["logs"]) == len(cpu["logs"]) >= 10
    a, b = torch.tensor(gpu["logs"]), torch.tensor(cpu["logs"])
    assert bool((a[:, 1] > 0).all()) and bool((a[:, 2] > 0).all())
    assert torch.allclose(a[:, 0], 0.5 * a[:, 2] + 0.5 * 4 * a[:, 1], rtol=1e-4)
    tol = 0.02 if variant == "fp8" else 0.01
    noise = float((a[:, 0] - b[:, 0]).abs().mean())
    assert noise <= tol * float(b[:, 0].abs().mean()), (variant, gpu["logs"], cpu["logs"])
    klnoise = float((a[:, 1] - b[:, 1]).abs().mean())
    assert klnoise <= 4 * tol * float(b[:, 1].abs().mean()) + 1e-4, (variant, gpu["logs"], cpu["logs"])
    if variant == "plain":
        off = _train(tmp_path, "cpu", variant, False)
        assert all(kl == -1.0 for _, kl, _ in off["logs"])
        plain = torch.tensor([x for x, _, _ in off["logs"]])
        assert float((b[:, 0] - plain).abs().mean()) > 2 * noise, (float((b[:, 0] - plain).abs().mean()), noise)


def test_logged_distill_kl_matches_the_batch(workdir):
    """A fixed device batch through the graphed micro-batch: the distill_kl / distill_ce the trainer copies to the host are the
    mean KL and CE of that batch under the weights it ran on, and loss = (1 - a) CE + a T^2 KL."""
    import logging
    import torch.nn.functional as F
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import synthetic_pretrain_dataset
    from acco_b200.launch import DistEnv
    m = _student("llama")
    ds = synthetic_pretrain_dataset(256, 200, 50257, 256, seed=0)
    args = AttrDict(method_name="acco", batch_size=4, max_length=256, nb_steps_tot=64, warmup=0, learning_rate=1e-3, save=False,
                    tensorboard=False, distill_alpha=0.25, distill_temperature=2.0)
    t = DecoupledTrainer(model=m, train_dataset=ds, args=args, log=logging.getLogger("kd"), env=DistEnv(id_run="kd"), teacher=_teacher())
    g = torch.Generator(device=DEV).manual_seed(5)
    batch = {"input_ids": torch.randint(0, 50257, (4, 256), generator=g, device=DEV)}
    t.input_override = lambda: batch
    for _ in range(3):
        t._drain()                  # nothing in flight: the next micro-batch runs on the weights bound now
        with torch.no_grad():
            s = t.model(**batch).logits[:, :-1].reshape(-1, 50257).float()
            tl = t.teacher(**batch).logits[:, :-1].reshape(-1, 50257).float()
        tgt = batch["input_ids"][:, 1:].reshape(-1)
        ce = float(F.cross_entropy(s, tgt))
        kl = float(F.kl_div(torch.log_softmax(s / 2, -1), torch.log_softmax(tl / 2, -1), reduction="batchmean", log_target=True))
        t.step()
        torch.cuda.synchronize()
        got_ce, got_kl = (float(v) for v in t.distill_host)
        assert t._graphs is not None and not getattr(t, "_graphs_disabled", None)
        assert abs(got_kl - kl) <= 1e-3 * kl + 1e-6, (got_kl, kl)
        assert abs(got_ce - ce) <= 1e-4 * ce, (got_ce, ce)
        assert abs(float(t.loss_host) - (0.75 * got_ce + 0.25 * 4 * got_kl)) <= 1e-5 * float(t.loss_host)
