#!/usr/bin/env python
"""Cost and effect of DPO (train key ``dpo_beta``) and of the reference-free SimPO (``simpo_beta``) and ORPO (``orpo_lambda``), three
ways:

(a) ``kernels``: device time of the DPO forward (``dpo_fwd`` + ``dpo_reduce``) and in-place backward against the plain CE forward and
    backward on the same rows, at 2P x S x Vp = 2 x 4 x 1024 x 50304 and x 128256; CUDA events over many launches, the arms
    alternated, medians.  On a response row the DPO forward reads both rows and the backward reads and writes the policy's: 8 bytes
    per logit (CE: 6); prompt and padding rows are only zeroed (2 bytes).  Achieved bytes/s are reported against HBM3's 3.35 TB/s.
    Also the time and extra peak memory of the unfused PyTorch formulation (TRL's ``log_softmax`` of fp32 copies of both logits,
    gather, ``logsigmoid``, autograd).  SimPO and ORPO (``ce_fwd`` + ``pref_reduce``, then ``dpo_bwd``) read the policy's row only:
    6 bytes per logit of a response row, like the CE.
(b) ``trainer``: ACCO tokens/s and peak allocated memory with CUDA graphs on one GPU, SFT (padded rows) against DPO on the same
    [8, 1024] rows (4 pairs), and SimPO and ORPO on the same rows (no reference model), Llama-125M and the Llama-3.2-1B shape; the
    arms alternated ``--repeats`` times, medians.
(c) ``effect``: a small native Llama trained with DPO (beta 0.1; the reference being its initial weights), SimPO (beta 2, gamma 0.5)
    or ORPO (lambda 0.1) on ``synthetic_preference_dataset`` for ``--effect-steps`` micro-batches of 8 pairs; eval loss and accuracy
    before and after.  It reports; it asserts nothing.

    python tools/dpo_bench.py [--only kernels,trainer,effect] [--arms dpo,simpo,orpo] [--out dpo_bench.json]

Prints the card name and power limit with the numbers.  Needs a GPU."""
import argparse
import gc
import json
import logging
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBPS = 3.35
P, S = 4, 1024


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _labels(V, dev, seed=0):
    import torch
    g = torch.Generator(device=dev).manual_seed(seed)
    tok = torch.randint(0, V, (2 * P, S), generator=g, device=dev)
    col = torch.arange(S, device=dev)[None, :]
    a = torch.randint(1, S // 2, (2 * P, 1), generator=g, device=dev)
    lab = torch.where(col >= a, tok, torch.full_like(tok, -100))
    out = torch.full_like(lab, -100)
    out[:, :-1] = lab[:, 1:]
    return lab, out.reshape(-1)


def bench_kernels(res, arms, iters=20):
    import torch
    import torch.nn.functional as F
    from acco_b200 import ops
    C = ops.load_ext(required=True)
    for V, Vp in ((50257, 50304), (128256, 128256)):
        T = 2 * P * S
        s0 = (3 * torch.randn(T, Vp, device="cuda")).to(torch.bfloat16)
        r = (s0.float() + 0.5 * torch.randn(T, Vp, device="cuda")).to(torch.bfloat16)
        lab2d, lb = _labels(V, "cuda")
        buf = s0.clone()
        out = torch.zeros(3, device="cuda")
        one = torch.ones(1, device="cuda")

        def dpo():
            loss, lse, w = C.dpo_fwd(buf, r, lb, P, V, -100, 0.1, out)
            C.dpo_bwd_inplace(buf, lb, lse, w, one, P, V, -100)

        def ce():
            loss, inv_n, lse = C.ce_fwd(buf, lb, V, -100, 0.0, 0.0, None)
            C.ce_bwd_inplace(buf, lb, lse, inv_n, V, -100, 0.0, 0.0)

        def pref(orpo, coef, gamma):
            def f():
                loss, lse, w = C.pref_fwd(buf, lb, P, V, -100, orpo, coef, gamma, out)
                C.dpo_bwd_inplace(buf, lb, lse, w, one, P, V, -100)
            return f

        fns = {"dpo": dpo, "ce": ce, "simpo": pref(False, 2.0, 0.5), "orpo": pref(True, 0.1, 0.0)}
        fns = {k: f for k, f in fns.items() if k == "ce" or k in arms}
        times = {k: [] for k in fns}
        for f in fns.values():
            buf.copy_(s0)
            f()
        for _ in range(5):
            for name, f in fns.items():
                buf.copy_(s0)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    f()
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) * 1e3 / iters)
        us = {k: statistics.median(v) for k, v in times.items()}
        # unfused: TRL's formulation on fp32 copies, forward + backward
        x = s0[:, :V].view(2 * P, S, V)
        ref = r[:, :V].view(2 * P, S, V)
        del buf
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

        def unfused():
            xs = x.detach().requires_grad_(True)
            lbs, mask = lab2d[:, 1:], lab2d[:, 1:] != -100
            idx = torch.where(mask, lbs, torch.zeros_like(lbs))[..., None]
            lp = lambda z: (torch.log_softmax(z[:, :-1].float(), -1).gather(-1, idx)[..., 0] * mask).sum(-1)
            with torch.no_grad():
                lr = lp(ref)
            lpp = lp(xs)
            zz = 0.1 * ((lpp[:P] - lr[:P]) - (lpp[P:] - lr[P:]))
            (-F.logsigmoid(zz)).mean().backward()
            return xs.grad

        un_ms = extra = None
        if "dpo" in arms:
            un_ms, extra = _time_unfused(unfused)
        # bytes moved: a response row is read twice (DPO: three times) and written once; a prompt / padding row is only zeroed
        row_bytes, valid = Vp * 2, int((lb != -100).sum())
        dpo_bytes, ce_bytes = (4 * valid + (T - valid)) * row_bytes, (3 * valid + (T - valid)) * row_bytes
        del s0, r, x, ref
        gc.collect()
        torch.cuda.empty_cache()
        print(json.dumps({f"kernels_{V}": _kernel_row(res, V, T, Vp, valid, us, dpo_bytes, ce_bytes, arms, un_ms, extra)}), flush=True)


def _time_unfused(unfused):
    """Time (ms) and extra peak memory (GiB) of the unfused PyTorch formulation, forward + backward."""
    import torch
    unfused()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        g = unfused()
        del g
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 3, (torch.cuda.max_memory_allocated() - base) / 2 ** 30


def _kernel_row(res, V, T, Vp, valid, us, dpo_bytes, ce_bytes, arms, un_ms, extra):
    r = {"rows": T, "response_rows": valid, "Vp": Vp}
    for k, t_us in us.items():
        nbytes = dpo_bytes if k == "dpo" else ce_bytes       # SimPO / ORPO move the CE's bytes: one policy row, no reference
        r[f"{k}_fwd_bwd_us"], r[f"{k}_TBps"] = round(t_us, 1), round(nbytes / t_us / 1e6, 2)
        if k != "ce":
            r[f"{k}_over_ce"] = round(t_us / us["ce"], 3)
    if "dpo" in arms:
        r.update(unfused_ms=round(un_ms, 2), unfused_extra_peak_GiB=round(extra, 2))
    res[f"kernels_{V}"] = r
    return r


def _make(shape):
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    if shape == "llama125m":
        cfg = LlamaConfig(vocab_size=50257, hidden_size=768, intermediate_size=2048, num_hidden_layers=12, num_attention_heads=12,
                          max_position_embeddings=S)
    else:
        cfg = LlamaConfig(vocab_size=128256, hidden_size=2048, intermediate_size=8192, num_hidden_layers=16, num_attention_heads=32,
                          num_key_value_heads=8, max_position_embeddings=S, tie_word_embeddings=True)
    return cfg, LlamaForCausalLM


ARM_KEYS = {"sft": {}, "dpo": {"dpo_beta": 0.1}, "simpo": {"simpo_beta": 2.0, "simpo_gamma": 0.5}, "orpo": {"orpo_lambda": 0.1}}


def _run_trainer(shape, arm, steps, warm):
    import torch
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.launch import DistEnv
    cfg, cls = _make(shape)
    torch.manual_seed(0)
    m = cls(cfg)
    ref = None
    if arm == "dpo":
        torch.manual_seed(0)
        ref = cls(cfg)
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, cfg.vocab_size, (2 * P, S), generator=g, device="cuda")
    lab2d, _ = _labels(cfg.vocab_size, "cuda")
    batch = {"input_ids": ids, "labels": torch.where(lab2d != -100, ids, lab2d)}
    args = AttrDict(method_name="acco", batch_size=2 * P if arm == "sft" else P, n_grad_accumulation=1, max_length=S,
                    nb_steps_tot=10 ** 9, warmup=0, learning_rate=1e-5, save=False, tensorboard=False, const_len_batch=False,
                    log_every=10 ** 9, **ARM_KEYS[arm])
    t = DecoupledTrainer(model=m, train_dataset=None, args=args, log=logging.getLogger("dpo_bench"), env=DistEnv(id_run="dpo_bench"),
                         reference=ref)
    t.input_override = lambda: batch
    for _ in range(warm):
        t.step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    mb0 = t.micro_batches
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        t.step()
    e1.record()
    torch.cuda.synchronize()
    sec = e0.elapsed_time(e1) / 1e3
    out = {"tokens_per_s": round((t.micro_batches - mb0) * 2 * P * S / sec), "peak_GiB": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
           "graphs": t._graphs is not None and not getattr(t, "_graphs_disabled", None)}
    t._drain()
    from acco_b200.launch import shutdown_distributed
    shutdown_distributed()
    del t, m, ref
    gc.collect()
    torch.cuda.empty_cache()
    return out


def bench_trainer(res, arms, shapes, repeats, steps, warm):
    for shape in shapes:
        runs = {arm: [] for arm in ["sft"] + arms}
        for _ in range(repeats):
            for arm in runs:
                runs[arm].append(_run_trainer(shape, arm, steps, warm))
        r = {arm: {"tokens_per_s": statistics.median(x["tokens_per_s"] for x in v), "peak_GiB": max(x["peak_GiB"] for x in v),
                   "graphs": all(x["graphs"] for x in v), "runs": [x["tokens_per_s"] for x in v]} for arm, v in runs.items()}
        for arm in arms:
            r[f"{arm}_over_sft"] = round(r[arm]["tokens_per_s"] / r["sft"]["tokens_per_s"], 3)
        res[f"trainer_{shape}"] = r
        print(json.dumps({f"trainer_{shape}": r}), flush=True)


def bench_effect(res, arm, steps):
    import torch
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import synthetic_preference_dataset
    from acco_b200.launch import DistEnv
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(vocab_size=4096, hidden_size=384, intermediate_size=1024, num_hidden_layers=4, num_attention_heads=6,
                      max_position_embeddings=256)
    torch.manual_seed(0)
    m = LlamaForCausalLM(cfg)
    ref = None
    if arm == "dpo":
        torch.manual_seed(0)
        ref = LlamaForCausalLM(cfg)
    full = synthetic_preference_dataset(4000, 200, 4095, seed=3).train_test_split(0.05, seed=42)
    args = AttrDict(method_name="acco", batch_size=8, max_length=256, nb_steps_tot=steps, warmup=10, learning_rate=1e-4, save=False,
                    tensorboard=False, const_len_batch=False, max_eval_batches=20, log_every=10 ** 9, seed=1, **ARM_KEYS[arm])
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            t = DecoupledTrainer(model=m, train_dataset=full["train"], eval_dataset=full["test"], args=args,
                                 log=logging.getLogger("dpo_bench"), env=DistEnv(id_run="dpo_effect"), reference=ref)
            acc = lambda: t.eval_dpo_accuracy if arm == "dpo" else t.eval_pref_accuracy
            before = (float(t.eval_loop()), acc())
            t.train()
            after = (float(t.eval_loop()), acc())
        finally:
            os.chdir(cwd)
    key = "effect" if arm == "dpo" else f"effect_{arm}"
    res[key] = {"micro_batches": steps, "pairs_per_micro_batch": 8, **ARM_KEYS[arm], "eval_loss_before": round(before[0], 4),
                f"eval_{arm}_accuracy_before": round(before[1], 3), "eval_loss_after": round(after[0], 4),
                f"eval_{arm}_accuracy_after": round(after[1], 3)}
    print(json.dumps({key: res[key]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="kernels,trainer,effect")
    ap.add_argument("--arms", default="dpo,simpo,orpo", help="preference objectives measured next to CE / SFT")
    ap.add_argument("--shapes", default="llama125m,llama3-1b", help="model shapes of the trainer measurement")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--effect-steps", type=int, default=400)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dpo_bench needs a GPU")
    os.environ.setdefault("ACCO_ALLOW_NCCL_FALLBACK", "1")
    res = {"gpu": gpu_info()}
    print(json.dumps(res), flush=True)
    only, arms = set(a.only.split(",")), [x for x in a.arms.split(",") if x]
    if not set(arms) <= {"dpo", "simpo", "orpo"}:
        raise SystemExit(f"--arms takes dpo, simpo and orpo, got {a.arms!r}")
    if "kernels" in only:
        bench_kernels(res, arms)
    if "trainer" in only:
        bench_trainer(res, arms, a.shapes.split(","), a.repeats, a.steps, a.warmup)
    if "effect" in only:
        for arm in arms:
            bench_effect(res, arm, a.effect_steps)
    res["gpu_after"] = gpu_info()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
