#!/usr/bin/env python
"""Cost and effect of DPO (train key ``dpo_beta``), three ways:

(a) ``kernels``: device time of the DPO forward (``dpo_fwd`` + ``dpo_reduce``) and in-place backward against the plain CE forward and
    backward on the same rows, at 2P x S x Vp = 2 x 4 x 1024 x 50304 and x 128256; CUDA events over many launches, the arms
    alternated, medians.  On a response row the DPO forward reads both rows and the backward reads and writes the policy's: 8 bytes
    per logit (CE: 6); prompt and padding rows are only zeroed (2 bytes).  Achieved bytes/s are reported against HBM3's 3.35 TB/s.
    Also the time and extra peak memory of the unfused PyTorch formulation (TRL's ``log_softmax`` of fp32 copies of both logits,
    gather, ``logsigmoid``, autograd).
(b) ``trainer``: ACCO tokens/s and peak allocated memory with CUDA graphs on one GPU, SFT (padded rows) against DPO on the same
    [8, 1024] rows (4 pairs), Llama-125M and the Llama-3.2-1B shape; the arms alternated ``--repeats`` times, medians.
(c) ``effect``: a small native Llama trained with DPO (beta 0.1) on ``synthetic_preference_dataset`` for ``--effect-steps``
    micro-batches of 8 pairs, the reference being its initial weights; eval ``dpo_accuracy`` before and after.  It reports; it
    asserts nothing.

    python tools/dpo_bench.py [--only kernels,trainer,effect] [--out dpo_bench.json]

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


def bench_kernels(res, iters=20):
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

        times = {"dpo": [], "ce": []}
        for f in (dpo, ce):
            buf.copy_(s0)
            f()
        for _ in range(5):
            for name, f in (("dpo", dpo), ("ce", ce)):
                buf.copy_(s0)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    f()
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) * 1e3 / iters)
        dpo_us, ce_us = statistics.median(times["dpo"]), statistics.median(times["ce"])
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
        un_ms = e0.elapsed_time(e1) / 3
        extra = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
        # bytes moved: a response row is read twice (DPO: three times) and written once; a prompt / padding row is only zeroed
        row_bytes, valid = Vp * 2, int((lb != -100).sum())
        dpo_bytes, ce_bytes = (4 * valid + (T - valid)) * row_bytes, (3 * valid + (T - valid)) * row_bytes
        res[f"kernels_{V}"] = {"rows": T, "response_rows": valid, "Vp": Vp, "dpo_fwd_bwd_us": round(dpo_us, 1),
                               "ce_fwd_bwd_us": round(ce_us, 1), "dpo_over_ce": round(dpo_us / ce_us, 3),
                               "dpo_TBps": round(dpo_bytes / dpo_us / 1e6, 2), "ce_TBps": round(ce_bytes / ce_us / 1e6, 2),
                               "unfused_ms": round(un_ms, 2),
                               "unfused_extra_peak_GiB": round(extra, 2)}
        print(json.dumps({f"kernels_{V}": res[f"kernels_{V}"]}), flush=True)
        del s0, r, x, ref
        gc.collect()
        torch.cuda.empty_cache()


def _make(shape):
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    if shape == "llama125m":
        cfg = LlamaConfig(vocab_size=50257, hidden_size=768, intermediate_size=2048, num_hidden_layers=12, num_attention_heads=12,
                          max_position_embeddings=S)
    else:
        cfg = LlamaConfig(vocab_size=128256, hidden_size=2048, intermediate_size=8192, num_hidden_layers=16, num_attention_heads=32,
                          num_key_value_heads=8, max_position_embeddings=S, tie_word_embeddings=True)
    return cfg, LlamaForCausalLM


def _run_trainer(shape, dpo, steps, warm):
    import torch
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.launch import DistEnv
    cfg, cls = _make(shape)
    torch.manual_seed(0)
    m = cls(cfg)
    ref = None
    if dpo:
        torch.manual_seed(0)
        ref = cls(cfg)
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, cfg.vocab_size, (2 * P, S), generator=g, device="cuda")
    lab2d, _ = _labels(cfg.vocab_size, "cuda")
    batch = {"input_ids": ids, "labels": torch.where(lab2d != -100, ids, lab2d)}
    args = AttrDict(method_name="acco", batch_size=P if dpo else 2 * P, n_grad_accumulation=1, max_length=S, nb_steps_tot=10 ** 9,
                    warmup=0, learning_rate=1e-5, save=False, tensorboard=False, const_len_batch=False, dpo_beta=0.1 if dpo else None,
                    log_every=10 ** 9)
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


def bench_trainer(res, repeats, steps, warm):
    for shape in ("llama125m", "llama3-1b"):
        runs = {"sft": [], "dpo": []}
        for _ in range(repeats):
            for arm in ("sft", "dpo"):
                runs[arm].append(_run_trainer(shape, arm == "dpo", steps, warm))
        r = {arm: {"tokens_per_s": statistics.median(x["tokens_per_s"] for x in v), "peak_GiB": max(x["peak_GiB"] for x in v),
                   "graphs": all(x["graphs"] for x in v), "runs": [x["tokens_per_s"] for x in v]} for arm, v in runs.items()}
        r["dpo_over_sft"] = round(r["dpo"]["tokens_per_s"] / r["sft"]["tokens_per_s"], 3)
        res[f"trainer_{shape}"] = r
        print(json.dumps({f"trainer_{shape}": r}), flush=True)


def bench_effect(res, steps):
    import torch
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import synthetic_preference_dataset
    from acco_b200.launch import DistEnv
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(vocab_size=4096, hidden_size=384, intermediate_size=1024, num_hidden_layers=4, num_attention_heads=6,
                      max_position_embeddings=256)
    torch.manual_seed(0)
    m = LlamaForCausalLM(cfg)
    torch.manual_seed(0)
    ref = LlamaForCausalLM(cfg)
    full = synthetic_preference_dataset(4000, 200, 4095, seed=3).train_test_split(0.05, seed=42)
    args = AttrDict(method_name="acco", batch_size=8, max_length=256, nb_steps_tot=steps, warmup=10, learning_rate=1e-4, save=False,
                    tensorboard=False, const_len_batch=False, dpo_beta=0.1, max_eval_batches=20, log_every=10 ** 9, seed=1)
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            t = DecoupledTrainer(model=m, train_dataset=full["train"], eval_dataset=full["test"], args=args,
                                 log=logging.getLogger("dpo_bench"), env=DistEnv(id_run="dpo_effect"), reference=ref)
            before = (float(t.eval_loop()), t.eval_dpo_accuracy)
            t.train()
            after = (float(t.eval_loop()), t.eval_dpo_accuracy)
        finally:
            os.chdir(cwd)
    res["effect"] = {"micro_batches": steps, "pairs_per_micro_batch": 8, "eval_loss_before": round(before[0], 4),
                     "eval_dpo_accuracy_before": round(before[1], 3), "eval_loss_after": round(after[0], 4),
                     "eval_dpo_accuracy_after": round(after[1], 3)}
    print(json.dumps({"effect": res["effect"]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="kernels,trainer,effect")
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
    only = set(a.only.split(","))
    if "kernels" in only:
        bench_kernels(res)
    if "trainer" in only:
        bench_trainer(res, a.repeats, a.steps, a.warmup)
    if "effect" in only:
        bench_effect(res, a.effect_steps)
    res["gpu_after"] = gpu_info()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
