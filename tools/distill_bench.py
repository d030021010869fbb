#!/usr/bin/env python
"""Cost and effect of knowledge distillation (train key ``distill_teacher`` / ``DecoupledTrainer(teacher=...)``), three ways:

(a) ``kernels``: device time of the KD forward (``kd_fwd`` + ``kd_reduce``) and in-place backward against the plain CE forward
    and backward, at T x Vp = 8192 x 50304 (V = 50257) and 4096 x 128256, temperature 1 and 2; CUDA events over many launches,
    the arms alternated, medians.  The KD forward reads both rows, the backward reads both and writes the student's: 10 bytes per
    logit (CE: 6), reported against HBM3's 3.35 TB/s.  Also the time and peak memory of the unfused PyTorch formulation
    (``log_softmax`` of fp32 copies of both logits, autograd) at the same shapes.
(b) ``trainer``: ACCO tokens/s and peak allocated memory with CUDA graphs on one GPU, without and with a random-weight teacher:
    Llama-125M at 8 x 1024 (teacher: Llama-125M) and the Llama-3.2-1B shape at 4 x 1024 (teacher: the Llama-3-8B shape); the
    arms alternated ``--repeats`` times, medians.
(c) ``effect``: a Llama-125M teacher trained for ``--effect-steps`` micro-batches of 8 x 1024 ``synthetic_pretrain_dataset`` rows;
    then a smaller native Llama student (6 layers, width 384) trained for the same number of micro-batches on the same seed, without
    and with distillation (a = 0.5, T = 2); the eval cross-entropy of each on held-out rows.  It reports; it asserts nothing.

    python tools/distill_bench.py [--only kernels,trainer,effect] [--out distill_bench.json]

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
SEQ = 1024
ALPHA = 0.5


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def _unfused(s, t, lab, T):
    import torch
    import torch.nn.functional as F
    x = s.detach().requires_grad_(True)
    xf, tf = x.float(), t.float()
    loss = (1 - ALPHA) * F.cross_entropy(xf, lab) + ALPHA * T * T * F.kl_div(
        torch.log_softmax(xf / T, -1), torch.log_softmax(tf / T, -1), reduction="batchmean", log_target=True)
    loss.backward()


def bench_kernels(launches, samples):
    import torch
    from acco_b200 import ops
    C = ops.load_ext(required=True)
    out = []
    for Tn, V, Vp in ((8192, 50257, 50304), (4096, 128256, 128256)):
        g = torch.Generator(device="cuda").manual_seed(0)
        s = (2 * torch.randn(Tn, Vp, device="cuda", generator=g)).bfloat16()
        t = (3 * torch.randn(Tn, Vp, device="cuda", generator=g)).bfloat16()
        lab = torch.randint(0, V, (Tn,), device="cuda", generator=g)
        scratch = s.clone()                      # the backward overwrites its input; its cost does not depend on the values
        kd_out = torch.zeros(2, device="cuda")
        res = {"T": Tn, "V": V, "Vp": Vp}
        arms = {}
        _, inv_n, lse = C.ce_fwd(s, lab, V, -100)
        arms["ce"] = (lambda: C.ce_fwd(s, lab, V, -100),
                      lambda lse=lse, inv_n=inv_n: C.ce_bwd_inplace(scratch, lab, lse, inv_n, V, -100), 6)
        for T in (1.0, 2.0):
            _, inv_k, lse3 = C.kd_fwd(s, t, lab, V, -100, ALPHA, T, kd_out)
            arms[f"kd_T{T:g}"] = (lambda T=T: C.kd_fwd(s, t, lab, V, -100, ALPHA, T, kd_out),
                                  lambda T=T, lse3=lse3, inv_k=inv_k: C.kd_bwd_inplace(scratch, t, lab, lse3, inv_k, V, -100, ALPHA, T), 10)
        acc = {k: {"fwd": [], "bwd": []} for k in arms}
        for fwd, bwd, _ in arms.values():
            for _ in range(10):
                fwd(), bwd()
        torch.cuda.synchronize()
        for _ in range(samples):
            for k, (fwd, bwd, _) in arms.items():
                acc[k]["fwd"].append(timed(fwd, launches))
                acc[k]["bwd"].append(timed(bwd, launches))
        for k, (_, _, nbytes) in arms.items():
            f, b = statistics.median(acc[k]["fwd"]), statistics.median(acc[k]["bwd"])
            tbps = Tn * Vp * nbytes / ((f + b) * 1e-3) / 1e12
            res[k] = {"fwd_us": 1e3 * f, "bwd_us": 1e3 * b, "total_us": 1e3 * (f + b),
                      "total_min_max_us": [1e3 * (min(acc[k]["fwd"]) + min(acc[k]["bwd"])), 1e3 * (max(acc[k]["fwd"]) + max(acc[k]["bwd"]))],
                      "bytes_per_logit": nbytes, "TBps": tbps, "share_of_3.35_TBps": tbps / HBM_TBPS}
        for T in (1.0, 2.0):
            res[f"kd_T{T:g}_over_ce"] = res[f"kd_T{T:g}"]["total_us"] / res["ce"]["total_us"]
        # the unfused PyTorch formulation, fp32 copies of both logits and autograd
        for T in (1.0, 2.0):
            _unfused(s, t, lab, T)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            ms = statistics.median(timed(lambda: _unfused(s, t, lab, T), 3) for _ in range(3))
            res[f"unfused_T{T:g}"] = {"total_us": 1e3 * ms, "peak_extra_GB": (torch.cuda.max_memory_allocated() - base) / 1e9}
        kd_mem = {}
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        _, inv_k, lse3 = C.kd_fwd(s, t, lab, V, -100, ALPHA, 2.0, kd_out)
        C.kd_bwd_inplace(scratch, t, lab, lse3, inv_k, V, -100, ALPHA, 2.0)
        torch.cuda.synchronize()
        kd_mem["peak_extra_GB"] = (torch.cuda.max_memory_allocated() - base) / 1e9
        res["kd_T2_memory"] = kd_mem
        print(json.dumps(res), flush=True)
        out.append(res)
        del s, t, scratch
        torch.cuda.empty_cache()
    return out


def _trainer(student, teacher, B, ds, tag):
    import torch
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.launch import DistEnv
    from acco_b200.models import preset
    torch.manual_seed(0)
    model = preset(student, device="cuda", dtype=torch.bfloat16) if isinstance(student, str) else student
    t_model = None
    if teacher is not None:
        torch.manual_seed(1)
        t_model = preset(teacher, device="cuda", dtype=torch.bfloat16) if isinstance(teacher, str) else teacher
    args = AttrDict(method_name="acco", batch_size=B, n_grad_accumulation=1, max_length=SEQ, learning_rate=6e-4, weight_decay=0.1,
                    adam_beta1=0.9, adam_beta2=0.95, scheduler_name="cosine", warmup=100, nb_steps_tot=10 ** 12, use_mixed_precision=True,
                    const_len_batch=True, eval=False, save=False, tensorboard=False, seed=1, log_every=10 ** 9, distill_alpha=ALPHA,
                    distill_temperature=2.0)
    log = logging.getLogger("distill_bench")
    log.setLevel(logging.WARNING)
    return DecoupledTrainer(model=model, train_dataset=ds, args=args, log=log, env=DistEnv(id_run=tag), teacher=t_model)


def _close(t):
    """Stop the trainer's work; the caller drops its last reference and calls :func:`_free` (the trainer sits in reference cycles, so
    its memory returns only at a collection after that)."""
    t._drain()
    if t._feeder is not None:
        t._feeder.close()
    t.teacher = None


def _free():
    import torch
    gc.collect()
    torch.cuda.empty_cache()


def run_e2e(student, teacher, B, ds, warmup, micro):
    import torch
    torch.cuda.reset_peak_memory_stats()
    t = _trainer(student, teacher, B, ds, f"{student}-{teacher}")
    while t.micro_batches < warmup:
        t.step()
    torch.cuda.synchronize()
    m0 = t.micro_batches
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    while t.micro_batches < m0 + micro:
        t.step()
    e1.record()
    torch.cuda.synchronize()
    n = t.micro_batches - m0
    ms = e0.elapsed_time(e1) / n
    out = {"ms_per_micro_batch": ms, "tokens_per_s": B * SEQ / (ms * 1e-3), "peak_allocated_GB": torch.cuda.max_memory_allocated() / 1e9,
           "graphs": t._graphs is not None and not getattr(t, "_graphs_disabled", None),
           "distill_kl": float(t.distill_host[1]) if teacher else None}
    _close(t)
    del t
    _free()
    return out


def bench_trainer(repeats, warmup, micro):
    from acco_b200.data import synthetic_pretrain_dataset
    from acco_b200.models import PRESETS
    out = []
    for student, teacher, B in (("llama125m", "llama125m", 8), ("llama3-1b", "llama3-8b", 4)):
        V = PRESETS[student][1]["vocab_size"]
        ds = synthetic_pretrain_dataset(3000, 400, V, SEQ, seed=0)
        res = {"student": student, "teacher": teacher, "batch": B, "seq": SEQ, "runs": {"none": [], teacher: []}}
        for _ in range(repeats):
            for tch in (None, teacher):
                try:
                    r = run_e2e(student, tch, B, ds, warmup, micro)
                except RuntimeError as e:            # e.g. out of memory: reported, not hidden
                    r = {"error": f"{type(e).__name__}: {str(e)[:300]}"}
                    _free()
                res["runs"][tch or "none"].append(r)
                print(student, tch, json.dumps(r), flush=True)
        for k, v in res["runs"].items():
            ok = [r for r in v if "tokens_per_s" in r]
            if ok:
                res[f"{k}_median_tokens_per_s"] = statistics.median(r["tokens_per_s"] for r in ok)
                res[f"{k}_median_peak_GB"] = statistics.median(r["peak_allocated_GB"] for r in ok)
        out.append(res)
    return out


def bench_effect(steps, eval_batches=20):
    import torch
    import torch.nn.functional as F
    from acco_b200.data import stack_collate, synthetic_pretrain_dataset
    from acco_b200.models import PRESETS, LlamaConfig, LlamaForCausalLM
    V = PRESETS["llama125m"][1]["vocab_size"]
    B = 8
    n_rows = (steps + eval_batches + 2) * B
    ds = synthetic_pretrain_dataset(2 * n_rows * SEQ // 400, 400, V, SEQ, seed=0)
    assert len(ds) >= n_rows, len(ds)
    eval_ids = [stack_collate([ds[j] for j in range((steps + 1 + i) * B, (steps + 2 + i) * B)])["input_ids"].cuda()
                for i in range(eval_batches)]

    def train(model, teacher):
        t = _trainer(model, teacher, B, ds, "effect")
        k = [0]

        def nxt():
            i = k[0]
            k[0] += 1
            return {"input_ids": stack_collate([ds[j] for j in range(i * B, (i + 1) * B)])["input_ids"].cuda()}
        t.input_override = nxt
        while t.micro_batches < steps:
            t.step()
        t._drain()
        with torch.no_grad():
            ce = statistics.fmean(float(F.cross_entropy(t.model(input_ids=x).logits[:, :-1].reshape(-1, V).float(),
                                                        x[:, 1:].reshape(-1))) for x in eval_ids)
        trained = t.model
        _close(t)
        del t
        _free()
        return trained, ce

    def small():
        torch.manual_seed(3)
        return LlamaForCausalLM(LlamaConfig(vocab_size=V, hidden_size=384, intermediate_size=1024, num_hidden_layers=6, num_attention_heads=6,
                                            max_position_embeddings=SEQ)).to("cuda", torch.bfloat16)
    out = {"teacher": "llama125m", "student": "llama 6 x 384", "batch": B, "seq": SEQ, "micro_batches": steps, "alpha": ALPHA,
           "temperature": 2.0, "eval_rows": eval_batches * B}
    teacher, out["teacher_eval_ce"] = train("llama125m", None)
    teacher.requires_grad_(False)
    _, out["student_eval_ce_without"] = train(small(), None)
    _, out["student_eval_ce_with"] = train(small(), teacher)
    print("effect", json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="kernels,trainer,effect")
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--samples", type=int, default=7)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=10, help="micro-batches before the timed window")
    ap.add_argument("--micro", type=int, default=30, help="micro-batches in the timed window")
    ap.add_argument("--effect-steps", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("distill_bench needs a GPU")
    os.environ.setdefault("ACCO_ALLOW_NCCL_FALLBACK", "1")
    parts = a.only.split(",")
    rep = {"gpu": gpu_info(), "alpha": ALPHA}
    print("GPU:", rep["gpu"], flush=True)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)                            # the trainer writes nothing here with save / tensorboard off; keep the tree clean anyway
        try:
            if "kernels" in parts:
                rep["kernels"] = bench_kernels(a.launches, a.samples)
            if "trainer" in parts:
                rep["trainer"] = bench_trainer(a.repeats, a.warmup, a.micro)
            if "effect" in parts:
                rep["effect"] = bench_effect(a.effect_steps)
        finally:
            os.chdir(cwd)
    rep["gpu_after"] = gpu_info()
    print(json.dumps(rep))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
