#!/usr/bin/env python
"""Cost of label smoothing (train key ``label_smoothing_factor``) on the native models, three ways:

(a) ``kernels``: device time of the cross-entropy forward (``ce_fwd`` + ``ce_reduce``) and in-place backward at eps = 0 and eps = 0.1,
    T x Vp = 8192 x 50304 (V = 50257) and 4096 x 128256; CUDA events over many launches, the two arms alternated.  The forward
    reads the logits once, the backward reads and writes them: 6 bytes per logit in all.
(b) ``microbatch``: one training micro-batch (forward + backward into ``.grad``) of Llama-125M at 8 x 1024 and of the Llama-3.2-1B
    preset at 4 x 1024 with eps = 0.1, on the fused route (``model.label_smoothing``) and on the ``LabelSmoother`` route the trainer
    takes for non-native models (forced by wrapping the model), eager and replayed from a CUDA graph.  Reports time and the peak of
    ``torch.cuda.max_memory_allocated`` above what was allocated before the micro-batch.
(c) ``trainer``: acco-ft tokens/s (Llama-125M, micro-batches of 4 x 512 padded SFT rows, 2 per half-round, ACCO, one GPU) with
    eps = 0.1, fused route vs ``LabelSmoother`` route.  Tokens are the padded ones the trainer counts.

    python tools/label_smoothing_bench.py [--only kernels,microbatch,trainer] [--out label_smoothing_bench.json]

Prints the card name and power limit with the numbers.  Needs a GPU."""
import argparse
import json
import logging
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

EPS = 0.1


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


def bench_kernels(launches, samples):
    import torch
    from acco_b200 import ops
    C = ops.load_ext(required=True)
    out = []
    for T, V, Vp in ((8192, 50257, 50304), (4096, 128256, 128256)):
        g = torch.Generator(device="cuda").manual_seed(0)
        lg = (2 * torch.randn(T, Vp, device="cuda", generator=g)).bfloat16()
        lab = torch.randint(0, V, (T,), device="cuda", generator=g)
        scratch = lg.clone()                     # the backward overwrites its input; its cost does not depend on the values
        res = {"T": T, "V": V, "Vp": Vp}
        ms = {}
        for eps in (0.0, EPS):
            _, inv_n, lse = C.ce_fwd(lg, lab, V, -100, eps)
            fwd = lambda eps=eps: C.ce_fwd(lg, lab, V, -100, eps)
            bwd = lambda eps=eps, lse=lse, inv_n=inv_n: C.ce_bwd_inplace(scratch, lab, lse, inv_n, V, -100, eps)
            for _ in range(10):
                fwd(), bwd()
            ms[eps] = (fwd, bwd, {"fwd": [], "bwd": []})
        torch.cuda.synchronize()
        for _ in range(samples):
            for eps, (fwd, bwd, acc) in ms.items():
                acc["fwd"].append(timed(fwd, launches))
                acc["bwd"].append(timed(bwd, launches))
        for eps, (_, _, acc) in ms.items():
            f, b = statistics.median(acc["fwd"]), statistics.median(acc["bwd"])
            res[f"eps={eps}"] = {"fwd_us": 1e3 * f, "bwd_us": 1e3 * b, "total_us": 1e3 * (f + b),
                                 "fwd_min_max_us": [1e3 * min(acc["fwd"]), 1e3 * max(acc["fwd"])],
                                 "bwd_min_max_us": [1e3 * min(acc["bwd"]), 1e3 * max(acc["bwd"])],
                                 "TBps": T * Vp * 6 / ((f + b) * 1e-3) / 1e12}
        res["smoothed_over_plain_pct"] = 100.0 * (res[f"eps={EPS}"]["total_us"] / res["eps=0.0"]["total_us"] - 1.0)
        out.append(res)
        del lg, scratch
        torch.cuda.empty_cache()
    return out


class Wrapped:
    """Builds a non-native view of a native model: logits only, so the loss goes through ``LabelSmoother`` (the trainer's route
    for HF-style models)."""

    @staticmethod
    def make(m):
        import torch

        class _W(torch.nn.Module):
            def __init__(self):
                super().__init__()
                self.m = m

            def forward(self, input_ids=None, labels=None, attention_mask=None, **kw):
                return {"logits": self.m(input_ids=input_ids).logits}
        return _W()


def bench_microbatch(iters, samples):
    import torch
    from acco_b200.models import preset
    from acco_b200.utils.misc import LabelSmoother
    out = []
    for name, B, S in (("llama125m", 8, 1024), ("llama3-1b", 4, 1024)):
        torch.manual_seed(0)
        m = preset(name, device=torch.device("cuda"), dtype=torch.bfloat16)
        V = m.config.vocab_size
        ids = torch.randint(0, V, (B, S), device="cuda")
        labels = ids.clone()
        smoother = LabelSmoother(EPS)

        def fused():
            m.label_smoothing = EPS
            loss = m(input_ids=ids, labels=labels)[0]
            loss.backward()
            return loss

        def old():
            m.label_smoothing = 0.0
            loss = smoother({"logits": m(input_ids=ids).logits}, labels, shift_labels=True)
            loss.backward()
            return loss

        res = {"model": name, "B": B, "S": S, "V": V}
        for route, fn in (("fused", fused), ("label_smoother", old)):
            for p in m.parameters():
                p.grad = None
            fn()                                        # allocates .grad
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            fn()
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
            eager = statistics.median(timed(fn, iters) for _ in range(samples))
            r = {"eager_ms": eager, "peak_extra_GiB": peak / 2 ** 30}
            try:
                st = torch.cuda.Stream()
                st.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(st):
                    for _ in range(3):
                        fn()
                torch.cuda.current_stream().wait_stream(st)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    fn()
                r["graph_ms"] = statistics.median(timed(graph.replay, iters) for _ in range(samples))
                del graph
            except Exception as e:                      # report, do not hide: a route that cannot be captured is a finding
                r["graph_ms"] = f"capture failed: {type(e).__name__}: {str(e)[:200]}"
            res[route] = r
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
        f, o = res["fused"], res["label_smoother"]
        res["memory_saved_GiB"] = o["peak_extra_GiB"] - f["peak_extra_GiB"]
        res["eager_saved_pct"] = 100.0 * (1.0 - f["eager_ms"] / o["eager_ms"])
        out.append(res)
        del m
        torch.cuda.empty_cache()
    return out


def bench_trainer(steps, warmup):
    import torch
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import ByteTokenizer, synthetic_sft_dataset
    from acco_b200.launch import DistEnv, shutdown_distributed
    from acco_b200.models import preset
    os.environ.setdefault("ACCO_ALLOW_NCCL_FALLBACK", "1")
    out = {}
    for route in ("fused", "label_smoother", "fused", "label_smoother"):
        torch.manual_seed(0)
        m = preset("llama125m", dtype=torch.float32)
        V = m.config.vocab_size
        model = m if route == "fused" else Wrapped.make(m)
        tok = ByteTokenizer()
        tok.pad_token_id = tok.eos_token_id = V - 1
        ds = synthetic_sft_dataset(4000, 300, V - 1, 512, seed=1)
        args = AttrDict(method_name="acco", batch_size=4, n_grad_accumulation=2, max_length=512, nb_steps_tot=100000, warmup=0,
                        learning_rate=2e-5, adam_beta2=0.95, scheduler_name="cosine", save=False, tensorboard=False, const_len_batch=False,
                        use_mixed_precision=True, label_smoothing_factor=EPS, seed=1, log_every=10 ** 9)
        cwd = os.getcwd()
        with tempfile.TemporaryDirectory() as tmp:
            os.chdir(tmp)
            try:
                t = DecoupledTrainer(model=model, tokenizer=tok, train_dataset=ds, args=args, log=logging.getLogger("lsb"),
                                     env=DistEnv(id_run="lsb"))
                for _ in range(warmup):
                    t.step()
                torch.cuda.synchronize()
                tok0, t0 = t._tokens_seen, time.perf_counter()
                for _ in range(steps):
                    t.step()
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                tps = (t._tokens_seen - tok0) / dt
                graphs = t._use_graphs()
                t._drain()
            finally:
                os.chdir(cwd)
                shutdown_distributed()
        out.setdefault(route, {"tokens_per_s": [], "graphs": graphs})["tokens_per_s"].append(tps)
        del t, model, m
        torch.cuda.empty_cache()
    for r in out.values():
        r["median_tokens_per_s"] = statistics.median(r["tokens_per_s"])
    out["fused_over_label_smoother_pct"] = 100.0 * (out["fused"]["median_tokens_per_s"] / out["label_smoother"]["median_tokens_per_s"] - 1.0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="kernels,microbatch,trainer")
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--samples", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("label_smoothing_bench needs a GPU")
    parts = a.only.split(",")
    rep = {"gpu": gpu_info(), "eps": EPS}
    print("GPU:", rep["gpu"], flush=True)
    if "kernels" in parts:
        rep["kernels"] = bench_kernels(a.launches, a.samples)
        print(json.dumps(rep["kernels"], indent=1), flush=True)
    if "microbatch" in parts:
        rep["microbatch"] = bench_microbatch(a.iters, a.samples)
        print(json.dumps(rep["microbatch"], indent=1), flush=True)
    if "trainer" in parts:
        rep["trainer"] = bench_trainer(a.steps, a.warmup)
        print(json.dumps(rep["trainer"], indent=1), flush=True)
    print(json.dumps(rep))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
