#!/usr/bin/env python
"""Multi-GPU check + micro-benchmark of KERNEL A (fused RS + AdamW + AG) against the NCCL library path.

    torchrun --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tools/symm_check.py --numel 20000000

For every transport available (p2p, multimem) it runs an ACCO round sequence (tentative / real /
tentative / real ...) on rank-specific random gradients with rank-specific micro-batch counts, on
BOTH backends, and after every round checks: identical global counts; fp32 master / Adam state /
stash agree with the NCCL+fused-local-AdamW path within bf16-reduction tolerance; the gathered
parameters are bit-identical on all ranks; the consumed accumulator is zero.  Then it times the
round (CUDA events, max over ranks) and reports achieved NVLink bytes/s and the HBM floor.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch
import torch.distributed as dist
import torch.nn as nn

from acco_b200.launch import discover_env, init_distributed
from acco_b200.optim import ShardedAdamW
from acco_b200.parallel.arena import FlatArena
from acco_b200.parallel.backend import TorchDistBackend
from acco_b200.parallel.schedule import RoundScheduler
from acco_b200.ops import fused_adamw_shard


class Flat(nn.Module):
    def __init__(self, n):
        super().__init__()
        self.w = nn.Parameter(torch.empty(n))


def build(kind, n, env, dev, mode_env=None):
    if mode_env:
        os.environ["ACCO_SYMM_MODE"] = mode_env
    torch.manual_seed(0)
    m = Flat(n)
    with torch.no_grad():
        m.w.normal_(0, 0.02)
    m.to(dev, torch.bfloat16)
    if kind == "symm":
        from acco_b200.parallel.symm import SymmBackend
        be = SymmBackend(env.rank, env.world_size, dev)
    else:
        be = TorchDistBackend(env.rank, env.world_size, dev, fused_adam=fused_adamw_shard)
    ar = FlatArena(m, env.world_size, env.rank, torch.bfloat16, dev, align=1024, allocator=be.allocator())
    opt = ShardedAdamW(ar.shard(ar.theta[0]), lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1)
    be.attach(ar, opt)
    return be, ar, opt


def fill_grads(ar, idx, rnd, rank):
    g = torch.Generator(device=ar.device).manual_seed(1000 * rnd + rank)
    ar.acc[idx].copy_((torch.randn(ar.layout.padded, generator=g, device=ar.device) * 0.01).to(torch.bfloat16))
    ar.acc[idx][ar.numel:].zero_()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--numel", type=int, default=20_000_003)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--bench-numel", type=int, default=123_587_328)
    ap.add_argument("--bench-iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--grids", default="", help="comma list of CTA counts to sweep for the fused kernel (0 = default)")
    a = ap.parse_args()
    env = init_distributed(discover_env())
    dev = torch.device("cuda", env.local_rank)
    W, rank = env.world_size, env.rank
    report = {"world": W, "numel": a.numel, "modes": {}}
    ref_be, ref_ar, ref_opt = build("nccl", a.numel, env, dev)
    modes = ["p2p", "multimem"]
    for mode in modes:
        try:
            be, ar, opt = build("symm", a.numel, env, dev, mode_env=mode)
        except Exception as e:
            report["modes"][mode] = {"available": False, "why": f"{type(e).__name__}: {str(e)[:200]}"}
            continue
        # fresh reference state
        ref_be, ref_ar, ref_opt = build("nccl", a.numel, env, dev)
        import dataclasses
        from acco_b200.optim import adamw_shard_update_
        s1, s2 = RoundScheduler("acco"), RoundScheduler("acco")
        ok, worst = True, {}
        # the oracle optimizer: same initial state; every round it is fed THE KERNEL'S OWN reduced gradient (read back from the stash,
        # which the validation plans make every round write), so master / m / v / theta must then agree to fp32 round-off on BOTH
        # transports - no "Adam amplifies a 1-ulp difference" escape hatch.  The reduced gradient itself is checked separately,
        # element-wise, against the exact fp32 sum of the ranks' bf16 gradients.
        oracle = ShardedAdamW(ar.shard(ar.theta[0]).clone(), lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1)
        oracle_stash_count = 0
        prev_stash = torch.zeros_like(opt.stash)
        for r in range(a.rounds):
            p1, p2 = s1.next_plan(), s2.next_plan()
            p1v = dataclasses.replace(p1, write_stash=True)          # validation: the gradient the update used lands in the stash
            for arena in (ar, ref_ar):
                fill_grads(arena, p1.read_acc, r, rank)
            cnt = 1 + (rank + r) % 3
            lr = 1e-3 * (1 + r)
            be.launch_round(p1v, lr, cnt)
            ref_be.launch_round(p2, lr, cnt)
            torch.cuda.synchronize()
            t1, t2 = be.finish_round(p1v), ref_be.finish_round(p2)
            s1.complete(p1, t1)
            s2.complete(p2, t2)
            S = ar.layout.size_slice
            lo_, hi_ = rank * S, (rank + 1) * S
            # ---- (1) the reduction: exact fp32 sum of every rank's bf16 gradient for MY slice
            exact = torch.zeros(S, device=dev, dtype=torch.float64)
            mag = torch.zeros(S, device=dev, dtype=torch.float32)
            for q in range(W):
                gq = torch.Generator(device=dev).manual_seed(1000 * r + q)
                full = (torch.randn(ar.layout.padded, generator=gq, device=dev) * 0.01).to(torch.bfloat16)
                full[ar.numel:].zero_()
                exact += full[lo_:hi_].double()
                mag += full[lo_:hi_].float().abs()
            exact = exact.float()                                      # sum of W bf16 values: exact in fp64, one rounding to fp32
            used = opt.stash.clone()                                   # gradient the kernel fed to AdamW this round
            base_prev = prev_stash if p1.add_stash else torch.zeros_like(prev_stash)
            if mode == "multimem":
                # the switch adds in fp32 and returns bf16: the result must be one of the two bf16 neighbours of the exact sum
                bits = exact.view(torch.int32)
                toward0 = (bits & -65536).view(torch.float32)
                away0 = ((bits & -65536) + 65536).view(torch.float32)
                cands = (base_prev + toward0, base_prev + away0, base_prev + exact.to(torch.bfloat16).float())
                hit = (used == cands[0]) | (used == cands[1]) | (used == cands[2])
                red_bad = int((~hit).sum().item())
                red_err = float(((used - base_prev) - exact).abs().max())
            else:
                # p2p: fp32 accumulation of 8 bf16 values in registers - exact up to fp32 summation order
                red_err = float((used - (base_prev + exact)).abs().max())
                # (tolerance relative to the magnitude of the TERMS: the sum itself may cancel to ~0)
                red_bad = int(((used - (base_prev + exact)).abs() > 2e-7 * (mag + base_prev.abs()) + 1e-12).sum().item())
            prev_stash = used
            # ---- (2) the update: oracle AdamW on the kernel's own reduced gradient
            tot_cnt = sum(1 + (q + r) % 3 for q in range(W))
            upd_cnt = tot_cnt + (oracle_stash_count if p1.add_stash else 0)
            o_plan = dataclasses.replace(p1, add_stash=False, write_stash=False)
            hp = oracle.hyper(lr, o_plan, 1.0 / upd_cnt)
            o_out = torch.empty(S, device=dev, dtype=torch.bfloat16)
            adamw_shard_update_(used, oracle.master, oracle.exp_avg, oracle.exp_avg_sq, torch.zeros_like(used), o_out, hp)
            oracle.after_launch(p1)
            if p1.write_stash:
                oracle_stash_count = tot_cnt
            mine = ar.theta[p1.write_theta][lo_:hi_]
            theta_mismatch = (mine != o_out)
            # tolerance of the pushed bf16 weight: one bf16 ulp of the value (the fp32 results agree to ~1e-8, which decides the
            # rounding direction for ~1e-4 of the elements) plus that fp32 slack for weights that are themselves ~0
            ulp = o_out.float().abs() * 2.0 ** -7 + 1e-7
            errs = {
                "count": abs(t1 - upd_cnt),
                "count_vs_nccl": abs(t1 - t2),
                "reduced_grad_bad_elements": red_bad,
                "reduced_grad_max_abs_err": red_err,
                "master": float((opt.master - oracle.master).abs().max()),
                "exp_avg": float((opt.exp_avg - oracle.exp_avg).abs().max()),
                "exp_avg_sq": float((opt.exp_avg_sq - oracle.exp_avg_sq).abs().max()),
                "theta_frac_not_bit_identical": float(theta_mismatch.float().mean()),
                "theta_max_err_in_ulps": float(((mine.float() - o_out.float()).abs() / ulp).max()),
                "master_vs_nccl": float((opt.master - ref_opt.master).abs().max()),
                "theta_vs_nccl": float((ar.theta[p1.write_theta].float() - ref_ar.theta[p2.write_theta].float()).abs().max()),
                "acc_left": float(ar.acc[p1.read_acc].float().abs().max()),
            }
            chk = ar.theta[p1.write_theta].view(torch.int16).to(torch.int64).sum().reshape(1)
            lo, hi = chk.clone(), chk.clone()
            dist.all_reduce(lo, op=dist.ReduceOp.MIN)
            dist.all_reduce(hi, op=dist.ReduceOp.MAX)
            errs["rank_divergence"] = int((hi - lo).item())
            for k, v in errs.items():
                worst[k] = max(worst.get(k, 0), v)
            # gates (identical for both transports): counts exact; every reduced element exact (p2p) / a bf16 neighbour of the exact
            # sum (multimem); optimizer state equal to the oracle's to fp32 round-off (fast-math sqrt / div in the kernel); the pushed
            # bf16 weights bit-identical except where the fp32 value sits on a rounding boundary (<= 1 ulp, < 0.1 % of elements);
            # all ranks hold bit-identical gathered weights; the consumed accumulator is zero.  *_vs_nccl is informational only
            # (NCCL reduces in bf16 around a ring).
            mscale = float(oracle.master.abs().max())
            good = (errs["count"] == 0 and errs["count_vs_nccl"] == 0 and errs["rank_divergence"] == 0 and errs["acc_left"] == 0
                    and errs["reduced_grad_bad_elements"] == 0
                    and errs["master"] <= 4e-6 * max(mscale, 1e-2) and errs["exp_avg"] <= 1e-7 and errs["exp_avg_sq"] <= 1e-9
                    and errs["theta_max_err_in_ulps"] <= 1.01 and errs["theta_frac_not_bit_identical"] < 1e-3)
            ok = ok and good
        flag = torch.tensor([1 if ok else 0], device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        report["modes"][mode] = {"available": True, "backend": be.name, "ok": bool(flag.item()), "worst": worst}
        del be, ar, opt
        torch.cuda.empty_cache()

    # ------------------------------------------------------------------ timing
    n = a.bench_numel
    grids = [int(g) for g in a.grids.split(",")] if a.grids else [0]
    combos = [("nccl", None, 0)] + [("symm", m, g) for m in ("p2p", "multimem") for g in grids]
    for kind, mode, grid in combos:
        key = (mode or "nccl") + (f"@grid{grid}" if grid else "")
        os.environ["ACCO_ROUND_GRID"] = str(grid)
        if kind == "symm" and not report["modes"].get(mode, {}).get("available"):
            continue
        try:
            be, ar, opt = build(kind, n, env, dev, mode_env=mode)
        except Exception as e:
            report.setdefault("timing", {})[key] = {"error": str(e)[:200]}
            continue
        sched = RoundScheduler("dpu")
        times = []
        for it in range(a.bench_iters + 3):
            plan = sched.next_plan()
            dist.barrier()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            be.launch_round(plan, 1e-3, 1)
            e1.record()
            torch.cuda.synchronize()
            sched.complete(plan, be.finish_round(plan))
            t = torch.tensor([e0.elapsed_time(e1)], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            if it >= 3:
                times.append(float(t.item()))
        ms = sorted(times)[len(times) // 2]
        S = ar.layout.size_slice
        link_bytes = 2.0 * S * (W - 1)                       # per direction per GPU: RS ingress == AG egress
        hbm_bytes = S * (2 * W + 12 + 12 + 2 * W) + ar.layout.padded * 2   # reads+writes incl. accumulator zeroing
        report.setdefault("timing", {})[key] = {
            "backend": be.name, "ms_median": ms, "ms_min": min(times), "numel": n, "slice": S,
            "nvlink_GBps_per_dir": link_bytes / (ms * 1e-3) / 1e9, "nvlink_frac_of_450": link_bytes / (ms * 1e-3) / 450e9,
            "roofline_ms": max(link_bytes / 450e9, hbm_bytes / 3.35e12) * 1e3,
        }
        del be, ar, opt
        torch.cuda.empty_cache()
    # ---- what the fabric + NCCL's own NVLS kernels sustain for the same bytes: an all-reduce of the whole accumulator does exactly the
    # traffic of one round (switch-reduce every 1/W slice, multicast it back) without the AdamW / zeroing work
    try:
        buf = torch.zeros(((n + 1023) // 1024) * 1024, device=dev, dtype=torch.bfloat16)
        times = []
        for it in range(a.bench_iters + 3):
            dist.barrier()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            dist.all_reduce(buf)
            e1.record()
            torch.cuda.synchronize()
            t = torch.tensor([e0.elapsed_time(e1)], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            if it >= 3:
                times.append(float(t.item()))
        ms = sorted(times)[len(times) // 2]
        report.setdefault("timing", {})["nccl_allreduce_same_bytes"] = {
            "ms_median": ms, "numel": int(buf.numel()), "bus_GBps": 2.0 * (W - 1) / W * buf.numel() * 2 / (ms * 1e-3) / 1e9,
            "note": "NCCL all-reduce (NVLS when available) of a bf16 buffer the size of the gradient accumulator: the collective-only floor "
                    "of a round on this fabric"}
    except Exception as e:      # noqa: BLE001
        report.setdefault("timing", {})["nccl_allreduce_same_bytes"] = {"error": str(e)[:200]}
    if rank == 0:
        print(json.dumps(report, indent=1))
        if a.out:
            os.makedirs(os.path.dirname(a.out), exist_ok=True)
            json.dump(report, open(a.out, "w"), indent=1)
    dist.barrier()
    dist.destroy_process_group()
    bad = [m for m, v in report["modes"].items() if v.get("available") and not v.get("ok")]
    if not any(v.get("available") for v in report["modes"].values()):
        bad.append("no symmetric-memory transport available")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
