#!/usr/bin/env python
"""RMSNorm / LayerNorm kernels of this tree against another build of the extension (typically the previous commit's):
same seeded inputs through both, outputs compared, then kernel times alternated between the two in one process.

    python tools/norm_parity.py --parent-ext /path/to/other/_C.so [--out norm_parity.json] [--iters 30] [--rounds 5]

The other build is loaded as a second module (``acco_parent._C``) and driven through its own bindings: either the
unified ``norm_fwd`` / ``norm_bwd`` or the older per-norm ones (``rmsnorm_fwd``, ``add_rmsnorm_fwd``, ``rmsnorm_bwd``,
``add_rmsnorm_bwd``, ``layernorm_fwd``, ``layernorm_bwd``).

Rules (widths up to 1024 take the warp-per-row kernels, which must not change at all):
* H <= 1024: y, h, mean, rstd, dh and dw / db (fp32 and accumulated into a bf16 .grad) bitwise equal;
* H > 1024 (only the reduction order may differ): h bitwise; mean / rstd within 2e-6 relative; y and dh within one bf16
  ulp per element; fp32 dw / db within 1e-5 * max|dw|; accumulated bf16 dw / db within one bf16 ulp.
Shapes the other build does not cover are skipped.  Timing: T = 8192, L2 flushed before every launch
(``kernel_bench.timed``), the two builds alternated ``--rounds`` times; the spread is the largest relative difference
between two rounds of the other build, and the check is new median <= other median * (1 + spread)."""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch

from acco_b200 import ops
from kernel_bench import timed

DEV = "cuda"
EPS = 1e-5
PARITY_T = (1000, 8192)
PARITY_H = (64, 768, 1024, 2048, 2560, 4096, 8192, 12288)
TIMING_H = (768, 2048, 2560, 4096, 8192)
SHIPPED = {"rmsnorm": (768, 2048, 4096), "layernorm": (768, 2560)}


def load_module(path):
    spec = importlib.util.spec_from_file_location("acco_parent._C", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class Unified:
    """A build with ``norm_fwd`` / ``norm_bwd`` (any width the kernels cover: H % 8 == 0, H <= 16384)."""

    def __init__(self, C):
        self.C = C

    def covers(self, layer, H):
        return H % 8 == 0 and H <= 16384

    def fwd(self, a, r, w, b):
        return tuple(self.C.norm_fwd(a, r, w, b, EPS))

    def bwd(self, dy, de, h, w, mean, rstd, wg, bg):
        return tuple(self.C.norm_bwd(dy, de, h, w, mean, rstd, wg, bg))


class PerNorm:
    """A build with the per-norm bindings (RMSNorm up to H = 16384, LayerNorm up to 8192)."""

    def __init__(self, C):
        self.C = C

    def covers(self, layer, H):
        return H % 8 == 0 and H <= (8192 if layer else 16384)

    def fwd(self, a, r, w, b):
        C = self.C
        if b is None:
            if r is None:
                y, rstd = C.rmsnorm_fwd(a, w, EPS)
                return y, None, None, rstd
            y, h, rstd = C.add_rmsnorm_fwd(a, r, w, EPS)
            return y, h, None, rstd
        out = C.layernorm_fwd(a, r, w, b, EPS)
        return (out[0], None, out[1], out[2]) if r is None else tuple(out)

    def bwd(self, dy, de, h, w, mean, rstd, wg, bg):
        C = self.C
        if mean is None:
            return tuple(C.rmsnorm_bwd(dy, h, w, rstd, wg) if de is None else C.add_rmsnorm_bwd(dy, de, h, w, rstd, wg))
        return tuple(C.layernorm_bwd(dy, de, h, w, mean, rstd, wg, bg))


def wrap(C):
    return Unified(C) if hasattr(C, "norm_fwd") else PerNorm(C)


def bf(shape, gen, scale=1.0, shift=0.0):
    return (torch.randn(*shape, generator=gen) * scale + shift).to(DEV, torch.bfloat16)


def inputs(T, H, seed):
    g = torch.Generator().manual_seed(seed)
    return dict(a=bf((T, H), g), r=bf((T, H), g), w=bf((H,), g, 0.1, 1.0), b=bf((H,), g, 0.1), dy=bf((T, H), g), de=bf((T, H), g),
                wg=bf((H,), g, 0.5), bg=bf((H,), g, 0.5))


def ulp_ok(new, old):
    """|new - old| <= one bf16 ulp of the larger magnitude, elementwise."""
    n, o = new.float(), old.float()
    mag = torch.maximum(n.abs(), o.abs()).clamp_min(torch.finfo(torch.bfloat16).tiny)
    _, e = torch.frexp(mag)
    return bool(((n - o).abs() <= torch.ldexp(torch.ones_like(mag), e - 8)).all())


def compare(name, new, old, exact, kind, fails):
    if new is None and old is None:
        return
    if exact or kind == "bits":
        ok = torch.equal(new, old)
    elif kind == "stat":
        ok = bool(((new - old).abs() <= 2e-6 * old.abs()).all())
    elif kind == "ulp":
        ok = ulp_ok(new, old)
    else:                                       # fp32 parameter-gradient sums
        ok = bool(((new - old).abs() <= 1e-5 * old.abs().max()).all())
    if not ok:
        d = (new.float() - old.float()).abs().max().item()
        fails.append(f"{name}: max |diff| {d:.3e}")


def parity(new, old, fails):
    n = 0
    for layer in (False, True):
        kind = "layernorm" if layer else "rmsnorm"
        for T in PARITY_T:
            for H in PARITY_H:
                if not (old.covers(layer, H) and new.covers(layer, H)):
                    print(f"skip {kind} T={T} H={H}: not covered by the other build", flush=True)
                    continue
                x = inputs(T, H, seed=T * 100003 + H)
                b = x["b"] if layer else None
                exact = H <= 1024
                for res in (False, True):
                    tag = f"{'add_' if res else ''}{kind} T={T} H={H}"
                    r = x["r"] if res else None
                    fn, fo = new.fwd(x["a"], r, x["w"], b), old.fwd(x["a"], r, x["w"], b)
                    for nm, i, k in (("y", 0, "ulp"), ("h", 1, "bits"), ("mean", 2, "stat"), ("rstd", 3, "stat")):
                        compare(f"{tag} {nm}", fn[i], fo[i], exact, k, fails)
                    # the backward of both builds sees the same saved tensors (the other build's forward outputs)
                    h = fo[1] if res else x["a"]
                    de = x["de"] if res else None
                    dn, do = new.bwd(x["dy"], de, h, x["w"], fo[2], fo[3], None, None), old.bwd(x["dy"], de, h, x["w"], fo[2], fo[3], None, None)
                    compare(f"{tag} dh", dn[0], do[0], exact, "ulp", fails)
                    compare(f"{tag} dw|db fp32", dn[1], do[1], exact, "sum", fails)
                    acc = {}
                    for side, impl in (("new", new), ("old", old)):
                        wg, bg = x["wg"].clone(), (x["bg"].clone() if layer else None)
                        impl.bwd(x["dy"], de, h, x["w"], fo[2], fo[3], wg, bg)
                        acc[side] = (wg, bg)
                    compare(f"{tag} dw accumulated", acc["new"][0], acc["old"][0], exact, "ulp", fails)
                    if layer:
                        compare(f"{tag} db accumulated", acc["new"][1], acc["old"][1], exact, "ulp", fails)
                    n += 1
    return n


def timing(new, old, iters, rounds):
    T = 8192
    rows = []
    for layer in (False, True):
        kind = "layernorm" if layer else "rmsnorm"
        for H in TIMING_H:
            if not (old.covers(layer, H) and new.covers(layer, H)):
                continue
            x = inputs(T, H, seed=7)
            b = x["b"] if layer else None
            _, _, mean, rstd = old.fwd(x["a"], None, x["w"], b)
            wg, bg = x["wg"].clone(), (x["bg"].clone() if layer else None)
            cases = {
                "fwd": lambda impl: impl.fwd(x["a"], None, x["w"], b),
                "add_fwd": lambda impl: impl.fwd(x["a"], x["r"], x["w"], b),
                "bwd_accum": lambda impl: impl.bwd(x["dy"], None, x["a"], x["w"], mean, rstd, wg, bg),
                "add_bwd_accum": lambda impl: impl.bwd(x["dy"], x["de"], x["a"], x["w"], mean, rstd, wg, bg),
            }
            for case, fn in cases.items():
                t_old, t_new = [], []
                for _ in range(rounds):
                    t_old.append(timed(lambda: fn(old), iters, True))
                    t_new.append(timed(lambda: fn(new), iters, True))
                med = lambda v: sorted(v)[len(v) // 2]
                spread = (max(t_old) - min(t_old)) / min(t_old)
                m_old, m_new = med(t_old), med(t_new)
                rows.append(dict(norm=kind, H=H, case=case, parent_ms=m_old, new_ms=m_new, ratio=m_new / m_old, spread=spread,
                                 shipped=H in SHIPPED[kind], ok=m_new <= m_old * (1 + spread)))
                r = rows[-1]
                print(f"{kind:9s} H={H:5d} {case:14s} parent {m_old * 1e3:8.1f} us  new {m_new * 1e3:8.1f} us  "
                      f"new/parent {r['ratio']:.3f}  spread {spread:.3f}  {'shipped' if r['shipped'] else '':7s} "
                      f"{'ok' if r['ok'] else 'SLOWER'}", flush=True)
    return rows


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-ext", required=True, help="path of the other build's _C*.so")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-timing", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    new, old = wrap(ops.load_ext(required=True)), wrap(load_module(a.parent_ext))
    print("card:", card(), flush=True)
    fails = []
    n = parity(new, old, fails)
    print(f"parity: {n} shape/variant cases, {len(fails)} failures", flush=True)
    for f in fails:
        print("  FAIL", f)
    rows = [] if a.no_timing else timing(new, old, a.iters, a.rounds)
    slow = [r for r in rows if r["shipped"] and not r["ok"]]
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump({"card": card(), "parity_cases": n, "parity_failures": fails, "timing": rows}, open(a.out, "w"), indent=1)
    print(f"timing: {len(rows)} cases, {len(slow)} shipped-shape cases slower than parent * (1 + spread)")
    sys.exit(1 if fails or slow else 0)


if __name__ == "__main__":
    main()
