"""KERNEL A on one H100: ``rs_adam_ag_kernel`` and ``round_norm_kernel`` against the fp64 oracle and bounds of
``test_round_oracle.py``, at every local-mode instantiation (G, O in {bf16, fp32}, with and without a no-decay table, the default
and the ``kSmall`` footprint), through both entry points (``adamw_shard`` with a device ``inv_count``; ``rs_adam_ag`` mode 0 with the
in-kernel count, plain and clipped by ``round_norm``'s output), and the P2P instantiation at world 1.  Exact identities (outputs,
commit flags, stash, guard cells, counters) are checked bit for bit.  fp64 references are computed on chunks of the shard.
Run with ``pytest -m gpu -s`` to see the worst error / bound ratio per output."""
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops  # noqa: E402
from acco_b200.parallel.schedule import COMMIT_ALL, COMMIT_NONE, COMMIT_PARAM, COMMIT_STATE, RoundScheduler  # noqa: E402
from test_round_oracle import (Hyper, Round, bf16_rn, f32s, keep_mask, norm_bounds, norm_ref, ratio, round_bounds,  # noqa: E402
                               round_count, round_inputs, round_ref)

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = 1 << 22                     # elements per fp64 reference chunk
GUARD = 8                           # sentinel elements on each side of every tensor the kernel writes
SENTINEL = -96.0
DT = {"bf16": torch.bfloat16, "fp32": torch.float32}
HYPERS = [Hyper(lr=1e-3, b2=0.95, step=1), Hyper(lr=3e-4, b2=0.999, step=2), Hyper(lr=1e-3, b2=0.9999, step=1000),
          Hyper(lr=6e-4, b2=0.95, step=10 ** 6)]
STASH_USE = [(False, False), (False, True), (True, False)]          # (add_stash, write_stash): none, write, add
WORST = {}


@pytest.fixture(scope="module")
def C():
    return ops.load_ext(required=True)


@pytest.fixture(autouse=True)
def _free_between_cases():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def note(name, worst):
    for k, r in worst.items():
        WORST[k] = max(WORST.get(k, 0.0), r)
    print(f"\n[round] {name}: worst error/bound " + " ".join(f"{k}={r:.3f}" for k, r in worst.items()))


# ================================================================================================= geometry
def small_mode() -> bool:
    return os.environ.get("ACCO_ROUND_LOCAL_SMALL", "") == "1"


def default_grid(C, S: int, mode: int = 0) -> int:
    """``default_grid`` of the binding (the ``kSmall`` launch then clamps to one CTA per SM)."""
    want = max(-(-(S // 8) // 256), 1)
    return min(want, C.num_sms() * (4 if mode == 0 else 1))


def vectors_per_pass(C, grid: int, mode: int = 0) -> int:
    """Vectors one pass of the grid-stride loop covers: grid x threads x the ``kU`` unroll."""
    if mode == 0 and small_mode():
        return min(grid, C.num_sms()) * 256 * 2
    return grid * 512 * (4 if mode == 0 else 1)


def wrap_sizes(C, grid: int, mode: int = 0):
    """Shard sizes of +-1 vector around one and two full passes, and one that leaves some ``kU`` slots of the last pass empty."""
    p = vectors_per_pass(C, grid, mode)
    step = p // (4 if mode == 0 and not small_mode() else 2 if mode == 0 else 1)     # vectors per unrolled slot
    return [8 * n for n in (p - 1, p + 1, 2 * p - 1, 2 * p + 1, p + step + 5)]


def no_decay_ranges(S: int):
    """Ranges that start and end inside vectors, at the first element, and past the end of the shard."""
    cand = sorted([(0, 1), (3, 11), (S // 3 + 1, S // 3 + 13), (S // 2 + 5, S // 2 + 6), (S - 1, S + 4)])
    out = []
    for lo, hi in cand:
        if out and lo <= out[-1][1]:
            out[-1] = (out[-1][0], max(out[-1][1], hi))
        else:
            out.append((lo, hi))
    return out


# ================================================================================================= state with guard cells
class State:
    """Shard state, gradient sum and output, each a view between two runs of ``GUARD`` sentinel elements."""

    def __init__(self, S, gdt, odt, seed, eps_dominated=False, stash_count=0):
        grad, master, m, v, stash = round_inputs(S, gdt, seed=seed, eps_dominated=eps_dominated, device=DEV)
        self.S = S
        self.bufs = {}
        for name, x in (("grad", grad), ("master", master), ("m", m), ("v", v), ("stash", stash),
                        ("out", torch.zeros(S, dtype=odt, device=DEV))):
            buf = torch.full((S + 2 * GUARD,), SENTINEL, dtype=x.dtype, device=DEV)
            buf[GUARD:GUARD + S] = x
            self.bufs[name] = buf
            setattr(self, name, buf[GUARD:GUARD + S])
        self.scratch = torch.tensor([stash_count, -5, 0, 0], dtype=torch.int32, device=DEV)
        self.init = {k: getattr(self, k).clone() for k in ("grad", "master", "m", "v", "stash")}

    def guards_ok(self) -> bool:
        return all(bool((b[:GUARD] == SENTINEL).all()) and bool((b[GUARD + self.S:] == SENTINEL).all()) for b in self.bufs.values())


def launch(C, entry, st: State, hp: Hyper, rd: Round, grid=0, table=None, mode=0, pads=(), max_norm=None, norm_out=None):
    """One round through ``adamw_shard`` ("shard": ``rd.inv`` as a device scalar), ``rs_adam_ag`` ("round": in-kernel count) or
    ``round_norm`` + ``rs_adam_ag`` ("clipped").  Returns the ``rd`` the oracle must use (the clipped round's ``inv_eff``)."""
    gbf, obf = st.grad.dtype == torch.bfloat16, st.out.dtype == torch.bfloat16
    tab = None if table is None else torch.tensor(table, dtype=torch.int64, device=DEV).view(-1, 2)
    if entry == "shard":
        inv_t = torch.tensor([rd.inv], dtype=torch.float32, device=DEV)
        C.adamw_shard(st.grad, st.master, st.m, st.v, st.stash, st.out, inv_t, st.scratch, hp.lr, hp.b1, hp.b2, hp.eps, hp.wd, hp.step,
                      rd.commit, rd.add_stash, rd.write_stash, tab, 0)
        return rd
    inv = None
    if entry == "clipped":
        C.round_norm([st.grad.data_ptr()], list(pads), 0, st.stash, st.scratch, norm_out, st.S, 0, 1, rd.local_count, rd.add_stash, gbf,
                     mode, grid, max_norm)
        inv = norm_out
    C.rs_adam_ag([st.grad.data_ptr()], [st.out.data_ptr()], list(pads), 0, 0, st.master, st.m, st.v, st.stash, st.scratch, st.S, 0, 1,
                 rd.local_count, hp.lr, hp.b1, hp.b2, hp.eps, hp.wd, hp.step, rd.commit, rd.add_stash, rd.write_stash, gbf, obf, mode, grid,
                 None, inv, tab)
    if entry == "clipped":
        return Round(rd.commit, rd.add_stash, rd.write_stash, rd.local_count, rd.stash_count, float(norm_out[1]))
    return rd


def bound_ratios(got, init, hp: Hyper, rd: Round, keep=None, finite_only=False):
    """Worst error / bound of ``m1``, ``v1``, ``p1`` (each only if present in ``got``), on chunks."""
    S = init["master"].numel()
    worst = {}
    for lo in range(0, S, CHUNK):
        sl = slice(lo, min(S, lo + CHUNK))
        o = round_ref(init["grad"][sl], init["master"][sl], init["m"][sl], init["v"][sl], init["stash"][sl], hp, rd,
                      None if keep is None else keep[sl])
        b = round_bounds(o, hp, rd)
        for k, bn in (("m1", "m"), ("v1", "v"), ("p1", "p")):
            if k not in got:
                continue
            want, g = o[k], got[k][sl]
            if finite_only:
                fin = torch.isfinite(want)
                want, g, bb = want[fin], g[fin], b[bn][fin]
            else:
                bb = b[bn]
            worst[k] = max(worst.get(k, 0.0), ratio(g, want, bb))
    return worst


def check_round(C, entry, st: State, hp, rd, grid=0, table=None, mode=0, pads=(), name=""):
    """Launch one COMMIT_ALL round and check everything: bounds, exact output and stash, guard cells, counters."""
    S = st.S
    keep = keep_mask(S, table, device=DEV) if table else None
    norm_out = torch.zeros(3 + 4 * C.num_sms() + 8, device=DEV)
    max_norm = None
    if entry == "clipped":
        total = round_count(rd)[0]
        max_norm = 0.5 * norm_ref(st.grad, st.stash, rd.add_stash, total, 1.0)["norm"]
    rd_used = launch(C, entry, st, hp, rd, grid, table, mode, pads, max_norm, norm_out)
    torch.cuda.synchronize()
    got = {"m1": st.m, "v1": st.v, "p1": st.master}
    worst = bound_ratios(got, st.init, hp, rd_used, keep)
    assert all(r <= 1.0 for r in worst.values()), (name, worst)
    if st.out.dtype == torch.float32:
        assert torch.equal(st.out, st.master), name
    else:
        assert torch.equal(st.out, bf16_rn(st.master.double())), name                  # round to nearest even, of the committed master'
    acc = st.init["grad"].float() + (st.init["stash"] if rd.add_stash else 0.0)
    assert torch.equal(st.stash, acc if rd.write_stash else st.init["stash"]), name     # f32(acc), unscaled
    assert torch.equal(st.grad, st.init["grad"]) and st.guards_ok(), name
    total, after = round_count(rd)
    assert st.scratch.tolist()[:2] == [after, total], name                              # stash_count, total_out
    assert int(st.scratch[3]) == 0, name                                                 # done_ctas reset by the last CTA
    if entry == "clipped":
        nb = norm_bounds(st.init["grad"], st.init["stash"], rd.add_stash, total, max_norm, grid or default_grid(C, S, mode), float(norm_out[2]))
        no = norm_ref(st.init["grad"], st.init["stash"], rd.add_stash, total, max_norm)
        worst["sumsq"] = abs(float(norm_out[2]) - no["sumsq"]) / nb["sumsq"]
        worst["norm"] = abs(float(norm_out[0]) - nb["want_norm"]) / nb["norm"]
        worst["inv_eff"] = abs(float(norm_out[1]) - nb["want_inv_eff"]) / nb["inv_eff"]
        assert max(worst["sumsq"], worst["norm"], worst["inv_eff"]) <= 1.0, (name, worst)
    return worst


def configs(C, entry, mode=0):
    """(S, grid) pairs: 8 and 8 * 37 elements, the wrap sizes at the default grid, and (rs_adam_ag) at forced grids 1, 3 and 7."""
    out = [(8, 0), (8 * 37, 0)]
    full = default_grid(C, 1 << 40, mode)
    out += [(S, 0) for S in wrap_sizes(C, full, mode)]
    if entry != "shard":
        for g in (1, 3, 7):
            out += [(S, g) for S in wrap_sizes(C, g, mode)]
    return out


def run_variant(C, entry, gname, oname, nodecay, mode=0, pads=()):
    """Every size of ``configs`` with the hyperparameter edges, eps-dominated elements and stash uses cycled through."""
    worst = {}
    for i, (S, grid) in enumerate(configs(C, entry, mode)):
        hp = HYPERS[i % len(HYPERS)]
        add, write = STASH_USE[i % 3]
        stash_count = 3 + i % 4
        if entry == "shard":
            rd = Round(COMMIT_ALL, add, write, 0, stash_count, f32s(1.0 / (2 + i % 5)))
        else:
            rd = Round(COMMIT_ALL, add, write, 1 + i % 6, stash_count)
        st = State(S, DT[gname], DT[oname], seed=i + 17 * nodecay, eps_dominated=i % 2 == 1, stash_count=stash_count)
        table = no_decay_ranges(S) if nodecay else None
        w = check_round(C, entry, st, hp, rd, grid, table, mode, pads, name=f"{entry} {gname}->{oname} S={S} grid={grid}")
        for k, r in w.items():
            worst[k] = max(worst.get(k, 0.0), r)
        del st
    return worst


# ================================================================================================= against the bounds
VARIANTS = [(g, o, nd) for g in ("bf16", "fp32") for o in ("bf16", "fp32") for nd in (False, True)]


@pytest.mark.parametrize("entry", ["shard", "round", "clipped"])
@pytest.mark.parametrize("gname,oname,nodecay", VARIANTS)
def test_round_against_bounds(C, entry, gname, oname, nodecay):
    """m', v', master' within the fp64 bounds; out == master' (fp32) or bf16_rn(master') bit for bit; the stash write is f32(acc);
    guard cells, counters."""
    note(f"{entry} {gname}->{oname} nodecay={nodecay}", run_variant(C, entry, gname, oname, nodecay))


@pytest.mark.parametrize("gname,oname,nodecay", VARIANTS)
def test_commit_modes_and_stash(C, gname, oname, nodecay):
    """Every commit mode x stash use from the same state: the output is identical across the four modes, m' and v' between STATE
    and ALL, master' between PARAM and ALL; what a mode does not commit keeps its bits; counters follow the count rule."""
    S = 8 * 4099
    table = no_decay_ranges(S) if nodecay else None
    hp = Hyper(lr=1e-3, b2=0.999, step=3)
    for add, write in STASH_USE:
        res = {}
        rd0 = Round(COMMIT_ALL, add, write, 5, 7)
        for commit in (COMMIT_NONE, COMMIT_PARAM, COMMIT_STATE, COMMIT_ALL):
            st = State(S, DT[gname], DT[oname], seed=5, stash_count=7)
            rd = Round(commit, add, write, 5, 7)
            launch(C, "round", st, hp, rd, table=table)
            torch.cuda.synchronize()
            res[commit] = st
            if not commit & COMMIT_PARAM:
                assert torch.equal(st.master, st.init["master"]), (commit, add, write)
            if not commit & COMMIT_STATE:
                assert torch.equal(st.m, st.init["m"]) and torch.equal(st.v, st.init["v"]), (commit, add, write)
            total, after = round_count(rd)
            assert st.scratch.tolist() == [after, total, 0, 0] and st.guards_ok()
        a = res[COMMIT_ALL]
        for commit, st in res.items():
            assert torch.equal(st.out, a.out) and torch.equal(st.stash, a.stash), commit
        assert torch.equal(res[COMMIT_STATE].m, a.m) and torch.equal(res[COMMIT_STATE].v, a.v)
        assert torch.equal(res[COMMIT_PARAM].master, a.master)
        w = bound_ratios({"m1": a.m, "v1": a.v, "p1": a.master}, a.init, hp, rd0, keep_mask(S, table, device=DEV) if table else None)
        assert all(r <= 1.0 for r in w.values()), w


@pytest.mark.parametrize("gname,oname", [(g, o) for g in ("bf16", "fp32") for o in ("bf16", "fp32")])
def test_zero_gradient_probes(C, gname, oname):
    """Zero gradient and moments: lr * wd = 0.5 halves the master exactly and lr = 0 leaves it unchanged, through both entry points
    of the default instantiations (denominator eps, update exactly 0)."""
    S = 8 * 3001
    for entry in ("shard", "round"):
        for lr, wd, factor in ((0.5, 1.0, 0.5), (0.0, 0.1, 1.0)):
            st = State(S, DT[gname], DT[oname], seed=9)
            for t in (st.grad, st.m, st.v, st.stash):
                t.zero_()
            st.init = {k: getattr(st, k).clone() for k in ("grad", "master", "m", "v", "stash")}
            rd = Round(COMMIT_ALL, False, False, 0 if entry == "shard" else 4, 0, 0.25 if entry == "shard" else None)
            launch(C, entry, st, Hyper(lr=lr, wd=wd, step=1), rd)
            torch.cuda.synchronize()
            want = st.init["master"] * factor
            assert torch.equal(st.master, want), (entry, lr)
            assert torch.equal(st.out, want.to(st.out.dtype)), (entry, lr)
            assert bool((st.m == 0).all()) and bool((st.v == 0).all())


def test_round_with_count_zero_scales_by_one(C):
    """local_count 0 without the stash: total_out 0 and the gradient is applied unscaled (1 / max(0, 1))."""
    S = 8 * 513
    st = State(S, torch.float32, torch.float32, seed=4, stash_count=9)
    rd = Round(COMMIT_ALL, False, False, 0, 9)
    w = check_round(C, "round", st, Hyper(step=4), rd, name="count 0")
    assert st.scratch.tolist()[:2] == [9, 0]
    note("count 0", w)


# ================================================================================================= non-finite gradients
@pytest.mark.parametrize("gname", ["bf16", "fp32"])
@pytest.mark.parametrize("entry", ["shard", "round"])
def test_non_finite_gradients_stay_in_their_element(C, gname, entry):
    """A NaN, +inf or -inf gradient at each of the 8 positions of a vector: the non-finite outputs are exactly the oracle's, and
    every other element of the vector (and the shard) stays within its bound."""
    vals = (math.nan, math.inf, -math.inf)
    S = 8 * 64
    st = State(S, DT[gname], torch.float32, seed=6)
    for j in range(8):
        for k, x in enumerate(vals):
            st.grad[8 * (3 * j + k + 1) + j] = x
    st.init["grad"] = st.grad.clone()
    rd = Round(COMMIT_ALL, False, False, 0 if entry == "shard" else 3, 0, 0.25 if entry == "shard" else None)
    launch(C, entry, st, Hyper(step=2), rd)
    torch.cuda.synchronize()
    o = round_ref(st.init["grad"], st.init["master"], st.init["m"], st.init["v"], st.init["stash"], Hyper(step=2), rd)
    for k, got in (("m1", st.m), ("v1", st.v), ("p1", st.master), ("p1", st.out)):
        want = o[k]
        assert torch.equal(torch.isnan(got), torch.isnan(want)), k
        assert torch.equal(torch.isinf(got), torch.isinf(want)), k
        inf = torch.isinf(want)
        assert torch.equal(torch.sign(got[inf]), torch.sign(want[inf].float())), k
    assert int(torch.isnan(st.master).sum()) == 24                       # the update of a non-finite element is NaN, nothing more
    w = bound_ratios({"m1": st.m, "v1": st.v, "p1": st.master}, st.init, Hyper(step=2), rd, finite_only=True)
    assert all(r <= 1.0 for r in w.values()), w


# ================================================================================================= norm pass
def run_norm(C, grad, stash, scratch, out, S, local_count, add, grid, max_norm):
    C.round_norm([grad.data_ptr()], [], 0, stash, scratch, out, S, 0, 1, local_count, add, grad.dtype == torch.bfloat16, 0, grid, max_norm)


@pytest.mark.parametrize("gname", ["bf16", "fp32"])
def test_norm_pass(C, gname):
    """sumsq, norm and inv_eff within bound at wrapping sizes and forced grids; repeat gives the same bits and the counter resets;
    a zero gradient gives a coefficient of exactly 1; a NaN gives a NaN norm and inv_eff."""
    worst = {}
    out = torch.zeros(3 + 4 * C.num_sms() + 8, device=DEV)
    cases = []
    for grid in (0, 1, 3, 7):
        g = grid or 4 * C.num_sms()
        per = g * 256 * 4
        cases += [(8 * n, grid) for n in (per - 1, per + 1, 2 * per + 3)]
    cases += [(8, 0), (8 * 37, 5)]
    for i, (S, grid) in enumerate(cases):
        add = i % 2 == 1
        gen = torch.Generator(device=DEV).manual_seed(i)
        grad = (torch.randn(S, device=DEV, generator=gen) * 3).to(DT[gname])
        stash = torch.randn(S, device=DEV, generator=gen)
        scratch = torch.tensor([4, 0, 0, 0], dtype=torch.int32, device=DEV)
        local_count = 1 + i % 5
        total = local_count + (4 if add else 0)
        max_norm = (0.5 if i % 3 else 4.0) * norm_ref(grad, stash, add, total, 1.0)["norm"]
        run_norm(C, grad, stash, scratch, out, S, local_count, add, grid, max_norm)
        first = out.clone()
        run_norm(C, grad, stash, scratch, out, S, local_count, add, grid, max_norm)
        assert torch.equal(out[:3], first[:3]) and int(scratch[3]) == 0
        b = norm_bounds(grad, stash, add, total, max_norm, grid or default_grid(C, S), float(out[2]))
        o = norm_ref(grad, stash, add, total, max_norm)
        w = {"sumsq": abs(float(out[2]) - o["sumsq"]) / b["sumsq"], "norm": abs(float(out[0]) - b["want_norm"]) / b["norm"],
             "inv_eff": abs(float(out[1]) - b["want_inv_eff"]) / b["inv_eff"]}
        assert max(w.values()) <= 1.0, (S, grid, w)
        for k, r in w.items():
            worst[k] = max(worst.get(k, 0.0), r)
    z = torch.zeros(8 * 1000, dtype=DT[gname], device=DEV)
    scratch = torch.zeros(4, dtype=torch.int32, device=DEV)
    run_norm(C, z, torch.zeros(8 * 1000, device=DEV), scratch, out, 8 * 1000, 4, False, 0, 1.0)
    assert float(out[0]) == 0.0 and float(out[1]) == 0.25               # coefficient exactly 1, inv = rcp(4) exact
    z[77] = math.nan
    run_norm(C, z, torch.zeros(8 * 1000, device=DEV), scratch, out, 8 * 1000, 4, False, 0, 1.0)
    assert math.isnan(float(out[0])) and math.isnan(float(out[1]))
    note(f"norm {gname}", worst)


# ================================================================================================= a round sequence, eager and graphed
CLIP = 0.05                         # max_grad_norm of the clipped sequence: every round clips


def acco_round(C, st: State, acc, lc, plan, r, step, clip, norm_out, snap):
    """One round of an ACCO plan (tentative: write the stash, commit nothing; real: add it, commit all) through the in-kernel count,
    then a copy of the output, the counters and the norm pass's result into ``snap``."""
    hp = Hyper(lr=1e-3 * (1 - r / 16), b2=0.999, step=step + 1)
    inv = None
    if clip:
        C.round_norm([acc.data_ptr()], [], 0, st.stash, st.scratch, norm_out, st.S, 0, 1, lc, plan.add_stash, True, 0, 0, CLIP)
        inv = norm_out
    C.rs_adam_ag([acc.data_ptr()], [st.out.data_ptr()], [], 0, 0, st.master, st.m, st.v, st.stash, st.scratch, st.S, 0, 1, lc,
                 hp.lr, hp.b1, hp.b2, hp.eps, hp.wd, hp.step, plan.commit, plan.add_stash, plan.write_stash, True, False, 0, 0, None, inv, None)
    snap["out"].copy_(st.out)
    snap["scratch"].copy_(st.scratch)
    snap["norm"].copy_(norm_out[:3])
    return hp


def acco_sequence(C, st: State, accs, counts, clip: bool, norm_out, snaps):
    sched = RoundScheduler("acco")
    step = 0
    for r, (acc, lc) in enumerate(zip(accs, counts)):
        plan = sched.next_plan()
        acco_round(C, st, acc, lc, plan, r, step, clip, norm_out, snaps[r])
        step += 1 if plan.commit & COMMIT_STATE else 0


@pytest.mark.parametrize("clip", [False, True])
def test_acco_round_sequence_eager_and_graphed(C, clip):
    """Each round against the oracle applied to the kernel's own state before it (as ``tools/symm_check.py`` does); then the same
    sequence captured once in a CUDA graph and replayed from the same initial state matches eager bit for bit, counters included."""
    S = 8 * 70001
    rounds = 8
    st = State(S, torch.bfloat16, torch.float32, seed=21)
    for t in (st.m, st.v, st.stash):
        t.zero_()
    gen = torch.Generator(device=DEV).manual_seed(22)
    accs = [(torch.randn(S, device=DEV, generator=gen) * (1 + r)).bfloat16() for r in range(rounds)]
    counts = [2, 3, 1, 4, 2, 2, 5, 3]
    norm_out = torch.zeros(3 + 4 * C.num_sms(), device=DEV)
    start = {k: getattr(st, k).clone() for k in ("master", "m", "v", "stash", "out", "scratch")}

    def snaps_new():
        return [{"out": torch.empty_like(st.out), "scratch": torch.empty_like(st.scratch), "norm": torch.empty(3, device=DEV)}
                for _ in range(rounds)]

    # eager, one round at a time, each checked against the oracle from the kernel's own state before it
    eager = snaps_new()
    sched = RoundScheduler("acco")
    step, worst = 0, {}
    for r in range(rounds):
        before = {"grad": accs[r], "master": st.master.clone(), "m": st.m.clone(), "v": st.v.clone(), "stash": st.stash.clone()}
        sc_before = st.scratch.clone()
        plan = sched.next_plan()
        hp = acco_round(C, st, accs[r], counts[r], plan, r, step, clip, norm_out, eager[r])
        torch.cuda.synchronize()
        rd = Round(plan.commit, plan.add_stash, plan.write_stash, counts[r], int(sc_before[0]), float(norm_out[1]) if clip else None)
        got = {"p1": st.out}
        if plan.commit & COMMIT_STATE:
            got.update(m1=st.m, v1=st.v)
        w = bound_ratios(got, before, hp, rd)
        assert all(x <= 1.0 for x in w.values()), (r, w)
        for k, x in w.items():
            worst[k] = max(worst.get(k, 0.0), x)
        total, after = round_count(rd)
        assert st.scratch.tolist() == [after, total, 0, 0], r
        if plan.write_stash:
            assert torch.equal(st.stash, accs[r].float() + (before["stash"] if plan.add_stash else 0))
        if not plan.commit:
            assert torch.equal(st.master, before["master"]) and torch.equal(st.m, before["m"]) and torch.equal(st.v, before["v"])
        if plan.commit & COMMIT_STATE:
            step += 1
    final = {k: getattr(st, k).clone() for k in ("master", "m", "v", "stash", "out", "scratch")}
    note(f"sequence clip={clip}", worst)

    # the same sequence in one CUDA graph, replayed from the initial state
    graphed = snaps_new()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for k, x in start.items():
            getattr(st, k).copy_(x)
        acco_sequence(C, st, accs, counts, clip, norm_out, graphed)          # warm-up on the side stream, as before a capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        acco_sequence(C, st, accs, counts, clip, norm_out, graphed)
    for k, x in start.items():
        getattr(st, k).copy_(x)
    for snap in graphed:
        for t in snap.values():
            t.fill_(-1)
    g.replay()
    torch.cuda.synchronize()
    for r in range(rounds):
        for k in ("out", "scratch", "norm"):
            if k == "norm" and not clip:
                continue
            assert torch.equal(graphed[r][k], eager[r][k]), (r, k)
    for k, x in final.items():
        assert torch.equal(getattr(st, k), x), k


# ================================================================================================= P2P at world 1
@pytest.mark.parametrize("gname,oname,nodecay", VARIANTS)
def test_p2p_instantiation_at_world_one(C, gname, oname, nodecay):
    """Mode 1 with one rank: peer loads and stores on local memory, the count exchange through the signal pad, the end barrier.
    Every flag such a round waits on is written earlier by the same thread: the gate kernel publishes pad[0] (and the count in
    pad[2]) before it waits on pad[0], and the last CTA writes pad[1] before it waits on it.  The epoch advances by one per round."""
    pad = torch.zeros(5 + 3, dtype=torch.int32, device=DEV)             # [0, 5W) for W = 1, plus a guard
    pads = [pad.data_ptr()]
    worst = {}
    sizes = [(8 * 37, 0), (8 * (2 * 3 * 512 + 1), 3), (8 * (C.num_sms() * 512 + 1), 0)]
    for r, (S, grid) in enumerate(sizes):
        st = State(S, DT[gname], DT[oname], seed=30 + r, stash_count=2)
        st.scratch[2] = r                                                   # the epoch of the previous round
        rd = Round(COMMIT_ALL, *STASH_USE[r % 3], 3 + r, 2)
        w = check_round(C, "round", st, HYPERS[r], rd, grid, no_decay_ranges(S) if nodecay else None, mode=1, pads=pads,
                        name=f"p2p S={S}")
        assert int(st.scratch[2]) == r + 1 and pad.tolist()[:3] == [r + 1, r + 1, 3 + r] and pad.tolist()[5:] == [0, 0, 0]
        for k, x in w.items():
            worst[k] = max(worst.get(k, 0.0), x)
    note(f"p2p {gname}->{oname} nodecay={nodecay}", worst)


# ================================================================================================= kSmall
def test_small_instantiations_in_a_subprocess():
    """The 256-thread local instantiations (ACCO_ROUND_LOCAL_SMALL=1, read once per process), with and without a table, through
    both entry points: the bounds, the exact checks and the zero-gradient probes."""
    code = f"""
import sys, torch
sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})
import test_round_kernels_gpu as T
from acco_b200 import ops
C = ops.load_ext(required=True)
for g, o, nd in T.VARIANTS:
    for entry in ("shard", "round", "clipped"):
        for k, r in T.run_variant(C, entry, g, o, nd).items():
            T.WORST[k] = max(T.WORST.get(k, 0.0), r)
for g in ("bf16", "fp32"):
    for o in ("bf16", "fp32"):
        T.test_zero_gradient_probes(C, g, o)
print("small ok, worst error/bound", " ".join(f"{{k}}={{v:.3f}}" for k, v in sorted(T.WORST.items())))
"""
    env = dict(os.environ, ACCO_ROUND_LOCAL_SMALL="1")
    p = subprocess.run([sys.executable, "-c", code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0 and "small ok" in p.stdout, p.stdout[-3000:]
    print("\n[round] kSmall: " + p.stdout.strip().splitlines()[-1])


# ================================================================================================= binding checks
def test_bindings_reject_misaligned_short_and_foreign_tensors(C):
    """Rejected before any launch.  Alignment and device cases use zero-length shards and length cases short views inside a larger
    allocation, so even a binding without the checks would touch no memory outside the test's own buffers."""
    big = torch.zeros(64, device=DEV)
    i32 = torch.zeros(4, dtype=torch.int32, device=DEV)
    one = torch.ones(1, device=DEV)
    e = lambda: big[:0]
    mis = big[1:1]                                                       # empty, 4 bytes past a 16-byte boundary
    hyper = (1e-3, 0.9, 0.95, 1e-8, 0.1, 1, COMMIT_ALL, False, False)

    def shard(**kw):
        a = dict(grad_sum=e(), master=e(), exp_avg=e(), exp_avg_sq=e(), stash=e(), out=e(), inv_count=one, scratch=i32)
        a.update(kw)
        C.adamw_shard(a["grad_sum"], a["master"], a["exp_avg"], a["exp_avg_sq"], a["stash"], a["out"], a["inv_count"], a["scratch"], *hyper)

    def rnd(S=0, acc=None, theta=None, **kw):
        a = dict(master=big[:S], exp_avg=big[:S], exp_avg_sq=big[:S], stash=big[:S])
        a.update(kw)
        C.rs_adam_ag([acc if acc is not None else big.data_ptr()], [theta if theta is not None else big.data_ptr()], [], 0, 0,
                     a["master"], a["exp_avg"], a["exp_avg_sq"], a["stash"], i32, S, 0, 1, 1, *hyper, False, False, 0, 0, None)

    shard()                                                              # the well-formed zero-length calls are accepted
    rnd()
    torch.cuda.synchronize()
    for name in ("grad_sum", "master", "exp_avg", "exp_avg_sq", "stash", "out"):
        with pytest.raises(RuntimeError, match="aligned"):
            shard(**{name: mis})
    for name in ("master", "exp_avg", "exp_avg_sq", "stash"):
        with pytest.raises(RuntimeError, match="aligned"):
            rnd(**{name: mis})
    with pytest.raises(RuntimeError, match="aligned"):
        rnd(acc=big.data_ptr() + 4)
    with pytest.raises(RuntimeError, match="aligned"):
        rnd(theta=big.data_ptr() + 8)
    # exp_avg / exp_avg_sq that do not hold S elements (short views inside the 64-element allocation)
    S = 16
    full = lambda: torch.zeros(64, device=DEV)
    for name in ("exp_avg", "exp_avg_sq"):
        args = {k: full()[:S] for k in ("grad_sum", "master", "exp_avg", "exp_avg_sq", "stash", "out")}
        args[name] = full()[:8]
        with pytest.raises(RuntimeError, match="elements"):
            shard(**args)
        args = {k: full()[:S] for k in ("master", "exp_avg", "exp_avg_sq", "stash")}
        args[name] = full()[:8]
        with pytest.raises(RuntimeError, match="elements"):
            rnd(S, **args)
    # zero-length shard tensors on another device (a launch would dereference none of them)
    for name in ("grad_sum", "out"):
        with pytest.raises(RuntimeError, match="device"):
            shard(**{name: torch.zeros(0)})
    torch.cuda.synchronize()
    assert bool((big == 0).all())


def test_report_worst_ratios():
    """Print the worst error / bound per output over the file (``-s``)."""
    if WORST:
        print("\n[round] worst over the file: " + " ".join(f"{k}={v:.3f}" for k, v in sorted(WORST.items())))
