"""The fused all-gather GEMM (gather mode of ``csrc/gemm_wgmma.cu``, ``ops.gemm.GatheredWeight`` / ``gemm_tn_gather``) on the CPU:
the round state its GPU tests start from, a model of its flag protocol with the mutants that model must catch, and the ownership
tables the trainer builds.

* ``emulated_round_state``: what rank ``rank`` and its peers hold after a round that skipped the pulled ranges.  The local copy is
  fresh except inside ``pulled_ranges(r)`` of every other rank ``r`` (those hold the stale value), and peer ``r`` is fresh only inside
  its own slice (poison elsewhere).  ``test_gather_gemm_gpu.py`` builds every input with it, one device buffer per emulated rank.
* ``run_protocol``: the producer thread of every CTA, transcribed at the granularity of its synchronisation.  Units are decoded as
  ``decode_unit`` does in gather mode (BN 256, one K split, ``band = num_sn``, ``pm = pn = 1``; ``test_properties._gemm_units`` is
  the twin of the decoder) and unit ``t`` goes to CTA ``t % G``.  A gatherer (m-block 0 of a column with ``owner >= 0``) loads from
  the owner, issues the TMA store into the local copy, waits for it (``cp.async.bulk.wait_group 0``) and then publishes both half
  flags of ``(n_blk, kb)`` for epoch ``e = *epoch + 1``.  A waiter takes the fast path when both flags of the last k-block are at
  ``e`` or later, and otherwise polls each k-block's two flags before its load.  TMA stores land as late as allowed (at the wait),
  and CTAs are interleaved one step at a time, round robin or at random.  Checked, over two consecutive calls:

  - ``deadlock``: every CTA finishes;
  - ``read-before-store``: a waiter loads ``(n_blk, kb)`` only after that k-block's write-through has landed in this call;
  - ``flag-ahead-of-store``: no flag is published before its store has landed;
  - ``teardown``: the last CTA resets the done counter and advances ``*epoch`` to ``e``, and every gathered flag equals ``e``.

  Flags only rise, so whether the protocol deadlocks does not depend on the interleaving.  The kernel assumes that all ``G`` CTAs
  are resident at once (one per SM); ``resident < G`` models a grid beyond that, and the GPU tests assert that the model clears
  their exact case before they launch it.
"""
from __future__ import annotations

import random
from typing import Dict, List, Optional, Sequence, Tuple

import pytest
import torch
from hypothesis import given, settings, strategies as st

from acco_b200.ops.gemm import TILE_K, TILE_N, GatheredWeight, fused_ag_tables
from test_properties import _gemm_units

H100_SMS = 132
GPU_CTA_CAPS = (0, 1, 2, 7, 131)       # max_ctas values of test_gather_gemm_gpu.py (0: one CTA per SM)
MASK = 0xFFFFFFFF


# ---------------------------------------------------------------------------------------------- round state
def pulled_by_others(W: int, rank: int, weights: Sequence[Tuple[int, int, int]], size_slice: int) -> List[Tuple[int, int]]:
    """Flat-buffer ranges ``[lo, hi)`` that rank ``rank`` pulls from their owners: ``pulled_ranges(r)`` of every ``r != rank`` for
    every weight ``(n, k, offset)``."""
    out = []
    for n, k, off in weights:
        gw = GatheredWeight(n, k, off, [0] * W, size_slice, rank, "cpu")
        for r in range(W):
            if r != rank:
                out += gw.pulled_ranges(r, size_slice)
    return sorted(out)


def emulated_round_state(truth: torch.Tensor, stale, W: int, rank: int, weights: Sequence[Tuple[int, int, int]], size_slice: int,
                         poison=float("nan")):
    """``(local, peers)`` after a round that skipped the pulled ranges.  ``truth``: the fresh flat buffer (``size_slice * W``
    elements, or any length that covers every weight); ``stale``: a tensor like ``truth`` or a scalar; ``weights``: the
    ``(n, k, offset)`` of every gathered matrix.  ``local`` is fresh except in the ranges this rank pulls, which hold ``stale``;
    ``peers[r]`` is a separate buffer, fresh inside rank ``r``'s slice and ``poison`` everywhere else."""
    local = truth.clone()
    for lo, hi in pulled_by_others(W, rank, weights, size_slice):
        local[lo:hi] = stale[lo:hi] if torch.is_tensor(stale) else stale
    peers = []
    for r in range(W):
        p = torch.full_like(truth, poison)
        lo, hi = min(r * size_slice, truth.numel()), min((r + 1) * size_slice, truth.numel())
        p[lo:hi] = truth[lo:hi]
        peers.append(p)
    return local, peers


LAYOUT_CASES = [(2, 2304, 768, 768 * 100, 1024 * 1200), (8, 4096, 768, 8 * 12345, 1024 * 900), (4, 1000, 64, 0, 1024 * 16),
                (8, 50304, 768, 0, 15448064)]                                                       # test_gather_layout.py
ROUND_STATE_CASES = LAYOUT_CASES + [
    (1, 2304, 768, 800, 2304 * 768 + 2048),            # world 1: nothing is pulled
    (3, 2304, 768, 8 * 1001, 800 * 768),               # world 3, offset off every slice boundary
    (8, 4096, 64, 8 * 77, 4096 * 64 // 8 + 256),        # world 8, every slice holds two tiles plus a bit
    (8, 1000, 768, 24, 200 * 768),                     # slice smaller than one 256-row tile: every tile straddles
    (4, 1000, 96, 8 * 5, 300 * 96),                    # N not a multiple of 256 (ragged last tile)
]


def _tile_of(e: torch.Tensor, k: int, off: int) -> torch.Tensor:
    return (e - off) // (TILE_N * k)


@pytest.mark.parametrize("W,n,k,offset,slice_", ROUND_STATE_CASES)
def test_emulated_round_state_matches_the_ownership_tables(W, n, k, offset, slice_):
    """Every element of every rank's local copy and of every peer buffer, against ``GatheredWeight.owners``: a tile this rank
    gathers holds ``stale`` locally and ``truth`` on its owner; every other element of the local copy is fresh; a peer is fresh in
    its own slice only.  Values are element indices (int64), stale = -1 - index, poison = -2^40.  Above 2^22 elements only the
    pulled ranges are compared with the tables (the buffers would take gigabytes)."""
    L = offset + n * k + 1000                           # the weight plus a neighbouring parameter
    assert L <= slice_ * W
    for rank in range(W):
        owners = GatheredWeight(n, k, offset, [0] * W, slice_, rank, "cpu").owners
        tiles = [(offset + t * TILE_N * k, offset + min((t + 1) * TILE_N, n) * k) for t in range(len(owners))]
        assert pulled_by_others(W, rank, [(n, k, offset)], slice_) == [tiles[t] for t, o in enumerate(owners) if o >= 0]
        assert all(o != rank and lo // slice_ == (hi - 1) // slice_ == o for (lo, hi), o in zip(tiles, owners) if o >= 0)
    if L > 1 << 22:
        return
    truth = torch.arange(L, dtype=torch.int64)
    stale = -1 - truth
    poison = -(1 << 40)
    num_n = -(-n // TILE_N)
    e = torch.arange(L)
    in_w = (e >= offset) & (e < offset + n * k)
    tile = torch.where(in_w, _tile_of(e, k, offset), torch.zeros_like(e))
    for rank in range(W):
        gw = GatheredWeight(n, k, offset, [0] * W, slice_, rank, "cpu")
        local, peers = emulated_round_state(truth, stale, W, rank, [(n, k, offset)], slice_, poison)
        owner = torch.tensor(gw.owners, dtype=torch.int64)[tile]
        gathered = in_w & (owner >= 0)
        assert torch.equal(local[gathered], stale[gathered])
        assert torch.equal(local[~gathered], truth[~gathered])
        for r, p in enumerate(peers):
            mine = (e >= r * slice_) & (e < (r + 1) * slice_)
            assert torch.equal(p[mine], truth[mine]) and bool((p[~mine] == poison).all())
        # a gathered tile is whole on its owner: the kernel reads fresh bits from it
        for t in range(num_n):
            o = gw.owners[t]
            if o >= 0:
                lo, hi = offset + t * TILE_N * k, offset + min((t + 1) * TILE_N, n) * k
                assert o != rank and torch.equal(peers[o][lo:hi], truth[lo:hi])
        if W == 1:
            assert torch.equal(local, truth) and all(o == -1 for o in gw.owners)
    if slice_ < TILE_N * k:
        assert all(o == -1 for r in range(W) for o in GatheredWeight(n, k, offset, [0] * W, slice_, r, "cpu").owners[:-1])


# ---------------------------------------------------------------------------------------------- ownership preconditions
@pytest.mark.parametrize("n,k,offset,peers,slice_,what", [
    (512, 256, 1028, 2, 1 << 20, "offset"),
    (512, 260, 1024, 2, 1 << 20, "K"),
    (516, 256, 1024, 2, 1 << 20, "N"),
    (512, 256, 1024, 9, 1 << 20, "peers"),
    (512, 256, 1024, 2, (1024 + 512 * 256) // 2 - 8, "past"),      # the last 16 elements have no owner among the peers
])
def test_gathered_weight_rejects_tables_the_kernel_cannot_serve(n, k, offset, peers, slice_, what):
    with pytest.raises(ValueError):
        GatheredWeight(n, k, offset, [1 << 30] * peers, slice_, 0, "cpu")


def test_gathered_weight_accepts_the_edges_of_its_preconditions():
    GatheredWeight(8, 8, 8, [1 << 30] * 8, 9, 0, "cpu")                         # 8 peers, the matrix ends on the last element
    gw = GatheredWeight(512, 256, 1024, [1 << 30] * 2, (1024 + 512 * 256) // 2, 0, "cpu")
    assert gw.owners == [-1, 1]                                                  # tile 0 straddles, tile 1 is rank 1's


# ---------------------------------------------------------------------------------------------- one table builder
class _Toy(torch.nn.Module):
    """Parameters at chosen flat offsets: each candidate is preceded by a pad parameter of the given size."""

    def __init__(self, shapes, pads):
        super().__init__()
        self.ps = torch.nn.ParameterList()
        self.cands = []
        for (n, k), pad in zip(shapes, pads):
            if pad:
                self.ps.append(torch.nn.Parameter(torch.zeros(pad)))
            p = torch.nn.Parameter(torch.zeros(n, k))
            self.ps.append(p)
            self.cands.append(p)

    def fused_ag_candidates(self):
        return list(self.cands)


def test_fused_ag_tables_is_the_trainers_table():
    """``fused_ag_tables`` on a toy model: one ``GatheredWeight`` per theta buffer with that buffer's bases, weights whose offset, K
    or N is not a multiple of 8 skipped, and the pulled ranges equal to the union of every rank's ``pulled_ranges``."""
    from acco_b200.parallel.arena import FlatArena
    W, rank = 4, 1
    shapes = [(768, 256), (1024, 96), (260, 64), (512, 100), (512, 64), (256, 64)]
    pads = [0, 0, 8, 0, 4, 4]                           # the fifth weight sits at an offset that is 4 mod 8, the sixth at 0 mod 8
    model = _Toy(shapes, pads)
    arena = FlatArena(model, W, rank, torch.float32, "cpu", align=1024, double_buffer=True)
    S = arena.layout.size_slice
    bases = [[(1 << 32) * (i + 1) + r * (1 << 28) for r in range(W)] for i in range(2)]
    table, pulled = fused_ag_tables(model, arena, bases, S, rank, "cpu")
    by_id = {id(p): o for p, o in zip(arena.params, arena.offsets)}
    kept = [p for p in model.cands if by_id[id(p)] % 8 == 0 and p.shape[0] % 8 == 0 and p.shape[1] % 8 == 0]
    assert [id(p) for p in kept] == list(table) and len(kept) == 3
    want = []
    for p in kept:
        gws = table[id(p)]
        assert len(gws) == 2
        for i, gw in enumerate(gws):
            assert (gw.n, gw.k, gw.offset, gw.rank) == (p.shape[0], p.shape[1], by_id[id(p)], rank)
            assert gw.peer_ptrs == [b + 2 * gw.offset for b in bases[i]]
            assert gw.owners == GatheredWeight(gw.n, gw.k, gw.offset, bases[i], S, rank, "cpu").owners
        for r in range(W):
            want += gws[0].pulled_ranges(r, S)
    assert pulled == want and pulled


# ---------------------------------------------------------------------------------------------- the flag protocol
MUTANTS = {
    "m_blocks_descending": "m-blocks walked in descending order (waiters before their gatherer)",
    "pm2_lockstep": "a pm = 2 cluster whose two CTAs move through units in lockstep",
    "fast_path_first_kblock": "the fast path tests the first k-block's flags instead of the last",
    "flag_before_wait_group": "flags published before cp.async.bulk.wait_group 0",
    "epoch_not_incremented": "epoch taken as *epoch instead of *epoch + 1",
    "oversubscribed": "G larger than the number of resident CTAs",
}


def _ge(v: int, e: int) -> bool:
    """``(int32_t)(v - e) >= 0``, the kernel's comparison of a flag with the epoch."""
    return ((v - e) & MASK) < 0x80000000


class _State:
    def __init__(self):
        self.flags: Dict[Tuple[int, int, int], int] = {}
        self.E = 0                    # *epoch
        self.done = 0                 # done counter
        self.landed = set()           # (n_blk, kb) whose write-through has landed in this call
        self.violations: List[Tuple[str, str]] = []

    def flag(self, key) -> int:
        return self.flags.get(key, 0)


def _actor(s: _State, ctas: List[list], num_k: int, owners: Sequence[int], G: int, mutant: Optional[str]):
    """The producer thread(s) of one CTA (or of a lock-stepped cluster: ``ctas`` holds each CTA's unit list).  Yields ``None`` after
    every step, or the flag key it is blocked on."""
    epoch = s.E if mutant == "epoch_not_incremented" else (s.E + 1) & MASK
    yield None
    for step in zip(*ctas):
        roles = []
        for mb, n, kb0, kb1 in step:
            owner = owners[n]
            gatherer, waiter = owner >= 0 and mb == 0, owner >= 0 and mb != 0
            fast = not waiter
            if waiter:
                kc = 0 if mutant == "fast_path_first_kblock" else num_k - 1
                fast = _ge(s.flag((n, kc, 0)), epoch) and _ge(s.flag((n, kc, 1)), epoch)
            roles.append((n, gatherer, waiter, fast))
        yield None
        kb0, kb1 = step[0][2], step[0][3]
        for kb in range(kb0, kb1):
            for n, gatherer, waiter, fast in roles:
                if waiter and not fast:
                    for h in (0, 1):
                        while not _ge(s.flag((n, kb, h)), epoch):
                            yield (n, kb, h)
                if waiter and (n, kb) not in s.landed:
                    s.violations.append(("read-before-store", f"tile {n} k-block {kb}"))
            yield None                                             # the stage is full
            for n, gatherer, waiter, fast in roles:
                if not gatherer:
                    continue
                yield None                                         # TMA store into the local copy issued
                steps = ("publish", "land") if mutant == "flag_before_wait_group" else ("land", "publish")
                for what in steps:
                    if what == "land":
                        s.landed.add((n, kb))                      # cp.async.bulk.wait_group 0 returns
                    else:
                        if (n, kb) not in s.landed:
                            s.violations.append(("flag-ahead-of-store", f"tile {n} k-block {kb}"))
                        s.flags[(n, kb, 0)] = s.flags[(n, kb, 1)] = epoch
                    yield None
    for _ in ctas:                                                 # teardown: done counter, last CTA advances the epoch
        s.done += 1
        if s.done == G:
            s.done = 0
            s.E = epoch
    yield None


def gather_units(M: int, N: int, K: int, G: int, pm: int = 1, descending: bool = False):
    """Per cluster, per CTA: the ``(mb, n_blk, kb0, kb1)`` units of a gather-mode launch of ``G`` CTAs."""
    num_mb = -(-M // 128)
    num_smb = -(-num_mb // pm)
    out: Dict[int, Dict[int, list]] = {}
    for cl, cta, mb, n, kb0, kb1 in _gemm_units(M, N, K, TILE_N, 1, pm, 1, max(1, G // pm)):
        if descending:
            mb = num_smb * pm - 1 - mb
        out.setdefault(cl, {}).setdefault(cta, []).append((mb, n, kb0, kb1))
    return [[ctas[c] for c in sorted(ctas)] for _, ctas in sorted(out.items())]


def run_protocol(M: int, N: int, K: int, G: int, owners: Optional[Sequence[int]] = None, mutant: Optional[str] = None,
                 resident: Optional[int] = None, schedule: str = "rr", seed: int = 0, calls: int = 2) -> List[Tuple[str, str]]:
    """Run ``calls`` consecutive gather-mode launches of ``G`` CTAs (``owners``: the tile owner table, default every column
    gathered) and return the violations found, ``[(check, detail)]``; empty when the protocol is clean."""
    num_n, num_k = -(-N // TILE_N), -(-K // TILE_K)
    owners = list(owners) if owners is not None else [1] * num_n
    pm = 2 if mutant == "pm2_lockstep" else 1
    clusters = gather_units(M, N, K, G, pm, descending=mutant == "m_blocks_descending")
    G = len(clusters) * pm                                          # the grid the host launches: min(units, slots)
    if mutant == "oversubscribed" and resident is None:
        resident = max(1, G // 3)
    resident = len(clusters) if resident is None else resident
    s = _State()
    rng = random.Random(seed)
    for call in range(calls):
        s.landed = set()
        actors = [_actor(s, ctas, num_k, owners, G, mutant) for ctas in clusters]
        blocked: Dict[int, Tuple[int, int, int]] = {}
        epoch = {}
        waiting = list(range(len(actors)))                          # not yet resident, in launch order
        active = waiting[:resident]
        waiting = waiting[resident:]
        while active:
            progressed = False
            n_act = len(active)
            start = rng.randrange(n_act) if schedule == "random" else 0
            for i in range(n_act):
                a = active[(start + i) % n_act]
                key = blocked.get(a)
                if key is not None and not _ge(s.flag(key), epoch[a]):
                    continue
                if a not in epoch:
                    epoch[a] = s.E if mutant == "epoch_not_incremented" else (s.E + 1) & MASK
                try:
                    r = next(actors[a])
                except StopIteration:
                    active.remove(a)
                    if waiting:
                        active.append(waiting.pop(0))
                    progressed = True
                    break
                if r is None:
                    blocked.pop(a, None)
                    progressed = True
                else:
                    if key is None or r != key:
                        progressed = True
                    blocked[a] = r
                if schedule == "random":
                    break
            if not progressed:
                stuck = sorted(blocked.get(a) for a in active if a in blocked)
                s.violations.append(("deadlock", f"call {call + 1}: {len(active)} resident CTAs blocked, e.g. on flag {stuck[:1]}"))
                return s.violations
        gathered = [n for n in range(num_n) if owners[n] >= 0]
        if s.done != 0 or any(s.flag((n, kb, h)) != s.E for n in gathered for kb in range(num_k) for h in (0, 1)) or \
                (mutant != "epoch_not_incremented" and s.E != call + 1):
            s.violations.append(("teardown", f"call {call + 1}: epoch {s.E}, done {s.done}"))
    return s.violations


def protocol_clears(M: int, N: int, K: int, G: int, owners: Sequence[int]) -> bool:
    """What the GPU tests assert before each launch: the model of their exact case finishes with no violation."""
    return run_protocol(M, N, K, G, owners) == []


def grid_of(M: int, N: int, max_ctas: int, sms: int = H100_SMS) -> int:
    """The gather launch's grid: one CTA per unit, at most one per SM, at most ``max_ctas`` (0: no cap)."""
    units = -(-M // 128) * -(-N // TILE_N)
    cap = sms if max_ctas <= 0 else min(max_ctas, sms)
    return min(units, cap)


MODEL_SHAPES = [(1, 2304, 768), (128, 2304, 768), (129, 776, 776), (1000, 2304, 768), (2048, 768, 2048), (127, 8, 64),
                (1000, 1024, 2048)]


@pytest.mark.parametrize("M,N,K", MODEL_SHAPES)
def test_protocol_is_clean_at_every_grid(M, N, K):
    """G = 1 ... 16, 131, 132 and every grid the GPU tests launch at this shape, round robin and at three random interleavings;
    every column gathered, and a table with local columns between gathered ones."""
    num_n = -(-N // TILE_N)
    units = -(-M // 128) * num_n
    grids = {min(G, units) for G in set(range(1, 17)) | {131, 132}} | {grid_of(M, N, c) for c in GPU_CTA_CAPS}
    for owners in ([1] * num_n, [(-1 if n % 3 == 1 else n % 4) for n in range(num_n)]):
        for G in sorted(grids):
            assert run_protocol(M, N, K, G, owners) == [], (G, owners)
            for seed in range(3):
                assert run_protocol(M, N, K, G, owners, schedule="random", seed=seed) == [], (G, seed)


@settings(max_examples=60, deadline=None)
@given(M=st.integers(1, 1500), n8=st.integers(1, 400), k8=st.integers(1, 100), G=st.integers(1, 132), pattern=st.integers(0, 2 ** 12 - 1),
       seed=st.integers(0, 3))
def test_protocol_is_clean_for_any_shape_and_grid(M, n8, k8, G, pattern, seed):
    N, K = 8 * n8, 8 * k8
    num_n = -(-N // TILE_N)
    owners = [(n % 8) if (pattern >> (n % 12)) & 1 else -1 for n in range(num_n)]
    assert run_protocol(M, N, K, G, owners, schedule="random" if seed else "rr", seed=seed) == []


# each mutant at a shape and grid where the kernel's real protocol is clean, and the check that must catch it
MUTANT_CASES = [
    ("m_blocks_descending", (1000, 2304, 768, 7), "deadlock"),
    ("pm2_lockstep", (1000, 2304, 768, 16), "deadlock"),
    ("fast_path_first_kblock", (1000, 2304, 768, 7), "read-before-store"),
    ("flag_before_wait_group", (1000, 2304, 768, 72), "flag-ahead-of-store"),
    ("epoch_not_incremented", (1000, 2304, 768, 72), "read-before-store"),
    ("oversubscribed", (1000, 2304, 768, 7), "deadlock"),
]


def test_every_protocol_mutant_is_caught():
    """Prints one row per mutant: the case, the first check that caught it, and every check that fired."""
    assert sorted(m for m, _, _ in MUTANT_CASES) == sorted(MUTANTS)
    rows = []
    for mutant, (M, N, K, G), want in MUTANT_CASES:
        assert run_protocol(M, N, K, G) == [], "the unmutated protocol must be clean here"
        v = run_protocol(M, N, K, G, mutant=mutant)
        checks = sorted({c for c, _ in v})
        rows.append((mutant, f"M {M} N {N} K {K} G {G}", v[0][0] if v else "-", ", ".join(checks)))
        assert v and v[0][0] == want, (mutant, v[:3])
    w = [max(len(r[i]) for r in rows) for i in range(4)]
    print("\nflag-protocol mutants:")
    print(f"  {'mutant':<{w[0]}}  {'case':<{w[1]}}  {'caught by':<{w[2]}}  all checks that fired")
    for r in rows:
        print(f"  {r[0]:<{w[0]}}  {r[1]:<{w[1]}}  {r[2]:<{w[2]}}  {r[3]}")


def test_oversubscription_is_the_only_limit_on_the_grid():
    """With every CTA resident the protocol is clean at any grid; the same grid with fewer resident CTAs than it launches can
    deadlock.  The GPU tests stay at one CTA per SM (``max_ctas`` <= the SM count)."""
    M, N, K = 1000, 2304, 768
    for G in (3, 7, 16):
        assert run_protocol(M, N, K, G) == []
    assert any(c == "deadlock" for c, _ in run_protocol(M, N, K, 7, resident=3))
