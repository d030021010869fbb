"""Property-based tests (hypothesis) for the pure-Python building blocks."""
import numpy as np
import pytest
import torch

hypothesis = pytest.importorskip("hypothesis")
from hypothesis import given, settings, strategies as st

from acco_b200.data.packing import pack_const_len
from acco_b200.optim import AdamHyper, adamw_shard_update_
from acco_b200.parallel.arena import ShardLayout
from acco_b200.parallel.schedule import COMMIT_ALL, COMMIT_NONE, RoundScheduler
from acco_b200.utils.hostlist import collect_hostlist, expand_hostlist


@settings(max_examples=200, deadline=None)
@given(n=st.integers(1, 10 ** 9), world=st.integers(1, 16), align=st.sampled_from([1, 8, 1024]))
def test_shard_layout_partitions_the_vector(n, world, align):
    lay = ShardLayout(n, world, align)
    assert lay.size_slice % align == 0 and lay.padded >= n and lay.padded - n < world * max(align, 1) + world
    covered = 0
    for r in range(world):
        lo, hi = lay.bounds(r)
        assert 0 <= lo <= hi <= n and hi - lo <= lay.size_slice
        assert lo == min(r * lay.size_slice, n)
        covered += hi - lo
    assert covered == n
    assert lay.owner_of(n - 1) < world


@settings(max_examples=100, deadline=None)
@given(lens=st.lists(st.integers(0, 30), min_size=0, max_size=40), L=st.integers(1, 17), eos=st.integers(0, 5))
def test_packing_is_concatenate_with_eos_then_reshape(lens, L, eos):
    rng = np.random.default_rng(sum(lens) + L)
    docs = [rng.integers(10, 99, size=n).tolist() for n in lens]
    flat = [t for d in docs for t in (d + [eos])]
    rows = len(flat) // L
    got = pack_const_len(docs, L, eos)
    assert got.shape == (rows, L)
    assert got.reshape(-1).tolist() == flat[: rows * L]


@settings(max_examples=60, deadline=None)
@given(hosts=st.lists(st.tuples(st.sampled_from(["n", "gpu", "node-a"]), st.integers(0, 300)), min_size=1, max_size=25, unique=True))
def test_hostlist_roundtrip(hosts):
    names = [f"{p}{i}" for p, i in hosts]
    assert sorted(expand_hostlist(collect_hostlist(names))) == sorted(names)


@settings(max_examples=50, deadline=None)
@given(method=st.sampled_from(["acco", "dpu", "ddp"]), warm=st.integers(0, 3), n=st.integers(1, 12),
       counts=st.lists(st.integers(1, 5), min_size=12, max_size=12))
def test_scheduler_invariants(method, warm, n, counts):
    s = RoundScheduler(method, n_warmup_rounds=warm)
    prev_write = None
    stash = 0
    total = 0
    for i in range(n):
        before = s.compute_buffers(round_in_flight=False)
        p = s.next_plan()
        assert p.read_acc == before["acc"]                      # the round consumes what compute was just writing
        if prev_write is not None:
            assert before["theta"] == prev_write                # compute runs on the newest gathered weights
        during = s.compute_buffers(round_in_flight=True)
        assert during["acc"] != p.read_acc and during["theta"] != p.write_theta
        c = counts[i]
        upd = c + (stash if p.add_stash else 0)
        if p.write_stash:
            stash = c
        s.complete(p, upd)
        if p.counts_toward_total:
            total += upd
        assert (p.commit == COMMIT_NONE) == (p.kind == "tentative")
        assert (p.commit == COMMIT_ALL) == (p.kind != "tentative")
        prev_write = p.write_theta
    assert s.count_grad_tot == total and s.count_com == n


@settings(max_examples=40, deadline=None)
@given(seed=st.integers(0, 10 ** 6), n1=st.integers(1, 4), n2=st.integers(1, 4))
def test_tentative_plus_real_equals_one_large_batch_step(seed, n1, n2):
    """ACCO's two half-rounds commit exactly the AdamW step of the mean over all n1+n2 micro-gradients."""
    g = torch.Generator().manual_seed(seed)
    p0 = torch.randn(32, generator=g)
    grads = [torch.randn(32, generator=g) for _ in range(n1 + n2)]
    master, m, v, stash, out = p0.clone(), torch.zeros(32), torch.zeros(32), torch.zeros(32), torch.zeros(32)
    adamw_shard_update_(sum(grads[:n1]), master, m, v, stash, out, AdamHyper(lr=1e-2, step=1, inv_count=1.0 / n1, commit=COMMIT_NONE, write_stash=True))
    assert torch.equal(master, p0)
    adamw_shard_update_(sum(grads[n1:]), master, m, v, stash, out, AdamHyper(lr=1e-2, step=1, inv_count=1.0 / (n1 + n2), commit=COMMIT_ALL, add_stash=True))
    ref = p0.clone().requires_grad_(True)
    opt = torch.optim.AdamW([ref], lr=1e-2, betas=(0.9, 0.999), weight_decay=0.01)
    ref.grad = sum(grads) / (n1 + n2)
    opt.step()
    torch.testing.assert_close(master, ref.detach(), rtol=1e-5, atol=1e-6)


# ----------------------------------------------------------------------------------------------
# GEMM work decomposition (mirrors `decode_unit` / the unit loops of csrc/gemm_wgmma.cu)
# ----------------------------------------------------------------------------------------------
def _gemm_units(M, N, K, bn, splits, pm, pn, slots):
    """Python twin of the device-side tile scheduler: yields (cluster, cta, mb, n_blk, kb0, kb1) for every unit every CTA runs.
    A CTA computes 128-row tiles; a cluster is pm x pn CTAs (cluster rank = pi * pn + pj) owning a super-tile of pm x pn tiles."""
    BM, BK = 128, 64
    num_n, num_k = -(-N // bn), -(-K // BK)
    num_mb = -(-M // BM)
    num_sn = -(-num_n // pn)
    tiles = -(-num_mb // pm) * num_sn
    splits = max(1, min(splits, num_k))
    kbs = -(-num_k // splits)
    splits = -(-num_k // kbs)
    num_units = tiles * splits
    grid_clusters = min(num_units, slots)
    for cl in range(grid_clusters):
        for cta in range(pm * pn):
            pi, pj = divmod(cta, pn)
            t = cl
            while t < num_units:
                s, tile = divmod(t, tiles)
                smb, sn = divmod(tile, num_sn)
                yield cl, cta, smb * pm + pi, sn * pn + pj, s * kbs, min(num_k, s * kbs + kbs)
                t += grid_clusters
    return


@settings(max_examples=150, deadline=None)
@given(M=st.integers(1, 3000), N=st.integers(8, 1500), K=st.integers(8, 4000), bn=st.sampled_from([64, 128, 256]),
       splits=st.integers(1, 9), pm=st.sampled_from([1, 2]), pn=st.sampled_from([1, 2]), slots=st.integers(1, 132))
def test_gemm_tile_scheduler_covers_every_output_k_block_exactly_once(M, N, K, bn, splits, pm, pn, slots):
    """Every real (m-block, n-block, k-block) triple is computed by exactly one CTA; phantom tiles (odd counts under clusters) lie
    entirely outside the matrix (TMA zero-fills their loads, the epilogue stores nothing); all CTAs of a cluster run the same number
    of k-iterations (they share pipeline stages through multicast), and no split is empty."""
    BM = 128
    num_mb, num_n, num_k = -(-M // BM), -(-N // bn), -(-K // 64)
    seen = {}
    per_cta_iters = {}
    for cl, cta, mb, n_blk, kb0, kb1 in _gemm_units(M, N, K, bn, splits, pm, pn, slots):
        assert kb1 > kb0                                             # no empty split
        per_cta_iters[(cl, cta)] = per_cta_iters.get((cl, cta), 0) + (kb1 - kb0)
        real = mb < num_mb and n_blk < num_n
        if not real:
            assert mb * BM >= M or n_blk * bn >= N                   # phantom tile: fully out of range
            continue
        for kb in range(kb0, kb1):
            key = (mb, n_blk, kb)
            assert key not in seen, key
            seen[key] = True
    assert len(seen) == num_mb * num_n * num_k
    by_cluster = {}
    for (cl, cta), it in per_cta_iters.items():
        by_cluster.setdefault(cl, set()).add(it)
    assert all(len(v) == 1 for v in by_cluster.values())           # lock-step inside a cluster
