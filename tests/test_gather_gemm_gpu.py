"""Gather mode of the wgmma GEMM (``ops.gemm.gemm_tn_gather`` / ``GatherLinearFn``, train key ``fused_ag_gemm``) on one H100, with W
ranks emulated by W separate device buffers handed to the kernel as the peers' flat buffers.

The protocol needs no second GPU: the peer pointers are plain device addresses for ``cuTensorMapEncode``, and the flags, epoch and
done counter are local words shared by the CTAs of one grid.  So these tests run the real gatherer and waiter roles, the write-through,
the flags and the epoch logic.  They leave out only the NVLink path itself (peer reads bypass the local L2), which the ``multigpu``
tests cover.

Every case runs three calls through one ``GatheredWeight`` with new fresh weights each call: the stale value is NaN in the first and
the previous call's weights in the others, so a waiter that loads early sees finite but wrong bits.  Inputs come from
``test_gather_oracle.emulated_round_state``.  Per call: the exact tier bit for bit against ``bf16_rn`` of the fp64 product, or the
random tier within the fp64 bound and statistics of ``test_gemm_oracle`` and bit-equal to the same launch on a complete copy with an
all-local table; the write-through (the weight's local copy equals the fresh weights, the rest of the flat buffer and every peer buffer
unchanged); the epoch, done counter and flags; the launch count.  Before each launch the CPU protocol model must clear the case at
its grid.  Negative controls show that the checks see a wrong owner, a pulled tile left local and a plain GEMM on the stale copy."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops  # noqa: E402
from acco_b200.ops.gemm import TILE_K, TILE_N, GatheredWeight, fused_ag_tables, gemm_nn, gemm_tn, gemm_tn_gather, gemm_tt_acc  # noqa: E402
from test_gather_oracle import emulated_round_state, grid_of, protocol_clears  # noqa: E402
from test_gemm_oracle import check_random, dense_exact, exact_result, ints  # noqa: E402

DEV = "cuda"
NAN = float("nan")


def sms() -> int:
    return ops.load_ext(required=True).num_sms()


def ceil8(x) -> int:
    return -(-int(x) // 8) * 8


def layout(N: int, K: int, W: int, rank: int, kind: str):
    """``(offset, size_slice)`` of one weight in a flat buffer of ``W`` slices.  ``remote``: the whole weight inside one other rank's
    slice; ``one``: one owner boundary inside the weight; ``several``: the weight spread over every slice; ``every``: slices shorter
    than one 256-row tile, so every tile straddles a boundary and nothing is gathered."""
    NK = N * K
    if kind == "remote":
        S = ceil8(NK + 2048)
        o = W - 1 if rank != W - 1 else 0
        return o * S + 1024, S
    if kind == "one":
        S = ceil8(NK * 0.55) + 1024
        return S - ceil8(NK * 0.45), S
    if kind == "every":
        assert every_fits(N, K, W)
        return 1000, ceil8(TILE_N * K * 0.6)
    return 1000, ceil8((NK + 2048) / W)                               # several


def every_fits(N: int, K: int, W: int) -> bool:
    """Whether W slices shorter than one tile hold the weight (the ``every`` layout)."""
    return W * ceil8(TILE_N * K * 0.6) >= 1000 + N * K + 1024


def fresh(L: int, tier: str, seed: int) -> torch.Tensor:
    """Fresh weights: ``exact`` dense-exact integers, ``ints`` values in {-1, 0, 1} (the chains), ``random`` N(0, 1)."""
    if tier == "ints":
        return ints((L,), 1, seed, DEV)
    if tier == "exact":
        return dense_exact(1, L, seed, DEV)[0]
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(L, generator=g, device=DEV).to(torch.bfloat16)


def bits_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Bitwise equality (NaN payloads and signed zeros included)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    return torch.equal(a.contiguous().reshape(-1).view(torch.int16), b.contiguous().reshape(-1).view(torch.int16))


class Emulation:
    """One weight [N, K] at ``offset`` in a flat buffer of ``W`` slices of ``S``: the local flat buffer of rank ``rank``, W peer buffers
    (one per emulated rank, this rank's own included) and the ``GatheredWeight`` over them."""

    def __init__(self, N, K, W, rank, kind, tier, seed=0):
        self.N, self.K, self.W, self.rank, self.tier, self.seed = N, K, W, rank, tier, seed
        self.offset, self.S = layout(N, K, W, rank, kind)
        self.L = self.S * W
        assert self.offset + N * K <= self.L and self.offset % 8 == 0
        self.local = torch.empty(self.L, dtype=torch.bfloat16, device=DEV)
        self.peers = [torch.empty(self.L, dtype=torch.bfloat16, device=DEV) for _ in range(W)]
        self.gw = GatheredWeight(N, K, self.offset, [p.data_ptr() for p in self.peers], self.S, rank, DEV)
        self.truth = None
        self.round = 0

    @property
    def weights(self):
        return [(self.N, self.K, self.offset)]

    def w(self, flat) -> torch.Tensor:
        return flat[self.offset:self.offset + self.N * self.K].view(self.N, self.K)

    def next_round(self):
        """New fresh weights; the local copy's pulled tiles hold the stale value (NaN first, then the previous weights)."""
        stale = NAN if self.truth is None else self.truth
        self.round += 1
        self.truth = fresh(self.L, self.tier, 1000 * self.seed + self.round)
        local, peers = emulated_round_state(self.truth, stale, self.W, self.rank, self.weights, self.S, NAN)
        self.local.copy_(local)
        for p, q in zip(self.peers, peers):
            p.copy_(q)
        del local, peers

    def gathered_tiles(self):
        return [t for t, o in enumerate(self.gw.owners) if o >= 0]


def check_call(em: Emulation, y: torch.Tensor, x: torch.Tensor, before_local: torch.Tensor, epoch0: int, tag: str,
               ref: torch.Tensor = None):
    """The checks of one call (module docstring).  Returns the random tier's ratios (or None)."""
    N, K, off = em.N, em.K, em.offset
    tw = em.w(em.truth)
    stats = None
    if em.tier == "exact":
        assert bits_equal(y, exact_result(x, tw)), f"{tag}: y differs from bf16_rn(x w^T)"
    else:
        stats = check_random(y, x, tw)
        assert all(v <= 1.0 for v in stats.values()), (tag, stats)
        assert ref is not None and bits_equal(y, ref), f"{tag}: y differs from the all-local launch on a complete copy"
    # write-through: the weight's local copy is the fresh weights, the rest of the flat buffer is unchanged
    assert bits_equal(em.w(em.local), tw), f"{tag}: local copy not written through"
    assert bits_equal(em.local[:off], before_local[:off]) and bits_equal(em.local[off + N * K:], before_local[off + N * K:]), \
        f"{tag}: local buffer changed outside the weight"
    for r, p in enumerate(em.peers):                                 # every peer buffer unchanged: fresh in its slice, NaN elsewhere
        lo, hi = r * em.S, (r + 1) * em.S
        assert bits_equal(p[lo:hi], em.truth[lo:hi]), f"{tag}: peer {r} changed"
        assert bool(p[:lo].isnan().all()) and bool(p[hi:].isnan().all()), f"{tag}: peer {r} changed"
    # state and flags
    st = em.gw.state.tolist()
    assert st == [epoch0 + 1, 0], (tag, st, epoch0)
    num_n, num_k = -(-N // TILE_N), -(-K // TILE_K)
    fl = em.gw.flags.view(num_n, num_k, 2)
    owners = torch.tensor(em.gw.owners, device=DEV)
    assert bool((fl[owners >= 0] == epoch0 + 1).all()), f"{tag}: gathered flags not at the new epoch"
    assert bool((fl[owners < 0] == 0).all()), f"{tag}: flags of local tiles touched"
    return stats


def run_gather(em: Emulation, x: torch.Tensor, max_ctas: int, tag: str):
    """One call: re-poison, launch, check.  Returns the random tier's ratios."""
    em.next_round()
    before = em.local.clone()
    epoch0 = int(em.gw.state[0])
    n0 = ops.launch_counts().get("gemm_gather", 0)
    y = gemm_tn_gather(x, em.w(em.local), em.gw, max_ctas=max_ctas)
    assert ops.launch_counts().get("gemm_gather", 0) == n0 + 1
    ref = None
    if em.tier == "random":
        ref_gw = GatheredWeight(em.N, em.K, em.offset, [p.data_ptr() for p in em.peers], em.S, em.rank, DEV)
        ref_gw.tile_owner.fill_(-1)
        ref = gemm_tn_gather(x, em.w(em.truth).clone(), ref_gw, max_ctas=max_ctas)
    torch.cuda.synchronize()
    return check_call(em, y, x, before, epoch0, tag, ref)


SHAPES = [(2304, 768), (768, 2048), (16384, 2048), (50304, 768), (128256, 2048), (776, 776), (8, 64)]
MS = [1, 127, 128, 129, 1000, 2048, 8192]
KINDS = ["remote", "one", "several", "every"]
CAPS = [0, 1, 2, 7, 131]


def _cases():
    """A rotation through the product: every shape meets every M, both tiers, W 2 / 4 / 8 with the local rank first, in the middle
    and last, all four slice layouts and every CTA cap.  The three largest weights run on the default grid only, at M 128, 2048 and
    8192."""
    out = []
    for i, (N, K) in enumerate(SHAPES):
        big = N >= 16384
        for j, M in enumerate(MS):
            if big and M not in (128, 2048, 8192):
                continue
            W = (2, 4, 8)[(i + j) % 3]
            rank = (0, W // 2, W - 1)[(i + 2 * j) % 3]
            kind = KINDS[(i + j) % 4]
            if kind == "every" and not every_fits(N, K, W):
                kind = "several"
            cap = 0 if big else CAPS[(i + 3 * j) % 5]
            tier = ("exact", "random")[(i + j) % 2]
            out.append((M, N, K, W, rank, kind, cap, tier))
    return out


CASES = _cases()


@pytest.mark.parametrize("M,N,K,W,rank,kind,cap,tier", CASES, ids=[f"M{c[0]}-N{c[1]}-K{c[2]}-W{c[3]}r{c[4]}-{c[5]}-cap{c[6]}-{c[7]}" for c in CASES])
def test_gather_gemm(M, N, K, W, rank, kind, cap, tier):
    em = Emulation(N, K, W, rank, kind, tier, seed=M + N + K)
    G = grid_of(M, N, cap, sms())
    assert protocol_clears(M, N, K, G, em.gw.owners), "the flag-protocol model does not clear this case"
    x = dense_exact(M, K, 7, DEV) if tier == "exact" else \
        torch.randn(M, K, generator=torch.Generator(device=DEV).manual_seed(7), device=DEV).to(torch.bfloat16)
    worst = {}
    for call in range(3):
        stats = run_gather(em, x, cap, f"call {call + 1}")
        for k, v in (stats or {}).items():
            worst[k] = max(worst.get(k, 0.0), v)
    gathered = len(em.gathered_tiles())
    desc = ", ".join(f"{k} {v:.3f}" for k, v in sorted(worst.items())) or "bit-exact"
    print(f"\ngather M {M} N {N} K {K} W {W} rank {rank} {kind} cap {cap} grid {G}: {gathered}/{len(em.gw.owners)} tiles gathered; {desc}")


# ---------------------------------------------------------------------------------------------- negative controls
def test_negative_controls_are_detected():
    """Three broken calls that keep every pointer valid, each of which the checks above must reject."""
    M, N, K, W, rank = 1000, 2304, 768, 4, 0
    x = dense_exact(M, K, 3, DEV)
    found = {}

    def detected(fn) -> bool:
        try:
            fn()
        except AssertionError:
            return True
        return False

    for control in ("wrong owner", "pulled tile left local", "plain gemm on the stale copy"):
        em = Emulation(N, K, W, rank, "several", "exact", seed=5)
        tiles = em.gathered_tiles()
        assert len(tiles) >= 2
        t = tiles[len(tiles) // 2]
        if control == "wrong owner":
            o = em.gw.owners[t]
            em.gw.tile_owner[t] = (o + 1) % W                       # that rank's buffer holds NaN over this tile
        elif control == "pulled tile left local":
            em.gw.tile_owner[t] = -1

        def broken():
            for call in range(2):                                    # the second call sees finite stale bits
                if control == "plain gemm on the stale copy":
                    em.next_round()
                    y = gemm_tn(x, em.w(em.local))
                    torch.cuda.synchronize()
                    assert bits_equal(y, exact_result(x, em.w(em.truth)))
                else:
                    run_gather(em, x, 0, f"{control}, call {call + 1}")
        found[control] = detected(broken)
        print(f"\nnegative control '{control}': {'detected' if found[control] else 'NOT detected'}")
    assert all(found.values()), found


# ---------------------------------------------------------------------------------------------- chains, graphs, PDL
def _chain_operands(M, N, K):
    """Exact through the chain: x has one +-1 per row, w is in {-1, 0, 1}, dy has four +-1 per row, so y, dx = dy w and every
    partial of the wgrad are small integers that bf16 and fp32 hold exactly in any order."""
    g = torch.Generator(device=DEV).manual_seed(11)
    x = torch.zeros(M, K, dtype=torch.bfloat16, device=DEV)
    x[torch.arange(M, device=DEV), torch.randint(0, K, (M,), generator=g, device=DEV)] = \
        (torch.randint(0, 2, (M,), generator=g, device=DEV) * 2 - 1).to(torch.bfloat16)
    dy = torch.zeros(M, N, dtype=torch.bfloat16, device=DEV)
    for _ in range(4):
        dy[torch.arange(M, device=DEV), torch.randint(0, N, (M,), generator=g, device=DEV)] = \
            (torch.randint(0, 2, (M,), generator=g, device=DEV) * 2 - 1).to(torch.bfloat16)
    return x, dy, ints((N, K), 8, 12, DEV)


def _chain(x, dy, w_local, gw, grad):
    y = gemm_tn_gather(x, w_local, gw)
    dx = gemm_nn(dy, w_local)                       # reads the copy the gather just completed
    gemm_tt_acc(dy, x, grad)
    return y, dx


def _check_chain(em, x, dy, y, dx, grad, g0, tag):
    tw = em.w(em.truth)
    clean = tw.clone()
    g_clean = g0.clone()
    y_c, dx_c = gemm_tn(x, clean), gemm_nn(dy, clean)
    gemm_tt_acc(dy, x, g_clean)
    torch.cuda.synchronize()
    for got, want, exact, name in ((y, y_c, exact_result(x, tw), "y"), (dx, dx_c, exact_result(dy, tw.t()), "dx"),
                                   (grad, g_clean, exact_result(dy.t(), x.t(), C=g0), "grad")):
        assert bits_equal(got, want) and bits_equal(got, exact), f"{tag}: {name}"
    assert bits_equal(em.w(em.local), tw), f"{tag}: write-through"


def test_chain_eager_and_graph():
    """The gather GEMM, then the dgrad reading the copy it completed and the wgrad, back to back with no host sync: eagerly for three
    calls, then captured once in a CUDA graph and replayed for three more, with the fresh weights and the stale copy rewritten between
    replays.  The epoch is read from device memory, so every replay gathers again."""
    M, N, K = 1000, 2304, 768
    em = Emulation(N, K, 4, 1, "several", "ints", seed=9)
    assert protocol_clears(M, N, K, grid_of(M, N, 0, sms()), em.gw.owners)
    x, dy, g0 = _chain_operands(M, N, K)
    grad = g0.clone()
    for call in range(3):
        em.next_round()
        grad.copy_(g0)
        y, dx = _chain(x, dy, em.w(em.local), em.gw, grad)
        torch.cuda.synchronize()
        _check_chain(em, x, dy, y, dx, grad, g0, f"eager call {call + 1}")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            grad.copy_(g0)
            y, dx = _chain(x, dy, em.w(em.local), em.gw, grad)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    for call in range(3):
        em.next_round()                                             # rewrites truth, peers and the stale copy in place
        e0 = int(em.gw.state[0])
        graph.replay()
        torch.cuda.synchronize()
        assert int(em.gw.state[0]) == e0 + 1
        _check_chain(em, x, dy, y, dx, grad, g0, f"graph replay {call + 1}")


def test_chain_without_programmatic_dependent_launch():
    """``ACCO_GEMM_PDL`` is read once per process: the chain again in a fresh one with PDL off."""
    if os.environ.get("ACCO_GEMM_PDL") == "0":
        pytest.skip("already the PDL-off run")
    env = dict(os.environ, ACCO_GEMM_PDL="0")
    py = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    p = subprocess.run(py + ["-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                        f"{os.path.abspath(__file__)}::test_chain_eager_and_graph"], env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600, cwd=os.path.dirname(os.path.abspath(__file__)))
    assert p.returncode == 0 and "1 passed" in p.stdout, p.stdout[-3000:]


# ---------------------------------------------------------------------------------------------- the linear layer
@pytest.mark.parametrize("grad_dtype", [torch.bfloat16, torch.float32], ids=["bf16-grad", "fp32-main_grad"])
def test_linear_forward_backward(grad_dtype):
    """``ops.linear(x, w, gathered=gw)`` forward and backward over two micro-batches (the second without ``gathered``, as the model
    runs it) against the same calls on a complete local copy with an all-local table: y, dx and the accumulated gradient bit for bit
    (exact operands), into a bf16 ``.grad`` or an fp32 ``main_grad`` with no ``.grad`` beside it."""
    M, N, K = 1000, 2304, 768
    em = Emulation(N, K, 4, 2, "several", "ints", seed=13)
    x0, dy, g0 = _chain_operands(M, N, K)
    em.next_round()

    def setup(flat, table):
        w = em.w(flat).detach().requires_grad_(True)
        gbuf = g0.to(grad_dtype).clone()
        if grad_dtype == torch.float32:
            w.main_grad = gbuf
        else:
            w.grad = gbuf
        return w, gbuf, table

    complete = em.truth.clone()
    ref_gw = GatheredWeight(N, K, em.offset, [p.data_ptr() for p in em.peers], em.S, em.rank, DEV)
    ref_gw.tile_owner.fill_(-1)
    runs = {}
    for name, flat, table in (("gathered", em.local, em.gw), ("complete", complete, ref_gw)):
        w, gbuf, table = setup(flat, table)
        outs = []
        for mb in range(2):
            x = x0.clone().requires_grad_(True)
            y = ops.linear(x, w, gathered=table if mb == 0 else None)
            y.backward(dy)
            outs += [y.detach(), x.grad]
        torch.cuda.synchronize()
        assert w.grad is None if grad_dtype == torch.float32 else w.grad is gbuf
        runs[name] = outs + [gbuf]
    for a, b in zip(runs["gathered"], runs["complete"]):
        assert a.dtype == b.dtype and torch.equal(a, b)
    assert bits_equal(em.w(em.local), em.w(em.truth))
    want = exact_result(dy.t(), x0.t(), C=g0).to(grad_dtype)
    if grad_dtype == torch.bfloat16:                                 # two micro-batches: g0 + 2 dy^T x, all exact integers
        want = exact_result(dy.t(), x0.t(), C=want)
    else:
        want = g0.double() + 2 * (dy.double().t() @ x0.double())
    assert torch.equal(runs["gathered"][-1].double(), want.double())


# ---------------------------------------------------------------------------------------------- model wiring
LLAMA125 = dict(vocab_size=50257, hidden_size=768, intermediate_size=2048, num_hidden_layers=2, num_attention_heads=12,
                num_key_value_heads=12, max_position_embeddings=1024)
LLAMA1B_UNTIED = dict(vocab_size=128256, hidden_size=2048, intermediate_size=8192, num_hidden_layers=2, num_attention_heads=32,
                      num_key_value_heads=8, max_position_embeddings=8192, rope_theta=500000.0, tie_word_embeddings=False,
                      rope_scaling=dict(rope_type="llama3", factor=32.0, low_freq_factor=1.0, high_freq_factor=4.0,
                                        original_max_position_embeddings=8192))
MODEL_CASES = [("llama125m", LLAMA125, 4, 1, 8, 1024), ("llama1b-untied-128256", LLAMA1B_UNTIED, 2, 1, 2, 2048)]
GRAD_REL_TOL = 2.0 ** -6


class _Rank:
    """One emulated rank's model in a ``FlatArena(world=W, rank)`` with the symmetric backend's slice alignment, W peer buffers per
    theta buffer and the trainer's tables over them."""

    def __init__(self, cfg, W, rank, peers=None):
        from acco_b200.models import LlamaConfig, LlamaForCausalLM
        from acco_b200.parallel.arena import FlatArena
        torch.manual_seed(0)
        self.model = LlamaForCausalLM(LlamaConfig(**cfg)).to(DEV).to(torch.bfloat16)
        self.arena = FlatArena(self.model, W, rank, torch.bfloat16, DEV, align=1024)
        self.W, self.rank, self.S = W, rank, self.arena.layout.size_slice
        L = self.arena.layout.padded
        self.peers = peers or [[torch.empty(L, dtype=torch.bfloat16, device=DEV) for _ in range(W)] for _ in range(2)]
        bases = [[p.data_ptr() for p in ps] for ps in self.peers]
        self.table, _ = fused_ag_tables(self.model, self.arena, bases, self.S, rank, DEV)
        self.model._ag_table = self.table
        off = {id(p): o for p, o in zip(self.arena.params, self.arena.offsets)}
        self.weights = [(p.shape[0], p.shape[1], off[id(p)]) for p in self.model.fused_ag_candidates() if id(p) in self.table]

    def micro_batch(self, ids, pending):
        m = self.model
        m._ag_idx, m._ag_pending = self.arena.live, pending
        self.arena.acc[self.arena.grad_idx].zero_()
        loss = m(input_ids=ids, labels=ids).loss
        loss.backward()
        return loss.detach()


def _round(ranks, idx, truth, stale):
    """Round state for ``theta[idx]``: ``ranks[0]`` gets the stale copy, the twin ``ranks[1]`` the complete one; both share peers."""
    a, twin = ranks
    local, peers = emulated_round_state(truth, stale, a.W, a.rank, a.weights, a.S, NAN)
    a.arena.theta[idx].copy_(local)
    twin.arena.theta[idx].copy_(truth)
    for p, q in zip(a.peers[idx], peers):
        p.copy_(q)


def _fresh_theta(arena, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    t = arena.theta[0].clone()
    n = arena.numel
    t[:n] = (t[:n].float() + 0.02 * torch.randn(n, generator=g, device=DEV)).to(torch.bfloat16)
    return t


def _grads_close(a, b, tag):
    for (pa, pb) in zip(a.arena.params, b.arena.params):
        ga, gb = pa.grad.float(), pb.grad.float()
        rel = float((ga - gb).norm() / gb.norm().clamp_min(1e-30))
        assert rel <= GRAD_REL_TOL, (tag, tuple(pa.shape), rel)


@pytest.mark.parametrize("case", MODEL_CASES, ids=[c[0] for c in MODEL_CASES])
def test_model_micro_batch_gathers_like_a_complete_copy(case):
    """One pending micro-batch as the trainer runs it, against a twin whose local copy is already complete (same tables, same
    peers): loss and logits bit for bit; ``theta[live]`` equal to the fresh weights afterwards; every gradient within
    ``GRAD_REL_TOL`` of the twin's (the split-K wgrad and dgrad add their partials in arrival order, so gradient bits vary from run to
    run; a stale tile moves a gradient by O(1)); the next micro-batch (nothing pending) equal to the twin's.  Then both theta buffers:
    a flip with ``point_params`` and a gather into ``theta[1]``.  The step is held to the whole-step fp64 criterion of
    ``test_step_oracle.step_ratios``, and one replay of the pending micro-batch's CUDA graph (``MicroBatchGraphs``, keyed as
    ``gradient_step`` keys it) gathers a new round."""
    from acco_b200.parallel.graphs import MicroBatchGraphs
    from test_step_oracle import hf_from_native, hf_grads, native_grads, run_step, step_ratios, zipf_ids
    name, cfg, W, rank, B, S = case
    a = _Rank(cfg, W, rank)
    twin = _Rank(cfg, W, rank, peers=a.peers)
    assert a.table and all(len(v) == 2 for v in a.table.values())
    assert any(o >= 0 for gws in a.table.values() for o in gws[0].owners)
    V = a.model.config.vocab_size
    ids = [zipf_ids(B * S, V, seed=200 + i).view(B, S).to(DEV) for i in range(3)]
    truth = _fresh_theta(a.arena, 1)
    for idx in (0, 1):
        a.arena.point_params(idx)
        twin.arena.point_params(idx)
        stale = NAN if idx == 0 else truth
        truth = _fresh_theta(a.arena, 10 + idx)
        _round((a, twin), idx, truth, stale)
        n0 = ops.launch_counts().get("gemm_gather", 0)
        la, lt = a.micro_batch(ids[0], True), twin.micro_batch(ids[0], True)
        torch.cuda.synchronize()
        assert ops.launch_counts().get("gemm_gather", 0) - n0 == 2 * len(a.table)
        assert bits_equal(la, lt) and bool(torch.isfinite(la)), (idx, float(la), float(lt))
        assert bits_equal(a.arena.theta[idx], truth), f"theta[{idx}] is not the fresh weights after the pending forward"
        _grads_close(a, twin, f"theta[{idx}] pending")
        if idx == 0:                                                 # whole-step criterion against HF fp64, HF bf16 as yardstick
            hf16 = hf_from_native(a.model, torch.bfloat16, DEV, attn="sdpa")
            hf64 = hf_from_native(a.model, torch.float64, DEV, attn="eager")
            run_step(hf16, [ids[0]], 0.0, hf_V=V)
            run_step(hf64, [ids[0]], 0.0, hf_V=V)
            r = step_ratios(native_grads(a.model), hf_grads(hf64), hf_grads(hf16), "model.embed_tokens.weight", ids[0])
            worst = max(r.items(), key=lambda kv: kv[1])
            print(f"\n{name}: worst e(ours) / (2 e(HF bf16) + floor) = {worst[1]:.3f} ({worst[0]})")
            assert worst[1] <= 1.0, r
            del hf16, hf64
        la, lt = a.micro_batch(ids[1], False), twin.micro_batch(ids[1], False)
        assert bits_equal(la, lt), (idx, float(la), float(lt))
        _grads_close(a, twin, f"theta[{idx}] next micro-batch")
        with torch.no_grad():
            a.model._ag_pending = twin.model._ag_pending = False
            assert bits_equal(a.model(input_ids=ids[2]).logits, twin.model(input_ids=ids[2]).logits)

    # CUDA graph of the pending micro-batch, keyed as gradient_step keys it, replayed after a new emulated round
    idx = a.arena.live

    def step(b):
        a.model._ag_idx, a.model._ag_pending = a.arena.live, True
        loss = a.model(input_ids=b["input_ids"], labels=b["input_ids"]).loss
        loss.backward()
        return loss.detach()

    graphs = MicroBatchGraphs(step, DEV)
    host = {"input_ids": ids[0]}
    key = (a.arena.live, a.arena.grad_idx, True, MicroBatchGraphs.signature(host))
    graphs.capture(key, host, cleanup=lambda: a.arena.acc[a.arena.grad_idx].zero_())
    stale, truth = truth, _fresh_theta(a.arena, 99)
    _round((a, twin), idx, truth, stale)
    a.arena.acc[a.arena.grad_idx].zero_()
    e0 = [int(gws[idx].state[0]) for gws in a.table.values()]
    la = graphs.replay(key, host)
    lt = twin.micro_batch(ids[0], True)
    torch.cuda.synchronize()
    assert [int(gws[idx].state[0]) for gws in a.table.values()] == [e + 1 for e in e0]
    assert float(la) == float(lt), (float(la), float(lt))
    assert bits_equal(a.arena.theta[idx], truth)
    _grads_close(a, twin, "graph replay")
