"""An fp64 oracle of causal / sliding-window / document-masked attention, written from first principles, and the tolerances the GPU
tests of the flash-attention kernels (``test_attention_kernels_gpu.py``) use, with the evidence that they are the right size.

The oracle decides visibility from per-token document ids and row positions alone (``kv <= q``, ``q - kv < window``, same document)
and returns O, LSE, dQ, dK and dV in fp64 through an explicit backward.  It shares no code with ``ops.attention``: the production
SDPA fallback builds its mask with ``_window_mask`` / ``_seg_mask``, so a reference built on them could not catch their bugs.

The margin table (``test_margin_table``) runs every GPU case, or a scaled-down twin of it, on the CPU and asserts two things:

* the blockwise emulator of the kernels (``attention_blockwise_ref`` / ``attention_blockwise_bwd_ref``, which copy the kernels' bf16
  rounding points) stays within half of each tolerance of the oracle, so an honest bf16 kernel passes with room to spare;
* every mask mutant (window +-1, diagonal excluded, one key into the future, segment start -1 / +1, scale 1/8 for 1.0) lands more
  than 3x a tolerance away from the oracle, either on the dense comparison or on one of the mask-edge probes, and the table says
  which check caught it.  Probes plant a key that dominates the softmax just outside (and a twin just inside) each mask edge."""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import numpy as np
import pytest
import torch

D = 64

# Dense tolerances: O and LSE max abs error; dQ / dK / dV max abs error relative to the largest oracle gradient.  Sized by the
# margin table: the emulator reaches 7.9e-3 on O at scale 1.0 (GPT-Neo's sharp softmax) and 6.5e-3 on dK, so these are the tightest
# round values it passes with half to spare.  The LSE comes from fp32 scores of exact bf16 products: the kernels stay below 5e-6 on
# an H100 (GPT-Neo scale 1.0), the emulator below 4e-6.  A one-key mask error is below the O / dV tolerances on the dense
# comparison (one key among hundreds); the LSE and the probes are what see it, by factors of thousands.
TOL = {"o": 2e-2, "lse": 5e-5, "dq": 1.5e-2, "dk": 1.5e-2, "dv": 1.5e-2}
# Probe tolerance (values near the planted 64 carry bf16 output rounding): |got - want| <= PROBE_ATOL + PROBE_RTOL * |want|.
PROBE_ATOL, PROBE_RTOL = 1e-2, 1e-2
# A probe query's LSE is about 128 * scale: fp32 scores carry a relative error, on top of TOL["lse"].
PROBE_LSE_RTOL = 1e-5
PLANT_V = 64.0


# ---------------------------------------------------------------------------------------------- rows and visibility
def doc_ids(lengths: Sequence[Sequence[int]], S: int) -> torch.Tensor:
    """Sample lengths of each row -> int64 document ids [B, S] (0, 1, 2, ... along each row)."""
    rows = []
    for row in lengths:
        assert sum(row) == S and all(n > 0 for n in row), row
        rows.append(torch.repeat_interleave(torch.arange(len(row)), torch.tensor(list(row))))
    return torch.stack(rows)


def seg_starts_of(lengths: Sequence[Sequence[int]], S: int) -> torch.Tensor:
    """The kernels' encoding of the same rows: int32 [B*S], the row position at which each token's sample starts."""
    out = np.zeros((len(lengths), S), dtype=np.int32)
    for b, row in enumerate(lengths):
        a = 0
        for n in row:
            out[b, a:a + n] = a
            a += n
    return torch.from_numpy(out.reshape(-1))


def lengths_of_seg(seg: torch.Tensor, B: int, S: int) -> List[List[int]]:
    """Inverse of :func:`seg_starts_of` (for rows made by ``test_packing.random_seg``)."""
    seg = seg.view(B, S).tolist()
    out = []
    for row in seg:
        starts = sorted(set(row)) + [S]
        out.append([starts[i + 1] - starts[i] for i in range(len(starts) - 1)])
    return out


def visibility(doc: torch.Tensor, window: int, mutant: Optional[str] = None) -> torch.Tensor:
    """bool [B, S, S] (query, key): key kv is visible from query q iff kv <= q, q - kv < window (window <= 0 or >= S: no window)
    and both tokens belong to the same document.  ``mutant`` moves one edge by one key (for the margin table)."""
    B, S = doc.shape
    pos = torch.arange(S, device=doc.device)
    qp, kp = pos[:, None], pos[None, :]
    vis = kp <= qp + (1 if mutant == "future" else 0)
    if mutant == "diag":
        vis = vis & (kp != qp)
    if 0 < window < S:
        w = window + {"window+1": 1, "window-1": -1}.get(mutant, 0)
        vis = vis & (qp - kp < w)
    if mutant in ("seg-1", "seg+1"):
        new = torch.ones_like(doc, dtype=torch.bool)
        new[:, 1:] = doc[:, 1:] != doc[:, :-1]
        start = torch.where(new, pos[None, :], torch.zeros_like(pos)[None, :]).cummax(dim=1).values
        shift = -1 if mutant == "seg-1" else 1
        return vis[None] & (kp[None] >= (start + shift)[:, :, None])
    return vis[None] & (doc[:, :, None] == doc[:, None, :])


# ---------------------------------------------------------------------------------------------- the oracle
def oracle(q, k, v, d_o, scale: float, vis: torch.Tensor, groups: Optional[Sequence[int]] = None,
           vis_bwd: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """q [B,S,Hq,D], k / v [B,S,Hk,D], d_o [B,S,Hq,D] or None, vis bool [B,S,S] -> fp64 {o [B,S,h,D], lse [B,h,S] (natural log),
    dq [B,S,h,D], dk / dv [B,S,g,D]} for the KV groups ``groups`` (default: all) and their h = len(groups) * Hq/Hk query heads.
    A query that sees no key gets O = 0 and LSE = -inf.  ``vis_bwd`` (margin table only): a different mask for the backward, which
    then rebuilds P as exp(score - LSE) the way the kernel's backward does, so a backward-only mask error can be modelled."""
    B, S, Hq, _ = q.shape
    Hk = k.shape[2]
    G = Hq // Hk
    groups = list(range(Hk)) if groups is None else list(groups)
    vis = vis.to(q.device)
    o, lse, dq, dk, dv = [], [], [], [], []
    for g in groups:
        K, V = k[:, :, g].double(), v[:, :, g].double()
        dK = torch.zeros_like(K)
        dV = torch.zeros_like(V)
        for h in range(g * G, (g + 1) * G):
            Q = q[:, :, h].double()
            s = (Q @ K.transpose(1, 2) * scale).masked_fill(~vis, float("-inf"))
            m = s.amax(dim=-1, keepdim=True)
            m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
            e = torch.exp(s - m)
            l = e.sum(dim=-1, keepdim=True)
            p = e / torch.where(l > 0, l, torch.ones_like(l))
            O = p @ V
            o.append(O)
            lse.append((torch.log(l) + m).squeeze(-1))
            if vis_bwd is not None:
                L = lse[-1][..., None]
                s = (Q @ K.transpose(1, 2) * scale).masked_fill(~vis_bwd.to(q.device), float("-inf"))
                p = torch.where(torch.isfinite(L), torch.exp(s - torch.where(torch.isfinite(L), L, torch.zeros_like(L))), torch.zeros_like(s))
            del s, e
            if d_o is not None:
                dO = d_o[:, :, h].double()
                dV += p.transpose(1, 2) @ dO
                ds = p * (dO @ V.transpose(1, 2) - (dO * O).sum(dim=-1, keepdim=True))
                dq.append(ds @ K * scale)
                dK += ds.transpose(1, 2) @ Q * scale
                del ds
            del p
        dk.append(dK)
        dv.append(dV)
    out = {"o": torch.stack(o, dim=2), "lse": torch.stack(lse, dim=1)}
    if d_o is not None:
        out.update(dq=torch.stack(dq, dim=2), dk=torch.stack(dk, dim=2), dv=torch.stack(dv, dim=2))
    return out


def heads_of(groups: Sequence[int], Hq: int, Hk: int) -> List[int]:
    G = Hq // Hk
    return [h for g in groups for h in range(g * G, (g + 1) * G)]


# ---------------------------------------------------------------------------------------------- inputs and metrics
def make_qkv(B, S, Hq, Hk, seed, d=D):
    """The inputs of the existing kernel tests: bf16 ``qkv [B*S, (Hq+2Hk)*d]`` (randn * 0.7) and ``d_o [B*S, Hq*d]`` (randn * 0.5)."""
    g = torch.Generator().manual_seed(seed)
    qkv = (torch.randn(B * S, (Hq + 2 * Hk) * d, generator=g) * 0.7).to(torch.bfloat16)
    d_o = (torch.randn(B * S, Hq * d, generator=g) * 0.5).to(torch.bfloat16)
    return qkv, d_o


def split(qkv, B, S, Hq, Hk, d=D):
    x = qkv.view(B, S, Hq + 2 * Hk, d)
    return x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:]


def dense_errors(got: Dict[str, torch.Tensor], want: Dict[str, torch.Tensor]) -> Dict[str, float]:
    """Error per quantity in the units of ``TOL``: max abs for O / LSE, max abs over the largest oracle value for gradients.
    A non-finite difference (a row that lost all its keys) counts as infinite.  A gradient that is zero everywhere (rows of length-1
    samples: every softmax is a single 1, so dK = 0) is compared in absolute terms."""
    out = {}
    for name in ("o", "lse", "dq", "dk", "dv"):
        if name not in got or name not in want:
            continue
        diff = torch.nan_to_num((got[name].double() - want[name].double()).abs(), nan=math.inf)
        err = float(diff.max())
        if name.startswith("d"):
            err /= float(want[name].abs().max()) or 1.0
        out[name] = err
    return out


def dense_ratios(got, want) -> Dict[str, float]:
    return {k: e / TOL[k] for k, e in dense_errors(got, want).items()}


# ---------------------------------------------------------------------------------------------- mask-edge probes
# A probe owns one (batch row, head) slot.  Its queries get the vector u (2.0 in the first 8 dims: |u|^2 = 32), the planted key gets
# 4u, so its score 128 * scale beats every random key by far.  `out` queries must not see the key, `inn` queries must.
U_DIMS = 8


def probes(S: int, window: int, lengths_row: Optional[Sequence[int]], B: int) -> List[dict]:
    """Probes of one configuration: just outside and just inside the window edge (kv = q - window, q - window + 1), the diagonal
    (kv = q + 1, kv = q), each sample start (kv = seg[q] - 1, seg[q]) and the row offset (the last key of the previous batch row).
    Positions are rows of batch row 0 unless the probe says otherwise."""
    w = window if 0 < window < S else 0
    doc = None if lengths_row is None else doc_ids([lengths_row], S)[0]
    same = (lambda a, b: True) if doc is None else (lambda a, b: bool(doc[a] == doc[b]))
    out = []
    if w:
        for q_out in sorted({w, 127, 128, 191, 255, 256, 385, 511, 512, S - 1}):
            kp = q_out - w
            if kp >= 0 and same(kp, q_out) and same(kp, q_out - 1):
                out.append(dict(kind="window", kp=kp, out=[q_out], inn=[q_out - 1]))
    for kp in sorted({1, 64, 128, 129, S - 64}):
        if kp < S and same(kp - 1, kp):
            out.append(dict(kind="diag", kp=kp, out=[kp - 1], inn=[kp]))
    if lengths_row is not None:
        starts = np.cumsum([0] + list(lengths_row))[:-1].tolist()
        ends = np.cumsum(list(lengths_row)).tolist()
        picked = [i for i, s0 in enumerate(starts) if s0 in (63, 64, 65, 127, 128, 129, 256, S - 1)]
        picked += [i for i in range(1, len(starts)) if i not in picked][:max(0, 6 - len(picked))]
        for i in sorted(picked)[:8]:
            s0, s1 = starts[i], ends[i]
            if s0 == 0:
                continue
            out.append(dict(kind="seg-out", kp=s0 - 1, out=[s0], inn=[s0 - 1]))
            out.append(dict(kind="seg-in", kp=s0, out=[], inn=[min(s0 + 1, s1 - 1)]))
    if B >= 2:
        out.append(dict(kind="row", kp=S - 1, out=[], inn=[S - 1], next_row=[0, 1]))
    return out


def probe_slots(plist: List[dict], B: int) -> int:
    """Heads needed so that every probe gets a (row, head) slot of its own (the row probe takes one head in rows 0 and 1)."""
    n_rows = sum(1 for p in plist if p["kind"] != "row")
    return (n_rows + B - 1) // B + (1 if any(p["kind"] == "row" for p in plist) else 0)


def plant(qkv, d_o, B, S, H, plist: List[dict], value: Optional[float]):
    """Write the probes into MHA inputs (Hq = Hk = H) in place.  ``value``: the planted key's value (all dims; None keeps the random
    value).  ``d_o`` (or None): 4.0 on every ``out`` query, so a key that leaks into one of them in the backward swamps its dK / dV
    rows.  -> list of (probe, b, h)."""
    q, k, v = split(qkv, B, S, H, H)
    u = torch.zeros(D, dtype=qkv.dtype)
    u[:U_DIMS] = 2.0
    dO = None if d_o is None else d_o.view(B, S, H, D)
    slots = [(b, h) for h in range(H - (1 if any(p["kind"] == "row" for p in plist) else 0)) for b in range(B)]
    placed = []
    for p in plist:
        if p["kind"] == "row":
            b, h = 0, H - 1
            q[1, p["next_row"], h] = u
            if dO is not None:
                dO[1, p["next_row"], h] = 4.0
        else:
            b, h = slots.pop(0)
        q[b, p["out"] + p["inn"], h] = u
        k[b, p["kp"], h] = 4 * u
        if value is not None:
            v[b, p["kp"], h] = value
        if dO is not None and p["out"]:
            dO[b, p["out"], h] = 4.0
        placed.append((p, b, h))
    return placed


def _probe_q_rows(p, b):
    rows = [(b, s) for s in p["out"] + p["inn"]]
    if p["kind"] == "row":
        rows += [(1, s) for s in p["next_row"]]
    return rows


def probe_fwd_ratios(got, want, placed) -> Dict[str, float]:
    """Worst error / allowed error over the probe queries' O rows and LSE values."""
    ro = rl = 0.0
    for p, b, h in placed:
        for bb, s in _probe_q_rows(p, b):
            for name in ("o", "lse"):
                g = got[name][bb, s, h] if name == "o" else got[name][bb, h, s]
                w = want[name][bb, s, h] if name == "o" else want[name][bb, h, s]
                allowed = PROBE_ATOL + PROBE_RTOL * w.abs() if name == "o" else TOL["lse"] + PROBE_LSE_RTOL * w.abs()
                r = torch.nan_to_num((g.double() - w).abs() / allowed, nan=math.inf).max()
                if name == "o":
                    ro = max(ro, float(r))
                else:
                    rl = max(rl, float(r))
    return {"probe_o": ro, "probe_lse": rl}


def probe_bwd_ratios(got, want, placed) -> Dict[str, float]:
    """Worst error of the planted keys' dK / dV rows, relative to the largest oracle gradient, over the dense tolerance."""
    out = {}
    for name in ("dk", "dv"):
        scale = float(want[name].abs().max()) or 1.0
        r = 0.0
        for p, b, h in placed:
            r = max(r, float(torch.nan_to_num((got[name][b, p["kp"], h].double() - want[name][b, p["kp"], h]).abs(), nan=math.inf).max()))
        out["probe_" + name] = r / scale / TOL[name]
    return out


def check_probes_live(want, placed) -> None:
    """The oracle itself shows every probe is live: an ``inn`` query's O is the planted value, an ``out`` query's O is far from it."""
    for p, b, h in placed:
        for s in p["inn"]:
            assert float((want["o"][b, s, h] - PLANT_V).abs().max()) < 1.0, (p, "inside query does not see the planted key")
        outs = [(b, s) for s in p["out"]] + ([(1, s) for s in p["next_row"]] if p["kind"] == "row" else [])
        for bb, s in outs:
            assert float((want["o"][bb, s, h] - PLANT_V).abs().min()) > 32.0, (p, "outside query is dominated by the planted key")


# ---------------------------------------------------------------------------------------------- row layouts of packed rows
def row_lengths(kind: str, B: int, S: int, seed: int = 0) -> List[List[int]]:
    if kind == "random":
        from test_packing import random_seg
        return lengths_of_seg(random_seg(B, S, seed=seed), B, S)
    if kind == "len1":
        return [[1] * S for _ in range(B)]
    if kind == "edges":                      # samples starting at 63, 64, 65, 127, 128, 129: warpgroup and CTA edges
        return [[63, 1, 1, 62, 1, 1, S - 129] for _ in range(B)]
    if kind == "wg2":                        # a sample starting at 64, the forward's second warpgroup
        return [[64, S - 64] for _ in range(B)]
    if kind == "single":
        return [[S] for _ in range(B)]
    raise ValueError(kind)


SEG_KINDS = ("random", "len1", "edges", "wg2", "single")
GPTNEO_WINDOWS = (0, 1, 63, 64, 65, 127, 128, 129, 256, 300, 1024, 2048)


def mutants(S: int, window: int, segmented: bool, scale: float) -> List[str]:
    out = ["diag", "future"]
    if 0 < window < S:
        out += ["window+1"] + (["window-1"] if window > 1 else [])
    if segmented:
        out += ["seg-1", "seg+1"]
    if scale == 1.0:
        out.append("scale")
    return out


# ---------------------------------------------------------------------------------------------- CPU self-checks of the oracle
def _fp64_inputs(B, S, Hq, Hk, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, S, h, D, generator=g, dtype=torch.float64) * 0.7 for h in (Hq, Hk, Hk))
    d_o = torch.randn(B, S, Hq, D, generator=g, dtype=torch.float64) * 0.5
    return q, k, v, d_o


@pytest.mark.parametrize("B,S,Hq,Hk,window,scale,layout", [
    (1, 64, 1, 1, 0, 0.125, None), (2, 96, 4, 2, 17, 1.0, None), (1, 128, 2, 1, 1, 0.125, None), (2, 80, 2, 2, 0, 0.125, "random"),
    (2, 128, 4, 1, 40, 1.0, "random"), (1, 64, 2, 2, 0, 1.0, "len1")])
def test_oracle_matches_causal_attention_ref_and_masked_sdpa(B, S, Hq, Hk, window, scale, layout):
    from acco_b200.ops.attention import causal_attention_ref
    q, k, v, d_o = _fp64_inputs(B, S, Hq, Hk, S + Hq + window)
    lengths = [[S]] * B if layout is None else row_lengths(layout, B, S, seed=S)
    vis = visibility(doc_ids(lengths, S), window)
    want = oracle(q, k, v, d_o, scale, vis)
    seg = None if layout is None else seg_starts_of(lengths, S)
    ref = causal_attention_ref(q, k, v, scale=scale, window=window or None, seg=seg)   # fp32 math inside
    assert float((want["o"] - ref).abs().max()) < 1e-5
    # dense SDPA in fp64 with the oracle's mask, gradients by autograd
    qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
    o = torch.nn.functional.scaled_dot_product_attention(qg.transpose(1, 2), kg.transpose(1, 2), vg.transpose(1, 2),
                                                         attn_mask=vis[:, None], scale=scale, enable_gqa=Hq != Hk).transpose(1, 2)
    gq, gk, gv = torch.autograd.grad(o, (qg, kg, vg), d_o)
    for name, ref_t in (("o", o.detach()), ("dq", gq), ("dk", gk), ("dv", gv)):
        assert float((want[name] - ref_t).abs().max()) < 1e-10, name
    s = torch.einsum("bqhd,bkhd->bhqk", q, k.repeat_interleave(Hq // Hk, dim=2)) * scale
    lse = s.masked_fill(~vis[:, None], float("-inf")).logsumexp(dim=-1)
    assert float((want["lse"] - lse).abs().max()) < 1e-10


def test_oracle_visibility_is_the_documented_rule():
    """Brute force over every (q, kv) pair of a packed row, with the rule spelled out token by token."""
    S, window = 40, 7
    lengths = [[5, 1, 1, 13, 20]]
    doc = doc_ids(lengths, S)[0].tolist()
    vis = visibility(doc_ids(lengths, S), window)[0]
    for q in range(S):
        for kv in range(S):
            assert bool(vis[q, kv]) == (kv <= q and q - kv < window and doc[kv] == doc[q]), (q, kv)
    seg = seg_starts_of(lengths, S).tolist()
    assert all(seg[s] == min(i for i in range(S) if doc[i] == doc[s]) for s in range(S))


def test_oracle_head_subset_matches_the_full_run():
    q, k, v, d_o = _fp64_inputs(1, 128, 8, 2, 3)
    vis = visibility(doc_ids([[128]], 128), 0)
    full = oracle(q, k, v, d_o, 0.125, vis)
    part = oracle(q, k, v, d_o, 0.125, vis, groups=[1])
    hs = heads_of([1], 8, 2)
    for name in ("o", "dq"):
        assert torch.equal(part[name], full[name][:, :, hs])
    assert torch.equal(part["lse"], full["lse"][:, hs])
    for name in ("dk", "dv"):
        assert torch.equal(part[name], full[name][:, :, [1]])


def test_oracle_lse_and_empty_rows():
    """LSE normalises the probabilities; a query with no visible key (the diagonal mutant at q = 0) gets O = 0, LSE = -inf."""
    q, k, v, d_o = _fp64_inputs(1, 64, 1, 1, 5)
    vis = visibility(doc_ids([[64]], 64), 9, mutant="diag")
    r = oracle(q, k, v, d_o, 0.125, vis)
    assert float(r["lse"][0, 0, 0]) == -math.inf and float(r["o"][0, 0, 0].abs().max()) == 0.0
    s = (q[0, :, 0] @ k[0, :, 0].T * 0.125).masked_fill(~vis[0], float("-inf"))
    p = torch.exp(s[1:] - r["lse"][0, 0, 1:, None])
    assert torch.allclose(p.sum(-1), torch.ones(63, dtype=torch.float64), atol=1e-12)
    assert bool(torch.isfinite(r["dk"]).all())


# ---------------------------------------------------------------------------------------------- the margin table
def _cases():
    """(name, B, S, Hq, Hk, scale, window, layout) of every GPU case: the case itself where it is cheap on a CPU, else a twin with
    the same S, window, scale and row layout and fewer rows / heads (a different S for Llama-3.2-1B, whose rows are too long)."""
    cs = [("small", 1, 128, 1, 1, 0.125, 0, None), ("gqa4", 2, 256, 4, 1, 0.125, 0, None),
          ("llama125m", 1, 1024, 1, 1, 0.125, 0, None), ("llama3.2-1b", 1, 2048, 4, 1, 0.125, 0, None)]
    cs += [(f"gptneo-w{w}", 1, 1024, 1, 1, 1.0, w, None) for w in GPTNEO_WINDOWS]
    cs += [(f"seg-{kind}-w{w}-s{sc}", 1, 1024, 1, 1, sc, w, kind) for kind in SEG_KINDS for w in (0, 256) for sc in (1.0, 0.125)]
    return cs


def margin_row(name, B, S, Hq, Hk, scale, window, layout):
    """-> (emulator ratios, {mutant: (check, ratio)}): the emulator's error over each tolerance, and for every mutant the check that
    separates it from the oracle by the widest margin (ratios are error / tolerance)."""
    from acco_b200.ops.attention import attention_blockwise_bwd_ref, attention_blockwise_ref
    lengths = [[S]] * B if layout is None else row_lengths(layout, B, S, seed=S + window)
    doc = doc_ids(lengths, S)
    seg = None if layout is None else seg_starts_of(lengths, S)
    qkv, d_o = make_qkv(B, S, Hq, Hk, seed=S + window + Hq)
    q, k, v = split(qkv, B, S, Hq, Hk)
    dO = d_o.view(B, S, Hq, D)
    want = oracle(q, k, v, dO, scale, visibility(doc, window))
    eo, el = attention_blockwise_ref(q, k, v, scale, window or None, seg)
    edq, edk, edv = attention_blockwise_bwd_ref(q, k, v, eo, dO, el, scale, window or None, seg)
    emu = dense_ratios({"o": eo, "lse": el, "dq": edq, "dk": edk, "dv": edv}, want)

    # probes: MHA with enough heads for one slot per probe (a twin of the GPU probe case: same S, window, scale, layout)
    pl = probes(S, window, None if layout is None else lengths[0], 2)
    Hp = probe_slots(pl, 2)
    plen = [[S]] * 2 if layout is None else [lengths[0]] * 2
    pdoc = doc_ids(plen, S)
    fq, _ = make_qkv(2, S, Hp, Hp, seed=7)
    placed = plant(fq, None, 2, S, Hp, pl, PLANT_V)
    bq, bd = make_qkv(2, S, Hp, Hp, seed=8)
    plant(bq, bd, 2, S, Hp, pl, None)
    f_split, b_split = split(fq, 2, S, Hp, Hp), split(bq, 2, S, Hp, Hp)
    f_want = oracle(*f_split, None, scale, visibility(pdoc, window))
    check_probes_live(f_want, placed)
    b_want = oracle(*b_split, bd.view(2, S, Hp, D), scale, visibility(pdoc, window))

    def best(ratios):
        k_ = max(ratios, key=ratios.get)
        return k_, ratios[k_]

    caught = {}
    for mut in mutants(S, window, layout is not None, scale):
        if mut == "scale":
            got = oracle(q, k, v, dO, 0.125, visibility(doc, window))
            ratios = {"dense_" + n: r for n, r in dense_ratios(got, want).items()}
            ratios.update(probe_fwd_ratios(oracle(*f_split, None, 0.125, visibility(pdoc, window)), f_want, placed))
            caught[mut] = best(ratios)
            continue
        vis_m, pvis_m = visibility(doc, window, mut), visibility(pdoc, window, mut)
        if torch.equal(vis_m, visibility(doc, window)) and torch.equal(pvis_m, visibility(pdoc, window)):
            caught[mut] = ("equivalent", math.inf)     # the edge never binds in these rows (e.g. no sample is longer than the window)
            continue
        # the same mask error in the forward (and so in the LSE the backward consumes) ...
        got = oracle(q, k, v, None, scale, vis_m)
        ratios = {"dense_" + n: r for n, r in dense_ratios(got, want).items()}
        ratios.update(probe_fwd_ratios(oracle(*f_split, None, scale, pvis_m), f_want, placed))
        caught[mut] = best(ratios)
        # ... and in the backward alone, on top of an honest forward
        got = oracle(q, k, v, dO, scale, visibility(doc, window), vis_bwd=vis_m)
        ratios = {"dense_" + n: r for n, r in dense_ratios(got, want).items() if n.startswith("d")}
        ratios.update(probe_bwd_ratios(oracle(*b_split, bd.view(2, S, Hp, D), scale, visibility(pdoc, window), vis_bwd=pvis_m),
                                       b_want, placed))
        caught[mut + " (bwd)"] = best(ratios)
    return emu, caught


def margin_table(cases=None) -> List[tuple]:
    return [(c[0],) + margin_row(*c) for c in (cases or _cases())]


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c[0])
def test_margin_table(case):
    emu, caught = margin_row(*case)
    for name, r in emu.items():
        assert r < 0.5, (case[0], "emulator", name, r)
    for mut, (check, r) in caught.items():
        assert r > 3.0, (case[0], mut, check, r)


if __name__ == "__main__":                  # print the margin table: python tests/test_attention_oracle.py
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    for name, emu, caught in margin_table():
        print(f"{name:24s} emulator/tol " + " ".join(f"{k}={v:.2f}" for k, v in emu.items()))
        print(" " * 25 + "mutants " + "  ".join(f"{m}:{c}={r:.3g}" for m, (c, r) in caught.items()))
