"""The row-wise kernels (norms, RoPE, SwiGLU, GELU-new, cross-entropy) against the fp64 oracles and bounds of
``test_rowwise_oracle.py``, through the bindings, at every norm instantiation and at token counts where every grid-stride loop wraps;
plus the branches that live in the ``ops`` autograd glue.  fp64 references are computed on row chunks (peak well under 8 GB).
Run with ``pytest -m gpu -s`` to see the worst error / bound ratio and the share of outputs off the correctly rounded value."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops  # noqa: E402
from test_rowwise_oracle import (FTZ, bf16_rn, ce_inputs, ce_loss_bound, ce_ref, finite_bf16, gelu_ref,  # noqa: E402
                                 norm_bounds, norm_geometry, norm_grid, norm_inputs, norm_ref, out_bound, param_bound, ratio,
                                 rope_ref, rope_tables64, rows_per_owner, swiglu_ref)

DEV = "cuda"
EPS = 1e-5
CHUNK = 1 << 22                     # elements per fp64 reference chunk


@pytest.fixture(scope="module")
def C():
    return ops.load_ext(required=True)


@pytest.fixture(autouse=True)
def _free_between_cases():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def report(name, r, share=None):
    print(f"\n[rowwise] {name}: worst error/bound {r:.3f}" + ("" if share is None else f", not correctly rounded {100 * share:.3f} %"))


def off_rn(got, y64) -> int:
    """Elements that differ from the correctly rounded ``bf16_rn(y64)`` (values that round to inf compared as inf)."""
    return int((got.view(torch.int16) != bf16_rn(y64).view(torch.int16)).sum())


# ================================================================================================= norms
WIDTHS = [64, 256, 512, 768, 776, 1024, 1032, 2048, 2560, 4096, 4104, 8192, 12288, 16384]


def wrapping_T(H: int, sms: int) -> int:
    """A token count where the forward and the backward loops both run at least 2 rows per warp / CTA, with a ragged last sweep."""
    owners = []
    for bwd in (False, True):
        cap = norm_grid(1 << 30, H, sms, bwd) * (1 if H > 1024 else 8)
        owners.append(cap)
    big = max(owners)
    return 2 * big + big // 2 + 3


def run_norm(C, T, H, layer, residual, extra, seed, probes=True):
    """Forward, then the backward twice (fp32 dw | db, and accumulated into bf16 ``.grad`` views with guard cells); every output
    against the oracle on row chunks.  Returns the worst ratio per output, and the share of y and dh elements off the correctly
    rounded value."""
    a, w, b, r, dy, ex = norm_inputs(T, H, layer, residual, extra, seed, device=DEV)
    if probes and T > 8:
        a[5], a[6] = 1.5, 0.0                                      # constant row (zero variance) and a row of exact zeros
        if residual:
            r[5], r[6] = 0.25, 0.0
    y, h, mean, rstd = C.norm_fwd(a, r, w, b, EPS)
    hs = h if residual else a
    dh, dwdb = C.norm_bwd(dy, ex, hs, w, mean, rstd, None, None)
    guard = torch.randn(2, H + 16, device=DEV).to(torch.bfloat16)
    keep = guard.clone()
    wg, bg = guard[0, 8:8 + H], guard[1, 8:8 + H]
    g0w, g0b = wg.clone(), bg.clone()
    dh2, empty = C.norm_bwd(dy, ex, hs, w, mean, rstd, wg, bg if layer else None)
    assert empty.numel() == 0 and torch.equal(dh2, dh)
    for i in range(2 if layer else 1):                             # guard cells around the .grad views stay untouched
        assert torch.equal(guard[i, :8], keep[i, :8]) and torch.equal(guard[i, 8 + H:], keep[i, 8 + H:])
    if not layer:
        assert torch.equal(guard[1], keep[1])
    grid = norm_grid(T, H, C.num_sms(), True)
    worst, off = {}, 0
    dw64 = torch.zeros(H, dtype=torch.float64, device=DEV)
    db64, E_dw, E_db = torch.zeros_like(dw64), torch.zeros_like(dw64), torch.zeros_like(dw64)
    step = max(1, CHUNK // H)
    for r0 in range(0, T, step):
        sl = slice(r0, r0 + step)
        o = norm_ref(a[sl], w, b, None if r is None else r[sl], dy[sl], None if ex is None else ex[sl], EPS)
        bnd = norm_bounds(o, w, H, T, grid, layer, dy[sl], None if ex is None else ex[sl])
        got = {"y": y[sl], "rstd": rstd[sl], "dh": dh[sl]}
        if layer:
            got["mean"] = mean[sl]
        for k, v in got.items():
            worst[k] = max(worst.get(k, 0.0), ratio(v, o[k], bnd[k]))
        off += off_rn(y[sl], o["y"]) + off_rn(dh[sl], o["dh"])
        if residual:
            assert torch.equal(h[sl].double(), o["h"]), "h must be bf16_rn(a + r)"
        dw64 += o["dw"]
        db64 += o["db"]
        E_dw += bnd["E_dw"]
        E_db += bnd["E_db"]
        del o, bnd
    worst["dw"] = ratio(dwdb[:H], dw64, param_bound(dw64, E_dw))
    worst["dw_accum"] = ratio(wg, g0w.double() + dw64, param_bound(dw64, E_dw, g0w))
    if layer:
        worst["db"] = ratio(dwdb[H:], db64, param_bound(db64, E_db))
        worst["db_accum"] = ratio(bg, g0b.double() + db64, param_bound(db64, E_db, g0b))
    return worst, off / (2 * T * H)


@pytest.mark.parametrize("residual", [False, True], ids=["plain", "residual"])
@pytest.mark.parametrize("layer", [False, True], ids=["rms", "layer"])
@pytest.mark.parametrize("H", WIDTHS)
def test_norm_wrapped_against_fp64(C, H, layer, residual):
    """Every instantiation (warp VPT 1-4, CTA VPT 1 / 2 / 4, ragged widths) at a T where both loops wrap with a ragged last sweep."""
    sms = C.num_sms()
    T = wrapping_T(H, sms)
    for bwd in (False, True):
        g = norm_grid(T, H, sms, bwd)
        owners = g * (1 if H > 1024 else 8)
        assert rows_per_owner(T, H, g) >= 2 and T % owners != 0
    worst, share = run_norm(C, T, H, layer, residual, residual, seed=H + 2 * layer + residual)
    vpt, cta, _ = norm_geometry(H)
    report(f"norm H={H} {'layer' if layer else 'rms'} res={residual} T={T} ({'cta' if cta else 'warp'} vpt {vpt})", max(worst.values()), share)
    for k, v in worst.items():
        assert v <= 1.0, (k, v, worst)


@pytest.mark.parametrize("T", [1, 7])
@pytest.mark.parametrize("layer", [False, True], ids=["rms", "layer"])
@pytest.mark.parametrize("H", [256, 776, 4104])
def test_norm_few_rows(C, T, H, layer):
    worst, _ = run_norm(C, T, H, layer, True, True, seed=T * H, probes=False)
    for k, v in worst.items():
        assert v <= 1.0, (k, v, worst)


def _norm_glue(layer, residual, with_bias_grad=True):
    T, H = 600, 1032
    a, w, b, r, dy, ex = norm_inputs(T, H, layer, residual, residual, seed=7, device=DEV)
    a.requires_grad_(True)
    w.requires_grad_(True)
    g0w = torch.randn(H, device=DEV).to(torch.bfloat16)
    w.grad = g0w.clone()
    keep_w = w.grad
    g0b = None
    if layer:
        b.requires_grad_(True)
        if with_bias_grad:
            g0b = torch.randn(H, device=DEV).to(torch.bfloat16)
            b.grad = g0b.clone()
    if residual:
        r.requires_grad_(True)
        y, h = (ops.add_layernorm(a, r, w, b, EPS) if layer else ops.add_rmsnorm(a, r, w, EPS))
        torch.autograd.backward([y, h], [dy, ex])
    else:
        y = ops.layernorm(a, w, b, EPS) if layer else ops.rmsnorm(a, w, EPS)
        y.backward(dy)
    o = norm_ref(a.detach(), w.detach(), b.detach() if layer else None, r.detach() if residual else None, dy, ex, EPS)
    grid = norm_grid(T, H, torch.cuda.get_device_properties(0).multi_processor_count, True)
    bnd = norm_bounds(o, w.detach(), H, T, grid, layer, dy, ex)
    assert ratio(y.detach(), o["y"], bnd["y"]) <= 1.0
    assert ratio(a.grad, o["dh"], bnd["dh"]) <= 1.0
    if residual:
        assert torch.equal(a.grad, r.grad)
    return o, bnd, w, b, g0w, g0b, keep_w


@pytest.mark.parametrize("layer", [False, True], ids=["rms", "layer"])
def test_norm_glue_accumulates_into_existing_grad(layer):
    """``add_rmsnorm`` / ``add_layernorm`` add dw (and db) into the parameters' existing bf16 ``.grad`` in place."""
    o, bnd, w, b, g0w, g0b, keep_w = _norm_glue(layer, residual=True)
    assert w.grad is keep_w
    assert ratio(w.grad, g0w.double() + o["dw"], param_bound(o["dw"], bnd["E_dw"], g0w)) <= 1.0
    if layer:
        assert ratio(b.grad, g0b.double() + o["db"], param_bound(o["db"], bnd["E_db"], g0b)) <= 1.0


def test_layernorm_glue_with_only_weight_grad_accumulates_neither():
    """LayerNorm accumulates both parameters or neither: with ``w.grad`` present and ``b.grad`` absent, dw and db come back as
    fresh bf16 gradients (autograd then adds dw to ``w.grad``: one more bf16 rounding of dw)."""
    o, bnd, w, b, g0w, _, keep_w = _norm_glue(True, residual=False, with_bias_grad=False)
    E_extra = 2.0 ** -7 * o["dw"].abs()
    assert ratio(w.grad, g0w.double() + o["dw"], param_bound(o["dw"], bnd["E_dw"] + E_extra, g0w)) <= 1.0
    assert ratio(b.grad, o["db"], out_bound(o["db"], bnd["E_db"])) <= 1.0


# ================================================================================================= RoPE
ROPE = [  # (D, Hq, Hk, S, B): tokens B * S > SMs * 32 * 8 (the warp loop wraps)
    (64, 12, 12, 8192, 5), (128, 32, 8, 8192, 5), (16, 4, 2, 4096, 9), (32, 4, 4, 4096, 9), (256, 2, 1, 4096, 9)]


def rope_check(qkv_out, qkv_in, cos, sin, n_rot, S=None, inverse=False, pos=None):
    T, n, D = qkv_in.shape
    step = max(1, CHUNK // (n * D))
    worst, off, tot = 0.0, 0, 0
    for r0 in range(0, T, step):
        sl = slice(r0, r0 + step)
        p = None if pos is None else pos[sl]
        if p is None:
            p = torch.arange(r0, min(T, r0 + step), device=DEV) % S
        y64, E = rope_ref(qkv_in[sl], cos, sin, n_rot, inverse=inverse, pos=p)
        worst = max(worst, ratio(qkv_out[sl], y64, out_bound(y64, 2 * E)))
        off += off_rn(qkv_out[sl, :n_rot], y64[:, :n_rot])
        tot += y64[:, :n_rot].numel()
    return worst, off / tot


@pytest.mark.parametrize("D,Hq,Hk,S,B", ROPE)
def test_rope_wrapped_against_fp64(C, D, Hq, Hk, S, B):
    T = B * S
    assert T > C.num_sms() * 32 * 8
    n = Hq + 2 * Hk
    g = torch.Generator(device=DEV).manual_seed(D + Hq)
    x = torch.randn(T, n, D, generator=g, device=DEV).to(torch.bfloat16)
    cos, sin = (t.to(DEV) for t in rope_tables64(S, D, 500000.0))
    y = x.clone()
    C.rope_qkv_inplace(y, cos, sin, B, S, Hq + Hk, n, D, False)
    r, share = rope_check(y, x, cos, sin, Hq + Hk, S=S)
    assert torch.equal(y[:, Hq + Hk:], x[:, Hq + Hk:])                      # V heads untouched
    z = y.clone()
    C.rope_qkv_inplace(z, cos, sin, B, S, Hq + Hk, n, D, True)
    ri, _ = rope_check(z, y, cos, sin, Hq + Hk, S=S, inverse=True)
    report(f"rope D={D} {Hq}/{Hk} T={T}", max(r, ri), share)
    assert r <= 1.0 and ri <= 1.0


def test_rope_per_token_tables_for_packed_rows(C):
    """Packed rows: documents restart their positions; the tables are gathered per token (one row of length T, S = T)."""
    D, Hq, Hk = 64, 12, 12
    n = Hq + 2 * Hk
    doc = torch.tensor([0, 700, 701, 5000, 12000, 20000, 36000], device=DEV)
    T = 36100
    assert T > C.num_sms() * 32 * 8
    starts = torch.zeros(T, dtype=torch.long, device=DEV)
    starts[doc] = doc
    pos = torch.arange(T, device=DEV) - torch.cummax(starts, 0).values
    cos_s, sin_s = (t.to(DEV) for t in rope_tables64(8192 * 4, D, 500000.0))
    cos, sin = cos_s[pos].contiguous(), sin_s[pos].contiguous()
    g = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randn(T, n, D, generator=g, device=DEV).to(torch.bfloat16)
    y = x.clone()
    C.rope_qkv_inplace(y, cos, sin, 1, T, Hq + Hk, n, D, False)
    r, _ = rope_check(y, x, cos_s, sin_s, Hq + Hk, pos=pos)
    assert r <= 1.0


def quarter_turns(S, D, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    k = torch.randint(0, 4, (S, D // 2), generator=g, device=DEV)
    cos = torch.tensor([1.0, 0.0, -1.0, 0.0], device=DEV)[k].contiguous()
    sin = torch.tensor([0.0, 1.0, 0.0, -1.0], device=DEV)[k].contiguous()
    return cos, sin


@pytest.mark.parametrize("D,Hq,Hk", [(64, 12, 12), (128, 32, 8), (16, 4, 2), (256, 2, 1)])
def test_rope_quarter_turns_are_exact_signed_permutations(C, D, Hq, Hk):
    B, S = 3, 777
    n = Hq + 2 * Hk
    cos, sin = quarter_turns(S, D, D)
    g = torch.Generator(device=DEV).manual_seed(D)
    x = torch.randn(B * S, n, D, generator=g, device=DEV).to(torch.bfloat16)
    x[x == 0] = 1.0                                              # no zeros: every output is one input with a sign
    y = x.clone()
    C.rope_qkv_inplace(y, cos, sin, B, S, Hq + Hk, n, D, False)
    y64, _ = rope_ref(x, cos, sin, Hq + Hk, S)
    assert torch.equal(y.double(), y64)
    assert torch.equal(y[:, Hq + Hk:].view(torch.int16), x[:, Hq + Hk:].view(torch.int16))
    z = y.clone()
    C.rope_qkv_inplace(z, cos, sin, B, S, Hq + Hk, n, D, True)
    assert torch.equal(z.view(torch.int16), x.view(torch.int16))


@pytest.mark.parametrize("D,Hq,Hk", [(64, 12, 12), (128, 32, 8)])
def test_rope_pack_bwd_strided_views(C, D, Hq, Hk):
    """dq from a transposed [B, H, S, D] buffer, dk / dv slices of one wider buffer: identity tables give a bitwise copy of the
    gather, random tables the inverse rotation of q and k within the bound."""
    B, S = 2, 9000
    g = torch.Generator(device=DEV).manual_seed(D)
    dq = torch.randn(B, Hq, S, D, generator=g, device=DEV).to(torch.bfloat16).transpose(1, 2)
    kv = torch.randn(B, S, 2 * Hk + 1, D, generator=g, device=DEV).to(torch.bfloat16)
    dk, dv = kv[:, :, 1:Hk + 1], kv[:, :, Hk + 1:]
    want = torch.cat([dq, dk, dv], 2).reshape(B * S, Hq + 2 * Hk, D)
    one, zero = torch.ones(S, D // 2, device=DEV), torch.zeros(S, D // 2, device=DEV)
    out = C.rope_pack_bwd(dq, dk, dv, one, zero).view(B * S, Hq + 2 * Hk, D)
    assert torch.equal(out.view(torch.int16), want.view(torch.int16))
    cos, sin = (t.to(DEV) for t in rope_tables64(S, D, 500000.0))
    out = C.rope_pack_bwd(dq, dk, dv, cos, sin).view(B * S, Hq + 2 * Hk, D)
    r, _ = rope_check(out, want, cos, sin, Hq + Hk, S=S, inverse=True)
    assert r <= 1.0


# ================================================================================================= SwiGLU / GELU
def as_rows(v: torch.Tensor, I: int, fill: float = 1.0) -> torch.Tensor:
    n = -(-v.numel() // I) * I
    out = torch.full((n,), fill, dtype=v.dtype, device=v.device)
    out[:v.numel()] = v
    return out.view(-1, I)


def test_swiglu_every_finite_bf16_gate(C):
    xs = finite_bf16().to(DEV)
    I = 1024
    worst, off, tot = {}, 0, 0
    for up in (1.0, -0.75, 3.5):
        g = as_rows(xs, I)
        u = torch.full_like(g, up)
        out = C.swiglu_fwd(torch.cat([g, u], 1).contiguous())
        for dval in (1.0, -2.5):
            d = torch.full_like(g, dval)
            dgu = C.swiglu_bwd(d, torch.cat([g, u], 1).contiguous())
            o = swiglu_ref(g, u, d)
            for k, got in (("out", out), ("dgate", dgu[:, :I]), ("dup", dgu[:, I:])):
                worst[k] = max(worst.get(k, 0.0), ratio(got, o[k], o["b_" + k]))
                off += off_rn(got, o[k])
                tot += got.numel()
    report("swiglu exhaustive", max(worst.values()), off / tot)
    for k, v in worst.items():
        assert v <= 1.0, (k, v)


def test_gelu_every_finite_bf16_input(C):
    x = as_rows(finite_bf16().to(DEV), 1024)
    worst, off, tot = {}, 0, 0
    y = C.gelu_fwd(x)
    o = gelu_ref(x)
    worst["y"] = ratio(y, o["y"], o["b_y"])
    off, tot = off_rn(y, o["y"]), y.numel()
    for dval in (1.0, -0.375):
        d = torch.full_like(x, dval)
        dx = C.gelu_bwd(d, x)
        o = gelu_ref(x, d)
        worst[f"dx{dval}"] = ratio(dx, o["dx"], o["b_dx"])
        off += off_rn(dx, o["dx"])
        tot += dx.numel()
    report("gelu exhaustive", max(worst.values()), off / tot)
    for k, v in worst.items():
        assert v <= 1.0, (k, v)


@pytest.mark.parametrize("T,I", [(4096, 8192), (4096, 14336)], ids=["llama3.2-1b", "llama3-8b"])
def test_swiglu_training_shapes(C, T, I):
    g = torch.Generator(device=DEV).manual_seed(I)
    gu = (torch.randn(T, 2 * I, generator=g, device=DEV) * 2).to(torch.bfloat16)
    d = torch.randn(T, I, generator=g, device=DEV).to(torch.bfloat16)
    assert T * I // 8 > 2 * C.num_sms() * 8 * 4 * 256                      # the grid-stride loop wraps
    out = C.swiglu_fwd(gu)
    dgu = C.swiglu_bwd(d, gu)
    worst = 0.0
    step = max(1, CHUNK // I)
    for r0 in range(0, T, step):
        sl = slice(r0, r0 + step)
        o = swiglu_ref(gu[sl, :I], gu[sl, I:], d[sl])
        worst = max(worst, ratio(out[sl], o["out"], o["b_out"]), ratio(dgu[sl, :I], o["dgate"], o["b_dgate"]),
                    ratio(dgu[sl, I:], o["dup"], o["b_dup"]))
    report(f"swiglu T={T} I={I}", worst)
    assert worst <= 1.0


@pytest.mark.parametrize("I", [3072, 10240], ids=["gptneo", "gptneoLarge"])
def test_gelu_training_shapes(C, I):
    T = 8192
    g = torch.Generator(device=DEV).manual_seed(I)
    x = (torch.randn(T, I, generator=g, device=DEV) * 2).to(torch.bfloat16)
    d = torch.randn(T, I, generator=g, device=DEV).to(torch.bfloat16)
    assert T * I // 8 > 2 * C.num_sms() * 16 * 256
    y = C.gelu_fwd(x)
    dx = C.gelu_bwd(d, x)
    worst = 0.0
    step = max(1, CHUNK // I)
    for r0 in range(0, T, step):
        sl = slice(r0, r0 + step)
        o = gelu_ref(x[sl], d[sl])
        worst = max(worst, ratio(y[sl], o["y"], o["b_y"]), ratio(dx[sl], o["dx"], o["b_dx"]))
    report(f"gelu T={T} I={I}", worst)
    assert worst <= 1.0


# ================================================================================================= cross-entropy
def run_ce(C, lg, lab, V, dloss=1.0, rows=128):
    """Kernel forward + backward (on a copy: the backward overwrites the logits) against the oracle on row chunks."""
    T, Vp = lg.shape
    loss, inv_n, lse = C.ce_fwd(lg, lab, V, -100)
    n = int((lab != -100).sum())
    scale = torch.tensor([dloss], device=DEV) * inv_n
    grad = lg.clone()
    C.ce_bwd_inplace(grad, lab, lse, scale, V, -100)
    inv64 = 1.0 / n if n else 0.0
    worst = {"lse": 0.0, "grad": 0.0}
    row_sum = E_sum = abs_sum = 0.0
    off = tot = 0
    for r0 in range(0, T, rows):
        sl = slice(r0, r0 + rows)
        o = ce_ref(lg[sl], lab[sl], V, scale=float(scale))           # the scale is an input of the backward kernel
        worst["lse"] = max(worst["lse"], ratio(lse[sl], o["lse"], o["b_lse"]))
        worst["grad"] = max(worst["grad"], ratio(grad[sl], o["grad"], o["b_grad"]))
        if Vp > V:
            assert bool((grad[sl, V:] == 0).all()), "padding columns must get exactly zero gradient"
        off += off_rn(grad[sl, :V], o["grad"][:, :V])
        tot += o["grad"][:, :V].numel()
        row_sum += float(o["row"].sum())
        abs_sum += float(o["row"].abs().sum())
        E_sum += float(o["E_row"].sum())
        del o
    loss64 = row_sum * inv64
    worst["loss"] = abs(float(loss) - loss64) / ce_loss_bound(E_sum, abs_sum, T, loss64, inv64)
    worst["inv_n"] = abs(float(inv_n) - inv64) / max(2 * 2.0 ** -22 * inv64, FTZ)
    assert torch.isfinite(lse).all() and math.isfinite(float(loss))
    return worst, off / max(tot, 1)


CE_SHAPES = [(50257, 50304), (128256, 128256), (131, 136), (1000, 1000), (8, 8), (1, 8)]


@pytest.mark.parametrize("V,Vp,pad", [(V, Vp, pad) for V, Vp in CE_SHAPES for pad in ((None, math.nan, math.inf) if Vp > V else (None,))])
def test_cross_entropy_against_fp64(C, V, Vp, pad):
    """Padding columns left random, or filled with NaN / +inf: excluded from the softmax, gradient exactly 0."""
    lg, lab = ce_inputs(64, V, Vp, seed=V, pad_fill=pad, device=DEV)
    worst, share = run_ce(C, lg, lab, V, dloss=2.5)
    report(f"ce V={V}/{Vp} pad={pad}", max(worst.values()), share)
    for k, v in worst.items():
        assert v <= 1.0, (k, v, worst)


def test_cross_entropy_llama3_bench_microbatch(C):
    """T = 4096 rows of the Llama-3 vocabulary (the Llama-3.2-1B micro-batch), 1 GiB of logits; fp64 reference on 64-row chunks."""
    lg, lab = ce_inputs(4096, 128256, 128256, seed=1, device=DEV)
    worst, share = run_ce(C, lg, lab, 128256, rows=64)
    report("ce T=4096 V=128256", max(worst.values()), share)
    for k, v in worst.items():
        assert v <= 1.0, (k, v, worst)


def test_cross_entropy_all_ignored_batch_is_pinned_to_zero(C):
    """Every row ignored: the kernels return loss 0, inv_n 0, lse 0 and an all-zero gradient.  HF's mean over zero rows is NaN;
    the trainer sums such losses over micro-batches and rounds, so a NaN would poison the whole step.  Pinned on purpose."""
    lg, lab = ce_inputs(40, 1000, 1008, seed=2, pad_fill=math.nan, device=DEV)
    lab[:] = -100
    loss, inv_n, lse = C.ce_fwd(lg, lab, 1000, -100)
    assert float(loss) == 0.0 and float(inv_n) == 0.0 and bool((lse == 0).all())
    grad = lg.clone()
    C.ce_bwd_inplace(grad, lab, lse, torch.ones(1, device=DEV) * inv_n, 1000, -100)
    assert bool((grad == 0).all())


def test_cross_entropy_glue_scale_is_dloss_times_inv_n():
    """``softmax_cross_entropy`` backward scales by ``dloss * inv_n`` (the mean's 1 / n and the upstream gradient)."""
    V, Vp = 50257, 50304
    lg, lab = ce_inputs(300, V, Vp, seed=5, device=DEV)
    keep = lg.clone()
    x = lg.clone().requires_grad_(True)
    loss = ops.softmax_cross_entropy(x * 1.0, lab, V, -100)
    (loss * 3.0).backward()
    n = int((lab != -100).sum())
    for r0 in range(0, 300, 100):
        o = ce_ref(keep[r0:r0 + 100], lab[r0:r0 + 100], V, scale=3.0 / n)
        assert ratio(x.grad[r0:r0 + 100], o["grad"], o["b_grad"]) <= 1.0
