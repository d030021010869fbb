"""Sample packing for fine-tuning (``packing: True``), CPU side:

* ``pack_sft`` (first-fit-decreasing rows) and ``PackedCollator`` (labels / positions contract, equivalence with ``PadCollator``);
* the segment-aware attention specification (document masking): blockwise forward / backward references against a dense fp32
  masked reference, and the loop ranges of the segmented kernels against brute-force visibility;
* the models: a packed row gives every sample the logits, losses and gradients it gets alone;
* the autograd glue of the segmented kernels (fake extension) and the trainer wiring."""
import math

import numpy as np
import pytest
import torch

from acco_b200.data import PackedCollator, PadCollator, TokenDataset, pack_sft, synthetic_documents, synthetic_sft_dataset
from acco_b200.ops.attention import (attention_blockwise_bwd_ref, attention_blockwise_ref, bwd_query_blocks_seg, causal_attention_ref,
                                     fwd_key_blocks_seg, segment_starts)

from helpers import LOG, base_args, tiny_model

PAD = 95


# ---------------------------------------------------------------------------------------------- pack_sft
def test_pack_sft_places_every_sample_whole_and_in_order():
    docs = [d.tolist() for d in synthetic_documents(300, 40, 96, seed=4, min_len=1, max_len=200)] + [list(range(90))]
    out = pack_sft(docs, 64)
    assert out == pack_sft(docs, 64)                                              # deterministic
    seen = []
    for row, lens in zip(out["input_ids"], out["doc_lens"]):
        assert len(row) <= 64 and sum(lens) == len(row) and all(n > 0 for n in lens)
        a = 0
        for n in lens:
            seen.append(tuple(row[a:a + n]))
            a += n
    want = sorted(tuple(d[:64]) for d in docs)                                    # truncated like truncate_docs
    assert sorted(seen) == want


def test_pack_sft_first_fit_decreasing():
    out = pack_sft([[1] * 3, [2] * 6, [3] * 5, [4] * 2, [5] * 4], 8)
    assert out["doc_lens"] == [[6, 2], [5, 3], [4]]
    assert out["input_ids"][0] == [2] * 6 + [4] * 2


def test_pack_sft_efficiency_on_alpaca_shaped_data():
    ds = synthetic_sft_dataset(5000, 180, 50257, 512)
    packed = ds.map(lambda b: pack_sft(b["input_ids"], 512), batched=True, remove_columns=ds.column_names)   # per 1000 samples
    real = sum(len(r) for r in ds["input_ids"])
    assert sum(len(r) for r in packed["input_ids"]) == real
    assert real / (len(packed) * 512) >= 0.95


# ---------------------------------------------------------------------------------------------- PackedCollator
def test_packed_collator_contract():
    rows = [{"input_ids": [5, 6, 7, 8, 9, PAD, 11], "doc_lens": [3, 1, 3]}, {"input_ids": [20, 21], "doc_lens": [2]}]
    out = PackedCollator(PAD, 10)(rows)
    assert all(v.shape == (2, 10) and v.dtype == torch.int64 for v in out.values())
    assert out["position_ids"].tolist() == [[0, 1, 2, 0, 0, 1, 2, 0, 1, 2], [0, 1, 0, 1, 2, 3, 4, 5, 6, 7]]
    assert out["input_ids"].tolist() == [[5, 6, 7, 8, 9, PAD, 11, PAD, PAD, PAD], [20, 21] + [PAD] * 8]
    assert out["labels"].tolist() == [[-100, 6, 7, -100, -100, -100, 11, -100, -100, -100], [-100, 21] + [-100] * 8]
    keep = PackedCollator(PAD, 10, mask_all_pad_tokens=False)(rows)
    assert keep["labels"][0, 5] == PAD


@pytest.mark.parametrize("row", [{"input_ids": [1, 2, 3], "doc_lens": [2, 2]}, {"input_ids": [1, 2, 3], "doc_lens": [3, 0]},
                                 {"input_ids": [1, 2, 3], "doc_lens": [4, -1]}, {"input_ids": list(range(12)), "doc_lens": [12]}])
def test_packed_collator_rejects_malformed_rows(row):
    with pytest.raises(ValueError):
        PackedCollator(PAD, 10)([row])


def _pairs_padded(batch):
    """(context, target) pairs a padded batch trains: position t of row b predicts labels[b, t+1] from tokens [0, t]."""
    ids, lab = batch["input_ids"], batch["labels"]
    return sorted((tuple(ids[b, :t + 1].tolist()), int(lab[b, t + 1])) for b in range(ids.shape[0]) for t in range(ids.shape[1] - 1)
                  if lab[b, t + 1] != -100)


def _pairs_packed(batch):
    """Same for packed rows: the context of position t is the tokens of its own sample up to t (document masking)."""
    ids, lab, pos = batch["input_ids"], batch["labels"], batch["position_ids"]
    out = []
    for b in range(ids.shape[0]):
        for t in range(ids.shape[1] - 1):
            if lab[b, t + 1] != -100:
                a = t - int(pos[b, t])
                out.append((tuple(ids[b, a:t + 1].tolist()), int(lab[b, t + 1])))
    return sorted(out)


@pytest.mark.parametrize("mask_all", [True, False])
def test_packed_collator_trains_the_pairs_of_the_pad_collator(mask_all):
    rng = np.random.default_rng(0)
    docs = [rng.integers(0, 96, size=int(n)).tolist() for n in rng.integers(1, 30, size=60)]
    for d in docs[::7]:
        d[len(d) // 2] = PAD                                                      # pad ids inside samples follow the PadCollator rule
    packed = pack_sft(docs, 32)
    rows = [{"input_ids": r, "doc_lens": l} for r, l in zip(packed["input_ids"], packed["doc_lens"])]
    got = _pairs_packed(PackedCollator(PAD, 32, mask_all_pad_tokens=mask_all)(rows))
    want = _pairs_padded(PadCollator(PAD, mask_all_pad_tokens=mask_all, max_length=32)([{"input_ids": d} for d in docs]))
    assert got == want


# ---------------------------------------------------------------------------------------------- attention specification
LENS = (1, 63, 64, 65, 127, 128, 129)


def random_seg(B, S, seed, whole_row=False):
    """int32 [B*S] segment starts of rows cut into samples drawn from LENS (the last one takes what is left)."""
    rng = np.random.default_rng(seed)
    seg = np.zeros((B, S), dtype=np.int32)
    for b in range(B):
        a = 0
        while a < S:
            n = S if whole_row else int(rng.choice(LENS))
            n = min(n, S - a)
            seg[b, a:a + n] = a
            a += n
    return torch.from_numpy(seg.reshape(-1))


def test_segment_starts_encoding():
    pos = torch.tensor([[0, 1, 2, 0, 1, 0], [0, 1, 2, 3, 4, 5]])
    assert segment_starts(pos).tolist() == [0, 0, 0, 3, 3, 5, 0, 0, 0, 0, 0, 0]
    assert segment_starts(pos).dtype == torch.int32


@pytest.mark.parametrize("window", [None, 256])
@pytest.mark.parametrize("Hq,Hk", [(4, 4), (32, 8)])
@pytest.mark.parametrize("whole_row", [False, True])
def test_segmented_blockwise_references_match_dense_masked_attention(window, Hq, Hk, whole_row):
    B, S = (1, 512) if Hq == 32 else (2, 512)
    seg = random_seg(B, S, seed=Hq + (window or 0), whole_row=whole_row)
    torch.manual_seed(0)
    q, k, v = (torch.randn(B, S, h, 64, requires_grad=True) for h in (Hq, Hk, Hk))
    ref = causal_attention_ref(q, k, v, window=window, seg=seg)
    d_o = torch.randn_like(ref)
    gq, gk, gv = torch.autograd.grad(ref, (q, k, v), d_o)
    with torch.no_grad():
        o, lse = attention_blockwise_ref(q, k, v, None, window, seg=seg)
        dq, dk, dv = attention_blockwise_bwd_ref(q, k, v, o, d_o, lse, None, window, seg=seg)
    assert (o - ref).abs().max() < 1e-2
    att = (q.detach().transpose(1, 2) @ k.detach().repeat_interleave(Hq // Hk, 2).transpose(1, 2).transpose(-1, -2)) / 8.0
    i = torch.arange(S)
    vis = (i[None, :] <= i[:, None]) & (i[None, :] > i[:, None] - (window or S))
    vis = vis[None] & (i[None, None, :] >= seg.view(B, S)[:, :, None].long())
    assert torch.allclose(lse, att.masked_fill(~vis[:, None], float("-inf")).logsumexp(-1), atol=1e-4)
    for got, want in ((dq, gq), (dk, gk), (dv, gv)):
        assert (got - want).abs().max() / want.abs().max() < 1e-2
    if whole_row:                                                                 # one sample per row: the unsegmented schedule
        o0, lse0 = attention_blockwise_ref(q.detach(), k.detach(), v.detach(), None, window)
        assert torch.equal(o0, o) and torch.equal(lse0, lse)


@pytest.mark.parametrize("S", [512, 1024])
@pytest.mark.parametrize("window", [None, 256, 300])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_segmented_block_ranges_cover_exactly_the_visible_pairs(S, window, seed):
    """The kernels' loop bounds: forward CTA = 128 queries over 64-key blocks, backward CTA = 64 keys over 64-query blocks (and the
    128 x 128 tiles of the blockwise references)."""
    win = min(window or S, S)
    seg = random_seg(1, S, seed).long()
    i = torch.arange(S)
    vis = (i[None, :] <= i[:, None]) & (i[None, :] + win > i[:, None]) & (i[None, :] >= seg[:, None])   # [q, kv]
    for bq, bk in ((128, 128), (128, 64), (64, 64)):
        blocks = vis.view(S // bq, bq, S // bk, bk).any(dim=3).any(dim=1)
        want = {(m, n) for m in range(S // bq) for n in range(S // bk) if blocks[m, n]}
        if bq >= bk:
            assert {(m, j) for m in range(S // bq) for j in fwd_key_blocks_seg(m, win, seg, bq, bk)} == want
        if bq == bk:
            assert {(m, n) for n in range(S // bk) for m in bwd_query_blocks_seg(n, S, win, seg, bq, bk)} == want


# ---------------------------------------------------------------------------------------------- models
def _tiny_gptneo():
    from acco_b200.models import GPTConfig, GPTForCausalLM
    torch.manual_seed(3)
    return GPTForCausalLM(GPTConfig(vocab_size=96, hidden_size=32, num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=64,
                                    attention_layers="alternating", window_size=5, pad_vocab_multiple=8))


@pytest.mark.parametrize("family", ["llama", "gptneo"])
def test_packed_row_equals_each_sample_alone(family):
    model = tiny_model() if family == "llama" else _tiny_gptneo()       # tiny Llama: GQA 4 / 2; GPT-Neo: local layer, window 5
    rng = np.random.default_rng(1)
    docs = [rng.integers(0, 95, size=n).tolist() for n in (9, 1, 13, 6)]
    L = 32
    batch = PackedCollator(PAD, L)([{"input_ids": sum(docs, []), "doc_lens": [len(d) for d in docs]}])

    def per_token_loss(logits, labels):
        tgt = torch.full_like(labels, -100)
        tgt[:, :-1] = labels[:, 1:]
        return torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]).float(), tgt.reshape(-1), reduction="none",
                                                 ignore_index=-100)

    model.zero_grad(set_to_none=True)
    logits = model(batch["input_ids"], position_ids=batch["position_ids"]).logits
    lp = per_token_loss(logits, batch["labels"])
    lp.sum().backward()
    g_packed = [p.grad.clone() for p in model.parameters()]
    model.zero_grad(set_to_none=True)
    a, total = 0, 0.0
    for d in docs:
        ids = torch.tensor([d])
        lab = PadCollator(PAD)([{"input_ids": d}])["labels"]
        la = per_token_loss(model(ids).logits, lab)
        assert torch.allclose(lp[a:a + len(d)], la, atol=1e-5)
        total = total + la.sum()
        a += len(d)
    total.backward()
    for gp, p in zip(g_packed, model.parameters()):
        assert torch.allclose(gp, p.grad, atol=1e-5), float((gp - p.grad).abs().max())


def test_position_ids_of_one_sample_per_row_change_nothing():
    model = tiny_model()
    ids = torch.randint(0, 95, (2, 16))
    pos = torch.arange(16).expand(2, 16)
    assert torch.allclose(model(ids).logits, model(ids, position_ids=pos).logits, atol=1e-6)


# ---------------------------------------------------------------------------------------------- autograd glue (fake extension)
class _FakeSegExt:
    """acco_b200._C stand-in on the CPU: attention entry points backed by the segment-aware blockwise specification, RoPE kernels by
    their reference math (table row t % S, like the kernels).  Records the ``seg`` each entry point received."""
    seen = []

    @staticmethod
    def attn_supported(B, S, Hq, Hk, D, scale):
        return D == 64 and S % 128 == 0 and Hq % Hk == 0 and scale > 0

    @staticmethod
    def attn_fwd(qkv, B, S, Hq, Hk, D, sc, window, seg=None):
        _FakeSegExt.seen.append(("fwd", seg))
        x = qkv.view(B, S, Hq + 2 * Hk, D)
        o, lse = attention_blockwise_ref(x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:], sc, window, seg=seg)
        return o.reshape(B * S, Hq * D), lse

    @staticmethod
    def attn_bwd(qkv, o, d_o, lse, B, S, Hq, Hk, D, sc, window, seg=None):
        _FakeSegExt.seen.append(("bwd", seg))
        x = qkv.view(B, S, Hq + 2 * Hk, D)
        dq, dk, dv = attention_blockwise_bwd_ref(x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:], o.view(B, S, Hq, D),
                                                 d_o.view(B, S, Hq, D), lse, sc, window, seg=seg)
        return dq.reshape(B * S, Hq * D), dk.reshape(B * S, Hk * D), dv.reshape(B * S, Hk * D)

    @staticmethod
    def rope_qkv_inplace(qkv, cos, sin, B, S, n_rot, n_total, D, inverse):
        from acco_b200.ops.rope import apply_rope_ref
        x = qkv.view(B, S, n_total, D)
        x[:, :, :n_rot] = apply_rope_ref(x[:, :, :n_rot], cos, -sin if inverse else sin)

    @staticmethod
    def rope_pack_bwd(dq, dk, dv, cos, sin):
        from acco_b200.ops.rope import apply_rope_ref
        B, S = dq.shape[:2]
        return torch.cat([apply_rope_ref(dq, cos, -sin), apply_rope_ref(dk, cos, -sin), dv], dim=2).reshape(B * S, -1)


@pytest.mark.parametrize("rope,window,scale", [(True, None, None), (False, 160, 1.0)])
def test_segmented_attention_autograd_glue(monkeypatch, rope, window, scale):
    from acco_b200 import ops
    from acco_b200.ops import attention as A
    from acco_b200.ops.rope import rope_qkv_ref, rope_tables
    monkeypatch.delenv("ACCO_ATTN", raising=False)                                # packed rows take the own kernels regardless
    monkeypatch.setattr(ops, "load_ext", lambda required=False: _FakeSegExt)
    _FakeSegExt.seen = []
    B, S, Hq, Hk, D = 2, 256, 4, 2, 64
    seg = random_seg(B, S, seed=5)
    pos = (torch.arange(S).repeat(B) - seg.long())
    torch.manual_seed(1)
    qkv = (torch.randn(B * S, (Hq + 2 * Hk) * D) * 0.5).requires_grad_()
    if rope:
        cos, sin = rope_tables(S, D, 10000.0, "cpu")
        cos, sin = cos[pos], sin[pos]                                             # per-token tables [B*S, D/2]
    else:
        cos, sin = A._identity_tables(S, D, "cpu")
    d_o = torch.randn(B * S, Hq * D)
    out = A._RopeAttentionFn.apply(qkv.clone(), cos, sin, B, S, Hq, Hk, D, rope, scale, window, seg)
    out.backward(d_o)
    assert [k for k, _ in _FakeSegExt.seen] == ["fwd", "bwd"] and all(s is seg for _, s in _FakeSegExt.seen)
    got = qkv.grad.clone()
    q2 = qkv.detach().clone().requires_grad_()
    y = rope_qkv_ref(q2, cos, sin, 1, B * S, Hq, Hk, D) if rope else q2
    y = y.view(B, S, Hq + 2 * Hk, D)
    ref = causal_attention_ref(y[:, :, :Hq], y[:, :, Hq:Hq + Hk], y[:, :, Hq + Hk:], scale=scale, window=window, seg=seg).reshape(B * S, Hq * D)
    ref.backward(d_o)
    assert (out - ref).abs().max() < 2e-2
    assert (got - q2.grad).abs().max() / q2.grad.abs().max() < 2e-2


# ---------------------------------------------------------------------------------------------- trainer
def _sft_trainer(**kw):
    from acco_b200 import DecoupledTrainer
    from acco_b200.data import ByteTokenizer
    from acco_b200.launch import DistEnv
    tok = ByteTokenizer()
    tok.pad_token_id = tok.eos_token_id = PAD
    model = kw.pop("model", None) or tiny_model()
    ds = synthetic_sft_dataset(400, 8, 96, 32, seed=1)
    ev = synthetic_sft_dataset(40, 8, 96, 32, seed=2)
    a = dict(const_len_batch=False, packing=True, max_length=32)
    a.update(kw)
    args = base_args(**a)
    return DecoupledTrainer(model=model, tokenizer=tok, train_dataset=ds, eval_dataset=ev, args=args, log=LOG, env=DistEnv(id_run="pack"))


def test_trainer_packing_trains_and_evaluates_padded(workdir):
    t = _sft_trainer(nb_steps_tot=80, learning_rate=5e-3, batch_size=2)
    assert isinstance(t.train_dataloader.collate_fn, PackedCollator) and isinstance(t.eval_dataloader.collate_fn, PadCollator)
    assert t.train_dataset.column_names == ["input_ids", "doc_lens"] and len(t.train_dataset) < 400
    losses = []
    while not t.finished():
        t.step()
        losses.append(float(t.loss_host))
    t._finish("")
    assert all(math.isfinite(x) for x in losses)
    assert sum(losses[-10:]) / 10 < sum(losses[:10]) / 10 - 0.2
    assert torch.isfinite(t.eval_loop())


@pytest.mark.parametrize("bad", [{"const_len_batch": True}, {"group_by_length": True}, {"model": "hf"}])
def test_trainer_packing_rejects_invalid_combinations(workdir, bad):
    if bad.get("model") == "hf":
        class HFLike(torch.nn.Module):
            def __init__(self):
                super().__init__()
                self.w = torch.nn.Parameter(torch.zeros(4))

            def forward(self, input_ids=None, labels=None, **kw):
                return ((self.w ** 2).sum(),)
        bad = {"model": HFLike()}
    with pytest.raises(ValueError, match="packing"):
        _sft_trainer(**bad)
