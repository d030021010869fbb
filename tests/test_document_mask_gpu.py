"""Document masking of pre-training rows on the H100 (``document_mask: True``):

* the segmented flash-attention kernels, forward and backward, at pre-training shapes (Llama-125M heads at S = 1024, the
  Llama-3.2-1B heads 32 / 8 at S = 1024 and 2048, GPT-Neo's 256-token window at scale 1.0) on rows cut by ``DocumentCollator``:
  one from the openwebtext-shaped synthetic corpus, one with boundaries at 127 / 128 / 129 and on other block edges.  They are
  checked against the fp32 reference (every head) and the blockwise references (the kernels' own loop bounds and rounding points;
  the first and the last KV group), with the tolerances of ``test_packing_gpu.py``;
* the per-document oracle on bf16 weights, on the kernels: a masked row's loss and gradients against every document run alone;
* the one-GPU ACCO trainer with CUDA graphs, alone and with ``fp8`` / ``max_grad_norm``, against the fp32 CPU trainer, with one
  graph captured per buffer pair and replayed across batches of different segmentations."""
import logging
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops
from acco_b200.data import DocumentCollator, synthetic_pretrain_dataset
from acco_b200.ops.attention import attention_blockwise_bwd_ref, attention_blockwise_ref, causal_attention_ref, segment_starts

from test_document_mask import doc_rows

DEV = "cuda"
D = 64
O_TOL, G_TOL = 2e-2, 3e-2          # test_packing_gpu.py: O max abs error; dQ / dK / dV max error relative to the largest gradient
# segment starts on the 64- and 128-token block edges and one either side of them (consecutive starts: one-token documents)
EDGE_STARTS = (1, 63, 64, 65, 127, 128, 129, 191, 192, 255, 256, 257, 383, 384, 511, 512, 513, 639, 640, 767, 768, 895, 896, 1023,
               1024, 1025, 1151, 1279, 1280, 1535, 1536, 1537, 1791, 1792, 2047)


def corpus_row(S, V, seed):
    ds = synthetic_pretrain_dataset(64, 900, V, S, eos_token_id=V - 1, seed=seed)
    rows = np.stack([np.asarray(ds[i]["input_ids"]) for i in range(len(ds))])
    return rows[int(np.argmax((rows == V - 1).sum(1)))]                       # the row with the most documents


def edge_row(S, V, seed):
    row = np.random.default_rng(seed).integers(0, V - 1, size=S)
    for s in EDGE_STARTS:
        if s < S:
            row[s - 1] = V - 1                                                    # the EOS before column s opens a segment at s
    return row


def rows_seg(S, V=50257, seed=0):
    rows = np.stack([corpus_row(S, V, seed), edge_row(S, V, seed)])
    batch = DocumentCollator(V - 1)([{"input_ids": r} for r in rows])
    return segment_starts(batch["position_ids"]), batch


ATTN_CASES = {
    "llama125m_s1024": (1024, 12, 12, 0, 0.125),
    "llama3.2-1b_s1024": (1024, 32, 8, 0, 0.125),
    "llama3.2-1b_s2048": (2048, 32, 8, 0, 0.125),
    "gptneo_w256_s1024": (1024, 12, 12, 256, 1.0),
}


@pytest.mark.parametrize("case", list(ATTN_CASES))
def test_segmented_kernels_at_pretraining_shapes(case):
    S, Hq, Hk, window, sc = ATTN_CASES[case]
    B = 2
    C = ops.load_ext(required=True)
    seg, batch = rows_seg(S, seed=S + Hq)
    starts = [(batch["position_ids"][b] == 0).nonzero().flatten().tolist() for b in range(B)]
    assert len(starts[0]) >= 2 and {127, 128, 129} <= set(starts[1]), starts
    g = torch.Generator().manual_seed(S + Hq + window)
    amp = 0.7 * math.sqrt(0.125 / sc)                                             # the same logit spread at scale 1.0 (GPT-Neo)
    qkv = (torch.randn(B * S, (Hq + 2 * Hk) * D, generator=g) * amp).to(DEV, torch.bfloat16)
    d_o = (torch.randn(B * S, Hq * D, generator=g) * 0.5).to(DEV, torch.bfloat16)
    seg_d = seg.to(DEV)
    o, lse = C.attn_fwd(qkv, B, S, Hq, Hk, D, sc, window, seg_d)
    dq, dk, dv = C.attn_bwd(qkv, o, d_o, lse, B, S, Hq, Hk, D, sc, window, seg_d)
    torch.cuda.synchronize()
    got = {"o": o.view(B, S, Hq, D).float().cpu(), "dq": dq.view(B, S, Hq, D).float().cpu(), "dk": dk.view(B, S, Hk, D).float().cpu(),
           "dv": dv.view(B, S, Hk, D).float().cpu()}
    assert bool(torch.isfinite(lse).all())
    x = qkv.view(B, S, Hq + 2 * Hk, D)
    # fp32 reference (dense masked attention, autograd) on the device
    q, k, v = (t.float().requires_grad_() for t in (x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:]))
    ref = causal_attention_ref(q, k, v, scale=sc, window=window or None, seg=seg_d)
    gq, gk, gv = torch.autograd.grad(ref, (q, k, v), d_o.view(B, S, Hq, D).float())
    fp32 = {"o": ref.detach().cpu(), "dq": gq.cpu(), "dk": gk.cpu(), "dv": gv.cpu()}
    del q, k, v, ref, gq, gk, gv
    # blockwise references (the kernels' tiles, loop bounds and bf16 rounding points) for the first and the last KV group: a Python
    # loop over 128 x 128 tiles, run on the device
    G = Hq // Hk
    hq = list(range(G)) + list(range(Hq - G, Hq))
    hk = [0, Hk - 1]
    with torch.device(DEV):
        bo, blse = attention_blockwise_ref(x[:, :, hq], x[:, :, [Hq + h for h in hk]], x[:, :, [Hq + Hk + h for h in hk]], sc, window,
                                           seg=seg_d)
        bdq, bdk, bdv = attention_blockwise_bwd_ref(x[:, :, hq], x[:, :, [Hq + h for h in hk]], x[:, :, [Hq + Hk + h for h in hk]], bo,
                                                    d_o.view(B, S, Hq, D)[:, :, hq], blse, sc, window, seg=seg_d)
    block = {"o": bo.float().cpu(), "dq": bdq.float().cpu(), "dk": bdk.float().cpu(), "dv": bdv.float().cpu()}
    sub = {"o": hq, "dq": hq, "dk": hk, "dv": hk}
    report = []
    for ref_name, want in (("fp32", fp32), ("blockwise", block)):
        for name in ("o", "dq", "dk", "dv"):
            g_ = got[name] if ref_name == "fp32" else got[name][:, :, sub[name]]
            err = float((g_ - want[name]).abs().max())
            if name != "o":
                err /= float(want[name].abs().max())
            report.append(f"{ref_name}.{name}={err:.2e}")
            assert err < (O_TOL if name == "o" else G_TOL), (case, ref_name, name, err)
    lse_err = float((lse[:, hq] - blse).abs().max())
    report.append(f"blockwise.lse={lse_err:.2e}")
    assert lse_err < 1e-2
    print(f"[doc-mask attn] {case}: " + " ".join(report))


# ---------------------------------------------------------------------------------------------- per-document oracle, bf16 kernels
ORACLE_LENS = [[127, 1, 1, 128, 129, 190, 448], [700, 324]]                     # GPT-Neo: 700 and 448 outgrow the 256 window


def _bf16_model(family):
    from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    if family == "llama":
        m = LlamaForCausalLM(LlamaConfig(vocab_size=1000, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                                         num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=1024))
        names = [n for l in m.model.layers for n in (l.self_attn.qkv_proj, l.self_attn.o_proj)]
    else:
        m = GPTForCausalLM(GPTConfig(vocab_size=1000, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                                     max_position_embeddings=1024, attention_layers="alternating", window_size=256))
        names = [blk.attn.attention.qkv_proj for blk in m.transformer.h]
    return m.to(DEV, torch.bfloat16), names


@pytest.mark.parametrize("family", ["llama", "gptneo"])
def test_per_document_oracle_on_the_kernels(family):
    """Tolerances of the whole-model test of ``test_packing_gpu.py``: mean token loss within 3e-2, attention-weight gradients with
    cosine similarity > 0.99.  The documents alone run the unsegmented path (SDPA), so the two sides share no attention code.
    The fp64 check of document-masked steps at training widths, tensor by tensor under the whole-step criterion, is
    ``test_step_matrix_gpu.py``."""
    model, watched = _bf16_model(family)
    rows = doc_rows(ORACLE_LENS, np.random.default_rng(2), eos=999)
    batch = DocumentCollator(999)([{"input_ids": r} for r in rows])
    ids, pos, lab = (batch[k].to(DEV) for k in ("input_ids", "position_ids", "labels"))
    ops.reset_launch_counts()
    n_masked = int((lab[:, 1:] != -100).sum())
    loss = model(ids, position_ids=pos, labels=lab).loss * n_masked             # mean -> sum over the row's targets
    loss.backward()
    counts = ops.launch_counts()
    assert counts.get("attn_fwd_seg", 0) == 2 and counts.get("attn_bwd_seg", 0) == 4, counts
    g_masked = [p.grad.float().clone() for p in watched]
    model.zero_grad(set_to_none=True)
    total, n_alone = 0.0, 0
    for b in range(ids.shape[0]):
        starts = (batch["position_ids"][b] == 0).nonzero().flatten().tolist() + [ids.shape[1]]
        for a, e in zip(starts[:-1], starts[1:]):
            if e - a < 2:
                continue                                                          # a one-token document has no target
            d = ids[b:b + 1, a:e]
            part = model(d, labels=d).loss * (e - a - 1)
            part.backward()
            total += float(part)
            n_alone += e - a - 1
    assert n_alone == n_masked
    lm, la = float(loss) / n_masked, total / n_alone
    cos = [float(torch.nn.functional.cosine_similarity(gm.flatten(), p.grad.float().flatten(), dim=0)) for gm, p in zip(g_masked, watched)]
    print(f"[doc-mask oracle] {family}: mean loss masked {lm:.5f} alone {la:.5f}, gradient cosines {[round(c, 5) for c in cos]}")
    assert abs(lm - la) < 3e-2 and min(cos) > 0.99, (lm, la, cos)


# ---------------------------------------------------------------------------------------------- trainer
def _make(tmp_path, monkeypatch, mixed=True, steps=16, **kw):
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import ByteTokenizer
    from acco_b200.launch import DistEnv
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    monkeypatch.chdir(tmp_path)
    torch.manual_seed(0)
    cfg = LlamaConfig(vocab_size=1000, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, max_position_embeddings=256)
    ds = synthetic_pretrain_dataset(512, 100, 1000, 256, eos_token_id=999, seed=0)              # ~2.5 documents per row
    args = AttrDict(method_name="acco", batch_size=4, n_grad_accumulation=2, max_length=256, nb_steps_tot=steps, warmup=0,
                    learning_rate=1e-3, save=False, tensorboard=False, use_mixed_precision=mixed, static_accumulation=True, seed=1,
                    document_mask=True, **kw)
    return DecoupledTrainer(model=LlamaForCausalLM(cfg), tokenizer=ByteTokenizer(eos_token_id=999), train_dataset=ds, args=args,
                            log=logging.getLogger("dm"), env=DistEnv(id_run="dm"))


def _train(t):
    losses = []
    while not t.finished():
        t.step()
        losses.append(float(t.loss_host))
    t._drain()
    return losses


TRAINER_CASES = {"plain": {}, "fp8": dict(fp8=True), "max_grad_norm": dict(max_grad_norm=0.5)}


@pytest.mark.parametrize("case", list(TRAINER_CASES))
def test_trainer_document_mask_with_cuda_graphs(tmp_path, monkeypatch, case):
    from acco_b200.parallel.graphs import MicroBatchGraphs
    monkeypatch.delenv("ACCO_ATTN", raising=False)
    kw = TRAINER_CASES[case]
    captures, segmentations, replays = [], set(), [0]
    capture, replay = MicroBatchGraphs.capture, MicroBatchGraphs.replay

    def capture_spy(self, key, example, cleanup=None):
        captures.append(key)
        return capture(self, key, example, cleanup)

    def replay_spy(self, key, inputs):
        replays[0] += 1
        segmentations.add(inputs["position_ids"].cpu().numpy().tobytes())
        return replay(self, key, inputs)
    monkeypatch.setattr(MicroBatchGraphs, "capture", capture_spy)
    monkeypatch.setattr(MicroBatchGraphs, "replay", replay_spy)
    ops.reset_launch_counts()
    t = _make(tmp_path, monkeypatch, **kw)
    assert isinstance(t.train_dataloader.collate_fn, DocumentCollator)
    got = _train(t)
    counts = ops.launch_counts()
    keys = list(t._graphs._graphs) if t._graphs is not None else []
    assert keys and not getattr(t, "_graphs_disabled", None)
    assert len(captures) == len(keys) == len(set(captures)) <= 4, captures  # one capture per (parameter, accumulator) buffer pair
    assert replays[0] == t.micro_batches and len(segmentations) > len(keys), (replays, len(segmentations))
    assert counts.get("attn_fwd_seg", 0) > 0 and counts.get("attn_bwd_seg", 0) > 0 and counts.get("attn_fwd", 0) == 0, counts
    assert all(math.isfinite(x) for x in got)
    with monkeypatch.context() as mp:                                            # the fp32 CPU trainer on the same data and weights
        mp.setattr(torch.cuda, "is_available", lambda: False)
        ref = _train(_make(tmp_path, mp, mixed=False, **{k: v for k, v in kw.items() if k != "fp8"}))
    print(f"{case}: losses bf16 kernels {got[:3]} ... {got[-3:]}, fp32 CPU {ref[:3]} ... {ref[-3:]}")
    assert len(got) == len(ref)
    tol = 0.06 if case == "fp8" else 0.03
    torch.testing.assert_close(torch.tensor(got), torch.tensor(ref), rtol=tol, atol=0)
