"""Document masking for const-len pre-training rows (``document_mask: True``), CPU side:

* ``DocumentCollator`` against a per-token oracle of its contract (segments, positions, labels);
* the per-document oracle: a masked row's summed token loss and its parameter gradients equal those of every document run alone
  as its own row (positions from 0), in fp32, for a GQA Llama and a GPT-Neo whose documents outgrow the local layers' window;
  two mutants (positions left at ``arange``, the cross-document label kept) fail the same check;
* the trainer: its validation, the ACCO / DPU / DDP trainers with the key on, the key off leaving the batches unchanged, and the
  command line on the synthetic pre-training corpus."""
import copy
import math
import os
import sys

import numpy as np
import pytest
import torch

from acco_b200.data import ByteTokenizer, DocumentCollator, stack_collate, synthetic_pretrain_dataset

from helpers import LOG, base_args, tiny_model

EOS = 95
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def oracle(row, eos):
    """Per token, straight from the contract: -> (position_ids, labels)."""
    pos, lab, start = [], [], 0
    for s, tok in enumerate(row):
        if s > 0 and row[s - 1] == eos:
            start = s
        pos.append(s - start)
        lab.append(-100 if (s == start and s > 0) else tok)
    return pos, lab


def random_rows(B, S, n_eos, rng, eos=EOS):
    rows = rng.integers(0, eos, size=(B, S))
    for r in rows:
        r[rng.choice(S, size=n_eos, replace=False)] = eos
    return rows


# ---------------------------------------------------------------------------------------------- DocumentCollator
def _check_collator(rows, eos=EOS):
    out = DocumentCollator(eos)([{"input_ids": r} for r in rows])
    assert set(out) == {"input_ids", "labels", "position_ids"}
    assert all(v.dtype == torch.int64 and v.shape == rows.shape for v in out.values())
    assert out["input_ids"].tolist() == rows.tolist()
    for b, r in enumerate(rows.tolist()):
        pos, lab = oracle(r, eos)
        assert out["position_ids"][b].tolist() == pos
        assert out["labels"][b].tolist() == lab
    seg = torch.arange(rows.shape[1]) - out["position_ids"]
    assert bool((seg[:, 1:] >= seg[:, :-1]).all())                              # the segmented kernels' precondition
    return out


@pytest.mark.parametrize("n_eos", [0, 1, 2, 5, 17, 40])
@pytest.mark.parametrize("S", [64, 256])
def test_collator_matches_the_per_token_oracle(n_eos, S):
    rng = np.random.default_rng(S + n_eos)
    _check_collator(random_rows(4, S, n_eos, rng))


@pytest.mark.parametrize("case", ["eos_first", "eos_last", "eos_run", "eos_run_at_end", "all_eos", "eos_at_1"])
def test_collator_edges(case):
    rng = np.random.default_rng(7)
    r = rng.integers(0, EOS, size=(1, 32))
    if case == "eos_first":
        r[0, 0] = EOS
    elif case == "eos_last":
        r[0, 31] = EOS                                                            # opens no segment
    elif case == "eos_run":
        r[0, 10:14] = EOS                                                         # one-token segments
    elif case == "eos_run_at_end":
        r[0, 28:] = EOS
    elif case == "all_eos":
        r[:] = EOS
    elif case == "eos_at_1":
        r[0, 1] = EOS
    out = _check_collator(r)
    if case == "eos_last":
        assert out["position_ids"][0].tolist() == list(range(32))
    if case == "eos_run":
        assert out["position_ids"][0, 10:16].tolist() == [10, 0, 0, 0, 0, 1]
        assert out["labels"][0, 11:15].tolist() == [-100] * 4
    if case == "all_eos":
        assert out["position_ids"][0].tolist() == [0] * 32
        assert out["labels"][0].tolist() == [EOS] + [-100] * 31


def test_collator_without_eos_is_the_plain_row():
    rows = np.random.default_rng(3).integers(0, EOS, size=(3, 48))
    out = _check_collator(rows)
    assert torch.equal(out["position_ids"], torch.arange(48).expand(3, 48))
    assert torch.equal(out["labels"], out["input_ids"])
    assert torch.equal(out["input_ids"], stack_collate([{"input_ids": r} for r in rows])["input_ids"])


def test_collator_keeps_eos_targets_and_reads_packed_rows():
    """Rows from ``pack_const_len``: every EOS stays a target, and each document's positions restart right after its EOS."""
    ds = synthetic_pretrain_dataset(200, 30, 96, 64, eos_token_id=EOS, seed=2)
    out = DocumentCollator(EOS)([ds[i] for i in range(len(ds))])
    ids, lab, pos = out["input_ids"], out["labels"], out["position_ids"]
    assert bool((lab[ids == EOS] == EOS).all())
    assert int((ids == EOS).sum()) > len(ds)                                      # several documents per row
    after = torch.zeros_like(ids, dtype=torch.bool)
    after[:, 1:] = ids[:, :-1] == EOS
    assert bool((pos[after] == 0).all()) and bool((lab[after] == -100).all())
    assert int((lab == -100).sum()) == int(after.sum())


# ---------------------------------------------------------------------------------------------- per-document oracle
def _tiny_gptneo(window=256, n_pos=1024):
    from acco_b200.models import GPTConfig, GPTForCausalLM
    torch.manual_seed(3)
    return GPTForCausalLM(GPTConfig(vocab_size=96, hidden_size=32, num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=n_pos,
                                    attention_layers="alternating", window_size=window, pad_vocab_multiple=8))


def doc_rows(lens_per_row, rng, eos=EOS):
    """Rows made of documents: every length but the last of a row ends in EOS (the last one runs off the row's end, as in
    ``pack_const_len``); the first one plays the tail of a document cut by the previous row."""
    rows = []
    for lens in lens_per_row:
        r = []
        for i, n in enumerate(lens):
            d = rng.integers(0, eos, size=n).tolist()
            if i < len(lens) - 1:
                d[-1] = eos
            r += d
        rows.append(r)
    return np.asarray(rows, dtype=np.int64)


def token_loss(logits, labels):
    """Summed next-token loss with the models' label shift."""
    tgt = torch.full_like(labels, -100)
    tgt[:, :-1] = labels[:, 1:]
    return torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]).float(), tgt.reshape(-1), ignore_index=-100,
                                             reduction="sum")


def per_document_errors(model, batch, position_ids=None, labels=None):
    """-> (loss error, worst gradient error relative to the largest gradient) between the masked rows and the documents alone."""
    ids = batch["input_ids"]
    pos = batch["position_ids"] if position_ids is None else position_ids
    lab = batch["labels"] if labels is None else labels
    params = [p for p in model.parameters() if p.requires_grad]
    masked = token_loss(model(ids, position_ids=pos).logits, lab)
    g_masked = torch.autograd.grad(masked, params, allow_unused=True)
    alone = 0.0
    for b in range(ids.shape[0]):
        starts = (batch["position_ids"][b] == 0).nonzero().flatten().tolist() + [ids.shape[1]]
        for a, e in zip(starts[:-1], starts[1:]):
            d = ids[b:b + 1, a:e]
            alone = alone + token_loss(model(d).logits, d)
    g_alone = torch.autograd.grad(alone, params, allow_unused=True)
    gerr = 0.0
    for gm, ga in zip(g_masked, g_alone):
        gm = torch.zeros(()) if gm is None else gm
        ga = torch.zeros(()) if ga is None else ga
        gerr = max(gerr, float((gm - ga).abs().max() / max(float(ga.abs().max()), 1e-12)))
    return abs(float(masked.detach()) - float(alone.detach())) / float(alone.detach()), gerr


LOSS_TOL, GRAD_TOL = 1e-5, 1e-4          # fp32: reassociation only
ORACLE_ROWS = {
    # (Llama rows, GPT-Neo rows): GPT-Neo's documents reach past its 256-token window, so its local layer cuts inside a segment
    "llama": ([[5, 40, 1, 1, 60, 21], [128], [127, 1]], 128),
    "gptneo": ([[100, 300, 1, 1, 366], [600, 168], [767, 1]], 768),
}


@pytest.mark.parametrize("family", ["llama", "gptneo"])
def test_masked_rows_equal_each_document_alone(family):
    lens, S = ORACLE_ROWS[family]
    assert all(sum(r) == S for r in lens)
    model = tiny_model(vocab=96, hidden=32) if family == "llama" else _tiny_gptneo()     # tiny Llama: GQA 4 / 2
    batch = DocumentCollator(EOS)([{"input_ids": r} for r in doc_rows(lens, np.random.default_rng(5))])
    lerr, gerr = per_document_errors(model, batch)
    print(f"{family}: loss {lerr:.2e}, gradients {gerr:.2e}")
    assert lerr < LOSS_TOL and gerr < GRAD_TOL, (lerr, gerr)
    # mutants: positions left at arange (no restart, no mask), and the cross-document prediction kept as a target
    B, S = batch["input_ids"].shape
    lerr_pos, gerr_pos = per_document_errors(model, batch, position_ids=torch.arange(S).expand(B, S))
    lerr_lab, gerr_lab = per_document_errors(model, batch, labels=batch["input_ids"])
    print(f"{family} mutants: arange positions {lerr_pos:.2e} / {gerr_pos:.2e}, cross-document label {lerr_lab:.2e} / {gerr_lab:.2e}")
    for name, le, ge in (("positions", lerr_pos, gerr_pos), ("label", lerr_lab, gerr_lab)):
        assert le > 100 * LOSS_TOL or ge > 100 * GRAD_TOL, (name, le, ge)


# ---------------------------------------------------------------------------------------------- trainer
class _HFLike(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(4))

    def forward(self, input_ids=None, labels=None, **kw):
        return ((self.w ** 2).sum(),)


def _trainer(tokenizer="byte", model=None, dataset=None, **kw):
    from acco_b200 import DecoupledTrainer
    from acco_b200.launch import DistEnv
    tok = ByteTokenizer(eos_token_id=EOS) if tokenizer == "byte" else tokenizer
    ds = dataset if dataset is not None else synthetic_pretrain_dataset(400, 12, 96, 32, eos_token_id=EOS, seed=1)
    ev = synthetic_pretrain_dataset(40, 12, 96, 32, eos_token_id=EOS, seed=2)
    a = dict(document_mask=True, max_length=32, batch_size=2)
    a.update(kw)
    return DecoupledTrainer(model=model or tiny_model(), tokenizer=tok, train_dataset=ds, eval_dataset=ev, args=base_args(**a), log=LOG,
                            env=DistEnv(id_run="docmask"))


def _tok(eos):
    t = ByteTokenizer()
    t.eos_token_id = eos
    return t


@pytest.mark.parametrize("bad,match", [
    ({"document_mask": "yes"}, "true or false"),
    ({"document_mask": 1}, "true or false"),
    ({"const_len_batch": False}, "const_len_batch=True"),
    ({"model": "hf"}, "native model"),
    ({"tokenizer": None}, "eos_token_id"),
    ({"tokenizer": _tok(None)}, "eos_token_id"),
    ({"tokenizer": _tok(95.0)}, "eos_token_id"),
    ({"tokenizer": _tok(True)}, "eos_token_id"),
])
def test_trainer_rejects_invalid_combinations(workdir, bad, match):
    bad = dict(bad)
    if bad.get("model") == "hf":
        bad["model"] = _HFLike()
    with pytest.raises(ValueError, match=match):
        _trainer(**bad)


def test_trainer_accepts_a_numpy_eos_id(workdir):
    t = _trainer(tokenizer=_tok(np.int64(EOS)), nb_steps_tot=2)
    assert isinstance(t.train_dataloader.collate_fn, DocumentCollator) and t.train_dataloader.collate_fn.eos == EOS


@pytest.mark.parametrize("method", ["acco", "dpu", "ddp"])
def test_trainers_run_with_document_masking(workdir, monkeypatch, method):
    seen = []
    model = tiny_model()
    fwd = model.forward

    def forward(input_ids, **kw):
        seen.append(kw.get("position_ids"))
        return fwd(input_ids, **kw)
    monkeypatch.setattr(model, "forward", forward)
    t = _trainer(model=model, method_name=method, nb_steps_tot=40, learning_rate=5e-3)
    assert isinstance(t.train_dataloader.collate_fn, DocumentCollator) and isinstance(t.eval_dataloader.collate_fn, DocumentCollator)
    losses = []
    while not t.finished():
        t.step()
        losses.append(float(t.loss_host))
    t._finish("")
    assert t.sched.count_grad_tot >= 40 and all(math.isfinite(x) for x in losses)
    assert seen and all(p is not None for p in seen)
    assert any(bool((p[:, 1:] == 0).any()) for p in seen)                         # positions restarted inside rows
    assert sum(losses[-10:]) / 10 < sum(losses[:10]) / 10, losses
    n = len(seen)
    assert torch.isfinite(t.eval_loop()) and len(seen) > n and all(p is not None for p in seen[n:])


def test_key_off_keeps_stack_collate_batches(workdir):
    t = _trainer(document_mask=False, nb_steps_tot=2)
    loader = t.train_dataloader
    assert loader.collate_fn is stack_collate and t.eval_dataloader.collate_fn is stack_collate
    twin = copy.deepcopy(loader)
    for idx, got in zip(twin.index_batches(), loader):
        want = stack_collate([t.train_dataset[int(i)] for i in idx])
        assert list(got) == ["input_ids"] and torch.equal(got["input_ids"], want["input_ids"])
    on = _trainer(nb_steps_tot=2)
    assert isinstance(on.train_dataloader.collate_fn, DocumentCollator)
    for idx, got in zip(copy.deepcopy(on.train_dataloader).index_batches(), on.train_dataloader):
        assert torch.equal(got["input_ids"], stack_collate([on.train_dataset[int(i)] for i in idx])["input_ids"])   # same rows


def test_cli_pretraining_with_document_mask(workdir, monkeypatch):
    sys.path.insert(0, ROOT)
    import main as cli
    from acco_b200.data import collate
    calls = []
    orig = collate.DocumentCollator.__call__

    def call(self, batch):
        calls.append(self.eos)
        return orig(self, batch)
    monkeypatch.setattr(collate.DocumentCollator, "__call__", call)
    stats = cli.main(["train=acco", "model=tiny", "data=synthetic", "train.nb_steps_tot=6", "train.batch_size=2", "train.max_length=32",
                      "train.use_mixed_precision=False", "data.synthetic_docs=200", "data.synthetic_mean_len=12", "train.warmup=0",
                      "run_name=docmask", "train.save=False", "train.document_mask=true", "train.dataloader_num_workers=0"])
    assert stats["count_grad_tot"] >= 6
    assert calls and set(calls) == {511}                                          # the tiny model's vocab_size - 1
