import numpy as np
import pytest
import torch

from acco_b200.data import (BatchLoader, ByteTokenizer, DeviceFeeder, PadCollator, TokenDataset, load_from_disk,
                            make_const_len_tokenize_fn, make_truncate_tokenize_fn, pack_const_len, stack_collate,
                            synthetic_pretrain_dataset, synthetic_sft_dataset, synthetic_text_dataset)


def test_pack_const_len_semantics():
    # concat docs + EOS, cut into rows, drop the tail (trainer_base.py:84-97)
    docs = [[1, 2, 3], [4, 5], [6, 7, 8, 9]]
    rows = pack_const_len(docs, 4, eos_token_id=0)
    assert rows.tolist() == [[1, 2, 3, 0], [4, 5, 0, 6], [7, 8, 9, 0]]
    rows = pack_const_len(docs, 5, eos_token_id=0)
    assert rows.tolist() == [[1, 2, 3, 0, 4], [5, 0, 6, 7, 8]]          # tail [9, 0] dropped
    assert pack_const_len([], 4, 0).shape == (0, 4)


def test_tokenize_fns_and_map():
    tok = ByteTokenizer()
    ds = synthetic_text_dataset(20, 12, seed=0)
    packed = ds.map(make_const_len_tokenize_fn(tok, "text", 16), batched=True, remove_columns=ds.column_names)
    assert packed.column_names == ["input_ids"] and all(len(r) == 16 for r in packed["input_ids"])
    flat = np.concatenate([np.asarray(r) for r in packed["input_ids"]])
    assert (flat == tok.eos_token_id).sum() >= 1
    trunc = ds.map(make_truncate_tokenize_fn(tok, "text", 10), batched=True, remove_columns=ds.column_names)
    assert len(trunc) == 20 and max(len(r) for r in trunc["input_ids"]) <= 10


def test_dataset_shard_split_disk(tmp_path):
    ds = TokenDataset({"input_ids": torch.arange(40).reshape(10, 4)})
    a, b = ds.shard(2, 0), ds.shard(2, 1)
    assert len(a) == len(b) == 5 and a[0]["input_ids"].tolist() == [0, 1, 2, 3] and b[0]["input_ids"].tolist() == [4, 5, 6, 7]
    sp = ds.train_test_split(0.2, seed=42)
    assert len(sp["train"]) == 8 and len(sp["test"]) == 2
    sp2 = ds.train_test_split(0.2, seed=42)
    assert torch.equal(sp["test"]["input_ids"], sp2["test"]["input_ids"])
    ds.save_to_disk(str(tmp_path / "d"))
    assert torch.equal(load_from_disk(str(tmp_path / "d"))["input_ids"], ds["input_ids"])


def test_collators():
    b = stack_collate([{"input_ids": [1, 2, 3]}, {"input_ids": [4, 5, 6]}])
    assert b["input_ids"].dtype == torch.long and b["input_ids"].shape == (2, 3)
    eos = 9
    col = PadCollator(pad_token_id=eos)
    out = col([{"input_ids": [1, 2, eos, 3]}, {"input_ids": [4, 5]}])
    assert out["input_ids"].tolist() == [[1, 2, eos, 3], [4, 5, eos, eos]]
    assert out["attention_mask"].tolist() == [[1, 1, 1, 1], [1, 1, 0, 0]]
    # pad == eos  =>  every EOS label is masked, also the real one
    assert out["labels"].tolist() == [[1, 2, -100, 3], [4, 5, -100, -100]]
    out2 = PadCollator(eos, mask_all_pad_tokens=False)([{"input_ids": [1, 2, eos, 3]}, {"input_ids": [4, 5]}])
    assert out2["labels"].tolist() == [[1, 2, eos, 3], [4, 5, -100, -100]]


def test_loader_and_feeder_epoch_restart():
    ds = synthetic_pretrain_dataset(40, 30, 100, 8, seed=0)
    n_rows = len(ds)
    ld = BatchLoader(ds, 4, stack_collate, shuffle=True, drop_last=True, seed=1)
    assert len(ld) == n_rows // 4
    seen = [b["input_ids"] for b in ld]
    assert len(seen) == len(ld) and all(s.shape == (4, 8) for s in seen)
    fd = DeviceFeeder(ld, torch.device("cpu"), prefetch=2)
    for _ in range(2 * len(ld) + 1):           # crosses epoch boundaries without StopIteration
        assert fd.next()["input_ids"].shape == (4, 8)
    assert fd.epochs >= 1
    fd.close()


def test_sft_shapes():
    ds = synthetic_sft_dataset(32, 20, 200, 24, seed=0)
    lens = [len(r) for r in ds["input_ids"]]
    assert max(lens) <= 24 and len(set(lens)) > 3


def test_native_packer_matches_numpy_reference():
    """csrc/host_data.cpp (used automatically when the extension is built) == the pure-numpy packing rule."""
    from acco_b200.data import packing
    rng = np.random.default_rng(0)
    docs = [rng.integers(1, 100, size=int(n)).tolist() for n in rng.integers(0, 40, size=200)]

    def reference(docs, L, eos):
        flat = []
        for d in docs:
            flat += list(d) + [eos]
        rows = len(flat) // L
        return np.asarray(flat[: rows * L], dtype=np.int64).reshape(rows, L)

    for L in (1, 7, 16, 33):
        got = packing.pack_const_len(docs, L, eos_token_id=0)
        assert got.dtype == np.int64 and np.array_equal(got, reference(docs, L, 0))
    if packing._native() is None:
        pytest.skip("extension not built: only the numpy path was exercised")


def test_group_by_length_batches_have_similar_lengths():
    ds = synthetic_sft_dataset(400, 40, 200, 128, seed=3)
    plain = BatchLoader(ds, 8, PadCollator(199, pad_to_multiple_of=1), shuffle=True, seed=0)
    grouped = BatchLoader(ds, 8, PadCollator(199, pad_to_multiple_of=1), shuffle=True, seed=0, group_by_length=True, mega_batch_mult=10)

    def waste(loader):
        pad = tot = 0
        seen = 0
        for b in loader:
            pad += int((b["attention_mask"] == 0).sum())
            tot += b["attention_mask"].numel()
            seen += b["input_ids"].shape[0]
        return pad / tot, seen
    wp, n1 = waste(plain)
    wg, n2 = waste(grouped)
    assert n1 == n2 == 400 and wg < 0.5 * wp        # same rows, far less padding
    first = next(iter(grouped))
    assert first["input_ids"].shape[1] == max(len(r) for r in ds["input_ids"])   # longest row comes first


def test_feeder_with_worker_processes_matches_in_thread_order():
    """`dataloader_num_workers >= 2` fans collation out to persistent worker processes; batches and their order are unchanged."""
    import torch
    from acco_b200.data import BatchLoader, DeviceFeeder, stack_collate, synthetic_pretrain_dataset
    ds = synthetic_pretrain_dataset(64, 12, 50, 8, seed=3)
    a = DeviceFeeder(BatchLoader(ds, 4, stack_collate, shuffle=True, seed=5), torch.device("cpu"), num_workers=0)
    b = DeviceFeeder(BatchLoader(ds, 4, stack_collate, shuffle=True, seed=5), torch.device("cpu"), num_workers=2)
    try:
        assert b.num_workers == 2
        n = len(a.loader)
        for _ in range(n + 3):                       # crosses an epoch boundary: persistent workers keep serving
            assert torch.equal(a.next()["input_ids"], b.next()["input_ids"])
    finally:
        a.close()
        b.close()


def test_feeder_counts_real_tokens_from_the_attention_mask():
    """SFT batches are ragged + padded: throughput must count non-pad tokens (attention-mask sum), not batch x padded length."""
    import torch
    from acco_b200.data import BatchLoader, DeviceFeeder, PadCollator, stack_collate, synthetic_pretrain_dataset, synthetic_sft_dataset
    ds = synthetic_sft_dataset(40, 10, 95, 32, seed=2)
    f = DeviceFeeder(BatchLoader(ds, 4, PadCollator(pad_token_id=95, max_length=32), shuffle=False), torch.device("cpu"))
    try:
        want = 0
        for _ in range(5):
            b = f.next()
            want += int(b["attention_mask"].sum())
        assert f.tokens_real == want and want < 5 * 4 * 32
    finally:
        f.close()
    g = DeviceFeeder(BatchLoader(synthetic_pretrain_dataset(64, 12, 50, 8, seed=3), 4, stack_collate), torch.device("cpu"))
    try:
        g.next(), g.next_host()
        assert g.tokens_real == 2 * 4 * 8
    finally:
        g.close()


def test_feeder_thread_is_joined_before_the_interpreter_exits():
    """A feeder whose producer thread is still running torch / numpy code when the interpreter finalises used to abort the process
    (`terminate called without an active exception`, exit code 134): a finished job looked like a crash to its launcher.  Both an
    explicit `close()` and a forgotten one (finalizer at exit) must end with exit code 0."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys, torch; sys.path.insert(0, %r);"
            "from acco_b200.data import synthetic_pretrain_dataset;"
            "from acco_b200.data.loader import BatchLoader, DeviceFeeder;"
            "from acco_b200.data.collate import stack_collate;"
            "ds = synthetic_pretrain_dataset(256, 600, 5000, 512, seed=0);"
            "f = DeviceFeeder(BatchLoader(ds, 8, stack_collate, seed=0), torch.device('cpu'), prefetch=4);"
            "[f.next() for _ in range(100)];"
            "f.close() if sys.argv[1] == 'close' else None" % root)
    for mode in ("close", "forget"):
        p = subprocess.run([sys.executable, "-c", code, mode], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
        assert p.returncode == 0, (mode, p.returncode, p.stdout[-500:])
