from .collate import PREFERENCE_COLUMNS, DocumentCollator, PackedCollator, PadCollator, PreferenceCollator, stack_collate
from .dataset import TokenDataset, load_from_disk
from .loader import BatchLoader, DeviceFeeder
from .packing import (make_const_len_tokenize_fn, make_packed_tokenize_fn, make_preference_tokenize_fn, make_truncate_tokenize_fn,
                      pack_const_len, pack_sft, truncate_docs)
from .synthetic import (synthetic_documents, synthetic_pretrain_dataset, synthetic_preference_dataset, synthetic_sft_dataset,
                        synthetic_text_dataset, synthetic_token_batches)
from .tokenizer import ByteTokenizer

__all__ = [
    "DocumentCollator", "PackedCollator", "PadCollator", "PreferenceCollator", "PREFERENCE_COLUMNS", "stack_collate", "TokenDataset", "load_from_disk", "BatchLoader", "DeviceFeeder",
    "make_const_len_tokenize_fn", "make_truncate_tokenize_fn", "make_packed_tokenize_fn", "make_preference_tokenize_fn", "pack_const_len", "pack_sft",
    "truncate_docs",
    "synthetic_documents", "synthetic_pretrain_dataset", "synthetic_preference_dataset", "synthetic_sft_dataset", "synthetic_text_dataset",
    "synthetic_token_batches", "ByteTokenizer",
]
