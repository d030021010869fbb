import logging

import torch
import torch.nn as nn

from acco_b200 import AttrDict
from acco_b200.models import LlamaConfig, LlamaForCausalLM

LOG = logging.getLogger("acco-test")


def tiny_model(seed=0, vocab=96, hidden=32, layers=2):
    torch.manual_seed(seed)
    return LlamaForCausalLM(LlamaConfig(vocab_size=vocab, hidden_size=hidden, intermediate_size=48, num_hidden_layers=layers,
                                        num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=32,
                                        pad_vocab_multiple=8))


def base_args(**kw):
    a = dict(method_name="acco", batch_size=2, n_grad_accumulation=1, max_length=16, nb_steps_tot=12, warmup=0,
             use_mixed_precision=False, learning_rate=1e-2, weight_decay=0.0, scheduler_name="constant", save=False,
             tensorboard=False, const_len_batch=True, eval=False, n_warmup_steps=0, seed=123, log_every=10)
    a.update(kw)
    return AttrDict(a)


class ToyQuadratic(nn.Module):
    """Loss whose k-th evaluation has gradient 0.1*(k+1)*p  (the toy of the golden-trace test)."""

    def __init__(self, p0):
        super().__init__()
        self.p = nn.Parameter(torch.tensor(p0, dtype=torch.float32))
        self.k = 0

    def forward(self, input_ids=None, labels=None, **kw):
        loss = 0.05 * (self.k + 1) * (self.p ** 2).sum()
        self.k += 1
        return (loss,)
