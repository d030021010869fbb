"""Native GPT-2 / GPT-Neo style causal LM (LayerNorm, learned positions, GELU-new MLP,
global and sliding-window local attention).

The reference's default pre-training model is ``GPTNeoForCausalLM`` built from
``config/model/gpt-neo-125M.json`` (`/root/reference/main.py:39-41`): 12 layers alternating global / local
(window 256) attention, **no 1/sqrt(d) scaling of QK^T** and fp32 eager attention
(`transformers/models/gpt_neo/modeling_gpt_neo.py:105-130`), q/k/v projections without bias,
tied LM head.  ``arch='gptneo'`` reproduces exactly that; ``arch='gpt2'`` is the same block
with scaled, all-global attention (benchmark configuration 1's "GPT-2 small").

GPU layout (same recipe as the native Llama): activations are ``[T = B*S, H]`` row-major bf16; q/k/v are ONE fused
``[3H, H]`` weight and one wgmma GEMM; biases are added in the GEMM epilogue; residual-add + LayerNorm, GELU-new and the
softmax-CE are single sm_90a kernels (``ops.layernorm`` / ``ops.cross_entropy``); the vocabulary is padded to a multiple of
128 rows (50257 -> 50304; padded logits are masked inside the CE kernel and get zero gradient); wgrad GEMMs and the
LayerNorm dw/db reductions accumulate straight into the flat gradient arena.  ``state_dict()`` / ``load_state_dict()`` speak
HF GPT-Neo key names (``transformer.h.N.attn.attention.q_proj.weight`` ...) and un-padded shapes, so checkpoints interchange.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from .. import ops
from .base import NativeCausalLM, NativeConfig
from .output import CausalLMOutput

__all__ = ["GPTConfig", "GPTForCausalLM"]


@dataclass
class GPTConfig(NativeConfig):
    vocab_size: int = 50257
    hidden_size: int = 768
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    intermediate_size: Optional[int] = None
    max_position_embeddings: int = 1024
    layer_norm_epsilon: float = 1e-5
    attention_layers: Any = "alternating"   # "global" | "alternating" | explicit list of "global"/"local"
    window_size: int = 256
    scale_attn: bool = False                # GPT-Neo: False (no 1/sqrt(d)); GPT-2: True
    tie_word_embeddings: bool = True
    initializer_range: float = 0.02
    pad_vocab_multiple: int = 128
    model_type: str = "gpt_neo"

    def __post_init__(self):
        if self.intermediate_size is None:
            self.intermediate_size = 4 * self.hidden_size
        if isinstance(self.attention_layers, str):
            if self.attention_layers == "global":
                self.attention_layers = ["global"] * self.num_hidden_layers
            elif self.attention_layers == "alternating":
                self.attention_layers = [("global", "local")[i % 2] for i in range(self.num_hidden_layers)]
            else:
                raise ValueError("attention_layers must be 'global', 'alternating' or a list")
        assert len(self.attention_layers) == self.num_hidden_layers

    @classmethod
    def from_dict(cls, d: Dict[str, Any]) -> "GPTConfig":
        d = dict(d)
        # accept HF GPT-Neo json spellings
        if "num_layers" in d:
            d.setdefault("num_hidden_layers", d["num_layers"])
        if "num_heads" in d:
            d.setdefault("num_attention_heads", d["num_heads"])
        if "attention_types" in d and "attention_layers" not in d:
            layers: List[str] = []
            for kinds, rep in d["attention_types"]:
                layers.extend(list(kinds) * int(rep))
            d["attention_layers"] = layers
        return super().from_dict(d)

    def flops_per_token(self, seq_len: int) -> float:
        H, I, L = self.hidden_size, self.intermediate_size, self.num_hidden_layers
        mm = L * (4 * H * H + 2 * H * I) + self.vocab_size * H
        attn = L * 2 * H * seq_len / 2
        return 3.0 * 2.0 * (mm + attn)


class _LN(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim))
        self.bias = nn.Parameter(torch.zeros(dim))


class _Lin(nn.Module):
    def __init__(self, i: int, o: int):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(o, i))
        self.bias = nn.Parameter(torch.zeros(o))


class _Attention(nn.Module):
    def __init__(self, cfg: GPTConfig):
        super().__init__()
        H = cfg.hidden_size
        self.qkv_proj = nn.Parameter(torch.empty(3 * H, H))        # q | k | v rows, no bias (HF: three bias-free Linear)
        self.out_proj = _Lin(H, H)


class _AttnWrap(nn.Module):
    def __init__(self, cfg: GPTConfig):
        super().__init__()
        self.attention = _Attention(cfg)


class _MLP(nn.Module):
    def __init__(self, cfg: GPTConfig):
        super().__init__()
        self.c_fc = _Lin(cfg.hidden_size, cfg.intermediate_size)
        self.c_proj = _Lin(cfg.intermediate_size, cfg.hidden_size)


class _Block(nn.Module):
    def __init__(self, cfg: GPTConfig, kind: str):
        super().__init__()
        self.ln_1 = _LN(cfg.hidden_size)
        self.attn = _AttnWrap(cfg)
        self.ln_2 = _LN(cfg.hidden_size)
        self.mlp = _MLP(cfg)
        self.kind = kind


class _Transformer(nn.Module):
    def __init__(self, cfg: GPTConfig):
        super().__init__()
        self.wte = nn.Parameter(torch.empty(cfg.padded_vocab, cfg.hidden_size))
        self.wpe = nn.Parameter(torch.empty(cfg.max_position_embeddings, cfg.hidden_size))
        self.h = nn.ModuleList([_Block(cfg, k) for k in cfg.attention_layers])
        self.ln_f = _LN(cfg.hidden_size)


class GPTForCausalLM(NativeCausalLM):
    _hf_ignored_suffixes = (".attn.attention.bias", "masked_bias")      # HF's causal-mask buffers

    def __init__(self, config: GPTConfig):
        super().__init__(config)
        self.transformer = _Transformer(config)
        self.lm_head = None if config.tie_word_embeddings else nn.Parameter(torch.empty(config.padded_vocab, config.hidden_size))
        self.reset_parameters()

    def _init_fill(self, name: str) -> Optional[float]:
        if name.endswith("bias"):
            return 0.0
        return 1.0 if ".ln_" in name else None

    @property
    def embed_weight(self) -> torch.Tensor:
        return self.transformer.wte

    def num_parameters(self, padded: bool = False) -> int:
        n = sum(p.numel() for p in self.parameters())
        if not padded:
            pad = (self.config.padded_vocab - self.config.vocab_size) * self.config.hidden_size
            n -= pad * (1 if self.lm_head is None else 2)
        return n

    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                labels: Optional[torch.Tensor] = None, position_ids: Optional[torch.Tensor] = None,
                teacher_logits: Optional[torch.Tensor] = None, reference_logits: Optional[torch.Tensor] = None,
                preference_pairs: bool = False, **unused) -> CausalLMOutput:
        """HF-style call; ``attention_mask`` is accepted for API compatibility (right padding + causal attention: logits at
        non-pad positions do not depend on it; pad positions carry ``labels == -100``).  ``position_ids [B, S]`` marks packed rows
        (``PackedCollator``): the learned positions are gathered per token and no token attends to another sample.
        ``teacher_logits [B*S, Vp]`` (with labels): the loss is the distillation objective; ``reference_logits [B*S, Vp]`` (with
        labels, ``B = 2P`` rows of preference pairs): the DPO objective; ``preference_pairs=True`` (with labels, the same rows): the
        model's SimPO or ORPO objective (:meth:`_lm_output`)."""
        B, S = input_ids.shape
        return self._lm_output(self.padded_logits(input_ids, position_ids), labels, B, S, teacher_logits, reference_logits,
                               preference_pairs)

    def padded_logits(self, input_ids: torch.Tensor, position_ids: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The LM head's output ``[B*S, Vp]``, vocabulary padding included (a distillation teacher's logits)."""
        cfg = self.config
        B, S = input_ids.shape
        T = B * S
        Hh, D, H = cfg.num_attention_heads, cfg.head_dim, cfg.hidden_size
        eps = cfg.layer_norm_epsilon
        fp8 = self.fp8
        tr = self.transformer
        scale = (1.0 / math.sqrt(D)) if cfg.scale_attn else 1.0
        seg = None
        if position_ids is None:
            h = (ops.embedding(input_ids.reshape(T), tr.wte).view(B, S, H) + ops.main_grad_param(tr.wpe, S)).view(T, H)
        else:
            h = ops.embedding(input_ids.reshape(T), tr.wte) + ops.embedding(position_ids.reshape(T), tr.wpe)
            seg = ops.segment_starts(position_ids)
        branch = None          # output of the previous residual branch, not yet added to h
        for blk in tr.h:
            a = blk.attn.attention
            if branch is None:
                n = ops.layernorm(h, blk.ln_1.weight, blk.ln_1.bias, eps)
            else:
                n, h = ops.add_layernorm(branch, h, blk.ln_1.weight, blk.ln_1.bias, eps)
            qkv = ops.linear(n, a.qkv_proj, fp8=fp8)                                                       # [T, 3H]
            att = ops.packed_causal_attention(qkv, B, S, Hh, Hh, D, scale=scale,
                                              window=cfg.window_size if blk.kind == "local" else None, seg=seg)   # [T, H]
            o = ops.linear(att, a.out_proj.weight, a.out_proj.bias, fp8=fp8)
            n, h = ops.add_layernorm(o, h, blk.ln_2.weight, blk.ln_2.bias, eps)
            f = ops.linear(n, blk.mlp.c_fc.weight, blk.mlp.c_fc.bias, fp8=fp8)
            branch = ops.linear(ops.gelu_new(f), blk.mlp.c_proj.weight, blk.mlp.c_proj.bias, fp8=fp8)
        if branch is None:
            n = ops.layernorm(h, tr.ln_f.weight, tr.ln_f.bias, eps)
        else:
            n, h = ops.add_layernorm(branch, h, tr.ln_f.weight, tr.ln_f.bias, eps)
        return ops.linear(n, self.head_weight)                                                  # [T, Vp]

    def _hf_tensors(self) -> List[Tuple[str, torch.Tensor]]:
        """HF ``GPTNeoForCausalLM`` keys: the fused QKV weight is split back into HF's three projections."""
        H, V = self.config.hidden_size, self.config.vocab_size
        tr = self.transformer
        t = [("transformer.wte.weight", tr.wte[:V]), ("transformer.wpe.weight", tr.wpe)]
        for i, blk in enumerate(tr.h):
            b, a, mlp = f"transformer.h.{i}.", blk.attn.attention, blk.mlp
            t += [(b + "ln_1.weight", blk.ln_1.weight), (b + "ln_1.bias", blk.ln_1.bias),
                  (b + "attn.attention.q_proj.weight", a.qkv_proj[:H]),
                  (b + "attn.attention.k_proj.weight", a.qkv_proj[H:2 * H]),
                  (b + "attn.attention.v_proj.weight", a.qkv_proj[2 * H:]),
                  (b + "attn.attention.out_proj.weight", a.out_proj.weight), (b + "attn.attention.out_proj.bias", a.out_proj.bias),
                  (b + "ln_2.weight", blk.ln_2.weight), (b + "ln_2.bias", blk.ln_2.bias),
                  (b + "mlp.c_fc.weight", mlp.c_fc.weight), (b + "mlp.c_fc.bias", mlp.c_fc.bias),
                  (b + "mlp.c_proj.weight", mlp.c_proj.weight), (b + "mlp.c_proj.bias", mlp.c_proj.bias)]
        t += [("transformer.ln_f.weight", tr.ln_f.weight), ("transformer.ln_f.bias", tr.ln_f.bias),
              ("lm_head.weight", self.head_weight[:V])]
        return t
