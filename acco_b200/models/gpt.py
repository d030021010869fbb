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
from collections import OrderedDict
from dataclasses import dataclass, asdict
from typing import Any, Dict, List, Optional

import torch
import torch.nn as nn

from .. import ops
from .output import CausalLMOutput

__all__ = ["GPTConfig", "GPTForCausalLM"]


@dataclass
class GPTConfig:
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

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads

    @property
    def padded_vocab(self) -> int:
        m = max(int(self.pad_vocab_multiple), 1)
        return ((self.vocab_size + m - 1) // m) * m

    def to_dict(self) -> Dict[str, Any]:
        return asdict(self)

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
        keys = cls.__dataclass_fields__.keys()
        return cls(**{k: v for k, v in d.items() if k in keys})

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


class GPTForCausalLM(nn.Module):
    def __init__(self, config: GPTConfig):
        super().__init__()
        self.config = config
        self.transformer = _Transformer(config)
        self.lm_head = None if config.tie_word_embeddings else nn.Parameter(torch.empty(config.padded_vocab, config.hidden_size))
        self.reset_parameters()

    @torch.no_grad()
    def reset_parameters(self) -> None:
        std = self.config.initializer_range
        V = self.config.vocab_size
        for name, p in self.named_parameters():
            if name.endswith("bias"):
                p.zero_()
            elif ".ln_" in name or name.endswith("ln_f.weight"):
                p.fill_(1.0)
            else:
                p.normal_(0.0, std)
        # alignment padding rows of the vocabulary are exactly zero and stay zero
        self.transformer.wte[V:].zero_()
        if self.lm_head is not None:
            self.lm_head[V:].zero_()

    @property
    def head_weight(self) -> torch.Tensor:
        return self.transformer.wte if self.lm_head is None else self.lm_head

    def num_parameters(self, padded: bool = False) -> int:
        n = sum(p.numel() for p in self.parameters())
        if not padded:
            pad = (self.config.padded_vocab - self.config.vocab_size) * self.config.hidden_size
            n -= pad * (1 if self.lm_head is None else 2)
        return n

    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                labels: Optional[torch.Tensor] = None, **unused) -> CausalLMOutput:
        """HF-style call; ``attention_mask`` is accepted for API compatibility (right padding + causal attention: logits at
        non-pad positions do not depend on it; pad positions carry ``labels == -100``)."""
        cfg = self.config
        B, S = input_ids.shape
        T = B * S
        Hh, D, H = cfg.num_attention_heads, cfg.head_dim, cfg.hidden_size
        eps = cfg.layer_norm_epsilon
        tr = self.transformer
        scale = (1.0 / math.sqrt(D)) if cfg.scale_attn else 1.0
        h = (ops.embedding(input_ids.reshape(T), tr.wte).view(B, S, H) + tr.wpe[:S]).view(T, H)
        branch = None          # output of the previous residual branch, not yet added to h
        for blk in tr.h:
            a = blk.attn.attention
            if branch is None:
                n = ops.layernorm(h, blk.ln_1.weight, blk.ln_1.bias, eps)
            else:
                n, h = ops.add_layernorm(branch, h, blk.ln_1.weight, blk.ln_1.bias, eps)
            qkv = ops.linear(n, a.qkv_proj)                                                       # [T, 3H]
            att = ops.packed_causal_attention(qkv, B, S, Hh, Hh, D, scale=scale,
                                              window=cfg.window_size if blk.kind == "local" else None)   # [T, H]
            o = ops.linear(att, a.out_proj.weight, a.out_proj.bias)
            n, h = ops.add_layernorm(o, h, blk.ln_2.weight, blk.ln_2.bias, eps)
            f = ops.linear(n, blk.mlp.c_fc.weight, blk.mlp.c_fc.bias)
            branch = ops.linear(ops.gelu_new(f), blk.mlp.c_proj.weight, blk.mlp.c_proj.bias)
        if branch is None:
            n = ops.layernorm(h, tr.ln_f.weight, tr.ln_f.bias, eps)
        else:
            n, h = ops.add_layernorm(branch, h, tr.ln_f.weight, tr.ln_f.bias, eps)
        logits = ops.linear(n, self.head_weight)                                                  # [T, Vp]
        if labels is None:
            return CausalLMOutput(loss=None, logits=logits.view(B, S, -1)[..., : cfg.vocab_size])
        shifted = torch.full_like(labels, -100)
        shifted[:, :-1] = labels[:, 1:]
        loss = ops.softmax_cross_entropy(logits, shifted.reshape(T), cfg.vocab_size, -100)
        return CausalLMOutput(loss=loss, logits=None)

    # ------------------------------------------------------------------ HF-compatible checkpoints
    def state_dict(self, *args, destination=None, prefix: str = "", keep_vars: bool = False, **kw):
        """HF ``GPTNeoForCausalLM`` key names and shapes (fused QKV split, vocab padding removed); the tensors are views of the
        live parameters (hence of the flat arena)."""
        cfg = self.config
        H, V = cfg.hidden_size, cfg.vocab_size
        get = (lambda p: p) if keep_vars else (lambda p: p.detach())
        sd = destination if destination is not None else OrderedDict()
        tr = self.transformer
        sd[prefix + "transformer.wte.weight"] = get(tr.wte)[:V]
        sd[prefix + "transformer.wpe.weight"] = get(tr.wpe)
        for i, blk in enumerate(tr.h):
            b = f"{prefix}transformer.h.{i}."
            a = blk.attn.attention
            qkv = get(a.qkv_proj)
            sd[b + "ln_1.weight"], sd[b + "ln_1.bias"] = get(blk.ln_1.weight), get(blk.ln_1.bias)
            sd[b + "attn.attention.q_proj.weight"] = qkv[:H]
            sd[b + "attn.attention.k_proj.weight"] = qkv[H:2 * H]
            sd[b + "attn.attention.v_proj.weight"] = qkv[2 * H:]
            sd[b + "attn.attention.out_proj.weight"], sd[b + "attn.attention.out_proj.bias"] = get(a.out_proj.weight), get(a.out_proj.bias)
            sd[b + "ln_2.weight"], sd[b + "ln_2.bias"] = get(blk.ln_2.weight), get(blk.ln_2.bias)
            sd[b + "mlp.c_fc.weight"], sd[b + "mlp.c_fc.bias"] = get(blk.mlp.c_fc.weight), get(blk.mlp.c_fc.bias)
            sd[b + "mlp.c_proj.weight"], sd[b + "mlp.c_proj.bias"] = get(blk.mlp.c_proj.weight), get(blk.mlp.c_proj.bias)
        sd[prefix + "transformer.ln_f.weight"], sd[prefix + "transformer.ln_f.bias"] = get(tr.ln_f.weight), get(tr.ln_f.bias)
        sd[prefix + "lm_head.weight"] = get(self.head_weight)[:V]
        return sd

    @torch.no_grad()
    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        cfg = self.config
        H, V = cfg.hidden_size, cfg.vocab_size
        sd = {k: v for k, v in dict(state_dict).items() if not k.endswith(".attn.attention.bias") and not k.endswith("masked_bias")}
        used, missing = set(), []

        def put(dst: torch.Tensor, name: str):
            if name in sd:
                used.add(name)
                dst.copy_(sd[name].to(dst.dtype))
            else:
                missing.append(name)

        tr = self.transformer
        put(tr.wte[:V], "transformer.wte.weight")
        put(tr.wpe, "transformer.wpe.weight")
        for i, blk in enumerate(tr.h):
            b = f"transformer.h.{i}."
            a = blk.attn.attention
            put(blk.ln_1.weight, b + "ln_1.weight"), put(blk.ln_1.bias, b + "ln_1.bias")
            put(a.qkv_proj[:H], b + "attn.attention.q_proj.weight")
            put(a.qkv_proj[H:2 * H], b + "attn.attention.k_proj.weight")
            put(a.qkv_proj[2 * H:], b + "attn.attention.v_proj.weight")
            put(a.out_proj.weight, b + "attn.attention.out_proj.weight"), put(a.out_proj.bias, b + "attn.attention.out_proj.bias")
            put(blk.ln_2.weight, b + "ln_2.weight"), put(blk.ln_2.bias, b + "ln_2.bias")
            put(blk.mlp.c_fc.weight, b + "mlp.c_fc.weight"), put(blk.mlp.c_fc.bias, b + "mlp.c_fc.bias")
            put(blk.mlp.c_proj.weight, b + "mlp.c_proj.weight"), put(blk.mlp.c_proj.bias, b + "mlp.c_proj.bias")
        put(tr.ln_f.weight, "transformer.ln_f.weight"), put(tr.ln_f.bias, "transformer.ln_f.bias")
        if self.lm_head is not None:
            put(self.lm_head[:V], "lm_head.weight")
        elif "lm_head.weight" in sd:
            used.add("lm_head.weight")
        unexpected = [k for k in sd if k not in used]
        if strict and (missing or unexpected):
            raise RuntimeError(f"load_state_dict: missing={missing[:5]} unexpected={unexpected[:5]}")
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)
