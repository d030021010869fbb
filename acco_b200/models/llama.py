"""Native Llama-family causal LM (RMSNorm, RoPE, GQA, SwiGLU, tied or untied head).

Role in the reference: the model is "whatever HF returns" (`main.py:33-41`; Llama-3 for the
finetuning configs, `README.md:76-82`), called as ``model(**inputs, labels=input_ids)`` with
``outputs[0]`` the loss (`trainer_decoupled.py:28-34`).  This implementation keeps that calling
convention and the HF **checkpoint key names** (``model.layers.N.self_attn.q_proj.weight`` ...),
but is laid out for the GPU kernel path:

* activations are ``[T = B*S, H]`` row-major bf16 throughout; QKV and gate|up are single fused
  GEMMs (one weight each in the flat arena; split back to HF names only in ``state_dict()``);
* the LM head / embedding is padded to a multiple of 128 rows so the logits GEMM has aligned
  leading dimensions (50257 -> 50304); padded columns are masked inside the fused CE kernel;
* residual add + RMSNorm, RoPE (in place on the QKV buffer), SwiGLU and the softmax-CE are
  single hand-written sm_90a kernels (``acco_b200/ops``); wgrad GEMMs accumulate directly into
  the flat gradient arena.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from .. import ops
from .base import NativeCausalLM, NativeConfig
from .output import CausalLMOutput

__all__ = ["LlamaConfig", "LlamaForCausalLM"]


@dataclass
class LlamaConfig(NativeConfig):
    vocab_size: int = 50257
    hidden_size: int = 768
    intermediate_size: int = 2048
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    num_key_value_heads: Optional[int] = None
    max_position_embeddings: int = 1024
    rms_norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    rope_scaling: Optional[Dict[str, Any]] = None       # HF dict (``rope_type: llama3`` for Llama-3.1 / 3.2 checkpoints)
    tie_word_embeddings: bool = True
    initializer_range: float = 0.02
    pad_vocab_multiple: int = 128
    model_type: str = "llama"

    def __post_init__(self):
        if self.num_key_value_heads is None:
            self.num_key_value_heads = self.num_attention_heads
        assert self.hidden_size % self.num_attention_heads == 0
        assert self.num_attention_heads % self.num_key_value_heads == 0

    def num_parameters(self, padded: bool = False) -> int:
        H, I, L = self.hidden_size, self.intermediate_size, self.num_hidden_layers
        D, Hq, Hk = self.head_dim, self.num_attention_heads, self.num_key_value_heads
        V = self.padded_vocab if padded else self.vocab_size
        per_layer = (Hq + 2 * Hk) * D * H + H * Hq * D + 3 * H * I + 2 * H
        n = V * H + L * per_layer + H
        if not self.tie_word_embeddings:
            n += V * H
        return n

    def flops_per_token(self, seq_len: int) -> float:
        """Training FLOPs per token (fwd+bwd = 3x fwd), matmuls + causal attention."""
        H, I, L = self.hidden_size, self.intermediate_size, self.num_hidden_layers
        D, Hq, Hk = self.head_dim, self.num_attention_heads, self.num_key_value_heads
        mm = L * ((Hq + 2 * Hk) * D * H + Hq * D * H + 3 * H * I) + self.vocab_size * H
        attn = L * 2 * Hq * D * seq_len / 2   # QK^T and PV, causal half
        return 3.0 * 2.0 * (mm + attn)


class _Norm(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim))


class _Attn(nn.Module):
    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        D, Hq, Hk, H = cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.hidden_size
        self.qkv_proj = nn.Parameter(torch.empty((Hq + 2 * Hk) * D, H))
        self.o_proj = nn.Parameter(torch.empty(H, Hq * D))


class _MLP(nn.Module):
    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        self.gate_up_proj = nn.Parameter(torch.empty(2 * cfg.intermediate_size, cfg.hidden_size))
        self.down_proj = nn.Parameter(torch.empty(cfg.hidden_size, cfg.intermediate_size))


class _Layer(nn.Module):
    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        self.input_layernorm = _Norm(cfg.hidden_size)
        self.self_attn = _Attn(cfg)
        self.post_attention_layernorm = _Norm(cfg.hidden_size)
        self.mlp = _MLP(cfg)


class _Body(nn.Module):
    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        self.embed_tokens = nn.Parameter(torch.empty(cfg.padded_vocab, cfg.hidden_size))
        self.layers = nn.ModuleList([_Layer(cfg) for _ in range(cfg.num_hidden_layers)])
        self.norm = _Norm(cfg.hidden_size)


class LlamaForCausalLM(NativeCausalLM):
    _hf_ignored_suffixes = ("rotary_emb.inv_freq",)

    def __init__(self, config: LlamaConfig):
        super().__init__(config)
        self.model = _Body(config)
        if config.tie_word_embeddings:
            self.lm_head = None
        else:
            self.lm_head = nn.Parameter(torch.empty(config.padded_vocab, config.hidden_size))
        self._rope_cache: Dict[Any, Any] = {}
        # fused all-gather + GEMM (KERNEL B): {id(param): [GatheredWeight for theta[0], theta[1]]}, set by the trainer
        self._ag_table: Dict[int, Any] = {}
        self._ag_idx = 0
        self._ag_pending = False
        self.reset_parameters()

    def _init_fill(self, name: str) -> Optional[float]:
        return 1.0 if name.endswith("norm.weight") else None

    @property
    def embed_weight(self) -> torch.Tensor:
        return self.model.embed_tokens

    def num_parameters(self) -> int:
        return sum(p.numel() for p in self.parameters())

    def _rope(self, S: int, device) -> Any:
        key = (S, str(device))
        if key not in self._rope_cache:
            self._rope_cache[key] = ops.rope_tables(S, self.config.head_dim, self.config.rope_theta, device, scaling=self.config.rope_scaling)
        return self._rope_cache[key]

    def fused_ag_candidates(self):
        """Weights whose first forward use is a GEMM (so their all-gather can be fused into it)."""
        out = []
        for layer in self.model.layers:
            out += [layer.self_attn.qkv_proj, layer.self_attn.o_proj, layer.mlp.gate_up_proj, layer.mlp.down_proj]
        if self.lm_head is not None:
            out.append(self.lm_head)
        return out

    def _gw(self, p):
        if not self._ag_pending:
            return None
        e = self._ag_table.get(id(p))
        return None if e is None else e[self._ag_idx]

    # ------------------------------------------------------------------ forward
    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                labels: Optional[torch.Tensor] = None, position_ids: Optional[torch.Tensor] = None,
                teacher_logits: Optional[torch.Tensor] = None, reference_logits: Optional[torch.Tensor] = None,
                preference_pairs: bool = False, **unused) -> CausalLMOutput:
        """HF-style call.  ``attention_mask`` is accepted for API compatibility; with right
        padding and causal attention the logits at non-pad positions do not depend on it, and pad
        positions carry ``labels == -100`` (the collator's job), so it is not applied.
        ``position_ids [B, S]`` marks packed rows (``PackedCollator``): positions restart at 0 for every sample, RoPE uses them
        and no token attends to another sample.
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
        D, Hq, Hk = cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads
        cos, sin = self._rope(S, input_ids.device)
        seg = None
        if position_ids is not None:
            pos = position_ids.reshape(T)
            cos, sin = cos[pos], sin[pos]                                                   # per-token tables [T, D/2]
            seg = ops.segment_starts(position_ids)
        eps = cfg.rms_norm_eps
        fp8 = self.fp8

        h = ops.embedding(input_ids.reshape(T), self.model.embed_tokens)                   # [T, H]
        branch = None          # output of the previous residual branch, not yet added to h
        for layer in self.model.layers:
            if branch is None:
                n = ops.rmsnorm(h, layer.input_layernorm.weight, eps)
            else:
                n, h = ops.add_rmsnorm(branch, h, layer.input_layernorm.weight, eps)
            qkv = ops.linear(n, layer.self_attn.qkv_proj, gathered=self._gw(layer.self_attn.qkv_proj), fp8=fp8)   # [T, (Hq+2Hk)D]
            att = ops.rope_causal_attention(qkv, cos, sin, B, S, Hq, Hk, D, seg=seg)       # [T, Hq*D]
            o = ops.linear(att, layer.self_attn.o_proj, gathered=self._gw(layer.self_attn.o_proj), fp8=fp8)
            n, h = ops.add_rmsnorm(o, h, layer.post_attention_layernorm.weight, eps)
            gu = ops.linear(n, layer.mlp.gate_up_proj, gathered=self._gw(layer.mlp.gate_up_proj), fp8=fp8)
            branch = ops.linear(ops.swiglu(gu), layer.mlp.down_proj, gathered=self._gw(layer.mlp.down_proj), fp8=fp8)
        if branch is None:
            n = ops.rmsnorm(h, self.model.norm.weight, eps)
        else:
            n, h = ops.add_rmsnorm(branch, h, self.model.norm.weight, eps)
        return ops.linear(n, self.head_weight, gathered=self._gw(self.head_weight) if self.lm_head is not None else None)   # [T, Vp]

    def _hf_tensors(self) -> List[Tuple[str, torch.Tensor]]:
        """HF ``LlamaForCausalLM`` keys: the fused QKV and gate|up weights are split back into HF's projections."""
        cfg = self.config
        D, Hq, Hk, V, I = cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.vocab_size, cfg.intermediate_size
        t = [("model.embed_tokens.weight", self.model.embed_tokens[:V])]
        for i, layer in enumerate(self.model.layers):
            b = f"model.layers.{i}."
            qkv, gu = layer.self_attn.qkv_proj, layer.mlp.gate_up_proj
            t += [(b + "self_attn.q_proj.weight", qkv[: Hq * D]),
                  (b + "self_attn.k_proj.weight", qkv[Hq * D: (Hq + Hk) * D]),
                  (b + "self_attn.v_proj.weight", qkv[(Hq + Hk) * D:]),
                  (b + "self_attn.o_proj.weight", layer.self_attn.o_proj),
                  (b + "mlp.gate_proj.weight", gu[:I]),
                  (b + "mlp.up_proj.weight", gu[I:]),
                  (b + "mlp.down_proj.weight", layer.mlp.down_proj),
                  (b + "input_layernorm.weight", layer.input_layernorm.weight),
                  (b + "post_attention_layernorm.weight", layer.post_attention_layernorm.weight)]
        t += [("model.norm.weight", self.model.norm.weight), ("lm_head.weight", self.head_weight[:V])]
        return t
