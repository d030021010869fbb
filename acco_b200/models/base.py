"""What the native Llama and GPT-Neo models share: config helpers, the training switches, initialisation, the loss tail and
the HF checkpoint format.

Each model describes its checkpoint once, as a table of ``(HF key, view of the live parameter)`` pairs (``_hf_tensors``);
``state_dict()`` and ``load_state_dict()`` both walk that table, so saving and loading cannot drift apart."""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import asdict
from typing import Any, Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from .. import ops
from .output import CausalLMOutput

__all__ = ["NativeConfig", "NativeCausalLM"]


class NativeConfig:
    """Mixin for the config dataclasses (``vocab_size``, ``hidden_size``, ``num_attention_heads``, ``pad_vocab_multiple``)."""

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
    def from_dict(cls, d: Dict[str, Any]):
        """Build from a mapping, ignoring keys that are not fields (HF ``config.json`` carries many)."""
        keys = cls.__dataclass_fields__.keys()
        return cls(**{k: v for k, v in dict(d).items() if k in keys})


class NativeCausalLM(nn.Module):
    """Base of the native causal LMs.  A subclass registers its parameters, including ``lm_head`` (``None`` when the head is
    tied to the input embedding), then calls :meth:`reset_parameters`.  It provides ``embed_weight``, ``_init_fill``,
    ``_hf_tensors`` and ``_hf_ignored_suffixes``.  This class registers no parameter, buffer or submodule."""

    _hf_ignored_suffixes: Tuple[str, ...] = ()      # checkpoint keys ending so are never reported as unexpected

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.fp8 = False             # FP8 GEMMs for the block linears of training micro-batches (train key `fp8`, ops/fp8.py)
        self.label_smoothing = 0.0   # label smoothing of the loss when labels are given (train key `label_smoothing_factor`)
        self.z_loss_weight = 0.0     # z * mean lse^2 added to the loss (train key `z_loss_weight`, ops/cross_entropy.py)
        self.z_loss_out: Optional[torch.Tensor] = None   # one fp32 on the device: receives the z-term of each loss computed
        # knowledge distillation (train key `distill_teacher`): the weight a and temperature T of a forward given teacher_logits,
        # and two fp32 on the device that receive each such loss's mean CE and mean KL (ops.distill_cross_entropy)
        self.distill_alpha = 0.5
        self.distill_temperature = 1.0
        self.distill_out: Optional[torch.Tensor] = None
        # DPO (train key `dpo_beta`): beta of a forward given reference_logits, and three fp32 on the device that receive each such
        # loss's mean chosen reward, mean rejected reward and accuracy (ops.dpo_loss)
        self.dpo_beta = 0.1
        self.dpo_out: Optional[torch.Tensor] = None
        # reference-free preference objectives (train keys `simpo_beta` / `simpo_gamma`, `orpo_lambda`): the one set (not None) is the
        # loss of a forward given preference_pairs=True; three fp32 on the device receive its logged means (ops.simpo_loss / orpo_loss)
        self.simpo_beta: Optional[float] = None
        self.simpo_gamma = 0.5
        self.orpo_lambda: Optional[float] = None
        self.pref_out: Optional[torch.Tensor] = None

    @property
    def embed_weight(self) -> torch.Tensor:
        raise NotImplementedError

    @property
    def head_weight(self) -> torch.Tensor:
        return self.embed_weight if self.lm_head is None else self.lm_head

    # ------------------------------------------------------------------ init
    def _init_fill(self, name: str) -> Optional[float]:
        """The constant parameter ``name`` starts at, or None to draw it from N(0, initializer_range)."""
        raise NotImplementedError

    @torch.no_grad()
    def reset_parameters(self) -> None:
        std = self.config.initializer_range
        for name, p in self.named_parameters():
            fill = self._init_fill(name)
            if fill is None:
                p.normal_(0.0, std)
            else:
                p.fill_(fill)
        # alignment padding rows of the vocabulary are exactly zero and stay zero
        V = self.config.vocab_size
        self.embed_weight[V:].zero_()
        if self.lm_head is not None:
            self.lm_head[V:].zero_()

    # ------------------------------------------------------------------ loss
    def _lm_output(self, logits: torch.Tensor, labels: Optional[torch.Tensor], B: int, S: int,
                   teacher_logits: Optional[torch.Tensor] = None, reference_logits: Optional[torch.Tensor] = None,
                   preference_pairs: bool = False) -> CausalLMOutput:
        """Logits ``[B*S, Vp]`` -> the logits cut to ``vocab_size`` without labels, else the mean cross-entropy loss, or with
        ``teacher_logits`` (a teacher's :meth:`padded_logits` on the same tokens) the distillation objective, over the same rows.
        With ``reference_logits`` (a frozen reference's :meth:`padded_logits`) the ``B = 2P`` rows are ``P`` preference pairs, chosen
        rows first, and the loss is the DPO objective over the response tokens the labels keep (``ops.dpo_loss``).  With
        ``preference_pairs=True`` the rows are laid out the same way and the loss is the reference-free objective set on the model:
        SimPO (``simpo_beta``, ``simpo_gamma``; ``ops.simpo_loss``) or ORPO (``orpo_lambda``; ``ops.orpo_loss``)."""
        V = self.config.vocab_size
        if labels is None:
            if teacher_logits is not None or reference_logits is not None or preference_pairs:
                raise ValueError("teacher_logits / reference_logits / preference_pairs need labels: the loss is taken over the rows the "
                                 "labels keep")
            return CausalLMOutput(loss=None, logits=logits.view(B, S, -1)[..., :V])
        if teacher_logits is not None and reference_logits is not None:
            raise ValueError("give teacher_logits (distillation) or reference_logits (DPO), not both")
        if preference_pairs and (teacher_logits is not None or reference_logits is not None):
            raise ValueError("preference_pairs (SimPO / ORPO) needs no frozen model: give it without teacher_logits / reference_logits")
        # HF shift: position t predicts token t+1; the last position has no target
        shifted = torch.full_like(labels, -100)
        shifted[:, :-1] = labels[:, 1:]
        if teacher_logits is not None:
            if self.label_smoothing or self.z_loss_weight:
                raise ValueError("distillation cannot be combined with label smoothing or the z-loss")
            loss = ops.distill_cross_entropy(logits, teacher_logits, shifted.reshape(B * S), V, self.distill_alpha,
                                             self.distill_temperature, out=self.distill_out)
            return CausalLMOutput(loss=loss, logits=None)
        if reference_logits is not None:
            if self.label_smoothing or self.z_loss_weight:
                raise ValueError("DPO cannot be combined with label smoothing or the z-loss")
            if B % 2:
                raise ValueError(f"DPO needs an even number of rows (P chosen, then P rejected), got {B}")
            loss = ops.dpo_loss(logits, reference_logits, shifted.reshape(B * S), B // 2, V, self.dpo_beta, out=self.dpo_out)
            return CausalLMOutput(loss=loss, logits=None)
        if preference_pairs:
            if self.label_smoothing or self.z_loss_weight:
                raise ValueError("SimPO / ORPO cannot be combined with label smoothing or the z-loss")
            if (self.simpo_beta is None) == (self.orpo_lambda is None):
                raise ValueError(f"preference_pairs needs exactly one objective set on the model: simpo_beta={self.simpo_beta!r}, "
                                 f"orpo_lambda={self.orpo_lambda!r}")
            if B % 2:
                raise ValueError(f"preference pairs need an even number of rows (P chosen, then P rejected), got {B}")
            if self.simpo_beta is not None:
                loss = ops.simpo_loss(logits, shifted.reshape(B * S), B // 2, V, self.simpo_beta, self.simpo_gamma, out=self.pref_out)
            else:
                loss = ops.orpo_loss(logits, shifted.reshape(B * S), B // 2, V, self.orpo_lambda, out=self.pref_out)
            return CausalLMOutput(loss=loss, logits=None)
        loss = ops.softmax_cross_entropy(logits, shifted.reshape(B * S), V, -100, label_smoothing=self.label_smoothing,
                                         z_loss=self.z_loss_weight, z_loss_out=self.z_loss_out)
        return CausalLMOutput(loss=loss, logits=None)

    def padded_logits(self, input_ids: torch.Tensor, position_ids: Optional[torch.Tensor] = None) -> torch.Tensor:
        raise NotImplementedError

    # ------------------------------------------------------------------ HF-compatible checkpoints
    def _hf_tensors(self) -> List[Tuple[str, torch.Tensor]]:
        """``(HF key, view of the live parameter)`` in checkpoint order, with HF shapes (fused weights split, vocabulary padding
        removed) and ``lm_head.weight`` last."""
        raise NotImplementedError

    def state_dict(self, *args, destination=None, prefix: str = "", keep_vars: bool = False, **kw):
        """HF key names and shapes.  The tensors are views of the live parameters (hence of the flat arena), like the
        reference's checkpoints (`trainer_decoupled.py:568-573`)."""
        sd = destination if destination is not None else OrderedDict()
        for key, t in self._hf_tensors():
            sd[prefix + key] = t if keep_vars else t.detach()
        return sd

    @torch.no_grad()
    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        """Copy an HF-keyed state dict into the parameters.  A tied head takes its weights from the embedding, so it neither
        needs nor reports ``lm_head.weight``."""
        sd = dict(state_dict)
        used, missing = set(), []
        for key, dst in self._hf_tensors():
            if key == "lm_head.weight" and self.lm_head is None:
                used.add(key)
            elif key in sd:
                used.add(key)
                dst.copy_(sd[key].to(dst.dtype))
            else:
                missing.append(key)
        unexpected = [k for k in sd if k not in used and not k.endswith(self._hf_ignored_suffixes)]
        if strict and (missing or unexpected):
            raise RuntimeError(f"load_state_dict: missing={missing[:5]} unexpected={unexpected[:5]}")
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)
