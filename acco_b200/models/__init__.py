"""Model families: native Llama (RMSNorm/RoPE/GQA/SwiGLU) and GPT-2 / GPT-Neo (LayerNorm/learned
positions/global+local attention), both callable HF-style (``model(**inputs, labels=...)[0]`` is
the loss) and both loading/saving HF checkpoint key names.  Any other HF-style ``nn.Module`` can
be handed to :class:`~acco_b200.trainer.DecoupledTrainer` as well."""
from __future__ import annotations

import json
import os
from typing import Any, Mapping

from .base import NativeCausalLM, NativeConfig
from .gpt import GPTConfig, GPTForCausalLM
from .llama import LlamaConfig, LlamaForCausalLM
from .output import CausalLMOutput

__all__ = ["NativeConfig", "NativeCausalLM", "LlamaConfig", "LlamaForCausalLM", "GPTConfig", "GPTForCausalLM", "CausalLMOutput",
           "build_model", "PRESETS", "preset", "from_pretrained", "load_hf_state_dict"]

PRESETS = {
    # name: (arch, kwargs)          parameter counts: logical (un-padded vocab)
    "llama125m": ("llama", dict(vocab_size=50257, hidden_size=768, intermediate_size=2048, num_hidden_layers=12,
                                num_attention_heads=12, num_key_value_heads=12, max_position_embeddings=1024,
                                rope_theta=10000.0, tie_word_embeddings=True)),
    "llama3-1b": ("llama", dict(vocab_size=128256, hidden_size=2048, intermediate_size=8192, num_hidden_layers=16,
                                num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=8192,
                                rope_theta=500000.0, tie_word_embeddings=True)),
    "llama3-8b": ("llama", dict(vocab_size=128256, hidden_size=4096, intermediate_size=14336, num_hidden_layers=32,
                                num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=8192,
                                rope_theta=500000.0, tie_word_embeddings=False)),
    "gpt2-small": ("gpt2", dict(vocab_size=50257, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                                max_position_embeddings=1024, attention_layers="global")),
    "gptneo": ("gptneo", dict(vocab_size=50257, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                              max_position_embeddings=1024, attention_layers="alternating", window_size=256)),
    "tiny": ("llama", dict(vocab_size=512, hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                           num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=128)),
}


def preset(name: str, device=None, dtype=None):
    arch, kw = PRESETS[name]
    return build_model(dict(arch=arch, **kw), device=device, dtype=dtype)


def build_model(model_cfg: Mapping[str, Any], config_root: str = None, device=None, dtype=None):
    """Instantiate a randomly initialised model from a ``config/model/*.yaml`` mapping.

    ``arch: llama | gpt2 | gptneo``.  For ``gptneo`` a ``config_path`` pointing at an HF json
    (reference layout, `config/model/gptneo.yaml`) is honoured when the file exists.
    ``device`` / ``dtype``: construct *and initialise* the parameters there (an 8B model is 32 GB of fp32 on the
    host otherwise - per rank)."""
    if device is not None or dtype is not None:
        import torch
        old = torch.get_default_dtype()
        try:
            if dtype is not None:
                torch.set_default_dtype(dtype)
            if device is not None:
                with torch.device(device):
                    return build_model(model_cfg, config_root)
            return build_model(model_cfg, config_root)
        finally:
            torch.set_default_dtype(old)
    cfg = dict(model_cfg)
    arch = str(cfg.get("arch", "llama")).lower()
    if arch == "llama":
        return LlamaForCausalLM(LlamaConfig.from_dict(cfg))
    if arch in ("gpt2", "gptneo", "gpt_neo"):
        path = cfg.get("config_path")
        if path and config_root:
            full = os.path.join(config_root, str(path).lstrip("/"))
            if os.path.isfile(full):
                with open(full) as f:
                    js = json.load(f)
                js.update({k: v for k, v in cfg.items() if k in ("attention_layers",) and not isinstance(v, str)})
                cfg = {**js, **{k: v for k, v in cfg.items() if k not in js and k != "attention_layers"}}
        cfg.setdefault("scale_attn", arch == "gpt2")
        if arch == "gpt2":
            cfg["attention_layers"] = "global"
        return GPTForCausalLM(GPTConfig.from_dict(cfg))
    raise ValueError(f"unknown model arch {arch!r}")


# ----------------------------------------------------------------------------------------------
# Pretrained checkpoints (`/root/reference/main.py:33-35`: ``AutoModelForCausalLM.from_pretrained(config_path)`` when finetuning)
# ----------------------------------------------------------------------------------------------
def load_hf_state_dict(path: str) -> Mapping[str, Any]:
    """Tensors of an HF checkpoint directory (``*.safetensors`` shards, ``pytorch_model*.bin``) or of a single ``.pt/.bin/.safetensors``
    file, as one flat ``{name: tensor}`` mapping on the CPU."""
    import glob

    import torch
    files = [path] if os.path.isfile(path) else (sorted(glob.glob(os.path.join(path, "*.safetensors")))
                                                 or sorted(glob.glob(os.path.join(path, "pytorch_model*.bin")))
                                                 or sorted(glob.glob(os.path.join(path, "*.pt"))))
    if not files:
        raise FileNotFoundError(f"no *.safetensors / pytorch_model*.bin / *.pt under {path!r}")
    sd = {}
    for f in files:
        if f.endswith(".safetensors"):
            from safetensors.torch import load_file
            sd.update(load_file(f, device="cpu"))
        else:
            sd.update(torch.load(f, map_location="cpu"))
    return sd


def _native_config_from_hf(hf: Mapping[str, Any]):
    """HF ``config.json`` -> native model config, or None when the architecture has no native implementation."""
    mt = str(hf.get("model_type", "")).lower()
    if mt == "llama" and not hf.get("attention_bias", False) and not hf.get("mlp_bias", False) \
            and hf.get("head_dim") in (None, int(hf["hidden_size"]) // int(hf["num_attention_heads"])):
        rs = hf.get("rope_scaling") or None
        if rs is not None and str(rs.get("rope_type", rs.get("type", "default"))) not in ("default", "llama3", "linear"):
            return None
        return LlamaConfig.from_dict({**hf, "rope_scaling": rs, "rope_theta": hf.get("rope_theta", 10000.0)})
    if mt == "gpt_neo":
        cfg = GPTConfig.from_dict({**hf, "scale_attn": False})
        return cfg if str(hf.get("activation_function", "gelu_new")) == "gelu_new" else None
    return None


def from_pretrained(path: str, device=None, dtype=None, native: bool = True):
    """Load a pretrained causal LM for finetuning.

    ``path``: an HF checkpoint directory (``config.json`` + safetensors / bin shards).  Llama-family and GPT-Neo checkpoints are
    loaded into the *native* models (kernel path; same key names, so ``load_state_dict`` takes the HF tensors as they are); any other
    architecture - or ``native=False`` - goes through ``transformers.AutoModelForCausalLM.from_pretrained`` exactly like the
    reference, and the trainer drives that ``nn.Module`` through its generic (eager / CUDA-graph) path.  A hub id works too when
    the files are in the local HF cache (there is no network on the training nodes)."""
    cfg_file = os.path.join(path, "config.json")
    if native and os.path.isfile(cfg_file):
        with open(cfg_file) as f:
            hf = json.load(f)
        cfg = _native_config_from_hf(hf)
        if cfg is not None:
            arch = "llama" if isinstance(cfg, LlamaConfig) else "gptneo"
            model = build_model({"arch": arch, **cfg.to_dict()}, device=device, dtype=dtype)
            missing, unexpected = model.load_state_dict(load_hf_state_dict(path), strict=False)
            missing = [k for k in missing if not k.endswith("lm_head.weight")]
            if missing:
                raise RuntimeError(f"checkpoint {path!r} lacks {missing[:5]} ...")
            return model
    from transformers import AutoModelForCausalLM
    model = AutoModelForCausalLM.from_pretrained(path, torch_dtype=dtype)
    return model.to(device) if device is not None else model
