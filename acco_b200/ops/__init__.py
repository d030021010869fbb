"""Hot ops.  Every op has two implementations with identical semantics:

* a hand-written **sm_90a CUDA kernel** (``acco_b200/csrc/*.cu``, built in-tree into
  ``acco_b200/_C.so`` by ``__graft_entry__.build()``) - the path that runs on an H100;
* a plain **PyTorch fp32 reference** (``*_ref`` functions) - the CPU path and the numerics oracle
  used by ``tests/``.

On a CUDA tensor the kernel path is mandatory: if the extension is missing the op raises
instead of silently falling back (set ``ACCO_ALLOW_FALLBACK=1`` to permit the eager fallback,
e.g. when bisecting a kernel bug).
"""
from __future__ import annotations

import glob
import importlib.util
import os
import threading
from typing import Dict, Optional

import torch

_EXT = None
_EXT_ERR: Optional[BaseException] = None
_LOCK = threading.Lock()
_PKG_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# launch accounting for bench.py's ``gpu_launches`` (our own kernels only)
_launch_counts: Dict[str, int] = {}
_counting = True


def count_launch(name: str, n: int = 1) -> None:
    if _counting:
        _launch_counts[name] = _launch_counts.get(name, 0) + n


def launch_counts() -> Dict[str, int]:
    return dict(_launch_counts)


def reset_launch_counts() -> None:
    _launch_counts.clear()


def total_launches() -> int:
    return sum(_launch_counts.values())


def ext_path() -> Optional[str]:
    cands = sorted(glob.glob(os.path.join(_PKG_DIR, "_C*.so")))
    return cands[-1] if cands else None


def load_ext(required: bool = False):
    """Import the in-tree extension module (``acco_b200/_C*.so``)."""
    global _EXT, _EXT_ERR
    if _EXT is not None:
        return _EXT
    with _LOCK:
        if _EXT is not None:
            return _EXT
        path = ext_path()
        if path is None:
            _EXT_ERR = FileNotFoundError(
                f"acco_b200/_C*.so not found under {_PKG_DIR}; run `python -c 'import __graft_entry__ as g; g.build()'`")
        else:
            try:
                spec = importlib.util.spec_from_file_location("acco_b200._C", path)
                mod = importlib.util.module_from_spec(spec)
                spec.loader.exec_module(mod)
                _EXT = mod
                _EXT_ERR = None
            except BaseException as e:  # pragma: no cover
                _EXT_ERR = e
        if _EXT is None and required:
            raise RuntimeError(f"acco_b200 CUDA extension unavailable: {_EXT_ERR}")
        return _EXT


def have_ext() -> bool:
    return load_ext() is not None


def use_kernels(*tensors: torch.Tensor, bf16_only: bool = True) -> bool:
    """True -> dispatch to the sm_90a kernels.  CUDA tensors without the extension are an
    error unless ``ACCO_ALLOW_FALLBACK=1``.  The activation kernels are bf16-only: fp32 CUDA
    tensors (``use_mixed_precision=False`` / fp32 DDP weights, not a hot configuration) take the
    PyTorch path."""
    if not tensors or not all(t.is_cuda for t in tensors if t is not None):
        return False
    if bf16_only and any(t.is_floating_point() and t.dtype != torch.bfloat16 for t in tensors if t is not None):
        return False
    if os.environ.get("ACCO_FORCE_EAGER") == "1":
        return False
    if load_ext() is not None:
        return True
    if os.environ.get("ACCO_ALLOW_FALLBACK") == "1":
        return False
    raise RuntimeError(
        "acco_b200: CUDA tensors given but the sm_90a extension is not built/loaded "
        f"({_EXT_ERR}). Build it with __graft_entry__.build() or set ACCO_ALLOW_FALLBACK=1.")


from .norm import rmsnorm, add_rmsnorm, rmsnorm_ref, add_rmsnorm_ref  # noqa: E402
from .layernorm import layernorm, add_layernorm, gelu_new, layernorm_ref, add_layernorm_ref, gelu_new_ref  # noqa: E402
from .rope import rope_qkv, rope_qkv_ref, apply_rope_ref, rope_tables  # noqa: E402
from .embedding import embedding  # noqa: E402
from .swiglu import swiglu, swiglu_ref  # noqa: E402
from .cross_entropy import softmax_cross_entropy, softmax_cross_entropy_ref  # noqa: E402
from .linear import linear, LinearFn  # noqa: E402
from .attention import causal_attention, causal_attention_ref, rope_causal_attention, packed_causal_attention  # noqa: E402
from .adam import fused_adamw_shard  # noqa: E402

__all__ = [
    "load_ext", "have_ext", "use_kernels", "ext_path",
    "count_launch", "launch_counts", "reset_launch_counts", "total_launches",
    "rmsnorm", "add_rmsnorm", "rmsnorm_ref", "add_rmsnorm_ref",
    "layernorm", "add_layernorm", "gelu_new", "layernorm_ref", "add_layernorm_ref", "gelu_new_ref",
    "rope_qkv", "rope_qkv_ref", "apply_rope_ref", "rope_tables", "embedding",
    "swiglu", "swiglu_ref",
    "softmax_cross_entropy", "softmax_cross_entropy_ref",
    "linear", "LinearFn",
    "causal_attention", "causal_attention_ref", "rope_causal_attention", "packed_causal_attention",
    "fused_adamw_shard",
]
