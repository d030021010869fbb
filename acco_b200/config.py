"""Hydra-compatible config composition without Hydra.

The reference composes ``config/config.yaml`` + one file from each of the groups
``data/ train/ model/`` with Hydra (`main.py:25`, `config/config.yaml:2-5`) and passes
``cfg.train`` whole as the trainer's ``args`` (`main.py:60`).  Hydra/omegaconf are not
installed on the (offline) GPU image, so this module re-implements the subset that the
reference relies on, on top of PyYAML:

* ``defaults:`` list of ``{group: option}`` entries -> ``<config_dir>/<group>/<option>.yaml``
  mounted at key ``group``;
* command-line overrides ``group=option`` (re-select a group file), ``a.b.c=value`` (set a
  leaf, YAML-typed), ``+a.b=value`` (add a new key), ``~a.b`` (delete);
* ``${now:%Y-%m-%d}`` and ``${a.b}`` interpolation;
* attribute access on the result (:class:`AttrDict`), ``to_container`` for CSV logging
  (replaces ``OmegaConf.to_container`` used at `trainer_decoupled.py:582`).
"""
from __future__ import annotations

import copy
import datetime as _dt
import os
import re
from typing import Any, Dict, Iterable, List, Mapping, Optional

import yaml

__all__ = ["AttrDict", "compose", "to_container", "load_yaml", "apply_overrides", "default_config_dir"]


class AttrDict(dict):
    """dict with attribute access, recursively applied.  ``args.batch_size`` works like a
    Hydra ``DictConfig`` for every access pattern in the reference trainer."""

    def __init__(self, *a, **kw):
        super().__init__()
        for k, v in dict(*a, **kw).items():
            self[k] = v

    @staticmethod
    def _wrap(v):
        if isinstance(v, Mapping) and not isinstance(v, AttrDict):
            return AttrDict(v)
        if isinstance(v, list):
            return [AttrDict._wrap(x) for x in v]
        return v

    def __setitem__(self, k, v):
        super().__setitem__(k, AttrDict._wrap(v))

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:  # pragma: no cover - message path
            raise AttributeError(f"config has no key {k!r}") from e

    def __setattr__(self, k, v):
        self[k] = v

    def __delattr__(self, k):
        del self[k]

    def get(self, k, default=None):
        return self[k] if k in self else default

    def copy(self):
        return AttrDict(copy.deepcopy(dict(self)))

    def __deepcopy__(self, memo):
        return AttrDict({k: copy.deepcopy(v, memo) for k, v in self.items()})


def to_container(cfg: Any, resolve: bool = True) -> Any:
    """Plain ``dict``/``list`` copy of a config (stand-in for ``OmegaConf.to_container``).

    Also accepts ``argparse.Namespace``-like objects so results logging works with any
    ``args`` a user hands to :class:`~acco_b200.trainer.DecoupledTrainer`."""
    if isinstance(cfg, Mapping):
        return {k: to_container(v) for k, v in cfg.items()}
    if isinstance(cfg, (list, tuple)):
        return [to_container(v) for v in cfg]
    if hasattr(cfg, "__dict__") and not isinstance(cfg, type):
        return {k: to_container(v) for k, v in vars(cfg).items() if not k.startswith("_")}
    return cfg


def default_config_dir() -> str:
    here = os.path.dirname(os.path.abspath(__file__))
    return os.path.join(os.path.dirname(here), "config")


def load_yaml(path: str) -> Dict[str, Any]:
    with open(path, "r") as f:
        data = yaml.safe_load(f)
    return data or {}


def _parse_value(text: str) -> Any:
    """YAML-typed scalar parsing, with the float forms PyYAML misses (``6e-4``) and WITHOUT the YAML-1.1 surprises Hydra's override
    grammar does not have: ``12:30`` is a string (not the base-60 integer 750), ``010`` is 10 (not octal 8), ``1_000`` stays text."""
    t = text.strip()
    if re.fullmatch(r"[+-]?\d+(:\d+)+", t) or re.fullmatch(r"[+-]?\d+(_\d+)+", t):
        return text
    if re.fullmatch(r"[+-]?0\d+", t):
        return int(t, 10)
    try:
        v = yaml.safe_load(text)
    except yaml.YAMLError:
        return text
    if isinstance(v, str):
        if re.fullmatch(r"[+-]?(\d+\.?\d*|\.\d+)([eE][+-]?\d+)?", v):
            try:
                return float(v)
            except ValueError:
                pass
    return v


def _fix_scalars(node: Any) -> Any:
    """PyYAML (YAML 1.1) reads ``6e-4`` as a string; Hydra/OmegaConf read a float."""
    if isinstance(node, dict):
        return {k: _fix_scalars(v) for k, v in node.items()}
    if isinstance(node, list):
        return [_fix_scalars(v) for v in node]
    if isinstance(node, str) and re.fullmatch(r"[+-]?(\d+\.?\d*|\.\d+)[eE][+-]?\d+", node.strip()):
        return float(node)
    return node


def _set_path(cfg: Dict[str, Any], dotted: str, value: Any, create: bool) -> None:
    keys = dotted.split(".")
    node = cfg
    for k in keys[:-1]:
        if k not in node or not isinstance(node[k], dict):
            if not create:
                raise KeyError(f"override {dotted!r}: no such config node {k!r} (use +{dotted}=... to add)")
            node[k] = {}
        node = node[k]
    if keys[-1] not in node and not create:
        raise KeyError(f"override {dotted!r}: key does not exist (use +{dotted}=... to add)")
    node[keys[-1]] = value


def _del_path(cfg: Dict[str, Any], dotted: str) -> None:
    keys = dotted.split(".")
    node = cfg
    for k in keys[:-1]:
        node = node[k]
    node.pop(keys[-1], None)


def _get_path(cfg: Mapping, dotted: str) -> Any:
    node: Any = cfg
    for k in dotted.split("."):
        node = node[k]
    return node


_INTERP = re.compile(r"\$\{([^${}]+)\}")


def _resolve(node: Any, root: Mapping, now: _dt.datetime) -> Any:
    if isinstance(node, dict):
        return {k: _resolve(v, root, now) for k, v in node.items()}
    if isinstance(node, list):
        return [_resolve(v, root, now) for v in node]
    if not isinstance(node, str) or "${" not in node:
        return node

    def sub(m: "re.Match[str]") -> str:
        expr = m.group(1).strip()
        if expr.startswith("now:"):
            return now.strftime(expr[4:])
        if expr.startswith("oc.env:") or expr.startswith("env:"):
            name, _, dflt = expr.split(":", 1)[1].partition(",")
            return os.environ.get(name.strip(), dflt.strip())
        return str(_get_path(root, expr))

    whole = _INTERP.fullmatch(node)
    if whole and not whole.group(1).startswith(("now:", "oc.env:", "env:")):
        return _get_path(root, whole.group(1).strip())  # keep the referenced type
    return _INTERP.sub(sub, node)


def apply_overrides(cfg: Dict[str, Any], overrides: Iterable[str], groups: Mapping[str, str], config_dir: str) -> Dict[str, str]:
    """Apply Hydra-style overrides in place; returns the final ``group -> option`` map."""
    chosen = dict(groups)
    deferred: List[str] = []
    for ov in overrides:
        if "=" in ov and not ov.startswith(("+", "~")):
            key, _, val = ov.partition("=")
            if "." not in key and os.path.isdir(os.path.join(config_dir, key)):
                chosen[key] = val
                continue
        deferred.append(ov)
    for group, option in chosen.items():
        path = os.path.join(config_dir, group, f"{option}.yaml")
        if not os.path.exists(path):
            avail = sorted(os.path.splitext(f)[0] for f in os.listdir(os.path.join(config_dir, group)) if f.endswith(".yaml"))
            raise FileNotFoundError(f"config group {group!r} has no option {option!r}; available: {avail}")
        cfg[group] = _fix_scalars(load_yaml(path))
    for ov in deferred:
        if ov.startswith("~"):
            _del_path(cfg, ov[1:].split("=")[0])
            continue
        create = ov.startswith("+")
        key, sep, val = ov.lstrip("+").partition("=")
        if not sep:
            raise ValueError(f"bad override {ov!r}; expected key=value")
        _set_path(cfg, key, _parse_value(val), create)
    return chosen


def compose(
    config_dir: Optional[str] = None,
    config_name: str = "config.yaml",
    overrides: Optional[Iterable[str]] = None,
    now: Optional[_dt.datetime] = None,
) -> AttrDict:
    """Compose the root config: root yaml + ``defaults`` groups + CLI overrides.

    ``compose(overrides=["train=ddp", "model=llama125m", "train.batch_size=4"])`` mirrors
    ``python main.py train=ddp model=llama125m train.batch_size=4`` of the reference
    (`README.md:52-58`)."""
    config_dir = config_dir or default_config_dir()
    root = _fix_scalars(load_yaml(os.path.join(config_dir, config_name)))
    defaults = root.pop("defaults", []) or []
    groups: Dict[str, str] = {}
    for entry in defaults:
        if isinstance(entry, dict):
            for g, opt in entry.items():
                groups[str(g)] = str(opt)
        elif isinstance(entry, str) and entry != "_self_":
            groups[entry] = entry
    chosen = apply_overrides(root, list(overrides or []), groups, config_dir)
    root = _resolve(root, root, now or _dt.datetime.now())
    cfg = AttrDict(root)
    cfg["_groups_"] = chosen
    return cfg
