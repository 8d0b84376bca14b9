"""A small Hydra-compatible config loader for the slamkit CLI surface (SURVEY.md §5, §8 b-3).

`hydra-core` / `omegaconf` are not dependencies of this package, and the hot paths must not depend on them, so this module
re-implements the subset of Hydra 1.3 semantics that the reference's `config/` tree and README one-liners use:
`defaults:` lists (group selection, nested `/group: name`, `override /group: name`, `_self_`), the
`# @package _global_` directive, `group=name` and dotted `key=value` / `+key=value` command-line overrides, `???`
mandatory values, and attribute-style access to the composed tree (`cfg.tokeniser.params.dedup`).
"""
from __future__ import annotations

import os
import re
from typing import Any, Dict, List, Optional

import yaml

MISSING = "???"


class Cfg(dict):
    """dict with attribute access and `.get`, enough of DictConfig for the CLI code."""

    def __getattr__(self, k):
        try:
            v = self[k]
        except KeyError as e:
            raise AttributeError(k) from e
        if v == MISSING:
            raise ValueError(f"Missing mandatory value: {k}")
        return v

    def __setattr__(self, k, v):
        self[k] = v


_FLOAT_RE = re.compile(r"^[+-]?(\d+\.?\d*|\.\d+)[eE][+-]?\d+$")


def _wrap(x):
    if isinstance(x, str) and _FLOAT_RE.match(x):      # PyYAML reads `1e-3` as a string; Hydra/OmegaConf as a float
        return float(x)
    if isinstance(x, dict):
        return Cfg({k: _wrap(v) for k, v in x.items()})
    if isinstance(x, list):
        return [_wrap(v) for v in x]
    return x


def _merge(dst: dict, src: dict) -> dict:
    for k, v in src.items():
        if isinstance(v, dict) and isinstance(dst.get(k), dict):
            _merge(dst[k], v)
        else:
            dst[k] = v
    return dst


def _set_path(tree: dict, dotted: str, value, create: bool) -> None:
    keys = dotted.split(".")
    cur = tree
    for k in keys[:-1]:
        if k not in cur or not isinstance(cur[k], dict):
            if not create and k not in cur:
                raise KeyError(f"Could not override '{dotted}': key '{k}' not in config (use +{dotted}=... to add)")
            cur[k] = {} if not isinstance(cur.get(k), dict) else cur[k]
        cur = cur[k]
    if not create and keys[-1] not in cur:
        raise KeyError(f"Could not override '{dotted}': no such key (use +{dotted}=... to add)")
    cur[keys[-1]] = value


class _Loader:
    def __init__(self, root: str):
        self.root = root

    def read(self, rel: str):
        path = os.path.join(self.root, rel + ".yaml")
        if not os.path.exists(path):
            raise FileNotFoundError(f"config '{rel}' not found under {self.root}")
        text = open(path).read()
        is_global = any(l.strip().replace(" ", "") == "#@package_global_" for l in text.splitlines()[:5])
        return yaml.safe_load(text) or {}, is_global

    def compose(self, rel: str, package: List[str], choices: Dict[str, str]) -> dict:
        """Compose file `rel` (e.g. 'tokeniser/unit_hubert_25'); its content lands under `package` unless the file
        carries `# @package _global_`."""
        body, is_global = self.read(rel)
        defaults = body.pop("defaults", [])
        group_dir = os.path.dirname(rel)
        out: dict = {}
        seen_self = False

        def place(tree: dict, pkg: List[str]) -> dict:
            for k in reversed(pkg):
                tree = {k: tree}
            return tree

        own_pkg = [] if is_global else package
        for d in defaults:
            if d == "_self_":
                _merge(out, place(body, own_pkg))
                seen_self = True
                continue
            if isinstance(d, str):                      # sibling file in the same group
                _merge(out, self.compose(os.path.join(group_dir, d) if group_dir else d, package, choices))
                continue
            (k, v), = d.items()
            k = k.replace("override ", "").strip()
            absolute = k.startswith("/")
            grp = k.lstrip("/")
            grp_path = grp if absolute else (os.path.join(group_dir, grp) if group_dir else grp)
            choice = choices.get(grp_path, v)
            if choice is None:
                continue
            choices.setdefault(grp_path, choice)
            _merge(out, self.compose(os.path.join(grp_path, choice), grp_path.split("/"), choices))
        if not seen_self:
            _merge(out, place(body, own_pkg))
        return out


def _pre_scan_overrides(loader: _Loader, rel: str, choices: Dict[str, str], cli: Dict[str, str]) -> None:
    """`override /group: name` entries anywhere in the defaults tree win over the primary defaults list."""
    body, _ = loader.read(rel)
    group_dir = os.path.dirname(rel)
    for d in body.get("defaults", []):
        if isinstance(d, str):
            if d != "_self_":
                _pre_scan_overrides(loader, os.path.join(group_dir, d) if group_dir else d, choices, cli)
            continue
        (k, v), = d.items()
        is_override = k.startswith("override ")
        k = k.replace("override ", "").strip()
        grp = k.lstrip("/")
        grp_path = grp if k.startswith("/") else (os.path.join(group_dir, grp) if group_dir else grp)
        if is_override:
            choices[grp_path] = v
        pick = cli.get(grp_path, choices.get(grp_path, v))
        if pick is not None:
            _pre_scan_overrides(loader, os.path.join(grp_path, pick), choices, cli)


def load_config(config_name: str, overrides: Optional[List[str]] = None, config_dir: Optional[str] = None) -> Cfg:
    config_dir = config_dir or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "config")
    loader = _Loader(config_dir)
    overrides = list(overrides or [])
    choices: Dict[str, str] = {}
    value_overrides = []
    for ov in overrides:
        if "=" not in ov:
            raise ValueError(f"bad override '{ov}' (expected key=value)")
        k, v = ov.split("=", 1)
        add = k.startswith("+")
        k = k.lstrip("+")
        if not add and "." not in k and os.path.isdir(os.path.join(config_dir, k)):
            choices[k] = v                               # config-group selection, e.g. tokeniser=unit_hubert_25
        else:
            value_overrides.append((k, yaml.safe_load(v), add))
    scan: Dict[str, str] = {}
    _pre_scan_overrides(loader, config_name, scan, choices)
    for k, v in scan.items():
        choices.setdefault(k, v)
    tree = loader.compose(config_name, [], choices)
    for k, v, add in value_overrides:
        _set_path(tree, k, v, create=add)
    return _wrap(tree)


def require(cfg: Cfg, *dotted: str) -> None:
    """Raise like Hydra does when a `???` value was not supplied."""
    for d in dotted:
        cur: Any = cfg
        for k in d.split("."):
            cur = cur[k]
        if cur == MISSING:
            raise ValueError(f"Missing mandatory value: {d}")


def to_container(cfg) -> Any:
    if isinstance(cfg, dict):
        return {k: to_container(v) for k, v in cfg.items()}
    if isinstance(cfg, list):
        return [to_container(v) for v in cfg]
    return cfg
