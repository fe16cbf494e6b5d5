"""Reading Demucs v3 / v4 model packages without the reference's Python classes.

A `.th` file is `torch.save({"klass": HTDemucs, "args": ..., "kwargs": {...}, "state": {...}, ...})`
(uvr_lib_v5/demucs/states.py:34-64); a bag is a YAML file listing signatures, per-source weights and a segment
(demucs/repo.py:120-137).  Only the data is needed here -- the class object is replaced by a named placeholder while unpickling.
"""
from __future__ import annotations

import os
import pickle
import types
from fractions import Fraction

import numpy as np
import torch
import yaml

from .demucs import HTDemucsConfig
from .demucs_v3 import DemucsConfig
from .hdemucs import HDemucsConfig

# constructor arguments that must keep the value the H100 graph was built for (htdemucs.py:36-98)
_REQUIRED = dict(cac=True, wiener_iters=0, end_iters=0, wiener_residual=False, rewrite=True, multi_freqs=None, context_enc=0, t_emb="sin", t_norm_in=True,
                 t_norm_in_group=False, t_group_norm=False, t_norm_first=True, t_norm_out=True, t_layer_scale=True, t_gelu=True, t_weight_pos_embed=1.0,
                 t_sparse_self_attn=False, t_sparse_cross_attn=False, t_cross_first=False, channels_time=None, use_train_segment=True)
_MAPPED = ("sources", "audio_channels", "channels", "growth", "nfft", "depth", "kernel_size", "stride", "context", "dconv_depth", "dconv_comp", "bottom_channels",
           "t_layers", "t_heads", "t_hidden_scale", "freq_emb", "emb_scale", "samplerate", "segment")


# HDemucs (v3) constructor arguments (hdemucs.py:360-400): values the H100 graph is built for, and the ones that map onto HDemucsConfig
_HD_REQUIRED = dict(cac=True, wiener_iters=0, end_iters=0, wiener_residual=False, rewrite=True, hybrid=True, channels_time=None)
_HD_MAPPED = ("sources", "audio_channels", "channels", "growth", "nfft", "depth", "hybrid_old", "freq_emb", "emb_scale", "kernel_size", "time_stride", "stride", "context",
              "context_enc", "norm_starts", "norm_groups", "dconv_mode", "dconv_depth", "dconv_comp", "dconv_attn", "dconv_lstm", "samplerate", "segment")


# Demucs (v3 time-domain) constructor arguments (demucs.py:236-272): values the H100 graph is built for, and the ones that map onto DemucsConfig
_V3_REQUIRED = dict(glu=True, gelu=True, rewrite=True, normalize=True, resample=True)
_V3_MAPPED = ("sources", "audio_channels", "channels", "growth", "depth", "kernel_size", "stride", "context", "norm_starts", "norm_groups", "dconv_mode",
              "dconv_depth", "dconv_comp", "dconv_attn", "dconv_lstm", "samplerate", "segment")


class _Placeholder:
    """Stands in for a class the package pickled by reference (e.g. demucs.htdemucs.HTDemucs)."""


# Globals a Demucs package legitimately pickles: tensor rebuild helpers / storages, plain containers, Fraction, numpy scalars and omegaconf containers (the
# training config some packages carry).  EVERYTHING else -- first of all the model class itself -- becomes an inert placeholder instead of being imported:
# a crafted .th cannot name an arbitrary callable (the reference's plain torch.load would execute it).
_ALLOWED_MODULES = ("torch._utils", "torch.storage", "torch._tensor", "torch.serialization", "collections", "fractions", "numpy", "numpy.core.multiarray", "numpy._core.multiarray",
                    "numpy.core.numeric", "numpy._core.numeric", "omegaconf.dictconfig", "omegaconf.listconfig", "omegaconf.base", "omegaconf.nodes", "builtins")
_ALLOWED_BUILTINS = {"set", "frozenset", "dict", "list", "tuple", "int", "float", "bool", "str", "bytes", "bytearray", "complex", "slice", "range", "object"}


class _TolerantUnpickler(pickle.Unpickler):
    def find_class(self, module, name):
        allowed = module in _ALLOWED_MODULES or (module == "torch" and (name.endswith("Storage") or name in ("Size", "device", "dtype", "Tensor") or name.startswith(("float", "int", "uint", "bfloat", "bool", "half", "double", "long", "short", "complex"))))
        if module == "builtins" and name not in _ALLOWED_BUILTINS:
            allowed = False
        if allowed:
            try:
                return super().find_class(module, name)
            except (ImportError, AttributeError):
                pass
        return type(name, (_Placeholder,), {"__module__": module})


_pickle_shim = types.ModuleType("b200sep_tolerant_pickle")
_pickle_shim.Unpickler = _TolerantUnpickler
_pickle_shim.load = lambda f, **kw: _TolerantUnpickler(f, **kw).load()
_pickle_shim.__dict__.update({k: getattr(pickle, k) for k in ("UnpicklingError", "HIGHEST_PROTOCOL", "dump", "dumps", "loads", "Pickler")})


def load_package(path: str) -> dict:
    return torch.load(path, map_location="cpu", pickle_module=_pickle_shim, weights_only=False)


def _hdemucs_config(kwargs: dict) -> HDemucsConfig:
    for k, v in _HD_REQUIRED.items():
        if k in kwargs and kwargs[k] != v:
            raise NotImplementedError(f"HDemucs option {k}={kwargs[k]!r} is outside the supported structure (needs {v!r})")
    if kwargs.get("multi_freqs"):
        raise NotImplementedError("HDemucs multi_freqs (MultiWrap band splitting) is not supported")
    fields = {k: kwargs[k] for k in _HD_MAPPED if k in kwargs}
    if "sources" in fields:
        fields["sources"] = tuple(fields["sources"])
    return HDemucsConfig(**fields)


def _demucs_v3_config(kwargs: dict) -> DemucsConfig:
    for k, v in _V3_REQUIRED.items():
        if k in kwargs and kwargs[k] != v:
            raise NotImplementedError(f"Demucs option {k}={kwargs[k]!r} is outside the supported structure (needs {v!r})")
    if kwargs.get("lstm_layers", 0):
        raise NotImplementedError("Demucs lstm_layers > 0 (the bottleneck BLSTM) is not supported")
    fields = {k: kwargs[k] for k in _V3_MAPPED if k in kwargs}
    if "sources" in fields:
        fields["sources"] = tuple(fields["sources"])
    cfg = DemucsConfig(**fields)
    if cfg.kernel_size != 2 * cfg.stride:
        raise NotImplementedError(f"Demucs kernel_size={cfg.kernel_size} with stride={cfg.stride}: only kernel_size == 2 * stride is supported")
    return cfg


def config_from_package(package: dict):
    klass = package["klass"]
    name = getattr(klass, "__name__", str(klass))
    # v1 / v2 packages pickle classes of the same name from demucs.model / model_v2 / tasnet: only demucs.demucs.Demucs is the v3 network
    v3 = name == "Demucs" and getattr(klass, "__module__", "").rsplit(".", 1)[-1] == "demucs"
    if name not in ("HTDemucs", "HDemucs") and not v3:
        raise NotImplementedError(f"model class {getattr(klass, '__module__', '?')}.{name}: the H100 Demucs path covers HTDemucs (v4), HDemucs (v3 hybrid) and "
                                  "Demucs (v3 time-domain, module demucs.demucs) packages; Demucs v1 / v2 models are not built")
    kwargs = dict(package.get("kwargs", {}))
    if package.get("args"):
        raise ValueError("positional constructor arguments in a Demucs package are not supported")
    if name == "HDemucs":
        return _hdemucs_config(kwargs)
    if v3:
        return _demucs_v3_config(kwargs)
    for k, v in _REQUIRED.items():
        if k in kwargs and kwargs[k] != v:
            raise NotImplementedError(f"HTDemucs option {k}={kwargs[k]!r} is outside the supported structure (needs {v!r})")
    if kwargs.get("norm_starts", 4) < kwargs.get("depth", 4):
        raise NotImplementedError("encoder/decoder GroupNorm (norm_starts < depth) is not supported")
    fields = {k: kwargs[k] for k in _MAPPED if k in kwargs}
    if "sources" in fields:
        fields["sources"] = tuple(fields["sources"])
    fields.setdefault("bottom_channels", 0)  # constructor defaults (htdemucs.py:56-133) where they differ from HTDemucsConfig's
    fields.setdefault("segment", 10)
    fields["segment"] = Fraction(fields["segment"])
    if "t_max_period" in kwargs:
        fields["max_period"] = float(kwargs["t_max_period"])
    return HTDemucsConfig(**fields)


def state_from_package(package: dict) -> dict:
    state = package["state"]
    if state.get("__quantized"):
        raise NotImplementedError("DiffQ-quantized Demucs packages are not supported")
    return {k: v.detach().to(torch.float32).numpy() for k, v in state.items()}  # packages may store half precision (states.py:67-77)


def load_demucs(model_path: str):
    """get_model(name, repo) of demucs/pretrained.py:58-79 for a local repo: `model_path` is a bag `.yaml` or a single `.th`.
    -> (list of (HTDemucsConfig / HDemucsConfig / DemucsConfig, state dict), bag weights or None, bag segment or None)"""
    repo = os.path.dirname(os.path.abspath(model_path))
    if model_path.endswith((".yaml", ".yml")):
        with open(model_path) as f:
            bag = yaml.safe_load(f)
        files = {}
        for fn in os.listdir(repo):  # LocalRepo.scan (repo.py:70-84): "<sig>.th" or "<sig>-<checksum>.th"
            if fn.endswith(".th"):
                files[fn[:-3].split("-")[0]] = os.path.join(repo, fn)
        models = []
        for sig in bag["models"]:
            if sig not in files:
                raise FileNotFoundError(f"Demucs bag {model_path} needs model {sig}.th in {repo}")
            pkg = load_package(files[sig])
            models.append((config_from_package(pkg), state_from_package(pkg)))
        return models, bag.get("weights"), bag.get("segment")
    pkg = load_package(model_path)
    return [(config_from_package(pkg), state_from_package(pkg))], None, None
