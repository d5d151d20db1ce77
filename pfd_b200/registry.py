"""Model registry + config bank with the reference's plugin surface.

Mirrors lib/model_zoo/common/get_model.py:32-124 (`get_model()` singleton, `@register(name)`,
`get_model()(cfg)` with cfg.type / cfg.args / cfg.pth|pretrained / strict_sd) and the part of
lib/cfg_helper.py:102-146 that app.py uses (`model_cfg_bank()(name)`).  `install_into_reference()`
registers the pfd_b200 classes under the reference's own type names inside the reference's registry,
so `app.py` (run from the reference tree) builds the pfd_b200 pipeline unchanged — see INTEGRATION.md.
"""
from __future__ import annotations

import copy
import os.path as osp
from typing import Any, Callable, Dict

import torch


class AttrDict(dict):
    """Small attr-dict (the reference uses easydict.EasyDict for configs)."""

    def __init__(self, d=None, **kw):
        super().__init__()
        for k, v in dict(d or {}, **kw).items():
            self[k] = v

    @staticmethod
    def _wrap(v):
        if isinstance(v, dict) and not isinstance(v, AttrDict):
            return AttrDict(v)
        if isinstance(v, (list, tuple)):
            return type(v)(AttrDict._wrap(x) for x in v)
        return v

    def __setitem__(self, k, v):
        super().__setitem__(k, self._wrap(v))

    __setattr__ = __setitem__

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __deepcopy__(self, memo):
        return AttrDict({k: copy.deepcopy(v, memo) for k, v in self.items()})


def _singleton(cls):
    inst = {}

    def get(*a, **k):
        if cls not in inst:
            inst[cls] = cls(*a, **k)
        return inst[cls]
    return get


@_singleton
class get_model(object):
    def __init__(self):
        self.model: Dict[str, Callable] = {}

    def register(self, model, name):
        self.model[name] = model

    def __call__(self, cfg, verbose=False):
        if cfg is None:
            return None
        from . import _register_all  # noqa: F401  (registers the built-in types on first use)
        t = cfg["type"]
        if t not in self.model:
            raise ValueError(f"pfd_b200: unknown model type '{t}' (known: {sorted(self.model)})")
        args = copy.deepcopy(cfg.get("args", {}))
        net = self.model[t](**args)
        pretrained = cfg.get("pretrained", None) or cfg.get("pth", None)
        if pretrained is not None:
            ext = osp.splitext(pretrained)[1]
            if ext == ".safetensors":
                from safetensors.torch import load_file
                sd = load_file(pretrained, cfg.get("map_location", "cpu"))
            else:
                sd = torch.load(pretrained, map_location=cfg.get("map_location", "cpu"))
                if ext == ".ckpt":
                    sd = sd["state_dict"]
            net.load_state_dict(sd, strict=cfg.get("strict_sd", True))
        return net


def register(name):
    def wrapper(cls):
        get_model().register(cls, name)
        return cls
    return wrapper


def install_into_reference():
    """Register pfd_b200 classes in the *reference's* registry (lib.model_zoo.common.get_model) under
    the reference type names, and swap the sampler / PPE_MLP symbols app.py imports.  Must be called
    from a process whose CWD / sys.path is the reference tree (as app.py runs).  The reference modules
    are imported eagerly first because get_model.__call__ imports them lazily and their @register
    decorators would otherwise overwrite ours (get_model.py:72-85, SURVEY.md §8b)."""
    import importlib
    from . import _register_all  # noqa: F401
    ref_zoo = importlib.import_module("lib.model_zoo")
    for m in ("pfd", "autokl", "openaimodel", "controlnet", "seecoder", "swin", "ddim"):
        importlib.import_module(f"lib.model_zoo.{m}")
    ref_get_model = importlib.import_module("lib.model_zoo.common.get_model").get_model
    for name, cls in get_model().model.items():
        ref_get_model().register(cls, name)
    from . import ddim as our_ddim, seecoder as our_seecoder
    importlib.import_module("lib.model_zoo.ddim").DDIMSampler = our_ddim.DDIMSampler
    importlib.import_module("lib.model_zoo.seecoder").PPE_MLP = our_seecoder.PPE_MLP
    return ref_zoo
