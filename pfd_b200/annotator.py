"""The process-global network of a ControlNet annotator (HED, PiDiNet, M-LSD, OpenPose).

Like the reference's module-global annotator networks, each network lives outside any pipeline's state dict: it is read
from its checkpoint on first use (never downloaded) or installed with ``set``, and follows the input to its device.
"""
from __future__ import annotations

import os
import sys
from typing import Callable, Dict, Optional

import torch
import torch.nn as nn


def read_state_dict(path: str) -> Dict[str, torch.Tensor]:
    """What the reference's annotators accept (e.g. pidinet/__init__.py:52-65): a .safetensors file, or a torch file
    (read with weights_only=True) with or without a top-level 'state_dict'; 'module.' is removed from the keys."""
    if os.path.splitext(path)[1].lower() == ".safetensors":
        import safetensors.torch
        sd = safetensors.torch.load_file(path, device="cpu")
    else:
        sd = torch.load(path, map_location="cpu", weights_only=True)
    sd = sd.get("state_dict", sd)
    return {k.replace("module.", ""): v for k, v in sd.items()}


class AnnotatorNetwork:
    """One annotator's installed network and its default checkpoint.  The network itself stays in the annotator
    module's ``_network`` global (``owner`` is the module's name), where the module's own code and callers that save
    and restore it find it.  ``name`` starts the missing-file error text."""

    def __init__(self, owner: str, cls: Callable[[], nn.Module], default_path: str, name: str,
                 read: Callable[[str], Dict[str, torch.Tensor]] = read_state_dict):
        self.module = sys.modules[owner]
        self.cls, self.default_path, self.name, self.read = cls, default_path, name, read

    @property
    def installed(self) -> Optional[nn.Module]:
        return self.module._network

    def set(self, m: Optional[nn.Module]) -> None:
        """Install the process-wide network (or None to drop it)."""
        self.module._network = m

    def load(self, path: Optional[str] = None) -> nn.Module:
        """Read the checkpoint (default: the reference's location relative to the working directory) with strict=True
        and install it.  Raises FileNotFoundError when the file is absent; never downloads."""
        path = path or self.default_path
        if not os.path.isfile(path):
            raise FileNotFoundError(f"{self.name} weights not found: {path}")
        m = self.cls()
        m.load_state_dict(self.read(path), strict=True)
        m.eval()
        self.set(m)
        return m

    def get(self) -> nn.Module:
        """The installed network, loading it from the default path on first use."""
        return self.installed if self.installed is not None else self.load()

    def available(self) -> bool:
        """True when a network is installed or the default checkpoint exists (so get() can load it)."""
        return self.installed is not None or os.path.isfile(self.default_path)

    def on(self, x: torch.Tensor) -> nn.Module:
        """get(), moved to x's device (the reference's annotators move their network to the input's device)."""
        net = self.get()
        if next(net.parameters()).device != x.device:
            net.to(x.device)
        return net
