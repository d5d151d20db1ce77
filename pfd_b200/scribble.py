"""Scribble annotators (ControlNet.preprocess type 'scribble') on the pfd_b200 kernels (controlnet.py:432-491).

    method='hed'     the HED network (hed.py), then make_scribble on its uint8 levels: float32 Gaussian blur
                     (sigma 3), non-maximum suppression along four 3-tap lines, `> 127`, uint8 Gaussian blur (sigma 3,
                     OpenCV's bit-exact fixed-point path), `> 4`                        (pfd_scribble_hed_f32)
    method='xdog'    difference of float32 Gaussians (sigma 0.5 and 5) of the uint8 RGB image, minimum over the
                     channels, uint8 truncation, edge where uint8(2 * uint8(255 - dog)) > threshold
                                                                                        (pfd_scribble_xdog_f32)
    method='pidinet' (the reference's default) needs the PiDiNet network, which pfd_b200 does not provide.

The reference's xdog branch cannot run as written (it passes device= to a one-argument function and would return nine
channels); this is what its lines compute, as three equal channels like every other type.  The product
2 * (255 - dog) is uint8 arithmetic in numpy and wraps mod 256 (255 - dog = 128 gives 0, not an edge); that is kept.
"""
from __future__ import annotations

import math

import torch

from . import native as nv


def preprocess_scribble(x: torch.Tensor, method: str = "pidinet", threshold=32) -> torch.Tensor:
    """ControlNet.preprocess(x, type='scribble', method=...) for a CUDA [B,3,H,W] image in [0,1] -> float32
    [B,3,H,W] with 1.0 on scribble pixels."""
    if method == "hed":
        from .hed import preprocess_hed
        return nv.scribble_hed(preprocess_hed(x))
    if method == "xdog":
        # the uint8 edge strength e (0..254) is compared as e > threshold: for a fractional threshold that is
        # e > floor(threshold); clamping keeps the integer in range without changing any decision
        t = min(max(math.floor(threshold), -1), 255)
        return nv.scribble_xdog(x, t)
    if method == "pidinet":
        raise NotImplementedError("scribble method 'pidinet' needs the PiDiNet network, which pfd_b200 does not "
                                  "provide: use method='hed' or method='xdog', or feed a ready control map "
                                  "(do_preprocess=False)")
    raise ValueError(f"unknown scribble method {method!r} (pfd_b200 runs 'hed' and 'xdog'; 'pidinet' is not "
                     "implemented)")
