"""pfd_b200 — H100-native (sm_90a) implementation of the Prompt-Free-Diffusion inference hot path.

Public surface (mirrors the reference's lib.model_zoo / lib.cfg_helper plugin API):
    from pfd_b200 import get_model, register, model_cfg_bank, DDIMSampler, Sampler, set_deterministic, randn
    net = get_model()(model_cfg_bank()('pfd_seecoder_with_controlnet')); net.to('cuda')
    c = net.ctx_encode(img, 'image'); x, _ = DDIMSampler(net).sample(...); im = net.vae_decode(x, 'image')
All arithmetic runs in the hand-written CUDA kernels behind include/pfd_b200.h (pfd_b200/native.py);
there is no torch / CPU fallback.
"""
from .registry import AttrDict, get_model, register, install_into_reference  # noqa: F401
from .configs import model_cfg_bank  # noqa: F401


def set_deterministic(flag: bool = True) -> None:
    """Switch deterministic mode on or off (pfd_set_option "deterministic", include/pfd_b200.h): outputs become a
    bitwise function of each sample's own inputs, whatever else is in its batch and on however many GPUs and SMs.
    Every cached CUDA graph and packed plan is invalidated, so nothing captured in one mode replays in the other."""
    from . import graphs, native
    native.set_env_option("deterministic", int(bool(flag)))
    graphs.invalidate()


def is_deterministic() -> bool:
    """True when deterministic mode is on (set_deterministic, or PFD_DETERMINISTIC=1 at start-up)."""
    from . import native
    return native.deterministic()


def randn(shape, seeds, stream=0, draw=0, device=None):
    """Per-sample seeded fp16 N(0, 1) noise, exactly what the samplers draw for x_info["seeds"] (pfd_b200/rng.py):
    stream 0 = x_T, 1 = per-step sampler noise at schedule position `draw`, 2 = img2img forward noise."""
    from . import rng
    return rng.randn(shape, seeds, stream=stream, draw=draw, device=device)


def __getattr__(name):
    if name == "DDIMSampler":
        from .ddim import DDIMSampler
        return DDIMSampler
    if name == "Sampler":
        from .sampler import Sampler
        return Sampler
    raise AttributeError(name)
