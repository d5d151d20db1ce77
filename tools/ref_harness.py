"""Import harness for the UNMODIFIED reference (SHI-Labs/Prompt-Free-Diffusion).

The reference tree is its verbatim staged copy oracle/_ref (oracle/install_reference.py, run by build(); git-ignored)
or the checkout named by PFD_REFERENCE.  Used by tools/make_golden*.py to pin
the oracle / write the golden fixtures, by bench.py's reference arms (the reference's own modules timed on the
host CPU and in eager fp16 on the same GPU) and by the optional reference-side parity tests.  Recipe: SURVEY.md
App. D.  Nothing here is imported by the product.
"""
import os
import sys
import types

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _find_reference():
    for cand in (os.environ.get("PFD_REFERENCE"), os.path.join(_ROOT, "oracle", "_ref")):
        if cand and os.path.isdir(os.path.join(cand, "lib", "model_zoo")):
            return cand
    return None


REF = _find_reference()


def available() -> bool:
    return REF is not None


class EasyDict(dict):
    """Minimal attr-dict stand-in for the `easydict` package (lib/cfg_helper.py:13)."""

    def __init__(self, d=None, **kw):
        super().__init__()
        d = dict(d or {}, **kw)
        for k, v in d.items():
            self[k] = v

    @classmethod
    def _wrap(cls, v):
        if isinstance(v, dict) and not isinstance(v, EasyDict):
            return cls(v)
        if isinstance(v, (list, tuple)):
            return type(v)(cls._wrap(x) for x in v)
        return v

    def __setitem__(self, k, v):
        super().__setitem__(k, self._wrap(v))

    def __setattr__(self, k, v):
        self[k] = v

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def update(self, *a, **kw):
        for k, v in dict(*a, **kw).items():
            self[k] = v

    def __deepcopy__(self, memo):
        import copy
        return EasyDict({k: copy.deepcopy(v, memo) for k, v in self.items()})


def install_shims():
    sys.modules.setdefault("easydict", types.SimpleNamespace(EasyDict=EasyDict))
    if "matplotlib" not in sys.modules:
        mpl = types.ModuleType("matplotlib")
        mpl.__path__ = []
        plt = types.ModuleType("matplotlib.pyplot")
        mpl.pyplot = plt
        sys.modules.update({"matplotlib": mpl, "matplotlib.pyplot": plt})
    if "omegaconf" not in sys.modules:
        oc = types.ModuleType("omegaconf")
        ocl = types.ModuleType("omegaconf.listconfig")
        ocl.ListConfig = type("ListConfig", (list,), {})
        oc.listconfig = ocl
        sys.modules.update({"omegaconf": oc, "omegaconf.listconfig": ocl})
    import torch
    if torch.cuda.device_count() == 0:
        torch.cuda.device_count = lambda: 1  # lib/sync.py:31-41 divides by device_count()


_imported = False


def import_reference():
    """chdir into the reference tree (cfg_helper resolves 'configs/model' relative to CWD) and import."""
    global _imported
    if REF is None:
        raise RuntimeError("reference tree not found (neither PFD_REFERENCE nor oracle/_ref)")
    install_shims()
    os.chdir(REF)                       # cfg_helper resolves 'configs/model' relative to the CWD on every call
    if not _imported:
        sys.path.insert(0, REF)
        _imported = True
    from lib.cfg_helper import model_cfg_bank
    from lib.model_zoo import get_model
    return model_cfg_bank, get_model


class skip_random_init:
    """Make torch.nn.init.* no-ops while the reference constructs its modules: random initialisation of 1.6 B
    parameters takes ~40 s on 8 CPU cores and every floating-point tensor is overwritten by fill_reference_net()
    anyway.  (Construction must stay on the CPU: register_schedule calls .numpy() on freshly created tensors,
    diffusion_utils.py:30, so a torch.device('cuda') context breaks it.)"""
    NAMES = ("uniform_", "normal_", "trunc_normal_", "constant_", "ones_", "zeros_", "xavier_uniform_",
             "xavier_normal_", "kaiming_uniform_", "kaiming_normal_", "orthogonal_")

    def __enter__(self):
        import torch
        self.saved = {n: getattr(torch.nn.init, n) for n in self.NAMES if hasattr(torch.nn.init, n)}
        for n in self.saved:
            setattr(torch.nn.init, n, lambda tensor, *a, **k: tensor)
        return self

    def __exit__(self, *e):
        import torch
        for n, f in self.saved.items():
            setattr(torch.nn.init, n, f)


def build_reference_net(name="pfd_seecoder_with_controlnet", overrides=None, device=None, fast=False):
    """Build the reference pipeline on the CPU.  `overrides(cfgm)` may shrink the config.  fast=True skips the random
    initialisation (use only when fill_reference_net() follows).  `device` is accepted for callers that move the
    net afterwards; construction itself is always on the CPU."""
    import contextlib
    import torch
    model_cfg_bank, get_model = import_reference()
    cfgm = model_cfg_bank()(name)
    cfgm.args.vae_cfg_list[0][1].pop("pth", None)  # autokl.yaml:26 points to an absent checkpoint
    if overrides is not None:
        overrides(cfgm)
    torch.manual_seed(0)
    with (skip_random_init() if fast else contextlib.nullcontext()):
        net = get_model()(cfgm)
    net.eval()
    return net, cfgm


def fill_reference_net(net, seed=0):
    """Load the name-seeded synthetic weights (pfd_b200/weights.py) into a reference net, on whatever device its
    parameters live (values are generated on the CPU, so they are identical everywhere)."""
    if _ROOT not in sys.path:
        sys.path.insert(0, _ROOT)
    from pfd_b200.weights import SCHEDULE_BUFFERS, fill_module_
    fill_module_(net, seed=seed, skip=SCHEDULE_BUFFERS)
    return net


def cpu_sampler(net):
    """DDIMSampler whose register_buffer does not force .to('cuda') (ddim.py:17-21)."""
    from lib.model_zoo.ddim import DDIMSampler

    class CPUSampler(DDIMSampler):
        def register_buffer(self, name, attr):
            setattr(self, name, attr)

    return CPUSampler(net)
