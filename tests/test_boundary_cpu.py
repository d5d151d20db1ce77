"""The reference-facing boundary (SURVEY.md §8b): `pfd_b200.install_into_reference()` registers the pfd_b200 classes
in the REFERENCE's own registry, so the reference's `model_cfg_bank` / `get_model` (what app.py calls, app.py:111)
build the pfd_b200 pipeline, and reference-built state dicts load with strict=True (app.py:137-162).

Needs the reference tree (its copy staged under oracle/_ref by build(), or PFD_REFERENCE); skipped otherwise.
Runs in a child process because the harness chdir()s into the reference tree and patches sys.modules."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

CHILD = r'''
import json, os, sys
ROOT = sys.argv[1]
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch
import ref_harness as rh
model_cfg_bank, get_model = rh.import_reference()
res = {}
# 1. a state dict built by the UNMODIFIED reference classes (VAE: 84 M parameters, real tensors)
cfg_vae = model_cfg_bank()("autokl_v2"); cfg_vae.pop("pth", None)
torch.manual_seed(0)
ref_vae = get_model()(cfg_vae)
res["ref_vae_class"] = type(ref_vae).__module__
ref_sd = {k: v.clone() for k, v in ref_vae.state_dict().items()}
# 2. install pfd_b200 into the reference's registry
import pfd_b200
from pfd_b200.registry import install_into_reference
install_into_reference()
import lib.model_zoo.ddim as ref_ddim, lib.model_zoo.seecoder as ref_see
res["sampler_swapped"] = ref_ddim.DDIMSampler.__module__
res["ppe_swapped"] = ref_see.PPE_MLP.__module__
# 3. the reference's bank + registry now build pfd_b200 classes (full pipeline on the meta device: names/shapes only)
cfgm = model_cfg_bank()("pfd_seecoder_with_controlnet")
cfgm.args.vae_cfg_list[0][1].pop("pth", None)
with torch.device("meta"):
    net = get_model()(cfgm, verbose=False)        # verbose=True sums the parameters on the host (get_model.py:108-115)
res["net_class"] = type(net).__module__ + "." + type(net).__name__
res["children"] = {n: type(m).__module__ for n, m in [("vae", net.vae["image"]), ("ctx", net.ctx["image"]),
                                                     ("diffuser", net.diffuser["image"]), ("ctl", net.ctl)]}
res["shapes"] = {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in net.state_dict().items()}
res["to_returns_none"] = net.to("meta") is None and net.device == "meta"
# 4. round trip: reference-built VAE state dict -> pfd_b200 VAE built through the reference registry, strict
ours = get_model()(cfg_vae)
res["ours_vae_class"] = type(ours).__module__
missing = ours.load_state_dict(ref_sd, strict=True)
back = ours.state_dict()
res["roundtrip_keys_equal"] = sorted(back) == sorted(ref_sd)
res["roundtrip_values_equal"] = all(torch.equal(back[k], ref_sd[k]) for k in ref_sd)
# 5. and back into the reference class
ref_vae.load_state_dict(back, strict=True)
print("RESULT " + json.dumps(res))
'''


def test_install_into_reference_builds_pfd_b200_through_the_reference_registry():
    import ref_harness as rh
    if not rh.available():
        pytest.skip("reference tree not present (oracle/_ref or PFD_REFERENCE)")
    r = subprocess.run([sys.executable, "-c", CHILD, ROOT], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1]
    res = json.loads(line[len("RESULT "):])
    assert res["ref_vae_class"].startswith("lib.model_zoo"), "the first build must come from the unmodified reference"
    assert res["net_class"] == "pfd_b200.pfd.PromptFreeDiffusion_with_control"
    assert all(m.startswith("pfd_b200.") for m in res["children"].values()), res["children"]
    assert res["ours_vae_class"].startswith("pfd_b200.")
    assert res["sampler_swapped"] == "pfd_b200.ddim" and res["ppe_swapped"] == "pfd_b200.seecoder"
    assert res["to_returns_none"]                                        # pfd.py:100-102 / app.py:127
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "state_dict_shapes.json")))
    assert res["shapes"] == gold, "state-dict layout built through the reference registry differs from the reference's"
    assert len(gold) == 1902
    assert res["roundtrip_keys_equal"] and res["roundtrip_values_equal"]
