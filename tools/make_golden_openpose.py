"""Write tests/golden/openpose_outputs.npz and tests/golden/openpose_state_dict_shapes.json from the UNMODIFIED
reference.

The reference annotator (lib/model_zoo/controlnet_annotator/openpose, staged under oracle/_ref by build()) is imported
through tools/ref_harness.py, with a stand-in `skimage` (openpose/hand.py imports skimage.measure.label, which the body
path never calls).  OpenposeDetector.load_model is replaced by a stub that installs a Body built with Body.__new__
around a bodypose_model filled with oracle/openpose_oracle.synth_state_dict, and placeholder hand / face models, so
nothing is loaded or downloaded.  For 'planted' cases the network is replaced by a stand-in that returns Gaussian
heatmaps and limb-aligned PAFs of known skeletons at the network's output size.

Per case i the npz holds `case_i` = [kind (0 network, 1 planted), seed, H, W] (the image is
oracle/hed_oracle.hed_image(seed, H, W)), the stage-6 maps the reference computed (`l1_i` [38,h8,w8], `l2_i` [19,h8,w8]), Body.__call__'s `candidate_i` [N,4]
and `subset_i` [M,20], and the reference's ControlNet.preprocess(x, type='openpose') output as uint8 (`pre_i`).

    python tools/make_golden_openpose.py
"""
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import hed_oracle as HO  # noqa: E402
from oracle import openpose_oracle as O  # noqa: E402
from tools import ref_harness  # noqa: E402

# network cases: H < 184, H = 184, the exact 2x path (368), 512^2, 512x640, 768x512, and H = 172 where int(H * s) = 183
NETWORK = [(71, 150, 200), (72, 184, 184), (73, 368, 368), (74, 512, 512), (75, 512, 640), (76, 768, 512),
           (77, 172, 251)]
# planted cases: (seed, H, W) with overlapping people, one cut by the right border, a zero-length limb and a merge
PLANTED = [(81, 512, 640)]


def planted_people(H, W):
    """Skeletons in image pixels, and the limbs left out of each one's PAF."""
    base = np.array([[0, -120], [0, -80], [-40, -80], [-60, -20], [-70, 40], [40, -80], [60, -20], [70, 40],
                     [-24, 40], [-28, 120], [-30, 200], [24, 40], [28, 120], [30, 200], [-16, -136], [16, -136],
                     [-32, -124], [32, -124]], np.float64)
    a = base + [W * 0.3, H * 0.5]
    b = base * 0.9 + [W * 0.5, H * 0.52]                 # overlaps a
    c = base + [W - 24, H * 0.5]                         # cut by the right border
    c[16] = c[14]                                        # reye == rear: a limb of length 0
    d = base * 0.8 + [W * 0.75, H * 0.45]                # no neck-nose PAF: its head row merges at the ear links
    return [a, b, c, d], [(), (), (), (12,)]


def stage6_planted(H, W):
    h, w = O.resized_size(H, W)
    hp, wp = h + (-h) % 8, w + (-w) % 8
    s = h / H
    people, skip = planted_people(H, W)
    heat, paf = O.planted_maps([p * s / 8 - 0.5 for p in people], hp // 8, wp // 8, sigma=1.0, width=0.75, skip=skip)
    l1 = torch.from_numpy(paf).permute(2, 0, 1)[None].contiguous()
    l2 = torch.from_numpy(np.concatenate([heat, np.zeros_like(heat[:, :, :1])], 2)).permute(2, 0, 1)[None].contiguous()
    return l1, l2


def main():
    out_dir = os.path.join(ROOT, "tests", "golden")
    ref_harness.import_reference()
    if "skimage" not in sys.modules:
        sk = types.ModuleType("skimage")
        skm = types.ModuleType("skimage.measure")
        skm.label = lambda *a, **k: (_ for _ in ()).throw(RuntimeError("hand path not used"))
        sk.measure = skm
        sys.modules.update({"skimage": sk, "skimage.measure": skm})
    import lib.model_zoo.controlnet_annotator.openpose as refop
    from lib.model_zoo.controlnet import ControlNet
    from lib.model_zoo.controlnet_annotator.openpose.body import Body
    from lib.model_zoo.controlnet_annotator.openpose.model import bodypose_model

    model = bodypose_model()
    model.load_state_dict(O.synth_state_dict(0), strict=True)
    model.eval()
    shapes = {k: list(v.shape) for k, v in model.state_dict().items()}
    with open(os.path.join(out_dir, "openpose_state_dict_shapes.json"), "w") as f:
        json.dump(shapes, f, indent=1)
        f.write("\n")
    body = Body.__new__(Body)
    body.model = model

    def stub_load(self):
        self.body_estimation = body
        self.hand_estimation = types.SimpleNamespace(model=torch.nn.Module())
        self.face_estimation = types.SimpleNamespace(model=torch.nn.Module())
    refop.OpenposeDetector.load_model = stub_load

    captured, returned = [], []
    call = Body.__call__

    def recording_call(self, img):
        cand, subset = call(self, img)
        returned.append((np.asarray(cand, np.float64).reshape(-1, 4), np.asarray(subset, np.float64).reshape(-1, 20)))
        return cand, subset
    Body.__call__ = recording_call

    class Planted(torch.nn.Module):
        def __init__(self, l1, l2):
            super().__init__()
            self.l1, self.l2 = l1, l2

        def forward(self, x):
            return self.l1.clone(), self.l2.clone()

    arrays = {}
    cases = [(0, *c) for c in NETWORK] + [(1, *c) for c in PLANTED]
    for i, (kind, seed, H, W) in enumerate(cases):
        img = np.ascontiguousarray(HO.hed_image(seed, H, W))
        if kind == 1:
            body.model = Planted(*stage6_planted(H, W))
        else:
            body.model = model
        hook = body.model.register_forward_hook(lambda mod, inp, out: captured.append(
            (out[0][0].detach().numpy().copy(), out[1][0].detach().numpy().copy())))
        captured.clear()
        returned.clear()
        x = HO.image_to_tensor(img)
        with torch.no_grad():
            y = ControlNet.preprocess(None, x, type="openpose")
        hook.remove()
        assert y.shape == (1, 3, H, W) and y.dtype == torch.float32 and len(captured) == 1 and len(returned) == 1
        cand, subset = returned[0]
        arrays[f"case_{i}"] = np.array([kind, seed, H, W], np.int64)
        arrays[f"l1_{i}"], arrays[f"l2_{i}"] = captured[0][0].astype(np.float32), captured[0][1].astype(np.float32)
        arrays[f"candidate_{i}"], arrays[f"subset_{i}"] = cand, subset
        arrays[f"pre_{i}"] = (y[0].permute(1, 2, 0).numpy() * 255).round().astype(np.uint8)
        h, w = O.resized_size(H, W)
        heat, paf = O.reference_maps(captured[0][0], captured[0][1], h, w, H, W)
        ties = O.near_ties(heat, paf, cand, subset, H, W)
        print(f"[golden-openpose] case {i}: {'planted' if kind else 'network'} {H}x{W}: {len(cand)} peaks, "
              f"{len(subset)} persons {subset[:, 19].astype(int).tolist()}, near-ties {ties}")
    path = os.path.join(out_dir, "openpose_outputs.npz")
    np.savez_compressed(path, **arrays)
    print(f"[golden-openpose] wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
