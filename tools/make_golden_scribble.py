"""Write tests/golden/scribble_outputs.npz from the UNMODIFIED reference.

The reference (staged under oracle/_ref by build()) is imported through tools/ref_harness.py; its HED annotator's
ControlNetHED_Apache2 is filled with the name-seeded synthetic weights (oracle/hed_oracle.synth_state_dict) and assigned
to the module's `netNetwork` global, so apply_hed never reaches its checkpoint download.  The reference's own
ControlNet.preprocess(x, type='scribble', method='hed') then runs on the CPU (cv2 on the host) for seeded images
oracle/hed_oracle.hed_image(seed, H, W).  Per case i the npz holds `case_i` = [seed, H, W], the reference's uint8 HED
map `hed_i` (apply_hed) and its uint8 scribble map `scribble_i` (channel 0 of the output times 255), so that the
post-process can be checked on its own, apart from the fp16 network's level error.  There is no xdog golden: that
reference branch raises before it computes anything.

    python tools/make_golden_scribble.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import hed_oracle as O  # noqa: E402
from tools import ref_harness  # noqa: E402

CASES = [(41, 33, 31), (42, 97, 131), (43, 200, 168), (44, 256, 256)]


def main():
    out_dir = os.path.join(ROOT, "tests", "golden")
    ref_harness.import_reference()
    import lib.model_zoo.controlnet_annotator.hed as refhed
    from lib.model_zoo.controlnet import ControlNet

    net = refhed.ControlNetHED_Apache2()
    O.fill_synthetic(net, seed=0)
    net.eval()
    refhed.netNetwork = net                              # apply_hed uses it as is: no checkpoint, no download

    arrays = {}
    for i, (seed, H, W) in enumerate(CASES):
        img = O.hed_image(seed, H, W)
        x = O.image_to_tensor(img)                       # ToPILImage(x) gives back img exactly
        hed = refhed.apply_hed(img, device="cpu")
        # preprocess reads nothing from the module for a tensor input; no 1.6 B-parameter ControlNet is built for it
        with torch.no_grad():
            y = ControlNet.preprocess(None, x, type="scribble", method="hed")
        assert refhed.netNetwork is net
        assert y.shape == (1, 3, H, W) and y.dtype == torch.float32
        scr = (y[0, 0].numpy() * 255).round().astype(np.uint8)
        assert set(np.unique(scr).tolist()) <= {0, 255}
        arrays[f"case_{i}"] = np.array([seed, H, W], np.int64)
        arrays[f"hed_{i}"] = hed
        arrays[f"scribble_{i}"] = scr
        print(f"[golden-scribble] case {i}: {H}x{W}, scribble 255 on {(scr == 255).mean():.1%} of pixels, "
              f"HED levels > 127 on {(hed > 127).mean():.1%}")
    path = os.path.join(out_dir, "scribble_outputs.npz")
    np.savez_compressed(path, **arrays)
    print(f"[golden-scribble] wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
