"""Write tests/golden/hed_outputs.npz and tests/golden/hed_state_dict_shapes.json from the UNMODIFIED reference.

The reference annotator (lib/model_zoo/controlnet_annotator/hed, staged under oracle/_ref by build()) is imported
through tools/ref_harness.py, its ControlNetHED_Apache2 is filled with the name-seeded synthetic weights
(oracle/hed_oracle.synth_state_dict) and assigned to the module's `netNetwork` global BEFORE apply_hed runs, so
apply_hed never reaches its checkpoint download.  apply_hed then runs on the CPU in fp32 on seeded images whose sides are
not multiples of 16.  The npz holds, per case i: the image seed and shape (`case_i` = [seed, H, W]; the image is
oracle/hed_oracle.hed_image(seed, H, W)), the uint8 output (`u8_i`) and the five side maps of the reference network,
sampled with stride `side_i_k_stride` in both directions where they are large (`side_i_k`, full shape in
`side_i_k_shape`).

    python tools/make_golden_hed.py
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import hed_oracle as O  # noqa: E402
from tools import ref_harness  # noqa: E402

CASES = [(11, 33, 31), (12, 97, 131), (13, 256, 256)]
MAX_SIDE_SAMPLES = 4096


def main():
    out_dir = os.path.join(ROOT, "tests", "golden")
    ref_harness.import_reference()
    import lib.model_zoo.controlnet_annotator.hed as refhed
    from einops import rearrange

    net = refhed.ControlNetHED_Apache2()
    O.fill_synthetic(net, seed=0)
    net.eval()
    refhed.netNetwork = net                              # apply_hed uses it as is: no checkpoint, no download
    shapes = {k: list(v.shape) for k, v in net.state_dict().items()}
    with open(os.path.join(out_dir, "hed_state_dict_shapes.json"), "w") as f:
        json.dump(shapes, f, indent=1)
        f.write("\n")

    arrays = {}
    for i, (seed, H, W) in enumerate(CASES):
        img = O.hed_image(seed, H, W)
        u8 = refhed.apply_hed(img, device="cpu")
        assert refhed.netNetwork is net
        with torch.no_grad():                            # the side maps apply_hed resizes (hed/__init__.py:115-117)
            sides = net(rearrange(torch.from_numpy(img.copy()).float(), "h w c -> 1 c h w"))
        arrays[f"case_{i}"] = np.array([seed, H, W], np.int64)
        arrays[f"u8_{i}"] = u8
        for k, s in enumerate(sides):
            s = s[0, 0].numpy().astype(np.float32)
            stride = 1
            while (s.shape[0] // stride) * (s.shape[1] // stride) > MAX_SIDE_SAMPLES:
                stride += 1
            arrays[f"side_{i}_{k}"] = s[::stride, ::stride].copy()
            arrays[f"side_{i}_{k}_stride"] = np.array(stride, np.int64)
            arrays[f"side_{i}_{k}_shape"] = np.array(s.shape, np.int64)
        inner = float(((u8 > 0) & (u8 < 255)).mean())
        print(f"[golden-hed] case {i}: {H}x{W}, {inner:.1%} of pixels strictly between 0 and 255, "
              f"side std {[round(float(s.std()), 3) for s in sides]}")
    path = os.path.join(out_dir, "hed_outputs.npz")
    np.savez_compressed(path, **arrays)
    print(f"[golden-hed] wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
