"""Write tests/golden/pidinet_outputs.npz and tests/golden/pidinet_state_dict_shapes.json from the UNMODIFIED reference.

The reference annotator (lib/model_zoo/controlnet_annotator/pidinet, staged under oracle/_ref by build()) is imported
through tools/ref_harness.py; its pidinet() is filled with the synthetic weights of oracle/pidinet_oracle.synth_state_dict
(name-seeded, classifier gain 10) and assigned to the module's `netNetwork` global BEFORE apply_pidinet runs, so
apply_pidinet never reaches its checkpoint download.  Per case i the npz holds `case_i` = [seed, H, W] (the image is
oracle/hed_oracle.hed_image(seed, H, W)), apply_pidinet's uint8 map `u8_i`, the four pre-sigmoid side maps of the
reference network (the MapReduce outputs before F.interpolate), sampled with stride `side_i_k_stride` where they are
large (`side_i_k`, full shape in `side_i_k_shape`), and the reference's own ControlNet.preprocess(x, type='scribble')
output with the default method as uint8 (`scribble_i`).

    python tools/make_golden_pidinet.py
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import hed_oracle as HO  # noqa: E402
from oracle import pidinet_oracle as O  # noqa: E402
from tools import ref_harness  # noqa: E402

CASES = [(51, 33, 31), (52, 97, 131), (53, 200, 168), (54, 256, 256)]
MAX_SIDE_SAMPLES = 4096


def main():
    out_dir = os.path.join(ROOT, "tests", "golden")
    ref_harness.import_reference()
    import lib.model_zoo.controlnet_annotator.pidinet as refpidi
    from lib.model_zoo.controlnet import ControlNet

    net = refpidi.pidinet()
    O.fill_synthetic(net, seed=0)
    net.eval()
    refpidi.netNetwork = net                             # apply_pidinet uses it as is: no checkpoint, no download
    shapes = {k: list(v.shape) for k, v in net.state_dict().items()}
    with open(os.path.join(out_dir, "pidinet_state_dict_shapes.json"), "w") as f:
        json.dump(shapes, f, indent=1)
        f.write("\n")

    # the MapReduce outputs, captured by hooks during the network's own forward
    captured = []
    for m in net.conv_reduces:
        m.register_forward_hook(lambda mod, inp, out: captured.append(out[0, 0].detach().numpy().astype(np.float32)))

    arrays = {}
    for i, (seed, H, W) in enumerate(CASES):
        img = HO.hed_image(seed, H, W)
        captured.clear()
        u8 = refpidi.apply_pidinet(img, device="cpu")
        assert refpidi.netNetwork is net
        sides = list(captured)
        assert len(sides) == 4 and u8.shape == (H, W) and u8.dtype == np.uint8
        x = HO.image_to_tensor(img)                      # ToPILImage(x) gives back img exactly
        with torch.no_grad():
            y = ControlNet.preprocess(None, x, type="scribble")
        assert refpidi.netNetwork is net
        assert y.shape == (1, 3, H, W) and y.dtype == torch.float32
        scr = (y[0, 0].numpy() * 255).round().astype(np.uint8)
        assert set(np.unique(scr).tolist()) <= {0, 255}
        arrays[f"case_{i}"] = np.array([seed, H, W], np.int64)
        arrays[f"u8_{i}"] = u8
        arrays[f"scribble_{i}"] = scr
        for k, s in enumerate(sides):
            stride = 1
            while (s.shape[0] // stride) * (s.shape[1] // stride) > MAX_SIDE_SAMPLES:
                stride += 1
            arrays[f"side_{i}_{k}"] = s[::stride, ::stride].copy()
            arrays[f"side_{i}_{k}_stride"] = np.array(stride, np.int64)
            arrays[f"side_{i}_{k}_shape"] = np.array(s.shape, np.int64)
        inner = float(((u8 > 0) & (u8 < 255)).mean())
        _, acts = O.network_sides(O.synth_state_dict(0), img, return_acts=True)
        print(f"[golden-pidinet] case {i}: {H}x{W}, {inner:.1%} of pixels strictly between 0 and 255, levels "
              f"{int(u8.min())}..{int(u8.max())}, scribble 255 on {(scr == 255).mean():.1%}, largest |block output| "
              f"{max(acts):.3f}, side std {[round(float(s.std()), 3) for s in sides]}")
    path = os.path.join(out_dir, "pidinet_outputs.npz")
    np.savez_compressed(path, **arrays)
    print(f"[golden-pidinet] wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
