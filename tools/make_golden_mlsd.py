"""Write tests/golden/mlsd_outputs.npz and tests/golden/mlsd_state_dict_shapes.json from the UNMODIFIED reference.

The reference annotator (lib/model_zoo/controlnet_annotator/mlsd, staged under oracle/_ref by build()) is imported
through tools/ref_harness.py; its MobileV2_MLSD_Large is filled with the synthetic weights of
oracle/mlsd_oracle.synth_state_dict (name-seeded, output gains) and assigned to the module's `mlsdmodel` global BEFORE
apply_mlsd runs, so apply_mlsd never loads or downloads a checkpoint.  Per case i the npz holds `case_i` = [seed, H, W]
(the image is oracle/hed_oracle.hed_image(seed, H, W)), `thr_i` = [thr_v, thr_d], the network's output channels
7..11 `maps_i` (fp32 [5, H/2, W/2]; absent when pred_lines raised), the segment list pred_lines returned, as
apply_mlsd converts it with int() (`segs_i`, int64 [n, 4], top-k order; empty when it raised),
apply_mlsd's uint8 map `lines_i` and the reference's own ControlNet.preprocess(x, type='mlsd', thr_v=, thr_d=) output
as uint8 (`pre_i`).

    python tools/make_golden_mlsd.py
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import hed_oracle as HO  # noqa: E402
from oracle import mlsd_oracle as O  # noqa: E402
from tools import ref_harness  # noqa: E402

# (seed, H, W, thr_v, thr_d): conforming sizes (33 and 257 are 16k + 1), a size whose decoder concat fails (200x168),
# one with fewer than 200 map cells (16x32), and non-default thresholds
CASES = [(61, 33, 48, 0.1, 0.1), (62, 96, 128, 0.1, 0.1), (63, 257, 176, 0.1, 0.1), (64, 256, 256, 0.1, 0.1),
         (65, 200, 168, 0.1, 0.1), (66, 16, 32, 0.1, 0.1), (67, 128, 160, 0.3, 30.0)]


def main():
    out_dir = os.path.join(ROOT, "tests", "golden")
    ref_harness.import_reference()
    import lib.model_zoo.controlnet_annotator.mlsd as refmlsd
    from lib.model_zoo.controlnet import ControlNet
    from lib.model_zoo.controlnet_annotator.mlsd.models.mbv2_mlsd_large import MobileV2_MLSD_Large

    net = MobileV2_MLSD_Large()
    O.fill_synthetic(net, seed=0)
    net.eval()
    refmlsd.mlsdmodel = net                              # apply_mlsd uses it as is: no checkpoint, no download
    shapes = {k: list(v.shape) for k, v in net.state_dict().items()}
    with open(os.path.join(out_dir, "mlsd_state_dict_shapes.json"), "w") as f:
        json.dump(shapes, f, indent=1)
        f.write("\n")

    captured, returned = [], []
    net.block23.register_forward_hook(lambda mod, inp, out: captured.append(out[0, 7:12].detach().numpy().copy()))
    pred_lines = refmlsd.pred_lines

    def recording_pred_lines(*a, **k):
        lines = pred_lines(*a, **k)
        returned.append(np.array([[int(v) for v in line] for line in lines], np.int64).reshape(-1, 4))
        return lines
    refmlsd.pred_lines = recording_pred_lines

    arrays = {}
    for i, (seed, H, W, thr_v, thr_d) in enumerate(CASES):
        img = np.ascontiguousarray(HO.hed_image(seed, H, W))  # cv2.line refuses a non-contiguous output array
        captured.clear()
        returned.clear()
        lines = refmlsd.apply_mlsd(img, thr_v, thr_d, device="cpu")
        assert refmlsd.mlsdmodel is net and lines.shape == (H, W) and lines.dtype == np.uint8
        x = HO.image_to_tensor(img)                      # ToPILImage(x) gives back img exactly
        with torch.no_grad():
            y = ControlNet.preprocess(None, x, type="mlsd", thr_v=thr_v, thr_d=thr_d)
        assert y.shape == (1, 3, H, W) and y.dtype == torch.float32
        pre = (y[0, 0].numpy() * 255).round().astype(np.uint8)
        arrays[f"case_{i}"] = np.array([seed, H, W], np.int64)
        arrays[f"thr_{i}"] = np.array([thr_v, thr_d], np.float64)
        arrays[f"lines_{i}"] = lines
        arrays[f"pre_{i}"] = pre
        ran = len(returned) > 0                          # pred_lines returned (every conforming case here has segments)
        assert ran == O.size_supported(H, W), f"case {i}: size rule disagrees with the reference"
        if ran:
            arrays[f"maps_{i}"] = captured[0].astype(np.float32)
        segs = returned[0] if ran else np.zeros((0, 4), np.int64)
        arrays[f"segs_{i}"] = segs
        msg = ""
        if ran:
            heat = O.heat_map(captured[0][0])
            peaks = int((heat > np.float32(thr_v)).sum())
            below = int(((heat > 0) & (heat <= np.float32(thr_v))).sum())
            length = np.hypot(segs[:, 2] - segs[:, 0], segs[:, 3] - segs[:, 1]) if len(segs) else np.zeros(1)
            outside = int(((segs[:, [0, 2]] < 0) | (segs[:, [0, 2]] >= W)).any(1).sum() +
                          ((segs[:, [1, 3]] < 0) | (segs[:, [1, 3]] >= H)).any(1).sum()) if len(segs) else 0
            msg = (f"{peaks} peaks above thr_v, {below} below, {len(segs)} segments, median length "
                   f"{np.median(length):.1f} px, {outside} endpoint(s) outside, ")
        print(f"[golden-mlsd] case {i}: {H}x{W} thr ({thr_v}, {thr_d}): {msg}{(lines > 0).mean():.2%} line pixels, "
              f"preprocess == apply_mlsd: {np.array_equal(pre, lines)}")
    path = os.path.join(out_dir, "mlsd_outputs.npz")
    np.savez_compressed(path, **arrays)
    print(f"[golden-mlsd] wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
