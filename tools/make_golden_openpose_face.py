"""Write tests/golden/openpose_face_outputs.npz and tests/golden/openpose_face_state_dict_shapes.json from the
UNMODIFIED reference.

The reference annotator (lib/model_zoo/controlnet_annotator/openpose, staged under oracle/_ref by build()) is imported
through tools/ref_harness.py with a stand-in `skimage` (hand.py imports it; the face path never calls it).
OpenposeDetector.load_model is replaced by a stub: the body network is a stand-in that returns planted stage-6 maps
(oracle/openpose_oracle.planted_maps) of known skeletons, so the face boxes are controlled, and the face model is a
Face built with Face.__new__ around either a FaceNet filled with oracle/openpose_face_oracle.synth_state_dict (kind 0)
or a stand-in that returns planted 71 x 48 x 48 maps (kind 1, openpose_face_oracle.planted_face_maps).  Nothing is loaded or downloaded.

Per case i the npz holds `case_i` = [kind, image, H, W, gain x 1000] (the image is oracle/hed_oracle.hed_image(image,
H, W)), the planted body maps `l1_i` [38,h8,w8] / `l2_i` [19,h8,w8], Body.__call__'s `candidate_i` / `subset_i`,
`boxes_i` int [F, 4] (person, x, y, w) from util.faceDetect, for kind 0 FaceNet's `hs_i` (float32 [F,71,48,48],
hs[-1]; kind 1's are oracle/openpose_face_oracle.planted_face_maps(image)), the landmarks `lmk_i` (int [F,71,2], crop
pixels, -1 for a channel without one) and ControlNet.preprocess(x, type='openpose_withface') as uint8 (`pre_i`).
Face.__call__'s input is checked against oracle/openpose_face_oracle.face_input (cv2 on the crop) rather than stored.

    python tools/make_golden_openpose_face.py
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
from oracle import openpose_face_oracle as FO  # noqa: E402
from oracle import openpose_oracle as O  # noqa: E402
from tools import ref_harness  # noqa: E402

GAIN = 0.35                     # synthetic FaceNet head gain: some channels cross 0.05, some do not
H, W = 768, 1024


def skeleton(nose, e, body=1.0):
    """18 keypoints with the nose at `nose`, eyes (+-e, -e) and ears (+-1.6 e, -0.3 e) from it (faceDetect's width is
    3 e), and a body of scale `body` below."""
    base = np.array([[0, 0], [0, 40], [-40, 40], [-60, 100], [-70, 160], [40, 40], [60, 100], [70, 160],
                     [-24, 160], [-28, 240], [-30, 320], [24, 160], [28, 240], [30, 320], [0, 0], [0, 0],
                     [0, 0], [0, 0]], np.float64) * body
    nose = np.asarray(nose, np.float64)
    k = base + nose
    k[14], k[15] = nose + [-e, -e], nose + [e, -e]
    k[16], k[17] = nose + [-1.6 * e, -0.3 * e], nose + [1.6 * e, -0.3 * e]
    return k


def planted_people(image):
    """Image 0: a LANCZOS4 face (box 168) overlapped by a smaller one, a 384 box (eye 64 px from the nose), and a face
    at the right edge whose crop is 450 x 325 (INTER_AREA emulated by the bilinear variant).  Image 1: a 420 box
    (INTER_AREA), a person without a nose and a face whose box is below 20 px.  Image 1 runs the synthetic FaceNet,
    whose hs[-1] is stored, so it has a single face box: that keeps the golden file small."""
    if image == 0:
        return [skeleton([200, 250], 28, 1.2), skeleton([250, 262], 20, 1.1), skeleton([560, 300], 64, 1.3),
                skeleton([W - 100, 330], 75, 1.2)]
    nonose = skeleton([640, 260], 30, 1.2)
    nonose[0] = np.nan
    return [skeleton([300, 300], 70, 1.2), nonose, skeleton([860, 250], 3, 1.0)]


def stage6_planted(image):
    h, w = O.resized_size(H, W)
    hp, wp = h + (-h) % 8, w + (-w) % 8
    s = h / H
    heat, paf = O.planted_maps([p * s / 8 - 0.5 for p in planted_people(image)], hp // 8, wp // 8, sigma=1.0,
                               width=0.75)
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
    from lib.model_zoo.controlnet_annotator.openpose import util as refutil
    from lib.model_zoo.controlnet_annotator.openpose.body import Body
    from lib.model_zoo.controlnet_annotator.openpose.face import Face, FaceNet

    facenet = FaceNet()
    facenet.load_state_dict(FO.synth_state_dict(0, GAIN), strict=True)
    facenet.eval()
    shapes = {k: list(v.shape) for k, v in facenet.state_dict().items()}
    with open(os.path.join(out_dir, "openpose_face_state_dict_shapes.json"), "w") as f:
        json.dump(shapes, f, indent=1)
        f.write("\n")
    body = Body.__new__(Body)
    face = Face.__new__(Face)

    def stub_load(self):
        self.body_estimation = body
        self.hand_estimation = types.SimpleNamespace(model=torch.nn.Module())
        self.face_estimation = face
    refop.OpenposeDetector.load_model = stub_load

    class Planted(torch.nn.Module):
        def __init__(self, *maps):
            super().__init__()
            self.maps = maps

        def forward(self, x):
            out = tuple(m.clone() for m in self.maps)
            return out if len(out) > 1 else [out[0][None]]

    rec = {"cand": [], "boxes": [], "x": [], "hs": [], "lmk": []}
    call, detect, peaks = Body.__call__, refutil.faceDetect, Face.compute_peaks_from_heatmaps

    def body_call(self, img):
        cand, subset = call(self, img)
        rec["cand"].append((np.asarray(cand, np.float64).reshape(-1, 4), np.asarray(subset, np.float64).reshape(-1, 20)))
        return cand, subset

    def face_detect(b, img):
        r = detect(b, img)
        rec["boxes"].append(r)
        return r

    def face_peaks(self, maps):
        p = peaks(self, maps)
        rec["lmk"].append(np.asarray(p, np.int64).reshape(-1, 2))
        return p
    Body.__call__, Face.compute_peaks_from_heatmaps = body_call, face_peaks
    refutil.faceDetect = face_detect

    arrays = {}
    cases = [(0, 1, GAIN), (1, 0, 0.0)]         # (kind, image, gain): synthetic FaceNet / planted face maps
    for i, (kind, image, gain) in enumerate(cases):
        img = np.ascontiguousarray(HO.hed_image(90 + image, H, W))
        body.model = Planted(*stage6_planted(image))
        face.model = facenet if kind == 0 else Planted(FO.planted_face_maps(image))
        def record(mod, inp, out):
            rec["x"].append(inp[0][0].numpy().copy())
            rec["hs"].append(out[-1][0].numpy().copy())
        hook = face.model.register_forward_hook(record)
        for v in rec.values():
            v.clear()
        with torch.no_grad():
            y = ControlNet.preprocess(None, HO.image_to_tensor(img), type="openpose_withface")
        hook.remove()
        cand, subset = rec["cand"][0]
        boxes = [(p, *b) for p, b in enumerate(rec["boxes"]) if b is not None]
        # a channel compute_peaks skips gets no entry: place the recorded landmarks by the channels that pass 0.05
        lmk = np.full((len(boxes), 71, 2), -1, np.int64)
        for f, (hs, (p, bx, by, bw)) in enumerate(zip(rec["hs"], boxes)):
            ch, cw = min(by + bw, H) - by, min(bx + bw, W) - bx
            maps = FO.heatmaps(hs, ch, cw)
            passing = [c for c in range(71) if (maps[c] > 0.05).any()]
            lmk[f, passing] = rec["lmk"][f]
        arrays[f"case_{i}"] = np.array([kind, image, H, W, round(gain * 1000)], np.int64)
        l1, l2 = stage6_planted(image)
        arrays[f"l1_{i}"], arrays[f"l2_{i}"] = l1[0].numpy(), l2[0].numpy()
        arrays[f"candidate_{i}"], arrays[f"subset_{i}"] = cand, subset
        arrays[f"boxes_{i}"] = np.array(boxes, np.int64).reshape(-1, 4)
        if kind == 0:
            arrays[f"hs_{i}"] = np.stack(rec["hs"]).astype(np.float32)
        for f, b in enumerate(arrays[f"boxes_{i}"]):            # the oracle's crop and resize is the reference's
            assert np.array_equal(FO.face_input(img[:, :, ::-1], b[1:])[1], rec["x"][f][None])
        arrays[f"lmk_{i}"] = lmk
        arrays[f"pre_{i}"] = (y[0].permute(1, 2, 0).numpy() * 255).round().astype(np.uint8)
        crops = [(min(b[2] + b[3], H) - b[2], min(b[1] + b[3], W) - b[1]) for b in arrays[f"boxes_{i}"]]
        print(f"[golden-openpose-face] case {i}: {len(subset)} persons, boxes {arrays[f'boxes_{i}'].tolist()}, crops "
              f"{crops}, landmarks per face {(lmk[..., 0] >= 0).sum(1).tolist()}, near-ties "
              f"{[FO.near_ties(FO.heatmaps(hs, *c)) for hs, c in zip(rec['hs'], crops)]}")
    path = os.path.join(out_dir, "openpose_face_outputs.npz")
    np.savez_compressed(path, **arrays)
    print(f"[golden-openpose-face] wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
