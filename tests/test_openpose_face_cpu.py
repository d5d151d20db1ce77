"""OpenPose face annotator on the CPU: FaceNet's state-dict layout, the oracle against the reference's goldens, the
area-emulated bilinear resize tables against cv2, and the missing-weight messages."""
import json
import os

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _goldens():
    z = np.load(os.path.join(GOLDEN, "openpose_face_outputs.npz"))
    return z, len([k for k in z.files if k.startswith("case_")])


def test_state_dict_layout_matches_reference():
    from pfd_b200.openpose_face import FacePose
    with open(os.path.join(GOLDEN, "openpose_face_state_dict_shapes.json")) as f:
        ref = json.load(f)
    sd = FacePose().state_dict()
    assert list(sd) == list(ref)
    assert {k: list(v.shape) for k, v in sd.items()} == ref
    assert len(sd) == 104 and sum(v.numel() for v in sd.values()) == 38425706


@pytest.mark.parametrize("suffix", [".pth", "_wrapped.pth", ".safetensors"])
def test_raw_wrapped_and_safetensors_checkpoints_load_strict(tmp_path, suffix):
    from oracle import openpose_face_oracle as FO
    from pfd_b200 import openpose_face
    sd = FO.synth_state_dict(3)
    path = str(tmp_path / f"facenet{suffix}")
    if suffix == ".safetensors":
        import safetensors.torch
        safetensors.torch.save_file({k: v.contiguous() for k, v in sd.items()}, path)
    else:
        torch.save({"state_dict": sd} if "wrapped" in suffix else sd, path)
    prev = openpose_face._network
    try:
        m = openpose_face.load_face(path)
        assert all(torch.equal(m.state_dict()[k], v) for k, v in sd.items())
    finally:
        openpose_face.set_network(prev)


def test_oracle_reproduces_reference_goldens():
    from oracle import hed_oracle as HO
    from oracle import openpose_face_oracle as FO
    z, n = _goldens()
    for i in range(n):
        kind, image, H, W, gain = (int(v) for v in z[f"case_{i}"])
        cand, subset, boxes = z[f"candidate_{i}"], z[f"subset_{i}"], z[f"boxes_{i}"]
        bgr = np.ascontiguousarray(HO.hed_image(90 + image, H, W)[:, :, ::-1])
        got = [(p, *b) for p, b in ((p, FO.face_box(FO.person_keypoints(cand, row), H, W))
                                    for p, row in enumerate(subset)) if b is not None]
        assert np.array_equal(np.array(got).reshape(-1, 4), boxes), f"case {i}: face boxes"
        if kind == 0:
            sd = FO.synth_state_dict(0, gain / 1000)
            x = np.concatenate([FO.face_input(bgr, b[1:])[1] for b in boxes])
            with torch.no_grad():
                hs = FO.network(sd, torch.from_numpy(x)).numpy()
            err = np.abs(hs - z[f"hs_{i}"]).max()
            assert err < 1e-4, f"case {i}: hs[-1] off by {err}"
            hs = z[f"hs_{i}"]
        else:
            hs = np.stack([FO.planted_face_maps(image).numpy()] * len(boxes))
        dots = [[] for _ in range(len(subset))]
        for f, (p, bx, by, bw) in enumerate(boxes):
            maps = FO.heatmaps(hs[f], min(by + bw, H) - by, min(bx + bw, W) - bx)
            lmk = FO.peaks(maps)
            assert np.array_equal(lmk, z[f"lmk_{i}"][f]), f"case {i} face {f}: landmarks"
            dots[p] = FO.landmarks_to_pixels(lmk, (bx, by, bw), H, W)
        assert np.array_equal(FO.draw(cand, subset, dots, H, W), z[f"pre_{i}"]), f"case {i}: canvas"


CROPS = [(330, 600), (600, 330), (200, 600), (383, 385), (100, 500), (250, 384), (383, 900), (20, 1000), (450, 325)]


@pytest.mark.parametrize("h,w", CROPS)
def test_area_emulated_bilinear_tables_match_cv2(h, w):
    """cv2.resize(INTER_AREA) of a crop with a side below 384 runs OpenCV's bilinear variant; the tables of
    openpose_tables.area_linear_axis with VResizeLinear's fixed-point rounding give its bits."""
    import cv2
    from pfd_b200 import openpose_tables as T
    rng = np.random.default_rng(h * 1000 + w)
    x = rng.integers(0, 256, (h, w), dtype=np.uint8)
    plan = T.resize_plan(h, w, 384, 384, area=True, fixed=True)
    assert plan[0] == "linear"
    (iy, wy), (ix, wx) = plan[1], plan[2]
    xi = x.astype(np.int64)
    rows = xi[:, ix[:, 0]] * wx[None, :, 0] + xi[:, ix[:, 1]] * wx[None, :, 1]
    r0, r1 = rows[iy[:, 0]], rows[iy[:, 1]]
    got = (((wy[:, 0, None] * (r0 >> 4)) >> 16) + ((wy[:, 1, None] * (r1 >> 4)) >> 16) + 2) >> 2
    ref = cv2.resize(x, (384, 384), interpolation=cv2.INTER_AREA)
    assert np.array_equal(np.clip(got, 0, 255).astype(np.uint8), ref)


def test_missing_face_weights_message(tmp_path, monkeypatch):
    from pfd_b200 import openpose_face
    prev = openpose_face._network
    openpose_face.set_network(None)
    monkeypatch.chdir(tmp_path)
    try:
        with pytest.raises(NotImplementedError) as e:
            openpose_face.preprocess_openpose_face(torch.zeros((1, 3, 64, 64)))
    finally:
        openpose_face.set_network(prev)
    msg = str(e.value)
    for s in ("facenet.pth", openpose_face.DEFAULT_PATH, "load_face", "set_network", "type='openpose'"):
        assert s in msg


def test_face_hand_type_message():
    from pfd_b200.controlnet import ControlNet
    with pytest.raises(NotImplementedError) as e:
        ControlNet.preprocess(type("C", (), {"get_device": lambda self: torch.device("cpu")})(),
                              torch.zeros((1, 3, 8, 8)), type="openpose_withfacehand")
    assert "type='openpose'" in str(e.value) and "'openpose_withface'" in str(e.value)
