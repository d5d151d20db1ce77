"""OpenPose body annotator: host-side tables, weight loading and the oracle, checked without a GPU."""
import numpy as np
import pytest
import torch

CASES = [(512, 640, 184, 230), (368, 368, 184, 184), (100, 150, 184, 276), (768, 512, 184, 122),
         (501, 333, 184, 122), (552, 552, 184, 184), (184, 230, 512, 640), (184, 230, 100, 125), (184, 184, 92, 92)]


@pytest.mark.parametrize("h,w,H,W", CASES)
def test_resize_restatement_matches_cv2(h, w, H, W):
    cv2 = pytest.importorskip("cv2")
    from oracle import openpose_oracle as O
    rng = np.random.default_rng(h * w)
    for area in (False, True):
        if area and (H > h or W > w):
            continue
        flag = cv2.INTER_AREA if area else cv2.INTER_LANCZOS4
        u8 = rng.integers(0, 256, (h, w)).astype(np.uint8)
        assert np.array_equal(O.resize(u8, H, W, area), cv2.resize(u8, (W, H), interpolation=flag))
        f = rng.standard_normal((h, w)).astype(np.float32)
        assert np.abs(O.resize(f, H, W, area) - cv2.resize(f, (W, H), interpolation=flag)).max() <= 2e-6


def test_state_dict_layout_and_raw_cmu_keys(tmp_path):
    from pfd_b200 import openpose
    sd = openpose.BodyPose().state_dict()
    assert len(sd) == 184 and sum(v.numel() for v in sd.values()) == 52311446
    raw = {k.split(".", 1)[1]: torch.randn(v.shape) for k, v in sd.items()}      # util.transfer's source format
    p = tmp_path / "body_pose_model.pth"
    torch.save(raw, p)
    prev = openpose._network
    try:
        m = openpose.load_openpose(str(p))
        assert torch.equal(m.model3_2.Mconv4_stage3_L2.weight, raw["Mconv4_stage3_L2.weight"])
    finally:
        openpose.set_network(prev)


def test_colour_and_sine_tables():
    from pfd_b200 import openpose_tables as T
    c = T.color_table()
    assert c.shape == (35, 3) and list(c[0]) == [153, 0, 0] and list(c[17]) == [255, 0, 0]
    assert T.SIN_TABLE[90] == 1.0 and T.SIN_TABLE[1] == np.float32(0.0174524)


def test_absent_weights_raise(tmp_path, monkeypatch):
    from pfd_b200 import openpose
    prev = openpose._network
    openpose.set_network(None)
    monkeypatch.chdir(tmp_path)
    try:
        assert not openpose.available()
        with pytest.raises(NotImplementedError, match="set_network"):
            openpose.preprocess_openpose(torch.zeros((1, 3, 8, 8)))
        with pytest.raises(FileNotFoundError):
            openpose.load_openpose()
    finally:
        openpose.set_network(prev)


def _goldens():
    import os
    path = os.path.join(os.path.dirname(__file__), "golden", "openpose_outputs.npz")
    z = np.load(path)
    n = len([k for k in z.files if k.startswith("case_")])
    return z, n


def test_oracle_network_matches_reference_maps():
    from oracle import hed_oracle as HO
    from oracle import openpose_oracle as O
    z, n = _goldens()
    sd = O.synth_state_dict(0)
    for i in range(n):
        kind, seed, H, W = (int(v) for v in z[f"case_{i}"])
        if kind:
            continue
        x, _ = O.network_input(HO.hed_image(seed, H, W))
        with torch.no_grad():
            l1, l2 = O.network(sd, torch.from_numpy(x))
        assert np.abs(l1[0].numpy() - z[f"l1_{i}"]).max() <= 1e-4, f"case {i}"
        assert np.abs(l2[0].numpy() - z[f"l2_{i}"]).max() <= 1e-4, f"case {i}"


def test_oracle_decode_and_draw_reproduce_reference():
    pytest.importorskip("cv2")
    from oracle import openpose_oracle as O
    z, n = _goldens()
    for i in range(n):
        kind, seed, H, W = (int(v) for v in z[f"case_{i}"])
        h, w = O.resized_size(H, W)
        heat, paf = O.reference_maps(z[f"l1_{i}"], z[f"l2_{i}"], h, w, H, W)
        cand, subset = O.decode(heat, paf, H)
        assert np.array_equal(cand, z[f"candidate_{i}"]), f"case {i}: candidates"
        assert np.array_equal(subset, z[f"subset_{i}"]), f"case {i}: subsets"
        assert np.array_equal(O.draw(cand, subset, H, W), z[f"pre_{i}"]), f"case {i}: canvas"
        if kind:
            assert not any(O.near_ties(heat, paf, cand, subset, H, W).values()), f"case {i}: near-ties"
            assert len(subset) == 4                       # the person without a neck-nose link was merged
