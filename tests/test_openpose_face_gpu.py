"""OpenPose face annotator on the GPU (pfd_b200/openpose_face.py, csrc/openpose.cu) against the reference's goldens,
the CPU oracle and cv2."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GAIN = 0.35


@pytest.fixture(scope="module")
def nets():
    from oracle import openpose_face_oracle as FO
    from oracle import openpose_oracle as O
    from pfd_b200 import openpose, openpose_face
    prev = openpose._network, openpose_face._network
    body = openpose.BodyPose()
    body.load_state_dict(O.synth_state_dict(0), strict=True)
    face = openpose_face.FacePose()
    face.load_state_dict(FO.synth_state_dict(0, GAIN), strict=True)
    body, face = body.cuda().eval(), face.cuda().eval()
    openpose.set_network(body)
    openpose_face.set_network(face)
    yield body, face
    openpose.set_network(prev[0])
    openpose_face.set_network(prev[1])


def _goldens():
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "openpose_face_outputs.npz"))
    return z, len([k for k in z.files if k.startswith("case_")])


def _case(z, i):
    from oracle import hed_oracle as HO
    kind, image, H, W, gain = (int(v) for v in z[f"case_{i}"])
    img = HO.hed_image(90 + image, H, W)
    maps = torch.from_numpy(np.concatenate([z[f"l1_{i}"], z[f"l2_{i}"]])[None]).cuda()
    return kind, image, H, W, img, HO.image_to_tensor(img).cuda(), maps


def _u8(out):
    return (out.permute(1, 2, 0).cpu().numpy() * 255).round().astype(np.uint8)


def _ref_maps(z, i, kind, image):
    from oracle import openpose_face_oracle as FO
    if kind == 0:
        return torch.from_numpy(z[f"hs_{i}"])
    return torch.stack([FO.planted_face_maps(image)] * len(z[f"boxes_{i}"]))


def test_face_boxes_match_reference(nets):
    from pfd_b200 import openpose_face
    z, n = _goldens()
    for i in range(n):
        kind, image, H, W, _, x, maps = _case(z, i)
        _, info = openpose_face.apply(*nets, x, debug=True, body_maps=maps,
                                      face_maps=lambda inp, boxes: _ref_maps(z, i, kind, image).cuda())
        got = info["face_boxes"].numpy()
        ref = z[f"boxes_{i}"]
        assert len(got) == len(ref), f"case {i}: {len(got)} faces, reference {len(ref)}"
        assert np.array_equal(got[:, :4], np.concatenate([np.zeros((len(ref), 1), int), ref[:, :3]], 1))
        assert np.array_equal(got[:, 4], np.minimum(ref[:, 2] + ref[:, 3], H) - ref[:, 2])
        assert np.array_equal(got[:, 5], np.minimum(ref[:, 1] + ref[:, 3], W) - ref[:, 1])


def test_face_input_matches_cv2_and_tables(nets):
    """Every crop of the goldens (LANCZOS4, copy, INTER_AREA and the area-emulated bilinear) plus direct boxes."""
    from oracle import openpose_face_oracle as FO
    from pfd_b200 import native as nv
    from pfd_b200 import openpose_face
    from pfd_b200 import openpose_tables as T
    z, n = _goldens()
    seen = set()
    for i in range(n):
        _, _, H, W, img, x, _ = _case(z, i)
        boxes = [tuple(b[1:]) for b in z[f"boxes_{i}"]] + [(W - 300, H - 500, 520), (0, 0, 768), (5, 7, 100)]
        for bx, by, bw in boxes:
            ch, cw = min(by + bw, H) - by, min(bx + bw, W) - bx
            plan, tabs = openpose_face._resize(ch, cw, x.device)
            ref_plan = T.resize_plan(ch, cw, 384, 384, area=768 / (ch + cw) < 1, fixed=True)
            assert plan[0] == ref_plan[0]
            for (di, dw), (ri, rw) in zip(tabs or (), ref_plan[1:]):
                assert np.array_equal(di.cpu().numpy(), ri) and np.array_equal(dw.cpu().numpy(), rw)
            seen.add(plan[0])
            out = torch.empty((384, 384, 16), device="cuda", dtype=torch.float16)
            nv.openpose_face_input(x, 0, (bx, by, ch, cw), 384, plan, tabs, out)
            got = out[..., :3].float().permute(2, 0, 1).cpu().numpy()
            ref = FO.face_input(np.ascontiguousarray(img[:, :, ::-1]), (bx, by, bw))[1][0]
            lv = np.abs(got - ref) * 256
            assert lv.max() <= 1 and (lv == 0).mean() >= 0.999, f"{ch}x{cw} ({plan[0]}): {lv.max()} levels"
            if plan[0] in ("copy", "linear", "block"):
                assert (lv == 0).all(), f"{ch}x{cw} ({plan[0]})"
            assert (out[..., 3:] == 0).all()
    assert seen >= {"copy", "sep", "linear", "block"}


def test_network_matches_fp32_oracle(nets):
    from oracle import openpose_face_oracle as FO
    z, _ = _goldens()
    _, _, H, W, img, _, _ = _case(z, 1)
    bgr = np.ascontiguousarray(img[:, :, ::-1])
    x = np.concatenate([FO.face_input(bgr, b[1:])[1] for b in z["boxes_1"]])
    inp = torch.zeros((len(x), 384, 384, 16), dtype=torch.float16)
    inp[..., :3] = torch.from_numpy(x).permute(0, 2, 3, 1).half()
    got = nets[1].network(inp.cuda()).cpu()
    with torch.no_grad():
        ref = FO.network(FO.synth_state_dict(0, GAIN), torch.from_numpy(x))
    rel = ((got - ref).pow(2).mean() / ref.pow(2).mean()).sqrt().item()
    assert rel < 5e-3, f"stage-6 face maps rel rms {rel:.3e}"


def test_landmarks_and_canvas_exact_on_reference_maps(nets):
    """Given the reference's body maps and hs[-1] (or the planted face maps), the landmarks and the canvas equal the
    reference's, except where the oracle reports a near-tie."""
    from oracle import openpose_face_oracle as FO
    from pfd_b200 import openpose_face
    z, n = _goldens()
    for i in range(n):
        kind, image, H, W, _, x, maps = _case(z, i)
        hs = _ref_maps(z, i, kind, image)
        out, info = openpose_face.apply(*nets, x, debug=True, body_maps=maps, face_maps=lambda inp, b: hs.cuda())
        lmk = info["face_landmarks"].cpu().numpy()
        ties = 0
        for f, (p, bx, by, bw) in enumerate(z[f"boxes_{i}"]):
            near = FO.near_ties(FO.heatmaps(hs[f].numpy(), min(by + bw, H) - by, min(bx + bw, W) - bx))
            ties += len(near)
            keep = np.setdiff1d(np.arange(71), near)
            assert np.array_equal(lmk[f, keep], z[f"lmk_{i}"][f, keep]), f"case {i} face {f}: landmarks"
        if ties == 0:
            ours = _u8(out[0])
            assert np.array_equal(ours, z[f"pre_{i}"]), f"case {i}: {(ours != z[f'pre_{i}']).any(2).sum()} pixels"


def test_dots_match_cv2_on_random_landmarks(nets):
    """Random landmarks on random canvas sizes: the float32 round trip int(float32((p + x) / W) * W), which lands one
    pixel short for a few percent of positions, the -1 rule at crop row / column 0, and border clipping."""
    import cv2
    from oracle import openpose_face_oracle as FO
    from pfd_b200 import native as nv
    from pfd_b200 import openpose_face
    rng = np.random.default_rng(11)
    short = 0
    for trial in range(12):
        H, W = (int(v) for v in rng.integers(64, 700, 2))
        nf = 3
        boxes = np.zeros((nf, 6), np.int32)
        lmk = np.zeros((nf, 71, 2), np.int32)
        ref = np.zeros((H, W, 3), np.uint8)
        for f in range(nf):
            bw = int(rng.integers(20, min(H, W)))
            bx, by = int(rng.integers(0, W - 10)), int(rng.integers(0, H - 10))
            ch, cw = min(by + bw, H) - by, min(bx + bw, W) - bx
            boxes[f] = (0, 0, bx, by, ch, cw)
            lmk[f] = np.stack([rng.integers(0, cw, 71), rng.integers(0, ch, 71)], 1)
            lmk[f, :3] = 0
            lmk[f, 3] = -1
            for px, py in FO.landmarks_to_pixels(lmk[f], (bx, by, bw), H, W):
                cv2.circle(ref, (px, py), 3, (255, 255, 255), thickness=-1)
            v = (lmk[f, 4:, 0] + bx).astype(np.float32)
            short += int(((v / np.float32(W)).astype(np.float32) * np.float32(W)).astype(np.int64).__ne__(v).sum())
        persons = torch.full((1, nv.PFD_OPENPOSE_MAX_PERSONS, 18), -1, dtype=torch.int32, device="cuda")
        npers = torch.ones((1,), dtype=torch.int32, device="cuda")
        xy = torch.zeros((1, 18, nv.PFD_OPENPOSE_MAX_PEAKS, 2), dtype=torch.int32, device="cuda")
        P = nets[0]._plans(H, W, torch.device("cuda"))
        out = nv.openpose_face_draw(persons, npers, xy, H, W, P["sintab"], openpose_face._color_table("cuda"),
                                    torch.from_numpy(boxes).cuda(), torch.from_numpy(lmk).cuda(), nf)
        ours = _u8(out[0])
        assert np.array_equal(ours, ref), f"trial {trial} ({H}x{W}): {(ours != ref).any(2).sum()} pixels differ"
    assert short > 0                       # the one-pixel-short round trip occurred


def test_end_to_end_synthetic_facenet(nets, ctl):
    from pfd_b200 import openpose_face
    z, _ = _goldens()
    kind, image, H, W, _, x, maps = _case(z, 0)
    out, info = openpose_face.apply(*nets, x, debug=True, body_maps=maps)
    lmk = info["face_landmarks"].cpu().numpy()
    ref = z["lmk_0"]
    both = (lmk[..., 0] >= 0) & (ref[..., 0] >= 0)
    close = (np.abs(lmk - ref).max(-1) <= 1) & both
    fa = close.sum() / max((ref[..., 0] >= 0).sum(), 1)
    fb = close.sum() / max((lmk[..., 0] >= 0).sum(), 1)
    eq = (_u8(out[0]) == z["pre_0"]).all(2).mean()
    print(f"[face e2e] landmarks within 1 px {fa:.4f} / {fb:.4f}, canvas pixels equal {eq:.5f}")
    assert fa >= 0.99 and fb >= 0.99, f"landmarks matched {fa:.4f} / {fb:.4f}"
    assert eq >= 0.99, f"{eq:.4f} of canvas pixels equal"


@pytest.fixture(scope="module")
def ctl():
    from pfd_b200.controlnet import ControlNet
    return ControlNet(32, 4, 32, 3, 1, [], channel_mult=(1,), use_spatial_transformer=True, context_dim=32,
                      num_heads=1, legacy=False).cuda()


def test_batch_equals_single_zero_faces_and_dispatch(nets, ctl):
    import pfd_b200
    from pfd_b200 import native as nv
    from pfd_b200 import openpose_face
    z, _ = _goldens()
    xs, ms = [], []
    for i in (0, 1):
        _, _, H, W, _, x, maps = _case(z, i)
        xs.append(x)
        ms.append(maps)
    was = nv.deterministic()
    pfd_b200.set_deterministic(True)
    try:
        both = openpose_face.apply(*nets, torch.cat(xs), body_maps=torch.cat(ms))
        for k in range(2):
            one = openpose_face.apply(*nets, xs[k], body_maps=ms[k])
            assert torch.equal(both[k], one[0]), f"image {k}: batch differs from single"
        # the public entry runs the same pipeline on the network's own body maps
        x = xs[0][..., :384, :512].contiguous()
        assert torch.equal(ctl.preprocess(x, type="openpose_withface_v11p"), openpose_face.apply(*nets, x))
    finally:
        pfd_b200.set_deterministic(was)
    # no nose anywhere: no face box, and the canvas is exactly the body annotator's
    nonose = ms[1].clone()
    nonose[:, 38] = 0
    out, info = openpose_face.apply(*nets, xs[1], debug=True, body_maps=nonose)
    assert len(info["face_boxes"]) == 0 and int(info["npersons"][0]) > 0
    assert torch.equal(out, nets[0].apply(xs[1], maps=nonose))


def test_capture_raises(nets):
    from pfd_b200 import openpose_face
    x = torch.rand((1, 3, 184, 184), device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="CUDA graph"):
        with torch.cuda.graph(g, stream=s):
            openpose_face.preprocess_openpose_face(x)
