"""M-LSD annotator, CPU side: the oracle (oracle/mlsd_oracle.py) against the reference's outputs in
tests/golden/mlsd_outputs.npz, its line rasteriser against cv2.line, the size rule, BN folding, and the parameter
layout / loader / absent-weights behaviour of pfd_b200.mlsd."""
import json
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _cases(z):
    i = 0
    while f"case_{i}" in z:
        yield i, [int(v) for v in z[f"case_{i}"]], [float(v) for v in z[f"thr_{i}"]]
        i += 1


def _rows(a):
    return sorted(map(tuple, np.asarray(a).reshape(-1, 4).tolist()))


def test_oracle_reproduces_reference_outputs():
    from oracle import hed_oracle as HO
    from oracle import mlsd_oracle as O
    z = np.load(os.path.join(GOLDEN, "mlsd_outputs.npz"))
    sd = O.synth_state_dict(0)
    n = zeros = 0
    for i, (seed, H, W), (thr_v, thr_d) in _cases(z):
        img = np.ascontiguousarray(HO.hed_image(seed, H, W))
        lines, segs, maps = O.apply_mlsd(sd, img, thr_v, thr_d)
        assert np.array_equal(z[f"pre_{i}"], z[f"lines_{i}"]), f"case {i}: reference preprocess != apply_mlsd"
        if maps is None:
            assert f"maps_{i}" not in z and not z[f"lines_{i}"].any() and not lines.any()
            zeros += 1
        else:
            ref = z[f"maps_{i}"]
            assert maps.shape == ref.shape == (5, H // 2, W // 2)
            err = np.abs(maps - ref).max() / np.abs(ref).max()
            assert err <= 1e-5, f"case {i}: map error {err:.2e}"
            # exactness of the decode and the drawing, on the reference's own maps
            assert O.decode(ref, thr_v, thr_d).tolist() == z[f"segs_{i}"].tolist(), f"case {i}: segments"
            assert np.array_equal(O.draw_lines(H, W, z[f"segs_{i}"]), z[f"lines_{i}"]), f"case {i}: line map"
            assert _rows(segs) == _rows(z[f"segs_{i}"]), f"case {i}: segments from the oracle's own map"
            assert np.array_equal(lines, z[f"lines_{i}"]), f"case {i}: line map from the oracle's own map"
        n += 1
    assert n == 7 and zeros == 2


def test_goldens_exercise_every_decision():
    """The synthetic gains make every step of the decode matter on the golden images."""
    from oracle import mlsd_oracle as O
    z = np.load(os.path.join(GOLDEN, "mlsd_outputs.npz"))
    over_topk = below = long_outside = thr_d_cut = 0
    for i, (seed, H, W), (thr_v, thr_d) in _cases(z):
        if f"maps_{i}" not in z:
            continue
        heat = O.heat_map(z[f"maps_{i}"][0])
        over_topk += (heat > np.float32(thr_v)).sum() > O.TOPK
        below += ((heat > 0) & (heat <= np.float32(thr_v))).sum() > 0
        s = z[f"segs_{i}"]
        length = np.hypot(s[:, 2] - s[:, 0], s[:, 3] - s[:, 1])
        out = ((s[:, [0, 2]] < 0) | (s[:, [0, 2]] >= W) | (s[:, [1, 3]] < 0) | (s[:, [1, 3]] >= H)).any(1)
        long_outside += int(((length >= 20) & out).sum())
        thr_d_cut += len(s) < min(O.TOPK, int((heat > np.float32(thr_v)).sum()))
    assert over_topk >= 1 and below >= 1 and long_outside >= 100 and thr_d_cut >= 1


def test_line_oracle_equals_cv2():
    cv2 = pytest.importorskip("cv2")
    from oracle.mlsd_oracle import draw_lines, random_segments
    H, W = 64, 80
    segs = random_segments(12000, H, W)
    for s in segs:
        img = np.zeros((H, W, 3), np.uint8)
        cv2.line(img, (int(s[0]), int(s[1])), (int(s[2]), int(s[3])), [255, 255, 255], 1)
        assert np.array_equal(draw_lines(H, W, s[None]), img[:, :, 0]), f"segment {s.tolist()}"
        rev = np.zeros((H, W, 3), np.uint8)
        cv2.line(rev, (int(s[2]), int(s[3])), (int(s[0]), int(s[1])), [255, 255, 255], 1)
        assert np.array_equal(draw_lines(H, W, s[None, [2, 3, 0, 1]]), rev[:, :, 0]), f"reversed {s.tolist()}"


@pytest.mark.parametrize("H,W", [(512, 512), (256, 384), (33, 48), (257, 176), (200, 168), (97, 131), (16, 32),
                                 (32, 32), (17, 240), (16, 224), (31, 64), (34, 64)])
def test_size_rule_predicts_reference_failures(H, W):
    """pfd_b200.mlsd.size_supported and the oracle's agree with whether the reference network + topk run."""
    from oracle import mlsd_oracle as O
    from pfd_b200.mlsd import size_supported
    from tools import ref_harness
    if not ref_harness.available():
        pytest.skip("reference tree not staged (build() stages it under oracle/_ref)")
    ref_harness.import_reference()
    from lib.model_zoo.controlnet_annotator.mlsd.models.mbv2_mlsd_large import MobileV2_MLSD_Large
    torch.manual_seed(0)
    net = MobileV2_MLSD_Large().eval()
    x = torch.zeros((1, 4, H, W))
    try:
        with torch.no_grad():
            out = net(x)
        torch.topk(torch.sigmoid(out[:, 0]).reshape(-1), O.TOPK)
        ran = True
    except Exception:
        ran = False
    assert size_supported(H, W) == O.size_supported(H, W) == ran


def test_bn_folding_matches_reference_modules():
    """fold_bn (ours and the oracle's) equals Conv2d -> BatchNorm2d(eval) in float64."""
    from oracle.mlsd_oracle import fold_bn as oracle_fold
    from pfd_b200.mlsd import MLSD, fold_bn
    g = torch.Generator().manual_seed(3)
    for cout, cin, k, bias in ((32, 4, 3, False), (64, 128, 3, True), (24, 96, 1, False)):
        conv = torch.nn.Conv2d(cin, cout, k, padding=k // 2, bias=bias).double()
        bn = torch.nn.BatchNorm2d(cout).double().eval()
        with torch.no_grad():
            for t in (bn.weight, bn.bias, bn.running_mean):
                t.copy_(torch.randn(cout, generator=g, dtype=torch.float64))
            bn.running_var.copy_(0.2 + torch.rand(cout, generator=g, dtype=torch.float64))
        x = torch.randn((2, cin, 7, 9), generator=g, dtype=torch.float64)
        ref = bn(conv(x))
        sd = {"c.weight": conv.weight.detach(), "b.weight": bn.weight.detach(), "b.bias": bn.bias.detach(),
              "b.running_mean": bn.running_mean, "b.running_var": bn.running_var}
        if bias:
            sd["c.bias"] = conv.bias.detach()
        w, b = oracle_fold(sd, "c", "b")
        y = torch.nn.functional.conv2d(x, w, b, padding=k // 2)
        assert torch.allclose(y, ref, rtol=0, atol=1e-12)
        w32, b32 = fold_bn(conv.float(), bn.float())
        y32 = torch.nn.functional.conv2d(x, w32.double(), b32.double(), padding=k // 2)
        assert torch.allclose(y32, ref, rtol=1e-5, atol=1e-5)
    assert isinstance(MLSD(), torch.nn.Module)


def test_state_dict_layout_matches_reference():
    from oracle.mlsd_oracle import state_dict_shapes
    from pfd_b200.mlsd import MLSD
    m = MLSD()
    ours = {k: list(v.shape) for k, v in m.state_dict().items()}
    with open(os.path.join(GOLDEN, "mlsd_state_dict_shapes.json")) as f:
        table = json.load(f)
    assert ours == table and list(ours) == list(table)
    assert len(ours) == 362 and sum(p.numel() for p in m.parameters()) == 1533680
    assert ours == {k: list(v) for k, v in state_dict_shapes().items()}


def _write(tmp_path, sd, name, kind):
    path = str(tmp_path / name)
    if kind == "safetensors":
        import safetensors.torch
        safetensors.torch.save_file({k: v.contiguous() for k, v in sd.items()}, path)
    elif kind == "wrapped":
        torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, path)
    else:
        torch.save(sd, path)
    return path


@pytest.mark.parametrize("kind", ["pth", "wrapped", "safetensors"])
def test_load_mlsd_checkpoint_forms(tmp_path, kind):
    from oracle.mlsd_oracle import synth_state_dict
    from pfd_b200 import mlsd
    sd = synth_state_dict(3)
    path = _write(tmp_path, sd, "mlsd_large_512_fp32." + ("safetensors" if kind == "safetensors" else "pth"), kind)
    saved = mlsd._network
    try:
        m = mlsd.load_mlsd(path)
        assert mlsd.get_network() is m
        for k, v in m.state_dict().items():
            assert torch.equal(v, sd[k])
        sd.pop("block23.conv3.bias")
        with pytest.raises(RuntimeError):
            mlsd.load_mlsd(_write(tmp_path, sd, "broken." + ("safetensors" if kind == "safetensors" else "pth"), kind))
    finally:
        mlsd.set_network(saved)


def test_absent_weights(tmp_path, monkeypatch):
    from pfd_b200 import mlsd
    import torch.hub

    def no_download(*a, **k):
        raise AssertionError("tried to download")
    monkeypatch.setattr(torch.hub, "download_url_to_file", no_download)
    monkeypatch.chdir(tmp_path)
    saved = mlsd._network
    try:
        mlsd.set_network(None)
        assert not mlsd.available()
        with pytest.raises(FileNotFoundError, match="missing.pth"):
            mlsd.load_mlsd(str(tmp_path / "missing.pth"))
        with pytest.raises(FileNotFoundError, match="mlsd_large_512_fp32.pth"):
            mlsd.get_network()
        with pytest.raises(NotImplementedError) as e:
            mlsd.preprocess_mlsd(torch.rand((1, 3, 32, 32)))
        msg = str(e.value)
        assert mlsd.DEFAULT_PATH in msg and "pfd_b200.mlsd.load_mlsd" in msg and "set_network" in msg
    finally:
        mlsd.set_network(saved)
