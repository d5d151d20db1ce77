"""PiDiNet annotator, CPU side: the oracle (oracle/pidinet_oracle.py) against the reference's outputs in
tests/golden/pidinet_outputs.npz and against torch, the PDC weight conversions, and the parameter layout / loader /
absent-weights behaviour of pfd_b200.pidinet."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _cases(z):
    i = 0
    while f"case_{i}" in z:
        yield i, [int(v) for v in z[f"case_{i}"]]
        i += 1


def test_oracle_reproduces_reference_outputs():
    from oracle import hed_oracle as HO
    from oracle import pidinet_oracle as O
    z = np.load(os.path.join(GOLDEN, "pidinet_outputs.npz"))
    sd = O.synth_state_dict(0)
    n = 0
    for i, (seed, H, W) in _cases(z):
        img = HO.hed_image(seed, H, W)
        sides, acts = O.network_sides(sd, img, return_acts=True)
        # fp16 headroom of the GPU path: every block output of the network stays small on these images
        assert max(acts) < 8, f"case {i}: block output magnitude {max(acts)}"
        for k, s in enumerate(sides):
            st = int(z[f"side_{i}_{k}_stride"])
            assert tuple(s.shape) == tuple(z[f"side_{i}_{k}_shape"])
            ref = z[f"side_{i}_{k}"]
            got = s[::st, ::st]
            rel = np.sqrt(np.mean((got - ref) ** 2) / np.mean(ref ** 2))
            assert rel <= 1e-5, f"case {i} side {k}: rel rms {rel:.2e}"
        u8, pre = O.fuse(sd, sides, H, W)
        ref_u8 = z[f"u8_{i}"]
        differ = (u8 != ref_u8) & ~O.near_integer(pre)
        assert u8.shape == (H, W) and not differ.any(), f"case {i}: {int(differ.sum())} uint8 levels differ"
        inner = float(((ref_u8 > 0) & (ref_u8 < 255)).mean())
        assert inner >= 0.3 and int(ref_u8.max()) - int(ref_u8.min()) >= 150, f"case {i}: uninformative levels"
        n += 1
    assert n == 4


@pytest.mark.parametrize("op", ["cv", "cd", "ad", "rd"])
def test_pdc_conversion_equals_pixel_difference_form(op):
    from oracle import pidinet_oracle as O
    from pfd_b200.pidinet import convert_pdc
    g = torch.Generator().manual_seed(7)
    for C, H, W in ((6, 9, 11), (3, 5, 4)):
        x = torch.randn((2, C, H, W), generator=g, dtype=torch.float64)
        w = torch.randn((C, 1, 3, 3), generator=g, dtype=torch.float64)
        ref = O.pdc_reference_form(op, x, w)
        for conv in (O.convert_pdc, convert_pdc):
            k = conv(op, w)
            assert k.shape[-1] == (5 if op == "rd" else 3)
            y = F.conv2d(x, k, padding=k.shape[-1] // 2, groups=C)
            assert torch.allclose(y, ref, rtol=0, atol=1e-12), f"{op}: {(y - ref).abs().max().item():.2e}"
        assert torch.equal(O.convert_pdc(op, w), convert_pdc(op, w))


@pytest.mark.parametrize("src,dst", [((17, 13), (131, 97)), ((25, 21), (200, 168)), ((8, 8), (256, 256)),
                                     ((64, 80), (512, 640)), ((12, 16), (97, 131)), ((50, 42), (200, 168)),
                                     ((96, 80), (768, 640)), ((33, 31), (33, 31))])
def test_bilinear_rule_matches_torch_bit_for_bit(src, dst):
    from oracle.pidinet_oracle import resize_bilinear
    s = np.random.RandomState(sum(src) + sum(dst)).randn(*src).astype(np.float32)
    ref = F.interpolate(torch.from_numpy(s)[None, None], dst, mode="bilinear", align_corners=False)[0, 0].numpy()
    out = resize_bilinear(s, *dst)
    assert out.dtype == np.float32 and out.shape == ref.shape and np.array_equal(out, ref)


@pytest.mark.parametrize("src,dst", [((4, 4), (33, 31)), ((8, 8), (64, 64)), ((2, 3), (8, 9))])
def test_bilinear_rule_small_outputs_within_ulps(src, dst):
    """PyTorch takes another CPU path for H + W <= 128; the values agree to float32 rounding."""
    from oracle.pidinet_oracle import resize_bilinear
    s = np.random.RandomState(sum(src) + sum(dst)).randn(*src).astype(np.float32)
    ref = F.interpolate(torch.from_numpy(s)[None, None], dst, mode="bilinear", align_corners=False)[0, 0].numpy()
    assert np.abs(resize_bilinear(s, *dst) - ref).max() <= 4e-7 * np.abs(s).max()


def test_state_dict_layout_matches_reference():
    from oracle.pidinet_oracle import state_dict_shapes
    from pfd_b200.pidinet import PiDiNet
    ours = {k: list(v.shape) for k, v in PiDiNet().state_dict().items()}
    with open(os.path.join(GOLDEN, "pidinet_state_dict_shapes.json")) as f:
        table = json.load(f)
    assert ours == table and list(ours) == list(table)
    assert len(ours) == 83 and sum(int(np.prod(s)) for s in ours.values()) == 710149
    assert ours == {k: list(v) for k, v in state_dict_shapes().items()}


def test_cdcm_fragment_packing():
    """pack_cdcm puts W_d[n, c, ky, kx] where pfd_pidinet_cdcm_f16's lanes read it."""
    from pfd_b200.pidinet import pack_cdcm
    ws = [torch.randn((24, 24, 3, 3)) for _ in range(4)]
    pk = pack_cdcm(ws).float()
    for s, j, lane, e in ((0, 0, 0, 0), (53, 2, 31, 3), (1, 1, 17, 2), (26, 0, 5, 1), (40, 2, 9, 2)):
        g, t = lane // 4, lane % 4
        krow = 16 * s + (8 if e >= 2 else 0) + 2 * t + (e % 2)
        tap, c = krow // 24, krow % 24
        d, t9 = tap // 9, tap % 9
        assert pk[s, j, lane, e] == ws[d][8 * j + g, c, t9 // 3, t9 % 3].half().float()


def _write(tmp_path, sd, name, kind):
    path = str(tmp_path / name)
    if kind == "safetensors":
        import safetensors.torch
        safetensors.torch.save_file({k: v.contiguous() for k, v in sd.items()}, path)
    else:
        torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, path)
    return path


@pytest.mark.parametrize("kind", ["pth", "safetensors"])
def test_load_pidinet_checkpoint_forms(tmp_path, kind):
    from oracle.pidinet_oracle import synth_state_dict
    from pfd_b200 import pidinet
    sd = synth_state_dict(3)
    path = _write(tmp_path, sd, "table5_pidinet." + kind, kind)
    saved = pidinet._network
    try:
        m = pidinet.load_pidinet(path)
        assert pidinet.get_network() is m
        for k, v in m.state_dict().items():
            assert torch.equal(v, sd[k])
        sd.pop("classifier.bias")
        with pytest.raises(RuntimeError):
            pidinet.load_pidinet(_write(tmp_path, sd, "broken." + kind, kind))
    finally:
        pidinet.set_network(saved)


def test_absent_weights(tmp_path, monkeypatch):
    from pfd_b200 import pidinet
    from pfd_b200.scribble import preprocess_scribble
    import torch.hub

    def no_download(*a, **k):
        raise AssertionError("tried to download")
    monkeypatch.setattr(torch.hub, "download_url_to_file", no_download)
    monkeypatch.chdir(tmp_path)
    saved = pidinet._network
    try:
        pidinet.set_network(None)
        with pytest.raises(FileNotFoundError, match="missing.pth"):
            pidinet.load_pidinet(str(tmp_path / "missing.pth"))
        with pytest.raises(FileNotFoundError, match="table5_pidinet.pth"):
            pidinet.get_network()
        x = torch.rand((1, 3, 16, 16))
        for kw in ({}, {"method": "pidinet"}):
            with pytest.raises(NotImplementedError, match="method='hed'.*method='xdog'") as e:
                preprocess_scribble(x, **kw)
            msg = str(e.value)
            assert pidinet.DEFAULT_PATH in msg and "pfd_b200.pidinet.load_pidinet" in msg and "set_network" in msg
        with pytest.raises(ValueError):
            preprocess_scribble(x, method="canny")
    finally:
        pidinet.set_network(saved)
