"""HED soft-edge annotator, CPU side: the oracle (oracle/hed_oracle.py) against the reference's outputs in
tests/golden/hed_outputs.npz and against cv2.resize, and the parameter layout / loader of pfd_b200.hed."""
import json
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _golden():
    return np.load(os.path.join(GOLDEN, "hed_outputs.npz"))


def _cases(z):
    i = 0
    while f"case_{i}" in z:
        yield i, [int(v) for v in z[f"case_{i}"]]
        i += 1


def test_oracle_reproduces_reference_outputs():
    from oracle import hed_oracle as O
    z = _golden()
    sd = O.synth_state_dict(0)
    n = 0
    for i, (seed, H, W) in _cases(z):
        u8, pre, sides = O.apply_hed(sd, O.hed_image(seed, H, W))
        for k, s in enumerate(sides):
            st = int(z[f"side_{i}_{k}_stride"])
            assert tuple(s.shape) == tuple(z[f"side_{i}_{k}_shape"])
            ref = z[f"side_{i}_{k}"]
            got = s[::st, ::st]
            rel = np.sqrt(np.mean((got - ref) ** 2) / np.mean(ref ** 2))
            assert rel <= 1e-4, f"case {i} side {k}: rel rms {rel:.2e}"
        ref_u8 = z[f"u8_{i}"]
        differ = (u8 != ref_u8) & ~O.near_integer(pre)
        assert u8.shape == (H, W) and not differ.any(), f"case {i}: {int(differ.sum())} uint8 levels differ"
        n += 1
    assert n == 3


@pytest.mark.parametrize("src,dst", [((17, 13), (131, 97)), ((13, 17), (97, 131)), ((2, 3), (33, 31)),
                                     ((16, 16), (256, 256)), ((8, 8), (33, 31)), ((1, 1), (5, 7)),
                                     ((33, 31), (33, 31)), ((64, 80), (64, 80))])
def test_resize_matches_cv2(src, dst):
    cv2 = pytest.importorskip("cv2")
    from oracle.hed_oracle import resize_linear
    s = np.random.RandomState(sum(src) + sum(dst)).randn(*src).astype(np.float32) * 7
    ref = cv2.resize(s, (dst[1], dst[0]), interpolation=cv2.INTER_LINEAR)
    out = resize_linear(s, *dst)
    assert out.dtype == np.float32 and out.shape == ref.shape
    assert np.abs(out - ref).max() <= 1e-6 * np.abs(ref).max()
    if src == dst:
        assert np.array_equal(out, ref)


def test_state_dict_layout_matches_reference():
    from oracle.hed_oracle import state_dict_shapes
    from pfd_b200.hed import ControlNetHED
    ours = {k: list(v.shape) for k, v in ControlNetHED().state_dict().items()}
    with open(os.path.join(GOLDEN, "hed_state_dict_shapes.json")) as f:
        table = json.load(f)
    assert ours == table and list(ours) == list(table)
    assert ours == {k: list(v) for k, v in state_dict_shapes().items()}
    from tools import ref_harness
    if ref_harness.available():
        cwd = os.getcwd()
        try:
            ref_harness.import_reference()
            import lib.model_zoo.controlnet_annotator.hed as refhed
            ref = {k: list(v.shape) for k, v in refhed.ControlNetHED_Apache2().state_dict().items()}
        finally:
            os.chdir(cwd)
        assert ours == ref


def test_load_hed_missing_file_raises_without_download(tmp_path, monkeypatch):
    from pfd_b200 import hed
    import torch.hub

    def no_download(*a, **k):
        raise AssertionError("load_hed tried to download")
    monkeypatch.setattr(torch.hub, "download_url_to_file", no_download)
    saved = hed._network
    try:
        with pytest.raises(FileNotFoundError, match="missing.pth"):
            hed.load_hed(str(tmp_path / "missing.pth"))
        monkeypatch.chdir(tmp_path)
        hed.set_network(None)
        with pytest.raises(FileNotFoundError, match="ControlNetHED.pth"):
            hed.get_network()
    finally:
        hed.set_network(saved)


def test_load_hed_strict_round_trip(tmp_path):
    from oracle.hed_oracle import synth_state_dict
    from pfd_b200 import hed
    import safetensors.torch
    sd = synth_state_dict(3)
    # the forms every annotator loader accepts: plain, a 'state_dict' with 'module.' keys, safetensors
    wrapped, st = str(tmp_path / "wrapped.pth"), str(tmp_path / "ControlNetHED.safetensors")
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, wrapped)
    safetensors.torch.save_file({k: v.contiguous() for k, v in sd.items()}, st)
    path = str(tmp_path / "ControlNetHED.pth")
    torch.save(sd, path)
    saved = hed._network
    try:
        for p in (path, wrapped, st):
            m = hed.load_hed(p)
            assert hed.get_network() is m
            for k, v in m.state_dict().items():
                assert torch.equal(v, sd[k])
        sd.pop("norm")
        torch.save(sd, path)
        with pytest.raises(RuntimeError):
            hed.load_hed(path)
    finally:
        hed.set_network(saved)

