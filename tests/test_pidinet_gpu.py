"""PiDiNet annotator on the GPU (ControlNet.preprocess type 'scribble', default method 'pidinet'): the fp16 network
against the fp32 oracle (oracle/pidinet_oracle.py) and the reference's outputs (tests/golden), batch invariance, graph
capture and weight swaps.

The bounds are HED's, set before anything was measured.  Measured on an H100 80GB HBM3 with the synthetic weights:
per-stage side maps within 4.1e-3 relative rms of the oracle (bound 5e-3); levels max |d| 1, mean |d| <= 0.17, 100 %
within 1, against both the oracle and the reference's maps; end-to-end scribble flips 0 %, 0.17 %, 0.08 % and 0.24 %
of the pixels on the four golden cases (33x31, 97x131, 200x168, 256x256; bound 1 %)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fp32_oracle():
    """The oracle runs its convolutions on the GPU in true fp32 (no TF32)."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.fixture(scope="module")
def pidi_net():
    """Installs the synthetic network for this module and restores whatever was installed before (the scribble and
    HED tests that run later expect no PiDiNet network)."""
    from oracle.pidinet_oracle import fill_synthetic
    from pfd_b200 import pidinet
    m = fill_synthetic(pidinet.PiDiNet().cuda(), seed=0)
    saved = pidinet._network
    pidinet.set_network(m)
    yield m
    pidinet.set_network(saved)


@pytest.fixture(scope="module")
def ctl():
    """A small ControlNet: preprocess does not depend on the ControlNet's own size."""
    from pfd_b200.controlnet import ControlNet
    return ControlNet(32, 4, 32, 3, 1, [], channel_mult=(1,), use_spatial_transformer=True, context_dim=32,
                      num_heads=1, legacy=False).cuda()


def _image(shape, dtype):
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.rand(shape, generator=g)
    x = 0.5 * F.avg_pool2d(x, 9, 1, 4) + 0.5 * F.avg_pool2d(x, 3, 1, 1)
    return ((x - x.min()) / (x.max() - x.min())).to(dtype)


def _levels(out):
    return (out[:, 0].double() * 255).round().to(torch.int64).cpu().numpy()


def _check_levels(lv, ref, what):
    d = np.abs(lv.astype(np.int64) - ref.astype(np.int64))
    inner = float(((ref > 0) & (ref < 255)).mean())
    print(f"[pidinet] {what}: max |d| {d.max()}, mean |d| {d.mean():.4f}, within 1: {(d <= 1).mean():.4%}, "
          f"unsaturated {inner:.1%}")
    assert inner >= 0.30, f"{what}: only {inner:.1%} of pixels strictly between 0 and 255"
    assert d.max() <= 3 and d.mean() <= 0.25 and (d <= 1).mean() >= 0.99, what


def _rel_rms(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.sqrt(np.mean((a - b) ** 2) / np.mean(b ** 2)))


SHAPES = [((1, 3, 512, 512), torch.float16), ((2, 3, 131, 97), torch.float32), ((1, 3, 768, 640), torch.float32),
          ((1, 3, 33, 31), torch.float16), ((1, 3, 8, 8), torch.float32)]


@pytest.mark.parametrize("shape,dtype", SHAPES)
def test_pidinet_matches_oracle(pidi_net, fp32_oracle, shape, dtype):
    from oracle import hed_oracle as HO
    from oracle import pidinet_oracle as O
    x = _image(shape, dtype).cuda()
    out, sides = pidi_net.apply(x, return_sides=True)
    B, _, H, W = shape
    assert out.dtype == torch.float32 and out.is_cuda and out.shape == (B, 3, H, W)
    assert torch.equal(out[:, 0], out[:, 1]) and torch.equal(out[:, 0], out[:, 2])
    sd = {k: v.detach().cpu() for k, v in pidi_net.state_dict().items()}
    lv = _levels(out)
    for b in range(B):
        ref_u8, _, ref_sides = O.apply_pidinet(sd, HO.to_pil_u8(x[b]), device="cuda")
        rels = [_rel_rms(s[b].cpu().numpy(), r) for s, r in zip(sides, ref_sides)]
        print(f"[pidinet] {tuple(shape)} image {b}: side rel rms {['%.2e' % r for r in rels]}")
        assert max(rels) <= 5e-3, f"image {b}: side rel rms {rels}"
        _check_levels(lv[b], ref_u8, f"{tuple(shape)} {dtype} image {b}")


def test_golden_reference_outputs(pidi_net, ctl):
    from oracle import hed_oracle as HO
    z = np.load(os.path.join(ROOT, "tests", "golden", "pidinet_outputs.npz"))
    i = 0
    while f"case_{i}" in z:
        seed, H, W = (int(v) for v in z[f"case_{i}"])
        x = HO.image_to_tensor(HO.hed_image(seed, H, W)).cuda()
        from pfd_b200.pidinet import preprocess_pidinet
        _check_levels(_levels(preprocess_pidinet(x))[0], z[f"u8_{i}"], f"golden {H}x{W}")
        scr = ctl.preprocess(x, type="scribble")
        assert torch.equal(ctl.preprocess(x, type="scribble", method="pidinet"), scr)
        got = (scr[0, 0].cpu().numpy() * 255).round().astype(np.uint8)
        flips = float((got != z[f"scribble_{i}"]).mean())
        print(f"[pidinet] golden scribble {H}x{W}: {flips:.3%} of pixels flipped")
        assert flips <= 0.01, f"{H}x{W}: {flips:.3%} of scribble pixels differ"
        i += 1
    assert i == 4


def test_scribble_output_contract(pidi_net, ctl):
    x = _image((2, 3, 96, 120), torch.float16).cuda()
    out = ctl.preprocess(x, type="scribble")
    assert out.dtype == torch.float32 and out.shape == (2, 3, 96, 120)
    assert torch.equal(out[:, 0], out[:, 1]) and torch.equal(out[:, 0], out[:, 2])
    assert set(torch.unique(out).tolist()) <= {0.0, 1.0}
    assert torch.equal(ctl.preprocess(x, type="scribble", method="pidinet"), out)


def test_batch_equals_single_in_deterministic_mode(pidi_net, ctl):
    import pfd_b200
    from pfd_b200 import native as nv
    was = nv.deterministic()
    pfd_b200.set_deterministic(True)
    try:
        x = _image((3, 3, 72, 88), torch.float32).cuda()
        batch = ctl.preprocess(x, type="scribble")
        lv = pidi_net.apply(x)
        for b in range(3):
            assert torch.equal(ctl.preprocess(x[b:b + 1], type="scribble"), batch[b:b + 1]), f"sample {b}"
            assert torch.equal(pidi_net.apply(x[b:b + 1]), lv[b:b + 1]), f"sample {b} levels"
    finally:
        pfd_b200.set_deterministic(was)


def test_graph_capture_equals_eager(pidi_net, ctl):
    x = _image((2, 3, 96, 80), torch.float16).cuda()
    eager = ctl.preprocess(x, type="scribble")
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ctl.preprocess(x, type="scribble")                             # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ctl.preprocess(x, type="scribble")
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_weight_swap_repacks(pidi_net, fp32_oracle):
    from oracle import hed_oracle as HO
    from oracle import pidinet_oracle as O
    x = _image((1, 3, 120, 136), torch.float32).cuda()
    a = pidi_net.apply(x)
    old = {k: v.clone() for k, v in pidi_net.state_dict().items()}
    try:
        sd2 = O.synth_state_dict(2)
        pidi_net.load_state_dict({k: v.cuda() for k, v in sd2.items()}, strict=True)
        b = pidi_net.apply(x)
        assert (a != b).float().mean().item() > 0.5, "stale packed weights after load_state_dict"
        ref_u8, _, _ = O.apply_pidinet(sd2, HO.to_pil_u8(x[0]), device="cuda")
        _check_levels(_levels(b)[0], ref_u8, "after weight swap")
    finally:
        pidi_net.load_state_dict(old, strict=True)
    assert torch.equal(pidi_net.apply(x), a)


def test_small_inputs_raise(pidi_net, ctl):
    for shape in ((1, 3, 7, 64), (1, 3, 64, 7)):
        with pytest.raises(ValueError):
            ctl.preprocess(torch.rand(shape).cuda(), type="scribble")


def test_absent_weights_still_raise(ctl, tmp_path, monkeypatch):
    from pfd_b200 import pidinet
    monkeypatch.chdir(tmp_path)
    saved = pidinet._network
    pidinet.set_network(None)
    try:
        x = torch.rand((1, 3, 32, 32)).cuda()
        for kw in ({}, {"method": "pidinet"}):
            with pytest.raises(NotImplementedError, match="method='hed'.*method='xdog'"):
                ctl.preprocess(x, type="scribble", **kw)
    finally:
        pidinet.set_network(saved)
