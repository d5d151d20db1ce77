"""Scribble annotators on the GPU (ControlNet.preprocess type 'scribble', methods 'hed' and 'xdog'): the kernels against
the numpy oracle (oracle/scribble_oracle.py), the reference's outputs (tests/golden/scribble_outputs.npz), batching,
deterministic mode and CUDA-graph replay."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# End-to-end method='hed' against the reference's golden scribble maps: the fp16 HED network moves levels by up to 3
# (test_hed_gpu.py), which moves some NMS / `> 127` decisions and, through the 19x19 blur, the pixels around them.
# Measured on an H100 80GB HBM3 (700 W power limit): 0 %, 0.23 %, 0.36 % and 0.46 % of the pixels of the four golden
# cases (33x31, 97x131, 200x168, 256x256) differ; the bound is about twice the largest.
E2E_FLIP_BOUND = 0.01


@pytest.fixture(scope="module")
def hed_net():
    from oracle.hed_oracle import fill_synthetic
    from pfd_b200 import hed
    m = fill_synthetic(hed.ControlNetHED().cuda(), seed=0)
    saved = hed._network
    hed.set_network(m)
    yield m
    hed.set_network(saved)


@pytest.fixture(scope="module")
def ctl():
    """A small ControlNet: preprocess does not depend on the ControlNet's own size."""
    from pfd_b200.controlnet import ControlNet
    return ControlNet(32, 4, 32, 3, 1, [], channel_mult=(1,), use_spatial_transformer=True, context_dim=32,
                      num_heads=1, legacy=False).cuda()


@pytest.fixture
def det():
    import pfd_b200
    was = pfd_b200.is_deterministic()
    pfd_b200.set_deterministic(True)
    yield
    pfd_b200.set_deterministic(was)


def _golden():
    z = np.load(os.path.join(ROOT, "tests", "golden", "scribble_outputs.npz"))
    i = 0
    while f"case_{i}" in z:
        seed, H, W = (int(v) for v in z[f"case_{i}"])
        yield seed, H, W, z[f"hed_{i}"], z[f"scribble_{i}"]
        i += 1


def _check_map(out, B, H, W):
    assert out.dtype == torch.float32 and out.is_cuda and out.shape == (B, 3, H, W)
    assert torch.equal(out[:, 0], out[:, 1]) and torch.equal(out[:, 0], out[:, 2])
    assert bool(((out == 0) | (out == 1)).all())


def _u8(out):
    return (out[:, 0] * 255).to(torch.uint8).cpu().numpy()


def test_post_process_on_golden_hed_maps():
    from oracle import scribble_oracle as S
    from pfd_b200 import native as nv
    cases = list(_golden())
    assert len(cases) == 4
    for _, H, W, hed_u8, ref in cases:
        levels = torch.from_numpy(hed_u8).float().div(255.0)[None, None].cuda()
        out, nms = nv.scribble_hed(levels, return_nms=True)
        _check_map(out, 1, H, W)
        _, exempt = S.make_scribble(hed_u8)
        bad = (_u8(out)[0] != ref) & ~exempt
        assert not bad.any(), f"{H}x{W}: {int(bad.sum())} pixels differ from the reference away from near-ties"
        assert exempt.mean() <= 1e-3, exempt.mean()
        zc, zp = S.nms_threshold(S.blur_f64(hed_u8, 3.0), S.TOL)
        z = nms.cpu().numpy()[0] == 255
        assert not (zc & ~z).any() and not (z & ~zp).any(), f"{H}x{W}: NMS decision outside the tie tolerance"
        assert 0.05 < (ref == 255).mean() < 0.95


@pytest.mark.parametrize("B,H,W", [(2, 97, 131), (1, 9, 7), (3, 1, 1), (1, 1, 40), (2, 300, 257), (1, 64, 64)])
def test_u8_blur_is_exact(B, H, W):
    from oracle import scribble_oracle as S
    from pfd_b200 import native as nv
    rng = np.random.RandomState(B * 1000 + H + W)
    z = rng.randint(0, 256, (B, H, W)).astype(np.uint8)
    z[-1] = np.where(rng.rand(H, W) > 0.97, 255, 0)                   # sparse 255-dots, as after the NMS
    blurred, out = nv.scribble_blur_u8(torch.from_numpy(z).cuda())
    _check_map(out, B, H, W)
    bl = blurred.cpu().numpy()
    for b in range(B):
        assert np.array_equal(bl[b], S.blur_u8(z[b])), f"image {b}"
    assert np.array_equal(_u8(out), np.where(bl > 4, 255, 0))


XDOG_SHAPES = [((1, 3, 9, 7), torch.float32), ((2, 3, 97, 131), torch.float16), ((1, 3, 768, 640), torch.float32),
               ((1, 3, 33, 31), torch.float16), ((1, 3, 256, 256), torch.float16)]


@pytest.mark.parametrize("shape,dtype", XDOG_SHAPES)
def test_xdog_matches_oracle(ctl, shape, dtype):
    from oracle import hed_oracle as HO
    from oracle import scribble_oracle as S
    B, _, H, W = shape
    x = torch.cat([HO.image_to_tensor(S.scribble_image(10 * b + H, H, W), dtype) for b in range(B)]).cuda()
    wrap = 0
    values = [S.xdog_value(HO.to_pil_u8(x[b])) for b in range(B)]
    for threshold in (0, 32, 200):
        out = ctl.preprocess(x, type="scribble", method="xdog", threshold=threshold)
        _check_map(out, B, H, W)
        got = _u8(out)
        for b in range(B):
            v = values[b]
            dogs = [np.floor(np.clip(v + s, 0, 255)).astype(np.uint8) for s in (-S.TOL, 0.0, S.TOL)]
            e = [S.xdog_from_dog(d, threshold) for d in dogs]
            exempt = (e[0] != e[1]) | (e[2] != e[1])
            bad = (got[b] != np.where(e[1], 255, 0)) & ~exempt
            assert not bad.any(), f"threshold {threshold} image {b}: {int(bad.sum())} pixels differ"
            assert exempt.mean() <= 1e-3, exempt.mean()
            wrap += int((255 - dogs[1].astype(np.int64) >= 128).sum())
    if H * W >= 4096:
        assert wrap > 0, "no pixel in the uint8 wrap range"
    assert torch.equal(ctl.preprocess(x, type="scribble", method="xdog"),                 # the default threshold
                       ctl.preprocess(x, type="scribble", method="xdog", threshold=32))


def test_xdog_wrap_pixels_are_not_edges(ctl):
    """255 - dog = 128 .. 144 gives 2 * (255 - dog) mod 256 = 0 .. 32: no edge at threshold 32."""
    from oracle import hed_oracle as HO
    from oracle import scribble_oracle as S
    img = S.scribble_image(2, 256, 256)
    x = HO.image_to_tensor(img).cuda()
    got = _u8(ctl.preprocess(x, type="scribble", method="xdog"))[0]
    _, exempt, dog = S.xdog(HO.to_pil_u8(x[0]), 32)
    inv = 255 - dog.astype(np.int64)
    low_wrap = (inv >= 128) & (inv <= 144) & ~exempt
    high_wrap = (inv > 144) & ~exempt
    assert low_wrap.sum() > 0 and high_wrap.sum() > 0
    assert (got[low_wrap] == 0).all() and (got[high_wrap] == 255).all()


def test_preprocess_hed_end_to_end(hed_net, ctl):
    from oracle import hed_oracle as HO
    from oracle import scribble_oracle as S
    worst = 0.0
    for seed, H, W, _, ref in _golden():
        x = HO.image_to_tensor(HO.hed_image(seed, H, W)).cuda()
        out = ctl.preprocess(x, type="scribble", method="hed", size=[64, 64])
        _check_map(out, 1, H, W)
        got = _u8(out)[0]
        # exact against the oracle on this run's own HED levels (only the network's level error is left to the golden)
        levels = (ctl.preprocess(x, type="hed")[0, 0].double() * 255).round().to(torch.uint8).cpu().numpy()
        want, exempt = S.make_scribble(levels)
        assert not ((got != want) & ~exempt).any() and exempt.mean() <= 1e-3
        flips = float((got != ref).mean())
        print(f"[scribble] end-to-end {H}x{W}: {flips:.4%} of pixels differ from the reference")
        worst = max(worst, flips)
    assert worst <= E2E_FLIP_BOUND, worst


def test_inputs_like_other_types(hed_net, ctl, tmp_path):
    import PIL.Image
    from oracle import hed_oracle as HO
    img = HO.hed_image(7, 40, 56)
    x = HO.image_to_tensor(img).cuda()
    path = os.path.join(str(tmp_path), "img.png")
    PIL.Image.fromarray(img).save(path)
    for method in ("hed", "xdog"):
        a = ctl.preprocess(x, type="scribble", method=method)
        _check_map(a, 1, 40, 56)
        assert torch.equal(ctl.preprocess(path, type="scribble", method=method), a)
        assert torch.equal(ctl.preprocess(x.cpu(), type="scribble", method=method), a)
        gray = x[:, :1]
        assert torch.equal(ctl.preprocess(gray, type="scribble", method=method),
                           ctl.preprocess(gray.repeat(1, 3, 1, 1), type="scribble", method=method))


@pytest.mark.parametrize("method", ["hed", "xdog"])
def test_batch_equals_singles_deterministic(hed_net, ctl, det, method):
    from oracle import hed_oracle as HO
    x = torch.cat([HO.image_to_tensor(HO.hed_image(s, 96, 80)) for s in (1, 2, 3)]).cuda().half()
    batch = ctl.preprocess(x, type="scribble", method=method)
    singles = torch.cat([ctl.preprocess(x[b:b + 1], type="scribble", method=method) for b in range(3)])
    assert torch.equal(batch, singles)


def test_graph_replay_equals_eager(hed_net, ctl):
    from oracle import hed_oracle as HO
    x = torch.cat([HO.image_to_tensor(HO.hed_image(s, 96, 80)) for s in (4, 5)]).cuda().half()
    run = lambda: (ctl.preprocess(x, type="scribble", method="hed"),                # noqa: E731
                   ctl.preprocess(x, type="scribble", method="xdog", threshold=20))
    eager = run()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()                                                                        # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = run()
    for o in outs:
        o.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(outs[0], eager[0]) and torch.equal(outs[1], eager[1])


def test_methods_that_do_not_run(ctl):
    x = torch.rand((1, 3, 32, 32)).cuda()
    with pytest.raises(ValueError):
        ctl.preprocess(x, type="scribble", method="canny")
    for kw in ({}, {"method": "pidinet"}):
        with pytest.raises(NotImplementedError, match="method='hed'.*method='xdog'"):
            ctl.preprocess(x, type="scribble", **kw)
