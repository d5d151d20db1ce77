"""HED soft-edge annotator on the GPU (ControlNet.preprocess types 'hed' / 'softedge_v11p'): the fp16 network and the
three glue kernels against the fp32 oracle (oracle/hed_oracle.py), the reference's outputs (tests/golden) and torch."""
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
    print(f"[hed] {what}: max |d| {d.max()}, mean |d| {d.mean():.4f}, within 1: {(d <= 1).mean():.4%}, "
          f"unsaturated {inner:.1%}")
    assert inner >= 0.30, f"{what}: only {inner:.1%} of pixels strictly between 0 and 255"
    assert d.max() <= 3 and d.mean() <= 0.25 and (d <= 1).mean() >= 0.99, what


def _rel_rms(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.sqrt(np.mean((a - b) ** 2) / np.mean(b ** 2)))


SHAPES = [((1, 3, 512, 512), torch.float16), ((2, 3, 131, 97), torch.float32), ((1, 3, 768, 640), torch.float32),
          ((1, 3, 33, 31), torch.float16)]


@pytest.mark.parametrize("shape,dtype", SHAPES)
def test_preprocess_hed_matches_oracle(hed_net, ctl, fp32_oracle, shape, dtype):
    from oracle import hed_oracle as O
    from pfd_b200.hed import SCALE
    x = _image(shape, dtype).cuda()
    out = ctl.preprocess(x, type="hed", size=[64, 64])
    B, _, H, W = shape
    assert out.dtype == torch.float32 and out.is_cuda and out.shape == (B, 3, H, W)
    assert torch.equal(out[:, 0], out[:, 1]) and torch.equal(out[:, 0], out[:, 2])
    assert torch.equal(ctl.preprocess(x, type="softedge_v11p"), out)
    _, sides = hed_net.apply(x, return_sides=True)
    sd = {k: v.detach() for k, v in hed_net.state_dict().items()}
    lv = _levels(out)
    for b in range(B):
        ref_u8, _, ref_sides = O.apply_hed(sd, O.to_pil_u8(x[b]), device="cuda")
        for k, (s, r) in enumerate(zip(sides, ref_sides)):
            rel = _rel_rms(s[b].cpu().numpy() / SCALE, r)
            assert rel <= 5e-3, f"image {b} side {k}: rel rms {rel:.2e}"
        _check_levels(lv[b], ref_u8, f"{tuple(shape)} {dtype} image {b}")
    if B > 1:
        singles = torch.cat([ctl.preprocess(x[b:b + 1], type="hed") for b in range(B)])
        d = (_levels(singles) - lv)
        # the GEMM may split K differently for another M: allow rare one-level flips, nothing more
        assert np.abs(d).max() <= 1 and (d != 0).mean() <= 1e-3, f"batch vs single: {(d != 0).mean():.2e}"


def test_fuse_kernel_matches_oracle_exactly(fp32_oracle):
    from oracle import hed_oracle as O
    from pfd_b200 import native as nv
    sd = O.synth_state_dict(0)
    for seed, H, W in ((21, 97, 131), (22, 33, 31), (23, 200, 168)):
        sides = O.network_sides(sd, O.hed_image(seed, H, W), device="cuda")
        ref_u8, pre = O.fuse(sides, H, W)
        out = nv.hed_fuse([torch.from_numpy(s)[None].cuda() for s in sides], H, W, inv_scale=1.0)
        assert out.shape == (1, 3, H, W) and torch.equal(out[:, 0], out[:, 2])
        lv = _levels(out)[0]
        bad = (lv != ref_u8) & ~O.near_integer(pre)
        assert not bad.any(), f"{H}x{W}: {int(bad.sum())} levels differ away from integer boundaries"
        # the float32 values are exactly level / 255 (ToTensor)
        assert torch.equal(out[0, 0].cpu(), torch.from_numpy(lv.astype(np.float32)) / 255.0)


@pytest.mark.parametrize("B,h,w,C", [(2, 7, 9, 64), (1, 16, 16, 128), (2, 5, 3, 512), (1, 1, 1, 8), (1, 33, 31, 256),
                                     (1, 2, 2, 24)])
def test_pool_side_kernel_against_torch(B, h, w, C):
    from pfd_b200 import native as nv
    g = torch.Generator().manual_seed(B * 1000 + h * 100 + w + C)
    x = torch.relu(torch.randn((B, h, w, C), generator=g)).half().cuda()
    pw = torch.randn((C,), generator=g).cuda()
    pb = torch.randn((1,), generator=g).cuda()
    side, pooled = nv.hed_pool_side(x, pw, pb, pool=True)
    if h >= 2 and w >= 2:
        ref_pool = F.max_pool2d(x.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
        assert pooled.shape == ref_pool.shape and torch.equal(pooled, ref_pool)
    else:                                                              # floor semantics: nothing to pool
        assert pooled.shape == (B, h // 2, w // 2, C)
    ref_side = (x.double() @ pw.double()) + pb.double()
    err = (side.double() - ref_side).abs().max().item()
    assert side.shape == (B, h, w) and err <= 1e-5 * (x.double().abs() @ pw.double().abs()).max().item() + 1e-6
    side2, none = nv.hed_pool_side(x, pw, pb, pool=False)
    assert none is None and torch.equal(side2, side)


def test_golden_reference_outputs(hed_net, ctl):
    from oracle import hed_oracle as O
    z = np.load(os.path.join(ROOT, "tests", "golden", "hed_outputs.npz"))
    i = 0
    while f"case_{i}" in z:
        seed, H, W = (int(v) for v in z[f"case_{i}"])
        x = O.image_to_tensor(O.hed_image(seed, H, W)).cuda()
        _check_levels(_levels(ctl.preprocess(x, type="hed"))[0], z[f"u8_{i}"], f"golden {H}x{W}")
        i += 1
    assert i == 3


def test_graph_capture_equals_eager(hed_net):
    x = _image((2, 3, 96, 80), torch.float16).cuda()
    eager = hed_net.apply(x)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        hed_net.apply(x)                                               # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = hed_net.apply(x)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_weight_swap_repacks(hed_net, ctl, fp32_oracle):
    from oracle import hed_oracle as O
    x = _image((1, 3, 120, 136), torch.float32).cuda()
    a = ctl.preprocess(x, type="hed")
    # seed 2: most output levels of this image stay strictly between 0 and 255 (seed 1 saturates 95 % of them)
    old = {k: v.clone() for k, v in hed_net.state_dict().items()}
    try:
        hed_net.load_state_dict({k: v.cuda() for k, v in O.synth_state_dict(2).items()}, strict=True)
        b = ctl.preprocess(x, type="hed")
        assert (a != b).float().mean().item() > 0.5, "stale packed weights after load_state_dict"
        ref_u8, _, _ = O.apply_hed(O.synth_state_dict(2), O.to_pil_u8(x[0]), device="cuda")
        _check_levels(_levels(b)[0], ref_u8, "after weight swap")
    finally:
        hed_net.load_state_dict(old, strict=True)
    assert torch.equal(ctl.preprocess(x, type="hed"), a)


def test_other_annotators_still_raise(ctl):
    x = torch.rand((1, 3, 32, 32)).cuda()
    for t in ("mlsd", "normal", "openpose", "scribble", "seg"):
        with pytest.raises(NotImplementedError):
            ctl.preprocess(x, type=t)
