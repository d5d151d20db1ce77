"""The annotator layer kernels (PiDiNet, M-LSD, OpenPose) and the shared ToPILImage quantiser against float64 references
of their own contracts (annotator_ref.py), element by element, at image borders, odd sizes, maps smaller than the
kernel window, the last partial 16x16 CDCM tile and the last 8-channel vector.

Integer cases (exact products and sums) must equal the reference exactly; random cases must stay within the bound
derived from the kernel's rounding points.  Data movement (pools, im2col, the pooled output of the depthwise conv, the
quantiser) is compared bit for bit.  Every grid-stride kernel also runs once with more work items than one pass of its
capped grid (16 blocks per SM), and a batch of three images must give the bits of the images run one at a time.
"""
import pytest
import torch

import annotator_ref as R
from pfd_b200 import native as nv

pytestmark = pytest.mark.gpu


def _c(t):
    return t.cuda()


def _op_head(x, w, b, relu, buf, off):
    out = _c(buf)
    nv.openpose_head(_c(x), _c(w), _c(b), relu, out, off)
    return out


def _upsample(x, buf):
    out = _c(buf)
    nv.mlsd_upsample(_c(x), out[..., out.shape[-1] // 2:])
    return out


RUN = {
    "roundtrip": lambda v: nv.image_u8_roundtrip(_c(v)),
    "hed_input": lambda img, norm, scale, cpad: nv.hed_input(_c(img), _c(torch.tensor(norm, dtype=torch.float32)),
                                                             scale, cpad),
    "mlsd_input": lambda img: nv.mlsd_input(_c(img)),
    "pool": lambda x: nv.openpose_pool(_c(x)),
    "im2col": lambda x: nv.im2col7x7(_c(x)),
    "dw": lambda x, wt, pool: nv.pidinet_dw(_c(x), _c(wt), pool),
    "mlsd_dw": lambda x, wt, b, s: nv.mlsd_dw(_c(x), _c(wt), _c(b), s),
    "reduce": lambda x, w, b: nv.pidinet_reduce(_c(x), _c(w), _c(b)),
    "cdcm": lambda m, wpk: nv.pidinet_cdcm(_c(m), _c(wpk)),
    "side": lambda u, prm: nv.pidinet_side(_c(u), _c(prm)),
    "fuse": lambda sides, cls, H, W: nv.pidinet_fuse([_c(s) for s in sides], _c(cls), H, W),
    "upsample": _upsample,
    "mlsd_head": lambda x, w, b: nv.mlsd_head(_c(x), _c(w), _c(b)),
    "op_head": _op_head,
}


def _ok(res, what):
    ok, worst = res
    print(f"[{what}] worst {worst:.3g}")
    assert ok, f"{what}: worst {worst}"


def _ids(cases):
    return ["x".join(str(v) for v in c) for c in cases]


# ------------------------------------------------------------------------------------------------- quantiser
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_quantiser(dtype):
    _ok(R.check_quant(RUN["roundtrip"], RUN["hed_input"], RUN["mlsd_input"], dtype), f"quant {dtype}")


# ------------------------------------------------------------------------------------------------- data movement
@pytest.mark.parametrize("integer", [True, False])
@pytest.mark.parametrize("case", R.POOL_CASES, ids=_ids(R.POOL_CASES))
def test_openpose_pool(case, integer):
    _ok(R.check_pool(RUN["pool"], case, integer, 11), f"pool {case}")


@pytest.mark.parametrize("case", R.IM2COL_CASES, ids=_ids(R.IM2COL_CASES))
def test_im2col7x7(case):
    _ok(R.check_im2col(RUN["im2col"], case, 12), f"im2col {case}")


# ------------------------------------------------------------------------------------------------- PiDiNet
@pytest.mark.parametrize("integer", [True, False])
@pytest.mark.parametrize("case", R.DW_CASES, ids=_ids(R.DW_CASES))
def test_pidinet_dw(case, integer):
    _ok(R.check_dw(RUN["dw"], case, integer, 13), f"pidinet_dw {case}")


@pytest.mark.parametrize("integer", [True, False])
@pytest.mark.parametrize("case", R.REDUCE_CASES, ids=_ids(R.REDUCE_CASES))
def test_pidinet_reduce(case, integer):
    _ok(R.check_reduce(RUN["reduce"], case, integer, 14), f"pidinet_reduce {case}")


@pytest.mark.parametrize("case", R.CDCM_CASES, ids=_ids(R.CDCM_CASES))
def test_pidinet_cdcm_integer(case):
    _ok(R.check_cdcm(RUN["cdcm"], case, True, 15), f"pidinet_cdcm {case}")


@pytest.mark.parametrize("case", [(1, 33, 31), (2, 17, 64), (1, 65, 48)], ids=_ids([(1, 33, 31), (2, 17, 64), (1, 65, 48)]))
def test_pidinet_cdcm_random(case):
    _ok(R.check_cdcm(RUN["cdcm"], case, False, 16), f"pidinet_cdcm random {case}")


@pytest.mark.parametrize("case", R.SIDE_CASES, ids=_ids(R.SIDE_CASES))
def test_pidinet_side(case):
    _ok(R.check_side(RUN["side"], case, 17), f"pidinet_side {case}")


@pytest.mark.parametrize("case", R.FUSE_CASES, ids=_ids(R.FUSE_CASES))
def test_pidinet_fuse(case):
    _ok(R.check_fuse(RUN["fuse"], case, 18), f"pidinet_fuse {case} near-integer pixels")


# ------------------------------------------------------------------------------------------------- M-LSD
@pytest.mark.parametrize("integer", [True, False])
@pytest.mark.parametrize("case", R.MLSD_DW_CASES, ids=_ids(R.MLSD_DW_CASES))
def test_mlsd_dw(case, integer):
    _ok(R.check_mlsd_dw(RUN["mlsd_dw"], case, integer, 19), f"mlsd_dw {case}")


@pytest.mark.parametrize("case", R.UPSAMPLE_CASES, ids=_ids(R.UPSAMPLE_CASES))
def test_mlsd_upsample(case):
    _ok(R.check_upsample(RUN["upsample"], case, 20), f"mlsd_upsample {case}")


@pytest.mark.parametrize("integer", [True, False])
@pytest.mark.parametrize("case", R.MLSD_HEAD_CASES, ids=_ids(R.MLSD_HEAD_CASES))
def test_mlsd_head(case, integer):
    _ok(R.check_mlsd_head(RUN["mlsd_head"], case, integer, 21), f"mlsd_head {case}")


# ------------------------------------------------------------------------------------------------- OpenPose head
@pytest.mark.parametrize("integer", [True, False])
@pytest.mark.parametrize("case", R.OP_HEAD_CASES, ids=_ids(R.OP_HEAD_CASES))
def test_openpose_head(case, integer):
    _ok(R.check_op_head(RUN["op_head"], case, integer, 22), f"openpose_head {case}")


# ------------------------------------------------------------------------------------------------- grid-stride passes
def _items(block=256):
    """More work items than one pass of a capped grid: 16 blocks per SM of `block` threads, plus a ragged tail."""
    return 16 * torch.cuda.get_device_properties(0).multi_processor_count * block + 77


def _side(n):
    return int(n ** 0.5) + 1


def test_grid_stride_quantiser():
    n = _items()
    vals = R.rand((n,), 30, 0.0, 1.0).half()
    assert R.bit_mismatches(RUN["roundtrip"](vals), R.to_u8_ref(vals).float() / 255) == 0
    img = R.rand((1, 3, 7, _items() // 7 + 1), 31, 0.0, 1.0).float()
    assert R.bit_mismatches(RUN["hed_input"](img, R.HED_NORM, R.HED_SCALE, 3),
                            R.hed_input_ref(img, R.HED_NORM, R.HED_SCALE, 3)) == 0
    assert R.bit_mismatches(RUN["mlsd_input"](img), R.mlsd_input_ref(img)) == 0


def test_grid_stride_data_movement():
    s = _side(_items() // 8)                             # C = 64: 8 vectors per pixel
    _ok(R.check_pool(RUN["pool"], (1, 2 * s + 1, 2 * s, 64), False, 32), "pool large")
    s = _side(_items() // 49) + 1                        # C = 8: 49 items per pixel
    _ok(R.check_im2col(RUN["im2col"], (1, s, s, 8), 33), "im2col large")


def test_grid_stride_pidinet():
    s = _side(_items() // 8)
    _ok(R.check_dw(RUN["dw"], (1, s, s, 64, 3, False), False, 34), "pidinet_dw large")
    _ok(R.check_dw(RUN["dw"], (1, 2 * s + 1, 2 * s, 64, 3, True), True, 35), "pidinet_dw pool large")
    s = _side(_items(128))
    _ok(R.check_reduce(RUN["reduce"], (1, s, s, 8), False, 36), "pidinet_reduce large")
    s = _side(_items())
    _ok(R.check_side(RUN["side"], (1, s, s), 37), "pidinet_side large")
    _ok(R.check_fuse(RUN["fuse"], (1, s, s + 3), 38), "pidinet_fuse large")


def test_grid_stride_mlsd_openpose():
    s = _side(_items())
    _ok(R.check_mlsd_dw(RUN["mlsd_dw"], (1, s, s, 8, 1), False, 39), "mlsd_dw large")
    _ok(R.check_mlsd_dw(RUN["mlsd_dw"], (1, 2 * s + 1, 2 * s, 8, 2), True, 40), "mlsd_dw stride 2 large")
    s = _side(_items() // 32)                             # 4 output pixels x 8 vectors per input pixel
    _ok(R.check_upsample(RUN["upsample"], (1, s, s), 41), "mlsd_upsample large")
    s = _side(_items(128))
    _ok(R.check_mlsd_head(RUN["mlsd_head"], (1, s, s, 8), False, 42), "mlsd_head large")
    s = _side(_items() // 19)
    _ok(R.check_op_head(RUN["op_head"], (1, s, s, 8, 19, False, 21, 1), False, 43), "openpose_head large")


# ------------------------------------------------------------------------------------------------- batch invariance
def _batch_cases():
    """name -> (inputs with a leading batch of 3, call(inputs) -> output with the batch leading)."""
    g = 50
    x16 = R.randn((3, 19, 21, 64), g).half().cuda()
    img = R.rand((3, 3, 13, 17), g, 0.0, 1.0).float().cuda()
    w9 = R.randn((9, 64), g + 1, 0.3).float().cuda()
    w25 = R.randn((25, 64), g + 2, 0.3).float().cuda()
    b64 = R.randn((64,), g + 3).float().cuda()
    m, Ws = R.cdcm_inputs(3, 19, 21, False, g)
    from pfd_b200.pidinet import pack_cdcm
    wpk = pack_cdcm(list(Ws)).cuda()
    u = R.randn((3, 19, 21, R.D), g).float().cuda()
    prm = R.side_params(g).cuda()
    sides, cls = R.fuse_inputs(3, 37, 45, g)
    sides, cls = [s.cuda() for s in sides], cls.cuda()
    wr, br = R.randn((64, R.D), g + 4, 0.2).float().cuda(), R.randn((R.D,), g + 5).float().cuda()
    w5, b5 = R.randn((5, 64), g + 6, 0.1).float().cuda(), R.randn((5,), g + 7).float().cuda()
    w19, b19 = R.randn((19, 64), g + 8, 0.1).float().cuda(), R.randn((19,), g + 9).float().cuda()

    def head(x):
        out = torch.zeros((x.shape[0], 21, x.shape[1], x.shape[2]), device=x.device)
        nv.openpose_head(x, w19, b19, False, out, 1)
        return out

    def up(x):
        out = torch.zeros((x.shape[0], 2 * x.shape[1], 2 * x.shape[2], 128), device=x.device, dtype=torch.float16)
        nv.mlsd_upsample(x, out[..., 64:])
        return out

    return {
        "roundtrip": ([img], lambda i: nv.image_u8_roundtrip(i)),
        "hed_input": ([img], lambda i: nv.hed_input(i, torch.tensor(R.HED_NORM, device="cuda").float(), R.HED_SCALE)),
        "mlsd_input": ([img], lambda i: nv.mlsd_input(i)),
        "pidinet_dw3": ([x16], lambda x: nv.pidinet_dw(x, w9)),
        "pidinet_dw5": ([x16], lambda x: nv.pidinet_dw(x, w25)),
        "pidinet_dw_pool": ([x16], lambda x: torch.cat(nv.pidinet_dw(x, w9, pool=True), -1)),
        "pidinet_reduce": ([x16], lambda x: nv.pidinet_reduce(x, wr, br)),
        "pidinet_cdcm": ([m.cuda()], lambda x: nv.pidinet_cdcm(x, wpk)),
        "pidinet_side": ([u], lambda x: nv.pidinet_side(x, prm)),
        "pidinet_fuse": (sides, lambda *s: nv.pidinet_fuse(list(s), cls, 37, 45)),
        "mlsd_dw1": ([x16.abs() * 2], lambda x: nv.mlsd_dw(x, w9, b64, 1)),
        "mlsd_dw2": ([x16.abs() * 2], lambda x: nv.mlsd_dw(x, w9, b64, 2)),
        "mlsd_upsample": ([x16], up),
        "mlsd_head": ([x16], lambda x: nv.mlsd_head(x, w5, b5)),
        "openpose_pool": ([x16], lambda x: nv.openpose_pool(x)),
        "im2col7x7": ([x16], lambda x: nv.im2col7x7(x).reshape(x.shape[0], -1)),
        "openpose_head": ([x16], head),
    }


BATCH_KERNELS = ["roundtrip", "hed_input", "mlsd_input", "pidinet_dw3", "pidinet_dw5", "pidinet_dw_pool",
                 "pidinet_reduce", "pidinet_cdcm", "pidinet_side", "pidinet_fuse", "mlsd_dw1", "mlsd_dw2",
                 "mlsd_upsample", "mlsd_head", "openpose_pool", "im2col7x7", "openpose_head"]


@pytest.fixture(scope="module")
def batch_cases():
    return _batch_cases()


@pytest.mark.parametrize("name", BATCH_KERNELS)
def test_batch_of_three_matches_single_images(batch_cases, name):
    inputs, call = batch_cases[name]
    whole = call(*inputs)
    singles = torch.cat([call(*[t[n:n + 1].contiguous() for t in inputs]) for n in range(3)])
    torch.cuda.synchronize()
    assert R.bits_equal(whole.cpu(), singles.cpu()), name
