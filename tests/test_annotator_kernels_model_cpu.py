"""CPU model of the annotator layer-kernel tests (test_annotator_kernels_gpu.py): numpy emulations of the kernels'
arithmetic and index rules (annotator_ref.py) stand in for the kernels and run through the same checks and cases.
The emulations pass every check; each listed mutant (annotator_ref.MUTANTS) fails at least one case, so a kernel with
that defect would fail the GPU test too.
"""
import pytest
import torch

import annotator_ref as R


def _cases(kernel):
    """[(label, check(run) -> (ok, worst))] of one kernel, as the GPU test runs them (its large grid-stride and batch
    cases aside)."""
    out = []
    both = (True, False)
    if kernel == "quant":
        for dt in (torch.float16, torch.float32):
            out.append((f"{dt}", lambda r, dt=dt: R.check_quant(r["roundtrip"], r["hed_input"], r["mlsd_input"], dt)))
    table = {
        "pool": (R.POOL_CASES, both, lambda r, c, i, s: R.check_pool(r["pool"], c, i, s)),
        "im2col": (R.IM2COL_CASES, (False,), lambda r, c, i, s: R.check_im2col(r["im2col"], c, s)),
        "dw": (R.DW_CASES, both, lambda r, c, i, s: R.check_dw(r["dw"], c, i, s)),
        "mlsd_dw": (R.MLSD_DW_CASES, both, lambda r, c, i, s: R.check_mlsd_dw(r["mlsd_dw"], c, i, s)),
        "reduce": (R.REDUCE_CASES, both, lambda r, c, i, s: R.check_reduce(r["reduce"], c, i, s)),
        "cdcm": (R.CDCM_CASES, both, lambda r, c, i, s: R.check_cdcm(r["cdcm"], c, i, s, r.get("pack"))),
        "side": (R.SIDE_CASES, (False,), lambda r, c, i, s: R.check_side(r["side"], c, s)),
        "fuse": (R.FUSE_CASES, (False,), lambda r, c, i, s: R.check_fuse(r["fuse"], c, s)),
        "upsample": (R.UPSAMPLE_CASES, (False,), lambda r, c, i, s: R.check_upsample(r["upsample"], c, s)),
        "mlsd_head": (R.MLSD_HEAD_CASES, both, lambda r, c, i, s: R.check_mlsd_head(r["mlsd_head"], c, i, s)),
        "op_head": (R.OP_HEAD_CASES, both, lambda r, c, i, s: R.check_op_head(r["op_head"], c, i, s)),
    }
    if kernel in table:
        cases, kinds, fn = table[kernel]
        for k, case in enumerate(cases):
            for integer in kinds:
                out.append((f"{case} {'int' if integer else 'rand'}",
                            lambda r, c=case, i=integer, s=100 + k: fn(r, c, i, s)))
    return out


KERNELS = ["quant", "pool", "im2col", "dw", "mlsd_dw", "reduce", "cdcm", "side", "fuse", "upsample", "mlsd_head",
           "op_head"]
MUTANT_KERNELS = {
    "dw_drop_last_col": ["dw"], "ceil_pool": ["pool", "dw"], "mlsd_sym_pad": ["mlsd_dw"],
    "mlsd_relu6_out_only": ["mlsd_dw"], "upsample_align_false": ["upsample"], "csam_pad_u": ["side"],
    "cdcm_swap_dilations": ["cdcm"], "cdcm_pack_lanes_swapped": ["cdcm"], "quant_fp32_product": ["quant"],
    "fuse_unclamped_i1": ["fuse"], "head_relu_paf": ["op_head"],
}


def test_every_mutant_has_a_kernel():
    assert set(MUTANT_KERNELS) == set(R.MUTANTS)


@pytest.mark.parametrize("kernel", KERNELS)
def test_model_passes_every_check(kernel):
    runners = R.model_runners()
    worst_int = worst_rand = 0.0
    failed = []
    for label, check in _cases(kernel):
        ok, worst = check(runners)
        if not ok:
            failed.append((label, worst))
        if label.endswith("rand"):
            worst_rand = max(worst_rand, worst)
        else:
            worst_int = max(worst_int, worst)
    print(f"[model {kernel}] {len(_cases(kernel))} cases, integer mismatches {worst_int:g}, "
          f"random max err/bound {worst_rand:.3g}")
    assert not failed, failed


@pytest.mark.parametrize("mutant", list(R.MUTANTS))
def test_mutant_is_rejected(mutant):
    runners = R.model_runners(mutant)
    if mutant == "cdcm_pack_lanes_swapped":
        runners = dict(R.model_runners(), pack=R.pack_cdcm_lanes_swapped)
    rejected, total = [], 0
    for kernel in MUTANT_KERNELS[mutant]:
        for label, check in _cases(kernel):
            total += 1
            ok, worst = check(runners)
            if not ok:
                rejected.append(f"{kernel} {label} ({worst:.3g})")
    print(f"[mutant {mutant}] {R.MUTANTS[mutant]}: rejected by {len(rejected)} of {total} cases, e.g. "
          f"{rejected[:2]}")
    assert rejected, f"{mutant} passes every case"


def test_fp32_product_changes_131_fp16_levels():
    """The quantiser's product must be rounded in fp16: rounded in fp32 instead, 131 of the 15 361 fp16 inputs in
    [0, 1] truncate to another level."""
    x = R.quant_inputs_f16()
    assert torch.equal(R.to_u8_model(x), R.to_u8_ref(x))
    assert int((R.to_u8_model(x, "quant_fp32_product") != R.to_u8_ref(x)).sum()) == 131


def test_cdcm_unpack_inverts_pack():
    """The emulation's fragment decoding is the inverse of pidinet.pack_cdcm: K = (dilation, ky, kx, channel)."""
    from pfd_b200.pidinet import pack_cdcm
    Ws = R.ints((4, 24, 24, 3, 3), -8, 8, 3).float()
    dense = R.cdcm_unpack(pack_cdcm(list(Ws)))
    assert torch.equal(dense, Ws.permute(0, 3, 4, 2, 1).reshape(864, 24).double())


def test_fuse_resize_model_is_the_oracle_resize():
    from oracle.pidinet_oracle import resize_bilinear
    for k, (h, w, H, W) in enumerate([(4, 5, 37, 45), (1, 1, 9, 8), (16, 12, 131, 97), (64, 61, 67, 61)]):
        s = R.randn((h, w), k).float().numpy()
        assert (R.resize_model(s, H, W) == resize_bilinear(s, H, W)).all(), (h, w, H, W)
