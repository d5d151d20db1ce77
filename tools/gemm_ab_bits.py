"""Compare the GEMM outputs of two builds of the library bit for bit, over a matrix of the UNet's Linear and conv
shapes (batch 8 = one CFG pair of batch 4 at 512 x 512) and the epilogues they run.  Each build runs in its own
process (PFD_B200_LIB); inputs come from fixed CPU seeds, so both processes see the same data.

    python tools/gemm_ab_bits.py --lib-a OLD.so [--lib-b NEW.so]     # --lib-b defaults to the in-tree library
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to("cuda", torch.float16)


def cases(nv):
    """name -> callable returning the output tensor."""
    out = {}
    # Linears: (M, N, K, epilogue)
    for M, N, K, ep in [(32768, 320, 320, "bias_res"), (32768, 320, 1280, "bias_res"), (32768, 320, 320, "none"),
                        (8192, 640, 640, "bias_res"), (8192, 640, 2560, "bias_res"), (8192, 640, 640, "none"),
                        (2048, 1280, 1280, "bias_res"), (2048, 1280, 5120, "bias_res"), (512, 1280, 1280, "bias_res"),
                        (1184, 1280, 768, "none"), (32768, 960, 320, "none"), (1000, 328, 192, "bias_res")]:
        x, w = rnd(M, K), rnd(N, K, scale=K ** -0.5, seed=1)
        b = rnd(N, seed=2) if ep == "bias_res" else None
        r = rnd(M, N, seed=3) if ep == "bias_res" else None
        out[f"linear_{M}x{N}x{K}_{ep}"] = (lambda x=x, w=w, b=b, r=r: nv.linear(x, w, b, residual=r))
    # GEGLU projections of the three transformer widths
    for M, C in [(32768, 320), (8192, 640), (2048, 1280)]:
        x, w, b = rnd(M, C), rnd(8 * C, C, scale=C ** -0.5, seed=1), rnd(8 * C, seed=2)
        wp, bp, bn = nv.pack_geglu(w, b)
        out[f"geglu_{M}x{C}"] = (lambda x=x, wp=wp, bp=bp, bn=bn: nv.linear(x, wp, bp, act=nv.ACT_GEGLU, bn_force=bn))
    # head-split q / k / v projection ([B, T, heads*d] -> [B, heads, T, d]) and the swapped V^T product (element-strided)
    B, T, heads, d = 8, 4096, 5, 64
    xq, wq, bq = rnd(B * T, 320), rnd(320, 320, scale=320 ** -0.5, seed=1), rnd(320, seed=2)

    def head_split(x=xq, w=wq, b=bq):
        o = torch.empty((B, heads, T, d), device="cuda", dtype=torch.float16)
        nv.gemm_raw([(x, 1, 320, (320, 320 * T, 320 * T))], in_w=T, in_h=1, stride=1, W=T, H=1, NB=B, w=w, N=320,
                    K=320, bias=b, out=o, so=(heads * T * d, 0, 0, d, T * d, 1), ndiv=1, cdiv=d)
        return o

    def v_transposed(x=xq, w=wq, b=bq):
        o = torch.empty((B, heads, d, T), device="cuda", dtype=torch.float16)
        nv.gemm_raw([(x, 1, 320, (320, 320 * T, 320 * T))], in_w=T, in_h=1, stride=1, W=T, H=1, NB=B, w=w, N=320,
                    K=320, bias=b, out=o, so=(heads * d * T, 0, 0, 1, d * T, T), ndiv=1, cdiv=d)
        return o
    out["head_split_8x4096x320"] = head_split
    out["v_transposed_8x4096x320"] = v_transposed
    # 3x3 convs: ResBlock conv1 (bias + time-embedding row add + SiLU), conv2 (bias + identity residual), plain
    for NB, H, C, N in [(8, 64, 320, 320), (8, 32, 640, 640), (8, 16, 1280, 1280), (8, 8, 1280, 1280)]:
        x = rnd(NB, H, H, C)
        wp = rnd(N, 9 * C, scale=(9 * C) ** -0.5, seed=1)
        b, ra, r = rnd(N, seed=2), rnd(NB, N, seed=5), rnd(NB, H, H, N, seed=3)
        out[f"conv_{NB}x{H}x{H}x{C}->{N}_rowadd_silu"] = (
            lambda x=x, wp=wp, b=b, ra=ra: nv.conv3x3(x, wp, b, rowadd=ra, act=nv.ACT_SILU))
        out[f"conv_{NB}x{H}x{H}x{C}->{N}_res"] = (lambda x=x, wp=wp, b=b, r=r: nv.conv3x3(x, wp, b, residual=r))
        out[f"conv_{NB}x{H}x{H}x{C}->{N}_plain"] = (lambda x=x, wp=wp, b=b: nv.conv3x3(x, wp, b))
    return out


def dump(path):
    from pfd_b200 import native as nv
    nv.load()
    res = {}
    for name, fn in cases(nv).items():
        res[name] = fn().cpu()
        torch.cuda.synchronize()
    torch.save(res, path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-a", required=True)
    ap.add_argument("--lib-b", default=None)
    ap.add_argument("--dump", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.dump:
        dump(args.dump)
        return
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for tag, lib in (("a", args.lib_a), ("b", args.lib_b)):
            env = dict(os.environ)
            env.pop("PFD_B200_LIB", None)
            if lib:
                env["PFD_B200_LIB"] = os.path.abspath(lib)
            p = os.path.join(tmp, tag + ".pt")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--lib-a", "-", "--dump", p], env=env, check=True)
            paths.append(p)
        a, b = (torch.load(p) for p in paths)
    ndiff = 0
    for name in a:
        x, y = a[name], b[name]
        diff = (x != y).sum().item()
        ndiff += diff > 0
        print(json.dumps({"case": name, "shape": list(x.shape), "elements_differing": diff,
                          "max_abs_diff": (x.float() - y.float()).abs().max().item()}))
    print(json.dumps({"cases": len(a), "cases_differing": ndiff}))
    sys.exit(1 if ndiff else 0)


if __name__ == "__main__":
    main()
