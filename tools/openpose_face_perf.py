"""CUDA-event times of the OpenPose face annotator (pfd_b200/openpose_face.py) with synthetic weights: FaceNet alone at
1, 4 and 16 faces (TFLOP/s counted from its shapes), the whole 'openpose_withface' call against 'openpose' on planted
bodies with four faces at 512^2 and 1024^2, and the oracle's fp32 eager FaceNet one face at a time, as Face.__call__
runs it.  Prints one line per case and the card's name and power limit."""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def face_flops() -> float:
    """Multiply-adds x 2 of FaceNet on one 384 x 384 face, from its layer shapes (about 232 GFLOP)."""
    from pfd_b200.openpose_face import TRUNK, stage_layers
    f, h = 0.0, 384
    for v in TRUNK:
        if v == "pool":
            h //= 2
        else:
            f += 2 * h * h * v[1] * v[2] * 9
    for i in range(1, 7):
        f += sum(2 * h * h * cin * cout * k * k for _, cin, cout, k in stage_layers(i))
    return f


def timed(fn, iters):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def planted_maps(body, S):
    """Body stage-6 maps of four standing people whose face boxes are about S / 6 wide."""
    from oracle import openpose_oracle as O
    from tools.make_golden_openpose_face import skeleton
    P = body._plans(S, S, torch.device("cuda"))
    s = P["h"] / S
    e = S / 36
    people = [skeleton([S * (0.15 + 0.23 * k), S * 0.3], e, S / 1024) for k in range(4)]
    heat, paf = O.planted_maps([p * s / 8 - 0.5 for p in people], P["hp"] // 8, P["wp"] // 8, sigma=1.0, width=0.75)
    maps = np.concatenate([paf, heat, np.zeros_like(heat[:, :, :1])], 2).transpose(2, 0, 1)[None]
    return torch.from_numpy(np.ascontiguousarray(maps)).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    from oracle import openpose_face_oracle as FO
    from oracle import openpose_oracle as O
    from pfd_b200 import openpose, openpose_face
    body = openpose.BodyPose()
    body.load_state_dict(O.synth_state_dict(0), strict=True)
    face = openpose_face.FacePose()
    sd = FO.synth_state_dict(0, 0.35)
    face.load_state_dict(sd, strict=True)
    body, face = body.cuda().eval(), face.cuda().eval()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print(f"[openpose_face_perf] device: {q}")
    gf = face_flops()
    for N in (1, 4, 16):
        inp = torch.randn((N, 384, 384, 16), device="cuda").half()
        inp[..., 3:] = 0
        ms = timed(lambda: face.network(inp), a.iters)
        print(f"[openpose_face_perf] FaceNet, {N} faces: {ms:.2f} ms ({ms / N:.2f} ms per face), "
              f"{N * gf / (ms * 1e-3) / 1e12:.0f} TFLOP/s at {gf / 1e9:.0f} GFLOP per face")
    for S in (512, 1024):
        x = torch.rand((1, 3, S, S), device="cuda")
        maps = planted_maps(body, S)
        _, info = openpose_face.apply(body, face, x, debug=True, body_maps=maps)
        nf = len(info["face_boxes"])
        t_face = timed(lambda: openpose_face.apply(body, face, x, body_maps=maps), a.iters)
        t_body = timed(lambda: body.apply(x, maps=maps), a.iters)
        print(f"[openpose_face_perf] {S}x{S} planted bodies, {nf} faces: 'openpose_withface' {t_face:.2f} ms, "
              f"'openpose' {t_body:.2f} ms (both from the same stage-6 body maps)")
    with torch.no_grad():
        x = torch.rand((1, 3, 384, 384)) - 0.5
        sdg = {k: v.cuda() for k, v in sd.items()}
        ms = timed(lambda: FO.network(sdg, x.cuda()), a.iters)
    print(f"[openpose_face_perf] oracle fp32 eager FaceNet, one face: {ms:.2f} ms "
          f"({gf / (ms * 1e-3) / 1e12:.0f} TFLOP/s)")


if __name__ == "__main__":
    main()
