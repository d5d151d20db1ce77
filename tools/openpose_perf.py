"""CUDA-event time per ControlNet.preprocess(type='openpose') call (pfd_b200/openpose.py) with synthetic weights, at
several image sizes and batch 1 / 4, with the network's TFLOP/s counted from its shapes.  Prints one line per case and
the card's name and power limit."""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def network_flops(hp: int, wp: int) -> float:
    """Multiply-adds x 2 of bodypose_model on an hp x wp input, from its layer shapes."""
    from pfd_b200.openpose import VGG, _layers
    f, h, w = 0.0, hp, wp
    for v in VGG:
        if v == "pool":
            h, w = h // 2, w // 2
        else:
            f += 2 * h * w * v[1] * v[2] * 9
    for i in range(1, 7):
        for L in (1, 2):
            f += sum(2 * h * w * cin * cout * k * k for _, cin, cout, k in _layers(i, L))
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="512,768,1024,1536")
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    from oracle import openpose_oracle as O
    from pfd_b200 import openpose
    net = openpose.BodyPose()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    net = net.cuda().eval()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print(f"[openpose_perf] device: {q}")
    for S in (int(s) for s in a.sizes.split(",")):
        for B in (1, 4):
            x = torch.rand((B, 3, S, S), device="cuda")
            for _ in range(3):
                net.apply(x)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                net.apply(x)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.iters
            P = net._plans(S, S, x.device)
            tf = B * network_flops(P["hp"], P["wp"]) / (ms * 1e-3) / 1e12
            print(f"[openpose_perf] {B}x{S}x{S}: {ms:.2f} ms per preprocess call, network {tf:.1f} TFLOP/s over the "
                  "whole call")


if __name__ == "__main__":
    main()
