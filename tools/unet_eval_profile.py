"""One CFG-pair UNet evaluation (batch 4 -> 8 rows, 64x64 latents) run eagerly twice: meant to be run under
`ncu --metrics gpu__time_duration.sum --cache-control none --clock-control none` with PFD_GEMM_TRACE=1 so that
the per-launch device times can be joined with the GEMM call descriptors."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench

net = bench.synth_net(bench.CONFIGS[2]).half()
net.to("cuda")
B, L = 4, 64
torch.manual_seed(0)
img = torch.rand((1, 3, 512, 512), device="cuda").half()
c = net.ctx_encode(img, "image").repeat(B, 1, 1)
u = torch.zeros_like(c)
c_full = torch.cat([u, c])
prep = net.prepare_context(c_full, "image")
x = torch.randn((B, 4, L, L), device="cuda", dtype=torch.float16)
t_in = torch.full((2 * B,), 501, device="cuda", dtype=torch.long)
c_info = {"type": "image", "c": prep["c"], "_pfd_prepared": prep, "control": None}
for i in range(2):
    torch.cuda.synchronize()
    sys.stderr.write("EVALMARK %d\n" % i)
    sys.stderr.flush()
    net.apply_model({"type": "image", "x": torch.cat([x, x])}, t_in, c_info)
torch.cuda.synchronize()
sys.stderr.write("EVALMARK end\n")
