"""Multi-GPU batch split on real GPUs (SURVEY.md §8e, VERDICT r1 item 8): ONE request of B images sharded over the ranks
with pfd_b200/parallel.py - rank-0 SeeCoder encode -> NCCL broadcast, full-batch randn with the request seed + slice,
all-gather of the decoded images - must reproduce the single-GPU result for the same seed.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29533 tools/split_check.py [--deterministic]

--deterministic runs every rank in deterministic mode (pfd_b200.set_deterministic) and requires the gathered batch to
equal the single-GPU batch bit for bit.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--deterministic", action="store_true")
    args = ap.parse_args()
    world, rank, local = int(os.environ["WORLD_SIZE"]), int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from pfd_b200 import DDIMSampler, get_model, model_cfg_bank, parallel as par
    from pfd_b200.weights import SCHEDULE_BUFFERS, fill_module_
    if args.deterministic:
        from pfd_b200 import set_deterministic
        set_deterministic(True)
    net = get_model()(model_cfg_bank()("pfd_seecoder"))
    fill_module_(net, seed=0, skip=SCHEDULE_BUFFERS)
    net = net.half()
    net.to("cuda")
    B, L, steps, seed = int(os.environ.get("SPLIT_B", "5")), 32, 4, 20          # 5 images over 2 ranks: ragged shards
    img = torch.rand((1, 3, 256, 256), generator=torch.Generator().manual_seed(1)).cuda().half()
    sampler = DDIMSampler(net)

    def run(xt, c1):
        n = xt.shape[0]
        c = c1.repeat(n, 1, 1)
        x, _ = sampler.sample(steps=steps, x_info={"type": "image", "xt": xt},
                              c_info={"type": "image", "conditioning": c, "unconditional_conditioning": torch.zeros_like(c),
                                      "unconditional_guidance_scale": 2.0, "control": None},
                              shape=[n, 4, L, L], verbose=False, eta=0.0)
        return net.vae_decode(x, "image")

    c1 = net.ctx_encode(img, "image") if rank == 0 else None
    c1 = par.broadcast_conditioning(c1, 0, shape=(1, 148, 768), dtype=torch.float16, device="cuda")
    xt = par.sharded_noise([B, 4, L, L], seed=seed, rank=rank, world=world, device="cuda", dtype=torch.float16)
    full = par.gather_images(run(xt, c1), B)
    res = None
    if rank == 0:
        torch.manual_seed(seed)                                               # the single-GPU reference RNG call (ddim.py:105)
        xt_full = torch.randn([B, 4, L, L], device="cuda", dtype=torch.float16)
        a, b = par.shard_range(B, world, 0)
        same_noise = bool(torch.equal(xt_full[a:b], xt))
        single = run(xt_full, c1)
        diff = (full.float() - single.float())
        rel = (diff.pow(2).mean() / single.float().pow(2).mean()).sqrt().item()
        res = {"world": world, "batch": B, "shards": [par.shard_range(B, world, r) for r in range(world)],
               "noise_slice_equals_single_gpu_randn": same_noise, "rel_rms_gathered_vs_single_gpu": rel,
               "max_abs": diff.abs().max().item(), "shape": list(full.shape),
               "deterministic": args.deterministic, "exact_equal": bool(torch.equal(full, single))}
        print("SPLIT_RESULT " + json.dumps(res), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0 and not (res["noise_slice_equals_single_gpu_randn"] and res["rel_rms_gathered_vs_single_gpu"] < 3e-3
                          and (res["exact_equal"] or not args.deterministic)):
        sys.exit(1)


if __name__ == "__main__":
    main()
