#!/usr/bin/env python
"""BASELINE config[4] / SURVEY.md §8d config 5: the reference's DDP training step on synthetic views.

    torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tools/train_step_bench.py \
        [--impl ours|reference] [--batch 4] [--frames 10] [--res 224] [--steps 5] [--warmup 2]

One step = `spann3r/training.py:216-228`: forward of a batch of `--batch` sequences per rank -> `ConfLoss_t(Regr3D_t(L21,
norm_mode='avg_dis', fix_first=False), alpha=0.4).compute_frame_loss` (the REFERENCE's criterion, imported from the staged
copy under oracle/_ref: losses are callers of the path, SURVEY.md §2) -> backward -> DDP gradient all-reduce (NCCL, 2.63 GB
fp32 per rank, `DistributedDataParallel(find_unused_parameters=True, static_graph=True)` as `training.py:322-325`) -> AdamW.

--impl ours: `spann3r_b200.Spann3R` in training mode = the sm_90a kernels forward (attn_thresh=0, Philox memory dropout,
ungated add_mem) + the PyTorch-RECOMPUTE backward of `spann3r_b200/train.py` (native dgrad / wgrad not written yet: backward
time is eager PyTorch and is reported as such).  --impl reference: the unmodified reference module, eager PyTorch both ways.

Rank 0 prints one JSON line: steps/s (device time, max over ranks), forward / backward split, and the EXPOSED all-reduce time
= step time with gradient synchronisation minus step time under `no_sync()` (same compute, no collective)."""
import argparse
import contextlib
import io
import json
import os
import sys
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def synthetic_views(B, F_, res, device, seed):
    """Views with the keys `compute_frame_loss` reads (spann3r/loss.py:138-178): img, pts3d (world frame), valid_mask,
    camera_pose (cam-to-world), true_shape; a smooth random surface per frame."""
    g = torch.Generator().manual_seed(seed)
    views = []
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, res), torch.linspace(-1, 1, res), indexing="ij")
    for f in range(F_):
        img = torch.rand(B, 3, res, res, generator=g) * 2 - 1
        z = 2.0 + 0.3 * torch.rand(B, 1, 1, generator=g) + 0.2 * torch.sin(3 * xs + f)[None] * torch.rand(B, 1, 1, generator=g)
        pts = torch.stack((xs[None] * z, ys[None] * z, z), dim=-1)
        pose = torch.eye(4).repeat(B, 1, 1)
        pose[:, :3, 3] = 0.05 * f * torch.randn(B, 3, generator=g)
        views.append({"img": img.to(device), "pts3d": (pts + pose[:, None, None, :3, 3]).to(device),
                      "valid_mask": torch.ones(B, res, res, dtype=torch.bool, device=device), "camera_pose": pose.to(device),
                      "true_shape": torch.tensor([[res, res]] * B)})
    return views


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    try:     # torchrun exports OMP_NUM_THREADS=1: building the models is host work, give each rank its share of the cores
        torch.set_num_threads(max(1, len(os.sched_getaffinity(0)) // 2 // max(world, 1)))
    except Exception:
        pass
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    from baseline import ref_loader
    from spann3r_b200 import synth
    sd = synth.make_state_dict(sharpen=True)
    with contextlib.redirect_stdout(io.StringIO()):
        if a.impl == "reference":
            model = ref_loader.build_model(sd, synth.DUST3R_ARGS).to(dev)
        else:
            from spann3r_b200 import Spann3R
            ref_loader.load()                      # only for the criterion below
            model = Spann3R(dus3r_name=None)
            model.load_state_dict(sd, strict=True)
            model = model.to(dev)
    from dust3r.losses import L21          # noqa: the reference's criterion (staged copy)
    from spann3r.loss import ConfLoss_t, Regr3D_t   # noqa
    criterion = ConfLoss_t(Regr3D_t(L21, norm_mode="avg_dis", fix_first=False), alpha=0.4).to(dev)
    model.train()
    ddp = model
    if world > 1:
        ddp = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local], find_unused_parameters=True, static_graph=True)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-6, betas=(0.9, 0.95))
    batch = synthetic_views(a.batch, a.frames, a.res, dev, seed=1000 * rank + 1)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]

    def step(sync=True):
        opt.zero_grad(set_to_none=True)
        ctx = contextlib.nullcontext() if (sync or world == 1) else ddp.no_sync()
        with ctx, contextlib.redirect_stdout(io.StringIO()):
            ev[0].record()
            preds, preds_all = ddp(batch)
            ev[1].record()
            loss, details, factor = criterion.compute_frame_loss(batch, preds_all)
            loss = loss + factor
            loss.backward()
            ev[2].record()
        opt.step()
        ev[3].record()
        return loss

    def timed(n, sync):
        tot = [0.0, 0.0, 0.0]
        last = None
        for _ in range(n):
            if world > 1:
                dist.barrier()
            torch.cuda.synchronize(dev)
            last = step(sync)
            torch.cuda.synchronize(dev)
            tot[0] += ev[0].elapsed_time(ev[3]); tot[1] += ev[0].elapsed_time(ev[1]); tot[2] += ev[1].elapsed_time(ev[2])
        t = torch.tensor([x / n for x in tot], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t.tolist(), float(last)

    t0 = time.time()
    for _ in range(a.warmup):
        l0 = float(step(True))
    (ms, fwd, bwd), l1 = timed(a.steps, True)
    (ms_ns, _, _), _ = timed(max(2, a.steps // 2), False) if world > 1 else ((ms, 0, 0), 0)
    if rank == 0:
        nparam = sum(p.numel() for p in model.parameters())
        print(json.dumps({
            "what": "DDP training step (SURVEY 8d config 5)", "impl": a.impl, "n_gpus": world, "batch_per_gpu": a.batch,
            "frames": a.frames, "resolution": a.res, "steps": a.steps, "warmup": a.warmup,
            "ms_per_step": ms, "steps_per_s": 1e3 / ms, "sequences_per_s": world * a.batch * 1e3 / ms,
            "forward_ms": fwd, "loss_backward_ms": bwd, "optimizer_ms": ms - fwd - bwd,
            "ms_per_step_no_sync": ms_ns, "exposed_allreduce_ms": max(0.0, ms - ms_ns) if world > 1 else None,
            "gradient_bytes_per_rank": 4 * nparam, "loss_first": l0, "loss_last": l1,
            "backward": "PyTorch recompute (spann3r_b200/train.py)" if a.impl == "ours" else "PyTorch autograd (reference)",
            "forward": "sm_90a kernels (libspann3r_b200.so)" if a.impl == "ours" else "PyTorch eager (reference)",
            "wall_s": time.time() - t0}), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
