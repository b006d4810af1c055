#!/usr/bin/env python
"""The value stage (`s3r_engine_value`: value encoder + value_norm + value_out + `cur_v + feat_k1`) of the default model
against `Spann3R(use_feat=True)` (768-wide encoder, 16 heads of 48 run in 64-wide slots, fed with the decoder tokens).

    python tools/bench_value_stage.py [--res 224x224,384x512] [--batch 1] [--iters 50] [--warmup 10] [--mem-pos-enc]

Synthetic weights (synth.make_state_dict); the engine first runs one encode / decode / heads so that its inputs are real
activations.  Per (resolution, model) one JSON line: the mean of `--iters` value-stage calls timed with CUDA events
after `--warmup` untimed ones, and the launches / algorithmic tensor-core FLOPs of one call.  The first line names the
card and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def time_it(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", default="224x224,384x512", help="comma-separated HxW")
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--mem-pos-enc", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_value_stage: no CUDA device (timings need the GPU)")
    from spann3r_b200 import Spann3R, synth
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": torch.cuda.get_device_name(), "nvidia_smi": q, "batch": a.batch, "iters": a.iters,
                      "warmup": a.warmup, "mem_pos_enc": a.mem_pos_enc}), flush=True)
    for use_feat in (False, True):
        spec = synth.usefeat_spec() if use_feat else synth.load_spec()
        m = Spann3R(dus3r_name=None, use_feat=use_feat, mem_pos_enc=a.mem_pos_enc)
        m.load_state_dict(synth.make_state_dict(spec, seed=0, sharpen=True), strict=True)
        m = m.cuda().eval()
        for res in a.res.split(","):
            H, W = (int(v) for v in res.lower().split("x"))
            B = a.batch
            eng = m._engine_for(B, H, W)
            fr = synth.make_frames(2, H, W, batch=B)
            feats = eng.encode(torch.cat([f["img"] for f in fr]).cuda())
            f1, f2 = feats[:B].contiguous(), feats[B:].contiguous()
            with torch.no_grad():
                eng.decode(f1, f2)
                k1, _ = eng.keyheads(f1, f2)
                pts, _ = eng.heads()
            p1 = pts[0].contiguous()

            def call():
                return m._value(eng, p1, k1, H > W)
            call()
            torch.cuda.synchronize()
            eng.take_flops()
            eng.take_launches()
            call()
            flops, launches = eng.take_flops(), eng.take_launches()
            ms = time_it(call, a.iters, a.warmup)
            print(json.dumps({"model": "use_feat" if use_feat else "default", "res": [H, W], "batch": B, "ms": round(ms, 4),
                              "launches": launches, "gflop": round(flops / 1e9, 2),
                              "tflops": round(flops / ms / 1e9, 1)}), flush=True)
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
