#!/usr/bin/env python
"""Independent sequences batched (`Spann3R.forward_sequences`) against one sequence at a time (`Spann3R.forward`).

Two workloads on the sharpened synthetic checkpoint:
  eval     16 sequences at 224 x 224, lengths drawn with a seed from 8..40 (the resolution demo.py / eval.py use; real
           datasets mix sequence lengths like this)
  config3  8 sequences of 10 frames at 384 x 512 (BASELINE config 3's per-GPU shape)
Arms: `forward` per sequence (B = 1) and `forward_sequences` with max_batch 2, 4 and 8, alternated round by round in one
process after a warm-up of every arm.  Each arm's time runs between two device synchronisations; frames/s counts the
input frames.  The worst per-sequence rel-L2 of each batched arm is taken against the B = 1 arm of the same round.
Prints one JSON line per (workload, arm) and a header line with the card's name and power limit.

    python tools/bench_sequences.py [--rounds 3] [--workloads eval,config3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [x.strip() for x in q.split(",")[:2]]
    except Exception as ex:  # the numbers are still reported, without the power limit
        info["power_limit"] = f"unavailable ({ex!r})"
    return info


def workloads(names):
    from spann3r_b200 import synth
    out = {}
    if "eval" in names:
        g = torch.Generator().manual_seed(2024)
        lengths = torch.randint(8, 41, (16,), generator=g).tolist()
        out["eval"] = [synth.make_frames(n, 224, 224, seed0=1000 * s + 1) for s, n in enumerate(lengths)]
    if "config3" in names:
        out["config3"] = [synth.make_frames(10, 384, 512, seed0=100 * s + 1) for s in range(8)]
    return out


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def worst_rel(res, ref):
    w = 0.0
    for (p, _), (r, _) in zip(res, ref):
        for a, b in zip(p, r):
            for k in b:
                w = max(w, rel_l2(a[k], b[k]))
    return w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default="eval,config3")
    ap.add_argument("--batches", default="2,4,8")
    args = ap.parse_args()
    from spann3r_b200 import Spann3R, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_sequences needs the GPU")
    m = Spann3R(dus3r_name=None)
    m.load_state_dict(synth.make_state_dict(sharpen=True), strict=True)
    m = m.cuda().eval()
    print(json.dumps({"card": card()}), flush=True)
    batches = [int(b) for b in args.batches.split(",")]
    for name, seqs in workloads(args.workloads.split(",")).items():
        n_frames = sum(len(q) for q in seqs)
        arms = {"B1": lambda: [m(q) for q in seqs]}
        for mb in batches:
            arms[f"max_batch={mb}"] = (lambda mb=mb: m.forward_sequences(seqs, max_batch=mb))
        for run in arms.values():           # warm-up: engines, plans, every bank length the timed rounds meet
            run()
        torch.cuda.synchronize()
        times = {a: [] for a in arms}
        worst = {a: 0.0 for a in arms}
        for _ in range(args.rounds):
            outs = {}
            for a, run in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                outs[a] = run()
                torch.cuda.synchronize()
                times[a].append(time.perf_counter() - t0)
            for a in arms:
                worst[a] = max(worst[a], worst_rel(outs[a], outs["B1"]))
            del outs
        for a in arms:
            ts = sorted(times[a])
            print(json.dumps({"workload": name, "arm": a, "sequences": len(seqs), "frames": n_frames,
                              "lengths": [len(q) for q in seqs] if name == "eval" else None,
                              "frames_per_s_median": round(n_frames / ts[len(ts) // 2], 1),
                              "frames_per_s_min": round(n_frames / ts[-1], 1),
                              "frames_per_s_max": round(n_frames / ts[0], 1),
                              "worst_rel_l2_vs_B1": worst[a]}), flush=True)


if __name__ == "__main__":
    main()
