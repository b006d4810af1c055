#!/usr/bin/env python
"""Offline reconstruction: the reference's pair-graph route against the native one, on the sharpened synthetic checkpoint.

Routes, alternated round by round in one process after a warm-up of every route and shape:
  graph        what demo.py / eval.py --offline do today, restated on the CUDA model: `inference(make_pairs(complete,
               symmetrize=True), model.dust3r, batch_size=2)` -- batches of 2 pairs symmetrised to 4 pair forwards, every
               map copied to the host -- then `offline_reconstruction(frames, graph)` with its serial next-best-view loop.
  max_batch=K  `offline_reconstruction(frames, max_batch=K)`: batched pair scores on the device, then next-best-view
               candidates scored K at a time.
Cases: F in {4, 10, 20} at 224 x 224 (the resolution demo.py / eval.py use) and F = 10 at 384 x 512.  Each time runs
between two device synchronisations.  Per route: median / min / max wall time, images encoded and engine decode calls in
one run, and whether idx_used equals the graph route's.  Prints a header line with the card's name and power limit,
then one JSON line per (case, route).

    python tools/bench_offline.py [--rounds 3] [--cases 4x224x224,10x224x224,20x224x224,10x384x512]
"""
import argparse
import contextlib
import io
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


class Counts:
    """Images encoded and decode calls of every engine, counted at the Engine class."""

    def __init__(self):
        from spann3r_b200.engine import Engine
        self.images = self.decodes = 0
        enc, dec = Engine.encode, Engine.decode

        def encode(eng, img):
            self.images += img.shape[0]
            return enc(eng, img)

        def decode(eng, f1, f2, want_all=False):
            self.decodes += 1
            return dec(eng, f1, f2, want_all)
        Engine.encode, Engine.decode = encode, decode

    def take(self):
        out = (self.images, self.decodes)
        self.images = self.decodes = 0
        return out


def graph_route(m, frames):
    """dust3r.inference.inference(make_pairs(frames, 'complete', symmetrize=True), m.dust3r, batch_size=2) as the
    reference runs it, then offline_reconstruction(frames, graph)."""
    n = len(frames)
    pairs = [(i, j) for i in range(n) for j in range(i)]
    pairs += [(j, i) for i, j in pairs]
    v1, v2, c1, c2 = [], [], [], []
    for s in range(0, len(pairs), 2):
        chunk = pairs[s: s + 2]
        a = [x for i, j in chunk for x in (i, j)]           # _interleave_imgs of the symmetrised batch
        b = [x for i, j in chunk for x in (j, i)]
        r1, r2 = m.dust3r({"img": torch.cat([frames[i]["img"] for i in a])}, {"img": torch.cat([frames[i]["img"] for i in b])})
        v1 += a
        v2 += b
        c1 += list(r1["conf"].cpu().unbind(0))
        c2 += list(r2["conf"].cpu().unbind(0))
        r1["pts3d"].cpu(), r2["pts3d_in_other_view"].cpu()   # to_cpu of the whole result, as the reference does
    graph = {"view1": {"idx": v1}, "view2": {"idx": v2}, "pred1": {"conf": c1}, "pred2": {"conf": c2}}
    return m.offline_reconstruction(frames, graph)[2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--cases", default="4x224x224,10x224x224,20x224x224,10x384x512")
    ap.add_argument("--batches", default="1,4,8")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_offline needs the GPU")
    from spann3r_b200 import Spann3R, synth
    m = Spann3R(dus3r_name=None)
    m.load_state_dict(synth.make_state_dict(sharpen=True), strict=True)
    m = m.cuda().eval()
    counts = Counts()
    print(json.dumps({"card": card()}), flush=True)
    for case in args.cases.split(","):
        n, H, W = (int(x) for x in case.split("x"))
        frames = [{"img": f["img"].cuda()} for f in synth.make_frames(n, H, W)]
        routes = {"graph": lambda: graph_route(m, frames)}
        for mb in (int(b) for b in args.batches.split(",")):
            routes[f"max_batch={mb}"] = (lambda mb=mb: m.offline_reconstruction(frames, max_batch=mb)[2])
        times = {r: [] for r in routes}
        used, work = {}, {}
        with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
            for r, run in routes.items():       # warm-up: engines and plans of every batch size
                used[r] = run()
                work[r] = counts.take()
            for _ in range(args.rounds):
                for r, run in routes.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    idx = run()
                    torch.cuda.synchronize()
                    times[r].append(time.perf_counter() - t0)
                    assert idx == used[r], (r, idx, used[r])
                counts.take()
        for r in routes:
            ts = sorted(times[r])
            print(json.dumps({"case": case, "route": r, "s_median": round(ts[len(ts) // 2], 4), "s_min": round(ts[0], 4),
                              "s_max": round(ts[-1], 4), "images_encoded": work[r][0], "decode_calls": work[r][1],
                              "idx_used_equal_to_graph": used[r] == used["graph"], "idx_used": used[r]}), flush=True)


if __name__ == "__main__":
    main()
