#!/usr/bin/env python
"""In-process A/B of one planner option (s3r_set_option): two models in ONE process, planned under option=off / option=on,
timed ALTERNATELY on the same sequences -- robust against the box-to-box and minute-to-minute clock / power drift that
makes separate bench.py runs differ by +-1.5 %.  Prints one JSON line per option.

    python tools/ab_inproc.py prefetch_b=1,0 [--rounds 12]
"""
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spann3r_b200 import Spann3R, _lib, synth  # noqa: E402

rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 12
specs = [a for a in sys.argv[1:] if "=" in a]
sd = synth.make_state_dict(sharpen=True)
frames = [[{"img": f["img"].cuda()} for f in synth.make_frames(10, 384, 512, seed0=1 + 100 * s)] for s in range(2)]
L = _lib.lib()
for spec in specs:
    name, vals = spec.split("=")
    a, b = (int(v) for v in vals.split(","))
    models = {}
    for v in (a, b):
        _lib.check(L.s3r_set_option(name.encode(), v), "s3r_set_option")
        m = Spann3R(dus3r_name=None)
        m.load_state_dict(sd, strict=True)
        m = m.cuda().eval()
        for i in range(3):
            m(frames[i % 2])                       # plans are built here, under this option value
        models[v] = m
    _lib.check(L.s3r_set_option(name.encode(), a), "s3r_set_option")
    torch.cuda.synchronize()
    ms = {a: [], b: []}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(rounds):
        for v in ((a, b) if r % 2 == 0 else (b, a)):
            e0.record()
            for i in range(2):
                models[v](frames[i])
            e1.record()
            torch.cuda.synchronize()
            ms[v].append(e0.elapsed_time(e1) / 2)
    ma, mb = statistics.median(ms[a]), statistics.median(ms[b])
    ratios = sorted(y / x for x, y in zip(ms[a], ms[b]))
    print(json.dumps({"option": name, "values": [a, b], "median_ms_per_seq": [ma, mb], "ratio_b_over_a_median": ratios[len(ratios) // 2],
                      "ratio_min_max": [ratios[0], ratios[-1]], "rounds": rounds,
                      "frames_per_s": [10 / (ma / 1e3), 10 / (mb / 1e3)]}), flush=True)
    del models
    torch.cuda.empty_cache()
