#!/usr/bin/env python
"""GPU PnP (s3r_pnp_ransac) vs cv2.solvePnPRansac on the host, per 512x384 frame (demo.py:166-180 runs the latter once per
frame on a CPU copy of the pointmap).  Prints one JSON line; run on the GPU box:  python tools/bench_pnp.py"""
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spann3r_b200 import synth  # noqa: E402
from spann3r_b200.postprocess import solve_pnp_ransac  # noqa: E402

B = 10
case = synth.PNP_CASES[1]
maps = [synth.make_pointmap_case(case[0], case[1], case[2], case[3], case[4], case[5], case[6], 100 + j) for j in range(B)]
K = maps[0][1]
batch = torch.stack([torch.from_numpy(m[0]) for m in maps]).cuda()
for _ in range(3):
    solve_pnp_ransac(batch, K)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(10):
    ok, rvec, tvec, inl = solve_pnp_ransac(batch, K)
e1.record()
torch.cuda.synchronize()
gpu_ms = e0.elapsed_time(e1) / 10 / B
# end to end incl. reading the poses back (what a caller needs on the host)
t0 = time.time()
for _ in range(10):
    ok, rvec, tvec, inl = solve_pnp_ransac(batch, K)
    poses = torch.cat((rvec, tvec), 1).cpu()
e2e_ms = (time.time() - t0) / 10 / B * 1e3
res = {"what": "camera pose per 512x384 frame, batch of 10 frames per call, 20 % outliers", "gpu_ms_per_frame": gpu_ms,
       "gpu_e2e_ms_per_frame_incl_pose_readback": e2e_ms, "all_ok": bool(ok.all()),
       "algorithmic_bytes_per_frame": 384 * 512 * 12 * (2 + 16), "passes": "score + mask + 16 Gauss-Newton passes"}
try:
    import cv2
    H, W = case[0], case[1]
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    p2 = np.stack((u, v), -1).reshape(-1, 2).astype(np.float32)
    t0 = time.time()     # ONE frame: on a contended many-core host cv2 took 7.6 s per frame
    cv2.solvePnPRansac(maps[0][0].reshape(-1, 3), p2, K.astype(np.float32), np.zeros(4, np.float32))
    res["cv2_ms_per_frame"] = (time.time() - t0) * 1e3
    res["cv2"] = cv2.__version__
    res["speedup_e2e"] = res["cv2_ms_per_frame"] / e2e_ms
except Exception as ex:  # cv2 is the reference's dependency, not ours
    res["cv2_ms_per_frame"] = None
    res["cv2_error"] = repr(ex)[:100]
print(json.dumps(res))
