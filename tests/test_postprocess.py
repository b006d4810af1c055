"""Post-path focal estimate (SURVEY.md section 8f rank 4, first step): oracle vs golden values from the REAL reference
function (CPU), CUDA path vs both (GPU).  Floating point: sums over ~2e5 pixels in a different order -> 1e-4 relative."""
import importlib.util
import json
import os

import pytest
import torch

from conftest import GOLDEN, ROOT

TOL = 1e-4
HERE = os.path.dirname(os.path.abspath(__file__))


def _pointmap():
    spec = importlib.util.spec_from_file_location("make_golden_focal", os.path.join(ROOT, "tools", "make_golden_focal.py"))
    src = open(spec.origin).read().replace('from dust3r.post_process import estimate_focal_knowing_depth  # noqa: E402', '')
    ns = {"__name__": "golden_helper", "__file__": spec.origin}
    exec(compile(src, spec.origin, "exec"), ns)
    return ns["pointmap"]


def _cases():
    return json.load(open(os.path.join(GOLDEN, "focal.json")))["cases"]


def test_oracle_matches_reference_golden():
    from oracle.postprocess_oracle import focal_weiszfeld
    pm = _pointmap()
    for c in _cases():
        pts = pm(c["seed"], c["B"], c["H"], c["W"], c["f_true"])
        f = focal_weiszfeld(pts, (c["W"] / 2, c["H"] / 2))
        for a, b in zip(f.tolist(), c["focal"]):
            assert abs(a - b) <= 2e-6 * abs(b), (a, b)
            assert abs(a - c["f_true"]) < 0.05 * c["f_true"]      # and it does recover the synthetic camera


def test_median_mode_oracle_and_device_math_are_bit_exact(tmp_path):
    """focal_mode='median' selects an ELEMENT of the vote set, so the bar is bit-exact: (a) the oracle restatement and (b) the
    product's device math header (csrc/focal_math.cuh: votes + ordered keys) driven on the host through the same 4 x 8-bit
    radix select the CUDA kernels perform (tests/native/focal_host_check.cpp), both against the REAL reference's values."""
    import ctypes as C
    import subprocess
    from oracle.postprocess_oracle import focal_median
    so = str(tmp_path / "focal_host_check.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-x", "c++",
                           os.path.join(HERE, "native", "focal_host_check.cpp"), "-o", so])
    L = C.CDLL(so)
    L.focal_median_host.restype = C.c_float
    L.focal_median_host.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float]
    pm = _pointmap()
    for c in _cases():
        pts = pm(c["seed"], c["B"], c["H"], c["W"], c["f_true"])
        f = focal_median(pts, (c["W"] / 2, c["H"] / 2))
        assert f.tolist() == c["focal_median"]
        for b in range(c["B"]):
            p = pts[b].contiguous()
            assert L.focal_median_host(p.data_ptr(), c["H"], c["W"], c["W"] / 2, c["H"] / 2) == c["focal_median"][b]
    # all votes NaN -> NaN, like torch.nanmedian
    nanmap = torch.full((8, 8, 3), float("nan"))
    assert L.focal_median_host(nanmap.data_ptr(), 8, 8, 4.0, 4.0) != L.focal_median_host(nanmap.data_ptr(), 8, 8, 4.0, 4.0)


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100")
def test_cuda_focal_median_is_bit_exact():
    """The CUDA radix select (s3r_focal_median) against the real reference's values, bit for bit."""
    from spann3r_b200.postprocess import estimate_focal_knowing_depth
    pm = _pointmap()
    for c in _cases():
        pts = pm(c["seed"], c["B"], c["H"], c["W"], c["f_true"])
        f = estimate_focal_knowing_depth(pts.cuda(), (c["W"] / 2, c["H"] / 2), focal_mode="median").cpu()
        assert f.tolist() == c["focal_median"], (f.tolist(), c["focal_median"])
    nanmap = torch.full((1, 16, 16, 3), float("nan")).cuda()
    assert torch.isnan(estimate_focal_knowing_depth(nanmap, (8.0, 8.0), focal_mode="median")).all()


@pytest.mark.gpu
def test_cuda_focal_matches_reference():
    from oracle.postprocess_oracle import focal_weiszfeld
    from spann3r_b200.postprocess import estimate_focal_knowing_depth
    pm = _pointmap()
    for c in _cases():
        pts = pm(c["seed"], c["B"], c["H"], c["W"], c["f_true"])
        pp = torch.tensor((c["W"] / 2, c["H"] / 2))
        f = estimate_focal_knowing_depth(pts.cuda(), pp, focal_mode="weiszfeld").cpu()
        ref = focal_weiszfeld(pts, pp)
        for a, b, g in zip(f.tolist(), ref.tolist(), c["focal"]):
            assert abs(a - g) <= TOL * abs(g), (a, g)
            assert abs(a - b) <= TOL * abs(b), (a, b)
    # clipping (min_focal / max_focal in units of the 60-degree base focal, post_process.py:55-56)
    c = _cases()[0]
    pts = pm(c["seed"], c["B"], c["H"], c["W"], c["f_true"])
    f = estimate_focal_knowing_depth(pts.cuda(), (c["W"] / 2, c["H"] / 2), focal_mode="weiszfeld", min_focal=1.0,
                                     max_focal=1.0).cpu()
    assert abs(float(f[0]) - max(c["H"], c["W"]) / 1.1547005383792515) < 1e-2
