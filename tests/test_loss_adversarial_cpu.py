"""The criteria without a GPU, at the inputs where they go wrong:
  * the per-pixel math header (csrc/loss_math.cuh) compiled for the CPU (tests/native/loss_host_check.cpp) against a
    numpy float32 restatement in the reference's operation order, bit for bit, on random and adversarial values
    (+-0.0, subnormals, +-inf, NaN, one ulp either side of a tie); conf_term and pred_grad, which call logf / work in
    fp64, against fp64 within a stated bound; the radix-select median against numpy's sorted lower median;
  * the PyTorch restatement (oracle/loss_oracle.py) against the reference's own criteria on the adversarial cases of
    tests/golden/loss_adv_*.npz (tools/make_golden_loss_adv.py), at full resolution, NaN for NaN."""
import json
import os

import numpy as np
import pytest
import torch

import loss_host as lh
from conftest import GOLDEN
from oracle import loss_oracle as lo
from spann3r_b200 import synth
from test_loss_cpu import oracle_kwargs, slot_tensors

U = 2.0 ** -24          # unit roundoff of fp32
F32 = np.float32
ADV = sorted(synth.LOSS_ADV_CASES)


def _special():
    one_up, one_down = np.nextafter(F32(1), F32(2)), np.nextafter(F32(1), F32(0))
    return np.array([0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, -1.1754942e-38, 1.17549435e-38, 3e-39, np.inf, -np.inf,
                     np.nan, 1.0, -1.0, one_up, one_down, 3.0, np.nextafter(F32(3), F32(4)), 3.4028235e38,
                     -3.4028235e38, 2.0 ** -126, 0.5, 1e20, -1e-20], F32)


def adversarial(rng, n):
    """n float32 values: a third random normal, a third log-uniform over the whole fp32 range with random signs, a
    third drawn from the special values above."""
    a = rng.standard_normal(n).astype(F32)
    b = (rng.choice([-1, 1], n) * 10.0 ** rng.uniform(-44, 38, n)).astype(F32)
    c = rng.choice(_special(), n)
    return rng.permutation(np.concatenate([a, b, c])[:n])


def same_bits(a, b):
    """Equal bit patterns, with any NaN equal to any NaN (the payload is not part of the arithmetic's contract)."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a.view(np.uint32)[~na], b.view(np.uint32)[~nb]))


# numpy float32 restatement, every step rounded, in the reference's order
def np_norm3(v):
    return np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])


def np_align(p, factor, shift, mul):
    f, s, m = F32(factor), F32(shift), F32(mul)
    return np.stack([(p[:, 0] / f) * m, (p[:, 1] / f) * m, ((p[:, 2] / f) - s) * m], 1)


def np_stage_value(p, factor, shift, centre, kind):
    f = F32(factor)
    x, y, z = p[:, 0] / f, p[:, 1] / f, p[:, 2] / f
    if kind == 0:
        return z
    zs = z - F32(shift)
    if kind in (1, 2, 3):
        return (x, y, zs)[kind - 1]
    c = np.asarray(centre, F32)
    return np_norm3(np.stack([x - c[0], y - c[1], zs - c[2]], 1))


def np_order_key(v):
    u = np.asarray(v, F32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


@pytest.fixture(scope="module")
def rng():
    return np.random.default_rng(20261018)


def _vectors(rng, n):
    return adversarial(rng, 3 * n).reshape(n, 3)


def test_norm3_l21_align_stage_values_are_bit_exact(rng):
    with np.errstate(all="ignore"):
        for trial in range(4):
            n = 4096
            p, q = _vectors(rng, n), _vectors(rng, n)
            if trial == 1:                       # ties: q one ulp either side of p, or equal
                q = np.nextafter(p, rng.choice([-np.inf, np.inf], p.shape).astype(F32))
                q[::3] = p[::3]
            assert same_bits(lh.norm3(p), np_norm3(p))
            u, d = lh.l21(p, q)
            assert same_bits(u, p - q) and same_bits(d, np_norm3(p - q))
            for factor, shift, mul in [(1.0, 0.0, 1.0), (0.37, 1.25, 2.5), (1e-8, -3.0, 1e-3), (3e-39, 0.0, 7.0),
                                       (np.inf, 1.0, 1.0), (2.0, np.nan, 1.0), (1.5, -0.0, np.inf), (-0.0, 0.0, 1.0)]:
                assert same_bits(lh.align(p, factor, shift, mul), np_align(p, factor, shift, mul)), (factor, shift, mul)
                centre = adversarial(rng, 3)
                for kind in range(5):
                    assert same_bits(lh.stage_value(p, factor, shift, centre, kind),
                                     np_stage_value(p, factor, shift, centre, kind)), (factor, shift, kind)
    # identity alignment leaves every coordinate bit-identical (the criteria without normalisation rely on it)
    p = _vectors(rng, 1024)
    assert same_bits(lh.align(p, 1.0, 0.0, 1.0), p)


def test_order_key_is_monotone_and_inverts(rng):
    v = adversarial(rng, 1 << 14)
    v = v[~np.isnan(v)]
    k = lh.order_key(v)
    assert np.array_equal(k, np_order_key(v))
    assert same_bits(lh.key_value(k), v)
    o = np.argsort(k, kind="stable")
    s = v[o]
    assert np.all(s[:-1] <= s[1:])                              # key order is float order
    # -0.0 sorts just below +0.0, and every other neighbour pair keeps its float order strictly
    assert lh.order_key(np.array([-0.0], F32))[0] + 1 == lh.order_key(np.array([0.0], F32))[0]
    assert np.all(np.diff(lh.order_key(np.array([-np.inf, -3.4028235e38, -1e-45, -0.0, 0.0, 1e-45, 3.4028235e38,
                                                 np.inf], F32)).astype(np.int64)) > 0)


def test_conf_term_within_fp64_bound(rng):
    """d c - alpha log c: logf of the C library and np.log / CUDA's logf may differ by an ulp, so the bound is on the
    fp64 value: 2 roundings of the products, 1 of the difference and 1 ulp of log, each <= u of its operand:
    |err| <= 4 u (|d c| + alpha |log c|) (+ the smallest subnormal for results near 0)."""
    n = 1 << 14
    d = np.abs(rng.standard_normal(n)).astype(F32) * F32(3)
    d[:64] = 0.0
    c = (1 + np.exp(rng.standard_normal(n))).astype(F32)
    c[64:128] = 1.0
    c[128:192] = 1e30
    c[192:256] = np.nextafter(F32(1), F32(2))
    for alpha in (0.0, 0.2, 0.4, 1.0):
        got = lh.conf_term(d, c, alpha).astype(np.float64)
        dd, cc = d.astype(np.float64), c.astype(np.float64)
        ref = dd * cc - np.float64(F32(alpha)) * np.log(cc)
        bound = 4 * U * (np.abs(dd * cc) + alpha * np.abs(np.log(cc))) + 1e-45
        assert np.all(np.abs(got - ref) <= bound), (alpha, np.max(np.abs(got - ref) / bound))
        if alpha == 0.0:
            assert same_bits(lh.conf_term(d, c, alpha), d * c - F32(0) * np.log(c))


def test_pred_grad_within_fp64_bound(rng):
    """pred_grad against the same formula in fp64 with the exact fp64 norm: the header takes |p| as the fp32 norm3
    (<= 3 u relative: 2 additions, 1 square root, the squares' roundings inside them) and rounds the result to fp32
    (u), so |err| <= 8 u (|g_d scale / d| |u| + |coef / (|p| (1 + |p|))| |p|) + the fp32 subnormal floor.  d == 0 and
    p == 0 give exactly 0 for their term, as torch's norm backward."""
    n = 1 << 13
    p = rng.standard_normal((n, 3)).astype(F32) * F32(2)
    q = rng.standard_normal((n, 3)).astype(F32)
    q[:256] = p[:256]                                          # d == 0
    p[256:300] = 0.0                                           # |p| == 0
    q[300:400] = np.nextafter(p[300:400], F32(np.inf))         # d at the ulp scale: the ill-conditioned end
    u, d = lh.l21(p, q)
    for g_d, scale, coef, lg in [(0.7, 1.3, 0.0, 0), (1.0, 2.0, -0.25, 0), (-3e-3, 0.5, 1e-2, 1), (0.0, 1.0, 0.3, 1),
                                 (1e30, 1.0, 0.0, 0)]:
        got = lh.pred_grad(p, u, d, g_d, scale, coef, lg).astype(np.float64)
        pd, ud, dd = p.astype(np.float64), u.astype(np.float64), d.astype(np.float64)
        nrm = np.linalg.norm(pd, axis=1)
        with np.errstate(all="ignore"):
            s1 = np.where(dd > 0, g_d * scale / dd, 0.0)[:, None]
            s2 = np.where(nrm > 0, coef / nrm / (1.0 + nrm if lg else 1.0), 0.0)[:, None]
        ref = s1 * ud + s2 * pd
        bound = 8 * U * (np.abs(s1) * np.abs(ud) + np.abs(s2) * np.abs(pd)) + 1e-45
        assert np.all(np.abs(got - ref) <= bound), (g_d, scale, coef, lg)
        if coef == 0.0:
            assert np.all(got[:256] == 0.0) and not np.signbit(got[:256]).any()


def _np_lower_median(v):
    v = np.sort(v[~np.isnan(v)], kind="stable")
    return v[(len(v) - 1) // 2] if len(v) else F32(np.nan)


@pytest.mark.parametrize("kind", range(5))
def test_radix_median_is_the_lower_median(rng, kind):
    """The host radix select over stage values: the lower median of numpy's sort, on sets with many ties at the middle
    ranks, ties straddling rank (n - 1) / 2, +-inf and NaN among the values, odd / even / 0 / 1 / 2 valid values."""
    with np.errstate(all="ignore"):
        for trial in range(12):
            n = int(rng.choice([1, 2, 3, 4, 257, 1000, 4096]))
            p = rng.standard_normal((n, 3)).astype(F32)
            if trial % 3 == 1:                              # heavy ties: values from a 3-element alphabet
                p = rng.choice(np.array([-1.5, 0.25, 2.0], F32), (n, 3))
            if trial % 3 == 2:
                p[rng.random((n, 3)) < 0.05] = np.inf
                p[rng.random((n, 3)) < 0.05] = -np.inf
                p[rng.random((n, 3)) < 0.1] = np.nan
            valid = rng.random(n) < 0.8
            if trial == 0:
                valid[:] = False
            factor, shift = F32(rng.uniform(0.5, 2)), F32(rng.standard_normal())
            centre = rng.standard_normal(3).astype(F32)
            vals = np_stage_value(p, factor, shift, centre, kind)[valid]
            got = lh.median(p, valid, factor, shift, centre, kind)
            ref = _np_lower_median(vals)
            assert same_bits(got, ref) or (got == 0 and ref == 0), (trial, got, ref)
            t = torch.from_numpy(vals).nanmedian() if len(vals) else torch.tensor(float("nan"))
            assert (np.isnan(got) and t.isnan()) or got == t.item()
    # an even count whose two middle values differ: the lower one
    p = np.zeros((4, 3), F32)
    p[:, 2] = [1.0, 2.0, 2.0 + 2 ** -22, 5.0]
    assert lh.median(p, np.ones(4, bool), 1.0, 0.0, np.zeros(3), 0) == 2.0
    # -0.0 and +0.0 are one value to torch.nanmedian; the radix select ranks -0.0 first
    p[:, 2] = [-0.0, 0.0, 0.0, -0.0]
    m = lh.median(p, np.ones(4, bool), 1.0, 0.0, np.zeros(3), 0)
    assert m == 0 and np.signbit(m)


# ---------------------------------------------------------------------------------------------------------------------
def load_adv_golden(name):
    return dict(np.load(os.path.join(GOLDEN, f"loss_adv_{name}.npz")))


def close(a, b, rtol):
    """a within rtol (|b| + rms(b)) of b elementwise, NaN exactly where b is NaN, +-inf equal."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    fin = np.isfinite(b)
    if not np.array_equal(a[~fin & ~np.isnan(b)], b[~fin & ~np.isnan(b)]) or not np.isfinite(a[fin]).all():
        return False
    if not fin.any():
        return True
    rms = np.sqrt(np.mean(b[fin] ** 2))
    return bool(np.all(np.abs(a[fin] - b[fin]) <= rtol * (np.abs(b[fin]) + rms)))


def test_adversarial_goldens_are_small_and_cover_the_issues():
    for name in ADV:
        g = load_adv_golden(name)
        assert os.path.getsize(os.path.join(GOLDEN, f"loss_adv_{name}.npz")) < 1 << 20
        assert json.loads(str(g["case"])) == json.loads(json.dumps(synth.LOSS_ADV_CASES[name], sort_keys=True))
    assert str(load_adv_golden("empty_term")["raises"]) == "TypeError"   # torch.stack of a tensor and the int 0
    assert np.isnan(load_adv_golden("empty_b_ssi")["mon_vals"]).all()


@pytest.mark.parametrize("name", ADV)
def test_oracle_matches_adversarial_goldens(name):
    """fp32 PyTorch restatement vs the reference, full resolution.  Both are fp32 with the same per-pixel operations;
    they differ in the order of the norm factor's sums (<= n u relative for n pooled values, ~1e-6 here), which moves
    maps by that relative amount and the gradients of the worst-conditioned pixels by up to (|pr| + |gt|) / d times
    it: rtol 1e-5 (maps, scalars) and 1e-4 (gradients) of |ref| + rms(ref)."""
    case = synth.LOSS_ADV_CASES[name]
    g = load_adv_golden(name)
    gts, preds = synth.make_loss_adv_case(name)
    okw = oracle_kwargs(case["criterion"])
    dist_clip = case.get("kw", {}).get("dist_clip")
    out = lo.criterion(gts, preds, dtype=torch.float32, dist_clip=dist_clip, check_empty=False, **okw)
    F = len(gts)
    for i in range(F):
        assert close(out["gt_pts"][i], g[f"gt_{i}"], 1e-5), i
        assert np.array_equal(out["masks"][i].numpy(), g[f"mask_{i}"])
    for k in range(F - 1):
        assert close(out["pr_l"][k].detach(), g[f"pr_l_{k}"], 1e-5), k
        assert close(out["pr_r"][k].detach(), g[f"pr_r_{k}"], 1e-5), k
    for key in ("gt_factor", "pr_factor"):
        if g[key].size == 0:
            assert out[key] is None
        else:
            assert close(out[key].detach().flatten(), g[key], 1e-6)
    assert list(out["monitoring"]) == list(g["mon_keys"])
    assert close([float(v) for v in out["monitoring"].values()], g["mon_vals"], 1e-5)
    if case["call"] != "loss":
        return
    if str(g["raises"]):
        gts, preds = synth.make_loss_adv_case(name)
        with pytest.raises(ValueError, match="without a valid pixel"):
            lo.criterion(gts, preds, dtype=torch.float32, dist_clip=dist_clip, **okw)
        return
    gts, preds = synth.make_loss_adv_case(name)
    for p, c in slot_tensors(preds).values():
        p.requires_grad_(True)
        c.requires_grad_(True)
    out = lo.criterion(gts, preds, dtype=torch.float32, dist_clip=dist_clip, **okw)
    (out["loss"] + out["factor_loss"]).backward()
    assert close(float(out["loss"]), g["loss"], 1e-5) and close(float(out["factor_loss"]), g["factor_loss"], 1e-5)
    assert list(out["details"]) == list(g["detail_keys"])
    assert close(list(out["details"].values()), g["detail_vals"], 1e-5)
    for (side, k), (p, c) in slot_tensors(preds).items():
        assert close(p.grad, g[f"grad_pts_{side}_{k}"], 1e-4), (side, k)
        gc = c.grad if c.grad is not None else torch.zeros_like(c)
        assert close(gc, g[f"grad_conf_{side}_{k}"], 1e-4), (side, k)
