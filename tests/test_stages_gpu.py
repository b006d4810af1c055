"""Every engine stage against the fp64 oracle, at each image geometry the engine serves.

The reference is oracle.spann3r_oracle run in float64 on the GPU (state dict and images in double).  Each stage is
isolated the way test_model_gpu.py::test_stagewise_vs_oracle does it: its input is the fp64 oracle's input of that stage
rounded to fp32, and the same rounded values (in double) feed the reference.  `keyheads` and `heads` read the engine's
own last decode (the key-head input and the DPT hooks are written by `decode`), so their bars include the decoder's error.

Geometries: 224 x 224 at B = 1 and B = 2, 384 x 512, the portrait 512 x 384 (value encoder reads the transposed map), 336 x
512 (odd patch rows: refinenet4's output is cropped), 512 x 336 (odd patch columns, portrait), 208 x 240 (13 x 15 = 195
tokens: V^T is padded to 196, both crop dimensions odd) on the sharpened checkpoint, and the raw one at 224 x 224 and 384 x
512.  Encode takes 2 B + 1 images (an odd count).

The two raw-checkpoint geometries duplicate the sharpened ones at the same size: the checkpoints differ only in
norm_q.weight (`test_raw_and_sharpened_checkpoints_differ_only_in_norm_q`), which only the memory read uses, so every stage
here computes the same bits on both.  They are kept so that the raw checkpoint's stages stay covered if that changes.

Two errors per tensor:
  global  relative L2;
  local   token tensors: the worst row's L2 error over the RMS row norm; maps: the worst pixel's error (over its
          channels) over the RMS pixel norm, the border rows and columns reported apart ("border") from the interior.
Each bar is about 3x the worst error measured over the geometries on H100 80GB HBM3 cards at 400 W and at 700 W power
limits (every error was the same on both); the measured values are in the comments.  Global bars never exceed the 224 x 224 bars of test_stagewise_vs_oracle (2e-4,
heads 3e-4).

Bitwise: two heads() calls give the same bits, and heads() with per-launch profiling on (one stream) the same bits as
with it off (pyramid levels 2-4 on side streams).
"""
import pytest
import torch

from conftest import get_state_dict, rel_l2

# (global, local, border) per stage; worst measured over all geometries in the comment (global / local / border)
BARS = {
    "encode": (2e-4, 2.7e-4, None),        # 8.3e-5 / 8.9e-5 (224 x 224; 4.6-4.8e-5 at 672-768 tokens); global at the ceiling
    "decode": (9e-5, 1e-4, None),          # 3.0e-5 / 3.2e-5 (224 x 224, B = 2)
    "keyheads": (7.5e-5, 8e-5, None),      # 2.5e-5 / 2.6e-5 (208 x 240)
    "pts3d": (1.4e-4, 2.6e-4, 1.9e-4),     # 4.6e-5 / 8.6e-5 / 6.2e-5
    "conf": (2.3e-6, 5.2e-6, 3e-6),        # 7.5e-7 / 1.7e-6 / 1.0e-6
    "value": (7e-5, 7.2e-5, None),         # 2.3e-5 / 2.4e-5 (208 x 240, RoPE)
    "value_usefeat": (4.2e-5, 4.5e-5, None),   # 1.4e-5 / 1.5e-5 (208 x 240, RoPE)
}

GEOMS = [
    # id, sharpened checkpoint, B, H, W
    ("224", True, 1, 224, 224),
    ("224_b2", True, 2, 224, 224),
    ("384x512", True, 1, 384, 512),
    ("512x384", True, 1, 512, 384),
    ("336x512", True, 1, 336, 512),
    ("512x336", True, 1, 512, 336),
    ("208x240", True, 1, 208, 240),
    ("224_raw", False, 1, 224, 224),          # same stage bits as "224" (see the module docstring)
    ("384x512_raw", False, 1, 384, 512),      # same stage bits as "384x512"
]
USEFEAT_GEOMS = ("208x240", "512x336")


# ------------------------------------------------------------------------------------------------
# error measures (pure; checked on the CPU at the end of the file)
# ------------------------------------------------------------------------------------------------
def row_err(a: torch.Tensor, b: torch.Tensor) -> float:
    """[..., C] tensors: max over rows of |a_r - b_r| / RMS_r |b_r| (L2 over the last axis)."""
    a, b = a.double().reshape(-1, a.shape[-1]), b.double().reshape(-1, b.shape[-1])
    return float((a - b).norm(dim=-1).max() / b.norm(dim=-1).pow(2).mean().sqrt().clamp_min(1e-300))


def map_err(a: torch.Tensor, b: torch.Tensor):
    """[B, H, W] or [B, H, W, C] maps: (worst interior pixel, worst border pixel) error over the RMS pixel norm."""
    a, b = a.double(), b.double()
    if a.dim() == 3:
        a, b = a[..., None], b[..., None]
    e = (a - b).norm(dim=-1)
    rms = float(b.norm(dim=-1).pow(2).mean().sqrt().clamp_min(1e-300))
    border = torch.zeros_like(e, dtype=torch.bool)
    border[:, 0], border[:, -1], border[:, :, 0], border[:, :, -1] = True, True, True, True
    inner = e[~border]
    return (float(inner.max()) if inner.numel() else 0.0) / rms, float(e[border].max()) / rms


def check(geom, stage, name, got, ref, kind="tokens", bars=None):
    g, lb, bb = bars or BARS[stage]
    glob = rel_l2(got, ref)
    if kind == "tokens":
        loc, bor = row_err(got, ref), None
    else:
        loc, bor = map_err(got, ref)
    print(f"STAGE {geom:12s} {stage:14s} {name:18s} global {glob:.2e} local {loc:.2e}" +
          (f" border {bor:.2e}" if bor is not None else ""))
    assert bool(torch.isfinite(got).all()), (geom, stage, name)
    assert glob < g, (geom, stage, name, "global", glob, g)
    assert loc < lb, (geom, stage, name, "local", loc, lb)
    if bor is not None:
        assert bor < bb, (geom, stage, name, "border", bor, bb)


# ------------------------------------------------------------------------------------------------
# fixtures: one geometry at a time (module-scoped parametrized fixture: pytest groups the tests by geometry)
# ------------------------------------------------------------------------------------------------
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from spann3r_b200 import _lib
    _lib.require_device()


_MODELS = {}   # (sharpen, use_feat) -> (model, fp64 state dict on the GPU); emptied when the module ends


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    """The models and fp64 state dicts take several GB of device memory: give it back to later test modules."""
    yield
    _MODELS.clear()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _model(sharpen, use_feat=False):
    from spann3r_b200 import Spann3R, synth
    key = (sharpen, use_feat)
    if key not in _MODELS:
        m = Spann3R(dus3r_name=None, use_feat=use_feat)
        sd = synth.make_state_dict(synth.usefeat_spec(), seed=0, sharpen=sharpen) if use_feat else get_state_dict(sharpen)
        m.load_state_dict(sd, strict=True)
        sd64 = {k: v.double().cuda() for k, v in sd.items()}
        _MODELS[key] = (m.cuda().eval(), sd64)
    return _MODELS[key]


class Case:
    """One geometry: a test-owned engine (2 B + 1 images) and the fp64 oracle's stage inputs / outputs."""

    def __init__(self, gid, sharpen, B, H, W):
        from oracle import spann3r_oracle as orc
        from spann3r_b200 import synth
        from spann3r_b200.engine import Engine
        self.gid, self.B, self.H, self.W = gid, B, H, W
        self.model, sd = _model(sharpen)
        self.sd = sd
        nimg = 2 * B + 1
        self.eng = Engine(self.model._weights(), B, H, W, max_images=nimg)
        frames = synth.make_frames(nimg, H, W, seed0=7)
        self.img = torch.cat([f["img"] for f in frames]).cuda().contiguous()
        with torch.no_grad():
            feats, pos = orc.encode_image(sd, self.img.double())
            self.ref_feats = feats
            self.pos = pos
            # decoder input: the fp64 encoder output rounded to fp32
            self.f1, self.f2 = feats[:B].float().contiguous(), feats[B:2 * B].float().contiguous()
            self.p1, self.p2 = pos[:B], pos[B:2 * B]
            self.rdec1, self.rdec2 = orc.decoder(sd, self.f1.double(), self.p1, self.f2.double(), self.p2)
            self.rk1 = orc.key_head(sd, 1, self.f1.double(), self.rdec1[-1])
            self.rk2 = orc.key_head(sd, 2, self.f2.double(), self.rdec2[-1])
            self.r1 = orc.dpt_head(sd, "dust3r.downstream_head1", self.rdec1, H, W)
            self.r2 = orc.dpt_head(sd, "dust3r.downstream_head2", self.rdec2, H, W)

    def decode(self):
        return self.eng.decode(self.f1, self.f2, want_all=True)


@pytest.fixture(scope="module", params=GEOMS, ids=[g[0] for g in GEOMS])
def case(request):
    _need_gpu()
    c = Case(*request.param)
    yield c
    del c.eng
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------
# stages
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_encode(case):
    feats = case.eng.encode(case.img)
    for i in range(feats.shape[0]):
        check(case.gid, "encode", f"img{i}", feats[i], case.ref_feats[i])


@pytest.mark.gpu
def test_decode(case):
    dec = case.decode()
    for l in range(12):
        for s, rdec in ((0, case.rdec1), (1, case.rdec2)):
            for b in range(case.B):
                check(case.gid, "decode", f"l{l}s{s}b{b}", dec[l, s, b], rdec[l + 1][b])


@pytest.mark.gpu
def test_keyheads(case):
    case.decode()
    k1, k2 = case.eng.keyheads(case.f1, case.f2)
    for b in range(case.B):
        check(case.gid, "keyheads", f"head1b{b}", k1[b], case.rk1[b])
        check(case.gid, "keyheads", f"head2b{b}", k2[b], case.rk2[b])


@pytest.mark.gpu
def test_heads(case):
    """pts3d and conf of both heads in the head's own (H, W) layout; bitwise: repeated, and profiled (one stream)."""
    case.decode()
    pts, conf = case.eng.heads()
    for h, r in ((0, case.r1), (1, case.r2)):
        for b in range(case.B):
            check(case.gid, "pts3d", f"head{h + 1}b{b}", pts[h, b:b + 1], r["pts3d"][b:b + 1], kind="map")
            check(case.gid, "conf", f"head{h + 1}b{b}", conf[h, b:b + 1], r["conf"][b:b + 1], kind="map")
    pts_b, conf_b = case.eng.heads()
    assert torch.equal(pts, pts_b) and torch.equal(conf, conf_b), "two heads() calls differ"
    case.eng.profile(True)
    try:
        pts_p, conf_p = case.eng.heads()
        case.eng.profile_read()
    finally:
        case.eng.profile(False)
    assert torch.equal(pts, pts_p) and torch.equal(conf, conf_p), "heads() on one stream differs from the side streams"


@pytest.mark.gpu
@pytest.mark.parametrize("rope", [False, True], ids=["norope", "rope"])
def test_value(case, rope):
    """Default value encoder on head 1's fp64 pointmap rounded to fp32 (portrait frames: read transposed, as the
    landscape view the reference's head wrapper hands it), + feat_k1."""
    from oracle import spann3r_oracle as orc
    portrait = case.H > case.W
    pts = case.r1["pts3d"].float().contiguous()                 # [B, H, W, 3], the head's own layout
    k1 = case.rk1.float().contiguous()
    got = case.eng.value(pts, k1, transposed=portrait, rope=rope)
    land = pts.double().swapaxes(1, 2) if portrait else pts.double()
    with torch.no_grad():
        ref = orc.encode_cur_value(case.sd, land, mem_pos_enc=rope) + k1.double()
    for b in range(case.B):
        check(case.gid, "value", f"{'rope' if rope else 'norope'}b{b}", got[b], ref[b])


@pytest.mark.gpu
@pytest.mark.parametrize("rope", [False, True], ids=["norope", "rope"])
def test_value_usefeat(case, rope):
    """use_feat value encoder (tokens=True) on the fp64 decoder's dec1[-1] rounded to fp32, + feat_k1."""
    if case.gid not in USEFEAT_GEOMS:
        pytest.skip("use_feat value stage runs at " + ", ".join(USEFEAT_GEOMS))
    from oracle import usefeat_oracle as ufo
    from spann3r_b200.engine import Engine
    m, sdu = _model(True, use_feat=True)
    eng = Engine(m._weights(), case.B, case.H, case.W)
    assert all(torch.equal(sdu[k], case.sd[k]) for k in case.sd if k.startswith("dust3r."))
    tok = case.rdec1[-1].float().contiguous()
    k1 = case.rk1.float().contiguous()
    got = eng.value(tok, k1, rope=rope, tokens=True)
    with torch.no_grad():
        ref = ufo.encode_cur_value(sdu, tok.double(), case.p1, mem_pos_enc=rope) + k1.double()
    del eng
    for b in range(case.B):
        check(case.gid, "value_usefeat", f"{'rope' if rope else 'norope'}b{b}", got[b], ref[b])


# ------------------------------------------------------------------------------------------------
# CPU: the error measures
# ------------------------------------------------------------------------------------------------
def test_row_err_finds_one_bad_row():
    g = torch.Generator().manual_seed(0)
    b = torch.randn(2, 300, 64, generator=g, dtype=torch.float64)
    a = b.clone()
    a[1, 123] += 0.01 * b[1, 123].norm() * torch.randn(64, generator=g, dtype=torch.float64) / 8
    rms = float(b.norm(dim=-1).pow(2).mean().sqrt())
    assert abs(row_err(a, b) - float((a - b)[1, 123].norm()) / rms) < 1e-12
    assert rel_l2(a, b) < row_err(a, b) / 10          # the global measure dilutes it by ~sqrt(rows)
    assert row_err(b, b) == 0.0


def test_map_err_splits_border_from_interior():
    b = torch.ones(1, 9, 12, 3, dtype=torch.float64)
    a = b.clone()
    a[0, 8, 5, 1] += 0.5            # last row: border
    a[0, 4, 6, 0] += 0.1            # interior
    inner, border = map_err(a, b)
    rms = 3 ** 0.5
    assert abs(inner - 0.1 / rms) < 1e-12 and abs(border - 0.5 / rms) < 1e-12
    c = torch.ones(2, 5, 7, dtype=torch.float64)
    d = c.clone()
    d[1, 2, 0] = 1.25               # first column: border
    assert map_err(d, c) == (0.0, 0.25)


def test_raw_and_sharpened_checkpoints_differ_only_in_norm_q():
    """Why the raw geometries give the same stage bits as the sharpened ones (module docstring)."""
    raw, sharp = get_state_dict(False), get_state_dict(True)
    assert raw.keys() == sharp.keys()
    assert [k for k in raw if not torch.equal(raw[k], sharp[k])] == ["norm_q.weight"]
