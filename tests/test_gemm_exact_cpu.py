"""The premise and the sensitivity of the bit-exact GEMM tests (test_gemm_exact_gpu.py), on the CPU.

Premise: for every case the GPU file runs, the generator's worst case -- the absolute products of an output plus its bias
and residuals -- stays within 2^22 quanta, so the kernel has exactly one correct fp32 answer.

Sensitivity: on a representative case of every case list, each defect model a split-bf16 kernel tends to have (a product
left out or added, a k-block dropped, the wrong tap, a shifted row, the lo plane truncated) changes at least one element
of every output tile it touches, so `torch.equal` on the GPU cannot pass a kernel with that defect.  Three of them are the
defects a relative-L2 bar of 3e-5 lets through on random normal data: a_hi * b_lo missing for one k-block of one tile,
A's lo plane of the last row read from the row above, and the output's lo plane truncated instead of rounded."""
import pytest
import torch

import gemm_exact as E

# ------------------------------------------------------------------------------------------------ premise
@pytest.mark.parametrize("geom", E.GEOMETRY)
def test_premise_geometry(geom):
    G, NB, H, W, Kc, taps, N = geom
    g = E.pick_gen(Kc * taps)
    assert g.bound(Kc * taps) + 3 * E.EPI_MAX <= E.BUDGET


@pytest.mark.parametrize("name,G,rows,K,N", E.SWEEP)
def test_premise_sweep(name, G, rows, K, N):
    g = E.pick_gen(K)
    assert g.bound(K) + 3 * E.EPI_MAX <= E.BUDGET
    assert g.s >= 4, g   # hi and lo still far apart at the longest contraction


@pytest.mark.parametrize("rows,Kc,N,bn", E.RING)
def test_premise_ring(rows, Kc, N, bn):
    assert E.pick_gen(Kc).bound(Kc) + 3 * E.EPI_MAX <= E.BUDGET


@pytest.mark.parametrize("shape", E.wgrad_cases())
def test_premise_wgrad(shape):
    nb, h, w, n, kc, taps = shape
    P = nb * h * w
    assert E.pick_gen(P, E.BUDGET).bound(P) <= E.BUDGET


def test_premise_small_outputs():
    """stats_out sums squares: with outputs |x| <= X quanta, 32 X^2 <= 2^22.  EPI_QKV rounds to tf32: |x| < 2^11."""
    assert 32 * (E.Gen(1, 0).bound(E.STATS_KC) + 3 * E.STATS_EPI) ** 2 <= E.BUDGET
    assert E.Gen(1, 1).bound(E.QKV_KC) + E.QKV_BIAS < 1 << 11


def test_planes_are_the_values():
    g = E.Gen(4, 8)
    hi, lo = E.planes((1000,), g, seed=1)
    assert torch.equal(hi.float() / 256, hi.float().div(256).round()) and hi.float().abs().max() <= 4 * 256
    assert torch.equal(lo.float(), lo.float().round()) and lo.float().abs().max() <= 4
    # outputs of ~2^20 quanta have more bits than hi + lo hold: the lo plane is rounded, and truncation shows
    x = E.ints((1000,), 1 << 20, 1.0, seed=2)
    h, l_ = E.split_ref(x)
    ht, lt = E.split_trunc(x)
    assert torch.equal(h, x.to(torch.bfloat16)) and torch.equal(h, ht)
    assert (l_ != lt).float().mean() > 0.2


# ------------------------------------------------------------------------------------------------ sensitivity
class Model:
    """Output of the exact kernel and of its defect models on one case (fp64, linear or 3x3)."""

    def __init__(self, a, b, G, taps, q, seed):
        """a planes [G*NB, H, W, Kc], b planes [G*N, taps*Kc]; bias and residual drawn as the GPU file draws them (up to
        2^19 quanta each), so that outputs are large enough for the lo plane to be rounded."""
        self.a, self.b, self.G, self.taps = a, b, G, taps
        self.shape = a[0].shape
        self.N = n = b[0].shape[0] // G
        NB, H, W = self.shape[0] // G, self.shape[1], self.shape[2]
        self.epi = (E.ints((G, 1, 1, 1, n), E.EPI_MAX, q, seed + 5) +
                    E.ints((G, NB, H, W, n), E.EPI_MAX, q, seed + 6)).double()
        self.exp = self.out(self.acc())

    def per_group(self, f, a=None):
        """f(a_g, b_g) -> [NB, H, W, N] over the groups -> [G, NB, H, W, N]."""
        a = self.a if a is None else a
        NB = self.shape[0] // self.G
        return torch.stack([f(tuple(t[g * NB:(g + 1) * NB].double() for t in a),
                              tuple(t[g * self.N:(g + 1) * self.N].double() for t in self.b)) for g in range(self.G)])

    def prod(self, x, y):
        return self.per_group(lambda a, b: E.conv_ref(a[x], b[y], self.taps))

    def acc(self, a=None):
        """The three products, on other A planes if given."""
        return self.per_group(lambda a_, b: E.conv_ref(a_[0], b[0] + b[1], self.taps) + E.conv_ref(a_[1], b[0], self.taps), a)

    def out(self, acc):
        return acc + self.epi

    def tiles(self):
        NB, H, W = self.shape[0] // self.G, self.shape[1], self.shape[2]
        return E.tile_ids(self.G * NB, H, W, self.N).view(self.G, NB, H, W, self.N)


def _assert_every_tile(model, got, region, what):
    """Every tile with an element in `region` has an element where `got` differs from the expected output."""
    tiles = model.tiles()
    diff = got != model.exp
    touched = torch.unique(tiles[region])
    hit = torch.unique(tiles[diff & region])
    missed = sorted(set(touched.tolist()) - set(hit.tolist()))
    assert not missed, f"{what}: {len(missed)} of {len(touched)} touched tiles unchanged, e.g. {missed[:8]}"


def _kblock(model, tap, c0, c1):
    """The three products' contribution of channels [c0, c1) of one tap."""
    kc = model.shape[-1]

    def f(a, b):
        wh, wl = (t.view(model.N, model.taps, kc).clone() for t in b)
        keep = torch.zeros_like(wh)
        keep[:, tap, c0:c1] = 1
        wh, wl = (wh * keep).view(model.N, -1), (wl * keep).view(model.N, -1)
        return E.conv_ref(a[0], wh + wl, model.taps) + E.conv_ref(a[1], wh, model.taps)
    return model.per_group(f)


def _reach(model, tap):
    """Outputs a tap can reach at all (3x3: not where its shift lands in the zero padding), over every column."""
    NB, H, W = model.shape[0] // model.G, model.shape[1], model.shape[2]
    w = torch.zeros(1, model.taps, 1, dtype=torch.float64)
    w[0, tap] = 1
    r = E.conv_ref(torch.ones(NB, H, W, 1, dtype=torch.float64), w.view(1, -1), model.taps) > 0
    return r.expand(NB, H, W, model.N).unsqueeze(0).expand(model.G, NB, H, W, model.N)


def _global_models(model):
    hh, hl, lh = model.prod(0, 0), model.prod(0, 1), model.prod(1, 0)
    ll = model.prod(1, 1)
    kc = model.shape[-1]
    kpt = (kc + 31) // 32
    last = model.taps - 1
    everywhere = torch.ones_like(model.exp, dtype=torch.bool)
    ms = {"hh only": (hh, everywhere), "hh + hl": (hh + hl, everywhere), "hh + lh": (hh + lh, everywhere),
          "+ lo lo": (hh + hl + lh + ll, everywhere)}
    acc = hh + hl + lh
    mid, tm = kpt // 2, model.taps // 2
    ms["first k-block dropped"] = (acc - _kblock(model, 0, 0, min(32, kc)), _reach(model, 0))
    ms["middle k-block dropped"] = (acc - _kblock(model, tm, 32 * mid, min(32 * mid + 32, kc)), _reach(model, tm))
    ms["last k-block dropped"] = (acc - _kblock(model, last, 32 * (kpt - 1), kc), _reach(model, last))
    if kc % 32:
        ms["ragged channel tail dropped"] = (acc - _kblock(model, tm, kc - kc % 32, kc), _reach(model, tm))
    return {k: (model.out(v), r) for k, (v, r) in ms.items()}


def _check_global(model):
    for what, (got, region) in _global_models(model).items():
        _assert_every_tile(model, got, region, what)


def _check_truncated_lo(model):
    hi, lo = E.split_ref(model.exp)
    ht, lt = E.split_trunc(model.exp)
    assert torch.equal(hi, ht)
    tiles = model.tiles()
    touched = torch.unique(tiles)
    hit = torch.unique(tiles[lo != lt])
    assert len(hit) == len(touched), ("lo truncated", len(hit), len(touched))


def _check_table_defects(model):
    """The three defects that pass a 3e-5 relative-L2 bar on random data, each in the tiles it touches."""
    G, NB, H, W, N = model.exp.shape
    acc = model.exp - model.epi
    kc = model.shape[-1]
    tiles = model.tiles()
    t0 = int(tiles[0, 0, 0, 0, 0])
    region = tiles == t0
    tm = model.taps // 2
    hl_kb = model.per_group(lambda a, b: E.conv_ref(a[0], _mask_kblock(b[1], model.taps, kc, tm, 0, min(32, kc)), model.taps))
    _assert_every_tile(model, model.out(acc - torch.where(region, hl_kb, 0)), region, "a_hi b_lo missing, one k-block of one tile")
    hl = model.prod(0, 1)
    _assert_every_tile(model, model.out(acc - torch.where(region, hl, 0)), region, "a_hi b_lo missing over K in one tile")
    if H == 1:   # linear: the last row's lo plane read from the row above
        al = model.a[1].clone()
        al[:, :, -1] = al[:, :, -2]
        row = torch.zeros_like(region)
        row[:, :, :, -1] = True
        got = model.out(model.acc((model.a[0], al)))
        _assert_every_tile(model, got, row, "A lo of the last row from the row above")
        # a row shifted in the ragged last tile: every row of that tile reads the A row above it
        first = (W - 1) // 128 * 128
        if first > 0 and W % 128:
            a2 = tuple(t.clone() for t in model.a)
            for t, s in zip(a2, model.a):
                t[:, :, first:] = s[:, :, first - 1:W - 1]
            rows = torch.zeros_like(region)
            rows[:, :, :, first:] = True
            _assert_every_tile(model, model.out(model.acc(a2)), rows, "row shifted in the ragged last tile")


def _mask_kblock(w, taps, kc, tap, c0, c1):
    m = torch.zeros(taps, kc, dtype=w.dtype)
    m[tap, c0:c1] = 1
    return (w.view(w.shape[0], taps, kc) * m).view(w.shape[0], -1)


def _linear_model(G, rows, Kc, N, seed):
    g = E.pick_gen(Kc)
    a = E.planes((G, 1, rows, Kc), g, seed)
    b = E.planes((G * N, Kc), g, seed + 1)
    return Model(a, b, G, 1, g.q, seed)


@pytest.mark.parametrize("G,rows,Kc,N", [(1, 333, 200, 160), (2, 77, 40, 96)])
def test_defects_change_every_tile_linear(G, rows, Kc, N):
    """The geometry list: ragged M, a channel tail (200 = 6 x 32 + 8), partial column tiles, two groups."""
    model = _linear_model(G, rows, Kc, N, seed=10)
    _check_global(model)
    _check_truncated_lo(model)
    _check_table_defects(model)


def test_defects_change_every_tile_sweep():
    """dec.proj of the sweep: groups 2, 768 rows, K = N = 768."""
    model = _linear_model(2, 768, 768, 768, seed=20)
    _check_global(model)
    _check_truncated_lo(model)
    _check_table_defects(model)


def test_defects_change_every_tile_ring():
    """The ragged ring-wrap launch: 7700 rows (60 tiles + 20 rows), 160 channels, N = 1056."""
    model = _linear_model(1, 7700, 160, 1056, seed=30)
    _check_global(model)
    _check_table_defects(model)


@pytest.mark.parametrize("NB,H,W,Kc,N", [(2, 13, 19, 40, 96), (3, 7, 7, 24, 32)])
def test_defects_change_every_tile_conv3x3(NB, H, W, Kc, N):
    g = E.pick_gen(9 * Kc)
    a = E.planes((NB, H, W, Kc), g, seed=40)
    b = E.planes((N, 9 * Kc), g, seed=41)
    model = Model(a, b, 1, 9, g.q, seed=40)
    _check_global(model)
    _check_truncated_lo(model)
    _check_table_defects(model)
    # the wrong tap: tap 4's weights applied at the shift of tap 5 (and tap 0's at tap 1)
    everywhere = torch.ones_like(model.exp, dtype=torch.bool)
    for t, u in ((4, 5), (0, 1)):
        def moved(a_, b_, t=t, u=u):   # tap t's weights against the A box of tap u's shift
            wh, wl = (torch.zeros(N, 9, Kc, dtype=torch.float64) for _ in range(2))
            wh[:, u], wl[:, u] = b_[0].view(N, 9, Kc)[:, t], b_[1].view(N, 9, Kc)[:, t]
            wh, wl = wh.view(N, -1), wl.view(N, -1)
            return E.conv_ref(a_[0], wh + wl, 9) + E.conv_ref(a_[1], wh, 9)
        got = model.out(model.acc() - _kblock(model, t, 0, Kc) + model.per_group(moved))
        _assert_every_tile(model, got, everywhere, f"tap {t} read at the shift of tap {u}")


@pytest.mark.parametrize("shape", [(2, 37, 53, 128, 96, 9), (3, 19, 23, 192, 256, 1), (1, 7, 7, 256, 768, 9)])
def test_defects_change_every_tile_wgrad(shape):
    """s3r_conv_wgrad's defect models: products, a 64-pixel k-block (first, middle, the ragged last), the wrong tap.
    Tiles: 128 dY channels x 128 X channels of one tap."""
    nb, h, w, n, kc, taps = shape
    g = E.pick_gen(nb * h * w, E.BUDGET)
    dy = E.planes((nb, h, w, n), g, seed=50)
    x = E.planes((nb, h, w, kc), g, seed=51)
    exp = E.wgrad_ref(dy, x, taps)
    tiles = (torch.arange(n)[:, None, None] // 128 * 1000 + torch.arange(taps)[None, :, None] * 10 +
             torch.arange(kc)[None, None, :] // 128)
    touched = set(torch.unique(tiles).tolist())

    def check(got, what, region=None):
        want = touched if region is None else set(torch.unique(tiles[region.expand_as(tiles)]).tolist())
        hit = set(torch.unique(tiles[got != exp]).tolist())
        assert want <= hit, (what, len(want - hit))

    def masked(px):   # the reference over the pixels where px is True only, and the (tap) outputs those pixels reach
        m = px.view(nb, h, w, 1).to(torch.bfloat16)
        one = torch.ones(nb, h, w, 1, dtype=torch.bfloat16)
        reach = E.wgrad_ref((one * m, one * 0), (one, one * 0), taps) > 0
        return E.wgrad_ref(tuple(t * m for t in dy), x, taps), reach

    yh, yl = dy
    xh, xl = x
    hh = E.wgrad_ref((yh, torch.zeros_like(yl)), (xh, torch.zeros_like(xl)), taps)
    check(hh, "hh only")
    check(E.wgrad_ref((yh, torch.zeros_like(yl)), x, taps), "hh + hl")
    check(hh + E.wgrad_ref((torch.zeros_like(yh), yl), (xh, torch.zeros_like(xl)), taps), "hh + lh")
    ll = E.wgrad_ref((yl, torch.zeros_like(yl)), (torch.zeros_like(xh), xl), taps)
    check(exp + ll, "+ lo lo")
    box = E.row_tiles(nb, h, w, pix=64)
    nbox = int(box.max()) + 1
    for kb, what in ((0, "first"), (nbox // 2, "middle"), (nbox - 1, "last")):
        part, reach = masked(box == kb)
        check(exp - part, f"{what} 64-pixel k-block dropped", reach)
    if taps == 9:
        # tap 4 (no shift) computed with the shift of tap 5
        xs = tuple(torch.cat((t[:, :, 1:], torch.zeros_like(t[:, :, :1])), 2) for t in x)
        wrong = exp.clone()
        wrong[:, 4] = E.wgrad_ref(dy, xs, 1)[:, 0]
        hit = set(torch.unique(tiles[:, 4][wrong[:, 4] != exp[:, 4]]).tolist())
        assert hit == set(torch.unique(tiles[:, 4]).tolist()), "tap 4 read at the shift of tap 5"
