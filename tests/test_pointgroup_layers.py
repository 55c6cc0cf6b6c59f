"""PointGroup's U-Net on the device layer by layer (catgrasp_b200/pointgroup.py, cg_spconv.cu) against the layer plan of
oracle/pointgroup_ref.py, and the offset head and the conv kernel on their own at their tile edges.

The forward's end-to-end checks (test_pointgroup_kernels.py) see the final offsets only, after ~60 layers in series.
Here every convolution of a forward is captured (PointGroupNet._conv and .head wrapped, their outputs filled with NaN
before the call) and
  - matched to exactly one plan record by its weights, bit for bit;
  - checked for wiring exactly: its input and residual are bit-equal to the outputs the plan names (the encoder half
    first in a concatenation), its table to the oracle's table of its level, its count word to the level's count,
    its BN (scale, shift) and bias to the float32 of the state dict's float64 values;
  - held within 2x the one-layer bound of ``pointgroup_ref.layer`` on the device's own inputs;
  - checked to leave its padding rows (at or past the count) NaN;
and the poisoned forward's offsets are bit-equal to an unpoisoned one's, so no layer reads a padding row.

Seeded mutations, each caught (first failing test shown, then whether test_pointgroup_kernels.py and
test_spconv_kernels.py, which held the forward to 1e-3 of its largest offset, catch it too):
  - BN eps 1e-5 -> 1e-4 in weights._bn_affine              test_layers_golden[hnm] (BN of the first conv)  missed
  - level 5's conv.0 and deconv.0 BN swapped in packing     test_layers_golden[hnm] (BN of unet.u.u.u.u.conv.2)  missed
  - the second tail block's residual taken from the first
    tail block's input (its encoder half, the same shape)   test_layers_golden[hnm] (residual)  test_forward_golden
  - the conv kernel's store guard r >= n made r >= M        test_layers_golden[hnm] (a padding row written)  missed
  - offset_head_kernel reading W1 transposed                test_layers_golden[hnm] (head bound)  test_forward_golden
  - gather3_kernel giving site 0 to a point with no site    test_head_count_word[16]  missed
"""
import json
import os
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from catgrasp_b200 import pointgroup, spconv, synthetic, weights   # noqa: E402
from oracle import pointgroup_ref as PR                               # noqa: E402
from oracle import spconv_ref as S                                    # noqa: E402
from oracle.encoder_ref import bound_ratio                            # noqa: E402

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "pointgroup.npz"))
KEY_SHAPES = [(k, tuple(s)) for k, s in json.loads(str(G["key_shapes"]))]
M16, REPS16 = int(G["m"]), int(G["block_reps"])
TILE = 64            # the conv kernel's output rows per CTA
NAN = float("nan")


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _eq(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


class Capture:
    """PointGroupNet._conv and .head as the product makes them, with NaN-filled outputs, recording every call."""

    def __init__(self, monkeypatch):
        self.convs, self.heads = [], []
        cap = self

        def conv(net, x, nbr, W, n, rows, bn=None, bias=None, residual=None):
            K, Cin, Cout = W.shape
            out = torch.full((rows, Cout), NAN, dtype=torch.float32, device=net.device)
            scale, shift = (None, None) if bn is None else bn
            net.ctx.call("cg_spconv_conv_dev", net.ctx.h, x, Cin, nbr, K, n, rows, W, Cout, scale, shift, bias,
                         residual, out)
            cap.convs.append(dict(x=x, table=nbr, W=W, n=n, rows=rows, bn=bn, bias=bias, res=residual, out=out))
            return out

        def head(net, level, x, p2v):
            h = net.w["head"]
            N = p2v.shape[0]
            site = torch.full((level.rows, 3), NAN, dtype=torch.float32, device=net.device)
            out = torch.full((N, 3), NAN, dtype=torch.float32, device=net.device)
            net.ctx.call("cg_pointgroup_head_dev", net.ctx.h, x, net.m, level.n, level.rows, h["bn"][0], h["bn"][1],
                         h["W1"], h["b1"], h["W2"], h["b2"], p2v, N, site, out)
            cap.heads.append(dict(x=x, n=level.n, p2v=p2v, site=site, out=out))
            return out

        monkeypatch.setattr(pointgroup.PointGroupNet, "_conv", conv)
        monkeypatch.setattr(pointgroup.PointGroupNet, "head", head)


def _bn32(sd, p):
    """float32 of the float64 BN affine, as the plan defines it."""
    g, b, mu, var = (np.asarray(sd[p + s], np.float64) for s in (".weight", ".bias", ".running_mean", ".running_var"))
    s = g / np.sqrt(var + PR.BN_EPS)
    return s.astype(np.float32), (b - mu * s).astype(np.float32)


def _sample(count, seed, n=2048):
    """The first and last two 64-row tiles of a level's count and a seeded sample of its rows."""
    last = max(0, (count - 1) // TILE * TILE - TILE)
    rng = np.random.RandomState(seed)
    return np.unique(np.concatenate([np.arange(min(TILE, count)), np.arange(last, count), rng.randint(0, count, n)]))


def _scene(sd, m, reps, locs, shape, feats, monkeypatch, expect_dropped=(), sampled=False):
    """One forward through the patched net, every layer checked (module docstring), on every live row or, ``sampled``,
    on ``_sample``'s rows of each level.  Returns the levels' counts."""
    net = pointgroup.PointGroupNet(sd, m, reps, device=0)
    locs = np.asarray(locs, dtype=np.int64)
    feats = np.ascontiguousarray(feats, dtype=np.float32)
    level, p2v = spconv.index(torch.from_numpy(locs.astype(np.int32)).cuda(), tuple(int(s) for s in shape))
    f = torch.from_numpy(feats).cuda()
    want = net.offsets(level, p2v, f).cpu().numpy()

    dev_levels = pointgroup.pyramid(level)
    cap = Capture(monkeypatch)
    got = net.offsets(level, p2v, f, levels=dev_levels).cpu().numpy()
    monkeypatch.undo()
    assert np.isfinite(got).all() and _eq(got, want)   # padding rows poisoned with NaN reach no offset

    # the levels: device sites and tables against levels_of
    order_sites = np.unique(S.pack(locs))
    ref_levels = PR.levels_of(S.unpack(order_sites).astype(np.int64), tuple(int(s) for s in shape))
    counts, rows = [], []
    for (lv, dn, up), (rvox, rnbr, rdn, rup) in zip(dev_levels, ref_levels):
        n = lv.count()
        assert n == len(rvox) and np.array_equal(_np(lv.vox)[:n], rvox)
        counts.append(n)
        rows.append(lv.rows)
    for i in expect_dropped:
        assert (ref_levels[i][3] < 0).all(1).any(), f"level {i} drops no child"

    # the voxel features, in key order, as the oracle forms them
    locs4 = np.concatenate([np.zeros((len(locs), 1), np.int64), locs], 1)
    vl, _, v2p = PR.voxelization_idx(locs4)
    vfeats = PR.voxelization(feats, v2p)[np.argsort(S.pack(vl[:, 1:]), kind="stable")]

    recs = PR.plan(m, reps)
    by_w = {}
    for r in recs:
        w32 = np.asarray(sd[r.name + ".weight"], np.float64).astype(np.float32).reshape(r.K, r.cin, r.cout)
        by_w.setdefault(w32.tobytes(), []).append(r)
    level_of = {PR.VFEATS: 0, **{r.name: r.level for r in recs}}
    outs = {PR.VFEATS: vfeats}
    seen = set()
    assert len(cap.convs) == len(recs)
    for call in cap.convs:
        W = _np(call["W"])
        match = by_w.get(W.tobytes(), [])
        assert len(match) == 1, f"weights {W.shape} match {len(match)} plan records"
        rec = match[0]
        assert rec.name not in seen and W.shape == (rec.K, rec.cin, rec.cout)
        seen.add(rec.name)
        L, n = rec.level, counts[rec.level]
        # wiring, bit for bit
        assert int(call["n"].item()) == n and call["rows"] == rows[L], rec.name
        tab = _np(call["table"])
        ref_tab = PR.table(rec, ref_levels)
        if ref_tab is None:
            assert tab is None, rec.name
        else:
            assert tab.shape == (rows[L], rec.K) and np.array_equal(tab[:n], ref_tab), rec.name
            assert (tab[n:] == -1).all(), rec.name
        nin = counts[level_of[rec.src[0]]]
        x = _np(call["x"])
        assert x.shape == (rows[level_of[rec.src[0]]], rec.cin), rec.name
        x = x[:nin]
        assert _eq(x, np.concatenate([outs[s][:nin] for s in rec.src], 1)), f"{rec.name}: input"
        res = _np(call["res"])
        if rec.res is None:
            assert res is None, rec.name
        else:
            res = res[:n]
            assert _eq(res, np.concatenate([outs[s][:n] for s in rec.res], 1)), f"{rec.name}: residual"
        if rec.bn is None:
            assert call["bn"] is None, rec.name
        else:
            s, t = _bn32(sd, rec.bn)
            assert _eq(_np(call["bn"][0]), s) and _eq(_np(call["bn"][1]), t), f"{rec.name}: BN {rec.bn}"
        assert _eq(_np(call["bias"]), np.asarray(sd[rec.name + ".bias"], np.float32)), f"{rec.name}: bias"
        # the output: padding untouched, live rows within 2x the one-layer bound
        out = _np(call["out"])
        assert np.isnan(out[n:]).all(), f"{rec.name}: a padding row was written"
        sample = _sample(n, zlib.crc32(rec.name.encode())) if sampled else None
        y, ey = PR.layer(sd, rec, x, res, ref_levels, rows=sample)
        live = out[:n] if sample is None else out[sample]
        ratio = bound_ratio(live, y, ey).max()
        print(f"  {rec.name:60s} {rec.kind:5s} L{L} K{rec.K:2d} {rec.cin:4d}->{rec.cout:4d} "
              f"rows {len(live):6d}  worst/2x bound {ratio:.3e}")
        assert ratio <= 1.0, rec.name
        outs[rec.name] = out
    assert seen == {r.name for r in recs}

    # the head on the device's own level-1 features; the gather bit for bit
    (hd,) = cap.heads
    n0 = counts[0]
    xh = _np(hd["x"])
    assert _eq(xh[:n0], outs[recs[-1].name][:n0])
    site = _np(hd["site"])
    assert np.isnan(site[n0:]).all()
    y, ey = PR.head(sd, xh[:n0].astype(np.float64), 0.0)
    ratio = bound_ratio(site[:n0], y, ey).max()
    print(f"  {'head':60s} rows {n0:6d}  worst/2x bound {ratio:.3e}")
    assert ratio <= 1.0
    assert _eq(_np(hd["out"]), site[_np(hd["p2v"])])
    return counts


@pytest.fixture(scope="module")
def sd16():
    return PR.synthetic_state_dict(KEY_SHAPES, int(G["seed"]))


def _pile(n_points, n_objects, seed):
    sc = synthetic.make_pile(n_points, n_objects=n_objects, seed=seed)
    _, locs, feats, shape = PR.host_front(sc["cloud_xyz"], sc["cloud_normal"])
    return locs, shape, feats


@pytest.mark.parametrize("cls", ("hnm", "nut", "screw"))
def test_layers_golden(cls, sd16, monkeypatch):
    feats = PR.host_front(G[f"{cls}_cloud_xyz"], G[f"{cls}_cloud_normal"])[2]
    _scene(sd16, M16, REPS16, G[f"{cls}_locs"], G[f"{cls}_spatial_shape"], feats, monkeypatch)


def test_layers_m32(monkeypatch):
    sd = PR.synthetic_state_dict(list(weights.pointgroup_keys(32, 2).items()), 5)
    _scene(sd, 32, 2, *_pile(6000, 4, 14), monkeypatch)


def test_layers_m12_block_reps_1(monkeypatch):
    # every layer's Cout (12 ... 84) leaves a partial 16-column tile
    sd = PR.synthetic_state_dict(list(weights.pointgroup_keys(12, 1).items()), 7)
    _scene(sd, 12, 1, *_pile(4000, 3, 16), monkeypatch)


def test_layers_one_site(sd16, monkeypatch):
    rng = np.random.RandomState(17)
    locs = np.tile([[37, 90, 5]], (3, 1))
    feats = rng.randn(3, PR.INPUT_C).astype(np.float32)
    counts = _scene(sd16, M16, REPS16, locs, (128, 128, 128), feats, monkeypatch)
    assert counts == [1] * PR.LEVELS


def test_layers_odd_shape(sd16, monkeypatch):
    # 135 -> 67 -> 33 -> 16: the last plane of each of the first three levels has no parent, so those children's
    # up-conv rows are the bias alone
    rng = np.random.RandomState(18)
    locs = rng.randint(100, 135, (6000, 3))
    locs[:300, 0] = 134
    locs[300:600, 1] = 134
    locs[600:900, 2] = 134
    nrm = rng.randn(len(locs), 3)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    feats = np.concatenate([nrm, locs / 500.0], 1).astype(np.float32)
    _scene(sd16, M16, REPS16, locs, (135, 135, 135), feats, monkeypatch, expect_dropped=(0, 1, 2))


def test_layers_pile_120k(sd16, monkeypatch):
    # the largest pile of test_pointgroup_kernels.test_forward_pile; above ~20k points, a sample of rows
    counts = _scene(sd16, M16, REPS16, *_pile(120000, 60, 13), monkeypatch, sampled=True)
    assert counts[0] > 4 * TILE


# ---------------------------------------------------------------- the offset head on its own
def _head_sd(m, seed):
    keys = [("output_layer.0" + s, (m,)) for s in (".weight", ".bias", ".running_mean", ".running_var")]
    keys += [("offset.0.weight", (m, m)), ("offset.0.bias", (m,))]
    keys += [("offset.1" + s, (m,)) for s in (".weight", ".bias", ".running_mean", ".running_var")]
    keys += [("offset.3.weight", (3, m)), ("offset.3.bias", (3,))]
    return PR.synthetic_state_dict(keys, seed, offset_scale=1.0)


def _head_weights(sd):
    """float32 (s0, t0, W1 [in][out], b1, W2 [in][out], b2), offset.1 folded into offset.0 in float64."""
    s0, t0 = _bn32(sd, "output_layer.0")
    g, b, mu, var = (np.asarray(sd["offset.1" + s], np.float64) for s in (".weight", ".bias", ".running_mean",
                                                                            ".running_var"))
    s = g / np.sqrt(var + PR.BN_EPS)
    W1 = np.asarray(sd["offset.0.weight"], np.float64) * s[:, None]
    b1 = (np.asarray(sd["offset.0.bias"], np.float64) - mu) * s + b
    W2, b2 = np.asarray(sd["offset.3.weight"], np.float64), np.asarray(sd["offset.3.bias"], np.float64)
    return [np.ascontiguousarray(a, dtype=np.float32) for a in (s0, t0, W1.T, b1, W2.T, b2)]


def _head(sd, x, n, p2v):
    """cg_pointgroup_head_dev with NaN-filled outputs: (site (V,3), out (N,3)) as numpy."""
    from catgrasp_b200 import _lib
    ctx = _lib.Context.get(0)
    V, m = x.shape
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
    site = torch.full((V, 3), NAN, device="cuda")
    out = torch.full((len(p2v), 3), NAN, device="cuda")
    ctx.call("cg_pointgroup_head_dev", ctx.h, dev(x), m, dev(np.int32([n])), V, *map(dev, _head_weights(sd)),
             dev(p2v.astype(np.int32)), len(p2v), site, out)
    return site.cpu().numpy(), out.cpu().numpy()


@pytest.mark.parametrize("V", [1, 7, 8, 9, 1000])
@pytest.mark.parametrize("m", [1, 3, 16, 31, 32, 33, 64, 200, 512])
def test_head(m, V):
    sd = _head_sd(m, 100 + m)
    x = (np.random.RandomState(V).randn(V, m) * 2).astype(np.float32)
    p2v = np.random.RandomState(V + 1).randint(0, V, 2 * V + 3)
    site, out = _head(sd, x, V, p2v)
    y, ey = PR.head(sd, x.astype(np.float64), 0.0)
    ratio = bound_ratio(site, y, ey).max()
    assert ratio <= 1.0, ratio
    assert _eq(out, site[p2v])
    again = _head(sd, x, V, p2v)
    assert _eq(again[0], site) and _eq(again[1], out)


@pytest.mark.parametrize("m", [16, 33])
def test_head_count_word(m):
    """Site rows at or past the count word are not written; a point whose site is at or past it, or negative, gets
    NaN; a count word past the rows is clamped to them."""
    V, n = 1000, 337
    sd = _head_sd(m, 7)
    x = np.random.RandomState(8).randn(V, m).astype(np.float32)
    p2v = np.random.RandomState(9).randint(0, V, 3000)
    p2v[:4] = (-1, -(1 << 31), V, V + 5)
    p2v[4:7] = (n - 1, n, 0)
    site, out = _head(sd, x, n, p2v)
    assert np.isnan(site[n:]).all() and np.isfinite(site[:n]).all()
    y, ey = PR.head(sd, x[:n].astype(np.float64), 0.0)
    assert bound_ratio(site[:n], y, ey).max() <= 1.0
    live = (p2v >= 0) & (p2v < n)
    assert _eq(out[live], site[p2v[live]])
    assert np.isnan(out[~live]).all() and (~live).sum() >= 5
    full, full_out = _head(sd, x, V + 12345, p2v)
    y, ey = PR.head(sd, x.astype(np.float64), 0.0)
    assert bound_ratio(full, y, ey).max() <= 1.0
    ok = (p2v >= 0) & (p2v < V)
    assert _eq(full_out[ok], full[p2v[ok]]) and np.isnan(full_out[~ok]).all()


# ---------------------------------------------------------------- the conv kernel at its tile edges
def _conv(x, nbr, W, n, bn, bias, res):
    from catgrasp_b200 import _lib
    ctx = _lib.Context.get(0)
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
    K, Cin, Cout = W.shape
    Mrows = x.shape[0] if nbr is None else nbr.shape[0]
    out = torch.full((Mrows, Cout), NAN, device="cuda")
    scale, shift = (None, None) if bn is None else bn
    ctx.call("cg_spconv_conv_dev", ctx.h, dev(x), Cin, dev(nbr), K, dev(np.int32([n])), Mrows, dev(W), Cout,
             dev(scale), dev(shift), dev(bias), dev(res), out)
    return out.cpu().numpy()


@pytest.mark.parametrize("V", [63, 65])
@pytest.mark.parametrize("cout", [1, 3, 15, 17, 31, 33, 63, 65, 80, 129])
@pytest.mark.parametrize("cin", [1, 31, 33, 48, 80, 112])
@pytest.mark.parametrize("K", [27, 8, 1])
def test_conv_tile_edges(K, cin, cout, V):
    """V live rows of V + 5 (so the last tile holds padding rows), against spconv_ref.conv with and without BN,
    bias and residual; two runs bitwise equal and the padding rows left as they were."""
    rng = np.random.RandomState(K * 100000 + cin * 1000 + cout * 10 + V)
    Mrows = V + 5
    Vin = Mrows if K == 1 else 2 * V + 3
    nbr = None
    if K > 1:
        nbr = np.where(rng.rand(Mrows, K) < 0.4, rng.randint(0, Vin, (Mrows, K)), -1).astype(np.int32)
        nbr[V // 2] = -1                                            # a row with no input: bias and residual only
    x = rng.randn(Vin, cin).astype(np.float32)
    W = (rng.randn(K, cin, cout) / np.sqrt(K * cin)).astype(np.float32)
    bn = ((rng.rand(cin) + 0.5).astype(np.float32), rng.randn(cin).astype(np.float32))
    bias, res = rng.randn(cout).astype(np.float32), rng.randn(Mrows, cout).astype(np.float32)
    for on in (False, True):
        args = (bn, bias, res) if on else (None, None, None)
        got = _conv(x, nbr, W, V, *args)
        assert _eq(got, _conv(x, nbr, W, V, *args))
        assert np.isnan(got[V:]).all(), "a padding row was written"
        y, ey = S.conv(x, nbr, W, *args, rows=np.arange(V))
        ratio = bound_ratio(got[:V], y, ey).max()
        assert ratio <= 1.0, (on, ratio)
