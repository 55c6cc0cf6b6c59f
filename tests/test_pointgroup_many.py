"""Several frames in one pass through PointGroup's sparse U-Net: spconv.index_many and the batched down step
(cg_spconv_index_many_dev, cg_spconv_down_many_dev), PointGroupNet.offsets on a batched level and
PointGroupPredictor.predict_many, each held bit for bit to the one-frame calls.

  - tables: at every pyramid level, frame b's sites, count and nbr / down / up entries equal the one-frame call's plus
    its row base, for frames of different sizes and odd and even shapes, one site, shape 1 on an axis, identical
    frames, and sites on the top planes of 2^w-wide fields next to the following frame's origin;
  - network: each frame's offsets equal PointGroupNet.offsets on that frame alone, at m = 16 and 32 and block_reps 1;
  - predictor: predict_many's labels and xyz_shifted equal a loop of predict, for numpy and CUDA input;
  - rejections before any launch.
"""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from catgrasp_b200 import _lib, pointgroup, spconv, synthetic, weights   # noqa: E402
from catgrasp_b200.predicter import PointGroupPredictor                     # noqa: E402
from oracle import pointgroup_ref as PR                                      # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
G = np.load(os.path.join(GOLDEN, "pointgroup.npz"))
SEG = np.load(os.path.join(GOLDEN, "segment.npz"))
CLASSES = ("hnm", "nut", "screw")
KEY_SHAPES = [(k, tuple(s)) for k, s in json.loads(str(G["key_shapes"]))]
M16, REPS = int(G["m"]), int(G["block_reps"])


def _coords(shape, n, seed):
    rng = np.random.RandomState(seed)
    return np.stack([rng.randint(0, s, n) for s in shape], 1).astype(np.int32)


def _carry_frames(side):
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.int32)
    top, origin = g[(g == side - 1).any(1)], g[(g == 0).any(1)]
    return [top, origin, np.concatenate([top, origin]), origin[::3]], [(side,) * 3] * 4


BATCHES = {
    "mixed": ([_coords((13, 11, 12), 300, 1), _coords((9, 10, 7), 200, 2), _coords((20, 16, 17), 1500, 3),
               np.array([[2, 3, 4]] * 3, np.int32), _coords((2, 3, 4), 5, 4), _coords((130, 129, 128), 60000, 5)],
              [(13, 11, 12), (9, 10, 7), (20, 16, 17), (5, 5, 5), (2, 3, 4), (130, 129, 128)]),
    "shape_1": ([_coords((8, 9, 10), 200, 6), _coords((1, 6, 7), 30, 7), _coords((9, 1, 9), 40, 8)],
                [(8, 9, 10), (1, 6, 7), (9, 1, 9)]),
    "identical": ([_coords((6, 6, 6), 80, 9), _coords((6, 6, 6), 80, 9), _coords((7, 5, 6), 50, 10)],
                  [(6, 6, 6), (6, 6, 6), (7, 5, 6)]),
    "carry": _carry_frames(16),
    "one_site_first": ([np.array([[0, 0, 0]], np.int32), _coords((11, 12, 13), 400, 11)], [(1, 1, 1), (11, 12, 13)]),
    "seven_levels": ([_coords((135, 128, 129), 50000, 13), _coords((128, 128, 128), 20000, 14),
                      _coords((200, 141, 128), 30000, 15)], [(135, 128, 129), (128, 128, 128), (200, 141, 128)]),
}


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _rebase(t, base):
    return np.where(t >= 0, t + base, -1)


def _single_pyramid(coords, shape, depth):
    level, p2v = spconv.index(_cuda(coords), shape)
    out = [(level, None, None)]
    for _ in range(depth - 1):
        coarse, dn, up = spconv.down(out[-1][0])
        out[-1] = (out[-1][0], dn, up)
        out.append((coarse, None, None))
    return out, p2v


def _depth(shapes):
    """Levels every frame's one-frame pyramid can build (a coarse shape of 0 takes no further down step), at most 7."""
    d, shapes = 1, [tuple(s) for s in shapes]
    while d < 7 and min(min(s) for s in shapes) >= 1:
        shapes = [spconv.coarse_shape(s) for s in shapes]
        d += 1
    return d


def _np(t):
    return t.cpu().numpy()


def check_tables(frames, shapes):
    depth = _depth(shapes)
    level, p2v = spconv.index_many([_cuda(c) for c in frames], shapes)
    batched = [(level, None, None)]
    for _ in range(depth - 1):
        coarse, dn, up = spconv.down(batched[-1][0])
        batched[-1] = (batched[-1][0], dn, up)
        batched.append((coarse, None, None))
    singles = [_single_pyramid(c, s, depth) for c, s in zip(frames, shapes)]
    p2v, start = _np(p2v), 0
    for i in range(depth):
        blv, bdn, bup = batched[i]
        n = [sp[0][i][0].count() for sp in singles]
        base = np.cumsum([0] + n)
        assert blv.count() == base[-1]
        assert blv.shapes == tuple(tuple(sp[0][i][0].shape) for sp in singles)
        if i:
            assert blv.rows == spconv.down_rows(batched[i - 1][0].rows, batched[i - 1][0].shapes)
        vox, nbr, frame = _np(blv.vox), _np(blv.nbr), _np(blv.frame)
        assert (nbr[base[-1]:] == -1).all()
        if bdn is not None:
            dn, up, nxt = _np(bdn), _np(bup), np.cumsum([0] + [sp[0][i + 1][0].count() for sp in singles])
            assert (dn[nxt[-1]:] == -1).all() and (up[base[-1]:] == -1).all()
        for b, (sp, sp2v) in enumerate(singles):
            lv, sdn, sup = sp[i]
            rows = slice(base[b], base[b + 1])
            assert (frame[rows] == b).all()
            assert np.array_equal(vox[rows], _np(lv.vox)[:n[b]])
            assert np.array_equal(nbr[rows], _rebase(_np(lv.nbr)[:n[b]], base[b]))
            if i == 0:
                assert np.array_equal(p2v[start:start + len(frames[b])], _np(sp2v) + base[b])
                start += len(frames[b])
            if sdn is not None:
                assert np.array_equal(dn[nxt[b]:nxt[b + 1]], _rebase(_np(sdn)[:nxt[b + 1] - nxt[b]], base[b]))
                assert np.array_equal(up[rows], _rebase(_np(sup)[:n[b]], nxt[b]))
    return depth


@pytest.mark.parametrize("name", list(BATCHES))
def test_tables_equal_the_frames(name):
    frames, shapes = BATCHES[name]
    assert check_tables(frames, shapes) >= 2


def test_carry_batch_is_on_the_field_edge():
    """The carry batch's largest shape is exactly 2^w: a site at x = 2^w - 1 plus one would key the next frame."""
    frames, shapes = BATCHES["carry"]
    assert spconv.key_layout(shapes) == (2, 4) and max(frames[0][:, 0]) == 15 and (frames[1][:, 0] == 0).any()


def test_one_frame_equals_the_single_call():
    frames, shapes = [_coords((129, 128, 131), 50000, 12)], [(129, 128, 131)]
    check_tables(frames, shapes)
    a, _ = spconv.index_many([_cuda(frames[0])], shapes)
    b, _ = spconv.index(_cuda(frames[0]), shapes[0])
    assert torch.equal(a.vox, b.vox) and torch.equal(a.nbr, b.nbr) and not a.frame.any()


# ---------------------------------------------------------------------------------------------------- network


def _front(cls):
    _, locs, feats, shape = PR.host_front(G[f"{cls}_cloud_xyz"], G[f"{cls}_cloud_normal"])
    return locs, feats, tuple(int(s) for s in shape)


def _pile(n_points, seed):
    sc = synthetic.make_pile(n_points, n_objects=max(2, n_points // 2000), seed=seed)
    _, locs, feats, shape = PR.host_front(sc["cloud_xyz"], sc["cloud_normal"])
    return locs, feats, tuple(int(s) for s in shape)


def _net(m, reps, seed):
    keys = KEY_SHAPES if (m, reps) == (M16, REPS) else list(weights.pointgroup_keys(m, reps).items())
    return pointgroup.PointGroupNet(PR.synthetic_state_dict(keys, seed), m, reps, device=0)


def check_offsets(net, fronts):
    level, p2v = spconv.index_many([_cuda(f[0]) for f in fronts], [f[2] for f in fronts])
    feats = _cuda(np.concatenate([f[1] for f in fronts]))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = net.offsets(level, p2v, feats)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    start = 0
    for locs, f, shape in fronts:
        lv, sp2v = spconv.index(_cuda(locs), shape)
        want = net.offsets(lv, sp2v, _cuda(f))
        assert torch.equal(got[start:start + len(locs)].view(torch.int32), want.view(torch.int32))
        start += len(locs)
    assert start == got.shape[0]


@pytest.mark.parametrize("m, reps, seed", [(M16, REPS, int(G["seed"])), (32, 2, 5), (8, 1, 6)])
def test_offsets_equal_the_frames(m, reps, seed):
    fronts = [_pile(3000, 21), _front("nut"), _pile(500, 22), _front("hnm"), _front("screw"), _pile(20000, 23)]
    check_offsets(_net(m, reps, seed), fronts)


def test_offsets_one_frame():
    check_offsets(_net(M16, REPS, int(G["seed"])), [_front("nut")])


# ---------------------------------------------------------------------------------------------------- predictor


@pytest.fixture(scope="module")
def predictor(tmp_path_factory):
    import yaml
    d = tmp_path_factory.mktemp("artifacts-pg-many")
    cfg = {"downsample_size": 0.0005,
           "GENERAL": {"input_channel": 3, "scale": 500, "full_scale": [128, 999999], "mode": 4},
           "STRUCTURE": {"m": M16, "block_residual": True, "block_reps": REPS, "use_coords": True},
           "GROUP": {"prepare_epochs": 999999}}
    (d / "config_pointgroup.yaml").write_text(yaml.safe_dump(cfg))
    sd = PR.synthetic_state_dict(KEY_SHAPES, int(G["seed"]))
    torch.save({"state_dict": {"module." + k: torch.from_numpy(v) for k, v in sd.items()}},
               str(d / "best_val.pth.tar"))
    return PointGroupPredictor("nut", artifact_dir=str(d), device=0)


def _frames():
    out = [{"cloud_xyz": G[f"{c}_cloud_xyz"].copy(), "cloud_normal": G[f"{c}_cloud_normal"].copy()} for c in CLASSES]
    seg = SEG["nut_cloud_xyz"].copy()
    out.insert(1, {"cloud_xyz": seg, "cloud_normal": np.tile(np.float32([0, 0, -1]), (len(seg), 1))})
    sc = synthetic.make_pile(8000, n_objects=4, seed=31)
    out.append({"cloud_xyz": sc["cloud_xyz"].astype(np.float32), "cloud_normal": sc["cloud_normal"].astype(np.float32)})
    return out


def _same(a, b):
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))
    return a.is_cuda and b.is_cuda and _same(a.cpu().numpy(), b.cpu().numpy())


@pytest.mark.parametrize("kind", ["numpy", "cuda"])
def test_predict_many_equals_the_loop(predictor, kind):
    frames = _frames()
    if kind == "cuda":
        frames = [{k: _cuda(v) for k, v in d.items()} for d in frames]
    want, shifted = [], []
    for d in frames:
        want.append(predictor.predict(d))
        shifted.append(predictor.xyz_shifted)
    predictor.xyz_shifted = None
    got = predictor.predict_many(frames)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert _same(g, w)
    assert _same(predictor.xyz_shifted, shifted[-1])
    one = predictor.predict_many(frames[-1:])
    assert _same(one[0], want[-1]) and _same(predictor.xyz_shifted, shifted[-1])


def test_predict_many_rejections(predictor):
    ctx = predictor.model.ctx
    good = _frames()[0]
    bad_shape = {"cloud_xyz": good["cloud_xyz"][:, :2], "cloud_normal": good["cloud_normal"][:, :2]}
    no_normal = {"cloud_xyz": good["cloud_xyz"]}
    mixed = [good, {k: _cuda(v) for k, v in good.items()}]
    with pytest.raises(KeyError) as loop_err:
        predictor.predict(no_normal)
    marker = object()
    predictor.xyz_shifted = marker
    torch.cuda.synchronize()
    ctx.reset_launch_count()
    with pytest.raises(ValueError, match="no frames"):
        predictor.predict_many([])
    with pytest.raises(ValueError, match="all numpy arrays or all CUDA tensors"):
        predictor.predict_many(mixed)
    with pytest.raises(ValueError, match="frame 1 has cloud_xyz"):
        predictor.predict_many([good, bad_shape])
    with pytest.raises(KeyError) as err:
        predictor.predict_many([good, no_normal])
    assert err.value.args == loop_err.value.args
    with pytest.raises(ValueError, match="M >= 1"):
        predictor.predict({"cloud_xyz": good["cloud_xyz"][:0], "cloud_normal": good["cloud_normal"][:0]})
    assert ctx.launch_count() == 0 and predictor.xyz_shifted is marker


def test_keys_that_do_not_fit_are_refused_before_launch():
    """f + 3w <= 63: two frames of 2^21 per axis (w = 21, f = 1) are refused by Python and by the C entry, with no
    launch; one frame of 2^21 per axis still indexes, through both entries."""
    ctx = _lib.Context.get(0)
    big = (1 << 21,) * 3
    c = np.array([[0, 0, 0], [(1 << 21) - 1] * 3, [(1 << 21) - 1, (1 << 21) - 2, (1 << 21) - 1]], np.int32)
    torch.cuda.synchronize()
    ctx.reset_launch_count()
    with pytest.raises(ValueError, match="f \\+ 3 w <= 63"):
        spconv.index_many([_cuda(c), _cuda(c)], [big, big])
    ct = _cuda(np.concatenate([c, c]))
    out = [torch.empty(s, dtype=torch.int32, device="cuda") for s in ((6, 3), (1,), (6,), (6,), (6, 27))]
    with pytest.raises(_lib.CgError, match="f \\+ 3 w <= 63"):
        ctx.call("cg_spconv_index_many_dev", ctx.h, ct, 6, 2, np.int32([0, 3, 6]), np.int32([big, big]), *out)
    with pytest.raises(_lib.CgError, match="f \\+ 3 w <= 63"):
        ctx.call("cg_spconv_down_many_dev", ctx.h, ct, out[2], out[1], 6, 2, np.int32([big, big]), 6, out[0], out[1],
                 out[2], out[4], torch.empty((6, 8), dtype=torch.int32, device="cuda"),
                 torch.empty((6, 8), dtype=torch.int32, device="cuda"))
    assert ctx.launch_count() == 0
    one, _ = spconv.index(_cuda(c), big)
    many, _ = spconv.index_many([_cuda(c)], [big])
    for lv in (one, many):
        assert lv.count() == 3
        nbr = _np(lv.nbr)
        assert nbr[1, 9 * 1 + 3 * 2 + 1] == 2                   # (2^21-1, 2^21-2, 2^21-1) + (0, 1, 0)
        assert (nbr[2] >= 0).sum() == 2                          # itself and the site below in y, nothing past 2^21
    assert torch.equal(one.vox, many.vox) and torch.equal(one.nbr, many.nbr)
    fits = [(1 << 20,) * 3] * 8                                  # f = 3, w = 20: exactly 63 bits
    check_tables([c // 2] * 8, fits)
