"""oracle/spconv_ref.py against dense torch convolutions on zero-filled grids (spconv's own test contract,
test/test_conv.py: the weight (kx, ky, kz, Cin, Cout) permuted to torch's layout), CPU only.

Grids of 5 ... 13 sites per axis, odd and even, with isolated sites and sites on every face and corner:
  SubM k3   == conv3d(padding=1) read at the sites
  SubM k1   == x @ W
  down      == conv3d(stride=2) read at the parents; the parents are those of the children inside the coarse shape
  up        == conv_transpose3d(stride=2) zero-padded to the fine shape, read at the sites (a child on an odd axis's
               last plane gets nothing)
and the error bound holds a float32 evaluation (torch's own summation order) of each.
"""
import itertools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import spconv_ref as R

SHAPES = [(5, 5, 5), (6, 7, 8), (13, 12, 11), (9, 13, 6), (12, 12, 12)]


def _sites(shape, seed, density=0.3):
    """Random sites plus every corner and a site on each face centre, in shuffled order with
    duplicates (so the level is a proper subset of the rows)."""
    rng = np.random.RandomState(seed)
    X, Y, Z = shape
    grid = np.stack(np.meshgrid(np.arange(X), np.arange(Y), np.arange(Z), indexing="ij"), -1).reshape(-1, 3)
    pick = grid[rng.rand(len(grid)) < density]
    corners = np.array(list(itertools.product([0, X - 1], [0, Y - 1], [0, Z - 1])))
    faces = np.array([[0, Y // 2, Z // 2], [X - 1, Y // 2, Z // 2], [X // 2, 0, Z // 2], [X // 2, Y - 1, Z // 2],
                      [X // 2, Y // 2, 0], [X // 2, Y // 2, Z - 1]])
    c = np.concatenate([pick, corners, faces, pick[: len(pick) // 3]])
    return c[rng.permutation(len(c))].astype(np.int32)


def _weights(K, cin, cout, seed):
    return (np.random.RandomState(seed).randn(*K, cin, cout) / np.sqrt(np.prod(K) * cin)).astype(np.float32)


def _feats(n, c, seed):
    return np.random.RandomState(seed).randn(n, c).astype(np.float32)


def _at(g, vox):
    v = np.asarray(vox, dtype=np.int64)
    return g[0][:, v[:, 0], v[:, 1], v[:, 2]].T


def _within(f32, y, ey):
    assert (np.abs(np.asarray(f32, dtype=np.float64) - y) <= ey).all()


def test_index_matches_brute_force():
    coords = _sites((7, 6, 9), 0)
    vox, p2v, nbr = R.index(coords)
    assert (vox[p2v] == coords).all()
    assert len({tuple(v) for v in vox}) == len(vox) == len({tuple(c) for c in coords})
    assert (np.diff(R.pack(vox)) > 0).all()
    where = {tuple(v): i for i, v in enumerate(vox)}
    for i, v in enumerate(vox):
        for k in range(27):
            q = (v[0] + k // 9 - 1, v[1] + k // 3 % 3 - 1, v[2] + k % 3 - 1)
            assert nbr[i, k] == where.get(q, -1)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("cin, cout", [(6, 16), (32, 16)])
def test_subm_k3_equals_dense_conv(shape, cin, cout):
    vox, _, nbr = R.index(_sites(shape, sum(shape)))
    x = _feats(len(vox), cin, 1)
    W = _weights((3, 3, 3), cin, cout, 2)
    y, ey = R.conv(x, nbr, W)
    wt = torch.from_numpy(W).permute(4, 3, 0, 1, 2)
    dense = F.conv3d(torch.from_numpy(R.dense_grid(vox, x, shape)), wt.double(), padding=1).numpy()
    np.testing.assert_allclose(y, _at(dense, vox), rtol=0, atol=1e-12)
    f32 = F.conv3d(torch.from_numpy(R.dense_grid(vox, x, shape)).float(), wt, padding=1).numpy()
    _within(_at(f32, vox), y, ey)


def test_subm_k3_isolated_site_sees_only_itself():
    coords = np.array([[0, 0, 0], [4, 4, 4], [4, 4, 5]], dtype=np.int32)
    vox, _, nbr = R.index(coords)
    assert (nbr[0] == [-1] * 13 + [0] + [-1] * 13).all()
    x, W = _feats(3, 4, 3), _weights((3, 3, 3), 4, 5, 4)
    y, _ = R.conv(x, nbr, W)
    np.testing.assert_allclose(y[0], x[0].astype(np.float64) @ W[1, 1, 1].astype(np.float64), rtol=0, atol=1e-15)


def test_subm_k1_is_a_matrix_product():
    x, W = _feats(17, 12, 5), _weights((1, 1, 1), 12, 7, 6)
    y, ey = R.conv(x, None, W)
    np.testing.assert_allclose(y, x.astype(np.float64) @ W[0, 0, 0].astype(np.float64), rtol=0, atol=1e-13)
    _within(x @ W[0, 0, 0], y, ey)


@pytest.mark.parametrize("shape", SHAPES)
def test_down_equals_strided_dense_conv(shape):
    vox, _, _ = R.index(_sites(shape, 3 * sum(shape)))
    cvox, cnbr, dn, up, cs = R.down(vox, shape)
    assert cs == tuple((s - 2) // 2 + 1 for s in shape)
    kept = vox[(vox >> 1 < np.array(cs)).all(1)]
    assert {tuple(p) for p in cvox} == {tuple(p) for p in kept >> 1}
    if any(s % 2 for s in shape):
        assert len(kept) < len(vox)                     # an odd axis's last plane is dropped
    assert (cnbr == R.neighbours(cvox)).all()
    x, W = _feats(len(vox), 16, 7), _weights((2, 2, 2), 16, 24, 8)
    y, ey = R.conv(x, dn, W)
    wt = torch.from_numpy(W).permute(4, 3, 0, 1, 2)
    g = torch.from_numpy(R.dense_grid(vox, x, shape))
    dense = F.conv3d(g, wt.double(), stride=2).numpy()
    assert dense.shape[2:] == cs
    np.testing.assert_allclose(y, _at(dense, cvox), rtol=0, atol=1e-12)
    _within(_at(F.conv3d(g.float(), wt, stride=2).numpy(), cvox), y, ey)


@pytest.mark.parametrize("shape", SHAPES)
def test_up_equals_transposed_dense_conv(shape):
    vox, _, _ = R.index(_sites(shape, 5 * sum(shape)))
    cvox, _, dn, up, cs = R.down(vox, shape)
    x, W = _feats(len(cvox), 24, 9), _weights((2, 2, 2), 24, 16, 10)
    b = np.random.RandomState(11).randn(16).astype(np.float32)
    y, ey = R.conv(x, up, W, bias=b)
    wt = torch.from_numpy(W).permute(3, 4, 0, 1, 2)
    g = torch.from_numpy(R.dense_grid(cvox, x, cs))
    pad = [(0, s - 2 * c) for s, c in zip(shape, cs)]
    dense = F.pad(F.conv_transpose3d(g, wt.double(), stride=2), [p for q in reversed(pad) for p in q]).numpy()
    np.testing.assert_allclose(y, _at(dense, vox) + b, rtol=0, atol=1e-12)
    dropped = (up < 0).all(1)
    assert dropped.any() == any(s % 2 for s in shape)
    assert (y[dropped] == b.astype(np.float64)).all()
    f32 = F.pad(F.conv_transpose3d(g.float(), wt, stride=2), [p for q in reversed(pad) for p in q]).numpy()
    _within(_at(f32, vox) + b, y, ey)


def test_down_then_up_pairs_are_inverse():
    vox, _, _ = R.index(_sites((11, 10, 9), 12))
    _, _, dn, up, _ = R.down(vox, (11, 10, 9))
    for p, k in zip(*np.nonzero(dn >= 0)):
        assert up[dn[p, k], k] == p
    assert (up >= 0).sum() == (dn >= 0).sum()


def test_bn_prologue_acts_on_present_rows_only():
    """Absent neighbours contribute 0, not ReLU(shift): normalising a dense grid everywhere gives another answer."""
    shape = (6, 6, 6)
    vox, _, nbr = R.index(_sites(shape, 13, density=0.1))
    x, W = _feats(len(vox), 8, 14), _weights((3, 3, 3), 8, 8, 15)
    s = np.random.RandomState(16).rand(8).astype(np.float32) + 0.5
    t = np.abs(np.random.RandomState(17).randn(8)).astype(np.float32) + 0.1
    y, ey = R.conv(x, nbr, W, bn=(s, t))
    a = np.maximum(x.astype(np.float64) * s + t, 0)
    wt = torch.from_numpy(W).permute(4, 3, 0, 1, 2).double()
    good = F.conv3d(torch.from_numpy(R.dense_grid(vox, a, shape)), wt, padding=1).numpy()
    np.testing.assert_allclose(y, _at(good, vox), rtol=0, atol=1e-12)
    g = R.dense_grid(vox, x, shape)
    everywhere = np.maximum(g * s.reshape(1, -1, 1, 1, 1) + t.reshape(1, -1, 1, 1, 1), 0)
    wrong = _at(F.conv3d(torch.from_numpy(everywhere), wt, padding=1).numpy(), vox)
    assert (np.abs(wrong - y) > 2 * ey).any()


def test_bound_grows_with_input_bound_and_residual():
    vox, _, nbr = R.index(_sites((5, 6, 7), 18))
    x, W = _feats(len(vox), 6, 19), _weights((3, 3, 3), 6, 4, 20)
    res = _feats(len(vox), 4, 21)
    y0, e0 = R.conv(x, nbr, W)
    y1, e1 = R.conv(x, nbr, W, residual=res, ex=np.full(x.shape, 1e-6), eres=np.full(res.shape, 1e-7))
    np.testing.assert_allclose(y1, y0 + res, rtol=0, atol=1e-12)
    assert (e1 > e0 + 1e-7).all()
