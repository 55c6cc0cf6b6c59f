"""cg_spconv.cu (catgrasp_b200.spconv) against oracle/spconv_ref.py: the level, neighbour, down and up tables bit for
bit, and every convolution type within 2x the oracle's float64 bound, bitwise equal across two runs.

Seeded kernel mutations, each caught (first failing test shown):
  - k <-> 26 - k in the neighbour table (convolution for correlation)  test_index_tables
  - k <-> K - 1 - k in the conv kernel's weight offset                 test_subm_k3
  - BN + ReLU applied at absent neighbours                             test_subm_k3 (positive shifts)
  - the odd-plane drop ignored (no bound on the parent index)          test_index_tables (odd shapes)
  - the inverse offset mirrored (7 - k in the up table)                test_index_tables
  - the last output tile skipped                                       test_subm_k3 at V = tile + 1
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from catgrasp_b200 import spconv   # noqa: E402
from oracle import spconv_ref as R  # noqa: E402
from oracle.encoder_ref import bound_ratio  # noqa: E402

TILE = 64


def _coords(shape, n, seed):
    rng = np.random.RandomState(seed)
    return np.stack([rng.randint(0, s, n) for s in shape], 1).astype(np.int32)


def _sites(V, seed, side=9):
    """V distinct sites of a side^3 block (dense enough that most have neighbours), in shuffled order."""
    rng = np.random.RandomState(seed)
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3)
    return g[rng.permutation(len(g))[:V]].astype(np.int32), (side,) * 3


def _rand(shape, seed, scale=1.0):
    return (np.random.RandomState(seed).randn(*shape) * scale).astype(np.float32)


def _bn(C, seed):
    rng = np.random.RandomState(seed)
    return (rng.rand(C) + 0.5).astype(np.float32), (np.abs(rng.randn(C)) + 0.2).astype(np.float32)


def _cuda(*a):
    return [None if x is None else torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a]


def _check(x, nbr, W, n, bn=None, bias=None, res=None, rows=None):
    """Kernel vs oracle within 2x the bound on `rows` (default all), and two runs bitwise equal."""
    xt, nt, Wt, bt, rt = _cuda(x, nbr, W, bias, res)
    bnt = None if bn is None else tuple(_cuda(*bn))
    nw = torch.tensor([n], dtype=torch.int32, device="cuda")
    got = spconv.conv(xt, nt, Wt, nw, bn=bnt, bias=bt, residual=rt)
    again = spconv.conv(xt, nt, Wt, nw, bn=bnt, bias=bt, residual=rt)
    assert torch.equal(got.view(torch.int32), again.view(torch.int32))
    assert not got[n:].any()
    rows = np.arange(n) if rows is None else rows
    y, ey = R.conv(x, nbr, W, bn=bn, bias=bias, residual=res, rows=rows)
    ratio = bound_ratio(got.cpu().numpy()[rows], y, ey)
    assert ratio.max() <= 1.0, ratio.max()
    return got


@pytest.mark.parametrize("shape, n", [((1, 1, 1), 1), ((3, 3, 3), 2), ((5, 7, 9), 200), ((6, 6, 6), 400),
                                      ((13, 11, 12), 3000), ((129, 130, 128), 60000), ((128, 128, 128), 1 << 20)])
def test_index_tables(shape, n):
    coords = _coords(shape, n, sum(shape) + n)
    level, p2v = spconv.index(torch.from_numpy(coords).cuda(), shape)
    vox, p2v_r, nbr = R.index(coords)
    V = level.count()
    assert V == len(vox)
    assert (level.vox[:V].cpu().numpy() == vox).all()
    assert (p2v.cpu().numpy() == p2v_r).all()
    got_nbr = level.nbr.cpu().numpy()
    assert (got_nbr[:V] == nbr).all() and (got_nbr[V:] == -1).all()
    coarse, dn, up = spconv.down(level)
    cvox, cnbr, dn_r, up_r, cs = R.down(vox, shape)
    P = coarse.count()
    assert coarse.shape == cs and P == len(cvox)
    assert (coarse.vox[:P].cpu().numpy() == cvox).all()
    assert (coarse.nbr[:P].cpu().numpy() == cnbr).all() and (coarse.nbr[P:] == -1).all()
    dn, up = dn.cpu().numpy(), up.cpu().numpy()
    assert (dn[:P] == dn_r).all() and (dn[P:] == -1).all()
    assert (up[:V] == up_r).all() and (up[V:] == -1).all()


def test_pyramid():
    """Seven levels down from a 135 x 128 x 129 cloud (odd axes at several levels), each equal to the oracle's."""
    shape = (135, 128, 129)
    coords = _coords(shape, 50000, 5)
    level, _ = spconv.index(torch.from_numpy(coords).cuda(), shape)
    vox, _, _ = R.index(coords)
    for _ in range(6):
        level, dn, up = spconv.down(level)
        cvox, cnbr, dn_r, up_r, shape = R.down(vox, shape)
        P = level.count()
        assert level.shape == shape and P == len(cvox)
        assert level.rows == max(1, min(len(vox), int(np.prod(shape))))   # sized by the bound, not the point count
        assert (level.vox[:P].cpu().numpy() == cvox).all()
        assert (level.nbr[:P].cpu().numpy() == cnbr).all()
        assert (dn[:P].cpu().numpy() == dn_r).all() and (up[:len(vox)].cpu().numpy() == up_r).all()
        vox = cvox


@pytest.mark.parametrize("V", [1, 2, TILE - 1, TILE, TILE + 1, 2 * TILE + 1, 700])
@pytest.mark.parametrize("cin, cout", [(6, 16), (16, 16), (32, 48), (64, 112), (192, 112), (96, 65)])
def test_subm_k3(V, cin, cout):
    sites, _ = _sites(V, V + cin)
    _, _, nbr = R.index(sites)
    x = _rand((V, cin), 1)
    W = _rand((3, 3, 3, cin, cout), 2, 1 / np.sqrt(27 * cin))
    _check(x, nbr, W, V)
    _check(x, nbr, W, V, bn=_bn(cin, 3), res=_rand((V, cout), 4))


@pytest.mark.parametrize("V", [1, TILE + 1, 1000])
@pytest.mark.parametrize("cin, cout", [(6, 16), (192, 112), (224, 224)])
def test_k1(V, cin, cout):
    x = _rand((V, cin), 5)
    W = _rand((1, 1, 1, cin, cout), 6, 1 / np.sqrt(cin))
    _check(x, None, W, V, bn=_bn(cin, 7))
    _check(x, None, W, V, bias=_rand((cout,), 8), res=_rand((V, cout), 9))


@pytest.mark.parametrize("shape", [(9, 9, 9), (10, 11, 12), (17, 16, 15)])
@pytest.mark.parametrize("cin, cout", [(16, 32), (112, 96)])
def test_down_and_up(shape, cin, cout):
    vox, _, _ = R.index(_coords(shape, int(0.4 * np.prod(shape)), 11))
    cvox, _, dn, up, _ = R.down(vox, shape)
    x = _rand((len(vox), cin), 12)
    Wd = _rand((2, 2, 2, cin, cout), 13, 1 / np.sqrt(8 * cin))
    _check(x, dn, Wd, len(cvox), bn=_bn(cin, 14))
    xc = _rand((len(cvox), cout), 15)
    Wu = _rand((2, 2, 2, cout, cin), 16, 1 / np.sqrt(cout))
    _check(xc, up, Wu, len(vox), bn=_bn(cout, 17), bias=_rand((cin,), 18))
    dropped = (up < 0).all(1)
    assert dropped.any() == any(s % 2 for s in shape)


def test_large_level():
    """~2^20 sites: a sample of rows, the first and the last two tiles within the bound."""
    shape = (128, 128, 128)
    coords = _coords(shape, 1 << 20, 21)
    level, _ = spconv.index(torch.from_numpy(coords).cuda(), shape)
    V = level.count()
    nbr = level.nbr[:V].cpu().numpy()
    rng = np.random.RandomState(22)
    rows = np.unique(np.concatenate([np.arange(TILE), np.arange(V - 2 * TILE, V), rng.randint(0, V, 4096)]))
    x = _rand((V, 16), 23)
    W = _rand((3, 3, 3, 16, 32), 24, 1 / np.sqrt(27 * 16))
    _check(x, nbr, W, V, bn=_bn(16, 25), bias=_rand((32,), 26), rows=rows)


def test_count_word_limits_the_rows():
    """Rows from the device count on are not written: the table may be larger than the level."""
    sites, _ = _sites(100, 30)
    _, _, nbr = R.index(sites)
    x = _rand((100, 8), 31)
    W = _rand((3, 3, 3, 8, 8), 32, 0.1)
    _check(x, nbr, W, 37)


def test_count_word_past_the_table_is_clamped():
    """A count word larger than the table (another level's, say) writes only the table's rows."""
    sites, _ = _sites(100, 33)
    _, _, nbr = R.index(sites)
    xt, nt, Wt = _cuda(_rand((100, 8), 34), nbr, _rand((3, 3, 3, 8, 16), 35, 0.1))
    want = spconv.conv(xt, nt, Wt, torch.tensor([100], dtype=torch.int32, device="cuda"))
    big = torch.full((1,), 1 << 20, dtype=torch.int32, device="cuda")
    assert torch.equal(spconv.conv(xt, nt, Wt, big).view(torch.int32), want.view(torch.int32))


def test_conv_refuses_wrong_shapes():
    sites, _ = _sites(50, 36)
    _, _, nbr = R.index(sites)
    x, nt, W = _cuda(_rand((50, 8), 37), nbr, _rand((3, 3, 3, 8, 16), 38))
    n = torch.tensor([50], dtype=torch.int32, device="cuda")
    ones = lambda c: torch.ones(c, device="cuda")   # noqa: E731
    for kw in (dict(bias=ones(15)), dict(bn=(ones(7), ones(8))), dict(bn=(ones(8), ones(9))),
               dict(residual=torch.ones(50, 15, device="cuda"))):
        with pytest.raises(ValueError):
            spconv.conv(x, nt, W, n, **kw)
    with pytest.raises(ValueError):
        spconv.conv(x[:49], nt, W, n)                        # the table names row 49
    with pytest.raises(ValueError):
        spconv.conv(x, nt, W, torch.tensor([50, 50], dtype=torch.int32, device="cuda"))
