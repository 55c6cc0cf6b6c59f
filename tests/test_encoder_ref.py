"""CPU tests of the float64 encoder reference (oracle/encoder_ref.py) that the tensor-core kernel tests rely on.

1. It computes the same network as the fp32 torch oracle (oracle/pointnet_ref.py), which is pinned to the
   reference's golden vectors.
2. Its error bound is tight enough to catch the localized trunk bugs that the end-to-end tolerances miss: a skipped
   tile, a skipped warp, swapped columns, a wrong reduction in one channel, a row offset by one point.
"""
import numpy as np
import pytest
import torch

from catgrasp_b200.synthetic import make_state_dict
from catgrasp_b200.weights import pack_blob
from oracle.encoder_ref import FoldedNet, bound_ratio, f2key, key2f


@pytest.fixture(scope="module")
def cls_ref():
    sd = make_state_dict("cls", 10, seed=0)
    blob, n_out = pack_blob(sd, "cls")
    return sd, FoldedNet(blob, "cls", n_out)


def _x(B, N, seed):
    rng = np.random.RandomState(seed)
    return rng.normal(0, 1, (B, N, 6)).astype(np.float32)


def test_key_twins_round_trip():
    v = np.array([0.0, -0.0, 1.5, -1.5, 3e38, -3e38, 1e-45, -1e-45, np.inf, -np.inf], np.float32)
    k = f2key(v)
    assert np.array_equal(key2f(k).view(np.uint32), v.view(np.uint32))
    order = np.argsort(v.astype(np.float64) - 1e-300 * np.signbit(v), kind="stable")   # -0 below +0
    assert np.all(np.diff(k[order].astype(np.int64)) > 0)            # keys sort like the floats
    assert f2key(np.float32(-np.inf)) > 0                              # a zero key is below every float


@pytest.mark.parametrize("kind,n_out,seed", [("cls", 10, 0), ("seg", 300, 1)])
def test_float64_path_matches_fp32_oracle(kind, n_out, seed):
    """Logits and the 1024-channel encoder feature agree with oracle/pointnet_ref.py to fp32 round-off."""
    from oracle import pointnet_ref
    sd = make_state_dict(kind, n_out, seed=seed)
    blob, n = pack_blob(sd, kind)
    ref = FoldedNet(blob, kind, n)
    x = _x(3, 300, 7)
    out = ref.forward(x, engine=0)
    sdt = pointnet_ref._sd(sd)
    with torch.no_grad():
        g32 = pointnet_ref.encoder(sdt, torch.from_numpy(x).permute(0, 2, 1), True)[0].numpy()
    fwd = pointnet_ref.pointnet_cls_forward if kind == "cls" else pointnet_ref.pointnet_seg_forward
    lg32 = fwd(sd, x)[0].numpy()
    for got, want, e in ((g32, out["gC"], out["egC"]), (lg32, out["logits"], out["elogits"])):
        d = np.abs(got.astype(np.float64) - want)
        # the fp32 oracle runs unfolded conv + BN in fp32: its error is of the order of the fp32 engine's bound
        assert d.max() <= 4 * e.max(), (d.max(), e.max())
        assert d.max() < 1e-5 * max(1.0, np.abs(want).max())


def _perturbations(N, ch):
    """Bugs a wrong fragment map, ring phase or tile bound would produce, as (name, zmax(z)) over the pre-bias
    128 -> 1024 outputs z (B,N,1024) of a trunk; ``ch`` is the channel whose max becomes a mean."""
    last = (N - 1) // 128 * 128
    warp_rows = np.ones(N, bool)
    warp_rows[[n for n in range(N) if 48 <= n % 128 < 64]] = False    # warp 3 of every tile

    def swap_pairs(z):
        m = z.amax(1).clone()
        h = 5                                                            # one 64-channel half-chunk
        idx = torch.arange(64 * h, 64 * h + 64)
        m[:, idx] = m[:, idx.view(32, 2).flip(1).reshape(-1)]
        return m

    def mean_ch(z):
        m = z.amax(1).clone()
        m[:, ch] = z[:, :, ch].mean(1)
        return m

    shift = np.minimum(np.arange(N) + 1, N - 1)                         # load_row reads point n + 1
    return [("last tile ignored", lambda z: z[:, :last].amax(1)),
            ("one warp's rows ignored", lambda z: z[:, torch.from_numpy(warp_rows)].amax(1)),
            ("column pairs swapped", swap_pairs),
            (f"channel {ch} mean", mean_ch),
            ("row offset by one", lambda z: z[:, torch.from_numpy(shift)].amax(1))]


@pytest.mark.parametrize("engine", [1, 3])
@pytest.mark.parametrize("trunk", ["A", "B", "C"])
def test_checker_rejects_localized_trunk_bugs(cls_ref, engine, trunk):
    """B=8, N=1000 (the last tile is points 896-999): each perturbed max-pool output lies outside twice the bound
    of the unperturbed one, so a kernel with that bug fails the GPU tests."""
    _, ref = cls_ref
    x = _x(8, 1000, 0)
    full = ref.forward(x, engine=0)
    kw = {"A": {}, "B": {"T3": full["T3"]}, "C": {"T3": full["T3"], "T64": full["T64"]}}[trunk]
    z, ez, _, _ = ref.trunk_pre(trunk, x, engine=engine, **kw)
    g = ref.finish(trunk, z.amax(1)).numpy()
    eg = ez.amax(1).numpy()
    assert bound_ratio(g, g, eg).max() == 0
    # a channel that the ReLU of trunks A and B holds at 0 on every point is 0 whatever the reduction: the mean bug
    # goes to channel 517 or, if that one is dead, the next live channel
    ch = 517 + int(np.argmax((g[:, 517:] > 0).any(0)))
    for name, red in _perturbations(1000, ch):
        gp = ref.finish(trunk, red(z)).numpy()
        r = bound_ratio(gp, g, eg)
        print(f"trunk {trunk} engine {engine} {name}: {int((r > 1).sum())} values past 2x the bound, "
              f"max ratio {r.max():.3g}")
        assert r.max() > 1, (trunk, engine, name)
