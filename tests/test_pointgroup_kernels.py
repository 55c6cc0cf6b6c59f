"""PointGroup on the device (catgrasp_b200/pointgroup.py, the voxel-mean and offset-head kernels of cg_spconv.cu,
PointGroupPredictor) against oracle/pointgroup_ref.py and tests/golden/pointgroup.npz.

The oracle's propagated bound is rigorous but grows by the weights' absolute row sums at every one of the U-Net's
~60 layers in series, so on its own it cannot tell a wiring error from rounding.  Every forward is therefore also held
to REL of the largest float64 offset, which fp32 rounding stays far inside and any wiring error leaves.

Seeded mutations, each caught (first failing test shown):
  - decoder half first in the concatenation            test_forward_golden (REL)
  - the tail's k1 identity branch skipped               test_forward_golden (REL)
  - the residual taken after the BN, not the raw input  test_forward_golden (REL)
  - the head's BN left out (b1, W1 unfolded)            test_forward_golden (REL)
  - a coarse level's table used in a tail block         test_forward_golden (REL)
  - a site's points summed in reverse order             test_voxel_mean[777-6-2] (bit for bit)
  - the scale applied after the min is subtracted       test_sites_scale_before_min (locs bit for bit)
"""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from catgrasp_b200 import pointgroup, spconv, synthetic, weights   # noqa: E402
from catgrasp_b200.predicter import PointGroupPredictor              # noqa: E402
from oracle import pointgroup_ref as PR                               # noqa: E402
from oracle.encoder_ref import bound_ratio                            # noqa: E402

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "pointgroup.npz"))
CLASSES = ("hnm", "nut", "screw")
KEY_SHAPES = [(k, tuple(s)) for k, s in json.loads(str(G["key_shapes"]))]
M, REPS = int(G["m"]), int(G["block_reps"])
REL = 1e-3


@pytest.fixture(scope="module")
def sd16():
    return PR.synthetic_state_dict(KEY_SHAPES, int(G["seed"]))


@pytest.fixture(scope="module")
def net16(sd16):
    return pointgroup.PointGroupNet(sd16, M, REPS, device=0)


def _level(sites, shape):
    return spconv.index(torch.from_numpy(np.ascontiguousarray(sites, dtype=np.int32)).cuda(), tuple(shape))


def _run(net, locs, shape, feats):
    """Device offsets twice (bitwise equal) from point sites and features."""
    level, p2v = _level(locs, shape)
    f = torch.from_numpy(np.ascontiguousarray(feats, dtype=np.float32)).cuda()
    a = net.offsets(level, p2v, f)
    b = net.offsets(level, p2v, f)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    return a.cpu().numpy()


def _check(got, off, bound):
    assert bound_ratio(got, off, bound).max() <= 1.0
    scale = np.abs(off).max()
    assert np.abs(got - off).max() <= REL * scale, np.abs(got - off).max() / scale


def _oracle(sd, m, reps, locs, shape, feats):
    locs4 = np.concatenate([np.zeros((len(locs), 1), np.int64), locs], 1)
    vl, p2v, v2p = PR.voxelization_idx(locs4)
    off, bound, _, _ = PR.forward(sd, m, reps, vl[:, 1:], shape, PR.voxelization(feats, v2p), p2v)
    return off, bound


@pytest.mark.parametrize("N,C,seed", [(1, 6, 0), (2, 6, 1), (777, 6, 2), (4096 + 5, 3, 3), (1 << 20, 6, 4)])
def test_voxel_mean(N, C, seed):
    rng = np.random.RandomState(seed)
    side = max(2, int(round((N / 4) ** (1 / 3))))
    locs = rng.randint(0, side, (N, 3)).astype(np.int64)
    if N > 4096:
        locs[rng.permutation(N - 1)[:4096]] = (0, 0, 0)        # one site with at least 4096 points
    if N > 1:
        locs[-1] = (side, side, side)                          # one site with exactly one point
    feats = (rng.randn(N, C) * rng.uniform(0.1, 10, C)).astype(np.float32)
    level, p2v = _level(locs, locs.max(0) + 1)
    got = pointgroup.voxel_mean(level, p2v, torch.from_numpy(feats).cuda()).cpu().numpy()
    locs4 = np.concatenate([np.zeros((N, 1), np.int64), locs], 1)
    vl, rp2v, v2p = PR.voxelization_idx(locs4)
    want = PR.voxelization(feats, v2p)
    # the device's sites come in key order, the reference's in first-seen order: match them by coordinates
    dev_sites = level.vox.cpu().numpy().astype(np.int64)
    order = np.argsort(spconv_key(vl[:, 1:]))
    assert np.array_equal(dev_sites, vl[order, 1:])
    assert np.array_equal(got.view(np.uint32), want[order].view(np.uint32))
    assert v2p[:, 0].max() >= (4096 if N > 4096 else 1) and (v2p[:, 0] == 1).any()
    assert np.array_equal(p2v.cpu().numpy(), np.argsort(order)[rp2v])


def spconv_key(c):
    c = np.asarray(c, dtype=np.int64)
    return (c[:, 0] << 42) | (c[:, 1] << 21) | c[:, 2]


@pytest.mark.parametrize("cls", CLASSES)
def test_forward_golden(cls, net16):
    got = _run(net16, G[f"{cls}_locs"], G[f"{cls}_spatial_shape"],
               PR.host_front(G[f"{cls}_cloud_xyz"], G[f"{cls}_cloud_normal"])[2])
    _check(got, G[f"{cls}_offsets64"], G[f"{cls}_bound"])


@pytest.mark.parametrize("n_points,seed", [(500, 11), (20000, 12), (120000, 13)])
def test_forward_pile(n_points, seed, sd16, net16):
    sc = synthetic.make_pile(n_points, n_objects=max(2, n_points // 2000), seed=seed)
    _, locs, feats, shape = PR.host_front(sc["cloud_xyz"], sc["cloud_normal"])
    _check(_run(net16, locs, shape, feats), *_oracle(sd16, M, REPS, locs, shape, feats))


def test_forward_m32():
    keys = list(weights.pointgroup_keys(32, 2).items())
    sd = PR.synthetic_state_dict(keys, 5)
    net = pointgroup.PointGroupNet(sd, 32, 2, device=0)
    sc = synthetic.make_pile(6000, n_objects=4, seed=14)
    _, locs, feats, shape = PR.host_front(sc["cloud_xyz"], sc["cloud_normal"])
    _check(_run(net, locs, shape, feats), *_oracle(sd, 32, 2, locs, shape, feats))


def test_forward_block_reps_1():
    sd = PR.synthetic_state_dict(list(weights.pointgroup_keys(8, 1).items()), 6)
    net = pointgroup.PointGroupNet(sd, 8, 1, device=0)
    sc = synthetic.make_pile(3000, n_objects=3, seed=15)
    _, locs, feats, shape = PR.host_front(sc["cloud_xyz"], sc["cloud_normal"])
    _check(_run(net, locs, shape, feats), *_oracle(sd, 8, 1, locs, shape, feats))


def test_forward_does_not_synchronise(net16):
    cls = "nut"
    level, p2v = _level(G[f"{cls}_locs"], G[f"{cls}_spatial_shape"])
    f = torch.from_numpy(PR.host_front(G[f"{cls}_cloud_xyz"], G[f"{cls}_cloud_normal"])[2]).cuda()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = net16.offsets(level, p2v, f)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert out.shape == (len(G[f"{cls}_locs"]), 3)


@pytest.fixture(scope="module")
def artifact_dir(tmp_path_factory, sd16):
    import yaml
    d = tmp_path_factory.mktemp("artifacts-pg")
    cfg = {"downsample_size": 0.0005,
           "GENERAL": {"input_channel": 3, "scale": 500, "full_scale": [128, 999999], "mode": 4},
           "STRUCTURE": {"m": M, "block_residual": True, "block_reps": REPS, "use_coords": True},
           "GROUP": {"prepare_epochs": 999999}}
    (d / "config_pointgroup.yaml").write_text(yaml.safe_dump(cfg))
    torch.save({"state_dict": {"module." + k: torch.from_numpy(v) for k, v in sd16.items()}},
               str(d / "best_val.pth.tar"))
    return str(d)


@pytest.mark.parametrize("cls", CLASSES)
def test_host_front_golden(cls, artifact_dir):
    p = PointGroupPredictor(cls, artifact_dir=artifact_dir, device=0)
    xo, locs, feats, shape = p.host_front({"cloud_xyz": G[f"{cls}_cloud_xyz"], "cloud_normal": G[f"{cls}_cloud_normal"]})
    assert np.array_equal(xo, G[f"{cls}_xyz_original_all"])
    assert np.array_equal(locs, G[f"{cls}_locs"]) and tuple(shape) == tuple(G[f"{cls}_spatial_shape"])


@pytest.mark.parametrize("cls", CLASSES)
def test_predict_golden(cls, artifact_dir):
    p = PointGroupPredictor(cls, artifact_dir=artifact_dir, device=0)
    data = {"cloud_xyz": G[f"{cls}_cloud_xyz"].copy(), "cloud_normal": G[f"{cls}_cloud_normal"].copy()}
    labels = p.predict(data)
    assert labels.dtype == np.int64 and np.array_equal(labels, G[f"{cls}_labels_all"])
    want = G[f"{cls}_xyz_shifted"]
    assert p.xyz_shifted.shape == want.shape
    # float32 point + float32 offset: the offset's error plus one rounding of the sum
    lim = REL * np.abs(G[f"{cls}_offsets64"]).max() + np.spacing(np.abs(want))
    assert (np.abs(p.xyz_shifted.astype(np.float64) - want) <= lim).all()


def _order_sensitive_xs(xmin, count):
    """float32 x > xmin where trunc(fl(fl(x * 500) - fl(xmin * 500))) differs from trunc(fl(fl(x - xmin) * 500))."""
    f, out = np.float32, []
    for k in range(1, 400):
        x = f(xmin + f(k) / f(500))
        for _ in range(40):
            x = np.nextafter(x, f(-1))
        for _ in range(80):
            if int(f(f(x * f(500)) - f(xmin * f(500)))) != int(f(f(x - xmin) * f(500))):
                out.append(x)
                break
            x = np.nextafter(x, f(1))
        if len(out) == count:
            return np.array(out, np.float32)
    raise AssertionError("no order-sensitive coordinates found")


def test_sites_scale_before_min(artifact_dir):
    # sites are trunc((xyz * scale) - min), the scale first, as the reference computes them; here the other order
    # truncates differently.  Points 2 mm apart in y, so each is alone in its voxel and snaps to itself.
    xmin = np.float32(0.0123457)
    xs = np.concatenate([[xmin], _order_sensitive_xs(xmin, 6)]).astype(np.float32)
    xyz = np.stack([xs, np.arange(len(xs), dtype=np.float32) * np.float32(0.002),
                    np.full(len(xs), 0.7, np.float32)], 1)
    nrm = np.tile(np.float32([0, 0, 1]), (len(xs), 1))
    p = PointGroupPredictor("nut", artifact_dir=artifact_dir, device=0)
    xo, locs, _, shape = p.host_front({"cloud_xyz": xyz, "cloud_normal": nrm})
    rxo, rlocs, _, rshape = PR.host_front(xyz, nrm)
    assert np.array_equal(xo, rxo) and np.array_equal(locs, rlocs) and tuple(shape) == tuple(rshape)
    alt = ((rxo - rxo.min(0)) * np.float32(500)).astype(np.int64)
    assert (alt != rlocs).any()
