"""GPU: NunocsPredicter.predict_many against a loop of predict, and its batched device entries against the
single-object ones.

- Equivalence with the loop, bit for bit: every returned array, numpy's generator afterwards and the attributes
  data_transformed, confidence_z, pred_bins, best_ratio and nocs_pose, for B in {1, 2, 5, 16} objects cut from a
  synthetic pile (masked counts below, at and above n_pts), in both subsample modes, with the kd-tree evaluation off
  and on, for numpy and CUDA input.
- A batch that mixes objects with a pose and a collinear object without one.
- Batch independence of the device work: an object's forward outputs and pose-search record are the same alone,
  first and last in a batch of 16.
- The reference's numbers: the two NUNOCS goldens as object 0 of a batch reproduce the recorded results.
- Chunking: a batch long enough to split the forward and the pose search into several passes gives the bits of
  batches short enough to run in one.
- Engines: the batched forward equals the single-object forward, object by object, on every trunk engine.
"""
import copy
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ENGINES = [int(e) for e in os.environ.get("CG_TEST_ENGINES", "0,1,2,3").split(",")]


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.cuda.set_device(0)
    return 0


def _predicter(tmp, n_pts, state_dict, normalizer=True):
    from catgrasp_b200.predicter import NunocsPredicter
    from catgrasp_b200.synthetic import write_artifacts
    d = write_artifacts(str(tmp), "seg", n_pts, with_normalizer=normalizer, state_dict=state_dict)
    return NunocsPredicter("nut", artifact_dir=d, device=0)


@pytest.fixture(scope="module")
def lattice(cuda, tmp_path_factory):
    from catgrasp_b200.synthetic import make_lattice_seg_state_dict
    return _predicter(tmp_path_factory.mktemp("lat"), 512, make_lattice_seg_state_dict(seed=5), normalizer=False)


@pytest.fixture(scope="module")
def objects():
    """16 objects of a pile (about 400-900 points each) with a few points under z = 0.1, and one cut to exactly 512."""
    from catgrasp_b200.synthetic import make_pile
    scene = make_pile(12000, n_objects=16, seed=7)
    out = []
    for k in range(16):
        m = scene["object_id"] == k
        xyz, nrm = scene["cloud_xyz"][m].copy(), scene["cloud_normal"][m].copy()
        xyz[:3, 2] = 0.05                                     # masked out
        out.append({"cloud_xyz": xyz, "cloud_normal": nrm})
    big = next(i for i, o in enumerate(out) if len(o["cloud_xyz"]) > 520)
    out[big] = {k: v[:515] for k, v in out[big].items()}       # 512 points with z >= 0.1
    return out


def _np(v):
    return v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)


def _eq(a, b, what):
    if a is None or b is None:
        assert a is None and b is None, what
        return
    assert type(a) is type(b), (what, type(a), type(b))
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for k in a:
            _eq(a[k], b[k], f"{what}[{k}]")
        return
    if isinstance(a, torch.Tensor):
        assert a.is_cuda == b.is_cuda, what
    if isinstance(a, (float, int)):
        assert a == b, what
        return
    x, y = _np(a), _np(b)
    assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), what


ATTRS = ("data_transformed", "confidence_z", "pred_bins", "best_ratio", "nocs_pose")


def _run(pred, fn, seed=0):
    for a in ATTRS:
        pred.__dict__.pop(a, None)
    np.random.seed(seed)
    out = fn()
    st = np.random.get_state()
    return out, (st[1].copy(), st[2]), {a: getattr(pred, a, None) for a in ATTRS}


def _check_equal_to_loop(pred, datas, ids=None):
    keep = copy.deepcopy([{k: _np(v) for k, v in d.items()} for d in datas])
    want = _run(pred, lambda: [pred.predict(copy.deepcopy(d), None if ids is None else ids[b])
                               for b, d in enumerate(datas)])
    got = _run(pred, lambda: pred.predict_many(datas, ids=ids))
    assert len(got[0]) == len(datas)
    for b, (w, g) in enumerate(zip(want[0], got[0])):
        _eq(w[0], g[0], f"nocs[{b}]")
        _eq(w[1], g[1], f"pose[{b}]")
    assert np.array_equal(want[1][0], got[1][0]) and want[1][1] == got[1][1], "numpy state"
    for a in ATTRS:
        _eq(want[2][a], got[2][a], a)
    for d, k in zip(datas, keep):                              # not modified
        assert d.keys() == k.keys() and all(_np(d[n]).tobytes() == k[n].tobytes() for n in k)
    return got[0]


@pytest.mark.parametrize("B", [1, 2, 5, 16])
@pytest.mark.parametrize("mode", ["host", "device"])
@pytest.mark.parametrize("kd", [False, True])
@pytest.mark.parametrize("cuda_in", [False, True])
def test_equals_the_loop(lattice, objects, B, mode, kd, cuda_in):
    pred = lattice
    pred.subsample, pred.use_kdtree_for_eval = mode, kd
    try:
        datas = objects[:B] if B < 16 else objects[5:] + objects[:5]
        if cuda_in:
            datas = [{k: torch.from_numpy(v).cuda() for k, v in d.items()} for d in datas]
        out = _check_equal_to_loop(pred, datas)
        if cuda_in:
            assert all(r[1] is None or (r[1].is_cuda and r[0].is_cuda) for r in out)
        else:
            assert all(r[1] is None or isinstance(r[1], np.ndarray) for r in out)
    finally:
        pred.subsample, pred.use_kdtree_for_eval = "host", False


def test_given_ids_equal_the_loop(lattice, objects):
    rng = np.random.RandomState(4)
    datas = objects[:4]
    ids = [None if b % 2 else rng.randint(0, int((d["cloud_xyz"][:, 2] >= 0.1).sum()), 512).astype(np.int64)
           for b, d in enumerate(datas)]
    for mode in ("host", "device"):
        lattice.subsample = mode
        try:
            _check_equal_to_loop(lattice, datas, ids=ids)
        finally:
            lattice.subsample = "host"


def _collinear(n=700):
    t = np.linspace(0.0, 1.0, n)
    xyz = np.stack([0.03 * t, np.zeros(n), np.full(n, 0.7)], 1)
    nrm = np.tile([0.0, 0.0, -1.0], (n, 1))
    return {"cloud_xyz": xyz, "cloud_normal": nrm}


@pytest.mark.parametrize("mode", ["host", "device"])
def test_failure_slots(lattice, objects, mode):
    lattice.subsample = mode
    try:
        datas = [objects[0], _collinear(), objects[1], _collinear(300), objects[2]]
        out = _check_equal_to_loop(lattice, datas)
        assert out[1] == (None, None) and out[3] == (None, None)
        assert any(r[1] is not None for r in out)
    finally:
        lattice.subsample = "host"


def test_batch_independence_of_the_device_work(lattice, objects):
    """Fixed inputs (no draws): object k's forward outputs and record alone, first and last in a batch of 16."""
    from catgrasp_b200.aligning import ransac9d_pose_many
    pred, n = lattice, 512
    rng = np.random.RandomState(0)
    x = torch.from_numpy(rng.normal(0, 1, (16, n, 6)).astype(np.float32)).cuda()
    src = torch.from_numpy(rng.uniform(-0.5, 0.5, (16, n, 3))).cuda()
    R = np.linalg.qr(rng.normal(size=(3, 3)))[0] * 0.02
    tgt = src @ torch.from_numpy(R).cuda().T + 0.7 + torch.from_numpy(rng.normal(0, 4e-4, (16, n, 3))).cuda()
    ids = torch.from_numpy(rng.randint(0, n, (16, 2 * 2000, 4)).astype(np.int32)).cuda()

    def rec(order):
        o = torch.tensor(order).cuda()
        return ransac9d_pose_many(src[o], tgt[o], ids[o], pred.THRESHOLDS, max_scale=[0.05] * 3,
                                  min_scale=[0.005] * 3, max_dimensions=[1.2] * 3).cpu().numpy()

    def fwd(order):
        o = torch.tensor(order).cuda()
        return [t.cpu().numpy() for t in pred.model.nunocs_many_dev(x[o].contiguous(), 100)]

    others = [k for k in range(16) if k != 3]
    for got_rec, got_fwd, row in ((rec([3]), fwd([3]), 0), (rec([3] + others[:15]), fwd([3] + others[:15]), 0),
                                  (rec(others[:15] + [3]), fwd(others[:15] + [3]), 15)):
        assert got_rec[row].tobytes() == rec([3])[0].tobytes()
        for a, b in zip(got_fwd, fwd([3])):
            assert a[row].tobytes() == b[0].tobytes()
    assert (rec(list(range(16)))[:, 2 * 19] >= 0).any()        # some object has a pose


def _golden_predicter(g, tmp, sd):
    from catgrasp_b200.predicter import NunocsPredicter
    from catgrasp_b200.synthetic import write_artifacts
    d = write_artifacts(str(tmp), "seg", n_pts=8192, state_dict=sd, normalizer=(g["mean"], g["std"]))
    return NunocsPredicter("nut", artifact_dir=d, device=0)


def test_reference_numbers_inside_a_batch(cuda, golden_dir, objects, tmp_path):
    from catgrasp_b200.synthetic import make_lattice_seg_state_dict, make_state_dict
    gl = np.load(os.path.join(golden_dir, "host_nunocs_lattice.npz"))
    gr = np.load(os.path.join(golden_dir, "host_nunocs_random.npz"))
    pl = _golden_predicter(gl, tmp_path / "l", make_lattice_seg_state_dict(seed=int(gl["weight_seed"]), mean=gl["mean"],
                                                                           std=gl["std"]))
    pr = _golden_predicter(gr, tmp_path / "r", make_state_dict("seg", 300, seed=int(gr["weight_seed"])))
    lat = {"cloud_xyz": gl["cloud_xyz"], "cloud_normal": gl["cloud_normal"].astype(np.float64)}
    ran = {"cloud_xyz": gr["cloud_xyz"].astype(np.float64), "cloud_normal": gr["cloud_normal"].astype(np.float64)}
    # alone: the recorded state afterwards; first of a batch: the recorded results (its draws come first)
    for batch in ([lat], [lat, objects[0], ran, objects[1]]):
        np.random.seed(0)
        out = pl.predict_many(batch)
        if len(batch) == 1:
            np.testing.assert_array_equal(np.random.rand(2), gl["next_rand"])
            assert pl.best_ratio == float(gl["best_ratio"])
            np.testing.assert_array_equal(pl.pred_bins.reshape(-1, 3), gl["nocs_bins"])
        nocs, tf = out[0]
        np.testing.assert_array_equal(np.asarray(nocs, np.float32), gl["nocs_cloud"])
        np.testing.assert_allclose(tf, gl["transform"], rtol=0, atol=1e-9)
    for batch in ([ran], [ran, objects[2], lat]):
        np.random.seed(0)
        out = pr.predict_many(batch)
        assert bool(gr["returned_none"]) and out[0] == (None, None)
        if len(batch) == 1:
            np.testing.assert_array_equal(np.random.rand(2), gr["next_rand"])
            np.testing.assert_array_equal(pr.data_transformed["keep_ids"], gr["keep_ids"])
            np.testing.assert_array_equal(pr.data_transformed["input"].astype(np.float32), gr["input"])


def test_chunking_gives_the_bits_of_short_batches(cuda, objects, tmp_path):
    """n_pts 1024: CG_NUNOCS_MANY_PASS_POINTS = 2^18 makes forward passes of 256 objects, and 2 x 10 000 hypotheses
    make pose-search launches of 52 objects (CG_RANSAC_MANY_PASS_PAIRS = 2^20); 260 objects need both to split.
    Batches of 50 run each in one pass."""
    from catgrasp_b200.synthetic import make_lattice_seg_state_dict
    pred = _predicter(tmp_path, 1024, make_lattice_seg_state_dict(seed=5), normalizer=False)
    pred.subsample = "device"
    datas = [objects[b % 16] for b in range(260)]
    np.random.seed(3)
    whole = pred.predict_many(datas)
    st_whole = np.random.get_state()[1].copy()
    np.random.seed(3)
    parts = []
    for b0 in range(0, 260, 50):
        parts += pred.predict_many(datas[b0:b0 + 50])
    assert np.array_equal(np.random.get_state()[1], st_whole)
    assert sum(r[1] is not None for r in whole) > 0
    for b, (w, p) in enumerate(zip(whole, parts)):
        _eq(w[0], p[0], f"nocs[{b}]")
        _eq(w[1], p[1], f"pose[{b}]")


@pytest.mark.parametrize("engine", ENGINES)
def test_batched_forward_equals_single_on_every_engine(lattice, engine):
    """B = 11 > 8: the per-cloud FC layers run in two groups; each object's outputs are its B = 1 forward's."""
    net = lattice.model
    keep = net.ctx.get_engine()
    rng = np.random.RandomState(engine)
    x = rng.normal(0, 1, (11, 512, 6)).astype(np.float32)
    try:
        net.ctx.set_engine(engine)
        many = net.nunocs_many_host(x, 100)
        many_dev = [t.cpu().numpy() for t in net.nunocs_many_dev(torch.from_numpy(x).cuda(), 100)]
        for b in range(11):
            one = net.nunocs_host(x[b], 100)
            for k in range(3):
                assert many[k][b].tobytes() == one[k].tobytes(), (engine, b, k)
                assert many_dev[k][b].tobytes() == one[k].tobytes(), (engine, b, k)
    finally:
        net.ctx.set_engine(keep)
