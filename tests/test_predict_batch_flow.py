"""GraspPredicter.score on a shard of the candidate list: the shard's rows of the full call, bit for bit, with numpy's
global generator left where the full call leaves it, and predict_batch as the host-side view of the same numbers."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# A launch's batch size selects the FC kernel (up to 8 rows, up to 63, tensor cores beyond), and only launches of one
# class agree bit for bit: every launch here, of a shard, a chunk or the whole list, scores at most 8 candidates.
B, N_PTS, CHUNK = 8, 256, 3
SHARDS = ((0, 0), (3, 3), (B, B), (2, 7), (0, B))


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def predicter(cuda, tmp_path_factory):
    from catgrasp_b200.predicter import GraspPredicter
    from catgrasp_b200.synthetic import write_artifacts
    adir = write_artifacts(str(tmp_path_factory.mktemp("flow") / "artifacts-47"), "cls", n_pts=N_PTS, seed=0)
    gp = GraspPredicter("nut", artifact_dir=adir)
    gp.chunk = CHUNK                          # the host draw of the full list runs in chunks of 3, 3 and 2
    return gp


def _scene(points):
    """(data, poses): a pile of 1500 points, cut to its first ``points`` valid ones (fewer than N_PTS: the draw is with
    replacement and walks numpy's stream differently)."""
    from catgrasp_b200.synthetic import make_candidates, make_pile
    scene = make_pile(1500, n_objects=3, seed=9)
    keep = np.nonzero(scene["cloud_xyz"][:, 2] >= 0.1)[0][:points]
    data = {"cloud_xyz": scene["cloud_xyz"][keep], "cloud_normal": scene["cloud_normal"][keep]}
    return data, list(make_candidates(data["cloud_xyz"], data["cloud_normal"], B, seed=10))


def _check_shards(gp, data, poses, **kw):
    np.random.seed(7)
    full = gp.score(data, poses, **kw)
    after = np.random.rand(2)
    assert full.is_cuda and full.dtype == torch.float32 and full.shape == (B, gp.model.n_out)
    for lo, hi in SHARDS:
        np.random.seed(7)
        part = gp.score(data, poses, shard=(lo, hi), **kw)
        assert np.array_equal(np.random.rand(2), after), (lo, hi)
        assert part.is_cuda and part.dtype == torch.float32 and part.shape == (hi - lo, gp.model.n_out), (lo, hi)
        assert torch.equal(part, full[lo:hi]), (lo, hi)
    return full, after


@pytest.mark.parametrize("points", (1200, 200))
@pytest.mark.parametrize("mode", ("host", "device"))
def test_score_shard_is_rows_of_full_call_on_the_same_stream(predicter, mode, points):
    data, poses = _scene(points)
    full, after = _check_shards(predicter, data, poses, subsample=mode)
    np.random.seed(7)
    out = predicter.predict_batch(data, poses, subsample=mode)     # the same call, as the reference's result list
    assert np.array_equal(np.random.rand(2), after)
    probs = full.cpu().numpy()
    assert len(out) == B and all(len(o) == 3 for o in out)
    assert all(np.array_equal(o[2], p) for o, p in zip(out, probs))
    assert all(o[0] == p.argmax() and o[1] == p[o[0]] for o, p in zip(out, probs))
    assert all(o[0].dtype == np.int64 and o[1].dtype == np.float32 and o[2].dtype == np.float32 for o in out)


def test_score_shard_with_given_ids_leaves_numpy_alone(predicter):
    data, poses = _scene(1200)
    ids = np.random.RandomState(12).randint(0, 1200, (B, N_PTS)).astype(np.int32)
    _, after = _check_shards(predicter, data, poses, ids=ids)
    np.random.seed(7)
    assert np.array_equal(np.random.rand(2), after)


def test_an_empty_candidate_list_gives_an_empty_list(predicter):
    data, _ = _scene(1200)
    np.random.seed(7)
    after = np.random.rand(2)
    for mode in ("host", "device"):
        np.random.seed(7)
        assert predicter.predict_batch(data, [], subsample=mode) == []
        assert np.array_equal(np.random.rand(2), after)
