"""CPU: NunocsPredicter.predict_many's host logic, which needs no device.

- The whole list is checked before any random number is drawn: every rejected call leaves numpy's generator as it
  was, including when the failing object comes after valid ones, and so does a rejected one-object predict.
- draw_nunocs_many (the host-mode draws of B objects in one walk of numpy's generator) equals the loop's draws, word for
  word: per object draw_subsample_ids' np.random.choice, then a _LegacyDraw of 2H RANSAC 4-subsets, and the same state
  afterwards.
"""
import numpy as np
import pytest

from catgrasp_b200 import _lib
from catgrasp_b200.predicter import NunocsPredicter, _LegacyDraw, draw_nunocs_many, draw_subsample_ids


def _predicter(n_pts=64, subsample="host"):
    """A NunocsPredicter without a network: predict_many's checks run before anything touches the model."""
    p = object.__new__(NunocsPredicter)
    p.cfg = {"n_pts": n_pts, "ce_loss_bins": 100}
    p.ransac_max_iter = 10
    p.subsample = subsample
    p.use_kdtree_for_eval = False
    p.kdtree_eval_resolution = 0.003
    return p


def _obj(M, seed, z=0.7):
    rng = np.random.RandomState(seed)
    xyz = rng.uniform(-0.02, 0.02, (M, 3))
    xyz[:, 2] += z
    nrm = rng.normal(size=(M, 3))
    return {"cloud_xyz": xyz, "cloud_normal": nrm / np.linalg.norm(nrm, axis=1, keepdims=True)}


def _state():
    s = np.random.get_state()
    return s[0], s[1].copy(), s[2], s[3], s[4]


def _same(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def _rejects(p, datas, match, ids=None, one=False):
    """predict_many(datas) raises, or with ``one`` predict on the one object, and draws nothing."""
    np.random.seed(11)
    before = _state()
    with pytest.raises(ValueError, match=match):
        if one:
            p.predict(datas[0], ids=None if ids is None else ids[0])
        else:
            p.predict_many(datas, ids=ids)
    assert _same(before, _state())


@pytest.mark.parametrize("mode", ["host", "device"])
def test_empty_masked_cloud_is_rejected_before_any_draw(mode):
    p = _predicter(subsample=mode)
    far = _obj(50, 2, z=0.05)                      # every point below z = 0.1: predict's np.random.choice raises
    _rejects(p, [_obj(100, 1), _obj(30, 3), far], "cannot be empty unless no samples are taken")
    _rejects(p, [far], "cannot be empty")
    _rejects(p, [far], "cannot be empty", one=True)


def test_malformed_and_mixed_inputs_are_rejected_before_any_draw():
    p = _predicter()
    good = _obj(100, 1)
    _rejects(p, [good, {"cloud_xyz": good["cloud_xyz"]}], "cloud_normal")
    _rejects(p, [good, "not a dict"], "not a dict")
    _rejects(p, [good, {"cloud_xyz": good["cloud_xyz"], "cloud_normal": good["cloud_normal"][:5]}], r"\(M,3\)")
    _rejects(p, [good, {"cloud_xyz": good["cloud_xyz"][:, :2], "cloud_normal": good["cloud_normal"][:, :2]}],
             r"\(M,3\)")
    _rejects(p, [good, {"cloud_xyz": good["cloud_xyz"].tolist(), "cloud_normal": good["cloud_normal"]}],
             "all numpy arrays or all CUDA tensors|\\(M,3\\)")
    _rejects(p, [good, good], "2 objects", ids=[None])
    _rejects(p, [good], "ids\\[0\\] has shape", ids=[np.arange(10)])
    _rejects(p, [good, good], "indexes outside", ids=[None, np.arange(64) + 40])
    _rejects(p, [good, good], "indexes outside", ids=[np.arange(64) - 1, None])
    _rejects(p, [good], "ids\\[0\\] has shape", ids=[np.arange(10)], one=True)
    _rejects(p, [good], "indexes outside", ids=[np.arange(64) + 40], one=True)


def test_bad_kdtree_resolution_is_rejected_before_any_draw():
    p = _predicter()
    p.use_kdtree_for_eval = True
    p.kdtree_eval_resolution = -1.0
    _rejects(p, [_obj(100, 1)], "kdtree_eval_resolution")


def test_too_few_points_per_object_is_rejected_before_any_draw():
    _rejects(_predicter(n_pts=3), [_obj(100, 1)], "larger sample than population")
    _rejects(_predicter(n_pts=3), [_obj(100, 1)], "larger sample than population", one=True)


def test_empty_list_draws_nothing():
    np.random.seed(5)
    before = _state()
    assert _predicter().predict_many([]) == []
    assert _same(before, _state())


def _host_rng_or_skip():
    try:
        _lib.load()
    except (_lib.CgError, OSError) as e:
        pytest.skip(f"host RNG library not loadable: {e}")


@pytest.mark.parametrize("given", [False, True])
def test_batched_host_draw_equals_the_loop(given):
    """Counts below, at and above n_pts (with and without replacement), one M of 1 (randint with rng 0 consumes
    nothing), and with ``given`` some objects whose subset is passed in (not drawn)."""
    _host_rng_or_skip()
    n_pts, n_hyp = 64, 2 * 37
    Ms = [10, 64, 500, 1, 65, 3000]
    ids = [None, np.arange(n_pts), None, None, np.arange(n_pts), None] if given else None
    np.random.seed(1234)
    want_sub, want_hyp = [], []
    for b, M in enumerate(Ms):
        want_sub.append(draw_subsample_ids(M, n_pts) if ids is None or ids[b] is None else None)
        d = _LegacyDraw()
        want_hyp.append(d.draw(n_pts, 4, n_hyp))
        d.commit()
    want_state = _state()
    np.random.seed(1234)
    subs, hyp = draw_nunocs_many(Ms, n_pts, n_hyp, given=ids)
    assert _same(want_state, _state())
    assert hyp.dtype == np.int32 and hyp.shape == (len(Ms), n_hyp, 4)
    for b in range(len(Ms)):
        if want_sub[b] is None:
            assert subs[b] is None
        else:
            assert subs[b].tobytes() == want_sub[b].astype(np.int32).tobytes(), b
        assert hyp[b].tobytes() == want_hyp[b].tobytes(), b
