"""The several-frame pick's argument refusals (CPU only): compute_candidate_grasp_many, segment_table_many and
estimate_normals_many refuse a bad frame list or bad offsets with ValueError before any device work."""
import numpy as np
import pytest
import torch

from catgrasp_b200 import cloud, pick

K = np.array([[600.0, 0, 31.5], [0, 600.0, 23.5], [0, 0, 1]])


def _many(depths, Ks, masks, envs):
    return pick.compute_candidate_grasp_many(depths, Ks, masks, envs, None, None, None, {}, {}, [np.eye(4)], {})


def test_pick_many_refuses_bad_frame_lists():
    d, m = np.ones((48, 64), np.float32), np.zeros((48, 64), bool)
    with pytest.raises(ValueError, match="no frames"):
        _many([], [], [], [])
    with pytest.raises(ValueError, match="2 depths, 1 Ks"):
        _many([d, d], [K], [m, m], [{}, {}])
    with pytest.raises(ValueError, match="envs"):
        _many([d], [K], [m], [])
    with pytest.raises(ValueError, match="frame 1"):
        _many([d, d], [K, K], [m, m[:, :10]], [{}, {}])
    with pytest.raises(ValueError, match="frame 0"):
        _many([d[0]], [K], [m[0]], [{}])
    with pytest.raises(ValueError, match="frame 0"):
        _many([d], [K[:2]], [m], [{}])


def test_pick_one_frame_refuses_at_its_first_next():
    """compute_candidate_grasp stays a generator: nothing is checked or run before its first next()."""
    g = pick.compute_candidate_grasp(np.ones((4, 4)), K, np.zeros((3, 3)), None, None, None, {}, {}, {}, [], {})
    with pytest.raises(ValueError, match="mask of its shape"):
        next(g)


def test_segment_table_many_refuses_bad_offsets():
    lab, x = torch.zeros(10, dtype=torch.int64), torch.zeros(10, 3)
    for off, nl in (([0, 4, 9], [1, 1]), ([0, 6, 4, 10], [1, 1, 1]), ([0, 10], [1, 1]), ([1, 10], [1]),
                    ([0, 10], [0]), ([0], [])):
        with pytest.raises(ValueError, match="segment_table_many"):
            pick.segment_table_many(lab, x, off, nl)
    with pytest.raises(ValueError, match="CUDA"):
        pick.segment_table_many(lab, x, [0, 10], [1])      # well-formed, but not on the device
    with pytest.raises(ValueError, match="int32 / int64"):
        pick.segment_table_many(lab.float(), x, [0, 10], [1])


def test_estimate_normals_many_refuses_bad_offsets():
    p = np.zeros((10, 3))
    for off in ([0, 4, 9], [0, 6, 4, 10], [0], [1, 10]):
        with pytest.raises(ValueError, match="estimate_normals_many"):
            cloud.estimate_normals_many(p, off, 0.002, 30)
