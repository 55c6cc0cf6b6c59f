"""The per-pick control stages without a GPU: oracle/pick_ref.py against tests/golden/pick_control.npz (the
reference's own compute_candidate_grasp with fixed collaborators, see make_golden_pick.py), and the summation order
the ranking kernel restates against numpy's own sum."""
import os

import numpy as np
import pytest

from oracle import pick_ref

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "pick_control.npz"))
SCENES = ("mixed", "equal", "none")


@pytest.mark.parametrize("name", SCENES)
def test_segment_stage_matches_golden(name):
    t = pick_ref.segment_table(G[f"{name}_labels"], G[f"{name}_cloud_xyz"])
    assert t["order"] == G[f"{name}_visits"].tolist()
    for k, idx in enumerate(t["indices"]):
        assert np.array_equal(G[f"{name}_cloud_xyz"][idx], G[f"{name}_ob_pts_{k}"])
    # one colour draw per inlier segment, then nothing until the first object
    np.random.seed(int(G["seed"]))
    for _ in t["inlier_ids"]:
        np.random.randint(0, 255, size=(3))
    st = np.random.get_state()
    assert np.array_equal(st[1], G[f"{name}_rng_key"]) and st[2] == int(G[f"{name}_rng_pos"])


def test_golden_covers_the_branches():
    t = pick_ref.segment_table(G["mixed_labels"], G["mixed_cloud_xyz"])
    small = t["count"] < 500
    assert small.sum() >= 2 and not t["inlier"][small].any()
    assert ((~small) & ~t["inlier"]).any()                                         # low density
    ext = t["max"] - t["min"]
    assert any(t["inlier"][l] and (ext[l] == 0).any() for l in range(len(ext)))    # zero extent, inlier
    counts = [t["count"][l] for l in t["order"]]
    assert len(set(counts)) < len(counts)                                           # equal counts
    assert G["none_visits"].size == 0 and int(G["none_n_yield"]) == 0


@pytest.mark.parametrize("name", ("mixed", "equal"))
def test_ranking_matches_golden(name):
    n_classes = int(G["n_classes"])
    for k in range(int(G[f"{name}_n_yield"])):
        p_G, p_T_G, perm = pick_ref.rank_grasps(G[f"{name}_probs_{k}"], G[f"{name}_p_T_given_G_{k}"], n_classes)
        assert np.array_equal(perm, G[f"{name}_order_{k}"])
        assert np.array_equal(p_G[perm].view(np.uint64), G[f"{name}_p_G_{k}"].view(np.uint64))
        assert np.array_equal(p_T_G[perm].view(np.uint64), G[f"{name}_p_T_G_{k}"].view(np.uint64))


def pairwise_restated(a):
    """The order cg_pick.cu's rank kernel sums in (numpy's pairwise_sum for n <= 128)."""
    n = len(a)
    if n < 8:
        r = 0.0
        for v in a:
            r += v
        return r
    r = list(a[:8])
    i = 8
    while i < n - n % 8:
        for j in range(8):
            r[j] += a[i + j]
        i += 8
    res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    for v in a[i:]:
        res += v
    return res


@pytest.mark.parametrize("C", [3, 7, 8, 10, 17, 64, 128])
def test_summation_order_is_numpys(C):
    rng = np.random.RandomState(C)
    z = rng.normal(0, 30, (4000, C))
    e = np.exp(z - z.max(1, keepdims=True))
    probs = (e / e.sum(1, keepdims=True)).astype(np.float32)
    seq_differs = 0
    for row in probs:
        a = row * np.arange(C)
        assert pairwise_restated(a) == a.sum()
        s = 0.0
        for v in a:
            s += v
        seq_differs += s != a.sum()
    if C >= 8:
        assert seq_differs > 0          # the rows are wide enough to tell the orders apart
