"""CPU: cg_host_legacy_choice for small subsets (n_pts <= 16, the slot-following path of csrc/cg_host_rng.cpp) against
numpy's own ``np.random.choice(M, n_pts, replace=False)``, one call per draw: the same indices and the generator left
in the same state, on every instruction-set level and thread count; and the sequence one host-mode
NunocsPredicter.predict makes.  Also the device draw's keying of NunocsPredicter's device mode, restated by
oracle/draw_ref.py."""
import numpy as np
import pytest

from catgrasp_b200 import _lib
from catgrasp_b200.predicter import _LegacyDraw


def _state():
    st = np.random.get_state()
    return st[1].copy(), st[2], st[3], st[4]


def _same_state(a, b):
    return np.array_equal(a[0], b[0]) and a[1:] == b[1:]


def _numpy_draws(M, n_pts, count):
    out = np.empty((count, n_pts), np.int32)
    for c in range(count):
        out[c] = np.random.choice(M, size=n_pts, replace=False)
    return out


@pytest.mark.parametrize("n_pts", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("isa", [-1, 0])
def test_small_subsets_equal_numpy(n_pts, isa):
    lib = _lib.load()
    try:
        lib.cg_host_rng_isa(isa)
        for M in sorted({n_pts, n_pts + 1, 2047, 2048, 2049, 8192, 65537}):
            for count in (0, 1, 7, 2000):
                if M == 65537 and count == 2000:
                    count = 150                               # numpy's own draw is the slow side here
                for nthreads in (1, 0):
                    np.random.seed(M * 31 + n_pts + count)
                    np.random.randn(1)                        # a cached gaussian in the state tuple
                    ref = _numpy_draws(M, n_pts, count)
                    ref_state = _state()
                    np.random.seed(M * 31 + n_pts + count)
                    np.random.randn(1)
                    d = _LegacyDraw()
                    got = d.draw(M, n_pts, count, nthreads=nthreads)
                    d.commit()
                    assert np.array_equal(got, ref), (M, n_pts, count, nthreads)
                    assert _same_state(_state(), ref_state), (M, n_pts, count, nthreads)
    finally:
        lib.cg_host_rng_isa(-1)


@pytest.mark.parametrize("isa", [-1, 0])
def test_host_predict_sequence(isa):
    """What host-mode predict draws: the 8192-of-M cloud subset (np.random.choice(np.arange(M), 8192)), then the two
    thresholds' 10 000 subsets of 4 of 8192 each, as one C call that continues where the reference's loops would."""
    lib = _lib.load()
    try:
        lib.cg_host_rng_isa(isa)
        M, n, H = 12000, 8192, 10000
        np.random.seed(11)
        ref_sub = np.random.choice(np.arange(M), size=n, replace=M < n)
        ref = _numpy_draws(n, 4, 2 * H)
        ref_next = np.random.rand(3)
        np.random.seed(11)
        d = _LegacyDraw()
        sub = d.draw(M, n, 1, nthreads=1)[0]
        got = d.draw(n, 4, 2 * H)
        d.commit()
        assert np.array_equal(sub, ref_sub) and np.array_equal(got, ref)
        assert np.array_equal(np.random.rand(3), ref_next)
    finally:
        lib.cg_host_rng_isa(-1)


def test_device_mode_keying():
    """Device mode draws candidate 0 = the cloud subset and candidates 1 .. 2H = the hypotheses (1 + h for the first
    threshold, 1 + H + h for the second) from one seed; a hypothesis's four indices are distinct."""
    from oracle.draw_ref import draw_ids
    seed, M, n, H = 0x1234_5678_9abc_def0, 9000, 8192, 10000
    both = draw_ids(n, 4, 2 * H, seed, first_candidate=1)
    assert np.array_equal(both[:H], draw_ids(n, 4, H, seed, first_candidate=1))
    assert np.array_equal(both[H:], draw_ids(n, 4, H, seed, first_candidate=1 + H))
    assert ((both >= 0) & (both < n)).all()
    s = np.sort(both, axis=1)
    assert (s[:, 1:] != s[:, :-1]).all()
    sub = draw_ids(M, n, 1, seed, first_candidate=0)[0]
    assert len(np.unique(sub)) == n and sub.min() >= 0 and sub.max() < M
