"""The iiwa14 IK kernel (csrc/cg_ik.cu) against its numpy twin (oracle/ik_ref.py) and the reference's ikfast
solver as pinned in tests/golden/ik_iiwa14.npz, and filterGraspPose's built-in IK test against the reference build's
survivors and counters."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

from make_golden_ik import IK_LOWER, IK_UPPER, TIGHT_LOWER, TIGHT_UPPER, digest, filter_case, inputs  # noqa: E402
from make_golden_mycpp import IK_CASES, filter_inputs, ik_frames  # noqa: E402
from oracle import ik_ref, mycpp_ref  # noqa: E402

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(HERE, "golden", "ik_iiwa14.npz"))


@pytest.fixture(scope="module")
def poses():
    P, fam, _ = inputs()
    return P, fam, ik_ref.in_band(P)


def _angles_close(a, b, tol):
    d = np.abs(np.angle(np.exp(1j * (a - b))))
    return np.where(np.isnan(a) & np.isnan(b), True, d <= tol)


def test_kernel_equals_twin(poses):
    from catgrasp_b200.ik import iiwa14_ik
    P, _, band = poses
    cnt, sol = iiwa14_ik(P, IK_UPPER, IK_LOWER, solutions=True)
    rc, rsol = ik_ref.iiwa14_ik(P, IK_UPPER, IK_LOWER)
    assert cnt.dtype == np.int8 and sol.shape == (len(P), 8, 7)
    assert (np.isnan(sol) == np.isnan(rsol)).all()
    assert _angles_close(sol, rsol, 1e-12)[~band].all()
    assert _angles_close(sol, rsol, 1e-9).all()
    assert (cnt[~band] == rc[~band]).all()


def test_kernel_matches_ikfast_outside_bands(poses):
    from catgrasp_b200.ik import iiwa14_ik
    P, _, band = poses
    ca = iiwa14_ik(torch.from_numpy(P).cuda(), IK_UPPER, IK_LOWER).cpu().numpy()
    cb = iiwa14_ik(P, TIGHT_UPPER, TIGHT_LOWER)
    assert (ca[~band] == GOLD["count_a"][~band]).all()
    assert (cb[~band] == GOLD["count_b"][~band]).all()
    _, sol = iiwa14_ik(P, IK_UPPER, IK_LOWER, solutions=True)
    assert ((~np.isnan(sol[:, :, 0])).sum(axis=1) == GOLD["nsol"])[~band].all()


def test_kernel_edge_cases():
    from catgrasp_b200.ik import iiwa14_ik
    empty = iiwa14_ik(np.zeros((0, 4, 4), np.float32), IK_UPPER, IK_LOWER, solutions=True)
    assert empty[0].shape == (0,) and empty[1].shape == (0, 8, 7)
    q = np.random.RandomState(5).uniform(-1.5, 1.5, (333, 7))
    q[:, 2] = 0
    P = ik_ref.iiwa14_fk(q).astype(np.float32)            # 333: not a multiple of the block size
    P[7, 0, 3] = np.nan
    P[8, 2, 2] = np.inf
    P[9, 1, 0] = -np.inf
    cnt, sol = iiwa14_ik(P, IK_UPPER, IK_LOWER, solutions=True)
    rc, _ = ik_ref.iiwa14_ik(P, IK_UPPER, IK_LOWER)
    assert (cnt[7:10] == 0).all() and np.isnan(sol[7:10]).all()
    assert (cnt == rc).all()
    assert (iiwa14_ik(P, IK_UPPER, IK_LOWER) == cnt).all()              # no solution buffer
    assert (iiwa14_ik(P, IK_LOWER, IK_UPPER) == 0).all()                # lower > upper
    with pytest.raises(ValueError):
        iiwa14_ik(P, IK_UPPER[:6], IK_LOWER[:6])


def _sdfs(g):
    from catgrasp_b200.sdf import Sdf3D
    return (Sdf3D(g["open"]["sdf"], g["open"]["origin"], g["open"]["res"], device=0),
            Sdf3D(g["enclosed"]["sdf"], g["enclosed"]["origin"], g["enclosed"]["res"], device=0))


def _run_filter(grasps, sym, nocs, c2n, g, p1, p2, cam, ee, fdir, adjust, mode, verbose, as_tensor):
    from catgrasp_b200 import my_cpp
    so, se = _sdfs(g)
    my_cpp.register_gripper_sdf(g["open"]["V"], g["open"]["F"], so)
    my_cpp.register_gripper_sdf(g["enclosed"]["V"], g["enclosed"]["F"], se)
    old = my_cpp.DEFAULT_SDF_MODE
    my_cpp.DEFAULT_SDF_MODE = mode
    try:
        gp = torch.as_tensor(np.asarray(grasps, np.float64)).cuda() if as_tensor else grasps
        return my_cpp.filterGraspPose(gp, sym, nocs, c2n, cam, ee, g["gripper_in_grasp"], fdir, True, adjust,
                                      list(IK_UPPER), list(IK_LOWER), g["open"]["V"], g["open"]["F"], g["enclosed"]["V"],
                                      g["enclosed"]["F"], p1, p2, 0.0005, verbose)
    finally:
        my_cpp.DEFAULT_SDF_MODE = old


@pytest.mark.parametrize("as_tensor", [False, True])
@pytest.mark.parametrize("k", range(len(IK_CASES)))
def test_filterGraspPose_builtin_ik_equals_reference(k, as_tensor):
    from catgrasp_b200 import my_cpp
    my_cpp.set_ik_solver(None)
    S, scale, mode, adjust, fdir = IK_CASES[k]
    (p1, p2, P, sym, nocs, c2n, g), dg = filter_inputs(S, scale)
    cam, ee = ik_frames()
    gold = np.load(os.path.join(HERE, "golden", "mycpp_filter.npz"))
    assert (digest(dg, cam, ee, IK_UPPER, IK_LOWER) == gold[f"ik_inputs_sha_{k}"]).all()
    out = _run_filter(P, sym, nocs, c2n, g, p1, p2, cam, ee, fdir, adjust, mode, False, as_tensor)
    got = mycpp_ref.sort_poses(np.array(out).reshape(-1, 4, 4)).view(np.uint32)
    assert got.shape == gold[f"ik_survivors_{k}"].shape and (got == gold[f"ik_survivors_{k}"]).all()


@pytest.mark.parametrize("k", range(len(IK_CASES)))
def test_ik_counts_on_filter_survivors(k):
    from catgrasp_b200.ik import iiwa14_ik
    from catgrasp_b200.my_cpp import _mm4_f32, grasp_in_cam_unshifted
    from oracle import filter_ref
    S, scale, mode, adjust, fdir = IK_CASES[k]
    (p1, p2, P, sym, nocs, c2n, g), _ = filter_inputs(S, scale)
    cam, ee = ik_frames()
    st, _, _ = filter_ref.filter_ref(P, sym, nocs, c2n, g["gripper_in_grasp"], fdir, adjust, mode, g["open"], p1,
                                     g["enclosed"], p2)
    u = grasp_in_cam_unshifted(P, sym, nocs, c2n)
    f = lambda m: np.asarray(m, np.float64).astype(np.float32)      # noqa: E731
    eb = np.array([_mm4_f32(_mm4_f32(f(cam), u[q]), f(ee)) for q in np.nonzero(st == 0)[0]])
    runs = np.load(os.path.join(HERE, "golden", "mycpp_ref_runs.npz"))
    assert (iiwa14_ik(eb, IK_UPPER, IK_LOWER).astype(np.int64) == runs[f"ik_counts_{k}"]).all()


def test_filter_case_survivors_and_counters(capsys):
    from catgrasp_b200 import my_cpp
    my_cpp.set_ik_solver(None)
    c = filter_case()
    assert (digest(c["grasps"], c["p1"], c["p2"], c["cam"], c["ee"]) == GOLD["filter_sha"]).all()
    capsys.readouterr()
    out = _run_filter(c["grasps"], c["sym"], c["nocs_pose"], c["c2n"], c["g"], c["p1"], c["p2"], c["cam"], c["ee"],
                      False, False, 0, True, False)
    txt = capsys.readouterr().out
    got = mycpp_ref.sort_poses(np.array(out).reshape(-1, 4, 4)).view(np.uint32)
    assert got.shape == GOLD["filter_survivors"].shape and (got == GOLD["filter_survivors"]).all()
    a, i, o, e, n = GOLD["filter_counters"]
    assert f"n_approach_dir_rej={a}, n_ik_rej={i}, n_open_gripper_rej={o}, n_close_gripper_rej={e}" in txt, txt
    assert len(out) == n


def test_device_route_equals_hook_route():
    """filter_grasp_pose_raw(..., ik=...) on CUDA tensors gives the per-pair status of the host-hook route with the
    reference's ikfast (or, without the oracle build, its restatement) as the hook."""
    from catgrasp_b200 import _lib, my_cpp
    from catgrasp_b200.my_cpp import _mm4_f32, grasp_in_cam_unshifted
    try:
        from oracle import mycpp_ref_ik
        hook = (lambda T, up, lo: len(mycpp_ref_ik.ik_within_limits(T, up, lo)) > 0) if mycpp_ref_ik.available() else None
    except Exception:
        hook = None
    if hook is None:
        hook = lambda T, up, lo: ik_ref.iiwa14_ik(T[None], up, lo)[0][0] > 0      # noqa: E731
    c = filter_case()
    so, se = _sdfs(c["g"])
    args = (c["grasps"], c["sym"], c["nocs_pose"], c["c2n"], c["gripper_in_grasp"], False, False, so, c["p1"], se, c["p2"])
    st0, _, _ = my_cpp.filter_grasp_pose_raw(*args, split_status=True)
    gp = torch.as_tensor(c["grasps"]).cuda()
    st, off, po = my_cpp.filter_grasp_pose_raw(gp, *args[1:], split_status=True,
                                               ik=(c["cam"], c["ee"], IK_UPPER, IK_LOWER))
    st, off, po = st.cpu().numpy(), off.cpu().numpy(), po.cpu().numpy()
    u = grasp_in_cam_unshifted(c["grasps"], c["sym"], c["nocs_pose"], c["c2n"])
    f = lambda m: np.asarray(m, np.float64).astype(np.float32)      # noqa: E731
    want = st0.copy()
    for q in np.nonzero(st0 != _lib.CG_ST_REJ_DIR)[0]:
        if not hook(_mm4_f32(_mm4_f32(f(c["cam"]), u[q]), f(c["ee"])), IK_UPPER, IK_LOWER):
            want[q] = _lib.CG_ST_REJ_IK
    assert (st == want).all()
    rej = st == _lib.CG_ST_REJ_IK
    assert rej.any() and (off[rej] == -1).all() and (po[rej] == 0).all()
