"""GPU (-m gpu): the collision filter kernel (csrc/cg_collide.cu) point by point, on both of its scan paths.

Every launch is compared bit for bit with oracle/filter_ref.c (status, offset, poses as uint32) and, where the
geometry is built for it, with a closed-form expectation.  Three settings run each case:
  padded   -- the gripper proxy with 5 cells of positive padding: trilinear lookups through the hit queue;
  cropped  -- the proxy cropped one cell inside the gripper's bounding box: boundary cells inside the palm and fingers
              are negative, so the plain trilinear scan runs and clamped lookups of points outside the grid can hit;
  nearest  -- the padded proxy with nearest-cell lookups (out-of-grid points are dropped).
Geometry: every group of points sits on one line along its gripper's z axis, 5 cm apart; a point of another group is
then outside the gripper's grid box in z and clamps onto a z face above the fingers or the gap, where sd >= 4 mm in
every setting, so each candidate pose sees only its own group."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

EYE = np.eye(4)
TH = 0.7                                                  # gripper rotation about the camera z axis
R = np.array([[np.cos(TH), -np.sin(TH), 0], [np.sin(TH), np.cos(TH), 0], [0, 0, 1.0]])
BASE = np.array([0.31, -0.17, 0.55])
SPACING = 0.05
FINGER = np.array([0.0225, 0.029, 0.0])                  # centre of finger 1 in the gripper frame
GAP = np.array([0.0225, 0.0, 0.0])                       # centre of the gap between the fingers
SETTINGS = ["padded", "cropped", "nearest"]


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def grids(cuda):
    from catgrasp_b200.sdf import Sdf3D
    from catgrasp_b200.synthetic import make_gripper_proxy
    g = make_gripper_proxy()
    out = {"gig": g["gripper_in_grasp"]}
    for name in ("open", "enclosed"):
        d = g[name]
        c = 6                                              # 5 cells of padding + 1 inside the bounding box
        crop = {"sdf": np.ascontiguousarray(d["sdf"][c:-c, c:-c, c:-c]),
                "origin": (d["origin"].astype(np.float64) + c * float(d["res"])).astype(np.float32), "res": d["res"]}
        assert (crop["sdf"][0] < 0).any() and (crop["sdf"][-1] < 0).any()
        for setting, dd in (("padded", d), ("cropped", crop), ("nearest", d)):
            out[(setting, name)] = (dd, Sdf3D(dd["sdf"], dd["origin"], dd["res"]))
    return out


def _mode(setting):
    return 1 if setting == "nearest" else 0


def _run(grids, setting, poses, p1, p2, adjust=False, split=False, margin=0.0, fdir=False, encl=True, gig=None,
         sdfs=None):
    """kernel vs filter_ref.c, bit for bit; returns (status, offset, poses)."""
    from catgrasp_b200 import my_cpp
    from oracle import filter_ref
    if sdfs is None:
        (do, so), (de, se) = grids[(setting, "open")], grids[(setting, "enclosed")]
    else:
        (do, so), (de, se) = sdfs
    if not encl:
        de, se = None, None
    gig = grids["gig"] if gig is None else gig
    p1 = np.asarray(p1, np.float64).reshape(-1, 3)
    p2 = np.asarray(p2, np.float64).reshape(-1, 3)
    mode = _mode(setting)
    st, off, out = my_cpp.filter_grasp_pose_raw(poses, [EYE], EYE, EYE, gig, fdir, adjust, so, p1, se, p2, sdf_mode=mode,
                                                sdf_margin=margin, split_status=split)
    rst, roff, rout = filter_ref.filter_ref(poses, [EYE], EYE, EYE, gig, fdir, adjust, mode, do, p1, de, p2,
                                            margin=margin, split=split)
    assert np.array_equal(st, rst), np.nonzero(st != rst)[0][:10]
    assert np.array_equal(off, roff)
    assert np.array_equal(out.view(np.uint32), rout.view(np.uint32))
    return st, off, out


def _pose_at(origin, gig):
    """grasp pose whose gripper frame (rotation R) has its origin at ``origin`` (camera frame)"""
    gp = np.eye(4)
    gp[:3, :3] = R
    gp[:3, 3] = origin
    return gp @ np.linalg.inv(gig)


def _line(P):
    return BASE[None] + R[:, 2][None] * (SPACING * (np.arange(P) - P // 2))[:, None]


# ------------------------------------------------------------------ hit position sweep
SWEEP_P = [1, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025, 2047, 2048, 2049, 4095, 4096, 4097, 20000, 40000]


def _sweep_indices(P):
    head = min(P, 1024)
    stride = P // head
    idx = {0, 1, P - 1, P - 2}
    for k in range(1, P // 1024 + 1):                    # 1024-point chunk edges
        idx |= {1024 * k - 1, 1024 * k}
    for j in (1, 2, 511, 512, 1022, 1023):               # strided-head sample edges
        idx |= {j * stride - 1, j * stride, j * stride + 1}
    idx |= {1023 * stride + 1, (1023 * stride + P) // 2}  # after the last head sample: only the full scan sees them
    if stride > 2:
        idx |= {stride // 2, 511 * stride + stride // 2}  # between head samples
    return sorted(i for i in idx if 0 <= i < P)


@pytest.mark.parametrize("which", ["object", "background"])
@pytest.mark.parametrize("setting", SETTINGS)
def test_single_hit_found_at_every_scan_position(grids, setting, which):
    """One point per candidate lies in a finger; the rest of the set is on the line.  Each candidate must find its point
    wherever the scan order puts it: first/last, chunk edges, strided-head samples and the points the head skips."""
    gig = grids["gig"]
    for P in SWEEP_P:
        pts = _line(P)
        idx = _sweep_indices(P)
        poses = [_pose_at(pts[i] - R @ FINGER, gig) for i in idx]
        poses.append(_pose_at(pts[0] + R[:, 2] * SPACING / 2 - R @ FINGER, gig))   # between two points: no hit
        poses = np.stack(poses)
        none = np.zeros((0, 3))
        p1, p2 = (pts, none) if which == "object" else (none, pts)
        st, off, _ = _run(grids, setting, poses, p1, p2, split=True)
        hit = 3 if which == "object" else 4
        assert (st[:-1] == hit).all(), (P, [idx[k] for k in np.nonzero(st[:-1] != hit)[0][:8]])
        assert st[-1] == 0 and off[-1] == 0, P
        assert (off[:-1] == -1).all()


# ------------------------------------------------------------------ lateral offsets and split status
DELTAS_MM = [0, 1, -1, 2, -2]


def _winner(n, m):
    """A at depth n + 0.25 mm inside finger 1 (y face 25 mm), B at m + 0.25 mm inside finger 2; the gripper moves by
    Delta along its y axis, so A's depth becomes n + 0.25 - Delta and B's m + 0.25 + Delta.  With the voxel margin
    (0.433 mm) a depth of 0.25 mm hits and -0.75 mm does not, for trilinear and nearest-cell lookups alike."""
    for k, d in enumerate(DELTAS_MM):
        if not (n - d >= 0 or m + d >= 0):
            return k
    return -1


OFFSET_CASES = [(-1, -1), (0, -2), (-2, 0), (1, -3), (-3, 1), (2, 2)]   # winners 0, 1, 2, 3, 4, none


def _groups(gig, groups):
    """groups: list of (object points, background points) in gripper coordinates -> poses, p1, p2 (camera frame)"""
    poses, p1, p2 = [], [], []
    for c, (obj, bg) in enumerate(groups):
        o = BASE + R[:, 2] * SPACING * c
        poses.append(_pose_at(o, gig))
        p1 += [o + R @ np.asarray(q) for q in obj]
        p2 += [o + R @ np.asarray(q) for q in bg]
    return np.stack(poses), np.array(p1).reshape(-1, 3), np.array(p2).reshape(-1, 3)


@pytest.mark.parametrize("setting", SETTINGS)
def test_winning_offset_closed_form(grids, setting):
    from catgrasp_b200.my_cpp import voxel_margin
    assert [_winner(n, m) for n, m in OFFSET_CASES] == [0, 1, 2, 3, 4, -1]
    groups = [([(0.0225, 0.025 + (n + 0.25) * 1e-3, 0.0), (0.0225, -0.025 - (m + 0.25) * 1e-3, 0.0)], [])
              for n, m in OFFSET_CASES]
    poses, p1, p2 = _groups(grids["gig"], groups)
    st, off, out = _run(grids, setting, poses, p1, p2, adjust=True, margin=voxel_margin(0.0005))
    assert off.tolist() == [0, 1, 2, 3, 4, -1], off.tolist()
    assert st.tolist() == [0, 0, 0, 0, 0, 3]
    shift = np.einsum("ij,ij->i", out[:5, :3, 3] - poses[:5, :3, 3], poses[:5, :3, 1]) * 1e3
    assert np.abs(shift - np.array(DELTAS_MM)).max() < 1e-3


@pytest.mark.parametrize("setting", SETTINGS)
def test_split_status_closed_form(grids, setting):
    """3 = the object's points hit the open gripper (also when the background hits too), 4 = only the background hits
    the enclosed gripper (a point in the gap), 0 = neither."""
    from catgrasp_b200.my_cpp import voxel_margin
    inA = (0.0225, 0.025 + 1.25e-3, 0.0)
    free = (0.0225, 0.025 - 0.75e-3, 0.0)
    groups = [([inA], []), ([free], [GAP]), ([inA], [GAP]), ([free], []), ([], [GAP]), ([inA], [])]
    poses, p1, p2 = _groups(grids["gig"], groups)
    st, off, _ = _run(grids, setting, poses, p1, p2, split=True, margin=voxel_margin(0.0005))
    assert st.tolist() == [3, 4, 3, 0, 4, 3]
    st, _, _ = _run(grids, setting, poses, p1, p2, split=False, margin=voxel_margin(0.0005))
    assert st.tolist() == [3, 3, 3, 0, 3, 3]


@pytest.mark.parametrize("setting", SETTINGS)
def test_points_outside_the_cropped_grid(grids, setting):
    """A point in finger 1 just beyond the cropped grid's y face hits in every setting; a point 20 cm out along the
    gripper's y axis clamps onto that face, so only the cropped grid's plain scan reports it (sdf.py clamps)."""
    from catgrasp_b200.my_cpp import voxel_margin
    near, far = (0.0225, 0.03275, 0.0), (0.0225, 0.2, 0.0)
    groups = [([near], []), ([far], []), ([], [near]), ([], [far]), ([], [])]
    poses, p1, p2 = _groups(grids["gig"], groups)
    st, _, _ = _run(grids, setting, poses, p1, p2, margin=voxel_margin(0.0005))
    far_hit = 3 if setting == "cropped" else 0
    assert st.tolist() == [3, far_hit, 3, far_hit, 0]


# ------------------------------------------------------------------ a full hit queue
def _free_points(n, rng):
    """gripper coordinates inside the padded grid box and the cropped one, in free space of both grippers:
    above the fingers and the gap, |z| in [10.7, 13.8] mm, x >= 3 mm (sd >= 0.7 mm > margin + 1e-4)"""
    x = rng.uniform(0.003, 0.043, n)
    y = rng.uniform(-0.031, 0.031, n)
    z = rng.uniform(0.0107, 0.0138, n) * rng.choice([-1, 1], n)
    return np.stack([x, y, z], 1)


@pytest.mark.parametrize("setting", SETTINGS)
def test_full_hit_queue(grids, setting):
    """Every point of every 1024-point chunk needs the eight-corner lookup, so the queue fills to its capacity; the one
    colliding point (if any) sits at index 0, 1023, 1024 or P-1."""
    from catgrasp_b200.my_cpp import voxel_margin
    gig = grids["gig"]
    rng = np.random.RandomState(7)
    o = BASE
    pose = _pose_at(o, gig)[None]
    for P in (1024, 1025, 3000):
        base = _free_points(P, rng)
        for hit in (None, 0, 1023, 1024, P - 1):
            if hit is not None and hit >= P:
                continue
            q = base.copy()
            if hit is not None:
                q[hit] = FINGER
            pts = o[None] + q @ R.T
            none = np.zeros((0, 3))
            for which in ("object", "background"):
                p1, p2 = (pts, none) if which == "object" else (none, pts)
                st, _, _ = _run(grids, setting, pose, p1, p2, margin=voxel_margin(0.0005))
                assert st[0] == (0 if hit is None else 3), (P, hit, which)


# ------------------------------------------------------------------ empty sets and thin grids
def test_empty_point_sets(grids):
    from catgrasp_b200.my_cpp import grasp_in_cam_unshifted
    from catgrasp_b200.synthetic import make_filter_case
    p1, p2, poses, sym, nocs_pose, c2n, g = make_filter_case(43, 48, 1)
    poses = np.einsum("ij,qjk->qik", nocs_pose @ c2n, poses)     # camera frame
    none = np.zeros((0, 3))
    for setting in SETTINGS:
        for a, b, encl in ((none, none, True), (none, none, False), (p1, none, True), (p1, none, False), (none, p2, True)):
            st, off, out = _run(grids, setting, poses, a, b, adjust=True, fdir=True, encl=encl)
            if len(a) == 0 and len(b) == 0:
                assert set(st.tolist()) <= {0, 1} and (off[st == 0] == 0).all()
                ref = grasp_in_cam_unshifted(poses, [EYE], EYE, EYE)
                assert np.array_equal(out[st == 0].view(np.uint32), ref[st == 0].view(np.uint32))


THIN = [(1, 7, 5), (2, 6, 4), (5, 1, 2), (1, 1, 1), (2, 2, 2), (3, 2, 1)]


@pytest.mark.parametrize("shape", THIN)
def test_thin_grids(cuda, shape):
    """1 or 2 cells on an axis: every cell is a boundary cell (cg_sdf_create's boundary scan) and the lookup has no
    upper neighbour on that axis.  Grids with and without a negative boundary cell, both lookups, margin 0 and > 0."""
    from catgrasp_b200.my_cpp import voxel_margin
    from catgrasp_b200.sdf import Sdf3D
    rng = np.random.RandomState(sum(shape))
    res = 0.004
    origin = np.array([0.1, -0.05, 0.6], np.float32)
    box = np.array(shape) * res
    pts = origin[None] + rng.uniform(-0.01, 1, (3000, 3)) * (box + 0.02)[None] - 0.005
    poses = np.stack([_jitter(rng) for _ in range(48)])
    for neg in (False, True):
        data = rng.uniform(0.0002, 0.004, shape).astype(np.float32)
        if neg:
            data.reshape(-1)[rng.randint(data.size)] = -0.002
        d = {"sdf": data, "origin": origin, "res": np.float32(res)}
        s = Sdf3D(data, origin, res)
        for mode_setting in ("padded", "nearest"):
            for margin in (0.0, voxel_margin(0.0005)):
                st, _, _ = _run(None, mode_setting, poses, pts[:1500], pts[1500:], adjust=True, margin=margin,
                                gig=EYE, sdfs=((d, s), (d, s)))
                assert (st == 0).any() or (st == 3).any()


def _jitter(rng, rot=0.02, tr=0.003):
    a = rng.normal(0, rot, 3)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + K + K @ K / 2
    u, _, vt = np.linalg.svd(T[:3, :3])
    T[:3, :3] = u @ vt
    T[:3, 3] = rng.normal(0, tr, 3)
    return T


# ------------------------------------------------------------------ the out-of-box shortcut at a positive margin
def _threshold(m):
    """smallest float32 boundary value for which make_view keeps the shortcut at margin m"""
    b = np.float32(m)
    while not (float(b) * (1.0 - 2.0 ** -19) - 2.0 ** -140 >= float(np.float32(m))):
        b = np.nextafter(b, np.float32(1))
    return b


def test_shortcut_threshold_is_a_few_ulps():
    from catgrasp_b200.my_cpp import voxel_margin
    m = np.float32(voxel_margin(0.0005))
    t = _threshold(m)
    n = int(t.view(np.int32) - m.view(np.int32))
    assert 8 <= n <= 40, n


@pytest.mark.parametrize("ulps", [0, 1, 7, "threshold", "2m"])
def test_margin_at_the_shortcut_edge(cuda, ulps):
    """A grid with a negative interior and every boundary cell = b, points all outside the box (clamped onto faces,
    edges and corners) in both sets.  For b just above the margin, rounded interpolation weights can put a clamped
    lookup below it: the kernel must scan such grids like the oracle does.  From the threshold up no lookup can."""
    from catgrasp_b200.my_cpp import voxel_margin
    from catgrasp_b200.sdf import Sdf3D
    m = np.float32(voxel_margin(0.0005))
    if ulps == "threshold":
        b = _threshold(m)
    elif ulps == "2m":
        b = np.float32(2 * m)
    else:
        b = np.float32(m)
        for _ in range(ulps):
            b = np.nextafter(b, np.float32(1))
    shape, res = (40, 30, 20), 0.001
    data = np.full(shape, -0.01, np.float32)
    data[0], data[-1], data[:, 0], data[:, -1], data[:, :, 0], data[:, :, -1] = b, b, b, b, b, b
    origin = np.array([-0.02, -0.015, 0.6], np.float32)
    d = {"sdf": data, "origin": origin, "res": np.float32(res)}
    s = Sdf3D(data, origin, res)
    rng = np.random.RandomState(11)
    lo, hi = origin - 0.02, origin + (np.array(shape) - 1) * res + 0.02
    pts = rng.uniform(lo, hi, (20000, 3))
    rel = (pts - origin) / res
    inside = ((rel > -6) & (rel < np.array(shape) - 1 + 6)).all(1)          # 5 mm clear of the box
    pts = pts[~inside][:8000]
    poses = np.stack([_jitter(rng, rot=0.002, tr=0.001) for _ in range(64)])   # moves the box by < 2.5 mm
    none = np.zeros((0, 3))
    rejected = 0
    for a, c in ((pts, none), (none, pts)):
        st, _, _ = _run(None, "padded", poses, a, c, margin=float(m), gig=EYE, sdfs=((d, s), (d, s)))
        rejected += int((st != 0).sum())
    print(f"b = m + {ulps} ulps: {rejected} of 128 poses rejected")
    if ulps == 0:
        assert rejected > 0                               # the case the old shortcut rule got wrong
    if ulps in ("threshold", "2m"):
        assert rejected == 0                              # the bound of make_view: no clamped lookup below m


# ------------------------------------------------------------------ float64 predicate
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("adjust,fdir", [(True, True), (False, True), (True, False)])
@pytest.mark.parametrize("S,scale", [(1, (1, 1, 1)), (12, (1.0, 1.1, 0.9))])
def test_kernel_agrees_with_float64_predicate(cuda, mode, adjust, fdir, S, scale):
    from catgrasp_b200 import my_cpp
    from catgrasp_b200.sdf import Sdf3D
    from catgrasp_b200.synthetic import make_filter_case
    from oracle import filter64
    p1, p2, poses, sym, nocs_pose, c2n, g = make_filter_case(43, 128, S, scale)
    poses = poses[:32] if S > 1 else poses
    so = Sdf3D(g["open"]["sdf"], g["open"]["origin"], g["open"]["res"])
    se = Sdf3D(g["enclosed"]["sdf"], g["enclosed"]["origin"], g["enclosed"]["res"])
    st, off, out = my_cpp.filter_grasp_pose_raw(poses, sym, nocs_pose, c2n, g["gripper_in_grasp"], fdir, adjust, so, p1,
                                                se, p2, sdf_mode=mode)
    r = filter64.filter64(poses, sym, nocs_pose, c2n, g["gripper_in_grasp"], fdir, adjust, mode, g["open"], p1,
                          g["enclosed"], p2)
    bad, undecided = filter64.compare(r, st, off, out)
    print(f"float64 predicate: {len(st)} poses, {undecided} undecided")
    assert bad == 0 and undecided <= 0.02 * len(st)


def test_k2_sample_agrees_with_float64_predicate(cuda):
    from catgrasp_b200 import my_cpp
    from catgrasp_b200.sdf import Sdf3D
    from catgrasp_b200.synthetic import make_candidates, make_gripper_proxy, make_pile
    from oracle import filter64
    scene = make_pile(20000, seed=1)
    obj = scene["object_id"] == 3
    p1, p2 = scene["cloud_xyz"][obj], scene["cloud_xyz"][~obj]
    poses = make_candidates(p1, scene["cloud_normal"][obj], 4096, seed=1)
    sel = np.random.RandomState(5).choice(len(poses), 512, replace=False)
    g = make_gripper_proxy()
    so = Sdf3D(g["open"]["sdf"], g["open"]["origin"], g["open"]["res"])
    se = Sdf3D(g["enclosed"]["sdf"], g["enclosed"]["origin"], g["enclosed"]["res"])
    st, off, out = my_cpp.filter_grasp_pose_raw(poses, [EYE], EYE, EYE, g["gripper_in_grasp"], True, True, so, p1, se, p2)
    r = filter64.filter64(poses[sel], [EYE], EYE, EYE, g["gripper_in_grasp"], True, True, 0, g["open"], p1,
                          g["enclosed"], p2)
    bad, undecided = filter64.compare(r, st[sel], off[sel], out[sel])
    print(f"K2 sample: 512 poses, {undecided} undecided")
    assert bad == 0 and undecided <= 0.02 * 512
    assert (r["status"] == 0).any() and (r["status"] == 3).any() and (r["status"] == 1).any()
