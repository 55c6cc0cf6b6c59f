"""CPU ORACLE (test infrastructure only): numpy restatement of run_grasp_simulation.py:50-73
(compute_grasp_affordance_worker) and pybullet_env/env_grasp.py:243-283 (get_finger_contact_area).
PINNED: tests/test_affordance_golden.py checks it against values produced by the reference's own functions
(tests/golden/make_golden_affordance.py)."""
import numpy as np


def _finger_contact_area(box, ob_in_finger, ob_pts, ob_normals, grip_dir, surface_tol):
    """box = (xmin, xmax, zmin, zmax) of the finger mesh vertices.  Returns (surface_pts in the camera frame, dist) or None."""
    grip_dir = np.array(grip_dir, dtype=float)
    grip_dir = grip_dir / np.linalg.norm(grip_dir)
    R, t = ob_in_finger[:3, :3], ob_in_finger[:3, 3]
    cur_pts = (R @ ob_pts.T).T + t
    cur_normals = (R @ ob_normals.T).T
    m = (cur_pts[:, 0] >= box[0]) & (cur_pts[:, 0] <= box[1]) & (cur_pts[:, 2] >= box[2]) & (cur_pts[:, 2] <= box[3])
    if m.sum() == 0:
        return None
    w_pts, w_n = cur_pts[m], cur_normals[m]
    if np.allclose(grip_dir, np.array([0, 1, 0])):
        dist = np.abs(w_pts[:, 1] - w_pts[:, 1].min())
    elif np.allclose(grip_dir, np.array([0, -1, 0])):
        dist = np.abs(w_pts[:, 1] - w_pts[:, 1].max())
    else:
        raise RuntimeError(f"grip_dir={grip_dir}")
    c = dist <= surface_tol
    if c.sum() == 0:
        return None
    dist = dist[c]
    n = w_n[c][np.abs(dist).argmin()].copy()
    n /= np.linalg.norm(n)
    if np.dot(n, grip_dir) > 0:
        return None
    homo = np.concatenate((w_pts[c], np.ones((c.sum(), 1))), axis=-1)
    return (np.linalg.inv(ob_in_finger) @ homo.T).T[:, :3], dist


def grasp_affordance(grasp_poses, finger_mesh_in_grasp, pts_in_cam, normals_in_cam, canonical_affordance, kdtree, finger_boxes,
                     grip_dirs, surface_tol=0.005):
    """p(T|G) per grasp (NaN where the reference returns None) and contact-patch sizes (G, F)."""
    out = np.full(len(grasp_poses), np.nan)
    ncon = np.zeros((len(grasp_poses), len(finger_boxes)), np.int32)
    for i, grasp_in_cam in enumerate(grasp_poses):
        cam_in_finger = np.linalg.inv(finger_mesh_in_grasp) @ np.linalg.inv(grasp_in_cam)
        scores = []
        for f, box in enumerate(finger_boxes):
            r = _finger_contact_area(box, cam_in_finger, pts_in_cam, normals_in_cam, grip_dirs[f], surface_tol)
            if r is None:
                continue
            surface_pts, _ = r
            ncon[i, f] = len(surface_pts)
            _, idx = kdtree.query(surface_pts)
            scores.append(canonical_affordance[idx].mean())
        if scores:
            v = np.array(scores).mean()
            if np.isfinite(v):
                out[i] = v
    return out, ncon


U = 2.0 ** -53


def finger_decisions(R, t, pts, nrm, box, sgn, tol, exact=False):
    """Every decision the kernel makes for one finger of one grasp (env_grasp.py:243-283), with the point set of each
    and whether rounding could change it.  The kernel forms q = fma(r2, z, fma(r1, y, r0 x)) + t; numpy's R @ p + t
    rounds differently, each by at most 3 u (|r| |p| + |t|) per coordinate, so ``slack`` = 8 u (|r| |p| + |t|) bounds
    the gap between the two.  A point within the slack of a box edge or of |y - y_ext| = tol, a second in-patch point
    within twice the slack of the closest one (np.argmin's pick), or a normal whose y / |n| is within 8 u of 0 makes
    the finger *undecided*.  exact=True (dyadic inputs under signed axis permutations: every product and sum exact)
    sets the slack to 0.
    Returns dict(inbox, y_ext, patch (indices), jstar, facing_away, dropped, undecided)."""
    q = pts @ R.T + t
    slack = np.zeros(len(pts)) if exact else 8 * U * (np.abs(pts) @ np.abs(R).T + np.abs(t)).max(axis=1)
    x, y, z = q[:, 0], q[:, 1], q[:, 2]
    inbox = (x >= box[0]) & (x <= box[1]) & (z >= box[2]) & (z <= box[3])
    near = lambda v, e: np.abs(v - e) <= slack                 # noqa: E731
    und = bool((near(x, box[0]) | near(x, box[1]) | near(z, box[2]) | near(z, box[3])).any())
    out = {"inbox": np.nonzero(inbox)[0], "y_ext": None, "patch": np.zeros(0, np.int64), "jstar": None,
           "facing_away": None, "dropped": True, "undecided": und}
    if not inbox.any():                                       # within_finger_mask.sum()==0 (:253-254)
        return out
    y_ext = sgn * (sgn * y[inbox]).min()
    d = np.abs(y - y_ext)
    # the kernel's y_ext can differ by one point's slack: widen every |d - tol| test by the largest in-box slack
    sl = slack + (slack[inbox].max() if not exact else 0.0)
    out["undecided"] = und or bool((inbox & (np.abs(d - tol) <= sl)).any())
    patch = np.nonzero(inbox & (d <= tol))[0]
    out["y_ext"], out["patch"] = y_ext, patch
    if patch.size == 0:                                       # contact_mask.sum()==0 (:268-269)
        return out
    j = patch[np.argmin(d[patch])]
    if not exact and ((d[patch] <= d[j] + 2 * sl[patch]) & (patch != j)).any():
        out["undecided"] = True
    n = R @ nrm[j]
    out["jstar"] = j
    out["facing_away"] = bool((n[1] / np.linalg.norm(n)) * sgn > 0)
    if not exact and abs(n[1]) <= 8 * U * (np.abs(R[1]) @ np.abs(nrm[j])):
        out["undecided"] = True
    out["dropped"] = out["facing_away"]
    return out


def grasp_affordance_pointwise_nn(grasp_poses, finger_mesh_in_grasp, pts_in_cam, normals_in_cam, aff_of_pts, finger_boxes,
                                  grip_signs, surface_tol=0.005, exact=False, decisions=False):
    """The formulation the CUDA kernel uses: the nearest-canonical-point affordance is attached to every (down-sampled)
    point once (``aff_of_pts``) instead of being queried per contact patch.  Identical to grasp_affordance() except where a
    point is equidistant from two canonical points (a voxel mean of two points is): the reference's per-patch query breaks
    such ties by the rounding noise of its transform round trip (env_grasp.py:282), so a patch mean can differ by one
    point's affordance / patch size (observed <= 2.3e-4).
    Per finger the decisions come from finger_decisions(); with decisions=True also returns, per grasp, the list of
    per-finger decision dicts and whether any of them is undecided."""
    T = np.linalg.inv(finger_mesh_in_grasp) @ np.linalg.inv(np.asarray(grasp_poses, np.float64))
    out = np.full(len(T), np.nan)
    ncon = np.zeros((len(T), len(finger_boxes)), np.int32)
    per, und = [], np.zeros(len(T), bool)
    for gi in range(len(T)):
        R, t = T[gi, :3, :3], T[gi, :3, 3]
        tot, nf, fd = 0.0, 0, []
        for f, sgn in enumerate(grip_signs):
            r = finger_decisions(R, t, pts_in_cam, normals_in_cam, finger_boxes[f], sgn, surface_tol, exact=exact)
            fd.append(r)
            und[gi] |= r["undecided"]
            if r["dropped"]:
                continue
            ncon[gi, f] = len(r["patch"])
            tot += aff_of_pts[r["patch"]].mean()
            nf += 1
        per.append(fd)
        if nf:
            out[gi] = tot / nf
    if decisions:
        return out, ncon, per, und
    return out, ncon
