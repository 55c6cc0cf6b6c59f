"""Cone grasp-pose enumeration with the structure of the reference's
``dexnet/grasping/grasp_sampler.py::PointConeGraspSampler`` (SURVEY.md 8f F3).

Split of work (file:line = dexnet/grasping/grasp_sampler.py unless stated):
  host   * the view-sphere directions (``hinter_sampling`` Utils.py:293-391, cone mask / rotation / random subset
           :140-149) -- per scene, a few dozen vectors;
         * the local frame ``R0`` of every surface sample (:227-263: kd-tree ball query, normal scatter matrix,
           ``np.linalg.eig``) -- kept on the host so eigenvector signs and the numpy-RNG stream are the reference's;
  device * the R0 @ R_sphere @ R_inplane x approach-depth enumeration (:266-286) and the optional
           ``center_ob_between_gripper`` shift (:191-203) -- csrc/cg_cone.cu; the poses stay on the GPU and feed
           ``my_cpp.filter_grasp_pose_raw`` without a host round trip.

``cone_grasp_poses`` consumes the global numpy RNG exactly like ``sample_grasps`` (:131-158).
"""
import math

import numpy as np
import torch
from scipy.spatial import cKDTree

from . import _lib


def euler_matrix(ai, aj, ak, axes="sxyz"):
    """Static-frame x-y-z Euler angles -> 4x4, the published formula of the ``transformations`` module the reference
    imports (Utils.py:10; used at grasp_sampler.py:144,:268 with axes='sxyz')."""
    if axes != "sxyz":
        raise NotImplementedError("only the 'sxyz' convention the reference uses")
    si, sj, sk = math.sin(ai), math.sin(aj), math.sin(ak)
    ci, cj, ck = math.cos(ai), math.cos(aj), math.cos(ak)
    cc, cs = ci * ck, ci * sk
    sc, ss = si * ck, si * sk
    M = np.identity(4)
    M[0, 0] = cj * ck
    M[0, 1] = sj * sc - cs
    M[0, 2] = sj * cc + ss
    M[1, 0] = cj * sk
    M[1, 1] = sj * ss + cc
    M[1, 2] = sj * cs - sc
    M[2, 0] = -sj
    M[2, 1] = cj * si
    M[2, 2] = cj * ci
    return M


def normalizeRotation(pose):
    """Utils.py:172-179."""
    new_pose = pose.copy()
    scales = np.linalg.norm(pose[:3, :3], axis=0)
    new_pose[:3, :3] /= scales.reshape(1, 3)
    return new_pose


def directionVecToRotation(direction, ref=np.array([0, 0, 1])):
    """Utils.py:262-290 (float64; the fp32 C++ twin is catgrasp_b200.my_cpp.directionVecToRotation)."""
    direction = direction / np.linalg.norm(direction)
    v = np.cross(direction, ref)
    if (v == 0).all():
        return np.eye(3)
    s = np.linalg.norm(v)
    c = direction.dot(ref)
    v_skew = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])
    if s == 0:
        R = np.array([[1, 0, 0], [0, -1, 0], [0, 0, -1]])
    else:
        R = (np.identity(3) + v_skew + v_skew.dot(v_skew) * (1 - c) / (s ** 2)).T
    return normalizeRotation(R)


_ICO_C = (1.0 + math.sqrt(5.0)) / 2.0
_ICO_PTS = [(-1.0, _ICO_C, 0.0), (1.0, _ICO_C, 0.0), (-1.0, -_ICO_C, 0.0), (1.0, -_ICO_C, 0.0), (0.0, -1.0, _ICO_C),
            (0.0, 1.0, _ICO_C), (0.0, -1.0, -_ICO_C), (0.0, 1.0, -_ICO_C), (_ICO_C, 0.0, -1.0), (_ICO_C, 0.0, 1.0),
            (-_ICO_C, 0.0, -1.0), (-_ICO_C, 0.0, 1.0)]
_ICO_FACES = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
              (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10),
              (8, 6, 7), (9, 8, 1)]


def hinter_sampling(min_n_pts, radius=1):
    """View-sphere sampling by icosahedron subdivision (Hinterstoisser et al., BMVC 2008), with the vertex numbering
    and the breadth-first / azimuth ordering of Utils.py:293-391.  Returns (points (V,3), creation level per point)."""
    pts = [list(p) for p in _ICO_PTS]
    level = [0] * len(pts)
    faces = list(_ICO_FACES)
    depth = 0
    while len(pts) < min_n_pts:
        depth += 1
        midpoint = {}
        split = []
        for f in faces:
            mids = []
            for a, b in ((f[0], f[1]), (f[1], f[2]), (f[2], f[0])):
                key = (a, b) if a < b else (b, a)
                if key not in midpoint:
                    midpoint[key] = len(pts)
                    pts.append((0.5 * (np.array(pts[key[0]]) + np.array(pts[key[1]]))).tolist())
                    level.append(depth)
                mids.append(midpoint[key])
            m01, m12, m20 = mids
            split += [(f[0], m01, m20), (m01, f[1], m12), (m01, m12, m20), (m20, m12, f[2])]
        faces = split
    pts = np.array(pts)
    pts *= np.reshape(radius / np.linalg.norm(pts, axis=1), (pts.shape[0], 1))
    neigh = {}
    for f in faces:
        for i in range(3):
            neigh.setdefault(f[i], set()).add(f[(i + 1) % 3])
            neigh[f[i]].add(f[(i + 2) % 3])
    two_pi = 2.0 * math.pi
    azimuth = lambda i: (math.atan2(pts[i][1], pts[i][0]) + two_pi) % two_pi      # noqa: E731
    order = []
    seen = [False] * len(pts)
    frontier = [int(np.argmax(pts[:, 2]))]
    while len(order) != len(pts):
        frontier = sorted(frontier, key=azimuth)          # stable: azimuth ties keep the set's iteration order
        reached = []
        for i in frontier:
            order.append(i)
            seen[i] = True
            reached += [j for j in neigh[i]]
        frontier = [j for j in set(reached) if not seen[j]]
    return pts[np.array(order), :], [level[i] for i in order]


def cone_sphere_points(n_sphere_dir, cone_deg=60.0):
    """grasp_sampler.py:140-149: sphere directions within ``cone_deg`` of +z, turned onto +x, at most ``n_sphere_dir`` of
    them (``np.random.choice`` without replacement from the global numpy RNG)."""
    sphere_pts = hinter_sampling(min_n_pts=1000, radius=1)[0]
    sphere_pts = sphere_pts / np.linalg.norm(sphere_pts, axis=-1).reshape(-1, 1)
    sphere_pts = sphere_pts[sphere_pts[:, 2] >= np.cos(cone_deg * np.pi / 180)]
    rot_y = euler_matrix(0, np.pi / 2, 0, axes="sxyz")[:3, :3]
    sphere_pts = (rot_y @ sphere_pts.T).T
    if sphere_pts.shape[0] > n_sphere_dir:
        ids = np.random.choice(np.arange(len(sphere_pts)), size=n_sphere_dir, replace=False)
        sphere_pts = sphere_pts[ids]
    return sphere_pts


def compute_cloud_resolution(pts, n_sample=100):
    """Utils.py:492-501 (consumes the numpy RNG)."""
    ids = np.random.choice(len(pts), size=n_sample).astype(int)
    sample_pts = pts[ids]
    background_ids = np.array(list(set(np.arange(len(pts))) - set(ids))).astype(int)
    dists, _ = cKDTree(pts[background_ids]).query(sample_pts)
    dists = np.array(dists[np.isfinite(dists)])
    return np.sort(dists)[:10].mean()


def surface_frame(selected_surface, selected_normal, points_for_sample, normals_for_sample, r_ball, kdtree=None):
    """grasp_sampler.py:227-263: R0 = [approach | major | minor] at one surface sample.  Like the reference it
    normalises the touched rows of ``normals_for_sample`` in place and doubles ``r_ball`` until the ball holds a
    neighbour; returns (R0 (3,3) float64, r_ball actually used)."""
    if kdtree is None:
        kdtree = cKDTree(points_for_sample)
    while True:
        M = np.zeros((3, 3))
        kd_indices = kdtree.query_ball_point(selected_surface.reshape(1, 3), r=r_ball)
        kd_indices = np.array(kd_indices[0]).astype(int).reshape(-1)
        sqr_distances = np.linalg.norm(selected_surface.reshape(1, 3) - points_for_sample[kd_indices], axis=-1) ** 2
        for k in range(len(kd_indices)):
            if sqr_distances[k] != 0:
                normal = normals_for_sample[kd_indices[k]].reshape(-1, 1)      # a view: normalised in place (:241-243)
                if np.linalg.norm(normal) != 0:
                    normal /= np.linalg.norm(normal)
                M += np.matmul(normal, normal.T)
        if sum(sum(M)) != 0:
            break
        r_ball *= 2                                                              # :246-249
    approach_normal = -selected_normal.reshape(3)
    approach_normal /= np.linalg.norm(approach_normal)
    eigval, eigvec = np.linalg.eig(M)
    minor_pc = eigvec[:, np.argmin(eigval)].reshape(3)
    minor_pc = minor_pc - np.dot(approach_normal, minor_pc) / np.dot(approach_normal, approach_normal) * approach_normal
    minor_pc /= np.linalg.norm(minor_pc)
    major_pc = np.cross(minor_pc, approach_normal)
    major_pc = major_pc / np.linalg.norm(major_pc)
    R0 = np.concatenate((approach_normal.reshape(3, 1), major_pc.reshape(3, 1), minor_pc.reshape(3, 1)), axis=1)
    return R0, r_ball


def enumerate_poses(surface_pts, R0s, sphere_pts, hand_depth, approach_step, init_bite, points_for_center=None,
                    inplane_deg=np.arange(0, 180, 30), device=0):
    """Device part: (S,3) samples with frames (S,3,3) -> poses ((P,4,4) float64 cuda, (P,4,4) float32 cuda),
    P = S * (1 + len(sphere_pts) * len(inplane_deg)) * len(np.arange(0, hand_depth, approach_step)), in the reference's
    order.  ``points_for_center`` (M,3) applies center_ob_between_gripper (:191-203)."""
    ref = np.array([1, 0, 0])
    R_sphere = np.stack([directionVecToRotation(direction=sp.copy(), ref=ref) for sp in sphere_pts]) \
        if len(sphere_pts) else np.zeros((0, 3, 3))
    R_inplane = np.stack([euler_matrix(x_rot * np.pi / 180, 0, 0, axes="sxyz")[:3, :3] for x_rot in inplane_deg])
    depths = np.arange(0, hand_depth, approach_step).astype(np.float64)
    S, NS, NI, ND = len(surface_pts), len(R_sphere), len(R_inplane), len(depths)
    P = S * (1 + NS * NI) * ND
    ctx, d_surf, d_R0, d_sph, d_inp, d_dep, d_pts = _lib.inputs(
        surface_pts, R0s, R_sphere, R_inplane, depths, points_for_center, dtype=torch.float64, ctx=_lib.Context.get(device))
    out64 = torch.empty((P, 4, 4), dtype=torch.float64, device=d_surf.device)
    out32 = torch.empty((P, 4, 4), dtype=torch.float32, device=d_surf.device)
    if P == 0:
        return out64, out32
    ctx.call("cg_cone_poses_dev", ctx.h, d_surf, d_R0, S, d_sph, NS, d_inp, NI, d_dep, ND, float(init_bite), out64, out32)
    if d_pts is not None:
        ctx.call("cg_center_grasps_dev", ctx.h, out64, out32, P, d_pts, d_pts.shape[0])
    return out64, out32


def cone_frames(points_for_sample, normals_for_sample, max_num_samples=200, n_sphere_dir=100):
    """Host half of PointConeGraspSampler.sample_grasps (:131-158, :227-263): returns (sample_ids that yield poses,
    R0s (S,3,3), sphere_pts).  Frames are the reference's bit for bit -- including the ill-defined ones it produces when
    the smallest principal direction is parallel to the approach axis (the projected vector is rounding noise, so such
    an R0 is not orthonormal).  Same numpy-RNG consumption as the reference: cloud resolution sample, sphere subset, shuffle of the
    surface samples; then ``np.random.seed(state[1][0])`` once per surface sample as :227 does."""
    resolution = compute_cloud_resolution(points_for_sample)
    r_ball = resolution * 3
    sphere_pts = cone_sphere_points(n_sphere_dir)
    sample_ids = np.arange(len(points_for_sample))
    np.random.shuffle(sample_ids)
    if len(sample_ids) > max_num_samples:
        sample_ids = sample_ids[:max_num_samples]
    seed = np.random.get_state()[1][0]
    kdtree = cKDTree(points_for_sample)
    R0s, keep = [], []
    for i in sample_ids:
        np.random.seed(seed)
        R0, r_ball = surface_frame(points_for_sample[i], normals_for_sample[i], points_for_sample, normals_for_sample,
                                   r_ball, kdtree)
        # np.linalg.eig may answer a (numerically) repeated eigenvalue with a complex pair; the reference then drops every
        # rotation built from that frame (``np.iscomplex(R).any()``, :273) -- here the whole surface sample is dropped.
        if np.iscomplexobj(R0):
            if np.iscomplex(R0).any():
                continue
            R0 = R0.real
        R0s.append(R0)
        keep.append(i)
    return np.array(keep, dtype=sample_ids.dtype), np.array(R0s).reshape(-1, 3, 3), sphere_pts


def cone_grasp_poses(points_for_sample, normals_for_sample, hand_depth, init_bite, max_num_samples=200, n_sphere_dir=100,
                     approach_step=0.003, center_ob_between_gripper=False, device=0):
    """PointConeGraspSampler.sample_grasps up to its filterGraspPose call (:131-203): the candidate poses in the camera
    frame, on the GPU, as ((P,4,4) float64, (P,4,4) float32) CUDA tensors."""
    sample_ids, R0s, sphere_pts = cone_frames(points_for_sample, normals_for_sample, max_num_samples, n_sphere_dir)
    return enumerate_poses(points_for_sample[sample_ids], R0s, sphere_pts, hand_depth, approach_step, init_bite,
                           points_for_center=points_for_sample if center_ob_between_gripper else None, device=device)
