"""Affordance transfer with the structure of the reference's ``compute_grasp_affordance`` (run_grasp_simulation.py:50-107;
SURVEY.md 8f F4), all grasps of an object in one launch (csrc/cg_affordance.cu).

Host (once per object): the canonical cloud in the camera frame, its 2 mm down-sampled copy with normals, and for every
down-sampled point the affordance of its nearest canonical point (the kd-tree query of run_grasp_simulation.py:62 does not
depend on the grasp: contact points are a subset of the down-sampled cloud).  Device (per grasp): finger-frame transform,
finger-extent test, contact patch, normal test, mean affordance.
"""
import numpy as np
import torch
from scipy.spatial import cKDTree

from . import _lib


def finger_boxes_from_meshes(finger_meshes):
    """x / z extent of each finger mesh's vertices (pybullet_env/env_grasp.py:252)."""
    return np.array([[m.vertices[:, 0].min(), m.vertices[:, 0].max(), m.vertices[:, 2].min(), m.vertices[:, 2].max()]
                     for m in finger_meshes], dtype=np.float64)


def compute_grasp_affordance(grasp_poses, finger_mesh_in_grasp, canonical_pts_in_cam, canonical_normals_in_cam,
                             canonical_cloud_in_cam, canonical_affordance, finger_boxes, grip_dirs, surface_tol=0.005,
                             device=0):
    """Returns (p_T_given_G (G,) float64 with NaN where the reference drops the grasp (run_grasp_simulation.py:66-67),
    contact-patch sizes (G, F) int32)."""
    poses = np.asarray(grasp_poses, dtype=np.float64).reshape(-1, 4, 4)
    G = poses.shape[0]
    boxes = np.ascontiguousarray(finger_boxes, dtype=np.float64).reshape(-1, 4)
    F = boxes.shape[0]
    dirs = []
    for d in np.asarray(grip_dirs, dtype=np.float64).reshape(F, 3):
        d = d / np.linalg.norm(d)
        if np.allclose(d, [0, 1, 0]):
            dirs.append(1)
        elif np.allclose(d, [0, -1, 0]):
            dirs.append(-1)
        else:
            raise RuntimeError(f"grip_dir={d}")                            # env_grasp.py:266-267
    if G == 0:
        return np.zeros(0), np.zeros((0, F), np.int32)
    pts = np.ascontiguousarray(canonical_pts_in_cam, dtype=np.float64)
    _, nn = cKDTree(np.asarray(canonical_cloud_in_cam, dtype=np.float64)).query(pts)       # :62, once per object
    aff = np.ascontiguousarray(np.asarray(canonical_affordance, dtype=np.float64)[nn])
    cam_in_finger = np.linalg.inv(np.asarray(finger_mesh_in_grasp, np.float64)) @ np.linalg.inv(poses)   # :52
    ctx, d_T, d_pts, d_nrm, d_aff = _lib.inputs(cam_in_finger, pts, canonical_normals_in_cam, aff, dtype=torch.float64,
                                                ctx=_lib.Context.get(device))
    out_p = torch.empty((G,), dtype=torch.float64, device=d_T.device)
    out_c = torch.zeros((G, 4), dtype=torch.int32, device=d_T.device)
    ctx.call("cg_grasp_affordance_dev", ctx.h, d_T, G, d_pts, d_nrm, d_aff, pts.shape[0], boxes,
             np.array(dirs, dtype=np.intc), F, float(surface_tol), out_p, out_c)
    return out_p.cpu().numpy(), out_c.cpu().numpy()[:, :F]
