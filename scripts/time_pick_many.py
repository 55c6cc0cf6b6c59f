"""compute_candidate_grasp_many against a loop of compute_candidate_grasp, on B = 1, 4 and 8 render_depth piles (the
reference K at a reduced frame size, seeds 0 .. B-1, synthetic weights), with the renderer's id map as the
segmentation (a segmenter without predict_many) and with PointGroupPredictor (m = 16, synthetic weights, predict_many):

  - the shared scene stages: the sum of the ``timings`` entries of back-projection and masks, normals, segmentation,
    segment table and 1 mm scene, each ending in a synchronise (over the frames for the loop, once for the batch);
  - the whole call with every generator consumed, on the host clock from a synchronised device to a synchronise,
    without ``timings``.

The loop and the batch alternate, each warmed up first, from the same numpy state; every yielded dict and numpy's
state after it are compared bit for bit.

    python scripts/time_pick_many.py [--reps 3] [--frames 1 4 8] [--scale 0.5] [--objects 8]
"""
import _harness
import argparse
import tempfile
import time

import numpy as np
import torch

from catgrasp_b200 import pick, synthetic
from time_pick import CFG_RUN, IdSegmenter
from time_pointgroup import _predictor

SHARED = ("back-projection and masks", "normals", "segmentation", "segment table", "1 mm scene")


class IdMapSegmenter:
    """The renderer's id map of each frame, found by the frame's point count and first point."""

    def __init__(self):
        self.by_key = {}

    @staticmethod
    def _key(xyz):
        return (int(xyz.shape[0]), tuple(xyz[0].tolist()))

    def add(self, xyz, labels):
        self.by_key[self._key(xyz)] = IdSegmenter(labels)

    def predict(self, data):
        return self.by_key[self._key(data["cloud_xyz"])].predict(data)


def _setup(tmp):
    from catgrasp_b200.predicter import GraspPredicter, NunocsPredicter
    gp = GraspPredicter("nut", artifact_dir=synthetic.write_artifacts(f"{tmp}/cls", "cls", 2048, seed=3), device=0)
    npd = NunocsPredicter("nut", artifact_dir=synthetic.write_artifacts(
        f"{tmp}/seg", "seg", 2048, with_normalizer=False, state_dict=synthetic.make_lattice_seg_state_dict(seed=5)),
        device=0)
    g = synthetic.make_gripper_proxy()
    box = [0.0, 0.045, -0.010, 0.010]
    gripper = {"vertices": g["open"]["V"], "faces": g["open"]["F"], "enclosed_vertices": g["enclosed"]["V"],
               "enclosed_faces": g["enclosed"]["F"], "hand_depth": 0.012, "init_bite": 0.002,
               "grasp_in_gripper": np.linalg.inv(g["gripper_in_grasp"]), "finger_boxes": np.array([box, box]),
               "grip_dirs": np.array([[0, -1, 0], [0, 1, 0]]), "finger_mesh_in_grasp": g["gripper_in_grasp"]}
    cam = np.eye(4)
    cam[:3, :3] = np.diag([1.0, -1.0, -1.0])
    cam[:3, 3] = [0.6, 0.0, 0.85]
    eeg = np.eye(4)
    eeg[:3, :3] = np.array([[0, 0, 1], [0, 1, 0], [-1, 0, 0]], float).T
    eeg[:3, 3] = [-0.17, 0, 0]
    up = np.deg2rad([170, 120, 170, 120, 170, 120, 175])
    env = {"cam_in_world": cam, "bin_in_world": np.eye(4), "ee_in_grasp": eeg, "upper": up, "lower": -up}
    rng = np.random.RandomState(31)
    pts, nrm = synthetic.sample_hex_nut(3000, rng)
    lo, s = pts.min(0), (pts.max(0) - pts.min(0)).max()
    poses = synthetic.make_candidates(pts, nrm, 200, seed=32)
    poses[:, :3, 3] = (poses[:, :3, 3] - lo) / s
    canonical = {"canonical_grasps": poses, "canonical_scores": rng.uniform(0.9, 1, 200),
                 "canonical_cloud": (pts - lo) / s, "canonical_normals": nrm,
                 "canonical_affordance": np.clip(0.5 + 0.5 * np.sin(40 * pts[:, 0]), 0, 1)}
    return gp, npd, gripper, env, canonical


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--scale", type=float, default=0.5, help="frame size and focal length as a share of the reference")
    ap.add_argument("--objects", type=int, default=8)
    a = ap.parse_args()
    print("card:", _harness.card())
    K = _harness.REFERENCE_K.copy()
    K[:2] *= a.scale
    H, W = (int(round(v * a.scale)) for v in _harness.REFERENCE_HW)
    dev = torch.device("cuda", 0)
    tmp = tempfile.mkdtemp()
    gp, npd, gripper, env, canonical = _setup(tmp)
    frames, idmap = [], IdMapSegmenter()
    from catgrasp_b200 import cloud
    for seed in range(max(a.frames)):
        depth, ids = synthetic.render_depth(K, H, W, n_objects=a.objects, seed=seed)
        d, bg = torch.from_numpy(depth).to(dev), torch.from_numpy(ids < 0).to(dev)
        pts = cloud.depth2xyzmap(d, K)[bg == 0].reshape(-1, 3)
        idmap.add(pts, torch.from_numpy(ids[ids >= 0].astype(np.int64)).to(dev))
        frames.append((d, bg))
    print(f"frames {H} x {W}, {a.objects} objects, no-background points per frame "
          f"{min(int((f[1] == 0).sum()) for f in frames)} to {max(int((f[1] == 0).sum()) for f in frames)}")
    segmenters = {"id map": idmap, "PointGroup": _predictor(16, tmp)}

    def loop(fr, seg, timings):
        out = []
        for d, bg in fr:
            for r in pick.compute_candidate_grasp(d, K, bg, seg, npd, gp, gripper, env, canonical, [np.eye(4)],
                                                  CFG_RUN, timings=timings):
                out.append((r, np.random.get_state()))
        return out

    def many(fr, seg, timings):
        out = []
        gens = pick.compute_candidate_grasp_many([f[0] for f in fr], [K] * len(fr), [f[1] for f in fr],
                                                 [env] * len(fr), seg, npd, gp, gripper, canonical, [np.eye(4)],
                                                 CFG_RUN, timings=timings)
        for g in gens:
            for r in g:
                out.append((r, np.random.get_state()))
        return out

    for sname, seg in segmenters.items():
        for B in a.frames:
            fr = frames[:B]
            forms = {"loop": loop, "many": many}
            outs, shared, whole = {}, {f: [] for f in forms}, {f: [] for f in forms}
            for rep in range(a.reps + 1):                      # round 0 warms both forms up
                for f, fn in forms.items():
                    np.random.seed(0)
                    timings = {}
                    fn(fr, seg, timings)
                    np.random.seed(0)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    outs[f] = fn(fr, seg, None)
                    torch.cuda.synchronize()
                    if rep:
                        shared[f].append(sum(timings.get(k, 0.0) for k in SHARED))
                        whole[f].append((time.perf_counter() - t0) * 1e3)
            eq = len(outs["loop"]) == len(outs["many"]) and all(
                _same(r, w) and np.array_equal(st[1], wst[1]) and st[2] == wst[2]
                for (r, st), (w, wst) in zip(outs["loop"], outs["many"]))
            print(f"{sname}, B = {B}: {len(outs['many'])} objects yielded; many == loop bit for bit, numpy state "
                  f"included: {eq}")
            for f in forms:
                print(f"  {f:5s} shared stages {_harness.summary(shared[f])}")
                print(f"  {f:5s} whole call    {_harness.summary(whole[f])}")
            print(f"  loop / many (medians): shared stages {np.median(shared['loop']) / np.median(shared['many']):.2f}"
                  f", whole call {np.median(whole['loop']) / np.median(whole['many']):.2f}")


if __name__ == "__main__":
    main()
