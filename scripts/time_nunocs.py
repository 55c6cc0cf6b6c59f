"""Time of one object's NunocsPredicter.predict (an object of the time_pick.py pile, 'nut' synthetic lattice weights,
n_pts 2048, 2 x 10 000 RANSAC hypotheses) in three forms, run alternately:
  old    -- the straight composition: predict_nocs, then estimate9DTransform at 0.003 and 0.005 (10 000 numpy
            np.random.choice calls each) and predict's post-processing;
  host   -- predict with subsample = "host" (same numbers: one C draw of the 2 x 10 000 subsets, one fused launch);
  device -- predict with subsample = "device" (device draws, one fused launch);
then the fused launch alone (cg_ransac9d_pose_dev, CUDA events) and the host draw of 20 000 subsets of 4 of 8192
against cg_host_legacy_skip over the same stream.

    python scripts/time_nunocs.py [--reps 5]
"""
import argparse
import copy
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from catgrasp_b200 import cloud, synthetic   # noqa: E402
from catgrasp_b200.predicter import NunocsPredicter, _LegacyDraw   # noqa: E402

K = np.array([2257.7500557850776, 0, 1032, 0, 2257.4882391629421, 772, 0, 0, 1], np.float64).reshape(3, 3)


def spread(ts):
    ts = np.asarray(ts)
    return f"median {np.median(ts):9.2f} ms  min {ts.min():9.2f}  max {ts.max():9.2f}  (n={len(ts)})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("GPU:", smi)
    from test_ransac_pose import old_predict
    depth, ids = synthetic.render_depth(K, 1544, 2064, n_objects=16, seed=1)
    xyz = cloud.depth2xyzmap(depth, K)
    lab = ids[ids >= 0]
    pts = xyz[ids >= 0].reshape(-1, 3)
    big = np.bincount(lab).argmax()
    ob = pts[lab == big]
    data = {"cloud_xyz": ob, "cloud_normal": cloud.estimate_normals(ob, 0.002, 30)}
    tmp = tempfile.mkdtemp()
    npd = NunocsPredicter("nut", artifact_dir=synthetic.write_artifacts(
        f"{tmp}/seg", "seg", 2048, with_normalizer=False, state_dict=synthetic.make_lattice_seg_state_dict(seed=5)),
        device=0)
    print(f"object: {len(ob)} points, n_pts {npd.cfg['n_pts']}, H = {npd.ransac_max_iter} per threshold")

    def run(mode):
        np.random.seed(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if mode == "old":
            out = old_predict(npd, copy.deepcopy(data))[1]
        else:
            npd.subsample = mode
            out = npd.predict(copy.deepcopy(data))[1]
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    times, poses = {"old": [], "host": [], "device": []}, {}
    for m in times:
        run(m)                                                # warm-up
    for _ in range(a.reps):
        for m in times:
            t, poses[m] = run(m)
            times[m].append(t)
    same = (poses["old"] is None and poses["host"] is None) or \
        (poses["old"] is not None and poses["host"] is not None and poses["old"].tobytes() == poses["host"].tobytes())
    print(f"host pose == old pose bit for bit: {same}")
    for m in ("old", "host", "device"):
        print(f"predict {m:7s} {spread(times[m])}")

    # the fused launch alone
    from catgrasp_b200.aligning import ransac9d_pose
    dev = torch.device("cuda", 0)
    npd.subsample = "device"
    np.random.seed(0)
    nocs, _ = npd.predict(copy.deepcopy(data))
    src = torch.from_numpy(np.asarray(nocs, np.float64)).to(dev)
    tgt = torch.from_numpy(npd.data_transformed["cloud_xyz_original"]).to(dev)
    hyp = npd.model.draw_ids_dev(src.shape[0], 4, 2 * npd.ransac_max_iter, 1, first_candidate=1)
    kw = dict(max_scale=npd.max_scale, min_scale=npd.min_scale, max_dimensions=npd.MAX_DIMENSIONS)
    for _ in range(3):
        ransac9d_pose(src, tgt, hyp, npd.THRESHOLDS, **kw)
    ev = []
    for _ in range(20):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ransac9d_pose(src, tgt, hyp, npd.THRESHOLDS, **kw)
        e1.record()
        ev.append((e0, e1))
    torch.cuda.synchronize()
    print(f"fused launch (N = {src.shape[0]}, 2 x {npd.ransac_max_iter}) {spread([x.elapsed_time(y) for x, y in ev])}")

    # the host draw against the walk alone
    td, ts = [], []
    for _ in range(a.reps):
        np.random.seed(1)
        d = _LegacyDraw()
        t0 = time.perf_counter()
        d.draw(8192, 4, 20000)
        td.append((time.perf_counter() - t0) * 1e3)
        np.random.seed(1)
        d = _LegacyDraw()
        t0 = time.perf_counter()
        d.skip(8192, 4, 20000)
        ts.append((time.perf_counter() - t0) * 1e3)
    print(f"host draw 20000 x (4 of 8192)      {spread(td)}")
    print(f"cg_host_legacy_skip, same stream   {spread(ts)}")
    print(f"draw / skip (medians) {np.median(td) / np.median(ts):.2f}")


if __name__ == "__main__":
    main()
