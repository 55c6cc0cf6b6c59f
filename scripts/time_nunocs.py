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
import _harness
import argparse
import copy
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from catgrasp_b200 import cloud, synthetic   # noqa: E402
from catgrasp_b200.predicter import NunocsPredicter, _LegacyDraw   # noqa: E402

K = _harness.REFERENCE_K


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print("card:", _harness.card())
    from test_ransac_pose import old_predict
    depth, ids = synthetic.render_depth(K, *_harness.REFERENCE_HW, n_objects=16, seed=1)
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

    times, poses = {"old": [], "host": [], "device": []}, {}

    def run(mode):
        if mode == "old":
            poses[mode] = old_predict(npd, copy.deepcopy(data))[1]
        else:
            npd.subsample = mode
            poses[mode] = npd.predict(copy.deepcopy(data))[1]

    for m in times:                                           # warm-up
        np.random.seed(0)
        run(m)
    for _ in range(a.reps):
        for m in times:
            np.random.seed(0)
            times[m] += _harness.wall_ms(lambda: run(m), 1, 0)
    same = (poses["old"] is None and poses["host"] is None) or \
        (poses["old"] is not None and poses["host"] is not None and poses["old"].tobytes() == poses["host"].tobytes())
    print(f"host pose == old pose bit for bit: {same}")
    for m in ("old", "host", "device"):
        print(f"predict {m:7s} {_harness.summary(times[m])}")

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
    ts = _harness.queued_ms(lambda: ransac9d_pose(src, tgt, hyp, npd.THRESHOLDS, **kw), 20, 3)
    print(f"fused launch (N = {src.shape[0]}, 2 x {npd.ransac_max_iter}) {_harness.summary(ts)}")

    # the host draw against the walk alone
    td, ts = [], []
    for _ in range(a.reps):
        np.random.seed(1)
        d = _LegacyDraw()
        td += _harness.wall_ms(lambda: d.draw(8192, 4, 20000), 1, 0)
        np.random.seed(1)
        d = _LegacyDraw()
        ts += _harness.wall_ms(lambda: d.skip(8192, 4, 20000), 1, 0)
    print(f"host draw 20000 x (4 of 8192)      {_harness.summary(td)}")
    print(f"cg_host_legacy_skip, same stream   {_harness.summary(ts)}")
    print(f"draw / skip (medians) {np.median(td) / np.median(ts):.2f}")


if __name__ == "__main__":
    main()
