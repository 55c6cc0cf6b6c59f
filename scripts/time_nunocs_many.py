"""NunocsPredicter.predict_many against the loop of predict calls it replaces, on the 16 objects of the time_pick.py
pile ('nut' synthetic lattice weights, 2 x 10 000 RANSAC hypotheses per object), in both subsample modes; the two
forms run alternately, each from the same numpy seed, and their results are compared bit for bit.  Then the batched
fused pose search alone (cg_ransac9d_pose_many_dev, CUDA events) at B = 1, 4 and 16 objects, and B single-object
launches (cg_ransac9d_pose_dev) for comparison.

    python scripts/time_nunocs_many.py [--reps 5] [--n-pts 2048]
"""
import _harness
import argparse
import tempfile

import numpy as np
import torch

from catgrasp_b200 import cloud, synthetic
from catgrasp_b200.predicter import NunocsPredicter

K = _harness.REFERENCE_K


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n-pts", type=int, default=2048)
    a = ap.parse_args()
    print("card:", _harness.card())
    depth, ids = synthetic.render_depth(K, *_harness.REFERENCE_HW, n_objects=16, seed=1)
    xyz = cloud.depth2xyzmap(depth, K)
    lab = ids[ids >= 0]
    pts = xyz[ids >= 0].reshape(-1, 3)
    datas = []
    for k in np.unique(lab):
        ob = pts[lab == k]
        datas.append({"cloud_xyz": ob, "cloud_normal": cloud.estimate_normals(ob, 0.002, 30)})
    tmp = tempfile.mkdtemp()
    npd = NunocsPredicter("nut", artifact_dir=synthetic.write_artifacts(
        f"{tmp}/seg", "seg", a.n_pts, with_normalizer=False, state_dict=synthetic.make_lattice_seg_state_dict(seed=5)),
        device=0)
    print(f"{len(datas)} objects of {min(len(d['cloud_xyz']) for d in datas)} to "
          f"{max(len(d['cloud_xyz']) for d in datas)} points, n_pts {a.n_pts}, H = {npd.ransac_max_iter} per threshold")

    forms = {"loop": lambda: [npd.predict(d) for d in datas], "many": lambda: npd.predict_many(datas)}
    for mode in ("host", "device"):
        npd.subsample = mode
        times, out = {f: [] for f in forms}, {}

        def run(f):
            np.random.seed(0)
            out[f] = forms[f]()
        for f in forms:                                       # warm-up
            run(f)
        for _ in range(a.reps):
            for f in forms:
                times[f] += _harness.wall_ms(lambda: run(f), 1, 0)
        same = all(_same(x[0], y[0]) and _same(x[1], y[1]) for x, y in zip(out["loop"], out["many"]))
        n_pose = sum(r[1] is not None for r in out["many"])
        print(f"{mode}: many == loop bit for bit: {same}; {n_pose} of {len(datas)} objects with a pose")
        for f in forms:
            print(f"  {mode} {f:5s} {_harness.summary(times[f])}")
        print(f"  {mode} loop / many (medians) {np.median(times['loop']) / np.median(times['many']):.2f}")

    # the batched fused launch alone, against B single-object launches on the same inputs
    from catgrasp_b200.aligning import ransac9d_pose, ransac9d_pose_many
    npd.subsample = "device"
    np.random.seed(0)
    dev = torch.device("cuda", 0)
    srcs, tgts = [], []
    for d in datas:                                           # each object's NOCS cloud and cloud_xyz_original
        npd.predict(d)
        dt = npd.data_transformed
        x = torch.as_tensor(np.asarray(dt["input"], np.float32)).to(dev)
        srcs.append(npd.model.nunocs_dev(x, int(npd.cfg["ce_loss_bins"]))[0].to(torch.float64))
        tgts.append(torch.as_tensor(np.asarray(dt["cloud_xyz_original"], np.float64)).to(dev))
    src, tgt = torch.stack(srcs), torch.stack(tgts)
    H = npd.ransac_max_iter
    hyp = torch.stack([npd.model.draw_ids_dev(a.n_pts, 4, 2 * H, 100 + b, first_candidate=1)
                       for b in range(len(datas))])
    kw = dict(max_scale=npd.max_scale, min_scale=npd.min_scale, max_dimensions=npd.MAX_DIMENSIONS)
    for B in [b for b in (1, 4, 16) if b <= len(datas)]:
        s, t, h = src[:B].contiguous(), tgt[:B].contiguous(), hyp[:B].contiguous()
        tm = _harness.queued_ms(lambda: ransac9d_pose_many(s, t, h, npd.THRESHOLDS, **kw), 20, 3)
        ts = _harness.queued_ms(lambda: [ransac9d_pose(s[b], t[b], h[b], npd.THRESHOLDS, **kw) for b in range(B)],
                                20, 3)
        print(f"pose search B = {B:2d} (N = {a.n_pts}, 2 x {H}): one launch   {_harness.summary(tm)}")
        print(f"pose search B = {B:2d} (N = {a.n_pts}, 2 x {H}): {B:2d} launches {_harness.summary(ts)}")


if __name__ == "__main__":
    main()
