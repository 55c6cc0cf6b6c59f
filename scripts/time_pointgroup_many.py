"""PointGroup on several frames in one pass against one frame at a time, on full-resolution rendered piles (the frame
of time_pointgroup.py, under seeds 0 .. B-1), at B = 1, 4 and 8 and m = 16 and 32 (block_reps 2, synthetic weights):

  - the network part, batched (spconv.index_many, the pyramid, one voxel mean, one U-Net forward and one head) against
    the same steps per frame, from the fronts' device tensors; CUDA events around each form, ending in a synchronise;
  - PointGroupPredictor.predict_many against a loop of predict; host clock ending in a synchronise.

The two forms alternate, each is warmed up first, and their outputs are compared bit for bit.

    python scripts/time_pointgroup_many.py [--reps 5] [--frames 1 4 8] [--m 16 32]
"""
import _harness
import argparse
import tempfile

import numpy as np
import torch

from catgrasp_b200 import pointgroup, spconv, synthetic
from time_pointgroup import _predictor

K = _harness.REFERENCE_K


def frame(seed, objects):
    depth, _ = synthetic.render_depth(K, *_harness.REFERENCE_HW, n_objects=objects, seed=seed, bin_size=0.2)
    v, u = np.nonzero(depth >= 0.1)
    z = depth[v, u].astype(np.float64)
    xyz = np.stack([(u - K[0, 2]) * z / K[0, 0], (v - K[1, 2]) * z / K[1, 1], z], 1).astype(np.float32)
    return {"cloud_xyz": xyz, "cloud_normal": np.tile(np.float32([0, 0, -1]), (len(xyz), 1))}


def net_batched(net, fronts):
    level, p2v = spconv.index_many([f[1] for f in fronts], [f[3] for f in fronts])
    return net.offsets(level, p2v, torch.cat([f[2] for f in fronts]))


def net_per_frame(net, fronts):
    out = []
    for _, locs, feats, shape in fronts:
        level, p2v = spconv.index(locs, shape)
        out.append(net.offsets(level, p2v, feats))
    return torch.cat(out)


def same(a, b):
    if isinstance(a, torch.Tensor):
        a, b = a.cpu().numpy(), b.cpu().numpy()
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def alternate(forms, reps, timer):
    """{form: [ms]} with the forms run in turn, `reps` rounds after one warm-up round, and each form's last output."""
    out = {f: fn() for f, fn in forms.items()}
    times = {f: [] for f in forms}
    for _ in range(reps):
        for f, fn in forms.items():
            times[f] += timer(lambda: out.__setitem__(f, fn()), 1, 0)
    return times, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--m", type=int, nargs="+", default=[16, 32])
    ap.add_argument("--objects", type=int, default=16)
    a = ap.parse_args()
    print("card:", _harness.card())
    datas = [frame(s, a.objects) for s in range(max(a.frames))]
    print(f"{len(datas)} frames of {min(len(d['cloud_xyz']) for d in datas)} to "
          f"{max(len(d['cloud_xyz']) for d in datas)} points")
    with tempfile.TemporaryDirectory() as tmp:
        for m in a.m:
            p = _predictor(m, tmp)
            fronts = [p.device_front(d) for d in datas]
            print(f"m = {m}: {min(len(f[1]) for f in fronts)} to {max(len(f[1]) for f in fronts)} points after the "
                  f"0.5 mm down-sampling, shapes {sorted(set(f[3] for f in fronts))}")
            for B in a.frames:
                fr, ds = fronts[:B], datas[:B]
                t, out = alternate({"per frame": lambda: net_per_frame(p.model, fr),
                                    "batched": lambda: net_batched(p.model, fr)}, a.reps, _harness.synced_ms)
                print(f"  B = {B} network  batched == per frame bit for bit: {same(out['per frame'], out['batched'])}")
                for f in t:
                    print(f"    {f:10s} {_harness.summary(t[f])}")
                print(f"    per frame / batched (medians) {np.median(t['per frame']) / np.median(t['batched']):.2f}")
                t, out = alternate({"loop": lambda: [p.predict(d) for d in ds],
                                    "many": lambda: p.predict_many(ds)}, a.reps, _harness.wall_ms)
                eq = all(same(x, y) for x, y in zip(out["loop"], out["many"]))
                print(f"  B = {B} predict  predict_many == loop bit for bit: {eq}")
                for f in t:
                    print(f"    {f:10s} {_harness.summary(t[f])}")
                print(f"    loop / many (medians) {np.median(t['loop']) / np.median(t['many']):.2f}")


if __name__ == "__main__":
    main()
