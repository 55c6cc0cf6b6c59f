"""PointGroup's front and clustering on several frames in one pass against one frame at a time, on the full-resolution
rendered piles of time_pointgroup_many.py (seeds 0 .. B-1), at B = 1, 4 and 8 (m = 16, block_reps 2, synthetic
weights):

  - front + clustering: device_front_many and the batched pointgroup labels against device_front and pointgroup_labels
    per frame, with the network's offsets computed once beforehand; host clock ending in a synchronise;
  - PointGroupPredictor.predict_many against a loop of predict; host clock ending in a synchronise;
  - the split of the per-frame form at B = 1: device time (kernels and copies, summed from torch.profiler in a run of
    its own) against the wall time of the same call, the rest being host round trips, allocation and launch gaps.

The two forms alternate, each is warmed up first, and their outputs are compared bit for bit.

    python scripts/time_pointgroup_front_many.py [--reps 5] [--frames 1 4 8]
"""
import _harness
import argparse
import tempfile
import time

import numpy as np
import torch

from catgrasp_b200 import segment, spconv
from time_pointgroup import _predictor
from time_pointgroup_many import alternate, frame, same


def front_cluster_per_frame(p, datas, offs, bw):
    out = []
    for d, off in zip(datas, offs):
        xo, _, _, _ = p.device_front(d)
        out.append(segment.pointgroup_labels(xo, off, torch.from_numpy(d["cloud_xyz"]).cuda(), bw)[0])
    return torch.cat(out)


def front_cluster_batched(p, datas, offs, bw):
    xo, _, _, _, row_off = p.device_front_many(datas)
    clouds = [torch.from_numpy(d["cloud_xyz"]).cuda().to(torch.float64) for d in datas]
    cloud_off = np.cumsum([0] + [len(c) for c in clouds])
    return segment._pointgroup_labels_cat(xo, torch.cat(offs), row_off, torch.cat(clouds), cloud_off, bw)[0]


def device_ms(fn):
    """Summed device time (kernels, copies, sets) of one call of fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(e.self_device_time_total for e in prof.key_averages()) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--objects", type=int, default=16)
    a = ap.parse_args()
    print("card:", _harness.card())
    datas = [frame(s, a.objects) for s in range(max(a.frames))]
    print(f"{len(datas)} frames of {min(len(d['cloud_xyz']) for d in datas)} to "
          f"{max(len(d['cloud_xyz']) for d in datas)} points")
    bw = segment.MEANSHIFT_BANDWIDTH["nut"]
    with tempfile.TemporaryDirectory() as tmp:
        p = _predictor(16, tmp)
        offs = []
        for d in datas:
            xo, locs, feats, shape = p.device_front(d)
            level, p2v = spconv.index(locs, shape)
            offs.append(p.model.offsets(level, p2v, feats))
        for B in a.frames:
            ds, of = datas[:B], offs[:B]
            t, out = alternate({"per frame": lambda: front_cluster_per_frame(p, ds, of, bw),
                                "batched": lambda: front_cluster_batched(p, ds, of, bw)}, a.reps, _harness.wall_ms)
            print(f"  B = {B} front + clustering  batched == per frame bit for bit: "
                  f"{same(out['per frame'], out['batched'])}")
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
        for name, fn in (("per frame", lambda: front_cluster_per_frame(p, datas[:1], offs[:1], bw)),
                         ("batched", lambda: front_cluster_batched(p, datas[:1], offs[:1], bw))):
            fn()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
            dev = device_ms(fn)
            print(f"  split, one frame, {name}: wall {wall:.1f} ms, device work {dev:.1f} ms, host round trips, "
                  f"allocation and gaps {wall - dev:.1f} ms")


if __name__ == "__main__":
    main()
