"""Time PointGroupPredictor.predict on a full-resolution rendered pile (the one time_spconv.py uses), broken into its
stages: the host front (keep mask, 0.5 mm down-sampling and snap, sites; wall clock), the voxelisation (spconv.index,
the six down steps and the voxel mean; wall clock, it synchronises once in index), the U-Net forward and the offset
head (CUDA events), and pointgroup_labels (wall clock).  Also the host time to enqueue the forward against its GPU
time.  Weights are oracle/pointgroup_ref.synthetic_state_dict at m = 16 and m = 32 (block_reps 2); normals all face
the camera (no stage's time depends on their values).  Median of 5 after 2 warm-up runs.

    python scripts/time_pointgroup.py [--objects 16] [--m 16 32]
"""
import _harness
import argparse
import os
import tempfile
import time

import numpy as np
import torch
import yaml

from catgrasp_b200 import pointgroup, spconv, synthetic, weights
from catgrasp_b200.predicter import PointGroupPredictor
from catgrasp_b200.segment import MEANSHIFT_BANDWIDTH, pointgroup_labels
from oracle.pointgroup_ref import synthetic_state_dict

K = _harness.REFERENCE_K


def _predictor(m, tmp):
    cfg = {"downsample_size": 0.0005,
           "GENERAL": {"input_channel": 3, "scale": 500, "full_scale": [128, 999999], "mode": 4},
           "STRUCTURE": {"m": m, "block_residual": True, "block_reps": 2, "use_coords": True}}
    d = os.path.join(tmp, f"m{m}")
    os.makedirs(d)
    with open(os.path.join(d, "config_pointgroup.yaml"), "w") as f:
        yaml.safe_dump(cfg, f)
    sd = synthetic_state_dict(list(weights.pointgroup_keys(m, 2).items()), 0)
    torch.save({"state_dict": {k: torch.from_numpy(v) for k, v in sd.items()}}, os.path.join(d, "best_val.pth.tar"))
    return PointGroupPredictor("nut", artifact_dir=d, device=0)


def stages(p, data):
    """One predict, stage by stage: dict of ms."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    t0 = time.perf_counter()
    xo, locs, feats, shape = p.host_front(data)
    t1 = time.perf_counter()
    dev = p.model.device
    level, p2v = spconv.index(torch.from_numpy(locs).to(dev), shape)
    levels = pointgroup.pyramid(level)
    f = torch.from_numpy(feats).to(dev)
    vf = pointgroup.voxel_mean(level, p2v, f)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    ev[0].record()
    x = p.model.unet(levels, vf)
    t_enq = time.perf_counter()
    ev[1].record()
    off = p.model.head(level, x, p2v)
    ev[2].record()
    torch.cuda.synchronize()
    t3 = time.perf_counter()
    off = off.cpu().numpy()
    pointgroup_labels(xo, off, data["cloud_xyz"], MEANSHIFT_BANDWIDTH[p.class_name])
    t4 = time.perf_counter()
    return {"host front": (t1 - t0) * 1e3, "voxelisation": (t2 - t1) * 1e3, "forward (GPU)": ev[0].elapsed_time(ev[1]),
            "forward enqueue (host)": (t_enq - t2) * 1e3, "head (GPU)": ev[1].elapsed_time(ev[2]),
            "pointgroup_labels": (t4 - t3) * 1e3, "total": (t4 - t0) * 1e3, "points": len(locs),
            "sites": level.count(), "levels": [lv.count() for lv, _, _ in levels]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--objects", type=int, default=16)
    ap.add_argument("--m", type=int, nargs="+", default=[16, 32])
    args = ap.parse_args()
    print("card:", _harness.card())
    depth, _ = synthetic.render_depth(K, *_harness.REFERENCE_HW, n_objects=args.objects, seed=0, bin_size=0.2)
    v, u = np.nonzero(depth >= 0.1)
    z = depth[v, u].astype(np.float64)
    xyz = np.stack([(u - K[0, 2]) * z / K[0, 0], (v - K[1, 2]) * z / K[1, 1], z], 1).astype(np.float32)
    data = {"cloud_xyz": xyz, "cloud_normal": np.tile(np.float32([0, 0, -1]), (len(xyz), 1))}
    print(f"input points {len(xyz)}")
    with tempfile.TemporaryDirectory() as tmp:
        for m in args.m:
            p = _predictor(m, tmp)
            for _ in range(2):
                stages(p, data)
            runs = [stages(p, data) for _ in range(5)]
            r0 = runs[0]
            print(f"m = {m}: {r0['points']} points after the 0.5 mm down-sampling, {r0['sites']} level-1 sites, "
                  f"levels {r0['levels']}")
            for k in ("host front", "voxelisation", "forward (GPU)", "forward enqueue (host)", "head (GPU)",
                      "pointgroup_labels", "total"):
                print(f"  {k:24s} {_harness.summary([r[k] for r in runs])}")


if __name__ == "__main__":
    main()
