"""Time the sparse convolution primitives (cg_spconv.cu) on a rendered pile at PointGroup's 2 mm cells: the level
build (after a 0.5 mm down-sampling, as predict does), the six down steps of the U-Net's pyramid, and one
BN + ReLU + SubM k3 layer per level at the widths of an m = 16 / 32 network (level i has i * m channels), both as a
Python call and as the kernel alone (ten launches through the C entry).  CUDA events, median of 20 after 5 warm-up
runs.  Prints the card, its power limit, per-level site counts and the FLOPs of each layer
(2 * present pairs * Cin * Cout).

    python scripts/time_spconv.py [--objects 16] [--m 16]
"""
import _harness
import argparse

import numpy as np
import torch

from catgrasp_b200 import _lib, spconv, synthetic

K = _harness.REFERENCE_K


def _time(fn):
    return float(np.median(_harness.queued_ms(fn, 20, 5)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--objects", type=int, default=16)
    ap.add_argument("--m", type=int, default=16)
    args = ap.parse_args()
    print("card:", _harness.card())
    depth, _ = synthetic.render_depth(K, *_harness.REFERENCE_HW, n_objects=args.objects, seed=0, bin_size=0.2)
    v, u = np.nonzero(depth >= 0.1)
    z = depth[v, u].astype(np.float64)
    xyz = np.stack([(u - K[0, 2]) * z / K[0, 0], (v - K[1, 2]) * z / K[1, 1], z], 1)
    xyz = np.unique(np.floor(xyz / 0.0005), axis=0) * 0.0005 * 500    # predict's 0.5 mm down-sampling, then scale 500
    locs = (xyz - xyz.min(0)).astype(np.int64)
    shape = tuple(int(max(s, 128)) for s in locs.max(0) + 1)
    c = torch.from_numpy(locs).cuda()
    print(f"points {len(locs)}, spatial shape {shape}")
    t_index = _time(lambda: spconv.index(c, shape))
    levels = [spconv.index(c, shape)[0]]
    for _ in range(6):
        levels.append(spconv.down(levels[-1])[0])
    t_down = _time(lambda: [spconv.down(lv) for lv in levels[:-1]])
    print(f"level build {t_index:.3f} ms (incl. its coordinate check and count synchronisations); "
          f"six down steps {t_down:.3f} ms (incl. Python / ctypes per call)")
    rng = np.random.RandomState(1)
    total_ms = total_flop = 0.0
    for i, lv in enumerate(levels):
        C = (i + 1) * args.m
        V = lv.count()
        pairs = int((lv.nbr[:V] >= 0).sum())
        x = torch.from_numpy(rng.randn(lv.rows, C).astype(np.float32)).cuda()
        W = torch.from_numpy((rng.randn(27, C, C) * 0.05).astype(np.float32)).cuda()
        bn = (torch.ones(C, device="cuda"), torch.zeros(C, device="cuda"))
        call_ms = _time(lambda: spconv.conv(x, lv.nbr, W, lv.n, bn=bn))
        # the kernel alone: ten launches queued through the C entry into one preallocated output, per launch
        ctx, out = _lib.Context.get(x.device.index), torch.empty(lv.rows, C, device="cuda")
        cargs = (ctx.h, x, C, lv.nbr, 27, lv.n, lv.rows, W, C, bn[0], bn[1], None, None, out)
        ms = _time(lambda: [ctx.call("cg_spconv_conv_dev", *cargs) for _ in range(10)]) / 10
        flop = 2.0 * pairs * C * C
        total_ms += ms
        total_flop += flop
        print(f"level {i + 1}: {V:7d} sites ({lv.rows} rows), {pairs:8d} pairs, SubM k3 {C}->{C}: kernel {ms:.4f} ms "
              f"({flop / ms / 1e9:.2f} TFLOP/s), Python call {call_ms:.3f} ms, {flop / 1e9:.3f} GFLOP")
    print(f"one SubM layer per level, kernels: {total_ms:.3f} ms, {total_flop / 1e9:.3f} GFLOP")


if __name__ == "__main__":
    main()
