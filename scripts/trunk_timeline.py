"""Phase timeline of the tensor-core trunk kernel (developer tool, needs an H100).

Builds a developer copy of the library (CG_EXPERIMENTS, in a temporary directory; the package's own build is not
touched), then runs one K2-sized grasp-Q forward (B candidates x N points: the STN3d, STNkd and encoder trunks) per
engine with CG_TRUNK_TIMELINE=1.  Every trunk launch prints one line to stderr: clock64() cycles of one consumer warp
per 128 points (engine 3 runs 256-point tiles, engines 1 and 2 128-point tiles), averaged over the warps of 8 sampled
CTAs, split into
  start   W2 landed (once per CTA, spread over its tiles)
  input   waiting for the helpers to fill the input tile X0, and reading this warp's rows from it
  front   6->64 FMA, L1, L2
  x3      waiting for the other warpgroup to leave the previous tile's L3, storing X3, and the barrier after it
  l3      128->1024 and the max; of which wgmma-wait = waiting for a wgmma group, ring-wait = waiting for W3 slots
and the tensor-busy estimate: the tensor work of 128 points at 2048 dense fp16 / bf16 MAC per clock per SM over their
cycles.  The same line gives the helper warps' cycles per 128 points, averaged over the helper warps of the sampled
CTAs:
  x0 build       gathering the cloud rows, the float64 transform, and storing them into X0
  x0-empty wait  waiting for the consumers to finish reading the previous tile's X0
  t64            converting and storing each candidate's T64 operand image (encoder trunk), with its wait
  fold           the global fold of each finished candidate's max, with its wait
The helpers keep up when x0-empty wait is large beside x0 build and the consumers' input stays small.

    python scripts/trunk_timeline.py [--engines 3,1] [-B 4096] [-N 1024]
"""
import argparse
import os
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--engines", default="3,1")
    ap.add_argument("-B", type=int, default=4096)
    ap.add_argument("-N", type=int, default=1024)
    args = ap.parse_args()

    with tempfile.TemporaryDirectory(prefix="cg_timeline_") as td:
        from catgrasp_b200 import build
        build.NVCC_FLAGS.append("-DCG_EXPERIMENTS")
        build.LIB_DIR = td
        build.LIB = os.path.join(td, "libcatgrasp_b200.so")
        build.build(force=True)
        from catgrasp_b200 import _lib
        _lib.LIB_PATH = build.LIB
        os.environ["CG_TRUNK_TIMELINE"] = "1"

        import numpy as np
        import torch
        from catgrasp_b200.net import PointNetCls
        from catgrasp_b200.synthetic import make_candidates, make_pile, make_state_dict
        torch.cuda.set_device(0)
        net = PointNetCls(make_state_dict("cls", 10, seed=0), device=0)
        scene = make_pile(20000, n_objects=6, seed=3)
        poses = make_candidates(scene["cloud_xyz"], scene["cloud_normal"], args.B, seed=4)
        rng = np.random.default_rng(0)
        ids = np.stack([rng.choice(20000, args.N, replace=False) for _ in range(args.B)]).astype(np.int32)
        for e in [int(x) for x in args.engines.split(",")]:
            net.ctx.set_engine(e)
            for rep in range(2):   # the first forward includes module load and weight upload
                print(f"--- engine {e}, forward {rep}", file=sys.stderr, flush=True)
                net.graspq_host(scene["cloud_xyz"], scene["cloud_normal"], poses, ids)
                torch.cuda.synchronize()
        del net
        shutil.rmtree(td, ignore_errors=True)


if __name__ == "__main__":
    main()
