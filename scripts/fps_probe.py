"""Developer probe: FPS kernel time (CUDA events) for a cloud size; CG_FPS_CLUSTER=<n> (experiments build) sets the cluster size.

    python scripts/fps_probe.py [N ...]
"""
import _harness
import argparse, os
import numpy as np, torch
from catgrasp_b200 import _lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("N", type=int, nargs="*", default=[4096, 20000], help="cloud sizes")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    print("card:", _harness.card())
    ctx = _lib.Context.get(0); ctx.use_torch_stream()
    for N in a.N:
        xyz = torch.from_numpy(np.random.RandomState(0).uniform(-1, 1, (1, N, 3)).astype(np.float32)).cuda()
        st = torch.zeros(1, dtype=torch.int32, device="cuda"); o = torch.empty((1, 1024), dtype=torch.int32, device="cuda")
        f = lambda: ctx.check(ctx.lib.cg_fps_dev(ctx.h, _lib.ptr(xyz), 1, N, 1024, _lib.ptr(st), _lib.ptr(o)))
        ms = float(np.mean(_harness.queued_ms(f, 10, 1)))
        print(f"cluster={os.environ.get('CG_FPS_CLUSTER','auto')} N={N}: {ms:.3f} ms ({ms/1023*1e3:.2f} us/round)")


if __name__ == "__main__":
    main()
