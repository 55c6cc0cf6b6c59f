"""Times Sdf3D.from_mesh (csrc/cg_sdf_build.cu) on the gripper proxy, the proxy with tessellated faces (~12 k and
~200 k triangles of the same geometry) and the hex nut, at 1 mm and 0.5 mm cells.

One build = the blocking cg_sdf_from_mesh call (host-side Morton sort and snapping, uploads, the three kernels, the
download of the grid for its boundary statistics), bracketed by CUDA events on the stream it runs on; median of
repeats after warm-up.  The brute-force oracle's host time for the same grid is extrapolated from a sample of nodes, as
context.  With culling, going from 12 k to 200 k triangles of the same geometry should cost far less than 16x."""
import _harness
import argparse
import ctypes as C
import time

import numpy as np
import torch

from catgrasp_b200 import _lib
from catgrasp_b200.synthetic import make_gripper_proxy, make_hex_nut_mesh, tessellated_box_mesh
from oracle.sdf_mesh_ref import grid_geometry, node_positions, sdf_mesh_ref


def tessellated_proxy(m):
    V0 = make_gripper_proxy()["open"]["V"]
    Vs, Fs, off = [], [], 0
    for b in range(V0.shape[0] // 8):
        V, F = tessellated_box_mesh(V0[8 * b:8 * b + 8].min(0), V0[8 * b:8 * b + 8].max(0), m)
        Vs.append(V); Fs.append(F + off); off += V.shape[0]
    return np.concatenate(Vs), np.concatenate(Fs).astype(np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=11)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-sample", type=int, default=256)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    print("card:", _harness.card())
    ctx = _lib.Context.get(0)
    ctx.use_torch_stream()
    g = make_gripper_proxy()["open"]
    meshes = [("proxy", g["V"], g["F"]), ("proxy_tess12k", *tessellated_proxy(18)),
              ("proxy_tess200k", *tessellated_proxy(75)), ("hex_nut", *make_hex_nut_mesh(n_seg=480))]
    rng = np.random.RandomState(0)
    times = {}
    print(f"{'mesh':>16} {'res mm':>6} {'cells':>9} {'triangles':>9} {'ms/build':>9} {'spread':>13} {'oracle s (extrap.)':>18}")
    for res in (0.001, 0.0005):
        for name, V, F in meshes:
            V = np.ascontiguousarray(V, np.float64)
            F = np.ascontiguousarray(F, np.int32)
            ms = []
            for it in range(a.warmup + a.repeats):
                h = C.c_void_p()
                t = _harness.synced_ms(lambda: ctx.check(ctx.lib.cg_sdf_from_mesh(
                    ctx.h, _lib.ptr(V), V.shape[0], _lib.ptr(F), F.shape[0], C.c_float(res), 5, C.byref(h))), 1, 0)
                ctx.lib.cg_sdf_destroy(h)          # outside the timed build
                if it >= a.warmup:
                    ms += t
            dims, origin, r32 = grid_geometry(V, res, 5)
            ncell = int(np.prod(dims))
            idx = np.stack([rng.randint(0, d, a.oracle_sample) for d in dims], 1)
            t0 = time.perf_counter()
            sdf_mesh_ref(V, F, node_positions(origin, r32, idx))
            t_or = (time.perf_counter() - t0) * ncell / a.oracle_sample
            med = float(np.median(ms))
            times[(name, res)] = med
            print(f"{name:>16} {res * 1e3:6.1f} {ncell:9d} {F.shape[0]:9d} {med:9.2f} "
                  f"{min(ms):6.2f}-{max(ms):6.2f} {t_or:18.1f}")
    for res in (0.001, 0.0005):
        r = times[("proxy_tess200k", res)] / times[("proxy_tess12k", res)]
        print(f"res {res * 1e3:.1f} mm: 200 k / 12 k triangles (17.4x more) -> {r:.2f}x the build time")


if __name__ == "__main__":
    main()
