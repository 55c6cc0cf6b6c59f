"""Timing of the per-scene kernels (FPS, ball query, grouping, occupancy grid, RANSAC, filter) on one H100."""
import _harness
import time, json
import numpy as np, torch
from catgrasp_b200 import _lib, pointnet2 as pn2, my_cpp
from catgrasp_b200 import grasp_sampler as gs
from catgrasp_b200.aligning import estimate9DTransform
from catgrasp_b200.synthetic import make_mlp_state_dict, make_pile


def timeit(fn, n=10):
    """Host-clock time per call over `n` calls queued back to back, after one warm-up call."""
    def calls():
        for _ in range(n):
            fn()          # each result dropped at once, so the next call reuses its memory
    fn()
    return _harness.wall_ms(calls, 1, 0)[0] / n


def kernel_ms(fn, n=10):
    """CUDA-event time of the kernels alone (inputs resident, no host work in between)."""
    return float(np.mean(_harness.queued_ms(fn, n, 1)))


def main():
    torch.cuda.set_device(0)
    print("card:", _harness.card())
    out = {}
    for N in (20000, 40000):
        sc = make_pile(N, seed=1)
        xyz = torch.from_numpy((sc["cloud_xyz"] - sc["cloud_xyz"].mean(0)).astype(np.float32))[None].cuda()
        start = torch.tensor([0])
        out[f"fps_N{N}_1024_ms"] = timeit(lambda: pn2.farthest_point_sample(xyz, 1024, start_idx=start))
        ctx = _lib.Context.get(0); ctx.use_torch_stream()
        st32 = torch.zeros(1, dtype=torch.int32, device="cuda"); o32 = torch.empty((1, 1024), dtype=torch.int32, device="cuda")
        out[f"fps_N{N}_1024_cluster_kernel_ms"] = kernel_ms(lambda: ctx.check(ctx.lib.cg_fps_dev(ctx.h, _lib.ptr(xyz), 1, N, 1024, _lib.ptr(st32), _lib.ptr(o32))))
        out[f"fps_N{N}_1024_single_cta_kernel_ms"] = kernel_ms(lambda: ctx.check(ctx.lib.cg_fps_single_cta_dev(ctx.h, _lib.ptr(xyz), 1, N, 1024, _lib.ptr(st32), _lib.ptr(o32))))
        idx = pn2.farthest_point_sample(xyz, 1024, start_idx=start)
        new_xyz = pn2.index_points(xyz, idx)
        out[f"ball_query_N{N}_S1024_k32_ms"] = timeit(lambda: pn2.query_ball_point(0.004, 32, xyz, new_xyz))
        out[f"sample_and_group_N{N}_ms"] = timeit(lambda: pn2.sample_and_group(1024, 0.004, 32, xyz, xyz, start_idx=start), n=5)
    # one SA(1024, 0.2, 32) layer [6 -> 64 -> 64 -> 128] on a 20k-point scene (coordinates centred and scaled to the unit cube, as
    # PointNet++ runs them) and one FP layer back onto the dense cloud
    sc = make_pile(20000, seed=1)
    c = sc["cloud_xyz"] - sc["cloud_xyz"].mean(0)
    xyz_n = torch.from_numpy((c / np.abs(c).max()).astype(np.float32).T.copy())[None].cuda()
    nrm_n = torch.from_numpy(sc["cloud_normal"].astype(np.float32).T.copy())[None].cuda()
    sa = pn2.PointNetSetAbstraction(1024, 0.2, 32, 6, [64, 64, 128], False, make_mlp_state_dict([6, 64, 64, 128], seed=1), device=0)
    fp = pn2.PointNetFeaturePropagation(131, [128, 128, 64], make_mlp_state_dict([131, 128, 128, 64], seed=2, conv2d=False), device=0)
    st1 = torch.tensor([0])
    l1x, l1p = sa(xyz_n, nrm_n, start_idx=st1)
    out["sa_1024_r0.2_k32_N20000_ms"] = kernel_ms(lambda: sa(xyz_n, nrm_n, start_idx=st1), n=5)
    out["fp_1024_to_20000_ms"] = kernel_ms(lambda: fp(xyz_n, l1x, nrm_n, l1p), n=5)
    sa_flop = 2.0 * (6 * 64 + 64 * 64 + 64 * 128) * 1024 * 32
    out["sa_mlp_gflop"] = sa_flop / 1e9
    K = np.eye(3)
    t = time.perf_counter(); occ = my_cpp.makeOccupancyGridFromCloudScan(sc["cloud_xyz"], K, 0.001); out["occupancy_20k_1mm_ms"] = (time.perf_counter() - t) * 1e3
    out["occupancy_points"] = int(occ.shape[0])
    rng = np.random.RandomState(0)
    src = np.round(rng.uniform(-0.5, 0.5, (8192, 3)) / 0.01) * 0.01
    T = np.eye(4); T[:3, :3] *= 0.02; T[:3, 3] = [0, 0, 0.7]
    tgt = (T @ np.c_[src, np.ones(8192)].T).T[:, :3] + rng.normal(0, 0.0004, (8192, 3))
    np.random.seed(0)
    t = time.perf_counter(); estimate9DTransform(src, tgt, 0.003, max_iter=10000, max_scale=[0.05] * 3, min_scale=[0.005] * 3, max_dimensions=np.array([1.2] * 3)); out["ransac_10000x8192_total_ms"] = (time.perf_counter() - t) * 1e3
    # K5-scale cone enumeration: ~1M poses, centred on a 10k-point object
    rng = np.random.RandomState(0)
    S = 1024
    surf = rng.uniform(-0.01, 0.01, (S, 3)) + [0, 0, 0.7]
    R0s = np.stack([np.linalg.qr(rng.normal(size=(3, 3)))[0] for _ in range(S)])
    sph = gs.cone_sphere_points(30)
    obj = rng.uniform(-0.01, 0.01, (10000, 3)) + [0, 0, 0.7]
    def run():
        return gs.enumerate_poses(surf, R0s, sph, 0.03, 0.005, 0.002, points_for_center=obj)
    p64, p32 = run(); torch.cuda.synchronize()
    out["cone_poses"] = int(p64.shape[0])
    out["cone_enumerate_center_10k_ms"] = timeit(run, n=5)
    out["cone_enumerate_only_ms"] = timeit(lambda: gs.enumerate_poses(surf, R0s, sph, 0.03, 0.005, 0.002), n=5)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
