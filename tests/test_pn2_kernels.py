"""GPU tests (-m gpu) of the PointNet++ kernels (csrc/cg_pn2.cu, csrc/cg_sa.cu) against oracle/pn2_ref.py.

Every comparison is exact (bit for bit) unless a bound is named:
- FPS in every (cluster size, points per thread) configuration cg_fps_dev picks, at the range edges, on clouds with
  exact distance ties everywhere (a shuffled lattice, every point twice), and at its edge cases;
- ball query with points exactly on the sphere, nsample around the 32-lane step and beyond any ball, empty balls;
- square_distance / index_points / group_points off the tile multiples and with empty-ball indices;
- 3-NN and interpolation across the 1024-point sparse tiles, with ties at the 3rd / 4th neighbour and coinciding
  points, against the fp32 contract of three_nn_kernel / three_interp_kernel;
- the SA / FP stacks on engines 0 and 1 within twice the bound of the float64 reference (pn2_ref.SharedMLP64), engine 3
  bit-identical to engine 1; every comparison against a bound prints its largest error / (2 x bound) ratio;
- shared-MLP layers beyond 65535 row tiles (4.19 M rows on the FMA kernel, 8.39 M on tensor cores).
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pn2_ref
from oracle.encoder_ref import bound_ratio, u_bf16x3, u_fp32

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)
    from catgrasp_b200 import _lib
    c = _lib.Context.get(0)
    c.use_torch_stream()
    return c


def _dev(a, dtype=torch.float32):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)


def _ptr(t):
    from catgrasp_b200 import _lib
    return _lib.ptr(t)


def _same(a, b):
    """Same shape and bit pattern (NaN matches NaN whatever its payload)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype.kind == "f":
        a, b = a.astype(np.float32), b.astype(np.float32)
        return bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())
    return bool((a == b).all())


def _lattice(n, rng, side=None):
    """n points of a shuffled integer lattice scaled by 1/16, centred: every coordinate, difference, square and
    expanded-form term is exact in fp32, so equal distances are exactly equal."""
    side = side or int(np.ceil(n ** (1 / 3)))
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3)
    g = g[rng.permutation(len(g))[:n]] - side // 2
    return (g / 16.0).astype(np.float32)


def _twice(n, rng):
    """n / 2 random points, each appearing twice at far-apart indices."""
    p = rng.uniform(-1, 1, (n // 2, 3)).astype(np.float32)
    return np.concatenate([p, p[rng.permutation(n // 2)]])


# ------------------------------------------------------------------------------------------ FPS
def _fps(ctx, xyz, npoint, start, single_cta=False):
    B, N, _ = xyz.shape
    out = torch.full((B, npoint), -7, dtype=torch.int32, device="cuda")
    fn = ctx.lib.cg_fps_single_cta_dev if single_cta else ctx.lib.cg_fps_dev
    ctx.use_torch_stream()
    x, st = _dev(xyz), _dev(start, torch.int32)          # held: a freed temporary's memory would be reused
    ctx.check(fn(ctx.h, _ptr(x), B, N, npoint, _ptr(st), _ptr(out)))
    return out.cpu().numpy()


def _check_fps(ctx, xyz, npoint, start):
    N = xyz.shape[1]
    ref = pn2_ref.farthest_point_sample(xyz, npoint, start)
    got = _fps(ctx, xyz, npoint, start)
    assert np.array_equal(got, ref), (N, pn2_ref.fps_config(N))
    if N <= 56320:
        assert np.array_equal(_fps(ctx, xyz, npoint, start, single_cta=True), ref), N


# one N inside each of the nine (cluster, points per thread) ranges of cg_fps_dev, and both sides of every edge
FPS_SIZES = [1, 777, 2048, 2049, 3000, 4096, 4097, 5000, 5632, 5633, 7000, 8192, 8193, 10000, 13312, 13313, 15000,
             16384, 16385, 20000, 32768, 32769, 50000, 65536, 65537, 100000, 131072]
FPS_CONFIGS = {(2, 4), (2, 8), (2, 16), (4, 8), (4, 16), (8, 8), (8, 16), (8, 32), (16, 32)}
TIE_SIZES = [1000, 3000, 7000, 10000, 20000, 50000, 100000]


def test_fps_sizes_cover_every_launch_config():
    assert {pn2_ref.fps_config(n) for n in FPS_SIZES} == FPS_CONFIGS
    assert len({pn2_ref.fps_config(n) for n in TIE_SIZES}) >= 4


def _npoint(N):
    return min(N, 128 if N <= 16384 else 48)    # the numpy oracle costs O(N) per round


@pytest.mark.parametrize("N", FPS_SIZES)
def test_fps_every_config_vs_oracle(ctx, N):
    """B = 3 clouds with starts 0, N - 1 and N / 2."""
    xyz = np.random.RandomState(N).uniform(-1, 1, (3, N, 3)).astype(np.float32)
    _check_fps(ctx, xyz, _npoint(N), np.array([0, N - 1, N // 2]))


@pytest.mark.parametrize("N", TIE_SIZES)
def test_fps_exact_ties(ctx, N):
    """Ties everywhere: the first maximum (lowest index) must win in the thread, the warp, the CTA and the cluster."""
    rng = np.random.RandomState(N + 1)
    lat = np.stack([_lattice(N, rng) for _ in range(3)])
    _check_fps(ctx, lat, _npoint(N), np.array([0, N - 1, N // 3]))
    two = np.stack([_twice(N, rng) for _ in range(3)])
    _check_fps(ctx, two, _npoint(N), np.array([N - 1, 0, N // 2 + 1]))


def test_fps_edges(ctx):
    """npoint = 1; npoint > N (all distances 0: index 0 repeats, as in the reference); N = 1; N above the limit."""
    from catgrasp_b200 import _lib
    rng = np.random.RandomState(11)
    xyz = rng.uniform(-1, 1, (3, 3000, 3)).astype(np.float32)
    _check_fps(ctx, xyz, 1, np.array([5, 0, 2999]))
    small = rng.uniform(-1, 1, (2, 5, 3)).astype(np.float32)
    ref = pn2_ref.farthest_point_sample(small, 12, np.array([3, 4]))
    assert (ref[:, 5:] == 0).all()
    _check_fps(ctx, small, 12, np.array([3, 4]))
    _check_fps(ctx, rng.uniform(-1, 1, (3, 1, 3)).astype(np.float32), 4, np.array([0, 0, 0]))
    big = torch.zeros((1, 131073, 3), device="cuda")
    out = torch.zeros((1, 4), dtype=torch.int32, device="cuda")
    rc = ctx.lib.cg_fps_dev(ctx.h, _ptr(big), 1, 131073, 4, None, _ptr(out))
    assert rc == _lib.CG_EINVAL and b"fps: N too large" in ctx.lib.cg_last_error(ctx.h)
    rc = ctx.lib.cg_fps_dev(ctx.h, _ptr(big), 1, 131072, 4, None, _ptr(out))
    assert rc == _lib.CG_OK, ("131072 points need the 16-CTA cluster, which this device does not co-schedule: "
                              + ctx.lib.cg_last_error(ctx.h).decode())


# ------------------------------------------------------------------------------------------ ball query
def _ball(ctx, radius, nsample, xyz, new_xyz):
    from catgrasp_b200 import pointnet2 as pn2
    return pn2.query_ball_point(radius, nsample, _dev(xyz), _dev(new_xyz)).cpu().numpy()


@pytest.mark.parametrize("N", [1, 31, 33, 1000])
@pytest.mark.parametrize("nsample", [1, 31, 32, 33, 64, 300])
def test_ball_query_boundary_vs_oracle(ctx, N, nsample):
    """r = 0.25 on a lattice of spacing 1/16: points at exactly d^2 = r^2 (d^2 <= r^2 is in the ball); 300 is more
    than any ball holds (257 lattice points); centroids far away have empty balls (N in every slot); B = 2 clouds."""
    rng = np.random.RandomState(N * 7 + nsample)
    xyz = np.stack([_lattice(N, rng, side=10), _lattice(N, rng, side=10)])
    on_sphere = xyz[:, :1] + np.array([0.25, 0, 0], np.float32)        # point 0 lies exactly on its sphere
    cent = np.concatenate([xyz[:, rng.randint(0, N, 40)], np.full((2, 3, 3), 5.0, np.float32), on_sphere], axis=1)
    ref = pn2_ref.query_ball_point(0.25, nsample, xyz, cent)
    d = np.stack([pn2_ref.sq_expanded(cent[b], xyz[b]) for b in range(2)])
    assert (d[:, 43, 0] == np.float32(0.0625)).all() and (ref[:, 43, 0] == 0).all()
    assert (ref[:, 40:43] == N).all()
    assert np.array_equal(_ball(ctx, 0.25, nsample, xyz, cent), ref)


# ------------------------------------------------------------------------------------------ dense helpers
@pytest.mark.parametrize("S,N", [(1, 1), (65, 257), (130, 1000), (64, 256)])
def test_square_distance_index_group_points(ctx, S, N):
    from catgrasp_b200 import pointnet2 as pn2
    B = 3
    rng = np.random.RandomState(S + N)
    xyz = rng.uniform(-1, 1, (B, N, 3)).astype(np.float32)
    src = rng.uniform(-1, 1, (B, S, 3)).astype(np.float32)
    assert _same(pn2.square_distance(_dev(src), _dev(xyz)).cpu().numpy(), pn2_ref.square_distance(src, xyz))
    K = 5
    idx = rng.randint(0, N + 1, (B, S, K)).astype(np.int32)            # N marks an empty ball
    idx[:, 0, :] = N
    for D in (0, 7):
        pts = rng.normal(0, 1, (B, N, D)).astype(np.float32) if D else None
        valid = idx < N
        safe = np.where(valid, idx, 0)
        want = np.stack([xyz[b][safe[b]] - src[b][:, None] for b in range(B)]).astype(np.float32)
        if D:
            want = np.concatenate([want, np.stack([pts[b][safe[b]] for b in range(B)])], -1)
        want[~valid] = 0.0
        out = torch.full((B, S, K, 3 + D), float("nan"), device="cuda")
        ctx.use_torch_stream()
        t = [_dev(xyz), _dev(pts), _dev(src), _dev(idx, torch.int32)]
        ctx.check(ctx.lib.cg_group_points_dev(ctx.h, *map(_ptr, t), B, N, D, S, K, _ptr(out)))
        assert _same(out.cpu().numpy(), want), D
    feats = rng.normal(0, 1, (B, N, 9)).astype(np.float32)
    flat = idx.reshape(B, -1)
    want = np.stack([feats[b][np.where(flat[b] < N, flat[b], 0)] for b in range(B)])
    want[flat == N] = 0.0
    assert _same(pn2.index_points(_dev(feats), _dev(flat, torch.int64)).cpu().numpy(), want)


# ------------------------------------------------------------------------------------------ 3-NN / interpolation
def _interp(ctx, xyz1, xyz2, p1, p2):
    B, N, _ = xyz1.shape
    S, D2 = p2.shape[1], p2.shape[2]
    D1 = 0 if p1 is None else p1.shape[2]
    out = torch.full((B, N, D1 + D2), float("nan"), device="cuda")
    idx = torch.full((B, N, 3), -7, dtype=torch.int32, device="cuda")
    w = torch.full((B, N, 3), float("nan"), device="cuda")
    ctx.use_torch_stream()
    t = [_dev(xyz1), _dev(xyz2), _dev(p1), _dev(p2)]
    ctx.check(ctx.lib.cg_three_interp_dev(ctx.h, _ptr(t[0]), _ptr(t[1]), _ptr(t[2]), D1, _ptr(t[3]), D2, B, N, S,
                                          _ptr(out), _ptr(idx), _ptr(w)))
    return out.cpu().numpy(), idx.cpu().numpy(), w.cpu().numpy()


def _check_interp(ctx, xyz1, xyz2, p1, p2):
    out, idx, w = _interp(ctx, xyz1, xyz2, p1, p2)
    ridx, rw = pn2_ref.three_nn(xyz1, xyz2)
    k = ridx.shape[2]
    assert np.array_equal(idx[:, :, :k], ridx)
    assert _same(w[:, :, :k], rw)
    if k == 2:                                         # S = 2: the third slot is index 0 with weight 0
        assert (idx[:, :, 2] == 0).all() and (w[:, :, 2] == 0).all()
    assert _same(out, pn2_ref.three_interp(p1, p2, ridx, rw))
    return ridx


NN_CASES = [(2, 129, 0, 33), (3, 1, 4, 1), (4, 127, 0, 256), (1023, 129, 3, 33), (1024, 127, 0, 1),
            (1025, 129, 16, 33), (1025, 1, 0, 256), (3000, 5000, 0, 33), (3000, 127, 8, 256), (2, 1, 5, 1)]


@pytest.mark.parametrize("S,N,D1,D2", NN_CASES)
def test_three_nn_interp_vs_oracle(ctx, S, N, D1, D2):
    rng = np.random.RandomState(S * 31 + N)
    B = 2
    xyz2 = rng.uniform(-1, 1, (B, S, 3)).astype(np.float32)
    xyz1 = rng.uniform(-1, 1, (B, N, 3)).astype(np.float32)
    p1 = rng.normal(0, 1, (B, N, D1)).astype(np.float32) if D1 else None
    p2 = rng.normal(0, 1, (B, S, D2)).astype(np.float32)
    _check_interp(ctx, xyz1, xyz2, p1, p2)


@pytest.mark.parametrize("S", [4, 1500, 3000])
def test_three_nn_lattice_ties(ctx, S):
    """Sparse points on a lattice, dense points on lattice points, edge midpoints, face centres and cell centres:
    ties at every rank, in particular between the 3rd and 4th neighbour, across the sparse tiles."""
    rng = np.random.RandomState(S)
    B, N = 2, 600
    xyz2 = np.stack([_lattice(S, rng, side=max(2, int(np.ceil(S ** (1 / 3))))) for _ in range(B)])
    base = xyz2[:, rng.randint(0, S, N)]
    half = np.float32(1 / 32)
    off = (rng.randint(0, 2, (B, N, 3)) * half).astype(np.float32)
    xyz1 = (base + off).astype(np.float32)
    p2 = rng.normal(0, 1, (B, S, 33)).astype(np.float32)
    ridx = _check_interp(ctx, xyz1, xyz2, rng.normal(0, 1, (B, N, 2)).astype(np.float32), p2)
    if S >= 1500:
        d = np.stack([np.sort(pn2_ref.sq_expanded(xyz1[b], xyz2[b]), 1)[:, 2:4] for b in range(B)])
        assert (d[..., 0] == d[..., 1]).mean() > 0.3           # 3rd / 4th neighbour ties are common
    assert ridx.shape == (B, N, 3)


@pytest.mark.parametrize("S", [3, 1025])
def test_three_nn_coinciding_points(ctx, S):
    """Dense points equal to sparse points: the expanded-form distance is about 0 and may be negative."""
    rng = np.random.RandomState(S + 5)
    B, N = 2, 300
    xyz2 = rng.uniform(-1, 1, (B, S, 3)).astype(np.float32)
    xyz1 = np.concatenate([xyz2[:, rng.randint(0, S, N - 50)], rng.uniform(-1, 1, (B, 50, 3)).astype(np.float32)], 1)
    _check_interp(ctx, xyz1, xyz2, None, rng.normal(0, 1, (B, S, 256)).astype(np.float32))


# ------------------------------------------------------------------------------------------ SA / FP stacks
def _report(label, engine, got, ref, err):
    assert np.isfinite(got).all(), label
    r = float(bound_ratio(got, ref, err).max())
    print(f"\nRATIO engine={engine} {label} = {r:.3g}")
    assert r <= 1.0, (label, engine, r)
    return r


SA_CASES = {   # name: (B, N, D, npoint, radius, nsample, mlp, group_all)
    "rows<64": (1, 200, 3, 4, 0.3, 8, [64, 48], False),
    "rows%128!=0": (2, 500, 3, 37, 0.3, 16, [64, 64, 128], False),
    "K=1": (2, 300, 3, 100, 0.2, 1, [64, 128], False),
    "width48": (2, 400, 3, 64, 0.3, 8, [64, 48], False),
    "width192": (2, 400, 3, 64, 0.3, 8, [64, 192], False),
    "group_all": (2, 300, 61, None, None, None, [128, 256], True),
}


@pytest.mark.parametrize("case", list(SA_CASES))
def test_set_abstraction_vs_float64(ctx, case):
    from catgrasp_b200.pointnet2 import PointNetSetAbstraction
    from catgrasp_b200.synthetic import make_mlp_state_dict
    B, N, D, npoint, radius, nsample, mlp, group_all = SA_CASES[case]
    rng = np.random.RandomState(len(case) * 13 + N)
    xyz = rng.uniform(-0.5, 0.5, (B, N, 3)).astype(np.float32)
    pts = rng.normal(0, 1, (B, N, D)).astype(np.float32)
    dims = [3 + D] + mlp
    sd = make_mlp_state_dict(dims, seed=N + len(mlp), conv2d=True)
    sa = PointNetSetAbstraction(npoint, radius, nsample, 3 + D, mlp, group_all, sd, device=0)
    ref = pn2_ref.SharedMLP64(sd, len(mlp))
    start = np.arange(B) * 7 % N
    if group_all:
        grouped = np.concatenate([xyz, pts], -1)[:, None]
    else:
        new_xyz, grouped, _, _ = pn2_ref.sample_and_group(npoint, radius, nsample, xyz, pts, start)
    G, K = B * grouped.shape[1], grouped.shape[2]
    got = {}
    for engine in (0, 1, 3):
        ctx.set_engine(engine)
        try:
            gx, gp = sa(_dev(xyz).permute(0, 2, 1), _dev(pts).permute(0, 2, 1), start_idx=start)
        finally:
            ctx.set_engine(3)
        got[engine] = gp.permute(0, 2, 1).reshape(G, -1).cpu().numpy()
        if not group_all:
            assert np.array_equal(gx.permute(0, 2, 1).cpu().numpy(), new_xyz)
        if engine < 3:
            want, err = ref.group_max(grouped.reshape(G, K, -1), engine)
            tc = ref.on_tc(engine, G * K)
            _report(f"SA {case} G={G} K={K} dims={dims} tc={tc}", engine, got[engine], want, err)
    assert np.array_equal(got[3].view(np.uint32), got[1].view(np.uint32))


FP_CASES = {   # name: (B, N, S, D1, D2, mlp)
    "D1=0": (2, 300, 50, 0, 64, [64, 48]),
    "S=1": (2, 200, 1, 16, 48, [128]),
    "S=2": (2, 150, 2, 0, 64, [64, 64]),
    "S=2 D1>0": (1, 40, 2, 5, 59, [192]),
}


@pytest.mark.parametrize("case", list(FP_CASES))
def test_feature_propagation_vs_float64(ctx, case):
    from catgrasp_b200.pointnet2 import PointNetFeaturePropagation
    from catgrasp_b200.synthetic import make_mlp_state_dict
    B, N, S, D1, D2, mlp = FP_CASES[case]
    rng = np.random.RandomState(N + S)
    xyz1 = rng.uniform(-1, 1, (B, N, 3)).astype(np.float32)
    xyz2 = rng.uniform(-1, 1, (B, S, 3)).astype(np.float32)
    p1 = rng.normal(0, 1, (B, N, D1)).astype(np.float32) if D1 else None
    p2 = rng.normal(0, 1, (B, S, D2)).astype(np.float32)
    dims = [D1 + D2] + mlp
    sd = make_mlp_state_dict(dims, seed=N + S, conv2d=False)
    fp = PointNetFeaturePropagation(D1 + D2, mlp, sd, device=0)
    ref = pn2_ref.SharedMLP64(sd, len(mlp))
    if S == 1:
        feat = np.repeat(p2, N, axis=1)
        feat = feat if p1 is None else np.concatenate([p1, feat], -1)
    else:
        ridx, rw = pn2_ref.three_nn(xyz1, xyz2)
        feat = pn2_ref.three_interp(p1, p2, ridx, rw)
    got = {}
    for engine in (0, 1, 3):
        ctx.set_engine(engine)
        try:
            args = (_dev(xyz1).permute(0, 2, 1), _dev(xyz2).permute(0, 2, 1),
                    None if p1 is None else _dev(p1).permute(0, 2, 1), _dev(p2).permute(0, 2, 1))
            if S == 1:
                out = fp(*args)
            else:
                out, idx, w = fp(*args, return_nn=True)
                assert idx.shape == (B, N, min(S, 3)) and w.shape == (B, N, min(S, 3))
                assert np.array_equal(idx.cpu().numpy(), ridx) and _same(w.cpu().numpy(), rw)
        finally:
            ctx.set_engine(3)
        got[engine] = out.permute(0, 2, 1).reshape(B * N, -1).cpu().numpy()
        if engine < 3:
            want, err = ref.rows(feat.reshape(B * N, -1), engine)
            _report(f"FP {case} R={B * N} dims={dims} tc={ref.on_tc(engine, B * N)}", engine, got[engine], want, err)
    assert np.array_equal(got[3].view(np.uint32), got[1].view(np.uint32))


# ------------------------------------------------------------------------------------------ beyond 65535 row tiles
def _sample_rows(R, tile):
    """The first two tiles, and the rows from two tiles before the 65536th row tile to the end."""
    edge = 65535 * tile
    return np.concatenate([np.arange(2 * tile), np.arange(edge - 2 * tile, R)])


@pytest.mark.parametrize("R,K,N,engine,tile", [(4194305, 6, 64, 1, 64),      # FMA tiled kernel (64-row tiles)
                                                (8388609, 64, 64, 1, 128)])  # tensor cores (128-row tiles)
def test_shared_mlp_beyond_65535_row_tiles(ctx, R, K, N, engine, tile):
    """One fully-connected + ReLU layer over more rows than gridDim.y can hold in tiles.  A private context, so that
    its multi-GB workspace is released when the test ends."""
    from catgrasp_b200 import _lib
    pc = _lib.Context(0)
    h = C.c_void_p()
    try:
        pc.set_engine(engine)
        pc.use_torch_stream()
        rng = np.random.RandomState(R)
        W = (rng.uniform(-1, 1, (K, N)) / np.sqrt(K)).astype(np.float32)
        b = rng.uniform(-0.1, 0.1, N).astype(np.float32)
        pc.check(pc.lib.cg_mlp_create(pc.h, 1, (C.c_int * 2)(K, N), (C.c_void_p * 1)(W.ctypes.data),
                                      (C.c_void_p * 1)(b.ctypes.data), C.byref(h)))
        gen = torch.Generator(device="cuda").manual_seed(R)
        x = torch.randn((R, K), generator=gen, device="cuda")
        out = torch.full((R, N), float("nan"), device="cuda")
        pc.check(pc.lib.cg_shared_mlp_dev(h, _ptr(x), R, _ptr(out)))
        rows = _sample_rows(R, tile)
        sel = torch.from_numpy(rows).cuda()
        xs, got = x[sel].cpu().numpy().astype(np.float64), out[sel].cpu().numpy()
        assert not torch.isnan(out).any().item()
        del x, out
    finally:
        if h:
            pc.lib.cg_mlp_destroy(h)
        torch.cuda.synchronize()
        pc.lib.cg_ctx_destroy(pc.h)
        torch.cuda.empty_cache()
    tc = engine >= 1 and R >= 64 and K % 64 == 0 and N >= 64
    assert tc == (tile == 128)
    W64 = W.astype(np.float64)
    want = np.maximum(xs @ W64 + b, 0.0)
    err = (u_bf16x3(K) if tc else u_fp32(K)) * (np.abs(xs) @ np.abs(W64) + np.abs(b))
    _report(f"rows R={R} K={K} N={N} {'tc' if tc else 'fma'}", engine, got, want, err)


def test_set_abstraction_beyond_65535_row_tiles(ctx):
    """128 clouds x 1024 centroids x 32 members = 4,194,304 rows > 65535 x 64 on the first (FMA) layer."""
    from catgrasp_b200 import pointnet2 as pn2
    from catgrasp_b200.pointnet2 import PointNetSetAbstraction
    from catgrasp_b200.synthetic import make_mlp_state_dict
    B, N, S, K = 128, 1100, 1024, 32
    rng = np.random.RandomState(2)
    xyz = _dev(rng.uniform(-0.5, 0.5, (B, N, 3)).astype(np.float32))
    pts = _dev(rng.normal(0, 1, (B, N, 3)).astype(np.float32))
    start = np.arange(B) % N
    sd = make_mlp_state_dict([6, 16], seed=3, conv2d=True)
    sa = PointNetSetAbstraction(S, 0.2, K, 6, [16], False, sd, device=0)
    ref = pn2_ref.SharedMLP64(sd, 1)
    ctx.set_engine(1)
    try:
        _, out = sa(xyz.permute(0, 2, 1), pts.permute(0, 2, 1), start_idx=start)
        got = out.permute(0, 2, 1).reshape(B * S, -1)
        _, grouped = pn2.sample_and_group(S, 0.2, K, xyz, pts, start_idx=start)
        groups = _sample_rows(B * S * K, 64)[::K] // K
        groups = np.unique(np.concatenate([groups, groups + 1]).clip(0, B * S - 1))
        sel = torch.from_numpy(groups).cuda()
        gin = grouped.reshape(B * S, K, 6)[sel].cpu().numpy()
        g = got[sel].cpu().numpy()
        del out, got, grouped
    finally:
        ctx.set_engine(3)
    want, err = ref.group_max(gin, 1, rows=B * S * K)
    _report(f"SA rows={B * S * K}", 1, g, want, err)
