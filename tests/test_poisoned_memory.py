"""GPU tests (-m gpu): every entry point writes each byte of scratch and output memory before it reads it.

Nothing under a call is fresh memory.  A context's two workspace arenas (``ws`` for the ``*_dev`` entries' scratch,
``io`` for the ``*_host`` entries' staged copies) only grow and are never cleared, and the Python wrappers take their
outputs from ``torch.empty``, which hands back recycled blocks.  Each case here runs the protocol of ``_protocol``:

1. a warm call, so both arenas reach the case's size;
2. a clean call, whose result A is held to the case's reference (the helpers of the existing tests);
3. for each byte in ``PATTERNS``, every byte of both arenas set to it (``Context.fill_workspaces``) and every CUDA
   tensor from ``torch.empty`` / ``torch.empty_like`` filled with it (the ``poison`` fixture), then the call again:
   the result must equal A bit for bit -- counts, offsets, permutations and the slots the contract defines as unused
   (-1, NaN, zeros, ``order[n_kept:]``) included.  0xFF reads as NaN, as -1 and as all-ones keys; 0x7F as 3.4e38
   and as large positive counts.

``test_big_then_small`` runs each family's largest case, then its smallest without poisoning, and requires the small
case's clean result: what a real call leaves behind, as in a pick that runs fifteen entry points on one context.

Carves and the tests that cover them (``cg_ws_carve`` / ``cg_io_stage`` call sites).  Pieces that hold indices are
named with the step that writes them before any read, so a poisoned index never reaches a kernel:

- cg_net.cu:214 cls_forward_impl (forward, graspq_dev, graspq_host): gmax keys (cleared by cudaMemsetAsync before
  each trunk), f1, f2, T3, T64, logits.  No indices.  Cases ``pointnet-cls-*``, ``pointnet-graspq-*``.
- cg_net.cu:249 seg_forward_impl (forward, nunocs_dev / _host / many): encoder pieces, pf, biasg, y1..y3, logits.  No
  indices.  Cases ``pointnet-seg-*``, ``pointnet-nunocs-*``, ``nets-nunocs-many-*``.
- cg_net.cu:319 graspq_forward_many_dev: encoder pieces, logits.  No indices.  ``nets-graspq-many-*``.
- cg_net.cu:364 / 434 / 479 (io) graspq_host, nunocs_host, nunocs_many_host: ids are copied in from the host before
  the compute step.  ``pointnet-graspq-*``, ``pointnet-nunocs-*``, ``nets-nunocs-many-*``.
- cg_net.cu:414 encoder_probe_dev: a test hook, used only for the references.
- cg_sa.cu:123 run_mlp (shared MLP, grouped MLP + max): two ping-pong activation buffers.  No indices.
  ``pn2-sa-*``, ``pn2-fp-*``.
- cg_sa.cu:214 three_interp without out_idx / out_weight: idx written by three_nn_kernel before three_interp_kernel
  reads it.  ``pn2-interp-scratch``.
- cg_cloud.cu:476 cloud_index_build (one set and many): vin (point ids, written by the key kernel), cid (written by
  the scan), dU / doff (the cell count, written by a kernel; the set offsets, copied from the host).
  ``cloud-*``, ``meanshift-*``.
- cg_cloud.cu:670 nearest_many_dev: qoff, copied from the host first.  ``cloud-many-*``.
- cg_meanshift.cu:368 meanshift (one set and many): vA / vB (seed ids, written by seed_key_kernel and the sorts),
  gid (scan of head), gseed / gcount / nmodes (group_kernel), rseed / supp / kept (written per mode before use).
  ``meanshift-*``.
- cg_spconv.cu:241 spconv index / down (one frame and many): rA / rB (row ids, written by the key kernels and the
  sort), vid (scan), d_off / d_cs (copied from the host).  ``spconv-index-down-*``, ``spconv-many-frames``.
- cg_spconv.cu:512 voxel_mean: rA / rB (written by site_key_kernel and the sort), first / last (cleared by
  cudaMemsetAsync, then written by site_run_kernel).  ``spconv-voxel-mean-*``.
- cg_pick.cu:240 segment_table: cnt / kmin / kmax (seg_init_kernel over all L labels), rank / seg_len
  (seg_order_kernel), pval (seg_points_kernel).  ``pick-table-*``.
- cg_pick.cu:295 rank_grasps: idx (rank_score_kernel).  ``pick-rank-*``.
- cg_ransac.cu:626 ransac9d: out_T per object (written for each valid hypothesis and read only for the winner), keys
  (cleared per launch; a winning key carries a hypothesis index), err (cleared), tmean (voxel means), the kd-tree
  workspaces (hash tables cleared in the kernel).  ``pose-*``.
- cg_ransac.cu:674 / 695 (io) ransac9d_host, ransac9d_kdtree_host: ids copied from the host; out_T cleared before the
  kernel.  ``pose-host-*``, ``pose-kdtree-*``.
- cg_collide.cu:435 (io) filter_grasp_pose_host: no indices.  ``filter-S*``, ``filter-full-hit-queue``.
- cg_occupancy.cu:136 (io) occupancy_from_scan_host: the mask, cleared before occ_mark_kernel.  ``others-occupancy``.

Families and references: PointNet (check_encoder / FoldedNet of test_tc_kernels), batched nets (the single-call
loop and oracle.draw_ref), PointNet++ (oracle.pn2_ref and its float64 shared MLP), cloud (oracle.cloud_ref and
test_cloud_index_many.check_index), mean shift (oracle.meanshift_ref), sparse U-Net (oracle.spconv_ref), pick
(oracle.pick_ref), pose (ransac64 through test_ransac_kernel.check), filter / IK (filter_ref.c and ik_ref), others
(filter_ref.occupancy_ref, the cone and affordance oracles).
"""
import numpy as np
import pytest
import torch

from test_filter_kernel import grids  # noqa: F401
from test_tc_kernels import ENGINES, check_encoder, cls_pair, cuda, probe, seg_pair  # noqa: F401

pytestmark = pytest.mark.gpu

PATTERNS = (0xFF, 0x7F)
_EMPTY, _EMPTY_LIKE = torch.empty, torch.empty_like


# ------------------------------------------------------------------------------------------ protocol
@pytest.fixture
def poison(monkeypatch):
    """poison(byte): from now on every CUDA tensor from torch.empty / torch.empty_like comes back with each byte of
    its storage set to ``byte``; poison(None) stops it.  CPU tensors are untouched; monkeypatch restores torch."""
    state = {"byte": None}

    def filled(fn):
        def wrapper(*args, **kwargs):
            t = fn(*args, **kwargs)
            if state["byte"] is not None and t.is_cuda:
                s = t.untyped_storage()
                if s.nbytes():
                    raw = _EMPTY(0, dtype=torch.uint8, device=t.device)
                    raw.set_(s, 0, (s.nbytes(),))
                    raw.fill_(state["byte"])
            return t
        return wrapper

    monkeypatch.setattr(torch, "empty", filled(_EMPTY))
    monkeypatch.setattr(torch, "empty_like", filled(_EMPTY_LIKE))
    return lambda byte: state.__setitem__("byte", byte)


def _host(r):
    """The results as host data (synchronises): tensors and arrays copied, containers kept."""
    if isinstance(r, torch.Tensor):
        return r.detach().cpu().numpy().copy()
    if isinstance(r, np.ndarray):
        return r.copy()
    if isinstance(r, dict):
        return {k: _host(v) for k, v in r.items()}
    if isinstance(r, (tuple, list)):
        return [_host(v) for v in r]
    return np.asarray(r)


def _assert_same(a, b, where=""):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), where
        for k in a:
            _assert_same(a[k], b[k], f"{where}/{k}")
    elif isinstance(a, list):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, f"{where}/{i}")
    else:
        a, b = np.asarray(a), np.asarray(b)
        assert a.dtype == b.dtype and a.shape == b.shape, (where, a.dtype, b.dtype, a.shape, b.shape)
        assert a.tobytes() == b.tobytes(), (where, int((a.reshape(-1) != b.reshape(-1)).sum()) if a.size else 0)


def _ctx():
    from catgrasp_b200 import _lib
    return _lib.Context.get(0)


def _protocol(poison, run, check=None):
    """Warm call, clean call A (held to check(A)), then each pattern over both arenas and the outputs: A again."""
    ctx = _ctx()
    _host(run())
    A = _host(run())
    if check is not None:
        check(A)
    for byte in PATTERNS:
        torch.cuda.synchronize()
        ctx.fill_workspaces(byte)
        poison(byte)
        try:
            got = _host(run())
        finally:
            poison(None)
        _assert_same(A, got, f"pattern 0x{byte:02X}")
    return A


def _cu(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)


# ------------------------------------------------------------------------------------------ cases
# Each builder takes the fixtures dict and returns (run, check): run() makes the call and returns its outputs, check(A)
# holds the clean result to the reference.  A family's cases are listed smallest first, largest last.
CASES = {}


def case(family, label, **params):
    def deco(fn):
        CASES[f"{family}-{label}"] = (family, fn, params)
        return fn
    return deco


# PointNet cls / seg --------------------------------------------------------------------------------------------
def _engine_run(engine, call):
    def run():
        _ctx().set_engine(engine)
        try:
            return call()
        finally:
            _ctx().set_engine(3)
    return run


for _e in ENGINES:
    for _B, _N in ((1, 1), (9, 255), (9, 257), (131, 256)):
        @case("pointnet", f"cls-B{_B}-N{_N}-e{_e}", engine=_e, B=_B, N=_N)
        def _cls(fx, engine, B, N):
            net, ref = fx["cls_pair"]
            x = np.random.RandomState(B * 7 + N).normal(0, 1, (B, N, 6)).astype(np.float32)

            def check(A):
                net.ctx.set_engine(engine)
                try:
                    check_encoder(ref, engine, probe(net, B, N, x=x), x, logits=A[0], label="poisoned cls")
                finally:
                    net.ctx.set_engine(3)
            return _engine_run(engine, lambda: net.forward(x, return_probs=True)), check

    for _B, _N, _k in ((2, 3, "rows"), (4, 300, "tiled"), (5, 431, "tc"), (17, 129, "tc")):
        @case("pointnet", f"seg-B{_B}-N{_N}-{_k}-e{_e}", engine=_e, B=_B, N=_N)
        def _seg(fx, engine, B, N):
            net, ref = fx["seg_pair"]
            x = np.random.RandomState(B * 11 + N).normal(0, 1, (B, N, 6)).astype(np.float32)

            def check(A):
                net.ctx.set_engine(engine)
                try:
                    check_encoder(ref, engine, probe(net, B, N, x=x, want_pf=True), x, logits=A, label="poisoned seg")
                finally:
                    net.ctx.set_engine(3)
            return _engine_run(engine, lambda: net.forward(x)), check

    @case("pointnet", f"graspq-B131-N255-e{_e}", engine=_e)
    def _graspq(fx, engine):
        from catgrasp_b200.synthetic import make_candidates, make_pile
        from oracle.encoder_ref import fused_input
        net, ref = fx["cls_pair"]
        B, N, M = 131, 255, 400
        scene = make_pile(M, n_objects=3, seed=41)
        xyz, nrm = scene["cloud_xyz"], scene["cloud_normal"]
        poses = make_candidates(xyz, nrm, B, seed=42)
        rng = np.random.RandomState(43)
        ids = rng.randint(0, M, (B, N)).astype(np.int32)
        mean = np.concatenate([rng.normal(0, 0.002, 3), rng.normal(0, 0.05, 3)])
        std = np.concatenate([rng.uniform(0.008, 0.012, 3), rng.uniform(0.5, 0.6, 3)])
        d = [_cu(a, t) for a, t in ((xyz, torch.float64), (nrm, torch.float64), (poses, torch.float64),
                                    (ids, torch.int32), (mean, torch.float64), (std, torch.float64))]

        def call():
            return net.graspq_dev(*d), net.graspq_host(xyz, nrm, poses, ids, mean, std)

        def check(A):
            _assert_same(A[0], A[1], "graspq dev vs host")
            net.ctx.set_engine(engine)
            try:
                got = probe(net, B, N, fused=(xyz, nrm, poses, ids, mean, std))
            finally:
                net.ctx.set_engine(3)
            x, ex = fused_input(xyz, nrm, poses, ids, mean, std)
            check_encoder(ref, engine, got, x, ex, label="poisoned graspq")
        return _engine_run(engine, call), check

    @case("pointnet", f"nunocs-N257-e{_e}", engine=_e)
    def _nunocs(fx, engine):
        net, _ = fx["seg_pair"]
        x = np.random.RandomState(257).normal(0, 1, (257, 6)).astype(np.float32)

        def call():
            return net.nunocs_dev(x, 100), net.nunocs_host(x, 100), net.forward(x[None])

        def check(A):
            _assert_same(A[0], A[1], "nunocs dev vs host")
            lg = A[2][0].reshape(257, 3, 100)
            np.testing.assert_array_equal(A[0][2], lg.argmax(-1))
        return _engine_run(engine, call), check


# batched nets --------------------------------------------------------------------------------------------------
for _groups in ((1,), (1, 7, 9, 64, 3, 2)):
    @case("nets", f"graspq-many-{len(_groups)}groups", groups=_groups)
    def _graspq_many(fx, groups):
        from catgrasp_b200.synthetic import make_candidates, make_pile
        net, _ = fx["cls_pair"]
        B, N, M = sum(groups), 128, 500
        scene = make_pile(M, n_objects=3, seed=51)
        xyz, nrm = scene["cloud_xyz"], scene["cloud_normal"]
        poses = make_candidates(xyz, nrm, B, seed=52)
        ids = np.random.RandomState(53).randint(0, M, (B, N)).astype(np.int32)
        d = [_cu(a, t) for a, t in ((xyz, torch.float64), (nrm, torch.float64), (poses, torch.float64),
                                    (ids, torch.int32))]

        def check(A):
            r = np.cumsum((0,) + tuple(groups))
            for a, b in zip(r[:-1], r[1:]):
                p, lab = net.graspq_dev(d[0], d[1], d[2][a:b].contiguous(), d[3][a:b].contiguous())
                _assert_same(A[0][a:b], p.cpu().numpy(), f"rows {a}:{b}")
                _assert_same(A[1][a:b], lab.cpu().numpy(), f"labels {a}:{b}")
        return lambda: net.graspq_many_dev(*d, groups), check


@case("nets", "draw-ids-many")
def _draw_many(fx):
    from test_graspq_many import _draw_ids_many_ref
    net, _ = fx["cls_pair"]
    args = ([10, 500, 3, 1000, 7], 128, [0, 1, 5, 300, 0], [1, 2, 3, 4, 5], [0, 10, 510, 513, 1513])
    return (lambda: net.draw_ids_many_dev(*args)), (lambda A: _assert_same(A, _draw_ids_many_ref(*args), "draw"))


for _B, _N in ((1, 257), (3, 40), (65535, 64)):
    @case("nets", f"nunocs-many-B{_B}-N{_N}", B=_B, N=_N)
    def _nunocs_many(fx, B, N):
        net, _ = fx["seg_pair"]
        x = np.random.RandomState(B + N).normal(0, 1, (B, N, 6)).astype(np.float32)
        xd = _cu(x, torch.float32)
        small = B * N < 10000

        def call():
            return (net.nunocs_many_dev(xd, 100),) + ((net.nunocs_many_host(x, 100),) if small else ())

        def check(A):
            if small:
                _assert_same(A[0], A[1], "many dev vs host")
            for b in sorted({0, B // 2, B - 1}):
                one = _host(net.nunocs_dev(xd[b], 100))
                for k in range(3):
                    _assert_same(A[0][k][b], one[k], f"object {b} output {k}")
        return call, check


# PointNet++ ----------------------------------------------------------------------------------------------------
@case("pn2", "fps-ball-group")
def _pn2_prims(fx):
    from catgrasp_b200 import pointnet2 as pn2
    from oracle import pn2_ref
    rng = np.random.RandomState(61)
    B, N, S, K = 2, 1000, 64, 33
    xyz = rng.uniform(-0.5, 0.5, (B, N, 3)).astype(np.float32)
    pts = rng.normal(0, 1, (B, N, 5)).astype(np.float32)
    start = np.array([0, N - 1], np.int32)
    x, p, st = _cu(xyz, torch.float32), _cu(pts, torch.float32), _cu(start, torch.int64)

    def call():
        fi = pn2.farthest_point_sample(x, S, start_idx=st)
        new_xyz = pn2.index_points(x, fi)
        bi = pn2.query_ball_point(0.2, K, x, new_xyz)
        return fi, bi, pn2.index_points(p, bi), pn2.square_distance(new_xyz, x)

    def check(A):
        fi = pn2_ref.farthest_point_sample(xyz, S, start)
        np.testing.assert_array_equal(A[0], fi)
        new_xyz = pn2_ref.index_points(xyz, fi)
        bi = pn2_ref.query_ball_point(0.2, K, xyz, new_xyz)
        np.testing.assert_array_equal(A[1], bi)
        _assert_same(A[2], pn2_ref.index_points(pts, bi).astype(np.float32), "grouped points")
        _assert_same(A[3], pn2_ref.square_distance(new_xyz, xyz).astype(np.float32), "square distance")
    return call, check


@case("pn2", "interp-scratch")
def _pn2_interp(fx):
    from catgrasp_b200 import _lib
    from oracle import pn2_ref
    rng = np.random.RandomState(62)
    B, N, S, D1, D2 = 2, 129, 33, 3, 17
    xyz1, xyz2 = rng.uniform(-1, 1, (B, N, 3)).astype(np.float32), rng.uniform(-1, 1, (B, S, 3)).astype(np.float32)
    p1, p2 = rng.normal(0, 1, (B, N, D1)).astype(np.float32), rng.normal(0, 1, (B, S, D2)).astype(np.float32)
    t = [_cu(a, torch.float32) for a in (xyz1, xyz2, p1, p2)]

    def call():
        out = torch.empty((B, N, D1 + D2), dtype=torch.float32, device="cuda")
        ctx = _lib.Context.get(0)
        ctx.call("cg_three_interp_dev", ctx.h, t[0], t[1], t[2], D1, t[3], D2, B, N, S, out, None, None)
        return out

    def check(A):
        ridx, rw = pn2_ref.three_nn(xyz1, xyz2)
        ref = pn2_ref.three_interp(p1, p2, ridx, rw)
        assert np.array_equal(np.isnan(A), np.isnan(ref)) and np.array_equal(A[~np.isnan(A)], ref[~np.isnan(ref)])
    return call, check


for _name, (_B, _N, _D, _np_, _r, _ns, _mlp) in {"sa-small": (1, 200, 3, 4, 0.3, 8, [64, 48]),
                                                  "sa-partial-tile": (2, 500, 3, 37, 0.3, 16, [64, 64, 128])}.items():
    @case("pn2", _name, B=_B, N=_N, D=_D, npoint=_np_, radius=_r, nsample=_ns, mlp=_mlp)
    def _sa(fx, B, N, D, npoint, radius, nsample, mlp):
        from catgrasp_b200.pointnet2 import PointNetSetAbstraction
        from catgrasp_b200.synthetic import make_mlp_state_dict
        from oracle import pn2_ref
        from oracle.encoder_ref import bound_ratio
        rng = np.random.RandomState(N + 63)
        xyz = rng.uniform(-0.5, 0.5, (B, N, 3)).astype(np.float32)
        pts = rng.normal(0, 1, (B, N, D)).astype(np.float32)
        sd = make_mlp_state_dict([3 + D] + mlp, seed=N, conv2d=True)
        sa = PointNetSetAbstraction(npoint, radius, nsample, 3 + D, mlp, False, sd, device=0)
        start = np.arange(B) * 7 % N
        x, p = _cu(xyz, torch.float32).permute(0, 2, 1), _cu(pts, torch.float32).permute(0, 2, 1)
        fx["keep"].append(sa)

        def check(A):
            new_xyz, grouped, _, _ = pn2_ref.sample_and_group(npoint, radius, nsample, xyz, pts, start)
            np.testing.assert_array_equal(A[0].transpose(0, 2, 1), new_xyz)
            G, K = B * npoint, nsample
            want, err = pn2_ref.SharedMLP64(sd, len(mlp)).group_max(grouped.reshape(G, K, -1), 1)
            assert bound_ratio(A[1].transpose(0, 2, 1).reshape(G, -1), want, err).max() <= 1.0
        return _engine_run(1, lambda: sa(x, p, start_idx=start)), check


@case("pn2", "fp-interp-mlp")
def _fp(fx):
    from catgrasp_b200.pointnet2 import PointNetFeaturePropagation
    from catgrasp_b200.synthetic import make_mlp_state_dict
    from oracle import pn2_ref
    from oracle.encoder_ref import bound_ratio
    rng = np.random.RandomState(64)
    B, N, S, D2, mlp = 2, 300, 50, 64, [64, 48]
    xyz1, xyz2 = rng.uniform(-1, 1, (B, N, 3)).astype(np.float32), rng.uniform(-1, 1, (B, S, 3)).astype(np.float32)
    p2 = rng.normal(0, 1, (B, S, D2)).astype(np.float32)
    sd = make_mlp_state_dict([D2] + mlp, seed=N + S, conv2d=False)
    fp = PointNetFeaturePropagation(D2, mlp, sd, device=0)
    fx["keep"].append(fp)
    args = (_cu(xyz1, torch.float32).permute(0, 2, 1), _cu(xyz2, torch.float32).permute(0, 2, 1), None,
            _cu(p2, torch.float32).permute(0, 2, 1))

    def check(A):
        ridx, rw = pn2_ref.three_nn(xyz1, xyz2)
        np.testing.assert_array_equal(A[1], ridx)
        want, err = pn2_ref.SharedMLP64(sd, len(mlp)).rows(pn2_ref.three_interp(None, p2, ridx, rw).reshape(B * N, -1), 1)
        assert bound_ratio(A[0].transpose(0, 2, 1).reshape(B * N, -1), want, err).max() <= 1.0
    return _engine_run(1, lambda: fp(*args, return_nn=True)), check


# cloud ---------------------------------------------------------------------------------------------------------
def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


for _n, _nn in ((1, 1), (3000, 64)):
    @case("cloud", f"one-set-P{_n}-max_nn{_nn}", n=_n, max_nn=_nn)
    def _cloud(fx, n, max_nn):
        from catgrasp_b200 import cloud
        from oracle import cloud_ref
        rng = np.random.RandomState(n + 70)
        pts = rng.uniform(-0.02, 0.02, (n, 3)) + [0, 0, 0.6]
        q = rng.uniform(-0.021, 0.021, (257, 3)) + [0, 0, 0.6]
        nrm = rng.normal(0, 1, (n, 3))
        vs, rad = 0.003, 0.004

        def call():
            ix = cloud.CloudIndex(pts, vs)
            m, mn = ix.voxel_means(nrm)
            d, i = cloud.nearest(pts, q, 0.002)
            ix2 = cloud.CloudIndex(pts, rad)
            return (m, mn, d, i, ix2.within(q, rad, False), ix2.within(q, rad, True),
                    ix2.normals(rad, max_nn, (0.0, 0.0, 0.0), neighbours=True))

        def check(A):
            rm, rn, _ = cloud_ref.voxel_down_sample(pts, vs, nrm)
            _assert_same(A[0], rm, "voxel means")
            _assert_same(A[1], rn, "voxel normals")
            rd, ri = cloud_ref.nearest(pts, q, 0.002)
            _assert_same(A[2], rd, "nearest d")
            assert (A[3] == ri).all()
            assert (A[4].astype(bool) == cloud_ref.within(pts, q, rad, False)).all()
            assert (A[5].astype(bool) == cloud_ref.within(pts, q, rad, True)).all()
            nbr, cnt = cloud_ref.neighbours(pts, rad, max_nn)
            np.testing.assert_array_equal(A[6][2], cnt)
            np.testing.assert_array_equal(A[6][1], nbr)
        return call, check


@case("cloud", "depth2xyz")
def _depth(fx):
    from catgrasp_b200 import cloud
    from oracle import cloud_ref
    K = np.array([[600.0, 0, 63.5], [0, 601.0, 47.5], [0, 0, 1]])
    depth = np.random.RandomState(71).uniform(0.0, 1.2, (97, 129)).astype(np.float32)
    d = _cu(depth, torch.float32)
    return (lambda: cloud.depth2xyzmap(d, K)), (lambda A: _assert_same(A, cloud_ref.depth2xyzmap(depth, K), "xyz"))


for _kind in ("one-point-sets", "top-cell-next-to-next-set"):
    @case("cloud", f"many-{_kind}", kind=_kind)
    def _cloud_many(fx, kind):
        from catgrasp_b200 import cloud
        from test_cloud_index_many import _tables, check_index, check_nearest_many
        rng = np.random.RandomState(72)
        cell = 0.004
        if kind == "one-point-sets":
            sets = [rng.uniform(0, 0.1, (1, 3)), rng.uniform(0, 0.1, (300, 3)), rng.uniform(0, 0.1, (1, 3))]
        else:
            a = rng.uniform(0, 0.05, (200, 3))
            a[0] = a.min(0) - cell / 2 + [cell * 63.999, cell * 63.999, cell * 63.999]
            sets = [a, a.max(0) + rng.uniform(0, 0.05, (150, 3))]
        pts = np.concatenate(sets)
        off = np.cumsum([0] + [len(s) for s in sets])
        qs = [rng.uniform(0, 0.1, (k, 3)) for k in (5, 0, 40)][:len(sets)]
        q = np.concatenate(qs)
        qoff = np.cumsum([0] + [len(s) for s in qs])

        def call():
            ix = cloud.CloudIndex(pts, cell, set_offsets=off)
            return list(_tables(ix)) + list(ix.voxel_means()[:1]) + list(ix.nearest_many(q, qoff, 0.01))

        def check(A):
            check_index(sets, cell)
            check_nearest_many(sets, qs, cell, 0.01)
        return call, check


# mean shift ----------------------------------------------------------------------------------------------------
def _ms_attrs(m):
    return [m.seed_centers_, m.seed_counts_, m.seed_iters_, m.cluster_centers_, m.labels_]


for _name, _mi in (("one-point", 300), ("identical", 300), ("pile-iter0", 0), ("pile-iter1", 1), ("pile", 300)):
    @case("meanshift", _name, name=_name, max_iter=_mi)
    def _ms(fx, name, max_iter):
        from catgrasp_b200 import segment
        from test_meanshift_kernel import _check, _pile
        if name == "one-point":
            X = np.array([[0.1, 0.2, 0.3]])
        elif name == "identical":
            X = np.tile([[0.01, -0.02, 0.5]], (77, 1))
        else:
            X = _pile(3000, 5, 81, 0.6)
        bw = 0.02
        return (lambda: _ms_attrs(segment.MeanShift(bandwidth=bw, max_iter=max_iter).fit(X))), \
            (lambda A: _assert_same(A, _host(_ms_attrs(_check(X, bw, max_iter))), "meanshift vs checked run"))


@case("meanshift", "many-sets")
def _ms_many(fx):
    from catgrasp_b200 import segment
    from test_meanshift_kernel import _pile
    from test_cloud_index_many import check_meanshift_many
    Xs = [np.array([[0.1, 0.2, 0.3]]), np.tile([[0.0, 0.0, 0.5]], (9, 1)), _pile(2000, 4, 82, 0.6)]

    def call():
        return [_ms_attrs(m) for m in segment.MeanShift(bandwidth=0.02, max_iter=300).fit_many(Xs)]

    def check(A):
        got = check_meanshift_many(Xs, 0.02)
        _assert_same(A, _host([_ms_attrs(m) for m in got]), "many vs checked run")
    return call, check


# sparse U-Net --------------------------------------------------------------------------------------------------
for _shape, _n in (((1, 1, 1), 1), ((1, 7, 9), 40), ((13, 11, 12), 3000)):
    @case("spconv", "index-down-" + "x".join(map(str, _shape)), shape=_shape, n=_n)
    def _sp_index(fx, shape, n):
        from catgrasp_b200 import spconv
        from oracle import spconv_ref as R
        from test_spconv_kernels import _coords
        c = _coords(shape, n, n)
        ct = _cu(c, torch.int32)

        def call():
            lv, p2v = spconv.index(ct, shape)
            co, down, up = spconv.down(lv)
            P = co.count()        # coarse rows from the count on are capacity: out_vox is not written there
            return lv.vox, lv.nbr, p2v, co.vox[:P], co.nbr, co.n, down, up

        def check(A):
            vox, p2v, nbr = R.index(c)
            cvox, cnbr, dn, up, _ = R.down(vox, shape)
            V, P = len(vox), len(cvox)
            assert int(A[5][0]) == P
            _assert_same([A[0], A[1], A[2]], [vox.astype(np.int32), nbr, p2v], "fine level")
            _assert_same([A[3][:P], A[4][:P], A[6][:P], A[7]], [cvox.astype(np.int32), cnbr, dn, up], "coarse level")
            assert (A[4][P:] == -1).all() and (A[6][P:] == -1).all()
        return call, check


for _V in (1, 63, 64, 65):
    @case("spconv", f"conv-k3-k1-V{_V}", V=_V)
    def _sp_conv(fx, V):
        from catgrasp_b200 import spconv
        from oracle import spconv_ref as R
        from oracle.encoder_ref import bound_ratio
        from test_spconv_kernels import _bn, _rand, _sites
        _, _, nbr = R.index(_sites(V, V)[0])
        x, W3, W1 = _rand((V, 16), 1), _rand((3, 3, 3, 16, 32), 2, 0.05), _rand((1, 1, 1, 32, 16), 3, 0.2)
        bias, bn = _rand((32,), 4), _bn(16, 5)
        t = [_cu(a, torch.float32) for a in (x, W3, W1, bias)]
        nt, bnt = _cu(nbr, torch.int32), tuple(_cu(a, torch.float32) for a in bn)
        nw = torch.tensor([V], dtype=torch.int32, device="cuda")

        def call():
            y = spconv.conv(t[0], nt, t[1], nw, bn=bnt, bias=t[3])
            return y, spconv.conv(y, None, t[2], nw, residual=t[0])

        def check(A):
            y, ey = R.conv(x, nbr, W3, bn=bn, bias=bias)
            assert bound_ratio(A[0], y, ey).max() <= 1.0
            z, ez = R.conv(A[0], None, W1, residual=x, ex=None)
            assert bound_ratio(A[1], z, ez).max() <= 1.0
        return call, check


@case("spconv", "voxel-mean-head")
def _sp_mean(fx):
    from test_pointgroup_layers import _head, _head_sd
    rng = np.random.RandomState(91)
    N, V, m = 700, 65, 16
    p2v = rng.randint(0, V, N).astype(np.int32)
    p2v[:3] = -1
    feats = rng.normal(0, 1, (N, 3)).astype(np.float32)
    x = rng.normal(0, 1, (V, m)).astype(np.float32)
    sd = _head_sd(m, 92)
    p2v_t, f_t, x_t = _cu(p2v, torch.int32), _cu(feats, torch.float32), _cu(x, torch.float32)

    from test_pointgroup_layers import _head_weights
    nv = torch.tensor([V], dtype=torch.int32, device="cuda")
    hw = [_cu(a, torch.float32) for a in _head_weights(sd)]
    ctx = _ctx()

    def call():
        mean = torch.empty((V, 3), dtype=torch.float32, device="cuda")
        ctx.call("cg_pointgroup_voxel_mean_dev", ctx.h, f_t, N, 3, p2v_t, nv, V, mean)
        site, out = torch.empty((V, 3), device="cuda"), torch.empty((N, 3), device="cuda")
        ctx.call("cg_pointgroup_head_dev", ctx.h, x_t, m, nv, V, *hw, p2v_t, N, site, out)
        return mean, site, out

    def check(A):
        _assert_same(A[1:], _host(list(_head(sd, x, V, p2v))), "head vs NaN-initialised run")
        ref = np.zeros((V, 3), np.float32)
        for v in range(V):
            sel = feats[p2v == v]
            inv = np.float32(1.0) / np.float32(len(sel)) if len(sel) else np.float32(0)
            for r in sel:
                ref[v] = ref[v] + inv * r
        _assert_same(A[0], ref, "voxel mean")
    return call, check


@case("spconv", "many-frames")
def _sp_many(fx):
    from catgrasp_b200 import spconv
    from test_spconv_kernels import _coords
    shapes = [(1, 1, 1), (5, 7, 9), (13, 11, 12)]
    cs = [_cu(_coords(s, n, i), torch.int32) for i, (s, n) in enumerate(zip(shapes, (1, 100, 2000)))]

    def call():
        lv, p2v = spconv.index_many(cs, shapes)
        co, down, up = spconv.down(lv)
        P = co.count()        # coarse rows from the count on are capacity: out_vox / out_frame are not written there
        return lv.vox, lv.nbr, lv.frame, p2v, co.vox[:P], co.nbr, co.frame[:P], co.n, down, up

    def check(A):
        base = 0
        for b, (c, s) in enumerate(zip(cs, shapes)):
            lv, p2v = spconv.index(c, s)
            V = lv.vox.shape[0]
            _assert_same(A[0][base:base + V], lv.vox.cpu().numpy(), f"frame {b} sites")
            nb = lv.nbr.cpu().numpy()
            _assert_same(A[1][base:base + V], np.where(nb >= 0, nb + base, -1).astype(np.int32), f"frame {b} nbr")
            base += V
    return call, check


# pick ----------------------------------------------------------------------------------------------------------
for _M, _L in ((0, 1), (1, 1), (5000, 7), (20000, 512), (20000, 513)):
    @case("pick", f"table-M{_M}-L{_L}", M=_M, L=_L)
    def _table(fx, M, L):
        from catgrasp_b200 import pick
        from test_pick_kernels import _check_table
        rng = np.random.RandomState(M + L)
        labels = rng.randint(0, L, M).astype(np.int64)
        labels[:min(L, M)] = np.arange(min(L, M))
        xyz = rng.uniform(-0.1, 0.1, (M, 3)).astype(np.float32) * rng.uniform(0.01, 1, (L, 3))[labels].astype(np.float32)
        lab, x = _cu(labels, torch.int64), _cu(xyz, torch.float32)

        def check(A):
            if M > 0:
                _check_table(labels, xyz)
            n = int(A["n_kept"][0])
            assert (A["order"][n:] == -1).all() and (A["offsets"][n:] == A["offsets"][n]).all()
        return (lambda: pick.segment_table(lab, x, L)), check


for _G, _C in ((0, 10), (1, 5), (1, 10), (7, 5), (700, 10)):
    @case("pick", f"rank-G{_G}-C{_C}", G=_G, C=_C)
    def _rank(fx, G, C):
        from catgrasp_b200 import pick
        from oracle import pick_ref
        from test_pick_kernels import _softmax_rows
        rng = np.random.RandomState(G + C)
        probs, pt = _softmax_rows(rng, G, C), rng.uniform(0, 1, G)
        pt[: G // 3] = 0.25
        d = (_cu(probs, torch.float32), _cu(pt, torch.float64))

        def check(A):
            for a, r in zip(A, pick_ref.rank_grasps(probs, pt, C + 1)):
                _assert_same(a, np.asarray(r).astype(a.dtype), "rank")
        return (lambda: pick.rank_grasps(*d, C + 1)), check


# pose ----------------------------------------------------------------------------------------------------------
for _N in (4, 129):
    @case("pose", f"host-N{_N}", N=_N)
    def _ransac_host(fx, N):
        from test_ransac_kernel import _exact_case, check, kernel
        rng = np.random.RandomState(N)
        src, tgt = _exact_case(N, rng)
        ids = np.array([rng.choice(N, 4, replace=False) for _ in range(60)], np.int32)
        ids[1] = [0, 0, 1, 2]            # a repeated point: invalid, its T slot is the cleared one
        return (lambda: kernel(src, tgt, ids)), (lambda A: check(src, tgt, ids))

    @case("pose", f"dev-N{_N}", N=_N)
    def _ransac_dev(fx, N):
        from test_ransac_kernel import _exact_case
        from test_ransac_pose import fused, same_as_host
        rng = np.random.RandomState(N + 1)
        src, tgt = _exact_case(N, rng)
        ids = np.array([rng.choice(N, 4, replace=False) for _ in range(120)], np.int32)

        def check(A):
            _assert_same(A[0], _host(same_as_host(src, tgt, ids[:60])), "one threshold")
            for t, sub, thr in ((0, ids[:60], 0.003), (1, ids[60:], 0.005)):
                one = fused(src, tgt, sub, (thr,))
                for k in ("winner", "count", "T", "count_ratio"):
                    assert one[k][0].tobytes() == A[1][k][t].tobytes(), (t, k)
        return (lambda: (fused(src, tgt, ids[:60]), fused(src, tgt, ids, (0.003, 0.005)))), check


@case("pose", "all-invalid")
def _ransac_invalid(fx):
    from test_ransac_kernel import _exact_case, kernel
    from test_ransac_pose import fused
    rng = np.random.RandomState(5)
    src, tgt = _exact_case(129, rng)
    ids = np.array([rng.choice(129, 4, replace=False) for _ in range(50)], np.int32)
    tiny = np.array([1e-6] * 3)

    def check(A):
        ratio, T, valid = A[0]
        assert not valid.any() and not ratio.any() and not T.any()
        assert A[1]["winner"][0] == -1 and A[1]["best_ratio"] == 0.0 and not A[1]["pose"].any()
    return (lambda: (kernel(src, tgt, ids, max_s=tiny), fused(src, tgt, ids, max_s=tiny))), check


@case("pose", "many-objects")
def _ransac_many(fx):
    from catgrasp_b200.aligning import ransac9d_pose_many
    from test_ransac_kernel import _exact_case
    from test_ransac_pose import fused
    from test_ransac_ref import MAX_D, MAX_S, MIN_S
    rng = np.random.RandomState(7)
    B, N, H = 3, 129, 40
    cases = [_exact_case(N, rng) for _ in range(B)]
    src, tgt = np.stack([c[0] for c in cases]), np.stack([c[1] for c in cases])
    ids = np.stack([[rng.choice(N, 4, replace=False) for _ in range(2 * H)] for _ in range(B)]).astype(np.int32)
    d = (_cu(src, torch.float64), _cu(tgt, torch.float64), _cu(ids, torch.int32))

    def check(A):
        for b in range(B):
            one = fused(src[b], tgt[b], ids[b], (0.003, 0.005))
            assert one["record"].tobytes() == A[b].tobytes(), b
    return (lambda: ransac9d_pose_many(*d, (0.003, 0.005), max_scale=MAX_S, min_scale=MIN_S, max_dimensions=MAX_D)), check


@case("pose", "kdtree-host-and-dev")
def _ransac_kd(fx):
    from test_ransac_kdtree import LOOSE, _draws, _pile, check, kd_kernel, kd_pose, pose_equals_host
    src, tgt = _pile(129, 8)
    ids = [_draws(129, 40, 9), _draws(129, 40, 10)]
    thrs, res = (0.003, 0.005), 0.004

    def check_all(A):
        _assert_same(A[0], _host(list(check(src, tgt, ids[0], thrs[0], res, **LOOSE))), "kd host vs oracle")
        _assert_same(A[1], _host(pose_equals_host(src, tgt, ids, thrs, res, **LOOSE)), "kd pose vs host rule")
    return (lambda: (kd_kernel(src, tgt, ids[0], thrs[0], res, **LOOSE),
                     kd_pose(src, tgt, np.r_[ids[0], ids[1]], thrs, res, **LOOSE))), check_all


# filter / IK ---------------------------------------------------------------------------------------------------
def _filter_case(S, empty=False, seed=43):
    from catgrasp_b200.synthetic import make_filter_case
    p1, p2, poses, sym, nocs, c2n, _ = make_filter_case(seed, 48, S)
    if empty:
        p1, p2 = np.zeros((0, 3)), np.zeros((0, 3))
    return p1, p2, poses, sym, nocs, c2n


for _S, _empty in ((1, True), (1, False), (12, False)):
    @case("filter", f"S{_S}" + ("-empty" if _empty else ""), S=_S, empty=_empty)
    def _filter(fx, S, empty):
        from catgrasp_b200 import my_cpp
        from oracle import filter_ref
        p1, p2, poses, sym, nocs, c2n = _filter_case(S, empty)
        gig = fx["grids"]["gig"]
        (do, so), (de, se) = fx["grids"][("padded", "open")], fx["grids"][("padded", "enclosed")]
        args = lambda gp: (gp, sym, nocs, c2n, gig, True, True, so, p1, se, p2)   # noqa: E731
        gd = _cu(np.asarray(poses), torch.float32)

        def call():
            return (my_cpp.filter_grasp_pose_raw(*args(poses), sdf_mode=0),
                    my_cpp.filter_grasp_pose_raw(*args(gd), sdf_mode=0))

        def check(A):
            _assert_same(A[0], A[1], "host vs dev")
            r = filter_ref.filter_ref(poses, sym, nocs, c2n, gig, True, True, 0, do, np.asarray(p1, np.float64), de,
                                      np.asarray(p2, np.float64))
            for a, b in zip(A[0], r):
                assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).astype(a.dtype).view(np.uint8))
        return call, check


@case("filter", "full-hit-queue")
def _filter_queue(fx):
    from catgrasp_b200 import my_cpp
    from catgrasp_b200.my_cpp import voxel_margin
    from test_filter_kernel import BASE, EYE, FINGER, R, _free_points, _pose_at, _run
    gig = fx["grids"]["gig"]
    pose = _pose_at(BASE, gig)[None]
    q = _free_points(1025, np.random.RandomState(7))
    q[1024] = FINGER
    pts = BASE[None] + q @ R.T
    none = np.zeros((0, 3))
    so, se = fx["grids"][("padded", "open")][1], fx["grids"][("padded", "enclosed")][1]

    def call():
        return my_cpp.filter_grasp_pose_raw(pose, [EYE], EYE, EYE, gig, False, False, so, pts, se, none, sdf_mode=0,
                                            sdf_margin=voxel_margin(0.0005))

    def check(A):
        st, off, out = _run(fx["grids"], "padded", pose, pts, none, margin=voxel_margin(0.0005))
        _assert_same(A, _host([st, off, out]), "vs filter_ref")
        assert A[0][0] == 3
    return call, check


@case("filter", "apply-ik")
def _filter_ik(fx):
    from catgrasp_b200 import my_cpp
    from test_ik_kernel import IK_LOWER, IK_UPPER
    p1, p2, poses, sym, nocs, c2n = _filter_case(4, seed=44)
    gig = fx["grids"]["gig"]
    so, se = fx["grids"][("padded", "open")][1], fx["grids"][("padded", "enclosed")][1]
    cam, ee = np.eye(4), np.eye(4)
    cam[:3, 3] = [0.5, 0.0, 0.4]
    gd = _cu(np.asarray(poses), torch.float32)

    def call():
        return my_cpp.filter_grasp_pose_raw(gd, sym, nocs, c2n, gig, True, True, so, p1, se, p2, sdf_mode=0,
                                            ik=(cam, ee, IK_UPPER, IK_LOWER))

    def check(A):
        st, off, out = _host(my_cpp.filter_grasp_pose_raw(gd, sym, nocs, c2n, gig, True, True, so, p1, se, p2,
                                                          sdf_mode=0))
        ik = A[0] == 2
        keep = ~ik
        assert (st[ik] != 1).all() and (A[1][ik] == -1).all() and not A[2][ik].any()
        _assert_same([A[0][keep], A[1][keep], A[2][keep]], [st[keep], off[keep], out[keep]], "non-IK pairs")
    return call, check


@case("filter", "iiwa14-ik-Q333")
def _ik(fx):
    from catgrasp_b200.ik import iiwa14_ik
    from oracle import ik_ref
    from test_ik_kernel import IK_LOWER, IK_UPPER
    q = np.random.RandomState(5).uniform(-1.5, 1.5, (333, 7))
    q[:, 2] = 0
    P = ik_ref.iiwa14_fk(q).astype(np.float32)
    P[7, 0, 3] = np.nan
    Pd = _cu(P, torch.float32)

    def check(A):
        rc, _ = ik_ref.iiwa14_ik(P, IK_UPPER, IK_LOWER)
        assert (A[0] == rc).all() and np.isnan(A[1][7]).all()
    return (lambda: iiwa14_ik(Pd, IK_UPPER, IK_LOWER, solutions=True)), check


# others --------------------------------------------------------------------------------------------------------
@case("others", "occupancy")
def _occ(fx):
    from catgrasp_b200 import my_cpp
    from test_occupancy_geometry import _kernel_vs_oracle, _pile
    pts = _pile(31)
    return (lambda: my_cpp.makeOccupancyGridFromCloudScan(pts, np.eye(3), 0.001)), \
        (lambda A: _assert_same(A, _kernel_vs_oracle(pts, 0.001)[0], "vs occupancy_ref"))


@case("others", "cone-pick-sized")
def _cone(fx):
    from catgrasp_b200 import _lib
    from catgrasp_b200 import grasp_sampler as gs
    from catgrasp_b200.synthetic import make_pile
    from test_cone_kernels import INIT_BITE, _dev, run, tables
    scene = make_pile(2400, n_objects=6, seed=21)
    m = scene["object_id"] == int(np.argmax(np.bincount(scene["object_id"])))
    pts, nrm = scene["cloud_xyz"][m].copy(), scene["cloud_normal"][m].copy()
    np.random.seed(5)
    ids, R0s, sph = gs.cone_frames(pts, nrm, np.inf, 30)
    surf = pts[ids]
    Rs, Ri = tables(sph, np.arange(0, 180, 30))
    depths = np.arange(0, 0.03, 0.002)
    P = len(surf) * (1 + len(Rs) * len(Ri)) * len(depths)
    t = [_dev(a) for a in (surf, R0s, Rs, Ri, depths, pts)]
    ctx = _lib.Context.get(0)

    def call():
        o64 = torch.empty((P, 4, 4), dtype=torch.float64, device="cuda")
        o32 = torch.empty((P, 4, 4), dtype=torch.float32, device="cuda")
        ctx.call("cg_cone_poses_dev", ctx.h, t[0], t[1], len(surf), t[2], len(Rs), t[3], len(Ri), t[4], len(depths),
                 float(INIT_BITE), o64, o32)
        ctx.call("cg_center_grasps_dev", ctx.h, o64, o32, P, t[5], len(pts))
        return o64, o32

    def check(A):
        _assert_same(A, _host(run(ctx, surf, R0s, Rs, Ri, depths, pts)), "vs NaN-initialised run")
    return call, check


for _P in (1, 129):
    @case("others", f"affordance-P{_P}", P=_P)
    def _aff(fx, P):
        from test_affordance_kernel import BOXES, compare, dyadic_cloud, kernel
        rng = np.random.RandomState(P)
        pts, nrm, aff = dyadic_cloud(rng, P)
        cif = np.stack([np.eye(4)] * 9)
        cif[:, :3, 3] = rng.randint(-4, 5, (9, 3)) / 16.0
        dirs = [1, -1]
        args = (cif, pts, nrm, aff, BOXES[:2], dirs, 0.0625)
        return (lambda: kernel(*args)), (lambda A: _assert_same(A, _host(list(compare(*args))), "vs oracle"))


# ------------------------------------------------------------------------------------------ tests
@pytest.fixture(scope="module")
def fx(request, cuda):  # noqa: F811
    """The nets and grids the cases share, made once."""
    out = {"keep": []}

    class _Lazy(dict):
        def __missing__(self, k):
            self[k] = request.getfixturevalue(k)
            return self[k]
    return _Lazy(out)


@pytest.mark.parametrize("name", list(CASES))
def test_poisoned(fx, poison, name):
    family, build, params = CASES[name]
    run, check = build(fx, **params)
    _protocol(poison, run, check)


FAMILIES = sorted({f for f, _, _ in CASES.values()})


@pytest.mark.parametrize("family", FAMILIES)
def test_big_then_small(fx, family):
    names = [n for n, (f, _, _) in CASES.items() if f == family]
    small, big = names[0], names[-1]
    run_s, _ = CASES[small][1](fx, **CASES[small][2])
    run_b, _ = CASES[big][1](fx, **CASES[big][2])
    _host(run_s())
    A = _host(run_s())
    _host(run_b())
    _assert_same(A, _host(run_s()), f"{small} after {big}")
