"""CPU tests: the C ABI library loads and exports every symbol of include/*.h, host logic,
weight folding, and that the product path fails loudly without a GPU / without the extension."""
import copy
import os
import re

import numpy as np
import pytest
import torch

from catgrasp_b200 import _lib
from catgrasp_b200.synthetic import make_gripper_proxy, make_pile, make_candidates, make_state_dict
from catgrasp_b200.weights import BLOB_ORDER, pack_blob, strip_module_prefix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "catgrasp_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(cg_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from catgrasp_b200 import build
    build.build()
    lib = _lib.load()
    syms = _header_symbols()
    assert len(syms) >= 25
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/catgrasp_b200.h but not exported"
        assert s in _lib.SIGNATURES, f"{s} has no ctypes prototype"
    assert set(_lib.SIGNATURES) == set(syms)
    assert b"sm_90a" in lib.cg_version()


def test_no_cpu_fallback_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.CgError):
        _lib.Context(0)


def test_missing_extension_fails_loudly(monkeypatch):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libcatgrasp_b200.so")
    with pytest.raises(_lib.CgError, match="no CPU fallback"):
        _lib.load()


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "catgrasp_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), f
                assert not re.search(r"#\s*include\s*[<\"][^>\"]*oracle", txt), f      # comments may name the oracle file
                assert not re.search(r"(CDLL|dlopen)\([^)]*oracle", txt), f


@pytest.mark.parametrize("kind,n_out", [("cls", 10), ("seg", 300)])
def test_blob_size_matches_library(kind, n_out):
    lib = _lib.load()
    blob, n = pack_blob(make_state_dict(kind, n_out, seed=3), kind)
    assert n == n_out and blob.dtype == np.float32
    assert blob.size == lib.cg_net_blob_floats(0 if kind == "cls" else 1, n_out)
    assert len(BLOB_ORDER) == 20


def test_bn_folding_matches_conv_bn():
    """Folded (Wt, b) reproduce conv1d + eval BatchNorm (pointnet2.py:171) to fp32 round-off."""
    import torch.nn.functional as F
    from catgrasp_b200.weights import _fold
    sd = strip_module_prefix(make_state_dict("cls", 10, seed=5))
    x = torch.randn(2, 64, 50)
    y = F.conv1d(x, sd["feat.stn.conv2.weight"], sd["feat.stn.conv2.bias"])
    y = F.batch_norm(y, sd["feat.stn.bn2.running_mean"], sd["feat.stn.bn2.running_var"], sd["feat.stn.bn2.weight"],
                     sd["feat.stn.bn2.bias"], training=False, eps=1e-5)
    Wt, b = _fold(sd, "feat.stn.conv2", "feat.stn.bn2")
    y2 = torch.einsum("bkn,kc->bcn", x.double(), torch.from_numpy(Wt)) + torch.from_numpy(b)[None, :, None]
    assert (y.double() - y2).abs().max() < 1e-5


def test_checkpoint_key_check():
    sd = strip_module_prefix(make_state_dict("cls", 10, seed=0))
    bad = copy.copy(sd)
    bad.pop("fc3.bias")
    with pytest.raises(RuntimeError):
        pack_blob(bad, "cls")
    with pytest.raises(RuntimeError):
        pack_blob(sd, "seg")


def test_host_id_draw_consumes_rng_like_reference():
    """draw_subsample_ids == the ids GraspDataset.transform draws (dataset_grasp.py:72-73), candidate by candidate."""
    from catgrasp_b200.predicter import draw_subsample_ids
    from oracle.transforms_ref import grasp_transform
    scene = make_pile(700, n_objects=2, seed=1)
    data = {"cloud_xyz": scene["cloud_xyz"], "cloud_normal": scene["cloud_normal"]}
    for n_pts in (256, 700, 1024):
        np.random.seed(9)
        ref = [grasp_transform(copy.deepcopy(data), np.eye(4), {"n_pts": n_pts})["ids"] for _ in range(3)]
        after_ref = np.random.rand()
        np.random.seed(9)
        ids = draw_subsample_ids(700, n_pts, count=3)
        assert np.random.rand() == after_ref
        assert np.array_equal(ids, np.stack(ref))


def test_sdf_file_layout_roundtrip(tmp_path):
    """sdf_file.py:76-84: values are stored i fastest, k slowest and land in data[i][j][k]."""
    from catgrasp_b200.sdf import parse_sdf_file, write_sdf_file
    rng = np.random.RandomState(0)
    data = rng.normal(size=(4, 5, 6)).astype(np.float32)
    p = str(tmp_path / "g.sdf")
    write_sdf_file(p, data, [0.1, 0.2, 0.3], 0.001)
    d2, origin, res = parse_sdf_file(p)
    assert np.allclose(d2, data, atol=1e-6) and np.allclose(origin, [0.1, 0.2, 0.3]) and res == 0.001
    lines = open(p).read().split("\n")
    assert float(lines[3]) == pytest.approx(float(data[0, 0, 0]), abs=1e-6)
    assert float(lines[4]) == pytest.approx(float(data[1, 0, 0]), abs=1e-6)      # i is the fastest index


def _mm4(A, B):
    O = np.zeros((4, 4), np.float32)
    for r in range(4):
        for c in range(4):
            s = np.float32(A[r, 0] * B[0, c])
            for k in (1, 2, 3):
                s = np.float32(s + np.float32(A[r, k] * B[k, c]))
            O[r, c] = s
    return O


def test_filter_oracle_pose_logic_matches_eigen_order():
    """oracle/filter_ref.c pose arithmetic == an independent numpy fp32 restatement of
    common.cpp:159,190-197,265 (sequential fp32 products, normalise by division, float step values)."""
    from oracle import filter_ref
    rng = np.random.RandomState(0)
    scene = make_pile(400, n_objects=2, seed=2)
    poses = make_candidates(scene["cloud_xyz"], scene["cloud_normal"], 16, seed=3)
    g = make_gripper_proxy()
    far = scene["cloud_xyz"][:50] + 10.0                       # nothing collides: offset 0 must win
    nocs = np.eye(4); nocs[:3, :3] *= np.array([1.0, 1.2, 0.8]); nocs[:3, 3] = [0.01, -0.02, 0.03]
    c2n = np.eye(4); c2n[:3, 3] = rng.normal(0, 0.01, 3)
    sym = np.eye(4); sym[:3, :3] = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]])
    st, off, out = filter_ref.filter_ref(poses, [sym], nocs, c2n, g["gripper_in_grasp"], False, True, 0, g["open"], far,
                                         g["enclosed"], far)
    assert (st == 0).all() and (off == 0).all()
    f = lambda m: np.asarray(m, np.float64).astype(np.float32)
    c2c = _mm4(f(nocs), f(c2n))
    for i in range(len(poses)):
        G = _mm4(c2c, _mm4(f(sym), f(poses[i])))
        for col in range(3):
            x, y, z = G[0, col], G[1, col], G[2, col]
            n = np.sqrt(np.float32(np.float32(np.float32(x * x) + np.float32(y * y)) + np.float32(z * z)))
            G[:3, col] = np.array([x / n, y / n, z / n], np.float32)
        assert np.array_equal(G.view(np.uint32), out[i].view(np.uint32))
    # everything collides -> zero matrices, offset -1, status 3 (common.cpp:289-293)
    inside = (np.linalg.inv(np.eye(4)) @ np.eye(4))[:3, 3][None] + poses[0][:3, 3][None] - 0.035 * poses[0][:3, 0][None]
    st, off, out = filter_ref.filter_ref(poses[:1], [np.eye(4)], np.eye(4), np.eye(4), g["gripper_in_grasp"], False, True,
                                         0, g["open"], np.repeat(inside, 4, 0) - 0.02 * poses[0][:3, 0][None], None,
                                         np.zeros((0, 3)))
    assert st[0] == 3 and off[0] == -1 and (out == 0).all()
    # the float accumulator of common.cpp:255 (SURVEY Appendix A7)
    s1 = np.float32(0.001); s2 = np.float32(s1 + np.float32(0.001)); s3 = np.float32(s2 + np.float32(0.001))
    assert float(s1) == 0.0010000000474974513 and float(s2) == 0.0020000000949949026 and not (float(s3) <= 0.003)


def test_sdf_oracle_fp32_vs_reference_formula():
    """C fp32 trilinear / nearest lookups agree with the float64 restatement of sdf.py:292-359."""
    from oracle import filter_ref, sdf_ref
    g = make_gripper_proxy()["open"]
    rng = np.random.RandomState(1)
    dims = np.array(g["sdf"].shape)
    gc = rng.uniform(-3, dims.max() + 3, (4000, 3)).astype(np.float32)
    tri = filter_ref.sdf_lookup_ref(g["sdf"], gc, 0)
    assert np.abs(tri - sdf_ref.signed_distance(g["sdf"], gc.T)).max() < 1e-6
    near = filter_ref.sdf_lookup_ref(g["sdf"], gc, 1)
    assert np.array_equal(near, sdf_ref.signed_distance_nearest(g["sdf"], gc.T).astype(np.float32))


def test_occupancy_oracle_semantics():
    """oracle/occupancy_ref.c (common.cpp:324-431): samples at/behind the observed surface are reported, samples in
    front of it are not; geometry follows the reference's float arithmetic."""
    from oracle import filter_ref
    rng = np.random.RandomState(0)
    # a fronto-parallel wall at z = 0.70 m seen from the origin
    xy = rng.uniform(-0.02, 0.02, (6000, 2))
    pts = np.c_[xy, np.full(6000, 0.70) + rng.uniform(0, 0.0005, 6000)].astype(np.float32)
    res = 0.002
    flags, org, dims = filter_ref.occupancy_ref(pts, res)
    pad = np.float32(0.005)
    mn, mx = pts.min(0), pts.max(0)
    assert np.array_equal(org, mn - pad)
    assert all(int(dims[a]) == int((mx[a] + pad - (mn[a] - pad)) / np.float32(res)) for a in range(3))
    zi = np.arange(dims[2])
    z = org[2] + zi.astype(np.float32) * np.float32(res)
    inner = flags[4:-4, 4:-4, :]                      # rays through the wall's interior
    assert not inner[:, :, z < 0.697].any()           # free space in front of the wall
    assert inner[:, :, z > 0.703].mean() > 0.95       # occluded space behind it


def test_bench_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` (the driver's reference arm) runs without a GPU and prints one JSON line with the
    keys the contract names; under torchrun only rank 0 works."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
           "--cpu-sample", "32", "--config", "K1", "--nunocs-pts", "512", "--n-pts", "256"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=root)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["metric"] == "candidate grasps scored/sec" and line["value"] > 0
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    assert line["config"]["config"] == "K1" and "PORT" in line["cpu_baseline"]["sample"]
    assert line["e2e"] == {"value": line["value"], "unit": line["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    env = dict(os.environ, RANK="1", WORLD_SIZE="2")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=120, cwd=root, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""        # other ranks exit 0 without work


def test_host_pose_composition_is_bit_identical_to_the_oracle():
    """my_cpp.grasp_in_cam_unshifted (host fp32, feeds the IK stage) == oracle/filter_ref.c's pose arithmetic, which is
    itself bit-identical to the reference's compiled filterGraspPose (tests/test_mycpp_golden.py)."""
    from catgrasp_b200.my_cpp import grasp_in_cam_unshifted
    from catgrasp_b200.synthetic import make_filter_case
    from oracle import filter_ref
    p1, p2, poses, sym, nocs_pose, c2n, g = make_filter_case(43, 64, 12, (1.0, 1.1, 0.9))
    none = np.zeros((0, 3))
    st, off, out = filter_ref.filter_ref(poses, sym, nocs_pose, c2n, g["gripper_in_grasp"], False, False, 0, g["open"], none,
                                         g["enclosed"], none)
    assert (st == 0).all()
    u = grasp_in_cam_unshifted(poses, sym, nocs_pose, c2n)
    assert np.array_equal(u.view(np.uint32), out.view(np.uint32))


# ------------------------------------------------------------------ the subset draw (host half of GraspDataset.transform)
@pytest.mark.parametrize("M,n_pts,count", [(20000, 1024, 24), (3000, 1024, 40), (2048, 2048, 9), (1024, 1024, 12),
                                           (700, 1024, 12), (1, 5, 3), (2, 2, 4), (5, 8, 6), (1025, 1024, 7)])
@pytest.mark.parametrize("nthreads,isa", [(1, -1), (0, -1), (3, 0), (3, 1)])
def test_c_legacy_choice_equals_numpy(M, n_pts, count, nthreads, isa):
    """cg_host_legacy_choice continues numpy's GLOBAL MT19937 stream exactly like the reference's per-candidate
    ``np.random.choice(np.arange(M), size=n_pts, replace=M < n_pts)`` (dataset_grasp.py:72-73): same indices, and the
    generator is left in the same state (next uniform AND next gaussian draws agree), single- and multi-threaded."""
    from catgrasp_b200 import _lib
    from catgrasp_b200.predicter import _LegacyDraw, draw_subsample_ids_numpy
    _lib.load().cg_host_rng_isa(isa)        # -1: best of AVX-512 / AVX2 / scalar on this host; 0 / 1: capped
    np.random.seed(123)
    np.random.rand(3)
    np.random.randn(1)                      # leaves a cached gaussian in the state tuple
    ref = draw_subsample_ids_numpy(M, n_pts, count)
    ref_next = (np.random.rand(4), np.random.randn(3))
    np.random.seed(123)
    np.random.rand(3)
    np.random.randn(1)
    d = _LegacyDraw()
    a = d.draw(M, n_pts, count // 2, nthreads=nthreads)          # two chunks: the pipelined predict_batch does this
    b = d.draw(M, n_pts, count - count // 2, nthreads=nthreads)
    d.commit()
    _lib.load().cg_host_rng_isa(-1)
    got_next = (np.random.rand(4), np.random.randn(3))
    assert np.array_equal(np.concatenate([a, b]), ref)
    assert np.array_equal(ref_next[0], got_next[0]) and np.array_equal(ref_next[1], got_next[1])


@pytest.mark.parametrize("isa", [0, 1, 2])
def test_c_legacy_skip_equals_draw(isa):
    """cg_host_legacy_skip (the stream walk of a sharded call) leaves the generator exactly where drawing leaves it, on
    every instruction-set level, including sizes around the power-of-two mask changes."""
    from catgrasp_b200 import _lib
    from catgrasp_b200.predicter import _LegacyDraw
    lib = _lib.load()
    try:
        lib.cg_host_rng_isa(isa)
        for M, n_pts, count in ((20000, 1024, 9), (16384, 1024, 5), (16385, 1024, 5), (4097, 4096, 3), (33, 16, 50), (700, 1024, 7)):
            np.random.seed(5 + M)
            a = _LegacyDraw()
            a.draw(M, n_pts, count, nthreads=1)
            np.random.seed(5 + M)
            b = _LegacyDraw()
            b.skip(M, n_pts, count)
            assert np.array_equal(a.key, b.key) and a.pos.value == b.pos.value, (M, n_pts)
    finally:
        lib.cg_host_rng_isa(-1)


def test_draw_subsample_ids_wrapper_consumes_like_reference():
    from catgrasp_b200.predicter import draw_subsample_ids, draw_subsample_ids_numpy
    np.random.seed(7)
    ref = draw_subsample_ids_numpy(5000, 256, 33)
    r2 = np.random.rand(2)
    np.random.seed(7)
    got = draw_subsample_ids(5000, 256, count=33)
    assert np.array_equal(ref, got) and np.array_equal(r2, np.random.rand(2))
    np.random.seed(8)
    one = draw_subsample_ids(900, 64)
    np.random.seed(8)
    assert np.array_equal(one, np.random.choice(np.arange(900), size=64, replace=False))


def test_device_draw_oracle_properties():
    """oracle/draw_ref.py (the pin of cg_draw_ids_dev): distinct in-range indices without replacement, keys depend on
    (seed, global candidate index) only -> a shard draws what the unsharded call draws."""
    from oracle.draw_ref import draw_ids
    full = draw_ids(20000, 1024, 64, seed=99, first_candidate=0)
    assert full.min() >= 0 and full.max() < 20000
    assert all(len(set(r.tolist())) == 1024 for r in full)
    part = draw_ids(20000, 1024, 16, seed=99, first_candidate=32)
    assert np.array_equal(part, full[32:48])
    assert not np.array_equal(full[0], full[1])
    assert not np.array_equal(draw_ids(20000, 1024, 2, seed=100), full[:2])
    rep = draw_ids(700, 1024, 8, seed=1)
    assert rep.min() >= 0 and rep.max() < 700
    perm = draw_ids(1024, 1024, 3, seed=5)
    assert all(sorted(r.tolist()) == list(range(1024)) for r in perm)        # M == n_pts: a permutation
    cnt = np.bincount(draw_ids(20000, 1024, 2048, seed=42).ravel(), minlength=20000)
    e = 2048 * 1024 / 20000
    assert 0.85 < ((cnt - e) ** 2 / e).sum() / 19999 < 1.1                   # chi2 / dof ~ (1 - n/M)
