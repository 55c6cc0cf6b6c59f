"""The mesh -> signed-distance grid builder (csrc/cg_sdf_build.cu, Sdf3D.from_mesh) and its oracles
(oracle/sdf_mesh_ref.c: brute-force float64 distance, sign by winding number; oracle/sdf_parity_exact.py: the exact
ray parity of the builder's contract).

CPU tests pin the distance oracle: against the analytic box-union SDF of the gripper proxy, a numpy restatement,
half-space tests on convex hulls and an analytic inside test of a hex nut with a bore.  GPU tests compare the builder
with the oracles node by node (magnitudes equal to float32(|d_ref|) bit for bit, signs equal to the exact parity
wherever |d| > res * 2^-16 and to the winding number wherever |d| >= res * 2^-12, exact geometry, bitwise repeatable),
check that bad input is refused, and run the collision filter on built grids.  tests/test_sdf_build_edges.py takes
the builder to its grid, brick, tile and lattice edges."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

from catgrasp_b200.synthetic import (_box_mesh, _box_sdf, hex_nut_mesh_inside, make_filter_case, make_gripper_proxy,
                                     make_hex_nut_mesh, tessellated_box_mesh)
from oracle.sdf_mesh_ref import grid_geometry, node_positions, sdf_mesh_ref
from oracle.sdf_parity_exact import parity_lines

SIGN_TOL = 2.0 ** -12          # winding-number signs are compared where |d_ref| >= res * 2^-12
PARITY_TOL = 2.0 ** -16        # parity signs where |d_ref| > res * 2^-16: twice the snap bound of the builder


def _proxy_boxes(name):
    V = make_gripper_proxy()[name]["V"]
    return [(V[8 * b:8 * b + 8].min(0), V[8 * b:8 * b + 8].max(0)) for b in range(V.shape[0] // 8)]


def _proxy_node_positions(rng, n):
    """n seeded nodes of make_gripper_proxy's own grid at its own float64 positions lo + i * 0.001"""
    g = make_gripper_proxy()["open"]
    dims = np.array(g["sdf"].shape)
    lo = np.array([-0.040, -0.033, -0.015]) - 5 * 0.001
    idx = np.stack([rng.randint(0, d, n) for d in dims], 1)
    return idx, lo[None] + 0.001 * idx


def _tessellated_proxy(name, m):
    Vs, Fs, off = [], [], 0
    for lo, hi in _proxy_boxes(name):
        V, F = tessellated_box_mesh(lo, hi, m)
        Vs.append(V); Fs.append(F + off); off += V.shape[0]
    return np.concatenate(Vs), np.concatenate(Fs).astype(np.int32)


def _hull_mesh(seed, n=40):
    from scipy.spatial import ConvexHull
    rng = np.random.RandomState(seed)
    P = rng.normal(size=(n, 3)) * np.array([0.02, 0.012, 0.009]) + np.array([0.1, -0.05, 0.7])
    h = ConvexHull(P)
    F = h.simplices.copy()
    nrm = np.cross(P[F[:, 1]] - P[F[:, 0]], P[F[:, 2]] - P[F[:, 0]])
    flip = np.einsum("ij,ij->i", nrm, h.equations[:, :3]) < 0          # orient every face outward
    F[flip] = F[flip][:, ::-1]
    return P, F.astype(np.int32), h.equations


# ------------------------------------------------------------------ CPU: the oracle
@pytest.mark.parametrize("name", ["open", "enclosed"])
def test_oracle_matches_analytic_proxy_at_proxy_nodes(name):
    """Touching, non-overlapping boxes: the distance to the concatenated box meshes is the min of the box SDFs."""
    g = make_gripper_proxy()
    idx, P = _proxy_node_positions(np.random.RandomState(1), 4000)
    ana = np.min(np.stack([_box_sdf(P, lo, hi) for lo, hi in _proxy_boxes(name)]), 0)
    sd, _ = sdf_mesh_ref(g[name]["V"], g[name]["F"], P)
    assert np.abs(sd - ana).max() <= 1e-12
    # the builder's geometry is the proxy's, and its float32 node positions move values by at most ~6.1e-9 m
    dims, origin, res = grid_geometry(g[name]["V"], 0.001, 5)
    assert np.array_equal(dims, g[name]["sdf"].shape) and np.array_equal(origin, g[name]["origin"])
    sd32, _ = sdf_mesh_ref(g[name]["V"], g[name]["F"], node_positions(origin, res, idx))
    grid = g[name]["sdf"][idx[:, 0], idx[:, 1], idx[:, 2]].astype(np.float64)
    assert np.abs(sd32 - grid).max() <= 6.2e-9 + np.spacing(np.float32(0.05))


def _numpy_sdf(V, F, P):
    """Restatement: closest point by barycentric least squares (Gram system) when it falls inside, else the three
    edges; winding number by Van Oosterom-Strackee, all in numpy."""
    a, b, c = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    best = np.full(P.shape[0], np.inf)
    om = np.zeros(P.shape[0])
    for t in range(F.shape[0]):
        e0, e1, w = b[t] - a[t], c[t] - a[t], P - a[t]
        a00, a01, a11 = e0 @ e0, e0 @ e1, e1 @ e1
        det = a00 * a11 - a01 * a01
        cand = []
        if det > 1e-30 * (a00 * a11):
            s = (a11 * (w @ e0) - a01 * (w @ e1)) / det
            u = (a00 * (w @ e1) - a01 * (w @ e0)) / det
            q = a[t] + s[:, None] * e0 + u[:, None] * e1
            ins = (s >= 0) & (u >= 0) & (s + u <= 1)
            cand.append(np.where(ins, ((P - q) ** 2).sum(1), np.inf))
        for p0, p1 in ((a[t], b[t]), (b[t], c[t]), (c[t], a[t])):
            d = p1 - p0
            L = d @ d
            tt = np.clip(((P - p0) @ d) / L, 0, 1) if L > 0 else np.zeros(P.shape[0])
            cand.append((((P - p0) - tt[:, None] * d) ** 2).sum(1))
        best = np.minimum(best, np.min(cand, 0))
        A, B, Cc = a[t] - P, b[t] - P, c[t] - P
        la, lb, lc = (np.linalg.norm(X, axis=1) for X in (A, B, Cc))
        num = np.einsum("ij,ij->i", A, np.cross(B, Cc))
        den = la * lb * lc + np.einsum("ij,ij->i", A, B) * lc + np.einsum("ij,ij->i", A, Cc) * lb + \
            np.einsum("ij,ij->i", B, Cc) * la
        om += 2 * np.arctan2(num, den)
    w = om / (4 * np.pi)
    return np.where(np.abs(w) > 0.5, -1, 1) * np.sqrt(best), w


@pytest.mark.parametrize("case", ["tetra", "box", "degenerate"])
def test_oracle_matches_numpy_restatement(case):
    rng = np.random.RandomState(7)
    if case == "tetra":
        V = np.array([[0, 0, 0], [0.01, 0, 0], [0, 0.012, 0], [0.001, 0.002, 0.009]])
        F = np.array([[0, 2, 1], [0, 1, 3], [1, 2, 3], [0, 3, 2]], np.int32)
    elif case == "box":
        V, F = tessellated_box_mesh([-0.01, 0.0, 0.02], [0.005, 0.008, 0.03], 2)
    else:                                           # a box with a zero-area pair and a point triangle
        V, F = _box_mesh(np.zeros(3), np.array([0.01, 0.02, 0.015]))
        V = np.concatenate([V, [[0.005, 0.0, 0.0]]])
        F = np.concatenate([F, [[0, 1, 8], [1, 0, 8], [2, 2, 2]]]).astype(np.int32)
    P = V.min(0) - 0.004 + rng.uniform(size=(3000, 3)) * (V.max(0) - V.min(0) + 0.008)
    sd, w = sdf_mesh_ref(V, F, P)
    sd_np, w_np = _numpy_sdf(V, F, P)
    assert np.all(np.isfinite(sd))
    assert np.abs(np.abs(sd) - np.abs(sd_np)).max() <= 1e-15
    assert np.abs(w - w_np).max() <= 1e-9
    far = np.abs(sd_np) > 1e-9
    assert np.array_equal(np.sign(sd[far]), np.sign(sd_np[far]))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_sign_on_convex_hulls(seed):
    V, F, eq = _hull_mesh(seed)
    rng = np.random.RandomState(seed + 10)
    P = V.min(0) - 0.005 + rng.uniform(size=(5000, 3)) * (V.max(0) - V.min(0) + 0.01)
    sd, w = sdf_mesh_ref(V, F, P)
    h = P @ eq[:, :3].T + eq[:, 3]
    inside = (h < 0).all(1)
    clear = np.abs(h).min(1) > 1e-9
    assert clear.sum() > 4900 and inside[clear].sum() > 500
    assert np.array_equal(sd[clear] < 0, inside[clear])
    assert np.allclose(np.abs(w[clear]), inside[clear].astype(float), atol=1e-9)
    # the distance of an inside point is its distance to the nearest face plane
    assert np.allclose(-sd[inside & clear], np.abs(h[inside & clear]).min(1), rtol=0, atol=1e-15)


def test_oracle_sign_on_hex_nut():
    V, F = make_hex_nut_mesh()
    rng = np.random.RandomState(3)
    P = rng.uniform(-0.013, 0.013, size=(20000, 3)) * np.array([1, 1, 0.5])
    sd, w = sdf_mesh_ref(V, F, P)
    ins = hex_nut_mesh_inside(P)
    clear = np.abs(sd) > 1e-9
    assert ins[clear].sum() > 2000 and (~ins[clear]).sum() > 2000
    assert np.array_equal(sd[clear] < 0, ins[clear])
    bore = (np.hypot(P[:, 0], P[:, 1]) < 0.004) & (np.abs(P[:, 2]) < 0.003)      # the hole is outside (genus 1)
    assert bore.sum() > 100 and (sd[bore] > 0).all()


# ------------------------------------------------------------------ GPU: builder vs oracle
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)


def _dyadic_mesh():
    r = 2.0 ** -10
    V1, F1 = tessellated_box_mesh([0, 0, 0], [8 * r, 6 * r, 4 * r], 2)
    V2, F2 = tessellated_box_mesh([8 * r, 2 * r, 0], [12 * r, 4 * r, 2 * r], 2)
    return np.concatenate([V1, V2]), np.concatenate([F1, F2 + V1.shape[0]]).astype(np.int32), r


def _shell_mesh():
    """A box with a 0.4 mm wall around a cavity; the far walls hold the node planes x = 12, y = 10, z = 8 mm."""
    Vo, Fo = _box_mesh(np.array([0.0, 0.0, 0.0]), np.array([0.0123, 0.0103, 0.0083]))
    Vi, Fi = _box_mesh(np.array([0.0004, 0.0004, 0.0004]), np.array([0.0119, 0.0099, 0.0079]))
    return np.concatenate([Vo, Vi]), np.concatenate([Fo, Fi[:, ::-1] + 8]).astype(np.int32)


def _degenerate_box():
    V, F = _box_mesh(np.array([0.001, -0.002, 0.0]), np.array([0.011, 0.006, 0.007]))
    V = np.concatenate([V, [(V[0] + V[1]) / 2]])
    return V, np.concatenate([F, [[0, 1, 8], [1, 0, 8]]]).astype(np.int32)


def _gpu_case(name):
    """(V, F, res, padding, sample): sample = None checks every node, else (n random nodes, slab index along x)"""
    g = make_gripper_proxy()
    if name in ("proxy_open", "proxy_enclosed"):
        d = g[name.split("_")[1]]
        return d["V"], d["F"], 0.001, 5, None
    if name in ("proxy_pad0", "proxy_pad1"):
        return g["open"]["V"], g["open"]["F"], 0.001, int(name[-1]), None
    if name == "proxy_tess200k":
        V, F = _tessellated_proxy("open", 75)
        return V, F, 0.001, 5, (1500, 50)
    if name == "hex_nut":
        V, F = make_hex_nut_mesh()
        return V, F, 0.0005, 3, None
    if name.startswith("hull"):
        V, F, _ = _hull_mesh(int(name[-1]))
        return V, F, 0.001, 4, None
    if name == "thin_shell":
        V, F = _shell_mesh()
        return V, F, 0.001, 2, None
    if name == "dyadic":
        V, F, r = _dyadic_mesh()
        return V, F, r, 2, None
    if name == "degenerate_pair":
        V, F = _degenerate_box()
        return V, F, 0.001, 3, None
    raise KeyError(name)


GPU_CASES = ["proxy_open", "proxy_enclosed", "proxy_pad0", "proxy_pad1", "proxy_tess200k", "hex_nut", "hull0", "hull1",
             "thin_shell", "dyadic", "degenerate_pair"]


def on_lattice(V, origin, res):
    """True when every vertex coordinate is origin + an integer multiple of res * 2^-16 exactly (small meshes only):
    the builder's snap then moves nothing, so its sign is the exact parity at every node, on the surface too."""
    V = np.asarray(V, np.float64)
    if V.size > 3000:
        return False
    step = Fraction(float(res)) / 2 ** 16
    return all(((Fraction(float(v)) - Fraction(float(o))) / step).denominator == 1 for col, o in zip(V.T, origin)
               for v in col)


def check_nodes(built, V, F, idx, winding=True):
    """Compare the built grid with the oracles at the nodes idx (n, 3): |value| equal to float32(|d_ref|) bit for bit,
    the sign equal to the exact ray parity wherever |d_ref| > res * 2^-16 (at every node, zeros included, when the
    mesh lies on the snap lattice), and (``winding``: closed non-overlapping meshes, where the two rules coincide) to
    the winding number wherever |d_ref| >= res * 2^-12.
    Returns (nodes checked, signs decided by parity, magnitude mismatches, inside nodes)."""
    origin, res = built.origin_, built.resolution_
    sd, _ = sdf_mesh_ref(V, F, node_positions(origin, res, idx))
    got = built.data_[idx[:, 0], idx[:, 1], idx[:, 2]]
    assert np.all(np.isfinite(got))
    mag = np.abs(got).view(np.uint32) != np.abs(sd).astype(np.float32).view(np.uint32)
    assert not mag.any(), (int(mag.sum()), idx[mag][:5], got[mag][:5], sd[mag][:5])
    lines, inv = np.unique(idx[:, 1:], axis=0, return_inverse=True)
    inside, open_, _ = parity_lines(V, F, origin, res, built.dims_, lines)
    assert not open_.any()
    par = inside[inv.reshape(-1), idx[:, 0]]
    decided = (np.abs(sd) > res * PARITY_TOL) | on_lattice(V, origin, res)
    wrong = decided & (np.signbit(got) != par)
    assert not wrong.any(), (int(wrong.sum()), idx[wrong][:5], got[wrong][:5], sd[wrong][:5])
    if winding:
        wdec = np.abs(sd) >= res * SIGN_TOL
        wrong = wdec & (np.signbit(got) != (sd < 0))
        assert not wrong.any(), (idx[wrong][:5], got[wrong][:5], sd[wrong][:5])
    return idx.shape[0], int(decided.sum()), int(mag.sum()), int((decided & par).sum())


def report(capsys, name, stats):
    n, dec, mis, ins = stats
    with capsys.disabled():
        print(f"\n  {name}: {n} nodes checked, {dec} signs decided ({ins} inside), {mis} magnitude mismatches")


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_CASES)
def test_builder_matches_oracle(name, capsys):
    _cuda()
    from catgrasp_b200.sdf import Sdf3D
    V, F, res, pad, sample = _gpu_case(name)
    built = Sdf3D.from_mesh(V, F, res, pad)
    dims, origin, res32 = grid_geometry(V, res, pad)
    assert np.array_equal(built.data_.shape, dims) and np.array_equal(built.dims_, dims)
    assert np.array_equal(built.origin_, origin) and built.resolution_ == float(res32)
    if sample is None:
        idx = np.stack(np.meshgrid(*[np.arange(d) for d in dims], indexing="ij"), -1).reshape(-1, 3)
    else:
        n, i_slab = sample
        rng = np.random.RandomState(5)
        rand = np.stack([rng.randint(0, d, n) for d in dims], 1)
        jj, kk = np.meshgrid(np.arange(dims[1]), np.arange(dims[2]), indexing="ij")
        slab = np.stack([np.full(jj.size, i_slab), jj.reshape(-1), kk.reshape(-1)], 1)
        idx = np.concatenate([rand, slab])
    stats = check_nodes(built, V, F, idx)
    report(capsys, name, stats)
    assert stats[3] > 0 and stats[1] > idx.shape[0] // 2
    again = Sdf3D.from_mesh(V, F, res, pad)
    assert np.array_equal(again.data_.view(np.uint32), built.data_.view(np.uint32))


@pytest.mark.gpu
def test_builder_grid_is_close_to_analytic_proxy():
    """Built proxy grids vs make_gripper_proxy's analytic grids: same geometry, values within the node-position shift."""
    _cuda()
    from catgrasp_b200.sdf import Sdf3D
    g = make_gripper_proxy()
    for name in ("open", "enclosed"):
        b = Sdf3D.from_mesh(g[name]["V"], g[name]["F"])
        assert np.array_equal(b.origin_, g[name]["origin"]) and b.data_.shape == g[name]["sdf"].shape
        assert np.abs(b.data_.astype(np.float64) - g[name]["sdf"]).max() <= 6.2e-9 + np.spacing(np.float32(0.05))


def _raw_build(V, F, res, pad, nv=None, nf=None):
    from catgrasp_b200 import _lib
    ctx = _lib.Context.get(0)
    V = np.ascontiguousarray(V, np.float64).reshape(-1, 3)
    F = np.ascontiguousarray(F, np.int32).reshape(-1, 3)
    h = C.c_void_p()
    rc = ctx.lib.cg_sdf_from_mesh(ctx.h, _lib.ptr(V), V.shape[0] if nv is None else nv, _lib.ptr(F),
                                  F.shape[0] if nf is None else nf, C.c_float(res), int(pad), C.byref(h))
    msg = ctx.lib.cg_last_error(ctx.h).decode()
    if h.value:
        ctx.lib.cg_sdf_destroy(h)
    return rc, h.value, msg


@pytest.mark.gpu
def test_builder_rejects_bad_input():
    _cuda()
    from catgrasp_b200 import _lib
    g = make_gripper_proxy()["open"]
    V, F = g["V"], g["F"]
    rc, h, _ = _raw_build(V, F, 0.001, 5)
    assert rc == _lib.CG_OK and h
    # an open mesh: one triangle of the palm's largest face (x = -0.04, 60 x 30 mm) removed
    big = np.nonzero(np.isclose(V[F].max(1)[:, 0], -0.04) & np.isclose(V[F].min(1)[:, 0], -0.04))[0]
    assert big.size == 2
    Vn = V.copy()
    Vn[0, 1] = np.nan
    Fo = F.copy()
    Fo[3, 1] = V.shape[0]
    cases = {"open": (V, np.delete(F, big[0], axis=0), 0.001, 5), "index": (V, Fo, 0.001, 5),
             "negative_index": (V, -F, 0.001, 5), "nan": (Vn, F, 0.001, 5), "res0": (V, F, 0.0, 5),
             "res_neg": (V, F, -0.001, 5), "res_nan": (V, F, float("nan"), 5), "pad": (V, F, 0.001, -1),
             "nf0": (V, np.zeros((0, 3), np.int32), 0.001, 5), "too_big": (V, F, 1e-6, 5)}
    for key, (v, f, r, p) in cases.items():
        rc, h, msg = _raw_build(v, f, r, p)
        assert rc == _lib.CG_EINVAL and not h, (key, rc)
        if key == "open":
            assert "not closed" in msg
    with pytest.raises(_lib.CgError, match="not closed"):
        from catgrasp_b200.sdf import Sdf3D
        Sdf3D.from_mesh(V, np.delete(F, big[0], axis=0))


# ------------------------------------------------------------------ GPU: the collision filter on built grids
EYE = np.eye(4)


def _built_pair():
    from catgrasp_b200.sdf import Sdf3D
    g = make_gripper_proxy()
    return Sdf3D.from_mesh(g["open"]["V"], g["open"]["F"]), Sdf3D.from_mesh(g["enclosed"]["V"], g["enclosed"]["F"])


def _as_dict(s):
    return {"sdf": s.data_, "origin": s.origin_, "res": np.float32(s.resolution_)}


@pytest.mark.gpu
@pytest.mark.parametrize("margin", [0.0, 0.0005])
def test_filter_on_built_grid_equals_filter_on_its_values(margin):
    """A built grid behaves in the filter exactly like the same values passed through cg_sdf_create (this covers the
    boundary statistics of the out-of-box shortcut)."""
    _cuda()
    from catgrasp_b200 import my_cpp
    from catgrasp_b200.sdf import Sdf3D
    p1, p2, poses, sym, nocs, c2n, g = make_filter_case(11, 48, 12)
    bo, be = _built_pair()
    co, ce = (Sdf3D(b.data_, b.origin_, b.resolution_) for b in (bo, be))
    for adjust in (False, True):
        args = (poses, sym, nocs, c2n, g["gripper_in_grasp"], True, adjust)
        a = my_cpp.filter_grasp_pose_raw(*args, bo, p1, be, p2, sdf_margin=margin)
        b = my_cpp.filter_grasp_pose_raw(*args, co, p1, ce, p2, sdf_margin=margin)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        assert np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32))


def _filter_args(seed, G, S):
    p1, p2, poses, sym, nocs, c2n, g = make_filter_case(seed, G, S)
    gp = make_gripper_proxy()
    return (poses, sym, nocs, c2n, EYE, EYE, g["gripper_in_grasp"], True, False, True, None, None,
            gp["open"]["V"], gp["open"]["F"], gp["enclosed"]["V"], gp["enclosed"]["F"], p1, p2, 0.003, False)


@pytest.mark.gpu
def test_filterGraspPose_without_registration(monkeypatch, capsys):
    """The 20 reference arguments and no registered SDF: the grids are built from the meshes.  The result equals
    filter_ref.c on the built grids bit for bit, and the analytic-grid result wherever filter64's verdict holds for
    every grid within the largest |built - analytic| difference."""
    _cuda()
    from catgrasp_b200 import my_cpp
    from catgrasp_b200.sdf import Sdf3D
    from oracle import filter_ref
    from oracle.filter64 import filter64
    monkeypatch.setattr(my_cpp, "_SDF_REGISTRY", {})
    a = _filter_args(5, 40, 12)
    (poses, sym, nocs, c2n, _, _, gig, fdir, _, adjust, _, _, Vo, Fo, Ve, Fe, p1, p2, _, _) = a
    got = my_cpp.filterGraspPose(*a)
    assert len(my_cpp._SDF_REGISTRY) == 2
    bo = my_cpp._sdf_for(Vo, Fo)
    be = my_cpp._sdf_for(Ve, Fe)
    st, off, out = filter_ref.filter_ref(poses, sym, nocs, c2n, gig, fdir, adjust, 0, _as_dict(bo), p1, _as_dict(be), p2)
    ref = [out[q] for q in np.nonzero(st == 0)[0]]
    assert len(got) == len(ref) and all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(got, ref))
    # against the analytic grids
    g = make_gripper_proxy()
    D = max(float(np.abs(bo.data_.astype(np.float64) - g["open"]["sdf"]).max()),
            float(np.abs(be.data_.astype(np.float64) - g["enclosed"]["sdf"]).max()))
    assert D <= 1e-8
    monkeypatch.setattr(my_cpp, "_SDF_REGISTRY", {})
    my_cpp.register_gripper_sdf(Vo, Fo, Sdf3D(g["open"]["sdf"], g["open"]["origin"], g["open"]["res"]))
    my_cpp.register_gripper_sdf(Ve, Fe, Sdf3D(g["enclosed"]["sdf"], g["enclosed"]["origin"], g["enclosed"]["res"]))
    ana = my_cpp.filter_grasp_pose_raw(poses, sym, nocs, c2n, gig, fdir, adjust, my_cpp._sdf_for(Vo, Fo), p1,
                                       my_cpp._sdf_for(Ve, Fe), p2)
    built = filter_ref.filter_ref(poses, sym, nocs, c2n, gig, fdir, adjust, 0, _as_dict(bo), p1, _as_dict(be), p2)
    lo = filter64(poses, sym, nocs, c2n, gig, fdir, adjust, 0, g["open"], p1, g["enclosed"], p2, margin=-2 * D)
    hi = filter64(poses, sym, nocs, c2n, gig, fdir, adjust, 0, g["open"], p1, g["enclosed"], p2, margin=2 * D)
    sure = lo["decided"] & hi["decided"] & (lo["status"] == hi["status"]) & (lo["offset"] == hi["offset"])
    assert sure.sum() > 0.9 * sure.size
    assert np.array_equal(ana[0][sure], built[0][sure]) and np.array_equal(ana[1][sure], built[1][sure])
    with capsys.disabled():
        print(f"\n  filter on built vs analytic grids: {int(sure.sum())} of {sure.size} poses decided within "
              f"max |built - analytic| = {D:.3e} m, all equal")


@pytest.mark.gpu
def test_registered_sdf_takes_precedence(monkeypatch):
    _cuda()
    from catgrasp_b200 import my_cpp
    from catgrasp_b200.sdf import Sdf3D
    monkeypatch.setattr(my_cpp, "_SDF_REGISTRY", {})
    a = _filter_args(6, 24, 6)
    assert len(my_cpp.filterGraspPose(*a)) > 0
    g = make_gripper_proxy()
    solid = -np.ones_like(g["open"]["sdf"])            # everything inside: every pose collides
    my_cpp.register_gripper_sdf(a[12], a[13], Sdf3D(solid, g["open"]["origin"], g["open"]["res"]))
    assert my_cpp.filterGraspPose(*a) == []


@pytest.mark.gpu
def test_collision_manager_without_registration(monkeypatch):
    _cuda()
    from catgrasp_b200 import my_cpp
    monkeypatch.setattr(my_cpp, "_SDF_REGISTRY", {})
    g = make_gripper_proxy()["open"]
    cm = my_cpp.CollisionManager()
    cm.registerMesh(g["V"], g["F"])
    pose = np.eye(4)
    pose[:3, 3] = [0.2, 0.1, 0.5]
    cm.setTransform(pose, 0)
    cm.registerPointCloud(np.array([[0.2 + 0.0225, 0.1 + 0.029, 0.5]]), 0.003)        # inside finger 1
    assert cm.isAnyCollision()
    cm.registerPointCloud(np.array([[0.2 + 0.0225, 0.1, 0.5], [0.3, 0.1, 0.5]]), 0.003)   # between the fingers, far
    assert not cm.isAnyCollision()


@pytest.mark.gpu
def test_sdf_file_round_trip_of_built_grid(tmp_path):
    _cuda()
    from catgrasp_b200 import my_cpp
    from catgrasp_b200.sdf import read_sdf_file, write_sdf_file
    p1, p2, poses, sym, nocs, c2n, g = make_filter_case(8, 32, 6)
    bo, be = _built_pair()
    files = []
    for name, b in (("open", bo), ("enclosed", be)):
        path = str(tmp_path / f"gripper_{name}.sdf")
        write_sdf_file(path, b.data_, b.origin_, b.resolution_)
        files.append(read_sdf_file(path))
    assert np.array_equal(files[0].data_.view(np.uint32), bo.data_.view(np.uint32))
    assert np.array_equal(files[0].origin_, bo.origin_) and files[0].resolution_ == bo.resolution_
    args = (poses, sym, nocs, c2n, g["gripper_in_grasp"], True, True)
    a = my_cpp.filter_grasp_pose_raw(*args, bo, p1, be, p2)
    b = my_cpp.filter_grasp_pose_raw(*args, files[0], p1, files[1], p2)
    assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))
