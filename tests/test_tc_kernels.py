"""GPU tests (-m gpu) of the trunk and fully-connected kernels at the level of their own outputs.

Each kernel output is compared with the float64 reference of oracle/encoder_ref.py, within twice its rigorous error
bound, on every engine: the three trunks' 1024-channel max-pool outputs, the point feature of a PointNetSeg, T3, T64
and the head logits (each FC chain given the GPU's own input keys), and single FC layers through a one-layer cg_mlp.
The end-to-end tolerances of test_gpu_parity.py cannot see a trunk that skips a tile; these can
(tests/test_encoder_ref.py).  Every comparison against a bound prints its largest error / (2 x bound) ratio, so a
loss of precision shows before it fails.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle.encoder_ref import FoldedNet, bound_ratio, fused_input, key2f, u_bf16x3, u_fp32

pytestmark = pytest.mark.gpu

ENGINES = [int(e) for e in os.environ.get("CG_TEST_ENGINES", "0,1,2,3").split(",")]
CHUNK_B = 16384   # candidates per internal pass of the cls forward (cg_net.cu)


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _build(kind, n_out, sd, cuda):
    from catgrasp_b200.net import PointNetCls, PointNetSeg
    from catgrasp_b200.weights import pack_blob
    net = (PointNetCls if kind == "cls" else PointNetSeg)(sd, device=0)
    blob, n = pack_blob(sd, kind)
    return net, FoldedNet(blob, kind, n, device=cuda)


@pytest.fixture(scope="module")
def cls_pair(cuda):
    from catgrasp_b200.synthetic import make_state_dict
    return _build("cls", 10, make_state_dict("cls", 10, seed=0), cuda)


@pytest.fixture(scope="module")
def seg_pair(cuda):
    from catgrasp_b200.synthetic import make_state_dict
    return _build("seg", 300, make_state_dict("seg", 300, seed=1), cuda)


def _dev(a, dtype):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)


def probe(net, B, N, x=None, fused=None, want_pf=False):
    """cg_encoder_probe_dev: the three trunks' max-pool outputs (decoded from their keys), T3, T64 and optionally the
    point feature.  fused = (xyz, nrm, poses, ids, mean, std) with ids / mean / std possibly None."""
    from catgrasp_b200 import _lib
    ctx = net.ctx
    ctx.use_torch_stream()
    keys = torch.zeros((3, B, 1024), dtype=torch.int32, device="cuda")
    T3 = torch.empty((B, 9), dtype=torch.float32, device="cuda")
    T64 = torch.empty((B, 4096), dtype=torch.float32, device="cuda")
    pf = torch.empty((B, N, 64), dtype=torch.float32, device="cuda") if want_pf else None
    if fused is None:
        xd = _dev(x, torch.float32)
        args = (_lib.ptr(xd), None, None, 0, None, None, None, None)
    else:
        xyz, nrm, poses, ids, mean, std = fused
        t = [_dev(xyz, torch.float64), _dev(nrm, torch.float64), _dev(poses, torch.float64), _dev(ids, torch.int32),
             _dev(mean, torch.float64), _dev(std, torch.float64)]
        args = (None, _lib.ptr(t[0]), _lib.ptr(t[1]), len(xyz), _lib.ptr(t[2]), _lib.ptr(t[3]), _lib.ptr(t[4]),
                _lib.ptr(t[5]))
    ctx.check(ctx.lib.cg_encoder_probe_dev(net.h, *args, B, N, _lib.ptr(keys), _lib.ptr(T3), _lib.ptr(T64),
                                           _lib.ptr(pf)))
    torch.cuda.synchronize()
    k = keys.cpu().numpy().view(np.uint32)
    out = {"keys": k, "gA": key2f(k[0]), "gB": key2f(k[1]), "gC": key2f(k[2]),
           "T3": T3.cpu().numpy(), "T64": T64.cpu().numpy()}
    if want_pf:
        out["pf"] = pf.cpu().numpy()
    return out


def _ratio(label, got, ref, err):
    r = bound_ratio(got, ref, err)
    assert np.isfinite(np.asarray(got)).all(), label
    return float(r.max())


def check_encoder(ref, engine, got, x, ex=None, logits=None, label=""):
    """Every trunk output given its own inputs (trunks B and C take the GPU's T3 / T64), and every FC chain given the
    GPU's keys.  Returns {name: largest error / (2 x bound)}; all must be <= 1."""
    B = got["gA"].shape[0]
    r = {}
    A = ref.trunk("A", x, ex, engine=engine)
    r["A"] = _ratio("A", got["gA"], A["g"], A["eg"])
    Bt = ref.trunk("B", x, ex, T3=got["T3"], engine=engine)
    r["B"] = _ratio("B", got["gB"], Bt["g"], Bt["eg"])
    want_pf = "pf" in got
    Ct = ref.trunk("C", x, ex, T3=got["T3"], T64=got["T64"], engine=engine, want_pf=want_pf)
    r["C"] = _ratio("C", got["gC"], Ct["g"], Ct["eg"])
    if want_pf:
        r["pf"] = _ratio("pf", got["pf"], Ct["pf"], Ct["epf"])
    T3, eT3 = ref.stn_fc("A", got["gA"], engine=engine)
    r["T3"] = _ratio("T3", got["T3"], T3, eT3)
    T64, eT64 = ref.stn_fc("B", got["gB"], engine=engine)
    r["T64"] = _ratio("T64", got["T64"], T64, eT64)
    if logits is not None:
        if ref.kind == "cls":
            lg, elg = ref.cls_head(got["gC"], engine=engine)
        else:
            lg, elg = ref.seg_head(got["gC"], np.zeros_like(got["gC"]), got["pf"], np.zeros_like(got["pf"]), engine)
        r["logits"] = _ratio("logits", logits, lg, elg)
    print(f"\nRATIO engine={engine} {label} B={B} " + " ".join(f"{k}={v:.3g}" for k, v in r.items()))
    bad = {k: v for k, v in r.items() if not v <= 1.0}
    assert not bad, (label, bad)
    return r


# ------------------------------------------------------------------------------------------ trunk features
X_SHAPES = ([(1, n) for n in (1, 63, 64, 65, 127, 128, 129, 1000, 2048, 8192)] +
            [(3, n) for n in (1, 63, 65, 128, 129, 1000, 8192)] +
            [(130, 64), (130, 129), (130, 1000), (528, 1), (528, 129), (528, 1000)] +
            [(100, 1100),      # 9 tiles split over 5 CTAs as 2+2+2+2+1
             (600, 2048)])     # one CTA runs all 16 tiles of a candidate: the W3 ring goes through many phases


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("B,N", X_SHAPES)
def test_trunks_and_fc_vs_float64(cls_pair, engine, B, N):
    net, ref = cls_pair
    net.ctx.set_engine(engine)
    x = np.random.RandomState(B * 10007 + N).normal(0, 1, (B, N, 6)).astype(np.float32)
    got = probe(net, B, N, x=x)
    logits = net.forward(x).cpu().numpy()
    check_encoder(ref, engine, got, x, logits=logits, label=f"x_direct N={N}")


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("with_ids,with_norm", [(True, True), (True, False), (False, True), (False, False)])
def test_trunks_fused_input_vs_float64(cls_pair, engine, with_ids, with_norm):
    """The fused grasp-Q input: subset ids (M < N draws with replacement) or none (point n = cloud point n, N <= M),
    with and without the mean / std normaliser."""
    from catgrasp_b200.synthetic import make_candidates, make_pile
    net, ref = cls_pair
    net.ctx.set_engine(engine)
    B, N = 130, 600
    M = 400 if with_ids else 700
    scene = make_pile(M, n_objects=3, seed=31)
    xyz, nrm = scene["cloud_xyz"], scene["cloud_normal"]
    poses = make_candidates(xyz, nrm, B, seed=32)
    rng = np.random.RandomState(33)
    ids = rng.randint(0, M, (B, N)).astype(np.int32) if with_ids else None
    mean = std = None
    if with_norm:
        mean = np.concatenate([rng.normal(0, 0.002, 3), rng.normal(0, 0.05, 3)])
        std = np.concatenate([rng.uniform(0.008, 0.012, 3), rng.uniform(0.5, 0.6, 3)])
    got = probe(net, B, N, fused=(xyz, nrm, poses, ids, mean, std))
    x, ex = fused_input(xyz, nrm, poses, ids if with_ids else np.tile(np.arange(N), (B, 1)), mean, std)
    check_encoder(ref, engine, got, x, ex, label=f"fused ids={with_ids} norm={with_norm} N={N}")


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("B,N", [(2, 1000), (1, 8192), (3, 65)])
def test_seg_point_feature_and_logits_vs_float64(seg_pair, engine, B, N):
    net, ref = seg_pair
    net.ctx.set_engine(engine)
    x = np.random.RandomState(N + B).normal(0, 1, (B, N, 6)).astype(np.float32)
    got = probe(net, B, N, x=x, want_pf=True)
    logits = net.forward(x).cpu().numpy()
    check_encoder(ref, engine, got, x, logits=logits, label=f"seg N={N}")


@pytest.mark.parametrize("engine", ENGINES)
def test_all_negative_channels(cuda, engine):
    """Encoder channels that are negative at every point (trunk C has no ReLU), and STN channels the ReLU holds at 0:
    the negative half of the key order and the zero-initialised key buffer."""
    from catgrasp_b200.synthetic import make_state_dict
    sd = make_state_dict("cls", 10, seed=4)
    neg = np.arange(0, 1024, 37)
    for bn in ("module.feat.bn3", "module.feat.stn.bn3", "module.feat.fstn.bn3"):
        bias = sd[bn + ".bias"].clone()
        bias[neg] = -50.0
        sd[bn + ".bias"] = bias
    net, ref = _build("cls", 10, sd, cuda)
    net.ctx.set_engine(engine)
    B, N = 5, 300
    x = np.random.RandomState(5).normal(0, 1, (B, N, 6)).astype(np.float32)
    got = probe(net, B, N, x=x)
    assert (got["gC"][:, neg] < -10).all()
    assert (got["gA"][:, neg] == 0).all() and (got["gB"][:, neg] == 0).all()
    check_encoder(ref, engine, got, x, logits=net.forward(x).cpu().numpy(), label="negative channels")


# ------------------------------------------------------------------------------------------ single FC layers
def _fma_kernel(M, K, N, num_sms):
    """Which FMA kernel cg_linear_launch (cg_linear.cu) picks when the layer is not on tensor cores."""
    if M <= 8:
        return "rows"
    if N >= 128 and K % 16 == 0 and -(-N // 128) * -(-M // 64) >= num_sms:
        return "wide"
    return "tiled"


def _mlp1(cuda, engine, R, K, N, seed):
    """One-layer cg_mlp (fully-connected + ReLU) on R rows vs float64; returns the largest error / (2 x bound)."""
    from catgrasp_b200 import _lib
    ctx = _lib.Context.get(0)
    ctx.set_engine(engine)
    rng = np.random.RandomState(seed)
    W = rng.uniform(-1, 1, (K, N)).astype(np.float32) / np.float32(np.sqrt(K))
    b = rng.uniform(-0.1, 0.1, N).astype(np.float32)
    x = rng.normal(0, 1, (R, K)).astype(np.float32)
    dims = (C.c_int * 2)(K, N)
    h = C.c_void_p()
    ctx.check(ctx.lib.cg_mlp_create(ctx.h, 1, dims, (C.c_void_p * 1)(W.ctypes.data), (C.c_void_p * 1)(b.ctypes.data),
                                    C.byref(h)))
    try:
        ctx.use_torch_stream()
        xd = _dev(x, torch.float32)
        out = torch.full((R, N), float("nan"), dtype=torch.float32, device="cuda")
        ctx.check(ctx.lib.cg_shared_mlp_dev(h, _lib.ptr(xd), R, _lib.ptr(out)))
        got = out.cpu().numpy()
    finally:
        ctx.lib.cg_mlp_destroy(h)
        ctx.set_engine(3)
    tc = engine >= 1 and R >= 64 and K % 64 == 0 and N >= 64
    u = u_bf16x3(K) if tc else u_fp32(K)
    W64, x64 = W.astype(np.float64), x.astype(np.float64)
    y = np.maximum(x64 @ W64 + b, 0.0)
    e = u * (np.abs(x64) @ np.abs(W64) + np.abs(b))
    r = _ratio("mlp", got, y, e)
    print(f"\nRATIO engine={engine} fc R={R} K={K} N={N} {'tc' if tc else _fma_kernel(R, K, N, 132)}={r:.3g}")
    assert r <= 1.0, (R, K, N, r)
    return r


@pytest.mark.parametrize("K", [64, 128, 192, 256, 1024])
@pytest.mark.parametrize("N", [64, 72, 128, 130, 300, 4096])
def test_fc_tensor_core_k_blocks(cuda, K, N):
    """Engine 1, tensor-core FC: 1, 2, 3, 4 and 16 K-blocks against the 3-stage ring (4 and 16 refill it); column
    tiles that end inside a tile; R = 129 ends inside a 128-row tile."""
    _mlp1(cuda, 1, 129, K, N, seed=K * 7 + N)


@pytest.mark.parametrize("R", [64, 65, 127, 128, 129, 1000])
@pytest.mark.parametrize("K,N", [(192, 130), (256, 4096)])
def test_fc_tensor_core_rows(cuda, R, K, N):
    _mlp1(cuda, 1, R, K, N, seed=R)


@pytest.mark.parametrize("engine", [0, 1])
@pytest.mark.parametrize("R,K,N,kernel", [(5, 100, 72, "rows"), (8, 1024, 300, "rows"),
                                          (3000, 80, 300, "wide"), (2816, 1024, 300, "wide"),
                                          (200, 100, 72, "tiled"), (1000, 1024, 300, "tiled"), (65, 6, 64, "tiled")])
def test_fc_fma_kernels(cuda, engine, R, K, N, kernel):
    """The FMA kernels, each selected by the rules of cg_linear_launch: on engine 0, and on engine 1 where the layer
    cannot go to tensor cores (K not a multiple of 64, or too few rows)."""
    on_tc = engine >= 1 and R >= 64 and K % 64 == 0 and N >= 64
    if on_tc:
        pytest.skip("tensor-core layer: covered by the tests above")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert _fma_kernel(R, K, N, sms) == kernel
    _mlp1(cuda, engine, R, K, N, seed=R + K + N)


# ------------------------------------------------------------------------------------------ batches over CHUNK_B
@pytest.mark.parametrize("engine", ENGINES)
def test_cls_batch_over_chunk(cls_pair, engine):
    """B = 16384 + 100 runs as two internal passes.  Both the x input and the fused grasp-Q input must give, bit for
    bit, what separate calls on the two parts give, and a sample must agree with the float64 reference."""
    from catgrasp_b200.synthetic import make_candidates, make_pile
    net, ref = cls_pair
    net.ctx.set_engine(engine)
    B, N = CHUNK_B + 100, 24
    x = np.random.RandomState(9).normal(0, 1, (B, N, 6)).astype(np.float32)
    xd = _dev(x, torch.float32)
    full = net.forward(xd).cpu().numpy()
    head = net.forward(xd[:CHUNK_B]).cpu().numpy()
    tail = net.forward(xd[CHUNK_B:]).cpu().numpy()
    assert np.array_equal(full[:CHUNK_B].view(np.uint32), head.view(np.uint32))
    assert np.array_equal(full[CHUNK_B:].view(np.uint32), tail.view(np.uint32))
    # a sample against the float64 network (end to end, at the logit tolerance of tests/test_gpu_parity.py: error
    # bounds carried through every layer are rigorous but far too loose to be useful)
    sel = np.array([0, 1, 4097, CHUNK_B - 1, CHUNK_B, CHUNK_B + 1, B - 1])
    tol = 5e-4 * (4 if engine >= 2 else 1)
    lg = ref.forward(x[sel], engine=engine)["logits"]
    assert np.abs(full[sel] - lg).max() < tol
    # fused input: the per-pass offsets of poses and ids
    M = 2000
    scene = make_pile(M, n_objects=4, seed=41)
    xyz, nrm = scene["cloud_xyz"], scene["cloud_normal"]
    poses = make_candidates(xyz, nrm, 64, seed=42)[np.random.RandomState(43).randint(0, 64, B)]
    ids = np.random.RandomState(44).randint(0, M, (B, N)).astype(np.int32)
    t = [_dev(a, torch.float64) for a in (xyz, nrm, poses)]
    d_ids = _dev(ids, torch.int32)
    pf, _ = net.graspq_dev(t[0], t[1], t[2], d_ids)
    ph, _ = net.graspq_dev(t[0], t[1], t[2][:CHUNK_B].contiguous(), d_ids[:CHUNK_B].contiguous())
    pt, _ = net.graspq_dev(t[0], t[1], t[2][CHUNK_B:].contiguous(), d_ids[CHUNK_B:].contiguous())
    pf, ph, pt = (a.cpu().numpy() for a in (pf, ph, pt))
    assert np.array_equal(pf[:CHUNK_B].view(np.uint32), ph.view(np.uint32))
    assert np.array_equal(pf[CHUNK_B:].view(np.uint32), pt.view(np.uint32))
    xs, _ = fused_input(xyz, nrm, poses[sel], ids[sel])
    lg = ref.forward(xs, engine=engine)["logits"]
    p = np.exp(lg - lg.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    assert np.abs(pf[sel] - p).max() < 1e-4


# ------------------------------------------------------------------------------------------ the fp16 range
def test_fp16_weight_range_falls_back_to_engine1(cuda):
    """A folded STN3d W3 entry beyond 65504: engines 2 and 3 run that trunk on the engine-1 kernel (bit-identical
    keys), while the encoder trunk still changes engine."""
    from catgrasp_b200.synthetic import make_state_dict
    sd = make_state_dict("cls", 10, seed=6)
    g = sd["module.feat.stn.bn3.weight"].clone()
    g[100] = 1e7
    sd["module.feat.stn.bn3.weight"] = g
    w = sd["module.feat.stn.fc1.weight"].clone()
    w[:, 100] = 0.0                       # keep T3 ordinary: the huge channel does not feed the STN's FC layers
    sd["module.feat.stn.fc1.weight"] = w
    net, ref = _build("cls", 10, sd, cuda)
    assert not ref.f16_ok("A") and ref.f16_ok("B") and ref.f16_ok("C")
    B, N = 4, 500
    x = np.random.RandomState(6).normal(0, 1, (B, N, 6)).astype(np.float32)
    got = {}
    for e in (1, 2, 3):
        net.ctx.set_engine(e)
        got[e] = probe(net, B, N, x=x)
        check_encoder(ref, e, got[e], x, label="W3 beyond fp16")
    for e in (2, 3):
        assert np.array_equal(got[e]["keys"][0], got[1]["keys"][0]), e
        assert not np.array_equal(got[e]["keys"][2], got[1]["keys"][2]), e
    net.ctx.set_engine(3)


def _overflow_state_dict():
    """Eight STN3d layer-2 channels scaled by 1e6 (outputs far beyond 65504 wherever they are positive) and their
    layer-3 weights by 1e-6, so that the network stays ordinary and only the fp16 clamp changes the result."""
    from catgrasp_b200.synthetic import make_state_dict
    sd = make_state_dict("cls", 10, seed=8)
    ch = np.arange(8)
    g = sd["module.feat.stn.bn2.weight"].clone()
    g[ch] *= 1e6
    sd["module.feat.stn.bn2.weight"] = g
    w = sd["module.feat.stn.conv3.weight"].clone()
    w[:, ch] *= 1e-6
    sd["module.feat.stn.conv3.weight"] = w
    return sd


def test_fp16_activation_overflow_is_reported(cuda, tmp_path, capsys):
    """Layer-2 outputs beyond 65504: engines 2 and 3 clamp them and must raise the overflow flag (engine 1 must not);
    reading the flag clears it; GraspPredicter on engine 2 or 3 then re-runs on engine 1: over several chunks, with
    either draw or caller-given ids, without touching numpy's generator, and leaving the shared context as it was."""
    from catgrasp_b200.predicter import GraspPredicter
    from catgrasp_b200.synthetic import make_candidates, make_pile, write_artifacts
    sd = _overflow_state_dict()
    net, ref = _build("cls", 10, sd, cuda)
    x = np.random.RandomState(8).normal(0, 1, (16, 400, 6)).astype(np.float32)
    lg = {}
    for e in (1, 2, 3):
        net.ctx.set_engine(e)
        net.ctx.fp16_overflow()
        lg[e] = net.forward(x).cpu().numpy()
        assert net.ctx.fp16_overflow() == (e >= 2), e
        assert net.ctx.fp16_overflow() is False
    net.ctx.set_engine(3)
    assert np.isfinite(lg[1]).all()
    assert not np.array_equal(lg[2], lg[1]) and not np.array_equal(lg[3], lg[1])
    adir = write_artifacts(str(tmp_path / "artifacts-47"), "cls", n_pts=256, state_dict=sd)
    scene = make_pile(1500, n_objects=3, seed=9)
    data = {"cloud_xyz": scene["cloud_xyz"], "cloud_normal": scene["cloud_normal"]}
    poses = list(make_candidates(scene["cloud_xyz"], scene["cloud_normal"], 13, seed=10))
    M = int((scene["cloud_xyz"][:, 2] >= 0.1).sum())
    given = np.random.RandomState(11).randint(0, M, (13, 256)).astype(np.int32)
    ctx = net.ctx
    for tag, kw in (("host", {"subsample": "host"}), ("device", {"subsample": "device"}), ("ids", {"ids": given})):
        out, nxt = {}, {}
        for e in (1, 2, 3):
            gp = GraspPredicter("nut", artifact_dir=adir, engine=e)
            gp.chunk = 5                      # the host draw runs in chunks of 5, 5 and 3
            for call in (0, 1):               # the second call: no state survives the first
                capsys.readouterr()
                np.random.seed(3)
                probs = np.stack([o[2] for o in gp.predict_batch(data, poses, **kw)])
                nxt[e] = np.random.rand(2)
                assert ("re-running on engine 1" in capsys.readouterr().out) == (e >= 2), (tag, e, call)
                assert ctx.get_engine() == 3 and ctx.fp16_overflow() is False, (tag, e, call)
                assert np.array_equal(probs.view(np.uint32), out.setdefault(e, probs).view(np.uint32)), (tag, e, call)
        for e in (2, 3):                      # the re-run: engine 1's bits, numpy's generator where engine 1 leaves it
            assert np.array_equal(out[e].view(np.uint32), out[1].view(np.uint32)), (tag, e)
            assert np.array_equal(nxt[e], nxt[1]), (tag, e)
