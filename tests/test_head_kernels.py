"""GPU tests (-m gpu) of what the networks compute after their logits, and of the host entry points that feed them.

- softmax_kernel (cg_linear.cu): the grasp-Q probabilities against a float64 softmax within a written-out bound, and
  the label as the reference takes it: softmax, then the argmax of the float32 probabilities, the first maximum
  winning (predicter.py:86-89).
- nunocs_post_kernel: the NUNOCS bins (first maximum of each axis' logits), coords bit for bit against the reference's
  float32 arithmetic (predicter.py:145-150) and confidence_z against float64.
- The seg head's per-cloud bias (the global half of its first conv) on every FC kernel cg_linear_launch picks for it.
- cg_graspq_forward_host given its ids pageable, pinned, as a view into a pinned buffer and in a reused pinned buffer.

Most of the post-processing tests use nets whose last layer has zero weights.  Every FC kernel then returns that
layer's bias as the logits, bit for bit (the products are zero, and so are the bf16 hi / lo parts of 0), so ties,
near-ties and underflow are set by construction.  Every comparison against a bound prints its largest
error / (2 x bound) ratio.
"""
import numpy as np
import pytest
import torch

from oracle.encoder_ref import FoldedNet, bound_ratio
from test_tc_kernels import (CHUNK_B, ENGINES, _build, _dev, _fma_kernel, check_encoder, cls_pair,  # noqa: F401
                             cuda, probe, seg_pair)

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
EXPF = 2.0 ** -22        # expf: at most 2 ulp (CUDA C++ Programming Guide, single-precision mathematical functions)
SUB = 2.0 ** -148        # absolute error of an expf result or a quotient in the subnormal range (2 ulp of 2^-149)


# ------------------------------------------------------------------------------------------ references
def softmax64(lg):
    """float64 softmax over the last axis of float32 logits, and the shifted logits d = l - max."""
    l = np.asarray(lg, np.float64)
    d = l - l.max(-1, keepdims=True)
    e = np.exp(d)
    return e / e.sum(-1, keepdims=True), d


def softmax_bound(p, d):
    """Bound on |p32 - p| for p32_i = expf(fl(l_i - m)) / sum_j expf(fl(l_j - m)) in float32:
        fl(l - m)        relative 2^-24 of d, which changes exp(d) by |d| 2^-24 (relative)
        expf             2 ulp = 2^-22 relative; SUB absolute where the result is subnormal
        the sum          C - 1 roundings of positive terms: (C - 1) 2^-24 relative; C SUB absolute
        the division     2^-24 relative, SUB absolute for a subnormal quotient
    The sum holds expf(0) = 1 (the maximum), so an absolute error of the sum moves p by at most that much."""
    C = p.shape[-1]
    dm = np.abs(d).max(-1, keepdims=True)
    return p * ((np.abs(d) + dm) * U32 + 2 * EXPF + C * U32) + (C + 2) * SUB


def conf_bound(conf, d):
    """Bound on confidence_z = 1 / sum_k expf(fl(l_k - m)) over one axis (the softmax probability at its argmax)."""
    bins = d.shape[-1]
    return conf * (np.abs(d).max(-1) * U32 + EXPF + bins * U32) + (bins + 2) * SUB


def ref_coords(bins_idx, bins):
    """predicter.py:145-150: pred.argmax(dim=-1).float() * bin_resolution, then .numpy() - 0.5, on the CPU."""
    return (torch.from_numpy(np.asarray(bins_idx, np.int64)).float() * (1 / bins)).numpy() - 0.5


def report(label, got, ref, err):
    r = float(bound_ratio(got, ref, err).max())
    print(f"\nRATIO {label} {r:.3g}")
    assert r <= 1.0, (label, r)


def assert_bits(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), what


def bias_net(kind, bias, seed):
    """A PointNetCls / PointNetSeg whose last layer (fc3 / conv4) has zero weights: its logits are ``bias`` on every
    row.  Returns (net, state_dict)."""
    from catgrasp_b200.net import PointNetCls, PointNetSeg
    from catgrasp_b200.synthetic import make_state_dict
    bias = np.asarray(bias, np.float32)
    sd = make_state_dict(kind, bias.size, seed=seed)
    last = "module.fc3" if kind == "cls" else "module.conv4"
    sd[last + ".weight"] = torch.zeros_like(sd[last + ".weight"])
    sd[last + ".bias"] = torch.from_numpy(bias.copy())
    return (PointNetCls if kind == "cls" else PointNetSeg)(sd, device=0), sd


# ------------------------------------------------------------------------------------------ softmax, logits set
SOFTMAX_NOUT = [1, 2, 10, 31, 32]
SOFTMAX_B = [1, 7, 8, 9, CHUNK_B + 3]      # 8 rows per block; B > CHUNK_B runs two internal passes


def softmax_case(case, C, rng):
    """(logits (C,) float32, the label the reference gives) for one case; None where C is too small for it."""
    t = rng.uniform(-4.0, -1.0, C).astype(np.float32)
    if case == "equal":                     # every class the same: probabilities 1/C, label 0
        t[:] = np.float32(0.3)
        return t, 0
    if case == "tie":                       # an exact tie at the maximum, two random classes
        if C < 2:
            return None
        i, j = sorted(rng.choice(C, 2, replace=False))
        t[i] = t[j] = np.float32(2.5)
        return t, i
    if case == "tie_ends":                  # lanes 0 and C - 1
        if C < 3:
            return None
        t[0] = t[C - 1] = np.float32(2.5)
        return t, 0
    if case in ("near_tie", "near_tie_mirror"):
        # logits 0 and 1e-30: expf(-1e-30) rounds to 1, so both probabilities are equal and the lower class wins,
        # whichever of the two logits is larger
        if C < 2:
            return None
        i = C - 2 if C > 2 else 0
        t[i], t[i + 1] = (0.0, 1e-30) if case == "near_tie" else (1e-30, 0.0)
        return t, i
    if case == "underflow":                 # logits +-90: expf(-180) underflows to 0; ties among the +90 classes
        t = np.where(rng.rand(C) < 0.5, 90.0, -90.0).astype(np.float32)
        t[rng.randint(C)] = 90.0
        return t, int(np.argmax(t))
    raise ValueError(case)


SOFTMAX_CASES = [(C, case) for C in SOFTMAX_NOUT
                 for case in ("equal", "tie", "tie_ends", "near_tie", "near_tie_mirror", "underflow")
                 if softmax_case(case, C, np.random.RandomState(0)) is not None]


@pytest.mark.parametrize("C,case", SOFTMAX_CASES)
def test_softmax_and_label_on_set_logits(cuda, C, case):
    """Probabilities within the float64 bound, label == argmax of the written probabilities (lowest class on a tie) ==
    the fp32 torch oracle's softmax + argmax, through cg_graspq_forward_dev (probs + label) and cg_cls_forward_dev
    (logits + probs), at every row of every batch size."""
    from oracle.pointnet_ref import pointnet_cls_forward
    rng = np.random.RandomState(C * 131 + len(case))
    lg, want = softmax_case(case, C, rng)
    net, sd = bias_net("cls", lg, seed=C)
    M, N = 32, 4
    cloud = np.random.RandomState(1).normal(0, 0.05, (2, M, 3))
    x1 = np.random.RandomState(2).normal(0, 1, (1, N, 6)).astype(np.float32)
    ref_lg = pointnet_cls_forward(sd, x1)[0]
    assert_bits(ref_lg.numpy()[0], lg, "oracle logits == the bias")
    oracle_label = int(ref_lg.softmax(dim=1).argmax(dim=1)[0])
    assert oracle_label == want, (oracle_label, want)
    p64, d = softmax64(lg)
    err = softmax_bound(p64, d)
    xyz, nrm = _dev(cloud[0], torch.float64), _dev(cloud[1], torch.float64)
    for B in SOFTMAX_B:
        poses = torch.eye(4, dtype=torch.float64, device="cuda").expand(B, 4, 4).contiguous()
        ids = torch.zeros((B, N), dtype=torch.int32, device="cuda")
        probs, label = net.graspq_dev(xyz, nrm, poses, ids)
        x = torch.zeros((B, N, 6), dtype=torch.float32, device="cuda")
        logits, probs2 = net.forward(x, return_probs=True)
        probs, label, logits, probs2 = (a.cpu().numpy() for a in (probs, label, logits, probs2))
        assert_bits(logits, np.broadcast_to(lg, (B, C)), f"logits == the bias, B={B}")
        assert_bits(probs, np.broadcast_to(probs[0], (B, C)), f"every row alike, B={B}")
        assert_bits(probs2, probs, f"cls forward probs == graspq probs, B={B}")
        report(f"softmax C={C} {case} B={B}", probs[0], p64, err)
        assert (label == np.argmax(probs[0])).all(), (B, np.unique(label), probs[0])
        assert (label == oracle_label).all(), (B, np.unique(label), oracle_label)


def test_softmax_rejects_more_than_32_classes(cuda):
    """The softmax runs one warp per row: a PointNetCls with 33 outputs is refused with CG_EINVAL and a message."""
    from catgrasp_b200._lib import CgError
    with pytest.raises(CgError, match="error -1: invalid argument: n_out"):
        bias_net("cls", np.zeros(33, np.float32), seed=33)


# ------------------------------------------------------------------------------------------ NUNOCS, logits set
NUNOCS_BINS = [1, 31, 32, 33, 100, 129]


def nunocs_row(case, bins, rng):
    """(logits (bins,) float32, the first-maximum bin) of one axis; None where bins is too small for the case.
    A value one ulp below the maximum sits before (or in the same lane as) the winner where there is room."""
    top = np.float32(1.5)
    below = np.nextafter(top, np.float32(-np.inf))
    t = rng.uniform(-3.0, 1.0, bins).astype(np.float32)
    if case == "same_lane":                 # ties at k and k + 32: one lane sees both
        if bins < 33:
            return None
        k = rng.randint(0, bins - 32)
        t[k] = t[k + 32] = top
        if k > 0:
            t[rng.randint(0, k)] = below
        return t, k
    if case == "next_lane":                 # ties at k and k + 1: two lanes meet in the shuffle
        if bins < 2:
            return None
        k = rng.randint(0, bins - 1)
        t[k] = t[k + 1] = top
        if k > 0:
            t[k - 1] = below
        return t, k
    if case == "last":                      # the maximum in the last bin
        t[bins - 1] = top
        if bins > 32:
            t[bins - 33] = below
        return t, bins - 1
    if case == "equal":
        t[:] = top
        return t, 0
    raise ValueError(case)


@pytest.mark.parametrize("bins", NUNOCS_BINS)
def test_nunocs_post_on_set_logits(cuda, bins):
    """Bins, coords and confidence_z of cg_nunocs_forward_dev / _host for logits set per axis.  Every case sits on
    every axis once (the cases rotate over the three axes), so confidence_z sees each of them."""
    cases = [c for c in ("same_lane", "next_lane", "last", "equal")
             if nunocs_row(c, bins, np.random.RandomState(0)) is not None]
    for rot in range(len(cases)):
        rng = np.random.RandomState(bins * 17 + rot)
        rows = [nunocs_row(cases[(a + rot) % len(cases)], bins, rng) for a in range(3)]
        lg = np.stack([r[0] for r in rows])                         # (3, bins)
        want = np.array([r[1] for r in rows], np.int32)
        assert (np.argmax(lg, -1) == want).all()
        net, _ = bias_net("seg", lg.reshape(-1), seed=bins + rot)
        p64, d = softmax64(lg[2])
        conf64 = p64[want[2]]
        err = conf_bound(conf64, d)
        label = f"bins={bins} axes={[cases[(a + rot) % len(cases)] for a in range(3)]}"
        for N in (1, 100):                  # the head's last layer on the few-row FMA kernel, and on the wider ones
            x = np.random.RandomState(N).normal(0, 1, (N, 6)).astype(np.float32)
            logits = net.forward(x[None]).cpu().numpy()[0]
            assert_bits(logits, np.broadcast_to(lg.reshape(-1), (N, 3 * bins)), f"logits == the bias, N={N}")
            c, z, b = (a.cpu().numpy() for a in net.nunocs_dev(x, bins))
            hc, hz, hb = net.nunocs_host(x, bins)
            assert_bits(hc, c, "host coords == dev coords")
            assert_bits(hz, z, "host conf_z == dev conf_z")
            assert np.array_equal(hb, b), "host bins == dev bins"
            assert (b == want).all(), (label, N, b[0], want)
            assert_bits(c, np.broadcast_to(ref_coords(want, bins), (N, 3)), f"coords {label}")
            report(f"conf_z {label} N={N}", z, np.full(N, conf64), np.full(N, err))


def test_reference_coords_round_the_resolution_to_float32_first():
    """The reference's bin * (1 / bins) multiplies a float32 tensor by a Python float: torch rounds the scalar to
    float32 first, so its coords are float32(bin) * float32(1 / bins) - 0.5 in float32, which is what the kernel does."""
    for bins in NUNOCS_BINS + [3, 7, 10, 50, 64, 1000]:
        k = np.arange(bins)
        want = (k.astype(np.float32) * np.float32(1 / bins)) - np.float32(0.5)
        assert want.dtype == np.float32
        assert_bits(ref_coords(k, bins), want, bins)
        assert np.float32(1 / bins) == np.float32(1) / np.float32(bins)     # the kernel's 1.0f / bins


# ------------------------------------------------------------------------------------------ the GPU's own logits
@pytest.fixture(scope="module")
def seg_nets(cuda):
    from catgrasp_b200.net import PointNetSeg
    from catgrasp_b200.synthetic import make_state_dict
    return {bins: PointNetSeg(make_state_dict("seg", 3 * bins, seed=50 + bins), device=0) for bins in (33, 100)}


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("bins", [33, 100])
@pytest.mark.parametrize("N", [1, 7, 8, 8193])
def test_nunocs_post_on_gpu_logits(seg_nets, engine, bins, N):
    """cg_seg_forward_dev's logits and cg_nunocs_forward_dev on the same input: first-maximum bins, coords bit for
    bit, confidence_z within its float64 bound; the host entry point equal to the device one bit for bit."""
    net = seg_nets[bins]
    net.ctx.set_engine(engine)
    x = np.random.RandomState(N * 3 + bins).normal(0, 1, (N, 6)).astype(np.float32)
    lg = net.forward(x[None]).cpu().numpy()[0].reshape(N, 3, bins)
    c, z, b = (a.cpu().numpy() for a in net.nunocs_dev(x, bins))
    hc, hz, hb = net.nunocs_host(x, bins)
    net.ctx.set_engine(3)
    assert_bits(hc, c, "host coords == dev coords")
    assert_bits(hz, z, "host conf_z == dev conf_z")
    assert np.array_equal(hb, b)
    want = np.argmax(lg, -1)
    assert np.array_equal(b, want)
    assert_bits(c, ref_coords(want, bins), "coords")
    p64, d = softmax64(lg[:, 2])
    conf64 = p64[np.arange(N), want[:, 2]]
    report(f"engine={engine} conf_z bins={bins} N={N}", z, conf64, conf_bound(conf64, d))


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("B", [1, 9, 4097])
def test_cls_probs_on_gpu_logits(cls_pair, engine, B):
    net, _ = cls_pair
    net.ctx.set_engine(engine)
    x = np.random.RandomState(B).normal(0, 1, (B, 32, 6)).astype(np.float32)
    logits, probs = (a.cpu().numpy() for a in net.forward(x, return_probs=True))
    net.ctx.set_engine(3)
    p64, d = softmax64(logits)
    report(f"engine={engine} cls probs B={B}", probs, p64, softmax_bound(p64, d))


# ------------------------------------------------------------------------------------------ seg head, per-cloud bias
# (B, N, kernel of the 64 -> 512 point half that adds the per-cloud bias); P = B x N rows
SEG_SHAPES = [(2, 3, "rows"), (8, 1, "rows"), (1, 8, "rows"), (4, 300, "tiled"), (3, 1000, "wide"),
              (5, 431, "tc"), (17, 129, "tc")]      # cloud boundaries inside 64- and 128-row tiles
SEG_RUNS = [(e, B, N, k) for e in ENGINES for B, N, k in SEG_SHAPES
            if k == "rows" or (k == "tc") == (e >= 1)]


@pytest.fixture(scope="module")
def seg_passthrough(cuda):
    """A PointNetSeg whose conv2, conv3 and conv4 pass their first channels through unchanged (weights 0 and 1, a
    BatchNorm that folds to the identity, bias 0): its logits are the first 128 channels of the layer that adds the
    per-cloud bias.  Random layers after that one widen the float64 bound of the logits past what another cloud's
    bias row changes; with these the bound stays near that layer's own."""
    from catgrasp_b200.synthetic import make_state_dict
    n_out = 300
    sd = make_state_dict("seg", n_out, seed=2)
    for conv, bn, cout, cin in (("conv2", "bn2", 256, 512), ("conv3", "bn3", 128, 256), ("conv4", None, n_out, 128)):
        w = torch.zeros((cout, cin, 1))
        k = torch.arange(min(cout, cin))
        w[k, k, 0] = 1.0
        sd[f"module.{conv}.weight"] = w
        sd[f"module.{conv}.bias"] = torch.zeros(cout)
        if bn:
            sd[f"module.{bn}.weight"] = torch.ones(cout)
            sd[f"module.{bn}.bias"] = torch.zeros(cout)
            sd[f"module.{bn}.running_mean"] = torch.zeros(cout)
            sd[f"module.{bn}.running_var"] = torch.full((cout,), 1 - 1e-5)   # var + eps = 1: the fold is exact
    net, ref = _build("seg", n_out, sd, cuda)
    for name in ("HEAD2", "HEAD3", "HEAD4"):
        assert set(torch.unique(ref.W[name]).tolist()) == {0.0, 1.0} and not ref.b[name].any(), name
    return net, ref


@pytest.mark.parametrize("engine,B,N,kernel", SEG_RUNS)
def test_seg_head_per_cloud_bias_on_every_fc_kernel(seg_pair, seg_passthrough, engine, B, N, kernel):
    """The point half of the seg head's first conv adds cloud b's row of the global half to points b*N .. b*N+N-1.
    Checked on a random net and on one whose logits are that layer's output (seg_passthrough)."""
    P = B * N
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert FoldedNet.fc_on_tc(engine, P, 64, 512) == (kernel == "tc")
    if kernel != "tc":
        assert _fma_kernel(P, 64, 512, sms) == kernel
    x = np.random.RandomState(B * 1009 + N).normal(0, 1, (B, N, 6)).astype(np.float32)
    for which, (net, ref) in (("random", seg_pair), ("passthrough", seg_passthrough)):
        net.ctx.set_engine(engine)
        got = probe(net, B, N, x=x, want_pf=True)
        logits = net.forward(x).cpu().numpy()
        net.ctx.set_engine(3)
        check_encoder(ref, engine, got, x, logits=logits, label=f"seg head {which} {kernel} N={N}")


# ------------------------------------------------------------------------------------------ host entry points
@pytest.fixture(scope="module")
def pile(cuda):
    from catgrasp_b200.synthetic import make_candidates, make_pile
    scene = make_pile(2000, n_objects=4, seed=61)
    xyz, nrm = scene["cloud_xyz"], scene["cloud_normal"]
    return xyz, nrm, make_candidates(xyz, nrm, 64, seed=62)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("B,N", [(130, 300), (CHUNK_B + 100, 24)])
@pytest.mark.parametrize("norm", [False, True])
def test_graspq_host_ids_from_any_host_memory(cls_pair, pile, engine, B, N, norm):
    """cg_graspq_forward_host reads pinned ids in place (mapped host memory) and copies pageable ones: both, a view at
    a non-zero offset into a larger pinned buffer, and a pinned buffer refilled between two calls give what
    cg_graspq_forward_dev gives with device ids, bit for bit.  B > CHUNK_B offsets the mapped pointer in its second
    internal pass."""
    net, _ = cls_pair
    net.ctx.set_engine(engine)
    xyz, nrm, cand = pile
    rng = np.random.RandomState(B + N + norm)
    poses = cand[rng.randint(0, len(cand), B)]
    ids1, ids2 = rng.randint(0, len(xyz), (2, B, N)).astype(np.int32)
    mean = std = None
    if norm:
        mean = np.concatenate([rng.normal(0, 0.002, 3), rng.normal(0, 0.05, 3)])
        std = np.concatenate([rng.uniform(0.008, 0.012, 3), rng.uniform(0.5, 0.6, 3)])
    d = [_dev(a, torch.float64) for a in (xyz, nrm, poses, mean, std)]

    def dev(ids):
        p, l = net.graspq_dev(d[0], d[1], d[2], _dev(ids, torch.int32), d[3], d[4])
        return p.cpu().numpy(), l.cpu().numpy()

    def host(ids, how, want):
        p, l = net.graspq_host(xyz, nrm, poses, ids, mean, std)
        assert_bits(p, want[0], f"probs, ids {how}")
        assert np.array_equal(l, want[1]), f"labels, ids {how}"

    want1, want2 = dev(ids1), dev(ids2)
    assert not np.array_equal(want1[0], want2[0])
    host(ids1, "pageable", want1)
    pinned = torch.from_numpy(ids1.copy()).pin_memory()
    assert pinned.is_pinned()
    host(pinned, "pinned", want1)
    off = 777
    big = torch.full((off + B * N + 5,), -1, dtype=torch.int32).pin_memory()
    view = big[off: off + B * N].view(B, N)
    view.copy_(torch.from_numpy(ids1))
    host(view, f"view at element {off} of a pinned buffer", want1)
    pinned.copy_(torch.from_numpy(ids2))
    host(pinned, "pinned, refilled", want2)
    net.ctx.set_engine(3)
