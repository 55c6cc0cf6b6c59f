"""GPU tests (-m gpu): the tensor-core trunk's max-pool keys do not depend on how its persistent grid cuts the batch.

The trunk kernel (engines 1-3) runs one CTA per SM over a balanced range of 128-point tiles, and ranges start and end
inside candidates.  The per-point arithmetic does not depend on the range and the max is exact, so the keys of a
candidate must be the same bit for bit whether it runs in a batch, in a sub-batch cut at another offset, or alone.

Trunks B and C take T3 / T64 from FC layers whose kernel is chosen by the row count (cg_linear_launch), so their keys
are compared where those inputs are the same: between batches of >= 64 rows, and for a candidate alone wherever its T3
(and T64) equal the batch's.  Trunk A depends on the input alone and is compared everywhere.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TC_ENGINES = [1, 2, 3]
CHUNK_B = 16384   # candidates per internal pass of the cls forward (cg_net.cu)
M_SCENE = 3000


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def nets(cuda):
    from catgrasp_b200.net import PointNetCls, PointNetSeg
    from catgrasp_b200.synthetic import make_state_dict
    return {"ids": PointNetCls(make_state_dict("cls", 10, seed=0), device=0),
            "x": PointNetSeg(make_state_dict("seg", 300, seed=1), device=0)}


@pytest.fixture(scope="module")
def scene(cuda):
    from catgrasp_b200.synthetic import make_candidates, make_pile
    s = make_pile(M_SCENE, n_objects=4, seed=21)
    poses = make_candidates(s["cloud_xyz"], s["cloud_normal"], 4096, seed=22)
    return [torch.from_numpy(np.ascontiguousarray(a)).to("cuda", torch.float64)
            for a in (s["cloud_xyz"], s["cloud_normal"], poses)]


def make_inputs(src, B, N, seed):
    """Per-candidate inputs on the device: (poses, ids) for the fused grasp-Q input, or (x,) for the x input."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if src == "ids":
        ids = torch.randint(0, M_SCENE, (B, N), generator=g, device="cuda", dtype=torch.int32)
        pose_idx = torch.randint(0, 4096, (B,), generator=g, device="cuda")
        return pose_idx, ids
    return (torch.randn((B, N, 6), generator=g, device="cuda", dtype=torch.float32),)


def rows(inp, sel):
    return tuple(a[sel].contiguous() for a in inp)


def probe(net, scene, src, inp):
    """cg_encoder_probe_dev on device tensors: keys (3,B,1024) i32, T3, T64 and (x input) the point feature."""
    from catgrasp_b200 import _lib
    ctx = net.ctx
    ctx.use_torch_stream()
    if src == "ids":
        pose_idx, ids = inp
        B, N = ids.shape
        poses = scene[2][pose_idx].contiguous()
        args = (None, _lib.ptr(scene[0]), _lib.ptr(scene[1]), M_SCENE, _lib.ptr(poses), _lib.ptr(ids), None, None)
        pf = None
    else:
        (x,) = inp
        B, N = x.shape[:2]
        args = (_lib.ptr(x), None, None, 0, None, None, None, None)
        pf = torch.empty((B, N, 64), dtype=torch.float32, device="cuda")
    keys = torch.zeros((3, B, 1024), dtype=torch.int32, device="cuda")
    T3 = torch.empty((B, 9), dtype=torch.float32, device="cuda")
    T64 = torch.empty((B, 4096), dtype=torch.float32, device="cuda")
    ctx.check(ctx.lib.cg_encoder_probe_dev(net.h, *args, B, N, _lib.ptr(keys), _lib.ptr(T3), _lib.ptr(T64),
                                           _lib.ptr(pf)))
    torch.cuda.synchronize()
    return {"keys": keys, "T3": T3.view(torch.int32), "T64": T64.view(torch.int32),
            "pf": None if pf is None else pf.view(torch.int32)}


def same(a, b):
    return a.shape == b.shape and torch.equal(a, b)


def assert_rows_equal(full, sel, sub, label):
    """Every output of a sub-batch of >= 64 rows equals the batch's rows sel, bit for bit."""
    for t in range(3):
        assert same(full["keys"][t][sel], sub["keys"][t]), (label, "trunk", "ABC"[t])
    assert same(full["T3"][sel], sub["T3"]), (label, "T3")
    assert same(full["T64"][sel], sub["T64"]), (label, "T64")
    if sub["pf"] is not None:
        assert same(full["pf"][sel], sub["pf"]), (label, "pf")


def assert_alone_equal(full, b, one, label):
    """A candidate run alone: trunk A always; trunks B / C (and the point feature) where their T3 / T64 agree."""
    assert same(full["keys"][0][b:b + 1], one["keys"][0]), (label, b, "trunk A")
    if same(full["T3"][b:b + 1], one["T3"]):
        assert same(full["keys"][1][b:b + 1], one["keys"][1]), (label, b, "trunk B")
        if same(full["T64"][b:b + 1], one["T64"]):
            assert same(full["keys"][2][b:b + 1], one["keys"][2]), (label, b, "trunk C")
            if one["pf"] is not None:
                assert same(full["pf"][b:b + 1], one["pf"]), (label, b, "pf")


@pytest.mark.parametrize("src", ["ids", "x"])
@pytest.mark.parametrize("N", [1, 127, 128, 129, 1024, 8192])
@pytest.mark.parametrize("engine", TC_ENGINES)
def test_keys_do_not_depend_on_the_cut(nets, scene, engine, N, src):
    """B = 133 candidates (one more than the SMs of an H100 SXM: ranges start inside candidates, or hold 1 or 2
    one-tile candidates at N <= 128) against sub-batches cut at other offsets, 64 copies of one candidate (its tiles
    spread over many ranges), and candidates alone."""
    net = nets[src]
    net.ctx.set_engine(engine)
    B = 133
    inp = make_inputs(src, B, N, seed=N * 7 + engine)
    full = probe(net, scene, src, inp)
    for lo, hi in [(0, 64), (64, B), (5, 69), (69, B), (1, 132)]:
        sel = torch.arange(lo, hi, device="cuda")
        assert_rows_equal(full, sel, probe(net, scene, src, rows(inp, sel)), f"rows {lo}:{hi}")
    for b in (0, 1, 66, 131, 132):
        sel = torch.full((64,), b, device="cuda")
        assert_rows_equal(full, sel, probe(net, scene, src, rows(inp, sel)), f"64 x row {b}")
        one = probe(net, scene, src, rows(inp, torch.tensor([b], device="cuda")))
        assert_alone_equal(full, b, one, "alone")
    net.ctx.set_engine(3)


@pytest.mark.parametrize("src", ["ids", "x"])
@pytest.mark.parametrize("N", [129, 1024])
@pytest.mark.parametrize("B", [1, 2, 131, 132, 133, 4096])
@pytest.mark.parametrize("engine", TC_ENGINES)
def test_batch_sizes_against_a_4096_batch(nets, scene, engine, B, N, src):
    """Batches of B candidates taken from the head and the tail of a 4096-candidate batch; at B = 1, 2 the grid has
    fewer CTAs than SMs (B x ntiles < 132) and every CTA holds one tile."""
    net = nets[src]
    net.ctx.set_engine(engine)
    inp = make_inputs(src, 4096, N, seed=B + N)
    full = probe(net, scene, src, inp)
    for lo in (0, 4096 - B):
        sel = torch.arange(lo, lo + B, device="cuda")
        sub = probe(net, scene, src, rows(inp, sel))
        if B >= 64:
            assert_rows_equal(full, sel, sub, f"rows {lo}:{lo + B}")
        else:
            for i in range(B):
                row = {"keys": sub["keys"][:, i:i + 1], "T3": sub["T3"][i:i + 1], "T64": sub["T64"][i:i + 1],
                       "pf": None if sub["pf"] is None else sub["pf"][i:i + 1]}
                assert_alone_equal(full, lo + i, row, f"rows {lo}+{i}")
    net.ctx.set_engine(3)


@pytest.mark.parametrize("engine", TC_ENGINES)
def test_grasp_q_batch_over_chunk(nets, scene, engine):
    """B = 16385 runs as two internal passes (the second one candidate): the probabilities equal, bit for bit, those
    of separate calls on the two parts."""
    net = nets["ids"]
    net.ctx.set_engine(engine)
    B, N = CHUNK_B + 1, 129
    pose_idx, ids = make_inputs("ids", B, N, seed=5)
    poses = scene[2][pose_idx].contiguous()
    full, _ = net.graspq_dev(scene[0], scene[1], poses, ids)
    head, _ = net.graspq_dev(scene[0], scene[1], poses[:CHUNK_B].contiguous(), ids[:CHUNK_B].contiguous())
    tail, _ = net.graspq_dev(scene[0], scene[1], poses[CHUNK_B:].contiguous(), ids[CHUNK_B:].contiguous())
    torch.cuda.synchronize()
    assert torch.equal(full[:CHUNK_B].view(torch.int32), head.view(torch.int32))
    assert torch.equal(full[CHUNK_B:].view(torch.int32), tail.view(torch.int32))
    net.ctx.set_engine(3)


def test_fp16_overflow_is_reported_from_every_range(cuda):
    """Layer-2 outputs beyond 65504 in one candidate only, near the end of a 133-candidate batch: engines 2 and 3 must
    raise the overflow flag, engine 1 must not, and the other candidates' keys are those of a batch without it."""
    from catgrasp_b200.net import PointNetCls
    from catgrasp_b200.synthetic import make_state_dict
    sd = make_state_dict("cls", 10, seed=8)
    net = PointNetCls(sd, device=0)
    B, N, hot = 133, 1024, 130
    (x,) = make_inputs("x", B, N, seed=8)
    x_hot = x.clone()
    x_hot[hot] *= 1e5   # the STN3d trunk's layer-2 activations of this candidate leave the fp16 range
    for e in (1, 2, 3):
        net.ctx.set_engine(e)
        net.ctx.fp16_overflow()
        cold = probe(net, None, "x", (x,))
        assert net.ctx.fp16_overflow() is False, e
        hot_run = probe(net, None, "x", (x_hot,))
        assert net.ctx.fp16_overflow() == (e >= 2), e
        keep = torch.arange(B, device="cuda") != hot
        assert torch.equal(cold["keys"][0][keep], hot_run["keys"][0][keep]), e
    net.ctx.set_engine(3)
