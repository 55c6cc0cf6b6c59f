"""The ctypes prototype table (catgrasp_b200/_lib.py) against include/catgrasp_b200.h, and the checks Context.call
makes before a launch.

CPU: every pointer parameter of the header has a space in SIGNATURES (HostBuf / DevBuf, or c_void_p for a handle),
every entry has the stream its kind needs, and the parameter types accept and refuse what they should.
GPU: bad arguments raise before the entry point is called.  The ctypes function is replaced by a recording stub, so a
missing check fails the test instead of launching with a bad pointer; the context still works afterwards.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from catgrasp_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HANDLE = re.compile(r"\bcg_(ctx|net|sdf|mlp|cloud_index)\s*\*\s*\w+$")


def _prototypes():
    """{name: [(declaration, mark)]} from the header; mark is 'host' / 'device' for a parameter marked in a comment."""
    src = open(os.path.join(ROOT, "include", "catgrasp_b200.h")).read()
    src = re.sub(r"/\*\s*(host|device)\s*\*/", r"@\1", src)
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for name, params in re.findall(r"\b(cg_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", src):
        decls = [p.strip() for p in params.split(",") if p.strip() not in ("", "void")]
        out[name] = [(re.sub(r"\s*@\w+", "", d), (re.findall(r"@(\w+)", d) or [None])[0]) for d in decls]
    return out


def test_every_pointer_parameter_has_a_space():
    protos = _prototypes()
    assert set(protos) == set(_lib.SIGNATURES)
    for name, params in protos.items():
        argtypes = _lib.SIGNATURES[name][1]
        assert len(argtypes) == len(params), name
        for (decl, mark), t in zip(params, argtypes):
            if HANDLE.search(decl) or decl == "void *cuda_stream":
                assert t is C.c_void_p, (name, decl)
            elif "*" in decl or "[" in decl:
                device = mark == "device" or (mark is None and name.endswith("_dev") and "**" not in decl)
                assert t is (_lib.DevBuf if device else _lib.HostBuf), (name, decl)
            else:
                assert t not in (_lib.HostBuf, _lib.DevBuf, C.c_void_p), (name, decl)


def test_every_entry_has_the_stream_of_its_kind():
    streams = {name: s for name, (_, _, s) in _lib.SIGNATURES.items()}
    for name, s in streams.items():
        if name.endswith("_dev"):
            assert s == _lib.TORCH, name
        elif name.endswith("_host"):
            assert s == _lib.OWN, name
    assert streams["cg_cloud_index_create"] == _lib.TORCH
    for name in ("cg_net_create", "cg_sdf_create", "cg_mlp_create", "cg_sdf_from_mesh", "cg_sdf_download"):
        assert streams[name] == _lib.OWN, name
    for name in ("cg_sdf_geometry", "cg_cloud_index_info", "cg_net_destroy", "cg_sdf_destroy", "cg_mlp_destroy",
                 "cg_cloud_index_destroy", "cg_ctx_set_stream", "cg_ctx_synchronize"):
        assert streams[name] is None, name


def test_host_parameter_takes_host_buffers_and_raw_pointers():
    a = np.arange(6, dtype=np.float32)
    t = torch.arange(6, dtype=torch.float32)
    assert _lib.HostBuf.from_param(a).value == a.ctypes.data
    assert _lib.HostBuf.from_param(t).value == t.data_ptr()
    assert _lib.HostBuf.from_param(None) is None
    p = C.c_void_p(1234)
    assert _lib.HostBuf.from_param(p) is p
    v = C.c_int()
    assert _lib.HostBuf.from_param(C.byref(v)) is not None
    assert _lib.HostBuf.from_param((C.c_float * 3)()) is not None
    with pytest.raises(ValueError):
        _lib.HostBuf.from_param(a[::2])
    with pytest.raises(ValueError):
        _lib.HostBuf.from_param(t.reshape(2, 3)[:, :2])
    with pytest.raises(ValueError):
        _lib.HostBuf.from_param(np.zeros((3, 2), np.float32).T)


def test_device_parameter_refuses_host_buffers():
    p = C.c_void_p(1234)
    assert _lib.DevBuf.from_param(p) is p
    assert _lib.DevBuf.from_param(None) is None
    assert _lib.DevBuf.from_param(4096) is not None
    with pytest.raises(TypeError):
        _lib.DevBuf.from_param(np.zeros(3))
    with pytest.raises(TypeError):
        _lib.DevBuf.from_param(torch.zeros(3))


def test_raw_calls_keep_taking_ptr_arguments():
    """A raw prototype call with _lib.ptr() pointers and ctypes arrays still reaches the library (no device needed)."""
    lib = _lib.load()
    p = np.array([[0.0, 0.0, 0.0], [0.01, 0.02, 0.03]], np.float32)
    dims, org = (C.c_int * 3)(), (C.c_float * 3)()
    assert lib.cg_occupancy_grid_geometry(_lib.ptr(p), 2, C.c_float(0.005), dims, org) == _lib.CG_OK
    d2, o2 = np.empty(3, np.int32), np.empty(3, np.float32)
    assert lib.cg_occupancy_grid_geometry(p, 2, 0.005, d2, o2) == _lib.CG_OK
    assert list(d2) == list(dims) and list(o2) == list(org)


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)
    return _lib.Context.get(0)


@pytest.fixture
def stub(monkeypatch):
    """stub(ctx, name): replace entry `name` of ctx's library by a recorder; returns the list of its calls."""
    def install(ctx, name):
        calls = []
        monkeypatch.setattr(ctx.lib, name, lambda *a: calls.append(a) or 0)
        return calls
    return install


def _refused(ctx, calls, fn, *errors):
    before = ctx.launch_count()
    with pytest.raises(errors or (_lib.CgError, TypeError, ValueError)):
        fn()
    assert calls == [] and ctx.launch_count() == before


def _still_works(ctx):
    """A launch no test stubs runs and gives its answer: every point's ball holds points 0 and 1 first."""
    from catgrasp_b200.pointnet2 import query_ball_point
    before = ctx.launch_count()
    a = torch.rand((1, 5, 3), device="cuda")
    got = query_ball_point(10.0, 2, a, a).cpu()
    assert (got == torch.tensor([0, 1])).all() and ctx.launch_count() > before


@pytest.mark.gpu
def test_host_parameter_refuses_a_cuda_tensor(ctx):
    with pytest.raises(TypeError):
        _lib.HostBuf.from_param(torch.zeros(3, device="cuda"))
    t = torch.zeros(3, device="cuda")
    assert _lib.DevBuf.from_param(t).value == t.data_ptr()
    with pytest.raises(ValueError):
        _lib.DevBuf.from_param(torch.zeros((4, 4), device="cuda")[:, :2])


@pytest.mark.gpu
def test_cpu_index_and_cpu_points_are_refused(ctx, stub):
    from catgrasp_b200.pointnet2 import index_points, square_distance
    pts = torch.rand((2, 16, 3), device="cuda")
    calls = stub(ctx, "cg_index_points_dev")
    _refused(ctx, calls, lambda: index_points(pts, torch.zeros((2, 4), dtype=torch.long)), TypeError)
    calls = stub(ctx, "cg_square_distance_dev")
    _refused(ctx, calls, lambda: square_distance(pts, torch.rand((2, 8, 3))), TypeError)
    _still_works(ctx)


@pytest.mark.gpu
def test_sliced_ids_are_refused(ctx, stub):
    from catgrasp_b200.net import PointNetCls
    from catgrasp_b200.synthetic import make_state_dict
    net = PointNetCls(make_state_dict("cls", 10, seed=0), device=0)
    xyz = torch.rand((64, 3), dtype=torch.float64, device="cuda")
    poses = torch.eye(4, dtype=torch.float64, device="cuda").repeat(3, 1, 1)
    ids = torch.zeros((3, 1024), dtype=torch.int32, device="cuda")
    calls = stub(net.ctx, "cg_graspq_forward_dev")
    _refused(net.ctx, calls, lambda: net.graspq_dev(xyz, xyz, poses, ids[:, :512]), ValueError)
    _refused(net.ctx, calls, lambda: net.graspq_dev(xyz.cpu().numpy(), xyz, poses, ids), TypeError)   # host array
    _still_works(ctx)


@pytest.mark.gpu
def test_inputs_on_another_device_than_the_handle_are_refused(ctx, stub):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from catgrasp_b200.net import PointNetCls
    from catgrasp_b200.synthetic import make_state_dict
    net = PointNetCls(make_state_dict("cls", 10, seed=0), device=0)
    d1 = torch.device("cuda", 1)
    xyz = torch.rand((64, 3), dtype=torch.float64, device=d1)
    poses = torch.eye(4, dtype=torch.float64, device=d1).repeat(3, 1, 1)
    ids = torch.zeros((3, 256), dtype=torch.int32, device=d1)
    calls = stub(net.ctx, "cg_graspq_forward_dev")
    out = (torch.empty((3, 10), device="cuda"), torch.empty((3,), dtype=torch.int32, device="cuda"))
    _refused(net.ctx, calls, lambda: net.graspq_dev(xyz, xyz, poses, ids, out=out), _lib.CgError)
    _still_works(ctx)
