"""Sdf3D container and ``.sdf`` reader (meshpy/meshpy/sdf.py:217-289, sdf_file.py:59-87)."""
import ctypes as C

import numpy as np
import torch

from . import _lib


class Sdf3D:
    """A signed-distance grid resident in HBM.

    data[i][j][k] (float32), origin (3,), resolution: the grid coordinate of a
    point x in the SDF frame is (x - origin) / resolution (sdf.py:252-264).
    """

    def __init__(self, sdf_data, origin, resolution, device=None, ctx=None):
        self.data_ = np.ascontiguousarray(sdf_data, dtype=np.float32)
        assert self.data_.ndim == 3
        self.origin_ = np.ascontiguousarray(origin, dtype=np.float32).reshape(3)
        self.resolution_ = float(np.float32(resolution))
        self.dims_ = np.array(self.data_.shape)
        # ``ctx``: a library context of its own (= its own stream and workspace) lets the collision filter run
        # concurrently with the networks of the per-device default context (bench.py does this)
        self.ctx = ctx if ctx is not None else _lib.Context.get(device)
        h = C.c_void_p()
        self.ctx.call("cg_sdf_create", self.ctx.h, self.data_, *self.data_.shape, self.origin_, self.resolution_,
                      C.byref(h))
        self.h = h

    @classmethod
    def from_mesh(cls, vertices, faces, resolution=0.001, padding=5, device=None, ctx=None):
        """Signed-distance grid of a closed triangle mesh, built on the GPU (replaces make_sdf.py:30-36 / SDFGen).

        vertices (N,3), faces (M,3); ``resolution`` is the cell size and ``padding`` the number of cells added on
        every side of the mesh's bounding box (make_sdf.py's defaults: 1 mm, 5 cells).  Values are exact distances to
        the nearest triangle, negative inside.  ``write_sdf_file(path, s.data_, s.origin_, s.resolution_)`` stores the
        result as a ``.sdf`` file.  Raises CgError for an open mesh or invalid input."""
        V = np.ascontiguousarray(vertices, dtype=np.float64)
        F = np.asarray(faces)
        if V.ndim != 2 or V.shape[1] != 3 or F.ndim != 2 or F.shape[1] != 3:
            raise ValueError(f"from_mesh: vertices and faces must be (N,3), got {V.shape} and {F.shape}")
        if F.size and (F.min() < np.iinfo(np.int32).min or F.max() > np.iinfo(np.int32).max):
            raise ValueError("from_mesh: face index out of the int32 range")
        F = np.ascontiguousarray(F, dtype=np.int32)
        self = cls.__new__(cls)
        self.ctx = ctx if ctx is not None else _lib.Context.get(device)
        self.h = None
        h = C.c_void_p()
        self.ctx.call("cg_sdf_from_mesh", self.ctx.h, V, V.shape[0], F, F.shape[0], float(resolution), int(padding),
                      C.byref(h))
        self.h = h
        dims = np.empty(3, np.int32)
        self.origin_ = np.empty(3, np.float32)
        res = C.c_float()
        self.ctx.call("cg_sdf_geometry", self.h, dims, self.origin_, C.byref(res))
        self.data_ = np.empty(tuple(dims), np.float32)
        self.ctx.call("cg_sdf_download", self.h, self.data_)
        self.resolution_ = float(res.value)
        self.dims_ = np.array(self.data_.shape)
        return self

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.ctx.call("cg_sdf_destroy", self.h)
                self.h = None
        except Exception:
            pass

    def _lookup(self, coords, mode):
        _, c = _lib.inputs(coords, dtype=torch.float32, ctx=self.ctx)
        c = c.reshape(3, -1).t().contiguous()          # reference passes (3,N)
        P = c.shape[0]
        out = torch.empty((P,), dtype=torch.float32, device=c.device)
        self.ctx.call("cg_sdf_lookup_dev", self.h, c, P, mode, out)
        return out

    def _signed_distance(self, coords, fast=False):
        """sdf.py:292-343: coords (3,N) in GRID units -> (N,) trilinear (or nearest when fast)."""
        return self._lookup(coords, _lib.CG_SDF_NEAREST if fast else _lib.CG_SDF_TRILINEAR)

    def transform_pt_obj_to_grid(self, x_sdf):
        """sdf.py:252-264 for (N,3) points."""
        return (np.asarray(x_sdf, dtype=np.float32) - self.origin_[None]) / np.float32(self.resolution_)


def parse_sdf_file(path):
    """sdf_file.py:59-87: header ``nx ny nz`` / ``ox oy oz`` / ``res`` then values, i fastest, k slowest.
    Host-only: returns (data[i][j][k] float64, origin (3,), resolution)."""
    with open(path, "r") as f:
        nx, ny, nz = [int(v) for v in f.readline().split()]
        origin = np.array([float(v) for v in f.readline().split()])
        res = float(f.readline())
        vals = np.loadtxt(f, dtype=np.float64).reshape(-1)
    assert vals.size == nx * ny * nz, "truncated .sdf file"
    data = vals.reshape(nz, ny, nx).transpose(2, 1, 0)   # file order: k slowest, i fastest -> data[i][j][k]
    return np.ascontiguousarray(data), origin, res


def read_sdf_file(path, device=None):
    """SdfFile(path).read() (sdf_file.py:41-87) -> device-resident Sdf3D."""
    data, origin, res = parse_sdf_file(path)
    return Sdf3D(data, origin, res, device=device)


def write_sdf_file(path, data, origin, res):
    """Inverse of read_sdf_file (the layout SDFGen emits, make_sdf.py:30-34)."""
    data = np.asarray(data)
    nx, ny, nz = data.shape
    with open(path, "w") as f:
        f.write(f"{nx} {ny} {nz}\n")
        f.write(" ".join(repr(float(v)) for v in origin) + "\n")
        f.write(repr(float(res)) + "\n")
        np.savetxt(f, data.transpose(2, 1, 0).reshape(-1), fmt="%.9g")
