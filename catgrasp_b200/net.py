"""Device-resident PointNetCls / PointNetSeg (pointnet2.py:275-329) behind the C ABI."""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .weights import pack_blob


class _Net:
    kind = None
    kind_id = None

    def __init__(self, state_dict, device=None):
        self.ctx = _lib.Context.get(device)
        blob, n_out = pack_blob(state_dict, self.kind)
        self.n_out = n_out
        expect = self.ctx.call("cg_net_blob_floats", self.kind_id, n_out)
        if expect != blob.size:
            raise _lib.CgError(f"weight blob has {blob.size} floats, library expects {expect}")
        h = C.c_void_p()
        self.ctx.call("cg_net_create", self.ctx.h, self.kind_id, n_out, blob, blob.size, C.byref(h))
        self.h = h
        self.device = torch.device("cuda", self.ctx.device)

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.ctx.call("cg_net_destroy", self.h)
                self.h = None
        except Exception:
            pass

    def _empty(self, *shape, dtype=torch.float32):
        return torch.empty(shape, dtype=dtype, device=self.device)

    def draw_ids_dev(self, M, n_pts, count, seed, first_candidate=0, out=None):
        """Counter-based subset draw on the device (cg_draw_ids_dev): (count, n_pts) int32 cuda tensor (``out`` if
        given)."""
        ids = self._empty(count, n_pts, dtype=torch.int32) if out is None else out
        self.ctx.call("cg_draw_ids_dev", self.ctx.h, int(M), int(n_pts), int(count), int(seed), int(first_candidate), ids)
        return ids

    def draw_ids_many_dev(self, Ms, n_pts, counts, seeds, bases, out=None):
        """cg_draw_ids_dev for several objects in one launch (cg_draw_ids_many_dev): a (sum(counts), n_pts) int32 CUDA
        tensor whose rows of object o are ``draw_ids_dev(Ms[o], n_pts, counts[o], seeds[o]) + bases[o]``."""
        n_obj = len(Ms)
        rows = np.zeros(n_obj + 1, np.int64)
        rows[1:] = np.cumsum(np.asarray(counts, np.int64))
        ids = self._empty(int(rows[-1]), n_pts, dtype=torch.int32) if out is None else out
        if n_obj == 0 or rows[-1] == 0:
            return ids
        _, m, s, r, b = _lib.inputs(np.asarray(Ms, np.int32), np.asarray(seeds, np.uint64).view(np.int64), rows,
                                    np.asarray(bases, np.int32), dtype=(torch.int32, torch.int64, torch.int64,
                                                                        torch.int32), ctx=self.ctx)
        self.ctx.call("cg_draw_ids_many_dev", self.ctx.h, n_obj, m, s, r, b, int(n_pts), int(rows[-1]), ids)
        return ids


class PointNetCls(_Net):
    """forward(x:(B,N,6)) -> logits (B,n_out); mirrors pointnet2.py:289-299 (first return value)."""
    kind, kind_id = "cls", _lib.CG_NET_CLS

    def forward(self, x, return_probs=False):
        _, x = _lib.inputs(x, dtype=torch.float32, ctx=self.ctx)
        B, N, D = x.shape
        assert D == 6
        logits = self._empty(B, self.n_out)
        probs = torch.empty_like(logits) if return_probs else None
        self.ctx.call("cg_cls_forward_dev", self.h, x, B, N, logits, probs)
        return (logits, probs) if return_probs else logits

    __call__ = forward

    def graspq_dev(self, cloud_xyz, cloud_nrm, poses, ids, mean=None, std=None, out=None):
        """Fused transform + forward + softmax on device tensors; returns (probs (B,n_out) f32, label (B,) i32)."""
        M = cloud_xyz.shape[0]
        B = poses.shape[0]
        N = ids.shape[1]
        probs, label = out if out is not None else (self._empty(B, self.n_out), self._empty(B, dtype=torch.int32))
        self.ctx.call("cg_graspq_forward_dev", self.h, cloud_xyz, cloud_nrm, M, poses, B, ids, N, mean, std, probs, label)
        return probs, label

    def graspq_many_dev(self, cloud_xyz, cloud_nrm, poses, ids, groups, mean=None, std=None, out=None):
        """graspq_dev over the candidates of several objects (cg_graspq_forward_many_dev): the clouds concatenated,
        ``ids`` rebased to their rows, ``groups`` the row counts of the graspq_dev launches to reproduce (their FC
        kernels, and so their bits).  Returns (probs (B,n_out) f32, label (B,) i32 or None); ``out`` = (probs, label
        or None)."""
        M, B, N = cloud_xyz.shape[0], poses.shape[0], ids.shape[1]
        groups = np.ascontiguousarray(groups, dtype=np.int32)
        probs, label = out if out is not None else (self._empty(B, self.n_out), self._empty(B, dtype=torch.int32))
        self.ctx.call("cg_graspq_forward_many_dev", self.h, cloud_xyz, cloud_nrm, M, poses, B, ids, N, mean, std,
                      groups, len(groups), probs, label)
        return probs, label

    def graspq_host(self, cloud_xyz, cloud_nrm, poses, ids, mean=None, std=None, out_probs=None, out_label=None):
        """Reference-facing blocking call on HOST buffers (numpy or pinned torch CPU tensors)."""
        M = cloud_xyz.shape[0]
        B = poses.shape[0]
        N = ids.shape[1]
        if out_probs is None:
            out_probs = np.empty((B, self.n_out), dtype=np.float32)
        if out_label is None:
            out_label = np.empty((B,), dtype=np.int32)
        self.ctx.call("cg_graspq_forward_host", self.h, cloud_xyz, cloud_nrm, M, poses, B, ids, N, mean, std, out_probs,
                      out_label)
        return out_probs, out_label


class PointNetSeg(_Net):
    """forward(x:(B,N,6)) -> logits (B,N,n_out); mirrors pointnet2.py:316-329."""
    kind, kind_id = "seg", _lib.CG_NET_SEG

    def forward(self, x):
        _, x = _lib.inputs(x, dtype=torch.float32, ctx=self.ctx)
        B, N, D = x.shape
        assert D == 6
        out = self._empty(B, N, self.n_out)
        self.ctx.call("cg_seg_forward_dev", self.h, x, B, N, out)
        return out

    __call__ = forward

    def nunocs_host(self, x, bins):
        """x (N,6) float32 host -> (coords (N,3) f32, conf_z (N,) f32, bins (N,3) i32); predicter.py:142-150."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        N = x.shape[0]
        coords = np.empty((N, 3), np.float32)
        conf = np.empty((N,), np.float32)
        b = np.empty((N, 3), np.int32)
        self.ctx.call("cg_nunocs_forward_host", self.h, x, N, int(bins), coords, conf, b)
        return coords, conf, b

    def nunocs_dev(self, x, bins):
        _, x = _lib.inputs(x, dtype=torch.float32, ctx=self.ctx)
        N = x.shape[0]
        coords = self._empty(N, 3)
        conf = self._empty(N)
        b = self._empty(N, 3, dtype=torch.int32)
        self.ctx.call("cg_nunocs_forward_dev", self.h, x, N, int(bins), coords, conf, b)
        return coords, conf, b

    def nunocs_many_host(self, x, bins):
        """x (B,N,6) float32 host -> (coords (B,N,3) f32, conf_z (B,N) f32, bins (B,N,3) i32): nunocs_host on each
        x[b], bit for bit, in one batched forward (cg_nunocs_forward_many_host)."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        B, N, _ = x.shape
        coords = np.empty((B, N, 3), np.float32)
        conf = np.empty((B, N), np.float32)
        b = np.empty((B, N, 3), np.int32)
        self.ctx.call("cg_nunocs_forward_many_host", self.h, x, B, N, int(bins), coords, conf, b)
        return coords, conf, b

    def nunocs_many_dev(self, x, bins):
        """nunocs_many_host on the device: CUDA tensors in and out, no synchronisation."""
        _, x = _lib.inputs(x, dtype=torch.float32, ctx=self.ctx)
        B, N, _ = x.shape
        coords = self._empty(B, N, 3)
        conf = self._empty(B, N)
        b = self._empty(B, N, 3, dtype=torch.int32)
        self.ctx.call("cg_nunocs_forward_many_dev", self.h, x, B, N, int(bins), coords, conf, b)
        return coords, conf, b
