"""Clustering of the segmentation's shifted points on the device (csrc/cg_meanshift.cu): sklearn's MeanShift as
PointGroupPredictor.predict uses it (predicter.py:332), and the label propagation around it (:308-338).

Numpy in, numpy out; CUDA tensor in, CUDA tensor out (see _lib).  Centres keep X's dtype (float32 or float64); labels
are int64.  Labels are the nearest kept centre in float64 d2, ties to the smaller centre index.  Centres are summed in
int64 fixed point, so they do not depend on the order of X's rows; sklearn's own centres move by a few float32 ulps
when the rows are permuted, its labels do not.
"""
import numbers

import numpy as np
import torch

from . import _lib
from .cloud import CloudIndex, _query_cell

MEANSHIFT_BANDWIDTH = {"hnm": 0.005, "nut": 0.007, "screw": 0.009}   # predicter.py:317-330
DOWNSAMPLE = 0.002                                                     # predicter.py:309
LABEL_REACH = 4.0      # first nearest-centre query bound, in bandwidths; points beyond it are queried again unbounded


def _as_points(X):
    """X as an (N,3) float32 / float64 numpy array or tensor (other dtypes widened to float64, as sklearn does);
    ValueError for a wrong shape, no rows or a non-finite value."""
    if isinstance(X, torch.Tensor):
        if X.dtype not in (torch.float32, torch.float64):
            X = X.to(torch.float64)
        finite = lambda a: bool(torch.isfinite(a).all())      # noqa: E731
    else:
        X = np.asarray(X)
        if X.dtype not in (np.float32, np.float64):
            X = X.astype(np.float64)
        finite = lambda a: bool(np.isfinite(a).all())         # noqa: E731
    if X.ndim != 2 or X.shape[1] != 3:
        raise ValueError(f"Expected a 2D array of shape (n_samples, 3), got shape {tuple(X.shape)}")
    if X.shape[0] == 0:
        raise ValueError("Found array with 0 sample(s) (shape=(0, 3)) while a minimum of 1 is required")
    if not finite(X):
        raise ValueError("Input X contains NaN or infinity")
    return X


def _nearest_many(ref, ref_off, query, query_off, reach):
    """Index of the nearest ref point for every query, per set (ref, query: float64 device tensors, set s the rows
    [off[s], off[s + 1]) of each, every ref set non-empty): the index into ref of each query's nearest point of its own
    set, ties to the smaller index.  First within `reach`, then, for the queries with nothing that close, within the
    diagonal of the box around every set's points and those queries, which covers each set's own, so none goes
    unanswered.  One index build for the whole batch, and at most one more, shared by every set, for those queries."""
    _, idx = CloudIndex(ref, _query_cell(ref, reach), ref.device.index, set_offsets=ref_off).nearest_many(
        query, query_off, reach)
    miss = torch.nonzero(idx < 0).reshape(-1)
    if miss.numel():
        q = query[miss]
        miss_off = np.searchsorted(miss.cpu().numpy(), np.asarray(query_off), side="left")
        span = torch.maximum(ref.amax(0), q.amax(0)) - torch.minimum(ref.amin(0), q.amin(0))
        bound = float(torch.linalg.norm(span)) * (1 + 1e-9)
        _, far = CloudIndex(ref, _query_cell(ref, bound), ref.device.index, set_offsets=ref_off).nearest_many(
            q, miss_off, bound)
        if bool((far < 0).any()):
            raise _lib.CgError("nearest: a query found no point within the joint bounding box's diagonal")
        idx[miss] = far
    return idx.to(torch.int64)


def _set_ids(off, device):
    """(N,) int64 device tensor: the set of each row, for offsets off (S + 1 host ints)."""
    off = np.asarray(off, dtype=np.int64)
    return torch.repeat_interleave(torch.arange(len(off) - 1, device=device),
                                   torch.from_numpy(np.diff(off)).to(device))


def _fit_many(x, off, bw, max_iter):
    """MeanShift per set on the device: x (N,3) float32 / float64 CUDA, set s the rows [off[s], off[s + 1]).  Returns
    (centres set-major, centre offsets (S + 1) numpy, labels (N,) int64 per set, n_iter (S,) numpy, seed centres,
    seed counts (N,) int64, seed iterations (N,) int64).  Synchronises once after the clustering, once more in the
    labelling (twice when a point has no centre within LABEL_REACH bandwidths)."""
    ctx = _lib.Context.get(x.device.index)
    f64 = x.dtype == torch.float64
    off = np.asarray(off, dtype=np.int64)
    S = len(off) - 1
    index = CloudIndex(x, bw, x.device.index, set_offsets=off)
    P = x.shape[0]
    seed_c = torch.empty_like(x)
    seed_n = torch.empty((P,), dtype=torch.int32, device=x.device)
    seed_it = torch.empty_like(seed_n)
    cen = torch.empty_like(x)
    coff = torch.empty((S + 1,), dtype=torch.int32, device=x.device)
    ctx.call("cg_meanshift_many_dev", index.h, x, int(f64), float(bw), int(max_iter), seed_c, seed_n, seed_it, cen,
             coff)
    n_iter = torch.stack([seed_it[a:b].amax() for a, b in zip(off[:-1].tolist(), off[1:].tolist())])
    host = torch.cat([coff, n_iter]).cpu().numpy().astype(np.int64)                  # one synchronisation
    coff_h, n_iter = host[:S + 1], host[S + 1:]
    if (np.diff(coff_h) < 1).any():
        raise ValueError("CloudIndex needs at least one point")                        # as fit: a set with no centre
    centres = cen[:int(coff_h[-1])].contiguous()
    labels = _nearest_many(centres.to(torch.float64), coff_h, x.to(torch.float64), off, LABEL_REACH * bw)
    labels = labels - torch.from_numpy(coff_h[:-1]).to(x.device)[_set_ids(off, x.device)]
    return centres, coff_h, labels, n_iter, seed_c, seed_n.to(torch.int64), seed_it.to(torch.int64)


class MeanShift:
    """sklearn.cluster.MeanShift for the arguments the reference passes: every point seeds an ascent (seeds=None,
    bin_seeding=False) and every point is labelled (cluster_all=True).  n_jobs is accepted and ignored.

    fit(X) sets cluster_centers_ (K,3) in X's dtype, labels_ (N,) int64 and n_iter_, and also the per-seed results
    seed_centers_ (N,3), seed_counts_ (N,) (points within bandwidth of the final centre, 0 when none) and
    seed_iters_ (N,); it is fit_many with one set.  X holds at most 2^21 points."""

    def __init__(self, bandwidth=None, cluster_all=True, n_jobs=None, seeds=None, bin_seeding=False, max_iter=300):
        self.bandwidth = bandwidth
        self.cluster_all = cluster_all
        self.n_jobs = n_jobs
        self.seeds = seeds
        self.bin_seeding = bin_seeding
        self.max_iter = max_iter

    def _check_params(self):
        if self.bandwidth is None:
            raise NotImplementedError("MeanShift: bandwidth=None (estimate_bandwidth) is not supported")
        if self.seeds is not None:
            raise NotImplementedError("MeanShift: explicit seeds are not supported")
        if self.bin_seeding:
            raise NotImplementedError("MeanShift: bin_seeding=True is not supported")
        if not self.cluster_all:
            raise NotImplementedError("MeanShift: cluster_all=False is not supported")
        bw = self.bandwidth
        if isinstance(bw, bool) or not isinstance(bw, numbers.Real) or not (np.isfinite(bw) and bw > 0):
            raise ValueError(f"MeanShift: bandwidth must be a positive finite number, got {bw!r}")
        it = self.max_iter
        if isinstance(it, bool) or not isinstance(it, numbers.Integral) or not 0 <= it < 2 ** 31:
            raise ValueError(f"MeanShift: max_iter must be an integer >= 0, got {it!r}")

    def fit(self, X, y=None):
        vars(self).update(vars(self.fit_many([X])[0]))
        return self

    def fit_predict(self, X, y=None):
        return self.fit(X).labels_

    def fit_many(self, Xs):
        """fit for several point sets in one pass: a list of fitted MeanShift instances, the s-th as fit leaves it
        for Xs[s] alone, bit for bit.  The sets are numpy arrays or CUDA tensors (not mixed) of one dtype, each of at
        most 2^21 points; each set's results come back in its own kind and dtype."""
        self._check_params()
        Xs = [_as_points(X) for X in list(Xs)]
        if not Xs:
            raise ValueError("MeanShift.fit_many: no point sets")
        kinds = {getattr(X, "is_cuda", False) for X in Xs}
        dtypes = {str(X.dtype).split(".")[-1] for X in Xs}
        if len(kinds) > 1 or len(dtypes) > 1:
            raise ValueError(f"MeanShift.fit_many: the sets must share one kind and dtype, got {sorted(dtypes)}")
        f64 = dtypes == {"float64"}
        ctx, *xs = _lib.inputs(*Xs, dtype=torch.float64 if f64 else torch.float32)
        off = np.cumsum([0] + [len(x) for x in xs])
        centres, coff, labels, n_iter, seed_c, seed_n, seed_it = _fit_many(torch.cat(xs), off, float(self.bandwidth),
                                                                           self.max_iter)
        out = []
        for s, X in enumerate(Xs):
            a, b, c, d = off[s], off[s + 1], coff[s], coff[s + 1]
            m = MeanShift(bandwidth=self.bandwidth, cluster_all=self.cluster_all, n_jobs=self.n_jobs,
                          seeds=self.seeds, bin_seeding=self.bin_seeding, max_iter=self.max_iter)
            m.n_iter_ = int(n_iter[s])
            (m.cluster_centers_, m.labels_, m.seed_centers_, m.seed_counts_, m.seed_iters_) = _lib.returned(
                X, centres[c:d].contiguous(), labels[a:b].contiguous(), seed_c[a:b].contiguous(),
                seed_n[a:b].contiguous(), seed_it[a:b].contiguous())
            out.append(m)
        return out


def pointgroup_labels(xyz_original_all, pt_offsets, cloud_xyz, bandwidth):
    """predicter.py:308-338 after the network: the 2 mm voxel down-sampling of the network's points, each voxel mean
    snapped to its nearest point, those points moved by their offsets (float32), clustered by MeanShift, and every
    point of cloud_xyz labelled with its nearest snapped point's cluster.  Returns (labels_all (M,) int64,
    xyz_shifted (U,3) float32): pointgroup_labels_many with one frame."""
    return pointgroup_labels_many([xyz_original_all], [pt_offsets], [cloud_xyz], bandwidth)[0]


def _pointgroup_labels_cat(xo, off, xo_off, cloud, cloud_off, bandwidth):
    """pointgroup_labels over several frames laid end to end, on the device: xo / off (N,3) float32 with frame b at
    rows [xo_off[b], xo_off[b + 1]), cloud (M,3) float64 with frame b at [cloud_off[b], cloud_off[b + 1]).  Returns
    (labels_all (M,) int64, xyz_shifted (U,3) float32, its frame offsets (B + 1) numpy).  One 2 mm index, one snap
    index and one snap check for all frames."""
    ds = CloudIndex(xo, DOWNSAMPLE, xo.device.index, set_offsets=xo_off)                  # :308-310
    down, _ = ds.voxel_means()
    down_off = ds.cell_offsets
    del ds
    # :311-313 snap: a voxel mean and its members share a voxel, so the nearest member is within the diagonal; the
    # bound is widened by 1e-9 relative so rounding at a voxel face cannot exclude it
    snap = DOWNSAMPLE * np.sqrt(3.0) * (1 + 1e-9)
    _, ids = CloudIndex(xo, snap, xo.device.index, set_offsets=xo_off).nearest_many(down, down_off, snap)
    if bool((ids < 0).any()):
        raise _lib.CgError("pointgroup_labels: a voxel mean has no point within its voxel's diagonal")
    ids = ids.to(torch.int64)
    xyz_down = xo[ids]
    xyz_shifted = xyz_down + off[ids]                                                    # :314, float32
    if not bool(torch.isfinite(xyz_shifted).all() & torch.isfinite(cloud).all()):        # as _as_points, at once
        raise ValueError("Input X contains NaN or infinity")
    ms = MeanShift(bandwidth=bandwidth)
    ms._check_params()
    labels = _fit_many(xyz_shifted, down_off, float(ms.bandwidth), ms.max_iter)[2]            # :332
    nearest = _nearest_many(xyz_down.to(torch.float64), down_off, cloud, cloud_off, LABEL_REACH * DOWNSAMPLE)
    return labels[nearest], xyz_shifted, down_off                                         # :334-336


def pointgroup_labels_many(xyz_original_alls, pt_offsetss, cloud_xyzs, bandwidth):
    """pointgroup_labels for several frames in one pass: a list of (labels_all, xyz_shifted), the b-th as
    pointgroup_labels gives it for frame b alone, bit for bit.  The arrays are numpy arrays or CUDA tensors; frame b's
    results are CUDA tensors where xyz_original_alls[b] is one, else numpy.  The number of index builds and
    synchronisations does not grow with the number of frames."""
    xos, offs, clouds = list(xyz_original_alls), list(pt_offsetss), list(cloud_xyzs)
    if not xos or len(offs) != len(xos) or len(clouds) != len(xos):
        raise ValueError("pointgroup_labels_many: need one offsets array and one cloud per frame, and a frame")
    xos, offs, clouds = [_as_points(a) for a in xos], [_as_points(a) for a in offs], [_as_points(a) for a in clouds]
    for b, (xo, off) in enumerate(zip(xos, offs)):
        if off.shape[0] != xo.shape[0]:
            raise ValueError(f"pointgroup_labels_many: frame {b}'s pt_offsets must have one row per point")
    ctx, *t = _lib.inputs(*xos, *offs, *clouds, dtype=(torch.float32,) * (2 * len(xos)) + (torch.float64,) * len(xos))
    B = len(xos)
    xo_off = np.cumsum([0] + [len(a) for a in xos])
    cloud_off = np.cumsum([0] + [len(a) for a in clouds])
    labels, shifted, sh_off = _pointgroup_labels_cat(torch.cat(t[:B]), torch.cat(t[B:2 * B]), xo_off,
                                                     torch.cat(t[2 * B:]), cloud_off, bandwidth)
    return [_lib.returned(xos[b], labels[cloud_off[b]:cloud_off[b + 1]].contiguous(),
                          shifted[sh_off[b]:sh_off[b + 1]].contiguous()) for b in range(B)]
