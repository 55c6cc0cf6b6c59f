"""Exact rational statement of the scan occupancy rule -- ORACLE, test infrastructure only.

oracle/occupancy_ref.c and csrc/cg_occupancy.cu share one float64 arithmetic and one control flow, so a mistake common
to both (the ``+ 2r`` early exit, the handling of negative steps, a tie broken towards the wrong axis) would pass every
comparison between them.  This module restates the rule of my_cpp/common.cpp:324-431 without that arithmetic:

* inputs, in the reference's float32 arithmetic: the sample grid (geometry of common.cpp:352-377, samples
  ``origin + float(i) * res``) and each sample's float32 norm ``dq = sqrtf((x*x + y*y) + z*z)``;
* occupied cells: ``floor(p / res)`` of the scan points, in exact rationals;
* the walk: cell (0,0,0) is tested first; then a DDA along the ray from the origin through the exact sample
  coordinates (not the float-normalised direction).  The next boundary on axis a is crossed at
  ``t_a = (k_a + [step_a > 0]) * res / s_a`` (t = 1 at the sample), and the smallest t_a is found by exact
  cross-multiplication.  The kernel's early exit (``tmax > dq + 2 res``) is not used.  The walk stops only where no
  later cell can be reported: when it has left the occupied cells' bounding box for good (steps are monotone), or when
  the next cell is entered farther than ``dq + 0.87 res`` from the origin.  A cell centre is within sqrt(3)/2 res
  (0.8660 res) of every point of its cell, so every later centre is then farther than dq; 0.87 > sqrt(3)/2 is the
  whole argument.  This one test is made in float64, where the margin of 0.0039 res dwarfs the rounding;
* the verdict: the first occupied cell's centre c is reported when ``|c|^2 <= dq^2``, exactly.

A sample is *undecided* when the kernel's arithmetic may legitimately order things differently from the exact rule:
two crossing parameters within a relative TIE_REL of each other (the kernel's direction is the float32-normalised
sample, so it can order near-ties either way) with an occupied cell among the ones either order would visit, or a
final comparison within a relative CMP_REL.  Ties whose alternative cells are all free cannot change the verdict and
leave the sample decided.

Pure Python: keep grids small (a few thousand samples, rays of tens of cells), or pass a subset of samples.
"""
from fractions import Fraction
from itertools import combinations

import numpy as np

TIE_REL = 1e-6
CMP_REL = 1e-9
PAD = np.float32(0.005)


def geometry(pts, res):
    """(dims (3,) int, origin (3,) float32, res float32): common.cpp:352-366, :375-377 in float32."""
    p = np.ascontiguousarray(np.asarray(pts, np.float64).astype(np.float32)).reshape(-1, 3)
    r = np.float32(res)
    mn, mx = p.min(0), p.max(0)
    dims = (((mx + PAD) - (mn - PAD)) / r).astype(np.int64)
    return dims, (mn - PAD).astype(np.float32), r


def samples_of(origin, r, idx3):
    """(S,3) float32 sample coordinates of grid indices idx3 (S,3), and their float32 norms."""
    s = (origin[None, :] + idx3.astype(np.float32) * r).astype(np.float32)
    q = (s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]) + s[:, 2] * s[:, 2]
    return s, np.sqrt(q.astype(np.float32)).astype(np.float32)


def _floor_div(x, r):
    q = x / r
    return q.numerator // q.denominator


def occupancy_exact(pts, res, samples=None):
    """Flags, decided and tied (bool) for the samples with raster indices ``samples`` (all samples by default, in
    (xi, yi, zi) raster order).  ``tied`` marks samples whose walk met an exact tie between crossing parameters."""
    p = np.asarray(pts, np.float64).astype(np.float32).reshape(-1, 3)
    dims, origin, r32 = geometry(p, res)
    nx, ny, nz = (int(d) for d in dims)
    if samples is None:
        samples = np.arange(nx * ny * nz)
    samples = np.asarray(samples, np.int64)
    idx3 = np.stack([samples // (ny * nz), (samples // nz) % ny, samples % nz], 1)
    s32, dq32 = samples_of(origin, r32, idx3)
    r = Fraction(float(r32))
    occ = {tuple(_floor_div(Fraction(float(v)), r) for v in row) for row in p}
    kmin = [min(c[a] for c in occ) for a in range(3)]
    kmax = [max(c[a] for c in occ) for a in range(3)]
    flags = np.zeros(len(samples), np.uint8)
    decided = np.ones(len(samples), bool)
    tied = np.zeros(len(samples), bool)
    for i in range(len(samples)):
        f, d, t = _walk(s32[i], dq32[i], r, float(r32), occ, kmin, kmax)
        flags[i], decided[i], tied[i] = f, d, t
    return flags, decided, tied


def _walk(s32, dq32, r, rf, occ, kmin, kmax):
    """(flag, decided, tied) of one sample."""
    if not dq32 > 0:
        return 0, True, False                                # a sample at the origin is never reported
    sf = [Fraction(float(v)) for v in s32]
    den = max(v.denominator for v in sf)                     # powers of two: the largest is a common multiple
    S = [v.numerator * (den // v.denominator) for v in sf]  # integer sample, up to the common scale
    step = [(v > 0) - (v < 0) for v in S]
    snorm = float(np.linalg.norm(np.asarray(s32, np.float64)))
    reach = float(dq32) + 0.87 * rf
    k = [0, 0, 0]
    tied = False
    hit = (0, 0, 0) in occ
    while not hit:
        if any((k[a] < kmin[a] and step[a] <= 0) or (k[a] > kmax[a] and step[a] >= 0) for a in range(3)):
            return 0, True, tied                             # left the occupied cells' bounding box for good
        moving = [a for a in range(3) if step[a]]
        num = {a: abs(k[a] + (1 if step[a] > 0 else 0)) for a in moving}    # t_a = num[a] * r / |S_a| (scaled)
        m = moving[0]
        for a in moving[1:]:
            if num[a] * abs(S[m]) < num[m] * abs(S[a]):
                m = a
        if num[m] * rf / abs(float(sf[m])) * snorm > reach:
            return 0, True, tied                             # every later cell centre is farther than the sample
        tm = num[m] / abs(S[m])
        group = [a for a in moving if num[a] * abs(S[m]) == num[m] * abs(S[a])]
        tied |= len(group) > 1
        group += [a for a in moving if a not in group and num[a] / abs(S[a]) <= tm * (1 + TIE_REL)]
        if len(group) > 1:
            # either order passes through the cells k + (a proper subset of the group's steps); free cells cannot
            # change the verdict, an occupied one can
            for n in range(1, len(group)):
                for sub in combinations(group, n):
                    c = list(k)
                    for a in sub:
                        c[a] += step[a]
                    if tuple(c) in occ:
                        return 0, False, tied
        for a in group:
            k[a] += step[a]
        hit = tuple(k) in occ
    c2 = sum(((ka + Fraction(1, 2)) * r) ** 2 for ka in k)
    d2 = Fraction(float(dq32)) ** 2
    if abs(c2 - d2) <= CMP_REL * d2:
        return int(c2 <= d2), False, tied
    return int(c2 <= d2), True, tied
