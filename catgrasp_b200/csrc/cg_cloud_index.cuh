// cg_cloud_index.cuh -- the uniform-grid point index of cg_cloud.cu and the device helpers that query it, shared by
// every source that searches a cloud (cg_cloud.cu, cg_meanshift.cu, cg_ransac.cu).  See cg_cloud.cu for the index's layout.
#pragma once
#include <cmath>
#include <vector>
#include "cg_common.cuh"

// one set of a many-set index: its origin, its largest occupied cell per axis
struct CloudSet {
  double o[3];
  int64_t mc[3];
};

struct cg_cloud_index {
  cg_ctx *ctx = nullptr;
  int P = 0, U = 0;            // points, occupied cells
  double cell = 0.0;
  double origin[3] = {0, 0, 0};
  double hi[3] = {0, 0, 0};    // max_bound of the points
  int bits = 1;                // bits per axis in a key
  int64_t maxc[3] = {0, 0, 0}; // largest occupied cell coordinate per axis
  double *spts = nullptr;      // (P,3) points in key order
  int32_t *perm = nullptr;     // (P) original index of each sorted point
  uint64_t *ukey = nullptr;    // (U) ascending unique keys
  int32_t *start = nullptr;    // (U+1) first sorted point of each cell; start[U] = P
  // the sets (cg_cloud_index_create_many; one set otherwise): set s holds points [poff[s], poff[s+1]) in the caller's
  // order and in key order, and cells [coff[s], coff[s+1]); its keys carry the prefix s << 3 bits.  origin, hi and
  // maxc above are set 0's.  The device copies exist only when S > 1.
  int S = 1;
  std::vector<int32_t> poff, coff;          // host, S+1 each
  std::vector<double> set_hi;               // host, (S,3): each set's max_bound
  std::vector<CloudSet> sets;               // host, S
  const CloudSet *d_sets = nullptr;         // device (S), inside the spts allocation
  const int32_t *d_poff = nullptr;          // device (S+1), inside the spts allocation
};

namespace {

constexpr int MAX_AXIS_BITS = 21;
constexpr double RANGE_SLACK = 1e-6;   // cells

struct IndexView {
  const double *spts;
  const int32_t *perm;
  const uint64_t *ukey;
  const int32_t *start;
  int U, bits;
  double cell, ox, oy, oz;
  int64_t mx, my, mz;
  uint64_t prefix;         // the set field of every key this view searches (0 for a one-set index)
  const CloudSet *sets;    // a many-set index's table (S > 1), else null
  const int32_t *poff;     // (S+1) its point offsets, else null
  int S;

  // the view of set s alone: its origin, its cell range and its key prefix, so a query sees only set s's cells
  __device__ __forceinline__ IndexView in_set(int s) const {
    IndexView v = *this;
    const CloudSet &r = sets[s];
    v.ox = r.o[0]; v.oy = r.o[1]; v.oz = r.o[2];
    v.mx = r.mc[0]; v.my = r.mc[1]; v.mz = r.mc[2];
    v.prefix = (uint64_t)s << (3 * bits);
    return v;
  }
};

inline IndexView view_of(const cg_cloud_index *ix) {
  return IndexView{ix->spts, ix->perm, ix->ukey, ix->start, ix->U, ix->bits, ix->cell, ix->origin[0], ix->origin[1],
                   ix->origin[2], ix->maxc[0], ix->maxc[1], ix->maxc[2], 0ull, ix->d_sets, ix->d_poff, ix->S};
}

// the s with off[s] <= i < off[s + 1] (off ascending, every range non-empty, 0 <= i < off[S])
__device__ __forceinline__ int set_of(const int32_t *off, int S, int i) {
  int lo = 0, hi = S;
  while (hi - lo > 1) {
    const int m = (lo + hi) >> 1;
    if (off[m] <= i) lo = m; else hi = m;
  }
  return lo;
}

__device__ __forceinline__ double dist2(double ax, double ay, double az, double bx, double by, double bz) {
  const double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by), dz = __dsub_rn(az, bz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__device__ __forceinline__ uint64_t pack(int64_t x, int64_t y, int64_t z, int b) {
  return ((uint64_t)x << (2 * b)) | ((uint64_t)y << b) | (uint64_t)z;
}

// a point's cell key: floor((p - origin) / cell) per axis, each operation rounded on its own, packed x major.  The
// caller guarantees every coordinate lies in [0, 2^bits).
__device__ __forceinline__ uint64_t cell_key(double px, double py, double pz, double ox, double oy, double oz, double cell,
                                             int bits) {
  const int64_t x = (int64_t)floor(__ddiv_rn(__dsub_rn(px, ox), cell));
  const int64_t y = (int64_t)floor(__ddiv_rn(__dsub_rn(py, oy), cell));
  const int64_t z = (int64_t)floor(__ddiv_rn(__dsub_rn(pz, oz), cell));
  return pack(x, y, z, bits);
}

// cells [lo, hi] on one axis that can hold a point within R of q; false when none of them is occupied
__device__ __forceinline__ bool axis_range(double q, double o, double R, double cell, int64_t maxc, int64_t &lo, int64_t &hi) {
  const double d = __dsub_rn(q, o);
  const double flo = floor(__ddiv_rn(__dsub_rn(d, R), cell) - RANGE_SLACK);
  const double fhi = floor(__ddiv_rn(__dadd_rn(d, R), cell) + RANGE_SLACK);
  if (!(flo <= (double)maxc) || !(fhi >= 0.0)) return false;   // also false for NaN
  lo = flo < 0.0 ? 0 : (int64_t)flo;
  hi = fhi > (double)maxc ? maxc : (int64_t)fhi;
  return true;
}

__device__ __forceinline__ int lower_bound(const uint64_t *a, int lo, int hi, uint64_t k) {
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (a[m] < k) lo = m + 1; else hi = m;
  }
  return lo;
}

__device__ __forceinline__ int upper_bound(const uint64_t *a, int lo, int hi, uint64_t k) {
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (a[m] <= k) lo = m + 1; else hi = m;
  }
  return lo;
}

// The cell range of a query: per (x, y) column, the contiguous run [s, e) of sorted points in cells z_lo..z_hi.  The
// range is clamped to the view's largest cells, below 2^bits, so a column's keys never carry into the next set's.
struct Columns {
  int64_t x0, x1, y0, y1, z0, z1;
  bool any;
  __device__ __forceinline__ Columns(const IndexView &V, double qx, double qy, double qz, double R) {
    any = axis_range(qx, V.ox, R, V.cell, V.mx, x0, x1) && axis_range(qy, V.oy, R, V.cell, V.my, y0, y1) &&
          axis_range(qz, V.oz, R, V.cell, V.mz, z0, z1);
  }
  // as above, with the origin and cell range of `r` when it is not null (a set's row the caller keeps in shared memory,
  // read axis by axis where it is used, so a long-lived query holds no registers for it)
  __device__ __forceinline__ Columns(const IndexView &V, const volatile CloudSet *r, double qx, double qy, double qz,
                                     double R) {
    any = axis_range(qx, r ? r->o[0] : V.ox, R, V.cell, r ? r->mc[0] : V.mx, x0, x1) &&
          axis_range(qy, r ? r->o[1] : V.oy, R, V.cell, r ? r->mc[1] : V.my, y0, y1) &&
          axis_range(qz, r ? r->o[2] : V.oz, R, V.cell, r ? r->mc[2] : V.mz, z0, z1);
  }
  // the occupied cells [a, b) of column (cx, cy), as positions in the cell table
  __device__ __forceinline__ void cells(const IndexView &V, int64_t cx, int64_t cy, int &a, int &b) const {
    a = lower_bound(V.ukey, 0, V.U, V.prefix | pack(cx, cy, z0, V.bits));
    b = upper_bound(V.ukey, a, V.U, V.prefix | pack(cx, cy, z1, V.bits));
  }
  __device__ __forceinline__ void run(const IndexView &V, int64_t cx, int64_t cy, int &s, int &e) const {
    int a, b;
    cells(V, cx, cy, a, b);
    s = V.start[a];
    e = V.start[b];
  }
};

}  // namespace
