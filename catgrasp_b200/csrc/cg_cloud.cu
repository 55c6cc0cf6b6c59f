// cg_cloud.cu -- point-cloud preparation on the device: the open3d / scipy steps between the camera and the ported
// stages (run_grasp_simulation.py:97, :113-139, :171-175, :198-211, :245-251).
//
// Every query runs against one structure, cg_cloud_index: the points binned into a uniform grid of cells of size `cell`
// with origin min_bound - cell/2 (open3d VoxelDownSample's origin).  A point's cell is floor((p - origin) / cell) per
// axis in float64, in that order; the three cell coordinates are packed into one 64-bit key (x major, z minor) and the
// points are radix-sorted by (key, index), so a cell's members are contiguous and in ascending point index.  The unique
// keys, ascending, with each cell's first sorted point, form the cell table; a query binary-searches it once per (x, y)
// column of its cell range, because the cells of a column are consecutive keys and their points one contiguous run.
// Nothing depends on atomic arrival order: the results are a function of the inputs alone.  The index structure and
// its query helpers are in cg_cloud_index.cuh, shared with cg_meanshift.cu.
//
// A many-set index (cg_cloud_index_create_many) holds S point sets laid end to end, each with what a one-set index
// over it alone has: its own bounds, so its own origin (its min_bound - cell/2), its own largest cells and the 2^21
// cell limit per axis.  Every set shares `cell`.  A key is s << 3b | x << 2b | y << b | z: b is the smallest width that
// holds every set's largest cell, and the set field takes bit_length(S - 1) bits; a batch whose key needs more than
// 63 bits is refused.  So the sorted points, the cell table and the voxel means are set-major, and set s's block is its
// one-set index shifted by its first point (perm, start) and carrying its prefix (keys).  S = 1 is today's layout.  A
// query of set s searches set s's cells only (IndexView::in_set); the build synchronises twice whatever S is.  The
// many-set queries are nearest (queries carry a set table) and normals (each sorted point finds its set from poff).
//
// Decisions are float64 with the reference's operation order and no FMA contraction:
//   d2 = (dx*dx + dy*dy) + dz*dz     scipy's sqeuclidean_distance_double (cKDTree.query, query_ball_point)
// and a cell range is widened by 1e-6 cells on each side, far more than the rounding of (q - origin +- R) / cell for
// coordinates below 2^21 cells, so the candidate set always contains every point the float64 predicate accepts.
#include <algorithm>
#include <cmath>
#include <cub/cub.cuh>
#include "cg_cloud_index.cuh"

namespace {

// ---- index construction ------------------------------------------------------------------------------------------

constexpr int BT = 256;

// per block: min xyz, max xyz, and 1.0 when a coordinate is not finite.  Blocks [s * nbs, (s + 1) * nbs) cover set s,
// the points [off[s], off[s + 1]) (off null: one set, the P points)
__global__ void __launch_bounds__(BT) bounds_kernel(const double *__restrict__ pts, int P, const int32_t *__restrict__ off,
                                                    int nbs, double *__restrict__ part) {
  double v[7] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY, 0.0};
  const int s = off ? blockIdx.x / nbs : 0, c = blockIdx.x - s * nbs;
  const int lo = off ? off[s] : 0, hi = off ? off[s + 1] : P;
  for (int i = lo + c * BT + threadIdx.x; i < hi; i += nbs * BT) {
    for (int a = 0; a < 3; a++) {
      const double x = pts[3 * (size_t)i + a];
      if (!isfinite(x)) v[6] = 1.0;
      v[a] = fmin(v[a], x);
      v[3 + a] = fmax(v[3 + a], x);
    }
  }
  __shared__ double sh[7][BT / 32];
  for (int a = 0; a < 7; a++) {
    double x = v[a];
    for (int o = 16; o; o >>= 1) {
      const double y = __shfl_xor_sync(0xffffffffu, x, o);
      x = (a < 3) ? fmin(x, y) : fmax(x, y);
    }
    if ((threadIdx.x & 31) == 0) sh[a][threadIdx.x >> 5] = x;
  }
  __syncthreads();
  if (threadIdx.x < 7) {
    const int a = threadIdx.x;
    double x = sh[a][0];
    for (int w = 1; w < BT / 32; w++) x = (a < 3) ? fmin(x, sh[a][w]) : fmax(x, sh[a][w]);
    part[(size_t)blockIdx.x * 7 + a] = x;
  }
}

// block s: set s's bounds from its nb partials
__global__ void __launch_bounds__(BT) bounds_final_kernel(const double *__restrict__ part, int nb, double *__restrict__ out) {
  if (threadIdx.x >= 7) return;
  const int a = threadIdx.x;
  const double *p = part + (size_t)blockIdx.x * nb * 7;
  double x = p[a];
  for (int b = 1; b < nb; b++) x = (a < 3) ? fmin(x, p[(size_t)b * 7 + a]) : fmax(x, p[(size_t)b * 7 + a]);
  out[(size_t)blockIdx.x * 7 + a] = x;
}

// sets null: one set with origin (ox, oy, oz); else point i's set from off, with that set's origin and prefix
__global__ void key_kernel(const double *__restrict__ pts, int P, double ox, double oy, double oz, double cell, int bits,
                           const CloudSet *__restrict__ sets, const int32_t *__restrict__ off, int S,
                           uint64_t *__restrict__ keys, int32_t *__restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  uint64_t prefix = 0;
  if (sets) {
    const int s = set_of(off, S, i);
    ox = sets[s].o[0]; oy = sets[s].o[1]; oz = sets[s].o[2];
    prefix = (uint64_t)s << (3 * bits);
  }
  keys[i] = prefix | cell_key(pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2], ox, oy, oz, cell, bits);
  vals[i] = i;
}

__global__ void head_flag_kernel(const uint64_t *__restrict__ keys, int P, int32_t *__restrict__ flag) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < P) flag[j] = (j == 0 || keys[j] != keys[j - 1]) ? 1 : 0;
}

// cell table and the points in key order; cid = exclusive scan of the head flags.  coff (S+1): each set's first cell
// (set = key >> sh; every set has a point, so a cell), coff[S] = U
__global__ void table_kernel(const uint64_t *__restrict__ keys, const int32_t *__restrict__ perm, const int32_t *__restrict__ cid,
                             const double *__restrict__ pts, int P, int sh, uint64_t *__restrict__ ukey,
                             int32_t *__restrict__ start, double *__restrict__ spts, int *__restrict__ U,
                             int32_t *__restrict__ coff) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  const bool head = j == 0 || keys[j] != keys[j - 1];
  if (head) {
    ukey[cid[j]] = keys[j];
    start[cid[j]] = j;
    if (j == 0 || (keys[j] >> sh) != (keys[j - 1] >> sh)) coff[keys[j] >> sh] = cid[j];
  }
  if (j == P - 1) {                       // cells = heads before the last point, plus the last point if it is one
    const int u = cid[j] + (head ? 1 : 0);
    start[u] = P;
    *U = u;
    coff[(keys[j] >> sh) + 1] = u;
  }
  const size_t o = 3 * (size_t)perm[j];
  spts[3 * (size_t)j] = pts[o];
  spts[3 * (size_t)j + 1] = pts[o + 1];
  spts[3 * (size_t)j + 2] = pts[o + 2];
}

// ---- voxel down-sampling (open3d VoxelDownSample) ----------------------------------------------------------------

// one thread per occupied cell: members summed in ascending point index, divided by the count; the normal sum is
// normalised (Eigen's normalized(): unchanged when its squared norm is 0)
__global__ void voxel_kernel(IndexView V, const double *__restrict__ nrm, double *__restrict__ out_pts,
                             double *__restrict__ out_nrm) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= V.U) return;
  const int s = V.start[u], e = V.start[u + 1];
  double sx = 0.0, sy = 0.0, sz = 0.0, nx = 0.0, ny = 0.0, nz = 0.0;
  for (int k = s; k < e; k++) {
    sx = __dadd_rn(sx, V.spts[3 * (size_t)k]);
    sy = __dadd_rn(sy, V.spts[3 * (size_t)k + 1]);
    sz = __dadd_rn(sz, V.spts[3 * (size_t)k + 2]);
    if (nrm) {
      const size_t o = 3 * (size_t)V.perm[k];
      nx = __dadd_rn(nx, nrm[o]);
      ny = __dadd_rn(ny, nrm[o + 1]);
      nz = __dadd_rn(nz, nrm[o + 2]);
    }
  }
  const double c = (double)(e - s);
  out_pts[3 * (size_t)u] = __ddiv_rn(sx, c);
  out_pts[3 * (size_t)u + 1] = __ddiv_rn(sy, c);
  out_pts[3 * (size_t)u + 2] = __ddiv_rn(sz, c);
  if (nrm) {
    const double q = __dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz));
    if (q > 0.0) {
      const double n = sqrt(q);
      nx = __ddiv_rn(nx, n); ny = __ddiv_rn(ny, n); nz = __ddiv_rn(nz, n);
    }
    out_nrm[3 * (size_t)u] = nx;
    out_nrm[3 * (size_t)u + 1] = ny;
    out_nrm[3 * (size_t)u + 2] = nz;
  }
}

// ---- nearest point within a bound (cKDTree.query) ----------------------------------------------------------------

// qoff null: every query searches the whole (one-set) index; else the queries [qoff[s], qoff[s + 1]) search set s
// only, and the answer is the point's index in the whole index (set s's first point plus its index in the set)
__global__ void nearest_kernel(IndexView V0, const int32_t *__restrict__ qoff, const double *__restrict__ q, int Q,
                               double max_dist, int32_t *__restrict__ out_idx, double *__restrict__ out_dist) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Q) return;
  const IndexView V = qoff ? V0.in_set(set_of(qoff, V0.S, i)) : V0;
  const double qx = q[3 * (size_t)i], qy = q[3 * (size_t)i + 1], qz = q[3 * (size_t)i + 2];
  double best = INFINITY;
  int bi = 0x7fffffff;
  const Columns C(V, qx, qy, qz, max_dist);
  if (C.any) {
    for (int64_t cx = C.x0; cx <= C.x1; cx++)
      for (int64_t cy = C.y0; cy <= C.y1; cy++) {
        int s, e;
        C.run(V, cx, cy, s, e);
        for (int k = s; k < e; k++) {
          const double d2 = dist2(qx, qy, qz, V.spts[3 * (size_t)k], V.spts[3 * (size_t)k + 1], V.spts[3 * (size_t)k + 2]);
          const int id = V.perm[k];
          if (d2 < best || (d2 == best && id < bi)) { best = d2; bi = id; }   // ties: the smaller index
        }
      }
  }
  const double d = sqrt(best);
  const bool ok = bi != 0x7fffffff && d <= max_dist;
  out_idx[i] = ok ? bi : -1;
  out_dist[i] = ok ? d : INFINITY;
}

// ---- radius membership (query_ball_point) and the crop -----------------------------------------------------------

// mark[i] = some indexed point p has d2(q_i, p) <= r2 (compare_sqrt == 0) or sqrt(d2) <= r (compare_sqrt == 1)
__global__ void radius_mask_kernel(IndexView V, const double *__restrict__ q, int Q, double r, double r2, int compare_sqrt,
                                   uint8_t *__restrict__ mark) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Q) return;
  const double qx = q[3 * (size_t)i], qy = q[3 * (size_t)i + 1], qz = q[3 * (size_t)i + 2];
  bool hit = false;
  const Columns C(V, qx, qy, qz, r);
  if (C.any) {
    for (int64_t cx = C.x0; cx <= C.x1 && !hit; cx++)
      for (int64_t cy = C.y0; cy <= C.y1 && !hit; cy++) {
        int s, e;
        C.run(V, cx, cy, s, e);
        for (int k = s; k < e; k++) {
          const double d2 = dist2(qx, qy, qz, V.spts[3 * (size_t)k], V.spts[3 * (size_t)k + 1], V.spts[3 * (size_t)k + 2]);
          if (compare_sqrt ? sqrt(d2) <= r : d2 <= r2) { hit = true; break; }
        }
      }
  }
  mark[i] = hit ? 1 : 0;
}

// ---- normal estimation (open3d EstimateNormals, KDTreeSearchParamHybrid) + correct_pcd_normal_direction -------------
//
// One warp per point.  The warp walks the point's columns 32 candidates at a time and appends the ones with
// d2 <= r*r to a per-warp buffer in shared memory.  When the buffer could overflow it is compacted to its max_nn
// smallest (d2, index) keys, which always frees room because max_nn <= NRM_MAX_NN < NRM_CAP - 32; a final compaction
// leaves the neighbourhood at [0, n) in (d2, index) order.  A compaction ranks every entry against all the others
// (keys are unique: they contain the index), so no thread keeps a heap and the selection is order-independent.

constexpr int NW = 4;                 // warps per CTA
constexpr int NRM_CAP = 256;          // candidate slots per warp
constexpr int NRM_SLOTS = NRM_CAP / 32;

struct NbrBuf {
  double d2[NRM_CAP];
  int32_t id[NRM_CAP];    // original point index (the tie key)
  int32_t pos[NRM_CAP];   // sorted position (where its coordinates are)
};

__device__ __forceinline__ bool key_less(double da, int ia, double db, int ib) { return da < db || (da == db && ia < ib); }

// keep the max_nn smallest keys of buf[0, n), in key order at [0, min(n, max_nn))
__device__ int compact(NbrBuf &B, int n, int max_nn, int lane) {
  double rd[NRM_SLOTS];
  int ri[NRM_SLOTS], rp[NRM_SLOTS], rr[NRM_SLOTS];
#pragma unroll
  for (int s = 0; s < NRM_SLOTS; s++) {
    const int i = lane + 32 * s;
    rd[s] = i < n ? B.d2[i] : INFINITY;
    ri[s] = i < n ? B.id[i] : 0x7fffffff;
    rp[s] = i < n ? B.pos[i] : 0;
    rr[s] = 0;
  }
  for (int m = 0; m < n; m++) {
    const double dm = B.d2[m];
    const int im = B.id[m];
#pragma unroll
    for (int s = 0; s < NRM_SLOTS; s++) rr[s] += key_less(dm, im, rd[s], ri[s]) ? 1 : 0;
  }
  __syncwarp();
#pragma unroll
  for (int s = 0; s < NRM_SLOTS; s++) {
    const int i = lane + 32 * s;
    if (i < n && rr[s] < max_nn) {
      B.d2[rr[s]] = rd[s];
      B.id[rr[s]] = ri[s];
      B.pos[rr[s]] = rp[s];
    }
  }
  __syncwarp();
  return n < max_nn ? n : max_nn;
}

// eigenvector of the smallest eigenvalue of a symmetric 3x3 matrix: cyclic Jacobi rotations until the off-diagonal
// part is below 1e-17 of the matrix's norm (backward stable, so the vector's error is O(u ||A|| / gap))
__device__ void smallest_eigvec(double a[3][3], double out[3]) {
  double v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  const double fro = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2] +
                     2.0 * (a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2]);
  for (int sweep = 0; sweep < 32; sweep++) {
    const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
    if (off <= 1e-34 * fro) break;
#pragma unroll
    for (int p = 0; p < 2; p++)
#pragma unroll
      for (int q = p + 1; q < 3; q++) {
        const double apq = a[p][q];
        if (apq == 0.0) continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
        const double t = fabs(theta) > 1e150 ? 0.5 / theta : copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
        for (int k = 0; k < 3; k++) {                 // A <- A J  (columns p, q)
          const double akp = a[k][p], akq = a[k][q];
          a[k][p] = c * akp - s * akq;
          a[k][q] = s * akp + c * akq;
        }
#pragma unroll
        for (int k = 0; k < 3; k++) {                 // A <- J^T A  (rows p, q)
          const double apk = a[p][k], aqk = a[q][k];
          a[p][k] = c * apk - s * aqk;
          a[q][k] = s * apk + c * aqk;
        }
        a[p][q] = a[q][p] = 0.0;
#pragma unroll
        for (int k = 0; k < 3; k++) {                 // V <- V J
          const double vkp = v[k][p], vkq = v[k][q];
          v[k][p] = c * vkp - s * vkq;
          v[k][q] = s * vkp + c * vkq;
        }
      }
  }
  const int m01 = a[1][1] < a[0][0] ? 1 : 0;                   // first smallest diagonal entry
  const double l01 = m01 ? a[1][1] : a[0][0];
  const int m = a[2][2] < l01 ? 2 : m01;
#pragma unroll
  for (int k = 0; k < 3; k++) out[k] = m == 0 ? v[k][0] : (m == 1 ? v[k][1] : v[k][2]);
}

// A many-set index (V0.S > 1): sorted point j belongs to the set whose point range holds j (the sorted points are
// set-major) and searches that set's cells only, so its neighbours, counts and normal are those of a one-set index over
// the set alone; ids stay indices into the whole index.  The minimum of one CTA per SM keeps ptxas from trading the
// set's view for a stack frame and spills.
__global__ void __launch_bounds__(NW * 32, 1) normals_kernel(IndexView V0, int P, double r, double r2, int max_nn,
                                                             double vx, double vy, double vz, double *__restrict__ out_n,
                                                             int32_t *__restrict__ out_nbr, int32_t *__restrict__ out_cnt) {
  __shared__ NbrBuf bufs[NW];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  NbrBuf &B = bufs[w];
  for (int j = blockIdx.x * NW + w; j < P; j += gridDim.x * NW) {
    IndexView V = V0;
    if (V0.S > 1) V = V0.in_set(set_of(V0.poff, V0.S, j));
    const double qx = V.spts[3 * (size_t)j], qy = V.spts[3 * (size_t)j + 1], qz = V.spts[3 * (size_t)j + 2];
    const Columns C(V, qx, qy, qz, r);
    int n = 0;
    if (C.any) {
      for (int64_t cx = C.x0; cx <= C.x1; cx++)
        for (int64_t cy = C.y0; cy <= C.y1; cy++) {
          int s, e;
          C.run(V, cx, cy, s, e);
          for (int base = s; base < e; base += 32) {
            const int k = base + lane;
            double d2 = INFINITY;
            bool hit = false;
            if (k < e) {
              d2 = dist2(qx, qy, qz, V.spts[3 * (size_t)k], V.spts[3 * (size_t)k + 1], V.spts[3 * (size_t)k + 2]);
              hit = d2 <= r2;
            }
            const unsigned bal = __ballot_sync(0xffffffffu, hit);
            if (!bal) continue;
            if (n + 32 > NRM_CAP) n = compact(B, n, max_nn, lane);
            if (hit) {
              const int at = n + __popc(bal & ((1u << lane) - 1u));
              B.d2[at] = d2;
              B.id[at] = V.perm[k];
              B.pos[at] = k;
            }
            n += __popc(bal);
            __syncwarp();
          }
        }
    }
    n = compact(B, n, max_nn, lane);
    const int orig = V.perm[j];
    if (out_nbr)
      for (int t = lane; t < max_nn; t += 32) out_nbr[(size_t)orig * max_nn + t] = t < n ? B.id[t] : -1;
    if (lane == 0) {
      if (out_cnt) out_cnt[orig] = n;
      double nx = 0.0, ny = 0.0, nz = 1.0;
      if (n >= 3) {
        // two-pass float64 covariance about the mean, neighbours in (d2, index) order
        double sx = 0.0, sy = 0.0, sz = 0.0;
        for (int t = 0; t < n; t++) {
          const size_t o = 3 * (size_t)B.pos[t];
          sx = __dadd_rn(sx, V.spts[o]); sy = __dadd_rn(sy, V.spts[o + 1]); sz = __dadd_rn(sz, V.spts[o + 2]);
        }
        const double cn = (double)n;
        const double mx = __ddiv_rn(sx, cn), my = __ddiv_rn(sy, cn), mz = __ddiv_rn(sz, cn);
        double c00 = 0.0, c01 = 0.0, c02 = 0.0, c11 = 0.0, c12 = 0.0, c22 = 0.0;
        for (int t = 0; t < n; t++) {
          const size_t o = 3 * (size_t)B.pos[t];
          const double dx = __dsub_rn(V.spts[o], mx), dy = __dsub_rn(V.spts[o + 1], my), dz = __dsub_rn(V.spts[o + 2], mz);
          c00 = __dadd_rn(c00, __dmul_rn(dx, dx)); c01 = __dadd_rn(c01, __dmul_rn(dx, dy));
          c02 = __dadd_rn(c02, __dmul_rn(dx, dz)); c11 = __dadd_rn(c11, __dmul_rn(dy, dy));
          c12 = __dadd_rn(c12, __dmul_rn(dy, dz)); c22 = __dadd_rn(c22, __dmul_rn(dz, dz));
        }
        double A[3][3] = {{__ddiv_rn(c00, cn), __ddiv_rn(c01, cn), __ddiv_rn(c02, cn)},
                          {__ddiv_rn(c01, cn), __ddiv_rn(c11, cn), __ddiv_rn(c12, cn)},
                          {__ddiv_rn(c02, cn), __ddiv_rn(c12, cn), __ddiv_rn(c22, cn)}};
        const bool zero = A[0][0] == 0.0 && A[0][1] == 0.0 && A[0][2] == 0.0 && A[1][1] == 0.0 && A[1][2] == 0.0 &&
                          A[2][2] == 0.0;
        if (!zero) {
          double ev[3];
          smallest_eigvec(A, ev);
          const double l = sqrt(ev[0] * ev[0] + ev[1] * ev[1] + ev[2] * ev[2]);
          if (l > 0.0) { nx = ev[0] / l; ny = ev[1] / l; nz = ev[2] / l; }
        }
      }
      // Utils.py:205-213 correct_pcd_normal_direction, numpy's operation order
      const double ux = __dsub_rn(vx, qx), uy = __dsub_rn(vy, qy), uz = __dsub_rn(vz, qz);
      const double un = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), __dmul_rn(uz, uz)));
      const double wx = __ddiv_rn(ux, un), wy = __ddiv_rn(uy, un), wz = __ddiv_rn(uz, un);
      const double nn = __dadd_rn(sqrt(__dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz))), 1e-10);
      nx = __ddiv_rn(nx, nn); ny = __ddiv_rn(ny, nn); nz = __ddiv_rn(nz, nn);
      const double dot = __dadd_rn(__dadd_rn(__dmul_rn(wx, nx), __dmul_rn(wy, ny)), __dmul_rn(wz, nz));
      if (dot < 0.0) { nx = -nx; ny = -ny; nz = -nz; }
      out_n[3 * (size_t)orig] = nx;
      out_n[3 * (size_t)orig + 1] = ny;
      out_n[3 * (size_t)orig + 2] = nz;
    }
    __syncwarp();
  }
}

// ---- back-projection (Utils.py:239-251 depth2xyzmap) ---------------------------------------------------------------

// x = (u - cx) * z / fx, y = (v - cy) * z / fy in float64 left to right, narrowed to float32; depth < 0.1 (compared in
// the depth's own type, as numpy compares an array with a Python float) gives (0, 0, 0)
template <typename T>
__global__ void depth2xyz_kernel(const T *__restrict__ depth, int H, int W, double fx, double cx, double fy, double cy,
                                 float *__restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)H * W) return;
  const T z = depth[i];
  float x = 0.f, y = 0.f, zz = 0.f;
  if (!(z < (T)0.1)) {
    const double zd = (double)z;
    const double u = (double)(i % W), v = (double)(i / W);
    x = (float)__ddiv_rn(__dmul_rn(__dsub_rn(u, cx), zd), fx);
    y = (float)__ddiv_rn(__dmul_rn(__dsub_rn(v, cy), zd), fy);
    zz = (float)zd;
  }
  out[3 * i] = x;
  out[3 * i + 1] = y;
  out[3 * i + 2] = zz;
}

unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace

extern "C" int cg_depth2xyz_dev(cg_ctx *ctx, const void *depth, int depth_is_f64, int H, int W, const double *K, float *out_xyz) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, depth && K && out_xyz && H > 0 && W > 0, "depth2xyz: bad arguments");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const int64_t n = (int64_t)H * W;
  if (depth_is_f64)
    depth2xyz_kernel<double><<<blocks(n, 256), 256, 0, ctx->stream>>>((const double *)depth, H, W, K[0], K[2], K[4], K[5], out_xyz);
  else
    depth2xyz_kernel<float><<<blocks(n, 256), 256, 0, ctx->stream>>>((const float *)depth, H, W, K[0], K[2], K[4], K[5], out_xyz);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

namespace {

int bit_length(int v) {
  int n = 0;
  while (v >> n) n++;
  return n;
}

// The one build behind cg_cloud_index_create (off null: one set of P points) and cg_cloud_index_create_many (S sets,
// set s the points [off[s], off[s + 1]) of pts, off on the host).  Synchronises twice: the bounds, then the cells.
int cloud_index_build(cg_ctx *ctx, const double *pts, int P, const int32_t *off, int S, double cell, cg_cloud_index **out) {
  const bool many = off != nullptr;
  CG_REQUIRE(ctx, pts && out && P > 0, "cloud_index: null argument or no points");
  CG_REQUIRE(ctx, cell > 0.0 && std::isfinite(cell), "cloud_index: cell size must be positive and finite");
  if (many) {
    CG_REQUIRE(ctx, off[0] == 0 && off[S] == P, "cloud_index: the set offsets must run from 0 to the point count");
    for (int s = 0; s < S; s++) CG_REQUIRE(ctx, off[s] < off[s + 1], "cloud_index: every set needs at least one point");
  }
  *out = nullptr;
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const int nb = (int)std::min<int64_t>(blocks(P, BT), 2 * (int64_t)ctx->num_sms);
  const int nbs = std::max(1, nb / S);   // bounds blocks per set; one set keeps nb
  const size_t Sz = (size_t)S;
  // workspace: bounds partials | keys in/out | vals | head flags | scanned ids | U and the cell offsets | set offsets
  // (many sets) | CUB temp
  size_t sort_tmp = 0, scan_tmp = 0;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (uint64_t *)nullptr, (uint64_t *)nullptr, (int32_t *)nullptr,
                                               (int32_t *)nullptr, P, 0, 3 * MAX_AXIS_BITS, ctx->stream));
  CG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (int32_t *)nullptr, (int32_t *)nullptr, P, ctx->stream));
  const size_t tmp = std::max(sort_tmp, scan_tmp);
  double *part; uint64_t *kin, *kout; int32_t *vin, *flag, *cid, *dU, *doff; void *dtmp;
  int rc = cg_ws_carve(ctx, [&](cg_arena &ar) {
    part = ar.take<double>(7 * ((size_t)nbs * Sz + Sz));
    kin = ar.take<uint64_t>(P); kout = ar.take<uint64_t>(P);
    vin = ar.take<int32_t>(P); flag = ar.take<int32_t>(P); cid = ar.take<int32_t>(P);
    dU = ar.take<int32_t>(Sz + 2);
    doff = ar.take<int32_t>(many ? Sz + 1 : 0);
    dtmp = ar.take<char>(tmp);
  });
  if (rc != CG_OK) return rc;
  double *bnd = part + 7 * (size_t)nbs * Sz;
  // the set offsets, from pageable memory: staged at once, no synchronisation
  if (many) CG_CUDA(ctx, cudaMemcpyAsync(doff, off, sizeof(int32_t) * (Sz + 1), cudaMemcpyHostToDevice, ctx->stream));

  bounds_kernel<<<nbs * S, BT, 0, ctx->stream>>>(pts, P, many ? doff : nullptr, nbs, part);
  CG_LAUNCH_CHECK(ctx);
  bounds_final_kernel<<<S, BT, 0, ctx->stream>>>(part, nbs, bnd);
  CG_LAUNCH_CHECK(ctx);
  std::vector<double> hb(7 * Sz);
  CG_CUDA(ctx, cudaMemcpyAsync(hb.data(), bnd, sizeof(double) * hb.size(), cudaMemcpyDeviceToHost, ctx->stream));
  CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));

  cg_cloud_index ix;   // goes to the heap only when every step below has succeeded
  ix.ctx = ctx;
  ix.P = P;
  ix.cell = cell;
  ix.S = S;
  ix.sets.resize(Sz);
  ix.set_hi.resize(3 * Sz);
  int64_t maxc = 0;
  for (int s = 0; s < S; s++) {
    const double *h = &hb[7 * (size_t)s];
    CG_REQUIRE(ctx, h[6] == 0.0, "cloud_index: a coordinate is NaN or infinite");
    for (int a = 0; a < 3; a++) {
      const double o = h[a] - cell * 0.5;                               // open3d: min_bound - voxel_size * 0.5
      const double top = floor((h[3 + a] - o) / cell);                  // the largest point's cell (floor is monotone)
      CG_REQUIRE(ctx, top < (double)(1 << MAX_AXIS_BITS),
                 "cloud_index: the cloud spans 2^21 or more cells on an axis; use a larger cell");
      ix.sets[s].o[a] = o;
      ix.sets[s].mc[a] = (int64_t)top;
      ix.set_hi[3 * (size_t)s + a] = h[3 + a];
      maxc = std::max(maxc, ix.sets[s].mc[a]);
    }
  }
  for (int a = 0; a < 3; a++) {
    ix.origin[a] = ix.sets[0].o[a];
    ix.hi[a] = ix.set_hi[a];
    ix.maxc[a] = ix.sets[0].mc[a];
  }
  int bits = 1;
  while ((int64_t(1) << bits) <= maxc) bits++;
  ix.bits = bits;
  const int set_bits = bit_length(S - 1), key_bits = set_bits + 3 * bits;
  CG_REQUIRE(ctx, key_bits <= 63,
             "cloud_index: " + std::to_string(S) + " sets need " + std::to_string(set_bits) + " set bits and the "
             "largest set spans " + std::to_string(maxc + 1) + " cells, " + std::to_string(bits) + " bits per axis; "
             "the key holds set bits + 3 * bits <= 63");
  ix.poff = many ? std::vector<int32_t>(off, off + S + 1) : std::vector<int32_t>{0, P};
  // the set table and the set offsets (many sets) live behind the sorted points, in one allocation
  const size_t pts_bytes = sizeof(double) * 3 * (size_t)P;
  const size_t set_bytes = many ? sizeof(CloudSet) * Sz + sizeof(int32_t) * (Sz + 1) : 0;
  DevBuf spts, perm, ukey, start;
  if ((rc = dev_alloc(ctx, spts, pts_bytes + set_bytes))) return rc;
  if ((rc = dev_alloc(ctx, perm, sizeof(int32_t) * (size_t)P))) return rc;
  if ((rc = dev_alloc(ctx, ukey, sizeof(uint64_t) * (size_t)P))) return rc;
  if ((rc = dev_alloc(ctx, start, sizeof(int32_t) * ((size_t)P + 1)))) return rc;
  ix.spts = static_cast<double *>(spts.p); ix.perm = static_cast<int32_t *>(perm.p);
  ix.ukey = static_cast<uint64_t *>(ukey.p); ix.start = static_cast<int32_t *>(start.p);
  if (many) {
    CloudSet *d_sets = reinterpret_cast<CloudSet *>(static_cast<char *>(spts.p) + pts_bytes);
    int32_t *d_poff = reinterpret_cast<int32_t *>(d_sets + S);
    CG_CUDA(ctx, cudaMemcpyAsync(d_sets, ix.sets.data(), sizeof(CloudSet) * Sz, cudaMemcpyHostToDevice, ctx->stream));
    CG_CUDA(ctx, cudaMemcpyAsync(d_poff, off, sizeof(int32_t) * (Sz + 1), cudaMemcpyHostToDevice, ctx->stream));
    ix.d_sets = d_sets;
    ix.d_poff = d_poff;
  }

  key_kernel<<<blocks(P, 256), 256, 0, ctx->stream>>>(pts, P, ix.origin[0], ix.origin[1], ix.origin[2], cell, bits,
                                                      ix.d_sets, many ? doff : nullptr, S, kin, vin);
  CG_LAUNCH_CHECK(ctx);
  size_t tb = tmp;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(dtmp, tb, kin, kout, vin, ix.perm, P, 0, key_bits, ctx->stream));
  head_flag_kernel<<<blocks(P, 256), 256, 0, ctx->stream>>>(kout, P, flag);
  CG_LAUNCH_CHECK(ctx);
  tb = tmp;
  CG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(dtmp, tb, flag, cid, P, ctx->stream));
  table_kernel<<<blocks(P, 256), 256, 0, ctx->stream>>>(kout, ix.perm, cid, pts, P, 3 * bits, ix.ukey, ix.start, ix.spts,
                                                        dU, dU + 1);
  CG_LAUNCH_CHECK(ctx);
  std::vector<int32_t> hu(Sz + 2);
  CG_CUDA(ctx, cudaMemcpyAsync(hu.data(), dU, sizeof(int32_t) * hu.size(), cudaMemcpyDeviceToHost, ctx->stream));
  CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  ix.U = hu[0];
  ix.coff.assign(hu.begin() + 1, hu.end());
  spts.release(); perm.release(); ukey.release(); start.release();   // owned by the index now
  *out = new cg_cloud_index(std::move(ix));
  return CG_OK;
}

}  // namespace

extern "C" int cg_cloud_index_create(cg_ctx *ctx, const double *pts, int P, double cell, cg_cloud_index **out) {
  if (!ctx) return CG_EINVAL;
  return cloud_index_build(ctx, pts, P, nullptr, 1, cell, out);
}

extern "C" int cg_cloud_index_create_many(cg_ctx *ctx, const double *pts, const int32_t *set_offsets, int S, double cell,
                                          cg_cloud_index **out) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, set_offsets && S >= 1, "cloud_index_many: null set offsets or S < 1");
  return cloud_index_build(ctx, pts, set_offsets[S], set_offsets, S, cell, out);
}

extern "C" int cg_cloud_index_sets(const cg_cloud_index *ix, int *out_sets, int32_t *out_cell_offsets) {
  if (!ix) return CG_EINVAL;
  if (out_sets) *out_sets = ix->S;
  if (out_cell_offsets) std::copy(ix->coff.begin(), ix->coff.end(), out_cell_offsets);
  return CG_OK;
}

extern "C" int cg_cloud_index_tables_dev(const cg_cloud_index *ix, double *out_pts, int32_t *out_perm,
                                         uint64_t *out_keys, int32_t *out_start) {
  if (!ix) return CG_EINVAL;
  cg_ctx *ctx = ix->ctx;
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t P = (size_t)ix->P, U = (size_t)ix->U;
  if (out_pts) CG_CUDA(ctx, cudaMemcpyAsync(out_pts, ix->spts, sizeof(double) * 3 * P, cudaMemcpyDeviceToDevice, ctx->stream));
  if (out_perm) CG_CUDA(ctx, cudaMemcpyAsync(out_perm, ix->perm, sizeof(int32_t) * P, cudaMemcpyDeviceToDevice, ctx->stream));
  if (out_keys) CG_CUDA(ctx, cudaMemcpyAsync(out_keys, ix->ukey, sizeof(uint64_t) * U, cudaMemcpyDeviceToDevice, ctx->stream));
  if (out_start)
    CG_CUDA(ctx, cudaMemcpyAsync(out_start, ix->start, sizeof(int32_t) * (U + 1), cudaMemcpyDeviceToDevice, ctx->stream));
  return CG_OK;
}

extern "C" void cg_cloud_index_destroy(cg_cloud_index *ix) {
  if (!ix) return;
  cudaSetDevice(ix->ctx->device);
  cudaStreamSynchronize(ix->ctx->stream);
  cudaFree(ix->spts);
  cudaFree(ix->perm);
  cudaFree(ix->ukey);
  cudaFree(ix->start);
  delete ix;
}

extern "C" int cg_cloud_index_info(const cg_cloud_index *ix, int *out_points, int *out_cells, double *out_cell, double *out_origin) {
  if (!ix) return CG_EINVAL;
  if (out_points) *out_points = ix->P;
  if (out_cells) *out_cells = ix->U;
  if (out_cell) *out_cell = ix->cell;
  if (out_origin)
    for (int a = 0; a < 3; a++) out_origin[a] = ix->origin[a];
  return CG_OK;
}

extern "C" int cg_voxel_down_sample_dev(const cg_cloud_index *ix, const double *normals, double *out_pts, double *out_normals) {
  if (!ix) return CG_EINVAL;
  cg_ctx *ctx = ix->ctx;
  CG_REQUIRE(ctx, out_pts && (!normals || out_normals), "voxel_down_sample: null output");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  voxel_kernel<<<blocks(ix->U, 128), 128, 0, ctx->stream>>>(view_of(ix), normals, out_pts, normals ? out_normals : nullptr);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_cloud_nearest_dev(const cg_cloud_index *ix, const double *query, int Q, double max_dist, int32_t *out_idx,
                                    double *out_dist) {
  if (!ix) return CG_EINVAL;
  cg_ctx *ctx = ix->ctx;
  CG_REQUIRE(ctx, ix->S == 1, "cloud_nearest: the index holds several sets; use cg_cloud_nearest_many_dev");
  CG_REQUIRE(ctx, Q >= 0 && (Q == 0 || (query && out_idx && out_dist)), "cloud_nearest: bad arguments");   // empty: NULL allowed
  CG_REQUIRE(ctx, max_dist >= 0.0 && std::isfinite(max_dist), "cloud_nearest: max_dist must be finite and >= 0");
  if (Q == 0) return CG_OK;
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  nearest_kernel<<<blocks(Q, 128), 128, 0, ctx->stream>>>(view_of(ix), nullptr, query, Q, max_dist, out_idx, out_dist);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_cloud_nearest_many_dev(const cg_cloud_index *ix, const double *query, const int32_t *query_offsets, int Q,
                                         double max_dist, int32_t *out_idx, double *out_dist) {
  if (!ix) return CG_EINVAL;
  cg_ctx *ctx = ix->ctx;
  const int S = ix->S;
  CG_REQUIRE(ctx, query_offsets, "cloud_nearest_many: null query offsets");
  CG_REQUIRE(ctx, Q >= 0 && (Q == 0 || (query && out_idx && out_dist)), "cloud_nearest_many: bad arguments");
  CG_REQUIRE(ctx, query_offsets[0] == 0 && query_offsets[S] == Q,
             "cloud_nearest_many: the query offsets must run from 0 to Q, one range per set");
  for (int s = 0; s < S; s++)
    CG_REQUIRE(ctx, query_offsets[s] <= query_offsets[s + 1], "cloud_nearest_many: the query offsets must not decrease");
  CG_REQUIRE(ctx, max_dist >= 0.0 && std::isfinite(max_dist), "cloud_nearest_many: max_dist must be finite and >= 0");
  if (Q == 0) return CG_OK;
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  int32_t *qoff = nullptr;
  if (S > 1) {
    const int rc = cg_ws_carve(ctx, [&](cg_arena &ar) { qoff = ar.take<int32_t>((size_t)S + 1); });
    if (rc != CG_OK) return rc;
    // from pageable memory: staged at once, no synchronisation
    CG_CUDA(ctx, cudaMemcpyAsync(qoff, query_offsets, sizeof(int32_t) * ((size_t)S + 1), cudaMemcpyHostToDevice,
                                 ctx->stream));
  }
  nearest_kernel<<<blocks(Q, 128), 128, 0, ctx->stream>>>(view_of(ix), qoff, query, Q, max_dist, out_idx, out_dist);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_cloud_radius_mask_dev(const cg_cloud_index *ix, const double *query, int Q, double r, int compare_sqrt,
                                        uint8_t *out_mask) {
  if (!ix) return CG_EINVAL;
  cg_ctx *ctx = ix->ctx;
  CG_REQUIRE(ctx, ix->S == 1, "cloud_radius_mask: the index holds several sets, and the queries carry none");
  CG_REQUIRE(ctx, Q >= 0 && (Q == 0 || (query && out_mask)), "cloud_radius_mask: bad arguments");   // empty: NULL allowed
  CG_REQUIRE(ctx, r >= 0.0 && std::isfinite(r), "cloud_radius_mask: r must be finite and >= 0");
  if (Q == 0) return CG_OK;
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  radius_mask_kernel<<<blocks(Q, 128), 128, 0, ctx->stream>>>(view_of(ix), query, Q, r, r * r, compare_sqrt ? 1 : 0, out_mask);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

namespace {

// the one launch behind cg_cloud_normals_dev and cg_cloud_normals_many_dev; a many-set index's sets are in its view
int cloud_normals(const cg_cloud_index *ix, const char *what, double radius, int max_nn, const double *view_point,
                  double *out_normals, int32_t *out_nbr, int32_t *out_nbr_count) {
  cg_ctx *ctx = ix->ctx;
  CG_REQUIRE(ctx, view_point && out_normals, std::string(what) + ": null argument");
  CG_REQUIRE(ctx, radius >= 0.0 && std::isfinite(radius), std::string(what) + ": radius must be finite and >= 0");
  CG_REQUIRE(ctx, max_nn >= 1 && max_nn <= CG_CLOUD_MAX_NN, std::string(what) + ": 1 <= max_nn <= CG_CLOUD_MAX_NN");
  static_assert(CG_CLOUD_MAX_NN <= NRM_CAP - 32, "compaction must free room");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const int grid = (int)std::min<int64_t>(blocks(ix->P, NW), 16 * (int64_t)ctx->num_sms);
  normals_kernel<<<grid, NW * 32, 0, ctx->stream>>>(view_of(ix), ix->P, radius, radius * radius, max_nn, view_point[0],
                                                    view_point[1], view_point[2], out_normals, out_nbr, out_nbr_count);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

}  // namespace

extern "C" int cg_cloud_normals_dev(const cg_cloud_index *ix, double radius, int max_nn, const double *view_point,
                                    double *out_normals, int32_t *out_nbr, int32_t *out_nbr_count) {
  if (!ix) return CG_EINVAL;
  CG_REQUIRE(ix->ctx, ix->S == 1, "cloud_normals: the index holds several sets; use cg_cloud_normals_many_dev");
  return cloud_normals(ix, "cloud_normals", radius, max_nn, view_point, out_normals, out_nbr, out_nbr_count);
}

extern "C" int cg_cloud_normals_many_dev(const cg_cloud_index *ix, double radius, int max_nn, const double *view_point,
                                         double *out_normals, int32_t *out_nbr, int32_t *out_nbr_count) {
  if (!ix) return CG_EINVAL;
  return cloud_normals(ix, "cloud_normals_many", radius, max_nn, view_point, out_normals, out_nbr, out_nbr_count);
}
