// cg_meanshift.cu -- sklearn's MeanShift(bandwidth, seeds=None, bin_seeding=False, cluster_all=True) on the device:
// the clustering of the segmentation's shifted points (predicter.py:332).
//
// Every point of X seeds one flat-kernel ascent.  Per ascent step the neighbour set is every point with
//   d2 = (dx*dx + dy*dy) + dz*dz <= bw*bw      float64, no FMA (the kd-tree's rule, cg_cloud_index.cuh::dist2)
// found through a cg_cloud_index over X (cell = bw scans at most 4 x 4 x 4 cells).  The new mean is summed in int64
// fixed point, so it does not depend on summation order, lane split or scheduling:
//   q(p) = llrint((p - origin) * 2^(41-E)),  E = the smallest integer with 2^E >= max(p - origin) + bw
//   m    = dtype((double)(sum q) * 2^(E-41) / n + origin)       dtype = X's own (float32 or float64)
// Every q is below 2^41, so the sums stay below 2^62 for P <= 2^21 points.  The ascent stops on an empty set, when
// sqrt((dx*dx + dy*dy) + dz*dz) <= 1e-3 bw for the step (dx = m - old in X's dtype, widened), or after max_iter steps,
// as sklearn's _mean_shift_single_seed does.
//
// The modes then follow sklearn's post-processing exactly:
//   1. seeds with a non-empty set are collapsed by centre value (-0.0 == +0.0): the centre of the lowest seed, the
//      count of the highest (a Python dict keeps the first key and the last value);
//   2. they are ordered by (count, x, y, z) descending;
//   3. greedy suppression in that order: a centre still unique removes every later centre with d2 <= bw*bw.
// Steps 1-2 are stable radix sorts (z, y, x descending, then count), so ties are decided by seed index and the order
// is a function of the values alone.  Step 3 is sequential by definition; one warp walks the sorted list and finds
// each kept centre's neighbours through a grid of the modes (the same cells as the index over X), so its cost grows
// with the number of modes times their local density, not with its square.
//
// Over a many-set index (cg_meanshift_many_dev) every set is clustered as cg_meanshift_dev clusters it alone: the
// fixed point takes the set's own origin and E, an ascent searches its own set's cells only, the collapse and the
// (count, x, y, z) order take the set as the most significant key, and the suppression runs one warp per set.  The
// centres come out set-major.  The 2^21-point limit is per set, as the int64 sums are.
#include <algorithm>
#include <cmath>
#include <cub/cub.cuh>
#include "cg_cloud_index.cuh"

namespace {

constexpr int MS_WARPS = 8;          // ascent: warps (seeds) per CTA
constexpr int MS_MAX_POINTS = 1 << 21;
constexpr int QBITS = 41;            // fixed-point bits below 2^E

__device__ __forceinline__ float narrow(double x, float) { return __double2float_rn(x); }
__device__ __forceinline__ double narrow(double x, double) { return x; }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }

// ascending uint64 order == ascending value order, with -0.0 and +0.0 on one key (never 0 for a finite value)
__device__ __forceinline__ uint64_t order_key(double x) {
  const uint64_t b = (uint64_t)__double_as_longlong(x == 0.0 ? 0.0 : x);
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}

// set_scale (many sets; null for one): (S,2) each set's scale and unscale
__global__ void quantise_kernel(IndexView V, int P, double scale, const double *__restrict__ set_scale,
                                long long *__restrict__ q) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const double *__restrict__ spts = V.spts;
  double ox = V.ox, oy = V.oy, oz = V.oz;
  if (set_scale) {                                    // sorted points are set-major, at the same offsets as X's
    const int t = set_of(V.poff, V.S, i);
    ox = V.sets[t].o[0]; oy = V.sets[t].o[1]; oz = V.sets[t].o[2];
    scale = set_scale[2 * t];
  }
  q[3 * (size_t)i] = __double2ll_rn(__dmul_rn(__dsub_rn(spts[3 * (size_t)i], ox), scale));
  q[3 * (size_t)i + 1] = __double2ll_rn(__dmul_rn(__dsub_rn(spts[3 * (size_t)i + 1], oy), scale));
  q[3 * (size_t)i + 2] = __double2ll_rn(__dmul_rn(__dsub_rn(spts[3 * (size_t)i + 2], oz), scale));
}

// one warp per seed: lanes split each column's run of candidates, the int64 sums and the count are warp-reduced
template <typename T>
__global__ void __launch_bounds__(MS_WARPS * 32) ascent_kernel(IndexView V0, const long long *__restrict__ q,
                                                               const T *__restrict__ X, int P, double bw, double bw2,
                                                               double stop, double unscale,
                                                               const double *__restrict__ set_scale, int max_iter,
                                                               T *__restrict__ out_c, int32_t *__restrict__ out_n,
                                                               int32_t *__restrict__ out_it) {
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x * MS_WARPS + (threadIdx.x >> 5);
  if (s >= P) return;   // the whole warp leaves together
  // many sets: seed s searches its own set t with that set's fixed point.  The warp's row is kept in shared memory and
  // read where it is used, so the set's origin and range hold no registers across the ascent.
  __shared__ CloudSet rows[MS_WARPS];
  __shared__ double unscales[MS_WARPS];
  const int wi = threadIdx.x >> 5;
  int t = 0;
  if (set_scale) {
    t = set_of(V0.poff, V0.S, s);
    if (lane == 0) {
      rows[wi] = V0.sets[t];
      unscales[wi] = set_scale[2 * t + 1];
    }
    __syncwarp();
  }
  const volatile CloudSet &row = rows[wi];
  T m[3] = {X[3 * (size_t)s], X[3 * (size_t)s + 1], X[3 * (size_t)s + 2]};
  int it = 0, n = 0;
  for (;;) {
    const double qx = (double)m[0], qy = (double)m[1], qz = (double)m[2];
    long long sum[3] = {0, 0, 0};
    int c = 0;
    IndexView V = V0;
    if (set_scale) V.prefix = (uint64_t)t << (3 * V0.bits);
    const Columns C(V, set_scale ? &row : nullptr, qx, qy, qz, bw);
    if (C.any)
      for (int64_t cx = C.x0; cx <= C.x1; cx++)
        for (int64_t cy = C.y0; cy <= C.y1; cy++) {
          int b, e;
          C.run(V, cx, cy, b, e);
          for (int k = b + lane; k < e; k += 32) {
            const double d2 = dist2(qx, qy, qz, V.spts[3 * (size_t)k], V.spts[3 * (size_t)k + 1], V.spts[3 * (size_t)k + 2]);
            if (d2 <= bw2) {
              c++;
              sum[0] += q[3 * (size_t)k];
              sum[1] += q[3 * (size_t)k + 1];
              sum[2] += q[3 * (size_t)k + 2];
            }
          }
        }
    for (int w = 16; w; w >>= 1) {
      c += __shfl_xor_sync(0xffffffffu, c, w);
#pragma unroll
      for (int a = 0; a < 3; a++) sum[a] += __shfl_xor_sync(0xffffffffu, sum[a], w);
    }
    n = c;
    if (n == 0) break;                                  // nothing within bw: the seed keeps its mean, count 0
    const T old[3] = {m[0], m[1], m[2]};
    const double cn = (double)n;
    double o[3] = {V0.ox, V0.oy, V0.oz}, us = unscale;
    if (set_scale) {
      o[0] = row.o[0]; o[1] = row.o[1]; o[2] = row.o[2];
      us = unscales[wi];
    }
#pragma unroll
    for (int a = 0; a < 3; a++)
      m[a] = narrow(__dadd_rn(__ddiv_rn(__dmul_rn(__ll2double_rn(sum[a]), us), cn), o[a]), T());
    const double dx = (double)sub_rn(m[0], old[0]), dy = (double)sub_rn(m[1], old[1]), dz = (double)sub_rn(m[2], old[2]);
    const double step = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
    if (step <= stop || it == max_iter) break;
    it++;
  }
  if (lane == 0) {
    out_c[3 * (size_t)s] = m[0];
    out_c[3 * (size_t)s + 1] = m[1];
    out_c[3 * (size_t)s + 2] = m[2];
    out_n[s] = n;
    out_it[s] = it;
  }
}

// sort key of axis `a` for the seed at each position (position j of the previous pass's order, or j itself on the
// first pass); seeds with an empty set get the x key 0, below every finite value, so they sort last.  a = 3 (many
// sets, the last pass): S - 1 - the seed's set, so the descending sort puts set 0 first
template <typename T>
__global__ void seed_key_kernel(const T *__restrict__ c, const int32_t *__restrict__ n, int P, int a,
                                const int32_t *__restrict__ poff, int S, const int32_t *__restrict__ order,
                                uint64_t *__restrict__ key, int32_t *__restrict__ val) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  const int s = order ? order[j] : j;
  if (a == 3) key[j] = (uint64_t)(S - 1 - set_of(poff, S, s));
  else key[j] = (a == 0 && n[s] == 0) ? 0ull : order_key((double)c[3 * (size_t)s + a]);
  if (!order) val[j] = j;
}

template <typename T>
__device__ __forceinline__ bool same_centre(const T *c, int s, int t) {
  return order_key((double)c[3 * (size_t)s]) == order_key((double)c[3 * (size_t)t]) &&
         order_key((double)c[3 * (size_t)s + 1]) == order_key((double)c[3 * (size_t)t + 1]) &&
         order_key((double)c[3 * (size_t)s + 2]) == order_key((double)c[3 * (size_t)t + 2]);
}

// seeds s and t are in different sets (poff null: one set)
__device__ __forceinline__ bool other_set(const int32_t *poff, int S, int s, int t) {
  return poff && set_of(poff, S, s) != set_of(poff, S, t);
}

// head[j] = position j starts a group of equal centres (seeds in value order, empty ones last; many sets: set-major)
template <typename T>
__global__ void head_kernel(const T *__restrict__ c, const int32_t *__restrict__ n, int P, const int32_t *__restrict__ poff,
                            int S, const int32_t *__restrict__ order, int32_t *__restrict__ head) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  const int s = order[j];
  head[j] = n[s] > 0 && (j == 0 || !same_centre(c, s, order[j - 1]) || other_set(poff, S, s, order[j - 1])) ? 1 : 0;
}

// per group: its first (lowest) seed and the count of its last (highest) seed; the number of groups
template <typename T>
__global__ void group_kernel(const T *__restrict__ c, const int32_t *__restrict__ n, int P, const int32_t *__restrict__ poff,
                             int S, const int32_t *__restrict__ order, const int32_t *__restrict__ head,
                             const int32_t *__restrict__ gid, int32_t *__restrict__ gseed, int32_t *__restrict__ gcount,
                             int32_t *__restrict__ nmodes) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  if (j == P - 1) *nmodes = gid[j] + head[j];
  const int s = order[j];
  if (n[s] == 0) return;
  const int g = gid[j] + head[j] - 1;   // gid counts the heads before j
  if (head[j]) gseed[g] = s;
  if (j == P - 1 || n[order[j + 1]] == 0 || !same_centre(c, s, order[j + 1]) || other_set(poff, S, s, order[j + 1]))
    gcount[g] = n[s];
}

// count sort key: groups are already in descending (x, y, z) (many sets: set-major); a stable ascending sort on
// set << 32 | P - count puts them in descending (count, x, y, z) per set; slots past the last group sort after every
// group.  One set: the set field is 0.
__global__ void count_key_kernel(const int32_t *__restrict__ gcount, const int32_t *__restrict__ gseed,
                                 const int32_t *__restrict__ nmodes, int P, const int32_t *__restrict__ poff, int S,
                                 uint64_t *__restrict__ key, int32_t *__restrict__ val) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= P) return;
  const uint64_t set = g < *nmodes ? (poff ? (uint64_t)set_of(poff, S, gseed[g]) : 0ull) : (uint64_t)(S - 1);
  key[g] = (set << 32) | (g < *nmodes ? (uint64_t)(P - gcount[g]) : (uint64_t)P + 1);
  val[g] = g;
}

// the modes in rank order (float64 copies) and their cells in the index's grid, clamped to its range so a centre
// rounded just outside the points' bounding box is still found; slots past the last mode get the largest key
template <typename T>
__global__ void rank_kernel(IndexView V0, const T *__restrict__ c, const int32_t *__restrict__ gseed,
                            const int32_t *__restrict__ rank_group, const int32_t *__restrict__ nmodes, int P,
                            double *__restrict__ rc, int32_t *__restrict__ rseed, uint64_t *__restrict__ key,
                            int32_t *__restrict__ val, int32_t *__restrict__ supp) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= P) return;
  val[r] = r;
  supp[r] = 0;
  if (r >= *nmodes) {
    key[r] = ~0ull;
    return;
  }
  const int s = gseed[rank_group[r]];
  rseed[r] = s;
  const IndexView V = V0.S > 1 ? V0.in_set(set_of(V0.poff, V0.S, s)) : V0;   // the seed's set: its grid and prefix
  const double o[3] = {V.ox, V.oy, V.oz};
  const int64_t mc[3] = {V.mx, V.my, V.mz};
  int64_t cc[3];
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const double x = (double)c[3 * (size_t)s + a];
    rc[3 * (size_t)r + a] = x;
    const double f = floor(__ddiv_rn(__dsub_rn(x, o[a]), V.cell));
    cc[a] = f < 0.0 ? 0 : (f > (double)mc[a] ? mc[a] : (int64_t)f);
  }
  key[r] = V.prefix | pack(cc[0], cc[1], cc[2], V.bits);
}

// the first rank in [0, M) whose mode is in set t or later (ranks are set-major)
__device__ int first_rank_of_set(const int32_t *rseed, const int32_t *poff, int S, int M, int t) {
  int lo = 0, hi = M;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (set_of(poff, S, rseed[m]) < t) lo = m + 1; else hi = m;
  }
  return lo;
}

// sequential greedy suppression (one warp per set, block t for set t): mode r, if still unique, marks every later mode
// within bw; the modes of each column of r's cell range are the run [lower_bound, upper_bound) of the sorted mode keys,
// and the set's prefix keeps that run in set t
__global__ void __launch_bounds__(32) suppress_kernel(IndexView V0, const double *__restrict__ rc,
                                                      const uint64_t *__restrict__ mkey, const int32_t *__restrict__ mrank,
                                                      const int32_t *__restrict__ rseed, const int32_t *__restrict__ nmodes,
                                                      double bw, double bw2, int32_t *supp_) {
  volatile int32_t *supp = supp_;
  const int lane = threadIdx.x;
  const int M = *nmodes;
  const int t = blockIdx.x;
  const IndexView V = V0.S > 1 ? V0.in_set(t) : V0;
  const int r0 = V0.S > 1 ? first_rank_of_set(rseed, V0.poff, V0.S, M, t) : 0;
  const int r1 = V0.S > 1 ? first_rank_of_set(rseed, V0.poff, V0.S, M, t + 1) : M;
  for (int r = r0; r < r1; r++) {
    if (supp[r]) continue;   // uniform across the warp: every lane read the same flag after the last __syncwarp
    const double qx = rc[3 * (size_t)r], qy = rc[3 * (size_t)r + 1], qz = rc[3 * (size_t)r + 2];
    const Columns C(V, qx, qy, qz, bw);
    if (C.any) {
      const int ny = (int)(C.y1 - C.y0 + 1);
      const int ncol = (int)(C.x1 - C.x0 + 1) * ny;
      for (int col = lane; col < ncol; col += 32) {
        const int64_t cx = C.x0 + col / ny, cy = C.y0 + col % ny;
        const int a = lower_bound(mkey, 0, M, V.prefix | pack(cx, cy, C.z0, V.bits));
        const int b = upper_bound(mkey, a, M, V.prefix | pack(cx, cy, C.z1, V.bits));
        for (int k = a; k < b; k++) {
          const int j = mrank[k];
          if (j > r && dist2(qx, qy, qz, rc[3 * (size_t)j], rc[3 * (size_t)j + 1], rc[3 * (size_t)j + 2]) <= bw2)
            supp[j] = 1;
        }
      }
    }
    __syncwarp();
  }
}

__global__ void kept_kernel(const int32_t *__restrict__ supp, const int32_t *__restrict__ nmodes, int P,
                            int32_t *__restrict__ kept) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < P) kept[r] = r < *nmodes && !supp[r] ? 1 : 0;
}

// kept modes in rank order, each the value of its lowest seed (so -0.0 survives as the first seed had it).  out_n
// (null: not written) = how many; out_off (many sets; null: not written) = (S+1) each set's first kept mode, out_off[S]
// = how many
template <typename T>
__global__ void emit_kernel(const T *__restrict__ c, const int32_t *__restrict__ rseed, const int32_t *__restrict__ kept,
                            const int32_t *__restrict__ pos, int P, const int32_t *__restrict__ nmodes,
                            const int32_t *__restrict__ poff, int S, T *__restrict__ out, int32_t *__restrict__ out_n,
                            int32_t *__restrict__ out_off) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= P) return;
  if (r == P - 1 && out_n) *out_n = pos[r] + kept[r];
  if (out_off) {
    const int M = *nmodes;
    if (r < M) {                  // the sets after the previous mode's, up to this mode's, start at this mode
      const int t = set_of(poff, S, rseed[r]), tp = r == 0 ? -1 : set_of(poff, S, rseed[r - 1]);
      for (int u = tp + 1; u <= t; u++) out_off[u] = pos[r];
    }
    if (r == P - 1) {             // the sets after the last mode's, and the end
      const int tl = M == 0 ? -1 : set_of(poff, S, rseed[M - 1]);
      for (int u = tl + 1; u <= S; u++) out_off[u] = pos[r] + kept[r];
    }
  }
  if (!kept[r]) return;
  const int s = rseed[r];
  const size_t k = (size_t)pos[r];
  out[3 * k] = c[3 * (size_t)s];
  out[3 * k + 1] = c[3 * (size_t)s + 1];
  out[3 * k + 2] = c[3 * (size_t)s + 2];
}

unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

int bit_length(int v) {
  int n = 0;
  while (v >> n) n++;
  return n;
}

// The clustering behind cg_meanshift_dev (out_k: the centre count) and cg_meanshift_many_dev (out_off: the centre
// offsets per set).  A one-set index passes no set tables, so its kernels take the one-set branches.
template <typename T>
int meanshift(const cg_cloud_index *ix, const T *X, double bw, int max_iter, T *seed_c, int32_t *seed_n,
              int32_t *seed_it, T *out_c, int32_t *out_k, int32_t *out_off) {
  cg_ctx *ctx = ix->ctx;
  const int P = ix->P, S = ix->S;
  const bool many = S > 1;
  const IndexView V = view_of(ix);
  // per set, E: the smallest integer with 2^E >= max(p - origin) + bw (p - origin is monotone in p, so the max is
  // at hi)
  std::vector<double> sc(2 * (size_t)S);
  for (int t = 0; t < S; t++) {
    double umax = 0.0;
    for (int a = 0; a < 3; a++) umax = std::max(umax, ix->set_hi[3 * (size_t)t + a] - ix->sets[t].o[a]);
    int e2 = 0;
    const double fr = std::frexp(umax + bw, &e2);
    const int E = fr == 0.5 ? e2 - 1 : e2;
    sc[2 * (size_t)t] = std::ldexp(1.0, QBITS - E);
    sc[2 * (size_t)t + 1] = std::ldexp(1.0, E - QBITS);
  }
  const double scale = sc[0], unscale = sc[1];

  size_t sort_tmp = 0, scan_tmp = 0;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (uint64_t *)nullptr, (uint64_t *)nullptr, (int32_t *)nullptr,
                                               (int32_t *)nullptr, P, 0, 64, ctx->stream));
  CG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (int32_t *)nullptr, (int32_t *)nullptr, P, ctx->stream));
  const size_t tmp = std::max(sort_tmp, scan_tmp);
  const size_t Pz = (size_t)P;
  long long *q; double *rc; uint64_t *kA, *kB; void *dtmp;
  int32_t *vA, *vB, *head, *gid, *gseed, *gcount, *rseed, *supp, *kept, *nmodes;
  double *d_sc;
  const int rc_ = cg_ws_carve(ctx, [&](cg_arena &ar) {
    q = ar.take<long long>(3 * Pz);
    rc = ar.take<double>(3 * Pz);
    kA = ar.take<uint64_t>(Pz); kB = ar.take<uint64_t>(Pz);
    vA = ar.take<int32_t>(Pz); vB = ar.take<int32_t>(Pz); head = ar.take<int32_t>(Pz);
    gid = ar.take<int32_t>(Pz); gseed = ar.take<int32_t>(Pz); gcount = ar.take<int32_t>(Pz);
    rseed = ar.take<int32_t>(Pz); supp = ar.take<int32_t>(Pz); kept = ar.take<int32_t>(Pz);
    nmodes = ar.take<int32_t>(1);
    d_sc = ar.take<double>(many ? sc.size() : 0);
    dtmp = ar.take<char>(tmp);
  });
  if (rc_ != CG_OK) return rc_;
  cudaStream_t st = ctx->stream;
  const unsigned g256 = blocks(P, 256);
  // the set scales, from pageable memory: staged at once, no synchronisation
  if (many) CG_CUDA(ctx, cudaMemcpyAsync(d_sc, sc.data(), sizeof(double) * sc.size(), cudaMemcpyHostToDevice, st));
  const double *set_scale = many ? d_sc : nullptr;
  const int32_t *poff = many ? ix->d_poff : nullptr;

  quantise_kernel<<<g256, 256, 0, st>>>(V, P, scale, set_scale, q);
  CG_LAUNCH_CHECK(ctx);
  ascent_kernel<T><<<blocks(P, MS_WARPS), MS_WARPS * 32, 0, st>>>(V, q, X, P, bw, bw * bw, 1e-3 * bw, unscale, set_scale,
                                                                  max_iter, seed_c, seed_n, seed_it);
  CG_LAUNCH_CHECK(ctx);

  // seeds in descending (x, y, z), equal centres by ascending seed index, empty ones last: z, y, x passes, then (many
  // sets) a set pass that makes the order set-major
  size_t tb;
  const int32_t *order = nullptr;
  int32_t *vin = vA, *vout = vB;
  for (int a = 2; a >= (many ? -1 : 0); a--) {
    const int axis = a < 0 ? 3 : a;
    seed_key_kernel<T><<<g256, 256, 0, st>>>(seed_c, seed_n, P, axis, poff, S, order, kA, vin);
    CG_LAUNCH_CHECK(ctx);
    tb = tmp;
    CG_CUDA(ctx, cub::DeviceRadixSort::SortPairsDescending(dtmp, tb, kA, kB, vin, vout, P, 0,
                                                           axis == 3 ? bit_length(S - 1) : 64, st));
    order = vout;
    std::swap(vin, vout);
  }
  // order (= vin after the swap) holds the seeds in value order
  head_kernel<T><<<g256, 256, 0, st>>>(seed_c, seed_n, P, poff, S, order, head);
  CG_LAUNCH_CHECK(ctx);
  tb = tmp;
  CG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(dtmp, tb, head, gid, P, st));
  group_kernel<T><<<g256, 256, 0, st>>>(seed_c, seed_n, P, poff, S, order, head, gid, gseed, gcount, nmodes);
  CG_LAUNCH_CHECK(ctx);
  int32_t *ord_free = vout;   // the buffer not holding `order`
  count_key_kernel<<<g256, 256, 0, st>>>(gcount, gseed, nmodes, P, poff, S, kA, ord_free);
  CG_LAUNCH_CHECK(ctx);
  int32_t *rank_group = head;   // head is consumed: reuse it for the rank -> group table
  tb = tmp;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(dtmp, tb, kA, kB, ord_free, rank_group, P, 0,
                                               many ? 32 + bit_length(S - 1) : 23, st));
  rank_kernel<T><<<g256, 256, 0, st>>>(V, seed_c, gseed, rank_group, nmodes, P, rc, rseed, kA, vA, supp);
  CG_LAUNCH_CHECK(ctx);
  tb = tmp;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(dtmp, tb, kA, kB, vA, vB, P, 0, 64, st));
  suppress_kernel<<<S, 32, 0, st>>>(V, rc, kB, vB, rseed, nmodes, bw, bw * bw, supp);
  CG_LAUNCH_CHECK(ctx);
  kept_kernel<<<g256, 256, 0, st>>>(supp, nmodes, P, kept);
  CG_LAUNCH_CHECK(ctx);
  tb = tmp;
  CG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(dtmp, tb, kept, gid, P, st));
  emit_kernel<T><<<g256, 256, 0, st>>>(seed_c, rseed, kept, gid, P, nmodes, poff, S, out_c, out_k, out_off);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

}  // namespace

namespace {

int meanshift_checked(const cg_cloud_index *ix, const char *who, const void *X, int x_is_f64, double bandwidth,
                      int max_iter, void *seed_c, int32_t *seed_n, int32_t *seed_it, void *out_c, int32_t *out_k,
                      int32_t *out_off) {
  cg_ctx *ctx = ix->ctx;
  const std::string w = who;
  CG_REQUIRE(ctx, X && seed_c && seed_n && seed_it && out_c && (out_k || out_off), w + ": null argument");
  CG_REQUIRE(ctx, bandwidth > 0.0 && std::isfinite(bandwidth), w + ": bandwidth must be positive and finite");
  CG_REQUIRE(ctx, ix->cell == bandwidth, w + ": the index must be built with cell = bandwidth");
  CG_REQUIRE(ctx, max_iter >= 0, w + ": max_iter must be >= 0");
  for (int t = 0; t < ix->S; t++)
    CG_REQUIRE(ctx, ix->poff[t + 1] - ix->poff[t] <= MS_MAX_POINTS,
               w + ": at most 2^21 points" + (ix->S > 1 ? " per set" : "") + " (the int64 sums must stay below 2^62)");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  if (x_is_f64)
    return meanshift<double>(ix, (const double *)X, bandwidth, max_iter, (double *)seed_c, seed_n, seed_it,
                             (double *)out_c, out_k, out_off);
  return meanshift<float>(ix, (const float *)X, bandwidth, max_iter, (float *)seed_c, seed_n, seed_it, (float *)out_c,
                          out_k, out_off);
}

}  // namespace

extern "C" int cg_meanshift_dev(const cg_cloud_index *ix, const void *X, int x_is_f64, double bandwidth, int max_iter,
                                void *out_seed_centres, int32_t *out_seed_counts, int32_t *out_seed_iters,
                                void *out_centres, int32_t *out_n_centres) {
  if (!ix) return CG_EINVAL;
  CG_REQUIRE(ix->ctx, ix->S == 1, "meanshift: the index holds several sets; use cg_meanshift_many_dev");
  CG_REQUIRE(ix->ctx, out_n_centres, "meanshift: null argument");
  return meanshift_checked(ix, "meanshift", X, x_is_f64, bandwidth, max_iter, out_seed_centres, out_seed_counts,
                           out_seed_iters, out_centres, out_n_centres, nullptr);
}

extern "C" int cg_meanshift_many_dev(const cg_cloud_index *ix, const void *X, int x_is_f64, double bandwidth, int max_iter,
                                     void *out_seed_centres, int32_t *out_seed_counts, int32_t *out_seed_iters,
                                     void *out_centres, int32_t *out_centre_offsets) {
  if (!ix) return CG_EINVAL;
  CG_REQUIRE(ix->ctx, out_centre_offsets, "meanshift_many: null argument");
  return meanshift_checked(ix, "meanshift_many", X, x_is_f64, bandwidth, max_iter, out_seed_centres, out_seed_counts,
                           out_seed_iters, out_centres, nullptr, out_centre_offsets);
}
