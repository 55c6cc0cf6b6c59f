// cg_pick.cu -- the glue of the per-pick call (catgrasp_b200/pick.py): the segment table of the segmentation's labels
// (run_grasp_simulation.py:217-240, :253-259, :273) and the ranking of an object's scored grasps (:311-328).
//
// Both entries take device pointers, run on the context's stream and never synchronise.  Every result the host needs
// for a decision (how many segments are kept, in which order) is a device word the caller reads back.
//
// Segment table.  Labels are dense in [0, L).  Per label: the point count (int32 atomics), the exact per-axis min and
// max (the coordinate widened to float64, which is exact, and mapped to an order-preserving uint64 for atomicMin /
// atomicMax), then the inlier test evaluated in the cloud's dtype the way numpy evaluates :223-234.  Kept labels are
// ordered by one radix sort of (count << 32 | label) descending: count descending, ties in descending label order, as
// reversed(sorted(items, key=count)) gives them.  The kept points are grouped by one stable radix sort of (rank in
// that order, point index), so each segment's indices come out ascending, as `scene_seg == seg_id` selects them.
//
// Several frames (cg_segment_table_many_dev) run as one table of L = sum L_b labels: frame b's labels are the rows
// [loff[b], loff[b+1]) and its points [poff[b], poff[b+1]).  A kernel finds a point's or a row's frame by a binary
// search of those offsets (null for one frame) and shifts frame-local labels to rows and back.  The label sort is
// segmented by frame; the point sort key is frame b's offset slot (loff[b] + b) plus the rank, so frame b's points
// stay in its own range [poff[b], poff[b+1]); the offsets are one scan by frame over L + B slots, each frame's first
// slot 0.  Every output block is what the one-frame table of that frame gives, bit for bit.
//
// Ranking.  p_G = (pred * arange(C)).sum() / denom, denom = len(cfg_grasp['classes']) - 1, with numpy's pairwise
// summation order (8 <= C <= 128: eight accumulators over the first C - C % 8 terms, combined
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the rest in sequence; C < 8: left to right).  The products are exact in float64.  The permutation is Python's stable
// sorted(key=-p_T_G): one stable radix sort of an order-preserving key in which -0.0 and +0.0 are one value.
#include <cub/cub.cuh>
#include "cg_common.cuh"

namespace {

constexpr int ST_THREADS = 256;
constexpr int ST_SMEM_L = 512;   // labels held per CTA in shared memory; a larger table takes global atomics

unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

// order-preserving map of a double onto uint64 (NaN excluded): a < b  <=>  key(a) < key(b)
__device__ __forceinline__ uint64_t ord_key(double v) {
  const uint64_t b = (uint64_t)__double_as_longlong(v);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double ord_val(uint64_t k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// the b with off[b] <= i < off[b + 1] (off ascending from 0, ranges may be empty, 0 <= i < off[B])
__device__ __forceinline__ int frame_of(const int32_t *__restrict__ off, int B, int64_t i) {
  int lo = 0, hi = B;
  while (hi - lo > 1) {
    const int m = (lo + hi) >> 1;
    if (off[m] <= i) lo = m; else hi = m;
  }
  return lo;
}

__device__ __forceinline__ int64_t load_label(const void *labels, int is_i64, int64_t i) {
  return is_i64 ? static_cast<const int64_t *>(labels)[i] : (int64_t) static_cast<const int32_t *>(labels)[i];
}
__device__ __forceinline__ double load_x(const void *x, int is_f64, int64_t i) {
  return is_f64 ? static_cast<const double *>(x)[i] : (double)static_cast<const float *>(x)[i];
}

__global__ void seg_init_kernel(int L, int32_t *__restrict__ count, uint64_t *__restrict__ kmin,
                                uint64_t *__restrict__ kmax) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  count[l] = 0;
  for (int a = 0; a < 3; a++) {
    kmin[3 * (size_t)l + a] = ~0ull;
    kmax[3 * (size_t)l + a] = 0ull;
  }
}

// count, min and max per label; labels outside [0, L) are skipped.  SMEM: per-CTA privatised tables (L <= ST_SMEM_L).
// Several frames (poff non-null): point i's frame-local label l is row loff[b] + l, skipped outside [0, L_b)
template <bool SMEM>
__global__ void __launch_bounds__(ST_THREADS) seg_stats_kernel(const void *__restrict__ labels, int lab_i64,
                                                               const void *__restrict__ x, int x_f64, int M, int L,
                                                               const int32_t *__restrict__ poff,
                                                               const int32_t *__restrict__ loff, int B,
                                                               int32_t *__restrict__ count,
                                                               uint64_t *__restrict__ kmin,
                                                               uint64_t *__restrict__ kmax) {
  __shared__ int32_t s_cnt[SMEM ? ST_SMEM_L : 1];
  __shared__ uint64_t s_min[SMEM ? 3 * ST_SMEM_L : 1], s_max[SMEM ? 3 * ST_SMEM_L : 1];
  if (SMEM) {
    for (int l = threadIdx.x; l < L; l += blockDim.x) {
      s_cnt[l] = 0;
      for (int a = 0; a < 3; a++) {
        s_min[3 * l + a] = ~0ull;
        s_max[3 * l + a] = 0ull;
      }
    }
    __syncthreads();
  }
  int32_t *cnt = SMEM ? s_cnt : count;
  uint64_t *mn = SMEM ? s_min : kmin, *mx = SMEM ? s_max : kmax;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t l = load_label(labels, lab_i64, i);
    if (poff) {
      const int b = frame_of(poff, B, i);
      if (l < 0 || l >= loff[b + 1] - loff[b]) continue;
      l += loff[b];
    } else if (l < 0 || l >= L) {
      continue;
    }
    atomicAdd(&cnt[l], 1);
    for (int a = 0; a < 3; a++) {
      const unsigned long long k = ord_key(load_x(x, x_f64, 3 * i + a));
      atomicMin((unsigned long long *)&mn[3 * l + a], k);
      atomicMax((unsigned long long *)&mx[3 * l + a], k);
    }
  }
  if (SMEM) {
    __syncthreads();
    for (int l = threadIdx.x; l < L; l += blockDim.x) {
      if (s_cnt[l] == 0) continue;
      atomicAdd(&count[l], s_cnt[l]);
      for (int a = 0; a < 3; a++) {
        atomicMin((unsigned long long *)&kmin[3 * l + a], (unsigned long long)s_min[3 * l + a]);
        atomicMax((unsigned long long *)&kmax[3 * l + a], (unsigned long long)s_max[3 * l + a]);
      }
    }
  }
}

// run_grasp_simulation.py:223-234 in the cloud's dtype: ext = max - min, q = ext / 0.001, prod = (q0 * q1) * q2, all
// rounded in that dtype; density = n / prod in float64 (int64 / float32 promotes to float64).  A zero extent gives
// prod = 0 and density = inf: an inlier, as in numpy.
__global__ void seg_decide_kernel(int L, int x_f64, const int32_t *__restrict__ count,
                                  const uint64_t *__restrict__ kmin, const uint64_t *__restrict__ kmax,
                                  double *__restrict__ out_min, double *__restrict__ out_max,
                                  int32_t *__restrict__ out_count, uint8_t *__restrict__ out_inlier,
                                  uint64_t *__restrict__ sort_key) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  const int n = count[l];
  double lo[3], hi[3];
  for (int a = 0; a < 3; a++) {
    lo[a] = n ? ord_val(kmin[3 * (size_t)l + a]) : 0.0;
    hi[a] = n ? ord_val(kmax[3 * (size_t)l + a]) : 0.0;
    out_min[3 * (size_t)l + a] = lo[a];
    out_max[3 * (size_t)l + a] = hi[a];
  }
  bool inlier = n >= 500;
  if (inlier) {
    double prod;
    if (x_f64) {
      double q[3];
      for (int a = 0; a < 3; a++) q[a] = __ddiv_rn(__dsub_rn(hi[a], lo[a]), 0.001);
      prod = __dmul_rn(__dmul_rn(q[0], q[1]), q[2]);
    } else {
      float q[3];
      for (int a = 0; a < 3; a++) q[a] = __fdiv_rn(__fsub_rn((float)hi[a], (float)lo[a]), 0.001f);
      prod = (double)__fmul_rn(__fmul_rn(q[0], q[1]), q[2]);
    }
    const double density = __ddiv_rn((double)n, prod);
    inlier = !(density < 0.01);
  }
  out_count[l] = n;
  out_inlier[l] = inlier;
  sort_key[l] = inlier ? ((uint64_t)n << 32) | (uint32_t)l : 0ull;   // kept keys are > 0: n >= 500
}

// the sorted keys -> the kept labels in order (frame-local), their rank per row, the kept count per frame, and the
// offset slots: frame b's slot loff[b] + b is 0 and slot loff[b] + b + 1 + k the k-th kept segment's count (0 past
// the kept ones).  Several frames (loff non-null): each slot's frame also goes to slot_frame, the scan's key
__global__ void seg_order_kernel(int L, const uint64_t *__restrict__ sorted_key, const uint8_t *__restrict__ inlier,
                                 const int32_t *__restrict__ loff, int B, int32_t *__restrict__ order,
                                 int32_t *__restrict__ rank, int32_t *__restrict__ n_kept, int32_t *__restrict__ seg_len,
                                 int32_t *__restrict__ slot_frame) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= L) return;
  const int b = loff ? frame_of(loff, B, k) : 0;
  const int base = loff ? loff[b] : 0, Lb = loff ? loff[b + 1] - base : L, kk = k - base;
  int32_t *len = seg_len + base + b;
  const uint64_t key = sorted_key[k];
  if (key) {
    const int l = (int)(uint32_t)key;
    order[k] = l - base;
    rank[l] = kk;
    len[kk + 1] = (int32_t)(key >> 32);
    if (kk + 1 == Lb || sorted_key[k + 1] == 0ull) n_kept[b] = kk + 1;
  } else {
    order[k] = -1;
    len[kk + 1] = 0;
    if (kk == 0) n_kept[b] = 0;
  }
  if (kk == 0) len[0] = 0;
  if (slot_frame) {
    slot_frame[base + b + kk + 1] = b;
    if (kk == 0) slot_frame[base + b] = b;
  }
  if (!inlier[k]) rank[k] = -1;
}

// scene_seg with outliers set to -1 (:240), and the compaction key of every point: its segment's rank, or L past the
// last segment.  Several frames (poff non-null): the rank plus frame b's offset slot loff[b] + b, L_b past its last
// segment, and the point's index within its frame
__global__ void seg_points_kernel(const void *__restrict__ labels, int lab_i64, int M, int L,
                                  const int32_t *__restrict__ poff, const int32_t *__restrict__ loff, int B,
                                  const int32_t *__restrict__ rank, void *__restrict__ out_labels,
                                  uint32_t *__restrict__ pkey, int32_t *__restrict__ pval) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const int b = poff ? frame_of(poff, B, i) : 0;
  const int base = poff ? loff[b] : 0, Lb = poff ? loff[b + 1] - base : L;
  const int64_t l = load_label(labels, lab_i64, i);
  const int r = (l >= 0 && l < Lb) ? rank[base + l] : -1;
  const int64_t out = r >= 0 ? l : -1;
  if (lab_i64)
    static_cast<int64_t *>(out_labels)[i] = out;
  else
    static_cast<int32_t *>(out_labels)[i] = (int32_t)out;
  pkey[i] = (uint32_t)(base + b) + (r >= 0 ? (uint32_t)r : (uint32_t)Lb);
  pval[i] = poff ? i - poff[b] : i;
}

// numpy's pairwise_sum (loops_utils.h) for n <= 128 terms
__device__ __forceinline__ double numpy_pairwise_sum(const float *__restrict__ row, int n) {
  if (n < 8) {
    double res = 0.0;
    for (int c = 0; c < n; c++) res = __dadd_rn(res, __dmul_rn((double)row[c], (double)c));
    return res;
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; j++) r[j] = __dmul_rn((double)row[j], (double)j);
  int i = 8;
  for (; i < n - (n % 8); i += 8) {
#pragma unroll
    for (int j = 0; j < 8; j++) r[j] = __dadd_rn(r[j], __dmul_rn((double)row[i + j], (double)(i + j)));
  }
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                         __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; i++) res = __dadd_rn(res, __dmul_rn((double)row[i], (double)i));
  return res;
}

__global__ void rank_score_kernel(const float *__restrict__ probs, int G, int C, int denom,
                                  const double *__restrict__ p_t_given_g,
                                  double *__restrict__ p_g, double *__restrict__ p_tg, uint64_t *__restrict__ key,
                                  int32_t *__restrict__ idx) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const double pg = __ddiv_rn(numpy_pairwise_sum(probs + (size_t)g * C, C), (double)denom);
  const double ptg = __dmul_rn(p_t_given_g[g], pg);
  p_g[g] = pg;
  p_tg[g] = ptg;
  // ascending in -p_T_G: the complement of the order key of p_T_G, with -0.0 folded onto +0.0
  key[g] = ~ord_key(ptg == 0.0 ? 0.0 : ptg);
  idx[g] = g;
}

}  // namespace

namespace {

// The one table behind cg_segment_table_dev (B = 1, poff = {0, M}, loff = {0, L}) and cg_segment_table_many_dev.
// poff and loff are host arrays of B + 1; the frame tables reach the device only when B > 1.
int segment_table(cg_ctx *ctx, const void *labels, int labels_is_i64, const void *x, int x_is_f64, int B,
                  const int32_t *poff, const int32_t *loff, void *out_labels, int32_t *out_count, double *out_min,
                  double *out_max, uint8_t *out_inlier, int32_t *out_order, int32_t *out_n_kept, int32_t *out_offsets,
                  int32_t *out_index) {
  const int M = poff[B], L = loff[B];
  const bool many = B > 1;
  CG_REQUIRE(ctx, out_count && out_min && out_max && out_inlier && out_order && out_n_kept && out_offsets,
             "segment_table: null argument");
  CG_REQUIRE(ctx, M == 0 || (labels && x && out_labels && out_index), "segment_table: null argument");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t Lz = (size_t)L, Mz = (size_t)M, Bz = (size_t)B, slots = Lz + Bz;
  size_t tmp_l = 0, tmp_m = 0, tmp_s = 0;
  int lbits = 1;
  while ((1ll << lbits) <= (int64_t)(L + B - 1)) lbits++;   // point keys are offset slots in [0, L + B)
  if (many)
    CG_CUDA(ctx, cub::DeviceSegmentedRadixSort::SortKeysDescending(nullptr, tmp_l, (uint64_t *)nullptr, (uint64_t *)nullptr,
                                                                   L, B, (int32_t *)nullptr, (int32_t *)nullptr, 0, 64, st));
  else
    CG_CUDA(ctx, cub::DeviceRadixSort::SortKeysDescending(nullptr, tmp_l, (uint64_t *)nullptr, (uint64_t *)nullptr, L,
                                                          0, 64, st));
  if (M > 0)
    CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, tmp_m, (uint32_t *)nullptr, (uint32_t *)nullptr,
                                                 (int32_t *)nullptr, (int32_t *)nullptr, M, 0, lbits, st));
  if (many)
    CG_CUDA(ctx, cub::DeviceScan::InclusiveSumByKey(nullptr, tmp_s, (int32_t *)nullptr, (int32_t *)nullptr,
                                                    (int32_t *)nullptr, (int)slots, ::cuda::std::equal_to<>(), st));
  else
    CG_CUDA(ctx, cub::DeviceScan::InclusiveSum(nullptr, tmp_s, (int32_t *)nullptr, (int32_t *)nullptr, (int)slots, st));
  const size_t tmp_bytes = std::max(tmp_l, std::max(tmp_m, tmp_s));
  int32_t *cnt, *rank, *seg_len, *slot_frame, *pval, *dpoff, *dloff;
  uint64_t *kmin, *kmax, *key, *key_sorted;
  uint32_t *pkey, *pkey_sorted;
  void *tmp;
  const int rc = cg_ws_carve(ctx, [&](cg_arena &ar) {
    cnt = ar.take<int32_t>(Lz); rank = ar.take<int32_t>(Lz); seg_len = ar.take<int32_t>(slots);
    slot_frame = ar.take<int32_t>(many ? slots : 0);
    dpoff = ar.take<int32_t>(many ? Bz + 1 : 0); dloff = ar.take<int32_t>(many ? Bz + 1 : 0);
    kmin = ar.take<uint64_t>(3 * Lz); kmax = ar.take<uint64_t>(3 * Lz);
    key = ar.take<uint64_t>(Lz); key_sorted = ar.take<uint64_t>(Lz);
    pkey = ar.take<uint32_t>(Mz); pkey_sorted = ar.take<uint32_t>(Mz); pval = ar.take<int32_t>(Mz);
    tmp = ar.take<char>(tmp_bytes);
  });
  if (rc != CG_OK) return rc;
  if (many) {   // from pageable memory: staged at once, no synchronisation
    CG_CUDA(ctx, cudaMemcpyAsync(dpoff, poff, sizeof(int32_t) * (Bz + 1), cudaMemcpyHostToDevice, st));
    CG_CUDA(ctx, cudaMemcpyAsync(dloff, loff, sizeof(int32_t) * (Bz + 1), cudaMemcpyHostToDevice, st));
  } else {
    dpoff = dloff = slot_frame = nullptr;
  }
  seg_init_kernel<<<blocks(L, 256), 256, 0, st>>>(L, cnt, kmin, kmax);
  CG_LAUNCH_CHECK(ctx);
  if (M > 0) {
    const unsigned g = std::min<unsigned>(blocks(M, ST_THREADS), 4u * (unsigned)ctx->num_sms);
    if (L <= ST_SMEM_L)
      seg_stats_kernel<true><<<g, ST_THREADS, 0, st>>>(labels, labels_is_i64, x, x_is_f64, M, L, dpoff, dloff, B, cnt,
                                                       kmin, kmax);
    else
      seg_stats_kernel<false><<<g, ST_THREADS, 0, st>>>(labels, labels_is_i64, x, x_is_f64, M, L, dpoff, dloff, B, cnt,
                                                        kmin, kmax);
    CG_LAUNCH_CHECK(ctx);
  }
  seg_decide_kernel<<<blocks(L, 256), 256, 0, st>>>(L, x_is_f64, cnt, kmin, kmax, out_min, out_max, out_count,
                                                    out_inlier, key);
  CG_LAUNCH_CHECK(ctx);
  size_t tb = tmp_bytes;
  if (many)
    CG_CUDA(ctx, cub::DeviceSegmentedRadixSort::SortKeysDescending(tmp, tb, key, key_sorted, L, B, dloff, dloff + 1, 0,
                                                                   64, st));
  else
    CG_CUDA(ctx, cub::DeviceRadixSort::SortKeysDescending(tmp, tb, key, key_sorted, L, 0, 64, st));
  seg_order_kernel<<<blocks(L, 256), 256, 0, st>>>(L, key_sorted, out_inlier, dloff, B, out_order, rank, out_n_kept,
                                                   seg_len, slot_frame);
  CG_LAUNCH_CHECK(ctx);
  // offsets: each frame's slots scanned on their own, its first slot 0
  tb = tmp_bytes;
  if (many)
    CG_CUDA(ctx, cub::DeviceScan::InclusiveSumByKey(tmp, tb, slot_frame, seg_len, out_offsets, (int)slots,
                                                    ::cuda::std::equal_to<>(), st));
  else
    CG_CUDA(ctx, cub::DeviceScan::InclusiveSum(tmp, tb, seg_len, out_offsets, (int)slots, st));
  if (M > 0) {
    seg_points_kernel<<<blocks(M, 256), 256, 0, st>>>(labels, labels_is_i64, M, L, dpoff, dloff, B, rank, out_labels,
                                                      pkey, pval);
    CG_LAUNCH_CHECK(ctx);
    // stable: within a segment the point indices stay ascending
    tb = tmp_bytes;
    CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp, tb, pkey, pkey_sorted, pval, out_index, M, 0, lbits, st));
  }
  return CG_OK;
}

}  // namespace

extern "C" int cg_segment_table_dev(cg_ctx *ctx, const void *labels, int labels_is_i64, const void *x, int x_is_f64,
                                    int M, int L, void *out_labels, int32_t *out_count, double *out_min,
                                    double *out_max, uint8_t *out_inlier, int32_t *out_order, int32_t *out_n_kept,
                                    int32_t *out_offsets, int32_t *out_index) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, M >= 0 && L >= 1 && L < (1 << 30), "segment_table: M must be >= 0 and L in [1, 2^30)");
  const int32_t poff[2] = {0, M}, loff[2] = {0, L};
  return segment_table(ctx, labels, labels_is_i64, x, x_is_f64, 1, poff, loff, out_labels, out_count, out_min, out_max,
                       out_inlier, out_order, out_n_kept, out_offsets, out_index);
}

extern "C" int cg_segment_table_many_dev(cg_ctx *ctx, const void *labels, int labels_is_i64, const void *x, int x_is_f64,
                                         int B, const int32_t *point_offsets, const int32_t *label_offsets,
                                         void *out_labels, int32_t *out_count, double *out_min, double *out_max,
                                         uint8_t *out_inlier, int32_t *out_order, int32_t *out_n_kept,
                                         int32_t *out_offsets, int32_t *out_index) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, B >= 1 && point_offsets && label_offsets, "segment_table_many: B >= 1 and both offset tables");
  CG_REQUIRE(ctx, point_offsets[0] == 0 && label_offsets[0] == 0, "segment_table_many: the offsets must start at 0");
  int64_t L = 0;
  for (int b = 0; b < B; b++) {
    CG_REQUIRE(ctx, point_offsets[b] <= point_offsets[b + 1], "segment_table_many: the point offsets must not decrease");
    CG_REQUIRE(ctx, label_offsets[b] < label_offsets[b + 1], "segment_table_many: every frame needs L_b >= 1 labels");
    L = label_offsets[b + 1];
  }
  CG_REQUIRE(ctx, L + B < (1 << 30), "segment_table_many: the frames' labels plus B must be below 2^30");
  return segment_table(ctx, labels, labels_is_i64, x, x_is_f64, B, point_offsets, label_offsets, out_labels, out_count,
                       out_min, out_max, out_inlier, out_order, out_n_kept, out_offsets, out_index);
}

extern "C" int cg_rank_grasps_dev(cg_ctx *ctx, const float *probs, int G, int C, int denom, const double *p_T_given_G,
                                  double *out_p_G, double *out_p_T_G, int32_t *out_perm) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, G >= 0 && C >= 1 && C <= 128 && denom >= 1,
             "rank_grasps: G must be >= 0, C in [1, 128] and denom >= 1");
  if (G == 0) return CG_OK;
  CG_REQUIRE(ctx, probs && p_T_given_G && out_p_G && out_p_T_G && out_perm, "rank_grasps: null argument");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  size_t sort_tmp = 0;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (uint64_t *)nullptr, (uint64_t *)nullptr,
                                               (int32_t *)nullptr, (int32_t *)nullptr, G, 0, 64, st));
  uint64_t *key, *key_sorted;
  int32_t *idx;
  void *tmp;
  const size_t Gz = (size_t)G;
  const int rc = cg_ws_carve(ctx, [&](cg_arena &ar) {
    key = ar.take<uint64_t>(Gz); key_sorted = ar.take<uint64_t>(Gz); idx = ar.take<int32_t>(Gz);
    tmp = ar.take<char>(sort_tmp);
  });
  if (rc != CG_OK) return rc;
  rank_score_kernel<<<blocks(G, 256), 256, 0, st>>>(probs, G, C, denom, p_T_given_G, out_p_G, out_p_T_G, key, idx);
  CG_LAUNCH_CHECK(ctx);
  size_t tb = sort_tmp;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp, tb, key, key_sorted, idx, out_perm, G, 0, 64, st));
  return CG_OK;
}
