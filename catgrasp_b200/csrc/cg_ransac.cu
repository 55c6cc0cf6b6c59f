// cg_ransac.cu -- hypothesis scoring of the NUNOCS 9-DoF RANSAC (SURVEY.md 8f F1).
//
// Replaces the loop body of aligning.py:36-81 (estimate9DTransform_worker) for all hypotheses at once:
//   4-point affine (cv2.estimateAffine3D on 4 correspondences = the exact affine through them, or the minimum-norm
//   least-squares affine when the 4 points are affinely dependent, aligning.py:23-33)
//   -> per-axis scales and scale gates (:41-43) -> R = A / scales, singular values in [0.8, 1.2] (:45-49)
//   -> R := U V^T, det > 0 (:51-53) -> T = [R diag(scales) | t] (:55)
//   -> extent of inv(T) target <= max_dimensions (:58-62) -> inlier ratio |T src - tgt| <= threshold (:64-67).
// One CTA per hypothesis: thread 0 does the 4x4 solve / 3x3 polar step in float64, all threads stream the N points.
// The 4-subsets come from the host (the reference's numpy RNG calls, aligning.py:91-97) or from cg_draw_ids_dev.
//
// cg_ransac9d_pose_dev runs the same kernel over one or two thresholds (one set of H subsets each) and also does what
// the host did with the scores: the first maximum among valid hypotheses per threshold (aligning.py:115) through a
// 64-bit atomicMax key, then, in the last CTA to finish (fence + counter), predict's choice between the thresholds
// (predicter.py:152-172: det test, inlier ratio at 3 mm, strict `>`).  Nothing comes back to the host.
//
// With a KdEval the same kernel scores by aligning.py:68-79 instead (use_kdtree_for_eval): for src_t = T [source, 1],
//   count = #{i : some voxel mean of the target is within thr of src_t[i]} + #{j : some voxel mean of src_t is within
//   thr of target[j]},   ratio = count / 2N.
// cKDTree's `nearest distance <= thr` is an existence test, so neither side needs a tree.  The target's voxel means
// come from a cg_cloud_index of the target (cell = resolution), built once per call; each CTA bins its own src_t into
// an open-addressing hash table of cells in a workspace of its own, sums each voxel in ascending point index (one
// warp per quarter of the table, so no sum depends on arrival order) and divides by the count, as voxel_kernel does.
// All of it is float64 without FMA: src_t = ((T00 x + T01 y) + T02 z) + T03, cells floor((p - origin) / r) with
// origin = min_bound - r * 0.5, distances cg_cloud_index.cuh's dist2 and a correctly rounded sqrt.  In this mode the
// grid is persistent (one workspace per CTA, CTAs loop over the hypotheses).
#include <algorithm>
#include <memory>
#include "cg_cloud_index.cuh"

namespace {

constexpr int RT = 128;

// solve M x = b for three right-hand sides, M 4x4 (rows = [src_i, 1]); partial pivoting; false if singular
__device__ bool solve4(double M[4][4], double B[4][3], double X[4][3]) {
  int perm[4] = {0, 1, 2, 3};
  for (int c = 0; c < 4; c++) {
    int p = c;
    double best = fabs(M[perm[c]][c]);
    for (int r = c + 1; r < 4; r++)
      if (fabs(M[perm[r]][c]) > best) { best = fabs(M[perm[r]][c]); p = r; }
    if (best < 1e-12) return false;
    const int t = perm[c]; perm[c] = perm[p]; perm[p] = t;
    const int pr = perm[c];
    for (int r = c + 1; r < 4; r++) {
      const int rr = perm[r];
      const double f = M[rr][c] / M[pr][c];
      for (int k = c; k < 4; k++) M[rr][k] -= f * M[pr][k];
      for (int k = 0; k < 3; k++) B[rr][k] -= f * B[pr][k];
    }
  }
  for (int k = 0; k < 3; k++)
    for (int c = 3; c >= 0; c--) {
      double s = B[perm[c]][k];
      for (int j = c + 1; j < 4; j++) s -= M[perm[c]][j] * X[j][k];
      X[c][k] = s / M[perm[c]][c];
    }
  return true;
}

// Minimum-norm least-squares solution X = pinv(M) B, the answer cv2.estimateAffine3D gives on 4 points when M is
// singular: it solves the 12x12 system (M's singular values, each three times) with DECOMP_SVD, which drops singular
// values <= 2 DBL_EPSILON * (sum of the 12) = 6 DBL_EPSILON * sum_j sigma_j(M) (OpenCV 4.13, bisected on cv2).
// One-sided (Hestenes) Jacobi on the columns of M: M V = W with orthogonal columns w_j = sigma_j u_j, so
// pinv(M) B = sum over kept j of v_j (w_j^T B) / sigma_j^2.  Small singular values come out to ~eps * sigma_max
// (an eigen-decomposition of M^T M would give sqrt(eps) * sigma_max, above the threshold).
__device__ void minnorm4(const double Min[4][4], const double B[4][3], double X[4][3]) {
  double W[4][4], V[4][4];
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) { W[i][j] = Min[i][j]; V[i][j] = (i == j) ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 30; sweep++) {
    bool rotated = false;
    for (int p = 0; p < 3; p++)
      for (int q = p + 1; q < 4; q++) {
        double a = 0.0, b = 0.0, g = 0.0;
        for (int i = 0; i < 4; i++) { a += W[i][p] * W[i][p]; b += W[i][q] * W[i][q]; g += W[i][p] * W[i][q]; }
        if (fabs(g) <= 1e-300 || fabs(g) <= 2.220446049250313e-16 * sqrt(a * b)) continue;
        rotated = true;
        const double zeta = (b - a) / (2.0 * g);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
        for (int i = 0; i < 4; i++) {
          const double wp = W[i][p], wq = W[i][q];
          W[i][p] = c * wp - s * wq; W[i][q] = s * wp + c * wq;
          const double vp = V[i][p], vq = V[i][q];
          V[i][p] = c * vp - s * vq; V[i][q] = s * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
  double sig2[4], sum = 0.0;
  for (int j = 0; j < 4; j++) {
    sig2[j] = W[0][j] * W[0][j] + W[1][j] * W[1][j] + W[2][j] * W[2][j] + W[3][j] * W[3][j];
    sum += sqrt(sig2[j]);
  }
  const double cut = 6.0 * 2.220446049250313e-16 * sum;
  for (int r = 0; r < 4; r++)
    for (int k = 0; k < 3; k++) X[r][k] = 0.0;
  for (int j = 0; j < 4; j++) {
    if (!(sqrt(sig2[j]) > cut)) continue;
    for (int k = 0; k < 3; k++) {
      const double proj = (W[0][j] * B[0][k] + W[1][j] * B[1][k] + W[2][j] * B[2][k] + W[3][j] * B[3][k]) / sig2[j];
      for (int r = 0; r < 4; r++) X[r][k] += V[r][j] * proj;
    }
  }
}

// symmetric 3x3 eigen-decomposition by cyclic Jacobi: A = V diag(w) V^T
__device__ void jacobi3(double A[3][3], double V[3][3], double w[3]) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) V[i][j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 30; sweep++) {
    const double off = fabs(A[0][1]) + fabs(A[0][2]) + fabs(A[1][2]);
    if (off < 1e-300) break;
    for (int p = 0; p < 2; p++)
      for (int q = p + 1; q < 3; q++) {
        if (fabs(A[p][q]) < 1e-300) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; k++) {
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - s * akq;
          A[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; k++) {
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - s * aqk;
          A[q][k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 3; k++) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
  }
  for (int i = 0; i < 3; i++) w[i] = A[i][i];
}

// Gates of one launch, by value: the scale gates, the optional extent gate and up to two thresholds.
struct Gates {
  double thr[2];
  double min_scale[3], max_scale[3], max_dims[3];
  int has_max_dims;
};

// The fused selection (cg_ransac9d_pose_dev); keys == nullptr switches it off (cg_ransac9d_host).
//   keys[t]: per-threshold atomicMax of (count << 32) | (0xFFFFFFFF - h) over valid hypotheses (0: none valid);
//   keys[n_thr]: the completion counter.  record: see include/catgrasp_b200.h.
struct Fuse {
  unsigned long long *keys;
  double *record;
  double ratio_thr;
  int n_thr;
};

constexpr int REC_PER_THR = 19;   // winner, count, T (16), count at ratio_thr

// The kd-tree evaluation (ws == nullptr switches it off).  Each CTA owns ws + blockIdx.x * stride: src_t (N,3), each
// point's hash slot (N), then the table of 2^cap_log2 >= 2N cells: keys, counts, sums (later means).
struct KdEval {
  IndexView tv;            // the target's index (cell = r); the mean of cell table entry u is tmean[u]
  const double *tmean;
  double r;
  char *ws;
  size_t stride;
  int cap_log2;
  int *err;                // set to 1 when a transformed source is not finite or spans 2^KD_BITS voxels on an axis
};

constexpr int KD_BITS = MAX_AXIS_BITS;                    // bits per axis of a source voxel key
constexpr uint64_t KD_EMPTY = ~0ull;                      // no key has all 63 + 1 bits set
constexpr int KD_PARTS = RT / 32;                         // warps, each summing the voxels of one quarter of the table
// The per-CTA workspaces of one call stay under 1 GiB (about 100 N bytes each) unless that leaves fewer CTAs than
// SMs; below that the grid is the kernel's resident CTAs.
constexpr size_t KD_WS_BYTES = size_t(1) << 30;

__host__ __device__ inline size_t kd_src_bytes(int N) { return ((size_t)N * 3 * sizeof(double) + 255) & ~size_t(255); }
__host__ __device__ inline size_t kd_slot_bytes(int N) { return ((size_t)N * sizeof(int32_t) + 255) & ~size_t(255); }
__host__ inline size_t kd_stride(int N, int cap_log2) {
  const size_t cap = size_t(1) << cap_log2;
  return kd_src_bytes(N) + kd_slot_bytes(N) + cap * (sizeof(uint64_t) + sizeof(int32_t) + 3 * sizeof(double));
}

__device__ __forceinline__ unsigned kd_hash(uint64_t key, int cap_log2) {
  return (unsigned)((key * 0x9E3779B97F4A7C15ull) >> (64 - cap_log2));
}

// some point of pts[a, b) has sqrt(dist2(q, p)) <= thr
__device__ __forceinline__ bool any_within(const double *pts, int a, int b, double qx, double qy, double qz, double thr) {
  for (int u = a; u < b; u++)
    if (sqrt(dist2(qx, qy, qz, pts[3 * (size_t)u], pts[3 * (size_t)u + 1], pts[3 * (size_t)u + 2])) <= thr) return true;
  return false;
}

// aligning.py:68-79 for the hypothesis T (shared, 12 doubles) at threshold thr: the two-way count, in thread 0, or -1
// when the transformed source cannot be binned (k.err is then set).  Called by all RT threads.
__device__ int kd_count(const KdEval &k, const double *__restrict__ src, const double *__restrict__ tgt, int N,
                        const double *T, double thr, double (*red)[6], int *redc) {
  __shared__ double so[3];
  __shared__ int64_t smaxc[3];
  __shared__ int sbad;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  char *base = k.ws + (size_t)blockIdx.x * k.stride;
  double *P = reinterpret_cast<double *>(base);
  int32_t *pslot = reinterpret_cast<int32_t *>(base + kd_src_bytes(N));
  const unsigned cap = 1u << k.cap_log2, cmask = cap - 1u;
  uint64_t *hkey = reinterpret_cast<uint64_t *>(base + kd_src_bytes(N) + kd_slot_bytes(N));
  int32_t *hcnt = reinterpret_cast<int32_t *>(hkey + cap);
  double *hsum = reinterpret_cast<double *>(hcnt + cap);   // cap * 4 bytes keeps it 8-byte aligned (cap >= 8)

  // src_t, its bounds, and an empty table
  double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  int bad = 0;
  for (int i = tid; i < N; i += RT) {
    const double x = src[(size_t)i * 3], y = src[(size_t)i * 3 + 1], z = src[(size_t)i * 3 + 2];
    for (int a = 0; a < 3; a++) {
      const double v = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[a * 4], x), __dmul_rn(T[a * 4 + 1], y)),
                                           __dmul_rn(T[a * 4 + 2], z)), T[a * 4 + 3]);
      P[(size_t)i * 3 + a] = v;
      if (!isfinite(v)) bad = 1;
      mn[a] = fmin(mn[a], v); mx[a] = fmax(mx[a], v);
    }
  }
  for (unsigned j = tid; j < cap; j += RT) {
    hkey[j] = KD_EMPTY; hcnt[j] = 0;
    hsum[3 * (size_t)j] = 0.0; hsum[3 * (size_t)j + 1] = 0.0; hsum[3 * (size_t)j + 2] = 0.0;
  }
  for (int o = 16; o > 0; o >>= 1)
    for (int a = 0; a < 3; a++) {
      mn[a] = fmin(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = fmax(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
  if (lane == 0)
    for (int a = 0; a < 3; a++) { red[wid][a] = mn[a]; red[wid][3 + a] = mx[a]; }
  bad = __syncthreads_or(bad);
  if (tid == 0) {
    for (int w = 1; w < RT / 32; w++)
      for (int a = 0; a < 3; a++) { mn[a] = fmin(mn[a], red[w][a]); mx[a] = fmax(mx[a], red[w][3 + a]); }
    for (int a = 0; a < 3; a++) {
      so[a] = __dsub_rn(mn[a], __dmul_rn(k.r, 0.5));                     // open3d: min_bound - voxel_size * 0.5
      const double top = floor(__ddiv_rn(__dsub_rn(mx[a], so[a]), k.r));  // the largest point's cell (floor is monotone)
      if (!(top < (double)(1 << KD_BITS))) bad = 1;
      smaxc[a] = bad ? 0 : (int64_t)top;
    }
    sbad = bad;
    if (bad) atomicExch(k.err, 1);
  }
  __syncthreads();
  if (sbad) return -1;
  const double ox = so[0], oy = so[1], oz = so[2];

  // cells of the table; a cell's slot depends on arrival order, nothing computed from it does
  for (int i = tid; i < N; i += RT) {
    const uint64_t key = cell_key(P[(size_t)i * 3], P[(size_t)i * 3 + 1], P[(size_t)i * 3 + 2], ox, oy, oz, k.r, KD_BITS);
    unsigned h = kd_hash(key, k.cap_log2);
    for (;;) {
      const uint64_t prev = atomicCAS((unsigned long long *)&hkey[h], (unsigned long long)KD_EMPTY, (unsigned long long)key);
      if (prev == KD_EMPTY || prev == key) break;
      h = (h + 1) & cmask;
    }
    pslot[i] = (int32_t)h;
  }
  __syncthreads();

  // voxel sums in ascending point index: warp w owns the slots h % KD_PARTS == w and walks the points in order; the
  // lowest lane of each group of equal slots adds the group's points one by one
  for (int b0 = 0; b0 < N; b0 += 32) {
    const int i = b0 + lane;
    const int h = i < N ? pslot[i] : -1;
    const bool mine = h >= 0 && (h % KD_PARTS) == wid;
    const unsigned act = __ballot_sync(0xffffffffu, mine);
    if (mine) {
      const unsigned grp = __match_any_sync(act, h);
      if (lane == __ffs(grp) - 1) {
        double sx = hsum[3 * (size_t)h], sy = hsum[3 * (size_t)h + 1], sz = hsum[3 * (size_t)h + 2];
        for (unsigned m = grp; m; m &= m - 1) {
          const size_t o = 3 * (size_t)(b0 + __ffs(m) - 1);
          sx = __dadd_rn(sx, P[o]); sy = __dadd_rn(sy, P[o + 1]); sz = __dadd_rn(sz, P[o + 2]);
        }
        hsum[3 * (size_t)h] = sx; hsum[3 * (size_t)h + 1] = sy; hsum[3 * (size_t)h + 2] = sz;
        hcnt[h] += __popc(grp);
      }
    }
    __syncwarp();
  }
  __syncthreads();
  for (unsigned j = tid; j < cap; j += RT) {
    const int c = hcnt[j];
    if (c == 0) continue;
    const double dc = (double)c;
    hsum[3 * (size_t)j] = __ddiv_rn(hsum[3 * (size_t)j], dc);
    hsum[3 * (size_t)j + 1] = __ddiv_rn(hsum[3 * (size_t)j + 1], dc);
    hsum[3 * (size_t)j + 2] = __ddiv_rn(hsum[3 * (size_t)j + 2], dc);
  }
  __syncthreads();

  int cnt = 0;
  // dists1 <= thr: src_t against the target's voxel means, through the target's cell table
  for (int i = tid; i < N; i += RT) {
    const double qx = P[(size_t)i * 3], qy = P[(size_t)i * 3 + 1], qz = P[(size_t)i * 3 + 2];
    const Columns C(k.tv, qx, qy, qz, thr);
    bool hit = false;
    if (C.any)
      for (int64_t cx = C.x0; cx <= C.x1 && !hit; cx++)
        for (int64_t cy = C.y0; cy <= C.y1 && !hit; cy++) {
          int a, b;
          C.cells(k.tv, cx, cy, a, b);
          hit = any_within(k.tmean, a, b, qx, qy, qz, thr);
        }
    cnt += hit ? 1 : 0;
  }
  // dists2 <= thr: the target against src_t's voxel means, cell by cell through the table.  The cell range is
  // axis_range's, widened by RANGE_SLACK cells: a rounded mean may lie an ulp outside its voxel.
  for (int j = tid; j < N; j += RT) {
    const double qx = tgt[(size_t)j * 3], qy = tgt[(size_t)j * 3 + 1], qz = tgt[(size_t)j * 3 + 2];
    int64_t x0, x1, y0, y1, z0, z1;
    bool hit = false;
    if (axis_range(qx, ox, thr, k.r, smaxc[0], x0, x1) && axis_range(qy, oy, thr, k.r, smaxc[1], y0, y1) &&
        axis_range(qz, oz, thr, k.r, smaxc[2], z0, z1))
      for (int64_t cx = x0; cx <= x1 && !hit; cx++)
        for (int64_t cy = y0; cy <= y1 && !hit; cy++)
          for (int64_t cz = z0; cz <= z1 && !hit; cz++) {
            const uint64_t key = pack(cx, cy, cz, KD_BITS);
            for (unsigned h = kd_hash(key, k.cap_log2);; h = (h + 1) & cmask) {
              const uint64_t kh = hkey[h];
              if (kh == KD_EMPTY) break;
              if (kh == key) { hit = any_within(hsum, (int)h, (int)h + 1, qx, qy, qz, thr); break; }
            }
          }
    cnt += hit ? 1 : 0;
  }
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) redc[wid] = cnt;
  __syncthreads();
  int c = 0;
  if (tid == 0)
    for (int w = 0; w < RT / 32; w++) c += redc[w];
  return c;
}

// The fused selection after the CTA's last pair: the last CTA to finish (fence + counter) reads each threshold's winner
// and its T, counts the winner's residuals <= f.ratio_thr and makes predict's choice between the thresholds
// (predicter.py:152-172's loop), into f.record.  Called by all RT threads; T and win are shared scratch.
__device__ void select_pose(const Fuse &f, const double *src, const double *tgt, int N, int H, const double *out_T,
                            double *T, int *redc, int &win) {
  __shared__ int last;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) {
    __threadfence();   // this CTA's T and key before its count
    last = atomicAdd(&f.keys[f.n_thr], 1ull) == (unsigned long long)gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double *rec = f.record;
  double best_ratio = 0.0;
  int chosen = -1;
  for (int t = 0; t < f.n_thr; t++) {
    if (tid == 0) {
      const unsigned long long key = atomicAdd(&f.keys[t], 0ull);
      win = key ? (int)(0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFull)) : -1;
    }
    __syncthreads();
    const int w = win;
    if (w >= 0 && tid < 12) T[tid] = __ldcg(&out_T[((size_t)t * H + w) * 16 + tid]);   // the scoring pass's T, not a recompute
    __syncthreads();
    int cnt = 0;
    if (w >= 0)
      for (int i = tid; i < N; i += RT) {
        const double sx = src[(size_t)i * 3], sy = src[(size_t)i * 3 + 1], sz = src[(size_t)i * 3 + 2];
        const double ex = T[0] * sx + T[1] * sy + T[2] * sz + T[3] - tgt[(size_t)i * 3];
        const double ey = T[4] * sx + T[5] * sy + T[6] * sz + T[7] - tgt[(size_t)i * 3 + 1];
        const double ez = T[8] * sx + T[9] * sy + T[10] * sz + T[11] - tgt[(size_t)i * 3 + 2];
        if (sqrt(ex * ex + ey * ey + ez * ez) <= f.ratio_thr) cnt++;
      }
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) redc[wid] = cnt;
    __syncthreads();
    if (tid == 0) {
      double *r = rec + (size_t)t * REC_PER_THR;
      int c3 = 0;
      for (int w2 = 0; w2 < RT / 32; w2++) c3 += redc[w2];
      r[0] = (double)w;
      r[1] = w >= 0 ? (double)(int)(__ldcg(&f.keys[t]) >> 32) : 0.0;
      for (int k = 0; k < 16; k++) r[2 + k] = w >= 0 ? __ldcg(&out_T[((size_t)t * H + w) * 16 + k]) : 0.0;
      r[18] = (double)c3;
      if (w >= 0) {
        // predict's checks on the winner: det(T[:3,:3]) >= 0, then ratio > best_ratio (the first threshold wins a tie;
        // a winner with no point within ratio_thr is not a pose)
        const double det = T[0] * (T[5] * T[10] - T[6] * T[9]) - T[1] * (T[4] * T[10] - T[6] * T[8]) +
                           T[2] * (T[4] * T[9] - T[5] * T[8]);
        const double ratio = (double)c3 / (double)N;
        if (!(det < 0) && ratio > best_ratio) { best_ratio = ratio; chosen = t; }
      }
    }
    __syncthreads();
  }
  if (tid == 0) {
    double *r = rec + (size_t)f.n_thr * REC_PER_THR;
    r[0] = (double)chosen;
    for (int k = 0; k < 16; k++) r[1 + k] = chosen >= 0 ? rec[(size_t)chosen * REC_PER_THR + 2 + k] : 0.0;
    r[17] = best_ratio;
  }
}

// Launched with RT threads.  __maxnreg__ rather than __launch_bounds__(RT): with the kd-tree path inlined, the launch
// bound lets ptxas settle on 128 registers and spill the scoring loop; 168 keeps 3 CTAs per SM, as before that path.
// Thread 0's hypothesis and the residual count stay in the kernel body: moved into __device__ functions, even verbatim,
// they change ptxas's register allocation and cost 0.2-0.7 % of the residual launch (H100 80GB HBM3, 700 W).
__global__ void __maxnreg__(168) ransac9d_kernel(const double *__restrict__ src, const double *__restrict__ tgt, int N,
                                                 const int32_t *__restrict__ ids, int H, int NB, const Gates g,
                                                 double *__restrict__ out_ratio, double *__restrict__ out_T,
                                                 unsigned char *__restrict__ out_valid, const Fuse f, const KdEval kd) {
  __shared__ double T[12], Ti[12];
  __shared__ int ok;
  __shared__ double red[RT / 32][6];
  __shared__ int redc[RT / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // Object blockIdx.y of a batched pose search (cg_ransac9d_pose_many_dev): its source, target, subsets, T workspace,
  // keys and record.  Every other launch has gridDim.y == 1.
  const size_t obj = blockIdx.y;
  src += obj * N * 3;
  tgt += obj * N * 3;
  ids += obj * NB * 4;
  out_T += obj * NB * 16;
  Fuse fo = f;
  fo.keys += obj * (f.n_thr + 1);
  fo.record += obj * (f.n_thr * REC_PER_THR + 18);
  // NB = (threshold, hypothesis) pairs: pair b scores hypothesis b % H of threshold b / H with the subset ids[b].  One
  // CTA per pair (gridDim.x == NB), or, with the kd-tree evaluation, fewer CTAs that each take every gridDim.x-th pair.
  for (int b = blockIdx.x; b < NB; b += gridDim.x) {
    const double thr = b < H ? g.thr[0] : g.thr[1];   // no run-time index into the parameter block
    if (tid == 0) {
      ok = 0;
      double M[4][4], B[4][3], X[4][3], M0[4][4], B0[4][3];
      for (int i = 0; i < 4; i++) {
        const int id = ids[(size_t)b * 4 + i];
        // cv2.estimateAffine3D (aligning.py:27) narrows its inputs to CV_32F before the double-precision solve:
        // the four sample points go through float, the residual pass below keeps the caller's float64.
        for (int k = 0; k < 3; k++) {
          M[i][k] = M0[i][k] = (double)(float)src[(size_t)id * 3 + k];
          B[i][k] = B0[i][k] = (double)(float)tgt[(size_t)id * 3 + k];
        }
        M[i][3] = M0[i][3] = 1.0;
      }
      // X[j][k]: dst_k = sum_j X[j][k] * [src,1]_j  -> A[k][j] = X[j][k].  A pivot below 1e-12 (duplicate, coplanar or
      // nearly so) sends the subset to the minimum-norm solve; it is as rare as such subsets are.
      if (!solve4(M, B, X)) minnorm4(M0, B0, X);
      bool good = true;
      double A[3][3], t[3], sc[3];
      {
        for (int k = 0; k < 3; k++) {
          for (int j = 0; j < 3; j++) A[k][j] = X[j][k];
          t[k] = X[3][k];
        }
        for (int j = 0; j < 3; j++) {   // scales = column norms (aligning.py:41)
          sc[j] = sqrt(A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j]);
          if (sc[j] > g.max_scale[j] || sc[j] < g.min_scale[j]) good = false;
        }
      }
      if (good) {
        double R[3][3], G[3][3], V[3][3], w[3];
        for (int i = 0; i < 3; i++)
          for (int j = 0; j < 3; j++) R[i][j] = A[i][j] / sc[j];
        for (int i = 0; i < 3; i++)
          for (int j = 0; j < 3; j++) G[i][j] = R[0][i] * R[0][j] + R[1][i] * R[1][j] + R[2][i] * R[2][j];
        jacobi3(G, V, w);             // R^T R = V diag(w) V^T, singular values = sqrt(w)
        double smin = 1e300, smax = 0.0;
        for (int i = 0; i < 3; i++) {
          const double s = sqrt(fmax(w[i], 0.0));
          smin = fmin(smin, s); smax = fmax(smax, s);
        }
        if (smin < 0.8 || smax > 1.2) good = false;
        if (good) {
          // U V^T = R V diag(1/s) V^T
          double Q[3][3];
          for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
              double acc = 0.0;
              for (int k = 0; k < 3; k++) acc += V[i][k] * V[j][k] / sqrt(w[k]);
              Q[i][j] = acc;
            }
          double Ro[3][3];
          for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) Ro[i][j] = R[i][0] * Q[0][j] + R[i][1] * Q[1][j] + R[i][2] * Q[2][j];
          const double det = Ro[0][0] * (Ro[1][1] * Ro[2][2] - Ro[1][2] * Ro[2][1]) -
                             Ro[0][1] * (Ro[1][0] * Ro[2][2] - Ro[1][2] * Ro[2][0]) +
                             Ro[0][2] * (Ro[1][0] * Ro[2][1] - Ro[1][1] * Ro[2][0]);
          if (det < 0) good = false;
          if (good) {
            for (int i = 0; i < 3; i++) {
              for (int j = 0; j < 3; j++) T[i * 4 + j] = Ro[i][j] * sc[j];
              T[i * 4 + 3] = t[i];
            }
            // inverse: (Ro S)^-1 = S^-1 Ro^T
            for (int i = 0; i < 3; i++) {
              for (int j = 0; j < 3; j++) Ti[i * 4 + j] = Ro[j][i] / sc[i];
              Ti[i * 4 + 3] = -(Ti[i * 4 + 0] * t[0] + Ti[i * 4 + 1] * t[1] + Ti[i * 4 + 2] * t[2]);
            }
            ok = 1;
          }
        }
      }
    }
    __syncthreads();
    if (ok) {
      double mn[3] = {1e300, 1e300, 1e300}, mx[3] = {-1e300, -1e300, -1e300};
      int cnt = 0;
      for (int i = tid; i < N; i += RT) {
        const double sx = src[(size_t)i * 3], sy = src[(size_t)i * 3 + 1], sz = src[(size_t)i * 3 + 2];
        const double tx = tgt[(size_t)i * 3], ty = tgt[(size_t)i * 3 + 1], tz = tgt[(size_t)i * 3 + 2];
        const double ex = T[0] * sx + T[1] * sy + T[2] * sz + T[3] - tx;
        const double ey = T[4] * sx + T[5] * sy + T[6] * sz + T[7] - ty;
        const double ez = T[8] * sx + T[9] * sy + T[10] * sz + T[11] - tz;
        if (sqrt(ex * ex + ey * ey + ez * ez) <= thr) cnt++;
        if (g.has_max_dims) {
          for (int k = 0; k < 3; k++) {
            const double c = Ti[k * 4] * tx + Ti[k * 4 + 1] * ty + Ti[k * 4 + 2] * tz + Ti[k * 4 + 3];
            mn[k] = fmin(mn[k], c); mx[k] = fmax(mx[k], c);
          }
        }
      }
      for (int o = 16; o > 0; o >>= 1) {
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        for (int k = 0; k < 3; k++) {
          mn[k] = fmin(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], o));
          mx[k] = fmax(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
        }
      }
      if (lane == 0) {
        redc[wid] = cnt;
        for (int k = 0; k < 3; k++) { red[wid][k] = mn[k]; red[wid][3 + k] = mx[k]; }
      }
      __syncthreads();
      int c = 0;
      bool good = true;
      if (tid == 0) {
        for (int w2 = 0; w2 < RT / 32; w2++) {
          c += redc[w2];
          for (int k = 0; k < 3; k++) { mn[k] = fmin(mn[k], red[w2][k]); mx[k] = fmax(mx[k], red[w2][3 + k]); }
        }
        if (g.has_max_dims)
          for (int k = 0; k < 3; k++)
            if (mx[k] - mn[k] > g.max_dims[k]) good = false;
      }
      const int den = kd.ws ? 2 * N : N;
      if (kd.ws) {                            // the gates above decide first; the kd-tree count replaces the residual count
        if (tid == 0) ok = good;
        __syncthreads();
        if (ok) c = kd_count(kd, src, tgt, N, T, thr, red, redc);
        if (c < 0) good = false;
      }
      if (tid == 0) {
        if (out_valid) {
          out_valid[b] = good ? 1 : 0;
          out_ratio[b] = good ? (double)c / (double)den : 0.0;
        }
        if (good) {
          for (int k = 0; k < 12; k++) out_T[(size_t)b * 16 + k] = T[k];
          out_T[(size_t)b * 16 + 12] = 0.0; out_T[(size_t)b * 16 + 13] = 0.0; out_T[(size_t)b * 16 + 14] = 0.0;
          out_T[(size_t)b * 16 + 15] = 1.0;
          // count / N is monotone in count, so the largest key is the host's first maximum among valid hypotheses
          if (fo.keys)
            atomicMax(&fo.keys[b / H], ((unsigned long long)c << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)(b % H)));
        }
      }
    } else if (tid == 0 && out_valid) {
      out_valid[b] = 0; out_ratio[b] = 0.0;
    }
    __syncthreads();                         // T, Ti, ok, red and redc are the next pair's
  }
  if (fo.keys) select_pose(fo, src, tgt, N, H, out_T, T, redc, ok);
}

Gates make_gates(const double *thresholds, int n_thr, const double min_scale[3], const double max_scale[3],
                 const double *max_dims) {
  Gates g{};
  for (int t = 0; t < 2; t++) g.thr[t] = thresholds[t < n_thr ? t : 0];
  for (int k = 0; k < 3; k++) { g.min_scale[k] = min_scale[k]; g.max_scale[k] = max_scale[k]; g.max_dims[k] = max_dims ? max_dims[k] : 0.0; }
  g.has_max_dims = max_dims != nullptr;
  return g;
}

bool good_resolution(double r) { return std::isfinite(r) && r > 0.0; }

// Every launch of ransac9d_kernel: H hypotheses for each of n_thr thresholds on device inputs.  Without a record it
// writes cg_ransac9d_host's per-hypothesis out_ratio, out_T (zeroed first) and out_valid; with one, the fused selection
// writes cg_ransac9d_pose_dev's record and every T goes to the workspace.  kd_r > 0 scores by the kd-tree evaluation
// at that resolution: the target's index and voxel means, a persistent grid with one workspace per CTA, and the
// kernel's error word read back.  That synchronises the stream twice in cg_cloud_index_create, once for the error word
// and once more when the index is destroyed.
// With a record, B objects (B > 1 only without kd_r): src / tgt (B,N,3), ids (B,nb,4), record B records; the grid's y
// is the object, CG_RANSAC_MANY_PASS_PAIRS / nb objects per launch at most, the launches in object order over one
// workspace.
int ransac9d(cg_ctx *ctx, const double *src, const double *tgt, int N, const int32_t *ids, int H, int n_thr,
             const Gates &g, double kd_r, double *out_ratio, double *out_T, unsigned char *out_valid, double *record,
             double ratio_thr, int B = 1) {
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const int nb = n_thr * H;
  const bool kd = kd_r > 0.0;
  CG_REQUIRE(ctx, B == 1 || (record && !kd), "ransac9d: several objects need the fused selection without kd_r");
  const int per_launch = (int)std::min<long long>(B, std::max<long long>(1, CG_RANSAC_MANY_PASS_PAIRS / nb));
  std::unique_ptr<cg_cloud_index, void (*)(cg_cloud_index *)> ix(nullptr, cg_cloud_index_destroy);
  int grid = nb, cap_log2 = 3;
  size_t stride = 0;
  if (kd) {
    cg_cloud_index *p = nullptr;
    int rc = cg_cloud_index_create(ctx, tgt, N, kd_r, &p);
    ix.reset(p);
    if (rc) return rc;
    while ((size_t(1) << cap_log2) < 2 * (size_t)N) cap_log2++;
    stride = kd_stride(N, cap_log2);
    int per_sm = 0;
    CG_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ransac9d_kernel, RT, 0));
    const long long resident = (long long)std::max(per_sm, 1) * ctx->num_sms;
    const long long budget = std::max<long long>(ctx->num_sms, (long long)(KD_WS_BYTES / stride));
    grid = (int)std::min<long long>({(long long)nb, resident, budget});
  }
  unsigned long long *keys = nullptr;   // per-threshold keys, then the completion counter
  double *tmean = nullptr;              // the target's voxel means
  int *err = nullptr;
  char *ws = nullptr;                   // one workspace per CTA
  int rc = cg_ws_carve(ctx, [&](cg_arena &ar) {
    if (record) {   // per object: every valid hypothesis's T, read back by the last CTA; keys and counter
      out_T = ar.take<double>((size_t)per_launch * nb * 16);
      keys = ar.take<unsigned long long>((size_t)per_launch * (n_thr + 1));
    }
    if (kd) {
      tmean = ar.take<double>((size_t)ix->U * 3);
      err = ar.take<int>(1);
      ws = ar.take<char>(stride * (size_t)grid);
    }
  });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  if (kd) {
    if ((rc = cg_voxel_down_sample_dev(ix.get(), nullptr, tmean, nullptr))) return rc;
    CG_CUDA(ctx, cudaMemsetAsync(err, 0, sizeof(int), st));
  }
  if (!record) CG_CUDA(ctx, cudaMemsetAsync(out_T, 0, (size_t)H * 128, st));
  const KdEval k = kd ? KdEval{view_of(ix.get()), tmean, kd_r, ws, stride, cap_log2, err} : KdEval{};
  const size_t rec_len = (size_t)n_thr * REC_PER_THR + 18;
  for (int b0 = 0; b0 < B; b0 += per_launch) {
    const int nob = std::min(per_launch, B - b0);
    if (record)
      CG_CUDA(ctx, cudaMemsetAsync(keys, 0, (size_t)nob * (n_thr + 1) * sizeof(unsigned long long), st));
    const Fuse f = record ? Fuse{keys, record + (size_t)b0 * rec_len, ratio_thr, n_thr} : Fuse{};
    const size_t o = (size_t)b0 * N * 3;
    ransac9d_kernel<<<dim3(grid, nob), RT, 0, st>>>(src + o, tgt + o, N, ids + (size_t)b0 * nb * 4, H, nb, g, out_ratio,
                                                   out_T, out_valid, f, k);
    CG_LAUNCH_CHECK(ctx);
  }
  if (!kd) return CG_OK;
  int h = 0;
  CG_CUDA(ctx, cudaMemcpyAsync(&h, err, sizeof(int), cudaMemcpyDeviceToHost, st));
  CG_CUDA(ctx, cudaStreamSynchronize(st));
  CG_REQUIRE(ctx, h == 0, "ransac9d_kdtree: a transformed source is not finite or spans 2^21 or more voxels on an axis");
  return CG_OK;
}

}  // namespace

extern "C" int cg_ransac9d_host(cg_ctx *ctx, const double *source, const double *target, int N, const int32_t *ids, int H,
                                double pass_threshold, const double min_scale[3], const double max_scale[3],
                                const double *max_dims, double *out_ratio, double *out_T, unsigned char *out_valid) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, source && target && ids && N >= 4 && H > 0 && min_scale && max_scale, "ransac9d: bad arguments");
  CG_REQUIRE(ctx, out_ratio && out_T && out_valid, "ransac9d: outputs");
  const Gates g = make_gates(&pass_threshold, 1, min_scale, max_scale, max_dims);
  const double *d_src, *d_tgt; const int32_t *d_ids; double *d_ratio, *d_T; unsigned char *d_valid;
  return cg_io_stage(ctx, [&](cg_io_pieces &io) {
    d_src = io.in(source, (size_t)N * 3);
    d_tgt = io.in(target, (size_t)N * 3);
    d_ids = io.in(ids, (size_t)H * 4);
    d_ratio = io.out(out_ratio, H);
    d_T = io.out(out_T, (size_t)H * 16);
    d_valid = io.out(out_valid, H);
  }, [&] { return ransac9d(ctx, d_src, d_tgt, N, d_ids, H, 1, g, 0.0, d_ratio, d_T, d_valid, nullptr, 0.0); });
}

extern "C" int cg_ransac9d_kdtree_host(cg_ctx *ctx, const double *source, const double *target, int N, const int32_t *ids,
                                       int H, double pass_threshold, const double min_scale[3], const double max_scale[3],
                                       const double *max_dims, double resolution, double *out_ratio, double *out_T,
                                       unsigned char *out_valid) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, source && target && ids && N >= 4 && H > 0 && min_scale && max_scale, "ransac9d_kdtree: bad arguments");
  CG_REQUIRE(ctx, N <= CG_RANSAC_KD_MAX_N, "ransac9d_kdtree: N > CG_RANSAC_KD_MAX_N");
  CG_REQUIRE(ctx, good_resolution(resolution), "ransac9d_kdtree: resolution must be positive and finite");
  CG_REQUIRE(ctx, out_ratio && out_T && out_valid, "ransac9d_kdtree: outputs");
  const Gates g = make_gates(&pass_threshold, 1, min_scale, max_scale, max_dims);
  const double *d_src, *d_tgt; const int32_t *d_ids; double *d_ratio, *d_T; unsigned char *d_valid;
  return cg_io_stage(ctx, [&](cg_io_pieces &io) {
    d_src = io.in(source, (size_t)N * 3);
    d_tgt = io.in(target, (size_t)N * 3);
    d_ids = io.in(ids, (size_t)H * 4);
    d_ratio = io.out(out_ratio, H);
    d_T = io.out(out_T, (size_t)H * 16);
    d_valid = io.out(out_valid, H);
  }, [&] { return ransac9d(ctx, d_src, d_tgt, N, d_ids, H, 1, g, resolution, d_ratio, d_T, d_valid, nullptr, 0.0); });
}

extern "C" int cg_ransac9d_pose_dev(cg_ctx *ctx, const double *source, const double *target, int N, const int32_t *ids,
                                    int H, const double *thresholds, int n_thr, const double min_scale[3],
                                    const double max_scale[3], const double *max_dims, double ratio_threshold,
                                    double *out_record) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, source && target && ids && N >= 4 && H > 0 && thresholds && (n_thr == 1 || n_thr == 2) && min_scale &&
                      max_scale && out_record, "ransac9d_pose: bad arguments");
  CG_REQUIRE(ctx, (long long)H * n_thr <= 0x7FFFFFFFll, "ransac9d_pose: too many hypotheses");
  const Gates g = make_gates(thresholds, n_thr, min_scale, max_scale, max_dims);
  return ransac9d(ctx, source, target, N, ids, H, n_thr, g, 0.0, nullptr, nullptr, nullptr, out_record, ratio_threshold);
}

extern "C" int cg_ransac9d_pose_many_dev(cg_ctx *ctx, const double *source, const double *target, int B, int N,
                                         const int32_t *ids, int H, const double *thresholds, int n_thr,
                                         const double min_scale[3], const double max_scale[3], const double *max_dims,
                                         double ratio_threshold, double *out_records) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, source && target && ids && N >= 4 && H > 0 && thresholds && (n_thr == 1 || n_thr == 2) && min_scale &&
                      max_scale && out_records, "ransac9d_pose_many: bad arguments");
  CG_REQUIRE(ctx, B >= 1 && B <= CG_NUNOCS_MANY_MAX_B, "ransac9d_pose_many: 1 <= B <= CG_NUNOCS_MANY_MAX_B");
  CG_REQUIRE(ctx, (long long)H * n_thr <= 0x7FFFFFFFll, "ransac9d_pose_many: too many hypotheses");
  const Gates g = make_gates(thresholds, n_thr, min_scale, max_scale, max_dims);
  return ransac9d(ctx, source, target, N, ids, H, n_thr, g, 0.0, nullptr, nullptr, nullptr, out_records,
                  ratio_threshold, B);
}

extern "C" int cg_ransac9d_kdtree_pose_dev(cg_ctx *ctx, const double *source, const double *target, int N,
                                           const int32_t *ids, int H, const double *thresholds, int n_thr,
                                           const double min_scale[3], const double max_scale[3], const double *max_dims,
                                           double ratio_threshold, double resolution, double *out_record) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, source && target && ids && N >= 4 && H > 0 && thresholds && (n_thr == 1 || n_thr == 2) && min_scale &&
                      max_scale && out_record, "ransac9d_kdtree_pose: bad arguments");
  CG_REQUIRE(ctx, (long long)H * n_thr <= 0x7FFFFFFFll, "ransac9d_kdtree_pose: too many hypotheses");
  CG_REQUIRE(ctx, N <= CG_RANSAC_KD_MAX_N, "ransac9d_kdtree_pose: N > CG_RANSAC_KD_MAX_N");
  CG_REQUIRE(ctx, good_resolution(resolution), "ransac9d_kdtree_pose: resolution must be positive and finite");
  const Gates g = make_gates(thresholds, n_thr, min_scale, max_scale, max_dims);
  return ransac9d(ctx, source, target, N, ids, H, n_thr, g, resolution, nullptr, nullptr, nullptr, out_record,
                  ratio_threshold);
}
