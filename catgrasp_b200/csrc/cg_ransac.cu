// cg_ransac.cu -- hypothesis scoring of the NUNOCS 9-DoF RANSAC (SURVEY.md 8f F1).
//
// Replaces the loop body of aligning.py:36-81 (estimate9DTransform_worker) for all hypotheses at once:
//   4-point affine (cv2.estimateAffine3D on 4 correspondences = the exact affine through them, or the minimum-norm
//   least-squares affine when the 4 points are affinely dependent, aligning.py:23-33)
//   -> per-axis scales and scale gates (:41-43) -> R = A / scales, singular values in [0.8, 1.2] (:45-49)
//   -> R := U V^T, det > 0 (:51-53) -> T = [R diag(scales) | t] (:55)
//   -> extent of inv(T) target <= max_dimensions (:58-62) -> inlier ratio |T src - tgt| <= threshold (:64-67).
// One CTA per hypothesis: thread 0 does the 4x4 solve / 3x3 polar step in float64, all threads stream the N points.
// The 4-subsets are drawn on the host with the reference's numpy RNG calls (aligning.py:91-97).
#include "cg_common.cuh"

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

__global__ void __launch_bounds__(RT) ransac9d_kernel(const double *__restrict__ src, const double *__restrict__ tgt, int N,
                                                      const int32_t *__restrict__ ids, int H, double thr,
                                                      const double *__restrict__ min_scale,
                                                      const double *__restrict__ max_scale,
                                                      const double *__restrict__ max_dims, double *__restrict__ out_ratio,
                                                      double *__restrict__ out_T, unsigned char *__restrict__ out_valid) {
  __shared__ double T[12], Ti[12];
  __shared__ int ok;
  __shared__ double red[RT / 32][6];
  __shared__ int redc[RT / 32];
  const int h = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) {
    ok = 0;
    double M[4][4], B[4][3], X[4][3], M0[4][4], B0[4][3];
    for (int i = 0; i < 4; i++) {
      const int id = ids[h * 4 + i];
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
        if (sc[j] > max_scale[j] || sc[j] < min_scale[j]) good = false;
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
  if (!ok) {
    if (tid == 0) { out_valid[h] = 0; out_ratio[h] = 0.0; }
    return;
  }
  double mn[3] = {1e300, 1e300, 1e300}, mx[3] = {-1e300, -1e300, -1e300};
  int cnt = 0;
  for (int i = tid; i < N; i += RT) {
    const double sx = src[(size_t)i * 3], sy = src[(size_t)i * 3 + 1], sz = src[(size_t)i * 3 + 2];
    const double tx = tgt[(size_t)i * 3], ty = tgt[(size_t)i * 3 + 1], tz = tgt[(size_t)i * 3 + 2];
    const double ex = T[0] * sx + T[1] * sy + T[2] * sz + T[3] - tx;
    const double ey = T[4] * sx + T[5] * sy + T[6] * sz + T[7] - ty;
    const double ez = T[8] * sx + T[9] * sy + T[10] * sz + T[11] - tz;
    if (sqrt(ex * ex + ey * ey + ez * ez) <= thr) cnt++;
    if (max_dims) {
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
  if (tid == 0) {
    int c = 0;
    for (int w2 = 0; w2 < RT / 32; w2++) {
      c += redc[w2];
      for (int k = 0; k < 3; k++) { mn[k] = fmin(mn[k], red[w2][k]); mx[k] = fmax(mx[k], red[w2][3 + k]); }
    }
    bool good = true;
    if (max_dims)
      for (int k = 0; k < 3; k++)
        if (mx[k] - mn[k] > max_dims[k]) good = false;
    out_valid[h] = good ? 1 : 0;
    out_ratio[h] = good ? (double)c / (double)N : 0.0;
    if (good) {
      for (int k = 0; k < 12; k++) out_T[(size_t)h * 16 + k] = T[k];
      out_T[(size_t)h * 16 + 12] = 0.0; out_T[(size_t)h * 16 + 13] = 0.0; out_T[(size_t)h * 16 + 14] = 0.0;
      out_T[(size_t)h * 16 + 15] = 1.0;
    }
  }
}

}  // namespace

extern "C" int cg_ransac9d_host(cg_ctx *ctx, const double *source, const double *target, int N, const int32_t *ids, int H,
                                double pass_threshold, const double min_scale[3], const double max_scale[3],
                                const double *max_dims, double *out_ratio, double *out_T, unsigned char *out_valid) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, source && target && ids && N >= 4 && H > 0 && min_scale && max_scale, "ransac9d: bad arguments");
  CG_REQUIRE(ctx, out_ratio && out_T && out_valid, "ransac9d: outputs");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  double *d_src, *d_tgt, *d_par, *d_ratio, *d_T; int32_t *d_ids; unsigned char *d_valid;
  int rc = cg_io_carve(ctx, [&](cg_arena &ar) {
    d_src = ar.take<double>((size_t)N * 3);
    d_tgt = ar.take<double>((size_t)N * 3);
    d_ids = ar.take<int32_t>((size_t)H * 4);
    d_par = ar.take<double>(9);
    d_ratio = ar.take<double>(H);
    d_T = ar.take<double>((size_t)H * 16);
    d_valid = ar.take<unsigned char>(H);
  });
  if (rc) return rc;
  double par[9];
  for (int k = 0; k < 3; k++) { par[k] = min_scale[k]; par[3 + k] = max_scale[k]; par[6 + k] = max_dims ? max_dims[k] : 0.0; }
  cudaStream_t st = ctx->stream;
  CG_CUDA(ctx, cudaMemcpyAsync(d_src, source, (size_t)N * 24, cudaMemcpyHostToDevice, st));
  CG_CUDA(ctx, cudaMemcpyAsync(d_tgt, target, (size_t)N * 24, cudaMemcpyHostToDevice, st));
  CG_CUDA(ctx, cudaMemcpyAsync(d_ids, ids, (size_t)H * 16, cudaMemcpyHostToDevice, st));
  CG_CUDA(ctx, cudaMemcpyAsync(d_par, par, sizeof(par), cudaMemcpyHostToDevice, st));
  CG_CUDA(ctx, cudaMemsetAsync(d_T, 0, (size_t)H * 128, st));
  ransac9d_kernel<<<H, RT, 0, st>>>(d_src, d_tgt, N, d_ids, H, pass_threshold, d_par, d_par + 3, max_dims ? d_par + 6 : nullptr,
                                    d_ratio, d_T, d_valid);
  CG_LAUNCH_CHECK(ctx);
  CG_CUDA(ctx, cudaMemcpyAsync(out_ratio, d_ratio, (size_t)H * 8, cudaMemcpyDeviceToHost, st));
  CG_CUDA(ctx, cudaMemcpyAsync(out_T, d_T, (size_t)H * 128, cudaMemcpyDeviceToHost, st));
  CG_CUDA(ctx, cudaMemcpyAsync(out_valid, d_valid, (size_t)H, cudaMemcpyDeviceToHost, st));
  CG_CUDA(ctx, cudaStreamSynchronize(st));
  return CG_OK;
}
