// cg_linear.cu -- batched fully-connected layers and the small epilogue kernels
// of the PointNet heads (fp32 SIMT; < 1% of the path's FLOPs, SURVEY.md 8a N3-N6).
//
//   Y[M][N] = act( X[M][K] @ Wt[K][N] + bias[row / bias_row_div][N] )
//
// replaces nn.Linear / nn.Conv1d(k=1) + folded BatchNorm + ReLU of
// pointnet2.py:176-183, :214-221, :295-298 and the PointNetSeg head :323-327.
#include "cg_net.cuh"

namespace {

constexpr int BM = 64, BN = 64, BK = 16;

__global__ void __launch_bounds__(256) linear_kernel(const float *__restrict__ X, int M, int K,
                                                      const float *__restrict__ Wt,
                                                      const float *__restrict__ bias, int N, int relu,
                                                      int bias_row_div, int x_is_keys,
                                                      float *__restrict__ Y) {
  __shared__ __align__(16) float xs[BK][BM + 4];
  __shared__ __align__(16) float ws[BK][BN + 4];
  const long long tile = cg_row_tile();
  if (tile * BM >= M) return;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = (int)tile * BM, n0 = blockIdx.x * BN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += BK) {
    // X tile: 64 rows x 16 k  (each thread: one row, 4 consecutive k)
    {
      const int r = tid >> 2, kq = (tid & 3) * 4;
      const int m = m0 + r;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (m < M) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const int k = k0 + kq + q;
          if (k < K) {
            float f = X[(size_t)m * K + k];
            if (x_is_keys) f = cg_key2f(__float_as_uint(f));
            v[q] = f;
          }
        }
      }
#pragma unroll
      for (int q = 0; q < 4; q++) xs[kq + q][r] = v[q];
    }
    // W tile: 16 k x 64 n  (each thread: one k row, 4 consecutive n)
    {
      const int r = tid >> 4, nq = (tid & 15) * 4;
      const int k = k0 + r;
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const int n = n0 + nq + q;
        ws[r][nq + q] = (k < K && n < N) ? Wt[(size_t)k * N + n] : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; kk++) {
      const float4 a = *reinterpret_cast<const float4 *>(&xs[kk][ty * 4]);
      const float4 b = *reinterpret_cast<const float4 *>(&ws[kk][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
    const float *brow = bias ? (bias + (size_t)(bias_row_div > 0 ? (m / bias_row_div) : 0) * N) : nullptr;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j] + (brow ? brow[n] : 0.f);
      if (relu) v = fmaxf(v, 0.f);
      Y[(size_t)m * N + n] = v;
    }
  }
}


// Larger register tile for the wide FC layers: 64 x 128 outputs per CTA, 4 x 8 per thread, BK = 16, global->register
// prefetch of the next k-tile while the current one is consumed from shared memory.
constexpr int LM = 64, LN = 128, LK = 16;

__global__ void __launch_bounds__(256) linear_wide_kernel(const float *__restrict__ X, int M, int K,
                                                           const float *__restrict__ Wt,
                                                           const float *__restrict__ bias, int N, int relu,
                                                           int bias_row_div, int x_is_keys,
                                                           float *__restrict__ Y) {
  __shared__ __align__(16) float xs[2][LK][LM + 4];
  __shared__ __align__(16) float ws[2][LK][LN + 4];
  const long long tile = cg_row_tile();
  if (tile * LM >= M) return;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;            // 16 x 16 threads: ty -> 4 rows, tx -> 8 cols (2 x float4)
  const int m0 = (int)tile * LM, n0 = blockIdx.x * LN;
  float acc[4][8];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 8; j++) acc[i][j] = 0.f;
  // X tile 64 x 16: thread -> row (tid >> 2), 4 consecutive k ((tid & 3) * 4)
  const int xr = tid >> 2, xk = (tid & 3) * 4;
  // W tile 16 x 128: thread -> k row (tid >> 4), 8 consecutive n ((tid & 15) * 8)
  const int wr = tid >> 4, wn = (tid & 15) * 8;
  const bool xrow_ok = (m0 + xr) < M;
  const float *xp = X + (size_t)(m0 + xr) * K + xk;
  float4 xreg = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 wreg0 = xreg, wreg1 = xreg;
  const bool vecN = ((N & 3) == 0);
  auto gload = [&](int k0) {
    if (xrow_ok) {
      xreg = *reinterpret_cast<const float4 *>(xp + k0);
      if (x_is_keys) {
        xreg.x = cg_key2f(__float_as_uint(xreg.x)); xreg.y = cg_key2f(__float_as_uint(xreg.y));
        xreg.z = cg_key2f(__float_as_uint(xreg.z)); xreg.w = cg_key2f(__float_as_uint(xreg.w));
      }
    }
    const float *wp = Wt + (size_t)(k0 + wr) * N + n0 + wn;
    if (vecN && n0 + wn + 8 <= N) {
      wreg0 = *reinterpret_cast<const float4 *>(wp);
      wreg1 = *reinterpret_cast<const float4 *>(wp + 4);
    } else {
      float t[8];
#pragma unroll
      for (int q = 0; q < 8; q++) t[q] = (n0 + wn + q < N) ? wp[q] : 0.f;
      wreg0 = make_float4(t[0], t[1], t[2], t[3]);
      wreg1 = make_float4(t[4], t[5], t[6], t[7]);
    }
  };
  auto sstore = [&](int buf) {
    xs[buf][xk + 0][xr] = xreg.x; xs[buf][xk + 1][xr] = xreg.y; xs[buf][xk + 2][xr] = xreg.z; xs[buf][xk + 3][xr] = xreg.w;
    *reinterpret_cast<float4 *>(&ws[buf][wr][wn]) = wreg0;
    *reinterpret_cast<float4 *>(&ws[buf][wr][wn + 4]) = wreg1;
  };
  gload(0);
  sstore(0);
  __syncthreads();
  const int nk = K / LK;
  for (int kt = 0; kt < nk; kt++) {
    const int buf = kt & 1;
    if (kt + 1 < nk) gload((kt + 1) * LK);
#pragma unroll
    for (int kk = 0; kk < LK; kk++) {
      const float4 a = *reinterpret_cast<const float4 *>(&xs[buf][kk][ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4 *>(&ws[buf][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4 *>(&ws[buf][kk][64 + tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kt + 1 < nk) sstore(buf ^ 1);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
    const float *brow = bias ? (bias + (size_t)(bias_row_div > 0 ? (m / bias_row_div) : 0) * N) : nullptr;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const int n = n0 + ((j < 4) ? (tx * 4 + j) : (64 + tx * 4 + j - 4));
      if (n >= N) continue;
      float v = acc[i][j] + (brow ? brow[n] : 0.f);
      if (relu) v = fmaxf(v, 0.f);
      Y[(size_t)m * N + n] = v;
    }
  }
}


// Few-row variant (M <= 8: the per-scene NUNOCS heads, B = 1): 16 output columns per CTA, K split over 64 thread
// groups whose partial sums meet in shared memory -- latency-bound GEMV work that the tiled kernels serialise badly
// (a 1024->512 layer is 32 CTAs of 16 dependent loop steps; with 64 columns x 16 slices it was 8 CTAs of 64 steps).
constexpr int RM = CG_FC_FEW_ROWS;
constexpr int RQ = 4;     // column quads per CTA
constexpr int RS = 64;    // k-slices per CTA
constexpr int RC = RQ * 4;

// With groups.n > 0 one launch runs groups.n independent row groups, blockIdx.y picking one: group g is rows
// (groups.g[g] >> 4) .. + (groups.g[g] & 15) - 1 of X and Y, and each of its rows gets the sums a launch on that group
// alone gives (row m of a group uses bias row m / bias_row_div counted from the group's first row).
__global__ void __launch_bounds__(256) linear_rows_kernel(const float *__restrict__ X, int M, int K,
                                                           const float *__restrict__ Wt,
                                                           const float *__restrict__ bias, int N, int relu,
                                                           int bias_row_div, int x_is_keys,
                                                           float *__restrict__ Y,
                                                           const __grid_constant__ cg_fc_row_groups groups) {
  __shared__ float red[RS][RM][RC + 1];
  if (groups.n > 0) {
    const int32_t g = groups.g[blockIdx.y];
    X += (size_t)(g >> 4) * K;
    Y += (size_t)(g >> 4) * N;
    M = g & 15;
  }
  const int tid = threadIdx.x;
  const int nq = tid % RQ, ks = tid / RQ;          // RQ column quads x RS k-slices
  const int n = blockIdx.x * RC + nq * 4;
  float acc[RM][4];
#pragma unroll
  for (int m = 0; m < RM; m++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[m][j] = 0.f;
  const int kper = (K + RS - 1) / RS;
  const int k0 = ks * kper, k1 = min(K, k0 + kper);
  const bool vec = ((N & 3) == 0) && (n + 4 <= N);
#pragma unroll 4
  for (int k = k0; k < k1; k++) {
    float w[4];
    if (vec) {
      const float4 t = *reinterpret_cast<const float4 *>(Wt + (size_t)k * N + n);
      w[0] = t.x; w[1] = t.y; w[2] = t.z; w[3] = t.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; j++) w[j] = (n + j < N) ? Wt[(size_t)k * N + n + j] : 0.f;
    }
#pragma unroll
    for (int m = 0; m < RM; m++) {
      if (m < M) {
        float x = X[(size_t)m * K + k];
        if (x_is_keys) x = cg_key2f(__float_as_uint(x));
#pragma unroll
        for (int j = 0; j < 4; j++) acc[m][j] = fmaf(x, w[j], acc[m][j]);
      }
    }
  }
#pragma unroll
  for (int m = 0; m < RM; m++)
#pragma unroll
    for (int j = 0; j < 4; j++) red[ks][m][nq * 4 + j] = acc[m][j];
  __syncthreads();
  for (int o = tid; o < M * RC; o += 256) {
    const int m = o / RC, c = o % RC;
    const int col = blockIdx.x * RC + c;
    if (col >= N) continue;
    float v = 0.f;
#pragma unroll 8
    for (int s2 = 0; s2 < RS; s2++) v += red[s2][m][c];
    if (bias) v += bias[(size_t)(bias_row_div > 0 ? (m / bias_row_div) : 0) * N + col];
    if (relu) v = fmaxf(v, 0.f);
    Y[(size_t)m * N + col] = v;
  }
}

// softmax over C <= 32 classes, one warp per row (predicter.py:86-90).  The label is the argmax of the probabilities
// as written, the lowest class winning a tie, as the reference takes it (softmax, then argmax): logits closer than
// expf resolves, such as 0 and 1e-30, give equal probabilities and so the lower class, not the larger logit.
__global__ void softmax_kernel(const float *__restrict__ logits, int B, int C, float *__restrict__ probs,
                               int32_t *__restrict__ label) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= B) return;
  const float v = (lane < C) ? logits[(size_t)row * C + lane] : -INFINITY;
  float m = v;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  const float e = (lane < C) ? expf(v - m) : 0.f;
  float s = e;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float p = e / s;
  if (lane < C && probs) probs[(size_t)row * C + lane] = p;
  if (label) {
    float pm = (lane < C) ? p : -1.f;   // lanes past C never win: every probability is >= 0
    int am = lane;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float op = __shfl_xor_sync(0xffffffffu, pm, o);
      const int oa = __shfl_xor_sync(0xffffffffu, am, o);
      if (op > pm || (op == pm && oa < am)) { pm = op; am = oa; }
    }
    if (lane == 0) label[row] = am;
  }
}

// NUNOCS post-processing (predicter.py:144-150): one warp per (point, axis)
__global__ void nunocs_post_kernel(const float *__restrict__ logits, int P, int bins,
                                   float *__restrict__ coords, float *__restrict__ conf_z,
                                   int32_t *__restrict__ out_bins) {
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= P * 3) return;
  const int p = w / 3, ax = w % 3;
  const float *row = logits + (size_t)p * 3 * bins + (size_t)ax * bins;
  float m = -INFINITY;
  int am = 0x7fffffff;
  for (int k = lane; k < bins; k += 32) {
    const float v = row[k];
    if (v > m) { m = v; am = k; }   // strict: first maximum wins inside a lane
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const int oa = __shfl_xor_sync(0xffffffffu, am, o);
    if (om > m || (om == m && oa < am)) { m = om; am = oa; }
  }
  if (lane == 0) {
    const float res = 1.0f / (float)bins;          // bin_resolution, predicter.py:145
    if (coords) coords[(size_t)p * 3 + ax] = __fsub_rn(__fmul_rn((float)am, res), 0.5f);  // :146 then :150, two roundings
    if (out_bins) out_bins[(size_t)p * 3 + ax] = am;
  }
  if (ax == 2 && conf_z) {
    float s = 0.f;
    for (int k = lane; k < bins; k += 32) s += expf(row[k] - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) conf_z[p] = 1.0f / s;           // softmax prob at the argmax, :147-148
  }
}

}  // namespace

int cg_linear_launch(cg_ctx *ctx, const cg_layer &L, const float *X, int M, float *Y, unsigned flags,
                     const float *row_bias, int rows_per_bias) {
  const int K = L.K, N = L.C;
  CG_REQUIRE(ctx, M > 0 && K > 0 && N > 0, "linear: bad shape");
  const float *Wt = L.Wt, *bias = row_bias ? row_bias : L.b;
  const int relu = (flags & CG_FC_RELU) != 0, x_is_keys = (flags & CG_FC_KEYS) != 0, bias_row_div = rows_per_bias;
  if (ctx->engine >= 1 && L.tc && M >= 64)
    return cg_linear_tc_launch(ctx, X, M, K, L.tc, bias, N, relu, bias_row_div, x_is_keys, Y);
  if (M <= RM) {
    cg_fc_row_groups one;
    one.n = 0;
    linear_rows_kernel<<<(N + RC - 1) / RC, 256, 0, ctx->stream>>>(X, M, K, Wt, bias, N, relu, bias_row_div, x_is_keys, Y,
                                                                   one);
    CG_LAUNCH_CHECK(ctx);
    return CG_OK;
  }
  const long wide_ctas = (long)((N + LN - 1) / LN) * ((M + LM - 1) / LM);
  if (N >= 128 && (K % LK) == 0 && (K % 4) == 0 && wide_ctas >= ctx->num_sms) {
    const dim3 gridw = cg_row_tile_grid((N + LN - 1) / LN, ((long long)M + LM - 1) / LM);
    linear_wide_kernel<<<gridw, 256, 0, ctx->stream>>>(X, M, K, Wt, bias, N, relu, bias_row_div, x_is_keys, Y);
    CG_LAUNCH_CHECK(ctx);
    return CG_OK;
  }
  const dim3 grid = cg_row_tile_grid((N + BN - 1) / BN, ((long long)M + BM - 1) / BM);
  linear_kernel<<<grid, 256, 0, ctx->stream>>>(X, M, K, Wt, bias, N, relu, bias_row_div, x_is_keys, Y);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

int cg_linear_launch_groups(cg_ctx *ctx, const cg_layer &L, const float *X, const int32_t *rows, int n_groups, float *Y,
                            unsigned flags) {
  const int K = L.K, N = L.C;
  CG_REQUIRE(ctx, K > 0 && N > 0 && n_groups > 0, "linear_groups: bad shape");
  const int relu = (flags & CG_FC_RELU) != 0, x_is_keys = (flags & CG_FC_KEYS) != 0;
  cg_fc_row_groups few;
  few.n = 0;
  auto flush = [&]() -> int {
    if (few.n == 0) return CG_OK;
    linear_rows_kernel<<<dim3((N + RC - 1) / RC, few.n), 256, 0, ctx->stream>>>(X, 0, K, L.Wt, L.b, N, relu, 0,
                                                                              x_is_keys, Y, few);
    CG_LAUNCH_CHECK(ctx);
    few.n = 0;
    return CG_OK;
  };
  long long total = 0;
  for (int i = 0; i < n_groups; i++) {
    CG_REQUIRE(ctx, rows[i] > 0, "linear_groups: empty group");
    total += rows[i];
  }
  CG_REQUIRE(ctx, total < (1 << 27), "linear_groups: 2^27 rows or more");
  int r0 = 0, rc;
  for (int i = 0; i < n_groups; r0 += rows[i++]) {
    const int m = rows[i];
    if (m <= RM) {   // the kernel cg_linear_launch takes for m rows, m <= 8 (it never takes tensor cores below 64)
      few.g[few.n++] = (r0 << 4) | m;
      if (few.n == CG_FC_GROUPS_PER_LAUNCH && (rc = flush())) return rc;
    } else if ((rc = cg_linear_launch(ctx, L, X + (size_t)r0 * K, m, Y + (size_t)r0 * N, flags))) {
      return rc;
    }
  }
  return flush();
}

int cg_softmax_launch(cg_ctx *ctx, const float *logits, int B, int C, float *probs, int32_t *label) {
  CG_REQUIRE(ctx, C >= 1 && C <= 32, "softmax: 1 <= n_out <= 32");
  const int wpb = 8;
  softmax_kernel<<<(B + wpb - 1) / wpb, wpb * 32, 0, ctx->stream>>>(logits, B, C, probs, label);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

int cg_nunocs_post_launch(cg_ctx *ctx, const float *logits, int P, int bins, float *coords, float *conf_z,
                          int32_t *out_bins) {
  CG_REQUIRE(ctx, P > 0 && bins > 0, "nunocs_post: bad shape");
  const int wpb = 8;
  const long warps = (long)P * 3;
  nunocs_post_kernel<<<(unsigned)((warps + wpb - 1) / wpb), wpb * 32, 0, ctx->stream>>>(logits, P, bins, coords,
                                                                                     conf_z, out_bins);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}
