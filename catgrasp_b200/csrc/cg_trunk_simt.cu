// cg_trunk_simt.cu -- fp32 SIMT "trunk" kernel (engine 0).
//
// One trunk = the per-point shared-MLP chain of a PointNet block followed by
// the max over points, fused so that no (N x C) activation ever reaches HBM:
//
//   input rows (built in-kernel from cloud + pose + ids, or read directly)
//     -> [xyz @ T3]                      pointnet2.py:245-250
//     -> conv 6->64 + BN + ReLU          pointnet2.py:171 / :252
//     -> [conv 64->64 + BN + ReLU | h @ T64]   pointnet2.py:209 / :255-259
//     -> conv 64->128 + BN + ReLU        pointnet2.py:172 / :210 / :263
//     -> conv 128->1024 + BN [+ ReLU]    pointnet2.py:173 / :211 / :264
//     -> max over points                 pointnet2.py:174 / :212 / :265
//
// The per-candidate input build restates GraspDataset.transform
// (dataset_grasp.py:63-91) in float64 and narrows to fp32 exactly where the
// reference does (predicter.py:84 `.cuda().float()`).
//
// Tiling: one CTA = 256 threads = one tile of 128 points; every layer is a
// register-tiled (8 points x 8|4 channels per thread) fp32 GEMM whose operands
// live in shared memory in k-major order; the 128->1024 layer streams its
// weights through a 3-stage cp.async ring in 32-row slices and reduces its
// output straight into a shared running max.
#include "cg_trunk_common.cuh"

namespace {
using namespace cg_trunk;

constexpr int KS = 32;       // W3 rows per ring stage
constexpr int NSTAGE = 3;
constexpr int RING_FLOATS = NSTAGE * KS * 128;  // 12288

struct SmemLayout {
  float in_s[8 * TP];          //  4 KB   [k][p]
  float regA[64 * TP];         // 32 KB   regA ++ regC = h2 [128][TP]
  float regC[64 * TP];         // 32 KB
  float regB[64 * TP];         // 32 KB
  float ring[RING_FLOATS];     // 48 KB
  uint32_t gmax_s[1024];       //  4 KB
  float w0[6 * 64];
  float bias0[64];
  float bias1[64];
  float bias2[128];
  double pinv[12];             // Rinv (9) + tinv (3)
  double mean[6];
  double sden[6];
  float T3[9];
};

__device__ __forceinline__ void load_slice(float *ring, int s, const float *__restrict__ W3, int tid) {
  // slice s: chunk = s>>2 (128 channels), rows (s&3)*32 .. +32 of W3t [128][1024]
  const int stage = s % NSTAGE;
  const int chunk = s >> 2, k0 = (s & 3) * KS;
  float *dst = ring + stage * (KS * 128);
  const float *src = W3 + (size_t)k0 * 1024 + chunk * 128;
#pragma unroll
  for (int it = 0; it < (KS * 128) / (NT * 4); it++) {
    const int e = (it * NT + tid) * 4;   // float index inside the slice
    const int r = e >> 7, c = e & 127;
    cp_async16(dst + e, src + (size_t)r * 1024 + c);
  }
}

__global__ void __launch_bounds__(NT, 1) trunk_simt_kernel(const cg_trunk_args a, int tiles_per_cta) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SmemLayout &S = *reinterpret_cast<SmemLayout *>(smem_raw);
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.y;
  const int N = a.N;
  const int ntiles = (N + TP - 1) / TP;
  const int tile_begin = blockIdx.x * tiles_per_cta;
  const int tile_end = min(ntiles, tile_begin + tiles_per_cta);
  if (tile_begin >= tile_end) return;

  // ---- per-CTA constants -------------------------------------------------
  for (int i = tid; i < 1024; i += NT) S.gmax_s[i] = 0u;
  for (int i = tid; i < 6 * 64; i += NT) S.w0[i] = a.l0.Wt[i];
  if (tid < 64) {
    S.bias0[tid] = a.l0.b[tid];
    S.bias1[tid] = (a.stage1_mode == 1) ? a.l1.b[tid] : 0.f;
  }
  if (tid < 128) S.bias2[tid] = a.l2.b[tid];
  if (tid < 9) S.T3[tid] = a.T3 ? a.T3[b * 9 + tid] : 0.f;
  if (a.in.x_direct == nullptr) {
    if (tid == 0) pose_inverse(a.in.poses + (size_t)b * 16, S.pinv);
    if (tid < 6) {
      S.mean[tid] = a.in.mean ? a.in.mean[tid] : 0.0;
      S.sden[tid] = a.in.stdv ? (a.in.stdv[tid] + 1e-15) : 1.0;
    }
  }
  __syncthreads();

  for (int tile = tile_begin; tile < tile_end; tile++) {
    // ---- stage W1 / W2 into the ring area (ring is idle here) -------------
    float *w1s = S.ring;          // [64][64]
    float *w2s = S.ring + 4096;   // [64][128]
    if (a.stage1_mode != 0) {
      const float *src = (a.stage1_mode == 1) ? a.l1.Wt : (a.T64 + (size_t)b * 4096);
      for (int e = tid * 4; e < 4096; e += NT * 4) cp_async16(w1s + e, src + e);
    }
    for (int e = tid * 4; e < 8192; e += NT * 4) cp_async16(w2s + e, a.l2.Wt + e);
    cp_async_commit();

    // ---- build the (128 x 6) input tile -----------------------------------
    if (tid < TP) {
      int n = tile * TP + tid;
      if (n >= N) n = N - 1;  // duplicate a valid point: cannot change a max
      float v[6];
      if (a.in.x_direct) {
        const float *xr = a.in.x_direct + ((size_t)b * N + n) * 6;
#pragma unroll
        for (int k = 0; k < 6; k++) v[k] = xr[k];
      } else {
        const int id = a.in.ids ? a.in.ids[(size_t)b * N + n] : n;
        const double *px = a.in.cloud_xyz + (size_t)id * 3;
        const double *pn = a.in.cloud_nrm + (size_t)id * 3;
        const double x = px[0], y = px[1], z = px[2];
        const double nx = pn[0], ny = pn[1], nz = pn[2];
        double w[6];
        pose_transform(S.pinv, x, y, z, nx, ny, nz, w);
#pragma unroll
        for (int k = 0; k < 6; k++) v[k] = (float)((w[k] - S.mean[k]) / S.sden[k]);
      }
      if (a.T3) apply_t3(S.T3, v);
#pragma unroll
      for (int k = 0; k < 6; k++) S.in_s[k * TP + tid] = v[k];
    }
    __syncthreads();

    // ---- stage 0: 6 -> 64 ---------------------------------------------------
    float *h0 = (a.stage1_mode != 0) ? S.regA : S.regB;
    mlp_layer<6, 64, 4, true, true>(S.in_s, S.w0, S.bias0, h0, tx, ty);
    cp_async_wait<0>();
    __syncthreads();

    // ---- stage 1: optional 64 -> 64 ----------------------------------------
    if (a.stage1_mode == 1) {
      mlp_layer<64, 64, 4, true, true>(S.regA, w1s, S.bias1, S.regB, tx, ty);
      __syncthreads();
    } else if (a.stage1_mode == 2) {
      mlp_layer<64, 64, 4, false, false>(S.regA, w1s, S.bias1, S.regB, tx, ty);
      __syncthreads();
    }
    if (a.pf_out) {  // PointNetSeg point feature (pointnet2.py:261)
      const int p = tid & (TP - 1);
      const int n = tile * TP + p;
      if (n < N) {
        float *dst = a.pf_out + ((size_t)b * N + n) * 64;
        for (int c = (tid >> 7) * 4; c < 64; c += 8) {
          float4 o = make_float4(S.regB[(c + 0) * TP + p], S.regB[(c + 1) * TP + p],
                                 S.regB[(c + 2) * TP + p], S.regB[(c + 3) * TP + p]);
          *reinterpret_cast<float4 *>(dst + c) = o;
        }
      }
    }

    // ---- stage 2: 64 -> 128, output h2 = regA ++ regC ------------------------
    mlp_layer<64, 128, 8, true, true>(S.regB, w2s, S.bias2, S.regA, tx, ty);
    __syncthreads();  // h2 complete; ring (w1s/w2s) free

    // ---- stage 3: 128 -> 1024 streamed, fused max ----------------------------
    const float *h2 = S.regA;
    load_slice(S.ring, 0, a.l3.Wt, tid);
    cp_async_commit();
    load_slice(S.ring, 1, a.l3.Wt, tid);
    cp_async_commit();
    float acc[8][8];
    const int p0 = ty * 4, p1 = 64 + ty * 4;
    const int c0 = tx * 4, c1 = 64 + tx * 4;
    for (int s = 0; s < 32; s++) {
      cp_async_wait<NSTAGE - 2>();
      __syncthreads();
      if (s + NSTAGE - 1 < 32) load_slice(S.ring, s + NSTAGE - 1, a.l3.Wt, tid);
      cp_async_commit();
      const int ks = s & 3;
      if (ks == 0) {
#pragma unroll
        for (int i = 0; i < 8; i++)
#pragma unroll
          for (int j = 0; j < 8; j++) acc[i][j] = 0.f;
      }
      const float *w = S.ring + (s % NSTAGE) * (KS * 128);
      const float *hh = h2 + ks * KS * TP;
#pragma unroll 8
      for (int kk = 0; kk < KS; kk++) {
        float av[8], bv[8];
        *reinterpret_cast<float4 *>(&av[0]) = *reinterpret_cast<const float4 *>(&hh[kk * TP + p0]);
        *reinterpret_cast<float4 *>(&av[4]) = *reinterpret_cast<const float4 *>(&hh[kk * TP + p1]);
        *reinterpret_cast<float4 *>(&bv[0]) = *reinterpret_cast<const float4 *>(&w[kk * 128 + c0]);
        *reinterpret_cast<float4 *>(&bv[4]) = *reinterpret_cast<const float4 *>(&w[kk * 128 + c1]);
#pragma unroll
        for (int i = 0; i < 8; i++)
#pragma unroll
          for (int j = 0; j < 8; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      if (ks == 3) {
        const int chunk = s >> 2;
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const int c = chunk * 128 + ((j < 4) ? (c0 + j) : (c1 + j - 4));
          float m = acc[0][j];
#pragma unroll
          for (int i = 1; i < 8; i++) m = fmaxf(m, acc[i][j]);
          m += __ldg(&a.l3.b[c]);  // bias is constant over points: add after the max
          if (a.relu3) m = fmaxf(m, 0.f);
          m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
          if ((tid & 31) < 16) atomicMax(&S.gmax_s[c], cg_f2key(m));
        }
      }
    }
    cp_async_wait<0>();
    __syncthreads();  // ring + h2 free for the next tile
  }

  for (int i = tid; i < 1024; i += NT) atomicMax(&a.gmax_keys[(size_t)b * 1024 + i], S.gmax_s[i]);
}

}  // namespace

int cg_trunk_launch_simt(cg_ctx *ctx, const cg_trunk_args &a) {
  CG_REQUIRE(ctx, a.B > 0 && a.N > 0, "trunk: B,N must be positive");
  CG_REQUIRE(ctx, a.B <= 65535, "trunk: B > 65535 must be chunked by the caller");
  static bool attr_set[CG_MAX_DEVICES] = {};   // the attribute is per device
  const size_t smem = sizeof(SmemLayout);
  if (!attr_set[ctx->device]) {
    CG_CUDA(ctx, cudaFuncSetAttribute(trunk_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set[ctx->device] = true;
  }
  const int ntiles = (a.N + TP - 1) / TP;
  // enough CTAs to fill the machine ~4x over; one CTA per candidate when B is large
  int splits = 1;
  while ((long)a.B * splits < 4L * ctx->num_sms && splits < ntiles) splits *= 2;
  const int tiles_per_cta = (ntiles + splits - 1) / splits;
  dim3 grid((ntiles + tiles_per_cta - 1) / tiles_per_cta, a.B);
  trunk_simt_kernel<<<grid, NT, smem, ctx->stream>>>(a, tiles_per_cta);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}
