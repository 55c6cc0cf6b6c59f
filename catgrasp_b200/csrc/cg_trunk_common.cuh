// cg_trunk_common.cuh -- device helpers shared by the fp32-SIMT trunk (engine 0) and the
// tensor-core trunk (engines 1-3): register-tiled fp32 layers over k-major shared-memory tiles, the
// float64 pose inverse and transform of an input row, its T3 product, and cp.async wrappers.
#pragma once
#include "cg_net.cuh"

namespace cg_trunk {

constexpr int TP = 128;      // points per tile
constexpr int NT = 256;      // threads per CTA
__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
  uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// out[C][TP] = act(W^T h + b): h is [K][TP], w is [K][C]; NC = channels per thread (4 or 8).
template <int K, int C, int NC, bool RELU, bool BIAS>
__device__ __forceinline__ void mlp_layer(const float *__restrict__ hin, const float *__restrict__ w,
                                          const float *__restrict__ bias, float *__restrict__ hout,
                                          int tx, int ty) {
  static_assert(C == 16 * NC, "channel tiling");
  float acc[8][NC];
#pragma unroll
  for (int i = 0; i < 8; i++)
#pragma unroll
    for (int j = 0; j < NC; j++) acc[i][j] = 0.f;
  const int p0 = ty * 4, p1 = 64 + ty * 4;
  const int c0 = tx * 4, c1 = 64 + tx * 4;
#pragma unroll 4
  for (int k = 0; k < K; k++) {
    float a[8], b[NC];
    *reinterpret_cast<float4 *>(&a[0]) = *reinterpret_cast<const float4 *>(&hin[k * TP + p0]);
    *reinterpret_cast<float4 *>(&a[4]) = *reinterpret_cast<const float4 *>(&hin[k * TP + p1]);
    *reinterpret_cast<float4 *>(&b[0]) = *reinterpret_cast<const float4 *>(&w[k * C + c0]);
    if (NC == 8) *reinterpret_cast<float4 *>(&b[4]) = *reinterpret_cast<const float4 *>(&w[k * C + c1]);
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
      for (int j = 0; j < NC; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
  }
#pragma unroll
  for (int j = 0; j < NC; j++) {
    const int c = (j < 4) ? (c0 + j) : (c1 + j - 4);
    const float bb = BIAS ? bias[c] : 0.f;
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
      v[i] = acc[i][j] + bb;
      if (RELU) v[i] = fmaxf(v[i], 0.f);
    }
    *reinterpret_cast<float4 *>(&hout[c * TP + p0]) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4 *>(&hout[c * TP + p1]) = make_float4(v[4], v[5], v[6], v[7]);
  }
}

// 3x3 inverse by cofactors in float64 + tinv = -Rinv t  (np.linalg.inv of a pose, dataset_grasp.py:69-70)
static __device__ void pose_inverse(const double *P, double *out) {
  const double a = P[0], b = P[1], c = P[2], d = P[4], e = P[5], f = P[6], g = P[8], h = P[9], i = P[10];
  const double A = e * i - f * h, Bc = -(d * i - f * g), Cc = d * h - e * g;
  const double det = a * A + b * Bc + c * Cc;
  const double r = 1.0 / det;
  out[0] = A * r;  out[1] = -(b * i - c * h) * r;  out[2] = (b * f - c * e) * r;
  out[3] = Bc * r; out[4] = (a * i - c * g) * r;   out[5] = -(a * f - c * d) * r;
  out[6] = Cc * r; out[7] = -(a * h - b * g) * r;  out[8] = (a * e - b * d) * r;
  const double tx = P[3], ty = P[7], tz = P[11];
  out[9] = -(out[0] * tx + out[1] * ty + out[2] * tz);
  out[10] = -(out[3] * tx + out[4] * ty + out[5] * tz);
  out[11] = -(out[6] * tx + out[7] * ty + out[8] * tz);
}

// One cloud row (x, y, z, nx, ny, nz) into the candidate's frame in float64: w[0..2] = Rinv xyz + tinv,
// w[3..5] = Rinv nrm, with R = pose_inverse's output.  Both trunks then normalise w and narrow it to float, but not
// in the same way: engine 0 divides by (std + 1e-15), engines 1-3 multiply by its reciprocal, so engine 0's input
// rows can differ from the other engines' in the last bit.
__device__ __forceinline__ void pose_transform(const double *R, double x, double y, double z, double nx, double ny,
                                               double nz, double *w) {
  w[0] = R[0] * x + R[1] * y + R[2] * z + R[9];
  w[1] = R[3] * x + R[4] * y + R[5] * z + R[10];
  w[2] = R[6] * x + R[7] * y + R[8] * z + R[11];
  w[3] = R[0] * nx + R[1] * ny + R[2] * nz;
  w[4] = R[3] * nx + R[4] * ny + R[5] * nz;
  w[5] = R[6] * nx + R[7] * ny + R[8] * nz;
}

// xyz @ T3 (pointnet2.py:248) of one input row v[6]; the normals pass through (:245-250)
__device__ __forceinline__ void apply_t3(const float *t3, float *v) {
  const float x = v[0], y = v[1], z = v[2];
  v[0] = fmaf(z, t3[6], fmaf(y, t3[3], x * t3[0]));
  v[1] = fmaf(z, t3[7], fmaf(y, t3[4], x * t3[1]));
  v[2] = fmaf(z, t3[8], fmaf(y, t3[5], x * t3[2]));
}


}  // namespace cg_trunk
