// cg_pose.cuh -- the float32 pose arithmetic of the reference's filterGraspPose (my_cpp/common.cpp:159,190-197,216),
// shared by the collision filter (cg_collide.cu) and the IK pass (cg_ik.cu) so that both compose poses with the same
// operations in the same order.  Every operation is spelled with an explicit rounding intrinsic (no FMA contraction),
// which oracle/filter_ref.c and my_cpp._mm4_f32 reproduce bit for bit.
#pragma once

namespace {

__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }

// Eigen fixed-size 4x4 float product as compiled by the reference build (SSE2, no FMA):
// out(r,c) = ((a(r,0)b(0,c) + a(r,1)b(1,c)) + a(r,2)b(2,c)) + a(r,3)b(3,c)
__device__ void mm4(const float *A, const float *B, float *O) {
#pragma unroll
  for (int r = 0; r < 4; r++)
#pragma unroll
    for (int c = 0; c < 4; c++) {
      float s = mul(A[r * 4 + 0], B[0 * 4 + c]);
      s = add(s, mul(A[r * 4 + 1], B[1 * 4 + c]));
      s = add(s, mul(A[r * 4 + 2], B[2 * 4 + c]));
      s = add(s, mul(A[r * 4 + 3], B[3 * 4 + c]));
      O[r * 4 + c] = s;
    }
}

// Eigen normalize(): v /= sqrt(x*x + y*y + z*z)   (common.cpp:194-197)
__device__ void normalize_col(float *G, int col) {
  const float x = G[0 * 4 + col], y = G[1 * 4 + col], z = G[2 * 4 + col];
  const float n = __fsqrt_rn(add(add(mul(x, x), mul(y, y)), mul(z, z)));
  G[0 * 4 + col] = __fdiv_rn(x, n);
  G[1 * 4 + col] = __fdiv_rn(y, n);
  G[2 * 4 + col] = __fdiv_rn(z, n);
}

}  // namespace
