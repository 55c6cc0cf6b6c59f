// cg_cone.cu -- cone pose enumeration on the device (SURVEY.md 8f F3).
//
// Replaces the inner loops of dexnet/grasping/grasp_sampler.py::PointConeGraspSampler:
//   * sample_one_surface_point (:266-286): Rs = [R0] + [R0 @ R_sphere @ R_inplane for sphere_pts x in-plane angles];
//     R = normalizeRotation(R) (Utils.py:172-179: divide every column by its norm); for d in arange(0, hand_depth, step):
//     pose = [R | selected_surface + init_bite * R[:,0] + R[:,0] * d];
//   * sample_grasps (:191-203), center_ob_between_gripper: every pose is shifted along its y axis by the centre of the
//     object's extent in the grasp frame: pose = pose @ [I | (0, cy, 0)], cy = (max_y + min_y) / 2 of inv(pose) * points.
// The per-surface-point frame R0 (kd-tree ball query, normal scatter matrix, LAPACK eig: :227-263) stays on the host so
// that eigenvector signs are the reference's; this file is the part whose work grows with the number of poses.
//
// All arithmetic is float64 like the reference's numpy.  3x3 products are fma chains (numpy hands them to BLAS, whose
// summation order is not defined), so rotations built from sphere and in-plane tables are within a rounding bound of
// the exact product, not bit-exact; the column normalisation and the translation are evaluated in numpy's order with
// correctly rounded operations, so R0's own poses are numpy's bit for bit.  Centring inverts by cofactors where the
// reference calls np.linalg.inv: bounded, not bit-exact.  oracle/cone_ref.py derives the bounds, tests/test_cone_kernels.py
// checks them.  A float32 copy (what pybind narrows to when the poses enter filterGraspPose, common.h:60) is written
// alongside for cg_filter_grasp_pose_dev: the float64 pose narrowed, after centring too.
#include "cg_common.cuh"

namespace {

__device__ __forceinline__ void mm3(const double *A, const double *B, double *O) {
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++)
      O[r * 3 + c] = fma(A[r * 3 + 2], B[6 + c], fma(A[r * 3 + 1], B[3 + c], A[r * 3] * B[c]));
}

// one thread per (surface point s, rotation r): r == 0 is R0 itself, r >= 1 is (sphere (r-1)/NI, in-plane (r-1)%NI)
__global__ void cone_pose_kernel(const double *__restrict__ surf, const double *__restrict__ R0, int S,
                                 const double *__restrict__ Rsph, int NS, const double *__restrict__ Rinp, int NI,
                                 const double *__restrict__ depths, int ND, double init_bite, double *__restrict__ out64,
                                 float *__restrict__ out32) {
  const int NR = 1 + NS * NI;
  const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long)S * NR) return;
  const int s = (int)(t / NR), r = (int)(t % NR);
  double R[9];
  if (r == 0) {
    for (int k = 0; k < 9; k++) R[k] = R0[(size_t)s * 9 + k];
  } else {
    double T[9];
    mm3(R0 + (size_t)s * 9, Rsph + (size_t)((r - 1) / NI) * 9, T);   // (R0 @ R_sphere) @ R_inplane, left to right (:269)
    mm3(T, Rinp + (size_t)((r - 1) % NI) * 9, R);
  }
  for (int c = 0; c < 3; c++) {                                        // normalizeRotation, Utils.py:176-178
    const double x = R[c], y = R[3 + c], z = R[6 + c];
    const double n = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
    R[c] = x / n;
    R[3 + c] = y / n;
    R[6 + c] = z / n;
  }
  const double px = surf[(size_t)s * 3], py = surf[(size_t)s * 3 + 1], pz = surf[(size_t)s * 3 + 2];
  for (int k = 0; k < ND; k++) {
    const double d = depths[k];
    double P[16];
    for (int i = 0; i < 3; i++) {
      P[i * 4] = R[i * 3];
      P[i * 4 + 1] = R[i * 3 + 1];
      P[i * 4 + 2] = R[i * 3 + 2];
    }
    // selected_surface + init_bite*approach_dir + approach_dir*d, evaluated left to right (:279)
    P[3] = __dadd_rn(__dadd_rn(px, __dmul_rn(init_bite, R[0])), __dmul_rn(R[0], d));
    P[7] = __dadd_rn(__dadd_rn(py, __dmul_rn(init_bite, R[3])), __dmul_rn(R[3], d));
    P[11] = __dadd_rn(__dadd_rn(pz, __dmul_rn(init_bite, R[6])), __dmul_rn(R[6], d));
    P[12] = 0.0; P[13] = 0.0; P[14] = 0.0; P[15] = 1.0;
    const size_t o = ((size_t)t * ND + k) * 16;
    for (int i = 0; i < 16; i++) out64[o + i] = P[i];
    if (out32)
      for (int i = 0; i < 16; i++) out32[o + i] = (float)P[i];
  }
}

constexpr int CT = 128;

// one CTA per pose: y extent of the object in the grasp frame, then shift the pose along its own y axis
__global__ void __launch_bounds__(CT) center_grasp_kernel(double *__restrict__ poses64, float *__restrict__ poses32, int P,
                                                          const double *__restrict__ pts, int M) {
  const int p = blockIdx.x, tid = threadIdx.x;
  double *T = poses64 + (size_t)p * 16;
  const double yx = T[1], yy = T[5], yz = T[9];          // second column: the grasp frame's y axis in the camera frame
  const double tx = T[3], ty = T[7], tz = T[11];
  // second row of inv(R) by cofactors: the reference inverts the pose numerically (:194) and its frames are not always
  // orthonormal (see grasp_sampler.cone_frames), so the transpose is not a substitute
  const double a = T[0], b = T[1], c = T[2], d = T[4], e = T[5], f = T[6], g = T[8], h = T[9], i = T[10];
  const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
  const double ix = (f * g - d * i) / det, iy = (a * i - c * g) / det, iz = (c * d - a * f) / det;
  double lo = 1e300, hi = -1e300;
  for (int j = tid; j < M; j += CT) {
    const double *q = pts + (size_t)j * 3;
    const double y = fma(iz, q[2] - tz, fma(iy, q[1] - ty, ix * (q[0] - tx)));
    lo = fmin(lo, y);
    hi = fmax(hi, y);
  }
  __shared__ double slo[CT / 32], shi[CT / 32];
  for (int o = 16; o; o >>= 1) {
    lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((tid & 31) == 0) { slo[tid >> 5] = lo; shi[tid >> 5] = hi; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < CT / 32; w++) { lo = fmin(lo, slo[w]); hi = fmax(hi, shi[w]); }
    const double cy = (hi + lo) / 2;                       // (max + min) / 2, :197
    const double nx = fma(yx, cy, tx), ny = fma(yy, cy, ty), nz = fma(yz, cy, tz);
    T[3] = nx; T[7] = ny; T[11] = nz;
    if (poses32) {
      float *F = poses32 + (size_t)p * 16;
      F[3] = (float)nx; F[7] = (float)ny; F[11] = (float)nz;
    }
  }
}

}  // namespace

extern "C" int cg_cone_poses_dev(cg_ctx *ctx, const double *surface_pts, const double *R0, int S, const double *R_sphere,
                                 int NS, const double *R_inplane, int NI, const double *depths, int ND, double init_bite,
                                 double *out_poses64, float *out_poses32) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, surface_pts && R0 && depths && out_poses64 && S > 0 && ND > 0 && NS >= 0 && NI >= 0, "cone_poses: bad arguments");
  CG_REQUIRE(ctx, (NS == 0 || NI == 0) || (R_sphere && R_inplane), "cone_poses: rotation tables missing");
  // each factor is checked before the next product, so no product of int arguments can overflow 64 bits
  const long long lim = 1LL << 31, nr = 1 + (long long)NS * NI, n = nr < lim ? (long long)S * nr : lim;
  CG_REQUIRE(ctx, n < lim && n * ND < lim, "cone_poses: 2^31 poses or more in one call");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  cone_pose_kernel<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(surface_pts, R0, S, R_sphere, NS, R_inplane, NI, depths, ND,
                                                                        init_bite, out_poses64, out_poses32);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_center_grasps_dev(cg_ctx *ctx, double *poses64, float *poses32, int P, const double *pts, int M) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, poses64 && pts && P >= 0 && M > 0, "center_grasps: bad arguments");
  if (P == 0) return CG_OK;
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  center_grasp_kernel<<<P, CT, 0, ctx->stream>>>(poses64, poses32, P, pts, M);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}
