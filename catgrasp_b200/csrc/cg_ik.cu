// cg_ik.cu -- closed-form inverse kinematics of the KUKA iiwa14 with the free joint 2 fixed at 0, in float64, and the
// IK feasibility test of the reference's filterGraspPose (my_cpp/common.cpp:9-72, :214-226) as a post-pass over the
// collision filter's output.
//
// The chain: base -> shoulder 0.36 m, shoulder -> elbow 0.42 m, elbow -> wrist 0.40 m, wrist -> end effector 0.081 m;
// joint axes z, +y, z, -y, z, +y, z.  With joint 2 = 0 the shoulder (joints 0, 1) and the wrist (4, 5, 6) are
// spherical: the wrist centre p - 0.081 R z gives q0 (two branches), q3 (law of cosines, two signs) and q1; then
// R_03^T R = Rz(q4) Ry(q5) Rz(q6) gives the wrist angles (two branches).  oracle/ik_ref.py is the numpy twin (same
// steps and constants); the special cases reproduce the reference's generated ikfast solver, bisected against it
// (tests/golden/make_golden_ik.py, DESIGN.md X5).
//
// Branch slot b = 4*s + 2*e + w of the (8,7) solution block, unused slots NaN:
//   s = 0: q0 = atan2(y, x) of the wrist centre, s = 1: q0 + pi;  e = 0: q3 >= 0, e = 1: q3 < 0;
//   w = 0: q5 >= 0 (or the lumped singular solution), w = 1: the flipped wrist (q4 + pi, -q5, q6 + pi).
// Every angle is wrapped to [-pi, pi].
#include "cg_common.cuh"
#include "cg_pose.cuh"

namespace {

constexpr double D_BS = 0.36, D_SE = 0.42, D_EW = 0.40, D_WF = 0.081;
constexpr double PI = 3.141592653589793;
// ikfast returns no solution when the wrist centre lies within 1 mm of the joint-0 axis (bisected to 1e-3 m at three
// arm configurations); the pose is reachable, but the reference calls it IK-infeasible
constexpr double SHOULDER_BAND = 1e-3;
// the law-of-cosines value c3 is accepted up to 1e-7 beyond [-1, 1] and clamped (ikfast's sin/cos slack)
constexpr double REACH_SLACK = 1e-7;
// ikfast merges two solutions whose sine and cosine differ by less than 1e-6: the elbow pair +-q3 when |2 sin q3| < 1e-6
constexpr double ELBOW_MERGE = 1e-6;
// below this |sin q5| the wrist is singular: one solution per arm branch, q6 = 0 and q4 = q4 + q6 (q4 - q6 at q5 = pi)
// (arms with q5 <= 3e-7 mostly give 6 solutions in ikfast)
constexpr double WRIST_SINGULAR = 1e-6;
// from WRIST_SINGULAR up to this |sin q5| ikfast returns neither wrist solution of the arm branch: over 60 random arms
// the last q5 that lost the branch was 1.6e-3 .. 4.9e-3 (median 2.5e-3), and every arm lost it from 1e-5 to 2e-4
constexpr double WRIST_DROP = 2.5e-3;

// ikfast checks each solution against the input matrix, which the reference passes unchecked (a float32 product, maybe
// of a scaled or sheared pose): a solution is kept only when Rz(q4) Ry(q5) Rz(q6) reproduces R_03^T R to within this,
// entry by entry.  Tolerances from 1e-5 to 1e-4 all reproduce ikfast on the fixture and the filter cases; 3e-6 does not.
constexpr double ROT_RESIDUAL = 3e-5;

constexpr int IK_BLOCK = 128;

// max |Rz(q4) Ry(q5) Rz(q6) - M| over the 9 entries
__device__ double wrist_residual(double q4, double q5, double q6, const double *M) {
  double s4, c4, s5, c5, s6, c6;
  sincos(q4, &s4, &c4);
  sincos(q5, &s5, &c5);
  sincos(q6, &s6, &c6);
  const double W[9] = {c4 * c5 * c6 - s4 * s6, -c4 * c5 * s6 - s4 * c6, c4 * s5,
                       s4 * c5 * c6 + c4 * s6, -s4 * c5 * s6 + c4 * c6, s4 * s5,
                       -s5 * c6, s5 * s6, c5};
  double r = 0.0;
#pragma unroll
  for (int k = 0; k < 9; k++) r = fmax(r, fabs(W[k] - M[k]));
  return r;
}

struct IkLimits {
  double up[7], lo[7];
};

__device__ __forceinline__ double wrap(double a) {
  if (a > PI) a -= 2.0 * PI;
  if (a < -PI) a += 2.0 * PI;
  return a;
}

// One pose: rows 0..2 of ee_in_base (float32, widened).  Returns the number of slots whose 7 joints all satisfy
// lo[i] <= q[i] <= up[i]; writes the (8,7) block to sol when it is not null.
__device__ int iiwa14_ik_one(const float *T, const IkLimits &lim, double *sol) {
  double R[9], p[3];
  bool finite = true;
#pragma unroll
  for (int r = 0; r < 3; r++) {
#pragma unroll
    for (int c = 0; c < 3; c++) {
      R[r * 3 + c] = (double)T[r * 4 + c];
      finite = finite && isfinite(R[r * 3 + c]);
    }
    p[r] = (double)T[r * 4 + 3];
    finite = finite && isfinite(p[r]);
  }
  const double vx = p[0] - D_WF * R[2];
  const double vy = p[1] - D_WF * R[5];
  const double vz = (p[2] - D_WF * R[8]) - D_BS;
  const double rho = sqrt(vx * vx + vy * vy);
  double c3 = ((vx * vx + vy * vy + vz * vz) - (D_SE * D_SE + D_EW * D_EW)) / (2.0 * D_SE * D_EW);
  const bool ok = finite && rho >= SHOULDER_BAND && c3 >= -1.0 - REACH_SLACK && c3 <= 1.0 + REACH_SLACK;
  int count = 0;
  if (!ok) {
    if (sol)
      for (int k = 0; k < 56; k++) sol[k] = __longlong_as_double(0x7ff8000000000000LL);
    return 0;
  }
  c3 = fmin(fmax(c3, -1.0), 1.0);
  const double s3 = sqrt(1.0 - c3 * c3);
  const bool elbow_two = 2.0 * s3 >= ELBOW_MERGE;
  const double q0a = atan2(vy, vx);
  for (int s = 0; s < 2; s++) {
    const double q0 = s == 0 ? q0a : wrap(q0a + PI);
    const double r = s == 0 ? rho : -rho;
    double s0, c0;
    sincos(q0, &s0, &c0);
    for (int e = 0; e < 2; e++) {
      const double q3 = atan2(e == 0 ? s3 : -s3, c3);
      double sq3, cq3;
      sincos(q3, &sq3, &cq3);
      const double ux = -D_EW * sq3;
      const double uz = D_SE + D_EW * cq3;
      const double q1 = wrap(atan2(r, vz) - atan2(ux, uz));
      // M = R_03^T R, R_03 = Rz(q0) Ry(q1 - q3): rows of R_03^T are Ry(b)^T Rz(q0)^T
      double sb, cb;
      sincos(q1 - q3, &sb, &cb);
      const double a0[3] = {cb * c0, cb * s0, -sb}, a1[3] = {-s0, c0, 0.0}, a2[3] = {sb * c0, sb * s0, cb};
      double M[9];
#pragma unroll
      for (int c = 0; c < 3; c++) {
        M[0 * 3 + c] = a0[0] * R[0 * 3 + c] + a0[1] * R[1 * 3 + c] + a0[2] * R[2 * 3 + c];
        M[1 * 3 + c] = a1[0] * R[0 * 3 + c] + a1[1] * R[1 * 3 + c] + a1[2] * R[2 * 3 + c];
        M[2 * 3 + c] = a2[0] * R[0 * 3 + c] + a2[1] * R[1 * 3 + c] + a2[2] * R[2 * 3 + c];
      }
      const double s5 = sqrt(M[2] * M[2] + M[5] * M[5]);
      const double c5 = M[8];
      const bool sing = s5 < WRIST_SINGULAR;
      const bool drop = !sing && s5 < WRIST_DROP;
      const bool arm = e == 0 || elbow_two;
      const double q4g = atan2(M[5], M[2]), q5g = acos(fmin(fmax(c5, -1.0), 1.0)), q6g = atan2(M[7], -M[6]);
      for (int w = 0; w < 2; w++) {
        double q[7];
        q[0] = q0; q[1] = q1; q[2] = 0.0; q[3] = q3;
        if (w == 0 && sing) {
          q[4] = c5 >= 0.0 ? atan2(M[3], M[0]) : atan2(-M[3], -M[0]);
          q[5] = c5 >= 0.0 ? 0.0 : PI;
          q[6] = 0.0;
        } else if (w == 0) {
          q[4] = q4g; q[5] = q5g; q[6] = q6g;
        } else {
          q[4] = wrap(q4g + PI); q[5] = -q5g; q[6] = wrap(q6g + PI);
        }
        bool valid = arm && !drop && (w == 0 || !sing);
        if (valid) valid = wrist_residual(q[4], q[5], q[6], M) <= ROT_RESIDUAL;
        if (valid) {
          bool in = true;
#pragma unroll
          for (int k = 0; k < 7; k++) in = in && q[k] >= lim.lo[k] && q[k] <= lim.up[k];
          count += in;
        }
        if (sol) {
          const int slot = 4 * s + 2 * e + w;
#pragma unroll
          for (int k = 0; k < 7; k++) sol[slot * 7 + k] = valid ? q[k] : __longlong_as_double(0x7ff8000000000000LL);
        }
      }
    }
  }
  return count;
}

__global__ void __launch_bounds__(IK_BLOCK) ik_kernel(const float *__restrict__ ee, int Q, const IkLimits lim,
                                                      int8_t *__restrict__ out_count, double *__restrict__ out_sol) {
  const int i = blockIdx.x * IK_BLOCK + threadIdx.x;
  if (i >= Q) return;
  float T[12];
#pragma unroll
  for (int k = 0; k < 12; k++) T[k] = __ldg(ee + (size_t)i * 16 + k);
  out_count[i] = (int8_t)iiwa14_ik_one(T, lim, out_sol ? out_sol + (size_t)i * 56 : nullptr);
}

// common.cpp:214-226 after the filter kernel: every pair the approach test kept gets IK on its UN-shifted grasp_in_cam
// (composed exactly as filter_kernel does), ee_in_base = cam_in_world * grasp_in_cam * ee_in_grasp left to right
// (:216); a pair without an in-limit solution is the reference's IK rejection -- IK precedes the collision tests, so it
// takes the attribution whatever the collision verdict was.
__global__ void __launch_bounds__(IK_BLOCK) filter_ik_kernel(const cg_filter_params prm, const float *__restrict__ grasp_poses,
                                                             const float *__restrict__ sym, int S, long Q,
                                                             const cg_ik_params ik, const IkLimits lim,
                                                             uint8_t *__restrict__ status, int8_t *__restrict__ offset,
                                                             float *__restrict__ out_poses) {
  const long q = (long)blockIdx.x * IK_BLOCK + threadIdx.x;
  if (q >= Q || status[q] == CG_ST_REJ_DIR) return;
  const int i = (int)(q / S), j = (int)(q % S);
  float c2c[16], tmp[16], g[16], ce[16], eb[16];
  mm4(prm.nocs_pose, prm.canonical_to_nocs, c2c);            // common.cpp:159
  mm4(sym + (size_t)j * 16, grasp_poses + (size_t)i * 16, tmp);  // :190
  mm4(c2c, tmp, g);                                          // :191
  for (int col = 0; col < 3; col++) normalize_col(g, col);   // :194-197
  mm4(ik.cam_in_world, g, ce);                               // :216
  mm4(ce, ik.ee_in_grasp, eb);
  if (iiwa14_ik_one(eb, lim, nullptr) > 0) return;
  status[q] = CG_ST_REJ_IK;
  offset[q] = -1;
#pragma unroll
  for (int k = 0; k < 16; k++) out_poses[q * 16 + k] = 0.f;
}

IkLimits make_limits(const double *upper, const double *lower) {
  IkLimits l;
  for (int k = 0; k < 7; k++) { l.up[k] = upper[k]; l.lo[k] = lower[k]; }
  return l;
}

}  // namespace

extern "C" int cg_iiwa14_ik_dev(cg_ctx *ctx, const float *ee_in_base, int Q, const double upper[7],
                                const double lower[7], int8_t *out_count, double *out_solutions) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, Q >= 0 && upper && lower, "iiwa14_ik: Q / limits");
  if (Q == 0) return CG_OK;
  CG_REQUIRE(ctx, ee_in_base && out_count, "iiwa14_ik: poses / counts");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  ik_kernel<<<(Q + IK_BLOCK - 1) / IK_BLOCK, IK_BLOCK, 0, ctx->stream>>>(ee_in_base, Q, make_limits(upper, lower),
                                                                          out_count, out_solutions);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_filter_apply_ik_dev(cg_ctx *ctx, const cg_filter_params *prm, const float *grasp_poses, int G,
                                      const float *symmetry_tfs, int S, const cg_ik_params *ik, uint8_t *status,
                                      int8_t *offset, float *out_poses) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, prm && ik && grasp_poses && symmetry_tfs && G > 0 && S > 0, "filter_ik: poses");
  CG_REQUIRE(ctx, status && offset && out_poses, "filter_ik: filter outputs");
  CG_REQUIRE(ctx, (long)G * S < 2147483647L, "filter_ik: too many pairs");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const long Q = (long)G * S;
  filter_ik_kernel<<<(unsigned)((Q + IK_BLOCK - 1) / IK_BLOCK), IK_BLOCK, 0, ctx->stream>>>(
      *prm, grasp_poses, symmetry_tfs, S, Q, *ik, make_limits(ik->upper, ik->lower), status, offset, out_poses);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}
