// cg_affordance.cu -- affordance transfer per grasp (SURVEY.md 8f F4).
//
// Replaces run_grasp_simulation.py:50-73 (compute_grasp_affordance_worker) with pybullet_env/env_grasp.py:243-283
// (get_finger_contact_area) for G grasps at once: the object's canonical cloud (already in the camera frame) is moved
// into the finger frame of each grasp; per finger, the points inside the finger's x/z extent are kept (:252), the
// contact patch is the part of them within `surface_tol` of the extreme y in the closing direction (:261-270), the
// patch is dropped when the normal at its closest point faces along the closing direction (:275-281), and the
// finger's score is the mean affordance of the patch (nearest canonical point, precomputed per point on the host,
// :62-63).  A grasp's p(T|G) is the mean over its fingers with a patch; no patch at all -> NaN (the reference drops the grasp).
//
// float64 like the reference's numpy; one CTA per grasp, two sweeps over the points per finger.
#include "cg_common.cuh"

namespace {

constexpr int AT = 128;
constexpr int MAXF = 4;

struct FingerSpec {
  double xmin[MAXF], xmax[MAXF], zmin[MAXF], zmax[MAXF];
  int dir[MAXF];   // +1: closes along +y (patch at the smallest y), -1: along -y (patch at the largest y)
  int n;
};

__device__ __forceinline__ double block_min(double v, double *sh) {
  for (int o = 16; o; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = sh[0];
  for (int w = 1; w < AT / 32; w++) r = fmin(r, sh[w]);
  return r;
}

__device__ __forceinline__ double block_sum(double v, double *sh) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = sh[0];
  for (int w = 1; w < AT / 32; w++) r += sh[w];
  return r;
}

__global__ void __launch_bounds__(AT) affordance_kernel(const double *__restrict__ cam_in_finger, int G,
                                                        const double *__restrict__ pts, const double *__restrict__ nrm,
                                                        const double *__restrict__ aff, int P, FingerSpec fs, double tol,
                                                        double *__restrict__ out_p, int *__restrict__ out_contacts) {
  __shared__ double sh[AT / 32];
  __shared__ int sh_i[AT / 32];
  const int g = blockIdx.x, tid = threadIdx.x;
  const double *T = cam_in_finger + (size_t)g * 16;
  const double r00 = T[0], r01 = T[1], r02 = T[2], t0 = T[3];
  const double r10 = T[4], r11 = T[5], r12 = T[6], t1 = T[7];
  const double r20 = T[8], r21 = T[9], r22 = T[10], t2 = T[11];
  double total = 0.0;
  int nf = 0;
  for (int f = 0; f < fs.n; f++) {
    const double sgn = (double)fs.dir[f];
    // sweep 1: extreme y (in the closing direction) of the points inside the finger's x/z extent; s*y is minimised
    double ext = 1e300;
    for (int j = tid; j < P; j += AT) {
      const double px = pts[3 * j], py = pts[3 * j + 1], pz = pts[3 * j + 2];
      const double qx = fma(r02, pz, fma(r01, py, r00 * px)) + t0;
      const double qz = fma(r22, pz, fma(r21, py, r20 * px)) + t2;
      if (qx >= fs.xmin[f] && qx <= fs.xmax[f] && qz >= fs.zmin[f] && qz <= fs.zmax[f]) {
        const double qy = fma(r12, pz, fma(r11, py, r10 * px)) + t1;
        ext = fmin(ext, sgn * qy);
      }
    }
    ext = block_min(ext, sh);
    if (ext > 1e299) {                               // within_finger_mask.sum()==0 (:253-254)
      if (tid == 0) out_contacts[g * MAXF + f] = 0;
      continue;
    }
    const double y_ext = sgn * ext;
    // sweep 2: contact patch, its affordance sum, and the first point closest to the finger surface
    double sum = 0.0, cnt = 0.0, best_d = 1e300;
    int best_j = 0x7fffffff;
    for (int j = tid; j < P; j += AT) {
      const double px = pts[3 * j], py = pts[3 * j + 1], pz = pts[3 * j + 2];
      const double qx = fma(r02, pz, fma(r01, py, r00 * px)) + t0;
      const double qz = fma(r22, pz, fma(r21, py, r20 * px)) + t2;
      if (qx >= fs.xmin[f] && qx <= fs.xmax[f] && qz >= fs.zmin[f] && qz <= fs.zmax[f]) {
        const double qy = fma(r12, pz, fma(r11, py, r10 * px)) + t1;
        const double d = fabs(qy - y_ext);
        if (d <= tol) {
          sum += aff[j];
          cnt += 1.0;
          if (d < best_d) { best_d = d; best_j = j; }        // ascending j per thread: keeps the first minimum
        }
      }
    }
    const double dmin = block_min(best_d, sh);
    int cand = (best_d == dmin) ? best_j : 0x7fffffff;        // np.argmin: first index attaining the minimum
    for (int o = 16; o; o >>= 1) cand = min(cand, __shfl_xor_sync(0xffffffffu, cand, o));
    __syncthreads();
    if ((tid & 31) == 0) sh_i[tid >> 5] = cand;
    __syncthreads();
    int jstar = sh_i[0];
    for (int w = 1; w < AT / 32; w++) jstar = min(jstar, sh_i[w]);
    if (jstar == 0x7fffffff) {                       // empty patch: tol < 0 or NaN (contact_mask.sum()==0, :268-269)
      if (tid == 0) out_contacts[g * MAXF + f] = 0;
      continue;
    }
    sum = block_sum(sum, sh);
    cnt = block_sum(cnt, sh);
    // normal at the closest point, rotated into the finger frame; only the sign of its y component matters (:277-281)
    const double ny = fma(r12, nrm[3 * jstar + 2], fma(r11, nrm[3 * jstar + 1], r10 * nrm[3 * jstar]));
    const double nx = fma(r02, nrm[3 * jstar + 2], fma(r01, nrm[3 * jstar + 1], r00 * nrm[3 * jstar]));
    const double nz = fma(r22, nrm[3 * jstar + 2], fma(r21, nrm[3 * jstar + 1], r20 * nrm[3 * jstar]));
    const double nn = sqrt(nx * nx + ny * ny + nz * nz);
    const bool facing_away = (ny / nn) * sgn > 0.0;
    if (facing_away) {
      if (tid == 0) out_contacts[g * MAXF + f] = 0;
      continue;
    }
    if (tid == 0) out_contacts[g * MAXF + f] = (int)cnt;
    total += sum / cnt;
    nf++;
  }
  if (tid == 0) out_p[g] = nf > 0 ? total / (double)nf : nan("");
}

}  // namespace

extern "C" int cg_grasp_affordance_dev(cg_ctx *ctx, const double *cam_in_finger, int G, const double *pts, const double *nrm,
                                       const double *affordance, int P, const double *finger_boxes, const int *grip_dirs,
                                       int F, double surface_tol, double *out_p, int *out_contacts) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, cam_in_finger && pts && nrm && affordance && finger_boxes && grip_dirs && out_p && out_contacts,
             "grasp_affordance: null argument");
  CG_REQUIRE(ctx, G >= 0 && P > 0 && F >= 1 && F <= MAXF, "grasp_affordance: 1 <= fingers <= 4, P > 0");
  if (G == 0) return CG_OK;
  FingerSpec fs;
  fs.n = F;
  for (int f = 0; f < F; f++) {
    fs.xmin[f] = finger_boxes[4 * f]; fs.xmax[f] = finger_boxes[4 * f + 1];
    fs.zmin[f] = finger_boxes[4 * f + 2]; fs.zmax[f] = finger_boxes[4 * f + 3];
    CG_REQUIRE(ctx, grip_dirs[f] == 1 || grip_dirs[f] == -1, "grasp_affordance: grip_dir must be +1 or -1 (closing along +-y)");
    fs.dir[f] = grip_dirs[f];
  }
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  affordance_kernel<<<G, AT, 0, ctx->stream>>>(cam_in_finger, G, pts, nrm, affordance, P, fs, surface_tol, out_p, out_contacts);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}
