// cg_occupancy.cu -- occupancy / occlusion grid from a depth scan.
//
// Replaces my_cpp/common.cpp:324-431 (makeOccupancyGridFromCloudScan): an octomap OcTree is filled with the scan
// points and, for every sample of a regular grid over the padded bounding box (pitch = resolution, pad 5 mm), a ray is
// cast from the sensor origin through the sample; the sample is reported when the first occupied cell on that ray is
// not farther than the sample itself (i.e. the sample is on or behind the observed surface).
//
// octomap is not available (SURVEY.md 8c): this file and oracle/occupancy_ref.c restate the semantic with the same
// operations in the same order so that they agree bit for bit -- occupied set = cells floor(p / res) of the scan points
// (dense bit mask over their bounding box); the ray is a 3-D DDA from the origin cell whose next-boundary parameters
// are recomputed from the integer cell index at every step (no accumulation); a hit counts when |cell centre| <=
// |sample|.  The oracle is compiled with -ffp-contract=off; nvcc contracts a*b + c into an FMA by default, so every
// floating-point operation of the cast kernel is written as an explicit round-to-nearest intrinsic, which nvcc never
// fuses (tests/test_codegen.py checks the PTX for FMAs).  An exact rational statement of the rule, without
// the kernel's arithmetic or its early exit, is oracle/occupancy_exact.py.
// The reference's own function, compiled against a restatement of the octomap calls it makes (oracle/build_ref.py,
// oracle/ref_shim/octomap/octomap.h), returns exactly the same samples (tests/test_mycpp_golden.py); parity with the
// octomap library itself stays unpinned (not installed, version not pinned by the reference).
#include "cg_common.cuh"

namespace {

struct OccGrid {
  float x0, y0, z0;      // first sample = min - pad (float arithmetic of common.cpp:375-377)
  int nx, ny, nz;        // sample counts (common.cpp:364-366)
  int kx0, ky0, kz0;     // smallest occupied cell index per axis
  int dx, dy, dz;        // extent of the occupied-cell bounding box
  float res;
};

__global__ void occ_mark_kernel(const float *__restrict__ pts, int P, OccGrid g, unsigned *__restrict__ mask) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const double r = (double)g.res;
  const int kx = (int)floor((double)pts[3 * i] / r) - g.kx0;
  const int ky = (int)floor((double)pts[3 * i + 1] / r) - g.ky0;
  const int kz = (int)floor((double)pts[3 * i + 2] / r) - g.kz0;
  const size_t bit = ((size_t)kx * g.dy + ky) * g.dz + kz;
  atomicOr(&mask[bit >> 5], 1u << (bit & 31));
}

__device__ __forceinline__ bool occ_test(const unsigned *mask, const OccGrid &g, int kx, int ky, int kz) {
  const int ix = kx - g.kx0, iy = ky - g.ky0, iz = kz - g.kz0;
  if (ix < 0 || iy < 0 || iz < 0 || ix >= g.dx || iy >= g.dy || iz >= g.dz) return false;
  const size_t bit = ((size_t)ix * g.dy + iy) * g.dz + iz;
  return (mask[bit >> 5] >> (bit & 31)) & 1u;
}

__global__ void occ_cast_kernel(OccGrid g, const unsigned *__restrict__ mask, unsigned char *__restrict__ flags) {
  const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long total = (long)g.nx * g.ny * g.nz;
  if (t >= total) return;
  const int zi = (int)(t % g.nz), yi = (int)((t / g.nz) % g.ny), xi = (int)(t / ((long)g.nz * g.ny));
  const float x = __fadd_rn(g.x0, __fmul_rn((float)xi, g.res));
  const float y = __fadd_rn(g.y0, __fmul_rn((float)yi, g.res));
  const float z = __fadd_rn(g.z0, __fmul_rn((float)zi, g.res));
  const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
  unsigned char out = 0;
  if (nrm > 0.f) {
    const double d[3] = {(double)__fdiv_rn(x, nrm), (double)__fdiv_rn(y, nrm), (double)__fdiv_rn(z, nrm)};
    const double r = (double)g.res, dist_q = (double)nrm;
    int k[3] = {0, 0, 0};
    int step[3];
    for (int a = 0; a < 3; a++) step[a] = (d[a] > 0.0) - (d[a] < 0.0);
    // the origin cell itself (octomap's castRay tests the start node first)
    bool hit = occ_test(mask, g, 0, 0, 0);
    double cdist = sqrt(__dmul_rn(__dmul_rn(0.75, r), r));    // 3.0 * 0.25 * r * r
    const double reach = __dadd_rn(dist_q, __dmul_rn(2.0, r));
    while (!hit) {
      double tmax[3];
      for (int a = 0; a < 3; a++)
        tmax[a] = step[a] ? __ddiv_rn(__dmul_rn((double)(k[a] + (step[a] > 0 ? 1 : 0)), r), d[a]) : 1e300;
      const int dim = (tmax[0] < tmax[1]) ? ((tmax[0] < tmax[2]) ? 0 : 2) : ((tmax[1] < tmax[2]) ? 1 : 2);
      if (tmax[dim] > reach) break;   // any later cell centre is farther than the sample
      k[dim] += step[dim];
      if (occ_test(mask, g, k[0], k[1], k[2])) {
        const double cx = __dmul_rn(__dadd_rn((double)k[0], 0.5), r), cy = __dmul_rn(__dadd_rn((double)k[1], 0.5), r),
                     cz = __dmul_rn(__dadd_rn((double)k[2], 0.5), r);
        cdist = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz)));
        hit = true;
      }
    }
    if (hit && cdist <= dist_q) out = 1;      // common.cpp:388-393
  }
  flags[t] = out;
}

}  // namespace

// Host-only helper: grid geometry exactly as common.cpp:352-366,375-377 computes it (float arithmetic).
extern "C" int cg_occupancy_grid_geometry(const float *pts_host, int P, float resolution, int dims[3], float origin[3]) {
  if (!pts_host || P <= 0 || !(resolution > 0.f) || !dims || !origin) return CG_EINVAL;
  float mn[3] = {pts_host[0], pts_host[1], pts_host[2]}, mx[3] = {pts_host[0], pts_host[1], pts_host[2]};
  for (int i = 1; i < P; i++)
    for (int a = 0; a < 3; a++) {
      mn[a] = fminf(mn[a], pts_host[3 * i + a]);
      mx[a] = fmaxf(mx[a], pts_host[3 * i + a]);
    }
  const float pad = 0.005f;
  for (int a = 0; a < 3; a++) {
    const float n = (mx[a] + pad - (mn[a] - pad)) / resolution;     // int max_xi = (xmax+pad-(xmin-pad))/resolution
    if (!(n < 2147483648.f)) return CG_EINVAL;                        // the conversion to int would overflow
    dims[a] = (int)n;
    origin[a] = mn[a] - pad;
  }
  return CG_OK;
}

extern "C" int cg_occupancy_from_scan_host(cg_ctx *ctx, const float *pts_host, int P, float resolution,
                                           unsigned char *out_flags_host) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, pts_host && P > 0 && resolution > 0.f && out_flags_host, "occupancy: bad arguments");
  int dims[3];
  float org[3];
  int rc = cg_occupancy_grid_geometry(pts_host, P, resolution, dims, org);
  if (rc) return rc;
  OccGrid g;
  g.x0 = org[0]; g.y0 = org[1]; g.z0 = org[2];
  g.nx = dims[0]; g.ny = dims[1]; g.nz = dims[2];
  g.res = resolution;
  const long total = (long)g.nx * g.ny * g.nz;
  CG_REQUIRE(ctx, total > 0 && total < (1L << 31), "occupancy: grid size");
  int kmin[3] = {INT32_MAX, INT32_MAX, INT32_MAX}, kmax[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
  for (int i = 0; i < P; i++)
    for (int a = 0; a < 3; a++) {
      const int k = (int)floor((double)pts_host[3 * i + a] / (double)resolution);
      kmin[a] = k < kmin[a] ? k : kmin[a];
      kmax[a] = k > kmax[a] ? k : kmax[a];
    }
  g.kx0 = kmin[0]; g.ky0 = kmin[1]; g.kz0 = kmin[2];
  g.dx = kmax[0] - kmin[0] + 1; g.dy = kmax[1] - kmin[1] + 1; g.dz = kmax[2] - kmin[2] + 1;
  const size_t bits = (size_t)g.dx * g.dy * g.dz;
  CG_REQUIRE(ctx, bits < (size_t(1) << 33), "occupancy: occupied-cell bounding box too large");
  const size_t words = (bits + 31) / 32;
  const float *d_pts; unsigned *d_mask; unsigned char *d_flags;
  return cg_io_stage(ctx, [&](cg_io_pieces &io) {
    d_pts = io.in(pts_host, (size_t)P * 3);
    d_mask = io.take<unsigned>(words);
    d_flags = io.out(out_flags_host, (size_t)total);
  }, [&] {
    CG_CUDA(ctx, cudaMemsetAsync(d_mask, 0, words * 4, ctx->stream));
    occ_mark_kernel<<<(P + 255) / 256, 256, 0, ctx->stream>>>(d_pts, P, g, d_mask);
    CG_LAUNCH_CHECK(ctx);
    occ_cast_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(g, d_mask, d_flags);
    CG_LAUNCH_CHECK(ctx);
    return CG_OK;
  });
}
