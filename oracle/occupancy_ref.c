/*
 * occupancy_ref.c -- CPU ORACLE for the scan occupancy / occlusion grid.  TEST INFRASTRUCTURE ONLY.
 *
 * Restates my_cpp/common.cpp:324-431 (makeOccupancyGridFromCloudScan): grid geometry :352-366,:375-377, ray
 * direction :378-380, "first occupied cell not farther than the sample" :383-393.  octomap (OcTree::insertPointCloud,
 * castRay) is not in /root/reference nor installed: the traversal below is a restatement of the SEMANTIC (occupied set
 * = cells floor(p/res) containing a scan point; 3-D DDA from the origin cell; hit reported at the cell centre) with
 * the CUDA kernel's operations in the kernel's order, none contracted (-ffp-contract=off here, explicit _rn intrinsics
 * there).  oracle/occupancy_exact.py states the same rule in exact rationals, without this arithmetic or the early
 * exit.  PARITY with octomap itself is UNPINNED; the control flow is pinned:
 * the reference's compiled function on oracle/ref_shim/octomap/octomap.h returns the same samples (tests/test_mycpp_golden.py).
 */
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

void occupancy_geometry_ref(const float *pts, int P, float res, int *dims, float *origin) {
  float mn[3] = {pts[0], pts[1], pts[2]}, mx[3] = {pts[0], pts[1], pts[2]};
  for (int i = 1; i < P; i++)
    for (int a = 0; a < 3; a++) {
      mn[a] = fminf(mn[a], pts[3 * i + a]);
      mx[a] = fmaxf(mx[a], pts[3 * i + a]);
    }
  const float pad = 0.005f;
  for (int a = 0; a < 3; a++) {
    dims[a] = (int)((mx[a] + pad - (mn[a] - pad)) / res);
    origin[a] = mn[a] - pad;
  }
}

void occupancy_ref(const float *pts, int P, float res, unsigned char *flags) {
  int dims[3];
  float org[3];
  occupancy_geometry_ref(pts, P, res, dims, org);
  int kmin[3] = {INT_MAX, INT_MAX, INT_MAX}, kmax[3] = {INT_MIN, INT_MIN, INT_MIN};
  for (int i = 0; i < P; i++)
    for (int a = 0; a < 3; a++) {
      const int k = (int)floor((double)pts[3 * i + a] / (double)res);
      if (k < kmin[a]) kmin[a] = k;
      if (k > kmax[a]) kmax[a] = k;
    }
  const int dx = kmax[0] - kmin[0] + 1, dy = kmax[1] - kmin[1] + 1, dz = kmax[2] - kmin[2] + 1;
  const size_t bits = (size_t)dx * dy * dz;
  unsigned char *occ = (unsigned char *)calloc(bits, 1);
  for (int i = 0; i < P; i++) {
    const int kx = (int)floor((double)pts[3 * i] / (double)res) - kmin[0];
    const int ky = (int)floor((double)pts[3 * i + 1] / (double)res) - kmin[1];
    const int kz = (int)floor((double)pts[3 * i + 2] / (double)res) - kmin[2];
    occ[((size_t)kx * dy + ky) * dz + kz] = 1;
  }
  const double r = (double)res;
#pragma omp parallel for schedule(dynamic) collapse(2)
  for (int xi = 0; xi < dims[0]; xi++)
    for (int yi = 0; yi < dims[1]; yi++)
      for (int zi = 0; zi < dims[2]; zi++) {
        const float x = org[0] + (float)xi * res, y = org[1] + (float)yi * res, z = org[2] + (float)zi * res;
        const float nrm = sqrtf((x * x + y * y) + z * z);
        unsigned char out = 0;
        if (nrm > 0.f) {
          const double d[3] = {(double)(x / nrm), (double)(y / nrm), (double)(z / nrm)};
          const double dist_q = (double)nrm;
          int k[3] = {0, 0, 0}, step[3];
          for (int a = 0; a < 3; a++) step[a] = (d[a] > 0.0) - (d[a] < 0.0);
#define OCC(KX, KY, KZ) (((KX) - kmin[0]) >= 0 && ((KY) - kmin[1]) >= 0 && ((KZ) - kmin[2]) >= 0 && ((KX) - kmin[0]) < dx && \
                         ((KY) - kmin[1]) < dy && ((KZ) - kmin[2]) < dz && occ[((size_t)((KX) - kmin[0]) * dy + ((KY) - kmin[1])) * dz + ((KZ) - kmin[2])])
          int hit = OCC(0, 0, 0);
          double cdist = sqrt(3.0 * 0.25 * r * r);
          while (!hit) {
            double tmax[3];
            for (int a = 0; a < 3; a++)
              tmax[a] = step[a] ? ((double)(k[a] + (step[a] > 0 ? 1 : 0)) * r) / d[a] : 1e300;
            const int dim = (tmax[0] < tmax[1]) ? ((tmax[0] < tmax[2]) ? 0 : 2) : ((tmax[1] < tmax[2]) ? 1 : 2);
            if (tmax[dim] > dist_q + 2.0 * r) break;
            k[dim] += step[dim];
            if (OCC(k[0], k[1], k[2])) {
              const double cx = ((double)k[0] + 0.5) * r, cy = ((double)k[1] + 0.5) * r, cz = ((double)k[2] + 0.5) * r;
              cdist = sqrt(cx * cx + cy * cy + cz * cz);
              hit = 1;
            }
          }
          if (hit && cdist <= dist_q) out = 1;
        }
        flags[((size_t)xi * dims[1] + yi) * dims[2] + zi] = out;
      }
  free(occ);
}
