/* sdf_mesh_ref.c -- ORACLE for catgrasp_b200/csrc/cg_sdf_build.cu (test infrastructure only).
 *
 * Brute-force float64 signed distance from query points to a closed triangle mesh:
 *   distance: exact point-triangle distance, minimised over every triangle (a zero-area triangle counts as its
 *             segments / point);
 *   sign:     the generalized winding number, the sum over triangles of the solid angle (Van Oosterom & Strackee,
 *             IEEE Trans. Biomed. Eng. 30(2), 1983) over 4 pi; inside where |w| > 1/2.  This is independent of the
 *             ray parity the kernel uses.
 * Query points are given explicitly (not a grid), so large meshes can be checked on a sample of nodes and the
 * analytic proxy's own node positions can be evaluated. */
#include <math.h>
#include <omp.h>

static double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

static void cross3(const double *a, const double *b, double *o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

static double seg_d2(const double *p, const double *a, const double *b) {
  double d[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, w[3] = {p[0] - a[0], p[1] - a[1], p[2] - a[2]};
  double L = dot3(d, d), t = L > 0.0 ? dot3(w, d) / L : 0.0;
  if (t < 0.0) t = 0.0;
  if (t > 1.0) t = 1.0;
  double r[3] = {w[0] - t * d[0], w[1] - t * d[1], w[2] - t * d[2]};
  return dot3(r, r);
}

static double tri_d2(const double *p, const double *a, const double *b, const double *c) {
  double ab[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, ac[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
  double n[3];
  cross3(ab, ac, n);
  double nn = dot3(n, n);
  if (nn > 0.0) {
    const double *v[3] = {a, b, c};
    int inside = 1;
    for (int e = 0; e < 3 && inside; e++) {
      const double *s = v[e], *t = v[(e + 1) % 3];
      double d[3] = {t[0] - s[0], t[1] - s[1], t[2] - s[2]}, w[3] = {p[0] - s[0], p[1] - s[1], p[2] - s[2]}, x[3];
      cross3(d, w, x);
      inside = dot3(x, n) >= 0.0;
    }
    if (inside) {
      double w[3] = {p[0] - a[0], p[1] - a[1], p[2] - a[2]};
      double h = dot3(w, n);
      return h * h / nn;
    }
  }
  double d0 = seg_d2(p, a, b), d1 = seg_d2(p, b, c), d2 = seg_d2(p, c, a);
  return fmin(d0, fmin(d1, d2));
}

/* solid angle of triangle (a,b,c) seen from p (signed by orientation) */
static double solid_angle(const double *p, const double *a, const double *b, const double *c) {
  double A[3] = {a[0] - p[0], a[1] - p[1], a[2] - p[2]}, B[3] = {b[0] - p[0], b[1] - p[1], b[2] - p[2]},
         Cc[3] = {c[0] - p[0], c[1] - p[1], c[2] - p[2]}, x[3];
  double la = sqrt(dot3(A, A)), lb = sqrt(dot3(B, B)), lc = sqrt(dot3(Cc, Cc));
  cross3(B, Cc, x);
  double num = dot3(A, x);
  double den = la * lb * lc + dot3(A, B) * lc + dot3(A, Cc) * lb + dot3(B, Cc) * la;
  return 2.0 * atan2(num, den);
}

/* V (nv,3), F (nf,3), Q (nq,3) -> out_sd (nq) signed distance, out_wind (nq) winding number (may be NULL);
 * nthreads <= 0: OpenMP's default team */
void sdf_mesh_ref(const double *V, const int *F, int nf, const double *Q, long nq, int nthreads, double *out_sd,
                  double *out_wind) {
#pragma omp parallel for schedule(dynamic, 16) num_threads(nthreads > 0 ? nthreads : omp_get_max_threads())
  for (long q = 0; q < nq; q++) {
    const double *p = Q + 3 * q;
    double best = INFINITY, om = 0.0;
    for (int f = 0; f < nf; f++) {
      const double *a = V + 3 * F[3 * f], *b = V + 3 * F[3 * f + 1], *c = V + 3 * F[3 * f + 2];
      best = fmin(best, tri_d2(p, a, b, c));
      om += solid_angle(p, a, b, c);
    }
    const double w = om / (4.0 * M_PI), d = sqrt(best);
    out_sd[q] = fabs(w) > 0.5 ? -d : d;
    if (out_wind) out_wind[q] = w;
  }
}
