// extern "C" entry points into the reference's IK (my_cpp/common.cpp:9-72 get_ik_within_limits and the generated ikfast
// solver's ComputeFk), linked against oracle/_ref/libmycpp_ref.so by oracle/build_ref_ik.py, for oracle/mycpp_ref_ik.py.
// ORACLE / test infrastructure only.
#include "common.h"

#include <limits>

// Every solution get_ik_within_limits returns with limits of -inf / +inf (none is rejected by a limit), in the order
// ikfast produced them.  Writes at most `cap` rows of 7 doubles; returns the solution count.
extern "C" int ref_ik_solutions(const float *ee_in_base, double *out, int cap) {
  Eigen::Matrix4f m;
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) m(r, c) = ee_in_base[r * 4 + c];
  const double inf = std::numeric_limits<double>::infinity();
  std::vector<double> up(7, inf), lo(7, -inf);
  std::vector<std::vector<double>> sols = get_ik_within_limits(m, up, lo);
  for (size_t i = 0; i < sols.size() && (int)i < cap; i++)
    for (int k = 0; k < 7; k++) out[i * 7 + k] = sols[i][k];
  return (int)sols.size();
}

// ikfast ComputeFk: joints (7) -> trans (3), rot (9, row-major), float64
extern "C" void ref_ik_fk(const double *q, double *trans, double *rot) { ComputeFk(q, trans, rot); }
