// cg_sdf_build.cu -- signed-distance grid of a closed triangle mesh (replaces make_sdf.py:30-36, which runs the external
// SDFGen binary, and the .sdf files it writes, sdf_file.py:59-87).
//
// Grid: per axis n = ceil(extent / res - 1e-4) + 1 + 2 * padding nodes, origin = float32(min vertex - padding * res);
// node (i,j,k) sits at origin + (i,j,k) * res, evaluated in float64 from the float32 origin and res (the positions the
// filter's lookups assume).  The 1e-4 is a tolerance in cells: an extent of a whole number of cells gains no node.
//
// Value: the exact Euclidean distance from the node to the nearest triangle in float64, rounded once to float32,
// negative inside.  A zero-area triangle counts as its segment or point.
//
// Distance pass: one CTA per brick of 4x8x8 nodes.  Triangles are sorted by the Morton code of their centroids and
// grouped into tiles of 32 with a float64 AABB; a CTA first processes the tile nearest to its brick and the tiles next to
// the brick in Morton order, then sweeps all tiles and skips a tile whose AABB lies farther from the brick's AABB than
// the brick's largest per-node best distance (plus a slack far above the float64 error of a point-triangle distance);
// each warp applies the same test to its own 2x4x4 sub-brick and best distances.  A skipped tile cannot hold a triangle
// nearer to any node than that node's best, so the result is the brute-force minimum, and since the minimum does not
// depend on the order the grid is bitwise deterministic.
//
// Sign pass: ray parity along +x (SDFGen's method).  The yz coordinates of every vertex are snapped to a fixed-point
// lattice (2^16 steps per cell) on which the grid lines are lattice points, so the crossing test of a line with a
// projected triangle is exact in int64.  Lines through an edge or a vertex are resolved by a half-open rule that is
// the same as moving the line by (eps, eps^2) in (y, z): a closed mesh is crossed an even number of times on every
// line.  A crossing at x_c counts for every node with x_i > x_c; a line with an odd total means the mesh is open and
// the build fails.  Snapping moves the geometry by at most res * 2^-17, so the sign is exact for nodes farther than that
// from the surface.  Parity is not the winding number: where closed parts overlap, a line crosses two surfaces and the
// overlap comes out positive (outside), as SDFGen's odd-crossing rule gives it.  That is the contract, not a bug to fix.
#include <math.h>
#include <algorithm>
#include "cg_common.cuh"

namespace {

constexpr int BX = 4, BY = 8, BZ = 8, BT = BX * BY * BZ;   // brick of nodes per CTA, k fastest
constexpr int TILE = 32;                                   // triangles per culling tile
constexpr int TRI_D = 9;                                   // doubles per triangle: a, b, c
constexpr int SNAP_BITS = 16;                              // fixed-point steps per cell: 2^16
constexpr int MAX_CELLS_AXIS = 2048;                       // keeps snapped coordinates < 2^28: orient2d exact in int64
constexpr int SEED_TILES = 1;                              // tiles on either side of the brick's Morton position

struct Geom {
  int nx, ny, nz;
  double o[3];   // float32 origin, widened
  double res;    // float32 resolution, widened
};

__device__ __forceinline__ double node_x(const Geom &g, int a, int i) { return __dadd_rn(g.o[a], __dmul_rn((double)i, g.res)); }

// The point-triangle distance is spelled with explicitly rounded operations (no FMA contraction) in the operation order
// of oracle/sdf_mesh_ref.c, so that both compute the same float64 value: a node exactly on a face comes out 0 on both.
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }

struct V3 {
  double x, y, z;
};
__device__ __forceinline__ V3 vsub(const V3 &a, const V3 &b) { return {dsub(a.x, b.x), dsub(a.y, b.y), dsub(a.z, b.z)}; }
__device__ __forceinline__ double vdot(const V3 &a, const V3 &b) {
  return __dadd_rn(__dadd_rn(dmul(a.x, b.x), dmul(a.y, b.y)), dmul(a.z, b.z));
}
__device__ __forceinline__ V3 vcross(const V3 &a, const V3 &b) {
  return {dsub(dmul(a.y, b.z), dmul(a.z, b.y)), dsub(dmul(a.z, b.x), dmul(a.x, b.z)), dsub(dmul(a.x, b.y), dmul(a.y, b.x))};
}

// squared distance from p to the segment s -> t (s == t: the point s)
__device__ __forceinline__ double seg_d2(const V3 &p, const V3 &s, const V3 &t) {
  const V3 d = vsub(t, s), w = vsub(p, s);
  const double L = vdot(d, d);
  double u = L > 0.0 ? __ddiv_rn(vdot(w, d), L) : 0.0;
  u = fmin(fmax(u, 0.0), 1.0);
  const V3 r = {dsub(w.x, dmul(u, d.x)), dsub(w.y, dmul(u, d.y)), dsub(w.z, dmul(u, d.z))};
  return vdot(r, r);
}

// squared distance from p to triangle T = (a, b, c): the plane distance when p projects inside, else the nearest edge.
// A zero-area triangle has no inside and reduces to its edges; no NaN for any finite input.
__device__ double tri_d2(const V3 &p, const double *T) {
  const V3 a = {T[0], T[1], T[2]}, b = {T[3], T[4], T[5]}, c = {T[6], T[7], T[8]};
  const V3 n = vcross(vsub(b, a), vsub(c, a));
  const double nn = vdot(n, n);
  if (nn > 0.0) {
    // p projects inside iff it is on the inner side of all three edges: ((t - s) x (p - s)) . n >= 0
    if (vdot(vcross(vsub(b, a), vsub(p, a)), n) >= 0.0 && vdot(vcross(vsub(c, b), vsub(p, b)), n) >= 0.0 &&
        vdot(vcross(vsub(a, c), vsub(p, c)), n) >= 0.0) {
      const double h = vdot(vsub(p, a), n);
      return __ddiv_rn(dmul(h, h), nn);
    }
  }
  return fmin(seg_d2(p, a, b), fmin(seg_d2(p, b, c), seg_d2(p, c, a)));
}

__host__ __device__ __forceinline__ uint32_t morton_spread(uint32_t v) {   // 10 bits -> every third bit
  v &= 0x3ffu;
  v = (v | (v << 16)) & 0x030000ffu;
  v = (v | (v << 8)) & 0x0300f00fu;
  v = (v | (v << 4)) & 0x030c30c3u;
  v = (v | (v << 2)) & 0x09249249u;
  return v;
}

struct MortonFrame {
  double lo[3], scale[3];   // q_a = clamp((x_a - lo_a) * scale_a, 0, 1023)
};

__host__ __device__ __forceinline__ uint32_t morton_code(const MortonFrame &m, double x, double y, double z) {
  const double c[3] = {x, y, z};
  uint32_t q[3];
  for (int a = 0; a < 3; a++) q[a] = (uint32_t)fmin(fmax((c[a] - m.lo[a]) * m.scale[a], 0.0), 1023.0);
  return (morton_spread(q[0]) << 2) | (morton_spread(q[1]) << 1) | morton_spread(q[2]);
}

// squared gap between two AABBs (0 when they overlap)
__device__ __forceinline__ double box_gap2(const double *blo, const double *bhi, const double *t) {
  double s = 0.0;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const double g = fmax(fmax(t[a] - bhi[a], blo[a] - t[3 + a]), 0.0);
    s += g * g;
  }
  return s;
}

// tris (ntiles*TILE, 9) Morton-ordered (the last tile padded with repeats of the last triangle), tbox (ntiles, 6) =
// lo xyz, hi xyz; tcode (ntiles) = Morton code of each tile's first triangle.  Writes unsigned distances.
__global__ void __launch_bounds__(BT) sdf_distance_kernel(const Geom g, const double *__restrict__ tris,
                                                          const double *__restrict__ tbox,
                                                          const uint32_t *__restrict__ tcode, int ntiles,
                                                          const MortonFrame mf, double slack, float *__restrict__ grid) {
  __shared__ double s_tri[TILE * TRI_D];
  __shared__ double s_wmax[BT / 32];
  __shared__ unsigned s_mask[BT / 32];
  const int nbx = (g.nx + BX - 1) / BX, nby = (g.ny + BY - 1) / BY;
  const int b = blockIdx.x;
  const int i0 = (b % nbx) * BX, j0 = ((b / nbx) % nby) * BY, k0 = (b / (nbx * nby)) * BZ;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  // each warp holds a compact 2x4x4 sub-brick (warps 2x2x2 in the brick), so that its own bound is tight
  const int wi0 = i0 + 2 * (warp >> 2), wj0 = j0 + 4 * ((warp >> 1) & 1), wk0 = k0 + 4 * (warp & 1);
  const int i = wi0 + (lane >> 4), j = wj0 + ((lane >> 2) & 3), k = wk0 + (lane & 3);
  const bool active = i < g.nx && j < g.ny && k < g.nz;
  const V3 p = {node_x(g, 0, i), node_x(g, 1, j), node_x(g, 2, k)};
  const double wlo[3] = {node_x(g, 0, wi0), node_x(g, 1, wj0), node_x(g, 2, wk0)};
  const double whi[3] = {node_x(g, 0, wi0 + 1), node_x(g, 1, wj0 + 3), node_x(g, 2, wk0 + 3)};
  const double blo[3] = {node_x(g, 0, i0), node_x(g, 1, j0), node_x(g, 2, k0)};
  const double bhi[3] = {node_x(g, 0, min(i0 + BX, g.nx) - 1), node_x(g, 1, min(j0 + BY, g.ny) - 1),
                         node_x(g, 2, min(k0 + BZ, g.nz) - 1)};
  double best = INFINITY;
  double thr2 = INFINITY;    // skip a tile whose gap^2 to the brick exceeds this; block-uniform
  double wthr2 = INFINITY;   // the same for the warp's sub-brick and the warp's largest best; warp-uniform

  auto process = [&](int tile) {
    for (int e = t; e < TILE * TRI_D; e += BT) s_tri[e] = tris[(size_t)tile * TILE * TRI_D + e];
    __syncthreads();
    if (active && box_gap2(wlo, whi, tbox + (size_t)tile * 6) <= wthr2) {
#pragma unroll 2
      for (int e = 0; e < TILE; e++) best = fmin(best, tri_d2(p, s_tri + e * TRI_D));
    }
    double m = active ? best : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    const double rw = sqrt(m) + slack;
    wthr2 = rw * rw;
    if (lane == 0) s_wmax[warp] = m;
    __syncthreads();   // also: every thread is done with s_tri before the next tile overwrites it
    double mb = s_wmax[0];
#pragma unroll
    for (int w = 1; w < BT / 32; w++) mb = fmax(mb, s_wmax[w]);
    const double r = sqrt(mb) + slack;
    thr2 = r * r;
  };

  // Seed the bound with the tile whose AABB is nearest to the brick's (ties: lowest index) -- Morton neighbours alone can
  // lie across a jump of the curve, far from the brick, and a loose bound lets the sweep process most tiles -- then
  // with the tiles next to the brick's centre in Morton order.
  {
    double gb = INFINITY;
    int tb = 0;
    for (int tile = t; tile < ntiles; tile += BT) {
      const double gg = box_gap2(blo, bhi, tbox + (size_t)tile * 6);
      if (gg < gb) { gb = gg; tb = tile; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double og = __shfl_xor_sync(0xffffffffu, gb, o);
      const int ot = __shfl_xor_sync(0xffffffffu, tb, o);
      if (og < gb || (og == gb && ot < tb)) { gb = og; tb = ot; }
    }
    if (lane == 0) { s_wmax[warp] = gb; s_mask[warp] = (unsigned)tb; }
    __syncthreads();
    gb = s_wmax[0];
    tb = (int)s_mask[0];
    for (int w = 1; w < BT / 32; w++)
      if (s_wmax[w] < gb || (s_wmax[w] == gb && (int)s_mask[w] < tb)) { gb = s_wmax[w]; tb = (int)s_mask[w]; }
    process(tb);   // its first barrier orders these reads before s_wmax is rewritten
  }
  const uint32_t key = morton_code(mf, 0.5 * (blo[0] + bhi[0]), 0.5 * (blo[1] + bhi[1]), 0.5 * (blo[2] + bhi[2]));
  int lo = 0, hi = ntiles;   // last tile whose first code <= key (0 if none)
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (tcode[mid] <= key) lo = mid; else hi = mid;
  }
  const int s0 = max(0, lo - SEED_TILES), s1 = min(ntiles - 1, lo + SEED_TILES);
  for (int tile = s0; tile <= s1; tile++) process(tile);

  // sweep: test BT tiles at once, then process the survivors in order against the bound as it tightens
  for (int c = 0; c < ntiles; c += BT) {
    const int tile = c + t;
    const bool cand = tile < ntiles && (tile < s0 || tile > s1) && box_gap2(blo, bhi, tbox + (size_t)tile * 6) <= thr2;
    const unsigned m = __ballot_sync(0xffffffffu, cand);
    if (lane == 0) s_mask[warp] = m;
    __syncthreads();
    for (int w = 0; w < BT / 32; w++) {
      unsigned mm = s_mask[w];
      while (mm) {
        const int bit = __ffs(mm) - 1;
        mm &= mm - 1;
        const int tt = c + w * 32 + bit;
        if (box_gap2(blo, bhi, tbox + (size_t)tt * 6) <= thr2) process(tt);   // same on every thread
      }
    }
    __syncthreads();   // s_mask is rewritten by the next chunk
  }
  if (active) grid[((size_t)i * g.ny + j) * g.nz + k] = __double2float_rn(sqrt(best));
}

struct SnapTri {
  long long y[3], z[3];   // yz on the lattice: round((c - origin) / res * 2^16)
  double x[3];
};

__device__ __forceinline__ long long orient2d(long long au, long long av, long long bu, long long bv, long long pu,
                                              long long pv) {
  return (bu - au) * (pv - av) - (bv - av) * (pu - au);
}

// w == 0 (the line runs through the edge a->b of a counter-clockwise triangle) counts as inside iff moving the line by
// (eps, eps^2) moves it inside: cross(d, (eps, eps^2)) = du eps^2 - dv eps > 0
__device__ __forceinline__ bool edge_in(long long w, long long du, long long dv) {
  return w > 0 || (w == 0 && (dv < 0 || (dv == 0 && du > 0)));
}

// one warp per triangle; cnt[slot * nlines + line], line = j * nz + k, slot = first node with x_i > x_c (nx: beyond)
__global__ void __launch_bounds__(256) sdf_crossings_kernel(const Geom g, const SnapTri *__restrict__ st, int nf,
                                                            int *__restrict__ cnt) {
  const int f = (int)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (f >= nf) return;
  const SnapTri T = st[f];
  long long u0 = T.y[0], v0 = T.z[0], u1 = T.y[1], v1 = T.z[1], u2 = T.y[2], v2 = T.z[2];
  double x1 = T.x[1], x2 = T.x[2];
  const double x0 = T.x[0];
  const long long W = orient2d(u0, v0, u1, v1, u2, v2);
  if (W == 0) return;   // zero projected area: no crossing
  if (W < 0) {          // counter-clockwise in (y, z)
    long long tu = u1, tv = v1;
    u1 = u2; v1 = v2; u2 = tu; v2 = tv;
    const double tx = x1; x1 = x2; x2 = tx;
  }
  const double Wd = (double)(W < 0 ? -W : W);
  const long long S = 1ll << SNAP_BITS;
  const long long umin = min(u0, min(u1, u2)), umax = max(u0, max(u1, u2));
  const long long vmin = min(v0, min(v1, v2)), vmax = max(v0, max(v1, v2));
  // grid lines j with j*S in [umin, umax] (floor division for negative coordinates)
  const long long jlo = max(0ll, (umin >= 0 ? (umin + S - 1) / S : -((-umin) / S)));
  const long long jhi = min((long long)g.ny - 1, (umax >= 0 ? umax / S : -((-umax + S - 1) / S)));
  const long long klo = max(0ll, (vmin >= 0 ? (vmin + S - 1) / S : -((-vmin) / S)));
  const long long khi = min((long long)g.nz - 1, (vmax >= 0 ? vmax / S : -((-vmax + S - 1) / S)));
  if (jlo > jhi || klo > khi) return;
  const long long nk = khi - klo + 1, nl = (jhi - jlo + 1) * nk;
  const size_t nlines = (size_t)g.ny * g.nz;
  for (long long l = lane; l < nl; l += 32) {
    const long long j = jlo + l / nk, k = klo + l % nk;
    const long long pu = j * S, pv = k * S;
    const long long w0 = orient2d(u1, v1, u2, v2, pu, pv);
    const long long w1 = orient2d(u2, v2, u0, v0, pu, pv);
    const long long w2 = orient2d(u0, v0, u1, v1, pu, pv);
    if (!(edge_in(w0, u2 - u1, v2 - v1) && edge_in(w1, u0 - u2, v0 - v2) && edge_in(w2, u1 - u0, v1 - v0))) continue;
    const double xc = ((double)w0 * x0 + (double)w1 * x1 + (double)w2 * x2) / Wd;
    // first node with x_i > xc
    const double tc = fmin(fmax((xc - g.o[0]) / g.res, -1.0), (double)g.nx);
    int s = (int)floor(tc) + 1;
    s = min(max(s, 0), g.nx);
    while (s > 0 && node_x(g, 0, s - 1) > xc) s--;
    while (s < g.nx && node_x(g, 0, s) <= xc) s++;
    atomicAdd(cnt + (size_t)s * nlines + (size_t)(j * g.nz + k), 1);
  }
}

// one thread per line: prefix parity along x, negate the inside nodes; an odd total marks the mesh open
__global__ void sdf_parity_kernel(const Geom g, const int *__restrict__ cnt, float *__restrict__ grid, int *open_flag) {
  const size_t nlines = (size_t)g.ny * g.nz;
  const size_t line = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (line >= nlines) return;
  int run = 0;
  for (int i = 0; i < g.nx; i++) {
    run += cnt[(size_t)i * nlines + line];
    if (run & 1) grid[(size_t)i * nlines + line] = -grid[(size_t)i * nlines + line];
  }
  run += cnt[(size_t)g.nx * nlines + line];
  if (run & 1) atomicOr(open_flag, 1);
}

}  // namespace

extern "C" int cg_sdf_from_mesh(cg_ctx *ctx, const double *vertices, int nv, const int32_t *faces, int nf,
                                float resolution, int padding, cg_sdf **out) {
  if (!ctx || !out) return CG_EINVAL;
  *out = nullptr;
  CG_REQUIRE(ctx, vertices && faces && nv > 0 && nf > 0, "sdf_from_mesh: empty mesh (nv, nf must be > 0)");
  CG_REQUIRE(ctx, resolution > 0.f && isfinite(resolution), "sdf_from_mesh: resolution must be finite and > 0");
  CG_REQUIRE(ctx, padding >= 0, "sdf_from_mesh: padding must be >= 0");
  double vlo[3] = {INFINITY, INFINITY, INFINITY}, vhi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (size_t e = 0; e < (size_t)nv * 3; e++) {
    CG_REQUIRE(ctx, isfinite(vertices[e]), "sdf_from_mesh: non-finite vertex coordinate");
    vlo[e % 3] = fmin(vlo[e % 3], vertices[e]);
    vhi[e % 3] = fmax(vhi[e % 3], vertices[e]);
  }
  for (size_t e = 0; e < (size_t)nf * 3; e++)
    CG_REQUIRE(ctx, faces[e] >= 0 && faces[e] < nv, "sdf_from_mesh: face index out of range");

  // grid geometry
  const double res = (double)resolution;
  Geom g;
  int dims[3];
  for (int a = 0; a < 3; a++) {
    const double n = ceil((vhi[a] - vlo[a]) / res - 1e-4) + 1.0 + 2.0 * (double)padding;
    CG_REQUIRE(ctx, n <= MAX_CELLS_AXIS, "sdf_from_mesh: more than 2048 nodes along an axis (coarser resolution?)");
    dims[a] = (int)n;
    g.o[a] = (double)(float)(vlo[a] - (double)padding * res);
  }
  g.nx = dims[0]; g.ny = dims[1]; g.nz = dims[2];
  g.res = res;
  const size_t ncell = (size_t)g.nx * g.ny * g.nz, nlines = (size_t)g.ny * g.nz;
  CG_REQUIRE(ctx, (g.nx + 1) * nlines < (size_t)2147483647, "sdf_from_mesh: grid too large (>= 2^31 nodes)");

  // Morton-ordered triangles in tiles of TILE (the last tile padded with its last triangle: a repeat changes no minimum)
  MortonFrame mf;
  for (int a = 0; a < 3; a++) {
    mf.lo[a] = vlo[a];
    mf.scale[a] = vhi[a] > vlo[a] ? 1023.0 / (vhi[a] - vlo[a]) : 0.0;
  }
  std::vector<uint64_t> order((size_t)nf);
  for (int f = 0; f < nf; f++) {
    double c[3];
    for (int a = 0; a < 3; a++)
      c[a] = (vertices[3 * (size_t)faces[3 * (size_t)f] + a] + vertices[3 * (size_t)faces[3 * (size_t)f + 1] + a] +
              vertices[3 * (size_t)faces[3 * (size_t)f + 2] + a]) / 3.0;
    order[f] = ((uint64_t)morton_code(mf, c[0], c[1], c[2]) << 32) | (uint32_t)f;
  }
  std::sort(order.begin(), order.end());
  const int ntiles = (nf + TILE - 1) / TILE;
  std::vector<double> tris((size_t)ntiles * TILE * TRI_D), tbox((size_t)ntiles * 6);
  std::vector<uint32_t> tcode(ntiles);
  for (int s = 0; s < ntiles * TILE; s++) {
    const int f = (int)(uint32_t)order[std::min(s, nf - 1)];
    for (int v = 0; v < 3; v++)
      for (int a = 0; a < 3; a++) tris[(size_t)s * TRI_D + 3 * v + a] = vertices[3 * (size_t)faces[3 * (size_t)f + v] + a];
  }
  for (int t = 0; t < ntiles; t++) {
    tcode[t] = (uint32_t)(order[(size_t)t * TILE] >> 32);
    double *bx = &tbox[(size_t)t * 6];
    for (int a = 0; a < 3; a++) { bx[a] = INFINITY; bx[3 + a] = -INFINITY; }
    for (int s = t * TILE; s < (t + 1) * TILE; s++)
      for (int v = 0; v < 3; v++)
        for (int a = 0; a < 3; a++) {
          bx[a] = fmin(bx[a], tris[(size_t)s * TRI_D + 3 * v + a]);
          bx[3 + a] = fmax(bx[3 + a], tris[(size_t)s * TRI_D + 3 * v + a]);
        }
  }
  // Slack of the culling test: the float64 distance of a node to a triangle or to an AABB is off by a few ulps of the
  // largest coordinate involved; 2^-30 of it is far above that and far below any float32 spacing of the result.
  double mag = 0.0;
  for (int a = 0; a < 3; a++)
    mag = fmax(mag, fmax(fmax(fabs(vlo[a]), fabs(vhi[a])), fmax(fabs(g.o[a]), fabs(g.o[a] + (dims[a] - 1) * res))));
  const double slack = 2.0 * ldexp(mag, -30);

  // yz of every triangle on the fixed-point lattice
  const double S = ldexp(1.0, SNAP_BITS);
  std::vector<SnapTri> snap((size_t)nf);
  for (int f = 0; f < nf; f++)
    for (int v = 0; v < 3; v++) {
      const double *p = vertices + 3 * (size_t)faces[3 * (size_t)f + v];
      snap[f].x[v] = p[0];
      snap[f].y[v] = llrint((p[1] - g.o[1]) / res * S);
      snap[f].z[v] = llrint((p[2] - g.o[2]) / res * S);
    }

  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  DevBuf d_grid, d_tris, d_tbox, d_tcode, d_snap, d_cnt, d_flag;
  int rc;
  if ((rc = dev_alloc(ctx, d_grid, ncell * sizeof(float)))) return rc;
  if ((rc = dev_alloc(ctx, d_tris, tris.size() * sizeof(double)))) return rc;
  if ((rc = dev_alloc(ctx, d_tbox, tbox.size() * sizeof(double)))) return rc;
  if ((rc = dev_alloc(ctx, d_tcode, tcode.size() * sizeof(uint32_t)))) return rc;
  if ((rc = dev_alloc(ctx, d_snap, snap.size() * sizeof(SnapTri)))) return rc;
  if ((rc = dev_alloc(ctx, d_cnt, (g.nx + 1) * nlines * sizeof(int)))) return rc;
  if ((rc = dev_alloc(ctx, d_flag, sizeof(int)))) return rc;
  CG_CUDA(ctx, cudaMemcpyAsync(d_tris.p, tris.data(), tris.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  CG_CUDA(ctx, cudaMemcpyAsync(d_tbox.p, tbox.data(), tbox.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  CG_CUDA(ctx, cudaMemcpyAsync(d_tcode.p, tcode.data(), tcode.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  CG_CUDA(ctx, cudaMemcpyAsync(d_snap.p, snap.data(), snap.size() * sizeof(SnapTri), cudaMemcpyHostToDevice, st));
  CG_CUDA(ctx, cudaMemsetAsync(d_cnt.p, 0, (g.nx + 1) * nlines * sizeof(int), st));
  CG_CUDA(ctx, cudaMemsetAsync(d_flag.p, 0, sizeof(int), st));

  float *grid = static_cast<float *>(d_grid.p);
  const int nbricks = ((g.nx + BX - 1) / BX) * ((g.ny + BY - 1) / BY) * ((g.nz + BZ - 1) / BZ);
  sdf_distance_kernel<<<nbricks, BT, 0, st>>>(g, static_cast<const double *>(d_tris.p),
                                              static_cast<const double *>(d_tbox.p),
                                              static_cast<const uint32_t *>(d_tcode.p), ntiles, mf, slack, grid);
  CG_LAUNCH_CHECK(ctx);
  sdf_crossings_kernel<<<(unsigned)(((size_t)nf * 32 + 255) / 256), 256, 0, st>>>(
      g, static_cast<const SnapTri *>(d_snap.p), nf, static_cast<int *>(d_cnt.p));
  CG_LAUNCH_CHECK(ctx);
  sdf_parity_kernel<<<(unsigned)((nlines + 255) / 256), 256, 0, st>>>(g, static_cast<const int *>(d_cnt.p), grid,
                                                                      static_cast<int *>(d_flag.p));
  CG_LAUNCH_CHECK(ctx);

  std::vector<float> host(ncell);
  int open = 0;
  CG_CUDA(ctx, cudaMemcpyAsync(host.data(), grid, ncell * sizeof(float), cudaMemcpyDeviceToHost, st));
  CG_CUDA(ctx, cudaMemcpyAsync(&open, d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  CG_CUDA(ctx, cudaStreamSynchronize(st));
  CG_REQUIRE(ctx, !open, "sdf_from_mesh: mesh is not closed (a grid line along x crosses it an odd number of times)");

  cg_sdf *s = new cg_sdf();
  s->ctx = ctx; s->nx = g.nx; s->ny = g.ny; s->nz = g.nz; s->res = resolution;
  for (int a = 0; a < 3; a++) s->origin[a] = (float)g.o[a];
  cg_sdf_border_stats(s, host.data());
  s->grid = static_cast<float *>(d_grid.release());
  *out = s;
  return CG_OK;
}

extern "C" int cg_sdf_geometry(const cg_sdf *sdf, int dims[3], float origin[3], float *resolution) {
  if (!sdf || !dims || !origin || !resolution) return CG_EINVAL;
  dims[0] = sdf->nx; dims[1] = sdf->ny; dims[2] = sdf->nz;
  for (int a = 0; a < 3; a++) origin[a] = sdf->origin[a];
  *resolution = sdf->res;
  return CG_OK;
}

extern "C" int cg_sdf_download(cg_sdf *sdf, float *grid_host) {
  if (!sdf) return CG_EINVAL;
  cg_ctx *ctx = sdf->ctx;
  CG_REQUIRE(ctx, grid_host, "sdf_download: NULL output");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t bytes = (size_t)sdf->nx * sdf->ny * sdf->nz * sizeof(float);
  CG_CUDA(ctx, cudaMemcpyAsync(grid_host, sdf->grid, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return CG_OK;
}
