// cg_spconv.cu -- sparse 3-D convolution with spconv 1.x semantics, the layer types of PointGroup's U-Net
// (SubMConv3d k3 / k1, SparseConv3d k2 s2, SparseInverseConv3d k2; PointGroup/model/pointgroup/pointgroup.py).
//
// A level is a set of distinct integer sites (x, y, z), each in [0, 2^21), packed into the 63-bit key
// x << 42 | y << 21 | z and held in ascending key order: row-major over (x, y, z), z fastest.  The order of a level's
// rows reaches no output of the network (every gather goes through a table), so key order is the contract.
//
// Every convolution is one gather table nbr[Vout][K] (input row or -1) and one weight array W[K][Cin][Cout]:
//   out[r] = (sum_k W[k]^T act(in[nbr[r][k]]) + bias) + residual[r]
// with act(v) = max(v * scale + shift, 0) per channel when a BN prologue is given, else v, and an absent (-1) row
// contributing nothing -- not act(0): spconv's BN and ReLU run on the active rows only.
//   SubM k3  nbr[v][k] = the site v + (kx-1, ky-1, kz-1), k = 9 kx + 3 ky + kz   (cross-correlation, geometry.h)
//   SubM k1  no table: row r reads row r
//   down     down[p][k] = the child c with c = 2 p + (kx, ky, kz), k = 4 kx + 2 ky + kz; a child whose parent index
//            on some axis is >= (S - 2) / 2 + 1 is dropped (getValidOutPos), so an odd axis loses its last plane
//   up       up[c][k] = parent(c) for k = c - 2 parent(c), -1 elsewhere: the down pairs with in and out swapped and
//            the same k (spconv_ops.h indice_inverse_conv); a dropped child reads nothing and gets the bias only
// The sum runs over k ascending, then input channel ascending, as one fp32 FMA chain per output: two runs are bitwise
// equal, and the result does not depend on the tile shape or on Vout.
//
// Table builds size every output from a row bound the caller gives, write the true count to a device word and never
// synchronise, so a network forward needs no host round trip after the first level's count.  A coarse level's bound
// is min(the finer level's rows, the cells of the coarse shape): every parent has a child and is a coarse cell.
#include <cub/cub.cuh>
#include "cg_common.cuh"

namespace {

constexpr int SP_BITS = 21;
constexpr int SP_MAX = 1 << SP_BITS;
constexpr uint64_t SP_NONE = ~0ull;   // sorts after every site key

constexpr int CT_R = 64;              // conv tile: output rows per CTA
constexpr int CT_K = 32;              //            input channels per shared-memory stage
constexpr int CT_THREADS = 256;       // 16 x 16 threads, 4 rows x NJ channels each (16 NJ channels per CTA)

__host__ __device__ __forceinline__ uint64_t sp_key(int x, int y, int z) {
  return ((uint64_t)x << (2 * SP_BITS)) | ((uint64_t)y << SP_BITS) | (uint64_t)z;
}
__device__ __forceinline__ int sp_coord(uint64_t key, int axis) {
  return (int)((key >> (SP_BITS * (2 - axis))) & (SP_MAX - 1));
}

unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

__global__ void point_key_kernel(const int32_t *__restrict__ coords, int N, uint64_t *__restrict__ key,
                                 int32_t *__restrict__ val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  key[i] = sp_key(coords[3 * (size_t)i], coords[3 * (size_t)i + 1], coords[3 * (size_t)i + 2]);
  val[i] = i;
}

// parent key of every child row below *nvox whose parent lies inside the coarse shape (sx, sy, sz), else SP_NONE
__global__ void parent_key_kernel(const int32_t *__restrict__ vox, const int32_t *__restrict__ nvox, int M, int sx,
                                  int sy, int sz, uint64_t *__restrict__ key, int32_t *__restrict__ val) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= M) return;
  val[v] = v;
  if (v >= *nvox) {
    key[v] = SP_NONE;
    return;
  }
  const int px = vox[3 * (size_t)v] >> 1, py = vox[3 * (size_t)v + 1] >> 1, pz = vox[3 * (size_t)v + 2] >> 1;
  key[v] = px < sx && py < sy && pz < sz ? sp_key(px, py, pz) : SP_NONE;
}

__global__ void head_kernel(const uint64_t *__restrict__ key, int M, int32_t *__restrict__ head) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < M) head[j] = key[j] != SP_NONE && (j == 0 || key[j] != key[j - 1]) ? 1 : 0;
}

// sorted (key, row) pairs -> the level: its keys and sites in key order, its size, and each row's site (-1: none)
__global__ void emit_level_kernel(const uint64_t *__restrict__ key, const int32_t *__restrict__ row,
                                  const int32_t *__restrict__ head, const int32_t *__restrict__ vid, int M,
                                  uint64_t *__restrict__ vkey, int32_t *__restrict__ vox, int32_t *__restrict__ nvox,
                                  int32_t *__restrict__ row_site) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= M) return;
  if (j == M - 1) *nvox = vid[j] + head[j];
  if (key[j] == SP_NONE) {
    row_site[row[j]] = -1;
    return;
  }
  const int v = vid[j] + head[j] - 1;
  row_site[row[j]] = v;
  if (head[j]) {
    vkey[v] = key[j];
    for (int a = 0; a < 3; a++) vox[3 * (size_t)v + a] = sp_coord(key[j], a);
  }
}

// nbr[v][k] for every (v, k) with v < M: the site at v + (kx-1, ky-1, kz-1) by binary search, -1 when absent or v is
// past the level's size
__global__ void nbr_kernel(const uint64_t *__restrict__ vkey, const int32_t *__restrict__ nvox, int M,
                           int32_t *__restrict__ nbr) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)M * 27) return;
  const int v = (int)(t / 27), k = (int)(t % 27);
  const int n = *nvox;
  int found = -1;
  if (v < n) {
    const uint64_t key = vkey[v];
    const int x = sp_coord(key, 0) + k / 9 - 1, y = sp_coord(key, 1) + k / 3 % 3 - 1, z = sp_coord(key, 2) + k % 3 - 1;
    if (x >= 0 && y >= 0 && z >= 0 && x < SP_MAX && y < SP_MAX && z < SP_MAX) {
      const uint64_t q = sp_key(x, y, z);
      int lo = 0, hi = n;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (vkey[mid] < q) lo = mid + 1; else hi = mid;
      }
      if (lo < n && vkey[lo] == q) found = lo;
    }
  }
  nbr[t] = found;
}

// down[p][k] = child, up[c][k] = parent; both tables were set to -1 before
__global__ void pairs_kernel(const int32_t *__restrict__ vox, const int32_t *__restrict__ parent, int M,
                             int32_t *__restrict__ down, int32_t *__restrict__ up) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= M) return;
  const int p = parent[c];
  if (p < 0) return;
  const int k = (vox[3 * (size_t)c] & 1) << 2 | (vox[3 * (size_t)c + 1] & 1) << 1 | (vox[3 * (size_t)c + 2] & 1);
  down[8 * (size_t)p + k] = c;
  up[8 * (size_t)c + k] = p;
}

// sorted (key, row) pairs of M rows -> head flags, their scan, the level (at most Mout sites, the caller's bound) and
// its neighbour table (Mout rows)
int build_level(cg_ctx *ctx, const uint64_t *skey, const int32_t *srow, int M, int Mout, int32_t *head, int32_t *vid,
                void *tmp, size_t tmp_bytes, uint64_t *vkey, int32_t *vox, int32_t *nvox, int32_t *row_site,
                int32_t *nbr) {
  cudaStream_t st = ctx->stream;
  head_kernel<<<blocks(M, 256), 256, 0, st>>>(skey, M, head);
  CG_LAUNCH_CHECK(ctx);
  size_t tb = tmp_bytes;
  CG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp, tb, head, vid, M, st));
  emit_level_kernel<<<blocks(M, 256), 256, 0, st>>>(skey, srow, head, vid, M, vkey, vox, nvox, row_site);
  CG_LAUNCH_CHECK(ctx);
  nbr_kernel<<<blocks((int64_t)Mout * 27, 256), 256, 0, st>>>(vkey, nvox, Mout, nbr);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

// scratch of one level build over M rows
struct LevelWs {
  uint64_t *kA, *kB, *vkey;
  int32_t *rA, *rB, *head, *vid;
  void *tmp;
  size_t tmp_bytes;
};

int carve_level(cg_ctx *ctx, int M, LevelWs &w) {
  size_t sort_tmp = 0, scan_tmp = 0;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (uint64_t *)nullptr, (uint64_t *)nullptr,
                                               (int32_t *)nullptr, (int32_t *)nullptr, M, 0, 64, ctx->stream));
  CG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (int32_t *)nullptr, (int32_t *)nullptr, M, ctx->stream));
  w.tmp_bytes = std::max(sort_tmp, scan_tmp);
  const size_t Mz = (size_t)M;
  return cg_ws_carve(ctx, [&](cg_arena &ar) {
    w.kA = ar.take<uint64_t>(Mz); w.kB = ar.take<uint64_t>(Mz); w.vkey = ar.take<uint64_t>(Mz);
    w.rA = ar.take<int32_t>(Mz); w.rB = ar.take<int32_t>(Mz);
    w.head = ar.take<int32_t>(Mz); w.vid = ar.take<int32_t>(Mz);
    w.tmp = ar.take<char>(w.tmp_bytes);
  });
}

// one output tile of CT_R rows x 16 NJ channels (NJ = 1, 2 or 4, picked from Cout so a narrow layer does not run
// zero columns); see the file comment for the arithmetic, which does not depend on NJ.  Rows from min(*nout, M) on
// are not touched: M is the row count of nbr, residual and out.
template <int NJ>
__global__ void __launch_bounds__(CT_THREADS) spconv_kernel(
    const float *__restrict__ in, int Cin, const int32_t *__restrict__ nbr, int K, const int32_t *__restrict__ nout,
    int M, const float *__restrict__ W, int Cout, const float *__restrict__ scale, const float *__restrict__ shift,
    const float *__restrict__ bias, const float *__restrict__ res, float *__restrict__ out) {
  constexpr int CT_C = 16 * NJ;
  __shared__ float As[CT_R][CT_K + 1];
  __shared__ float Ws[CT_K][CT_C];
  __shared__ int32_t src[CT_R];
  const int n = min(*nout, M);
  const int r0 = blockIdx.x * CT_R;
  if (r0 >= n) return;   // the whole CTA leaves together
  const int c0 = blockIdx.y * CT_C;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float acc[4][NJ];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < NJ; j++) acc[i][j] = 0.f;

  for (int k = 0; k < K; k++) {
    int s = -1;
    if (tid < CT_R) {
      const int r = r0 + tid;
      s = r < n ? (nbr ? nbr[(size_t)r * K + k] : r) : -1;
    }
    __syncthreads();   // the previous offset's readers of src are done
    if (tid < CT_R) src[tid] = s;
    if (!__syncthreads_or(s >= 0)) continue;   // no row of the tile has this offset
    for (int cb = 0; cb < Cin; cb += CT_K) {
      for (int e = tid; e < CT_R * CT_K; e += CT_THREADS) {
        const int row = e / CT_K, ci = e % CT_K, c = cb + ci;
        const int sr = src[row];
        float a = 0.f;
        if (sr >= 0 && c < Cin) {
          a = in[(size_t)sr * Cin + c];
          if (scale) a = fmaxf(fmaf(a, scale[c], shift[c]), 0.f);
        }
        As[row][ci] = a;
      }
      for (int e = tid; e < CT_K * CT_C; e += CT_THREADS) {
        const int ci = e / CT_C, co = e % CT_C, c = cb + ci, o = c0 + co;
        Ws[ci][co] = c < Cin && o < Cout ? W[((size_t)k * Cin + c) * Cout + o] : 0.f;
      }
      __syncthreads();
      const int kn = min(CT_K, Cin - cb);
      for (int ci = 0; ci < kn; ci++) {
        float a[4], w[NJ];
#pragma unroll
        for (int i = 0; i < 4; i++) a[i] = As[ty + 16 * i][ci];
#pragma unroll
        for (int j = 0; j < NJ; j++) w[j] = Ws[ci][tx + 16 * j];
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < NJ; j++) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int r = r0 + ty + 16 * i;
    if (r >= n) continue;
#pragma unroll
    for (int j = 0; j < NJ; j++) {
      const int o = c0 + tx + 16 * j;
      if (o >= Cout) continue;
      float v = acc[i][j];
      if (bias) v = __fadd_rn(v, bias[o]);
      if (res) v = __fadd_rn(v, res[(size_t)r * Cout + o]);
      out[(size_t)r * Cout + o] = v;
    }
  }
}

}  // namespace

extern "C" int cg_spconv_index_dev(cg_ctx *ctx, const int32_t *coords, int N, int32_t *out_vox, int32_t *out_nvox,
                                   int32_t *out_p2v, int32_t *out_nbr) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, N >= 1, "spconv_index: N must be >= 1");
  CG_REQUIRE(ctx, N <= (1 << 30) / 27, "spconv_index: at most 2^30 / 27 points (the neighbour table's int32 index)");
  CG_REQUIRE(ctx, coords && out_vox && out_nvox && out_p2v && out_nbr, "spconv_index: null argument");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  LevelWs w;
  const int rc = carve_level(ctx, N, w);
  if (rc != CG_OK) return rc;
  cudaStream_t st = ctx->stream;
  point_key_kernel<<<blocks(N, 256), 256, 0, st>>>(coords, N, w.kA, w.rA);
  CG_LAUNCH_CHECK(ctx);
  size_t tb = w.tmp_bytes;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.kA, w.kB, w.rA, w.rB, N, 0, 3 * SP_BITS, st));
  return build_level(ctx, w.kB, w.rB, N, N, w.head, w.vid, w.tmp, w.tmp_bytes, w.vkey, out_vox, out_nvox, out_p2v,
                     out_nbr);
}

extern "C" int cg_spconv_down_dev(cg_ctx *ctx, const int32_t *vox, const int32_t *nvox, int M, const int32_t *shape,
                                  int out_rows, int32_t *out_vox, int32_t *out_nvox, int32_t *out_nbr,
                                  int32_t *out_down, int32_t *out_up) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, M >= 1 && M <= (1 << 30) / 27, "spconv_down: M must be in [1, 2^30 / 27]");
  CG_REQUIRE(ctx, vox && nvox && shape && out_vox && out_nvox && out_nbr && out_down && out_up,
             "spconv_down: null argument");
  int cs[3];
  int64_t cells = 1;
  for (int a = 0; a < 3; a++) {
    CG_REQUIRE(ctx, shape[a] >= 1 && shape[a] <= SP_MAX, "spconv_down: shape must be in [1, 2^21] per axis");
    cs[a] = shape[a] >= 2 ? (shape[a] - 2) / 2 + 1 : 0;   // get_conv_output_size for k2 s2 p0
    cells *= cs[a];
  }
  // a parent has at least one child and is a cell of the coarse shape
  CG_REQUIRE(ctx, out_rows >= std::max<int64_t>(1, std::min<int64_t>(M, cells)),
             "spconv_down: out_rows must be at least min(M, coarse cells) and >= 1");
  CG_REQUIRE(ctx, out_rows <= (1 << 30) / 27, "spconv_down: out_rows must be <= 2^30 / 27");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  LevelWs w;
  int rc = carve_level(ctx, M, w);
  if (rc != CG_OK) return rc;
  cudaStream_t st = ctx->stream;
  parent_key_kernel<<<blocks(M, 256), 256, 0, st>>>(vox, nvox, M, cs[0], cs[1], cs[2], w.kA, w.rA);
  CG_LAUNCH_CHECK(ctx);
  size_t tb = w.tmp_bytes;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.kA, w.kB, w.rA, w.rB, M, 0, 64, st));
  // rA is free after the sort: it takes each child's parent row (-1: dropped, or a row past *nvox)
  rc = build_level(ctx, w.kB, w.rB, M, out_rows, w.head, w.vid, w.tmp, w.tmp_bytes, w.vkey, out_vox, out_nvox, w.rA,
                   out_nbr);
  if (rc != CG_OK) return rc;
  CG_CUDA(ctx, cudaMemsetAsync(out_down, 0xff, sizeof(int32_t) * 8 * (size_t)out_rows, st));
  CG_CUDA(ctx, cudaMemsetAsync(out_up, 0xff, sizeof(int32_t) * 8 * (size_t)M, st));
  pairs_kernel<<<blocks(M, 256), 256, 0, st>>>(vox, w.rA, M, out_down, out_up);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_spconv_conv_dev(cg_ctx *ctx, const float *in, int Cin, const int32_t *nbr, int K,
                                  const int32_t *nout, int M, const float *W, int Cout, const float *bn_scale,
                                  const float *bn_shift, const float *bias, const float *residual, float *out) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, Cin >= 1 && Cout >= 1 && K >= 1 && M >= 1, "spconv_conv: Cin, Cout, K and M must be >= 1");
  CG_REQUIRE(ctx, nbr || K == 1, "spconv_conv: without a gather table K must be 1");
  CG_REQUIRE(ctx, in && nout && W && out, "spconv_conv: null argument");
  CG_REQUIRE(ctx, !bn_scale == !bn_shift, "spconv_conv: give both BN scale and shift, or neither");
  CG_REQUIRE(ctx, (size_t)M * (size_t)K < ((size_t)1 << 31) && (size_t)M * Cout < ((size_t)1 << 40),
             "spconv_conv: table or output too large");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const int nj = Cout <= 16 ? 1 : Cout <= 32 ? 2 : 4;
  const dim3 grid(blocks(M, CT_R), blocks(Cout, 16 * nj));
  auto kernel = nj == 1 ? spconv_kernel<1> : nj == 2 ? spconv_kernel<2> : spconv_kernel<4>;
  kernel<<<grid, CT_THREADS, 0, ctx->stream>>>(in, Cin, nbr, K, nout, M, W, Cout, bn_scale, bn_shift, bias, residual,
                                               out);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}
