// cg_spconv.cu -- sparse 3-D convolution with spconv 1.x semantics, the layer types of PointGroup's U-Net
// (SubMConv3d k3 / k1, SparseConv3d k2 s2, SparseInverseConv3d k2; PointGroup/model/pointgroup/pointgroup.py).
//
// A level is a set of distinct integer sites (x, y, z), each in [0, 2^21), packed into the 63-bit key
// x << 42 | y << 21 | z and held in ascending key order: row-major over (x, y, z), z fastest.  The order of a level's
// rows reaches no output of the network (every gather goes through a table), so key order is the contract.
//
// A batched level holds the sites of B > 1 frames, each on its own spatial shape S_b, with the frame above the
// coordinates: key = b << 3w | x << 2w | y << w | z, where w is the smallest width with 2^w >= every S_b on every axis
// and the frame field takes f = bit_length(B - 1) bits; f + 3w <= 63, else the batch is refused.  So a batched level is
// its frames' one-frame levels one after another, frame b's rows starting at its row base (the sites of the frames
// before it), and every table entry of frame b is the one-frame entry plus that base.  Neighbours are bounded by the
// field, 2^w, so no coordinate carries into the next field.  With one frame the layout is the one above (f = 0,
// w = 21), whatever the shape.
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
// is max(1, min(the finer level's rows, the cells of the coarse shapes summed over the frames)): every parent has a
// child and is a coarse cell of its child's frame.
#include <cub/cub.cuh>
#include "cg_common.cuh"

namespace {

constexpr int SP_BITS = 21;
constexpr int SP_MAX = 1 << SP_BITS;
constexpr uint64_t SP_NONE = ~0ull;   // sorts after every site key

constexpr int CT_R = 64;              // conv tile: output rows per CTA
constexpr int CT_K = 32;              //            input channels per shared-memory stage
constexpr int CT_THREADS = 256;       // 16 x 16 threads, 4 rows x NJ channels each (16 NJ channels per CTA)

// the key of site (x, y, z) of frame b in fields of w bits
__host__ __device__ __forceinline__ uint64_t sp_key(int b, int x, int y, int z, int w) {
  return ((uint64_t)b << (3 * w)) | ((uint64_t)x << (2 * w)) | ((uint64_t)y << w) | (uint64_t)z;
}
__device__ __forceinline__ int sp_coord(uint64_t key, int axis, int w) {
  return (int)((key >> (w * (2 - axis))) & ((1ull << w) - 1));
}

unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

// each point's key; frame b's points are rows [off[b], off[b + 1]) of coords (off null: one frame)
__global__ void point_key_kernel(const int32_t *__restrict__ coords, int N, const int32_t *__restrict__ off, int B,
                                 int w, uint64_t *__restrict__ key, int32_t *__restrict__ val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  int b = 0;
  if (off) {   // the last frame whose first row is <= i
    int lo = 0, hi = B - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (off[mid] <= i) lo = mid; else hi = mid - 1;
    }
    b = lo;
  }
  key[i] = sp_key(b, coords[3 * (size_t)i], coords[3 * (size_t)i + 1], coords[3 * (size_t)i + 2], w);
  val[i] = i;
}

// parent key of every child row below *nvox whose parent lies inside its frame's coarse shape cshape[3 b ..], else
// SP_NONE; frame[v] is the child's frame (null: frame 0)
__global__ void parent_key_kernel(const int32_t *__restrict__ vox, const int32_t *__restrict__ frame,
                                  const int32_t *__restrict__ nvox, int M, const int32_t *__restrict__ cshape, int w,
                                  uint64_t *__restrict__ key, int32_t *__restrict__ val) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= M) return;
  val[v] = v;
  if (v >= *nvox) {
    key[v] = SP_NONE;
    return;
  }
  const int b = frame ? frame[v] : 0;
  const int px = vox[3 * (size_t)v] >> 1, py = vox[3 * (size_t)v + 1] >> 1, pz = vox[3 * (size_t)v + 2] >> 1;
  const int *cs = cshape + 3 * (size_t)b;
  key[v] = px < cs[0] && py < cs[1] && pz < cs[2] ? sp_key(b, px, py, pz, w) : SP_NONE;
}

__global__ void head_kernel(const uint64_t *__restrict__ key, int M, int32_t *__restrict__ head) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < M) head[j] = key[j] != SP_NONE && (j == 0 || key[j] != key[j - 1]) ? 1 : 0;
}

// sorted (key, row) pairs -> the level: its keys, sites and frames (frame null: not written) in key order, its size,
// and each row's site (-1: none)
__global__ void emit_level_kernel(const uint64_t *__restrict__ key, const int32_t *__restrict__ row,
                                  const int32_t *__restrict__ head, const int32_t *__restrict__ vid, int M, int w,
                                  uint64_t *__restrict__ vkey, int32_t *__restrict__ vox, int32_t *__restrict__ frame,
                                  int32_t *__restrict__ nvox, int32_t *__restrict__ row_site) {
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
    for (int a = 0; a < 3; a++) vox[3 * (size_t)v + a] = sp_coord(key[j], a, w);
    if (frame) frame[v] = (int)(key[j] >> (3 * w));
  }
}

// nbr[v][k] for every (v, k) with v < M: the site at v + (kx-1, ky-1, kz-1) of the same frame by binary search, -1 when
// absent, outside the w-bit fields or v is past the level's size
__global__ void nbr_kernel(const uint64_t *__restrict__ vkey, const int32_t *__restrict__ nvox, int M, int w,
                           int32_t *__restrict__ nbr) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)M * 27) return;
  const int v = (int)(t / 27), k = (int)(t % 27);
  const int n = *nvox;
  int found = -1;
  if (v < n) {
    const uint64_t key = vkey[v];
    const int lim = 1 << w;
    const int x = sp_coord(key, 0, w) + k / 9 - 1, y = sp_coord(key, 1, w) + k / 3 % 3 - 1,
              z = sp_coord(key, 2, w) + k % 3 - 1;
    if (x >= 0 && y >= 0 && z >= 0 && x < lim && y < lim && z < lim) {
      const uint64_t q = sp_key((int)(key >> (3 * w)), x, y, z, w);
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

// sorted (key, row) pairs of M rows -> head flags, their scan, the level (at most Mout sites, the caller's bound; its
// frames too when frame is given) and its neighbour table (Mout rows)
int build_level(cg_ctx *ctx, const uint64_t *skey, const int32_t *srow, int M, int Mout, int w, int32_t *head,
                int32_t *vid, void *tmp, size_t tmp_bytes, uint64_t *vkey, int32_t *vox, int32_t *frame,
                int32_t *nvox, int32_t *row_site, int32_t *nbr) {
  cudaStream_t st = ctx->stream;
  head_kernel<<<blocks(M, 256), 256, 0, st>>>(skey, M, head);
  CG_LAUNCH_CHECK(ctx);
  size_t tb = tmp_bytes;
  CG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp, tb, head, vid, M, st));
  emit_level_kernel<<<blocks(M, 256), 256, 0, st>>>(skey, srow, head, vid, M, w, vkey, vox, frame, nvox, row_site);
  CG_LAUNCH_CHECK(ctx);
  nbr_kernel<<<blocks((int64_t)Mout * 27, 256), 256, 0, st>>>(vkey, nvox, Mout, w, nbr);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

int bit_length(int v) {
  int n = 0;
  while (v >> n) n++;
  return n;
}

// The one table build behind cg_spconv_{index,down}_dev and their _many forms, for B frames on the host shapes
// (3 per frame; null for a one-frame index, which needs no shape).  Checks its arguments before any launch.
//   index (coords given): the M points coords, frame b's at rows [off[b], off[b + 1]) (off: host, null for one
//     frame) -> the level of their sites in out_rows = M rows, out_p2v = each point's site
//   down (vox given): the M rows of a level with *nvox sites, site v of frame frame[v] (null: one frame) -> the level
//     of their parents in out_rows rows, out_down (out_rows,8) and out_up (M,8)
// out_frame (null: not written) takes each site's frame.
int spconv_tables(cg_ctx *ctx, const std::string &who, int B, const int32_t *shapes, const int32_t *off,
                  const int32_t *coords, const int32_t *vox, const int32_t *frame, const int32_t *nvox, int M,
                  int out_rows, int32_t *out_vox, int32_t *out_nvox, int32_t *out_frame, int32_t *out_nbr,
                  int32_t *out_p2v, int32_t *out_down, int32_t *out_up) {
  const bool down = vox != nullptr;
  CG_REQUIRE(ctx, B >= 1, who + ": B must be >= 1");
  // the key layout (file comment): one frame keeps f = 0, w = 21
  int f = 0, w = SP_BITS, smax = 1;
  if (shapes) {
    for (int i = 0; i < 3 * B; i++) {
      CG_REQUIRE(ctx, shapes[i] >= 1 && shapes[i] <= SP_MAX, who + ": shape must be in [1, 2^21] per axis");
      smax = std::max(smax, shapes[i]);
    }
  }
  if (B > 1) {
    f = bit_length(B - 1);
    w = bit_length(smax - 1);
    CG_REQUIRE(ctx, f + 3 * w <= 63,
               who + ": " + std::to_string(B) + " frames need " + std::to_string(f) + " frame bits and a largest "
               "shape of " + std::to_string(smax) + " needs " + std::to_string(w) + " bits per axis; the key holds "
               "f + 3 w <= 63");
  }
  std::vector<int32_t> cs;
  if (down) {
    // get_conv_output_size for k2 s2 p0, per frame; a parent has at least one child and is a cell of its frame
    int64_t cells = 0;
    cs.resize(3 * (size_t)B);
    for (int b = 0; b < B; b++) {
      int64_t n = 1;
      for (int a = 0; a < 3; a++) {
        const int S = shapes[3 * b + a];
        cs[3 * b + a] = S >= 2 ? (S - 2) / 2 + 1 : 0;
        n *= cs[3 * b + a];
      }
      cells += n;
    }
    CG_REQUIRE(ctx, out_rows >= std::max<int64_t>(1, std::min<int64_t>(M, cells)),
               who + ": out_rows must be at least min(M, coarse cells) and >= 1");
    CG_REQUIRE(ctx, out_rows <= (1 << 30) / 27, who + ": out_rows must be <= 2^30 / 27");
  } else if (off) {
    CG_REQUIRE(ctx, off[0] == 0 && off[B] == M, who + ": the frame offsets must run from 0 to N");
    for (int b = 0; b < B; b++) CG_REQUIRE(ctx, off[b] <= off[b + 1], who + ": the frame offsets must not decrease");
  }
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  size_t sort_tmp = 0, scan_tmp = 0;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (uint64_t *)nullptr, (uint64_t *)nullptr,
                                               (int32_t *)nullptr, (int32_t *)nullptr, M, 0, 64, st));
  CG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (int32_t *)nullptr, (int32_t *)nullptr, M, st));
  const size_t tmp_bytes = std::max(sort_tmp, scan_tmp), Mz = (size_t)M;
  const size_t n_off = !down && off ? (size_t)B + 1 : 0;
  uint64_t *kA, *kB, *vkey;
  int32_t *rA, *rB, *head, *vid, *d_off, *d_cs;
  void *tmp;
  int rc = cg_ws_carve(ctx, [&](cg_arena &ar) {
    kA = ar.take<uint64_t>(Mz); kB = ar.take<uint64_t>(Mz); vkey = ar.take<uint64_t>(Mz);
    rA = ar.take<int32_t>(Mz); rB = ar.take<int32_t>(Mz);
    head = ar.take<int32_t>(Mz); vid = ar.take<int32_t>(Mz);
    tmp = ar.take<char>(tmp_bytes);
    d_off = ar.take<int32_t>(n_off); d_cs = ar.take<int32_t>(cs.size());
  });
  if (rc != CG_OK) return rc;
  // the frame tables, from pageable memory: staged at once, no synchronisation
  if (n_off) CG_CUDA(ctx, cudaMemcpyAsync(d_off, off, sizeof(int32_t) * n_off, cudaMemcpyHostToDevice, st));
  if (down) CG_CUDA(ctx, cudaMemcpyAsync(d_cs, cs.data(), sizeof(int32_t) * cs.size(), cudaMemcpyHostToDevice, st));
  size_t tb = tmp_bytes;
  if (!down) {
    point_key_kernel<<<blocks(M, 256), 256, 0, st>>>(coords, M, n_off ? d_off : nullptr, B, w, kA, rA);
    CG_LAUNCH_CHECK(ctx);
    CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp, tb, kA, kB, rA, rB, M, 0, f + 3 * w, st));
    return build_level(ctx, kB, rB, M, M, w, head, vid, tmp, tmp_bytes, vkey, out_vox, out_frame, out_nvox, out_p2v,
                       out_nbr);
  }
  parent_key_kernel<<<blocks(M, 256), 256, 0, st>>>(vox, frame, nvox, M, d_cs, w, kA, rA);
  CG_LAUNCH_CHECK(ctx);
  // all 64 bits: a dropped child's SP_NONE sorts after every parent key
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp, tb, kA, kB, rA, rB, M, 0, 64, st));
  // rA is free after the sort: it takes each child's parent row (-1: dropped, or a row past *nvox)
  rc = build_level(ctx, kB, rB, M, out_rows, w, head, vid, tmp, tmp_bytes, vkey, out_vox, out_frame, out_nvox, rA,
                   out_nbr);
  if (rc != CG_OK) return rc;
  CG_CUDA(ctx, cudaMemsetAsync(out_down, 0xff, sizeof(int32_t) * 8 * (size_t)out_rows, st));
  CG_CUDA(ctx, cudaMemsetAsync(out_up, 0xff, sizeof(int32_t) * 8 * Mz, st));
  pairs_kernel<<<blocks(M, 256), 256, 0, st>>>(vox, rA, M, out_down, out_up);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
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

// ---- PointGroup's voxelisation (pointgroup_ops mode 4) and offset head around the U-Net ----

// each point's site as a sort key; a point naming no site below *nvox sorts last as ~0u
__global__ void site_key_kernel(const int32_t *__restrict__ p2v, int N, const int32_t *__restrict__ nvox, int V,
                                uint32_t *__restrict__ key, int32_t *__restrict__ val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int v = p2v[i];
  key[i] = v >= 0 && v < min(*nvox, V) ? (uint32_t)v : ~0u;
  val[i] = i;
}

// the sorted keys' runs: site v's points are sorted positions [first[v], last[v]); both were set to 0 before
__global__ void site_run_kernel(const uint32_t *__restrict__ key, int N, int32_t *__restrict__ first,
                                int32_t *__restrict__ last) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N || key[j] == ~0u) return;
  if (j == 0 || key[j - 1] != key[j]) first[key[j]] = j;
  if (j == N - 1 || key[j + 1] != key[j]) last[key[j]] = j + 1;
}

// one thread per (site, channel): out = 0; for each point in ascending index out = fl(out + fl(fl(1/n) * x)), the
// arithmetic of voxelize_fp_cuda_ with average = true, whose atomicAdd rules out a fused multiply-add
__global__ void voxel_mean_kernel(const float *__restrict__ feats, int C, const int32_t *__restrict__ perm,
                                  const int32_t *__restrict__ first, const int32_t *__restrict__ last,
                                  const int32_t *__restrict__ nvox, int V, float *__restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)min(*nvox, V) * C) return;
  const int v = (int)(t / C), c = (int)(t % C);
  const int b = first[v], e = last[v];
  const float mult = e > b ? __fdiv_rn(1.f, (float)(e - b)) : 1.f;
  float acc = 0.f;
  for (int j = b; j < e; j++) acc = __fadd_rn(acc, __fmul_rn(mult, feats[(size_t)perm[j] * C + c]));
  out[t] = acc;
}

constexpr int HD_WARPS = 8;   // offset head: sites (one warp each) per CTA

// one warp per site: a = ReLU(x * s0 + t0) (output_layer), h = ReLU(W1^T a + b1) (Linear with its BN folded in),
// out = W2^T h + b2; each output one fp32 FMA chain over the input channels ascending, then the bias
__global__ void __launch_bounds__(HD_WARPS * 32) offset_head_kernel(
    const float *__restrict__ in, int m, const int32_t *__restrict__ nvox, int V, const float *__restrict__ s0,
    const float *__restrict__ t0, const float *__restrict__ W1, const float *__restrict__ b1,
    const float *__restrict__ W2, const float *__restrict__ b2, float *__restrict__ out) {
  extern __shared__ float hd_sh[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int v = blockIdx.x * HD_WARPS + w;
  if (v >= min(*nvox, V)) return;   // the whole warp leaves together
  float *a = hd_sh + (size_t)w * 2 * m, *h = a + m;
  for (int c = lane; c < m; c += 32) a[c] = fmaxf(fmaf(in[(size_t)v * m + c], s0[c], t0[c]), 0.f);
  __syncwarp();
  for (int o = lane; o < m; o += 32) {
    float acc = 0.f;
    for (int c = 0; c < m; c++) acc = fmaf(a[c], W1[(size_t)c * m + o], acc);
    h[o] = fmaxf(__fadd_rn(acc, b1[o]), 0.f);
  }
  __syncwarp();
  if (lane < 3) {
    float acc = 0.f;
    for (int c = 0; c < m; c++) acc = fmaf(h[c], W2[3 * c + lane], acc);
    out[3 * (size_t)v + lane] = __fadd_rn(acc, b2[lane]);
  }
}

// out[i] = site[p2v[i]] (3 floats), NaN for a point naming no site below *nvox
__global__ void gather3_kernel(const float *__restrict__ site, const int32_t *__restrict__ p2v, int N,
                               const int32_t *__restrict__ nvox, int V, float *__restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 3 * (int64_t)N) return;
  const int i = (int)(t / 3), j = (int)(t % 3);
  const int v = p2v[i];
  out[t] = v >= 0 && v < min(*nvox, V) ? site[3 * (size_t)v + j] : __int_as_float(0x7fc00000);
}

}  // namespace

extern "C" int cg_spconv_index_dev(cg_ctx *ctx, const int32_t *coords, int N, int32_t *out_vox, int32_t *out_nvox,
                                   int32_t *out_p2v, int32_t *out_nbr) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, N >= 1, "spconv_index: N must be >= 1");
  CG_REQUIRE(ctx, N <= (1 << 30) / 27, "spconv_index: at most 2^30 / 27 points (the neighbour table's int32 index)");
  CG_REQUIRE(ctx, coords && out_vox && out_nvox && out_p2v && out_nbr, "spconv_index: null argument");
  return spconv_tables(ctx, "spconv_index", 1, nullptr, nullptr, coords, nullptr, nullptr, nullptr, N, N, out_vox,
                       out_nvox, nullptr, out_nbr, out_p2v, nullptr, nullptr);
}

extern "C" int cg_spconv_index_many_dev(cg_ctx *ctx, const int32_t *coords, int N, int B, const int32_t *offsets,
                                        const int32_t *shapes, int32_t *out_vox, int32_t *out_nvox,
                                        int32_t *out_frame, int32_t *out_p2v, int32_t *out_nbr) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, N >= 1, "spconv_index_many: N must be >= 1");
  CG_REQUIRE(ctx, N <= (1 << 30) / 27,
             "spconv_index_many: at most 2^30 / 27 points (the neighbour table's int32 index)");
  CG_REQUIRE(ctx, coords && offsets && shapes && out_vox && out_nvox && out_frame && out_p2v && out_nbr,
             "spconv_index_many: null argument");
  return spconv_tables(ctx, "spconv_index_many", B, shapes, offsets, coords, nullptr, nullptr, nullptr, N, N, out_vox,
                       out_nvox, out_frame, out_nbr, out_p2v, nullptr, nullptr);
}

extern "C" int cg_spconv_down_dev(cg_ctx *ctx, const int32_t *vox, const int32_t *nvox, int M, const int32_t *shape,
                                  int out_rows, int32_t *out_vox, int32_t *out_nvox, int32_t *out_nbr,
                                  int32_t *out_down, int32_t *out_up) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, M >= 1 && M <= (1 << 30) / 27, "spconv_down: M must be in [1, 2^30 / 27]");
  CG_REQUIRE(ctx, vox && nvox && shape && out_vox && out_nvox && out_nbr && out_down && out_up,
             "spconv_down: null argument");
  return spconv_tables(ctx, "spconv_down", 1, shape, nullptr, nullptr, vox, nullptr, nvox, M, out_rows, out_vox,
                       out_nvox, nullptr, out_nbr, nullptr, out_down, out_up);
}

extern "C" int cg_spconv_down_many_dev(cg_ctx *ctx, const int32_t *vox, const int32_t *frame, const int32_t *nvox,
                                       int M, int B, const int32_t *shapes, int out_rows, int32_t *out_vox,
                                       int32_t *out_nvox, int32_t *out_frame, int32_t *out_nbr, int32_t *out_down,
                                       int32_t *out_up) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, M >= 1 && M <= (1 << 30) / 27, "spconv_down_many: M must be in [1, 2^30 / 27]");
  CG_REQUIRE(ctx, vox && frame && nvox && shapes && out_vox && out_nvox && out_frame && out_nbr && out_down && out_up,
             "spconv_down_many: null argument");
  return spconv_tables(ctx, "spconv_down_many", B, shapes, nullptr, nullptr, vox, frame, nvox, M, out_rows, out_vox,
                       out_nvox, out_frame, out_nbr, nullptr, out_down, out_up);
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

extern "C" int cg_pointgroup_voxel_mean_dev(cg_ctx *ctx, const float *feats, int N, int C, const int32_t *p2v,
                                            const int32_t *nvox, int V, float *out) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, N >= 1 && C >= 1 && V >= 1, "pointgroup_voxel_mean: N, C and V must be >= 1");
  CG_REQUIRE(ctx, (int64_t)V * C < ((int64_t)1 << 40) && (int64_t)N * C < ((int64_t)1 << 40),
             "pointgroup_voxel_mean: features too large");
  CG_REQUIRE(ctx, feats && p2v && nvox && out, "pointgroup_voxel_mean: null argument");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  size_t sort_tmp = 0;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (uint32_t *)nullptr, (uint32_t *)nullptr,
                                               (int32_t *)nullptr, (int32_t *)nullptr, N, 0, 32, st));
  uint32_t *kA, *kB;
  int32_t *rA, *rB, *first, *last;
  void *tmp;
  const size_t Nz = (size_t)N, Vz = (size_t)V;
  const int rc = cg_ws_carve(ctx, [&](cg_arena &ar) {
    kA = ar.take<uint32_t>(Nz); kB = ar.take<uint32_t>(Nz);
    rA = ar.take<int32_t>(Nz); rB = ar.take<int32_t>(Nz);
    first = ar.take<int32_t>(Vz); last = ar.take<int32_t>(Vz);
    tmp = ar.take<char>(sort_tmp);
  });
  if (rc != CG_OK) return rc;
  site_key_kernel<<<blocks(N, 256), 256, 0, st>>>(p2v, N, nvox, V, kA, rA);
  CG_LAUNCH_CHECK(ctx);
  // a stable sort: each site's points stay in ascending index order
  size_t tb = sort_tmp;
  CG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp, tb, kA, kB, rA, rB, N, 0, 32, st));
  CG_CUDA(ctx, cudaMemsetAsync(first, 0, sizeof(int32_t) * Vz, st));
  CG_CUDA(ctx, cudaMemsetAsync(last, 0, sizeof(int32_t) * Vz, st));
  site_run_kernel<<<blocks(N, 256), 256, 0, st>>>(kB, N, first, last);
  CG_LAUNCH_CHECK(ctx);
  voxel_mean_kernel<<<blocks((int64_t)V * C, 256), 256, 0, st>>>(feats, C, rB, first, last, nvox, V, out);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_pointgroup_head_dev(cg_ctx *ctx, const float *in, int m, const int32_t *nvox, int V,
                                      const float *bn_scale, const float *bn_shift, const float *W1, const float *b1,
                                      const float *W2, const float *b2, const int32_t *p2v, int N, float *out_site,
                                      float *out) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, m >= 1 && m <= 512, "pointgroup_head: m must be in [1, 512]");
  CG_REQUIRE(ctx, V >= 1 && N >= 1 && (int64_t)V * m < ((int64_t)1 << 40), "pointgroup_head: V and N must be >= 1");
  CG_REQUIRE(ctx, in && nvox && bn_scale && bn_shift && W1 && b1 && W2 && b2 && p2v && out_site && out,
             "pointgroup_head: null argument");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t shm = sizeof(float) * HD_WARPS * 2 * (size_t)m;
  if (shm > 48 * 1024)
    CG_CUDA(ctx, cudaFuncSetAttribute(offset_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
  offset_head_kernel<<<blocks(V, HD_WARPS), HD_WARPS * 32, shm, st>>>(in, m, nvox, V, bn_scale, bn_shift, W1, b1, W2,
                                                                      b2, out_site);
  CG_LAUNCH_CHECK(ctx);
  gather3_kernel<<<blocks(3 * (int64_t)N, 256), 256, 0, st>>>(out_site, p2v, N, nvox, V, out);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}
