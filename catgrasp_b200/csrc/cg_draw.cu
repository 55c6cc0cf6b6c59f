// cg_draw.cu -- opt-in device-side point-subset draw for the grasp-Q scorer (subsample="device").
//
// The reference draws each candidate's n_pts point subset with the global numpy generator on the host
// (np.random.choice, dataset_grasp.py:72-73) -- a full Fisher-Yates shuffle of the M scene points per candidate, which
// caps GraspPredicter.predict_batch at a few thousand candidates/s however fast the GPU is.  This kernel draws a
// statistically equivalent subset on the device with a counter-based generator: NOT the reference's numbers (it cannot
// be: the MT19937 stream is sequential), same distribution:
//   M >= n_pts  (reference: replace=False)  ids[b][n] = P_b(n), n = 0..n_pts-1, where P_b is a keyed pseudo-random
//               PERMUTATION of [0, M): an 8-round balanced Feistel network over the smallest even-width power of two
//               >= M, cycle-walked back into range -> n_pts distinct, uniformly distributed indices, no memory, no
//               sequential dependency;
//   M <  n_pts  (reference: replace=True)   ids[b][n] = floor(u * M), u from a 32-bit hash of (seed, candidate, n).
// The key depends on (seed, first_candidate + b) only, so a candidate gets the same subset whichever rank scores it.
#include "cg_common.cuh"

namespace {

__device__ __forceinline__ uint32_t mix32(uint32_t x) {   // lowbias32 finaliser (full-avalanche 32-bit bijection)
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}

// With n_obj > 0 the launch draws for n_obj objects: global row r belongs to the object o with
// obj_row[o] <= r < obj_row[o + 1], is that object's candidate r - obj_row[o] under its own M and seed, and its ids
// are written plus obj_base[o]; M, seed_lo, seed_hi and first_candidate are then unused.
__global__ void draw_ids_kernel(int M, int n_pts, int count, uint32_t seed_lo, uint32_t seed_hi, long long first_candidate,
                                int32_t *__restrict__ out, int n_obj, const int32_t *__restrict__ obj_M,
                                const uint64_t *__restrict__ obj_seed, const int64_t *__restrict__ obj_row,
                                const int32_t *__restrict__ obj_base) {
  const long long total = (long long)count * n_pts;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    int b = (int)(idx / n_pts);
    const int n = (int)(idx - (long long)b * n_pts);
    int Mo = M, base = 0;
    uint32_t slo = seed_lo, shi = seed_hi;
    long long cand0 = first_candidate;
    if (n_obj > 0) {   // the last object whose first row is <= b (objects with no rows share their successor's)
      int lo = 0, hi = n_obj - 1;
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (obj_row[mid] <= b) lo = mid;
        else hi = mid - 1;
      }
      Mo = obj_M[lo];
      slo = (uint32_t)obj_seed[lo];
      shi = (uint32_t)(obj_seed[lo] >> 32);
      base = obj_base[lo];
      b -= (int)obj_row[lo];
      cand0 = 0;
    }
    // Feistel geometry: domain 2^(2h) >= M
    int bits = 32 - __clz((unsigned)(Mo - 1) | 1u);
    if (Mo <= 1) bits = 1;
    const int h = (bits + 1) >> 1;
    const uint32_t hmask = (1u << h) - 1u;
    const unsigned long long cand = (unsigned long long)(cand0 + b);
    const uint32_t k0 = mix32(slo ^ mix32((uint32_t)cand + 0x9e3779b9u));
    const uint32_t k1 = mix32(shi ^ mix32((uint32_t)(cand >> 32) + 0x85ebca6bu) ^ k0);
    uint32_t v;
    if (Mo < n_pts) {
      const uint32_t u = mix32(k0 ^ mix32((uint32_t)n * 0x9e3779b1u + k1));
      v = (uint32_t)(((unsigned long long)u * (unsigned)Mo) >> 32);
    } else {
      uint32_t x = (uint32_t)n;
      do {   // cycle walking: re-encrypt until the value falls into [0, M); the domain is < 4M, so < 4 rounds on average
        uint32_t L = x >> h, R = x & hmask;
#pragma unroll
        for (int r = 0; r < 8; r++) {
          const uint32_t f = mix32(R ^ (r & 1 ? k1 : k0) ^ ((uint32_t)r * 0x9e3779b9u)) & hmask;
          const uint32_t nl = R;
          R = L ^ f;
          L = nl;
        }
        x = (L << h) | R;
      } while (x >= (uint32_t)Mo);
      v = x;
    }
    out[idx] = (int32_t)v + base;
  }
}

}  // namespace

extern "C" int cg_draw_ids_dev(cg_ctx *ctx, int M, int n_pts, int count, uint64_t seed, int64_t first_candidate,
                               int32_t *out_ids) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, out_ids && M > 0 && n_pts > 0 && count > 0, "draw_ids: bad arguments");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const long long total = (long long)count * n_pts;
  int blocks = (int)((total + 255) / 256);
  const int cap = ctx->num_sms * 16;
  if (blocks > cap) blocks = cap;
  draw_ids_kernel<<<blocks, 256, 0, ctx->stream>>>(M, n_pts, count, (uint32_t)seed, (uint32_t)(seed >> 32), first_candidate,
                                                   out_ids, 0, nullptr, nullptr, nullptr, nullptr);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}

extern "C" int cg_draw_ids_many_dev(cg_ctx *ctx, int n_obj, const int32_t *M, const uint64_t *seed,
                                    const int64_t *row_offsets, const int32_t *base, int n_pts, int rows,
                                    int32_t *out_ids) {
  if (!ctx) return CG_EINVAL;
  CG_REQUIRE(ctx, out_ids && M && seed && row_offsets && base && n_obj > 0 && n_pts > 0 && rows > 0,
             "draw_ids_many: bad arguments");
  CG_CUDA(ctx, cudaSetDevice(ctx->device));
  const long long total = (long long)rows * n_pts;
  long long blocks = (total + 255) / 256;
  const int cap = ctx->num_sms * 16;
  if (blocks > cap) blocks = cap;
  draw_ids_kernel<<<(int)blocks, 256, 0, ctx->stream>>>(0, n_pts, rows, 0u, 0u, 0, out_ids, n_obj, M, seed, row_offsets,
                                                        base);
  CG_LAUNCH_CHECK(ctx);
  return CG_OK;
}
