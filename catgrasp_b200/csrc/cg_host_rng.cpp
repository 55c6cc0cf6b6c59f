// cg_host_rng.cu -- host-side helper: the reference's per-candidate point-subset draw, bit-identical and fast.
//
// The reference draws every candidate's subset with ONE call of the GLOBAL legacy numpy generator
//     ids = np.random.choice(np.arange(M), size=n_pts, replace=(M < n_pts))        (dataset_grasp.py:72-73)
// i.e. for M >= n_pts a full Fisher-Yates shuffle of arange(M) (RandomState.permutation -> _shuffle_raw, one
// masked-rejection random_interval(i) per element, i = M-1 .. 1) and for M < n_pts n_pts masked-rejection draws
// (RandomState.randint -> random_bounded_uint64_fill, 32-bit path).  A drop-in must consume exactly the same
// MT19937 words, otherwise every later np.random call of the host program diverges from the reference run.
// Doing that through numpy costs a Python-level call + an arange + a copy per candidate (~0.3 ms at M = 20 000);
// this file restates the generator (MT19937 genrand_int32, numpy/random/src/mt19937) and the two draw loops in C:
// the caller passes numpy's state in (np.random.get_state()), gets ids for `count` candidates and the advanced
// state back (np.random.set_state()).  tests/test_abi_and_host.py checks ids AND the post-state against numpy itself.
#if (defined(__x86_64__) || defined(__i386__)) && !defined(CG_HOST_RNG_SCALAR_ONLY)
#define CG_X86 1
#include <immintrin.h>
#else
#define CG_X86 0   // e.g. aarch64 (Grace): the scalar walk and replay below
#endif
#include <stdint.h>
#include <string.h>
#include <time.h>

#include <atomic>
#include <thread>
#include <vector>

#include "../../include/catgrasp_b200.h"

// Layout of the work: (1) regenerating the 624-word state and tempering a block of raw words have no loop-carried
// dependency inside a vector -> AVX-512 / AVX2 variants picked at load time (scalar fallback); (2) which words a shuffle
// ACCEPTS does not depend on the permutation, only on the running index i (`i -= (word & mask) <= i`), so the calling
// thread walks the stream alone ("skip": 16 words per step while no word falls inside the 16-wide ambiguity window under
// i) and snapshots the generator at every candidate boundary; (3) worker threads replay the real shuffles from the
// snapshots.  Above position n_pts a swap only needs its downward half (position i is never read again).

namespace {

constexpr int MT_N = 624, MT_M = 397;
constexpr uint32_t MT_MAG = 0x9908b0dfu, MT_UP = 0x80000000u, MT_LO = 0x7fffffffu;

inline uint32_t mt_mix(uint32_t a, uint32_t b, uint32_t far) {
  const uint32_t y = (a & MT_UP) | (b & MT_LO);
  return far ^ (y >> 1) ^ ((y & 1u) ? MT_MAG : 0u);
}
inline uint32_t temper1(uint32_t y) {
  y ^= (y >> 11);
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= (y >> 18);
  return y;
}
inline uint32_t mask_of(uint32_t max) {
  uint32_t mask = max;
  mask |= mask >> 1;
  mask |= mask >> 2;
  mask |= mask >> 4;
  mask |= mask >> 8;
  mask |= mask >> 16;
  return mask;
}

// ---- scalar -------------------------------------------------------------------------------------------------------
void refill_scalar(uint32_t *mt) {
  int kk = 0;
  for (; kk < MT_N - MT_M; kk++) mt[kk] = mt_mix(mt[kk], mt[kk + 1], mt[kk + MT_M]);
  for (; kk < MT_N - 1; kk++) mt[kk] = mt_mix(mt[kk], mt[kk + 1], mt[kk + (MT_M - MT_N)]);
  mt[MT_N - 1] = mt_mix(mt[MT_N - 1], mt[0], mt[MT_M - 1]);
}
void temper_scalar(const uint32_t *in, uint32_t *out, int n) {
  for (int k = 0; k < n; k++) out[k] = temper1(in[k]);
}
// Accept scan over tempered words w[0..avail): i -= ((w & mask) <= i) per word, mask = smallest all-ones >= i.
// Stops when i reaches 0 or the words run out; returns the number of words consumed.
int scan_scalar(const uint32_t *w, int avail, uint32_t &i_io, uint32_t &mask_io) {
  uint32_t i = i_io, mask = mask_io;
  int k = 0;
  while (k < avail && i >= 1) {
    const uint32_t lim = mask >> 1, m = mask;   // the mask is constant while i stays in (mask >> 1, mask]
    while (k < avail && i > lim) {
      i -= ((w[k] & m) <= i) ? 1u : 0u;
      k++;
    }
    if (i <= lim) mask >>= 1;
  }
  i_io = i;
  mask_io = mask;
  return k;
}

// Upper part of a replay (positions >= low are never read after their own step, so p[j] = p[i] is the whole swap):
// consumes words while i >= low; p[dummy] swallows the store of a rejected word.
int upper_scalar(const uint32_t *w, int avail, uint32_t &i_io, uint32_t &mask_io, uint32_t low, int32_t *p, uint32_t dummy) {
  uint32_t i = i_io, mask = mask_io;
  int k = 0;
  for (; k < avail && i >= low; k++) {
    const uint32_t j = w[k] & mask;
    const uint32_t acc = (j <= i) ? 1u : 0u;
    p[acc ? j : dummy] = p[i];
    i -= acc;
    if ((mask >> 1) >= i) mask >>= 1;   // smallest all-ones mask >= i
  }
  i_io = i;
  mask_io = mask;
  return k;
}

// The scan with the accepted words kept: step i's j goes to js[top - i] (top = M - 1), so js lists the shuffle's
// swap partners from i = M-1 down.  A rejected word's store lands in the slot the next accepted word overwrites.
int record_scalar(const uint32_t *w, int avail, uint32_t &i_io, uint32_t &mask_io, uint32_t *js, uint32_t top) {
  uint32_t i = i_io, mask = mask_io;
  int k = 0;
  while (k < avail && i >= 1) {
    const uint32_t lim = mask >> 1, m = mask;
    while (k < avail && i > lim) {
      const uint32_t j = w[k] & m;
      js[top - i] = j;
      i -= (j <= i) ? 1u : 0u;
      k++;
    }
    if (i <= lim) mask >>= 1;
  }
  i_io = i;
  mask_io = mask;
  return k;
}

// Backward pass over the steps i = i0 .. M-1 (js[M-1-i] = j_i) for output slots that sit below every remaining i: the
// swap at step i moves a slot's element only if the slot tracks position j_i, and then it came from position i.
void follow_scalar(const uint32_t *js, uint32_t M, uint32_t i, uint32_t *pos, int n) {
  for (; i < M; i++) {
    const uint32_t j = js[M - 1 - i];
    for (int k = 0; k < n; k++)
      if (pos[k] == j) { pos[k] = i; break; }
  }
}

#if CG_X86
// ---- AVX2 ---------------------------------------------------------------------------------------------------------
#define CG_AVX2 __attribute__((target("avx2,popcnt")))
CG_AVX2 inline __m256i mix8(__m256i a, __m256i b, __m256i far) {
  const __m256i y = _mm256_or_si256(_mm256_and_si256(a, _mm256_set1_epi32((int)MT_UP)), _mm256_and_si256(b, _mm256_set1_epi32((int)MT_LO)));
  const __m256i odd = _mm256_sub_epi32(_mm256_setzero_si256(), _mm256_and_si256(y, _mm256_set1_epi32(1)));
  return _mm256_xor_si256(_mm256_xor_si256(far, _mm256_srli_epi32(y, 1)), _mm256_and_si256(odd, _mm256_set1_epi32((int)MT_MAG)));
}
CG_AVX2 void refill_avx2(uint32_t *mt) {
  int kk = 0;
  for (; kk + 8 <= MT_N - MT_M; kk += 8)
    _mm256_storeu_si256((__m256i *)(mt + kk), mix8(_mm256_loadu_si256((const __m256i *)(mt + kk)), _mm256_loadu_si256((const __m256i *)(mt + kk + 1)),
                                                   _mm256_loadu_si256((const __m256i *)(mt + kk + MT_M))));
  for (; kk < MT_N - MT_M; kk++) mt[kk] = mt_mix(mt[kk], mt[kk + 1], mt[kk + MT_M]);
  for (; kk + 8 <= MT_N - 1; kk += 8)
    _mm256_storeu_si256((__m256i *)(mt + kk), mix8(_mm256_loadu_si256((const __m256i *)(mt + kk)), _mm256_loadu_si256((const __m256i *)(mt + kk + 1)),
                                                   _mm256_loadu_si256((const __m256i *)(mt + kk + (MT_M - MT_N)))));
  for (; kk < MT_N - 1; kk++) mt[kk] = mt_mix(mt[kk], mt[kk + 1], mt[kk + (MT_M - MT_N)]);
  mt[MT_N - 1] = mt_mix(mt[MT_N - 1], mt[0], mt[MT_M - 1]);
}
CG_AVX2 void temper_avx2(const uint32_t *in, uint32_t *out, int n) {
  int k = 0;
  for (; k + 8 <= n; k += 8) {
    __m256i y = _mm256_loadu_si256((const __m256i *)(in + k));
    y = _mm256_xor_si256(y, _mm256_srli_epi32(y, 11));
    y = _mm256_xor_si256(y, _mm256_and_si256(_mm256_slli_epi32(y, 7), _mm256_set1_epi32((int)0x9d2c5680u)));
    y = _mm256_xor_si256(y, _mm256_and_si256(_mm256_slli_epi32(y, 15), _mm256_set1_epi32((int)0xefc60000u)));
    y = _mm256_xor_si256(y, _mm256_srli_epi32(y, 18));
    _mm256_storeu_si256((__m256i *)(out + k), y);
  }
  for (; k < n; k++) out[k] = temper1(in[k]);
}
CG_AVX2 int scan_avx2(const uint32_t *w, int avail, uint32_t &i_io, uint32_t &mask_io) {
  uint32_t i = i_io, mask = mask_io;
  int k = 0;
  const __m256i lane = _mm256_setr_epi32(0, 1, 2, 3, 4, 5, 6, 7);
  while (k < avail && i >= 1) {
    const uint32_t lim = mask >> 1, m = mask;
    // 8 words at once: lane l sees i lowered by at most l accepts, so (w <= i - l) is a sure accept and (w > i) a sure
    // reject (values < 2^31: signed compares are exact); anything in between is replayed word by word
    const __m256i vm = _mm256_set1_epi32((int)m);
    while (k + 8 <= avail && i > lim + 8) {
      const __m256i v = _mm256_and_si256(_mm256_loadu_si256((const __m256i *)(w + k)), vm);
      const __m256i lo = _mm256_sub_epi32(_mm256_set1_epi32((int)i), lane);
      const int rej = _mm256_movemask_ps(_mm256_castsi256_ps(_mm256_cmpgt_epi32(v, _mm256_set1_epi32((int)i))));
      const int nacc = _mm256_movemask_ps(_mm256_castsi256_ps(_mm256_cmpgt_epi32(v, lo)));   // NOT a sure accept
      if (rej != nacc) break;
      i -= 8u - (uint32_t)__builtin_popcount((unsigned)nacc);
      k += 8;
    }
    for (int n = 0; n < 8 && k < avail && i > lim; n++, k++) i -= ((w[k] & m) <= i) ? 1u : 0u;
    if (i <= lim) mask >>= 1;
  }
  i_io = i;
  mask_io = mask;
  return k;
}

// ---- AVX-512 ------------------------------------------------------------------------------------------------------
#define CG_AVX512 __attribute__((target("avx512f,popcnt")))
CG_AVX512 inline __m512i mix16(__m512i a, __m512i b, __m512i far) {
  const __m512i y = _mm512_or_si512(_mm512_and_si512(a, _mm512_set1_epi32((int)MT_UP)), _mm512_and_si512(b, _mm512_set1_epi32((int)MT_LO)));
  const __m512i odd = _mm512_sub_epi32(_mm512_setzero_si512(), _mm512_and_si512(y, _mm512_set1_epi32(1)));
  return _mm512_xor_si512(_mm512_xor_si512(far, _mm512_srli_epi32(y, 1)), _mm512_and_si512(odd, _mm512_set1_epi32((int)MT_MAG)));
}
CG_AVX512 void refill_avx512(uint32_t *mt) {
  int kk = 0;
  for (; kk + 16 <= MT_N - MT_M; kk += 16)
    _mm512_storeu_si512(mt + kk, mix16(_mm512_loadu_si512(mt + kk), _mm512_loadu_si512(mt + kk + 1), _mm512_loadu_si512(mt + kk + MT_M)));
  for (; kk < MT_N - MT_M; kk++) mt[kk] = mt_mix(mt[kk], mt[kk + 1], mt[kk + MT_M]);
  for (; kk + 16 <= MT_N - 1; kk += 16)
    _mm512_storeu_si512(mt + kk, mix16(_mm512_loadu_si512(mt + kk), _mm512_loadu_si512(mt + kk + 1), _mm512_loadu_si512(mt + kk + (MT_M - MT_N))));
  for (; kk < MT_N - 1; kk++) mt[kk] = mt_mix(mt[kk], mt[kk + 1], mt[kk + (MT_M - MT_N)]);
  mt[MT_N - 1] = mt_mix(mt[MT_N - 1], mt[0], mt[MT_M - 1]);
}
CG_AVX512 void temper_avx512(const uint32_t *in, uint32_t *out, int n) {
  int k = 0;
  for (; k + 16 <= n; k += 16) {
    __m512i y = _mm512_loadu_si512(in + k);
    y = _mm512_xor_si512(y, _mm512_srli_epi32(y, 11));
    y = _mm512_xor_si512(y, _mm512_and_si512(_mm512_slli_epi32(y, 7), _mm512_set1_epi32((int)0x9d2c5680u)));
    y = _mm512_xor_si512(y, _mm512_and_si512(_mm512_slli_epi32(y, 15), _mm512_set1_epi32((int)0xefc60000u)));
    y = _mm512_xor_si512(y, _mm512_srli_epi32(y, 18));
    _mm512_storeu_si512(out + k, y);
  }
  for (; k < n; k++) out[k] = temper1(in[k]);
}
CG_AVX512 int scan_avx512(const uint32_t *w, int avail, uint32_t &i_io, uint32_t &mask_io) {
  uint32_t i = i_io, mask = mask_io;
  int k = 0;
  const __m512i lane = _mm512_setr_epi32(0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15);
  while (k < avail && i >= 1) {
    const uint32_t lim = mask >> 1, m = mask;
    const __m512i vm = _mm512_set1_epi32((int)m);
    while (k + 16 <= avail && i > lim + 16) {
      const __m512i v = _mm512_and_si512(_mm512_loadu_si512(w + k), vm);
      const __mmask16 rej = _mm512_cmpgt_epu32_mask(v, _mm512_set1_epi32((int)i));
      const __mmask16 nacc = _mm512_cmpgt_epu32_mask(v, _mm512_sub_epi32(_mm512_set1_epi32((int)i), lane));
      if (rej != nacc) break;
      i -= 16u - (uint32_t)__builtin_popcount((unsigned)nacc);
      k += 16;
    }
    for (int n = 0; n < 16 && k < avail && i > lim; n++, k++) i -= ((w[k] & m) <= i) ? 1u : 0u;
    if (i <= lim) mask >>= 1;
  }
  i_io = i;
  mask_io = mask;
  return k;
}

CG_AVX512 int upper_avx512(const uint32_t *w, int avail, uint32_t &i_io, uint32_t &mask_io, uint32_t low, int32_t *p, uint32_t dummy) {
  uint32_t i = i_io, mask = mask_io;
  int k = 0;
  const __m512i lane = _mm512_setr_epi32(0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15);
  alignas(64) uint32_t js[16];
  while (k < avail && i >= low) {
    const uint32_t lim = mask >> 1, m = mask;
    const __m512i vm = _mm512_set1_epi32((int)m);
    // 16 words decided at once (same test as the scan), accepted targets compressed, then the ordered scatter
    while (k + 16 <= avail && i > lim + 16 && i >= low + 16) {
      const __m512i v = _mm512_and_si512(_mm512_loadu_si512(w + k), vm);
      const __mmask16 rej = _mm512_cmpgt_epu32_mask(v, _mm512_set1_epi32((int)i));
      const __mmask16 nacc = _mm512_cmpgt_epu32_mask(v, _mm512_sub_epi32(_mm512_set1_epi32((int)i), lane));
      if (rej != nacc) break;
      const uint32_t cnt = 16u - (uint32_t)__builtin_popcount((unsigned)nacc);
      _mm512_store_si512(js, _mm512_maskz_compress_epi32((__mmask16)~nacc, v));
      for (uint32_t n = 0; n < cnt; n++) p[js[n]] = p[i - n];
      i -= cnt;
      k += 16;
    }
    for (int n = 0; n < 16 && k < avail && i > lim && i >= low; n++, k++) {
      const uint32_t j = w[k] & m;
      const uint32_t acc = (j <= i) ? 1u : 0u;
      p[acc ? j : dummy] = p[i];
      i -= acc;
    }
    if (i <= lim) mask >>= 1;
  }
  i_io = i;
  mask_io = mask;
  return k;
}

CG_AVX512 int record_avx512(const uint32_t *w, int avail, uint32_t &i_io, uint32_t &mask_io, uint32_t *js, uint32_t top) {
  uint32_t i = i_io, mask = mask_io;
  int k = 0;
  const __m512i lane = _mm512_setr_epi32(0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15);
  while (k < avail && i >= 1) {
    const uint32_t lim = mask >> 1, m = mask;
    const __m512i vm = _mm512_set1_epi32((int)m);
    while (k + 16 <= avail && i > lim + 16) {
      const __m512i v = _mm512_and_si512(_mm512_loadu_si512(w + k), vm);
      const __mmask16 rej = _mm512_cmpgt_epu32_mask(v, _mm512_set1_epi32((int)i));
      const __mmask16 nacc = _mm512_cmpgt_epu32_mask(v, _mm512_sub_epi32(_mm512_set1_epi32((int)i), lane));
      if (rej != nacc) break;
      // accepted j's in step order; the full 16-wide store writes past them into slots later steps overwrite
      _mm512_storeu_si512(js + (top - i), _mm512_maskz_compress_epi32((__mmask16)~nacc, v));
      i -= 16u - (uint32_t)__builtin_popcount((unsigned)nacc);
      k += 16;
    }
    for (int n = 0; n < 16 && k < avail && i > lim; n++, k++) {
      const uint32_t j = w[k] & m;
      js[top - i] = j;
      i -= (j <= i) ? 1u : 0u;
    }
    if (i <= lim) mask >>= 1;
  }
  i_io = i;
  mask_io = mask;
  return k;
}

CG_AVX512 void follow_avx512(const uint32_t *js, uint32_t M, uint32_t i, uint32_t *pos, int n) {
  __m512i P[16];   // the tracked positions, broadcast
  for (int k = 0; k < n; k++) P[k] = _mm512_set1_epi32((int)pos[k]);
  // 32 steps at a time: steps i .. i+15 are lanes 15 .. 0 of js[M-16-i ..], steps i+16 .. i+31 lanes 15 .. 0 of
  // js[M-32-i ..]; the earliest hit is the highest set lane, and the scan resumes right after it
  while (i + 32 <= M) {
    const __m512i lo = _mm512_loadu_si512(js + (M - 16 - i)), hi = _mm512_loadu_si512(js + (M - 32 - i));
    __mmask16 hlo = 0, hhi = 0;
    for (int k = 0; k < n; k++) {
      hlo |= _mm512_cmpeq_epu32_mask(lo, P[k]);
      hhi |= _mm512_cmpeq_epu32_mask(hi, P[k]);
    }
    if (!(hlo | hhi)) {
      i += 32;
      continue;
    }
    const uint32_t step = hlo ? i + (uint32_t)__builtin_clz((unsigned)hlo) - 16u : i + (uint32_t)__builtin_clz((unsigned)hhi);
    const uint32_t j = js[M - 1 - step];
    for (int k = 0; k < n; k++)
      if (pos[k] == j) { pos[k] = step; P[k] = _mm512_set1_epi32((int)step); break; }
    i = step + 1;
  }
  follow_scalar(js, M, i, pos, n);
}

#endif   // CG_X86

struct Isa {
  void (*refill)(uint32_t *);
  void (*temper)(const uint32_t *, uint32_t *, int);
  int (*scan)(const uint32_t *, int, uint32_t &, uint32_t &);
  int (*upper)(const uint32_t *, int, uint32_t &, uint32_t &, uint32_t, int32_t *, uint32_t);
  int (*record)(const uint32_t *, int, uint32_t &, uint32_t &, uint32_t *, uint32_t);
  void (*follow)(const uint32_t *, uint32_t, uint32_t, uint32_t *, int);
  int level;
};
Isa pick_isa(int force) {
#if CG_X86
  __builtin_cpu_init();
  int level = __builtin_cpu_supports("avx512f") ? 2 : (__builtin_cpu_supports("avx2") ? 1 : 0);
  if (force >= 0 && force < level) level = force;
  if (level == 2) return {refill_avx512, temper_avx512, scan_avx512, upper_avx512, record_avx512, follow_avx512, 2};
  if (level == 1) return {refill_avx2, temper_avx2, scan_avx2, upper_scalar, record_scalar, follow_scalar, 1};
#else
  (void)force;
#endif
  return {refill_scalar, temper_scalar, scan_scalar, upper_scalar, record_scalar, follow_scalar, 0};
}
Isa g_isa = pick_isa(-1);

struct Mt {
  uint32_t *key;
  int pos;
  inline uint32_t next() {
    if (pos == MT_N) {
      g_isa.refill(key);
      pos = 0;
    }
    return temper1(key[pos++]);
  }
};

// One candidate's shuffle from generator state g (advanced in place); writes the first n_pts entries to out.
// p has M + 1 entries (p[M] swallows the store of a rejected word, so a rejection costs no branch and no
// store-to-load forwarding stall on p[i]).
void shuffle_one(Mt &g, int64_t M, int32_t n_pts, int32_t *p, int32_t *out) {
  for (int32_t i = 0; i < (int32_t)M; i++) p[i] = i;
  uint32_t mask = mask_of((uint32_t)(M - 1));
  uint32_t i = (uint32_t)(M - 1);
  const uint32_t low = (uint32_t)n_pts, dummy = (uint32_t)M;
  uint32_t tmp[MT_N];
  while (i >= 1) {
    if (g.pos == MT_N) {
      g_isa.refill(g.key);
      g.pos = 0;
    }
    const int avail = MT_N - g.pos;
    g_isa.temper(g.key + g.pos, tmp, avail);
    int k = (i >= low) ? g_isa.upper(tmp, avail, i, mask, low, p, dummy) : 0;
    for (; k < avail && i >= 1; k++) {
      const uint32_t j = tmp[k] & mask;
      const uint32_t acc = (j <= i) ? 1u : 0u;
      const uint32_t jj = acc ? j : dummy;
      const int32_t t = p[jj];
      p[jj] = p[i];
      p[acc ? i : dummy] = t;
      i -= acc;
      if ((mask >> 1) >= i) mask >>= 1;
    }
    g.pos += k;
  }
  memcpy(out, p, (size_t)n_pts * sizeof(int32_t));
}

// Advances g exactly as shuffle_one would, without touching a permutation: the sequential part of the threaded draw.
void shuffle_skip(Mt &g, int64_t M) {
  uint32_t mask = mask_of((uint32_t)(M - 1));
  uint32_t i = (uint32_t)(M - 1);
  uint32_t tmp[MT_N];
  while (i >= 1) {
    if (g.pos == MT_N) {
      g_isa.refill(g.key);
      g.pos = 0;
    }
    const int avail = MT_N - g.pos;
    g_isa.temper(g.key + g.pos, tmp, avail);
    g.pos += g_isa.scan(tmp, avail, i, mask);
  }
}

// Small subsets (n_pts <= SLOT_MAX): follow the n_pts output slots instead of replaying the shuffle.  The walk keeps
// every step's j (js needs M - 1 + 16 entries); the element that ends in slot k is found by undoing the swaps from the
// last step (i = 1) up: a slot's position changes at step i only if it is i or j_i.  Above the slots (i >= n_pts) a
// tracked position is always below i, so only j_i == position matters, and that is rare: the backward pass is n_pts
// compares per step, a fraction of the walk's cost.
constexpr int SLOT_MAX = 16;

void shuffle_slots(Mt &g, int64_t M, int32_t n_pts, uint32_t *js, int32_t *out) {
  const uint32_t top = (uint32_t)(M - 1);
  uint32_t mask = mask_of(top);
  uint32_t i = top;
  uint32_t tmp[MT_N];
  while (i >= 1) {
    if (g.pos == MT_N) {
      g_isa.refill(g.key);
      g.pos = 0;
    }
    const int avail = MT_N - g.pos;
    g_isa.temper(g.key + g.pos, tmp, avail);
    g.pos += g_isa.record(tmp, avail, i, mask, js, top);
  }
  uint32_t pos[SLOT_MAX];
  for (int k = 0; k < n_pts; k++) pos[k] = (uint32_t)k;
  uint32_t s = 1;
  for (; s < (uint32_t)n_pts && s < (uint32_t)M; s++) {   // the steps among the slots: the full swap
    const uint32_t j = js[top - s];
    for (int k = 0; k < n_pts; k++) {
      if (pos[k] == s) pos[k] = j;
      else if (pos[k] == j) pos[k] = s;
    }
  }
  g_isa.follow(js, (uint32_t)M, s, pos, n_pts);
  for (int k = 0; k < n_pts; k++) out[k] = (int32_t)pos[k];
}

inline void backoff(int &spins) {
  if (++spins < 4096) {
#if CG_X86
    _mm_pause();
#else
    std::this_thread::yield();
#endif
  } else {   // the walker is far behind (or descheduled): stop burning the core
    struct timespec ts = {0, 20000};
    nanosleep(&ts, nullptr);
  }
}

}  // namespace

// Developer/test hook: cap the instruction set (0 scalar, 1 AVX2, 2 AVX-512; -1 = best available).  Returns the level in use.
extern "C" int cg_host_rng_isa(int force) {
  g_isa = pick_isa(force);
  return g_isa.level;
}

// key: 624 words, *pos in [0, 624] (numpy's state tuple fields 1 and 2), both updated in place.
// out: (count, n_pts) int32.  M < 2^31.  nthreads <= 0: one thread per host core (at most 12).
// The generator is inherently sequential, but which words a candidate consumes does not depend on its permutation:
// the calling thread walks the stream (snapshotting the state at every candidate boundary) while worker threads
// replay the real shuffles from those snapshots.
extern "C" int cg_host_legacy_choice(uint32_t *key, int32_t *pos, int64_t M, int32_t n_pts, int32_t count, int32_t *out,
                                     int32_t nthreads) {
  if (!key || !pos || !out || M <= 0 || M >= (1ll << 31) || n_pts <= 0 || count < 0 || *pos < 0 || *pos > MT_N)
    return CG_EINVAL;
  Mt g{key, *pos};
  if (M < n_pts) {
    // replace=True: randint(0, M, size=n_pts): value = next_uint32 & mask until value <= M-1 (masked rejection)
    const uint32_t rng = (uint32_t)(M - 1);
    const uint32_t mask = mask_of(rng);
    for (int64_t c = 0; c < count; c++) {
      int32_t *o = out + c * (int64_t)n_pts;
      for (int i = 0; i < n_pts; i++) {
        uint32_t v;
        if (rng == 0) v = 0;   // random_bounded_uint64_fill: rng == 0 consumes nothing
        else
          while ((v = (g.next() & mask)) > rng) {
          }
        o[i] = (int32_t)v;
      }
    }
    *pos = g.pos;
    return CG_OK;
  }
  // replace=False: permutation(M)[:n_pts]: shuffle arange(M) from the top, j = random_interval(i)
  if (n_pts <= SLOT_MAX) {   // one thread: the walk is the whole cost, workers would only wait for it
    std::vector<uint32_t> js((size_t)M + 16);
    for (int64_t c = 0; c < count; c++) shuffle_slots(g, M, n_pts, js.data(), out + c * (int64_t)n_pts);
    *pos = g.pos;
    return CG_OK;
  }
  if (nthreads <= 0) {
    // the walk is ~6x faster than one replay: a dozen workers keep up with it, more only add wake-up traffic
    nthreads = (int32_t)std::thread::hardware_concurrency();
    if (nthreads > 12) nthreads = 12;
  }
  if (nthreads > count) nthreads = count;
  if (nthreads < 2 || count < 4 || M < 2048) {
    std::vector<int32_t> perm((size_t)M + 1);
    for (int64_t c = 0; c < count; c++) shuffle_one(g, M, n_pts, perm.data(), out + c * (int64_t)n_pts);
    *pos = g.pos;
    return CG_OK;
  }
  struct Snap { uint32_t key[MT_N]; int pos; };
  std::vector<Snap> snaps((size_t)count);
  struct alignas(64) Counter { std::atomic<int> v{0}; };
  Counter ready, next;   // separate cache lines: the walker publishes `ready`, the workers contend on `next`
  auto worker = [&]() {
    std::vector<int32_t> perm((size_t)M + 1);
    for (;;) {
      const int c = next.v.fetch_add(1, std::memory_order_relaxed);
      if (c >= count) return;
      int spins = 0;
      while (ready.v.load(std::memory_order_acquire) <= c) backoff(spins);
      Mt lg{snaps[(size_t)c].key, snaps[(size_t)c].pos};
      shuffle_one(lg, M, n_pts, perm.data(), out + (int64_t)c * n_pts);
    }
  };
  std::vector<std::thread> pool;
  for (int t = 0; t < nthreads - 1; t++) pool.emplace_back(worker);
  for (int c = 0; c < count; c++) {
    memcpy(snaps[(size_t)c].key, key, sizeof(uint32_t) * MT_N);
    snaps[(size_t)c].pos = g.pos;
    ready.v.store(c + 1, std::memory_order_release);
    shuffle_skip(g, M);
  }
  worker();   // the walking thread helps with what is left
  for (auto &t : pool) t.join();
  *pos = g.pos;
  return CG_OK;
}

// Advance the generator over `count` candidates without producing indices (a rank that scores candidates [lo, hi) of a
// list still has to leave numpy's generator where the reference's full loop leaves it).
extern "C" int cg_host_legacy_skip(uint32_t *key, int32_t *pos, int64_t M, int32_t n_pts, int32_t count) {
  if (!key || !pos || M <= 0 || M >= (1ll << 31) || n_pts <= 0 || count < 0 || *pos < 0 || *pos > MT_N) return CG_EINVAL;
  Mt g{key, *pos};
  if (M < n_pts) {
    const uint32_t rng = (uint32_t)(M - 1);
    const uint32_t mask = mask_of(rng);
    if (rng != 0)
      for (int64_t i = 0; i < (int64_t)count * n_pts; i++)
        while ((g.next() & mask) > rng) {
        }
  } else {
    for (int c = 0; c < count; c++) shuffle_skip(g, M);
  }
  *pos = g.pos;
  return CG_OK;
}
