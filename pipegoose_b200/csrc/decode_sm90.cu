// Split-KV ("flash-decoding") ALiBi attention for one decoding step of a KV-cached generation, sm_90a.
//
//   qkv     : [B, H*3*D] bf16, the step's QKV projection, each row laid out [head][q|k|v][D]
//   k_cache : [B, H, capacity, D] bf16, v_cache likewise           out : [B, H*D] bf16
//   lead    : int32 [B] leading pad positions of each row (nullptr: none)
//
// Every row decodes one token at column `pos`.  The kernel writes the new k / v into cache[:, :, pos]; row b's query
// then attends to keys lead[b] <= k <= pos with score = q.k * scale + slope[h] * (k - pos) (the same softmax as
// slope * k), softmax and sums in fp32.
//
// Grid (split, head, row).  A row's key range is cut into `splits` contiguous chunks, one per CTA.  A CTA's four warps
// stream their chunk with 16-byte loads: a key's D bf16 are spread over LPK lanes (8 dims each), so a warp reads
// 32 / LPK keys per load and keeps U keys of K and V in flight per lane.  Every key group keeps an online softmax
// (m, l, o) in registers; the groups are merged through shared memory.  With one split that merge is the output.
// Otherwise each CTA writes its partial (m, l, o[D]) to the fp32 workspace, and the CTA that takes the last ticket of
// its (row, head) merges the partials in split order and resets the ticket: no CTA waits for another, and the result
// has no atomics in its arithmetic, so it is bitwise reproducible.
//
// The key at `pos` is read from the qkv row, not from the cache, by the one lane group that handles it; that group
// also stores it into the cache.  No other thread touches cache[:, :, pos], so the write never races a read and the
// cache can be read through the non-coherent path.
//
// Paged form (PAGED = true, continuous batching): the caches are page pools k_pool / v_pool [num_pages, H, 64, D] and
// every row has its own position pos[b] (int32 [B] on the device).  Row b's position p lives in page
// table[b, p / 64] (int32 [B, max_pages]) at slot p % 64.  Row b writes its new k / v into the slot of pos[b] and
// attends to keys 0 <= k <= pos[b]; there is no lead.  The grid is sized for the longest row (`pos` holds the host's
// bound on max(pos[b])); each row cuts its own range into `splits` chunks, so the bound only shapes the grid.  The page
// holding pos[b] belongs to row b alone; other pages may be shared between rows and are only read.  So the write of
// pos[b]'s slot races no read either.
//
// paged_kv_write_kernel stores the k / v of a packed prefill into the pools: token n's heads go to slot[n]
// (page * 64 + offset), 16 bytes per thread.
//
// paged_kv_copy_kernel copies the leading slots of pages (beam search forks a shared partly filled page): for every
// pair i = (src, dst, count) and every layer of the [n_layer, pages, H, 64, D] pools, slots 0 .. count - 1 of K and V
// of page src go to page dst, 16 bytes per thread, with their fp32 scales over FP8 pools.
//
// FP8 pools (e4m3 codes [num_pages, H, 64, D] and fp32 scales [num_pages, H, 64], one per position, head and K | V):
// a row x of D values is stored as scale = amax / 448 and code_i = e4m3_rn_satfinite(x_i * (448 / amax)), all codes 0
// and scale 0 when amax == 0; it reads back as float(code) * scale.  ops/attention.py holds the same quantizer for the
// CPU, bit for bit (IEEE division: the build has no fast-math).  Positions a step computes itself are read from its
// bf16 qkv, exactly; only positions of earlier steps are read from the FP8 pools.
//   paged_kv_write_fp8_kernel   the quantizing form of paged_kv_write_kernel: one half-warp per (token, head, K|V) row.
//   decode_attention_fp8_kernel the paged split-KV kernel over FP8 pools: a lane loads 16 codes (16 B), the score is
//                               (q.code_k) * s_k and a key's value weight p * s_v.  The key at pos[b] joins every
//                               key group's loop after it, from qkv; warp 0 of split 0 quantizes it into its slot.
//                               The loop never reads that slot, so the store races nothing.
//   kv_dequantize_kernel        whole pages src[i] of the FP8 pools into pages dst[i] of bf16 pools (the staging
//                               pool of a prefill with cached prefixes).
#include "launch.h"
#include "pdl_launch.cuh"
#include "ptx.cuh"
#include <cuda_fp8.h>
#include <cmath>
#include <cstdio>

namespace pg {

constexpr int kDecWarps = 4;
constexpr int kDecThreads = kDecWarps * 32;
constexpr int kDecUnroll = 4;        // keys of K and V in flight per lane group
constexpr int kDecMinChunk = 64;     // fewest keys a split is given
constexpr int kDecTargetCtas = 132 * 4;
constexpr float kDecLog2e = 1.4426950408889634f;
constexpr int kPageShift = 6;        // 64 positions per page of the paged pools
constexpr int kPageSize = 1 << kPageShift;
constexpr int kAppendMaxTokens = 8;  // most tokens a row appends in one append-attention call

struct DecodeArgs {
  const __nv_bfloat16* qkv;
  __nv_bfloat16* k_cache;
  __nv_bfloat16* v_cache;
  const float* slopes;
  union {
    const int* lead;         // contiguous form: [B] leading pads
    const int* cu_seqlens;   // append form: [B + 1], row b's tokens are qkv rows cu_seqlens[b] .. cu_seqlens[b+1] - 1
  };
  __nv_bfloat16* out;
  float* part;   // [B*H, splits, D + 2]: (m, l, o[D]) per split (splits > 1)
  int* ticket;   // [B*H], zero between calls
  int H, capacity, pos, splits;
  float scale_log2;
  // paged form only (k_cache / v_cache are then the pools, capacity and lead unused)
  const int* table;     // [B, max_pages] page ids
  const int* row_pos;   // [B] each row's new-token position
  int max_pages;
  // FP8 pools only (k_cache / v_cache then hold e4m3 codes)
  float* k_scales;      // [num_pages, H, 64]
  float* v_scales;
};

PG_DEVICE void bf16x8_to_f32(const uint4& r, float* f) {
  const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(p[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

// The end of the decode kernels, once per query: merge the CTA's key groups (lane sub of group grp holds o for dims
// sub * E ..), then, with one split, store the output row `out`, otherwise this split's partial and, in the CTA that
// takes the last ticket, the merge of all splits.  `bh` indexes the query's ticket and partials.
template <int D, int NG, int E>
PG_DEVICE void decode_merge(const DecodeArgs& a, size_t bh, int split, int grp, int sub, bool active, float m, float l,
                            const float (&o)[E], float* s_m, float* s_l, float (*s_o)[D], int& s_last,
                            __nv_bfloat16* out) {
  if (sub == 0) {
    s_m[grp] = m;
    s_l[grp] = l;
  }
  if (active) {
#pragma unroll
    for (int i = 0; i < E; ++i) s_o[grp][sub * E + i] = o[i];
  }
  __syncthreads();
  const int d = threadIdx.x;
  float M = -INFINITY, L = 0.f, O = 0.f;
  if (d < D) {
#pragma unroll
    for (int g = 0; g < NG; ++g) M = fmaxf(M, s_m[g]);
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      const float w = s_m[g] == -INFINITY ? 0.f : exp2f(s_m[g] - M);
      L = fmaf(w, s_l[g], L);
      O = fmaf(w, s_o[g][d], O);
    }
  }
  if (a.splits == 1) {   // this CTA saw every key, including pos: L > 0
    if (d < D) out[d] = __float2bfloat16(O / L);
    return;
  }

  float* part = a.part + bh * a.splits * (D + 2);
  float* mine = part + static_cast<size_t>(split) * (D + 2);
  if (d == 0) {
    mine[0] = M;   // -inf for an empty split (a row whose key range is shorter than the split count)
    mine[1] = L;
  }
  if (d < D) mine[2 + d] = O;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(a.ticket + bh, 1) == a.splits - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (d < D) {
    float Mg = -INFINITY;
    for (int sp = 0; sp < a.splits; ++sp) Mg = fmaxf(Mg, __ldcg(part + static_cast<size_t>(sp) * (D + 2)));
    float Lg = 0.f, Og = 0.f;
    for (int sp = 0; sp < a.splits; ++sp) {
      const float* p = part + static_cast<size_t>(sp) * (D + 2);
      const float ms = __ldcg(p);
      const float w = ms == -INFINITY ? 0.f : exp2f(ms - Mg);
      Lg = fmaf(w, __ldcg(p + 1), Lg);
      Og = fmaf(w, __ldcg(p + 2 + d), Og);
    }
    out[d] = __float2bfloat16(Og / Lg);
  }
  if (threadIdx.x == 0) a.ticket[bh] = 0;
}

template <int D, bool PAGED>
__global__ void __launch_bounds__(kDecThreads) decode_attention_kernel(const DecodeArgs a) {
  constexpr int VEC = D / 8;                  // lanes holding a key's dims (8 bf16 = 16 B each)
  constexpr int LPK = VEC <= 8 ? 8 : 16;      // lanes per key: VEC rounded up to a power of two (shuffle reduction)
  constexpr int KPW = 32 / LPK;               // keys per warp per load
  constexpr int NG = kDecWarps * KPW;         // key groups per CTA
  static_assert(D % 8 == 0 && VEC <= 16, "head size");
  __shared__ float s_m[NG], s_l[NG];
  __shared__ float s_o[NG][D];
  __shared__ int s_last;

  pdl_launch_dependents();
  pdl_wait();
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int H = a.H;
  const int pos = PAGED ? __ldg(a.row_pos + b) : a.pos;
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPK;
  const int grp = (threadIdx.x >> 5) * KPW + lane / LPK;
  const bool active = sub < VEC;

  const int lo = !PAGED && a.lead != nullptr ? min(max(a.lead[b], 0), pos) : 0;
  const int chunk = (pos - lo + a.splits) / a.splits;   // ceil((pos - lo + 1) / splits)
  const int k0 = lo + split * chunk;
  const int k1 = min(k0 + chunk, pos + 1);

  const size_t bh = static_cast<size_t>(b) * H + h;
  const __nv_bfloat16* row = a.qkv + (static_cast<size_t>(b) * H + h) * 3 * D;
  const uint4* kc = reinterpret_cast<const uint4*>(PAGED ? a.k_cache : a.k_cache + bh * a.capacity * D);
  const uint4* vc = reinterpret_cast<const uint4*>(PAGED ? a.v_cache : a.v_cache + bh * a.capacity * D);
  const int* tab = PAGED ? a.table + static_cast<size_t>(b) * a.max_pages : nullptr;
  // uint4 offset of key k from kc / vc
  auto key_at = [&](int k) -> size_t {
    if constexpr (PAGED)
      return ((static_cast<size_t>(__ldg(tab + (k >> kPageShift))) * H + h) * kPageSize + (k & (kPageSize - 1))) * VEC;
    else
      return static_cast<size_t>(k) * VEC;
  };
  const uint4* k_new = reinterpret_cast<const uint4*>(row + D);
  const uint4* v_new = reinterpret_cast<const uint4*>(row + 2 * D);

  float q[8];
  {
    uint4 r = make_uint4(0, 0, 0, 0);
    if (active) r = reinterpret_cast<const uint4*>(row)[sub];
    bf16x8_to_f32(r, q);
#pragma unroll
    for (int i = 0; i < 8; ++i) q[i] *= a.scale_log2;
  }
  const float slope_log2 = a.slopes[h] * kDecLog2e;

  // online softmax of this lane group's keys, base-2 exponents
  float m = -INFINITY, l = 0.f, o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = 0.f;
  // the trip count is the same for every thread of the CTA: the shuffles below are never divergent
  for (int kb = k0; kb < k1; kb += NG * kDecUnroll) {
    uint4 kr[kDecUnroll], vr[kDecUnroll];
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) {
      const int k = kb + u * NG + grp;
      kr[u] = vr[u] = make_uint4(0, 0, 0, 0);
      if (active && k < k1) {
        if (k == pos) {
          kr[u] = k_new[sub];
          vr[u] = v_new[sub];
          if constexpr (PAGED) {
            reinterpret_cast<uint4*>(a.k_cache)[key_at(pos) + sub] = kr[u];
            reinterpret_cast<uint4*>(a.v_cache)[key_at(pos) + sub] = vr[u];
          } else {
            reinterpret_cast<uint4*>(a.k_cache + (bh * a.capacity + pos) * D)[sub] = kr[u];
            reinterpret_cast<uint4*>(a.v_cache + (bh * a.capacity + pos) * D)[sub] = vr[u];
          }
        } else {
          const size_t at = key_at(k);
          kr[u] = __ldg(kc + at + sub);
          vr[u] = __ldg(vc + at + sub);
        }
      }
    }
    float s[kDecUnroll];
    float mx = m;
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) {
      float kf[8];
      bf16x8_to_f32(kr[u], kf);
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) dot = fmaf(q[i], kf[i], dot);
#pragma unroll
      for (int off = LPK / 2; off > 0; off >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, off);
      const int k = kb + u * NG + grp;
      s[u] = k < k1 ? fmaf(slope_log2, static_cast<float>(k - pos), dot) : -INFINITY;
      mx = fmaxf(mx, s[u]);
    }
    const float ref = mx == -INFINITY ? 0.f : mx;   // a group with no key yet: keep l = o = 0
    const float corr = exp2f(m - ref);
    l *= corr;
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] *= corr;
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) {
      const float p = exp2f(s[u] - ref);
      float vf[8];
      bf16x8_to_f32(vr[u], vf);
      l += p;
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = fmaf(p, vf[i], o[i]);
    }
    m = mx;
  }

  decode_merge<D, NG>(a, bh, split, grp, sub, active, m, l, o, s_m, s_l, s_o, s_last, a.out + bh * D);
}

// Paged append attention (speculative verification): row b appends n = cu_seqlens[b+1] - cu_seqlens[b] tokens
// (1 <= n <= NQ) at positions pos[b] .. pos[b] + n - 1; query i attends to keys 0 .. pos[b] + i.  The layout of
// decode_attention_kernel<D, true>, with NQ queries per CTA: every key of the chunk is loaded once and scored against
// all of the row's queries, each with its own online softmax.  Keys pos[b] .. are read from qkv by the one lane group
// that handles each, which also stores it into its pool slot; no thread reads a slot this launch writes.  Each query
// then goes through decode_merge with its own ticket and partials (index (b * H + h) * kAppendMaxTokens + i).
template <int D, int NQ>
__global__ void __launch_bounds__(kDecThreads) append_attention_kernel(const DecodeArgs a) {
  constexpr int VEC = D / 8;
  constexpr int LPK = VEC <= 8 ? 8 : 16;
  constexpr int KPW = 32 / LPK;
  constexpr int NG = kDecWarps * KPW;
  constexpr int U = NQ <= 2 ? kDecUnroll : 2;   // keys in flight per lane group: fewer with more queries (registers)
  static_assert(D % 8 == 0 && VEC <= 16 && NQ <= kAppendMaxTokens, "head size / queries");
  __shared__ float s_m[NG], s_l[NG];
  __shared__ float s_o[NG][D];
  __shared__ int s_last;

  pdl_launch_dependents();
  pdl_wait();
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int H = a.H;
  const int pos = __ldg(a.row_pos + b);
  const int t0 = __ldg(a.cu_seqlens + b);
  const int n = __ldg(a.cu_seqlens + b + 1) - t0;
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPK;
  const int grp = (threadIdx.x >> 5) * KPW + lane / LPK;
  const bool active = sub < VEC;

  const int chunk = (pos + n - 1 + a.splits) / a.splits;   // ceil((pos + n) / splits)
  const int k0 = split * chunk;
  const int k1 = min(k0 + chunk, pos + n);

  const size_t tstride = static_cast<size_t>(H) * 3 * D;     // one token of qkv
  const __nv_bfloat16* tok = a.qkv + static_cast<size_t>(t0) * tstride + static_cast<size_t>(h) * 3 * D;
  const uint4* kc = reinterpret_cast<const uint4*>(a.k_cache);
  const uint4* vc = reinterpret_cast<const uint4*>(a.v_cache);
  const int* tab = a.table + static_cast<size_t>(b) * a.max_pages;
  auto key_at = [&](int k) -> size_t {
    return ((static_cast<size_t>(__ldg(tab + (k >> kPageShift))) * H + h) * kPageSize + (k & (kPageSize - 1))) * VEC;
  };

  float q[NQ][8];
#pragma unroll
  for (int j = 0; j < NQ; ++j) {
    uint4 r = make_uint4(0, 0, 0, 0);
    if (active && j < n) r = reinterpret_cast<const uint4*>(tok + j * tstride)[sub];
    bf16x8_to_f32(r, q[j]);
#pragma unroll
    for (int i = 0; i < 8; ++i) q[j][i] *= a.scale_log2;
  }
  const float slope_log2 = a.slopes[h] * kDecLog2e;

  float m[NQ], l[NQ], o[NQ][8];
#pragma unroll
  for (int j = 0; j < NQ; ++j) {
    m[j] = -INFINITY;
    l[j] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) o[j][i] = 0.f;
  }
  // the trip count is the same for every thread of the CTA: the shuffles below are never divergent
  for (int kb = k0; kb < k1; kb += NG * U) {
    uint4 kr[U], vr[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int k = kb + u * NG + grp;
      kr[u] = vr[u] = make_uint4(0, 0, 0, 0);
      if (active && k < k1) {
        if (k >= pos) {   // a new token: from qkv, and into its slot
          const __nv_bfloat16* t = tok + (k - pos) * tstride;
          kr[u] = reinterpret_cast<const uint4*>(t + D)[sub];
          vr[u] = reinterpret_cast<const uint4*>(t + 2 * D)[sub];
          reinterpret_cast<uint4*>(a.k_cache)[key_at(k) + sub] = kr[u];
          reinterpret_cast<uint4*>(a.v_cache)[key_at(k) + sub] = vr[u];
        } else {
          const size_t at = key_at(k);
          kr[u] = __ldg(kc + at + sub);
          vr[u] = __ldg(vc + at + sub);
        }
      }
    }
    float s[U][NQ];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float kf[8];
      bf16x8_to_f32(kr[u], kf);
      const int k = kb + u * NG + grp;
#pragma unroll
      for (int j = 0; j < NQ; ++j) {
        s[u][j] = -INFINITY;
        if (j < n) {   // uniform over the CTA
          float dot = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) dot = fmaf(q[j][i], kf[i], dot);
#pragma unroll
          for (int off = LPK / 2; off > 0; off >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, off);
          if (k < k1 && k <= pos + j) s[u][j] = fmaf(slope_log2, static_cast<float>(k - pos - j), dot);
        }
      }
    }
    float ref[NQ];
#pragma unroll
    for (int j = 0; j < NQ; ++j) {
      float mx = m[j];
#pragma unroll
      for (int u = 0; u < U; ++u) mx = fmaxf(mx, s[u][j]);
      ref[j] = mx == -INFINITY ? 0.f : mx;   // a group with no key yet: keep l = o = 0
      const float corr = exp2f(m[j] - ref[j]);
      l[j] *= corr;
#pragma unroll
      for (int i = 0; i < 8; ++i) o[j][i] *= corr;
      m[j] = mx;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float vf[8];
      bf16x8_to_f32(vr[u], vf);
#pragma unroll
      for (int j = 0; j < NQ; ++j) {
        const float p = exp2f(s[u][j] - ref[j]);
        l[j] += p;
#pragma unroll
        for (int i = 0; i < 8; ++i) o[j][i] = fmaf(p, vf[i], o[j][i]);
      }
    }
  }

  const size_t bh = static_cast<size_t>(b) * H + h;
#pragma unroll
  for (int j = 0; j < NQ; ++j) {
    if (j < n) {
      if (j > 0) __syncthreads();   // the previous query's merge has read the shared buffers
      decode_merge<D, NG>(a, bh * kAppendMaxTokens + j, split, grp, sub, active, m[j], l[j], o[j], s_m, s_l, s_o,
                          s_last, a.out + (static_cast<size_t>(t0 + j) * H + h) * D);
    }
  }
}

#define PG_CHECK_LAUNCH(name)                                                       \
  do {                                                                              \
    cudaError_t e__ = cudaGetLastError();                                           \
    if (e__ != cudaSuccess) {                                                       \
      fprintf(stderr, "pipegoose_b200: %s launch failed: %s\n", name, cudaGetErrorString(e__)); \
      return -1;                                                                    \
    }                                                                               \
  } while (0)

template <int D, bool PAGED>
static int launch_decode(const DecodeArgs& a, int B, cudaStream_t s) {
  if (launch_pdl(decode_attention_kernel<D, PAGED>, dim3(a.splits, a.H, B), dim3(kDecThreads), 0, s, a) != cudaSuccess)
    return -1;
  PG_CHECK_LAUNCH("decode_attention");
  return 0;
}

template <bool PAGED>
static int launch_decode_d(const DecodeArgs& a, int B, int D, cudaStream_t s) {
  switch (D) {
    case 64: return launch_decode<64, PAGED>(a, B, s);
    case 80: return launch_decode<80, PAGED>(a, B, s);
    case 128: return launch_decode<128, PAGED>(a, B, s);
    default: return -1;
  }
}

__global__ void __launch_bounds__(256) paged_kv_write_kernel(const uint4* __restrict__ qkv, const int* __restrict__ slot,
                                                             uint4* __restrict__ k_pool, uint4* __restrict__ v_pool,
                                                             int N, int H, int vec) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;   // (n, h, k|v, 16-byte column)
  if (i >= static_cast<long long>(N) * H * 2 * vec) return;
  const int c = static_cast<int>(i % vec);
  long long r = i / vec;
  const int kv = static_cast<int>(r & 1);
  r >>= 1;
  const int h = static_cast<int>(r % H);
  const long long n = r / H;
  const int s = __ldg(slot + n);
  const uint4 x = __ldg(qkv + ((n * H + h) * 3 + 1 + kv) * vec + c);
  const size_t dst = ((static_cast<size_t>(s >> kPageShift) * H + h) * kPageSize + (s & (kPageSize - 1))) * vec + c;
  (kv ? v_pool : k_pool)[dst] = x;
}

// One thread per (pair, layer, head, K|V, slot, 16-byte column); threads of slots >= count return at once.  The column-0
// thread of a row also copies its scale (FP8 pools).
__global__ void __launch_bounds__(256) paged_kv_copy_kernel(const int* __restrict__ pairs, uint4* __restrict__ k_pools,
                                                            uint4* __restrict__ v_pools, float* __restrict__ k_scales,
                                                            float* __restrict__ v_scales, int n, int layers,
                                                            int pages, int H, int vec) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(n) * layers * H * 2 * kPageSize * vec) return;
  const int c = static_cast<int>(i % vec);
  long long r = i / vec;
  const int slot = static_cast<int>(r % kPageSize);
  r /= kPageSize;
  const int kv = static_cast<int>(r & 1);
  r >>= 1;
  const int h = static_cast<int>(r % H);
  r /= H;
  const int layer = static_cast<int>(r % layers);
  const int p = static_cast<int>(r / layers);
  if (slot >= __ldg(pairs + 3 * p + 2)) return;
  const long long base = static_cast<long long>(layer) * pages;
  const size_t from = ((base + __ldg(pairs + 3 * p)) * H + h) * kPageSize + slot;
  const size_t to = ((base + __ldg(pairs + 3 * p + 1)) * H + h) * kPageSize + slot;
  uint4* pool = kv ? v_pools : k_pools;
  pool[to * vec + c] = pool[from * vec + c];
  float* scales = kv ? v_scales : k_scales;
  if (c == 0 && scales != nullptr) scales[to] = scales[from];
}

// ---- FP8 pools
constexpr float kFp8Max = 448.0f;   // largest finite e4m3

PG_DEVICE void fp8x16_to_f32(const uint4& r, float* f) {
  const __nv_fp8x2_storage_t* p = reinterpret_cast<const __nv_fp8x2_storage_t*>(&r);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float2 t = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2(p[i], __NV_E4M3)));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

// Quantize one row of vec * 8 bf16 (src) into e4m3 codes and its scale.  The row belongs to a half-warp: lane sub < vec
// holds values 8 * sub .. 8 * sub + 7, the others take part in the amax shuffles only.  Every lane of the warp calls it.
PG_DEVICE void quantize_row_fp8(const uint4* src, int sub, int vec, uint8_t* codes, float* scale) {
  float x[8];
  bf16x8_to_f32(sub < vec ? src[sub] : make_uint4(0, 0, 0, 0), x);
  float a = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) a = fmaxf(a, fabsf(x[i]));
#pragma unroll
  for (int off = 8; off > 0; off >>= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, off));
  if (sub >= vec) return;
  uint2 c = make_uint2(0, 0);
  if (a > 0.f) {
    const float inv = kFp8Max / a;
    __nv_fp8x2_storage_t* cp = reinterpret_cast<__nv_fp8x2_storage_t*>(&c);
#pragma unroll
    for (int i = 0; i < 4; ++i)
      cp[i] = __nv_cvt_float2_to_fp8x2(make_float2(x[2 * i] * inv, x[2 * i + 1] * inv), __NV_SATFINITE, __NV_E4M3);
  }
  reinterpret_cast<uint2*>(codes)[sub] = c;
  if (sub == 0) *scale = a / kFp8Max;
}

// One half-warp per (token, head, K|V) row: lanes 0-15 of warp (n, h) quantize its key, lanes 16-31 its value.
__global__ void __launch_bounds__(256) paged_kv_write_fp8_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                                 const int* __restrict__ slot, uint8_t* k_pool,
                                                                 uint8_t* v_pool, float* k_scales, float* v_scales,
                                                                 int N, int H, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;   // (n, h)
  if (w >= static_cast<long long>(N) * H) return;   // whole warps
  const int lane = threadIdx.x & 31, kv = lane >> 4;
  const int h = static_cast<int>(w % H);
  const long long n = w / H;
  const int s = __ldg(slot + n);
  const size_t at = (static_cast<size_t>(s >> kPageShift) * H + h) * kPageSize + (s & (kPageSize - 1));
  quantize_row_fp8(reinterpret_cast<const uint4*>(qkv + ((n * H + h) * 3 + 1 + kv) * D), lane & 15, D / 8,
                   (kv ? v_pool : k_pool) + at * D, (kv ? v_scales : k_scales) + at);
}

template <int D>
__global__ void __launch_bounds__(kDecThreads) decode_attention_fp8_kernel(const DecodeArgs a) {
  constexpr int VEC = D / 16;                 // lanes holding a key's codes (16 e4m3 = 16 B each)
  constexpr int LPK = VEC <= 4 ? 4 : 8;       // lanes per key: VEC rounded up to a power of two (shuffle reduction)
  constexpr int KPW = 32 / LPK;
  constexpr int NG = kDecWarps * KPW;
  static_assert(D % 16 == 0 && VEC <= 8, "head size");
  __shared__ float s_m[NG], s_l[NG];
  __shared__ float s_o[NG][D];
  __shared__ int s_last;

  pdl_launch_dependents();
  pdl_wait();
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int H = a.H;
  const int pos = __ldg(a.row_pos + b);
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPK;
  const int grp = (threadIdx.x >> 5) * KPW + lane / LPK;
  const bool active = sub < VEC;

  const int chunk = (pos + a.splits) / a.splits;   // ceil((pos + 1) / splits)
  const int k0 = split * chunk;
  const int k1 = min(k0 + chunk, pos + 1);
  const int kend = min(k1, pos);                    // the keys read from the pools: all before pos

  const size_t bh = static_cast<size_t>(b) * H + h;
  const __nv_bfloat16* row = a.qkv + bh * 3 * D;
  const uint4* kc = reinterpret_cast<const uint4*>(a.k_cache);
  const uint4* vc = reinterpret_cast<const uint4*>(a.v_cache);
  const int* tab = a.table + static_cast<size_t>(b) * a.max_pages;
  auto slot_at = [&](int k) -> size_t {   // pool row of key k: its scale, and its codes at D bytes per row
    return (static_cast<size_t>(__ldg(tab + (k >> kPageShift))) * H + h) * kPageSize + (k & (kPageSize - 1));
  };

  if (split == 0 && threadIdx.x < 32) {   // store pos: lanes 0-15 its key, 16-31 its value
    const size_t at = slot_at(pos);
    const int kv = lane >> 4;
    quantize_row_fp8(reinterpret_cast<const uint4*>(row + (1 + kv) * D), lane & 15, D / 8,
                     reinterpret_cast<uint8_t*>(kv ? a.v_cache : a.k_cache) + at * D, (kv ? a.v_scales : a.k_scales) + at);
  }

  const uint4* q_row = reinterpret_cast<const uint4*>(row);
  const uint4* k_new = reinterpret_cast<const uint4*>(row + D);
  const uint4* v_new = reinterpret_cast<const uint4*>(row + 2 * D);
  float q[16];
  bf16x8_to_f32(active ? q_row[2 * sub] : make_uint4(0, 0, 0, 0), q);
  bf16x8_to_f32(active ? q_row[2 * sub + 1] : make_uint4(0, 0, 0, 0), q + 8);
#pragma unroll
  for (int i = 0; i < 16; ++i) q[i] *= a.scale_log2;
  const float slope_log2 = a.slopes[h] * kDecLog2e;

  float m = -INFINITY, l = 0.f, o[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i] = 0.f;
  // the trip count is the same for every thread of the CTA: the shuffles below are never divergent
  for (int kb = k0; kb < kend; kb += NG * kDecUnroll) {
    uint4 kr[kDecUnroll], vr[kDecUnroll];
    float sk[kDecUnroll], sv[kDecUnroll];
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) {
      const int k = kb + u * NG + grp;
      kr[u] = vr[u] = make_uint4(0, 0, 0, 0);
      sk[u] = sv[u] = 0.f;
      if (k < kend) {
        const size_t at = slot_at(k);
        sk[u] = __ldg(a.k_scales + at);
        sv[u] = __ldg(a.v_scales + at);
        if (active) {
          kr[u] = __ldg(kc + at * VEC + sub);
          vr[u] = __ldg(vc + at * VEC + sub);
        }
      }
    }
    float s[kDecUnroll];
    float mx = m;
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) {
      float kf[16];
      fp8x16_to_f32(kr[u], kf);
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) dot = fmaf(q[i], kf[i], dot);
#pragma unroll
      for (int off = LPK / 2; off > 0; off >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, off);
      const int k = kb + u * NG + grp;
      s[u] = k < kend ? fmaf(slope_log2, static_cast<float>(k - pos), dot * sk[u]) : -INFINITY;
      mx = fmaxf(mx, s[u]);
    }
    const float ref = mx == -INFINITY ? 0.f : mx;   // a group with no key yet: keep l = o = 0
    const float corr = exp2f(m - ref);
    l *= corr;
#pragma unroll
    for (int i = 0; i < 16; ++i) o[i] *= corr;
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) {
      const float p = exp2f(s[u] - ref);
      const float w = p * sv[u];
      float vf[16];
      fp8x16_to_f32(vr[u], vf);
      l += p;
#pragma unroll
      for (int i = 0; i < 16; ++i) o[i] = fmaf(w, vf[i], o[i]);
    }
    m = mx;
  }

  if (k0 <= pos && pos < k1) {   // this CTA's range ends at pos: its key and value from qkv, exact, in group 0
    float kf[16], vf[16];
    bf16x8_to_f32(active ? k_new[2 * sub] : make_uint4(0, 0, 0, 0), kf);
    bf16x8_to_f32(active ? k_new[2 * sub + 1] : make_uint4(0, 0, 0, 0), kf + 8);
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) dot = fmaf(q[i], kf[i], dot);
#pragma unroll
    for (int off = LPK / 2; off > 0; off >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, off);
    const float s = grp == 0 ? dot : -INFINITY;
    const float mx = fmaxf(m, s);
    const float ref = mx == -INFINITY ? 0.f : mx;
    const float corr = exp2f(m - ref);
    const float p = exp2f(s - ref);
    bf16x8_to_f32(active ? v_new[2 * sub] : make_uint4(0, 0, 0, 0), vf);
    bf16x8_to_f32(active ? v_new[2 * sub + 1] : make_uint4(0, 0, 0, 0), vf + 8);
    l = fmaf(l, corr, p);
#pragma unroll
    for (int i = 0; i < 16; ++i) o[i] = fmaf(p, vf[i], o[i] * corr);
    m = mx;
  }

  decode_merge<D, NG>(a, bh, split, grp, sub, active, m, l, o, s_m, s_l, s_o, s_last, a.out + bh * D);
}

// One thread per 16 codes: (page i, head, slot, K|V, 16-column group) -> 16 bf16 of page dst[i].
__global__ void __launch_bounds__(256) kv_dequantize_kernel(const uint4* __restrict__ k_pool,
                                                            const uint4* __restrict__ v_pool,
                                                            const float* __restrict__ k_scales,
                                                            const float* __restrict__ v_scales,
                                                            const int* __restrict__ src, const int* __restrict__ dst,
                                                            uint4* __restrict__ k_out, uint4* __restrict__ v_out,
                                                            int n, int rows, int vec) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(n) * rows * 2 * vec) return;
  const int c = static_cast<int>(i % vec);
  long long r = i / vec;
  const int kv = static_cast<int>(r & 1);
  r >>= 1;
  const int row = static_cast<int>(r % rows);   // head * 64 + slot
  const int pi = static_cast<int>(r / rows);
  const size_t from = static_cast<size_t>(__ldg(src + pi)) * rows + row;
  const size_t to = static_cast<size_t>(__ldg(dst + pi)) * rows + row;
  const float sc = __ldg((kv ? v_scales : k_scales) + from);
  float f[16];
  fp8x16_to_f32(__ldg((kv ? v_pool : k_pool) + from * vec + c), f);
  uint4 y[2];
  __nv_bfloat162* yp = reinterpret_cast<__nv_bfloat162*>(y);
#pragma unroll
  for (int j = 0; j < 8; ++j) yp[j] = __floats2bfloat162_rn(f[2 * j] * sc, f[2 * j + 1] * sc);
  uint4* out = (kv ? v_out : k_out) + (to * vec + c) * 2;
  out[0] = y[0];
  out[1] = y[1];
}

}  // namespace pg

using namespace pg;

extern "C" int pg_decode_splits(int B, int H, int span) {
  const int rows = B * H > 0 ? B * H : 1;
  const int by_len = (span + kDecMinChunk - 1) / kDecMinChunk;
  const int by_grid = (kDecTargetCtas + rows - 1) / rows;
  const int n = by_len < by_grid ? by_len : by_grid;
  return n > 1 ? n : 1;
}

extern "C" int pg_decode_attention(const void* qkv, void* k_cache, void* v_cache, const float* slopes, const int* lead,
                                   void* out, float* part, int* ticket, int B, int H, int D, int capacity, int pos,
                                   int splits, float softmax_scale, cudaStream_t s) {
  if (pos < 0 || pos >= capacity || splits < 1 || (splits > 1 && (part == nullptr || ticket == nullptr))) return -1;
  DecodeArgs a;
  a.qkv = static_cast<const __nv_bfloat16*>(qkv);
  a.k_cache = static_cast<__nv_bfloat16*>(k_cache);
  a.v_cache = static_cast<__nv_bfloat16*>(v_cache);
  a.slopes = slopes;
  a.lead = lead;
  a.out = static_cast<__nv_bfloat16*>(out);
  a.part = part;
  a.ticket = ticket;
  a.H = H;
  a.capacity = capacity;
  a.pos = pos;
  a.splits = splits;
  a.scale_log2 = kDecLog2e * (softmax_scale > 0.f ? softmax_scale : 1.0f / sqrtf(static_cast<float>(D)));
  a.table = nullptr;
  a.row_pos = nullptr;
  a.max_pages = 0;
  return launch_decode_d<false>(a, B, D, s);
}

extern "C" int pg_paged_decode_attention(const void* qkv, void* k_pool, void* v_pool, const int* table, const int* pos,
                                         const float* slopes, void* out, float* part, int* ticket, int B, int H, int D,
                                         int max_pages, int max_pos, int splits, float softmax_scale, cudaStream_t s) {
  if (max_pos < 0 || max_pages < 1 || splits < 1 || (splits > 1 && (part == nullptr || ticket == nullptr))) return -1;
  DecodeArgs a;
  a.qkv = static_cast<const __nv_bfloat16*>(qkv);
  a.k_cache = static_cast<__nv_bfloat16*>(k_pool);
  a.v_cache = static_cast<__nv_bfloat16*>(v_pool);
  a.slopes = slopes;
  a.lead = nullptr;
  a.out = static_cast<__nv_bfloat16*>(out);
  a.part = part;
  a.ticket = ticket;
  a.H = H;
  a.capacity = 0;
  a.pos = max_pos;
  a.splits = splits;
  a.scale_log2 = kDecLog2e * (softmax_scale > 0.f ? softmax_scale : 1.0f / sqrtf(static_cast<float>(D)));
  a.table = table;
  a.row_pos = pos;
  a.max_pages = max_pages;
  return launch_decode_d<true>(a, B, D, s);
}

extern "C" int pg_paged_append_attention(const void* qkv, void* k_pool, void* v_pool, const int* table,
                                         const int* cu_seqlens, const int* pos, const float* slopes, void* out,
                                         float* part, int* ticket, int B, int N, int H, int D, int max_pages,
                                         int max_pos, int max_tokens, int splits, float softmax_scale,
                                         cudaStream_t s) {
  if (max_pos < 0 || max_pages < 1 || splits < 1 || max_tokens < 1 || max_tokens > kAppendMaxTokens || N < B ||
      N > static_cast<long long>(B) * max_tokens || ticket == nullptr || (splits > 1 && part == nullptr))
    return -1;
  if (B == 0) return 0;
  DecodeArgs a;
  a.qkv = static_cast<const __nv_bfloat16*>(qkv);
  a.k_cache = static_cast<__nv_bfloat16*>(k_pool);
  a.v_cache = static_cast<__nv_bfloat16*>(v_pool);
  a.slopes = slopes;
  a.cu_seqlens = cu_seqlens;
  a.out = static_cast<__nv_bfloat16*>(out);
  a.part = part;
  a.ticket = ticket;
  a.H = H;
  a.capacity = 0;
  a.pos = max_pos;
  a.splits = splits;
  a.scale_log2 = kDecLog2e * (softmax_scale > 0.f ? softmax_scale : 1.0f / sqrtf(static_cast<float>(D)));
  a.table = table;
  a.row_pos = pos;
  a.max_pages = max_pages;
  a.k_scales = a.v_scales = nullptr;
  // the query tile: the smallest power of two that holds the longest row (more queries cost registers and keys in
  // flight for every row)
  const int most = max_tokens;
  const dim3 grid(splits, H, B), block(kDecThreads);
  cudaError_t e;
#define PG_APPEND_CASE(DD)                                                                      \
  case DD:                                                                                      \
    e = most <= 1   ? launch_pdl(append_attention_kernel<DD, 1>, grid, block, 0, s, a)          \
        : most <= 2 ? launch_pdl(append_attention_kernel<DD, 2>, grid, block, 0, s, a)          \
        : most <= 4 ? launch_pdl(append_attention_kernel<DD, 4>, grid, block, 0, s, a)          \
                    : launch_pdl(append_attention_kernel<DD, 8>, grid, block, 0, s, a);         \
    break;
  switch (D) {
    PG_APPEND_CASE(64)
    PG_APPEND_CASE(80)
    PG_APPEND_CASE(128)
    default: return -1;
  }
#undef PG_APPEND_CASE
  if (e != cudaSuccess) return -1;
  PG_CHECK_LAUNCH("append_attention");
  return 0;
}

extern "C" int pg_paged_kv_write(const void* qkv, const int* slot, void* k_pool, void* v_pool, int N, int H, int D,
                                 cudaStream_t s) {
  if (N < 0 || H < 1 || D % 8 != 0) return -1;
  if (N == 0) return 0;
  const long long n = static_cast<long long>(N) * H * 2 * (D / 8);
  if (launch_pdl(paged_kv_write_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, s,
                 static_cast<const uint4*>(qkv), slot, static_cast<uint4*>(k_pool), static_cast<uint4*>(v_pool), N, H,
                 D / 8) != cudaSuccess)
    return -1;
  PG_CHECK_LAUNCH("paged_kv_write");
  return 0;
}

extern "C" int pg_paged_kv_write_fp8(const void* qkv, const int* slot, void* k_pool, void* v_pool, float* k_scales,
                                     float* v_scales, int N, int H, int D, cudaStream_t s) {
  if (N < 0 || H < 1 || D % 8 != 0 || D / 8 > 16) return -1;
  if (N == 0) return 0;
  const long long threads = static_cast<long long>(N) * H * 32;
  if (launch_pdl(paged_kv_write_fp8_kernel, dim3(static_cast<unsigned>((threads + 255) / 256)), dim3(256), 0, s,
                 static_cast<const __nv_bfloat16*>(qkv), slot, static_cast<uint8_t*>(k_pool),
                 static_cast<uint8_t*>(v_pool), k_scales, v_scales, N, H, D) != cudaSuccess)
    return -1;
  PG_CHECK_LAUNCH("paged_kv_write_fp8");
  return 0;
}

extern "C" int pg_paged_decode_attention_fp8(const void* qkv, void* k_pool, void* v_pool, float* k_scales,
                                             float* v_scales, const int* table, const int* pos, const float* slopes,
                                             void* out, float* part, int* ticket, int B, int H, int D, int max_pages,
                                             int max_pos, int splits, float softmax_scale, cudaStream_t s) {
  if (max_pos < 0 || max_pages < 1 || splits < 1 || (splits > 1 && (part == nullptr || ticket == nullptr))) return -1;
  DecodeArgs a;
  a.qkv = static_cast<const __nv_bfloat16*>(qkv);
  a.k_cache = static_cast<__nv_bfloat16*>(k_pool);
  a.v_cache = static_cast<__nv_bfloat16*>(v_pool);
  a.slopes = slopes;
  a.lead = nullptr;
  a.out = static_cast<__nv_bfloat16*>(out);
  a.part = part;
  a.ticket = ticket;
  a.H = H;
  a.capacity = 0;
  a.pos = max_pos;
  a.splits = splits;
  a.scale_log2 = kDecLog2e * (softmax_scale > 0.f ? softmax_scale : 1.0f / sqrtf(static_cast<float>(D)));
  a.table = table;
  a.row_pos = pos;
  a.max_pages = max_pages;
  a.k_scales = k_scales;
  a.v_scales = v_scales;
  cudaError_t e;
  switch (D) {
    case 64: e = launch_pdl(decode_attention_fp8_kernel<64>, dim3(splits, H, B), dim3(kDecThreads), 0, s, a); break;
    case 80: e = launch_pdl(decode_attention_fp8_kernel<80>, dim3(splits, H, B), dim3(kDecThreads), 0, s, a); break;
    case 128: e = launch_pdl(decode_attention_fp8_kernel<128>, dim3(splits, H, B), dim3(kDecThreads), 0, s, a); break;
    default: return -1;
  }
  if (e != cudaSuccess) return -1;
  PG_CHECK_LAUNCH("decode_attention_fp8");
  return 0;
}

extern "C" int pg_paged_kv_dequantize(const void* k_pool, const void* v_pool, const float* k_scales,
                                      const float* v_scales, const int* src, const int* dst, void* k_out, void* v_out,
                                      int n, int H, int D, cudaStream_t s) {
  if (n < 0 || H < 1 || D % 16 != 0) return -1;
  if (n == 0) return 0;
  const long long threads = static_cast<long long>(n) * H * kPageSize * 2 * (D / 16);
  if (launch_pdl(kv_dequantize_kernel, dim3(static_cast<unsigned>((threads + 255) / 256)), dim3(256), 0, s,
                 static_cast<const uint4*>(k_pool), static_cast<const uint4*>(v_pool), k_scales, v_scales, src, dst,
                 static_cast<uint4*>(k_out), static_cast<uint4*>(v_out), n, H * kPageSize, D / 16) != cudaSuccess)
    return -1;
  PG_CHECK_LAUNCH("kv_dequantize");
  return 0;
}

extern "C" int pg_paged_kv_copy(const int* pairs, void* k_pools, void* v_pools, float* k_scales, float* v_scales, int n,
                                int layers, int pages, int H, int row_bytes, cudaStream_t s) {
  if (n < 0 || layers < 1 || pages < 1 || H < 1 || row_bytes % 16 != 0 || (k_scales == nullptr) != (v_scales == nullptr))
    return -1;
  if (n == 0) return 0;
  const long long threads = static_cast<long long>(n) * layers * H * 2 * kPageSize * (row_bytes / 16);
  if (launch_pdl(paged_kv_copy_kernel, dim3(static_cast<unsigned>((threads + 255) / 256)), dim3(256), 0, s, pairs,
                 static_cast<uint4*>(k_pools), static_cast<uint4*>(v_pools), k_scales, v_scales, n, layers, pages, H,
                 row_bytes / 16) != cudaSuccess)
    return -1;
  PG_CHECK_LAUNCH("paged_kv_copy");
  return 0;
}
