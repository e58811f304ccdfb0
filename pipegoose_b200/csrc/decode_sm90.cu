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
// bound on max(pos[b])); each row cuts its own range into `splits` chunks, so the bound only shapes the grid.  Rows
// own disjoint pages, so the write of pos[b]'s slot races no read either.
//
// paged_kv_write_kernel stores the k / v of a packed prefill into the pools: token n's heads go to slot[n]
// (page * 64 + offset), 16 bytes per thread.
#include "launch.h"
#include "pdl_launch.cuh"
#include "ptx.cuh"
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

struct DecodeArgs {
  const __nv_bfloat16* qkv;
  __nv_bfloat16* k_cache;
  __nv_bfloat16* v_cache;
  const float* slopes;
  const int* lead;
  __nv_bfloat16* out;
  float* part;   // [B*H, splits, D + 2]: (m, l, o[D]) per split (splits > 1)
  int* ticket;   // [B*H], zero between calls
  int H, capacity, pos, splits;
  float scale_log2;
  // paged form only (k_cache / v_cache are then the pools, capacity and lead unused)
  const int* table;     // [B, max_pages] page ids
  const int* row_pos;   // [B] each row's new-token position
  int max_pages;
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

  // merge the CTA's key groups
  if (sub == 0) {
    s_m[grp] = m;
    s_l[grp] = l;
  }
  if (active) {
#pragma unroll
    for (int i = 0; i < 8; ++i) s_o[grp][sub * 8 + i] = o[i];
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
  __nv_bfloat16* out = a.out + bh * D;
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
