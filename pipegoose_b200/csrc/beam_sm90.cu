// Beam search's candidate choice (continuous batching), sm_90a: a fused log-softmax and top-k over the rows of every
// request.
//
//   logits : [N, V] bf16 or fp32, row stride ld (elements)       scores : fp32 [N], each row's running beam score
//   cu     : int32 [R + 1], request r owns rows cu[r] .. cu[r+1] - 1
//
// For every request r the kernel returns the k (<= 16) best candidates (row n, token v) of its rows by
//   score = scores[n] + (logit[n, v] - lse[n]),   lse[n] = log(sum_v exp(logit[n, v])),
// in fp32, sorted by descending score; equal scores go to the lower (row, token), which is what a stable descending
// sort over the flat index n * V + v gives.  -inf logits (vocabulary padding) take no part in the sums, as in
// ce_stats_kernel; they stay candidates with a score of -inf.  Optionally it also writes lse[n].
//
// Grid (split, row).  A row's vocabulary is cut into `splits` chunks, one per CTA of 256 threads.  Each thread keeps an
// online (max, sum-exp) and its own top-KP raw logits (KP, a power of two >= k, in registers) over the 16-byte vectors
// it reads.  The CTA reduces both in a fixed order and writes its partial (m, s) and top-KP to the workspace.  A
// request's best k candidates are among each row's best k logits (within a row the score is monotone in the logit), so
// the CTA that takes the request's last arrival ticket merges the partials: each row's lse from its splits in split
// order, then k rounds of a block-wide arg-max over rows x splits x KP candidates.  It then resets the ticket.  No CTA
// waits for another and no atomic touches the arithmetic, so the result is bitwise reproducible.
#include "launch.h"
#include "pdl_launch.cuh"
#include "ptx.cuh"
#include <climits>
#include <cmath>
#include <cstdio>

namespace pg {

constexpr int kBeamThreads = 256;
constexpr int kBeamMaxCand = 4096;     // candidates a merging CTA holds: rows * splits * KP of one request
constexpr int kBeamMaxRows = 64;       // rows of one request
constexpr int kBeamMinChunk = 2048;    // fewest logits a CTA is given
constexpr int kBeamTargetCtas = 132 * 4;

struct BeamArgs {
  const void* logits;
  const float* scores;
  const int* cu;
  float* part_stat;     // [N, splits, 2]: (m, s)
  float* part_val;      // [N, splits, KP]
  int* part_idx;        // [N, splits, KP], INT_MAX: no candidate
  int* ticket;          // [R], zero between calls
  float* out_score;     // [R, k]
  int* out_token;       // [R, k]
  int* out_row;         // [R, k]
  float* lse;           // [N] or nullptr
  long long ld;
  int V, R, k, chunk, splits;
};

// Does (va, ia) come before (vb, ib)?  Higher value first, then lower index.
PG_DEVICE bool beam_before(float va, int ia, float vb, int ib) { return va > vb || (va == vb && ia < ib); }

template <int KP>
PG_DEVICE void beam_push(float (&v)[KP], int (&id)[KP], float x, int i) {
  if (x < v[KP - 1] || !beam_before(x, i, v[KP - 1], id[KP - 1])) return;
  v[KP - 1] = x;
  id[KP - 1] = i;
#pragma unroll
  for (int j = KP - 1; j > 0; --j) {
    if (beam_before(v[j], id[j], v[j - 1], id[j - 1])) {
      const float tv = v[j]; v[j] = v[j - 1]; v[j - 1] = tv;
      const int ti = id[j]; id[j] = id[j - 1]; id[j - 1] = ti;
    }
  }
}

// Block-wide best (value, index) of every thread's pair; every thread gets it.  Ends with a barrier, so the scratch
// arrays can be reused at once.
PG_DEVICE void beam_block_best(float& v, int& i, float* sv, int* si) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (beam_before(ov, oi, v, i)) { v = ov; i = oi; }
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { sv[w] = v; si[w] = i; }
  __syncthreads();
  v = sv[0];
  i = si[0];
#pragma unroll
  for (int j = 1; j < kBeamThreads / 32; ++j)
    if (beam_before(sv[j], si[j], v, i)) { v = sv[j]; i = si[j]; }
  __syncthreads();
}

template <typename T>
PG_DEVICE float beam_load(const T* p) {
  if constexpr (sizeof(T) == 2) return __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(p));
  else return *p;
}

template <typename T, int KP>
__global__ void __launch_bounds__(kBeamThreads) beam_topk_kernel(const BeamArgs a) {
  __shared__ float s_val[kBeamMaxCand];
  __shared__ int s_idx[kBeamMaxCand];
  __shared__ float s_rv[kBeamThreads / 32], s_lse[kBeamMaxRows];
  __shared__ int s_ri[kBeamThreads / 32];
  __shared__ int s_last;
  pdl_launch_dependents();
  pdl_wait();
  const int split = blockIdx.x, n = blockIdx.y, tid = threadIdx.x;
  const int c0 = split * a.chunk, c1 = max(c0, min(a.V, c0 + a.chunk));
  const T* row = static_cast<const T*>(a.logits) + static_cast<long long>(n) * a.ld;

  // ---- this CTA's chunk: online (m, s) and top-KP per thread
  float m = -INFINITY, s = 0.f;
  float v[KP];
  int id[KP];
#pragma unroll
  for (int j = 0; j < KP; ++j) { v[j] = -INFINITY; id[j] = INT_MAX; }
  auto take = [&](float x, int i) {
    beam_push<KP>(v, id, x, i);
    if (x == -INFINITY) return;
    const float nm = fmaxf(m, x);
    s = s * __expf(m - nm) + __expf(x - nm);
    m = nm;
  };
  constexpr int E = 16 / sizeof(T);                       // elements per 16-byte load
  const uintptr_t addr = reinterpret_cast<uintptr_t>(row + c0);
  int head = static_cast<int>(((16 - (addr & 15)) & 15) / sizeof(T));   // elements before the first aligned vector
  if ((addr & (sizeof(T) - 1)) != 0) head = c1 - c0;      // misaligned element type: scalar loads only
  head = min(head, c1 - c0);
  const int nvec = (c1 - c0 - head) / E;
  const int body = c0 + head, tail = body + nvec * E;
  if (tid < head) take(beam_load(row + c0 + tid), c0 + tid);
  for (int q = tid; q < nvec; q += kBeamThreads) {
    const uint4 raw = ld_global_nc_v4(row + body + q * E);
    float f[E];
    if constexpr (sizeof(T) == 2) {
      const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 t = unpack_bf16x2(w[j]);
        f[2 * j] = t.x;
        f[2 * j + 1] = t.y;
      }
    } else {
      f[0] = __uint_as_float(raw.x); f[1] = __uint_as_float(raw.y);
      f[2] = __uint_as_float(raw.z); f[3] = __uint_as_float(raw.w);
    }
    const int i0 = body + q * E;
    float cm = -INFINITY;
#pragma unroll
    for (int j = 0; j < E; ++j) {
      beam_push<KP>(v, id, f[j], i0 + j);
      cm = fmaxf(cm, f[j]);
    }
    if (cm == -INFINITY) continue;         // E masked logits: exp(-inf - -inf) would be NaN
    const float nm = fmaxf(m, cm);
    float add = 0.f;
#pragma unroll
    for (int j = 0; j < E; ++j) add += __expf(f[j] - nm);
    s = s * __expf(m - nm) + add;
    m = nm;
  }
  for (int i = tail + tid; i < c1; i += kBeamThreads) take(beam_load(row + i), i);

  // ---- CTA partial: (m, s) in warp order, then the CTA's top-KP by KP rounds of a block arg-max over list heads
  {
    const float wm = warp_max(m);
    float ws = warp_sum(s * (m == -INFINITY ? 0.f : __expf(m - wm)));
    const int lane = tid & 31, w = tid >> 5;
    if (lane == 0) { s_rv[w] = wm; s_lse[w] = ws; }
    __syncthreads();
    if (tid == 0) {
      float gm = -INFINITY, gs = 0.f;
      for (int j = 0; j < kBeamThreads / 32; ++j) gm = fmaxf(gm, s_rv[j]);
      for (int j = 0; j < kBeamThreads / 32; ++j) gs += s_rv[j] == -INFINITY ? 0.f : s_lse[j] * expf(s_rv[j] - gm);
      float* st = a.part_stat + (static_cast<long long>(n) * a.splits + split) * 2;
      st[0] = gm;
      st[1] = gs;
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < KP; ++j) { s_val[tid * KP + j] = v[j]; s_idx[tid * KP + j] = id[j]; }
  __syncthreads();
  {
    int h = 0;                                             // this thread's list head
    float* pv = a.part_val + (static_cast<long long>(n) * a.splits + split) * KP;
    int* pi = a.part_idx + (static_cast<long long>(n) * a.splits + split) * KP;
    for (int r = 0; r < KP; ++r) {
      float bv = h < KP ? s_val[tid * KP + h] : -INFINITY;
      int bi = h < KP ? s_idx[tid * KP + h] : INT_MAX;
      const int mine = bi;
      beam_block_best(bv, bi, s_rv, s_ri);
      if (bi != INT_MAX && mine == bi) ++h;               // token indices are unique within a row
      if (tid == 0) { pv[r] = bv; pi[r] = bi; }
    }
  }

  // ---- the last CTA of the request merges
  int r = 0, lo = 0, hi = a.R;                             // r: the request whose rows hold n
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(a.cu + mid + 1) <= n) lo = mid + 1; else hi = mid;
  }
  r = lo;
  const int first = __ldg(a.cu + r), rows = __ldg(a.cu + r + 1) - first;
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const int prev = atomicAdd(a.ticket + r, 1);
    s_last = prev == rows * a.splits - 1;
    if (s_last) a.ticket[r] = 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (tid < rows) {
    const float* st = a.part_stat + static_cast<long long>(first + tid) * a.splits * 2;
    float gm = -INFINITY, gs = 0.f;
    for (int j = 0; j < a.splits; ++j) gm = fmaxf(gm, __ldcg(st + 2 * j));
    for (int j = 0; j < a.splits; ++j) {
      const float mj = __ldcg(st + 2 * j);
      if (mj != -INFINITY) gs += __ldcg(st + 2 * j + 1) * expf(mj - gm);
    }
    const float l = gm == -INFINITY ? -INFINITY : gm + logf(gs);
    s_lse[tid] = l;
    if (a.lse != nullptr) a.lse[first + tid] = l;
  }
  __syncthreads();
  const int per_row = a.splits * KP, C = rows * per_row;
  for (int e = tid; e < C; e += kBeamThreads) {
    const int j = e / per_row;
    const long long off = static_cast<long long>(first) * per_row + e;
    const int idx = __ldcg(a.part_idx + off);
    if (idx == INT_MAX) {
      s_val[e] = -INFINITY;
      s_idx[e] = INT_MAX;
    } else {
      s_val[e] = __ldg(a.scores + first + j) + (__ldcg(a.part_val + off) - s_lse[j]);
      s_idx[e] = j * a.V + idx;
    }
  }
  __syncthreads();
  for (int q = 0; q < a.k; ++q) {
    float bv = -INFINITY;
    int bi = INT_MAX, be = -1;
    for (int e = tid; e < C; e += kBeamThreads)
      if (beam_before(s_val[e], s_idx[e], bv, bi)) { bv = s_val[e]; bi = s_idx[e]; be = e; }
    const int mine = bi;
    beam_block_best(bv, bi, s_rv, s_ri);
    if (be >= 0 && mine == bi && bi != INT_MAX) { s_val[be] = -INFINITY; s_idx[be] = INT_MAX; }
    if (tid == 0) {
      const long long o = static_cast<long long>(r) * a.k + q;
      a.out_score[o] = bv;
      a.out_token[o] = bi == INT_MAX ? -1 : bi % a.V;
      a.out_row[o] = bi == INT_MAX ? -1 : first + bi / a.V;
    }
    __syncthreads();
  }
}

}  // namespace pg

using namespace pg;

#define PG_CHECK_LAUNCH(name)                                                       \
  do {                                                                              \
    cudaError_t e__ = cudaGetLastError();                                           \
    if (e__ != cudaSuccess) {                                                       \
      fprintf(stderr, "pipegoose_b200: %s launch failed: %s\n", name, cudaGetErrorString(e__)); \
      return -1;                                                                    \
    }                                                                               \
  } while (0)

extern "C" int pg_beam_topk_kp(int k) { return k <= 2 ? 2 : k <= 4 ? 4 : k <= 8 ? 8 : 16; }

extern "C" int pg_beam_topk_splits(int N, int V, int k, int max_rows) {
  const int kp = pg_beam_topk_kp(k);
  int s = (kBeamTargetCtas + N - 1) / (N > 0 ? N : 1);
  const int by_len = (V + kBeamMinChunk - 1) / kBeamMinChunk;
  const int by_smem = kBeamMaxCand / (kp * (max_rows > 0 ? max_rows : 1));
  s = s < by_len ? s : by_len;
  s = s < by_smem ? s : by_smem;
  if (s < 1) s = 1;
  const int chunk = ((V + s - 1) / s + 63) / 64 * 64;    // whole 64-element chunks; no split is left empty
  return (V + chunk - 1) / chunk;
}

extern "C" int pg_beam_topk(const void* logits, int fp32, long long ld, const float* scores, const int* cu,
                            float* part, int* ticket, float* out_score, int* out_token, int* out_row, float* lse, int N,
                            int V, int R, int k, int max_rows, int splits, cudaStream_t s) {
  const int kp = pg_beam_topk_kp(k);
  if (N < 1 || R < 1 || V < k || k < 1 || k > 16 || max_rows < 1 || max_rows > kBeamMaxRows || splits < 1 ||
      max_rows * splits * kp > kBeamMaxCand)
    return -1;
  BeamArgs a;
  a.logits = logits;
  a.scores = scores;
  a.cu = cu;
  const long long slots = static_cast<long long>(N) * splits;
  a.part_stat = part;
  a.part_val = part + slots * 2;
  a.part_idx = reinterpret_cast<int*>(part + slots * (2 + kp));
  a.ticket = ticket;
  a.out_score = out_score;
  a.out_token = out_token;
  a.out_row = out_row;
  a.lse = lse;
  a.ld = ld;
  a.V = V;
  a.R = R;
  a.k = k;
  a.splits = splits;
  a.chunk = ((V + splits - 1) / splits + 63) / 64 * 64;
  const dim3 grid(splits, N), block(kBeamThreads);
  cudaError_t e;
#define PG_BEAM_CASE(KK)                                                                                     \
  case KK:                                                                                                   \
    e = fp32 ? launch_pdl(beam_topk_kernel<float, KK>, grid, block, 0, s, a)                                 \
             : launch_pdl(beam_topk_kernel<__nv_bfloat16, KK>, grid, block, 0, s, a);                        \
    break;
  switch (kp) {
    PG_BEAM_CASE(2)
    PG_BEAM_CASE(4)
    PG_BEAM_CASE(8)
    PG_BEAM_CASE(16)
    default: return -1;
  }
#undef PG_BEAM_CASE
  if (e != cudaSuccess) return -1;
  PG_CHECK_LAUNCH("beam_topk");
  return 0;
}
