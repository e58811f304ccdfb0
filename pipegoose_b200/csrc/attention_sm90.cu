// Causal ALiBi flash attention for sm_90a on Bloom's fused QKV layout.
//
//   qkv : [B*S, H*3*D] bf16, each row laid out [head][q|k|v][D]      out : [B*S, H*D] bf16
//   scores = q.k / sqrt(D) + slope[head] * (key_pos - query_pos)  (== slope * key_pos under softmax)
//
// Forward: one CTA per (128-query block, head, batch).  A TMA warp streams Q once and K/V blocks
// through a 2-stage ring; two consumer warpgroups own 64 query rows each and compute S = Q K^T with
// wgmma (fp32 accumulators in registers), the online softmax in registers (a row is spread over the
// four threads of a quad), and O += P V with P taken straight from registers as the A operand (the
// accumulator fragment of S is the A fragment of P).  [S, S] never exists.
//
// Backward: one CTA per (128-key block, head, batch) looping over the 64-row query blocks at or below
// the diagonal.  A pre-kernel writes each query's (lse * log2e, -delta * scale) pair and zeroes
// the fp32 dQ buffer; the TMA warp loads a query block's pairs next to its Q and dO.  Two consumer
// warpgroups own 64 keys each: S^T = K Q^T and dP^T = V dO^T on the tensor cores, P^T / dS^T
// recomputed in registers, dV += P^T dO and dK += dS^T Q with P^T / dS^T as register A operands
// (dV, dK accumulate in registers across the loop).  dS^T of all 128 keys is staged in shared memory
// and each warpgroup computes half of dQ = dS K by output columns, contracting over all 128 keys; its
// fp32 tile goes through shared memory and one thread adds it into the dQ buffer with a TMA reduce.
//
// Packed sequences (SEG = true): seg_start[b*S + s] is the row-relative position where the document holding token s
// begins (non-decreasing along a row), and query q sees key k iff seg_start[q] <= k <= q.  The forward starts its key
// loop at the block holding the CTA's first query's document start; the backward ends its query loop at the end of the
// document holding the key block's last key.  Key / query blocks outside those ranges hold no visible pair and are
// never loaded.  SEG = false compiles to the kernels without the lower bound.
//
// Paged prefill (PAGED = true, inference only, no LSE): one CTA per (128-query block, head, sequence r).  The queries
// are the new tokens cu_seqlens[r] .. cu_seqlens[r+1]-1 of a packed qkv, at positions start[r], start[r]+1, ...; their
// keys and values are read from the page pools [num_pages, H, 64, D] through the block table, never from qkv, so a
// cached prefix and the new tokens (already stored by paged_kv_write) are read the same way.  Query at position p sees
// keys 0 <= k <= p.  A 128-key block is two pages, each loaded as 64-row TMA boxes at an 8 KB offset, which lands in
// the same swizzled layout as one 128-row box: the consumer loop is shared.  Pool slots past the CTA's last query
// position may hold anything (NaN included): the second page of the last block is not loaded when it lies wholly
// past it, and V rows past it are zeroed in shared memory before P.V (a masked p = 0 times NaN would still be NaN).
// D = 80 runs as D = 128: the pool maps have 80 columns, so TMA's out-of-bounds fill zeroes K / V columns 80..127.
#include "launch.h"
#include "pdl_launch.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"
#include <cstdio>
#include <cstring>
#include <mutex>
#include <unordered_map>

namespace pg {

int make_tmap_bf16_2d(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld,
                      uint32_t box_rows, uint32_t box_cols);
int make_tmap_f32_3d(CUtensorMap* out, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t box1);

constexpr int ATT_BM = 128;      // queries per forward CTA
constexpr int ATT_BN = 128;      // keys per block
constexpr int ATT_BWD_BM = 64;   // queries per backward step
constexpr int kAttThreads = 384;  // warpgroup 0: warp 0 TMA; warpgroups 1, 2: consumers
constexpr float kLog2e = 1.4426950408889634f;

PG_DEVICE float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// A operand (k16 slice kk) of a bf16 product from an fp32 accumulator fragment (columns 16 kk .. 16 kk + 15)
template <int R>
PG_DEVICE void acc_to_a(const float (&d)[R], int kk, uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(d[8 * kk + 0], d[8 * kk + 1]);
  a[1] = pack_bf16x2(d[8 * kk + 2], d[8 * kk + 3]);
  a[2] = pack_bf16x2(d[8 * kk + 4], d[8 * kk + 5]);
  a[3] = pack_bf16x2(d[8 * kk + 6], d[8 * kk + 7]);
}

constexpr int kAttRegsLight = 24;
constexpr int kAttRegsConsumer = 240;

template <int D>
struct AttFwdCfg {
  static constexpr int kTileBytes = ATT_BM * D * 2;  // Q, K or V tile: D/64 atoms of [128 rows x 128 B]
  static constexpr int kStages = 2;
  static constexpr int kSmemBytes = kTileBytes * (1 + 2 * kStages) + 256 + 1024 /*align*/;
};

struct AttFwdArgs {
  __nv_bfloat16* out;
  float* lse;  // [B, H, S] natural log
  const float* slopes;
  int B, S, H, ld_out;
  float scale_log2;  // log2(e) / sqrt(D)
  const int* seg_start;  // [B*S] document start of every token (SEG only)
  // PAGED only (B = number of sequences, S = max_len, the host bound on new tokens per sequence)
  const int* cu_seqlens;  // [B+1] rows of each sequence in qkv
  const int* start;       // [B] position of each sequence's first new token
  const int* table;       // [B, max_pages] pages of each sequence
  int max_pages, H_pool;  // table width; heads per page of the pools
  int d_out;              // columns stored per head (80 for bloom-3b on the D = 128 instantiation)
};

template <int D, bool SEG, bool PAGED = false>
__global__ void __launch_bounds__(kAttThreads, 1)
    attention_fwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, const AttFwdArgs args,
                         const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v) {
  using Cfg = AttFwdCfg<D>;
  constexpr int ST = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Cfg::kTileBytes;
  uint8_t* sV = sK + ST * Cfg::kTileBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + ST * Cfg::kTileBytes);
  uint64_t* q_full = bars;            // 1
  uint64_t* kv_full = bars + 1;       // ST
  uint64_t* kv_empty = kv_full + ST;  // ST

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) pdl_launch_dependents();
  const int num_qb = (args.S + ATT_BM - 1) / ATT_BM;
  const int qb = num_qb - 1 - blockIdx.x;  // longest (most key blocks) first
  const int head = blockIdx.y, batch = blockIdx.z;
  int num_kb = qb + 1;
  int row0 = batch * args.S + qb * ATT_BM;  // global row of the first query
  // (PAGED: qkv's heads are d_out wide, e.g. 80 on the D = 128 instantiation; K / V come from the pools)
  const int col_q = head * 3 * (PAGED ? args.d_out : D), col_k = col_q + D, col_v = col_q + 2 * D;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tm_qkv);
    if constexpr (PAGED) {
      tma_prefetch_desc(&tm_k);
      tma_prefetch_desc(&tm_v);
    }
    mbar_init(q_full, 1);
    for (int i = 0; i < ST; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);  // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // prologue above overlapped the predecessor; Q/K/V are read below
  // first key block with a visible pair: seg_start is non-decreasing, so the first query's document start is the CTA's
  // lowest.  Producer and consumers run the same j0 .. num_kb - 1.
  int j0 = 0;
  if constexpr (SEG) j0 = args.seg_start[row0] / ATT_BN;
  // PAGED: the sequence's new tokens n_new, the position of the CTA's first query and of its last real one
  int n_new = 0, p_first = 0, p_last = 0;
  if constexpr (PAGED) {
    const int n0 = args.cu_seqlens[batch];
    n_new = args.cu_seqlens[batch + 1] - n0;
    if (qb * ATT_BM >= n_new) return;  // past this sequence's end (the grid is sized from the longest)
    p_first = args.start[batch] + qb * ATT_BM;
    p_last = args.start[batch] + min(n_new, qb * ATT_BM + ATT_BM) - 1;
    row0 = n0 + qb * ATT_BM;
    num_kb = p_last / ATT_BN + 1;
  }

  if (warp < 4) {
    setmaxnreg_dec<kAttRegsLight>();
    if (warp == 0) {
      // ===================== TMA producer =====================
      if (lane == 0) {
        mbar_arrive_expect_tx(q_full, Cfg::kTileBytes);
#pragma unroll
        for (int a = 0; a < D / 64; ++a) tma_load_2d(sQ + a * 16384, &tm_qkv, q_full, col_q + a * 64, row0);
      }
      int stage = 0;
      uint32_t phase = 0;
      for (int j = j0; j < num_kb; ++j) {
        mbar_wait(&kv_empty[stage], phase ^ 1);
        if (PAGED && lane == 0) {
          // one 64-row box per page and atom; the second page is skipped when it holds no key <= p_last
          const int pages = j * ATT_BN + 64 <= p_last ? 2 : 1;
          const int* trow = args.table + static_cast<size_t>(batch) * args.max_pages + 2 * j;
          mbar_arrive_expect_tx(&kv_full[stage], pages * Cfg::kTileBytes);
          for (int pg = 0; pg < pages; ++pg) {
            const int prow = (trow[pg] * args.H_pool + head) * 64;
#pragma unroll
            for (int a = 0; a < D / 64; ++a) {
              const int off = stage * Cfg::kTileBytes + a * 16384 + pg * 8192;
              tma_load_2d(sK + off, &tm_k, &kv_full[stage], a * 64, prow);
              tma_load_2d(sV + off, &tm_v, &kv_full[stage], a * 64, prow);
            }
          }
        } else if (lane == 0) {
          const int krow = batch * args.S + j * ATT_BN;
          mbar_arrive_expect_tx(&kv_full[stage], 2 * Cfg::kTileBytes);
#pragma unroll
          for (int a = 0; a < D / 64; ++a) {
            tma_load_2d(sK + stage * Cfg::kTileBytes + a * 16384, &tm_qkv, &kv_full[stage], col_k + a * 64, krow);
            tma_load_2d(sV + stage * Cfg::kTileBytes + a * 16384, &tm_qkv, &kv_full[stage], col_v + a * 64, krow);
          }
        }
        __syncwarp();
        if (++stage == ST) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }
  setmaxnreg_inc<kAttRegsConsumer>();
  // ===================== consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) =====================
  const int wg = (warp >> 2) - 1, wl = warp & 3;
  const int tid_wg = threadIdx.x & 127;
  const int t4 = lane & 3;
  int qpos[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) qpos[hh] = qb * ATT_BM + 64 * wg + 16 * wl + (lane >> 2) + 8 * hh;
  int qrow[2] = {0, 0};  // PAGED: row index inside the sequence; qpos the position, rows past the end read the last
  if constexpr (PAGED) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      qrow[hh] = qpos[hh];
      qpos[hh] = min(p_first - qb * ATT_BM + qpos[hh], p_last);
    }
  }
  const float slope2 = args.slopes[head] * kLog2e;
  int seg[2] = {0, 0};  // document start of each row (padded rows of the last block read the last token's)
  if constexpr (SEG) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) seg[hh] = args.seg_start[batch * args.S + min(qpos[hh], args.S - 1)];
  }
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float s[ATT_BN / 2];
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  const uint32_t aQ = smem_u32(sQ) + wg * 8192;
  mbar_wait(q_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int j = j0; j < num_kb; ++j) {
    mbar_wait(&kv_full[stage], phase);
    const uint32_t aK = smem_u32(sK + stage * Cfg::kTileBytes), aV = smem_u32(sV + stage * Cfg::kTileBytes);
    if constexpr (PAGED) {
      // V rows past p_last (unwritten slots, or the page that was not loaded) -> 0 before P.V; the two consumer
      // warpgroups split the rows and meet at a named barrier.  Masked K rows need nothing: their scores become -inf.
      const int r0 = p_last + 1 - j * ATT_BN;
      if (r0 < ATT_BN) {
        uint8_t* v = sV + stage * Cfg::kTileBytes;
        const int chunks = (ATT_BN - r0) * 8;  // 16-byte chunks per atom
        for (int c = threadIdx.x - 128; c < chunks * (D / 64); c += 256) {
          const int a = c / chunks, rc = c - a * chunks;
          *reinterpret_cast<uint4*>(v + a * 16384 + (r0 + (rc >> 3)) * 128 + (rc & 7) * 16) = make_uint4(0, 0, 0, 0);
        }
        fence_proxy_async_smem();
        named_bar_sync(1, 256);
      }
    }
    // S = Q K^T
    wgmma_fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < D / 16; ++k) {
      const uint32_t off = (k >> 2) * 16384 + (k & 3) * 32;
      Wgmma<ATT_BN, 0, 0>::mma(s, make_wgmma_desc_sw128(aQ + off, 0, 1024), make_wgmma_desc_sw128(aK + off, 0, 1024),
                               k != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    // x = s*scale_log2 + slope2*(kpos - qpos); the causal mask only matters on the diagonal block
    // (PAGED: query blocks start at start[r], off the key grid; a block holds keys past some query iff its last key
    // lies past the CTA's first query)
    const bool diag = PAGED ? (j * ATT_BN + ATT_BN - 1 > p_first) : (j == qb);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const float bias0 = slope2 * static_cast<float>(j * ATT_BN - qpos[hh]);
      const int lim = qpos[hh] - j * ATT_BN;  // column c is visible iff c <= lim
      const int lo = seg[hh] - j * ATT_BN;    // ... and (SEG) c >= lo
      float mx = -INFINITY;
#pragma unroll
      for (int jn = 0; jn < ATT_BN / 8; ++jn) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * jn + 2 * t4 + e;
          float x = fmaf(s[4 * jn + 2 * hh + e], args.scale_log2, fmaf(slope2, static_cast<float>(col), bias0));
          if (diag && col > lim) x = -INFINITY;
          if (SEG && col < lo) x = -INFINITY;
          s[4 * jn + 2 * hh + e] = x;
          mx = fmaxf(mx, x);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[hh], mx);
      // SEG: a row whose document starts after this block has seen nothing yet (m_new = -inf); subtracting 0 keeps
      // alpha and p at exp2(-inf) = 0 instead of exp2(-inf - -inf) = NaN
      const float m_sub = (SEG && m_new == -INFINITY) ? 0.f : m_new;
      const float alpha = fast_exp2(m_run[hh] - m_sub);  // m_run = -inf on the first block -> 0
      float rs = 0.f;
#pragma unroll
      for (int jn = 0; jn < ATT_BN / 8; ++jn) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float p = fast_exp2(s[4 * jn + 2 * hh + e] - m_sub);
          s[4 * jn + 2 * hh + e] = p;
          rs += p;
        }
      }
      l_run[hh] = l_run[hh] * alpha + rs;  // per-thread partial over its columns; the quad is summed at the end
      m_run[hh] = m_new;
#pragma unroll
      for (int jn = 0; jn < D / 8; ++jn) {
        o[4 * jn + 2 * hh] *= alpha;
        o[4 * jn + 2 * hh + 1] *= alpha;
      }
    }
    // O += P V   (P from registers, packed before the fence so that no wgmma waits on a register write; V MN-major:
    // D/64 atoms of [128 keys x 64] 16 KB apart)
    uint32_t pa[ATT_BN / 16][4];
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk) acc_to_a(s, kk, pa[kk]);
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk)
      WgmmaRS<D, 1>::mma(o, pa[kk], make_wgmma_desc_sw128(aV + kk * 2048, 16384, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    if (tid_wg == 0) mbar_arrive(&kv_empty[stage]);
    if (++stage == ST) {
      stage = 0;
      phase ^= 1;
    }
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float l = l_run[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv_l = 1.f / l;
    if constexpr (PAGED) {
      if (qrow[hh] < n_new) {
        __nv_bfloat16* orow = args.out + static_cast<size_t>(row0 - qb * ATT_BM + qrow[hh]) * args.ld_out + head * args.d_out;
#pragma unroll
        for (int jn = 0; jn < D / 8; ++jn)
          if (8 * jn < args.d_out)
            *reinterpret_cast<uint32_t*>(orow + 8 * jn + 2 * t4) =
                pack_bf16x2(o[4 * jn + 2 * hh] * inv_l, o[4 * jn + 2 * hh + 1] * inv_l);
      }
    } else if (qpos[hh] < args.S) {
      __nv_bfloat16* orow = args.out + static_cast<size_t>(batch * args.S + qpos[hh]) * args.ld_out + head * D;
#pragma unroll
      for (int jn = 0; jn < D / 8; ++jn)
        *reinterpret_cast<uint32_t*>(orow + 8 * jn + 2 * t4) =
            pack_bf16x2(o[4 * jn + 2 * hh] * inv_l, o[4 * jn + 2 * hh + 1] * inv_l);
      if (t4 == 0)
        args.lse[(static_cast<size_t>(batch) * args.H + head) * args.S + qpos[hh]] =
            (m_run[hh] + log2f(l)) * 0.6931471805599453f;
    }
  }
}

// -----------------------------------------------------------------------------------------------
// backward
// -----------------------------------------------------------------------------------------------
// Per-query statistics of the backward loop: stats[b,h,i] = (lse[b,h,i] * log2e, -delta[b,h,i] * scale) with
// delta = sum_d dO[i,d] * O[i,d], rows of S_pad (S rounded up to 64) pairs so that the kernel loads a query block's
// 512 bytes with one bulk copy (pairs past S are never written; the kernel does not use them).  The same pass zeroes
// the row's fp32 dQ accumulator.  One warp per token row: every lane loads 16-byte chunks of the [H*D] row (fully
// coalesced), the D/8 lanes that share a head reduce with shuffles.
__global__ void __launch_bounds__(256) attention_bwd_prep_kernel(const __nv_bfloat16* __restrict__ dout,
                                                                 const __nv_bfloat16* __restrict__ out,
                                                                 const float* __restrict__ lse, float2* __restrict__ stats,
                                                                 float* __restrict__ dq_acc, int B, int S, int S_pad,
                                                                 int H, int D, float scale) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= B * S) return;
  const int cph = D / 8;                 // 16-byte chunks (= lanes) per head: 8 or 16
  const int nchunks = H * cph;
  const __nv_bfloat16* a = dout + static_cast<size_t>(row) * H * D;
  const __nv_bfloat16* b = out + static_cast<size_t>(row) * H * D;
  float4* dq_row = reinterpret_cast<float4*>(dq_acc + static_cast<size_t>(row) * H * D);
  for (int c = lane; c < H * D / 4; c += 32) dq_row[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int bidx = row / S, spos = row % S;
  for (int c0 = 0; c0 < nchunks; c0 += 32) {
    const int c = c0 + lane;
    float s = 0.f;
    if (c < nchunks) {
      const uint4 x = ld_global_nc_v4(a + c * 8), y = ld_global_nc_v4(b + c * 8);
      const uint32_t xw[4] = {x.x, x.y, x.z, x.w}, yw[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(xw[j]), g = unpack_bf16x2(yw[j]);
        s += f.x * g.x + f.y * g.y;
      }
    }
    for (int o = cph >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (c < nchunks && (lane & (cph - 1)) == 0) {
      const int head = c / cph;
      const size_t bh = static_cast<size_t>(bidx) * H + head;
      stats[bh * S_pad + spos] = make_float2(lse[bh * S + spos] * kLog2e, -s * scale);
    }
  }
}

template <int D>
struct AttBwdCfg {
  static constexpr int kKVBytes = ATT_BN * D * 2;     // K or V tile: D/64 atoms of [128 keys x 128 B]
  static constexpr int kQBytes = ATT_BWD_BM * D * 2;  // Q or dO tile: D/64 atoms of [64 queries x 128 B]
  static constexpr int kQStages = 2;
  static constexpr int kdSBytes = ATT_BN * ATT_BWD_BM * 2;  // dS^T [128 keys x 64 queries], one swizzled atom
  static constexpr int kdQCols = D / 2;                     // dQ columns per consumer warpgroup
  static constexpr int kdQBytes = ATT_BWD_BM * kdQCols * 4;  // fp32 [64 queries x D/2]: D/64 boxes of [64 x 32]
  static constexpr int kStatBytes = ATT_BWD_BM * 8;         // (lse2, nds) of a query block
  static constexpr int kSegBytes = ATT_BWD_BM * 4;          // seg_start of a query block (SEG)
  // K, V; Q, dO, the statistics and seg_start per stage; dS^T and the dQ tiles double-buffered (step it uses buffer
  // it & 1)
  static constexpr int kSmemBytes = 2 * kKVBytes + kQStages * (2 * kQBytes + kStatBytes + kSegBytes) + 2 * kdSBytes +
                                    2 * 2 * kdQBytes + 256 + 1024 /*align*/;
  static_assert(kSmemBytes <= 227 * 1024, "attention backward: shared memory");
};

struct AttBwdArgs {
  const float2* stats;      // [B, H, S_pad] (lse * log2e, -delta * scale), see attention_bwd_prep_kernel
  const float* slopes;
  __nv_bfloat16* dqkv;      // [B*S, H*3*D]
  int B, S, H, S_pad;
  float scale, scale_log2;
  const int* seg_start;     // [B*S] document start of every token (SEG only)
};

// tm_dq: fp32 map over the zeroed dQ accumulator [B, S, H*D] with [64 x 32] boxes; a box's rows past S are clipped,
// so no query of the next sequence is touched.
template <int D, bool SEG>
__global__ void __launch_bounds__(kAttThreads, 1)
    attention_bwd_kernel(const __grid_constant__ CUtensorMap tm_kv, const __grid_constant__ CUtensorMap tm_q,
                         const __grid_constant__ CUtensorMap tm_do, const __grid_constant__ CUtensorMap tm_dq,
                         const AttBwdArgs args) {
  using Cfg = AttBwdCfg<D>;
  constexpr int QS = Cfg::kQStages;
  constexpr int DQN = Cfg::kdQCols;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sK = smem;
  uint8_t* sV = sK + Cfg::kKVBytes;
  uint8_t* sQ = sV + Cfg::kKVBytes;
  uint8_t* sdO = sQ + QS * Cfg::kQBytes;
  uint8_t* sdS = sdO + QS * Cfg::kQBytes;  // [2][kdSBytes]
  uint8_t* sdQ = sdS + 2 * Cfg::kdSBytes;  // [2 buffers][2 warpgroups][kdQBytes]
  float2* sStat = reinterpret_cast<float2*>(sdQ + 4 * Cfg::kdQBytes);  // [QS][64]
  int* sSeg = reinterpret_cast<int*>(sStat + QS * ATT_BWD_BM);         // [QS][64] (SEG)
  uint64_t* bars = reinterpret_cast<uint64_t*>(sSeg + QS * ATT_BWD_BM);
  uint64_t* kv_full = bars;         // 1
  uint64_t* q_full = bars + 1;      // QS
  uint64_t* q_empty = q_full + QS;  // QS

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) pdl_launch_dependents();
  const int num_qb = (args.S + ATT_BWD_BM - 1) / ATT_BWD_BM;
  const int jb = blockIdx.x;  // key block
  const int head = blockIdx.y, batch = blockIdx.z;
  const int qb0 = jb * (ATT_BN / ATT_BWD_BM);  // first query block that sees these keys
  int n_iter = num_qb - qb0;
  const int col_q = head * 3 * D, col_k = col_q + D, col_v = col_q + 2 * D;
  const int krow0 = batch * args.S + jb * ATT_BN;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tm_kv);
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_do);
    tma_prefetch_desc(&tm_dq);
    mbar_init(kv_full, 1);
    for (int i = 0; i < QS; ++i) {
      mbar_init(&q_full[i], 1);
      mbar_init(&q_empty[i], 2);  // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // prologue above overlapped the predecessor; Q/K/V, dO, the statistics and the zeroed dQ are used below
  if constexpr (SEG) {
    // the last query that sees a key of this block ends the document holding its last key: the first q > k_last with
    // seg_start[q] > k_last, found by binary search over the row's non-decreasing seg_start.  Every thread computes the
    // same count, so the producer and the consumers agree on it.
    const int* seg_row = args.seg_start + static_cast<size_t>(batch) * args.S;
    const int k_last = min(jb * ATT_BN + ATT_BN - 1, args.S - 1);
    int lo = k_last + 1, hi = args.S;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (seg_row[mid] > k_last) hi = mid;
      else lo = mid + 1;
    }
    n_iter = (lo + ATT_BWD_BM - 1) / ATT_BWD_BM - qb0;
  }

  if (warp < 4) {
    setmaxnreg_dec<kAttRegsLight>();
    if (warp == 0) {
      // ===================== TMA producer =====================
      if (lane == 0) {
        mbar_arrive_expect_tx(kv_full, 2 * Cfg::kKVBytes);
#pragma unroll
        for (int a = 0; a < D / 64; ++a) {
          tma_load_2d(sK + a * 16384, &tm_kv, kv_full, col_k + a * 64, krow0);
          tma_load_2d(sV + a * 16384, &tm_kv, kv_full, col_v + a * 64, krow0);
        }
      }
      const float2* stat_row = args.stats + (static_cast<size_t>(batch) * args.H + head) * args.S_pad;
      int stage = 0;
      uint32_t phase = 0;
      for (int it = 0; it < n_iter; ++it) {
        const int qrow = batch * args.S + (qb0 + it) * ATT_BWD_BM;
        mbar_wait(&q_empty[stage], phase ^ 1);
        if constexpr (SEG) {
          // the block's document starts (0 past S), published to the consumers by lane 0's arrive on q_full
          const int q0 = (qb0 + it) * ATT_BWD_BM;
          for (int i = lane; i < ATT_BWD_BM; i += 32)
            st_shared_s32(smem_u32(sSeg + stage * ATT_BWD_BM + i), q0 + i < args.S ? args.seg_start[qrow + i] : 0);
          __syncwarp();
        }
        if (lane == 0) {
          mbar_arrive_expect_tx(&q_full[stage], 2 * Cfg::kQBytes + Cfg::kStatBytes);
#pragma unroll
          for (int a = 0; a < D / 64; ++a) {
            tma_load_2d(sQ + stage * Cfg::kQBytes + a * 8192, &tm_q, &q_full[stage], col_q + a * 64, qrow);
            tma_load_2d(sdO + stage * Cfg::kQBytes + a * 8192, &tm_do, &q_full[stage], head * D + a * 64, qrow);
          }
          bulk_load_1d(sStat + stage * ATT_BWD_BM, stat_row + (qb0 + it) * ATT_BWD_BM, Cfg::kStatBytes, &q_full[stage]);
        }
        __syncwarp();
        if (++stage == QS) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }
  setmaxnreg_inc<kAttRegsConsumer>();
  // ===================== consumers: warpgroup wg owns keys [64 wg, 64 wg + 64) of the block =====================
  const int wg = (warp >> 2) - 1, wl = warp & 3;
  const int tid_wg = threadIdx.x & 127;
  const int t4 = lane & 3;
  int kr[2], kpos[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    kr[hh] = 64 * wg + 16 * wl + (lane >> 2) + 8 * hh;  // key row inside the block
    kpos[hh] = jb * ATT_BN + kr[hh];
  }
  const float slope2 = args.slopes[head] * kLog2e;
  const uint32_t aK = smem_u32(sK) + wg * 8192, aV = smem_u32(sV) + wg * 8192;
  // dQ: this warpgroup's output columns [DQN wg, DQN wg + DQN) of K (MN-major: D/64 atoms 16 KB apart, 2 bytes a column)
  const uint32_t aKdq = smem_u32(sK) + (wg * DQN / 64) * 16384 + (wg * DQN % 64) * 2;
  const uint32_t adS0 = smem_u32(sdS), aTile0 = smem_u32(sdQ + wg * Cfg::kdQBytes);
  const uint32_t aStat0 = smem_u32(sStat) + t4 * 16, aSeg0 = smem_u32(sSeg) + t4 * 8;
  float dv[D / 2], dk[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) {
    dv[i] = 0.f;
    dk[i] = 0.f;
  }
  mbar_wait(kv_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int it = 0; it < n_iter; ++it) {
    const int qb = qb0 + it;
    mbar_wait(&q_full[stage], phase);
    const uint32_t aQ = smem_u32(sQ + stage * Cfg::kQBytes), adO = smem_u32(sdO + stage * Cfg::kQBytes);
    float st[ATT_BWD_BM / 2], dpt[ATT_BWD_BM / 2];
    // S^T = K Q^T, dP^T = V dO^T   (64 keys x 64 queries, contraction over D)
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < D / 16; ++k) {
      const uint32_t okv = (k >> 2) * 16384 + (k & 3) * 32, oq = (k >> 2) * 8192 + (k & 3) * 32;
      Wgmma<ATT_BWD_BM, 0, 0>::mma(st, make_wgmma_desc_sw128(aK + okv, 0, 1024), make_wgmma_desc_sw128(aQ + oq, 0, 1024),
                                   k != 0 ? 1u : 0u);
    }
#pragma unroll
    for (int k = 0; k < D / 16; ++k) {
      const uint32_t okv = (k >> 2) * 16384 + (k & 3) * 32, oq = (k >> 2) * 8192 + (k & 3) * 32;
      Wgmma<ATT_BWD_BM, 0, 0>::mma(dpt, make_wgmma_desc_sw128(aV + okv, 0, 1024), make_wgmma_desc_sw128(adO + oq, 0, 1024),
                                   k != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(st);
    wgmma_fence_regs(dpt);
    // p = exp2(s*scale_log2 + slope2*(kpos-qpos) - lse2); dS = p * (dP - delta) * scale.  Masked (key after query)
    // and out-of-sequence queries get p = 0.
    const uint32_t aStat = aStat0 + stage * Cfg::kStatBytes, aSeg = aSeg0 + stage * Cfg::kSegBytes;
#pragma unroll
    for (int jn = 0; jn < ATT_BWD_BM / 8; ++jn) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int qpos = qb * ATT_BWD_BM + 8 * jn + 2 * t4 + e;
        const bool q_ok = qpos < args.S;
        const float2 sv = ld_shared_v2_f32(aStat + jn * 64 + e * 8);  // (lse2, nds) of query qpos
        const float lse2 = q_ok ? sv.x : 0.f;
        const float nds = q_ok ? sv.y : 0.f;
        int seg_q = 0;
        if constexpr (SEG) seg_q = ld_shared_s32(aSeg + jn * 32 + e * 4);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int i = 4 * jn + 2 * hh + e;
          float p = fast_exp2(fmaf(st[i], args.scale_log2, fmaf(slope2, static_cast<float>(kpos[hh] - qpos), -lse2)));
          if (!q_ok || kpos[hh] > qpos) p = 0.f;
          if (SEG && kpos[hh] < seg_q) p = 0.f;
          st[i] = p;
          dpt[i] = p * fmaf(dpt[i], args.scale, nds);
        }
      }
    }
    // dS^T (bf16) -> shared memory, [128 keys x 64 queries] with the 128-byte swizzle, for the dQ product below
    const uint32_t adS = adS0 + (it & 1) * Cfg::kdSBytes;
#pragma unroll
    for (int jn = 0; jn < ATT_BWD_BM / 8; ++jn) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = kr[hh];
        const uint32_t off = r * 128 + ((jn ^ (r & 7)) << 4) + t4 * 4;
        st_shared_b32(adS + off, pack_bf16x2(dpt[4 * jn + 2 * hh], dpt[4 * jn + 2 * hh + 1]));
      }
    }
    // dV += P^T dO ; dK += dS^T Q   (contraction over the 64 queries; dO / Q MN-major: D/64 atoms 8 KB apart)
    uint32_t pa[ATT_BWD_BM / 16][4], dsa[ATT_BWD_BM / 16][4];  // packed before the fence (see the forward)
#pragma unroll
    for (int kk = 0; kk < ATT_BWD_BM / 16; ++kk) {
      acc_to_a(st, kk, pa[kk]);
      acc_to_a(dpt, kk, dsa[kk]);
    }
    wgmma_fence_regs(dv);
    wgmma_fence_regs(dk);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < ATT_BWD_BM / 16; ++kk)
      WgmmaRS<D, 1>::mma(dv, pa[kk], make_wgmma_desc_sw128(adO + kk * 2048, 8192, 1024), 1u);
#pragma unroll
    for (int kk = 0; kk < ATT_BWD_BM / 16; ++kk)
      WgmmaRS<D, 1>::mma(dk, dsa[kk], make_wgmma_desc_sw128(aQ + kk * 2048, 8192, 1024), 1u);
    wgmma_commit();
    fence_proxy_async_smem();  // dS^T writes -> async-proxy (wgmma) reads
    // this warpgroup's dQ tile buffer was last added by step it - 2: wait until that reduce has read it
    if (tid_wg == 0) tma_store_wait_read<1>();
    // both halves of dS^T are written (the other warpgroup last read this buffer in step it - 2, before it arrived
    // here in step it - 1), and the tile is free
    named_bar_sync(1, 256);
    // dQ[:, DQN wg .. + DQN] = dS K over all 128 keys.  A = dS (MN-major: queries contiguous in the dS^T rows),
    // B = K (MN-major: D contiguous)
    float dq[DQN / 2];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk)
      Wgmma<DQN, 1, 1>::mma(dq, make_wgmma_desc_sw128(adS + kk * 2048, 8192, 1024),
                            make_wgmma_desc_sw128(aKdq + kk * 2048, 16384, 1024), kk != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(dq);
    wgmma_fence_regs(dv);
    wgmma_fence_regs(dk);
    const uint32_t aTile = aTile0 + (it & 1) * 2 * Cfg::kdQBytes;
    // fp32 tile -> shared memory: D/64 boxes of [64 queries x 32 columns], 128-byte rows with the 128-byte swizzle
    // (16-byte chunk c of row r at c ^ (r & 7))
#pragma unroll
    for (int jn = 0; jn < DQN / 8; ++jn) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = 16 * wl + (lane >> 2) + 8 * hh;
        const int chunk = 2 * (jn & 3) + (t4 >> 1);
        const uint32_t off = (jn >> 2) * 8192 + r * 128 + ((chunk ^ (r & 7)) << 4) + (t4 & 1) * 8;
        st_shared_v2_f32(aTile + off, dq[4 * jn + 2 * hh], dq[4 * jn + 2 * hh + 1]);
      }
    }
    fence_proxy_async_smem();  // tile writes -> async-proxy (TMA) reads
    // every wgmma of this step has retired (the wait above covers the dV / dK group): Q / dO / the statistics are free
    named_bar_sync(2 + wg, 128);
    if (tid_wg == 0) {
#pragma unroll
      for (int b = 0; b < DQN / 32; ++b)
        tma_reduce_add_3d(&tm_dq, sdQ + ((it & 1) * 2 + wg) * Cfg::kdQBytes + b * 8192, head * D + wg * DQN + b * 32,
                          qb * ATT_BWD_BM, batch);
      tma_store_commit();
      mbar_arrive(&q_empty[stage]);
    }
    if (++stage == QS) {
      stage = 0;
      phase ^= 1;
    }
  }
  // dK, dV of this key block
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    if (kpos[hh] >= args.S) continue;
    __nv_bfloat16* dk_row = args.dqkv + static_cast<size_t>(batch * args.S + kpos[hh]) * (args.H * 3 * D) + col_k;
    __nv_bfloat16* dv_row = dk_row + D;
#pragma unroll
    for (int jn = 0; jn < D / 8; ++jn) {
      *reinterpret_cast<uint32_t*>(dk_row + 8 * jn + 2 * t4) = pack_bf16x2(dk[4 * jn + 2 * hh], dk[4 * jn + 2 * hh + 1]);
      *reinterpret_cast<uint32_t*>(dv_row + 8 * jn + 2 * t4) = pack_bf16x2(dv[4 * jn + 2 * hh], dv[4 * jn + 2 * hh + 1]);
    }
  }
  // the dQ sums are complete (and the tiles read) before the CTA exits, so the convert kernel that follows reads them
  if (tid_wg == 0) tma_store_wait<0>();
}

// dq fp32 [rows, H*D] -> bf16 into dqkv[rows, H*3*D] (q slot of every head)
__global__ void __launch_bounds__(256) attention_dq_convert_kernel(const float* __restrict__ dq,
                                                                   __nv_bfloat16* __restrict__ dqkv, int64_t rows,
                                                                   int H, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t idx = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  const int64_t total = rows * H * D;
  if (idx >= total) return;
  const int64_t row = idx / (H * D);
  const int rem = static_cast<int>(idx % (H * D));
  const int head = rem / D, d = rem % D;
  const float4 a = *reinterpret_cast<const float4*>(dq + idx);
  const float4 b = *reinterpret_cast<const float4*>(dq + idx + 4);
  st_global_v4(dqkv + row * (H * 3 * D) + head * 3 * D + d,
               make_uint4(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w), pack_bf16x2(b.x, b.y), pack_bf16x2(b.z, b.w)));
}

}  // namespace pg

using namespace pg;

static int att_tmap(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  struct Key {
    const void* p;
    uint64_t r, c;
    uint32_t b;
    bool operator==(const Key& o) const { return p == o.p && r == o.r && c == o.c && b == o.b; }
  };
  struct H {
    size_t operator()(const Key& k) const {
      return reinterpret_cast<size_t>(k.p) ^ (k.r * 1315423911u) ^ (k.c << 20) ^ (static_cast<size_t>(k.b) << 40);
    }
  };
  static std::unordered_map<Key, CUtensorMap, H> cache;
  static std::mutex mu;
  std::lock_guard<std::mutex> g(mu);
  Key key{ptr, rows, cols, box_rows};
  auto it = cache.find(key);
  if (it != cache.end()) {
    *out = it->second;
    return 0;
  }
  if (make_tmap_bf16_2d(out, ptr, rows, cols, cols, box_rows, 64) != 0) return -1;
  if (cache.size() > 4096) cache.clear();
  cache.emplace(key, *out);
  return 0;
}

#define PG_CHECK_LAUNCH(name)                                                       \
  do {                                                                              \
    cudaError_t e__ = cudaGetLastError();                                           \
    if (e__ != cudaSuccess) {                                                       \
      fprintf(stderr, "pipegoose_b200: %s launch failed: %s\n", name, cudaGetErrorString(e__)); \
      return -1;                                                                    \
    }                                                                               \
  } while (0)

template <int D, bool SEG>
static int launch_att_fwd(const CUtensorMap& tm, const AttFwdArgs& a, cudaStream_t s) {
  using Cfg = AttFwdCfg<D>;
  static bool set = false;
  if (!set) {
    if (cudaFuncSetAttribute(attention_fwd_kernel<D, SEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes) != cudaSuccess) return -1;
    set = true;
  }
  dim3 grid((a.S + ATT_BM - 1) / ATT_BM, a.H, a.B);
  // the pool maps are unused here: the qkv map fills their slots
  if (launch_pdl(attention_fwd_kernel<D, SEG>, grid, dim3(kAttThreads), Cfg::kSmemBytes, s, tm, a, tm, tm) != cudaSuccess)
    return -1;
  PG_CHECK_LAUNCH("attention_fwd");
  return 0;
}

// softmax_scale <= 0: 1/sqrt(D).  An explicit scale lets a head that was zero-padded to a supported width (e.g. D=80
// -> 128: the padded columns contribute nothing to Q.K) keep the scale of its true width.
// seg_start: int32 [B*S] row-relative document starts (packed sequences), nullptr: one document per row.
extern "C" int pg_attention_fwd(const void* qkv, const float* slopes, void* out, float* lse, int B, int S, int H,
                                int D, float softmax_scale, const int* seg_start, cudaStream_t s) {
  if (D != 64 && D != 128) return -1;
  CUtensorMap tm;
  if (att_tmap(&tm, qkv, static_cast<uint64_t>(B) * S, static_cast<uint64_t>(H) * 3 * D, ATT_BM) != 0) return -1;
  AttFwdArgs a;
  a.out = (__nv_bfloat16*)out;
  a.lse = lse;
  a.slopes = slopes;
  a.B = B; a.S = S; a.H = H;
  a.ld_out = H * D;
  a.scale_log2 = kLog2e * (softmax_scale > 0.f ? softmax_scale : 1.0f / sqrtf(static_cast<float>(D)));
  a.seg_start = seg_start;
  if (seg_start != nullptr) return D == 64 ? launch_att_fwd<64, true>(tm, a, s) : launch_att_fwd<128, true>(tm, a, s);
  return D == 64 ? launch_att_fwd<64, false>(tm, a, s) : launch_att_fwd<128, false>(tm, a, s);
}

template <int D>
static int launch_att_fwd_paged(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                                const AttFwdArgs& a, cudaStream_t s) {
  using Cfg = AttFwdCfg<D>;
  static bool set = false;
  if (!set) {
    if (cudaFuncSetAttribute(attention_fwd_kernel<D, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes) != cudaSuccess) return -1;
    set = true;
  }
  dim3 grid((a.S + ATT_BM - 1) / ATT_BM, a.H, a.B);
  if (launch_pdl(attention_fwd_kernel<D, false, true>, grid, dim3(kAttThreads), Cfg::kSmemBytes, s, tq, a, tk, tv) != cudaSuccess)
    return -1;
  PG_CHECK_LAUNCH("attention_fwd_paged");
  return 0;
}

// Paged prefill attention (PAGED, see the top of the file): qkv [N, H*3*D] holds the new tokens of R sequences
// (cu_seqlens int32 [R+1], start int32 [R], table int32 [R, max_pages], all on the device); out [N, H*D].  max_len >= the
// most new tokens of any sequence sizes the grid.  k_pool / v_pool [num_pages, H, 64, D] are read, never written.
// D = 80 runs on the D = 128 instantiation (pool maps of 80 columns: out-of-bounds columns read as zero).
extern "C" int pg_paged_prefill_attention(const void* qkv, const void* k_pool, const void* v_pool, const int* table,
                                          const int* cu_seqlens, const int* start, const float* slopes, void* out, int N,
                                          int R, int H, int D, int num_pages, int max_pages, int max_len,
                                          float softmax_scale, cudaStream_t s) {
  if (D != 64 && D != 80 && D != 128) return -1;
  if (N <= 0 || R <= 0 || max_len <= 0) return 0;
  const uint64_t pool_rows = static_cast<uint64_t>(num_pages) * H * 64;
  if (pool_rows >= (1ull << 31)) return -1;  // TMA row coordinates are int32
  CUtensorMap tq, tk, tv;
  if (att_tmap(&tq, qkv, static_cast<uint64_t>(N), static_cast<uint64_t>(H) * 3 * D, ATT_BM) != 0) return -1;
  if (att_tmap(&tk, k_pool, pool_rows, D, 64) != 0) return -1;
  if (att_tmap(&tv, v_pool, pool_rows, D, 64) != 0) return -1;
  AttFwdArgs a;
  memset(&a, 0, sizeof(a));
  a.out = (__nv_bfloat16*)out;
  a.slopes = slopes;
  a.B = R; a.S = max_len; a.H = H;
  a.ld_out = H * D;
  a.scale_log2 = kLog2e * (softmax_scale > 0.f ? softmax_scale : 1.0f / sqrtf(static_cast<float>(D)));
  a.cu_seqlens = cu_seqlens;
  a.start = start;
  a.table = table;
  a.max_pages = max_pages;
  a.H_pool = H;
  a.d_out = D;
  return D == 64 ? launch_att_fwd_paged<64>(tq, tk, tv, a, s) : launch_att_fwd_paged<128>(tq, tk, tv, a, s);
}

template <int D, bool SEG>
static int launch_att_bwd(const CUtensorMap& tkv, const CUtensorMap& tq, const CUtensorMap& tdo, const CUtensorMap& tdq,
                          const AttBwdArgs& a, cudaStream_t s) {
  using Cfg = AttBwdCfg<D>;
  static bool set = false;
  if (!set) {
    if (cudaFuncSetAttribute(attention_bwd_kernel<D, SEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes) != cudaSuccess) return -1;
    set = true;
  }
  // key block fastest: the CTAs of one (head, batch) run together and share its Q / dO / statistics reads and dQ
  // reduce-adds in L2 (with the key block slowest, longest first, the backward measured 12 % slower at D = 64 and
  // 61 % slower at D = 128 on an H100)
  dim3 grid((a.S + ATT_BN - 1) / ATT_BN, a.H, a.B);
  if (launch_pdl(attention_bwd_kernel<D, SEG>, grid, dim3(kAttThreads), Cfg::kSmemBytes, s, tkv, tq, tdo, tdq, a) != cudaSuccess)
    return -1;
  PG_CHECK_LAUNCH("attention_bwd");
  return 0;
}

// dq_acc: fp32 workspace [B*S, H*D] (any contents: the pre-kernel zeroes it); stats: fp32 workspace of
// pg_attention_bwd_stats_floats(B, S, H) floats
extern "C" int pg_attention_bwd(const void* qkv, const float* slopes, const void* out, const float* lse,
                                const void* dout, void* dqkv, float* dq_acc, float* stats, int B, int S, int H,
                                int D, float softmax_scale, const int* seg_start, cudaStream_t s) {
  if (D != 64 && D != 128) return -1;
  const int64_t rows = static_cast<int64_t>(B) * S;
  const int S_pad = (S + ATT_BWD_BM - 1) / ATT_BWD_BM * ATT_BWD_BM;
  CUtensorMap tkv, tq, tdo, tdq;
  if (att_tmap(&tkv, qkv, rows, static_cast<uint64_t>(H) * 3 * D, ATT_BN) != 0) return -1;
  if (att_tmap(&tq, qkv, rows, static_cast<uint64_t>(H) * 3 * D, ATT_BWD_BM) != 0) return -1;
  if (att_tmap(&tdo, dout, rows, static_cast<uint64_t>(H) * D, ATT_BWD_BM) != 0) return -1;
  if (make_tmap_f32_3d(&tdq, dq_acc, static_cast<uint64_t>(H) * D, S, B, ATT_BWD_BM) != 0) return -1;
  const float scale = softmax_scale > 0.f ? softmax_scale : 1.0f / sqrtf(static_cast<float>(D));
  if (launch_pdl(attention_bwd_prep_kernel, dim3((unsigned)((rows * 32 + 255) / 256)), dim3(256), 0, s,
                 (const __nv_bfloat16*)dout, (const __nv_bfloat16*)out, lse, reinterpret_cast<float2*>(stats), dq_acc, B,
                 S, S_pad, H, D, scale) != cudaSuccess)
    return -1;
  PG_CHECK_LAUNCH("attention_bwd_prep");
  AttBwdArgs a;
  a.stats = reinterpret_cast<const float2*>(stats);
  a.slopes = slopes;
  a.dqkv = (__nv_bfloat16*)dqkv;
  a.B = B; a.S = S; a.H = H; a.S_pad = S_pad;
  a.scale = scale;
  a.scale_log2 = a.scale * kLog2e;
  a.seg_start = seg_start;
  const int rc = seg_start != nullptr
                     ? (D == 64 ? launch_att_bwd<64, true>(tkv, tq, tdo, tdq, a, s) : launch_att_bwd<128, true>(tkv, tq, tdo, tdq, a, s))
                     : (D == 64 ? launch_att_bwd<64, false>(tkv, tq, tdo, tdq, a, s) : launch_att_bwd<128, false>(tkv, tq, tdo, tdq, a, s));
  if (rc != 0) return rc;
  const int64_t total = rows * H * D;
  if (launch_pdl(attention_dq_convert_kernel, dim3((unsigned)((total / 8 + 255) / 256)), dim3(256), 0, s, (const float*)dq_acc,
                 (__nv_bfloat16*)dqkv, (int64_t)rows, H, D) != cudaSuccess) return -1;
  PG_CHECK_LAUNCH("attention_dq_convert");
  return 0;
}

extern "C" int64_t pg_attention_bwd_stats_floats(int B, int S, int H) {
  return static_cast<int64_t>(B) * H * ((S + ATT_BWD_BM - 1) / ATT_BWD_BM * ATT_BWD_BM) * 2;
}
