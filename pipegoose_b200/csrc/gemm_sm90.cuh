// Persistent, warp-specialised bf16 GEMM for sm_90a:
//   TMA (cp.async.bulk.tensor) -> 128B-swizzled smem ring -> wgmma.mma_async issued by two
//   consumer warpgroups (64 rows of the 128-row tile each, fp32 accumulators in registers) ->
//   epilogue by the same warpgroups: for bf16 and plain fp32 outputs in the accumulator-fragment layout with TMA
//   stores / reduce-adds (epilogue_tma, epilogue_tma_f32), otherwise accumulators handed over through shared memory
//   (the general epilogue).
//
// One kernel serves the three operand layouts a transformer training step needs
//   NT : Y  = X  · Wᵀ   (A K-major,  B K-major)    forward
//   NN : dX = dY · W    (A K-major,  B MN-major)   dgrad
//   TN : dW = dYᵀ · X   (A MN-major, B MN-major)   wgrad
// and the fused compute+collective forms used by tensor parallelism
//   all-gather -> GEMM : M is split into `num_chunks` row chunks that become readable
//                        at different times (a comm CTA group or a peer publishes a
//                        flag per chunk); tiles are visited chunk by chunk, starting at
//                        the local chunk, and the TMA producer acquires the chunk flag.
//   GEMM -> reduce-scatter : the epilogue stores each tile straight into the owner
//                        rank's staging slot through its NVLink peer mapping and bumps a
//                        per-owner arrival counter with a system-scope release.
// The epilogue applies bias / tanh-GELU (also emitting the pre-activation) /
// GELU-backward / residual add / fp32 accumulate, so none of those is a separate pass.
// FP8 operands (FMT, the FP8 linear layers): NT only, TMA epilogue only, per-tensor scales applied in the epilogue.
#pragma once
#include "grad_rs.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace pg {

constexpr int kMaxPeers = 8;

enum EpiFlags : int {
  EPI_BIAS = 1,        // acc += bias[col]
  EPI_GELU = 2,        // out = gelu_tanh(acc); if aux_out != null, aux_out = acc (pre-activation)
  EPI_RESIDUAL = 4,    // out = acc + residual[row, col]
  EPI_OUT_F32 = 8,     // out is fp32
  EPI_ACCUM = 16,      // out += acc (fp32 out only)
  EPI_DGELU = 32,      // out = acc * gelu_tanh'(aux_in[row, col])
  EPI_SCATTER = 64,    // MoE combine: out row -> out_peer[src][row_ret[row]], scaled by row_scale[row]
  EPI_ATOMIC = 128,    // fp32 out += acc with red.global.add (split-K partial sums)
  EPI_BGRAD = 256,     // bias_grad[m] += sum_k A[k, m] (wgrad: the bias gradient from the dY operand, A MN-major)
};
// (GemmArgs::ce_part != null) lm_head: besides the bf16 logits the epilogue emits, per row and per half tile, the online
// softmax partials (max, sum exp(x - max)) of the logits it holds in registers — the cross entropy never re-reads the
// [tokens, vocab] logits for its statistics (csrc/elementwise.cu: ce_combine merges the partials)

struct GemmArgs {
  int M, N, K;
  int k_splits;  // >1: the K loop is split over k_splits work items per tile (partial sums added: EPI_ATOMIC)
  void* out;
  int ldc;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* residual;
  int ldr;
  void* aux;  // EPI_GELU: pre-activation output; EPI_DGELU: pre-activation input (bf16, ld = ldc)
  int flags;
  // ---- chunked traversal (fused collectives); num_chunks == 1 for a plain GEMM
  int num_chunks;
  int chunk_rows;   // rows per chunk (multiple of 128 when num_chunks > 1)
  int first_chunk;  // chunk visited first (the local one)
  // all-gather -> GEMM: chunk c is readable once chunk_flags[c] >= flag_value
  const uint32_t* chunk_flags;
  uint32_t flag_value;
  // comm CTAs (blockIdx.x < n_comm) pull every rank's shard into the local gathered A matrix with
  // bulk async copies (peer global -> smem -> local global) and publish chunk_flags (+1 per CTA)
  int n_comm;
  const void* ag_src[kMaxPeers];     // rank r's shard (NVLink peer mapping; ag_src[my_rank] is local)
  void* ag_dst;                      // local gathered matrix [num_chunks * chunk_rows, K]
  uint64_t ag_chunk_bytes;           // bytes of one shard
  uint32_t* ag_peer_flag[kMaxPeers]; // &peer_r.shard_ready[my_rank]: tell rank r that my shard is readable
  const uint32_t* ag_ready;          // local shard_ready[src] (written by src), wait >= ag_epoch
  uint32_t ag_epoch;
  int my_rank;
  int a_local_chunk;  // >= 0: tiles of this chunk load A through tma_a_local (rows relative to the chunk)
  // grouped GEMM (one chunk per expert): B / bias of chunk c start b_chunk_rows*c rows / bias_chunk_stride*c
  // elements further (stacked expert weights)
  int b_chunk_rows;
  int bias_chunk_stride;
  // EPI_SCATTER: row r (inside its chunk) came from rank r / scatter_rows_per_src; it returns to row
  // row_ret[r] of that rank's buffer out_peer[rank] (row_ret < 0: empty slot), scaled by row_scale[r]
  const int* row_ret;
  const float* row_scale;
  int scatter_rows_per_src;
  // GEMM -> reduce-scatter: rows of chunk c go to out_peer[c] (row index relative to chunk),
  // then arrive_ctr[c] (+1 per finished tile, release.sys)
  void* out_peer[kMaxPeers];
  uint32_t* arrive_ctr[kMaxPeers];
  // fused reduction of the LOCAL chunk (visited last): once every peer's arrival counter reached rs_wait_value,
  // the epilogue of this rank's own tiles adds the peers' staged partial tiles (+ bias + residual) and writes the
  // final rows to `out`; no separate reduce kernel, the own partial never goes through memory
  const __nv_bfloat16* rs_in[kMaxPeers];  // local staging slot of source s (rs_in[my_rank] unused); null = off
  const uint32_t* rs_wait_ctr;            // local arrival counters, one per source
  uint32_t rs_wait_value;
  float* ce_part;  // [M, 2 * n_blks, 2] fp32 (max, sumexp) partials; slot 2 * n_blk + half (null: off)
  int ce_valid;    // logits columns >= ce_valid are vocabulary padding: excluded from the statistics
  // wgrad -> data-parallel reduce-scatter (fp32 outputs): every 16-byte group of the tile is added into the gradient
  // buffer of the rank that owns its ZeRO-1 slice (local L2 atomics / NVLink peer atomics); grad_rs.world <= 1: off
  PgGradRS grad_rs;
  float* bias_grad;  // EPI_BGRAD: fp32 [M]
  // FP8 operands (FMT != FMT_BF16): value = code * scale_inv, one fp32 device scalar per operand; the epilogue multiplies
  // every accumulator by a_scale_inv * b_scale_inv before anything else
  const float* a_scale_inv;
  const float* b_scale_inv;
};

// Operand formats of the kernel.  FP8 (A e4m3 or e5m2, B e4m3) is K-major only and runs the TMA epilogue only: a
// k-block is 128 codes, i.e. the same 128-byte swizzled rows, stage sizes and descriptors as a 64-wide bf16 k-block.
enum GemmFmt : int { FMT_BF16 = 0, FMT_E4M3 = 1, FMT_E5M2 = 2 };

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int WG_K = 16;           // K of one wgmma instruction
constexpr int kGemmThreads = 384;  // warpgroup 0: warp 0 TMA, warp 1 epilogue-operand TMA; warpgroups 1, 2: wgmma + epilogue
constexpr int kAccLd = 68;         // fp32 accumulator hand-over rows: 64 columns + 4 of padding (bank spread)

// Shared-memory budget.  TMA_EPI = false (general epilogue): the per-warp staging buffers and the fp32 accumulator
// hand-over.  TMA_EPI = true (TMA-store epilogue): the whole 128 x BN bf16 output tile as [64 x 64] 128B-swizzled
// slots (slot 2-D index: warpgroup, 64-column group) plus the tile's bias slice; the slots first receive the
// tile's residual / GELU' input and are then overwritten in place by the output.  The stage count is what is left:
// 3 at BN = 256 and 4 at BN = 192 (as for the general epilogue), 6 at BN = 128, 8 at BN = 64.
template <int BN, bool TMA_EPI = false>
struct GemmCfg {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiStageBytes = TMA_EPI ? 0 : 8 * 32 * 64;  // 8 epilogue warps x [32 rows x 64 B]
  static constexpr int kAccStageBytes = TMA_EPI ? 0 : 2 * 64 * kAccLd * 4;  // per consumer warpgroup: [64 x 64] fp32
  static constexpr int kSlotBytes = 64 * 64 * 2;
  static constexpr int kSlots = TMA_EPI ? 2 * (BN / 64) : 0;
  static constexpr int kBiasBytes = TMA_EPI ? BN * 2 : 0;
  static constexpr int kFixedBytes =
      kEpiStageBytes + kAccStageBytes + kSlots * kSlotBytes + kBiasBytes + 1024 /*align*/ + 256 /*barriers*/;
  static constexpr int kMaxStages = (227 * 1024 - kFixedBytes) / kStageBytes;  // 227 KB: sm_90 opt-in maximum
  static constexpr int kStages = kMaxStages > 8 ? 8 : kMaxStages;
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
};

PG_DEVICE float gelu_tanh(float x) {
  // Bloom's GELU: x * 0.5 * (1 + tanh(0.79788456 x (1 + 0.044715 x^2)))
  float u = 0.79788456f * x * (1.0f + 0.044715f * x * x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  return 0.5f * x * (1.0f + t);
}
PG_DEVICE float gelu_tanh_grad(float x) {
  float u = 0.79788456f * x * (1.0f + 0.044715f * x * x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  return 0.5f * x * ((1.0f - t * t) * (0.79788456f + 0.1070322243f * x * x)) + 0.5f * (1.0f + t);
}

struct TileCoord {
  int m_blk, n_blk, chunk;
};

// Tiles are enumerated chunk-major (chunk order rotated to start at first_chunk); inside a
// chunk, groups of 8 row-blocks sweep all column-blocks so that concurrently resident CTAs
// share A and B tiles through L2.
PG_DEVICE TileCoord map_tile(int t, int m_blks_per_chunk, int n_blks, int num_chunks,
                             int first_chunk) {
  const int per_chunk = m_blks_per_chunk * n_blks;
  const int ci = t / per_chunk;
  int r = t - ci * per_chunk;
  int chunk = first_chunk + ci;
  if (chunk >= num_chunks) chunk -= num_chunks;
  constexpr int G = 8;
  const int per_group = G * n_blks;
  const int g = r / per_group;
  const int first_m = g * G;
  const int gsz = min(m_blks_per_chunk - first_m, G);
  r -= g * per_group;
  TileCoord c;
  c.n_blk = r / gsz;
  c.m_blk = chunk * m_blks_per_chunk + first_m + (r - c.n_blk * gsz);
  c.chunk = chunk;
  return c;
}

// The bf16 matrix the epilogue reads element-wise (GELU' pre-activation or residual; the same choice in both
// epilogues), null: none.
PG_DEVICE const void* epi_input(const GemmArgs& a) {
  return (a.flags & EPI_DGELU) ? a.aux : (a.flags & EPI_RESIDUAL) ? static_cast<const void*>(a.residual) : nullptr;
}

// TMA-store epilogue of one tile for consumer warpgroup wg (tile rows [64 wg, 64 wg + 64)), bf16 output, one chunk.
// Bias, cross-entropy partials, GELU (+ pre-activation), GELU' and residual are applied in fp32 on the accumulator
// fragments with the general epilogue's arithmetic, in its order, so the bf16 results are the same bits.  The
// bias slice and the residual / GELU' input were loaded into shared memory by the producer warpgroup under the main
// loop (epi_full).  The bf16 results are written in place into the warpgroup's 128B-swizzled [64 x 64] slots and
// leave with TMA stores (clipped at the M / N edges) that nobody waits for here: the storing thread waits for
// them to have READ the slots during the next tile's first k-block, or at kernel exit.
//
// Fragment element acc[4 j + 2 hh + e] is row 16 wl + lane / 4 + 8 hh, column 8 j + 2 (lane % 4) + e of the
// warpgroup's 64 x BN block (wgmma.cuh); the pair (e = 0, 1) is one 4-byte word of slot j / 8, whose 16-byte chunk
// j % 8 of row r sits at chunk (j % 8) ^ (r % 8) (r % 8 = lane / 4): the 32 lanes of a warp hit 32 different banks.
template <int BN>
PG_DEVICE void epilogue_tma(float (&acc)[BN / 2], const GemmArgs& args, const CUtensorMap* tma_out,
                            const CUtensorMap* tma_aux, uint8_t* wslots, const uint8_t* bias_s, uint64_t* epi_full,
                            uint32_t epi_parity, bool has_in, int m_blk, int n_blk, int n_blks, int wg, int tid_wg) {
  constexpr int kSlotBytes = 64 * 64 * 2;
  const int lane = tid_wg & 31;
  const int wl = tid_wg >> 5;
  const int quad = lane & 3;
  const int m0 = m_blk * BM + 64 * wg;
  const int n0 = n_blk * BN;
  uint8_t* my_row = wslots + (16 * wl + (lane >> 2)) * 128 + quad * 4;
  auto word = [&](int j, int hh) -> uint32_t* {
    return reinterpret_cast<uint32_t*>(my_row + (j >> 3) * kSlotBytes + hh * (8 * 128) + (((j & 7) ^ (lane >> 2)) << 4));
  };
  auto store_tile = [&](const CUtensorMap* map) {
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) *word(j, hh) = pack_bf16x2(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]);
    fence_proxy_async_smem();
    named_bar_sync(2 + wg, 128);
    if (tid_wg == 0) {
#pragma unroll
      for (int s = 0; s < BN / 64; ++s) tma_store_2d(map, wslots + s * kSlotBytes, n0 + 64 * s, m0);
      tma_store_commit();
    }
  };

  if (has_in) {
    mbar_wait(epi_full, epi_parity);
  } else {
    named_bar_sync(2 + wg, 128);  // the storing thread saw the previous tile's stores read the slots
  }
  if (args.flags & EPI_BIAS) {
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(bias_s + (8 * j + 2 * quad) * 2));
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        acc[4 * j + 2 * hh] += b.x;
        acc[4 * j + 2 * hh + 1] += b.y;
      }
    }
  }
  if (args.ce_part != nullptr) {
    // statistics of the values as they are STORED (rounded to bf16); per row and tile half [BN/2 h, BN/2 (h + 1)):
    // each thread of a quad holds a quarter of the row's columns, the quad merges them with shuffles
    const int lim = min(args.N, args.ce_valid) - n0;  // columns [0, lim) of the tile enter the statistics
    float mx[2][2], sm[2][2];                         // [hh][half]
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        mx[hh][hf] = -INFINITY;
        sm[hh][hf] = 0.f;
      }
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = acc[4 * j + 2 * hh + e];
          v = __bfloat162float(__float2bfloat16_rn(v));
          if (8 * j + 2 * quad + e < lim) mx[hh][j >= BN / 16] = fmaxf(mx[hh][j >= BN / 16], v);
        }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        mx[hh][hf] = fmaxf(mx[hh][hf], __shfl_xor_sync(0xffffffffu, mx[hh][hf], 1));
        mx[hh][hf] = fmaxf(mx[hh][hf], __shfl_xor_sync(0xffffffffu, mx[hh][hf], 2));
      }
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * j + 2 * quad + e < lim)
            sm[hh][j >= BN / 16] += exp2f((acc[4 * j + 2 * hh + e] - mx[hh][j >= BN / 16]) * 1.4426950408889634f);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        sm[hh][hf] += __shfl_xor_sync(0xffffffffu, sm[hh][hf], 1);
        sm[hh][hf] += __shfl_xor_sync(0xffffffffu, sm[hh][hf], 2);
      }
    // lane 4 i + hh writes row 16 wl + i + 8 hh: both halves of the tile, slots 2 n_blk and 2 n_blk + 1
    const int row = m0 + 16 * wl + (lane >> 2) + 8 * quad;
    if (quad < 2 && row < args.M) {
      const float4 v = quad == 0 ? make_float4(mx[0][0], sm[0][0], mx[0][1], sm[0][1])
                                 : make_float4(mx[1][0], sm[1][0], mx[1][1], sm[1][1]);
      *reinterpret_cast<float4*>(args.ce_part + (static_cast<size_t>(row) * n_blks + n_blk) * 4) = v;
    }
  }
  if (args.flags & EPI_GELU) {
    if (args.aux != nullptr) store_tile(tma_aux);  // the pre-activation
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = gelu_tanh(acc[i]);
    if (args.aux != nullptr) {
      if (tid_wg == 0) tma_store_wait_read<0>();
      named_bar_sync(2 + wg, 128);
    }
  }
  if (epi_input(args) != nullptr) {
    const bool dgelu = (args.flags & EPI_DGELU) != 0;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const float2 z = unpack_bf16x2(*word(j, hh));
        if (dgelu) {
          acc[4 * j + 2 * hh] *= gelu_tanh_grad(z.x);
          acc[4 * j + 2 * hh + 1] *= gelu_tanh_grad(z.y);
        } else {
          acc[4 * j + 2 * hh] += z.x;
          acc[4 * j + 2 * hh + 1] += z.y;
        }
      }
  }
  store_tile(tma_out);
}

// TMA epilogue of one tile for consumer warpgroup wg, plain fp32 output (wgrad into a main grad).  The warpgroup's
// BN / 64 slots of 8 KB hold [64 rows x 32] fp32 each (one 128-byte row per tile row, 128B-swizzled), so its
// 64 x BN block leaves in two rounds of BN / 2 columns; the second round reuses the slots once the first round's
// transfers have read them.  With EPI_ACCUM (accumulate, or a split-K partial) the slots are added to the output
// with TMA reduce-adds, else stored.  Both are clipped at the M / N edges.
//
// Fragment pair acc[4 j + 2 hh + (0, 1)] (row r = 16 wl + lane / 4 + 8 hh, columns 8 j + 2 quad + (0, 1)) is 8 bytes
// of 16-byte chunk 2 (j % 4) + quad / 2 of row r in slot (j % (BN / 16)) / 4 of round j / (BN / 16), stored at chunk
// position chunk ^ (r % 8): a warp's 256 bytes cover every bank twice (the minimum for 8-byte stores).
template <int BN>
PG_DEVICE void epilogue_tma_f32(const float (&acc)[BN / 2], const GemmArgs& args, const CUtensorMap* tma_out,
                                uint8_t* wslots, int m_blk, int n_blk, int wg, int tid_wg) {
  constexpr int kSlotBytes = 64 * 32 * 4;
  constexpr int JR = BN / 16;  // fragment column groups per round
  const int lane = tid_wg & 31;
  const int wl = tid_wg >> 5;
  const int quad = lane & 3;
  const int m0 = m_blk * BM + 64 * wg;
  const int n0 = n_blk * BN;
  const bool add = (args.flags & EPI_ACCUM) != 0;
  uint8_t* my_row = wslots + (16 * wl + (lane >> 2)) * 128 + (quad & 1) * 8;
  named_bar_sync(2 + wg, 128);  // the storing thread saw the previous tile's transfers read the slots
#pragma unroll
  for (int rd = 0; rd < 2; ++rd) {
    if (rd == 1) {
      if (tid_wg == 0) tma_store_wait_read<0>();
      named_bar_sync(2 + wg, 128);
    }
#pragma unroll
    for (int jj = 0; jj < JR; ++jj) {
      const int j = rd * JR + jj;
      const int chunk = 2 * (jj & 3) + (quad >> 1);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
        *reinterpret_cast<float2*>(my_row + (jj >> 2) * kSlotBytes + hh * (8 * 128) + ((chunk ^ (lane >> 2)) << 4)) =
            make_float2(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]);
    }
    fence_proxy_async_smem();
    named_bar_sync(2 + wg, 128);
    if (tid_wg == 0) {
#pragma unroll
      for (int s = 0; s < BN / 64; ++s) {
        const int c0 = n0 + rd * (BN / 2) + 32 * s;
        if (add)
          tma_reduce_add_2d(tma_out, wslots + s * kSlotBytes, c0, m0);
        else
          tma_store_2d(tma_out, wslots + s * kSlotBytes, c0, m0);
      }
      tma_store_commit();
    }
  }
}

// Register budget: the block owns the SM's register file (384 threads x 168 at launch); the producer warpgroup gives
// registers back (40) and the two consumer warpgroups take them (232): 128*40 + 256*232 <= 64 K.  A consumer thread
// holds BN/2 fp32 accumulators (128 at BN = 256) plus the epilogue's working set.
constexpr int kGemmLightRegs = 40;
constexpr int kGemmConsumerRegs = 232;

// TMA_EPI selects the epilogue (the host picks the TMA-store one for every bf16-output, single-chunk call with
// 16-byte-aligned matrices, see gemm_sm90.cu); the producer and the main loop are the same for both.  FMT: the operand
// format (GemmFmt); FP8 changes the k-block width in elements, the wgmma instruction, the promotion of each k-block's
// partial sums into the fp32 accumulators and the dequantizing scale.
// tma_out / tma_aux / tma_in ([64 x 64] boxes, 128B swizzle over out, aux and epi_input()) are read only by it.
template <int BN, bool A_MN, bool B_MN, bool TMA_EPI, int FMT>
__global__ void __launch_bounds__(kGemmThreads, 1)
    gemm_bf16_kernel(const __grid_constant__ CUtensorMap tma_a,
                     const __grid_constant__ CUtensorMap tma_b,
                     const __grid_constant__ CUtensorMap tma_a_local,
                     const __grid_constant__ CUtensorMap tma_out,
                     const __grid_constant__ CUtensorMap tma_aux,
                     const __grid_constant__ CUtensorMap tma_in, const GemmArgs args) {
  using Cfg = GemmCfg<BN, TMA_EPI>;
  constexpr int STAGES = Cfg::kStages;
  static_assert(FMT == FMT_BF16 || (!A_MN && !B_MN && TMA_EPI), "FP8 operands are K-major and use the TMA epilogue");
  constexpr int KB = FMT == FMT_BF16 ? BK : 2 * BK;  // elements of a k-block (128-byte rows either way)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * Cfg::kABytes;
  uint8_t* smem_epi = smem + STAGES * Cfg::kStageBytes;
  float* smem_acc = reinterpret_cast<float*>(smem_epi + Cfg::kEpiStageBytes);
  uint8_t* smem_slots = smem_epi;  // TMA_EPI: kSlots x [64 x 64] bf16, then the bias slice
  uint8_t* smem_bias = smem_slots + Cfg::kSlots * Cfg::kSlotBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_epi + Cfg::kEpiStageBytes + Cfg::kAccStageBytes +
                                               Cfg::kSlots * Cfg::kSlotBytes + Cfg::kBiasBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  uint64_t* epi_full = bars + 2 * STAGES;       // TMA_EPI: the tile's bias / epilogue input landed in smem
  uint64_t* epi_empty = bars + 2 * STAGES + 1;  // TMA_EPI: both warpgroups' previous stores have read the slots
  // TMA_EPI: the producer warpgroup prefetches epilogue operands (uniform over the grid)
  const bool has_in = TMA_EPI && ((args.flags & EPI_BIAS) || epi_input(args) != nullptr);
  // warps 2, 3 sum the A stages into the bias gradient (uniform over the grid; wgrad layout only)
  const bool bgrad = A_MN && (args.flags & EPI_BGRAD) != 0;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) pdl_launch_dependents();  // the next kernel may start its prologue under this one's tail

  const int chunk_rows = (args.num_chunks > 1) ? args.chunk_rows : args.M;
  const int m_blks_per_chunk = (chunk_rows + BM - 1) / BM;
  const int unit0 = static_cast<int>(blockIdx.x) - args.n_comm;
  const int unit_stride = static_cast<int>(gridDim.x) - args.n_comm;
  const int n_blks = (args.N + BN - 1) / BN;
  const int num_tiles = m_blks_per_chunk * n_blks * args.num_chunks;
  const int num_kb = (args.K + KB - 1) / KB;
  const int k_splits = args.k_splits > 1 ? args.k_splits : 1;
  const int kb_per_split = (num_kb + k_splits - 1) / k_splits;
  const int num_work = num_tiles * k_splits;  // work item t: tile t % num_tiles, K split t / num_tiles

  if (static_cast<int>(blockIdx.x) < args.n_comm) {
    // ============================ communication CTA ============================
    // One thread drives a ring of bulk copies: peer shard -> shared memory -> local gathered
    // matrix, 16 KB per copy, 8 loads in flight per CTA (~1 MB in flight over 8 CTAs: the NVLink
    // bandwidth-delay product).
    pdl_wait();  // predecessors (the kernel that produced this rank's shard) are complete and visible
    constexpr uint32_t kSlice = 16 * 1024;
    constexpr int kCommStages = 12;  // smem ring slots
    constexpr int kLoadsInFlight = 10;  // => up to kCommStages - kLoadsInFlight stores may still be reading smem
    uint64_t* cbar = reinterpret_cast<uint64_t*>(smem + kCommStages * kSlice);
    if (threadIdx.x == 0) {
      for (int i = 0; i < kCommStages; ++i) mbar_init(&cbar[i], 1);
      fence_mbar_init();
      if (blockIdx.x == 0) {
        // my shard was produced by the previous kernel on this stream: publish it to every peer
        fence_acq_rel_sys();
        for (int p = 0; p < args.num_chunks; ++p)
          if (p != args.my_rank) st_release_sys(args.ag_peer_flag[p], args.ag_epoch);
      }
      uint32_t ph[kCommStages];
      for (int i = 0; i < kCommStages; ++i) ph[i] = 0;
      const uint64_t nslices = (args.ag_chunk_bytes + kSlice - 1) / kSlice;
      const uint64_t first = blockIdx.x, step = args.n_comm;
      const uint64_t mine = (nslices > first) ? (nslices - first + step - 1) / step : 0;
      uint64_t ring = 0;  // slices issued so far over all shards -> ring slot = ring % kCommStages
      for (int i = 1; i <= args.num_chunks; ++i) {
        // remote shards first (rank+1, rank+2, ...); the local one last: the GEMM reads it in place,
        // the copy into the gathered matrix is only needed by later consumers (wgrad)
        int src = args.my_rank + i;
        if (src >= args.num_chunks) src -= args.num_chunks;
        if (src != args.my_rank) {
          spin_until_ge_quiet(args.ag_ready + src, args.ag_epoch);  // site 1
        }
        const uint8_t* from = reinterpret_cast<const uint8_t*>(args.ag_src[src]);
        uint8_t* to = reinterpret_cast<uint8_t*>(args.ag_dst) + static_cast<uint64_t>(src) * args.ag_chunk_bytes;
        uint64_t issued = 0, stored = 0;
        while (stored < mine) {
          while (issued < mine && issued - stored < kLoadsInFlight) {
            const int st = static_cast<int>((ring + issued) % kCommStages);
            const uint64_t off = (first + issued * step) * kSlice;
            const uint32_t bytes = static_cast<uint32_t>(min(static_cast<uint64_t>(kSlice), args.ag_chunk_bytes - off));
            // the store that last used this slot is >= kCommStages - kLoadsInFlight stores old
            tma_store_wait_read<kCommStages - kLoadsInFlight>();
            mbar_arrive_expect_tx(&cbar[st], bytes);
            bulk_load_1d(smem + st * kSlice, from + off, bytes, &cbar[st]);
            ++issued;
          }
          const int st = static_cast<int>((ring + stored) % kCommStages);
          const uint64_t off = (first + stored * step) * kSlice;
          const uint32_t bytes = static_cast<uint32_t>(min(static_cast<uint64_t>(kSlice), args.ag_chunk_bytes - off));
          mbar_wait(&cbar[st], ph[st]);
          ph[st] ^= 1;
          bulk_store_1d(to + off, smem + st * kSlice, bytes);
          tma_store_commit();
          ++stored;
        }
        ring += mine;
        tma_store_wait<0>();  // this CTA's part of the shard is written
        fence_proxy_async_global();
        __threadfence();
        atomicAdd(const_cast<uint32_t*>(args.chunk_flags) + src, 1u);
      }
    }
    return;
  }

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    if constexpr (TMA_EPI) {
      tma_prefetch_desc(&tma_out);
      tma_prefetch_desc(&tma_aux);
      tma_prefetch_desc(&tma_in);
    }
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], bgrad ? 4 : 2);  // one arrival per consumer warpgroup (+ warps 2, 3: EPI_BGRAD)
    }
    if constexpr (TMA_EPI) {
      mbar_init(epi_full, 1);
      mbar_init(epi_empty, 2);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // everything above overlapped the previous kernel's tail; operands / epilogue inputs are read below

  // each register re-balancing instruction dominates the code of its warpgroup(s): ptxas allocates per region
  if (warp < 4) {
    setmaxnreg_dec<kGemmLightRegs>();
  if (warp == 0) {
    // ============================ TMA producer ============================
    int stage = 0;
    uint32_t phase = 0;
    int seen_chunk = -1;
    for (int t = unit0; t < num_work; t += unit_stride) {
      const TileCoord tc = map_tile(t % num_tiles, m_blks_per_chunk, n_blks, args.num_chunks, args.first_chunk);
      const int kb_begin = (t / num_tiles) * kb_per_split;
      const int kb_end = min(num_kb, kb_begin + kb_per_split);
      if (args.chunk_flags != nullptr && tc.chunk != seen_chunk && tc.chunk != args.a_local_chunk) {
        if (lane == 0) {
          spin_until_ge_quiet(args.chunk_flags + tc.chunk, args.flag_value);  // site 2
          fence_proxy_async_global();
        }
        __syncwarp();
        seen_chunk = tc.chunk;
      }
      int m0 = tc.m_blk * BM;
      const int n0 = tc.n_blk * BN;
      // all-gather -> GEMM: the local shard is read in place from its (peer-visible) staging buffer
      const CUtensorMap* map_a = &tma_a;
      if (args.a_local_chunk >= 0 && tc.chunk == args.a_local_chunk) {
        map_a = &tma_a_local;
        m0 -= tc.chunk * chunk_rows;
      }
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (lane == 0) {
          uint8_t* sa = smem_a + stage * Cfg::kABytes;
          uint8_t* sb = smem_b + stage * Cfg::kBBytes;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if constexpr (!A_MN) {
            tma_load_2d(sa, map_a, &full_bar[stage], kb * KB, m0);
          } else {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i)
              tma_load_2d(sa + i * (BK * 128), map_a, &full_bar[stage], m0 + i * 64, kb * BK);
          }
          if constexpr (!B_MN) {
            tma_load_2d(sb, &tma_b, &full_bar[stage], kb * KB, n0 + tc.chunk * args.b_chunk_rows);
          } else {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)
              tma_load_2d(sb + i * (BK * 128), &tma_b, &full_bar[stage], n0 + i * 64, kb * BK + tc.chunk * args.b_chunk_rows);
          }
        }
        __syncwarp();
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else if (TMA_EPI && warp == 1 && has_in) {
    // ============================ epilogue operand prefetch (TMA_EPI) ============================
    // The tile's bias slice and residual / GELU' sub-tiles go into the slots as soon as both warpgroups released them
    // (early in the tile's main loop), so the epilogue never waits on global memory.
    const void* in = epi_input(args);
    uint32_t parity = 0;
    for (int t = unit0; t < num_work; t += unit_stride) {
      const TileCoord tc = map_tile(t % num_tiles, m_blks_per_chunk, n_blks, args.num_chunks, args.first_chunk);
      const int n0 = tc.n_blk * BN;
      if (lane == 0) {
        mbar_wait(epi_empty, parity ^ 1);
        const uint32_t bias_bytes = (args.flags & EPI_BIAS) ? min(BN, args.N - n0) * 2 : 0;
        mbar_arrive_expect_tx(epi_full, bias_bytes + (in != nullptr ? Cfg::kSlots * Cfg::kSlotBytes : 0));
        if (bias_bytes > 0) bulk_load_1d(smem_bias, args.bias + n0, bias_bytes, epi_full);
        if (in != nullptr) {
#pragma unroll
          for (int s = 0; s < Cfg::kSlots; ++s)
            tma_load_2d(smem_slots + s * Cfg::kSlotBytes, &tma_in, epi_full, n0 + 64 * (s % (BN / 64)),
                        tc.m_blk * BM + 64 * (s / (BN / 64)));
        }
      }
      __syncwarp();
      parity ^= 1;
    }
  } else if (A_MN && bgrad && (warp == 2 || warp == 3)) {
    // ============================ bias gradient (EPI_BGRAD) ============================
    // bias_grad[m] = sum over k of A[k, m], read from the stages the main loop consumes: warp 2 + i sums the
    // [64 k x 64 m] box i of every stage it owns, lane l columns 2 l, 2 l + 1 (16-byte chunk l / 4 of a 128-byte
    // row, at chunk (l / 4) ^ (k % 8)).  Every tile of an M block streams the same A, so a tile sums only the
    // k-blocks with kb % n_blks == n_blk: each k-block is read once per M block, whatever the split.  The warp
    // releases each stage with its own arrival on the empty barrier and adds its sums once per work item.
    const int i = warp - 2;
    int stage = 0;
    uint32_t phase = 0;
    for (int t = unit0; t < num_work; t += unit_stride) {
      const TileCoord tc = map_tile(t % num_tiles, m_blks_per_chunk, n_blks, args.num_chunks, args.first_chunk);
      const int kb_begin = (t / num_tiles) * kb_per_split;
      const int kb_end = min(num_kb, kb_begin + kb_per_split);
      float s0 = 0.f, s1 = 0.f;
      bool summed = false;
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        if (kb % n_blks == tc.n_blk) {
          const uint8_t* box = smem_a + stage * Cfg::kABytes + i * (BK * 128) + (lane & 3) * 4;
#pragma unroll 8
          for (int k = 0; k < BK; ++k) {
            const float2 v =
                unpack_bf16x2(*reinterpret_cast<const uint32_t*>(box + k * 128 + (((lane >> 2) ^ (k & 7)) << 4)));
            s0 += v.x;
            s1 += v.y;
          }
          summed = true;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      const int m = tc.m_blk * BM + 64 * i + 2 * lane;
      if (summed && m < args.M) {
        atomicAdd(args.bias_grad + m, s0);
        if (m + 1 < args.M) atomicAdd(args.bias_grad + m + 1, s1);
      }
    }
  }
  } else {
    setmaxnreg_inc<kGemmConsumerRegs>();
    // ============================ consumers: wgmma main loop + epilogue ============================
    // Warpgroup wg (0, 1) computes rows [64 wg, 64 wg + 64) of the tile with m64 x BN x k16 wgmma, keeping one group
    // of four in flight: the stage of k-block kb is released once the group of kb + 1 is issued and kb's retired.
    // General epilogue: 8 warps; warp e = 4 wg + w (w = warp in its warpgroup) owns tile rows [32q, 32q+32) with
    // q = 2 wg + (w & 1) (one row per thread) and every second 32-column chunk (c = h, h+2, ..., h = w >> 1).  The
    // accumulators reach the row-per-thread layout through shared memory, 64 columns (two chunks) per round.  Every
    // global access is coalesced through a per-warp [32 rows x 64 B] staging buffer (16-byte chunks XOR-swizzled by
    // row pair): 4 lanes cover one 64-byte row segment, 8 rows per instruction.  Epilogue inputs (residual / GELU'
    // pre-activation) are prefetched one chunk ahead into registers.
    const int e = warp - 4;
    const int wg = e >> 2;
    const int wl = e & 3;
    const int q = 2 * wg + (wl & 1);
    const int h = wl >> 1;
    const int tid_wg = threadIdx.x & 127;
    float* acc_stage = smem_acc + wg * 64 * kAccLd;
    constexpr int NCH = BN / 32;
    constexpr int NRD = BN / 64;  // hand-over rounds
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    const bool out_f32 = (args.flags & EPI_OUT_F32) != 0;
    const __nv_bfloat16* in_ptr = nullptr;
    int in_ld = 0;
    if (!out_f32) {
      if (args.flags & EPI_DGELU) {
        in_ptr = reinterpret_cast<const __nv_bfloat16*>(args.aux);
        in_ld = args.ldc;
      } else if (args.flags & EPI_RESIDUAL) {
        in_ptr = args.residual;
        in_ld = args.ldr;
      }
    }
    uint8_t* stg_warp = smem_epi + e * 2048;
    uint8_t* stg_own = stg_warp + lane * 64;         // this thread's row (64 B)
    const int own_sw = (lane >> 1) & 3;               // swizzle of this thread's row
    const int co_r = lane >> 2;                       // coalesced pattern: row inside a group of 8
    const int co_ch = lane & 3;                       // 16-byte chunk of the 64-byte segment
    bool rs_ready = false;                            // peers' partial tiles of the local chunk have landed
    uint32_t epi_parity = 0;                          // TMA_EPI: phase of epi_full for this tile
    for (int t = unit0; t < num_work; t += unit_stride) {
      const TileCoord tc = map_tile(t % num_tiles, m_blks_per_chunk, n_blks, args.num_chunks, args.first_chunk);
      {
        const int kb_begin = (t / num_tiles) * kb_per_split;
        const int kb_end = min(num_kb, kb_begin + kb_per_split);
        int prev_stage = -1;
        wgmma_fence_regs(acc);
        if constexpr (FMT != FMT_BF16) {
          // FP8 wgmma accumulates with less than fp32 precision: each 128-wide k-block is summed by the tensor cores
          // into `part` alone and then added into the fp32 accumulators (promotion), so that error does not grow
          // with K.  The stage is released as soon as its k-block retired.
          float part[BN / 2];
          for (int kb = kb_begin; kb < kb_end; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = smem_u32(smem_a + stage * Cfg::kABytes) + wg * (64 * 128);
            const uint32_t sb = smem_u32(smem_b + stage * Cfg::kBBytes);
            wgmma_fence_regs(part);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / WG_K; ++k)  // k32 step k: bytes [32 k, 32 k + 32) of the K-major rows
              WgmmaFp8<BN, FMT == FMT_E5M2>::mma(part, make_wgmma_desc_sw128(sa + k * 32, 0, 1024),
                                                 make_wgmma_desc_sw128(sb + k * 32, 0, 1024), k > 0 ? 1u : 0u);
            wgmma_commit();
            if constexpr (TMA_EPI) {
              if (kb == kb_begin && t != unit0 && tid_wg == 0) {
                tma_store_wait_read<0>();
                if (has_in) mbar_arrive(epi_empty);
              }
            }
            wgmma_wait<0>();
            wgmma_fence_regs(part);
            if (tid_wg == 0) mbar_arrive(&empty_bar[stage]);
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = kb > kb_begin ? acc[i] + part[i] : part[i];
            if (++stage == STAGES) {
              stage = 0;
              phase ^= 1;
            }
          }
        } else {
        for (int kb = kb_begin; kb < kb_end; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          // this warpgroup's 64 rows: the second half of a K-major tile, or the second 64-wide atom of an MN-major one
          const uint32_t sa = smem_u32(smem_a + stage * Cfg::kABytes) + wg * (64 * 128);
          const uint32_t sb = smem_u32(smem_b + stage * Cfg::kBBytes);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / WG_K; ++k) {
            const uint64_t da = A_MN ? make_wgmma_desc_sw128(sa + k * (WG_K * 128), BK * 128, 1024)
                                     : make_wgmma_desc_sw128(sa + k * (WG_K * 2), 0, 1024);
            const uint64_t db = B_MN ? make_wgmma_desc_sw128(sb + k * (WG_K * 128), BK * 128, 1024)
                                     : make_wgmma_desc_sw128(sb + k * (WG_K * 2), 0, 1024);
            Wgmma<BN, A_MN, B_MN>::mma(acc, da, db, (kb > kb_begin || k > 0) ? 1u : 0u);
          }
          wgmma_commit();
          if constexpr (TMA_EPI) {
            // the previous tile's stores have long read the slots: hand them to the operand prefetch / next epilogue
            if (kb == kb_begin && t != unit0 && tid_wg == 0) {
              tma_store_wait_read<0>();
              if (has_in) mbar_arrive(epi_empty);
            }
          }
          wgmma_wait<1>();
          if (prev_stage >= 0 && tid_wg == 0) mbar_arrive(&empty_bar[prev_stage]);
          prev_stage = stage;
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (prev_stage >= 0 && tid_wg == 0) mbar_arrive(&empty_bar[prev_stage]);
        }
      }
      if constexpr (FMT != FMT_BF16) {
        // dequantize once: the product of the two per-tensor scales (read after pdl_wait: the casts wrote them)
        const float s = *args.a_scale_inv * *args.b_scale_inv;
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] *= s;
      }
      if constexpr (TMA_EPI) {
        uint8_t* wslots = smem_slots + wg * (BN / 64) * Cfg::kSlotBytes;
        if (out_f32) {
          epilogue_tma_f32<BN>(acc, args, &tma_out, wslots, tc.m_blk, tc.n_blk, wg, tid_wg);
          continue;
        }
        epilogue_tma<BN>(acc, args, &tma_out, &tma_aux, wslots, smem_bias, epi_full, epi_parity, has_in, tc.m_blk,
                         tc.n_blk, n_blks, wg, tid_wg);
        epi_parity ^= 1;
        continue;
      }
      const int row = tc.m_blk * BM + q * 32 + lane;
      const int n0 = tc.n_blk * BN;
      // destination row pointer (possibly on a peer GPU)
      uint8_t* out_base = reinterpret_cast<uint8_t*>(args.out);
      int out_row = row;
      int row_limit = args.M;
      if (args.num_chunks > 1) {
        row_limit = (tc.chunk + 1) * chunk_rows;
        if (args.out_peer[0] != nullptr && !(args.flags & EPI_SCATTER)) {
          out_base = reinterpret_cast<uint8_t*>(args.out_peer[tc.chunk]);
          out_row = row - tc.chunk * chunk_rows;
        }
      }
      // GEMM -> reduce-scatter with the reduction fused into the local chunk's epilogue
      const bool rs_mode = args.rs_wait_ctr != nullptr && args.num_chunks > 1;
      const bool rs_local = rs_mode && tc.chunk == args.my_rank;
      if (rs_local) {
        out_base = reinterpret_cast<uint8_t*>(args.out);
        out_row = row - tc.chunk * chunk_rows;
        if (!rs_ready) {
          // peers computed my chunk FIRST; by the time I reach it their tiles have normally landed
          if (lane == 0) {
            for (int s2 = 0; s2 < args.num_chunks; ++s2)
              if (s2 != args.my_rank) spin_until_ge_quiet(args.rs_wait_ctr + s2, args.rs_wait_value);  // site 3
          }
          __syncwarp();
          rs_ready = true;
        }
      }
      const bool row_ok = row < row_limit && row < args.M;
      const int warp_row0 = tc.m_blk * BM + q * 32;  // first row handled by this warp
      const int warp_out_row0 = out_row - lane;               // its destination row index
      const int rows_ok = max(0, min(32, min(row_limit, args.M) - warp_row0));
      const int local_row0 = warp_row0 - tc.chunk * chunk_rows;
      // bias / residual of a fused reduce-scatter belong to the final (local) rows, not to partials sent to peers;
      // the residual is then the local token shard [chunk_rows, N]
      const bool use_in = in_ptr != nullptr && (!rs_mode || rs_local);
      const bool use_bias = (args.flags & EPI_BIAS) && (!rs_mode || rs_local);
      uint4 pre[4];
      auto prefetch_in = [&](int c) {
        const int col = n0 + c * 32 + co_ch * 8;
        const __nv_bfloat16* base = in_ptr + static_cast<size_t>(rs_local ? local_row0 : warp_row0) * in_ld;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int rr = i * 8 + co_r;
          pre[i] = make_uint4(0, 0, 0, 0);
          if (rr < rows_ok && col < args.N) pre[i] = ld_global_nc_v4(base + static_cast<size_t>(rr) * in_ld + col);
        }
      };
      if (use_in && h < NCH) prefetch_in(h);
      float ce_m = -INFINITY, ce_s = 0.f;  // online softmax partial of this thread's row over this warp's chunks
#pragma unroll 1
      for (int rd = 0; rd < NRD; ++rd) {
        // columns [64 rd, 64 rd + 64): fragments -> shared memory (the previous round's readers are done)
        named_bar_sync(2 + wg, 128);
#pragma unroll
        for (int r2 = 0; r2 < NRD; ++r2) {
          if (r2 == rd) {  // constant register indices
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
              for (int hh = 0; hh < 2; ++hh) {
                const int fr = 16 * wl + (lane >> 2) + 8 * hh;
                const int fc = 8 * j + 2 * (lane & 3);
                *reinterpret_cast<float2*>(acc_stage + fr * kAccLd + fc) =
                    make_float2(acc[32 * r2 + 4 * j + 2 * hh], acc[32 * r2 + 4 * j + 2 * hh + 1]);
              }
            }
          }
        }
        named_bar_sync(2 + wg, 128);
        const int c = 2 * rd + h;
        uint32_t v[32];
        {
          const float* src = acc_stage + (32 * (wl & 1) + lane) * kAccLd + 32 * h;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 x = *reinterpret_cast<const float4*>(src + 4 * i);
            v[4 * i] = __float_as_uint(x.x);
            v[4 * i + 1] = __float_as_uint(x.y);
            v[4 * i + 2] = __float_as_uint(x.z);
            v[4 * i + 3] = __float_as_uint(x.w);
          }
        }
        if (use_in) {
          // park the prefetched inputs in the staging buffer, start fetching the next chunk's
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int rr = i * 8 + co_r;
            *reinterpret_cast<uint4*>(stg_warp + rr * 64 + ((co_ch ^ ((rr >> 1) & 3)) << 4)) = pre[i];
          }
          __syncwarp();
          if (c + 2 < NCH) prefetch_in(c + 2);
        }
        const int col0 = n0 + c * 32;
        const int ncols = max(0, min(32, args.N - col0));  // multiple of 8
        float f[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) f[i] = __uint_as_float(v[i]);
        const bool active = row_ok && ncols > 0;
        if (active && use_bias) {
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            if (g * 8 < ncols) {
              const uint4 bb = ld_global_nc_v4(args.bias + tc.chunk * args.bias_chunk_stride + col0 + g * 8);
              const uint32_t bw[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float2 bf = unpack_bf16x2(bw[j]);
                f[g * 8 + 2 * j] += bf.x;
                f[g * 8 + 2 * j + 1] += bf.y;
              }
            }
          }
        }
        if (out_f32) {
          // fp32 output (wgrad into the main-grad buffer): each thread owns a full 128-byte line
          if (active && args.grad_rs.world > 1) {
            // gradient reduce-scatter fused into the wgrad: the line goes to the owner of its ZeRO-1 slice
            const float* o = reinterpret_cast<const float*>(out_base) + static_cast<size_t>(out_row) * args.ldc + col0;
            const long long off = (o - args.grad_rs.local) - args.grad_rs.start;
            const long long own0 = grs_owner(args.grad_rs, off);
            const bool one_owner = off - own0 * args.grad_rs.seg + 32 <= args.grad_rs.seg;
            float* t0 = grs_target(args.grad_rs, o);
#pragma unroll
            for (int g = 0; g < 8; ++g) {
              if (g * 4 < ncols) {
                const float4 val = make_float4(f[g * 4], f[g * 4 + 1], f[g * 4 + 2], f[g * 4 + 3]);
                grs_add4_at(args.grad_rs, one_owner ? t0 + g * 4 : grs_target(args.grad_rs, o + g * 4), val);
              }
            }
            continue;
          }
          if (active) {
            float* o = reinterpret_cast<float*>(out_base) + static_cast<size_t>(out_row) * args.ldc + col0;
#pragma unroll
            for (int g = 0; g < 8; ++g) {
              if (g * 4 < ncols) {
                float4 val = make_float4(f[g * 4], f[g * 4 + 1], f[g * 4 + 2], f[g * 4 + 3]);
                if (args.flags & EPI_ATOMIC) {
                  red_add_v4_f32(o + g * 4, val);  // split-K partial sums
                } else {
                  if (args.flags & EPI_ACCUM) {
                    const float4 old = *reinterpret_cast<const float4*>(o + g * 4);
                    val.x += old.x; val.y += old.y; val.z += old.z; val.w += old.w;
                  }
                  *reinterpret_cast<float4*>(o + g * 4) = val;
                }
              }
            }
          }
          continue;
        }
        // coalesced store of the staged [32 x 64 B] block to rows dst_row0.. of a bf16 matrix
        auto store_block = [&](__nv_bfloat16* base, int dst_row0, int ld) {
          __syncwarp();
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int rr = i * 8 + co_r;
            if (rr < rows_ok && co_ch * 8 < ncols) {
              const uint4 val = *reinterpret_cast<const uint4*>(stg_warp + rr * 64 + ((co_ch ^ ((rr >> 1) & 3)) << 4));
              st_global_v4(base + static_cast<size_t>(dst_row0 + rr) * ld + col0 + co_ch * 8, val);
            }
          }
          __syncwarp();
        };
        auto stage_own = [&]() {
#pragma unroll
          for (int g = 0; g < 4; ++g)
            *reinterpret_cast<uint4*>(stg_own + ((g ^ own_sw) << 4)) =
                make_uint4(pack_bf16x2(f[g * 8 + 0], f[g * 8 + 1]), pack_bf16x2(f[g * 8 + 2], f[g * 8 + 3]),
                           pack_bf16x2(f[g * 8 + 4], f[g * 8 + 5]), pack_bf16x2(f[g * 8 + 6], f[g * 8 + 7]));
        };
        if (args.ce_part != nullptr) {
          // statistics of the values as they are STORED (rounded to bf16), so that the later softmax over the stored
          // logits is normalised exactly
          const int lim = min(ncols, args.ce_valid - col0);
          if (lim > 0) {
            float cm = -INFINITY;
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              f[i] = __bfloat162float(__float2bfloat16_rn(f[i]));
              if (i < lim) cm = fmaxf(cm, f[i]);
            }
            const float nm = fmaxf(ce_m, cm);
            float sum = 0.f;
#pragma unroll
            for (int i = 0; i < 32; ++i)
              if (i < lim) sum += exp2f((f[i] - nm) * 1.4426950408889634f);
            ce_s = ce_s * exp2f((ce_m - nm) * 1.4426950408889634f) + sum;
            ce_m = nm;
          }
        }
        if (args.flags & EPI_GELU) {
          if (args.aux != nullptr) {
            // the pre-activation goes out through the same staged, coalesced path
            stage_own();
            store_block(reinterpret_cast<__nv_bfloat16*>(args.aux), warp_row0, args.ldc);
          }
#pragma unroll
          for (int i = 0; i < 32; ++i) f[i] = gelu_tanh(f[i]);
        }
        if (use_in) {
          const bool dgelu = (args.flags & EPI_DGELU) != 0;
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            const uint4 z = *reinterpret_cast<const uint4*>(stg_own + ((g ^ own_sw) << 4));
            const uint32_t zw[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float2 zf = unpack_bf16x2(zw[j]);
              if (dgelu) {
                f[g * 8 + 2 * j] *= gelu_tanh_grad(zf.x);
                f[g * 8 + 2 * j + 1] *= gelu_tanh_grad(zf.y);
              } else {
                f[g * 8 + 2 * j] += zf.x;
                f[g * 8 + 2 * j + 1] += zf.y;
              }
            }
          }
        }
        if (rs_local) {
          // add every peer's staged partial of this chunk (local memory, written through NVLink and acquired above)
#pragma unroll 1
          for (int src = 0; src < args.num_chunks; ++src) {
            if (src == args.my_rank) continue;
            const __nv_bfloat16* base = args.rs_in[src] + static_cast<size_t>(local_row0) * args.N + col0 + co_ch * 8;
            __syncwarp();
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int rr = i * 8 + co_r;
              uint4 val = make_uint4(0, 0, 0, 0);
              if (rr < rows_ok && co_ch * 8 < ncols) val = ld_global_v4(base + static_cast<size_t>(rr) * args.N);
              *reinterpret_cast<uint4*>(stg_warp + rr * 64 + ((co_ch ^ ((rr >> 1) & 3)) << 4)) = val;
            }
            __syncwarp();
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              const uint4 z = *reinterpret_cast<const uint4*>(stg_own + ((g ^ own_sw) << 4));
              const uint32_t zw[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float2 zf = unpack_bf16x2(zw[j]);
                f[g * 8 + 2 * j] += zf.x;
                f[g * 8 + 2 * j + 1] += zf.y;
              }
            }
          }
          __syncwarp();
        }
        if (active && (args.flags & EPI_SCATTER)) {
          const float sc = args.row_scale[row];
#pragma unroll
          for (int i = 0; i < 32; ++i) f[i] *= sc;
        }
        stage_own();
        if (args.flags & EPI_SCATTER) {
          __syncwarp();
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int rr = i * 8 + co_r;
            if (rr < rows_ok && co_ch * 8 < ncols) {
              const int gr = warp_row0 + rr;
              const int ret = args.row_ret[gr];
              if (ret >= 0) {
                const uint4 val = *reinterpret_cast<const uint4*>(stg_warp + rr * 64 + ((co_ch ^ ((rr >> 1) & 3)) << 4));
                const int src = (gr - tc.chunk * chunk_rows) / args.scatter_rows_per_src;
                st_global_v4(reinterpret_cast<__nv_bfloat16*>(args.out_peer[src]) +
                                 static_cast<size_t>(ret) * args.ldc + col0 + co_ch * 8, val);
              }
            }
          }
          __syncwarp();
        } else {
          store_block(reinterpret_cast<__nv_bfloat16*>(out_base), warp_out_row0, args.ldc);
        }
      }
      if (args.ce_part != nullptr && row_ok) {
        float2* dst = reinterpret_cast<float2*>(args.ce_part) + static_cast<size_t>(row) * (2 * n_blks) + 2 * tc.n_blk + h;
        *dst = make_float2(ce_m, ce_s);
      }
      if (args.num_chunks > 1 && args.arrive_ctr[0] != nullptr && !(args.flags & EPI_SCATTER) && !rs_local) {
        // all eight epilogue warps have stored their part of this tile -> publish to the owner
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (warp == 4 && lane == 0) {
          fence_acq_rel_sys();
          red_add_release_sys(args.arrive_ctr[tc.chunk], 1u);
        }
      }
    }
    // TMA_EPI: the last stores complete before the CTA (and its shared memory) goes away
    if (TMA_EPI && tid_wg == 0) tma_store_wait<0>();
  }
}

}  // namespace pg
