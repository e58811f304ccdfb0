// Host side of the wgmma GEMM: TMA tensor-map construction (driver entry point resolved at
// run time so the library links without libcuda), tile-shape selection, launch.
#include "gemm_sm90.cuh"
#include "launch.h"
#include "pdl_launch.cuh"

#include <cstdio>
#include <cstring>
#include <mutex>
#include <unordered_map>

namespace pg {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || p == nullptr) {
      fprintf(stderr, "pipegoose_b200: cuTensorMapEncodeTiled not available (%s)\n",
              cudaGetErrorString(e));
      return nullptr;
    }
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// 2-D tensor map over a row-major [rows, cols] matrix (cols contiguous, leading dimension ld elements) of esize-byte
// elements (1: FP8 codes as UINT8, 2: bf16, 4: fp32) with a [box_rows, box_cols] box and 128-byte swizzle.
static int make_tmap_2d(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld,
                        uint32_t box_rows, uint32_t box_cols, int esize) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return -1;
  // driver entry points need the primary context bound to the calling thread (autograd worker
  // threads have not necessarily touched the runtime yet)
  cudaFree(nullptr);
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * esize};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = esize == 4   ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                 : esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                              : CU_TENSOR_MAP_DATA_TYPE_UINT8;
  CUresult r = enc(out, dt, 2, const_cast<void*>(ptr), dims,
                   strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr,
            "pipegoose_b200: cuTensorMapEncodeTiled failed (%d) ptr=%p rows=%llu cols=%llu ld=%llu "
            "box=%ux%u\n",
            (int)r, ptr, (unsigned long long)rows, (unsigned long long)cols,
            (unsigned long long)ld, box_rows, box_cols);
    return -1;
  }
  return 0;
}

int make_tmap_bf16_2d(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols,
                      uint64_t ld, uint32_t box_rows, uint32_t box_cols) {
  return make_tmap_2d(out, ptr, rows, cols, ld, box_rows, box_cols, 2);
}

// 3-D fp32 tensor map over a contiguous [d2, d1, d0] tensor (d0 contiguous) with a [1, box1, 32] box and 128-byte
// swizzle (32 fp32 = one 128-byte row), for TMA reduce-adds of fp32 tiles.
int make_tmap_f32_3d(CUtensorMap* out, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t box1) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return -1;
  cudaFree(nullptr);
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {d0 * 4, d0 * d1 * 4};
  cuuint32_t box[3] = {32, box1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "pipegoose_b200: cuTensorMapEncodeTiled (fp32, 3-D) failed (%d) ptr=%p dims=%llu x %llu x %llu\n",
            (int)r, ptr, (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2);
    return -1;
  }
  return 0;
}

struct TmapKey {
  const void* ptr;
  uint64_t rows, cols, ld;
  uint32_t box_rows;
  int esize;
  bool operator==(const TmapKey& o) const {
    return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows && esize == o.esize;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr);
    h ^= k.rows * 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
    h ^= k.cols * 0xC2B2AE3D27D4EB4Full + (h << 6) + (h >> 2);
    h ^= (k.ld * 31 + k.box_rows * 8 + k.esize) + (h << 6) + (h >> 2);
    return h;
  }
};

// [box_rows x 128 / esize] boxes: 128-byte box rows (64 bf16, 32 fp32 or 128 FP8 codes)
static int cached_tmap(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols,
                       uint64_t ld, uint32_t box_rows, int esize = 2) {
  static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  static std::mutex mu;
  TmapKey key{ptr, rows, cols, ld, box_rows, esize};
  std::lock_guard<std::mutex> g(mu);
  auto it = cache.find(key);
  if (it != cache.end()) {
    *out = it->second;
    return 0;
  }
  if (make_tmap_2d(out, ptr, rows, cols, ld, box_rows, 128 / esize, esize) != 0) return -1;
  if (cache.size() > 8192) cache.clear();
  cache.emplace(key, *out);
  return 0;
}

static int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// The three tensor maps of the TMA-store epilogue ([64 x 64] boxes over out / aux / the epilogue input)
struct EpiMaps {
  CUtensorMap out, aux, in;
};

template <int BN, bool A_MN, bool B_MN, bool TMA_EPI, int FMT = FMT_BF16>
static int launch_cfg(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tal, const EpiMaps& em,
                      const GemmArgs& args, int max_ctas, cudaStream_t stream) {
  using Cfg = GemmCfg<BN, TMA_EPI>;
  auto kern = gemm_bf16_kernel<BN, A_MN, B_MN, TMA_EPI, FMT>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e =
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      fprintf(stderr, "pipegoose_b200: cudaFuncSetAttribute failed: %s\n", cudaGetErrorString(e));
      return -1;
    }
    attr_set = true;
  }
  const int chunk_rows = args.num_chunks > 1 ? args.chunk_rows : args.M;
  const int tiles = ((chunk_rows + BM - 1) / BM) * ((args.N + BN - 1) / BN) * args.num_chunks *
                    (args.k_splits > 1 ? args.k_splits : 1);
  int units = max_ctas - args.n_comm;  // CTAs that run GEMM tiles
  if (units < 1) units = 1;
  if (tiles < units) units = tiles;
  if (units < 1) units = 1;
  const int grid = units + args.n_comm;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid, 1, 1);
  cfg.blockDim = dim3(kGemmThreads, 1, 1);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, ta, tb, tal, em.out, em.aux, em.in, args);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) {
    fprintf(stderr, "pipegoose_b200: gemm launch failed: %s\n", cudaGetErrorString(e));
    return -1;
  }
  return 0;
}

// Tile width (and, for fp32-accumulating outputs, a K split) by a wave-quantisation cost model:
// cost = waves * (k-blocks per work item * BN / efficiency(BN)) + one exposed epilogue.
// cheap_split: partial sums leave through the TMA epilogue's reduce-adds, which cost what a plain store costs.
// kblk: elements of a k-block (BK for bf16, 2 BK for FP8); max_bn: widest tile allowed.
static int pick_bn(int M_rows, int N, int K, int kblk, int max_bn, int chunks, int ctas, bool allow_split,
                   bool cheap_split, int* k_splits) {
  const int cand[4] = {256, 192, 128, 64};
  const float eff[4] = {1.0f, 0.93f, 0.82f, 0.55f};  // 128 x BN tiles
  const int num_kb = (K + kblk - 1) / kblk;
  int best = 256;
  float best_cost = 1e30f;
  *k_splits = 1;
  for (int i = 0; i < 4; ++i) {
    const int bn = cand[i];
    if (bn > max_bn || (bn > 64 && N <= bn / 2)) continue;
    const long tiles = (long)((M_rows + BM - 1) / BM) * ((N + bn - 1) / bn) * chunks;
    const int max_split = allow_split ? 8 : 1;
    for (int s = 1; s <= max_split; ++s) {
      const int per = (num_kb + s - 1) / s;
      if (s > 1 && (per < 16 || (long)(s - 1) * per >= num_kb)) break;
      const long waves = (tiles * s + ctas - 1) / ctas;
      // the epilogue of the last wave is exposed; per-thread atomics cost about twice a plain store
      const float epi = (s > 1 && !cheap_split ? 16.0f : 8.0f) * (float)bn;
      const float cost = (float)waves * (float)per * (float)bn / eff[i] + epi;
      if (cost < best_cost * 0.97f) {
        best_cost = cost;
        best = bn;
        *k_splits = s;
      }
    }
  }
  return best;
}

}  // namespace pg

using namespace pg;

static int g_cta_cap = 0;
extern "C" void pg_set_gemm_cta_cap(int ctas) { g_cta_cap = ctas > 0 ? ctas : 0; }

extern "C" int pg_gemm_bf16(const PgGemmDesc* d, cudaStream_t stream) {
  if (d->M <= 0 || d->N <= 0 || d->K <= 0) return 0;
  GemmArgs args;
  memset(&args, 0, sizeof(args));
  args.M = d->M;
  args.N = d->N;
  args.K = d->K;
  args.out = d->out;
  args.ldc = d->ldc;
  args.bias = reinterpret_cast<const __nv_bfloat16*>(d->bias);
  args.residual = reinterpret_cast<const __nv_bfloat16*>(d->residual);
  args.ldr = d->ldr;
  args.aux = d->aux;
  args.flags = d->flags;
  args.num_chunks = d->num_chunks > 1 ? d->num_chunks : 1;
  args.chunk_rows = d->chunk_rows;
  args.first_chunk = d->first_chunk;
  args.chunk_flags = d->chunk_flags;
  args.flag_value = d->flag_value;
  for (int i = 0; i < kMaxPeers; ++i) {
    args.out_peer[i] = d->out_peer[i];
    args.arrive_ctr[i] = d->arrive_ctr[i];
    args.rs_in[i] = reinterpret_cast<const __nv_bfloat16*>(d->rs_in[i]);
  }
  args.rs_wait_ctr = d->rs_wait_ctr;
  args.rs_wait_value = d->rs_wait_value;
  args.ce_part = d->ce_part;
  args.ce_valid = d->ce_valid > 0 ? d->ce_valid : d->N;
  args.grad_rs = d->grad_rs;
  args.bias_grad = d->bias_grad;
  args.a_scale_inv = d->a_scale_inv;
  args.b_scale_inv = d->b_scale_inv;
  const bool fp8 = d->fmt != FMT_BF16;
  const int kblk = fp8 ? 2 * BK : BK;
  if (fp8 && (d->fmt != FMT_E4M3 && d->fmt != FMT_E5M2)) {
    fprintf(stderr, "pipegoose_b200: unknown GEMM operand format %d\n", d->fmt);
    return -1;
  }
  if (fp8 && (d->a_mn || d->b_mn || d->num_chunks > 1 || d->n_comm > 0 || d->grad_rs.world > 1 ||
              d->ce_part != nullptr || (d->flags & (EPI_BGRAD | EPI_SCATTER)) || d->a_scale_inv == nullptr ||
              d->b_scale_inv == nullptr || (d->K % 16) != 0 || (d->lda % 16) != 0 || (d->ldb % 16) != 0 ||
              (reinterpret_cast<uintptr_t>(d->A) & 15) != 0 || (reinterpret_cast<uintptr_t>(d->B) & 15) != 0)) {
    fprintf(stderr, "pipegoose_b200: the FP8 GEMM needs K-major 16-byte-aligned operands (K %% 16 == 0), both scales, "
                    "one chunk and no fused collective, scatter or bias gradient\n");
    return -1;
  }
  if ((args.flags & EPI_BGRAD) &&
      (!d->a_mn || args.bias_grad == nullptr || d->num_chunks > 1 || d->n_comm > 0)) {
    fprintf(stderr, "pipegoose_b200: the fused bias gradient needs an MN-major A, a bias_grad buffer and one chunk\n");
    return -1;
  }
  if (args.grad_rs.world > 1) {
    if (!(d->flags & EPI_OUT_F32) || args.num_chunks > 1 || (d->ldc % 4) != 0) {
      fprintf(stderr, "pipegoose_b200: gradient reduce-scatter epilogue needs a plain fp32 output with ldc %% 4 == 0\n");
      return -1;
    }
    args.flags |= EPI_ACCUM;  // contributions are ADDED into the owners' buffers (zeroed by the optimizer step)
  }
  args.b_chunk_rows = d->b_chunk_rows;
  args.bias_chunk_stride = d->bias_chunk_stride;
  args.row_ret = d->row_ret;
  args.row_scale = d->row_scale;
  args.scatter_rows_per_src = d->scatter_rows_per_src > 0 ? d->scatter_rows_per_src : 1;
  args.n_comm = d->n_comm;
  args.ag_dst = d->ag_dst;
  args.ag_chunk_bytes = d->ag_chunk_bytes;
  args.ag_ready = d->ag_ready;
  args.ag_epoch = d->ag_epoch;
  args.my_rank = d->my_rank;
  for (int i = 0; i < kMaxPeers; ++i) {
    args.ag_src[i] = d->ag_src[i];
    args.ag_peer_flag[i] = d->ag_peer_flag[i];
  }
  if (args.num_chunks > 1 && (args.chunk_rows % BM) != 0) {
    fprintf(stderr, "pipegoose_b200: chunk_rows (%d) must be a multiple of %d\n", args.chunk_rows, BM);
    return -1;
  }
  int max_ctas = d->max_ctas > 0 ? d->max_ctas : num_sms();
  if (d->max_ctas <= 0 && g_cta_cap > 0 && g_cta_cap < max_ctas) max_ctas = g_cta_cap;
  const int chunk_rows = args.num_chunks > 1 ? args.chunk_rows : args.M;
  if ((args.flags & EPI_DGELU) && (args.flags & EPI_RESIDUAL)) {
    fprintf(stderr, "pipegoose_b200: EPI_DGELU and EPI_RESIDUAL are mutually exclusive\n");
    return -1;
  }
  // split-K only where the epilogue can add partial sums: plain fp32 outputs (wgrad into main grads)
  const bool allow_split = (args.flags & EPI_OUT_F32) && args.num_chunks == 1 && args.bias == nullptr &&
                           d->k_splits != 1 && (d->ldc % 4) == 0;
  // the TMA epilogue serves plain fp32 outputs (see tma_epi below)
  const bool f32_tma = (args.flags & EPI_OUT_F32) && args.num_chunks == 1 && args.bias == nullptr &&
                       (d->ldc % 4) == 0 && args.grad_rs.world <= 1 && args.n_comm == 0 && args.ce_part == nullptr &&
                       !(args.flags & (EPI_GELU | EPI_RESIDUAL | EPI_DGELU | EPI_SCATTER)) &&
                       (reinterpret_cast<uintptr_t>(args.out) & 15) == 0;
  int auto_splits = 1;
  // FP8 promotes each k-block's partial sums into a second set of accumulators: tiles up to 128 wide
  int bn = pick_bn(chunk_rows, args.N, args.K, kblk, fp8 ? 128 : 256, args.num_chunks, max_ctas - args.n_comm,
                   allow_split, f32_tma, &auto_splits);
  if (args.ce_part != nullptr && d->block_n <= 0) {
    // the partials are laid out per 256-column tile (two per row and tile): fix the tile width
    bn = 256;
    auto_splits = 1;
  }
  if (d->block_n > 0) {
    bn = d->block_n;
    auto_splits = 1;
  }
  args.k_splits = (allow_split && d->k_splits > 1) ? d->k_splits : auto_splits;
  {
    const int num_kb = (args.K + kblk - 1) / kblk;
    if (args.k_splits > num_kb) args.k_splits = num_kb;
    if (args.k_splits > 1) {
      const int per = (num_kb + args.k_splits - 1) / args.k_splits;
      args.k_splits = (num_kb + per - 1) / per;  // no empty split
    }
  }
  if (args.k_splits > 1) {
    if (!(args.flags & EPI_ACCUM)) {
      // partial sums are added atomically: an overwriting GEMM starts from zero
      cudaMemset2DAsync(args.out, (size_t)args.ldc * 4, 0, (size_t)args.N * 4, (size_t)args.M, stream);
    }
    args.flags |= EPI_ATOMIC | EPI_ACCUM;
  }

  CUtensorMap ta, tb, tal;
  args.a_local_chunk = -1;
  // A: K-major  -> matrix [M, K] (ld = lda), box [128 rows, 64]
  //    MN-major -> matrix [K, M] (ld = lda), box [64 k-rows, 64]
  const int op_esize = fp8 ? 1 : 2;
  if (!d->a_mn) {
    if (cached_tmap(&ta, d->A, d->M, d->K, d->lda, BM, op_esize) != 0) return -1;
  } else {
    if (cached_tmap(&ta, d->A, d->K, d->M, d->lda, BK) != 0) return -1;
  }
  const uint64_t b_groups = d->b_chunk_rows > 0 ? (uint64_t)args.num_chunks : 1;  // stacked expert weights
  if (!d->b_mn) {
    if (cached_tmap(&tb, d->B, d->N * b_groups, d->K, d->ldb, bn, op_esize) != 0) return -1;
  } else {
    if (cached_tmap(&tb, d->B, d->K * b_groups, d->N, d->ldb, BK) != 0) return -1;
  }

  tal = ta;
  if (d->a_local != nullptr && !d->a_mn && args.num_chunks > 1) {
    // the local shard of an all-gather -> GEMM is read in place: [chunk_rows, K] matrix
    if (cached_tmap(&tal, d->a_local, args.chunk_rows, d->K, d->K, BM) != 0) return -1;
    args.a_local_chunk = d->my_rank;
  }

  // The TMA-store epilogue serves every call with a bf16 output, one chunk (no fused collective, no MoE scatter)
  // and 16-byte-aligned matrices (TMA's requirement).  The GELU pre-activation output cannot share the slots with
  // an epilogue input, so that combination also stays on the general epilogue.  It also serves plain fp32 outputs
  // (f32_tma: no bias or other epilogue input, no gradient reduce-scatter), split or not: partial sums and
  // accumulation leave as TMA reduce-adds.
  auto aligned = [](const void* p, int ld) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0 && (ld % 8) == 0; };
  const void* epi_in = (args.flags & EPI_DGELU) ? args.aux : (args.flags & EPI_RESIDUAL) ? args.residual : nullptr;
  const int in_ld = (args.flags & EPI_DGELU) ? args.ldc : args.ldr;
  const bool gelu_aux = (args.flags & EPI_GELU) && args.aux != nullptr;
  const bool tma_epi = f32_tma || (!(args.flags & (EPI_OUT_F32 | EPI_SCATTER)) && args.num_chunks == 1 &&
                                   args.n_comm == 0 && args.grad_rs.world <= 1 && args.k_splits == 1 &&
                                   aligned(args.out, args.ldc) &&
                                   (!gelu_aux || (aligned(args.aux, args.ldc) && epi_in == nullptr)) &&
                                   (epi_in == nullptr || aligned(epi_in, in_ld)) &&
                                   (!(args.flags & EPI_BIAS) || aligned(args.bias, 8)));
  EpiMaps em;
  memset(&em, 0, sizeof(em));
  if (f32_tma) {
    if (cached_tmap(&em.out, args.out, args.M, args.N, args.ldc, 64, 4) != 0) return -1;
    em.aux = em.in = em.out;
  } else if (tma_epi) {
    if (cached_tmap(&em.out, args.out, args.M, args.N, args.ldc, 64) != 0) return -1;
    em.aux = em.in = em.out;
    if (gelu_aux && cached_tmap(&em.aux, args.aux, args.M, args.N, args.ldc, 64) != 0) return -1;
    if (epi_in != nullptr && cached_tmap(&em.in, epi_in, args.M, args.N, in_ld, 64) != 0) return -1;
  }

  if (fp8) {
    if (!tma_epi) {
      fprintf(stderr, "pipegoose_b200: the FP8 GEMM runs the TMA epilogue only: 16-byte-aligned bf16 output, bias, "
                      "residual and GELU' input (no GELU pre-activation together with an epilogue input), or a plain "
                      "fp32 output\n");
      return -1;
    }
#define PG_DISPATCH_FP8(FMT)                                                                          \
  switch (bn) {                                                                                       \
    case 128: return launch_cfg<128, false, false, true, FMT>(ta, tb, tal, em, args, max_ctas, stream); \
    case 64: return launch_cfg<64, false, false, true, FMT>(ta, tb, tal, em, args, max_ctas, stream);   \
    default: fprintf(stderr, "pipegoose_b200: FP8 block_n must be 64 or 128, got %d\n", bn); return -1; \
  }
    if (d->fmt == FMT_E4M3) {
      PG_DISPATCH_FP8(FMT_E4M3)
    } else {
      PG_DISPATCH_FP8(FMT_E5M2)
    }
#undef PG_DISPATCH_FP8
  }

#define PG_DISPATCH_BN(AMN, BMN, EPI)                                                                    \
  switch (bn) {                                                                                          \
    case 256: return launch_cfg<256, AMN, BMN, EPI>(ta, tb, tal, em, args, max_ctas, stream);             \
    case 192: return launch_cfg<192, AMN, BMN, EPI>(ta, tb, tal, em, args, max_ctas, stream);             \
    case 128: return launch_cfg<128, AMN, BMN, EPI>(ta, tb, tal, em, args, max_ctas, stream);             \
    case 64: return launch_cfg<64, AMN, BMN, EPI>(ta, tb, tal, em, args, max_ctas, stream);               \
    default: fprintf(stderr, "pipegoose_b200: bad block_n %d\n", bn); return -1;                         \
  }
#define PG_DISPATCH_EPI(AMN, BMN) \
  if (tma_epi) {                  \
    PG_DISPATCH_BN(AMN, BMN, true) \
  } else {                        \
    PG_DISPATCH_BN(AMN, BMN, false) \
  }
  if (!d->a_mn && !d->b_mn) {
    PG_DISPATCH_EPI(false, false)
  } else if (!d->a_mn && d->b_mn) {
    PG_DISPATCH_EPI(false, true)
  } else if (d->a_mn && d->b_mn) {
    PG_DISPATCH_EPI(true, true)
  } else {
    PG_DISPATCH_EPI(true, false)
  }
#undef PG_DISPATCH_EPI
#undef PG_DISPATCH_BN
}
