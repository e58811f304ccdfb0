// Swapping KV-cache pages between the device pools and a pinned host pool (continuous batching with preemption),
// sm_90a.
//
//   k_pools / v_pools : [layers, pages, H, 64, D] bf16 or e4m3 codes        pairs : int32 [n, 2] (pool page, host slot)
//   k_scales / v_scales : fp32 [layers, pages, H, 64] (FP8 pools only)
//   host_kv : [slots, layers, 2, H, 64, D], the pools' dtype          host_scales : fp32 [slots, layers, 2, H, 64]
//
// A host slot is one contiguous region: every layer's K then V of one page, so a page crosses PCIe as one stream.  The
// kernel reads and writes the pinned host pool directly, through its device pointer (zero-copy), so one launch moves
// every pair, layer, K and V and the scales, with no copy-engine call per page.
//
// The copy is one flat index space of 16-byte words: first the data words, ((pair * layers + layer) * 2 + kv) * cv + c
// with cv = H * 64 * D * elem / 16 words per (page, layer, K|V), then likewise the scale words (sv = H * 64 * 4 / 16).
// Consecutive threads take consecutive words, which are consecutive on both sides (a pool page's K of one layer is
// contiguous too), so every access is a coalesced 16-byte one.  A thread loads kSwapUnroll words, one block stride
// apart, into registers before it stores any: loads from host memory take a PCIe round trip each, so several are kept
// in flight per thread.
#include "launch.h"
#include "pdl_launch.cuh"
#include "ptx.cuh"
#include <cstdio>

namespace pg {

constexpr int kSwapThreads = 256;
constexpr int kSwapUnroll = 8;

struct SwapArgs {
  const int* pairs;
  uint4* k_pools;
  uint4* v_pools;
  uint4* k_scales;         // nullptr: bf16 pools
  uint4* v_scales;
  uint4* host_kv;
  uint4* host_scales;
  long long data_words;    // n * layers * 2 * cv
  long long total_words;   // data_words + n * layers * 2 * sv (FP8 pools)
  int layers;
  int pages;
  int cv;
  int sv;
};

// Device-side and host-side address of word i.
__device__ __forceinline__ void swap_word(const SwapArgs& a, long long i, uint4*& dev, uint4*& host) {
  const bool data = i < a.data_words;
  const long long j = data ? i : i - a.data_words;
  const int w = data ? a.cv : a.sv;
  const int c = static_cast<int>(j % w);
  long long r = j / w;
  const int kv = static_cast<int>(r & 1);
  r >>= 1;
  const int layer = static_cast<int>(r % a.layers);
  const int p = static_cast<int>(r / a.layers);
  const int page = __ldg(a.pairs + 2 * p);
  const int slot = __ldg(a.pairs + 2 * p + 1);
  uint4* pool = data ? (kv ? a.v_pools : a.k_pools) : (kv ? a.v_scales : a.k_scales);
  dev = pool + (static_cast<size_t>(layer) * a.pages + page) * w + c;
  host = (data ? a.host_kv : a.host_scales) + ((static_cast<size_t>(slot) * a.layers + layer) * 2 + kv) * w + c;
}

template <bool TO_HOST>
__global__ void __launch_bounds__(kSwapThreads) paged_kv_swap_kernel(const SwapArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const long long base = static_cast<long long>(blockIdx.x) * kSwapThreads * kSwapUnroll + threadIdx.x;
  uint4 v[kSwapUnroll];
  uint4* dst[kSwapUnroll];
#pragma unroll
  for (int u = 0; u < kSwapUnroll; ++u) {
    const long long i = base + static_cast<long long>(u) * kSwapThreads;
    dst[u] = nullptr;
    if (i < a.total_words) {
      uint4 *dev, *host;
      swap_word(a, i, dev, host);
      v[u] = TO_HOST ? *dev : *host;
      dst[u] = TO_HOST ? host : dev;
    }
  }
#pragma unroll
  for (int u = 0; u < kSwapUnroll; ++u)
    if (dst[u] != nullptr) *dst[u] = v[u];
}

}  // namespace pg

using namespace pg;

extern "C" int pg_paged_kv_swap(const int* pairs, void* k_pools, void* v_pools, float* k_scales, float* v_scales,
                                void* host_kv, float* host_scales, int n, int layers, int pages, int H, int row_bytes,
                                int to_host, cudaStream_t s) {
  if (n < 0 || layers < 1 || pages < 1 || H < 1 || row_bytes % 16 != 0 || (k_scales == nullptr) != (v_scales == nullptr) ||
      (k_scales == nullptr) != (host_scales == nullptr))
    return -1;
  if (n == 0) return 0;
  SwapArgs a;
  a.pairs = pairs;
  a.k_pools = static_cast<uint4*>(k_pools);
  a.v_pools = static_cast<uint4*>(v_pools);
  a.k_scales = reinterpret_cast<uint4*>(k_scales);
  a.v_scales = reinterpret_cast<uint4*>(v_scales);
  a.host_kv = static_cast<uint4*>(host_kv);
  a.host_scales = reinterpret_cast<uint4*>(host_scales);
  a.layers = layers;
  a.pages = pages;
  a.cv = H * 64 * (row_bytes / 16);
  a.sv = H * 64 * 4 / 16;
  a.data_words = static_cast<long long>(n) * layers * 2 * a.cv;
  a.total_words = a.data_words + (k_scales != nullptr ? static_cast<long long>(n) * layers * 2 * a.sv : 0);
  const long long per_block = static_cast<long long>(kSwapThreads) * kSwapUnroll;
  const dim3 grid(static_cast<unsigned>((a.total_words + per_block - 1) / per_block)), block(kSwapThreads);
  const cudaError_t e = to_host ? launch_pdl(paged_kv_swap_kernel<true>, grid, block, 0, s, a)
                                : launch_pdl(paged_kv_swap_kernel<false>, grid, block, 0, s, a);
  if (e != cudaSuccess || cudaGetLastError() != cudaSuccess) {
    fprintf(stderr, "pipegoose_b200: paged_kv_swap launch failed: %s\n", cudaGetErrorString(e));
    return -1;
  }
  return 0;
}
