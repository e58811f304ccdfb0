// Mixture-of-experts routing and NVLink all-to-all dispatch.
//
//   moe_route     one warp per token: fp32 gate (x . Wg + b) [* jitter], softmax, top-k, position of
//                 the token inside its expert's per-source capacity window (atomic counter), and the
//                 partial sums of the Switch load-balancing loss / router z-loss.
//   moe_dispatch  permute + all-to-all in one pass: every (token, k) that won a slot is copied straight
//                 into the owner rank's expert buffer through its NVLink peer mapping
//                 (row = expert_local * T*C + src_rank*C + pos), together with the return address
//                 (k*n + token) and the gate weight; the owner's per-expert arrival counters are
//                 bumped with a system-scope release so the expert GEMM (chunk = expert) can start on
//                 an expert as soon as all sources finished pushing.
// Combine is the epilogue of the last expert GEMM (EPI_SCATTER in gemm_sm90.cuh): each output row is
// scaled by its gate weight and stored into the source rank's combine buffer at the return address.
#include "launch.h"
#include "ptx.cuh"
#include <cstdio>

namespace pg {

constexpr int kMaxExperts = 64;
constexpr int kMaxTopK = 2;

__global__ void __launch_bounds__(256) moe_route_kernel(
    const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ wg,
    const __nv_bfloat16* __restrict__ bg, const float* __restrict__ jitter, int n, int h, int E, int top_k,
    int capacity, float* __restrict__ probs, int* __restrict__ topk_idx, float* __restrict__ topk_prob,
    int* __restrict__ pos, int* __restrict__ counts, float* __restrict__ prob_sum, float* __restrict__ zsum,
    float* __restrict__ lse_out) {
  extern __shared__ __nv_bfloat16 s_w[];  // [E, h]
  for (int i = threadIdx.x; i < E * h / 8; i += blockDim.x)
    reinterpret_cast<uint4*>(s_w)[i] = ld_global_nc_v4(wg + i * 8);
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  for (int t = blockIdx.x * warps_per_block + (threadIdx.x >> 5); t < n; t += gridDim.x * warps_per_block) {
    float acc[kMaxExperts / 4];  // E <= 16 handled in registers per lane; larger E loops below
    float logit[kMaxExperts];
    const __nv_bfloat16* xr = x + static_cast<size_t>(t) * h;
    for (int e0 = 0; e0 < E; e0 += kMaxExperts / 4) {
      const int ne = min(kMaxExperts / 4, E - e0);
#pragma unroll
      for (int j = 0; j < kMaxExperts / 4; ++j) acc[j] = 0.f;
      for (int c = lane; c < h / 8; c += 32) {
        const uint4 xv = ld_global_nc_v4(xr + c * 8);
        const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
        float xf[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(xw[j]);
          xf[2 * j] = f.x;
          xf[2 * j + 1] = f.y;
        }
#pragma unroll
        for (int j = 0; j < kMaxExperts / 4; ++j) {
          if (j < ne) {
            const uint4 wv = *reinterpret_cast<const uint4*>(s_w + static_cast<size_t>(e0 + j) * h + c * 8);
            const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float2 f = unpack_bf16x2(ww[q]);
              acc[j] += xf[2 * q] * f.x + xf[2 * q + 1] * f.y;
            }
          }
        }
      }
#pragma unroll
      for (int j = 0; j < kMaxExperts / 4; ++j) {
        const float s = warp_sum(acc[j]);
        if (j < ne) logit[e0 + j] = s;
      }
    }
    if (lane == 0) {
      float mx = -INFINITY;
      for (int e = 0; e < E; ++e) {
        float l = logit[e] + (bg ? __bfloat162float(bg[e]) : 0.f);
        if (jitter) l *= jitter[static_cast<size_t>(t) * E + e];
        logit[e] = l;
        mx = fmaxf(mx, l);
      }
      float se = 0.f;
      for (int e = 0; e < E; ++e) se += expf(logit[e] - mx);
      const float lse = mx + logf(se);
      atomicAdd(zsum, lse * lse);
      if (lse_out) lse_out[t] = lse;
      float p[kMaxExperts];
      for (int e = 0; e < E; ++e) {
        p[e] = expf(logit[e] - lse);
        probs[static_cast<size_t>(t) * E + e] = p[e];
        atomicAdd(&prob_sum[e], p[e]);
      }
      // A token whose probabilities are not finite (a NaN or +-inf input, weight or logit makes all of them NaN) is
      // dropped for every k: expert 0, weight 0, no slot, not counted.  Its NaN still reaches probs / lse / prob_sum /
      // zsum, and so the losses, as on the eager path.
      if (!isfinite(lse)) {
        for (int k = 0; k < top_k; ++k) {
          topk_idx[t * top_k + k] = 0;
          topk_prob[t * top_k + k] = 0.f;
          pos[t * top_k + k] = -1;
        }
        continue;
      }
      int chosen[kMaxTopK] = {-1, -1};
      for (int k = 0; k < top_k; ++k) {
        int best = -1;
        float bp = -1.f;
        for (int e = 0; e < E; ++e)
          if (e != chosen[0] && p[e] > bp) {
            bp = p[e];
            best = e;
          }
        chosen[k] = best;
        int slot = atomicAdd(&counts[best], 1);
        if (slot >= capacity) slot = -1;  // over capacity: dropped (passes through on the residual path)
        topk_idx[t * top_k + k] = best;
        topk_prob[t * top_k + k] = bp;
        pos[t * top_k + k] = slot;
      }
    }
  }
}

struct MoePeers {
  __nv_bfloat16* buf[PG_MAX_PEERS];  // expert input buffers [E_local * T * C, h]
  int* row_ret[PG_MAX_PEERS];        // return address per buffer row (k * n + token), -1 = empty
  float* row_scale[PG_MAX_PEERS];    // gate weight per buffer row
  uint32_t* arrive[PG_MAX_PEERS];    // per local expert arrival counters on the owner
};

// scale_by_prob: 0 = copy rows (forward dispatch of x); 1 = multiply rows by the gate prob
// (backward dispatch of dy: d(expert out) = p * dy)
__global__ void __launch_bounds__(256) moe_dispatch_kernel(
    const __nv_bfloat16* __restrict__ x, const int* __restrict__ topk_idx, const float* __restrict__ topk_prob,
    const int* __restrict__ pos, MoePeers peers, int n, int h, int top_k, int E_local, int T, int C, int my_rank,
    int scale_by_prob) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int total = n * top_k;
  for (int i = blockIdx.x * warps_per_block + (threadIdx.x >> 5); i < total; i += gridDim.x * warps_per_block) {
    const int slot = pos[i];
    if (slot < 0) continue;
    const int t = i / top_k, k = i - t * top_k;
    const int e = topk_idx[i];
    const int owner = e / E_local, el = e - owner * E_local;
    const int row = el * (T * C) + my_rank * C + slot;
    const float p = topk_prob[i];
    const __nv_bfloat16* src = x + static_cast<size_t>(t) * h;
    __nv_bfloat16* dst = peers.buf[owner] + static_cast<size_t>(row) * h;
    for (int c = lane; c < h / 8; c += 32) {
      uint4 v = ld_global_nc_v4(src + c * 8);
      if (scale_by_prob) {
        uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(w[j]);
          w[j] = pack_bf16x2(f.x * p, f.y * p);
        }
        v = make_uint4(w[0], w[1], w[2], w[3]);
      }
      st_global_v4(dst + c * 8, v);
    }
    if (lane == 0) {
      peers.row_ret[owner][row] = k * n + t;
      peers.row_scale[owner][row] = p;
    }
  }
  __syncthreads();
  if (threadIdx.x < T * E_local) {
    const int owner = threadIdx.x / E_local, el = threadIdx.x % E_local;
    fence_acq_rel_sys();
    red_add_release_sys(peers.arrive[owner] + el, 1u);
  }
}

// fill int32 buffer with a value / zero helpers for the per-step buffers
__global__ void fill_i32_kernel(int* p, int v, int64_t n) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
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

extern "C" int pg_moe_route(const void* x, const void* wg, const void* bg, const float* jitter, int n, int h, int E,
                            int top_k, int capacity, float* probs, int* topk_idx, float* topk_prob, int* pos,
                            int* counts, float* prob_sum, float* zsum, float* lse_out, cudaStream_t s) {
  if (n == 0) return 0;
  // top_k distinct experts must exist: with top_k > E the last picks would find no expert
  if (E < 1 || E > kMaxExperts || top_k < 1 || top_k > kMaxTopK || top_k > E || h % 8 != 0) return -1;
  const size_t smem = static_cast<size_t>(E) * h * 2;
  if (smem > 200 * 1024) return -1;
  static bool set = false;
  if (!set) {
    cudaFuncSetAttribute(moe_route_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    set = true;
  }
  int blocks = (n + 7) / 8;
  if (blocks > 132 * 2) blocks = 132 * 2;
  moe_route_kernel<<<blocks, 256, smem, s>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)wg,
                                             (const __nv_bfloat16*)bg, jitter, n, h, E, top_k, capacity, probs,
                                             topk_idx, topk_prob, pos, counts, prob_sum, zsum, lse_out);
  PG_CHECK_LAUNCH("moe_route");
  return 0;
}

extern "C" int pg_moe_dispatch(const void* x, const int* topk_idx, const float* topk_prob, const int* pos,
                               void* const* peer_buf, int* const* peer_row_ret, float* const* peer_row_scale,
                               uint32_t* const* peer_arrive, int n, int h, int top_k, int E_local, int T, int C,
                               int my_rank, int scale_by_prob, int blocks, cudaStream_t s) {
  MoePeers p;
  for (int i = 0; i < PG_MAX_PEERS; ++i) {
    p.buf[i] = nullptr; p.row_ret[i] = nullptr; p.row_scale[i] = nullptr; p.arrive[i] = nullptr;
  }
  for (int i = 0; i < T; ++i) {
    p.buf[i] = (__nv_bfloat16*)peer_buf[i];
    p.row_ret[i] = peer_row_ret[i];
    p.row_scale[i] = peer_row_scale[i];
    p.arrive[i] = peer_arrive[i];
  }
  if (T * E_local > 256) return -1;
  moe_dispatch_kernel<<<blocks, 256, 0, s>>>((const __nv_bfloat16*)x, topk_idx, topk_prob, pos, p, n, h, top_k,
                                             E_local, T, C, my_rank, scale_by_prob);
  PG_CHECK_LAUNCH("moe_dispatch");
  return 0;
}

extern "C" int pg_fill_i32(int* p, int v, int64_t n, cudaStream_t s) {
  if (n == 0) return 0;
  fill_i32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p, v, n);
  PG_CHECK_LAUNCH("fill_i32");
  return 0;
}
