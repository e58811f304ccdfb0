// Collective kernels over NVLink peer mappings (NVSwitch: every peer at full bandwidth, so all
// of these are direct all-to-all patterns, no rings):
//   rs_reduce      second half of GEMM->reduce-scatter: sum the T staged partial tiles (+bias,
//                  +residual) once every source's arrival counter says its tiles landed
//   allreduce_f32  data-parallel gradient bucket: two-shot (reduce-scatter by pulling peers'
//                  slices, then all-gather by pushing the reduced slice), fused with the 1/dp
//                  scale; reduce_scatter_only leaves rank r with slice r (ZeRO-1)
//   allgather_bf16 ZeRO-1 parameter all-gather: push my updated bf16 slices to every peer
//   barrier_peers  flag barrier (release/acquire at system scope)
// plus the cudaIpc-based symmetric allocation helpers.
#include "launch.h"
#include "ptx.cuh"
#include <cstdio>
#include <cstring>

namespace pg {

__global__ void __launch_bounds__(256) rs_reduce_kernel(
    const __nv_bfloat16* __restrict__ staging, int num_src, int64_t src_stride,
    const uint32_t* __restrict__ arrive_ctr, uint32_t expected, const __nv_bfloat16* __restrict__ bias,
    const __nv_bfloat16* __restrict__ residual, __nv_bfloat16* __restrict__ out, int rows, int cols) {
  if (threadIdx.x == 0) {
    for (int s = 0; s < num_src; ++s) spin_until_ge(arrive_ctr + s, expected, 10);
  }
  __syncthreads();
  const int64_t nvec = static_cast<int64_t>(rows) * cols / 8;
  const int cvec = cols / 8;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int s = 0; s < num_src; ++s) {
      const uint4 v = ld_global_v4(staging + s * src_stride + i * 8);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(w[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
    if (bias != nullptr) {
      const uint4 v = ld_global_nc_v4(bias + (i % cvec) * 8);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(w[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
    if (residual != nullptr) {
      const uint4 v = ld_global_nc_v4(residual + i * 8);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(w[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
    st_global_v4(out + i * 8, make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                                         pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7])));
  }
}

struct PeerPtrs {
  float* buf[PG_MAX_PEERS];
  uint32_t* flag[PG_MAX_PEERS];
};

// Reduce-scatter without a GEMM in front (vocab-parallel embedding: every rank holds a partial [T * rows, cols] matrix):
// row block c goes to rank c's staging slot of this source, then this CTA bumps rank c's arrival counter — the same
// protocol the GEMM -> reduce-scatter epilogue speaks, so the owner's rs_reduce kernel consumes both.
struct RsPushArgs {
  __nv_bfloat16* out_peer[PG_MAX_PEERS];
  uint32_t* arrive_ctr[PG_MAX_PEERS];
};
__global__ void __launch_bounds__(256) rs_push_kernel(const __nv_bfloat16* __restrict__ x, RsPushArgs a, int num_chunks,
                                                      int first_chunk, int64_t chunk_elems) {
  const int64_t nvec = chunk_elems / 8;
  for (int i = 0; i < num_chunks; ++i) {
    int c = first_chunk + i;
    if (c >= num_chunks) c -= num_chunks;
    const __nv_bfloat16* src = x + c * chunk_elems;
    __nv_bfloat16* dst = a.out_peer[c];
    for (int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec;
         v += static_cast<int64_t>(gridDim.x) * blockDim.x)
      st_global_v4(dst + v * 8, ld_global_nc_v4(src + v * 8));
    __syncthreads();
    if (threadIdx.x == 0) {
      fence_acq_rel_sys();
      red_add_release_sys(a.arrive_ctr[c], 1u);
    }
  }
}

// flag layout per rank: flags[phase * PG_MAX_PEERS + src]
PG_DEVICE void peer_barrier(const PeerPtrs& p, int world, int rank, uint32_t value, int phase) {
  // executed by one block; thread t < world signals peer t, then waits for peer t's signal
  if (threadIdx.x < world) {
    fence_acq_rel_sys();
    st_release_sys(p.flag[threadIdx.x] + phase * PG_MAX_PEERS + rank, value);
    spin_until_ge(p.flag[rank] + phase * PG_MAX_PEERS + threadIdx.x, value, 11 + phase);
  }
}

// Two-shot all-reduce (average) of buf[offset : offset+n) in place on every rank.
// grid-wide phases are separated by a device-wide counter (cooperative-free: all CTAs resident).
template <int kU>
__device__ __forceinline__ void allreduce_f32_body(const PeerPtrs& p, float* __restrict__ mc, int world, int rank,
                                                   int64_t offset, int64_t n, int64_t bucket_elems, float scale,
                                                   int rs_only, uint32_t epoch, uint32_t* __restrict__ grid_ctr) {
  // phase 0: everyone's bucket is complete locally (kernel boundary) -> cross-rank barrier
  if (blockIdx.x == 0) peer_barrier(p, world, rank, epoch, 0);
  // release the other CTAs of this rank
  __syncthreads();
  if (threadIdx.x == 0) {
    if (blockIdx.x == 0) {
      __threadfence();
      atomicExch(grid_ctr, epoch);
    } else {
      spin_until_ge(grid_ctr, epoch, 13);
    }
  }
  __syncthreads();
  // [offset, offset + n) is a run of buckets of bucket_elems elements (the last one may be shorter; every length is a
  // multiple of world * 4): ONE launch, one barrier pair, reduces them all — each bucket slice-wise, so that the ZeRO-1
  // ownership (rank r owns slice r of every bucket) is the same as with one launch per bucket
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t b0 = 0; b0 < n; b0 += bucket_elems) {
  const int64_t seg = min(bucket_elems, n - b0) / world;
  const int64_t my0 = offset + b0 + rank * seg;
  const int64_t nvec = seg / 4;
  // reduce my slice: pull the same slice from every peer.  kU independent 16-byte loads per thread per
  // peer are issued before any is consumed (NVLink latency ~2 us: bytes in flight, not threads, set the rate)
  if (mc != nullptr) {
    // NVLS: ONE multimem.ld_reduce per 16 bytes returns the sum over all replicas (reduced inside the NVSwitch, 1/world
    // of the bytes of a pull from every peer cross this GPU's links); the all-gather half is ONE multimem.st
    for (int64_t i0 = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i0 < nvec; i0 += stride * kU) {
      float4 v[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int64_t i = i0 + u * stride;
        v[u] = (i < nvec) ? multimem_ld_reduce_add_v4_f32(mc + my0 + i * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int64_t i = i0 + u * stride;
        if (i >= nvec) continue;
        float4 r = v[u];
        r.x *= scale; r.y *= scale; r.z *= scale; r.w *= scale;
        if (rs_only) {
          *reinterpret_cast<float4*>(p.buf[rank] + my0 + i * 4) = r;
        } else {
          multimem_st_v4_f32(mc + my0 + i * 4, r);
        }
      }
    }
  } else
  for (int64_t i0 = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i0 < nvec; i0 += stride * kU) {
    float4 acc[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
    for (int s = 0; s < world; ++s) {
      int src = rank + s;
      if (src >= world) src -= world;
      const float* base = p.buf[src] + my0;
      float4 v[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int64_t i = i0 + u * stride;
        v[u] = (i < nvec) ? *reinterpret_cast<const float4*>(base + i * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        acc[u].x += v[u].x; acc[u].y += v[u].y; acc[u].z += v[u].z; acc[u].w += v[u].w;
      }
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int64_t i = i0 + u * stride;
      if (i >= nvec) continue;
      float4 r = acc[u];
      r.x *= scale; r.y *= scale; r.z *= scale; r.w *= scale;
      if (rs_only) {
        *reinterpret_cast<float4*>(p.buf[rank] + my0 + i * 4) = r;
      } else {
#pragma unroll 1
        for (int s = 0; s < world; ++s) {
          int dst = rank + s;
          if (dst >= world) dst -= world;
          *reinterpret_cast<float4*>(p.buf[dst] + my0 + i * 4) = r;
        }
      }
    }
  }
  }  // buckets
  // phase 1: all ranks finished reading my buffer / writing into it
  __syncthreads();
  __shared__ uint32_t last;
  if (threadIdx.x == 0) {
    __threadfence_system();
    const uint32_t old = atomicAdd(grid_ctr + 1, 1u);
    last = (old == gridDim.x - 1) ? 1u : 0u;
    if (last) atomicExch(grid_ctr + 1, 0u);
  }
  __syncthreads();
  if (last) peer_barrier(p, world, rank, epoch, 1);
}

__global__ void __launch_bounds__(512) allreduce_f32_kernel(PeerPtrs p, float* __restrict__ mc, int world, int rank,
                                                            int64_t offset, int64_t n, int64_t bucket_elems, float scale,
                                                            int rs_only, uint32_t epoch, uint32_t* __restrict__ grid_ctr) {
  allreduce_f32_body<8>(p, mc, world, rank, offset, n, bucket_elems, scale, rs_only, epoch, grid_ctr);
}

// Small form: 128 threads x <= 64 registers and a few bytes of shared memory.  A persistent GEMM CTA holds its SM's
// whole register file (see gemm_sm90.cuh), so neither form runs next to a GEMM CTA: while backward computes, the
// GEMM grids are capped (pg_set_gemm_cta_cap, ops/comm.py) to leave the reducer's SMs free.
// 2 CTAs per SM x 128 threads x 4 x 16 B = 16 KB in flight per SM (2.4 MB over the chip: the NVLink bandwidth-delay product)
__global__ void __launch_bounds__(128, 8) /* <= 64 registers per thread */
    allreduce_f32_small_kernel(PeerPtrs p, float* __restrict__ mc, int world, int rank, int64_t offset, int64_t n,
                               int64_t bucket_elems, float scale, int rs_only, uint32_t epoch,
                               uint32_t* __restrict__ grid_ctr) {
  allreduce_f32_body<4>(p, mc, world, rank, offset, n, bucket_elems, scale, rs_only, epoch, grid_ctr);
}

struct PeerPtrsBf16 {
  __nv_bfloat16* buf[PG_MAX_PEERS];
  uint32_t* flag[PG_MAX_PEERS];
};

// push my slice of every region of the flat bf16 parameter buffer to all peers.  Regions: [0, head) and then
// [head + k*bucket, head + (k+1)*bucket) up to total; a region of length len is owned slice-wise (len / world each)
__global__ void __launch_bounds__(512) allgather_bf16_kernel(PeerPtrsBf16 p, __nv_bfloat16* __restrict__ mc, int world,
                                                             int rank, int64_t head_elems, int64_t bucket_elems,
                                                             int64_t total_elems, uint32_t epoch,
                                                             uint32_t* __restrict__ grid_ctr) {
  const int64_t nb = (total_elems - head_elems + bucket_elems - 1) / bucket_elems;
  for (int64_t b = (head_elems > 0 ? -1 : 0); b < nb; ++b) {
    const int64_t start = b < 0 ? 0 : head_elems + b * bucket_elems;
    const int64_t len = b < 0 ? head_elems : min(bucket_elems, total_elems - start);
    const int64_t seg = len / world;
    const int64_t my0 = start + rank * seg;
    const int64_t nvec = seg / 8;
    constexpr int kU = 4;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i0 = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i0 < nvec; i0 += stride * kU) {
      uint4 v[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int64_t i = i0 + u * stride;
        v[u] = (i < nvec) ? ld_global_v4(p.buf[rank] + my0 + i * 8) : make_uint4(0, 0, 0, 0);
      }
      if (mc != nullptr) {
        // NVLS: one store, the switch writes every replica (this rank's own copy included: same value)
#pragma unroll
        for (int u = 0; u < kU; ++u) {
          const int64_t i = i0 + u * stride;
          if (i < nvec) multimem_st_v4_b32(mc + my0 + i * 8, v[u]);
        }
        continue;
      }
#pragma unroll 1
      for (int s = 1; s < world; ++s) {
        int dst = rank + s;
        if (dst >= world) dst -= world;
#pragma unroll
        for (int u = 0; u < kU; ++u) {
          const int64_t i = i0 + u * stride;
          if (i < nvec) st_global_v4(p.buf[dst] + my0 + i * 8, v[u]);
        }
      }
    }
  }
  __syncthreads();
  __shared__ uint32_t last;
  if (threadIdx.x == 0) {
    __threadfence_system();
    const uint32_t old = atomicAdd(grid_ctr + 1, 1u);
    last = (old == gridDim.x - 1) ? 1u : 0u;
    if (last) atomicExch(grid_ctr + 1, 0u);
  }
  __syncthreads();
  if (last) {
    PeerPtrs q;
    for (int i = 0; i < PG_MAX_PEERS; ++i) q.flag[i] = p.flag[i];
    peer_barrier(q, world, rank, epoch, 1);
  }
}

// NVLS self-test: out[i] = sum over replicas of in[i] (multimem.ld_reduce), then mc_out[i] = that (multimem.st)
__global__ void multimem_selftest_kernel(const float* __restrict__ mc_in, float* __restrict__ mc_out, float* __restrict__ out,
                                         int64_t nvec) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float4 v = multimem_ld_reduce_add_v4_f32(mc_in + i * 4);
    *reinterpret_cast<float4*>(out + i * 4) = v;
    if (mc_out != nullptr) multimem_st_v4_f32(mc_out + i * 4, v);
  }
}

// GEMM -> reduce-scatter, NVLS form: every rank keeps its partial product [T * rows, cols] in its own symmetric
// buffer; rank r sums rows [r * rows, (r+1) * rows) of all replicas with multimem.ld_reduce (bf16x2, fp32 accumulation
// inside the switch) once every source's tiles of that block are complete (+ bias + residual)
__global__ void __launch_bounds__(256) rs_reduce_mc_kernel(
    const __nv_bfloat16* __restrict__ mc_partial, const uint32_t* __restrict__ arrive_ctr, int num_src, uint32_t expected,
    const __nv_bfloat16* __restrict__ bias, const __nv_bfloat16* __restrict__ residual, __nv_bfloat16* __restrict__ out,
    int rows, int cols) {
  if (threadIdx.x == 0) {
    for (int s = 0; s < num_src; ++s) spin_until_ge(arrive_ctr + s, expected, 14);
  }
  __syncthreads();
  const int64_t nvec = static_cast<int64_t>(rows) * cols / 8;
  const int cvec = cols / 8;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const uint4 v = multimem_ld_reduce_add_v4_bf16x2(mc_partial + i * 8);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    float acc[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      acc[2 * j] = f.x;
      acc[2 * j + 1] = f.y;
    }
    if (bias != nullptr) {
      const uint4 b = ld_global_nc_v4(bias + (i % cvec) * 8);
      const uint32_t bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(bw[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
    if (residual != nullptr) {
      const uint4 r = ld_global_nc_v4(residual + i * 8);
      const uint32_t rw[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(rw[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
    st_global_v4(out + i * 8, make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                                         pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7])));
  }
}

__global__ void barrier_kernel(PeerPtrs p, int world, int rank, uint32_t epoch) {
  peer_barrier(p, world, rank, epoch, 0);
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

extern "C" int pg_rs_reduce(const void* staging, int num_src, int64_t src_stride_elems,
                            const uint32_t* arrive_ctr, uint32_t expected, const void* bias,
                            const void* residual, void* out, int rows, int cols, cudaStream_t s) {
  if (rows == 0) return 0;
  if (cols % 8 != 0) return -1;
  const int64_t nvec = static_cast<int64_t>(rows) * cols / 8;
  int blocks = static_cast<int>((nvec + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  rs_reduce_kernel<<<blocks, 256, 0, s>>>((const __nv_bfloat16*)staging, num_src, src_stride_elems,
                                          arrive_ctr, expected, (const __nv_bfloat16*)bias,
                                          (const __nv_bfloat16*)residual, (__nv_bfloat16*)out, rows, cols);
  PG_CHECK_LAUNCH("rs_reduce");
  return 0;
}

// grid_ctr: two uint32 in LOCAL memory right after the flag area: peer_flags[rank] + 2*PG_MAX_PEERS
extern "C" int pg_allreduce_f32(float* const* peer_bufs, float* mc_buf, int world, int rank, int64_t offset_elems,
                                int64_t n, int64_t bucket_elems, float scale, int reduce_scatter_only,
                                uint32_t* const* peer_flags, uint32_t epoch, int blocks, cudaStream_t s) {
  if (n == 0) return 0;
  if (bucket_elems <= 0 || bucket_elems > n) bucket_elems = n;
  if (bucket_elems % (world * 4) != 0 || (n % bucket_elems) % (world * 4) != 0) return -1;
  PeerPtrs p;
  memset(&p, 0, sizeof(p));
  for (int i = 0; i < world; ++i) {
    p.buf[i] = peer_bufs[i];
    p.flag[i] = peer_flags[i];
  }
  // overlapped with backward: a handful of CTAs on the SMs the persistent GEMMs leave free (pg_set_gemm_cta_cap);
  // after backward (nothing else runs): enough CTAs to keep ~3 MB in flight over NVLink
  if (blocks < 0) {  // small form: -blocks CTAs of 128 threads
    allreduce_f32_small_kernel<<<-blocks, 128, 0, s>>>(p, mc_buf, world, rank, offset_elems, n, bucket_elems, scale,
                                                       reduce_scatter_only, epoch, peer_flags[rank] + 2 * PG_MAX_PEERS);
    PG_CHECK_LAUNCH("allreduce_f32_small");
    return 0;
  }
  if (blocks == 0) blocks = 24;
  allreduce_f32_kernel<<<blocks, 512, 0, s>>>(p, mc_buf, world, rank, offset_elems, n, bucket_elems, scale,
                                              reduce_scatter_only, epoch,
                                              peer_flags[rank] + 2 * PG_MAX_PEERS);
  PG_CHECK_LAUNCH("allreduce_f32");
  return 0;
}

extern "C" int pg_allgather_bf16(void* const* peer_bufs, void* mc_buf, int world, int rank, int64_t head_elems,
                                 int64_t bucket_elems, int64_t total_elems,
                                 uint32_t* const* peer_flags, uint32_t epoch, cudaStream_t s) {
  if (bucket_elems <= 0 || head_elems % (world * 8) != 0) return -1;
  PeerPtrsBf16 p;
  memset(&p, 0, sizeof(p));
  for (int i = 0; i < world; ++i) {
    p.buf[i] = (__nv_bfloat16*)peer_bufs[i];
    p.flag[i] = peer_flags[i];
  }
  const int blocks = 32;
  allgather_bf16_kernel<<<blocks, 512, 0, s>>>(p, (__nv_bfloat16*)mc_buf, world, rank, head_elems, bucket_elems,
                                               total_elems, epoch, peer_flags[rank] + 2 * PG_MAX_PEERS);
  PG_CHECK_LAUNCH("allgather_bf16");
  return 0;
}

extern "C" int pg_rs_push(const void* x, int num_chunks, int first_chunk, int64_t chunk_elems, void* const* out_peer,
                          uint32_t* const* arrive_ctr, int blocks, cudaStream_t s) {
  if (chunk_elems % 8 != 0 || num_chunks > PG_MAX_PEERS) return -1;
  RsPushArgs a;
  memset(&a, 0, sizeof(a));
  for (int i = 0; i < num_chunks; ++i) {
    a.out_peer[i] = (__nv_bfloat16*)out_peer[i];
    a.arrive_ctr[i] = arrive_ctr[i];
  }
  rs_push_kernel<<<blocks, 256, 0, s>>>((const __nv_bfloat16*)x, a, num_chunks, first_chunk, chunk_elems);
  PG_CHECK_LAUNCH("rs_push");
  return 0;
}

extern "C" int pg_multimem_selftest(const float* mc_in, float* mc_out, float* out, int64_t n, cudaStream_t s) {
  if (n % 4 != 0) return -1;
  multimem_selftest_kernel<<<64, 256, 0, s>>>(mc_in, mc_out, out, n / 4);
  PG_CHECK_LAUNCH("multimem_selftest");
  return 0;
}

extern "C" int pg_rs_reduce_mc(const void* mc_partial, const uint32_t* arrive_ctr, int num_src, uint32_t expected,
                               const void* bias, const void* residual, void* out, int rows, int cols, cudaStream_t s) {
  if (rows == 0) return 0;
  if (cols % 8 != 0) return -1;
  const int64_t nvec = static_cast<int64_t>(rows) * cols / 8;
  int blocks = static_cast<int>((nvec + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  rs_reduce_mc_kernel<<<blocks, 256, 0, s>>>((const __nv_bfloat16*)mc_partial, arrive_ctr, num_src, expected,
                                             (const __nv_bfloat16*)bias, (const __nv_bfloat16*)residual,
                                             (__nv_bfloat16*)out, rows, cols);
  PG_CHECK_LAUNCH("rs_reduce_mc");
  return 0;
}

extern "C" int pg_barrier_peers(uint32_t* const* peer_flags, int world, int rank, uint32_t epoch,
                                cudaStream_t s) {
  PeerPtrs p;
  memset(&p, 0, sizeof(p));
  for (int i = 0; i < world; ++i) p.flag[i] = peer_flags[i];
  barrier_kernel<<<1, 32, 0, s>>>(p, world, rank, epoch);
  PG_CHECK_LAUNCH("barrier_peers");
  return 0;
}

extern "C" int pg_symm_alloc(int64_t nbytes, void** ptr, void* handle64) {
  cudaError_t e = cudaMalloc(ptr, nbytes);
  if (e != cudaSuccess) {
    fprintf(stderr, "pipegoose_b200: symmetric cudaMalloc(%lld) failed: %s\n", (long long)nbytes, cudaGetErrorString(e));
    return -1;
  }
  cudaMemset(*ptr, 0, nbytes);
  cudaIpcMemHandle_t h;
  e = cudaIpcGetMemHandle(&h, *ptr);
  if (e != cudaSuccess) {
    fprintf(stderr, "pipegoose_b200: cudaIpcGetMemHandle failed: %s\n", cudaGetErrorString(e));
    return -1;
  }
  static_assert(sizeof(h) == 64, "ipc handle size");
  memcpy(handle64, &h, 64);
  return 0;
}

extern "C" int pg_symm_open(const void* handle64, void** ptr) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  cudaError_t e = cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    fprintf(stderr, "pipegoose_b200: cudaIpcOpenMemHandle failed: %s\n", cudaGetErrorString(e));
    return -1;
  }
  return 0;
}

extern "C" int pg_symm_close(void* ptr) { return cudaIpcCloseMemHandle(ptr) == cudaSuccess ? 0 : -1; }
extern "C" int pg_symm_free(void* ptr) { return cudaFree(ptr) == cudaSuccess ? 0 : -1; }
