// Per-tensor FP8 casts of the FP8 linear layers (current scaling: the scale comes from the tensor being cast, on the
// device, with no host sync).  The format, defined by ops.kernels.fp8_quantize_reference:
//   amax = max |x|,  fmax = 448 (e4m3) or 57344 (e5m2)
//   scale = min(fmax / amax, FLT_MAX) (IEEE division; 1 when amax = 0),  code = rn_satfinite(x * scale)
//   scale_inv = amax / fmax (1 when amax = 0, NaN when amax is not finite)
// so that x ~ code * scale_inv.  A non-finite amax makes scale_inv NaN instead of saturating: an inf or NaN in a
// gradient reaches the gradient norm through the GEMMs that use its codes.
//   fp8_amax_kernel : amax of bf16 [R, C] into an fp32 device scalar, by atomic max on the bits of |x| (bf16 |x| orders
//                     like its bit pattern, NaN above inf), so the result does not depend on the order.
//   fp8_cast_kernel : one 64 x 64 tile per block; writes each of codes [R, C], transposed codes [C, R] (staged through
//                     shared memory, 16-byte stores when R % 16 == 0), scale_inv, and the fp32 column sums of x added
//                     into colsum (the bias gradient of a dY), each only when its pointer is set.
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cfloat>

#include "launch.h"
#include "ptx.cuh"

namespace pg {

constexpr int kCastTile = 64;
constexpr int kCastThreads = 256;
constexpr int kCastLd = kCastTile + 4;  // bytes per staged code row: 4-byte aligned, rows 0 / 16 / 32 / 48 spread

__global__ void __launch_bounds__(256) fp8_amax_kernel(const uint4* __restrict__ x, int64_t nvec,
                                                       unsigned* __restrict__ amax_bits) {
  unsigned m = 0;  // two bf16 |x| bit patterns, max per halfword
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const uint4 v = __ldg(x + i);
    m = __vmaxu2(m, v.x & 0x7FFF7FFFu);
    m = __vmaxu2(m, v.y & 0x7FFF7FFFu);
    m = __vmaxu2(m, v.z & 0x7FFF7FFFu);
    m = __vmaxu2(m, v.w & 0x7FFF7FFFu);
  }
  unsigned r = max(m & 0xFFFFu, m >> 16);
  r = __reduce_max_sync(0xffffffffu, r);
  __shared__ unsigned s_m[8];
  if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = r;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < static_cast<int>(blockDim.x >> 5); ++w) r = max(r, s_m[w]);
    atomicMax(amax_bits, r << 16);  // the fp32 bits of the bf16 value
  }
}

template <bool E5M2>
PG_DEVICE uint16_t cvt_fp8x2(float lo, float hi) {
  return __nv_cvt_float2_to_fp8x2(make_float2(lo, hi), __NV_SATFINITE, E5M2 ? __NV_E5M2 : __NV_E4M3);
}

template <bool E5M2>
__global__ void __launch_bounds__(kCastThreads) fp8_cast_kernel(const __nv_bfloat16* __restrict__ x, int R, int C,
                                                                const float* __restrict__ amax_p, uint8_t* codes,
                                                                uint8_t* codes_t, float* scale_inv, float* colsum) {
  constexpr float kFmax = E5M2 ? 57344.0f : 448.0f;
  __shared__ __align__(16) uint8_t tile[kCastTile * kCastLd];
  __shared__ float part[8][kCastTile];
  const float amax = *amax_p;
  float scale = 1.0f;
  if (amax != 0.0f) scale = fminf(__fdiv_rn(kFmax, amax), FLT_MAX);
  if (scale_inv != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0)
    *scale_inv = amax == 0.0f ? 1.0f : (isfinite(amax) ? __fdiv_rn(amax, kFmax) : __int_as_float(0x7fffffff));

  const int r0 = blockIdx.y * kCastTile;
  const int c0 = blockIdx.x * kCastTile;
  const int t = threadIdx.x;
  const int g = t & 7;  // 8-column group of the tile
  float cs[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) cs[j] = 0.f;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = (t >> 3) + 32 * h;
    const int row = r0 + r, col = c0 + 8 * g;
    uint2 cw = make_uint2(0, 0);
    if (row < R && col < C) {  // C % 8 == 0: a group is whole or absent
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * C + col));
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      uint16_t p[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(w[j]);
        cs[2 * j] += f.x;
        cs[2 * j + 1] += f.y;
        p[j] = cvt_fp8x2<E5M2>(f.x * scale, f.y * scale);
      }
      cw = make_uint2(p[0] | (static_cast<uint32_t>(p[1]) << 16), p[2] | (static_cast<uint32_t>(p[3]) << 16));
      if (codes != nullptr) *reinterpret_cast<uint2*>(codes + static_cast<size_t>(row) * C + col) = cw;
    }
    uint32_t* st = reinterpret_cast<uint32_t*>(tile + r * kCastLd + 8 * g);
    st[0] = cw.x;
    st[1] = cw.y;
  }
  if (colsum != nullptr) {
    // lanes l, l + 8, l + 16, l + 24 of a warp hold the same columns: fold them, then the 8 warps in fixed order
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      cs[j] += __shfl_xor_sync(0xffffffffu, cs[j], 8);
      cs[j] += __shfl_xor_sync(0xffffffffu, cs[j], 16);
    }
    if ((t & 31) < 8) {
#pragma unroll
      for (int j = 0; j < 8; ++j) part[t >> 5][8 * g + j] = cs[j];
    }
  }
  __syncthreads();
  if (colsum != nullptr && t < kCastTile && c0 + t < C) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += part[w][t];
    atomicAdd(colsum + c0 + t, s);
  }
  if (codes_t != nullptr) {
    // transposed row c0 + c (a column of x), rows r0 + 16 q .. r0 + 16 q + 15 of x: 4 threads per 64-byte segment
    const int c = t >> 2, q = t & 3;
    if (c0 + c < C) {
      uint32_t w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint8_t* src = tile + (16 * q + 4 * i) * kCastLd + c;
        w[i] = src[0] | (src[kCastLd] << 8) | (src[2 * kCastLd] << 16) | (static_cast<uint32_t>(src[3 * kCastLd]) << 24);
      }
      const int rr = r0 + 16 * q;
      uint8_t* dst = codes_t + static_cast<size_t>(c0 + c) * R + rr;
      if ((R & 15) == 0) {
        if (rr < R) *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
      } else {
        for (int i = 0; i < 16 && rr + i < R; ++i) dst[i] = static_cast<uint8_t>(w[i >> 2] >> (8 * (i & 3)));
      }
    }
  }
}

}  // namespace pg

using namespace pg;

extern "C" int pg_fp8_amax(const void* x, int64_t n, float* amax, cudaStream_t s) {
  if ((n & 7) != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0) return -1;
  cudaMemsetAsync(amax, 0, sizeof(float), s);
  const int64_t nvec = n / 8;
  if (nvec > 0) {
    const int64_t want = (nvec + kCastThreads - 1) / kCastThreads;
    const int blocks = static_cast<int>(want < 1024 ? want : 1024);
    fp8_amax_kernel<<<blocks, kCastThreads, 0, s>>>(reinterpret_cast<const uint4*>(x), nvec,
                                                    reinterpret_cast<unsigned*>(amax));
  }
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int pg_fp8_cast(const void* x, int R, int C, int e5m2, const float* amax, void* codes, void* codes_t,
                           float* scale_inv, float* colsum, cudaStream_t s) {
  if (R < 0 || C < 0 || (C & 7) != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0 ||
      (reinterpret_cast<uintptr_t>(codes) & 7) != 0 || (reinterpret_cast<uintptr_t>(codes_t) & 15) != 0)
    return -1;
  if (R == 0 || C == 0) {
    if (scale_inv == nullptr) return 0;
    R = C = 0;  // still write scale_inv
  }
  const dim3 grid(R == 0 ? 1 : (C + kCastTile - 1) / kCastTile, R == 0 ? 1 : (R + kCastTile - 1) / kCastTile);
  auto* xb = reinterpret_cast<const __nv_bfloat16*>(x);
  auto* cp = reinterpret_cast<uint8_t*>(codes);
  auto* ct = reinterpret_cast<uint8_t*>(codes_t);
  if (e5m2)
    fp8_cast_kernel<true><<<grid, kCastThreads, 0, s>>>(xb, R, C, amax, cp, ct, scale_inv, colsum);
  else
    fp8_cast_kernel<false><<<grid, kCastThreads, 0, s>>>(xb, R, C, amax, cp, ct, scale_inv, colsum);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
