// Memory-bound kernels of the training step: LayerNorm (fwd/bwd, optionally fused with the
// embedding gather), bias-gradient column sums, embedding backward, vocab-parallel
// cross-entropy (stats / finalize+dlogits), fused Adam on flat fp32 shards, grad utilities.
// All bf16 I/O is 16-byte vectorised; statistics and accumulation are fp32.
#include "grad_rs.cuh"
#include "launch.h"
#include "pdl_launch.cuh"
#include "ptx.cuh"
#include <cstdio>
#include <cstring>

namespace pg {

constexpr int kMaxChunks = 32;  // 16B chunks per lane -> rows up to 32*32*8 = 8192 elements

// ---------------------------------------------------------------------------------------------
// LayerNorm forward: one warp per row.  src row = x[row] or, when ids != nullptr, table[ids[row]]
// (embedding gather fused with word_embeddings_layernorm); rows whose id falls outside
// [vocab_start, vocab_end) read as zero (vocab-parallel embedding).
// ---------------------------------------------------------------------------------------------
template <int CH>
__global__ void __launch_bounds__(256) layernorm_fwd_kernel(
    const __nv_bfloat16* __restrict__ x, const int64_t* __restrict__ ids, int vocab_start,
    int vocab_end, const __nv_bfloat16* __restrict__ gamma, const __nv_bfloat16* __restrict__ beta,
    __nv_bfloat16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out,
    int rows, int h, float eps, int apply_ln) {
  pdl_launch_dependents();
  pdl_wait();  // before any exit: a kernel that completes must imply its predecessors completed
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const int nchunks = h >> 3;
  const __nv_bfloat16* src = x + static_cast<size_t>(warp) * h;
  bool zero_row = false;
  if (ids != nullptr) {
    const int64_t id = ids[warp];
    if (id < vocab_start || id >= vocab_end) zero_row = true;
    src = x + static_cast<size_t>(id - vocab_start) * h;
  }
  uint4 v[CH];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks && !zero_row) {
      v[i] = ld_global_nc_v4(src + c * 8);
      const uint32_t w[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(w[j]);
        sum += f.x + f.y;
      }
    } else {
      v[i] = make_uint4(0, 0, 0, 0);
    }
  }
  __nv_bfloat16* dst = y + static_cast<size_t>(warp) * h;
  if (!apply_ln) {
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int c = lane + 32 * i;
      if (c < nchunks) st_global_v4(dst + c * 8, v[i]);
    }
    return;
  }
  sum = warp_sum(sum);
  const float mean = sum / h;
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      const uint32_t w[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(w[j]);
        var += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
      }
    }
  }
  var = warp_sum(var) / h;
  const float rstd = rsqrtf(var + eps);
  if (lane == 0) {
    if (mean_out) mean_out[warp] = mean;
    if (rstd_out) rstd_out[warp] = rstd;
  }
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      const uint4 g = ld_global_nc_v4(gamma + c * 8);
      const uint4 b = ld_global_nc_v4(beta + c * 8);
      const uint32_t w[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
      const uint32_t gw[4] = {g.x, g.y, g.z, g.w};
      const uint32_t bw[4] = {b.x, b.y, b.z, b.w};
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(w[j]);
        const float2 gg = unpack_bf16x2(gw[j]);
        const float2 bb = unpack_bf16x2(bw[j]);
        o[j] = pack_bf16x2((f.x - mean) * rstd * gg.x + bb.x, (f.y - mean) * rstd * gg.y + bb.y);
      }
      st_global_v4(dst + c * 8, make_uint4(o[0], o[1], o[2], o[3]));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// LayerNorm backward, two kernels:
//   dx      : one warp per row; dx = rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat)) (+ dx_extra,
//             the residual-stream gradient that bypasses the LN)
//   dparams : column reduction  dgamma[n] += sum_m dy*xhat,  dbeta[n] += sum_m dy  straight into the
//             fp32 main-grad vectors (one atomic per column per block)
// ---------------------------------------------------------------------------------------------
template <int CH>
__global__ void __launch_bounds__(256) layernorm_bwd_dx_kernel(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
    const __nv_bfloat16* __restrict__ gamma, const float* __restrict__ mean,
    const float* __restrict__ rstd, const __nv_bfloat16* __restrict__ dx_extra,
    __nv_bfloat16* __restrict__ dx, int rows, int h) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int nchunks = h >> 3;
  const float mu = mean[row], rs = rstd[row];
  const __nv_bfloat16* dyr = dy + static_cast<size_t>(row) * h;
  const __nv_bfloat16* xr = x + static_cast<size_t>(row) * h;
  uint4 vdy[CH], vx[CH];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      vdy[i] = ld_global_nc_v4(dyr + c * 8);
      vx[i] = ld_global_nc_v4(xr + c * 8);
      const uint4 g = ld_global_nc_v4(gamma + c * 8);
      const uint32_t aw[4] = {vdy[i].x, vdy[i].y, vdy[i].z, vdy[i].w};
      const uint32_t bw[4] = {vx[i].x, vx[i].y, vx[i].z, vx[i].w};
      const uint32_t gw[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 d = unpack_bf16x2(aw[j]);
        const float2 xx = unpack_bf16x2(bw[j]);
        const float2 gg = unpack_bf16x2(gw[j]);
        const float g0 = d.x * gg.x, g1 = d.y * gg.y;
        s1 += g0 + g1;
        s2 += g0 * (xx.x - mu) * rs + g1 * (xx.y - mu) * rs;
      }
    }
  }
  s1 = warp_sum(s1) / h;
  s2 = warp_sum(s2) / h;
  __nv_bfloat16* dxr = dx + static_cast<size_t>(row) * h;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      const uint4 g = ld_global_nc_v4(gamma + c * 8);
      const uint32_t aw[4] = {vdy[i].x, vdy[i].y, vdy[i].z, vdy[i].w};
      const uint32_t bw[4] = {vx[i].x, vx[i].y, vx[i].z, vx[i].w};
      const uint32_t gw[4] = {g.x, g.y, g.z, g.w};
      uint32_t ew[4] = {0, 0, 0, 0};
      if (dx_extra != nullptr) {
        const uint4 ex = ld_global_nc_v4(dx_extra + static_cast<size_t>(row) * h + c * 8);
        ew[0] = ex.x; ew[1] = ex.y; ew[2] = ex.z; ew[3] = ex.w;
      }
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 d = unpack_bf16x2(aw[j]);
        const float2 xx = unpack_bf16x2(bw[j]);
        const float2 gg = unpack_bf16x2(gw[j]);
        const float2 e = unpack_bf16x2(ew[j]);
        const float a0 = rs * (d.x * gg.x - s1 - (xx.x - mu) * rs * s2) + e.x;
        const float a1 = rs * (d.y * gg.y - s1 - (xx.y - mu) * rs * s2) + e.y;
        o[j] = pack_bf16x2(a0, a1);
      }
      st_global_v4(dxr + c * 8, make_uint4(o[0], o[1], o[2], o[3]));
    }
  }
}

__global__ void __launch_bounds__(256) layernorm_bwd_params_kernel(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
    const float* __restrict__ mean, const float* __restrict__ rstd, float* __restrict__ dgamma,
    float* __restrict__ dbeta, int rows, int h, int rows_per_block) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[2][8][256];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int col0 = blockIdx.x * 256 + lane * 8;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(rows, r0 + rows_per_block);
  float dg[8] = {0, 0, 0, 0, 0, 0, 0, 0}, db[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col0 < h) {
    for (int r = r0 + wib; r < r1; r += 8) {
      const float mu = mean[r], rs = rstd[r];
      const uint4 a = ld_global_nc_v4(dy + static_cast<size_t>(r) * h + col0);
      const uint4 b = ld_global_nc_v4(x + static_cast<size_t>(r) * h + col0);
      const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
      const uint32_t bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 d = unpack_bf16x2(aw[j]);
        const float2 xx = unpack_bf16x2(bw[j]);
        dg[2 * j] += d.x * (xx.x - mu) * rs;
        dg[2 * j + 1] += d.y * (xx.y - mu) * rs;
        db[2 * j] += d.x;
        db[2 * j + 1] += d.y;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    red[0][wib][lane * 8 + j] = dg[j];
    red[1][wib][lane * 8 + j] = db[j];
  }
  __syncthreads();
  const int c = threadIdx.x;
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    s0 += red[0][w][c];
    s1 += red[1][w][c];
  }
  if (blockIdx.x * 256 + c < h) {
    atomicAdd(&dgamma[blockIdx.x * 256 + c], s0);
    atomicAdd(&dbeta[blockIdx.x * 256 + c], s1);
  }
}

// ---------------------------------------------------------------------------------------------
// column sum: out[n] += sum_m x[m, n]   (bias gradients into the fp32 main grad)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) colsum_kernel(const __nv_bfloat16* __restrict__ x, int ld,
                                                     float* __restrict__ out, int rows, int cols,
                                                     int rows_per_block) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[8][256];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int col0 = blockIdx.x * 256 + lane * 8;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(rows, r0 + rows_per_block);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col0 < cols) {
    for (int r = r0 + wib; r < r1; r += 8) {
      const uint4 v = ld_global_nc_v4(x + static_cast<size_t>(r) * ld + col0);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(w[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[wib][lane * 8 + j] = acc[j];
  __syncthreads();
  const int c = threadIdx.x;
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) s += red[w][c];
  if (blockIdx.x * 256 + c < cols) atomicAdd(&out[blockIdx.x * 256 + c], s);
}

// ---------------------------------------------------------------------------------------------
// embedding backward: dW[id - vocab_start, :] += dx[row, :]  (fp32 main grad, atomics)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) embedding_bwd_kernel(const __nv_bfloat16* __restrict__ dx,
                                                            const int64_t* __restrict__ ids,
                                                            float* __restrict__ dw, int rows, int h,
                                                            int vocab_start, int vocab_end, const PgGradRS grs) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const int64_t id = ids[warp];
  if (id < vocab_start || id >= vocab_end) return;
  float* dst = dw + static_cast<size_t>(id - vocab_start) * h;
  const __nv_bfloat16* src = dx + static_cast<size_t>(warp) * h;
  for (int c = lane; c < (h >> 3); c += 32) {
    const uint4 v = ld_global_nc_v4(src + c * 8);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    if (grs.world > 1) {
      // data-parallel reduce-scatter fused into the scatter-add: the row goes to the owner of its ZeRO-1 slice
      const float2 a = unpack_bf16x2(w[0]), b = unpack_bf16x2(w[1]), c2 = unpack_bf16x2(w[2]), d = unpack_bf16x2(w[3]);
      grs_add4(grs, dst + c * 8, make_float4(a.x, a.y, b.x, b.y));
      grs_add4(grs, dst + c * 8 + 4, make_float4(c2.x, c2.y, d.x, d.y));
      continue;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      atomicAdd(dst + c * 8 + 2 * j, f.x);
      atomicAdd(dst + c * 8 + 2 * j + 1, f.y);
    }
  }
}

// dst_local[i] += scale * src[i], added into the buffers of the ranks that own the ZeRO-1 slices (see PgGradRS):
// gradients that autograd delivered (or any torch-side gradient) join the in-kernel reduce-scatter here
template <bool SRC_F32>
__global__ void __launch_bounds__(256) grad_rs_accum_kernel(const void* __restrict__ src_, float* __restrict__ dst_local,
                                                            int64_t n, float scale, const PgGradRS grs) {
  const int64_t i4 = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i4 >= n) return;
  float f[4] = {0.f, 0.f, 0.f, 0.f};
  const int cnt = (n - i4) < 4 ? static_cast<int>(n - i4) : 4;
  if (SRC_F32) {
    const float* src = reinterpret_cast<const float*>(src_);
    for (int j = 0; j < cnt; ++j) f[j] = src[i4 + j] * scale;
  } else {
    const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(src_);
    for (int j = 0; j < cnt; ++j) f[j] = __bfloat162float(src[i4 + j]) * scale;
  }
  if (cnt == 4) {
    grs_add4(grs, dst_local + i4, make_float4(f[0], f[1], f[2], f[3]));
  } else {
    for (int j = 0; j < cnt; ++j) red_add_f32(grs_target(grs, dst_local + i4 + j), f[j]);
  }
}

// ---------------------------------------------------------------------------------------------
// vocab-parallel cross entropy, two kernels around one tiny cross-rank exchange.
//   ce_stats:    per row (max, sum exp(x - max), logit[target] if the target is local else 0)
//   ce_finalize: given the *global* (max, sumexp, target logit) per row: loss[row] and, in
//                place, dlogits = (softmax - onehot) * grad_scale   (ignore_index rows -> 0)
// One block per row, online softmax, bf16 logits read once per kernel.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512) ce_stats_kernel(const __nv_bfloat16* __restrict__ logits,
                                                       int ld, const int64_t* __restrict__ targets,
                                                       float* __restrict__ stats, int vocab_local,
                                                       int vocab_start) {
  const int row = blockIdx.x;
  const __nv_bfloat16* lr = logits + static_cast<size_t>(row) * ld;
  float m = -INFINITY, s = 0.f;
  const int nchunks = vocab_local >> 3;
  for (int c = threadIdx.x; c < nchunks; c += blockDim.x) {
    const uint4 v = ld_global_nc_v4(lr + c * 8);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    float f[8];
    float cm = -INFINITY;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = unpack_bf16x2(w[j]);
      f[2 * j] = t.x;
      f[2 * j + 1] = t.y;
      cm = fmaxf(cm, fmaxf(t.x, t.y));
    }
    if (cm == -INFINITY) continue;  // eight masked (-inf) logits, e.g. vocabulary padding: exp(-inf - -inf) would be NaN
    const float nm = fmaxf(m, cm);
    float add = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) add += __expf(f[j] - nm);
    s = s * __expf(m - nm) + add;
    m = nm;
  }
  for (int c = nchunks * 8 + threadIdx.x; c < vocab_local; c += blockDim.x) {  // tail
    const float f = __bfloat162float(lr[c]);
    if (f == -INFINITY) continue;
    const float nm = fmaxf(m, f);
    s = s * __expf(m - nm) + __expf(f - nm);
    m = nm;
  }
  __shared__ float sm[16], ss[16];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  float wm = warp_max(m);
  s = s * ((m == -INFINITY) ? 0.f : __expf(m - wm));
  s = warp_sum(s);
  if (lane == 0) {
    sm[wib] = wm;
    ss[wib] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float gm = -INFINITY;
    const int nw = blockDim.x >> 5;
    for (int i = 0; i < nw; ++i) gm = fmaxf(gm, sm[i]);
    float gs = 0.f;
    for (int i = 0; i < nw; ++i) gs += (sm[i] == -INFINITY) ? 0.f : ss[i] * __expf(sm[i] - gm);
    const int64_t t = targets[row] - vocab_start;
    float tl = 0.f;
    if (t >= 0 && t < vocab_local) tl = __bfloat162float(lr[t]);
    stats[row * 3 + 0] = gm;
    stats[row * 3 + 1] = gs;
    stats[row * 3 + 2] = tl;
  }
}

__global__ void __launch_bounds__(512) ce_finalize_kernel(
    __nv_bfloat16* __restrict__ logits, int ld, const int64_t* __restrict__ targets,
    const float* __restrict__ gstats, float* __restrict__ loss_rows, int vocab_local,
    int vocab_start, const float* __restrict__ grad_scale_ptr, int64_t ignore_index, int write_grad) {
  const int row = blockIdx.x;
  const float gm = gstats[row * 3 + 0], gs = gstats[row * 3 + 1], tl = gstats[row * 3 + 2];
  const int64_t tg = targets[row];
  const bool ignored = (tg == ignore_index);
  if (threadIdx.x == 0) loss_rows[row] = ignored ? 0.f : (logf(gs) + gm - tl);
  if (!write_grad) return;
  const float grad_scale = grad_scale_ptr ? *grad_scale_ptr : 1.0f;
  const float inv = ignored ? 0.f : grad_scale / gs;
  const int64_t t = tg - vocab_start;
  __nv_bfloat16* lr = logits + static_cast<size_t>(row) * ld;
  const int nchunks = vocab_local >> 3;
  for (int c = threadIdx.x; c < nchunks; c += blockDim.x) {
    const uint4 v = ld_global_v4(lr + c * 8);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    float f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 q = unpack_bf16x2(w[j]);
      f[2 * j] = __expf(q.x - gm) * inv;
      f[2 * j + 1] = __expf(q.y - gm) * inv;
    }
    if (!ignored && t >= c * 8 && t < c * 8 + 8) f[t - c * 8] -= grad_scale;
    st_global_v4(lr + c * 8, make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]),
                                        pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7])));
  }
  for (int c = nchunks * 8 + threadIdx.x; c < vocab_local; c += blockDim.x) {
    float f = __expf(__bfloat162float(lr[c]) - gm) * inv;
    if (!ignored && t == c) f -= grad_scale;
    lr[c] = __float2bfloat16(f);
  }
}

// ---------------------------------------------------------------------------------------------
// fused Adam(W) on a flat shard: fp32 master / moments, fp32 grads (already averaged),
// writes the bf16 model copy.  grad_scale folds in loss-scale / clipping coefficients.
// ---------------------------------------------------------------------------------------------
// One element of the step.  Every operation is rounded explicitly, leaving the compiler no multiply-add contraction to
// choose: adam_kernel's vector and scalar paths and adam_strided_kernel give the same bits for the same inputs.
__device__ __forceinline__ void adam_update(float& p, float& m, float& v, float g, float lr, float beta1, float beta2,
                                            float eps, float weight_decay, float bc1, float bc2, float grad_scale,
                                            int adamw) {
  g = __fmul_rn(g, grad_scale);
  if (!adamw && weight_decay != 0.f) g = __fmaf_rn(weight_decay, p, g);
  m = __fmaf_rn(beta1, m, __fmul_rn(__fsub_rn(1.f, beta1), g));
  v = __fmaf_rn(beta2, v, __fmul_rn(__fmul_rn(__fsub_rn(1.f, beta2), g), g));
  const float denom = __fadd_rn(__fsqrt_rn(__fdiv_rn(v, bc2)), eps);
  if (adamw && weight_decay != 0.f) p = __fmul_rn(p, __fsub_rn(1.f, __fmul_rn(lr, weight_decay)));
  p = __fsub_rn(p, __fdiv_rn(__fmul_rn(lr, __fdiv_rn(m, bc1)), denom));
}

__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ master,
                                                   float* __restrict__ exp_avg,
                                                   float* __restrict__ exp_avg_sq,
                                                   const float* __restrict__ grad,
                                                   __nv_bfloat16* __restrict__ param_bf16, int64_t n,
                                                   float lr, float beta1, float beta2, float eps,
                                                   float weight_decay, float bc1, float bc2,
                                                   float grad_scale, int adamw, int zero_grad) {
  const int64_t i4 = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i4 >= n) return;
  if (i4 + 4 <= n) {
    float4 p = *reinterpret_cast<float4*>(master + i4);
    float4 m = *reinterpret_cast<float4*>(exp_avg + i4);
    float4 v = *reinterpret_cast<float4*>(exp_avg_sq + i4);
    const float4 g4 = *reinterpret_cast<const float4*>(grad + i4);
    // in-kernel gradient reduce-scatter: the owner clears its slice right after consuming it, so that the peers'
    // next red.global.add contributions start from zero (no separate memset pass over the gradients)
    if (zero_grad) *reinterpret_cast<float4*>(const_cast<float*>(grad) + i4) = make_float4(0.f, 0.f, 0.f, 0.f);
    float pp[4] = {p.x, p.y, p.z, p.w}, mm[4] = {m.x, m.y, m.z, m.w}, vv[4] = {v.x, v.y, v.z, v.w};
    const float gg[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j)
      adam_update(pp[j], mm[j], vv[j], gg[j], lr, beta1, beta2, eps, weight_decay, bc1, bc2, grad_scale, adamw);
    *reinterpret_cast<float4*>(master + i4) = make_float4(pp[0], pp[1], pp[2], pp[3]);
    *reinterpret_cast<float4*>(exp_avg + i4) = make_float4(mm[0], mm[1], mm[2], mm[3]);
    *reinterpret_cast<float4*>(exp_avg_sq + i4) = make_float4(vv[0], vv[1], vv[2], vv[3]);
    if (param_bf16) {
      uint2 o = make_uint2(pack_bf16x2(pp[0], pp[1]), pack_bf16x2(pp[2], pp[3]));
      *reinterpret_cast<uint2*>(param_bf16 + i4) = o;
    }
  } else {
    for (int64_t i = i4; i < n; ++i) {
      float p = master[i], m = exp_avg[i], v = exp_avg_sq[i];
      adam_update(p, m, v, grad[i], lr, beta1, beta2, eps, weight_decay, bc1, bc2, grad_scale, adamw);
      master[i] = p;
      exp_avg[i] = m;
      exp_avg_sq[i] = v;
      if (param_bf16) param_bf16[i] = __float2bfloat16(p);
      if (zero_grad) const_cast<float*>(grad)[i] = 0.f;
    }
  }
}

// bf16 -> fp32 accumulate / copy with scale: dst (+)= scale * src
__global__ void __launch_bounds__(256) accum_bf16_to_f32_kernel(const __nv_bfloat16* __restrict__ src,
                                                               float* __restrict__ dst, int64_t n,
                                                               float scale, int accumulate) {
  const int64_t i8 = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  if (i8 >= n) return;
  if (i8 + 8 <= n) {
    const uint4 v = ld_global_nc_v4(src + i8);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    float f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = unpack_bf16x2(w[j]);
      f[2 * j] = t.x * scale;
      f[2 * j + 1] = t.y * scale;
    }
    float4* d = reinterpret_cast<float4*>(dst + i8);
    if (accumulate) {
      const float4 a = d[0], b = d[1];
      f[0] += a.x; f[1] += a.y; f[2] += a.z; f[3] += a.w;
      f[4] += b.x; f[5] += b.y; f[6] += b.z; f[7] += b.w;
    }
    d[0] = make_float4(f[0], f[1], f[2], f[3]);
    d[1] = make_float4(f[4], f[5], f[6], f[7]);
  } else {
    for (int64_t i = i8; i < n; ++i) {
      const float t = __bfloat162float(src[i]) * scale;
      dst[i] = accumulate ? dst[i] + t : t;
    }
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



#define PG_DISPATCH_CH(h, BODY)                                  \
  do {                                                           \
    const int ch__ = ((h) / 8 + 31) / 32;                        \
    if (ch__ <= 1) { constexpr int CH = 1; BODY; }               \
    else if (ch__ <= 2) { constexpr int CH = 2; BODY; }          \
    else if (ch__ <= 4) { constexpr int CH = 4; BODY; }          \
    else if (ch__ <= 8) { constexpr int CH = 8; BODY; }          \
    else if (ch__ <= 10) { constexpr int CH = 10; BODY; }        \
    else if (ch__ <= 16) { constexpr int CH = 16; BODY; }        \
    else if (ch__ <= 32) { constexpr int CH = 32; BODY; }        \
    else { fprintf(stderr, "pipegoose_b200: hidden size %d too large\n", (h)); return -1; } \
  } while (0)

extern "C" int pg_layernorm_fwd(const void* x, const int64_t* ids, int vocab_start, int vocab_end,
                                const void* gamma, const void* beta, void* y, float* mean,
                                float* rstd, int rows, int h, float eps, int apply_ln,
                                cudaStream_t s) {
  if (rows == 0) return 0;
  if (h % 8 != 0) return -1;
  const int blocks = (rows * 32 + 255) / 256;
  PG_DISPATCH_CH(h, (launch_pdl(layernorm_fwd_kernel<CH>, dim3(blocks), dim3(256), 0, s,
                                (const __nv_bfloat16*)x, ids, vocab_start, vocab_end,
                                (const __nv_bfloat16*)gamma, (const __nv_bfloat16*)beta, (__nv_bfloat16*)y,
                                mean, rstd, rows, h, eps, apply_ln)));
  PG_CHECK_LAUNCH("layernorm_fwd");
  return 0;
}

extern "C" int pg_layernorm_bwd(const void* dy, const void* x, const void* gamma, const float* mean,
                                const float* rstd, const void* dx_extra, void* dx, float* dgamma,
                                float* dbeta, int rows, int h, cudaStream_t s) {
  if (rows == 0) return 0;
  if (h % 8 != 0) return -1;
  const int blocks = (rows * 32 + 255) / 256;
  PG_DISPATCH_CH(h, (launch_pdl(layernorm_bwd_dx_kernel<CH>, dim3(blocks), dim3(256), 0, s,
                                (const __nv_bfloat16*)dy, (const __nv_bfloat16*)x,
                                (const __nv_bfloat16*)gamma, mean, rstd, (const __nv_bfloat16*)dx_extra,
                                (__nv_bfloat16*)dx, rows, h)));
  PG_CHECK_LAUNCH("layernorm_bwd_dx");
  if (dgamma != nullptr) {
    const int cb = (h + 255) / 256;
    int rsplit = (132 * 4 + cb - 1) / cb;
    if (rsplit > (rows + 63) / 64) rsplit = (rows + 63) / 64;
    if (rsplit < 1) rsplit = 1;
    const int rpb = (rows + rsplit - 1) / rsplit;
    launch_pdl(layernorm_bwd_params_kernel, dim3(cb, rsplit), dim3(256), 0, s,
               (const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, mean, rstd, dgamma, dbeta, rows, h, rpb);
    PG_CHECK_LAUNCH("layernorm_bwd_params");
  }
  return 0;
}

extern "C" int pg_colsum(const void* x, int ld, float* out, int rows, int cols, cudaStream_t s) {
  if (rows == 0 || cols == 0) return 0;
  const int cb = (cols + 255) / 256;
  int rsplit = (132 * 4 + cb - 1) / cb;
  if (rsplit > (rows + 63) / 64) rsplit = (rows + 63) / 64;
  if (rsplit < 1) rsplit = 1;
  const int rpb = (rows + rsplit - 1) / rsplit;
  launch_pdl(colsum_kernel, dim3(cb, rsplit), dim3(256), 0, s, (const __nv_bfloat16*)x, ld, out, rows, cols, rpb);
  PG_CHECK_LAUNCH("colsum");
  return 0;
}

extern "C" int pg_embedding_bwd(const void* dx, const int64_t* ids, float* dw, int rows, int h,
                                int vocab_start, int vocab_end, const PgGradRS* grad_rs, cudaStream_t s) {
  if (rows == 0) return 0;
  PgGradRS grs;
  memset(&grs, 0, sizeof(grs));
  if (grad_rs != nullptr) grs = *grad_rs;
  embedding_bwd_kernel<<<(rows * 32 + 255) / 256, 256, 0, s>>>((const __nv_bfloat16*)dx, ids, dw,
                                                               rows, h, vocab_start, vocab_end, grs);
  PG_CHECK_LAUNCH("embedding_bwd");
  return 0;
}

extern "C" int pg_grad_rs_accum(const void* src, int src_is_f32, float* dst_local, int64_t n, float scale,
                                const PgGradRS* grad_rs, cudaStream_t s) {
  if (n == 0) return 0;
  if (grad_rs == nullptr || grad_rs->world <= 1) return -1;
  const int64_t threads = (n + 3) / 4;
  const unsigned blocks = (unsigned)((threads + 255) / 256);
  if (src_is_f32) {
    grad_rs_accum_kernel<true><<<blocks, 256, 0, s>>>(src, dst_local, n, scale, *grad_rs);
  } else {
    grad_rs_accum_kernel<false><<<blocks, 256, 0, s>>>(src, dst_local, n, scale, *grad_rs);
  }
  PG_CHECK_LAUNCH("grad_rs_accum");
  return 0;
}

extern "C" int pg_ce_stats(const void* logits, int ld, const int64_t* targets, float* stats,
                           int rows, int vocab_local, int vocab_start, cudaStream_t s) {
  if (rows == 0) return 0;
  ce_stats_kernel<<<rows, 512, 0, s>>>((const __nv_bfloat16*)logits, ld, targets, stats,
                                       vocab_local, vocab_start);
  PG_CHECK_LAUNCH("ce_stats");
  return 0;
}

// one warp per row: merge the nparts (max, sumexp) partials of the lm_head GEMM epilogue, fetch the target logit
__global__ void __launch_bounds__(256) ce_combine_kernel(const float2* __restrict__ part, int nparts,
                                                         const __nv_bfloat16* __restrict__ logits, int ld,
                                                         const int64_t* __restrict__ targets, float* __restrict__ stats,
                                                         int rows, int vocab_local, int vocab_start) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float2* pr = part + static_cast<size_t>(row) * nparts;
  float m = -INFINITY, s = 0.f;
  for (int i = lane; i < nparts; i += 32) {
    const float2 v = pr[i];
    if (v.y > 0.f) {
      const float nm = fmaxf(m, v.x);
      s = s * __expf(m - nm) + v.y * __expf(v.x - nm);
      m = nm;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, off);
    const float os = __shfl_xor_sync(0xffffffffu, s, off);
    const float nm = fmaxf(m, om);
    if (nm > -INFINITY) {
      s = s * __expf(m - nm) + os * __expf(om - nm);
      m = nm;
    }
  }
  if (lane == 0) {
    const int64_t t = targets[row] - vocab_start;
    float tl = 0.f;
    if (t >= 0 && t < vocab_local) tl = __bfloat162float(logits[static_cast<size_t>(row) * ld + t]);
    stats[row * 3 + 0] = m;
    stats[row * 3 + 1] = s;
    stats[row * 3 + 2] = tl;
  }
}

extern "C" int pg_ce_combine(const float* part, int nparts, const void* logits, int ld, const int64_t* targets,
                             float* stats, int rows, int vocab_local, int vocab_start, cudaStream_t s) {
  if (rows == 0) return 0;
  ce_combine_kernel<<<(rows * 32 + 255) / 256, 256, 0, s>>>(reinterpret_cast<const float2*>(part), nparts,
                                                           (const __nv_bfloat16*)logits, ld, targets, stats, rows,
                                                           vocab_local, vocab_start);
  PG_CHECK_LAUNCH("ce_combine");
  return 0;
}

extern "C" int pg_ce_finalize(void* logits, int ld, const int64_t* targets, const float* gstats,
                              float* loss_rows, int rows, int vocab_local, int vocab_start,
                              const float* grad_scale, int64_t ignore_index, int write_grad,
                              cudaStream_t s) {
  if (rows == 0) return 0;
  ce_finalize_kernel<<<rows, 512, 0, s>>>((__nv_bfloat16*)logits, ld, targets, gstats, loss_rows,
                                          vocab_local, vocab_start, grad_scale, ignore_index,
                                          write_grad);
  PG_CHECK_LAUNCH("ce_finalize");
  return 0;
}

extern "C" int pg_adam(float* master, float* m, float* v, const float* grad, void* param_bf16,
                       int64_t n, float lr, float beta1, float beta2, float eps, float wd,
                       float bc1, float bc2, float grad_scale, int adamw, int zero_grad, cudaStream_t s) {
  if (n == 0) return 0;
  const int64_t threads = (n + 3) / 4;
  adam_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(
      master, m, v, grad, (__nv_bfloat16*)param_bf16, n, lr, beta1, beta2, eps, wd, bc1, bc2,
      grad_scale, adamw, zero_grad);
  PG_CHECK_LAUNCH("adam");
  return 0;
}

// one thread per four consecutive elements of one bucket slice (seg % 4 == 0)
__global__ void __launch_bounds__(256) adam_strided_kernel(float* __restrict__ master, float* __restrict__ exp_avg,
                                                           float* __restrict__ exp_avg_sq, float* __restrict__ grad,
                                                           __nv_bfloat16* __restrict__ param_bf16, int64_t seg,
                                                           int64_t bucket_stride, int64_t total, float lr, float beta1,
                                                           float beta2, float eps, float weight_decay, float bc1, float bc2,
                                                           float grad_scale, int adamw, int zero_grad) {
  const int64_t i4 = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i4 >= total) return;
  const int64_t b = i4 / seg;
  const int64_t f4 = b * bucket_stride + (i4 - b * seg);  // offset in the flat gradient / parameter buffers
  float4 p = *reinterpret_cast<float4*>(master + i4);
  float4 m = *reinterpret_cast<float4*>(exp_avg + i4);
  float4 v = *reinterpret_cast<float4*>(exp_avg_sq + i4);
  const float4 g4 = *reinterpret_cast<const float4*>(grad + f4);
  if (zero_grad) *reinterpret_cast<float4*>(grad + f4) = make_float4(0.f, 0.f, 0.f, 0.f);
  float pp[4] = {p.x, p.y, p.z, p.w}, mm[4] = {m.x, m.y, m.z, m.w}, vv[4] = {v.x, v.y, v.z, v.w};
  const float gg[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
  for (int j = 0; j < 4; ++j)
    adam_update(pp[j], mm[j], vv[j], gg[j], lr, beta1, beta2, eps, weight_decay, bc1, bc2, grad_scale, adamw);
  *reinterpret_cast<float4*>(master + i4) = make_float4(pp[0], pp[1], pp[2], pp[3]);
  *reinterpret_cast<float4*>(exp_avg + i4) = make_float4(mm[0], mm[1], mm[2], mm[3]);
  *reinterpret_cast<float4*>(exp_avg_sq + i4) = make_float4(vv[0], vv[1], vv[2], vv[3]);
  if (param_bf16) *reinterpret_cast<uint2*>(param_bf16 + f4) = make_uint2(pack_bf16x2(pp[0], pp[1]), pack_bf16x2(pp[2], pp[3]));
}

extern "C" int pg_adam_strided(float* master, float* m, float* v, float* grad, void* param_bf16, int64_t seg,
                               int64_t bucket_stride, int64_t nb, float lr, float beta1, float beta2, float eps, float wd,
                               float bc1, float bc2, float grad_scale, int adamw, int zero_grad, cudaStream_t s) {
  if (nb <= 0 || seg <= 0) return 0;
  if (seg % 4 != 0 || bucket_stride % 4 != 0) return -1;
  const int64_t total = seg * nb;
  const int64_t threads = total / 4;
  adam_strided_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(master, m, v, grad, (__nv_bfloat16*)param_bf16, seg,
                                                                       bucket_stride, total, lr, beta1, beta2, eps, wd, bc1,
                                                                       bc2, grad_scale, adamw, zero_grad);
  PG_CHECK_LAUNCH("adam_strided");
  return 0;
}

extern "C" int pg_accum_bf16_to_f32(const void* src, float* dst, int64_t n, float scale,
                                    int accumulate, cudaStream_t s) {
  if (n == 0) return 0;
  const int64_t threads = (n + 7) / 8;
  accum_bf16_to_f32_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(
      (const __nv_bfloat16*)src, dst, n, scale, accumulate);
  PG_CHECK_LAUNCH("accum_bf16_to_f32");
  return 0;
}
