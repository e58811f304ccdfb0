// C launch API shared between the CUDA translation units (nvcc) and the torch bindings (g++).
// Every entry point returns 0 on success and enqueues on the given stream.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PG_MAX_PEERS 8

// In-kernel data-parallel gradient reduce-scatter (ZeRO-1): the flat fp32 gradient buffer of every data-parallel rank is
// peer-mapped; elements [start, start + world * seg) are owned slice-wise (rank r owns [start + r*seg, start + (r+1)*seg)).
// A kernel that produces a gradient (wgrad GEMM epilogue, embedding backward, gradient fold) adds it with
// red.global.add straight into the OWNER's buffer — no local copy, no separate reduction kernel, nothing exposed
// after backward except one peer barrier.  world <= 1: plain local accumulation.
typedef struct PgGradRS {
  float* peer[PG_MAX_PEERS];  // flat gradient buffer of data-parallel rank r (peer[my rank] is the local buffer)
  const float* local;         // this rank's flat gradient buffer (gradient pointers handed to kernels point into it)
  long long start;            // first element of the in-kernel reduce-scatter region
  long long seg;              // elements per owner slice (multiple of 4)
  int world;
  int scalar_red;             // 1: four scalar red.global.add.f32 instead of one red.global.add.v4.f32
} PgGradRS;

typedef struct PgGemmDesc {
  const void* A;  // bf16
  const void* B;  // bf16
  int M, N, K;
  int lda, ldb;
  int a_mn;  // 0: A is [M, K] row-major (K-major); 1: A is [K, M] row-major (MN-major)
  int b_mn;  // 0: B is [N, K] row-major (K-major); 1: B is [K, N] row-major (MN-major)
  void* out;
  int ldc;
  const void* bias;      // bf16 [N]
  const void* residual;  // bf16 [M, ldr]
  int ldr;
  void* aux;  // bf16 [M, ldc]
  int flags;  // EpiFlags
  int block_n;   // 0 = auto
  int k_splits;  // 0 = auto (fp32 outputs only), 1 = never split, >1 = forced
  int max_ctas;  // 0 = all SMs
  int num_chunks, chunk_rows, first_chunk;
  const uint32_t* chunk_flags;
  uint32_t flag_value;
  void* out_peer[PG_MAX_PEERS];
  uint32_t* arrive_ctr[PG_MAX_PEERS];
  // GEMM -> reduce-scatter with the reduction fused into the local chunk's epilogue (see GemmArgs)
  const void* rs_in[PG_MAX_PEERS];
  const uint32_t* rs_wait_ctr;
  uint32_t rs_wait_value;
  // all-gather -> GEMM communication CTAs
  int n_comm;
  const void* ag_src[PG_MAX_PEERS];
  void* ag_dst;
  uint64_t ag_chunk_bytes;
  uint32_t* ag_peer_flag[PG_MAX_PEERS];
  const uint32_t* ag_ready;
  uint32_t ag_epoch;
  int my_rank;
  const void* a_local;  // all-gather -> GEMM: this rank's shard [chunk_rows, K] (read in place)
  // grouped GEMM / MoE combine
  int b_chunk_rows, bias_chunk_stride;
  const int* row_ret;
  const float* row_scale;
  int scatter_rows_per_src;
  // fp32 output (wgrad): add the tile into the owners' gradient buffers (see PgGradRS); world <= 1: off
  PgGradRS grad_rs;
  // lm_head: per-row online-softmax partials [M, 2 * ceil(N / block_n), 2] fp32 written by the epilogue (null: off);
  // columns >= ce_valid are padding.  block_n is forced to 256 so that the caller can size the buffer.
  float* ce_part;
  int ce_valid;
  // wgrad (a_mn): with EPI_BGRAD (256) in flags, bias_grad[m] (fp32 [M]) += sum over k of A[k, m], the bias gradient
  // summed from the dY stages the GEMM already loads
  float* bias_grad;
  // FP8 operands: fmt 1 = A e4m3, 2 = A e5m2 (B e4m3 in both; 0 = bf16).  A [M, K] and B [N, K] codes, both K-major
  // (a_mn = b_mn = 0), K % 16 == 0; value = code * scale_inv with one fp32 device scalar per operand.  Only the TMA
  // epilogue's cases: bf16 out with bias / bias + GELU (+ pre-activation) / bias + residual / GELU', or plain fp32 out.
  int fmt;
  const float* a_scale_inv;
  const float* b_scale_inv;
} PgGemmDesc;

// ---- attention_sm90.cu
// seg_start: int32 [B*S] row-relative document starts of packed sequences (nullptr: one document per row)
int pg_attention_fwd(const void* qkv, const float* slopes, void* out, float* lse, int B, int S, int H, int D,
                     float softmax_scale, const int* seg_start, cudaStream_t s);
// dq_acc: fp32 workspace [B*S, H*D], any contents; stats: fp32 workspace of pg_attention_bwd_stats_floats(B, S, H)
int pg_attention_bwd(const void* qkv, const float* slopes, const void* out, const float* lse, const void* dout,
                     void* dqkv, float* dq_acc, float* stats, int B, int S, int H, int D, float softmax_scale,
                     const int* seg_start, cudaStream_t s);
int64_t pg_attention_bwd_stats_floats(int B, int S, int H);
// Paged prefill: the new tokens of R sequences packed in qkv [N, H*3*D] (sequence r: rows cu_seqlens[r] ..
// cu_seqlens[r+1]-1 at positions start[r], start[r]+1, ...) attend to keys 0 <= k <= p of their own sequence, all read
// from k_pool / v_pool [num_pages, H, 64, D] through table [R, max_pages] (the caller stores the new k / v first).
// cu_seqlens, start, table: int32 on the device; max_len >= every sequence's new tokens (host bound, sizes the grid).
// out [N, H*D].  D in {64, 80, 128}.  No LSE: inference only.
int pg_paged_prefill_attention(const void* qkv, const void* k_pool, const void* v_pool, const int* table,
                               const int* cu_seqlens, const int* start, const float* slopes, void* out, int N, int R,
                               int H, int D, int num_pages, int max_pages, int max_len, float softmax_scale,
                               cudaStream_t s);

// ---- decode_sm90.cu
// One decoding step of B rows at column pos: writes the new k / v of qkv [B, H*3*D] into k_cache / v_cache
// [B, H, capacity, D], then out [B, H*D] = softmax(q.k * scale + slope * (k - pos)) V over keys lead[b] <= k <= pos
// (lead: int32 [B] or nullptr).  D in {64, 80, 128}.  splits > 1: part is an fp32 workspace of B*H*splits*(D+2)
// floats and ticket an int32 [B*H] array that is zero before the call and zero again after it.
int pg_decode_attention(const void* qkv, void* k_cache, void* v_cache, const float* slopes, const int* lead, void* out,
                        float* part, int* ticket, int B, int H, int D, int capacity, int pos, int splits,
                        float softmax_scale, cudaStream_t s);
// split count for B*H rows whose key ranges are at most `span` keys long
int pg_decode_splits(int B, int H, int span);
// The paged form: k_pool / v_pool [num_pages, H, 64, D]; row b's position p is slot p % 64 of page
// table[b * max_pages + p / 64].  Row b writes its new k / v at pos[b] (int32 [B], device) and attends to keys
// 0 <= k <= pos[b].  max_pos >= every pos[b] sizes the grid (splits from pg_decode_splits(B, H, max_pos + 1)).
int pg_paged_decode_attention(const void* qkv, void* k_pool, void* v_pool, const int* table, const int* pos,
                              const float* slopes, void* out, float* part, int* ticket, int B, int H, int D,
                              int max_pages, int max_pos, int splits, float softmax_scale, cudaStream_t s);
// Append form (speculative verification): row b appends the n_b = cu_seqlens[b+1] - cu_seqlens[b] tokens (1 <= n_b <= 8,
// sum N) of qkv [N, H*3*D] at positions pos[b] .. pos[b] + n_b - 1, writing their k / v into their slots; token i
// attends to keys 0 .. pos[b] + i.  Every key is read once per CTA for all of the row's tokens.  max_pos >= every
// pos[b] + n_b - 1 sizes the grid (splits from pg_decode_splits(B, H, max_pos + 1)); max_tokens (1 .. 8) >= every n_b
// picks the query tile (1, 2, 4 or 8 queries per CTA).  Both are host bounds the caller guarantees.  splits > 1: part
// holds B*H*8*splits*(D+2) floats; ticket is an int32 [B*H*8] array, zero before the call and zero again after it.
int pg_paged_append_attention(const void* qkv, void* k_pool, void* v_pool, const int* table, const int* cu_seqlens,
                              const int* pos, const float* slopes, void* out, float* part, int* ticket, int B, int N,
                              int H, int D, int max_pages, int max_pos, int max_tokens, int splits,
                              float softmax_scale, cudaStream_t s);
// Prefill: the k / v of every token n of qkv [N, H*3*D] into pool slot slot[n] (page * 64 + offset), all heads.
int pg_paged_kv_write(const void* qkv, const int* slot, void* k_pool, void* v_pool, int N, int H, int D,
                      cudaStream_t s);
// FP8 pools: e4m3 codes k_pool / v_pool [num_pages, H, 64, D] with fp32 scales k_scales / v_scales [num_pages, H, 64],
// one per position and head (value = float(code) * scale).  pg_paged_kv_write_fp8 quantizes every token's k / v into
// its slot.  pg_paged_decode_attention_fp8 is pg_paged_decode_attention over those pools: the key and value at pos[b]
// come from qkv exactly and are quantized into their slot.  pg_paged_kv_dequantize writes pages src[i] (int32 [n]) of
// the FP8 pools, dequantized to bf16, into pages dst[i] of k_out / v_out [*, H, 64, D]: the staging pool through which
// pg_paged_prefill_attention reads a cached prefix held in FP8 pools.
int pg_paged_kv_write_fp8(const void* qkv, const int* slot, void* k_pool, void* v_pool, float* k_scales,
                          float* v_scales, int N, int H, int D, cudaStream_t s);
int pg_paged_decode_attention_fp8(const void* qkv, void* k_pool, void* v_pool, float* k_scales, float* v_scales,
                                  const int* table, const int* pos, const float* slopes, void* out, float* part,
                                  int* ticket, int B, int H, int D, int max_pages, int max_pos, int splits,
                                  float softmax_scale, cudaStream_t s);
int pg_paged_kv_dequantize(const void* k_pool, const void* v_pool, const float* k_scales, const float* v_scales,
                           const int* src, const int* dst, void* k_out, void* v_out, int n, int H, int D,
                           cudaStream_t s);
// Beam-search forks: for every pair i of pairs (int32 [n, 3]: src page, dst page, count) and every layer of the pools
// k_pools / v_pools [layers, pages, H, 64, D] (row_bytes = D * element size), slots 0 .. count - 1 of page src are
// copied into page dst, with their fp32 scales [layers, pages, H, 64] when k_scales / v_scales are given (FP8 pools).
int pg_paged_kv_copy(const int* pairs, void* k_pools, void* v_pools, float* k_scales, float* v_scales, int n,
                     int layers, int pages, int H, int row_bytes, cudaStream_t s);

// ---- kv_swap_sm90.cu
// Preemption: for every pair i of pairs (int32 [n, 2]: pool page, host slot), every layer, K and V of page `page` of the
// pools [layers, pages, H, 64, D] (row_bytes = D * element size) move to or from slot `slot` of host_kv [slots, layers,
// 2, H, 64, D] (to_host != 0: pool -> host), with the fp32 scales [layers, pages, H, 64] <-> host_scales [slots,
// layers, 2, H, 64] when given (FP8 pools; all three or none).  host_kv / host_scales are device pointers of pinned
// host memory (cudaHostGetDevicePointer).  The caller guarantees that every id is in range.
int pg_paged_kv_swap(const int* pairs, void* k_pools, void* v_pools, float* k_scales, float* v_scales, void* host_kv,
                     float* host_scales, int n, int layers, int pages, int H, int row_bytes, int to_host,
                     cudaStream_t s);

// ---- beam_sm90.cu
// Beam search's candidate choice: for every request r (rows cu[r] .. cu[r+1] - 1 of logits [N, V], bf16 or, with
// fp32 != 0, fp32, row stride ld) the k (1 .. 16) best (score, token, row) by score = scores[row] + (logit - lse[row]),
// descending, ties to the lower (row, token); lse (nullable, fp32 [N]) receives each row's logsumexp.  max_rows
// (<= 64) bounds the rows of one request; splits comes from pg_beam_topk_splits(N, V, k, max_rows).  part holds
// N * splits * (2 + 2 * pg_beam_topk_kp(k)) floats; ticket is an int32 [R] array, zero before the call and after it.
int pg_beam_topk_kp(int k);
int pg_beam_topk_splits(int N, int V, int k, int max_rows);
int pg_beam_topk(const void* logits, int fp32, long long ld, const float* scores, const int* cu, float* part,
                 int* ticket, float* out_score, int* out_token, int* out_row, float* lse, int N, int V, int R, int k,
                 int max_rows, int splits, cudaStream_t s);

// ---- moe.cu
int pg_moe_route(const void* x, const void* wg, const void* bg, const float* jitter, int n, int h, int E, int top_k,
                 int capacity, float* probs, int* topk_idx, float* topk_prob, int* pos, int* counts,
                 float* prob_sum, float* zsum, float* lse_out, cudaStream_t s);
int pg_moe_dispatch(const void* x, const int* topk_idx, const float* topk_prob, const int* pos,
                    void* const* peer_buf, int* const* peer_row_ret, float* const* peer_row_scale,
                    uint32_t* const* peer_arrive, int n, int h, int top_k, int E_local, int T, int C, int my_rank,
                    int scale_by_prob, int blocks, cudaStream_t s);
int pg_fill_i32(int* p, int v, int64_t n, cudaStream_t s);

// ---- comm.cu
// out[rows, cols] = sum_src staging[src][rows, cols] (+ bias) (+ residual), after every source's
// arrival counter reached `expected`
int pg_rs_reduce(const void* staging, int num_src, int64_t src_stride_elems, const uint32_t* arrive_ctr,
                 uint32_t expected, const void* bias, const void* residual, void* out, int rows, int cols,
                 cudaStream_t s);
// flat fp32 gradient bucket: in-place all-reduce / reduce-scatter average over NVLink peers
// mc_buf != null: the reduce half is ONE multimem.ld_reduce per 16 bytes (summed inside the NVSwitch), the all-gather
// half ONE multimem.st
// [offset, offset + n) may be a run of buckets of bucket_elems elements (0: one bucket): each is reduced slice-wise
int pg_allreduce_f32(float* const* peer_bufs, float* mc_buf, int world, int rank, int64_t offset_elems, int64_t n,
                     int64_t bucket_elems, float scale, int reduce_scatter_only, uint32_t* const* peer_flags,
                     uint32_t epoch, int blocks, cudaStream_t s);
// ZeRO-1 parameter all-gather: regions [0, head) and then [head + k*bucket, ...) up to total; every rank pushes its
// 1/world slice of each region to all peers (mc_buf != null: ONE multimem.st per 16 bytes through the NVSwitch)
int pg_allgather_bf16(void* const* peer_bufs, void* mc_buf, int world, int rank, int64_t head_elems,
                      int64_t bucket_elems, int64_t total_elems, uint32_t* const* peer_flags, uint32_t epoch,
                      cudaStream_t s);
int pg_barrier_peers(uint32_t* const* peer_flags, int world, int rank, uint32_t epoch, cudaStream_t s);
// reduce-scatter without a GEMM: push row block c of x [num_chunks * chunk_elems] to rank c's staging slot and bump its
// arrival counter by `blocks` (one per CTA); the owner runs pg_rs_reduce on the slots
int pg_rs_push(const void* x, int num_chunks, int first_chunk, int64_t chunk_elems, void* const* out_peer,
               uint32_t* const* arrive_ctr, int blocks, cudaStream_t s);
// NVLS
int pg_multimem_selftest(const float* mc_in, float* mc_out, float* out, int64_t n, cudaStream_t s);
int pg_rs_reduce_mc(const void* mc_partial, const uint32_t* arrive_ctr, int num_src, uint32_t expected, const void* bias,
                    const void* residual, void* out, int rows, int cols, cudaStream_t s);
// symmetric memory (VMM + multicast; symm_vmm.cu)
int pg_vmm_probe(int world, int* mc_supported, int64_t* gran);
int pg_vmm_alloc(int64_t nbytes, void** ptr, int* fd, uint64_t* handle);
int pg_vmm_import(int fd, int64_t nbytes, void** ptr, uint64_t* handle);
int pg_vmm_unmap(void* ptr, int64_t nbytes, uint64_t handle);
int pg_mc_create(int world, int64_t nbytes, int* fd, uint64_t* mc_handle);
int pg_mc_import(int fd, uint64_t* mc_handle);
int pg_mc_add_device(uint64_t mc_handle);
int pg_mc_bind(uint64_t mc_handle, uint64_t mem_handle, int64_t nbytes, void** mc_ptr);
// symmetric memory (cudaIpc)
int pg_symm_alloc(int64_t nbytes, void** ptr, void* handle64);
int pg_symm_open(const void* handle64, void** ptr);
int pg_symm_close(void* ptr);
int pg_symm_free(void* ptr);

int pg_gemm_bf16(const PgGemmDesc* d, cudaStream_t stream);
// persistent GEMM grids use at most `ctas` CTAs (0 = all SMs): leaves SMs to overlapped communication kernels
void pg_set_gemm_cta_cap(int ctas);

// ---- elementwise.cu
int pg_layernorm_fwd(const void* x, const int64_t* ids, int vocab_start, int vocab_end,
                     const void* gamma, const void* beta, void* y, float* mean, float* rstd,
                     int rows, int h, float eps, int apply_ln, cudaStream_t s);
int pg_layernorm_bwd(const void* dy, const void* x, const void* gamma, const float* mean,
                     const float* rstd, const void* dx_extra, void* dx, float* dgamma, float* dbeta,
                     int rows, int h, cudaStream_t s);
int pg_colsum(const void* x, int ld, float* out, int rows, int cols, cudaStream_t s);
int pg_embedding_bwd(const void* dx, const int64_t* ids, float* dw, int rows, int h,
                     int vocab_start, int vocab_end, const PgGradRS* grad_rs, cudaStream_t s);
// dst (a range of the local flat gradient buffer) += scale * src, added into the owners' buffers (src: bf16 or fp32)
int pg_grad_rs_accum(const void* src, int src_is_f32, float* dst_local, int64_t n, float scale,
                     const PgGradRS* grad_rs, cudaStream_t s);
int pg_ce_stats(const void* logits, int ld, const int64_t* targets, float* stats, int rows,
                int vocab_local, int vocab_start, cudaStream_t s);
// merge the GEMM epilogue's partials [rows, nparts, 2] into stats [rows, 3] = (max, sumexp, logit[target] or 0)
int pg_ce_combine(const float* part, int nparts, const void* logits, int ld, const int64_t* targets, float* stats,
                  int rows, int vocab_local, int vocab_start, cudaStream_t s);
int pg_ce_finalize(void* logits, int ld, const int64_t* targets, const float* gstats,
                   float* loss_rows, int rows, int vocab_local, int vocab_start,
                   const float* grad_scale, int64_t ignore_index, int write_grad, cudaStream_t s);
int pg_adam(float* master, float* m, float* v, const float* grad, void* param_bf16, int64_t n,
            float lr, float beta1, float beta2, float eps, float wd, float bc1, float bc2,
            float grad_scale, int adamw, int zero_grad, cudaStream_t s);
// ZeRO-1 form: ONE launch updates this rank's slice of nb equally sized buckets — optimizer state element b * seg + w
// belongs to flat element first + b * bucket_stride + w (w < seg)
int pg_adam_strided(float* master, float* m, float* v, float* grad, void* param_bf16, int64_t seg, int64_t bucket_stride,
                    int64_t nb, float lr, float beta1, float beta2, float eps, float wd, float bc1, float bc2,
                    float grad_scale, int adamw, int zero_grad, cudaStream_t s);
int pg_accum_bf16_to_f32(const void* src, float* dst, int64_t n, float scale, int accumulate,
                         cudaStream_t s);

// ---- fp8_cast.cu (per-tensor FP8 casts of the FP8 linear layers; format in fp8_cast.cu)
// amax (fp32 device scalar) = max |x| over n bf16 elements (n % 8 == 0, x 16-byte aligned)
int pg_fp8_amax(const void* x, int64_t n, float* amax, cudaStream_t s);
// x bf16 [R, C] contiguous (C % 8 == 0) -> codes [R, C], codes_t [C, R], scale_inv (fp32 scalar), colsum (fp32 [C], added
// into), each written when not null; e5m2: 1 for e5m2 codes, 0 for e4m3
int pg_fp8_cast(const void* x, int R, int C, int e5m2, const float* amax, void* codes, void* codes_t, float* scale_inv,
                float* colsum, cudaStream_t s);

#ifdef __cplusplus
}
#endif
