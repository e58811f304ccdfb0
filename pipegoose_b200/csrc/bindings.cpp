// torch <-> kernel glue.  Only argument checking and pointer plumbing lives here; every op
// enqueues on the current CUDA stream and raises if the launch API reports a failure.
#include <torch/extension.h>
#include <c10/cuda/CUDAStream.h>
#include <c10/cuda/CUDAGuard.h>

#include "launch.h"
#include <cmath>

namespace {

cudaStream_t cur_stream() { return c10::cuda::getCurrentCUDAStream().stream(); }

bool parse_grad_rs(const py::dict& d, PgGradRS* out);

void check_bf16_2d(const torch::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.scalar_type() == torch::kBFloat16, name, " must be bf16");
  TORCH_CHECK(t.dim() == 2 && t.stride(1) == 1, name, " must be 2-D with unit inner stride");
  TORCH_CHECK(t.stride(0) % 8 == 0, name, " leading dimension must be a multiple of 8");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0, name, " must be 16B aligned");
}

// out[M,N] = epilogue(op(A) * op(B)).  a_mn/b_mn select the stored layout (see launch.h).
void gemm(const torch::Tensor& a, const torch::Tensor& b, torch::Tensor out, bool a_mn, bool b_mn,
          const c10::optional<torch::Tensor>& bias, const c10::optional<torch::Tensor>& residual,
          const c10::optional<torch::Tensor>& aux, int64_t flags, int64_t block_n,
          int64_t max_ctas, int64_t num_chunks, int64_t first_chunk, int64_t chunk_flags_ptr,
          int64_t flag_value, std::vector<int64_t> out_peer_ptrs,
          std::vector<int64_t> arrive_ctr_ptrs, const py::dict& ag,
          const c10::optional<torch::Tensor>& bias_grad) {
  check_bf16_2d(a, "a");
  check_bf16_2d(b, "b");
  c10::cuda::CUDAGuard guard(a.device());
  PgGemmDesc d;
  memset(&d, 0, sizeof(d));
  const int64_t M = a_mn ? a.size(1) : a.size(0);
  const int64_t K = a_mn ? a.size(0) : a.size(1);
  const int64_t groups = ag.contains("b_chunk_rows") ? num_chunks : 1;  // stacked (grouped) B
  const int64_t N = b_mn ? b.size(1) : b.size(0) / groups;
  const int64_t Kb = b_mn ? b.size(0) / groups : b.size(1);
  TORCH_CHECK(K == Kb, "gemm: contraction dims differ: ", K, " vs ", Kb);
  TORCH_CHECK(N % 8 == 0, "gemm: N must be a multiple of 8");
  d.A = a.data_ptr();
  d.B = b.data_ptr();
  d.M = (int)M; d.N = (int)N; d.K = (int)K;
  d.lda = (int)a.stride(0);
  d.ldb = (int)b.stride(0);
  d.a_mn = a_mn; d.b_mn = b_mn;
  TORCH_CHECK(out.is_cuda() && out.dim() == 2 && out.stride(1) == 1, "out must be 2-D cuda");
  const bool f32 = out.scalar_type() == torch::kFloat32;
  TORCH_CHECK(f32 || out.scalar_type() == torch::kBFloat16, "out must be bf16 or fp32");
  if (out_peer_ptrs.empty()) {
    TORCH_CHECK(out.size(0) == M && out.size(1) == N, "out shape mismatch");
  }
  d.out = out.data_ptr();
  d.ldc = (int)out.stride(0);
  TORCH_CHECK(d.ldc % 8 == 0, "out leading dimension must be a multiple of 8");
  // both epilogues write 16-byte groups (vector stores / TMA)
  TORCH_CHECK(reinterpret_cast<uintptr_t>(d.out) % 16 == 0, "out must be 16B aligned");
  d.flags = (int)flags | (f32 ? 8 : 0);
  if (bias.has_value()) {
    TORCH_CHECK(bias->scalar_type() == torch::kBFloat16 && bias->numel() % N == 0 && bias->is_contiguous(), "bias must be contiguous bf16 [N] (or [groups, N])");
    d.bias = bias->data_ptr();
    d.flags |= 1;
  }
  if (residual.has_value()) {
    check_bf16_2d(*residual, "residual");
    // fused reduce-scatter: the residual is the local token shard [M / num_chunks, N]
    TORCH_CHECK((residual->size(0) == M || (ag.contains("rs_in") && residual->size(0) * num_chunks == M)) &&
                    residual->size(1) == N, "residual shape mismatch");
    d.residual = residual->data_ptr();
    d.ldr = (int)residual->stride(0);
    d.flags |= 4;
  }
  if (aux.has_value()) {
    check_bf16_2d(*aux, "aux");
    TORCH_CHECK(aux->size(0) == M && aux->size(1) == N && aux->stride(0) == out.stride(0), "aux must match out");
    d.aux = aux->data_ptr();
  }
  d.block_n = (int)block_n;
  d.max_ctas = (int)max_ctas;
  d.num_chunks = (int)num_chunks;
  d.first_chunk = (int)first_chunk;
  if (num_chunks > 1) {
    TORCH_CHECK(M % num_chunks == 0, "M must divide into chunks");
    d.chunk_rows = (int)(M / num_chunks);
    TORCH_CHECK(num_chunks <= PG_MAX_PEERS, "too many chunks");
  }
  d.chunk_flags = reinterpret_cast<const uint32_t*>(chunk_flags_ptr);
  d.flag_value = (uint32_t)flag_value;
  for (size_t i = 0; i < out_peer_ptrs.size() && i < PG_MAX_PEERS; ++i) d.out_peer[i] = reinterpret_cast<void*>(out_peer_ptrs[i]);
  for (size_t i = 0; i < arrive_ctr_ptrs.size() && i < PG_MAX_PEERS; ++i) d.arrive_ctr[i] = reinterpret_cast<uint32_t*>(arrive_ctr_ptrs[i]);
  if (ag.contains("b_chunk_rows")) {
    d.b_chunk_rows = ag["b_chunk_rows"].cast<int>();
    d.bias_chunk_stride = ag.contains("bias_chunk_stride") ? ag["bias_chunk_stride"].cast<int>() : 0;
    if (ag.contains("row_ret")) {
      d.row_ret = reinterpret_cast<const int*>(ag["row_ret"].cast<int64_t>());
      d.row_scale = reinterpret_cast<const float*>(ag["row_scale"].cast<int64_t>());
      d.scatter_rows_per_src = ag["rows_per_src"].cast<int>();
    }
  }
  if (ag.contains("rs_in")) {
    auto in = ag["rs_in"].cast<std::vector<int64_t>>();
    for (size_t i = 0; i < in.size() && i < PG_MAX_PEERS; ++i) d.rs_in[i] = reinterpret_cast<const void*>(in[i]);
    d.rs_wait_ctr = reinterpret_cast<const uint32_t*>(ag["rs_wait"].cast<int64_t>());
    d.rs_wait_value = (uint32_t)ag["rs_wait_value"].cast<int64_t>();
    d.my_rank = ag["rank"].cast<int>();
  }
  if (ag.contains("ce_part")) {
    // lm_head + cross entropy: the epilogue also writes the online-softmax partials (fp32 [M, 2 * ceil(N/256), 2])
    TORCH_CHECK(!f32 && num_chunks >= 1, "ce_part needs a bf16 logits output");
    d.ce_part = reinterpret_cast<float*>(ag["ce_part"].cast<int64_t>());
    d.ce_valid = ag.contains("ce_valid") ? ag["ce_valid"].cast<int>() : 0;
  }
  if (ag.contains("grad_rs")) {
    TORCH_CHECK(f32, "grad_rs needs an fp32 output");
    parse_grad_rs(ag["grad_rs"].cast<py::dict>(), &d.grad_rs);
  }
  if (bias_grad.has_value()) {
    // wgrad with the bias gradient summed from the dY operand: bias_grad[m] += sum_k a[k, m]
    TORCH_CHECK(a_mn && num_chunks == 1 && !ag.contains("n_comm"), "bias_grad needs a wgrad (a_mn) GEMM of one chunk");
    TORCH_CHECK(bias_grad->is_cuda() && bias_grad->scalar_type() == torch::kFloat32 && bias_grad->is_contiguous() &&
                    bias_grad->numel() == M, "bias_grad must be a contiguous fp32 CUDA tensor of ", M, " elements");
    d.bias_grad = bias_grad->data_ptr<float>();
    d.flags |= 256;
  }
  if (ag.contains("k_splits")) d.k_splits = ag["k_splits"].cast<int>();
  if (ag.contains("n_comm")) {
    d.n_comm = ag["n_comm"].cast<int>();
    d.ag_dst = reinterpret_cast<void*>(ag["dst"].cast<int64_t>());
    d.ag_chunk_bytes = (uint64_t)ag["chunk_bytes"].cast<int64_t>();
    d.ag_ready = reinterpret_cast<const uint32_t*>(ag["ready"].cast<int64_t>());
    d.ag_epoch = (uint32_t)ag["epoch"].cast<int64_t>();
    d.my_rank = ag["rank"].cast<int>();
    d.a_local = reinterpret_cast<const void*>(ag["local"].cast<int64_t>());
    auto src = ag["src"].cast<std::vector<int64_t>>();
    auto pf = ag["peer_flag"].cast<std::vector<int64_t>>();
    for (size_t i = 0; i < src.size() && i < PG_MAX_PEERS; ++i) d.ag_src[i] = reinterpret_cast<const void*>(src[i]);
    for (size_t i = 0; i < pf.size() && i < PG_MAX_PEERS; ++i) d.ag_peer_flag[i] = reinterpret_cast<uint32_t*>(pf[i]);
  }
  TORCH_CHECK(pg_gemm_bf16(&d, cur_stream()) == 0, "pg_gemm_bf16 failed");
}


bool is_fp8(const torch::Tensor& t) {
  return t.scalar_type() == torch::kFloat8_e4m3fn || t.scalar_type() == torch::kFloat8_e5m2;
}

// out[M, N] = epilogue(a_scale_inv * b_scale_inv * (a[M, K] · b[N, K]ᵀ)) over FP8 codes, both K-major: a e4m3 or e5m2,
// b e4m3.  bf16 out: bias, gelu (pre-activation into aux), residual, or dgelu (out *= gelu'(aux)); fp32 out: overwrite
// or accumulate, k_splits 0 = auto, 1 = never, > 1 = forced.
void gemm_fp8(const torch::Tensor& a, const torch::Tensor& b, const torch::Tensor& a_scale_inv,
              const torch::Tensor& b_scale_inv, torch::Tensor out, const c10::optional<torch::Tensor>& bias,
              const c10::optional<torch::Tensor>& residual, const c10::optional<torch::Tensor>& aux, bool gelu,
              bool dgelu, bool accumulate, int64_t block_n, int64_t k_splits) {
  for (const torch::Tensor* t : {&a, &b}) {
    TORCH_CHECK(t->is_cuda() && t->device() == a.device(), "gemm_fp8: operands must be CUDA tensors on one device");
    TORCH_CHECK(t->dim() == 2 && t->stride(1) == 1, "gemm_fp8: operands must be 2-D with unit inner stride");
    TORCH_CHECK(t->stride(0) % 16 == 0 && reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0,
                "gemm_fp8: operand rows must be 16-byte aligned (leading dimension a multiple of 16)");
  }
  TORCH_CHECK(is_fp8(a), "gemm_fp8: a must be float8_e4m3fn or float8_e5m2");
  TORCH_CHECK(b.scalar_type() == torch::kFloat8_e4m3fn, "gemm_fp8: b must be float8_e4m3fn");
  const int64_t M = a.size(0), K = a.size(1), N = b.size(0);
  TORCH_CHECK(b.size(1) == K, "gemm_fp8: contraction dims differ: ", K, " vs ", b.size(1));
  TORCH_CHECK(K % 16 == 0, "gemm_fp8: K (", K, ") must be a multiple of 16");
  TORCH_CHECK(N % 8 == 0, "gemm_fp8: N must be a multiple of 8");
  for (const torch::Tensor* t : {&a_scale_inv, &b_scale_inv})
    TORCH_CHECK(t->is_cuda() && t->device() == a.device() && t->scalar_type() == torch::kFloat32 && t->numel() >= 1,
                "gemm_fp8: scale_inv must be an fp32 CUDA scalar");
  c10::cuda::CUDAGuard guard(a.device());
  TORCH_CHECK(out.is_cuda() && out.dim() == 2 && out.stride(1) == 1 && out.size(0) == M && out.size(1) == N,
              "gemm_fp8: out must be a 2-D CUDA tensor [M, N] with unit inner stride");
  const bool f32 = out.scalar_type() == torch::kFloat32;
  TORCH_CHECK(f32 || out.scalar_type() == torch::kBFloat16, "gemm_fp8: out must be bf16 or fp32");
  TORCH_CHECK(out.stride(0) % 8 == 0 && reinterpret_cast<uintptr_t>(out.data_ptr()) % 16 == 0,
              "gemm_fp8: out must be 16-byte aligned with a leading dimension that is a multiple of 8");
  TORCH_CHECK(!f32 || (!bias.has_value() && !residual.has_value() && !aux.has_value() && !gelu && !dgelu),
              "gemm_fp8: an fp32 out takes no epilogue input");
  TORCH_CHECK(f32 || (!accumulate && k_splits <= 1), "gemm_fp8: accumulate / k_splits need an fp32 out");
  TORCH_CHECK(!(gelu && dgelu) && !(dgelu && residual.has_value()), "gemm_fp8: gelu, dgelu and residual conflict");
  TORCH_CHECK((gelu || dgelu) || !aux.has_value(), "gemm_fp8: aux is the GELU pre-activation (gelu / dgelu)");
  TORCH_CHECK(!dgelu || aux.has_value(), "gemm_fp8: dgelu needs aux");
  TORCH_CHECK(block_n == 0 || block_n == 64 || block_n == 128, "gemm_fp8: block_n must be 0 (auto), 64 or 128");
  PgGemmDesc d;
  memset(&d, 0, sizeof(d));
  d.A = a.data_ptr();
  d.B = b.data_ptr();
  d.M = (int)M; d.N = (int)N; d.K = (int)K;
  d.lda = (int)a.stride(0);
  d.ldb = (int)b.stride(0);
  d.out = out.data_ptr();
  d.ldc = (int)out.stride(0);
  d.flags = (f32 ? 8 : 0) | (gelu ? 2 : 0) | (dgelu ? 32 : 0) | (accumulate ? 16 : 0);
  if (bias.has_value()) {
    TORCH_CHECK(bias->is_cuda() && bias->scalar_type() == torch::kBFloat16 && bias->numel() == N && bias->is_contiguous(),
                "gemm_fp8: bias must be contiguous bf16 [N]");
    d.bias = bias->data_ptr();
    d.flags |= 1;
  }
  if (residual.has_value()) {
    check_bf16_2d(*residual, "residual");
    TORCH_CHECK(residual->size(0) == M && residual->size(1) == N, "gemm_fp8: residual must be [M, N]");
    d.residual = residual->data_ptr();
    d.ldr = (int)residual->stride(0);
    d.flags |= 4;
  }
  if (aux.has_value()) {
    check_bf16_2d(*aux, "aux");
    TORCH_CHECK(aux->size(0) == M && aux->size(1) == N && aux->stride(0) == out.stride(0), "gemm_fp8: aux must match out");
    d.aux = aux->data_ptr();
  }
  d.block_n = (int)block_n;
  d.k_splits = (int)k_splits;
  d.num_chunks = 1;
  d.fmt = a.scalar_type() == torch::kFloat8_e5m2 ? 2 : 1;
  d.a_scale_inv = a_scale_inv.data_ptr<float>();
  d.b_scale_inv = b_scale_inv.data_ptr<float>();
  TORCH_CHECK(pg_gemm_bf16(&d, cur_stream()) == 0, "gemm_fp8 failed");
}

// Per-tensor FP8 cast of x bf16 [R, C] (contiguous, C % 8 == 0): amax (fp32 workspace, >= 1 element) = max |x|, then
// each given output: codes [R, C] and codes_t [C, R] (float8_e5m2 when e5m2, else float8_e4m3fn), scale_inv (fp32
// scalar) and colsum (fp32 [C], the column sums of x added into it).  Format: csrc/fp8_cast.cu.
void fp8_quantize(const torch::Tensor& x, bool e5m2, torch::Tensor amax, const c10::optional<torch::Tensor>& codes,
                  const c10::optional<torch::Tensor>& codes_t, const c10::optional<torch::Tensor>& scale_inv,
                  const c10::optional<torch::Tensor>& colsum) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && x.dim() == 2 && x.scalar_type() == torch::kBFloat16,
              "fp8_quantize: x must be a contiguous 2-D bf16 CUDA tensor");
  const int64_t R = x.size(0), C = x.size(1);
  TORCH_CHECK(C % 8 == 0, "fp8_quantize: the column count (", C, ") must be a multiple of 8");
  TORCH_CHECK(R < (int64_t(1) << 31) && C < (int64_t(1) << 31), "fp8_quantize: x is too large");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0, "fp8_quantize: x must be 16-byte aligned");
  c10::cuda::CUDAGuard guard(x.device());
  auto on_dev = [&](const torch::Tensor& t) { return t.is_cuda() && t.device() == x.device() && t.is_contiguous(); };
  TORCH_CHECK(on_dev(amax) && amax.scalar_type() == torch::kFloat32 && amax.numel() >= 1,
              "fp8_quantize: amax must be an fp32 CUDA workspace on x's device");
  const auto dt = e5m2 ? torch::kFloat8_e5m2 : torch::kFloat8_e4m3fn;
  if (codes.has_value())
    TORCH_CHECK(on_dev(*codes) && codes->scalar_type() == dt && codes->size(0) == R && codes->size(1) == C &&
                    reinterpret_cast<uintptr_t>(codes->data_ptr()) % 8 == 0,
                "fp8_quantize: codes must be a contiguous 8-byte-aligned ", e5m2 ? "float8_e5m2" : "float8_e4m3fn",
                " tensor [R, C]");
  if (codes_t.has_value())
    TORCH_CHECK(on_dev(*codes_t) && codes_t->scalar_type() == dt && codes_t->size(0) == C && codes_t->size(1) == R &&
                    reinterpret_cast<uintptr_t>(codes_t->data_ptr()) % 16 == 0,
                "fp8_quantize: codes_t must be a contiguous 16-byte-aligned ", e5m2 ? "float8_e5m2" : "float8_e4m3fn",
                " tensor [C, R]");
  if (scale_inv.has_value())
    TORCH_CHECK(on_dev(*scale_inv) && scale_inv->scalar_type() == torch::kFloat32 && scale_inv->numel() >= 1,
                "fp8_quantize: scale_inv must be an fp32 CUDA scalar");
  if (colsum.has_value())
    TORCH_CHECK(on_dev(*colsum) && colsum->scalar_type() == torch::kFloat32 && colsum->numel() == C,
                "fp8_quantize: colsum must be a contiguous fp32 CUDA tensor of ", C, " elements");
  TORCH_CHECK(pg_fp8_amax(x.data_ptr(), x.numel(), amax.data_ptr<float>(), cur_stream()) == 0, "fp8_amax failed");
  TORCH_CHECK(pg_fp8_cast(x.data_ptr(), (int)R, (int)C, e5m2 ? 1 : 0, amax.data_ptr<float>(),
                          codes.has_value() ? codes->data_ptr() : nullptr,
                          codes_t.has_value() ? codes_t->data_ptr() : nullptr,
                          scale_inv.has_value() ? scale_inv->data_ptr<float>() : nullptr,
                          colsum.has_value() ? colsum->data_ptr<float>() : nullptr, cur_stream()) == 0,
              "fp8_cast failed");
}

// {"peer": [ptr per data-parallel rank], "local": ptr, "start": elems, "seg": elems, "scalar": 0/1} -> PgGradRS
bool parse_grad_rs(const py::dict& d, PgGradRS* out) {
  memset(out, 0, sizeof(*out));
  if (!d.contains("peer")) return false;
  auto peers = d["peer"].cast<std::vector<int64_t>>();
  TORCH_CHECK(peers.size() >= 2 && peers.size() <= PG_MAX_PEERS, "grad_rs: 2..", PG_MAX_PEERS, " peers");
  for (size_t i = 0; i < peers.size(); ++i) out->peer[i] = reinterpret_cast<float*>(peers[i]);
  out->local = reinterpret_cast<const float*>(d["local"].cast<int64_t>());
  out->start = d["start"].cast<int64_t>();
  out->seg = d["seg"].cast<int64_t>();
  out->world = (int)peers.size();
  out->scalar_red = d.contains("scalar") ? d["scalar"].cast<int>() : 0;
  TORCH_CHECK(out->seg > 0 && out->seg % 4 == 0 && out->start % 4 == 0, "grad_rs: start / seg must be multiples of 4");
  return true;
}

#define PG_CUDA(t) TORCH_CHECK((t).is_cuda() && (t).is_contiguous(), #t " must be a contiguous CUDA tensor")
#define PG_BF16(t) TORCH_CHECK((t).scalar_type() == torch::kBFloat16, #t " must be bf16")
#define PG_F32(t) TORCH_CHECK((t).scalar_type() == torch::kFloat32, #t " must be fp32")
#define PG_ALIGNED(t, bytes) \
  TORCH_CHECK(reinterpret_cast<uintptr_t>((t).data_ptr()) % (bytes) == 0, #t " must be " #bytes "-byte aligned")

const void* opt_ptr(const c10::optional<torch::Tensor>& t) { return t.has_value() ? t->data_ptr() : nullptr; }

// y = LN(x) (or LN(table[ids]) / table[ids] when ids is given); returns nothing, fills y/mean/rstd
void layernorm_fwd(const torch::Tensor& x, const c10::optional<torch::Tensor>& ids, int64_t vocab_start,
                   int64_t vocab_end, const torch::Tensor& gamma, const torch::Tensor& beta, torch::Tensor y,
                   c10::optional<torch::Tensor> mean, c10::optional<torch::Tensor> rstd, double eps, bool apply_ln) {
  PG_CUDA(x); PG_BF16(x); PG_CUDA(y); PG_BF16(y); PG_CUDA(gamma); PG_BF16(gamma); PG_CUDA(beta); PG_BF16(beta);
  c10::cuda::CUDAGuard guard(x.device());
  const int h = (int)y.size(-1);
  const int rows = (int)(y.numel() / h);
  TORCH_CHECK(x.size(-1) == h, "hidden size mismatch");
  const int64_t* idp = nullptr;
  if (ids.has_value()) { PG_CUDA(*ids); TORCH_CHECK(ids->scalar_type() == torch::kInt64 && ids->numel() == rows, "ids must be int64 [rows]"); idp = ids->data_ptr<int64_t>(); }
  else { TORCH_CHECK(x.numel() == y.numel(), "x/y size mismatch"); }
  float* mp = mean.has_value() ? mean->data_ptr<float>() : nullptr;
  float* rp = rstd.has_value() ? rstd->data_ptr<float>() : nullptr;
  TORCH_CHECK(pg_layernorm_fwd(x.data_ptr(), idp, (int)vocab_start, (int)vocab_end, gamma.data_ptr(), beta.data_ptr(),
                               y.data_ptr(), mp, rp, rows, h, (float)eps, apply_ln, cur_stream()) == 0, "layernorm_fwd failed");
}

void layernorm_bwd(const torch::Tensor& dy, const torch::Tensor& x, const torch::Tensor& gamma, const torch::Tensor& mean,
                   const torch::Tensor& rstd, const c10::optional<torch::Tensor>& dx_extra, torch::Tensor dx,
                   c10::optional<torch::Tensor> dgamma, c10::optional<torch::Tensor> dbeta) {
  PG_CUDA(dy); PG_BF16(dy); PG_CUDA(x); PG_BF16(x); PG_CUDA(dx); PG_BF16(dx); PG_CUDA(mean); PG_F32(mean); PG_CUDA(rstd); PG_F32(rstd);
  c10::cuda::CUDAGuard guard(x.device());
  const int h = (int)x.size(-1);
  const int rows = (int)(x.numel() / h);
  float* dg = nullptr; float* db = nullptr;
  if (dgamma.has_value()) { PG_F32(*dgamma); PG_F32(*dbeta); dg = dgamma->data_ptr<float>(); db = dbeta->data_ptr<float>(); }
  TORCH_CHECK(pg_layernorm_bwd(dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), mean.data_ptr<float>(), rstd.data_ptr<float>(),
                               opt_ptr(dx_extra), dx.data_ptr(), dg, db, rows, h, cur_stream()) == 0, "layernorm_bwd failed");
}

void colsum(const torch::Tensor& x, torch::Tensor out) {
  check_bf16_2d(x, "x"); PG_CUDA(out); PG_F32(out);
  c10::cuda::CUDAGuard guard(x.device());
  TORCH_CHECK(out.numel() == x.size(1), "out must have one entry per column");
  TORCH_CHECK(pg_colsum(x.data_ptr(), (int)x.stride(0), out.data_ptr<float>(), (int)x.size(0), (int)x.size(1), cur_stream()) == 0, "colsum failed");
}

void embedding_bwd(const torch::Tensor& dx, const torch::Tensor& ids, torch::Tensor dw, int64_t vocab_start, int64_t vocab_end,
                   const py::dict& grad_rs) {
  PG_CUDA(dx); PG_BF16(dx); PG_CUDA(ids); PG_CUDA(dw); PG_F32(dw);
  c10::cuda::CUDAGuard guard(dx.device());
  const int h = (int)dx.size(-1);
  const int rows = (int)(dx.numel() / h);
  TORCH_CHECK(ids.scalar_type() == torch::kInt64 && ids.numel() == rows, "ids must be int64 [rows]");
  // the kernel adds rows in chunks of 8 columns: any other width would drop the last columns
  TORCH_CHECK(h % 8 == 0, "embedding_bwd: hidden size must be a multiple of 8");
  PG_ALIGNED(dx, 16);
  PgGradRS grs;
  const bool inl = parse_grad_rs(grad_rs, &grs);
  TORCH_CHECK(pg_embedding_bwd(dx.data_ptr(), ids.data_ptr<int64_t>(), dw.data_ptr<float>(), rows, h, (int)vocab_start, (int)vocab_end,
                               inl ? &grs : nullptr, cur_stream()) == 0, "embedding_bwd failed");
}

void ce_stats(const torch::Tensor& logits, const torch::Tensor& targets, torch::Tensor stats, int64_t vocab_start) {
  check_bf16_2d(logits, "logits"); PG_CUDA(targets); PG_CUDA(stats); PG_F32(stats);
  c10::cuda::CUDAGuard guard(logits.device());
  const int rows = (int)logits.size(0);
  TORCH_CHECK(targets.scalar_type() == torch::kInt64 && targets.numel() == rows && stats.numel() == rows * 3, "bad targets/stats");
  TORCH_CHECK(pg_ce_stats(logits.data_ptr(), (int)logits.stride(0), targets.data_ptr<int64_t>(), stats.data_ptr<float>(), rows, (int)logits.size(1), (int)vocab_start, cur_stream()) == 0, "ce_stats failed");
}

void ce_combine(const torch::Tensor& part, const torch::Tensor& logits, const torch::Tensor& targets, torch::Tensor stats,
                int64_t vocab_start) {
  check_bf16_2d(logits, "logits"); PG_CUDA(part); PG_F32(part); PG_CUDA(targets); PG_CUDA(stats); PG_F32(stats);
  c10::cuda::CUDAGuard guard(logits.device());
  const int rows = (int)logits.size(0);
  TORCH_CHECK(part.dim() == 3 && part.size(0) == rows && part.size(2) == 2, "part must be [rows, nparts, 2]");
  TORCH_CHECK(targets.scalar_type() == torch::kInt64 && targets.numel() == rows && stats.numel() == rows * 3, "bad targets/stats");
  TORCH_CHECK(pg_ce_combine(part.data_ptr<float>(), (int)part.size(1), logits.data_ptr(), (int)logits.stride(0), targets.data_ptr<int64_t>(),
                            stats.data_ptr<float>(), rows, (int)logits.size(1), (int)vocab_start, cur_stream()) == 0, "ce_combine failed");
}

void ce_finalize(torch::Tensor logits, const torch::Tensor& targets, const torch::Tensor& gstats, torch::Tensor loss_rows,
                 int64_t vocab_start, const c10::optional<torch::Tensor>& grad_scale, int64_t ignore_index, bool write_grad) {
  const float* gsp = nullptr;
  if (grad_scale.has_value()) { PG_CUDA(*grad_scale); PG_F32(*grad_scale); gsp = grad_scale->data_ptr<float>(); }
  check_bf16_2d(logits, "logits"); PG_CUDA(targets); PG_CUDA(gstats); PG_F32(gstats); PG_CUDA(loss_rows); PG_F32(loss_rows);
  c10::cuda::CUDAGuard guard(logits.device());
  const int rows = (int)logits.size(0);
  TORCH_CHECK(pg_ce_finalize(logits.data_ptr(), (int)logits.stride(0), targets.data_ptr<int64_t>(), gstats.data_ptr<float>(), loss_rows.data_ptr<float>(),
                             rows, (int)logits.size(1), (int)vocab_start, gsp, ignore_index, write_grad, cur_stream()) == 0, "ce_finalize failed");
}

void adam_step(torch::Tensor master, torch::Tensor m, torch::Tensor v, const torch::Tensor& grad, c10::optional<torch::Tensor> param_bf16,
               double lr, double beta1, double beta2, double eps, double wd, int64_t step, double grad_scale, bool adamw,
               bool zero_grad) {
  PG_CUDA(master); PG_F32(master); PG_CUDA(m); PG_F32(m); PG_CUDA(v); PG_F32(v); PG_CUDA(grad); PG_F32(grad);
  c10::cuda::CUDAGuard guard(master.device());
  const int64_t n = master.numel();
  TORCH_CHECK(m.numel() == n && v.numel() == n && grad.numel() == n, "adam: size mismatch");
  // float4 accesses of the fp32 buffers, 8-byte stores of four bf16 parameters
  PG_ALIGNED(master, 16); PG_ALIGNED(m, 16); PG_ALIGNED(v, 16); PG_ALIGNED(grad, 16);
  void* pb = nullptr;
  if (param_bf16.has_value()) { PG_CUDA(*param_bf16); PG_BF16(*param_bf16); TORCH_CHECK(param_bf16->numel() == n, "adam: bf16 param size mismatch");
    PG_ALIGNED(*param_bf16, 8); pb = param_bf16->data_ptr(); }
  const double bc1 = 1.0 - std::pow(beta1, (double)step), bc2 = 1.0 - std::pow(beta2, (double)step);
  TORCH_CHECK(pg_adam(master.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(), grad.data_ptr<float>(), pb, n, (float)lr, (float)beta1, (float)beta2,
                      (float)eps, (float)wd, (float)bc1, (float)bc2, (float)grad_scale, adamw, zero_grad, cur_stream()) == 0, "adam failed");
}

// ZeRO-1: this rank's slice (seg elements at flat offset first + b * bucket_stride) of nb equally sized buckets in ONE launch;
// master / m / v hold the nb slices back to back
void adam_step_strided(torch::Tensor master, torch::Tensor m, torch::Tensor v, torch::Tensor flat_grad, c10::optional<torch::Tensor> flat_param,
                       int64_t first, int64_t seg, int64_t bucket_stride, int64_t nb, double lr, double beta1, double beta2, double eps,
                       double wd, int64_t step, double grad_scale, bool adamw, bool zero_grad) {
  PG_CUDA(master); PG_F32(master); PG_CUDA(m); PG_F32(m); PG_CUDA(v); PG_F32(v); PG_CUDA(flat_grad); PG_F32(flat_grad);
  c10::cuda::CUDAGuard guard(master.device());
  TORCH_CHECK(master.numel() == seg * nb && m.numel() == seg * nb && v.numel() == seg * nb, "adam_strided: state size mismatch");
  TORCH_CHECK(first >= 0 && first + (nb - 1) * bucket_stride + seg <= flat_grad.numel(), "adam_strided: range outside the flat buffer");
  // float4 accesses from flat_grad + first (seg and bucket_stride are checked by the launcher), 8-byte parameter stores
  TORCH_CHECK(first % 4 == 0, "adam_strided: first must be a multiple of 4");
  PG_ALIGNED(master, 16); PG_ALIGNED(m, 16); PG_ALIGNED(v, 16); PG_ALIGNED(flat_grad, 16);
  void* pb = nullptr;
  if (flat_param.has_value()) { PG_CUDA(*flat_param); PG_BF16(*flat_param); TORCH_CHECK(flat_param->numel() == flat_grad.numel(), "flat sizes differ");
    PG_ALIGNED(*flat_param, 8); pb = reinterpret_cast<char*>(flat_param->data_ptr()) + 2 * first; }
  const double bc1 = 1.0 - std::pow(beta1, (double)step), bc2 = 1.0 - std::pow(beta2, (double)step);
  TORCH_CHECK(pg_adam_strided(master.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(), flat_grad.data_ptr<float>() + first, pb, seg,
                              bucket_stride, nb, (float)lr, (float)beta1, (float)beta2, (float)eps, (float)wd, (float)bc1, (float)bc2,
                              (float)grad_scale, adamw, zero_grad, cur_stream()) == 0, "adam_strided failed");
}

void accum_bf16_to_f32(const torch::Tensor& src, torch::Tensor dst, double scale, bool accumulate) {
  PG_CUDA(src); PG_BF16(src); PG_CUDA(dst); PG_F32(dst);
  c10::cuda::CUDAGuard guard(src.device());
  TORCH_CHECK(src.numel() == dst.numel(), "size mismatch");
  // 16-byte loads of src and float4 stores to dst
  PG_ALIGNED(src, 16); PG_ALIGNED(dst, 16);
  TORCH_CHECK(pg_accum_bf16_to_f32(src.data_ptr(), dst.data_ptr<float>(), src.numel(), (float)scale, accumulate, cur_stream()) == 0, "accum failed");
}


// dst (a view into the local flat fp32 gradient buffer) += scale * src through the in-kernel reduce-scatter
void grad_rs_accum(const torch::Tensor& src, torch::Tensor dst, double scale, const py::dict& grad_rs) {
  PG_CUDA(src); PG_CUDA(dst); PG_F32(dst);
  TORCH_CHECK(src.scalar_type() == torch::kBFloat16 || src.scalar_type() == torch::kFloat32, "src must be bf16 or fp32");
  TORCH_CHECK(src.numel() == dst.numel(), "size mismatch");
  c10::cuda::CUDAGuard guard(src.device());
  PgGradRS grs;
  TORCH_CHECK(parse_grad_rs(grad_rs, &grs), "grad_rs_accum needs a grad_rs descriptor");
  TORCH_CHECK(pg_grad_rs_accum(src.data_ptr(), src.scalar_type() == torch::kFloat32, dst.data_ptr<float>(), src.numel(), (float)scale,
                               &grs, cur_stream()) == 0, "grad_rs_accum failed");
}

// seg_start: optional int32 [B*S] row-relative document starts of packed sequences (see attention_sm90.cu)
const int* seg_start_ptr(const c10::optional<torch::Tensor>& seg_start, const torch::Tensor& qkv, int64_t B, int64_t S) {
  if (!seg_start.has_value()) return nullptr;
  const torch::Tensor& t = *seg_start;
  TORCH_CHECK(t.is_cuda() && t.device() == qkv.device(), "seg_start must be on the device of qkv");
  TORCH_CHECK(t.scalar_type() == torch::kInt32, "seg_start must be int32");
  TORCH_CHECK(t.is_contiguous(), "seg_start must be contiguous");
  TORCH_CHECK(t.numel() == B * S, "seg_start must hold B*S = ", B * S, " entries, got ", t.numel());
  return t.data_ptr<int>();
}

void attention_fwd(const torch::Tensor& qkv, const torch::Tensor& slopes, torch::Tensor out, torch::Tensor lse,
                   int64_t B, int64_t S, int64_t H, int64_t D, double softmax_scale,
                   const c10::optional<torch::Tensor>& seg_start) {
  PG_CUDA(qkv); PG_BF16(qkv); PG_CUDA(out); PG_BF16(out); PG_CUDA(slopes); PG_F32(slopes); PG_CUDA(lse); PG_F32(lse);
  c10::cuda::CUDAGuard guard(qkv.device());
  TORCH_CHECK(qkv.numel() == B * S * H * 3 * D && out.numel() == B * S * H * D && lse.numel() == B * H * S && slopes.numel() == H, "attention_fwd: shape mismatch");
  const int* seg = seg_start_ptr(seg_start, qkv, B, S);
  TORCH_CHECK(pg_attention_fwd(qkv.data_ptr(), slopes.data_ptr<float>(), out.data_ptr(), lse.data_ptr<float>(), (int)B, (int)S, (int)H, (int)D, (float)softmax_scale, seg, cur_stream()) == 0, "attention_fwd failed");
}

void attention_bwd(const torch::Tensor& qkv, const torch::Tensor& slopes, const torch::Tensor& out, const torch::Tensor& lse,
                   const torch::Tensor& dout, torch::Tensor dqkv, int64_t B, int64_t S, int64_t H, int64_t D,
                   double softmax_scale, const c10::optional<torch::Tensor>& seg_start) {
  PG_CUDA(qkv); PG_BF16(qkv); PG_CUDA(out); PG_BF16(out); PG_CUDA(dout); PG_BF16(dout); PG_CUDA(dqkv); PG_BF16(dqkv); PG_CUDA(lse); PG_F32(lse);
  c10::cuda::CUDAGuard guard(qkv.device());
  TORCH_CHECK(dout.numel() == out.numel() && dqkv.numel() == qkv.numel(), "attention_bwd: shape mismatch");
  const int* seg = seg_start_ptr(seg_start, qkv, B, S);
  auto dq_acc = torch::empty({B * S, H * D}, qkv.options().dtype(torch::kFloat32));
  auto stats = torch::empty({pg_attention_bwd_stats_floats((int)B, (int)S, (int)H)}, qkv.options().dtype(torch::kFloat32));
  TORCH_CHECK(pg_attention_bwd(qkv.data_ptr(), slopes.data_ptr<float>(), out.data_ptr(), lse.data_ptr<float>(), dout.data_ptr(), dqkv.data_ptr(),
                               dq_acc.data_ptr<float>(), stats.data_ptr<float>(), (int)B, (int)S, (int)H, (int)D, (float)softmax_scale, seg, cur_stream()) == 0, "attention_bwd failed");
}

// One decoding step (decode_sm90.cu): writes the new k / v of qkv [B, H*3*D] at column pos of k_cache / v_cache
// [B, H, capacity, D] and returns attention over keys lead[b] .. pos in out [B, H*D].  ticket: int32, at least B*H
// entries, all zero (the kernel leaves them zero).
void decode_attention(const torch::Tensor& qkv, torch::Tensor k_cache, torch::Tensor v_cache, const torch::Tensor& slopes,
                      int64_t pos, const c10::optional<torch::Tensor>& lead, torch::Tensor out, torch::Tensor ticket,
                      double softmax_scale) {
  PG_CUDA(qkv); PG_BF16(qkv); PG_CUDA(k_cache); PG_BF16(k_cache); PG_CUDA(v_cache); PG_BF16(v_cache);
  PG_CUDA(out); PG_BF16(out); PG_CUDA(slopes); PG_F32(slopes); PG_CUDA(ticket);
  TORCH_CHECK(ticket.scalar_type() == torch::kInt32, "ticket must be int32");
  TORCH_CHECK(k_cache.dim() == 4 && v_cache.sizes() == k_cache.sizes(), "k_cache / v_cache must be [B, H, capacity, D]");
  const int64_t B = k_cache.size(0), H = k_cache.size(1), cap = k_cache.size(2), D = k_cache.size(3);
  TORCH_CHECK(D == 64 || D == 80 || D == 128, "decode_attention: head size ", D, " has no kernel (64, 80, 128)");
  TORCH_CHECK(qkv.numel() == B * H * 3 * D && out.numel() == B * H * D && slopes.numel() == H, "decode_attention: shape mismatch");
  TORCH_CHECK(ticket.numel() >= B * H, "ticket must hold at least B*H = ", B * H, " entries");
  TORCH_CHECK(0 <= pos && pos < cap, "decode_attention: pos ", pos, " outside the cache capacity ", cap);
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&qkv, &k_cache, &v_cache, &out, &slopes, &ticket})
    TORCH_CHECK(t->device() == qkv.device(), "decode_attention: tensors on different devices");
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&qkv, &k_cache, &v_cache})
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0, "decode_attention: qkv and caches must be 16B aligned");
  const int* lp = nullptr;
  if (lead.has_value()) {
    PG_CUDA(*lead);
    TORCH_CHECK(lead->scalar_type() == torch::kInt32 && lead->numel() == B && lead->device() == qkv.device(),
                "lead must be int32 [B] on the device of qkv");
    lp = lead->data_ptr<int>();
  }
  c10::cuda::CUDAGuard guard(qkv.device());
  const int splits = pg_decode_splits((int)B, (int)H, (int)pos + 1);
  torch::Tensor part;
  if (splits > 1) part = torch::empty({B * H * splits * (D + 2)}, qkv.options().dtype(torch::kFloat32));
  TORCH_CHECK(pg_decode_attention(qkv.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), slopes.data_ptr<float>(), lp,
                                  out.data_ptr(), splits > 1 ? part.data_ptr<float>() : nullptr, ticket.data_ptr<int>(),
                                  (int)B, (int)H, (int)D, (int)cap, (int)pos, splits, (float)softmax_scale,
                                  cur_stream()) == 0, "decode_attention failed");
}

void check_pools(const torch::Tensor& qkv, const torch::Tensor& k_pool, const torch::Tensor& v_pool, const char* op) {
  PG_CUDA(qkv); PG_BF16(qkv); PG_CUDA(k_pool); PG_BF16(k_pool); PG_CUDA(v_pool); PG_BF16(v_pool);
  TORCH_CHECK(k_pool.dim() == 4 && v_pool.sizes() == k_pool.sizes(), op, ": k_pool / v_pool must be [num_pages, H, 64, D]");
  TORCH_CHECK(k_pool.size(2) == 64, op, ": the pools' page dimension must be 64, got ", k_pool.size(2));
  const int64_t D = k_pool.size(3);
  TORCH_CHECK(D == 64 || D == 80 || D == 128, op, ": head size ", D, " has no kernel (64, 80, 128)");
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&k_pool, &v_pool})
    TORCH_CHECK(t->device() == qkv.device(), op, ": tensors on different devices");
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&qkv, &k_pool, &v_pool})
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0, op, ": qkv and pools must be 16B aligned");
}

// One decoding step over paged pools (decode_sm90.cu, PAGED): row b writes its new k / v of qkv [B, H*3*D] at
// position pos[b] (the slot of page table[b, pos[b] / 64]) and attends to keys 0 .. pos[b]; out [B, H*D].  table
// (int32 [B, max_pages]) and pos (int32 [B]) stay on the device: the caller guarantees pos[b] <= max_pos, that
// table[b, 0 .. pos[b] / 64] are pages of the pool and that no two rows share a page.  ticket as for decode_attention.
void paged_decode_attention(const torch::Tensor& qkv, torch::Tensor k_pool, torch::Tensor v_pool,
                            const torch::Tensor& table, const torch::Tensor& pos, int64_t max_pos,
                            const torch::Tensor& slopes, torch::Tensor out, torch::Tensor ticket, double softmax_scale) {
  check_pools(qkv, k_pool, v_pool, "paged_decode_attention");
  PG_CUDA(out); PG_BF16(out); PG_CUDA(slopes); PG_F32(slopes); PG_CUDA(ticket); PG_CUDA(table); PG_CUDA(pos);
  TORCH_CHECK(ticket.scalar_type() == torch::kInt32 && table.scalar_type() == torch::kInt32 &&
              pos.scalar_type() == torch::kInt32, "paged_decode_attention: ticket, table and pos must be int32");
  TORCH_CHECK(table.dim() == 2 && table.size(1) >= 1, "paged_decode_attention: table must be [B, max_pages]");
  const int64_t B = table.size(0), H = k_pool.size(1), D = k_pool.size(3), max_pages = table.size(1);
  TORCH_CHECK(pos.numel() == B && qkv.numel() == B * H * 3 * D && out.numel() == B * H * D && slopes.numel() == H,
              "paged_decode_attention: shape mismatch");
  TORCH_CHECK(ticket.numel() >= B * H, "ticket must hold at least B*H = ", B * H, " entries");
  TORCH_CHECK(0 <= max_pos && max_pos < max_pages * 64, "paged_decode_attention: max_pos ", max_pos,
              " outside the ", max_pages, " pages of a table row");
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&out, &slopes, &ticket, &table, &pos})
    TORCH_CHECK(t->device() == qkv.device(), "paged_decode_attention: tensors on different devices");
  if (B == 0) return;
  c10::cuda::CUDAGuard guard(qkv.device());
  const int splits = pg_decode_splits((int)B, (int)H, (int)max_pos + 1);
  torch::Tensor part;
  if (splits > 1) part = torch::empty({B * H * splits * (D + 2)}, qkv.options().dtype(torch::kFloat32));
  TORCH_CHECK(pg_paged_decode_attention(qkv.data_ptr(), k_pool.data_ptr(), v_pool.data_ptr(), table.data_ptr<int>(),
                                        pos.data_ptr<int>(), slopes.data_ptr<float>(), out.data_ptr(),
                                        splits > 1 ? part.data_ptr<float>() : nullptr, ticket.data_ptr<int>(), (int)B,
                                        (int)H, (int)D, (int)max_pages, (int)max_pos, splits, (float)softmax_scale,
                                        cur_stream()) == 0, "paged_decode_attention failed");
}

// Paged append attention (decode_sm90.cu, speculative verification): row b appends the tokens of qkv [N, H*3*D] rows
// cu_seqlens[b] .. cu_seqlens[b+1]-1 (1 to 8 of them) at positions pos[b] ..; each writes its k / v into its slot and
// attends to keys 0 .. its own position; out [N, H*D].  table, cu_seqlens and pos stay on the device: the caller
// guarantees that every row appends 1 to max_tokens (<= 8) tokens, pos[b] + its tokens - 1 <= max_pos, that table[b]
// holds pages of the pool for those positions and that no two rows share a page.  max_tokens picks the kernel's query
// tile.  ticket: int32, at least 8*B*H entries, all zero.
void paged_append_attention(const torch::Tensor& qkv, torch::Tensor k_pool, torch::Tensor v_pool,
                            const torch::Tensor& table, const torch::Tensor& cu_seqlens, const torch::Tensor& pos,
                            int64_t max_pos, int64_t max_tokens, const torch::Tensor& slopes, torch::Tensor out,
                            torch::Tensor ticket, double softmax_scale) {
  check_pools(qkv, k_pool, v_pool, "paged_append_attention");
  PG_CUDA(out); PG_BF16(out); PG_CUDA(slopes); PG_F32(slopes); PG_CUDA(ticket); PG_CUDA(table); PG_CUDA(cu_seqlens);
  PG_CUDA(pos);
  TORCH_CHECK(ticket.scalar_type() == torch::kInt32 && table.scalar_type() == torch::kInt32 &&
              cu_seqlens.scalar_type() == torch::kInt32 && pos.scalar_type() == torch::kInt32,
              "paged_append_attention: ticket, table, cu_seqlens and pos must be int32");
  TORCH_CHECK(table.dim() == 2 && table.size(1) >= 1 && table.is_contiguous(),
              "paged_append_attention: table must be a contiguous [B, max_pages]");
  const int64_t B = table.size(0), H = k_pool.size(1), D = k_pool.size(3), max_pages = table.size(1);
  TORCH_CHECK(cu_seqlens.numel() == B + 1 && pos.numel() == B && cu_seqlens.is_contiguous() && pos.is_contiguous(),
              "paged_append_attention: cu_seqlens must be [B+1] and pos [B] for the B = ", B, " table rows");
  TORCH_CHECK(qkv.dim() == 2 && qkv.size(1) == H * 3 * D && qkv.is_contiguous(),
              "paged_append_attention: qkv must be a contiguous [N, H*3*D]");
  const int64_t N = qkv.size(0);
  TORCH_CHECK(1 <= max_tokens && max_tokens <= 8, "paged_append_attention: max_tokens ", max_tokens,
              " outside 1 .. 8");
  TORCH_CHECK(B <= N && N <= max_tokens * B, "paged_append_attention: ", N, " tokens for ", B,
              " rows: every row appends 1 to max_tokens = ", max_tokens, " tokens");
  TORCH_CHECK(out.numel() == N * H * D && out.is_contiguous() && slopes.numel() == H,
              "paged_append_attention: shape mismatch");
  TORCH_CHECK(ticket.numel() >= 8 * B * H, "ticket must hold at least 8*B*H = ", 8 * B * H, " entries");
  TORCH_CHECK(0 <= max_pos && max_pos < max_pages * 64, "paged_append_attention: max_pos ", max_pos,
              " outside the ", max_pages, " pages of a table row");
  for (const torch::Tensor* t :
       std::initializer_list<const torch::Tensor*>{&out, &slopes, &ticket, &table, &cu_seqlens, &pos})
    TORCH_CHECK(t->device() == qkv.device(), "paged_append_attention: tensors on different devices");
  if (B == 0) return;
  c10::cuda::CUDAGuard guard(qkv.device());
  const int splits = pg_decode_splits((int)B, (int)H, (int)max_pos + 1);
  torch::Tensor part;
  if (splits > 1) part = torch::empty({B * H * 8 * splits * (D + 2)}, qkv.options().dtype(torch::kFloat32));
  TORCH_CHECK(pg_paged_append_attention(qkv.data_ptr(), k_pool.data_ptr(), v_pool.data_ptr(), table.data_ptr<int>(),
                                        cu_seqlens.data_ptr<int>(), pos.data_ptr<int>(), slopes.data_ptr<float>(),
                                        out.data_ptr(), splits > 1 ? part.data_ptr<float>() : nullptr,
                                        ticket.data_ptr<int>(), (int)B, (int)N, (int)H, (int)D, (int)max_pages,
                                        (int)max_pos, (int)max_tokens, splits, (float)softmax_scale,
                                        cur_stream()) == 0,
              "paged_append_attention failed");
}

// Paged prefill attention (attention_sm90.cu, PAGED): the new tokens of R sequences packed in qkv [N, H*3*D] (sequence
// r: rows cu_seqlens[r] .. cu_seqlens[r+1]-1 at positions start[r], ...) attend to keys 0 .. p of their own sequence,
// read from the pools through table [R, max_pages]; out [N, H*D].  The pools are not written.  cu_seqlens, start and
// table stay on the device: the caller guarantees max_len >= every sequence's new tokens, that table[r] holds pages of
// the pool for positions 0 .. start[r] + new tokens - 1, and that those slots were written.
void paged_prefill_attention(const torch::Tensor& qkv, const torch::Tensor& k_pool, const torch::Tensor& v_pool,
                             const torch::Tensor& table, const torch::Tensor& cu_seqlens, const torch::Tensor& start,
                             int64_t max_len, const torch::Tensor& slopes, torch::Tensor out, double softmax_scale) {
  check_pools(qkv, k_pool, v_pool, "paged_prefill_attention");
  PG_CUDA(out); PG_BF16(out); PG_CUDA(slopes); PG_F32(slopes); PG_CUDA(table); PG_CUDA(cu_seqlens); PG_CUDA(start);
  TORCH_CHECK(table.scalar_type() == torch::kInt32 && cu_seqlens.scalar_type() == torch::kInt32 &&
              start.scalar_type() == torch::kInt32, "paged_prefill_attention: table, cu_seqlens and start must be int32");
  TORCH_CHECK(table.dim() == 2 && table.size(1) >= 1 && table.is_contiguous(),
              "paged_prefill_attention: table must be a contiguous [R, max_pages]");
  const int64_t R = table.size(0), H = k_pool.size(1), D = k_pool.size(3), max_pages = table.size(1);
  const int64_t num_pages = k_pool.size(0);
  TORCH_CHECK(cu_seqlens.numel() == R + 1 && start.numel() == R, "paged_prefill_attention: cu_seqlens must be [R+1] and "
              "start [R] for the R = ", R, " table rows");
  TORCH_CHECK(qkv.dim() == 2 && qkv.size(1) == H * 3 * D && qkv.is_contiguous(),
              "paged_prefill_attention: qkv must be a contiguous [N, H*3*D]");
  const int64_t N = qkv.size(0);
  TORCH_CHECK(out.numel() == N * H * D && out.is_contiguous() && slopes.numel() == H,
              "paged_prefill_attention: shape mismatch");
  TORCH_CHECK(1 <= max_len && max_len <= max_pages * 64, "paged_prefill_attention: max_len ", max_len,
              " outside 1 .. the ", max_pages * 64, " positions of a table row");
  TORCH_CHECK(num_pages * H * 64 < (int64_t(1) << 31), "paged_prefill_attention: pools of ", num_pages * H * 64,
              " rows exceed the 2^31 rows a tensor map addresses");
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&out, &slopes, &table, &cu_seqlens, &start})
    TORCH_CHECK(t->device() == qkv.device(), "paged_prefill_attention: tensors on different devices");
  if (N == 0 || R == 0) return;
  c10::cuda::CUDAGuard guard(qkv.device());
  TORCH_CHECK(pg_paged_prefill_attention(qkv.data_ptr(), k_pool.data_ptr(), v_pool.data_ptr(), table.data_ptr<int>(),
                                         cu_seqlens.data_ptr<int>(), start.data_ptr<int>(), slopes.data_ptr<float>(),
                                         out.data_ptr(), (int)N, (int)R, (int)H, (int)D, (int)num_pages,
                                         (int)max_pages, (int)max_len, (float)softmax_scale, cur_stream()) == 0,
              "paged_prefill_attention failed");
}

// Prefill cache write: the k / v of every token n of qkv [N, H*3*D] into pool slot slot[n] (page * 64 + offset).  The
// caller guarantees every slot lies in the pool.
void paged_kv_write(const torch::Tensor& qkv, const torch::Tensor& slot, torch::Tensor k_pool, torch::Tensor v_pool) {
  check_pools(qkv, k_pool, v_pool, "paged_kv_write");
  PG_CUDA(slot);
  TORCH_CHECK(slot.scalar_type() == torch::kInt32 && slot.device() == qkv.device(), "paged_kv_write: slot must be int32 on the device of qkv");
  const int64_t N = slot.numel(), H = k_pool.size(1), D = k_pool.size(3);
  TORCH_CHECK(qkv.numel() == N * H * 3 * D, "paged_kv_write: qkv must be [N, H*3*D] for the N = ", N, " slots");
  c10::cuda::CUDAGuard guard(qkv.device());
  TORCH_CHECK(pg_paged_kv_write(qkv.data_ptr(), slot.data_ptr<int>(), k_pool.data_ptr(), v_pool.data_ptr(), (int)N,
                                (int)H, (int)D, cur_stream()) == 0, "paged_kv_write failed");
}

// FP8 pools: e4m3 codes [num_pages, H, 64, D] and fp32 scales [num_pages, H, 64] for K and for V.
void check_fp8_pools(const torch::Tensor& k_pool, const torch::Tensor& v_pool, const torch::Tensor& k_scales,
                     const torch::Tensor& v_scales, const torch::Device& device, const char* op) {
  PG_CUDA(k_pool); PG_CUDA(v_pool); PG_CUDA(k_scales); PG_CUDA(v_scales);
  TORCH_CHECK(k_pool.scalar_type() == torch::kFloat8_e4m3fn && v_pool.scalar_type() == torch::kFloat8_e4m3fn, op,
              ": k_pool / v_pool must be float8_e4m3fn");
  PG_F32(k_scales); PG_F32(v_scales);
  TORCH_CHECK(k_pool.dim() == 4 && v_pool.sizes() == k_pool.sizes(), op, ": k_pool / v_pool must be [num_pages, H, 64, D]");
  TORCH_CHECK(k_pool.size(2) == 64, op, ": the pools' page dimension must be 64, got ", k_pool.size(2));
  const int64_t D = k_pool.size(3);
  TORCH_CHECK(D == 64 || D == 80 || D == 128, op, ": head size ", D, " has no kernel (64, 80, 128)");
  TORCH_CHECK(k_scales.sizes() == k_pool.sizes().slice(0, 3) && v_scales.sizes() == k_scales.sizes(), op,
              ": k_scales / v_scales must be [num_pages, H, 64] like the pools, got ", k_scales.sizes(), " and ",
              v_scales.sizes());
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&k_pool, &v_pool, &k_scales, &v_scales})
    TORCH_CHECK(t->device() == device, op, ": tensors on different devices");
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&k_pool, &v_pool})
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0, op, ": pools must be 16B aligned");
}

// paged_kv_write into FP8 pools: every token's k / v quantized into its slot, with their scales.
void paged_kv_write_fp8(const torch::Tensor& qkv, const torch::Tensor& slot, torch::Tensor k_pool, torch::Tensor v_pool,
                        torch::Tensor k_scales, torch::Tensor v_scales) {
  PG_CUDA(qkv); PG_BF16(qkv); PG_CUDA(slot);
  check_fp8_pools(k_pool, v_pool, k_scales, v_scales, qkv.device(), "paged_kv_write_fp8");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(qkv.data_ptr()) % 16 == 0, "paged_kv_write_fp8: qkv must be 16B aligned");
  TORCH_CHECK(slot.scalar_type() == torch::kInt32 && slot.device() == qkv.device(), "paged_kv_write_fp8: slot must be int32 on the device of qkv");
  const int64_t N = slot.numel(), H = k_pool.size(1), D = k_pool.size(3);
  TORCH_CHECK(qkv.numel() == N * H * 3 * D, "paged_kv_write_fp8: qkv must be [N, H*3*D] for the N = ", N, " slots");
  c10::cuda::CUDAGuard guard(qkv.device());
  TORCH_CHECK(pg_paged_kv_write_fp8(qkv.data_ptr(), slot.data_ptr<int>(), k_pool.data_ptr(), v_pool.data_ptr(),
                                    k_scales.data_ptr<float>(), v_scales.data_ptr<float>(), (int)N, (int)H, (int)D,
                                    cur_stream()) == 0, "paged_kv_write_fp8 failed");
}

// paged_decode_attention over FP8 pools.  The key and value at pos[b] enter the attention from qkv, exactly, and are
// quantized into their slot.
void paged_decode_attention_fp8(const torch::Tensor& qkv, torch::Tensor k_pool, torch::Tensor v_pool,
                                torch::Tensor k_scales, torch::Tensor v_scales, const torch::Tensor& table,
                                const torch::Tensor& pos, int64_t max_pos, const torch::Tensor& slopes, torch::Tensor out,
                                torch::Tensor ticket, double softmax_scale) {
  PG_CUDA(qkv); PG_BF16(qkv);
  check_fp8_pools(k_pool, v_pool, k_scales, v_scales, qkv.device(), "paged_decode_attention_fp8");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(qkv.data_ptr()) % 16 == 0, "paged_decode_attention_fp8: qkv must be 16B aligned");
  PG_CUDA(out); PG_BF16(out); PG_CUDA(slopes); PG_F32(slopes); PG_CUDA(ticket); PG_CUDA(table); PG_CUDA(pos);
  TORCH_CHECK(ticket.scalar_type() == torch::kInt32 && table.scalar_type() == torch::kInt32 &&
              pos.scalar_type() == torch::kInt32, "paged_decode_attention_fp8: ticket, table and pos must be int32");
  TORCH_CHECK(table.dim() == 2 && table.size(1) >= 1, "paged_decode_attention_fp8: table must be [B, max_pages]");
  const int64_t B = table.size(0), H = k_pool.size(1), D = k_pool.size(3), max_pages = table.size(1);
  TORCH_CHECK(pos.numel() == B && qkv.numel() == B * H * 3 * D && out.numel() == B * H * D && slopes.numel() == H,
              "paged_decode_attention_fp8: shape mismatch");
  TORCH_CHECK(ticket.numel() >= B * H, "ticket must hold at least B*H = ", B * H, " entries");
  TORCH_CHECK(0 <= max_pos && max_pos < max_pages * 64, "paged_decode_attention_fp8: max_pos ", max_pos,
              " outside the ", max_pages, " pages of a table row");
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&out, &slopes, &ticket, &table, &pos})
    TORCH_CHECK(t->device() == qkv.device(), "paged_decode_attention_fp8: tensors on different devices");
  if (B == 0) return;
  c10::cuda::CUDAGuard guard(qkv.device());
  const int splits = pg_decode_splits((int)B, (int)H, (int)max_pos + 1);
  torch::Tensor part;
  if (splits > 1) part = torch::empty({B * H * splits * (D + 2)}, qkv.options().dtype(torch::kFloat32));
  TORCH_CHECK(pg_paged_decode_attention_fp8(qkv.data_ptr(), k_pool.data_ptr(), v_pool.data_ptr(),
                                            k_scales.data_ptr<float>(), v_scales.data_ptr<float>(), table.data_ptr<int>(),
                                            pos.data_ptr<int>(), slopes.data_ptr<float>(), out.data_ptr(),
                                            splits > 1 ? part.data_ptr<float>() : nullptr, ticket.data_ptr<int>(), (int)B,
                                            (int)H, (int)D, (int)max_pages, (int)max_pos, splits, (float)softmax_scale,
                                            cur_stream()) == 0, "paged_decode_attention_fp8 failed");
}

// Pages src[i] (int32 [n]) of the FP8 pools, dequantized, into pages dst[i] of the bf16 pools k_out / v_out
// [*, H, 64, D].  The caller guarantees that every id is a page of its pool.
void paged_kv_dequantize(const torch::Tensor& k_pool, const torch::Tensor& v_pool, const torch::Tensor& k_scales,
                         const torch::Tensor& v_scales, const torch::Tensor& src, const torch::Tensor& dst,
                         torch::Tensor k_out, torch::Tensor v_out) {
  check_fp8_pools(k_pool, v_pool, k_scales, v_scales, k_pool.device(), "paged_kv_dequantize");
  PG_CUDA(src); PG_CUDA(dst); PG_CUDA(k_out); PG_BF16(k_out); PG_CUDA(v_out); PG_BF16(v_out);
  TORCH_CHECK(src.scalar_type() == torch::kInt32 && dst.scalar_type() == torch::kInt32 && src.numel() == dst.numel(),
              "paged_kv_dequantize: src and dst must be int32 page lists of one length");
  TORCH_CHECK(k_out.dim() == 4 && v_out.sizes() == k_out.sizes() && k_out.size(1) == k_pool.size(1) &&
              k_out.size(2) == 64 && k_out.size(3) == k_pool.size(3),
              "paged_kv_dequantize: k_out / v_out must be [pages, H, 64, D] like the pools");
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&src, &dst, &k_out, &v_out})
    TORCH_CHECK(t->device() == k_pool.device(), "paged_kv_dequantize: tensors on different devices");
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&k_out, &v_out})
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0, "paged_kv_dequantize: outputs must be 16B aligned");
  c10::cuda::CUDAGuard guard(k_pool.device());
  TORCH_CHECK(pg_paged_kv_dequantize(k_pool.data_ptr(), v_pool.data_ptr(), k_scales.data_ptr<float>(),
                                     v_scales.data_ptr<float>(), src.data_ptr<int>(), dst.data_ptr<int>(),
                                     k_out.data_ptr(), v_out.data_ptr(), (int)src.numel(), (int)k_pool.size(1),
                                     (int)k_pool.size(3), cur_stream()) == 0, "paged_kv_dequantize failed");
}

// KV pools as paged_kv_copy and paged_kv_swap take them: contiguous [n_layer, pages, H, 64, D] bf16, or FP8 codes with
// fp32 scales [n_layer, pages, H, 64], on one device and 16-byte aligned.  Returns whether they are FP8 and sets the
// bytes of one pool row.
static bool check_kv_pools(const char* op, const torch::Tensor& k_pools, const torch::Tensor& v_pools,
                           const c10::optional<torch::Tensor>& k_scales, const c10::optional<torch::Tensor>& v_scales,
                           int64_t* row_bytes) {
  PG_CUDA(k_pools); PG_CUDA(v_pools);
  TORCH_CHECK(k_pools.dim() == 5 && v_pools.sizes() == k_pools.sizes() && k_pools.size(3) == 64 &&
              k_pools.scalar_type() == v_pools.scalar_type() && k_pools.is_contiguous() && v_pools.is_contiguous(),
              op, ": k_pools / v_pools must be contiguous [n_layer, pages, H, 64, D] of one dtype");
  const bool fp8 = k_pools.scalar_type() == torch::kFloat8_e4m3fn;
  TORCH_CHECK(fp8 || k_pools.scalar_type() == torch::kBFloat16, op, ": pools must be bf16 or float8_e4m3fn");
  TORCH_CHECK(fp8 == k_scales.has_value() && fp8 == v_scales.has_value(),
              op, ": float8_e4m3fn pools need k_scales and v_scales, and bf16 pools take none");
  if (fp8) {
    for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&*k_scales, &*v_scales}) {
      PG_CUDA((*t)); PG_F32((*t));
      TORCH_CHECK(t->sizes() == k_pools.sizes().slice(0, 4) && t->is_contiguous() && t->device() == k_pools.device(),
                  op, ": scales must be contiguous fp32 [n_layer, pages, H, 64] like the pools");
      TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0, op, ": scales must be 16B aligned");
    }
  }
  *row_bytes = k_pools.size(4) * k_pools.element_size();
  TORCH_CHECK(*row_bytes % 16 == 0, op, ": a pool row of ", *row_bytes, " bytes is not a whole number of 16-byte words");
  TORCH_CHECK(v_pools.device() == k_pools.device(), op, ": tensors on different devices");
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&k_pools, &v_pools})
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0, op, ": pools must be 16B aligned");
  return fp8;
}

// Beam-search forks: slots 0 .. count - 1 of page src into page dst, for every pair (int32 [n, 3]: src, dst, count)
// and every layer of the pools [n_layer, pages, H, 64, D] (bf16, or FP8 codes with fp32 scales [n_layer, pages, H,
// 64]).  The caller guarantees that every id is a page of the pools and that no dst is also a src.
void paged_kv_copy(const torch::Tensor& pairs, torch::Tensor k_pools, torch::Tensor v_pools,
                   const c10::optional<torch::Tensor>& k_scales, const c10::optional<torch::Tensor>& v_scales) {
  PG_CUDA(pairs);
  TORCH_CHECK(pairs.scalar_type() == torch::kInt32 && pairs.dim() == 2 && pairs.size(1) == 3 && pairs.is_contiguous(),
              "paged_kv_copy: pairs must be contiguous int32 [n, 3] (src, dst, count)");
  int64_t row_bytes;
  const bool fp8 = check_kv_pools("paged_kv_copy", k_pools, v_pools, k_scales, v_scales, &row_bytes);
  TORCH_CHECK(pairs.device() == k_pools.device(), "paged_kv_copy: tensors on different devices");
  c10::cuda::CUDAGuard guard(k_pools.device());
  TORCH_CHECK(pg_paged_kv_copy(pairs.data_ptr<int>(), k_pools.data_ptr(), v_pools.data_ptr(),
                               fp8 ? k_scales->data_ptr<float>() : nullptr, fp8 ? v_scales->data_ptr<float>() : nullptr,
                               (int)pairs.size(0), (int)k_pools.size(0), (int)k_pools.size(1), (int)k_pools.size(2),
                               (int)row_bytes, cur_stream()) == 0, "paged_kv_copy failed");
}

// The device pointer of a pinned host tensor (refused if it is not pinned host memory).
static void* pinned_device_ptr(const torch::Tensor& t, const char* what) {
  cudaPointerAttributes attr;
  const cudaError_t e = cudaPointerGetAttributes(&attr, t.data_ptr());
  if (e != cudaSuccess) (void)cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess && attr.type == cudaMemoryTypeHost,
              "paged_kv_swap: ", what, " must be in pinned host memory (Tensor.pin_memory())");
  void* dev = nullptr;
  const cudaError_t g = cudaHostGetDevicePointer(&dev, t.data_ptr(), 0);
  if (g != cudaSuccess) (void)cudaGetLastError();
  TORCH_CHECK(g == cudaSuccess && dev != nullptr, "paged_kv_swap: ", what, " has no device mapping: ",
              cudaGetErrorString(g));
  return dev;
}

// Preemption: K and V (and their scales over FP8 pools) of pool page `page` of every layer to or from host slot `slot`,
// for every pair (int32 [n, 2]: page, slot).  host_kv is pinned [slots, n_layer, 2, H, 64, D] in the pools' dtype,
// host_scales pinned fp32 [slots, n_layer, 2, H, 64] (FP8 pools only).  The caller guarantees that every id is in range.
void paged_kv_swap(const torch::Tensor& pairs, torch::Tensor k_pools, torch::Tensor v_pools,
                   const c10::optional<torch::Tensor>& k_scales, const c10::optional<torch::Tensor>& v_scales,
                   torch::Tensor host_kv, const c10::optional<torch::Tensor>& host_scales, bool to_host) {
  PG_CUDA(pairs);
  TORCH_CHECK(pairs.scalar_type() == torch::kInt32 && pairs.dim() == 2 && pairs.size(1) == 2 && pairs.is_contiguous(),
              "paged_kv_swap: pairs must be contiguous int32 [n, 2] (page, slot)");
  int64_t row_bytes;
  const bool fp8 = check_kv_pools("paged_kv_swap", k_pools, v_pools, k_scales, v_scales, &row_bytes);
  TORCH_CHECK(pairs.device() == k_pools.device(), "paged_kv_swap: tensors on different devices");
  const auto L = k_pools.size(0), H = k_pools.size(2), D = k_pools.size(4);
  TORCH_CHECK(!host_kv.is_cuda() && host_kv.is_contiguous() && host_kv.scalar_type() == k_pools.scalar_type() &&
              host_kv.dim() == 6 && host_kv.size(1) == L && host_kv.size(2) == 2 && host_kv.size(3) == H &&
              host_kv.size(4) == 64 && host_kv.size(5) == D,
              "paged_kv_swap: host_kv must be a contiguous host tensor [slots, n_layer, 2, H, 64, D] of the pools' dtype");
  TORCH_CHECK(fp8 == host_scales.has_value(),
              "paged_kv_swap: float8_e4m3fn pools need host_scales, and bf16 pools take none");
  if (fp8)
    TORCH_CHECK(!host_scales->is_cuda() && host_scales->is_contiguous() &&
                host_scales->scalar_type() == torch::kFloat32 && host_scales->sizes() == host_kv.sizes().slice(0, 5),
                "paged_kv_swap: host_scales must be a contiguous fp32 host tensor [slots, n_layer, 2, H, 64]");
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&host_kv, fp8 ? &*host_scales : &host_kv})
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0, "paged_kv_swap: host tensors must be 16B aligned");
  void* host = pinned_device_ptr(host_kv, "host_kv");
  float* scales = fp8 ? static_cast<float*>(pinned_device_ptr(*host_scales, "host_scales")) : nullptr;
  c10::cuda::CUDAGuard guard(k_pools.device());
  TORCH_CHECK(pg_paged_kv_swap(pairs.data_ptr<int>(), k_pools.data_ptr(), v_pools.data_ptr(),
                               fp8 ? k_scales->data_ptr<float>() : nullptr, fp8 ? v_scales->data_ptr<float>() : nullptr,
                               host, scales, (int)pairs.size(0), (int)L, (int)k_pools.size(1), (int)H, (int)row_bytes,
                               to_host ? 1 : 0, cur_stream()) == 0, "paged_kv_swap failed");
}

// Beam search's candidate choice (csrc/beam_sm90.cu): per request r (rows cu[r] .. cu[r+1] - 1 of logits [N, V], bf16
// or fp32, unit inner stride) the k best (score, token, row), written to out_score / out_token / out_row [R, k], and
// each row's logsumexp into lse [N] when given.  max_rows is the host's bound on one request's rows.
void beam_topk(const torch::Tensor& logits, const torch::Tensor& scores, const torch::Tensor& cu, int64_t k,
               int64_t max_rows, torch::Tensor out_score, torch::Tensor out_token, torch::Tensor out_row,
               const c10::optional<torch::Tensor>& lse, torch::Tensor ticket) {
  TORCH_CHECK(logits.is_cuda(), "beam_topk: logits must be a CUDA tensor");
  PG_CUDA(scores); PG_F32(scores); PG_CUDA(cu); PG_CUDA(out_score); PG_F32(out_score);
  PG_CUDA(out_token); PG_CUDA(out_row); PG_CUDA(ticket);
  const bool fp32 = logits.scalar_type() == torch::kFloat32;
  TORCH_CHECK(fp32 || logits.scalar_type() == torch::kBFloat16, "beam_topk: logits must be bf16 or fp32");
  TORCH_CHECK(logits.dim() == 2 && logits.stride(1) == 1 && logits.size(0) >= 1,
              "beam_topk: logits must be [N, V] with unit inner stride");
  const int64_t N = logits.size(0), V = logits.size(1), R = cu.numel() - 1;
  TORCH_CHECK(cu.scalar_type() == torch::kInt32 && R >= 1 && cu.is_contiguous(), "beam_topk: cu must be int32 [R + 1]");
  TORCH_CHECK(out_token.scalar_type() == torch::kInt32 && out_row.scalar_type() == torch::kInt32 &&
              ticket.scalar_type() == torch::kInt32, "beam_topk: out_token, out_row and ticket must be int32");
  TORCH_CHECK(scores.numel() == N && scores.is_contiguous(), "beam_topk: scores must be fp32 [N]");
  TORCH_CHECK(1 <= k && k <= 16 && k <= V, "beam_topk: k must be in 1 .. min(16, V), got ", k);
  TORCH_CHECK(1 <= max_rows && max_rows <= 64, "beam_topk: a request holds 1 .. 64 rows, got ", max_rows);
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&out_score, &out_token, &out_row})
    TORCH_CHECK(t->numel() == R * k && t->is_contiguous(), "beam_topk: outputs must be contiguous [R, k]");
  TORCH_CHECK(ticket.numel() >= R, "beam_topk: ticket must hold at least R = ", R, " entries");
  if (lse.has_value()) {
    PG_CUDA((*lse)); PG_F32((*lse));
    TORCH_CHECK(lse->numel() == N && lse->is_contiguous(), "beam_topk: lse must be fp32 [N]");
  }
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&scores, &cu, &out_score, &out_token, &out_row, &ticket})
    TORCH_CHECK(t->device() == logits.device(), "beam_topk: tensors on different devices");
  c10::cuda::CUDAGuard guard(logits.device());
  const int splits = pg_beam_topk_splits((int)N, (int)V, (int)k, (int)max_rows);
  torch::Tensor part = torch::empty({N * splits * (2 + 2 * pg_beam_topk_kp((int)k))}, scores.options());
  TORCH_CHECK(pg_beam_topk(logits.data_ptr(), fp32 ? 1 : 0, logits.stride(0), scores.data_ptr<float>(), cu.data_ptr<int>(),
                           part.data_ptr<float>(), ticket.data_ptr<int>(), out_score.data_ptr<float>(),
                           out_token.data_ptr<int>(), out_row.data_ptr<int>(),
                           lse.has_value() ? lse->data_ptr<float>() : nullptr, (int)N, (int)V, (int)R, (int)k,
                           (int)max_rows, splits, cur_stream()) == 0, "beam_topk failed");
}

void moe_route(const torch::Tensor& x, const torch::Tensor& wg, const c10::optional<torch::Tensor>& bg,
               const c10::optional<torch::Tensor>& jitter, int64_t top_k, int64_t capacity, torch::Tensor probs,
               torch::Tensor topk_idx, torch::Tensor topk_prob, torch::Tensor pos, torch::Tensor counts,
               torch::Tensor prob_sum, torch::Tensor zsum, torch::Tensor lse) {
  PG_CUDA(x); PG_BF16(x); PG_CUDA(wg); PG_BF16(wg); PG_CUDA(probs); PG_F32(probs);
  c10::cuda::CUDAGuard guard(x.device());
  const int n = (int)x.size(0), h = (int)x.size(1), E = (int)wg.size(0);
  const float* jp = jitter.has_value() ? jitter->data_ptr<float>() : nullptr;
  TORCH_CHECK(pg_moe_route(x.data_ptr(), wg.data_ptr(), opt_ptr(bg), jp, n, h, E, (int)top_k, (int)capacity,
                           probs.data_ptr<float>(), topk_idx.data_ptr<int>(), topk_prob.data_ptr<float>(), pos.data_ptr<int>(),
                           counts.data_ptr<int>(), prob_sum.data_ptr<float>(), zsum.data_ptr<float>(), lse.data_ptr<float>(), cur_stream()) == 0, "moe_route failed");
}

void moe_dispatch(const torch::Tensor& x, const torch::Tensor& topk_idx, const torch::Tensor& topk_prob, const torch::Tensor& pos,
                  std::vector<int64_t> peer_buf, std::vector<int64_t> peer_row_ret, std::vector<int64_t> peer_row_scale,
                  std::vector<int64_t> peer_arrive, int64_t top_k, int64_t E_local, int64_t C, int64_t my_rank, bool scale_by_prob, int64_t blocks) {
  PG_CUDA(x); PG_BF16(x);
  c10::cuda::CUDAGuard guard(x.device());
  const int T = (int)peer_buf.size();
  TORCH_CHECK(T >= 1 && T <= PG_MAX_PEERS, "moe_dispatch: 1..", PG_MAX_PEERS, " peer buffers, got ", T);
  TORCH_CHECK(peer_row_ret.size() == peer_buf.size() && peer_row_scale.size() == peer_buf.size() &&
                  peer_arrive.size() == peer_buf.size(), "moe_dispatch: the four peer lists must have the same length");
  void* bufs[PG_MAX_PEERS]; int* rets[PG_MAX_PEERS]; float* scs[PG_MAX_PEERS]; uint32_t* arr[PG_MAX_PEERS];
  for (int i = 0; i < T; ++i) { bufs[i] = reinterpret_cast<void*>(peer_buf[i]); rets[i] = reinterpret_cast<int*>(peer_row_ret[i]);
    scs[i] = reinterpret_cast<float*>(peer_row_scale[i]); arr[i] = reinterpret_cast<uint32_t*>(peer_arrive[i]); }
  TORCH_CHECK(pg_moe_dispatch(x.data_ptr(), topk_idx.data_ptr<int>(), topk_prob.data_ptr<float>(), pos.data_ptr<int>(), bufs, rets, scs, arr,
                              (int)x.size(0), (int)x.size(1), (int)top_k, (int)E_local, T, (int)C, (int)my_rank, scale_by_prob, (int)blocks, cur_stream()) == 0, "moe_dispatch failed");
}

// ---------------------------------------------------------------- symmetric memory / collectives
py::tuple symm_alloc(int64_t nbytes) {
  void* ptr = nullptr;
  char handle[64];
  TORCH_CHECK(pg_symm_alloc(nbytes, &ptr, handle) == 0, "symm_alloc failed");
  return py::make_tuple(reinterpret_cast<int64_t>(ptr), py::bytes(handle, 64));
}
int64_t symm_open(const std::string& handle) {
  TORCH_CHECK(handle.size() == 64, "bad ipc handle");
  void* ptr = nullptr;
  TORCH_CHECK(pg_symm_open(handle.data(), &ptr) == 0, "symm_open failed");
  return reinterpret_cast<int64_t>(ptr);
}
void symm_close(int64_t ptr) { pg_symm_close(reinterpret_cast<void*>(ptr)); }
void symm_free(int64_t ptr) { pg_symm_free(reinterpret_cast<void*>(ptr)); }

torch::Tensor tensor_from_ptr(int64_t ptr, int64_t nbytes, int64_t device_index) {
  auto opts = torch::TensorOptions().dtype(torch::kUInt8).device(torch::kCUDA, (int)device_index);
  return torch::from_blob(reinterpret_cast<void*>(ptr), {nbytes}, [](void*) {}, opts);
}

void rs_reduce(int64_t staging_ptr, int64_t num_src, int64_t src_stride, int64_t ctr_ptr, int64_t expected,
               const c10::optional<torch::Tensor>& bias, const c10::optional<torch::Tensor>& residual, torch::Tensor out) {
  PG_CUDA(out); PG_BF16(out);
  c10::cuda::CUDAGuard guard(out.device());
  TORCH_CHECK(pg_rs_reduce(reinterpret_cast<const void*>(staging_ptr), (int)num_src, src_stride,
                           reinterpret_cast<const uint32_t*>(ctr_ptr), (uint32_t)expected, opt_ptr(bias), opt_ptr(residual),
                           out.data_ptr(), (int)out.size(0), (int)out.size(1), cur_stream()) == 0, "rs_reduce failed");
}

void allreduce_f32(std::vector<int64_t> peer_bufs, int64_t rank, int64_t offset, int64_t n, double scale, bool rs_only,
                   std::vector<int64_t> peer_flags, int64_t epoch, int64_t blocks, int64_t mc_buf, int64_t bucket_elems) {
  float* bufs[PG_MAX_PEERS]; uint32_t* flags[PG_MAX_PEERS];
  const int world = (int)peer_bufs.size();
  TORCH_CHECK(world <= PG_MAX_PEERS && peer_flags.size() == peer_bufs.size(), "bad peer lists");
  for (int i = 0; i < world; ++i) { bufs[i] = reinterpret_cast<float*>(peer_bufs[i]); flags[i] = reinterpret_cast<uint32_t*>(peer_flags[i]); }
  TORCH_CHECK(pg_allreduce_f32(bufs, reinterpret_cast<float*>(mc_buf), world, (int)rank, offset, n, bucket_elems, (float)scale, rs_only, flags,
                               (uint32_t)epoch, (int)blocks, cur_stream()) == 0, "allreduce_f32 failed");
}

void allgather_bf16(std::vector<int64_t> peer_bufs, int64_t rank, int64_t bucket_elems, int64_t total_elems,
                    std::vector<int64_t> peer_flags, int64_t epoch, int64_t head_elems, int64_t mc_buf) {
  void* bufs[PG_MAX_PEERS]; uint32_t* flags[PG_MAX_PEERS];
  const int world = (int)peer_bufs.size();
  TORCH_CHECK(world <= PG_MAX_PEERS && peer_flags.size() == peer_bufs.size(), "bad peer lists");
  for (int i = 0; i < world; ++i) { bufs[i] = reinterpret_cast<void*>(peer_bufs[i]); flags[i] = reinterpret_cast<uint32_t*>(peer_flags[i]); }
  TORCH_CHECK(pg_allgather_bf16(bufs, reinterpret_cast<void*>(mc_buf), world, (int)rank, head_elems, bucket_elems, total_elems, flags,
                                (uint32_t)epoch, cur_stream()) == 0, "allgather_bf16 failed");
}

void rs_push(const torch::Tensor& x, int64_t num_chunks, int64_t first_chunk, std::vector<int64_t> out_peer,
             std::vector<int64_t> arrive_ctr, int64_t blocks) {
  PG_CUDA(x); PG_BF16(x);
  c10::cuda::CUDAGuard guard(x.device());
  TORCH_CHECK((int64_t)out_peer.size() == num_chunks && (int64_t)arrive_ctr.size() == num_chunks && x.numel() % num_chunks == 0, "rs_push: bad lists");
  void* outs[PG_MAX_PEERS]; uint32_t* ctrs[PG_MAX_PEERS];
  for (int i = 0; i < num_chunks; ++i) { outs[i] = reinterpret_cast<void*>(out_peer[i]); ctrs[i] = reinterpret_cast<uint32_t*>(arrive_ctr[i]); }
  TORCH_CHECK(pg_rs_push(x.data_ptr(), (int)num_chunks, (int)first_chunk, x.numel() / num_chunks, outs, ctrs, (int)blocks, cur_stream()) == 0, "rs_push failed");
}

void multimem_selftest(int64_t mc_in, int64_t mc_out, torch::Tensor out) {
  PG_CUDA(out); PG_F32(out);
  c10::cuda::CUDAGuard guard(out.device());
  TORCH_CHECK(pg_multimem_selftest(reinterpret_cast<const float*>(mc_in), reinterpret_cast<float*>(mc_out), out.data_ptr<float>(),
                                   out.numel(), cur_stream()) == 0, "multimem_selftest failed");
}

void rs_reduce_mc(int64_t mc_partial, int64_t ctr_ptr, int64_t num_src, int64_t expected, const c10::optional<torch::Tensor>& bias,
                  const c10::optional<torch::Tensor>& residual, torch::Tensor out) {
  PG_CUDA(out); PG_BF16(out);
  c10::cuda::CUDAGuard guard(out.device());
  TORCH_CHECK(pg_rs_reduce_mc(reinterpret_cast<const void*>(mc_partial), reinterpret_cast<const uint32_t*>(ctr_ptr), (int)num_src,
                              (uint32_t)expected, opt_ptr(bias), opt_ptr(residual), out.data_ptr(), (int)out.size(0), (int)out.size(1),
                              cur_stream()) == 0, "rs_reduce_mc failed");
}

// ---- VMM + multicast symmetric memory (symm_vmm.cu)
py::tuple vmm_probe(int64_t world) {
  int mc = 0; int64_t gran = 0;
  const int rc = pg_vmm_probe((int)world, &mc, &gran);
  return py::make_tuple(rc == 0, mc != 0, gran);
}
py::tuple vmm_alloc(int64_t nbytes) {
  void* ptr = nullptr; int fd = -1; uint64_t h = 0;
  TORCH_CHECK(pg_vmm_alloc(nbytes, &ptr, &fd, &h) == 0, "vmm_alloc failed");
  return py::make_tuple(reinterpret_cast<int64_t>(ptr), fd, (int64_t)h);
}
py::tuple vmm_import(int64_t fd, int64_t nbytes) {
  void* ptr = nullptr; uint64_t h = 0;
  TORCH_CHECK(pg_vmm_import((int)fd, nbytes, &ptr, &h) == 0, "vmm_import failed");
  return py::make_tuple(reinterpret_cast<int64_t>(ptr), (int64_t)h);
}
void vmm_unmap(int64_t ptr, int64_t nbytes, int64_t handle) { pg_vmm_unmap(reinterpret_cast<void*>(ptr), nbytes, (uint64_t)handle); }
py::tuple mc_create(int64_t world, int64_t nbytes) {
  int fd = -1; uint64_t h = 0;
  TORCH_CHECK(pg_mc_create((int)world, nbytes, &fd, &h) == 0, "mc_create failed");
  return py::make_tuple(fd, (int64_t)h);
}
int64_t mc_import(int64_t fd) {
  uint64_t h = 0;
  TORCH_CHECK(pg_mc_import((int)fd, &h) == 0, "mc_import failed");
  return (int64_t)h;
}
void mc_add_device(int64_t mc) { TORCH_CHECK(pg_mc_add_device((uint64_t)mc) == 0, "mc_add_device failed"); }
int64_t mc_bind(int64_t mc, int64_t mem, int64_t nbytes) {
  void* p = nullptr;
  TORCH_CHECK(pg_mc_bind((uint64_t)mc, (uint64_t)mem, nbytes, &p) == 0, "mc_bind failed");
  return reinterpret_cast<int64_t>(p);
}

void barrier_peers(std::vector<int64_t> peer_flags, int64_t rank, int64_t epoch) {
  uint32_t* flags[PG_MAX_PEERS];
  const int world = (int)peer_flags.size();
  for (int i = 0; i < world; ++i) flags[i] = reinterpret_cast<uint32_t*>(peer_flags[i]);
  TORCH_CHECK(pg_barrier_peers(flags, world, (int)rank, (uint32_t)epoch, cur_stream()) == 0, "barrier_peers failed");
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("gemm", &gemm, "wgmma bf16 GEMM with fused epilogue / chunked collectives",
        py::arg("a"), py::arg("b"), py::arg("out"), py::arg("a_mn") = false, py::arg("b_mn") = false,
        py::arg("bias") = py::none(), py::arg("residual") = py::none(), py::arg("aux") = py::none(),
        py::arg("flags") = 0, py::arg("block_n") = 0, py::arg("max_ctas") = 0,
        py::arg("num_chunks") = 1, py::arg("first_chunk") = 0, py::arg("chunk_flags_ptr") = 0,
        py::arg("flag_value") = 0, py::arg("out_peer_ptrs") = std::vector<int64_t>{},
        py::arg("arrive_ctr_ptrs") = std::vector<int64_t>{}, py::arg("ag") = py::dict(),
        py::arg("bias_grad") = py::none());
  m.def("gemm_fp8", &gemm_fp8, "wgmma FP8 GEMM (K-major e4m3 / e5m2 x e4m3 codes, per-tensor scales)", py::arg("a"),
        py::arg("b"), py::arg("a_scale_inv"), py::arg("b_scale_inv"), py::arg("out"), py::arg("bias") = py::none(),
        py::arg("residual") = py::none(), py::arg("aux") = py::none(), py::arg("gelu") = false, py::arg("dgelu") = false,
        py::arg("accumulate") = false, py::arg("block_n") = 0, py::arg("k_splits") = 0);
  m.def("fp8_quantize", &fp8_quantize, py::arg("x"), py::arg("e5m2"), py::arg("amax"), py::arg("codes") = py::none(),
        py::arg("codes_t") = py::none(), py::arg("scale_inv") = py::none(), py::arg("colsum") = py::none());
  m.def("layernorm_fwd", &layernorm_fwd);
  m.def("layernorm_bwd", &layernorm_bwd);
  m.def("colsum", &colsum);
  m.def("embedding_bwd", &embedding_bwd, py::arg("dx"), py::arg("ids"), py::arg("dw"), py::arg("vocab_start"), py::arg("vocab_end"),
        py::arg("grad_rs") = py::dict());
  m.def("grad_rs_accum", &grad_rs_accum);
  m.def("ce_stats", &ce_stats);
  m.def("ce_combine", &ce_combine);
  m.def("ce_finalize", &ce_finalize);
  m.def("adam_step", &adam_step, py::arg("master"), py::arg("m"), py::arg("v"), py::arg("grad"), py::arg("param_bf16"), py::arg("lr"),
        py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("wd"), py::arg("step"), py::arg("grad_scale"), py::arg("adamw"),
        py::arg("zero_grad") = false);
  m.def("adam_step_strided", &adam_step_strided);
  m.def("accum_bf16_to_f32", &accum_bf16_to_f32);
  m.def("attention_fwd", &attention_fwd, py::arg("qkv"), py::arg("slopes"), py::arg("out"), py::arg("lse"), py::arg("B"),
        py::arg("S"), py::arg("H"), py::arg("D"), py::arg("softmax_scale") = 0.0, py::arg("seg_start") = py::none());
  m.def("attention_bwd", &attention_bwd, py::arg("qkv"), py::arg("slopes"), py::arg("out"), py::arg("lse"), py::arg("dout"),
        py::arg("dqkv"), py::arg("B"), py::arg("S"), py::arg("H"), py::arg("D"), py::arg("softmax_scale") = 0.0,
        py::arg("seg_start") = py::none());
  m.def("decode_attention", &decode_attention, py::arg("qkv"), py::arg("k_cache"), py::arg("v_cache"), py::arg("slopes"),
        py::arg("pos"), py::arg("lead"), py::arg("out"), py::arg("ticket"), py::arg("softmax_scale") = 0.0);
  m.def("paged_decode_attention", &paged_decode_attention, py::arg("qkv"), py::arg("k_pool"), py::arg("v_pool"),
        py::arg("table"), py::arg("pos"), py::arg("max_pos"), py::arg("slopes"), py::arg("out"), py::arg("ticket"),
        py::arg("softmax_scale") = 0.0);
  m.def("paged_append_attention", &paged_append_attention, py::arg("qkv"), py::arg("k_pool"), py::arg("v_pool"),
        py::arg("table"), py::arg("cu_seqlens"), py::arg("pos"), py::arg("max_pos"), py::arg("max_tokens"),
        py::arg("slopes"), py::arg("out"), py::arg("ticket"), py::arg("softmax_scale") = 0.0);
  m.def("paged_prefill_attention", &paged_prefill_attention, py::arg("qkv"), py::arg("k_pool"), py::arg("v_pool"),
        py::arg("table"), py::arg("cu_seqlens"), py::arg("start"), py::arg("max_len"), py::arg("slopes"), py::arg("out"),
        py::arg("softmax_scale"));
  m.def("paged_kv_write", &paged_kv_write, py::arg("qkv"), py::arg("slot"), py::arg("k_pool"), py::arg("v_pool"));
  m.def("paged_kv_write_fp8", &paged_kv_write_fp8, py::arg("qkv"), py::arg("slot"), py::arg("k_pool"),
        py::arg("v_pool"), py::arg("k_scales"), py::arg("v_scales"));
  m.def("paged_decode_attention_fp8", &paged_decode_attention_fp8, py::arg("qkv"), py::arg("k_pool"),
        py::arg("v_pool"), py::arg("k_scales"), py::arg("v_scales"), py::arg("table"), py::arg("pos"),
        py::arg("max_pos"), py::arg("slopes"), py::arg("out"), py::arg("ticket"), py::arg("softmax_scale") = 0.0);
  m.def("paged_kv_dequantize", &paged_kv_dequantize, py::arg("k_pool"), py::arg("v_pool"), py::arg("k_scales"),
        py::arg("v_scales"), py::arg("src"), py::arg("dst"), py::arg("k_out"), py::arg("v_out"));
  m.def("paged_kv_copy", &paged_kv_copy, py::arg("pairs"), py::arg("k_pools"), py::arg("v_pools"),
        py::arg("k_scales") = py::none(), py::arg("v_scales") = py::none());
  m.def("paged_kv_swap", &paged_kv_swap, py::arg("pairs"), py::arg("k_pools"), py::arg("v_pools"), py::arg("k_scales"),
        py::arg("v_scales"), py::arg("host_kv"), py::arg("host_scales"), py::arg("to_host"));
  m.def("beam_topk", &beam_topk, py::arg("logits"), py::arg("scores"), py::arg("cu"), py::arg("k"), py::arg("max_rows"),
        py::arg("out_score"), py::arg("out_token"), py::arg("out_row"), py::arg("lse"), py::arg("ticket"));
  m.def("moe_route", &moe_route);
  m.def("moe_dispatch", &moe_dispatch);
  m.def("symm_alloc", &symm_alloc);
  m.def("symm_open", &symm_open);
  m.def("symm_close", &symm_close);
  m.def("symm_free", &symm_free);
  m.def("tensor_from_ptr", &tensor_from_ptr);
  m.def("rs_reduce", &rs_reduce);
  m.def("allreduce_f32", &allreduce_f32, py::arg("peer_bufs"), py::arg("rank"), py::arg("offset"), py::arg("n"),
        py::arg("scale"), py::arg("rs_only"), py::arg("peer_flags"), py::arg("epoch"), py::arg("blocks") = 0, py::arg("mc_buf") = 0, py::arg("bucket_elems") = 0);
  m.def("set_gemm_cta_cap", [](int64_t n) { pg_set_gemm_cta_cap((int)n); });
  m.def("allgather_bf16", &allgather_bf16, py::arg("peer_bufs"), py::arg("rank"), py::arg("bucket_elems"), py::arg("total_elems"),
        py::arg("peer_flags"), py::arg("epoch"), py::arg("head_elems") = 0, py::arg("mc_buf") = 0);
  m.def("rs_push", &rs_push);
  m.def("multimem_selftest", &multimem_selftest);
  m.def("rs_reduce_mc", &rs_reduce_mc);
  m.def("vmm_probe", &vmm_probe);
  m.def("vmm_alloc", &vmm_alloc);
  m.def("vmm_import", &vmm_import);
  m.def("vmm_unmap", &vmm_unmap);
  m.def("mc_create", &mc_create);
  m.def("mc_import", &mc_import);
  m.def("mc_add_device", &mc_add_device);
  m.def("mc_bind", &mc_bind);
  m.def("barrier_peers", &barrier_peers);
}
