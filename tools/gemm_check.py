"""GPU dev harness: correctness of the wgmma GEMM in every layout/epilogue + throughput vs cuBLAS.
Writes the results as JSON to --out (default: gemm_check.json in the current directory).

    python tools/gemm_check.py [all|epi] [--so path/to/_C.so] [--out results.json]

--so times another build of the extension (e.g. an older commit's) with the same harness."""
import json, os, sys, time, importlib.util
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
argv = sys.argv[1:]
def _opt(name, default):
    if name in argv:
        i = argv.index(name); v = argv[i + 1]; del argv[i:i + 2]; return v
    return default
SO = _opt("--so", os.path.join(ROOT, "pipegoose_b200", "_C.so"))
OUT = _opt("--out", "gemm_check.json")
spec = importlib.util.spec_from_file_location("_C", SO)
_C = importlib.util.module_from_spec(spec); spec.loader.exec_module(_C)

dev = "cuda"
torch.manual_seed(0)
results = {"correctness": [], "perf": []}

def gelu(x):
    return x * 0.5 * (1.0 + torch.tanh(0.79788456 * x * (1 + 0.044715 * x * x)))

def run_case(M, N, K, a_mn, b_mn, bn, epi):
    A = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
    B = torch.randn(N, K, device=dev, dtype=torch.bfloat16)
    ref = A.float() @ B.float().t()
    a_st = A.t().contiguous() if a_mn else A
    b_st = B.t().contiguous() if b_mn else B
    bias = res = aux = None
    flags = 0
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    if epi == "bias":
        bias = torch.randn(N, device=dev, dtype=torch.bfloat16); ref = ref + bias.float()
    elif epi == "bias_gelu":
        bias = torch.randn(N, device=dev, dtype=torch.bfloat16); pre = ref + bias.float(); ref = gelu(pre)
        aux = torch.empty(M, N, device=dev, dtype=torch.bfloat16); flags = 2
    elif epi == "bias_res":
        bias = torch.randn(N, device=dev, dtype=torch.bfloat16); res = torch.randn(M, N, device=dev, dtype=torch.bfloat16)
        ref = ref + bias.float() + res.float()
    elif epi == "f32acc":
        out = torch.randn(M, N, device=dev, dtype=torch.float32); ref = ref + out; flags = 16
    elif epi == "f32over":
        out = torch.full((M, N), 7.0, device=dev, dtype=torch.float32)
    elif epi == "dgelu":
        aux = torch.randn(M, N, device=dev, dtype=torch.bfloat16); flags = 32
        z = aux.float().requires_grad_(True); g = torch.autograd.grad(gelu(z).sum(), z)[0]; ref = ref * g
    _C.gemm(a_st, b_st, out, a_mn, b_mn, bias, res, aux, flags, bn)
    torch.cuda.synchronize()
    err = (out.float() - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-6
    rel = err / scale
    ok = rel < 2e-2
    if epi == "bias_gelu":
        e2 = (aux.float() - pre).abs().max().item() / (pre.abs().max().item() + 1e-6)
        ok = ok and e2 < 2e-2
    results["correctness"].append(dict(M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, bn=bn, epi=epi, rel_err=rel, ok=bool(ok)))
    print(("OK  " if ok else "FAIL"), M, N, K, "a_mn", a_mn, "b_mn", b_mn, "bn", bn, epi, "rel", f"{rel:.2e}", flush=True)
    return ok

all_ok = True
stage = argv[0] if argv else "all"
# smallest first: one tile, one k-block
for (a_mn, b_mn) in [(False, False), (False, True), (True, True), (True, False)]:
    for bn in [128, 256, 64, 192]:
        all_ok &= run_case(128, bn, 64, a_mn, b_mn, bn, "none")
        all_ok &= run_case(256, 512, 256, a_mn, b_mn, bn, "none")
for (a_mn, b_mn) in [(False, False), (False, True), (True, True)]:
    all_ok &= run_case(4096, 1024, 1024, a_mn, b_mn, 0, "none")
    all_ok &= run_case(1000, 264, 200, a_mn, b_mn, 0, "none") if not a_mn else True
    all_ok &= run_case(1024, 328, 520, a_mn, b_mn, 0, "none")
for epi in ["bias", "bias_gelu", "bias_res", "f32acc", "dgelu"]:
    all_ok &= run_case(2048, 1024, 512, False, False, 0, epi)
    all_ok &= run_case(640, 328, 136, False, False, 128, epi)
all_ok &= run_case(1024, 4096, 8192, True, True, 0, "f32acc")
# small outputs with a long K: the host picks a split-K (atomic fp32 partial sums), overwrite and accumulate
for epi in ["f32acc", "f32over"]:
    all_ok &= run_case(1024, 1024, 8192, True, True, 0, epi)
    all_ok &= run_case(512, 768, 4096, True, True, 0, epi)
    all_ok &= run_case(256, 264, 2048, True, True, 0, epi)
results["all_ok"] = bool(all_ok)

def bench(fn, iters=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    ts = []
    for _ in range(iters):
        flush.zero_()
        s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record(); torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2], ts[0]

# fused-epilogue GEMMs at the flagship (bloom-560m, 8192 tokens) shapes
def epi_perf():
    M, h = 8192, 1024
    x = torch.randn(M, h, device=dev, dtype=torch.bfloat16)
    x4 = torch.randn(M, 4 * h, device=dev, dtype=torch.bfloat16)
    w1 = torch.randn(4 * h, h, device=dev, dtype=torch.bfloat16)
    w2 = torch.randn(h, 4 * h, device=dev, dtype=torch.bfloat16)
    wd = torch.randn(h, h, device=dev, dtype=torch.bfloat16)
    b4 = torch.randn(4 * h, device=dev, dtype=torch.bfloat16)
    b1 = torch.randn(h, device=dev, dtype=torch.bfloat16)
    o1 = torch.empty(M, h, device=dev, dtype=torch.bfloat16)
    o4 = torch.empty(M, 4 * h, device=dev, dtype=torch.bfloat16)
    z4 = torch.randn(M, 4 * h, device=dev, dtype=torch.bfloat16)
    g1 = torch.zeros(h, h, device=dev, dtype=torch.float32)
    g4 = torch.zeros(4 * h, h, device=dev, dtype=torch.float32)
    w3 = torch.randn(3 * h, h, device=dev, dtype=torch.bfloat16)
    b3 = torch.randn(3 * h, device=dev, dtype=torch.bfloat16)
    o3 = torch.empty(M, 3 * h, device=dev, dtype=torch.bfloat16)
    V = 250880  # bloom vocabulary: lm_head logits with the cross-entropy partials in the epilogue
    wv = torch.randn(V, h, device=dev, dtype=torch.bfloat16) * 0.05
    ov = torch.empty(M, V, device=dev, dtype=torch.bfloat16)
    ce_part = torch.empty(M, 2 * ((V + 255) // 256), 2, device=dev, dtype=torch.float32)
    ce_ag = {"ce_part": ce_part.data_ptr(), "ce_valid": V}
    # wgrad operands: dy of qkv [M, 3h]; fp32 main grads of fc2 [h, 4h], qkv [3h, h] and the lm_head table [V, h]
    x3 = torch.randn(M, 3 * h, device=dev, dtype=torch.bfloat16)
    g14 = torch.zeros(h, 4 * h, device=dev, dtype=torch.float32)
    g3 = torch.zeros(3 * h, h, device=dev, dtype=torch.float32)
    gv = torch.zeros(V, h, device=dev, dtype=torch.float32)
    cases = {
        "fc1_bias_gelu_aux": (lambda: _C.gemm(x, w1, o4, False, False, b4, None, z4, 2), 2.0 * M * h * 4 * h),
        "fc1_bias_only": (lambda: _C.gemm(x, w1, o4, False, False, b4, None, None, 0), 2.0 * M * h * 4 * h),
        "fc2_bias_residual": (lambda: _C.gemm(x4, w2, o1, False, False, b1, x, None, 0), 2.0 * M * h * 4 * h),
        "dense_bias_residual": (lambda: _C.gemm(x, wd, o1, False, False, b1, x, None, 0), 2.0 * M * h * h),
        "fc2_dgrad_dgelu": (lambda: _C.gemm(x, w2, o4, False, True, None, None, z4, 32), 2.0 * M * h * 4 * h),
        "fc1_dgrad": (lambda: _C.gemm(x4, w1, o1, False, True), 2.0 * M * h * 4 * h),
        "dense_dgrad": (lambda: _C.gemm(x, wd, o1, False, True), 2.0 * M * h * h),
        "qkv_bias": (lambda: _C.gemm(x, w3, o3, False, False, b3, None, None, 0), 2.0 * M * h * 3 * h),
        "lm_head_ce": (lambda: _C.gemm(x, wv, ov, False, False, None, None, None, 0, ag=ce_ag), 2.0 * M * h * V),
        "dense_wgrad_f32acc": (lambda: _C.gemm(x, x, g1, True, True, None, None, None, 16), 2.0 * M * h * h),
        "dense_wgrad_f32over": (lambda: _C.gemm(x, x, g1, True, True, None, None, None, 0), 2.0 * M * h * h),
        "fc1_wgrad_f32acc": (lambda: _C.gemm(x4, x, g4, True, True, None, None, None, 16), 2.0 * M * h * 4 * h),
        "fc2_wgrad_f32acc": (lambda: _C.gemm(x, x4, g14, True, True, None, None, None, 16), 2.0 * M * h * 4 * h),
        "qkv_wgrad_f32acc": (lambda: _C.gemm(x3, x, g3, True, True, None, None, None, 16), 2.0 * M * h * 3 * h),
        "lm_head_wgrad_f32over": (lambda: _C.gemm(ov, x, gv, True, True, None, None, None, 0), 2.0 * M * h * V),
    }
    # "+ bias sum": the wgrad that also produces the bias gradient (dy's column sums); a build without the fused form
    # (no bias_grad argument) runs the wgrad and then the column-sum kernel, as its training step does
    bg = torch.zeros(V, device=dev, dtype=torch.float32)
    try:
        _C.gemm(x, x, g1, True, True, None, None, None, 16, bias_grad=bg[:h])
        fused = True
    except TypeError:
        fused = False

    def with_bias(dy, xx, g, flags):
        if fused:
            return lambda: _C.gemm(dy, xx, g, True, True, None, None, None, flags, bias_grad=bg[:dy.shape[1]])
        return lambda: (_C.gemm(dy, xx, g, True, True, None, None, None, flags), _C.colsum(dy, bg[:dy.shape[1]]))

    for name, (dy, xx, g, flags, fl) in {"dense_wgrad_f32acc": (x, x, g1, 16, 2.0 * M * h * h),
                                         "fc1_wgrad_f32acc": (x4, x, g4, 16, 2.0 * M * h * 4 * h),
                                         "fc2_wgrad_f32acc": (x, x4, g14, 16, 2.0 * M * h * 4 * h),
                                         "qkv_wgrad_f32acc": (x3, x, g3, 16, 2.0 * M * h * 3 * h),
                                         "lm_head_wgrad_f32over": (ov, x, gv, 0, 2.0 * M * h * V)}.items():
        cases[name + "_bias"] = (with_bias(dy, xx, g, flags), fl)
    out = {}
    for name, (fn, fl) in cases.items():
        row = {}
        med, best = bench(fn)
        row["auto"] = dict(ms=med, tflops=fl / med / 1e9)
        out[name] = row
        print(name, "  ".join(f"{t}: {v['ms']*1e3:.1f} us {v['tflops']:.0f} TF" for t, v in row.items()), flush=True)
    del wv, ov, ce_part, gv
    return out

# Plain NT GEMM at M = 8192, N = 4096, BN = 256 over K: time per tile round = fixed + per_kb * (K / 64).  The fit
# separates the steady-state cost of a 64-deep k-block from the per-tile cost outside the main loop (prologue,
# epilogue, pipeline fill).
def k_sweep():
    M, N, bn = 8192, 4096, 256
    rounds = -(-((M // 128) * (N // bn)) // torch.cuda.get_device_properties(0).multi_processor_count)
    rows = []
    for K in (512, 1024, 2048, 4096):
        A = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
        B = torch.randn(N, K, device=dev, dtype=torch.bfloat16)
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        med, _ = bench(lambda: _C.gemm(A, B, out, False, False, None, None, None, 0, bn))
        rows.append(dict(K=K, ms=med, us_per_round=med * 1e3 / rounds))
    kb = np.array([r["K"] / 64 for r in rows]); t = np.array([r["us_per_round"] for r in rows])
    per_kb, fixed = np.polyfit(kb, t, 1)
    res = dict(M=M, N=N, bn=bn, rounds=rounds, rows=rows, per_kblock_us=float(per_kb), fixed_per_tile_us=float(fixed))
    print("k_sweep", json.dumps(res), flush=True)
    return res

results["epi_perf"] = epi_perf()
results["k_sweep"] = k_sweep()
if stage == "epi":
    os.makedirs(os.path.dirname(os.path.abspath(OUT)), exist_ok=True)
    json.dump(results, open(OUT, "w"), indent=1)
    print("ALL_OK", all_ok)
    sys.exit(0)

shapes = [(8192, 8192, 8192), (8192, 3072, 1024), (8192, 1024, 1024), (8192, 4096, 1024), (8192, 1024, 4096),
          (4096, 1024, 1024), (16384, 12288, 4096), (8192, 250880 // 2, 1024)]
for (M, N, K) in shapes:
    A = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
    B = torch.randn(N, K, device=dev, dtype=torch.bfloat16)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    fl = 2.0 * M * N * K
    med, best = bench(lambda: torch.matmul(A, B.t(), out=out))
    row = dict(M=M, N=N, K=K, cublas_ms=med, cublas_tflops=fl / med / 1e9, cublas_best_tflops=fl / best / 1e9)
    for bn in [256, 192, 128]:
        med, best = bench(lambda: _C.gemm(A, B, out, False, False, None, None, None, 0, bn))
        row[f"ours_bn{bn}_ms"] = med
        row[f"ours_bn{bn}_tflops"] = fl / med / 1e9
        row[f"ours_bn{bn}_best_tflops"] = fl / best / 1e9
    # dgrad / wgrad layouts at auto BN
    Bt = B.t().contiguous()
    med, _ = bench(lambda: _C.gemm(A, Bt, out, False, True))
    row["ours_nn_tflops"] = fl / med / 1e9
    At = A.t().contiguous()
    med, _ = bench(lambda: _C.gemm(At, Bt, out, True, True))
    row["ours_tn_tflops"] = fl / med / 1e9
    results["perf"].append(row)
    print(json.dumps(row), flush=True)
    del A, B, out, Bt, At

os.makedirs(os.path.dirname(os.path.abspath(OUT)), exist_ok=True)
json.dump(results, open(OUT, "w"), indent=1)
print("ALL_OK", all_ok)
