"""Run each hot kernel a few times at a flagship-model shape (for `ncu --set full -k regex:<name>`)."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pipegoose_b200.ops import native, kernels as K
n = native()
dev = "cuda"
which = sys.argv[1] if len(sys.argv) > 1 else "gemm"
torch.manual_seed(0)
if which == "gemm":
    M, N, Kd = 8192, 4096, 1024  # bloom-560m fc1
    a = torch.randn(M, Kd, device=dev, dtype=torch.bfloat16); b = torch.randn(N, Kd, device=dev, dtype=torch.bfloat16)
    bias = torch.randn(N, device=dev, dtype=torch.bfloat16)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16); aux = torch.empty_like(out)
    for _ in range(6): n.gemm(a, b, out, False, False, bias, None, aux, 2)
elif which == "gemm_pair":
    # lm_head-like (long N) shape
    M, N, Kd = 8192, 32768, 1024
    a = torch.randn(M, Kd, device=dev, dtype=torch.bfloat16); b = torch.randn(N, Kd, device=dev, dtype=torch.bfloat16)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    for _ in range(6): n.gemm(a, b, out)
elif which == "gemm_big":
    M = N = Kd = 8192
    a = torch.randn(M, Kd, device=dev, dtype=torch.bfloat16); b = torch.randn(N, Kd, device=dev, dtype=torch.bfloat16)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    for _ in range(6): n.gemm(a, b, out)
elif which == "lm_head_ce":
    # lm_head logits GEMM with the cross-entropy statistics in its epilogue (bloom-560m, 8192 tokens, TP2 shard of the vocabulary)
    M, N, Kd = 8192, 125440, 1024
    a = torch.randn(M, Kd, device=dev, dtype=torch.bfloat16); b = torch.randn(N, Kd, device=dev, dtype=torch.bfloat16) * 0.05
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    part = K.ce_partials_buffer(M, N, dev)
    for _ in range(4): n.gemm(a, b, out, ag={"ce_part": part.data_ptr(), "ce_valid": N})
elif which == "attn":
    B, S, H, D = 8, 1024, 16, 64
    qkv = torch.randn(B * S, H * 3 * D, device=dev, dtype=torch.bfloat16); slopes = K.alibi_slopes(H, device=dev)
    out = torch.empty(B * S, H * D, device=dev, dtype=torch.bfloat16); lse = torch.empty(B, H, S, device=dev)
    dout = torch.randn_like(out); dqkv = torch.empty_like(qkv)
    for _ in range(4):
        n.attention_fwd(qkv, slopes, out, lse, B, S, H, D)
        n.attention_bwd(qkv, slopes, out, lse, dout, dqkv, B, S, H, D)
torch.cuda.synchronize()
