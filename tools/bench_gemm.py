#!/usr/bin/env python
"""Micro-benchmark of the wgmma GEMM (for ncu captures): python tools/bench_gemm.py M N K [iters]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from whisperlivekit_b200.dims import DIMS
from whisperlivekit_b200.engine import WhisperEngine

M, N, K = (int(x) for x in sys.argv[1:4]) if len(sys.argv) >= 4 else (24000, 5120, 1280)
iters = int(sys.argv[4]) if len(sys.argv) > 4 else 5
out_bf16 = os.environ.get("OUT", "bf16") == "bf16"
gelu = int(os.environ.get("GELU", "1"))        # bit 0: GELU, bit 1: fp32 residual accumulated in place (OUT=f32)
eng = WhisperEngine(DIMS["micro"], None, [(0, 0)], precision="bf16", max_sessions=1, max_batch=1)
A = torch.randn(M, K, device="cuda").bfloat16()
ROT = int(os.environ.get("ROTATE", "1"))          # > 1: cycle through that many weight copies (HBM-streaming regime)
Ws = [(torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16() for _ in range(ROT)]
W = Ws[0]
b = torch.randn(N, device="cuda")
C = torch.empty(M, N, device="cuda", dtype=torch.bfloat16 if out_bf16 else torch.float32)
torch.cuda.synchronize()
for _ in range(2):
    eng.op_gemm(os.environ.get("BACKEND", "tcgen05"), A.data_ptr(), 1, K, W.data_ptr(), 1, K, b.data_ptr(), C.data_ptr(), 1 if out_bf16 else 0, N, M, N, K, gelu)
eng.timer_record(0)
for i in range(iters):
    eng.op_gemm(os.environ.get("BACKEND", "tcgen05"), A.data_ptr(), 1, K, Ws[i % ROT].data_ptr(), 1, K, b.data_ptr(), C.data_ptr(), 1 if out_bf16 else 0, N, M, N, K, gelu)
eng.timer_record(1)
ms = eng.timer_elapsed_ms(0, 1) / iters
print(f"gemm rot={ROT} {M}x{N}x{K} gelu={int(gelu)} out={"bf16" if out_bf16 else "f32"}: {ms:.3f} ms  {2.0*M*N*K/ms/1e9:.1f} TFLOP/s")
