#!/usr/bin/env python
"""Time the fused encoder attention alone: python tools/bench_attn.py [streams] [iters]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from whisperlivekit_b200.dims import ModelDimensions
from whisperlivekit_b200.engine import WhisperEngine
B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 10
d, H = 1280, 20
e = WhisperEngine(ModelDimensions(80, 1500, d, H, 1, 51864, 448, 64, 1, 1), None, [(0, 0)], precision="bf16", max_sessions=1, max_batch=1)
qkv = (torch.randn(B * 1500, 3 * d, device="cuda") * 0.35).bfloat16()
out = torch.empty(B * 1500, d, device="cuda", dtype=torch.bfloat16)
torch.cuda.synchronize()
for _ in range(3):
    e.op_encoder_attention("tcgen05", qkv.data_ptr(), 1, B, out.data_ptr())
e.timer_record(0)
for _ in range(iters):
    e.op_encoder_attention("tcgen05", qkv.data_ptr(), 1, B, out.data_ptr())
e.timer_record(1)
e.sync()
ms = e.timer_elapsed_ms(0, 1) / iters
exps = B * H * 1500 * 1536
print(f"attn B={B}: {ms*1e3:.1f} us  {4.0*B*H*1500*1500*64/ms/1e9:.0f} TFLOP/s  {exps/ms/1e6/132:.2f} Gexp/s/SM  pad={os.environ.get('WLK_ATTN_SMEM_PAD','0')}")
