#!/usr/bin/env python
"""Diagnose the wgmma attention kernel against fp32 torch: where (rows / dims) do errors sit?"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from whisperlivekit_b200.dims import ModelDimensions
from whisperlivekit_b200.engine import WhisperEngine

for d, H, B, scale in [(128, 2, 1, 0.8), (128, 2, 1, 0.1), (384, 6, 2, 0.8)]:
    e2 = WhisperEngine(ModelDimensions(80, 1500, d, H, 1, 51864, 448, 64, 1, 1), None, [(0, 0)], precision="bf16",
                       max_sessions=1, max_batch=1)
    g = torch.Generator(device="cuda").manual_seed(d)
    qkv = (torch.randn(B * 1500, 3 * d, device="cuda", generator=g) * scale).bfloat16()
    out = torch.full((B * 1500, d), float("nan"), device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    e2.op_encoder_attention("tcgen05", qkv.data_ptr(), 1, B, out.data_ptr())
    e2.sync()
    x = qkv.float().view(B, 1500, 3, H, 64)
    q, k, v = x[:, :, 0].transpose(1, 2), x[:, :, 1].transpose(1, 2), x[:, :, 2].transpose(1, 2)
    ref = (torch.softmax(q @ k.transpose(-1, -2), dim=-1) @ v).transpose(1, 2).reshape(B * 1500, d)
    err = (out.float() - ref).abs()
    print(f"d={d} H={H} B={B} scale={scale}: nan={int(torch.isnan(out.float()).sum())} max_err={err.nan_to_num(9).max().item():.4f}")
    e = err.nan_to_num(9).view(B, 1500, H, 2, 32)
    bad_rows = (e.amax(dim=(2, 3, 4)) > 2e-2)
    print("  bad rows per batch:", bad_rows.sum(dim=1).tolist(), " first bad:", [int(torch.nonzero(br)[0]) if br.any() else -1 for br in bad_rows])
    print("  max err per (head, dim half):", e.amax(dim=(0, 1, 4)).tolist())
    rows128 = e[0].amax(dim=(1, 2, 3))
    print("  max err per 128-row tile (batch 0):", [round(rows128[i:i + 128].max().item(), 3) for i in range(0, 1500, 128)])
    print("  max err by row%128 quadrant:", [round(torch.stack([rows128[i::128][:11] for i in range(qd * 32, qd * 32 + 32)]).max().item(), 3) for qd in range(4)])
    e2.close()
