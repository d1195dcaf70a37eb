"""GPU: the causal tower's attention (qwen_attention_kernel) and the windowed tower's fp32 attention
(qwin_attn_simt_kernel) run one shared core, attend_row_warp (csrc/attn_warp.cuh), and differ only in where they find
their keys.  A block-bidirectional causal job at start 0 whose left context covers the whole job sees exactly keys
0 .. n - 1, as one windowed block of the same n rows does, so on the same q / k / v the two kernels must agree bit for
bit."""
import pytest
import torch

from test_gpu_qwen_tower_kernels import ATTN_L, ATTN_LAYER, DEV, Q_STEPS_CAP, causal_engine, gen, tower_dims
from whisperlivekit_b200.qwen_engine import window_attention

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("H", [2, 14])
@pytest.mark.parametrize("n", [1, 17, 64, 128])
def test_causal_and_window_attention_share_one_core(n, H):
    d, left = 64 * H, Q_STEPS_CAP
    g = gen(100 * n + H)
    qkv = torch.randn(n, 3 * d, device=DEV, generator=g)
    qkv[:, :d] *= 0.125
    ring = torch.full((ATTN_L, 2, H, left + Q_STEPS_CAP, 64), float("nan"), device=DEV)
    ring[ATTN_LAYER, 0, :, :n] = qkv[:, d:2 * d].view(n, H, 64).transpose(0, 1)     # key at position p in slot p
    ring[ATTN_LAYER, 1, :, :n] = qkv[:, 2 * d:].view(n, H, 64).transpose(0, 1)
    q = qkv[:, :d].contiguous()
    causal = torch.full((n, d), float("nan"), device=DEV)
    eng = causal_engine("fp32", tower_dims(d, left=left, bidir=True, n_layer=ATTN_L))
    torch.cuda.synchronize()
    eng.op_attention(ATTN_LAYER, q.data_ptr(), [0], [n], [ring.data_ptr()], causal.data_ptr())
    torch.cuda.synchronize()
    eng.close()
    window = window_attention(qkv, [n], 0)
    assert torch.isfinite(causal).all()
    assert torch.equal(causal, window), float((causal - window).abs().max())
