"""GPU: the persistent encoder self-attention kernel (bf16, `op_encoder_attention("tcgen05", ...)`) on the walks it can
take.  Each CTA walks work tiles (query tile, head, stream); the CTA that computes a row, and where in its walk, must not
change the row: outputs are checked against fp32 softmax(QK^T)V and, bit for bit, against the same streams run one
at a time."""
import pytest
import torch

pytestmark = pytest.mark.gpu

GUARD = 256          # rows past the output that the kernel must leave alone


def _engine(d, H):
    from whisperlivekit_b200.dims import ModelDimensions
    from whisperlivekit_b200.engine import WhisperEngine
    return WhisperEngine(ModelDimensions(80, 1500, d, H, 1, 51864, 448, 64, 1, 1), None, [(0, 0)], precision="bf16",
                         max_sessions=1, max_batch=1)


def _attend(e, qkv, B, d):
    """the op on qkv [B*1500, 3d]; the output buffer is NaN-filled and GUARD rows longer than the output"""
    out = torch.full((B * 1500 + GUARD, d), float("nan"), device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    e.op_encoder_attention("tcgen05", qkv.data_ptr(), 1, B, out.data_ptr())
    e.sync()
    assert torch.isnan(out[B * 1500:].float()).all(), "rows past the output were written"
    return out[:B * 1500]


def _reference(qkv, B, d, H):
    x = qkv.float().view(B, 1500, 3, H, 64)
    q, k, v = x[:, :, 0].transpose(1, 2), x[:, :, 1].transpose(1, 2), x[:, :, 2].transpose(1, 2)
    return (torch.softmax(q @ k.transpose(-1, -2), dim=-1) @ v).transpose(1, 2).reshape(B * 1500, d)


# (1280, 20, 3): 480 work tiles of 192 query rows, so CTAs get an uneven number of them; (128, 2, 1): 16 work tiles,
# fewer than the SMs; (640, 10, 5): 400 work tiles over five streams
@pytest.mark.parametrize("d,H,B", [(1280, 20, 3), (128, 2, 1), (640, 10, 5)])
def test_encoder_attention_pp_walks(d, H, B):
    e = _engine(d, H)
    g = torch.Generator(device="cuda").manual_seed(d + 7 * H + B)
    qkv = (torch.randn(B * 1500, 3 * d, device="cuda", generator=g) * 0.8).bfloat16()
    out = _attend(e, qkv, B, d)
    # every row of every query tile is written, the ragged last one (rows 1344..1499 of 192) included
    assert not torch.isnan(out.float()).any()
    assert (out.float() - _reference(qkv, B, d, H)).abs().max().item() < 2e-2
    # each stream alone (another walk, another grid) gives the same bits
    for b in range(B):
        alone = _attend(e, qkv[b * 1500:(b + 1) * 1500].contiguous(), 1, d)
        assert torch.equal(alone, out[b * 1500:(b + 1) * 1500]), b
    # and a second run the same bits again
    assert torch.equal(_attend(e, qkv, B, d), out)
    e.close()


def test_encoder_attention_pp_last_key_tile():
    """The last key tile holds keys 1408..1499; the 36 rows past them in the loaded tile belong to the next stream (or
    are zero-filled past the tensor) and must get no weight.  Giving the next stream's keys huge scores and values
    makes any weight on them visible."""
    d, H, B = 128, 2, 2
    e = _engine(d, H)
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(B, 1500, 3, H, 64, device="cuda", generator=g) * 0.5
    x[1, :36, 1] *= 40.0                                      # stream 1's first keys: far above anything in stream 0
    x[1, :36, 2] += 1000.0
    qkv = x.reshape(B * 1500, 3 * d).bfloat16()
    out = _attend(e, qkv, B, d)
    assert not torch.isnan(out.float()).any()
    assert (out.float() - _reference(qkv, B, d, H)).abs()[:1500].max().item() < 2e-2
    e.close()
