"""GPU: op-level checks of the hand-written kernels through the C ABI (wlk_op_*),
against plain torch fp32 references of the same op."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from whisperlivekit_b200.dims import DIMS


@pytest.fixture(scope="module")
def eng():
    from whisperlivekit_b200.engine import WhisperEngine
    e = WhisperEngine(DIMS["micro"], None, [(0, 0)], precision="bf16", max_sessions=1, max_batch=1)
    yield e
    e.close()


def _gemm(eng, backend, A, W, bias, gelu, out_dtype):
    M, K = A.shape
    N = W.shape[0]
    Cm = torch.empty(M, N, device="cuda", dtype=out_dtype)
    code = {torch.float32: 0, torch.bfloat16: 1}
    torch.cuda.synchronize()
    eng.op_gemm(backend, A.data_ptr(), code[A.dtype], A.stride(0), W.data_ptr(), code[W.dtype], W.stride(0),
                bias.data_ptr() if bias is not None else None, Cm.data_ptr(), code[out_dtype], Cm.stride(0),
                M, N, K, gelu)
    eng.sync()
    return Cm


def _ref(A, W, bias, gelu):
    r = A.float() @ W.float().t()
    if bias is not None:
        r = r + bias
    if gelu:
        r = torch.nn.functional.gelu(r)
    return r


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (1500, 384, 384), (37, 51, 20), (16, 1280, 1280), (3, 51864, 128)])
@pytest.mark.parametrize("gelu", [False, True])
def test_gemm_simt_fp32(eng, M, N, K, gelu):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N)
    A = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g)
    out = _gemm(eng, "simt", A, W, b, gelu, torch.float32)
    ref = _ref(A.double(), W.double(), b.double(), gelu).float() if not gelu else _ref(A, W, b, gelu)
    assert (out - ref).abs().max().item() < 2e-4 * max(1.0, ref.abs().max().item())


SHAPES_TC = [(128, 256, 64), (256, 256, 128), (1500, 1280, 1280), (3000, 384, 240), (1000, 3840, 1280),
             (129, 264, 72), (64, 128, 5120), (4500, 5120, 1280), (12000, 1280, 5120),
             (16, 3840, 1280), (64, 1280, 1280), (1, 51864, 384), (200, 1280, 5120)]


@pytest.mark.parametrize("M,N,K", SHAPES_TC)
def test_gemm_tcgen05_bf16(eng, M, N, K):
    """Tensor-core (wgmma) GEMM vs fp32 reference on the same bf16-rounded operands: only the fp32
    accumulation order differs, so the bound is tight (1e-3 relative to the output scale)."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g)
    for gelu in (False, True):
        out = _gemm(eng, "tcgen05", A, W, b, gelu, torch.float32)
        ref = _ref(A, W, b, gelu)
        err = (out - ref).abs().max().item()
        assert err < 1e-3 * max(1.0, ref.abs().max().item()), (M, N, K, gelu, err)
    out_bf = _gemm(eng, "tcgen05", A, W, b, False, torch.bfloat16)
    ref = _ref(A, W, b, False)
    assert (out_bf.float() - ref).abs().max().item() < 2e-2 * max(1.0, ref.abs().max().item())
    simt = _gemm(eng, "simt", A, W, b, False, torch.float32)
    assert (simt - _gemm(eng, "tcgen05", A, W, b, False, torch.float32)).abs().max().item() < 1e-3 * max(1.0, ref.abs().max().item())


def test_gemm_tcgen05_strided_overlapping_rows(eng):
    """The conv stem feeds the GEMM overlapping rows (pitch < row length) through the TMA map."""
    g = torch.Generator(device="cuda").manual_seed(5)
    base = torch.randn(3002 * 80, device="cuda", generator=g).bfloat16()
    A = torch.as_strided(base, (3000, 240), (80, 1))
    W = (torch.randn(384, 240, device="cuda", generator=g) / 15).bfloat16()
    out = _gemm(eng, "tcgen05", A, W, None, False, torch.float32)
    ref = A.float() @ W.float().t()
    assert (out - ref).abs().max().item() < 1e-3 * ref.abs().max().item()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_encoder_attention_simt(eng, dtype):
    d, H, B = 128, 2, 2
    g = torch.Generator(device="cuda").manual_seed(3)
    qkv = (torch.randn(B * 1500, 3 * d, device="cuda", generator=g) * 0.8).to(dtype)
    out = torch.empty(B * 1500, d, device="cuda", dtype=dtype)
    torch.cuda.synchronize()
    eng.op_encoder_attention("simt", qkv.data_ptr(), 0 if dtype == torch.float32 else 1, B, out.data_ptr())
    eng.sync()
    x = qkv.float().view(B, 1500, 3, H, 64)
    q, k, v = x[:, :, 0].transpose(1, 2), x[:, :, 1].transpose(1, 2), x[:, :, 2].transpose(1, 2)
    ref = (torch.softmax(q @ k.transpose(-1, -2), dim=-1) @ v).transpose(1, 2).reshape(B * 1500, d)
    tol = 2e-5 if dtype == torch.float32 else 1e-2
    assert (out.float() - ref).abs().max().item() < tol


@pytest.mark.parametrize("d,H,B", [(128, 2, 1), (384, 6, 2), (1280, 20, 1)])
def test_encoder_attention_tcgen05(eng, d, H, B):
    """Fused tensor-core attention vs fp32 softmax(QK^T)V on the same bf16 inputs.  P is rounded to
    bf16 before the PV product (8 mantissa bits): tolerance 2e-2 on outputs of O(1)."""
    from whisperlivekit_b200.dims import ModelDimensions
    from whisperlivekit_b200.engine import WhisperEngine
    e2 = WhisperEngine(ModelDimensions(80, 1500, d, H, 1, 51864, 448, 64, 1, 1), None, [(0, 0)], precision="bf16",
                       max_sessions=1, max_batch=1)
    g = torch.Generator(device="cuda").manual_seed(d)
    qkv = (torch.randn(B * 1500, 3 * d, device="cuda", generator=g) * 0.8).bfloat16()
    out = torch.full((B * 1500, d), float("nan"), device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    e2.op_encoder_attention("tcgen05", qkv.data_ptr(), 1, B, out.data_ptr())
    e2.sync()
    x = qkv.float().view(B, 1500, 3, H, 64)
    q, k, v = x[:, :, 0].transpose(1, 2), x[:, :, 1].transpose(1, 2), x[:, :, 2].transpose(1, 2)
    ref = (torch.softmax(q @ k.transpose(-1, -2), dim=-1) @ v).transpose(1, 2).reshape(B * 1500, d)
    assert not torch.isnan(out.float()).any()
    assert (out.float() - ref).abs().max().item() < 2e-2
    e2.close()


def test_encoder_attention_tcgen05_moving_reference():
    """The online softmax keeps a running maximum per row and rescales O and l in registers whenever a key tile raises it.
    With random inputs the maximum settles in the first tiles: here the keys of later tiles are scaled up so that most rows
    move it by large factors several times, at different tiles."""
    from whisperlivekit_b200.dims import ModelDimensions
    from whisperlivekit_b200.engine import WhisperEngine
    d, H, B = 256, 4, 2
    e2 = WhisperEngine(ModelDimensions(80, 1500, d, H, 1, 51864, 448, 64, 1, 1), None, [(0, 0)], precision="bf16",
                       max_sessions=1, max_batch=1)
    g = torch.Generator(device="cuda").manual_seed(77)
    x = torch.randn(B, 1500, 3, H, 64, device="cuda", generator=g) * 0.7
    ramp = torch.ones(1500, device="cuda")
    ramp[400:] = 1.8; ramp[700:] = 2.6; ramp[1000:] = 3.5; ramp[1300:] = 4.5       # key norms grow tile by tile
    x[:, :, 1] *= ramp[None, :, None, None]
    x[1, :, 1, 1] *= torch.linspace(1.0, 0.2, 1500, device="cuda")[:, None]         # ... and one head where they shrink
    qkv = x.reshape(B * 1500, 3 * d).bfloat16()
    out = torch.full((B * 1500, d), float("nan"), device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    e2.op_encoder_attention("tcgen05", qkv.data_ptr(), 1, B, out.data_ptr())
    e2.sync()
    xf = qkv.float().view(B, 1500, 3, H, 64)
    q, k, v = xf[:, :, 0].transpose(1, 2), xf[:, :, 1].transpose(1, 2), xf[:, :, 2].transpose(1, 2)
    s = q @ k.transpose(-1, -2)
    jump = (s[..., 1280:].amax(-1) - s[..., :128].amax(-1)) * 1.4427                # log2 units, last tile vs first
    assert (jump > 8).float().mean().item() > 0.5                                   # the path under test is really taken
    ref = (torch.softmax(s, dim=-1) @ v).transpose(1, 2).reshape(B * 1500, d)
    assert not torch.isnan(out.float()).any()
    assert (out.float() - ref).abs().max().item() < 3e-2
    e2.close()


@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (512, 512, 256), (1500, 1280, 1280), (3000, 384, 240),
                                   (257, 300, 72), (24000, 1280, 1280), (4500, 5120, 1280)])
def test_gemm_tcgen05_cta_pair(eng, M, N, K):
    """The 128-wide-tile instantiation (backend "tcgen05_pair") vs fp32 reference and vs the 64-wide one ("tcgen05_1cta")."""
    g = torch.Generator(device="cuda").manual_seed(M + 3 * N + K)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g)
    out = _gemm(eng, "tcgen05_pair", A, W, b, True, torch.float32)
    ref = _ref(A, W, b, True)
    assert not torch.isnan(out).any()
    assert (out - ref).abs().max().item() < 1e-3 * max(1.0, ref.abs().max().item())
    one = _gemm(eng, "tcgen05_1cta", A, W, b, True, torch.float32)
    assert (out - one).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("M,N,K", [(16, 1280, 1280), (64, 1280, 5120), (1, 384, 1536), (48, 512, 512)])
def test_gemm_tcgen05_split_k_in_place(eng, M, N, K):
    """Decoder-shaped GEMMs updating the fp32 residual stream in place (x += A W^T + b): the short/narrow
    case is split along K with fp32 atomics."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g)
    x0 = torch.randn(M, N, device="cuda", generator=g)
    x = x0.clone()
    torch.cuda.synchronize()
    eng.op_gemm("tcgen05", A.data_ptr(), 1, K, W.data_ptr(), 1, K, b.data_ptr(), x.data_ptr(), 0, N, M, N, K, 2)
    eng.sync()
    ref = x0 + A.float() @ W.float().t() + b
    assert (x - ref).abs().max().item() < 1e-3 * max(1.0, ref.abs().max().item())
