"""GPU: the 128 x 128 ping-pong wgmma GEMM (backend "tcgen05_pair", and "tcgen05" where it picks 128-wide tiles) through
wlk_op_gemm, against an fp32 reference of the same bf16 operands and against the 64-wide kernel ("tcgen05_1cta").

The two consumer warpgroups of a CTA take alternate tiles of its walk and skip each other's k-slabs in the shared ring,
so the shapes cover every way a walk can end: one tile per CTA (the second consumer idle), tile counts below 2 x SMs
(some CTAs with one tile, some with two), exact multiples of the grid, odd tile counts per CTA, ragged M and N, fewer
k-slabs than the ring is deep, and long K."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from whisperlivekit_b200.dims import DIMS

CODE = {torch.float32: 0, torch.bfloat16: 1}


@pytest.fixture(scope="module")
def eng():
    from whisperlivekit_b200.engine import WhisperEngine
    e = WhisperEngine(DIMS["micro"], None, [(0, 0)], precision="bf16", max_sessions=1, max_batch=1)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(eng, backend, A, lda, W, bias, C, gelu_bits, M, N, K):
    torch.cuda.synchronize()
    eng.op_gemm(backend, A.data_ptr(), 1, lda, W.data_ptr(), 1, K, bias.data_ptr() if bias is not None else None,
                C.data_ptr(), CODE[C.dtype], C.stride(0), M, N, K, gelu_bits)
    eng.sync()
    return C


def _operands(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g)
    return A, W, b, g


def _check(eng, A, lda, W, b, gelu, out_dtype, M, N, K):
    ref = A.float() @ W.float().t() + b
    if gelu:
        ref = torch.nn.functional.gelu(ref)
    scale = max(1.0, ref.abs().max().item())
    out = _run(eng, "tcgen05_pair", A, lda, W, b, torch.full((M, N), float("nan"), device="cuda", dtype=out_dtype),
               int(gelu), M, N, K)
    assert not torch.isnan(out.float()).any()
    tol = 1e-3 if out_dtype == torch.float32 else 8e-3          # bf16 output: one rounding of the result
    assert (out.float() - ref).abs().max().item() < tol * scale
    one = _run(eng, "tcgen05_1cta", A, lda, W, b, torch.empty(M, N, device="cuda", dtype=out_dtype), int(gelu), M, N, K)
    if out_dtype == torch.float32:
        assert (out - one).abs().max().item() < 1e-4 * scale
    else:
        assert (out.float() - one.float()).abs().max().item() <= 8e-3 * scale


# (M, N) sized from the SM count: tiles per CTA 1 (fewer tiles than SMs, and a two-tile grid with a ragged M), 1 or 2
# (fewer than 2 x SMs), exactly 2, exactly 3 (odd), and 7 or 8 with a ragged last m block
def _walk_shapes(sms):
    return [(40 * 128, 128), (sms + 7, 128), (10 * 128, sms // 10 * 128 + 128),
            (2 * sms * 128 // 12, 12 * 128), (3 * sms * 128 // 12, 12 * 128), (7 * sms * 128 // 12 + 77, 12 * 128)]


@pytest.mark.parametrize("walk", range(6))
@pytest.mark.parametrize("gelu", [False, True])
def test_pingpong_walks(eng, sms, walk, gelu):
    M, N = _walk_shapes(sms)[walk]
    K = 1280
    A, W, b, _ = _operands(M, N, K, 100 + walk)
    _check(eng, A, K, W, b, gelu, torch.float32, M, N, K)


@pytest.mark.parametrize("M,N,K", [(1000, 1000, 1280), (129, 264, 72), (3001, 200, 384), (2000, 640, 256),
                                   (1500, 1280, 5120), (300, 51, 320)])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_pingpong_ragged_and_k(eng, M, N, K, out_dtype):
    """M and N off the tile grid, K below the ring depth (4 to 6 k-slabs against 6 stages) and K = 5120."""
    A, W, b, _ = _operands(M, N, K, M + N + K)
    _check(eng, A, K, W, b, True, out_dtype, M, N, K)


def test_pingpong_overlapping_rows(eng):
    """The conv stem's operand: rows of pitch 128 reading 384 columns of one buffer."""
    g = torch.Generator(device="cuda").manual_seed(9)
    M, N, K, lda = 6000, 1280, 384, 128
    base = torch.randn((M - 1) * lda + K, device="cuda", generator=g).bfloat16()
    A = torch.as_strided(base, (M, K), (lda, 1))
    W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g)
    _check(eng, A, lda, W, b, True, torch.float32, M, N, K)


@pytest.mark.parametrize("M,N,K", [(24000, 1280, 1280), (1500, 1280, 5120), (777, 384, 1280), (130, 130, 64)])
@pytest.mark.parametrize("backend", ["tcgen05_pair", "tcgen05"])
def test_pingpong_residual_in_place(eng, M, N, K, backend):
    """x += A W^T + b on the fp32 residual stream: C aliases the residual (attention-out and FC2)."""
    A, W, b, g = _operands(M, N, K, 7 * M + K)
    x0 = torch.randn(M, N, device="cuda", generator=g)
    ref = x0 + A.float() @ W.float().t() + b
    scale = max(1.0, ref.abs().max().item())
    x = _run(eng, backend, A, K, W, b, x0.clone(), 2, M, N, K)
    assert (x - ref).abs().max().item() < 1e-3 * scale
    y = _run(eng, "tcgen05_1cta", A, K, W, b, x0.clone(), 2, M, N, K)
    assert (x - y).abs().max().item() < 1e-4 * scale
