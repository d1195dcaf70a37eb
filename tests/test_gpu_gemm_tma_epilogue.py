"""GPU: the ping-pong wgmma GEMM's staged epilogue through wlk_op_gemm: a plain row-major output leaves by TMA tile
stores out of shared memory.  Each result is checked against an fp32 reference of the same bf16 operands, and bitwise
against the same kernel's register-path epilogue, which the kernel runs when C's row pitch is not a multiple of 16
bytes (no tensor map can address it).  The fp32 residual accumulated in place (x += A W^T + b) stays on the register
path; it is checked here at the same shapes and pitches.

The shapes cover TMA clipping (ragged M and N, a sub-tile wholly past N, rows and columns of the buffer beyond the
problem left untouched), 1500-row stream boundaries inside a tile, walks with more tiles per consumer than it has
staging buffers, walks that leave the second consumer idle, and cluster-padding tiles of the 2 x 2 clusters."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from whisperlivekit_b200.dims import DIMS

CODE = {torch.float32: 0, torch.bfloat16: 1}
SENTINEL = -4096.0                     # exact in bf16 and fp32; never produced by these problems
K = 1280

# (M, N): ragged M and N; a tile's last fp32 sub-tile wholly past N, four tiles (one per CTA: the second consumer idle);
# two 1500-row streams; 40 tiles of 128 x 128 (one per CTA); 16 streams (~14 tiles per CTA, 7 per consumer); 36 x 5
# tiles (odd n blocks: 2 x 2 cluster padding)
SHAPES = [(1000, 1000), (130, 200), (3000, 1280), (40 * 128, 128), (24000, 1280), (4500, 640)]
# output type and epilogue bits of wlk_op_gemm (1: GELU, 2: fp32 residual accumulated in place)
MODES = {"bf16_gelu": (torch.bfloat16, 1), "bf16_bias": (torch.bfloat16, 0), "f32_gelu": (torch.float32, 1),
         "f32_residual": (torch.float32, 2)}


@pytest.fixture(scope="module")
def eng():
    from whisperlivekit_b200.engine import WhisperEngine
    e = WhisperEngine(DIMS["micro"], None, [(0, 0)], precision="bf16", max_sessions=1, max_batch=1)
    yield e
    e.close()


def _gemm(eng, backend, A, W, b, C, bits, M, N):
    torch.cuda.synchronize()
    eng.op_gemm(backend, A.data_ptr(), 1, K, W.data_ptr(), 1, K, b.data_ptr(), C.data_ptr(), CODE[C.dtype], C.stride(0),
                M, N, K, bits)
    eng.sync()


def _buffer(M, N, ld, dtype, x0):
    """[M + 3, ld] filled with SENTINEL; x0 (the residual) in its [M, N] corner."""
    C = torch.full((M + 3, ld), SENTINEL, device="cuda", dtype=dtype)
    if x0 is not None:
        C[:M, :N] = x0
    return C


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("backend", ["tcgen05_pair", "tcgen05_pp2x2"])
@pytest.mark.parametrize("shape", range(len(SHAPES)))
def test_tma_epilogue(eng, shape, backend, mode):
    M, N = SHAPES[shape]
    dtype, bits = MODES[mode]
    g = torch.Generator(device="cuda").manual_seed(1000 * shape + 17 * bits + (dtype == torch.float32))
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g)
    x0 = torch.randn(M, N, device="cuda", generator=g) if bits & 2 else None

    es = torch.finfo(dtype).bits // 8
    ld_tma = (N + 7) // 8 * 8 + 8                 # 16-byte pitch, columns past N: the staged path
    ld_reg = N + 1 if (N + 1) * es % 16 else N + 2  # pitch off 16 bytes: the register path
    C = _buffer(M, N, ld_tma, dtype, x0)
    _gemm(eng, backend, A, W, b, C, bits, M, N)
    R = _buffer(M, N, ld_reg, dtype, x0)
    _gemm(eng, backend, A, W, b, R, bits, M, N)

    # nothing outside the [M, N] box was written (TMA clips at M and N)
    assert bool((C[M:] == SENTINEL).all()) and bool((C[:M, N:] == SENTINEL).all())
    assert bool((R[M:] == SENTINEL).all()) and bool((R[:M, N:] == SENTINEL).all())
    out = C[:M, :N]
    # the same arithmetic in the same order as the register path: bitwise equal
    assert torch.equal(out, R[:M, :N])

    ref = A.float() @ W.float().t() + b
    if bits & 1:
        ref = torch.nn.functional.gelu(ref)
    if x0 is not None:
        ref = ref + x0
    scale = max(1.0, ref.abs().max().item())
    tol = 1e-3 if dtype == torch.float32 else 8e-3          # bf16 output: one rounding of the result
    assert not torch.isnan(out.float()).any()
    assert (out.float() - ref).abs().max().item() < tol * scale
