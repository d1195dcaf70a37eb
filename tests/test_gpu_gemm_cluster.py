"""GPU: the 128 x 128 ping-pong wgmma GEMM in thread-block clusters (backends "tcgen05_pp2x1", "tcgen05_pp1x2",
"tcgen05_pp2x2", and "tcgen05" where it picks 128-wide tiles) against the same kernel on lone CTAs ("tcgen05_pair").

A cluster only changes which CTA loads which rows of a k-slab from L2: every output element gets the same wgmmas in the
same K order, so the outputs must be bitwise equal to the lone-CTA kernel's.  The shapes are those of
tests/test_gpu_gemm_pingpong.py plus the cases that only clusters have: an odd number of m blocks (the cluster's second
tile lies past M), N off a multiple of 256 (past N for 1x2), fewer cluster-tiles than the grid holds (down to one), and
fewer k-slabs than the ring is deep."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from whisperlivekit_b200.dims import DIMS

CODE = {torch.float32: 0, torch.bfloat16: 1}
CLUSTERS = ["tcgen05_pp2x1", "tcgen05_pp1x2", "tcgen05_pp2x2"]


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


def _auto_is_128(M, N, sms):
    """gemm_tcgen05's auto path takes 128-wide tiles while they cover half the SMs (else the 64-wide kernel)."""
    return N >= 128 and -(-M // 128) * -(-N // 128) >= sms // 2


def _equal_to_lone(eng, sms, A, lda, W, b, gelu, out_dtype, M, N, K):
    """Every cluster shape (and auto, where it runs this kernel) writes exactly what the lone-CTA kernel writes, and
    nothing outside [M, N] (C is a view into a NaN-filled buffer one tile larger each way)."""
    def out():
        buf = torch.full((M + 128, N + 136), float("nan"), device="cuda", dtype=out_dtype)
        return buf, buf[:M, :N]
    ref_buf, ref = out()
    _run(eng, "tcgen05_pair", A, lda, W, b, ref, int(gelu), M, N, K)
    assert not torch.isnan(ref.float()).any()
    for backend in CLUSTERS + (["tcgen05"] if _auto_is_128(M, N, sms) else []):
        buf, C = out()
        _run(eng, backend, A, lda, W, b, C, int(gelu), M, N, K)
        assert torch.equal(C, ref), backend
        assert torch.equal(buf.isnan(), ref_buf.isnan()), backend


def _walk_shapes(sms):
    return [(40 * 128, 128), (sms + 7, 128), (10 * 128, sms // 10 * 128 + 128),
            (2 * sms * 128 // 12, 12 * 128), (3 * sms * 128 // 12, 12 * 128), (7 * sms * 128 // 12 + 77, 12 * 128)]


@pytest.mark.parametrize("walk", range(6))
@pytest.mark.parametrize("gelu", [False, True])
def test_cluster_walks(eng, sms, walk, gelu):
    M, N = _walk_shapes(sms)[walk]
    K = 1280
    A, W, b, _ = _operands(M, N, K, 100 + walk)
    _equal_to_lone(eng, sms, A, K, W, b, gelu, torch.float32, M, N, K)


@pytest.mark.parametrize("M,N,K", [(1000, 1000, 1280), (129, 264, 72), (3001, 200, 384), (2000, 640, 256),
                                   (1500, 1280, 5120), (300, 51, 320)])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_cluster_ragged_and_k(eng, sms, M, N, K, out_dtype):
    A, W, b, _ = _operands(M, N, K, M + N + K)
    _equal_to_lone(eng, sms, A, K, W, b, True, out_dtype, M, N, K)


@pytest.mark.parametrize("M,N,K", [
    (563 * 128 - 61, 1280, 1280),    # odd num_m (the 48-stream encoder's 563) with a ragged last block
    (9 * 128 + 5, 3 * 128 + 40, 640),  # odd num_m and odd num_n, both ragged: every cluster shape has idle tiles
    (4000, 384, 1280),               # N = 3 x 128: not a multiple of 256
    (4000, 640 + 8, 1280),           # N a multiple of neither 128 nor 256
    (128, 128, 1280),                # a single tile: one cluster-tile, most of the cluster idle
    (100, 70, 64),                   # a single partial tile and one k-slab
    (3 * 128, 2 * 128, 1280),        # fewer cluster-tiles than the device holds clusters
    (7000, 1280, 192),               # three k-slabs: fewer than the six-deep ring
    (2 * 128 + 1, 1280, 320),        # five k-slabs, odd num_m
])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_cluster_edges(eng, sms, M, N, K, out_dtype):
    A, W, b, _ = _operands(M, N, K, 3 * M + N + K)
    _equal_to_lone(eng, sms, A, K, W, b, True, out_dtype, M, N, K)


def test_cluster_overlapping_rows(eng, sms):
    """The conv stem's operand: rows of pitch 128 reading 384 columns of one buffer."""
    g = torch.Generator(device="cuda").manual_seed(9)
    M, N, K, lda = 6000, 1280, 384, 128
    base = torch.randn((M - 1) * lda + K, device="cuda", generator=g).bfloat16()
    A = torch.as_strided(base, (M, K), (lda, 1))
    W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g)
    _equal_to_lone(eng, sms, A, lda, W, b, True, torch.float32, M, N, K)


@pytest.mark.parametrize("M,N,K", [(24000, 1280, 1280), (1500, 1280, 5120), (777, 384, 1280), (130, 130, 64)])
def test_cluster_residual_in_place(eng, sms, M, N, K):
    """x += A W^T + b on the fp32 residual stream, C aliasing the residual (attention-out and FC2)."""
    A, W, b, g = _operands(M, N, K, 7 * M + K)
    x0 = torch.randn(M, N, device="cuda", generator=g)
    y = _run(eng, "tcgen05_pair", A, K, W, b, x0.clone(), 2, M, N, K)
    for backend in CLUSTERS + (["tcgen05"] if _auto_is_128(M, N, sms) else []):
        x = _run(eng, backend, A, K, W, b, x0.clone(), 2, M, N, K)
        assert torch.equal(x, y), backend
