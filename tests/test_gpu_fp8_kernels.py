"""GPU: the FP8 (WLK_PREC_FP8) kernels op by op -- per-row e4m3 quantization, the LayerNorm with e4m3 output and the FC1
output-scale bound it writes, and the e4m3 wgmma GEMM with the encoder's three epilogues -- against float64 references
on the decoded operands, so that what is left is the kernels' own rounding and the FP8 tensor cores' accumulation."""
import json
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from whisperlivekit_b200.dims import DIMS

F32, BF16, E4M3 = 0, 1, 3
FMAX = 448.0
# |C - ref| <= TAU * sum_k |a_k w_k| (+ one output ulp): the FP8 wgmma accumulates all of K in its own accumulator, which
# keeps fewer bits than fp32 (DESIGN.md section 3 records the measured worst ratio next to this bound)
TAU = 2.0 ** -9


@pytest.fixture(scope="module")
def eng():
    from whisperlivekit_b200.engine import WhisperEngine
    e = WhisperEngine(DIMS["micro"], None, [(0, 0)], precision="bf16", max_sessions=1, max_batch=1)
    yield e
    e.close()


def _dec(q):
    return q.view(torch.float8_e4m3fn).double()


def _quantize(eng, x):
    """-> (e4m3 bytes as uint8, fp32 row scales) of a 2-D fp32 / bf16 tensor, by wlk_op_quantize_rows"""
    rows, cols = x.shape
    q = torch.full((rows, cols), 0x55, device="cuda", dtype=torch.uint8)
    s = torch.full((rows,), -1.0, device="cuda")
    torch.cuda.synchronize()
    eng.op_quantize_rows(x.data_ptr(), F32 if x.dtype == torch.float32 else BF16, x.stride(0), rows, cols, q.data_ptr(),
                         q.stride(0), s.data_ptr())
    eng.sync()
    return q, s


def _e4m3_ulp(v):
    """spacing of e4m3 at |v| (subnormal spacing 2^-9 below 2^-6)"""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -6)))
    return torch.pow(2.0, e - 3)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_quantize_rows_matches_torch(eng, dtype):
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(6, 1280, device="cuda", generator=g)
    x[1] *= 1e4
    x[2] *= 1e-6
    x[3] = 0.0
    x[3, 17] = -3.5                                    # single spike
    x[4] = 0.0                                         # all zero
    x = x.to(dtype)
    q, s = _quantize(eng, x)
    xf = x.float()
    amax = xf.abs().amax(dim=1)
    assert torch.equal(s, amax / torch.full_like(amax, FMAX))     # (a tensor / scalar division multiplies by 1/448)
    nz = amax > 0
    ref = (xf[nz] / s[nz, None]).clamp(-FMAX, FMAX).to(torch.float8_e4m3fn).view(torch.uint8)
    assert torch.equal(q[nz], ref)
    assert s[4].item() == 0.0 and int(q[4].abs().sum()) == 0 and not torch.isnan(_dec(q)).any()


def _ln64(x, w, b):
    x = x.double()
    mu = x.mean(dim=1, keepdim=True)
    var = ((x - mu) ** 2).mean(dim=1, keepdim=True)
    return (x - mu) / torch.sqrt(var + 1e-5) * w.double() + b.double()


def _gelu64(h):
    return 0.5 * h * (1.0 + torch.erf(h / math.sqrt(2.0)))


def test_layernorm_fp8_scales_bytes_and_fc1_bound(eng):
    d, R = 1280, 64
    g = torch.Generator(device="cuda").manual_seed(5)
    W1 = torch.randn(4 * d, d, device="cuda", generator=g) * 0.02
    b1 = torch.randn(4 * d, device="cuda", generator=g) * 0.5
    w = 1.0 + 0.1 * torch.randn(d, device="cuda", generator=g)
    b = 0.1 * torch.randn(d, device="cuda", generator=g)
    x = torch.randn(R, d, device="cuda", generator=g) * 3.0
    # adversarial rows: parallel to a weight row (after the LayerNorm's affine map), so Cauchy-Schwarz is nearly tight
    for r in range(R // 2, R):
        x[r] = (W1[r * 37 % (4 * d)] - b) / w
    W1q, s1 = _quantize(eng, W1)
    W1h = _dec(W1q) * s1.double()[:, None]
    wnorm = float(W1h.norm(dim=1).max())
    bmax = float(b1.abs().max())
    out = torch.zeros(R, d, device="cuda", dtype=torch.uint8)
    s_a = torch.zeros(R, device="cuda")
    s_h = torch.zeros(R, device="cuda")
    torch.cuda.synchronize()
    eng.op_layernorm_fp8(x.data_ptr(), d, w.data_ptr(), b.data_ptr(), R, d, out.data_ptr(), d, s_a.data_ptr(),
                         s_h.data_ptr(), wnorm, bmax)
    eng.sync()
    y = _ln64(x, w, b)
    amax = y.abs().amax(dim=1)
    assert torch.allclose(s_a.double(), amax / FMAX, rtol=1e-5, atol=0)
    ref = (y / s_a.double()[:, None]).clamp(-FMAX, FMAX)
    refq = ref.float().to(torch.float8_e4m3fn).double()
    assert ((_dec(out) - refq).abs() <= _e4m3_ulp(refq) + 1e-12).all()

    yh = _dec(out) * s_a.double()[:, None]
    h = yh @ W1h.T + b1.double()
    gmax = _gelu64(h).abs().amax(dim=1)
    cap = FMAX * s_h.double()
    assert (gmax <= cap * (1 + 1e-5)).all(), float((gmax / cap).max())
    # the FC1 kernel's e4m3 output of these rows saturates nowhere
    hid = torch.zeros(R, 4 * d, device="cuda", dtype=torch.uint8)
    torch.cuda.synchronize()
    eng.op_gemm_fp8("tcgen05", out.data_ptr(), s_a.data_ptr(), d, W1q.data_ptr(), s1.data_ptr(), d, b1.data_ptr(),
                    hid.data_ptr(), E4M3, 4 * d, R, 4 * d, d, c_scale_ptr=s_h.data_ptr(), gelu=True)
    eng.sync()
    assert not (_dec(hid).abs() >= FMAX).any()
    # slack of the bound, and the error against exact per-row amax quantization of the hidden (reported)
    hid_ref = _gelu64(h)
    exact_s = hid_ref.abs().amax(dim=1, keepdim=True) / FMAX
    exact = (hid_ref / exact_s).float().to(torch.float8_e4m3fn).double() * exact_s
    got = _dec(hid) * s_h.double()[:, None]
    den = hid_ref.abs().amax(dim=1)
    print(json.dumps(dict(
        bound_slack_random=float((cap / gmax)[: R // 2].median()), bound_slack_adversarial=float((cap / gmax)[R // 2:].max()),
        hidden_err_bound=float(((got - hid_ref).abs().amax(dim=1) / den).max()),
        hidden_err_exact_amax=float(((exact - hid_ref).abs().amax(dim=1) / den).max()))))


# epilogues of the encoder's three e4m3 GEMMs: (N, K) and the epilogue
EPIS = {"qkv": (3840, 1280), "fc1": (5120, 1280), "fc2": (1280, 5120), "qkv_ragged_n": (1000, 1280)}
VARIANTS = ["tcgen05", "tcgen05_pair", "tcgen05_pp2x1", "tcgen05_pp1x2", "tcgen05_pp2x2"]
_WORST = {}


@pytest.mark.parametrize("epi", list(EPIS))
@pytest.mark.parametrize("M", [1, 127, 128, 1500, 3077])
def test_gemm_fp8(eng, M, epi):
    N, K = EPIS[epi]
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N + K)
    A32 = torch.randn(M, K, device="cuda", generator=g) * (1 + torch.rand(M, 1, device="cuda", generator=g) * 4)
    W32 = torch.randn(N, K, device="cuda", generator=g) * 0.03
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    Aq, sa = _quantize(eng, A32)
    Wq, sw = _quantize(eng, W32)
    Ah, Wh = _dec(Aq) * sa.double()[:, None], _dec(Wq) * sw.double()[:, None]
    acc = Ah @ Wh.T
    S = Ah.abs() @ Wh.abs().T                               # sum_k |a_k w_k|
    x0 = torch.randn(M, N, device="cuda", generator=g)
    qk = 64 ** -0.25
    if epi.startswith("qkv"):
        ref = acc + bias.double()
        ref[:, : 2 * (N // 3) // 8 * 8] *= qk               # (the epilogue scales whole 8-column chunks)
        err_scale = S * qk
        c_type, ldc, tdtype = BF16, N, torch.bfloat16
    elif epi == "fc1":
        h = acc + bias.double()
        ref = _gelu64(h)
        err_scale = S * 1.13                                 # |GELU'| <= 1.13
        c_scale = (ref.abs().amax(dim=1) / FMAX * 1.25).float().clamp_min(1e-30)
        c_type, ldc, tdtype = E4M3, N, torch.uint8
    else:
        ref = acc + bias.double() + x0.double()
        err_scale = S
        c_type, ldc, tdtype = F32, N, torch.float32

    outs = []
    for v in VARIANTS + ["tcgen05"]:
        C = x0.clone() if c_type == F32 else torch.zeros(M, ldc, device="cuda", dtype=tdtype)
        torch.cuda.synchronize()
        kw = dict(gelu=epi == "fc1", accumulate=c_type == F32)
        if epi.startswith("qkv"):
            kw.update(col_scale=qk, scale_cols=2 * (N // 3) // 8 * 8)
        if c_type == E4M3:
            kw.update(c_scale_ptr=c_scale.data_ptr())
        eng.op_gemm_fp8(v, Aq.data_ptr(), sa.data_ptr(), K, Wq.data_ptr(), sw.data_ptr(), K, bias.data_ptr(), C.data_ptr(),
                        c_type, ldc, M, N, K, **kw)
        eng.sync()
        outs.append(C)
        if c_type == E4M3:
            got = _dec(C) * c_scale.double()[:, None]
            out_ulp = _e4m3_ulp(ref / c_scale.double()[:, None]) * c_scale.double()[:, None]
        else:
            got = C.double()
            out_ulp = ref.abs() * (2.0 ** -8 if c_type == BF16 else 2.0 ** -23)
        excess = (got - ref).abs() - out_ulp
        ratio = float((excess / err_scale.clamp_min(1e-30)).max())
        _WORST[(epi, K)] = max(_WORST.get((epi, K), 0.0), ratio)
        assert ratio <= TAU, (v, ratio)
    assert torch.equal(outs[0], outs[-1])                   # two identical launches: the same bits
    print(json.dumps(dict(epi=epi, M=M, K=K, worst_ratio=_WORST[(epi, K)])))


def test_fp8_gemm_refuses_the_64_wide_kernel(eng):
    from whisperlivekit_b200._lib import WlkError
    A = torch.zeros(128, 128, device="cuda", dtype=torch.uint8)
    s = torch.ones(128, device="cuda")
    C = torch.zeros(128, 128, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(WlkError):
        eng.op_gemm_fp8("tcgen05_1cta", A.data_ptr(), s.data_ptr(), 128, A.data_ptr(), s.data_ptr(), 128, None,
                        C.data_ptr(), BF16, 128, 128, 128, 128)


_FORCED = """
import torch
from whisperlivekit_b200._lib import WlkError
from whisperlivekit_b200.dims import DIMS
from whisperlivekit_b200.engine import WhisperEngine
e = WhisperEngine(DIMS["micro"], None, [(0, 0)], precision="bf16", max_sessions=1, max_batch=1)
A = torch.zeros(128, 128, device="cuda", dtype=torch.uint8)
s = torch.ones(128, device="cuda")
C = torch.zeros(128, 128, device="cuda", dtype=torch.bfloat16)
torch.cuda.synchronize()
try:
    e.op_gemm_fp8("tcgen05", A.data_ptr(), s.data_ptr(), 128, A.data_ptr(), s.data_ptr(), 128, None, C.data_ptr(), 1,
                  128, 128, 128, 128)
    print("ACCEPTED")
except WlkError as err:
    print("REFUSED", err)
e.close()
"""


@pytest.mark.parametrize("variant", ["1", "6"])
def test_forced_64_wide_variant_refuses_e4m3(variant):
    """WLK_GEMM_VARIANT (read once per process: a child process) forcing a 64-wide kernel makes the auto e4m3 GEMM fail
    with a clear error instead of running a kernel that has no e4m3 form"""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, WLK_GEMM_VARIANT=variant, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-c", _FORCED], capture_output=True, text=True, env=env, cwd=root, timeout=300)
    assert "REFUSED" in r.stdout and "no e4m3 kernel" in r.stdout, (r.stdout, r.stderr[-2000:])
