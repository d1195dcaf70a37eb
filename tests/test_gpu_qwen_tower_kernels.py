"""GPU: the Qwen3 audio-tower kernels (csrc/qwen.cu) one at a time through the op-level entry points (wlk_qwen_op_*, and
wlk_qwen_window_attention for the windowed tower's attention), each against a float64 torch reference of the same op on
the same inputs rounded to the activation type (fp32 in fp32 mode, bf16 in bf16 mode).  The whole-tower tests
(test_gpu_qwen.py, test_gpu_qwen_window.py) run d_model 128 with 8 conv channels and bound bf16 at 6e-2 .. 8e-2; these
bound each kernel at its own rounding, at the 0.6B geometry and at the edges production reaches: rings that wrap, left
contexts up to the 511-key limit, conv inputs shorter than a chunk, attention blocks up to the 256-key limit, and the
closed-form positional rows every causal stream uses past 1500 steps.

Every test prints its measured maximum next to its bound.  Measured on an H100 80GB HBM3 (700 W power limit), worst case
over the parameters:
  positions         0 past the table at every width and position up to 2^30 - 1 (bound 2^-22); table rows bit-equal.
                    CPU and CUDA torch disagree on about a third of the closed-form entries, so the reference is
                    evaluated on the device
  conv stem         fp32 0.18 of its bound (stage 1), 0.03 (GEMM stages); bf16 0.50 (the output's rounding)
  qkv scatter       fp32 0.002 of its bound (5.9e-6); bf16 0.46 (the output's rounding)
  causal attention  fp32 1.3e-6 x max|V| (4.4e-6 with the moving maximum; bound 3e-5); bf16 0.50 of 3e-5 max|V| + 1 ulp
  window attention  fp32 1.3e-6 x max|V| (bound 3e-5); bf16 0.29 of 2^-8 max|V| + 1 ulp (3.0e-3 x max|V|)

Mutations each of these catches (applied to a scratch copy):
  - the closed form's frequencies from the fp32 quotient -logf(1e4) / (half - 1), what the engine did before it took the
    reference's fp32 frequencies: test_positions fails at d 896, 1.2e-4 off at step 1500, 2.4e-4 at 4095, 3.9e-3 at
    45000, 6.2e-2 at 2^20 and 2.0 at 2^30 - 1
  - qwen_attention_kernel's window starting at p - left_ctx (one key too many): every test_causal_attention set fails
    (the extra key's ring slot holds NaN)
  - qwin_attn_mma_kernel masking key pairs with k0 + 1 > nk (the zero pad key of an odd block joins the softmax):
    test_window_attention[bf16] fails, 70x its bound
  - qwen_im2col_kernel without its t < len clip (a short window's conv reads steps past the previous stage's length):
    test_conv_stem[windowed] fails in both precisions"""
import dataclasses
import math

import pytest
import torch
import torch.nn.functional as F

from test_gpu_qwen_text_kernels import bf16_ulp
from whisperlivekit_b200._lib import WlkError
from whisperlivekit_b200.qwen_dims import (QWEN_DIMS, QwenTowerDims, QwenWindowDims, sinusoid_table,
                                           synthetic_tower_state_dict)
from whisperlivekit_b200.qwen_engine import QwenTowerEngine, QwenWindowEngine, window_attention

pytestmark = pytest.mark.gpu

DEV = "cuda"
ACT = {"fp32": torch.float32, "bf16": torch.bfloat16}
SENTINEL = -768.0                      # exact in bf16 and fp32, far from any output
Q_STEPS_CAP = 128                      # steps one session contributes to a round; ring = left context + 128


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def tower_dims(d=128, C=8, max_positions=40, left=25, bidir=False, n_layer=2):
    return QwenTowerDims(conv_channels=C, d_model=d, n_head=d // 64, n_layer=n_layer, ffn_dim=256, out_dim=64,
                         max_positions=max_positions, block_frames=0, left_context_steps=left, block_bidirectional=bidir)


def causal_engine(precision, dims, max_batch=1):
    return QwenTowerEngine(dims, None, precision=precision, max_sessions=1, max_batch=max_batch)


def fp32_ulp(y):
    a = y.double().abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 23)


def act_ulp(precision, y):
    return fp32_ulp(y) if precision == "fp32" else bf16_ulp(y)


# ---------------------------------------------------------------------------------------------------------------------
# positional rows

POS_D = [128, 896, 1024, 1280]


def closed_form(d, positions, device):
    """The reference's closed form (causal.py _position_embedding, restated in oracle/qwen_oracle.py _pos) with
    offset = p and length 1 for every p, evaluated by torch on `device`."""
    half = d // 2
    inv = torch.exp(-math.log(10000.0) / float(max(1, half - 1)) * torch.arange(half, device=device, dtype=torch.float32))
    rows = []
    for p in positions:
        scaled = torch.arange(p, p + 1, device=device, dtype=torch.float32)[:, None] * inv[None, :]
        rows.append(torch.cat([scaled.sin(), scaled.cos()], dim=1))
    return torch.cat(rows)


@pytest.mark.parametrize("max_positions", [40, 1500])
@pytest.mark.parametrize("d", POS_D)
def test_positions(d, max_positions):
    """Rows inside the table are the table's rows, bit for bit.  Past it the kernel evaluates sin / cos of
    fp32(p) * inv_freq[j]: with the reference's fp32 frequencies the argument is the same fp32 number the reference forms,
    so the only difference left is sinf / cosf against torch's sin / cos of that argument, each within 2 ulp of the
    exact value (for any argument: the reduction is exact): bound 2^-22 absolute (4 ulp at 1).  A frequency one ulp off
    moves the angle by p * 2^-24 * inv: 1e-4 rad at step 1500 and 60 rad at 2^30 - 1."""
    T = max_positions
    positions = [0, T - 1, T, T + 1, 4095, 45000, 2 ** 20, 2 ** 30 - 1]
    eng = causal_engine("fp32", tower_dims(d, max_positions=T, n_layer=1))
    table = sinusoid_table(T, d)
    eng.load_tensor("positional_embedding.positional_embedding", table)
    out = torch.full((len(positions), d), float("nan"), device=DEV)
    torch.cuda.synchronize()
    eng.op_positions(positions, out.data_ptr())
    eng.close()
    inside = [i for i, p in enumerate(positions) if p < T]
    past = [p for p in positions if p >= T]
    assert torch.equal(out[inside].cpu(), torch.from_numpy(table[[positions[i] for i in inside]])), "table rows differ"
    ref = closed_form(d, past, DEV)
    err = (out[len(inside):].double() - ref.double()).abs().amax(1).tolist()
    cpu = closed_form(d, past, "cpu")
    n_cpu = int((cpu != ref.cpu()).sum())
    tag = f"positions[d={d} table={T}]"
    print(f"{tag}: max |err| = {max(err):.2e} (bound {2.0 ** -22:.2e}); by position "
          + " ".join(f"{p}:{e:.1e}" for p, e in zip(past, err))
          + f"; CPU and CUDA torch disagree on {n_cpu} of {cpu.numel()} entries")
    assert max(err) <= 2.0 ** -22, dict(zip(past, err))


def test_positions_need_only_the_table():
    eng = causal_engine("fp32", tower_dims())
    out = torch.zeros(2, 128, device=DEV)
    with pytest.raises(WlkError, match="positional_embedding"):
        eng.op_positions([0, 1], out.data_ptr())
    eng.load_tensor("positional_embedding.positional_embedding", sinusoid_table(40, 128))
    with pytest.raises(WlkError, match="position"):
        eng.op_positions([0, -1], out.data_ptr())
    with pytest.raises(WlkError, match="position"):
        eng.op_positions([2 ** 30], out.data_ptr())
    eng.op_positions([0, 39], out.data_ptr())
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# conv stem

CONV_TAPS = ("conv2d1.weight", "conv2d1.bias", "conv2d2.weight", "conv2d2.bias", "conv2d3.weight", "conv2d3.bias")
WINDOW_CHUNKS = [(100, 1), (100, 37), (100, 99), (100, 100), (1, 1), (2, 2), (7, 7), (64, 64), (99, 99)]   # (p0, avail)


def conv_len(n):
    return (n - 1) // 2 + 1


def gelu64(z):
    return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))


@pytest.mark.parametrize("C", [8, 480])
@pytest.mark.parametrize("mode", ["causal", "windowed"])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_conv_stem(precision, mode, C):
    """Each stage against float64 F.conv2d (3x3, stride 2, pad 1) + exact-erf GELU applied to the kernel's own output of
    the previous stage (the first to the chunk's mel frames, zero at and past avail, p0 frames long), compared only on the
    steps inside that stage's conv length.  The windowed chunks put NaN in the frames at and past avail: nothing may read
    them.  Bound per element: the output's rounding to act (1 ulp of the reference, half for the rounding and half for
    the fp32 result's own error straddling a boundary), plus the fp32 sum of K products (9 for conv1, 9C = 4320 at C 480
    for the im2col GEMMs) at worst K + 1 roundings of 2^-23 relative (2^-23: tensor cores may truncate) of
    sum |x| |w| + |b|, times GELU's slope (<= 1.13), plus 2^-21 |z| for the fp32 erff and its products (z the
    pre-activation: 1 + erf(z / sqrt 2) cancels for negative z)."""
    act = ACT[precision]
    if mode == "causal":
        dims = tower_dims(C=C)
        eng = causal_engine(precision, dims)
        chunks, T0 = [(8, 8)] * 6, 8
    else:
        dims = QwenWindowDims(conv_channels=C, d_model=128, n_head=2, n_layer=2, ffn_dim=256, out_dim=64, max_positions=40,
                              n_window_infer=200, left_context_frames=400, right_context_frames=64)
        eng = QwenWindowEngine(dims, None, precision=precision, max_sessions=1, max_batch=1)
        chunks, T0 = WINDOW_CHUNKS, 100
    sd = synthetic_tower_state_dict(dataclasses.replace(dims, n_layer=0), seed=C)
    for name in CONV_TAPS:
        eng.load_tensor(name, sd[name])
    n, M = len(chunks), dims.n_mels
    g = gen(C + T0)
    mel = torch.randn(n, T0, M, device=DEV, generator=g) * 0.8
    for k, (p0, avail) in enumerate(chunks):
        mel[k, avail:] = float("nan")
    T1 = T0 // 2
    T2 = conv_len(T1)
    T3 = conv_len(T2)
    a1 = torch.full((n, M // 2, T1, C), float("nan"), dtype=act, device=DEV)
    a2 = torch.full((n, M // 4, T2, C), float("nan"), dtype=act, device=DEV)
    a3 = torch.full((n, T3, M // 8, C), float("nan"), dtype=act, device=DEV)
    torch.cuda.synchronize()
    eng.op_conv_stem(mel.data_ptr(), [a for _, a in chunks], [p for p, _ in chunks], a1.data_ptr(), a2.data_ptr(),
                     a3.data_ptr())
    eng.close()
    W = {k: torch.from_numpy(sd[k]).to(DEV).double() for k in CONV_TAPS}
    w2 = W["conv2d2.weight"].to(act).double()           # the engine keeps the GEMM weights in act
    w3 = W["conv2d3.weight"].to(act).double()
    got1 = a1.permute(0, 3, 1, 2).double()              # [n][C][F][T]
    got2 = a2.permute(0, 3, 1, 2).double()
    got3 = a3.permute(0, 3, 2, 1).double()
    worst = {1: 0.0, 2: 0.0, 3: 0.0}
    errs = {1: 0.0, 2: 0.0, 3: 0.0}
    for k, (p0, avail) in enumerate(chunks):
        x = mel[k, :p0].double().clone()
        x[avail:] = 0.0
        inp = x.t()[None, None]                         # [1][1][n_mels][p0]
        L1 = conv_len(p0)
        L2 = conv_len(L1)
        L3 = conv_len(L2)
        stages = [(1, inp, W["conv2d1.weight"], W["conv2d1.bias"], got1[k:k + 1, :, :, :L1], 9),
                  (2, got1[k:k + 1, :, :, :L1], w2, W["conv2d2.bias"], got2[k:k + 1, :, :, :L2], 9 * C),
                  (3, got2[k:k + 1, :, :, :L2], w3, W["conv2d3.bias"], got3[k:k + 1, :, :, :L3], 9 * C)]
        for s, src, w, b, got, K in stages:
            assert torch.isfinite(src).all(), f"stage {s} input of chunk {k} (p0 {p0}, avail {avail}) is not finite"
            z = F.conv2d(src, w, b, stride=2, padding=1)
            ref = gelu64(z)
            mag = F.conv2d(src.abs(), w.abs(), b.abs(), stride=2, padding=1)
            allowed = act_ulp(precision, ref) + 1.13 * (K + 1) * 2.0 ** -23 * mag + 2.0 ** -21 * z.abs()
            assert got.shape == ref.shape, (s, got.shape, ref.shape)
            err = (got - ref).abs()
            ratio = float((err / allowed).max()) if torch.isfinite(err).all() else float("inf")
            worst[s] = max(worst[s], ratio)
            errs[s] = max(errs[s], float(err.max()))
    tag = f"conv_stem[{precision} {mode} C={C}]"
    print(f"{tag}: " + ", ".join(f"stage {s} max |err| {errs[s]:.2e} = {worst[s]:.3f} of its bound" for s in (1, 2, 3)))
    assert max(worst.values()) <= 1.0, (tag, worst)


def test_conv_stem_rejects_what_it_cannot_hold():
    dims = QwenWindowDims(conv_channels=8, d_model=128, n_head=2, n_layer=1, ffn_dim=256, out_dim=64, max_positions=40,
                          n_window_infer=200, left_context_frames=400, right_context_frames=64)
    eng = QwenWindowEngine(dims, None, precision="fp32", max_sessions=1, max_batch=1)
    n = 33
    mel = torch.zeros(n, 100, 128, device=DEV)
    a = torch.zeros(n * 64 * 50 * 8, device=DEV)
    args = (a.data_ptr(), a.data_ptr(), a.data_ptr())
    with pytest.raises(WlkError, match="not loaded"):
        eng.op_conv_stem(mel.data_ptr(), [100], [100], *args)
    sd = synthetic_tower_state_dict(dataclasses.replace(dims, n_layer=0), seed=1)
    for name in CONV_TAPS:
        eng.load_tensor(name, sd[name])
    with pytest.raises(WlkError, match="workspace"):
        eng.op_conv_stem(mel.data_ptr(), [100] * n, [100] * n, *args)
    for avail, p0 in ((0, 100), (64, 63), (100, 101)):
        with pytest.raises(WlkError, match="avail"):
            eng.op_conv_stem(mel.data_ptr(), [avail], [p0], *args)
    eng.op_conv_stem(mel.data_ptr(), [100] * 32, [100] * 32, *args)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# causal QKV projection with the K/V ring scatter

@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_qkv_scatter(precision):
    """The 0.6B geometry (d 896, 14 heads, left context 150: rings of 278 slots) over rows of three sessions at positions
    that wrap the ring (0, ring - 1, ring, 1000, 2^30 - 130 ...).  Values: float64 xn W^T + b on the act-rounded xn and W,
    the q columns times 0.125.  Bound: the fp32 sum of d = 896 products, at worst 898 roundings of 2^-23 relative (tensor
    cores may truncate) of sum |xn| |W| + |b|, plus the output's rounding to act (1 ulp).  Placement: the rings are
    prefilled with a sentinel and exactly the rows' (layer, K / V, head, slot) entries change."""
    act = ACT[precision]
    dims = dataclasses.replace(QWEN_DIMS["qwen3-asr-0.6b"], n_layer=2)
    d, H, layer, n_slots = dims.d_model, dims.n_head, 1, 3
    ring = dims.left_context_steps + Q_STEPS_CAP
    eng = causal_engine(precision, dims)
    g = gen(896)
    Wq = torch.randn(3 * d, d, device=DEV, generator=g) * (1.6 / math.sqrt(d))
    bq = torch.randn(3 * d, device=DEV, generator=g) * 0.02
    p = f"layers.{layer}.self_attn."
    for i, part in enumerate(("q_proj", "k_proj", "v_proj")):
        eng.load_tensor(p + part + ".weight", Wq[i * d:(i + 1) * d].cpu().numpy())
        eng.load_tensor(p + part + ".bias", bq[i * d:(i + 1) * d].cpu().numpy())
    positions = [0, ring - 1, ring, 1000, 2 ** 30 - 130, 1, 555, ring + 1, 2 ** 30 - 131, 277 * 3]
    slot = [r % n_slots for r in range(len(positions))]
    keys = [(s, p_ % ring) for s, p_ in zip(slot, positions)]
    assert len(set(keys)) == len(keys), "two rows of one session on one ring slot"
    R = len(positions)
    xn = torch.randn(R, d, device=DEV, generator=g).to(act)
    rings = [torch.full((dims.n_layer, 2, H, ring, 64), SENTINEL, dtype=act, device=DEV) for _ in range(n_slots)]
    q_out = torch.full((R, d), float("nan"), dtype=act, device=DEV)
    torch.cuda.synchronize()
    eng.op_qkv(layer, xn.data_ptr(), slot, positions, [r.data_ptr() for r in rings], q_out.data_ptr())
    eng.close()
    for s in range(n_slots):
        want = torch.zeros(dims.n_layer, 2, H, ring, dtype=torch.bool, device=DEV)
        for r in range(R):
            if slot[r] == s:
                want[layer, :, :, positions[r] % ring] = True
        changed = (rings[s] != SENTINEL).any(-1)
        assert torch.equal(changed, want), f"session {s}: K/V written outside the rows' ring slots"
    x, w = xn.double(), Wq.to(act).double()
    ref = x @ w.t() + bq.double()
    ref[:, :d] *= 0.125
    mag = x.abs() @ w.abs().t() + bq.double().abs()
    mag[:, :d] *= 0.125
    got = torch.empty(R, 3 * d, dtype=torch.float64, device=DEV)
    got[:, :d] = q_out.double()
    for r in range(R):
        got[r, d:2 * d] = rings[slot[r]][layer, 0, :, positions[r] % ring].reshape(d).double()
        got[r, 2 * d:] = rings[slot[r]][layer, 1, :, positions[r] % ring].reshape(d).double()
    allowed = act_ulp(precision, ref) + (d + 2) * 2.0 ** -23 * mag
    err = (got - ref).abs()
    ratio = float((err / allowed).max())
    print(f"qkv[{precision}]: max |err| = {float(err.max()):.2e} (q {float(err[:, :d].max()):.1e}, k "
          f"{float(err[:, d:2 * d].max()):.1e}, v {float(err[:, 2 * d:].max()):.1e}), {ratio:.3f} of the bound")
    assert ratio <= 1.0, ratio


# ---------------------------------------------------------------------------------------------------------------------
# causal attention over the K/V ring

ATTN_L, ATTN_LAYER = 2, 1
ATTN_STEPS = [1, 24, 128]


class Round:
    """One round of jobs.  Job j holds n_steps[j] rows at positions starts[j] ..; its ring has random K / V at the slots
    of every position some row may see ([start - left + 1, start + n - 1], clipped at 0) in the tested layer, and NaN
    in every other slot and in the other layer: a key outside every query's window must never be read."""

    def __init__(self, act, H, left, starts, n_steps, g, k_fn=None):
        self.ring = left + Q_STEPS_CAP
        self.left, self.H = left, H
        self.jobs, self.rings = [], []
        row = 0
        for j, (p0, n) in enumerate(zip(starts, n_steps)):
            k0 = max(0, p0 - left + 1)
            kpos = torch.arange(k0, p0 + n, device=DEV)
            slots = kpos % self.ring
            k = torch.randn(H, len(kpos), 64, device=DEV, generator=g)
            v = torch.rand(H, len(kpos), 64, device=DEV, generator=g) * 2 - 1
            if k_fn is not None:
                k = k_fn(kpos, k)
            rg = torch.full((ATTN_L, 2, H, self.ring, 64), float("nan"), dtype=act, device=DEV)
            rg[ATTN_LAYER, 0][:, slots] = k.to(act)
            rg[ATTN_LAYER, 1][:, slots] = v.to(act)
            self.rings.append(rg)
            self.jobs.append((row, n, p0, kpos, slots))
            row += n
        self.rows = row
        self.starts, self.n_steps = list(starts), list(n_steps)

    def run(self, eng, q):
        out = torch.full((self.rows, self.H * 64), float("nan"), dtype=q.dtype, device=DEV)
        torch.cuda.synchronize()
        eng.op_attention(ATTN_LAYER, q.data_ptr(), self.starts, self.n_steps, [r.data_ptr() for r in self.rings],
                         out.data_ptr())
        return out

    def reference(self, q, bidir):
        """float64 softmax(q k^T) v (q arrives pre-scaled) over keys [p - left + 1, p] (causal) or
        [p - left + 1, last row of the job] (block-bidirectional), clipped at 0 (reference causal.py:330-346)."""
        out = torch.empty(self.rows, self.H * 64, dtype=torch.float64, device=DEV)
        for (row, n, p0, kpos, slots), rg in zip(self.jobs, self.rings):
            k = rg[ATTN_LAYER, 0][:, slots].double()
            v = rg[ATTN_LAYER, 1][:, slots].double()
            qp = p0 + torch.arange(n, device=DEV)
            hi = torch.full_like(qp, p0 + n - 1) if bidir else qp
            allowed = (kpos[None, :] >= qp[:, None] - self.left + 1) & (kpos[None, :] <= hi[:, None])
            qs = q[row:row + n].double().view(n, self.H, 64).transpose(0, 1)
            sc = (qs @ k.transpose(1, 2)).masked_fill(~allowed[None], -math.inf)
            out[row:row + n] = (torch.softmax(sc, -1) @ v).transpose(0, 1).reshape(n, self.H * 64)
        return out

    def max_v(self):
        return max(float(rg[ATTN_LAYER, 1][:, s].float().abs().max()) for (_, _, _, _, s), rg in zip(self.jobs, self.rings))


def check_fp32_softmax(precision, got, ref, max_v, tag):
    """fp32 softmax on fp32 or bf16 operands (SIMT, one warp per query): 3e-5 x max|V|.  The largest rounding term is the
    sequential P V sum of a lane over up to 511 keys (511 roundings of 2^-24: 3e-5 relative if every one went the same
    way, a few 1e-7 in practice); the 64-term score dots and expf add a few 1e-7 at the scores used here.  bf16 adds the
    output's rounding: one ulp of the reference."""
    assert torch.isfinite(got.float()).all(), f"{tag}: non-finite outputs (a key outside the window was read)"
    err = (got.double() - ref).abs()
    allowed = 3e-5 * max_v + (bf16_ulp(ref) if precision == "bf16" else 0.0)
    ratio = float((err / allowed).max())
    print(f"{tag}: max |err| = {float(err.max()):.3e} = {float(err.max()) / max_v:.2e} x max|V|, {ratio:.3f} of the bound")
    assert ratio <= 1.0, (tag, ratio)


@pytest.mark.parametrize("bidir", [False, True])
@pytest.mark.parametrize("left", [1, 25, 150, 384])
@pytest.mark.parametrize("H", [2, 14])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_causal_attention(precision, H, left, bidir):
    """Five jobs in one round at starts 0, left - 1 (the first row whose window reaches position 0), ring - 3 (the
    job's rows wrap the ring), 1000 and 2^30 - 200, with 1, 24 and 128 steps rotating over them.  left 384 is the
    limit: 384 + 127 = 511 keys for the last query of a bidirectional 128-step job."""
    act = ACT[precision]
    eng = causal_engine(precision, tower_dims(64 * H, left=left, bidir=bidir, n_layer=ATTN_L))
    ring = left + Q_STEPS_CAP
    starts = [0, left - 1, ring - 3, 1000, 2 ** 30 - 200]
    i = [1, 25, 150, 384].index(left) + (3 if bidir else 0)
    n_steps = [ATTN_STEPS[(j + i) % 3] for j in range(len(starts))]
    g = gen(1000 * H + left + int(bidir))
    rd = Round(act, H, left, starts, n_steps, g)
    q = (torch.randn(rd.rows, H * 64, device=DEV, generator=g) * 0.25).to(act)
    got = rd.run(eng, q)
    eng.close()
    check_fp32_softmax(precision, got, rd.reference(q, bidir), rd.max_v(),
                       f"causal attention[{precision} H={H} left={left} {'bidir' if bidir else 'causal'} steps={n_steps}]")


@pytest.mark.parametrize("bidir", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_causal_attention_moving_maximum(precision, bidir):
    """Key norms grow with position (up to 4x over a query's 511 keys) and fall in one head, so the maximum score sits at
    the newest keys for most rows and at the oldest for that head's rows: the softmax's maximum is far from its first
    keys."""
    act = ACT[precision]
    H, left = 14, 384
    eng = causal_engine(precision, tower_dims(64 * H, left=left, bidir=bidir, n_layer=ATTN_L))
    g = gen(511)

    def k_fn(kpos, k):
        ramp = 1.0 + 3.0 * (kpos - kpos[0]).float() / max(1, int(kpos[-1] - kpos[0]))
        k = k * ramp[None, :, None]
        k[5] = k[5] / ramp[:, None] ** 2
        return k

    rd = Round(act, H, left, [3000, 2 ** 30 - 200], [128, 128], g, k_fn)
    q = (torch.randn(rd.rows, H * 64, device=DEV, generator=g) * 0.2).to(act)
    got = rd.run(eng, q)
    eng.close()
    row, n, p0, kpos, slots = rd.jobs[0]
    k = rd.rings[0][ATTN_LAYER, 0][:, slots].float()
    sc = q[row:row + n].float().view(n, H, 64).transpose(0, 1) @ k.transpose(1, 2)
    jump = (sc[..., -64:].amax(-1) - sc[..., :64].amax(-1)).abs() * 1.4427
    assert (jump > 4).float().mean().item() > 0.5, jump
    check_fp32_softmax(precision, got, rd.reference(q, bidir), rd.max_v(),
                       f"causal attention moving maximum[{precision} {'bidir' if bidir else 'causal'}]")


def test_causal_attention_rejects_what_the_kernel_assumes_away():
    eng = causal_engine("fp32", tower_dims(left=25, n_layer=ATTN_L))
    rg = torch.zeros(ATTN_L, 2, 2, 25 + Q_STEPS_CAP, 64, device=DEV)
    q = torch.zeros(2 * Q_STEPS_CAP, 128, device=DEV)
    out = torch.zeros_like(q)

    def call(starts, n_steps, layer=ATTN_LAYER):
        eng.op_attention(layer, q.data_ptr(), starts, n_steps, [rg.data_ptr()] * len(starts), out.data_ptr())

    call([0, 2 ** 30 - 129], [128, 128])                       # accepted
    for starts, n_steps in (([0], [0]), ([0], [129]), ([5, 0], [24, -1])):
        with pytest.raises(WlkError, match="n_steps"):
            call(starts, n_steps)
    with pytest.raises(WlkError, match="negative start"):
        call([-1], [1])
    with pytest.raises(WlkError, match="overflow"):
        call([2 ** 30 - 128], [128])
    with pytest.raises(WlkError, match="jobs"):
        call([], [])
    for layer in (-1, ATTN_L):
        with pytest.raises(WlkError, match="layer"):
            call([0], [1], layer=layer)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# windowed tower: block-diagonal attention

BLOCK_LENS = [1, 15, 16, 17, 63, 64, 65, 129, 241, 255, 256]
EXTRA_ROWS = 7                         # rows past the streams: never written


def window_reference(qkv, rows, d):
    """float64 softmax(q k^T) v within each stream (one block per stream), on the act-rounded inputs."""
    x = qkv.double()
    out = torch.empty(sum(rows), d, dtype=torch.float64, device=DEV)
    r0 = 0
    for n in rows:
        blk = x[r0:r0 + n].view(n, 3, d // 64, 64).permute(1, 2, 0, 3)      # [q|k|v][head][row][64]
        out[r0:r0 + n] = (torch.softmax(blk[0] @ blk[1].transpose(1, 2), -1) @ blk[2]).transpose(0, 1).reshape(n, d)
        r0 += n
    return out


def run_window(qkv, rows):
    d = qkv.shape[1] // 3
    out = torch.full((qkv.shape[0], d), float("nan"), dtype=qkv.dtype, device=DEV)
    window_attention(qkv, rows, 0, out=out)
    total = sum(rows)
    assert torch.isnan(out[total:].float()).all(), "rows past the streams were written"
    return out[:total]


def check_window(precision, got, ref, max_v, tag):
    """fp32 (SIMT, fp32 softmax over <= 256 keys): 3e-5 x max|V| as for the causal kernel, with half its keys.  bf16
    (mma.sync, fp32 online softmax): P is rounded to bf16 for the P V product (2^-9 relative per entry, at most
    2^-9 max|V| on the output) while l sums the unrounded P (another 2^-9 max|V|), so 2^-8 max|V|, plus the output's own
    rounding to bf16 (one ulp of the reference)."""
    assert torch.isfinite(got.float()).all(), f"{tag}: non-finite outputs"
    err = (got.double() - ref).abs()
    allowed = 3e-5 * max_v if precision == "fp32" else 2.0 ** -8 * max_v + bf16_ulp(ref)
    ratio = float((err / allowed).max())
    print(f"{tag}: max |err| = {float(err.max()):.3e} = {float(err.max()) / max_v:.2e} x max|V|, {ratio:.3f} of the bound")
    assert ratio <= 1.0, (tag, ratio)


@pytest.mark.parametrize("d", [256, 896])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_window_attention(precision, d):
    """One stream per block length: 1, 15 / 16 / 17 (a 16-key MMA step and one past it), 63 / 64 / 65 (a 64-key tile),
    129, 241, 255 and 256 (the limit), in one launch; NaN-prefilled output rows past the streams stay NaN."""
    act = ACT[precision]
    g = gen(d + 7)
    R = sum(BLOCK_LENS) + EXTRA_ROWS
    qkv = torch.randn(R, 3 * d, device=DEV, generator=g) * 1.5
    qkv[:, :d] *= 0.125
    qkv = qkv.to(act)
    got = run_window(qkv, BLOCK_LENS)
    max_v = float(qkv[:sum(BLOCK_LENS), 2 * d:].float().abs().max())
    check_window(precision, got, window_reference(qkv[:sum(BLOCK_LENS)], BLOCK_LENS, d), max_v,
                 f"window attention[{precision} d={d}]")


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_window_attention_moving_maximum(precision):
    """Key norms step up with every 64-key tile (up to 5x at the fourth) and fall in one head, so the online softmax's
    running maximum rises at every tile edge for most rows; blocks of 256, 255, 129 and 65 rows."""
    act = ACT[precision]
    d, rows = 896, [256, 255, 129, 65]
    g = gen(64)
    R = sum(rows) + EXTRA_ROWS
    qkv = torch.randn(R, 3 * d, device=DEV, generator=g)
    qkv[:, :d] *= 0.125
    r0 = 0
    for n in rows:
        ramp = 1.0 + 4.0 * (torch.arange(n, device=DEV) // 64).float() / 3.0
        k = qkv[r0:r0 + n, d:2 * d].view(n, d // 64, 64)
        k *= ramp[:, None, None]
        k[:, 3] /= ramp[:, None] ** 2
        r0 += n
    qkv = qkv.to(act)
    got = run_window(qkv, rows)
    q = qkv[:256, :d].float().view(256, d // 64, 64).transpose(0, 1)
    k = qkv[:256, d:2 * d].float().view(256, d // 64, 64).transpose(0, 1)
    sc = q @ k.transpose(1, 2)
    jump = (sc[..., -64:].amax(-1) - sc[..., :64].amax(-1)).abs() * 1.4427
    assert (jump > 4).float().mean().item() > 0.5, jump
    max_v = float(qkv[:sum(rows), 2 * d:].float().abs().max())
    check_window(precision, got, window_reference(qkv[:sum(rows)], rows, d), max_v, f"window moving maximum[{precision}]")


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_window_attention_rejects_a_257_row_block(precision):
    qkv = torch.zeros(300, 3 * 128, dtype=ACT[precision], device=DEV)
    with pytest.raises(WlkError, match="exceeds 256"):
        window_attention(qkv, [257], 0)
    with pytest.raises(WlkError, match="exceeds 256"):
        window_attention(qkv, [300], 257)
    window_attention(qkv, [300], 256)
