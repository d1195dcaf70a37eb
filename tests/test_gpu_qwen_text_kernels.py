"""GPU: the Qwen3 text-decoder kernels (csrc/qwen_text.cu) one at a time through the op-level entry points
(wlk_qtext_op_*), each against a float64 torch reference of the same op on the same inputs rounded to the activation
type (fp32 in fp32 mode, bf16 in bf16 mode).  The whole-forward tests (test_gpu_qwen_text.py) bound bf16 logits at
8e-2 .. 5.7e-1, wide enough to hide an attention mask off by one key or a RoPE angle off by 1e-3 rad; these bound each
kernel at its own rounding.

Every test prints its measured maximum next to its bound.  Measured on an H100 80GB HBM3 (700 W power limit), worst case
over the parameters:
  qk_rope    fp32 1.6e-7 x |out|max (bound 2e-6); bf16 1 ulp (bound 1 ulp)
  attention  fp32 1.9e-6 x max|V| (4.9e-6 with the moving maximum; bound 3e-5);
             bf16 0.38 of its bound 2^-8 max|V| + 1 ulp (2.9e-3 at max|V| = 1)
  magnet     rows at or past the magnet exactly 8, rows before it within [-1, 1], both precisions
  rmsnorm    fp32 1.8e-7 x |ref| (bound 2e-6); bf16 1 ulp (bound 1 ulp)
  swiglu     fp32 2.1e-7 x |ref| (bound 5e-7); bf16 0 ulp (bound 1 ulp)
With the RoPE frequencies rounded once from a double-precision pow (what the engine did before it took HF's fp32
values), test_qk_rope fails in every parameter set: fp32 q off by 2.6e-5 x |out|max at position 1100 and 1.2e-3 at
32767 (theta 1e6), bf16 by up to 154 ulp.  With the bf16 kernel's causal mask one key short, test_attention_magnet_keys
fails."""
import math

import numpy as np
import pytest
import torch

from whisperlivekit_b200._lib import WlkError
from whisperlivekit_b200.qwen_dims import QwenTextDims, rope_inv_freq
from whisperlivekit_b200.qwen_text_engine import QwenTextEngine

pytestmark = pytest.mark.gpu

DEV = "cuda"
ACT = {"fp32": torch.float32, "bf16": torch.bfloat16}
MAX_CTX = 32768
HD = 128
EPS = float(np.float32(1e-6))          # the engine's rms_eps, as the kernels see it
SCALE = HD ** -0.5


def make_engine(precision, H=16, KV=8, L=3, d=256, F=512, theta=1e6, max_ctx=MAX_CTX):
    dims = QwenTextDims(vocab=256, d_model=d, n_layer=L, n_head=H, n_kv_head=KV, ffn_dim=F, rope_theta=theta,
                        rms_eps=1e-6, tied=False, max_ctx=max_ctx)
    return QwenTextEngine(dims, None, precision=precision, max_sessions=1, max_batch=1)


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def bf16_ulp(y):
    """Spacing of bf16 numbers at |y| (8 significant bits); subnormal spacing below 2^-126."""
    a = y.double().abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def within_one_bf16_ulp(got, ref, what):
    """bf16 output of an fp32 computation: the kernel rounds its fp32 value once, so it may sit one ulp from the
    correctly rounded float64 reference when its few-ulp fp32 error straddles a rounding boundary, never further."""
    want = ref.to(torch.bfloat16).double()
    err = (got.double() - want).abs()
    ulps = float((err / bf16_ulp(want)).max())
    print(f"{what}: max {ulps:.2f} bf16 ulp (bound 1)")
    assert ulps <= 1.0, (what, ulps)


# ---------------------------------------------------------------------------------------------------------------------
# q/k RMSNorm + RoPE + K/V scatter

ROPE_POS = [0, 1, 63, 64, 1023, 1100, 4095, 8191, 32767]
SENTINEL = -768.0                      # exact in bf16 and fp32, far from any output


def rope_reference(qkv, qn, kn, pos, H, KV, theta):
    """HF Qwen3: per-head RMSNorm, angle = fp32(pos) * inv_freq rounded to fp32 (the fp32 [64, 1] @ [1, T] matmul of
    Qwen3RotaryEmbedding has one product per entry), then cos / sin and rotate_half in float64."""
    R = qkv.shape[0]
    inv = torch.as_tensor(rope_inv_freq(theta, HD), device=DEV)
    ang = (torch.as_tensor(pos, dtype=torch.float32, device=DEV)[:, None] * inv[None, :]).double()
    cos = torch.cat([ang.cos(), ang.cos()], -1)[:, None]
    sin = torch.cat([ang.sin(), ang.sin()], -1)[:, None]
    x = qkv.double().view(R, H + 2 * KV, HD)

    def rms(v, w):
        return w.double() * (v / torch.sqrt(v.pow(2).mean(-1, keepdim=True) + EPS))

    def rot(v):
        return torch.cat([-v[..., HD // 2:], v[..., :HD // 2]], -1)

    q, k = rms(x[:, :H], qn), rms(x[:, H:H + KV], kn)
    return q * cos + rot(q) * sin, k * cos + rot(k) * sin, x[:, H + KV:]


@pytest.mark.parametrize("H,KV", [(16, 8), (8, 2), (8, 1)])
@pytest.mark.parametrize("theta", [1e6, 1e4])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_qk_rope(precision, theta, H, KV):
    """Bound: fp32 |out - ref| <= 2e-6 x |out|max per tensor.  The kernel's path to an output is a 128-term fp32 sum of
    squares (<= 8 roundings: 5 shuffle levels + 4 warps), rsqrtf (2 ulp), three products, cosf / sinf (2 ulp) and the
    rotation's two roundings: about 1.5e-6 relative at worst, typically a few 1e-7.  An inv_freq entry one ulp off moves
    the angle by 6e-5 rad at position 1100 and 2e-3 rad at 32767, 30x to 1000x that bound.  bf16: one ulp of the rounded
    reference.  V is copied as is (bit-exact), and only (layer, kv head, position) of each row's slot changes."""
    L, layer, n_slots = 3, 2, 2
    act = ACT[precision]
    eng = make_engine(precision, H, KV, L=L, theta=theta)
    g = gen(100 * H + KV + int(theta))
    R = len(ROPE_POS)
    W = (H + 2 * KV) * HD
    qkv = torch.randn(R, W, device=DEV, generator=g) * 3.0
    qn = 1.0 + 0.3 * torch.randn(HD, device=DEV, generator=g)
    kn = 1.0 + 0.3 * torch.randn(HD, device=DEV, generator=g)
    slot = [r % n_slots for r in range(R)]                   # alternate slots: rows need not be packed here
    caches = [torch.full((L, 2, KV, MAX_CTX, HD), SENTINEL, dtype=act, device=DEV) for _ in range(n_slots)]
    qout = torch.full((R, H * HD), float("nan"), dtype=act, device=DEV)
    torch.cuda.synchronize()
    eng.op_qk_rope(qkv.data_ptr(), qn.data_ptr(), kn.data_ptr(), ROPE_POS, slot, [c.data_ptr() for c in caches], layer,
                   qout.data_ptr())
    q_ref, k_ref, v_ref = rope_reference(qkv, qn, kn, ROPE_POS, H, KV, theta)
    # placement: exactly the rows' (layer, head, position) entries changed, in every slot
    for s in range(n_slots):
        want = torch.zeros(L, 2, KV, MAX_CTX, dtype=torch.bool, device=DEV)
        for r in range(R):
            if slot[r] == s:
                want[layer, :, :, ROPE_POS[r]] = True
        changed = (caches[s] != SENTINEL).any(-1)
        assert torch.equal(changed, want), f"slot {s}: K/V written outside the rows' cache entries"
    k_got = torch.stack([caches[slot[r]][layer, 0, :, ROPE_POS[r]] for r in range(R)])
    v_got = torch.stack([caches[slot[r]][layer, 1, :, ROPE_POS[r]] for r in range(R)])
    assert torch.equal(v_got, qkv.view(R, H + 2 * KV, HD)[:, H + KV:].to(act)), "V must be stored unnormalised, unrotated"
    q_got = qout.view(R, H, HD)
    tag = f"qk_rope[{precision} theta={theta:g} H={H} KV={KV}]"
    if precision == "fp32":
        for name, got, ref in (("q", q_got, q_ref), ("k", k_got, k_ref)):
            scale = float(ref.abs().max())
            per_pos = ((got.double() - ref).abs().amax(dim=(1, 2)) / scale).tolist()
            worst = max(per_pos)
            print(f"{tag} {name}: max |err| / |out|max = {worst:.2e} (bound 2e-6); by position "
                  + " ".join(f"{p}:{e:.1e}" for p, e in zip(ROPE_POS, per_pos)))
            assert worst <= 2e-6, (name, dict(zip(ROPE_POS, per_pos)))
    else:
        within_one_bf16_ulp(q_got, q_ref, f"{tag} q")
        within_one_bf16_ulp(k_got, k_ref, f"{tag} k")
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# causal GQA attention over the cache

ATTN_SHAPES = [(4, 4), (16, 8), (8, 2), (8, 1), (32, 4)]      # G = 1, 2, 4, 8 and 8 at KV = 4
ROW_COUNTS = [1, 15, 16, 17, 33, 40]
STARTS = [0, 1, 47, 63, 64, 1000, None]                         # None: max_ctx - rows (the last row at 32767)
ATTN_L, ATTN_LAYER = 2, 1


class Batch:
    """Sessions packed as a forward packs them: session j holds rows[j] rows at positions starts[j] ..; its cache has
    random K / V at every position up to its last row and NaN at every position past it (and in the other layer), the
    contract being that keys past a row's own position are neither read nor multiplied."""

    def __init__(self, act, KV, rows, starts, g, k_fn=None, v_fn=None):
        self.sessions, self.pos, self.slot, self.caches = [], [], [], []
        row0 = 0
        for s, (n, p0) in enumerate(zip(rows, starts)):
            T = p0 + n
            c = torch.full((ATTN_L, 2, KV, MAX_CTX, HD), float("nan"), dtype=act, device=DEV)
            k = torch.randn(KV, T, HD, device=DEV, generator=g)
            v = torch.rand(KV, T, HD, device=DEV, generator=g) * 2 - 1
            if k_fn is not None:
                k = k_fn(s, k)
            if v_fn is not None:
                v = v_fn(s, v)
            c[ATTN_LAYER, 0, :, :T] = k.to(act)
            c[ATTN_LAYER, 1, :, :T] = v.to(act)
            self.caches.append(c)
            self.sessions.append((row0, n, p0, s))
            self.pos += list(range(p0, T))
            self.slot += [s] * n
            row0 += n
        self.rows = row0

    def run(self, eng, q, H):
        out = torch.full((self.rows, H * HD), float("nan"), dtype=q.dtype, device=DEV)
        torch.cuda.synchronize()
        eng.op_attention(q.data_ptr(), self.pos, self.slot, [c.data_ptr() for c in self.caches], ATTN_LAYER, out.data_ptr())
        return out

    def reference(self, q, H, KV):
        """float64 softmax(q k^T / sqrt(128)) v over positions 0 .. pos, KV heads repeated like HF repeat_kv."""
        out = torch.empty(self.rows, H * HD, dtype=torch.float64, device=DEV)
        G = H // KV
        for row0, n, p0, s in self.sessions:
            T = p0 + n
            k = self.caches[s][ATTN_LAYER, 0, :, :T].double().repeat_interleave(G, dim=0)
            v = self.caches[s][ATTN_LAYER, 1, :, :T].double().repeat_interleave(G, dim=0)
            qs = q[row0:row0 + n].double().view(n, H, HD).transpose(0, 1)
            sc = (qs @ k.transpose(1, 2)) * SCALE
            mask = torch.arange(T, device=DEV)[None, :] > (p0 + torch.arange(n, device=DEV))[:, None]
            p = torch.softmax(sc.masked_fill(mask, -math.inf), dim=-1)
            out[row0:row0 + n] = (p @ v).transpose(0, 1).reshape(n, H * HD)
        return out

    def max_v(self):
        return max(float(c[ATTN_LAYER, 1, :, :p0 + n].float().abs().max()) for (_, n, p0, _), c in zip(self.sessions, self.caches))


def check_attention(precision, got, ref, max_v, tag):
    """fp32 (SIMT, fp32 online softmax): 3e-5 x max|V| -- the sums run over up to 32768 keys in fp32, a few 1e-7
    relative per key tile, far below.  bf16 (mma.sync): P is rounded to bf16 for the P V product (2^-9 relative per entry,
    at most 2^-9 max|V| on the output) while l sums the unrounded P (another 2^-9 max|V| of normalisation mismatch), so
    2^-8 max|V|, plus the output's own rounding to bf16 (one ulp of the reference)."""
    assert torch.isfinite(got.float()).all(), f"{tag}: non-finite outputs (a key past a row's position was read)"
    err = (got.double() - ref).abs()
    if precision == "fp32":
        bound = 3e-5 * max_v
        worst = float(err.max())
        print(f"{tag}: max |err| = {worst:.3e} = {worst / max_v:.2e} x max|V| (bound 3e-5 x max|V| = {bound:.3e})")
        assert worst <= bound, (tag, worst, bound)
    else:
        allowed = 2.0 ** -8 * max_v + bf16_ulp(ref)
        ratio = float((err / allowed).max())
        print(f"{tag}: max |err| = {float(err.max()):.3e}, {ratio:.2f} of the bound 2^-8 max|V| + 1 ulp")
        assert ratio <= 1.0, (tag, ratio)


@pytest.mark.parametrize("H,KV", ATTN_SHAPES)
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_attention(precision, H, KV):
    """Seven sessions in one batch, row counts 1 .. 40 (tiles of 1, 15 and 16 rows, 17 = 16 + 1) paired with start
    positions 0, 1, 47, 63, 64 (a tile that starts on / just before a 64-key block edge), 1000 and max_ctx - rows; the
    pairing rotates with the shape so each count meets several starts."""
    act = ACT[precision]
    eng = make_engine(precision, H, KV, L=ATTN_L)
    i = ATTN_SHAPES.index((H, KV))
    g = gen(7 * H + KV)
    rows = [ROW_COUNTS[(j + i) % len(ROW_COUNTS)] for j in range(len(STARTS))]
    starts = [MAX_CTX - n if p is None else p for n, p in zip(rows, STARTS)]
    b = Batch(act, KV, rows, starts, g)
    q = (torch.randn(b.rows, H * HD, device=DEV, generator=g) * 1.5).to(act)
    got = b.run(eng, q, H)
    check_attention(precision, got, b.reference(q, H, KV), b.max_v(), f"attention[{precision} H={H} KV={KV}]")
    eng.close()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_attention_1024_rows(precision):
    """A full 1024-row round: one session of 1000 rows starting mid-block (position 7, 63 tiles) and one of 24 ending
    at max_ctx - 1."""
    H, KV = 16, 8
    act = ACT[precision]
    eng = make_engine(precision, H, KV, L=ATTN_L)
    g = gen(1024)
    b = Batch(act, KV, [1000, 24], [7, MAX_CTX - 24], g)
    assert b.rows == 1024
    q = (torch.randn(b.rows, H * HD, device=DEV, generator=g) * 1.5).to(act)
    got = b.run(eng, q, H)
    check_attention(precision, got, b.reference(q, H, KV), b.max_v(), f"attention 1024 rows[{precision}]")
    eng.close()


# one magnet position per KV head of each session: on a row's own position (and so one past its predecessor's), on
# 16-row tile seams (15 / 16) and on 64-key block edges (63 / 64, 1023 / 1024)
MAGNET_SESSIONS = [(80, 0, [0, 1, 15, 16, 17, 47, 63, 64]),
                   (40, 1000, [1000, 1001, 1015, 1016, 1023, 1024, 1025, 1039]),
                   (33, 47, [47, 48, 62, 63, 64, 65, 78, 79])]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_attention_magnet_keys(precision):
    """Every query of KV head h shares a direction that only the key at magnet position m_h has (score 28 above all
    others), and V there is 8 in every dimension while other V lie in [-1, 1].  A row at position >= m_h must come out
    8 to within 1e-6 (the other keys' total weight is below 1e-8), a row before it must stay within [-1, 1].  A mask off
    by one key in either direction, or a wrong 64-key block edge, moves a row by about 7: no tolerance hides that."""
    H, KV = 16, 8
    act = ACT[precision]
    eng = make_engine(precision, H, KV, L=ATTN_L)
    g = gen(20)
    rows = [n for n, _, _ in MAGNET_SESSIONS]
    starts = [p for _, p, _ in MAGNET_SESSIONS]

    def k_fn(s, k):
        k = k * 0.5
        k[..., 0] = 0.0
        for h, m in enumerate(MAGNET_SESSIONS[s][2]):
            k[h, m] = 0.0
            k[h, m, 0] = 40.0
        return k

    def v_fn(s, v):
        for h, m in enumerate(MAGNET_SESSIONS[s][2]):
            v[h, m] = 8.0
        return v

    b = Batch(act, KV, rows, starts, g, k_fn, v_fn)
    q = torch.randn(b.rows, H, HD, device=DEV, generator=g) * 0.5
    q[..., 0] = 8.0                                           # score of the magnet: 8 * 40 / sqrt(128) = 28.3
    q = q.reshape(b.rows, H * HD).to(act)
    got = b.run(eng, q, H)
    G = H // KV
    o = got.float().view(b.rows, KV, G, HD)
    worst_near, worst_far, wrong = 0.0, 0.0, []
    for row0, n, p0, s in b.sessions:
        for h, m in enumerate(MAGNET_SESSIONS[s][2]):
            for r in range(n):
                x = o[row0 + r, h]
                if p0 + r >= m:
                    dev = float((x - 8.0).abs().max())     # NaN compares false: taken as wrong below
                    worst_near = max(worst_near, dev)
                    if not dev <= 1e-6:
                        wrong.append((s, h, m, p0 + r, "at or past the magnet", float(x.min()), float(x.max())))
                else:
                    far = float(x.abs().max())
                    worst_far = max(worst_far, far)
                    if not far <= 1.01:
                        wrong.append((s, h, m, p0 + r, "before the magnet", float(x.min()), float(x.max())))
    print(f"magnet[{precision}]: rows at or past the magnet within {worst_near:.1e} of 8, rows before it max |out| "
          f"{worst_far:.3f}; {len(wrong)} (session, head, magnet, position) rows wrong")
    assert not wrong, (len(wrong), wrong[:12])
    check_attention(precision, got, b.reference(q, H, KV), b.max_v(), f"magnet[{precision}]")
    eng.close()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_attention_moving_maximum(precision):
    """The online softmax rescales O and l whenever a key block raises a row's running maximum.  With random keys the
    maximum settles early; here key norms rise block by block (64 keys) up to 6x, and fall in one KV head, so most
    rows move their maximum by large factors many times, at different blocks."""
    H, KV = 16, 8
    act = ACT[precision]
    eng = make_engine(precision, H, KV, L=ATTN_L)
    g = gen(77)
    T_end = 4096

    def k_fn(s, k):
        T = k.shape[1]
        blk = torch.arange(T, device=DEV) // 64
        ramp = 1.0 + 5.0 * blk.float() / float(blk.max())
        k = k * ramp[None, :, None]
        k[3] = k[3] * torch.linspace(1.0, 0.2, T, device=DEV)[:, None] / ramp[:, None]    # ... falling in one head
        return k

    b = Batch(act, KV, [16, 40], [T_end - 16, 1000], g, k_fn)
    q = torch.randn(b.rows, H * HD, device=DEV, generator=g).to(act)
    got = b.run(eng, q, H)
    # the path under test is really taken: last block's max score vs the first block's, in log2 units
    row0, n, p0, s = b.sessions[0]
    k = b.caches[s][ATTN_LAYER, 0, :, :T_end].float().repeat_interleave(H // KV, dim=0)
    sc = (q[row0:row0 + n].float().view(n, H, HD).transpose(0, 1) @ k.transpose(1, 2)) * SCALE
    jump = (sc[..., -64:].amax(-1) - sc[..., :64].amax(-1)) * 1.4427
    assert (jump > 8).float().mean().item() > 0.5, jump
    check_attention(precision, got, b.reference(q, H, KV), b.max_v(), f"moving maximum[{precision}]")
    eng.close()


def test_attention_rejects_what_the_kernels_assume_away():
    H, KV = 4, 2
    eng = make_engine("bf16", H, KV, L=ATTN_L, max_ctx=64)
    cache = torch.zeros(ATTN_L, 2, KV, 64, HD, dtype=torch.bfloat16, device=DEV)
    q = torch.zeros(1025, H * HD, dtype=torch.bfloat16, device=DEV)
    out = torch.zeros_like(q)
    kv = [cache.data_ptr(), cache.data_ptr()]

    def call(pos, slot, layer=ATTN_LAYER):
        eng.op_attention(q.data_ptr(), pos, slot, kv, layer, out.data_ptr())

    call([3, 4, 5, 0, 1], [0, 0, 0, 1, 1])                    # packed: accepted
    with pytest.raises(WlkError, match="rows"):
        call([], [])
    with pytest.raises(WlkError, match="rows"):
        call(list(range(1025)), [0] * 1025)
    with pytest.raises(WlkError, match="not contiguous"):
        call([0, 0, 1], [0, 1, 0])
    with pytest.raises(WlkError, match="does not follow"):
        call([5, 7], [0, 0])
    with pytest.raises(WlkError, match="does not follow"):
        call([5, 4], [0, 0])
    with pytest.raises(WlkError, match="position"):
        call([63, 64], [0, 0])
    with pytest.raises(WlkError, match="position"):
        call([-1], [0])
    with pytest.raises(WlkError, match="slot"):
        call([0], [2])
    with pytest.raises(WlkError, match="layer"):
        call([0], [0], layer=ATTN_L)
    with pytest.raises(WlkError, match="layer"):
        call([0], [0], layer=-1)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# RMSNorm and SwiGLU

@pytest.mark.parametrize("d", [256, 1024, 2048])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_rmsnorm(precision, d):
    """Rows at ordinary scale, at 1e4, all zero, and at 1e-4 where mean(x^2) = 1e-8 is 1 % of eps (eps anywhere but
    inside the square root changes those rows by ~10x), plus one row with a single large entry.  Bound: fp32
    |out - ref| <= 2e-6 |ref| element by element: the sum of squares takes <= 8 serial adds per thread, 5 shuffle levels
    and 8 warp partials (<= 21 roundings of 2^-24, 1.3e-6, all terms positive), then +eps, rsqrtf (2 ulp) and two
    products: ~1e-6 at worst.  bf16: one ulp of the rounded reference."""
    act = ACT[precision]
    eng = make_engine(precision, d=d)
    g = gen(d)
    x = torch.randn(10, d, device=DEV, generator=g)
    x[4:6] *= 1e4
    x[6] = 0.0
    x[7:9] *= 1e-4
    x[9] = 0.01 * x[9]
    x[9, d // 3] = 50.0
    w = 1.0 + 0.2 * torch.randn(d, device=DEV, generator=g)
    ref = w.double() * (x.double() / torch.sqrt(x.double().pow(2).mean(-1, keepdim=True) + EPS))
    out = torch.full((10, d), SENTINEL, dtype=act, device=DEV)
    torch.cuda.synchronize()
    eng.op_rmsnorm(x.data_ptr(), w.data_ptr(), out.data_ptr(), 10)
    tag = f"rmsnorm[{precision} d={d}]"
    if precision == "fp32":
        rel = float(((out.double() - ref).abs() / ref.abs().clamp_min(1e-30)).max())
        print(f"{tag}: max |err| / |ref| = {rel:.2e} (bound 2e-6)")
        assert torch.equal(out[6], torch.zeros_like(out[6]))
        assert rel <= 2e-6, rel
    else:
        within_one_bf16_ulp(out, ref, tag)
    # the final norm's row map: rows marked -1 are skipped, output rows nobody maps to keep their contents
    out_row = [3, -1, 0, 7, -1, 1, 9, 2, -1, 4]
    mapped = torch.full((10, d), SENTINEL, dtype=act, device=DEV)
    torch.cuda.synchronize()
    eng.op_rmsnorm(x.data_ptr(), w.data_ptr(), mapped.data_ptr(), 10, out_row)
    for r, o in enumerate(out_row):
        if o >= 0:
            assert torch.equal(mapped[o], out[r]), (r, o)
    for o in set(range(10)) - set(out_row):
        assert (mapped[o] == SENTINEL).all(), o
    eng.close()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_swiglu(precision):
    """silu(g) * u against float64, gates at the fp32 edges of exp (+-88 is where exp(-g) nears FLT_MAX; at -100 it
    overflows to inf and the kernel returns -0 for -3.7e-42) and a random bulk.  Bound: fp32 |out - ref| <= 5e-7 |ref| +
    1e-40: expf (2 ulp) passes into 1 / (1 + e) with a factor <= 1, then 1 + e, the division and the product round once
    each, 3.5 ulp of 2^-23 at worst; the absolute 1e-40 covers the underflowed -100 gates.  bf16: one ulp of the rounded
    reference (subnormal spacing for the underflowed ones)."""
    act = ACT[precision]
    F, R = 512, 37
    eng = make_engine(precision, F=F)
    g = gen(5)
    gate = torch.randn(R, F, device=DEV, generator=g) * 6.0
    up = torch.randn(R, F, device=DEV, generator=g) * 2.0
    specials = torch.tensor([-100.0, -88.0, -20.0, 0.0, 20.0, 88.0, 100.0], device=DEV)
    gate[:, :7] = specials
    idx = torch.randint(0, R * F, (300,), device=DEV, generator=g)
    gate.view(-1)[idx] = specials[torch.arange(300, device=DEV) % 7]
    gu = torch.cat([gate, up], dim=1).contiguous()
    hid = torch.full((R, F), SENTINEL, dtype=act, device=DEV)
    torch.cuda.synchronize()
    eng.op_swiglu(gu.data_ptr(), hid.data_ptr(), R)
    ref = torch.nn.functional.silu(gate.double()) * up.double()
    tag = f"swiglu[{precision}]"
    if precision == "fp32":
        err = (hid.double() - ref).abs()
        ratio = float((err / (5e-7 * ref.abs() + 1e-40)).max())
        big = ref.abs() > 1e-30
        rel = float((err[big] / ref.abs()[big]).max())
        print(f"{tag}: max |err| / |ref| = {rel:.2e} where |ref| > 1e-30; {ratio:.2f} of the bound 5e-7 |ref| + 1e-40")
        assert ratio <= 1.0, ratio
    else:
        within_one_bf16_ulp(hid, ref, tag)
    eng.close()
