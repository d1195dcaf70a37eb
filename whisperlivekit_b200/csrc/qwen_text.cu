// Qwen3-ASR text decoder (HF Qwen3Model + lm_head) behind the C ABI (wlk_qtext_* in include/wlk_b200.h).
//   reference third_party/qwen3-asr-causal/src/qwen3_asr_causal/model.py:
//     text model wiring :1498-1507, generate_full_hypothesis_rolling :991-1250,
//     generate_full_hypothesis_from_cached_audio :839-989, _GreedyControlSession :254-438
// The host's TextDecodeDriver (whisperlivekit_b200/qwen_text_engine.py) holds the reference generate logic; this file owns
// the forward over a croppable per-session KV cache, the decode controls + argmax over the logit rows, and the two
// generate loops run in one call each (generate_full, generate_rolling).
//
// Data layout (per round, R <= QT_ROUND_ROWS rows packed over the sessions of the call, each session's rows in position
// order, so a row always finds the keys of its predecessors either in earlier rounds or in this round's scatter):
//   residual x   fp32 [R][d];  xn act [R][d];  qkv fp32 [R][(H + 2 KV) * 128];  q act [R][H * 128];
//   K/V per session act [L][K|V][KV][max_ctx][128] (written by the QK-norm + RoPE kernel);  gate|up fp32 [R][2F]
//   hlog act [logit rows][d]: final-normed rows the lm_head runs on, in groups of logit_group rows (256 MB of fp32 logits)
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include "../../include/wlk_b200.h"
#include "host.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

namespace wlk {
namespace {

constexpr int QT_HD = 128;              // head_dim the kernels specialise on
constexpr int QT_ROUND_ROWS = 1024;     // rows of one forward round (workspace bound)
constexpr size_t QT_LOGIT_BYTES = (size_t)256 << 20;   // logits workspace: lm_head + pick run in groups of rows that fit
constexpr int QT_PICK_THREADS = 512;

__device__ __forceinline__ float block_reduce_sum(float v, float* red) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
    __syncthreads();
    if (l == 0) red[w] = v;
    __syncthreads();
    float r = 0.f;
    for (int i = 0; i < nw; ++i) r += red[i];
    return r;
}

// x[r] = embed_tokens[src] (src >= 0) or the embedding row up[-1 - src] (rows up_ld floats apart: the uploaded host rows,
// or the caller's device rows).  With tok set, src[r] indexes it instead: the token a pick left on the device.
__global__ void qt_embed_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ tok, const float* __restrict__ emb,
                                const float* __restrict__ up, int64_t up_ld, float* __restrict__ x, int d) {
    const int r = blockIdx.x;
    const int s = tok ? tok[src[r]] : src[r];
    const float* from = s >= 0 ? emb + (int64_t)s * d : up + (int64_t)(-1 - s) * up_ld;
    for (int i = threadIdx.x; i < d; i += blockDim.x) x[(int64_t)r * d + i] = from[i];
}

// fp32 rows [R][cols] with row pitch ld -> act [R][cols] (the frame adapter's GEMM operand)
template <typename T>
__global__ void qt_rows_to_act_kernel(const float* __restrict__ in, int64_t ld, T* __restrict__ out, int cols) {
    const int r = blockIdx.x;
    for (int i = threadIdx.x; i < cols; i += blockDim.x) out[(int64_t)r * cols + i] = from_f32<T>(in[(int64_t)r * ld + i]);
}

// Qwen3RMSNorm: w * (x * rsqrt(mean(x^2) + eps)), fp32 statistics; out row = out_row ? out_row[r] : r (skip when < 0)
template <typename T>
__global__ void qt_rmsnorm_kernel(const float* __restrict__ x, const float* __restrict__ w, T* __restrict__ out,
                                  const int32_t* __restrict__ out_row, int d, float eps) {
    __shared__ float red[32];
    const int r = blockIdx.x;
    const int o = out_row ? out_row[r] : r;
    if (o < 0) return;
    const float* xr = x + (int64_t)r * d;
    float s = 0.f;
    for (int i = threadIdx.x; i < d; i += blockDim.x) s += xr[i] * xr[i];
    s = block_reduce_sum(s, red);
    const float inv = rsqrtf(s / (float)d + eps);
    for (int i = threadIdx.x; i < d; i += blockDim.x) out[(int64_t)o * d + i] = from_f32<T>(w[i] * (xr[i] * inv));
}

// After the fused QKV GEMM: per-head RMSNorm (q_norm / k_norm over 128 dims), HF rotate-half RoPE at the row's position,
// q -> qout [R][H*128], k / v -> the session cache.  grid (R, H + 2 KV), 128 threads (one per dim).
template <typename T>
__global__ void __launch_bounds__(QT_HD)
qt_qk_rope_kernel(const float* __restrict__ qkv, const float* __restrict__ qn, const float* __restrict__ kn,
                  const float* __restrict__ inv_freq, const int32_t* __restrict__ row_pos, const int32_t* __restrict__ row_slot,
                  void* const* __restrict__ kv_ptrs, T* __restrict__ qout, int layer, int H, int KV, int max_ctx, float eps) {
    __shared__ float red[4];
    __shared__ float vals[QT_HD];
    const int r = blockIdx.x, hh = blockIdx.y, i = threadIdx.x;
    const int W = (H + 2 * KV) * QT_HD;
    float v = qkv[(int64_t)r * W + hh * QT_HD + i];
    const int pos = row_pos[r];
    T* kvbase = reinterpret_cast<T*>(kv_ptrs[row_slot[r]]);
    if (hh >= H + KV) {                                            // v head: straight to the cache
        const int kh = hh - H - KV;
        kvbase[((((int64_t)layer * 2 + 1) * KV + kh) * max_ctx + pos) * QT_HD + i] = from_f32<T>(v);
        return;
    }
    const float s = block_reduce_sum(v * v, red);
    v = (hh < H ? qn[i] : kn[i]) * (v * rsqrtf(s / (float)QT_HD + eps));
    vals[i] = v;
    __syncthreads();
    const int j = i & (QT_HD / 2 - 1);
    const float ang = (float)pos * inv_freq[j];
    const float c = cosf(ang), sn = sinf(ang);
    const float rot = i < QT_HD / 2 ? -vals[i + QT_HD / 2] : vals[i - QT_HD / 2];
    const float o = v * c + rot * sn;
    if (hh < H) qout[(int64_t)r * H * QT_HD + hh * QT_HD + i] = from_f32<T>(o);
    else kvbase[((((int64_t)layer * 2 + 0) * KV + (hh - H)) * max_ctx + pos) * QT_HD + i] = from_f32<T>(o);
}

// fp32 mode: causal GQA attention over the session cache: the query at position p attends to cache positions 0 .. p (its own
// block's keys were scattered before this kernel).  grid (R, KV); one warp per query head of the KV group, so the
// group's heads stream the same K/V rows (L1-shared) instead of one pass per head.  Online fp32 softmax, scale 128^-0.5.
template <typename T>
__global__ void __launch_bounds__(256)
qt_attention_kernel(const T* __restrict__ q, const int32_t* __restrict__ row_pos, const int32_t* __restrict__ row_slot,
                    void* const* __restrict__ kv_ptrs, T* __restrict__ out, int layer, int H, int KV, int max_ctx) {
    __shared__ float qs[8][QT_HD];
    const int r = blockIdx.x, kh = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int G = H / KV;
    if (warp >= G) return;
    const int h = kh * G + warp;
    const int pos = row_pos[r];
    const T* kv = reinterpret_cast<const T*>(kv_ptrs[row_slot[r]]);
    const T* kb = kv + (((int64_t)layer * 2 + 0) * KV + kh) * max_ctx * QT_HD;
    const T* vb = kv + (((int64_t)layer * 2 + 1) * KV + kh) * max_ctx * QT_HD;
    const float scale = 0.08838834764831845f;                      // 128^-0.5
#pragma unroll
    for (int e = 0; e < 4; ++e) qs[warp][lane + 32 * e] = to_f32(q[(int64_t)r * H * QT_HD + h * QT_HD + lane + 32 * e]) * scale;
    __syncwarp();
    float m = -INFINITY, l = 0.f, acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k0 = 0; k0 <= pos; k0 += 32) {
        const int k = k0 + lane;
        float sc = -INFINITY;
        if (k <= pos) {
            const T* kr = kb + (int64_t)k * QT_HD;
            float a = 0.f;
#pragma unroll 16
            for (int e = 0; e < QT_HD; ++e) a = fmaf(qs[warp][e], to_f32(kr[e]), a);
            sc = a;
        }
        const float mt = warp_max(sc);
        const float mn = fmaxf(m, mt);
        const float corr = expf(m - mn);                           // m = -inf on the first tile: corr = 0
        const float p = k <= pos ? expf(sc - mn) : 0.f;
        l = l * corr + warp_sum(p);
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[e] *= corr;
        const int nk = min(32, pos + 1 - k0);
        for (int j = 0; j < nk; ++j) {
            const float pj = __shfl_sync(0xffffffffu, p, j);
            const T* vr = vb + (int64_t)(k0 + j) * QT_HD;
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[e] = fmaf(pj, to_f32(vr[lane + 32 * e]), acc[e]);
        }
        m = mn;
    }
    const float inv = 1.0f / l;
#pragma unroll
    for (int e = 0; e < 4; ++e) out[(int64_t)r * H * QT_HD + h * QT_HD + lane + 32 * e] = from_f32<T>(acc[e] * inv);
}

// bf16 mode: the same attention on warp-level tensor cores (mma.sync m16n8k16, bf16 operands, fp32 accumulate).
// One CTA per (tile of <= 16 consecutive query rows of one session, KV head), one warp per query head of the group:
// the CTA stages 64-key K and V tiles in shared memory once and every head of the group runs its 16 x 64 score MMA,
// the online fp32 softmax and the P V MMA on them, so a tile's K/V leave HBM once per KV group.  Rows past n_rows of a
// tile carry zero queries and are not stored; row r attends to keys 0 .. pos0 + r.
struct QTAttnTile { int32_t row0, n_rows, slot, pos0; };
constexpr int QT_KT = 64;                         // keys per shared-memory tile
constexpr int QT_KPAD = QT_HD + 8;                // padded row: the fragment loads of a quad hit distinct banks


__global__ void __launch_bounds__(256)
qt_attention_mma_kernel(const bf16* __restrict__ q, const QTAttnTile* __restrict__ tiles, void* const* __restrict__ kv_ptrs,
                        bf16* __restrict__ out, int layer, int H, int KV, int max_ctx) {
    __shared__ __align__(16) bf16 ks[QT_KT][QT_KPAD];
    __shared__ __align__(16) bf16 vs[QT_KT][QT_KPAD];
    const QTAttnTile tl = tiles[blockIdx.x];
    const int kh = blockIdx.y, G = H / KV, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int h = kh * G + warp;
    const bf16* kv = reinterpret_cast<const bf16*>(kv_ptrs[tl.slot]);
    const bf16* kb = kv + (((int64_t)layer * 2 + 0) * KV + kh) * max_ctx * QT_HD;
    const bf16* vb = kv + (((int64_t)layer * 2 + 1) * KV + kh) * max_ctx * QT_HD;
    const int kend = tl.pos0 + tl.n_rows;
    const bool ok0 = g < tl.n_rows, ok1 = g + 8 < tl.n_rows;
    const bf16* q0 = q + (int64_t)(tl.row0 + g) * H * QT_HD + h * QT_HD;
    const bf16* q1 = q + (int64_t)(tl.row0 + g + 8) * H * QT_HD + h * QT_HD;
    uint32_t qa[8][4];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
        const int c = kk * 16 + 2 * t;
        qa[kk][0] = ok0 ? *reinterpret_cast<const uint32_t*>(q0 + c) : 0u;
        qa[kk][1] = ok1 ? *reinterpret_cast<const uint32_t*>(q1 + c) : 0u;
        qa[kk][2] = ok0 ? *reinterpret_cast<const uint32_t*>(q0 + c + 8) : 0u;
        qa[kk][3] = ok1 ? *reinterpret_cast<const uint32_t*>(q1 + c + 8) : 0u;
    }
    const int lim0 = min(tl.pos0 + g, kend - 1), lim1 = min(tl.pos0 + g + 8, kend - 1);
    const float scale = 0.08838834764831845f;                      // 128^-0.5
    float o[16][4];
#pragma unroll
    for (int n = 0; n < 16; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    for (int k0 = 0; k0 < kend; k0 += QT_KT) {
        __syncthreads();                                           // the previous tile is consumed
        for (int i = threadIdx.x; i < QT_KT * (QT_HD / 8); i += blockDim.x) {
            const int r = i / (QT_HD / 8), c = (i % (QT_HD / 8)) * 8;
            uint4 kz = make_uint4(0, 0, 0, 0), vz = kz;
            if (k0 + r < kend) {
                kz = *reinterpret_cast<const uint4*>(kb + (int64_t)(k0 + r) * QT_HD + c);
                vz = *reinterpret_cast<const uint4*>(vb + (int64_t)(k0 + r) * QT_HD + c);
            }
            *reinterpret_cast<uint4*>(&ks[r][c]) = kz;
            *reinterpret_cast<uint4*>(&vs[r][c]) = vz;
        }
        __syncthreads();
        float s[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&ks[8 * j + g][kk * 16 + 2 * t]);
                const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&ks[8 * j + g][kk * 16 + 2 * t + 8]);
                ptx::mma_bf16_16816(s[j], qa[kk], b0, b1);
            }
        }
        float mx0 = m0, mx1 = m1;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = k0 + 8 * j + 2 * t + (e & 1);
                const bool ok = key <= (e < 2 ? lim0 : lim1);
                s[j][e] = ok ? s[j][e] * scale : -INFINITY;
                if (e < 2) mx0 = fmaxf(mx0, s[j][e]); else mx1 = fmaxf(mx1, s[j][e]);
            }
#pragma unroll
        for (int off = 1; off <= 2; off <<= 1) {
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off));
        }
        const float c0 = expf(m0 - mx0), c1 = expf(m1 - mx1);     // the first tile always holds key 0: mx is finite
        float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s[j][0] = expf(s[j][0] - mx0); s[j][1] = expf(s[j][1] - mx0);
            s[j][2] = expf(s[j][2] - mx1); s[j][3] = expf(s[j][3] - mx1);
            sum0 += s[j][0] + s[j][1];
            sum1 += s[j][2] + s[j][3];
        }
#pragma unroll
        for (int off = 1; off <= 2; off <<= 1) {
            sum0 += __shfl_xor_sync(0xffffffffu, sum0, off);
            sum1 += __shfl_xor_sync(0xffffffffu, sum1, off);
        }
        l0 = l0 * c0 + sum0;
        l1 = l1 * c1 + sum1;
#pragma unroll
        for (int n = 0; n < 16; ++n) { o[n][0] *= c0; o[n][1] *= c0; o[n][2] *= c1; o[n][3] *= c1; }
#pragma unroll
        for (int kk = 0; kk < QT_KT / 16; ++kk) {
            const uint32_t pa[4] = {ptx::pack_bf16x2(s[2 * kk][0], s[2 * kk][1]), ptx::pack_bf16x2(s[2 * kk][2], s[2 * kk][3]),
                                    ptx::pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]), ptx::pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3])};
            const int kr = 16 * kk + 2 * t;
#pragma unroll
            for (int n = 0; n < 16; ++n) {
                const int c = 8 * n + g;
                const uint32_t b0 = ptx::pack_bf16_pair(vs[kr][c], vs[kr + 1][c]);
                const uint32_t b1 = ptx::pack_bf16_pair(vs[kr + 8][c], vs[kr + 9][c]);
                ptx::mma_bf16_16816(o[n], pa, b0, b1);
            }
        }
        m0 = mx0; m1 = mx1;
    }
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
    for (int n = 0; n < 16; ++n) {
        const int c = h * QT_HD + 8 * n + 2 * t;
        if (ok0) *reinterpret_cast<uint32_t*>(out + (int64_t)(tl.row0 + g) * H * QT_HD + c) = ptx::pack_bf16x2(o[n][0] * i0, o[n][1] * i0);
        if (ok1) *reinterpret_cast<uint32_t*>(out + (int64_t)(tl.row0 + g + 8) * H * QT_HD + c) = ptx::pack_bf16x2(o[n][2] * i1, o[n][3] * i1);
    }
}

// SwiGLU: hid[r][j] = silu(gate[r][j]) * up[r][j], gate|up = gu[r][0:F] | gu[r][F:2F] (fp32, down_proj(act(gate) * up))
template <typename T>
__global__ void qt_swiglu_kernel(const float* __restrict__ gu, T* __restrict__ hid, int rows, int F) {
    const int64_t total = (int64_t)rows * F;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / F, j = i % F;
        const float g = gu[r * 2 * F + j], u = gu[r * 2 * F + F + j];
        hid[i] = from_f32<T>(g / (1.0f + expf(-g)) * u);
    }
}

struct PickArgs {
    float* logits; int64_t ld; int vocab;
    const int32_t* hist; const int32_t* hist_off; const int32_t* hist_len;
    const int32_t* suppress; int n_suppress;
    float penalty; int penalize; int ngram; int max_consec; int wait_id;
    int32_t* picks; float* values;
    // device-resident histories (gen != null): row j picks for session row_sess[j], whose history is its first `step`
    // tokens gen[row_sess[j]][0 .. step) (row_step[j] tokens instead when row_step is set); the pick is appended there
    // and left in next[row_sess[j]] for the next forward
    int32_t* gen; int gen_ld; const int32_t* row_sess; int step; int32_t* next; const int32_t* row_step;
};

// _GreedyControlSession.controlled_logits + argmax (model.py:335-418), one CTA per logit row, in place on the row:
// suppress (-inf) -> repetition penalty on the unique in-vocab history (first occurrence claims the token in a shared
// vocab bitmap) -> n-gram ban (finfo(float32).min) -> max-consecutive (only the wait score stays) -> argmax, lowest index on
// ties.  The modified set is a few hundred ids; the argmax then reads each logit once.
__global__ void __launch_bounds__(QT_PICK_THREADS) qt_pick_kernel(PickArgs a) {
    extern __shared__ uint32_t seen[];
    __shared__ float bv[QT_PICK_THREADS / 32];
    __shared__ int bi[QT_PICK_THREADS / 32];
    const int row = blockIdx.x, tid = threadIdx.x;
    float* lg = a.logits + (int64_t)row * a.ld;
    const int sess = a.gen ? a.row_sess[row] : 0;
    int32_t* gh = a.gen ? a.gen + (int64_t)sess * a.gen_ld : nullptr;
    const int32_t* h = a.gen ? gh : a.hist + a.hist_off[row];
    const int n = a.gen ? (a.row_step ? a.row_step[row] : a.step) : a.hist_len[row];
    auto emit = [&](int pick, float value) {                          // thread 0, after every read of the history
        a.picks[row] = pick;
        if (a.values) a.values[row] = value;
        if (gh) { gh[n] = pick; a.next[sess] = pick; }
    };
    const int words = (a.vocab + 31) / 32;
    const float fmin = -3.4028234663852886e38f;
    for (int i = tid; i < a.n_suppress; i += blockDim.x) lg[a.suppress[i]] = -INFINITY;
    for (int i = tid; i < words; i += blockDim.x) seen[i] = 0u;
    __syncthreads();
    if (a.penalize) {
        for (int i = tid; i < n; i += blockDim.x) {
            const int t = h[i];
            if (t < 0 || t >= a.vocab) continue;
            const uint32_t bit = 1u << (t & 31);
            if (atomicOr(&seen[t >> 5], bit) & bit) continue;          // not the first occurrence
            const float x = lg[t];
            lg[t] = x < 0.f ? x * a.penalty : x / a.penalty;
        }
    }
    __syncthreads();
    if (a.ngram > 0) {
        const int pre = a.ngram - 1;
        for (int s = tid; s <= n - a.ngram; s += blockDim.x) {
            bool match = true;
            for (int k = 0; k < pre && match; ++k) match = h[s + k] == h[n - pre + k];
            const int t = h[s + pre];
            if (match && t >= 0 && t < a.vocab) lg[t] = fmin;
        }
    }
    __syncthreads();
    if (a.max_consec > 0 && a.wait_id >= 0 && a.wait_id < a.vocab && n >= a.max_consec) {
        if (tid == 0) {                                               // every other entry is finfo.min
            const float w = lg[a.wait_id];
            const int pick = (w > fmin || a.wait_id == 0) ? a.wait_id : 0;
            emit(pick, pick == a.wait_id ? w : fmin);
        }
        return;
    }
    float best = -INFINITY;
    int besti = 0x7fffffff;
    for (int v = tid; v < a.vocab; v += blockDim.x) {
        const float x = lg[v];
        if (x > best || (x == best && v < besti)) { best = x; besti = v; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
        if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
    }
    if ((tid & 31) == 0) { bv[tid >> 5] = best; bi[tid >> 5] = besti; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
            if (bv[w] > best || (bv[w] == best && bi[w] < besti)) { best = bv[w]; besti = bi[w]; }
        if (besti == 0x7fffffff) besti = 0;                            // NaN row: torch.argmax would say 0 too
        emit(besti, best);
    }
}

// Draft verification of generate_full_hypothesis_rolling (model.py:991-1250), one CTA per session.  Session i's verify
// picks are picks[base[i] .. base[i] + dl[i]], row j picked after draft[:j]; accepted = the first j whose pick differs
// from draft[j], else dl.  The pick after the accepted prefix (the correction, or the tail's first pick when all of the
// draft stands) starts the continuation: gen row i becomes draft[:accepted] + [that pick] (the pick only while it fits
// gen_ld), next[i] holds it for the next forward and res[i] = (accepted, pick) is what the host reads.
__global__ void qt_verify_kernel(const int32_t* __restrict__ picks, const int32_t* __restrict__ base,
                                 const int32_t* __restrict__ draft, const int32_t* __restrict__ draft_off,
                                 const int32_t* __restrict__ dl, int32_t* __restrict__ gen, int gen_ld,
                                 int32_t* __restrict__ next, int32_t* __restrict__ res) {
    __shared__ int acc;
    const int i = blockIdx.x, n = dl[i];
    const int32_t* p = picks + base[i];
    const int32_t* d = draft + draft_off[i];
    if (threadIdx.x == 0) acc = n;
    __syncthreads();
    for (int j = threadIdx.x; j < n; j += blockDim.x)
        if (p[j] != d[j]) atomicMin(&acc, j);
    __syncthreads();
    const int a = acc;
    int32_t* g = gen + (int64_t)i * gen_ld;
    for (int j = threadIdx.x; j < a; j += blockDim.x) g[j] = d[j];
    if (threadIdx.x == 0) {
        const int tok = p[a];
        if (a < gen_ld) g[a] = tok;
        next[i] = tok;
        res[2 * i] = a;
        res[2 * i + 1] = tok;
    }
}

struct QTLayerW {
    void *Wqkv = nullptr, *Wo = nullptr, *Wgu = nullptr, *Wd = nullptr;
    float *qn = nullptr, *kn = nullptr, *ln1 = nullptr, *ln2 = nullptr;
};

struct QTSession {
    bool open = false;
    int len = 0;
    void* kv = nullptr;
};

// QwenAudioSurgeryFrameAdapter (reference model.py:631-691): proj [d][in_dim] without bias, then `nb` blocks of
// x + scale * down(silu(gate(n)) * up(n)), n = RMSNorm(x) with eps 1e-6 (the reference's own RMSNorm, model.py:83-91).
// Tensors are stashed on load and packed by finalize, which derives in_dim, nb and the hidden width from their shapes.
struct QTAdapter {
    int in_dim = 0, hidden = 0, nb = 0;
    float scale = 0.f;
    void* Wp = nullptr;                              // act [d][in_dim]
    std::vector<float*> norm;                        // fp32 [d]
    std::vector<void*> Wgu, Wd;                      // act [2 hidden][d] (gate | up), [d][hidden]
    void* a_in = nullptr;                            // act [QT_ROUND_ROWS][in_dim]
    float* a_gu = nullptr;                           // fp32 [QT_ROUND_ROWS][2 hidden]
    void* a_hid = nullptr;                           // act [QT_ROUND_ROWS][hidden]
};
constexpr float QT_ADAPTER_EPS = 1e-6f;

}  // namespace
}  // namespace wlk

using namespace wlk;

struct wlk_qtext : EngineBase {
    wlk_qtext_dims dims{};
    size_t kv_bytes = 0;
    float *emb = nullptr, *normw = nullptr, *inv_freq = nullptr;
    void* head = nullptr;                               // lm_head [V][d] act type (the embedding table when tied)
    std::vector<QTLayerW> L;
    SessionTable<QTSession> sess;
    float *x = nullptr, *qkv = nullptr, *gu = nullptr, *up = nullptr, *logits = nullptr, *values_d = nullptr;
    void *xn = nullptr, *qb = nullptr, *att = nullptr, *hid = nullptr, *hlog = nullptr;
    int32_t* picks_d = nullptr;
    float* up_h = nullptr;                               // pinned: the round's host embedding rows, one H2D copy per round
    int32_t* pick_d = nullptr; size_t pick_cap = 0;      // device copy of a pick call's histories, suppress list, offsets
    int32_t* gen_d = nullptr; size_t gen_cap = 0;        // generate_full: per-session token histories + next tokens
    int logit_group = 0;
    int up_rows = 0;                                     // rows of `up` (uploaded embedding rows)
    int logit_cap = 0, n_logit = 0;                      // rows of hlog; rows the last forward kept
    std::map<std::string, std::pair<std::vector<int64_t>, std::vector<float>>> adapter_stash;   // until finalize
    bool has_adapter = false;
    QTAdapter ad;
};

namespace {

// bf16 runs every GEMM on the wgmma kernels (cfg->gemm_backend is not consulted); a shape they do not take is an error
void tgemm(wlk_qtext* t, GemmArgs& g) { t->gemm.run(g, t->act == DT_BF16, t->st, t->num_sms, "text decoder"); }

// Pack the stashed adapter tensors (no-op when none were loaded).
void build_adapter(wlk_qtext* t) {
    auto& st = t->adapter_stash;
    if (st.empty()) return;
    const int d = t->dims.d_model;
    auto get = [&](const std::string& name) -> std::pair<std::vector<int64_t>, std::vector<float>>& {
        auto it = st.find(name);
        WLK_CHECK(it != st.end(), "adapter tensor %s missing", name.c_str());
        return it->second;
    };
    auto& proj = get("adapter.proj.weight");
    WLK_CHECK(proj.first.size() == 2 && proj.first[0] == d && proj.first[1] >= 8 && proj.first[1] % 8 == 0,
              "adapter.proj.weight must be [d_model][in_dim] with in_dim a multiple of 8");
    QTAdapter& A = t->ad;
    A.in_dim = (int)proj.first[1];
    int nb = 0;
    while (st.count("adapter.blocks." + std::to_string(nb) + ".norm.weight")) ++nb;
    A.nb = nb;
    size_t used = 1;
    if (nb > 0) {
        auto& rs = get("adapter.residual_scale");
        WLK_CHECK(rs.second.size() == 1, "adapter.residual_scale must hold one value");
        A.scale = rs.second[0];
        used++;
        A.hidden = (int)get("adapter.blocks.0.mlp.gate.weight").first[0];
        WLK_CHECK(A.hidden >= 8 && A.hidden % 8 == 0, "adapter hidden width %d must be a positive multiple of 8", A.hidden);
    } else if (st.count("adapter.residual_scale")) {
        used++;
    }
    const size_t es = t->es();
    size_t* aw = &t->bytes_weights;
    A.Wp = t->allocs.take((size_t)d * A.in_dim * es, aw);
    t->upload.put(proj.second.data(), proj.second.size(), A.Wp, t->act, t->st);
    const int64_t H = A.hidden;
    for (int i = 0; i < nb; ++i) {
        const std::string p = "adapter.blocks." + std::to_string(i) + ".";
        auto& nw = get(p + "norm.weight");
        auto& g = get(p + "mlp.gate.weight");
        auto& u = get(p + "mlp.up.weight");
        auto& dn = get(p + "mlp.down.weight");
        WLK_CHECK(nw.first == std::vector<int64_t>{d}, "%snorm.weight must be [d_model]", p.c_str());
        WLK_CHECK(g.first == (std::vector<int64_t>{H, d}) && u.first == (std::vector<int64_t>{H, d}),
                  "%smlp.gate / mlp.up must be [hidden][d_model] with the hidden width of block 0", p.c_str());
        WLK_CHECK(dn.first == (std::vector<int64_t>{d, H}), "%smlp.down.weight must be [d_model][hidden]", p.c_str());
        float* nd = (float*)t->allocs.take((size_t)d * 4, aw);
        t->upload.put(nw.second.data(), nw.second.size(), nd, DT_F32, t->st);
        void* gu = t->allocs.take((size_t)2 * H * d * es, aw);
        t->upload.put(g.second.data(), g.second.size(), gu, t->act, t->st);
        t->upload.put(u.second.data(), u.second.size(), (char*)gu + (size_t)H * d * es, t->act, t->st);
        void* wd = t->allocs.take((size_t)d * H * es, aw);
        t->upload.put(dn.second.data(), dn.second.size(), wd, t->act, t->st);
        A.norm.push_back(nd); A.Wgu.push_back(gu); A.Wd.push_back(wd);
        used += 4;
    }
    WLK_CHECK(used == st.size(), "%zu adapter tensors do not belong to an adapter of %d blocks", st.size() - used, nb);
    size_t* ws = &t->bytes_workspace;
    A.a_in = t->allocs.take((size_t)QT_ROUND_ROWS * A.in_dim * es, ws);
    if (nb > 0) {
        A.a_gu = (float*)t->allocs.take((size_t)QT_ROUND_ROWS * 2 * H * 4, ws);
        A.a_hid = t->allocs.take((size_t)QT_ROUND_ROWS * H * es, ws);
    }
    st.clear();
    t->has_adapter = true;
}

void create(const wlk_qtext_dims* dims, const wlk_config* cfg, wlk_qtext** out) {
    WLK_CHECK(dims && cfg && out, "null argument");
    const wlk_qtext_dims& D = *dims;
    WLK_CHECK(D.head_dim == QT_HD, "head_dim must be %d", QT_HD);
    WLK_CHECK(D.n_kv_head >= 1 && D.n_head % D.n_kv_head == 0 && D.n_head / D.n_kv_head <= 8, "n_head must be a multiple (<= 8x) of n_kv_head");
    WLK_CHECK(D.d_model % 8 == 0 && D.ffn_dim % 8 == 0 && D.vocab >= 1, "d_model and ffn_dim must be multiples of 8");
    WLK_CHECK(D.max_ctx >= 1 && D.max_ctx <= 32768, "max_ctx must be in [1, 32768]");
    WLK_CHECK((size_t)(D.vocab + 31) / 32 * 4 <= 200 * 1024, "vocab too large for the pick kernel's bitmap");
    WLK_CHECK(cfg->max_sessions >= 1 && cfg->max_batch >= 1, "max_sessions / max_batch must be >= 1");

    auto* t = new wlk_qtext();
    t->open(*cfg);
    t->dims = D;
    t->act = cfg->precision == WLK_PREC_BF16 ? DT_BF16 : DT_F32;
    const size_t es = t->es();
    const int d = D.d_model, F = D.ffn_dim, H = D.n_head, KV = D.n_kv_head;
    const size_t W = (size_t)(H + 2 * KV) * QT_HD;
    WeightTable& T = t->weights;
    T.rule = WeightTable::EXACT;
    T.wt = t->act;
    // the fp32 embedding rows, and lm_head in the activation type: a copy of the embedding table when tied
    WeightTable::Entry& emb = T.f32("embed_tokens.weight", t->emb, {D.vocab, d});
    if (D.tied) {
        T.buf(t->head, (size_t)D.vocab * d * es);
        emb.dst.push_back(WeightTable::Dst(t->head, 0, t->act));
    } else {
        T.mat("lm_head.weight", t->head, {D.vocab, d});
    }
    T.f32("norm.weight", t->normw, {d});
    T.f32("rotary_emb.inv_freq", t->inv_freq, {QT_HD / 2}).optional = true;   // the host's own RoPE frequencies
    t->L.resize(D.n_layer);
    for (int i = 0; i < D.n_layer; ++i) {
        const std::string p = "layers." + std::to_string(i) + ".";
        QTLayerW& Lw = t->L[i];
        const std::string a = p + "self_attn.", m = p + "mlp.";
        T.fused(Lw.Wqkv, t->act, {{a + "q_proj.weight", H * QT_HD}, {a + "k_proj.weight", KV * QT_HD}, {a + "v_proj.weight", KV * QT_HD}}, d);
        T.mat(a + "o_proj.weight", Lw.Wo, {d, H * QT_HD});
        T.fused(Lw.Wgu, t->act, {{m + "gate_proj.weight", F}, {m + "up_proj.weight", F}}, d);
        T.mat(m + "down_proj.weight", Lw.Wd, {d, F});
        T.f32(a + "q_norm.weight", Lw.qn, {QT_HD});
        T.f32(a + "k_norm.weight", Lw.kn, {QT_HD});
        T.f32(p + "input_layernorm.weight", Lw.ln1, {d});
        T.f32(p + "post_attention_layernorm.weight", Lw.ln2, {d});
    }
    T.allocate(t->allocs, &t->bytes_weights);
    {   // default inv_freq = 1 / theta^(2i / 128) in fp32 arithmetic like HF's default rope init (fp32 exponent, pow, then
        // 1 / x); libm's powf can still land one ulp away from torch's pow in a few entries, so hosts load
        // "rotary_emb.inv_freq" (whisperlivekit_b200/qwen_text_engine.py always does)
        std::vector<float> f(QT_HD / 2);
        for (int i = 0; i < QT_HD / 2; ++i) f[i] = 1.0f / powf(D.rope_theta, (float)(2 * i) / (float)QT_HD);
        CUDA_CHECK(cudaMemcpy(t->inv_freq, f.data(), f.size() * 4, cudaMemcpyHostToDevice));
    }
    const size_t R = QT_ROUND_ROWS;
    size_t* ws = &t->bytes_workspace;
    t->x = (float*)t->allocs.take(R * d * 4, ws);
    t->xn = t->allocs.take(R * d * es, ws);
    t->qkv = (float*)t->allocs.take(R * W * 4, ws);
    t->qb = t->allocs.take(R * H * QT_HD * es, ws);
    t->att = t->allocs.take(R * H * QT_HD * es, ws);
    t->gu = (float*)t->allocs.take(R * 2 * F * 4, ws);
    t->hid = t->allocs.take(R * F * es, ws);
    t->up_rows = (int)R;
    t->up = (float*)t->allocs.take(R * d * 4, ws);
    t->logit_cap = cfg->max_batch * 288;
    t->hlog = t->allocs.take((size_t)t->logit_cap * d * es, ws);
    t->logit_group = (int)std::max<size_t>(1, std::min<size_t>((size_t)t->logit_cap, QT_LOGIT_BYTES / ((size_t)D.vocab * 4)));
    t->logits = (float*)t->allocs.take((size_t)t->logit_group * D.vocab * 4, ws);
    t->picks_d = (int32_t*)t->allocs.take((size_t)t->logit_cap * 4, ws);
    t->values_d = (float*)t->allocs.take((size_t)t->logit_cap * 4, ws);
    if (t->act == DT_BF16) t->gemm.alloc(t->allocs, ws);
    t->stg.alloc(R * 32 + (size_t)cfg->max_batch * 16 + 8192, t->allocs, ws);
    CUDA_CHECK(cudaMallocHost(&t->up_h, R * d * 4));
    t->kv_bytes = (size_t)D.n_layer * 2 * KV * D.max_ctx * QT_HD * es;
    t->sess.slots.resize(cfg->max_sessions);
    CUDA_CHECK(cudaFuncSetAttribute(qt_pick_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    *out = t;
}

void destroy(wlk_qtext* t) {
    t->close([t] {
        for (auto& s : t->sess) if (s.kv) cudaFree(s.kv);
        if (t->up_h) cudaFreeHost(t->up_h);
        if (t->pick_d) cudaFree(t->pick_d);
        if (t->gen_d) cudaFree(t->gen_d);
    });
    delete t;
}

// Attention tiles of one round (the bf16 kernel's CTAs): <= 16 consecutive rows of one slot, a new tile whenever the
// slot changes.  Rows of a slot are contiguous and at consecutive positions, so a tile's row k sits at pos0 + k.
int make_tiles(const int32_t* pos, const int32_t* slot, int R, QTAttnTile* tiles) {
    int n = 0;
    for (int k = 0; k < R; ++k) {
        if (n == 0 || tiles[n - 1].slot != slot[k] || tiles[n - 1].n_rows == 16) tiles[n++] = QTAttnTile{k, 0, slot[k], pos[k]};
        tiles[n - 1].n_rows++;
    }
    return n;
}

// The per-kernel launches of a round, shared by run_round and the op-level entry points.
template <typename T>
void launch_rmsnorm(wlk_qtext* t, const float* x, const float* w, void* out, const int32_t* out_row_d, int R, float eps) {
    qt_rmsnorm_kernel<T><<<R, 256, 0, t->st>>>(x, w, (T*)out, out_row_d, t->dims.d_model, eps);
}

template <typename T>
void launch_qk_rope(wlk_qtext* t, const float* qkv, const float* qn, const float* kn, const int32_t* pos_d, const int32_t* slot_d,
                    void* const* kv_d, int layer, void* qout, int R) {
    const wlk_qtext_dims& D = t->dims;
    qt_qk_rope_kernel<T><<<dim3(R, D.n_head + 2 * D.n_kv_head), QT_HD, 0, t->st>>>(qkv, qn, kn, t->inv_freq, pos_d, slot_d, kv_d,
                                                                                 (T*)qout, layer, D.n_head, D.n_kv_head,
                                                                                 D.max_ctx, D.rms_eps);
}

template <typename T>
void launch_attention(wlk_qtext* t, const void* q, const int32_t* pos_d, const int32_t* slot_d, void* const* kv_d,
                      const QTAttnTile* tiles_d, int n_tiles, int layer, void* out, int R) {
    const int H = t->dims.n_head, KV = t->dims.n_kv_head;
    if (t->act == DT_BF16)
        qt_attention_mma_kernel<<<dim3(n_tiles, KV), 32 * (H / KV), 0, t->st>>>((const bf16*)q, tiles_d, kv_d, (bf16*)out,
                                                                              layer, H, KV, t->dims.max_ctx);
    else
        qt_attention_kernel<T><<<dim3(R, KV), 32 * (H / KV), 0, t->st>>>((const T*)q, pos_d, slot_d, kv_d, (T*)out, layer,
                                                                        H, KV, t->dims.max_ctx);
}

template <typename T>
void launch_swiglu(wlk_qtext* t, const float* gu, void* hid, int R, int F) {
    const int64_t total = (int64_t)R * F;
    const int blocks = (int)std::min<int64_t>((total + 255) / 256, 65535);
    qt_swiglu_kernel<T><<<blocks, 256, 0, t->st>>>(gu, (T*)hid, R, F);
}

template <typename T>
void run_round(wlk_qtext* t, int R, const int32_t* src_d, const int32_t* pos_d, const int32_t* slot_d, void* const* kv_d,
               const int32_t* logit_row_d, const QTAttnTile* tiles_d, int n_tiles, const float* up, int64_t up_ld,
               const int32_t* tok_d) {
    const wlk_qtext_dims& D = t->dims;
    const int d = D.d_model, F = D.ffn_dim, H = D.n_head, KV = D.n_kv_head;
    const int W = (H + 2 * KV) * QT_HD;
    qt_embed_kernel<<<R, 256, 0, t->st>>>(src_d, tok_d, t->emb, up, up_ld, t->x, d);
    for (int li = 0; li < D.n_layer; ++li) {
        QTLayerW& Lw = t->L[li];
        launch_rmsnorm<T>(t, t->x, Lw.ln1, t->xn, nullptr, R, D.rms_eps);
        {   GemmArgs g;
            g.A = t->xn; g.a_type = t->act; g.lda = d; g.W = Lw.Wqkv; g.w_type = t->act; g.ldw = d;
            g.M = R; g.N = W; g.K = d;
            g.epi.C = t->qkv; g.epi.c_type = DT_F32; g.epi.ldc = W;
            tgemm(t, g); }
        launch_qk_rope<T>(t, t->qkv, Lw.qn, Lw.kn, pos_d, slot_d, kv_d, li, t->qb, R);
        launch_attention<T>(t, t->qb, pos_d, slot_d, kv_d, tiles_d, n_tiles, li, t->att, R);
        {   GemmArgs g;
            g.A = t->att; g.a_type = t->act; g.lda = H * QT_HD; g.W = Lw.Wo; g.w_type = t->act; g.ldw = H * QT_HD;
            g.M = R; g.N = d; g.K = H * QT_HD;
            g.epi.residual = t->x; g.epi.ldr = d; g.epi.C = t->x; g.epi.c_type = DT_F32; g.epi.ldc = d;
            tgemm(t, g); }
        launch_rmsnorm<T>(t, t->x, Lw.ln2, t->xn, nullptr, R, D.rms_eps);
        {   GemmArgs g;
            g.A = t->xn; g.a_type = t->act; g.lda = d; g.W = Lw.Wgu; g.w_type = t->act; g.ldw = d;
            g.M = R; g.N = 2 * F; g.K = d;
            g.epi.C = t->gu; g.epi.c_type = DT_F32; g.epi.ldc = 2 * F;
            tgemm(t, g); }
        launch_swiglu<T>(t, t->gu, t->hid, R, F);
        {   GemmArgs g;
            g.A = t->hid; g.a_type = t->act; g.lda = F; g.W = Lw.Wd; g.w_type = t->act; g.ldw = F;
            g.M = R; g.N = d; g.K = F;
            g.epi.residual = t->x; g.epi.ldr = d; g.epi.C = t->x; g.epi.c_type = DT_F32; g.epi.ldc = d;
            tgemm(t, g); }
    }
    launch_rmsnorm<T>(t, t->x, t->normw, t->hlog, logit_row_d, R, D.rms_eps);
    CUDA_CHECK(cudaGetLastError());
}

// embeds: host rows [n_embeds][d_model] (staged through pinned memory), or, when embeds_ld > 0, device rows embeds_ld
// floats apart that the embedding gather reads in place.  With tok_d set, every row_src entry is an index into the
// device tokens tok_d [n_tok] instead (generate_full's decode steps: the picks never visit the host).
void forward(wlk_qtext* t, const int32_t* sids, int n, const int32_t* row_src, const int32_t* row_off, const float* embeds,
             int n_embeds, const int32_t* logit_rows, int64_t embeds_ld = 0, const int32_t* tok_d = nullptr, int n_tok = 0) {
    const wlk_qtext_dims& D = t->dims;
    const bool dev_rows = embeds_ld > 0;
    WLK_CHECK(t->finalized, "weights not finalized");
    WLK_CHECK(n >= 1 && n <= t->cfg.max_batch, "batch %d outside [1, %d]", n, t->cfg.max_batch);
    int n_logit = 0;
    t->sess.check_batch(sids, n);
    for (int i = 0; i < n; ++i) {
        QTSession& s = t->sess[sids[i]];
        const int r = row_off[i + 1] - row_off[i];
        WLK_CHECK(r >= 1, "session %d has no rows", sids[i]);
        WLK_CHECK(s.len + r <= D.max_ctx, "context full: session %d holds %d positions, %d more exceed max_ctx %d", sids[i], s.len, r, D.max_ctx);
        WLK_CHECK(logit_rows[i] >= 0 && logit_rows[i] <= r, "logit_rows[%d] = %d outside [0, %d]", i, logit_rows[i], r);
        n_logit += logit_rows[i];
    }
    WLK_CHECK(n_logit <= t->logit_cap, "%d logit rows exceed the engine's %d", n_logit, t->logit_cap);
    const int total = row_off[n] - row_off[0];
    for (int r = 0; r < total; ++r) {
        const int s = row_src[row_off[0] + r];
        if (tok_d) WLK_CHECK(s >= 0 && s < n_tok, "row %d: token index %d outside [0, %d)", r, s, n_tok);
        else WLK_CHECK(s < D.vocab && (s >= 0 || -1 - s < n_embeds), "row %d: source %d is neither a token id nor an embedding row", r, s);
    }
    // the packed row list: (session index, position, logit row or -1)
    std::vector<int> r_sess(total), r_pos(total), r_log(total);
    {   int r = 0, lg = 0;
        for (int i = 0; i < n; ++i) {
            const int cnt = row_off[i + 1] - row_off[i];
            for (int k = 0; k < cnt; ++k, ++r) {
                r_sess[r] = i; r_pos[r] = t->sess[sids[i]].len + k;
                r_log[r] = k >= cnt - logit_rows[i] ? lg++ : -1;
            }
        }
    }
    for (int r0 = 0; r0 < total; r0 += QT_ROUND_ROWS) {
        const int R = std::min(QT_ROUND_ROWS, total - r0);
        Stager sg(t->stg);                               // also waits until the previous round's copy out of up_h is done
        int32_t *src_d, *pos_d, *slot_d, *log_d;
        int32_t* src = sg.host<int32_t>(R, &src_d);
        int32_t* pos = sg.host<int32_t>(R, &pos_d);
        int32_t* slot = sg.host<int32_t>(R, &slot_d);
        int32_t* lrow = sg.host<int32_t>(R, &log_d);
        void** kv_d; void** kvp = sg.host<void*>(n, &kv_d);
        QTAttnTile* tiles_d; QTAttnTile* tiles = sg.host<QTAttnTile>(R, &tiles_d);
        for (int i = 0; i < n; ++i) kvp[i] = t->sess[sids[i]].kv;
        // embedding rows of this round go to `up` in the order they appear: packed into pinned memory, one copy
        int n_up = 0;
        for (int k = 0; k < R; ++k) {
            const int r = r0 + k;
            int s = row_src[row_off[0] + r];
            if (s < 0 && !dev_rows && !tok_d) {
                memcpy(t->up_h + (size_t)n_up * D.d_model, embeds + (size_t)(-1 - s) * D.d_model, (size_t)D.d_model * 4);
                s = -1 - n_up++;
            }
            src[k] = s; pos[k] = r_pos[r]; slot[k] = r_sess[r]; lrow[k] = r_log[r];
        }
        const int n_tiles = make_tiles(pos, slot, R, tiles);
        if (n_up) CUDA_CHECK(cudaMemcpyAsync(t->up, t->up_h, (size_t)n_up * D.d_model * 4, cudaMemcpyHostToDevice, t->st));
        sg.upload(t->st);                                // its event guards up_h as well
        const float* up = dev_rows ? embeds : t->up;
        const int64_t up_ld = dev_rows ? embeds_ld : D.d_model;
        if (t->act == DT_F32) run_round<float>(t, R, src_d, pos_d, slot_d, kv_d, log_d, tiles_d, n_tiles, up, up_ld, tok_d);
        else run_round<bf16>(t, R, src_d, pos_d, slot_d, kv_d, log_d, tiles_d, n_tiles, up, up_ld, tok_d);
    }
    // no host sync here: the pick (or logits) call that follows synchronizes once for the whole phase
    for (int i = 0; i < n; ++i) t->sess[sids[i]].len += row_off[i + 1] - row_off[i];
    t->n_logit = n_logit;
}

void head_group(wlk_qtext* t, int row0, int rows) {
    GemmArgs g;
    g.A = (const char*)t->hlog + (size_t)row0 * t->dims.d_model * t->es(); g.a_type = t->act; g.lda = t->dims.d_model;
    g.W = t->head; g.w_type = t->act; g.ldw = t->dims.d_model;
    g.M = rows; g.N = t->dims.vocab; g.K = t->dims.d_model;
    g.epi.C = t->logits; g.epi.c_type = DT_F32; g.epi.ldc = t->dims.vocab;
    tgemm(t, g);
}

// The in-vocab part of a suppress list; the reference only arms max-consecutive when the wait token is not suppressed
// (model.py:1067-1072), so a suppressed wait id becomes -1.
std::vector<int32_t> pick_suppress(wlk_qtext* t, const int32_t* suppress, int n_suppress, int* wait_id) {
    std::vector<int32_t> sup;
    for (int i = 0; i < n_suppress; ++i) if (suppress[i] >= 0 && suppress[i] < t->dims.vocab) sup.push_back(suppress[i]);
    for (int32_t v : sup) if (v == *wait_id) *wait_id = -1;
    return sup;
}

// The pick call's device buffer, grown on demand to `need` int32
int32_t* pick_buffer(wlk_qtext* t, size_t need) {
    if (need > t->pick_cap) {
        CUDA_CHECK(cudaStreamSynchronize(t->st));
        if (t->pick_d) CUDA_CHECK(cudaFree(t->pick_d));
        t->pick_d = nullptr;
        t->pick_cap = std::max(need, (size_t)1 << 16);
        CUDA_CHECK(cudaMalloc(&t->pick_d, t->pick_cap * 4));
    }
    return t->pick_d;
}

// lm_head + qt_pick_kernel over the N logit rows of the last forward, in groups of rows the logits workspace holds.
// a: everything but the logits; its per-row arrays (hist_off / hist_len or row_sess, picks, values) start at row 0.
void launch_picks(wlk_qtext* t, int N, const PickArgs& a) {
    const wlk_qtext_dims& D = t->dims;
    const size_t smem = (size_t)(D.vocab + 31) / 32 * 4;
    for (int g0 = 0; g0 < N; g0 += t->logit_group) {
        const int rows = std::min(t->logit_group, N - g0);
        head_group(t, g0, rows);
        PickArgs b = a;
        b.logits = t->logits; b.ld = D.vocab; b.vocab = D.vocab;
        if (b.gen) { b.row_sess += g0; if (b.row_step) b.row_step += g0; }
        else { b.hist_off += g0; b.hist_len += g0; }
        b.picks += g0;
        if (b.values) b.values += g0;
        qt_pick_kernel<<<rows, QT_PICK_THREADS, smem, t->st>>>(b);
        CUDA_CHECK(cudaGetLastError());
    }
}

void pick(wlk_qtext* t, const int32_t* hist, int n_hist, const int32_t* hist_off, const int32_t* hist_len, const int32_t* suppress,
          int n_suppress, float penalty, int ngram, int max_consec, int wait_id, int32_t* picks, float* values) {
    WLK_CHECK(t->finalized, "weights not finalized");
    const int N = t->n_logit;
    if (N == 0) return;
    for (int j = 0; j < N; ++j)
        WLK_CHECK(hist_off[j] >= 0 && hist_len[j] >= 0 && hist_off[j] + hist_len[j] <= n_hist, "history of row %d out of range", j);
    const std::vector<int32_t> sup = pick_suppress(t, suppress, n_suppress, &wait_id);
    // one device buffer: [2N offsets/lengths][suppress][histories]
    int32_t* meta_d = pick_buffer(t, (size_t)2 * N + sup.size() + (size_t)n_hist + 1);
    int32_t* hist_d = meta_d + 2 * N + sup.size();
    if (n_hist) CUDA_CHECK(cudaMemcpyAsync(hist_d, hist, (size_t)n_hist * 4, cudaMemcpyHostToDevice, t->st));
    CUDA_CHECK(cudaMemcpyAsync(meta_d, hist_off, (size_t)N * 4, cudaMemcpyHostToDevice, t->st));
    CUDA_CHECK(cudaMemcpyAsync(meta_d + N, hist_len, (size_t)N * 4, cudaMemcpyHostToDevice, t->st));
    if (!sup.empty()) CUDA_CHECK(cudaMemcpyAsync(meta_d + 2 * N, sup.data(), sup.size() * 4, cudaMemcpyHostToDevice, t->st));
    PickArgs a{};
    a.hist = hist_d; a.hist_off = meta_d; a.hist_len = meta_d + N;
    a.suppress = meta_d + 2 * N; a.n_suppress = (int)sup.size();
    a.penalty = penalty; a.penalize = penalty != 1.0f && penalty > 0.0f; a.ngram = ngram; a.max_consec = max_consec;
    a.wait_id = wait_id; a.picks = t->picks_d; a.values = t->values_d;
    launch_picks(t, N, a);
    CUDA_CHECK(cudaMemcpyAsync(picks, t->picks_d, (size_t)N * 4, cudaMemcpyDeviceToHost, t->st));
    if (values) CUDA_CHECK(cudaMemcpyAsync(values, t->values_d, (size_t)N * 4, cudaMemcpyDeviceToHost, t->st));
    CUDA_CHECK(cudaStreamSynchronize(t->st));            // the one host sync of a forward + pick phase
}

// The generate loops' device histories: gen_d holds n rows of max_new tokens, then n next tokens (returned).
int32_t* gen_buffer(wlk_qtext* t, int n, int max_new) {
    const size_t need = (size_t)n * max_new + n;
    if (need > t->gen_cap) {
        CUDA_CHECK(cudaStreamSynchronize(t->st));
        if (t->gen_d) CUDA_CHECK(cudaFree(t->gen_d));
        t->gen_d = nullptr;
        t->gen_cap = std::max(need, (size_t)1 << 14);
        CUDA_CHECK(cudaMalloc(&t->gen_d, t->gen_cap * 4));
    }
    return t->gen_d + (size_t)n * max_new;
}

// generate_full_hypothesis_from_cached_audio's cached path (model.py:839-989) for n caller-owned sessions at once: each
// session is reset and forwards its prefix (packed rounds as forward, one logit row per session), then every step
// forwards one row per session still decoding, in session order, and picks on it.  A session's generated tokens stay in
// gen_d, where the pick kernel appends each pick and leaves it for the next step's embedding gather, so a step uploads
// only its round staging and downloads only the picks the stop test needs.  Every session is reset on return.
void generate_full(wlk_qtext* t, const int32_t* sids, int n, const int32_t* row_src, const int32_t* row_off,
                   const float* embeds, int n_embeds, int64_t embeds_ld, int max_new, const int32_t* stop, int n_stop,
                   const int32_t* suppress, int n_suppress, float penalty, int ngram, int max_consec, int wait_id,
                   int32_t* tokens_out, int32_t* n_out) {
    const wlk_qtext_dims& D = t->dims;
    auto reset = [&] {                                   // every named session that is open, also when the call fails
        for (int i = 0; i < n; ++i)
            if (sids[i] >= 0 && sids[i] < (int)t->sess.size() && t->sess[sids[i]].open) t->sess[sids[i]].len = 0;
        t->n_logit = 0;                                  // no logit rows survive the call
    };
    try {
        WLK_CHECK(t->finalized, "weights not finalized");
        WLK_CHECK(n >= 1 && n <= t->cfg.max_batch, "batch %d outside [1, %d]", n, t->cfg.max_batch);
        WLK_CHECK(max_new >= 0, "max_new_tokens %d < 0", max_new);
        t->sess.check_batch(sids, n);
        for (int i = 0; i < n; ++i) {
            const int r = row_off[i + 1] - row_off[i];
            WLK_CHECK(r >= 1, "session %d has no rows", sids[i]);
            WLK_CHECK((int64_t)r + max_new <= D.max_ctx, "session %d: prefix %d + max_new_tokens %d exceed max_ctx %d", sids[i], r,
                      max_new, D.max_ctx);
        }
        for (int r = row_off[0]; r < row_off[n]; ++r)
            WLK_CHECK(row_src[r] < D.vocab && (row_src[r] >= 0 || -1 - row_src[r] < n_embeds),
                      "row %d: source %d is neither a token id nor an embedding row", r - row_off[0], row_src[r]);
        reset();
        for (int i = 0; i < n; ++i) n_out[i] = 0;
        if (max_new > 0) {
            const std::vector<int32_t> sup = pick_suppress(t, suppress, n_suppress, &wait_id);
            int32_t* next_d = gen_buffer(t, n, max_new);
            // pick buffer: [suppress][row -> session index of the step]
            int32_t* sup_d = pick_buffer(t, sup.size() + (size_t)n + 1);
            int32_t* row_sess_d = sup_d + sup.size();
            if (!sup.empty()) CUDA_CHECK(cudaMemcpyAsync(sup_d, sup.data(), sup.size() * 4, cudaMemcpyHostToDevice, t->st));
            PickArgs a{};
            a.suppress = sup_d; a.n_suppress = (int)sup.size();
            a.penalty = penalty; a.penalize = penalty != 1.0f && penalty > 0.0f; a.ngram = ngram; a.max_consec = max_consec;
            a.wait_id = wait_id; a.picks = t->picks_d; a.values = nullptr;
            a.gen = t->gen_d; a.gen_ld = max_new; a.row_sess = row_sess_d; a.next = next_d;

            std::vector<int32_t> live(n), live_sids(n), offs(n + 1), ones(n, 1), picks(n);
            for (int i = 0; i < n; ++i) { live[i] = i; offs[i] = i; }
            offs[n] = n;
            forward(t, sids, n, row_src, row_off, embeds, n_embeds, ones.data(), embeds_ld);
            for (int step = 0; !live.empty(); ++step) {
                const int m = (int)live.size();
                if (step > 0) {
                    for (int k = 0; k < m; ++k) live_sids[k] = sids[live[k]];
                    forward(t, live_sids.data(), m, live.data(), offs.data(), nullptr, 0, ones.data(), 0, next_d, n);
                }
                CUDA_CHECK(cudaMemcpyAsync(row_sess_d, live.data(), (size_t)m * 4, cudaMemcpyHostToDevice, t->st));
                a.step = step;
                launch_picks(t, m, a);
                CUDA_CHECK(cudaMemcpyAsync(picks.data(), t->picks_d, (size_t)m * 4, cudaMemcpyDeviceToHost, t->st));
                CUDA_CHECK(cudaStreamSynchronize(t->st));    // the one host sync of a step
                int kept = 0;
                for (int k = 0; k < m; ++k) {
                    const int i = live[k], tok = picks[k];
                    tokens_out[(size_t)i * max_new + step] = tok;
                    n_out[i] = step + 1;
                    bool stopped = step + 1 == max_new;
                    for (int s = 0; s < n_stop && !stopped; ++s) stopped = stop[s] == tok;
                    if (!stopped) live[kept++] = i;
                }
                live.resize(kept);
            }
        }
    } catch (...) {
        reset();
        throw;
    }
    reset();
}

// generate_full_hypothesis_rolling (model.py:991-1250) for n caller-owned sessions at once, with the rules of
// TextDecodeDriver._generate_rolling.  Session i holds the KV of its reused prefix; its rows (row_src / row_offsets, the
// last draft_len[i] of them the draft tokens) bring it to prefix_len[i] + draft_len[i] positions.  One forward keeps
// draft_len + 1 logit rows per session, picks on them with the draft prefixes as histories and verifies the drafts on the
// device (qt_verify_kernel); one download of (accepted, pick) per session lets the host crop each session to prefix +
// accepted.  Then every step forwards one row per session still decoding and picks over its device history; a step
// downloads only its picks.  On return every session holds prefix_len - tail_len positions ([head + audio_steps]); a
// failure after the checks resets every named session.
void generate_rolling(wlk_qtext* t, const int32_t* sids, int n, const int32_t* row_src, const int32_t* row_off,
                      const float* embeds, int n_embeds, int64_t embeds_ld, const int32_t* draft_len, const int32_t* prefix_len,
                      int tail_len, int max_new, const int32_t* stop, int n_stop, const int32_t* suppress, int n_suppress,
                      float penalty, int ngram, int max_consec, int wait_id, int32_t* tokens_out, int32_t* n_out,
                      int32_t* stats_out) {
    const wlk_qtext_dims& D = t->dims;
    WLK_CHECK(t->finalized, "weights not finalized");
    WLK_CHECK(n >= 1 && n <= t->cfg.max_batch, "batch %d outside [1, %d]", n, t->cfg.max_batch);
    WLK_CHECK(max_new >= 1, "max_new_tokens %d < 1", max_new);
    WLK_CHECK(tail_len >= 0, "tail_len %d < 0", tail_len);
    int n_verify = 0, n_draft = 0;
    t->sess.check_batch(sids, n);
    for (int i = 0; i < n; ++i) {
        const QTSession& s = t->sess[sids[i]];
        const int r = row_off[i + 1] - row_off[i], dl = draft_len[i], p = prefix_len[i];
        WLK_CHECK(dl >= 0 && dl <= max_new && dl + 1 <= r, "session %d: draft_len %d outside [0, min(max_new_tokens %d, rows %d - 1)]",
                  sids[i], dl, max_new, r);
        WLK_CHECK(p >= tail_len && s.len + r == p + dl, "session %d: %d held + %d rows is not prefix_len %d + draft_len %d "
                  "(tail_len %d)", sids[i], s.len, r, p, dl, tail_len);
        WLK_CHECK((int64_t)p + dl + max_new <= D.max_ctx, "session %d: prefix %d + draft %d + max_new_tokens %d exceed max_ctx %d",
                  sids[i], p, dl, max_new, D.max_ctx);
        for (int k = row_off[i + 1] - dl; k < row_off[i + 1]; ++k)
            WLK_CHECK(row_src[k] >= 0, "session %d: draft row %d is not a token", sids[i], k - row_off[i]);
        n_verify += dl + 1;
        n_draft += dl;
    }
    WLK_CHECK(n_verify <= t->logit_cap, "%d verify rows exceed the engine's %d logit rows", n_verify, t->logit_cap);
    for (int r = row_off[0]; r < row_off[n]; ++r)
        WLK_CHECK(row_src[r] < D.vocab && (row_src[r] >= 0 || -1 - row_src[r] < n_embeds),
                  "row %d: source %d is neither a token id nor an embedding row", r - row_off[0], row_src[r]);
    try {
        const std::vector<int32_t> sup = pick_suppress(t, suppress, n_suppress, &wait_id);
        int32_t* next_d = gen_buffer(t, n, max_new);
        // one upload: [suppress][hist_off V][hist_len V][drafts][base n][draft_off n][dl n]; then the per-step
        // [row_sess n][row_step n] and the verify results res [2n]
        std::vector<int32_t> meta(sup);
        const size_t o_hoff = meta.size(), o_hlen = o_hoff + n_verify, o_draft = o_hlen + n_verify,
                     o_base = o_draft + n_draft, o_doff = o_base + n, o_dl = o_doff + n, o_rs = o_dl + n, o_step = o_rs + n,
                     o_res = o_step + n;
        meta.resize(o_rs);
        std::vector<int32_t> logit_rows(n);
        for (int i = 0, v = 0, dd = 0; i < n; ++i) {
            const int dl = draft_len[i];
            meta[o_base + i] = v; meta[o_doff + i] = dd; meta[o_dl + i] = dl;
            for (int j = 0; j <= dl; ++j, ++v) { meta[o_hoff + v] = dd; meta[o_hlen + v] = j; }
            for (int j = 0; j < dl; ++j) meta[o_draft + dd + j] = row_src[row_off[i + 1] - dl + j];
            dd += dl;
            logit_rows[i] = dl + 1;
        }
        int32_t* buf = pick_buffer(t, o_res + 2 * (size_t)n);
        CUDA_CHECK(cudaMemcpyAsync(buf, meta.data(), meta.size() * 4, cudaMemcpyHostToDevice, t->st));
        PickArgs a{};
        a.suppress = buf; a.n_suppress = (int)sup.size();
        a.penalty = penalty; a.penalize = penalty != 1.0f && penalty > 0.0f; a.ngram = ngram; a.max_consec = max_consec;
        a.wait_id = wait_id; a.picks = t->picks_d; a.values = nullptr;

        // verify pass: every block in one forward, its picks and the draft check on the device
        forward(t, sids, n, row_src, row_off, embeds, n_embeds, logit_rows.data(), embeds_ld);
        PickArgs va = a;
        va.hist = buf + o_draft; va.hist_off = buf + o_hoff; va.hist_len = buf + o_hlen;
        launch_picks(t, n_verify, va);
        qt_verify_kernel<<<n, 128, 0, t->st>>>(t->picks_d, buf + o_base, buf + o_draft, buf + o_doff, buf + o_dl, t->gen_d,
                                                max_new, next_d, buf + o_res);
        CUDA_CHECK(cudaGetLastError());
        std::vector<int32_t> res(2 * (size_t)n), glen(n), steps(n), live, live_sids(n), offs(n + 1), ones(n, 1), picks(n),
            step_meta(2 * (size_t)n);
        CUDA_CHECK(cudaMemcpyAsync(res.data(), buf + o_res, res.size() * 4, cudaMemcpyDeviceToHost, t->st));
        CUDA_CHECK(cudaStreamSynchronize(t->st));        // the one host sync of the verify pass
        auto stops = [&](int tok) { for (int s = 0; s < n_stop; ++s) if (stop[s] == tok) return true; return false; };
        for (int i = 0; i < n; ++i) {
            const int dl = draft_len[i], acc = res[2 * i], tok = res[2 * i + 1];
            int32_t* out = tokens_out + (size_t)i * max_new;
            for (int j = 0; j < acc; ++j) out[j] = row_src[row_off[i + 1] - dl + j];
            glen[i] = acc;
            steps[i] = 0;
            if (acc < dl) t->sess[sids[i]].len = prefix_len[i] + acc;     // the corrected pick replaces draft[acc]
            if (acc < max_new) {                                          // the correction, or the tail's first pick
                out[glen[i]++] = tok;
                steps[i] = 1;
                if (!stops(tok) && glen[i] < max_new) live.push_back(i);
            }
            stats_out[4 * i] = acc;
            stats_out[4 * i + 2] = dl > 0 && acc == dl;
            stats_out[4 * i + 3] = acc < dl;
        }
        for (int i = 0; i <= n; ++i) offs[i] = i;
        // continuation: one row per live session, its device history growing by the step's pick
        while (!live.empty()) {
            const int m = (int)live.size();
            for (int k = 0; k < m; ++k) {
                live_sids[k] = sids[live[k]];
                step_meta[k] = live[k];
                step_meta[m + k] = glen[live[k]];
            }
            forward(t, live_sids.data(), m, live.data(), offs.data(), nullptr, 0, ones.data(), 0, next_d, n);
            CUDA_CHECK(cudaMemcpyAsync(buf + o_rs, step_meta.data(), (size_t)2 * m * 4, cudaMemcpyHostToDevice, t->st));
            PickArgs sa = a;
            sa.gen = t->gen_d; sa.gen_ld = max_new; sa.row_sess = buf + o_rs; sa.row_step = buf + o_rs + m; sa.next = next_d;
            launch_picks(t, m, sa);
            CUDA_CHECK(cudaMemcpyAsync(picks.data(), t->picks_d, (size_t)m * 4, cudaMemcpyDeviceToHost, t->st));
            CUDA_CHECK(cudaStreamSynchronize(t->st));    // the one host sync of a step
            int kept = 0;
            for (int k = 0; k < m; ++k) {
                const int i = live[k], tok = picks[k];
                tokens_out[(size_t)i * max_new + glen[i]++] = tok;
                steps[i]++;
                if (!stops(tok) && glen[i] < max_new) live[kept++] = i;
            }
            live.resize(kept);
        }
        for (int i = 0; i < n; ++i) {
            n_out[i] = glen[i];
            stats_out[4 * i + 1] = steps[i];
            t->sess[sids[i]].len = prefix_len[i] - tail_len;
        }
        t->n_logit = 0;
    } catch (...) {
        for (int i = 0; i < n; ++i) t->sess[sids[i]].len = 0;   // the checks above found every session open
        t->n_logit = 0;
        throw;
    }
}

void logits_out(wlk_qtext* t, int row0, int rows, float* out) {
    WLK_CHECK(t->finalized, "weights not finalized");
    WLK_CHECK(row0 >= 0 && rows >= 0 && row0 + rows <= t->n_logit, "logit rows [%d, %d) outside the last forward's %d", row0, row0 + rows, t->n_logit);
    for (int g0 = 0; g0 < rows; g0 += t->logit_group) {
        const int r = std::min(t->logit_group, rows - g0);
        head_group(t, row0 + g0, r);
        CUDA_CHECK(cudaMemcpyAsync(out + (size_t)g0 * t->dims.vocab, t->logits, (size_t)r * t->dims.vocab * 4, cudaMemcpyDeviceToHost, t->st));
        CUDA_CHECK(cudaStreamSynchronize(t->st));
    }
}

// ---- op-level entry points: one kernel of a round on caller-owned device buffers ----------------------------------

void op_rows(int rows) { WLK_CHECK(rows >= 1 && rows <= QT_ROUND_ROWS, "rows %d outside [1, %d]", rows, QT_ROUND_ROWS); }

// What the qk-rope and attention kernels index with: slot and position of each row, a layer, the slots' caches.
// `packed`: the rows are laid out as a forward packs them (each slot's rows contiguous, at consecutive positions), which
// the attention tiles assume.
void op_check_rows(wlk_qtext* t, const int32_t* pos, const int32_t* slot, int rows, void* const* kv, int n_slots, int layer,
                   bool packed) {
    op_rows(rows);
    WLK_CHECK(layer >= 0 && layer < t->dims.n_layer, "layer %d outside [0, %d)", layer, t->dims.n_layer);
    WLK_CHECK(n_slots >= 1, "no KV caches");
    std::vector<char> done(n_slots, 0);
    for (int r = 0; r < rows; ++r) {
        WLK_CHECK(slot[r] >= 0 && slot[r] < n_slots, "row %d: slot %d outside [0, %d)", r, slot[r], n_slots);
        WLK_CHECK(kv[slot[r]] != nullptr, "row %d: slot %d has no KV cache", r, slot[r]);
        WLK_CHECK(pos[r] >= 0 && pos[r] < t->dims.max_ctx, "row %d: position %d outside [0, %d)", r, pos[r], t->dims.max_ctx);
        if (!packed) continue;
        if (r > 0 && slot[r] == slot[r - 1]) {
            WLK_CHECK(pos[r] == pos[r - 1] + 1, "row %d: position %d does not follow %d of the same slot", r, pos[r], pos[r - 1]);
        } else {
            WLK_CHECK(!done[slot[r]], "row %d: the rows of slot %d are not contiguous", r, slot[r]);
            done[slot[r]] = 1;
        }
    }
}

void op_rmsnorm(wlk_qtext* t, const float* x, const float* w, void* out, int rows, const int32_t* out_row) {
    WLK_CHECK(x && w && out, "null argument");
    op_rows(rows);
    if (out_row) for (int r = 0; r < rows; ++r) WLK_CHECK(out_row[r] >= -1, "row %d: output row %d", r, out_row[r]);
    OpUpload up{t->st};
    const int32_t* out_row_d = out_row ? up.put(out_row, rows) : nullptr;
    if (t->act == DT_F32) launch_rmsnorm<float>(t, x, w, out, out_row_d, rows, t->dims.rms_eps);
    else launch_rmsnorm<bf16>(t, x, w, out, out_row_d, rows, t->dims.rms_eps);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(t->st));
}

void op_qk_rope(wlk_qtext* t, const float* qkv, const float* qn, const float* kn, const int32_t* pos, const int32_t* slot, int rows,
                void* const* kv, int n_slots, int layer, void* qout) {
    WLK_CHECK(qkv && qn && kn && pos && slot && kv && qout, "null argument");
    op_check_rows(t, pos, slot, rows, kv, n_slots, layer, false);
    OpUpload up{t->st};
    const int32_t* pos_d = up.put(pos, rows);
    const int32_t* slot_d = up.put(slot, rows);
    void* const* kv_d = up.put(kv, n_slots);
    if (t->act == DT_F32) launch_qk_rope<float>(t, qkv, qn, kn, pos_d, slot_d, kv_d, layer, qout, rows);
    else launch_qk_rope<bf16>(t, qkv, qn, kn, pos_d, slot_d, kv_d, layer, qout, rows);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(t->st));
}

void op_attention(wlk_qtext* t, const void* q, const int32_t* pos, const int32_t* slot, int rows, void* const* kv, int n_slots,
                  int layer, void* out) {
    WLK_CHECK(q && pos && slot && kv && out, "null argument");
    op_check_rows(t, pos, slot, rows, kv, n_slots, layer, true);
    std::vector<QTAttnTile> tiles(rows);
    const int n_tiles = make_tiles(pos, slot, rows, tiles.data());
    OpUpload up{t->st};
    const int32_t* pos_d = up.put(pos, rows);
    const int32_t* slot_d = up.put(slot, rows);
    void* const* kv_d = up.put(kv, n_slots);
    const QTAttnTile* tiles_d = up.put(tiles.data(), n_tiles);
    if (t->act == DT_F32) launch_attention<float>(t, q, pos_d, slot_d, kv_d, tiles_d, n_tiles, layer, out, rows);
    else launch_attention<bf16>(t, q, pos_d, slot_d, kv_d, tiles_d, n_tiles, layer, out, rows);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(t->st));
}

void op_swiglu(wlk_qtext* t, const float* gu, void* hid, int rows) {
    WLK_CHECK(gu && hid, "null argument");
    op_rows(rows);
    if (t->act == DT_F32) launch_swiglu<float>(t, gu, hid, rows, t->dims.ffn_dim);
    else launch_swiglu<bf16>(t, gu, hid, rows, t->dims.ffn_dim);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(t->st));
}

// The frame adapter over device rows, in chunks of QT_ROUND_ROWS: the residual stream lives in the forward's x workspace.
template <typename T>
void adapt_chunk(wlk_qtext* t, const float* in, int R, int64_t in_ld, float* out, int64_t out_ld) {
    const QTAdapter& A = t->ad;
    const int d = t->dims.d_model, H = A.hidden;
    qt_rows_to_act_kernel<T><<<R, 256, 0, t->st>>>(in, in_ld, (T*)A.a_in, A.in_dim);
    {   GemmArgs g;
        g.A = A.a_in; g.a_type = t->act; g.lda = A.in_dim; g.W = A.Wp; g.w_type = t->act; g.ldw = A.in_dim;
        g.M = R; g.N = d; g.K = A.in_dim;
        g.epi.C = t->x; g.epi.c_type = DT_F32; g.epi.ldc = d;
        tgemm(t, g); }
    for (int b = 0; b < A.nb; ++b) {
        launch_rmsnorm<T>(t, t->x, A.norm[b], t->xn, nullptr, R, QT_ADAPTER_EPS);
        {   GemmArgs g;
            g.A = t->xn; g.a_type = t->act; g.lda = d; g.W = A.Wgu[b]; g.w_type = t->act; g.ldw = d;
            g.M = R; g.N = 2 * H; g.K = d;
            g.epi.C = A.a_gu; g.epi.c_type = DT_F32; g.epi.ldc = 2 * H;
            tgemm(t, g); }
        launch_swiglu<T>(t, A.a_gu, A.a_hid, R, H);
        {   GemmArgs g;                                 // x + scale * down(...): col_scale, then the residual
            g.A = A.a_hid; g.a_type = t->act; g.lda = H; g.W = A.Wd[b]; g.w_type = t->act; g.ldw = H;
            g.M = R; g.N = d; g.K = H;
            g.epi.col_scale = A.scale; g.epi.scale_cols = d;
            g.epi.residual = t->x; g.epi.ldr = d; g.epi.C = t->x; g.epi.c_type = DT_F32; g.epi.ldc = d;
            tgemm(t, g); }
    }
    CUDA_CHECK(cudaMemcpy2DAsync(out, (size_t)out_ld * 4, t->x, (size_t)d * 4, (size_t)d * 4, R, cudaMemcpyDeviceToDevice, t->st));
    CUDA_CHECK(cudaGetLastError());
}

void adapt(wlk_qtext* t, const float* in, int rows, int64_t in_ld, float* out, int64_t out_ld) {
    WLK_CHECK(t->finalized, "weights not finalized");
    WLK_CHECK(t->has_adapter, "no adapter loaded");
    WLK_CHECK(rows >= 0, "rows %d < 0", rows);
    WLK_CHECK(in_ld >= t->ad.in_dim, "in_ld %lld < in_dim %d", (long long)in_ld, t->ad.in_dim);
    WLK_CHECK(out_ld >= t->dims.d_model, "out_ld %lld < d_model %d", (long long)out_ld, t->dims.d_model);
    WLK_CHECK(rows == 0 || (in && out), "null argument");
    for (int r0 = 0; r0 < rows; r0 += QT_ROUND_ROWS) {
        const int R = std::min(QT_ROUND_ROWS, rows - r0);
        if (t->act == DT_F32) adapt_chunk<float>(t, in + (int64_t)r0 * in_ld, R, in_ld, out + (int64_t)r0 * out_ld, out_ld);
        else adapt_chunk<bf16>(t, in + (int64_t)r0 * in_ld, R, in_ld, out + (int64_t)r0 * out_ld, out_ld);
    }
    CUDA_CHECK(cudaStreamSynchronize(t->st));          // out is complete when the call returns
}

}  // namespace

extern "C" {

int wlk_qtext_create(const wlk_qtext_dims* dims, const wlk_config* cfg, wlk_qtext** out) {
    WLK_API_BEGIN
    create(dims, cfg, out);
    WLK_API_END
}
int wlk_qtext_destroy(wlk_qtext* t) {
    WLK_API_BEGIN
    WLK_CHECK(t != nullptr, "null engine");
    CUDA_CHECK(cudaSetDevice(t->cfg.device));
    destroy(t);
    WLK_API_END
}
int wlk_qtext_load_tensor(wlk_qtext* t, const char* name, const float* host, const int64_t* shape, int ndim) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(name && host && shape && ndim >= 1, "bad arguments");
    if (std::string(name).rfind("adapter.", 0) == 0) {       // optional: the frame adapter, packed by finalize
        WLK_CHECK(!t->finalized, "adapter tensor %s loaded after finalize", name);
        t->adapter_stash[name] = {std::vector<int64_t>(shape, shape + ndim), std::vector<float>(host, host + numel(shape, ndim))};
    } else {
        t->weights.load(name, host, shape, ndim);
    }
    WLK_API_END
}
int wlk_qtext_finalize_weights(wlk_qtext* t) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    t->weights.require_all();
    build_adapter(t);
    t->upload.release();
    t->finalized = true;
    WLK_API_END
}
int wlk_qtext_memory(wlk_qtext* t, size_t* weights, size_t* sessions, size_t* workspace) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    t->memory(weights, sessions, workspace);
    WLK_API_END
}
int wlk_qtext_session_open(wlk_qtext* t, int32_t* sid) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(sid, "null out pointer");
    const int found = t->sess.free_slot();
    QTSession& s = t->sess[found];
    CUDA_CHECK(cudaMalloc(&s.kv, t->kv_bytes));
    t->bytes_sessions += t->kv_bytes;
    s.open = true; s.len = 0;
    *sid = found;
    WLK_API_END
}
int wlk_qtext_session_close(wlk_qtext* t, int32_t sid) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    QTSession& s = t->sess.at(sid);
    CUDA_CHECK(cudaStreamSynchronize(t->st));
    cudaFree(s.kv);
    t->bytes_sessions -= t->kv_bytes;
    s = QTSession{};
    WLK_API_END
}
int wlk_qtext_session_reset(wlk_qtext* t, int32_t sid) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    t->sess.at(sid).len = 0;
    WLK_API_END
}
int wlk_qtext_session_len(wlk_qtext* t, int32_t sid, int32_t* len) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(len, "null out pointer");
    *len = t->sess.at(sid).len;
    WLK_API_END
}
int wlk_qtext_crop(wlk_qtext* t, int32_t sid, int32_t len) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    QTSession& s = t->sess.at(sid);
    WLK_CHECK(len >= 0 && len <= s.len, "crop to %d outside [0, %d]", len, s.len);
    s.len = len;
    WLK_API_END
}
int wlk_qtext_forward(wlk_qtext* t, const int32_t* sids, int n, const int32_t* row_src, const int32_t* row_offsets,
                      const float* embeds_host, int32_t n_embeds, const int32_t* logit_rows) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(sids && row_src && row_offsets && logit_rows && (embeds_host || n_embeds == 0), "null argument");
    forward(t, sids, n, row_src, row_offsets, embeds_host, n_embeds, logit_rows);
    WLK_API_END
}
int wlk_qtext_forward_device(wlk_qtext* t, const int32_t* sids, int n, const int32_t* row_src, const int32_t* row_offsets,
                             const float* embeds_dev, int64_t embeds_ld, int32_t n_embeds, const int32_t* logit_rows) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(sids && row_src && row_offsets && logit_rows && (embeds_dev || n_embeds == 0), "null argument");
    WLK_CHECK(embeds_ld >= t->dims.d_model, "embeds_ld %lld < d_model %d", (long long)embeds_ld, t->dims.d_model);
    forward(t, sids, n, row_src, row_offsets, embeds_dev, n_embeds, logit_rows, embeds_ld);
    WLK_API_END
}
int wlk_qtext_adapt(wlk_qtext* t, const float* in_dev, int32_t rows, int64_t in_ld, float* out_dev, int64_t out_ld) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    adapt(t, in_dev, rows, in_ld, out_dev, out_ld);
    WLK_API_END
}
int wlk_qtext_adapter_dims(wlk_qtext* t, int32_t* in_dim, int32_t* n_blocks, int32_t* hidden) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    if (in_dim) *in_dim = t->has_adapter ? t->ad.in_dim : 0;
    if (n_blocks) *n_blocks = t->ad.nb;
    if (hidden) *hidden = t->ad.hidden;
    WLK_API_END
}
int wlk_qtext_pick(wlk_qtext* t, const int32_t* hist_tokens, int32_t n_hist_tokens, const int32_t* hist_off,
                   const int32_t* hist_len, const int32_t* suppress, int32_t n_suppress, float repetition_penalty,
                   int32_t no_repeat_ngram_size, int32_t max_consecutive, int32_t wait_token_id, int32_t* picks_out,
                   float* value_out) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(hist_off && hist_len && picks_out && (hist_tokens || n_hist_tokens == 0) && (suppress || n_suppress == 0), "null argument");
    pick(t, hist_tokens, n_hist_tokens, hist_off, hist_len, suppress, n_suppress, repetition_penalty, no_repeat_ngram_size,
         max_consecutive, wait_token_id, picks_out, value_out);
    WLK_API_END
}
int wlk_qtext_generate_full(wlk_qtext* t, const int32_t* sids, int32_t n, const int32_t* row_src, const int32_t* row_offsets,
                            const float* embeds, int64_t embeds_ld, int32_t n_embeds, int32_t max_new_tokens,
                            const int32_t* stop_ids, int32_t n_stop, const int32_t* suppress, int32_t n_suppress,
                            float repetition_penalty, int32_t no_repeat_ngram_size, int32_t max_consecutive,
                            int32_t wait_token_id, int32_t* tokens_out, int32_t* n_tokens_out) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(sids && row_src && row_offsets && (embeds || n_embeds == 0) && (stop_ids || n_stop == 0) &&
              (suppress || n_suppress == 0) && (tokens_out || max_new_tokens <= 0) && n_tokens_out, "null argument");
    WLK_CHECK(embeds_ld == 0 || embeds_ld >= t->dims.d_model, "embeds_ld %lld < d_model %d", (long long)embeds_ld, t->dims.d_model);
    generate_full(t, sids, n, row_src, row_offsets, embeds, n_embeds, embeds_ld, max_new_tokens, stop_ids, n_stop, suppress,
                  n_suppress, repetition_penalty, no_repeat_ngram_size, max_consecutive, wait_token_id, tokens_out, n_tokens_out);
    WLK_API_END
}
int wlk_qtext_generate_rolling(wlk_qtext* t, const int32_t* sids, int32_t n, const int32_t* row_src, const int32_t* row_offsets,
                               const float* embeds, int64_t embeds_ld, int32_t n_embeds, const int32_t* draft_len,
                               const int32_t* prefix_len, int32_t tail_len, int32_t max_new_tokens, const int32_t* stop_ids,
                               int32_t n_stop, const int32_t* suppress, int32_t n_suppress, float repetition_penalty,
                               int32_t no_repeat_ngram_size, int32_t max_consecutive, int32_t wait_token_id,
                               int32_t* tokens_out, int32_t* n_tokens_out, int32_t* stats_out) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(sids && row_src && row_offsets && (embeds || n_embeds == 0) && draft_len && prefix_len &&
              (stop_ids || n_stop == 0) && (suppress || n_suppress == 0) && tokens_out && n_tokens_out && stats_out,
              "null argument");
    WLK_CHECK(embeds_ld == 0 || embeds_ld >= t->dims.d_model, "embeds_ld %lld < d_model %d", (long long)embeds_ld, t->dims.d_model);
    generate_rolling(t, sids, n, row_src, row_offsets, embeds, n_embeds, embeds_ld, draft_len, prefix_len, tail_len,
                     max_new_tokens, stop_ids, n_stop, suppress, n_suppress, repetition_penalty, no_repeat_ngram_size,
                     max_consecutive, wait_token_id, tokens_out, n_tokens_out, stats_out);
    WLK_API_END
}
int wlk_qtext_logits(wlk_qtext* t, int32_t row0, int32_t n_rows, float* out_host) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    WLK_CHECK(out_host || n_rows == 0, "null output buffer");
    logits_out(t, row0, n_rows, out_host);
    WLK_API_END
}
int wlk_qtext_op_rmsnorm(wlk_qtext* t, const float* x, const float* w, void* out, int32_t rows, const int32_t* out_row_host) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    op_rmsnorm(t, x, w, out, rows, out_row_host);
    WLK_API_END
}
int wlk_qtext_op_qk_rope(wlk_qtext* t, const float* qkv, const float* q_norm_w, const float* k_norm_w, const int32_t* row_pos_host,
                         const int32_t* row_slot_host, int32_t rows, void* const* kv_ptrs_host, int32_t n_slots, int32_t layer,
                         void* q_out) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    op_qk_rope(t, qkv, q_norm_w, k_norm_w, row_pos_host, row_slot_host, rows, kv_ptrs_host, n_slots, layer, q_out);
    WLK_API_END
}
int wlk_qtext_op_attention(wlk_qtext* t, const void* q, const int32_t* row_pos_host, const int32_t* row_slot_host, int32_t rows,
                           void* const* kv_ptrs_host, int32_t n_slots, int32_t layer, void* out) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    op_attention(t, q, row_pos_host, row_slot_host, rows, kv_ptrs_host, n_slots, layer, out);
    WLK_API_END
}
int wlk_qtext_op_swiglu(wlk_qtext* t, const float* gu, void* hid, int32_t rows) {
    WLK_API_BEGIN
    WLK_ENTER(t, t->cfg.device);
    op_swiglu(t, gu, hid, rows);
    WLK_API_END
}

}  // extern "C"
