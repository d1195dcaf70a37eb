// Streaming Sortformer diarizer forward on the device (SURVEY.md section 8 row a16), behind the C ABI wlk_sf_* of
// include/wlk_b200.h.  Reference call sites: whisperlivekit/diarization/sortformer_backend.py
//   :120-126 streaming parameters, :175-196 mel front end (window 0.025 s, n_fft 512, 128 mels, normalize "NA"),
//   :212-234 per-stream state (fixed-size speaker cache / FIFO + lengths = NeMo's async layout),
//   :253-311 diarize(): 1.0 s of audio -> 101 mel frames (+ the previous chunk's last 99) -> forward_streaming_step.
// The arithmetic itself is NeMo's (3.0.0, absent from both containers); it is restated in oracle/sortformer_oracle.py
// (PARITY UNPINNED: never checked against NeMo) and this file follows that restatement:
//   front end   FilterbankFeatures: pre-emphasis 0.97, reflect-padded 512-point STFT with a centred 400-sample Hann
//               window, power, Slaney mel bank, log(x + 2^-24)
//   pre_encode  ConvSubsampling(dw_striding, 8x): conv2d 1->C k3 s2 + ReLU, 2 x (depthwise k3 s2, pointwise 1x1, ReLU),
//               Linear(C * n_mels/8 -> d_model)
//   encoder     17 FastConformer blocks over [speaker cache | FIFO | chunk] rows of each stream: half-step FF (SiLU),
//               Transformer-XL relative-position attention with untied biases, conv module (pointwise, GLU, depthwise k9,
//               BatchNorm(eval), SiLU, pointwise), half-step FF, LayerNorm
//   head        Linear(d_model -> 192), 18 post-LN Transformer blocks (ReLU FF), ReLU-Linear-ReLU-Linear-sigmoid
//   update      SortformerModules.streaming_update_async + _compress_spkcache for every stream (one CTA per stream)
// Streams are batched by packing their ragged sequences (<= spkcache + fifo + 25 rows each) into one row buffer: every
// GEMM of a step sees all streams of the call; attention, the conv module and the cache update run per stream.
// GEMMs go through the engine's wgmma / SIMT GEMM kernels (bf16 mode / fp32 parity mode); everything else is here.
#include <math.h>

#include <map>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/wlk_b200.h"
#include "host.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

namespace wlk {
namespace {

constexpr int SF_TP_CAP = 4096;         // rows of device-resident total_preds kept per session
constexpr int SF_TP_KEEP = 1024;        // tail kept when the buffer is trimmed (sortformer_backend.py:301-305)
constexpr float SF_LOG_GUARD = 5.9604644775390625e-08f;      // 2^-24
constexpr int SF_MAX_T = 512;           // rows of one stream's sequence (attention scratch is sized by it)

struct SfJob {                          // one per stream of a step (device array)
    const float* cache_cur; const float* fifo_cur;             // [spkcache_len][D], [fifo_len][D] fp32 (valid prefixes)
    float* cache_next; float* fifo_next;
    const float* cache_preds_cur; float* cache_preds_next;     // [spkcache_len][S]
    float* fifo_preds_next;                                    // [fifo_len][S]
    float* mean_sil;                                           // [D]
    int32_t* n_sil;                                            // [1]
    float* total_preds;                                        // append position of this step's chunk_preds
    float* prev_mel;                                           // [frames_per_chunk][n_mels]
    const float* pcm;                                          // this step's samples (device)
    int32_t n_samples, n_new_frames;                           // frames the samples give (n / hop + 1)
    int32_t has_prev;                                          // the previous chunk's last `prev_keep` frames lead the features
    int32_t feat_off, n_feat;                                  // rows of the feature buffer
    int32_t t1_off, t2_off, t3_off, T1, T2, T3;                // conv stem rows (time) per stage
    int32_t row_off, T;                                        // the stream's sequence in the packed row buffers
    int32_t sl, fl;                                            // valid speaker-cache / FIFO rows before the step
    int32_t lc, rc, max_chunk, clen;                           // streaming_update_async bookkeeping (host-mirrored)
    int32_t do_pop, pop, compress;
    int32_t out_off;                                           // row of chunk_preds in the step's output buffer
};

__device__ __forceinline__ float sigmoid_(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float silu_(float x) { return x / (1.0f + expf(-x)); }

// ---------------------------------------------------------------------------------------------------------------
// front end.  grid (frame, stream), 288 threads: thread k < 257 owns frequency bin k.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(288)
sf_mel_kernel(const SfJob* __restrict__ jobs, const float* __restrict__ window /*[win]*/, const float2* __restrict__ twiddle /*[n_fft]*/,
              const float* __restrict__ fbT /*[n_freq][n_mels]*/, const int2* __restrict__ span, float* __restrict__ feats,
              int n_fft, int win_len, int hop, int n_mels, int prev_keep) {
    extern __shared__ float sm[];
    float* xs = sm;                               // [win_len]
    float2* tw = reinterpret_cast<float2*>(xs + ((win_len + 3) & ~3));      // [n_fft]
    float* pw = reinterpret_cast<float*>(tw + n_fft);                        // [n_freq]
    const SfJob job = jobs[blockIdx.y];
    const int t = blockIdx.x;
    if (t >= job.n_new_frames) return;
    const int n_freq = n_fft / 2 + 1, N = job.n_samples;
    const int lead = (n_fft - win_len) / 2;       // the window sits centred in the n_fft frame (torch.stft)
    for (int i = threadIdx.x; i < n_fft; i += blockDim.x) tw[i] = twiddle[i];
    for (int i = threadIdx.x; i < win_len; i += blockDim.x) {
        int o = t * hop + lead + i - n_fft / 2;   // index into the pre-emphasised signal, reflect-padded by n_fft / 2
        if (o < 0) o = -o;
        if (o >= N) o = 2 * (N - 1) - o;
        const float v = o == 0 ? job.pcm[0] : job.pcm[o] - 0.97f * job.pcm[o - 1];
        xs[i] = v * window[i];
    }
    __syncthreads();
    const int k = threadIdx.x;
    if (k < n_freq) {
        float re = 0.f, im = 0.f;
        int idx = (k * lead) & (n_fft - 1);
        for (int i = 0; i < win_len; ++i) {
            const float2 w = tw[idx];
            re = fmaf(xs[i], w.x, re);
            im = fmaf(xs[i], w.y, im);
            idx = (idx + k) & (n_fft - 1);
        }
        pw[k] = re * re + im * im;
    }
    __syncthreads();
    for (int m = threadIdx.x; m < n_mels; m += blockDim.x) {
        const int2 sp = span[m];
        float acc = 0.f;
        for (int f = sp.x; f < sp.y; ++f) acc = fmaf(fbT[(int64_t)f * n_mels + m], pw[f], acc);
        const float v = logf(acc + SF_LOG_GUARD);
        const int lead_rows = job.has_prev ? prev_keep : 0;
        feats[(int64_t)(job.feat_off + lead_rows + t) * n_mels + m] = v;
        job.prev_mel[(int64_t)t * n_mels + m] = v;
    }
}

// the previous chunk's last `prev_keep` frames lead this step's features (sortformer_backend.py:277-283); runs BEFORE the
// mel kernel overwrites prev_mel.  grid (prev_keep, stream)
__global__ void sf_prev_feats_kernel(const SfJob* __restrict__ jobs, float* __restrict__ feats, int n_mels, int prev_keep,
                                     int frames_per_chunk) {
    const SfJob job = jobs[blockIdx.y];
    if (!job.has_prev) return;
    const int r = blockIdx.x;
    const float* src = job.prev_mel + (int64_t)(frames_per_chunk - prev_keep + r) * n_mels;
    float* dst = feats + (int64_t)(job.feat_off + r) * n_mels;
    for (int m = threadIdx.x; m < n_mels; m += blockDim.x) dst[m] = src[m];
}

// ---------------------------------------------------------------------------------------------------------------
// conv stem.  Activations are [time][freq][channel] (channels last) so the pointwise convolutions are plain GEMMs over
// (time, freq) rows and the final Linear reads rows of F * C.
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void sf_conv0_kernel(const SfJob* __restrict__ jobs, const float* __restrict__ feats, const float* __restrict__ w /*[C][3][3]*/,
                                const float* __restrict__ b, T* __restrict__ out, int n_mels, int C) {
    const SfJob job = jobs[blockIdx.y];
    const int F1 = (n_mels - 1) / 2 + 1;
    const int64_t total = (int64_t)job.T1 * F1 * C;
    const float* x = feats + (int64_t)job.feat_off * n_mels;
    T* o = out + (int64_t)job.t1_off * F1 * C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = i % C;
        int64_t r = i / C;
        const int f = r % F1;
        const int t = r / F1;
        float acc = b[c];
#pragma unroll
        for (int kt = 0; kt < 3; ++kt) {
            const int tt = 2 * t - 1 + kt;
            if (tt < 0 || tt >= job.n_feat) continue;
#pragma unroll
            for (int kf = 0; kf < 3; ++kf) {
                const int ff = 2 * f - 1 + kf;
                if (ff < 0 || ff >= n_mels) continue;
                acc = fmaf(w[c * 9 + kt * 3 + kf], x[(int64_t)tt * n_mels + ff], acc);
            }
        }
        o[i] = from_f32<T>(fmaxf(acc, 0.f));
    }
}

// depthwise 3x3 / stride 2 / pad 1 over [Ti][Fi][C] -> [To][Fo][C];  stage 1: rows t1 -> t2, stage 2: t2 -> t3
template <typename T>
__global__ void sf_dwconv_kernel(const SfJob* __restrict__ jobs, int stage, const T* __restrict__ in, const float* __restrict__ w,
                                 const float* __restrict__ b, T* __restrict__ out, int Fi, int C) {
    const SfJob job = jobs[blockIdx.y];
    const int Ti = stage == 1 ? job.T1 : job.T2, To = stage == 1 ? job.T2 : job.T3;
    const int ioff = stage == 1 ? job.t1_off : job.t2_off, ooff = stage == 1 ? job.t2_off : job.t3_off;
    const int Fo = (Fi - 1) / 2 + 1;
    const int64_t total = (int64_t)To * Fo * C;
    const T* x = in + (int64_t)ioff * Fi * C;
    T* o = out + (int64_t)ooff * Fo * C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = i % C;
        int64_t r = i / C;
        const int f = r % Fo;
        const int t = r / Fo;
        float acc = b[c];
#pragma unroll
        for (int kt = 0; kt < 3; ++kt) {
            const int tt = 2 * t - 1 + kt;
            if (tt < 0 || tt >= Ti) continue;
#pragma unroll
            for (int kf = 0; kf < 3; ++kf) {
                const int ff = 2 * f - 1 + kf;
                if (ff < 0 || ff >= Fi) continue;
                acc = fmaf(w[c * 9 + kt * 3 + kf], to_f32(x[((int64_t)tt * Fi + ff) * C + c]), acc);
            }
        }
        o[i] = from_f32<T>(acc);
    }
}

// rows of each stream's sequence: x = xscale * [speaker cache | FIFO | chunk].  grid (SF_MAX_T, stream)
__global__ void sf_assemble_kernel(const SfJob* __restrict__ jobs, const float* __restrict__ chunk /*[sum T3][D]*/, float* __restrict__ x,
                                   int D, float xscale) {
    const SfJob job = jobs[blockIdx.y];
    const int r = blockIdx.x;
    if (r >= job.T) return;
    const float* src = r < job.sl ? job.cache_cur + (int64_t)r * D
                     : r < job.sl + job.fl ? job.fifo_cur + (int64_t)(r - job.sl) * D
                                           : chunk + (int64_t)(job.t3_off + r - job.sl - job.fl) * D;
    float* dst = x + (int64_t)(job.row_off + r) * D;
    for (int i = threadIdx.x; i < D; i += blockDim.x) dst[i] = src[i] * xscale;
}

// ---------------------------------------------------------------------------------------------------------------
// attention over one stream's rows.  qkv [rows][3 d] (q | k | v; head h at columns h * dh).  RELPOS: Transformer-XL
// scores ((q + u) k_j + (q + v) p_{i-j}) / sqrt(dh), p from the per-layer table ptab[(center - (i - j))][d];
// otherwise plain softmax(q k^T) (q, k pre-scaled by the QKV GEMM).  Block = 4 warps x 4 queries; a lane owns keys
// lane, lane + 32, ... for the scores and two output dims for P V.  fp32 softmax.
// ---------------------------------------------------------------------------------------------------------------
template <typename T, bool RELPOS>
__global__ void __launch_bounds__(128)
sf_attention_kernel(const T* __restrict__ qkv, const SfJob* __restrict__ jobs, int n_head, int d, int dh,
                    const T* __restrict__ ptab, int center, const float* __restrict__ bias_u, const float* __restrict__ bias_v,
                    float score_scale, T* __restrict__ out) {
    constexpr int QPB = 16, MAXK = SF_MAX_T / 32;
    __shared__ float qs[QPB][2][64];
    __shared__ float ps[4][SF_MAX_T];
    const SfJob job = jobs[blockIdx.z];
    const int h = blockIdx.y, q0 = blockIdx.x * QPB;
    if (q0 >= job.T) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t ld = 3 * (int64_t)d;
    const T* base = qkv + (int64_t)job.row_off * ld + h * dh;
    for (int i = threadIdx.x; i < QPB * dh; i += 128) {
        const int qi = i / dh, e = i - qi * dh;
        float v = 0.f;
        if (q0 + qi < job.T) v = to_f32(base[(int64_t)(q0 + qi) * ld + e]);
        qs[qi][0][e] = RELPOS ? v + bias_u[h * dh + e] : v;
        qs[qi][1][e] = RELPOS ? v + bias_v[h * dh + e] : 0.f;
    }
    __syncthreads();
    for (int qq = 0; qq < QPB / 4; ++qq) {
        const int qi = warp * (QPB / 4) + qq, i = q0 + qi;
        if (i >= job.T) break;                                  // warp-uniform
        float sc[MAXK];
        float mx = -INFINITY;
#pragma unroll
        for (int m = 0; m < MAXK; ++m) {
            const int j = lane + 32 * m;
            sc[m] = -INFINITY;
            if (j < job.T) {
                const T* kr = base + (int64_t)j * ld + d;
                float acc = 0.f;
                for (int e = 0; e < dh; ++e) acc = fmaf(qs[qi][0][e], to_f32(kr[e]), acc);
                if (RELPOS) {
                    const T* pr = ptab + (int64_t)(center - (i - j)) * d + h * dh;
                    for (int e = 0; e < dh; ++e) acc = fmaf(qs[qi][1][e], to_f32(pr[e]), acc);
                }
                sc[m] = acc * score_scale;
                mx = fmaxf(mx, sc[m]);
            }
        }
        mx = warp_max(mx);
        float sum = 0.f;
#pragma unroll
        for (int m = 0; m < MAXK; ++m) {
            const int j = lane + 32 * m;
            if (j < job.T) { const float p = expf(sc[m] - mx); ps[warp][j] = p; sum += p; }
        }
        sum = warp_sum(sum);
        __syncwarp();
        const float inv = 1.0f / sum;
        for (int e0 = 2 * lane; e0 < dh; e0 += 64) {            // dh <= 64: one pass
            float a0 = 0.f, a1 = 0.f;
            const T* vr = base + 2 * (int64_t)d + e0;
            for (int j = 0; j < job.T; ++j) {
                const float p = ps[warp][j];
                a0 = fmaf(p, to_f32(vr[(int64_t)j * ld]), a0);
                a1 = fmaf(p, to_f32(vr[(int64_t)j * ld + 1]), a1);
            }
            T* o = out + (int64_t)(job.row_off + i) * d + h * dh + e0;
            o[0] = from_f32<T>(a0 * inv);
            o[1] = from_f32<T>(a1 * inv);
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------------------------
// bf16 mode: the same attention on warp-level tensor-core MMAs (mma.sync m16n8k16, bf16 operands, fp32 accumulate).
// The diarizer is ~2 % of a config-4 stream's FLOPs, its sequences are <= 401 rows and the relative-position term needs
// a per-row shift of the score tile, so a 16-query CTA with the scores staged in shared memory is the shape that fits;
// the wgmma pipeline of attn_tc.cu is reserved for the 1500-position Whisper encoder.
//   block = 16 queries of one (stream, head), 4 warps:
//     S[i][j]  = (q_i + u) . k_j                     warps split the 8-key column tiles          -> smem fp32
//     S[i][j] += (q_i + v) . p[c - (i - j)]          computed as a dense 16 x (T + 15) tile over the positions the block
//                                                    can touch, each element added at its shifted column (rel_shift)
//     P = exp(S * scale - max), row sums             a warp per 4 rows; P overwrites the row in place as bf16
//     O = P V / sum                                  warps split the 8-wide output column tiles
// ---------------------------------------------------------------------------------------------------------------

template <bool RELPOS>
__global__ void __launch_bounds__(128)
sf_attention_mma_kernel(const bf16* __restrict__ qkv, const SfJob* __restrict__ jobs, int n_head, int d, int dh,
                        const bf16* __restrict__ ptab, int center, const float* __restrict__ bias_u, const float* __restrict__ bias_v,
                        float score_scale, bf16* __restrict__ out) {
    constexpr int SP = SF_MAX_T + 8;                    // row pitch of S in floats (bank-friendly for the fragment loads)
    __shared__ float S[16][SP];
    __shared__ bf16 qs[2][16][72];                      // (q + u), (q + v), zero-padded to 64 columns
    __shared__ float rowinv[16];
    const SfJob job = jobs[blockIdx.z];
    const int h = blockIdx.y, i0 = blockIdx.x * 16, T = job.T;
    if (i0 >= T) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int64_t ld = 3 * (int64_t)d;
    const bf16* base = qkv + (int64_t)job.row_off * ld + h * dh;
    const bf16 zero = __float2bfloat16_rn(0.f);
    for (int i = threadIdx.x; i < 16 * 64; i += 128) {
        const int qi = i >> 6, e = i & 63;
        float v = 0.f;
        const bool live = e < dh && i0 + qi < T;
        if (live) v = to_f32(base[(int64_t)(i0 + qi) * ld + e]);
        qs[0][qi][e] = live ? __float2bfloat16_rn(RELPOS ? v + bias_u[h * dh + e] : v) : zero;
        qs[1][qi][e] = live && RELPOS ? __float2bfloat16_rn(v + bias_v[h * dh + e]) : zero;
    }
    __syncthreads();
    const int ksteps = (dh + 15) / 16;
    uint32_t au[4][4], av[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        if (ks < ksteps) {
            const int c0 = 16 * ks + 2 * t;
            au[ks][0] = *reinterpret_cast<const uint32_t*>(&qs[0][g][c0]);     au[ks][1] = *reinterpret_cast<const uint32_t*>(&qs[0][g + 8][c0]);
            au[ks][2] = *reinterpret_cast<const uint32_t*>(&qs[0][g][c0 + 8]); au[ks][3] = *reinterpret_cast<const uint32_t*>(&qs[0][g + 8][c0 + 8]);
            if (RELPOS) {
                av[ks][0] = *reinterpret_cast<const uint32_t*>(&qs[1][g][c0]);     av[ks][1] = *reinterpret_cast<const uint32_t*>(&qs[1][g + 8][c0]);
                av[ks][2] = *reinterpret_cast<const uint32_t*>(&qs[1][g][c0 + 8]); av[ks][3] = *reinterpret_cast<const uint32_t*>(&qs[1][g + 8][c0 + 8]);
            }
        }
    }
    // B fragment of a K-major row (key / position row `r`, columns 16 ks + 2t (+1) and + 8): zero past dh or when !ok
    auto bfrag = [&](const bf16* row, bool ok, int ks, uint32_t& b0, uint32_t& b1) {
        const int c0 = 16 * ks + 2 * t;
        b0 = ok && c0 < dh ? *reinterpret_cast<const uint32_t*>(row + c0) : 0u;
        b1 = ok && c0 + 8 < dh ? *reinterpret_cast<const uint32_t*>(row + c0 + 8) : 0u;
    };
    // ---- content term
    const int ntiles = (T + 7) / 8;
    for (int nt = warp; nt < ntiles; nt += 4) {
        const int j = 8 * nt + g;
        const bool ok = j < T;
        const bf16* kr = base + (int64_t)(ok ? j : 0) * ld + d;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            if (ks < ksteps) { uint32_t b0, b1; bfrag(kr, ok, ks, b0, b1); ptx::mma_bf16_16816(acc, au[ks], b0, b1); }
        }
        const int c = 8 * nt + 2 * t;
        S[g][c] = acc[0] * score_scale; S[g][c + 1] = acc[1] * score_scale;
        S[g + 8][c] = acc[2] * score_scale; S[g + 8][c + 1] = acc[3] * score_scale;
    }
    __syncthreads();
    if (RELPOS) {
        // positions the block can touch: table rows idx_lo .. idx_lo + T + 14, idx = center - (i - j)
        const int idx_lo = center - i0 - 15;
        const int mtiles = (T + 15 + 7) / 8;
        for (int mt = warp; mt < mtiles; mt += 4) {
            const int m = 8 * mt + g;
            const bool ok = m < T + 15;
            const bf16* pr = ptab + (int64_t)(idx_lo + (ok ? m : 0)) * d + h * dh;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                if (ks < ksteps) { uint32_t b0, b1; bfrag(pr, ok, ks, b0, b1); ptx::mma_bf16_16816(acc, av[ks], b0, b1); }
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int ii = g + (e >> 1) * 8, mm = 8 * mt + 2 * t + (e & 1);
                const int j = mm - 15 + ii;                      // rel_shift: column of S this position lands in for row ii
                if (j >= 0 && j < T) S[ii][j] += acc[e] * score_scale;
            }
        }
        __syncthreads();
    }
    // ---- softmax; P (unnormalised, bf16) overwrites the row in place
    const int Tp = (T + 15) & ~15;
    for (int rr = 0; rr < 4; ++rr) {
        const int row = warp * 4 + rr;
        float v[SF_MAX_T / 32];
        float mx = -INFINITY;
#pragma unroll
        for (int k = 0; k < SF_MAX_T / 32; ++k) {
            const int j = lane + 32 * k;
            v[k] = j < T ? S[row][j] : -INFINITY;
            mx = fmaxf(mx, v[k]);
        }
        mx = warp_max(mx);
        float sum = 0.f;
#pragma unroll
        for (int k = 0; k < SF_MAX_T / 32; ++k) { v[k] = lane + 32 * k < T ? expf(v[k] - mx) : 0.f; sum += v[k]; }
        sum = warp_sum(sum);
        __syncwarp();
        bf16* prow = reinterpret_cast<bf16*>(&S[row][0]);
#pragma unroll
        for (int k = 0; k < SF_MAX_T / 32; ++k) { const int j = lane + 32 * k; if (j < Tp) prow[j] = __float2bfloat16_rn(v[k]); }
        if (lane == 0) rowinv[row] = 1.0f / sum;
    }
    __syncthreads();
    // ---- O = P V
    const int otiles = (dh + 7) / 8, kk_n = Tp / 16;
    const bf16* vbase = base + 2 * (int64_t)d;
    for (int ot = warp; ot < otiles; ot += 4) {
        const int n = 8 * ot + g;                                // output column this lane's B fragment feeds
        const bool nok = n < dh;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int kk = 0; kk < kk_n; ++kk) {
            uint32_t a[4];
            const bf16* p0 = reinterpret_cast<const bf16*>(&S[g][0]) + 16 * kk + 2 * t;
            const bf16* p1 = reinterpret_cast<const bf16*>(&S[g + 8][0]) + 16 * kk + 2 * t;
            a[0] = *reinterpret_cast<const uint32_t*>(p0); a[1] = *reinterpret_cast<const uint32_t*>(p1);
            a[2] = *reinterpret_cast<const uint32_t*>(p0 + 8); a[3] = *reinterpret_cast<const uint32_t*>(p1 + 8);
            const int j0 = 16 * kk + 2 * t;
            auto vld = [&](int j) { return nok && j < T ? vbase[(int64_t)j * ld + n] : zero; };
            const uint32_t b0 = ptx::pack_bf16_pair(vld(j0), vld(j0 + 1)), b1 = ptx::pack_bf16_pair(vld(j0 + 8), vld(j0 + 9));
            ptx::mma_bf16_16816(acc, a, b0, b1);
        }
        const int c = 8 * ot + 2 * t;
        if (c < dh) {
            if (i0 + g < T) {
                const float inv = rowinv[g];
                *reinterpret_cast<__nv_bfloat162*>(out + (int64_t)(job.row_off + i0 + g) * d + h * dh + c) = __floats2bfloat162_rn(acc[0] * inv, acc[1] * inv);
            }
            if (i0 + g + 8 < T) {
                const float inv = rowinv[g + 8];
                *reinterpret_cast<__nv_bfloat162*>(out + (int64_t)(job.row_off + i0 + g + 8) * d + h * dh + c) = __floats2bfloat162_rn(acc[2] * inv, acc[3] * inv);
            }
        }
    }
}

// conv module middle: GLU over the 2 D columns of the pointwise output, depthwise k-tap conv along the stream's own rows
// (zero padding at the sequence ends), folded BatchNorm (y = A conv + B), SiLU.  grid (ceil(SF_MAX_T / 16), stream, D / 128)
template <typename T>
__global__ void __launch_bounds__(128)
sf_glu_dwconv_kernel(const T* __restrict__ in /*[rows][2D]*/, const SfJob* __restrict__ jobs, const float* __restrict__ w /*[D][K]*/,
                     const float* __restrict__ bnA, const float* __restrict__ bnB, T* __restrict__ out /*[rows][D]*/, int D, int K) {
    constexpr int TT = 16, KMAX = 16;
    __shared__ float g[TT + KMAX][128];
    const SfJob job = jobs[blockIdx.y];
    const int t0 = blockIdx.x * TT;
    if (t0 >= job.T) return;
    const int c = blockIdx.z * 128 + threadIdx.x, pad = (K - 1) / 2;
    const bool live = c < D;
    for (int r = 0; r < TT + K - 1; ++r) {
        const int t = t0 - pad + r;
        float v = 0.f;
        if (live && t >= 0 && t < job.T) {
            const T* row = in + (int64_t)(job.row_off + t) * 2 * D;
            v = to_f32(row[c]) * sigmoid_(to_f32(row[D + c]));
        }
        g[r][threadIdx.x] = v;
    }
    if (!live) return;
    float wk[KMAX];
    for (int k = 0; k < K; ++k) wk[k] = w[c * K + k];
    const float A = bnA[c], B = bnB[c];
    for (int r = 0; r < TT && t0 + r < job.T; ++r) {
        float acc = 0.f;
        for (int k = 0; k < K; ++k) acc = fmaf(wk[k], g[r + k][threadIdx.x], acc);
        out[(int64_t)(job.row_off + t0 + r) * D + c] = from_f32<T>(silu_(fmaf(A, acc, B)));
    }
}

template <typename T>
__global__ void sf_relu_kernel(const float* __restrict__ x, T* __restrict__ out, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = from_f32<T>(fmaxf(x[i], 0.f));
}

// sigmoid(W h + b), W [S][d]: warp per row
template <typename T>
__global__ void sf_spk_kernel(const T* __restrict__ h, const float* __restrict__ W, const float* __restrict__ b, float* __restrict__ preds,
                              int rows, int d, int S) {
    const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (row >= rows) return;
    for (int s = 0; s < S; ++s) {
        float acc = 0.f;
        for (int e = lane; e < d; e += 32) acc = fmaf(W[s * d + e], to_f32(h[(int64_t)row * d + e]), acc);
        acc = warp_sum(acc);
        if (lane == 0) preds[(int64_t)row * S + s] = sigmoid_(acc + b[s]);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// SortformerModules.streaming_update_async + _compress_spkcache, one CTA (256 threads) per stream.  Lengths and branch
// decisions do not depend on data and arrive precomputed in the job (host mirror); the data-dependent parts -- silence
// profile, scores, the three top-k selections and the sort -- run here.  Reads the *_cur buffers and the step's chunk /
// preds rows, writes the *_next buffers: no in-place hazards.
// ---------------------------------------------------------------------------------------------------------------
struct SfUpd {
    int D, S, CL, FL, sil_per_spk, n_cache;      // n_cache = CL + max_pop rows of NeMo's updated_spkcache
    float th, boost_latest, sil_th;
    int strong, weak, min_pos;
};

__global__ void __launch_bounds__(256)
sf_update_kernel(const SfJob* __restrict__ jobs, const float* __restrict__ chunk /*[sum T3][D]*/, const float* __restrict__ preds /*[rows][S]*/,
                 float* __restrict__ out_preds, SfUpd U) {
    extern __shared__ float sm[];
    const SfJob job = jobs[blockIdx.x];
    const int D = U.D, S = U.S, tid = threadIdx.x;
    const int sl = job.sl, fl = job.fl, clen = job.clen, pop = job.do_pop ? job.pop : 0;
    const float* P = preds + (int64_t)job.row_off * S;
    const float* Pf = P + (int64_t)sl * S;                          // fifo_preds[:fl] = preds[sl : sl + fl]
    const float* Pc = P + (int64_t)(sl + fl + job.lc) * S;          // chunk_preds[:clen]
    const float* chunk_rows = chunk + (int64_t)(job.t3_off + job.lc) * D;
    // row r of NeMo's updated_fifo (before the pop): the old FIFO, then the chunk
    auto up_fifo_row = [&](int r) -> const float* { return r < fl ? job.fifo_cur + (int64_t)r * D : chunk_rows + (int64_t)(r - fl) * D; };
    auto up_fifo_pred = [&](int r) -> const float* { return r < fl ? Pf + (int64_t)r * S : Pc + (int64_t)(r - fl) * S; };
    // row r of updated_spkcache: the old cache, then the popped FIFO rows
    auto up_cache_row = [&](int r) -> const float* { return r < sl ? job.cache_cur + (int64_t)r * D : up_fifo_row(r - sl); };

    // chunk_preds: the step's output and the tail of total_preds
    for (int i = tid; i < job.max_chunk * S; i += 256) {
        const float v = i < clen * S ? Pc[i] : 0.f;
        out_preds[(int64_t)job.out_off * S + i] = v;
        job.total_preds[i] = v;
    }
    // silence profile of the popped rows (_get_silence_profile)
    __shared__ int s_cnt;
    __shared__ float s_nsil_old;
    float* flag = sm;                                               // [n_cache] is_sil of the popped rows, later reused
    if (tid == 0) { s_cnt = 0; s_nsil_old = (float)*job.n_sil; }
    __syncthreads();
    if (pop > 0) {
        for (int r = tid; r < pop; r += 256) {
            const float* p = up_fifo_pred(r);
            float s = 0.f;
            for (int k = 0; k < S; ++k) s += p[k];
            const int is = s < U.sil_th;
            flag[r] = (float)is;
            if (is) atomicAdd(&s_cnt, 1);
        }
        __syncthreads();
        const int cnt = s_cnt;
        if (cnt > 0) {
            const float n_old = s_nsil_old, n_new = n_old + (float)cnt;
            for (int c = tid; c < D; c += 256) {
                float acc = 0.f;
                for (int r = 0; r < pop; ++r) if (flag[r] != 0.f) acc += up_fifo_row(r)[c];
                job.mean_sil[c] = (job.mean_sil[c] * n_old + acc) / fmaxf(n_new, 1.f);
            }
            if (tid == 0) *job.n_sil += cnt;
        }
        __syncthreads();
    }
    // new FIFO = updated_fifo[pop : pop + new_fl], zero behind it
    const int new_fl = fl + clen - pop;
    for (int r = 0; r < U.FL; ++r) {
        float* dst = job.fifo_next + (int64_t)r * D;
        if (r < new_fl) { const float* src = up_fifo_row(pop + r); for (int c = tid; c < D; c += 256) dst[c] = src[c]; }
        else for (int c = tid; c < D; c += 256) dst[c] = 0.f;
    }
    for (int i = tid; i < U.FL * S; i += 256) {
        const int r = i / S;
        job.fifo_preds_next[i] = r < new_fl ? up_fifo_pred(pop + r)[i - r * S] : 0.f;
    }
    const int sl2 = sl + pop;
    if (!job.compress) {
        for (int r = 0; r < U.CL; ++r) {
            float* dst = job.cache_next + (int64_t)r * D;
            if (r < sl2) { const float* src = up_cache_row(r); for (int c = tid; c < D; c += 256) dst[c] = src[c]; }
            else for (int c = tid; c < D; c += 256) dst[c] = 0.f;
        }
        for (int i = tid; i < U.CL * S; i += 256) {
            const int r = i / S;
            job.cache_preds_next[i] = r < sl ? job.cache_preds_cur[i] : r < sl2 ? up_fifo_pred(r - sl)[i - r * S] : 0.f;
        }
        return;
    }
    // ---- _compress_spkcache over n = n_cache rows (rows >= sl2 are zero: never speech)
    const int n = U.n_cache, nf = n + U.sil_per_spk;               // frames incl. the +inf silence pads
    float* pr = sm;                                                  // [n][S] updated_spkcache_preds
    float* sc = pr + n * S;                                          // [S][nf] scores, speaker-major (the flatten order)
    int* rank = reinterpret_cast<int*>(sc + S * nf);                 // [S][nf]
    int* sel = rank + S * nf;                                        // [CL] selected keys
    __shared__ int s_pos[8];
    __shared__ int s_nsel;
    __syncthreads();
    for (int i = tid; i < n * S; i += 256) {
        const int r = i / S;
        pr[i] = r < sl ? job.cache_preds_cur[i] : r < sl2 ? up_fifo_pred(r - sl)[i - r * S] : 0.f;
    }
    if (tid < 8) s_pos[tid] = 0;
    __syncthreads();
    const float NEG = -INFINITY;
    for (int r = tid; r < n; r += 256) {                            // _get_log_pred_scores + speech mask
        float l1s = 0.f;
        for (int k = 0; k < S; ++k) l1s += logf(fmaxf(1.0f - pr[r * S + k], U.th));
        for (int k = 0; k < S; ++k) {
            const float p = pr[r * S + k];
            float v = logf(fmaxf(p, U.th)) - logf(fmaxf(1.0f - p, U.th)) + l1s + 0.69314718055994531f;
            if (!(p > 0.5f)) v = NEG;
            sc[k * nf + r] = v;
            if (v > 0.f) atomicAdd(&s_pos[k], 1);
        }
    }
    __syncthreads();
    for (int i = tid; i < n * S; i += 256) {                        // _disable_low_scores, scores_boost_latest
        const int k = i / n, r = i - k * n;
        float v = sc[k * nf + r];
        if (v != NEG && !(v > 0.f) && s_pos[k] >= U.min_pos) v = NEG;
        if (r >= U.CL) v += U.boost_latest;
        sc[k * nf + r] = v;
    }
    __syncthreads();
    // _boost_topk_scores twice: rank within the speaker's column (ties: lower frame first)
    for (int pass = 0; pass < 2; ++pass) {
        const int kb = min(pass == 0 ? U.strong : U.weak, n);
        const float add = (pass == 0 ? 2.0f : 1.0f) * 0.69314718055994531f;
        for (int i = tid; i < n * S; i += 256) {
            const int k = i / n, r = i - k * n;
            const float v = sc[k * nf + r];
            int rk = 0;
            for (int r2 = 0; r2 < n; ++r2) { const float v2 = sc[k * nf + r2]; rk += (v2 > v) || (v2 == v && r2 < r); }
            rank[k * nf + r] = rk;
        }
        __syncthreads();
        for (int i = tid; i < n * S; i += 256) {
            const int k = i / n, r = i - k * n;
            if (rank[k * nf + r] < kb) sc[k * nf + r] += add;
        }
        __syncthreads();
    }
    for (int i = tid; i < U.sil_per_spk * S; i += 256) { const int k = i / U.sil_per_spk; sc[k * nf + n + (i - k * U.sil_per_spk)] = INFINITY; }
    if (tid == 0) s_nsel = 0;
    __syncthreads();
    // _get_topk_indices: the CL largest of the S * nf flattened scores (ties: lower flat index first)
    const int total = S * nf;
    for (int i = tid; i < total; i += 256) {
        const float v = sc[i];
        int rk = 0;
        for (int j = 0; j < total; ++j) { const float v2 = sc[j]; rk += (v2 > v) || (v2 == v && j < i); }
        if (rk < U.CL) {
            const int slot = atomicAdd(&s_nsel, 1);
            sel[slot] = v == NEG ? (1 << 30) + i : i;                // -inf picks sort behind everything: NeMo's max_index
        }
    }
    __syncthreads();
    // sort the selected keys, then gather (_gather_spkcache_and_preds)
    int* order = rank;                                              // [CL] key at sorted position
    for (int a = tid; a < U.CL; a += 256) {
        const int key = sel[a];
        int pos = 0;
        for (int b = 0; b < U.CL; ++b) pos += sel[b] < key;
        order[pos] = key;
    }
    __syncthreads();
    for (int q = 0; q < U.CL; ++q) {
        const int key = order[q];
        const int frame = key >= (1 << 30) ? -1 : key % nf;
        const bool disabled = frame < 0 || frame >= n;
        float* dst = job.cache_next + (int64_t)q * D;
        const float* src = disabled ? job.mean_sil : up_cache_row(frame);
        for (int c = tid; c < D; c += 256) dst[c] = src[c];
        if (tid < S) job.cache_preds_next[q * S + tid] = disabled ? 0.f : pr[frame * S + tid];
    }
}

__global__ void sf_bn_fold_kernel(const float* w, const float* b, const float* mean, const float* var, const float* conv_b, float* A, float* B, int d) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= d) return;
    const float a = w[c] / sqrtf(var[c] + 1e-5f);            // nn.BatchNorm1d eps
    A[c] = a;
    B[c] = b[c] + a * (conv_b[c] - mean[c]);
}

struct SfLayerW {
    void *W_ff1a, *W_ff1b, *W_ff2a, *W_ff2b, *Wqkv, *Wo, *Wpos, *Wpw1, *Wpw2;
    float *b_ff1a, *b_ff1b, *b_ff2a, *b_ff2b, *bqkv, *bo, *bpw1, *bpw2;
    float *ln_ff1w, *ln_ff1b, *ln_attw, *ln_attb, *ln_convw, *ln_convb, *ln_ff2w, *ln_ff2b, *ln_outw, *ln_outb;
    float *bias_u, *bias_v, *dw_w, *dw_b, *bn_w, *bn_b, *bn_mean, *bn_var, *bnA, *bnB;
    void* ptab;          // [2 SF_MAX_T - 1][D] linear_pos(PE(r)), activation type
};
struct SfTLayerW {
    void *Wqkv, *Wo, *W1, *W2;
    float *bqkv, *bo, *b1, *b2, *ln1w, *ln1b, *ln2w, *ln2b;
};

struct SfSession {
    bool open = false;
    float *cache[2] = {nullptr, nullptr}, *fifo[2] = {nullptr, nullptr}, *cache_preds[2] = {nullptr, nullptr}, *fifo_preds = nullptr;
    float *mean_sil = nullptr, *prev_mel = nullptr, *total_preds = nullptr;
    int32_t* n_sil = nullptr;
    int flip = 0, sl = 0, fl = 0, chunk_index = 0, tp_rows = 0;
    bool has_prev = false;
};

}  // namespace
}  // namespace wlk

using namespace wlk;

struct wlk_sf : EngineBase {
    wlk_sf_dims dims{};
    int gemm_backend = WLK_BACKEND_SIMT;
    int F1 = 0, F2 = 0, F3 = 0, frames_per_chunk = 0, prev_keep = 99, chunk_samples = 0, n_freq = 0;
    int max_T = 0, max_T3 = 0, max_feat = 0, max_pop = 0, max_chunk_cap = 0;
    // front end + conv stem
    float *window = nullptr, *fbT = nullptr; float2* twiddle = nullptr; int2* span = nullptr;
    float *c0w = nullptr, *c0b = nullptr, *dw1w = nullptr, *dw1b = nullptr, *dw2w = nullptr, *dw2b = nullptr, *pw1b = nullptr, *pw2b = nullptr, *outb = nullptr;
    void *Wpw1 = nullptr, *Wpw2 = nullptr, *Wout = nullptr;
    std::vector<SfLayerW> L;
    std::vector<SfTLayerW> TL;
    void *Wproj = nullptr, *Wh = nullptr; float *bproj = nullptr, *bh = nullptr, *Wspk = nullptr, *bspk = nullptr;
    float* pe_table = nullptr;          // [2 SF_MAX_T - 1][D] RelPositionalEncoding rows, fp32 (input of the per-layer tables)
    SessionTable<SfSession> sess;
    // workspaces
    float *pcm = nullptr, *feats = nullptr, *chunk = nullptr, *x = nullptr, *y = nullptr, *preds = nullptr, *out_preds = nullptr;
    void *a1 = nullptr, *a2 = nullptr, *a2p = nullptr, *a3 = nullptr, *a3p = nullptr, *xn = nullptr, *qkv = nullptr, *att = nullptr, *hid = nullptr, *cv = nullptr;
    float* out_h = nullptr;
};

namespace {

void gemm(wlk_sf* q, const void* A, int64_t lda, const void* W, int64_t ldw, int M, int N, int K, const float* bias, int act_fn,
          void* C, int c_type, int64_t ldc, const float* residual = nullptr, float scale = 1.f, int scale_cols = 0) {
    GemmArgs g;
    g.A = A; g.a_type = q->act; g.lda = lda; g.W = W; g.w_type = q->act; g.ldw = ldw;
    g.M = M; g.N = N; g.K = K;
    g.epi.bias = bias; g.epi.gelu = act_fn; g.epi.C = C; g.epi.c_type = c_type; g.epi.ldc = ldc;
    g.epi.residual = residual; g.epi.ldr = ldc; g.epi.col_scale = scale; g.epi.scale_cols = scale_cols;
    q->gemm.run(g, q->gemm_backend == WLK_BACKEND_TCGEN05, q->st, q->num_sms);
}

int sub_len(int t) { for (int i = 0; i < 3; ++i) t = (t + 2 - 3) / 2 + 1; return t; }

void finalize(wlk_sf* q) {
    const wlk_sf_dims& D = q->dims;
    q->weights.require_all();
    const int d = D.d_model, P = 2 * SF_MAX_T - 1;
    // RelPositionalEncoding rows for relative positions SF_MAX_T-1 ... -(SF_MAX_T-1); a row depends on its relative
    // position only, so one table serves every sequence length.  linear_pos of it is a constant per layer.
    std::vector<float> pe((size_t)P * d);
    for (int r = 0; r < P; ++r) {
        const double pos = (double)(SF_MAX_T - 1 - r);
        for (int i = 0; i < d; i += 2) {
            const double div = exp((double)i * -(log(10000.0) / d));
            pe[(size_t)r * d + i] = (float)sin(pos * div);
            pe[(size_t)r * d + i + 1] = (float)cos(pos * div);
        }
    }
    q->upload.put(pe.data(), pe.size(), q->pe_table, DT_F32, q->st);
    void* pe_act = q->pe_table;
    void* tmp = nullptr;
    if (q->act != DT_F32) {
        CUDA_CHECK(cudaMalloc(&tmp, (size_t)P * d * q->es()));
        convert_f32_to(q->pe_table, tmp, q->act, (int64_t)P * d, q->st);
        pe_act = tmp;
    }
    for (auto& L : q->L) {
        gemm(q, pe_act, d, L.Wpos, d, P, d, d, nullptr, 0, L.ptab, q->act, d);
        sf_bn_fold_kernel<<<(d + 127) / 128, 128, 0, q->st>>>(L.bn_w, L.bn_b, L.bn_mean, L.bn_var, L.dw_b, L.bnA, L.bnB, d);
    }
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(q->st));
    if (tmp) cudaFree(tmp);
    q->upload.release();
    q->finalized = true;
}

void create(const wlk_sf_dims* dims, const wlk_config* cfg, wlk_sf** out) {
    WLK_CHECK(dims && cfg && out, "null argument");
    const wlk_sf_dims& D = *dims;
    WLK_CHECK(D.n_fft >= 64 && (D.n_fft & (D.n_fft - 1)) == 0 && D.n_fft / 2 + 1 <= 288, "n_fft must be a power of two <= 512");
    WLK_CHECK(D.win_length >= 16 && D.win_length <= D.n_fft && (D.n_fft - D.win_length) % 2 == 0, "bad window length");
    WLK_CHECK(D.n_mels >= 8 && D.n_mels % 8 == 0, "n_mels must be a multiple of 8");
    WLK_CHECK(D.conv_channels % 8 == 0 && D.d_model % 8 == 0 && D.tf_d_model % 8 == 0 && D.tf_inner % 8 == 0, "widths must be multiples of 8");
    WLK_CHECK(D.d_model % D.n_head == 0 && D.d_model / D.n_head <= 64 && (D.d_model / D.n_head) % 8 == 0, "FastConformer heads must be a multiple of 8 and <= 64 wide");
    WLK_CHECK(D.tf_d_model % D.tf_n_head == 0 && D.tf_d_model / D.tf_n_head <= 64 && (D.tf_d_model / D.tf_n_head) % 8 == 0, "Transformer heads must be a multiple of 8 and <= 64 wide");
    WLK_CHECK(D.d_model <= 1280 && D.tf_d_model <= 1280 && D.d_model % 4 == 0 && D.tf_d_model % 4 == 0, "LayerNorm width limit");
    WLK_CHECK(D.conv_kernel >= 1 && D.conv_kernel <= 16 && D.conv_kernel % 2 == 1, "conv_kernel must be odd and <= 15");
    WLK_CHECK(D.n_spk >= 1 && D.n_spk <= 8, "n_spk must be in [1, 8]");
    WLK_CHECK(D.spkcache_len >= D.n_spk * (1 + D.spkcache_sil_frames_per_spk), "speaker cache too short for n_spk");
    WLK_CHECK(cfg->max_sessions >= 1 && cfg->max_batch >= 1, "max_sessions / max_batch must be >= 1");

    auto* q = new wlk_sf();
    q->open(*cfg);
    q->dims = D;
    q->act = cfg->precision == WLK_PREC_BF16 ? DT_BF16 : DT_F32;
    q->gemm_backend = q->act == DT_BF16 && cfg->gemm_backend != WLK_BACKEND_SIMT ? WLK_BACKEND_TCGEN05 : WLK_BACKEND_SIMT;
    q->n_freq = D.n_fft / 2 + 1;
    q->F1 = (D.n_mels - 1) / 2 + 1; q->F2 = (q->F1 - 1) / 2 + 1; q->F3 = (q->F2 - 1) / 2 + 1;
    // chunk duration = chunk_len * subsampling_factor * window_stride (sortformer_backend.py:190-194), hop = stride * 16 kHz
    q->chunk_samples = D.chunk_len * D.subsampling_factor * D.hop;
    q->frames_per_chunk = q->chunk_samples / D.hop + 1;
    q->prev_keep = 99;                                                  // sortformer_backend.py:278
    WLK_CHECK(q->prev_keep <= q->frames_per_chunk, "chunk shorter than the 99 context frames");
    q->max_feat = q->prev_keep + q->frames_per_chunk;
    q->max_T3 = sub_len(q->max_feat);
    q->max_T = D.spkcache_len + D.fifo_len + q->max_T3;
    WLK_CHECK(q->max_T <= SF_MAX_T, "spkcache_len + fifo_len + chunk rows = %d exceeds %d", q->max_T, SF_MAX_T);
    q->max_chunk_cap = q->max_T3;
    {   const int mc = q->max_T3;                                       // upper bound of max_chunk_len
        int mp = D.spkcache_update_period > mc ? D.spkcache_update_period : mc;
        if (mp > mc + D.fifo_len) mp = mc + D.fifo_len;
        q->max_pop = mp; }
    const size_t es = q->es();
    const int C = D.conv_channels, d = D.d_model, t = D.tf_d_model, ff = D.ff_mult * d, K = D.conv_kernel, S = D.n_spk;
    WeightTable& T = q->weights;
    T.rule = WeightTable::LEADING;
    T.wt = q->act;
    const int F = q->F3, P = 2 * SF_MAX_T - 1;
    T.buf(q->window, (size_t)D.win_length * 4);
    T.buf(q->twiddle, (size_t)D.n_fft * 8);
    T.buf(q->fbT, (size_t)q->n_freq * D.n_mels * 4);
    T.buf(q->span, (size_t)D.n_mels * 8);
    declare_mel_filters(T, q->fbT, q->span, D.n_mels, q->n_freq);    // the Slaney bank of librosa.filters.mel, as NeMo builds it
    const std::string pe = "encoder.pre_encode.";
    T.f32(pe + "conv.0.weight", q->c0w, {C, 9});
    T.f32(pe + "conv.0.bias", q->c0b, {C});
    T.f32(pe + "conv.2.weight", q->dw1w, {C, 9});
    T.f32(pe + "conv.2.bias", q->dw1b, {C});
    T.mat(pe + "conv.3.weight", q->Wpw1, {C, C});
    T.f32(pe + "conv.3.bias", q->pw1b, {C});
    T.f32(pe + "conv.5.weight", q->dw2w, {C, 9});
    T.f32(pe + "conv.5.bias", q->dw2b, {C});
    T.mat(pe + "conv.6.weight", q->Wpw2, {C, C});
    T.f32(pe + "conv.6.bias", q->pw2b, {C});
    // NeMo flattens [C][F] channel-major (x.transpose(1, 2).reshape(b, t, -1))
    T.mat(pe + "out.weight", q->Wout, {d, (int64_t)C * F}, swap_inner_axes(d, C, F));
    T.f32(pe + "out.bias", q->outb, {d});
    T.buf(q->pe_table, (size_t)P * d * 4);
    q->L.resize(D.n_layer);
    for (int i = 0; i < D.n_layer; ++i) {
        const std::string p = "encoder.layers." + std::to_string(i) + ".", a = p + "self_attn.", c = p + "conv.";
        SfLayerW& L = q->L[i];
        auto linear = [&](const std::string& n, void*& W, float*& b, int64_t rows, int64_t cols) {
            T.mat(n + ".weight", W, {rows, cols});
            T.f32(n + ".bias", b, {rows});
        };
        auto norm = [&](const std::string& n, float*& w, float*& b) {
            T.f32(n + ".weight", w, {d});
            T.f32(n + ".bias", b, {d});
        };
        norm(p + "norm_feed_forward1", L.ln_ff1w, L.ln_ff1b);
        linear(p + "feed_forward1.linear1", L.W_ff1a, L.b_ff1a, ff, d);
        linear(p + "feed_forward1.linear2", L.W_ff1b, L.b_ff1b, d, ff);
        norm(p + "norm_self_att", L.ln_attw, L.ln_attb);
        T.fused(L.Wqkv, q->act, {{a + "linear_q.weight", d}, {a + "linear_k.weight", d}, {a + "linear_v.weight", d}}, d);
        T.fused(L.bqkv, DT_F32, {{a + "linear_q.bias", d}, {a + "linear_k.bias", d}, {a + "linear_v.bias", d}}, 0);
        linear(a + "linear_out", L.Wo, L.bo, d, d);
        T.mat(a + "linear_pos.weight", L.Wpos, {d, d});
        T.f32(a + "pos_bias_u", L.bias_u, {D.n_head, d / D.n_head});
        T.f32(a + "pos_bias_v", L.bias_v, {D.n_head, d / D.n_head});
        norm(p + "norm_conv", L.ln_convw, L.ln_convb);
        linear(c + "pointwise_conv1", L.Wpw1, L.bpw1, 2 * d, d);
        T.f32(c + "depthwise_conv.weight", L.dw_w, {d, K});
        T.f32(c + "depthwise_conv.bias", L.dw_b, {d});
        norm(c + "batch_norm", L.bn_w, L.bn_b);
        T.f32(c + "batch_norm.running_mean", L.bn_mean, {d});
        T.f32(c + "batch_norm.running_var", L.bn_var, {d});
        T.add(c + "batch_norm.num_batches_tracked", {}, {}).optional = true;   // bookkeeping scalar of nn.BatchNorm1d
        linear(c + "pointwise_conv2", L.Wpw2, L.bpw2, d, d);
        norm(p + "norm_feed_forward2", L.ln_ff2w, L.ln_ff2b);
        linear(p + "feed_forward2.linear1", L.W_ff2a, L.b_ff2a, ff, d);
        linear(p + "feed_forward2.linear2", L.W_ff2b, L.b_ff2b, d, ff);
        norm(p + "norm_out", L.ln_outw, L.ln_outb);
        T.buf(L.bnA, (size_t)d * 4);
        T.buf(L.bnB, (size_t)d * 4);
        T.buf(L.ptab, (size_t)P * d * es);
    }
    q->TL.resize(D.tf_n_layer);
    for (int i = 0; i < D.tf_n_layer; ++i) {
        const std::string p = "transformer_encoder.layers." + std::to_string(i) + ".", a = p + "first_sub_layer.";
        SfTLayerW& L = q->TL[i];
        T.fused(L.Wqkv, q->act, {{a + "query_net.weight", t}, {a + "key_net.weight", t}, {a + "value_net.weight", t}}, t);
        T.fused(L.bqkv, DT_F32, {{a + "query_net.bias", t}, {a + "key_net.bias", t}, {a + "value_net.bias", t}}, 0);
        T.mat(a + "out_projection.weight", L.Wo, {t, t});
        T.f32(a + "out_projection.bias", L.bo, {t});
        T.f32(p + "layer_norm_1.weight", L.ln1w, {t});
        T.f32(p + "layer_norm_1.bias", L.ln1b, {t});
        T.mat(p + "second_sub_layer.dense_in.weight", L.W1, {D.tf_inner, t});
        T.f32(p + "second_sub_layer.dense_in.bias", L.b1, {D.tf_inner});
        T.mat(p + "second_sub_layer.dense_out.weight", L.W2, {t, D.tf_inner});
        T.f32(p + "second_sub_layer.dense_out.bias", L.b2, {t});
        T.f32(p + "layer_norm_2.weight", L.ln2w, {t});
        T.f32(p + "layer_norm_2.bias", L.ln2b, {t});
    }
    const std::string m = "sortformer_modules.";
    T.mat(m + "encoder_proj.weight", q->Wproj, {t, d});
    T.f32(m + "encoder_proj.bias", q->bproj, {t});
    T.mat(m + "first_hidden_to_hidden.weight", q->Wh, {t, t});
    T.f32(m + "first_hidden_to_hidden.bias", q->bh, {t});
    T.f32(m + "single_hidden_to_spks.weight", q->Wspk, {S, t});
    T.f32(m + "single_hidden_to_spks.bias", q->bspk, {S});
    T.allocate(q->allocs, &q->bytes_weights);
    {   // symmetric Hann window (torch.hann_window(periodic=False), as NeMo builds it) and exp(-2 pi i k / n_fft)
        std::vector<float> win(D.win_length);
        std::vector<float2> tw(D.n_fft);
        for (int i = 0; i < D.win_length; ++i) win[i] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * i / (D.win_length - 1)));
        for (int i = 0; i < D.n_fft; ++i) { const double a = 2.0 * M_PI * i / D.n_fft; tw[i] = make_float2((float)cos(a), (float)-sin(a)); }
        CUDA_CHECK(cudaMemcpyAsync(q->window, win.data(), win.size() * 4, cudaMemcpyHostToDevice, q->st));
        CUDA_CHECK(cudaMemcpyAsync(q->twiddle, tw.data(), tw.size() * 8, cudaMemcpyHostToDevice, q->st));
        CUDA_CHECK(cudaStreamSynchronize(q->st));
    }
    // workspaces for max_batch streams
    const size_t B = (size_t)cfg->max_batch;
    size_t* ws = &q->bytes_workspace;
    const size_t T1 = (q->max_feat - 1) / 2 + 1, T2 = (T1 - 1) / 2 + 1, T3 = (T2 - 1) / 2 + 1;
    const size_t R = B * q->max_T;
    q->pcm = (float*)q->allocs.take(B * q->chunk_samples * 4, ws);
    q->feats = (float*)q->allocs.take(B * q->max_feat * D.n_mels * 4, ws);
    q->a1 = q->allocs.take(B * T1 * q->F1 * C * es, ws);
    q->a2 = q->allocs.take(B * T2 * q->F2 * C * es, ws); q->a2p = q->allocs.take(B * T2 * q->F2 * C * es, ws);
    q->a3 = q->allocs.take(B * T3 * q->F3 * C * es, ws); q->a3p = q->allocs.take(B * T3 * q->F3 * C * es, ws);
    q->chunk = (float*)q->allocs.take(B * T3 * d * 4, ws);
    q->x = (float*)q->allocs.take(R * d * 4, ws);
    q->xn = q->allocs.take(R * d * es, ws);
    q->qkv = q->allocs.take(R * 3 * d * es, ws);
    q->att = q->allocs.take(R * d * es, ws);
    q->hid = q->allocs.take(R * (size_t)ff * es, ws);
    q->cv = q->allocs.take(R * d * es, ws);
    q->y = (float*)q->allocs.take(R * t * 4, ws);
    q->preds = (float*)q->allocs.take(R * S * 4, ws);
    q->out_preds = (float*)q->allocs.take(B * q->max_chunk_cap * S * 4, ws);
    CUDA_CHECK(cudaMallocHost(&q->out_h, B * q->max_chunk_cap * S * 4));
    if (q->gemm_backend == WLK_BACKEND_TCGEN05) q->gemm.alloc(q->allocs, ws);
    q->stg.alloc(B * sizeof(SfJob) + 4096, q->allocs, ws);
    q->sess.slots.resize(cfg->max_sessions);
    *out = q;
}

void free_session(SfSession& s) {
    for (int i = 0; i < 2; ++i) { if (s.cache[i]) cudaFree(s.cache[i]); if (s.fifo[i]) cudaFree(s.fifo[i]); if (s.cache_preds[i]) cudaFree(s.cache_preds[i]); }
    if (s.fifo_preds) cudaFree(s.fifo_preds);
    if (s.mean_sil) cudaFree(s.mean_sil);
    if (s.prev_mel) cudaFree(s.prev_mel);
    if (s.total_preds) cudaFree(s.total_preds);
    if (s.n_sil) cudaFree(s.n_sil);
    s = SfSession();
}

void destroy(wlk_sf* q) {
    q->close([q] {
        for (auto& s : q->sess) free_session(s);
        if (q->out_h) cudaFreeHost(q->out_h);
    });
    delete q;
}

void reset_session(wlk_sf* q, SfSession& s) {         // _init_streaming_state (sortformer_backend.py:212-234)
    const wlk_sf_dims& D = q->dims;
    for (int i = 0; i < 2; ++i) {
        CUDA_CHECK(cudaMemsetAsync(s.cache[i], 0, (size_t)D.spkcache_len * D.d_model * 4, q->st));
        CUDA_CHECK(cudaMemsetAsync(s.fifo[i], 0, (size_t)D.fifo_len * D.d_model * 4, q->st));
        CUDA_CHECK(cudaMemsetAsync(s.cache_preds[i], 0, (size_t)D.spkcache_len * D.n_spk * 4, q->st));
    }
    CUDA_CHECK(cudaMemsetAsync(s.fifo_preds, 0, (size_t)D.fifo_len * D.n_spk * 4, q->st));
    CUDA_CHECK(cudaMemsetAsync(s.mean_sil, 0, (size_t)D.d_model * 4, q->st));
    CUDA_CHECK(cudaMemsetAsync(s.n_sil, 0, 4, q->st));
    s.flip = 0; s.sl = 0; s.fl = 0; s.chunk_index = 0; s.tp_rows = 0; s.has_prev = false;
}

template <typename T>
void forward_typed(wlk_sf* q, int n, int R, int rows1, int rows2, int rows3, const SfJob* jobs) {
    const wlk_sf_dims& D = q->dims;
    const int C = D.conv_channels, d = D.d_model, t = D.tf_d_model, ff = D.ff_mult * d, H = D.n_head, dh = d / H, S = D.n_spk;
    // ---- pre_encode
    sf_conv0_kernel<T><<<dim3(64, n), 256, 0, q->st>>>(jobs, q->feats, q->c0w, q->c0b, (T*)q->a1, D.n_mels, C);
    sf_dwconv_kernel<T><<<dim3(32, n), 256, 0, q->st>>>(jobs, 1, (const T*)q->a1, q->dw1w, q->dw1b, (T*)q->a2, q->F1, C);
    gemm(q, q->a2, C, q->Wpw1, C, rows2 * q->F2, C, C, q->pw1b, 2, q->a2p, q->act, C);
    sf_dwconv_kernel<T><<<dim3(16, n), 256, 0, q->st>>>(jobs, 2, (const T*)q->a2p, q->dw2w, q->dw2b, (T*)q->a3, q->F2, C);
    gemm(q, q->a3, C, q->Wpw2, C, rows3 * q->F3, C, C, q->pw2b, 2, q->a3p, q->act, C);
    gemm(q, q->a3p, (int64_t)q->F3 * C, q->Wout, (int64_t)q->F3 * C, rows3, d, q->F3 * C, q->outb, 0, q->chunk, DT_F32, d);
    sf_assemble_kernel<<<dim3(q->max_T, n), 128, 0, q->st>>>(jobs, q->chunk, q->x, d, sqrtf((float)d));
    CUDA_CHECK(cudaGetLastError());
    (void)rows1;
    // ---- FastConformer blocks
    const float att_scale = 1.0f / sqrtf((float)dh);
    const int qblocks = (q->max_T + 15) / 16;
    for (int li = 0; li < D.n_layer; ++li) {
        SfLayerW& L = q->L[li];
        layernorm(q->x, d, L.ln_ff1w, L.ln_ff1b, q->xn, q->act, d, R, d, nullptr, q->st);
        gemm(q, q->xn, d, L.W_ff1a, d, R, ff, d, L.b_ff1a, 3, q->hid, q->act, ff);
        gemm(q, q->hid, ff, L.W_ff1b, ff, R, d, ff, L.b_ff1b, 0, q->x, DT_F32, d, q->x, 0.5f, d);
        layernorm(q->x, d, L.ln_attw, L.ln_attb, q->xn, q->act, d, R, d, nullptr, q->st);
        gemm(q, q->xn, d, L.Wqkv, d, R, 3 * d, d, L.bqkv, 0, q->qkv, q->act, 3 * d);
        if constexpr (std::is_same<T, bf16>::value)
            sf_attention_mma_kernel<true><<<dim3(qblocks, H, n), 128, 0, q->st>>>((const bf16*)q->qkv, jobs, H, d, dh, (const bf16*)L.ptab, SF_MAX_T - 1,
                                                                                  L.bias_u, L.bias_v, att_scale, (bf16*)q->att);
        else
            sf_attention_kernel<T, true><<<dim3(qblocks, H, n), 128, 0, q->st>>>((const T*)q->qkv, jobs, H, d, dh, (const T*)L.ptab, SF_MAX_T - 1,
                                                                                L.bias_u, L.bias_v, att_scale, (T*)q->att);
        gemm(q, q->att, d, L.Wo, d, R, d, d, L.bo, 0, q->x, DT_F32, d, q->x);
        layernorm(q->x, d, L.ln_convw, L.ln_convb, q->xn, q->act, d, R, d, nullptr, q->st);
        gemm(q, q->xn, d, L.Wpw1, d, R, 2 * d, d, L.bpw1, 0, q->hid, q->act, 2 * d);
        sf_glu_dwconv_kernel<T><<<dim3(qblocks, n, (d + 127) / 128), 128, 0, q->st>>>((const T*)q->hid, jobs, L.dw_w, L.bnA, L.bnB, (T*)q->cv, d, D.conv_kernel);
        gemm(q, q->cv, d, L.Wpw2, d, R, d, d, L.bpw2, 0, q->x, DT_F32, d, q->x);
        layernorm(q->x, d, L.ln_ff2w, L.ln_ff2b, q->xn, q->act, d, R, d, nullptr, q->st);
        gemm(q, q->xn, d, L.W_ff2a, d, R, ff, d, L.b_ff2a, 3, q->hid, q->act, ff);
        gemm(q, q->hid, ff, L.W_ff2b, ff, R, d, ff, L.b_ff2b, 0, q->x, DT_F32, d, q->x, 0.5f, d);
        layernorm(q->x, d, L.ln_outw, L.ln_outb, q->x, DT_F32, d, R, d, nullptr, q->st);
    }
    CUDA_CHECK(cudaGetLastError());
    // ---- encoder_proj + post-LN Transformer + speaker sigmoids
    convert_f32_to(q->x, q->xn, q->act, (int64_t)R * d, q->st);
    gemm(q, q->xn, d, q->Wproj, d, R, t, d, q->bproj, 0, q->y, DT_F32, t);
    const int TH = D.tf_n_head, tdh = t / TH;
    const float qk_scale = 1.0f / sqrtf(sqrtf((float)tdh));
    for (int li = 0; li < D.tf_n_layer; ++li) {
        SfTLayerW& L = q->TL[li];
        convert_f32_to(q->y, q->xn, q->act, (int64_t)R * t, q->st);
        gemm(q, q->xn, t, L.Wqkv, t, R, 3 * t, t, L.bqkv, 0, q->qkv, q->act, 3 * t, nullptr, qk_scale, 2 * t);
        if constexpr (std::is_same<T, bf16>::value)
            sf_attention_mma_kernel<false><<<dim3(qblocks, TH, n), 128, 0, q->st>>>((const bf16*)q->qkv, jobs, TH, t, tdh, nullptr, 0, nullptr, nullptr, 1.0f, (bf16*)q->att);
        else
            sf_attention_kernel<T, false><<<dim3(qblocks, TH, n), 128, 0, q->st>>>((const T*)q->qkv, jobs, TH, t, tdh, nullptr, 0, nullptr, nullptr, 1.0f, (T*)q->att);
        gemm(q, q->att, t, L.Wo, t, R, t, t, L.bo, 0, q->y, DT_F32, t, q->y);
        layernorm(q->y, t, L.ln1w, L.ln1b, q->y, DT_F32, t, R, t, nullptr, q->st);
        convert_f32_to(q->y, q->xn, q->act, (int64_t)R * t, q->st);
        gemm(q, q->xn, t, L.W1, t, R, D.tf_inner, t, L.b1, 2, q->hid, q->act, D.tf_inner);
        gemm(q, q->hid, D.tf_inner, L.W2, D.tf_inner, R, t, D.tf_inner, L.b2, 0, q->y, DT_F32, t, q->y);
        layernorm(q->y, t, L.ln2w, L.ln2b, q->y, DT_F32, t, R, t, nullptr, q->st);
    }
    sf_relu_kernel<T><<<256, 256, 0, q->st>>>(q->y, (T*)q->xn, (int64_t)R * t);
    gemm(q, q->xn, t, q->Wh, t, R, t, t, q->bh, 2, q->att, q->act, t);
    sf_spk_kernel<T><<<(R * 32 + 255) / 256, 256, 0, q->st>>>((const T*)q->att, q->Wspk, q->bspk, q->preds, R, t, S);
    CUDA_CHECK(cudaGetLastError());
}

// One diarize() step for n streams.  pcm != null: raw samples in (sample_off [n+1]); feats_host != null: features in
// (time-major [frames][n_mels] rows, frame_off [n+1], explicit left / right offsets = the forward_streaming_step seam).
void step(wlk_sf* q, const int32_t* sids, int n, const float* pcm_host, const int64_t* sample_off, const float* feats_host,
          const int32_t* frame_off, int left_offset, int right_offset, float* out_host, int32_t* out_rows) {
    const wlk_sf_dims& D = q->dims;
    WLK_CHECK(q->finalized, "weights not finalized");
    WLK_CHECK(n >= 1 && n <= q->cfg.max_batch, "batch %d outside [1, %d]", n, q->cfg.max_batch);
    WLK_CHECK((pcm_host != nullptr) != (feats_host != nullptr), "exactly one of pcm / features");
    const int S = D.n_spk, d = D.d_model;
    // ---- pass 1: validate and plan without touching any session
    std::vector<SfJob> jobs(n);
    int feat_rows = 0, r1 = 0, r2 = 0, r3 = 0, R = 0, out_off = 0;
    q->sess.check_batch(sids, n);
    for (int i = 0; i < n; ++i) {
        SfSession& s = q->sess[sids[i]];
        SfJob& j = jobs[i];
        memset(&j, 0, sizeof(j));
        int n_feat;
        if (pcm_host) {
            const int64_t ns = sample_off[i + 1] - sample_off[i];
            WLK_CHECK(ns == q->chunk_samples, "stream %d: a diarization step takes exactly %d samples (got %lld)", i, q->chunk_samples, (long long)ns);
            j.n_samples = (int)ns; j.n_new_frames = q->frames_per_chunk; j.has_prev = s.has_prev ? 1 : 0;
            n_feat = q->frames_per_chunk + (s.has_prev ? q->prev_keep : 0);
            j.lc = (int)nearbyint((s.chunk_index > 0 ? 8 : 0) / (double)D.encoder_subsampling);       // Python round(): ties to even            // sortformer_backend.py:289-290
            j.rc = (8 + D.encoder_subsampling - 1) / D.encoder_subsampling;
        } else {
            n_feat = frame_off[i + 1] - frame_off[i];
            WLK_CHECK(n_feat >= 8 && n_feat <= q->max_feat, "stream %d: %d feature frames outside [8, %d]", i, n_feat, q->max_feat);
            j.lc = (int)nearbyint(left_offset / (double)D.encoder_subsampling);
            j.rc = (right_offset + D.encoder_subsampling - 1) / D.encoder_subsampling;
        }
        j.feat_off = feat_rows; j.n_feat = n_feat;
        j.T1 = (n_feat - 1) / 2 + 1; j.T2 = (j.T1 - 1) / 2 + 1; j.T3 = (j.T2 - 1) / 2 + 1;
        j.t1_off = r1; j.t2_off = r2; j.t3_off = r3;
        j.sl = s.sl; j.fl = s.fl;
        j.row_off = R; j.T = s.sl + s.fl + j.T3;
        j.max_chunk = j.T3 - j.lc - j.rc;
        WLK_CHECK(j.max_chunk >= 1, "stream %d: chunk of %d rows leaves nothing after the %d + %d context rows", i, j.T3, j.lc, j.rc);
        j.clen = std::min(std::max(j.T3 - j.lc, 0), j.max_chunk);
        const int new_fl = s.fl + j.clen;
        j.do_pop = new_fl > D.fifo_len;
        if (j.do_pop) {
            int pop = D.spkcache_update_period;
            pop = std::max(pop, j.max_chunk - D.fifo_len + s.fl);
            pop = std::min(pop, new_fl);
            j.pop = pop;
            WLK_CHECK(pop <= q->max_pop, "pop-out of %d rows exceeds the planned %d", pop, q->max_pop);
        }
        j.compress = s.sl + j.pop > D.spkcache_len;
        j.out_off = out_off;
        feat_rows += n_feat; r1 += j.T1; r2 += j.T2; r3 += j.T3; R += j.T; out_off += j.max_chunk;
        const int cur = s.flip, nxt = s.flip ^ 1;
        j.cache_cur = s.cache[cur]; j.cache_next = s.cache[nxt]; j.fifo_cur = s.fifo[cur]; j.fifo_next = s.fifo[nxt];
        j.cache_preds_cur = s.cache_preds[cur]; j.cache_preds_next = s.cache_preds[nxt]; j.fifo_preds_next = s.fifo_preds;
        j.mean_sil = s.mean_sil; j.n_sil = s.n_sil; j.prev_mel = s.prev_mel;
        j.pcm = pcm_host ? q->pcm + (size_t)i * q->chunk_samples : nullptr;
    }
    // ---- total_preds room (trim like sortformer_backend.py:301-305, before the step's rows are appended)
    for (int i = 0; i < n; ++i) {
        SfSession& s = q->sess[sids[i]];
        if (s.tp_rows + jobs[i].max_chunk > SF_TP_CAP) {
            CUDA_CHECK(cudaMemcpyAsync(s.total_preds, s.total_preds + (size_t)(s.tp_rows - SF_TP_KEEP) * S, (size_t)SF_TP_KEEP * S * 4,
                                       cudaMemcpyDeviceToDevice, q->st));
            s.tp_rows = SF_TP_KEEP;
        }
        jobs[i].total_preds = s.total_preds + (size_t)s.tp_rows * S;
    }
    Stager sg(q->stg);
    SfJob* jd;
    memcpy(sg.host<SfJob>(n, &jd), jobs.data(), sizeof(SfJob) * n);
    sg.upload(q->st);
    if (pcm_host) {
        for (int i = 0; i < n; ++i)
            CUDA_CHECK(cudaMemcpyAsync(q->pcm + (size_t)i * q->chunk_samples, pcm_host + sample_off[i], (size_t)q->chunk_samples * 4,
                                       cudaMemcpyHostToDevice, q->st));
        sf_prev_feats_kernel<<<dim3(q->prev_keep, n), 128, 0, q->st>>>(jd, q->feats, D.n_mels, q->prev_keep, q->frames_per_chunk);
        const size_t smem = (size_t)((D.win_length + 3) & ~3) * 4 + (size_t)D.n_fft * 8 + (size_t)q->n_freq * 4;
        sf_mel_kernel<<<dim3(q->frames_per_chunk, n), 288, smem, q->st>>>(jd, q->window, q->twiddle, q->fbT, q->span, q->feats, D.n_fft,
                                                                          D.win_length, D.hop, D.n_mels, q->prev_keep);
    } else {
        for (int i = 0; i < n; ++i)
            CUDA_CHECK(cudaMemcpyAsync(q->feats + (size_t)jobs[i].feat_off * D.n_mels, feats_host + (size_t)frame_off[i] * D.n_mels,
                                       (size_t)jobs[i].n_feat * D.n_mels * 4, cudaMemcpyHostToDevice, q->st));
    }
    CUDA_CHECK(cudaGetLastError());
    if (q->act == DT_BF16) forward_typed<bf16>(q, n, R, r1, r2, r3, jd);
    else forward_typed<float>(q, n, R, r1, r2, r3, jd);
    // ---- streaming update
    SfUpd U;
    U.D = d; U.S = S; U.CL = D.spkcache_len; U.FL = D.fifo_len; U.sil_per_spk = D.spkcache_sil_frames_per_spk;
    U.n_cache = D.spkcache_len + q->max_pop;
    U.th = D.pred_score_threshold; U.boost_latest = D.scores_boost_latest; U.sil_th = D.sil_threshold;
    const int per_spk = D.spkcache_len / S - D.spkcache_sil_frames_per_spk;
    U.strong = (int)floor(per_spk * (double)D.strong_boost_rate);
    U.weak = (int)floor(per_spk * (double)D.weak_boost_rate);
    U.min_pos = (int)floor(per_spk * (double)D.min_pos_scores_rate);
    const int nf = U.n_cache + U.sil_per_spk;
    const size_t usm = ((size_t)U.n_cache * S + 2 * (size_t)S * nf + (size_t)U.CL) * 4 + 64;
    static bool seen_attr[64] = {};
    if (first_on_device(seen_attr)) CUDA_CHECK(cudaFuncSetAttribute(sf_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    WLK_CHECK(usm <= 96 * 1024, "speaker-cache scratch of %zu bytes exceeds the kernel's shared memory", usm);
    sf_update_kernel<<<n, 256, usm, q->st>>>(jd, q->chunk, q->preds, q->out_preds, U);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(q->out_h, q->out_preds, (size_t)out_off * S * 4, cudaMemcpyDeviceToHost, q->st));
    CUDA_CHECK(cudaStreamSynchronize(q->st));
    // ---- commit (the device work of the step has succeeded)
    int o = 0;
    for (int i = 0; i < n; ++i) {
        SfSession& s = q->sess[sids[i]];
        const SfJob& j = jobs[i];
        s.flip ^= 1;
        s.sl = std::min(j.sl + j.pop, D.spkcache_len);
        s.fl = j.fl + j.clen - j.pop;
        s.tp_rows += j.max_chunk;
        s.chunk_index += 1;
        if (pcm_host) s.has_prev = true;
        if (out_rows) out_rows[i] = o;
        o += j.max_chunk;
    }
    if (out_rows) out_rows[n] = o;
    if (out_host) memcpy(out_host, q->out_h, (size_t)o * S * 4);
}

}  // namespace

extern "C" {

int wlk_sf_create(const wlk_sf_dims* dims, const wlk_config* cfg, wlk_sf** out) {
    WLK_API_BEGIN
    create(dims, cfg, out);
    WLK_API_END
}
int wlk_sf_destroy(wlk_sf* q) {
    WLK_API_BEGIN
    WLK_CHECK(q != nullptr, "null engine");
    CUDA_CHECK(cudaSetDevice(q->cfg.device));
    destroy(q);
    WLK_API_END
}
int wlk_sf_load_tensor(wlk_sf* q, const char* name, const float* host, const int64_t* shape, int ndim) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(name && host && shape && ndim >= 1, "bad arguments");
    q->weights.load(name, host, shape, ndim);
    WLK_API_END
}
int wlk_sf_finalize_weights(wlk_sf* q) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    finalize(q);
    WLK_API_END
}
int wlk_sf_session_open(wlk_sf* q, int32_t* sid) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(sid != nullptr, "null argument");
    const wlk_sf_dims& D = q->dims;
    const int found = q->sess.free_slot();
    SfSession& s = q->sess[found];
    size_t* acct = &q->bytes_sessions;
    auto al = [&](size_t bytes) { void* p = nullptr; CUDA_CHECK(cudaMalloc(&p, bytes)); *acct += bytes; return p; };
    for (int k = 0; k < 2; ++k) {
        s.cache[k] = (float*)al((size_t)D.spkcache_len * D.d_model * 4);
        s.fifo[k] = (float*)al((size_t)D.fifo_len * D.d_model * 4);
        s.cache_preds[k] = (float*)al((size_t)D.spkcache_len * D.n_spk * 4);
    }
    s.fifo_preds = (float*)al((size_t)D.fifo_len * D.n_spk * 4);
    s.mean_sil = (float*)al((size_t)D.d_model * 4);
    s.prev_mel = (float*)al((size_t)q->frames_per_chunk * D.n_mels * 4);
    s.total_preds = (float*)al((size_t)SF_TP_CAP * D.n_spk * 4);
    s.n_sil = (int32_t*)al(16);
    s.open = true;
    reset_session(q, s);
    CUDA_CHECK(cudaStreamSynchronize(q->st));
    *sid = found;
    WLK_API_END
}
int wlk_sf_session_close(wlk_sf* q, int32_t sid) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    SfSession& s = q->sess.at(sid);
    CUDA_CHECK(cudaStreamSynchronize(q->st));
    free_session(s);
    WLK_API_END
}
int wlk_sf_session_reset(wlk_sf* q, int32_t sid) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    reset_session(q, q->sess.at(sid));
    CUDA_CHECK(cudaStreamSynchronize(q->st));
    WLK_API_END
}
int wlk_sf_step_audio(wlk_sf* q, const int32_t* sids, int n, const float* pcm_host, const int64_t* sample_offsets,
                      float* chunk_preds_host, int32_t* row_offsets_out) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(sids && pcm_host && sample_offsets, "null argument");
    step(q, sids, n, pcm_host, sample_offsets, nullptr, nullptr, 0, 0, chunk_preds_host, row_offsets_out);
    WLK_API_END
}
int wlk_sf_step_features(wlk_sf* q, const int32_t* sids, int n, const float* feats_host, const int32_t* frame_offsets,
                         int32_t left_offset, int32_t right_offset, float* chunk_preds_host, int32_t* row_offsets_out) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(sids && feats_host && frame_offsets, "null argument");
    WLK_CHECK(left_offset >= 0 && right_offset >= 0, "negative context offset");
    step(q, sids, n, nullptr, nullptr, feats_host, frame_offsets, left_offset, right_offset, chunk_preds_host, row_offsets_out);
    WLK_API_END
}
int wlk_sf_total_preds(wlk_sf* q, int32_t sid, const float** preds_dev, int32_t* n_rows) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    SfSession& s = q->sess.at(sid);
    if (preds_dev) *preds_dev = s.total_preds;
    if (n_rows) *n_rows = s.tp_rows;
    WLK_API_END
}
int wlk_sf_read_state(wlk_sf* q, int32_t sid, int32_t* lengths /*[4]: spkcache, fifo, n_sil, chunk_index*/, float* spkcache_host,
                      float* spkcache_preds_host, float* fifo_host, float* mean_sil_host) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    SfSession& s = q->sess.at(sid);
    const wlk_sf_dims& D = q->dims;
    CUDA_CHECK(cudaStreamSynchronize(q->st));
    if (lengths) {
        int32_t ns = 0;
        CUDA_CHECK(cudaMemcpy(&ns, s.n_sil, 4, cudaMemcpyDeviceToHost));
        lengths[0] = s.sl; lengths[1] = s.fl; lengths[2] = ns; lengths[3] = s.chunk_index;
    }
    if (spkcache_host) CUDA_CHECK(cudaMemcpy(spkcache_host, s.cache[s.flip], (size_t)D.spkcache_len * D.d_model * 4, cudaMemcpyDeviceToHost));
    if (spkcache_preds_host) CUDA_CHECK(cudaMemcpy(spkcache_preds_host, s.cache_preds[s.flip], (size_t)D.spkcache_len * D.n_spk * 4, cudaMemcpyDeviceToHost));
    if (fifo_host) CUDA_CHECK(cudaMemcpy(fifo_host, s.fifo[s.flip], (size_t)D.fifo_len * D.d_model * 4, cudaMemcpyDeviceToHost));
    if (mean_sil_host) CUDA_CHECK(cudaMemcpy(mean_sil_host, s.mean_sil, (size_t)D.d_model * 4, cudaMemcpyDeviceToHost));
    WLK_API_END
}
int wlk_sf_memory(wlk_sf* q, size_t* weights, size_t* sessions, size_t* workspace) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    q->memory(weights, sessions, workspace);
    WLK_API_END
}

}  // extern "C"
