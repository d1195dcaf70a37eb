// Qwen3-ASR audio towers behind the C ABI (wlk_qwen_* in include/wlk_b200.h), in one of two modes per engine:
//   causal   (wlk_qwen_create, SURVEY.md section 8 row a17): reference third_party/qwen3-asr-causal/src/qwen3_asr_causal/
//            causal.py: forward_chunk :713-782, _encode_ready_mels :642-681, _conv_one_block :230-248,
//            _position_embedding :204-228, _attention_chunk :292-376, _layer_chunk :378-421
//   windowed (wlk_qwen_window_create): QwenAudioSurgeryEncoder, reference model.py:441-608, over the stock tower
//            (transformers 5.5 modeling_qwen3_omni_moe.py:710-768)
// Both modes share the weights, the conv stem, the pre-LN layer stack and the head; each keeps its own planning, its
// conv_out step, its QKV destination and its attention.
//
// Causal: append-only execution, every mel frame transits the tower exactly once.  Sessions are batched per "round":
// round r holds the r-th ready block (or run of chunks) of every session in the call, so a block always finds the K/V
// its predecessor left in the session's ring.
//
// Data layout (R = encoder rows of a round or call):
//   conv stem    chunks of T0 mel frames fp32 [n][T0][n_mels] (causal: T0 = 8, one chunk per step; windowed: T0 = 100,
//                13 steps), NHWC activations [n][F][T][C]; conv2 / conv3 are im2col + GEMM (K = 9C, taps-major so a tap
//                is one contiguous run of C channels), conv_out is a GEMM over [steps][F*C] with its weight columns
//                permuted from the reference's (c, f) order at load time
//   residual x   fp32 [R][d]
//   causal       the sinusoid rows ride into conv_out as the GEMM's residual; q [R][d]; K/V rings per session
//                [L][K|V][H][ring][64], ring = left_context + 128 slots addressed by position % ring (written by the QKV
//                GEMM's scatter epilogue)
//   windowed     each chunk's valid steps are compacted into x with positional rows 0..12; qkv [R][3d]
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include "../../include/wlk_b200.h"
#include "attn_warp.cuh"
#include "host.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

namespace wlk {
namespace {

constexpr int Q_STEPS_CAP = 128;        // steps one session may contribute to one round

struct QJob {                           // one per session in a round (device array)
    void* kv;                           // the session's K/V rings
    int32_t start;                      // absolute position (encoder step index) of the round's first row
    int32_t n_steps;
    int32_t row_off;
    int32_t pad;
};

struct WChunk {                         // one conv chunk (device array)
    const float* src;                   // the chunk's first mel frame [frames][n_mels]
    int32_t avail;                      // frames of the window inside the chunk; frames beyond are zero
    int32_t p0;                         // conv input length: T0, or a window's length when it is under T0 frames
    int32_t dst_row;                    // residual row of the chunk's first valid step
    int32_t n_valid;                    // valid steps (windowed: mod-100 rule on avail)
};

// ---------------------------------------------------------------------------------------------------------
// conv2d1 (1 -> C, 3x3, stride 2, pad 1, GELU) over chunks laid out [n][T0][n_mels] (mel index = conv "height");
// chunk k's input ends at p0 (the conv's zero padding starts there).  out NHWC [n][n_mels / 2][T0 / 2][C]; steps past
// the chunk's conv length are computed but never read.
// ---------------------------------------------------------------------------------------------------------
template <typename T, int T0>
__global__ void qwen_conv1_kernel(const float* __restrict__ mel, const WChunk* __restrict__ jobs, const float* __restrict__ w,
                                  const float* __restrict__ b, T* __restrict__ out, int n_chunks, int n_mels, int C) {
    constexpr int T1 = T0 / 2;
    const int F1 = n_mels / 2;
    const int64_t total = (int64_t)n_chunks * F1 * T1 * C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = i % C;
        int64_t r = i / C;
        const int t = r % T1; r /= T1;
        const int f = r % F1;
        const int64_t ch = r / F1;
        const int p0 = jobs[ch].p0;
        const float* x = mel + ch * T0 * n_mels;
        float acc = b[c];
#pragma unroll
        for (int kf = 0; kf < 3; ++kf) {
            const int m = 2 * f - 1 + kf;
            if (m < 0 || m >= n_mels) continue;
#pragma unroll
            for (int kt = 0; kt < 3; ++kt) {
                const int fr = 2 * t - 1 + kt;
                if (fr < 0 || fr >= p0) continue;
                acc = fmaf(w[c * 9 + kf * 3 + kt], x[fr * n_mels + m], acc);
            }
        }
        out[i] = from_f32<T>(gelu_erf(acc));
    }
}

// im2col of a 3x3 / stride 2 / pad 1 conv over NHWC [n][Fi][Ti][C]: rows (n, fo, to), or (n, to, fo) when time_major
// (conv3, so that conv_out reads one step's [F][C] features as one row); columns (tap, c).  Input steps at or past
// the chunk's conv length at this stage read as zero (the conv's padding of a shorter input).
template <typename T>
__global__ void qwen_im2col_kernel(const T* __restrict__ src, const WChunk* __restrict__ jobs, T* __restrict__ dst, int n,
                                   int Fi, int Ti, int stage, int C, int time_major) {
    const int Fo = Fi / 2, To = (Ti + 1) / 2;
    const int64_t total = (int64_t)n * Fo * To * 9 * C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = i % C;
        int64_t r = i / C;
        const int tap = r % 9; r /= 9;
        int fo, to;
        if (time_major) { fo = r % Fo; r /= Fo; to = r % To; r /= To; }
        else { to = r % To; r /= To; fo = r % Fo; r /= Fo; }
        const int64_t ch = r;
        int len = jobs[ch].p0;                                   // conv input length at this stage
        for (int s = 0; s < stage; ++s) len = (len - 1) / 2 + 1;
        const int f = 2 * fo - 1 + tap / 3, t = 2 * to - 1 + tap % 3;
        T v = from_f32<T>(0.f);
        if (f >= 0 && f < Fi && t >= 0 && t < len) v = src[((ch * Fi + f) * Ti + t) * C + c];
        dst[i] = v;
    }
}

// positional rows: table[pos] while pos is inside the table, else the closed form sin | cos of fp32(pos) * inv_freq[j]
// (reference causal.py:204-228; inv_freq [d / 2] holds the reference's fp32 frequencies, see alloc_weights)
__global__ void qwen_pos_kernel(const int32_t* __restrict__ pos, const float* __restrict__ table, const float* __restrict__ inv_freq,
                                int max_positions, float* __restrict__ out, int rows, int d) {
    const int r = blockIdx.x;
    if (r >= rows) return;
    const int p = pos[r];
    const int half = d / 2;
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
        float v;
        if (p < max_positions) {
            v = table[(int64_t)p * d + i];
        } else {
            const float a = (float)p * inv_freq[i < half ? i : i - half];
            v = i < half ? sinf(a) : cosf(a);
        }
        out[(int64_t)r * d + i] = v;
    }
}

// ---------------------------------------------------------------------------------------------------------
// Attention of one round (reference causal.py:292-376): a query at position p sees keys at positions
//   [p - left_ctx + 1, block_max]   (block-bidirectional)   or   [p - left_ctx + 1, p]   (causal),
// clipped at 0; keys live in the session's ring at slot = position % ring (this round's keys were written by the
// QKV GEMM).  q arrives pre-scaled by head_dim^-0.5.  One warp per query (attend_row_warp), grid (head, job).
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128)
qwen_attention_kernel(const T* __restrict__ q, const QJob* __restrict__ jobs, int layer, int n_head, int d_model, int ring,
                      int left_ctx, int bidir, T* __restrict__ out) {
    __shared__ float qs[4][64];
    const QJob job = jobs[blockIdx.y];
    const int h = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const T* kbase = reinterpret_cast<const T*>(job.kv) + (((int64_t)layer * 2 + 0) * n_head + h) * ring * 64;
    const T* vbase = reinterpret_cast<const T*>(job.kv) + (((int64_t)layer * 2 + 1) * n_head + h) * ring * 64;
    const int block_max = job.start + job.n_steps - 1;
    for (int qi = warp; qi < job.n_steps; qi += 4) {
        const int p = job.start + qi;
        const int64_t row = job.row_off + qi;
        qs[warp][lane] = to_f32(q[row * d_model + h * 64 + lane]);
        qs[warp][lane + 32] = to_f32(q[row * d_model + h * 64 + lane + 32]);
        __syncwarp();
        const int lo = max(0, p - left_ctx + 1), hi = bidir ? block_max : p;
        // 16 keys per lane: ring <= 512
        attend_row_warp<T, 16>(qs[warp], hi - lo + 1, [&](int ki) { return kbase + (int64_t)((lo + ki) % ring) * 64; },
                               [&](int ki) { return vbase + (int64_t)((lo + ki) % ring) * 64; }, out + row * d_model + h * 64);
        __syncwarp();
    }
}

struct QLayerW {
    void *Wqkv = nullptr, *Wo = nullptr, *W1 = nullptr, *W2 = nullptr;
    float *bqkv = nullptr, *bo = nullptr, *b1 = nullptr, *b2 = nullptr;
    float *ln1w = nullptr, *ln1b = nullptr, *ln2w = nullptr, *ln2b = nullptr;
};

constexpr int QMEL_MAX_FRAMES = N_FRAMES;               // frames one featurized window may hold (30 s)
constexpr int QMEL_AUDIO_CAP = QMEL_MAX_FRAMES * HOP + 2 * N_FFT;

struct QSession {
    bool open = false;
    std::vector<float> pending;         // mel frames not yet consumed (host: the caller hands mels on the host)
    std::vector<float> tail;            // bounded mutable tail: the mel chunks of the steps that are still re-computable
    int64_t emitted = 0;                // encoder steps emitted so far == absolute position of the next step
    void* kv = nullptr;
    // incremental log-mel front end (reference features.py:32-112): the sample window lives on the device
    float* audio = nullptr; float* mel_raw = nullptr; float* mel_blockmax = nullptr;
    int64_t buf_len = 0, buf_start_frame = 0, mel_emitted = 0, total_samples = 0;
    // windowed engine (QwenAudioSurgeryState, reference model.py:36-43): the last left + right mel frames on the device
    float* win = nullptr;
    int64_t win_len = 0, frames_seen = 0, window_start = 0, last_in = 0, last_rec = 0, last_ctx = 0;
};

}  // namespace
}  // namespace wlk

using namespace wlk;

struct wlk_qwen : EngineBase {
    wlk_qwen_dims dims{};
    int gemm_backend = WLK_BACKEND_SIMT;
    int ring = 0, max_rows = 0, conv_chunks = 0;                 // conv_chunks: chunks the conv stem's workspace holds
    // weights
    float *c1w = nullptr, *c1b = nullptr, *c2b = nullptr, *c3b = nullptr, *bout = nullptr, *pos_table = nullptr, *pos_inv = nullptr;
    void *W2c = nullptr, *W3c = nullptr, *Wout = nullptr, *Wp1 = nullptr, *Wp2 = nullptr;
    float *lnpw = nullptr, *lnpb = nullptr, *bp1 = nullptr, *bp2 = nullptr;
    float *filtT = nullptr, *window = nullptr; float2* twiddle = nullptr; int2* filt_span = nullptr;   // mel front end
    float* mel_out = nullptr; size_t mel_out_cap = 0; float* audio_scratch = nullptr;
    std::vector<QLayerW> L;
    // sessions and workspaces
    SessionTable<QSession> sess;
    float *mel = nullptr, *x = nullptr, *outbuf = nullptr;                      // conv chunks, residual, head output
    void *a1 = nullptr, *col = nullptr, *a2 = nullptr, *a3 = nullptr;           // conv stem
    void *xn = nullptr, *att = nullptr, *hid = nullptr;                         // layer stack and head
    // causal engine: the positional rows of a round, q of a round (k / v go to the session rings)
    float* posbuf = nullptr; void* qb = nullptr;
    // windowed engine (wlk_qwen_window_create): geometry, rows of a full window, conv_out's rows, q/k/v, window scratch
    bool windowed = false;
    wlk_qwen_window_dims wd{};
    int win_rows = 0, win_block_chunks = 0;
    void* qkv = nullptr;
    float *xc = nullptr, *win_scratch = nullptr;
};

namespace {

void qgemm(wlk_qwen* q, GemmArgs& g) { q->gemm.run(g, q->gemm_backend == WLK_BACKEND_TCGEN05, q->st, q->num_sms); }

// The tower's weights (shared by the causal and the windowed engine) and the mel front end's constants.  The positional
// frequencies and the filterbank (only wlk_qwen_append_audio needs it) are optional.
void alloc_weights(wlk_qwen* q) {
    const wlk_qwen_dims& D = q->dims;
    WeightTable& T = q->weights;
    T.rule = WeightTable::EXACT;
    T.wt = q->act;
    const int C = D.conv_channels, d = D.d_model, F = D.n_mels / 8, ffn = D.ffn_dim;
    T.f32("conv2d1.weight", q->c1w, {C, 1, 3, 3});
    T.f32("conv2d1.bias", q->c1b, {C});
    T.mat("conv2d2.weight", q->W2c, {C, C, 3, 3}, swap_inner_axes(C, C, 9));
    T.f32("conv2d2.bias", q->c2b, {C});
    T.mat("conv2d3.weight", q->W3c, {C, C, 3, 3}, swap_inner_axes(C, C, 9));
    T.f32("conv2d3.bias", q->c3b, {C});
    // the reference flattens [C][F] (channel-major, causal.py:240-242)
    T.mat("conv_out.weight", q->Wout, {d, (int64_t)C * F}, swap_inner_axes(d, C, F));
    if (D.conv_out_bias) T.f32("conv_out.bias", q->bout, {d});
    T.f32("positional_embedding.positional_embedding", q->pos_table, {D.max_positions, d});
    T.f32("positional_embedding.inv_freq", q->pos_inv, {d / 2}).optional = true;
    T.f32("ln_post.weight", q->lnpw, {d});
    T.f32("ln_post.bias", q->lnpb, {d});
    T.mat("proj1.weight", q->Wp1, {d, d});
    T.f32("proj1.bias", q->bp1, {d});
    T.mat("proj2.weight", q->Wp2, {D.out_dim, d});
    T.f32("proj2.bias", q->bp2, {D.out_dim});
    q->L.resize(D.n_layer);
    for (int i = 0; i < D.n_layer; ++i) {
        const std::string p = "layers." + std::to_string(i) + ".";
        QLayerW& Lw = q->L[i];
        const std::string a = p + "self_attn.";
        T.fused(Lw.Wqkv, q->act, {{a + "q_proj.weight", d}, {a + "k_proj.weight", d}, {a + "v_proj.weight", d}}, d);
        T.fused(Lw.bqkv, DT_F32, {{a + "q_proj.bias", d}, {a + "k_proj.bias", d}, {a + "v_proj.bias", d}}, 0);
        T.mat(a + "out_proj.weight", Lw.Wo, {d, d});
        T.f32(a + "out_proj.bias", Lw.bo, {d});
        T.mat(p + "fc1.weight", Lw.W1, {ffn, d});
        T.f32(p + "fc1.bias", Lw.b1, {ffn});
        T.mat(p + "fc2.weight", Lw.W2, {d, ffn});
        T.f32(p + "fc2.bias", Lw.b2, {d});
        T.f32(p + "self_attn_layer_norm.weight", Lw.ln1w, {d});
        T.f32(p + "self_attn_layer_norm.bias", Lw.ln1b, {d});
        T.f32(p + "final_layer_norm.weight", Lw.ln2w, {d});
        T.f32(p + "final_layer_norm.bias", Lw.ln2b, {d});
    }
    T.buf(q->filtT, (size_t)N_FREQ * D.n_mels * 4);
    T.buf(q->window, N_FFT * 4);
    T.buf(q->twiddle, N_FFT * 8);
    T.buf(q->filt_span, (size_t)D.n_mels * 8);
    declare_mel_filters(T, q->filtT, q->filt_span, D.n_mels, N_FREQ).optional = true;
    T.allocate(q->allocs, &q->bytes_weights);
    {   // periodic Hann window and DFT twiddles exp(-2 pi i t / 400), evaluated in double
        std::vector<float> win(N_FFT);
        std::vector<float2> tw(N_FFT);
        for (int t = 0; t < N_FFT; ++t) {
            const double a = 2.0 * M_PI * t / N_FFT;
            win[t] = (float)(0.5 - 0.5 * cos(a));
            tw[t] = make_float2((float)cos(a), (float)-sin(a));
        }
        CUDA_CHECK(cudaMemcpyAsync(q->window, win.data(), N_FFT * 4, cudaMemcpyHostToDevice, q->st));
        CUDA_CHECK(cudaMemcpyAsync(q->twiddle, tw.data(), N_FFT * 8, cudaMemcpyHostToDevice, q->st));
        CUDA_CHECK(cudaStreamSynchronize(q->st));
    }
    {   // default frequencies of the closed-form positional rows, the reference's recipe: the scale -ln(1e4) / (half - 1)
        // is a double rounded once to fp32, times fp32(j), then fp32 exp.  The host's expf may still differ from the
        // device's exp by an ulp in a few entries, so hosts load "positional_embedding.inv_freq" evaluated on the device
        // (whisperlivekit_b200/qwen_engine.py always does)
        const int half = d / 2;
        const float scale = (float)(-std::log(10000.0) / (double)std::max(1, half - 1));
        std::vector<float> f(half);
        for (int j = 0; j < half; ++j) f[j] = std::exp(scale * (float)j);
        CUDA_CHECK(cudaMemcpyAsync(q->pos_inv, f.data(), f.size() * 4, cudaMemcpyHostToDevice, q->st));
        CUDA_CHECK(cudaStreamSynchronize(q->st));
    }
}

// The creation both modes share: the checks on the shared geometry, device, precision and GEMM backend, stream, weights,
// the conv stem's workspace (conv_chunks chunks of t0 frames at a time), the layer stack's and the head's workspace
// (max_rows rows), split-K scratch, the staging block and the sessions.  Each mode checks its own geometry before and
// adds its own buffers after.
wlk_qwen* create_common(const wlk_qwen_dims& D, const wlk_config* cfg, int max_rows, size_t conv_chunks, int t0,
                        size_t stg_bytes) {
    WLK_CHECK(D.n_mels % 8 == 0 && D.n_mels >= 8, "n_mels must be a multiple of 8");
    WLK_CHECK(D.d_model % 64 == 0 && D.d_model / D.n_head == 64 && D.d_model <= 1280, "heads must be 64 wide, d_model <= 1280");
    WLK_CHECK(D.conv_channels % 8 == 0, "conv_channels must be a multiple of 8");
    WLK_CHECK(cfg->max_sessions >= 1 && cfg->max_batch >= 1, "max_sessions / max_batch must be >= 1");

    auto* q = new wlk_qwen();
    q->open(*cfg);
    q->dims = D;
    q->act = cfg->precision == WLK_PREC_BF16 ? DT_BF16 : DT_F32;
    q->gemm_backend = q->act == DT_BF16 && cfg->gemm_backend != WLK_BACKEND_SIMT ? WLK_BACKEND_TCGEN05 : WLK_BACKEND_SIMT;
    q->max_rows = max_rows;
    q->conv_chunks = (int)conv_chunks;
    alloc_weights(q);
    const size_t es = q->es(), R = (size_t)max_rows, CH = conv_chunks;
    const int C = D.conv_channels, d = D.d_model, F = D.n_mels / 8, ffn = D.ffn_dim;
    const int t1 = t0 / 2, t2 = (t1 + 1) / 2, t3 = (t2 + 1) / 2;                 // steps after conv1 / 2 / 3
    size_t* ws = &q->bytes_workspace;
    q->mel = (float*)q->allocs.take(CH * t0 * D.n_mels * 4, ws);
    q->a1 = q->allocs.take(CH * (D.n_mels / 2) * t1 * C * es, ws);
    q->col = q->allocs.take(CH * (D.n_mels / 4) * t2 * 9 * C * es, ws);         // conv2's im2col is the larger one
    q->a2 = q->allocs.take(CH * (D.n_mels / 4) * t2 * C * es, ws);
    q->a3 = q->allocs.take(CH * t3 * F * C * es, ws);
    q->x = (float*)q->allocs.take(R * d * 4, ws);
    q->xn = q->allocs.take(R * d * es, ws);
    q->att = q->allocs.take(R * d * es, ws);
    q->hid = q->allocs.take(R * (size_t)std::max(ffn, d) * es, ws);
    q->outbuf = (float*)q->allocs.take(R * D.out_dim * 4, ws);
    q->audio_scratch = (float*)q->allocs.take((size_t)QMEL_AUDIO_CAP * 4, ws);
    if (q->gemm_backend == WLK_BACKEND_TCGEN05) q->gemm.alloc(q->allocs, ws);
    q->stg.alloc(stg_bytes, q->allocs, ws);
    q->sess.slots.resize(cfg->max_sessions);
    return q;
}

void create(const wlk_qwen_dims* dims, const wlk_config* cfg, wlk_qwen** out) {
    WLK_CHECK(dims && cfg && out, "null argument");
    const wlk_qwen_dims& D = *dims;
    WLK_CHECK(D.chunk_frames == 8, "the conv stem maps exactly 8 mel frames to one step");
    WLK_CHECK(D.block_frames % 8 == 0 && D.block_frames / 8 <= Q_STEPS_CAP, "block_frames must be a multiple of 8 and <= %d", 8 * Q_STEPS_CAP);
    WLK_CHECK(D.mutable_tail_steps >= 0 && D.mutable_tail_steps < Q_STEPS_CAP, "mutable_tail_steps must be in [0, %d)", Q_STEPS_CAP);
    WLK_CHECK(D.mutable_tail_steps == 0 || D.block_frames == 0, "fixed attention blocks and a mutable tail are exclusive");   // causal.py:127-131
    WLK_CHECK(D.left_context_steps >= 1 && D.left_context_steps + Q_STEPS_CAP <= 512, "left_context_steps must be in [1, %d]", 512 - Q_STEPS_CAP);
    const int steps_per_round = D.block_frames > 0 ? D.block_frames / 8 : Q_STEPS_CAP;
    const int max_rows = cfg->max_batch * steps_per_round;
    const size_t R = (size_t)max_rows;
    // a round stages its jobs, K/V pointers, one conv chunk per step and three int32 row maps
    const size_t stg = R * (16 + sizeof(WChunk)) + (size_t)cfg->max_batch * (sizeof(QJob) + sizeof(MelJob) + 64) + 4096;
    wlk_qwen* q = create_common(D, cfg, max_rows, R, 8, stg);
    q->ring = D.left_context_steps + Q_STEPS_CAP;
    size_t* ws = &q->bytes_workspace;
    q->posbuf = (float*)q->allocs.take(R * D.d_model * 4, ws);
    q->qb = q->allocs.take(R * D.d_model * q->es(), ws);
    *out = q;
}

void destroy(wlk_qwen* q) {
    q->close([q] {
        for (auto& s : q->sess) { if (s.kv) cudaFree(s.kv); if (s.win) cudaFree(s.win); if (s.audio) cudaFree(s.audio); if (s.mel_raw) cudaFree(s.mel_raw); if (s.mel_blockmax) cudaFree(s.mel_blockmax); }
        if (q->mel_out) cudaFree(q->mel_out);
    });
    delete q;
}

int grid_1d(int64_t total) { const int64_t b = (total + 255) / 256; return (int)(b > 65535 * 16 ? 65535 * 16 : b); }

// conv2d1 -> im2col -> conv2 GEMM -> im2col -> conv3 GEMM over nc chunks of T0 frames in q->mel; out q->a3, rows
// (chunk, step, f): one step's [F][C] features are one conv_out row
template <typename T, int T0>
void conv_stem(wlk_qwen* q, const WChunk* chunks_dev, int nc) {
    constexpr int T1 = T0 / 2, T2 = (T1 + 1) / 2, T3 = (T2 + 1) / 2;
    const wlk_qwen_dims& D = q->dims;
    const int C = D.conv_channels, F = D.n_mels / 8, F1 = D.n_mels / 2, F2 = D.n_mels / 4;
    qwen_conv1_kernel<T, T0><<<grid_1d((int64_t)nc * F1 * T1 * C), 256, 0, q->st>>>(q->mel, chunks_dev, q->c1w, q->c1b, (T*)q->a1,
                                                                                    nc, D.n_mels, C);
    qwen_im2col_kernel<T><<<grid_1d((int64_t)nc * F2 * T2 * 9 * C), 256, 0, q->st>>>((const T*)q->a1, chunks_dev, (T*)q->col,
                                                                                     nc, F1, T1, 1, C, 0);
    {   GemmArgs g;
        g.A = q->col; g.a_type = q->act; g.lda = 9 * C; g.W = q->W2c; g.w_type = q->act; g.ldw = 9 * C;
        g.M = nc * F2 * T2; g.N = C; g.K = 9 * C;
        g.epi.bias = q->c2b; g.epi.gelu = 1; g.epi.C = q->a2; g.epi.c_type = q->act; g.epi.ldc = C;
        qgemm(q, g); }
    qwen_im2col_kernel<T><<<grid_1d((int64_t)nc * F * T3 * 9 * C), 256, 0, q->st>>>((const T*)q->a2, chunks_dev, (T*)q->col,
                                                                                    nc, F2, T2, 2, C, 1);
    {   GemmArgs g;
        g.A = q->col; g.a_type = q->act; g.lda = 9 * C; g.W = q->W3c; g.w_type = q->act; g.ldw = 9 * C;
        g.M = nc * T3 * F; g.N = C; g.K = 9 * C;
        g.epi.bias = q->c3b; g.epi.gelu = 1; g.epi.C = q->a3; g.epi.c_type = q->act; g.epi.ldc = C;
        qgemm(q, g); }
}

// The QKV projection of layer li over rows [0, R) of xn (causal.py:343-346): bias, head_dim^-0.5 on the q columns;
// dst(epi) points the epilogue at the mode's destination
template <typename QkvDst>
void qkv_gemm(wlk_qwen* q, int li, const void* xn, int R, QkvDst dst) {
    const int d = q->dims.d_model;
    const QLayerW& L = q->L[li];
    GemmArgs g;
    g.A = xn; g.a_type = q->act; g.lda = d; g.W = L.Wqkv; g.w_type = q->act; g.ldw = d;
    g.M = R; g.N = 3 * d; g.K = d;
    g.epi.bias = L.bqkv; g.epi.col_scale = 0.125f; g.epi.scale_cols = d;
    g.epi.c_type = q->act;
    dst(g.epi);
    qgemm(q, g);
}

// The n_layer pre-LN layers over rows [0, R) of q->x (causal.py:378-421): LN, QKV, attention, out-proj + residual, LN,
// fc1 + GELU, fc2 + residual.  qkv_dst(epi, layer) points the QKV GEMM's epilogue at the mode's destination; attend(layer)
// runs the mode's attention from there into q->att.
template <typename QkvDst, typename Attend>
void run_layers(wlk_qwen* q, int R, QkvDst qkv_dst, Attend attend) {
    const wlk_qwen_dims& D = q->dims;
    const int d = D.d_model, ffn = D.ffn_dim;
    for (int li = 0; li < D.n_layer; ++li) {
        QLayerW& L = q->L[li];
        layernorm(q->x, d, L.ln1w, L.ln1b, q->xn, q->act, d, R, d, nullptr, q->st);
        qkv_gemm(q, li, q->xn, R, [&](Epilogue& e) { qkv_dst(e, li); });
        attend(li);
        {   GemmArgs g;
            g.A = q->att; g.a_type = q->act; g.lda = d; g.W = L.Wo; g.w_type = q->act; g.ldw = d;
            g.M = R; g.N = d; g.K = d;
            g.epi.bias = L.bo; g.epi.residual = q->x; g.epi.ldr = d; g.epi.C = q->x; g.epi.c_type = DT_F32; g.epi.ldc = d;
            qgemm(q, g); }
        layernorm(q->x, d, L.ln2w, L.ln2b, q->xn, q->act, d, R, d, nullptr, q->st);
        {   GemmArgs g;
            g.A = q->xn; g.a_type = q->act; g.lda = d; g.W = L.W1; g.w_type = q->act; g.ldw = d;
            g.M = R; g.N = ffn; g.K = d;
            g.epi.bias = L.b1; g.epi.gelu = 1; g.epi.C = q->hid; g.epi.c_type = q->act; g.epi.ldc = ffn;
            qgemm(q, g); }
        {   GemmArgs g;
            g.A = q->hid; g.a_type = q->act; g.lda = ffn; g.W = L.W2; g.w_type = q->act; g.ldw = ffn;
            g.M = R; g.N = d; g.K = ffn;
            g.epi.bias = L.b2; g.epi.residual = q->x; g.epi.ldr = d; g.epi.C = q->x; g.epi.c_type = DT_F32; g.epi.ldc = d;
            qgemm(q, g); }
    }
}

// head: ln_post -> proj1 -> GELU -> proj2 (causal.py:672-676) on `rows` rows of q->x into q->outbuf: rows [0, rows) when
// row_idx is null, else x's rows row_idx[0 .. rows) (row-wise ops: the same values as over every row)
void run_head(wlk_qwen* q, int rows, const int32_t* row_idx) {
    const wlk_qwen_dims& D = q->dims;
    const int d = D.d_model;
    if (rows > 0) {
        layernorm(q->x, d, q->lnpw, q->lnpb, q->xn, q->act, d, rows, d, row_idx, q->st);
        {   GemmArgs g;
            g.A = q->xn; g.a_type = q->act; g.lda = d; g.W = q->Wp1; g.w_type = q->act; g.ldw = d;
            g.M = rows; g.N = d; g.K = d;
            g.epi.bias = q->bp1; g.epi.gelu = 1; g.epi.C = q->hid; g.epi.c_type = q->act; g.epi.ldc = d;
            qgemm(q, g); }
        {   GemmArgs g;
            g.A = q->hid; g.a_type = q->act; g.lda = d; g.W = q->Wp2; g.w_type = q->act; g.ldw = d;
            g.M = rows; g.N = D.out_dim; g.K = d;
            g.epi.bias = q->bp2; g.epi.C = q->outbuf; g.epi.c_type = DT_F32; g.epi.ldc = D.out_dim;
            qgemm(q, g); }
    }
    CUDA_CHECK(cudaGetLastError());
}

// the positional rows of `rows` absolute positions (device array) -> out fp32 [rows][d]
void launch_positions(wlk_qwen* q, const int32_t* pos_dev, float* out, int rows) {
    qwen_pos_kernel<<<rows, 128, 0, q->st>>>(pos_dev, q->pos_table, q->pos_inv, q->dims.max_positions, out, rows, q->dims.d_model);
}

// the causal QKV destination: q -> qout [R][d]; k / v of row r -> ring kv_ptrs[slot[r]], layer li, ring slot ringpos[r]
void causal_qkv_dst(wlk_qwen* q, Epilogue& e, int li, void* qout, void* const* kv_ptrs_dev, const int32_t* slot_dev,
                    const int32_t* ringpos_dev) {
    const wlk_qwen_dims& D = q->dims;
    e.mode = EPI_SELF_QKV; e.C = qout; e.ldc = D.d_model;
    e.batch_ptrs = kv_ptrs_dev; e.row_slot = slot_dev; e.row_pos = ringpos_dev;
    e.layer = li; e.n_head = D.n_head; e.d_model = D.d_model; e.kv_len = q->ring;
}

// the causal attention of a round's jobs at layer li: q act [R][d] -> out act [R][d]
template <typename T>
void launch_causal_attention(wlk_qwen* q, int li, const void* qin, const QJob* jobs_dev, int n_jobs, void* out) {
    const wlk_qwen_dims& D = q->dims;
    qwen_attention_kernel<T><<<dim3(D.n_head, n_jobs), 128, 0, q->st>>>((const T*)qin, jobs_dev, li, D.n_head, D.d_model, q->ring,
                                                                        D.left_context_steps, D.block_bidirectional, (T*)out);
}

// one causal round: R steps, one 8-frame chunk each, staged in q->mel; the sinusoid rows of their absolute positions
// ride into conv_out as the GEMM's residual; the QKV GEMM scatters k / v into the session rings
template <typename T>
void run_round_typed(wlk_qwen* q, int n_jobs, int R, const QJob* jobs_dev, const WChunk* chunks_dev, void* const* kv_ptrs_dev,
                     const int32_t* slot_dev, const int32_t* ringpos_dev, const int32_t* abspos_dev) {
    const wlk_qwen_dims& D = q->dims;
    const int C = D.conv_channels, d = D.d_model, F = D.n_mels / 8;
    conv_stem<T, 8>(q, chunks_dev, R);
    launch_positions(q, abspos_dev, q->posbuf, R);
    {   GemmArgs g;
        g.A = q->a3; g.a_type = q->act; g.lda = (int64_t)F * C; g.W = q->Wout; g.w_type = q->act; g.ldw = (int64_t)F * C;
        g.M = R; g.N = d; g.K = F * C;
        g.epi.bias = D.conv_out_bias ? q->bout : nullptr; g.epi.residual = q->posbuf; g.epi.ldr = d;
        g.epi.C = q->x; g.epi.c_type = DT_F32; g.epi.ldc = d;
        qgemm(q, g); }
    CUDA_CHECK(cudaGetLastError());
    run_layers(q, R, [&](Epilogue& e, int li) { causal_qkv_dst(q, e, li, q->qb, kv_ptrs_dev, slot_dev, ringpos_dev); },
               [&](int li) { launch_causal_attention<T>(q, li, q->qb, jobs_dev, n_jobs, q->att); });
    run_head(q, R, nullptr);
}

// flush = false: forward_chunk (causal.py:713-782).  flush = true: flush_pending (causal.py:687-711) -- no new frames,
// the buffered whole 8-frame chunks are encoded as one piece regardless of the block size, the remainder is dropped.
// out_dev: `out` is device memory (the rows never leave the GPU).
void forward_chunk(wlk_qwen* q, const int32_t* sids, int n, const float* mels, const int32_t* frame_off, float* out,
                   int64_t cap_rows, int32_t* out_row_off, bool flush, bool out_dev = false) {
    const wlk_qwen_dims& D = q->dims;
    WLK_CHECK(q->finalized, "weights not finalized");
    WLK_CHECK(n >= 1 && n <= q->cfg.max_batch, "batch %d outside [1, %d]", n, q->cfg.max_batch);
    const int consume = (D.block_frames > 0 && !flush) ? D.block_frames : 8;
    const int steps_cap = (D.block_frames > 0 && !flush) ? D.block_frames / 8 : Q_STEPS_CAP;
    WLK_CHECK(!q->windowed, "this is a windowed engine: use wlk_qwen_window_forward");
    // append, split off what is ready (reference forward_chunk: causal.py:742-752).  Nothing of a session is committed
    // before the whole call has been validated and run: `rest` / `new_tail` replace pending / tail at the end.
    const int M = flush ? 0 : D.mutable_tail_steps;
    std::vector<std::vector<float>> ready(n), rest(n), new_tail(n);
    std::vector<int> done_steps(n, 0), total_steps(n, 0), freeze(n, 0);
    int64_t rows_total = 0;
    q->sess.check_batch(sids, n);
    for (int i = 0; i < n; ++i) {
        QSession& s = q->sess[sids[i]];
        std::vector<float> all(s.pending);
        if (!flush) {
            const int nf = frame_off[i + 1] - frame_off[i];
            WLK_CHECK(nf >= 0, "negative frame count");
            all.insert(all.end(), mels + (size_t)frame_off[i] * D.n_mels, mels + (size_t)frame_off[i + 1] * D.n_mels);
        }
        const int have = (int)(all.size() / D.n_mels);
        const int take = have / consume * consume;
        if ((D.block_frames == 0 || flush) && D.block_bidirectional)
            WLK_CHECK(take / 8 <= Q_STEPS_CAP, "bidirectional attention over %d steps in one call exceeds %d", take / 8, Q_STEPS_CAP);
        const bool empty_append = !flush && frame_off[i + 1] == frame_off[i];     // causal.py:731-736: touches nothing
        if (M > 0 && empty_append) {
            new_tail[i] = s.tail; total_steps[i] = 0; freeze[i] = 0;
        } else if (M > 0) {
            // _encode_mutable_tail (causal.py:548-640): the previously mutable chunks run again in front of the new ones,
            // at positions emitted .. (emitted counts frozen steps only); one round, so that every step sees the call's keys
            const int tail_steps = (int)(s.tail.size() / ((size_t)8 * D.n_mels));
            ready[i] = s.tail;
            ready[i].insert(ready[i].end(), all.begin(), all.begin() + (size_t)take * D.n_mels);
            total_steps[i] = tail_steps + take / 8;
            WLK_CHECK(total_steps[i] <= Q_STEPS_CAP, "mutable tail + new steps = %d exceed %d per call", total_steps[i], Q_STEPS_CAP);
            freeze[i] = std::max(0, total_steps[i] - M);               // leading blocks frozen until the tail fits (:617-627)
            new_tail[i].assign(ready[i].begin() + (size_t)freeze[i] * 8 * D.n_mels, ready[i].end());
        } else {
            ready[i].assign(all.begin(), all.begin() + (size_t)take * D.n_mels);
            total_steps[i] = take / 8;
        }
        if (!flush) rest[i].assign(all.begin() + (size_t)take * D.n_mels, all.end());   // flush: a sub-chunk remainder carries no decodable content (causal.py:697-705)
        out_row_off[i] = (int32_t)rows_total;
        rows_total += total_steps[i];
    }
    out_row_off[n] = (int32_t)rows_total;
    WLK_CHECK(rows_total <= cap_rows, "output buffer too small: %lld rows needed, %lld given", (long long)rows_total, (long long)cap_rows);
    // rounds
    for (;;) {
        std::vector<int> who;
        for (int i = 0; i < n; ++i) if (done_steps[i] < total_steps[i]) who.push_back(i);
        if (who.empty()) break;
        int nj = (int)who.size();
        Stager sg(q->stg);
        QJob* jobs_dev; QJob* jobs = sg.host<QJob>(nj, &jobs_dev);
        void** kv_dev; void** kvp = sg.host<void*>(nj, &kv_dev);
        int R = 0;
        std::vector<int> steps(nj);
        for (int k = 0; k < nj; ++k) { steps[k] = std::min(steps_cap, total_steps[who[k]] - done_steps[who[k]]); R += steps[k]; }
        if (R > q->max_rows) {                            // a flush may carry up to block-1 frames per session: trim the round
            int acc = 0, keep = 0;
            while (keep < nj && acc + steps[keep] <= q->max_rows) acc += steps[keep++];
            WLK_CHECK(keep >= 1, "round of %d steps exceeds the workspace (%d)", steps[0], q->max_rows);
            who.resize(keep); steps.resize(keep); R = acc; nj = keep;
        }
        WChunk* chunks_dev; WChunk* chunks = sg.host<WChunk>(R, &chunks_dev);
        int32_t *slot_dev, *ring_dev, *abs_dev;
        int32_t* slot = sg.host<int32_t>(R, &slot_dev);
        int32_t* ringpos = sg.host<int32_t>(R, &ring_dev);
        int32_t* abspos = sg.host<int32_t>(R, &abs_dev);
        int r = 0;
        for (int k = 0; k < nj; ++k) {
            const int i = who[k];
            QSession& s = q->sess[sids[i]];
            const int64_t start = s.emitted;
            WLK_CHECK(start + steps[k] < (int64_t)1 << 30, "stream position overflow");
            jobs[k] = QJob{s.kv, (int32_t)start, steps[k], r, 0};
            kvp[k] = s.kv;
            CUDA_CHECK(cudaMemcpyAsync(q->mel + (size_t)r * 8 * D.n_mels, ready[i].data() + (size_t)done_steps[i] * 8 * D.n_mels,
                                       (size_t)steps[k] * 8 * D.n_mels * 4, cudaMemcpyHostToDevice, q->st));
            for (int t = 0; t < steps[k]; ++t, ++r) {
                chunks[r] = WChunk{q->mel + (size_t)r * 8 * D.n_mels, 8, 8, r, 1};
                slot[r] = k; abspos[r] = (int32_t)(start + t); ringpos[r] = (int32_t)((start + t) % q->ring);
            }
        }
        sg.upload(q->st);
        if (q->act == DT_F32) run_round_typed<float>(q, nj, R, jobs_dev, chunks_dev, kv_dev, slot_dev, ring_dev, abs_dev);
        else run_round_typed<bf16>(q, nj, R, jobs_dev, chunks_dev, kv_dev, slot_dev, ring_dev, abs_dev);
        r = 0;
        for (int k = 0; k < nj; ++k) {
            const int i = who[k];
            CUDA_CHECK(cudaMemcpyAsync(out + ((size_t)out_row_off[i] + done_steps[i]) * D.out_dim, q->outbuf + (size_t)r * D.out_dim,
                                       (size_t)steps[k] * D.out_dim * 4, out_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                                       q->st));
            r += steps[k];
            done_steps[i] += steps[k];
            q->sess[sids[i]].emitted += M > 0 ? freeze[i] : steps[k];    // a mutable tail: only the frozen steps count (:638)
        }
        CUDA_CHECK(cudaStreamSynchronize(q->st));        // outbuf is reused by the next round
    }
    for (int i = 0; i < n; ++i) {                        // commit the host-side buffers
        QSession& s = q->sess[sids[i]];
        s.pending.swap(rest[i]);
        if (M > 0) s.tail.swap(new_tail[i]);
    }
}

// StreamingMelExtractor.append / .flush (reference features.py:86-110) for n sessions: the sample windows stay on the
// device, one launch pair featurizes every session's window, the newly determined frames come back [frames][n_mels].
void append_audio(wlk_qwen* q, const int32_t* sids, int n, const float* pcm, const int64_t* sample_off, float* out,
                  int64_t cap_frames, int32_t* frame_off, bool flush) {
    const wlk_qwen_dims& D = q->dims;
    WLK_CHECK(q->weights.loaded.count("mel_filters"), "load the \"mel_filters\" tensor [n_mels][201] before appending audio");
    WLK_CHECK(n >= 1 && n <= q->cfg.max_batch, "batch %d outside [1, %d]", n, q->cfg.max_batch);
    struct Plan { int first, last, frames; };
    std::vector<Plan> plan(n, Plan{0, 0, 0});
    std::vector<int> who;
    int64_t rows = 0;
    q->sess.check_batch(sids, n);
    for (int i = 0; i < n; ++i) {
        QSession& s = q->sess[sids[i]];
        if (!s.audio) {
            CUDA_CHECK(cudaMalloc(&s.audio, (size_t)QMEL_AUDIO_CAP * 4));
            CUDA_CHECK(cudaMalloc(&s.mel_raw, (size_t)MEL_STORE_FRAMES * D.n_mels * 4));
            CUDA_CHECK(cudaMalloc(&s.mel_blockmax, (size_t)(MEL_MAX_CTAS + MEL_MAX_PARTS) * 4));
            q->bytes_sessions += (size_t)QMEL_AUDIO_CAP * 4 + (size_t)(QMEL_MAX_FRAMES + 2) * D.n_mels * 4 + MEL_MAX_CTAS * 4;
        }
        int64_t upto;
        if (!flush) {
            const int64_t ns = sample_off[i + 1] - sample_off[i];
            WLK_CHECK(ns >= 0, "negative sample count");
            WLK_CHECK(s.buf_len + ns <= QMEL_AUDIO_CAP - 2 * N_FFT, "audio window overflow: append at most %d s at a time", QMEL_MAX_FRAMES / 100);
            if (ns) CUDA_CHECK(cudaMemcpyAsync(s.audio + s.buf_len, pcm + sample_off[i], (size_t)ns * 4, cudaMemcpyHostToDevice, q->st));
            s.buf_len += ns; s.total_samples += ns;
            frame_off[i] = (int32_t)rows;
            if (s.total_samples < N_FFT / 2 + 1) continue;                               // features.py:93-94
            upto = std::min((s.total_samples - N_FFT / 2) / HOP + 1, s.total_samples / HOP);   // :95-96
        } else {
            frame_off[i] = (int32_t)rows;
            upto = s.total_samples / HOP;                                                // :103
            if (upto <= s.mel_emitted) continue;
            if (s.buf_len < N_FFT + 1) {                                                 // :106-108 zero-pad a short tail
                CUDA_CHECK(cudaMemsetAsync(s.audio + s.buf_len, 0, (size_t)(N_FFT + 1 - s.buf_len) * 4, q->st));
                s.buf_len = N_FFT + 1;
            }
        }
        if (upto <= s.mel_emitted) continue;                                             // _emit, features.py:62-84
        int64_t first = s.mel_emitted - s.buf_start_frame, last = upto - s.buf_start_frame;
        const int64_t frames = s.buf_len / HOP;
        if (frames < last) { last = frames; upto = s.buf_start_frame + last; if (upto <= s.mel_emitted) continue; }
        WLK_CHECK(frames <= QMEL_MAX_FRAMES, "audio window of %lld frames exceeds %d", (long long)frames, QMEL_MAX_FRAMES);
        plan[i] = Plan{(int)first, (int)last, (int)frames};
        who.push_back(i);
        rows += last - first;
        s.mel_emitted = upto;
    }
    frame_off[n] = (int32_t)rows;
    WLK_CHECK(rows <= cap_frames, "output buffer too small: %lld frames needed, %lld given", (long long)rows, (long long)cap_frames);
    if (who.empty()) { CUDA_CHECK(cudaStreamSynchronize(q->st)); return; }
    const int nj = (int)who.size();
    if ((size_t)rows * D.n_mels > q->mel_out_cap) {
        if (q->mel_out) { CUDA_CHECK(cudaStreamSynchronize(q->st)); cudaFree(q->mel_out); q->mel_out = nullptr; }
        q->mel_out_cap = (size_t)rows * D.n_mels * 2;
        CUDA_CHECK(cudaMalloc(&q->mel_out, q->mel_out_cap * 4));
    }
    Stager sg(q->stg);
    MelJob* mj_dev; MelJob* mj = sg.host<MelJob>(nj, &mj_dev);
    int2* rng_dev; int2* rng = sg.host<int2>(nj, &rng_dev);
    int64_t* ooff_dev; int64_t* ooff = sg.host<int64_t>(nj, &ooff_dev);
    int max_frames = 1;
    for (int k = 0; k < nj; ++k) {
        const int i = who[k];
        QSession& s = q->sess[sids[i]];
        if (plan[i].frames > max_frames) max_frames = plan[i].frames;
        mj[k] = MelJob{s.audio, s.mel_raw, s.mel_blockmax, nullptr, (int32_t)s.buf_len, plan[i].frames, plan[i].frames, 1};
        rng[k] = make_int2(plan[i].first, plan[i].last);
        ooff[k] = frame_off[i];
    }
    sg.upload(q->st);
    mel_window_forward(mj_dev, rng_dev, ooff_dev, q->mel_out, nj, D.n_mels, q->filtT, q->window, q->twiddle, q->filt_span,
                       max_frames, q->st);
    CUDA_CHECK(cudaMemcpyAsync(out, q->mel_out, (size_t)rows * D.n_mels * 4, cudaMemcpyDeviceToHost, q->st));
    // drop the samples no longer needed: keep MARGIN (8) frames of history before the next frame to emit (features.py:77-83)
    for (int k = 0; k < nj; ++k) {
        QSession& s = q->sess[sids[who[k]]];
        const int64_t keep_from = std::max(s.buf_start_frame, s.mel_emitted - 8);
        const int64_t cut = (keep_from - s.buf_start_frame) * HOP;
        if (cut > 0) {
            const int64_t keep = s.buf_len - cut;
            if (keep > 0) {
                CUDA_CHECK(cudaMemcpyAsync(q->audio_scratch, s.audio + cut, (size_t)keep * 4, cudaMemcpyDeviceToDevice, q->st));
                CUDA_CHECK(cudaMemcpyAsync(s.audio, q->audio_scratch, (size_t)keep * 4, cudaMemcpyDeviceToDevice, q->st));
            }
            s.buf_len = keep > 0 ? keep : 0;
            s.buf_start_frame = keep_from;
        }
    }
    CUDA_CHECK(cudaStreamSynchronize(q->st));            // pcm / out belong to the caller; the staging block is reused
}

// =========================================================================================================
// Windowed engine: QwenAudioSurgeryEncoder (reference model.py:441-608) over the stock tower (transformers 5.5
// modeling_qwen3_omni_moe.py:710-768).  Per call, per session: the new frames join the session's device window (the
// last left + right frames); the window is cut into 100-frame chunks from its first frame, the tail chunk zero-padded
// to 100 (a window under 100 frames is one unpadded chunk); conv stem per chunk; the valid steps of every chunk (mod-100
// rule) are compacted with positional rows 0..12; layers with block-diagonal bidirectional attention; the head only on
// the rows the call emits.  All sessions of a call run in one pass, their rows back to back.
//
// Conv stem workspace: rounds of at most QW_CHUNKS_PER_ROUND chunks of conv_stem (im2col + GEMM).  An implicit-GEMM conv would need a new GEMM operand path; a fixed round keeps conv2's im2col at
// QW_CHUNKS_PER_ROUND x 800 x 9C elements (221 MB in bf16 at C = 480) whatever the batch, against 11.5 GB for 128
// sessions' 13 chunks at once, and 32 chunks = 25600 conv2 rows still fill the GEMM grid.
// =========================================================================================================
}  // namespace

// kernels live in wlk's anonymous namespace, like the causal tower's (one anonymous namespace per scope for nvcc's stubs)
namespace wlk {
namespace {

constexpr int QW_T0 = 100, QW_T3 = 13;  // conv chunk frames, steps after conv3
constexpr int QW_CHUNKS_PER_ROUND = 32;
constexpr int QW_KMAX = 256;            // keys one attention block may hold (a full default window is 164 rows)
constexpr int QW_QTILE = 64;            // query rows per attention CTA (4 warps x 16)
constexpr int QW_KSTRIDE = 72;          // smem row pitch (bf16) of the staged K / V: 64 + 8 keeps the fragment loads conflict-free

int window_steps(int64_t frames) {      // _get_feat_extract_output_lengths (mod-100 rule, model.py:164-174)
    if (frames <= 0) return 0;
    const int64_t leave = frames % 100;
    const int64_t feat = (leave - 1 >= 0 ? (leave - 1) / 2 : -1) + 1;        // floor division as torch does it
    const int64_t a = feat - 1 >= 0 ? (feat - 1) / 2 + 1 : 0;                // (feat - 1) // 2 + 1 with feat >= 0
    const int64_t b = a - 1 >= 0 ? (a - 1) / 2 + 1 : 0;
    return (int)std::max<int64_t>(0, b + (frames / 100) * 13);
}

size_t session_bytes(const wlk_qwen* q) {
    if (q->windowed) return (size_t)(q->wd.left_context_frames + q->wd.right_context_frames) * q->dims.n_mels * 4;
    return (size_t)q->dims.n_layer * 2 * q->dims.n_head * q->ring * 64 * q->es();
}

struct WAttn {                          // one query tile of one attention block (device array)
    int32_t row0;                       // first row of the block
    int32_t len;                        // rows (= keys) of the block
    int32_t q0;                         // the tile's first query, relative to row0
    int32_t pad;
};

// mel chunks [n][100][n_mels] from the session windows, zero beyond each chunk's frames
__global__ void qwin_gather_kernel(const WChunk* __restrict__ jobs, float* __restrict__ out, int n, int n_mels) {
    const int64_t total = (int64_t)n * QW_T0 * n_mels;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int m = i % n_mels;
        const int fr = (i / n_mels) % QW_T0;
        const WChunk j = jobs[i / ((int64_t)QW_T0 * n_mels)];
        out[i] = fr < j.avail ? j.src[(int64_t)fr * n_mels + m] : 0.f;
    }
}

// valid-step compaction: x[dst_row + j] = conv_out[chunk][j] + positional row j (rows restart in every chunk)
__global__ void qwin_compact_kernel(const float* __restrict__ xc, const WChunk* __restrict__ jobs, const float* __restrict__ table,
                                    float* __restrict__ x, int d) {
    const WChunk j = jobs[blockIdx.x];
    for (int s = 0; s < j.n_valid; ++s)
        for (int i = threadIdx.x; i < d; i += blockDim.x)
            x[(int64_t)(j.dst_row + s) * d + i] = xc[((int64_t)blockIdx.x * QW_T3 + s) * d + i] + table[(int64_t)s * d + i];
}

// Block-diagonal bidirectional attention, bf16 on tensor cores.  Grid (query tile, head), 4 warps.  The block's K and V
// (<= QW_KMAX rows of one head) are staged once in shared memory; each warp owns 16 query rows and runs mma.sync
// m16n8k16 for S = q k^T and O = P V over 64-key tiles with an fp32 online softmax (P is re-packed from the S
// accumulators, whose fragment layout is the A layout of the next MMA).  q arrives pre-scaled by head_dim^-0.5.
__global__ void __launch_bounds__(128)
qwin_attn_mma_kernel(const bf16* __restrict__ qkv, const WAttn* __restrict__ items, int d, bf16* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char qw_smem[];
    bf16* Ks = reinterpret_cast<bf16*>(qw_smem);
    bf16* Vs = Ks + QW_KMAX * QW_KSTRIDE;
    const WAttn it = items[blockIdx.x];
    const int h = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
    const int64_t ld = 3 * (int64_t)d;
    const int nk = it.len, nkp = (nk + 15) & ~15;
    for (int i = threadIdx.x; i < nkp * 8; i += 128) {
        const int r = i >> 3, c = (i & 7) * 8;
        uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
        if (r < nk) {
            const bf16* row = qkv + (int64_t)(it.row0 + r) * ld + h * 64 + c;
            kv = *reinterpret_cast<const uint4*>(row + d);
            vv = *reinterpret_cast<const uint4*>(row + 2 * d);
        }
        *reinterpret_cast<uint4*>(Ks + r * QW_KSTRIDE + c) = kv;
        *reinterpret_cast<uint4*>(Vs + r * QW_KSTRIDE + c) = vv;
    }
    __syncthreads();
    const int qr = it.q0 + warp * 16;                       // the warp's first query, relative to row0
    if (qr >= nk) return;
    uint32_t qa[4][4];
    {
        const int ra = qr + g, rb = qr + g + 8;
        const bf16* pa = qkv + (int64_t)(it.row0 + ra) * ld + h * 64;
        const bf16* pb = qkv + (int64_t)(it.row0 + rb) * ld + h * 64;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            const int c0 = ks * 16 + tq * 2;
            qa[ks][0] = ra < nk ? *reinterpret_cast<const uint32_t*>(pa + c0) : 0u;
            qa[ks][1] = rb < nk ? *reinterpret_cast<const uint32_t*>(pb + c0) : 0u;
            qa[ks][2] = ra < nk ? *reinterpret_cast<const uint32_t*>(pa + c0 + 8) : 0u;
            qa[ks][3] = rb < nk ? *reinterpret_cast<const uint32_t*>(pb + c0 + 8) : 0u;
        }
    }
    float o[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    for (int kt = 0; kt < nkp; kt += 64) {
        float s[8][4];
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const int kb = kt + nt * 8;
            s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
            if (kb < nkp) {
                const bf16* kr = Ks + (kb + g) * QW_KSTRIDE + tq * 2;
#pragma unroll
                for (int ks = 0; ks < 4; ++ks)
                    ptx::mma_bf16_16816(s[nt], qa[ks], *reinterpret_cast<const uint32_t*>(kr + ks * 16),
                                   *reinterpret_cast<const uint32_t*>(kr + ks * 16 + 8));
            }
            const int k0 = kb + tq * 2;
            if (k0 >= nk) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
            if (k0 + 1 >= nk) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
            mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
            mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float n0 = fmaxf(m0, mx0), n1 = fmaxf(m1, mx1);  // finite: every tile holds at least one key
        const float sc0 = __expf(m0 - n0), sc1 = __expf(m1 - n1);
        m0 = n0; m1 = n1;
        float r0 = 0.f, r1 = 0.f;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            s[nt][0] = __expf(s[nt][0] - n0); s[nt][1] = __expf(s[nt][1] - n0);
            s[nt][2] = __expf(s[nt][2] - n1); s[nt][3] = __expf(s[nt][3] - n1);
            r0 += s[nt][0] + s[nt][1]; r1 += s[nt][2] + s[nt][3];
        }
        r0 += __shfl_xor_sync(0xffffffffu, r0, 1); r0 += __shfl_xor_sync(0xffffffffu, r0, 2);
        r1 += __shfl_xor_sync(0xffffffffu, r1, 1); r1 += __shfl_xor_sync(0xffffffffu, r1, 2);
        l0 = l0 * sc0 + r0; l1 = l1 * sc1 + r1;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) { o[nt][0] *= sc0; o[nt][1] *= sc0; o[nt][2] *= sc1; o[nt][3] *= sc1; }
#pragma unroll
        for (int j = 0; j < 4; ++j) {                          // 16 keys per MMA
            const int kb = kt + j * 16;
            if (kb >= nkp) break;
            const uint32_t pa[4] = {ptx::pack_bf16x2(s[2 * j][0], s[2 * j][1]), ptx::pack_bf16x2(s[2 * j][2], s[2 * j][3]),
                                    ptx::pack_bf16x2(s[2 * j + 1][0], s[2 * j + 1][1]),
                                    ptx::pack_bf16x2(s[2 * j + 1][2], s[2 * j + 1][3])};
            const bf16* v0 = Vs + (kb + tq * 2) * QW_KSTRIDE + g;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const bf16* v = v0 + nt * 8;
                __nv_bfloat162 b0, b1;
                b0.x = v[0]; b0.y = v[QW_KSTRIDE];
                b1.x = v[8 * QW_KSTRIDE]; b1.y = v[9 * QW_KSTRIDE];
                ptx::mma_bf16_16816(o[nt], pa, *reinterpret_cast<uint32_t*>(&b0), *reinterpret_cast<uint32_t*>(&b1));
            }
        }
    }
    const float i0 = 1.f / l0, i1 = 1.f / l1;
    const int ra = qr + g, rb = qr + g + 8;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
        const int c = h * 64 + nt * 8 + tq * 2;
        if (ra < nk) *reinterpret_cast<__nv_bfloat162*>(out + (int64_t)(it.row0 + ra) * d + c) = __floats2bfloat162_rn(o[nt][0] * i0, o[nt][1] * i0);
        if (rb < nk) *reinterpret_cast<__nv_bfloat162*>(out + (int64_t)(it.row0 + rb) * d + c) = __floats2bfloat162_rn(o[nt][2] * i1, o[nt][3] * i1);
    }
}

// The fp32 parity variant: SIMT, one warp per query row (attend_row_warp), keys read from global memory.
__global__ void __launch_bounds__(128)
qwin_attn_simt_kernel(const float* __restrict__ qkv, const WAttn* __restrict__ items, int d, float* __restrict__ out) {
    __shared__ float qs[4][64];
    const WAttn it = items[blockIdx.x];
    const int h = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t ld = 3 * (int64_t)d;
    const float* kbase = qkv + (int64_t)it.row0 * ld + d + h * 64;
    const float* vbase = kbase + d;
    const int nk = it.len;
    for (int qi = it.q0 + warp; qi < min(nk, it.q0 + QW_QTILE); qi += 4) {
        const float* qrow = qkv + (int64_t)(it.row0 + qi) * ld + h * 64;
        qs[warp][lane] = qrow[lane];
        qs[warp][lane + 32] = qrow[lane + 32];
        __syncwarp();
        attend_row_warp<float, QW_KMAX / 32>(qs[warp], nk, [&](int ki) { return kbase + ki * ld; },
                                             [&](int ki) { return vbase + ki * ld; },
                                             out + (int64_t)(it.row0 + qi) * d + h * 64);
        __syncwarp();
    }
}

}  // namespace
}  // namespace wlk

namespace {

// the query tiles of stream blocks: stream i owns rows [row_off[i], row_off[i] + rows[i]), blocks of `block[i]` rows
void attn_items(const std::vector<int>& row_off, const std::vector<int>& rows, const std::vector<int>& block, std::vector<WAttn>& items) {
    items.clear();
    for (size_t i = 0; i < rows.size(); ++i) {
        const int blk = block[i] > 0 ? block[i] : rows[i];
        for (int b0 = 0; b0 < rows[i]; b0 += blk) {
            const int len = std::min(blk, rows[i] - b0);
            WLK_CHECK(len <= QW_KMAX, "attention block of %d rows exceeds %d", len, QW_KMAX);
            for (int q0 = 0; q0 < len; q0 += QW_QTILE) items.push_back(WAttn{row_off[i] + b0, len, q0, 0});
        }
    }
}

constexpr int QW_ATTN_SMEM = 2 * QW_KMAX * QW_KSTRIDE * 2;      // staged K and V of one block, bf16

// the mel frames of nc windowed chunks -> q->mel [nc][100][n_mels], zero at and past each chunk's avail
void launch_gather(wlk_qwen* q, const WChunk* chunks_dev, int nc) {
    qwin_gather_kernel<<<grid_1d((int64_t)nc * QW_T0 * q->dims.n_mels), 256, 0, q->st>>>(chunks_dev, q->mel, nc, q->dims.n_mels);
}

// the bf16 kernel's dynamic shared memory exceeds the default 48 KB: opt in once per device (at create, or per op call)
void window_attention_opt_in() {
    CUDA_CHECK(cudaFuncSetAttribute(qwin_attn_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, QW_ATTN_SMEM));
}

void launch_window_attention(int act, const void* qkv, const WAttn* items_dev, int n_items, int n_head, int d, void* out,
                             cudaStream_t st) {
    if (n_items == 0) return;
    if (act == DT_BF16) {
        const int smem = QW_ATTN_SMEM;
        qwin_attn_mma_kernel<<<dim3(n_items, n_head), 128, smem, st>>>((const bf16*)qkv, items_dev, d, (bf16*)out);
    } else {
        qwin_attn_simt_kernel<<<dim3(n_items, n_head), 128, 0, st>>>((const float*)qkv, items_dev, d, (float*)out);
    }
    CUDA_CHECK(cudaGetLastError());
}

void create_window(const wlk_qwen_window_dims* wdims, const wlk_config* cfg, wlk_qwen** out) {
    WLK_CHECK(wdims && cfg && out, "null argument");
    const wlk_qwen_window_dims& W = *wdims;
    WLK_CHECK(W.n_window == 50, "the mod-100 length rule needs n_window = 50 (100-frame chunks), got %d", W.n_window);
    WLK_CHECK(W.n_window_infer == 0 || W.n_window_infer >= 2 * W.n_window, "n_window_infer must be 0 or >= %d", 2 * W.n_window);
    WLK_CHECK(W.left_context_frames > 0 && W.right_context_frames >= 0, "left_context_frames must be > 0, right >= 0");
    WLK_CHECK(W.max_positions >= QW_T3, "the positional table needs at least %d rows", QW_T3);
    const int wframes = W.left_context_frames + W.right_context_frames;
    const int wrows = window_steps(wframes);
    const int chunks_per_block = W.n_window_infer / (2 * W.n_window);
    WLK_CHECK(std::min(wrows, W.n_window_infer ? QW_T3 * chunks_per_block : wrows) <= QW_KMAX,
              "attention blocks of more than %d rows are not supported", QW_KMAX);
    const wlk_qwen_dims D{W.n_mels, W.conv_channels, W.d_model, W.n_head, W.n_layer, W.ffn_dim, W.out_dim, W.max_positions,
                          8, 0, 1, 1, W.conv_out_bias, 0};
    const size_t R = (size_t)cfg->max_batch * wrows;
    const size_t max_chunks = (size_t)cfg->max_batch * ((wframes + QW_T0 - 1) / QW_T0);
    const size_t max_items = (size_t)cfg->max_batch * ((wrows + QW_QTILE - 1) / QW_QTILE + wrows);
    const size_t stg = R * 4 + max_chunks * sizeof(WChunk) + max_items * sizeof(WAttn) + (size_t)cfg->max_batch * (sizeof(MelJob) + 64) + 4096;
    wlk_qwen* q = create_common(D, cfg, (int)R, QW_CHUNKS_PER_ROUND, QW_T0, stg);
    q->windowed = true; q->wd = W;
    q->win_rows = wrows;
    q->win_block_chunks = chunks_per_block;
    if (q->act == DT_BF16) window_attention_opt_in();
    size_t* ws = &q->bytes_workspace;
    q->xc = (float*)q->allocs.take((size_t)QW_CHUNKS_PER_ROUND * QW_T3 * W.d_model * 4, ws);
    q->qkv = q->allocs.take(R * 3 * W.d_model * q->es(), ws);
    q->win_scratch = (float*)q->allocs.take((size_t)wframes * W.n_mels * 4, ws);
    *out = q;
}

// The tower over n windows (device pointers, win_len frames each, all > 0), rows emitted per window = [lo, hi) of its
// rows.  The emitted rows land in q->outbuf, back to back in window order; returns their count.
template <typename T>
int64_t run_windows(wlk_qwen* q, const std::vector<const float*>& wins, const std::vector<int>& wlen,
                    const std::vector<int>& lo, const std::vector<int>& hi) {
    const wlk_qwen_window_dims& W = q->wd;
    const int n = (int)wins.size();
    const int C = W.conv_channels, d = W.d_model, F = W.n_mels / 8, H = W.n_head;
    std::vector<int> row_off(n), rows(n), block(n);
    std::vector<WChunk> chunks;
    int R = 0;
    for (int i = 0; i < n; ++i) {
        row_off[i] = R;
        rows[i] = window_steps(wlen[i]);
        const int p0 = wlen[i] >= QW_T0 ? QW_T0 : wlen[i];
        for (int c = 0; c * QW_T0 < wlen[i]; ++c) {
            const int avail = std::min(QW_T0, wlen[i] - c * QW_T0);
            chunks.push_back(WChunk{wins[i] + (size_t)c * QW_T0 * W.n_mels, avail, p0, R + c * QW_T3, window_steps(avail)});
        }
        block[i] = q->win_block_chunks ? window_steps(p0) * q->win_block_chunks : 0;   // modeling_qwen3_omni_moe.py:748
        R += rows[i];
    }
    WLK_CHECK(R <= q->max_rows, "%d rows exceed the workspace (%d)", R, q->max_rows);
    std::vector<WAttn> items;
    attn_items(row_off, rows, block, items);
    std::vector<int32_t> emit;
    for (int i = 0; i < n; ++i) for (int r = lo[i]; r < hi[i]; ++r) emit.push_back(row_off[i] + r);
    const int E = (int)emit.size();
    Stager sg(q->stg);
    WChunk* chunks_dev; WAttn* items_dev; int32_t* emit_dev;
    memcpy(sg.host<WChunk>(chunks.size(), &chunks_dev), chunks.data(), chunks.size() * sizeof(WChunk));
    memcpy(sg.host<WAttn>(items.size(), &items_dev), items.data(), items.size() * sizeof(WAttn));
    memcpy(sg.host<int32_t>(E, &emit_dev), emit.data(), (size_t)E * 4);
    sg.upload(q->st);
    // conv stem, in rounds of at most QW_CHUNKS_PER_ROUND chunks
    for (size_t c0 = 0; c0 < chunks.size(); c0 += QW_CHUNKS_PER_ROUND) {
        const int nc = (int)std::min<size_t>(QW_CHUNKS_PER_ROUND, chunks.size() - c0);
        const WChunk* jd = chunks_dev + c0;
        launch_gather(q, jd, nc);
        conv_stem<T, QW_T0>(q, jd, nc);
        {   GemmArgs g;
            g.A = q->a3; g.a_type = q->act; g.lda = (int64_t)F * C; g.W = q->Wout; g.w_type = q->act; g.ldw = (int64_t)F * C;
            g.M = nc * QW_T3; g.N = d; g.K = F * C;
            g.epi.bias = W.conv_out_bias ? q->bout : nullptr; g.epi.C = q->xc; g.epi.c_type = DT_F32; g.epi.ldc = d;
            qgemm(q, g); }
        qwin_compact_kernel<<<nc, 128, 0, q->st>>>(q->xc, jd, q->pos_table, q->x, d);
        CUDA_CHECK(cudaGetLastError());
    }
    // pre-LN layers, block-diagonal attention; the head on the emitted rows only
    run_layers(q, R, [&](Epilogue& e, int) { e.C = q->qkv; e.ldc = 3 * d; },
               [&](int) { launch_window_attention(q->act, q->qkv, items_dev, (int)items.size(), H, d, q->att, q->st); });
    run_head(q, E, emit_dev);
    return E;
}

int64_t run_windows_any(wlk_qwen* q, const std::vector<const float*>& wins, const std::vector<int>& wlen,
                        const std::vector<int>& lo, const std::vector<int>& hi) {
    if (wins.empty()) return 0;
    return q->act == DT_F32 ? run_windows<float>(q, wins, wlen, lo, hi) : run_windows<bf16>(q, wins, wlen, lo, hi);
}

// QwenAudioSurgeryEncoder.forward_chunk (model.py:559-608) for n sessions
void window_forward(wlk_qwen* q, const int32_t* sids, int n, const float* mels, const int32_t* frame_off, float* out,
                    int64_t cap_rows, int32_t* out_row_off, bool out_dev) {
    const wlk_qwen_window_dims& W = q->wd;
    WLK_CHECK(q->windowed, "not a windowed engine: use wlk_qwen_forward_chunk");
    WLK_CHECK(q->finalized, "weights not finalized");
    WLK_CHECK(n >= 1 && n <= q->cfg.max_batch, "batch %d outside [1, %d]", n, q->cfg.max_batch);
    const int wframes = W.left_context_frames + W.right_context_frames;
    struct Plan { int nf, keep, drop_old, lo, hi, take; };
    std::vector<Plan> plan(n);
    int64_t rows_total = 0;
    q->sess.check_batch(sids, n);
    for (int i = 0; i < n; ++i) {                            // validate and plan; no session changes before the encode
        QSession& s = q->sess[sids[i]];
        const int nf = frame_off[i + 1] - frame_off[i];
        WLK_CHECK(nf >= 0, "negative frame count");
        Plan p{nf, (int)s.win_len, 0, 0, 0, 0};
        if (nf > 0) {
            const int64_t all = s.win_len + nf, len = std::min<int64_t>(all, wframes), drop = all - len;
            p.drop_old = (int)std::min<int64_t>(drop, s.win_len);
            p.keep = (int)(s.win_len - p.drop_old);
            const int64_t start = s.window_start + drop, seen = s.frames_seen + nf;
            const int ws = window_steps(start), fin = window_steps(std::max<int64_t>(0, seen - W.right_context_frames));
            const int nrows = window_steps(len);
            const int64_t e = std::max<int64_t>(s.emitted, ws) - ws;
            p.lo = (int)std::max<int64_t>(0, std::min<int64_t>(e, nrows));
            p.hi = std::max(p.lo, std::min(fin - ws, nrows));
            p.take = std::min(nf, wframes - p.keep);          // the newest frames that stay in the window
        }
        out_row_off[i] = (int32_t)rows_total;
        rows_total += p.hi - p.lo;
        plan[i] = p;
    }
    out_row_off[n] = (int32_t)rows_total;
    WLK_CHECK(rows_total <= cap_rows, "output buffer too small: %lld rows needed, %lld given", (long long)rows_total, (long long)cap_rows);
    // The device windows take the new frames, the tower encodes them, and only then do the session counters advance.
    // If the encode fails, the sessions that took frames are reset to the empty state (their device windows no longer
    // match their counters) and the error propagates.
    std::vector<const float*> wins;
    std::vector<int> wlen, lo, hi;
    const size_t fb = (size_t)W.n_mels * 4;
    try {
        for (int i = 0; i < n; ++i) {
            const Plan& p = plan[i];
            if (p.nf == 0) continue;                          // model.py:568-570: nothing changes
            QSession& s = q->sess[sids[i]];
            if (p.drop_old > 0 && p.keep > 0) {               // slide the kept frames to the front (via the scratch)
                CUDA_CHECK(cudaMemcpyAsync(q->win_scratch, s.win + (size_t)p.drop_old * W.n_mels, p.keep * fb, cudaMemcpyDeviceToDevice, q->st));
                CUDA_CHECK(cudaMemcpyAsync(s.win, q->win_scratch, p.keep * fb, cudaMemcpyDeviceToDevice, q->st));
            }
            CUDA_CHECK(cudaMemcpyAsync(s.win + (size_t)p.keep * W.n_mels, mels + ((size_t)frame_off[i + 1] - p.take) * W.n_mels,
                                       p.take * fb, cudaMemcpyHostToDevice, q->st));
            if (p.hi > p.lo) { wins.push_back(s.win); wlen.push_back(p.keep + p.take); lo.push_back(p.lo); hi.push_back(p.hi); }
        }
        const int64_t E = run_windows_any(q, wins, wlen, lo, hi);
        if (E) CUDA_CHECK(cudaMemcpyAsync(out, q->outbuf, (size_t)E * W.out_dim * 4,
                                          out_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, q->st));
        CUDA_CHECK(cudaStreamSynchronize(q->st));        // mels / out belong to the caller; the staging block is reused
    } catch (...) {
        for (int i = 0; i < n; ++i) {
            if (plan[i].nf == 0) continue;
            QSession& s = q->sess[sids[i]];
            s.win_len = s.frames_seen = s.window_start = s.emitted = s.last_in = s.last_rec = s.last_ctx = 0;
        }
        throw;
    }
    for (int i = 0; i < n; ++i) {                            // commit (model.py:573-607)
        const Plan& p = plan[i];
        if (p.nf == 0) continue;
        QSession& s = q->sess[sids[i]];
        s.window_start += s.win_len + p.nf - (p.keep + p.take);
        s.win_len = p.keep + p.take;
        s.frames_seen += p.nf;
        s.last_in = p.nf; s.last_rec = s.win_len; s.last_ctx = std::max<int64_t>(0, s.last_rec - s.last_in);
        if (p.hi > p.lo) s.emitted = window_steps(s.window_start) + p.hi;
    }
}

// forward_full (model.py:556-557) over stateless windows of at most left + right frames each (the workspace is sized for
// such windows); the call's windows are copied into a device buffer allocated for the call
void window_encode(wlk_qwen* q, int n, const float* mels, const int32_t* frame_off, float* out, int64_t cap_rows,
                   int32_t* out_row_off) {
    const wlk_qwen_window_dims& W = q->wd;
    WLK_CHECK(q->windowed, "not a windowed engine");
    WLK_CHECK(q->finalized, "weights not finalized");
    WLK_CHECK(n >= 1 && n <= q->cfg.max_batch, "batch %d outside [1, %d]", n, q->cfg.max_batch);
    const int wframes = W.left_context_frames + W.right_context_frames;
    int64_t rows_total = 0, frames_total = 0;
    for (int i = 0; i < n; ++i) {
        const int nf = frame_off[i + 1] - frame_off[i];
        WLK_CHECK(nf >= 0 && nf <= wframes, "window %d holds %d frames, outside [0, %d]", i, nf, wframes);
        out_row_off[i] = (int32_t)rows_total;
        rows_total += window_steps(nf);
        frames_total += nf;
    }
    out_row_off[n] = (int32_t)rows_total;
    WLK_CHECK(rows_total <= cap_rows, "output buffer too small: %lld rows needed, %lld given", (long long)rows_total, (long long)cap_rows);
    if (rows_total == 0) return;
    struct Staged { float* p = nullptr; ~Staged() { if (p) cudaFree(p); } } stage;   // one call's windows
    CUDA_CHECK(cudaMalloc(&stage.p, (size_t)frames_total * W.n_mels * 4));
    float* staged = stage.p;
    std::vector<const float*> wins;
    std::vector<int> wlen, lo, hi;
    CUDA_CHECK(cudaMemcpyAsync(staged, mels + (size_t)frame_off[0] * W.n_mels, (size_t)frames_total * W.n_mels * 4,
                               cudaMemcpyHostToDevice, q->st));
    for (int i = 0; i < n; ++i) {
        const int nf = frame_off[i + 1] - frame_off[i];
        if (nf == 0) continue;
        wins.push_back(staged + (size_t)(frame_off[i] - frame_off[0]) * W.n_mels);
        wlen.push_back(nf); lo.push_back(0); hi.push_back(window_steps(nf));
    }
    const int64_t E = run_windows_any(q, wins, wlen, lo, hi);
    CUDA_CHECK(cudaMemcpyAsync(out, q->outbuf, (size_t)E * W.out_dim * 4, cudaMemcpyDeviceToHost, q->st));
    CUDA_CHECK(cudaStreamSynchronize(q->st));
}

// ---- op-level entry points (kernel tests): one production launch on caller-owned device buffers, with the engine's
//      dims, precision and GEMM backend, on its stream, synchronized before returning ---------------------------------
void op_require(const wlk_qwen* q, std::initializer_list<std::string> names) {
    for (const std::string& n : names) WLK_CHECK(q->weights.loaded.count(n), "tensor %s is not loaded", n.c_str());
}

void op_positions(wlk_qwen* q, const int32_t* pos, int rows, float* out) {
    WLK_CHECK(pos && out, "null argument");
    WLK_CHECK(rows >= 1 && rows <= (1 << 20), "rows %d outside [1, %d]", rows, 1 << 20);
    op_require(q, {"positional_embedding.positional_embedding"});
    for (int r = 0; r < rows; ++r) WLK_CHECK(pos[r] >= 0 && pos[r] < (1 << 30), "row %d: position %d outside [0, 2^30)", r, pos[r]);
    OpUpload up{q->st};
    launch_positions(q, up.put(pos, rows), out, rows);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(q->st));
}

void op_conv_stem(wlk_qwen* q, const float* mel, const int32_t* avail, const int32_t* p0, int n, void* a1, void* a2, void* a3) {
    const wlk_qwen_dims& D = q->dims;
    WLK_CHECK(mel && avail && p0 && a1 && a2 && a3, "null argument");
    WLK_CHECK(n >= 1 && n <= q->conv_chunks, "%d chunks outside [1, %d] (the conv stem's workspace)", n, q->conv_chunks);
    op_require(q, {"conv2d1.weight", "conv2d1.bias", "conv2d2.weight", "conv2d2.bias", "conv2d3.weight", "conv2d3.bias"});
    const int T0 = q->windowed ? QW_T0 : 8;
    std::vector<WChunk> chunks(n);
    for (int k = 0; k < n; ++k) {
        if (q->windowed)
            WLK_CHECK(avail[k] >= 1 && avail[k] <= p0[k] && p0[k] <= T0, "chunk %d: avail %d, p0 %d (need 1 <= avail <= p0 <= %d)",
                      k, avail[k], p0[k], T0);
        else
            WLK_CHECK(avail[k] == 8 && p0[k] == 8, "chunk %d: a causal chunk is 8 frames (avail %d, p0 %d)", k, avail[k], p0[k]);
        chunks[k] = WChunk{mel + (size_t)k * T0 * D.n_mels, avail[k], p0[k], k, 0};
    }
    OpUpload up{q->st};
    const WChunk* chunks_dev = up.put(chunks.data(), n);
    if (q->windowed) launch_gather(q, chunks_dev, n);
    else CUDA_CHECK(cudaMemcpyAsync(q->mel, mel, (size_t)n * 8 * D.n_mels * 4, cudaMemcpyDeviceToDevice, q->st));
    if (q->act == DT_F32) { if (q->windowed) conv_stem<float, QW_T0>(q, chunks_dev, n); else conv_stem<float, 8>(q, chunks_dev, n); }
    else { if (q->windowed) conv_stem<bf16, QW_T0>(q, chunks_dev, n); else conv_stem<bf16, 8>(q, chunks_dev, n); }
    CUDA_CHECK(cudaGetLastError());
    const int T1 = T0 / 2, T2 = (T1 + 1) / 2, T3 = (T2 + 1) / 2;
    const size_t row = (size_t)D.conv_channels * q->es();
    CUDA_CHECK(cudaMemcpyAsync(a1, q->a1, (size_t)n * (D.n_mels / 2) * T1 * row, cudaMemcpyDeviceToDevice, q->st));
    CUDA_CHECK(cudaMemcpyAsync(a2, q->a2, (size_t)n * (D.n_mels / 4) * T2 * row, cudaMemcpyDeviceToDevice, q->st));
    CUDA_CHECK(cudaMemcpyAsync(a3, q->a3, (size_t)n * T3 * (D.n_mels / 8) * row, cudaMemcpyDeviceToDevice, q->st));
    CUDA_CHECK(cudaStreamSynchronize(q->st));
}

void op_qkv(wlk_qwen* q, int layer, const void* xn, const int32_t* slot, const int32_t* pos, int rows, void* const* kv,
            int n_slots, void* qout) {
    WLK_CHECK(!q->windowed, "a windowed engine has no K/V rings");
    WLK_CHECK(xn && slot && pos && kv && qout, "null argument");
    WLK_CHECK(layer >= 0 && layer < q->dims.n_layer, "layer %d outside [0, %d)", layer, q->dims.n_layer);
    WLK_CHECK(rows >= 1 && rows <= q->max_rows, "rows %d outside [1, %d]", rows, q->max_rows);
    WLK_CHECK(n_slots >= 1, "no K/V rings");
    const std::string p = "layers." + std::to_string(layer) + ".self_attn.";
    op_require(q, {p + "q_proj.weight", p + "k_proj.weight", p + "v_proj.weight", p + "q_proj.bias", p + "k_proj.bias",
                   p + "v_proj.bias"});
    std::vector<int32_t> ringpos(rows);
    for (int r = 0; r < rows; ++r) {
        WLK_CHECK(slot[r] >= 0 && slot[r] < n_slots, "row %d: slot %d outside [0, %d)", r, slot[r], n_slots);
        WLK_CHECK(kv[slot[r]] != nullptr, "row %d: slot %d has no K/V ring", r, slot[r]);
        WLK_CHECK(pos[r] >= 0 && pos[r] < (1 << 30), "row %d: position %d outside [0, 2^30)", r, pos[r]);
        ringpos[r] = pos[r] % q->ring;
    }
    OpUpload up{q->st};
    const int32_t* slot_d = up.put(slot, rows);
    const int32_t* ring_d = up.put(ringpos.data(), rows);
    void* const* kv_d = up.put(kv, n_slots);
    qkv_gemm(q, layer, xn, rows, [&](Epilogue& e) { causal_qkv_dst(q, e, layer, qout, kv_d, slot_d, ring_d); });
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(q->st));
}

void op_attention(wlk_qwen* q, int layer, const void* qin, const int32_t* start, const int32_t* n_steps, int n_jobs,
                  void* const* kv, void* out) {
    WLK_CHECK(!q->windowed, "a windowed engine has no K/V rings");
    WLK_CHECK(n_jobs >= 1 && n_jobs <= 65535, "%d jobs outside [1, 65535]", n_jobs);
    WLK_CHECK(qin && start && n_steps && kv && out, "null argument");
    WLK_CHECK(layer >= 0 && layer < q->dims.n_layer, "layer %d outside [0, %d)", layer, q->dims.n_layer);
    std::vector<QJob> jobs(n_jobs);
    int row = 0;
    for (int j = 0; j < n_jobs; ++j) {
        WLK_CHECK(n_steps[j] >= 1 && n_steps[j] <= Q_STEPS_CAP, "job %d: n_steps %d outside [1, %d]", j, n_steps[j], Q_STEPS_CAP);
        WLK_CHECK(start[j] >= 0, "job %d: negative start %d", j, start[j]);
        WLK_CHECK((int64_t)start[j] + n_steps[j] < ((int64_t)1 << 30), "job %d: stream position overflow", j);
        WLK_CHECK(kv[j] != nullptr, "job %d has no K/V ring", j);
        jobs[j] = QJob{kv[j], start[j], n_steps[j], row, 0};
        row += n_steps[j];
    }
    OpUpload up{q->st};
    const QJob* jobs_d = up.put(jobs.data(), n_jobs);
    if (q->act == DT_F32) launch_causal_attention<float>(q, layer, qin, jobs_d, n_jobs, out);
    else launch_causal_attention<bf16>(q, layer, qin, jobs_d, n_jobs, out);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(q->st));
}

}  // namespace

extern "C" {

int wlk_qwen_create(const wlk_qwen_dims* dims, const wlk_config* cfg, wlk_qwen** out) {
    WLK_API_BEGIN
    create(dims, cfg, out);
    WLK_API_END
}
int wlk_qwen_destroy(wlk_qwen* q) {
    WLK_API_BEGIN
    WLK_CHECK(q != nullptr, "null engine");
    CUDA_CHECK(cudaSetDevice(q->cfg.device));
    destroy(q);
    WLK_API_END
}
int wlk_qwen_load_tensor(wlk_qwen* q, const char* name, const float* host, const int64_t* shape, int ndim) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(name && host && shape && ndim >= 1, "bad arguments");
    q->weights.load(name, host, shape, ndim);
    WLK_API_END
}
int wlk_qwen_finalize_weights(wlk_qwen* q) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    q->weights.require_all();
    q->upload.release();
    q->finalized = true;
    WLK_API_END
}
int wlk_qwen_session_open(wlk_qwen* q, int32_t* sid) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(sid, "null out pointer");
    const int found = q->sess.free_slot();
    QSession& s = q->sess[found];
    const size_t bytes = session_bytes(q);
    CUDA_CHECK(cudaMalloc(q->windowed ? (void**)&s.win : &s.kv, bytes));
    q->bytes_sessions += bytes;
    s.open = true; s.emitted = 0; s.pending.clear(); s.tail.clear();
    *sid = found;
    WLK_API_END
}
int wlk_qwen_session_close(wlk_qwen* q, int32_t sid) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    QSession& s = q->sess.at(sid);
    CUDA_CHECK(cudaStreamSynchronize(q->st));
    cudaFree(q->windowed ? (void*)s.win : s.kv);
    q->bytes_sessions -= session_bytes(q);
    if (s.audio) {
        cudaFree(s.audio); cudaFree(s.mel_raw); cudaFree(s.mel_blockmax);
        q->bytes_sessions -= (size_t)QMEL_AUDIO_CAP * 4 + (size_t)(QMEL_MAX_FRAMES + 2) * q->dims.n_mels * 4 + MEL_MAX_CTAS * 4;
    }
    s = QSession{};
    WLK_API_END
}
int wlk_qwen_session_reset(wlk_qwen* q, int32_t sid) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    QSession& s = q->sess.at(sid);
    s.emitted = 0; s.pending.clear(); s.tail.clear();
    s.buf_len = s.buf_start_frame = s.mel_emitted = s.total_samples = 0;       // StreamingMelExtractor.reset, features.py:112
    s.win_len = s.frames_seen = s.window_start = s.last_in = s.last_rec = s.last_ctx = 0;
    WLK_API_END
}
int wlk_qwen_session_state(wlk_qwen* q, int32_t sid, int32_t* pending_frames, int64_t* emitted_steps) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    QSession& s = q->sess.at(sid);
    if (pending_frames) *pending_frames = (int32_t)(s.pending.size() / q->dims.n_mels);
    if (emitted_steps) *emitted_steps = s.emitted;
    WLK_API_END
}
int wlk_qwen_session_mutable_steps(wlk_qwen* q, int32_t sid, int32_t* mutable_steps) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    QSession& s = q->sess.at(sid);
    WLK_CHECK(mutable_steps != nullptr, "null argument");
    *mutable_steps = (int32_t)(s.tail.size() / ((size_t)8 * q->dims.n_mels));
    WLK_API_END
}
int wlk_qwen_forward_chunk(wlk_qwen* q, const int32_t* sids, int n, const float* mels_host, const int32_t* frame_offsets,
                           float* out_host, int64_t out_capacity_rows, int32_t* out_row_offsets) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(sids && frame_offsets && out_row_offsets && (mels_host || frame_offsets[n] == frame_offsets[0]), "null argument");
    WLK_CHECK(out_host || out_capacity_rows == 0, "null output buffer");
    forward_chunk(q, sids, n, mels_host, frame_offsets, out_host, out_capacity_rows, out_row_offsets, false);
    WLK_API_END
}
int wlk_qwen_flush_pending(wlk_qwen* q, const int32_t* sids, int n, float* out_host, int64_t out_capacity_rows,
                           int32_t* out_row_offsets) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(sids && out_row_offsets, "null argument");
    WLK_CHECK(out_host || out_capacity_rows == 0, "null output buffer");
    forward_chunk(q, sids, n, nullptr, nullptr, out_host, out_capacity_rows, out_row_offsets, true);
    WLK_API_END
}
int wlk_qwen_forward_chunk_device(wlk_qwen* q, const int32_t* sids, int n, const float* mels_host, const int32_t* frame_offsets,
                                  float* out_dev, int64_t out_capacity_rows, int32_t* out_row_offsets) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(sids && frame_offsets && out_row_offsets && (mels_host || frame_offsets[n] == frame_offsets[0]), "null argument");
    WLK_CHECK(out_dev || out_capacity_rows == 0, "null output buffer");
    forward_chunk(q, sids, n, mels_host, frame_offsets, out_dev, out_capacity_rows, out_row_offsets, false, true);
    WLK_API_END
}
int wlk_qwen_flush_pending_device(wlk_qwen* q, const int32_t* sids, int n, float* out_dev, int64_t out_capacity_rows,
                                  int32_t* out_row_offsets) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(sids && out_row_offsets, "null argument");
    WLK_CHECK(out_dev || out_capacity_rows == 0, "null output buffer");
    forward_chunk(q, sids, n, nullptr, nullptr, out_dev, out_capacity_rows, out_row_offsets, true, true);
    WLK_API_END
}
int wlk_qwen_session_get_pending(wlk_qwen* q, int32_t sid, float* mels_host, int64_t capacity_frames, int32_t* n_frames) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    QSession& s = q->sess.at(sid);
    WLK_CHECK(n_frames, "null argument");
    const int64_t have = (int64_t)(s.pending.size() / q->dims.n_mels);
    WLK_CHECK(have <= capacity_frames, "%lld pending frames exceed the buffer's %lld", (long long)have, (long long)capacity_frames);
    WLK_CHECK(mels_host || have == 0, "null output buffer");
    if (have) memcpy(mels_host, s.pending.data(), s.pending.size() * 4);
    *n_frames = (int32_t)have;
    WLK_API_END
}
int wlk_qwen_session_set_pending(wlk_qwen* q, int32_t sid, const float* mels_host, int32_t n_frames) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    QSession& s = q->sess.at(sid);
    WLK_CHECK(n_frames >= 0 && (mels_host || n_frames == 0), "bad arguments");
    s.pending.assign(mels_host, mels_host + (size_t)n_frames * q->dims.n_mels);
    WLK_API_END
}
int wlk_qwen_append_audio(wlk_qwen* q, const int32_t* sids, int n, const float* pcm_host, const int64_t* sample_offsets,
                          float* mel_out_host, int64_t out_capacity_frames, int32_t* frame_offsets_out, int32_t flush) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(sids && frame_offsets_out && (flush || sample_offsets), "null argument");
    WLK_CHECK(flush || pcm_host || sample_offsets[n] == sample_offsets[0], "null audio");
    WLK_CHECK(mel_out_host || out_capacity_frames == 0, "null output buffer");
    append_audio(q, sids, n, pcm_host, sample_offsets, mel_out_host, out_capacity_frames, frame_offsets_out, flush != 0);
    WLK_API_END
}
int wlk_qwen_window_create(const wlk_qwen_window_dims* dims, const wlk_config* cfg, wlk_qwen** out) {
    WLK_API_BEGIN
    create_window(dims, cfg, out);
    WLK_API_END
}
int wlk_qwen_window_forward(wlk_qwen* q, const int32_t* sids, int n, const float* mels_host, const int32_t* frame_offsets,
                            float* out, int64_t out_capacity_rows, int32_t* out_row_offsets, int32_t out_dev) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(sids && frame_offsets && out_row_offsets && (mels_host || frame_offsets[n] == frame_offsets[0]), "null argument");
    WLK_CHECK(out || out_capacity_rows == 0, "null output buffer");
    window_forward(q, sids, n, mels_host, frame_offsets, out, out_capacity_rows, out_row_offsets, out_dev != 0);
    WLK_API_END
}
int wlk_qwen_window_encode(wlk_qwen* q, int n, const float* mels_host, const int32_t* frame_offsets, float* out_host,
                           int64_t out_capacity_rows, int32_t* out_row_offsets) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(frame_offsets && out_row_offsets && (mels_host || frame_offsets[n] == frame_offsets[0]), "null argument");
    WLK_CHECK(out_host || out_capacity_rows == 0, "null output buffer");
    window_encode(q, n, mels_host, frame_offsets, out_host, out_capacity_rows, out_row_offsets);
    WLK_API_END
}
int wlk_qwen_window_state(wlk_qwen* q, int32_t sid, int64_t* fields) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(q->windowed, "not a windowed engine");
    WLK_CHECK(fields != nullptr, "null argument");
    QSession& s = q->sess.at(sid);
    const int64_t v[7] = {s.frames_seen, s.window_start, s.emitted, s.last_in, s.last_rec, s.last_ctx, s.win_len};
    memcpy(fields, v, sizeof(v));
    WLK_API_END
}
int wlk_qwen_window_attention(int device, int precision, const void* qkv, void* out, int d_model, const int32_t* stream_rows,
                              int n_streams, int block_rows) {
    WLK_API_BEGIN
    WLK_CHECK(qkv && out && stream_rows && n_streams >= 1 && d_model % 64 == 0 && block_rows >= 0, "bad arguments");
    use_device(device);
    if (precision != WLK_PREC_FP32) window_attention_opt_in();
    std::vector<int> row_off(n_streams), rows(n_streams), block(n_streams, block_rows);
    int r = 0;
    for (int i = 0; i < n_streams; ++i) { WLK_CHECK(stream_rows[i] >= 0, "negative row count"); row_off[i] = r; rows[i] = stream_rows[i]; r += rows[i]; }
    std::vector<WAttn> items;
    attn_items(row_off, rows, block, items);
    if (items.empty()) return 0;
    WAttn* items_dev = nullptr;
    CUDA_CHECK(cudaMalloc(&items_dev, items.size() * sizeof(WAttn)));
    cudaError_t ce = cudaMemcpy(items_dev, items.data(), items.size() * sizeof(WAttn), cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) {
        try {
            launch_window_attention(precision == WLK_PREC_FP32 ? DT_F32 : DT_BF16, qkv, items_dev, (int)items.size(),
                                    d_model / 64, d_model, out, nullptr);
            ce = cudaDeviceSynchronize();
        } catch (...) { cudaFree(items_dev); throw; }
    }
    cudaFree(items_dev);
    CUDA_CHECK(ce);
    WLK_API_END
}
int wlk_qwen_op_positions(wlk_qwen* q, const int32_t* pos_host, int32_t rows, float* out_dev) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    op_positions(q, pos_host, rows, out_dev);
    WLK_API_END
}
int wlk_qwen_op_conv_stem(wlk_qwen* q, const float* mel_dev, const int32_t* avail_host, const int32_t* p0_host, int32_t n_chunks,
                          void* a1_dev, void* a2_dev, void* a3_dev) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    op_conv_stem(q, mel_dev, avail_host, p0_host, n_chunks, a1_dev, a2_dev, a3_dev);
    WLK_API_END
}
int wlk_qwen_op_qkv(wlk_qwen* q, int32_t layer, const void* xn_dev, const int32_t* slot_host, const int32_t* pos_host, int32_t rows,
                    void* const* kv_ptrs_host, int32_t n_slots, void* q_out_dev) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    op_qkv(q, layer, xn_dev, slot_host, pos_host, rows, kv_ptrs_host, n_slots, q_out_dev);
    WLK_API_END
}
int wlk_qwen_op_attention(wlk_qwen* q, int32_t layer, const void* q_dev, const int32_t* start_host, const int32_t* n_steps_host,
                          int32_t n_jobs, void* const* kv_ptrs_host, void* out_dev) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    op_attention(q, layer, q_dev, start_host, n_steps_host, n_jobs, kv_ptrs_host, out_dev);
    WLK_API_END
}
int wlk_qwen_memory(wlk_qwen* q, size_t* weights, size_t* sessions, size_t* workspace) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    q->memory(weights, sessions, workspace);
    WLK_API_END
}

}  // extern "C"
