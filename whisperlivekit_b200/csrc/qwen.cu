// Qwen3-ASR causal-KV audio tower (SURVEY.md section 8 row a17) behind the C ABI (wlk_qwen_* in include/wlk_b200.h).
//   reference third_party/qwen3-asr-causal/src/qwen3_asr_causal/causal.py:
//     forward_chunk :713-782, _encode_ready_mels :642-681, _conv_one_block :230-248, _position_embedding :204-228,
//     _attention_chunk :292-376, _layer_chunk :378-421
// Append-only execution: every mel frame transits the tower exactly once.  Sessions are batched per "round":
// round r holds the r-th ready block (or run of chunks) of every session in the call, so a block always finds
// the K/V its predecessor left in the session's ring.
//
// Data layout (per round, R = encoder steps in the round, one step = one 8-frame mel chunk):
//   mel chunks   fp32 [R][8 frames][n_mels]                      (H2D from the caller's buffer)
//   conv stem    NHWC activations [R][F][T][C]; conv2 / conv3 are im2col + GEMM (K = 9C, taps-major so a tap is one
//                contiguous run of C channels), conv_out is a GEMM over [R][F*C] with its weight columns permuted
//                from the reference's (c, f) order at load time; the sinusoid rows ride in as the GEMM's residual
//   residual x   fp32 [R][d];  q [R][d];  K/V rings per session [L][K|V][H][ring][64], ring = left_context + 128
//                slots addressed by position % ring (written by the QKV GEMM's scatter epilogue)
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include "../../include/wlk_b200.h"
#include "host.cuh"
#include "kernels.cuh"

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

// ---------------------------------------------------------------------------------------------------------
// conv2d1: 1 -> C channels, 3x3, stride 2, pad 1, GELU.  in: chunk [T0 frames][n_mels] (mel index = conv "height").
// out: NHWC [F1][T1][C] with F1 = n_mels/2, T1 = T0/2.
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void qwen_conv1_kernel(const float* __restrict__ mel, const float* __restrict__ w, const float* __restrict__ b,
                                  T* __restrict__ out, int n_chunks, int n_mels, int t0, int C) {
    const int F1 = n_mels / 2, T1 = t0 / 2;
    const int64_t total = (int64_t)n_chunks * F1 * T1 * C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = i % C;
        int64_t r = i / C;
        const int t = r % T1; r /= T1;
        const int f = r % F1;
        const int64_t ch = r / F1;
        const float* x = mel + ch * t0 * n_mels;
        float acc = b[c];
#pragma unroll
        for (int kf = 0; kf < 3; ++kf) {
            const int m = 2 * f - 1 + kf;
            if (m < 0 || m >= n_mels) continue;
#pragma unroll
            for (int kt = 0; kt < 3; ++kt) {
                const int fr = 2 * t - 1 + kt;
                if (fr < 0 || fr >= t0) continue;
                acc = fmaf(w[c * 9 + kf * 3 + kt], x[fr * n_mels + m], acc);
            }
        }
        out[i] = from_f32<T>(gelu_erf(acc));
    }
}

// im2col for a 3x3 / stride 2 / pad 1 conv over NHWC [n][Fi][Ti][C] -> rows (n, fo, to), columns (tap, c)
template <typename T>
__global__ void qwen_im2col_kernel(const T* __restrict__ src, T* __restrict__ dst, int n, int Fi, int Ti, int C) {
    const int Fo = Fi / 2, To = (Ti + 1) / 2;
    const int64_t total = (int64_t)n * Fo * To * 9 * C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = i % C;
        int64_t r = i / C;
        const int tap = r % 9; r /= 9;
        const int to = r % To; r /= To;
        const int fo = r % Fo;
        const int64_t ch = r / Fo;
        const int f = 2 * fo - 1 + tap / 3, t = 2 * to - 1 + tap % 3;
        T v = from_f32<T>(0.f);
        if (f >= 0 && f < Fi && t >= 0 && t < Ti) v = src[((ch * Fi + f) * Ti + t) * C + c];
        dst[i] = v;
    }
}

// positional rows: table[pos] while pos is inside the table, else the closed form (reference causal.py:204-228)
__global__ void qwen_pos_kernel(const int32_t* __restrict__ pos, const float* __restrict__ table, int max_positions,
                                float* __restrict__ out, int rows, int d) {
    const int r = blockIdx.x;
    if (r >= rows) return;
    const int p = pos[r];
    const int half = d / 2;
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
        float v;
        if (p < max_positions) {
            v = table[(int64_t)p * d + i];
        } else {
            const int j = i < half ? i : i - half;
            const float inv = expf(-logf(10000.0f) / (float)max(1, half - 1) * (float)j);
            const float a = (float)p * inv;
            v = i < half ? sinf(a) : cosf(a);
        }
        out[(int64_t)r * d + i] = v;
    }
}

// ---------------------------------------------------------------------------------------------------------
// Attention of one round (reference causal.py:292-376): a query at position p sees keys at positions
//   [p - left_ctx + 1, block_max]   (block-bidirectional)   or   [p - left_ctx + 1, p]   (causal),
// clipped at 0; keys live in the session's ring at slot = position % ring (this round's keys were written by the
// QKV GEMM).  q arrives pre-scaled by head_dim^-0.5.  One warp per query, grid (head, job); fp32 softmax.
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128)
qwen_attention_kernel(const T* __restrict__ q, const QJob* __restrict__ jobs, int layer, int n_head, int d_model, int ring,
                      int left_ctx, int bidir, T* __restrict__ out) {
    constexpr int MAXK = 16;                    // keys per lane: ring <= 512
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
        const int nk = hi - lo + 1;
        float sc[MAXK];
        float mx = -INFINITY;
#pragma unroll
        for (int j = 0; j < MAXK; ++j) {
            const int ki = lane + 32 * j;
            sc[j] = -INFINITY;
            if (ki < nk) {
                const T* kr = kbase + (int64_t)((lo + ki) % ring) * 64;
                float acc = 0.f;
#pragma unroll 8
                for (int e = 0; e < 64; ++e) acc = fmaf(qs[warp][e], to_f32(kr[e]), acc);
                sc[j] = acc;
                mx = fmaxf(mx, acc);
            }
        }
        mx = warp_max(mx);
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < MAXK; ++j) {
            const float pexp = (lane + 32 * j < nk) ? expf(sc[j] - mx) : 0.f;
            sc[j] = pexp;
            sum += pexp;
        }
        sum = warp_sum(sum);
        float o0 = 0.f, o1 = 0.f;
#pragma unroll
        for (int j = 0; j < MAXK; ++j) {
            if (32 * j >= nk) break;
            for (int l = 0; l < 32; ++l) {
                const int ki = 32 * j + l;
                if (ki >= nk) break;
                const float pw = __shfl_sync(0xffffffffu, sc[j], l);
                const T* vr = vbase + (int64_t)((lo + ki) % ring) * 64;
                o0 = fmaf(pw, to_f32(vr[2 * lane]), o0);
                o1 = fmaf(pw, to_f32(vr[2 * lane + 1]), o1);
            }
        }
        const float inv = 1.0f / sum;
        out[row * d_model + h * 64 + 2 * lane] = from_f32<T>(o0 * inv);
        out[row * d_model + h * 64 + 2 * lane + 1] = from_f32<T>(o1 * inv);
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
};

}  // namespace
}  // namespace wlk

using namespace wlk;

struct wlk_qwen {
    wlk_qwen_dims dims{};
    wlk_config cfg{};
    int act = DT_F32, gemm_backend = WLK_BACKEND_SIMT, num_sms = 132;
    int ring = 0, max_rows = 0;
    cudaStream_t st = nullptr;
    std::mutex mu;
    DeviceAllocs allocs;
    size_t bytes_weights = 0, bytes_sessions = 0, bytes_workspace = 0;
    // weights
    float *c1w = nullptr, *c1b = nullptr, *c2b = nullptr, *c3b = nullptr, *bout = nullptr, *pos_table = nullptr;
    void *W2c = nullptr, *W3c = nullptr, *Wout = nullptr, *Wp1 = nullptr, *Wp2 = nullptr;
    float *lnpw = nullptr, *lnpb = nullptr, *bp1 = nullptr, *bp2 = nullptr;
    float *filtT = nullptr, *window = nullptr; float2* twiddle = nullptr; int2* filt_span = nullptr;   // mel front end
    bool have_filters = false;
    float* mel_out = nullptr; size_t mel_out_cap = 0; float* audio_scratch = nullptr;
    std::vector<QLayerW> L;
    std::set<std::string> loaded;
    bool finalized = false;
    WeightUpload upload;
    // sessions and workspaces
    std::vector<QSession> sess;
    float *mel = nullptr, *x = nullptr, *posbuf = nullptr, *outbuf = nullptr;
    void *a1 = nullptr, *col = nullptr, *a2 = nullptr, *a3 = nullptr, *xn = nullptr, *qb = nullptr, *att = nullptr, *hid = nullptr;
    void *qkv_scratch = nullptr;
    float* sk_scratch = nullptr; int* sk_counters = nullptr;      // this engine's split-K workspace (GemmArgs)
    uint8_t *stg_h = nullptr, *stg_d = nullptr; size_t stg_bytes = 0;
    size_t es() const { return dtype_size(act); }
};

namespace {

void qgemm(wlk_qwen* q, GemmArgs& g) {
    if (g.M <= 0) return;
    g.sk_scratch = q->sk_scratch; g.sk_scratch_floats = SK_SCRATCH_FLOATS;
    g.sk_counters = q->sk_counters; g.sk_max_tiles = SK_MAX_TILES;
    if (q->gemm_backend == WLK_BACKEND_TCGEN05 && gemm_tcgen05_supported(g, nullptr)) gemm_tcgen05(g, q->st, q->num_sms);
    else gemm_simt(g, q->st);
}

void load_tensor(wlk_qwen* q, const std::string& name, const float* host, const int64_t* shape, int ndim) {
    const wlk_qwen_dims& D = q->dims;
    const int C = D.conv_channels, d = D.d_model, F = D.n_mels / 8, ffn = D.ffn_dim;
    const int64_t n = numel(shape, ndim);
    auto mat = [&](void* dst, int64_t rows, int64_t cols) { expect_shape(name.c_str(), shape, ndim, {rows, cols}); q->upload.put(host, n, dst, q->act, q->st); };
    auto vec = [&](float* dst, int64_t len) { expect_shape(name.c_str(), shape, ndim, {len}); q->upload.put(host, n, dst, DT_F32, q->st); };
    if (name == "mel_filters") {
        // optional: only wlk_qwen_append_audio needs it.  [n_mels][201] (Slaney filterbank of the feature extractor)
        expect_shape(name.c_str(), shape, ndim, {D.n_mels, N_FREQ});
        std::vector<float> t((size_t)n);
        std::vector<int2> span(D.n_mels);
        for (int m = 0; m < D.n_mels; ++m) {
            int lo = N_FREQ, hi = 0;
            for (int k = 0; k < N_FREQ; ++k) {
                t[(size_t)k * D.n_mels + m] = host[(size_t)m * N_FREQ + k];
                if (host[(size_t)m * N_FREQ + k] != 0.f) { if (k < lo) lo = k; hi = k + 1; }
            }
            if (lo >= hi) { lo = 0; hi = 0; }
            span[m] = make_int2(lo, hi);
        }
        q->upload.put(t.data(), n, q->filtT, DT_F32, q->st);
        CUDA_CHECK(cudaMemcpyAsync(q->filt_span, span.data(), span.size() * 8, cudaMemcpyHostToDevice, q->st));
        CUDA_CHECK(cudaStreamSynchronize(q->st));
        q->have_filters = true;
    }
    else if (name == "conv2d1.weight") { expect_shape(name.c_str(), shape, ndim, {C, 1, 3, 3}); q->upload.put(host, n, q->c1w, DT_F32, q->st); }
    else if (name == "conv2d1.bias") vec(q->c1b, C);
    else if (name == "conv2d2.weight" || name == "conv2d3.weight") {
        // [Co][Ci][3][3] -> [Co][tap][Ci]: a tap's input channels are contiguous, like the im2col rows
        expect_shape(name.c_str(), shape, ndim, {C, C, 3, 3});
        std::vector<float> packed((size_t)n);
        for (int co = 0; co < C; ++co)
            for (int ci = 0; ci < C; ++ci)
                for (int tap = 0; tap < 9; ++tap)
                    packed[((size_t)co * 9 + tap) * C + ci] = host[((size_t)co * C + ci) * 9 + tap];
        q->upload.put(packed.data(), n, name == "conv2d2.weight" ? q->W2c : q->W3c, q->act, q->st);
    }
    else if (name == "conv2d2.bias") vec(q->c2b, C);
    else if (name == "conv2d3.bias") vec(q->c3b, C);
    else if (name == "conv_out.weight") {
        // the reference flattens [C][F] (channel-major, causal.py:240-242); activations here are [F][C]
        expect_shape(name.c_str(), shape, ndim, {d, (int64_t)C * F});
        std::vector<float> packed((size_t)n);
        for (int o = 0; o < d; ++o)
            for (int c = 0; c < C; ++c)
                for (int f = 0; f < F; ++f)
                    packed[(size_t)o * C * F + (size_t)f * C + c] = host[(size_t)o * C * F + (size_t)c * F + f];
        q->upload.put(packed.data(), n, q->Wout, q->act, q->st);
    }
    else if (name == "conv_out.bias") { WLK_CHECK(D.conv_out_bias, "this geometry has no conv_out bias"); vec(q->bout, d); }
    else if (name == "positional_embedding.positional_embedding") {
        expect_shape(name.c_str(), shape, ndim, {D.max_positions, d});
        q->upload.put(host, n, q->pos_table, DT_F32, q->st);
    }
    else if (name == "ln_post.weight") vec(q->lnpw, d);
    else if (name == "ln_post.bias") vec(q->lnpb, d);
    else if (name == "proj1.weight") mat(q->Wp1, d, d);
    else if (name == "proj1.bias") vec(q->bp1, d);
    else if (name == "proj2.weight") mat(q->Wp2, D.out_dim, d);
    else if (name == "proj2.bias") vec(q->bp2, D.out_dim);
    else if (name.rfind("layers.", 0) == 0) {
        const size_t dot = name.find('.', 7);
        WLK_CHECK(dot != std::string::npos, "unknown tensor %s", name.c_str());
        const int li = atoi(name.substr(7, dot - 7).c_str());
        WLK_CHECK(li >= 0 && li < D.n_layer, "layer index out of range in %s", name.c_str());
        const std::string rest = name.substr(dot + 1);
        QLayerW& Lw = q->L[li];
        const size_t es = q->es();
        auto part = [&](int which, bool is_weight) {            // q / k / v rows of the fused projection
            if (is_weight) { expect_shape(name.c_str(), shape, ndim, {d, d}); q->upload.put(host, n, (char*)Lw.Wqkv + (size_t)which * d * d * es, q->act, q->st); }
            else { expect_shape(name.c_str(), shape, ndim, {d}); q->upload.put(host, n, Lw.bqkv + (size_t)which * d, DT_F32, q->st); }
        };
        if (rest == "self_attn.q_proj.weight") part(0, true);
        else if (rest == "self_attn.k_proj.weight") part(1, true);
        else if (rest == "self_attn.v_proj.weight") part(2, true);
        else if (rest == "self_attn.q_proj.bias") part(0, false);
        else if (rest == "self_attn.k_proj.bias") part(1, false);
        else if (rest == "self_attn.v_proj.bias") part(2, false);
        else if (rest == "self_attn.out_proj.weight") mat(Lw.Wo, d, d);
        else if (rest == "self_attn.out_proj.bias") vec(Lw.bo, d);
        else if (rest == "self_attn_layer_norm.weight") vec(Lw.ln1w, d);
        else if (rest == "self_attn_layer_norm.bias") vec(Lw.ln1b, d);
        else if (rest == "final_layer_norm.weight") vec(Lw.ln2w, d);
        else if (rest == "final_layer_norm.bias") vec(Lw.ln2b, d);
        else if (rest == "fc1.weight") mat(Lw.W1, ffn, d);
        else if (rest == "fc1.bias") vec(Lw.b1, ffn);
        else if (rest == "fc2.weight") mat(Lw.W2, d, ffn);
        else if (rest == "fc2.bias") vec(Lw.b2, d);
        else WLK_CHECK(false, "unknown tensor %s", name.c_str());
    }
    else WLK_CHECK(false, "unknown tensor %s", name.c_str());
    q->loaded.insert(name);
}

std::vector<std::string> required(const wlk_qwen_dims& D) {
    std::vector<std::string> r = {"conv2d1.weight", "conv2d1.bias", "conv2d2.weight", "conv2d2.bias", "conv2d3.weight",
                                  "conv2d3.bias", "conv_out.weight", "positional_embedding.positional_embedding",
                                  "ln_post.weight", "ln_post.bias", "proj1.weight", "proj1.bias", "proj2.weight", "proj2.bias"};
    if (D.conv_out_bias) r.push_back("conv_out.bias");
    for (int i = 0; i < D.n_layer; ++i) {
        const std::string p = "layers." + std::to_string(i) + ".";
        for (const char* s : {"self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.out_proj", "fc1", "fc2",
                              "self_attn_layer_norm", "final_layer_norm"}) {
            r.push_back(p + s + ".weight");
            r.push_back(p + s + ".bias");
        }
    }
    return r;
}

void create(const wlk_qwen_dims* dims, const wlk_config* cfg, wlk_qwen** out) {
    WLK_CHECK(dims && cfg && out, "null argument");
    const wlk_qwen_dims& D = *dims;
    WLK_CHECK(D.n_mels % 8 == 0 && D.n_mels >= 8, "n_mels must be a multiple of 8");
    WLK_CHECK(D.chunk_frames == 8, "the conv stem maps exactly 8 mel frames to one step");
    WLK_CHECK(D.d_model % 64 == 0 && D.d_model / D.n_head == 64 && D.d_model <= 1280, "heads must be 64 wide, d_model <= 1280");
    WLK_CHECK(D.conv_channels % 8 == 0, "conv_channels must be a multiple of 8");
    WLK_CHECK(D.block_frames % 8 == 0 && D.block_frames / 8 <= Q_STEPS_CAP, "block_frames must be a multiple of 8 and <= %d", 8 * Q_STEPS_CAP);
    WLK_CHECK(D.mutable_tail_steps >= 0 && D.mutable_tail_steps < Q_STEPS_CAP, "mutable_tail_steps must be in [0, %d)", Q_STEPS_CAP);
    WLK_CHECK(D.mutable_tail_steps == 0 || D.block_frames == 0, "fixed attention blocks and a mutable tail are exclusive");   // causal.py:127-131
    WLK_CHECK(D.left_context_steps >= 1 && D.left_context_steps + Q_STEPS_CAP <= 512, "left_context_steps must be in [1, %d]", 512 - Q_STEPS_CAP);
    WLK_CHECK(cfg->max_sessions >= 1 && cfg->max_batch >= 1, "max_sessions / max_batch must be >= 1");
    const int num_sms = open_sm90_device(cfg->device);

    auto* q = new wlk_qwen();
    q->dims = D; q->cfg = *cfg;
    q->num_sms = num_sms;
    q->act = cfg->precision == WLK_PREC_BF16 ? DT_BF16 : DT_F32;
    q->gemm_backend = q->act == DT_BF16 && cfg->gemm_backend != WLK_BACKEND_SIMT ? WLK_BACKEND_TCGEN05 : WLK_BACKEND_SIMT;
    q->ring = D.left_context_steps + Q_STEPS_CAP;
    const int steps_per_round = D.block_frames > 0 ? D.block_frames / 8 : Q_STEPS_CAP;
    q->max_rows = cfg->max_batch * steps_per_round;
    CUDA_CHECK(cudaStreamCreateWithFlags(&q->st, cudaStreamNonBlocking));
    const size_t es = q->es();
    const int C = D.conv_channels, d = D.d_model, F = D.n_mels / 8, ffn = D.ffn_dim;
    size_t* aw = &q->bytes_weights;
    q->c1w = (float*)q->allocs.take((size_t)C * 9 * 4, aw); q->c1b = (float*)q->allocs.take(C * 4, aw);
    q->c2b = (float*)q->allocs.take(C * 4, aw); q->c3b = (float*)q->allocs.take(C * 4, aw);
    q->W2c = q->allocs.take((size_t)C * 9 * C * es, aw); q->W3c = q->allocs.take((size_t)C * 9 * C * es, aw);
    q->Wout = q->allocs.take((size_t)d * C * F * es, aw); q->bout = (float*)q->allocs.take(d * 4, aw);
    q->pos_table = (float*)q->allocs.take((size_t)D.max_positions * d * 4, aw);
    q->lnpw = (float*)q->allocs.take(d * 4, aw); q->lnpb = (float*)q->allocs.take(d * 4, aw);
    q->Wp1 = q->allocs.take((size_t)d * d * es, aw); q->bp1 = (float*)q->allocs.take(d * 4, aw);
    q->Wp2 = q->allocs.take((size_t)D.out_dim * d * es, aw); q->bp2 = (float*)q->allocs.take(D.out_dim * 4, aw);
    q->L.resize(D.n_layer);
    for (auto& Lw : q->L) {
        Lw.Wqkv = q->allocs.take((size_t)3 * d * d * es, aw); Lw.bqkv = (float*)q->allocs.take(3 * d * 4, aw);
        Lw.Wo = q->allocs.take((size_t)d * d * es, aw); Lw.bo = (float*)q->allocs.take(d * 4, aw);
        Lw.W1 = q->allocs.take((size_t)ffn * d * es, aw); Lw.b1 = (float*)q->allocs.take(ffn * 4, aw);
        Lw.W2 = q->allocs.take((size_t)d * ffn * es, aw); Lw.b2 = (float*)q->allocs.take(d * 4, aw);
        Lw.ln1w = (float*)q->allocs.take(d * 4, aw); Lw.ln1b = (float*)q->allocs.take(d * 4, aw);
        Lw.ln2w = (float*)q->allocs.take(d * 4, aw); Lw.ln2b = (float*)q->allocs.take(d * 4, aw);
    }
    const size_t R = (size_t)q->max_rows;
    size_t* ws = &q->bytes_workspace;
    q->mel = (float*)q->allocs.take(R * 8 * D.n_mels * 4, ws);
    q->a1 = q->allocs.take(R * (D.n_mels / 2) * 4 * C * es, ws);
    q->col = q->allocs.take(R * (D.n_mels / 4) * 2 * 9 * C * es, ws);              // conv2's im2col is the larger one
    q->a2 = q->allocs.take(R * (D.n_mels / 4) * 2 * C * es, ws);
    q->a3 = q->allocs.take(R * F * C * es, ws);
    q->posbuf = (float*)q->allocs.take(R * d * 4, ws);
    q->x = (float*)q->allocs.take(R * d * 4, ws);
    q->xn = q->allocs.take(R * d * es, ws); q->qb = q->allocs.take(R * d * es, ws); q->att = q->allocs.take(R * d * es, ws);
    q->hid = q->allocs.take(R * (size_t)(ffn > d ? ffn : d) * es, ws);
    q->outbuf = (float*)q->allocs.take(R * D.out_dim * 4, ws);
    q->filtT = (float*)q->allocs.take((size_t)N_FREQ * D.n_mels * 4, aw);
    q->window = (float*)q->allocs.take(N_FFT * 4, aw);
    q->twiddle = (float2*)q->allocs.take(N_FFT * 8, aw);
    q->filt_span = (int2*)q->allocs.take((size_t)D.n_mels * 8, aw);
    q->audio_scratch = (float*)q->allocs.take((size_t)QMEL_AUDIO_CAP * 4, ws);
    if (q->gemm_backend == WLK_BACKEND_TCGEN05) {
        q->sk_scratch = (float*)q->allocs.take(SK_SCRATCH_FLOATS * 4, ws);
        q->sk_counters = (int*)q->allocs.take(SK_MAX_TILES * 4, ws);
    }
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
    q->stg_bytes = R * 16 + (size_t)cfg->max_batch * (sizeof(QJob) + sizeof(MelJob) + 64) + 4096;
    CUDA_CHECK(cudaMallocHost(&q->stg_h, q->stg_bytes));
    q->stg_d = (uint8_t*)q->allocs.take(q->stg_bytes, ws);
    q->sess.resize(cfg->max_sessions);
    *out = q;
}

void destroy(wlk_qwen* q) {
    cudaStreamSynchronize(q->st);
    for (auto& s : q->sess) { if (s.kv) cudaFree(s.kv); if (s.audio) cudaFree(s.audio); if (s.mel_raw) cudaFree(s.mel_raw); if (s.mel_blockmax) cudaFree(s.mel_blockmax); }
    if (q->mel_out) cudaFree(q->mel_out);
    q->allocs.free_all();
    q->upload.release();
    if (q->stg_h) cudaFreeHost(q->stg_h);
    cudaStreamDestroy(q->st);
    delete q;
}

QSession& qsession(wlk_qwen* q, int32_t sid) {
    WLK_CHECK(sid >= 0 && sid < (int)q->sess.size() && q->sess[sid].open, "invalid session id %d", sid);
    return q->sess[sid];
}

template <typename T>
void run_round_typed(wlk_qwen* q, int n_jobs, int R, const QJob* jobs_dev, void* const* kv_ptrs_dev, const int32_t* slot_dev,
                     const int32_t* ringpos_dev, const int32_t* abspos_dev) {
    const wlk_qwen_dims& D = q->dims;
    const int C = D.conv_channels, d = D.d_model, F = D.n_mels / 8, ffn = D.ffn_dim, H = D.n_head;
    const int F1 = D.n_mels / 2, F2 = D.n_mels / 4;
    auto blocks = [](int64_t total) { int64_t b = (total + 255) / 256; return (int)(b > 65535 * 16 ? 65535 * 16 : b); };
    // conv stem
    qwen_conv1_kernel<T><<<blocks((int64_t)R * F1 * 4 * C), 256, 0, q->st>>>(q->mel, q->c1w, q->c1b, (T*)q->a1, R, D.n_mels, 8, C);
    qwen_im2col_kernel<T><<<blocks((int64_t)R * F2 * 2 * 9 * C), 256, 0, q->st>>>((const T*)q->a1, (T*)q->col, R, F1, 4, C);
    {   GemmArgs g;
        g.A = q->col; g.a_type = q->act; g.lda = 9 * C; g.W = q->W2c; g.w_type = q->act; g.ldw = 9 * C;
        g.M = R * F2 * 2; g.N = C; g.K = 9 * C;
        g.epi.bias = q->c2b; g.epi.gelu = 1; g.epi.C = q->a2; g.epi.c_type = q->act; g.epi.ldc = C;
        qgemm(q, g); }
    qwen_im2col_kernel<T><<<blocks((int64_t)R * F * 1 * 9 * C), 256, 0, q->st>>>((const T*)q->a2, (T*)q->col, R, F2, 2, C);
    {   GemmArgs g;
        g.A = q->col; g.a_type = q->act; g.lda = 9 * C; g.W = q->W3c; g.w_type = q->act; g.ldw = 9 * C;
        g.M = R * F; g.N = C; g.K = 9 * C;
        g.epi.bias = q->c3b; g.epi.gelu = 1; g.epi.C = q->a3; g.epi.c_type = q->act; g.epi.ldc = C;
        qgemm(q, g); }
    qwen_pos_kernel<<<R, 128, 0, q->st>>>(abspos_dev, q->pos_table, D.max_positions, q->posbuf, R, d);
    {   GemmArgs g;
        g.A = q->a3; g.a_type = q->act; g.lda = (int64_t)F * C; g.W = q->Wout; g.w_type = q->act; g.ldw = (int64_t)F * C;
        g.M = R; g.N = d; g.K = F * C;
        g.epi.bias = D.conv_out_bias ? q->bout : nullptr; g.epi.residual = q->posbuf; g.epi.ldr = d;
        g.epi.C = q->x; g.epi.c_type = DT_F32; g.epi.ldc = d;
        qgemm(q, g); }
    CUDA_CHECK(cudaGetLastError());
    // transformer layers with the per-session K/V rings
    for (int li = 0; li < D.n_layer; ++li) {
        QLayerW& L = q->L[li];
        layernorm(q->x, d, L.ln1w, L.ln1b, q->xn, q->act, d, R, d, nullptr, q->st);
        {   GemmArgs g;
            g.A = q->xn; g.a_type = q->act; g.lda = d; g.W = L.Wqkv; g.w_type = q->act; g.ldw = d;
            g.M = R; g.N = 3 * d; g.K = d;
            g.epi.bias = L.bqkv; g.epi.col_scale = 0.125f; g.epi.scale_cols = d;          // head_dim^-0.5 on q (causal.py:343-346)
            g.epi.mode = EPI_SELF_QKV; g.epi.C = q->qb; g.epi.ldc = d; g.epi.c_type = q->act;
            g.epi.batch_ptrs = kv_ptrs_dev; g.epi.row_slot = slot_dev; g.epi.row_pos = ringpos_dev;
            g.epi.layer = li; g.epi.n_head = H; g.epi.d_model = d; g.epi.kv_len = q->ring;
            qgemm(q, g); }
        qwen_attention_kernel<T><<<dim3(H, n_jobs), 128, 0, q->st>>>((const T*)q->qb, jobs_dev, li, H, d, q->ring,
                                                                    D.left_context_steps, D.block_bidirectional, (T*)q->att);
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
    // head: ln_post -> proj1 -> GELU -> proj2 (causal.py:672-676)
    layernorm(q->x, d, q->lnpw, q->lnpb, q->xn, q->act, d, R, d, nullptr, q->st);
    {   GemmArgs g;
        g.A = q->xn; g.a_type = q->act; g.lda = d; g.W = q->Wp1; g.w_type = q->act; g.ldw = d;
        g.M = R; g.N = d; g.K = d;
        g.epi.bias = q->bp1; g.epi.gelu = 1; g.epi.C = q->hid; g.epi.c_type = q->act; g.epi.ldc = d;
        qgemm(q, g); }
    {   GemmArgs g;
        g.A = q->hid; g.a_type = q->act; g.lda = d; g.W = q->Wp2; g.w_type = q->act; g.ldw = d;
        g.M = R; g.N = D.out_dim; g.K = d;
        g.epi.bias = q->bp2; g.epi.C = q->outbuf; g.epi.c_type = DT_F32; g.epi.ldc = D.out_dim;
        qgemm(q, g); }
    CUDA_CHECK(cudaGetLastError());
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
    // append, split off what is ready (reference forward_chunk: causal.py:742-752).  Nothing of a session is committed
    // before the whole call has been validated and run: `rest` / `new_tail` replace pending / tail at the end.
    const int M = flush ? 0 : D.mutable_tail_steps;
    std::vector<std::vector<float>> ready(n), rest(n), new_tail(n);
    std::vector<int> done_steps(n, 0), total_steps(n, 0), freeze(n, 0);
    int64_t rows_total = 0;
    for (int i = 0; i < n; ++i) {
        QSession& s = qsession(q, sids[i]);
        for (int j = 0; j < i; ++j) WLK_CHECK(sids[j] != sids[i], "session %d appears twice in the batch", sids[i]);
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
        // carve the staging block
        size_t off = 0;
        auto carve = [&](size_t bytes) { size_t o = (off + 255) / 256 * 256; off = o + bytes; WLK_CHECK(off <= q->stg_bytes, "staging overflow"); return o; };
        const size_t o_jobs = carve(nj * sizeof(QJob)), o_kv = carve(nj * sizeof(void*));
        int R = 0;
        std::vector<int> steps(nj);
        for (int k = 0; k < nj; ++k) { steps[k] = std::min(steps_cap, total_steps[who[k]] - done_steps[who[k]]); R += steps[k]; }
        if (R > q->max_rows) {                            // a flush may carry up to block-1 frames per session: trim the round
            int acc = 0, keep = 0;
            while (keep < nj && acc + steps[keep] <= q->max_rows) acc += steps[keep++];
            WLK_CHECK(keep >= 1, "round of %d steps exceeds the workspace (%d)", steps[0], q->max_rows);
            who.resize(keep); steps.resize(keep); R = acc; nj = keep;
        }
        const size_t o_slot = carve((size_t)R * 4), o_ring = carve((size_t)R * 4), o_abs = carve((size_t)R * 4);
        QJob* jobs = reinterpret_cast<QJob*>(q->stg_h + o_jobs);
        void** kvp = reinterpret_cast<void**>(q->stg_h + o_kv);
        int32_t* slot = reinterpret_cast<int32_t*>(q->stg_h + o_slot);
        int32_t* ringpos = reinterpret_cast<int32_t*>(q->stg_h + o_ring);
        int32_t* abspos = reinterpret_cast<int32_t*>(q->stg_h + o_abs);
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
                slot[r] = k; abspos[r] = (int32_t)(start + t); ringpos[r] = (int32_t)((start + t) % q->ring);
            }
        }
        CUDA_CHECK(cudaMemcpyAsync(q->stg_d, q->stg_h, off, cudaMemcpyHostToDevice, q->st));
        const QJob* jobs_dev = reinterpret_cast<const QJob*>(q->stg_d + o_jobs);
        void* const* kv_dev = reinterpret_cast<void* const*>(q->stg_d + o_kv);
        const int32_t* slot_dev = reinterpret_cast<const int32_t*>(q->stg_d + o_slot);
        const int32_t* ring_dev = reinterpret_cast<const int32_t*>(q->stg_d + o_ring);
        const int32_t* abs_dev = reinterpret_cast<const int32_t*>(q->stg_d + o_abs);
        if (q->act == DT_F32) run_round_typed<float>(q, nj, R, jobs_dev, kv_dev, slot_dev, ring_dev, abs_dev);
        else run_round_typed<bf16>(q, nj, R, jobs_dev, kv_dev, slot_dev, ring_dev, abs_dev);
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
        CUDA_CHECK(cudaStreamSynchronize(q->st));        // the staging block and outbuf are reused by the next round
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
    WLK_CHECK(q->have_filters, "load the \"mel_filters\" tensor [n_mels][201] before appending audio");
    WLK_CHECK(n >= 1 && n <= q->cfg.max_batch, "batch %d outside [1, %d]", n, q->cfg.max_batch);
    struct Plan { int first, last, frames; };
    std::vector<Plan> plan(n, Plan{0, 0, 0});
    std::vector<int> who;
    int64_t rows = 0;
    for (int i = 0; i < n; ++i) {
        QSession& s = qsession(q, sids[i]);
        for (int j = 0; j < i; ++j) WLK_CHECK(sids[j] != sids[i], "session %d appears twice in the batch", sids[i]);
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
    size_t off = 0;
    auto carve = [&](size_t bytes) { size_t o = (off + 255) / 256 * 256; off = o + bytes; WLK_CHECK(off <= q->stg_bytes, "staging overflow"); return o; };
    const size_t o_jobs = carve(nj * sizeof(MelJob)), o_rng = carve(nj * sizeof(int2)), o_off = carve(nj * sizeof(int64_t));
    MelJob* mj = reinterpret_cast<MelJob*>(q->stg_h + o_jobs);
    int2* rng = reinterpret_cast<int2*>(q->stg_h + o_rng);
    int64_t* ooff = reinterpret_cast<int64_t*>(q->stg_h + o_off);
    int max_frames = 1;
    for (int k = 0; k < nj; ++k) {
        const int i = who[k];
        QSession& s = q->sess[sids[i]];
        if (plan[i].frames > max_frames) max_frames = plan[i].frames;
        mj[k] = MelJob{s.audio, s.mel_raw, s.mel_blockmax, nullptr, (int32_t)s.buf_len, plan[i].frames, plan[i].frames, 1};
        rng[k] = make_int2(plan[i].first, plan[i].last);
        ooff[k] = frame_off[i];
    }
    CUDA_CHECK(cudaMemcpyAsync(q->stg_d, q->stg_h, off, cudaMemcpyHostToDevice, q->st));
    mel_window_forward(reinterpret_cast<const MelJob*>(q->stg_d + o_jobs), reinterpret_cast<const int2*>(q->stg_d + o_rng),
                       reinterpret_cast<const int64_t*>(q->stg_d + o_off), q->mel_out, nj, D.n_mels, q->filtT, q->window,
                       q->twiddle, q->filt_span, max_frames, q->st);
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
    load_tensor(q, name, host, shape, ndim);
    WLK_API_END
}
int wlk_qwen_finalize_weights(wlk_qwen* q) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    require_loaded(q->loaded, required(q->dims));
    q->upload.release();
    q->finalized = true;
    WLK_API_END
}
int wlk_qwen_session_open(wlk_qwen* q, int32_t* sid) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    WLK_CHECK(sid, "null out pointer");
    int found = -1;
    for (int i = 0; i < (int)q->sess.size(); ++i) if (!q->sess[i].open) { found = i; break; }
    WLK_CHECK(found >= 0, "all %d sessions in use", (int)q->sess.size());
    QSession& s = q->sess[found];
    const size_t bytes = (size_t)q->dims.n_layer * 2 * q->dims.n_head * q->ring * 64 * q->es();
    CUDA_CHECK(cudaMalloc(&s.kv, bytes));
    q->bytes_sessions += bytes;
    s.open = true; s.emitted = 0; s.pending.clear(); s.tail.clear();
    *sid = found;
    WLK_API_END
}
int wlk_qwen_session_close(wlk_qwen* q, int32_t sid) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    QSession& s = qsession(q, sid);
    CUDA_CHECK(cudaStreamSynchronize(q->st));
    cudaFree(s.kv);
    q->bytes_sessions -= (size_t)q->dims.n_layer * 2 * q->dims.n_head * q->ring * 64 * q->es();
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
    QSession& s = qsession(q, sid);
    s.emitted = 0; s.pending.clear(); s.tail.clear();
    s.buf_len = s.buf_start_frame = s.mel_emitted = s.total_samples = 0;       // StreamingMelExtractor.reset, features.py:112
    WLK_API_END
}
int wlk_qwen_session_state(wlk_qwen* q, int32_t sid, int32_t* pending_frames, int64_t* emitted_steps) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    QSession& s = qsession(q, sid);
    if (pending_frames) *pending_frames = (int32_t)(s.pending.size() / q->dims.n_mels);
    if (emitted_steps) *emitted_steps = s.emitted;
    WLK_API_END
}
int wlk_qwen_session_mutable_steps(wlk_qwen* q, int32_t sid, int32_t* mutable_steps) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    QSession& s = qsession(q, sid);
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
    QSession& s = qsession(q, sid);
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
    QSession& s = qsession(q, sid);
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
int wlk_qwen_memory(wlk_qwen* q, size_t* weights, size_t* sessions, size_t* workspace) {
    WLK_API_BEGIN
    WLK_ENTER(q, q->cfg.device);
    if (weights) *weights = q->bytes_weights;
    if (sessions) *sessions = q->bytes_sessions;
    if (workspace) *workspace = q->bytes_workspace;
    WLK_API_END
}

}  // extern "C"
