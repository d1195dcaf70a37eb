// Silero VAD forward on the device, batched over streams -- the ingest step before the path (SURVEY.md section 8f
// item 3).  Reference: the vendored TorchScript model whisperlivekit/silero_vad_models/silero_vad.jit, run one
// 512-sample window at a time per stream by VADIterator / FixedVADIterator (whisperlivekit/silero_vad_iterator.py:
// 20-29 init_jit_model, :288-331 FixedVADIterator); arithmetic restated in oracle/vad_oracle.py (16 kHz branch):
//   x = [64 context samples | 512 new], reflect-pad 64 on the right, conv1d with the [258,1,256] basis at hop 128
//   -> 4 frames, magnitude over the first / second 129 channels, four Conv1d(k=3,pad=1)+ReLU (129->128 s1, 128->64 s2,
//   64->64 s2, 64->128 s1), LSTMCell(128,128) on the stream's (h, c), ReLU -> Conv1d(128,1,k=1) -> sigmoid.
// One CTA per stream walks that stream's windows in order (the recurrence is per stream); the ~1.2 MB of weights are
// stored transposed so that consecutive threads read consecutive addresses, and are served from L2 to every CTA.
#include <mutex>
#include <set>
#include <vector>

#include "../../include/wlk_b200.h"
#include "common.cuh"
#include "host.cuh"

namespace wlk {
namespace {

constexpr int VW = 512, VCTX = 64, VX = VCTX + VW, VPAD = VX + 64;    // 576 samples in, 640 after the reflect pad
constexpr int NB = 129;                                                // frequency bins
constexpr int VSTATE = VCTX + 128 + 128;                               // context | h | c

struct VadWeights {
    float* basisT;       // [256][258]
    float *w0T, *b0;     // [129*3][128], [128]
    float *w1T, *b1;     // [128*3][64]
    float *w2T, *b2;     // [64*3][64]
    float *w3T, *b3;     // [64*3][128]
    float *wihT, *whhT;  // [128][512]
    float *bih, *bhh;    // [512]
    float *wdec, *bdec;  // [128], [1]
};
struct VadJob { float* state; const float* pcm; float* probs; int32_t n_windows; int32_t pad; };

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

__global__ void __launch_bounds__(256)
vad_forward_kernel(const VadJob* __restrict__ jobs, VadWeights W) {
    __shared__ float x[VPAD];
    __shared__ float ft[258][4];
    __shared__ float a0[NB][4];          // magnitude
    __shared__ float a1[128][4];
    __shared__ float a2[64][2];
    __shared__ float a3[64];
    __shared__ float a4[128];
    __shared__ float hs[128], cs[128], gates[512];
    __shared__ float red[8];
    const VadJob job = jobs[blockIdx.x];
    const int tid = threadIdx.x;
    if (tid < VCTX) x[tid] = job.state[tid];
    if (tid < 128) { hs[tid] = job.state[VCTX + tid]; cs[tid] = job.state[VCTX + 128 + tid]; }
    __syncthreads();
    for (int w = 0; w < job.n_windows; ++w) {
        for (int i = tid; i < VW; i += 256) x[VCTX + i] = job.pcm[(int64_t)w * VW + i];
        __syncthreads();
        if (tid < 64) x[VX + tid] = x[VX - 2 - tid];                       // F.pad(..., (0, 64), mode="reflect")
        __syncthreads();
        // ---- STFT as a strided conv: ft[c][t] = sum_j basis[c][j] x[128 t + j]
        for (int c = tid; c < 258; c += 256) {
            float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
            for (int j = 0; j < 256; ++j) {
                const float b = W.basisT[j * 258 + c];
                s0 = fmaf(b, x[j], s0); s1 = fmaf(b, x[128 + j], s1); s2 = fmaf(b, x[256 + j], s2); s3 = fmaf(b, x[384 + j], s3);
            }
            ft[c][0] = s0; ft[c][1] = s1; ft[c][2] = s2; ft[c][3] = s3;
        }
        __syncthreads();
        for (int i = tid; i < NB * 4; i += 256) {
            const int k = i >> 2, t = i & 3;
            const float re = ft[k][t], im = ft[NB + k][t];
            a0[k][t] = sqrtf(re * re + im * im);
        }
        __syncthreads();
        // ---- encoder.0: 129 -> 128, stride 1, 4 -> 4 frames.  thread = (co, frame pair)
        {
            const int co = tid & 127, t0 = (tid >> 7) * 2;
            float s0 = W.b0[co], s1 = s0;
            for (int ci = 0; ci < NB; ++ci) {
                const float w0 = W.w0T[(ci * 3 + 0) * 128 + co], w1 = W.w0T[(ci * 3 + 1) * 128 + co], w2 = W.w0T[(ci * 3 + 2) * 128 + co];
                const float xm = t0 > 0 ? a0[ci][t0 - 1] : 0.f, x0 = a0[ci][t0], x1 = a0[ci][t0 + 1], x2 = t0 + 2 < 4 ? a0[ci][t0 + 2] : 0.f;
                s0 = fmaf(w0, xm, fmaf(w1, x0, fmaf(w2, x1, s0)));
                s1 = fmaf(w0, x0, fmaf(w1, x1, fmaf(w2, x2, s1)));
            }
            a1[co][t0] = fmaxf(s0, 0.f); a1[co][t0 + 1] = fmaxf(s1, 0.f);
        }
        __syncthreads();
        // ---- encoder.1: 128 -> 64, stride 2, 4 -> 2 frames (out t reads in 2t-1 .. 2t+1).  thread = (co, t) for tid < 128
        if (tid < 128) {
            const int co = tid & 63, t = tid >> 6;
            float s = W.b1[co];
            for (int ci = 0; ci < 128; ++ci) {
                const float xm = t > 0 ? a1[ci][2 * t - 1] : 0.f;
                s = fmaf(W.w1T[(ci * 3 + 0) * 64 + co], xm, s);
                s = fmaf(W.w1T[(ci * 3 + 1) * 64 + co], a1[ci][2 * t], s);
                s = fmaf(W.w1T[(ci * 3 + 2) * 64 + co], a1[ci][2 * t + 1], s);
            }
            a2[co][t] = fmaxf(s, 0.f);
        }
        __syncthreads();
        // ---- encoder.2: 64 -> 64, stride 2, 2 -> 1 frame (reads in -1 (pad), 0, 1)
        if (tid < 64) {
            float s = W.b2[tid];
            for (int ci = 0; ci < 64; ++ci) {
                s = fmaf(W.w2T[(ci * 3 + 1) * 64 + tid], a2[ci][0], s);
                s = fmaf(W.w2T[(ci * 3 + 2) * 64 + tid], a2[ci][1], s);
            }
            a3[tid] = fmaxf(s, 0.f);
        }
        __syncthreads();
        // ---- encoder.3: 64 -> 128, stride 1, 1 -> 1 frame (only the centre tap sees data)
        if (tid < 128) {
            float s = W.b3[tid];
            for (int ci = 0; ci < 64; ++ci) s = fmaf(W.w3T[(ci * 3 + 1) * 128 + tid], a3[ci], s);
            a4[tid] = fmaxf(s, 0.f);
        }
        __syncthreads();
        // ---- LSTMCell: gates = W_ih y + b_ih + W_hh h + b_hh   (torch gate order i, f, g, o)
        for (int g = tid; g < 512; g += 256) {
            float s = W.bih[g] + W.bhh[g];
            for (int k = 0; k < 128; ++k) s = fmaf(W.wihT[k * 512 + g], a4[k], fmaf(W.whhT[k * 512 + g], hs[k], s));
            gates[g] = s;
        }
        __syncthreads();
        float part = 0.f;
        if (tid < 128) {
            const float ig = sigmoidf_(gates[tid]), fg = sigmoidf_(gates[128 + tid]), gg = tanhf(gates[256 + tid]), og = sigmoidf_(gates[384 + tid]);
            const float c = fg * cs[tid] + ig * gg;
            const float h = og * tanhf(c);
            cs[tid] = c; hs[tid] = h;
            part = fmaxf(h, 0.f) * W.wdec[tid];
        }
        part = warp_sum(part);
        if ((tid & 31) == 0) red[tid >> 5] = part;
        __syncthreads();
        if (tid == 0) {
            float s = W.bdec[0];
            for (int i = 0; i < 4; ++i) s += red[i];
            job.probs[w] = sigmoidf_(s);
        }
        if (tid < VCTX) x[tid] = x[VW + tid];                              // the window's last 64 samples: next context
        __syncthreads();
    }
    if (tid < VCTX) job.state[tid] = x[tid];
    if (tid < 128) { job.state[VCTX + tid] = hs[tid]; job.state[VCTX + 128 + tid] = cs[tid]; }
}

}  // namespace
}  // namespace wlk

using namespace wlk;

struct wlk_vad {
    int device = 0, max_sessions = 0;
    cudaStream_t st = nullptr;
    std::mutex mu;
    VadWeights w{};
    DeviceAllocs allocs;
    std::set<std::string> loaded;
    float* states = nullptr;                 // [max_sessions][VSTATE]
    std::vector<char> open;
    uint8_t *stg_h = nullptr, *stg_d = nullptr; size_t stg_bytes = 0;
};

namespace {
// host [rows][cols] -> device [cols][rows]
void put_T(wlk_vad* v, float* dst, const float* host, int rows, int cols) {
    std::vector<float> t((size_t)rows * cols);
    for (int r = 0; r < rows; ++r)
        for (int c = 0; c < cols; ++c) t[(size_t)c * rows + r] = host[(size_t)r * cols + c];
    CUDA_CHECK(cudaMemcpy(dst, t.data(), t.size() * 4, cudaMemcpyHostToDevice));
}
void ensure_staging(wlk_vad* v, size_t bytes) {
    if (bytes <= v->stg_bytes) return;
    if (v->stg_h) { CUDA_CHECK(cudaStreamSynchronize(v->st)); cudaFreeHost(v->stg_h); cudaFree(v->stg_d); }
    v->stg_bytes = bytes * 2;
    CUDA_CHECK(cudaMallocHost(&v->stg_h, v->stg_bytes));
    CUDA_CHECK(cudaMalloc(&v->stg_d, v->stg_bytes));
}
const char* kVadTensors[] = {"stft.forward_basis_buffer", "encoder.0.reparam_conv.weight", "encoder.0.reparam_conv.bias",
                             "encoder.1.reparam_conv.weight", "encoder.1.reparam_conv.bias", "encoder.2.reparam_conv.weight",
                             "encoder.2.reparam_conv.bias", "encoder.3.reparam_conv.weight", "encoder.3.reparam_conv.bias",
                             "decoder.rnn.weight_ih", "decoder.rnn.weight_hh", "decoder.rnn.bias_ih", "decoder.rnn.bias_hh",
                             "decoder.decoder.2.weight", "decoder.decoder.2.bias"};
}  // namespace

extern "C" {

int wlk_vad_create(int device, int max_sessions, wlk_vad** out) {
    WLK_API_BEGIN
    WLK_CHECK(out && max_sessions >= 1, "bad arguments");
    use_device(device);
    auto* v = new wlk_vad();
    v->device = device; v->max_sessions = max_sessions;
    CUDA_CHECK(cudaStreamCreateWithFlags(&v->st, cudaStreamNonBlocking));
    VadWeights& W = v->w;
    auto fv = [&](size_t n) { return (float*)v->allocs.take(n * 4, nullptr); };
    W.basisT = fv(256 * 258);
    W.w0T = fv(NB * 3 * 128); W.b0 = fv(128);
    W.w1T = fv(128 * 3 * 64); W.b1 = fv(64);
    W.w2T = fv(64 * 3 * 64); W.b2 = fv(64);
    W.w3T = fv(64 * 3 * 128); W.b3 = fv(128);
    W.wihT = fv(128 * 512); W.whhT = fv(128 * 512);
    W.bih = fv(512); W.bhh = fv(512);
    W.wdec = fv(128); W.bdec = fv(1);
    v->states = fv((size_t)max_sessions * VSTATE);
    v->open.assign(max_sessions, 0);
    *out = v;
    WLK_API_END
}
int wlk_vad_destroy(wlk_vad* v) {
    WLK_API_BEGIN
    WLK_CHECK(v != nullptr, "null engine");
    CUDA_CHECK(cudaSetDevice(v->device));
    cudaStreamSynchronize(v->st);
    v->allocs.free_all();
    if (v->stg_h) { cudaFreeHost(v->stg_h); cudaFree(v->stg_d); }
    cudaStreamDestroy(v->st);
    delete v;
    WLK_API_END
}
int wlk_vad_load_tensor(wlk_vad* v, const char* name, const float* host, int64_t n) {
    WLK_API_BEGIN
    WLK_ENTER(v, v->device);
    WLK_CHECK(name && host, "null argument");
    std::string s(name);
    if (s.rfind("_model.", 0) == 0) s = s.substr(7);
    VadWeights& W = v->w;
    auto expect = [&](int64_t want) { WLK_CHECK(n == want, "tensor %s has %lld elements, expected %lld", name, (long long)n, (long long)want); };
    auto plain = [&](float* dst, int64_t want) { expect(want); CUDA_CHECK(cudaMemcpy(dst, host, want * 4, cudaMemcpyHostToDevice)); };
    if (s == "stft.forward_basis_buffer") { expect(258 * 256); put_T(v, W.basisT, host, 258, 256); }
    else if (s == "encoder.0.reparam_conv.weight") { expect(128 * NB * 3); put_T(v, W.w0T, host, 128, NB * 3); }
    else if (s == "encoder.1.reparam_conv.weight") { expect(64 * 128 * 3); put_T(v, W.w1T, host, 64, 128 * 3); }
    else if (s == "encoder.2.reparam_conv.weight") { expect(64 * 64 * 3); put_T(v, W.w2T, host, 64, 64 * 3); }
    else if (s == "encoder.3.reparam_conv.weight") { expect(128 * 64 * 3); put_T(v, W.w3T, host, 128, 64 * 3); }
    else if (s == "encoder.0.reparam_conv.bias") plain(W.b0, 128);
    else if (s == "encoder.1.reparam_conv.bias") plain(W.b1, 64);
    else if (s == "encoder.2.reparam_conv.bias") plain(W.b2, 64);
    else if (s == "encoder.3.reparam_conv.bias") plain(W.b3, 128);
    else if (s == "decoder.rnn.weight_ih") { expect(512 * 128); put_T(v, W.wihT, host, 512, 128); }
    else if (s == "decoder.rnn.weight_hh") { expect(512 * 128); put_T(v, W.whhT, host, 512, 128); }
    else if (s == "decoder.rnn.bias_ih") plain(W.bih, 512);
    else if (s == "decoder.rnn.bias_hh") plain(W.bhh, 512);
    else if (s == "decoder.decoder.2.weight") plain(W.wdec, 128);
    else if (s == "decoder.decoder.2.bias") plain(W.bdec, 1);
    else WLK_CHECK(false, "unknown VAD tensor %s", name);
    v->loaded.insert(s);
    WLK_API_END
}
int wlk_vad_session_open(wlk_vad* v, int32_t* sid) {
    WLK_API_BEGIN
    WLK_ENTER(v, v->device);
    WLK_CHECK(sid, "null out pointer");
    for (auto t : kVadTensors) WLK_CHECK(v->loaded.count(t), "VAD tensor %s not loaded", t);
    int found = -1;
    for (int i = 0; i < v->max_sessions; ++i) if (!v->open[i]) { found = i; break; }
    WLK_CHECK(found >= 0, "all %d VAD sessions in use", v->max_sessions);
    CUDA_CHECK(cudaMemsetAsync(v->states + (size_t)found * VSTATE, 0, VSTATE * 4, v->st));
    v->open[found] = 1;
    *sid = found;
    WLK_API_END
}
int wlk_vad_session_reset(wlk_vad* v, int32_t sid) {           /* reset_states(): context, h, c <- 0 */
    WLK_API_BEGIN
    WLK_ENTER(v, v->device);
    WLK_CHECK(sid >= 0 && sid < v->max_sessions && v->open[sid], "invalid VAD session %d", sid);
    CUDA_CHECK(cudaMemsetAsync(v->states + (size_t)sid * VSTATE, 0, VSTATE * 4, v->st));
    WLK_API_END
}
int wlk_vad_session_close(wlk_vad* v, int32_t sid) {
    WLK_API_BEGIN
    WLK_ENTER(v, v->device);
    WLK_CHECK(sid >= 0 && sid < v->max_sessions && v->open[sid], "invalid VAD session %d", sid);
    v->open[sid] = 0;
    WLK_API_END
}
int wlk_vad_forward(wlk_vad* v, const int32_t* sids, int n, const float* pcm_host, const int32_t* window_offsets,
                    float* probs_host) {
    WLK_API_BEGIN
    WLK_ENTER(v, v->device);
    WLK_CHECK(sids && pcm_host && window_offsets && probs_host && n >= 1, "bad arguments");
    WLK_CHECK(window_offsets[0] == 0, "window_offsets must start at 0");
    const int total = window_offsets[n];
    for (int i = 0; i < n; ++i) {
        WLK_CHECK(sids[i] >= 0 && sids[i] < v->max_sessions && v->open[sids[i]], "invalid VAD session %d", sids[i]);
        WLK_CHECK(window_offsets[i + 1] >= window_offsets[i], "window_offsets must be non-decreasing");
        for (int j = 0; j < i; ++j) WLK_CHECK(sids[j] != sids[i], "session %d appears twice", sids[i]);
    }
    if (total == 0) return 0;
    const size_t o_pcm = 0, o_prob = (size_t)total * VW * 4, o_jobs = o_prob + (((size_t)total * 4 + 255) / 256) * 256;
    ensure_staging(v, o_jobs + sizeof(VadJob) * n);
    memcpy(v->stg_h + o_pcm, pcm_host, (size_t)total * VW * 4);
    VadJob* jobs = reinterpret_cast<VadJob*>(v->stg_h + o_jobs);
    for (int i = 0; i < n; ++i)
        jobs[i] = VadJob{v->states + (size_t)sids[i] * VSTATE, reinterpret_cast<const float*>(v->stg_d + o_pcm) + (size_t)window_offsets[i] * VW,
                         reinterpret_cast<float*>(v->stg_d + o_prob) + window_offsets[i], window_offsets[i + 1] - window_offsets[i], 0};
    CUDA_CHECK(cudaMemcpyAsync(v->stg_d, v->stg_h, o_jobs + sizeof(VadJob) * n, cudaMemcpyHostToDevice, v->st));
    vad_forward_kernel<<<n, 256, 0, v->st>>>(reinterpret_cast<const VadJob*>(v->stg_d + o_jobs), v->w);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(v->stg_h + o_prob, v->stg_d + o_prob, (size_t)total * 4, cudaMemcpyDeviceToHost, v->st));
    CUDA_CHECK(cudaStreamSynchronize(v->st));
    memcpy(probs_host, v->stg_h + o_prob, (size_t)total * 4);
    WLK_API_END
}

}  // extern "C"
