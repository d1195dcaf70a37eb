// Non-GEMM kernels of the streaming-Whisper hot path (sm_90a).  Everything here is
// bandwidth- or latency-bound SIMT code; the tensor-core kernels live in gemm_tc.cu / attn_tc.cu.
#include "attn_warp.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

namespace wlk {

// =====================================================================================
// block reductions
// =====================================================================================
template <int NT>
__device__ __forceinline__ float block_max(float v, float* red) {
    v = warp_max(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = (threadIdx.x < NT / 32) ? red[threadIdx.x] : -INFINITY;
    r = warp_max(r);
    __syncthreads();
    return r;            // valid in every thread of warp 0 .. broadcast below
}
template <int NT>
__device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = (threadIdx.x < NT / 32) ? red[threadIdx.x] : 0.f;
    r = warp_sum(r);
    __syncthreads();
    return r;
}
// all-thread broadcast versions
template <int NT>
__device__ __forceinline__ float block_max_all(float v, float* red) {
    float r = block_max<NT>(v, red);
    if (threadIdx.x == 0) red[0] = r;
    __syncthreads();
    r = red[0];
    __syncthreads();
    return r;
}
template <int NT>
__device__ __forceinline__ float block_sum_all(float v, float* red) {
    float r = block_sum<NT>(v, red);
    if (threadIdx.x == 0) red[0] = r;
    __syncthreads();
    r = red[0];
    __syncthreads();
    return r;
}

// =====================================================================================
// log-mel front end  (reference whisperlivekit/whisper/audio.py:110-157)
//   pass 1: per 8-frame CTA: reflect-padded framing, Hann window, 400-point real DFT (201 bins),
//           power, mel projection, log10(clamp 1e-10) -> raw[f][m], per-CTA max
//   pass 2: global max over the CTA maxima, max(x, gmax-8), (x+4)/4, convert, time-major store
//           with a zero row either side (the conv stem's padding) and the silence constant for
//           frames that see only the 30 s of zero padding.
// =====================================================================================
// Real-input DFT with the window's symmetry folded in: with s[j] = xw[j] + xw[400-j], d[j] = xw[j] - xw[400-j]
//   Re X[k] = xw[0] + (-1)^k xw[200] + sum_{j=1}^{199} s[j] cos(2 pi k j / 400)
//   Im X[k] =                        - sum_{j=1}^{199} d[j] sin(2 pi k j / 400)
// A thread owns one frequency bin and all MEL_FRAMES_PER_CTA frames of the CTA: per j it fetches one
// twiddle and the frames' (s, d) pairs as shared-memory broadcasts (every lane of a warp reads the same
// address), i.e. ~3 issued instructions per complex MAC pair instead of ~14 in the naive form.  The mel
// projection walks only each filter's non-zero span [lo, hi) (triangular filters: ~400 non-zeros in total).
__global__ void __launch_bounds__(224)
mel_power_kernel(const MelJob* __restrict__ jobs, int n_mels, const float* __restrict__ filtT /*[201][n_mels]*/,
                 const float* __restrict__ window, const float2* __restrict__ twiddle,
                 const int2* __restrict__ filt_span /*[n_mels] (lo, hi)*/) {
    constexpr int FR = MEL_FRAMES_PER_CTA;
    constexpr int HALF = N_FFT / 2;                  // 200
    __shared__ float2 sd[FR][HALF];                  // (s[j], d[j]); entry 0 holds (xw[0], xw[200])
    __shared__ float2 tw[N_FFT];
    __shared__ __align__(16) float pw[FR][N_FREQ + 3];   // first the TMA-staged samples of the CTA's frames, then the power spectra
    __shared__ float red[8];
    __shared__ __align__(8) uint64_t stage_bar;
    const MelJob job = jobs[blockIdx.y];
    const int f0 = blockIdx.x * FR;
    const int tid = threadIdx.x;
    const int n_valid = min(job.n_compute, job.n_total);
    if (f0 >= n_valid) {
        if (tid == 0) job.blockmax[blockIdx.x] = -10.0f;
        return;
    }
    if (f0 >= job.keep_lo && f0 + FR <= job.keep_hi) return;       // incremental: these rows of `raw` are still this window's
    // The samples the CTA's 16 frames touch are one contiguous run of (FR - 1) * HOP + N_FFT = 2800 floats.  Away from the
    // edges of the audio it is staged into shared memory by one bulk copy of the TMA engine (cp.async.bulk, completion
    // on an mbarrier) instead of 2800 strided per-thread loads; edge CTAs (reflection, zero padding) gather per sample.
    constexpr int SPAN = (FR - 1) * HOP + N_FFT;
    static_assert(SPAN <= FR * (N_FREQ + 3) && (SPAN * 4) % 16 == 0, "sample staging aliases pw");
    const int s_begin = f0 * HOP - HALF;
    const bool staged = s_begin >= 0 && s_begin + SPAN <= job.n && ((reinterpret_cast<uintptr_t>(job.audio + s_begin) & 15) == 0);
    float* stage = &pw[0][0];
    if (staged) {
        const uint32_t bar = ptx::smem_u32(&stage_bar);
        if (tid == 0) {
            ptx::mbar_init(bar, 1);
            ptx::fence_barrier_init();
            ptx::mbar_arrive_expect_tx(bar, SPAN * 4);
            ptx::tma_load_1d(ptx::smem_u32(stage), job.audio + s_begin, SPAN * 4, bar);
        }
        __syncthreads();
        ptx::mbar_wait(bar, 0);
    }
    for (int i = tid; i < N_FFT; i += 224) tw[i] = twiddle[i];
    // __fmul_rn: the product is rounded on its own in both branches (never contracted into the sums below), so a frame has
    // the same bits whether its CTA staged or gathered -- the incremental front end keeps rows across that difference
    auto sample = [&](int fr, int j) -> float {         // windowed sample j of frame fr
        if (staged) return __fmul_rn(stage[fr * HOP + j], window[j]);
        int s = (f0 + fr) * HOP - HALF + j;             // torch.stft(center=True): reflect pad n_fft/2
        if (s < 0) s = -s;
        if (job.pad && s >= job.n) s = 2 * (job.n - 1) - s;  // streaming window: reflect at the right edge too
        const float x = (s >= 0 && s < job.n) ? job.audio[s] : 0.f;   // right of the audio: the appended zeros
        return __fmul_rn(x, window[j]);
    };
    for (int i = tid; i < FR * HALF; i += 224) {
        const int fr = i / HALF, j = i - fr * HALF;
        if (j == 0) sd[fr][0] = make_float2(sample(fr, 0), sample(fr, HALF));
        else {
            const float a = sample(fr, j), b = sample(fr, N_FFT - j);
            sd[fr][j] = make_float2(a + b, a - b);
        }
    }
    __syncthreads();
    if (tid < N_FREQ) {
        const int k = tid;
        float re[FR], im[FR];
        const float sgn = (k & 1) ? -1.f : 1.f;
#pragma unroll
        for (int f = 0; f < FR; ++f) { re[f] = sd[f][0].x + sgn * sd[f][0].y; im[f] = 0.f; }
        int t = 0;
#pragma unroll 2
        for (int j = 1; j < HALF; ++j) {
            t += k;
            if (t >= N_FFT) t -= N_FFT;
            const float2 c = tw[t];
#pragma unroll
            for (int f = 0; f < FR; ++f) {
                const float2 v = sd[f][j];
                re[f] = fmaf(v.x, c.x, re[f]);
                im[f] = fmaf(v.y, c.y, im[f]);
            }
        }
#pragma unroll
        for (int f = 0; f < FR; ++f) pw[f][k] = re[f] * re[f] + im[f] * im[f];
    }
    __syncthreads();
    float lmax = -INFINITY;
    for (int idx = tid; idx < FR * n_mels; idx += 224) {
        const int fr = idx / n_mels, m = idx - fr * n_mels;
        const int f = f0 + fr;
        if (f >= n_valid) continue;
        const int2 sp = filt_span[m];
        float acc = 0.f;
        for (int k = sp.x; k < sp.y; ++k) acc = fmaf(filtT[k * n_mels + m], pw[fr][k], acc);
        const float v = log10f(fmaxf(acc, 1e-10f));
        if (f < MEL_STORE_FRAMES) job.raw[(int64_t)f * n_mels + m] = v;
        lmax = fmaxf(lmax, v);
    }
    // block max over 7 warps
    lmax = warp_max(lmax);
    if ((tid & 31) == 0) red[tid >> 5] = lmax;
    __syncthreads();
    if (tid == 0) {
        float bm = red[0];
        for (int w = 1; w < 7; ++w) bm = fmaxf(bm, red[w]);
        job.blockmax[blockIdx.x] = bm;
    }
}

template <typename TO>
__global__ void __launch_bounds__(256)
mel_finalize_kernel(const MelJob* __restrict__ jobs, int n_mels) {
    __shared__ float red[8];
    const MelJob job = jobs[blockIdx.y];
    float m = -10.0f;    // frames inside the zero padding contribute log10(1e-10)
    const int n_valid = min(job.n_compute, job.n_total);
    const int n_ctas = (n_valid + MEL_FRAMES_PER_CTA - 1) / MEL_FRAMES_PER_CTA;
    // stored rows: the partial maxima of mel_max_kernel (they cover kept and recomputed rows alike); frames past the
    // stored rows (audio longer than 30 s: always a full pass) only exist as the per-CTA maxima of this pass
    if (threadIdx.x < MEL_MAX_PARTS) m = fmaxf(m, job.blockmax[MEL_MAX_CTAS + threadIdx.x]);
    for (int i = MEL_STORE_FRAMES / MEL_FRAMES_PER_CTA + threadIdx.x; i < n_ctas; i += 256) m = fmaxf(m, job.blockmax[i]);
    const float gmax = block_max_all<256>(m, red);
    const float thr = gmax - 8.0f;
    TO* out = reinterpret_cast<TO*>(job.out);
    const int64_t total = (int64_t)MEL_ROWS * n_mels;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        int r = (int)(i / n_mels);
        float v = 0.f;
        if (r >= 1 && r <= N_FRAMES) {
            int f = r - 1;
            float raw = (f < n_valid) ? job.raw[(int64_t)f * n_mels + (i - (int64_t)r * n_mels)] : -10.0f;
            v = (fmaxf(raw, thr) + 4.0f) * 0.25f;
        }
        out[i] = from_f32<TO>(v);
    }
}

// partial maxima over the stored raw rows of every job: blockmax[MEL_MAX_CTAS + p], p < MEL_MAX_PARTS
__global__ void __launch_bounds__(256)
mel_max_kernel(const MelJob* __restrict__ jobs, int n_mels) {
    __shared__ float red[8];
    const MelJob job = jobs[blockIdx.y];
    const int n_rows = min(min(job.n_compute, job.n_total), MEL_STORE_FRAMES);
    const int64_t total4 = (int64_t)n_rows * n_mels / 4;                  // n_mels % 8 == 0
    const float4* r4 = reinterpret_cast<const float4*>(job.raw);
    float m = -INFINITY;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total4; i += (int64_t)MEL_MAX_PARTS * 256) {
        const float4 v = r4[i];
        m = fmaxf(m, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
    }
    m = block_max<256>(m, red);
    if (threadIdx.x == 0) job.blockmax[MEL_MAX_CTAS + blockIdx.x] = m;
}

void mel_forward(const MelJob* jobs_dev, int batch, int n_mels, const float* filtT, const float* window,
                 const float2* twiddle, const int2* filt_span, int out_type, int max_frames, cudaStream_t st) {
    int ctas = (max_frames + MEL_FRAMES_PER_CTA - 1) / MEL_FRAMES_PER_CTA;
    if (ctas < 1) ctas = 1;
    if (ctas > MEL_MAX_CTAS) ctas = MEL_MAX_CTAS;
    dim3 g1(ctas, batch);
    mel_power_kernel<<<g1, 224, 0, st>>>(jobs_dev, n_mels, filtT, window, twiddle, filt_span);
    CUDA_CHECK(cudaGetLastError());
    mel_max_kernel<<<dim3(MEL_MAX_PARTS, batch), 256, 0, st>>>(jobs_dev, n_mels);
    CUDA_CHECK(cudaGetLastError());
    dim3 g2(64, batch);
    if (out_type == DT_F32) mel_finalize_kernel<float><<<g2, 256, 0, st>>>(jobs_dev, n_mels);
    else mel_finalize_kernel<bf16><<<g2, 256, 0, st>>>(jobs_dev, n_mels);
    CUDA_CHECK(cudaGetLastError());
}

// Incremental front end of the Qwen3 streaming backend (reference third_party/qwen3-asr-causal/src/qwen3_asr_causal/
// features.py:50-84): features of one sample WINDOW -- reflect padding at both edges (MelJob.pad = 1), clamp against
// the window's own maximum -- of which frames [first, last) are emitted as fp32 [frames][n_mels].
__global__ void __launch_bounds__(256)
mel_window_finalize_kernel(const MelJob* __restrict__ jobs, const int2* __restrict__ ranges /* (first, last) */,
                           const int64_t* __restrict__ out_off, float* __restrict__ out, int n_mels) {
    __shared__ float red[8];
    const MelJob job = jobs[blockIdx.y];
    float m = -INFINITY;
    const int n_ctas = (job.n_compute + MEL_FRAMES_PER_CTA - 1) / MEL_FRAMES_PER_CTA;
    for (int i = threadIdx.x; i < n_ctas; i += 256) m = fmaxf(m, job.blockmax[i]);
    const float thr = block_max_all<256>(m, red) - 8.0f;
    const int2 r = ranges[blockIdx.y];
    const int64_t total = (int64_t)(r.y - r.x) * n_mels;
    float* o = out + out_off[blockIdx.y] * n_mels;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256)
        o[i] = (fmaxf(job.raw[(int64_t)r.x * n_mels + i], thr) + 4.0f) * 0.25f;
}
void mel_window_forward(const MelJob* jobs_dev, const int2* ranges_dev, const int64_t* out_off_dev, float* out_dev, int batch,
                        int n_mels, const float* filtT, const float* window, const float2* twiddle, const int2* filt_span,
                        int max_frames, cudaStream_t st) {
    int ctas = (max_frames + MEL_FRAMES_PER_CTA - 1) / MEL_FRAMES_PER_CTA;
    if (ctas < 1) ctas = 1;
    if (ctas > MEL_MAX_CTAS) ctas = MEL_MAX_CTAS;
    dim3 g1(ctas, batch);
    mel_power_kernel<<<g1, 224, 0, st>>>(jobs_dev, n_mels, filtT, window, twiddle, filt_span);
    CUDA_CHECK(cudaGetLastError());
    dim3 g2(8, batch);
    mel_window_finalize_kernel<<<g2, 256, 0, st>>>(jobs_dev, ranges_dev, out_off_dev, out_dev, n_mels);
    CUDA_CHECK(cudaGetLastError());
}

// mel computed by the caller (LocalAgreement: whisper.transcribe() builds it on the host) -> the engine's
// time-major layout with the conv padding rows: out[(f + 1) * n_mels + m] = mel[m * 3000 + f]
template <typename TO>
__global__ void mel_import_kernel(const float* __restrict__ mel, TO* __restrict__ out, int n_mels) {
    const int64_t total = (int64_t)MEL_ROWS * n_mels;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / n_mels), m = (int)(i - (int64_t)r * n_mels);
        const float v = (r >= 1 && r <= N_FRAMES) ? mel[(int64_t)m * N_FRAMES + (r - 1)] : 0.f;
        out[i] = from_f32<TO>(v);
    }
}
void mel_import(const float* mel_dev, void* out, int out_type, int n_mels, cudaStream_t st) {
    if (out_type == DT_F32) mel_import_kernel<float><<<256, 256, 0, st>>>(mel_dev, (float*)out, n_mels);
    else mel_import_kernel<bf16><<<256, 256, 0, st>>>(mel_dev, (bf16*)out, n_mels);
    CUDA_CHECK(cudaGetLastError());
}

// =====================================================================================
// small utilities
// =====================================================================================
template <typename T>
__global__ void zero_rows_kernel(T* base, int64_t row_elems, const int64_t* rows, int n_rows) {
    int r = blockIdx.x;
    if (r >= n_rows) return;
    T* p = base + rows[r] * row_elems;
    for (int64_t i = threadIdx.x; i < row_elems; i += blockDim.x) p[i] = from_f32<T>(0.f);
}
void zero_rows(void* base, int type, int64_t row_elems, const int64_t* rows, int n_rows, cudaStream_t st) {
    if (n_rows <= 0) return;
    if (type == DT_F32) zero_rows_kernel<float><<<n_rows, 256, 0, st>>>((float*)base, row_elems, rows, n_rows);
    else zero_rows_kernel<bf16><<<n_rows, 256, 0, st>>>((bf16*)base, row_elems, rows, n_rows);
    CUDA_CHECK(cudaGetLastError());
}

template <typename T>
__global__ void cvt_from_f32_kernel(const float* s, T* d, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        d[i] = from_f32<T>(s[i]);
}
template <typename T>
__global__ void cvt_to_f32_kernel(const T* s, float* d, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        d[i] = to_f32(s[i]);
}
void convert_f32_to(const float* src, void* dst, int dst_type, int64_t n, cudaStream_t st) {
    int grid = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
    if (grid < 1) grid = 1;
    if (dst_type == DT_F32) cvt_from_f32_kernel<float><<<grid, 256, 0, st>>>(src, (float*)dst, n);
    else cvt_from_f32_kernel<bf16><<<grid, 256, 0, st>>>(src, (bf16*)dst, n);
    CUDA_CHECK(cudaGetLastError());
}
// s16le PCM -> fp32 in [-1, 1): reference audio_processor.py:416-418 (np.int16 / 32768.0), exact in fp32
__global__ void pcm16_to_f32_kernel(const int16_t* __restrict__ s, float* __restrict__ d, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        d[i] = (float)s[i] * (1.0f / 32768.0f);
}
void pcm16_to_f32(const int16_t* src, float* dst, int64_t n, cudaStream_t st) {
    if (n <= 0) return;
    int grid = (int)((n + 255) / 256 < 1184 ? (n + 255) / 256 : 1184);
    pcm16_to_f32_kernel<<<grid, 256, 0, st>>>(src, dst, n);
    CUDA_CHECK(cudaGetLastError());
}

void convert_to_f32(const void* src, int src_type, float* dst, int64_t n, cudaStream_t st) {
    int grid = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
    if (grid < 1) grid = 1;
    if (src_type == DT_F32) cvt_to_f32_kernel<float><<<grid, 256, 0, st>>>((const float*)src, dst, n);
    else cvt_to_f32_kernel<bf16><<<grid, 256, 0, st>>>((const bf16*)src, dst, n);
    CUDA_CHECK(cudaGetLastError());
}

__global__ void split_planes_kernel(const float* __restrict__ s, bf16* __restrict__ hi, bf16* __restrict__ lo, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float x = s[i];
        const bf16 h = __float2bfloat16_rn(x);
        hi[i] = h;
        lo[i] = __float2bfloat16_rn(x - __bfloat162float(h));
    }
}
void split_f32_to_planes(const float* src, bf16* hi, bf16* lo, int64_t n, cudaStream_t st) {
    int grid = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
    if (grid < 1) grid = 1;
    split_planes_kernel<<<grid, 256, 0, st>>>(src, hi, lo, n);
    CUDA_CHECK(cudaGetLastError());
}

// =====================================================================================
// LayerNorm (fp32 statistics, reference whisper/model.py:39-41), one warp per row
// =====================================================================================
// The row (d <= 1280 floats) is read once with 128-bit loads and kept in registers for the two statistics
// passes and the normalisation; bf16 output is written 8 bytes at a time.
template <typename TO>
__device__ __forceinline__ void ln_store4(TO* o, float a, float b, float c, float d);
template <> __device__ __forceinline__ void ln_store4<float>(float* o, float a, float b, float c, float d) {
    *reinterpret_cast<float4*>(o) = make_float4(a, b, c, d);
}
template <> __device__ __forceinline__ void ln_store4<bf16>(bf16* o, float a, float b, float c, float d) {
    __nv_bfloat162 h0 = __floats2bfloat162_rn(a, b), h1 = __floats2bfloat162_rn(c, d);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&h0);
    u.y = *reinterpret_cast<uint32_t*>(&h1);
    *reinterpret_cast<uint2*>(o) = u;
}

template <typename TO>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ w, const float* __restrict__ b,
                 TO* __restrict__ out, int64_t ldo, int rows, int d, const int32_t* __restrict__ row_index) {
    ptx::griddep_launch();                   // programmatic dependent launch: see launch_pdl (common.cuh)
    ptx::griddep_wait();
    constexpr int MAXV = 10;                          // float4 per lane: d <= 1280
    const int warp = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const float4* xr = reinterpret_cast<const float4*>(x + (int64_t)(row_index ? row_index[warp] : warp) * ldx);
    const int nvec = d >> 2;
    float4 v[MAXV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int idx = lane + 32 * i;
        if (idx < nvec) { v[i] = xr[idx]; s += (v[i].x + v[i].y) + (v[i].z + v[i].w); }
        else v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const float mean = warp_sum(s) / d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        if (lane + 32 * i < nvec) {
            float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, dd = v[i].w - mean;
            q += (a * a + bb * bb) + (c * c + dd * dd);
        }
    }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / d + 1e-5f);
    const float4* w4 = reinterpret_cast<const float4*>(w);
    const float4* b4 = reinterpret_cast<const float4*>(b);
    TO* o = out + (int64_t)warp * ldo;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int idx = lane + 32 * i;
        if (idx < nvec) {
            const float4 ww = w4[idx], bb = b4[idx];
            ln_store4<TO>(o + 4 * idx, (v[i].x - mean) * rstd * ww.x + bb.x, (v[i].y - mean) * rstd * ww.y + bb.y,
                          (v[i].z - mean) * rstd * ww.z + bb.z, (v[i].w - mean) * rstd * ww.w + bb.w);
        }
    }
}
void layernorm(const float* x, int64_t ldx, const float* w, const float* b, void* out, int out_type, int64_t ldo,
               int rows, int d, const int32_t* row_index, cudaStream_t st) {
    if (rows <= 0) return;
    WLK_CHECK(d % 4 == 0 && d <= 1280 && ldx % 4 == 0 && ldo % 4 == 0, "layernorm: d=%d must be a multiple of 4 and <= 1280", d);
    int grid = (rows + 7) / 8;
    if (out_type == DT_F32) CUDA_CHECK(launch_pdl(layernorm_kernel<float>, dim3(grid), dim3(256), 0, st, x, ldx, w, b, (float*)out, ldo, rows, d, row_index));
    else CUDA_CHECK(launch_pdl(layernorm_kernel<bf16>, dim3(grid), dim3(256), 0, st, x, ldx, w, b, (bf16*)out, ldo, rows, d, row_index));
}

// =====================================================================================
// FP8 (WLK_PREC_FP8): per-row e4m3 quantization, one warp per row
// =====================================================================================
__device__ __forceinline__ float e4m3_to_f32(uint8_t b) {
    uint32_t h;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"((uint16_t)b));
    return __half2float(__ushort_as_half((uint16_t)(h & 0xffff)));
}

// scale = amax / 448 (0 for an all-zero row, whose bytes are then 0); byte = e4m3(x / scale), nearest even, saturated.
// x / scale is the correctly rounded fp32 quotient, so the bytes are those of (x / scale).clamp(+-448).to(e4m3fn).
template <typename TI>
__global__ void __launch_bounds__(256)
quantize_rows_kernel(const TI* __restrict__ src, int64_t lds, int rows, int cols, uint8_t* __restrict__ dst, int64_t ldd,
                     float* __restrict__ scale) {
    ptx::griddep_launch();
    ptx::griddep_wait();
    const int warp = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const TI* s = src + (int64_t)warp * lds;
    float amax = 0.f;
    for (int k = lane; k < cols; k += 32) amax = fmaxf(amax, fabsf(to_f32(s[k])));
    amax = warp_max(amax);
    const float sc = amax / E4M3_MAX;
    uint8_t* d = dst + (int64_t)warp * ldd;
    for (int k = lane; k < cols; k += 32)
        d[k] = sc > 0.f ? (uint8_t)(ptx::pack_e4m3x2(__fdiv_rn(to_f32(s[k]), sc), 0.f) & 0xff) : 0;
    if (lane == 0) scale[warp] = sc;
}
void quantize_rows(const void* src, int src_type, int64_t lds, int rows, int cols, uint8_t* dst, int64_t ldd, float* scale,
                   cudaStream_t st) {
    if (rows <= 0) return;
    WLK_CHECK(cols >= 1 && (src_type == DT_F32 || src_type == DT_BF16), "quantize_rows: fp32 or bf16 rows of >= 1 column");
    const int grid = (rows + 7) / 8;
    if (src_type == DT_F32)
        CUDA_CHECK(launch_pdl(quantize_rows_kernel<float>, dim3(grid), dim3(256), 0, st, (const float*)src, lds, rows, cols, dst, ldd, scale));
    else
        CUDA_CHECK(launch_pdl(quantize_rows_kernel<bf16>, dim3(grid), dim3(256), 0, st, (const bf16*)src, lds, rows, cols, dst, ldd, scale));
}

// LayerNorm with e4m3 output: y as layernorm_kernel computes it, s_a = max|y| / 448, bytes e4m3(y / s_a).  With `bound`
// = {max_n ||W1_n||, max_n |b1_n|} (the dequantized FC1 weight rows) also the FC1 output scale of the row,
// s_h = (||y^|| bound[0] + bound[1]) / 448 with y^ the dequantized row: by Cauchy-Schwarz no |h| and hence no GELU(h)
// exceeds 448 s_h (up to the accumulation's rounding, which the saturating convert absorbs).
__global__ void __launch_bounds__(256)
layernorm_fp8_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ w, const float* __restrict__ b,
                     uint8_t* __restrict__ out, int64_t ldo, float* __restrict__ s_a, float* __restrict__ s_h,
                     const float* __restrict__ bound, int rows, int d) {
    ptx::griddep_launch();
    ptx::griddep_wait();
    constexpr int MAXV = 10;                          // float4 per lane: d <= 1280
    const int warp = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const float4* xr = reinterpret_cast<const float4*>(x + (int64_t)warp * ldx);
    const int nvec = d >> 2;
    float4 v[MAXV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int idx = lane + 32 * i;
        if (idx < nvec) { v[i] = xr[idx]; s += (v[i].x + v[i].y) + (v[i].z + v[i].w); }
        else v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const float mean = warp_sum(s) / d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        if (lane + 32 * i < nvec) {
            float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, dd = v[i].w - mean;
            q += (a * a + bb * bb) + (c * c + dd * dd);
        }
    }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / d + 1e-5f);
    const float4* w4 = reinterpret_cast<const float4*>(w);
    const float4* b4 = reinterpret_cast<const float4*>(b);
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int idx = lane + 32 * i;
        if (idx < nvec) {
            const float4 ww = w4[idx], bb = b4[idx];
            v[i] = make_float4((v[i].x - mean) * rstd * ww.x + bb.x, (v[i].y - mean) * rstd * ww.y + bb.y,
                               (v[i].z - mean) * rstd * ww.z + bb.z, (v[i].w - mean) * rstd * ww.w + bb.w);
            amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v[i].x), fabsf(v[i].y)), fmaxf(fabsf(v[i].z), fabsf(v[i].w))));
        }
    }
    amax = warp_max(amax);
    const float sa = amax / E4M3_MAX;
    uint8_t* o = out + (int64_t)warp * ldo;
    float sq = 0.f;                                   // sum of the squared e4m3 values: ||y^|| = s_a sqrt(sq)
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int idx = lane + 32 * i;
        if (idx < nvec) {
            uint32_t u = 0;
            if (sa > 0.f) {
                const uint16_t lo = ptx::pack_e4m3x2(__fdiv_rn(v[i].x, sa), __fdiv_rn(v[i].y, sa));
                const uint16_t hi = ptx::pack_e4m3x2(__fdiv_rn(v[i].z, sa), __fdiv_rn(v[i].w, sa));
                u = (uint32_t)lo | ((uint32_t)hi << 16);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) { const float f = e4m3_to_f32((uint8_t)(u >> (8 * j))); sq += f * f; }
            *reinterpret_cast<uint32_t*>(o + 4 * idx) = u;
        }
    }
    sq = warp_sum(sq);
    if (lane == 0) {
        s_a[warp] = sa;
        if (s_h) s_h[warp] = (sa * sqrtf(sq) * bound[0] + bound[1]) / E4M3_MAX;
    }
}
void layernorm_fp8(const float* x, int64_t ldx, const float* w, const float* b, uint8_t* out, int64_t ldo, float* s_a,
                   float* s_h, const float* bound, int rows, int d, cudaStream_t st) {
    if (rows <= 0) return;
    WLK_CHECK(d % 4 == 0 && d <= 1280 && ldx % 4 == 0 && ldo % 4 == 0, "layernorm_fp8: d=%d must be a multiple of 4 and <= 1280", d);
    WLK_CHECK(!s_h || bound, "layernorm_fp8: the FC1 output scale needs the layer's bound");
    CUDA_CHECK(launch_pdl(layernorm_fp8_kernel, dim3((rows + 7) / 8), dim3(256), 0, st, x, ldx, w, b, out, ldo, s_a, s_h, bound,
                          rows, d));
}

// bound = {max_n s_w[n] ||e4m3 row n||, max_n |bias[n]|} of an e4m3 matrix [N][K] with row scales s_w: one block, a warp
// per row in a fixed order (deterministic)
__global__ void __launch_bounds__(1024)
fp8_fc1_bound_kernel(const uint8_t* __restrict__ wq, const float* __restrict__ s_w, const float* __restrict__ bias, int N, int K,
                     float* __restrict__ bound) {
    __shared__ float red[2][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float nmax = 0.f, bmax = 0.f;
    for (int n = warp; n < N; n += 32) {
        float sq = 0.f;
        for (int k = lane; k < K; k += 32) { const float f = e4m3_to_f32(wq[(int64_t)n * K + k]); sq += f * f; }
        nmax = fmaxf(nmax, s_w[n] * sqrtf(warp_sum(sq)));
        bmax = fmaxf(bmax, fabsf(bias[n]));
    }
    if (lane == 0) { red[0][warp] = nmax; red[1][warp] = bmax; }
    __syncthreads();
    if (warp == 0) {
        nmax = warp_max(red[0][lane]);
        bmax = warp_max(red[1][lane]);
        if (lane == 0) { bound[0] = nmax; bound[1] = bmax; }
    }
}
void fp8_fc1_bound(const uint8_t* wq, const float* s_w, const float* bias, int N, int K, float* bound, cudaStream_t st) {
    fp8_fc1_bound_kernel<<<1, 1024, 0, st>>>(wq, s_w, bias, N, K, bound);
    CUDA_CHECK(cudaGetLastError());
}

__global__ void embed_kernel(const int32_t* __restrict__ tok, const int32_t* __restrict__ pos,
                             const float* __restrict__ emb, const float* __restrict__ pos_emb, float* __restrict__ x,
                             int rows, int d) {
    ptx::griddep_launch();                   // programmatic dependent launch: see launch_pdl (common.cuh)
    ptx::griddep_wait();
    int r = blockIdx.x;
    if (r >= rows) return;
    const float* e = emb + (int64_t)tok[r] * d;
    const float* p = pos_emb + (int64_t)pos[r] * d;
    for (int i = threadIdx.x; i < d; i += blockDim.x) x[(int64_t)r * d + i] = e[i] + p[i];
}
void embed_tokens(const int32_t* tokens_dev, const int32_t* pos_dev, const float* emb, const float* pos_emb, float* x,
                  int rows, int d, cudaStream_t st) {
    if (rows <= 0) return;
    CUDA_CHECK(launch_pdl(embed_kernel, dim3(rows), dim3(256), 0, st, tokens_dev, pos_dev, emb, pos_emb, x, rows, d));
}

// =====================================================================================
// encoder self-attention, SIMT flash-style with fp32 arithmetic
//   (reference whisper/model.py:148-173: softmax((q s)(k s)^T) v, no mask, all 1500 positions)
//   grid (ceil(1500/64), H, batch), 256 threads; thread (ty, tx) owns rows ty*4.. x cols tx*4..
// =====================================================================================
template <typename T>
__global__ void __launch_bounds__(256)
enc_attn_simt_kernel(const T* __restrict__ qkv, int n_head, int d_model, T* __restrict__ out) {
    constexpr int BQ = 64, BKV = 64, D = 64, LD = D + 1;
    extern __shared__ float sm[];
    float* Qs = sm;                 // [BQ][LD]
    float* Ks = Qs + BQ * LD;       // [BKV][LD]
    float* Vs = Ks + BKV * LD;      // [BKV][LD]
    float* Ps = Vs + BKV * LD;      // [BQ][LD]
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
    const int64_t ld = 3 * (int64_t)d_model;
    const T* base = qkv + (int64_t)b * N_CTX * ld;

    for (int i = tid; i < BQ * D; i += 256) {
        int r = i >> 6, e = i & 63;
        int row = q0 + r;
        Qs[r * LD + e] = (row < N_CTX) ? to_f32(base[(int64_t)row * ld + h * D + e]) : 0.f;
    }
    float o[4][4], mrow[4], lrow[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        mrow[i] = -INFINITY; lrow[i] = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
    }
    for (int k0 = 0; k0 < N_CTX; k0 += BKV) {
        __syncthreads();
        for (int i = tid; i < BKV * D; i += 256) {
            int r = i >> 6, e = i & 63;
            int row = k0 + r;
            float kv = 0.f, vv = 0.f;
            if (row < N_CTX) {
                kv = to_f32(base[(int64_t)row * ld + d_model + h * D + e]);
                vv = to_f32(base[(int64_t)row * ld + 2 * d_model + h * D + e]);
            }
            Ks[r * LD + e] = kv;
            Vs[r * LD + e] = vv;
        }
        __syncthreads();
        float s[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
        for (int e = 0; e < D; ++e) {
            float a[4], c[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = Qs[(ty * 4 + i) * LD + e];
#pragma unroll
            for (int j = 0; j < 4; ++j) c[j] = Ks[(tx * 4 + j) * LD + e];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) s[i][j] = fmaf(a[i], c[j], s[i][j]);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float mx = -INFINITY;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (k0 + tx * 4 + j >= N_CTX) s[i][j] = -INFINITY;
                mx = fmaxf(mx, s[i][j]);
            }
#pragma unroll
            for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
            const float mnew = fmaxf(mrow[i], mx);
            const float corr = expf(mrow[i] - mnew);       // exp(-inf)=0 on the first tile
            float rs = 0.f;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float p = expf(s[i][j] - mnew);
                rs += p;
                Ps[(ty * 4 + i) * LD + tx * 4 + j] = p;
            }
#pragma unroll
            for (int off = 8; off > 0; off >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, off);
            lrow[i] = lrow[i] * corr + rs;
            mrow[i] = mnew;
#pragma unroll
            for (int j = 0; j < 4; ++j) o[i][j] *= corr;
        }
        __syncthreads();
#pragma unroll 8
        for (int c = 0; c < BKV; ++c) {
            float p[4], v[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) p[i] = Ps[(ty * 4 + i) * LD + c];
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = Vs[c * LD + tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) o[i][j] = fmaf(p[i], v[j], o[i][j]);
        }
    }
    T* ob = out + (int64_t)b * N_CTX * d_model;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int row = q0 + ty * 4 + i;
        if (row >= N_CTX) continue;
        float inv = 1.0f / lrow[i];
#pragma unroll
        for (int j = 0; j < 4; ++j) ob[(int64_t)row * d_model + h * D + tx * 4 + j] = from_f32<T>(o[i][j] * inv);
    }
}

void enc_attention_simt(const void* qkv, int type, int batch, int n_head, int d_model, void* out, cudaStream_t st) {
    dim3 grid((N_CTX + 63) / 64, n_head, batch);
    const int smem = 4 * 64 * 65 * 4;
    static bool seen[64] = {};
    if (first_on_device(seen)) {
        CUDA_CHECK(cudaFuncSetAttribute(enc_attn_simt_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        CUDA_CHECK(cudaFuncSetAttribute(enc_attn_simt_kernel<bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    }
    if (type == DT_F32) enc_attn_simt_kernel<float><<<grid, 256, smem, st>>>((const float*)qkv, n_head, d_model, (float*)out);
    else enc_attn_simt_kernel<bf16><<<grid, 256, smem, st>>>((const bf16*)qkv, n_head, d_model, (bf16*)out);
    CUDA_CHECK(cudaGetLastError());
}

// =====================================================================================
// decoder self-attention over the per-session self-KV cache (causal)
//   (reference whisper/model.py:109-114,130-146,148-173 with the triu(-inf) mask of :278)
//   grid (H, jobs), 128 threads; queries processed one after the other
// =====================================================================================
// One warp per query row (8 queries in flight per CTA), no block-level synchronisation: attend_row_warp (attn_warp.cuh).
template <typename T, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
dec_self_attn_kernel(const T* __restrict__ q, const DecJob* __restrict__ jobs, int layer, int n_head, int d_model,
                     int n_text_ctx, T* __restrict__ out) {
    ptx::griddep_launch();                   // programmatic dependent launch: see launch_pdl (common.cuh)
    ptx::griddep_wait();
    __shared__ float qs[WARPS][64];
    const DecJob job = jobs[blockIdx.y];
    const int h = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const T* Kc = reinterpret_cast<const T*>(job.self_kv) + (((int64_t)layer * 2 + 0) * n_head + h) * n_text_ctx * 64;
    const T* Vc = reinterpret_cast<const T*>(job.self_kv) + (((int64_t)layer * 2 + 1) * n_head + h) * n_text_ctx * 64;
    for (int t = warp; t < job.n_rows; t += WARPS) {
        const int64_t row = job.row_off + t;
        qs[warp][lane] = to_f32(q[row * d_model + h * 64 + lane]);
        qs[warp][lane + 32] = to_f32(q[row * d_model + h * 64 + lane + 32]);
        __syncwarp();
        // causal: keys 0 .. position; ceil(448 / 32) = 14 keys per lane
        attend_row_warp<T, 14>(qs[warp], job.offset + t + 1, [&](int key) { return Kc + (int64_t)key * 64; },
                               [&](int key) { return Vc + (int64_t)key * 64; }, out + row * d_model + h * 64);
        __syncwarp();
    }
}
void dec_self_attention(const void* q, int type, const DecJob* jobs, int n_jobs, int layer, int n_head, int d_model,
                        int n_text_ctx, void* out, int max_rows, cudaStream_t st) {
    WLK_CHECK(n_text_ctx <= 448, "dec_self_attention: n_text_ctx %d > 448", n_text_ctx);
    dim3 grid(n_head, n_jobs);
    if (max_rows <= 1) {                      // token step: one warp per (session, head), a single wave of tiny CTAs
        if (type == DT_F32) CUDA_CHECK(launch_pdl(dec_self_attn_kernel<float, 1>, grid, dim3(32), 0, st, (const float*)q, jobs, layer, n_head, d_model, n_text_ctx, (float*)out));
        else CUDA_CHECK(launch_pdl(dec_self_attn_kernel<bf16, 1>, grid, dim3(32), 0, st, (const bf16*)q, jobs, layer, n_head, d_model, n_text_ctx, (bf16*)out));
    } else {
        if (type == DT_F32) CUDA_CHECK(launch_pdl(dec_self_attn_kernel<float, 8>, grid, dim3(256), 0, st, (const float*)q, jobs, layer, n_head, d_model, n_text_ctx, (float*)out));
        else CUDA_CHECK(launch_pdl(dec_self_attn_kernel<bf16, 8>, grid, dim3(256), 0, st, (const bf16*)q, jobs, layer, n_head, d_model, n_text_ctx, (bf16*)out));
    }
}

// =====================================================================================
// decoder cross-attention over the persistent cross-K/V (1500 frames), with the alignment
// export: for alignment heads the softmaxed rows go to the session's alignment ring
//   (reference whisper/model.py:116-128,148-173; AlignAtt reads softmax(qk) of those heads,
//    simul_whisper.py:401-416)
//   grid (H, jobs), 256 threads, 8 queries per pass
// =====================================================================================
// K and V planes are streamed exactly once per block of QB queries with 128-bit loads: a group of LPK lanes
// covers one 64-wide row, so a warp instruction reads KPW whole rows (512 contiguous bytes); U such loads are
// issued back to back before any is consumed, which is what keeps enough bytes in flight to cover HBM latency.
// QB = 1 is the single-token decode step, QB = 8 the prefill.
template <typename T, int QB>
__global__ void __launch_bounds__(256)
dec_cross_attn_kernel(const T* __restrict__ q, const DecJob* __restrict__ jobs, int layer, int n_head, int d_model,
                      int n_text_ctx, const int32_t* __restrict__ align_rank, T* __restrict__ out, int only_align) {
    ptx::griddep_launch();                   // programmatic dependent launch: see launch_pdl (common.cuh)
    ptx::griddep_wait();
    constexpr int VN = RowVec<T>::N;          // elements per lane
    constexpr int LPK = 64 / VN;              // lanes per key row  (8 bf16 / 16 fp32)
    constexpr int KPW = 32 / LPK;             // key rows per warp instruction (4 / 2)
    constexpr int U = 8;                      // loads in flight per lane
    constexpr int KPI = KPW * U;              // keys per warp per outer iteration
    constexpr int KEYS_PER_WARP = (N_CTX + 7) / 8;
    typedef typename RowVec<T>::Raw Raw;
    extern __shared__ float sm[];
    float* sc = sm;                          // [QB][1500]
    float* qs = sc + QB * N_CTX;             // [QB][64]
    float* part = qs + QB * 64;              // [8 warps][QB][64]
    const DecJob job = jobs[blockIdx.y];
    const int h = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int sub = lane / LPK;              // which of the KPW rows of a warp instruction
    const int seg = (lane % LPK) * VN;       // first of this lane's VN dims
    const T* Kc = reinterpret_cast<const T*>(job.cross_kv) + (((int64_t)layer * 2 + 0) * n_head + h) * N_CTX * 64;
    const T* Vc = reinterpret_cast<const T*>(job.cross_kv) + (((int64_t)layer * 2 + 1) * n_head + h) * N_CTX * 64;
    const int rank = align_rank[layer * n_head + h];
    if (only_align && rank < 0) return;      // the other heads were done on the tensor cores
    const int kbeg = warp * KEYS_PER_WARP, kend = min(N_CTX, kbeg + KEYS_PER_WARP);
    for (int t0 = 0; t0 < job.n_rows; t0 += QB) {
        const int nq = min(QB, job.n_rows - t0);
        for (int i = tid; i < QB * 64; i += 256) {
            int qi = i >> 6, e = i & 63;
            qs[i] = (qi < nq) ? to_f32(q[(int64_t)(job.row_off + t0 + qi) * d_model + h * 64 + e]) : 0.f;
        }
        __syncthreads();
        // ---- scores: s[qi][key] = q[qi] . K[key]
        {
            float qr[QB][VN];
#pragma unroll
            for (int qi = 0; qi < QB; ++qi)
#pragma unroll
                for (int j = 0; j < VN; ++j) qr[qi][j] = qs[qi * 64 + seg + j];
            for (int k0 = kbeg; k0 < kend; k0 += KPI) {
                Raw raw[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int key = k0 + u * KPW + sub;
                    raw[u] = RowVec<T>::load(Kc + (int64_t)min(key, N_CTX - 1) * 64 + seg);
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int key = k0 + u * KPW + sub;
                    float kv[VN];
                    RowVec<T>::unpack(raw[u], kv);
#pragma unroll
                    for (int qi = 0; qi < QB; ++qi) {
                        float a = 0.f;
#pragma unroll
                        for (int j = 0; j < VN; ++j) a = fmaf(qr[qi][j], kv[j], a);
#pragma unroll
                        for (int o = LPK / 2; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
                        if ((lane % LPK) == 0 && key < kend) sc[qi * N_CTX + key] = a;
                    }
                }
            }
        }
        __syncthreads();
        // ---- softmax: warp w normalises query row w; alignment heads export the probabilities
        if (warp < nq) {
            float* r = sc + warp * N_CTX;
            float mx = -INFINITY;
            for (int k = lane; k < N_CTX; k += 32) mx = fmaxf(mx, r[k]);
            mx = warp_max(mx);
            float sum = 0.f;
            for (int k = lane; k < N_CTX; k += 32) { float p = expf(r[k] - mx); r[k] = p; sum += p; }
            sum = warp_sum(sum);
            const float inv = 1.0f / sum;
            float* arow = (rank >= 0)
                ? job.align + ((int64_t)rank * n_text_ctx + job.align_row0 + t0 + warp) * N_CTX : nullptr;
            for (int k = lane; k < N_CTX; k += 32) {
                float p = r[k] * inv;
                r[k] = p;
                if (arow) arow[k] = p;
            }
        }
        __syncthreads();
        // ---- out[qi][e] = sum_key p[qi][key] V[key][e]
        {
            float acc[QB][VN];
#pragma unroll
            for (int qi = 0; qi < QB; ++qi)
#pragma unroll
                for (int j = 0; j < VN; ++j) acc[qi][j] = 0.f;
            for (int k0 = kbeg; k0 < kend; k0 += KPI) {
                Raw raw[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int key = k0 + u * KPW + sub;
                    raw[u] = RowVec<T>::load(Vc + (int64_t)min(key, N_CTX - 1) * 64 + seg);
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int key = k0 + u * KPW + sub;
                    if (key < kend) {
                        float vv[VN];
                        RowVec<T>::unpack(raw[u], vv);
#pragma unroll
                        for (int qi = 0; qi < QB; ++qi) {
                            const float p = sc[qi * N_CTX + key];
#pragma unroll
                            for (int j = 0; j < VN; ++j) acc[qi][j] = fmaf(p, vv[j], acc[qi][j]);
                        }
                    }
                }
            }
            // fold the KPW row-groups of the warp, then the 8 warps through shared memory
#pragma unroll
            for (int qi = 0; qi < QB; ++qi)
#pragma unroll
                for (int j = 0; j < VN; ++j) {
                    float a = acc[qi][j];
#pragma unroll
                    for (int o = LPK; o < 32; o <<= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
                    acc[qi][j] = a;
                }
            if (sub == 0) {
#pragma unroll
                for (int qi = 0; qi < QB; ++qi)
#pragma unroll
                    for (int j = 0; j < VN; ++j) part[(warp * QB + qi) * 64 + seg + j] = acc[qi][j];
            }
        }
        __syncthreads();
        for (int i = tid; i < nq * 64; i += 256) {
            int qi = i >> 6, e = i & 63;
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) v += part[(w * QB + qi) * 64 + e];
            out[(int64_t)(job.row_off + t0 + qi) * d_model + h * 64 + e] = from_f32<T>(v);
        }
        __syncthreads();
    }
}

template <typename T, int QB>
static void launch_cross(const void* q, const DecJob* jobs, int n_jobs, int layer, int n_head, int d_model, int n_text_ctx,
                         const int32_t* align_rank, void* out, int only_align, cudaStream_t st) {
    dim3 grid(n_head, n_jobs);
    const int smem = (QB * N_CTX + QB * 64 + 8 * QB * 64) * 4;
    static bool seen[64] = {};
    if (first_on_device(seen))
        CUDA_CHECK(cudaFuncSetAttribute(dec_cross_attn_kernel<T, QB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CUDA_CHECK(launch_pdl(dec_cross_attn_kernel<T, QB>, grid, dim3(256), (size_t)smem, st, (const T*)q, jobs, layer, n_head, d_model, n_text_ctx, align_rank, (T*)out, only_align));
}
void dec_cross_attention(const void* q, int type, const DecJob* jobs, int n_jobs, int layer, int n_head, int d_model,
                         int n_text_ctx, const int32_t* align_rank, void* out, int max_rows, bool only_align_heads,
                         cudaStream_t st) {
    const bool single = max_rows <= 1;
    const int oa = only_align_heads ? 1 : 0;
    if (type == DT_F32) {
        if (single) launch_cross<float, 1>(q, jobs, n_jobs, layer, n_head, d_model, n_text_ctx, align_rank, out, oa, st);
        else launch_cross<float, 8>(q, jobs, n_jobs, layer, n_head, d_model, n_text_ctx, align_rank, out, oa, st);
    } else {
        if (single) launch_cross<bf16, 1>(q, jobs, n_jobs, layer, n_head, d_model, n_text_ctx, align_rank, out, oa, st);
        else launch_cross<bf16, 8>(q, jobs, n_jobs, layer, n_head, d_model, n_text_ctx, align_rank, out, oa, st);
    }
}

// =====================================================================================
// logits post-processing (reference simul_whisper.py:370-385, whisper/decoding.py:271-287)
// =====================================================================================
__global__ void __launch_bounds__(256)
no_speech_kernel(const LogitJob* __restrict__ jobs, int n_vocab, int no_speech_token, StepResult* __restrict__ res) {
    __shared__ float red[8];
    const float* lg = jobs[blockIdx.x].logits_sot;
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < n_vocab; i += 256) mx = fmaxf(mx, lg[i]);
    mx = block_max_all<256>(mx, red);
    float s = 0.f;
    for (int i = threadIdx.x; i < n_vocab; i += 256) s += expf(lg[i] - mx);
    s = block_sum_all<256>(s, red);
    if (threadIdx.x == 0) res[blockIdx.x].no_speech = expf(lg[no_speech_token] - mx) / s;
}
void no_speech_prob(const LogitJob* jobs, int n, int n_vocab, int no_speech_token, StepResult* res, cudaStream_t st) {
    no_speech_kernel<<<n, 256, 0, st>>>(jobs, n_vocab, no_speech_token, res);
    CUDA_CHECK(cudaGetLastError());
}

__global__ void suppress_kernel(const LogitJob* __restrict__ jobs, const int32_t* __restrict__ toks, int n_tokens) {
    float* lg = jobs[blockIdx.x].logits_last;
    for (int i = threadIdx.x; i < n_tokens; i += blockDim.x) lg[toks[i]] = -INFINITY;
}
void suppress_tokens(const LogitJob* jobs, int n, const int32_t* tokens_dev, int n_tokens, cudaStream_t st) {
    if (n_tokens <= 0) return;
    suppress_kernel<<<n, 128, 0, st>>>(jobs, tokens_dev, n_tokens);
    CUDA_CHECK(cudaGetLastError());
}
__global__ void bias_kernel(float* lg, const int32_t* toks, const float* bias, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) lg[toks[i]] += bias[i];
}
__global__ void bias_jobs_kernel(const LogitJob* __restrict__ jobs, const int32_t* __restrict__ job_of, const int32_t* __restrict__ toks,
                                 const float* __restrict__ bias, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) jobs[job_of[i]].logits_last[toks[i]] += bias[i];
}
void add_logit_bias_jobs(const LogitJob* jobs, const int32_t* job_of_dev, const int32_t* tokens_dev, const float* bias_dev, int n,
                         cudaStream_t st) {
    if (n <= 0) return;
    bias_jobs_kernel<<<(n + 127) / 128, 128, 0, st>>>(jobs, job_of_dev, tokens_dev, bias_dev, n);
    CUDA_CHECK(cudaGetLastError());
}
void add_logit_bias(float* logits, const int32_t* tokens_dev, const float* bias_dev, int n, cudaStream_t st) {
    if (n <= 0) return;
    bias_kernel<<<(n + 127) / 128, 128, 0, st>>>(logits, tokens_dev, bias_dev, n);
    CUDA_CHECK(cudaGetLastError());
}

__global__ void __launch_bounds__(256)
greedy_kernel(const LogitJob* __restrict__ jobs, int n_vocab, StepResult* __restrict__ res) {
    __shared__ float red[8];
    __shared__ int redi[8];
    const float* lg = jobs[blockIdx.x].logits_last;
    float mx = -INFINITY;
    int arg = 0x7fffffff;
    for (int i = threadIdx.x; i < n_vocab; i += 256) {
        float v = lg[i];
        if (v > mx) { mx = v; arg = i; }          // strictly greater: keeps the first index per thread
    }
    // argmax with lowest-index tie break (torch.argmax returns the first maximal element)
    for (int off = 16; off > 0; off >>= 1) {
        float om = __shfl_xor_sync(0xffffffffu, mx, off);
        int oa = __shfl_xor_sync(0xffffffffu, arg, off);
        if (om > mx || (om == mx && oa < arg)) { mx = om; arg = oa; }
    }
    if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = mx; redi[threadIdx.x >> 5] = arg; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w)
            if (red[w] > mx || (red[w] == mx && redi[w] < arg)) { mx = red[w]; arg = redi[w]; }
        red[0] = mx; redi[0] = arg;
    }
    __syncthreads();
    mx = red[0]; arg = redi[0];
    __syncthreads();
    float s = 0.f;
    for (int i = threadIdx.x; i < n_vocab; i += 256) s += expf(lg[i] - mx);
    s = block_sum_all<256>(s, red);
    if (threadIdx.x == 0) {
        res[blockIdx.x].token = arg;
        res[blockIdx.x].logprob = -logf(s);       // log_softmax at the argmax = mx - (mx + log s)
    }
}
void greedy_pick(const LogitJob* jobs, int n, int n_vocab, StepResult* res, cudaStream_t st) {
    greedy_kernel<<<n, 256, 0, st>>>(jobs, n_vocab, res);
    CUDA_CHECK(cudaGetLastError());
}

// =====================================================================================
// AlignAtt reduction (reference simul_whisper.py:418-437 + whisper/timing.py:19-54)
//   stats : per (head, frame) mean and 1/(std+1e-8) over the retained token rows (unbiased=False)
//   rows  : normalise, reflect-padded median-7 over frames, mean over heads, keep [:content_len]
//   argmax: most attended frame of the last row
// =====================================================================================
__global__ void __launch_bounds__(256)
align_stats_kernel(const LogitJob* __restrict__ jobs, int n_text_ctx) {
    const LogitJob job = jobs[blockIdx.z];
    const int a = blockIdx.y, f = blockIdx.x * 256 + threadIdx.x;
    if (f >= N_CTX) return;
    const float* p = job.align + (int64_t)a * n_text_ctx * N_CTX + f;
    const int T = job.row_end - job.row_begin;
    float s = 0.f;
    for (int r = job.row_begin; r < job.row_end; ++r) s += p[(int64_t)r * N_CTX];
    const float mean = s / T;
    float v = 0.f;
    for (int r = job.row_begin; r < job.row_end; ++r) { float d = p[(int64_t)r * N_CTX] - mean; v = fmaf(d, d, v); }
    const float sd = sqrtf(v / T);
    job.stats[((int64_t)a * N_CTX + f) * 2 + 0] = mean;
    job.stats[((int64_t)a * N_CTX + f) * 2 + 1] = 1.0f / (sd + 1e-8f);
}

__device__ __forceinline__ void cswap(float& a, float& b) { float lo = fminf(a, b), hi = fmaxf(a, b); a = lo; b = hi; }
__device__ __forceinline__ float median7(float* v) {
    // 7-input sorting network (16 compare-exchanges); v[3] is the median afterwards
    cswap(v[0], v[6]); cswap(v[2], v[3]); cswap(v[4], v[5]);
    cswap(v[0], v[2]); cswap(v[1], v[4]); cswap(v[3], v[6]);
    cswap(v[0], v[1]); cswap(v[2], v[5]); cswap(v[3], v[4]);
    cswap(v[1], v[2]); cswap(v[4], v[6]);
    cswap(v[2], v[3]); cswap(v[4], v[5]);
    cswap(v[1], v[2]); cswap(v[3], v[4]); cswap(v[5], v[6]);
    return v[3];
}

__global__ void __launch_bounds__(256)
align_rows_kernel(const LogitJob* __restrict__ jobs, int n_align, int n_text_ctx) {
    const LogitJob job = jobs[blockIdx.z];
    const int T = job.row_end - job.row_begin;
    const int n_out = job.full ? T : 1;
    if ((int)blockIdx.y >= n_out) return;
    const int r = job.full ? (job.row_begin + blockIdx.y) : (job.row_end - 1);
    const int f = blockIdx.x * 256 + threadIdx.x;
    if (f >= job.content_len) return;
    float acc = 0.f;
    for (int a = 0; a < n_align; ++a) {
        const float* p = job.align + ((int64_t)a * n_text_ctx + r) * N_CTX;
        const float* st = job.stats + (int64_t)a * N_CTX * 2;
        float v[7];
#pragma unroll
        for (int j = 0; j < 7; ++j) {
            int g = f + j - 3;
            if (g < 0) g = -g;                           // reflect (no edge repeat), F.pad(mode="reflect")
            if (g >= N_CTX) g = 2 * (N_CTX - 1) - g;
            g += job.rot;                                // ring-addressed encoder output (0 in parity mode)
            if (g >= N_CTX) g -= N_CTX;
            v[j] = (p[g] - st[g * 2]) * st[g * 2 + 1];
        }
        acc += median7(v);
    }
    job.attn_out[(int64_t)(r - job.row_begin) * N_CTX + f] = acc / n_align;
}

__global__ void __launch_bounds__(256)
align_argmax_kernel(const LogitJob* __restrict__ jobs, StepResult* __restrict__ res) {
    __shared__ float red[8];
    __shared__ int redi[8];
    const LogitJob job = jobs[blockIdx.x];
    const int T = job.row_end - job.row_begin;
    const float* row = job.attn_out + (int64_t)(T - 1) * N_CTX;
    float mx = -INFINITY;
    int arg = 0x7fffffff;
    for (int i = threadIdx.x; i < job.content_len; i += 256) {
        float v = row[i];
        if (v > mx) { mx = v; arg = i; }
    }
    for (int off = 16; off > 0; off >>= 1) {
        float om = __shfl_xor_sync(0xffffffffu, mx, off);
        int oa = __shfl_xor_sync(0xffffffffu, arg, off);
        if (om > mx || (om == mx && oa < arg)) { mx = om; arg = oa; }
    }
    if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = mx; redi[threadIdx.x >> 5] = arg; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w)
            if (red[w] > mx || (red[w] == mx && redi[w] < arg)) { mx = red[w]; arg = redi[w]; }
        res[blockIdx.x].frame = (arg == 0x7fffffff) ? 0 : arg;
    }
}

void align_reduce(const LogitJob* jobs, int n, int n_align, int n_text_ctx, StepResult* res, cudaStream_t st) {
    dim3 g1((N_CTX + 255) / 256, n_align, n);
    align_stats_kernel<<<g1, 256, 0, st>>>(jobs, n_text_ctx);
    CUDA_CHECK(cudaGetLastError());
    dim3 g2((N_CTX + 255) / 256, n_text_ctx, n);      // rows beyond the retained window exit immediately
    align_rows_kernel<<<g2, 256, 0, st>>>(jobs, n_align, n_text_ctx);
    CUDA_CHECK(cudaGetLastError());
    align_argmax_kernel<<<n, 256, 0, st>>>(jobs, res);
    CUDA_CHECK(cudaGetLastError());
}


// =====================================================================================
// incremental encoder helpers (engine.cu encode_incremental)
// =====================================================================================
// conv1 operand rows of a block: frame f in [2 p0 - 1, 2 p1) reads mel rows f .. f + 2 of the padded time-major buffer
// (row 0 is the zero pad row, frame f sits at row f + 1); frames outside [0, 3000) give zero rows (conv2's padding)
template <typename T>
__global__ void inc_gather_conv1_kernel(const IncJob* __restrict__ jobs, int n_mels, T* __restrict__ A1) {
    const IncJob job = jobs[blockIdx.y];
    const int nr = 2 * (job.p1 - job.p0) + 1, r = blockIdx.x;
    if (r >= nr) return;
    const int f = 2 * job.p0 - 1 + r, K = 3 * n_mels;
    T* dst = A1 + (int64_t)(job.row1_off + r) * K;
    const T* src = reinterpret_cast<const T*>(job.mel) + (int64_t)f * n_mels;    // rows f .. f + 2 are contiguous
    const bool ok = f >= 0 && f < N_FRAMES;
    for (int i = threadIdx.x; i < K; i += blockDim.x) dst[i] = ok ? src[i] : from_f32<T>(0.f);
}
void inc_gather_conv1(const IncJob* jobs, int n, int max_rows1, int n_mels, void* A1, int type, cudaStream_t st) {
    if (type == DT_BF16) inc_gather_conv1_kernel<bf16><<<dim3(max_rows1, n), 128, 0, st>>>(jobs, n_mels, (bf16*)A1);
    else inc_gather_conv1_kernel<float><<<dim3(max_rows1, n), 128, 0, st>>>(jobs, n_mels, (float*)A1);
    CUDA_CHECK(cudaGetLastError());
}
// conv2 operand rows: position p reads conv1 frames 2 p - 1 .. 2 p + 1 = packed conv1 rows 2 (p - p0) .. + 2 (contiguous);
// conv1 rows of frames outside the window are conv2's zero padding.  Also the row maps and the positional rows (by slot).
template <typename T>
__global__ void inc_gather_conv2_kernel(const IncJob* __restrict__ jobs, int d, const T* __restrict__ H1, T* __restrict__ A2,
                                        const float* __restrict__ enc_pos, float* __restrict__ posbuf, int32_t* __restrict__ row_slot,
                                        int32_t* __restrict__ row_pos) {
    const IncJob job = jobs[blockIdx.y];
    const int r = blockIdx.x;
    if (r >= job.p1 - job.p0) return;
    const int p = job.p0 + r;
    int slot = p + job.rot;
    if (slot >= N_CTX) slot -= N_CTX;
    const int64_t row = job.row_off + r;
    for (int k = 0; k < 3; ++k) {
        const int f = 2 * p - 1 + k;
        const bool ok = f >= 0 && f < N_FRAMES;
        const T* src = H1 + (int64_t)(job.row1_off + 2 * r + k) * d;
        T* dst = A2 + row * 3 * d + (int64_t)k * d;
        for (int i = threadIdx.x; i < d; i += blockDim.x) dst[i] = ok ? src[i] : from_f32<T>(0.f);
    }
    for (int i = threadIdx.x; i < d; i += blockDim.x) posbuf[row * d + i] = enc_pos[(int64_t)slot * d + i];
    if (threadIdx.x == 0) { row_slot[row] = blockIdx.y; row_pos[row] = slot; }
}
void inc_gather_conv2(const IncJob* jobs, int n, int max_rows, int d, const void* H1, void* A2, const float* enc_pos, float* posbuf,
                      int32_t* row_slot, int32_t* row_pos, int type, cudaStream_t st) {
    if (type == DT_BF16) inc_gather_conv2_kernel<bf16><<<dim3(max_rows, n), 256, 0, st>>>(jobs, d, (const bf16*)H1, (bf16*)A2, enc_pos, posbuf, row_slot, row_pos);
    else inc_gather_conv2_kernel<float><<<dim3(max_rows, n), 256, 0, st>>>(jobs, d, (const float*)H1, (float*)A2, enc_pos, posbuf, row_slot, row_pos);
    CUDA_CHECK(cudaGetLastError());
}
template <typename T>
__global__ void inc_scatter_rows_kernel(const IncJob* __restrict__ jobs, int d, const T* __restrict__ src) {
    const IncJob job = jobs[blockIdx.y];
    const int r = blockIdx.x;
    if (r >= job.p1 - job.p0) return;
    int slot = job.p0 + r + job.rot;
    if (slot >= N_CTX) slot -= N_CTX;
    const T* s = src + (int64_t)(job.row_off + r) * d;
    T* dst = reinterpret_cast<T*>(job.xa) + (int64_t)slot * d;
    for (int i = threadIdx.x; i < d; i += blockDim.x) dst[i] = s[i];
}
void inc_scatter_rows(const IncJob* jobs, int n, int max_rows, int d, const void* src, int type, cudaStream_t st) {
    if (type == DT_BF16) inc_scatter_rows_kernel<bf16><<<dim3(max_rows, n), 256, 0, st>>>(jobs, d, (const bf16*)src);
    else inc_scatter_rows_kernel<float><<<dim3(max_rows, n), 256, 0, st>>>(jobs, d, (const float*)src);
    CUDA_CHECK(cudaGetLastError());
}
// =====================================================================================
// Word-timestamp kernels of the LocalAgreement path: native replacements of the reference's two Triton
// kernels (whisper/triton_ops.py:13-103) with the semantics of its CPU path, which is the parity oracle
// (whisper/timing.py:19-54 median_filter, :57-105 dtw_cpu + backtrace).
// =====================================================================================
// median over a sliding window of odd width <= 15 along the last axis, reflect padding (no edge repeat)
__global__ void __launch_bounds__(256)
median_filter_kernel(const float* __restrict__ x, float* __restrict__ out, int rows, int cols, int width) {
    const int r = blockIdx.y;
    const int c = blockIdx.x * 256 + threadIdx.x;
    if (r >= rows || c >= cols) return;
    const float* xr = x + (int64_t)r * cols;
    const int pad = width / 2;
    float v[15];
    for (int j = 0; j < width; ++j) {
        int g = c + j - pad;
        if (g < 0) g = -g;
        if (g >= cols) g = 2 * (cols - 1) - g;
        v[j] = xr[g];
    }
    for (int a = 1; a < width; ++a) {                 // insertion sort (width is tiny)
        float key = v[a];
        int b = a - 1;
        while (b >= 0 && v[b] > key) { v[b + 1] = v[b]; --b; }
        v[b + 1] = key;
    }
    out[(int64_t)r * cols + c] = v[pad];
}
void median_filter(const float* x, float* out, int rows, int cols, int width, cudaStream_t st) {
    WLK_CHECK(width >= 1 && width <= 15 && (width & 1), "median_filter: width %d must be odd and <= 15", width);
    if (cols <= width / 2) {                          // timing.py:22-24: too short to pad, returned unchanged
        CUDA_CHECK(cudaMemcpyAsync(out, x, (size_t)rows * cols * 4, cudaMemcpyDeviceToDevice, st));
        return;
    }
    dim3 grid((cols + 255) / 256, rows);
    median_filter_kernel<<<grid, 256, 0, st>>>(x, out, rows, cols, width);
    CUDA_CHECK(cudaGetLastError());
}

// Dynamic time warping over x[N tokens, M frames]: anti-diagonal wavefront (thread = token row), three
// rotating diagonals in shared memory, byte trace in global memory, then the serial backtrace by one thread.
// Move choice follows dtw_cpu exactly: diagonal only if strictly cheaper than both, else up only if
// strictly cheaper than both, else left.  One CTA per problem (blockIdx.x = problem index).
struct DtwJob { const float* x; uint8_t* trace; int32_t* path; int32_t* path_len; int32_t N, M; };

__global__ void __launch_bounds__(512)
dtw_kernel(const DtwJob* __restrict__ jobs) {
    extern __shared__ float dsm[];
    const DtwJob job = jobs[blockIdx.x];
    const int N = job.N, M = job.M, tid = threadIdx.x;
    float* d0 = dsm;                       // diagonal k-2
    float* d1 = dsm + (N + 1);             // diagonal k-1
    float* d2 = dsm + 2 * (N + 1);         // diagonal k
    for (int i = tid; i <= N; i += 512) { d0[i] = INFINITY; d1[i] = INFINITY; d2[i] = INFINITY; }
    __syncthreads();
    if (tid == 0) d0[0] = 0.f;             // cost[0][0]; diagonal 1 (cost[0][1], cost[1][0]) stays inf
    __syncthreads();
    for (int k = 2; k <= N + M; ++k) {
        const int lo = max(1, k - M), hi = min(N, k - 1);
        for (int i = lo + tid; i <= hi; i += 512) {
            const int j = k - i;
            const float c0 = d0[i - 1], c1 = d1[i - 1], c2 = d1[i];
            float c; uint8_t t;
            if (c0 < c1 && c0 < c2) { c = c0; t = 0; }
            else if (c1 < c0 && c1 < c2) { c = c1; t = 1; }
            else { c = c2; t = 2; }
            d2[i] = __fadd_rn(job.x[(int64_t)(i - 1) * M + (j - 1)], c);
            job.trace[(int64_t)i * (M + 1) + j] = t;
        }
        if (tid == 0) { d2[0] = INFINITY; if (k <= N) d2[k] = INFINITY; }   // cost[0][k], cost[k][0]
        __syncthreads();
        float* tmp = d0; d0 = d1; d1 = d2; d2 = tmp;
        __syncthreads();
    }
    if (tid == 0) {                        // backtrace (timing.py:57-79), written in forward order
        int i = N, j = M, n = 0;
        int32_t* tmp = job.path + 2 * (N + M);           // scratch behind the two output rows
        while (i > 0 || j > 0) {
            tmp[2 * n] = i - 1; tmp[2 * n + 1] = j - 1; ++n;
            const int t = (i == 0) ? 2 : (j == 0) ? 1 : job.trace[(int64_t)i * (M + 1) + j];
            if (t == 0) { --i; --j; } else if (t == 1) --i; else --j;
        }
        for (int q = 0; q < n; ++q) {
            job.path[q] = tmp[2 * (n - 1 - q)];                 // text (token) indices
            job.path[(N + M) + q] = tmp[2 * (n - 1 - q) + 1];   // time (frame) indices
        }
        *job.path_len = n;
    }
}
void dtw_batch(const void* jobs_dev, int n_jobs, int max_tokens, cudaStream_t st) {
    const int smem = 3 * (max_tokens + 1) * 4;
    dtw_kernel<<<n_jobs, 512, smem, st>>>(reinterpret_cast<const DtwJob*>(jobs_dev));
    CUDA_CHECK(cudaGetLastError());
}

}  // namespace wlk
