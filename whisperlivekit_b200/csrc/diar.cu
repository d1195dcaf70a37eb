// Step after the diarization forward (SURVEY.md section 8f item 4): run-length speaker segments on the device.
//   reference whisperlivekit/diarization/sortformer_backend.py:313-363 (_process_predictions): of the frames x speakers
//   sigmoid matrix `total_preds` the LAST `len_prediction` frames are reduced to argmax over the first `max_speakers`
//   channels (arrival-ordered identities; np.argmax: first maximum wins, NaN counts as the maximum) and consecutive
//   equal speakers are merged into segments.  The reference copies the whole (ever growing) total_preds to the host
//   every chunk (:315); here only the (speaker, first frame, end frame) triples cross PCIe, for all streams in one call.
#include <vector>

#include "../../include/wlk_b200.h"
#include "common.cuh"
#include "host.cuh"

namespace wlk {
namespace {

constexpr int DIAR_MAX_FRAMES = 4096;      // frames of one chunk a stream may hand in (the reference: ~12 per 1 s step)

struct DiarJob { const float* preds; int32_t n_frames_total; int32_t len_prediction; int32_t n_spk; int32_t max_speakers; };

// one CTA per stream; thread t owns frames t, t + 256, ...
__global__ void __launch_bounds__(256)
diar_segments_kernel(const DiarJob* __restrict__ jobs, int32_t* __restrict__ seg_out /*[n][max_seg][3]*/,
                     int32_t* __restrict__ seg_count, int max_seg) {
    __shared__ int16_t spk[DIAR_MAX_FRAMES];
    __shared__ int warp_tot[8];
    __shared__ int base;
    const DiarJob job = jobs[blockIdx.x];
    const int n = min(job.len_prediction, job.n_frames_total);         // active_speakers[-len_prediction:]
    const float* p = job.preds + (int64_t)(job.n_frames_total - n) * job.n_spk;
    for (int f = threadIdx.x; f < n; f += 256) {
        const float* row = p + (int64_t)f * job.n_spk;
        int best = 0;
        float bv = row[0];
        bool nan_seen = bv != bv;
        for (int c = 1; c < job.max_speakers && !nan_seen; ++c) {     // np.argmax: first occurrence of the maximum; NaN is maximal
            const float v = row[c];
            if (v != v) { best = c; nan_seen = true; }
            else if (v > bv) { bv = v; best = c; }
        }
        spk[f] = (int16_t)best;
    }
    if (threadIdx.x == 0) base = 0;
    __syncthreads();
    int32_t* out = seg_out + (int64_t)blockIdx.x * max_seg * 3;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int f0 = 0; f0 < n; f0 += 256) {                              // block-wide exclusive scan of the boundary flags
        const int f = f0 + threadIdx.x;
        const int flag = (f < n && (f == 0 || spk[f] != spk[f - 1])) ? 1 : 0;
        int incl = flag;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        int woff = 0;
        for (int w = 0; w < warp; ++w) woff += warp_tot[w];
        const int idx = base + woff + incl - 1;                        // index of the segment that starts at frame f
        if (flag && idx < max_seg) {
            out[idx * 3 + 0] = spk[f];
            out[idx * 3 + 1] = f;
            if (idx > 0) out[(idx - 1) * 3 + 2] = f;                   // the previous segment ends where this one starts
        }
        __syncthreads();
        if (threadIdx.x == 255) base += woff + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const int total = base;
        if (total > 0 && total <= max_seg) out[(total - 1) * 3 + 2] = n;
        seg_count[blockIdx.x] = total;
    }
}

}  // namespace
}  // namespace wlk

using namespace wlk;

extern "C" int wlk_diar_segments(int device, const float* const* preds_dev, const int32_t* n_frames_total,
                                 const int32_t* len_prediction, int n_streams, int n_spk, int max_speakers,
                                 int32_t* seg_out_host, int32_t* seg_count_host, int max_seg) {
    WLK_API_BEGIN
    WLK_CHECK(preds_dev && n_frames_total && len_prediction && seg_out_host && seg_count_host, "null argument");
    WLK_CHECK(n_streams >= 1 && n_streams <= 65535 && max_seg >= 1, "bad stream / segment count");
    WLK_CHECK(n_spk >= 1 && max_speakers >= 1, "bad speaker count");
    // sortformer_backend.py:316-319
    WLK_CHECK(n_spk >= max_speakers, "Sortformer returned fewer speaker channels (%d) than configured (%d).", n_spk, max_speakers);
    use_device(device);
    std::vector<DiarJob> jobs(n_streams);
    for (int i = 0; i < n_streams; ++i) {
        WLK_CHECK(n_frames_total[i] >= 0 && len_prediction[i] >= 0, "negative frame count for stream %d", i);
        const int n = std::min(n_frames_total[i], len_prediction[i]);
        WLK_CHECK(n <= DIAR_MAX_FRAMES, "stream %d: %d frames in one chunk exceed %d", i, n, DIAR_MAX_FRAMES);
        WLK_CHECK(n == 0 || preds_dev[i] != nullptr, "stream %d: null predictions", i);
        jobs[i] = DiarJob{preds_dev[i], n_frames_total[i], len_prediction[i], n_spk, max_speakers};
    }
    DiarJob* jobs_dev = nullptr; int32_t *seg_dev = nullptr, *cnt_dev = nullptr;
    cudaStream_t st;
    CUDA_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    CUDA_CHECK(cudaMallocAsync(&jobs_dev, sizeof(DiarJob) * n_streams, st));
    CUDA_CHECK(cudaMallocAsync(&seg_dev, sizeof(int32_t) * 3 * (size_t)max_seg * n_streams, st));
    CUDA_CHECK(cudaMallocAsync(&cnt_dev, sizeof(int32_t) * n_streams, st));
    CUDA_CHECK(cudaMemcpyAsync(jobs_dev, jobs.data(), sizeof(DiarJob) * n_streams, cudaMemcpyHostToDevice, st));
    diar_segments_kernel<<<n_streams, 256, 0, st>>>(jobs_dev, seg_dev, cnt_dev, max_seg);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(seg_count_host, cnt_dev, sizeof(int32_t) * n_streams, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaMemcpyAsync(seg_out_host, seg_dev, sizeof(int32_t) * 3 * (size_t)max_seg * n_streams, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    cudaFreeAsync(jobs_dev, st); cudaFreeAsync(seg_dev, st); cudaFreeAsync(cnt_dev, st);
    cudaStreamSynchronize(st);
    cudaStreamDestroy(st);
    for (int i = 0; i < n_streams; ++i)
        WLK_CHECK(seg_count_host[i] <= max_seg, "stream %d produced %d segments, capacity %d", i, seg_count_host[i], max_seg);
    WLK_API_END
}
