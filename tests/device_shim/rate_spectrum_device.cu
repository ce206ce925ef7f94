// TEST INFRASTRUCTURE — not part of the product.
// Device harness for the decimator and its frequency shift (K11/K12, launch_decimate: modes_resample.cu) and
// the input spectrum pass (K13, launch_spectrum and launch_spectrum_pool: modes_spectrum.cu), so that
// tests/test_rate_kernels.py can check them byte for byte on spans, offsets and jobs it chooses, including
// the ones the decoder never builds.  It is linked against the product's own objects (build/modes_resample.o,
// build/modes_spectrum.o), exactly what libmodes_b200.so ships.
//
// Each entry runs exactly one launch, synchronises and downloads every zone the launch may write together with
// a guard zone after it, all filled with a sentinel before the launch, so a test also sees every byte the
// launch must leave alone.  The span is followed by 16 bytes of 0xa5 that must not be read as input.  Every
// argument is checked on the host first; a bad request returns an error and launches nothing.  The kernels
// read only inside in_bytes (and a pool job's hist and stage) and write only the zones allocated here.
#include <cstdint>
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#include "modes_internal.h"
#include "modes_resample_core.cuh"
#include "modes_spectrum_core.cuh"

namespace {
using namespace modes;

char g_err[256] = "";

int set_err(const char *what, cudaError_t e = cudaSuccess) {
    snprintf(g_err, sizeof(g_err), "%s%s%s", what, e != cudaSuccess ? ": " : "", e != cudaSuccess ? cudaGetErrorString(e) : "");
    return -1;
}

#define HCK(call)                                               \
    do {                                                        \
        cudaError_t e_ = (call);                                \
        if (e_ != cudaSuccess) return set_err(#call, e_);       \
    } while (0)

// Device memory freed on every return path.
struct Buffers {
    std::vector<void *> p;
    template <class T> cudaError_t alloc(T **out, size_t bytes) {
        void *q = nullptr;
        const cudaError_t e = cudaMalloc(&q, bytes ? bytes : 16);
        if (e == cudaSuccess) p.push_back(q);
        *out = static_cast<T *>(q);
        return e;
    }
    ~Buffers() { for (void *q : p) cudaFree(q); }
};

constexpr size_t kGuard = 256;                    // sentinel bytes after the body and after the carry block
constexpr uint64_t kMaxBytes = 1ull << 31;        // the largest span or body a request may ask for

// The span, uploaded with 16 bytes of 0xa5 after it.
int upload_span(Buffers &mem, const uint8_t *in, uint64_t in_bytes, uint8_t **d_in) {
    HCK(mem.alloc(d_in, in_bytes + 16));
    if (in_bytes) HCK(cudaMemcpy(*d_in, in, in_bytes, cudaMemcpyHostToDevice));
    HCK(cudaMemset(*d_in + in_bytes, 0xa5, 16));
    return 0;
}

}  // namespace

extern "C" {

const char *rate_error() { return g_err; }

// The step launch_decimate gets for offset_hz at 2 MHz * m (shift::step), or 0 with an error for an offset
// offset_fits refuses or an m the decoder does not take.
uint32_t rate_step(int m, int32_t offset_hz) {
    const InputRate *r = m >= 2 && m <= 5 ? find_input_rate(2000000u * (uint32_t)m) : nullptr;
    if (!r || !offset_fits(*r, offset_hz)) {
        set_err("rate or offset out of range");
        return 0;
    }
    return shift::step(offset_hz, r->hz);
}

// One launch_decimate: output samples [out_first, out_first + out_samples) of a 2 M MS/s stream into body and,
// with want_halo, the carry block before them into halo, from the span in (in_bytes bytes from input sample
// in_first; UC8 with shift -1, else int16 converted with the shift), each input sample rotated by offset_hz.
// body: 2 out_samples + kGuard bytes, halo: kHaloAlloc + kGuard bytes, both downloaded whole (sentinel 0x5a
// wherever the launch wrote nothing).
int decimate_run(int m, int shift, int32_t offset_hz, const uint8_t *in, uint64_t in_bytes, int64_t in_first,
                 int64_t out_first, uint64_t out_samples, int64_t out_end, int want_halo, uint8_t *body, uint8_t *halo) {
    if (m < 2 || m > 5) return set_err("m out of range");
    if (shift < -1 || shift > 15) return set_err("shift out of range");
    const uint32_t step = offset_hz ? rate_step(m, offset_hz) : 0;
    if (offset_hz && !step) return -1;
    if (!body || !halo || !out_samples || out_samples % 8 || out_first % 8 || 2 * out_samples > kMaxBytes)
        return set_err("output out of range");
    if (in_bytes > kMaxBytes || (in_bytes && !in)) return set_err("input out of range");
    // stream indices stay far from int64's edges: M n0 and 2 (M n0 - in_first) have room
    const int64_t kPos = (int64_t)1 << 56;
    if (in_first < -kPos || in_first > kPos || out_first < -kPos / 8 || out_first > kPos / 8) return set_err("position out of range");
    Buffers mem;
    uint8_t *d_in = nullptr, *d_body = nullptr, *d_halo = nullptr;
    if (upload_span(mem, in, in_bytes, &d_in)) return -1;
    HCK(mem.alloc(&d_body, 2 * out_samples + kGuard));
    HCK(mem.alloc(&d_halo, kHaloAlloc + kGuard));
    HCK(cudaMemset(d_body, 0x5a, 2 * out_samples + kGuard));
    HCK(cudaMemset(d_halo, 0x5a, kHaloAlloc + kGuard));
    const ResampleJob j{d_in, in_bytes, in_first, out_first, out_samples, out_end, d_body, want_halo ? d_halo : nullptr};
    launch_decimate(j, m, shift, step, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(body, d_body, 2 * out_samples + kGuard, cudaMemcpyDeviceToHost));
    HCK(cudaMemcpy(halo, d_halo, kHaloAlloc + kGuard, cudaMemcpyDeviceToHost));
    return 0;
}

// One launch_spectrum: the records of reference buffers first_buffer ... + n_buffers - 1 of a stream at the
// ratio out : in from the span (as decimate_run's).  records: n_buffers + 1 modes_spectrum; the first n_buffers
// start at zero, the last (the guard) is filled with 0x5a, and all are downloaded.
int spectrum_run(int shift, int out, int in_ratio, const uint8_t *in, uint64_t in_bytes, int64_t in_first,
                 int64_t first_buffer, uint32_t n_buffers, modes_spectrum *records) {
    if (shift < -1 || shift > 15) return set_err("shift out of range");
    const bool ratio_ok = (out == 1 && in_ratio >= 1 && in_ratio <= 5) || (out == 5 && in_ratio == 6);
    if (!ratio_ok) return set_err("ratio out of range");
    if (!records || !n_buffers || n_buffers > 4096) return set_err("records out of range");
    if (in_bytes > kMaxBytes || (in_bytes && !in)) return set_err("input out of range");
    const int64_t kPos = (int64_t)1 << 48;
    if (first_buffer < 0 || first_buffer > kPos / MODES_BUFFER_SAMPLES || in_first < -kPos || in_first > kPos)
        return set_err("position out of range");
    Buffers mem;
    uint8_t *d_in = nullptr;
    modes_spectrum *d_rec = nullptr;
    if (upload_span(mem, in, in_bytes, &d_in)) return -1;
    const size_t rec_bytes = (size_t)n_buffers * sizeof(modes_spectrum);
    HCK(mem.alloc(&d_rec, rec_bytes + sizeof(modes_spectrum)));
    HCK(cudaMemset(d_rec, 0, rec_bytes));
    HCK(cudaMemset(reinterpret_cast<uint8_t *>(d_rec) + rec_bytes, 0x5a, sizeof(modes_spectrum)));
    const ResampleJob j{d_in, in_bytes, in_first, 0, 0, INT64_MAX, nullptr, nullptr};
    launch_spectrum(j, shift, out, in_ratio, first_buffer, n_buffers, d_rec, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(records, d_rec, rec_bytes + sizeof(modes_spectrum), cudaMemcpyDeviceToHost));
    return 0;
}

// One launch_spectrum_pool over n_jobs jobs.  Job k reads its history, hist_bytes[k] = call0[k] - hist0[k] bytes
// at hist + hist_off[k], and its call, MODES_BUFFER_BYTES at stage + stage_off[k] (offsets into the two host
// arrays, multiples of 16); hist0 and call0 multiples of 16.  Its buffer's frames start at stream sample
// first[k].  max_frames: the most frames of a job (what the pool passes).  records as spectrum_run's.
int spectrum_pool_run(uint32_t n_jobs, const uint8_t *hist, uint64_t hist_total, const uint64_t *hist_off,
                      const uint8_t *stage, uint64_t stage_total, const uint64_t *stage_off, const int64_t *hist0,
                      const int64_t *call0, const int64_t *buffer, const int64_t *first, const uint32_t *frames,
                      uint32_t max_frames, modes_spectrum *records) {
    if (!n_jobs || n_jobs > 4096 || !records || !hist_off || !stage_off || !hist0 || !call0 || !buffer || !first || !frames)
        return set_err("jobs out of range");
    if (hist_total > kMaxBytes || stage_total > kMaxBytes || (hist_total && !hist) || !stage || hist_total % 16 || stage_total % 16)
        return set_err("input out of range");
    uint32_t most = 0;
    const int64_t kPos = (int64_t)1 << 48;
    for (uint32_t k = 0; k < n_jobs; k++) {
        if (hist0[k] % 16 || call0[k] % 16 || call0[k] < hist0[k] || hist0[k] < -kPos || call0[k] > kPos)
            return set_err("job bounds out of range");
        if (hist_off[k] % 16 || hist_off[k] > hist_total || (uint64_t)(call0[k] - hist0[k]) > hist_total - hist_off[k])
            return set_err("job history out of range");
        if (stage_off[k] % 16 || stage_off[k] > stage_total || MODES_BUFFER_BYTES > stage_total - stage_off[k])
            return set_err("job call out of range");
        if (first[k] < -kPos || first[k] > kPos || buffer[k] < 0 || frames[k] > 4096) return set_err("job frames out of range");
        most = frames[k] > most ? frames[k] : most;
    }
    if (max_frames < most || max_frames > 4096) return set_err("max_frames out of range");
    Buffers mem;
    uint8_t *d_hist = nullptr, *d_stage = nullptr;
    PoolSpectrumJob *d_jobs = nullptr;
    modes_spectrum *d_rec = nullptr;
    HCK(mem.alloc(&d_hist, hist_total));
    HCK(mem.alloc(&d_stage, stage_total));
    if (hist_total) HCK(cudaMemcpy(d_hist, hist, hist_total, cudaMemcpyHostToDevice));
    HCK(cudaMemcpy(d_stage, stage, stage_total, cudaMemcpyHostToDevice));
    std::vector<PoolSpectrumJob> jobs(n_jobs);
    for (uint32_t k = 0; k < n_jobs; k++)
        jobs[k] = PoolSpectrumJob{d_hist + hist_off[k], d_stage + stage_off[k], hist0[k], call0[k], buffer[k], first[k], frames[k], 0};
    HCK(mem.alloc(&d_jobs, n_jobs * sizeof(PoolSpectrumJob)));
    HCK(cudaMemcpy(d_jobs, jobs.data(), n_jobs * sizeof(PoolSpectrumJob), cudaMemcpyHostToDevice));
    const size_t rec_bytes = (size_t)n_jobs * sizeof(modes_spectrum);
    HCK(mem.alloc(&d_rec, rec_bytes + sizeof(modes_spectrum)));
    HCK(cudaMemset(d_rec, 0, rec_bytes));
    HCK(cudaMemset(reinterpret_cast<uint8_t *>(d_rec) + rec_bytes, 0x5a, sizeof(modes_spectrum)));
    launch_spectrum_pool(d_jobs, n_jobs, max_frames, d_rec, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(records, d_rec, rec_bytes + sizeof(modes_spectrum), cudaMemcpyDeviceToHost));
    return 0;
}

}  // extern "C"
