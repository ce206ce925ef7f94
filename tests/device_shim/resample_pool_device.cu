// TEST INFRASTRUCTURE — not part of the product.
// Device harness for the receiver pool's resampling launches (launch_resample_pool and
// launch_history_pool, modes_resample.cu), so that tests/test_pool_input_rate.py can check them byte for
// byte on jobs it lays out itself.  It is linked against the product's own object (build/modes_resample.o),
// exactly what libmodes_b200.so ships.
//
// Jobs name offsets into host arrays, which the harness uploads whole: `hist` (the receivers' input
// histories), `stage` (the call's buffers) and `out` (the batch's pairs for resampling, the histories'
// other halves for the history step).  It runs the one launch, synchronises and downloads `out` whole, so
// a test also sees every byte the launch must leave alone.  Every offset and span is checked on the host
// first; a bad request returns an error and runs nothing.
#include <cstdint>
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#include "modes_internal.h"

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

// [off, off + len) inside an array of n bytes, off a multiple of `align`.
bool inside(int64_t off, int64_t len, size_t n, int64_t align) {
    return off >= 0 && len >= 0 && off % align == 0 && (uint64_t)(off + len) <= n;
}

struct Arrays {
    uint8_t *hist = nullptr, *stage = nullptr, *out = nullptr;
};

int upload(Buffers &mem, Arrays &d, const uint8_t *hist, size_t hist_bytes, const uint8_t *stage, size_t stage_bytes,
           const uint8_t *out, size_t out_bytes) {
    HCK(mem.alloc(&d.hist, hist_bytes));
    HCK(mem.alloc(&d.stage, stage_bytes));
    HCK(mem.alloc(&d.out, out_bytes));
    if (hist_bytes) HCK(cudaMemcpy(d.hist, hist, hist_bytes, cudaMemcpyHostToDevice));
    if (stage_bytes) HCK(cudaMemcpy(d.stage, stage, stage_bytes, cudaMemcpyHostToDevice));
    if (out_bytes) HCK(cudaMemcpy(d.out, out, out_bytes, cudaMemcpyHostToDevice));
    return 0;
}

template <class Job> int run(Buffers &mem, const std::vector<Job> &jobs, Job **d_jobs) {
    HCK(mem.alloc(d_jobs, jobs.size() * sizeof(Job)));
    HCK(cudaMemcpy(*d_jobs, jobs.data(), jobs.size() * sizeof(Job), cudaMemcpyHostToDevice));
    return 0;
}

}  // namespace

extern "C" {

const char *rpool_error() { return g_err; }

// One resampling job: hist_off < 0 for none (call0 == hist0); out_first < 0: a 2 MHz pass-through job.
struct ShimResampleJob {
    int64_t hist_off, stage_off, hist0, call0, out_first, pad_tail_off, data_off;
};

int rpool_resample(const uint8_t *hist, size_t hist_bytes, const uint8_t *stage, size_t stage_bytes, uint8_t *out,
                   size_t out_bytes, const ShimResampleJob *jobs, uint32_t n_jobs) {
    if (!n_jobs || n_jobs > 4096 || !jobs || !out) return set_err("empty request");
    for (uint32_t i = 0; i < n_jobs; i++) {
        const ShimResampleJob &j = jobs[i];
        if (!inside(j.stage_off, MODES_BUFFER_BYTES, stage_bytes, 16) || !inside(j.data_off, MODES_BUFFER_BYTES, out_bytes, 16))
            return set_err("stage or data span out of range");
        if (j.out_first >= 0) {
            if (j.out_first % MODES_BUFFER_SAMPLES || j.hist0 < 0 || j.hist0 % 16 || j.call0 % 16 || j.call0 < j.hist0 ||
                !inside(j.pad_tail_off, MODES_CARRY_BYTES, out_bytes, 2))
                return set_err("resampling job out of range");
            if (j.call0 > j.hist0 && !inside(j.hist_off, j.call0 - j.hist0, hist_bytes, 16)) return set_err("history span out of range");
        }
    }
    Buffers mem;
    Arrays d;
    if (upload(mem, d, hist, hist_bytes, stage, stage_bytes, out, out_bytes)) return -1;
    std::vector<PoolResampleJob> dj(n_jobs);
    for (uint32_t i = 0; i < n_jobs; i++) {
        const ShimResampleJob &j = jobs[i];
        dj[i] = PoolResampleJob{j.hist_off >= 0 ? d.hist + j.hist_off : nullptr, d.stage + j.stage_off, j.hist0, j.call0, j.out_first,
                                j.out_first >= 0 ? d.out + j.pad_tail_off : nullptr, d.out + j.data_off};
    }
    PoolResampleJob *d_jobs = nullptr;
    if (run(mem, dj, &d_jobs)) return -1;
    launch_resample_pool(d_jobs, n_jobs, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(out, d.out, out_bytes, cudaMemcpyDeviceToHost));
    return 0;
}

// One history step: the stream bytes [keep, call0 + MODES_BUFFER_BYTES) to out + out_off.
struct ShimHistoryJob {
    int64_t hist_off, stage_off, hist0, call0, keep, out_off;
};

int rpool_history(const uint8_t *hist, size_t hist_bytes, const uint8_t *stage, size_t stage_bytes, uint8_t *out,
                  size_t out_bytes, const ShimHistoryJob *jobs, uint32_t n_jobs) {
    if (!n_jobs || n_jobs > 4096 || !jobs || !out) return set_err("empty request");
    uint64_t most = 0;
    for (uint32_t i = 0; i < n_jobs; i++) {
        const ShimHistoryJob &j = jobs[i];
        const int64_t end = j.call0 + MODES_BUFFER_BYTES;
        if (j.hist0 < 0 || j.hist0 % 16 || j.call0 % 16 || j.keep % 16 || j.keep < j.hist0 || j.call0 < j.hist0 || j.keep > end)
            return set_err("history job out of range");
        if (!inside(j.stage_off, MODES_BUFFER_BYTES, stage_bytes, 16) || !inside(j.out_off, end - j.keep, out_bytes, 16))
            return set_err("stage or output span out of range");
        if (j.call0 > j.keep && !inside(j.hist_off, j.call0 - j.hist0, hist_bytes, 16)) return set_err("history span out of range");
        if ((uint64_t)(end - j.keep) > most) most = (uint64_t)(end - j.keep);
    }
    Buffers mem;
    Arrays d;
    if (upload(mem, d, hist, hist_bytes, stage, stage_bytes, out, out_bytes)) return -1;
    std::vector<PoolHistoryJob> dj(n_jobs);
    for (uint32_t i = 0; i < n_jobs; i++) {
        const ShimHistoryJob &j = jobs[i];
        dj[i] = PoolHistoryJob{j.hist_off >= 0 ? d.hist + j.hist_off : nullptr, d.stage + j.stage_off, j.hist0, j.call0, j.keep,
                               d.out + j.out_off};
    }
    PoolHistoryJob *d_jobs = nullptr;
    if (run(mem, dj, &d_jobs)) return -1;
    launch_history_pool(d_jobs, n_jobs, most, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(out, d.out, out_bytes, cudaMemcpyDeviceToHost));
    return 0;
}

}  // extern "C"
