// TEST INFRASTRUCTURE — not part of the product.
// Device harness for the 16-bit input launches (launch_convert_sc16: K10 at 2 MHz; launch_resample_sc16:
// K9's int16 loader at 2.4 MS/s; modes_resample.cu), so that tests/test_input_format.py can check them
// byte for byte on spans it chooses, and scripts/input_format_time.py can time them.  It is linked
// against the product's own object (build/modes_resample.o), exactly what libmodes_b200.so ships.
//
// input_run uploads the span, fills the body and the carry block with a sentinel, runs the one launch,
// synchronises and downloads both whole, so a test also sees every byte the launch must leave alone.
// Every argument is checked on the host first; a bad request returns an error and runs nothing.
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

void launch(const ResampleJob &j, int rate24, int shift) {
    if (rate24) launch_resample_sc16(j, shift, 0);
    else launch_convert_sc16(j, shift, 0);
}

}  // namespace

extern "C" {

const char *input_error() { return g_err; }

// Output samples [out_first, out_first + out_samples) of a 16-bit stream into body (2 out_samples bytes)
// and, with want_halo, the carry block before them into halo (kHaloAlloc bytes), from the span in
// (in_bytes bytes from input sample in_first).  rate24: K9 (2.4 MS/s), else K10 (2 MHz; in_first a
// multiple of 4).  out_first a multiple of 8, out_samples of 8.
int input_run(const uint8_t *in, size_t in_bytes, int64_t in_first, int64_t out_first, uint64_t out_samples, int64_t out_end,
              int want_halo, int rate24, int shift, uint8_t *body, uint8_t *halo) {
    if (shift < 0 || shift > 15) return set_err("shift out of range");
    if (!body || !out_samples || out_samples % 8 || out_first % 8 || out_samples > (1ull << 31)) return set_err("output out of range");
    if (want_halo && !halo) return set_err("no carry block");
    if (!rate24 && in_first % 4) return set_err("K10 span must start at a multiple of 4 samples");
    if (in_bytes && !in) return set_err("no input");
    Buffers mem;
    uint8_t *d_in = nullptr, *d_body = nullptr, *d_halo = nullptr;
    HCK(mem.alloc(&d_in, in_bytes + 16));
    HCK(mem.alloc(&d_body, 2 * out_samples));
    HCK(mem.alloc(&d_halo, kHaloAlloc));
    if (in_bytes) HCK(cudaMemcpy(d_in, in, in_bytes, cudaMemcpyHostToDevice));
    HCK(cudaMemset(d_in + in_bytes, 0xa5, 16));           // past the span: must not be read as input
    HCK(cudaMemset(d_body, 0x5a, 2 * out_samples));
    HCK(cudaMemset(d_halo, 0x5a, kHaloAlloc));
    launch(ResampleJob{d_in, in_bytes, in_first, out_first, out_samples, out_end, d_body, want_halo ? d_halo : nullptr}, rate24, shift);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(body, d_body, 2 * out_samples, cudaMemcpyDeviceToHost));
    if (halo) HCK(cudaMemcpy(halo, d_halo, kHaloAlloc, cudaMemcpyDeviceToHost));
    return 0;
}

// Device time of reps launches over out_samples output samples (from buffer 0, with the carry block)
// from the int16 input they read (filled with a pattern), one pair of CUDA events around each: ms[k].
// floor_bytes: the bytes a launch must move (the input it reads and the output it writes).
int input_time(int rate24, int shift, uint64_t out_samples, int reps, float *ms, uint64_t *floor_bytes) {
    if (reps < 1 || !ms || !out_samples || out_samples % MODES_BUFFER_SAMPLES) return set_err("bad timing request");
    const uint64_t n_in = rate24 ? (6 * out_samples + 4) / 5 + 8 : out_samples;
    Buffers mem;
    uint8_t *d_in = nullptr, *d_body = nullptr, *d_halo = nullptr;
    HCK(mem.alloc(&d_in, 4 * n_in + 16));
    HCK(mem.alloc(&d_body, 2 * out_samples));
    HCK(mem.alloc(&d_halo, kHaloAlloc));
    HCK(cudaMemset(d_in, 0x35, 4 * n_in + 16));
    const ResampleJob j{d_in, 4 * n_in, 0, 0, out_samples, INT64_MAX, d_body, d_halo};
    cudaEvent_t a, b;
    HCK(cudaEventCreate(&a));
    HCK(cudaEventCreate(&b));
    for (int k = -2; k < reps; k++) {                      // two launches of warm-up
        HCK(cudaEventRecord(a, 0));
        launch(j, rate24, shift);
        HCK(cudaEventRecord(b, 0));
        HCK(cudaEventSynchronize(b));
        if (k >= 0) HCK(cudaEventElapsedTime(&ms[k], a, b));
    }
    HCK(cudaGetLastError());
    cudaEventDestroy(a);
    cudaEventDestroy(b);
    if (floor_bytes) *floor_bytes = 4 * n_in + 2 * out_samples;
    return 0;
}

// Device time of reps device-to-device copies of `bytes` bytes: ms[k].
int input_copy_time(uint64_t bytes, int reps, float *ms) {
    if (reps < 1 || !ms || !bytes) return set_err("bad timing request");
    Buffers mem;
    uint8_t *src = nullptr, *dst = nullptr;
    HCK(mem.alloc(&src, bytes));
    HCK(mem.alloc(&dst, bytes));
    HCK(cudaMemset(src, 0x35, bytes));
    cudaEvent_t a, b;
    HCK(cudaEventCreate(&a));
    HCK(cudaEventCreate(&b));
    for (int k = -2; k < reps; k++) {
        HCK(cudaEventRecord(a, 0));
        HCK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, 0));
        HCK(cudaEventRecord(b, 0));
        HCK(cudaEventSynchronize(b));
        if (k >= 0) HCK(cudaEventElapsedTime(&ms[k], a, b));
    }
    cudaEventDestroy(a);
    cudaEventDestroy(b);
    return 0;
}

}  // extern "C"
