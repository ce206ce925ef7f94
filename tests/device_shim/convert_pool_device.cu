// TEST INFRASTRUCTURE — not part of the product.
// Device harness for the receiver pool's conversion launch (launch_convert_pool, modes_resample.cu), so
// that tests/test_pool_input_format.py can check it byte for byte on jobs it lays out itself.  It is linked
// against the product's own object (build/modes_resample.o), exactly what libmodes_b200.so ships.
//
// Jobs name offsets into two host arrays, which the harness uploads whole: `in` (the call's 16-bit buffers)
// and `out` (the destinations, with whatever lies between them).  It runs the one launch, synchronises and
// downloads `out` whole, so a test also sees every byte the launch must leave alone.  Every offset and
// shift is checked on the host first; a bad request returns an error and runs nothing.
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

// [off, off + len) inside an array of n bytes, off a multiple of 16.
bool inside(int64_t off, int64_t len, size_t n) {
    return off >= 0 && len >= 0 && off % 16 == 0 && (uint64_t)(off + len) <= n;
}

}  // namespace

extern "C" {

const char *cpool_error() { return g_err; }

// One conversion job: the 2 x MODES_BUFFER_BYTES int16 bytes at in + in_off to the MODES_BUFFER_BYTES
// bytes at out + out_off with its shift.
struct ShimConvertJob {
    int64_t in_off, out_off, shift;
};

int cpool_convert(const uint8_t *in, size_t in_bytes, uint8_t *out, size_t out_bytes, const ShimConvertJob *jobs,
                  uint32_t n_jobs) {
    if (!n_jobs || n_jobs > 4096 || !jobs || !in || !out) return set_err("empty request");
    for (uint32_t i = 0; i < n_jobs; i++) {
        const ShimConvertJob &j = jobs[i];
        if (!inside(j.in_off, 2 * MODES_BUFFER_BYTES, in_bytes) || !inside(j.out_off, MODES_BUFFER_BYTES, out_bytes) ||
            j.shift < 0 || j.shift > 15)
            return set_err("conversion job out of range");
    }
    Buffers mem;
    uint8_t *d_in = nullptr, *d_out = nullptr;
    PoolConvertJob *d_jobs = nullptr;
    HCK(mem.alloc(&d_in, in_bytes));
    HCK(mem.alloc(&d_out, out_bytes));
    HCK(mem.alloc(&d_jobs, n_jobs * sizeof(PoolConvertJob)));
    HCK(cudaMemcpy(d_in, in, in_bytes, cudaMemcpyHostToDevice));
    HCK(cudaMemcpy(d_out, out, out_bytes, cudaMemcpyHostToDevice));
    std::vector<PoolConvertJob> dj(n_jobs);
    for (uint32_t i = 0; i < n_jobs; i++)
        dj[i] = PoolConvertJob{d_in + jobs[i].in_off, d_out + jobs[i].out_off, (int32_t)jobs[i].shift};
    HCK(cudaMemcpy(d_jobs, dj.data(), n_jobs * sizeof(PoolConvertJob), cudaMemcpyHostToDevice));
    launch_convert_pool(d_jobs, n_jobs, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(out, d_out, out_bytes, cudaMemcpyDeviceToHost));
    return 0;
}

}  // extern "C"
