// TEST INFRASTRUCTURE — not part of the product.
// Device harness for the receiver pool's gather launch (launch_gather_pool, modes_resample.cu), so that
// tests/test_pool_device_input.py can check it byte for byte on jobs it lays out itself.  It is linked against
// the product's own object (build/modes_resample.o), exactly what libmodes_b200.so ships.
//
// Jobs name offsets into three host arrays, which the harness uploads whole: `in` (the callers' buffers),
// `carry` (the device carries, both halves) and `out` (the batch's pairs).  It runs the one launch,
// synchronises and downloads `carry` and `out` whole, so a test also sees every byte the launch must leave
// alone.  Every offset is checked on the host first; a bad request returns an error and runs nothing.
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

}  // namespace

extern "C" {

const char *gpool_error() { return g_err; }

// One gather job: in_off < 0 for none (out + data_off already holds the buffer), carry_in_off < 0 for none
// (the stream starts).
struct ShimGatherJob {
    int64_t in_off, data_off, carry_in_off, carry_out_off, pad_tail_off;
};

int gpool_gather(const uint8_t *in, size_t in_bytes, uint8_t *carry, size_t carry_bytes, uint8_t *out, size_t out_bytes,
                 const ShimGatherJob *jobs, uint32_t n_jobs) {
    if (!n_jobs || n_jobs > 4096 || !jobs || !carry || !out) return set_err("empty request");
    for (uint32_t i = 0; i < n_jobs; i++) {
        const ShimGatherJob &j = jobs[i];
        if ((j.in_off >= 0 && !inside(j.in_off, MODES_BUFFER_BYTES, in_bytes, 16)) ||
            !inside(j.data_off, MODES_BUFFER_BYTES, out_bytes, 16) || !inside(j.pad_tail_off, MODES_CARRY_BYTES, out_bytes, 4) ||
            (j.carry_in_off >= 0 && !inside(j.carry_in_off, MODES_CARRY_BYTES, carry_bytes, 4)) ||
            !inside(j.carry_out_off, MODES_CARRY_BYTES, carry_bytes, 4) || j.carry_in_off == j.carry_out_off)
            return set_err("gather job out of range");
    }
    Buffers mem;
    uint8_t *d_in = nullptr, *d_carry = nullptr, *d_out = nullptr;
    PoolGatherJob *d_jobs = nullptr;
    HCK(mem.alloc(&d_in, in_bytes));
    HCK(mem.alloc(&d_carry, carry_bytes));
    HCK(mem.alloc(&d_out, out_bytes));
    HCK(mem.alloc(&d_jobs, n_jobs * sizeof(PoolGatherJob)));
    if (in_bytes) HCK(cudaMemcpy(d_in, in, in_bytes, cudaMemcpyHostToDevice));
    HCK(cudaMemcpy(d_carry, carry, carry_bytes, cudaMemcpyHostToDevice));
    HCK(cudaMemcpy(d_out, out, out_bytes, cudaMemcpyHostToDevice));
    std::vector<PoolGatherJob> dj(n_jobs);
    for (uint32_t i = 0; i < n_jobs; i++) {
        const ShimGatherJob &j = jobs[i];
        dj[i] = PoolGatherJob{j.in_off >= 0 ? d_in + j.in_off : nullptr, d_out + j.data_off,
                              j.carry_in_off >= 0 ? d_carry + j.carry_in_off : nullptr, d_carry + j.carry_out_off,
                              d_out + j.pad_tail_off};
    }
    HCK(cudaMemcpy(d_jobs, dj.data(), n_jobs * sizeof(PoolGatherJob), cudaMemcpyHostToDevice));
    launch_gather_pool(d_jobs, n_jobs, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(carry, d_carry, carry_bytes, cudaMemcpyDeviceToHost));
    HCK(cudaMemcpy(out, d_out, out_bytes, cudaMemcpyDeviceToHost));
    return 0;
}

}  // extern "C"
