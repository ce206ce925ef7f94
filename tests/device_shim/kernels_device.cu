// TEST INFRASTRUCTURE — not part of the product.
// Device harness for the recovery (modes_recover.cu) and signal (modes_signal.cu) passes, so that the
// GPU test suite (tests/test_kernel_edges.py) can run the constructed corpora of the host-shim tests
// through the shipped kernels.  It is linked against the product's own objects (build/*.o): the
// machine code under test is exactly what libmodes_b200.so ships.  The harness uploads one batch
// (body + carry block, laid out as submit() lays it out), fabricates the candidate records, sets the
// candidate count, calls the internal launchers of modes_internal.h and synchronises.
//
// The only device code compiled here is the two exhaustive sweeps of dev_sweeps(): the device build of
// modes_signal_core.cuh / modes_levels_core.cuh (the __CUDA_ARCH__ branches, which the host shims never
// compile) over all 2^32 inputs, each checked against a scalar restatement.
//
// Every request is validated on the host before anything is launched: each window v = t+18 .. t+18+223
// lies inside the batch's virtual sample array [0, 240 + N) and the capacity never exceeds the arrays.
// An invalid request returns an error and runs nothing.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>
#include <cuda_runtime.h>
#include "modes_internal.h"
#include "modes_levels_core.cuh"
#include "modes_signal_core.cuh"

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

struct Tables {
    uint16_t *lutn = nullptr;
    uint32_t *bit_syn = nullptr;
    int sm_count = 0;
    bool ok = false;
};

Tables &tables() {
    static Tables t = [] {
        Tables r;
        std::vector<uint16_t> lutn(kNLutEntries);
        uint32_t syn[112];
        build_lutn(lutn.data());
        build_bit_syndromes(syn);
        int dev = 0;
        cudaDeviceProp prop;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return r;
        r.sm_count = prop.multiProcessorCount;
        if (cudaMalloc(&r.lutn, sizeof(uint16_t) * kNLutEntries) != cudaSuccess ||
            cudaMalloc(&r.bit_syn, sizeof(syn)) != cudaSuccess ||
            cudaMemcpy(r.lutn, lutn.data(), sizeof(uint16_t) * kNLutEntries, cudaMemcpyHostToDevice) != cudaSuccess ||
            cudaMemcpy(r.bit_syn, syn, sizeof(syn), cudaMemcpyHostToDevice) != cudaSuccess)
            return r;
        r.ok = true;
        return r;
    }();
    return t;
}

// Device memory freed on every return path.
struct Buffers {
    std::vector<void *> p;
    template <class T> cudaError_t alloc(T **out, size_t bytes) {
        void *q = nullptr;
        const cudaError_t e = cudaMalloc(&q, bytes);
        if (e == cudaSuccess) p.push_back(q);
        *out = static_cast<T *>(q);
        return e;
    }
    ~Buffers() { for (void *q : p) cudaFree(q); }
};

// The windows of records at t[0..n) must lie inside the virtual array of n_buffers buffers.
int check_windows(uint32_t n_buffers, const int64_t *t, size_t stride, uint32_t n) {
    if (n_buffers == 0 || n_buffers > 4096) return set_err("n_buffers out of range");
    const int64_t limit = (int64_t)kHaloSamples + (int64_t)n_buffers * kBufSamples;
    for (uint32_t k = 0; k < n; k++) {
        int64_t tk;
        std::memcpy(&tk, reinterpret_cast<const uint8_t *>(t) + k * stride, sizeof(tk));
        if (tk < 0 || tk + 18 + 223 >= limit) {
            snprintf(g_err, sizeof(g_err), "record %u: window of t = %lld outside [0, %lld)", k, (long long)tk, (long long)limit);
            return -1;
        }
    }
    return 0;
}

// Body, carry block and counters of one batch on the device; counters[0] = counter.
int upload_batch(Buffers &mem, const uint8_t *body, uint32_t n_buffers, const uint8_t *carry476, uint32_t counter,
                 BatchView &in, uint32_t **d_counters) {
    const size_t body_bytes = (size_t)n_buffers * MODES_BUFFER_BYTES;
    uint8_t *d_body = nullptr, *d_halo = nullptr;
    HCK(mem.alloc(&d_body, body_bytes));
    HCK(mem.alloc(&d_halo, kHaloAlloc));
    HCK(mem.alloc(d_counters, 4 * sizeof(uint32_t)));
    uint8_t halo[kHaloAlloc];
    std::memset(halo, 127, sizeof(halo));
    if (carry476) std::memcpy(halo + (kHaloBytes - MODES_CARRY_BYTES), carry476, MODES_CARRY_BYTES);
    const uint32_t counters[4] = {counter, 0, 0, 0};
    HCK(cudaMemcpy(d_body, body, body_bytes, cudaMemcpyHostToDevice));
    HCK(cudaMemcpy(d_halo, halo, sizeof(halo), cudaMemcpyHostToDevice));
    HCK(cudaMemcpy(*d_counters, counters, sizeof(counters), cudaMemcpyHostToDevice));
    in = BatchView{d_body, d_halo, (uint64_t)n_buffers * kBufSamples};
    return 0;
}

constexpr unsigned long long kNone = ~0ull;

// isqrt32(x) for every 32-bit x: r^2 <= x < (r + 1)^2 in 64-bit integers.
__global__ void isqrt_sweep(unsigned long long *res) {
    const uint64_t step = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < (1ull << 32); x += step) {
        const uint64_t r = signal::isqrt32((uint32_t)x);
        if (!(r * r <= x && (r + 1) * (r + 1) > x)) {
            atomicAdd(&res[0], 1ull);
            atomicMin(&res[1], (unsigned long long)x);
        }
    }
}

__device__ bool rail(uint32_t b) { return b == 0 || b == 255; }

// Every word I0 Q0 I1 Q1 through signal::pair_mags / pulse_sq and levels::add_word / clipped_in, against
// a per-sample restatement: lutn[(I-127)^2 + (Q-127)^2], and I or Q at 0 or 255.
__global__ void word_sweep(const uint16_t *lutn, unsigned long long *res) {
    const uint64_t step = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < (1ull << 32); x += step) {
        const uint32_t w = (uint32_t)x;
        uint32_t m[2], clip = 0, near = 0;
        for (int s = 0; s < 2; s++) {
            const int i = (int)((w >> (16 * s)) & 0xff), q = (int)((w >> (16 * s + 8)) & 0xff);
            m[s] = lutn[(i - 127) * (i - 127) + (q - 127) * (q - 127)];
            clip += (rail(i) || rail(q)) ? 1u : 0u;
            near += (i == 0 || i >= 254 || q == 0 || q >= 254) ? 1u : 0u;   // |b - 127| >= 127
        }
        uint32_t first, second;
        signal::pair_mags(w, lutn, first, second);
        const uint32_t top = m[0] > m[1] ? m[0] : m[1];
        levels::Acc a;
        levels::acc_clear(a);
        const uint32_t maybe = levels::add_word(a, w, lutn);
        const bool ok = first == m[0] && second == m[1] && signal::pulse_sq(w, lutn) == top * top &&
                        a.sum_mag == m[0] + m[1] && a.sum_power == (uint64_t)m[0] * m[0] + (uint64_t)m[1] * m[1] &&
                        a.peak == top && a.clipped == 0 && (maybe != 0) == (near != 0) && levels::clipped_in(w) == clip;
        if (!ok) {
            atomicAdd(&res[0], 1ull);
            atomicMin(&res[1], (unsigned long long)x);
        }
    }
}

}  // namespace

extern "C" const char *dev_error() { return g_err; }

extern "C" int dev_sm_count() {
    Tables &T = tables();
    return T.ok ? T.sm_count : -1;
}

// Recovery records of n fabricated candidates (only t meaningful, every other byte 0xA5) into out
// (n records, filled with 0x5A before the launch), with counters[0] = counter (may exceed capacity).
extern "C" int dev_recover(const uint8_t *body, uint32_t n_buffers, const uint8_t *carry476, const int64_t *t, uint32_t n,
                           uint32_t capacity, uint32_t counter, uint8_t *out) {
    g_err[0] = 0;
    Tables &T = tables();
    if (!T.ok) return set_err("device tables");
    if (!body || !t || !out || n == 0) return set_err("empty request");
    if (capacity > n) return set_err("capacity exceeds the record arrays");
    if (check_windows(n_buffers, t, sizeof(int64_t), n)) return -1;
    std::vector<modes_candidate> recs(n);
    std::memset(recs.data(), 0xA5, n * sizeof(modes_candidate));
    for (uint32_t k = 0; k < n; k++) recs[k].t = t[k];
    Buffers mem;
    BatchView in{};
    uint32_t *d_counters = nullptr;
    if (upload_batch(mem, body, n_buffers, carry476, counter, in, &d_counters)) return -1;
    modes_candidate *d_recs = nullptr;
    modes_recovered *d_out = nullptr;
    HCK(mem.alloc(&d_recs, n * sizeof(modes_candidate)));
    HCK(mem.alloc(&d_out, n * sizeof(modes_recovered)));
    HCK(cudaMemcpy(d_recs, recs.data(), n * sizeof(modes_candidate), cudaMemcpyHostToDevice));
    HCK(cudaMemset(d_out, 0x5A, n * sizeof(modes_recovered)));
    const DeviceTables tab{T.lutn, nullptr, T.bit_syn, nullptr, nullptr};
    const ScanOutputs so{nullptr, capacity, nullptr, d_counters};
    launch_recover(in, tab, so, d_recs, capacity, d_out, T.sm_count, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(out, d_out, n * sizeof(modes_recovered), cudaMemcpyDeviceToHost));
    return 0;
}

// The signal pass over n whole candidate records (in place), counters[0] = counter, record capacity
// `capacity`.
extern "C" int dev_signal(const uint8_t *body, uint32_t n_buffers, const uint8_t *carry476, uint8_t *records, uint32_t n,
                          uint32_t capacity, uint32_t counter) {
    g_err[0] = 0;
    Tables &T = tables();
    if (!T.ok) return set_err("device tables");
    if (!body || !records || n == 0) return set_err("empty request");
    if (capacity > n) return set_err("capacity exceeds the record array");
    if (check_windows(n_buffers, reinterpret_cast<const int64_t *>(records), sizeof(modes_candidate), n)) return -1;
    Buffers mem;
    BatchView in{};
    uint32_t *d_counters = nullptr;
    if (upload_batch(mem, body, n_buffers, carry476, counter, in, &d_counters)) return -1;
    modes_candidate *d_recs = nullptr;
    HCK(mem.alloc(&d_recs, n * sizeof(modes_candidate)));
    HCK(cudaMemcpy(d_recs, records, n * sizeof(modes_candidate), cudaMemcpyHostToDevice));
    const DeviceTables tab{T.lutn, nullptr, nullptr, nullptr, nullptr};
    const ScanOutputs so{nullptr, capacity, nullptr, d_counters};
    launch_signal(in, tab, so, d_recs, T.sm_count, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(records, d_recs, n * sizeof(modes_candidate), cudaMemcpyDeviceToHost));
    return 0;
}

// out[0], out[1]: mismatches and first failing x of the isqrt32 sweep; out[2], out[3]: the same for
// the word sweep (first = 2^64 - 1 when none).
extern "C" int dev_sweeps(unsigned long long *out) {
    g_err[0] = 0;
    Tables &T = tables();
    if (!T.ok) return set_err("device tables");
    Buffers mem;
    unsigned long long *d_res = nullptr;
    HCK(mem.alloc(&d_res, 4 * sizeof(unsigned long long)));
    const unsigned long long init[4] = {0, kNone, 0, kNone};
    HCK(cudaMemcpy(d_res, init, sizeof(init), cudaMemcpyHostToDevice));
    isqrt_sweep<<<T.sm_count * 8, 256>>>(d_res);
    HCK(cudaGetLastError());
    word_sweep<<<T.sm_count * 8, 256>>>(T.lutn, d_res + 2);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(out, d_res, sizeof(init), cudaMemcpyDeviceToHost));
    return 0;
}
