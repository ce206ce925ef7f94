// TEST INFRASTRUCTURE — not part of the product.
// Device harness for the carrier measurement of the signal pass (modes_signal.cu), so that the GPU test
// suite (tests/test_carrier.py) can run constructed corpora through the shipped kernel with any of the three
// switches set.  It is linked against the product's own objects (build/modes_signal.o, modes_tables.o): the
// machine code under test is exactly what libmodes_b200.so ships.  It uploads one batch (body + carry block,
// laid out as submit() lays it out), takes fabricated candidate records and a carrier array (which the test
// fills with a sentinel, so that every entry the pass must not write can be checked), sets the candidate
// count, calls launch_signal and synchronises.  It compiles no device code of its own.
//
// Every request is validated on the host before anything is launched: the pass reads window samples
// 0 .. 16+2*112 of a record, so each v = t+2 .. t+242 must lie inside the batch's virtual sample array
// [0, 240 + N), and the capacity never exceeds the record array.  An invalid request returns an error and
// runs nothing.
#include <cstdint>
#include <cstdio>
#include <cstring>
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

struct Tables {
    uint16_t *lutn = nullptr;
    int sm_count = 0;
    bool ok = false;
};

Tables &tables() {
    static Tables t = [] {
        Tables r;
        std::vector<uint16_t> lutn(kNLutEntries);
        build_lutn(lutn.data());
        int dev = 0;
        cudaDeviceProp prop;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return r;
        r.sm_count = prop.multiProcessorCount;
        if (cudaMalloc(&r.lutn, sizeof(uint16_t) * kNLutEntries) != cudaSuccess ||
            cudaMemcpy(r.lutn, lutn.data(), sizeof(uint16_t) * kNLutEntries, cudaMemcpyHostToDevice) != cudaSuccess)
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

}  // namespace

extern "C" const char *car_error() { return g_err; }

extern "C" int car_sm_count() {
    Tables &T = tables();
    return T.ok ? T.sm_count : -1;
}

// The signal pass with the switches (signal, arrival, carrier) over n whole candidate records and n carrier
// records (both in place), counters[0] = counter (may exceed the capacity), record capacity `capacity`.
extern "C" int car_signal_pass(const uint8_t *body, uint32_t n_buffers, const uint8_t *carry476, uint8_t *records,
                               uint8_t *carrier, uint32_t n, uint32_t capacity, uint32_t counter, int signal, int arrival,
                               int measure_carrier) {
    g_err[0] = 0;
    Tables &T = tables();
    if (!T.ok) return set_err("device tables");
    if (!body || !records || !carrier || n == 0) return set_err("empty request");
    if (capacity > n) return set_err("capacity exceeds the record array");
    if (n_buffers == 0 || n_buffers > 4096) return set_err("n_buffers out of range");
    const int64_t limit = (int64_t)kHaloSamples + (int64_t)n_buffers * kBufSamples;
    for (uint32_t k = 0; k < n; k++) {
        int64_t tk;
        std::memcpy(&tk, records + (size_t)k * sizeof(modes_candidate), sizeof(tk));
        if (tk < 0 || tk + 242 >= limit) {
            snprintf(g_err, sizeof(g_err), "record %u: window of t = %lld outside [0, %lld)", k, (long long)tk, (long long)limit);
            return -1;
        }
    }
    Buffers mem;
    const size_t body_bytes = (size_t)n_buffers * MODES_BUFFER_BYTES;
    uint8_t *d_body = nullptr, *d_halo = nullptr;
    uint32_t *d_counters = nullptr;
    modes_candidate *d_recs = nullptr;
    modes_carrier *d_car = nullptr;
    HCK(mem.alloc(&d_body, body_bytes));
    HCK(mem.alloc(&d_halo, kHaloAlloc));
    HCK(mem.alloc(&d_counters, 4 * sizeof(uint32_t)));
    HCK(mem.alloc(&d_recs, n * sizeof(modes_candidate)));
    HCK(mem.alloc(&d_car, n * sizeof(modes_carrier)));
    uint8_t halo[kHaloAlloc];
    std::memset(halo, 127, sizeof(halo));
    if (carry476) std::memcpy(halo + (kHaloBytes - MODES_CARRY_BYTES), carry476, MODES_CARRY_BYTES);
    const uint32_t counters[4] = {counter, 0, 0, 0};
    HCK(cudaMemcpy(d_body, body, body_bytes, cudaMemcpyHostToDevice));
    HCK(cudaMemcpy(d_halo, halo, sizeof(halo), cudaMemcpyHostToDevice));
    HCK(cudaMemcpy(d_counters, counters, sizeof(counters), cudaMemcpyHostToDevice));
    HCK(cudaMemcpy(d_recs, records, n * sizeof(modes_candidate), cudaMemcpyHostToDevice));
    HCK(cudaMemcpy(d_car, carrier, n * sizeof(modes_carrier), cudaMemcpyHostToDevice));
    const BatchView in{d_body, d_halo, (uint64_t)n_buffers * kBufSamples};
    const DeviceTables tab{T.lutn, nullptr, nullptr, nullptr, nullptr};
    const ScanOutputs so{nullptr, capacity, nullptr, d_counters};
    launch_signal(in, tab, so, d_recs, T.sm_count, 0, signal != 0, arrival != 0, measure_carrier ? d_car : nullptr);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(records, d_recs, n * sizeof(modes_candidate), cudaMemcpyDeviceToHost));
    HCK(cudaMemcpy(carrier, d_car, n * sizeof(modes_carrier), cudaMemcpyDeviceToHost));
    return 0;
}
