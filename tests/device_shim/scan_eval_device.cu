// TEST INFRASTRUCTURE — not part of the product.
// Device harness for the preamble scan (K1, modes_scan2.cu), frame evaluation (K2, modes_eval_fused.cu
// and modes_kernels.cu) and the weak-preamble scan (modes_weak.cu), so that tests/test_persistent_kernels.py
// can run them with a chosen SM count.  The launchers size their persistent grids from sm_count, so a
// small sm_count puts every warp through many tiles and chunks with the kernels' machine code
// unchanged: it is linked against the product's own objects (build/*.o), exactly what
// libmodes_b200.so ships.  The harness uploads one batch (body + carry block, laid out as submit()
// lays it out), zeroes the four counters, calls the internal launchers of modes_internal.h and
// synchronises.  The frame-evaluation variant is the one MODES_EVAL_VARIANT selects (read per launch).
//
// Every request is validated on the host before anything is launched: 1 <= sm_count <= the device's
// SM count, each window (virtual samples v - 2 .. v + 240 of a position v) lies inside the batch's
// virtual sample array [0, 240 + N) and no capacity exceeds its array.  An invalid request returns
// an error and runs nothing.
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
    uint16_t *lutn = nullptr, *lut_iq = nullptr;
    uint32_t *bit_syn = nullptr, *fix_hash = nullptr, *pair_hash = nullptr;
    int sm_count = 0, max_blocks_per_sm = 0;
    bool ok = false;
    DeviceTables view() const { return DeviceTables{lutn, lut_iq, bit_syn, fix_hash, pair_hash}; }
};

template <class T> bool upload(T **dst, const T *src, size_t count) {
    return cudaMalloc(dst, sizeof(T) * count) == cudaSuccess &&
           cudaMemcpy(*dst, src, sizeof(T) * count, cudaMemcpyHostToDevice) == cudaSuccess;
}

// The full DeviceTables, built by the product's own builders (modes_tables.cpp), as the context builds them.
Tables &tables() {
    static Tables t = [] {
        Tables r;
        std::vector<uint16_t> lutn(kNLutEntries), lut_iq(kLutIqEntries);
        std::vector<uint32_t> fix(kFixHashSlots), pair(kPairHashSlots);
        uint32_t syn[112];
        build_lutn(lutn.data());
        build_lut_iq(lut_iq.data());
        build_bit_syndromes(syn);
        if (!build_fix_hash(syn, fix.data()) || !build_pair_hash(syn, pair.data())) return r;
        int dev = 0;
        cudaDeviceProp prop;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return r;
        r.sm_count = prop.multiProcessorCount;
        r.max_blocks_per_sm = prop.maxBlocksPerMultiProcessor;
        if (!upload(&r.lutn, lutn.data(), lutn.size()) || !upload(&r.lut_iq, lut_iq.data(), lut_iq.size()) ||
            !upload(&r.bit_syn, syn, 112) || !upload(&r.fix_hash, fix.data(), fix.size()) ||
            !upload(&r.pair_hash, pair.data(), pair.size()))
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

int check_common(const uint8_t *body, uint32_t n_buffers, int sm_count) {
    Tables &T = tables();
    if (!T.ok) return set_err("device tables");
    if (!body) return set_err("empty request");
    if (n_buffers == 0 || n_buffers > 8192) return set_err("n_buffers out of range");
    if (sm_count < 1 || sm_count > T.sm_count) return set_err("sm_count out of range");
    return 0;
}

// Body, carry block and counters of one batch on the device; counters[0] = counter, the rest 0.
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

}  // namespace

extern "C" const char *dev_error() { return g_err; }

// out[0]: the device's SM count; out[1]: the most CTAs an SM holds at once (bounds a persistent grid).
extern "C" int dev_limits(int *out) {
    g_err[0] = 0;
    Tables &T = tables();
    if (!T.ok) return set_err("device tables");
    out[0] = T.sm_count;
    out[1] = T.max_blocks_per_sm;
    return 0;
}

// K1 over one batch: cand_v_out[capacity] (filled with 0xFFFFFFFF before the launch), tiles_out
// [tiles_for(N)] (filled with 0xFF bytes), counters_out[4] as the kernel left them.
extern "C" int dev_scan(const uint8_t *body, uint32_t n_buffers, const uint8_t *carry476, int sm_count, uint32_t capacity,
                        uint32_t *cand_v_out, modes_tile *tiles_out, uint32_t *counters_out) {
    g_err[0] = 0;
    if (check_common(body, n_buffers, sm_count)) return -1;
    if (!cand_v_out || !tiles_out || !counters_out || capacity == 0) return set_err("empty request");
    Tables &T = tables();
    Buffers mem;
    BatchView in{};
    uint32_t *d_counters = nullptr;
    if (upload_batch(mem, body, n_buffers, carry476, 0, in, &d_counters)) return -1;
    const uint32_t n_tiles = tiles_for(in.n_samples);
    uint32_t *d_cand = nullptr;
    modes_tile *d_tiles = nullptr;
    HCK(mem.alloc(&d_cand, (size_t)capacity * sizeof(uint32_t)));
    HCK(mem.alloc(&d_tiles, (size_t)n_tiles * sizeof(modes_tile)));
    HCK(cudaMemset(d_cand, 0xFF, (size_t)capacity * sizeof(uint32_t)));
    HCK(cudaMemset(d_tiles, 0xFF, (size_t)n_tiles * sizeof(modes_tile)));
    const ScanOutputs so{d_cand, capacity, d_tiles, d_counters};
    launch_scan(in, T.view(), so, sm_count, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(cand_v_out, d_cand, (size_t)capacity * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    HCK(cudaMemcpy(tiles_out, d_tiles, (size_t)n_tiles * sizeof(modes_tile), cudaMemcpyDeviceToHost));
    HCK(cudaMemcpy(counters_out, d_counters, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return 0;
}

// K2 over the n positions v[] (the candidate array, n entries) with counters[0] = counter and record
// capacity `capacity` (<= n): records_out[n], filled with 0x5A bytes before the launch.
extern "C" int dev_eval(const uint8_t *body, uint32_t n_buffers, const uint8_t *carry476, const uint32_t *v, uint32_t n,
                        uint32_t capacity, uint32_t counter, int fix, int aggressive, int sm_count, modes_candidate *records_out) {
    g_err[0] = 0;
    if (check_common(body, n_buffers, sm_count)) return -1;
    if (!v || !records_out || n == 0) return set_err("empty request");
    if (capacity > n) return set_err("capacity exceeds the candidate and record arrays");
    const uint64_t n_samples = (uint64_t)n_buffers * kBufSamples;
    for (uint32_t k = 0; k < n; k++)
        if (v[k] < 2 || (uint64_t)v[k] >= n_samples) {
            snprintf(g_err, sizeof(g_err), "position %u: window of v = %u outside [0, %llu)", k, v[k],
                     (unsigned long long)(n_samples + kHaloSamples));
            return -1;
        }
    Tables &T = tables();
    Buffers mem;
    BatchView in{};
    uint32_t *d_counters = nullptr;
    if (upload_batch(mem, body, n_buffers, carry476, counter, in, &d_counters)) return -1;
    uint32_t *d_cand = nullptr;
    modes_candidate *d_rec = nullptr;
    HCK(mem.alloc(&d_cand, (size_t)n * sizeof(uint32_t)));
    HCK(mem.alloc(&d_rec, (size_t)n * sizeof(modes_candidate)));
    HCK(cudaMemcpy(d_cand, v, (size_t)n * sizeof(uint32_t), cudaMemcpyHostToDevice));
    HCK(cudaMemset(d_rec, 0x5A, (size_t)n * sizeof(modes_candidate)));
    const ScanOutputs so{d_cand, capacity, nullptr, d_counters};
    launch_eval(in, T.view(), so, d_rec, fix, aggressive, sm_count, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(records_out, d_rec, (size_t)n * sizeof(modes_candidate), cudaMemcpyDeviceToHost));
    return 0;
}

// The weak-preamble scan of the buffers first_buffer + i * buffer_step (< n_buffers) of one batch:
// pos_out[capacity] (filled with 0xFFFFFFFF before the launch), *count_out = the exact count.
extern "C" int dev_weak(const uint8_t *body, uint32_t n_buffers, const uint8_t *carry476, uint32_t first_buffer,
                        uint32_t buffer_step, int sm_count, uint32_t capacity, uint32_t scratch_cap, uint32_t *pos_out,
                        uint32_t *count_out) {
    g_err[0] = 0;
    if (check_common(body, n_buffers, sm_count)) return -1;
    if (!pos_out || !count_out || capacity == 0 || scratch_cap == 0) return set_err("empty request");
    if (buffer_step == 0 || first_buffer >= n_buffers) return set_err("scanned buffers outside the batch");
    const uint32_t n_scan = (n_buffers - first_buffer + buffer_step - 1) / buffer_step;
    Tables &T = tables();
    Buffers mem;
    BatchView in{};
    uint32_t *d_counters = nullptr;
    if (upload_batch(mem, body, n_buffers, carry476, 0, in, &d_counters)) return -1;
    const size_t n_tiles = weak_tiles_for(n_scan);
    uint32_t *d_pos = nullptr, *d_scratch = nullptr, *d_tiles = nullptr;
    HCK(mem.alloc(&d_pos, (size_t)capacity * sizeof(uint32_t)));
    HCK(mem.alloc(&d_scratch, (size_t)scratch_cap * sizeof(uint32_t)));
    HCK(mem.alloc(&d_tiles, 3 * n_tiles * sizeof(uint32_t)));
    HCK(cudaMemset(d_pos, 0xFF, (size_t)capacity * sizeof(uint32_t)));
    const WeakOutputs wo{first_buffer, buffer_step, n_scan, d_pos, capacity, d_scratch, scratch_cap, d_tiles, d_counters};
    launch_weak_scan(in, T.view(), wo, sm_count, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(pos_out, d_pos, (size_t)capacity * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    HCK(cudaMemcpy(count_out, d_counters + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return 0;
}
