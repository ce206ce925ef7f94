// TEST INFRASTRUCTURE — not part of the product.
// Device harness for the device resolve (K3, modes_resolve_gpu.cu), so that tests/test_resolve_device.py
// can run it on batches of any size with a chosen SM count and delivery capacity.  The launcher caps its
// replay grid at 4 CTAs of 8 warps per SM, so a small sm_count (or a batch of more than 32 * SM count
// buffers) puts warps through several buffers, and batches of more than 1024 buffers give each thread of
// the offsets kernel several buffers, with the kernels' machine code unchanged: it is linked against the
// product's own object (build/modes_resolve_gpu.o), exactly what libmodes_b200.so ships.
//
// One call uploads a candidate array, its tile array and a starting cache, runs launch_gpu_resolve and
// synchronises.  Every request is validated on the host before anything is launched: 1 <= sm_count <=
// the device's SM count, 1 <= n_buffers <= 65536, n_tiles == tiles_for(n_buffers * 131072), every
// tile's offset + count within the candidate array, capacity <= the delivery allocation, and an
// allocation of at least two deliveries per candidate (the most a batch can make).  An invalid request
// returns an error and runs nothing.  The delivery array is allocated with kGuardRecords more entries
// than that, all filled with kGuardByte before the launch and all copied back, so a write at or past
// the capacity shows up as a changed byte in the returned array, never as a write out of range.
#include <cstdint>
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#include "modes_internal.h"

namespace {
using namespace modes;

constexpr uint32_t kGuardRecords = 256;
constexpr int kGuardByte = 0xA5;
constexpr uint32_t kMaxBuffers = 65536;

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

int device_sm_count() {
    static const int n = [] {
        int dev = 0, v = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
        return v;
    }();
    return n;
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

extern "C" const char *dev_error() { return g_err; }

// out[0]: the device's SM count; out[1]: the guard records after a delivery allocation; out[2]: their byte.
extern "C" int dev_limits(int *out) {
    g_err[0] = 0;
    if (!out) return set_err("empty request");
    if (device_sm_count() < 1) return set_err("no CUDA device");
    out[0] = device_sm_count();
    out[1] = (int)kGuardRecords;
    out[2] = kGuardByte;
    return 0;
}

// launch_gpu_resolve over n_buffers buffers: records[n_records] and tiles[n_tiles] as the scan and frame
// evaluation leave them, the cache at the batch's start cache_in[1024], delivery capacity `capacity` in
// an allocation of alloc + kGuardRecords entries.  Outputs: out[alloc + kGuardRecords] (the whole
// allocation), stats_out[8], flags_out[3], cache_out[1024], n_deliv_out[n_buffers],
// offsets_out[n_buffers + 1] and start_out[n_buffers * 1024] (each buffer's final start cache).  Every
// output but `out` and the offsets is filled with 0xFF bytes on the device before the launch; the offsets
// are zeroed, so that an emit pass behind offsets the offsets kernel left unwritten stays in range.
extern "C" int dev_resolve(const modes_candidate *records, uint64_t n_records, const modes_tile *tiles, uint32_t n_tiles,
                           uint32_t n_buffers, const uint32_t *cache_in, int check_crc, int sm_count, uint32_t capacity,
                           uint32_t alloc, modes_delivery *out, uint64_t *stats_out, uint32_t *flags_out, uint32_t *cache_out,
                           uint32_t *n_deliv_out, uint32_t *offsets_out, uint32_t *start_out) {
    g_err[0] = 0;
    if (!tiles || !cache_in || !out || !stats_out || !flags_out || !cache_out || !n_deliv_out || !offsets_out || !start_out ||
        (n_records && !records))
        return set_err("empty request");
    if (device_sm_count() < 1) return set_err("no CUDA device");
    if (sm_count < 1 || sm_count > device_sm_count()) return set_err("sm_count out of range");
    if (n_buffers < 1 || n_buffers > kMaxBuffers) return set_err("n_buffers out of range");
    if (n_tiles != tiles_for((uint64_t)n_buffers * kBufSamples)) return set_err("n_tiles is not tiles_for(n_buffers * 131072)");
    for (uint32_t i = 0; i < n_tiles; i++)
        if ((uint64_t)tiles[i].offset + tiles[i].count > n_records) {
            snprintf(g_err, sizeof(g_err), "tile %u: records %u + %u outside the %llu candidates", i, tiles[i].offset,
                     tiles[i].count, (unsigned long long)n_records);
            return -1;
        }
    if (capacity > alloc) return set_err("capacity exceeds the delivery allocation");
    if (alloc < 2 * n_records) return set_err("the delivery allocation holds fewer than two deliveries per candidate");

    const size_t nb = n_buffers, n_out = (size_t)alloc + kGuardRecords;
    Buffers mem;
    modes_candidate *d_rec = nullptr;
    modes_tile *d_tiles = nullptr;
    uint32_t *d_start = nullptr, *d_end = nullptr, *d_written = nullptr, *d_readfirst = nullptr, *d_rerun = nullptr,
             *d_n_deliv = nullptr, *d_offsets = nullptr, *d_flags = nullptr, *d_cache_in = nullptr, *d_cache_out = nullptr;
    uint64_t *d_stats = nullptr;
    modes_delivery *d_out = nullptr;
    HCK(mem.alloc(&d_rec, (n_records ? n_records : 1) * sizeof(modes_candidate)));
    HCK(mem.alloc(&d_tiles, (size_t)n_tiles * sizeof(modes_tile)));
    HCK(mem.alloc(&d_start, nb * 1024 * sizeof(uint32_t)));
    HCK(mem.alloc(&d_end, nb * 1024 * sizeof(uint32_t)));
    HCK(mem.alloc(&d_written, nb * 32 * sizeof(uint32_t)));
    HCK(mem.alloc(&d_readfirst, nb * 32 * sizeof(uint32_t)));
    HCK(mem.alloc(&d_rerun, nb * sizeof(uint32_t)));
    HCK(mem.alloc(&d_n_deliv, nb * sizeof(uint32_t)));
    HCK(mem.alloc(&d_offsets, (nb + 1) * sizeof(uint32_t)));
    HCK(mem.alloc(&d_flags, 4 * sizeof(uint32_t)));
    HCK(mem.alloc(&d_cache_in, 1024 * sizeof(uint32_t)));
    HCK(mem.alloc(&d_cache_out, 1024 * sizeof(uint32_t)));
    HCK(mem.alloc(&d_stats, 8 * sizeof(uint64_t)));
    HCK(mem.alloc(&d_out, n_out * sizeof(modes_delivery)));
    if (n_records) HCK(cudaMemcpy(d_rec, records, n_records * sizeof(modes_candidate), cudaMemcpyHostToDevice));
    HCK(cudaMemcpy(d_tiles, tiles, (size_t)n_tiles * sizeof(modes_tile), cudaMemcpyHostToDevice));
    HCK(cudaMemcpy(d_cache_in, cache_in, 1024 * sizeof(uint32_t), cudaMemcpyHostToDevice));
    HCK(cudaMemset(d_out, kGuardByte, n_out * sizeof(modes_delivery)));
    HCK(cudaMemset(d_start, 0xFF, nb * 1024 * sizeof(uint32_t)));
    HCK(cudaMemset(d_n_deliv, 0xFF, nb * sizeof(uint32_t)));
    HCK(cudaMemset(d_offsets, 0, (nb + 1) * sizeof(uint32_t)));
    HCK(cudaMemset(d_flags, 0xFF, 4 * sizeof(uint32_t)));
    HCK(cudaMemset(d_cache_out, 0xFF, 1024 * sizeof(uint32_t)));
    HCK(cudaMemset(d_stats, 0xFF, 8 * sizeof(uint64_t)));
    HCK(cudaDeviceSynchronize());

    const GpuResolve g{d_start, d_end, d_written, d_readfirst, d_rerun, d_n_deliv, d_offsets, d_flags, d_cache_in, d_cache_out,
                       d_stats, d_out, capacity};
    launch_gpu_resolve(g, d_rec, d_tiles, n_tiles, n_buffers, check_crc, sm_count, 0);
    HCK(cudaGetLastError());
    HCK(cudaDeviceSynchronize());

    HCK(cudaMemcpy(out, d_out, n_out * sizeof(modes_delivery), cudaMemcpyDeviceToHost));
    HCK(cudaMemcpy(stats_out, d_stats, 8 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    HCK(cudaMemcpy(flags_out, d_flags, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    HCK(cudaMemcpy(cache_out, d_cache_out, 1024 * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    HCK(cudaMemcpy(n_deliv_out, d_n_deliv, nb * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    HCK(cudaMemcpy(offsets_out, d_offsets, (nb + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    HCK(cudaMemcpy(start_out, d_start, nb * 1024 * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return 0;
}
