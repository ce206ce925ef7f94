// modes_levels.cu — the level pass (modes_set_levels, modes_levels_device): for every reference
// buffer of a batch, the noise and clipping sums of modes_levels_core.cuh over its own 131072 samples,
// one modes_level record per buffer.
//
// A bandwidth-bound reduction over whole buffers already in HBM.  It is a separate kernel so that,
// with the feature off, nothing about the default kernels changes.  It reads the batch body only:
// the 238 carried samples of a buffer belong to the buffer before it, so every stream sample is
// counted exactly once.
//
// Shape: the magnitude table (lutn, 64 KB, keyed by I^2 + Q^2) is staged in shared memory once per
// CTA; a CTA then takes whole buffers, grid-stride.  Each thread reads 16-byte words at an 8 KB stride
// (four loads in flight), keeps its partial sums in registers (32-bit sum of magnitudes, 64-bit sum
// of squares), and the CTA reduces them with warp shuffles and one shared-memory step.  Lane 0 of warp
// 0 writes the buffer's record: exactly one writer per record and no accumulation in device memory,
// so a relaunch of the batch writes the same records.
#include <cstdint>
#include <cuda_runtime.h>
#include "modes_internal.h"
#include "modes_levels_core.cuh"

namespace modes {

constexpr int kLevelThreads = 512;
constexpr int kLevelWarps = kLevelThreads / 32;
constexpr int kLevelBlocksPerSm = 3;                                      // 3 x 64 KB of table per SM
constexpr int kLevelUnroll = 4;
constexpr int kLevelVecs = MODES_BUFFER_BYTES / 16;                       // 16-byte words per buffer
constexpr int kLevelLutBytes = (kNLutEntries * 2 + 15) / 16 * 16;
static_assert(kLevelVecs % (kLevelUnroll * kLevelThreads) == 0, "whole rounds per buffer");
// a thread's 32-bit sum of magnitudes, and a warp's, cannot overflow
static_assert((uint64_t)32 * (kBufSamples / kLevelThreads) * 65167u < (1ull << 32), "warp magnitude sum fits in 32 bits");

__global__ void __launch_bounds__(kLevelThreads, kLevelBlocksPerSm)
levels_kernel(const uint8_t *__restrict__ base, uint32_t n_buffers, uint64_t stride, const uint16_t *__restrict__ lutn,
              modes_level *__restrict__ out) {
    extern __shared__ uint4 s_raw[];
    uint16_t *s_lut = reinterpret_cast<uint16_t *>(s_raw);
    __shared__ uint64_t s_mag[kLevelWarps], s_pow[kLevelWarps];
    __shared__ uint32_t s_peak[kLevelWarps], s_clip[kLevelWarps];
    for (int i = threadIdx.x; i < (kNLutEntries - 1) / 8; i += kLevelThreads)
        s_raw[i] = __ldg(reinterpret_cast<const uint4 *>(lutn) + i);
    if (threadIdx.x == 0) s_lut[kNLutEntries - 1] = lutn[kNLutEntries - 1];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t b = blockIdx.x; b < n_buffers; b += gridDim.x) {
        const uint4 *p = reinterpret_cast<const uint4 *>(base + (uint64_t)b * stride) + threadIdx.x;
        levels::Acc a;
        levels::acc_clear(a);
        for (int i = 0; i < kLevelVecs; i += kLevelUnroll * kLevelThreads) {
            uint4 v[kLevelUnroll];
#pragma unroll
            for (int u = 0; u < kLevelUnroll; u++) v[u] = __ldcs(p + i + u * kLevelThreads);
#pragma unroll
            for (int u = 0; u < kLevelUnroll; u++) levels::add_quad(a, v[u].x, v[u].y, v[u].z, v[u].w, s_lut);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            a.sum_mag += __shfl_xor_sync(0xffffffffu, a.sum_mag, o);
            a.sum_power += __shfl_xor_sync(0xffffffffu, a.sum_power, o);
            a.peak = max(a.peak, __shfl_xor_sync(0xffffffffu, a.peak, o));
            a.clipped += __shfl_xor_sync(0xffffffffu, a.clipped, o);
        }
        if (lane == 0) { s_mag[warp] = a.sum_mag; s_pow[warp] = a.sum_power; s_peak[warp] = a.peak; s_clip[warp] = a.clipped; }
        __syncthreads();
        if (warp == 0) {
            uint64_t mag = lane < kLevelWarps ? s_mag[lane] : 0, pw = lane < kLevelWarps ? s_pow[lane] : 0;
            uint32_t peak = lane < kLevelWarps ? s_peak[lane] : 0, clip = lane < kLevelWarps ? s_clip[lane] : 0;
#pragma unroll
            for (int o = kLevelWarps / 2; o > 0; o >>= 1) {
                mag += __shfl_xor_sync(0xffffffffu, mag, o);
                pw += __shfl_xor_sync(0xffffffffu, pw, o);
                peak = max(peak, __shfl_xor_sync(0xffffffffu, peak, o));
                clip += __shfl_xor_sync(0xffffffffu, clip, o);
            }
            if (lane == 0) {
                modes_level r;
                r.buffer = b;
                r.n_samples = kBufSamples;
                r.clipped = clip;
                r.sum_mag = mag;
                r.sum_power = pw;
                r.peak = peak;
                r.pad = 0;
                out[b] = r;
            }
        }
        __syncthreads();                                                  // s_* are reused by the next buffer
    }
}

void launch_levels(const uint8_t *d_iq, uint32_t n_buffers, uint64_t stride_bytes, const DeviceTables &tab,
                   modes_level *out, int sm_count, cudaStream_t stream) {
    if (!n_buffers) return;
    // the opt-in to > 48 KB of dynamic shared memory is per device
    static bool configured[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 || !configured[dev]) {
        cudaFuncSetAttribute(levels_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kLevelLutBytes);
        if (dev >= 0 && dev < 64) configured[dev] = true;
    }
    const uint32_t most = (uint32_t)sm_count * kLevelBlocksPerSm;
    levels_kernel<<<n_buffers < most ? n_buffers : most, kLevelThreads, kLevelLutBytes, stream>>>(d_iq, n_buffers, stride_bytes,
                                                                                              tab.lutn, out);
}

}  // namespace modes
