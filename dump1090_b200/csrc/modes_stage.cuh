// modes_stage.cuh — the device loaders that stage input bytes for the kernels reading a stream's input
// span: K9-K12 (modes_resample.cu) and the spectrum pass K13 (modes_spectrum.cu).
#pragma once
#include "modes_internal.h"
#include "modes_input_core.cuh"

namespace modes {
// (an unnamed namespace, as the kernels that use them are in: their names stay those of each file's own)
namespace {

// Staging loaders: the 16 UC8 bytes of the tile's input at byte p of the converted stream relative to the
// job's first input sample (p a multiple of 16); bytes outside the job's span are no signal.
struct Uc8Input {
    __device__ __forceinline__ uint4 word(const ResampleJob &j, int64_t p) const {
        const int64_t in_bytes = (int64_t)j.in_bytes;
        if (p >= 0 && p + 16 <= in_bytes) return __ldg(reinterpret_cast<const uint4 *>(j.in + p));
        uint32_t b[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            uint32_t word = 0;
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int64_t pe = p + 4 * k + e;
                const uint32_t x = (pe >= 0 && pe < in_bytes) ? j.in[pe] : 127u;
                word |= x << (8 * e);
            }
            b[k] = word;
        }
        return make_uint4(b[0], b[1], b[2], b[3]);
    }
};

// SC16 / SC16Q11: the 8 samples of a word are 32 int16 bytes at 2 p; a sample is in the span when all 4
// of its bytes are (the trailing partial sample is not).  A missing sample reads as (0, 0), which
// converts to (127, 127) at every shift.
struct Sc16Input {
    int shift;
    __device__ __forceinline__ uint4 word(const ResampleJob &j, int64_t p) const {
        const int64_t b = 2 * p;
        const int64_t in_bytes = (int64_t)(j.in_bytes & ~(uint64_t)3);
        uint32_t w[8];
        if (b >= 0 && b + 32 <= in_bytes) {
            const uint4 lo = __ldg(reinterpret_cast<const uint4 *>(j.in + b));
            const uint4 hi = __ldg(reinterpret_cast<const uint4 *>(j.in + b + 16));
            w[0] = lo.x; w[1] = lo.y; w[2] = lo.z; w[3] = lo.w;
            w[4] = hi.x; w[5] = hi.y; w[6] = hi.z; w[7] = hi.w;
        } else {
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int64_t e = b + 4 * k;
                w[k] = (e >= 0 && e + 4 <= in_bytes) ? __ldg(reinterpret_cast<const uint32_t *>(j.in + e)) : 0u;
            }
        }
        uint32_t o[4];
#pragma unroll
        for (int k = 0; k < 4; k++)
            o[k] = input::convert_pair(w[2 * k], shift) | input::convert_pair(w[2 * k + 1], shift) << 16;
        return make_uint4(o[0], o[1], o[2], o[3]);
    }
};

// Stream byte p (a multiple of 16) of a job's input: the history [hist0, call0), the call [call0, + buffer),
// no signal elsewhere.
template <class Job>
__device__ __forceinline__ uint4 job_word(const Job &j, int64_t p) {
    if (p >= j.hist0 && p < j.call0) return __ldg(reinterpret_cast<const uint4 *>(j.hist + (p - j.hist0)));
    if (p >= j.call0 && p < j.call0 + MODES_BUFFER_BYTES) return __ldg(reinterpret_cast<const uint4 *>(j.stage + (p - j.call0)));
    return make_uint4(0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu);
}

}  // namespace
}  // namespace modes
