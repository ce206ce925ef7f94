/* modes_b200.h — C ABI of the H100-native Mode S / ADS-B demodulator.
 *
 * Drop-in boundary for dump1090's --ifile decode path.  The reference has no
 * plugin/FFI surface; the seam is its main loop (dump1090.c:2968-2990):
 *
 *     computeMagnitudeVector();                       dump1090.c:1454 / :2974
 *     detectModeS(Modes.magnitude, Modes.data_len/2); dump1090.c:1563 / :2986
 *         -> decodeModesMessage(&mm, msg)             dump1090.c:1091 / :1735
 *         -> useModesMessage(&mm)                     dump1090.c:1802 / :1777
 *
 * Each entry point below names the reference interface it replaces.  Plain C
 * types only; the library owns all device memory, streams and chunking, so
 * a caller passes raw file bytes in file order in pieces of any size and gets
 * back, in stream order, exactly the messages (and struct modesMessage fields)
 * the reference hands to useModesMessage() for the same bytes.
 *
 * There is no CPU fallback: modes_create() fails (NULL + modes_last_error)
 * when no CUDA device is usable.
 *
 * Threading: a context is not re-entrant (one thread at a time per modes_ctx, like the
 * reference's single decode thread); distinct contexts are independent.  Callbacks run on the
 * calling thread.  Status codes: 0 = ok, <0 = error with text in modes_last_error(ctx); the
 * library never calls exit().
 */
#ifndef MODES_B200_H
#define MODES_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MODES_B200_ABI_VERSION 3

/* Sizes fixed by the reference's buffering (dump1090.c:54, :61, :331). */
#define MODES_BUFFER_BYTES    262144      /* MODES_DATA_LEN: new bytes per reference buffer */
#define MODES_BUFFER_SAMPLES  131072
#define MODES_CARRY_BYTES     476         /* (MODES_FULL_LEN-1)*4 carried into the next buffer */
#define MODES_CARRY_SAMPLES   238

/* Replaces the four globals that change hot-path results: Modes.fix_errors
 * (dump1090.c:167, --no-fix :2873), Modes.aggressive (:179, :2896),
 * Modes.check_crc (:168, :2875), plus the EOF-buffer race made explicit
 * (dump1090.c:497 vs :2989; SURVEY.md fact 3). */
typedef struct modes_config {
    int32_t fix_errors;         /* 1 (default): 1-bit (2-bit if aggressive) CRC repair on DF11/17/18 */
    int32_t aggressive;         /* 0 (default) */
    int32_t check_crc;          /* 1 (default): deliver only messages with crcok */
    int32_t drop_eof_buffer;    /* 0 (default): decode the buffer that hit EOF; 1: drop it, as the
                                   stock binary does in most runs */
    int32_t device;             /* CUDA device ordinal, default 0 */
    int32_t profile;            /* 1: record per-kernel CUDA-event times (modes_get_kernel_times) */
    uint64_t max_batch_bytes;   /* device staging per in-flight batch; 0 = 64 MiB.  It counts the batch's
                                   2 MHz UC8 bytes: the input span a batch uploads at another rate or format
                                   is up to 10 times that (10 MS/s SC16) */
    int32_t n_gpus;             /* 0 or 1: one GPU (`device`).  N > 1: the streaming decode (modes_process /
                                   modes_finish) deals its batches of whole reference buffers round-robin to N
                                   devices starting at `device` — one stream, one pinned-to-device copy and
                                   two staging slots per GPU, every GPU behind its own PCIe link — and the
                                   calling thread resolves each group of N batches exactly (the speculative
                                   shard resolve of modes_resolver_run_shards).  With fewer than N devices
                                   present, devices are reused round-robin.  The stage-level entry points
                                   stay on `device`. */
    int32_t gpu_resolve;        /* 0 (default): the order-dependent half (retry/skip state machine, ICAO cache,
                                   statistics: dump1090.c:1769-1791, :898-983) is replayed on the host over the
                                   candidate records.  1: it runs on the GPU too — one warp per reference buffer,
                                   address caches handed from buffer to buffer and verified (SURVEY.md §8(f) item
                                   4); a batch whose caches do not settle in a few rounds is replayed in stream
                                   order on the device — and only 40-byte records of the delivered messages cross
                                   PCIe; the host builds the struct fields.  Same messages, same statistics, on
                                   any input within the density below (all flags included).  Streaming decode
                                   on one GPU only; a batch denser than one candidate per 64 samples is an error
                                   in this mode. */
} modes_config;

/* Replaces struct modesMessage (dump1090.c:211-260): same field names and
 * meaning, 32-bit fields in a fixed order.  Fields the reference leaves
 * unassigned for a given DF are 0 here.  nfixed and sample_pos are additions. */
typedef struct modes_message {
    uint8_t  msg[14];
    uint8_t  recovered;         /* 1: delivered by the soft-decision recovery (modes_set_recovery), not by the reference;
                                   2: the same at a weak preamble (modes_set_weak_preambles) */
    uint8_t  arrival;           /* MODES_EVAL_ARRIVAL code of the delivered attempt (modes_set_arrival): 0 = not measured,
                                   otherwise the arrival is (arrival - 8) 12 MHz ticks after 6 * sample_pos */
    int32_t  msgbits, msgtype, crcok;
    uint32_t crc;
    int32_t  errorbit, aa1, aa2, aa3, phase_corrected;
    int32_t  ca, iid;
    int32_t  metype, mesub, heading_is_valid, heading, aircraft_type;
    int32_t  fflag, tflag, raw_latitude, raw_longitude;
    char     flight[9];
    char     pad1[1];
    int16_t  carrier;           /* carrier code of the delivered attempt (modes_set_carrier): 0 = not measured,
                                   otherwise its frequency is (carrier - 16384) * 100 Hz above the bytes' centre */
    int32_t  ew_dir, ew_velocity, ns_dir, ns_velocity;
    int32_t  vert_rate_source, vert_rate_sign, vert_rate, velocity;
    int32_t  movement, movement_valid, ground_track, ground_track_valid;
    int32_t  fs, dr, um, identity;
    int32_t  altitude, unit;
    int32_t  nfixed;            /* bits repaired by the CRC fix (0/1/2) */
    int32_t  signal;            /* RMS pulse magnitude of the frame (see modes_frame_eval.signal); 0 = not measured */
    int64_t  sample_pos;        /* stream sample index of the preamble start */
} modes_message;

/* One evaluated frame attempt at one preamble position: everything
 * detectModeS()+decodeModesMessage() compute that is a pure function of the
 * samples and the flags (dump1090.c:1668-1735, :1099-1128). */
typedef struct modes_frame_eval {
    uint8_t  msg[14];           /* frame bytes, after the CRC fix if one was applied */
    uint8_t  msgtype;           /* DF of the demodulated frame (before any fix) */
    uint8_t  flags;             /* MODES_EVAL_* in bits 0-3; bits 4-7: the arrival code (MODES_EVAL_ARRIVAL_*) */
    uint8_t  errorbit;          /* first repaired bit, 0xFF = none */
    uint8_t  nfixed;
    uint16_t signal;            /* with modes_set_signal on and MODES_EVAL_DECODED set: floor(sqrt(floor(S / b))),
                                   S = sum over the b frame bits (b = 56 or 112 from msgtype) of the squared
                                   larger magnitude of the bit's two uncorrected samples (dump1090.c:1670-1671,
                                   magnitudes of :359-364); otherwise 0 */
    uint32_t crc;               /* 24-bit syndrome after the fix; 0 when not decoded */
} modes_frame_eval;

#define MODES_EVAL_GATE_OK   1  /* mean |low-high| >= 2550             dump1090.c:1723 */
#define MODES_EVAL_ERRORS    2  /* demodulation error in first 56 bits dump1090.c:1682 */
#define MODES_EVAL_DECODED   4  /* decodeModesMessage reached          dump1090.c:1731 */
#define MODES_EVAL_P2_VALID  8  /* pass[1] (phase-corrected retry) was evaluated */
#define MODES_EVAL_ARRIVAL_SHIFT 4      /* flags >> 4: arrival code, modes_set_arrival; 0 with the switch off */
#define MODES_EVAL_ARRIVAL_MASK  0xF0

/* One preamble candidate: a position that passes the tests of
 * dump1090.c:1602-1650, with the first attempt and the phase-corrected retry
 * (dump1090.c:1653-1664) both evaluated on the device. */
typedef struct modes_candidate {
    int64_t t;                  /* 131072*buffer_index + j  (j = index inside the reference buffer) */
    modes_frame_eval pass[2];
} modes_candidate;

/* Per scan tile: where its candidates sit in the candidate array.  Tiles are
 * in stream order; candidates inside a tile are in stream order.  How many positions a tile
 * covers is the scan kernel's business: size tile tables with modes_tile_count(). */
typedef struct modes_tile { uint32_t offset, count; } modes_tile;
#define MODES_TILE_SAMPLES 7936             /* 8 rows of 31 x 32 positions, see csrc/modes_scan2.cu */

/* Replaces Modes.stat_* (dump1090.c:186-195) in the order the reference prints
 * them (:2994-3003): valid_preamble, out_of_phase, demodulated, goodcrc,
 * badcrc, fixed, single_bit_fix, two_bits_fix. */
typedef struct modes_stats { int64_t v[8]; } modes_stats;

typedef struct modes_ctx modes_ctx;

/* Replaces useModesMessage(struct modesMessage*) (dump1090.c:1802): called on
 * the calling thread from modes_process/modes_finish/modes_resolve, in stream
 * order, once per message that passes the reference's gate (:1803).  The
 * pointer is valid only during the call. */
typedef void (*modes_sink_fn)(void *user, const modes_message *mm);

/* ---- lifecycle ---------------------------------------------------------- */
int         modes_abi_version(void);
void        modes_default_config(modes_config *cfg);                 /* modesInitConfig, dump1090.c:299 */
modes_ctx  *modes_create(const modes_config *cfg);                   /* modesInit, dump1090.c:321 */
void        modes_destroy(modes_ctx *ctx);
const char *modes_last_error(const modes_ctx *ctx);                  /* ctx may be NULL: create() error */
int         modes_set_sink(modes_ctx *ctx, modes_sink_fn fn, void *user);

/* Alternative to a callback: append every delivered message to a caller-owned
 * array (NULL/0 to stop).  modes_output_count() keeps counting past capacity. */
int    modes_set_output(modes_ctx *ctx, modes_message *out, size_t capacity);
size_t modes_output_count(const modes_ctx *ctx);

/* ---- streaming decode: the main loop, dump1090.c:2968-2990 -------------- */
/* Feed the next `nbytes` of the u8 I/Q stream (host memory, pinned or not).
 * Whole reference buffers are decoded as they complete.  0 = ok, <0 = error. */
int  modes_process(modes_ctx *ctx, const uint8_t *iq, size_t nbytes);
/* modes_process for bytes in device memory of the context's device (cfg.device): a CUDA SDR front end, a
 * torch pipeline or a capture read into GPU memory feeds the decoder without a copy through the host.
 *   Same output: a sequence of calls, then modes_finish, gives exactly what modes_process gives on the same
 *     bytes in the same call sizes: messages and every field, sample_pos, statistics, level, spectrum,
 *     recovery and weak records, signal and arrival codes, both drop_eof_buffer outcomes; at every input
 *     rate, format, offset and modes_set_* switch, with gpu_resolve and with n_gpus > 1 (whose other GPUs
 *     receive their batches from cfg.device's memory, peer to peer where the driver allows).
 *   Any pointer alignment and any byte count, odd counts and calls that split a buffer or a sample included.
 *   The bytes must be fully written before the call: it does not order itself after the caller's streams.
 *     When it returns, the decoder no longer reads d_iq, as modes_process returns with every copy done.
 *   One kind of memory per stream: from its first call until modes_finish / modes_reset a stream is fed
 *     either by modes_process or by modes_process_device; the other is refused with "in progress".
 *     modes_finish ends either.
 *   Refused: d_iq NULL with nbytes > 0, and memory that cudaPointerGetAttributes does not report as device
 *     memory of cfg.device (host, pinned, managed, or another device's), with a message naming it.
 * The stream's partial buffer, carry and input history then live on the device too; a stream fed from the
 * host allocates none of them. */
int  modes_process_device(modes_ctx *ctx, const void *d_iq, size_t nbytes);
/* End of stream: 127-pad and decode (or drop) the EOF buffer (dump1090.c:496-507). */
int  modes_finish(modes_ctx *ctx);
/* Forget stream position, carry, ICAO cache and statistics (a new --ifile run). */
int  modes_reset(modes_ctx *ctx);
int  modes_get_stats(const modes_ctx *ctx, modes_stats *out);

/* ---- 2.4, 4, 6, 8 and 10 MS/s input -------------------------------------- */
/* The sample rate of the bytes modes_process takes: 2000000 (the default, what dump1090 reads),
 * 2400000 (what dump1090-fa and readsb record from RTL-SDR dongles), or 4000000, 6000000, 8000000 and
 * 10000000 (what Airspy, SDRplay, USRP and other 16-bit radios usually record); any other value is
 * refused with a message that says "not supported".  It is
 * also refused between the first modes_process of a stream and modes_finish / modes_reset, and takes
 * effect for the stream that begins at create or reset.  On an n_gpus > 1 context it reaches every GPU.
 * A receiver of the pool has its own rate: modes_pool_set_input_rate below.
 *
 * At 2400000 every batch is first resampled to 2 MHz on the device by an exact 5:6 polyphase filter,
 * and the whole pipeline (and every modes_set_* pass) runs on those bytes unchanged, so a 2.4 MS/s
 * stream decodes to exactly what the 2 MHz decoder gives on the stream's resampled bytes:
 *   input   UC8 I/Q, zero at 127; n_in = ceil(bytes / 2), a trailing odd byte is an I whose Q is 127,
 *           and samples outside [0, n_in) read as (127, 127)
 *   output  sample n = 5q + r (r = 0..4) with base input index b = 6q + r, for I and Q separately
 *               y = clamp(127 + ((sum_k h[r][k] * (x[b + k - T/2 + 1] - 127) + 8192) >> 14), 0, 255)
 *           (int32 sum, arithmetic shift); N_out = ceil(5 n_in / 6) output samples
 *   taps    T = 6, signed 16-bit Q14, every branch summing to 16384: a Kaiser-windowed sinc (beta 5,
 *           cutoff 1.1 MHz) sampled at input offsets k - T/2 + 1 - 0.2 r (modes_resample_core.cuh)
 * The EOF buffer is 127 past N_out, as modes_finish pads a 2 MHz stream.  sample_pos counts 2 MHz
 * samples; output sample n sits at input time 1.2 n exactly, so 6 * sample_pos is the input time in
 * 12 MHz ticks and the Beast timestamps keep their meaning.  Level records describe the resampled
 * bytes (their clipping count can be lower than the input's).
 *
 * At 2000000 M (M = 2, 3, 4, 5) every batch is first decimated to 2 MHz on the device by an exact
 * integer filter, with the same consequences: the stream decodes to exactly what the 2 MHz decoder gives
 * on its decimated bytes, for every input format:
 *   output  sample n stands for input samples [M n, M n + M); for I and Q separately
 *               y = clamp(127 + ((sum_{k<T} h_M[k] * (x[M n - E + k] - 127) + 8192) >> 14), 0, 255)
 *           (int32 sum, arithmetic shift), T = M + 2E; N_out = ceil(n_in / M) output samples
 *   taps    signed 16-bit Q14, symmetric about input M n + (M - 1) / 2, each table summing to 16384
 *           (modes_resample_core.cuh has them)
 * Output sample n starts at input sample M n exactly, so 6 * sample_pos stays the 12 MHz time.  Level
 * records describe the decimated bytes. */
int  modes_set_input_rate(modes_ctx *ctx, uint32_t hz);
/* Where 1090 MHz sits in the capture's baseband, for a radio tuned off the channel (a zero-IF front end
 * tuned 1-3 MHz away from its DC spike, or a recording centred elsewhere): +2000000 means the radio was
 * tuned to 1088 MHz.  The decoder multiplies the input by e^{-j 2 pi offset_hz n / fs} before decimating.
 * 0, the default, is always taken.  Another value is taken only at 4000000 to 10000000 samples/s, with
 * |offset_hz| <= fs / 2 - 1 MHz (1, 2, 3 and 4 MHz at 4, 6, 8 and 10 MS/s); otherwise it is refused with
 * "not supported", and modes_set_input_rate likewise refuses a rate whose range excludes the offset
 * already set (so a caller who changes both sets the offset to 0 first).  Both setters are refused between
 * the first modes_process of a stream and modes_finish / modes_reset; modes_reset keeps the offset, and on
 * an n_gpus > 1 context it reaches every GPU.  Exactly, for input sample m counted from the stream's start
 * (int16 input after its conversion), xi = I - 127 and xq = Q - 127 (0 outside the stream):
 *   step    = round(offset_hz 2^32 / fs)                       (int64 arithmetic, stored as uint32)
 *   theta_m = (m step) mod 2^32                                (m taken mod 2^32 first)
 *   k_m     = ((theta_m + 2^21) >> 22) & 1023                  (the nearest of 1024 phases)
 *   c, s    = C[k_m], S[k_m]  with C[k] = round(16384 cos(2 pi k / 1024)), S[k] = round(16384 sin(2 pi k / 1024))
 *   u_i     = (xi c + xq s + 8192) >> 14,  u_q = (xq c - xi s + 8192) >> 14   (int32, arithmetic shift)
 *   y       = clamp(127 + ((sum_{k<T} h_M[k] u[M n - E + k] + 8192) >> 14), 0, 255)   for I and Q separately
 * with h_M, E and T the decimator's above (modes_resample_core.cuh has C and S).  The shift applied is
 * step fs / 2^32 Hz, within 0.002 Hz of offset_hz.  N_out, the EOF buffer, sample_pos, 6 * sample_pos as the
 * 12 MHz time and the arrival estimate keep their meaning: output n still starts at input sample M n.  At
 * offset 0 the output is the decimator's, byte for byte.  The receiver pool has no offset (it does not
 * take the decimated rates). */
int  modes_set_input_offset(modes_ctx *ctx, int32_t offset_hz);
/* The same per receiver of a pool (modes_pool_* below): 2000000 (the default) or 2400000; refused, with
 * "not supported", for any other value (the decimated rates included), a receiver out of range, and while the receiver has a stream in progress (from the
 * first modes_pool_submit / _ingest that names it until modes_pool_reset, which keeps the rate).  It
 * touches no device.  A 2.4 MS/s receiver's iq[i] is still MODES_BUFFER_BYTES of its stream (131072
 * input samples); a 2 MHz buffer of its resampled stream is decoded in the call whose input completes it
 * (its last sample and the filter's 4-sample lookahead have arrived): at most one per call, none in the
 * first call and in about one call in six after it.  A call in which no named receiver completes a buffer
 * delivers nothing and is still collected.  modes_pool_buffers counts the 2 MHz buffers decoded, and the
 * receiver's messages, sample_pos (2 MHz samples), statistics and level records (their buffer index a
 * 2 MHz buffer's) equal those of the 2 MHz decode, without the EOF buffer, of the first
 * modes_pool_buffers buffers of the receiver's resampled stream, with every switch, until
 * modes_pool_finish ends the stream with the buffers whose lookahead never arrives and the EOF buffer.  The pool's device
 * memory grows by a staging area (2 x 256 KiB per receiver of a batch) and about 1.1 MiB of input
 * history per 2.4 MS/s receiver. */
typedef struct modes_pool modes_pool;                /* the receiver pool: "many receivers on one GPU" below */
int  modes_pool_set_input_rate(modes_pool *p, uint32_t receiver, uint32_t hz);

/* ---- 16-bit input ---------------------------------------------------------- */
/* The sample format of the bytes modes_process takes, dump1090-fa's --iformat:
 *   MODES_INPUT_UC8      unsigned 8-bit I/Q, zero at 127 (the default, what dump1090 reads)
 *   MODES_INPUT_SC16     signed little-endian 16-bit I/Q (SoapySDR devices, Airspy-class tools)
 *   MODES_INPUT_SC16Q11  the same with 12-bit values (bladeRF)
 * shift: 0 ... 15, or negative for the format's default, which maps full scale to full scale: 8 for SC16,
 * 4 for SC16Q11.  Refused: an unknown format, a shift above 15, a shift other than 0 or negative with
 * UC8, and, as modes_set_input_rate, a call between the first modes_process of a stream and
 * modes_finish / modes_reset.  It takes effect for the stream that begins at create or reset (which keeps
 * it), reaches every GPU of an n_gpus > 1 context, and combines with either input rate.  A receiver of
 * the pool has its own format: modes_pool_set_input_format below.
 *
 * A 16-bit stream is converted to UC8 on the device, then decoded as a UC8 stream at the input rate
 * (at 2400000: converted, then resampled), so it decodes to exactly what the UC8 decoder gives on the
 * converted bytes:
 *   input   I, Q interleaved, 4 bytes a sample; n_in = floor(bytes / 4), 1-3 trailing bytes are ignored
 *   output  for a value v (I or Q) and the shift s, in int32 with an arithmetic shift (round half up):
 *               q = s ? (v + (1 << (s - 1))) >> s : v,   byte = clamp(127 + q, 0, 255)
 * At 2 MHz the EOF buffer is 127 past n_in, as modes_finish pads a UC8 stream.  Level records describe
 * the converted bytes, so their clipping count is the samples the shift saturated: a smaller shift
 * resolves weaker signals and clips strong ones sooner. */
#define MODES_INPUT_UC8      0u
#define MODES_INPUT_SC16     1u
#define MODES_INPUT_SC16Q11  2u
int  modes_set_input_format(modes_ctx *ctx, uint32_t format, int32_t shift);
/* The same per receiver of a pool (modes_pool_* below), with the same formats and shifts; refused for
 * what modes_set_input_format refuses, a receiver out of range, and, as modes_pool_set_input_rate, while
 * the receiver has a stream in progress (from the first modes_pool_submit / _ingest that names it until
 * modes_pool_reset, which keeps the format and the shift).  It touches no device and combines with either
 * input rate, set in either order.  One call still brings MODES_BUFFER_SAMPLES samples of every receiver
 * it names: iq[i] is MODES_BUFFER_BYTES bytes for a UC8 receiver and 2 x MODES_BUFFER_BYTES bytes of
 * little-endian int16 I/Q for an SC16 or SC16Q11 one, so the pool's schedule is the same at either format.
 * Everything the pool delivers for a 16-bit receiver (messages and their fields, sample_pos, statistics,
 * level records, recovery and weak statistics, modes_pool_buffers) equals what it delivers for a UC8
 * receiver at the same rate fed the converted bytes; level records describe the converted bytes.  A call
 * that names a 16-bit receiver converts its buffers on the device; the pool's device memory grows by a
 * staging area of 2 x 512 KiB per receiver of a batch (one per batch in flight), besides the 2 x 256 KiB
 * one a call that names a 2.4 MS/s receiver also uses.  modes_pool_resolve stays UC8 at 2 MHz. */
int  modes_pool_set_input_format(modes_pool *p, uint32_t receiver, uint32_t format, int32_t shift);

/* ---- stage-level entry points (tests, bench, multi-GPU sharding) -------- */
/* computeMagnitudeVector() alone (dump1090.c:1454-1469): nsamples I/Q pairs in
 * host memory -> nsamples u16 magnitudes in host memory, computed on the device. */
int  modes_compute_magnitude(modes_ctx *ctx, const uint8_t *iq, size_t nsamples, uint16_t *mag);

/* The device half of detectModeS() on data already in HBM.  d_iq: n_buffers *
 * MODES_BUFFER_BYTES bytes of device memory (16-byte aligned) holding whole
 * reference buffers of the stream; carry476: the MODES_CARRY_BYTES stream
 * bytes preceding d_iq (host memory), or NULL at stream start (no-signal).
 * Launches the scan and frame-evaluation kernels on the context's stream and
 * returns without waiting.  d_candidates (capacity cand_capacity records) and
 * d_tiles (modes_tile_count(n_buffers) entries) are device memory supplied by the caller, or
 * NULL to use the context's own workspace. */
int  modes_detect_device(modes_ctx *ctx, const void *d_iq, size_t n_buffers, const uint8_t *carry476,
                         void *d_candidates, size_t cand_capacity, void *d_tiles);
/* Same, from HOST memory (pinned for full speed): the library stages the buffers into its own device
 * memory with one asynchronous copy on the same stream, then launches the kernels. */
int  modes_detect_host(modes_ctx *ctx, const uint8_t *iq, size_t n_buffers, const uint8_t *carry476,
                       void *d_candidates, size_t cand_capacity, void *d_tiles);
/* The resampling of modes_set_input_rate(2400000) over a span already in device memory, for a job that
 * decodes its own shard of a 2.4 MS/s capture with modes_detect_device.  d_in: in_bytes bytes of the
 * stream's input from input sample in_first_sample on (16-byte aligned); every other input byte reads as
 * no signal (127), so the span must hold the input samples
 *     [floor(6 n0 / 5) - 2, floor(6 (n1 - 1) / 5) + 4)   with n0 = MODES_BUFFER_SAMPLES * first_buffer - 238,
 *                                                          n1 = MODES_BUFFER_SAMPLES * (first_buffer + n_buffers)
 * that exist.  Writes the 2 MHz reference buffers first_buffer ... first_buffer + n_buffers - 1 to d_out
 * (n_buffers * MODES_BUFFER_BYTES, 16-byte aligned); output samples at or past out_end are 127 (the
 * EOF buffer: out_end = N_out; negative = no limit).  carry476 (host memory, or NULL): the
 * MODES_CARRY_BYTES 2 MHz bytes before d_out, as modes_detect_device takes them; with it the call waits
 * for them, without it it returns at once.  Runs on the context's stream. */
int  modes_resample_device(modes_ctx *ctx, const void *d_in, size_t in_bytes, int64_t in_first_sample,
                           int64_t first_buffer, size_t n_buffers, int64_t out_end, void *d_out, uint8_t *carry476);
/* modes_resample_device at any rate modes_set_input_rate takes other than 2000000 (the call above is this
 * one at 2400000), UC8 input as there, the same arguments and the same behaviour.  At 2000000 M the span
 * must hold the input samples [M n0 - E, M n1 + E) that exist, with n0 = MODES_BUFFER_SAMPLES *
 * first_buffer - 240 and n1 as above (E: 2 for M = 2, 4 and 5; 1 for M = 3).  Any other rate is refused
 * with "not supported". */
int  modes_resample_device_at(modes_ctx *ctx, uint32_t hz, const void *d_in, size_t in_bytes, int64_t in_first_sample,
                              int64_t first_buffer, size_t n_buffers, int64_t out_end, void *d_out, uint8_t *carry476);
/* modes_resample_device_at with the input first rotated by offset_hz as modes_set_input_offset defines it,
 * the phase taken from each sample's stream index in_first_sample + i (so spans of one stream agree wherever
 * they are cut).  offset_hz 0 is modes_resample_device_at exactly; another offset is taken only at
 * 4000000 to 10000000 with |offset_hz| <= hz / 2 - 1 MHz, and refused with "not supported" otherwise. */
int  modes_resample_device_shift(modes_ctx *ctx, uint32_t hz, int32_t offset_hz, const void *d_in, size_t in_bytes,
                                 int64_t in_first_sample, int64_t first_buffer, size_t n_buffers, int64_t out_end,
                                 void *d_out, uint8_t *carry476);
/* Wait for the last modes_detect_device; returns the candidate count. */
int  modes_detect_wait(modes_ctx *ctx, uint64_t *n_candidates);
/* Copy the last result to host memory (arrays sized by the caller from
 * modes_detect_wait's count and modes_tile_count(n_buffers) tiles). */
int  modes_detect_fetch(modes_ctx *ctx, modes_candidate *candidates, modes_tile *tiles);

/* The sequential half of detectModeS(): retry/skip state machine
 * (dump1090.c:1769-1791), ICAO cache (:898-983, :1183-1210), statistics and the
 * sink gate (:1803), replayed over candidates in stream order.  buffer_base is
 * the stream index of the first reference buffer the arrays describe. */
int  modes_resolve(modes_ctx *ctx, const modes_candidate *candidates, const modes_tile *tiles,
                   size_t n_tiles, int64_t buffer_base);

/* The same sequential half as a standalone host object (no device needed): what
 * rank 0 runs over gathered candidate records in a multi-GPU job. */
typedef struct modes_resolver modes_resolver;
modes_resolver *modes_resolver_create(const modes_config *cfg);
void modes_resolver_destroy(modes_resolver *r);
int  modes_resolver_run(modes_resolver *r, const modes_candidate *candidates, const modes_tile *tiles,
                        size_t n_tiles, int64_t buffer_base, modes_sink_fn sink, void *user);
/* Several consecutive shards of one stream at once (one per GPU): resolved concurrently on host
 * threads by speculating the ICAO cache at each shard boundary and verifying it; the result is
 * identical to calling modes_resolver_run shard by shard. */
int  modes_resolver_run_shards(modes_resolver *r, size_t n_shards, const modes_candidate *const *candidates,
                               const modes_tile *const *tiles, const size_t *n_tiles, const int64_t *buffer_base,
                               modes_sink_fn sink, void *user);
/* One shard of a sharded decode, resolved where its records are (one rank or GPU thread per shard).
 * The only state crossing a shard boundary is the 1024-slot address cache (dump1090.c:335, :898-983):
 * a shard is resolved TENTATIVELY from a guess of the cache at its start — the job's starting cache
 * overwritten by what the tail of the previous shard leaves (modes_resolver_tail_cache, exchanged
 * between the shards' owners, 4 KiB) — the guess is compared with what the previous shard really
 * ended with (modes_resolver_get_cache after its tentative run), and a shard whose guess was wrong
 * is run again from the right cache.  modes_resolver_commit then delivers the messages and adds the
 * statistics.  dump1090_b200/sharded.py:resolve_distributed is the protocol over torch.distributed;
 * modes_resolver_run_shards is the same thing inside one process. */
#define MODES_ICAO_CACHE_SLOTS 1024
int  modes_resolver_get_cache(const modes_resolver *r, uint32_t cache[MODES_ICAO_CACHE_SLOTS]);  /* of the tentative run if one is pending */
int  modes_resolver_set_cache(modes_resolver *r, const uint32_t cache[MODES_ICAO_CACHE_SLOTS]);  /* NULL = empty; drops a pending run */
int  modes_resolver_tail_cache(const modes_resolver *r, const modes_candidate *candidates, const modes_tile *tiles,
                               size_t n_tiles, int64_t buffer_base, size_t n_tail_tiles, uint32_t cache[MODES_ICAO_CACHE_SLOTS]);
int  modes_resolver_run_tentative(modes_resolver *r, const modes_candidate *candidates, const modes_tile *tiles,
                                  size_t n_tiles, int64_t buffer_base);            /* records must stay valid until commit */
int  modes_resolver_commit(modes_resolver *r, modes_sink_fn sink, void *user);
int  modes_resolver_reset(modes_resolver *r);           /* forget ICAO cache, skip state, statistics */
int  modes_resolver_stats(const modes_resolver *r, modes_stats *out);
int    modes_resolver_set_output(modes_resolver *r, modes_message *out, size_t capacity);   /* like modes_set_output */
size_t modes_resolver_output_count(const modes_resolver *r);

/* decodeModesMessage() on frame bytes (the reference's hex door,
 * decodeHexMessage dump1090.c:2472-2502): CRC, fix and field decode run on the
 * device + resolve path with the context's ICAO cache: the frames see every address the stream
 * decoded so far, and the addresses they announce are seen by the stream's later batches, whether
 * the host or the device (gpu_resolve) resolves them. */
int  modes_decode_frame(modes_ctx *ctx, const uint8_t msg[14], modes_message *out);
/* n frames of 14 bytes each in one launch (device staging is kept by the context); decoded in
 * order, as n calls of modes_decode_frame would. */
int  modes_decode_frames(modes_ctx *ctx, const uint8_t *frames, size_t n, modes_message *out);

/* ---- presentation (SURVEY.md §8(f) item 1) -------------------------------- */
/* The reference's default (non --raw) text for one message: displayModesMessage()
 * (dump1090.c:1314-1450) plus the blank line of useModesMessage() (:1813), byte for byte.
 * check_crc = the --no-crc-check state (it changes one line, :1445).  Returns the length the text
 * needs; at most capacity-1 bytes + NUL are written.  Pure host code. */
size_t modes_format_message(const modes_message *mm, int check_crc, char *buf, size_t capacity);

/* SURVEY.md §8(f) item 2 — the raw TCP wire formats.  Output line of port 30002
 * (modesSendRawOutput, dump1090.c:2381-2393): "*" + UPPERCASE hex + ";\n". */
size_t modes_format_raw_net(const modes_message *mm, char *buf, size_t capacity);
/* Input line of port 30001, the parsing half of decodeHexMessage (dump1090.c:2472-2497).  Returns
 * the number of frame bytes written to msg (0..14; the rest zeroed) or -1 where the reference
 * discards the line.  Feed the bytes to modes_decode_frame() for the decoding half. */
int    modes_parse_hex_line(const char *line, uint8_t msg[14]);

/* ---- SURVEY.md §8(f) item 3 — aircraft tracker, CPR positions, SBS / JSON records -------------
 * The per-aircraft reduce over the delivered message stream that the reference's interactive
 * mode, HTTP map and SBS port share (dump1090.c:1822-2164).  Pure host code, no GPU involved.
 * Time is supplied by the caller in milliseconds: wall clock for a live feed (what the reference
 * uses, time()/mstime()), or stream time for a file: MODES_STREAM_EPOCH_MS + sample_pos / 2000.
 * The epoch matters: a new aircraft's odd/even CPR times start at 0, and the reference pairs two
 * frames when their times differ by <= 10 s (dump1090.c:2122) — with a clock that starts near 0
 * the first position frame of a file would be "paired" with the empty slot and decoded against
 * zeros.  mstime() is ~1.7e12, so the reference never does that; neither does a stream clock
 * that starts at the epoch below. */
#define MODES_STREAM_EPOCH_MS 1000000000000LL
typedef struct modes_tracker modes_tracker;

/* struct aircraft (dump1090.c:112-130) */
typedef struct modes_aircraft {
    uint32_t addr;                  /* ICAO address */
    char     hexaddr[7];            /* "%06x" */
    char     flight[9];
    int32_t  altitude, speed, track;
    int64_t  seen;                  /* seconds: now_ms / 1000 at the last message (time(NULL) in the reference) */
    int64_t  messages;
    int32_t  odd_cprlat, odd_cprlon, even_cprlat, even_cprlon;
    double   lat, lon;
    int64_t  odd_cprtime, even_cprtime;   /* ms (mstime() in the reference) */
} modes_aircraft;

/* check_crc: messages with crcok == 0 are ignored when set (dump1090.c:2073). */
modes_tracker *modes_tracker_create(int check_crc);
void   modes_tracker_destroy(modes_tracker *t);
/* interactiveReceiveData() (dump1090.c:2069-2164) incl. decodeCPR (:1952-1988), decodeCPRSurface
 * (:2004-2052), decodeMovementField (:2056-2066) and the receiver reference position.  Returns
 * the aircraft (valid until the next expire/destroy) or NULL when the message is ignored. */
const modes_aircraft *modes_tracker_update(modes_tracker *t, const modes_message *mm, int64_t now_ms);
size_t modes_tracker_count(const modes_tracker *t);
/* The aircraft in the reference's list order: most recently created first (dump1090.c:2080-2083). */
size_t modes_tracker_list(const modes_tracker *t, modes_aircraft *out, size_t capacity);
/* interactiveRemoveStaleAircrafts() (dump1090.c:2205-2229): drops aircraft not heard for more than
 * ttl_seconds; returns how many were removed. */
size_t modes_tracker_expire(modes_tracker *t, int64_t now_ms, int ttl_seconds);
/* Receiver reference position (running mean of decoded airborne positions, dump1090.c:2127-2141). */
void   modes_tracker_reference(const modes_tracker *t, double *lat, double *lon, int *count);
/* aircraftsToJson() (dump1090.c:2505-2551).  Returns the length needed; writes at most capacity-1 bytes + NUL. */
size_t modes_tracker_format_json(const modes_tracker *t, int metric, char *buf, size_t capacity);
/* The interactive-mode screen, interactiveShowData() (dump1090.c:2167-2199): clear-screen sequence,
 * header with the activity dot, one row per aircraft up to max_rows.  Same length convention. */
size_t modes_tracker_format_table(const modes_tracker *t, int metric, int max_rows, int64_t now_ms, char *buf, size_t capacity);
/* One SBS (BaseStation, port 30003) line for a message and its aircraft, modesSendSBSOutput()
 * (dump1090.c:2396-2446), newline included.  Returns the length needed, 0 for message types that
 * produce no line. */
size_t modes_format_sbs(const modes_message *mm, const modes_aircraft *a, char *buf, size_t capacity);
/* cprNLFunction (dump1090.c:1869-1931), exposed for tests. */
int    modes_cpr_nl(double lat);

/* ---- plumbing ----------------------------------------------------------- */
void *modes_stream(modes_ctx *ctx);                    /* the cudaStream_t modes_detect_device launches on */
int   modes_set_stream(modes_ctx *ctx, void *cuda_stream);   /* use the caller's stream for it (NULL: own) */
/* Device memory that other ranks on the same node can write into (CUDA IPC): rank 0 of a
 * multi-GPU job allocates the gather buffer with modes_device_alloc, exports it, and every other
 * rank maps it and passes its segment as d_candidates / d_tiles of modes_detect_device, so the
 * frame-evaluation kernel stores its records straight into rank 0's HBM over NVLink — the record
 * gather is fused into the kernel instead of following it as a collective. */
void *modes_device_alloc(size_t nbytes);
void  modes_device_free(void *p);
int   modes_ipc_export(const void *dptr, uint8_t handle[64]);
void *modes_ipc_open(const uint8_t handle[64]);          /* on the importing rank's current device */
int   modes_ipc_close(void *mapped);
int   modes_copy_to_host(void *dst_host, const void *src_device, size_t nbytes);   /* synchronous */
int   modes_device_memset(void *dst_device, int value, size_t nbytes);            /* synchronous */
/* Queue a device-to-device copy of the last modes_detect_device's counters {found, overflow,0,0}
 * (16 bytes) to `dst` (may be peer memory) on the detect stream. */
int   modes_detect_publish_count(modes_ctx *ctx, void *dst);
void *modes_host_alloc(size_t nbytes);                 /* pinned host memory for modes_process input */
void  modes_host_free(void *p);
/* cfg.profile: mean device time (CUDA events on the launching stream) per batch
 * since the previous call: [0] scan kernel (magnitude+preamble), [1] frame
 * evaluation kernel, [2] both, [3] number of batches averaged. */
int  modes_get_kernel_times(modes_ctx *ctx, float ms[4]);
/* Cumulative count of kernel launches issued by this context. */
uint64_t modes_launch_count(const modes_ctx *ctx);
/* How host threads wait for the GPU, process-wide (contexts read it when they are created).
 * 0 (default): the CUDA runtime's choice — on a many-core host it spins: lowest latency, one core
 * busy per waiting thread.  1: sleep until the GPU signals (cudaEventBlockingSync): for hosts that
 * run more GPU processes than they have cores to spare (e.g. one process per GPU under a small
 * container CPU quota).  The environment variable MODES_HOST_WAIT=block sets the initial value.
 * The helper threads that build message structs are sized from the CPUs this process may really
 * use (affinity mask cut down to the cgroup CPU quota); MODES_BUILD_THREADS=<n> overrides, e.g.
 * quota / ranks for several processes on one host. */
int  modes_set_host_wait(int mode);
/* Entries of the tile table of a batch of n_buffers reference buffers. */
size_t modes_tile_count(size_t n_buffers);

/* ---- many receivers on one GPU (SURVEY.md 8(f) item 4: batch across receivers, not across time) ----
 * One dump1090 process serves one RTL-SDR: rtlsdrCallback (dump1090.c:442-456) fills one buffer of
 * 131072 samples at a time, readDataFromFile/rtlsdrCallback prefix it with the last 238 samples of the
 * previous one (:481-485), and detectModeS keeps ONE address cache, skip state and set of statistics.
 * A pool keeps all of that per receiver for many independent 2 MHz streams and decodes one buffer of each
 * of them in ONE batch on the device (csrc/modes_pool.cpp: each buffer rides behind a resident pad buffer
 * whose tail is that receiver's carry, so the kernels are the single-stream ones).  Messages of a
 * receiver are delivered in its stream order with sample_pos counted in its own stream; receivers are
 * served in the order they are listed.  Every receiver's output equals a modes_ctx fed that receiver's
 * buffers alone. */
typedef void (*modes_pool_sink_fn)(void *user, uint32_t receiver, const modes_message *mm);
/* max_batch_receivers: most receivers one modes_pool_ingest call names (0: n_receivers); sizes the
 * resident batch (2 x 256 KiB per receiver).  No device is touched before the first modes_pool_ingest. */
modes_pool *modes_pool_create(const modes_config *cfg, size_t n_receivers, size_t max_batch_receivers);
void        modes_pool_destroy(modes_pool *p);
const char *modes_pool_last_error(const modes_pool *p);
/* iq[i]: the next MODES_BUFFER_BYTES of receiver receivers[i] (host memory, pinned for full speed); a
 * receiver may be named once per call and need not be named in every call. */
int  modes_pool_ingest(modes_pool *p, const uint32_t *receivers, const uint8_t *const *iq, size_t n,
                       modes_pool_sink_fn sink, void *user);
/* The two halves of modes_pool_ingest, for overlap: submit uploads the buffers and launches the kernels
 * and returns without waiting (the buffers must stay valid until the batch is collected); collect waits
 * for the OLDEST submitted batch, resolves it and delivers its messages.  Two batches may be in flight:
 *     submit(k+1); collect(k);      -- batch k+1 crosses PCIe and is scanned while batch k is resolved
 * A receiver may be named in both. */
int  modes_pool_submit(modes_pool *p, const uint32_t *receivers, const uint8_t *const *iq, size_t n);
int  modes_pool_collect(modes_pool *p, modes_pool_sink_fn sink, void *user);
/* modes_pool_submit / modes_pool_ingest for buffers in device memory of the pool's device (cfg.device): a CUDA
 * SDR front end, a GPU ingest of remote feeds or a torch pipeline feeds its receivers without a copy through
 * the host.  d_iq[i] is what iq[i] is for a host-fed call: MODES_BUFFER_BYTES for a UC8 receiver, twice that
 * for an SC16 or SC16Q11 one, at either input rate.
 *   Same output: the same messages and every field, sample_pos, statistics, modes_pool_buffers, and level,
 *     spectrum, recovery and weak records as host-fed calls of the same bytes in the same calls, with every
 *     switch and with two batches in flight.
 *   The bytes must be fully written before the call, which does not order itself after the caller's
 *     streams, and must not change until the matching modes_pool_collect returns (as a host-fed buffer).
 *   One kind of memory per receiver: from its first call until modes_pool_reset a receiver is fed either by
 *     host-fed calls or by device-fed calls; naming it in a call of the other kind is refused ("in progress").
 *   Refused, with a message naming the receiver: a NULL pointer, a buffer that is not 16-byte aligned, and
 *     memory that cudaPointerGetAttributes does not report as device memory of cfg.device (host, pinned,
 *     managed, or another device's).
 * The 2 MHz receivers' carries then live on the device (2 x 476 bytes per receiver of the pool, made on
 * the first device-fed call); host-fed calls make none of it. */
int  modes_pool_submit_device(modes_pool *p, const uint32_t *receivers, const void *const *d_iq, size_t n);
int  modes_pool_ingest_device(modes_pool *p, const uint32_t *receivers, const void *const *d_iq, size_t n,
                              modes_pool_sink_fn sink, void *user);
/* Ends the streams of the listed receivers: tails[i] holds tail_bytes[i] more bytes of receiver receivers[i]'s
 * stream (0 up to its buffer size: MODES_BUFFER_BYTES for a UC8 receiver, twice that for a 16-bit one), after
 * which its stream ends as modes_finish ends one.  A finite capture of any length is fed as its whole buffers
 * (modes_pool_submit / _ingest) and then its tail; a capture shorter than one buffer is a tail alone.
 *   Same output: after it, everything the pool has delivered for a receiver (messages and every field,
 *     sample_pos, signal, arrival and carrier, statistics, recovery and weak statistics, level and spectrum
 *     records, modes_pool_buffers) equals modes_process + modes_finish of a single-stream context with the same
 *     modes_config, rate, format, shift and switches on all the bytes the receiver was given.  cfg.drop_eof_buffer
 *     takes effect here: the EOF buffer is decoded (127 past the stream's end, its level record counting the real
 *     samples only) unless it is set.
 *   Synchronous, like modes_pool_ingest, and refused while a submitted batch is in flight.  It runs as at most
 *     two batches: first the whole 2 MHz buffers the tails complete (at 2 MHz a tail of a whole buffer, at
 *     2.4 MS/s the buffer whose filter lookahead had not arrived), then the EOF buffers.  Messages go to the sink
 *     and the output array batch by batch, each batch's in list order; each receiver's are in its stream order.
 *   Refused as modes_pool_ingest refuses (a receiver out of range or listed twice, more than max_batch
 *     receivers, a receiver fed from the other kind of memory), and for a tail longer than the receiver's buffer,
 *     a NULL tail of more than 0 bytes, and a receiver already finished.  Afterwards the receiver is finished:
 *     modes_pool_submit* and modes_pool_finish* naming it, and its rate and format setters, are refused until
 *     modes_pool_reset starts a new stream.  A receiver never fed may be finished (a capture shorter than a buffer).
 *   Staging: each tail is copied into a whole buffer padded with 127 (pinned host memory for modes_pool_finish,
 *     device memory for modes_pool_finish_device, one buffer of its format per listed receiver, kept for later
 *     calls). */
int  modes_pool_finish(modes_pool *p, const uint32_t *receivers, const uint8_t *const *tails, const size_t *tail_bytes,
                       size_t n, modes_pool_sink_fn sink, void *user);
/* The same with the tails in device memory of cfg.device, for receivers fed by modes_pool_submit_device (or never
 * fed): each is copied on the device, so it may end anywhere in its allocation; refused as a device-fed buffer is
 * (NULL, not 16-byte aligned, not device memory of cfg.device). */
int  modes_pool_finish_device(modes_pool *p, const uint32_t *receivers, const void *const *d_tails,
                              const size_t *tail_bytes, size_t n, modes_pool_sink_fn sink, void *user);
/* The host half alone, for candidate records produced elsewhere over a batch laid out as the pool lays
 * it out: buffer 2i = pad buffer of receivers[i] (no signal, last MODES_CARRY_BYTES = its carry), buffer
 * 2i+1 = its new buffer; candidates/tiles as modes_detect_fetch returns them for those 2n buffers.  The
 * buffers are 2 MHz buffers whatever the receivers' input rates. */
int  modes_pool_resolve(modes_pool *p, const uint32_t *receivers, size_t n, const modes_candidate *candidates,
                        const modes_tile *tiles, modes_pool_sink_fn sink, void *user);
/* Like modes_set_output: messages are ALSO written to a caller-owned array, all receivers' in delivery
 * order, receiver_of[k] naming the receiver of out[k]; the count keeps running past capacity, calling
 * it again restarts the array.  NULL, NULL, 0 turns it off.  The sink may then be NULL. */
int    modes_pool_set_output(modes_pool *p, modes_message *out, uint32_t *receiver_of, size_t capacity);
size_t modes_pool_output_count(const modes_pool *p);
int  modes_pool_stats(const modes_pool *p, uint32_t receiver, modes_stats *out);
int  modes_pool_reset(modes_pool *p, uint32_t receiver);        /* the receiver starts a new stream */
int64_t modes_pool_buffers(const modes_pool *p, uint32_t receiver);   /* buffers of it decoded so far */

/* ---- signal level and the Beast binary feed ----------------------------------------------------
 * Signal measurement is off by default.  When it is on, every batch submitted afterwards runs one
 * more kernel after frame evaluation, which writes modes_frame_eval.signal for every decoded
 * attempt; delivered messages carry it in modes_message.signal.  It is always measured on the
 * uncorrected samples, also for a phase-corrected retry.  Messages from the hex door have no
 * samples and keep signal = 0.  On an n_gpus > 1 context the setting reaches every GPU; a pool
 * applies it to all its device contexts.  Returns 0, or -1 for a NULL handle. */
int    modes_set_signal(modes_ctx *ctx, int on);
int    modes_pool_set_signal(modes_pool *p, int on);
/* One Beast frame for a message: 0x1a, '2' (7-byte frame) or '3' (14-byte frame), a 6-byte big-endian
 * 12 MHz timestamp = (6 * sample_pos) mod 2^48 (0 when sample_pos < 0) when arrival = 0, and
 * max(6 * sample_pos + arrival - 8, 0) mod 2^48 otherwise (modes_set_arrival), one signal byte
 * = min(255, (signal * 255 + 32767) / 65535), then the frame bytes; every 0x1a after the leading one
 * is doubled.  sample_pos counts the samples of one stream (of one receiver in a pool), so each
 * stream's clock is its own.  Returns the length the frame needs (at most 44); writes at most
 * capacity bytes and no terminating NUL.  Pure host code. */
size_t modes_format_beast(const modes_message *mm, uint8_t *buf, size_t capacity);

/* ---- arrival time to a sixth of a sample (multilateration-grade Beast timestamps) -------------
 * The Beast timestamp of a frame is 6 * sample_pos 12 MHz ticks: the preamble's sample, 500 ns coarse.
 * A pulse that starts d samples after a sample boundary puts about (1 - d) of its amplitude into that
 * sample and d into the next one, so the decoded frame's samples tell d.  For a decoded attempt
 * (MODES_EVAL_DECODED) of b bits (56 or 112, from msgtype) at buffer position j, with its frame bits
 * = its msg after any CRC fix and m = the reference's uncorrected magnitudes (dump1090.c:359-364):
 *   1. e = the nominal pulse pattern over the samples j .. j+17+2b: preamble pulses at 0, 2, 7 and 9;
 *      bit i puts a pulse at 16+2i when it is 1 and at 17+2i when it is 0; every other sample is empty.
 *   2. Every sample s in j+1 .. j+16+2b is classified by (e[s-1], e[s], e[s+1]):
 *        main (0,1,0), late (1,0,0), early (0,0,1), quiet (0,0,0); any other sample is not used.
 *      Every class is non-empty (the preamble alone has 3 main, 2 late, 1 early, 6 quiet samples).
 *   3. With mu = mean of m over quiet:  A = mean(main) - mu,  L = max(mean(late) - mu, 0),
 *      E = max(mean(early) - mu, 0).
 *   4. offset = round(6 (L - E) / (A + L + E)) ticks, halves rounded away from zero, clamped to
 *      [-7, 7]; the frame is not measured when A + L + E <= 0.  It is computed exactly in 64-bit
 *      integers from the class sums and counts (csrc/modes_arrival_core.cuh).
 * The code is 0 (not measured) or offset + 8 (1..15) and sits in bits 4-7 of modes_frame_eval.flags;
 * delivered messages carry it in modes_message.arrival.  The arrival of the frame is then
 * 6 * sample_pos + offset ticks.  Recovered messages (modes_message.recovered != 0) and frames from the
 * hex door are not measured (arrival = 0) and keep the coarse timestamp.
 *
 * Arrival measurement is off by default.  When it is on, every batch submitted afterwards runs the
 * signal pass's kernel (one more launch per batch when signal measurement is off, none more when it is
 * on).  On an n_gpus > 1 context the setting reaches every GPU; a pool applies it to all its device
 * contexts.  Returns 0, or -1 for a NULL handle. */
int    modes_set_arrival(modes_ctx *ctx, int on);
int    modes_pool_set_arrival(modes_pool *p, int on);

/* ---- carrier frequency of each message ------------------------------------------------------------
 * Where in frequency a frame arrived, relative to the centre of the 2 MHz bytes the scan reads: the median
 * over many aircraft is the receiver's own tuning error (its crystal error in ppm of 1090 MHz), a 4-10 MS/s
 * capture's offset shows whether modes_set_input_offset was right, and a frame far from its aircraft's usual
 * offset stands out.  For a decoded attempt (MODES_EVAL_DECODED) at buffer position j with b bits (56 or 112,
 * from msgtype), its frame bits = its msg after any CRC fix:
 *   1. The pulse sample of bit i is j+16+2i when the bit is 1 and j+17+2i when it is 0; the preamble's
 *      pulses are at j+0, 2, 7 and 9.
 *   2. The pairs are the pulse samples exactly two samples (1 us) apart: the preamble pairs (0, 2) and
 *      (7, 9), and the pulses of each two consecutive bits of equal value.
 *   3. With z = (I - 127) + i (Q - 127) of the 2 MHz bytes (resampled, decimated, shifted or converted on
 *      the other input paths), the record of the attempt is the sum of z_later conj(z_earlier) over the
 *      pairs:  re = sum (Ia Ib + Qa Qb),  im = sum (Ia Qb - Qa Ib)  (a the earlier sample), in int32.
 * The host converts the delivered attempt's record to f = atan2(im, re) / (2 pi 1 us), unambiguous within
 * +-500 kHz, and to the code 16384 + round(f / 100 Hz) (halves away from zero) in modes_message.carrier; a
 * frame above the centre of the bytes has f > 0.  The code is 0 (not measured) with the switch off, for
 * re = im = 0, for recovered messages and for frames from the hex door.  csrc/modes_carrier_core.cuh has
 * the arithmetic.
 *
 * Carrier measurement is off by default.  When it is on, every batch submitted afterwards runs the signal
 * pass's kernel (one more launch per batch when signal and arrival measurement are off, none more when one
 * is on), which writes one modes_carrier record per candidate to device memory; the records are copied to
 * the host beside the candidate records.  On an n_gpus > 1 context the setting reaches every GPU; a pool
 * applies it to all its device contexts.  It cannot be combined with gpu_resolve, whose delivery records
 * have no room for it.  Returns 0, or -1 for a NULL handle or with gpu_resolve. */
typedef struct modes_carrier {
    int32_t re[2], im[2];       /* the record of pass[k]; 0, 0 for an attempt not decoded */
} modes_carrier;
int    modes_set_carrier(modes_ctx *ctx, int on);
int    modes_pool_set_carrier(modes_pool *p, int on);

/* ---- receiver levels: noise floor, peak and clipping per buffer --------------------------------
 * What an operator reads of a receiver besides its messages: how loud the channel is, how close the
 * strongest samples come to full scale, and whether the ADC clips (gain too high).  One record per
 * reference buffer decoded, over the buffer's own samples (the 238 it carries over belong to the
 * buffer before it, so every stream sample is counted once), with m = the reference's magnitude
 * round(360 * sqrt((I-127)^2 + (Q-127)^2)) (dump1090.c:359-364, :1454-1469), m <= 65167.
 * Every field is an integer, so records do not depend on the order of the GPU's reduction.
 * On the scale of modes_message.signal (so that SNR = signal dB - noise dB):
 *     noise dBFS = 10 log10(sum sum_power / sum n_samples / 65535^2)
 *     peak dBFS  = 20 log10(max peak / 65535)
 *     clipped fraction = sum clipped / sum n_samples */
typedef struct modes_level {
    int64_t  buffer;            /* stream index of the buffer (in a pool: the receiver's own buffer index) */
    uint32_t n_samples;         /* stream samples in it: MODES_BUFFER_SAMPLES, fewer only in the EOF buffer
                                   (a trailing odd byte counts as a sample); the EOF padding adds nothing */
    uint32_t clipped;           /* samples whose I or Q byte is 0 or 255 */
    uint64_t sum_mag;           /* sum of m */
    uint64_t sum_power;         /* sum of m^2 */
    uint32_t peak;              /* max m, 0 for a buffer without signal */
    uint32_t pad;
} modes_level;

/* Level measurement is off by default.  When it is on, every batch the streaming decode submits
 * afterwards runs one more kernel over its buffers in HBM (one more launch per batch), and the
 * records are queued on the context in stream order: one per buffer decoded, none for an EOF buffer
 * dropped by drop_eof_buffer, n_samples = 0 for an all-padding EOF buffer that is decoded.  On an
 * n_gpus > 1 context the setting reaches every GPU.  modes_reset drops the queue.
 * modes_take_levels moves the oldest min(cap, queued) records to out and returns how many it moved;
 * with out = NULL it moves nothing and returns how many are queued.  Returns 0 / -1 (NULL handle). */
int    modes_set_levels(modes_ctx *ctx, int on);
size_t modes_take_levels(modes_ctx *ctx, modes_level *out, size_t cap);
/* Stage level: records of n_buffers whole buffers in device memory, buffer k at d_iq + k * stride_bytes
 * (16-byte aligned; stride 0 = MODES_BUFFER_BYTES), queued on the context's stream without waiting.
 * modes_levels_fetch waits and copies the n_buffers records of the last call to out in call order,
 * with buffer = k and n_samples = MODES_BUFFER_SAMPLES.  Independent of modes_set_levels. */
int    modes_levels_device(modes_ctx *ctx, const void *d_iq, size_t n_buffers, size_t stride_bytes);
int    modes_levels_fetch(modes_ctx *ctx, modes_level *out);
/* The pool measures the data buffers of every batch submitted while the switch is on (never the pad
 * buffers) and queues each receiver's records, buffer = the receiver's own buffer index, in its stream
 * order; modes_pool_reset clears the receiver's queue.  Same take convention as above. */
int    modes_pool_set_levels(modes_pool *p, int on);
size_t modes_pool_take_levels(modes_pool *p, uint32_t receiver, modes_level *out, size_t cap);

/* ---- input spectrum: where in frequency each buffer's input energy is --------------------------
 * The frequency-domain sibling of the levels above: where 1090 MHz sits in a capture (the offset to pass
 * modes_set_input_offset), where a zero-IF radio's DC spike is, whether an interferer or an image sits on
 * the channel, whether a 16-bit shift throws away the weak end.  One record per reference buffer decoded,
 * measured on the input it stands for, before resampling, decimation and the input offset; it changes no
 * message.  Exactly, in integers (modes_spectrum_core.cuh has the arithmetic):
 *   span     buffer b (2 MHz samples [b B, (b + 1) B), B = MODES_BUFFER_SAMPLES) stands for the input samples
 *            [s_b, s_{b+1}), s_b = floor(in b B / out) at the rate's ratio out : in (1:1 at 2000000, 5:6 at
 *            2400000, 1:M at 2000000 M); its F = floor((s_{b+1} - s_b) / 256) whole frames of 256 input
 *            samples start at s_b (F = 512, 614 and 512 M); the remainder is not measured
 *   sample   xi = I - 127, xq = Q - 127 of the UC8 bytes, a 16-bit stream's converted bytes (so a shift that
 *            clips or loses the weak end shows); samples past the stream's end are 0; no input offset
 *   window   v = (x w[n] + 8192) >> 14 (int32, arithmetic shift), w[n] = (16384 - C[4 n]) >> 1, a Q14 Hann
 *   FFT      radix-2 decimation in time over the bit-reversed frame, int32, no scaling; the butterfly of
 *            stage s = 0..7 (half = 2^s) on a = X[i], b = X[i + half] with k = (i mod half) 2^(7-s),
 *            c = C[4 k], s = S[4 k]:  t_re = (b_re c + b_im s + 8192) >> 14, t_im = (b_im c - b_re s + 8192) >> 14,
 *            X[i] = a + t, X[i + half] = a - t  (C, S: the 1024-phase tables of modes_set_input_offset)
 *   power    X_re^2 + X_im^2 as uint32 (|X| < 46400, so it fits), summed over the F frames in uint64
 *   record   power[i] = the sum of FFT bin (i + 128) mod 256: natural frequency order, bin i at
 *            (i - 128) fs / 256 Hz, bin 128 at DC
 * Off by default.  When it is on, every batch the streaming decode submits afterwards runs one more kernel
 * (one more launch per batch), on the same stream after the scan, over the input bytes already in HBM; the
 * records are queued as level records are: in stream order, one per buffer decoded (the EOF buffer's too,
 * unless drop_eof_buffer drops it), merged in stream order on an n_gpus > 1 context, dropped by modes_reset.
 * Same take convention as modes_take_levels.  Returns 0 / -1 (NULL handle). */
#define MODES_SPECTRUM_BINS 256
typedef struct modes_spectrum {
    int64_t  buffer;            /* stream index of the buffer (in a pool: the receiver's own buffer index) */
    uint32_t frames;            /* F */
    uint32_t pad;
    uint64_t power[MODES_SPECTRUM_BINS];
} modes_spectrum;
int    modes_set_spectrum(modes_ctx *ctx, int on);
size_t modes_take_spectra(modes_ctx *ctx, modes_spectrum *out, size_t cap);
/* The pool measures every buffer a receiver decodes while the switch is on, on the receiver's own input
 * (a 16-bit receiver's converted bytes), and queues its records under its own buffer index; its records
 * equal the single-stream decoder's for the receiver's stream.  modes_pool_reset clears the receiver's queue. */
int    modes_pool_set_spectrum(modes_pool *p, int on);
size_t modes_pool_take_spectra(modes_pool *p, uint32_t receiver, modes_spectrum *out, size_t cap);

/* ---- soft-decision recovery of weak DF17/DF18 frames of known aircraft -------------------------
 * Many weak frames pass the preamble test and fail the CRC because a few bits whose two half-bit
 * samples were nearly equal were sliced the wrong way.  The recovery pass asks which bits were
 * doubtful.  For a candidate at buffer position j, with the uncorrected magnitudes
 * a_i = m[j+16+2i], c_i = m[j+17+2i] (i < 112; dump1090.c:359-364, :1670-1671):
 *     hard bit b_i = a_i > c_i (a tie gives 0), confidence w_i = |a_i - c_i|
 *     only DF = b_0..b_4 in {17, 18} is searched (extended squitters: the parity must be exactly 0)
 *     s0 = the 24-bit syndrome of the 112 hard bits (dump1090.c:733-742)
 *     P  = the MODES_RECOVER_BITS positions in [5, 112) with the smallest (w_i, i); the DF is never flipped
 *     every subset S of P with XOR of the single-bit syndromes over S == s0 solves the frame:
 *       FOUND      one solution of least |S| (S may be empty): msg = the hard frame with S flipped, nflips = |S|
 *       AMBIGUOUS  two or more solutions share the least |S| (msg = the hard frame, nflips = that |S|)
 *       NOT_FOUND  no subset solves it (msg = the hard frame, nflips = 0)
 *     signal = floor(sqrt(floor(sum max(a_i, c_i)^2 / 112))) (the signal level of a long frame)
 * Candidates with another DF get status INELIGIBLE, the hard frame, nflips 0 and the signal.
 *
 * What is delivered is decided in stream order by the host resolve.  A recovered message is
 * delivered at candidate c (buffer b, position j) iff
 *   1. the reference's walk visits c (it is not inside a message the reference took),
 *   2. neither attempt at c was judged crcok (with check_crc = 0 the reference's crcok = 0
 *      deliveries at c come first),
 *   3. c is not within 241 positions after an earlier recovered message of the same buffer,
 *   4. its status is FOUND,
 *   5. its address (msg[1..3]) is in the ICAO address cache at that point (recovered messages never
 *      write the cache: an aircraft with no clean frame yet gets none), and
 *   6. the reference delivers no crcok message in the same buffer at j' with j < j' < j + 241
 *      (the same frame decoded a sample later).
 * It carries crcok = 1, crc = 0, errorbit = -1, phase_corrected = 0, iid = 0, nfixed = nflips,
 * recovered = 1, the fields of the frame, and signal = the record's signal when signal measurement
 * is on (0 otherwise).  The reference's messages and its eight statistics are unchanged.
 * Recovered messages are not the reference's: they are frames it does not decode. */
#define MODES_RECOVER_BITS 10
enum { MODES_RECOVER_INELIGIBLE = 0, MODES_RECOVER_FOUND = 1, MODES_RECOVER_AMBIGUOUS = 2, MODES_RECOVER_NOT_FOUND = 3 };

/* One record per candidate, at the candidate's index in the record array. */
typedef struct modes_recovered {
    uint8_t  msg[14];           /* the repaired frame if FOUND, otherwise the hard frame */
    uint8_t  status;            /* MODES_RECOVER_* */
    uint8_t  nflips;
    uint16_t signal;
    uint8_t  pad[2];
} modes_recovered;

typedef struct modes_recovery_stats {
    int64_t considered;         /* rules 1-2 hold and the DF is 17 or 18 */
    int64_t found;              /* of those, outside an earlier recovered message's span (rule 3) and FOUND */
    int64_t ambiguous;          /* ... and AMBIGUOUS */
    int64_t unknown_address;    /* FOUND, address not in the cache (rule 5) */
    int64_t dropped;            /* passed rules 1-5, dropped by rule 6 */
    int64_t delivered;
} modes_recovery_stats;

/* Recovery is off by default.  When it is on, every batch the streaming decode submits afterwards
 * runs one more kernel after frame evaluation (one more launch per batch), its records come back
 * with the candidate records, and the host resolve applies the rules above.  On an n_gpus > 1
 * context the setting reaches every GPU.  It cannot be combined with gpu_resolve = 1: the call then
 * fails and leaves the context as it was.  modes_reset clears the statistics. */
int    modes_set_recovery(modes_ctx *ctx, int on);
int    modes_get_recovery_stats(const modes_ctx *ctx, modes_recovery_stats *out);
/* Stage level: the records of the batch and candidate records of the last modes_detect_device /
 * _host call, queued on the context's stream after it without waiting.  d_out: capacity records in
 * device memory, or NULL for the context's own buffer, read with modes_recover_fetch (which waits
 * and copies as many records as modes_detect_wait reports).  Records beyond the capacity of either
 * array are not written. */
int    modes_recover_device(modes_ctx *ctx, void *d_out, size_t capacity);
int    modes_recover_fetch(modes_ctx *ctx, modes_recovered *out);
/* The host resolve with the rules above: recovered[k] belongs to candidates[k] (NULL: exactly
 * modes_resolver_run).  The records' signal is delivered as it is.  Batches must end at buffer
 * boundaries, as every decode path's do. */
int    modes_resolver_run_recovered(modes_resolver *r, const modes_candidate *candidates, const modes_recovered *recovered,
                                    const modes_tile *tiles, size_t n_tiles, int64_t buffer_base, modes_sink_fn sink, void *user);
/* modes_resolver_run_shards with recovery records, recovered[k][i] belonging to candidates[k][i]
 * (recovered = NULL: exactly modes_resolver_run_shards); the same as running the shards one by one
 * with modes_resolver_run_recovered. */
int    modes_resolver_run_shards_recovered(modes_resolver *r, size_t n_shards, const modes_candidate *const *candidates,
                                           const modes_recovered *const *recovered, const modes_tile *const *tiles,
                                           const size_t *n_tiles, const int64_t *buffer_base, modes_sink_fn sink, void *user);
int    modes_resolver_recovery_stats(const modes_resolver *r, modes_recovery_stats *out);
/* The pool: recovery for every batch submitted while the switch is on; statistics per receiver,
 * cleared by modes_pool_reset. */
int    modes_pool_set_recovery(modes_pool *p, int on);
int    modes_pool_recovery_stats(const modes_pool *p, uint32_t receiver, modes_recovery_stats *out);

/* ---- recovery at weak preambles ------------------------------------------------------------------
 * The recovery above only searches positions that passed the reference's preamble test, and at low
 * SNR that test rejects most weak frames before their bits are looked at.  A WEAK PREAMBLE is a
 * buffer position j in [0, 131070) (the positions the reference scans, dump1090.c:1593) where, with
 * m_x = m[j+x] (magnitudes of dump1090.c:359-364),
 *   1. the pulse shape holds: m0 > m1, m2 > m1, m7 > m8, m9 > m8,
 *   2. the mean pulse is more than twice the mean quiet sample:
 *        7 (m0+m2+m7+m9) > 8 (m4+m5+m6+m11+m12+m13+m14)
 *      (samples 1, 3, 8 and 10 are left out: a late pulse leaks into them),
 *   3. the hard DF is 17 or 18: b_i = m[16+2i] > m[17+2i], i < 5, and
 *   4. the reference's preamble test (dump1090.c:1602-1650, the "high" tests included) FAILS there,
 *      so weak positions and candidates are disjoint.
 * Every weak position gets the recovery record of a candidate at the same position (the same search,
 * the same modes_recovered record).  In the host resolve, the weak positions are merged into the
 * reference's walk in stream order.  A weak position (buffer b, j) starts the buffer's skip state like a
 * candidate does, is visited iff j is not inside a message the reference took (rule 1), and then goes
 * through rules 3-6 above as a candidate without a good attempt.  It shares the recovered-span skip
 * (rule 3) and the rule-6 drop with the candidates' recoveries.  It never changes the reference's
 * statistics or the address cache.
 * Messages delivered from weak positions carry recovered = 2 and otherwise the fields of recovered
 * messages.  Their statistics are kept apart: considered = weak positions visited, then found /
 * ambiguous / unknown_address / dropped / delivered as above; the recovery statistics keep counting
 * candidates only. */

/* Off by default, effective only while recovery is on: every batch the streaming decode submits
 * afterwards runs four more kernels (the weak-preamble scan, two that put its positions in stream order,
 * and the search over them), one more copy brings the positions and records back, and the resolve
 * merges them.  On an n_gpus > 1
 * context the setting reaches every GPU.  Refused (and the context left as it was) with gpu_resolve = 1.
 * modes_reset clears the statistics. */
int    modes_set_weak_preambles(modes_ctx *ctx, int on);
int    modes_get_weak_recovery_stats(const modes_ctx *ctx, modes_recovery_stats *out);
/* Stage level: the weak positions of the batch of the last modes_detect_device / _host call, in stream
 * order (t = 131072 * buffer + j, as modes_candidate.t), and their recovery records, queued on the
 * context's stream after it without waiting.  d_pos (u32) and d_rec: capacity entries of device memory
 * each, of which the first min(n, capacity) are written; both NULL: the context's own buffers, which
 * grow to hold every position.  modes_weak_fetch waits and sets *n to the number of weak positions of
 * the batch (which may exceed a caller's capacity); with the context's own buffers it also copies the
 * n positions and records to t and rec (either may be NULL). */
int    modes_weak_device(modes_ctx *ctx, void *d_pos, void *d_rec, size_t capacity);
int    modes_weak_fetch(modes_ctx *ctx, uint32_t *t, modes_recovered *rec, uint64_t *n);
/* modes_resolver_run_recovered with weak positions: weak_t[k] (sorted, t relative to buffer_base as
 * the candidates' t) and weak_rec[k], k < n_weak.  recovered must not be NULL when n_weak > 0.  With
 * n_weak = 0 it is exactly modes_resolver_run_recovered. */
int    modes_resolver_run_weak(modes_resolver *r, const modes_candidate *candidates, const modes_recovered *recovered,
                               const modes_tile *tiles, size_t n_tiles, int64_t buffer_base, const uint32_t *weak_t,
                               const modes_recovered *weak_rec, size_t n_weak, modes_sink_fn sink, void *user);
/* The same over shards (as modes_resolver_run_shards_recovered): weak_t[k], weak_rec[k], n_weak[k] of shard k. */
int    modes_resolver_run_shards_weak(modes_resolver *r, size_t n_shards, const modes_candidate *const *candidates,
                                      const modes_recovered *const *recovered, const modes_tile *const *tiles,
                                      const size_t *n_tiles, const int64_t *buffer_base, const uint32_t *const *weak_t,
                                      const modes_recovered *const *weak_rec, const size_t *n_weak, modes_sink_fn sink,
                                      void *user);
int    modes_resolver_weak_stats(const modes_resolver *r, modes_recovery_stats *out);
/* The pool: weak preambles for every batch submitted while both switches are on; statistics per
 * receiver, cleared by modes_pool_reset. */
int    modes_pool_set_weak_preambles(modes_pool *p, int on);
int    modes_pool_weak_stats(const modes_pool *p, uint32_t receiver, modes_recovery_stats *out);

#ifdef __cplusplus
}
#endif
#endif /* MODES_B200_H */
