"""ctypes binding of include/modes_b200.h — the Python host side of the C ABI.

Mirrors the reference's main-loop contract (dump1090.c:2968-2990): a `Decoder`
is fed raw u8 I/Q bytes and hands back, in stream order, the messages the
reference would pass to useModesMessage() (dump1090.c:1802).  Everything that
computes runs in libmodes_b200.so (CUDA, sm_90a).  There is no CPU fallback:
constructing a Decoder without a usable GPU raises.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from pathlib import Path

import numpy as np

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libmodes_b200.so"

BUFFER_BYTES = 262144
BUFFER_SAMPLES = 131072
CARRY_BYTES = 476
TILE_SAMPLES = 7936                       # MODES_TILE_SAMPLES
ICAO_CACHE_SLOTS = 1024                   # MODES_ICAO_CACHE_SLOTS
STREAM_EPOCH_MS = 1_000_000_000_000      # MODES_STREAM_EPOCH_MS: start of a file's stream clock for the tracker

EVAL_GATE_OK, EVAL_ERRORS, EVAL_DECODED, EVAL_P2_VALID = 1, 2, 4, 8
EVAL_ARRIVAL_SHIFT = 4                    # flags >> 4: arrival code (0 = not measured, else offset + 8 ticks)


class Config(C.Structure):
    _fields_ = [("fix_errors", C.c_int32), ("aggressive", C.c_int32), ("check_crc", C.c_int32),
                ("drop_eof_buffer", C.c_int32), ("device", C.c_int32), ("profile", C.c_int32),
                ("max_batch_bytes", C.c_uint64), ("n_gpus", C.c_int32), ("gpu_resolve", C.c_int32)]


_MSG_A = ("errorbit aa1 aa2 aa3 phase_corrected ca iid metype mesub heading_is_valid heading "
          "aircraft_type fflag tflag raw_latitude raw_longitude").split()
_MSG_B = ("ew_dir ew_velocity ns_dir ns_velocity vert_rate_source vert_rate_sign vert_rate velocity "
          "movement movement_valid ground_track ground_track_valid fs dr um identity altitude unit "
          "nfixed signal").split()


class Message(C.Structure):
    """struct modes_message == fields of struct modesMessage (dump1090.c:211-260)."""
    _fields_ = ([("msg", C.c_uint8 * 14), ("recovered", C.c_uint8), ("arrival", C.c_uint8), ("msgbits", C.c_int32),
                 ("msgtype", C.c_int32), ("crcok", C.c_int32), ("crc", C.c_uint32)]
                + [(n, C.c_int32) for n in _MSG_A]
                + [("flight", C.c_char * 9), ("pad1", C.c_char * 3)]
                + [(n, C.c_int32) for n in _MSG_B]
                + [("sample_pos", C.c_int64)])

    def hex(self) -> str:
        return bytes(self.msg[: self.msgbits // 8]).hex()

    def raw_line(self) -> str:
        """The --raw output line, dump1090.c:1324-1326."""
        return "*" + self.hex() + ";"

    def text(self, check_crc: int = 1) -> str:
        """The reference's default (non --raw) output for this message, dump1090.c:1314-1450."""
        buf = C.create_string_buffer(2048)
        n = lib().modes_format_message(C.byref(self), int(check_crc), buf, 2048)
        return buf.raw[:n].decode("latin1")

    def raw_net_line(self) -> str:
        """The TCP raw-output line (uppercase hex), dump1090.c:2381-2393."""
        buf = C.create_string_buffer(64)
        n = lib().modes_format_raw_net(C.byref(self), buf, 64)
        return buf.raw[:n].decode("latin1")

    def rssi_dbfs(self):
        """Signal level in dB relative to the largest magnitude (20 log10(signal / 65535)), or None
        when it was not measured (signal measurement off, or a frame from the hex door)."""
        return None if self.signal <= 0 else 20.0 * math.log10(self.signal / 65535.0)

    def timestamp_12mhz(self) -> int:
        """The 12 MHz Beast timestamp of this message: 6 * sample_pos, moved by the measured arrival
        offset (arrival - 8 ticks) when arrival != 0 (modes_set_arrival); clamped at 0 and taken
        modulo 2^48 as modes_format_beast writes it."""
        ticks = 6 * int(self.sample_pos) + (int(self.arrival) - 8 if self.arrival else 0)
        return 0 if ticks < 0 else ticks % (1 << 48)

    @property
    def carrier_code(self) -> int:
        """modes_message.carrier (bytes 106-107, the end of pad1): 0 = not measured, otherwise
        16384 + round(f / 100 Hz) for the frame's carrier f relative to the centre of the 2 MHz bytes
        (modes_set_carrier)."""
        return C.c_int16.from_address(C.addressof(self) + CARRIER_OFFSET).value

    def carrier_hz(self):
        """The frame's carrier frequency in Hz above the centre of the 2 MHz bytes the scan read (a
        multiple of 100 Hz within +-500 kHz), or None when it was not measured."""
        code = self.carrier_code
        return None if code == 0 else (code - CARRIER_CODE_ZERO) * CARRIER_STEP_HZ

    def beast(self) -> bytes:
        """The Beast binary frame of this message (modes_format_beast); its timestamp is
        timestamp_12mhz()."""
        buf = (C.c_uint8 * 64)()
        n = lib().modes_format_beast(C.byref(self), buf, 64)
        return bytes(buf[:n])

    def copy(self) -> "Message":
        m = Message()
        C.memmove(C.byref(m), C.byref(self), C.sizeof(Message))
        return m


CARRIER_OFFSET = 106                      # offsetof(modes_message, carrier): the last two bytes of pad1
CARRIER_CODE_ZERO = 16384                 # the carrier code of 0 Hz
CARRIER_STEP_HZ = 100                     # Hz per carrier code
assert C.sizeof(Message) == 200 and Message.pad1.offset == CARRIER_OFFSET - 1


class FrameEval(C.Structure):
    _fields_ = [("msg", C.c_uint8 * 14), ("msgtype", C.c_uint8), ("flags", C.c_uint8),
                ("errorbit", C.c_uint8), ("nfixed", C.c_uint8), ("signal", C.c_uint16), ("crc", C.c_uint32)]


class Candidate(C.Structure):
    _fields_ = [("t", C.c_int64), ("passes", FrameEval * 2)]


class Tile(C.Structure):
    _fields_ = [("offset", C.c_uint32), ("count", C.c_uint32)]


class Stats(C.Structure):
    _fields_ = [("v", C.c_int64 * 8)]


STAT_NAMES = ["valid_preamble", "out_of_phase", "demodulated", "goodcrc", "badcrc", "fixed",
              "single_bit_fix", "two_bits_fix"]

SINK_FN = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(Message))
POOL_SINK_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_uint32, C.POINTER(Message))

CANDIDATE_DTYPE = np.dtype([("t", "<i8"),
                            ("p", [("msg", "u1", 14), ("msgtype", "u1"), ("flags", "u1"), ("errorbit", "u1"),
                                   ("nfixed", "u1"), ("signal", "<u2"), ("crc", "<u4")], 2)], align=True)
TILE_DTYPE = np.dtype([("offset", "<u4"), ("count", "<u4")])
assert CANDIDATE_DTYPE.itemsize == C.sizeof(Candidate) == 56


class Level(C.Structure):
    """struct modes_level: noise, peak and clipping sums of one reference buffer."""
    _fields_ = [("buffer", C.c_int64), ("n_samples", C.c_uint32), ("clipped", C.c_uint32),
                ("sum_mag", C.c_uint64), ("sum_power", C.c_uint64), ("peak", C.c_uint32), ("pad", C.c_uint32)]


LEVEL_DTYPE = np.dtype([("buffer", "<i8"), ("n_samples", "<u4"), ("clipped", "<u4"), ("sum_mag", "<u8"),
                        ("sum_power", "<u8"), ("peak", "<u4"), ("pad", "<u4")])
assert LEVEL_DTYPE.itemsize == C.sizeof(Level) == 40
FULL_SCALE = 65535                        # the dBFS reference of rssi_dbfs() and level_summary()

# struct modes_recovered: one soft-decision recovery record per candidate (modes_set_recovery)
RECOVERED_DTYPE = np.dtype([("msg", "u1", 14), ("status", "u1"), ("nflips", "u1"), ("signal", "<u2"), ("pad", "u1", 2)])
assert RECOVERED_DTYPE.itemsize == 20
RECOVER_BITS = 10                         # MODES_RECOVER_BITS
RECOVER_INELIGIBLE, RECOVER_FOUND, RECOVER_AMBIGUOUS, RECOVER_NOT_FOUND = 0, 1, 2, 3
RECOVERY_STAT_NAMES = ["considered", "found", "ambiguous", "unknown_address", "dropped", "delivered"]


class RecoveryStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in RECOVERY_STAT_NAMES]

    def as_dict(self) -> dict:
        return {n: int(getattr(self, n)) for n in RECOVERY_STAT_NAMES}


def level_summary(records) -> dict:
    """Totals of level records (LEVEL_DTYPE): buffers, n_samples, clipped, and on the scale of
    Message.rssi_dbfs() (so that SNR = signal dB - noise dB)
        noise_dbfs = 10 log10(sum sum_power / sum n_samples / 65535^2)   (mean power)
        peak_dbfs  = 20 log10(max peak / 65535)
        clipped_fraction = sum clipped / sum n_samples
    With no samples the three derived values are None; with no power / a zero peak the dB values are -inf."""
    r = np.asarray(records, dtype=LEVEL_DTYPE)
    n = int(r["n_samples"].astype(np.uint64).sum()) if r.size else 0
    power = int(sum(int(v) for v in r["sum_power"]))
    peak = int(r["peak"].max()) if r.size else 0
    clipped = int(r["clipped"].astype(np.uint64).sum()) if r.size else 0
    out = dict(buffers=int(r.size), n_samples=n, clipped=clipped, noise_dbfs=None, peak_dbfs=None, clipped_fraction=None)
    if n:
        out["noise_dbfs"] = 10.0 * math.log10(power / n / FULL_SCALE ** 2) if power else -math.inf
        out["peak_dbfs"] = 20.0 * math.log10(peak / FULL_SCALE) if peak else -math.inf
        out["clipped_fraction"] = clipped / n
    return out

SPECTRUM_BINS = 256                       # MODES_SPECTRUM_BINS
# struct modes_spectrum: the input power spectrum of one reference buffer (modes_set_spectrum)
SPECTRUM_DTYPE = np.dtype([("buffer", "<i8"), ("frames", "<u4"), ("pad", "<u4"), ("power", "<u8", (SPECTRUM_BINS,))])
assert SPECTRUM_DTYPE.itemsize == 16 + 8 * SPECTRUM_BINS
BAND_HZ = 2_000_000                       # the width spectrum_summary searches: the 2 MHz the decoder keeps


def spectrum_summary(records, input_rate: int) -> dict:
    """What spectrum records (SPECTRUM_DTYPE) of a stream at input_rate say, for an operator:
        freq_hz[i]     = (i - 128) fs / 256, the centre of bin i (bin 128 is DC)
        power_db[i]    = 10 log10(sum power[i] / sum frames), the mean power per frame (-inf where it is 0)
        floor_db       = the median of the mean powers, with the DC bin and its two neighbours (the Hann
                         window's main lobe around DC) replaced by the mean of bins 126 and 130
        dc_excess_db   = 10 log10(mean DC power / mean of bins 126 and 130') (0 when both are 0): a zero-IF
                         radio's DC spike over the spectrum next to it
        band_offset_hz = the centre of the W = floor(256 * 2 MHz / fs) adjacent bins with the most power above
                         the floor (sum of max(mean - floor, 0); bins 127-129 replaced as for the floor; the
                         lowest such band on a tie): where the 2 MHz channel most likely sits, the offset
                         modes_set_input_offset takes
    The band search and the floor are exact integer arithmetic on the sums.  With no frames every derived
    value is None."""
    r = np.asarray(records, dtype=SPECTRUM_DTYPE)
    fs = int(input_rate)
    if fs not in INPUT_RATES:
        raise ValueError(f"{fs} samples/s is not supported {INPUT_RATES}")
    n = SPECTRUM_BINS
    frames = int(r["frames"].astype(np.uint64).sum()) if r.size else 0
    total = [sum(int(v) for v in r["power"][:, i]) for i in range(n)] if r.size else [0] * n
    out = dict(buffers=int(r.size), frames=frames, freq_hz=(np.arange(n) - n // 2) * (fs / n), power_db=None,
               floor_db=None, dc_excess_db=None, band_offset_hz=None)
    if not frames:
        return out
    out["power_db"] = np.array([10.0 * math.log10(t / frames) if t else -math.inf for t in total])
    dc, nb = 2 * total[n // 2], total[n // 2 - 2] + total[n // 2 + 2]
    out["dc_excess_db"] = 0.0 if dc == nb else math.inf if not nb else -math.inf if not dc else 10.0 * math.log10(dc / nb)
    t2 = [2 * t for t in total]                                         # twice the sums: the DC notch exact
    t2[n // 2 - 1: n // 2 + 2] = [nb] * 3
    srt = sorted(t2)
    floor4 = srt[n // 2 - 1] + srt[n // 2]                              # 4 x the median sum
    out["floor_db"] = 10.0 * math.log10(floor4 / 4 / frames) if floor4 else -math.inf
    above = [max(2 * t - floor4, 0) for t in t2]
    w = n * BAND_HZ // fs
    best, at = -1, 0
    for i0 in range(n - w + 1):
        score = sum(above[i0: i0 + w])
        if score > best:
            best, at = score, i0
    out["band_offset_hz"] = (at + (w - 1) / 2 - n // 2) * fs / n
    return out


def carrier_summary(messages) -> dict:
    """What the carrier frequencies of delivered messages (Message.carrier_hz(), modes_set_carrier) say
    about a receiver: the messages measured, the aircraft measured (distinct addresses aa1..aa3 among
    them), each aircraft's median offset in Hz (`per_aircraft`, keyed by the 24-bit address), and the
    receiver's estimate: the median over aircraft of their medians, in Hz (`receiver_hz`) and in ppm of
    1090 MHz (`receiver_ppm`; positive: frames arrive above the centre of the receiver's 2 MHz bytes, so
    its tuning is low).  Transponders scatter around 1090 MHz, so one aircraft says little; the median over
    many is the receiver's own offset.  With no measured message the estimates are None."""
    by_addr: dict[int, list[float]] = {}
    n = 0
    for m in messages:
        hz = m.carrier_hz()
        if hz is None:
            continue
        n += 1
        addr = (int(m.aa1) << 16) | (int(m.aa2) << 8) | int(m.aa3)
        by_addr.setdefault(addr, []).append(hz)
    per = {a: float(np.median(v)) for a, v in sorted(by_addr.items())}
    out = dict(messages=n, aircraft=len(per), per_aircraft=per, receiver_hz=None, receiver_ppm=None)
    if per:
        out["receiver_hz"] = float(np.median(list(per.values())))
        out["receiver_ppm"] = out["receiver_hz"] / 1090.0
    return out


_lib = None

# every symbol include/modes_b200.h declares
EXPORTS = ["modes_abi_version", "modes_default_config", "modes_create", "modes_destroy", "modes_last_error",
           "modes_set_sink", "modes_process", "modes_finish", "modes_reset", "modes_get_stats",
           "modes_compute_magnitude", "modes_detect_device", "modes_detect_host", "modes_detect_wait", "modes_detect_fetch",
           "modes_resolve", "modes_resolver_create", "modes_resolver_destroy", "modes_resolver_run",
           "modes_resolver_run_shards", "modes_resolver_get_cache", "modes_resolver_set_cache", "modes_resolver_tail_cache", "modes_resolver_run_tentative", "modes_resolver_commit", "modes_resolver_reset", "modes_resolver_stats", "modes_resolver_set_output", "modes_resolver_output_count", "modes_decode_frame", "modes_decode_frames", "modes_format_message", "modes_format_raw_net", "modes_parse_hex_line", "modes_stream", "modes_set_stream",
           "modes_set_output", "modes_output_count", "modes_device_alloc", "modes_device_free",
           "modes_ipc_export", "modes_ipc_open", "modes_ipc_close", "modes_copy_to_host", "modes_device_memset",
           "modes_detect_publish_count", "modes_host_alloc",
           "modes_host_free", "modes_get_kernel_times", "modes_launch_count", "modes_tile_count", "modes_set_host_wait",
           "modes_tracker_create", "modes_tracker_destroy", "modes_tracker_update", "modes_tracker_count",
           "modes_tracker_list", "modes_tracker_expire", "modes_tracker_reference", "modes_tracker_format_json",
           "modes_tracker_format_table", "modes_format_sbs", "modes_cpr_nl",
           "modes_pool_create", "modes_pool_destroy", "modes_pool_last_error", "modes_pool_ingest", "modes_pool_resolve",
           "modes_pool_stats", "modes_pool_reset", "modes_pool_buffers", "modes_pool_set_output", "modes_pool_output_count",
           "modes_pool_submit", "modes_pool_collect", "modes_set_signal", "modes_pool_set_signal", "modes_format_beast",
           "modes_set_levels", "modes_take_levels", "modes_levels_device", "modes_levels_fetch",
           "modes_pool_set_levels", "modes_pool_take_levels",
           "modes_set_recovery", "modes_get_recovery_stats", "modes_recover_device", "modes_recover_fetch",
           "modes_resolver_run_recovered", "modes_resolver_run_shards_recovered", "modes_resolver_recovery_stats", "modes_pool_set_recovery",
           "modes_pool_recovery_stats", "modes_set_weak_preambles", "modes_get_weak_recovery_stats", "modes_weak_device",
           "modes_weak_fetch", "modes_resolver_run_weak", "modes_resolver_run_shards_weak", "modes_resolver_weak_stats",
           "modes_pool_set_weak_preambles", "modes_pool_weak_stats", "modes_set_arrival", "modes_pool_set_arrival",
           "modes_set_input_rate", "modes_resample_device", "modes_pool_set_input_rate", "modes_set_input_format",
           "modes_pool_set_input_format", "modes_resample_device_at", "modes_set_input_offset",
           "modes_resample_device_shift", "modes_set_spectrum", "modes_take_spectra", "modes_pool_set_spectrum",
           "modes_pool_take_spectra", "modes_process_device", "modes_set_carrier", "modes_pool_set_carrier",
           "modes_pool_submit_device", "modes_pool_ingest_device", "modes_pool_finish", "modes_pool_finish_device"]

INPUT_RATES = (2_000_000, 2_400_000, 4_000_000, 6_000_000, 8_000_000, 10_000_000)      # modes_set_input_rate
INPUT_FORMATS = {"uc8": 0, "sc16": 1, "sc16q11": 2}     # modes_set_input_format: MODES_INPUT_*


def resampled_samples(n_input_bytes: int, rate: int = 2_400_000) -> int:
    """2 MHz samples of a UC8 stream of n_input_bytes bytes at `rate` (modes_set_input_rate), with
    n_in = ceil(bytes / 2): N_out = ceil(5 n_in / 6) at 2.4 MS/s, ceil(n_in / M) at 2 M MS/s, n_in at 2 MHz."""
    n_in = (int(n_input_bytes) + 1) // 2
    if rate == 2_400_000:
        return (5 * n_in + 5) // 6
    if rate not in INPUT_RATES:
        raise ValueError(f"{rate} samples/s is not supported {INPUT_RATES}")
    m = rate // 2_000_000
    return -(-n_in // m)


def lib():
    """Load libmodes_b200.so (built in-tree by `make` / __graft_entry__.build())."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `make` (no CPU fallback exists)")
        L = C.CDLL(str(LIB_PATH))
        L.modes_create.restype = C.c_void_p
        L.modes_create.argtypes = [C.POINTER(Config)]
        L.modes_destroy.argtypes = [C.c_void_p]
        L.modes_last_error.restype = C.c_char_p
        L.modes_last_error.argtypes = [C.c_void_p]
        L.modes_set_sink.argtypes = [C.c_void_p, SINK_FN, C.c_void_p]
        L.modes_process.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_process_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_finish.argtypes = [C.c_void_p]
        L.modes_reset.argtypes = [C.c_void_p]
        L.modes_get_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
        L.modes_compute_magnitude.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        L.modes_detect_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                          C.c_size_t, C.c_void_p]
        L.modes_detect_host.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                        C.c_size_t, C.c_void_p]
        L.modes_detect_wait.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        L.modes_detect_fetch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.modes_resolve.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64]
        L.modes_resolver_create.restype = C.c_void_p
        L.modes_resolver_create.argtypes = [C.POINTER(Config)]
        L.modes_resolver_destroy.argtypes = [C.c_void_p]
        L.modes_resolver_run.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64, SINK_FN,
                                         C.c_void_p]
        L.modes_resolver_run_shards.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p, SINK_FN, C.c_void_p]
        L.modes_resolver_reset.argtypes = [C.c_void_p]
        L.modes_resolver_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
        L.modes_resolver_set_output.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_resolver_output_count.restype = C.c_size_t
        L.modes_resolver_output_count.argtypes = [C.c_void_p]
        L.modes_decode_frame.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Message)]
        L.modes_decode_frames.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        L.modes_format_message.restype = C.c_size_t
        L.modes_format_message.argtypes = [C.POINTER(Message), C.c_int, C.c_char_p, C.c_size_t]
        L.modes_format_raw_net.restype = C.c_size_t
        L.modes_format_raw_net.argtypes = [C.POINTER(Message), C.c_char_p, C.c_size_t]
        L.modes_parse_hex_line.argtypes = [C.c_char_p, C.c_void_p]
        L.modes_stream.restype = C.c_void_p
        L.modes_stream.argtypes = [C.c_void_p]
        L.modes_set_stream.argtypes = [C.c_void_p, C.c_void_p]
        L.modes_set_output.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_output_count.restype = C.c_size_t
        L.modes_output_count.argtypes = [C.c_void_p]
        L.modes_device_alloc.restype = C.c_void_p
        L.modes_device_alloc.argtypes = [C.c_size_t]
        L.modes_device_free.argtypes = [C.c_void_p]
        L.modes_ipc_export.argtypes = [C.c_void_p, C.c_void_p]
        L.modes_ipc_open.restype = C.c_void_p
        L.modes_ipc_open.argtypes = [C.c_void_p]
        L.modes_ipc_close.argtypes = [C.c_void_p]
        L.modes_detect_publish_count.argtypes = [C.c_void_p, C.c_void_p]
        L.modes_copy_to_host.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_device_memset.argtypes = [C.c_void_p, C.c_int, C.c_size_t]
        L.modes_host_alloc.restype = C.c_void_p
        L.modes_host_alloc.argtypes = [C.c_size_t]
        L.modes_host_free.argtypes = [C.c_void_p]
        L.modes_get_kernel_times.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        L.modes_launch_count.restype = C.c_uint64
        L.modes_launch_count.argtypes = [C.c_void_p]
        L.modes_resolver_get_cache.argtypes = [C.c_void_p, C.c_void_p]
        L.modes_resolver_set_cache.argtypes = [C.c_void_p, C.c_void_p]
        L.modes_resolver_tail_cache.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64, C.c_size_t, C.c_void_p]
        L.modes_resolver_run_tentative.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64]
        L.modes_resolver_commit.argtypes = [C.c_void_p, SINK_FN, C.c_void_p]
        L.modes_tile_count.restype = C.c_size_t
        L.modes_tile_count.argtypes = [C.c_size_t]
        L.modes_pool_create.restype = C.c_void_p
        L.modes_pool_create.argtypes = [C.POINTER(Config), C.c_size_t, C.c_size_t]
        L.modes_pool_destroy.argtypes = [C.c_void_p]
        L.modes_pool_last_error.restype = C.c_char_p
        L.modes_pool_last_error.argtypes = [C.c_void_p]
        L.modes_pool_ingest.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, POOL_SINK_FN, C.c_void_p]
        L.modes_pool_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_pool_ingest_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, POOL_SINK_FN, C.c_void_p]
        L.modes_pool_submit_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_pool_collect.argtypes = [C.c_void_p, POOL_SINK_FN, C.c_void_p]
        L.modes_pool_finish.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, POOL_SINK_FN,
                                        C.c_void_p]
        L.modes_pool_finish_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, POOL_SINK_FN,
                                               C.c_void_p]
        L.modes_pool_resolve.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, POOL_SINK_FN, C.c_void_p]
        L.modes_pool_stats.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(Stats)]
        L.modes_pool_reset.argtypes = [C.c_void_p, C.c_uint32]
        L.modes_pool_set_output.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_pool_output_count.restype = C.c_size_t
        L.modes_pool_output_count.argtypes = [C.c_void_p]
        L.modes_pool_buffers.restype = C.c_int64
        L.modes_pool_buffers.argtypes = [C.c_void_p, C.c_uint32]
        L.modes_set_signal.argtypes = [C.c_void_p, C.c_int]
        L.modes_pool_set_signal.argtypes = [C.c_void_p, C.c_int]
        L.modes_set_arrival.argtypes = [C.c_void_p, C.c_int]
        L.modes_pool_set_arrival.argtypes = [C.c_void_p, C.c_int]
        L.modes_set_carrier.argtypes = [C.c_void_p, C.c_int]
        L.modes_pool_set_carrier.argtypes = [C.c_void_p, C.c_int]
        L.modes_format_beast.restype = C.c_size_t
        L.modes_format_beast.argtypes = [C.POINTER(Message), C.c_void_p, C.c_size_t]
        L.modes_set_levels.argtypes = [C.c_void_p, C.c_int]
        L.modes_take_levels.restype = C.c_size_t
        L.modes_take_levels.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_levels_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]
        L.modes_levels_fetch.argtypes = [C.c_void_p, C.c_void_p]
        L.modes_pool_set_levels.argtypes = [C.c_void_p, C.c_int]
        L.modes_pool_take_levels.restype = C.c_size_t
        L.modes_pool_take_levels.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t]
        L.modes_set_spectrum.argtypes = [C.c_void_p, C.c_int]
        L.modes_take_spectra.restype = C.c_size_t
        L.modes_take_spectra.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_pool_set_spectrum.argtypes = [C.c_void_p, C.c_int]
        L.modes_pool_take_spectra.restype = C.c_size_t
        L.modes_pool_take_spectra.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t]
        L.modes_set_recovery.argtypes = [C.c_void_p, C.c_int]
        L.modes_get_recovery_stats.argtypes = [C.c_void_p, C.POINTER(RecoveryStats)]
        L.modes_recover_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_recover_fetch.argtypes = [C.c_void_p, C.c_void_p]
        L.modes_resolver_run_recovered.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64,
                                                   SINK_FN, C.c_void_p]
        L.modes_resolver_run_shards_recovered.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                                          C.c_void_p, C.c_void_p, SINK_FN, C.c_void_p]
        L.modes_resolver_recovery_stats.argtypes = [C.c_void_p, C.POINTER(RecoveryStats)]
        L.modes_pool_set_recovery.argtypes = [C.c_void_p, C.c_int]
        L.modes_pool_recovery_stats.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(RecoveryStats)]
        L.modes_set_weak_preambles.argtypes = [C.c_void_p, C.c_int]
        L.modes_get_weak_recovery_stats.argtypes = [C.c_void_p, C.POINTER(RecoveryStats)]
        L.modes_weak_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_weak_fetch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
        L.modes_resolver_run_weak.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64,
                                              C.c_void_p, C.c_void_p, C.c_size_t, SINK_FN, C.c_void_p]
        L.modes_resolver_run_shards_weak.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, SINK_FN, C.c_void_p]
        L.modes_resolver_weak_stats.argtypes = [C.c_void_p, C.POINTER(RecoveryStats)]
        L.modes_pool_set_weak_preambles.argtypes = [C.c_void_p, C.c_int]
        L.modes_pool_weak_stats.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(RecoveryStats)]
        L.modes_set_input_rate.argtypes = [C.c_void_p, C.c_uint32]
        L.modes_pool_set_input_rate.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        L.modes_set_input_format.argtypes = [C.c_void_p, C.c_uint32, C.c_int32]
        L.modes_pool_set_input_format.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int32]
        L.modes_resample_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64, C.c_int64, C.c_size_t,
                                            C.c_int64, C.c_void_p, C.c_void_p]
        L.modes_resample_device_at.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_int64, C.c_int64,
                                               C.c_size_t, C.c_int64, C.c_void_p, C.c_void_p]
        L.modes_set_input_offset.argtypes = [C.c_void_p, C.c_int32]
        L.modes_resample_device_shift.argtypes = [C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.c_size_t, C.c_int64,
                                                  C.c_int64, C.c_size_t, C.c_int64, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def parse_hex_line(line: str | bytes):
    """decodeHexMessage's parser (dump1090.c:2472-2497): frame bytes, or None if the line is discarded."""
    if isinstance(line, str):
        line = line.encode("latin1")
    msg = (C.c_uint8 * 14)()
    n = lib().modes_parse_hex_line(line, msg)
    return None if n < 0 else bytes(msg)


def make_config(fix_errors=1, aggressive=0, check_crc=1, drop_eof_buffer=0, device=0, profile=0,
                max_batch_bytes=0, n_gpus=0, gpu_resolve=0) -> Config:
    cfg = Config()
    lib().modes_default_config(C.byref(cfg))
    cfg.fix_errors, cfg.aggressive, cfg.check_crc = int(fix_errors), int(aggressive), int(check_crc)
    cfg.drop_eof_buffer, cfg.device, cfg.profile = int(drop_eof_buffer), int(device), int(profile)
    if max_batch_bytes:
        cfg.max_batch_bytes = int(max_batch_bytes)
    cfg.n_gpus = int(n_gpus)
    cfg.gpu_resolve = int(gpu_resolve)
    return cfg


def tiles_for(n_buffers: int) -> int:
    """Entries of the tile table of a batch of n_buffers reference buffers (modes_tile_count)."""
    return int(lib().modes_tile_count(int(n_buffers)))


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def _is_cuda_tensor(x) -> bool:
    """A torch tensor in GPU memory (checked without importing torch: numpy and bytes have no is_cuda)."""
    return getattr(x, "is_cuda", False) is True


def _sync_stream(t) -> None:
    """Wait for the work queued on the tensor's current stream, which may still be writing it."""
    import torch
    torch.cuda.current_stream(t.device).synchronize()


class _Collector:
    """A sink that copies every delivered message."""

    def __init__(self):
        self.messages: list[Message] = []
        self.fn = SINK_FN(self._on)

    def _on(self, _user, mm):
        self.messages.append(mm.contents.copy())


class PinnedBuffer:
    """Page-locked host memory (modes_host_alloc) exposed as a numpy u8 array."""

    def __init__(self, nbytes: int):
        self.ptr = lib().modes_host_alloc(nbytes)
        if not self.ptr:
            raise MemoryError("modes_host_alloc failed")
        self.nbytes = nbytes
        self.array = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(self.ptr))

    def free(self):
        if self.ptr:
            lib().modes_host_free(self.ptr)
            self.ptr = None
            self.array = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Decoder:
    """One GPU decode context (modes_create ... modes_destroy).  signal=True measures the signal
    level of every decoded frame on the GPU (modes_set_signal): Message.signal, rssi_dbfs(), beast().
    levels=True measures every decoded buffer's noise, peak and clipping on the GPU
    (modes_set_levels): take_levels(), level_summary().  recover=True adds weak DF17/DF18 frames of
    known aircraft found by a soft-decision search on the GPU (modes_set_recovery), marked
    Message.recovered: recovery_stats().  weak_preambles=True (with recover=True) also searches the weak
    preambles the reference's preamble test rejects (modes_set_weak_preambles): Message.recovered = 2,
    weak_recovery_stats().  arrival=True measures every decoded frame's arrival time to a sixth of a
    sample on the GPU (modes_set_arrival): Message.arrival, timestamp_12mhz(), beast().
    input_rate=2_400_000 takes 2.4 MS/s bytes (what dump1090-fa and readsb record) and resamples them
    to 2 MHz on the GPU before the pipeline (modes_set_input_rate): the messages are exactly the 2 MHz
    decoder's on the resampled bytes.  Message.sample_pos still counts 2 MHz samples, and
    6 * sample_pos is the input time in 12 MHz ticks at either rate.  input_rate=4_000_000, 6_000_000,
    8_000_000 or 10_000_000 (what Airspy, SDRplay and USRP radios usually record) decimates by 2-5 on the GPU
    instead, with the same contract on the decimated bytes.
    input_format="sc16" or "sc16q11" takes signed 16-bit I/Q bytes (SoapySDR and Airspy-class tools,
    bladeRF) and converts them to 8-bit I/Q on the GPU with input_shift (None: the format's default)
    before the pipeline (modes_set_input_format): the messages are exactly the UC8 decoder's on the
    converted bytes, at either input rate.
    input_offset=+2_000_000 (Hz) decodes a 4-10 MS/s capture whose radio was tuned 2 MHz below 1090 MHz,
    as zero-IF radios are to keep their DC spike off the channel: the input is shifted back by that much on
    the GPU as it is decimated (modes_set_input_offset, |offset| <= input_rate / 2 - 1 MHz); 0 changes
    nothing.
    spectrum=True measures every decoded buffer's input power spectrum on the GPU, before resampling,
    decimation and the offset (modes_set_spectrum): take_spectra(), spectrum_summary().
    carrier=True measures every decoded frame's carrier frequency relative to the centre of the 2 MHz bytes
    on the GPU (modes_set_carrier): Message.carrier_code, carrier_hz(), carrier_summary().  It cannot be
    combined with gpu_resolve.
    process() and decode() also take a CUDA torch tensor of any dtype on the decoder's device, read as its
    raw bytes (e.g. int16 SC16 I/Q), and decode it where it is (modes_process_device): the output is what
    the same bytes give from host memory, without their two trips across PCIe."""

    def __init__(self, signal: bool = False, levels: bool = False, recover: bool = False, weak_preambles: bool = False,
                 arrival: bool = False, input_rate: int = 2_000_000, input_format: str = "uc8",
                 input_shift: int | None = None, input_offset: int = 0, spectrum: bool = False, carrier: bool = False,
                 **cfg):
        self.cfg = make_config(**cfg)
        self._h = lib().modes_create(C.byref(self.cfg))
        if not self._h:
            raise RuntimeError("modes_create failed: " + lib().modes_last_error(None).decode())
        if input_rate != 2_000_000:
            self.set_input_rate(input_rate)
        if input_format != "uc8" or input_shift is not None:
            self.set_input_format(input_format, input_shift)
        if input_offset:
            self.set_input_offset(input_offset)
        if signal:
            self.set_signal(True)
        if arrival:
            self.set_arrival(True)
        if levels:
            self.set_levels(True)
        if spectrum:
            self.set_spectrum(True)
        if carrier:
            self.set_carrier(True)
        if recover:
            self.set_recovery(True)
        if weak_preambles:
            self.set_weak_preambles(True)
        self._collector = _Collector()
        lib().modes_set_sink(self._h, self._collector.fn, None)

    # -- lifecycle
    def close(self):
        if self._h:
            lib().modes_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(lib().modes_last_error(self._h).decode())

    # -- streaming path (the --ifile main loop)
    def process(self, data) -> None:
        if _is_cuda_tensor(data):
            t = self._device_bytes(data)
            self.process_device_ptr(t.data_ptr(), t.numel() * t.element_size())
            return
        a = np.ascontiguousarray(data, dtype=np.uint8) if not isinstance(data, (bytes, bytearray)) \
            else np.frombuffer(data, dtype=np.uint8)
        self._check(lib().modes_process(self._h, _ptr(a), a.size))

    def process_ptr(self, ptr: int, nbytes: int) -> None:
        self._check(lib().modes_process(self._h, C.c_void_p(ptr), nbytes))

    def process_device_ptr(self, ptr: int, nbytes: int) -> None:
        """modes_process_device: nbytes of the stream at a device address of the decoder's device, fully
        written before the call and no longer read after it."""
        self._check(lib().modes_process_device(self._h, C.c_void_p(ptr), nbytes))

    def _device_bytes(self, t):
        """The CUDA tensor as a contiguous tensor on this decoder's device, its writers finished."""
        if t.device.index != self.cfg.device:
            raise ValueError(f"the tensor is on {t.device}, the decoder on cuda:{self.cfg.device}")
        if not t.is_contiguous():
            t = t.contiguous()
        _sync_stream(t)
        return t

    def finish(self) -> None:
        self._check(lib().modes_finish(self._h))

    def reset(self) -> None:
        self._check(lib().modes_reset(self._h))
        self._collector.messages = []

    def take_messages(self) -> list:
        out, self._collector.messages = self._collector.messages, []
        return out

    def decode(self, data, chunk: int | None = None) -> list:
        """Decode a whole stream like `dump1090 --ifile`: returns the message list.  A CUDA tensor is
        decoded in device memory, in calls of `chunk` bytes."""
        self.reset()
        if _is_cuda_tensor(data):
            t = self._device_bytes(data)
            ptr, n = t.data_ptr(), t.numel() * t.element_size()
            step = chunk or max(n, 1)
            for off in range(0, max(n, 1), step):
                self.process_device_ptr(ptr + off, min(step, n - off))
            self.finish()
            return self.take_messages()
        a = np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else \
            np.ascontiguousarray(data, dtype=np.uint8)
        if chunk:
            for off in range(0, a.size, chunk):
                self.process(a[off: off + chunk])
        else:
            self.process(a)
        self.finish()
        return self.take_messages()

    def set_output_array(self, capacity: int):
        """Deliver messages into a preallocated array instead of the Python callback
        (no per-message interpreter work).  Returns the ctypes array; capacity 0 restores the callback."""
        if capacity <= 0:
            self._out = None
            lib().modes_set_output(self._h, None, 0)
            lib().modes_set_sink(self._h, self._collector.fn, None)
            return None
        self._out = (Message * capacity)()
        lib().modes_set_sink(self._h, C.cast(None, SINK_FN), None)
        lib().modes_set_output(self._h, self._out, capacity)
        return self._out

    def rearm_output(self) -> None:
        lib().modes_set_output(self._h, self._out, len(self._out))

    def output_count(self) -> int:
        return int(lib().modes_output_count(self._h))

    def set_signal(self, on: bool) -> None:
        """Measure the signal level for batches submitted from now on (modes_set_signal)."""
        self._check(lib().modes_set_signal(self._h, int(bool(on))))

    def set_input_rate(self, hz: int) -> None:
        """The sample rate of the stream that begins at the next reset (decode() resets): one of INPUT_RATES
        (modes_set_input_rate); refused while a stream is in progress.  sample_pos counts 2 MHz samples at
        every rate, and 6 * sample_pos is the input time in 12 MHz ticks."""
        self._check(lib().modes_set_input_rate(self._h, int(hz)))

    def set_input_offset(self, hz: int) -> None:
        """Where 1090 MHz sits in the capture's baseband, in Hz (+2_000_000: the radio was tuned to 1088 MHz),
        for the stream that begins at the next reset (modes_set_input_offset): 0, or at the decimated rates
        |hz| <= input_rate / 2 - 1 MHz; refused while a stream is in progress.  set_input_rate refuses a rate
        that cannot take the offset already set, so set it to 0 before changing to such a rate."""
        self._check(lib().modes_set_input_offset(self._h, int(hz)))

    def set_input_format(self, fmt: str, shift: int | None = None) -> None:
        """The sample format of the stream that begins at the next reset: "uc8", "sc16" or "sc16q11"
        (INPUT_FORMATS, modes_set_input_format), with the shift 0 ... 15 that converts 16-bit values to
        8 bits (None: the format's default, 8 for sc16 and 4 for sc16q11); refused while a stream is in
        progress."""
        if fmt not in INPUT_FORMATS:
            raise ValueError(f"input format {fmt!r} is not one of {sorted(INPUT_FORMATS)}")
        self._check(lib().modes_set_input_format(self._h, INPUT_FORMATS[fmt], -1 if shift is None else int(shift)))

    def set_arrival(self, on: bool) -> None:
        """Measure the arrival time for batches submitted from now on (modes_set_arrival)."""
        self._check(lib().modes_set_arrival(self._h, int(bool(on))))

    def set_carrier(self, on: bool) -> None:
        """Measure the carrier frequency for batches submitted from now on (modes_set_carrier)."""
        self._check(lib().modes_set_carrier(self._h, int(bool(on))))

    def set_levels(self, on: bool) -> None:
        """Measure the buffers' levels for batches submitted from now on (modes_set_levels)."""
        self._check(lib().modes_set_levels(self._h, int(bool(on))))

    def set_recovery(self, on: bool) -> None:
        """Recover weak DF17/DF18 frames in batches submitted from now on (modes_set_recovery)."""
        self._check(lib().modes_set_recovery(self._h, int(bool(on))))

    def recovery_stats(self) -> dict:
        st = RecoveryStats()
        self._check(lib().modes_get_recovery_stats(self._h, C.byref(st)))
        return st.as_dict()

    def set_weak_preambles(self, on: bool) -> None:
        """Also recover at weak preambles in batches submitted from now on, while recovery is on
        (modes_set_weak_preambles)."""
        self._check(lib().modes_set_weak_preambles(self._h, int(bool(on))))

    def weak_recovery_stats(self) -> dict:
        st = RecoveryStats()
        self._check(lib().modes_get_weak_recovery_stats(self._h, C.byref(st)))
        return st.as_dict()

    def take_levels(self) -> np.ndarray:
        """The queued level records (LEVEL_DTYPE), oldest first, in stream order; the queue is emptied."""
        n = int(lib().modes_take_levels(self._h, None, 0))
        out = np.zeros(n, dtype=LEVEL_DTYPE)
        got = int(lib().modes_take_levels(self._h, _ptr(out), n)) if n else 0
        return out[:got]

    def set_spectrum(self, on: bool) -> None:
        """Measure the buffers' input spectra for batches submitted from now on (modes_set_spectrum)."""
        self._check(lib().modes_set_spectrum(self._h, int(bool(on))))

    def take_spectra(self) -> np.ndarray:
        """The queued spectrum records (SPECTRUM_DTYPE), oldest first, in stream order; the queue is emptied."""
        n = int(lib().modes_take_spectra(self._h, None, 0))
        out = np.zeros(n, dtype=SPECTRUM_DTYPE)
        got = int(lib().modes_take_spectra(self._h, _ptr(out), n)) if n else 0
        return out[:got]

    def set_stream(self, cuda_stream: int) -> None:
        self._check(lib().modes_set_stream(self._h, C.c_void_p(cuda_stream)))

    def stats(self) -> dict:
        st = Stats()
        self._check(lib().modes_get_stats(self._h, C.byref(st)))
        return dict(zip(STAT_NAMES, [int(x) for x in st.v]))

    # -- stage-level entry points
    def magnitude(self, iq: np.ndarray) -> np.ndarray:
        a = np.ascontiguousarray(iq, dtype=np.uint8)
        out = np.empty(a.size // 2, dtype=np.uint16)
        self._check(lib().modes_compute_magnitude(self._h, _ptr(a), a.size // 2, _ptr(out)))
        return out

    def detect_device(self, d_iq_ptr: int, n_buffers: int, carry: bytes | None = None,
                      d_candidates_ptr: int = 0, cand_capacity: int = 0, d_tiles_ptr: int = 0) -> None:
        carr = None
        if carry is not None:
            assert len(carry) == CARRY_BYTES
            carr = (C.c_uint8 * CARRY_BYTES).from_buffer_copy(carry)
        self._check(lib().modes_detect_device(self._h, C.c_void_p(d_iq_ptr), n_buffers, carr,
                                              C.c_void_p(d_candidates_ptr), cand_capacity,
                                              C.c_void_p(d_tiles_ptr)))

    def detect_host(self, host_ptr: int, n_buffers: int, carry: bytes | None = None,
                    d_candidates_ptr: int = 0, cand_capacity: int = 0, d_tiles_ptr: int = 0) -> None:
        carr = (C.c_uint8 * CARRY_BYTES).from_buffer_copy(carry) if carry is not None else None
        self._check(lib().modes_detect_host(self._h, C.c_void_p(host_ptr), n_buffers, carr,
                                            C.c_void_p(d_candidates_ptr), cand_capacity, C.c_void_p(d_tiles_ptr)))

    def detect_wait(self) -> int:
        n = C.c_uint64(0)
        self._check(lib().modes_detect_wait(self._h, C.byref(n)))
        return int(n.value)

    def detect_fetch(self, n_buffers: int):
        n = self.detect_wait()
        cands = np.zeros(max(n, 1), dtype=CANDIDATE_DTYPE)
        tiles = np.zeros(tiles_for(n_buffers), dtype=TILE_DTYPE)
        self._check(lib().modes_detect_fetch(self._h, _ptr(cands), _ptr(tiles)))
        return cands[:n], tiles

    def detect_fetch_into(self, cands: np.ndarray, tiles: np.ndarray):
        """Like detect_fetch, into caller-owned arrays (pinned memory for full PCIe speed); returns views."""
        n = self.detect_wait()
        if n > cands.size:
            raise RuntimeError(f"record buffer too small: {n} > {cands.size}")
        self._check(lib().modes_detect_fetch(self._h, _ptr(cands), _ptr(tiles)))
        return cands[:n], tiles

    def resolve(self, cands: np.ndarray, tiles: np.ndarray, buffer_base: int = 0) -> None:
        self._check(lib().modes_resolve(self._h, _ptr(np.ascontiguousarray(cands)), _ptr(np.ascontiguousarray(tiles)),
                                        tiles.size, buffer_base))

    def decode_frame(self, frame: bytes) -> Message:
        buf = (C.c_uint8 * 14)(*(list(frame) + [0] * (14 - len(frame))))
        m = Message()
        self._check(lib().modes_decode_frame(self._h, buf, C.byref(m)))
        return m

    def decode_frames(self, frames):
        """A batch of frames (each padded to 14 bytes) through the hex door in one launch, the
        address cache carried from frame to frame.  A list of frames gives a list of Message; an
        (n, 14) uint8 array is passed as it is and gives the ctypes array of n Message (view it
        with np.frombuffer), without a Python object per byte or per frame."""
        if isinstance(frames, np.ndarray):
            a = np.ascontiguousarray(frames, dtype=np.uint8).reshape(-1, 14)
            out = (Message * a.shape[0])()
            self._check(lib().modes_decode_frames(self._h, _ptr(a), a.shape[0], out))
            return out
        n = len(frames)
        buf = (C.c_uint8 * (14 * n))(*[b for f in frames for b in (list(f) + [0] * (14 - len(f)))])
        out = (Message * n)()
        self._check(lib().modes_decode_frames(self._h, buf, n, out))
        return [out[i] for i in range(n)]

    def resample_device(self, d_in_ptr: int, in_bytes: int, in_first_sample: int, first_buffer: int, n_buffers: int,
                        d_out_ptr: int, out_end: int = -1, want_carry: bool = True) -> bytes | None:
        """2 MHz reference buffers first_buffer ... of a 2.4 MS/s stream, from in_bytes of its input (input
        sample in_first_sample on) in device memory, into device memory at d_out_ptr (modes_resample_device).
        Output samples at or past out_end are 127 (negative: no limit).  Returns the CARRY_BYTES 2 MHz
        bytes before the first buffer (for detect_device), or None with want_carry=False (then nothing waits)."""
        carry = (C.c_uint8 * CARRY_BYTES)() if want_carry else None
        self._check(lib().modes_resample_device(self._h, C.c_void_p(d_in_ptr or None), int(in_bytes), int(in_first_sample),
                                                int(first_buffer), int(n_buffers), int(out_end), C.c_void_p(d_out_ptr),
                                                carry))
        return bytes(carry) if want_carry else None

    def resample_device_at(self, hz: int, d_in_ptr: int, in_bytes: int, in_first_sample: int, first_buffer: int,
                           n_buffers: int, d_out_ptr: int, out_end: int = -1, want_carry: bool = True) -> bytes | None:
        """resample_device at any of INPUT_RATES but 2 MHz (modes_resample_device_at): 2.4 MS/s resampled,
        4-10 MS/s decimated, UC8 input."""
        carry = (C.c_uint8 * CARRY_BYTES)() if want_carry else None
        self._check(lib().modes_resample_device_at(self._h, int(hz), C.c_void_p(d_in_ptr or None), int(in_bytes),
                                                   int(in_first_sample), int(first_buffer), int(n_buffers), int(out_end),
                                                   C.c_void_p(d_out_ptr), carry))
        return bytes(carry) if want_carry else None

    def resample_device_shift(self, hz: int, offset_hz: int, d_in_ptr: int, in_bytes: int, in_first_sample: int,
                              first_buffer: int, n_buffers: int, d_out_ptr: int, out_end: int = -1,
                              want_carry: bool = True) -> bytes | None:
        """resample_device_at with the input first shifted by offset_hz (modes_resample_device_shift), the phase
        from each sample's stream index; offset_hz 0 is resample_device_at exactly."""
        carry = (C.c_uint8 * CARRY_BYTES)() if want_carry else None
        self._check(lib().modes_resample_device_shift(self._h, int(hz), int(offset_hz), C.c_void_p(d_in_ptr or None),
                                                      int(in_bytes), int(in_first_sample), int(first_buffer),
                                                      int(n_buffers), int(out_end), C.c_void_p(d_out_ptr), carry))
        return bytes(carry) if want_carry else None

    def levels_device(self, d_iq_ptr: int, n_buffers: int, stride_bytes: int = 0) -> None:
        """Level records of n_buffers buffers in device memory, buffer k at d_iq_ptr + k * stride_bytes."""
        self._check(lib().modes_levels_device(self._h, C.c_void_p(d_iq_ptr), n_buffers, stride_bytes))
        self._levels_n = n_buffers

    def levels_fetch(self) -> np.ndarray:
        """The records of the last levels_device call (waits for them)."""
        out = np.zeros(getattr(self, "_levels_n", 0), dtype=LEVEL_DTYPE)
        self._check(lib().modes_levels_fetch(self._h, _ptr(out)))
        return out

    def recover_device(self, d_out_ptr: int = 0, capacity: int = 0) -> None:
        """Recovery records of the last detect_device / detect_host batch, into device memory, or (0) into
        the context's own buffer for recover_fetch()."""
        self._check(lib().modes_recover_device(self._h, C.c_void_p(d_out_ptr or None), capacity))

    def recover_fetch(self) -> np.ndarray:
        """The records of the last recover_device(0) call (RECOVERED_DTYPE), one per candidate record."""
        n = self.detect_wait()
        out = np.zeros(max(n, 1), dtype=RECOVERED_DTYPE)
        self._check(lib().modes_recover_fetch(self._h, _ptr(out)))
        return out[:n]

    def weak_device(self, d_pos_ptr: int = 0, d_rec_ptr: int = 0, capacity: int = 0) -> None:
        """Weak positions and their recovery records of the last detect_device / detect_host batch, into
        device memory (capacity entries each), or (0) into the context's own buffers for weak_fetch()."""
        self._check(lib().modes_weak_device(self._h, C.c_void_p(d_pos_ptr or None), C.c_void_p(d_rec_ptr or None), capacity))
        self._weak_ext = bool(d_pos_ptr)

    def weak_fetch(self):
        """(count, t, records) of the last weak_device call; t and records are empty for caller buffers."""
        n = C.c_uint64(0)
        self._check(lib().modes_weak_fetch(self._h, None, None, C.byref(n)))
        if getattr(self, "_weak_ext", False):
            return int(n.value), np.zeros(0, np.uint32), np.zeros(0, RECOVERED_DTYPE)
        t = np.zeros(max(n.value, 1), dtype=np.uint32)
        rec = np.zeros(max(n.value, 1), dtype=RECOVERED_DTYPE)
        self._check(lib().modes_weak_fetch(self._h, _ptr(t), _ptr(rec), C.byref(n)))
        return int(n.value), t[: n.value], rec[: n.value]

    def publish_count(self, dst_ptr: int) -> None:
        self._check(lib().modes_detect_publish_count(self._h, C.c_void_p(dst_ptr)))

    def kernel_times_ms(self):
        t = (C.c_float * 4)()
        lib().modes_get_kernel_times(self._h, C.byref(t))
        return [float(x) for x in t]

    def launch_count(self) -> int:
        return int(lib().modes_launch_count(self._h))

    @property
    def stream(self) -> int:
        return int(lib().modes_stream(self._h) or 0)


def _weak_arrays(weak):
    t, rec = weak
    t = np.ascontiguousarray(t, dtype=np.uint32)
    rec = np.ascontiguousarray(rec, dtype=RECOVERED_DTYPE)
    if rec.size != t.size:
        raise ValueError(f"{rec.size} weak records for {t.size} weak positions: one per position is needed")
    if t.size > 1 and not (np.diff(t.astype(np.int64)) > 0).all():
        raise ValueError("weak positions must be sorted and distinct")
    return t, rec


def _recovery_records(recovered, cands: np.ndarray) -> np.ndarray:
    rec = np.ascontiguousarray(recovered, dtype=RECOVERED_DTYPE)
    if rec.size < cands.size:
        raise ValueError(f"{rec.size} recovery records for {cands.size} candidates: one per candidate is needed")
    return rec


class Resolver:
    """The sequential half alone (no device): modes_resolver_*."""

    def __init__(self, **cfg):
        self.cfg = make_config(**cfg)
        self._h = lib().modes_resolver_create(C.byref(self.cfg))
        self._collector = _Collector()

    def run(self, cands: np.ndarray, tiles: np.ndarray, buffer_base: int = 0, recovered: np.ndarray | None = None,
            weak=None) -> None:
        """recovered: RECOVERED_DTYPE records, one per candidate, to add recovered messages
        (modes_resolver_run_recovered); None runs the reference's resolve alone.  weak: (t, records) of
        the weak preambles, t sorted (modes_resolver_run_weak; needs recovered)."""
        cands = np.ascontiguousarray(cands)
        tiles = np.ascontiguousarray(tiles)
        fn = C.cast(None, SINK_FN) if getattr(self, "_native", False) else self._collector.fn
        if weak is not None:
            if recovered is None:
                raise ValueError("weak preambles need the candidates' recovery records")
            rec = _recovery_records(recovered, cands)
            wt, wr = _weak_arrays(weak)
            rc = lib().modes_resolver_run_weak(self._h, _ptr(cands), _ptr(rec), _ptr(tiles), tiles.size, buffer_base,
                                               _ptr(wt), _ptr(wr), wt.size, fn, None)
        elif recovered is None:
            rc = lib().modes_resolver_run(self._h, _ptr(cands), _ptr(tiles), tiles.size, buffer_base, fn, None)
        else:
            rec = _recovery_records(recovered, cands)
            rc = lib().modes_resolver_run_recovered(self._h, _ptr(cands), _ptr(rec), _ptr(tiles), tiles.size, buffer_base,
                                                    fn, None)
        if rc:
            raise RuntimeError("modes_resolver_run failed")

    def recovery_stats(self) -> dict:
        st = RecoveryStats()
        if lib().modes_resolver_recovery_stats(self._h, C.byref(st)):
            raise RuntimeError("modes_resolver_recovery_stats failed")
        return st.as_dict()

    def weak_stats(self) -> dict:
        st = RecoveryStats()
        if lib().modes_resolver_weak_stats(self._h, C.byref(st)):
            raise RuntimeError("modes_resolver_weak_stats failed")
        return st.as_dict()

    def reset_state(self) -> None:
        lib().modes_resolver_reset(self._h)

    def run_shards(self, shards, recovered=None, weak=None) -> None:
        """shards: [(cands ndarray, tiles ndarray, buffer_base)] in stream order; resolved concurrently.
        recovered: a list of RECOVERED_DTYPE arrays, one per shard (modes_resolver_run_shards_recovered).
        weak: a list of (t, records) per shard (modes_resolver_run_shards_weak; needs recovered)."""
        n = len(shards)
        keep = [(np.ascontiguousarray(c), np.ascontiguousarray(t)) for c, t, _ in shards]
        cp = (C.c_void_p * n)(*[c.ctypes.data for c, _ in keep])
        tp = (C.c_void_p * n)(*[t.ctypes.data for _, t in keep])
        nt = (C.c_size_t * n)(*[t.size for _, t in keep])
        bb = (C.c_int64 * n)(*[int(b) for _, _, b in shards])
        fn = C.cast(None, SINK_FN) if getattr(self, "_native", False) else self._collector.fn
        if weak is not None:
            if recovered is None or len(recovered) != n or len(weak) != n:
                raise ValueError("weak preambles need one recovery array and one weak pair per shard")
            recs = [_recovery_records(r, c) for r, (c, _) in zip(recovered, keep)]
            wks = [_weak_arrays(w) for w in weak]
            rp = (C.c_void_p * n)(*[r.ctypes.data for r in recs])
            wtp = (C.c_void_p * n)(*[t.ctypes.data for t, _ in wks])
            wrp = (C.c_void_p * n)(*[r.ctypes.data for _, r in wks])
            nw = (C.c_size_t * n)(*[t.size for t, _ in wks])
            rc = lib().modes_resolver_run_shards_weak(self._h, n, cp, rp, tp, nt, bb, wtp, wrp, nw, fn, None)
        elif recovered is None:
            rc = lib().modes_resolver_run_shards(self._h, n, cp, tp, nt, bb, fn, None)
        else:
            if len(recovered) != n:
                raise ValueError(f"{len(recovered)} recovery arrays for {n} shards")
            recs = [_recovery_records(r, c) for r, (c, _) in zip(recovered, keep)]
            rp = (C.c_void_p * n)(*[r.ctypes.data for r in recs])
            rc = lib().modes_resolver_run_shards_recovered(self._h, n, cp, rp, tp, nt, bb, fn, None)
        if rc:
            raise RuntimeError("modes_resolver_run_shards failed")

    # ---- one shard of a sharded decode (see include/modes_b200.h and sharded.resolve_distributed)
    def get_cache(self) -> np.ndarray:
        out = np.zeros(ICAO_CACHE_SLOTS, dtype=np.uint32)
        lib().modes_resolver_get_cache(self._h, _ptr(out))
        return out

    def set_cache(self, cache=None) -> None:
        c = None if cache is None else np.ascontiguousarray(cache, dtype=np.uint32)
        lib().modes_resolver_set_cache(self._h, None if c is None else _ptr(c))

    def tail_cache(self, cands: np.ndarray, tiles: np.ndarray, buffer_base: int = 0, n_tail_tiles: int | None = None) -> np.ndarray:
        out = np.zeros(ICAO_CACHE_SLOTS, dtype=np.uint32)
        if n_tail_tiles is None:
            n_tail_tiles = max(tiles.size // 16, 128)
        if lib().modes_resolver_tail_cache(self._h, _ptr(cands), _ptr(tiles), tiles.size, buffer_base, n_tail_tiles, _ptr(out)):
            raise RuntimeError("modes_resolver_tail_cache failed")
        return out

    def run_tentative(self, cands: np.ndarray, tiles: np.ndarray, buffer_base: int = 0) -> None:
        self._held = (cands, tiles)                       # the records must outlive the commit
        if lib().modes_resolver_run_tentative(self._h, _ptr(cands), _ptr(tiles), tiles.size, buffer_base):
            raise RuntimeError("modes_resolver_run_tentative failed")

    def commit(self) -> None:
        fn = C.cast(None, SINK_FN) if getattr(self, "_native", False) else self._collector.fn
        if lib().modes_resolver_commit(self._h, fn, None):
            raise RuntimeError("modes_resolver_commit without a tentative run")
        self._held = None

    def take_messages(self):
        out, self._collector.messages = self._collector.messages, []
        return out

    def set_output_array(self, capacity: int):
        """Fill a preallocated array in place instead of calling back into Python per message."""
        self._out = (Message * capacity)() if capacity > 0 else None
        self._native = capacity > 0
        lib().modes_resolver_set_output(self._h, self._out, max(capacity, 0))
        return self._out

    def rearm_output(self) -> None:
        lib().modes_resolver_set_output(self._h, self._out, len(self._out))

    def output_count(self) -> int:
        return int(lib().modes_resolver_output_count(self._h))

    def stats(self) -> dict:
        st = Stats()
        lib().modes_resolver_stats(self._h, C.byref(st))
        return dict(zip(STAT_NAMES, [int(x) for x in st.v]))

    def close(self):
        if self._h:
            lib().modes_resolver_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- SURVEY.md 8(f) item 4: many receivers on one GPU ----------------------------------------

class ReceiverPool:
    """modes_pool_*: independent 2 MHz streams (one address cache, carry, skip state and set of
    statistics each, as one dump1090 process keeps per receiver), one buffer of each decoded per
    batch.  Messages are collected per receiver (`take(receiver)`).  signal=True: as for Decoder.
    levels=True: level records of every receiver's buffers (`take_levels(receiver)`).
    spectrum=True: input spectrum records of every receiver's buffers (`take_spectra(receiver)`).
    recover=True: as for Decoder, with statistics per receiver (`recovery_stats(receiver)`).
    weak_preambles=True: as for Decoder (`weak_recovery_stats(receiver)`).  arrival=True, carrier=True: as
    for Decoder.
    input_rate=2_400_000 sets every receiver to 2.4 MS/s at creation, set_input_rate(receiver, hz) one
    receiver (modes_pool_set_input_rate): a buffer is still BUFFER_BYTES of the receiver's stream, and its
    2 MHz buffers are decoded as their input completes (`buffers(receiver)` counts them).
    input_format="sc16" / "sc16q11" (and input_shift) sets every receiver's sample format at creation,
    set_input_format(receiver, fmt, shift) one receiver (modes_pool_set_input_format).  A buffer is the
    receiver's next BUFFER_SAMPLES samples as uint8 bytes: BUFFER_BYTES for a UC8 receiver, 2 * BUFFER_BYTES
    of little-endian int16 I/Q for an SC16 or SC16Q11 one; everything delivered for a 16-bit receiver
    equals what a UC8 receiver at its rate delivers on the converted bytes.
    ingest() and submit() also take CUDA torch tensors on the pool's device, either a list of one tensor per
    receiver or a 2-D tensor of one row per receiver, each read as its raw bytes (e.g. int16 SC16 I/Q), and
    decode them where they are (modes_pool_submit_device): the output is what the same bytes give from host
    memory, without their two trips across PCIe.  A receiver is fed from one kind of memory until
    reset(receiver).
    finish(receivers, tails) ends the listed receivers' streams with their last bytes (modes_pool_finish):
    everything delivered for a receiver then equals Decoder(same settings).decode(all its bytes), the EOF
    buffer included unless drop_eof_buffer=1.  decode_captures() decodes many finite captures this way."""

    def __init__(self, n_receivers: int, max_batch: int = 0, signal: bool = False, levels: bool = False,
                 recover: bool = False, weak_preambles: bool = False, arrival: bool = False,
                 input_rate: int = 2_000_000, input_format: str = "uc8", input_shift: int | None = None,
                 spectrum: bool = False, carrier: bool = False, **cfg):
        self.cfg = make_config(**cfg)
        self.n = n_receivers
        self._bytes = [BUFFER_BYTES] * n_receivers
        self._h = lib().modes_pool_create(C.byref(self.cfg), n_receivers, max_batch)
        if not self._h:
            raise RuntimeError("modes_pool_create failed")
        if signal:
            self.set_signal(True)
        if arrival:
            self.set_arrival(True)
        if levels:
            self.set_levels(True)
        if spectrum:
            self.set_spectrum(True)
        if carrier:
            self.set_carrier(True)
        if recover:
            self.set_recovery(True)
        if weak_preambles:
            self.set_weak_preambles(True)
        if input_rate != 2_000_000:
            for r in range(n_receivers):
                self.set_input_rate(r, input_rate)
        if input_format != "uc8" or input_shift is not None:
            for r in range(n_receivers):
                self.set_input_format(r, input_format, input_shift)
        self.messages = [[] for _ in range(n_receivers)]
        self._fn = POOL_SINK_FN(self._on)

    def _on(self, _user, receiver, mm):
        self.messages[receiver].append(mm.contents.copy())

    def _check(self, rc):
        if rc:
            raise RuntimeError(lib().modes_pool_last_error(self._h).decode())

    def _buffers(self, receivers, buffers):
        """The ids and the buffers as uint8 arrays, each of its receiver's size; ValueError otherwise."""
        ids = np.ascontiguousarray(receivers, dtype=np.uint32)
        bufs = [np.ascontiguousarray(b, dtype=np.uint8) for b in buffers]
        assert ids.size == len(bufs)
        for r, b in zip(ids.tolist(), bufs):
            want = self._bytes[r] if r < self.n else BUFFER_BYTES
            if b.size != want:
                raise ValueError(f"receiver {r}: a buffer of {b.size} bytes, its input format takes {want}")
        return ids, bufs

    def _device_buffers(self, receivers, buffers):
        """The ids, the device addresses of the CUDA tensors (a list of one per receiver, or the rows of a 2-D
        tensor), each read as its raw bytes and of its receiver's size, and the tensors to keep alive until the
        batch is collected; their writers finished.  ValueError otherwise."""
        ids = np.ascontiguousarray(receivers, dtype=np.uint32)
        if _is_cuda_tensor(buffers):
            t = self._on_device(buffers)
            if t.dim() != 2 or t.shape[0] != ids.size:
                raise ValueError(f"a tensor of shape {tuple(t.shape)} for {ids.size} receivers: one row per receiver")
            row = t.shape[1] * t.element_size()
            ptrs, sizes, keep = [t.data_ptr() + i * row for i in range(ids.size)], [row] * ids.size, [t]
        else:
            if not all(_is_cuda_tensor(b) for b in buffers):
                raise ValueError("a list that mixes CUDA tensors with host buffers: one kind of memory per call")
            keep = [self._on_device(b) for b in buffers]
            if len(keep) != ids.size:
                raise ValueError(f"{len(keep)} buffers for {ids.size} receivers")
            ptrs, sizes = [t.data_ptr() for t in keep], [t.numel() * t.element_size() for t in keep]
        for r, n in zip(ids.tolist(), sizes):
            want = self._bytes[r] if r < self.n else BUFFER_BYTES
            if n != want:
                raise ValueError(f"receiver {r}: a buffer of {n} bytes, its input format takes {want}")
        if keep:
            _sync_stream(keep[0])                            # one device, so one current stream for all
        return ids, (C.c_void_p * len(ptrs))(*ptrs), keep

    def _on_device(self, t):
        """The CUDA tensor as a contiguous tensor on this pool's device."""
        if t.device.index != self.cfg.device:
            raise ValueError(f"the tensor is on {t.device}, the pool on cuda:{self.cfg.device}")
        return t if t.is_contiguous() else t.contiguous()

    @staticmethod
    def _on_gpu(buffers) -> bool:
        return _is_cuda_tensor(buffers) or any(_is_cuda_tensor(b) for b in buffers)

    def ingest(self, receivers, buffers) -> None:
        """buffers[i]: the next buffer of receivers[i], uint8 bytes (numpy) of its format (class docstring),
        or CUDA tensors of those bytes (a list, or a 2-D tensor of one row per receiver)."""
        if self._on_gpu(buffers):
            ids, ptrs, _keep = self._device_buffers(receivers, buffers)
            self._check(lib().modes_pool_ingest_device(self._h, _ptr(ids), ptrs, ids.size, self._fn, None))
            return
        ids, bufs = self._buffers(receivers, buffers)
        ptrs = (C.c_void_p * len(bufs))(*[b.ctypes.data for b in bufs])
        self._check(lib().modes_pool_ingest(self._h, _ptr(ids), ptrs, ids.size, self._fn, None))

    def finish(self, receivers, tails) -> None:
        """tails[i]: the last bytes of receivers[i]'s stream, 0 up to its buffer size, uint8 bytes (numpy) or a
        CUDA tensor read as its raw bytes (for a device-fed or never-fed receiver); the streams then end as
        Decoder.finish() ends one.  Until reset(receiver), the receiver takes no more buffers."""
        ids = np.ascontiguousarray(receivers, dtype=np.uint32)
        if len(tails) != ids.size:
            raise ValueError(f"{len(tails)} tails for {ids.size} receivers")
        on_gpu = [_is_cuda_tensor(t) for t in tails]
        if any(on_gpu) and not all(on_gpu):
            raise ValueError("a list that mixes CUDA tensors with host buffers: one kind of memory per call")
        if any(on_gpu):
            keep = [self._on_device(t) for t in tails]
            ptrs, sizes = [t.data_ptr() for t in keep], [t.numel() * t.element_size() for t in keep]
        else:
            keep = [np.ascontiguousarray(t, dtype=np.uint8).reshape(-1) for t in tails]
            ptrs, sizes = [t.ctypes.data for t in keep], [t.size for t in keep]
        for r, n in zip(ids.tolist(), sizes):
            most = self._bytes[r] if r < self.n else BUFFER_BYTES
            if n > most:
                raise ValueError(f"receiver {r}: a tail of {n} bytes, its input format takes at most {most}")
        if any(on_gpu) and keep:
            _sync_stream(keep[0])
        fn = lib().modes_pool_finish_device if any(on_gpu) else lib().modes_pool_finish
        sizes = np.asarray(sizes, dtype=np.uintp)
        self._check(fn(self._h, _ptr(ids), (C.c_void_p * len(ptrs))(*ptrs), _ptr(sizes), ids.size, self._fn, None))

    def ingest_ptrs(self, receivers: np.ndarray, ptrs, sink=None) -> None:
        """The same from raw host addresses (pinned memory); sink: a POOL_SINK_FN or None to drop the messages."""
        fn = sink if sink is not None else C.cast(None, POOL_SINK_FN)
        self._check(lib().modes_pool_ingest(self._h, _ptr(receivers), ptrs, receivers.size, fn, None))

    def ingest_device_ptrs(self, receivers: np.ndarray, ptrs, sink=None) -> None:
        """modes_pool_ingest_device: the same from raw device addresses of the pool's device, written before the call."""
        fn = sink if sink is not None else C.cast(None, POOL_SINK_FN)
        self._check(lib().modes_pool_ingest_device(self._h, _ptr(receivers), ptrs, receivers.size, fn, None))

    def submit(self, receivers, buffers) -> None:
        """Upload + kernels, no waiting; `buffers` are kept alive until the matching collect()."""
        if self._on_gpu(buffers):
            ids, ptrs, keep = self._device_buffers(receivers, buffers)
            self._check(lib().modes_pool_submit_device(self._h, _ptr(ids), ptrs, ids.size))
            self._inflight = getattr(self, "_inflight", []) + [(ids, keep)]
            return
        ids, bufs = self._buffers(receivers, buffers)
        ptrs = (C.c_void_p * len(bufs))(*[b.ctypes.data for b in bufs])
        self._check(lib().modes_pool_submit(self._h, _ptr(ids), ptrs, ids.size))
        self._inflight = getattr(self, "_inflight", []) + [(ids, bufs)]

    def submit_ptrs(self, receivers: np.ndarray, ptrs) -> None:
        self._check(lib().modes_pool_submit(self._h, _ptr(receivers), ptrs, receivers.size))

    def submit_device_ptrs(self, receivers: np.ndarray, ptrs) -> None:
        """modes_pool_submit_device: raw device addresses, which must stay valid and unchanged until collect()."""
        self._check(lib().modes_pool_submit_device(self._h, _ptr(receivers), ptrs, receivers.size))

    def collect(self, sink="collect") -> None:
        """Wait for the oldest submitted batch, resolve it, deliver its messages (sink=None: only to the output array)."""
        fn = self._fn if sink == "collect" else (sink if sink is not None else C.cast(None, POOL_SINK_FN))
        self._check(lib().modes_pool_collect(self._h, fn, None))
        if getattr(self, "_inflight", None):
            self._inflight.pop(0)

    def resolve(self, receivers, cands: np.ndarray, tiles: np.ndarray) -> None:
        """The host half alone over records of a batch laid out pad, data, pad, data, ..."""
        ids = np.ascontiguousarray(receivers, dtype=np.uint32)
        cands = np.ascontiguousarray(cands); tiles = np.ascontiguousarray(tiles)
        assert tiles.size == tiles_for(2 * ids.size)
        self._check(lib().modes_pool_resolve(self._h, _ptr(ids), ids.size, _ptr(cands), _ptr(tiles), self._fn, None))

    def take(self, receiver: int) -> list:
        out, self.messages[receiver] = self.messages[receiver], []
        return out

    def set_output_array(self, capacity: int):
        """Messages of all receivers into one array (+ the receiver of each), restarted by rearm_output()."""
        self._out = (Message * capacity)()
        self._out_rx = np.zeros(capacity, dtype=np.uint32)
        self._check(lib().modes_pool_set_output(self._h, C.addressof(self._out), _ptr(self._out_rx), capacity))
        return self._out, self._out_rx

    def rearm_output(self) -> None:
        self._check(lib().modes_pool_set_output(self._h, C.addressof(self._out), _ptr(self._out_rx), len(self._out)))

    def output_count(self) -> int:
        return int(lib().modes_pool_output_count(self._h))

    def stats(self, receiver: int) -> dict:
        st = Stats()
        lib().modes_pool_stats(self._h, receiver, C.byref(st))
        return dict(zip(STAT_NAMES, [int(x) for x in st.v]))

    def set_signal(self, on: bool) -> None:
        """Measure the signal level for batches submitted from now on (modes_pool_set_signal)."""
        self._check(lib().modes_pool_set_signal(self._h, int(bool(on))))

    def set_arrival(self, on: bool) -> None:
        """Measure the arrival time for batches submitted from now on (modes_pool_set_arrival)."""
        self._check(lib().modes_pool_set_arrival(self._h, int(bool(on))))

    def set_carrier(self, on: bool) -> None:
        """Measure the carrier frequency for batches submitted from now on (modes_pool_set_carrier)."""
        self._check(lib().modes_pool_set_carrier(self._h, int(bool(on))))

    def set_levels(self, on: bool) -> None:
        """Measure the levels of batches submitted from now on (modes_pool_set_levels)."""
        self._check(lib().modes_pool_set_levels(self._h, int(bool(on))))

    def set_recovery(self, on: bool) -> None:
        """Recover weak DF17/DF18 frames in batches submitted from now on (modes_pool_set_recovery)."""
        self._check(lib().modes_pool_set_recovery(self._h, int(bool(on))))

    def recovery_stats(self, receiver: int) -> dict:
        st = RecoveryStats()
        self._check(lib().modes_pool_recovery_stats(self._h, receiver, C.byref(st)))
        return st.as_dict()

    def set_weak_preambles(self, on: bool) -> None:
        """Also recover at weak preambles in batches submitted from now on (modes_pool_set_weak_preambles)."""
        self._check(lib().modes_pool_set_weak_preambles(self._h, int(bool(on))))

    def weak_recovery_stats(self, receiver: int) -> dict:
        st = RecoveryStats()
        self._check(lib().modes_pool_weak_stats(self._h, receiver, C.byref(st)))
        return st.as_dict()

    def take_levels(self, receiver: int) -> np.ndarray:
        """The receiver's queued level records (LEVEL_DTYPE), its own buffer indices, oldest first."""
        n = int(lib().modes_pool_take_levels(self._h, receiver, None, 0))
        out = np.zeros(n, dtype=LEVEL_DTYPE)
        got = int(lib().modes_pool_take_levels(self._h, receiver, _ptr(out), n)) if n else 0
        return out[:got]

    def set_spectrum(self, on: bool) -> None:
        """Measure the input spectra of batches submitted from now on (modes_pool_set_spectrum)."""
        self._check(lib().modes_pool_set_spectrum(self._h, int(bool(on))))

    def take_spectra(self, receiver: int) -> np.ndarray:
        """The receiver's queued spectrum records (SPECTRUM_DTYPE), its own buffer indices, oldest first."""
        n = int(lib().modes_pool_take_spectra(self._h, receiver, None, 0))
        out = np.zeros(n, dtype=SPECTRUM_DTYPE)
        got = int(lib().modes_pool_take_spectra(self._h, receiver, _ptr(out), n)) if n else 0
        return out[:got]

    def buffers(self, receiver: int) -> int:
        return int(lib().modes_pool_buffers(self._h, receiver))

    def set_input_rate(self, receiver: int, hz: int) -> None:
        """The receiver's input sample rate, 2_000_000 or 2_400_000 (modes_pool_set_input_rate); refused
        while it has a stream in progress (until reset(receiver), which keeps the rate)."""
        self._check(lib().modes_pool_set_input_rate(self._h, int(receiver), int(hz)))

    def set_input_format(self, receiver: int, fmt: str, shift: int | None = None) -> None:
        """The receiver's sample format, one of INPUT_FORMATS, and its shift (None: the format's default)
        (modes_pool_set_input_format); refused while it has a stream in progress (until reset(receiver),
        which keeps the format)."""
        if fmt not in INPUT_FORMATS:
            raise ValueError(f"input format {fmt!r} is not one of {sorted(INPUT_FORMATS)}")
        self._check(lib().modes_pool_set_input_format(self._h, int(receiver), INPUT_FORMATS[fmt],
                                                      -1 if shift is None else int(shift)))
        self._bytes[receiver] = BUFFER_BYTES * (1 if fmt == "uc8" else 2)

    def reset(self, receiver: int) -> None:
        lib().modes_pool_reset(self._h, receiver)
        self.messages[receiver] = []

    def close(self):
        if self._h:
            lib().modes_pool_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def decode_captures(captures, *, input_rate: int = 2_000_000, input_format: str = "uc8", input_shift: int | None = None,
                    max_batch: int = 0, **switches_and_flags) -> list:
    """Decode many finite captures at once, each as one receiver of a ReceiverPool: returns each capture's
    messages, equal to Decoder(same settings).decode(capture).  captures: file paths or uint8 arrays, all of
    one rate and format.  Every capture is fed one buffer per call, in calls of up to max_batch receivers (0:
    all of them) with two batches in flight, and then finished with its tail.  switches_and_flags: the
    ReceiverPool switches (signal, levels, recover, ...) and modes_config flags (fix_errors, aggressive,
    check_crc, drop_eof_buffer, device)."""
    data = [np.fromfile(c, dtype=np.uint8) if isinstance(c, (str, os.PathLike)) else
            (np.frombuffer(c, dtype=np.uint8) if isinstance(c, (bytes, bytearray)) else
             np.ascontiguousarray(c, dtype=np.uint8).reshape(-1)) for c in captures]
    n = len(data)
    if not n:
        return []
    full = BUFFER_BYTES * (1 if input_format == "uc8" else 2)
    mb = max_batch if 0 < max_batch < n else n
    with ReceiverPool(n, max_batch=mb, input_rate=input_rate, input_format=input_format, input_shift=input_shift,
                      **switches_and_flags) as pool:
        whole = [d.size // full for d in data]
        in_flight = 0
        for k in range(max(whole)):
            ids = [i for i in range(n) if whole[i] > k]
            for g in range(0, len(ids), mb):
                group = ids[g: g + mb]
                if in_flight == 2:
                    pool.collect()
                    in_flight -= 1
                pool.submit(group, [data[i][k * full: (k + 1) * full] for i in group])
                in_flight += 1
        while in_flight:
            pool.collect()
            in_flight -= 1
        for g in range(0, n, mb):
            group = list(range(g, min(g + mb, n)))
            pool.finish(group, [data[i][whole[i] * full:] for i in group])
        return [pool.take(i) for i in range(n)]


# ---- SURVEY.md 8(f) item 3: aircraft tracker (host only) -------------------------------------

class Aircraft(C.Structure):
    """struct modes_aircraft == struct aircraft (dump1090.c:112-130)."""
    _fields_ = [("addr", C.c_uint32), ("hexaddr", C.c_char * 7), ("flight", C.c_char * 9),
                ("altitude", C.c_int32), ("speed", C.c_int32), ("track", C.c_int32),
                ("seen", C.c_int64), ("messages", C.c_int64),
                ("odd_cprlat", C.c_int32), ("odd_cprlon", C.c_int32), ("even_cprlat", C.c_int32), ("even_cprlon", C.c_int32),
                ("lat", C.c_double), ("lon", C.c_double), ("odd_cprtime", C.c_int64), ("even_cprtime", C.c_int64)]

    def as_tuple(self):
        return (self.addr, self.hexaddr, self.flight, self.altitude, self.speed, self.track, self.seen, self.messages,
                self.odd_cprlat, self.odd_cprlon, self.even_cprlat, self.even_cprlon, self.lat, self.lon,
                self.odd_cprtime, self.even_cprtime)


class Tracker:
    """Per-aircraft state over a delivered message stream: the reference's interactiveReceiveData
    with CPR position decoding, plus the SBS and JSON record formats.  Needs no GPU."""

    def __init__(self, check_crc: int = 1):
        L = lib()
        L.modes_tracker_create.restype = C.c_void_p
        L.modes_tracker_update.restype = C.POINTER(Aircraft)
        L.modes_tracker_update.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.modes_tracker_count.restype = C.c_size_t
        L.modes_tracker_count.argtypes = [C.c_void_p]
        L.modes_tracker_list.restype = C.c_size_t
        L.modes_tracker_list.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.modes_tracker_expire.restype = C.c_size_t
        L.modes_tracker_expire.argtypes = [C.c_void_p, C.c_int64, C.c_int]
        L.modes_tracker_reference.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.modes_tracker_format_json.restype = C.c_size_t
        L.modes_tracker_format_json.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]
        L.modes_tracker_destroy.argtypes = [C.c_void_p]
        L.modes_format_sbs.restype = C.c_size_t
        L.modes_format_sbs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        self._h = L.modes_tracker_create(int(check_crc))
        if not self._h:
            raise MemoryError("modes_tracker_create failed")

    def update(self, msg: "Message", now_ms: int):
        """Returns (Aircraft copy, SBS line) or None when the message is ignored."""
        p = lib().modes_tracker_update(self._h, C.byref(msg), int(now_ms))
        if not p:
            return None
        buf = C.create_string_buffer(512)
        n = lib().modes_format_sbs(C.byref(msg), p, buf, 512)
        a = Aircraft()
        C.memmove(C.byref(a), p, C.sizeof(Aircraft))
        return a, buf.raw[:n].decode("latin1")

    def aircraft(self):
        n = lib().modes_tracker_count(self._h)
        arr = (Aircraft * max(n, 1))()
        lib().modes_tracker_list(self._h, arr, n)
        return [arr[i] for i in range(n)]

    def expire(self, now_ms: int, ttl_seconds: int) -> int:
        return int(lib().modes_tracker_expire(self._h, int(now_ms), int(ttl_seconds)))

    def reference(self):
        lat, lon, cnt = C.c_double(), C.c_double(), C.c_int()
        lib().modes_tracker_reference(self._h, C.byref(lat), C.byref(lon), C.byref(cnt))
        return lat.value, lon.value, cnt.value

    def json(self, metric: int = 0) -> str:
        need = lib().modes_tracker_format_json(self._h, int(metric), None, 0)
        buf = C.create_string_buffer(need + 1)
        lib().modes_tracker_format_json(self._h, int(metric), buf, need + 1)
        return buf.raw[:need].decode("latin1")

    def table(self, now_ms: int, metric: int = 0, max_rows: int = 15) -> str:
        """The interactive-mode screen, dump1090.c:2167-2199."""
        f = lib().modes_tracker_format_table
        f.restype = C.c_size_t
        f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_size_t]
        need = f(self._h, int(metric), int(max_rows), int(now_ms), None, 0)
        buf = C.create_string_buffer(need + 1)
        f(self._h, int(metric), int(max_rows), int(now_ms), buf, need + 1)
        return buf.raw[:need].decode("latin1")

    def close(self):
        if self._h:
            lib().modes_tracker_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def cpr_nl(lat: float) -> int:
    f = lib().modes_cpr_nl
    f.restype = C.c_int
    f.argtypes = [C.c_double]
    return int(f(float(lat)))
