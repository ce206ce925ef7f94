"""Frames that exercise every path of the CRC repair (dump1090.c:795-894, decodeModesMessage
:1099-1128) and of the address cache behind it (:1196-1209).  TEST INFRASTRUCTURE.

Everything is derived from the Mode S generator polynomial through dump1090_b200.synth (its own
bitwise parity); nothing is read from the reference or from the product.  The low-weight codewords
of the code give the error patterns whose syndromes alias a 1- or 2-bit pattern: the decoder
"repairs" those into a different, parity-valid frame, and every implementation has to do exactly
what the reference does with them.

corpus() is a list of (frame14, label).  A label is "kind/base/detail": `kind` names the case
(see KINDS), `base` the transmitted frame (BASES), `detail` the flipped positions or the syndrome.
repair_stream(frac) puts the same frames on the air, one per 300-sample slot.
"""
from __future__ import annotations

import itertools
from functools import lru_cache

import numpy as np

from dump1090_b200 import synth

LONG, SHORT = 112, 56
ADDRESSES = (0x4840D6, 0xA1B2C3, 0x3C6586)
CONTROL_DFS = (0, 4, 5, 16, 20, 21, 24)        # never repaired: not DF 11/17/18
KINDS = ("clean", "flip1", "flip2", "mis1", "mis2", "flip3", "dfbit", "iid")
SLOT = 300


def nbits_of(df: int) -> int:
    """Frame length by downlink format (dump1090.c:746-753)."""
    return LONG if 16 <= df <= 21 else SHORT


def frame(df: int, low3: int, body: bytes) -> bytes:
    """A parity-valid frame of len(body) + 4 bytes, whatever length `df` implies."""
    data = bytes([((df & 31) << 3) | (low3 & 7)]) + body
    return data + synth.modes_parity(data).to_bytes(3, "big")


# ---- the code -------------------------------------------------------------------------------

@lru_cache(maxsize=None)
def bit_syndromes() -> tuple:
    """Syndrome of one flipped bit at position p (0..111) of a long frame: the parity of a data
    word with only bit p set, or the parity bit itself."""
    out = []
    for p in range(LONG):
        if p < LONG - 24:
            data = bytearray(11)
            data[p >> 3] = 0x80 >> (p & 7)
            out.append(synth.modes_parity(bytes(data)))
        else:
            out.append(1 << (LONG - 1 - p))
    return tuple(out)


def codewords(weight: int, positions) -> list:
    """Every set of `weight` (even) positions whose bit syndromes XOR to zero, as sorted tuples:
    meet in the middle on halves of weight/2."""
    syn = np.array(bit_syndromes(), dtype=np.int64)
    pos = np.array(sorted(positions))
    half = weight // 2
    combos = np.array(list(itertools.combinations(range(pos.size), half)), dtype=np.int64)
    s = np.bitwise_xor.reduce(syn[pos[combos]], axis=1)
    order = np.argsort(s, kind="stable")
    s, combos = s[order], combos[order]
    starts = np.flatnonzero(np.r_[True, s[1:] != s[:-1]])
    ends = np.r_[starts[1:], s.size]
    found = set()
    for a, b in zip(starts, ends):
        if b - a < 2:
            continue
        group = [set(pos[c].tolist()) for c in combos[a:b]]
        for x, y in itertools.combinations(group, 2):
            if not x & y:
                found.add(tuple(sorted(x | y)))
    return sorted(found)


@lru_cache(maxsize=None)
def long_codewords6() -> tuple:
    """Weight-6 codewords over positions 0..111 of a long frame."""
    return tuple(codewords(6, range(LONG)))


@lru_cache(maxsize=None)
def short_codewords8() -> tuple:
    """Weight-8 codewords over frame positions 0..55 of a short frame (table positions 56..111),
    in frame positions."""
    return tuple(tuple(p - (LONG - SHORT) for p in c) for c in codewords(8, range(LONG - SHORT, LONG)))


# ---- the frames ------------------------------------------------------------------------------

def _me(rng: synth.Counter) -> bytes:
    return bytes([(11 << 3) | rng.below(8)]) + bytes(rng.below(256) for _ in range(6))


@lru_cache(maxsize=None)
def _bases() -> dict:
    rng = synth.Counter(1090)
    b = {}
    for k, a in enumerate(ADDRESSES):
        aa = a.to_bytes(3, "big")
        tag = "abc"[k]
        b[f"df17{tag}"] = synth.make_frame(17, 5, aa + _me(rng))
        b[f"df18{tag}"] = synth.make_frame(18, 2, aa + _me(rng))
        b[f"df11{tag}"] = synth.make_frame(11, 5, aa)
        for df in CONTROL_DFS:
            body = bytes(rng.below(256) for _ in range(10 if 16 <= df <= 21 else 3))
            b[f"df{df}{tag}"] = synth.make_frame(df, rng.below(8), body, icao_for_ap=a)
        # parity-valid frames one DF bit away from DF 11 / 17 / 18 (short ones as short frames,
        # long ones as long frames)
        for target, body in ((11, aa), (17, aa + _me(rng)), (18, aa + _me(rng))):
            for k in range(5):
                b[f"src{target}_{k}{tag}"] = frame(target ^ (0x10 >> k), rng.below(8), body)
    return b


BASES = _bases()


def _pad(f: bytes) -> bytes:
    return f.ljust(14, b"\0")


def _flips(positions) -> str:
    return ",".join(str(p) for p in positions)


def _with_syndrome(f: bytes, s: int) -> bytes:
    """f with s XORed into its parity field: a frame whose syndrome is s."""
    return f[:-3] + (int.from_bytes(f[-3:], "big") ^ s).to_bytes(3, "big")


@lru_cache(maxsize=None)
def _corpus() -> tuple:
    out = []

    def add(kind, base, f, detail=""):
        out.append((_pad(f), f"{kind}/{base}/{detail}"))

    main = [n for n in BASES if n[:4] in ("df17", "df18", "df11")]
    controls = [n for n in BASES if n.startswith("df") and n not in main]
    for n in main + controls:                                  # announces every address first
        add("clean", n, BASES[n])
    for n in main + controls:
        f = BASES[n]
        for p in range(8 * len(f)):
            add("flip1", n, synth.flip_bits(f, [p]), str(p))
    for n in main:
        f = BASES[n]
        for pq in itertools.combinations(range(8 * len(f)), 2):
            add("flip2", n, synth.flip_bits(f, pq), _flips(pq))
    # miscorrections: error = codeword minus a 1- or 2-bit alias (which the decoder then flips)
    for n, cws in (("df17a", long_codewords6()), ("df18a", long_codewords6()), ("df11a", short_codewords8())):
        f = BASES[n]
        for c in cws:
            for k in (1, 2):
                for alias in itertools.combinations(c, k):
                    err = sorted(set(c) - set(alias))
                    add(f"mis{k}", n, synth.flip_bits(f, err), _flips(err))
    # three flipped bits outside the DF field: never repaired (no codeword of weight <= 5)
    rng = synth.Counter(3)
    for length, names in ((LONG, [n for n in main if nbits_of(BASES[n][0] >> 3) == LONG]),
                          (SHORT, [n for n in main if nbits_of(BASES[n][0] >> 3) == SHORT])):
        seen = set()
        while len(seen) < 1000:
            n = names[rng.below(len(names))]
            ps = tuple(sorted({5 + rng.below(length - 5) for _ in range(3)}))
            if len(ps) == 3 and (n, ps) not in seen:
                seen.add((n, ps))
                add("flip3", n, synth.flip_bits(BASES[n], ps), _flips(ps))
    # one DF bit flipped into DF 11 / 17 / 18
    for n in BASES:
        if n.startswith("src"):
            k = int(n.split("_")[1][0])
            add("dfbit", n, synth.flip_bits(BASES[n], [k]), str(k))
    # interrogator ids: a known DF11 address with every residual syndrome 1..79
    add("clean", "df11a", BASES["df11a"])
    for s in range(1, 80):
        add("iid", "df11a", _with_syndrome(BASES["df11a"], s), str(s))
    return tuple(out)


def corpus() -> list:
    """[(frame14 bytes, label)] in a fixed order; see the module docstring."""
    return list(_corpus())


def frames_array(items=None) -> np.ndarray:
    """The corpus frames as an (n, 14) uint8 array."""
    items = corpus() if items is None else items
    return np.frombuffer(b"".join(f for f, _ in items), dtype=np.uint8).reshape(-1, 14).copy()


def kind_of(label: str) -> str:
    return label.split("/", 1)[0]


def sent_of(label: str) -> bytes:
    """The frame that was transmitted before the errors of this item, padded to 14 bytes."""
    return _pad(BASES[label.split("/")[1]])


def coverage(items, msgs) -> dict:
    """What a decode of the corpus items exercised, from its messages (anything with the fields of
    checker.Msg, one per item): single-bit and two-bit repairs, miscorrections (a repair that
    yields a frame other than the transmitted one), DF11 frames repaired in their DF field, and
    DF11 frames accepted through the address cache with an interrogator id."""
    c = dict(single=0, pair=0, miscorrection=0, df11_df_bit=0, iid=0)
    for (f, label), m in zip(items, msgs):
        if m.iid:
            c["iid"] += 1
        if m.errorbit == -1:
            continue
        out = bytes(m.msg)
        nflip = sum(bin(a ^ b).count("1") for a, b in zip(f[: m.msgbits // 8], out))
        c["single" if nflip == 1 else "pair"] += 1
        if m.crcok and out[: m.msgbits // 8] != sent_of(label)[: m.msgbits // 8]:
            c["miscorrection"] += 1
        if m.msgtype == 11 and m.errorbit < 5:
            c["df11_df_bit"] += 1
    return c


# ---- the expected repair ----------------------------------------------------------------------

@lru_cache(maxsize=None)
def _byte_syndromes() -> np.ndarray:
    """[14, 256]: syndrome contribution of byte value v at byte k of a long frame."""
    syn = bit_syndromes()
    t = np.zeros((14, 256), dtype=np.int64)
    for k in range(14):
        for v in range(256):
            for j in range(8):
                if v & (0x80 >> j):
                    t[k, v] ^= syn[8 * k + j]
    return t


def syndromes(frames: np.ndarray) -> np.ndarray:
    """Syndrome of each (n, 14) frame over the length its DF field gives (dump1090.c:733-742)."""
    t = _byte_syndromes()
    longf = nbits_of_array(frames[:, 0] >> 3) == LONG
    s = np.zeros(frames.shape[0], dtype=np.int64)
    for k in range(14):
        s ^= np.where(longf, t[k, frames[:, k]], 0)
    for k in range(7):
        s ^= np.where(longf, 0, t[k + 7, frames[:, k]])
    return s


def nbits_of_array(df: np.ndarray) -> np.ndarray:
    return np.where((df >= 16) & (df <= 21), LONG, SHORT)


def table_lookup(table: np.ndarray, s: np.ndarray, bits: np.ndarray, maxfix: int):
    """fixBitErrors (dump1090.c:854-894) as array operations on the reference's own sorted
    bitErrorTable rows (syndrome, bits, pos0, pos1): which syndromes it repairs, how many bits, and
    the frame positions (pos1 is meaningless for one bit)."""
    i = np.minimum(np.searchsorted(table[:, 0], s), table.shape[0] - 1)
    nb, off = table[i, 1], LONG - bits
    p0, p1 = table[i, 2] - off, table[i, 3] - off
    ok = (table[i, 0] == s) & (nb <= maxfix) & (p0 >= 0) & (p0 < bits) & ((nb == 1) | ((p1 >= 0) & (p1 < bits)))
    return ok, np.where(ok, nb, 0), p0, p1


def model_repair(table: np.ndarray, frames: np.ndarray, fix: int, aggressive: int, s: np.ndarray | None = None):
    """decodeModesMessage's syndrome and repair (dump1090.c:1108-1128) on (n, 14) frames:
    (repaired frames, crc after the repair, errorbit or -1, bits fixed).  `s`: the frames'
    syndromes when the caller knows them."""
    df = frames[:, 0] >> 3
    bits = nbits_of_array(df)
    s = syndromes(frames) if s is None else s
    ok, nb, p0, p1 = table_lookup(table, s, bits, 2 if aggressive else 1)
    ok &= (s != 0) & bool(fix) & ((df == 11) | (df == 17) | (df == 18))
    out = frames.copy()
    for sel, p in ((ok, p0), (ok & (nb == 2), p1)):
        r = np.flatnonzero(sel)
        out[r, p[r] >> 3] ^= (0x80 >> (p[r] & 7)).astype(np.uint8)
    return out, np.where(ok, 0, s), np.where(ok, p0, -1), np.where(ok, nb, 0)


def sweep_chunks(base: bytes, chunk: int, with_zero: bool = True):
    """(syndromes, (n, 14) frames) covering base ^ S for every 24-bit S, S in the parity field."""
    f = np.frombuffer(base.ljust(14, b"\0"), dtype=np.uint8)
    nbytes = len(base)
    for lo in range(0 if with_zero else 1, 1 << 24, chunk):
        s = np.arange(lo, min(lo + chunk, 1 << 24), dtype=np.int64)
        frames = np.tile(f, (s.size, 1))
        for k in range(3):
            frames[:, nbytes - 3 + k] ^= (s >> (16 - 8 * k)).astype(np.uint8)
        yield s, frames


# ---- on the air ------------------------------------------------------------------------------

@lru_cache(maxsize=None)
def _stream(frac: float) -> bytes:
    rng = synth.Counter(77)
    frames = []
    for k, (f, _) in enumerate(_corpus()):
        nbytes = nbits_of(f[0] >> 3) // 8
        frames.append((SLOT * k + 40, f[:nbytes], 40.0, 2 * np.pi * rng.uniform(), frac))
    return synth.synth_stream(SLOT * len(frames) + 400, frames, sigma=0.8, seed=5).tobytes()


# A fractional offset at which the first attempt of some frames fails and the phase-corrected retry
# decodes and repairs them (found by scanning 0.05..0.95 with the oracle: at amplitude 40 only
# 0.45..0.55 lets the retry repair, and 0.55 the most, about 6 % of the repaired frames; see
# test_repair_stream_retries_carry_repairs).
RETRY_FRAC = 0.55


def repair_stream(frac: float = 0.0) -> np.ndarray:
    """The corpus as a u8 I/Q stream: one frame per 300-sample slot, amplitude 40, noise 0.8 LSB,
    every pulse delayed by `frac` of a sample."""
    return np.frombuffer(_stream(float(frac)), dtype=np.uint8).copy()
