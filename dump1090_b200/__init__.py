"""dump1090_b200 — H100-native Mode S / ADS-B demodulator (drop-in for dump1090's --ifile decode path).

The compute lives in libmodes_b200.so (hand-written sm_90a CUDA behind the C ABI
of include/modes_b200.h); this package is the thin Python host side.
"""
from . import api, synth  # noqa: F401
from .api import Decoder, Resolver, Message  # noqa: F401
