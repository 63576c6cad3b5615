"""The product's FarmHash (csrc/farmhash.cuh, the __host__ __device__ code the fingerprint / hash-partition kernels run,
compiled for the host inside libytgpu.so) against the reference's FarmHash: known answers of contrib/libs/farmhash
(tests/golden/farmhash_fingerprints.json) for every length class, and the oracle's restatement, which is pinned to the
same known answers (test_oracle_golden.py), for any byte string."""
import ctypes as C
import json
import os

import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

import oracle
from ytsaurus_b200 import capi

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "farmhash_fingerprints.json")
LENGTH_CLASSES = [0, 1, 3, 4, 7, 8, 16, 17, 32, 33, 63, 64, 65, 127, 128, 129, 191, 192, 193, 1023, 1024, 1025, 65536, 1 << 20]
# every length class of farmhashna::Hash64: 0, 1-3, 4-7, 8-16, 17-32, 33-64, >64 (incl. multiples of 64)
RANDOM_LENGTHS = list(range(0, 200)) + [255, 256, 257, 511, 512, 513, 1000, 4096, 65537]


def pattern_bytes(n):
    return bytes((i * 131 + 7) & 0xFF for i in range(n))


def det_bytes(n):
    """n pseudo-random bytes that depend on n only (splitmix64 stream seeded with n)."""
    out = bytearray()
    x = (0x9E3779B97F4A7C15 * (n + 1)) & (2**64 - 1)
    while len(out) < n:
        x = (x + 0x9E3779B97F4A7C15) & (2**64 - 1)
        z = x
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & (2**64 - 1)
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & (2**64 - 1)
        out += (z ^ (z >> 31)).to_bytes(8, "little")
    return bytes(out[:n])


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def _product():
    lib = capi.load()
    lib.ytgpu_hostcheck_fingerprint_bytes.restype = C.c_uint64
    lib.ytgpu_hostcheck_fingerprint_bytes.argtypes = [C.c_char_p, C.c_uint64]
    return lib


@settings(max_examples=1500, deadline=None)
@given(st.binary(max_size=400))
def test_fingerprint_of_any_byte_string(data):
    assert _product().ytgpu_hostcheck_fingerprint_bytes(data, len(data)) == oracle.farm_fingerprint_bytes(data)


@pytest.mark.parametrize("n", LENGTH_CLASSES)
def test_fingerprint_length_classes(n):
    data = pattern_bytes(n)
    assert _product().ytgpu_hostcheck_fingerprint_bytes(data, n) == int(golden()["fingerprint64_pattern_bytes"][str(n)])
