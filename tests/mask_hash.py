"""Host copy of the counter hash behind every in-kernel dropout / zoneout mask (t2_common.cuh: hash_u32, hash_seed, hash_bits32,
hash_uniform32, hash_keep16), in wrapping uint64 / uint32 numpy arithmetic, so that a test can rebuild the exact mask a kernel drew."""
import numpy as np

_U64 = np.uint64
_U32 = np.uint32


def hash_u32(seed, idx):
    idx = np.asarray(idx, dtype=_U64)
    with np.errstate(over="ignore"):
        z = _U64(seed) + _U64(0x9E3779B97F4A7C15) * (idx + _U64(1))
        z = (z ^ (z >> _U64(30))) * _U64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> _U64(27))) * _U64(0x94D049BB133111EB)
        z = z ^ (z >> _U64(31))
    return (z >> _U64(32)).astype(_U32)


def hash_seed(seed, stream):
    return int(hash_u32(seed, np.array([stream], dtype=_U64))[0])


def hash_bits32(hs, idx):
    idx = np.asarray(idx, dtype=_U64)
    lo = (idx & _U64(0xFFFFFFFF)).astype(_U32)
    hi = (idx >> _U64(32)).astype(_U32)
    with np.errstate(over="ignore"):
        h = _U32(hs) ^ (lo * _U32(0x9E3779B1)) ^ (hi * _U32(0x85EBCA77))
        h ^= h >> _U32(16)
        h *= _U32(0x85EBCA6B)
        h ^= h >> _U32(13)
        h *= _U32(0xC2B2AE35)
        h ^= h >> _U32(16)
    return h


def hash_uniform32(hs, idx):
    """U[0, 1) as float32: the top 24 bits of hash_bits32 times 2^-24"""
    return (hash_bits32(hs, idx) >> _U32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def keep_threshold16(p):
    """the 16-bit drop threshold the epilogues derive from a float32 rate: uint32(p * 65536.f)"""
    return int(np.float32(p) * np.float32(65536.0))


def hash_keep16(hs, idx, thr16):
    """pair form: one hash serves elements (idx & ~1, idx | 1), 16 bits each; kept iff its half >= thr16"""
    idx = np.asarray(idx, dtype=_U64)
    h = hash_bits32(hs, idx >> _U64(1))
    half = np.where((idx & _U64(1)) != 0, h >> _U32(16), h & _U32(0xFFFF))
    return half >= _U32(thr16)
