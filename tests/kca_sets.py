"""Which set of the evicting key cache a key falls in (consensus_b200/csrc/key_cache_assoc.cuh: kca_base), in Python, so
that a test can predict the per-set key counts of a launch.  tests/test_hostsim_key_cache_evict.py checks it against the
kernel's own function; the GPU tests take the seed and set count from sbv_debug_key_cache_sets."""
import numpy as np

M32 = 0xFFFFFFFF


def _mix(h, w):  # keygroup.cuh: kg_mix
    h = ((h ^ w) * 0x9E3779B1) & M32
    h ^= h >> 15
    return (h * 0x85EBCA77) & M32


def kc_hash(key: bytes, seed: int) -> int:  # key_cache.cuh: kc_hash over the key's little-endian 32-bit words
    h = seed & M32
    for w in np.frombuffer(key, "<u4").tolist():
        h = _mix(h, w)
    return h ^ (h >> 16)


def kca_set(key: bytes, seed: int, sets: int) -> int:
    return (kc_hash(key, seed) * sets) >> 32


def per_set_counts(keys, seed, sets):
    return np.bincount([kca_set(k, seed, sets) for k in keys], minlength=sets)
