"""oracle_ed25519 — CPU oracle for sbv_ed25519_verify_batch.  TEST INFRASTRUCTURE ONLY (never imported by consensus_b200).

`verify_batch` wraps liboracle_ed25519.so (ed25519_oracle.c: OpenSSL 3 EVP_PKEY_ED25519, multi-threaded);
`ref` is the independent pure-Python restatement of the accept set; `corpus` builds seeded corpora with every
corruption class.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import ref  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle_ed25519.so")


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "ed25519_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-C", _HERE, "liboracle_ed25519.so"])
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        _lib.orc_ed25519_bench.restype = C.c_double
    return _lib


def ncores() -> int:
    from oracle import ncores as n
    return n()


def _p8(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint8))


def _args(msgs, off, sig, pub):
    msgs = np.ascontiguousarray(msgs if len(msgs) else np.zeros(1, np.uint8), dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    sig = np.ascontiguousarray(sig, dtype=np.uint8)
    pub = np.ascontiguousarray(pub, dtype=np.uint8)
    n = off.size - 1
    assert sig.size == 64 * n and pub.size == 32 * n
    return msgs, off, sig, pub, n


def verify_batch(msgs, off, sig, pub, nthreads=None) -> np.ndarray:
    msgs, off, sig, pub, n = _args(msgs, off, sig, pub)
    ok = np.zeros(n, np.uint8)
    lib().orc_ed25519_verify_batch(C.c_size_t(n), _p8(msgs), off.ctypes.data_as(C.POINTER(C.c_uint64)), _p8(sig), _p8(pub), _p8(ok),
                                   C.c_int(nthreads or ncores()))
    return ok


def bench_verify(msgs, off, sig, pub, nthreads=None):
    """OpenSSL Ed25519 verification on nthreads cores; returns (seconds, verdicts)."""
    msgs, off, sig, pub, n = _args(msgs, off, sig, pub)
    ok = np.zeros(n, np.uint8)
    t = lib().orc_ed25519_bench(C.c_size_t(n), _p8(msgs), off.ctypes.data_as(C.POINTER(C.c_uint64)), _p8(sig), _p8(pub), _p8(ok),
                                C.c_int(nthreads or ncores()))
    return float(t), ok


def pubkey(seed: bytes) -> bytes:
    out = (C.c_uint8 * 32)()
    if lib().orc_ed25519_pubkey((C.c_uint8 * 32).from_buffer_copy(seed), out):
        raise ValueError("orc_ed25519_pubkey failed")
    return bytes(out)


def sign_batch(seeds, key_idx, msgs, off) -> np.ndarray:
    seeds = np.ascontiguousarray(seeds, dtype=np.uint8)
    key_idx = np.ascontiguousarray(key_idx, dtype=np.uint32)
    msgs = np.ascontiguousarray(msgs if len(msgs) else np.zeros(1, np.uint8), dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    n = key_idx.size
    sig = np.zeros((n, 64), np.uint8)
    if lib().orc_ed25519_sign_batch(C.c_size_t(n), _p8(seeds), key_idx.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(msgs),
                                    off.ctypes.data_as(C.POINTER(C.c_uint64)), _p8(sig)):
        raise RuntimeError("orc_ed25519_sign_batch failed")
    return sig
