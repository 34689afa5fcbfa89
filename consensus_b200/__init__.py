"""consensus_b200 — H100-native batched signature verification behind SmartBFT's api.Verifier.

The product is ``libsbv.so`` (hand-written sm_90a CUDA + a C ABI, include/sbv.h).  This package is
the thin ctypes binding used by the tests and bench.py; it never falls back to a CPU
implementation — if the library is missing or no CUDA device is usable, it raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsbv.so")

P256, P384, ED25519 = 0, 1, 2  # scheme tags of the mixed calls (the other calls take P256 / P384 only)
P256_SHA384, P384_SHA384 = 3, 4  # ECDSA over SHA-384: scheme tags of the mixed384 calls only
FIELD_BYTES = {P256: 32, P384: 48}
SHA256, SHA384, SHA512 = 0, 1, 2  # hash tags of the RSA calls (SBV_HASH_*)
HASH_BYTES = {SHA256: 32, SHA384: 48, SHA512: 64}
PSS_SALT_EQUALS_HASH, PSS_SALT_AUTO = -1, 0  # salt_len of the RSA-PSS calls (Go's PSSOptions.SaltLength)

SYMBOLS = [
    "sbv_create", "sbv_destroy", "sbv_last_error", "sbv_device_count", "sbv_verify_batch",
    "sbv_verify_batch_device", "sbv_verify_batch_der", "sbv_sha256_batch", "sbv_hash_verify_batch",
    "sbv_verify_mixed", "sbv_quorum", "sbv_compute_quorum", "sbv_set_keys", "sbv_kernel_launches",
    "sbv_probe_mad_rate", "sbv_profile_enable", "sbv_profile_read", "sbv_verify_registered",
    "sbv_verify_registered_device", "sbv_hash_verify_registered", "sbv_prepare_quorum", "sbv_verify_quorum",
    "sbv_comm_unique_id", "sbv_comm_init_rank", "sbv_comm_ranks", "sbv_gather_verdicts_device", "sbv_gather_words_device",
    "sbv_verify_batch_ranked", "sbv_host_alloc", "sbv_host_free", "sbv_ed25519_verify_batch",
    "sbv_ed25519_set_keys", "sbv_ed25519_verify_registered", "sbv_ed25519_verify_quorum", "sbv_mixed_verify_registered",
    "sbv_mixed_verify_quorum", "sbv_mixed_verify_batch", "sbv_sha384_batch", "sbv_hash384_verify_batch", "sbv_hash384_verify_registered",
    "sbv_key_cache_reserve", "sbv_key_cache_stats", "sbv_key_cache_reserve_evicting", "sbv_key_cache_stats_ex",
    "sbv_mixed384_verify_registered", "sbv_mixed384_verify_batch", "sbv_mixed384_verify_quorum",
    "sbv_sha512_batch", "sbv_rsa_verify_batch", "sbv_rsa_hash_verify_batch",
    "sbv_rsa_pss_verify_batch", "sbv_rsa_pss_hash_verify_batch",
    "sbv_rsa_set_keys", "sbv_rsa_verify_registered", "sbv_rsa_hash_verify_registered", "sbv_rsa_pss_verify_registered",
    "sbv_rsa_pss_hash_verify_registered", "sbv_rsa_verify_quorum", "sbv_rsa_pss_verify_quorum",
]


class EngineFault(RuntimeError):
    """An engine fault (CUDA error, bad argument).  Never a verdict — callers must fail-stop."""


_lib = None


def load_library() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise EngineFault(f"{LIB_PATH} is missing — run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(there is no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        lib.sbv_last_error.restype = C.c_char_p
        lib.sbv_kernel_launches.restype = C.c_uint64
        lib.sbv_probe_mad_rate.restype = C.c_double
        lib.sbv_destroy.restype = None
        lib.sbv_compute_quorum.restype = None
        _lib = lib
    return _lib


def _p8(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint8))


def _u8(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.uint8)
    return a


def compute_quorum(n: int):
    q, f = C.c_uint32(), C.c_uint32()
    load_library().sbv_compute_quorum(C.c_uint64(n), C.byref(q), C.byref(f))
    return q.value, f.value


class Engine:
    """One engine = 1..8 GPUs of one box (sbv_create)."""

    def __init__(self, devices=None, n_devices: int = 1):
        self._lib = load_library()
        self._h = C.c_void_p()
        if devices is not None:
            n_devices = len(devices)
            arr = (C.c_int * n_devices)(*devices)
        else:
            arr = None
        rc = self._lib.sbv_create(arr, C.c_int(n_devices), C.byref(self._h))
        if rc != 0:
            raise EngineFault(f"sbv_create failed ({rc}): no usable CUDA device? (there is no CPU fallback)")

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.sbv_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, rc, what):
        if rc != 0:
            raise EngineFault(f"{what} failed ({rc}): {self._lib.sbv_last_error(self._h).decode()}")

    @property
    def device_count(self) -> int:
        return self._lib.sbv_device_count(self._h)

    @property
    def kernel_launches(self) -> int:
        return int(self._lib.sbv_kernel_launches(self._h))

    def probe_mad_rate(self) -> float:
        return float(self._lib.sbv_probe_mad_rate(self._h))

    def profile_enable(self, on=True):
        self._check(self._lib.sbv_profile_enable(self._h, C.c_int(1 if on else 0)), "sbv_profile_enable")

    def profile_read(self):
        """(prep_ms, verify_ms, n_launch_pairs) summed since the last read; synchronise first."""
        p, v, k = C.c_double(), C.c_double(), C.c_uint64()
        self._check(self._lib.sbv_profile_read(self._h, C.byref(p), C.byref(v), C.byref(k)), "sbv_profile_read")
        return p.value, v.value, k.value

    def key_cache_reserve(self, p256=0, p384=0, ed25519=0):
        """Reserves, on every device, room for the tables of up to p256 / p384 / ed25519 keys that keys-per-item launches
        group, and empties any earlier cache; (0, 0, 0) frees it (sbv_key_cache_reserve)."""
        self._check(self._lib.sbv_key_cache_reserve(self._h, C.c_size_t(p256), C.c_size_t(p384), C.c_size_t(ed25519)),
                    "sbv_key_cache_reserve")

    def key_cache_stats(self, scheme) -> dict:
        """{capacity, resident, hits, misses} of one scheme's cache, summed over devices (sbv_key_cache_stats)."""
        out = (C.c_uint64 * 4)()
        self._check(self._lib.sbv_key_cache_stats(self._h, C.c_uint8(scheme), out), "sbv_key_cache_stats")
        return dict(zip(("capacity", "resident", "hits", "misses"), (int(v) for v in out)))

    def key_cache_reserve_evicting(self, p256=0, p384=0, ed25519=0):
        """As key_cache_reserve, but the caches replace their least recently used tables when full (16 ways per set;
        each capacity is rounded up to a multiple of 16); (0, 0, 0) frees them (sbv_key_cache_reserve_evicting)."""
        self._check(self._lib.sbv_key_cache_reserve_evicting(self._h, C.c_size_t(p256), C.c_size_t(p384), C.c_size_t(ed25519)),
                    "sbv_key_cache_reserve_evicting")

    def key_cache_stats_ex(self, scheme) -> dict:
        """{capacity, resident, hits, misses, evictions, given_up} of one scheme's cache, summed over devices
        (sbv_key_cache_stats_ex); the fill-once cache reports 0 for the last two."""
        out = (C.c_uint64 * 6)()
        self._check(self._lib.sbv_key_cache_stats_ex(self._h, C.c_uint8(scheme), out), "sbv_key_cache_stats_ex")
        return dict(zip(("capacity", "resident", "hits", "misses", "evictions", "given_up"), (int(v) for v in out)))

    # ---- host-buffer API (numpy arrays, or anything exposing a host pointer via .ctypes) ----
    def verify_batch(self, curve, r, s, qx, qy, digest, out=None) -> np.ndarray:
        L = FIELD_BYTES[curve]
        r, s, qx, qy, digest = map(_u8, (r, s, qx, qy, digest))
        n = r.size // L
        dlen = digest.size // n if n else 32
        ok = out if out is not None else np.zeros(n, np.uint8)
        self._check(self._lib.sbv_verify_batch(self._h, C.c_uint8(curve), C.c_size_t(n), _p8(r), _p8(s), _p8(qx), _p8(qy),
                                               _p8(digest), C.c_uint8(dlen), _p8(ok)), "sbv_verify_batch")
        return ok

    def verify_batch_ptr(self, curve, n, r, s, qx, qy, digest, dlen, ok):
        """Raw host pointers (ints) — used with pinned torch tensors."""
        vp = C.c_void_p
        self._check(self._lib.sbv_verify_batch(self._h, C.c_uint8(curve), C.c_size_t(n), vp(r), vp(s), vp(qx), vp(qy),
                                               vp(digest), C.c_uint8(dlen), vp(ok)), "sbv_verify_batch")

    def verify_batch_device(self, curve, n, d_r, d_s, d_qx, d_qy, d_digest, dlen, d_ok, stream=0, device_index=0):
        """Device pointers (ints); enqueued on `stream` (cudaStream_t as int), not synchronised."""
        vp = C.c_void_p
        self._check(self._lib.sbv_verify_batch_device(self._h, C.c_int(device_index), C.c_uint8(curve), C.c_size_t(n), vp(d_r),
                                                      vp(d_s), vp(d_qx), vp(d_qy), vp(d_digest), C.c_uint8(dlen), vp(d_ok),
                                                      vp(stream)), "sbv_verify_batch_device")

    def set_keys(self, curves, xy, ids=None, verification_seq=0):
        """Registers keys (slot i = key i) and builds their comb tables.  xy: (n, 2, L) or (n, 96) bytes."""
        curves = _u8(curves)
        n = curves.size
        xy = np.asarray(xy, dtype=np.uint8)
        if xy.size != n * 96:  # fixed-width per-curve arrays -> 48-byte slots
            L = xy.size // (2 * n)
            slots = np.zeros((n, 2, 48), np.uint8)
            slots[:, :, 48 - L:] = xy.reshape(n, 2, L)
            xy = slots
        xy = np.ascontiguousarray(xy.reshape(-1))
        ids = np.ascontiguousarray(ids if ids is not None else np.arange(n), dtype=np.uint64)
        self._check(self._lib.sbv_set_keys(self._h, C.c_uint64(verification_seq), C.c_size_t(n), ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                           _p8(curves), _p8(xy)), "sbv_set_keys")

    def verify_registered(self, curve, key_slot, r, s, digest) -> np.ndarray:
        key_slot = np.ascontiguousarray(key_slot, dtype=np.uint32)
        r, s, digest = map(_u8, (r, s, digest))
        n = key_slot.size
        dlen = digest.size // n if n else 32
        ok = np.zeros(n, np.uint8)
        self._check(self._lib.sbv_verify_registered(self._h, C.c_uint8(curve), C.c_size_t(n), key_slot.ctypes.data_as(C.POINTER(C.c_uint32)),
                                                    _p8(r), _p8(s), _p8(digest), C.c_uint8(dlen), _p8(ok)), "sbv_verify_registered")
        return ok

    def hash_verify_registered(self, curve, msgs, off, key_slot, r, s, _fn="sbv_hash_verify_registered") -> np.ndarray:
        msgs = _u8(msgs if len(msgs) else np.zeros(1, np.uint8))
        off = np.ascontiguousarray(off, dtype=np.uint64)
        key_slot = np.ascontiguousarray(key_slot, dtype=np.uint32)
        r, s = _u8(r), _u8(s)
        n = off.size - 1
        ok = np.zeros(n, np.uint8)
        self._check(getattr(self._lib, _fn)(self._h, C.c_uint8(curve), C.c_size_t(n), _p8(msgs), off.ctypes.data_as(C.POINTER(C.c_uint64)),
                                            key_slot.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(r), _p8(s), _p8(ok)), _fn)
        return ok

    def hash384_verify_registered(self, curve, msgs, off, key_slot, r, s) -> np.ndarray:
        """hash_verify_registered with e = the leftmost field bytes of SHA-384(M) (Go's ECDSAWithSHA384, ES384)."""
        return self.hash_verify_registered(curve, msgs, off, key_slot, r, s, _fn="sbv_hash384_verify_registered")

    def verify_registered_device(self, curve, n, d_slot, d_r, d_s, d_digest, dlen, d_ok, stream=0, device_index=0):
        vp = C.c_void_p
        self._check(self._lib.sbv_verify_registered_device(self._h, C.c_int(device_index), C.c_uint8(curve), C.c_size_t(n), vp(d_slot), vp(d_r),
                                                           vp(d_s), vp(d_digest), C.c_uint8(dlen), vp(d_ok), vp(stream)),
                    "sbv_verify_registered_device")

    def verify_batch_der(self, curve, sigs, sig_off, qxy, digest) -> np.ndarray:
        sigs = _u8(sigs if len(sigs) else np.zeros(1, np.uint8))
        sig_off = np.ascontiguousarray(sig_off, dtype=np.uint32)
        qxy, digest = _u8(qxy), _u8(digest)
        n = sig_off.size - 1
        dlen = digest.size // n if n else 32
        ok = np.zeros(n, np.uint8)
        self._check(self._lib.sbv_verify_batch_der(self._h, C.c_uint8(curve), C.c_size_t(n), _p8(sigs),
                                                   sig_off.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(qxy), _p8(digest),
                                                   C.c_uint8(dlen), _p8(ok)), "sbv_verify_batch_der")
        return ok

    def sha256_batch(self, msgs, off, _fn="sbv_sha256_batch", _width=32) -> np.ndarray:
        msgs = _u8(msgs if len(msgs) else np.zeros(1, np.uint8))
        off = np.ascontiguousarray(off, dtype=np.uint64)
        n = off.size - 1
        out = np.zeros((n, _width), np.uint8)
        self._check(getattr(self._lib, _fn)(self._h, C.c_size_t(n), _p8(msgs), off.ctypes.data_as(C.POINTER(C.c_uint64)), _p8(out)), _fn)
        return out

    def sha384_batch(self, msgs, off) -> np.ndarray:
        """SHA-384 of each message (msgs concatenated with off[n+1] byte offsets): n x 48 bytes."""
        return self.sha256_batch(msgs, off, _fn="sbv_sha384_batch", _width=48)

    def hash_verify_batch(self, curve, msgs, off, r, s, qx, qy, want_digest=False, _fn="sbv_hash_verify_batch", _width=32):
        msgs = _u8(msgs if len(msgs) else np.zeros(1, np.uint8))
        off = np.ascontiguousarray(off, dtype=np.uint64)
        r, s, qx, qy = map(_u8, (r, s, qx, qy))
        n = off.size - 1
        ok = np.zeros(n, np.uint8)
        dig = np.zeros((n, _width), np.uint8) if want_digest else None
        self._check(getattr(self._lib, _fn)(self._h, C.c_uint8(curve), C.c_size_t(n), _p8(msgs), off.ctypes.data_as(C.POINTER(C.c_uint64)),
                                            _p8(r), _p8(s), _p8(qx), _p8(qy), _p8(dig) if want_digest else None, _p8(ok)), _fn)
        return (ok, dig) if want_digest else ok

    def hash384_verify_batch(self, curve, msgs, off, r, s, qx, qy, want_digest=False):
        """hash_verify_batch with e = the leftmost field bytes of SHA-384(M) (Go's ECDSAWithSHA384, ES384); the digests, if
        asked for, are n x 48 bytes."""
        return self.hash_verify_batch(curve, msgs, off, r, s, qx, qy, want_digest, _fn="sbv_hash384_verify_batch", _width=48)

    def sha512_batch(self, msgs, off) -> np.ndarray:
        """SHA-512 of each message (msgs concatenated with off[n+1] byte offsets): n x 64 bytes."""
        return self.sha256_batch(msgs, off, _fn="sbv_sha512_batch", _width=64)

    def sha512_batch_ptr(self, n, msgs, off, digest_out):
        """Raw host pointers (ints) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_sha512_batch(self._h, C.c_size_t(n), vp(msgs), vp(off), vp(digest_out)), "sbv_sha512_batch")

    @staticmethod
    def _rsa_keys(modulus, pub_exp, key_slot):
        """The key arrays of an RSA call by their _ptr parameter names, and the item count they give: key_slot (registered), or
        modulus and pub_exp."""
        if key_slot is not None:
            key_slot = np.ascontiguousarray(key_slot, dtype=np.uint32)
            return {"key_slot": key_slot}, key_slot.size
        pub_exp = np.ascontiguousarray(pub_exp, dtype=np.uint32)
        return {"modulus": _u8(modulus), "pub_exp": pub_exp}, pub_exp.size

    def _rsa_digests(self, ptr, digest, sig, out, modulus=None, pub_exp=None, key_slot=None, **scalars):
        """The numpy form of the RSA calls over supplied digests: n = the keys' item count, k = the bytes per signature, and
        ptr (the call's _ptr form) given every array by keyword with the call's scalars.  Returns the verdicts (into out)."""
        keys, n = self._rsa_keys(modulus, pub_exp, key_slot)
        sig, digest = _u8(sig), _u8(digest)
        ok = out if out is not None else np.zeros(n, np.uint8)
        ptr(mod_bytes=sig.size // n if n else 256, n=n, digest=digest.ctypes.data, sig=sig.ctypes.data, ok=ok.ctypes.data,
            **{name: a.ctypes.data for name, a in keys.items()}, **scalars)
        return ok

    def _rsa_messages(self, ptr, hash, msgs, off, sig, want_digest, modulus=None, pub_exp=None, key_slot=None, **scalars):
        """The numpy form of the RSA calls that hash on the device: msgs concatenated with off[n+1] byte offsets, the rest as
        in _rsa_digests.  Returns the verdicts, and the n x hLen digests too with want_digest."""
        msgs = _u8(msgs if len(msgs) else np.zeros(1, np.uint8))
        off = np.ascontiguousarray(off, dtype=np.uint64)
        keys, _ = self._rsa_keys(modulus, pub_exp, key_slot)
        sig = _u8(sig)
        n = off.size - 1
        ok = np.zeros(n, np.uint8)
        dig = np.zeros((n, HASH_BYTES[hash]), np.uint8) if want_digest else None
        ptr(mod_bytes=sig.size // n if n else 256, hash=hash, n=n, msgs=msgs.ctypes.data, off=off.ctypes.data, sig=sig.ctypes.data,
            digest_out=dig.ctypes.data if want_digest else 0, ok=ok.ctypes.data, **{name: a.ctypes.data for name, a in keys.items()}, **scalars)
        return (ok, dig) if want_digest else ok

    def rsa_verify_batch(self, hash, digest, sig, modulus, pub_exp, out=None) -> np.ndarray:
        """RSA PKCS #1 v1.5 (Go crypto/rsa.VerifyPKCS1v15) over supplied digests: hash in {SHA256, SHA384, SHA512};
        digest = n x hLen bytes, sig and modulus = n x k bytes big-endian (k = 256, 384 or 512), pub_exp = n uint32."""
        return self._rsa_digests(self.rsa_verify_batch_ptr, digest, sig, out, hash=hash, modulus=modulus, pub_exp=pub_exp)

    def rsa_verify_batch_ptr(self, mod_bytes, hash, n, digest, sig, modulus, pub_exp, ok):
        """Raw host pointers (ints) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_rsa_verify_batch(self._h, C.c_uint32(mod_bytes), C.c_uint8(hash), C.c_size_t(n), vp(digest), vp(sig), vp(modulus),
                                                   vp(pub_exp), vp(ok)), "sbv_rsa_verify_batch")

    def rsa_hash_verify_batch(self, hash, msgs, off, sig, modulus, pub_exp, want_digest=False):
        """rsa_verify_batch with H = hash(M) computed on the device; msgs concatenated with off[n+1] byte offsets.  Returns
        the verdicts, and the n x hLen digests too with want_digest."""
        return self._rsa_messages(self.rsa_hash_verify_batch_ptr, hash, msgs, off, sig, want_digest, modulus=modulus, pub_exp=pub_exp)

    def rsa_hash_verify_batch_ptr(self, mod_bytes, hash, n, msgs, off, sig, modulus, pub_exp, digest_out, ok):
        """Raw host pointers (ints; digest_out may be 0) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_rsa_hash_verify_batch(self._h, C.c_uint32(mod_bytes), C.c_uint8(hash), C.c_size_t(n), vp(msgs), vp(off), vp(sig),
                                                        vp(modulus), vp(pub_exp), vp(digest_out or None), vp(ok)), "sbv_rsa_hash_verify_batch")

    def rsa_pss_verify_batch(self, hash, salt_len, digest, sig, modulus, pub_exp, out=None) -> np.ndarray:
        """RSA-PSS (Go crypto/rsa.VerifyPSS, MGF1 over the same hash) over supplied digests: salt_len = PSS_SALT_EQUALS_HASH,
        PSS_SALT_AUTO or the exact salt length; the other arguments as in rsa_verify_batch."""
        return self._rsa_digests(self.rsa_pss_verify_batch_ptr, digest, sig, out, hash=hash, salt_len=salt_len, modulus=modulus, pub_exp=pub_exp)

    def rsa_pss_verify_batch_ptr(self, mod_bytes, hash, salt_len, n, digest, sig, modulus, pub_exp, ok):
        """Raw host pointers (ints) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_rsa_pss_verify_batch(self._h, C.c_uint32(mod_bytes), C.c_uint8(hash), C.c_int32(salt_len), C.c_size_t(n), vp(digest),
                                                       vp(sig), vp(modulus), vp(pub_exp), vp(ok)), "sbv_rsa_pss_verify_batch")

    def rsa_pss_hash_verify_batch(self, hash, salt_len, msgs, off, sig, modulus, pub_exp, want_digest=False):
        """rsa_pss_verify_batch with H = hash(M) computed on the device; msgs concatenated with off[n+1] byte offsets.
        Returns the verdicts, and the n x hLen digests too with want_digest."""
        return self._rsa_messages(self.rsa_pss_hash_verify_batch_ptr, hash, msgs, off, sig, want_digest, salt_len=salt_len, modulus=modulus,
                                  pub_exp=pub_exp)

    def rsa_pss_hash_verify_batch_ptr(self, mod_bytes, hash, salt_len, n, msgs, off, sig, modulus, pub_exp, digest_out, ok):
        """Raw host pointers (ints; digest_out may be 0) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_rsa_pss_hash_verify_batch(self._h, C.c_uint32(mod_bytes), C.c_uint8(hash), C.c_int32(salt_len), C.c_size_t(n),
                                                            vp(msgs), vp(off), vp(sig), vp(modulus), vp(pub_exp), vp(digest_out or None), vp(ok)),
                    "sbv_rsa_pss_hash_verify_batch")

    def rsa_set_keys(self, mod_bytes, modulus, pub_exp):
        """Replaces the RSA key registry: slot i = (modulus i, pub_exp[i]), modulus i being mod_bytes[i] bytes (256, 384 or
        512) big-endian, the moduli concatenated in slot order; no keys empties it.  n0' and R^2 mod N are built once per
        key on every device; a slot whose key fails the key rule is kept, and its items reject."""
        mod_bytes = np.ascontiguousarray(mod_bytes, dtype=np.uint32).reshape(-1)
        pub_exp = np.ascontiguousarray(pub_exp, dtype=np.uint32).reshape(-1)
        modulus = _u8(modulus).reshape(-1)
        n = mod_bytes.size
        if pub_exp.size != n or modulus.size != int(mod_bytes.sum(dtype=np.uint64)):
            raise ValueError("pub_exp must hold one exponent and modulus mod_bytes[i] bytes per key")
        vp = C.c_void_p
        self._check(self._lib.sbv_rsa_set_keys(self._h, C.c_size_t(n), vp(mod_bytes.ctypes.data if n else None), vp(modulus.ctypes.data if n else None),
                                               vp(pub_exp.ctypes.data if n else None)), "sbv_rsa_set_keys")

    def rsa_verify_registered(self, hash, key_slot, digest, sig, out=None) -> np.ndarray:
        """rsa_verify_batch with the key of item i taken from registry slot key_slot[i] (rsa_set_keys); sig = n x k bytes,
        k the call's modulus size (a slot of another size rejects)."""
        return self._rsa_digests(self.rsa_verify_registered_ptr, digest, sig, out, hash=hash, key_slot=key_slot)

    def rsa_verify_registered_ptr(self, mod_bytes, hash, n, key_slot, digest, sig, ok):
        """Raw host pointers (ints) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_rsa_verify_registered(self._h, C.c_uint32(mod_bytes), C.c_uint8(hash), C.c_size_t(n), vp(key_slot), vp(digest),
                                                        vp(sig), vp(ok)), "sbv_rsa_verify_registered")

    def rsa_hash_verify_registered(self, hash, msgs, off, key_slot, sig, want_digest=False):
        """rsa_verify_registered with H = hash(M) computed on the device; msgs concatenated with off[n+1] byte offsets.
        Returns the verdicts, and the n x hLen digests too with want_digest."""
        return self._rsa_messages(self.rsa_hash_verify_registered_ptr, hash, msgs, off, sig, want_digest, key_slot=key_slot)

    def rsa_hash_verify_registered_ptr(self, mod_bytes, hash, n, msgs, off, key_slot, sig, digest_out, ok):
        """Raw host pointers (ints; digest_out may be 0) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_rsa_hash_verify_registered(self._h, C.c_uint32(mod_bytes), C.c_uint8(hash), C.c_size_t(n), vp(msgs), vp(off),
                                                             vp(key_slot), vp(sig), vp(digest_out or None), vp(ok)), "sbv_rsa_hash_verify_registered")

    def rsa_pss_verify_registered(self, hash, salt_len, key_slot, digest, sig, out=None) -> np.ndarray:
        """rsa_pss_verify_batch with the key of item i taken from registry slot key_slot[i] (rsa_set_keys)."""
        return self._rsa_digests(self.rsa_pss_verify_registered_ptr, digest, sig, out, hash=hash, salt_len=salt_len, key_slot=key_slot)

    def rsa_pss_verify_registered_ptr(self, mod_bytes, hash, salt_len, n, key_slot, digest, sig, ok):
        """Raw host pointers (ints) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_rsa_pss_verify_registered(self._h, C.c_uint32(mod_bytes), C.c_uint8(hash), C.c_int32(salt_len), C.c_size_t(n),
                                                            vp(key_slot), vp(digest), vp(sig), vp(ok)), "sbv_rsa_pss_verify_registered")

    def rsa_pss_hash_verify_registered(self, hash, salt_len, msgs, off, key_slot, sig, want_digest=False):
        """rsa_pss_verify_registered with H = hash(M) computed on the device; msgs concatenated with off[n+1] byte offsets.
        Returns the verdicts, and the n x hLen digests too with want_digest."""
        return self._rsa_messages(self.rsa_pss_hash_verify_registered_ptr, hash, msgs, off, sig, want_digest, salt_len=salt_len, key_slot=key_slot)

    def rsa_pss_hash_verify_registered_ptr(self, mod_bytes, hash, salt_len, n, msgs, off, key_slot, sig, digest_out, ok):
        """Raw host pointers (ints; digest_out may be 0) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_rsa_pss_hash_verify_registered(self._h, C.c_uint32(mod_bytes), C.c_uint8(hash), C.c_int32(salt_len), C.c_size_t(n),
                                                                 vp(msgs), vp(off), vp(key_slot), vp(sig), vp(digest_out or None), vp(ok)),
                    "sbv_rsa_pss_hash_verify_registered")

    def rsa_verify_quorum(self, hash, msgs, off, key_slot, sig, sig_off, instance, sender, signer, digest_match, n_instances, threshold,
                          self_id=None, _salt_len=None):
        """RSA commit votes against registered keys of any mix of sizes (rsa_set_keys): vote i's message msgs[off[i]:off[i+1]]
        is hashed on the device with `hash`, its signature sig[sig_off[i]:sig_off[i+1]] verified (PKCS #1 v1.5) under slot
        key_slot[i] at the size its length gives (a length other than 256, 384 or 512 bytes rejects), and the verdicts counted
        on the device; votes grouped by non-decreasing instance.  Returns (ok, valid_count, reached)."""
        msgs = _u8(msgs if len(msgs) else np.zeros(1, np.uint8))
        sig = _u8(sig if len(sig) else np.zeros(1, np.uint8))
        off = np.ascontiguousarray(off, dtype=np.uint64)
        sig_off = np.ascontiguousarray(sig_off, dtype=np.uint64)
        key_slot = np.ascontiguousarray(key_slot, dtype=np.uint32)
        instance = np.ascontiguousarray(instance, dtype=np.uint32)
        sender = np.ascontiguousarray(sender, dtype=np.uint16)
        signer = np.ascontiguousarray(signer, dtype=np.uint16)
        digest_match = _u8(digest_match)
        n = instance.size
        if off.size != n + 1 or sig_off.size != n + 1 or key_slot.size != n or sender.size != n or signer.size != n or digest_match.size != n:
            raise ValueError("off and sig_off must hold n + 1 offsets and every other column one entry per vote")
        ok = np.zeros(n, np.uint8)
        cnt = np.zeros(n_instances, np.uint32)
        reached = np.zeros(n_instances, np.uint8)
        if self_id is not None:
            self_id = np.ascontiguousarray(self_id, dtype=np.uint16)
        args = dict(n=n, msgs=msgs.ctypes.data, off=off.ctypes.data, key_slot=key_slot.ctypes.data, sig=sig.ctypes.data, sig_off=sig_off.ctypes.data,
                    instance=instance.ctypes.data, sender=sender.ctypes.data, signer=signer.ctypes.data, digest_match=digest_match.ctypes.data,
                    n_instances=n_instances, self_id=None if self_id is None else self_id.ctypes.data, threshold=threshold, ok=ok.ctypes.data,
                    valid_count=cnt.ctypes.data, reached=reached.ctypes.data)
        if _salt_len is None:
            self.rsa_verify_quorum_ptr(hash, **args)
        else:
            self.rsa_pss_verify_quorum_ptr(hash, _salt_len, **args)
        return ok, cnt, reached

    def rsa_verify_quorum_ptr(self, hash, n, msgs, off, key_slot, sig, sig_off, instance, sender, signer, digest_match, n_instances, self_id,
                              threshold, ok, valid_count, reached):
        """Raw host pointers (ints; self_id may be None) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_rsa_verify_quorum(self._h, C.c_uint8(hash), C.c_size_t(n), vp(msgs), vp(off), vp(key_slot), vp(sig), vp(sig_off),
                                                    vp(instance), vp(sender), vp(signer), vp(digest_match), C.c_size_t(n_instances), vp(self_id),
                                                    C.c_uint32(threshold), vp(ok), vp(valid_count), vp(reached)), "sbv_rsa_verify_quorum")

    def rsa_pss_verify_quorum(self, hash, salt_len, msgs, off, key_slot, sig, sig_off, instance, sender, signer, digest_match, n_instances,
                              threshold, self_id=None):
        """rsa_verify_quorum with RSA-PSS verdicts (salt_len as in rsa_pss_verify_batch)."""
        return self.rsa_verify_quorum(hash, msgs, off, key_slot, sig, sig_off, instance, sender, signer, digest_match, n_instances, threshold,
                                      self_id, _salt_len=salt_len)

    def rsa_pss_verify_quorum_ptr(self, hash, salt_len, n, msgs, off, key_slot, sig, sig_off, instance, sender, signer, digest_match, n_instances,
                                  self_id, threshold, ok, valid_count, reached):
        """Raw host pointers (ints; self_id may be None) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_rsa_pss_verify_quorum(self._h, C.c_uint8(hash), C.c_int32(salt_len), C.c_size_t(n), vp(msgs), vp(off), vp(key_slot),
                                                        vp(sig), vp(sig_off), vp(instance), vp(sender), vp(signer), vp(digest_match),
                                                        C.c_size_t(n_instances), vp(self_id), C.c_uint32(threshold), vp(ok), vp(valid_count), vp(reached)),
                    "sbv_rsa_pss_verify_quorum")

    def hash384_verify_batch_ptr(self, curve, n, msgs, off, r, s, qx, qy, digest_out, ok):
        """Raw host pointers (ints; digest_out may be 0) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_hash384_verify_batch(self._h, C.c_uint8(curve), C.c_size_t(n), vp(msgs), vp(off), vp(r), vp(s), vp(qx), vp(qy),
                                                       vp(digest_out or None), vp(ok)), "sbv_hash384_verify_batch")

    def ed25519_verify_batch(self, msgs, off, sig, pub, out=None) -> np.ndarray:
        """Ed25519 (Go crypto/ed25519.Verify): msgs concatenated with off[n+1] byte offsets, sig = n x 64 bytes (R || S),
        pub = n x 32 bytes.  Returns the n verdict bytes (into `out` if given)."""
        msgs = _u8(msgs if len(msgs) else np.zeros(1, np.uint8))
        off = np.ascontiguousarray(off, dtype=np.uint64)
        sig, pub = _u8(sig), _u8(pub)
        n = off.size - 1
        if sig.size != 64 * n or pub.size != 32 * n:
            raise ValueError("sig must hold 64 bytes and pub 32 bytes per message")
        ok = out if out is not None else np.zeros(n, np.uint8)
        self._check(self._lib.sbv_ed25519_verify_batch(self._h, C.c_size_t(n), _p8(msgs), off.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                       _p8(sig), _p8(pub), _p8(ok)), "sbv_ed25519_verify_batch")
        return ok

    def ed25519_verify_batch_ptr(self, n, msgs, off, sig, pub, ok):
        """Raw host pointers (ints) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_ed25519_verify_batch(self._h, C.c_size_t(n), vp(msgs), vp(off), vp(sig), vp(pub), vp(ok)),
                    "sbv_ed25519_verify_batch")

    def ed25519_set_keys(self, pub):
        """Replaces the Ed25519 key registry: slot i = the 32-byte encoding pub[i] (n x 32 bytes; n = 0 empties it) and
        builds a 384 KiB fixed-base table per decodable key on every device."""
        pub = _u8(pub)
        if pub.size % 32:
            raise ValueError("pub must hold 32 bytes per key")
        n = pub.size // 32
        self._check(self._lib.sbv_ed25519_set_keys(self._h, C.c_size_t(n), _p8(pub) if n else None), "sbv_ed25519_set_keys")

    def ed25519_verify_registered(self, msgs, off, key_slot, sig, out=None) -> np.ndarray:
        """Ed25519 with the key of item i taken from registry slot key_slot[i] (ed25519_set_keys): msgs concatenated with
        off[n+1] byte offsets, sig = n x 64 bytes (R || S).  Returns the n verdict bytes (into `out` if given)."""
        msgs = _u8(msgs if len(msgs) else np.zeros(1, np.uint8))
        off = np.ascontiguousarray(off, dtype=np.uint64)
        key_slot = np.ascontiguousarray(key_slot, dtype=np.uint32)
        sig = _u8(sig)
        n = off.size - 1
        if sig.size != 64 * n or key_slot.size != n:
            raise ValueError("sig must hold 64 bytes and key_slot one slot per message")
        ok = out if out is not None else np.zeros(n, np.uint8)
        self._check(self._lib.sbv_ed25519_verify_registered(self._h, C.c_size_t(n), _p8(msgs), off.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                            key_slot.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(sig), _p8(ok)),
                    "sbv_ed25519_verify_registered")
        return ok

    def ed25519_verify_registered_ptr(self, n, msgs, off, key_slot, sig, ok):
        """Raw host pointers (ints) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_ed25519_verify_registered(self._h, C.c_size_t(n), vp(msgs), vp(off), vp(key_slot), vp(sig), vp(ok)),
                    "sbv_ed25519_verify_registered")

    def ed25519_verify_quorum(self, msgs, off, key_slot, sig, instance, sender, signer, digest_match, n_instances, threshold,
                              self_id=None):
        """Ed25519 commit votes against registered keys (ed25519_set_keys): signatures verified, verdicts counted on the
        device.  msgs concatenated with off[n+1] byte offsets, sig = n x 64 bytes (R || S), votes grouped by
        non-decreasing instance.  Returns (ok, valid_count, reached)."""
        msgs = _u8(msgs if len(msgs) else np.zeros(1, np.uint8))
        off = np.ascontiguousarray(off, dtype=np.uint64)
        key_slot = np.ascontiguousarray(key_slot, dtype=np.uint32)
        instance = np.ascontiguousarray(instance, dtype=np.uint32)
        sender = np.ascontiguousarray(sender, dtype=np.uint16)
        signer = np.ascontiguousarray(signer, dtype=np.uint16)
        sig, digest_match = _u8(sig), _u8(digest_match)
        n = instance.size
        if off.size != n + 1 or sig.size != 64 * n or key_slot.size != n or sender.size != n or signer.size != n or digest_match.size != n:
            raise ValueError("off must hold n + 1 offsets, sig 64 bytes and every other column one entry per vote")
        ok = np.zeros(n, np.uint8)
        cnt = np.zeros(n_instances, np.uint32)
        reached = np.zeros(n_instances, np.uint8)
        sid = None
        if self_id is not None:
            self_id = np.ascontiguousarray(self_id, dtype=np.uint16)
            sid = self_id.ctypes.data_as(C.POINTER(C.c_uint16))
        u16 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint16))
        u32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))
        self._check(self._lib.sbv_ed25519_verify_quorum(self._h, C.c_size_t(n), _p8(msgs), off.ctypes.data_as(C.POINTER(C.c_uint64)), u32(key_slot),
                                                        _p8(sig), u32(instance), u16(sender), u16(signer), _p8(digest_match),
                                                        C.c_size_t(n_instances), sid, C.c_uint32(threshold), _p8(ok), u32(cnt), _p8(reached)),
                    "sbv_ed25519_verify_quorum")
        return ok, cnt, reached

    def ed25519_verify_quorum_ptr(self, n, msgs, off, key_slot, sig, instance, sender, signer, digest_match, n_instances, self_id, threshold,
                                  ok, valid_count, reached):
        """Raw host pointers (ints; self_id may be None) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(self._lib.sbv_ed25519_verify_quorum(self._h, C.c_size_t(n), vp(msgs), vp(off), vp(key_slot), vp(sig), vp(instance), vp(sender),
                                                        vp(signer), vp(digest_match), C.c_size_t(n_instances), vp(self_id), C.c_uint32(threshold),
                                                        vp(ok), vp(valid_count), vp(reached)), "sbv_ed25519_verify_quorum")

    def mixed_verify_registered(self, scheme, msgs, off, key_slot, sig96, out=None, _fn="sbv_mixed_verify_registered") -> np.ndarray:
        """Registered-key items of any scheme in one call: scheme[i] in {P256, P384, ED25519}, msgs concatenated with off[n+1]
        byte offsets, key_slot[i] a slot of the item's own registry (set_keys / ed25519_set_keys), sig96 = n x 96 bytes
        (P-256 r || s in [0, 64), P-384 r || s, Ed25519 R || S in [0, 64)).  Returns the n verdict bytes (into `out` if given)."""
        scheme = _u8(scheme)
        msgs = _u8(msgs if len(msgs) else np.zeros(1, np.uint8))
        off = np.ascontiguousarray(off, dtype=np.uint64)
        key_slot = np.ascontiguousarray(key_slot, dtype=np.uint32)
        sig96 = _u8(sig96)
        n = off.size - 1
        if scheme.size != n or sig96.size != 96 * n or key_slot.size != n:
            raise ValueError("scheme and key_slot must hold one entry and sig96 96 bytes per message")
        ok = out if out is not None else np.zeros(n, np.uint8)
        self._check(getattr(self._lib, _fn)(self._h, C.c_size_t(n), _p8(scheme), _p8(msgs), off.ctypes.data_as(C.POINTER(C.c_uint64)),
                                            key_slot.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(sig96), _p8(ok)), _fn)
        return ok

    def mixed_verify_registered_ptr(self, n, scheme, msgs, off, key_slot, sig96, ok, _fn="sbv_mixed_verify_registered"):
        """Raw host pointers (ints) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(getattr(self._lib, _fn)(self._h, C.c_size_t(n), vp(scheme), vp(msgs), vp(off), vp(key_slot), vp(sig96), vp(ok)), _fn)

    def mixed384_verify_registered(self, scheme, msgs, off, key_slot, sig96, out=None) -> np.ndarray:
        """mixed_verify_registered with ECDSA over SHA-384 too: scheme[i] in {P256, P384, ED25519, P256_SHA384, P384_SHA384};
        P256_SHA384 / P384_SHA384 items are packed as P256 / P384 items and hashed with SHA-384."""
        return self.mixed_verify_registered(scheme, msgs, off, key_slot, sig96, out, _fn="sbv_mixed384_verify_registered")

    def mixed384_verify_registered_ptr(self, n, scheme, msgs, off, key_slot, sig96, ok):
        self.mixed_verify_registered_ptr(n, scheme, msgs, off, key_slot, sig96, ok, _fn="sbv_mixed384_verify_registered")

    def mixed_verify_batch(self, scheme, msgs, off, sig96, key96, out=None, _fn="sbv_mixed_verify_batch") -> np.ndarray:
        """Items of any scheme with the key of each item in one call: scheme, msgs, off and sig96 as in
        mixed_verify_registered, key96 = n x 96 bytes (P-256 X || Y in [0, 64), P-384 X || Y, Ed25519 encoding in [0, 32)).
        Returns the n verdict bytes (into `out` if given)."""
        scheme = _u8(scheme)
        msgs = _u8(msgs if len(msgs) else np.zeros(1, np.uint8))
        off = np.ascontiguousarray(off, dtype=np.uint64)
        sig96, key96 = _u8(sig96), _u8(key96)
        n = off.size - 1
        if scheme.size != n or sig96.size != 96 * n or key96.size != 96 * n:
            raise ValueError("scheme must hold one entry and sig96 and key96 96 bytes per message")
        ok = out if out is not None else np.zeros(n, np.uint8)
        self._check(getattr(self._lib, _fn)(self._h, C.c_size_t(n), _p8(scheme), _p8(msgs), off.ctypes.data_as(C.POINTER(C.c_uint64)),
                                            _p8(sig96), _p8(key96), _p8(ok)), _fn)
        return ok

    def mixed_verify_batch_ptr(self, n, scheme, msgs, off, sig96, key96, ok, _fn="sbv_mixed_verify_batch"):
        """Raw host pointers (ints) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(getattr(self._lib, _fn)(self._h, C.c_size_t(n), vp(scheme), vp(msgs), vp(off), vp(sig96), vp(key96), vp(ok)), _fn)

    def mixed384_verify_batch(self, scheme, msgs, off, sig96, key96, out=None) -> np.ndarray:
        """mixed_verify_batch with ECDSA over SHA-384 too (scheme tags as in mixed384_verify_registered)."""
        return self.mixed_verify_batch(scheme, msgs, off, sig96, key96, out, _fn="sbv_mixed384_verify_batch")

    def mixed384_verify_batch_ptr(self, n, scheme, msgs, off, sig96, key96, ok):
        self.mixed_verify_batch_ptr(n, scheme, msgs, off, sig96, key96, ok, _fn="sbv_mixed384_verify_batch")

    def mixed_verify_quorum(self, scheme, msgs, off, key_slot, sig96, instance, sender, signer, digest_match, n_instances, threshold,
                            self_id=None, _fn="sbv_mixed_verify_quorum"):
        """Commit votes of a mixed consenter set: the items of mixed_verify_registered, verified and counted on the device
        (votes grouped by non-decreasing instance).  Returns (ok, valid_count, reached)."""
        scheme = _u8(scheme)
        msgs = _u8(msgs if len(msgs) else np.zeros(1, np.uint8))
        off = np.ascontiguousarray(off, dtype=np.uint64)
        key_slot = np.ascontiguousarray(key_slot, dtype=np.uint32)
        instance = np.ascontiguousarray(instance, dtype=np.uint32)
        sender = np.ascontiguousarray(sender, dtype=np.uint16)
        signer = np.ascontiguousarray(signer, dtype=np.uint16)
        sig96, digest_match = _u8(sig96), _u8(digest_match)
        n = instance.size
        if (off.size != n + 1 or scheme.size != n or sig96.size != 96 * n or key_slot.size != n or sender.size != n or signer.size != n
                or digest_match.size != n):
            raise ValueError("off must hold n + 1 offsets, sig96 96 bytes and every other column one entry per vote")
        ok = np.zeros(n, np.uint8)
        cnt = np.zeros(n_instances, np.uint32)
        reached = np.zeros(n_instances, np.uint8)
        sid = None
        if self_id is not None:
            self_id = np.ascontiguousarray(self_id, dtype=np.uint16)
            sid = self_id.ctypes.data_as(C.POINTER(C.c_uint16))
        u16 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint16))
        u32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))
        self._check(getattr(self._lib, _fn)(self._h, C.c_size_t(n), _p8(scheme), _p8(msgs), off.ctypes.data_as(C.POINTER(C.c_uint64)),
                                            u32(key_slot), _p8(sig96), u32(instance), u16(sender), u16(signer), _p8(digest_match),
                                            C.c_size_t(n_instances), sid, C.c_uint32(threshold), _p8(ok), u32(cnt), _p8(reached)), _fn)
        return ok, cnt, reached

    def mixed_verify_quorum_ptr(self, n, scheme, msgs, off, key_slot, sig96, instance, sender, signer, digest_match, n_instances, self_id,
                                threshold, ok, valid_count, reached, _fn="sbv_mixed_verify_quorum"):
        """Raw host pointers (ints; self_id may be None) — used with pinned buffers."""
        vp = C.c_void_p
        self._check(getattr(self._lib, _fn)(self._h, C.c_size_t(n), vp(scheme), vp(msgs), vp(off), vp(key_slot), vp(sig96), vp(instance),
                                            vp(sender), vp(signer), vp(digest_match), C.c_size_t(n_instances), vp(self_id),
                                            C.c_uint32(threshold), vp(ok), vp(valid_count), vp(reached)), _fn)

    def mixed384_verify_quorum(self, scheme, msgs, off, key_slot, sig96, instance, sender, signer, digest_match, n_instances, threshold,
                               self_id=None):
        """mixed_verify_quorum with ECDSA over SHA-384 too (scheme tags as in mixed384_verify_registered)."""
        return self.mixed_verify_quorum(scheme, msgs, off, key_slot, sig96, instance, sender, signer, digest_match, n_instances, threshold,
                                        self_id, _fn="sbv_mixed384_verify_quorum")

    def mixed384_verify_quorum_ptr(self, n, scheme, msgs, off, key_slot, sig96, instance, sender, signer, digest_match, n_instances, self_id,
                                   threshold, ok, valid_count, reached):
        self.mixed_verify_quorum_ptr(n, scheme, msgs, off, key_slot, sig96, instance, sender, signer, digest_match, n_instances, self_id,
                                     threshold, ok, valid_count, reached, _fn="sbv_mixed384_verify_quorum")

    def verify_mixed(self, curve_tag, r48, s48, qx48, qy48, digest32) -> np.ndarray:
        curve_tag, r48, s48, qx48, qy48, digest32 = map(_u8, (curve_tag, r48, s48, qx48, qy48, digest32))
        n = curve_tag.size
        ok = np.zeros(n, np.uint8)
        self._check(self._lib.sbv_verify_mixed(self._h, C.c_size_t(n), _p8(curve_tag), _p8(r48), _p8(s48), _p8(qx48), _p8(qy48),
                                               _p8(digest32), _p8(ok)), "sbv_verify_mixed")
        return ok

    # ---- one process per GPU ----
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        rc = load_library().sbv_comm_unique_id(buf)
        if rc != 0:
            raise EngineFault(f"sbv_comm_unique_id failed ({rc})")
        return bytes(buf)

    def comm_init_rank(self, uid: bytes, nranks: int, rank: int) -> int:
        buf = (C.c_uint8 * 128).from_buffer_copy(uid)
        ch = self._lib.sbv_comm_init_rank(self._h, buf, C.c_int(nranks), C.c_int(rank))
        if ch < 0:
            self._check(ch, "sbv_comm_init_rank")
        return ch

    def gather_verdicts_device(self, channel, d_ok, n, d_mask_all, stream=0):
        vp = C.c_void_p
        self._check(self._lib.sbv_gather_verdicts_device(self._h, C.c_int(channel), vp(d_ok), C.c_size_t(n), vp(d_mask_all), vp(stream)),
                    "sbv_gather_verdicts_device")

    def gather_words_device(self, channel, d_all, words, stream=0):
        vp = C.c_void_p
        self._check(self._lib.sbv_gather_words_device(self._h, C.c_int(channel), vp(d_all), C.c_size_t(words), vp(stream)), "sbv_gather_words_device")

    def verify_batch_ranked_ptr(self, channel, curve, n, r, s, qx, qy, digest, dlen, ok, mask_all):
        vp = C.c_void_p
        self._check(self._lib.sbv_verify_batch_ranked(self._h, C.c_int(channel), C.c_uint8(curve), C.c_size_t(n), vp(r), vp(s), vp(qx), vp(qy),
                                                      vp(digest), C.c_uint8(dlen), vp(ok), vp(mask_all)), "sbv_verify_batch_ranked")

    def verify_quorum(self, curve, r, s, qx, qy, digest, instance, sender, signer, digest_match, n_instances, threshold, self_id=None):
        """Commit votes: signatures verified, verdicts counted on the device.  Returns (ok, valid_count, reached)."""
        r, s, qx, qy, digest, digest_match = map(_u8, (r, s, qx, qy, digest, digest_match))
        instance = np.ascontiguousarray(instance, dtype=np.uint32)
        sender = np.ascontiguousarray(sender, dtype=np.uint16)
        signer = np.ascontiguousarray(signer, dtype=np.uint16)
        n = instance.size
        dlen = digest.size // n if n else 32
        ok = np.zeros(n, np.uint8)
        cnt = np.zeros(n_instances, np.uint32)
        reached = np.zeros(n_instances, np.uint8)
        sid = None
        if self_id is not None:
            self_id = np.ascontiguousarray(self_id, dtype=np.uint16)
            sid = self_id.ctypes.data_as(C.POINTER(C.c_uint16))
        u16 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint16))
        self._check(self._lib.sbv_verify_quorum(self._h, C.c_uint8(curve), C.c_size_t(n), _p8(r), _p8(s), _p8(qx), _p8(qy), _p8(digest), C.c_uint8(dlen),
                                                instance.ctypes.data_as(C.POINTER(C.c_uint32)), u16(sender), u16(signer), _p8(digest_match),
                                                C.c_size_t(n_instances), sid, C.c_uint32(threshold), _p8(ok),
                                                cnt.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(reached)), "sbv_verify_quorum")
        return ok, cnt, reached

    def prepare_quorum(self, instance, sender, digest_match, n_instances, threshold, self_id=None):
        instance = np.ascontiguousarray(instance, dtype=np.uint32)
        sender = np.ascontiguousarray(sender, dtype=np.uint16)
        digest_match = _u8(digest_match)
        cnt = np.zeros(n_instances, np.uint32)
        reached = np.zeros(n_instances, np.uint8)
        sid = None
        if self_id is not None:
            self_id = np.ascontiguousarray(self_id, dtype=np.uint16)
            sid = self_id.ctypes.data_as(C.POINTER(C.c_uint16))
        self._check(self._lib.sbv_prepare_quorum(self._h, C.c_size_t(instance.size), instance.ctypes.data_as(C.POINTER(C.c_uint32)),
                                                 sender.ctypes.data_as(C.POINTER(C.c_uint16)), _p8(digest_match), C.c_size_t(n_instances), sid,
                                                 C.c_uint32(threshold), cnt.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(reached)), "sbv_prepare_quorum")
        return cnt, reached

    def quorum(self, instance, sender, signer, digest_match, ok, n_instances, threshold, self_id=None):
        instance = np.ascontiguousarray(instance, dtype=np.uint32)
        sender = np.ascontiguousarray(sender, dtype=np.uint16)
        signer = np.ascontiguousarray(signer, dtype=np.uint16)
        digest_match, ok = _u8(digest_match), _u8(ok)
        cnt = np.zeros(n_instances, np.uint32)
        reached = np.zeros(n_instances, np.uint8)
        sid = None
        if self_id is not None:
            self_id = np.ascontiguousarray(self_id, dtype=np.uint16)
            sid = self_id.ctypes.data_as(C.POINTER(C.c_uint16))
        self._check(self._lib.sbv_quorum(self._h, C.c_size_t(instance.size), instance.ctypes.data_as(C.POINTER(C.c_uint32)),
                                         sender.ctypes.data_as(C.POINTER(C.c_uint16)), signer.ctypes.data_as(C.POINTER(C.c_uint16)),
                                         _p8(digest_match), _p8(ok), C.c_size_t(n_instances), sid, C.c_uint32(threshold),
                                         cnt.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(reached)), "sbv_quorum")
        return cnt, reached
