"""Registered RSA keys for the tests of sbv_rsa_set_keys and the registered verify calls, shared by the CPU simulation
(tests/test_hostsim_rsa_registered.py) and the GPU tests (tests/test_gpu_rsa_registered.py).

- corpus_registry: a registry of the distinct (modulus, exponent) pairs of one or more corpora of tests/rsa_cases.py,
  tests/rsa_pss_cases.py or tests/rsa_edges.py, and each item's slot in it;
- record: the record and limbs a slot must hold (rsa_keyed.cuh), from Python integers;
- record_keys: every golden key of tests/golden/rsa_keys.npz and every badkey class, over all three sizes."""
from __future__ import annotations

import math

import numpy as np

import rsa_cases
import rsa_edges
from oracle_rsa import ref

SIZES = (256, 384, 512)


class Registry:
    """Keys in slot order: mod_bytes (uint32), modulus (the moduli concatenated, uint8), exp (uint32)."""

    def __init__(self):
        self.keys, self._slot = [], {}

    def slot(self, mod: bytes, e: int) -> int:
        key = (bytes(mod), int(e))
        if key not in self._slot:
            self._slot[key] = len(self.keys)
            self.keys.append(key)
        return self._slot[key]

    def add(self, c) -> np.ndarray:
        """The slots of corpus c's items, adding their keys."""
        return np.array([self.slot(c["mod"][i].tobytes(), c["exp"][i]) for i in range(c["n"])], np.uint32)

    @property
    def n(self):
        return len(self.keys)

    def arrays(self):
        mb = np.array([len(m) for m, _ in self.keys], np.uint32)
        mods = np.frombuffer(b"".join(m for m, _ in self.keys) + b"\0", np.uint8)[:-1].copy()
        return mb, mods, np.array([e for _, e in self.keys], np.uint32)

    def offsets(self):
        """The byte offset of each modulus in the concatenation (rsa_reg_layout)."""
        return np.concatenate([[0], np.cumsum([len(m) for m, _ in self.keys])])[:-1].astype(np.uint64)


def corpus_registry(*corpora):
    """(registry, [slots of each corpus]) with every distinct (modulus, exponent) of the corpora in one slot."""
    reg = Registry()
    return reg, [reg.add(c) for c in corpora]


def key_valid(mod: bytes, e: int) -> bool:
    return int.from_bytes(mod, "big") % 2 == 1 and mod[0] != 0 and 2 <= e <= ref.E_MAX


def record(mod: bytes, e: int, off: int) -> np.ndarray:
    """The 8 + 2K words of sbv_debug_rsa_key for a key at byte offset off of the moduli: {k, valid, ntop, n0', e, limb offset
    (64 bits), 0}, the K limbs of N and the K of R^2 mod N (little-endian); n0' and R^2 are zero unless N is odd with a
    nonzero top limb (invalid keys with such an N have them)."""
    k, N = len(mod), int.from_bytes(mod, "big")
    valid = key_valid(mod, e)
    arith = N % 2 == 1 and N >> (8 * k - 32) != 0
    ninv = (-pow(N, -1, 2**32)) % 2**32 if arith else 0
    r2 = pow(2, 2 * 8 * k, N) if arith else 0
    head = [k, int(valid), mod[0], ninv, e, (off // 2) & 0xFFFFFFFF, (off // 2) >> 32, 0]
    limbs = np.frombuffer(N.to_bytes(k, "little") + r2.to_bytes(k, "little"), np.uint32)
    return np.concatenate([np.array(head, np.uint32), limbs])


def record_keys():
    """Every golden key (8k, 8k - 1, 8k - 4 and 8k - 7 bits, and the Blum keys) with e = 65537, then the keys of every badkey
    class of tests/rsa_cases.py, for each size; the sizes interleaved so that the build's per-size launches each gather
    slots from all over the registry."""
    per = {k: [] for k in SIZES}
    for k in SIZES:
        for b in (8 * k, 8 * k - 1, 8 * k - 4, 8 * k - 7):
            per[k].append((f"std_{b}", rsa_edges.key(f"std_{b}").n.to_bytes(k, "big"), 65537))
        per[k].append((f"blum_{8 * k}", rsa_edges.key(f"blum_{8 * k}").n.to_bytes(k, "big"), 3))
        c = rsa_cases.make_cases(k, ref.SHA256, short=True)
        for i, cl in enumerate(c["cls"]):
            if cl.startswith("badkey"):
                per[k].append((cl, c["mod"][i].tobytes(), int(c["exp"][i])))
    out = []
    for j in range(max(len(v) for v in per.values())):
        for k in SIZES:
            if j < len(per[k]):
                out.append(per[k][j])
    return out


def size_trap(mod: bytes, sig: bytes, k_slot: int, seed: int = 0):
    """A registered key of k_slot bytes whose slot, read as a key of k = len(mod) < k_slot bytes, would accept sig: the
    k_slot-byte modulus and the k-byte signature to use instead of sig.  The slot's first K limbs (its low k bytes) are N =
    mod; the K words after them, which a reader of the wrong size takes for R^2 mod N, are limbs of the slot's own N and R^2,
    c * R^2 mod N for some c.  The signature returned is S / c mod N, so that S * c * R -- not S * R -- starts the
    exponentiation and S^e mod N, the EM that sig recovers, comes out.  Only the size check of the registered kernels
    refuses it: the slot's key has another size than the call's."""
    import random
    rng = random.Random(f"size-trap-{len(mod)}-{k_slot}-{seed}")
    N, kc, ks = int.from_bytes(mod, "big"), len(mod), k_slot
    assert mod[0] != 0 and ks > kc
    R = 2 ** (8 * kc)
    S = int.from_bytes(sig, "big")
    while True:
        H = rng.getrandbits(8 * (ks - kc)) | 1 << (8 * (ks - kc) - 1)  # the high part of the slot's modulus, top bit set
        M = N + (H << (8 * kc))
        r2m = pow(2, 2 * 8 * ks, M)
        fake = int.from_bytes((M.to_bytes(ks, "little") + r2m.to_bytes(ks, "little"))[kc:2 * kc], "little")
        if fake >= N or math.gcd(fake, N) != 1:
            continue
        c = fake * pow(R * R, -1, N) % N
        return M.to_bytes(ks, "big"), (S * pow(c, -1, N) % N).to_bytes(kc, "big")
