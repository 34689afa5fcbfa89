"""Registered RSA keys in the CPU simulation (tools/hostsim).  hs_rsa_kprep builds a registry with k_rsa_kprep
(rsa_keyed.cuh) as sbv_rsa_set_keys launches it; hs_rsa_verify_registered and hs_rsa_pss_verify_registered run the
registered verify kernels in lockstep with the launchers' arguments over that registry.

- every record against Python integers: n0', R^2 mod N, N's leading byte, the limbs of N and the validity flag, for every
  golden key (8k, 8k - 1, 8k - 4 and 8k - 7 bits, and the Blum keys) and every badkey class, all three sizes in one
  registry (the badkey items whose N rsa_r2 can take, e = 1 with S = EM among them, have n0' and R^2 too, so that the
  verdict tests below reach the validity flag as the only refusal);
- the registered verdicts item for item against oracle_rsa.ref on a short corpus per size, for both paddings;
- the slots that reject: past the registry, a key of another size (crafted so that its bytes, read at the call's size,
  would accept), an invalid key, and any slot of an empty registry;
- the calls the entries refuse.
The GPU twin of this file is test_gpu_rsa_registered.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import rsa_cases
import rsa_pss_cases as pc
import rsa_registered as rr
from oracle_rsa import ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def kprep(hs, reg):
    """(rec, pool) of the registry as hs_rsa_kprep builds it."""
    mb, mods, exp = reg.arrays()
    rec = np.full(8 * reg.n, 0xA5A5A5A5, np.uint32)
    pool = np.full(max(int(mb.sum()) // 2, 1), 0xA5A5A5A5, np.uint32)
    assert hs.hs_rsa_kprep(C.c_size_t(reg.n), _p(mb), _p(mods), _p(exp), _p(rec), _p(pool)) == 0
    return rec, pool


def verify(hs, pad, k, hash, slots, sig, digest, nslots, rec, pool, salt_len=ref.SALT_AUTO):
    n = len(slots)
    ok = np.full(n, 7, np.uint8)
    sig = np.ascontiguousarray(sig).copy()
    slots, digest = np.ascontiguousarray(slots, np.uint32), np.ascontiguousarray(digest)
    if pad == "pss":
        rc = hs.hs_rsa_pss_verify_registered(C.c_uint32(k), C.c_uint8(hash), C.c_int32(salt_len), C.c_size_t(n), _p(sig), _p(slots), C.c_uint32(nslots),
                                             _p(rec), _p(pool), _p(digest), _p(ok))
    else:
        rc = hs.hs_rsa_verify_registered(C.c_uint32(k), C.c_uint8(hash), C.c_size_t(n), _p(sig), _p(slots), C.c_uint32(nslots), _p(rec), _p(pool),
                                         _p(digest), _p(ok))
    assert rc == 0
    return ok


def test_records_against_python_integers(hs):
    keys = rr.record_keys()
    reg = rr.Registry()
    for _, mod, e in keys:
        reg.slot(mod, e)
    assert reg.n == len(keys), "every key distinct"
    rec, pool = kprep(hs, reg)
    offs = reg.offsets()
    valid = 0
    for i, (name, mod, e) in enumerate(keys):
        want = rr.record(mod, e, int(offs[i]))
        k = len(mod)
        got = np.concatenate([rec[8 * i:8 * i + 8], pool[int(offs[i]) // 2:int(offs[i]) // 2 + k // 2]])
        assert got.tolist() == want.tolist(), (name, k)
        valid += int(want[1])
    assert valid == 15, "the golden keys are valid, every badkey class is not"


def _short_corpus(pad, k, hash):
    return (rsa_cases if pad == "pkcs1" else pc).make_cases(k, hash, seed=3, short=True)


# one hash per size and padding, so that every hash meets every padding and each size meets two hashes
CASES = [("pkcs1", 256, ref.SHA256), ("pkcs1", 384, ref.SHA384), ("pkcs1", 512, ref.SHA512),
         ("pss", 256, ref.SHA384), ("pss", 384, ref.SHA512), ("pss", 512, ref.SHA256)]


@pytest.mark.parametrize("pad,k,hash", CASES)
def test_verdicts_match_ref(hs, pad, k, hash):
    c = _short_corpus(pad, k, hash)
    other = rsa_cases.make_cases(256 if k != 256 else 384, ref.SHA256, seed=3, short=True)
    reg, (_, slots) = rr.corpus_registry(other, c)  # the corpus's keys sit behind slots of another size
    rec, pool = kprep(hs, reg)
    want = c["want"] if pad == "pkcs1" else pc.want(c, ref.SALT_AUTO)
    got = verify(hs, pad, k, hash, slots, c["sig"], c["digest"], reg.n, rec, pool)
    bad = [(cl, int(g), int(w)) for cl, g, w in zip(c["cls"], got, want) if g != w]
    assert not bad, bad
    assert 0 < int(want.sum()) < c["n"]


@pytest.mark.parametrize("pad", ["pkcs1", "pss"])
def test_slots_that_reject(hs, pad):
    """A valid item accepts through its slot and rejects through a slot past the registry, a slot of another size (one
    whose bytes, read at the call's size, would accept: rr.size_trap), an invalid key's slot, and any slot of an empty
    registry."""
    k, hash = 256, ref.SHA256
    c = _short_corpus(pad, k, hash)
    i = c["cls"].index("valid_e65537" if pad == "pkcs1" else "valid_salt_hlen")
    mod = c["mod"][i].tobytes()
    trap_mod, trap_sig = rr.size_trap(mod, c["sig"][i].tobytes(), 384)
    reg = rr.Registry()
    s_big = reg.slot(trap_mod, int(c["exp"][i]))
    s_bad = reg.slot(mod, 1)  # the same modulus with e = 1: the key rule refuses it
    s_good = reg.slot(mod, int(c["exp"][i]))
    rec, pool = kprep(hs, reg)
    slots = np.array([s_good, reg.n, 2**32 - 1, s_big, s_bad, s_good], np.uint32)
    sig, dig = np.repeat(c["sig"][i:i + 1], 6, 0), np.repeat(c["digest"][i:i + 1], 6, 0)
    sig[3] = np.frombuffer(trap_sig, np.uint8)
    assert verify(hs, pad, k, hash, slots, sig, dig, reg.n, rec, pool).tolist() == [1, 0, 0, 0, 0, 1]
    assert verify(hs, pad, k, hash, slots, sig, dig, 0, None, None).tolist() == [0] * 6


def test_entries_refuse_bad_calls(hs):
    z, sl, ok = np.zeros(512, np.uint8), np.zeros(1, np.uint32), np.full(1, 0x5A, np.uint8)
    mb, e = np.array([300], np.uint32), np.full(1, 65537, np.uint32)
    rec, pool = np.zeros(8, np.uint32), np.zeros(256, np.uint32)
    assert hs.hs_rsa_kprep(C.c_size_t(1), _p(mb), _p(z), _p(e), _p(rec), _p(pool)) == -1
    assert not rec.any()
    for m, h, s in ((255, 0, 0), (256, 3, 0), (256, 0, -2)):
        assert hs.hs_rsa_pss_verify_registered(C.c_uint32(m), C.c_uint8(h), C.c_int32(s), C.c_size_t(1), _p(z), _p(sl), C.c_uint32(1), _p(rec), _p(pool),
                                               _p(z), _p(ok)) == -1
        if s == 0:
            assert hs.hs_rsa_verify_registered(C.c_uint32(m), C.c_uint8(h), C.c_size_t(1), _p(z), _p(sl), C.c_uint32(1), _p(rec), _p(pool), _p(z),
                                               _p(ok)) == -1
        assert ok[0] == 0x5A
