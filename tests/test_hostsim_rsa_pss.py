"""RSA-PSS in the CPU simulation (tools/hostsim).  hs_rsa_pss_verify runs the whole device path with the arguments of
sbv_launch_rsa_pss: k_rsa_em (rsa_pss.cuh) in lockstep, a group of 16 lanes per item, then k_rsa_pss one thread per item.
hs_rsa_pss_decode runs k_rsa_pss alone over EMs computed here with Python integers, which keeps the lockstep
exponentiation (the slow part of the simulation) out of the salt-mode sweeps.

- every class of tests/rsa_pss_cases.py, on every size and hash, under auto, equals-hash and every explicit salt length
  of the corpus (each right, one short and one long) and 2^31 - 1, item for item against oracle_rsa.ref (decode only);
- the crafted classes item for item, and the salt modes picking their items;
- the whole path on a few items per size (valid, emLen = k - 1, a key-rule refusal, S = N, a PKCS #1 v1.5 signature),
  with EM and the unmasked DB as the kernels leave them over the signature buffer;
- the calls the entries refuse (salt_len < -1, a size or hash tag outside the set).
The GPU twin of this file is test_gpu_rsa_pss.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import rsa_pss_cases as pc
from oracle_rsa import ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")
PAIRS = [(k, h) for k in pc.SIZES for h in pc.HASHES]


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def recovered(c):
    """(EM over the signatures, the key and range verdicts) as k_rsa_em leaves them, in Python integers."""
    k = c["k"]
    em, ok = c["sig"].copy(), np.zeros(c["n"], np.uint8)
    for i in range(c["n"]):
        mod, e = c["mod"][i].tobytes(), int(c["exp"][i])
        n, s = int.from_bytes(mod, "big"), int.from_bytes(c["sig"][i].tobytes(), "big")
        if n % 2 and mod[0] and 2 <= e <= ref.E_MAX and s < n:
            em[i] = np.frombuffer(pow(s, e, n).to_bytes(k, "big"), np.uint8)
            ok[i] = 1
    return em, ok


def decode(hs, c, rec, salt_len, idx=None):
    idx = np.arange(c["n"]) if idx is None else idx
    em, ok = np.ascontiguousarray(rec[0][idx]), np.ascontiguousarray(rec[1][idx])
    mod, dig = np.ascontiguousarray(c["mod"][idx]), np.ascontiguousarray(c["digest"][idx])
    assert hs.hs_rsa_pss_decode(C.c_uint32(c["k"]), C.c_uint8(c["hash"]), C.c_int32(salt_len), C.c_size_t(len(idx)), _p(em), _p(mod), _p(dig),
                                _p(ok)) == 0
    return ok


def verify(hs, c, idx, salt_len, sig):
    mod, exp, dig = (np.ascontiguousarray(c[f][idx]) for f in ("mod", "exp", "digest"))
    ok = np.full(len(idx), 7, np.uint8)
    assert hs.hs_rsa_pss_verify(C.c_uint32(c["k"]), C.c_uint8(c["hash"]), C.c_int32(salt_len), C.c_size_t(len(idx)), _p(sig), _p(mod), _p(exp),
                                _p(dig), _p(ok)) == 0
    return ok


@pytest.mark.parametrize("k,hash", PAIRS)
def test_every_class_every_salt_mode(hs, k, hash):
    c = pc.make_cases(k, hash, seed=1)
    rec = recovered(c)
    for sl in pc.salt_lens(c):
        want = pc.want(c, sl)
        got = decode(hs, c, rec, sl)
        bad = [(c["cls"][i], int(g), int(w)) for i, (g, w) in enumerate(zip(got, want)) if g != w]
        assert not bad, (sl, bad)
        if sl in (ref.SALT_AUTO, ref.SALT_EQUALS_HASH):
            assert 0 < want.sum() < c["n"]


def test_salt_modes_pick_their_items(hs):
    """Auto accepts every valid salt length; equals-hash and an explicit length only the items of that length."""
    c = pc.make_cases(256, ref.SHA256, seed=1, short=True)
    rec = recovered(c)
    idx = np.array([i for i, cl in enumerate(c["cls"]) if cl.startswith("valid_salt_")])
    names = [c["cls"][i] for i in idx]
    assert decode(hs, c, rec, ref.SALT_AUTO, idx).tolist() == [1, 1, 1, 1]
    assert decode(hs, c, rec, ref.SALT_EQUALS_HASH, idx).tolist() == [int(nm == "valid_salt_hlen") for nm in names]
    S = pc.salts(256, ref.SHA256)
    for name in ("hlen", "mid", "max"):
        assert decode(hs, c, rec, S[name], idx).tolist() == [int(nm == f"valid_salt_{name}") for nm in names]
        assert decode(hs, c, rec, S[name] + 1, idx).tolist() == [0, 0, 0, 0]
        assert decode(hs, c, rec, S[name] - 1, idx).tolist() == [0, 0, 0, 0]
    assert decode(hs, c, rec, 2**31 - 1, idx).tolist() == [0, 0, 0, 0]


@pytest.mark.parametrize("k,hash", PAIRS)
def test_crafted_item_for_item(hs, k, hash):
    c = pc.make_cases(k, hash, seed=2, short=True)
    rec = recovered(c)
    idx = np.array([i for i, cl in enumerate(c["cls"]) if cl.startswith(("crafted", "cross"))])
    names = [c["cls"][i] for i in idx]
    assert any("top_bit" in nm for nm in names) and "crafted_bitlen_k-7_lead_byte" in names
    for sl in (ref.SALT_AUTO, ref.SALT_EQUALS_HASH, ref.HLEN[hash]):
        want = pc.want(c, sl)[idx]
        assert [nm for nm, w in zip(names, want) if w] == ["crafted_good"]
        got = decode(hs, c, rec, sl, idx)
        bad = [(nm, int(g), int(w)) for nm, g, w in zip(names, got, want) if g != w]
        assert not bad, (sl, bad)


# one hash per size for the 3072- and 4096-bit runs of the whole path, so that every hash meets a size above 2048 bits
WHOLE = [(256, ref.SHA256), (256, ref.SHA384), (256, ref.SHA512), (384, ref.SHA512), (512, ref.SHA384)]


@pytest.mark.parametrize("k,hash", WHOLE)
def test_whole_path_and_buffers(hs, k, hash):
    """k_rsa_em then k_rsa_pss: the verdicts, EM over the signature with DB unmasked in place, and the refused items'
    signatures left as they were."""
    c = pc.make_cases(k, hash, seed=1, short=True)
    names = ["valid_salt_hlen", f"valid_bitlen{8 * k - 7}_salt_hlen", "badkey_e1", "sigval_n", "cross_pkcs1"]
    if k != 256:
        names = names[:3]
    idx = np.array([c["cls"].index(nm) for nm in names])
    sig = np.ascontiguousarray(c["sig"][idx])
    got = verify(hs, c, idx, ref.SALT_AUTO, sig)
    assert got.tolist() == pc.want(c, ref.SALT_AUTO)[idx].tolist() == [1, 1, 0, 0, 0][:len(names)]
    hl = ref.HLEN[hash]
    for j, i in enumerate(idx[:2]):
        n = int.from_bytes(c["mod"][i].tobytes(), "big")
        em = pow(int.from_bytes(c["sig"][i].tobytes(), "big"), int(c["exp"][i]), n).to_bytes(k, "big")
        lead = 1 if c["mod"][i][0] == 1 else 0
        body = em[lead:]
        db_len = len(body) - hl - 1
        db = bytearray(x ^ y for x, y in zip(body[:db_len], ref.mgf1(body[db_len:db_len + hl], db_len, hash)))
        db[0] &= 0xFF >> (8 * len(body) - (n.bit_length() - 1))
        assert sig[j].tobytes() == em[:lead] + bytes(db) + body[db_len:], names[j]
    assert all(np.array_equal(sig[j], c["sig"][idx[j]]) for j in range(2, min(4, len(names))))  # e = 1, S = N: refused, S kept


def test_entries_refuse_bad_calls(hs):
    z, e, ok = np.zeros(512, np.uint8), np.full(1, 65537, np.uint32), np.full(1, 0x5A, np.uint8)
    for mb, h, sl in ((256, 0, -2), (256, 0, -2**31), (255, 0, 0), (256, 3, 0)):
        assert hs.hs_rsa_pss_verify(C.c_uint32(mb), C.c_uint8(h), C.c_int32(sl), C.c_size_t(1), _p(z), _p(z), _p(e), _p(z), _p(ok)) == -1
        assert hs.hs_rsa_pss_decode(C.c_uint32(mb), C.c_uint8(h), C.c_int32(sl), C.c_size_t(1), _p(z), _p(z), _p(z), _p(ok)) == -1
        assert ok[0] == 0x5A
