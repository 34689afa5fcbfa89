"""oracle_rsa.ref (the restatement of Go's crypto/rsa.VerifyPKCS1v15 in include/sbv.h) against OpenSSL, through
cryptography's RSAPublicNumbers(e, n).public_key().verify(sig, digest, PKCS1v15(), Prehashed(SHA-2)), over every class of
tests/rsa_cases.py whose key OpenSSL loads.

They agree on every class whose key OpenSSL loads but two, pinned here, where Go's rule as restated is the spec: an
exponent above 2^31 - 1 with a signature made under it (badkey_e_above_max, badkey_e4294967295).  OpenSSL accepts an odd
exponent up to its own, larger bound; Go's checkPub caps e at 2^31 - 1, so ref.py and the engine reject (the GPU and CPU
simulation files check the engine on the same items).  Classes whose key OpenSSL refuses to load (e = 0, 1 or even) are
only judged by ref.py; each rejects there."""
import math

import numpy as np
import pytest

import rsa_cases as rc
from oracle_rsa import ref

crypto = pytest.importorskip("cryptography")
from cryptography.exceptions import InvalidSignature  # noqa: E402
from cryptography.hazmat.primitives import hashes  # noqa: E402
from cryptography.hazmat.primitives.asymmetric import padding, rsa, utils  # noqa: E402

# the classes where OpenSSL accepts and Go's rule rejects (see the module docstring)
OPENSSL_ACCEPTS_GO_REJECTS = {"badkey_e_above_max", "badkey_e4294967295"}
HASH = {ref.SHA256: hashes.SHA256(), ref.SHA384: hashes.SHA384(), ref.SHA512: hashes.SHA512()}


def _openssl(hash, digest, sig, mod, e):
    """True / False, or None when OpenSSL refuses the key."""
    try:
        pub = rsa.RSAPublicNumbers(int(e), int.from_bytes(mod, "big")).public_key()
    except (ValueError, TypeError):
        return None
    try:
        pub.verify(sig, digest, padding.PKCS1v15(), utils.Prehashed(HASH[hash]))
        return True
    except (InvalidSignature, ValueError):
        return False


@pytest.mark.parametrize("k", rc.SIZES)
@pytest.mark.parametrize("hash", rc.HASHES)
def test_ref_matches_openssl(k, hash):
    c = rc.make_cases(k, hash)
    seen, refused, differ = set(), set(), set()
    for i, cl in enumerate(c["cls"]):
        got = _openssl(hash, c["digest"][i].tobytes(), c["sig"][i].tobytes(), c["mod"][i].tobytes(), c["exp"][i])
        want = bool(c["want"][i])
        seen.add(cl)
        if got is None:
            refused.add(cl)
            assert not want, cl
        elif got != want:
            differ.add(cl)
    assert differ == OPENSSL_ACCEPTS_GO_REJECTS, differ
    assert refused <= {"badkey_e0", "badkey_e1", "badkey_e2147483648", "badkey_even_n"}, refused
    # every valid class is loaded and accepted by both
    assert not {cl for cl in refused if cl.startswith(("valid", "msglen", "crafted"))}


def test_ref_pins_the_key_rule():
    """The key rule of step 1 on its own: e bounds, N parity and N's leading byte."""
    K = rc.key(2048)
    d = bytes(32)
    s = K.sign(256, ref.SHA256, d)
    mod = K.mod_bytes(256)
    assert ref.verify(256, ref.SHA256, d, s, mod, 65537)
    assert not ref.verify(256, ref.SHA256, d, s, mod, 2**31 + 1)  # a larger odd e is never accepted
    assert ref.verify(256, ref.SHA256, d, K.sign(256, ref.SHA256, d, 2**31 - 1), mod, 2**31 - 1)
    assert not ref.verify(256, ref.SHA256, d, s, (K.n ^ 1).to_bytes(256, "big"), 65537)
    assert not ref.verify(256, ref.SHA256, d, mod, mod, 65537)  # S = N


def test_encoding_layout():
    for k in rc.SIZES:
        for h in rc.HASHES:
            em = ref.encode(k, h, bytes(ref.HLEN[h]))
            t = len(ref.DIGEST_INFO[h]) + ref.HLEN[h]
            assert len(em) == k and em[:2] == b"\x00\x01" and em[2:k - t - 1] == b"\xff" * (k - t - 3) and em[k - t - 1] == 0
    assert np.array_equal(np.frombuffer(ref.DIGEST_INFO[ref.SHA256][-2:], np.uint8), [0x04, 0x20])


def test_large_exponent_is_pinned():
    """e > 2^31 - 1 with a signature made under it: OpenSSL accepts, Go's rule (and the engine) rejects."""
    K = rc.key(2048)
    e = 2**31 + 1
    while math.gcd(e, K.lam) != 1:
        e += 2
    d = bytes(range(32))
    s = K.sign(256, ref.SHA256, d, e)
    assert _openssl(ref.SHA256, d, s, K.mod_bytes(256), e) is True
    assert not ref.verify(256, ref.SHA256, d, s, K.mod_bytes(256), e)
