"""oracle_rsa.ref.pss_verify (the restatement of Go's crypto/rsa.VerifyPSS in include/sbv.h) against OpenSSL, through
cryptography's RSAPublicNumbers(e, n).public_key().verify(sig, digest, PSS(MGF1(h), salt), Prehashed(h)) with the salt
AUTO, DIGEST_LENGTH or an explicit length, over every class of tests/rsa_pss_cases.py whose key OpenSSL loads.

They agree everywhere but on two classes, pinned here, where Go's rule as restated is the spec: an exponent above
2^31 - 1 with a signature made under it (badkey_e_above_max, badkey_e4294967295), which OpenSSL accepts and Go's checkPub
refuses.  Classes whose key OpenSSL refuses to load (e = 0, 1 or even) are only judged by ref.py; each rejects there.

Signatures made by OpenSSL's own PSS signer, from the primes of the committed keys, must be accepted by ref: a check of
ref's decoding that does not go through ref.pss_encode."""
import math

import pytest

import rsa_pss_cases as pc
from oracle_rsa import ref

crypto = pytest.importorskip("cryptography")
from cryptography.exceptions import InvalidSignature  # noqa: E402
from cryptography.hazmat.primitives import hashes  # noqa: E402
from cryptography.hazmat.primitives.asymmetric import padding, rsa, utils  # noqa: E402

OPENSSL_ACCEPTS_GO_REJECTS = {"badkey_e_above_max", "badkey_e4294967295"}
HASH = {ref.SHA256: hashes.SHA256, ref.SHA384: hashes.SHA384, ref.SHA512: hashes.SHA512}


def _salt(salt_len):
    return {ref.SALT_AUTO: padding.PSS.AUTO, ref.SALT_EQUALS_HASH: padding.PSS.DIGEST_LENGTH}.get(salt_len, salt_len)


def _openssl(hash, salt_len, digest, sig, mod, e):
    """True / False, or None when OpenSSL refuses the key."""
    try:
        pub = rsa.RSAPublicNumbers(int(e), int.from_bytes(mod, "big")).public_key()
    except (ValueError, TypeError):
        return None
    try:
        pub.verify(sig, digest, padding.PSS(mgf=padding.MGF1(HASH[hash]()), salt_length=_salt(salt_len)), utils.Prehashed(HASH[hash]()))
        return True
    except (InvalidSignature, ValueError):
        return False


@pytest.mark.parametrize("k", pc.SIZES)
@pytest.mark.parametrize("hash", pc.HASHES)
def test_ref_matches_openssl(k, hash):
    c = pc.make_cases(k, hash)
    classes = set(c["cls"])
    for sl in pc.salt_lens(c):
        want = pc.want(c, sl)
        refused, differ = set(), set()
        for i, cl in enumerate(c["cls"]):
            got = _openssl(hash, sl, c["digest"][i].tobytes(), c["sig"][i].tobytes(), c["mod"][i].tobytes(), c["exp"][i])
            if got is None:
                refused.add(cl)
                assert not want[i], cl
            elif got != bool(want[i]):
                differ.add(cl)
        # the pinned pair differs only where the salt mode lets their encoding through
        assert differ <= OPENSSL_ACCEPTS_GO_REJECTS, (sl, differ)
        if sl in (ref.SALT_AUTO, ref.SALT_EQUALS_HASH):
            assert differ == OPENSSL_ACCEPTS_GO_REJECTS, (sl, differ)
            assert 0 < want.sum() < c["n"]
        assert refused <= {"badkey_e0", "badkey_e1", "badkey_e2147483648", "badkey_even_n"}, refused
    for prefix in ("valid", "msglen", "corrupt", "sigval", "crafted", "cross", "badkey"):
        assert any(cl.startswith(prefix) for cl in classes), prefix


@pytest.mark.parametrize("bits", [2048, 2041, 3072, 4089, 4096])
def test_openssl_signatures_are_accepted(bits):
    """OpenSSL signs with PSS from the committed primes (salt of hLen, the longest, and an explicit length); ref accepts
    each under auto and under the salt length it was made with, and rejects it under a length one longer."""
    k = -(-bits // 8)
    K = pc.key(bits)
    n, e = K.n, 65537
    d = pow(e, -1, (K.p - 1) * (K.q - 1))
    priv = rsa.RSAPrivateNumbers(K.p, K.q, d, d % (K.p - 1), d % (K.q - 1), pow(K.q, -1, K.p), rsa.RSAPublicNumbers(e, n)).private_key()
    mod = K.mod_bytes(k)
    em_len = (n.bit_length() - 1 + 7) // 8
    for hash in pc.HASHES:
        hl = ref.HLEN[hash]
        digest = ref.HASHLIB[hash](b"openssl signs this %d" % bits).digest()
        for salt, sl in ((padding.PSS.DIGEST_LENGTH, ref.SALT_EQUALS_HASH), (padding.PSS.MAX_LENGTH, em_len - hl - 2), (17, 17)):
            sig = priv.sign(digest, padding.PSS(mgf=padding.MGF1(HASH[hash]()), salt_length=salt), utils.Prehashed(HASH[hash]()))
            assert len(sig) == k
            assert ref.pss_verify(k, hash, digest, sig, mod, e, ref.SALT_AUTO)
            assert ref.pss_verify(k, hash, digest, sig, mod, e, sl)
            assert not ref.pss_verify(k, hash, digest, sig, mod, e, (hl if sl == ref.SALT_EQUALS_HASH else sl) + 1)
            assert not ref.pss_verify(k, hash, digest, sig, mod, e + 2 if math.gcd(e + 2, K.lam) == 1 else 3, ref.SALT_AUTO)


def test_large_exponent_is_pinned():
    """e > 2^31 - 1 with a PSS signature made under it: OpenSSL accepts, Go's rule (and the engine) rejects."""
    K = pc.key(2048)
    e = 2**31 + 1
    while math.gcd(e, K.lam) != 1:
        e += 2
    d = bytes(range(32))
    s = K.sign_pss(256, ref.SHA256, d, bytes(32), e)
    assert _openssl(ref.SHA256, ref.SALT_AUTO, d, s, K.mod_bytes(256), e) is True
    assert not ref.pss_verify(256, ref.SHA256, d, s, K.mod_bytes(256), e, ref.SALT_AUTO)


def test_salt_len_below_minus_one_is_not_a_verdict():
    with pytest.raises(AssertionError):
        ref.pss_verify(256, ref.SHA256, bytes(32), bytes(256), pc.key(2048).mod_bytes(256), 65537, -2)
