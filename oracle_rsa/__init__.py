"""oracle_rsa — CPU oracle for sbv_rsa_verify_batch / sbv_rsa_hash_verify_batch.  TEST INFRASTRUCTURE ONLY (never imported
by consensus_b200).  `ref` is the pure-Python restatement of Go's crypto/rsa.VerifyPKCS1v15 accept set, plus a seeded key
generator and a CRT signer."""
from . import ref  # noqa: F401
