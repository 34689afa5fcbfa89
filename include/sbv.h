/*
 * sbv.h — C ABI of the H100-native batched signature-verification engine.
 *
 * This is the drop-in boundary behind SmartBFT's application-implemented verifier plug-in:
 *   api.Verifier            /root/reference/pkg/api/dependencies.go:54-71
 *     VerifyConsenterSig    dependencies.go:60-62   (callers: internal/bft/view.go:834-838, 631-635,
 *                                                    internal/bft/viewchanger.go:718)
 *     VerifySignature       dependencies.go:63-64   (callers: viewchanger.go:598, 660, 983, 1022, 1076)
 *     VerifyRequest         dependencies.go:58-59   (callers: internal/bft/controller.go:239, 742-745,
 *                                                    internal/bft/requestpool.go:335-354)
 *     VerifyProposal        dependencies.go:56-57   (caller: view.go:555 — bulk VerifyRequest site)
 *   commit-vote collection  internal/bft/view.go:519-551 (processCommits), 827-849 (verifyVote),
 *                           internal/bft/util.go:114-143 (voteSet), 183-187 (computeQuorum)
 *   digests                 pkg/types/types.go:50-69 (Proposal.Digest), util.go:564-586
 *
 * A cgo (or any FFI) shim binds exactly these symbols; see INTEGRATION.md for the Go side.
 *
 * Conventions
 *  - Return value: 0 on success, < 0 on ENGINE FAULT (CUDA error, out of memory, bad argument).  A
 *    fault is never a verdict: the reference treats `error != nil` from a Verifier as "bad
 *    signature" (view.go:839-842, 386-393), so a host shim must fail-stop on a negative return,
 *    not convert it to a reject.
 *  - Per-item verdicts go to caller-owned arrays: 1 = accept, 0 = reject.
 *  - All pointers are HOST pointers unless the function name ends in _device.  Buffers are only
 *    read during the call and never retained (cgo pointer rules).  Pinned (cudaHostAlloc /
 *    cudaHostRegister) inputs are copied directly; pageable inputs are staged through the
 *    engine's own pinned ring.
 *  - Field elements and scalars are fixed-width big-endian: 32 bytes for P-256, 48 for P-384.
 *  - Accept set = Go crypto/ecdsa (Verify / VerifyASN1): key must be an on-curve affine point with
 *    coordinates < p; r, s in [1, n-1]; e = leftmost min(len, 32|48) digest bytes; R = (e/s)G +
 *    (r/s)Q must not be infinity; accept iff R.x mod n == r.  No low-S rule.
 *  - Thread-safe and re-entrant: the CUDA device is set explicitly per call, so calls may come from any
 *    OS thread (cgo).  Every host-buffer entry point owns a lane (stream, device buffers, pinned staging) for
 *    the duration of the call — six calls proceed concurrently and overlap their copies and kernels; a
 *    seventh waits.  A shard of >= 262,144 items (SBV_CHUNK_ITEMS) is uploaded in chunks on a second stream while
 *    the chunks that have arrived are hashed and verified.  On every return path, faults included, the lane has been drained: no copy into or out of
 *    the caller's buffers is in flight after the call returns, and on a fault the output arrays are untouched
 *    or partially written but never read as verdicts (the caller fail-stops).
 *  - Keys that repeat inside a keys-per-item batch are detected on the device and verified against a per-key
 *    fixed-base table built on the spot (SBV_GROUP_THRESHOLD, default 16 occurrences; 0 disables; at most
 *    SBV_GROUP_MAX_KEYS tables per launch, and when more keys repeat, which of them get one is not specified;
 *    launches below SBV_GROUP_MIN_BATCH items are not grouped): the verdicts
 *    are the same bit for bit, only cheaper.  ECDSA keys are grouped by (qx, qy), Ed25519 keys by their 32 encoded
 *    bytes; each device groups its own shard.
 *  - There is no CPU fallback: without a usable CUDA device sbv_create fails.
 */
#ifndef SBV_H
#define SBV_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sbv_engine sbv_engine;

/* Scheme tags.  The calls that take a curve (or a curve tag per item) accept SBV_P256 and SBV_P384 only and return
 * SBV_ERR_ARG for anything above; the sbv_mixed_* calls take the first three, where SBV_P256 and SBV_P384 are ECDSA over
 * SHA-256; only the sbv_mixed384_* calls also take SBV_P256_SHA384 and SBV_P384_SHA384, ECDSA over SHA-384. */
enum { SBV_P256 = 0, SBV_P384 = 1, SBV_ED25519 = 2, SBV_P256_SHA384 = 3, SBV_P384_SHA384 = 4 };
enum {
    SBV_OK = 0,
    SBV_ERR_ARG = -1,   /* bad argument */
    SBV_ERR_CUDA = -2,  /* CUDA runtime / driver error */
    SBV_ERR_NCCL = -3,  /* NCCL error (multi-device engines only) */
    SBV_ERR_NOMEM = -4
};

/* n_devices in {1,2,4,8}; device_ordinals == NULL means 0..n_devices-1.  With n_devices > 1 the
 * engine shards every batch across the devices and gathers the packed verdict bitmask with NCCL. */
int sbv_create(const int *device_ordinals, int n_devices, sbv_engine **out);
void sbv_destroy(sbv_engine *e);
/* Human-readable description of the last fault on this engine (a thread-local copy: valid until the calling
 * thread's next sbv_last_error). */
const char *sbv_last_error(const sbv_engine *e);
int sbv_device_count(const sbv_engine *e);

/* ECDSA verify, digests supplied.  SoA arrays of n fixed-width big-endian values. */
int sbv_verify_batch(sbv_engine *e, uint8_t curve, size_t n, const uint8_t *r, const uint8_t *s,
                     const uint8_t *qx, const uint8_t *qy, const uint8_t *digest, uint8_t digest_len,
                     uint8_t *ok);

/* Same, with every input already resident on device `device_index` (0-based position in the
 * engine's device list) and the verdicts left on the device.  Enqueued on `cuda_stream`
 * (a cudaStream_t; NULL = the legacy default stream) and NOT synchronised. */
int sbv_verify_batch_device(sbv_engine *e, int device_index, uint8_t curve, size_t n, const uint8_t *d_r,
                            const uint8_t *d_s, const uint8_t *d_qx, const uint8_t *d_qy,
                            const uint8_t *d_digest, uint8_t digest_len, uint8_t *d_ok, void *cuda_stream);

/* DER front end: sigs = concatenated ASN.1 SEQUENCE{INTEGER r, INTEGER s}, sig_off[n+1].  Parsed
 * with crypto/ecdsa.VerifyASN1 strictness (minimal lengths, minimal non-negative integers, no
 * trailing bytes); malformed items reject.  qxy = n * (X||Y). */
int sbv_verify_batch_der(sbv_engine *e, uint8_t curve, size_t n, const uint8_t *sigs, const uint32_t *sig_off,
                         const uint8_t *qxy, const uint8_t *digest, uint8_t digest_len, uint8_t *ok);

/* SHA-256 over a ragged batch: msgs concatenated, msg_off[n+1] byte offsets.  digest_out = 32n. */
int sbv_sha256_batch(sbv_engine *e, size_t n, const uint8_t *msgs, const uint64_t *msg_off, uint8_t *digest_out);

/* Fused SHA-256 -> ECDSA verify (VerifyRequest / VerifySignature shape): the message digest never
 * leaves the device.  digest_out may be NULL. */
int sbv_hash_verify_batch(sbv_engine *e, uint8_t curve, size_t n, const uint8_t *msgs, const uint64_t *msg_off,
                          const uint8_t *r, const uint8_t *s, const uint8_t *qx, const uint8_t *qy,
                          uint8_t *digest_out, uint8_t *ok);

/* ---- SHA-384 for ECDSA: the digest Go's crypto/x509 (ECDSAWithSHA384), JOSE ES384 and TLS ecdsa_secp384r1_sha384 pair
 * with P-384.  The three calls below are the SHA-256 forms with SHA-384 in place of SHA-256; msgs / msg_off as in
 * sbv_sha256_batch (msgs may be NULL when every message is empty).  The same argument checks run before anything is
 * written: SBV_ERR_ARG for a curve other than SBV_P256 / SBV_P384, null buffers, n >= 2^31 and decreasing offsets.
 * Multi-device engines shard them as the SHA-256 forms.  Mixed batches with SHA-384 items go through the sbv_mixed384_*
 * calls.  Out of scope, SHA-256 or digests only: sbv_verify_quorum, the DER front end and the _ranked and _device forms. */
/* SHA-384 over a ragged batch (msgs / msg_off as in sbv_sha256_batch); digest_out = 48n bytes. */
int sbv_sha384_batch(sbv_engine *e, size_t n, const uint8_t *msgs, const uint64_t *msg_off, uint8_t *digest_out);
/* sbv_hash_verify_batch with SHA-384: e = leftmost min(48, field bytes) of SHA-384(M) (the whole digest for P-384,
 * its leftmost 32 bytes for P-256, as crypto/ecdsa truncates).  The accept set is exactly that of sbv_verify_batch
 * with digest = SHA-384(M) and digest_len = 48, keys that repeat grouped as there.  digest_out (48n) may be NULL. */
int sbv_hash384_verify_batch(sbv_engine *e, uint8_t curve, size_t n, const uint8_t *msgs, const uint64_t *msg_off,
                             const uint8_t *r, const uint8_t *s, const uint8_t *qx, const uint8_t *qy,
                             uint8_t *digest_out, uint8_t *ok);
/* sbv_hash_verify_registered with SHA-384 (same e as above): the accept set is exactly that of sbv_verify_registered with
 * digest = SHA-384(M) and digest_len = 48. */
int sbv_hash384_verify_registered(sbv_engine *e, uint8_t curve, size_t n, const uint8_t *msgs, const uint64_t *msg_off,
                                  const uint32_t *key_slot, const uint8_t *r, const uint8_t *s, uint8_t *ok);

/* ---- RSA PKCS #1 v1.5 (RSASSA-PKCS1-v1_5, RFC 8017 §8.2.2), for a Verifier whose identities hold crypto/rsa keys
 * (crypto/x509 SHA256WithRSA, SHA384WithRSA, SHA512WithRSA).  Hash tags: */
enum { SBV_HASH_SHA256 = 0, SBV_HASH_SHA384 = 1, SBV_HASH_SHA512 = 2 };
/* Accept set = Go crypto/rsa.VerifyPKCS1v15(pub, hash, H, S).  k = mod_bytes (256, 384 or 512), modulus N (k bytes,
 * big-endian), public exponent e (uint32), digest H (hLen = 32, 48 or 64 bytes by the hash tag, taken as given: no
 * truncation), signature S (k bytes, big-endian):
 *  1. Key: reject unless N is odd, N's leading byte is nonzero (so Go's pub.Size() equals k and its k != len(sig)
 *     check passes) and 2 <= e <= 2^31 - 1 (the bounds of Go's checkPub).  The rule on N's parity is the engine's:
 *     Go's behaviour on an even modulus is not pinned by any test here, and no real key has one.
 *  2. Range: reject if S >= N (Go's bigmod SetBytes fails there), so S + N, the twin of a valid S, rejects.
 *  3. Recover: EM = S^e mod N as k bytes, big-endian.
 *  4. Compare: accept iff EM = 00 || 01 || FF..FF || 00 || DigestInfo(hash) || H byte for byte, the FF run k - tLen - 3
 *     bytes long, tLen = |DigestInfo| + hLen, with the DigestInfo prefixes of RFC 8017 §9.2 note 1 WITH the NULL
 *     parameters (the form without them rejects, as in Go).
 * RSA-PSS is not offered.  The checks: SBV_ERR_ARG for a mod_bytes other than 256 / 384 / 512, a hash tag above
 * SBV_HASH_SHA512, a null buffer (msgs may be NULL when every message is empty), n >= 2^31 and decreasing offsets, all
 * before anything is written or launched.  Multi-device engines shard by item as sbv_hash_verify_batch does.  Each
 * device's shard is uploaded whole (no chunked upload).  Out of scope: registered RSA keys, RSA items in the mixed and
 * commit-vote calls, and _device / _ranked forms. */
/* SHA-512 over a ragged batch (msgs / msg_off as in sbv_sha256_batch); digest_out = 64n bytes. */
int sbv_sha512_batch(sbv_engine *e, size_t n, const uint8_t *msgs, const uint64_t *msg_off, uint8_t *digest_out);
/* digests supplied: digest = n x hLen bytes; sig, modulus = n x mod_bytes bytes; pub_exp = n x uint32 */
int sbv_rsa_verify_batch(sbv_engine *e, uint32_t mod_bytes, uint8_t hash, size_t n, const uint8_t *digest,
                         const uint8_t *sig, const uint8_t *modulus, const uint32_t *pub_exp, uint8_t *ok);
/* fused SHA-2 -> RSA: H = hash(M) never leaves the device; digest_out (n x hLen) may be NULL */
int sbv_rsa_hash_verify_batch(sbv_engine *e, uint32_t mod_bytes, uint8_t hash, size_t n, const uint8_t *msgs,
                              const uint64_t *msg_off, const uint8_t *sig, const uint8_t *modulus,
                              const uint32_t *pub_exp, uint8_t *digest_out, uint8_t *ok);

/* Mixed-curve batch: curve_tag[i] in {SBV_P256, SBV_P384}; every field is stored in a 48-byte
 * slot (P-256 values right-aligned, i.e. 16 leading zero bytes); digest is 32 bytes per item. */
int sbv_verify_mixed(sbv_engine *e, size_t n, const uint8_t *curve_tag, const uint8_t *r48, const uint8_t *s48,
                     const uint8_t *qx48, const uint8_t *qy48, const uint8_t *digest32, uint8_t *ok);

/* Ed25519 verify over raw messages, for a Verifier whose keys are crypto/ed25519 keys (VerifyConsenterSig /
 * VerifySignature / VerifyRequest, dependencies.go:58-64).  msgs concatenated with msg_off[n+1] byte offsets (msgs may
 * be NULL when every message is empty); sig = 64n bytes (R || S), pub = 32n bytes, both as RFC 8032 encodes them.
 * Accept set = Go crypto/ed25519.Verify (pure Ed25519, no context): S < L; A decodes as edwards25519 Point.SetBytes does
 * (y >= p reduced, "-0" accepted, no subgroup check); k = SHA-512(R || A || M) mod L over the caller's bytes; accept iff
 * the canonical encoding of [S]B - [k]A equals R byte for byte (cofactorless; each signature on its own).  Messages are
 * hashed on the device.  The first call on an engine builds a 384 KiB table of B on every device.  Keys whose 32 bytes
 * repeat are grouped (see the top of this file): such a key gets a 48 KiB comb table built in the launch, with the same
 * settings and the same verdicts; two encodings of one point (y >= p, "-0") are two keys. */
int sbv_ed25519_verify_batch(sbv_engine *e, size_t n, const uint8_t *msgs, const uint64_t *msg_off, const uint8_t *sig,
                             const uint8_t *pub, uint8_t *ok);

/* Ed25519 key registry.  Consenter and client keys are configuration: they change only with a reconfiguration
 * (api.Verifier, dependencies.go:58-66).  sbv_ed25519_set_keys replaces the registry: slot i = the 32-byte encoding
 * pub[32i..32i+32); n = 0 empties it.  On every device it builds a fixed-base table per decodable key (8-bit signed
 * windows: 32 x 128 affine points = 384 KiB per key per device).  It waits for the launches that may still read the old
 * tables.  Independent of sbv_set_keys: neither call touches the other's registry.  A fault leaves the registry empty. */
int sbv_ed25519_set_keys(sbv_engine *e, size_t n, const uint8_t *pub);
/* sbv_ed25519_verify_batch with the key of item i taken from registry slot key_slot[i].  Same accept set: k hashes the
 * 32 bytes registered in the slot, not a re-encoding; a slot >= n, a registered key that does not decode and an empty
 * registry reject.  [k]A is fixed-base (32 additions, no doublings and no key decoding).  Every shard of one call, on
 * every device, reads the same registry: a concurrent sbv_ed25519_set_keys waits until the calls already enqueueing have
 * enqueued all their shards (and then for their kernels), and calls that start after it see the new registry. */
int sbv_ed25519_verify_registered(sbv_engine *e, size_t n, const uint8_t *msgs, const uint64_t *msg_off,
                                  const uint32_t *key_slot, const uint8_t *sig, uint8_t *ok);

/* Distinct-signer quorum count per consensus instance (processCommits, view.go:519-551).
 * Votes are given in arrival order.  A vote is registered iff signer == sender and sender !=
 * self_id[instance] and the sender has no earlier registered vote in the instance
 * (view.go:161-171, util.go:130-143); a registered vote is valid iff digest_match && ok
 * (view.go:829-842).  valid_count[i] = number of valid votes; reached[i] = valid_count[i] >=
 * threshold (the caller passes Quorum-1, view.go:531).  self_id may be NULL (no self filter). */
int sbv_quorum(sbv_engine *e, size_t n_votes, const uint32_t *instance, const uint16_t *sender,
               const uint16_t *signer, const uint8_t *digest_match, const uint8_t *ok, size_t n_instances,
               const uint16_t *self_id, uint32_t threshold, uint32_t *valid_count, uint8_t *reached);

/* Prepare collection in batch form (View.processPrepares, view.go:441-517): prepares carry no signature; the
 * first prepare of a sender burns its slot (util.go:130-143) and counts iff digest_match (view.go:452-459);
 * reached[i] = match_count[i] >= threshold (the caller passes Quorum-1, view.go:446). */
int sbv_prepare_quorum(sbv_engine *e, size_t n_votes, const uint32_t *instance, const uint16_t *sender,
                       const uint8_t *digest_match, size_t n_instances, const uint16_t *self_id, uint32_t threshold,
                       uint32_t *match_count, uint8_t *reached);

/* Commit-vote verification AND quorum collection in one call (verifyVote + processCommits, view.go:519-551,
 * 827-849; BASELINE configs[3]).  The n_votes signatures (SoA as in sbv_verify_batch) are verified, the verdicts stay
 * on the device and feed the distinct-signer count of sbv_quorum.  Votes must be grouped by instance with
 * non-decreasing instance ids, in arrival order inside an instance.  A multi-device engine shards BY INSTANCE so that
 * every count is local; the packed verdict mask and the packed `reached` mask travel in one NCCL all-gather.
 * Outputs: ok[n_votes], valid_count[n_instances], reached[n_instances]. */
int sbv_verify_quorum(sbv_engine *e, uint8_t curve, size_t n_votes, const uint8_t *r, const uint8_t *s, const uint8_t *qx,
                      const uint8_t *qy, const uint8_t *digest, uint8_t digest_len, const uint32_t *instance,
                      const uint16_t *sender, const uint16_t *signer, const uint8_t *digest_match, size_t n_instances,
                      const uint16_t *self_id, uint32_t threshold, uint8_t *ok, uint32_t *valid_count, uint8_t *reached);

/* sbv_verify_quorum for consenters with registered Ed25519 keys (verifyVote + processCommits, view.go:519-551, 827-849;
 * voteSet, util.go:130-143).  ok[i] = the verdict of sbv_ed25519_verify_registered for vote i: key from registry slot
 * key_slot[i], message msgs[msg_off[i]..msg_off[i+1]) hashed on the device (msgs may be NULL when every message is empty),
 * sig = 64 bytes per vote (R || S); a slot >= n, a registered key that does not decode and an empty registry reject.
 * valid_count / reached = sbv_quorum over those verdicts, with the same vote rules, self_id (NULL = no self filter) and
 * threshold (the caller passes Quorum-1).  The verdicts stay on the device.  Votes must be grouped by instance with
 * non-decreasing instance ids, in arrival order inside an instance.  A multi-device engine shards BY INSTANCE, as
 * sbv_verify_quorum does, and every shard of one call reads the same registry (as in sbv_ed25519_verify_registered).
 * Shards are uploaded whole: unlike the ECDSA calls, large Ed25519 shards are not uploaded in chunks.
 * Outputs: ok[n_votes], valid_count[n_instances], reached[n_instances]; n_instances == 0 does nothing. */
int sbv_ed25519_verify_quorum(sbv_engine *e, size_t n_votes, const uint8_t *msgs, const uint64_t *msg_off,
                              const uint32_t *key_slot, const uint8_t *sig, const uint32_t *instance,
                              const uint16_t *sender, const uint16_t *signer, const uint8_t *digest_match,
                              size_t n_instances, const uint16_t *self_id, uint32_t threshold, uint8_t *ok,
                              uint32_t *valid_count, uint8_t *reached);

/* Registered-key batch whose items may be of any scheme (a consenter or client set that mixes ECDSA and Ed25519 keys,
 * e.g. while it moves from one to the other).  scheme[i] in {SBV_P256, SBV_P384, SBV_ED25519}; msgs concatenated with
 * msg_off[n+1] byte offsets (msgs may be NULL when every message is empty); sig96 = one 96-byte row per item:
 *   P-256    r || s, 32 bytes each, big-endian, in bytes [0, 64)
 *   P-384    r || s, 48 bytes each, big-endian, filling the row
 *   Ed25519  R || S as RFC 8032 encodes them, in bytes [0, 64)
 * Bytes past the signature are ignored.  key_slot[i] indexes the registry of the item's own scheme: sbv_set_keys for
 * ECDSA, sbv_ed25519_set_keys for Ed25519 (slot 3 of an ECDSA item and slot 3 of an Ed25519 item are different keys).
 * ok[i] is byte for byte what the single-scheme call returns for item i: sbv_hash_verify_registered(scheme[i], ...)
 * for ECDSA items, sbv_ed25519_verify_registered for Ed25519 items.  The shard of each device is uploaded once, whole,
 * and split into the three families on the device; the ECDSA families run on the call's stream while the Ed25519 one
 * runs beside them on its second stream, and the verdicts are put back in item order on the device.  A tag > 2 returns
 * SBV_ERR_ARG with its index in sbv_last_error, before anything is written or launched.  Every shard of one call reads
 * the same Ed25519 registry, as in sbv_ed25519_verify_registered. */
int sbv_mixed_verify_registered(sbv_engine *e, size_t n, const uint8_t *scheme, const uint8_t *msgs, const uint64_t *msg_off,
                                const uint32_t *key_slot, const uint8_t *sig96, uint8_t *ok);
/* sbv_mixed_verify_registered with the key of each item carried in the call (client requests of a population that mixes
 * ECDSA and Ed25519 keys and comes and goes, so that no registry is rebuilt for it).  scheme, msgs, msg_off and sig96 as
 * in sbv_mixed_verify_registered; key96 = one 96-byte row per item, packed as sig96 is:
 *   P-256    X || Y, 32 bytes each, big-endian, in bytes [0, 64)
 *   P-384    X || Y, 48 bytes each, big-endian, filling the row
 *   Ed25519  the 32-byte RFC 8032 encoding, in bytes [0, 32)
 * Bytes past the key are ignored.  ok[i] is byte for byte what the single-scheme keys-per-item call returns for item i:
 * sbv_hash_verify_batch(scheme[i], ...) for ECDSA items (SHA-256 of the message; e = its leftmost 32 bytes for P-384
 * too), sbv_ed25519_verify_batch for Ed25519 items.  The shard of each device is uploaded once, whole, and split into the
 * three families on the device, keys included; the ECDSA families run on the call's stream while the Ed25519 one runs
 * beside them on its second stream, and the verdicts are put back in item order on the device.  Keys that repeat are
 * grouped per family and per device shard, with the SBV_GROUP_* settings of the single-scheme calls; an ECDSA key and an
 * Ed25519 key are never one group.  A tag > 2 returns SBV_ERR_ARG with its index in sbv_last_error, before anything is
 * written or launched.  No registry is read. */
int sbv_mixed_verify_batch(sbv_engine *e, size_t n, const uint8_t *scheme, const uint8_t *msgs, const uint64_t *msg_off,
                           const uint8_t *sig96, const uint8_t *key96, uint8_t *ok);
/* Commit votes of a mixed consenter set verified and counted in one call (verifyVote + processCommits,
 * view.go:519-551, 827-849): ok = the verdicts of sbv_mixed_verify_registered, valid_count / reached = sbv_quorum over
 * them, with the same vote rules, self_id (NULL = no self filter) and threshold.  The verdicts stay on the device.  Votes
 * must be grouped by instance with non-decreasing instance ids; a multi-device engine shards BY INSTANCE, as
 * sbv_verify_quorum does.  Outputs: ok[n_votes], valid_count[n_instances], reached[n_instances]; n_instances == 0 does
 * nothing. */
int sbv_mixed_verify_quorum(sbv_engine *e, size_t n_votes, const uint8_t *scheme, const uint8_t *msgs, const uint64_t *msg_off,
                            const uint32_t *key_slot, const uint8_t *sig96, const uint32_t *instance, const uint16_t *sender,
                            const uint16_t *signer, const uint8_t *digest_match, size_t n_instances, const uint16_t *self_id,
                            uint32_t threshold, uint8_t *ok, uint32_t *valid_count, uint8_t *reached);

/* The three mixed calls with ECDSA over SHA-384 among the items: each has the arguments of its sbv_mixed_* counterpart and
 * accepts scheme tags 0 to 4.  Tags 0 to 2 mean what they mean there; a batch of those tags only returns byte for byte
 * what the counterpart returns.  SBV_P256_SHA384 and SBV_P384_SHA384 items are packed as P-256 and P-384 items (sig96,
 * key96 and registry slots of sbv_set_keys alike) and are verified with e = the leftmost min(48, field bytes) of
 * SHA-384(M): ok[i] is byte for byte what sbv_hash384_verify_registered (or, keys per item, sbv_hash384_verify_batch)
 * returns for the item on its curve.  A tag > 4 returns SBV_ERR_ARG with its index in sbv_last_error, before anything is
 * written or launched; the other argument checks are those of the counterpart.  The split into the three curve families
 * is that of the counterpart, so keys that repeat are grouped per curve whichever hash their items use; each family is
 * hashed by one launch that picks SHA-256 or SHA-384 per item. */
int sbv_mixed384_verify_registered(sbv_engine *e, size_t n, const uint8_t *scheme, const uint8_t *msgs, const uint64_t *msg_off,
                                   const uint32_t *key_slot, const uint8_t *sig96, uint8_t *ok);
int sbv_mixed384_verify_batch(sbv_engine *e, size_t n, const uint8_t *scheme, const uint8_t *msgs, const uint64_t *msg_off,
                              const uint8_t *sig96, const uint8_t *key96, uint8_t *ok);
/* ok = the verdicts of sbv_mixed384_verify_registered; valid_count / reached as in sbv_mixed_verify_quorum (the same vote
 * rules, sharded by instance on a multi-device engine). */
int sbv_mixed384_verify_quorum(sbv_engine *e, size_t n_votes, const uint8_t *scheme, const uint8_t *msgs, const uint64_t *msg_off,
                               const uint32_t *key_slot, const uint8_t *sig96, const uint32_t *instance, const uint16_t *sender,
                               const uint16_t *signer, const uint8_t *digest_match, size_t n_instances, const uint16_t *self_id,
                               uint32_t threshold, uint8_t *ok, uint32_t *valid_count, uint8_t *reached);

/* computeQuorum(n) -> (q, f), internal/bft/util.go:183-187. */
void sbv_compute_quorum(uint64_t n, uint32_t *q, uint32_t *f);

/* Consenter key registry.  Keys are configuration in the reference: they change only with a
 * reconfiguration, i.e. a new VerificationSequence (dependencies.go:65-66).  sbv_set_keys replaces
 * the registry and precomputes, on every device, a fixed-base comb table per key
 * (8-bit signed windows: 33 x 128 affine points = 264 KiB per P-256 key, a few milliseconds for a thousand keys);
 * slot i of the registry is key i of this call.
 * xy = n * 96 bytes: X and Y in 48-byte slots (P-256 values right-aligned). */
int sbv_set_keys(sbv_engine *e, uint64_t verification_seq, size_t n, const uint64_t *ids, const uint8_t *curve,
                 const uint8_t *xy);

/* ECDSA verify against REGISTERED keys: key_slot[i] indexes the registry of sbv_set_keys.  Same accept
 * set as sbv_verify_batch; an unknown slot, a slot of another curve or an invalid registered key
 * rejects.  Both scalar multiplications are fixed-base (no doublings), which is ~5x less work than
 * the keys-per-item entry point. */
int sbv_verify_registered(sbv_engine *e, uint8_t curve, size_t n, const uint32_t *key_slot, const uint8_t *r,
                          const uint8_t *s, const uint8_t *digest, uint8_t digest_len, uint8_t *ok);
/* Fused SHA-256 -> registered-key verify (VerifyConsenterSig / VerifySignature / VerifyRequest with
 * registered consenter or client keys): messages hashed on the device. */
int sbv_hash_verify_registered(sbv_engine *e, uint8_t curve, size_t n, const uint8_t *msgs, const uint64_t *msg_off,
                               const uint32_t *key_slot, const uint8_t *r, const uint8_t *s, uint8_t *ok);
int sbv_verify_registered_device(sbv_engine *e, int device_index, uint8_t curve, size_t n, const uint32_t *d_key_slot,
                                 const uint8_t *d_r, const uint8_t *d_s, const uint8_t *d_digest, uint8_t digest_len,
                                 uint8_t *d_ok, void *cuda_stream);

/* ---- tables of repeated keys kept across launches (opt-in) ----
 * Keys that a keys-per-item launch groups (SBV_GROUP_THRESHOLD items or more of one key in a device's shard, within
 * SBV_GROUP_MIN_BATCH and SBV_GROUP_MAX_KEYS) get a fixed-base table built in the launch.  Client keys of a SmartBFT
 * deployment come back in every batch but are not configuration, so they cannot be registered; with a cache reserved, the
 * launch takes the tables of such keys from the cache instead of rebuilding them.  This covers sbv_verify_batch and its
 * _device, _der and _ranked forms, sbv_hash_verify_batch, sbv_hash384_verify_batch, sbv_verify_mixed, sbv_verify_quorum,
 * sbv_ed25519_verify_batch and sbv_mixed_verify_batch.
 *  - Only where a table comes from changes.  The cache serves only keys the launch groups anyway; keys below the threshold
 *    take the generic kernel, cached or not.  A hit puts the cached table into the launch's table slot; a miss is built as
 *    without a cache and then inserted if there is room.  A table is a pure function of the key bytes, so routing, the
 *    verification kernels and every verdict are bit for bit those of an engine without a cache.
 *  - Keyed by the exact bytes: qx || qy (64 bytes) for P-256, 96 bytes for P-384, the 32-byte encoding for Ed25519 (so
 *    y >= p and "-0" encodings are keys of their own, as in the grouping).  Entries are compared byte for byte, never by
 *    hash alone.
 *  - Only keys whose build flags them valid are inserted: an off-curve ECDSA key or an undecodable Ed25519 key is rebuilt,
 *    and rejected, in every launch.
 *  - Fill once, no eviction: a full cache stops inserting (sbv_key_cache_reserve_evicting below reserves a cache that
 *    replaces its least recently used entries instead).  Reserving again empties it (for example on a reconfiguration).
 *    It is independent of both registries and of verification_seq.
 *  - One cache per device: each device caches the keys of its own shards.
 *  - Two launches that miss the same key at once both build it; one of them inserts it.
 *
 * Reserve, on every device, room for the tables of up to p256 / p384 / ed25519 keys.  The sizes per key are the
 * per-launch table sizes: 32 KiB for P-256, 118 KiB for P-384, 47.8 KiB for Ed25519, plus a map of a power of two
 * >= 2 x capacity slots (72 to 104 bytes each).  Replaces and empties any earlier cache.  (0, 0, 0) frees it, and the
 * engine behaves as if none had been reserved: the same kernels, launch count and memory.  Excludes concurrent launches
 * as sbv_ed25519_set_keys does (it waits for the calls already enqueueing and drains every device).  SBV_ERR_NOMEM
 * leaves no cache on any device. */
int sbv_key_cache_reserve(sbv_engine *e, size_t p256, size_t p384, size_t ed25519);
/* Per scheme tag (SBV_P256 / SBV_P384 / SBV_ED25519; anything else is SBV_ERR_ARG), summed over devices, for the calls
 * that have returned (a _device call: once its stream has been synchronised): out[0] capacity, out[1] resident tables,
 * out[2] grouped keys served from the cache (hits), out[3] grouped valid keys built in the launch while a cache was
 * reserved (misses; invalid keys count as neither).  All zero without a cache. */
int sbv_key_cache_stats(sbv_engine *e, uint8_t scheme, uint64_t out[4]);
/* The evicting mode: reserves, on every device, caches that replace entries when full, so that the keys in use now stay
 * resident when the client population outgrows the cache or changes over time.  Which keys are served is as above: only
 * grouped keys, compared byte for byte, only valid keys inserted, one cache per device, and a table is a pure function of
 * the key bytes, so verdicts, routing and launch count are bit for bit those of an engine without a cache (the same two
 * extra launches per grouped launch as the fill-once mode).
 *  - Set-associative, 16 ways per set.  A requested capacity is rounded up to a multiple of 16 (out[0] of both stats calls
 *    reports the rounded capacity); the key bytes' hash picks the set.
 *  - Replacement: least recently used within the set, where "used" means looked up as a hit or inserted, ordered by a
 *    launch sequence number (one per grouped launch, per device and scheme).  A missed valid key takes an empty way, else
 *    the set's least recently used way that no launch is copying out of and that no launch at or after its own has used:
 *    a launch never evicts a table it has used itself.  With none, the insert is given up and counted.
 *  - Two launches that miss the same key at once may both insert it; both entries hold the same table.
 * The sizes per key are those of sbv_key_cache_reserve, plus 16 bytes of map per way beside the key bytes.  Works like
 * sbv_key_cache_reserve otherwise: per device and per scheme it replaces and empties any earlier cache of either mode,
 * (0, 0, 0) frees it, it excludes concurrent launches and drains every device, and SBV_ERR_NOMEM leaves no cache on any
 * device. */
int sbv_key_cache_reserve_evicting(sbv_engine *e, size_t p256, size_t p384, size_t ed25519);
/* out[0..3] as sbv_key_cache_stats; out[4] evictions (valid tables replaced by another key's table); out[5] inserts given
 * up (a missed valid key that found no way it could take: every way of its set busy with another key, being read, or
 * used by its own or a later launch).  The fill-once mode counts neither: out[4] is 0 as it never evicts, and out[5] is 0
 * because its kernels are left as they were (a full fill-once cache gives up every insert: out[3] - out[1] of them, less
 * the keys two launches inserted at once).  SBV_ERR_ARG for a scheme tag above SBV_ED25519 or a null out. */
int sbv_key_cache_stats_ex(sbv_engine *e, uint8_t scheme, uint64_t out[6]);

/* ---- one process per GPU (a Go host may run one node process per device; bench.py does under torchrun) ----
 * The engine of every process is one RANK; the only exchange is the all-gather of packed verdict / quorum bitmasks
 * over NCCL (NVLink / NVSwitch).  Rank 0 calls sbv_comm_unique_id and ships the 128 bytes to the others (any side
 * channel); every rank then calls sbv_comm_init_rank, which adds one CHANNEL (communicator) and returns its index.
 * The collectives of a channel must be issued in the same order on every rank, so concurrent caller threads take
 * one channel each (create as many as there are threads, in the same order on every rank). */
int sbv_comm_unique_id(uint8_t *id128);
int sbv_comm_init_rank(sbv_engine *e, const uint8_t *id128, int nranks, int rank);
int sbv_comm_ranks(const sbv_engine *e);
/* Device form: packs n verdict bytes into a bitmask and all-gathers the masks of all ranks,
 * d_mask_all[rank * ceil(n/32) + w]; enqueued on cuda_stream, not synchronised.  Every rank passes the same n. */
int sbv_gather_verdicts_device(sbv_engine *e, int channel, const uint8_t *d_ok, size_t n, uint32_t *d_mask_all, void *cuda_stream);
/* All-gather of `words` 32-bit words per rank, in place: the sender's words sit at d_all + rank * words. */
int sbv_gather_words_device(sbv_engine *e, int channel, uint32_t *d_all, size_t words, void *cuda_stream);
/* Host form: sbv_verify_batch for this rank's n items + the gather: ok[n] = this rank's verdict bytes,
 * mask_all[nranks * ceil(n/32)] = the packed verdicts of every rank. */
int sbv_verify_batch_ranked(sbv_engine *e, int channel, uint8_t curve, size_t n, const uint8_t *r, const uint8_t *s,
                            const uint8_t *qx, const uint8_t *qy, const uint8_t *digest, uint8_t digest_len, uint8_t *ok,
                            uint32_t *mask_all);

/* Pinned (page-locked, portable) host memory for batches the host marshals itself: buffers from here are DMA'd
 * directly by every entry point (no staging copy).  A cgo shim keeps C memory anyway (cgo pointer rules), so its
 * batch buffers should come from here.  NULL on failure. */
void *sbv_host_alloc(size_t bytes);
void sbv_host_free(void *p);

/* Introspection for benchmarks: number of kernel launches issued by this engine so far. */
uint64_t sbv_kernel_launches(const sbv_engine *e);
/* Optional CUDA-event timing inside every verify launch (off by default).  sbv_profile_read sums, over all
 * devices, prep_ms = launch start .. end of the scalar preparation (includes the key grouping) and verify_ms = the
 * verification kernels alone (the two halves of the fixed-base verification when keys were grouped, the generic kernel
 * otherwise), and
 * resets; the caller synchronises the streams it used first. */
int sbv_profile_enable(sbv_engine *e, int on);
int sbv_profile_read(sbv_engine *e, double *prep_ms, double *verify_ms, uint64_t *n_launch_pairs);
/* Peak-rate probe: dependent-free IMAD.WIDE.U32 loop on device 0; returns MAC32/s (0 on fault). */
double sbv_probe_mad_rate(sbv_engine *e);

#ifdef __cplusplus
}
#endif
#endif /* SBV_H */
