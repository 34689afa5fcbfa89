/*
 * oracle_ed25519/ed25519_oracle.c — CPU ORACLE for sbv_ed25519_verify_batch.  TEST INFRASTRUCTURE ONLY: tests/,
 * __graft_entry__.smoke() and tools/ed25519_bench.py load it; libsbv.so never links or calls it.
 *
 * Verification is OpenSSL 3 pure Ed25519 (EVP_PKEY_ED25519 + EVP_DigestVerify, no context), whose accept set agrees
 * with Go's crypto/ed25519.Verify on the cases the corpus covers (S >= L, keys with y >= p, "-0", small- and
 * mixed-order keys, non-canonical R); oracle_ed25519/ref.py restates that accept set independently and the tests
 * check the two against each other.
 */
#include <openssl/evp.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

static int verify_one(const uint8_t *msg, size_t len, const uint8_t *sig, const uint8_t *pub) {
    EVP_PKEY *k = EVP_PKEY_new_raw_public_key(EVP_PKEY_ED25519, NULL, pub, 32);
    if (!k) return 0;
    EVP_MD_CTX *c = EVP_MD_CTX_new();
    int ok = 0;
    if (c && EVP_DigestVerifyInit(c, NULL, NULL, NULL, k) == 1) ok = EVP_DigestVerify(c, sig, 64, msg, len) == 1;
    EVP_MD_CTX_free(c);
    EVP_PKEY_free(k);
    return ok;
}

typedef struct {
    size_t lo, hi;
    const uint8_t *msgs, *sig, *pub;
    const uint64_t *off;
    uint8_t *ok;
} job_t;

static void *run(void *arg) {
    job_t *j = (job_t *)arg;
    static const uint8_t empty[1] = {0};
    for (size_t i = j->lo; i < j->hi; i++) {
        const size_t len = (size_t)(j->off[i + 1] - j->off[i]);
        j->ok[i] = (uint8_t)verify_one(len ? j->msgs + j->off[i] : empty, len, j->sig + 64 * i, j->pub + 32 * i);
    }
    return NULL;
}

/* ok[i] = Ed25519 verdict of (msgs[off[i], off[i+1]), sig[64i..], pub[32i..]) */
void orc_ed25519_verify_batch(size_t n, const uint8_t *msgs, const uint64_t *off, const uint8_t *sig, const uint8_t *pub, uint8_t *ok,
                              int nthreads) {
    if (nthreads < 1) nthreads = 1;
    if ((size_t)nthreads > n) nthreads = n ? (int)n : 1;
    pthread_t th[256];
    job_t jobs[256];
    if (nthreads > 256) nthreads = 256;
    for (int t = 0; t < nthreads; t++) {
        jobs[t] = (job_t){n * t / nthreads, n * (t + 1) / nthreads, msgs, sig, pub, off, ok};
        if (t) pthread_create(&th[t], NULL, run, &jobs[t]);
    }
    run(&jobs[0]);
    for (int t = 1; t < nthreads; t++) pthread_join(th[t], NULL);
}

/* the verification above, timed (seconds of wall clock) — the CPU arm of tools/ed25519_bench.py */
double orc_ed25519_bench(size_t n, const uint8_t *msgs, const uint64_t *off, const uint8_t *sig, const uint8_t *pub, uint8_t *ok, int nthreads) {
    struct timespec a, b;
    clock_gettime(CLOCK_MONOTONIC, &a);
    orc_ed25519_verify_batch(n, msgs, off, sig, pub, ok, nthreads);
    clock_gettime(CLOCK_MONOTONIC, &b);
    return (double)(b.tv_sec - a.tv_sec) + 1e-9 * (double)(b.tv_nsec - a.tv_nsec);
}

/* public key of a 32-byte seed (RFC 8032 §5.1.5) */
int orc_ed25519_pubkey(const uint8_t *seed, uint8_t *pub) {
    EVP_PKEY *k = EVP_PKEY_new_raw_private_key(EVP_PKEY_ED25519, NULL, seed, 32);
    if (!k) return -1;
    size_t len = 32;
    int rc = EVP_PKEY_get_raw_public_key(k, pub, &len) == 1 && len == 32 ? 0 : -1;
    EVP_PKEY_free(k);
    return rc;
}

/* corpus signing: sig[64i..] = Ed25519 signature of message i under seed key_idx[i] (seeds: 32 bytes each) */
int orc_ed25519_sign_batch(size_t n, const uint8_t *seeds, const uint32_t *key_idx, const uint8_t *msgs, const uint64_t *off, uint8_t *sig) {
    static const uint8_t empty[1] = {0};
    EVP_MD_CTX *c = EVP_MD_CTX_new();
    if (!c) return -1;
    for (size_t i = 0; i < n; i++) {
        EVP_PKEY *k = EVP_PKEY_new_raw_private_key(EVP_PKEY_ED25519, NULL, seeds + 32 * (size_t)key_idx[i], 32);
        size_t sl = 64, len = (size_t)(off[i + 1] - off[i]);
        int good = k && EVP_MD_CTX_reset(c) == 1 && EVP_DigestSignInit(c, NULL, NULL, NULL, k) == 1 &&
                   EVP_DigestSign(c, sig + 64 * i, &sl, len ? msgs + off[i] : empty, len) == 1 && sl == 64;
        EVP_PKEY_free(k);
        if (!good) { EVP_MD_CTX_free(c); return -1; }
    }
    EVP_MD_CTX_free(c);
    return 0;
}
