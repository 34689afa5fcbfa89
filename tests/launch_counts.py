"""Kernel launches (sbv_kernel_launches) of one keys-per-item call on a one-device engine, as the pipelines enqueue them:
the first half (k_kg_insert, k_kg_assign, the table build, and k_kc_lookup + k_kc_insert with a cache reserved for the
scheme), then per chunk the hash, k_prep and the verification kernels.  A device's first Ed25519 call adds k_ed_btab_init,
which these counts leave out."""
P256, P384, ED = 0, 1, 2
BUILD = {P256: 5, P384: 4, ED: 4}  # k_kt_bases4 k_comb_affine k_comb_fill k_kt_inv k_kt_final / k_kt_bases4 k_kt_fill k_kt_inv k_kt_final / k_edc_*
DEFAULTS = {"SBV_GROUP_THRESHOLD": 16, "SBV_GROUP_MIN_BATCH": 0, "SBV_GROUP_MAX_KEYS": 8192, "SBV_CHUNK_ITEMS": 262144}


def _sort(n):  # the block-count sort ahead of a hash: k_sha_hist, k_sha_scan, k_sha_scatter
    return 3 if n >= 2048 else 0


def _first_half(scheme, n, env, cached):
    T = env["SBV_GROUP_THRESHOLD"]
    if T <= 0 or n < T or n < env["SBV_GROUP_MIN_BATCH"] or env["SBV_GROUP_MAX_KEYS"] <= 0:
        return None
    return 2 + BUILD[scheme] + (2 if scheme in cached else 0)


def ecdsa(curve, n, hashing=True, env=None, cached=(), chunked=True):
    """sbv_hash_verify_batch (hashing) or sbv_verify_batch; chunked=False: one chunk whatever SBV_CHUNK_ITEMS, as inside
    sbv_mixed_verify_batch."""
    env = {**DEFAULTS, **(env or {})}
    if n == 0:
        return 0
    first = _first_half(curve, n, env, cached)
    ci, chunks = env["SBV_CHUNK_ITEMS"], 1
    if chunked and ci > 0 and n >= ci:
        chunks = min(max(n // ci, 2), 32)
    per = (-(-n // chunks) + 255) // 256 * 256
    out = first or 0
    for lo in range(0, n, per):  # chunks past the last item launch nothing
        cn = min(per, n - lo)
        out += (_sort(cn) + 1 if hashing else 0) + 1 + (4 if first else 1)  # hash, k_prep, routing + generic + k_gpart + fixed-base / generic
    return out


def ed25519(n, env=None, cached=()):
    """sbv_ed25519_verify_batch: k_kg_route after the first half, the sort, k_ed_sha512, k_ed_verify, k_ed_verify_comb."""
    env = {**DEFAULTS, **(env or {})}
    if n == 0:
        return 0
    first = _first_half(ED, n, env, cached)
    return _sort(n) + 2 + (first + 2 if first else 0)


def mixed(counts, env=None, cached=()):
    """sbv_mixed_verify_batch over counts[scheme] items: the split (4), each family, k_mix_ok."""
    if sum(counts) == 0:
        return 0
    out = 5 + ed25519(counts[ED], env, cached)
    for c in (P256, P384):
        out += ecdsa(c, counts[c], True, env, cached, chunked=False)
    return out
