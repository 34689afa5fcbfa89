"""Every call that hashes on the device, past 32 bits (the CPU twin is test_hostsim_wide.py):

  a. messages whose bit length needs the high word: SHA-256 over 2^29 - 1 and 2^29 + 56 bytes, Ed25519 over M = 2^29 - 63
     bytes (bit length 2^32 + 8), each with a twin whose last byte is flipped;
  b. caller offsets past 2^32: the probe set of tests/wide_messages.py in a pageable, sparse buffer after 2^32 (the engine
     stages only the shard, so the kernels see small offsets);
  c. one shard larger than 4 GiB: a pinned blob of about 4,300 one-MiB fillers, then the probe set, so that the kernels,
     the chunked upload and the compacted blob of the mixed calls address bytes past 2^32.

Digests are compared where a call returns them, verdicts always, against hashlib and the OpenSSL oracles; quorum counts
against oracle.ecdsa_ref.count_commit_votes_batch.  Case c needs about 11 GiB of free device memory and 16 GiB of
available host memory (the pinned blob and the engine's pinned staging); the test skips, saying so, when the shared
machine has less.  One engine at a time: settings read at sbv_create (SBV_CHUNK_ITEMS, SBV_GROUP_THRESHOLD) get an
engine of their own, and the previous one is closed first."""
import ctypes as C
import os

import numpy as np
import pytest

import mixed_cases as mc
import wide_messages as wm
from oracle import ecdsa_ref
from oracle_ed25519 import ref

pytestmark = pytest.mark.gpu

GiB = 2**30
N_FILLERS = 4300


def _avail_host():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def _need(device_bytes, host_bytes):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < device_bytes:
        pytest.skip(f"needs {device_bytes / GiB:.1f} GiB of free device memory, {free / GiB:.1f} GiB free")
    if _avail_host() < host_bytes:
        pytest.skip(f"needs {host_bytes / GiB:.1f} GiB of available host memory, {_avail_host() / GiB:.1f} GiB available")


class Engines:
    """One engine at a time, created with the environment settings asked for, with the registries of `reg` loaded."""

    def __init__(self, reg):
        self.reg, self.env, self.eng = reg, None, None

    def get(self, **env):
        import consensus_b200 as sbv
        if self.eng is not None and env == self.env:
            return self.eng
        self.close()
        saved = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            self.eng = sbv.Engine(n_devices=1)
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k)
                else:
                    os.environ[k] = v
        self.env = env
        self.eng.set_keys(self.reg["ecdsa_curve"], self.reg["ecdsa_xy"])
        self.eng.ed25519_set_keys(self.reg["ed_pub"])
        return self.eng

    def close(self):
        if self.eng is not None:
            self.eng.close()
            self.eng = None


@pytest.fixture(scope="module")
def reg():
    return mc.registries(n256=1, n384=1, n_ed=1, seed=17)


@pytest.fixture(scope="module")
def engines(reg):
    e = Engines(reg)
    yield e
    e.close()


# ------------------------------------------------------------------------------------------------ the calls
CHUNKED = {"SBV_CHUNK_ITEMS": "256"}
GENERIC = {"SBV_GROUP_THRESHOLD": "0"}
SLOT = {wm.P256: 0, wm.P384: 1, wm.ED: 0}  # registries(n256=1, n384=1): ECDSA slot 0 is P-256, slot 1 P-384


def _votes(n):
    inst = (np.arange(n) // 4).astype(np.uint32)
    who = (np.arange(n) % 4 + 1).astype(np.uint16)
    return inst, who, who.copy(), np.ones(n, np.uint8), int(inst[-1]) + 1


def _sig96(it):
    n, tag, sg = it["n"], it["tag"], it["sigs"]
    rows = np.zeros((n, 96), np.uint8)
    for c, L in ((wm.P256, 32), (wm.P384, 48)):
        i = tag == c
        rows[i, :L], rows[i, L:2 * L] = sg[c][0][i], sg[c][1][i]
    rows[tag == wm.ED, :64] = sg[wm.ED][tag == wm.ED]
    return rows


def _keys(reg, c, n):
    L = {wm.P256: 32, wm.P384: 48}[c]
    xy = reg["ecdsa_xy"][SLOT[c]]
    return np.tile(xy[48 - L:48], (n, 1)), np.tile(xy[96 - L:], (n, 1))


def run_call(engines, name, it):
    """Runs call `name` on the items `it` and checks what it returns."""
    reg, msgs, off, n, exp = engines.reg, it["msgs"], it["off"], it["n"], it["exp"]
    sg = it["sigs"]
    if name == "sha256_batch":
        got = engines.get().sha256_batch(msgs, off)
        assert np.array_equal(got, it["dig"]), np.flatnonzero((got != it["dig"]).any(1))[:20]
    elif name in ("hash_verify_batch", "hash_verify_batch_chunked"):
        qx, qy = _keys(reg, wm.P256, n)
        ok, dig = engines.get(**(CHUNKED if name.endswith("chunked") else {})).hash_verify_batch(wm.P256, msgs, off, sg[wm.P256][0], sg[wm.P256][1], qx, qy,
                                                                                                 want_digest=True)
        assert np.array_equal(dig, it["dig"]), np.flatnonzero((dig != it["dig"]).any(1))[:20]
        assert np.array_equal(ok, exp[wm.P256]), np.flatnonzero(ok != exp[wm.P256])[:20]
    elif name in ("hash_verify_registered_p256", "hash_verify_registered_p384"):
        c = wm.P256 if name.endswith("p256") else wm.P384
        ok = engines.get().hash_verify_registered(c, msgs, off, np.full(n, SLOT[c], np.uint32), sg[c][0], sg[c][1])
        assert np.array_equal(ok, exp[c]), np.flatnonzero(ok != exp[c])[:20]
    elif name in ("ed25519_verify_batch_grouped", "ed25519_verify_batch_generic"):
        eng = engines.get(**(GENERIC if name.endswith("generic") else {}))
        ok = eng.ed25519_verify_batch(msgs, off, sg[wm.ED], np.tile(reg["ed_pub"][0], (n, 1)))
        assert np.array_equal(ok, exp[wm.ED]), np.flatnonzero(ok != exp[wm.ED])[:20]
    elif name == "ed25519_verify_registered":
        ok = engines.get().ed25519_verify_registered(msgs, off, np.zeros(n, np.uint32), sg[wm.ED])
        assert np.array_equal(ok, exp[wm.ED]), np.flatnonzero(ok != exp[wm.ED])[:20]
    elif name == "ed25519_verify_quorum":
        inst, snd, sgn, dm, ni = _votes(n)
        ok, cnt, reached = engines.get().ed25519_verify_quorum(msgs, off, np.zeros(n, np.uint32), sg[wm.ED], inst, snd, sgn, dm, ni, 3)
        want_cnt, want_reached = ecdsa_ref.count_commit_votes_batch(inst, snd, sgn, dm, exp[wm.ED], ni, 3)
        assert np.array_equal(ok, exp[wm.ED]), np.flatnonzero(ok != exp[wm.ED])[:20]
        assert np.array_equal(cnt, want_cnt) and np.array_equal(reached, want_reached)
    elif name in ("mixed_verify_registered", "mixed_verify_quorum"):
        tag = it["tag"]
        want = np.choose(tag, [exp[wm.P256], exp[wm.P384], exp[wm.ED]]).astype(np.uint8)
        slot = np.array([SLOT[int(t)] for t in tag], np.uint32)
        if name == "mixed_verify_registered":
            ok = engines.get().mixed_verify_registered(tag, msgs, off, slot, _sig96(it))
        else:
            inst, snd, sgn, dm, ni = _votes(n)
            ok, cnt, reached = engines.get().mixed_verify_quorum(tag, msgs, off, slot, _sig96(it), inst, snd, sgn, dm, ni, 3)
            want_cnt, want_reached = ecdsa_ref.count_commit_votes_batch(inst, snd, sgn, dm, want, ni, 3)
            assert np.array_equal(cnt, want_cnt) and np.array_equal(reached, want_reached)
        assert np.array_equal(ok, want), np.flatnonzero(ok != want)[:20]
    else:
        raise ValueError(name)


# grouped by the engine they need, so that engines are not recreated between neighbours
CALLS = ["sha256_batch", "hash_verify_batch", "hash_verify_registered_p256", "hash_verify_registered_p384", "ed25519_verify_batch_grouped",
         "ed25519_verify_registered", "ed25519_verify_quorum", "mixed_verify_registered", "mixed_verify_quorum", "hash_verify_batch_chunked",
         "ed25519_verify_batch_generic"]


def _items(reg, msgs, off, lay, seed):
    sigs, dig = wm.sign_items(reg, msgs, off, lay, seed)
    exp = wm.expected_ok(reg, msgs, off, sigs, dig)
    for c in (wm.P256, wm.P384, wm.ED):  # probes, spacers and fillers accept, twins reject
        assert np.array_equal(exp[c], wm.expected_kinds(lay)), (c, np.flatnonzero(exp[c] != wm.expected_kinds(lay))[:20])
    return {"msgs": msgs, "off": off, "n": lay.n, "tag": lay.tag, "sigs": sigs, "dig": dig, "exp": exp}


# ------------------------------------------------------------------------------------------------ a. huge messages
def test_sha256_bit_length_past_32_bits(engines):
    """The two long messages alone (no length sort below 2,048 items), then with 2,046 short ones (the sort runs and both
    land in its last bin)."""
    _need(3 * GiB, 4 * GiB)
    lens = list(wm.HUGE_SHA)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    buf = wm.pattern(int(off[-1]) + 2 * 2046 * 100 + 64, seed=1)
    want = np.frombuffer(b"".join(wm.sha256_ref(buf, off)), np.uint8).reshape(-1, 32)
    eng = engines.get()
    assert np.array_equal(eng.sha256_batch(buf, off), want)
    short = np.random.default_rng(2).integers(0, 200, 2046)
    off2 = np.concatenate([off, int(off[-1]) + np.cumsum(short)]).astype(np.uint64)
    want2 = np.frombuffer(b"".join(wm.sha256_ref(buf, off2)), np.uint8).reshape(-1, 32)
    assert np.array_equal(eng.sha256_batch(buf, off2), want2)


def _with_twins(lens, seed):
    """Each length followed by its twin (a copy with the last byte flipped)."""
    off = np.concatenate([[0], np.cumsum([ln for ln in lens for _ in (0, 1)])]).astype(np.uint64)
    buf = np.empty(int(off[-1]) + 16, np.uint8)
    for k, ln in enumerate(lens):
        a = int(off[2 * k])
        buf[a:a + ln] = wm.pattern(ln, seed + k)
        buf[a + ln:a + 2 * ln] = buf[a:a + ln]
        buf[a + 2 * ln - 1] ^= 0x01
    return buf, off


def test_hash_verify_batch_bit_length_past_32_bits(engines, reg):
    _need(5 * GiB, 9 * GiB)
    buf, off = _with_twins(wm.HUGE_SHA, 3)
    lay = wm.Layout(np.diff(off.astype(np.int64)), np.zeros(4, np.uint8), [wm.PROBE, wm.TWIN] * 2, [-1, 0, -1, 2])
    it = _items(reg, buf, off, lay, 4)
    assert [bytes(d) for d in it["dig"]] == wm.sha256_ref(buf, off)
    run_call(engines, "hash_verify_batch", it)


def test_ed25519_bit_length_past_32_bits(engines, reg):
    """SHA-512(R || A || M) and k = digest mod L through the debug hook, then the verdicts of sbv_ed25519_verify_batch."""
    _need(4 * GiB, 5 * GiB)
    buf, off = _with_twins([wm.HUGE_ED], 5)
    lay = wm.Layout(np.diff(off.astype(np.int64)), np.full(2, wm.ED, np.uint8), [wm.PROBE, wm.TWIN], [-1, 0])
    import oracle_ed25519 as oe
    sig = oe.sign_batch(reg["ed_seeds"][:1], np.zeros(2, np.uint32), buf, off)
    sig[1] = sig[0]  # the twin carries its probe's signature
    pub = np.tile(reg["ed_pub"][0], (2, 1))
    eng = engines.get()
    dig = np.zeros((2, 64), np.uint8)
    k = np.zeros((2, 8), np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert eng._lib.sbv_debug_ed25519_sha512(eng._h, C.c_size_t(2), p(buf), p(off), p(sig), p(pub), p(dig), p(k)) == 0
    want = wm.sha512_ref(buf, off, sig, pub)
    for i in range(2):
        assert bytes(dig[i]) == want[i], i
        assert sum(int(k[i, w]) << (32 * w) for w in range(8)) == int.from_bytes(want[i], "little") % ref.L, i
    assert np.array_equal(oe.verify_batch(buf, off, sig, pub), wm.expected_kinds(lay))
    assert np.array_equal(eng.ed25519_verify_batch(buf, off, sig, pub), wm.expected_kinds(lay))


# ------------------------------------------------------------------------------------------------ b. caller offsets past 2^32
@pytest.fixture(scope="module")
def far_items(reg):
    lay = wm.probe_layout()
    buf = wm.sparse(wm.FAR + lay.bytes + 64)
    off = wm.fill(buf, wm.FAR, lay, 41)
    assert int(off[0]) > 2**32
    return _items(reg, buf, off, lay, 42)


@pytest.mark.parametrize("name", CALLS)
def test_caller_offsets_past_2_32(engines, far_items, name):
    run_call(engines, name, far_items)


# ------------------------------------------------------------------------------------------------ c. one shard past 4 GiB
@pytest.fixture(scope="module")
def big_items(reg):
    """A pinned blob of N_FILLERS fillers of about 1 MiB, then the probe set; every item signed under every scheme."""
    import consensus_b200 as sbv
    lay = wm.probe_layout([2**20 + (i * 37) % 97 for i in range(N_FILLERS)])
    _need(11 * GiB, 16 * GiB)
    lib = sbv.load_library()
    lib.sbv_host_alloc.restype = C.c_void_p
    lib.sbv_host_free.argtypes = [C.c_void_p]
    size = lay.bytes + 64
    ptr = lib.sbv_host_alloc(C.c_size_t(size))
    assert ptr, "sbv_host_alloc failed"
    try:
        blob = np.ctypeslib.as_array((C.c_uint8 * size).from_address(ptr))
        block = wm.pattern(2**20 + 8192, seed=6)
        off = lay.offsets(0)
        for i in np.flatnonzero(lay.kind == wm.FILLER):
            a, b = int(off[i]), int(off[i + 1])
            s = (int(i) * 41) % 4096
            blob[a:b] = block[s:s + b - a]
            blob[a:a + 4] = np.frombuffer(int(i).to_bytes(4, "little"), np.uint8)
        wm.fill(blob, 0, lay, 43)
        blob[lay.bytes:] = 0
        p = int(np.flatnonzero(lay.kind == wm.PROBE)[0])
        assert int(off[p]) > 2**32 and int(off[-1]) - int(off[0]) > 4 * GiB
        yield _items(reg, blob, off, lay, 44)
    finally:
        lib.sbv_host_free(C.c_void_p(ptr))


@pytest.mark.parametrize("name", CALLS)
def test_shard_past_4_gib(engines, big_items, name):
    if name == "mixed_verify_registered":  # the P-256 fillers come first: the other families' regions start past 2^32
        tag, lens = big_items["tag"], np.diff(big_items["off"].astype(np.int64))
        assert int(lens[tag == wm.P256].sum()) > 2**32 and (tag[:N_FILLERS] == wm.P256).all()
    run_call(engines, name, big_items)
