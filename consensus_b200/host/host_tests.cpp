// host_tests.cpp — tests of the C++ host mirror.  `host_tests cpu` runs the reference-shaped tests
// with a mock verifier (no GPU); `host_tests gpu` runs the same call sites on the real engine with
// real ECDSA signatures (OpenSSL is used HERE ONLY, as the test's signer).
//
// Each test names the reference test it mirrors (/root/reference/internal/bft/*_test.go).
#include <array>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <thread>

#include "callsites.hpp"
#include "marshal.hpp"

using namespace sbft;

static int g_fail = 0, g_checks = 0;
#define CHECK(cond)                                                                      \
    do {                                                                                 \
        g_checks++;                                                                      \
        if (!(cond)) { g_fail++; fprintf(stderr, "  FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); } \
    } while (0)
#define RUN(t)                    \
    do {                          \
        int before = g_fail;      \
        t();                      \
        printf("%-58s %s\n", #t, g_fail == before ? "ok" : "FAILED"); \
    } while (0)

// ---- mock verifier, the shape of mocks/verifier_mock.go ----
struct MockVerifier : IVerifier {
    std::function<Error(const Signature &, const Proposal &)> consenter = [](const Signature &, const Proposal &) { return Error(); };
    std::function<Error(const Bytes &)> request = [](const Bytes &) { return Error(); };
    uint64_t verSeq = 1;
    int consenterCalls = 0, requestCalls = 0;
    std::pair<std::vector<RequestInfo>, Error> VerifyProposal(const Proposal &) override { return {{}, std::nullopt}; }
    std::pair<RequestInfo, Error> VerifyRequest(const Bytes &val) override { requestCalls++; return {RequestInfo{"c", std::string(val.begin(), val.end())}, request(val)}; }
    std::pair<Bytes, Error> VerifyConsenterSig(const Signature &s, const Proposal &p) override { consenterCalls++; return {AuxiliaryData(s.Msg), consenter(s, p)}; }
    Error VerifySignature(const Signature &) override { return std::nullopt; }
    uint64_t VerificationSequence() override { return verSeq; }
    std::vector<RequestInfo> RequestsFromProposal(const Proposal &) override { return {}; }
    Bytes AuxiliaryData(const Bytes &m) override { return m; }
};

// fixtures of view_test.go:31-122
static Proposal fixtureProposal() { return Proposal{{1}, {0}, ViewMetadata{1, 0, 0}.Marshal(), 1}; }
static Proposal fixtureWrongProposal() { return Proposal{{2}, {1}, {3}, 1}; }
static Vote prepareFrom(uint64_t sender, const std::string &digest) { Vote v; v.sender = sender; v.prepare = PrepareMsg{1, 0, digest, false}; return v; }
static Vote commitFrom(uint64_t sender, uint64_t signer, const std::string &digest) {
    Vote v; v.sender = sender;
    CommitMsg c; c.View = 1; c.Seq = 0; c.Digest = digest; c.Sig = ProtoSignature{signer, {4}, {}};
    v.commit = c;
    return v;
}

static void TestProposalDigestFixtures() {
    // DER of the view_test.go fixtures (values derived in SURVEY.md §8c)
    CHECK(hex(fixtureProposal().Der()) == "300d04010104010004020801020101");
    CHECK(hex(fixtureWrongProposal().Der()) == "300c040102040101040103020101");
    CHECK(fixtureProposal().Digest() == hex(sha256(fixtureProposal().Der())));
    CHECK(hex(sha256(Bytes{'a', 'b', 'c'})) == "ba7816bf8f01cfea414140de5dae2223b00361a396177a9cb410ff61f20015ad");
    CHECK(hex(sha256(Bytes{})) == "e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855");
    Bytes m(119, 'x');  // padding spills into a second block
    CHECK(sha256(m).size() == 32);
    CHECK(CommitSignaturesDigest({}).empty());  // util.go:565-567 nil for empty input
    CHECK(CommitSignaturesDigest({Signature{1, {4}, {5}}}).size() == 32);
    Proposal big{Bytes(300, 0xaa), {}, {}, 128};
    Bytes d = big.Der();
    CHECK(d[0] == 0x30 && d[1] == 0x82 && d[2] == 0x01 && d[3] == 0x38);
}

// tests/golden/digests_and_quorum.txt (the oracle's values; tests/test_golden.py pins the oracle to the same file)
struct GoldenProposal { Proposal p; const char *digest; };
static std::vector<GoldenProposal> goldenProposals() {
    return {
        {Proposal{{1}, {0}, {8, 1}, 1}, "45c32e94b3c427ee4a3f9b5964d3c5f9c15f3cfa7a28093eae8ca10d151fd892"},
        {Proposal{{2}, {1}, {3}, 1}, "d7707e2a07e57fdfdd54e73b869e3668f64db840920225cb3cc6bcaf509e45dd"},
        {Proposal{{}, {}, {}, 0}, "cc67164898e13d2ad50b32e740d8841aef5d0be6daefdf13492405ab087f793f"},
        {Proposal{Bytes(300, 0xaa), {'h'}, Bytes(130, 'm'), 128}, "99adadae41630b50ef7271ed34dfc1b9683e99a2ea7b2a41b76b337da9bef0ee"},
        {Proposal{{'p'}, {}, {}, -1}, "df1e849969833046e2920cedcad6355e1416526e8aee58b3d34114899c44e512"},
        {Proposal{{'p'}, {'q'}, {'r'}, (int64_t)1 << 40}, "ca563970278c698b36ace68926c2b505f7cae38ee36a3694e35909101a6dc562"},
    };
}
static const char *GOLDEN_COMMITSIGS = "ffc4b7e5e35c1ec4fe5cc27aab3f5ab06f2e721d97dd267e793e7c944105483b";
static std::vector<Signature> goldenCommitSigs() { return {Signature{1, {4}, {5}}, Signature{2, Bytes(70, 4), {}}}; }

static void TestGoldenDigests() {  // types.go:50-69, util.go:564-595 against the oracle's golden values
    for (auto &g : goldenProposals()) CHECK(g.p.Digest() == g.digest);
    CHECK(hex(CommitSignaturesDigest(goldenCommitSigs())) == GOLDEN_COMMITSIGS);
}

static void TestWireCodecs() {  // messages.proto:41-58, 92-96
    CommitMsg c; c.View = 3; c.Seq = 77; c.Digest = std::string(64, 'a'); c.Sig = ProtoSignature{9, {1, 2, 3}, {4, 5}}; c.Assist = true;
    Bytes w = MarshalCommit(c);
    CommitView v;
    CHECK(DecodeCommit(w.data(), w.size(), v));
    CHECK(v.View == 3 && v.Seq == 77 && v.Signer == 9 && v.has_sig && v.Assist);
    CHECK(v.digest_len == 64 && memcmp(v.digest, c.Digest.data(), 64) == 0);
    CHECK(v.value_len == 3 && v.value[2] == 3 && v.msg_len == 2 && v.msg[1] == 5);
    // golang/protobuf bytes of Commit{view:1, digest:"ab", signature:{signer:2, value:0x07}}
    const uint8_t golden[] = {0x08, 0x01, 0x1a, 0x02, 'a', 'b', 0x22, 0x05, 0x08, 0x02, 0x12, 0x01, 0x07};
    CommitMsg g; g.View = 1; g.Digest = "ab"; g.Sig = ProtoSignature{2, {7}, {}};
    Bytes gw = MarshalCommit(g);
    CHECK(gw.size() == sizeof golden && memcmp(gw.data(), golden, sizeof golden) == 0);
    for (size_t cut = 1; cut < w.size(); cut++) {  // every truncation is either rejected or decodes to a prefix — never reads out of bounds
        CommitView t;
        (void)DecodeCommit(w.data(), cut, t);
    }
    Bytes bad = w; bad[bad.size() - 3] = 0xff;  // length byte of the last field now overruns
    CommitView t;
    (void)DecodeCommit(bad.data(), bad.size(), t);
    PrepareMsg p{5, 6, "deadbeef", false}, q;
    Bytes pw = MarshalPrepare(p);
    CHECK(DecodePrepare(pw.data(), pw.size(), q) && q.View == 5 && q.Seq == 6 && q.Digest == "deadbeef" && !q.Assist);
    const uint8_t unknown_field[] = {0x08, 0x01, 0x78, 0x05};  // field 15 varint: skipped
    CHECK(DecodeCommit(unknown_field, sizeof unknown_field, t) && t.View == 1);
    const uint8_t field_zero[] = {0x00, 0x01};
    CHECK(!DecodeCommit(field_zero, sizeof field_zero, t));
}

static void TestQuorum() {  // util_test.go:135-163
    const int table[][3] = {{4, 1, 3}, {5, 1, 4}, {6, 1, 4}, {7, 2, 5}, {8, 2, 6}, {9, 2, 6}, {10, 3, 7}, {11, 3, 8}, {12, 3, 8}};
    for (auto &row : table) { int q, f; computeQuorum(row[0], q, f); CHECK(f == row[1]); CHECK(q == row[2]); }
    int q, f; computeQuorum(16, q, f); CHECK(q == 11 && f == 5);
}

static void TestBadPrepare() {  // view_test.go:362-464: a prepare with a wrong digest is logged and not counted
    Proposal p = fixtureProposal();
    ViewLog log;
    auto ids = processPrepares(p, 3, 1, {prepareFrom(2, fixtureWrongProposal().Digest()), prepareFrom(3, p.Digest()), prepareFrom(3, p.Digest()), prepareFrom(4, p.Digest())}, &log);
    CHECK((ids == std::vector<uint64_t>{3, 4}));
    CHECK(log.warnings.size() == 1 && log.warnings[0].find("Got wrong digest") != std::string::npos);
    // the wrong-digest voter burnt its slot: a later correct prepare from 2 is a double vote
    ids = processPrepares(p, 4, 1, {prepareFrom(2, "bad"), prepareFrom(2, p.Digest()), prepareFrom(3, p.Digest())}, nullptr);
    CHECK((ids == std::vector<uint64_t>{3}));
}

static void TestBadCommit() {  // view_test.go:466-531
    Proposal p = fixtureProposal();
    MockVerifier v;
    v.consenter = [](const Signature &, const Proposal &) { return Errorf(""); };
    ViewLog log;
    // commit with wrong digest from 1 -> "Got wrong digest"; commit from 2 -> "Couldn't verify 2's signature:"
    auto sigs = processCommits(v, p, 3, 4, {commitFrom(1, 1, fixtureWrongProposal().Digest()), commitFrom(2, 2, p.Digest())}, &log);
    CHECK(sigs.empty());
    CHECK(log.warnings.size() == 2);
    CHECK(log.warnings[0].find("Got wrong digest") != std::string::npos);
    CHECK(log.warnings[1].find("Couldn't verify 2's signature:") != std::string::npos);
    CHECK(v.consenterCalls == 1);  // the wrong-digest vote never reaches the verifier (view.go:829-832)
}

static void TestNormalPath() {  // view_test.go:533-673: n=4, Q=3, self=1, signer ID 4
    Proposal p = fixtureProposal();
    MockVerifier v;
    auto voters = processPrepares(p, 3, 1, {prepareFrom(2, p.Digest()), prepareFrom(3, p.Digest())});
    CHECK((voters == std::vector<uint64_t>{2, 3}));
    Bytes aux = PreparesFrom{voters}.Marshal();  // view.go:472-481
    PreparesFrom back;
    CHECK(PreparesFrom::Unmarshal(aux, back) && back.Ids == voters);
    auto sigs = processCommits(v, p, 3, 1, {commitFrom(2, 2, p.Digest()), commitFrom(3, 3, p.Digest())});
    CHECK(sigs.size() == 2);
    sigs.push_back(Signature{4, {4}, {}});  // decide() appends the node's own signature (view.go:856)
    CHECK(sigs.size() == 3);
    for (auto &s : sigs) CHECK(s.ID == 2 || s.ID == 3 || s.ID == 4);
    // Signer != sender is not registered (view.go:161-171); self votes are ignored; double votes dropped
    sigs = processCommits(v, p, 3, 1, {commitFrom(2, 3, p.Digest()), commitFrom(1, 1, p.Digest()), commitFrom(2, 2, p.Digest()), commitFrom(2, 2, p.Digest())});
    CHECK(sigs.size() == 1 && sigs[0].ID == 2);
    // more candidates than needed: only Quorum-1 are returned
    sigs = processCommits(v, p, 3, 1, {commitFrom(2, 2, p.Digest()), commitFrom(3, 3, p.Digest()), commitFrom(4, 4, p.Digest())});
    CHECK(sigs.size() == 2);
}

static void TestValidateLastDecision() {  // viewchanger_test.go:1415-1522, the same eight cases
    Bytes metadata = ViewMetadata{0, 1, 0}.Marshal();
    std::vector<ProtoSignature> lastSigs = {{1, {4}, {5}}, {2, {4}, {5}}, {3, {4}, {5}}};
    struct Case { const char *description; ViewData vd; bool verifyFails; bool valid; uint64_t sequence; };
    auto mk = [&](uint64_t nextView, std::optional<Proposal> ld, std::vector<ProtoSignature> sigs) { ViewData v; v.NextView = nextView; v.LastDecision = ld; v.LastDecisionSignatures = sigs; return v; };
    std::vector<Case> cases = {
        {"last decision is not set", mk(0, std::nullopt, {}), false, false, 0},
        {"last decision metadata is nil", mk(0, Proposal{}, {}), false, true, 0},
        {"unable to unmarshal last decision metadata", mk(0, Proposal{{}, {}, {0}, 0}, {}), false, false, 0},
        {"last decision view is greater or equal to requested next view", mk(1, Proposal{{}, {}, ViewMetadata{1, 1, 0}.Marshal(), 0}, {}), false, false, 0},
        {"not enough signatures", mk(1, Proposal{{}, {}, metadata, 0}, {}), false, false, 0},
        {"invalid signatures", mk(1, Proposal{{}, {}, metadata, 0}, lastSigs), true, false, 0},
        {"not enough valid signatures", mk(1, Proposal{{}, {}, metadata, 0}, {{0, {4}, {5}}, {0, {4}, {5}}, {1, {4}, {5}}}), false, false, 0},
        {"valid last decision", mk(1, Proposal{{}, {}, metadata, 0}, lastSigs), false, true, 1},
    };
    for (auto &c : cases) {
        MockVerifier v;
        if (c.verifyFails) v.consenter = [](const Signature &, const Proposal &) { return Errorf(""); };
        auto res = ValidateLastDecision(c.vd, 3, 4, v);
        if (c.valid) CHECK(!res.second); else CHECK(res.second.has_value());
        CHECK(res.first == c.sequence);
        if (g_fail) fprintf(stderr, "   case: %s\n", c.description);
    }
}

static void TestVerifyPrevCommitSignatures() {  // view.go:606-647
    Proposal prev = fixtureProposal();
    MockVerifier v;
    Bytes aux = PreparesFrom{{2, 3}}.Marshal();
    std::vector<ProtoSignature> sigs = {{2, {4}, aux}, {3, {4}, aux}, {4, {4}, aux}};
    auto res = verifyPrevCommitSignatures(v, sigs, prev, 1);
    CHECK(!res.second && res.first.size() == 3 && res.first[3].Ids == (std::vector<uint64_t>{2, 3}));
    res = verifyPrevCommitSignatures(v, sigs, prev, 2);  // verification sequence advanced -> skipped
    CHECK(!res.second && res.first.empty());
    v.consenter = [](const Signature &s, const Proposal &) { return s.ID == 3 ? Errorf("bad") : Error(); };
    res = verifyPrevCommitSignatures(v, sigs, prev, 1);
    CHECK(res.second && res.second->find("failed verifying consenter signature of 3") != std::string::npos);
    v.consenter = [](const Signature &, const Proposal &) { return Error(); };
    sigs[1].Msg = {0x0A, 0x05, 0x01};  // truncated packed field -> aux does not unmarshal
    res = verifyPrevCommitSignatures(v, sigs, prev, 1);
    CHECK(res.second && res.second->find("failed unmarshaling auxiliary input from 3") != std::string::npos);
}

static void TestReqPoolPrune() {  // requestpool_test.go:264-302
    Pool pool;
    MockVerifier v;
    Bytes req1{'1'}, req2{'2'};
    pool.Submit(req1, {"1", "1"});
    pool.Submit(req2, {"2", "2"});
    CHECK(pool.Size() == 2);
    v.request = [&](const Bytes &p) { return p == req1 ? Errorf("revoked") : Error(); };
    CHECK(pool.Prune(v) == 1);
    CHECK(pool.Size() == 1 && pool.requests()[0].second == (RequestInfo{"2", "2"}));
    uint64_t cached = 1;
    CHECK(!MaybePruneRevokedRequests(cached, v, pool));  // controller.go:736-738: unchanged sequence -> nothing
    v.verSeq = 2;
    CHECK(MaybePruneRevokedRequests(cached, v, pool) && cached == 2);
}

static void TestControllerLeaderRequestHandling() {  // controller_test.go:548-661
    Pool pool;
    MockVerifier v;
    CHECK(!HandleRequest(false, v, pool, {'x'}));  // not the leader: verifier not called
    CHECK(v.requestCalls == 0 && pool.Size() == 0);
    v.request = [](const Bytes &) { return Errorf("bad"); };
    CHECK(!HandleRequest(true, v, pool, {'x'}));   // bad request: not enqueued
    CHECK(v.requestCalls == 1 && pool.Size() == 0);
    v.request = [](const Bytes &) { return Error(); };
    CHECK(HandleRequest(true, v, pool, {'x'}));    // good: submitted
    CHECK(pool.Size() == 1);
}

static void TestAggregatorCoalesces() {
    std::atomic<int> calls{0};
    Aggregator agg([&](const std::vector<SigItem> &items) { calls++; std::vector<uint8_t> ok; for (auto &it : items) ok.push_back(it.r[0] & 1); return ok; },
                   std::chrono::microseconds(20000), 1 << 20);
    std::vector<std::thread> th;
    std::vector<int> res(15, -1);
    for (int i = 0; i < 15; i++) th.emplace_back([&, i] { SigItem it{}; it.r[0] = (uint8_t)i; res[i] = agg.submit(it); });  // N-1 concurrent callers
    for (auto &t : th) t.join();
    for (int i = 0; i < 15; i++) CHECK(res[i] == (i & 1));
    CHECK(calls.load() <= 3);  // coalesced (normally 1 batch)
    // size-capped flush does not wait for the deadline
    Aggregator agg2([&](const std::vector<SigItem> &items) { return std::vector<uint8_t>(items.size(), 1); }, std::chrono::microseconds(5000000), 1);
    auto t0 = std::chrono::steady_clock::now();
    SigItem it{};
    CHECK(agg2.submit(it));
    CHECK(std::chrono::steady_clock::now() - t0 < std::chrono::seconds(2));
    // a lone call is released by the deadline (processCommits must never deadlock, view.go:531)
    Aggregator agg3([&](const std::vector<SigItem> &items) { return std::vector<uint8_t>(items.size(), 0); }, std::chrono::microseconds(1000), 1 << 20);
    CHECK(!agg3.submit(it));
    // faults propagate as exceptions, never as verdicts
    Aggregator agg4([&](const std::vector<SigItem> &) -> std::vector<uint8_t> { throw EngineFault("boom"); }, std::chrono::microseconds(100), 4);
    bool threw = false;
    try { agg4.submit(it); } catch (const EngineFault &) { threw = true; }
    CHECK(threw);
}

// ================================================================================================ GPU part
#include "test_signer.hpp"

static void TestGpuVerifierEndToEnd() {
    GpuVerifier v({0});
    v.SetVerificationSequence(1);
    std::map<uint64_t, TestKey> keys;
    for (uint64_t id = 1; id <= 16; id++) { keys[id] = makeKey(); v.SetConsenterKey(id, keys[id].xy); }
    Proposal p = fixtureProposal();
    Bytes aux = PreparesFrom{{2, 3}}.Marshal();

    // single calls (the reference shape) — valid, wrong proposal, corrupted, unknown signer, malformed DER
    Signature good = signProposal(2, keys[2], p, aux);
    auto r = v.VerifyConsenterSig(good, p);
    CHECK(!r.second && r.first == aux && v.AuxiliaryData(good.Msg) == aux);
    CHECK(v.VerifyConsenterSig(good, fixtureWrongProposal()).second.has_value());
    Signature bad = good; bad.Value[bad.Value.size() - 1] ^= 1;
    CHECK(v.VerifyConsenterSig(bad, p).second.has_value());
    Signature other = good; other.ID = 3;
    CHECK(v.VerifyConsenterSig(other, p).second.has_value());
    Signature unknown = good; unknown.ID = 99;
    CHECK(v.VerifyConsenterSig(unknown, p).second.has_value());
    Signature trailing = good; trailing.Value.push_back(0);
    CHECK(v.VerifyConsenterSig(trailing, p).second.has_value());
    CHECK(!v.VerifySignature(good));
    Signature tampered = good; tampered.Msg.push_back(7);
    CHECK(v.VerifySignature(tampered).has_value());

    // TestNormalPath on real signatures, n=16 (Q=11): 15 concurrent single calls coalesce in the aggregator
    int q, f; computeQuorum(16, q, f);
    std::vector<Vote> votes;
    for (uint64_t id = 2; id <= 16; id++) {
        Signature s = signProposal(id, keys[id], p, aux);
        if (id == 5) s.Value[10] ^= 0x40;                 // Byzantine: bad signature
        Vote vt = commitFrom(id, id, id == 6 ? fixtureWrongProposal().Digest() : p.Digest());  // 6: wrong digest
        vt.commit->Sig = ProtoSignature{id, s.Value, s.Msg};
        votes.push_back(vt);
    }
    ViewLog log;
    auto sigs = processCommits(v, p, q, 1, votes, &log);
    CHECK((int)sigs.size() == q - 1);
    for (auto &s : sigs) CHECK(s.ID != 5 && s.ID != 6);
    CHECK(log.warnings.size() >= 1);

    uint64_t b0 = v.aggregator().batches();
    std::vector<std::thread> th; std::vector<int> okv(15, -1);
    for (int i = 0; i < 15; i++) th.emplace_back([&, i] { Signature s = signProposal(2 + i, keys[2 + i], p, aux); okv[i] = !v.VerifyConsenterSig(s, p).second; });
    for (auto &t : th) t.join();
    for (int i = 0; i < 15; i++) CHECK(okv[i] == 1);
    CHECK(v.aggregator().batches() - b0 <= 15);

    // ValidateLastDecision / verifyPrevCommitSignatures on real signatures
    Proposal last{{9}, {8}, ViewMetadata{0, 7, 0}.Marshal(), 1};
    ViewData vd; vd.NextView = 1; vd.LastDecision = last;
    for (uint64_t id = 1; id <= 11; id++) { Signature s = signProposal(id, keys[id], last, aux); vd.LastDecisionSignatures.push_back({id, s.Value, s.Msg}); }
    auto vr = ValidateLastDecision(vd, q, 16, v);
    CHECK(!vr.second && vr.first == 7);
    auto pc = verifyPrevCommitSignatures(v, vd.LastDecisionSignatures, last, 1);
    CHECK(!pc.second && pc.first.size() == 11);
    vd.LastDecisionSignatures[4].Value[12] ^= 1;
    CHECK(ValidateLastDecision(vd, q, 16, v).second.has_value());
    CHECK(verifyPrevCommitSignatures(v, vd.LastDecisionSignatures, last, 1).second.has_value());

    // requests: VerifyRequest / VerifyProposal / Pool.Prune
    TestKey ck = makeKey(); v.SetClientKey("alice", ck.xy);
    std::vector<Bytes> reqs; Bytes payload;
    for (int i = 0; i < 100; i++) {
        Bytes body(64 + i, (uint8_t)i);
        Bytes sig = signDer(ck, signed_part("alice", std::to_string(i), body));
        Bytes req = frame_request(sig, "alice", std::to_string(i), body);
        reqs.push_back(req);
        for (int k = 3; k >= 0; k--) payload.push_back((uint8_t)(req.size() >> (8 * k)));
        payload.insert(payload.end(), req.begin(), req.end());
    }
    auto one = v.VerifyRequest(reqs[3]);
    CHECK(!one.second && one.first == (RequestInfo{"alice", "3"}));
    Proposal prop{payload, {}, {}, 1};
    auto vp = v.VerifyProposal(prop);
    CHECK(!vp.second && vp.first.size() == 100 && vp.first[99] == (RequestInfo{"alice", "99"}));
    CHECK(v.RequestsFromProposal(prop) == vp.first);  // viewchanger.go:1178 agreement
    Bytes badPayload = payload; badPayload[badPayload.size() - 5] ^= 1;  // flips a byte of the last request body
    CHECK(v.VerifyProposal(Proposal{badPayload, {}, {}, 1}).second.has_value());
    CHECK(v.VerifyProposal(Proposal{payload, {}, {}, 2}).second.has_value());  // wrong verification sequence
    Pool pool;
    for (int i = 0; i < 100; i++) { Bytes rq = reqs[i]; if (i % 10 == 0) rq[rq.size() - 1] ^= 1; pool.Submit(rq, {"alice", std::to_string(i)}); }
    CHECK(pool.Prune(v) == 10 && pool.Size() == 90);
    // Proposal.Digest in batch on the GPU equals the host digest (types.go:50-69), incl. long-form DER lengths
    std::vector<Proposal> props = {fixtureProposal(), fixtureWrongProposal(), Proposal{}, Proposal{Bytes(70000, 0x5a), {1, 2, 3}, Bytes(200, 7), -5}, prop, last};
    auto dg = v.DigestBatch(props);
    for (size_t i = 0; i < props.size(); i++) CHECK(dg[i] == props[i].Digest());
    // ... and both digest kinds equal the ORACLE's golden values, not just the host mirror
    std::vector<Proposal> gp;
    for (auto &g : goldenProposals()) gp.push_back(g.p);
    auto gd = v.DigestBatch(gp);
    for (size_t i = 0; i < gp.size(); i++) CHECK(gd[i] == goldenProposals()[i].digest);
    std::vector<Signature> lastSigs;
    for (auto &ps : vd.LastDecisionSignatures) lastSigs.push_back(Signature{ps.Signer, ps.Value, ps.Msg});
    std::vector<std::vector<Signature>> sets = {goldenCommitSigs(), std::vector<Signature>(), lastSigs};
    auto cs = v.CommitSignaturesDigestBatch(sets);
    CHECK(hex(cs[0]) == GOLDEN_COMMITSIGS && cs[1].empty() && cs[2] == CommitSignaturesDigest(lastSigs));

    // wire Commits -> pinned SoA batch -> one verify + one quorum call (marshal.hpp), against processCommits vote by vote
    {
        CommitBatch batch;
        std::vector<Proposal> props3 = {fixtureProposal(), last, Proposal{{7, 7}, {1}, ViewMetadata{2, 9, 1}.Marshal(), 1}};
        std::vector<std::vector<Vote>> all_votes;
        auto slot_of = [&](uint64_t signer) { return signer >= 1 && signer <= 16 ? (int)v.ConsenterSlot(signer) : -1; };
        v.engine_batch({});  // registry pushed to the engine (sbv_set_keys)
        for (size_t pi = 0; pi < props3.size(); pi++) {
            const Proposal &pp = props3[pi];
            batch.begin_instance(pp.Digest(), 1);
            std::vector<Vote> vs;
            for (uint64_t id = 2; id <= 16; id++) {
                Signature sg = signProposal(id, keys[id], pp, aux);
                uint64_t sender = id, signer = id;
                std::string dig = pp.Digest();
                if (pi == 0 && id == 4) sg.Value[9] ^= 2;                   // bad signature
                if (pi == 1 && id == 7) dig = fixtureWrongProposal().Digest();  // wrong digest
                if (pi == 1 && id == 9) signer = 10;                        // signer != sender
                if (pi == 2 && id == 12) sender = 11;                       // second vote of sender 11
                if (pi == 2 && id >= 3 && id <= 8) sg.Value[11] ^= 1;       // six bad signatures: quorum fails
                Vote vt = commitFrom(sender, signer, dig);
                vt.commit->Sig = ProtoSignature{signer, sg.Value, sg.Msg};
                vs.push_back(vt);
                Bytes wire = MarshalCommit(*vt.commit);
                if (pi == 0 && id == 16) wire.resize(wire.size() - 3);     // truncated on the wire
                batch.add_wire_commit((uint16_t)sender, wire.data(), wire.size(), slot_of);
                if (pi == 0 && id == 16) vs.pop_back();                     // the reference never sees an undecodable message
            }
            all_votes.push_back(vs);
        }
        CHECK(batch.size() == 45 && batch.instances() == 3 && batch.malformed().size() == 1);
        std::vector<uint8_t> okv2, reached; std::vector<uint32_t> cnt;
        batch.verify_and_count(v.engine(), q - 1, okv2, cnt, reached);
        for (size_t pi = 0; pi < props3.size(); pi++) {
            // reference semantics, vote by vote: how many valid distinct foreign votes does the stream hold?
            VoteSet set(acceptCommits);
            int valid = 0;
            for (auto &vt : all_votes[pi]) {
                if (vt.sender == 1) continue;
                size_t before = set.votes().size();
                set.registerVote(vt.sender, vt);
                if (set.votes().size() == before) continue;
                Signature sg{vt.commit->Sig->Signer, vt.commit->Sig->Value, vt.commit->Sig->Msg};
                if (vt.commit->Digest == props3[pi].Digest() && !v.VerifyConsenterSig(sg, props3[pi]).second) valid++;
            }
            CHECK((int)cnt[pi] == valid);
            CHECK(reached[pi] == (valid >= q - 1 ? 1 : 0));
        }
        CHECK(reached[0] == 1 && reached[1] == 1 && reached[2] == 0);
    }
    for (auto &kv : keys) EC_KEY_free(kv.second.k);
    EC_KEY_free(ck.k);
}

// Ed25519 commits from the wire (marshal.hpp, CommitBatch::Ed25519): three instances with the Byzantine cases of the
// CommitBatch block above, plus a Commit without a Signature, a 63-byte Value, an unknown signer and a Signer beyond 16
// bits.  Without a GPU only the decoding rules are checked: which votes are inert and which are registered with a
// rejecting row.  On the GPU one sbv_ed25519_verify_quorum call is compared vote by vote with the VoteSet restatement.
static bool g_gpu = false;  // `host_tests gpu`
static void TestEd25519CommitBatch() {
    std::map<uint64_t, TestEdKey> keys;
    for (uint64_t id = 1; id <= 16; id++) keys[id] = makeEdKey();
    auto slot_of = [](uint64_t signer) { return signer >= 1 && signer <= 16 ? (int)signer - 1 : -1; };
    int q, f; computeQuorum(16, q, f);
    Proposal last{{9}, {8}, ViewMetadata{0, 7, 0}.Marshal(), 1};
    std::vector<Proposal> props3 = {fixtureProposal(), last, Proposal{{7, 7}, {1}, ViewMetadata{2, 9, 1}.Marshal(), 1}};
    Bytes aux = PreparesFrom{{2, 3}}.Marshal();
    struct WireVote { uint16_t sender; Bytes wire; std::optional<Vote> seen; EdCommit want; };  // seen: what the reference receives
    std::vector<std::vector<WireVote>> all(props3.size());
    for (size_t pi = 0; pi < props3.size(); pi++) {
        const Proposal &pp = props3[pi];
        for (uint64_t id = 2; id <= 16; id++) {
            Signature sg = signProposalEd25519(id, keys[id], pp, aux);
            uint64_t sender = id, signer = id;
            std::string dig = pp.Digest();
            EdCommit want = EdCommit::Verify;
            if (pi == 0 && id == 4) sg.Value[9] ^= 2;                                        // bad signature
            if (pi == 0 && id == 5) { sg.Value.resize(63); want = EdCommit::Rejecting; }     // 63-byte Value: registered, rejects
            if (pi == 1 && id == 7) dig = fixtureWrongProposal().Digest();                   // wrong digest
            if (pi == 1 && id == 9) signer = 10;                                             // signer != sender
            if (pi == 1 && id == 13) { sender = signer = 99; want = EdCommit::Rejecting; }   // unknown signer: registered, rejects
            if (pi == 2 && id == 12) sender = 11;                                            // second vote of sender 11
            if (pi == 2 && id >= 3 && id <= 8) sg.Value[11] ^= 1;                            // six bad signatures: quorum fails
            if (pi == 2 && id == 14) { signer = 70000; want = EdCommit::Inert; }             // Signer beyond the 16-bit column
            Vote vt = commitFrom(sender, signer, dig);
            vt.commit->Sig = ProtoSignature{signer, sg.Value, sg.Msg};
            if (pi == 0 && id == 15) { vt.commit->Sig.reset(); want = EdCommit::Inert; }     // no Signature
            Bytes wire = MarshalCommit(*vt.commit);
            std::optional<Vote> seen = vt;
            if (pi == 0 && id == 16) { wire.resize(wire.size() - 3); seen.reset(); want = EdCommit::Inert; }  // truncated on the wire
            all[pi].push_back({(uint16_t)sender, wire, seen, want});
        }
    }
    // the decoding rules
    size_t n_inert = 0, n_rejecting = 0;
    for (auto &votes : all)
        for (auto &w : votes) {
            CommitView c;
            uint32_t slot = 0;
            const EdCommit k = decode_ed25519_commit(w.wire.data(), w.wire.size(), slot_of, c, slot);
            CHECK(k == w.want);
            CHECK((k == EdCommit::Verify) == (slot != ED25519_NO_SLOT));
            if (k == EdCommit::Verify) CHECK(slot == c.Signer - 1 && c.value_len == 64);
            n_inert += k == EdCommit::Inert;
            n_rejecting += k == EdCommit::Rejecting;
        }
    CHECK(n_inert == 3 && n_rejecting == 2);
    if (!g_gpu) return;

    sbv_engine *e = nullptr;
    CHECK(sbv_create(nullptr, 1, &e) == SBV_OK);
    if (!e) return;
    Bytes reg(16 * 32);
    for (uint64_t id = 1; id <= 16; id++) memcpy(&reg[32 * (id - 1)], keys[id].pub, 32);
    CHECK(sbv_ed25519_set_keys(e, 16, reg.data()) == SBV_OK);
    std::vector<uint8_t> okv, reached; std::vector<uint32_t> cnt;
    {
        CommitBatch batch(CommitBatch::Ed25519);
        for (size_t pi = 0; pi < props3.size(); pi++) {
            batch.begin_instance(props3[pi].Digest(), 1);
            for (auto &w : all[pi]) batch.add_wire_commit(w.sender, w.wire.data(), w.wire.size(), slot_of);
        }
        CHECK(batch.size() == 45 && batch.instances() == 3 && batch.malformed().size() == 3 && batch.rejected().size() == 2);
        batch.verify_and_count(e, q - 1, okv, cnt, reached);
    }
    size_t i = 0;
    for (size_t pi = 0; pi < props3.size(); pi++) {
        VoteSet set(acceptCommits);
        int valid = 0;
        for (auto &w : all[pi]) {
            const size_t at = i++;
            bool sig_ok = false;
            if (w.seen && w.seen->commit->Sig) {
                const ProtoSignature &ps = *w.seen->commit->Sig;
                sig_ok = ps.Signer >= 1 && ps.Signer <= 16 && verifyEd25519(keys[ps.Signer].pub, ps.Value, ps.Msg);
            }
            CHECK(okv[at] == (w.want == EdCommit::Verify && sig_ok ? 1 : 0));  // inert and rejecting rows reject
            if (!w.seen || w.seen->sender == 1) continue;
            size_t before = set.votes().size();
            set.registerVote(w.seen->sender, *w.seen);
            if (set.votes().size() == before) continue;
            if (w.seen->commit->Digest == props3[pi].Digest() && sig_ok) valid++;
        }
        CHECK((int)cnt[pi] == valid);
        CHECK(reached[pi] == (valid >= q - 1 ? 1 : 0));
    }
    CHECK(reached[0] == 1 && reached[1] == 1 && reached[2] == 0);
    CHECK(cnt[0] == 11 && cnt[1] == 12 && cnt[2] == 7);
    sbv_destroy(e);
    for (auto &kv : keys) EVP_PKEY_free(kv.second.k);
}

// Commits of a mixed consenter set from the wire (marshal.hpp, CommitBatch::Mixed): consenters 1-7 hold P-256 keys, 8-9
// P-384 keys and 10-16 Ed25519 keys.  Three instances with the Byzantine cases of TestEd25519CommitBatch, plus a DER
// Value with a trailing byte, a 63-byte Ed25519 Value, a raw 64-byte Value from an ECDSA signer, a P-384 vote claiming an
// Ed25519 signer and an unknown signer (all registered, rejecting), and the inert cases.  Without a GPU only the decoding
// rules are checked; on the GPU one sbv_mixed_verify_quorum call is compared vote by vote with the VoteSet restatement.
static void TestMixedCommitBatch() {
    std::map<uint64_t, TestEcKey> ec;
    std::map<uint64_t, TestEdKey> ed;
    for (uint64_t id = 1; id <= 9; id++) ec[id] = makeEcKey(id <= 7 ? 32 : 48);
    for (uint64_t id = 10; id <= 16; id++) ed[id] = makeEdKey();
    auto key_of = [](uint64_t signer) -> MixedKey {
        if (signer >= 1 && signer <= 9) return {(uint8_t)(signer <= 7 ? SBV_P256 : SBV_P384), (int)signer - 1};
        if (signer >= 10 && signer <= 16) return {(uint8_t)SBV_ED25519, (int)signer - 10};
        return {(uint8_t)SBV_ED25519, -1};
    };
    // crypto/ecdsa.VerifyASN1 or crypto/ed25519.Verify under the signer's own key
    auto sig_valid = [&](uint64_t signer, const Bytes &val, const Bytes &msg) {
        if (signer >= 1 && signer <= 9) return CpuVerifier::check(ec[signer].k, val, msg);
        return signer >= 10 && signer <= 16 && verifyEd25519(ed[signer].pub, val, msg);
    };
    int q, f; computeQuorum(16, q, f);
    Proposal last{{9}, {8}, ViewMetadata{0, 7, 0}.Marshal(), 1};
    std::vector<Proposal> props3 = {fixtureProposal(), last, Proposal{{7, 7}, {1}, ViewMetadata{2, 9, 1}.Marshal(), 1}};
    Bytes aux = PreparesFrom{{2, 3}}.Marshal();
    struct WireVote { uint16_t sender; Bytes wire; std::optional<Vote> seen; EdCommit want; };
    std::vector<std::vector<WireVote>> all(props3.size());
    for (size_t pi = 0; pi < props3.size(); pi++) {
        const Proposal &pp = props3[pi];
        for (uint64_t id = 2; id <= 16; id++) {
            Signature sg; sg.ID = id;
            sg.Msg = pp.DigestRaw(); sg.Msg.insert(sg.Msg.end(), aux.begin(), aux.end());
            sg.Value = id <= 9 ? signDerEc(ec[id].k, sg.Msg) : signEd25519(ed[id], sg.Msg);
            uint64_t sender = id, signer = id;
            std::string dig = pp.Digest();
            EdCommit want = EdCommit::Verify;
            if (pi == 0 && id == 4) sg.Value[9] ^= 2;                                        // bad P-256 signature
            if (pi == 0 && id == 5) { sg.Value.push_back(0); want = EdCommit::Rejecting; }   // DER with a trailing byte
            if (pi == 0 && id == 8) sg.Value[20] ^= 4;                                       // bad P-384 signature
            if (pi == 0 && id == 11) { sg.Value.resize(63); want = EdCommit::Rejecting; }    // 63-byte Ed25519 Value
            if (pi == 1 && id == 2) { sg.Value.assign(64, 0x30); want = EdCommit::Rejecting; }  // raw 64 bytes from a P-256 signer
            if (pi == 1 && id == 7) dig = fixtureWrongProposal().Digest();                   // wrong digest
            if (pi == 1 && id == 9) { signer = 10; want = EdCommit::Rejecting; }             // P-384 DER under an Ed25519 signer
            if (pi == 1 && id == 13) { sender = signer = 99; want = EdCommit::Rejecting; }   // unknown signer
            if (pi == 2 && id == 12) sender = 11;                                            // second vote of sender 11
            if (pi == 2 && id >= 3 && id <= 8) sg.Value[11] ^= 1;                            // six bad signatures: quorum fails
            if (pi == 2 && id == 14) { signer = 70000; want = EdCommit::Inert; }             // Signer beyond the 16-bit column
            Vote vt = commitFrom(sender, signer, dig);
            vt.commit->Sig = ProtoSignature{signer, sg.Value, sg.Msg};
            if (pi == 0 && id == 15) { vt.commit->Sig.reset(); want = EdCommit::Inert; }     // no Signature
            Bytes wire = MarshalCommit(*vt.commit);
            std::optional<Vote> seen = vt;
            if (pi == 0 && id == 16) { wire.resize(wire.size() - 3); seen.reset(); want = EdCommit::Inert; }  // truncated on the wire
            all[pi].push_back({(uint16_t)sender, wire, seen, want});
        }
    }
    // the decoding rules
    size_t n_inert = 0, n_rejecting = 0;
    for (auto &votes : all)
        for (auto &w : votes) {
            CommitView c;
            uint8_t row[96], scheme = 0;
            uint32_t slot = 0;
            const EdCommit k = decode_mixed_commit(w.wire.data(), w.wire.size(), key_of, c, row, scheme, slot);
            CHECK(k == w.want);
            CHECK((k == EdCommit::Verify) == (slot != ED25519_NO_SLOT));
            if (k == EdCommit::Verify) {
                const MixedKey mk = key_of(c.Signer);
                CHECK(scheme == mk.scheme && (int)slot == mk.slot);
                if (scheme == SBV_ED25519) CHECK(c.value_len == 64 && memcmp(row, c.value, 64) == 0);
                if (scheme == SBV_P256) {
                    uint8_t r[32], s[32];
                    CHECK(parse_der_sig_span(c.value, c.value_len, r, s) && memcmp(row, r, 32) == 0 && memcmp(row + 32, s, 32) == 0);
                }
                if (scheme == SBV_P384) CHECK(std::any_of(row + 48, row + 96, [](uint8_t b) { return b != 0; }));
                if (scheme != SBV_P384) CHECK(std::all_of(row + 64, row + 96, [](uint8_t b) { return b == 0; }));
            } else {
                CHECK(std::all_of(row, row + 96, [](uint8_t b) { return b == 0; }));
            }
            n_inert += k == EdCommit::Inert;
            n_rejecting += k == EdCommit::Rejecting;
        }
    CHECK(n_inert == 3 && n_rejecting == 5);
    if (g_gpu) {
        sbv_engine *e = nullptr;
        CHECK(sbv_create(nullptr, 1, &e) == SBV_OK);
        if (!e) return;
        std::vector<uint64_t> ids(9);
        std::vector<uint8_t> curves(9), xy(9 * 96);
        for (uint64_t id = 1; id <= 9; id++) {
            ids[id - 1] = id;
            curves[id - 1] = id <= 7 ? SBV_P256 : SBV_P384;
            memcpy(&xy[96 * (id - 1)], ec[id].xy96, 96);
        }
        CHECK(sbv_set_keys(e, 1, 9, ids.data(), curves.data(), xy.data()) == SBV_OK);
        Bytes reg(7 * 32);
        for (uint64_t id = 10; id <= 16; id++) memcpy(&reg[32 * (id - 10)], ed[id].pub, 32);
        CHECK(sbv_ed25519_set_keys(e, 7, reg.data()) == SBV_OK);
        std::vector<uint8_t> okv, reached; std::vector<uint32_t> cnt;
        {
            CommitBatch batch(CommitBatch::Mixed);
            for (size_t pi = 0; pi < props3.size(); pi++) {
                batch.begin_instance(props3[pi].Digest(), 1);
                for (auto &w : all[pi]) batch.add_mixed_commit(w.sender, w.wire.data(), w.wire.size(), key_of);
            }
            CHECK(batch.size() == 45 && batch.instances() == 3 && batch.malformed().size() == 3 && batch.rejected().size() == 5);
            batch.verify_and_count(e, q - 1, okv, cnt, reached);
        }
        size_t i = 0;
        for (size_t pi = 0; pi < props3.size(); pi++) {
            VoteSet set(acceptCommits);
            int valid = 0;
            for (auto &w : all[pi]) {
                const size_t at = i++;
                bool sig_ok = false;
                if (w.seen && w.seen->commit->Sig) {
                    const ProtoSignature &ps = *w.seen->commit->Sig;
                    sig_ok = sig_valid(ps.Signer, ps.Value, ps.Msg);
                }
                CHECK(okv[at] == (w.want == EdCommit::Verify && sig_ok ? 1 : 0));  // inert and rejecting rows reject
                if (!w.seen || w.seen->sender == 1) continue;
                size_t before = set.votes().size();
                set.registerVote(w.seen->sender, *w.seen);
                if (set.votes().size() == before) continue;
                if (w.seen->commit->Digest == props3[pi].Digest() && sig_ok && w.want == EdCommit::Verify) valid++;
            }
            CHECK((int)cnt[pi] == valid);
            CHECK(reached[pi] == (valid >= q - 1 ? 1 : 0));
        }
        // instance 0: two bad signatures, two rejecting rows and two inert votes leave 9 < Q - 1; instance 1: a rejecting row,
        // a wrong digest, a foreign signer and an unknown signer leave 11; instance 2 as in TestEd25519CommitBatch
        CHECK(cnt[0] == 9 && cnt[1] == 11 && cnt[2] == 7);
        CHECK(reached[0] == 0 && reached[1] == 1 && reached[2] == 0);
        sbv_destroy(e);
    }
    for (auto &kv : ec) EC_KEY_free(kv.second.k);
    for (auto &kv : ed) EVP_PKEY_free(kv.second.k);
}

int main(int argc, char **argv) {
    std::string mode = argc > 1 ? argv[1] : "cpu";
    RUN(TestProposalDigestFixtures);
    RUN(TestGoldenDigests);
    RUN(TestWireCodecs);
    RUN(TestQuorum);
    RUN(TestBadPrepare);
    RUN(TestBadCommit);
    RUN(TestNormalPath);
    RUN(TestValidateLastDecision);
    RUN(TestVerifyPrevCommitSignatures);
    RUN(TestReqPoolPrune);
    RUN(TestControllerLeaderRequestHandling);
    RUN(TestAggregatorCoalesces);
    if (mode == "gpu") RUN(TestGpuVerifierEndToEnd);
    g_gpu = mode == "gpu";
    RUN(TestEd25519CommitBatch);
    RUN(TestMixedCommitBatch);
    printf("%d checks, %d failures\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
