// test_signer.hpp — TEST / BENCH INFRASTRUCTURE: an OpenSSL-backed signer (the reference's api.Signer,
// pkg/api/dependencies.go:46-52, is the application's job and is not part of the verification path)
// and a per-call CPU verifier used as the baseline arm of the n=4 simulator.  Never linked into libsbv.so.
#pragma once
#include <openssl/bn.h>
#include <openssl/ec.h>
#include <openssl/ecdsa.h>
#include <openssl/evp.h>
#include <openssl/obj_mac.h>

#include "callsites.hpp"

using namespace sbft;

struct TestKey { EC_KEY *k; uint8_t xy[64]; };
inline TestKey makeKey() {
    TestKey t;
    t.k = EC_KEY_new_by_curve_name(NID_X9_62_prime256v1);
    EC_KEY_generate_key(t.k);
    BIGNUM *x = BN_new(), *y = BN_new();
    EC_POINT_get_affine_coordinates(EC_KEY_get0_group(t.k), EC_KEY_get0_public_key(t.k), x, y, nullptr);
    BN_bn2binpad(x, t.xy, 32); BN_bn2binpad(y, t.xy + 32, 32);
    BN_free(x); BN_free(y);
    return t;
}
inline Bytes signDer(const TestKey &k, const Bytes &msg) {
    Bytes dig = sha256(msg);
    unsigned int len = ECDSA_size(k.k);
    Bytes sig(len);
    ECDSA_sign(0, dig.data(), 32, sig.data(), &len, k.k);
    sig.resize(len);
    return sig;
}
// Signer.SignProposal under the INTEGRATION.md convention: Msg = digest(prop) || aux
inline Signature signProposal(uint64_t id, const TestKey &k, const Proposal &p, const Bytes &aux) {
    Signature s; s.ID = id;
    s.Msg = p.DigestRaw(); s.Msg.insert(s.Msg.end(), aux.begin(), aux.end());
    s.Value = signDer(k, s.Msg);
    return s;
}


// An ECDSA key on P-256 (L = 32) or P-384 (L = 48); xy96 = X || Y in 48-byte slots, right-aligned, as sbv_set_keys takes
// them.  signDerEc: DER ECDSA over SHA-256(msg), as signDer.
struct TestEcKey { EC_KEY *k; uint8_t xy96[96]; };
inline TestEcKey makeEcKey(int L) {
    TestEcKey t{EC_KEY_new_by_curve_name(L == 32 ? NID_X9_62_prime256v1 : NID_secp384r1), {}};
    EC_KEY_generate_key(t.k);
    BIGNUM *x = BN_new(), *y = BN_new();
    EC_POINT_get_affine_coordinates(EC_KEY_get0_group(t.k), EC_KEY_get0_public_key(t.k), x, y, nullptr);
    BN_bn2binpad(x, t.xy96 + 48 - L, L); BN_bn2binpad(y, t.xy96 + 96 - L, L);
    BN_free(x); BN_free(y);
    return t;
}
inline Bytes signDerEc(EC_KEY *k, const Bytes &msg) {
    Bytes dig = sha256(msg);
    unsigned int len = ECDSA_size(k);
    Bytes sig(len);
    ECDSA_sign(0, dig.data(), 32, sig.data(), &len, k);
    sig.resize(len);
    return sig;
}

// Ed25519 consenter keys (OpenSSL EVP_PKEY_ED25519): Value = the raw 64-byte signature (R || S) over Signature.Msg.
struct TestEdKey { EVP_PKEY *k; uint8_t pub[32]; };
inline TestEdKey makeEdKey() {
    TestEdKey t{nullptr, {}};
    EVP_PKEY_CTX *ctx = EVP_PKEY_CTX_new_id(EVP_PKEY_ED25519, nullptr);
    EVP_PKEY_keygen_init(ctx);
    EVP_PKEY_keygen(ctx, &t.k);
    EVP_PKEY_CTX_free(ctx);
    size_t len = 32;
    EVP_PKEY_get_raw_public_key(t.k, t.pub, &len);
    return t;
}
inline Bytes signEd25519(const TestEdKey &k, const Bytes &msg) {
    Bytes sig(64);
    size_t len = 64;
    EVP_MD_CTX *ctx = EVP_MD_CTX_new();
    EVP_DigestSignInit(ctx, nullptr, nullptr, nullptr, k.k);
    EVP_DigestSign(ctx, sig.data(), &len, msg.data(), msg.size());
    EVP_MD_CTX_free(ctx);
    return sig;
}
// crypto/ed25519.Verify for the keys and signatures of the tests: a Value of any length other than 64 rejects
inline bool verifyEd25519(const uint8_t pub[32], const Bytes &sig, const Bytes &msg) {
    if (sig.size() != 64) return false;
    EVP_PKEY *k = EVP_PKEY_new_raw_public_key(EVP_PKEY_ED25519, nullptr, pub, 32);
    if (!k) return false;
    EVP_MD_CTX *ctx = EVP_MD_CTX_new();
    bool ok = EVP_DigestVerifyInit(ctx, nullptr, nullptr, nullptr, k) == 1 && EVP_DigestVerify(ctx, sig.data(), 64, msg.data(), msg.size()) == 1;
    EVP_MD_CTX_free(ctx);
    EVP_PKEY_free(k);
    return ok;
}
inline Signature signProposalEd25519(uint64_t id, const TestEdKey &k, const Proposal &p, const Bytes &aux) {
    Signature s; s.ID = id;
    s.Msg = p.DigestRaw(); s.Msg.insert(s.Msg.end(), aux.begin(), aux.end());
    s.Value = signEd25519(k, s.Msg);
    return s;
}

// One CPU ECDSA verification per call — the shape of a Go application calling crypto/ecdsa from
// VerifyConsenterSig / VerifyRequest (stand-in: OpenSSL ECDSA_verify; no Go toolchain here).
class CpuVerifier : public IVerifier {
  public:
    std::map<uint64_t, EC_KEY *> consenters;
    std::map<std::string, EC_KEY *> clients;
    uint64_t verSeq = 1;
    static bool check(EC_KEY *k, const Bytes &sig, const Bytes &msg) {
        Bytes dig = sha256(msg);
        return ECDSA_verify(0, dig.data(), 32, sig.data(), (int)sig.size(), k) == 1;
    }
    std::pair<Bytes, Error> VerifyConsenterSig(const Signature &sig, const Proposal &prop) override {
        Bytes d = prop.DigestRaw();
        if (sig.Msg.size() < 32 || memcmp(sig.Msg.data(), d.data(), 32)) return {Bytes(), Errorf("signature does not bind the proposal")};
        auto k = consenters.find(sig.ID);
        if (k == consenters.end() || !check(k->second, sig.Value, sig.Msg)) return {Bytes(), Errorf("invalid signature")};
        return {AuxiliaryData(sig.Msg), std::nullopt};
    }
    Error VerifySignature(const Signature &sig) override {
        auto k = consenters.find(sig.ID);
        if (k == consenters.end() || !check(k->second, sig.Value, sig.Msg)) return Errorf("invalid signature");
        return std::nullopt;
    }
    std::pair<RequestInfo, Error> VerifyRequest(const Bytes &val) override {
        ParsedRequest pr;
        if (!parse_request(val, pr)) return {RequestInfo(), Errorf("malformed request")};
        auto k = clients.find(pr.client);
        if (k == clients.end() || !check(k->second, pr.sig, pr.signedBytes)) return {RequestInfo(), Errorf("bad request signature")};
        return {RequestInfo{pr.client, pr.id}, std::nullopt};
    }
    std::pair<std::vector<RequestInfo>, Error> VerifyProposal(const Proposal &proposal) override {
        std::vector<Bytes> reqs; std::vector<RequestInfo> infos;
        if (!split_requests(proposal.Payload, reqs)) return {{}, Errorf("malformed proposal payload")};
        for (auto &r : reqs) { auto p = VerifyRequest(r); if (p.second) return {{}, p.second}; infos.push_back(p.first); }
        return {infos, std::nullopt};
    }
    uint64_t VerificationSequence() override { return verSeq; }
    std::vector<RequestInfo> RequestsFromProposal(const Proposal &) override { return {}; }
    Bytes AuxiliaryData(const Bytes &m) override { return m.size() >= 32 ? Bytes(m.begin() + 32, m.end()) : Bytes(); }
};

// naive_chain's verifier: accepts everything (examples/naive_chain/node.go:86-96)
class AcceptAllVerifier : public IVerifier {
  public:
    std::pair<std::vector<RequestInfo>, Error> VerifyProposal(const Proposal &) override { return {{}, std::nullopt}; }
    std::pair<RequestInfo, Error> VerifyRequest(const Bytes &) override { return {RequestInfo(), std::nullopt}; }
    std::pair<Bytes, Error> VerifyConsenterSig(const Signature &s, const Proposal &) override { return {AuxiliaryData(s.Msg), std::nullopt}; }
    Error VerifySignature(const Signature &) override { return std::nullopt; }
    uint64_t VerificationSequence() override { return 1; }
    std::vector<RequestInfo> RequestsFromProposal(const Proposal &) override { return {}; }
    Bytes AuxiliaryData(const Bytes &m) override { return m.size() >= 32 ? Bytes(m.begin() + 32, m.end()) : Bytes(); }
};
