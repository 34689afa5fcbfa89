// marshal.hpp — wire messages -> pinned SoA batches for the engine (north_star: "host code marshals incoming
// consensus-message and client-request signatures into pinned host batches").
//
//   Commit / Prepare / Signature wire codecs      /root/reference/smartbftprotos/messages.proto:41-58, 92-96
//   CommitBatch                                   the columns verifyVote + processCommits need
//                                                 (/root/reference/internal/bft/view.go:519-551, 827-849)
//
// A batch lives in PINNED host memory obtained from the engine (sbv_host_alloc), laid out exactly as the C ABI takes
// it: r[n][32], s[n][32], slot[n], msgs + msg_off[n+1] for sbv_hash_verify_registered, and instance / sender / signer /
// digest_match for the quorum stage.  Decoding a vote writes straight into those arrays — the DER signature is parsed
// into its r, s rows, Signature.Msg is appended to the message blob — so the engine DMAs from where the decoder wrote
// and no intermediate copy exists.
//
// An Ed25519 batch (CommitBatch::Ed25519) takes Commits whose Signature.Value is a raw 64-byte Ed25519 signature: the r and
// s columns together hold one 64-byte row (R || S) per vote, the slots index the engine's Ed25519 registry
// (sbv_ed25519_set_keys), and verify_and_count makes one sbv_ed25519_verify_quorum call.
//
// A mixed batch (CommitBatch::Mixed) takes Commits of a consenter set whose keys may be P-256, P-384 or Ed25519:
// key_of(signer) gives the signer's scheme and its slot of that scheme's registry, each vote gets a scheme tag and one
// 96-byte signature row (DER r, s parsed into r || s of the curve's width, or the raw R || S), and verify_and_count makes
// one sbv_mixed_verify_quorum call.
#pragma once
#include "verifier.hpp"
#include "callsites.hpp"

namespace sbft {

// ---- proto3 codecs (golang/protobuf field order and encodings) ----
namespace pb {
inline void bytes_field(Bytes &o, unsigned field, const uint8_t *p, size_t n) {
    varint(o, (uint64_t)field << 3 | 2); varint(o, n); o.insert(o.end(), p, p + n);
}
inline void u64_field(Bytes &o, unsigned field, uint64_t v) { if (v) { varint(o, (uint64_t)field << 3); varint(o, v); } }
}  // namespace pb

inline Bytes MarshalSignature(const ProtoSignature &s) {  // messages.proto:92-96
    Bytes o;
    pb::u64_field(o, 1, s.Signer);
    if (!s.Value.empty()) pb::bytes_field(o, 2, s.Value.data(), s.Value.size());
    if (!s.Msg.empty()) pb::bytes_field(o, 3, s.Msg.data(), s.Msg.size());
    return o;
}
inline Bytes MarshalCommit(const CommitMsg &c) {  // messages.proto:48-54
    Bytes o;
    pb::u64_field(o, 1, c.View);
    pb::u64_field(o, 2, c.Seq);
    if (!c.Digest.empty()) pb::bytes_field(o, 3, (const uint8_t *)c.Digest.data(), c.Digest.size());
    if (c.Sig) { Bytes s = MarshalSignature(*c.Sig); pb::bytes_field(o, 4, s.data(), s.size()); }
    if (c.Assist) { o.push_back(5 << 3); o.push_back(1); }
    return o;
}
inline Bytes MarshalPrepare(const PrepareMsg &p) {  // messages.proto:41-46
    Bytes o;
    pb::u64_field(o, 1, p.View);
    pb::u64_field(o, 2, p.Seq);
    if (!p.Digest.empty()) pb::bytes_field(o, 3, (const uint8_t *)p.Digest.data(), p.Digest.size());
    if (p.Assist) { o.push_back(4 << 3); o.push_back(1); }
    return o;
}

// A decoded Commit whose byte fields still point INTO the wire buffer (no copies).
struct CommitView {
    uint64_t View = 0, Seq = 0, Signer = 0;
    const uint8_t *digest = nullptr, *value = nullptr, *msg = nullptr;
    size_t digest_len = 0, value_len = 0, msg_len = 0;
    bool has_sig = false, Assist = false;
};
inline bool DecodeSignature(const uint8_t *p, const uint8_t *end, CommitView &out) {
    while (p < end) {
        uint64_t key, v;
        if (!pb::read_varint(p, end, key)) return false;
        const unsigned field = (unsigned)(key >> 3), wt = (unsigned)(key & 7);
        if (field == 0) return false;
        if (field == 1 && wt == 0) { if (!pb::read_varint(p, end, v)) return false; out.Signer = v; }
        else if ((field == 2 || field == 3) && wt == 2) {
            if (!pb::read_varint(p, end, v) || (uint64_t)(end - p) < v) return false;
            if (field == 2) { out.value = p; out.value_len = (size_t)v; } else { out.msg = p; out.msg_len = (size_t)v; }
            p += v;
        } else if (!pb::skip(p, end, wt)) return false;
    }
    return true;
}
inline bool DecodeCommit(const uint8_t *p, size_t n, CommitView &out) {
    out = CommitView();
    const uint8_t *end = p + n;
    while (p < end) {
        uint64_t key, v;
        if (!pb::read_varint(p, end, key)) return false;
        const unsigned field = (unsigned)(key >> 3), wt = (unsigned)(key & 7);
        if (field == 0) return false;
        if ((field == 1 || field == 2 || field == 5) && wt == 0) {
            if (!pb::read_varint(p, end, v)) return false;
            if (field == 1) out.View = v; else if (field == 2) out.Seq = v; else out.Assist = v != 0;
        } else if ((field == 3 || field == 4) && wt == 2) {
            if (!pb::read_varint(p, end, v) || (uint64_t)(end - p) < v) return false;
            if (field == 3) { out.digest = p; out.digest_len = (size_t)v; }
            else { out.has_sig = true; if (!DecodeSignature(p, p + v, out)) return false; }
            p += v;
        } else if (!pb::skip(p, end, wt)) return false;
    }
    return true;
}
inline bool DecodePrepare(const uint8_t *p, size_t n, PrepareMsg &out) {
    out = PrepareMsg();
    const uint8_t *end = p + n;
    while (p < end) {
        uint64_t key, v;
        if (!pb::read_varint(p, end, key)) return false;
        const unsigned field = (unsigned)(key >> 3), wt = (unsigned)(key & 7);
        if (field == 0) return false;
        if ((field == 1 || field == 2 || field == 4) && wt == 0) {
            if (!pb::read_varint(p, end, v)) return false;
            if (field == 1) out.View = v; else if (field == 2) out.Seq = v; else out.Assist = v != 0;
        } else if (field == 3 && wt == 2) {
            if (!pb::read_varint(p, end, v) || (uint64_t)(end - p) < v) return false;
            out.Digest.assign((const char *)p, (size_t)v);
            p += v;
        } else if (!pb::skip(p, end, wt)) return false;
    }
    return true;
}

// strict DER SEQUENCE{INTEGER r, INTEGER s} from a raw span, straight into two 32-byte rows
inline bool parse_der_sig_span(const uint8_t *sig, size_t n, uint8_t *r, uint8_t *s) {
    Bytes tmp(sig, sig + n);
    return parse_der_sig(tmp, r, s);
}

// How a wire Commit enters an Ed25519 batch, by the reference's registration rule (acceptCommits, view.go:161-171, then
// registerVote, util.go:130-143).  Only a Commit the reference would never register is Inert: undecodable bytes, no
// Signature, or a Signer that does not fit the 16-bit column.  Any other Commit is registered and burns its sender's
// slot; it is Rejecting when its Value is not exactly 64 bytes (crypto/ed25519.Verify rejects any other length) or its
// signer has no slot, and its row then carries ED25519_NO_SLOT, which rejects on the device.
enum class EdCommit { Inert, Rejecting, Verify };
constexpr uint32_t ED25519_NO_SLOT = 0xffffffffu;
template <class SlotOf>
inline EdCommit decode_ed25519_commit(const uint8_t *wire, size_t len, SlotOf &&slot_of, CommitView &c, uint32_t &slot) {
    slot = ED25519_NO_SLOT;
    if (!DecodeCommit(wire, len, c) || !c.has_sig || c.Signer > 0xffff) return EdCommit::Inert;
    const int s = slot_of(c.Signer);
    if (c.value_len != 64 || s < 0) return EdCommit::Rejecting;
    slot = (uint32_t)s;
    return EdCommit::Verify;
}

// Strict DER SEQUENCE{INTEGER r, INTEGER s} (crypto/ecdsa.VerifyASN1 rules) into r || s of width L each (32 for P-256,
// 48 for P-384), right-aligned.
inline bool parse_der_sig_width(const uint8_t *sig, size_t n, uint8_t *r, uint8_t *s, size_t L) {
    auto rd_int = [L](const uint8_t *&p, const uint8_t *end, uint8_t *out) {
        if (end - p < 2 || p[0] != 0x02) return false;
        size_t len = p[1];
        p += 2;
        if ((len & 0x80) || len == 0 || (size_t)(end - p) < len) return false;
        if (p[0] & 0x80) return false;
        if (len > 1 && p[0] == 0 && !(p[1] & 0x80)) return false;
        const uint8_t *v = p; size_t vl = len;
        if (vl > 1 && v[0] == 0) { v++; vl--; }
        if (vl > L) return false;
        memset(out, 0, L); memcpy(out + L - vl, v, vl);
        p += len;
        return true;
    };
    const uint8_t *p = sig, *end = sig + n;
    if (n < 2 || p[0] != 0x30) return false;
    size_t len;
    if (p[1] < 0x80) { len = p[1]; p += 2; }
    else if (p[1] == 0x81) { if (n < 3 || p[2] < 0x80) return false; len = p[2]; p += 3; }
    else return false;
    if ((size_t)(end - p) != len) return false;
    return rd_int(p, end, r) && rd_int(p, end, s) && p == end;
}

// A signer's key in a mixed consenter set: its scheme (SBV_P256, SBV_P384 or SBV_ED25519) and its slot of that
// scheme's registry (sbv_set_keys or sbv_ed25519_set_keys); slot < 0: the signer has no key.
struct MixedKey { uint8_t scheme; int slot; };

// How a wire Commit enters a mixed batch, by the same registration rule as decode_ed25519_commit: Inert for undecodable
// bytes, no Signature or a Signer beyond 16 bits; otherwise registered, and Rejecting when the signer has no key or its
// Value does not parse for the signer's scheme (strict DER for ECDSA, exactly 64 bytes for Ed25519).  row: the vote's
// 96-byte signature row, written for Verify and zeroed otherwise; scheme / slot: what the row is verified as (a rejecting
// or inert vote carries SBV_ED25519 or its signer's scheme and ED25519_NO_SLOT, which rejects on the device).
template <class KeyOf>
inline EdCommit decode_mixed_commit(const uint8_t *wire, size_t len, KeyOf &&key_of, CommitView &c, uint8_t *row, uint8_t &scheme, uint32_t &slot) {
    slot = ED25519_NO_SLOT;
    scheme = SBV_ED25519;
    memset(row, 0, 96);
    if (!DecodeCommit(wire, len, c) || !c.has_sig || c.Signer > 0xffff) return EdCommit::Inert;
    const MixedKey k = key_of(c.Signer);
    if (k.slot < 0 || k.scheme > SBV_ED25519) return EdCommit::Rejecting;
    scheme = k.scheme;
    bool parsed;
    if (k.scheme == SBV_ED25519) {
        parsed = c.value_len == 64;
        if (parsed) memcpy(row, c.value, 64);
    } else {
        const size_t L = k.scheme == SBV_P256 ? 32 : 48;
        parsed = parse_der_sig_width(c.value, c.value_len, row, row + L, L);
    }
    if (!parsed) { memset(row, 0, 96); return EdCommit::Rejecting; }
    slot = (uint32_t)k.slot;
    return EdCommit::Verify;
}

// One batch of commit votes (many instances = consensus sequences in flight, or many views during catch-up).
class CommitBatch {
  public:
    enum Scheme { EcdsaP256, Ed25519, Mixed };
    explicit CommitBatch(Scheme scheme = EcdsaP256) : ed25519_(scheme == Ed25519), mixed_(scheme == Mixed) {}
    size_t size() const { return n_; }
    size_t instances() const { return n_inst_; }
    void clear() { n_ = 0; msg_bytes_ = 0; n_inst_ = 0; malformed_.clear(); rejected_.clear(); }

    // Starts the votes of the next instance: `expected_digest` is proposal.Digest() (64 hex chars, view.go:524)
    // and `self` the local node id (its own vote never reaches the vote set).
    uint32_t begin_instance(const std::string &expected_digest, uint16_t self) {
        expected_ = expected_digest;
        self_.reserve((n_inst_ + 1) * 2, n_inst_ * 2);
        ((uint16_t *)self_.p)[n_inst_] = self;
        return (uint32_t)n_inst_++;
    }
    // Decodes one wire Commit received from `sender` and appends it to the current instance.  `slot_of(signer)` maps
    // the claimed signer to its slot of the engine's key registry (sbv_set_keys, or sbv_ed25519_set_keys for an Ed25519
    // batch), < 0 when unknown.  A mixed batch takes add_mixed_commit instead.
    // Malformed input never throws: the vote is recorded as one that cannot count (the reference drops such votes:
    // view.go:161-171, 839-842).  An Ed25519 batch follows decode_ed25519_commit instead.
    template <class SlotOf>
    void add_wire_commit(uint16_t sender, const uint8_t *wire, size_t len, SlotOf &&slot_of) {
        grow(n_ + 1);
        const size_t i = n_++;
        inst()[i] = (uint32_t)(n_inst_ - 1);
        snd()[i] = sender;
        CommitView c;
        if (ed25519_) {
            uint32_t slot = ED25519_NO_SLOT;
            const EdCommit k = n_inst_ > 0 ? decode_ed25519_commit(wire, len, slot_of, c, slot) : EdCommit::Inert;
            uint8_t *row = r() + 64 * i;
            slt()[i] = slot;
            if (k == EdCommit::Verify) memcpy(row, c.value, 64);
            else memset(row, 0, 64);
            if (k == EdCommit::Inert) {  // signer != sender keeps it out of the vote set
                sig()[i] = (uint16_t)(sender + 1); dm()[i] = 0;
                off()[i + 1] = msg_bytes_;
                malformed_.push_back(i);
                return;
            }
            if (k == EdCommit::Rejecting) rejected_.push_back(i);
            append_registered(i, c);
            return;
        }
        bool ok = n_inst_ > 0 && DecodeCommit(wire, len, c) && c.has_sig && c.Signer <= 0xffff;
        int slot = ok ? slot_of(c.Signer) : -1;
        ok = ok && slot >= 0 && parse_der_sig_span(c.value, c.value_len, r() + 32 * i, s() + 32 * i);
        if (!ok) {  // inert vote: signer != sender keeps it out of the vote set, r = s = 0 rejects on the device
            memset(r() + 32 * i, 0, 32); memset(s() + 32 * i, 0, 32);
            sig()[i] = (uint16_t)(sender + 1); slt()[i] = 0; dm()[i] = 0;
            off()[i + 1] = msg_bytes_;
            malformed_.push_back(i);
            return;
        }
        slt()[i] = (uint32_t)slot;
        append_registered(i, c);
    }
    // The same for a mixed batch (CommitBatch::Mixed only): key_of(signer) -> MixedKey gives the signer's scheme and slot, and
    // the vote follows decode_mixed_commit.
    template <class KeyOf>
    void add_mixed_commit(uint16_t sender, const uint8_t *wire, size_t len, KeyOf &&key_of) {
        grow(n_ + 1);
        const size_t i = n_++;
        inst()[i] = (uint32_t)(n_inst_ - 1);
        snd()[i] = sender;
        CommitView c;
        uint32_t slot = ED25519_NO_SLOT;
        uint8_t scheme = SBV_ED25519;
        uint8_t *row = rows_.p + 96 * i;
        EdCommit k = EdCommit::Inert;
        if (n_inst_ > 0) k = decode_mixed_commit(wire, len, key_of, c, row, scheme, slot);
        else memset(row, 0, 96);
        slt()[i] = slot;
        tags_.p[i] = scheme;
        if (k == EdCommit::Inert) {  // signer != sender keeps it out of the vote set
            sig()[i] = (uint16_t)(sender + 1); dm()[i] = 0;
            off()[i + 1] = msg_bytes_;
            malformed_.push_back(i);
            return;
        }
        if (k == EdCommit::Rejecting) rejected_.push_back(i);
        append_registered(i, c);
    }
    // Verifies every signature (SHA-256 of Signature.Msg on the device, registered keys) and counts the valid distinct
    // foreign votes per instance.  ok / count / reached are sized by the call.
    // An Ed25519 batch makes one sbv_ed25519_verify_quorum call (Signature.Msg hashed with SHA-512 on the device), a mixed
    // batch one sbv_mixed_verify_quorum call.
    void verify_and_count(sbv_engine *e, uint32_t threshold, std::vector<uint8_t> &ok, std::vector<uint32_t> &count, std::vector<uint8_t> &reached) {
        ok.assign(n_, 0); count.assign(n_inst_, 0); reached.assign(n_inst_, 0);
        if (n_ == 0 || n_inst_ == 0) return;
        if (mixed_) {
            if (sbv_mixed_verify_quorum(e, n_, tags_.p, msgs_.p, off(), slt(), rows_.p, inst(), snd(), sig(), dm(), n_inst_, (const uint16_t *)self_.p,
                                        threshold, ok.data(), count.data(), reached.data()) != SBV_OK)
                throw EngineFault(std::string("sbv_mixed_verify_quorum: ") + sbv_last_error(e));
            return;
        }
        if (ed25519_) {
            if (sbv_ed25519_verify_quorum(e, n_, msgs_.p, off(), slt(), r(), inst(), snd(), sig(), dm(), n_inst_, (const uint16_t *)self_.p, threshold,
                                          ok.data(), count.data(), reached.data()) != SBV_OK)
                throw EngineFault(std::string("sbv_ed25519_verify_quorum: ") + sbv_last_error(e));
            return;
        }
        if (sbv_hash_verify_registered(e, SBV_P256, n_, msgs_.p ? msgs_.p : (const uint8_t *)"", off(), slt(), r(), s(), ok.data()) != SBV_OK)
            throw EngineFault(std::string("sbv_hash_verify_registered: ") + sbv_last_error(e));
        if (sbv_quorum(e, n_, inst(), snd(), sig(), dm(), ok.data(), n_inst_, (const uint16_t *)self_.p, threshold, count.data(), reached.data()) != SBV_OK)
            throw EngineFault(std::string("sbv_quorum: ") + sbv_last_error(e));
    }
    const std::vector<size_t> &malformed() const { return malformed_; }
    const std::vector<size_t> &rejected() const { return rejected_; }  // Ed25519 / mixed: registered votes with a rejecting row
    const uint8_t *r_rows() const { return cols_.p; }
    const uint8_t *mixed_rows() const { return rows_.p; }    // mixed: the 96-byte signature rows
    const uint8_t *mixed_schemes() const { return tags_.p; }  // mixed: the scheme tag of every vote

  private:
    // signer, digest match and message of a vote that enters the vote set
    void append_registered(size_t i, const CommitView &c) {
        sig()[i] = (uint16_t)c.Signer;
        dm()[i] = (c.digest_len == expected_.size() && memcmp(c.digest, expected_.data(), c.digest_len) == 0) ? 1 : 0;
        msgs_.reserve(msg_bytes_ + c.msg_len + 16, msg_bytes_);
        if (c.msg_len) memcpy(msgs_.p + msg_bytes_, c.msg, c.msg_len);
        msg_bytes_ += c.msg_len;
        off()[i + 1] = msg_bytes_;
    }
    // column block (one pinned allocation): r, s, off, slot, instance, sender, signer, digest_match
    static constexpr size_t ROW = 32 + 32 + 8 + 4 + 4 + 2 + 2 + 1;
    void grow(size_t n) {
        if (n <= cap_) return;
        size_t nc = std::max(n, cap_ * 2 + 256);
        PinnedBuf nb;
        nb.reserve(nc * ROW + 64);
        auto at = [&](uint8_t *base, size_t capn, int k) {  // start of column k in a block sized for capn rows
            const size_t o[] = {0, 32 * capn, 64 * capn, 64 * capn + 8 * (capn + 1), 64 * capn + 8 * (capn + 1) + 4 * capn,
                                64 * capn + 8 * (capn + 1) + 8 * capn, 64 * capn + 8 * (capn + 1) + 10 * capn, 64 * capn + 8 * (capn + 1) + 12 * capn};
            return base + o[k];
        };
        const size_t w[] = {ed25519_ ? (size_t)64 : 32, ed25519_ ? (size_t)0 : 32, 8, 4, 4, 2, 2, 1};  // Ed25519: one 64-byte row over r and s
        if (cols_.p)
            for (int k = 0; k < 8; k++) memcpy(at(nb.p, nc, k), at(cols_.p, cap_, k), w[k] * (n_ + (k == 2 ? 1 : 0)));
        else
            memset(at(nb.p, nc, 2), 0, 8);
        std::swap(cols_.p, nb.p); std::swap(cols_.cap, nb.cap);
        if (mixed_) {  // the signature rows and scheme tags of a mixed batch live beside the column block
            rows_.reserve(nc * 96, n_ * 96);
            tags_.reserve(nc, n_);
        }
        cap_ = nc;
    }
    uint8_t *col(int k) const {
        const size_t c = cap_;
        const size_t o[] = {0, 32 * c, 64 * c, 64 * c + 8 * (c + 1), 64 * c + 8 * (c + 1) + 4 * c, 64 * c + 8 * (c + 1) + 8 * c,
                            64 * c + 8 * (c + 1) + 10 * c, 64 * c + 8 * (c + 1) + 12 * c};
        return cols_.p + o[k];
    }
    uint8_t *r() const { return col(0); }
    uint8_t *s() const { return col(1); }
    uint64_t *off() const { return (uint64_t *)col(2); }
    uint32_t *slt() const { return (uint32_t *)col(3); }
    uint32_t *inst() const { return (uint32_t *)col(4); }
    uint16_t *snd() const { return (uint16_t *)col(5); }
    uint16_t *sig() const { return (uint16_t *)col(6); }
    uint8_t *dm() const { return col(7); }

    PinnedBuf cols_, msgs_, self_, rows_, tags_;
    size_t cap_ = 0, n_ = 0, msg_bytes_ = 0, n_inst_ = 0;
    std::string expected_;
    std::vector<size_t> malformed_, rejected_;
    bool ed25519_ = false, mixed_ = false;
};

}  // namespace sbft
