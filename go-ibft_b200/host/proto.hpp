// proto.hpp -- host-side mirror of go-ibft's wire schema (reference messages/proto/messages.proto:7-110) and of
// IbftMessage.PayloadNoSig (reference messages/proto/helper.go:13-27).
//
// The reference is Go; no Go toolchain exists in the build image, so the host side above the C ABI is C++ with the same
// names and semantics (INTEGRATION.md shows the Go/cgo binding a maintainer would add).  Encoding follows protobuf-go
// v1.28.1 for this schema: fields in field-number order, zero scalars / empty bytes omitted, nil sub-messages omitted,
// present-but-empty sub-messages as `tag 00`, the set oneof member always emitted.  Checked byte-for-byte against wire
// bytes produced from the reference's own descriptor (tests/golden/proto_wire.json).
#pragma once
#include <cstdint>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

namespace ibft::host {

using Bytes = std::string;  // arbitrary bytes; like Go's string(key) it is directly usable as a map key

enum MessageType : uint32_t { PREPREPARE = 0, PREPARE = 1, COMMIT = 2, ROUND_CHANGE = 3 };  // messages.proto:7-12

struct View {  // messages.proto:15-21
  uint64_t height = 0, round = 0;
};
struct Proposal {  // messages.proto:104-110
  Bytes raw_proposal;
  uint64_t round = 0;
};
struct IbftMessage;
using MessagePtr = std::shared_ptr<IbftMessage>;

struct PreparedCertificate {  // messages.proto:87-94
  MessagePtr proposal_message;                 // nullptr == Go nil
  std::vector<MessagePtr> prepare_messages;    // empty == Go nil slice (indistinguishable on the wire)
};
struct RoundChangeCertificate {  // messages.proto:98-101
  std::vector<MessagePtr> round_change_messages;
};
struct PrePrepareMessage {  // messages.proto:47-57
  std::shared_ptr<Proposal> proposal;
  Bytes proposal_hash;
  std::shared_ptr<RoundChangeCertificate> certificate;
};
struct PrepareMessage {  // messages.proto:60-63
  Bytes proposal_hash;
};
struct CommitMessage {  // messages.proto:66-72
  Bytes proposal_hash, committed_seal;
};
struct RoundChangeMessage {  // messages.proto:75-83
  std::shared_ptr<Proposal> last_prepared_proposal;
  std::shared_ptr<PreparedCertificate> latest_prepared_certificate;
};

enum PayloadKind : uint8_t { PAYLOAD_NONE = 0, PAYLOAD_PREPREPARE = 5, PAYLOAD_PREPARE = 6, PAYLOAD_COMMIT = 7, PAYLOAD_ROUND_CHANGE = 8 };

struct IbftMessage {  // messages.proto:24-44
  std::shared_ptr<View> view;  // nullptr == nil view
  Bytes from, signature;
  uint32_t type = PREPREPARE;  // an int32 enum in protobuf-go: the bit pattern of int32(varint); encoded sign-extended
  PayloadKind payload_kind = PAYLOAD_NONE;  // which oneof member is set (independent of `type`, as in Go)
  // Where this message sits in the gossip frame it was decoded from: [wire_off, wire_off + wire_len) of *root_wire.  Set for the
  // top-level message AND for every message nested in its certificates (they share the root's bytes), so that the GPU verifier can
  // submit any of them as a raw-frame span without re-marshalling (IBFT_KIND_WIRE).  nullptr for messages built in memory.
  std::shared_ptr<const Bytes> root_wire;
  uint32_t wire_off = 0, wire_len = 0;
  bool has_wire() const { return root_wire != nullptr && wire_len != 0; }
  const char* wire_data() const { return root_wire->data() + wire_off; }
  PrePrepareMessage preprepare;
  PrepareMessage prepare;
  CommitMessage commit;
  RoundChangeMessage round_change;
};

struct DecodeError : std::runtime_error {
  using std::runtime_error::runtime_error;
};

// ----------------------------------------------------------------------------------------------- encoder
namespace wire {
inline void varint(Bytes& o, uint64_t v) {
  while (v >= 0x80) {
    o.push_back((char)(v | 0x80));
    v >>= 7;
  }
  o.push_back((char)v);
}
inline void f_varint(Bytes& o, uint32_t num, uint64_t v) {
  if (v == 0) return;
  varint(o, (uint64_t)num << 3);
  varint(o, v);
}
inline void f_bytes(Bytes& o, uint32_t num, const Bytes& b) {
  if (b.empty()) return;
  varint(o, ((uint64_t)num << 3) | 2);
  varint(o, b.size());
  o += b;
}
inline void f_msg(Bytes& o, uint32_t num, const Bytes& body) {  // present (possibly empty) sub-message
  varint(o, ((uint64_t)num << 3) | 2);
  varint(o, body.size());
  o += body;
}
}  // namespace wire

Bytes encode_message(const IbftMessage& m, bool with_signature = true);

inline Bytes encode_proposal(const Proposal& p) {
  Bytes o;
  wire::f_bytes(o, 1, p.raw_proposal);
  wire::f_varint(o, 2, p.round);
  return o;
}
inline Bytes encode_pc(const PreparedCertificate& pc) {
  Bytes o;
  if (pc.proposal_message) wire::f_msg(o, 1, encode_message(*pc.proposal_message));
  for (const auto& m : pc.prepare_messages) wire::f_msg(o, 2, m ? encode_message(*m) : Bytes());
  return o;
}
inline Bytes encode_rcc(const RoundChangeCertificate& r) {
  Bytes o;
  for (const auto& m : r.round_change_messages) wire::f_msg(o, 1, m ? encode_message(*m) : Bytes());
  return o;
}

inline Bytes encode_message(const IbftMessage& m, bool with_signature) {
  Bytes o;
  if (m.view) {
    Bytes v;
    wire::f_varint(v, 1, m.view->height);
    wire::f_varint(v, 2, m.view->round);
    wire::f_msg(o, 1, v);
  }
  wire::f_bytes(o, 2, m.from);
  if (with_signature) wire::f_bytes(o, 3, m.signature);
  wire::f_varint(o, 4, (uint64_t)(int64_t)(int32_t)m.type);  // protobuf-go: uint64(int64(int32 enum)), 10 bytes when negative
  switch (m.payload_kind) {
    case PAYLOAD_PREPREPARE: {
      Bytes b;
      if (m.preprepare.proposal) wire::f_msg(b, 1, encode_proposal(*m.preprepare.proposal));
      wire::f_bytes(b, 2, m.preprepare.proposal_hash);
      if (m.preprepare.certificate) wire::f_msg(b, 3, encode_rcc(*m.preprepare.certificate));
      wire::f_msg(o, 5, b);
      break;
    }
    case PAYLOAD_PREPARE: {
      Bytes b;
      wire::f_bytes(b, 1, m.prepare.proposal_hash);
      wire::f_msg(o, 6, b);
      break;
    }
    case PAYLOAD_COMMIT: {
      Bytes b;
      wire::f_bytes(b, 1, m.commit.proposal_hash);
      wire::f_bytes(b, 2, m.commit.committed_seal);
      wire::f_msg(o, 7, b);
      break;
    }
    case PAYLOAD_ROUND_CHANGE: {
      Bytes b;
      if (m.round_change.last_prepared_proposal) wire::f_msg(b, 1, encode_proposal(*m.round_change.last_prepared_proposal));
      if (m.round_change.latest_prepared_certificate) wire::f_msg(b, 2, encode_pc(*m.round_change.latest_prepared_certificate));
      wire::f_msg(o, 8, b);
      break;
    }
    default: break;
  }
  return o;
}

// messages/proto/helper.go:13-27: clone, Signature = nil, proto.Marshal -- the bytes that are hashed and signed
inline Bytes payload_no_sig(const IbftMessage& m) { return encode_message(m, false); }

// ----------------------------------------------------------------------------------------------- decoder
namespace wire {
// Nesting bound of the decoder.  A valid frame nests at most 4 messages deep (PREPREPARE -> RoundChangeCertificate ->
// ROUND_CHANGE -> PreparedCertificate -> PREPARE); decoding runs BEFORE any signature check, so an unauthenticated peer must
// not be able to exhaust the native stack with a few hundred KB of nested wrappers (protobuf-go caps recursion at 10,000 on
// growable stacks; a C++ frame is not growable).  Every sub-reader inherits depth + 1; decode_message refuses depth > kMaxDepth.
constexpr int kMaxDepth = 32;
struct Reader {
  const uint8_t* p;
  const uint8_t* end;
  int depth = 0;
  const std::shared_ptr<const Bytes>* root = nullptr;  // the frame being decoded (sub-readers inherit it): messages record their span
  bool done() const { return p >= end; }
  uint64_t varint() {
    uint64_t v = 0;
    int shift = 0;
    for (;;) {
      if (p >= end || shift > 63) throw DecodeError("truncated/overlong varint");
      uint8_t b = *p++;
      // protowire.ConsumeVarint: the 10th byte holds bit 63 only; anything above 1 overflows 64 bits
      if (shift == 63 && b > 1) throw DecodeError("variable length integer overflow");
      v |= (uint64_t)(b & 0x7F) << shift;
      shift += 7;
      if (!(b & 0x80)) return v;
    }
  }
  // returns false at end; otherwise field number, wire type and (for wt 0) value or (wt 2) the slice
  bool next(uint32_t& num, uint32_t& wt, uint64_t& val, Reader& sub) {
    if (done()) return false;
    uint64_t key = varint();
    num = (uint32_t)(key >> 3);
    wt = (uint32_t)(key & 7);
    if (num == 0 || (key >> 3) > 0x1FFFFFFFull) throw DecodeError("invalid field number");
    switch (wt) {
      case 0: val = varint(); break;
      case 3: skip_group(num, 0); break;  // a (deprecated) group: an unknown field to every message of this schema
      case 2: {
        uint64_t n = varint();
        if (n > (uint64_t)(end - p)) throw DecodeError("truncated bytes");
        sub = Reader{p, p + n, depth + 1, root};
        if (sub.depth > kMaxDepth) throw DecodeError("message nesting too deep");
        p += n;
        break;
      }
      case 1:
        if (end - p < 8) throw DecodeError("truncated fixed64");
        p += 8;
        break;
      case 5:
        if (end - p < 4) throw DecodeError("truncated fixed32");
        p += 4;
        break;
      default: throw DecodeError("unsupported wire type");
    }
    return true;
  }
  // moves past the END_GROUP tag that matches `number` (nested groups allowed)
  void skip_group(uint32_t number, int gdepth) {
    if (gdepth > kMaxDepth) throw DecodeError("group nesting too deep");
    for (;;) {
      uint64_t key = varint();
      uint32_t num = (uint32_t)(key >> 3), wt = (uint32_t)(key & 7);
      if (num == 0 || (key >> 3) > 0x1FFFFFFFull) throw DecodeError("invalid field number");
      if (wt == 4) {
        if (num != number) throw DecodeError("mismatched end group");
        return;
      }
      switch (wt) {
        case 0: varint(); break;
        case 1: if (end - p < 8) throw DecodeError("truncated fixed64"); p += 8; break;
        case 5: if (end - p < 4) throw DecodeError("truncated fixed32"); p += 4; break;
        case 2: {
          uint64_t n = varint();
          if (n > (uint64_t)(end - p)) throw DecodeError("truncated bytes");
          p += n;
          break;
        }
        case 3: skip_group(num, gdepth + 1); break;
        default: throw DecodeError("invalid wire type");
      }
    }
  }
  Bytes bytes() const { return Bytes((const char*)p, (size_t)(end - p)); }
};
}  // namespace wire

// The typed decoders MERGE the way protobuf-go's Unmarshal does, so that the model a frame decodes to is the one a Go node holds:
// a singular scalar / bytes field that appears again overwrites, a singular sub-message that appears again is merged field by
// field, repeated sub-messages accumulate, a different oneof member replaces the one set before (the same member again merges),
// and a known field with the wrong wire type is an unknown field (ignored by the model; kept by remarshal() below).
void decode_message_into(IbftMessage& m, wire::Reader r);
inline MessagePtr decode_message(wire::Reader r) {
  auto m = std::make_shared<IbftMessage>();
  if (r.root && *r.root) {
    m->root_wire = *r.root;
    m->wire_off = (uint32_t)(r.p - (const uint8_t*)(*r.root)->data());
    m->wire_len = (uint32_t)(r.end - r.p);
  }
  decode_message_into(*m, r);
  return m;
}
inline void decode_proposal_into(Proposal& p, wire::Reader r) {
  uint32_t num, wt;
  uint64_t val;
  wire::Reader sub{nullptr, nullptr, 0, nullptr};
  while (r.next(num, wt, val, sub)) {
    if (num == 1 && wt == 2) p.raw_proposal = sub.bytes();
    else if (num == 2 && wt == 0) p.round = val;
  }
}
inline void merge_message_field(MessagePtr& slot, wire::Reader sub) {
  if (!slot) {
    slot = decode_message(sub);
  } else {
    decode_message_into(*slot, sub);
    slot->root_wire = nullptr;  // assembled from two occurrences: there is no single span of the frame that IS this message
    slot->wire_off = slot->wire_len = 0;
  }
}
inline void decode_pc_into(PreparedCertificate& pc, wire::Reader r) {
  uint32_t num, wt;
  uint64_t val;
  wire::Reader sub{nullptr, nullptr, 0, nullptr};
  while (r.next(num, wt, val, sub)) {
    if (num == 1 && wt == 2) merge_message_field(pc.proposal_message, sub);
    else if (num == 2 && wt == 2) pc.prepare_messages.push_back(decode_message(sub));
  }
}
inline std::shared_ptr<PreparedCertificate> decode_pc(wire::Reader r) {
  auto pc = std::make_shared<PreparedCertificate>();
  decode_pc_into(*pc, r);
  return pc;
}
inline void decode_rcc_into(RoundChangeCertificate& c, wire::Reader r) {
  uint32_t num, wt;
  uint64_t val;
  wire::Reader sub{nullptr, nullptr, 0, nullptr};
  while (r.next(num, wt, val, sub))
    if (num == 1 && wt == 2) c.round_change_messages.push_back(decode_message(sub));
}

inline void decode_message_into(IbftMessage& mm, wire::Reader r) {
  IbftMessage* m = &mm;
  uint32_t num, wt;
  uint64_t val;
  wire::Reader sub{nullptr, nullptr, 0, nullptr};
  // a oneof member that differs from the one currently set starts from scratch; the same member again merges
  auto select = [&](PayloadKind k) {
    if (m->payload_kind != k) {
      m->preprepare = PrePrepareMessage();
      m->prepare = PrepareMessage();
      m->commit = CommitMessage();
      m->round_change = RoundChangeMessage();
      m->payload_kind = k;
    }
  };
  while (r.next(num, wt, val, sub)) {
    uint32_t n2, w2;
    uint64_t v2;
    wire::Reader s2{nullptr, nullptr, 0, nullptr};
    if (num == 1 && wt == 2) {
      if (!m->view) m->view = std::make_shared<View>();
      while (sub.next(n2, w2, v2, s2)) {
        if (n2 == 1 && w2 == 0) m->view->height = v2;
        else if (n2 == 2 && w2 == 0) m->view->round = v2;
      }
    } else if (num == 2 && wt == 2) {
      m->from = sub.bytes();
    } else if (num == 3 && wt == 2) {
      m->signature = sub.bytes();
    } else if (num == 4 && wt == 0) {
      m->type = (uint32_t)val;
    } else if (num == 5 && wt == 2) {
      select(PAYLOAD_PREPREPARE);
      while (sub.next(n2, w2, v2, s2)) {
        if (n2 == 1 && w2 == 2) {
          if (!m->preprepare.proposal) m->preprepare.proposal = std::make_shared<Proposal>();
          decode_proposal_into(*m->preprepare.proposal, s2);
        } else if (n2 == 2 && w2 == 2) {
          m->preprepare.proposal_hash = s2.bytes();
        } else if (n2 == 3 && w2 == 2) {
          if (!m->preprepare.certificate) m->preprepare.certificate = std::make_shared<RoundChangeCertificate>();
          decode_rcc_into(*m->preprepare.certificate, s2);
        }
      }
    } else if (num == 6 && wt == 2) {
      select(PAYLOAD_PREPARE);
      while (sub.next(n2, w2, v2, s2))
        if (n2 == 1 && w2 == 2) m->prepare.proposal_hash = s2.bytes();
    } else if (num == 7 && wt == 2) {
      select(PAYLOAD_COMMIT);
      while (sub.next(n2, w2, v2, s2)) {
        if (n2 == 1 && w2 == 2) m->commit.proposal_hash = s2.bytes();
        else if (n2 == 2 && w2 == 2) m->commit.committed_seal = s2.bytes();
      }
    } else if (num == 8 && wt == 2) {
      select(PAYLOAD_ROUND_CHANGE);
      while (sub.next(n2, w2, v2, s2)) {
        if (n2 == 1 && w2 == 2) {
          if (!m->round_change.last_prepared_proposal) m->round_change.last_prepared_proposal = std::make_shared<Proposal>();
          decode_proposal_into(*m->round_change.last_prepared_proposal, s2);
        } else if (n2 == 2 && w2 == 2) {
          if (!m->round_change.latest_prepared_certificate) m->round_change.latest_prepared_certificate = std::make_shared<PreparedCertificate>();
          decode_pc_into(*m->round_change.latest_prepared_certificate, s2);
        }
      }
    }
  }
}

inline MessagePtr decode_message(const uint8_t* data, size_t len) {
  auto root = std::make_shared<const Bytes>((const char*)data, len);
  const uint8_t* b = (const uint8_t*)root->data();
  return decode_message(wire::Reader{b, b + len, 0, &root});
}

// ----------------------------------------------------------------------------------------------- byte-exact re-marshal
// messages/proto/helper.go:13-27 is Clone + Signature = nil + proto.Marshal.  For a canonical frame that is the frame minus its
// signature TLV (what the device hashes).  For every OTHER parseable frame this restates protobuf-go's parse + marshal on a
// generic field tree (same rules as the typed decoder above, plus: unknown fields -- unknown numbers, wrong wire types, groups --
// are kept verbatim and re-emitted after the message's known fields), so that a GPU-backed node and a Go node hash the same
// bytes whatever a Byzantine validator signed.  Twin of oracle/ibft_proto.py remarshal(); checked against google.protobuf
// driven by the reference's descriptor (tests/golden/proto_wire.json "noncanonical").
namespace wire {
enum TreeType : uint8_t { T_IBFT = 0, T_VIEW, T_PREPREPARE, T_PREPARE, T_COMMIT, T_ROUND_CHANGE, T_PROPOSAL, T_RCC, T_PC };
// 0 unknown, 1 varint, 2 bytes, 3 sub-message, 4 repeated sub-message, 5 oneof member (sub-message); *sub = its type
inline int tree_field_kind(TreeType t, uint32_t f, TreeType* sub) {
  switch (t) {
    case T_IBFT:
      switch (f) {
        case 1: *sub = T_VIEW; return 3;
        case 2: case 3: return 2;
        case 4: return 1;
        case 5: *sub = T_PREPREPARE; return 5;
        case 6: *sub = T_PREPARE; return 5;
        case 7: *sub = T_COMMIT; return 5;
        case 8: *sub = T_ROUND_CHANGE; return 5;
        default: return 0;
      }
    case T_VIEW: return (f == 1 || f == 2) ? 1 : 0;
    case T_PREPREPARE:
      if (f == 1) { *sub = T_PROPOSAL; return 3; }
      if (f == 2) return 2;
      if (f == 3) { *sub = T_RCC; return 3; }
      return 0;
    case T_PREPARE: return f == 1 ? 2 : 0;
    case T_COMMIT: return (f == 1 || f == 2) ? 2 : 0;
    case T_ROUND_CHANGE:
      if (f == 1) { *sub = T_PROPOSAL; return 3; }
      if (f == 2) { *sub = T_PC; return 3; }
      return 0;
    case T_PROPOSAL: return f == 1 ? 2 : f == 2 ? 1 : 0;
    case T_RCC:
      if (f == 1) { *sub = T_IBFT; return 4; }
      return 0;
    case T_PC:
      if (f == 1) { *sub = T_IBFT; return 3; }
      if (f == 2) { *sub = T_IBFT; return 4; }
      return 0;
  }
  return 0;
}
struct TreeNode {
  struct Field {
    int kind = 0;
    uint64_t scalar = 0;
    Bytes bytes;
    std::vector<std::unique_ptr<TreeNode>> subs;  // one element for a singular sub-message
  };
  std::map<uint32_t, Field> fields;
  Bytes unknown;
};
inline void tree_parse_into(TreeNode& node, TreeType type, Reader r) {
  while (!r.done()) {
    const uint8_t* start = r.p;
    uint32_t num, wt;
    uint64_t val = 0;
    Reader sub{nullptr, nullptr, 0, nullptr};
    r.next(num, wt, val, sub);
    TreeType st = T_IBFT;
    int kind = tree_field_kind(type, num, &st);
    const uint32_t want = kind == 1 ? 0u : 2u;
    if (kind == 0 || wt != want) {
      node.unknown.append((const char*)start, (size_t)(r.p - start));
      continue;
    }
    if (kind == 5)  // a different oneof member replaces the one set before
      for (uint32_t other = 5; other <= 8; other++)
        if (other != num) node.fields.erase(other);
    TreeNode::Field& f = node.fields[num];
    f.kind = kind;
    if (kind == 1) f.scalar = (type == T_IBFT && num == 4) ? (uint64_t)(int64_t)(int32_t)val : val;  // the enum `type` is int32
    else if (kind == 2) f.bytes = sub.bytes();
    else if (kind == 4) {
      f.subs.push_back(std::make_unique<TreeNode>());
      tree_parse_into(*f.subs.back(), st, sub);
    } else {
      if (f.subs.empty()) f.subs.push_back(std::make_unique<TreeNode>());
      tree_parse_into(*f.subs[0], st, sub);  // a second occurrence merges into the first
    }
  }
}
inline Bytes tree_emit(const TreeNode& node, TreeType type, bool skip_signature) {
  Bytes o;
  for (auto& kv : node.fields) {
    const uint32_t num = kv.first;
    const TreeNode::Field& f = kv.second;
    if (skip_signature && type == T_IBFT && num == 3) continue;
    TreeType st = T_IBFT;
    tree_field_kind(type, num, &st);
    if (f.kind == 1) f_varint(o, num, f.scalar);
    else if (f.kind == 2) f_bytes(o, num, f.bytes);
    else
      for (auto& c : f.subs) f_msg(o, num, tree_emit(*c, st, false));
  }
  o += node.unknown;
  return o;
}
}  // namespace wire

// proto.Marshal(proto.Unmarshal(frame)), with the (known) signature field cleared first when !with_signature.  Throws DecodeError.
inline Bytes remarshal(const uint8_t* frame, size_t len, bool with_signature) {
  wire::TreeNode root;
  wire::tree_parse_into(root, wire::T_IBFT, wire::Reader{frame, frame + len, 0, nullptr});
  return wire::tree_emit(root, wire::T_IBFT, !with_signature);
}
// PayloadNoSig of a message: for one that was decoded from a frame, the re-marshal of exactly the bytes that arrived
inline Bytes payload_no_sig_exact(const IbftMessage& m) {
  if (m.has_wire()) return remarshal((const uint8_t*)m.wire_data(), m.wire_len, false);
  return payload_no_sig(m);
}

}  // namespace ibft::host
