// verify_core.cuh -- one signature check: (r, s, v, z) -> recovered signer address.
//
// This is the arithmetic behind core.Verifier.IsValidValidator (reference core/backend.go:41-45; callers
// core/ibft.go:735,1128,1213,1220) and core.Verifier.IsValidCommittedSeal (core/backend.go:53-55; caller
// core/ibft.go:943).  Conventions are those of SURVEY.md §8(c) and oracle/secp256k1.py: SEC 1 v2 §4.1.6 recovery
// with x = r only, 1 <= r,s < n, v in {0,1}, high-s accepted, address = Keccak-256(X||Y)[12:].
#pragma once
#include "../../include/ibft_verify.h"
#include "keccak.cuh"
#include "secp_ec.cuh"
#include "secp_modinv.cuh"
#include "sha256.cuh"

namespace ibft {

// modular inversions: safegcd divsteps by default, the Fermat ladders with -DIBFT_FERMAT (kept as a cross-check)
#if defined(IBFT_FERMAT)
#define IBFT_FE_INV fe_inv_fermat
#define IBFT_SC_INV sc_inv_fermat
#else
#define IBFT_FE_INV fe_inv_safegcd
#define IBFT_SC_INV sc_inv_safegcd
#endif

IBFT_HD fe fe_inv_for_table(const fe& a) { return IBFT_FE_INV(a); }

// digest of one item (kinds of include/ibft_verify.h).  Returns false for an unknown kind / out-of-range payload.
// want = false: only the structural checks (the chain warps of the split kernel never need z).
IBFT_HD bool item_digest(const ibft_sig_item& it, const uint8_t* arena, size_t arena_len, uint8_t* z, bool want = true) {
  switch (it.kind) {
    case IBFT_KIND_DIGEST:
#pragma unroll
      for (int i = 0; i < 32; i++) z[i] = it.digest[i];
      return true;
    case IBFT_KIND_PAYLOAD:
      if ((size_t)it.payload_off + it.payload_len > arena_len) return false;
      if (want) keccak256_bytes(arena + it.payload_off, it.payload_len, z);
      return true;
    case IBFT_KIND_PAYLOAD2: {
      uint64_t off2 = 0;
      uint32_t len2 = 0;
#pragma unroll
      for (int i = 0; i < 8; i++) off2 |= (uint64_t)it.digest[i] << (8 * i);
#pragma unroll
      for (int i = 0; i < 4; i++) len2 |= (uint32_t)it.digest[8 + i] << (8 * i);
      if ((size_t)it.payload_off + it.payload_len > arena_len || off2 > arena_len || (size_t)len2 > arena_len - off2) return false;
      if (want) keccak256_two_spans(arena + it.payload_off, it.payload_len, arena + off2, len2, z);
      return true;
    }
    case IBFT_KIND_SEAL: {
      // z = Keccak-256(proposalHash || 0x02), 0x02 = proto.MessageType_COMMIT (reference messages/proto/messages.proto:10)
      if (want) keccak256_commit_seal(it.digest, z);
      return true;
    }
    default:
      return false;
  }
}

// ------------------------------------------------------------------------------------------------------------
// Raw gossip frames (IBFT_KIND_WIRE / IBFT_KIND_WIRE_SEAL): top-level parse of a proto3 IbftMessage
// (reference messages/proto/messages.proto:24-44) with a canonical-encoding check.  protobuf-go emits fields in
// field-number order, omits zero scalars / empty bytes and uses minimal varints; only for such a frame does
// "frame minus the signature TLV" equal PayloadNoSig (clone, Signature = nil, Marshal: messages/proto/helper.go:13-27).
// Anything else is handed back to the host (status NEEDS_HOST), never guessed.  All four message types are accepted: the signed
// bytes of a ROUND_CHANGE / PREPREPARE frame include its nested certificates, which are validated by the same walk.
// ------------------------------------------------------------------------------------------------------------
struct wire_frame {
  uint32_t from_off, from_len;      // value of field 2
  uint32_t sig_tag_off, sig_end;    // the whole field-3 TLV
  uint32_t sig_off, sig_len;        // its value
  uint32_t type;                    // field 4
  uint32_t payload_field;           // 0, 6 (prepareData) or 7 (commitData)
  uint32_t hash_off, hash_len;      // proposalHash inside the payload
  uint32_t seal_off, seal_len;      // committedSeal (commitData only)
  bool has_view;
};

// minimal encoding required.  The 10th byte carries only bit 63: protobuf-go's protowire.ConsumeVarint rejects a 10th byte
// above 1 ("variable length integer overflow"), so such a frame never decodes on a Go node and must not be accepted here.
IBFT_HD bool wire_varint(const uint8_t* w, uint32_t len, uint32_t& pos, uint64_t& v) {
  v = 0;
  for (int shift = 0; shift < 64; shift += 7) {
    if (pos >= len) return false;
    uint8_t b = w[pos++];
    if (shift == 63 && b > 1) return false;
    v |= (uint64_t)(b & 0x7F) << shift;
    if (!(b & 0x80)) return !(b == 0 && shift > 0);  // a trailing zero group is a non-minimal encoding
  }
  return false;
}
// LEN field: reads the length, returns the value span; empty values are non-canonical (proto3 omits them)
IBFT_HD bool wire_len(const uint8_t* w, uint32_t len, uint32_t& pos, uint32_t& off, uint32_t& n, bool allow_empty) {
  uint64_t l;
  if (!wire_varint(w, len, pos, l)) return false;
  if (l > (uint64_t)(len - pos)) return false;
  if (l == 0 && !allow_empty) return false;
  off = pos;
  n = (uint32_t)l;
  pos += n;
  return true;
}

// Schema-driven canonical walk of a COMPLETE IbftMessage frame, nested certificates included (messages.proto:24-110):
//   IbftMessage { View view = 1; bytes from = 2; bytes signature = 3; MessageType type = 4;
//                 oneof payload { PrePrepareMessage = 5; PrepareMessage = 6; CommitMessage = 7; RoundChangeMessage = 8 } }
//   PrePrepareMessage { Proposal proposal = 1; bytes proposalHash = 2; RoundChangeCertificate certificate = 3 }
//   RoundChangeMessage { Proposal lastPreparedProposal = 1; PreparedCertificate latestPreparedCertificate = 2 }
//   PreparedCertificate { IbftMessage proposalMessage = 1; repeated IbftMessage prepareMessages = 2 }
//   RoundChangeCertificate { repeated IbftMessage roundChangeMessages = 1 }      Proposal { bytes rawProposal = 1; uint64 round = 2 }
// "canonical" = what protobuf-go emits for the decoded value (decode + encode reproduces the bytes): fields in field-number
// order (repeated fields contiguous), minimal varints, zero scalars / empty bytes omitted, sub-messages may be present-but-
// empty, at most one oneof member.  The walk is iterative (an explicit stack of open sub-messages, depth <= IBFT_WIRE_MAX_DEPTH)
// because device code cannot recurse; a valid frame nests IbftMessage -> payload -> certificate -> IbftMessage -> payload ->
// certificate -> IbftMessage -> payload = 8 levels (PREPREPARE carrying ROUND_CHANGE messages carrying prepared certificates).
#define IBFT_WIRE_MAX_DEPTH 12
enum wire_msg_type : uint8_t { WT_IBFT = 0, WT_VIEW, WT_PREPREPARE, WT_PREPARE, WT_COMMIT, WT_ROUND_CHANGE, WT_PROPOSAL, WT_RCC, WT_PC };
// field kinds: 0 unknown, 1 varint (non-zero), 2 bytes (non-empty), 3 + t sub-message of type t; bit 7: repeated
IBFT_HD uint32_t wire_field_kind(uint32_t msg, uint32_t field) {
  switch (msg) {
    case WT_IBFT:
      switch (field) {
        case 1: return 3 + WT_VIEW;
        case 2: case 3: return 2;
        case 4: return 1;
        case 5: return 3 + WT_PREPREPARE;
        case 6: return 3 + WT_PREPARE;
        case 7: return 3 + WT_COMMIT;
        case 8: return 3 + WT_ROUND_CHANGE;
        default: return 0;
      }
    case WT_VIEW: return (field == 1 || field == 2) ? 1u : 0u;
    case WT_PREPREPARE: return field == 1 ? 3u + WT_PROPOSAL : field == 2 ? 2u : field == 3 ? 3u + WT_RCC : 0u;
    case WT_PREPARE: return field == 1 ? 2u : 0u;
    case WT_COMMIT: return (field == 1 || field == 2) ? 2u : 0u;
    case WT_ROUND_CHANGE: return field == 1 ? 3u + WT_PROPOSAL : field == 2 ? 3u + WT_PC : 0u;
    case WT_PROPOSAL: return field == 1 ? 2u : field == 2 ? 1u : 0u;
    case WT_RCC: return field == 1 ? (0x80u | (3u + WT_IBFT)) : 0u;
    case WT_PC: return field == 1 ? 3u + WT_IBFT : field == 2 ? (0x80u | (3u + WT_IBFT)) : 0u;
    default: return 0;
  }
}

// true: canonical frame, `f` describes its TOP-LEVEL message (From, the signature TLV, type, which payload member, and for a
// flat PREPARE / COMMIT payload the proposalHash / committedSeal spans).  false: hand back to the host.
IBFT_HD bool parse_wire_frame(const uint8_t* w, uint32_t len, wire_frame& f) {
  f.from_off = f.from_len = f.sig_off = f.sig_len = f.type = f.payload_field = 0;
  f.hash_off = f.hash_len = f.seal_off = f.seal_len = 0;
  f.has_view = false;
  f.sig_tag_off = f.sig_end = 0xFFFFFFFFu;
  uint32_t end_stack[IBFT_WIRE_MAX_DEPTH];
  uint8_t type_stack[IBFT_WIRE_MAX_DEPTH], last_stack[IBFT_WIRE_MAX_DEPTH];
  int depth = 0;
  end_stack[0] = len;
  type_stack[0] = WT_IBFT;
  last_stack[0] = 0;
  uint32_t pos = 0;
  for (;;) {
    while (depth > 0 && pos == end_stack[depth]) depth--;   // close finished sub-messages
    if (depth == 0 && pos == len) break;
    const uint32_t end = end_stack[depth], msg = type_stack[depth];
    const uint32_t tag_off = pos;
    uint64_t key;
    if (!wire_varint(w, end, pos, key) || (key >> 35)) return false;
    const uint32_t field = (uint32_t)(key >> 3), wt = (uint32_t)(key & 7);
    const uint32_t kind = wire_field_kind(msg, field);
    if (kind == 0) return false;  // unknown field (or field 0)
    const bool repeated = kind & 0x80u;
    const uint32_t k = kind & 0x7Fu;
    uint32_t last = last_stack[depth];
    if (msg == WT_IBFT && last >= 5 && field >= 5) return false;  // the oneof holds at most one member
    if (repeated ? field < last : field <= last) return false;   // field-number order; only repeated fields may repeat
    last_stack[depth] = (uint8_t)field;
    if (k == 1) {
      uint64_t v;
      if (wt != 0 || !wire_varint(w, end, pos, v) || v == 0) return false;  // zero scalars are omitted
      if (msg == WT_IBFT && field == 4) {
        // IbftMessage.type is an enum: protobuf-go holds int32(v) and re-encodes it sign-extended, so a value above 2^31 - 1 is
        // not what it would emit.  The canonical form of a NEGATIVE type (10 bytes, v >= 2^63) is handed back too: the host
        // decides it, which is always allowed.  Checked at every depth: nested certificate messages are part of the signed bytes.
        if (v > 0x7FFFFFFFull) return false;
        if (depth == 0) f.type = (uint32_t)v;
      }
      continue;
    }
    uint32_t off, n;
    if (wt != 2 || !wire_len(w, end, pos, off, n, k != 2)) return false;  // bytes fields are never empty; sub-messages may be
    if (k == 2) {
      if (depth == 0) {
        if (field == 2) { f.from_off = off; f.from_len = n; }
        else { f.sig_tag_off = tag_off; f.sig_end = pos; f.sig_off = off; f.sig_len = n; }
      } else if (depth == 1 && (msg == WT_PREPARE || msg == WT_COMMIT)) {
        if (field == 1) { f.hash_off = off; f.hash_len = n; }
        else { f.seal_off = off; f.seal_len = n; }
      }
      continue;
    }
    // sub-message: descend (its bytes are [off, off + n); wire_len already moved pos past them, so step back in)
    if (depth == 0) {
      if (field == 1) f.has_view = true;
      else f.payload_field = field;
    }
    if (depth + 1 >= IBFT_WIRE_MAX_DEPTH) return false;
    depth++;
    end_stack[depth] = off + n;
    type_stack[depth] = (uint8_t)(k - 3);
    last_stack[depth] = 0;
    pos = off;
  }
  if (f.sig_tag_off == 0xFFFFFFFFu) { f.sig_tag_off = f.sig_end = len; }  // no signature field: nothing to cut out
  return true;
}

// Everything ecrecover needs for one item, whatever its kind.  Returns IBFT_ITEM_OK or IBFT_ITEM_NEEDS_HOST; *valid is false when
// the item is structurally invalid (verdict 0 without any arithmetic).
struct resolved_item {
  uint8_t r[32], s[32], z[32], signer[20];
  uint8_t v;
};
IBFT_HD int resolve_item(const ibft_sig_item& it, const uint8_t* arena, size_t arena_len, resolved_item& o, bool* valid,
                         bool want_digest = true) {
  *valid = false;
  if (it.kind == IBFT_KIND_WIRE || it.kind == IBFT_KIND_WIRE_SEAL) {
    if ((size_t)it.payload_off + it.payload_len > arena_len) return IBFT_ITEM_OK;
    const uint8_t* w = arena + it.payload_off;
    wire_frame f;
    if (!parse_wire_frame(w, it.payload_len, f)) return IBFT_ITEM_NEEDS_HOST;
    if (f.from_len != 20) return IBFT_ITEM_OK;  // can never equal a recovered address
#pragma unroll
    for (int i = 0; i < 20; i++) o.signer[i] = w[f.from_off + i];
    if (it.kind == IBFT_KIND_WIRE) {
      // IsValidValidator (core/backend.go:41-45): needs a view (for the height) and a 65-byte signature
      if (!f.has_view || f.sig_len != 65) return IBFT_ITEM_OK;
#pragma unroll
      for (int i = 0; i < 32; i++) { o.r[i] = w[f.sig_off + i]; o.s[i] = w[f.sig_off + 32 + i]; }
      o.v = w[f.sig_off + 64];
      if (want_digest) keccak256_two_spans(w, f.sig_tag_off, w + f.sig_end, it.payload_len - f.sig_end, o.z);
    } else {
      // IsValidCommittedSeal on the frame: ExtractCommitHash needs type == COMMIT and commitData (messages/helpers.go:51-62),
      // the seal is commitData.committedSeal with Signer = From (:38-48)
      if (f.type != 2 || f.payload_field != 7 || f.hash_len != 32 || f.seal_len != 65) return IBFT_ITEM_OK;
      if (want_digest) keccak256_commit_seal(w + f.hash_off, o.z);
#pragma unroll
      for (int i = 0; i < 32; i++) { o.r[i] = w[f.seal_off + i]; o.s[i] = w[f.seal_off + 32 + i]; }
      o.v = w[f.seal_off + 64];
    }
    *valid = true;
    return IBFT_ITEM_OK;
  }
#pragma unroll
  for (int i = 0; i < 32; i++) { o.r[i] = it.r[i]; o.s[i] = it.s[i]; }
#pragma unroll
  for (int i = 0; i < 20; i++) o.signer[i] = it.signer[i];
  o.v = it.v;
  *valid = item_digest(it, arena, arena_len, o.z, want_digest);
  return IBFT_ITEM_OK;
}

// Executor dispatch of Q = u1*G + u2*R -> affine (false = point at infinity).  The throughput path keeps its hand-scheduled
// Jacobian routine (ecmult_double); exec_levels runs the level-structured XYZZ routine of the latency path one product at a
// time (host emulation: differential test of the level wiring); exec_quad runs it on four lanes.  T must hold
// IBFT_RTAB_WORDS words per signature for the serial path, IBFT_QTAB_WORDS for the level-structured one.
struct exec_levels : exec_serial {};
IBFT_HD bool ecmult_affine(const exec_serial&, const sc& u1, const sc& u2, const aff& R, const gtab_view& G, const rtab_view& T,
                           fe& qx, fe& qy) {
  jac Q = ecmult_double(u1, u2, R, G, T);
  IBFT_STAGE(8);
  if (Q.inf || fe_is_zero(Q.z)) return false;
  fe zi = IBFT_FE_INV(Q.z);
  fe zi2 = fe_sqr(zi);
  qx = fe_normalize(fe_mul(Q.x, zi2));
  qy = fe_normalize(fe_mul(Q.y, fe_mul(zi2, zi)));
  return true;
}
template <class EX>
IBFT_HD bool ecmult_affine_levels(const EX& ex, const sc& u1, const sc& u2, const aff& R, const gtab_view& G, const rtab_view& T,
                                  fe& qx, fe& qy) {
  xyzz Q = ecmult_double_x(ex, u1, u2, R, G, qtab_view{T.base, T.stride});
  IBFT_STAGE(8);
  if (Q.inf || fe_is_zero(Q.zzz)) return false;
  fe i3 = IBFT_FE_INV(Q.zzz);     // 1/Z^3
  fe zi = fe_mul(Q.zz, i3);       // Z^2 / Z^3 = 1/Z
  qx = fe_normalize(fe_mul(Q.x, fe_sqr(zi)));
  qy = fe_normalize(fe_mul(Q.y, i3));
  return true;
}
IBFT_HD bool ecmult_affine(const exec_levels& ex, const sc& u1, const sc& u2, const aff& R, const gtab_view& G, const rtab_view& T,
                           fe& qx, fe& qy) {
  return ecmult_affine_levels(ex, u1, u2, R, G, T, qx, qy);
}
#if defined(__CUDACC__)
__device__ __forceinline__ bool ecmult_affine(const exec_quad& ex, const sc& u1, const sc& u2, const aff& R, const gtab_view& G,
                                              const rtab_view& T, fe& qx, fe& qy) {
  return ecmult_affine_levels(ex, u1, u2, R, G, T, qx, qy);
}
#endif

// The public key Q = r^-1 (s R - z G) of an in-range (r, s, v): R = lift_x(r, v) by a square root, then u1 G + u2 R by the
// executor's ecmult_affine.  false: r is not an abscissa, or Q is the point at infinity.
template <class EX>
IBFT_HD bool recover_key(const EX& ex, const sc& r, const sc& s, uint8_t v, const uint8_t* z_be, const gtab_view& G,
                         const rtab_view& T, fe& qx, fe& qy) {
  // R = lift_x(r, v)   (r < n < p: always a canonical field element)
  fe x;
#pragma unroll
  for (int i = 0; i < 8; i++) x.v[i] = r.v[i];
  fe y2 = fe_add(fe_mul(fe_sqr(x), x), fe_from_u32(7));
  fe y = fe_sqrt_candidate(y2);
  if (!fe_equal(fe_sqr(y), y2)) return false;  // x^3 + 7 is a non-residue: r is not an abscissa
  y = fe_normalize(y);
  if ((y.v[0] & 1u) != (uint32_t)v) y = fe_normalize(fe_neg(y));
  aff R;
  R.x = x;
  R.y = y;
  IBFT_STAGE(2);
  // u1 = -z/r, u2 = s/r  (mod n)
  sc z = sc_reduce_once(sc_from_be(z_be));
  sc rinv = IBFT_SC_INV(r);
  sc u1 = sc_neg(sc_mul(z, rinv));
  sc u2 = sc_mul(s, rinv);
  IBFT_STAGE(3);
  return ecmult_affine(ex, u1, u2, R, G, T, qx, qy);
}

#if IBFT_WC > 0 && !defined(IBFT_RECOVER_TABLE_INV)
// ------------------------------------------------------------------------------------------------------------
// The one-thread recovery (exec_serial: k_recover and the key registry's worklist pass) without a field inversion.
// -DIBFT_RECOVER_TABLE_INV keeps the composition above (affine table by one inversion, generator streams inside the window
// loop, inversion of Z at the end) for A/B runs.
//   1. u2 * R on the isomorphic curve E': phi(R) = (x c, c^2), c = x^3 + 7 = y^2, needs no square root; the table {1..8} phi(R)
//      is made "effective affine" without an inversion (ecmult_build_rtable_globalz), and the window loop walks the R streams
//      only.  Its result (X, Y, Z) on E' with the table's Z_8 is the Jacobian point A = (X, Y, W0 y) of E, W0 = Z Z_8: y stays
//      unknown.
//   2. u1 * G by a comb, no doubling, into B = (Xb, Yb, Zb): the wide comb over u1's own digits when the engine holds it
//      (ecmult_gen_wide, at most 12 additions), else the per-position comb over u1's GLV split (ecmult_gen_comb, 17).
//   3. A + B (recover_final): Z_A^2 = W0^2 c needs no root, so H and V = W0 Zb H do not depend on y; ONE exponentiation of
//      c V^4 gives y = sqrt(c) and 1 / (y V) = 1 / Z3 (fe_sqrt_inv), then S2 and the rest of the addition use y.
// A = (X, Y, W0) is held with Z = W0 (the factor y kept apart); the rare cases are exact: A = +-B, u1 = 0, a non-residue c.
// ------------------------------------------------------------------------------------------------------------
IBFT_HD bool recover_affine(const fe& x, const fe& y, const fe& zi, fe& qx, fe& qy) {
  const fe zi2 = fe_sqr(zi);
  qx = fe_normalize(fe_mul(x, zi2));
  qy = fe_normalize(fe_mul(y, fe_mul(zi2, zi)));
  return true;
}
// y = sqrt(c) with parity v and w = 1 / (y V); false when c is a non-residue
IBFT_HD bool recover_root(const fe& c, const fe& V, uint8_t v, fe& y, fe& w) {
  const fe_root_inv o = fe_sqrt_inv(c, V);
  if (!fe_equal(fe_sqr(o.y), c)) {
    IBFT_BRANCH(IBFT_BR_REC_NONRES);
    return false;
  }
  y = fe_normalize(o.y);
  w = o.w;
  if ((y.v[0] & 1u) != (uint32_t)v) {
    y = fe_normalize(fe_neg(y));
    w = fe_neg(w);
  }
  return true;
}
IBFT_HD bool recover_final(const jac& A, const fe& c, uint8_t v, const jac& B, fe& qx, fe& qy) {
  IBFT_OPCOUNT(IBFT_OP_REC_FINAL);
  fe y, w;
  if (B.inf) {  // u1 = 0: Q = A, Z_A = W0 y
    IBFT_BRANCH(IBFT_BR_REC_B_INF);
    if (A.inf || !recover_root(c, A.z, v, y, w)) return false;
    return recover_affine(A.x, A.y, w, qx, qy);
  }
  if (A.inf) {  // u2 R is never infinity (0 < u2 < n); Q = B, and c must still be a residue
    if (!recover_root(c, B.z, v, y, w)) return false;
    return recover_affine(B.x, B.y, fe_mul(y, w), qx, qy);  // 1 / Zb = y / (y Zb)
  }
  // add-1998-cmo-2 with Z1 = W0 y, Z2 = Zb: Z1Z1 = W0^2 c, S2 = Yb Z1 Z1Z1 = y (Yb W0 Z1Z1), Z3 = Z1 Z2 H = y V
  const fe z1z1 = fe_mul(fe_sqr(A.z), c);
  const fe z2z2 = fe_sqr(B.z);
  const fe u1 = fe_mul(A.x, z2z2);
  const fe h = fe_sub(fe_mul(B.x, z1z1), u1);
  const fe s1 = fe_mul(A.y, fe_mul(B.z, z2z2));
  const fe t2 = fe_mul(B.y, fe_mul(A.z, z1z1));  // S2 / y
  if (fe_is_zero(h)) {  // A = +-B (crafted signatures only): y first, then the sign of S2 - S1 decides
    if (!recover_root(c, A.z, v, y, w)) return false;
    if (!fe_is_zero(fe_sub(fe_mul(t2, y), s1))) {
      IBFT_BRANCH(IBFT_BR_REC_NEG);
      return false;  // A = -B: Q is the point at infinity
    }
    IBFT_BRANCH(IBFT_BR_REC_DBL);
    jac P = A;
    P.z = fe_mul(A.z, y);
    const jac D = jac_double(P);
    if (!recover_root(c, D.z, v, y, w)) return false;
    return recover_affine(D.x, D.y, fe_mul(y, w), qx, qy);
  }
  const fe V = fe_mul(fe_mul(A.z, B.z), h);
  if (!recover_root(c, V, v, y, w)) return false;
  const fe rr = fe_sub(fe_mul(t2, y), s1);
  const fe hh = fe_sqr(h);
  const fe hhh = fe_mul(h, hh);
  const fe vv = fe_mul(u1, hh);
  const fe x3 = fe_sub(fe_sub(fe_sqr(rr), hhh), fe_dbl(vv));
  const fe y3 = fe_sub(fe_mul(rr, fe_sub(vv, x3)), fe_mul(s1, hhh));
  return recover_affine(x3, y3, w, qx, qy);
}

// WIDE: u1*G by the wide comb, else by the per-position comb.  Each kernel instantiation holds only one of the two loops (the
// engine launches the wide one when it holds the table): with both behind a run-time branch the kernel ran 0.7 % slower on an H100.
template <bool WIDE>
IBFT_HD bool recover_key_serial(const sc& r, const sc& s, uint8_t v, const uint8_t* z_be, const gtab_view& G, const rtab_view& T,
                                fe& qx, fe& qy) {
  // u1 = -z/r, u2 = s/r  (mod n)
  sc z = sc_reduce_once(sc_from_be(z_be));
  sc rinv = IBFT_SC_INV(r);
  ecmult_digits dg;
  ecmult_split_into(sc_mul(s, rinv), dg, 0);
  const sc u1 = sc_neg(sc_mul(z, rinv));
#if IBFT_GEN_WIDE > 0
  if (WIDE) {
    ecmult_wide_into(u1, dg);
    // the 12 gathers out of 1.38 GiB start here, a whole window loop before the comb reads them (they are prefetched again
    // right before it, in case L2 let them go): +0.5 % on an H100 over prefetching only before the comb
    ecmult_gen_wide_prefetch(dg, G);
  } else
#endif
    ecmult_split_into(u1, dg, 2);
  IBFT_STAGE(3);
  // phi(R) on E' and its inversion-free table; c = x^3 + 7
  fe x;
#pragma unroll
  for (int i = 0; i < 8; i++) x.v[i] = r.v[i];
  fe c = fe_add(fe_mul(fe_sqr(x), x), fe_from_u32(7));
  aff Rp;
  Rp.x = fe_mul(x, c);
  Rp.y = fe_sqr(c);
  IBFT_STAGE(4);
  const fe z8 = ecmult_build_rtable_globalz(Rp, T);
  IBFT_STAGE(7);
  jac A = ecmult_streams(dg, G, T, false);
  IBFT_STAGE(8);
  // park A (and c) in this thread's slice of the table, dead from here on: the comb's accumulator takes their registers
  const bool a_inf = A.inf;
  T.store(0, A.x, A.y);
  T.store(1, fe_mul(A.z, z8), c);
  jac B;
#if IBFT_GEN_WIDE > 0
  if (WIDE) {
    ecmult_gen_wide_prefetch(dg, G);
    B = ecmult_gen_wide(dg, G);
  } else
#endif
  {
    ecmult_gen_comb_prefetch(dg, G);
    B = ecmult_gen_comb(dg, G);
  }
  T.load(0, A.x, A.y);
  T.load(1, A.z, c);
  A.inf = a_inf;
  return recover_final(A, c, v, B, qx, qy);
}
IBFT_HD bool recover_key(const exec_serial& ex, const sc& r, const sc& s, uint8_t v, const uint8_t* z_be, const gtab_view& G,
                         const rtab_view& T, fe& qx, fe& qy) {
#if !defined(__CUDA_ARCH__)
  // the host emulation supplies the comb entries through host_pos or host_wide; without them it runs the composition above
  if (G.has_wide()) return recover_key_serial<true>(r, s, v, z_be, G, T, qx, qy);
  if (G.host_pos == nullptr) return recover_key<exec_serial>(ex, r, s, v, z_be, G, T, qx, qy);
#endif
  (void)ex;
  return recover_key_serial<false>(r, s, v, z_be, G, T, qx, qy);
}
#if IBFT_GEN_WIDE > 0
// the one-thread recovery with u1*G from the wide comb (G.wide must be set)
struct exec_serial_wide : exec_serial {};
IBFT_HD bool recover_key(const exec_serial_wide&, const sc& r, const sc& s, uint8_t v, const uint8_t* z_be, const gtab_view& G,
                         const rtab_view& T, fe& qx, fe& qy) {
  return recover_key_serial<true>(r, s, v, z_be, G, T, qx, qy);
}
#endif
#endif

// Recover the signer of (r, s, v) over digest z.  Returns false when the signature is invalid; addr20 then zero.
template <class EX>
IBFT_HD bool ecrecover_address_x(const EX& ex, const uint8_t* r_be, const uint8_t* s_be, uint8_t v, const uint8_t* z_be,
                                 const gtab_view& G, const rtab_view& T, uint8_t* addr20, aff* key_out = nullptr) {
#pragma unroll
  for (int i = 0; i < 20; i++) addr20[i] = 0;
  sc r = sc_from_be(r_be), s = sc_from_be(s_be);
  if (v > 1) return false;
  if (sc_is_zero(r) || sc_is_zero(s) || sc_ge_n(r) || sc_ge_n(s)) return false;
  IBFT_STAGE(1);
  fe qx, qy;
  if (!recover_key(ex, r, s, v, z_be, G, T, qx, qy)) return false;
  if (key_out) { key_out->x = qx; key_out->y = qy; }
  IBFT_STAGE(9);
  keccak256_xy_address(qx, qy, addr20);
  IBFT_STAGE(10);
  return true;
}
IBFT_HD bool ecrecover_address(const uint8_t* r_be, const uint8_t* s_be, uint8_t v, const uint8_t* z_be,
                               const gtab_view& G, const rtab_view& T, uint8_t* addr20, aff* key_out = nullptr) {
  return ecrecover_address_x(exec_serial{}, r_be, s_be, v, z_be, G, T, addr20, key_out);
}

// Key registry: whether (x, y) may be the key of the entry of address addr20.  A known-key accept stands for "recovery yields
// exactly this key", so the signer it names is the entry's address; a key taken from anywhere but a recovery of this engine
// (another device's registry) has to show that it hashes to that address.  Both coordinates must be in the limb form a
// recovery stores (fully reduced, < p), the point on the curve, and its address addr20.
IBFT_HD bool key_matches_address(const fe& x, const fe& y, const uint8_t* addr20) {
  const fe xn = fe_normalize(x), yn = fe_normalize(y);
  uint32_t d = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) d |= (xn.v[i] ^ x.v[i]) | (yn.v[i] ^ y.v[i]);
  if (d != 0) return false;
  if (!fe_equal(fe_sqr(y), fe_add(fe_mul(fe_sqr(x), x), fe_from_u32(7)))) return false;
  uint8_t a[20];
  keccak256_xy_address(x, y, a);
#pragma unroll
  for (int i = 0; i < 20; i++) d |= (uint32_t)(a[i] ^ addr20[i]);
  return d == 0;
}

// Why one item is rejected (ibft_explain_batch): the recover path's decision, step by step, as an IBFT_REASON_* code.  The steps
// run in the order the verify kernels decide, so the first failing one is the reason.  member(group, signer) is the validator-set
// test of the kernels (true for a group without a table).  grouped: the call has groups (without, no item is ever of an unknown
// group, as in the verify calls).  addr20 = the recovered address when recovery succeeded, else zero.
template <class EX, class MEMBER>
IBFT_HD uint8_t explain_item(const EX& ex, const ibft_sig_item& it, const uint8_t* arena, size_t arena_len, bool grouped,
                             uint32_t n_groups, const gtab_view& G, const rtab_view& T, const MEMBER& member, uint8_t* addr20) {
#pragma unroll
  for (int i = 0; i < 20; i++) addr20[i] = 0;
  if (grouped && it.group >= n_groups) return IBFT_REASON_NO_GROUP;
  resolved_item ri;
  bool have = false;
  if (resolve_item(it, arena, arena_len, ri, &have) == IBFT_ITEM_NEEDS_HOST) return IBFT_REASON_NEEDS_HOST;
  if (!have) return IBFT_REASON_MALFORMED;
  if (ri.v > 1) return IBFT_REASON_BAD_V;
  const sc r = sc_from_be(ri.r), s = sc_from_be(ri.s);
  if (sc_is_zero(r) || sc_ge_n(r)) return IBFT_REASON_R_RANGE;
  if (sc_is_zero(s) || sc_ge_n(s)) return IBFT_REASON_S_RANGE;
  // recover_key answers false both for a non-residue and for the point at infinity: tell them apart first
  fe x;
#pragma unroll
  for (int i = 0; i < 8; i++) x.v[i] = r.v[i];
  const fe c = fe_add(fe_mul(fe_sqr(x), x), fe_from_u32(7));
  if (!fe_equal(fe_sqr(fe_sqrt_candidate(c)), c)) return IBFT_REASON_R_NOT_X;
  if (!ecrecover_address_x(ex, ri.r, ri.s, ri.v, ri.z, G, T, addr20)) return IBFT_REASON_NO_KEY;
  bool same = true;
#pragma unroll
  for (int i = 0; i < 20; i++) same = same && addr20[i] == ri.signer[i];
  if (!same) return IBFT_REASON_SIGNER_MISMATCH;
  if (!member(it.group, ri.signer)) return IBFT_REASON_NOT_VALIDATOR;
  return IBFT_REASON_OK;
}

#if IBFT_WC > 0
// ------------------------------------------------------------------------------------------------------------
// Split pipeline of the mid-size latency kernel (k_recover_split): one signature's serial chain is cut between a CHAIN warp
// and a HELPER warp that run on different schedulers of the SM.
//   helper, phase 1: digest, range checks, r^-1 mod n, u1 = -z/r, u2 = s/r, GLV split of both          -> digits of u2
//   helper, phase 2: y = sqrt(r^3 + 7) with the parity of v, u1*G as a comb over per-position tables     -> y, affine u1*G
//   chain:           u2*R WITHOUT knowing y: it works on the isomorphic curve E': Y^2 = X^3 + 7 y^6, where
//                    phi(R) = (x y^2, y^4) = (x c, c^2) with c = x^3 + 7 needs no square root (the a = 0 group law never
//                    uses b, and (X, Y) -> (beta X, Y) is the same endomorphism on E'), then maps the Jacobian result
//                    back with ONE multiplication, (X', Y', Z') -> (X', Y', Z' y), adds u1*G, converts, hashes.
// The chain warp's critical path loses sqrt, the scalar inversion, the GLV split, the digest and the generator stream.
// ------------------------------------------------------------------------------------------------------------
// helper phase 1, in three steps so that the r^-1 of several signatures can share ONE inversion (Montgomery's trick across
// the helper's passes): range check -> [batched inversion by the caller] -> digits of u2 = s/r -> digits of u1 = -z/r.
IBFT_HD bool split_sig_in_range(const resolved_item& ri) {
  sc r = sc_from_be(ri.r), s = sc_from_be(ri.s);
  if (ri.v > 1) return false;
  return !(sc_is_zero(r) || sc_is_zero(s) || sc_ge_n(r) || sc_ge_n(s));
}
IBFT_HD void split_helper_u2(const resolved_item& ri, const sc& rinv, ecmult_digits& dg) {
  ecmult_split_into(sc_mul(sc_from_be(ri.s), rinv), dg, 0);
}
IBFT_HD void split_helper_u1(const resolved_item& ri, const sc& rinv, ecmult_digits& dg) {
  sc z = sc_reduce_once(sc_from_be(ri.z));
  ecmult_split_into(sc_neg(sc_mul(z, rinv)), dg, 2);
}
// all of phase 1 for one signature (host emulation).  Returns false when (r, s, v) is out of range (verdict 0).
IBFT_HD bool split_helper_scalars(const resolved_item& ri, ecmult_digits& dg) {
  if (!split_sig_in_range(ri)) return false;
  sc rinv = IBFT_SC_INV(sc_from_be(ri.r));
  split_helper_u2(ri, rinv, dg);
  split_helper_u1(ri, rinv, dg);
  return true;
}
// helper phase 2.  Returns false when r is not an abscissa of the curve.  g_inf: u1*G is the point at infinity (u1 = 0).
IBFT_HD bool split_helper_point(const resolved_item& ri, const ecmult_digits& dg, const gtab_view& G, fe& y, bool& g_inf, fe& gx,
                                fe& gy) {
  sc r = sc_from_be(ri.r);
  fe x;
#pragma unroll
  for (int i = 0; i < 8; i++) x.v[i] = r.v[i];
  fe y2 = fe_add(fe_mul(fe_sqr(x), x), fe_from_u32(7));
  y = fe_sqrt_candidate(y2);
  if (!fe_equal(fe_sqr(y), y2)) return false;
  y = fe_normalize(y);
  if ((y.v[0] & 1u) != (uint32_t)ri.v) y = fe_normalize(fe_neg(y));
  jac P = ecmult_gen_comb(dg, G);
  g_inf = P.inf || fe_is_zero(P.z);
  if (!g_inf) {
    fe zi = IBFT_FE_INV(P.z), zi2 = fe_sqr(zi);
    gx = fe_mul(P.x, zi2);
    gy = fe_mul(P.y, fe_mul(zi2, zi));
  }
  return true;
}
// chain: phi(R) on E' from the abscissa alone; c = x^3 + 7 = y^2
IBFT_HD aff split_chain_point(const uint8_t* r_be, fe* c_out = nullptr) {
  sc r = sc_from_be(r_be);
  fe x;
#pragma unroll
  for (int i = 0; i < 8; i++) x.v[i] = r.v[i];
  fe c = fe_add(fe_mul(fe_sqr(x), x), fe_from_u32(7));
  aff Rp;
  Rp.x = fe_mul(x, c);
  Rp.y = fe_sqr(c);
  if (c_out) *c_out = c;
  return Rp;
}
// chain: map acc (= u2 * phi(R) on E') back, add u1*G, derive the address.  false = point at infinity.
IBFT_HD bool split_chain_finish(jac acc, const fe& y, bool g_inf, const fe& gx, const fe& gy, uint8_t* addr20,
                                aff* key_out = nullptr) {
#pragma unroll
  for (int i = 0; i < 20; i++) addr20[i] = 0;
  if (!acc.inf) acc.z = fe_mul(acc.z, y);
  if (!g_inf) acc = jac_add_affine(acc, gx, gy);
  if (acc.inf || fe_is_zero(acc.z)) return false;
  fe zi = IBFT_FE_INV(acc.z);
  fe zi2 = fe_sqr(zi);
  fe qx = fe_normalize(fe_mul(acc.x, zi2));
  fe qy = fe_normalize(fe_mul(acc.y, fe_mul(zi2, zi)));
  if (key_out) { key_out->x = qx; key_out->y = qy; }
  keccak256_xy_address(qx, qy, addr20);
  return true;
}
// the same for the four-lane chain (XYZZ accumulator): Z -> Z y means ZZ -> ZZ c, ZZZ -> ZZZ c y
template <class EX>
IBFT_HD bool split_chain_finish_x(const EX& ex, xyzz acc, const fe& c, const fe& y, bool g_inf, const fe& gx, const fe& gy,
                                  uint8_t* addr20, aff* key_out = nullptr) {
#pragma unroll
  for (int i = 0; i < 20; i++) addr20[i] = 0;
  if (!acc.inf) {
    fe a[4], b[4], o[4];
    a[0] = acc.zz; b[0] = c; a[1] = c; b[1] = y;
    ex.mul4(a, b, 2, o);
    acc.zz = o[0];
    a[0] = acc.zzz; b[0] = o[1];
    ex.mul4(a, b, 1, o);
    acc.zzz = o[0];
  }
  if (!g_inf) {
    xyzz q;
    q.x = gx; q.y = gy; q.zz = fe_from_u32(1); q.zzz = q.zz; q.inf = false;
    acc = xyzz_add_x(ex, acc, q);
  }
  if (acc.inf || fe_is_zero(acc.zzz)) return false;
  fe i3 = IBFT_FE_INV(acc.zzz);
  fe zi = fe_mul(acc.zz, i3);
  fe qx = fe_normalize(fe_mul(acc.x, fe_sqr(zi)));
  fe qy = fe_normalize(fe_mul(acc.y, i3));
  if (key_out) { key_out->x = qx; key_out->y = qy; }
  keccak256_xy_address(qx, qy, addr20);
  return true;
}
#endif

#if IBFT_WC > 0
// ------------------------------------------------------------------------------------------------------------
// Verification against a KNOWN public key.  Once a validator's signature has been recovered successfully its key Q is known
// (addr(Q) = the validator's address); later signatures of that validator are checked as u1*G + u2*Q == R with u1 = z/s,
// u2 = r/s, against a per-validator table of multiples of Q: no square root, no per-signature table, no address hash.
//   accept  <=>  the point equals R = (r, y) with the parity of y equal to v  <=>  recovery from (r, s, v, z) yields exactly Q
// (zG + rQ = sR  <=>  Q = r^-1 (sR - zG); x = r only, as in the recovery convention of this engine), hence accept implies the
// recover path's verdict 1.  A reject says "recovery would NOT yield Q" -- the caller then runs the recover path, so the
// final verdict is the recover path's in every case (also when the signature was made by another key with the same address).
// ------------------------------------------------------------------------------------------------------------
IBFT_HD bool ecdsa_verify_known(const resolved_item& ri, const gtab_view& G, const gtab_view& Qt) {
  sc r = sc_from_be(ri.r), s = sc_from_be(ri.s);
  if (ri.v > 1) return false;
  if (sc_is_zero(r) || sc_is_zero(s) || sc_ge_n(r) || sc_ge_n(s)) return false;
  sc z = sc_reduce_once(sc_from_be(ri.z));
  sc w = IBFT_SC_INV(s);
  ecmult_digits dg;
  ecmult_split_into(sc_mul(r, w), dg, 0);
  ecmult_split_into(sc_mul(z, w), dg, 2);
  jac P = ecmult_streams_known(dg, G, Qt);
  if (P.inf || fe_is_zero(P.z)) return false;
  fe zi = IBFT_FE_INV(P.z);
  fe zi2 = fe_sqr(zi);
  fe px = fe_normalize(fe_mul(P.x, zi2));
  fe py = fe_normalize(fe_mul(P.y, fe_mul(zi2, zi)));
  bool same = true;
#pragma unroll
  for (int i = 0; i < 8; i++) same = same && (px.v[i] == r.v[i]);  // r < n < p: canonical
  return same && ((py.v[0] & 1u) == (uint32_t)ri.v);
}

// The same verification cut between a chain warp and a helper warp (k_verify_split): the helper supplies w = s^-1, the digits
// of u2 = r w, and later the affine u1*G = (z w) G from the comb tables; the chain walks u2*Q and closes the check.
IBFT_HD void known_helper_u2(const resolved_item& ri, const sc& w, ecmult_digits& dg) { ecmult_split_into(sc_mul(sc_from_be(ri.r), w), dg, 0); }
IBFT_HD void known_helper_u1g(const resolved_item& ri, const sc& w, const gtab_view& G, bool& g_inf, fe& gx, fe& gy) {
  ecmult_digits dg;
#pragma unroll
  for (int k = 0; k < 6; k++) dg.ks[0][k] = dg.ks[1][k] = 0;
  dg.kneg[0] = dg.kneg[1] = false;
  ecmult_split_into(sc_mul(sc_reduce_once(sc_from_be(ri.z)), w), dg, 2);
  jac P = ecmult_gen_comb(dg, G);
  g_inf = P.inf || fe_is_zero(P.z);
  if (!g_inf) {
    fe zi = IBFT_FE_INV(P.z), zi2 = fe_sqr(zi);
    gx = fe_mul(P.x, zi2);
    gy = fe_mul(P.y, fe_mul(zi2, zi));
  }
}
// chain: acc = u2*Q (Jacobian); accept <=> acc + u1*G == (r, y) with parity(y) == v
IBFT_HD bool known_chain_finish(jac acc, bool g_inf, const fe& gx, const fe& gy, const resolved_item& ri) {
  if (!g_inf) acc = jac_add_affine(acc, gx, gy);
  if (acc.inf || fe_is_zero(acc.z)) return false;
  fe zi = IBFT_FE_INV(acc.z);
  fe zi2 = fe_sqr(zi);
  fe px = fe_normalize(fe_mul(acc.x, zi2));
  fe py = fe_normalize(fe_mul(acc.y, fe_mul(zi2, zi)));
  sc r = sc_from_be(ri.r);
  bool same = true;
#pragma unroll
  for (int i = 0; i < 8; i++) same = same && (px.v[i] == r.v[i]);
  return same && ((py.v[0] & 1u) == (uint32_t)ri.v);
}

// One comb position of a validator's key table: m * 2^(8 pos) * Q for m = 1..128 (affine, 16 words per entry), by 8*pos doublings
// and repeated addition; each entry normalised with its own inversion (built once per validator, off the hot path).
IBFT_HD void build_keytab_pos(const aff& Q, int pos, uint32_t* out) {
  jac P;
  P.x = Q.x; P.y = Q.y; P.z = fe_from_u32(1); P.inf = false;
  aff B = Q;
  if (pos > 0) {
    IBFT_ROLLED
    for (int t = 0; t < IBFT_WQ * pos; t++) P = jac_double(P);
    fe zi = IBFT_FE_INV(P.z), zi2 = fe_sqr(zi);
    B.x = fe_normalize(fe_mul(P.x, zi2));
    B.y = fe_normalize(fe_mul(P.y, fe_mul(zi2, zi)));
    P.x = B.x; P.y = B.y; P.z = fe_from_u32(1);
  }
  IBFT_ROLLED
  for (int m = 0; m < IBFT_KEYTAB_ENTRIES; m++) {
    if (m) P = jac_add_affine(P, B.x, B.y);  // the first addition is a doubling (handled by the adder)
    fe x = fe_zero(), y = fe_zero();
    if (!P.inf && !fe_is_zero(P.z)) {
      fe zi = IBFT_FE_INV(P.z), zi2 = fe_sqr(zi);
      x = fe_normalize(fe_mul(P.x, zi2));
      y = fe_normalize(fe_mul(P.y, fe_mul(zi2, zi)));
    }
#pragma unroll
    for (int i = 0; i < 8; i++) { out[16 * m + i] = x.v[i]; out[16 * m + 8 + i] = y.v[i]; }
  }
}
// the whole table of one validator (IBFT_KEYTAB_WORDS words)
IBFT_HD void build_keytab(const aff& Q, uint32_t* out) {
  IBFT_ROLLED
  for (int pos = 0; pos < IBFT_KEYTAB_POSITIONS; pos++)
    build_keytab_pos(Q, pos, out + (size_t)pos * IBFT_KEYTAB_ENTRIES * IBFT_GTAB_ENTRY_WORDS);
}
#endif

// ECDSA signing with a given nonce (the MessageConstructor side: reference core/backend.go:12-34 requires every built
// message to be signed and BuildCommitMessage to create a committed seal).  sig65 = R||S||V, s normalised to the low half.
// Returns false (sig65 all zero) when the key is 0 mod n -- no key recovers from such a signature -- or the nonce is unusable
// (k outside [1, n), R.x >= n, r = 0 or s = 0): the same rule as oracle_sign_with_k.
IBFT_HD bool ecdsa_sign(const uint8_t* d_be, const uint8_t* z_be, const uint8_t* k_be, const gtab_view& G, const rtab_view& T,
                        uint8_t* sig65) {
#pragma unroll
  for (int i = 0; i < 65; i++) sig65[i] = 0;
  sc k = sc_from_be(k_be);
  if (sc_is_zero(k) || sc_ge_n(k)) return false;
  sc d = sc_reduce_once(sc_from_be(d_be));
  if (sc_is_zero(d)) return false;
  sc z = sc_reduce_once(sc_from_be(z_be));
  aff g1;
  G.load(0, g1.x, g1.y);  // 1*G; its digit streams are all zero (u2 = 0), only the generator streams add
  sc zero;
#pragma unroll
  for (int i = 0; i < 8; i++) zero.v[i] = 0;
  jac Rj = ecmult_double(k, zero, g1, G, T);
  if (Rj.inf || fe_is_zero(Rj.z)) return false;
  fe zi = IBFT_FE_INV(Rj.z);
  fe zi2 = fe_sqr(zi);
  fe rx = fe_normalize(fe_mul(Rj.x, zi2));
  fe ry = fe_normalize(fe_mul(Rj.y, fe_mul(zi2, zi)));
  sc r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = rx.v[i];
  if (sc_ge_n(r) || sc_is_zero(r)) return false;
  sc s = sc_mul(IBFT_SC_INV(k), sc_add(z, sc_mul(r, d)));
  if (sc_is_zero(s)) return false;
  uint8_t v = (uint8_t)(ry.v[0] & 1u);
  if (sc_is_high(s)) {
    s = sc_neg(s);
    v ^= 1;
  }
  sc_to_be(r, sig65);
  sc_to_be(s, sig65 + 32);
  sig65[64] = v;
  return true;
}

// ECDSA signing with libsecp256k1's default nonce: secp256k1_ecdsa_sign_recoverable with nonce_function_rfc6979, which is what
// go-ethereum's crypto.Sign runs (the contract of ibft_sign_batch_rfc6979).  sig65 = R||S||V as ecdsa_sign makes it.  Returns
// false (sig65 all zero) for a key outside [1, n), for R.x >= n, where libsecp256k1 would answer with recovery id 2 or 3, and
// when four candidates gave no signature.
IBFT_HD bool ecdsa_sign_rfc6979(const uint8_t* d_be, const uint8_t* z_be, const gtab_view& G, const rtab_view& T, uint8_t* sig65) {
  const sc d = sc_from_be(d_be);
  if (!sc_is_zero(d) && !sc_ge_n(d)) {
    uint8_t zm[32], z1[32], k[32];
    sc_to_be(sc_reduce_once(sc_from_be(z_be)), zm);
    uint32_t carry = 1;  // z1 = (z mod n) + 1 < 2^256
    for (int i = 31; i >= 0; i--) {
      carry += zm[i];
      z1[i] = (uint8_t)carry;
      carry >>= 8;
    }
    for (uint32_t c = 0; c < 4; c++) {
      rfc6979_candidate(d_be, zm, c, k);
      const sc kc = sc_from_be(k);
      if (sc_is_zero(kc) || sc_ge_n(kc)) continue;  // libsecp256k1 moves on to the next candidate
      if (ecdsa_sign(d_be, zm, k, G, T, sig65)) return true;
      // With d and k in [1, n) ecdsa_sign refuses only R.x >= n (r = 0 would need R.x = n: no point has x = 0) and s = 0.
      // R does not depend on the digest, and s = k^-1 (z + r d) is k^-1 != 0 for the digest z + 1 where z gave 0.
      if (!ecdsa_sign(d_be, z1, k, G, T, sig65)) break;  // R.x >= n: refused
    }
  }
#pragma unroll
  for (int i = 0; i < 65; i++) sig65[i] = 0;
  return false;
}

}  // namespace ibft
