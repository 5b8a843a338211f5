// group_hash.cuh -- the proposal hash a PREPARE or COMMIT names, read as go-ibft reads it, for groups bound to the hash of the
// accepted proposal (ibft_group_hash, include/ibft_verify.h).
//
// go-ibft counts a PREPARE or a COMMIT only when it names the proposal this node accepted: handlePrepare filters with
// IsValidProposalHash(state.proposal, ExtractPrepareHash(m)) (reference core/ibft.go:855-889), handleCommit checks
// ExtractCommitHash(m) before the seal (core/ibft.go:931-967).  Both extractors (messages/helpers.go:51-62, :107-118) read the
// DECODED message: nil unless msg.Type is the wanted type and the payload oneof holds the matching member, else that member's
// proposalHash.  The bytes given here are a raw frame (IBFT_KIND_WIRE) or IbftMessage.PayloadNoSig() (IBFT_KIND_PAYLOAD), which
// the host may have re-marshalled from a non-canonical frame, so unknown fields, duplicates and groups survive in them (DESIGN
// §9).  The scan therefore applies protobuf-go's decoding rules rather than parse_wire_frame's canonical check:
//   * the last `type` (field 4, varint) wins, read as int32;
//   * a oneof member (fields 5-8) replaces a different one set before; the same member again merges into it;
//   * proposalHash (field 1 of PrepareMessage / CommitMessage) is bytes: its last occurrence wins, even when empty;
//   * a known field with the wrong wire type, and every unknown field (groups included), is skipped;
//   * anything protobuf-go refuses ANYWHERE in the message -- an overlong varint, a length past the end, field number 0, wire type
//     6 or 7, an unmatched end-group -- makes the whole message nil, so every sub-message is walked, certificates included.
// oracle/ibft_proto.py is the reference (tests/test_emul_group_hash.py compares the two).  The walk is iterative over an explicit
// stack of open messages and groups; one deeper than IBFT_PB_MAX_DEPTH reads as nil.  A message go-ibft builds nests at most 8
// levels (verify_core.cuh), so only a frame a Byzantine validator shaped on purpose can reach it, and it then loses only that
// validator's own vote.
#pragma once
#include "verify_core.cuh"

namespace ibft {

#define IBFT_PB_MAX_DEPTH 32
#define IBFT_PB_GROUP 0xFFu  // stack entry of an open group (its contents are skipped)

// protowire.ConsumeVarint: at most 10 bytes, the 10th holding only bit 63; non-minimal encodings are accepted
IBFT_HD bool pb_varint(const uint8_t* w, uint32_t end, uint32_t& pos, uint64_t& v) {
  v = 0;
  for (int shift = 0; shift < 64; shift += 7) {
    if (pos >= end) return false;
    const uint8_t b = w[pos++];
    if (shift == 63 && b > 1) return false;
    v |= (uint64_t)(b & 0x7F) << shift;
    if (!(b & 0x80)) return true;
  }
  return false;
}

// What ExtractPrepareHash (msg_type 1) or ExtractCommitHash (msg_type 2) returns for the IbftMessage encoded in w[0, len): true
// with the span [*hash_off, *hash_off + *hash_len) of proposalHash (empty when the member holds none), false for nil.
IBFT_HD bool extract_vote_hash(const uint8_t* w, uint32_t len, uint32_t msg_type, uint32_t* hash_off, uint32_t* hash_len) {
  uint32_t end_stack[IBFT_PB_MAX_DEPTH], group_num[IBFT_PB_MAX_DEPTH];
  uint8_t type_stack[IBFT_PB_MAX_DEPTH];
  int depth = 0;
  end_stack[0] = len;
  type_stack[0] = WT_IBFT;
  group_num[0] = 0;
  uint32_t type = 0, member = 0, h_off = 0, h_len = 0;
  uint32_t pos = 0;
  for (;;) {
    while (depth > 0 && type_stack[depth] != IBFT_PB_GROUP && pos == end_stack[depth]) depth--;  // close finished sub-messages
    if (depth == 0 && pos == len) break;
    const uint32_t end = end_stack[depth], msg = type_stack[depth];
    uint64_t key;
    if (!pb_varint(w, end, pos, key)) return false;
    const uint64_t num = key >> 3;
    const uint32_t wt = (uint32_t)(key & 7);
    if (num == 0 || num > 0x1FFFFFFFu) return false;
    uint64_t v = 0;
    uint32_t off = 0, n = 0;
    if (wt == 4) {  // end of a group: must close the innermost open group, with its number
      if (msg != IBFT_PB_GROUP || num != group_num[depth]) return false;
      depth--;
      continue;
    } else if (wt == 3) {
      if (depth + 1 >= IBFT_PB_MAX_DEPTH) return false;
      depth++;
      end_stack[depth] = end;  // a group ends at its end-group tag, inside the enclosing message
      type_stack[depth] = IBFT_PB_GROUP;
      group_num[depth] = (uint32_t)num;
      continue;
    } else if (wt == 0) {
      if (!pb_varint(w, end, pos, v)) return false;
    } else if (wt == 1 || wt == 5) {
      const uint32_t k = wt == 1 ? 8u : 4u;
      if (end - pos < k) return false;
      pos += k;
    } else if (wt == 2) {
      if (!pb_varint(w, end, pos, v) || v > (uint64_t)(end - pos)) return false;
      off = pos;
      n = (uint32_t)v;
      pos += n;
    } else {
      return false;  // wire types 6 and 7 do not exist
    }
    if (msg == IBFT_PB_GROUP) continue;  // a group's fields are skipped
    const uint32_t kind = wire_field_kind(msg, (uint32_t)num);
    const uint32_t k = kind & 0x7Fu;
    if (kind == 0 || wt != (k == 1 ? 0u : 2u)) continue;  // unknown field, or a known one with the wrong wire type
    if (k == 1) {
      if (depth == 0 && num == 4) type = (uint32_t)v;  // int32(v): the low 32 bits
      continue;
    }
    if (k == 2) {
      // depth 1 holds IbftMessage's members only: PrepareMessage is member 6, CommitMessage member 7
      if (depth == 1 && num == 1 && (msg == WT_PREPARE || msg == WT_COMMIT)) { h_off = off; h_len = n; }
      continue;
    }
    if (depth == 0 && num >= 5 && num != member) {  // a different oneof member replaces the one set before
      member = (uint32_t)num;
      h_off = h_len = 0;
    }
    if (depth + 1 >= IBFT_PB_MAX_DEPTH) return false;
    depth++;
    end_stack[depth] = off + n;
    type_stack[depth] = (uint8_t)(k - 3);
    pos = off;
  }
  if (type != msg_type || member != (msg_type == 1u ? 6u : 7u)) return false;
  *hash_off = h_off;
  *hash_len = h_len;
  return true;
}

// Whether an item of a group bound to `bound` (32 bytes) names it, by the group's extractor (msg_type 1 = PREPARE, 2 = COMMIT):
//   SEAL        digest (the proposalHash the caller extracted); COMMIT groups only
//   WIRE_SEAL   commitData.proposalHash of the frame, which must be a COMMIT; COMMIT groups only
//   WIRE        the group's extractor over the frame
//   PAYLOAD     the group's extractor over the PayloadNoSig bytes
//   others      no hash is knowable: never
// A hash of any length other than 32 never matches (bytes.Equal against a 32-byte hash).
IBFT_HD bool item_names_hash(const ibft_sig_item& it, const uint8_t* arena, size_t arena_len, uint32_t msg_type, const uint8_t* bound) {
  const uint8_t* h;
  switch (it.kind) {
    case IBFT_KIND_SEAL:
      if (msg_type != 2u) return false;
      h = it.digest;
      break;
    case IBFT_KIND_WIRE_SEAL:
    case IBFT_KIND_WIRE:
    case IBFT_KIND_PAYLOAD: {
      if (it.kind == IBFT_KIND_WIRE_SEAL && msg_type != 2u) return false;
      if ((size_t)it.payload_off + it.payload_len > arena_len) return false;
      const uint8_t* w = arena + it.payload_off;
      uint32_t off, n;
      if (!extract_vote_hash(w, it.payload_len, msg_type, &off, &n) || n != 32) return false;
      h = w + off;
      break;
    }
    default:
      return false;
  }
  bool eq = true;
  for (int i = 0; i < 32; i++) eq = eq && h[i] == bound[i];
  return eq;
}

}  // namespace ibft
