"""go-ibft wire schema (proto3) restated as plain Python: model, encoder, decoder, PayloadNoSig.

Oracle / test infrastructure only (see oracle/__init__.py).  Follows
messages/proto/messages.proto:7-110 (schema) and messages/proto/helper.go:13-27 (PayloadNoSig =
clone, Signature=nil, proto.Marshal).  Encoding rules are those of proto3 as emitted by
protobuf-go v1.28.1 (go.mod:9) for this schema: fields in field-number order, zero scalars and
empty bytes omitted, nil sub-messages omitted, present-but-empty sub-messages encoded as
``tag 00``, the set ``oneof payload`` member always emitted.  tests/test_oracle_proto.py checks
this encoder byte-for-byte against google.protobuf driven by the same schema.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Union

PREPREPARE, PREPARE, COMMIT, ROUND_CHANGE = 0, 1, 2, 3  # messages.proto:7-12


@dataclass
class View:  # messages.proto:15-21
    height: int = 0
    round: int = 0


@dataclass
class Proposal:  # messages.proto:104-110
    raw_proposal: bytes = b""
    round: int = 0


@dataclass
class PreparedCertificate:  # messages.proto:87-94
    proposal_message: Optional["IbftMessage"] = None
    prepare_messages: Optional[List["IbftMessage"]] = None  # None == Go nil slice


@dataclass
class RoundChangeCertificate:  # messages.proto:98-101
    round_change_messages: List["IbftMessage"] = field(default_factory=list)


@dataclass
class PrePrepareMessage:  # messages.proto:47-57
    proposal: Optional[Proposal] = None
    proposal_hash: bytes = b""
    certificate: Optional[RoundChangeCertificate] = None


@dataclass
class PrepareMessage:  # messages.proto:60-63
    proposal_hash: bytes = b""


@dataclass
class CommitMessage:  # messages.proto:66-72
    proposal_hash: bytes = b""
    committed_seal: bytes = b""


@dataclass
class RoundChangeMessage:  # messages.proto:75-83
    last_prepared_proposal: Optional[Proposal] = None
    latest_prepared_certificate: Optional[PreparedCertificate] = None


Payload = Union[PrePrepareMessage, PrepareMessage, CommitMessage, RoundChangeMessage, None]


@dataclass
class IbftMessage:  # messages.proto:24-44
    view: Optional[View] = None
    from_: bytes = b""
    signature: bytes = b""
    type: int = PREPREPARE  # an int32 enum, as in protobuf-go: decoded as int32(varint), encoded sign-extended
    payload: Payload = None

    # set by the decoder for a message that arrived in a NON-canonical encoding (unknown fields, duplicates, ...): the exact bytes,
    # because PayloadNoSig of such a message on a Go node is the protobuf re-marshal of what arrived, not of this model
    _wire: Optional[bytes] = field(default=None, repr=False, compare=False)

    def payload_no_sig(self) -> bytes:
        """messages/proto/helper.go:13-27."""
        if self._wire is not None:
            return payload_no_sig_from_wire(self._wire)
        return encode_ibft_message(self, with_signature=False)


# ----------------------------------------------------------------------------- encoder
def _varint(v: int) -> bytes:
    out = bytearray()
    v &= (1 << 64) - 1
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _f_varint(num: int, v: int) -> bytes:
    return b"" if v == 0 else _varint(num << 3) + _varint(v)


def _f_bytes(num: int, b: bytes) -> bytes:
    return b"" if len(b) == 0 else _varint((num << 3) | 2) + _varint(len(b)) + bytes(b)


def _f_msg(num: int, enc: Optional[bytes]) -> bytes:
    return b"" if enc is None else _varint((num << 3) | 2) + _varint(len(enc)) + enc


def encode_view(v: Optional[View]) -> Optional[bytes]:
    if v is None:
        return None
    return _f_varint(1, v.height) + _f_varint(2, v.round)


def encode_proposal(p: Optional[Proposal]) -> Optional[bytes]:
    if p is None:
        return None
    return _f_bytes(1, p.raw_proposal) + _f_varint(2, p.round)


def encode_pc(pc: Optional[PreparedCertificate]) -> Optional[bytes]:
    if pc is None:
        return None
    out = _f_msg(1, None if pc.proposal_message is None else encode_ibft_message(pc.proposal_message))
    for m in pc.prepare_messages or []:
        out += _f_msg(2, encode_ibft_message(m))
    return out


def encode_rcc(rcc: Optional[RoundChangeCertificate]) -> Optional[bytes]:
    if rcc is None:
        return None
    out = b""
    for m in rcc.round_change_messages:
        out += _f_msg(1, encode_ibft_message(m))
    return out


def encode_payload(p: Payload) -> bytes:
    if p is None:
        return b""
    if isinstance(p, PrePrepareMessage):
        body = _f_msg(1, encode_proposal(p.proposal)) + _f_bytes(2, p.proposal_hash) + _f_msg(3, encode_rcc(p.certificate))
        return _f_msg(5, body)
    if isinstance(p, PrepareMessage):
        return _f_msg(6, _f_bytes(1, p.proposal_hash))
    if isinstance(p, CommitMessage):
        return _f_msg(7, _f_bytes(1, p.proposal_hash) + _f_bytes(2, p.committed_seal))
    if isinstance(p, RoundChangeMessage):
        body = _f_msg(1, encode_proposal(p.last_prepared_proposal)) + _f_msg(2, encode_pc(p.latest_prepared_certificate))
        return _f_msg(8, body)
    raise TypeError(type(p))


def encode_ibft_message(m: IbftMessage, with_signature: bool = True) -> bytes:
    return (
        _f_msg(1, encode_view(m.view))
        + _f_bytes(2, m.from_)
        + (_f_bytes(3, m.signature) if with_signature else b"")
        + _f_varint(4, m.type)
        + encode_payload(m.payload)
    )


# ----------------------------------------------------------------------------- decoder
class DecodeError(ValueError):
    pass


def _int32(v: int) -> int:
    """protobuf-go's int32(v) of a decoded enum varint (IbftMessage.type)"""
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v & 0x80000000 else v


def _read_varint(buf: bytes, pos: int):
    shift = 0
    val = 0
    while True:
        if pos >= len(buf) or shift > 63:
            raise DecodeError("truncated/overlong varint")
        b = buf[pos]
        pos += 1
        if shift == 63 and b > 1:  # protowire.ConsumeVarint: the 10th byte holds bit 63 only
            raise DecodeError("variable length integer overflow")
        val |= (b & 0x7F) << shift
        shift += 7
        if not b & 0x80:
            return val & ((1 << 64) - 1), pos


def _fields(buf: bytes):
    pos = 0
    while pos < len(buf):
        key, pos = _read_varint(buf, pos)
        num, wt = key >> 3, key & 7
        if num == 0:
            raise DecodeError("field number 0")
        if wt == 0:
            v, pos = _read_varint(buf, pos)
        elif wt == 2:
            ln, pos = _read_varint(buf, pos)
            if pos + ln > len(buf):
                raise DecodeError("truncated bytes")
            v = buf[pos:pos + ln]
            pos += ln
        elif wt == 1:
            if pos + 8 > len(buf):
                raise DecodeError("truncated fixed64")
            v = buf[pos:pos + 8]
            pos += 8
        elif wt == 5:
            if pos + 4 > len(buf):
                raise DecodeError("truncated fixed32")
            v = buf[pos:pos + 4]
            pos += 4
        else:
            raise DecodeError(f"unsupported wire type {wt}")
        yield num, wt, v


# The typed decoders go through the generic field tree below (_parse_into), so that the MODEL a frame decodes to is the one
# protobuf-go builds: duplicated sub-messages merged, last scalar wins, a later oneof member replaces an earlier one, fields
# with a wrong wire type ignored (they are unknown fields).
def _view_from(n) -> View:
    return View(n.fields.get(1, 0), n.fields.get(2, 0))


def _proposal_from(n) -> Proposal:
    return Proposal(n.fields.get(1, b""), n.fields.get(2, 0))


def _pc_from(n) -> PreparedCertificate:
    pm = n.fields.get(1)
    reps = n.fields.get(2)
    return PreparedCertificate(None if pm is None else _message_from(pm), None if reps is None else [_message_from(x) for x in reps])


def _rcc_from(n) -> RoundChangeCertificate:
    return RoundChangeCertificate([_message_from(x) for x in n.fields.get(1, [])])


def _message_from(n) -> IbftMessage:
    m = IbftMessage()
    f = n.fields
    if 1 in f:
        m.view = _view_from(f[1])
    m.from_ = f.get(2, b"")
    m.signature = f.get(3, b"")
    m.type = f.get(4, 0)
    if 5 in f:
        g = f[5].fields
        m.payload = PrePrepareMessage(_proposal_from(g[1]) if 1 in g else None, g.get(2, b""), _rcc_from(g[3]) if 3 in g else None)
    elif 6 in f:
        m.payload = PrepareMessage(f[6].fields.get(1, b""))
    elif 7 in f:
        m.payload = CommitMessage(f[7].fields.get(1, b""), f[7].fields.get(2, b""))
    elif 8 in f:
        g = f[8].fields
        m.payload = RoundChangeMessage(_proposal_from(g[1]) if 1 in g else None, _pc_from(g[2]) if 2 in g else None)
    if n.raw is not None and encode_ibft_message(m) != n.raw:
        m._wire = n.raw
    return m


def _tree(buf: bytes, type_name: str):
    n = _Node()
    n.raw = bytes(buf)
    _parse_into(n, n.raw, type_name)
    return n


def decode_view(buf: bytes) -> View:
    return _view_from(_tree(buf, "View"))


def decode_proposal(buf: bytes) -> Proposal:
    return _proposal_from(_tree(buf, "Proposal"))


def decode_pc(buf: bytes) -> PreparedCertificate:
    return _pc_from(_tree(buf, "PreparedCertificate"))


def decode_rcc(buf: bytes) -> RoundChangeCertificate:
    return _rcc_from(_tree(buf, "RoundChangeCertificate"))


def decode_ibft_message(buf: bytes) -> IbftMessage:
    return _message_from(_tree(buf, "IbftMessage"))


# ----------------------------------------------------------------------------- byte-exact re-marshal of ANY parseable frame
# messages/proto/helper.go:13-27 is proto.Clone + Signature = nil + proto.Marshal.  For a frame protobuf-go itself produced the
# model encoder above reproduces those bytes.  For every OTHER parseable frame (a Byzantine validator may sign whatever bytes it
# likes and the honest Go nodes will re-marshal them the protobuf-go way) the result follows protobuf's parsing rules, restated
# here on a generic field tree:
#   * a known field with the wrong wire type, and every unknown field (groups included), is kept verbatim in the message's unknown
#     bytes and re-emitted AFTER its known fields, in arrival order;
#   * a singular scalar / bytes field that appears several times: the last occurrence wins;
#   * a singular sub-message that appears several times is MERGED field by field (the same rule, recursively);
#   * a oneof: a different member replaces the one set before, the same member again is merged;
#   * repeated sub-messages accumulate;
#   * an enum (IbftMessage.type) is int32: decoding keeps the low 32 bits as a signed value, encoding sign-extends it to 64 bits
#     (a negative type takes 10 bytes) and omits it when it is 0;
#   * a varint whose 10th byte is above 1 overflows 64 bits: a decode error (protowire.ConsumeVarint), wherever it appears;
#   * on output: fields in field-number order, zero scalars and empty bytes omitted, minimal varints.
_SCHEMA = {
    "IbftMessage": {1: ("msg", "View"), 2: ("bytes",), 3: ("bytes",), 4: ("enum",), 5: ("oneof", "PrePrepareMessage"),
                    6: ("oneof", "PrepareMessage"), 7: ("oneof", "CommitMessage"), 8: ("oneof", "RoundChangeMessage")},
    "View": {1: ("varint",), 2: ("varint",)},
    "PrePrepareMessage": {1: ("msg", "Proposal"), 2: ("bytes",), 3: ("msg", "RoundChangeCertificate")},
    "PrepareMessage": {1: ("bytes",)},
    "CommitMessage": {1: ("bytes",), 2: ("bytes",)},
    "RoundChangeMessage": {1: ("msg", "Proposal"), 2: ("msg", "PreparedCertificate")},
    "Proposal": {1: ("bytes",), 2: ("varint",)},
    "RoundChangeCertificate": {1: ("rep", "IbftMessage")},
    "PreparedCertificate": {1: ("msg", "IbftMessage"), 2: ("rep", "IbftMessage")},
}
_MAX_DEPTH = 100  # protobuf-go's default recursion limit is 10,000; anything legitimate needs 8


class _Node:
    __slots__ = ("fields", "unknown", "raw")

    def __init__(self):
        self.fields = {}
        self.unknown = bytearray()
        self.raw = None   # the bytes this node was parsed from; None once a second occurrence has been merged into it


def _skip_group(buf: bytes, pos: int, number: int, depth: int) -> int:
    """position just past the END_GROUP tag matching `number` (nested groups allowed)"""
    if depth > _MAX_DEPTH:
        raise DecodeError("nesting too deep")
    while True:
        key, pos = _read_varint(buf, pos)
        num, wt = key >> 3, key & 7
        if num == 0 or num > 0x1FFFFFFF:
            raise DecodeError("invalid field number")
        if wt == 4:
            if num != number:
                raise DecodeError("mismatched end group")
            return pos
        if wt == 0:
            _, pos = _read_varint(buf, pos)
        elif wt == 1:
            pos += 8
        elif wt == 5:
            pos += 4
        elif wt == 2:
            ln, pos = _read_varint(buf, pos)
            pos += ln
        elif wt == 3:
            pos = _skip_group(buf, pos, num, depth + 1)
        else:
            raise DecodeError("invalid wire type")
        if pos > len(buf):
            raise DecodeError("truncated group")


def _parse_into(node: _Node, buf: bytes, type_name: str, depth: int = 0) -> None:
    if depth > _MAX_DEPTH:
        raise DecodeError("nesting too deep")
    schema = _SCHEMA[type_name]
    pos = 0
    while pos < len(buf):
        start = pos
        key, pos = _read_varint(buf, pos)
        num, wt = key >> 3, key & 7
        if num == 0 or num > 0x1FFFFFFF:
            raise DecodeError("invalid field number")
        val = None
        if wt == 0:
            val, pos = _read_varint(buf, pos)
        elif wt == 1:
            pos += 8
        elif wt == 5:
            pos += 4
        elif wt == 2:
            ln, pos = _read_varint(buf, pos)
            val = buf[pos:pos + ln]
            pos += ln
        elif wt == 3:
            pos = _skip_group(buf, pos, num, depth + 1)
        else:
            raise DecodeError("invalid wire type")
        if pos > len(buf):
            raise DecodeError("truncated field")
        spec = schema.get(num)
        want = None if spec is None else (0 if spec[0] in ("varint", "enum") else 2)
        if spec is None or wt != want:
            node.unknown += buf[start:pos]
            continue
        kind = spec[0]
        if kind == "varint":
            node.fields[num] = val
        elif kind == "enum":
            node.fields[num] = _int32(val)
        elif kind == "bytes":
            node.fields[num] = bytes(val)
        elif kind == "rep":
            child = _Node()
            child.raw = bytes(val)
            _parse_into(child, val, spec[1], depth + 1)
            node.fields.setdefault(num, []).append(child)
        else:  # singular sub-message ("msg") or oneof member
            if kind == "oneof":
                for other in [k for k in node.fields if k != num and schema[k][0] == "oneof"]:
                    del node.fields[other]
            child = node.fields.get(num)
            if child is None:
                child = node.fields[num] = _Node()
                child.raw = bytes(val)
            else:
                child.raw = None
            _parse_into(child, val, spec[1], depth + 1)  # a second occurrence merges into the first


def _emit(node: _Node, type_name: str, skip: tuple = ()) -> bytes:
    schema = _SCHEMA[type_name]
    out = bytearray()
    for num in sorted(node.fields):
        if num in skip:
            continue
        spec, v = schema[num], node.fields[num]
        if spec[0] in ("varint", "enum"):
            out += _f_varint(num, v)
        elif spec[0] == "bytes":
            out += _f_bytes(num, v)
        elif spec[0] == "rep":
            for child in v:
                out += _f_msg(num, _emit(child, spec[1]))
        else:
            out += _f_msg(num, _emit(v, spec[1]))
    return bytes(out) + bytes(node.unknown)


def remarshal(frame: bytes, with_signature: bool = True) -> bytes:
    """proto.Marshal(proto.Unmarshal(frame)) the protobuf-go way; with_signature=False clears the (known) signature field first:
    IbftMessage.PayloadNoSig() for a message that arrived as `frame`."""
    root = _Node()
    _parse_into(root, bytes(frame), "IbftMessage")
    return _emit(root, "IbftMessage", skip=() if with_signature else (3,))


def payload_no_sig_from_wire(frame: bytes) -> bytes:
    return remarshal(frame, with_signature=False)
