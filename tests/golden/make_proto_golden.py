"""Generate tests/golden/proto_wire.json from the REFERENCE's own embedded descriptor.

Run in the authoring container only (needs /root/reference):
    python tests/golden/make_proto_golden.py
It reads the serialized FileDescriptorProto that protoc-gen-go embedded in
/root/reference/messages/proto/messages.pb.go (var file_messages_proto_messages_proto_rawDesc,
line 688+), loads it into google.protobuf, serialises a fixed list of messages with it and
records (case name, python-model repr, wire hex, wire hex with signature cleared = PayloadNoSig per
messages/proto/helper.go:13-27).  tests/test_oracle_proto.py replays the cases against
oracle/ibft_proto.py, and the C++ host codec is checked against the same file.
"""
import json
import os
import re
import sys

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))

from google.protobuf import descriptor_pb2, descriptor_pool, message_factory  # noqa: E402

from oracle import ibft_proto as ip  # noqa: E402
from edge_frames import EDGE_SEED, EDGE_VALIDATORS, EdgeFrames, sig_tlv, signed_variants  # noqa: E402

REF = "/root/reference/messages/proto/messages.pb.go"


def load_reference_classes():
    src = open(REF).read()
    m = re.search(r"file_messages_proto_messages_proto_rawDesc = \[\]byte\{(.*?)\n\}", src, re.S)
    raw = bytes(int(x, 16) for x in re.findall(r"0x([0-9a-fA-F]{2})", m.group(1)))
    fdp = descriptor_pb2.FileDescriptorProto.FromString(raw)
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    get = lambda n: message_factory.GetMessageClass(pool.FindMessageTypeByName(n))  # noqa: E731
    return {n: get(n) for n in ("IbftMessage", "View", "Proposal", "PreparedCertificate", "RoundChangeCertificate")}


def to_pb(cls, m: ip.IbftMessage):
    pb = cls["IbftMessage"]()
    fill_pb(pb, m)
    return pb


def fill_pb(pb, m: ip.IbftMessage):
    if m.view is not None:
        pb.view.SetInParent()
        pb.view.height = m.view.height
        pb.view.round = m.view.round
    pb.__setattr__("from", m.from_) if False else setattr(pb, "from", m.from_)
    pb.signature = m.signature
    pb.type = m.type
    p = m.payload
    if isinstance(p, ip.PrePrepareMessage):
        pb.preprepareData.SetInParent()
        if p.proposal is not None:
            pb.preprepareData.proposal.SetInParent()
            pb.preprepareData.proposal.rawProposal = p.proposal.raw_proposal
            pb.preprepareData.proposal.round = p.proposal.round
        pb.preprepareData.proposalHash = p.proposal_hash
        if p.certificate is not None:
            pb.preprepareData.certificate.SetInParent()
            for rc in p.certificate.round_change_messages:
                fill_pb(pb.preprepareData.certificate.roundChangeMessages.add(), rc)
    elif isinstance(p, ip.PrepareMessage):
        pb.prepareData.SetInParent()
        pb.prepareData.proposalHash = p.proposal_hash
    elif isinstance(p, ip.CommitMessage):
        pb.commitData.SetInParent()
        pb.commitData.proposalHash = p.proposal_hash
        pb.commitData.committedSeal = p.committed_seal
    elif isinstance(p, ip.RoundChangeMessage):
        pb.roundChangeData.SetInParent()
        if p.last_prepared_proposal is not None:
            pb.roundChangeData.lastPreparedProposal.SetInParent()
            pb.roundChangeData.lastPreparedProposal.rawProposal = p.last_prepared_proposal.raw_proposal
            pb.roundChangeData.lastPreparedProposal.round = p.last_prepared_proposal.round
        pc = p.latest_prepared_certificate
        if pc is not None:
            pb.roundChangeData.latestPreparedCertificate.SetInParent()
            if pc.proposal_message is not None:
                fill_pb(pb.roundChangeData.latestPreparedCertificate.proposalMessage, pc.proposal_message)
                pb.roundChangeData.latestPreparedCertificate.proposalMessage.SetInParent()
            for pm in pc.prepare_messages or []:
                fill_pb(pb.roundChangeData.latestPreparedCertificate.prepareMessages.add(), pm)


def cases():
    A = lambda i: bytes([0xA0 + i]) * 20  # noqa: E731
    H = b"\x22" * 32
    S = bytes(range(65))
    out = {}
    out["prepare_h1_r0"] = ip.IbftMessage(ip.View(1, 0), bytes(range(0xA0, 0xB4)), b"", ip.PREPARE, ip.PrepareMessage(H))
    out["prepare_h1e6_signed"] = ip.IbftMessage(ip.View(10**6, 0), A(1), S, ip.PREPARE, ip.PrepareMessage(H))
    out["commit_h1e6_signed"] = ip.IbftMessage(ip.View(10**6, 3), A(2), S, ip.COMMIT, ip.CommitMessage(H, S[::-1]))
    out["commit_empty_payload"] = ip.IbftMessage(ip.View(5, 0), A(2), S, ip.COMMIT, ip.CommitMessage())
    out["nil_view"] = ip.IbftMessage(None, A(3), S, ip.PREPARE, ip.PrepareMessage(H))
    out["empty_view"] = ip.IbftMessage(ip.View(0, 0), A(3), S, ip.PREPARE, ip.PrepareMessage(H))
    out["no_payload"] = ip.IbftMessage(ip.View(7, 1), A(4), S, ip.COMMIT, None)
    out["type_payload_mismatch"] = ip.IbftMessage(ip.View(7, 1), A(4), S, ip.PREPARE, ip.CommitMessage(H, S))
    out["all_default"] = ip.IbftMessage()
    out["big_varints"] = ip.IbftMessage(ip.View(2**64 - 1, 2**63), A(5), S, ip.ROUND_CHANGE, ip.RoundChangeMessage())
    pp0 = ip.IbftMessage(ip.View(9, 0), A(0), S, ip.PREPREPARE,
                         ip.PrePrepareMessage(ip.Proposal(b"block" * 50, 0), H, None))
    out["preprepare_r0"] = pp0
    preps = [ip.IbftMessage(ip.View(9, 0), A(i), S, ip.PREPARE, ip.PrepareMessage(H)) for i in (1, 2, 3)]
    pc = ip.PreparedCertificate(pp0, preps)
    rcs = [ip.IbftMessage(ip.View(9, 1), A(i), S, ip.ROUND_CHANGE,
                          ip.RoundChangeMessage(ip.Proposal(b"block" * 50, 0), pc)) for i in (0, 1, 2)]
    out["round_change_with_pc"] = rcs[0]
    out["round_change_empty"] = ip.IbftMessage(ip.View(9, 1), A(3), S, ip.ROUND_CHANGE, ip.RoundChangeMessage())
    out["round_change_pc_no_prepares"] = ip.IbftMessage(ip.View(9, 1), A(3), S, ip.ROUND_CHANGE,
                                                         ip.RoundChangeMessage(None, ip.PreparedCertificate(pp0, None)))
    out["round_change_pc_no_proposal"] = ip.IbftMessage(ip.View(9, 1), A(3), S, ip.ROUND_CHANGE,
                                                         ip.RoundChangeMessage(None, ip.PreparedCertificate(None, preps)))
    out["preprepare_r1_rcc"] = ip.IbftMessage(ip.View(9, 1), A(1), S, ip.PREPREPARE,
                                              ip.PrePrepareMessage(ip.Proposal(b"block" * 50, 1), H,
                                                                   ip.RoundChangeCertificate(rcs + [out["round_change_empty"]])))
    out["preprepare_empty_rcc"] = ip.IbftMessage(ip.View(9, 1), A(1), S, ip.PREPREPARE,
                                                 ip.PrePrepareMessage(ip.Proposal(b"", 0), b"", ip.RoundChangeCertificate([])))
    return out


def _tlvs(buf):
    out, pos = [], 0
    while pos < len(buf):
        s = pos
        key, pos = ip._read_varint(buf, pos)
        wt = key & 7
        if wt == 0:
            _, pos = ip._read_varint(buf, pos)
        elif wt == 2:
            ln, pos = ip._read_varint(buf, pos)
            pos += ln
        elif wt == 1:
            pos += 8
        elif wt == 5:
            pos += 4
        else:
            raise ValueError(wt)
        out.append(buf[s:pos])
    return out


def noncanonical_cases(cls):
    """Frames protobuf-go would NOT have produced but parses happily (a Byzantine validator may sign anything): duplicated and
    re-ordered fields, unknown fields, known numbers with the wrong wire type, groups, non-minimal varints, explicit zeros --
    with what google.protobuf (same descriptor) re-serialises them to, with and without the signature."""
    import random
    M = cls["IbftMessage"]
    rnd = random.Random(2024)
    unk = [bytes.fromhex(x) for x in ("4801", "5203616263", "5d01020304", "610102030405060708", "f80101", "1801", "0801", "2a00",
                                      "1a00", "7b08017c", "7b7c", "7b0a01617c", "2000", "20818000")]
    base = {n: to_pb(cls, m).SerializeToString(deterministic=True) for n, m in cases().items()}
    hand = {
        "view_split_in_two": bytes.fromhex("0a020805") + bytes.fromhex("0a021007") + base["prepare_h1_r0"][4:],
        "type_twice_last_wins": base["prepare_h1e6_signed"] + bytes.fromhex("2002"),
        "unknown_in_the_middle": base["commit_h1e6_signed"][:6] + bytes.fromhex("4801") + base["commit_h1e6_signed"][6:],
        "oneof_replaced": base["prepare_h1e6_signed"] + base["commit_h1e6_signed"][-103:],
        "signature_as_varint": bytes.fromhex("1801") + base["prepare_h1_r0"],
        "group_unknown": base["prepare_h1_r0"] + bytes.fromhex("7b0a0161087f7c"),
    }
    out = []
    for name, wire in hand.items():
        out.append((name, wire))
    names = sorted(base)
    for k in range(60):
        parts = _tlvs(base[names[k % len(names)]])
        for _ in range(rnd.randrange(1, 4)):
            op = rnd.randrange(5)
            if op == 0 and parts:
                parts.insert(rnd.randrange(len(parts) + 1), rnd.choice(parts))
            elif op == 1 and len(parts) > 1:
                i, j = rnd.randrange(len(parts)), rnd.randrange(len(parts))
                parts[i], parts[j] = parts[j], parts[i]
            elif op == 2:
                parts.insert(rnd.randrange(len(parts) + 1), rnd.choice(unk))
            elif op == 3 and parts:
                i = rnd.randrange(len(parts))
                key, pos = ip._read_varint(parts[i], 0)
                if key & 7 == 2:
                    ln, pos2 = ip._read_varint(parts[i], pos)
                    try:
                        inner = _tlvs(parts[i][pos2:pos2 + ln])
                    except Exception:
                        inner = []
                    if inner:
                        inner.insert(rnd.randrange(len(inner) + 1), rnd.choice(inner + unk))
                        body = b"".join(inner)
                        parts[i] = ip._varint(key) + ip._varint(len(body)) + body
            elif op == 4 and parts:
                del parts[rnd.randrange(len(parts))]
        out.append(("mutant_%02d" % k, b"".join(parts)))
    recs = []
    for name, wire in out:
        try:
            pb = M.FromString(wire)
        except Exception:
            recs.append({"name": name, "wire": wire.hex(), "parses": False})
            continue
        full = pb.SerializeToString(deterministic=True)
        pb.signature = b""
        recs.append({"name": name, "wire": wire.hex(), "parses": True, "remarshal": full.hex(),
                     "payload_no_sig": pb.SerializeToString(deterministic=True).hex()})
    return recs


# ----------------------------------------------------------------------------------------------------------- edge frames
# The frames of tests/edge_frames.py, each recorded by name and Keccak-256 with what protobuf answers for it: whether it decodes,
# whether decode + encode reproduces it (go_canonical), the Keccak-256 of its re-marshal and of its PayloadNoSig, its nesting
# levels, every `type` in it, and whether a Go node accepts its sender signature and committed seal.  upb (google.protobuf) and
# protobuf-go disagree in two places.  protowire.ConsumeVarint rejects a varint whose 10th byte is above 1 ("variable length
# integer overflow"), while upb masks such a VALUE varint to 64 bits and decodes the frame: for those rows go_parses is false by
# the protowire rule and the upb_* digests keep what upb did, so the difference stays visible.  The other way round,
# protobuf-go reads a TAG with ConsumeVarint (up to 10 bytes, field number at most 2^29 - 1) where upb refuses a tag longer than
# 5 bytes: for such a frame the go_* fields are upb's answers for the same frame with its tags re-encoded minimally, which
# protobuf-go reads identically, and upb_parses stays false.
def _pb_levels(pb):
    """nesting levels of a parsed message (the root is level 1; every present sub-message one more)"""
    subs = []
    for fd, v in pb.ListFields():
        if fd.message_type is None:
            continue
        subs += list(v) if fd.is_repeated else [v]
    return 1 + max((_pb_levels(s) for s in subs), default=0)


def _pb_types(pb):
    """IbftMessage.type of the message and of every IbftMessage nested in it"""
    out = [pb.type] if pb.DESCRIPTOR.name == "IbftMessage" else []
    for fd, v in pb.ListFields():
        if fd.message_type is not None:
            for s in (list(v) if fd.is_repeated else [v]):
                out += _pb_types(s)
    return out


class _Overflow(Exception):
    pass


def _protowire_read(buf: bytes, desc):
    """protobuf-go's reading of buf as `desc`: buf with every tag re-encoded minimally (sub-message length prefixes follow), which
    upb reads the way protobuf-go reads buf; None when buf is malformed.  Raises _Overflow where protowire.ConsumeVarint reports
    an overflow (a 10th byte above 1)."""
    out, pos = bytearray(), 0

    def rv():
        nonlocal pos
        v, shift, start = 0, 0, pos
        while True:
            b = buf[pos]
            pos += 1
            if shift == 63 and b > 1:
                raise _Overflow
            v |= (b & 0x7F) << shift
            shift += 7
            if not b & 0x80:
                return v, buf[start:pos]
    try:
        while pos < len(buf):
            key, _ = rv()
            out += ip._varint(key)
            num, wt = key >> 3, key & 7
            if wt == 0:
                out += rv()[1]
            elif wt in (1, 5):
                n = 8 if wt == 1 else 4
                out += buf[pos:pos + n]
                pos += n
            elif wt == 2:
                ln, raw = rv()
                body = buf[pos:pos + ln]
                pos += ln
                fd = desc.fields_by_number.get(num)
                inner = _protowire_read(body, fd.message_type) if fd is not None and fd.message_type is not None else body
                if inner is None:
                    return None
                out += (raw if inner == body else ip._varint(len(inner))) + inner
            else:
                return None
        return bytes(out) if pos == len(buf) else None
    except IndexError:
        return None


def edge_cases(cls):
    import workloads as wl
    from oracle import coracle as co
    M = cls["IbftMessage"]
    E = EdgeFrames()
    key = E.vs.keys[0]

    def keccak_hex(b):
        return co.keccak256(b).hex()

    def answers(wire):
        rec = {"upb_parses": False, "go_parses": False}
        try:
            go_src = _protowire_read(wire, M.DESCRIPTOR)  # None: protobuf-go cannot decode the frame
        except _Overflow:
            go_src = None
        try:
            pb, src = M.FromString(wire), wire
            rec.update(upb_parses=True)
        except Exception:
            if go_src is None or go_src == wire:
                return rec, None
            try:
                pb, src = M.FromString(go_src), go_src    # over-long tags: protobuf-go reads them, upb does not
            except Exception:
                return rec, None
        full = pb.SerializeToString(deterministic=True)
        nosig = M.FromString(src)
        nosig.signature = b""
        nosig = nosig.SerializeToString(deterministic=True)
        if go_src is None:
            rec.update(upb_remarshal_keccak=keccak_hex(full), upb_payload_no_sig_keccak=keccak_hex(nosig))  # upb's answer, not Go's
            return rec, None
        rec.update(go_parses=True, go_canonical=full == wire, go_remarshal_keccak=keccak_hex(full), go_payload_no_sig_keccak=keccak_hex(nosig),
                   go_levels=_pb_levels(pb), go_types=_pb_types(pb))
        # IsValidValidator (core/backend.go:41-45) and IsValidCommittedSeal on the frame, as a Go node decides them
        frm = getattr(pb, "from")
        sender = pb.HasField("view") and len(frm) == 20 and len(pb.signature) == 65 and \
            co.ecrecover_address(co.keccak256(nosig), pb.signature) == frm
        cd = pb.commitData
        seal = pb.type == ip.COMMIT and pb.WhichOneof("payload") == "commitData" and len(frm) == 20 and len(cd.proposalHash) == 32 and \
            len(cd.committedSeal) == 65 and co.ecrecover_address(wl.seal_digest(cd.proposalHash), cd.committedSeal) == frm
        rec.update(go_sender_valid=bool(sender), go_seal_valid=bool(seal))
        return rec, nosig

    recs, seen = [], set()
    for name, body in E.bases():
        _, go_nosig = answers(body(sig_tlv(b"\x00" * 65)))
        for vlab, wire in signed_variants(body, key, None if go_nosig is None else co.keccak256(go_nosig)):
            if wire in seen:      # the same bytes reached through two edges are recorded once
                continue
            seen.add(wire)
            rec, _ = answers(wire)
            recs.append({"name": "%s/%s" % (name, vlab), "wire_keccak": keccak_hex(wire), **rec})
    return recs


def main():
    cls = load_reference_classes()
    recs = []
    for name, m in cases().items():
        pb = to_pb(cls, m)
        wire = pb.SerializeToString(deterministic=True)
        pb.signature = b""
        nosig = pb.SerializeToString(deterministic=True)
        recs.append({"name": name, "model": repr(m), "wire": wire.hex(), "payload_no_sig": nosig.hex()})
    path = os.path.join(os.path.dirname(__file__), "proto_wire.json")
    edges = edge_cases(cls)
    text = json.dumps({"generator": "tests/golden/make_proto_golden.py",
                       "source": "descriptor embedded in reference messages/proto/messages.pb.go (protoc-gen-go v1.28.1)",
                       "cases": recs, "noncanonical": noncanonical_cases(cls), "edge_validators": [EDGE_SEED, EDGE_VALIDATORS],
                       "edges": "EDGES"}, indent=1)
    rows = ",\n  ".join(json.dumps(r, separators=(",", ":")) for r in edges)   # one edge frame per line
    open(path, "w").write(text.replace('"EDGES"', "[\n  " + rows + "\n ]"))
    print("wrote", path, len(recs), "cases", len(edges), "edge frames")


if __name__ == "__main__":
    main()
