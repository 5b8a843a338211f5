"""The raw gossip frames of tests/golden/proto_wire.json "edges": frames at protobuf's varint, enum, length and nesting edges.

The fixture records protobuf's answers for each frame by name (and the Keccak-256 of the frame); the frames themselves are built
here, by the generator (tests/golden/make_proto_golden.py) and by the tests alike.  Each base frame is a function of its
signature TLV and is signed by validator 0 of the fixture's table twice: over "frame minus the signature TLV" (the bytes the
device hashes) and over protobuf-go's PayloadNoSig (the bytes go-ibft hashes), whose digest the fixture records."""
import workloads as wl
from oracle import coracle as co
from oracle import ibft_proto as ip

EDGE_SEED, EDGE_VALIDATORS = 91, 4
EDGE_HASH = bytes(range(0x40, 0x60))


def _vmin(v):
    return ip._varint(v)


def _vwidth(v, w):
    """v in exactly w bytes (non-minimal when w is longer than needed)"""
    out = bytearray(((v >> (7 * i)) & 0x7F) | (0x80 if i < w - 1 else 0) for i in range(w))
    assert v >> (7 * w) == 0 or w == 10
    return bytes(out)


def _v10(low63, last):
    """a 10-byte varint: the low 63 bits of low63 in nine groups, then the raw byte `last`"""
    return bytes(((low63 >> (7 * i)) & 0x7F) | 0x80 for i in range(9)) + bytes([last])


def _varint_encodings(value_ok=True):
    """(label, encoding) pairs: minimal 1..10-byte values, 10-byte forms with every interesting last byte, non-minimal small values"""
    out = []
    if value_ok:
        for k in range(10):
            v = 1 << (7 * k)
            out.append(("min%d_2^%d" % (k + 1, 7 * k), _vmin(v)))
        out += [("min10_2^64-1", _vmin(2**64 - 1)), ("min5_2^32+5", _vmin(2**32 + 5))]
    for last, lab in ((0x00, "00"), (0x01, "01"), (0x02, "02"), (0x7F, "7f")):
        out.append(("ten_last%s" % lab, _v10(5, last)))
    out.append(("ten_last80_eleven01", _v10(5, 0x80) + b"\x01"))
    out += [("nonmin2_of5", _vwidth(5, 2)), ("nonmin3_of5", _vwidth(5, 3)), ("nonmin10_of5", _vwidth(5, 10))]
    return out


class EdgeFrames:
    def __init__(self):
        self.vs = wl.ValidatorSet(EDGE_SEED, EDGE_VALIDATORS)
        self.frm = self.vs.addrs[0]
        self.seal = wl.sign(self.vs.keys[0], wl.seal_digest(EDGE_HASH))

    @staticmethod
    def tlv(key: bytes, body: bytes, length: bytes = None):
        return key + (_vmin(len(body)) if length is None else length) + body

    def view(self, h=_vmin(100), r=_vmin(3), hkey=b"\x08", rkey=b"\x10"):
        return (hkey + h if h is not None else b"") + (rkey + r if r is not None else b"")

    def commit(self, view=None, type_enc=_vmin(2), type_key=b"\x20", body_len=None, tail=b"", view_len=None):
        """COMMIT frame as a function of its signature TLV (b"" = unsigned); type_enc None = no type field"""
        v = self.view() if view is None else view
        body = self.tlv(b"\x0a", EDGE_HASH) + self.tlv(b"\x12", self.seal)
        head = self.tlv(b"\x0a", v, view_len) + self.tlv(b"\x12", self.frm)
        rest = (type_key + type_enc if type_enc is not None else b"") + self.tlv(b"\x3a", body, body_len) + tail
        return lambda sig: head + sig + rest

    def prepare_view_last(self, view, view_len=None):
        """PREPARE frame whose view is its LAST field (a varint cut short inside the view runs into the end of the frame)"""
        head = self.tlv(b"\x12", self.frm)
        rest = b"\x20\x01" + self.tlv(b"\x32", self.tlv(b"\x0a", EDGE_HASH)) + self.tlv(b"\x0a", view, view_len)
        return lambda sig: head + sig + rest

    def preprepare(self, round_enc, raw=b"proposal"):
        prop = self.tlv(b"\x0a", raw) + (b"\x10" + round_enc if round_enc is not None else b"")
        body = self.tlv(b"\x0a", prop) + self.tlv(b"\x12", EDGE_HASH)
        head = self.tlv(b"\x0a", self.view()) + self.tlv(b"\x12", self.frm)
        rest = self.tlv(b"\x2a", body)
        return lambda sig: head + sig + rest

    def model_frame(self, m: ip.IbftMessage):
        """a frame built from the oracle model (canonical for in-range values); the signature TLV goes after `from`"""
        m.signature = b""
        enc = ip.encode_ibft_message(m)
        cut = len(ip._f_msg(1, ip.encode_view(m.view)) + ip._f_bytes(2, m.from_))
        return lambda sig: enc[:cut] + sig + enc[cut:]

    def bases(self):
        """(name, frame-of-signature-TLV)"""
        out = []
        vmin = _vmin
        # -- varints at every position the walker reads one
        for lab, e in _varint_encodings():
            out.append(("height_" + lab, self.commit(view=self.view(h=e))))
            out.append(("round_" + lab, self.commit(view=self.view(r=e))))
            out.append(("type_" + lab, self.commit(type_enc=e)))
            out.append(("proposal_round_" + lab, self.preprepare(e)))
        for lab, e in [("min1_2", vmin(2)), ("min5_2^32+2", vmin(2**32 + 2)), ("min10_2^63+2", vmin(2**63 + 2)), ("nonmin2_of2", _vwidth(2, 2)),
                       ("ten_last00_of2", _v10(2, 0)), ("ten_last01_of2", _v10(2, 1)), ("ten_last02_of2", _v10(2, 2))]:
            out.append(("type_commit_" + lab, self.commit(type_enc=e)))
        # the tag of `type` (0x20 = field 4, varint)
        for w in range(2, 11):
            out.append(("tag_nonmin%d" % w, self.commit(type_key=_vwidth(0x20, w))))
        for last, lab in ((0x00, "00"), (0x01, "01"), (0x02, "02"), (0x7F, "7f")):
            out.append(("tag_ten_last" + lab, self.commit(type_key=_v10(0x20, last))))
        out.append(("tag_ten_last80_eleven01", self.commit(type_key=_v10(0x20, 0x80) + b"\x01")))
        # a length prefix (commitData's, the last field of the frame; the view's, a sub-message in the middle)
        body_len = 2 + 32 + 2 + 65
        for w in range(1, 11):
            out.append(("len_width%d" % w, self.commit(body_len=_vwidth(body_len, w))))
        for last, lab in ((0x01, "01"), (0x02, "02"), (0x7F, "7f")):
            out.append(("len_ten_last" + lab, self.commit(body_len=_v10(body_len, last))))
        out.append(("len_ten_last80_eleven01", self.commit(body_len=_v10(body_len, 0x80) + b"\x01")))
        out.append(("len_one_past_frame", self.commit(body_len=vmin(body_len + 1))))
        out.append(("len_one_short", self.commit(body_len=vmin(body_len - 1))))
        out.append(("len_2^32_plus_len_5byte", self.commit(body_len=vmin(2**32 + body_len))))
        out.append(("len_2^32_plus_len_10byte", self.commit(body_len=_vwidth(2**32 + body_len, 10))))
        out.append(("len_2^63_plus_len", self.commit(body_len=vmin(2**63 + body_len))))
        vlen = len(self.view())
        out.append(("view_len_exact", self.commit(view_len=vmin(vlen))))
        out.append(("view_len_one_past", self.commit(view_len=vmin(vlen + 1))))
        out.append(("view_len_one_short", self.commit(view_len=vmin(vlen - 1))))
        out.append(("view_len_2^32_plus_len", self.commit(view_len=vmin(2**32 + vlen))))
        # varints cut short: at the end of a sub-message and at the end of the frame
        for lab, e in [("2", b"\x80"), ("10", _vmin(2**64 - 1)[:9]), ("ten_last80", _v10(5, 0x80))]:
            out.append(("trunc_height_end_of_view_" + lab, self.commit(view=self.view(h=e, r=None))))
            out.append(("trunc_round_end_of_view_" + lab, self.commit(view=self.view(r=e))))
            out.append(("trunc_round_end_of_frame_" + lab, self.prepare_view_last(self.view(r=e))))
            out.append(("trunc_proposal_round_end_of_proposal_" + lab, self.preprepare(e)))
            out.append(("trunc_type_end_of_frame_" + lab, lambda sig, e=e: self.commit()(sig)[: -(2 + 2 + 32 + 2 + 65 + 2)] + b"\x20" + e))
            out.append(("trunc_tag_end_of_frame_" + lab, self.commit(tail=e)))
            out.append(("trunc_len_end_of_frame_" + lab, self.commit(tail=b"\x12" + e)))
        # -- `type` at the int32 boundaries, at depth 0 and inside certificate messages at depths 3 and 6
        types = [("1", 1), ("2^31-1", 2**31 - 1), ("2^31", 2**31), ("2^32-1", 2**32 - 1), ("2^32", 2**32), ("2^32+1", 2**32 + 1),
                 ("2^32+2", 2**32 + 2), ("2^64-1", 2**64 - 1), ("2^64-2", 2**64 - 2), ("2^63", 2**63)]
        for lab, t in types:
            out.append(("type_depth0_" + lab, self.commit(type_enc=vmin(t))))
            out.append(("type_depth3_" + lab, self.model_frame(self.nested_type(t, 3))))
            out.append(("type_depth6_" + lab, self.model_frame(self.nested_type(t, 6))))
        # -- nesting: canonical frames 8 (the deepest a legitimate frame needs), 11, 12, 13 and 14 levels deep
        for levels in (8, 11, 12, 13, 14):
            out.append(("nesting_levels_%d" % levels, self.model_frame(self.nested_chain(levels))))
        return out

    def _msg(self, t, payload, k=1):
        return ip.IbftMessage(ip.View(100, 3), self.vs.addrs[k], b"\x05" * 65, t, payload)

    def nested_type(self, t, depth):
        """top PREPREPARE (depth 0) -> PrePrepareMessage -> RCC -> ROUND_CHANGE (depth 3) -> RoundChangeMessage -> PC -> PREPARE (depth 6);
        the message at `depth` carries type t"""
        inner = self._msg(t if depth == 6 else ip.PREPARE, ip.PrepareMessage(EDGE_HASH), 2)
        rc = self._msg(t if depth == 3 else ip.ROUND_CHANGE, ip.RoundChangeMessage(ip.Proposal(b"p", 0), ip.PreparedCertificate(None, [inner])), 1)
        return ip.IbftMessage(ip.View(100, 4), self.frm, b"", ip.PREPREPARE,
                              ip.PrePrepareMessage(ip.Proposal(b"proposal", 4), EDGE_HASH, ip.RoundChangeCertificate([rc])))

    def nested_chain(self, levels):
        """PREPREPARE -> RCC -> ROUND_CHANGE -> PC -> PREPREPARE -> ... whose deepest sub-message sits `levels` levels down (root = 1)"""
        # levels of a message at level L: PREPREPARE with a proposal reaches L + 2; each hop (IbftMessage -> payload ->
        # certificate -> IbftMessage) adds 3; a bare IbftMessage with a view reaches L + 1
        def build(lv, kind):
            if lv <= 2:
                return ip.IbftMessage(ip.View(100, 3), self.vs.addrs[1], b"\x05" * 65, ip.PREPARE, None)
            if lv == 3:
                return self._msg(ip.PREPREPARE, ip.PrePrepareMessage(ip.Proposal(b"p", 1), EDGE_HASH, None))
            if lv == 4:  # view (2), payload (2), certificate (3), an empty RCC message list -> PC with an empty message (4)
                return self._msg(ip.ROUND_CHANGE, ip.RoundChangeMessage(None, ip.PreparedCertificate(ip.IbftMessage(), None)))
            if kind == "pp":
                return self._msg(ip.PREPREPARE, ip.PrePrepareMessage(ip.Proposal(b"p", 1), EDGE_HASH,
                                                                     ip.RoundChangeCertificate([build(lv - 3, "rc")])))
            return self._msg(ip.ROUND_CHANGE, ip.RoundChangeMessage(ip.Proposal(b"p", 1), ip.PreparedCertificate(build(lv - 3, "pp"), None)))
        inner = build(levels - 3, "rc")
        return ip.IbftMessage(ip.View(100, 4), self.frm, b"", ip.PREPREPARE,
                              ip.PrePrepareMessage(ip.Proposal(b"proposal", 4), EDGE_HASH, ip.RoundChangeCertificate([inner])))


def sig_tlv(sig: bytes) -> bytes:
    return b"\x1a\x41" + sig


def signed_variants(body, key: int, go_digest):
    """(variant, frame) pairs of one base frame; go_digest = Keccak-256 of protobuf-go's PayloadNoSig (None: Go cannot decode it).
    The second variant exists only where the two signed byte strings differ, i.e. where the frame is not canonical."""
    cut = body(sig_tlv(wl.sign(key, co.keccak256(body(b"")))))
    out = [("signed_over_frame_minus_sig", cut)]
    if go_digest is not None:
        go = body(sig_tlv(wl.sign(key, go_digest)))
        if go != cut:
            out.append(("signed_over_go_payload_no_sig", go))
    return out
