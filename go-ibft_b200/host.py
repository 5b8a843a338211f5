"""ctypes binding of go-ibft_b200/host/libibfthost.so -- the C++ host-side mirror of the reference interfaces around the
hot path (proto codec, message store + batching shim, ValidatorManager, IBFT validation predicates, verifiers).

verifier kinds: "callback" (Python closures, the reference's mockBackend semantics) and "gpu" (C ABI -> CUDA kernels; fails
loudly without a device)."""
from __future__ import annotations

import ctypes
import os
import subprocess
from ctypes import CFUNCTYPE, POINTER, c_char_p, c_int, c_size_t, c_uint8, c_uint32, c_uint64, c_void_p

from . import build as _build
from .engine import EngineParams

HERE = os.path.dirname(os.path.abspath(__file__))
HOST_DIR = os.path.join(HERE, "host")
LIB = os.path.join(HOST_DIR, "libibfthost.so")

CB_VALID_PROPOSAL = CFUNCTYPE(c_int, POINTER(c_uint8), c_size_t)
CB_VALID_VALIDATOR = CFUNCTYPE(c_int, POINTER(c_uint8), c_size_t)
CB_PROPOSER = CFUNCTYPE(c_int, POINTER(c_uint8), c_size_t, c_uint64, c_uint64)
CB_PROPOSAL_HASH = CFUNCTYPE(c_int, POINTER(c_uint8), c_size_t, c_int, POINTER(c_uint8), c_size_t, c_int)
CB_SEAL = CFUNCTYPE(c_int, POINTER(c_uint8), c_size_t, c_int, POINTER(c_uint8), c_size_t, POINTER(c_uint8), c_size_t, c_int)
CB_REJECT = CFUNCTYPE(None, c_void_p, c_uint8, c_uint64, POINTER(c_uint8), c_size_t, POINTER(c_uint8), c_size_t, c_uint8, POINTER(c_uint8))


class Callbacks(ctypes.Structure):
    _fields_ = [("is_valid_proposal", CB_VALID_PROPOSAL), ("is_valid_validator", CB_VALID_VALIDATOR), ("is_proposer", CB_PROPOSER),
                ("is_valid_proposal_hash", CB_PROPOSAL_HASH), ("is_valid_committed_seal", CB_SEAL)]


_LIB = None


def build_host() -> str:
    _build.build()
    subprocess.check_call(["make", "-C", HOST_DIR, "-s"])
    return LIB


def load_host() -> ctypes.CDLL:
    global _LIB
    if _LIB is None:
        lib = ctypes.CDLL(build_host())
        lib.ibfthost_create.restype = c_void_p
        lib.ibfthost_create.argtypes = [c_int, POINTER(Callbacks), c_char_p, c_size_t, POINTER(EngineParams)]
        lib.ibfthost_create_multi.restype = c_void_p
        lib.ibfthost_create_multi.argtypes = [POINTER(Callbacks), c_char_p, c_size_t, POINTER(EngineParams), c_void_p, c_uint32]
        lib.ibfthost_destroy.argtypes = [c_void_p]
        lib.ibfthost_destroy.restype = None
        lib.ibfthost_set_validators.argtypes = [c_void_p, c_uint64, c_char_p, POINTER(c_uint32), c_char_p, c_uint32]
        lib.ibfthost_set_batching.argtypes = [c_void_p, c_int]
        lib.ibfthost_set_batching.restype = None
        lib.ibfthost_verify_committed_seals.argtypes = [c_void_p, c_char_p, c_size_t, c_char_p, c_char_p, c_uint32, POINTER(c_uint32)]
        lib.ibfthost_set_incremental_quorum.argtypes = [c_void_p, c_int]
        lib.ibfthost_set_incremental_quorum.restype = None
        lib.ibfthost_set_wire_frames.argtypes = [c_void_p, c_int]
        lib.ibfthost_set_wire_frames.restype = None
        lib.ibfthost_gpu_frames_handed_back.argtypes = [c_void_p]
        lib.ibfthost_gpu_frames_handed_back.restype = c_uint64
        lib.ibfthost_set_reject_hook.argtypes = [c_void_p, CB_REJECT, c_void_p]
        lib.ibfthost_set_reject_hook.restype = None
        lib.ibfthost_gpu_rejects.argtypes = [c_void_p, c_uint32]
        lib.ibfthost_gpu_rejects.restype = c_uint64
        lib.ibfthost_gpu_explain_calls.argtypes = [c_void_p]
        lib.ibfthost_gpu_explain_calls.restype = c_uint64
        lib.ibfthost_set_state.argtypes = [c_void_p, c_uint64, c_uint64, c_int, c_char_p, c_size_t]
        lib.ibfthost_get_state_name.argtypes = [c_void_p]
        for f in ("ibfthost_store_add", "ibfthost_add_message", "ibfthost_is_acceptable", "ibfthost_is_valid_validator"):
            getattr(lib, f).argtypes = [c_void_p, c_char_p, c_size_t]
        lib.ibfthost_add_messages.argtypes = [c_void_p, c_char_p, POINTER(c_uint32), c_uint32]
        lib.ibfthost_num_messages.argtypes = [c_void_p, c_uint64, c_uint64, c_uint32]
        lib.ibfthost_num_messages.restype = c_uint64
        lib.ibfthost_prune_by_height.argtypes = [c_void_p, c_uint64]
        lib.ibfthost_prune_by_height.restype = None
        lib.ibfthost_ingress_storm.argtypes = [c_void_p, c_char_p, POINTER(c_uint32), c_uint32, c_uint32, c_void_p, c_void_p]
        lib.ibfthost_ingress_storm.restype = ctypes.c_double
        lib.ibfthost_set_ingress.argtypes = [c_void_p, c_uint32, c_uint32, c_uint32]
        lib.ibfthost_set_ingress.restype = None
        for f in ("ibfthost_signal_count", "ibfthost_seal_count", "ibfthost_latest_pc_prepares", "ibfthost_gpu_device_calls", "ibfthost_gpu_items_verified",
                  "ibfthost_gpu_ingress_requests", "ibfthost_gpu_ingress_flushes"):
            getattr(lib, f).argtypes = [c_void_p]
            getattr(lib, f).restype = c_uint64
        lib.ibfthost_handle_commit.argtypes = [c_void_p, c_uint64, c_uint64]
        lib.ibfthost_handle_prepare.argtypes = [c_void_p, c_uint64, c_uint64]
        lib.ibfthost_handle_preprepare.argtypes = [c_void_p, c_uint64, c_uint64, c_char_p, c_size_t]
        lib.ibfthost_handle_round_change.argtypes = [c_void_p, c_uint64, c_uint64, c_char_p, c_size_t]
        lib.ibfthost_store_senders.argtypes = [c_void_p, c_uint64, c_uint64, c_uint32, c_char_p, c_size_t]
        lib.ibfthost_valid_pc.argtypes = [c_void_p, c_char_p, c_size_t, c_int, c_uint64, c_uint64]
        lib.ibfthost_validate_proposal.argtypes = [c_void_p, c_char_p, c_size_t, c_uint64, c_uint64]
        lib.ibfthost_has_quorum_senders.argtypes = [c_void_p, c_char_p, POINTER(c_uint32), c_uint32]
        lib.ibfthost_has_quorum_voted.argtypes = [c_void_p, c_void_p, c_uint32]
        lib.ibfthost_reencode.argtypes = [c_char_p, c_size_t, c_int, c_char_p, c_size_t]
        lib.ibfthost_reencode.restype = c_size_t
        lib.ibfthost_remarshal.argtypes = [c_char_p, c_size_t, c_int, c_char_p, c_size_t]
        lib.ibfthost_remarshal.restype = c_size_t
        lib.ibfthost_is_valid_committed_seal.argtypes = [c_void_p, c_char_p, c_size_t, c_char_p, c_size_t, c_char_p, c_size_t]
        lib.ibfthost_is_valid_proposal_hash.argtypes = [c_void_p, c_char_p, c_size_t, c_uint64, c_int, c_char_p, c_size_t]
        _LIB = lib
    return _LIB


def _bytes(p, n):
    return bytes(ctypes.cast(p, POINTER(c_uint8 * n)).contents) if (p and n) else b""


def reencode(wire: bytes, with_signature: bool = True):
    lib = load_host()
    buf = ctypes.create_string_buffer(len(wire) + 16)
    n = lib.ibfthost_reencode(wire, len(wire), int(with_signature), buf, len(buf))
    if n == ctypes.c_size_t(-1).value:
        return None
    return buf.raw[:n]


def remarshal(wire: bytes, with_signature: bool = True):
    """protobuf-go's Marshal(Unmarshal(wire)) restated by the C++ host codec (unknown fields kept, duplicates merged); None on a
    parse error.  with_signature=False: PayloadNoSig of a message that arrived as `wire`."""
    lib = load_host()
    n = lib.ibfthost_remarshal(wire, len(wire), int(with_signature), None, 0)
    if n == ctypes.c_size_t(-1).value:
        return None
    buf = ctypes.create_string_buffer(max(1, n))
    lib.ibfthost_remarshal(wire, len(wire), int(with_signature), buf, n)
    return buf.raw[:n]


class HostContext:
    """kind="callback": fns = dict of Python closures taking decoded arguments:
         is_valid_proposal(raw) / is_valid_validator(wire) / is_proposer(id, h, r) / is_valid_proposal_hash(proposal_wire|None, hash|None)
         / is_valid_committed_seal(hash|None, (signer, sig)|None)
       kind="gpu": is_proposer / is_valid_proposal closures only; signature work goes to the device -- to the devices listed in
       `devices` (one engine over all of them, ibft_engine_create_multi) when given."""

    def __init__(self, kind: str = "callback", fns: dict | None = None, node_id: bytes = b"", gpu_params: EngineParams | None = None,
                 devices: list[int] | None = None):
        self.lib = load_host()
        fns = fns or {}
        self._keep = []
        cbs = Callbacks()

        def wrap(tp, f):
            cb = tp(f)
            self._keep.append(cb)
            return cb
        if "is_valid_proposal" in fns:
            cbs.is_valid_proposal = wrap(CB_VALID_PROPOSAL, lambda p, n: int(bool(fns["is_valid_proposal"](_bytes(p, n)))))
        if "is_valid_validator" in fns:
            cbs.is_valid_validator = wrap(CB_VALID_VALIDATOR, lambda p, n: int(bool(fns["is_valid_validator"](_bytes(p, n)))))
        if "is_proposer" in fns:
            cbs.is_proposer = wrap(CB_PROPOSER, lambda p, n, h, r: int(bool(fns["is_proposer"](_bytes(p, n), h, r))))
        if "is_valid_proposal_hash" in fns:
            cbs.is_valid_proposal_hash = wrap(CB_PROPOSAL_HASH, lambda p, n, hp, h, hn, hh: int(bool(
                fns["is_valid_proposal_hash"](_bytes(p, n) if hp else None, _bytes(h, hn) if hh else None))))
        if "is_valid_committed_seal" in fns:
            cbs.is_valid_committed_seal = wrap(CB_SEAL, lambda h, hn, hh, s, sn, g, gn, hs: int(bool(
                fns["is_valid_committed_seal"](_bytes(h, hn) if hh else None, (_bytes(s, sn), _bytes(g, gn)) if hs else None))))
        if devices:
            if kind != "gpu" or gpu_params is None:
                raise ValueError("devices needs kind='gpu' and gpu_params")
            devs = (ctypes.c_int32 * len(devices))(*[int(d) for d in devices])
            self.ctx = self.lib.ibfthost_create_multi(ctypes.byref(cbs), node_id, len(node_id), ctypes.byref(gpu_params), devs, len(devices))
        else:
            self.ctx = self.lib.ibfthost_create(0 if kind == "callback" else 1, ctypes.byref(cbs), node_id, len(node_id),
                                                ctypes.byref(gpu_params) if gpu_params is not None else None)
        if not self.ctx:
            raise RuntimeError("ibfthost_create failed (a GPU verifier needs a CUDA device: there is no CPU fallback)")

    def close(self):
        if getattr(self, "ctx", None):
            self.lib.ibfthost_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _pack(items):
        lens = (c_uint32 * max(1, len(items)))(*[len(b) for b in items])
        return b"".join(items), lens

    def set_validators(self, height: int, addrs: list[bytes], powers: list[int] | None = None) -> int:
        blob, lens = self._pack(addrs)
        pw = b"".join(p.to_bytes(32, "big") for p in powers) if powers is not None else None
        return self.lib.ibfthost_set_validators(self.ctx, height, blob, lens, pw, len(addrs))

    def set_batching(self, on: bool):
        self.lib.ibfthost_set_batching(self.ctx, int(on))

    def set_incremental_quorum(self, on: bool):
        self.lib.ibfthost_set_incremental_quorum(self.ctx, int(on))

    def set_wire_frames(self, on: bool):
        self.lib.ibfthost_set_wire_frames(self.ctx, int(on))

    def set_reject_hook(self, fn):
        """GpuVerifier::onReject: fn(kind, height, message, from_, reason, recovered) once per rejected item -- kind IBFT_KIND_PAYLOAD /
        _WIRE (IsValidValidator: message = PayloadNoSig / the raw frame) or _SEAL (IsValidCommittedSeal: message = the proposal
        hash), reason REASON_*, recovered = the recovered address (20 bytes, zero when recovery was not reached).  None removes it."""
        if fn is None:
            self._reject_cb = None
            self.lib.ibfthost_set_reject_hook(self.ctx, CB_REJECT(), None)
            return
        self._reject_cb = CB_REJECT(lambda _u, kind, h, m, mn, f, fn_, reason, rec: fn(kind, h, _bytes(m, mn), _bytes(f, fn_), reason,
                                                                                        _bytes(rec, 20)))
        self.lib.ibfthost_set_reject_hook(self.ctx, self._reject_cb, None)

    def gpu_rejects(self, reason: int) -> int:
        return int(self.lib.ibfthost_gpu_rejects(self.ctx, reason))

    def gpu_explain_calls(self) -> int:
        return int(self.lib.ibfthost_gpu_explain_calls(self.ctx))

    def gpu_frames_handed_back(self) -> int:
        return int(self.lib.ibfthost_gpu_frames_handed_back(self.ctx))

    def set_state(self, height: int, rnd: int, state_name: int = 0, proposal_wire: bytes | None = None) -> int:
        return self.lib.ibfthost_set_state(self.ctx, height, rnd, state_name, proposal_wire, len(proposal_wire) if proposal_wire else 0)

    def state_name(self) -> int:
        return self.lib.ibfthost_get_state_name(self.ctx)

    def store_add(self, wire: bytes):
        return self.lib.ibfthost_store_add(self.ctx, wire, len(wire))

    def add_message(self, wire: bytes):
        return self.lib.ibfthost_add_message(self.ctx, wire, len(wire))

    def add_messages(self, wires: list[bytes]):
        blob, lens = self._pack(wires)
        return self.lib.ibfthost_add_messages(self.ctx, blob, lens, len(wires))

    def is_acceptable(self, wire: bytes) -> bool:
        return bool(self.lib.ibfthost_is_acceptable(self.ctx, wire, len(wire)))

    def num_messages(self, h, r, t) -> int:
        return int(self.lib.ibfthost_num_messages(self.ctx, h, r, t))

    def prune_by_height(self, h):
        self.lib.ibfthost_prune_by_height(self.ctx, h)

    def signal_count(self) -> int:
        return int(self.lib.ibfthost_signal_count(self.ctx))

    def _senders(self, fn, *args):
        buf = ctypes.create_string_buffer(1 << 22)
        rc = fn(self.ctx, *args, buf, len(buf))
        txt = buf.value.decode()
        return rc, sorted(bytes.fromhex(x) for x in txt.split("\n") if x != "") if rc > 0 else []

    def handle_commit(self, h, r) -> bool:
        return bool(self.lib.ibfthost_handle_commit(self.ctx, h, r))

    def handle_prepare(self, h, r) -> bool:
        return bool(self.lib.ibfthost_handle_prepare(self.ctx, h, r))

    def handle_preprepare(self, h, r):
        rc, s = self._senders(self.lib.ibfthost_handle_preprepare, h, r)
        return s[0] if rc else None

    def handle_round_change(self, h, r):
        rc, s = self._senders(self.lib.ibfthost_handle_round_change, h, r)
        return None if rc < 0 else s

    def store_senders(self, h, r, t):
        rc, s = self._senders(self.lib.ibfthost_store_senders, h, r, t)
        return s

    def seal_count(self) -> int:
        return int(self.lib.ibfthost_seal_count(self.ctx))

    def latest_pc_prepares(self) -> int:
        return int(self.lib.ibfthost_latest_pc_prepares(self.ctx))

    def valid_pc(self, pc_wire: bytes | None, round_limit: int, height: int) -> bool:
        return bool(self.lib.ibfthost_valid_pc(self.ctx, pc_wire, len(pc_wire) if pc_wire else 0, int(pc_wire is not None), round_limit, height))

    def validate_proposal(self, wire: bytes, h: int, r: int) -> bool:
        return bool(self.lib.ibfthost_validate_proposal(self.ctx, wire, len(wire), h, r))

    def has_quorum_senders(self, addrs: list[bytes]) -> bool:
        blob, lens = self._pack(addrs)
        return bool(self.lib.ibfthost_has_quorum_senders(self.ctx, blob, lens, len(addrs)))

    def has_quorum_voted(self, words) -> bool:
        import numpy as np
        w = np.ascontiguousarray(words, dtype=np.uint32)
        return bool(self.lib.ibfthost_has_quorum_voted(self.ctx, w.ctypes.data_as(c_void_p), len(w)))

    def is_valid_validator(self, wire: bytes) -> bool:
        return bool(self.lib.ibfthost_is_valid_validator(self.ctx, wire, len(wire)))

    def is_valid_committed_seal(self, phash: bytes | None, signer: bytes | None, sig: bytes = b"") -> bool:
        return bool(self.lib.ibfthost_is_valid_committed_seal(self.ctx, phash, len(phash) if phash else 0, signer,
                                                              len(signer) if signer else 0, sig, len(sig)))

    def is_valid_proposal_hash(self, raw: bytes | None, rnd: int, phash: bytes | None) -> bool:
        return bool(self.lib.ibfthost_is_valid_proposal_hash(self.ctx, raw or b"", len(raw) if raw else 0, rnd, int(raw is not None),
                                                             phash, len(phash) if phash else 0))

    def verify_committed_seals(self, phash: bytes, seals: list[tuple[bytes, bytes]]):
        """InsertProposal-side check: (has_quorum, n_valid) for (signer, signature) pairs over one proposal hash."""
        nv = c_uint32()
        rc = self.lib.ibfthost_verify_committed_seals(self.ctx, phash, len(phash), b"".join(s for s, _ in seals),
                                                      b"".join(g for _, g in seals), len(seals), ctypes.byref(nv))
        return bool(rc == 1), int(nv.value)

    def gpu_device_calls(self) -> int:
        return int(self.lib.ibfthost_gpu_device_calls(self.ctx))

    def gpu_items_verified(self) -> int:
        return int(self.lib.ibfthost_gpu_items_verified(self.ctx))

    # ---- ingress coalescer (single-message IsValidValidator calls from many threads)
    def set_ingress(self, max_batch: int = 4096, min_batch: int = 1, linger_us: int = 0):
        self.lib.ibfthost_set_ingress(self.ctx, max_batch, min_batch, linger_us)

    def ingress_storm(self, wires: list[bytes], threads: int):
        """Every wire message is checked with ONE single-message IsValidValidator call, from `threads` concurrent native
        threads.  Returns (verdicts uint8[n], per-call latency in us float32[n], elapsed us)."""
        import numpy as np
        n = len(wires)
        lens = (c_uint32 * n)(*[len(w) for w in wires])
        verdicts = np.zeros(n, dtype=np.uint8)
        lat = np.zeros(n, dtype=np.float32)
        us = self.lib.ibfthost_ingress_storm(self.ctx, b"".join(wires), lens, n, threads, verdicts.ctypes.data_as(c_void_p),
                                             lat.ctypes.data_as(c_void_p))
        if us < 0:
            raise ValueError("undecodable wire message")
        return verdicts, lat, float(us)

    def gpu_ingress_requests(self) -> int:
        return int(self.lib.ibfthost_gpu_ingress_requests(self.ctx))

    def gpu_ingress_flushes(self) -> int:
        return int(self.lib.ibfthost_gpu_ingress_flushes(self.ctx))
