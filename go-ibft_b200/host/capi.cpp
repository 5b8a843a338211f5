// capi.cpp -- C entry points over the host-side mirror (proto codec, store, validator manager, IBFT predicates, verifiers).
//
// Purpose: (1) the parity tests drive the C++ host logic and oracle/ibft_logic.py with identical wire bytes and compare
// every decision (tests/test_host_logic.py); (2) it is the shape of the calls the Go shim makes (INTEGRATION.md).
// Verifier kinds: 0 = callback verifier (function pointers; the reference's mockBackend), 1 = GPU verifier (C ABI ->
// CUDA kernels).  Everything is plain C types; byte strings are (ptr, len); variable-size outputs use caller buffers.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <thread>

#include "ibft_logic.hpp"

using namespace ibft::host;

extern "C" {

typedef int (*cb_is_valid_validator)(const uint8_t* wire, size_t len);
typedef int (*cb_is_proposer)(const uint8_t* id, size_t len, uint64_t height, uint64_t round);
typedef int (*cb_is_valid_proposal_hash)(const uint8_t* proposal_wire, size_t plen, int has_proposal, const uint8_t* hash, size_t hlen, int has_hash);
typedef int (*cb_is_valid_committed_seal)(const uint8_t* hash, size_t hlen, int has_hash, const uint8_t* signer, size_t slen,
                                          const uint8_t* sig, size_t siglen, int has_seal);
typedef int (*cb_is_valid_proposal)(const uint8_t* raw, size_t len);

struct ibfthost_callbacks {
  cb_is_valid_proposal is_valid_proposal;
  cb_is_valid_validator is_valid_validator;
  cb_is_proposer is_proposer;
  cb_is_valid_proposal_hash is_valid_proposal_hash;
  cb_is_valid_committed_seal is_valid_committed_seal;
};

struct ibfthost_ctx {
  std::unique_ptr<Verifier> verifier;
  GpuVerifier* gpu = nullptr;
  ValidatorManager vm;
  Messages messages;
  std::unique_ptr<IBFT> ibft;
  std::vector<uint64_t> signals;  // (type, height, round) triples
  std::string last_out;
};

static Bytes B(const uint8_t* p, size_t n) { return p ? Bytes((const char*)p, n) : Bytes(); }

static ibfthost_ctx* create_ctx(int kind, const ibfthost_callbacks* cbs, const uint8_t* id, size_t id_len,
                                const ibft_engine_params* gpu_params, const std::vector<int32_t>& devices) {
  auto* c = new ibfthost_ctx();
  if (kind == 0) {
    auto v = std::make_unique<CallbackVerifier>();
    v->id = B(id, id_len);
    if (cbs) {
      ibfthost_callbacks k = *cbs;
      if (k.is_valid_proposal) v->isValidProposalFn = [k](const Bytes& raw) { return k.is_valid_proposal((const uint8_t*)raw.data(), raw.size()) != 0; };
      if (k.is_valid_validator)
        v->isValidValidatorFn = [k](const IbftMessage& m) {
          Bytes w = encode_message(m);
          return k.is_valid_validator((const uint8_t*)w.data(), w.size()) != 0;
        };
      if (k.is_proposer) v->isProposerFn = [k](const Bytes& i, uint64_t h, uint64_t r) { return k.is_proposer((const uint8_t*)i.data(), i.size(), h, r) != 0; };
      if (k.is_valid_proposal_hash)
        v->isValidProposalHashFn = [k](const Proposal* p, const Bytes* h) {
          Bytes w = p ? encode_proposal(*p) : Bytes();
          return k.is_valid_proposal_hash((const uint8_t*)w.data(), w.size(), p != nullptr, h ? (const uint8_t*)h->data() : nullptr,
                                          h ? h->size() : 0, h != nullptr) != 0;
        };
      if (k.is_valid_committed_seal)
        v->isValidCommittedSealFn = [k](const Bytes* h, const CommittedSeal* s) {
          return k.is_valid_committed_seal(h ? (const uint8_t*)h->data() : nullptr, h ? h->size() : 0, h != nullptr,
                                           s ? (const uint8_t*)s->signer.data() : nullptr, s ? s->signer.size() : 0,
                                           s ? (const uint8_t*)s->signature.data() : nullptr, s ? s->signature.size() : 0, s != nullptr) != 0;
        };
    }
    c->verifier = std::move(v);
  } else {
    if (!gpu_params) { delete c; return nullptr; }
    auto v = std::make_unique<GpuVerifier>(*gpu_params, devices);
    if (!v->ok()) { delete c; return nullptr; }  // no CPU fallback: no engine, no context
    v->id = B(id, id_len);
    if (cbs && cbs->is_proposer) {
      auto f = cbs->is_proposer;
      v->isProposerFn = [f](const Bytes& i, uint64_t h, uint64_t r) { return f((const uint8_t*)i.data(), i.size(), h, r) != 0; };
    }
    if (cbs && cbs->is_valid_proposal) {
      auto f = cbs->is_valid_proposal;
      v->isValidProposalFn = [f](const Bytes& raw) { return f((const uint8_t*)raw.data(), raw.size()) != 0; };
    }
    c->gpu = v.get();
    c->verifier = std::move(v);
  }
  c->ibft = std::make_unique<IBFT>(*c->verifier, c->vm, c->messages);
  c->messages.on_signal = [c](uint32_t t, uint64_t h, uint64_t r) {
    c->signals.push_back(t);
    c->signals.push_back(h);
    c->signals.push_back(r);
  };
  return c;
}
ibfthost_ctx* ibfthost_create(int kind, const ibfthost_callbacks* cbs, const uint8_t* id, size_t id_len,
                              const ibft_engine_params* gpu_params) {
  return create_ctx(kind, cbs, id, id_len, gpu_params, {});
}
// a GPU verifier over several devices (ibft_engine_create_multi)
ibfthost_ctx* ibfthost_create_multi(const ibfthost_callbacks* cbs, const uint8_t* id, size_t id_len, const ibft_engine_params* gpu_params,
                                    const int32_t* devices, uint32_t n_devices) {
  if (!devices || n_devices == 0) return nullptr;
  return create_ctx(1, cbs, id, id_len, gpu_params, std::vector<int32_t>(devices, devices + n_devices));
}
void ibfthost_destroy(ibfthost_ctx* c) { delete c; }

// ValidatorManager.Init(height) with the embedder's GetVotingPowers result: n addresses (concatenated, lens[i] bytes each)
// and n 32-byte big-endian powers (NULL => 1).  Returns 0 ok, 5 = errVotingPowerNotCorrect, 1 = an address listed twice
// (GetVotingPowers returns a map, which cannot hold one twice), or the engine's status when it refuses the table.  A refused
// table changes nothing: the context keeps its previous table.
int ibfthost_set_validators(ibfthost_ctx* c, uint64_t height, const uint8_t* addrs, const uint32_t* lens, const uint8_t* powers_be, uint32_t n) {
  std::vector<Bytes> order;
  std::vector<u320> powers;
  size_t off = 0;
  for (uint32_t i = 0; i < n; i++) {
    order.push_back(B(addrs + off, lens[i]));
    off += lens[i];
    powers.push_back(powers_be ? u320::from_be32(powers_be + 32 * (size_t)i) : u320::from_u64(1));
  }
  // duplicates: a GPU context leaves the 20-byte addresses to the engine (GpuVerifier::SetValidators returns false); the
  // others -- every address of a callback context -- are checked here
  std::vector<Bytes> host_only;
  for (auto& a : order)
    if (!c->gpu || a.size() != 20) host_only.push_back(a);
  std::sort(host_only.begin(), host_only.end());
  if (std::adjacent_find(host_only.begin(), host_only.end()) != host_only.end()) return IBFT_ERR_INVALID_ARG;
  u320 total;
  for (auto& p : powers) total.add(p);
  if (total.is_zero()) return IBFT_ERR_VOTING_POWER;
  // the device table first: when the engine refuses it, the host ValidatorManager keeps its previous table too
  if (c->gpu && !c->gpu->SetValidators(height, order, powers)) {
    int rc = c->gpu->last_set_status();
    return rc != IBFT_OK ? rc : IBFT_ERR_CUDA;
  }
  if (!c->vm.SetVotingPowers(order, powers)) return IBFT_ERR_VOTING_POWER;
  return IBFT_OK;
}

void ibfthost_set_batching(ibfthost_ctx* c, int on) { c->ibft->batching = on != 0; }
void ibfthost_set_incremental_quorum(ibfthost_ctx* c, int on) { c->ibft->incremental_quorum = on != 0; }
// GPU verifier: submit PREPARE / COMMIT messages as raw frames (IBFT_KIND_WIRE)
void ibfthost_set_wire_frames(ibfthost_ctx* c, int on) { if (c->gpu) c->gpu->use_wire_frames = on != 0; }
uint64_t ibfthost_gpu_frames_handed_back(ibfthost_ctx* c) { return c->gpu ? c->gpu->frames_handed_back() : 0; }

// GpuVerifier::onReject: fn(user, kind, height, message, from, reason, recovered20) once per rejected item (see verifier.hpp);
// fn = NULL removes the hook.  Set it before the context is used from several threads.
typedef void (*cb_on_reject)(void* user, uint8_t kind, uint64_t height, const uint8_t* message, size_t mlen, const uint8_t* from,
                             size_t flen, uint8_t reason, const uint8_t* recovered20);
void ibfthost_set_reject_hook(ibfthost_ctx* c, cb_on_reject fn, void* user) {
  if (!c->gpu) return;
  if (!fn) { c->gpu->onReject = nullptr; return; }
  c->gpu->onReject = [fn, user](const GpuVerifier::Rejection& x) {
    fn(user, x.kind, x.height, (const uint8_t*)x.message.data(), x.message.size(), (const uint8_t*)x.from.data(), x.from.size(), x.reason,
       (const uint8_t*)x.recovered.data());
  };
}
// rejections reported with `reason` (IBFT_REASON_*), and the explain calls made for them
uint64_t ibfthost_gpu_rejects(ibfthost_ctx* c, uint32_t reason) { return c->gpu && reason < 256 ? c->gpu->rejects((uint8_t)reason) : 0; }
uint64_t ibfthost_gpu_explain_calls(ibfthost_ctx* c) { return c->gpu ? c->gpu->explain_calls() : 0; }

// state.view / state.name / state.proposalMessage
int ibfthost_set_state(ibfthost_ctx* c, uint64_t height, uint64_t round, int state_name, const uint8_t* proposal_wire, size_t len) {
  c->ibft->state.view = View{height, round};
  c->ibft->state.name = (StateName)state_name;
  try {
    c->ibft->state.proposal_message = proposal_wire ? decode_message(proposal_wire, len) : nullptr;
  } catch (const DecodeError&) { return IBFT_ERR_INVALID_ARG; }
  if (c->gpu) c->gpu->SetCurrentHeight(height);
  return IBFT_OK;
}
int ibfthost_get_state_name(ibfthost_ctx* c) { return (int)c->ibft->state.name; }

static MessagePtr dec(const uint8_t* w, size_t n) {
  try { return decode_message(w, n); } catch (const DecodeError&) { return nullptr; }
}

int ibfthost_store_add(ibfthost_ctx* c, const uint8_t* wire, size_t len) {  // messages.AddMessage
  auto m = dec(wire, len);
  if (!m) return IBFT_ERR_INVALID_ARG;
  c->messages.AddMessage(m);
  return IBFT_OK;
}
int ibfthost_add_message(ibfthost_ctx* c, const uint8_t* wire, size_t len) {  // IBFT.AddMessage
  auto m = dec(wire, len);
  if (!m) return IBFT_ERR_INVALID_ARG;
  c->ibft->AddMessage(m);
  return IBFT_OK;
}
// bulk ingress: `count` wire messages concatenated, lens[i] bytes each
int ibfthost_add_messages(ibfthost_ctx* c, const uint8_t* wires, const uint32_t* lens, uint32_t count) {
  std::vector<MessagePtr> batch;
  size_t off = 0;
  for (uint32_t i = 0; i < count; i++) {
    auto m = dec(wires + off, lens[i]);
    off += lens[i];
    if (m) batch.push_back(m);
  }
  c->ibft->AddMessages(batch);
  return IBFT_OK;
}
int ibfthost_is_acceptable(ibfthost_ctx* c, const uint8_t* wire, size_t len) {
  auto m = dec(wire, len);
  return m ? (int)c->ibft->isAcceptableMessage(*m) : 0;
}
uint64_t ibfthost_num_messages(ibfthost_ctx* c, uint64_t h, uint64_t r, uint32_t type) { return c->messages.numMessages(View{h, r}, type); }
void ibfthost_prune_by_height(ibfthost_ctx* c, uint64_t h) { c->messages.PruneByHeight(h); }
uint64_t ibfthost_signal_count(ibfthost_ctx* c) { return c->signals.size() / 3; }

// handlers: return the decision; senders of the resulting valid set are written, '\n'-joined hex, into out (for comparison)
static size_t put_senders(ibfthost_ctx* c, const std::vector<MessagePtr>& msgs, char* out, size_t cap) {
  static const char* hx = "0123456789abcdef";
  std::string s;
  for (auto& m : msgs) {
    for (unsigned char ch : m->from) { s.push_back(hx[ch >> 4]); s.push_back(hx[ch & 15]); }
    s.push_back('\n');
  }
  c->last_out = s;
  if (out && cap) {
    size_t n = std::min(cap - 1, s.size());
    memcpy(out, s.data(), n);
    out[n] = 0;
  }
  return s.size();
}
int ibfthost_handle_commit(ibfthost_ctx* c, uint64_t h, uint64_t r) { return (int)c->ibft->handleCommit(View{h, r}); }
int ibfthost_handle_prepare(ibfthost_ctx* c, uint64_t h, uint64_t r) { return (int)c->ibft->handlePrepare(View{h, r}); }
uint64_t ibfthost_seal_count(ibfthost_ctx* c) { return c->ibft->state.seals.size(); }
uint64_t ibfthost_latest_pc_prepares(ibfthost_ctx* c) { return c->ibft->state.latest_pc ? c->ibft->state.latest_pc->prepare_messages.size() : 0; }
// returns 1 and the accepted proposer (hex) when a valid PREPREPARE exists
int ibfthost_handle_preprepare(ibfthost_ctx* c, uint64_t h, uint64_t r, char* out, size_t cap) {
  auto m = c->ibft->handlePrePrepare(View{h, r});
  if (!m) return 0;
  put_senders(c, {m}, out, cap);
  return 1;
}
// returns -1 for the nil certificate, else the number of ROUND_CHANGE messages in the extended RCC (senders in out)
int ibfthost_handle_round_change(ibfthost_ctx* c, uint64_t h, uint64_t r, char* out, size_t cap) {
  bool found = false;
  auto msgs = c->ibft->handleRoundChangeMessage(View{h, r}, &found);
  if (!found) return -1;
  put_senders(c, msgs, out, cap);
  return (int)msgs.size();
}
// valid senders of a view after GetValidMessages with the always-true closure (store contents)
int ibfthost_store_senders(ibfthost_ctx* c, uint64_t h, uint64_t r, uint32_t type, char* out, size_t cap) {
  auto msgs = c->messages.Snapshot(View{h, r}, type);
  put_senders(c, msgs, out, cap);
  return (int)msgs.size();
}

// validPC on an encoded PreparedCertificate (NULL => nil certificate)
int ibfthost_valid_pc(ibfthost_ctx* c, const uint8_t* pc_wire, size_t len, int has_pc, uint64_t round_limit, uint64_t height) {
  if (!has_pc) return (int)c->ibft->validPC(nullptr, round_limit, height);
  try {
    auto pc = decode_pc(wire::Reader{pc_wire, pc_wire + len, 0, nullptr});
    return (int)c->ibft->validPC(pc.get(), round_limit, height);
  } catch (const DecodeError&) { return 0; }
}
int ibfthost_validate_proposal(ibfthost_ctx* c, const uint8_t* wire, size_t len, uint64_t h, uint64_t r) {
  auto m = dec(wire, len);
  if (!m) return 0;
  View v{h, r};
  return (int)(r == 0 ? c->ibft->validateProposal0(*m, v) : c->ibft->validateProposal(*m, v));
}
int ibfthost_has_quorum_senders(ibfthost_ctx* c, const uint8_t* addrs, const uint32_t* lens, uint32_t n) {
  std::set<Bytes> s;
  size_t off = 0;
  for (uint32_t i = 0; i < n; i++) { s.insert(B(addrs + off, lens[i])); off += lens[i]; }
  return (int)c->vm.HasQuorum(s);
}
// the quorum check reading the GPU's voted set (bit i = validator i in the order given to ibfthost_set_validators)
int ibfthost_has_quorum_voted(ibfthost_ctx* c, const uint32_t* words, uint32_t n_words) { return (int)c->vm.HasQuorumVoted(words, n_words); }

// codec: decode + re-encode (with / without signature); returns the encoded length (0 on decode error)
size_t ibfthost_reencode(const uint8_t* wire, size_t len, int with_signature, uint8_t* out, size_t cap) {
  auto m = dec(wire, len);
  if (!m) return (size_t)-1;
  Bytes e = encode_message(*m, with_signature != 0);
  if (out && cap >= e.size()) memcpy(out, e.data(), e.size());
  return e.size();
}

// PayloadNoSig of a frame as protobuf-go would produce it (Unmarshal, Signature = nil, Marshal): returns the length (or
// (size_t)-1 on a parse error) and writes the bytes when the buffer is large enough
size_t ibfthost_remarshal(const uint8_t* wire, size_t len, int with_signature, uint8_t* out, size_t cap) {
  try {
    Bytes e = remarshal(wire, len, with_signature != 0);
    if (out && cap >= e.size()) memcpy(out, e.data(), e.size());
    return e.size();
  } catch (const DecodeError&) { return (size_t)-1; }
}

// InsertProposal-side check (core/backend.go:78-81): n seals = n signers (20 bytes each) + n signatures (65 bytes each) over one
// proposal hash; returns 1 when the valid seals' distinct signers carry quorum, and the number of valid seals in *n_valid.
int ibfthost_verify_committed_seals(ibfthost_ctx* c, const uint8_t* hash, size_t hlen, const uint8_t* signers, const uint8_t* sigs,
                                    uint32_t n, uint32_t* n_valid) {
  if (!c->gpu) return -1;
  std::vector<CommittedSeal> seals;
  for (uint32_t i = 0; i < n; i++) seals.push_back(CommittedSeal{B(signers + 20 * (size_t)i, 20), B(sigs + 65 * (size_t)i, 65)});
  auto valid = c->gpu->VerifyCommittedSeals(B(hash, hlen), seals);
  std::set<Bytes> who;
  uint32_t cnt = 0;
  for (uint32_t i = 0; i < n; i++)
    if (valid[i]) { cnt++; who.insert(seals[i].signer); }
  if (n_valid) *n_valid = cnt;
  return (int)c->vm.HasQuorum(who);
}

// Ingress storm (test + bench harness of the coalescer): `count` wire messages are checked with SINGLE-message
// IsValidValidator calls from `threads` concurrent threads (thread t takes messages t, t+threads, ...), exactly the call
// pattern of the reference's gossip ingress (core/ibft.go:1101-1128).  verdicts[i] = the call's answer; lat_us[i] = its
// wall-clock latency (may be NULL).  Returns the elapsed wall time in microseconds, or -1 on a decode error.
double ibfthost_ingress_storm(ibfthost_ctx* c, const uint8_t* wires, const uint32_t* lens, uint32_t count, uint32_t threads,
                              uint8_t* verdicts, float* lat_us) {
  std::vector<MessagePtr> msgs(count);
  size_t off = 0;
  for (uint32_t i = 0; i < count; i++) {
    msgs[i] = dec(wires + off, lens[i]);
    off += lens[i];
    if (!msgs[i]) return -1.0;
  }
  if (threads == 0) threads = 1;
  auto t0 = std::chrono::steady_clock::now();
  std::vector<std::thread> pool;
  for (uint32_t t = 0; t < threads; t++) {
    pool.emplace_back([&, t]() {
      for (uint32_t i = t; i < count; i += threads) {
        auto a = std::chrono::steady_clock::now();
        bool ok = c->verifier->IsValidValidator(*msgs[i]);
        auto b = std::chrono::steady_clock::now();
        verdicts[i] = ok ? 1 : 0;
        if (lat_us) lat_us[i] = std::chrono::duration<float, std::micro>(b - a).count();
      }
    });
  }
  for (auto& th : pool) th.join();
  return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
}
void ibfthost_set_ingress(ibfthost_ctx* c, uint32_t max_batch, uint32_t min_batch, uint32_t linger_us) {
  if (!c->gpu) return;
  c->gpu->ingress_max_batch = max_batch ? max_batch : 1;
  c->gpu->ingress_min_batch = min_batch;
  c->gpu->ingress_linger_us = linger_us;
}
uint64_t ibfthost_gpu_ingress_requests(ibfthost_ctx* c) { return c->gpu ? c->gpu->ingress_requests() : 0; }
uint64_t ibfthost_gpu_ingress_flushes(ibfthost_ctx* c) { return c->gpu ? c->gpu->ingress_flushes() : 0; }

uint64_t ibfthost_gpu_device_calls(ibfthost_ctx* c) { return c->gpu ? c->gpu->device_calls() : 0; }
uint64_t ibfthost_gpu_items_verified(ibfthost_ctx* c) { return c->gpu ? c->gpu->items_verified() : 0; }
// single-message verifier calls through whatever verifier the context holds
int ibfthost_is_valid_validator(ibfthost_ctx* c, const uint8_t* wire, size_t len) {
  auto m = dec(wire, len);
  return m ? (int)c->verifier->IsValidValidator(*m) : 0;
}
int ibfthost_is_valid_committed_seal(ibfthost_ctx* c, const uint8_t* hash, size_t hlen, const uint8_t* signer, size_t slen,
                                     const uint8_t* sig, size_t siglen) {
  Bytes h = B(hash, hlen);
  CommittedSeal s{B(signer, slen), B(sig, siglen)};
  return (int)c->verifier->IsValidCommittedSeal(hash ? &h : nullptr, signer ? &s : nullptr);
}
int ibfthost_is_valid_proposal_hash(ibfthost_ctx* c, const uint8_t* raw, size_t rawlen, uint64_t round, int has_proposal,
                                    const uint8_t* hash, size_t hlen) {
  Proposal p{B(raw, rawlen), round};
  Bytes h = B(hash, hlen);
  return (int)c->verifier->IsValidProposalHash(has_proposal ? &p : nullptr, hash ? &h : nullptr);
}
}
