// verifier.hpp -- the plugin boundary of the hot path, mirrored from reference core/backend.go:37-56 (core.Verifier) plus
// Backend.ID (:84), and its GPU-backed implementation.
//
//   Verifier        same five methods, same argument meaning, bool-only results ("never panic, malformed => false":
//                   SURVEY.md §8b).  Prefetch() is the one addition: the batching shim announces the messages a handler is
//                   about to validate so that a GPU backend can verify all their signatures in ONE device call; the
//                   per-message methods then answer from the verdict cache, which keeps the reference's serial predicate
//                   code (and therefore its exact semantics, including pruning order) untouched.
//   CallbackVerifier  closure-backed verifier = the reference's mockBackend (core/mock_test.go:72-151): defaults true,
//                   IsProposer default false.  Used by the CPU tests of the host logic.
//   GpuVerifier     the production path: every signature check goes through the C ABI (include/ibft_verify.h) into the
//                   CUDA kernels.  There is NO CPU fallback: if the engine call fails the answer is `false` (no verdict is
//                   ever invented) and last_error() says why.
#pragma once
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <mutex>
#include <thread>
#include <unordered_map>

#include "../../include/ibft_verify.h"
#include "quorum.hpp"
#include "store.hpp"

namespace ibft::host {

class Verifier {
 public:
  virtual ~Verifier() = default;
  virtual bool IsValidProposal(const Bytes& raw_proposal) = 0;                                   // backend.go:39
  virtual bool IsValidValidator(const IbftMessage& msg) = 0;                                     // backend.go:41-45
  virtual bool IsProposer(const Bytes& id, uint64_t height, uint64_t round) = 0;                 // backend.go:47-48
  virtual bool IsValidProposalHash(const Proposal* proposal, const Bytes* hash) = 0;             // backend.go:50-51
  virtual bool IsValidCommittedSeal(const Bytes* proposal_hash, const CommittedSeal* seal) = 0;  // backend.go:53-55
  virtual Bytes ID() = 0;                                                                        // backend.go:84
  // Batching hook (no counterpart in the reference): sender signatures of `msgs` (+ their committed seals when
  // `with_seals`) are about to be checked.  Default: nothing.
  virtual void Prefetch(const std::vector<MessagePtr>& msgs, bool with_seals) {
    (void)msgs;
    (void)with_seals;
  }
};

class CallbackVerifier : public Verifier {
 public:
  std::function<bool(const Bytes&)> isValidProposalFn;
  std::function<bool(const IbftMessage&)> isValidValidatorFn;
  std::function<bool(const Bytes&, uint64_t, uint64_t)> isProposerFn;
  std::function<bool(const Proposal*, const Bytes*)> isValidProposalHashFn;
  std::function<bool(const Bytes*, const CommittedSeal*)> isValidCommittedSealFn;
  Bytes id;
  bool IsValidProposal(const Bytes& raw) override { return isValidProposalFn ? isValidProposalFn(raw) : true; }
  bool IsValidValidator(const IbftMessage& m) override { return isValidValidatorFn ? isValidValidatorFn(m) : true; }
  bool IsProposer(const Bytes& i, uint64_t h, uint64_t r) override { return isProposerFn ? isProposerFn(i, h, r) : false; }
  bool IsValidProposalHash(const Proposal* p, const Bytes* h) override { return isValidProposalHashFn ? isValidProposalHashFn(p, h) : true; }
  bool IsValidCommittedSeal(const Bytes* h, const CommittedSeal* s) override { return isValidCommittedSealFn ? isValidCommittedSealFn(h, s) : true; }
  Bytes ID() override { return id; }
};

class GpuVerifier : public Verifier {
 public:
  // embedder policy that is not signature work (SURVEY.md §8a a4): stays on the host
  std::function<bool(const Bytes&, uint64_t, uint64_t)> isProposerFn;
  std::function<bool(const Bytes&)> isValidProposalFn;
  // The proposal hash is the EMBEDDER's function (go-ibft only says "hash matches keccak(proposal)", core/ibft.go:648; a real node
  // hashes its block header).  Unset: the synthetic convention of SURVEY.md §8c, computed on the device.  Set: the embedder's
  // own hash -- also the place to hash ONE multi-megabyte proposal on a host core, where a single serial sponge is 20-30x
  // faster than on the device (DESIGN.md §3.3).  Either way it runs once per (proposal, round) thanks to the cache below.
  std::function<Bytes(const Bytes& raw_proposal, uint64_t round)> proposalHashFn;
  Bytes id;
  // Submit PREPARE / COMMIT messages as RAW FRAMES (IBFT_KIND_WIRE*): the device derives PayloadNoSig, From and the
  // signature from the gossip frame itself, so the host never re-marshals.  Frames the device hands back
  // (IBFT_ITEM_NEEDS_HOST: non-canonical encoding) are re-submitted through the marshalled path.
  bool use_wire_frames = false;
  // Ingress coalescer (see lookup_or_coalesce): a flush takes at most this many queued single-message checks, and a leader
  // that finds fewer than `ingress_min_batch` queued lingers up to `ingress_linger_us` for more (0 = flush at once: the
  // batching then comes from the checks that queue up WHILE a flush is on the device).
  uint32_t ingress_max_batch = 4096;
  uint32_t ingress_min_batch = 1;
  uint32_t ingress_linger_us = 0;
  uint32_t ingress_second_min = 32;  // queue length from which a SECOND flush goes up while one is still on the device

  explicit GpuVerifier(const ibft_engine_params& params) {
    params_ = params;
    int rc = ibft_engine_create(&params_, &engine_);
    if (rc != IBFT_OK) {
      engine_ = nullptr;
      error_ = ibft_last_error();
    }
  }
  ~GpuVerifier() override {
    if (engine_) ibft_engine_destroy(engine_);
  }
  bool ok() const { return engine_ != nullptr; }
  std::string last_error() const {
    std::lock_guard<std::mutex> lk(state_mu_);
    return error_;
  }
  ibft_engine* engine() { return engine_; }

  // ValidatorBackend.GetVotingPowers(height) pushed to the device (validator_manager.go:50-57): the table of `height`
  // occupies slot (height mod max_table_slots).  Addresses that are not 20 bytes can never equal a recovered signer and are
  // left out of the device table.
  bool SetValidators(uint64_t height, const std::vector<Bytes>& addrs, const std::vector<u320>& powers) {
    if (!engine_) return false;
    std::vector<uint8_t> a, p;
    for (size_t i = 0; i < addrs.size(); i++) {
      if (addrs[i].size() != 20) continue;
      a.insert(a.end(), addrs[i].begin(), addrs[i].end());
      for (int k = 3; k >= 0; k--)
        for (int j = 7; j >= 0; j--) p.push_back((uint8_t)(powers[i].l[k] >> (8 * j)));
    }
    uint32_t slot = (uint32_t)(height % params_.max_table_slots);
    {
      // the slot stops answering for its old height BEFORE the engine swaps the table
      std::lock_guard<std::mutex> lk(state_mu_);
      slot_height_.erase(slot);
      epoch_++;
      cache_.clear();
    }
    int rc = ibft_set_validators(engine_, slot, height, a.data(), p.data(), (uint32_t)(a.size() / 20));
    std::lock_guard<std::mutex> lk(state_mu_);
    if (rc != IBFT_OK) {
      error_ = ibft_last_error();
      return false;
    }
    slot_height_[slot] = height;
    if (height > current_height_.load()) hash_cache_.clear();  // proposals of finished heights are never asked for again
    current_height_ = height;
    epoch_++;
    cache_.clear();
    return true;
  }
  // committed seals carry no height: they are checked against the validators of the running sequence
  void SetCurrentHeight(uint64_t h) {
    std::lock_guard<std::mutex> lk(state_mu_);
    if (h > current_height_.load()) hash_cache_.clear();
    current_height_ = h;
  }

  bool IsValidProposal(const Bytes& raw) override { return isValidProposalFn ? isValidProposalFn(raw) : true; }
  bool IsProposer(const Bytes& i, uint64_t h, uint64_t r) override { return isProposerFn ? isProposerFn(i, h, r) : false; }
  Bytes ID() override { return id; }

  // The reference calls the verifier concurrently (gossip goroutines through AddMessage, the round goroutine and two
  // watchers: core/ibft.go:335-347, :1128) while the store holds its per-type mutex.  Every entry point below may be called
  // from any number of threads and never calls back into the store.  A cache miss does NOT become a device call of one item:
  // it joins the ingress queue (lookup_or_coalesce).
  bool IsValidValidator(const IbftMessage& m) override {
    Pending p;
    if (!sender_item(m, p)) return false;
    return lookup_or_coalesce(std::move(p));
  }
  bool IsValidCommittedSeal(const Bytes* proposal_hash, const CommittedSeal* seal) override {
    Pending p;
    if (!seal_item(proposal_hash, seal, p)) return false;
    return lookup_or_coalesce(std::move(p));
  }
  // Synthetic proposal-hash convention of SURVEY.md §8(c): Keccak-256(Keccak-256(rawProposal) || u64_be(round)); real
  // embedders hash an RLP header (out of scope).  Both sponges run in ONE device launch (ibft_proposal_hash_batch), once per
  // (proposal, round): the reference asks again for every PREPARE and COMMIT of the round (core/ibft.go:858, :938).
  bool IsValidProposalHash(const Proposal* proposal, const Bytes* hash) override {
    if (!engine_ || !proposal || !hash || hash->size() != 32) return false;
    Bytes key = proposal->raw_proposal;
    for (int j = 7; j >= 0; j--) key.push_back((char)(proposal->round >> (8 * j)));
    {
      std::lock_guard<std::mutex> lk(state_mu_);
      auto it = hash_cache_.find(key);
      if (it != hash_cache_.end()) return it->second == *hash;
    }
    uint8_t out[32];
    int rc = IBFT_OK;
    if (proposalHashFn) {
      Bytes h = proposalHashFn(proposal->raw_proposal, proposal->round);
      if (h.size() != 32) return false;
      memcpy(out, h.data(), 32);
    } else {
      uint32_t off = 0, len = (uint32_t)proposal->raw_proposal.size();
      uint64_t round = proposal->round;
      rc = ibft_proposal_hash_batch(engine_, (const uint8_t*)proposal->raw_proposal.data(), proposal->raw_proposal.size(), &off, &len,
                                    &round, 1, out);
      device_calls_++;
    }
    std::lock_guard<std::mutex> lk(state_mu_);
    if (rc != IBFT_OK) {
      error_ = ibft_last_error();
      return false;
    }
    // bounded: a validator flooding ROUND_CHANGE messages with distinct last_prepared_proposal values must not grow the cache
    // without limit (entries are proposal-sized); finished heights are dropped in SetValidators / SetCurrentHeight
    if (hash_cache_.size() >= kMaxHashCache) hash_cache_.clear();
    Bytes h((const char*)out, 32);
    hash_cache_[key] = h;
    return h == *hash;
  }

  void Prefetch(const std::vector<MessagePtr>& msgs, bool with_seals) override {
    std::vector<Pending> batch;
    std::unordered_map<Bytes, size_t> seen;
    {
      std::lock_guard<std::mutex> lk(state_mu_);
      int depth = 0;
      std::function<void(const IbftMessage&)> visit = [&](const IbftMessage& m) {
        if (depth > wire::kMaxDepth) return;  // same bound as the decoder
        depth++;
        Pending p;
        if (sender_item(m, p) && !cache_.count(p.key) && seen.emplace(p.key, batch.size()).second) batch.push_back(std::move(p));
        if (with_seals && m.payload_kind == PAYLOAD_COMMIT) {
          auto seal = ExtractCommittedSeal(m);
          Pending q;
          if (seal_item(ExtractCommitHash(m), seal.get(), q) && !cache_.count(q.key) && seen.emplace(q.key, batch.size()).second)
            batch.push_back(std::move(q));
        }
        // nested signatures: prepared certificates inside ROUND_CHANGE, round-change certificates inside PREPREPARE
        if (m.payload_kind == PAYLOAD_ROUND_CHANGE && m.round_change.latest_prepared_certificate) {
          auto& pc = *m.round_change.latest_prepared_certificate;
          if (pc.proposal_message) visit(*pc.proposal_message);
          for (auto& pm : pc.prepare_messages)
            if (pm) visit(*pm);
        }
        if (m.payload_kind == PAYLOAD_PREPREPARE && m.preprepare.certificate)
          for (auto& rc : m.preprepare.certificate->round_change_messages)
            if (rc) visit(*rc);
        depth--;
      };
      for (auto& m : msgs)
        if (m) visit(*m);
    }
    verify_pending(batch, nullptr);
  }

  // Re-verification of the >= Q committed seals of an imported block (Backend.InsertProposal, core/backend.go:78-81; the same
  // check a syncing node performs): all seals in ONE launch.  valid[i] = IsValidCommittedSeal(hash, seals[i]).
  std::vector<bool> VerifyCommittedSeals(const Bytes& proposal_hash, const std::vector<CommittedSeal>& seals) {
    std::vector<Pending> batch;
    std::vector<int> where(seals.size(), -1);  // index into batch, or -2 = answered from the cache (valid), -3 = cached invalid
    std::unordered_map<Bytes, size_t> seen;
    {
      std::lock_guard<std::mutex> lk(state_mu_);
      for (size_t i = 0; i < seals.size(); i++) {
        Pending p;
        if (!seal_item(&proposal_hash, &seals[i], p)) continue;
        auto c = cache_.find(p.key);
        if (c != cache_.end()) { where[i] = c->second ? -2 : -3; continue; }
        auto ins = seen.emplace(p.key, batch.size());
        where[i] = (int)ins.first->second;
        if (ins.second) batch.push_back(std::move(p));
      }
    }
    std::vector<int8_t> verdicts;
    verify_pending(batch, &verdicts);
    std::vector<bool> valid(seals.size(), false);
    for (size_t i = 0; i < seals.size(); i++) valid[i] = where[i] == -2 || (where[i] >= 0 && verdicts[(size_t)where[i]] == 1);
    return valid;
  }

  uint64_t device_calls() const { return device_calls_.load(); }
  uint64_t items_verified() const { return items_verified_.load(); }
  uint64_t frames_handed_back() const { return frames_handed_back_.load(); }
  uint64_t ingress_requests() const { return ingress_requests_.load(); }   // single-message checks that missed the cache
  uint64_t ingress_flushes() const { return ingress_flushes_.load(); }     // device calls the coalescer made for them

 private:
  static constexpr size_t kMaxHashCache = 64;
  struct Pending {
    Bytes key;  // exact-bytes cache key
    ibft_sig_item item;
    Bytes payload;                                 // marshalled items: PayloadNoSig
    std::shared_ptr<const Bytes> wire_root;        // raw-frame items: the span [wire_off, +wire_len) of the frame they came in
    uint32_t wire_off = 0, wire_len = 0;
    uint64_t height;
    const IbftMessage* fallback_payload_msg = nullptr;  // raw-frame items: the message to re-marshal if the device hands it back
  };
  // one queued single-message check of the ingress coalescer
  struct Req {
    Pending p;
    bool done = false;
    bool result = false;
    std::condition_variable cv;  // per request: a finished flush wakes its own callers only
  };
  mutable std::mutex state_mu_;  // cache_, hash_cache_, slot_height_, current_height_, epoch_, error_  (never held across a device call)
  ibft_engine_params params_{};
  ibft_engine* engine_ = nullptr;
  std::string error_;
  std::unordered_map<Bytes, bool> cache_;
  std::unordered_map<Bytes, Bytes> hash_cache_;
  std::map<uint32_t, uint64_t> slot_height_;
  std::atomic<uint64_t> current_height_{0};
  uint64_t epoch_ = 0;  // bumped by SetValidators: verdicts computed against a replaced table are not cached
  std::atomic<uint64_t> device_calls_{0}, items_verified_{0}, frames_handed_back_{0}, ingress_requests_{0}, ingress_flushes_{0};
  // ingress coalescer
  std::mutex ing_mu_;
  std::deque<std::shared_ptr<Req>> ing_queue_;
  int ing_leaders_ = 0;
  static constexpr int kMaxLeaders = 2;  // two flushes may be on the device at once (the engine has two lanes)

  static void put_sig(ibft_sig_item& it, const Bytes& sig, const Bytes& signer) {
    memset(&it, 0, sizeof it);
    memcpy(it.r, sig.data(), 32);
    memcpy(it.s, sig.data() + 32, 32);
    it.v = (uint8_t)sig[64];
    memcpy(it.signer, signer.data(), 20);
  }
  // IsValidValidator: signer of msg.Signature over Keccak-256(PayloadNoSig) == msg.From and From is a validator at
  // msg.View.Height (backend.go:41-45).  Structurally invalid => false without touching the device.
  bool sender_item(const IbftMessage& m, Pending& p, bool allow_wire = true) {
    if (!m.view || m.from.size() != 20 || m.signature.size() != 65) return false;
    p.height = m.view->height;
    if (allow_wire && use_wire_frames && m.has_wire()) {
      // any message type, top-level or nested in a certificate: the device walks the frame (canonical-encoding check included)
      // and hashes it with the signature TLV cut out -- no clone + marshal on the host
      memset(&p.item, 0, sizeof p.item);
      p.item.kind = IBFT_KIND_WIRE;
      p.wire_root = m.root_wire;
      p.wire_off = m.wire_off;
      p.wire_len = m.wire_len;
      p.fallback_payload_msg = &m;
      p.key.assign(1, 'W');
      for (int j = 7; j >= 0; j--) p.key.push_back((char)(p.height >> (8 * j)));
      p.key.append(m.wire_data(), m.wire_len);
      return true;
    }
    // marshalled path: for a message that was decoded from a frame, PayloadNoSig is the protobuf-go re-marshal of exactly the
    // bytes that arrived (unknown fields kept, duplicates merged) -- the model alone would lose them
    try {
      p.payload = payload_no_sig_exact(m);
    } catch (const DecodeError&) {
      return false;
    }
    put_sig(p.item, m.signature, m.from);
    p.item.kind = IBFT_KIND_PAYLOAD;
    p.key.assign(1, 'S');
    for (int j = 7; j >= 0; j--) p.key.push_back((char)(p.height >> (8 * j)));
    p.key += m.signature;
    p.key += p.payload;
    return true;
  }
  bool seal_item(const Bytes* proposal_hash, const CommittedSeal* seal, Pending& p) {
    if (!proposal_hash || !seal || proposal_hash->size() != 32 || seal->signer.size() != 20 || seal->signature.size() != 65) return false;
    p.height = current_height_.load();
    put_sig(p.item, seal->signature, seal->signer);
    memcpy(p.item.digest, proposal_hash->data(), 32);
    p.item.kind = IBFT_KIND_SEAL;
    p.key.assign(1, 'C');
    for (int j = 7; j >= 0; j--) p.key.push_back((char)(p.height >> (8 * j)));
    p.key += seal->signature;
    p.key += seal->signer;
    p.key += *proposal_hash;
    return true;
  }

  // INGRESS COALESCER.  The reference calls IsValidValidator once per inbound gossip message from any number of goroutines
  // (core/ibft.go:1101-1128).  One device call per message would cost a whole kernel launch and one serial chain for one signature and
  // serialise the callers.  Instead a miss is queued; a caller that finds fewer than two flushes in flight becomes a leader: it takes
  // everything queued (its own request included), makes a single device call for the batch, publishes the verdicts and wakes the
  // others (two leaders at most: the engine runs two host-buffer calls side by side, so the next batch goes up while the previous
  // one is still on the device).  Requests that
  // arrive while a flush is on the device pile up and form the next batch -- the batch size adapts to the arrival rate with no
  // timer (group commit); `ingress_linger_us` / `ingress_min_batch` add an optional wait for sparse traffic.  The verdict of
  // every request is exactly what a single-item call would have returned: same item, same table, same kernels.
  bool lookup_or_coalesce(Pending&& p) {
    {
      std::lock_guard<std::mutex> lk(state_mu_);
      auto it = cache_.find(p.key);
      if (it != cache_.end()) return it->second;
    }
    if (!engine_) return false;
    ingress_requests_++;
    auto req = std::make_shared<Req>();
    req->p = std::move(p);
    std::unique_lock<std::mutex> lk(ing_mu_);
    ing_queue_.push_back(req);
    while (!req->done) {
      // the first leader starts at once; a second one (while a flush is already on the device) only for a queue worth a launch of
      // its own -- otherwise the newcomers keep piling up behind the flush in flight and go up together when it returns
      if (ing_queue_.empty() || ing_leaders_ >= kMaxLeaders || (ing_leaders_ == 1 && ing_queue_.size() < ingress_second_min)) {
        req->cv.wait(lk);  // woken by the leader that decided this request, or by a finishing leader handing the lead over
        continue;
      }
      ing_leaders_++;
      if (ingress_linger_us && ing_queue_.size() < ingress_min_batch) {
        lk.unlock();
        std::this_thread::sleep_for(std::chrono::microseconds(ingress_linger_us));
        lk.lock();
      }
      std::vector<std::shared_ptr<Req>> taken;
      while (!ing_queue_.empty() && taken.size() < ingress_max_batch) {
        taken.push_back(std::move(ing_queue_.front()));
        ing_queue_.pop_front();
      }
      lk.unlock();
      // duplicates (the same message relayed by several peers) are verified once
      std::vector<Pending> batch;
      std::vector<size_t> slot_of(taken.size());
      std::unordered_map<Bytes, size_t> seen;
      for (size_t i = 0; i < taken.size(); i++) {
        auto ins = seen.emplace(taken[i]->p.key, batch.size());
        slot_of[i] = ins.first->second;
        if (ins.second) batch.push_back(taken[i]->p);
      }
      std::vector<int8_t> verdicts;
      verify_pending(batch, &verdicts);
      ingress_flushes_++;
      lk.lock();
      for (size_t i = 0; i < taken.size(); i++) {
        taken[i]->result = verdicts[slot_of[i]] == 1;  // no verdict (launch failure) => false, never true
        taken[i]->done = true;
        if (taken[i] != req) taken[i]->cv.notify_one();  // only the callers of THIS batch are woken (no thundering herd)
      }
      ing_leaders_--;
      if (!ing_queue_.empty()) ing_queue_.front()->cv.notify_one();  // somebody is waiting: hand the lead over
    }
    return req->result;
  }

  // One device call per engine-capacity chunk of the batch; groups = distinct heights (validator tables).
  // verdicts (optional): per batch entry 1 = valid, 0 = invalid, -1 = no verdict (the device call failed).
  void verify_pending(std::vector<Pending>& batch, std::vector<int8_t>* verdicts) {
    if (verdicts) verdicts->assign(batch.size(), -1);
    if (batch.empty() || !engine_) return;
    std::map<uint32_t, uint64_t> slot_height;
    uint64_t epoch;
    {
      std::lock_guard<std::mutex> lk(state_mu_);
      slot_height = slot_height_;
      epoch = epoch_;
    }
    size_t pos = 0;
    while (pos < batch.size()) {  // respect the engine's per-call capacity
      size_t n = std::min(batch.size() - pos, (size_t)params_.max_items);
      std::vector<ibft_sig_item> items(n);
      std::vector<ibft_group_desc> groups;
      std::map<uint64_t, uint16_t> group_of_height;
      std::unordered_map<const Bytes*, uint32_t> frame_at;  // root frame -> its offset in this call's arena
      Bytes arena;
      for (size_t i = 0; i < n; i++) {
        Pending& p = batch[pos + i];
        auto g = group_of_height.find(p.height);
        if (g == group_of_height.end()) {
          if (groups.size() >= params_.max_groups) { n = i; break; }
          uint32_t slot = (uint32_t)(p.height % params_.max_table_slots);
          auto sh = slot_height.find(slot);
          ibft_group_desc d{};
          // a height whose validator table is not resident cannot have members: its items are verified against an
          // empty answer (false) -- never against the wrong table (the engine checks d.height against the slot as well)
          d.table_slot = (sh != slot_height.end() && sh->second == p.height) ? (uint16_t)slot : (uint16_t)IBFT_NO_TABLE;
          d.height = p.height;
          groups.push_back(d);
          g = group_of_height.emplace(p.height, (uint16_t)(groups.size() - 1)).first;
        }
        items[i] = p.item;
        items[i].group = g->second;
        if (p.item.kind == IBFT_KIND_WIRE) {
          // a frame goes into the arena ONCE; messages nested in its certificates are spans inside it.  A nested message whose
          // root frame is not part of this batch contributes only its own bytes.
          auto placed = frame_at.find(p.wire_root.get());
          if (placed != frame_at.end()) {
            items[i].payload_off = placed->second + p.wire_off;
          } else {
            const bool whole = p.wire_off == 0 && p.wire_len == p.wire_root->size();
            if (arena.size() + p.wire_len > params_.max_payload_bytes) { n = i; break; }
            items[i].payload_off = (uint32_t)arena.size();
            if (whole) frame_at.emplace(p.wire_root.get(), (uint32_t)arena.size());
            arena.append(p.wire_root->data() + p.wire_off, p.wire_len);
          }
          items[i].payload_len = p.wire_len;
        } else if (p.item.kind == IBFT_KIND_PAYLOAD) {
          if (arena.size() + p.payload.size() > params_.max_payload_bytes) { n = i; break; }
          items[i].payload_off = (uint32_t)arena.size();
          items[i].payload_len = (uint32_t)p.payload.size();
          arena += p.payload;
        }
      }
      if (n == 0) {  // a single item that cannot fit: no verdict
        pos++;
        continue;
      }
      std::vector<uint32_t> bitmap((n + 31) / 32);
      std::vector<uint8_t> status(n, 0);
      int rc = ibft_verify_batch_ex(engine_, items.data(), (uint32_t)n, (const uint8_t*)arena.data(), arena.size(), groups.data(),
                                    (uint32_t)groups.size(), bitmap.data(), nullptr, nullptr, status.data(), nullptr, 0);
      device_calls_++;
      if (rc != IBFT_OK) {
        std::lock_guard<std::mutex> lk(state_mu_);
        error_ = ibft_last_error();  // launch failure => NO verdict is cached; callers see `false`
      } else {
        items_verified_ += n;
        std::vector<Pending> redo;
        std::vector<size_t> redo_of;
        {
          std::lock_guard<std::mutex> lk(state_mu_);
          const bool fresh = epoch == epoch_;  // the tables this batch was checked against are still the resident ones
          for (size_t i = 0; i < n; i++) {
            bool pass = (bitmap[i >> 5] >> (i & 31)) & 1u;
            // membership requires a resident table for the item's height
            if (groups[items[i].group].table_slot == IBFT_NO_TABLE) pass = false;
            Pending& p = batch[pos + i];
            if (status[i] == IBFT_ITEM_NEEDS_HOST && p.fallback_payload_msg) {
              // the device declined the frame (not canonical): same check through the marshalled path, same cache key
              Pending q;
              if (sender_item(*p.fallback_payload_msg, q, /*allow_wire=*/false)) {
                q.key = p.key;
                redo.push_back(std::move(q));
                redo_of.push_back(pos + i);
                continue;
              }
              pass = false;
            }
            if (fresh) cache_[p.key] = pass;
            if (verdicts) (*verdicts)[pos + i] = pass ? 1 : 0;
          }
        }
        if (!redo.empty()) {
          frames_handed_back_ += redo.size();
          std::vector<int8_t> rv;
          verify_pending(redo, &rv);
          if (verdicts)
            for (size_t k = 0; k < redo.size(); k++) (*verdicts)[redo_of[k]] = rv[k];
        }
      }
      pos += n;
    }
  }
};

}  // namespace ibft::host
