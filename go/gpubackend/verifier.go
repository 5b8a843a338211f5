package gpubackend

// COMPILE-UNVERIFIED (no Go toolchain in the authoring image).  Mirrors go-ibft_b200/host/verifier.hpp (GpuVerifier), which
// IS built and tested (tests/test_gpu_host.py, tests/test_gpu_round2.py): same cache keys, same "malformed => false", same
// Prefetch batching hook, same ingress coalescer, same table-epoch rule.

/*
#include "ibft_verify.h"
*/
import "C"

import (
	"encoding/binary"
	"math/big"
	"sync"
	"sync/atomic"
	"time"

	"github.com/0xPolygon/go-ibft/messages"
	"github.com/0xPolygon/go-ibft/messages/proto"
)

const maxHashCache = 64

// Verifier implements core.Verifier (core/backend.go:37-56) and messages.Prefetcher (go/patches/messages_messages.patch) on
// top of the engine.  Embed it in the node's Backend; the remaining Backend methods (message construction, BuildProposal,
// InsertProposal, ...) stay as they are.
type Verifier struct {
	Eng            *Engine
	IsProposerFn   func(id []byte, height, round uint64) bool // embedder policy, not signature work
	IsValidBlockFn func(raw []byte) bool
	// ProposalHashFn is the embedder's proposal hash (a real node hashes its block header).  nil: the synthetic convention of
	// SURVEY.md §8c on the device.  Also the place to hash ONE multi-megabyte proposal on a host core (DESIGN.md §3.3).
	ProposalHashFn func(raw []byte, round uint64) [32]byte

	// OnReject (optional) is called once per signature check the device rejected, with the reason and the recovered address (20
	// bytes, zero when recovery was not reached): after every device call that rejected items, one ExplainBatch call over them.
	// It runs after the verdicts are published and outside the verifier's locks.  Set it before the verifier is shared; nil
	// (the default) makes no extra device call.  Items of a height whose table is not resident are not reported.
	OnReject func(msg Item, reason Reason, recovered []byte)

	// ingress coalescer knobs (see lookupOrCoalesce)
	IngressMaxBatch int
	IngressMinBatch int
	IngressLinger   time.Duration

	mu            sync.Mutex // cache, hashCache, epoch -- never held across a device call
	cache         map[string]bool
	hashCache     map[string][32]byte
	epoch         uint64        // bumped by SetValidators: verdicts computed against a replaced table are not cached
	currentHeight atomic.Uint64 // committed seals carry no height: they are checked against the running sequence's validators

	ingMu     sync.Mutex
	ingCond   *sync.Cond
	ingQueue  []*ingressReq
	ingLeader bool
}

type ingressReq struct {
	it     Item
	key    string
	done   bool
	result bool
}

func NewVerifier(e *Engine) *Verifier {
	v := &Verifier{Eng: e, cache: map[string]bool{}, hashCache: map[string][32]byte{}, IngressMaxBatch: 4096, IngressMinBatch: 1}
	v.ingCond = sync.NewCond(&v.ingMu)
	return v
}

// SetValidators = ValidatorManager.Init's table pushed to the device (core/validator_manager.go:50-57).  Every cached verdict
// was computed against the old tables: the cache is emptied and in-flight batches will not write into it (epoch).
func (v *Verifier) SetValidators(height uint64, order [][]byte, powers map[string]*big.Int) error {
	v.mu.Lock()
	v.epoch++
	v.cache = map[string]bool{}
	v.mu.Unlock()
	err := v.Eng.SetValidators(height, order, powers)
	v.mu.Lock()
	v.epoch++
	v.cache = map[string]bool{}
	if height > v.currentHeight.Load() {
		v.hashCache = map[string][32]byte{} // proposals of finished heights are never asked for again
	}
	v.mu.Unlock()
	v.currentHeight.Store(height)
	return err
}

func (v *Verifier) SetCurrentHeight(h uint64) {
	v.mu.Lock()
	if h > v.currentHeight.Load() {
		v.hashCache = map[string][32]byte{}
	}
	v.mu.Unlock()
	v.currentHeight.Store(h)
}

func (v *Verifier) IsValidProposal(raw []byte) bool { return v.IsValidBlockFn == nil || v.IsValidBlockFn(raw) }
func (v *Verifier) IsProposer(id []byte, h, r uint64) bool {
	return v.IsProposerFn != nil && v.IsProposerFn(id, h, r)
}

func senderItem(m *proto.IbftMessage) (Item, string, bool) {
	if m == nil || m.View == nil || len(m.From) != 20 || len(m.Signature) != 65 {
		return Item{}, "", false
	}
	payload, err := m.PayloadNoSig() // messages/proto/helper.go:13-27
	if err != nil {
		return Item{}, "", false
	}
	var hb [8]byte
	binary.BigEndian.PutUint64(hb[:], m.View.Height)
	key := "S" + string(hb[:]) + string(m.Signature) + string(payload)
	return Item{Kind: C.IBFT_KIND_PAYLOAD, Sig: m.Signature, Signer: m.From, Payload: payload, Height: m.View.Height}, key, true
}

func (v *Verifier) sealItem(hash []byte, seal *messages.CommittedSeal) (Item, string, bool) {
	if hash == nil || seal == nil || len(hash) != 32 || len(seal.Signer) != 20 || len(seal.Signature) != 65 {
		return Item{}, "", false
	}
	h := v.currentHeight.Load()
	var hb [8]byte
	binary.BigEndian.PutUint64(hb[:], h)
	key := "C" + string(hb[:]) + string(seal.Signature) + string(seal.Signer) + string(hash)
	return Item{Kind: C.IBFT_KIND_SEAL, Sig: seal.Signature, Signer: seal.Signer, Hash: hash, Height: h}, key, true
}

// verifyBatch: one device call; verdicts are cached only if no validator table changed meanwhile.  nil on a failed launch.
func (v *Verifier) verifyBatch(items []Item, keys []string) []bool {
	if len(items) == 0 {
		return nil
	}
	v.mu.Lock()
	epoch := v.epoch
	v.mu.Unlock()
	res, err := v.Eng.VerifyBatch(items)
	if err != nil {
		return nil // launch failure: no verdict, never true
	}
	v.mu.Lock()
	if epoch == v.epoch {
		for i, k := range keys {
			v.cache[k] = res[i]
		}
	}
	v.mu.Unlock()
	return res
}

// lookupOrCoalesce: the reference calls IsValidValidator once per inbound gossip message from any number of goroutines
// (core/ibft.go:1101-1128).  A cache miss does NOT become a device call of one item: it joins the ingress queue; ONE caller at
// a time is the leader, takes everything queued (its own request included), makes a single device call, publishes the verdicts
// and wakes the others.  Requests arriving while a flush is on the device pile up and form the next batch (group commit).
func (v *Verifier) lookupOrCoalesce(it Item, key string) bool {
	v.mu.Lock()
	if ok, hit := v.cache[key]; hit {
		v.mu.Unlock()
		return ok
	}
	v.mu.Unlock()
	req := &ingressReq{it: it, key: key}
	v.ingMu.Lock()
	v.ingQueue = append(v.ingQueue, req)
	for !req.done {
		if v.ingLeader {
			v.ingCond.Wait()
			continue
		}
		v.ingLeader = true
		if v.IngressLinger > 0 && len(v.ingQueue) < v.IngressMinBatch {
			v.ingMu.Unlock()
			time.Sleep(v.IngressLinger)
			v.ingMu.Lock()
		}
		n := len(v.ingQueue)
		if n > v.IngressMaxBatch {
			n = v.IngressMaxBatch
		}
		taken := v.ingQueue[:n:n]
		v.ingQueue = append([]*ingressReq(nil), v.ingQueue[n:]...)
		v.ingMu.Unlock()
		// duplicates (the same message relayed by several peers) are verified once
		var items []Item
		var keys []string
		slot := make([]int, len(taken))
		seen := map[string]int{}
		for i, r := range taken {
			j, ok := seen[r.key]
			if !ok {
				j = len(items)
				seen[r.key] = j
				items, keys = append(items, r.it), append(keys, r.key)
			}
			slot[i] = j
		}
		res := v.verifyBatch(items, keys)
		v.ingMu.Lock()
		for i, r := range taken {
			r.result = res != nil && res[slot[i]]
			r.done = true
		}
		v.ingLeader = false
		v.ingCond.Broadcast()
		v.ingMu.Unlock()
		v.reportRejects(items, res)
		v.ingMu.Lock()
	}
	v.ingMu.Unlock()
	return req.result
}

// reportRejects: one ExplainBatch call over the items a device call rejected, then OnReject for each
func (v *Verifier) reportRejects(items []Item, res []bool) {
	if v.OnReject == nil || res == nil {
		return
	}
	var rejected []Item
	for i, ok := range res {
		if !ok {
			rejected = append(rejected, items[i])
		}
	}
	if len(rejected) == 0 {
		return
	}
	reasons, recovered, err := v.Eng.ExplainBatch(rejected)
	if err != nil {
		return
	}
	for i, r := range reasons {
		if r != ReasonOK { // ReasonOK: rejected on the host (no resident table), not by the device
			v.OnReject(rejected[i], r, recovered[i])
		}
	}
}

// IsValidValidator: signer of msg.Signature over Keccak-256(PayloadNoSig) == msg.From and From is a validator at
// msg.View.Height (core/backend.go:41-45).
func (v *Verifier) IsValidValidator(m *proto.IbftMessage) bool {
	it, key, ok := senderItem(m)
	return ok && v.lookupOrCoalesce(it, key)
}

// IsValidCommittedSeal (core/backend.go:53-55).
func (v *Verifier) IsValidCommittedSeal(hash []byte, seal *messages.CommittedSeal) bool {
	it, key, ok := v.sealItem(hash, seal)
	return ok && v.lookupOrCoalesce(it, key)
}

// IsValidProposalHash with the synthetic convention of SURVEY.md §8(c): Keccak-256(Keccak-256(raw) || u64_be(round)).
// A real embedder substitutes its own block hash here; the point is that it is computed once per (proposal, round), not once
// per PREPARE and COMMIT (core/ibft.go:858, :938).
func (v *Verifier) IsValidProposalHash(p *proto.Proposal, hash []byte) bool {
	if p == nil || len(hash) != 32 {
		return false
	}
	var rb [8]byte
	binary.BigEndian.PutUint64(rb[:], p.Round)
	key := string(p.RawProposal) + string(rb[:])
	v.mu.Lock()
	want, hit := v.hashCache[key]
	v.mu.Unlock()
	if !hit {
		if v.ProposalHashFn != nil {
			want = v.ProposalHashFn(p.RawProposal, p.Round)
		} else {
			var err error
			want, err = v.Eng.ProposalHash(p.RawProposal, p.Round)
			if err != nil {
				return false
			}
		}
		v.mu.Lock()
		if len(v.hashCache) >= maxHashCache { // entries are proposal-sized: bounded against ROUND_CHANGE floods
			v.hashCache = map[string][32]byte{}
		}
		v.hashCache[key] = want
		v.mu.Unlock()
	}
	return string(want[:]) == string(hash)
}

// Prefetch verifies, in ONE device call, every sender signature (and committed seal, and nested certificate signature) of
// the messages a handler is about to validate; the per-message methods above then answer from the cache.  Called by the
// batching shim in messages.GetValidMessages / GetExtendedRCC (go/patches/messages_messages.patch).
func (v *Verifier) Prefetch(msgs []*proto.IbftMessage, withSeals bool) {
	var items []Item
	var keys []string
	seen := map[string]bool{}
	depth := 0
	var visit func(m *proto.IbftMessage)
	add := func(it Item, key string, ok bool) {
		if !ok || seen[key] {
			return
		}
		v.mu.Lock()
		_, hit := v.cache[key]
		v.mu.Unlock()
		if !hit {
			seen[key] = true
			items, keys = append(items, it), append(keys, key)
		}
	}
	visit = func(m *proto.IbftMessage) {
		if m == nil || depth > 32 {
			return
		}
		depth++
		add(senderItem(m))
		if withSeals {
			if seal := messages.ExtractCommittedSeal(m); seal != nil {
				add(v.sealItem(messages.ExtractCommitHash(m), seal))
			}
		}
		if pc := messages.ExtractLatestPC(m); pc != nil {
			visit(pc.ProposalMessage)
			for _, p := range pc.PrepareMessages {
				visit(p)
			}
		}
		if rcc := messages.ExtractRoundChangeCertificate(m); rcc != nil {
			for _, rc := range rcc.RoundChangeMessages {
				visit(rc)
			}
		}
		depth--
	}
	for _, m := range msgs {
		visit(m)
	}
	v.reportRejects(items, v.verifyBatch(items, keys))
}
