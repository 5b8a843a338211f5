// Package gpubackend binds the H100 verification engine (include/ibft_verify.h, libibftverify.so) through cgo and
// implements the hot-path half of go-ibft's core.Backend: core.Verifier (core/backend.go:37-56).
//
// COMPILE-UNVERIFIED: the authoring image has no Go toolchain.  The C ABI below is exercised by the ctypes harness
// (go-ibft_b200/engine.py) and the C++ host mirror (go-ibft_b200/host) in the test-suite; this file shows the binding a
// maintainer adds on the Go side.
package gpubackend

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../go-ibft_b200 -libftverify -Wl,-rpath,${SRCDIR}/../../go-ibft_b200
#include <stdlib.h>
#include <string.h>
#include "ibft_verify.h"
*/
import "C"

import (
	"errors"
	"fmt"
	"math/big"
	"sync"
	"unsafe"
)

// Engine owns one ibft_engine (one per process per GPU).  The engine itself runs up to two host-buffer calls at a time (a
// full-capacity lane and a small lane for ingress batches); VerifyBatch may be called from any number of goroutines.
type Engine struct {
	h      *C.ibft_engine
	params C.ibft_engine_params
	mu     sync.RWMutex      // guards slotHeight
	// slotHeight[slot] = height of the validator table resident in that slot.  A message of another height that maps to the same
	// slot (height % slots) must NOT be checked against it: isAcceptableMessage admits any future height (core/ibft.go:1139-1148),
	// so H + k*slots would otherwise be answered from H's validator set.  The engine checks ibft_group_desc.height as well.
	slotHeight map[uint32]uint64
}

type Params struct {
	Device, MaxItems, MaxPayloadBytes, MaxGroups, MaxTableSlots, MaxValidators uint32
	// KeyCache sets IBFT_FLAG_KEY_CACHE: the engine learns every validator's public key from its first valid signature and
	// verifies (instead of recovering) that validator's later signatures against a per-validator comb table in device memory
	// (136 KiB per validator and resident table: 1.39 GB for 10,000 validators); verdicts are identical.  SetValidators for
	// the next height carries the tables over by address, so only newcomers are ever recovered again.  ~2.7x the recover
	// path's throughput, 0.48 ms instead of 0.8 ms for a 10k-validator COMMIT round (DESIGN.md section 3.1c).
	KeyCache bool
}

func lastError() error { return errors.New(C.GoString(C.ibft_last_error())) }

// NewEngine fails when no CUDA device is usable: there is no CPU fallback (IBFT_ERR_NO_DEVICE).
func NewEngine(p Params) (*Engine, error) {
	e := &Engine{slotHeight: map[uint32]uint64{}}
	e.params = C.ibft_engine_params{device: C.int32_t(p.Device), max_items: C.uint32_t(p.MaxItems),
		max_payload_bytes: C.uint32_t(p.MaxPayloadBytes), max_groups: C.uint32_t(p.MaxGroups),
		max_table_slots: C.uint32_t(p.MaxTableSlots), max_validators: C.uint32_t(p.MaxValidators)}
	if p.KeyCache {
		e.params.flags = C.IBFT_FLAG_KEY_CACHE
	}
	if rc := C.ibft_engine_create(&e.params, &e.h); rc != C.IBFT_OK {
		return nil, fmt.Errorf("ibft_engine_create: %w", lastError())
	}
	return e, nil
}

// RecoverPath values for SetRecoverPath (include/ibft_verify.h IBFT_PATH_*).  The verdicts are identical on every path.
const (
	PathAuto   = 0 // by batch size (default): small rounds take the latency kernels, large backlogs the throughput kernel
	PathThread = 1
	PathQuad   = 2
	PathSplit  = 3
	PathQSplit = 4
)

// SetRecoverPath pins the recover kernel (diagnostics / benchmarks); production code leaves it on PathAuto.
func (e *Engine) SetRecoverPath(path int) error {
	if rc := C.ibft_set_recover_path(e.h, C.int(path)); rc != C.IBFT_OK {
		return lastError()
	}
	return nil
}

func (e *Engine) Close() {
	if e.h != nil {
		C.ibft_engine_destroy(e.h)
		e.h = nil
	}
}

// SetValidators pushes Backend.GetVotingPowers(height) (core/validator_manager.go:50-57) to the device table of `height`.
// order fixes the validator index of each address (needed to read the voted-set bitmap back).
func (e *Engine) SetValidators(height uint64, order [][]byte, powers map[string]*big.Int) error {
	addrs := make([]byte, 0, 20*len(order))
	pw := make([]byte, 0, 32*len(order))
	for _, a := range order {
		if len(a) != 20 {
			continue // can never equal a recovered signer
		}
		addrs = append(addrs, a...)
		var buf [32]byte
		powers[string(a)].FillBytes(buf[:])
		pw = append(pw, buf[:]...)
	}
	slot := C.uint32_t(height % uint64(e.params.max_table_slots))
	var ap, pp *C.uint8_t
	if len(addrs) > 0 {
		ap, pp = (*C.uint8_t)(unsafe.Pointer(&addrs[0])), (*C.uint8_t)(unsafe.Pointer(&pw[0]))
	}
	// the slot stops answering for its old height BEFORE the engine swaps the table
	e.mu.Lock()
	delete(e.slotHeight, uint32(slot))
	e.mu.Unlock()
	if rc := C.ibft_set_validators(e.h, slot, C.uint64_t(height), ap, pp, C.uint32_t(len(addrs)/20)); rc != C.IBFT_OK {
		return fmt.Errorf("ibft_set_validators: %w", lastError())
	}
	e.mu.Lock()
	e.slotHeight[uint32(slot)] = height
	e.mu.Unlock()
	return nil
}

// Item is one signature check; it is marshalled into the packed 128-byte ibft_sig_item.
type Item struct {
	Kind    uint8 // C.IBFT_KIND_PAYLOAD (sender signature over PayloadNoSig) or C.IBFT_KIND_SEAL (committed seal)
	Sig     []byte
	Signer  []byte
	Hash    []byte // KIND_SEAL: proposal hash
	Payload []byte // KIND_PAYLOAD: IbftMessage.PayloadNoSig() (messages/proto/helper.go:13-27)
	Height  uint64
	Group   uint16 // VerifyGroups only: index into its groups (VerifyBatch groups items by Height)
}

// packItem marshals one item into its packed tuple (payload bytes appended to *arena); false for a malformed item, which is
// packed as IBFT_KIND_INVALID.
func packItem(p *C.ibft_sig_item, it Item, arena *[]byte) bool {
	if len(it.Sig) != 65 || len(it.Signer) != 20 || (it.Kind == C.IBFT_KIND_SEAL && len(it.Hash) != 32) {
		p.kind = C.IBFT_KIND_INVALID // malformed => false (messages/helpers.go:38-42 nil seal etc.)
		return false
	}
	C.memcpy(unsafe.Pointer(&p.r[0]), unsafe.Pointer(&it.Sig[0]), 32)
	C.memcpy(unsafe.Pointer(&p.s[0]), unsafe.Pointer(&it.Sig[32]), 32)
	p.v = C.uint8_t(it.Sig[64])
	C.memcpy(unsafe.Pointer(&p.signer[0]), unsafe.Pointer(&it.Signer[0]), 20)
	p.kind = C.uint8_t(it.Kind)
	if it.Kind == C.IBFT_KIND_SEAL {
		C.memcpy(unsafe.Pointer(&p.digest[0]), unsafe.Pointer(&it.Hash[0]), 32)
	} else {
		p.payload_off, p.payload_len = C.uint32_t(len(*arena)), C.uint32_t(len(it.Payload))
		*arena = append(*arena, it.Payload...)
	}
	return true
}

// VerifyBatch runs ONE device call for all items and returns one verdict per item.  A failed launch returns an error and
// NO verdicts (callers treat that as "not valid yet", never as true).  Go memory is only read during the call: the ABI
// copies into engine-owned pinned staging.
func (e *Engine) VerifyBatch(items []Item) ([]bool, error) {
	n := len(items)
	if n == 0 {
		return nil, nil
	}
	packed := make([]C.ibft_sig_item, n)
	var arena []byte
	groups := []C.ibft_group_desc{}
	groupOf := map[uint64]uint16{}
	noTable := map[uint16]bool{} // groups whose height has no resident table: verdict forced to false
	e.mu.RLock()
	for i, it := range items {
		p := &packed[i]
		if !packItem(p, it, &arena) {
			continue
		}
		g, ok := groupOf[it.Height]
		if !ok {
			g = uint16(len(groups))
			groupOf[it.Height] = g
			slot := uint32(it.Height % uint64(e.params.max_table_slots))
			d := C.ibft_group_desc{table_slot: C.IBFT_NO_TABLE, height: C.uint64_t(it.Height)}
			if h, set := e.slotHeight[slot]; set && h == it.Height {
				d.table_slot = C.uint16_t(slot)
			} else {
				// a height whose validator table is not resident has no members: false, never another height's table
				noTable[g] = true
			}
			groups = append(groups, d)
		}
		p.group = C.uint16_t(g)
	}
	e.mu.RUnlock()
	bitmap := make([]uint32, (n+31)/32)
	var ap *C.uint8_t
	if len(arena) > 0 {
		ap = (*C.uint8_t)(unsafe.Pointer(&arena[0]))
	}
	var gp *C.ibft_group_desc
	if len(groups) > 0 {
		gp = &groups[0]
	}
	// _ex: everything comes back with the call itself (a goroutine may change OS threads between two cgo calls, so the
	// "last call" getters are not usable from Go)
	rc := C.ibft_verify_batch_ex(e.h, &packed[0], C.uint32_t(n), ap, C.size_t(len(arena)), gp, C.uint32_t(len(groups)),
		(*C.uint32_t)(unsafe.Pointer(&bitmap[0])), nil, nil, nil, nil, 0)
	if rc != C.IBFT_OK {
		return nil, fmt.Errorf("ibft_verify_batch_ex: %w", lastError())
	}
	out := make([]bool, n)
	for i := range out {
		out[i] = bitmap[i/32]>>(uint(i)%32)&1 == 1 && !noTable[uint16(packed[i].group)]
	}
	return out, nil
}

// Quorum rules of a Group (include/ibft_verify.h IBFT_QUORUM_*): which of go-ibft's per-message-type decisions
// (hasQuorumByMsgType, core/ibft.go:1273-1284) the engine returns as the group's HasQuorum.
const (
	QuorumDefault    = uint16(C.IBFT_QUORUM_DEFAULT)    // HasQuorum: COMMIT, ROUND_CHANGE, validPC's PREPREPARE + PREPARE senders
	QuorumPrePrepare = uint16(C.IBFT_QUORUM_PREPREPARE) // at least one valid message
	QuorumPrepare    = uint16(C.IBFT_QUORUM_PREPARE)    // HasPrepareQuorum (core/validator_manager.go:99-127); needs Proposer
	ProposerNone     = uint32(C.IBFT_PROPOSER_NONE)     // the proposer is not a validator of the group's table
	ProposerUnset    = uint32(C.IBFT_PROPOSER_UNSET)    // there is no proposal message: HasQuorum is false
)

// Group is one quorum domain of VerifyGroups: the items of one (height, round, message type).
type Group struct {
	Height uint64
	Rule   uint16 // QuorumDefault, QuorumPrePrepare or QuorumPrepare
	// QuorumPrepare: the proposer's index in the validator table of Height (the order given to SetValidators, without the
	// entries it skipped), ProposerNone or ProposerUnset.  The caller decides who the proposer is (IsProposer).
	Proposer uint32
}

// GroupResult is the engine's quorum result of one Group (ibft_group_result).
type GroupResult struct {
	HasQuorum         bool
	NValid, NDistinct uint32
	Power             *big.Int // voting power of the distinct valid senders; under QuorumPrepare the proposer's is included
}

// VerifyGroups runs ONE device call for all items, each in groups[item.Group], and returns the verdicts and every group's
// quorum decision under its rule.  A group whose height has no resident validator table fails the call (IBFT_ERR_NO_TABLE).
func (e *Engine) VerifyGroups(items []Item, groups []Group) ([]bool, []GroupResult, error) {
	n := len(items)
	if n == 0 || len(groups) == 0 {
		return nil, nil, errors.New("VerifyGroups needs items and groups")
	}
	descs := make([]C.ibft_group_desc, len(groups))
	e.mu.RLock()
	for g, gr := range groups {
		slot := uint32(gr.Height % uint64(e.params.max_table_slots))
		if h, set := e.slotHeight[slot]; !set || h != gr.Height {
			e.mu.RUnlock()
			return nil, nil, fmt.Errorf("group %d: no validator table for height %d", g, gr.Height)
		}
		descs[g] = C.ibft_group_desc{table_slot: C.uint16_t(slot), flags: C.uint16_t(gr.Rule), height: C.uint64_t(gr.Height)}
		if gr.Rule == QuorumPrepare {
			descs[g].reserved = C.uint32_t(gr.Proposer)
		}
	}
	e.mu.RUnlock()
	packed := make([]C.ibft_sig_item, n)
	var arena []byte
	for i, it := range items {
		if int(it.Group) >= len(groups) {
			return nil, nil, fmt.Errorf("item %d: group %d out of range", i, it.Group)
		}
		packed[i].group = C.uint16_t(it.Group)
		packItem(&packed[i], it, &arena)
	}
	bitmap := make([]uint32, (n+31)/32)
	results := make([]C.ibft_group_result, len(groups))
	var ap *C.uint8_t
	if len(arena) > 0 {
		ap = (*C.uint8_t)(unsafe.Pointer(&arena[0]))
	}
	rc := C.ibft_verify_batch_ex(e.h, &packed[0], C.uint32_t(n), ap, C.size_t(len(arena)), &descs[0], C.uint32_t(len(descs)),
		(*C.uint32_t)(unsafe.Pointer(&bitmap[0])), &results[0], nil, nil, nil, 0)
	if rc != C.IBFT_OK {
		return nil, nil, fmt.Errorf("ibft_verify_batch_ex: %w", lastError())
	}
	out := make([]bool, n)
	for i := range out {
		out[i] = bitmap[i/32]>>(uint(i)%32)&1 == 1
	}
	res := make([]GroupResult, len(groups))
	for g, r := range results {
		p := new(big.Int)
		for k := 4; k >= 0; k-- {
			p.Lsh(p, 64).Or(p, new(big.Int).SetUint64(uint64(r.power[k])))
		}
		res[g] = GroupResult{HasQuorum: r.has_quorum != 0, NValid: uint32(r.n_valid), NDistinct: uint32(r.n_distinct), Power: p}
	}
	return out, res, nil
}

// ProposalHash = Keccak-256(Keccak-256(raw) || u64_be(round)), both sponges in one device launch (IsValidProposalHash,
// core/backend.go:50-51; the synthetic convention of SURVEY.md §8c -- a real embedder substitutes its block hash).
func (e *Engine) ProposalHash(raw []byte, round uint64) ([32]byte, error) {
	var out [32]byte
	off, ln, rd := C.uint32_t(0), C.uint32_t(len(raw)), C.uint64_t(round)
	var dp *C.uint8_t
	if len(raw) > 0 {
		dp = (*C.uint8_t)(unsafe.Pointer(&raw[0]))
	}
	if rc := C.ibft_proposal_hash_batch(e.h, dp, C.size_t(len(raw)), &off, &ln, &rd, 1, (*C.uint8_t)(unsafe.Pointer(&out[0]))); rc != C.IBFT_OK {
		return out, lastError()
	}
	return out, nil
}

// Keccak256 hashes on the device (IsValidProposalHash, core/backend.go:50-51).
func (e *Engine) Keccak256(data []byte) ([32]byte, error) {
	var out [32]byte
	off, ln := C.uint32_t(0), C.uint32_t(len(data))
	var dp *C.uint8_t
	if len(data) > 0 {
		dp = (*C.uint8_t)(unsafe.Pointer(&data[0]))
	}
	if rc := C.ibft_keccak256_batch(e.h, dp, C.size_t(len(data)), &off, &ln, 1, (*C.uint8_t)(unsafe.Pointer(&out[0]))); rc != C.IBFT_OK {
		return out, lastError()
	}
	return out, nil
}
