// Package mrq is the cgo binding of libmrq.so (include/mrq.h) — the Hopper-native multi-raft quorum
// engine.  SOURCE ONLY: there is no Go toolchain in the build image, so this file has never been compiled;
// it is the binding a maintainer of chzchzchz/raftsql would add next to raft.go (see INTEGRATION.md).
//
// cgo rules observed: C never retains a Go pointer after a call returns (every mrq_* entry point copies
// its inputs before returning); outputs are written into Go-owned slices passed for the duration of the
// call; there are no callbacks from C into Go.
package mrq

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../raftsql_b200 -lmrq
#include <stdlib.h>
#include "mrq.h"
*/
import "C"

import (
	"errors"
	"fmt"
	"unsafe"
)

// Message types (raftpb.MessageType numbering of the etcd v2.2/v2.3 era).
const (
	MsgApp           = C.MRQ_MSG_APP
	MsgAppResp       = C.MRQ_MSG_APP_RESP
	MsgVote          = C.MRQ_MSG_VOTE
	MsgVoteResp      = C.MRQ_MSG_VOTE_RESP
	MsgHeartbeat     = C.MRQ_MSG_HEARTBEAT
	MsgHeartbeatResp = C.MRQ_MSG_HEARTBEAT_RESP
	MsgReject        = C.MRQ_MSG_REJECT
)

// Out-word flags (the engine's stand-in for Ready.Messages, reference raft.go:227-230).
const (
	OutCampaign       = C.MRQ_OUT_CAMPAIGN
	OutBecameLeader   = C.MRQ_OUT_BECAME_LEADER
	OutBcastAppend    = C.MRQ_OUT_BCAST_APPEND
	OutBcastHeartbeat = C.MRQ_OUT_BCAST_HEARTBEAT
	OutSteppedDown    = C.MRQ_OUT_STEPPED_DOWN
	OutPropDropped    = C.MRQ_OUT_PROP_DROPPED
	OutPropForward    = C.MRQ_OUT_PROP_FORWARD
	OutCommitAdvanced = C.MRQ_OUT_COMMIT_ADVANCED
	OutVoteReplyShift = C.MRQ_OUT_VOTE_REPLY_SHIFT
	OutAckReplyShift  = C.MRQ_OUT_ACK_REPLY_SHIFT
)

const (
	RoleFollower  = C.MRQ_ROLE_FOLLOWER
	RoleCandidate = C.MRQ_ROLE_CANDIDATE
	RoleLeader    = C.MRQ_ROLE_LEADER
)

// Config mirrors raft.Config as the reference fills it (raft.go:152-159), for G groups.
type Config struct {
	Groups        uint64 // G
	GroupBase     uint64
	Replicas      uint32 // len(peers), raft.go:148
	SelfID        uint32 // raft.Config.ID, raft.go:153
	ElectionTick  uint32 // raft.go:154 (10)
	HeartbeatTick uint32 // raft.go:155 (1)
	Seed          uint64
	Device        int32
	InboxSlots    uint32
}

// Msg is one inbound raftpb.Message reduced to the fields the path reads.
type Msg struct {
	Group, Term, Index, LogTerm, Commit uint64
	Type, From                          uint8
}

// Engine is this node's replica of Config.Groups raft groups, resident on one H100.
// One goroutine drives one Engine, like the single select loop of reference raft.go:221-245.
type Engine struct {
	h *C.mrq_engine
	g uint64
	r uint32
}

func lastErr(h *C.mrq_engine) error { return errors.New(C.GoString(C.mrq_last_error(h))) }

// New is raft.StartNode for G groups (reference raft.go:161-165).
func New(c Config) (*Engine, error) {
	var cfg C.mrq_config
	C.mrq_config_default(&cfg)
	cfg.n_groups = C.uint64_t(c.Groups)
	cfg.group_base = C.uint64_t(c.GroupBase)
	cfg.n_replicas = C.uint32_t(c.Replicas)
	cfg.self_id = C.uint32_t(c.SelfID)
	if c.ElectionTick != 0 {
		cfg.election_tick = C.uint32_t(c.ElectionTick)
	}
	if c.HeartbeatTick != 0 {
		cfg.heartbeat_tick = C.uint32_t(c.HeartbeatTick)
	}
	cfg.seed = C.uint64_t(c.Seed)
	cfg.device = C.int32_t(c.Device)
	if c.InboxSlots != 0 {
		cfg.inbox_slots = C.uint32_t(c.InboxSlots)
	}
	var h *C.mrq_engine
	if rc := C.mrq_create(&cfg, &h); rc != 0 {
		return nil, fmt.Errorf("mrq_create: %d: %s", int(rc), C.GoString(C.mrq_last_error(nil)))
	}
	return &Engine{h: h, g: c.Groups, r: c.Replicas}, nil
}

// Close is node.Stop() (reference raft.go:141,195).
func (e *Engine) Close() {
	if e.h != nil {
		C.mrq_destroy(e.h)
		e.h = nil
	}
}

// Step posts the tick's inbound messages (node.Step, reference raft.go:268-270), sparse form.
func (e *Engine) Step(slot uint32, msgs []Msg) error {
	if len(msgs) == 0 {
		if rc := C.mrq_clear_inbox(e.h, C.uint32_t(slot)); rc != 0 {
			return lastErr(e.h)
		}
		return nil
	}
	buf := make([]C.mrq_msg, len(msgs))
	for i, m := range msgs {
		buf[i].group, buf[i].term, buf[i].index = C.uint64_t(m.Group), C.uint64_t(m.Term), C.uint64_t(m.Index)
		buf[i].logterm, buf[i].commit = C.uint64_t(m.LogTerm), C.uint64_t(m.Commit)
		buf[i]._type, buf[i].from = C.uint8_t(m.Type), C.uint8_t(m.From)
	}
	if rc := C.mrq_post_inbox_delta(e.h, C.uint32_t(slot), &buf[0], C.size_t(len(buf)), 0); rc != 0 {
		return lastErr(e.h)
	}
	return nil
}

// Propose is node.Propose (reference raft.go:211-215): count entries per group; payloads stay in Go.
func (e *Engine) Propose(slot uint32, groups []uint64, counts []uint32) error {
	if len(groups) == 0 {
		return nil
	}
	rc := C.mrq_propose(e.h, C.uint32_t(slot), (*C.uint64_t)(unsafe.Pointer(&groups[0])),
		(*C.uint32_t)(unsafe.Pointer(&counts[0])), C.size_t(len(groups)))
	if rc != 0 {
		return lastErr(e.h)
	}
	return nil
}

// Tick is node.Tick() for every group (reference raft.go:223-224) fused with the Step of the posted
// inbox: one sm_90a kernel launch.
func (e *Engine) Tick(slot uint32) error {
	if rc := C.mrq_tick(e.h, C.uint32_t(slot)); rc != 0 {
		return lastErr(e.h)
	}
	return nil
}

// Ready drains what <-node.Ready() would carry (reference raft.go:227): HardState{Term,Commit} and the
// per-group out word.  Slices must have Groups elements.
func (e *Engine) Ready(committed, term []uint64, role []uint8, out []uint32) error {
	var pc, pt *C.uint64_t
	var pr *C.uint8_t
	if committed != nil {
		pc = (*C.uint64_t)(unsafe.Pointer(&committed[0]))
	}
	if term != nil {
		pt = (*C.uint64_t)(unsafe.Pointer(&term[0]))
	}
	if role != nil {
		pr = (*C.uint8_t)(unsafe.Pointer(&role[0]))
	}
	if rc := C.mrq_sync_commits(e.h, pc, pr, pt); rc != 0 {
		return lastErr(e.h)
	}
	if out != nil {
		if rc := C.mrq_sync_out(e.h, (*C.uint32_t)(unsafe.Pointer(&out[0]))); rc != 0 {
			return lastErr(e.h)
		}
	}
	return nil
}

// QuorumCommit runs the standalone quorum kernel (maybeCommit on every leader group).
func (e *Engine) QuorumCommit() error {
	if rc := C.mrq_quorum_commit(e.h); rc != 0 {
		return lastErr(e.h)
	}
	return nil
}

// ---- the dense multi-raft path: byte frames on compact state (tick mode 4) ----------------------------------
// A host that leads (or follows) a million groups does not post messages one by one: per tick it encodes the
// whole inbox into ONE byte frame — R-1 sender bytes + 1 proposal byte per group (include/mrq_packed8.h) — ships
// it, ticks, and drains one byte per group (that tick's commit advance).  The frame buffers must be C memory
// (cgo: C may not keep Go pointers across calls, and the copy is asynchronous): AllocPinned / FreePinned.

// SetTickMode selects how Tick runs (include/mrq.h mrq_set_tick_mode); 4 = byte frames on compact state.
func (e *Engine) SetTickMode(mode int) error {
	if rc := C.mrq_set_tick_mode(e.h, C.int(mode)); rc != 0 {
		return lastErr(e.h)
	}
	return nil
}

// AllocPinned returns n bytes of page-locked C memory as a Go slice (not managed by the Go GC).
func AllocPinned(n int) []byte {
	p := C.mrq_alloc_pinned(C.size_t(n))
	if p == nil {
		return nil
	}
	return unsafe.Slice((*byte)(p), n)
}

// FreePinned releases a slice obtained from AllocPinned.
func FreePinned(b []byte) {
	if len(b) > 0 {
		C.mrq_free_pinned(unsafe.Pointer(&b[0]))
	}
}

// SetPackedBase hands the engine the window bases the frame builder starts from (one per group).
func (e *Engine) SetPackedBase(baseIndex, baseTerm []uint64) error {
	rc := C.mrq_set_packed_base(e.h, (*C.uint64_t)(unsafe.Pointer(&baseIndex[0])), (*C.uint64_t)(unsafe.Pointer(&baseTerm[0])))
	if rc != 0 {
		return lastErr(e.h)
	}
	return nil
}

// PostFrame starts the asynchronous copy of one byte frame (word: [R-1][G] in pinned memory, prop8: [G]) into
// inbox slot `slot`; wide carries the few messages that did not fit a byte.  Returns at once: the copy overlaps
// whatever tick is running.
func (e *Engine) PostFrame(slot uint32, word, prop8 []byte, wide []Msg) error {
	var v C.mrq_inbox_packed
	v.word = unsafe.Pointer(&word[0])
	v.prop_count8 = (*C.uint8_t)(unsafe.Pointer(&prop8[0]))
	v.word_bits = 8
	if len(wide) > 0 {
		// cgo: a struct handed to C must not hold pointers into Go memory, so the escape list lives in C memory for the
		// call (the engine copies it before returning: include/mrq.h, ownership rules)
		n := C.size_t(len(wide)) * C.size_t(unsafe.Sizeof(C.mrq_msg{}))
		cbuf := (*C.mrq_msg)(C.malloc(n))
		defer C.free(unsafe.Pointer(cbuf))
		buf := unsafe.Slice(cbuf, len(wide))
		for i, m := range wide {
			buf[i] = C.mrq_msg{}
			buf[i].group, buf[i].term, buf[i].index = C.uint64_t(m.Group), C.uint64_t(m.Term), C.uint64_t(m.Index)
			buf[i].logterm, buf[i].commit = C.uint64_t(m.LogTerm), C.uint64_t(m.Commit)
			buf[i]._type, buf[i].from = C.uint8_t(m.Type), C.uint8_t(m.From)
		}
		v.wide, v.n_wide = cbuf, C.size_t(len(wide))
	}
	if rc := C.mrq_post_inbox_packed(e.h, C.uint32_t(slot), &v); rc != 0 {
		return lastErr(e.h)
	}
	return nil
}

// DrainTick enqueues the copy of the last tick's commit advances (one byte per group, 255 = read the index in
// full with Ready) into pinned memory; Wait blocks until THAT copy has landed.
func (e *Engine) DrainTick(deltaPinned []byte) error {
	if rc := C.mrq_drain_tick_deltas(e.h, (*C.uint8_t)(unsafe.Pointer(&deltaPinned[0]))); rc != 0 {
		return lastErr(e.h)
	}
	return nil
}

// Wait blocks until the drain enqueued last has landed on the host.
func (e *Engine) Wait() error {
	if rc := C.mrq_drain_wait(e.h); rc != 0 {
		return lastErr(e.h)
	}
	return nil
}

// TickMany runs the ticks of the given inbox slots in ONE pair of kernel launches (tick mode 4: every thread
// carries its groups' state in registers from tick to tick) — a backlog of posted frames, or a replay.
func (e *Engine) TickMany(slots []uint32) error {
	if len(slots) == 0 {
		return nil
	}
	if rc := C.mrq_tick_many(e.h, (*C.uint32_t)(unsafe.Pointer(&slots[0])), C.uint32_t(len(slots))); rc != 0 {
		return lastErr(e.h)
	}
	return nil
}

// SlotOutputs reads the out words and commit advances of the tick that consumed `slot` in the last TickMany.
func (e *Engine) SlotOutputs(slot uint32, out []uint32, delta []byte) error {
	rc := C.mrq_sync_slot_outputs(e.h, C.uint32_t(slot), (*C.uint32_t)(unsafe.Pointer(&out[0])), (*C.uint8_t)(unsafe.Pointer(&delta[0])))
	if rc != 0 {
		return lastErr(e.h)
	}
	return nil
}

// Change-feed flags: which of HardState {Term, Vote} and SoftState {RaftState, Lead} a tick moved.
const (
	ChangeTerm = C.MRQ_CHANGE_TERM
	ChangeVote = C.MRQ_CHANGE_VOTE
	ChangeRole = C.MRQ_CHANGE_ROLE
	ChangeLead = C.MRQ_CHANGE_LEAD
)

// Change is one change-feed record: group's term, vote, role or lead after tick Tick differ from before it.
// TermStart is the new leader's empty entry (math.MaxUint64 unless Role == RoleLeader).
type Change struct {
	Tick, Term, TermStart uint64
	Group                 uint32
	Vote, Role, Lead      uint8
	What                  uint8 // Change* bits, never 0
}

// SetChangeCapacity turns the change feed on with room for n records between drains (0 turns it off).
func (e *Engine) SetChangeCapacity(n uint64) error {
	if rc := C.mrq_set_change_capacity(e.h, C.uint64_t(n)); rc != 0 {
		return lastErr(e.h)
	}
	return nil
}

// SyncChanges drains the change feed: every record since the previous drain, sorted by (Tick, Group).  lost > 0
// means records did not fit the capacity: the list is incomplete and the host must read the state in full.
func (e *Engine) SyncChanges() (changes []Change, lost uint64, err error) {
	buf := make([]C.mrq_change, 1024)
	var n, l C.uint64_t
	for {
		rc := C.mrq_sync_changes(e.h, &buf[0], C.uint64_t(len(buf)), &n, &l)
		if rc == C.MRQ_E_INVAL && uint64(n) > uint64(len(buf)) { // nothing was consumed: retry with room for all
			buf = make([]C.mrq_change, int(n))
			continue
		}
		if rc != 0 {
			return nil, 0, lastErr(e.h)
		}
		break
	}
	changes = make([]Change, int(n))
	for i := range changes {
		c := &buf[i]
		changes[i] = Change{Tick: uint64(c.tick), Term: uint64(c.term), TermStart: uint64(c.term_start), Group: uint32(c.group),
			Vote: uint8(c.vote), Role: uint8(c.role), Lead: uint8(c.lead), What: uint8(c.what)}
	}
	return changes, uint64(l), nil
}

// GroupState holds rows of listed groups: [n] per column, [R*n] replica-major for Match and Votes (element r*n+k
// belongs to groups[k]).  A nil column is skipped.
type GroupState struct {
	Term, Vote, Committed, LastIndex, LastTerm, TermStart, Match []uint64
	Role, Lead, SelfID, Votes                                    []uint8
	ElectionElapsed, HeartbeatElapsed, RandomizedTimeout         []uint16
}

// cState lays the non-nil columns of s out in C memory (cgo: a struct handed to C must not hold Go pointers) and
// returns the mrq_state over them, a copy-back for exports, and the free.
func (s *GroupState) cState(copyIn bool) (st C.mrq_state, copyBack func(), free func()) {
	var bufs []unsafe.Pointer
	var backs []func()
	col := func(p unsafe.Pointer, n int, size uintptr) unsafe.Pointer {
		if n == 0 {
			return nil
		}
		c := C.malloc(C.size_t(uintptr(n) * size))
		bufs = append(bufs, c)
		dst, src := unsafe.Slice((*byte)(c), uintptr(n)*size), unsafe.Slice((*byte)(p), uintptr(n)*size)
		if copyIn {
			copy(dst, src)
		}
		backs = append(backs, func() { copy(src, dst) })
		return c
	}
	u64 := func(v []uint64) *C.uint64_t {
		if len(v) == 0 {
			return nil
		}
		return (*C.uint64_t)(col(unsafe.Pointer(&v[0]), len(v), 8))
	}
	u8 := func(v []uint8) *C.uint8_t {
		if len(v) == 0 {
			return nil
		}
		return (*C.uint8_t)(col(unsafe.Pointer(&v[0]), len(v), 1))
	}
	u16 := func(v []uint16) *C.uint16_t {
		if len(v) == 0 {
			return nil
		}
		return (*C.uint16_t)(col(unsafe.Pointer(&v[0]), len(v), 2))
	}
	st.term, st.vote, st.committed, st.last_index = u64(s.Term), u64(s.Vote), u64(s.Committed), u64(s.LastIndex)
	st.last_term, st.term_start, st.match = u64(s.LastTerm), u64(s.TermStart), u64(s.Match)
	st.role, st.lead, st.self_id, st.votes = u8(s.Role), u8(s.Lead), u8(s.SelfID), u8(s.Votes)
	st.election_elapsed, st.heartbeat_elapsed, st.randomized_timeout = u16(s.ElectionElapsed), u16(s.HeartbeatElapsed), u16(s.RandomizedTimeout)
	copyBack = func() {
		for _, b := range backs {
			b()
		}
	}
	free = func() {
		for _, b := range bufs {
			C.free(b)
		}
	}
	return
}

// ExportGroups reads the rows of the listed local groups (duplicates allowed) into the non-nil columns of out, each
// sized for len(groups) rows: row k is exactly column groups[k] of a whole-engine export.  It writes no engine state
// and converts no representation, so it costs what n groups cost — e.g. the groups whose commit advance saturated at
// 255, or a status lookup.
func (e *Engine) ExportGroups(groups []uint64, out *GroupState) error {
	if len(groups) == 0 {
		return nil
	}
	st, copyBack, free := out.cState(false)
	defer free()
	if rc := C.mrq_export_groups(e.h, (*C.uint64_t)(unsafe.Pointer(&groups[0])), C.uint64_t(len(groups)), &st); rc != 0 {
		return lastErr(e.h)
	}
	copyBack()
	return nil
}

// ImportGroups overwrites the non-nil columns of the listed local groups (no duplicates) — e.g. one group replayed
// from its WAL — leaving every other group, and its compact state in tick mode 4, untouched.
func (e *Engine) ImportGroups(groups []uint64, in *GroupState) error {
	if len(groups) == 0 {
		return nil
	}
	st, _, free := in.cState(true)
	defer free()
	if rc := C.mrq_import_groups(e.h, (*C.uint64_t)(unsafe.Pointer(&groups[0])), C.uint64_t(len(groups)), &st); rc != 0 {
		return lastErr(e.h)
	}
	return nil
}
