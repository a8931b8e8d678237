/*
 * mrq.h — C-ABI of the Hopper-native multi-raft quorum engine ("mrq").
 *
 * This is the drop-in boundary for the hot path of chzchzchz/raftsql: everything the
 * reference reaches through github.com/coreos/etcd/raft's Node interface
 * (reference raft.go:152-165 construct, :214 Propose, :224 Tick, :227 Ready, :235 Advance,
 * :269 Step) — but for G independent raft groups at once, on one H100 (or one shard of G
 * on each of N H100s).  One engine == this node's replica of every group, exactly as one
 * reference process == this node's replica of one group (reference raft.go:62-78).
 *
 * Rules of the boundary (cgo / ctypes friendly):
 *   - plain C: opaque handle, POD structs, pointers + sizes; no C++/torch types;
 *   - every call returns 0 on success, <0 (MRQ_E_*) on error; mrq_last_error() gives text;
 *     the library never aborts or exits (contrast the reference's log.Fatalf sites,
 *     reference raft.go:102,107,114,126,251,256,263);
 *   - the caller owns every host buffer it passes; the engine copies before returning
 *     unless the call is documented as asynchronous-with-pinned-buffers;
 *   - one engine is driven by ONE thread at a time (mirrors the single select-loop goroutine,
 *     reference raft.go:221-245); distinct engines are independent;
 *   - no callbacks from C into the host.
 *
 * Identifiers: replica ids are 1..R (reference raft.go:150 `raft.Peer{ID: uint64(i + 1)}`),
 * 0 is etcd-raft's `None`.  All terms / indices are uint64 (raftpb).
 */
#ifndef MRQ_H
#define MRQ_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MRQ_ABI_VERSION 1u
#define MRQ_MAX_REPLICAS 8u /* ids and the vote record are packed 4+2 bits per replica */

/* ---- error codes ------------------------------------------------------------------- */
#define MRQ_OK 0
#define MRQ_E_INVAL (-1)   /* bad argument                                  */
#define MRQ_E_CUDA (-2)    /* CUDA runtime error (text in mrq_last_error)   */
#define MRQ_E_NOMEM (-3)   /* host or device allocation failed              */
#define MRQ_E_STATE (-4)   /* call not valid in this state                  */
#define MRQ_E_NCCL (-5)    /* NCCL not loadable / NCCL call failed          */
#define MRQ_E_NODEVICE (-6)/* no usable CUDA device: there is NO CPU fallback */

/* ---- roles (etcd-raft StateType order) -------------------------------------------------- */
#define MRQ_ROLE_FOLLOWER 0u
#define MRQ_ROLE_CANDIDATE 1u
#define MRQ_ROLE_LEADER 2u

/* ---- message types: etcd-raft raftpb.MessageType numbering of the v2.2/v2.3 era ------- */
#define MRQ_MSG_NONE 0u          /* empty inbox slot (MsgHup is local-only upstream)       */
#define MRQ_MSG_APP 3u           /* MsgApp, host-resolved: see mrq_inbox                   */
#define MRQ_MSG_APP_RESP 4u      /* MsgAppResp                                              */
#define MRQ_MSG_VOTE 5u          /* MsgVote                                                 */
#define MRQ_MSG_VOTE_RESP 6u     /* MsgVoteResp                                             */
#define MRQ_MSG_HEARTBEAT 8u     /* MsgHeartbeat                                            */
#define MRQ_MSG_HEARTBEAT_RESP 9u/* MsgHeartbeatResp                                        */
#define MRQ_MSG_TYPE_MASK 0x0Fu
#define MRQ_MSG_REJECT 0x80u     /* raftpb.Message.Reject, OR-ed into the type byte        */

/* ---- per-group output word (the engine's stand-in for Ready.Messages, raft.go:227-230) -- */
#define MRQ_OUT_CAMPAIGN 0x01u      /* campaign(): send MsgVote{Index:lastIndex,LogTerm:lastTerm} to all peers */
#define MRQ_OUT_BECAME_LEADER 0x02u /* becomeLeader(): an empty entry was appended at term_start               */
#define MRQ_OUT_BCAST_APPEND 0x04u  /* bcastAppend(): new entries and/or a new commit index to replicate       */
#define MRQ_OUT_BCAST_HEARTBEAT 0x08u /* MsgBeat fired: bcastHeartbeat()                                       */
#define MRQ_OUT_STEPPED_DOWN 0x10u  /* leader/candidate -> follower this tick                                  */
#define MRQ_OUT_PROP_DROPPED 0x20u  /* proposals dropped (candidate, or follower without a leader)             */
#define MRQ_OUT_PROP_FORWARD 0x40u  /* proposals to be forwarded to `lead` (follower with a leader)            */
#define MRQ_OUT_COMMIT_ADVANCED 0x80u /* committed[g] moved this tick                                          */
#define MRQ_OUT_VOTE_REPLY_SHIFT 8u /* bits 8..23: 2 bits per sender slot r: 0 none, 1 MsgVoteResp grant, 2 reject */
#define MRQ_OUT_ACK_REPLY_SHIFT 24u /* bits 24..31: 1 bit per sender slot r: reply MsgAppResp/MsgHeartbeatResp */

/* ---- configuration ------------------------------------------------------------------- */
typedef struct mrq_config {
  uint32_t abi_version;    /* MRQ_ABI_VERSION                                                     */
  uint32_t n_replicas;     /* R = len(peers), 1..MRQ_MAX_REPLICAS (reference raft.go:148)         */
  uint64_t n_groups;       /* G: raft groups owned by THIS engine (the shard, not the job total)  */
  uint64_t group_base;     /* global id of local group 0 (shard offset; keys the RNG / traces)    */
  uint32_t election_tick;  /* raft.Config.ElectionTick, reference raft.go:154 (10); 1..2047       */
  uint32_t heartbeat_tick; /* raft.Config.HeartbeatTick, reference raft.go:155 (1); 1..255        */
  uint64_t seed;           /* keys the randomized election timeout draw                           */
  uint32_t self_id;        /* raft.Config.ID, reference raft.go:153: 1..R for every group, or 0 = */
                           /* rotate: self id of global group g is (g % R) + 1                    */
  int32_t device;          /* CUDA device ordinal                                                 */
  void *stream;            /* optional cudaStream_t to run on (NULL: the engine creates one)      */
  uint32_t inbox_slots;    /* number of device inbox buffers to rotate through (>=1; default 2)   */
  uint32_t flags;          /* reserved, 0                                                         */
} mrq_config;

/* Fill a config with the reference's defaults (ElectionTick 10, HeartbeatTick 1; raft.go:154-155). */
void mrq_config_default(mrq_config *cfg);

typedef struct mrq_engine mrq_engine;

/* StartNode for G groups: every group a follower at term 0 with an empty log, like
 * raft.StartNode on a fresh MemoryStorage (reference raft.go:161-165) minus the conf-change
 * bootstrap entries (membership is the static peer list, reference raft.go:148-151). */
int mrq_create(const mrq_config *cfg, mrq_engine **out);
void mrq_destroy(mrq_engine *e);
/* Text of the last error on this engine (or of the last failed mrq_create when e == NULL). */
const char *mrq_last_error(const mrq_engine *e);

/* ---- state import / export (HardState + volatile state, SoA host arrays) -------------- */
/* All arrays have n_groups elements unless noted; a NULL pointer skips that column.
 * match / votes are replica-major: element [r * n_groups + g].  */
typedef struct mrq_state {
  uint64_t *term;        /* HardState.Term                                                     */
  uint64_t *vote;        /* HardState.Vote (0 = None)                                           */
  uint64_t *committed;   /* HardState.Commit                                                    */
  uint64_t *last_index;  /* raftLog.lastIndex()                                                 */
  uint64_t *last_term;   /* raftLog.lastTerm()                                                  */
  uint64_t *term_start;  /* index of the empty entry appended by becomeLeader (valid if leader; */
                         /* UINT64_MAX otherwise: the commit gate can never pass)               */
  uint64_t *match;       /* [R][G] Progress.Match (meaningful for leaders)                     */
  uint8_t *role;         /* MRQ_ROLE_*                                                          */
  uint8_t *lead;         /* raft.lead (0 = None)                                                */
  uint8_t *self_id;      /* this node's id in the group (1..R)                                  */
  uint8_t *votes;        /* [R][G] poll() record: 0 absent, 1 granted, 2 rejected               */
  uint16_t *election_elapsed;
  uint16_t *heartbeat_elapsed;
  uint16_t *randomized_timeout; /* in [ElectionTick, 2*ElectionTick-1]                          */
} mrq_state;

int mrq_export_state(mrq_engine *e, mrq_state *out); /* blocking: device -> caller arrays      */
int mrq_import_state(mrq_engine *e, const mrq_state *in); /* blocking: caller arrays -> device */
/* The same for a list of local groups, at a cost that follows n, not G (one kernel launch plus the copies).
 * `out` / `in` are mrq_state with n-row arrays: [n], and [R][n] for match / votes (element [r * n + k] belongs to
 * groups[k]); a NULL pointer skips that column.  n == 0: no-op.  groups == NULL with n > 0: MRQ_E_INVAL.  G == 0: OK.
 * Neither call records change-feed entries (as mrq_import_state: the feed does not record the host's own changes),
 * moves the mrq_sync_commit_deltas drain base (only mrq_sync_commits rebases it), or invalidates captured CUDA graphs
 * or mode-4 descriptor tables (only device memory contents change).
 *
 * mrq_export_groups: blocking.  Row k is exactly row groups[k] of what mrq_export_state would return at that point.
 * Duplicates are allowed.  Writes no engine state and converts no representation (tick mode 4's compact groups are
 * decoded in the kernel); a group >= G: MRQ_E_INVAL.
 * mrq_import_groups: blocking.  Overwrites the given columns of the listed groups, with the same effect on them as
 * "export everything, overwrite those rows, import everything" — on every later export, out word, commit advance,
 * change-feed record and counter except kernel_launches.  The other groups' state, including their compact
 * representation in tick mode 4, is untouched (unlike mrq_import_state, whose whole-engine conversion makes the next
 * mode-4 tick re-compact every group).  A duplicate or a group >= G: MRQ_E_INVAL, nothing changed.  With the fused
 * gather on (mrq_comm_set_mode(1)) an import of `committed` makes the next tick republish every full index.  */
int mrq_export_groups(mrq_engine *e, const uint64_t *groups, uint64_t n, mrq_state *out);
int mrq_import_groups(mrq_engine *e, const uint64_t *groups, uint64_t n, const mrq_state *in);
/* Progress.Next is message-construction state; without rejections it is exactly
 * max(term_start, match+1) (reset() sets Next = lastIndex+1 == term_start; maybeUpdate raises it
 * to n+1).  Exported as a convenience for the host's sendAppend.  out is [R][G].              */
int mrq_export_next(mrq_engine *e, uint64_t *next_out);
uint64_t mrq_tick_count(const mrq_engine *e);
int mrq_set_tick_count(mrq_engine *e, uint64_t t);

/* ---- the inbox: what node.Step(m) receives (reference raft.go:268-270) ---------------- */
/* Dense form: one slot per (sender replica r, group g) per tick, replica-major [r*G + g].
 * Field meaning per type (raftpb.Message fields):
 *   MSG_VOTE        term, index = candidate lastIndex, logterm = candidate lastTerm
 *   MSG_VOTE_RESP   term, REJECT bit
 *   MSG_APP_RESP    term, index = follower's acknowledged index, REJECT bit
 *   MSG_HEARTBEAT   term, commit
 *   MSG_HEARTBEAT_RESP term
 *   MSG_APP         term; HOST-RESOLVED: the host keeps the log, ran maybeAppend, and reports the
 *                   outcome: index/logterm = the log's (lastIndex,lastTerm) after the append,
 *                   commit = min(m.Commit, lastnewi).  With REJECT the log did not match: only
 *                   the term rule, electionElapsed=0 and lead=From apply.  What is reported must be a
 *                   log: logterm = 0 exactly when index = 0, and logterm <= term (no entry is newer
 *                   than the leader that sent it) — the engine keeps no per-entry terms and relies on
 *                   a new leader's own entries being the only ones of its term.
 * Slots are Step()ped in sender order r = 0..R-1, then proposals, then the tick — the
 * canonical per-tick serialisation (DESIGN.md §3).                                           */
typedef struct mrq_inbox {
  const uint8_t *type;     /* [R][G] MRQ_MSG_* | MRQ_MSG_REJECT                                */
  const uint64_t *term;    /* [R][G]                                                           */
  const uint64_t *index;   /* [R][G]                                                           */
  const uint64_t *logterm; /* [R][G]                                                           */
  const uint64_t *commit;  /* [R][G]                                                           */
  const uint32_t *prop_count; /* [G] entries proposed at this node this tick (raft.go:214); may be NULL */
} mrq_inbox;

/* Copy a dense inbox from host memory into inbox slot `slot` (async on the engine stream when the
 * source is pinned; the engine otherwise stages through its own pinned buffer).  NULL columns are
 * treated as all-zero.                                                                         */
int mrq_post_inbox_dense(mrq_engine *e, uint32_t slot, const mrq_inbox *in);

/* Sparse form: a list of messages, scattered into inbox slot `slot` on the device.  The slot is
 * cleared first unless `accumulate` is non-zero.  If several messages hit the same (from, group)
 * slot the last one in the list wins.                                                          */
typedef struct mrq_msg {
  uint64_t group; /* local group index 0..G-1 */
  uint64_t term;
  uint64_t index;
  uint64_t logterm;
  uint64_t commit;
  uint8_t type; /* MRQ_MSG_* | MRQ_MSG_REJECT */
  uint8_t from; /* sender id 1..R */
  uint8_t pad[6];
} mrq_msg;
int mrq_post_inbox_delta(mrq_engine *e, uint32_t slot, const mrq_msg *msgs, size_t n, int accumulate);

/* Packed dense form for the PCIe-bound host path: one 32-bit word per (sender, group) slot, decoded
 * on the device against two per-group BASE columns the host sets with mrq_set_packed_base (so the
 * decode never depends on engine state the host may be a few ticks behind on).  Exact; anything that
 * does not fit rides in the `wide` escape list:
 *   bits  0..3   type        bit 4 REJECT
 *   bits  5..6   term code c: term = base_term[g] + c for c in 0..2; c == 3 => escaped to `wide`
 *   bits  7..31  payload p (25 bits), by type:
 *        MSG_APP_RESP      index  = base_index[g] + p
 *        MSG_HEARTBEAT     commit = base_index[g] + p
 *        MSG_VOTE          logterm = base_term[g] + (p & 3), index = base_index[g] + (p >> 2)
 *        MSG_VOTE_RESP / MSG_HEARTBEAT_RESP   p unused
 *        MSG_APP           always escaped (needs three 64-bit fields)
 * Escaped / wide messages ride in `wide` (n_wide entries) and override their slot.
 *
 * 16-bit form (word_bits = 16; `word` then points at uint16_t[R][G]): bits 0..2 kind (0 none, 1 ack,
 * 2 ack|REJECT, 3 vote-resp grant, 4 vote-resp REJECT, 5 heartbeat, 6 heartbeat-resp, 7 escaped),
 * bits 3..4 term code as above, bits 5..15 payload p (ack index / heartbeat commit = base_index[g] + p).
 * MSG_VOTE and MSG_APP always escape.
 *
 * Byte form (word_bits = 8; `word` then points at uint8_t[R-1][G]): one byte per REMOTE sender — the row of
 * each group's own replica slot is left out — with a 64-entry index window that slides by a rule both sides
 * apply to the bytes alone (the device advances base_index itself).  Codec, row mapping and the window rule:
 * include/mrq_packed8.h; build frames with mrq_pack8 below.
 *
 * ASYNCHRONOUS: the copies run on the engine's copy stream so that the next tick's H2D overlaps the
 * current tick; `word`, `prop_count8` and `wide` should be page-locked (mrq_alloc_pinned) and must stay
 * valid and unmodified until a blocking call (mrq_sync_* / mrq_synchronize) made after the mrq_tick
 * that consumes the slot has returned.                                                         */
typedef struct mrq_inbox_packed {
  const void *word;           /* [R][G] uint32_t (word_bits 32 or 0) / uint16_t (16), or [R-1][G] uint8_t (8) */
  const uint8_t *prop_count8; /* [G] proposals (0..255) or NULL */
  const mrq_msg *wide;        /* escape list */
  size_t n_wide;
  uint32_t word_bits;         /* 0 or 32: 32-bit words; 16: 16-bit words; 8: the byte form */
  uint32_t reserved;          /* flags: MRQ_PACKED_KEEP, else 0 */
} mrq_inbox_packed;
/* tick mode 3 only: the byte frame stays in its slot after the tick that read it, so a sequence of slots can be
 * replayed (after restoring the state and the packed base) without posting again.                          */
#define MRQ_PACKED_KEEP 1u
int mrq_post_inbox_packed(mrq_engine *e, uint32_t slot, const mrq_inbox_packed *in);
/* Dense [G] decode bases for the packed form (NULL keeps the current column).  Blocking. */
int mrq_set_packed_base(mrq_engine *e, const uint64_t *base_index, const uint64_t *base_term);

/* Host-side frame builder for the byte form — the batched stand-in for rafthttp handing messages to
 * node.Step one at a time (reference raft.go:268-270): PURE CPU CODE (no engine, no device; usable from any thread).
 * Encodes the wide dense inbox `in` ([R][G] columns; prop_count may be NULL) of groups whose own ids are
 * self_id[G] (1..R) into word_out[R-1][G] (+ prop8_out[G] if not NULL), appends what does not fit to wide_out
 * (at most wide_cap entries; *n_wide = how many were needed) and slides base_index[G] exactly as the device
 * will when it decodes the frame — call it once per frame, in posting order, on the host's copy of the base
 * that was last given to mrq_set_packed_base.  MRQ_E_INVAL: bad arguments, more than 255 proposals for a
 * group, or wide_cap too small — base_index is then unchanged (the output buffers hold a discarded frame):
 * retry with room for *n_wide entries.  Large frames are built on several host threads (MRQ_HOST_THREADS).  */
int mrq_pack8(const mrq_inbox *in, const uint8_t *self_id, uint64_t n_groups, uint32_t n_replicas, uint64_t *base_index,
              const uint64_t *base_term, uint8_t *word_out, uint8_t *prop8_out, mrq_msg *wide_out, size_t wide_cap,
              size_t *n_wide);
/* The decode the device performs, on the host (same inline codec): word[R-1][G] -> the wide dense columns of
 * `out` ([R][G]; escaped and empty slots get type 0; only the columns Step() reads for a type are written,
 * the others are left as they were) and the slid base_index.  For tests and for debugging a frame builder. */
struct mrq_inbox_out;
int mrq_unpack8(const uint8_t *word, const uint8_t *self_id, uint64_t n_groups, uint32_t n_replicas, uint64_t *base_index,
                const uint64_t *base_term, const struct mrq_inbox_out *out);

/* Proposals only (node.Propose, reference raft.go:211-215): sparse (group, count) pairs added to
 * inbox slot `slot`'s prop_count.                                                             */
int mrq_propose(mrq_engine *e, uint32_t slot, const uint64_t *groups, const uint32_t *counts, size_t n);

/* Zero inbox slot `slot` on the device (async). */
int mrq_clear_inbox(mrq_engine *e, uint32_t slot);

/* ---- the hot path ------------------------------------------------------------------- */
/* One raft tick for every group: Step() every message of inbox slot `slot` in canonical order,
 * apply proposals, then Tick() (election / heartbeat timers, campaign).  Asynchronous on the
 * engine stream.  The fused sm_90a kernel covers SURVEY §8a rows a3–a16.  If a communicator is
 * attached (mrq_comm_init), the tick also all-gathers committed[] across ranks.               */
int mrq_tick(mrq_engine *e, uint32_t slot);
/* n ticks in one call, tick k consuming inbox slot slots[k].  The launch sequence for a slot list is
 * captured into a CUDA graph on first use and replayed afterwards (launch-bound regimes: small shards,
 * many GPUs).  Same results as n mrq_tick calls.                                               */
int mrq_tick_many(mrq_engine *e, const uint32_t *slots, uint32_t n);
/* Whether mrq_tick_many replays CUDA graphs: 0 never (plain launches), 1 always, 2 (default) only when
 * the engine holds few enough groups that the host launch rate, not the kernels, bounds the tick rate. */
int mrq_set_graph_mode(mrq_engine *e, int mode);
/* L2 residency hints of the tick kernel (default on): inbox columns are loaded evict-first, state columns
 * loaded / stored evict-last, so that a shard whose state fits the 50 MB L2 keeps it on-chip from tick to
 * tick and HBM carries (mostly) the inbox.  Results are unaffected; 0 turns the hints off.       */
int mrq_set_l2_policy(mrq_engine *e, int on);
/* n ticks with an empty inbox (timers only). */
int mrq_tick_idle(mrq_engine *e, uint32_t n);
/* How mrq_tick is launched: 0 = a lean fast kernel for the ticks that need no role machinery
 * (steady-state leaders, quiet / heart-beaten followers) + a general kernel over the compacted list of
 * the remaining groups (two launches); 2 = one launch doing both (each CTA compacts its stragglers in
 * shared memory and runs the general path on them); 1 = one general kernel over every group
 * (differential testing); 3 = mode 0 on the BYTE FORM of the inbox: a slot posted with word_bits = 8 is not
 * unpacked — the fast kernel reads the frame's bytes where the copy left them and the general kernel
 * materialises only the groups the fast one declines (a slot posted in any other form ticks as in mode 0;
 * no graph replay in this mode); 4 = the byte form on COMPACT STATE: every index-like column of a group
 * (lastIndex, committed, Progress.Match, the frame window) is held as a 32-bit offset from one per-group
 * 64-bit base, one thread owns four adjacent groups (128-bit column accesses), and the steady-state tick
 * moves ~82 B per group instead of 217; a group whose values do not fit, or whose tick needs the role
 * machinery, goes through the general path on the wide columns and is re-compacted; every call that
 * reads or writes wide state (import / export / sync / gen_trace / quorum / a wide post) converts first.
 * In mode 4 mrq_tick_many runs its whole slot sequence in ONE pair of launches (each thread carries its
 * groups' state in registers from tick to tick; per-tick out words and commit advances go to per-slot
 * buffers).  All modes give identical results.                                                   */
int mrq_set_tick_mode(mrq_engine *e, int mode);
/* mrq_tick_many in mode 4: 1 (default) = the state columns are written back after every tick of the
 * sequence (device state is exact at tick granularity), 0 = after the last tick only.           */
int mrq_set_write_through(mrq_engine *e, int on);

/* The standalone quorum kernel (K3; SURVEY §8a rows a15–a16): for every leader group,
 * mci = q-th largest of match[0..R-1][g]; committed = mci iff mci > committed && mci >= term_start.
 * Reads 8R+16 bytes per group, writes 8 when the commit index moves.  Asynchronous.           */
int mrq_quorum_commit(mrq_engine *e);

/* Which implementation mrq_quorum_commit uses: 0 = quad form, four groups per thread, two
 * 128-bit loads per column, 1 = TMA bulk-copy form (replica columns staged through shared memory with
 * cp.async.bulk + mbarrier; default, the fastest on H100), 2 = 128-bit LDG form, two groups per thread. */
int mrq_set_quorum_variant(mrq_engine *e, int variant);
/* The same kernel over caller-owned DEVICE columns (zero-copy integration; also what bench.py
 * rotates through so every timed launch reads cold HBM): d_match is [R][stride] replica-major,
 * d_committed / d_term_start are [n_groups]; stride must be a multiple of 4 and >= n_groups and
 * the columns 16-byte aligned.  Asynchronous on the engine stream.                             */
int mrq_quorum_commit_ext(mrq_engine *e, const uint64_t *d_match, uint64_t *d_committed, const uint64_t *d_term_start,
                          uint64_t n_groups, uint64_t stride, int variant);

/* Element-wise Progress.maybeUpdate on the device for a sparse list of acks (a14), without a tick:
 * match[from-1][group] = max(match, index).                                                    */
int mrq_match_update(mrq_engine *e, const uint64_t *groups, const uint8_t *from, const uint64_t *index, size_t n);

/* ---- outputs: the Ready() drain (reference raft.go:227-235) -------------------------- */
/* Blocking: waits for the stream, copies device -> caller.  NULL pointers are skipped.        */
int mrq_sync_commits(mrq_engine *e, uint64_t *committed_out, uint8_t *role_out, uint64_t *term_out);
/* Per-group output word of the last tick (MRQ_OUT_*). */
int mrq_sync_out(mrq_engine *e, uint32_t *out_words);
/* Compact commit drain for the host path: per-group advance of committed since the previous
 * drain, saturated to 255 in a byte.  255 means "read the full value": mrq_sync_commits with a
 * non-NULL committed_out rebases every group's drain to the values it returns.                 */
int mrq_sync_commit_deltas(mrq_engine *e, uint8_t *delta_out);
/* The same drain, split for pipelining hosts: mrq_drain_commit_deltas enqueues it (the destination must
 * be page-locked) and returns; mrq_drain_wait blocks until THAT drain has landed — not until the stream
 * is idle, so an mrq_post_inbox_packed issued in between keeps copying underneath.             */
int mrq_drain_commit_deltas(mrq_engine *e, uint8_t *delta_out_pinned);
int mrq_drain_wait(mrq_engine *e);
/* Mode 4 only: the tick kernels themselves write each group's commit advance of THAT tick (one byte,
 * 255 = "read the index in full") next to its out word, so draining the last tick is a plain
 * asynchronous copy (page-locked destination; mrq_drain_wait waits for it) — no extra kernel.
 * MRQ_E_STATE when the last tick was not a mode-4 tick on a byte frame.                           */
int mrq_drain_tick_deltas(mrq_engine *e, uint8_t *delta_out_pinned);
/* Mode 4, after mrq_tick_many: the out words and commit advances of the tick that consumed inbox slot `slot`
 * (every tick of the sequence writes to its slot's own buffers).  Blocking; a NULL pointer skips that column. */
int mrq_sync_slot_outputs(mrq_engine *e, uint32_t slot, uint32_t *out_words, uint8_t *delta_out);
int mrq_synchronize(mrq_engine *e);

/* ---- change feed: the groups whose HardState {Term, Vote} or SoftState {Lead, RaftState} moved (raft.go:227-235) ----
 * Recorded by the tick kernels themselves in every tick mode and every way of ticking (mrq_tick, mrq_tick_many,
 * mrq_tick_idle).  Commit advances are not recorded (they have their own drains); neither are changes the host makes
 * itself (mrq_import_state, mrq_set_tick_count).  Draining converts no state representation.                      */
#define MRQ_CHANGE_TERM 0x01u /* HardState.Term moved            */
#define MRQ_CHANGE_VOTE 0x02u /* HardState.Vote moved            */
#define MRQ_CHANGE_ROLE 0x04u /* SoftState.RaftState moved       */
#define MRQ_CHANGE_LEAD 0x08u /* SoftState.Lead moved            */
typedef struct mrq_change {   /* 32 bytes                        */
  uint64_t tick;              /* number of the tick that made the change (mrq_tick_count() before it) */
  uint64_t term;              /* after the tick                   */
  uint64_t term_start;        /* after the tick; UINT64_MAX unless leader (a new leader's empty entry) */
  uint32_t group;             /* local group index                */
  uint8_t vote, role, lead, what; /* after the tick; what = MRQ_CHANGE_* bits, never 0 */
} mrq_change;
/* 0 (default) = off.  Otherwise record up to max_records changes between drains.  Blocking; discards pending records. */
int mrq_set_change_capacity(mrq_engine *e, uint64_t max_records);
/* Blocking.  Every record since the previous drain, sorted by (tick, group), then reset.  Exactly one record per
 * (tick, group) whose term, vote, role or lead differs after that tick from before it.  *lost = records that did
 * not fit the capacity: the list is then incomplete (each returned record is still genuine) and the host must
 * read state in full.  cap < records pending: MRQ_E_INVAL, nothing consumed, *n_out = entries needed.
 * Feed off: MRQ_E_STATE. */
int mrq_sync_changes(mrq_engine *e, mrq_change *out, uint64_t cap, uint64_t *n_out, uint64_t *lost);

/* ---- synthetic vote/append traces, generated on the device (include/mrq_trace.h) -------- */
struct mrq_trace_params;
int mrq_gen_trace(mrq_engine *e, uint32_t slot, const struct mrq_trace_params *p, uint64_t tick);
/* Read an inbox slot back to host arrays (testing / oracle feeding). Non-const view required. */
typedef struct mrq_inbox_out {
  uint8_t *type;
  uint64_t *term, *index, *logterm, *commit;
  uint32_t *prop_count;
} mrq_inbox_out;
int mrq_read_inbox(mrq_engine *e, uint32_t slot, mrq_inbox_out *out);

/* ---- counters --------------------------------------------------------------------- */
typedef struct mrq_counters {
  uint64_t ticks;
  uint64_t kernel_launches;   /* kernels this library launched since create */
  uint64_t campaigns;         /* a10 */
  uint64_t elections_won;     /* a9  */
  uint64_t step_downs;        /* a12 */
  uint64_t commits_advanced;  /* a16: groups whose commit index moved */
  uint64_t votes_granted;     /* a13 */
  uint64_t errors;            /* invariant violations seen on device (e.g. commit > lastIndex) */
} mrq_counters;
int mrq_get_counters(mrq_engine *e, mrq_counters *out); /* blocking */

/* ---- timing on the engine stream (CUDA events) --------------------------------------- */
int mrq_timer_start(mrq_engine *e);
int mrq_timer_stop(mrq_engine *e, float *elapsed_ms); /* blocking */

/* ---- multi-GPU: groups shard across ranks; one all-gather of committed[] per tick -------- */
#define MRQ_COMM_ID_BYTES 128
/* NCCL is dlopen()ed on first use (libnccl.so.2); single-GPU use never needs it. */
int mrq_comm_unique_id(uint8_t id_out[MRQ_COMM_ID_BYTES]);
/* Attach this engine (rank `rank` of `world`) to a communicator.  Every rank must own the same
 * n_groups.  After this, mrq_tick() ends with ncclAllGather(committed[G]) -> gathered[world*G]. */
int mrq_comm_init(mrq_engine *e, const uint8_t id[MRQ_COMM_ID_BYTES], uint32_t rank, uint32_t world);
/* mode 0: ncclAllGather of uint64 committed[] (default); mode 1: peer-store gather fused into the
 * tick kernels over CUDA-IPC mapped peer buffers (requires mrq_ipc_attach): every tick each group's
 * commit index goes straight into every rank's buffer over NVLink — its low byte every tick, the
 * full 64-bit value only when anything above the low byte changed (or right after this call /
 * mrq_ipc_attach, which re-publish everything).  mrq_sync_gathered returns the stitched indices
 * in either mode.                                                                                */
int mrq_comm_set_mode(mrq_engine *e, uint32_t mode);
int mrq_sync_gathered(mrq_engine *e, uint64_t *gathered_out); /* blocking; world*G elements     */
/* CUDA-IPC plumbing for the fused peer-store gather: export this rank's gather buffer, then attach
 * every rank's handle (handles is world * MRQ_IPC_HANDLE_BYTES, in rank order).                  */
#define MRQ_IPC_HANDLE_BYTES 64
/* Size the gather buffer for `world` ranks (call before mrq_ipc_export when NCCL is not used). */
int mrq_ipc_prepare(mrq_engine *e, uint32_t world);
int mrq_ipc_export(mrq_engine *e, uint8_t handle_out[MRQ_IPC_HANDLE_BYTES]);
int mrq_ipc_attach(mrq_engine *e, const uint8_t *handles, uint32_t rank, uint32_t world);

/* ---- raw device pointers (zero-copy integration with a host that already lives on the GPU;
 * also lets tests / torch wrap the buffers).  `which` is an MRQ_PTR_* id.
 * In tick mode 4 some raw columns are exact only in the wide representation, i.e. right after a call
 * that converts (an export, mrq_sync_commits, ...): COMMITTED, LAST_INDEX and MATCH (kept as offsets
 * from a per-group base), and META's electionElapsed / heartbeatElapsed fields of a leader (kept as
 * phases against the tick number).                                                              */
#define MRQ_PTR_TERM 0
#define MRQ_PTR_META 1
#define MRQ_PTR_LAST_INDEX 2
#define MRQ_PTR_LAST_TERM 3
#define MRQ_PTR_COMMITTED 4
#define MRQ_PTR_TERM_START 5
#define MRQ_PTR_MATCH 6
#define MRQ_PTR_OUT 7
#define MRQ_PTR_GATHERED 8
void *mrq_device_ptr(mrq_engine *e, int which);
void *mrq_stream(mrq_engine *e);
/* Element stride between replica rows of the device's replica-major arrays (G rounded up to 128). */
uint64_t mrq_group_stride(const mrq_engine *e);
/* Page-locked host memory for asynchronous posts / drains (cudaHostAlloc / cudaFreeHost). */
void *mrq_alloc_pinned(size_t bytes);
void mrq_free_pinned(void *p);

/* Library/version probe: returns MRQ_ABI_VERSION; *sm_arch gets 90 (built for sm_90a). */
uint32_t mrq_version(uint32_t *sm_arch);

#ifdef __cplusplus
}
#endif
#endif /* MRQ_H */
