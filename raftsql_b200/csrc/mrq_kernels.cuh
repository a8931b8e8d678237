// mrq_kernels.cuh — sm_90a device code of the multi-raft quorum engine.
//
// One thread owns one raft group for one tick: the group's whole state lives in registers, the
// tick's messages are Step()ped in canonical order (sender ascending, proposals, timers), and only
// the columns that changed are written back.  All global accesses are column accesses with the
// group index fastest, so a warp reads/writes 256 contiguous bytes per u64 column.
//
// Restates (per group) what the reference reaches through etcd-raft's Node interface —
// reference raft.go:214 Propose, :224 Tick, :227 Ready, :235 Advance, :269 Step — i.e. SURVEY §8a
// rows a3–a16.  Integer only; tensor cores are not applicable.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/mrq.h"
#include "../../include/mrq_packed8.h"
#include "../../include/mrq_trace.h"

namespace mrq {

static constexpr uint64_t kNoGate = 0xFFFFFFFFFFFFFFFFull;  // term_start of a non-leader: gate never passes

// ---- packed per-group small state ("meta" column, one u64 per group) -----------------------
//  [0,2) role  [2,6) lead  [6,10) vote  [10,14) self id  [14,26) electionElapsed
//  [26,38) randomizedElectionTimeout  [38,46) heartbeatElapsed  [46,62) votes (2 bits x 8 slots)
//  [62] strict: some Progress.Match may exceed lastIndex (an out-of-range ack was seen this leadership)
//  [63] ltok:   the stored last_term equals term (always true for a leader after its first append) — lets
//               the steady-state path skip the last_term column entirely
struct Meta {
  uint32_t role, lead, vote, self, elapsed, rto, hb, votes, strict, ltok;
};
__host__ __device__ __forceinline__ uint64_t meta_pack(const Meta &m) {
  return (uint64_t)(m.role & 3u) | ((uint64_t)(m.lead & 15u) << 2) | ((uint64_t)(m.vote & 15u) << 6) |
         ((uint64_t)(m.self & 15u) << 10) | ((uint64_t)(m.elapsed & 0xFFFu) << 14) |
         ((uint64_t)(m.rto & 0xFFFu) << 26) | ((uint64_t)(m.hb & 0xFFu) << 38) |
         ((uint64_t)(m.votes & 0xFFFFu) << 46) | ((uint64_t)(m.strict & 1u) << 62) | ((uint64_t)(m.ltok & 1u) << 63);
}
__host__ __device__ __forceinline__ Meta meta_unpack(uint64_t w) {
  Meta m;
  m.role = (uint32_t)(w & 3u);
  m.lead = (uint32_t)((w >> 2) & 15u);
  m.vote = (uint32_t)((w >> 6) & 15u);
  m.self = (uint32_t)((w >> 10) & 15u);
  m.elapsed = (uint32_t)((w >> 14) & 0xFFFu);
  m.rto = (uint32_t)((w >> 26) & 0xFFFu);
  m.hb = (uint32_t)((w >> 38) & 0xFFu);
  m.votes = (uint32_t)((w >> 46) & 0xFFFFu);
  m.strict = (uint32_t)((w >> 62) & 1u);
  m.ltok = (uint32_t)((w >> 63) & 1u);
  return m;
}

// ---- device views -----------------------------------------------------------------------------
struct StateView {  // engine state, SoA; replica-major arrays use stride `gs` (padded G)
  uint64_t *term, *meta, *last_index, *last_term, *committed, *term_start, *match;
  uint32_t *out;
};
struct InboxView {  // one inbox slot, replica-major with stride `gs`
  uint8_t *type;
  uint64_t *term, *index, *logterm, *commit;
  uint32_t *prop;
};
// Device-side event counts.  Sharded: in steady state every group commits every tick, so one counter would
// take one same-address atomic per warp (tens of thousands per launch, serialised in one L2 slice).  CTAs
// spread over kCtrShards copies, each on its own 128-byte line; mrq_get_counters sums them.
static constexpr int kCtrShards = 64;
struct alignas(128) Counters {
  unsigned long long campaigns, elections_won, step_downs, commits_advanced, votes_granted, errors;
};
struct TickArgs {
  StateView s;
  InboxView in;  // in.type == nullptr: idle tick (timers only)
  Counters *ctr;
  uint64_t G, gs, group_base, seed;
  // The tick number lives in device memory so that a sequence of ticks can be replayed as a CUDA graph:
  // tick t reads tick_cur (written during tick t-1) and its first kernel writes tick_next = tick_cur + 1.
  const uint64_t *tick_cur;
  uint64_t *tick_next;
  uint32_t election_tick, heartbeat_tick;
  // Fused peer-store all-gather (multi-GPU mode 1): the commit index of every group this rank owns is stored
  // straight into every rank's gather buffer over NVLink.  NVLink bytes are what bounds a many-GPU job (N = 8:
  // 131,072 groups x 7 peers per GPU per tick), so the buffer is split: the LOW BYTE of every index is stored every
  // tick, the full 64-bit index only when anything above the low byte changed (every ~170 ticks per group at this
  // trace's commit rate) or when priming: ~1.05 B per group-tick per peer instead of 8.  mrq_sync_gathered stitches.
  uint8_t *peer_lo[8];
  uint64_t *peer_full[8];
  uint32_t world, rank, gather_prime;
  uint32_t l2_policy;  // 1: inbox evict-first / state evict-last hints in the fast kernel (see l2_policy())
  // fast/slow split: groups the fast kernel leaves untouched are listed here for the slow kernel
  uint32_t *slow_list;
  unsigned *slow_count, *slow_count_next;
  // Change feed (mrq_set_change_capacity): the general tick appends one record per group whose term, vote, role or
  // lead it moved.  change_count counts every record; only the first change_cap are written.  nullptr: feed off.
  mrq_change *changes;
  unsigned long long *change_count;
  uint64_t change_cap;
};

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------
// Every hot kernel lets the next launch in the stream start filling freed SMs while this grid's tail
// drains (launch_dependents), and touches global memory only after the previous grid has completed
// and flushed (wait).  No-ops when the launch did not ask for programmatic serialization.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// one group's commit index into every rank's gather buffer (see TickArgs)
template <class Args>
__device__ __forceinline__ void gather_store(const Args &a, const uint64_t i, const uint64_t committed, const uint64_t committed0) {
  const uint64_t at = (uint64_t)a.rank * a.G + i;
  const bool full = a.gather_prime || ((committed ^ committed0) >> 8) != 0;
#pragma unroll 1
  for (uint32_t p = 0; p < a.world; ++p) {
    a.peer_lo[p][at] = (uint8_t)committed;
    if (full) a.peer_full[p][at] = committed;
  }
}

// ---- cache-hinted accessors ---------------------------------------------------------------------
// (MRQ_HOST_EMULATION is defined only by tests/cpp/tick_host_test.cpp, which compiles the per-group tick
// functions of this header for the HOST and runs them over host arrays against the CPU checker; product
// builds never define it, so the block below is what they have always compiled.)
#ifndef MRQ_HOST_EMULATION
// Inbox columns are read exactly once per tick: stream them (read-only path, no L1 allocation).
__device__ __forceinline__ uint64_t ld_stream(const uint64_t *p) {
  uint64_t v;
  asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ uint32_t ld_stream_u8(const uint8_t *p) {
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.u8 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ uint32_t ld_stream_u32(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
// State columns are read and (sometimes) rewritten by the same thread: plain loads, no L1 allocation.
__device__ __forceinline__ uint64_t ld_state(const uint64_t *p) {
  uint64_t v;
  asm volatile("ld.global.L1::no_allocate.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_state(uint64_t *p, uint64_t v) {
  asm volatile("st.global.L1::no_allocate.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_state_u32(uint32_t *p, uint32_t v) {
  asm volatile("st.global.L1::no_allocate.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ---- L2 residency policy --------------------------------------------------------------------------------
// Every tick streams its inbox through L2 exactly once while the engine state is re-read every tick (the compact
// state of tick mode 4 is ~30 MB at the headline shape, next to H100's 50 MB L2).  Left alone the stream evicts the
// state and each tick re-reads it from HBM.  With cache-hinted accesses (createpolicy + .L2::cache_hint; the
// policy rides in the memory descriptor, no extra instructions) the inbox is marked evict-first and the state
// evict-last, so state columns stay on-chip from one tick to the next and HBM mostly carries the inbox.
__device__ __forceinline__ uint64_t l2_policy(uint32_t kind) {  // 0 normal, 1 evict-first, 2 evict-last
  uint64_t p;
  if (kind == 1u)
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  else if (kind == 2u)
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  else
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t ld_stream_p(const uint64_t *p, uint64_t pol) {
  uint64_t v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ uint32_t ld_stream_u8_p(const uint8_t *p, uint64_t pol) {
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ uint32_t ld_stream_u32_p(const uint32_t *p, uint64_t pol) {
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ uint64_t ld_state_p(const uint64_t *p, uint64_t pol) {
  uint64_t v;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void st_state_p(uint64_t *p, uint64_t v, uint64_t pol) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(p), "l"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_state_u32_p(uint32_t *p, uint32_t v, uint64_t pol) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.u32 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}
#else  // MRQ_HOST_EMULATION: the same accessors as plain memory operations
inline uint64_t ld_stream(const uint64_t *p) { return *p; }
inline uint32_t ld_stream_u8(const uint8_t *p) { return *p; }
inline uint32_t ld_stream_u32(const uint32_t *p) { return *p; }
inline uint64_t ld_state(const uint64_t *p) { return *p; }
inline void st_state(uint64_t *p, uint64_t v) { *p = v; }
inline void st_state_u32(uint32_t *p, uint32_t v) { *p = v; }
inline uint64_t l2_policy(uint32_t) { return 0; }
inline uint64_t ld_stream_p(const uint64_t *p, uint64_t) { return *p; }
inline uint32_t ld_stream_u8_p(const uint8_t *p, uint64_t) { return *p; }
inline uint32_t ld_stream_u32_p(const uint32_t *p, uint64_t) { return *p; }
inline uint64_t ld_state_p(const uint64_t *p, uint64_t) { return *p; }
inline void st_state_p(uint64_t *p, uint64_t v, uint64_t) { *p = v; }
inline void st_state_u32_p(uint32_t *p, uint32_t v, uint64_t) { *p = v; }
// The byte permute and the 16x2 lane instructions of compact_hot_pair, from the CUDA math API's definitions: per
// halfword, unsigned, the add wrapping mod 2^16.  (PRMT in its default mode: selector nibble n picks byte (s >> 4n) & 7
// of {b, a}.)
inline uint32_t __byte_perm(uint32_t a, uint32_t b, uint32_t s) {
  const uint64_t x = ((uint64_t)b << 32) | a;
  uint32_t r = 0;
  for (int n = 0; n < 4; ++n) r |= (uint32_t)((x >> (8 * ((s >> (4 * n)) & 7u))) & 0xFFu) << (8 * n);
  return r;
}
inline uint32_t lane16_of(uint32_t v, int s) { return (v >> s) & 0xFFFFu; }
inline uint32_t lanes16_pack(uint32_t lo, uint32_t hi) { return (lo & 0xFFFFu) | ((hi & 0xFFFFu) << 16); }
inline uint32_t __vminu2(uint32_t a, uint32_t b) {
  const uint32_t l0 = lane16_of(a, 0) < lane16_of(b, 0) ? lane16_of(a, 0) : lane16_of(b, 0);
  const uint32_t l1 = lane16_of(a, 16) < lane16_of(b, 16) ? lane16_of(a, 16) : lane16_of(b, 16);
  return lanes16_pack(l0, l1);
}
inline uint32_t __vmaxu2(uint32_t a, uint32_t b) {
  const uint32_t l0 = lane16_of(a, 0) > lane16_of(b, 0) ? lane16_of(a, 0) : lane16_of(b, 0);
  const uint32_t l1 = lane16_of(a, 16) > lane16_of(b, 16) ? lane16_of(a, 16) : lane16_of(b, 16);
  return lanes16_pack(l0, l1);
}
inline uint32_t __vimax3_u16x2(uint32_t a, uint32_t b, uint32_t c) { return __vmaxu2(__vmaxu2(a, b), c); }
inline uint32_t __viaddmax_u16x2(uint32_t a, uint32_t b, uint32_t c) {  // max(a + b, c) per lane, the sum wrapping
  return __vmaxu2(lanes16_pack(lane16_of(a, 0) + lane16_of(b, 0), lane16_of(a, 16) + lane16_of(b, 16)), c);
}
#endif

// ---- q-th largest of R values held in registers (a15: mis[q()-1] after a descending sort) -------
// 64-bit form: partial selection by bubbling maxima (q passes; R=5: 9 compare-exchanges, each
// 2 ISETP + 4 SEL because sm_90 has no 64-bit integer compare).  Used on the slow path only.
__device__ __forceinline__ void cswap_desc(uint64_t &hi, uint64_t &lo) {
  const uint64_t a = hi, b = lo;
  const bool sw = a < b;
  hi = sw ? b : a;
  lo = sw ? a : b;
}
template <int R>
__device__ __forceinline__ uint64_t quorum_index64(const uint64_t (&m)[R]) {
  constexpr int Q = R / 2 + 1;  // a7: q() = len(prs)/2 + 1
  uint64_t v[R];
#pragma unroll
  for (int i = 0; i < R; ++i) v[i] = m[i];
#pragma unroll
  for (int p = 0; p < Q; ++p) {
#pragma unroll
    for (int i = R - 1; i > p; --i) cswap_desc(v[i - 1], v[i]);
  }
  return v[Q - 1];
}
// 32-bit form on single-instruction min/max (VIMNMX.U32): the q-th largest of R uint32 values.
template <int R>
__device__ __forceinline__ uint32_t quorum_index32(const uint32_t (&d)[R]) {
  constexpr int Q = R / 2 + 1;
  if constexpr (R == 1) {
    return d[0];
  } else if constexpr (R == 2) {
    return min(d[0], d[1]);  // q = 2: the smaller one
  } else if constexpr (R == 3) {  // median of 3: 4 ops
    return max(min(d[0], d[1]), min(max(d[0], d[1]), d[2]));
  } else if constexpr (R == 5) {  // median of 5: 10 ops — drop the min and max of four, median3 with the fifth
    const uint32_t lo_ab = min(d[0], d[1]), hi_ab = max(d[0], d[1]);
    const uint32_t lo_cd = min(d[2], d[3]), hi_cd = max(d[2], d[3]);
    const uint32_t f = max(lo_ab, lo_cd), g = min(hi_ab, hi_cd);
    return max(min(d[4], f), min(max(d[4], f), g));
  } else {
    uint32_t v[R];
#pragma unroll
    for (int i = 0; i < R; ++i) v[i] = d[i];
#pragma unroll
    for (int p = 0; p < Q; ++p) {
#pragma unroll
      for (int i = R - 1; i > p; --i) {
        const uint32_t a = v[i - 1], b = v[i];
        v[i - 1] = max(a, b);
        v[i] = min(a, b);
      }
    }
    return v[Q - 1];
  }
}
// mci = q-th largest of match[].  Fast path: order statistics commute with the monotone map
// x -> max(x - committed, 0), so when every match is within 2^32 of `committed` (above) or below it
// (clamped to 0: such a value can never be the new commit index) the selection runs on 32-bit
// deltas; any other value falls back to the exact 64-bit network.  Returns the exact mci whenever
// mci > committed, and some value <= committed otherwise (callers only test mci > committed).
// d = max(m - c, 0) if that fits 32 bits; otherwise flags `bad`.  One borrow chain (3 instructions):
// b = all-ones iff m < c (behind: clamps to 0 whatever the distance), hi != 0 otherwise means too far ahead.
__device__ __forceinline__ void delta32(uint64_t m, uint64_t c, uint32_t &d, uint32_t &bad) {
  uint32_t lo, hi, b;
#ifndef MRQ_HOST_EMULATION
  asm("sub.cc.u32 %0, %3, %5;\n\t"
      "subc.cc.u32 %1, %4, %6;\n\t"
      "subc.u32 %2, 0, 0;"
      : "=r"(lo), "=r"(hi), "=r"(b)
      : "r"((uint32_t)m), "r"((uint32_t)(m >> 32)), "r"((uint32_t)c), "r"((uint32_t)(c >> 32)));
#else  // the same borrow chain in C
  const uint64_t diff = m - c;
  lo = (uint32_t)diff;
  hi = (uint32_t)(diff >> 32);
  b = m < c ? 0xFFFFFFFFu : 0u;
#endif
  d = ((b | hi) == 0u) ? lo : 0u;
  bad |= ~b & hi;
}
template <int R>
__device__ __forceinline__ uint64_t quorum_index(const uint64_t (&m)[R], uint64_t committed) {
  uint32_t d[R];
  uint32_t bad = 0;
#pragma unroll
  for (int r = 0; r < R; ++r) delta32(m[r], committed, d[r], bad);
  if (__builtin_expect(bad == 0u, 1)) return committed + quorum_index32<R>(d);
  return quorum_index64<R>(m);
}

// ---- one group's state machine, in registers ------------------------------------------------------
enum : uint32_t {
  D_TERM = 1u << 0, D_LI = 1u << 1, D_LT = 1u << 2, D_COMMIT = 1u << 3, D_GATE = 1u << 4, D_MATCH0 = 1u << 8
};

template <int R>
struct Group {
  uint64_t term, last_index, last_term, committed, gate;
  uint64_t match[R];
  uint32_t role, lead, vote, self, elapsed, rto, hb, votes, strict, ltok;
  uint32_t out, dirty, ev;  // ev: event bits for the counters
  bool lt_valid;
  bool pending;             // a Progress.Match rose and maybeCommit() has not been evaluated yet
  // context
  const uint64_t *lt_ptr;
  uint64_t seed, gg, tick_no;
  uint32_t et, ht;

  static constexpr uint32_t Q = R / 2 + 1;
  enum : uint32_t { EV_CAMPAIGN = 1, EV_WON = 2, EV_STEPDOWN = 4, EV_COMMIT = 8, EV_GRANT = 16, EV_ERROR = 32 };

  __device__ __forceinline__ uint64_t lastTerm() {  // raftLog.lastTerm(), loaded on first use
    if (!lt_valid) {
      last_term = ltok ? term : ld_state(lt_ptr);
      lt_valid = true;
    }
    return last_term;
  }
  __device__ __forceinline__ void setSelfMatch(uint64_t v) {
#pragma unroll
    for (int r = 0; r < R; ++r)
      if ((uint32_t)(r + 1) == self && match[r] != v) {
        match[r] = v;
        dirty |= D_MATCH0 << r;
      }
  }
  // a15 + a16: mci = q-th largest match; commit iff mci > committed && term(mci) == Term, where for a
  // leader term(i) == Term  <=>  term_start <= i <= lastIndex.
  __device__ __forceinline__ bool maybeCommit() {
    const uint64_t mci = quorum_index<R>(match, committed);
    if (mci > committed && mci >= gate && mci <= last_index) {
      committed = mci;
      dirty |= D_COMMIT;
      out |= MRQ_OUT_COMMIT_ADVANCED;
      ev |= EV_COMMIT;
      return true;
    }
    return false;
  }
  // upstream runs maybeCommit() after EVERY successful maybeUpdate.  Within a tick match[] only rises, so
  // the successive quorum indices are non-decreasing and the gate (>= term_start) is monotone in them: as
  // long as no match exceeds lastIndex, evaluating once after the last update commits exactly what the
  // sequence of evaluations would have.  (`strict` marks the other case — an out-of-range ack — and
  // makes every update evaluate immediately, as upstream does.)  Flushed before anything that reads
  // `committed`, changes role, or appends.
  __device__ __forceinline__ void flushCommit() {
    if (pending) {
      pending = false;
      if (maybeCommit()) out |= MRQ_OUT_BCAST_APPEND;  // stepLeader: if r.maybeCommit() { r.bcastAppend() }
    }
  }
  // a12 / upstream raft.reset(term)
  __device__ __forceinline__ void reset(uint64_t t) {
    if (term != t) {
      term = t;
      vote = 0;
      ltok = 0;  // every existing entry carries a smaller term
      dirty |= D_TERM;
    }
    lead = 0;
    elapsed = 0;
    hb = 0;
    votes = 0;
    rto = mrq_randomized_timeout(seed, gg, tick_no, et);
  }
  __device__ __forceinline__ void becomeFollower(uint64_t t, uint32_t ld) {
    flushCommit();
    if (role != MRQ_ROLE_FOLLOWER) {
      out |= MRQ_OUT_STEPPED_DOWN;
      ev |= EV_STEPDOWN;
    }
    reset(t);
    lead = ld;
    role = MRQ_ROLE_FOLLOWER;
    if (gate != kNoGate) {
      gate = kNoGate;
      dirty |= D_GATE;
    }
  }
  // a5: appendEntry(n entries stamped with Term) + self maybeUpdate + maybeCommit
  __device__ __forceinline__ void appendEntry(uint32_t n) {
    last_index += n;
    dirty |= D_LI;
    if (!ltok && (!lt_valid || last_term != term)) {
      last_term = term;
      lt_valid = true;
      dirty |= D_LT;
    }
    ltok = 1;
    setSelfMatch(last_index);
    pending = false;  // the evaluation below subsumes any deferred one: match only rose since
    maybeCommit();
  }
  __device__ __forceinline__ void becomeLeader() {
    reset(term);
    lead = self;
    role = MRQ_ROLE_LEADER;
    strict = 0;
    pending = false;
    out |= MRQ_OUT_BECAME_LEADER;
    ev |= EV_WON;
#pragma unroll
    for (int r = 0; r < R; ++r) {  // reset(): every Progress.Match = 0 (self: lastIndex, set by appendEntry)
      match[r] = 0;
      dirty |= D_MATCH0 << r;
    }
    gate = last_index + 1;  // index of the empty entry appended below: first entry of this term
    dirty |= D_GATE;
    appendEntry(1);
  }
  // a10
  __device__ __forceinline__ void campaign() {
    reset(term + 1);
    vote = self;
    role = MRQ_ROLE_CANDIDATE;
    ev |= EV_CAMPAIGN;
    votes |= 1u << (2u * (self - 1u));  // poll(self, true)
    if (Q == 1u) {
      becomeLeader();
      return;
    }
    out |= MRQ_OUT_CAMPAIGN;
  }
  __device__ __forceinline__ void commitTo(uint64_t c) {  // raftLog.commitTo: monotone; out of range = error
    if (committed < c) {
      if (last_index < c) {
        ev |= EV_ERROR;
        return;
      }
      committed = c;
      dirty |= D_COMMIT;
      out |= MRQ_OUT_COMMIT_ADVANCED;
      ev |= EV_COMMIT;
    }
  }
  __device__ __forceinline__ void replyVote(uint32_t r, bool reject) {
    out |= (reject ? 2u : 1u) << (MRQ_OUT_VOTE_REPLY_SHIFT + 2u * r);
  }
  __device__ __forceinline__ void handleAppend(uint32_t r, bool reject, uint64_t index, uint64_t logterm, uint64_t commit) {
    if (!reject) {
      if (last_index != index) {
        last_index = index;
        dirty |= D_LI;
      }
      if (!lt_valid || last_term != logterm) {
        last_term = logterm;
        lt_valid = true;
        dirty |= D_LT;
      }
      ltok = logterm == term;
      commitTo(commit);
    }
    out |= 1u << (MRQ_OUT_ACK_REPLY_SHIFT + r);
  }
  __device__ __forceinline__ void handleHeartbeat(uint32_t r, uint64_t commit) {
    commitTo(commit);
    out |= 1u << (MRQ_OUT_ACK_REPLY_SHIFT + r);
  }

  // upstream raft.Step(m) for the message in sender slot R_ (id R_+1); R_ is a compile-time slot so
  // match[] stays in registers.
  template <int R_>
  __device__ __forceinline__ void step(uint32_t ty, uint64_t mterm, uint64_t index, const uint64_t *p_logterm,
                                       const uint64_t *p_commit) {
    const uint32_t type = ty & MRQ_MSG_TYPE_MASK;
    const bool reject = (ty & MRQ_MSG_REJECT) != 0;
    const uint32_t from = R_ + 1;
    // a12: term rules
    if (mterm != 0) {
      if (mterm > term) {
        becomeFollower(mterm, type == MRQ_MSG_VOTE ? 0u : from);
      } else if (mterm < term) {
        return;
      }
    }
    if (role == MRQ_ROLE_LEADER) {
      if (type == MRQ_MSG_APP_RESP) {  // a14 + a15/a16
        if (!reject && match[R_] < index) {
          if (index > last_index && !strict) {  // out-of-range ack: from here on evaluate eagerly
            flushCommit();
            strict = 1;
          }
          match[R_] = index;
          dirty |= D_MATCH0 << R_;
          if (strict) {
            if (maybeCommit()) out |= MRQ_OUT_BCAST_APPEND;
          } else {
            pending = true;
          }
        }
      } else if (type == MRQ_MSG_VOTE) {
        replyVote(R_, true);
      }
      return;
    }
    if (role == MRQ_ROLE_CANDIDATE) {
      if (type == MRQ_MSG_VOTE_RESP) {  // a8 + a9
        if (((votes >> (2 * R_)) & 3u) == 0) votes |= (reject ? 2u : 1u) << (2 * R_);
        const uint32_t granted = __popc(votes & 0x5555u);
        const uint32_t total = __popc((votes | (votes >> 1)) & 0x5555u);
        if (granted == Q) {
          becomeLeader();
          out |= MRQ_OUT_BCAST_APPEND;
        } else if (total - granted == Q) {
          becomeFollower(term, 0);
        }
      } else if (type == MRQ_MSG_VOTE) {
        replyVote(R_, true);
      } else if (type == MRQ_MSG_APP) {
        becomeFollower(term, from);
        handleAppend(R_, reject, index, ld_stream(p_logterm), ld_stream(p_commit));
      } else if (type == MRQ_MSG_HEARTBEAT) {
        becomeFollower(term, from);
        handleHeartbeat(R_, ld_stream(p_commit));
      }
      return;
    }
    // follower
    if (type == MRQ_MSG_VOTE) {  // a13
      const uint64_t logterm = ld_stream(p_logterm);
      const uint64_t lt = lastTerm();
      const bool upToDate = logterm > lt || (logterm == lt && index >= last_index);
      if ((vote == 0 || vote == from) && upToDate) {
        elapsed = 0;
        vote = from;
        replyVote(R_, false);
        ev |= EV_GRANT;
      } else {
        replyVote(R_, true);
      }
    } else if (type == MRQ_MSG_APP) {
      elapsed = 0;
      lead = from;
      handleAppend(R_, reject, index, ld_stream(p_logterm), ld_stream(p_commit));
    } else if (type == MRQ_MSG_HEARTBEAT) {
      elapsed = 0;
      lead = from;
      handleHeartbeat(R_, ld_stream(p_commit));
    }
  }

  __device__ __forceinline__ void propose(uint32_t n) {  // a5
    if (role == MRQ_ROLE_LEADER) {
      appendEntry(n);  // (also settles a deferred evaluation; BCAST_APPEND is set either way)
      out |= MRQ_OUT_BCAST_APPEND;
    } else if (role == MRQ_ROLE_CANDIDATE || lead == 0) {
      out |= MRQ_OUT_PROP_DROPPED;
    } else {
      out |= MRQ_OUT_PROP_FORWARD;
    }
  }

  // a3 + a11: Tick()
  __device__ __forceinline__ void tick() {
    if (role == MRQ_ROLE_LEADER) {
      ++hb;
      ++elapsed;
      if (elapsed >= et) elapsed = 0;  // checkQuorum is off (reference raft.go:152-159)
      if (hb >= ht) {
        hb = 0;
        out |= MRQ_OUT_BCAST_HEARTBEAT;
      }
    } else {
      ++elapsed;
      if (elapsed >= rto) {
        elapsed = 0;
        campaign();
      }
    }
  }
};

template <int R, int I>
struct StepAll {
  __device__ static __forceinline__ void run(Group<R> &g, const uint32_t (&ty)[R], const uint64_t (&mt)[R],
                                             const uint64_t (&mi)[R], const InboxView &in, uint64_t gs, uint64_t i) {
    if ((ty[I] & MRQ_MSG_TYPE_MASK) != 0 && (uint32_t)(I + 1) != g.self)
      g.template step<I>(ty[I], mt[I], mi[I], in.logterm + (uint64_t)I * gs + i, in.commit + (uint64_t)I * gs + i);
    StepAll<R, I + 1>::run(g, ty, mt, mi, in, gs, i);
  }
};
template <int R>
struct StepAll<R, R> {
  __device__ static __forceinline__ void run(Group<R> &, const uint32_t (&)[R], const uint64_t (&)[R],
                                             const uint64_t (&)[R], const InboxView &, uint64_t, uint64_t) {}
};

__device__ __forceinline__ void count_events(Counters *c, uint32_t ev) {
  // warp-aggregate: one ballot per event class, lane 0 adds the popcount to this CTA's shard
  c += blockIdx.x & (kCtrShards - 1);
  const unsigned lane = threadIdx.x & 31u;
#pragma unroll
  for (int b = 0; b < 6; ++b) {
    const unsigned m = __ballot_sync(0xFFFFFFFFu, (ev >> b) & 1u);
    if (m != 0 && lane == 0) atomicAdd(&(&c->campaigns)[b], (unsigned long long)__popc(m));
  }
}

// Append one change-feed record per lane with what != 0.  Warp-aggregated over the lanes that reach this call (callers
// run the general tick under divergent guards): one atomic per warp with any change, so a mass election does not
// serialise one atomic per group on the counter.  Records at or past the capacity are counted, not written.
__device__ __forceinline__ void append_change(const TickArgs &a, const uint32_t what, const uint64_t tick_no, const uint64_t i,
                                              const uint64_t term, const uint64_t term_start, const uint32_t vote, const uint32_t role,
                                              const uint32_t lead) {
  const unsigned act = __activemask();
  const unsigned want = __ballot_sync(act, what != 0u);
  if (what == 0u) return;
  const unsigned lane = threadIdx.x & 31u;
  const int leader = __ffs((int)want) - 1;
  unsigned long long base = 0;
  if ((int)lane == leader) base = atomicAdd(a.change_count, (unsigned long long)__popc(want));
  base = __shfl_sync(want, base, leader);
  const unsigned long long at = base + (unsigned long long)__popc(want & ((1u << lane) - 1u));
  if (at < a.change_cap) {
    mrq_change c;
    c.tick = tick_no;
    c.term = term;
    c.term_start = term_start;
    c.group = (uint32_t)i;
    c.vote = (uint8_t)vote;
    c.role = (uint8_t)role;
    c.lead = (uint8_t)lead;
    c.what = (uint8_t)what;
    a.changes[at] = c;
  }
}

// ---- the general per-group tick: every message through the full state machine (a3–a16) ------------------
static constexpr int kTickThreads = 128;
template <int R>
__device__ __forceinline__ uint32_t general_group_tick(const TickArgs &a, const uint64_t i, const uint64_t tick_no) {
  uint32_t ev = 0;
  {
    const bool has_inbox = a.in.type != nullptr;
    // phase 1: group state + the tick's message types
    const uint64_t w_meta = ld_state(a.s.meta + i);
    Group<R> g;
    g.term = ld_state(a.s.term + i);
    g.last_index = ld_state(a.s.last_index + i);
    g.committed = ld_state(a.s.committed + i);
    g.gate = ld_state(a.s.term_start + i);
    uint32_t ty[R];
#pragma unroll
    for (int r = 0; r < R; ++r) ty[r] = has_inbox ? ld_stream_u8(a.in.type + (uint64_t)r * a.gs + i) : 0u;
    const uint32_t nprop = (has_inbox && a.in.prop) ? ld_stream_u32(a.in.prop + i) : 0u;
    // Progress.Match rides in the first wave of loads too (it is only meaningful for leaders, but waiting
    // for `role` would serialise a second round trip in front of the common case)
#pragma unroll
    for (int r = 0; r < R; ++r) g.match[r] = ld_state(a.s.match + (uint64_t)r * a.gs + i);
    const Meta m = meta_unpack(w_meta);
    g.role = m.role; g.lead = m.lead; g.vote = m.vote; g.self = m.self;
    g.elapsed = m.elapsed; g.rto = m.rto; g.hb = m.hb; g.votes = m.votes; g.strict = m.strict; g.ltok = m.ltok;
    g.out = 0; g.dirty = 0; g.ev = 0; g.lt_valid = false; g.last_term = 0; g.pending = false;
    g.lt_ptr = a.s.last_term + i;
    g.seed = a.seed; g.gg = a.group_base + i; g.tick_no = tick_no;
    const uint64_t committed0 = g.committed;
    g.et = a.election_tick; g.ht = a.heartbeat_tick;
    // phase 2: the present messages' term / index
    uint64_t mt[R], mi[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if ((uint32_t)(r + 1) == g.self) ty[r] = 0;  // a node does not message itself
      const bool present = (ty[r] & MRQ_MSG_TYPE_MASK) != 0;
      mt[r] = present ? ld_stream(a.in.term + (uint64_t)r * a.gs + i) : 0ull;
      mi[r] = present ? ld_stream(a.in.index + (uint64_t)r * a.gs + i) : 0ull;
    }
    if (g.role != MRQ_ROLE_LEADER) {
#pragma unroll
      for (int r = 0; r < R; ++r) g.match[r] = 0ull;  // not a leader: Progress is rebuilt by becomeLeader
    }
    // Step every message in sender order, then proposals, then the tick
    StepAll<R, 0>::run(g, ty, mt, mi, a.in, a.gs, i);
    if (nprop) g.propose(nprop);
    g.flushCommit();
    g.tick();
    // write back what changed
    Meta o;
    o.role = g.role; o.lead = g.lead; o.vote = g.vote; o.self = g.self;
    o.elapsed = g.elapsed; o.rto = g.rto; o.hb = g.hb; o.votes = g.votes; o.strict = g.strict; o.ltok = g.ltok;
    const uint64_t w_new = meta_pack(o);
    if (w_new != w_meta) st_state(a.s.meta + i, w_new);
    if (g.dirty & D_TERM) st_state(a.s.term + i, g.term);
    if (g.dirty & D_LI) st_state(a.s.last_index + i, g.last_index);
    if (g.dirty & D_LT) st_state(a.s.last_term + i, g.last_term);
    if (g.dirty & D_COMMIT) st_state(a.s.committed + i, g.committed);
    if (g.dirty & D_GATE) st_state(a.s.term_start + i, g.gate);
    if (g.role == MRQ_ROLE_LEADER) {
#pragma unroll
      for (int r = 0; r < R; ++r)
        if (g.dirty & (D_MATCH0 << r)) st_state(a.s.match + (uint64_t)r * a.gs + i, g.match[r]);
    }
    st_state_u32(a.s.out + i, g.out);
    if (a.world > 1) gather_store(a, i, g.committed, committed0);  // fused all-gather
    if (a.changes) {  // HardState {term, vote} / SoftState {lead, role} moved: the change feed
      // (D_TERM is set exactly when reset() moved the term; role, lead and vote are meta bits [0,2), [2,6), [6,10))
      const uint32_t d = (uint32_t)(w_new ^ w_meta);
      const uint32_t what = ((g.dirty & D_TERM) ? MRQ_CHANGE_TERM : 0u) | ((d & 0x3C0u) ? MRQ_CHANGE_VOTE : 0u) |
                            ((d & 0x3u) ? MRQ_CHANGE_ROLE : 0u) | ((d & 0x3Cu) ? MRQ_CHANGE_LEAD : 0u);
      append_change(a, what, tick_no, i, g.term, g.role == MRQ_ROLE_LEADER ? g.gate : kNoGate, g.vote, g.role, g.lead);
    }
    ev = g.ev;
  }
  return ev;
}

template <int R>
__device__ __forceinline__ uint32_t general_group_tick(const TickArgs &a, const uint64_t i) {
  return general_group_tick<R>(a, i, *a.tick_cur);
}

// ---- the tick, as two launches ------------------------------------------------------------------------------
// (1) tick_fast_kernel: one thread per group, for the ticks that need none of the role machinery —
//       * a leader whose inbox holds nothing but accepted, same-term, in-range MsgAppResp (steady state):
//         merge the acks (a14), append the proposals (a5), evaluate the quorum once (a15/a16), leader timers;
//       * a follower that hears nothing, or only a same-term MsgHeartbeat from its leader: election timer,
//         electionElapsed = 0, commitTo(m.Commit);
//     lean (no state machine inlined: small code, few registers, high occupancy).  Any other group is left
//     UNTOUCHED and its index appended to the slow list (one warp-aggregated atomic per warp).
// (2) tick_slow_kernel: grid-strides over the slow list and runs general_group_tick on each entry.
// A group is handled by exactly one of the two, and both are exact, so the pair equals the single kernel.
// The fast per-group tick.  Sets `slow` (and touches nothing) when the group needs the general path.
template <int R>
__device__ __forceinline__ void fast_group_tick(const TickArgs &a, const uint64_t i, bool &slow, uint32_t &ev) {
  // Every lane runs the same straight-line code (columns are padded to a multiple of the CTA size, so the
  // lanes past G read zero padding); `valid` only gates stores and the slow-list append.  That keeps the
  // warp collectives below on a full, converged warp.
  const bool valid = i < a.G;
  const uint64_t pol_stream = l2_policy(a.l2_policy ? 1u : 0u);  // inbox, out word: read/written once per tick
  const uint64_t pol_keep = l2_policy(a.l2_policy ? 2u : 0u);    // state columns: reused by the next tick
  {
    const bool has_inbox = a.in.type != nullptr;
    // one wave of independent loads: packed small state, the u64 state columns, Progress.Match, message types
    const uint64_t w_meta = ld_state_p(a.s.meta + i, pol_keep);
    const uint64_t term = ld_state_p(a.s.term + i, pol_keep);
    uint64_t last_index = ld_state_p(a.s.last_index + i, pol_keep);
    uint64_t committed = ld_state_p(a.s.committed + i, pol_keep);
    const uint64_t committed0 = committed;
    const uint64_t gate = ld_state_p(a.s.term_start + i, pol_keep);
    uint32_t ty[R];
#pragma unroll
    for (int r = 0; r < R; ++r) ty[r] = has_inbox ? ld_stream_u8_p(a.in.type + (uint64_t)r * a.gs + i, pol_stream) : 0u;
    const uint32_t nprop = (has_inbox && a.in.prop) ? ld_stream_u32_p(a.in.prop + i, pol_stream) : 0u;
    uint64_t match[R];
#pragma unroll
    for (int r = 0; r < R; ++r) match[r] = ld_state_p(a.s.match + (uint64_t)r * a.gs + i, pol_keep);
    Meta m = meta_unpack(w_meta);
    // second wave: term + (index | commit) of the messages that are present
    uint64_t mt[R], mx[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if ((uint32_t)(r + 1) == m.self) ty[r] = 0;  // a node does not message itself
      const bool present = ty[r] != 0u;
      const uint64_t *px = (ty[r] == MRQ_MSG_HEARTBEAT ? a.in.commit : a.in.index) + (uint64_t)r * a.gs + i;
      mt[r] = present ? ld_stream_p(a.in.term + (uint64_t)r * a.gs + i, pol_stream) : 0ull;
      mx[r] = present ? ld_stream_p(px, pol_stream) : 0ull;
    }
    uint32_t out = 0;
    uint32_t dirty = 0;
    if (m.role == MRQ_ROLE_LEADER) {
      bool ok = !m.strict && m.ltok;
#pragma unroll
      for (int r = 0; r < R; ++r)
        ok = ok && (ty[r] == 0u || (ty[r] == MRQ_MSG_APP_RESP && mt[r] == term && mx[r] <= last_index));
      slow = !ok;
      if (ok) {
        bool changed = false;
#pragma unroll
        for (int r = 0; r < R; ++r)
          if (ty[r] != 0u && match[r] < mx[r]) {  // Progress.maybeUpdate
            match[r] = mx[r];
            dirty |= D_MATCH0 << r;
            changed = true;
          }
        if (nprop) {  // appendEntry: lastTerm already equals Term (ltok), self Match = lastIndex
          last_index += nprop;
          dirty |= D_LI;
#pragma unroll
          for (int r = 0; r < R; ++r)
            if ((uint32_t)(r + 1) == m.self) {
              match[r] = last_index;
              dirty |= D_MATCH0 << r;
            }
          out |= MRQ_OUT_BCAST_APPEND;
          changed = true;
        }
        if (changed) {  // maybeCommit, once (see Group::flushCommit for why once is exact)
          const uint64_t mci = quorum_index<R>(match, committed);
          if (mci > committed && mci >= gate && mci <= last_index) {
            committed = mci;
            dirty |= D_COMMIT;
            out |= MRQ_OUT_COMMIT_ADVANCED | MRQ_OUT_BCAST_APPEND;
            ev |= Group<R>::EV_COMMIT;
          }
        }
        // tickHeartbeat
        ++m.hb;
        ++m.elapsed;
        if (m.elapsed >= a.election_tick) m.elapsed = 0;
        if (m.hb >= a.heartbeat_tick) {
          m.hb = 0;
          out |= MRQ_OUT_BCAST_HEARTBEAT;
        }
      }
    } else if (m.role == MRQ_ROLE_FOLLOWER) {
      bool ok = nprop == 0;
#pragma unroll
      for (int r = 0; r < R; ++r)
        ok = ok && (ty[r] == 0u || (ty[r] == MRQ_MSG_HEARTBEAT && (uint32_t)(r + 1) == m.lead && mt[r] == term &&
                                    mx[r] <= last_index));
      // the election timer must not fire this tick (campaign() is the slow path's business)
      bool heard = false;
#pragma unroll
      for (int r = 0; r < R; ++r) heard = heard || ty[r] != 0u;
      ok = ok && ((heard ? 1u : m.elapsed + 1u) < m.rto);
      slow = !ok;
      if (ok) {
#pragma unroll
        for (int r = 0; r < R; ++r)
          if (ty[r] != 0u) {  // stepFollower MsgHeartbeat: electionElapsed = 0, lead = From, commitTo, reply
            if (committed < mx[r]) {
              committed = mx[r];
              dirty |= D_COMMIT;
              out |= MRQ_OUT_COMMIT_ADVANCED;
              ev |= Group<R>::EV_COMMIT;
            }
            out |= 1u << (MRQ_OUT_ACK_REPLY_SHIFT + r);
          }
        m.elapsed = heard ? 1u : m.elapsed + 1u;  // reset by the heartbeat, then this tick's increment
      }
    } else {
      slow = true;
    }
    // Write-back is decided per WARP, not per lane: if any lane of the warp changed a column, every lane
    // this kernel owns rewrites it (unchanged lanes store the value they loaded).  Whole 32-byte sectors
    // are written, so L2 never has to fetch-and-merge partially written sectors from HBM.
    const uint64_t w_new = meta_pack(m);
    slow = slow && valid;
    const bool mine = valid && !slow;
    if (!mine) ev = 0;
    uint32_t wdirty = mine ? (dirty | (w_new != w_meta ? D_TERM : 0u)) : 0u;  // D_TERM bit reused: "meta changed"
    wdirty = __reduce_or_sync(0xFFFFFFFFu, wdirty);
    if (mine) {
      if (wdirty & D_TERM) st_state_p(a.s.meta + i, w_new, pol_keep);
      if (wdirty & D_LI) st_state_p(a.s.last_index + i, last_index, pol_keep);
      if (wdirty & D_COMMIT) st_state_p(a.s.committed + i, committed, pol_keep);
#pragma unroll
      for (int r = 0; r < R; ++r)
        if (wdirty & (D_MATCH0 << r)) st_state_p(a.s.match + (uint64_t)r * a.gs + i, match[r], pol_keep);
      st_state_u32_p(a.s.out + i, out, pol_stream);
      if (a.world > 1) gather_store(a, i, committed, committed0);  // fused all-gather
    }
  }
}

// ---- the tick on the BYTE FORM of the inbox (include/mrq_packed8.h), without the unpack pass -------------------
// (tick mode 3; validated on hardware in round 2 — tests/test_zz_packed8_gpu.py — and on the host against the CPU
// checker, tests/cpp/tick_host_test.cpp.  Tick mode 4 below supersedes it for dense multi-raft hosts.)
// Reads 4 sender bytes + 1 proposal byte + the two base words per group instead of the 73 B of wide inbox
// columns.  Same split as above: the fast function handles what needs none of the role machinery and leaves every
// other group untouched; the general one materialises that group's bytes into its wide inbox slot (escaped
// messages are already there: the host's wide list is scattered at post time) and runs general_group_tick.
// Whoever decodes a group slides its window (base_index), exactly once per frame.
struct Inbox8 {
  const uint8_t *word;        // [R-1][gs] one byte per remote sender
  const uint8_t *prop8;       // [gs] proposals, or nullptr
  uint64_t *base_index;       // [gs] window base, slid by the decode
  const uint64_t *base_term;  // [gs]
};
static constexpr uint32_t kTypeEscaped = 0xFFu;  // decode marker: "see the wide inbox slot" (never a message type)

// one sender byte -> (type, term, index | commit); `pay` of acks feeds the window rule
__device__ __forceinline__ void decode8(uint32_t w, uint64_t bi, uint64_t bt, uint32_t &ty, uint64_t &mt, uint64_t &mx,
                                        uint32_t &min_ack) {
  const mrq_p8_cell c = mrq_p8_decode(w, bi);
  ty = c.type;
  mt = c.type ? bt : 0ull;
  mx = (c.is_ack || c.is_hb) ? c.value : 0ull;
  if (c.is_ack) min_ack = c.pay < min_ack ? c.pay : min_ack;
  if (w == MRQ_P8_ESCAPE) ty = kTypeEscaped;
}

template <int R>
__device__ __forceinline__ void fast_group_tick8(const TickArgs &a, const Inbox8 &b, const uint64_t i, bool &slow, uint32_t &ev) {
  const bool valid = i < a.G;
  const uint64_t pol_stream = l2_policy(a.l2_policy ? 1u : 0u);
  const uint64_t pol_keep = l2_policy(a.l2_policy ? 2u : 0u);
  {
    const uint64_t w_meta = ld_state_p(a.s.meta + i, pol_keep);
    const uint64_t term = ld_state_p(a.s.term + i, pol_keep);
    uint64_t last_index = ld_state_p(a.s.last_index + i, pol_keep);
    uint64_t committed = ld_state_p(a.s.committed + i, pol_keep);
    const uint64_t committed0 = committed;
    const uint64_t gate = ld_state_p(a.s.term_start + i, pol_keep);
    const uint64_t bi = ld_state_p(b.base_index + i, pol_keep), bt = ld_state_p(b.base_term + i, pol_keep);
    uint32_t wb[R];  // the frame's bytes of this group, indexed by compact row (R-1 of them are used)
#pragma unroll
    for (int j = 0; j < R - 1; ++j) wb[j] = ld_stream_u8_p(b.word + (uint64_t)j * a.gs + i, pol_stream);
    const uint32_t nprop = b.prop8 ? ld_stream_u8_p(b.prop8 + i, pol_stream) : 0u;
    uint64_t match[R];
#pragma unroll
    for (int r = 0; r < R; ++r) match[r] = ld_state_p(a.s.match + (uint64_t)r * a.gs + i, pol_keep);
    Meta m = meta_unpack(w_meta);
    uint32_t ty[R];
    uint64_t mt[R], mx[R];
    uint32_t min_ack = MRQ_P8_NO_ACK;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      ty[r] = 0;
      mt[r] = mx[r] = 0;
      const uint32_t row = mrq_p8_row((uint32_t)r, m.self, (uint32_t)R);
      if (row >= (uint32_t)R - 1u) continue;  // the group's own slot: a node does not message itself
      uint32_t w = 0;
#pragma unroll
      for (int j = 0; j < R - 1; ++j)
        if ((uint32_t)j == row) w = wb[j];
      decode8(w, bi, bt, ty[r], mt[r], mx[r], min_ack);
    }
    uint32_t out = 0;
    uint32_t dirty = 0;
    if (m.role == MRQ_ROLE_LEADER) {
      bool ok = !m.strict && m.ltok;
#pragma unroll
      for (int r = 0; r < R; ++r)
        ok = ok && (ty[r] == 0u || (ty[r] == MRQ_MSG_APP_RESP && mt[r] == term && mx[r] <= last_index));
      slow = !ok;
      if (ok) {
        bool changed = false;
#pragma unroll
        for (int r = 0; r < R; ++r)
          if (ty[r] != 0u && match[r] < mx[r]) {  // Progress.maybeUpdate
            match[r] = mx[r];
            dirty |= D_MATCH0 << r;
            changed = true;
          }
        if (nprop) {  // appendEntry: lastTerm already equals Term (ltok), self Match = lastIndex
          last_index += nprop;
          dirty |= D_LI;
#pragma unroll
          for (int r = 0; r < R; ++r)
            if ((uint32_t)(r + 1) == m.self) {
              match[r] = last_index;
              dirty |= D_MATCH0 << r;
            }
          out |= MRQ_OUT_BCAST_APPEND;
          changed = true;
        }
        if (changed) {  // maybeCommit, once (see Group::flushCommit for why once is exact)
          const uint64_t mci = quorum_index<R>(match, committed);
          if (mci > committed && mci >= gate && mci <= last_index) {
            committed = mci;
            dirty |= D_COMMIT;
            out |= MRQ_OUT_COMMIT_ADVANCED | MRQ_OUT_BCAST_APPEND;
            ev |= Group<R>::EV_COMMIT;
          }
        }
        ++m.hb;  // tickHeartbeat
        ++m.elapsed;
        if (m.elapsed >= a.election_tick) m.elapsed = 0;
        if (m.hb >= a.heartbeat_tick) {
          m.hb = 0;
          out |= MRQ_OUT_BCAST_HEARTBEAT;
        }
      }
    } else if (m.role == MRQ_ROLE_FOLLOWER) {
      bool ok = nprop == 0;
#pragma unroll
      for (int r = 0; r < R; ++r)
        ok = ok && (ty[r] == 0u || (ty[r] == MRQ_MSG_HEARTBEAT && (uint32_t)(r + 1) == m.lead && mt[r] == term &&
                                    mx[r] <= last_index));
      bool heard = false;
#pragma unroll
      for (int r = 0; r < R; ++r) heard = heard || ty[r] != 0u;
      ok = ok && ((heard ? 1u : m.elapsed + 1u) < m.rto);  // the election timer must not fire this tick
      slow = !ok;
      if (ok) {
#pragma unroll
        for (int r = 0; r < R; ++r)
          if (ty[r] != 0u) {  // stepFollower MsgHeartbeat: electionElapsed = 0, lead = From, commitTo, reply
            if (committed < mx[r]) {
              committed = mx[r];
              dirty |= D_COMMIT;
              out |= MRQ_OUT_COMMIT_ADVANCED;
              ev |= Group<R>::EV_COMMIT;
            }
            out |= 1u << (MRQ_OUT_ACK_REPLY_SHIFT + r);
          }
        m.elapsed = heard ? 1u : m.elapsed + 1u;
      }
    } else {
      slow = true;
    }
    const uint64_t w_new = meta_pack(m);
    slow = slow && valid;
    const bool mine = valid && !slow;
    if (!mine) ev = 0;
    // the window: slid by this function only for the groups it handles (the general path slides its own)
    const uint64_t nb = mrq_p8_next_base(bi, min_ack);
    uint32_t wdirty = mine ? (dirty | (w_new != w_meta ? D_TERM : 0u) | (nb != bi ? D_GATE : 0u)) : 0u;  // D_GATE bit reused: "base moved"
    wdirty = __reduce_or_sync(0xFFFFFFFFu, wdirty);
    if (mine) {
      if (wdirty & D_TERM) st_state_p(a.s.meta + i, w_new, pol_keep);
      if (wdirty & D_LI) st_state_p(a.s.last_index + i, last_index, pol_keep);
      if (wdirty & D_COMMIT) st_state_p(a.s.committed + i, committed, pol_keep);
      if (wdirty & D_GATE) st_state_p(b.base_index + i, nb, pol_keep);
#pragma unroll
      for (int r = 0; r < R; ++r)
        if (wdirty & (D_MATCH0 << r)) st_state_p(a.s.match + (uint64_t)r * a.gs + i, match[r], pol_keep);
      st_state_u32_p(a.s.out + i, out, pol_stream);
      if (a.world > 1) gather_store(a, i, committed, committed0);
    }
  }
}

// The general path on the byte form: write this group's decoded messages into its wide inbox slot (an escaped
// sender keeps what the host's wide list scattered there), slide the window, then the unchanged general tick.
template <int R>
__device__ __forceinline__ uint32_t general_group_tick8(const TickArgs &a, const Inbox8 &b, const uint64_t i, const uint64_t tick_no) {
  const uint32_t self = meta_unpack(ld_state(a.s.meta + i)).self;
  const uint64_t bi = ld_state(b.base_index + i), bt = ld_state(b.base_term + i);
  uint32_t min_ack = MRQ_P8_NO_ACK;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const uint64_t o = (uint64_t)r * a.gs + i;
    const uint32_t row = mrq_p8_row((uint32_t)r, self, (uint32_t)R);
    if (row >= (uint32_t)R - 1u) {
      a.in.type[o] = 0;
      continue;
    }
    const uint32_t w = ld_stream_u8(b.word + (uint64_t)row * a.gs + i);
    if (w == MRQ_P8_ESCAPE) continue;  // the wide message is already in the slot
    const mrq_p8_cell c = mrq_p8_decode(w, bi);
    a.in.type[o] = c.type;
    if (c.type == 0) continue;
    a.in.term[o] = bt;
    if (c.is_ack) {
      a.in.index[o] = c.value;
      min_ack = c.pay < min_ack ? c.pay : min_ack;
    } else if (c.is_hb) {
      a.in.commit[o] = c.value;
    } else {
      a.in.index[o] = 0;
    }
  }
  if (a.in.prop) a.in.prop[i] = b.prop8 ? ld_stream_u8(b.prop8 + i) : 0u;
  const uint64_t nb = mrq_p8_next_base(bi, min_ack);
  if (nb != bi) st_state(b.base_index + i, nb);
  return general_group_tick<R>(a, i, tick_no);
}
template <int R>
__device__ __forceinline__ uint32_t general_group_tick8(const TickArgs &a, const Inbox8 &b, const uint64_t i) {
  return general_group_tick8<R>(a, b, i, *a.tick_cur);
}

template <int R>
__global__ void __launch_bounds__(kTickThreads, (R <= 5 ? 8 : (R == 6 ? 7 : 6))) tick_fast_kernel(const TickArgs a) {
  pdl_launch_dependents();
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t ev = 0;
  bool slow = false;
  pdl_wait();
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.tick_next = *a.tick_cur + 1;  // the next tick's number
  fast_group_tick<R>(a, i, slow, ev);
  // hand the groups this kernel did not touch to the slow kernel: one atomic per warp
  const unsigned smask = __ballot_sync(0xFFFFFFFFu, slow);
  if (smask != 0) {
    const unsigned lane = threadIdx.x & 31u;
    unsigned base = 0;
    if (lane == 0) base = atomicAdd(a.slow_count, (unsigned)__popc(smask));
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    if (slow) a.slow_list[base + __popc(smask & ((1u << lane) - 1u))] = (uint32_t)i;
  }
  if (__any_sync(0xFFFFFFFFu, ev != 0)) count_events(a.ctr, ev);
}

template <int R>
__global__ void __launch_bounds__(kTickThreads, (R <= 5 ? 6 : 5)) tick_slow_kernel(const TickArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const unsigned n = *a.slow_count;
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.slow_count_next = 0;  // the next tick's fast kernel starts from zero
  // whole warps iterate together so the warp-aggregated event counting stays converged
  const unsigned stride = gridDim.x * blockDim.x;
  const unsigned rounds = (n + stride - 1) / stride;
  unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
  for (unsigned it = 0; it < rounds; ++it, k += stride) {
    uint32_t ev = 0;
    if (k < n) ev = general_group_tick<R>(a, (uint64_t)a.slow_list[k]);
    if (__any_sync(0xFFFFFFFFu, ev != 0)) count_events(a.ctr, ev);
  }
}

// The same two launches on the byte form (tick mode 3): identical wrappers
// around fast_group_tick8 / general_group_tick8.
struct Tick8Args {
  TickArgs t;
  Inbox8 b;
};
template <int R>
__global__ void __launch_bounds__(kTickThreads, (R <= 5 ? 8 : (R == 6 ? 7 : 6))) tick_fast8_kernel(const Tick8Args a8) {
  const TickArgs &a = a8.t;
  pdl_launch_dependents();
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t ev = 0;
  bool slow = false;
  pdl_wait();
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.tick_next = *a.tick_cur + 1;  // the next tick's number
  fast_group_tick8<R>(a, a8.b, i, slow, ev);
  const unsigned smask = __ballot_sync(0xFFFFFFFFu, slow);
  if (smask != 0) {  // hand the groups this kernel did not touch to the slow kernel: one atomic per warp
    const unsigned lane = threadIdx.x & 31u;
    unsigned base = 0;
    if (lane == 0) base = atomicAdd(a.slow_count, (unsigned)__popc(smask));
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    if (slow) a.slow_list[base + __popc(smask & ((1u << lane) - 1u))] = (uint32_t)i;
  }
  if (__any_sync(0xFFFFFFFFu, ev != 0)) count_events(a.ctr, ev);
}
template <int R>
__global__ void __launch_bounds__(kTickThreads, (R <= 5 ? 6 : 5)) tick_slow8_kernel(const Tick8Args a8) {
  const TickArgs &a = a8.t;
  pdl_launch_dependents();
  pdl_wait();
  const unsigned n = *a.slow_count;
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.slow_count_next = 0;
  const unsigned stride = gridDim.x * blockDim.x;
  const unsigned rounds = (n + stride - 1) / stride;
  unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
  for (unsigned it = 0; it < rounds; ++it, k += stride) {
    uint32_t ev = 0;
    if (k < n) ev = general_group_tick8<R>(a, a8.b, (uint64_t)a.slow_list[k]);
    if (__any_sync(0xFFFFFFFFu, ev != 0)) count_events(a.ctr, ev);
  }
}

// Single-launch form of the same split: every lane runs the fast tick; the CTA then compacts the few lanes
// that need the general path into shared memory and runs general_group_tick on them with converged warps.
// One launch per tick instead of two (the second launch has a fixed cost even on an empty list, which matters
// once a GPU's shard is small), at the price of the general path's register budget for the whole kernel.
template <int R>
__global__ void __launch_bounds__(kTickThreads, (R <= 5 ? 6 : 5)) tick_fused_kernel(const TickArgs a) {
  __shared__ uint32_t s_list[kTickThreads];
  __shared__ unsigned s_n;
  pdl_launch_dependents();
  const uint64_t base = (uint64_t)blockIdx.x * blockDim.x;
  uint32_t ev = 0;
  bool slow = false;
  if (threadIdx.x == 0) s_n = 0;
  pdl_wait();
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.tick_next = *a.tick_cur + 1;
  fast_group_tick<R>(a, base + threadIdx.x, slow, ev);
  __syncthreads();
  const unsigned smask = __ballot_sync(0xFFFFFFFFu, slow);
  if (smask != 0) {  // warp-aggregated append to the CTA's list
    const unsigned lane = threadIdx.x & 31u;
    unsigned pos = 0;
    if (lane == 0) pos = atomicAdd(&s_n, (unsigned)__popc(smask));
    pos = __shfl_sync(0xFFFFFFFFu, pos, 0);
    if (slow) s_list[pos + __popc(smask & ((1u << lane) - 1u))] = threadIdx.x;
  }
  __syncthreads();
  const unsigned n = s_n;
  if (__any_sync(0xFFFFFFFFu, ev != 0)) count_events(a.ctr, ev);
  if (n != 0) {  // CTA-uniform
    uint32_t ev2 = 0;
    if (threadIdx.x < n) ev2 = general_group_tick<R>(a, base + s_list[threadIdx.x]);
    if (__any_sync(0xFFFFFFFFu, ev2 != 0)) count_events(a.ctr, ev2);
  }
}

// single-launch form (every group through the general path): kept for differential testing of the pair above
template <int R>
__global__ void __launch_bounds__(kTickThreads, (R <= 5 ? 6 : 5)) tick_general_kernel(const TickArgs a) {
  pdl_launch_dependents();
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  pdl_wait();
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.tick_next = *a.tick_cur + 1;
  uint32_t ev = 0;
  if (i < a.G) ev = general_group_tick<R>(a, i);
  if (__any_sync(0xFFFFFFFFu, ev != 0)) count_events(a.ctr, ev);
}

// ==== tick mode 4: the tick on COMPACT state + the byte inbox =====================================================
// The wide layout moves 217 B per group-tick at R = 5 (DESIGN.md §4.1), most of it 64-bit indices whose upper halves
// never change.  In mode 4 every index-like column of a group is a 16-bit OFFSET from one per-group u64 base
// `ibase[g]` that only the general path ever reads:
//     c.commit[g]        committed  - ibase
//     c.match[j][g]      Progress.Match of the j-th REMOTE sender - ibase, j = 0..R-2 in ascending id order — the row order
//                         of the byte frame (0 = "at or below ibase": the exact value stays in the wide column, and since
//                         ibase <= committed such a match can neither win a quorum nor be told apart by one)
//     c.match[R-1][g]    lastIndex - ibase            (a leader's own Match IS lastIndex; followers keep theirs here too)
//     c.win[g]           byte-inbox window base - ibase
//     c.gate[g]          term_start - ibase, read only while the gate is still closed (flag bit CF_GATE_OPEN clear)
//     c.flag[g]          CF_COMPACT (these columns, not the wide ones, are the truth for last_index / committed / match /
//                         window base), CF_TERM_OK (base_term == term: window messages carry the group's term),
//                         CF_GATE_OPEN (leader, term_start <= committed: the commit gate can no longer block)
// term, term_start, last_term never change on the fast path: they stay wide and are never read by it.  With the byte
// inbox (R-1 sender bytes + 1 proposal byte) the steady-state tick reads 8 (meta) + 1 + 2 + 2 + 2R + R = 28 B and
// writes 4 (out) + 1 (commit advance) + 2 + 2 + 2(R-1) + 1.5 = 18.5 B per group at R = 5: 46.5 B instead of 217 (a
// leader's timers run on the clock, c.clk below, so its meta word is not rewritten).
// One thread owns FOUR adjacent groups: every column access is one 64-bit (u16 x 4), 128-bit (u32 x 4) or two 128-bit
// (u64 x 4) loads or stores, which also cuts the instruction count per group-tick to a quarter of the scalar kernels'.
// Sixteen bits hold ~43k ticks of log growth at the steady trace's 1.5 proposals per tick; a group that outgrows
// them is re-based by the general path (compact_group picks a fresh base), exactly as a 32-bit one would be.
// Exactness: a group whose values do not fit (compact_span entries from its base), whose tick needs the role machinery, or
// whose frame holds anything but in-window acks / its leader's heartbeat is handed to the general path, which
// materialises the wide columns, runs the unchanged general tick on them, and re-compacts.
enum : uint32_t { CF_COMPACT = 1u, CF_TERM_OK = 2u, CF_GATE_OPEN = 4u };
enum : uint32_t { CD_META = 1u, CD_COMMIT = 2u, CD_WIN = 4u, CD_MATCH0 = 1u << 8, CD_MATCH_ANY = 0xFFu << 8 };
#ifndef MRQ_HOST_EMULATION
static constexpr uint32_t kCompactSpan = 0x7FFFFFFFu;  // offsets stay below 2^31: sums of two never wrap
#else
static uint32_t kCompactSpan = 0x7FFFFFFFu;  // (the host test lowers it to drive groups through the re-base path)
#endif

// The offset columns are `Off` wide in memory (the library: uint16_t; the host test also runs uint32_t); in registers
// every offset is a uint32_t.  The span an offset may reach is kCompactSpan clamped to the width minus one, so that
// the largest value of the type stays free for a gate that is closed for good (compact_group).
typedef uint16_t CompactOff;
template <typename Off>
__device__ __forceinline__ uint32_t compact_span() {
  const uint32_t w = (uint32_t)static_cast<Off>(~Off(0)) - 1u;
  return kCompactSpan < w ? kCompactSpan : w;
}

template <typename Off = uint32_t>
struct CompactViewT {
  uint8_t *flag;    // [gs]
  Off *commit;      // [gs]
  Off *win;         // [gs]
  Off *gate;        // [gs]
  uint32_t *iblo;   // [gs] low word of ibase (fused gather only)
  Off *match;       // [R][gs]
  uint64_t *ibase;  // [gs]
  uint32_t *clk;    // [gs] a compact leader's timer phases (see clk_phase); null: its timers stay in meta
};
using CompactView = CompactViewT<>;

// Clock-relative timers.  On a compact leader's tick both timers are pure clocks — electionElapsed goes to
// (el + 1) mod ElectionTick (checkQuorum is off, nothing else reads or resets it) and heartbeatElapsed to
// (hb + 1) mod HeartbeatTick — so, like the indices against ibase, they are stored against the engine's tick number T
// (the number of the next tick to run): c.clk holds p_el = (el - T) mod ET in bits [0,16) and p_hb = (hb - T) mod HT
// in bits [16,24), and the timers before tick T are (p + T) mod ET / HT.  The phases never change while the group
// stays a compact leader, so the batched tick neither stores them nor the meta word for it; meta's two timer fields
// are not the truth for such a group, as the wide committed / match columns are not.  Anything that changes role or
// term runs on the general path, which materialises the real timers into meta first.
__host__ __device__ __forceinline__ uint32_t clk_phase(uint32_t v, uint64_t T, uint32_t m) {  // (v - T) mod m, v < m
  const uint32_t tm = (uint32_t)(T % m);
  return v >= tm ? v - tm : v + m - tm;
}
__host__ __device__ __forceinline__ uint32_t clk_value(uint32_t p, uint64_t T, uint32_t m) {  // (p + T) mod m, p < m
  const uint32_t s = p + (uint32_t)(T % m);
  return s >= m ? s - m : s;
}

template <int R>
struct CGroup {  // one group's compact state, in registers
  uint64_t meta;
  uint32_t commit, win;
  uint32_t m[R];
};

// Row order.  The byte frame has R-1 rows: the remote senders in ascending id order (the group's own slot left out).
// The compact match column uses the SAME order — row j is the Match of the j-th remote sender — and its last row,
// R-1, is the group's own slot, i.e. lastIndex.  Frame row j therefore updates match row j with no mapping at all (the
// quorum index does not care about the order); the sender's id is only needed for a follower's reply bits.
__host__ __device__ __forceinline__ uint32_t crow_sender(uint32_t j, uint32_t self_id) {  // row j -> sender slot r (0-based)
  return j + (j + 1u >= self_id ? 1u : 0u);
}

// A settled leader: compact, its window messages carry its term, no strict mode, lastTerm == Term.  Only the general
// path changes role, strict, ltok or the flag, and a group that takes it leaves the fast kernels for the rest of the
// launch, so the answer holds for a whole launch.
__device__ __forceinline__ bool compact_settled(const uint32_t flag, const uint64_t meta) {
  constexpr uint64_t kSettled = 3ull | (1ull << 62) | (1ull << 63);  // role, strict, ltok
  return (flag & (CF_COMPACT | CF_TERM_OK)) == (CF_COMPACT | CF_TERM_OK) &&
         (meta & kSettled) == ((uint64_t)MRQ_ROLE_LEADER | (1ull << 63));
}

// The HOT case of a tick, straight-line: a settled leader whose frame holds nothing but in-window acks of its own term.
// This part does the acks, the proposals, the commit and the window; the callers below add the timers.  Returns false
// — with `g` untouched — for anything else; compact_step decides then.
template <int R, typename Off>
__device__ __forceinline__ bool compact_hot_log(CGroup<R> &g, bool hot, const uint32_t flag, const uint32_t (&wb)[R > 1 ? R - 1 : 1],
                                                const uint32_t nprop, const uint32_t gate, uint32_t &out, uint32_t &adv, uint32_t &dirty) {
  uint32_t li = g.m[R - 1];
  hot = hot && li + nprop <= compact_span<Off>();
  uint32_t nm[R];
  uint32_t d = 0, min_ack = MRQ_P8_NO_ACK, kinds = 0, mx_max = 0, moved = 0;
#pragma unroll
  for (int j = 0; j < R - 1; ++j) {
    const uint32_t w = wb[j];
    kinds |= w;
    const bool ack = (w & 1u) != 0u;  // (kind 3 is ruled out below)
    const uint32_t pay = w >> 2;
    const uint32_t mx = ack ? g.win + pay : 0u;
    mx_max = max(mx_max, mx);
    nm[j] = max(g.m[j], mx);          // Progress.maybeUpdate
    moved |= nm[j] ^ g.m[j];
    min_ack = ack ? min(min_ack, pay) : min_ack;
  }
  // an ack beyond lastIndex is upstream's strict path; heartbeats, responses, escapes: not the hot case
  if (!hot || mx_max > li || (kinds & 2u) != 0u) return false;
  uint32_t o = 0;
  li += nprop;  // appendEntry: lastTerm already equals Term (ltok), self Match = lastIndex
  nm[R - 1] = li;
  if (nprop) {
    moved = 1u;
    o |= MRQ_OUT_BCAST_APPEND;
  }
  d = moved != 0u ? CD_MATCH0 : 0u;  // one bit for the whole match column: the write-back stores all its rows
  uint32_t commit = g.commit, q = 0;
  if (d != 0u) {  // maybeCommit, once (see Group::flushCommit for why once is exact)
    uint32_t dl[R];
#pragma unroll
    for (int r = 0; r < R; ++r) dl[r] = max(nm[r], commit) - commit;
    q = quorum_index32<R>(dl);
    const bool open = (flag & CF_GATE_OPEN) != 0u || commit + q >= gate;
    q = (commit + q <= li && open) ? q : 0u;
  }
  if (q != 0u) {
    commit += q;
    d |= CD_COMMIT;
    o |= MRQ_OUT_COMMIT_ADVANCED | MRQ_OUT_BCAST_APPEND;
  }
  if (min_ack < MRQ_P8_NO_ACK && min_ack > MRQ_P8_SLACK) {  // the window slides for whoever decodes the frame
    g.win += min_ack - MRQ_P8_SLACK;
    d |= CD_WIN;
  }
  g.commit = commit;
#pragma unroll
  for (int r = 0; r < R; ++r) g.m[r] = nm[r];
  out = o;
  adv = q;
  dirty = d;
  return true;
}

// The hot step with the timers in meta (c.clk null).
template <int R, typename Off = uint32_t>
__device__ __forceinline__ bool compact_hot_step(CGroup<R> &g, const uint32_t flag, const uint32_t (&wb)[R > 1 ? R - 1 : 1],
                                                 const uint32_t nprop, const uint32_t gate, const uint32_t et, const uint32_t ht,
                                                 uint32_t &out, uint32_t &adv, uint32_t &dirty) {
  uint32_t o, d;
  if (!compact_hot_log<R, Off>(g, compact_settled(flag, g.meta), flag, wb, nprop, gate, o, adv, d)) return false;
  // tickHeartbeat on the packed word: electionElapsed bits [14,26), heartbeatElapsed bits [38,46)
  uint32_t lo = (uint32_t)g.meta, hi = (uint32_t)(g.meta >> 32);
  uint32_t el = ((lo >> 14) & 0xFFFu) + 1u;
  el = el >= et ? 0u : el;
  lo = (lo & ~(0xFFFu << 14)) | (el << 14);
  if (ht <= 1u) {  // HeartbeatTick 1 (reference raft.go:155; launch-uniform): every tick beats, the counter stays 0
    hi &= ~(0xFFu << 6);
    o |= MRQ_OUT_BCAST_HEARTBEAT;
  } else {
    uint32_t hb = ((hi >> 6) & 0xFFu) + 1u;
    if (hb >= ht) {
      hb = 0;
      o |= MRQ_OUT_BCAST_HEARTBEAT;
    }
    hi = (hi & ~(0xFFu << 6)) | (hb << 6);
  }
  const uint64_t nmeta = ((uint64_t)hi << 32) | lo;
  d |= nmeta != g.meta ? CD_META : 0u;
  g.meta = nmeta;
  out = o;
  dirty = d;
  return true;
}

// A compact leader's tickHeartbeat on the clock: its heartbeatElapsed is the byte at bit `shift` of `hbw`, a countdown
// kept in registers (only looked at when HeartbeatTick > 1).  Returns the out bit.
__device__ __forceinline__ uint32_t clk_heartbeat(const uint32_t ht, uint32_t &hbw, const uint32_t shift) {
  if (ht <= 1u) return MRQ_OUT_BCAST_HEARTBEAT;  // HeartbeatTick 1 (reference raft.go:155; launch-uniform): every tick beats
  uint32_t hb = ((hbw >> shift) & 0xFFu) + 1u;
  hb = hb >= ht ? 0u : hb;
  hbw = (hbw & ~(0xFFu << shift)) | (hb << shift);
  return hb == 0u ? MRQ_OUT_BCAST_HEARTBEAT : 0u;
}

// The hot step with clock-relative timers (c.clk): `settled` is compact_settled() of the group, evaluated once per
// launch, and its heartbeatElapsed is the byte at bit `shift` of `hbw` (clk_heartbeat).  The election timer needs no
// work at all, and neither meta nor c.clk changes.
template <int R, typename Off>
__device__ __forceinline__ bool compact_hot_step_clk(CGroup<R> &g, const bool settled, const uint32_t flag,
                                                     const uint32_t (&wb)[R > 1 ? R - 1 : 1], const uint32_t nprop, const uint32_t gate,
                                                     const uint32_t ht, uint32_t &hbw, const uint32_t shift, uint32_t &out, uint32_t &adv,
                                                     uint32_t &dirty) {
  if (!compact_hot_log<R, Off>(g, settled, flag, wb, nprop, gate, out, adv, dirty)) return false;
  out |= clk_heartbeat(ht, hbw, shift);
  return true;
}

// The (Q-1)-th largest of the R-1 remote rows per lane (Q = R/2 + 1), and their maximum in `vmax`.
template <int R>
__device__ __forceinline__ uint32_t pair_kth_largest(const uint32_t (&v)[R > 1 ? R - 1 : 1], uint32_t &vmax) {
  constexpr int N = R - 1, K = R / 2;  // the K-th largest of N
  if constexpr (N <= 0) {
    vmax = 0;
    return 0;
  } else if constexpr (N == 1) {
    vmax = v[0];
    return v[0];
  } else if constexpr (N == 2) {  // K = 1
    vmax = __vmaxu2(v[0], v[1]);
    return vmax;
  } else if constexpr (N == 3) {  // K = 2: the median of 3
    const uint32_t lo = __vminu2(v[0], v[1]), hi = __vmaxu2(v[0], v[1]);
    vmax = __vmaxu2(hi, v[2]);
    return __vmaxu2(lo, __vminu2(hi, v[2]));
  } else if constexpr (N == 4) {  // K = 2: the second largest of 4
    const uint32_t lo01 = __vminu2(v[0], v[1]), hi01 = __vmaxu2(v[0], v[1]);
    const uint32_t lo23 = __vminu2(v[2], v[3]), hi23 = __vmaxu2(v[2], v[3]);
    vmax = __vmaxu2(hi01, hi23);
    return __vimax3_u16x2(__vminu2(hi01, hi23), lo01, lo23);
  } else {  // partial selection: K passes of bubbling maxima to the front
    uint32_t w[N];
#pragma unroll
    for (int i = 0; i < N; ++i) w[i] = v[i];
#pragma unroll
    for (int p = 0; p < K; ++p) {
#pragma unroll
      for (int i = N - 1; i > p; --i) {
        const uint32_t a = w[i - 1], b = w[i];
        w[i - 1] = __vmaxu2(a, b);
        w[i] = __vminu2(a, b);
      }
    }
    vmax = w[0];
    return w[K - 1];
  }
}

// ---- the hot step of TWO groups at once, in the 16-bit lanes of Hopper's 16x2 integer instructions ----------------
// The quad kernel keeps each 16-bit offset column as two u32 words, the pair words: word 0 holds groups 0 (low half)
// and 1 (high half) of the quad, word 1 groups 2 and 3 — exactly as the column lies in memory.  compact_hot_pair runs
// compact_hot_log for both groups of one pair on those words, one VIMNMX / VIADDMNMX .U16x2 per step where the scalar
// step needs one instruction per group, and gives each lane exactly what the scalar step gives its group.  It applies
// only where that is cheap to make exact; otherwise it returns false with nothing changed, and the caller runs the
// scalar steps.  The caller vouches, once per launch, that both groups are settled leaders (compact_settled) still on
// the fast path.  Per tick it declines unless, in both lanes:
//   - every frame byte is "no message" or an ack (kind 0 or 1: no kind 2 or 3);
//   - every Match after the acks is <= lastIndex: for a settled (not strict) leader every stored Match is <= lastIndex,
//     so this is the scalar step's "no ack beyond lastIndex";
//   - lastIndex <= span - 255 and win <= 0xFFBF: no lane sum can wrap (win + 63 <= 0xFFFE, lastIndex + 255 <= span),
//     and the scalar "lastIndex + nprop <= span" holds.  A group is that close to the top only every ~43k ticks, for a
//     few hundred entries; the scalar step then makes the exact re-base decision.
// The commit is mci = max(commit, Q-th largest Match), never commit + q: an order statistic commutes with max(., commit),
// so this is the scalar max(m, commit) - commit network, and mci <= lastIndex by construction.  Since the new lastIndex
// is the largest row, the Q-th largest of R rows is the (Q-1)-th largest of the R-1 remote rows.  As in the scalar step,
// a lane whose Match and lastIndex did not move keeps its commit (after an import commit may sit below the quorum).
// `gate2`: c.gate in the lanes whose commit gate is still closed (CF_GATE_OPEN clear), 0 in the others; such a lane
// commits only an index >= its gate, as maybeCommit's term check does in the scalar step.
// Outputs per lane: `q2` the commit advance, `out2` MRQ_OUT_BCAST_APPEND / MRQ_OUT_COMMIT_ADVANCED (the heartbeat is
// the caller's), and `dirty` the pair's CD_MATCH0 / CD_COMMIT / CD_WIN.  `wq`: the quad's frame words (byte k = group k),
// `pq`: its proposal bytes, `hi`: 0 for groups 0/1, 1 for groups 2/3.
template <int R>
__device__ __forceinline__ bool compact_hot_pair(uint32_t &commit2, uint32_t &win2, uint32_t (&m2)[R], const uint32_t gate2,
                                                 const uint32_t (&wq)[R > 1 ? R - 1 : 1], const uint32_t pq, const int hi, uint32_t &q2,
                                                 uint32_t &out2, uint32_t &dirty) {
  constexpr uint32_t kLo = 0x00010001u;  // 1 in each lane
  const uint32_t span = compact_span<uint16_t>();
  if (span < 0xFFu) return false;  // (only a host test's tiny span)
  const uint32_t li_cap = (span - 0xFFu) * kLo, win_cap = 0xFFBFu * kLo;
  const uint32_t sel = hi ? 0x4342u : 0x4140u;  // the pair's two bytes into the low byte of each lane
  const uint32_t li = m2[R - 1];
  if (__vmaxu2(li, li_cap) != li_cap || __vmaxu2(win2, win_cap) != win_cap) return false;
  uint32_t nm[R > 1 ? R - 1 : 1], kinds = 0, moved = 0, mn = 0x01000100u;
#pragma unroll
  for (int j = 0; j < R - 1; ++j) {
    const uint32_t b = __byte_perm(wq[j], 0u, sel);  // a frame byte per lane: payload << 2 | kind
    kinds |= b;
    const uint32_t ack = (b & kLo) * 0xFFFFu;            // 0xFFFF in a lane with an ack
    const uint32_t pay = (b >> 2) & ack & 0x003F003Fu;   // the ack's payload, 0 elsewhere
    nm[j] = __viaddmax_u16x2(win2 & ack, pay, m2[j]);    // Progress.maybeUpdate(win + pay)
    moved |= nm[j] ^ m2[j];
    mn = __vminu2(mn, (b & ack) | (~ack & 0x01000100u));  // min ack byte; 0x100 (payload 64): no ack
  }
  if ((kinds & 0x00020002u) != 0u) return false;  // a heartbeat, a response, an escape: not the hot case
  uint32_t nmax = 0;
  const uint32_t kth = pair_kth_largest<R>(nm, nmax);
  if (R > 1 && __vmaxu2(nmax, li) != li) return false;  // an ack beyond lastIndex
  const uint32_t np = __byte_perm(pq, 0u, sel);
  const uint32_t nli = li + np;  // (no lane carries: li <= span - 255)
  moved |= np;
  const uint32_t mmask = __vminu2(moved, kLo) * 0xFFFFu;  // 0xFFFF in a lane whose Match or lastIndex moved
  const uint32_t mc = __vmaxu2(commit2, (R > 1 ? kth : nli) & mmask);
  const uint32_t shut = __vminu2(__vmaxu2(gate2, mc) ^ mc, kLo) * 0xFFFFu;  // 0xFFFF in a lane whose gate is above mc
  const uint32_t mci = (mc & ~shut) | (commit2 & shut);
  q2 = mci - commit2;  // (mci >= commit in both lanes: no lane borrows)
  // the window slides by min_ack - 16 when 16 < min_ack < 64: (min_ack & 63) maps the "no ack" 64 to 0
  const uint32_t slide16 = __vmaxu2((mn >> 2) & 0x003F003Fu, 0x00100010u);  // 16 + the slide
  const uint32_t nwin = win2 + slide16 - 0x00100010u;
  out2 = __vminu2(np | q2, kLo) * MRQ_OUT_BCAST_APPEND + __vminu2(q2, kLo) * MRQ_OUT_COMMIT_ADVANCED;
  dirty = (moved != 0u ? CD_MATCH0 : 0u) | (q2 != 0u ? CD_COMMIT : 0u) | (nwin != win2 ? CD_WIN : 0u);
#pragma unroll
  for (int j = 0; j < R - 1; ++j) m2[j] = nm[j];
  m2[R - 1] = nli;
  commit2 = mci;
  win2 = nwin;
  return true;
}


// One tick of one group on compact state, every case the compact form can express.  Returns true (and leaves `g`
// untouched) when the group needs the general path.  `wb[j]`: the frame's byte of row j, `nprop`: the proposal byte,
// `gate`: c.gate of the group (only looked at while CF_GATE_OPEN is clear).  Mirrors fast_group_tick8 in offset space.
// `clk_hb`: null when the timers are in meta; otherwise the timers are clock-relative and *clk_hb is the group's
// heartbeatElapsed, which a leader's tick advances in place of meta's timer fields (a leader then never sets CD_META).
template <int R, typename Off = uint32_t>
__device__ __forceinline__ bool compact_step(CGroup<R> &g, const uint32_t flag, const uint32_t (&wb)[R > 1 ? R - 1 : 1],
                                             const uint32_t nprop, const uint32_t gate, const uint32_t et, const uint32_t ht,
                                             uint32_t &out, uint32_t &adv, uint32_t &dirty, uint32_t *clk_hb = nullptr) {
  out = 0;
  adv = 0;
  dirty = 0;
  if (!(flag & CF_COMPACT)) return true;
  Meta m = meta_unpack(g.meta);
  uint32_t kind[R > 1 ? R - 1 : 1], pay[R > 1 ? R - 1 : 1];
  bool any_ack = false, any_hb = false;
  uint32_t min_ack = MRQ_P8_NO_ACK;
#pragma unroll
  for (int j = 0; j < R - 1; ++j) {
    kind[j] = wb[j] & 3u;
    pay[j] = (wb[j] >> 2) & 63u;
    if (kind[j] == 1u) {
      any_ack = true;
      min_ack = pay[j] < min_ack ? pay[j] : min_ack;
    } else if (kind[j] == 3u) {
      any_hb = true;
    } else if (kind[j] == 2u && (pay[j] <= 2u || pay[j] == 63u)) {
      return true;  // heartbeat-resp, vote-resp, or escaped to the wide list: the general path's business
    } else {
      kind[j] = 0;  // no message
    }
  }
  uint32_t li = g.m[R - 1];
  CGroup<R> n = g;
  if (m.role == MRQ_ROLE_LEADER) {
    if (m.strict || !m.ltok || any_hb) return true;
    if (any_ack && !(flag & CF_TERM_OK)) return true;
    if (li + nprop > compact_span<Off>()) return true;  // time to re-base
    bool changed = false;
#pragma unroll
    for (int j = 0; j < R - 1; ++j)
      if (kind[j] == 1u) {
        const uint32_t mx = g.win + pay[j];
        if (mx > li) return true;  // ack beyond lastIndex: upstream's strict path
        if (n.m[j] < mx) {         // Progress.maybeUpdate
          n.m[j] = mx;
          dirty |= CD_MATCH0 << j;
          changed = true;
        }
      }
    if (nprop) {  // appendEntry: lastTerm already equals Term (ltok), self Match = lastIndex
      li += nprop;
      n.m[R - 1] = li;
      dirty |= CD_MATCH0 << (R - 1);
      out |= MRQ_OUT_BCAST_APPEND;
      changed = true;
    }
    if (changed) {  // maybeCommit, once (see Group::flushCommit for why once is exact)
      uint32_t d[R];
#pragma unroll
      for (int r = 0; r < R; ++r) d[r] = max(n.m[r], n.commit) - n.commit;
      const uint32_t q = quorum_index32<R>(d);
      const uint32_t mci = n.commit + q;
      if (q != 0u && mci <= li && ((flag & CF_GATE_OPEN) != 0u || mci >= gate)) {
        adv = q;
        n.commit = mci;
        dirty |= CD_COMMIT;
        out |= MRQ_OUT_COMMIT_ADVANCED | MRQ_OUT_BCAST_APPEND;
      }
    }
    if (clk_hb) {  // tickHeartbeat on the clock: electionElapsed needs no work, heartbeatElapsed is the caller's
      const uint32_t hb = *clk_hb + 1u >= ht ? 0u : *clk_hb + 1u;
      if (hb == 0u) out |= MRQ_OUT_BCAST_HEARTBEAT;
      *clk_hb = hb;
    } else {
      ++m.hb;  // tickHeartbeat
      ++m.elapsed;
      if (m.elapsed >= et) m.elapsed = 0;
      if (m.hb >= ht) {
        m.hb = 0;
        out |= MRQ_OUT_BCAST_HEARTBEAT;
      }
    }
  } else if (m.role == MRQ_ROLE_FOLLOWER) {
    if (nprop != 0u || any_ack) return true;
    if (any_hb && !(flag & CF_TERM_OK)) return true;
#pragma unroll
    for (int j = 0; j < R - 1; ++j)
      if (kind[j] == 3u && (crow_sender((uint32_t)j, m.self) + 1u != m.lead || g.win + pay[j] > li)) return true;
    if ((any_hb ? 1u : m.elapsed + 1u) >= m.rto) return true;  // the election timer would fire: campaign() is general
#pragma unroll
    for (int j = 0; j < R - 1; ++j)
      if (kind[j] == 3u) {  // stepFollower MsgHeartbeat: electionElapsed = 0, lead = From, commitTo, reply
        const uint32_t mx = g.win + pay[j];
        if (n.commit < mx) {
          adv += mx - n.commit;
          n.commit = mx;
          dirty |= CD_COMMIT;
          out |= MRQ_OUT_COMMIT_ADVANCED;
        }
        out |= 1u << (MRQ_OUT_ACK_REPLY_SHIFT + crow_sender((uint32_t)j, m.self));
      }
    m.elapsed = any_hb ? 1u : m.elapsed + 1u;
  } else {
    return true;
  }
  if (min_ack < MRQ_P8_NO_ACK && min_ack > MRQ_P8_SLACK) {  // the window slides for whoever decodes the frame
    n.win = g.win + (min_ack - MRQ_P8_SLACK);
    dirty |= CD_WIN;
  }
  n.meta = meta_pack(m);
  if (n.meta != g.meta) dirty |= CD_META;
  g = n;
  return false;
}

// The wide values of a COMPACT group i, decoded from its compact columns and handed one by one to put(column, replica
// slot, value) — the columns the compact form holds differently: meta (only a leader's, whose real timers come from
// c.clk against `T`, the number of the next tick to run), committed, the window base, lastIndex, and the Match entries
// the compact form knows (a leader's own = lastIndex; a zero offset means the wide value, <= ibase, stands, and is not
// handed over).  Every other wide column is already exact.  materialise_group stores the values; the group-list export
// (export_group_row) reads them without writing any engine state.  Reads and stores interleave in the order of the
// former single function, so materialise_group compiles as it did.
enum : uint32_t { WV_META, WV_COMMITTED, WV_WINDOW, WV_LAST_INDEX, WV_MATCH };
template <typename Off, typename Put>
__device__ __forceinline__ void decode_compact_group(const StateView &s, const CompactViewT<Off> &c, uint64_t gs, uint32_t R, const uint64_t i,
                                                     const uint64_t T, const uint32_t et, const uint32_t ht, Put &&put) {
  Meta m = meta_unpack(s.meta[i]);
  if (c.clk && m.role == MRQ_ROLE_LEADER) {
    const uint32_t p = c.clk[i];
    m.elapsed = clk_value(p & 0xFFFFu, T, et);
    m.hb = clk_value((p >> 16) & 0xFFu, T, ht);
    put(WV_META, 0u, meta_pack(m));
  }
  const uint64_t ib = c.ibase[i];
  put(WV_COMMITTED, 0u, ib + c.commit[i]);
  put(WV_WINDOW, 0u, ib + c.win[i]);
  put(WV_LAST_INDEX, 0u, ib + c.match[(uint64_t)(R - 1u) * gs + i]);
  if (m.role == MRQ_ROLE_LEADER) {
    put(WV_MATCH, m.self - 1u, ib + c.match[(uint64_t)(R - 1u) * gs + i]);  // a leader's own Match is lastIndex
    for (uint32_t j = 0; j + 1u < R; ++j) {
      const uint32_t v = c.match[(uint64_t)j * gs + i];
      if (v != 0u) put(WV_MATCH, crow_sender(j, m.self), ib + v);  // 0: the wide value (<= ibase) stands
    }
  }
}

// compact -> wide for one group: the wide columns become exact copies (flag and c.clk untouched).  With c.clk, `T` is
// the number of the next tick to run and a leader's real timers are written into meta.
template <typename Off>
__device__ __forceinline__ void materialise_group(const StateView &s, const CompactViewT<Off> &c, uint64_t *base_index, uint64_t gs, uint32_t R,
                                                  const uint64_t i, const uint64_t T = 0, const uint32_t et = 1, const uint32_t ht = 1) {
  if (!(c.flag[i] & CF_COMPACT)) return;
  decode_compact_group(s, c, gs, R, i, T, et, ht, [&](const uint32_t col, const uint32_t r, const uint64_t v) {
    switch (col) {
      case WV_META: s.meta[i] = v; break;
      case WV_COMMITTED: s.committed[i] = v; break;
      case WV_WINDOW: base_index[i] = v; break;
      case WV_LAST_INDEX: s.last_index[i] = v; break;
      default: s.match[(uint64_t)r * gs + i] = v; break;
    }
  });
}

// wide -> compact for one group (after the general path, an import, or a new window base): picks a fresh ibase just
// below min(committed, window base) and writes the offsets; a group that does not fit stays wide (flag 0).  With c.clk,
// `T` is the number of the next tick to run and a leader's timers become phases against it; a leader whose timers are
// out of range (an import: el >= ET or hb >= HT) would not follow the modular rule on its next tick, so it stays wide
// until a general tick has normalised them.
template <typename Off>
__device__ __forceinline__ void compact_group(const StateView &s, const CompactViewT<Off> &c, const uint64_t *base_index,
                                              const uint64_t *base_term, uint64_t gs, uint32_t R, const uint64_t i, const uint64_t T = 0,
                                              const uint32_t et = 1, const uint32_t ht = 1) {
  const Meta m = meta_unpack(s.meta[i]);
  const uint64_t li = s.last_index[i], cm = s.committed[i], wb = base_index[i], gate = s.term_start[i];
  const uint64_t lo = cm < wb ? cm : wb;
  const uint64_t ib = lo ? lo - 1u : 0u;
  const uint64_t span = compact_span<Off>();
  bool fits = m.self >= 1 && m.self <= R && !m.strict && cm <= li && li - ib <= span && wb - ib <= span;
  const bool leader = m.role == MRQ_ROLE_LEADER;
  if (fits && leader) fits = s.match[(uint64_t)(m.self - 1u) * gs + i] == li;  // a leader's own Match is lastIndex
  if (fits && leader && c.clk) fits = m.elapsed < et && m.hb < ht;
  if (!fits) {
    c.flag[i] = 0;
    return;
  }
  if (leader && c.clk) c.clk[i] = clk_phase(m.elapsed, T, et) | (clk_phase(m.hb, T, ht) << 16);
  c.ibase[i] = ib;
  c.iblo[i] = (uint32_t)ib;
  c.commit[i] = (Off)(cm - ib);
  c.win[i] = (Off)(wb - ib);
  for (uint32_t j = 0; j + 1u < R; ++j) {
    Off v = 0;
    if (leader) {
      const uint64_t mv = s.match[(uint64_t)crow_sender(j, m.self) * gs + i];
      v = mv > ib ? (Off)(mv - ib) : (Off)0;  // mv <= lastIndex (not strict), so the offset fits
    }
    c.match[(uint64_t)j * gs + i] = v;
  }
  c.match[(uint64_t)(R - 1u) * gs + i] = (Off)(li - ib);
  constexpr Off kClosed = static_cast<Off>(~Off(0));  // closed for good: above every offset the span allows
  Off go = kClosed;  // (not a leader)
  if (leader) go = gate > ib ? (gate - ib >= (uint64_t)kClosed ? kClosed : (Off)(gate - ib)) : (Off)0;
  c.gate[i] = go;
  c.flag[i] = (uint8_t)(CF_COMPACT | (base_term[i] == s.term[i] ? CF_TERM_OK : 0u) | ((leader && gate <= cm) ? CF_GATE_OPEN : 0u));
}

// ---- rows of a list of groups (mrq_export_groups / mrq_import_groups) --------------------------------------------------
// The columns of mrq_state with n rows instead of G: row k belongs to the k-th listed group; match and votes are
// [R][n].  A null column is neither written (export) nor read (import).
struct GroupRows {
  uint64_t *term, *vote, *committed, *last_index, *last_term, *term_start, *match;
  uint8_t *role, *lead, *self_id, *votes;
  uint16_t *el, *hb, *rto;
};

// Row k of an export: group i exactly as mrq_export_state returns it (the wide columns, the compact ones decoded where
// the group is compact, meta unpacked as unpack_meta_kernel does).  `compact`: the engine's compact state is live (c is
// read only then).  Writes nothing but the row: no engine state, no representation change.
template <typename Off>
__device__ __forceinline__ void export_group_row(const StateView &s, const CompactViewT<Off> &c, const bool compact, uint64_t gs, uint32_t R,
                                                 const uint64_t i, const uint64_t T, const uint32_t et, const uint32_t ht, const GroupRows &o,
                                                 const uint64_t n, const uint64_t k) {
  uint64_t meta = s.meta[i], committed = s.committed[i], li = s.last_index[i];
  if (o.match)
    for (uint32_t r = 0; r < R; ++r) o.match[(uint64_t)r * n + k] = s.match[(uint64_t)r * gs + i];
  if (compact && (c.flag[i] & CF_COMPACT))
    decode_compact_group(s, c, gs, R, i, T, et, ht, [&](const uint32_t col, const uint32_t r, const uint64_t v) {
      switch (col) {
        case WV_META: meta = v; break;
        case WV_COMMITTED: committed = v; break;
        case WV_WINDOW: break;  // (the packed-inbox window base is not part of mrq_state)
        case WV_LAST_INDEX: li = v; break;
        default:
          if (o.match) o.match[(uint64_t)r * n + k] = v;
          break;
      }
    });
  const Meta m = meta_unpack(meta);
  if (o.term) o.term[k] = s.term[i];
  if (o.vote) o.vote[k] = m.vote;
  if (o.committed) o.committed[k] = committed;
  if (o.last_index) o.last_index[k] = li;
  if (o.last_term) o.last_term[k] = s.last_term[i];
  if (o.term_start) o.term_start[k] = s.term_start[i];
  if (o.role) o.role[k] = (uint8_t)m.role;
  if (o.lead) o.lead[k] = (uint8_t)m.lead;
  if (o.self_id) o.self_id[k] = (uint8_t)m.self;
  if (o.el) o.el[k] = (uint16_t)m.elapsed;
  if (o.hb) o.hb[k] = (uint16_t)m.hb;
  if (o.rto) o.rto[k] = (uint16_t)m.rto;
  if (o.votes)
    for (uint32_t r = 0; r < R; ++r) o.votes[(uint64_t)r * n + k] = (uint8_t)((m.votes >> (2 * r)) & 3u);
}

// Row k of an import into group i: what mrq_import_state does to that group, and nothing to any other.  A compact group
// is materialised first (`T`: the number of the next tick to run); then the given wide columns are overwritten and the
// given meta fields packed (pack_meta_kernel's rules), strict and ltok recomputed (fix_strict_kernel's rule), and, with
// the compact state live, the group re-compacted at T — a group that does not fit gets flag 0 and takes the general path
// on its next mode-4 tick, as after a whole-engine import.
template <typename Off>
__device__ __forceinline__ void import_group_row(const StateView &s, const CompactViewT<Off> &c, const bool compact, uint64_t *base_index,
                                                 const uint64_t *base_term, uint64_t gs, uint32_t R, const uint64_t i, const uint64_t T,
                                                 const uint32_t et, const uint32_t ht, const GroupRows &in, const uint64_t n, const uint64_t k) {
  if (compact) materialise_group(s, c, base_index, gs, R, i, T, et, ht);
  if (in.term) s.term[i] = in.term[k];
  if (in.committed) s.committed[i] = in.committed[k];
  if (in.last_index) s.last_index[i] = in.last_index[k];
  if (in.last_term) s.last_term[i] = in.last_term[k];
  if (in.term_start) s.term_start[i] = in.term_start[k];
  if (in.match)
    for (uint32_t r = 0; r < R; ++r) s.match[(uint64_t)r * gs + i] = in.match[(uint64_t)r * n + k];
  Meta m = meta_unpack(s.meta[i]);
  if (in.role) m.role = in.role[k];
  if (in.lead) m.lead = in.lead[k];
  if (in.self_id) m.self = in.self_id[k];
  if (in.vote) m.vote = (uint32_t)in.vote[k];
  if (in.el) m.elapsed = in.el[k];
  if (in.hb) m.hb = in.hb[k];
  if (in.rto) m.rto = in.rto[k];
  if (in.votes) {
    uint32_t w = 0;
    for (uint32_t r = 0; r < R; ++r) w |= (uint32_t)(in.votes[(uint64_t)r * n + k] & 3u) << (2 * r);
    m.votes = w;
  }
  m = meta_unpack(meta_pack(m));  // the fields as stored (an out-of-range role is masked before the strict rule reads it)
  uint32_t strict = 0;
  if (m.role == MRQ_ROLE_LEADER) {
    const uint64_t li = s.last_index[i];
    for (uint32_t r = 0; r < R; ++r) strict |= s.match[(uint64_t)r * gs + i] > li;
  }
  m.strict = strict;
  m.ltok = s.last_term[i] == s.term[i];
  s.meta[i] = meta_pack(m);
  if (compact) compact_group(s, c, base_index, base_term, gs, R, i, T, et, ht);
}

// One tick of a mode-4 launch: where its frame is, and where its per-tick outputs go.
struct TickDesc {
  const uint8_t *word8;  // [R-1][gs] the byte frame (in the slot's staging buffer)
  const uint8_t *prop8;  // [gs] proposal bytes, or nullptr
  InboxView in;          // the slot's wide inbox: escaped messages were scattered there; the general path decodes into it
  uint32_t *out;         // [gs] this tick's out words
  uint8_t *delta;        // [gs] this tick's commit advances, saturating at 255 ("read the index in full")
};
static constexpr uint32_t kMaxTicksPerLaunch = 96;  // descriptors of one launch live in shared memory (96 x 88 B)
template <typename Off = uint32_t>
struct Tick4ArgsT {
  TickArgs t;  // t.in and t.s.out are per tick (TickDesc)
  CompactViewT<Off> c;
  uint64_t *base_index;  // the wide window base (general path only)
  const uint64_t *base_term;
  TickDesc d0;            // nticks == 1: the descriptor rides in the kernel arguments
  const TickDesc *descs;  // nticks > 1: a table in device memory
  uint32_t nticks;
  uint32_t write_through;  // nticks > 1: 1 = the state columns are written after every tick, 0 = after the last one
  unsigned long long *slow_list64;  // (first general tick << 32) | group
};
using Tick4Args = Tick4ArgsT<>;

// The general path of mode 4 for one group, from tick t0 of the launch to its last tick.
template <int R, typename Off>
__device__ __forceinline__ uint32_t slow_group_ticks_c(const Tick4ArgsT<Off> &A, const uint64_t i, const uint32_t t0) {
  const TickArgs &a0 = A.t;
  const uint64_t tick0 = *a0.tick_cur;
  materialise_group(a0.s, A.c, A.base_index, a0.gs, (uint32_t)R, i, tick0 + t0, a0.election_tick, a0.heartbeat_tick);
  uint32_t ev = 0;
  for (uint32_t t = t0; t < A.nticks; ++t) {
    const TickDesc d = A.descs ? A.descs[t] : A.d0;
    TickArgs a = a0;
    a.in = d.in;
    a.s.out = d.out;
    const uint64_t c0 = a.s.committed[i];
    const Inbox8 b{d.word8, d.prop8, A.base_index, A.base_term};
    ev |= general_group_tick8<R>(a, b, i, tick0 + t);
    const uint64_t adv = a.s.committed[i] - c0;
    d.delta[i] = (uint8_t)(adv > 255u ? 255u : adv);
  }
  compact_group(a0.s, A.c, A.base_index, A.base_term, a0.gs, (uint32_t)R, i, tick0 + A.nticks, a0.election_tick, a0.heartbeat_tick);
  return ev;
}

#ifndef MRQ_HOST_EMULATION
// The complete compact step, OUT OF LINE for the quad kernel: the hot step covers the steady state, so this body runs for
// a few groups per tick — inlined four times it only bloated the loop (2,824 SASS instructions, 11 % of the issue
// slots lost to instruction fetch).  By value in, by value out: the caller's registers stay registers.
template <int R>
struct CStepResult {
  CGroup<R> g;
  uint32_t out, adv, dirty, slow, hb;
};
template <int R>
__device__ __noinline__ CStepResult<R> compact_step_cold(CGroup<R> g, uint32_t flag, uint32_t w0123, uint32_t w4567, uint32_t nprop,
                                                         uint32_t gate, uint32_t et, uint32_t ht, uint32_t hb) {
  uint32_t wb[R > 1 ? R - 1 : 1];
#pragma unroll
  for (int j = 0; j < (R > 1 ? R - 1 : 1); ++j) wb[j] = ((j < 4 ? w0123 : w4567) >> (8 * (j & 3))) & 0xFFu;  // the group's R-1 bytes, packed
  CStepResult<R> r;
  r.slow = compact_step<R, CompactOff>(g, flag, wb, nprop, gate, et, ht, r.out, r.adv, r.dirty, &hb) ? 1u : 0u;
  r.g = g;
  r.hb = hb;
  return r;
}
#endif

#ifndef MRQ_HOST_EMULATION
// Vector column accesses with the L2 residency policy of the scalar kernels
struct u32x4 {
  uint32_t v[4];
};
__device__ __forceinline__ u32x4 ld_v4u32_p(const uint32_t *p, uint64_t pol) {
  u32x4 r;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
               : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3])
               : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ void st_v4u32_p(uint32_t *p, const u32x4 &r, uint64_t pol) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "r"(r.v[0]), "r"(r.v[1]),
               "r"(r.v[2]), "r"(r.v[3]), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void ld_v2u64_p(const uint64_t *p, uint64_t pol, uint64_t &a, uint64_t &b) {
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;" : "=l"(a), "=l"(b) : "l"(p), "l"(pol));
}
__device__ __forceinline__ void st_v2u64_p(uint64_t *p, uint64_t a, uint64_t b, uint64_t pol) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.v2.u64 [%0], {%1, %2}, %3;" ::"l"(p), "l"(a), "l"(b), "l"(pol) : "memory");
}
// The 16-bit offset columns: a quad is one 64-bit access, two pair words (compact_hot_pair) as they lie in memory
__device__ __forceinline__ void ld_pairs_p(const uint16_t *p, uint64_t pol, uint32_t &a, uint32_t &b) {
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.u32 {%0, %1}, [%2], %3;" : "=r"(a), "=r"(b) : "l"(p), "l"(pol));
}
__device__ __forceinline__ void st_pairs_p(uint16_t *p, uint32_t a, uint32_t b, uint64_t pol) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.v2.u32 [%0], {%1, %2}, %3;" ::"l"(p), "r"(a), "r"(b), "l"(pol) : "memory");
}
__device__ __forceinline__ u32x4 ld_v4u16_p(const uint16_t *p, uint64_t pol) {  // (widened to one u32 per group)
  uint32_t a, b;
  ld_pairs_p(p, pol, a, b);
  return u32x4{{__byte_perm(a, 0u, 0x4410), __byte_perm(a, 0u, 0x4432), __byte_perm(b, 0u, 0x4410), __byte_perm(b, 0u, 0x4432)}};
}
// group k of a quad held as pair words: get / set its 16-bit lane
__device__ __forceinline__ uint32_t lane16(const uint32_t (&w)[2], int k) { return (w[k >> 1] >> (16 * (k & 1))) & 0xFFFFu; }
__device__ __forceinline__ void set_lane16(uint32_t (&w)[2], int k, uint32_t v) {
  w[k >> 1] = __byte_perm(w[k >> 1], v, (k & 1) ? 0x5410u : 0x3254u);
}
__device__ __forceinline__ uint32_t ld_stream_u16_p(const uint16_t *p, uint64_t pol) {
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u16 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void st_state_u16_p(uint16_t *p, uint32_t v, uint64_t pol) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.u16 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}

// THREADS x 4 groups per CTA.  128 for big shards; a shard of a many-GPU job is too small to fill 132 SMs with 512-group
// CTAs (131,072 groups = 256 of them), so the host picks 64 or 32 threads there: same register budget per SM, more CTAs.
template <int R, int THREADS>
#ifndef MRQ_T4_THREADS_PER_SM
#define MRQ_T4_THREADS_PER_SM 512  // resident threads per SM the register budget is cut for (development knob)
#endif
__global__ void __launch_bounds__(THREADS, (R <= 5 ? MRQ_T4_THREADS_PER_SM : 384) / THREADS) tick_fast4_kernel(const Tick4ArgsT<CompactOff> A) {
  const TickArgs &a = A.t;
  pdl_launch_dependents();
  const uint64_t i0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4u;
  const bool active = i0 < a.gs;       // the whole quad lies inside the padded row (gs is a multiple of 128)
  const uint64_t i = active ? i0 : 0;  // inactive lanes shadow quad 0: they load, never store
  const uint64_t pol_stream = l2_policy(a.l2_policy ? 1u : 0u);
  const uint64_t pol_keep = l2_policy(a.l2_policy ? 2u : 0u);
  pdl_wait();
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.tick_next = *a.tick_cur + A.nticks;
  // ---- the quad's state: one wave of independent 128-bit loads ---------------------------------------------------
  // The offsets stay packed as pair words (compact_hot_pair): cm2[p], wn2[p] and m2[p][r] hold groups 2p and 2p + 1.
  uint64_t meta[4];
  uint32_t flag[4], cm2[2], wn2[2], m2[2][R];
  {
    const uint32_t fw = ld_stream_u32_p(reinterpret_cast<const uint32_t *>(A.c.flag + i), pol_keep);
    ld_v2u64_p(a.s.meta + i, pol_keep, meta[0], meta[1]);
    ld_v2u64_p(a.s.meta + i + 2, pol_keep, meta[2], meta[3]);
    ld_pairs_p(A.c.commit + i, pol_keep, cm2[0], cm2[1]);
    ld_pairs_p(A.c.win + i, pol_keep, wn2[0], wn2[1]);
#pragma unroll
    for (int r = 0; r < R; ++r) ld_pairs_p(A.c.match + (uint64_t)r * a.gs + i, pol_keep, m2[0][r], m2[1][r]);
#pragma unroll
    for (int k = 0; k < 4; ++k) flag[k] = (fw >> (8 * k)) & 0xFFu;
  }
  uint32_t stopped = 0;  // bit k: group k is not this kernel's (padding, or handed to the general path at an earlier tick)
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (!active || i0 + k >= a.G) stopped |= 1u << k;
  uint32_t gt2[2] = {0u, 0u};  // c.gate in the lanes of the few groups whose commit gate is still closed, else 0
  if (((flag[0] & flag[1] & flag[2] & flag[3]) & CF_GATE_OPEN) == 0u) {
    ld_pairs_p(A.c.gate + i, pol_keep, gt2[0], gt2[1]);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (flag[k] & CF_GATE_OPEN) set_lane16(gt2, k, 0u);
  }
  const bool gather = a.world > 1;
  u32x4 iblo{};
  if (gather) iblo = ld_v4u32_p(A.c.iblo + i, pol_keep);
  uint32_t settled = 0;  // bit k: group k is a settled leader (compact_settled), for the whole launch
#pragma unroll
  for (int k = 0; k < 4; ++k) settled |= compact_settled(flag[k], meta[k]) ? 1u << k : 0u;
  // The compact leaders' heartbeatElapsed, one byte per group, counted in registers from the phases in c.clk.  With
  // HeartbeatTick 1 every tick beats and nothing needs counting.  (The bytes of other groups are never used.)
  uint32_t hb4 = 0;
  if (a.heartbeat_tick > 1u) {
    const u32x4 ck = ld_v4u32_p(A.c.clk + i, pol_keep);
    const uint64_t tick0 = *a.tick_cur;
#pragma unroll
    for (int k = 0; k < 4; ++k) hb4 |= (clk_value((ck.v[k] >> 16) & 0xFFu, tick0, a.heartbeat_tick) & 0xFFu) << (8 * k);
  }
  uint32_t acc_dirty = 0, ncommit = 0, ncommit2 = 0;  // ncommit2: the pair steps' count, per lane
  // Frames are loaded TWO ticks ahead of their use (a shard of a many-GPU job has too few warps per SM to hide a load
  // behind other warps: the thread's own next ticks have to cover it), and the per-tick descriptors come from shared
  // memory, so that a frame load never waits for a descriptor load first.
  __shared__ TickDesc s_desc[kMaxTicksPerLaunch];
  if (A.descs) {
    const uint32_t nw = A.nticks * (uint32_t)(sizeof(TickDesc) / 4);
    for (uint32_t w = threadIdx.x; w < nw; w += THREADS) reinterpret_cast<uint32_t *>(s_desc)[w] = reinterpret_cast<const uint32_t *>(A.descs)[w];
  } else if (threadIdx.x == 0) {
    s_desc[0] = A.d0;
  }
  __syncthreads();
  constexpr int NW = R > 1 ? R - 1 : 1;
  auto load_frame = [&](uint32_t t, uint32_t (&w)[NW], uint32_t &pbytes) {
    const TickDesc &dd = s_desc[t];
#pragma unroll
    for (int j = 0; j < R - 1; ++j) w[j] = ld_stream_u32_p(reinterpret_cast<const uint32_t *>(dd.word8 + (uint64_t)j * a.gs + i), pol_stream);
    if (R == 1) w[0] = 0;
    pbytes = dd.prop8 ? ld_stream_u32_p(reinterpret_cast<const uint32_t *>(dd.prop8 + i), pol_stream) : 0u;
  };
  uint32_t wb[NW], pb, wb1[NW], pb1 = 0;
  load_frame(0, wb, pb);
#pragma unroll
  for (int j = 0; j < NW; ++j) wb1[j] = 0;
  if (A.nticks > 1) load_frame(1, wb1, pb1);
  for (uint32_t t = 0; t < A.nticks; ++t) {
    uint32_t wb2[NW], pb2 = 0;
#pragma unroll
    for (int j = 0; j < NW; ++j) wb2[j] = 0;
    if (t + 2 < A.nticks) load_frame(t + 2, wb2, pb2);
    const TickDesc &d = s_desc[t];
    u32x4 outw{};
    uint32_t adv2[2] = {0u, 0u}, newly = 0, tdirty = 0;  // adv2: the commit advance bytes, in the pair words' lanes
    u32x4 lo_old{};
    if (gather) {
#pragma unroll
      for (int k = 0; k < 4; ++k) lo_old.v[k] = iblo.v[k] + lane16(cm2, k);
    }
    const uint32_t pair_ok = settled & ~stopped;
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      uint32_t q2, o2, pd;
      if (((pair_ok >> (2 * p)) & 3u) == 3u && compact_hot_pair<R>(cm2[p], wn2[p], m2[p], gt2[p], wb, pb, p, q2, o2, pd)) {
#pragma unroll
        for (int h = 0; h < 2; ++h) outw.v[2 * p + h] = ((o2 >> (16 * h)) & 0xFFFFu) | clk_heartbeat(a.heartbeat_tick, hb4, 8 * (2 * p + h));
        adv2[p] = __vminu2(q2, 0x00FF00FFu);
        ncommit2 += __vminu2(q2, 0x00010001u);
        tdirty |= pd;
        continue;
      }
      // the pair declined: the scalar steps, one group at a time, unpacked here and repacked after
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = 2 * p + h;
        if (stopped & (1u << k)) continue;
        CGroup<R> g;
        g.meta = meta[k];
        g.commit = lane16(cm2, k);
        g.win = lane16(wn2, k);
#pragma unroll
        for (int r = 0; r < R; ++r) g.m[r] = (m2[p][r] >> (16 * h)) & 0xFFFFu;
        uint32_t wk[R > 1 ? R - 1 : 1];
#pragma unroll
        for (int j = 0; j < (R > 1 ? R - 1 : 1); ++j) wk[j] = (wb[j] >> (8 * k)) & 0xFFu;
        uint32_t o, adv, dirty;
        const uint32_t np = (pb >> (8 * k)) & 0xFFu;
        bool slow = false;
        if (!compact_hot_step_clk<R, CompactOff>(g, (settled >> k) & 1u, flag[k], wk, np, lane16(gt2, k), a.heartbeat_tick, hb4, 8 * k, o, adv,
                                                 dirty)) {
          uint32_t p0 = 0, p1 = 0;  // the group's bytes, four to a word
#pragma unroll
          for (int j = 0; j < R - 1; ++j) {
            if (j < 4) p0 |= wk[j] << (8 * j);
            else p1 |= wk[j] << (8 * (j - 4));
          }
          const CStepResult<R> cr = compact_step_cold<R>(g, flag[k], p0, p1, np, lane16(gt2, k), a.election_tick, a.heartbeat_tick,
                                                         (hb4 >> (8 * k)) & 0xFFu);
          g = cr.g;
          o = cr.out;
          adv = cr.adv;
          dirty = cr.dirty;
          slow = cr.slow != 0u;
          hb4 = (hb4 & ~(0xFFu << (8 * k))) | ((cr.hb & 0xFFu) << (8 * k));
        }
        meta[k] = g.meta;
        set_lane16(cm2, k, g.commit);
        set_lane16(wn2, k, g.win);
#pragma unroll
        for (int r = 0; r < R; ++r) m2[p][r] = __byte_perm(m2[p][r], g.m[r], h ? 0x5410u : 0x3254u);
        if (slow) {
          newly |= 1u << k;
        } else {
          outw.v[k] = o;
          adv2[p] |= (adv > 255u ? 255u : adv) << (16 * h);
          tdirty |= dirty;
          ncommit += adv != 0u;
        }
      }
    }
    const uint32_t dw = __byte_perm(adv2[0], adv2[1], 0x6420);
    if (__any_sync(0xFFFFFFFFu, newly != 0u)) {  // hand those groups (from this tick on) to the general kernel
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const bool s = (newly >> k) & 1u;
        const unsigned smask = __ballot_sync(0xFFFFFFFFu, s);
        if (smask != 0) {
          const unsigned lane = threadIdx.x & 31u;
          unsigned base = 0;
          if (lane == 0) base = atomicAdd(a.slow_count, (unsigned)__popc(smask));
          base = __shfl_sync(0xFFFFFFFFu, base, 0);
          if (s) A.slow_list64[base + __popc(smask & ((1u << lane) - 1u))] = ((unsigned long long)t << 32) | (unsigned long long)(i0 + k);
        }
      }
      stopped |= newly;
    }
    acc_dirty |= tdirty;
    // ---- this tick's outputs (a stopped group's words are rewritten by the general kernel, which runs afterwards) --
    if (active) {
      st_v4u32_p(d.out + i, outw, pol_stream);
      st_state_u32_p(reinterpret_cast<uint32_t *>(d.delta + i), dw, pol_stream);
      if (gather) {  // fused all-gather: the quad's four low bytes in one 32-bit store per peer
        uint32_t lo4 = 0;
        bool carry = false;
        u32x4 lo;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          lo.v[k] = iblo.v[k] + lane16(cm2, k);
          lo4 |= (lo.v[k] & 0xFFu) << (8 * k);
          carry = carry || ((lo.v[k] ^ lo_old.v[k]) >> 8) != 0u;  // anything above the low byte moved (a wrap of the
        }                                                         // low word changes bits 8..31 too)
        const uint64_t at = (uint64_t)a.rank * a.G + i;
        const bool whole = i0 + 3 < a.G && (at & 3u) == 0u && stopped == 0u;
#pragma unroll 1
        for (uint32_t p = 0; p < a.world; ++p) {
          if (whole) {
            st_state_u32_p(reinterpret_cast<uint32_t *>(a.peer_lo[p] + at), lo4, pol_stream);
          } else {
#pragma unroll
            for (int k = 0; k < 4; ++k)
              if (!(stopped & (1u << k))) a.peer_lo[p][at + k] = (uint8_t)lo.v[k];
          }
        }
        if (a.gather_prime || carry) {  // the full index: only when more than its low byte changed (or when priming)
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (!(stopped & (1u << k)) && (a.gather_prime || ((lo.v[k] ^ lo_old.v[k]) >> 8) != 0u)) {
              const uint64_t full = A.c.ibase[i + k] + lane16(cm2, k);
#pragma unroll 1
              for (uint32_t p = 0; p < a.world; ++p) a.peer_full[p][at + k] = full;
            }
        }
      }
    }
    // ---- state write-back: per warp, whole quads (see fast_group_tick for why per warp) -----------------------------
    const bool last = t + 1 == A.nticks;
    if (A.write_through || last) {
      uint32_t wd = __reduce_or_sync(0xFFFFFFFFu, A.write_through ? tdirty : acc_dirty);
      if (active) {  // (a quad whose groups all left the fast path still owes the columns its earlier ticks changed)
        if (wd & CD_META) {
          st_v2u64_p(a.s.meta + i, meta[0], meta[1], pol_keep);
          st_v2u64_p(a.s.meta + i + 2, meta[2], meta[3], pol_keep);
        }
        if (wd & CD_COMMIT) st_pairs_p(A.c.commit + i, cm2[0], cm2[1], pol_keep);
        if (wd & CD_WIN) st_pairs_p(A.c.win + i, wn2[0], wn2[1], pol_keep);
        if (wd & CD_MATCH_ANY) {
#pragma unroll
          for (int r = 0; r < R; ++r) st_pairs_p(A.c.match + (uint64_t)r * a.gs + i, m2[0][r], m2[1][r], pol_keep);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < NW; ++j) {
      wb[j] = wb1[j];
      wb1[j] = wb2[j];
    }
    pb = pb1;
    pb1 = pb2;
  }
  // "commit advanced" events: one warp-reduced atomic
  const unsigned tot = __reduce_add_sync(0xFFFFFFFFu, ncommit + (ncommit2 & 0xFFFFu) + (ncommit2 >> 16));
  if (tot != 0 && (threadIdx.x & 31u) == 0)
    atomicAdd(&a.ctr[blockIdx.x & (kCtrShards - 1)].commits_advanced, (unsigned long long)tot);
}

// The same tick with ONE group per thread: for shards too small to occupy the GPU four groups to a thread (a warp then
// walks ~800 dependent instructions per tick alone on its scheduler, and that chain sets a small shard's floor).
// Scalar column accesses — the bytes no longer matter at this size, the number of warps in flight does.
template <int R>
__global__ void __launch_bounds__(128, 7) tick_fast1_kernel(const Tick4ArgsT<CompactOff> A) {
  const TickArgs &a = A.t;
  pdl_launch_dependents();
  const uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = i0 < a.G;
  const uint64_t i = i0 < a.gs ? i0 : 0;  // (columns are padded to gs: lanes past G read padding)
  const uint64_t pol_stream = l2_policy(a.l2_policy ? 1u : 0u);
  const uint64_t pol_keep = l2_policy(a.l2_policy ? 2u : 0u);
  pdl_wait();
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.tick_next = *a.tick_cur + A.nticks;
  __shared__ TickDesc s_desc[kMaxTicksPerLaunch];
  if (A.descs) {
    const uint32_t nw = A.nticks * (uint32_t)(sizeof(TickDesc) / 4);
    for (uint32_t w = threadIdx.x; w < nw; w += blockDim.x) reinterpret_cast<uint32_t *>(s_desc)[w] = reinterpret_cast<const uint32_t *>(A.descs)[w];
  } else if (threadIdx.x == 0) {
    s_desc[0] = A.d0;
  }
  __syncthreads();
  CGroup<R> g;
  const uint32_t flag = ld_stream_u8_p(A.c.flag + i, pol_keep);
  g.meta = ld_state_p(a.s.meta + i, pol_keep);
  g.commit = ld_stream_u16_p(A.c.commit + i, pol_keep);
  g.win = ld_stream_u16_p(A.c.win + i, pol_keep);
#pragma unroll
  for (int r = 0; r < R; ++r) g.m[r] = ld_stream_u16_p(A.c.match + (uint64_t)r * a.gs + i, pol_keep);
  const uint32_t gate = (flag & CF_GATE_OPEN) ? 0u : ld_stream_u16_p(A.c.gate + i, pol_keep);
  const bool gather = a.world > 1;
  const uint32_t iblo = gather ? ld_stream_u32_p(A.c.iblo + i, pol_keep) : 0u;
  const bool settled = compact_settled(flag, g.meta);  // (as in tick_fast4_kernel)
  uint32_t hb = 0;
  if (a.heartbeat_tick > 1u) hb = clk_value((ld_stream_u32_p(A.c.clk + i, pol_keep) >> 16) & 0xFFu, *a.tick_cur, a.heartbeat_tick) & 0xFFu;
  constexpr int NW = R > 1 ? R - 1 : 1;
  auto load_frame = [&](uint32_t t, uint32_t (&w)[NW], uint32_t &np) {
    const TickDesc &dd = s_desc[t];
#pragma unroll
    for (int j = 0; j < R - 1; ++j) w[j] = ld_stream_u8_p(dd.word8 + (uint64_t)j * a.gs + i, pol_stream);
    if (R == 1) w[0] = 0;
    np = dd.prop8 ? ld_stream_u8_p(dd.prop8 + i, pol_stream) : 0u;
  };
  uint32_t wb[NW], pb, wb1[NW], pb1 = 0;
  load_frame(0, wb, pb);
#pragma unroll
  for (int j = 0; j < NW; ++j) wb1[j] = 0;
  if (A.nticks > 1) load_frame(1, wb1, pb1);
  bool stopped = !valid;
  uint32_t acc_dirty = 0, ncommit = 0;
  __shared__ __align__(16) uint8_t s_lo[128];
  // CTA-wide gather stores need the whole CTA inside the shard and this rank's segment 4-byte aligned
  const bool cta_gather = gather && (uint64_t)(blockIdx.x + 1u) * 128u <= a.G && (((uint64_t)a.rank * a.G) & 3u) == 0u;
  for (uint32_t t = 0; t < A.nticks; ++t) {
    uint32_t wb2[NW], pb2 = 0;
#pragma unroll
    for (int j = 0; j < NW; ++j) wb2[j] = 0;
    if (t + 2 < A.nticks) load_frame(t + 2, wb2, pb2);
    const TickDesc &d = s_desc[t];
    uint32_t o = 0, adv = 0, dirty = 0;
    bool newly = false;
    const uint32_t lo_old = iblo + g.commit;
    if (!stopped) {
      if (!compact_hot_step_clk<R, CompactOff>(g, settled, flag, wb, pb, gate, a.heartbeat_tick, hb, 0, o, adv, dirty)) {
        uint32_t p0 = 0, p1 = 0;
#pragma unroll
        for (int j = 0; j < R - 1; ++j) {
          if (j < 4) p0 |= wb[j] << (8 * j);
          else p1 |= wb[j] << (8 * (j - 4));
        }
        const CStepResult<R> cr = compact_step_cold<R>(g, flag, p0, p1, pb, gate, a.election_tick, a.heartbeat_tick, hb);
        g = cr.g;
        o = cr.out;
        adv = cr.adv;
        dirty = cr.dirty;
        newly = cr.slow != 0u;
        hb = cr.hb;
      }
      if (newly) {
        o = 0;
        adv = 0;
        dirty = 0;
      }
      ncommit += adv != 0u;
    }
    const unsigned smask = __ballot_sync(0xFFFFFFFFu, newly);
    if (smask != 0) {  // hand those groups (from this tick on) to the general kernel
      const unsigned lane = threadIdx.x & 31u;
      unsigned base = 0;
      if (lane == 0) base = atomicAdd(a.slow_count, (unsigned)__popc(smask));
      base = __shfl_sync(0xFFFFFFFFu, base, 0);
      if (newly) A.slow_list64[base + __popc(smask & ((1u << lane) - 1u))] = ((unsigned long long)t << 32) | (unsigned long long)i0;
      stopped = stopped || newly;
    }
    acc_dirty |= dirty;
    if (valid) {  // this tick's outputs (a stopped group's are rewritten by the general kernel, which runs afterwards)
      st_state_u32_p(d.out + i, o, pol_stream);
      d.delta[i] = (uint8_t)(adv > 255u ? 255u : adv);
      if (gather && !cta_gather && !stopped) {  // (ragged CTA, or a shard size that breaks the 4-byte alignment: byte stores)
        const uint32_t lo = iblo + g.commit;
        const uint64_t at = (uint64_t)a.rank * a.G + i;
#pragma unroll 1
        for (uint32_t p = 0; p < a.world; ++p) a.peer_lo[p][at] = (uint8_t)lo;
      }
      if (gather && !stopped) {  // the full index: only when more than its low byte changed (or when priming)
        const uint32_t lo = iblo + g.commit;
        if (a.gather_prime || ((lo ^ lo_old) >> 8) != 0u) {
          const uint64_t at = (uint64_t)a.rank * a.G + i;
          const uint64_t fv = A.c.ibase[i] + g.commit;
#pragma unroll 1
          for (uint32_t p = 0; p < a.world; ++p) a.peer_full[p][at] = fv;
        }
      }
    }
    if (cta_gather) {
      // The CTA's 128 low bytes leave as ONE 128-byte store per peer (warp w serves peers w, w+4): NVLink moves a few
      // large writes far better than 32-byte ones (byte-wide peer stores took over half of an N = 8 tick).
      s_lo[threadIdx.x] = (uint8_t)(iblo + g.commit);  // (a stopped group's byte is rewritten by the general kernel later)
      __syncthreads();
      const uint32_t word = reinterpret_cast<const uint32_t *>(s_lo)[threadIdx.x & 31u];
      const uint64_t at0 = (uint64_t)a.rank * a.G + (uint64_t)blockIdx.x * 128u;
      for (uint32_t p = threadIdx.x >> 5; p < a.world; p += 4u)
        st_state_u32_p(reinterpret_cast<uint32_t *>(a.peer_lo[p] + at0) + (threadIdx.x & 31u), word, pol_stream);
      __syncthreads();
    }
    const bool last = t + 1 == A.nticks;
    if (A.write_through || last) {  // state write-back, per warp (see fast_group_tick)
      const uint32_t wd = __reduce_or_sync(0xFFFFFFFFu, A.write_through ? dirty : acc_dirty);
      if (valid) {
        if (wd & CD_META) st_state_p(a.s.meta + i, g.meta, pol_keep);
        if (wd & CD_COMMIT) st_state_u16_p(A.c.commit + i, g.commit, pol_keep);
        if (wd & CD_WIN) st_state_u16_p(A.c.win + i, g.win, pol_keep);
        if (wd & CD_MATCH_ANY) {
#pragma unroll
          for (int r = 0; r < R; ++r) st_state_u16_p(A.c.match + (uint64_t)r * a.gs + i, g.m[r], pol_keep);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < NW; ++j) {
      wb[j] = wb1[j];
      wb1[j] = wb2[j];
    }
    pb = pb1;
    pb1 = pb2;
  }
  const unsigned tot = __reduce_add_sync(0xFFFFFFFFu, ncommit);
  if (tot != 0 && (threadIdx.x & 31u) == 0)
    atomicAdd(&a.ctr[blockIdx.x & (kCtrShards - 1)].commits_advanced, (unsigned long long)tot);
}

template <int R>
__global__ void __launch_bounds__(kTickThreads, (R <= 5 ? 6 : 5)) tick_slow4_kernel(const Tick4ArgsT<CompactOff> A) {
  const TickArgs &a = A.t;
  pdl_launch_dependents();
  pdl_wait();
  const unsigned n = *a.slow_count;
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.slow_count_next = 0;
  const unsigned stride = gridDim.x * blockDim.x;
  const unsigned rounds = (n + stride - 1) / stride;
  unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
  for (unsigned it = 0; it < rounds; ++it, k += stride) {
    uint32_t ev = 0;
    if (k < n) {
      const unsigned long long e = A.slow_list64[k];
      ev = slow_group_ticks_c<R>(A, (uint64_t)(e & 0xFFFFFFFFull), (uint32_t)(e >> 32));
    }
    if (__any_sync(0xFFFFFFFFu, ev != 0)) count_events(a.ctr, ev);
  }
}

// whole-engine passes between the two representations (import / export / a new window base / a mode switch); `T` is
// the number of the next tick to run (the host's count at enqueue time: stream order makes it exact)
__global__ void __launch_bounds__(256) materialise_all_kernel(StateView s, CompactViewT<CompactOff> c, uint64_t *base_index, uint64_t gs, uint64_t G,
                                                               uint32_t R, int clear_flags, uint64_t T, uint32_t et, uint32_t ht) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  materialise_group(s, c, base_index, gs, R, i, T, et, ht);
  if (clear_flags) c.flag[i] = 0;
}
__global__ void __launch_bounds__(256) compact_all_kernel(StateView s, CompactViewT<CompactOff> c, const uint64_t *base_index,
                                                           const uint64_t *base_term, uint64_t gs, uint64_t G, uint32_t R, uint64_t T,
                                                           uint32_t et, uint32_t ht) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  compact_group(s, c, base_index, base_term, gs, R, i, T, et, ht);
}

// mrq_export_groups / mrq_import_groups: one thread per listed group (the host has checked the list: every group < G,
// and no duplicate in an import, so no two threads of an import touch one group).  `compact`: the compact state is live.
__global__ void __launch_bounds__(256) export_groups_kernel(StateView s, CompactViewT<CompactOff> c, int compact, uint64_t gs, uint32_t R,
                                                             const uint64_t *groups, uint64_t n, uint64_t T, uint32_t et, uint32_t ht,
                                                             GroupRows o) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  export_group_row(s, c, compact != 0, gs, R, groups[k], T, et, ht, o, n, k);
}
__global__ void __launch_bounds__(256) import_groups_kernel(StateView s, CompactViewT<CompactOff> c, int compact, uint64_t *base_index,
                                                             const uint64_t *base_term, uint64_t gs, uint32_t R, const uint64_t *groups,
                                                             uint64_t n, uint64_t T, uint32_t et, uint32_t ht, GroupRows in) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  import_group_row(s, c, compact != 0, base_index, base_term, gs, R, groups[k], T, et, ht, in, n, k);
}
#endif  // !MRQ_HOST_EMULATION

// ---- K3: the standalone quorum kernel (a15–a16) ------------------------------------------------------------
// Reads 8R+16 bytes per group (match[R], committed, term_start); writes committed where it moves.
// Precondition (checked by the fused tick, which has lastIndex in registers): match <= lastIndex.
struct QuorumArgs {
  const uint64_t *match;
  uint64_t *committed;
  const uint64_t *term_start;
  Counters *ctr;
  uint64_t G, gs;
};

template <int R>
__device__ __forceinline__ uint64_t quorum_commit_one(const uint64_t (&m)[R], uint64_t committed, uint64_t gate,
                                                      bool &moved) {
  const uint64_t mci = quorum_index<R>(m, committed);
  moved = mci > committed && mci >= gate;
  return moved ? mci : committed;
}

__device__ __forceinline__ void count_moved(Counters *ctr, unsigned nmoved) {
  if (ctr) {  // warp-shuffle reduction of the "commit advanced" count, one atomic per warp
    const unsigned tot = __reduce_add_sync(0xFFFFFFFFu, nmoved);
    if (tot != 0 && (threadIdx.x & 31u) == 0)
      atomicAdd(&ctr[blockIdx.x & (kCtrShards - 1)].commits_advanced, (unsigned long long)tot);
  }
}

// -- quad form: four groups per thread, every column read as TWO 128-bit loads per thread (sm_90's widest global
//    access, LDG.E.128), 2(R+2) independent 16-byte loads in flight per thread.
struct u64x4 {
  uint64_t v[4];
};
__device__ __forceinline__ u64x4 ld_plain_x4(const uint64_t *p) {
  u64x4 r;
  asm volatile("ld.global.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(r.v[0]), "=l"(r.v[1]) : "l"(p));
  asm volatile("ld.global.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(r.v[2]), "=l"(r.v[3]) : "l"(p + 2));
  return r;
}

// (.L2::256B: the streamed columns are read front to back, so each miss may as well bring its 256-byte neighbourhood)
__device__ __forceinline__ u64x4 ld_stream_x4_pf(const uint64_t *p) {
  u64x4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::256B.v2.u64 {%0, %1}, [%2];" : "=l"(r.v[0]), "=l"(r.v[1]) : "l"(p));
  asm volatile("ld.global.nc.L1::no_allocate.L2::256B.v2.u64 {%0, %1}, [%2];" : "=l"(r.v[2]), "=l"(r.v[3]) : "l"(p + 2));
  return r;
}
__device__ __forceinline__ void st_stream_x4(uint64_t *p, const u64x4 &v) {  // written once, not read back by this kernel
  asm volatile("st.global.cs.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(v.v[0]), "l"(v.v[1]) : "memory");
  asm volatile("st.global.cs.v2.u64 [%0], {%1, %2};" ::"l"(p + 2), "l"(v.v[2]), "l"(v.v[3]) : "memory");
}
__device__ __forceinline__ void st_stream_u64(uint64_t *p, uint64_t v) {
  asm volatile("st.global.cs.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

template <int R, int THREADS>
__global__ void __launch_bounds__(THREADS) quorum_kernel_quad(const QuorumArgs a) {
  pdl_launch_dependents();
  const uint64_t i = ((uint64_t)blockIdx.x * THREADS + threadIdx.x) * 4;
  unsigned nmoved = 0;
  pdl_wait();
  if (i + 3 < a.G) {
    u64x4 mv[R];
#pragma unroll
    for (int r = 0; r < R; ++r) mv[r] = ld_stream_x4_pf(a.match + (uint64_t)r * a.gs + i);
    const u64x4 cm = ld_plain_x4(a.committed + i);
    const u64x4 gt = ld_stream_x4_pf(a.term_start + i);
    u64x4 out;
    bool mvd[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint64_t m[R];
#pragma unroll
      for (int r = 0; r < R; ++r) m[r] = mv[r].v[k];
      out.v[k] = quorum_commit_one<R>(m, cm.v[k], gt.v[k], mvd[k]);
      nmoved += mvd[k];
    }
    if (nmoved == 4u) {  // the usual case under load: two 128-bit stores for the quad
      st_stream_x4(a.committed + i, out);
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (mvd[k]) st_stream_u64(a.committed + i + k, out.v[k]);
    }
  } else {
    for (uint64_t j = i; j < a.G; ++j) {  // ragged tail (< 4 groups)
      uint64_t m[R];
#pragma unroll
      for (int r = 0; r < R; ++r) m[r] = ld_stream(a.match + (uint64_t)r * a.gs + j);
      bool moved;
      const uint64_t c = quorum_commit_one<R>(m, ld_state(a.committed + j), ld_stream(a.term_start + j), moved);
      if (moved) st_state(a.committed + j, c);
      nmoved += moved;
    }
  }
  count_moved(a.ctr, nmoved);
}

// -- 128-bit form: two groups per thread.
__device__ __forceinline__ ulonglong2 ld_stream_v2(const uint64_t *p) {
  ulonglong2 v;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p));
  return v;
}
__device__ __forceinline__ ulonglong2 ld_plain_v2(const uint64_t *p) {
  ulonglong2 v;
  asm volatile("ld.global.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p));
  return v;
}

template <int R>
__global__ void __launch_bounds__(256) quorum_kernel_ldg(const QuorumArgs a) {
  pdl_launch_dependents();
  const uint64_t pair = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t i = pair * 2;
  unsigned nmoved = 0;
  pdl_wait();
  if (i + 1 < a.G) {
    ulonglong2 mv[R];
#pragma unroll
    for (int r = 0; r < R; ++r) mv[r] = ld_stream_v2(a.match + (uint64_t)r * a.gs + i);
    const ulonglong2 cm = ld_plain_v2(a.committed + i);
    const ulonglong2 gt = ld_stream_v2(a.term_start + i);
    uint64_t m0[R], m1[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      m0[r] = mv[r].x;
      m1[r] = mv[r].y;
    }
    bool mv0, mv1;
    const uint64_t c0 = quorum_commit_one<R>(m0, cm.x, gt.x, mv0);
    const uint64_t c1 = quorum_commit_one<R>(m1, cm.y, gt.y, mv1);
    if (mv0 && mv1) {
      asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};" ::"l"(a.committed + i), "l"(c0), "l"(c1) : "memory");
    } else if (mv0) {
      st_state(a.committed + i, c0);
    } else if (mv1) {
      st_state(a.committed + i + 1, c1);
    }
    nmoved = (unsigned)mv0 + (unsigned)mv1;
  } else if (i < a.G) {  // odd tail
    uint64_t m0[R];
#pragma unroll
    for (int r = 0; r < R; ++r) m0[r] = ld_stream(a.match + (uint64_t)r * a.gs + i);
    bool mv0;
    const uint64_t c0 = quorum_commit_one<R>(m0, ld_state(a.committed + i), ld_stream(a.term_start + i), mv0);
    if (mv0) st_state(a.committed + i, c0);
    nmoved = mv0;
  }
  count_moved(a.ctr, nmoved);
}

// -- TMA form: replica columns staged through shared memory by the bulk-copy engine.
// A persistent CTA walks tiles of TILE groups.  For each tile one elected thread issues R+2 1-D bulk
// copies (cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes — UBLKCP in SASS) of
// TILE*8 bytes each (match[0..R-1], committed, term_start) into one of STAGES shared-memory stages and
// arms that stage's mbarrier with the byte count; all threads wait on the barrier, select the quorum
// index from shared memory and store committed where it moves.  No registers are tied up by loads in
// flight: STAGES*(R+2)*TILE*8 bytes per CTA are outstanding regardless of occupancy.
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

template <int R, int TILE, int STAGES>
__global__ void __launch_bounds__(TILE) quorum_kernel_tma(const QuorumArgs a) {
  pdl_launch_dependents();
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int COLS = R + 2;
  uint64_t *tiles = reinterpret_cast<uint64_t *>(smem_raw);                     // [STAGES][COLS][TILE]
  uint64_t *bars = tiles + (size_t)STAGES * COLS * TILE;                        // [STAGES]
  const uint64_t ntiles = a.G / TILE;  // host guarantees G % TILE == 0 for this path (tail goes to an LDG form)
  const uint32_t tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) mbar_init(&bars[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();
  auto issue = [&](uint64_t tile, int s) {
    uint64_t *dst = tiles + (size_t)s * COLS * TILE;
    const uint64_t base = tile * TILE;
    mbar_expect_tx(&bars[s], (uint32_t)(COLS * TILE * 8));
#pragma unroll
    for (int r = 0; r < R; ++r) bulk_g2s(dst + (size_t)r * TILE, a.match + (uint64_t)r * a.gs + base, TILE * 8, &bars[s]);
    bulk_g2s(dst + (size_t)R * TILE, a.committed + base, TILE * 8, &bars[s]);
    bulk_g2s(dst + (size_t)(R + 1) * TILE, a.term_start + base, TILE * 8, &bars[s]);
  };
  // prologue: fill the pipeline
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      const uint64_t t = (uint64_t)blockIdx.x + (uint64_t)s * gridDim.x;
      if (t < ntiles) issue(t, s);
    }
  }
  unsigned nmoved = 0;
  int s = 0;
  uint32_t parity = 0;
  for (uint64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    mbar_wait(&bars[s], parity);
    const uint64_t *src = tiles + (size_t)s * COLS * TILE;
    uint64_t m[R];
#pragma unroll
    for (int r = 0; r < R; ++r) m[r] = src[(size_t)r * TILE + tid];
    const uint64_t cm = src[(size_t)R * TILE + tid];
    const uint64_t gt = src[(size_t)(R + 1) * TILE + tid];
    __syncthreads();  // everyone has drained this stage: it can be refilled
    if (tid == 0) {
      const uint64_t t = tile + (uint64_t)STAGES * gridDim.x;
      if (t < ntiles) issue(t, s);
    }
    bool moved;
    const uint64_t c = quorum_commit_one<R>(m, cm, gt, moved);
    if (moved) st_state(a.committed + tile * TILE + tid, c);
    nmoved += moved;
    if (++s == STAGES) {
      s = 0;
      parity ^= 1u;
    }
  }
  count_moved(a.ctr, nmoved);
}

// ---- a14 as a sparse pass: Progress.maybeUpdate for a list of acks -----------------------------------
__global__ void match_update_kernel(uint64_t *match, uint64_t gs, uint64_t G, uint32_t R, const uint64_t *groups,
                                    const uint8_t *from, const uint64_t *index, size_t n) {
  const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint64_t g = groups[k];
  const uint32_t f = from[k];
  if (g >= G || f < 1 || f > R) return;
  atomicMax(reinterpret_cast<unsigned long long *>(match + (uint64_t)(f - 1) * gs + g), (unsigned long long)index[k]);
}

// ---- inbox plumbing ---------------------------------------------------------------------------------------
struct MsgRec {  // device mirror of mrq_msg (40 bytes payload + 8)
  uint64_t group, term, index, logterm, commit;
  uint8_t type, from, pad[6];
};
static_assert(sizeof(MsgRec) == sizeof(mrq_msg), "mrq_msg layout");

__global__ void scatter_msgs_kernel(InboxView in, uint64_t gs, uint64_t G, uint32_t R, const MsgRec *msgs, size_t n) {
  const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const MsgRec m = msgs[k];
  if (m.group >= G || m.from < 1 || m.from > R) return;
  const uint64_t o = (uint64_t)(m.from - 1) * gs + m.group;
  in.type[o] = m.type;
  in.term[o] = m.term;
  in.index[o] = m.index;
  in.logterm[o] = m.logterm;
  in.commit[o] = m.commit;
}

__global__ void scatter_props_kernel(uint32_t *prop, uint64_t G, const uint64_t *groups, const uint32_t *counts, size_t n) {
  const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  if (groups[k] < G) atomicAdd(prop + groups[k], counts[k]);
}

// Packed inbox (include/mrq.h mrq_inbox_packed): one 32-bit word per slot, decoded against per-group
// base columns the host set with mrq_set_packed_base (robust to host/device pipelining: the decode
// never looks at engine state).  Exact: anything that does not fit escapes to the wide list.
__global__ void __launch_bounds__(256) unpack_inbox_kernel(InboxView in, const uint64_t *base_index,
                                                            const uint64_t *base_term, uint64_t gs, uint64_t G,
                                                            uint32_t R, const uint32_t *word, const uint8_t *prop8) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  const uint64_t bi = base_index[i], bt = base_term[i];
  for (uint32_t r = 0; r < R; ++r) {
    const uint64_t o = (uint64_t)r * gs + i;
    const uint32_t w = word[o];
    const uint32_t type = w & 15u;
    const uint32_t tc = (w >> 5) & 3u;
    const uint64_t pay = w >> 7;
    if (type == 0 || tc == 3u) {  // empty, or escaped to the wide list (scattered afterwards)
      in.type[o] = 0;
      continue;
    }
    in.type[o] = (uint8_t)(type | ((w & 16u) ? MRQ_MSG_REJECT : 0u));
    in.term[o] = bt + tc;
    // only the columns Step() reads for this type are written (index: acks/votes; commit: heartbeats)
    if (type == MRQ_MSG_APP_RESP) {
      in.index[o] = bi + pay;
    } else if (type == MRQ_MSG_HEARTBEAT) {
      in.commit[o] = bi + pay;
    } else if (type == MRQ_MSG_VOTE) {  // payload: bits 0..1 logterm - base_term, bits 2..24 index - base_index
      in.logterm[o] = bt + (pay & 3u);
      in.index[o] = bi + (pay >> 2);
    } else {
      in.index[o] = 0;
    }
  }
  if (in.prop) in.prop[i] = prop8 ? prop8[i] : 0u;
}

// 16-bit form: bits 0..2 kind (0 none, 1 ack, 2 ack|reject, 3 vote-resp grant, 4 vote-resp reject,
// 5 heartbeat, 6 heartbeat-resp, 7 escaped), bits 3..4 term code (term = base_term + c, c in 0..2; 3 = escaped),
// bits 5..15 payload p: ack index / heartbeat commit = base_index + p.  MsgVote / MsgApp always escape.
__global__ void __launch_bounds__(256) unpack16_inbox_kernel(InboxView in, const uint64_t *base_index,
                                                              const uint64_t *base_term, uint64_t gs, uint64_t G,
                                                              uint32_t R, const uint16_t *word, const uint8_t *prop8) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  const uint64_t bi = base_index[i], bt = base_term[i];
  for (uint32_t r = 0; r < R; ++r) {
    const uint64_t o = (uint64_t)r * gs + i;
    const uint32_t w = word[o];
    const uint32_t kind = w & 7u;
    const uint32_t tc = (w >> 3) & 3u;
    const uint64_t pay = w >> 5;
    if (kind == 0 || kind == 7u || tc == 3u) {
      in.type[o] = 0;
      continue;
    }
    in.term[o] = bt + tc;
    if (kind <= 2u) {
      in.type[o] = (uint8_t)(MRQ_MSG_APP_RESP | (kind == 2u ? MRQ_MSG_REJECT : 0u));
      in.index[o] = bi + pay;
    } else if (kind <= 4u) {
      in.type[o] = (uint8_t)(MRQ_MSG_VOTE_RESP | (kind == 4u ? MRQ_MSG_REJECT : 0u));
      in.index[o] = 0;
    } else if (kind == 5u) {
      in.type[o] = MRQ_MSG_HEARTBEAT;
      in.commit[o] = bi + pay;
    } else {
      in.type[o] = MRQ_MSG_HEARTBEAT_RESP;
      in.index[o] = 0;
    }
  }
  if (in.prop) in.prop[i] = prop8 ? prop8[i] : 0u;
}

// Byte form (include/mrq_packed8.h): R-1 rows of one byte per remote sender, the row of the group's own slot
// left out (the own id is the static `self` field of meta: it never changes while the engine runs, so the
// decode is still independent of anything a pipelined host could be behind on).  Also slides the window:
// base_index is read, used for this frame, and advanced for the next one.
// (the per-group body is a function of its own so that tests/cpp/tick_host_test.cpp can run it on the host)
__device__ __forceinline__ void unpack8_group(const InboxView &in, const uint64_t *meta, uint64_t *base_index,
                                              const uint64_t *base_term, uint64_t gs, uint32_t R, const uint8_t *word,
                                              const uint8_t *prop8, const uint64_t i) {
  const uint32_t self = meta_unpack(meta[i]).self;
  const uint64_t bi = base_index[i], bt = base_term[i];
  uint32_t min_ack = MRQ_P8_NO_ACK;
  for (uint32_t r = 0; r < R; ++r) {
    const uint64_t o = (uint64_t)r * gs + i;
    const uint32_t row = mrq_p8_row(r, self, R);
    if (row >= R - 1u) {  // the group's own slot (or an id outside 1..R): nothing is ever sent from there
      in.type[o] = 0;
      continue;
    }
    const mrq_p8_cell c = mrq_p8_decode(word[(uint64_t)row * gs + i], bi);
    in.type[o] = c.type;
    if (c.type == 0) continue;  // none, or escaped to the wide list (scattered afterwards)
    in.term[o] = bt;
    if (c.is_ack) {
      in.index[o] = c.value;
      min_ack = c.pay < min_ack ? c.pay : min_ack;
    } else if (c.is_hb) {
      in.commit[o] = c.value;
    } else {
      in.index[o] = 0;
    }
  }
  const uint64_t nb = mrq_p8_next_base(bi, min_ack);
  if (nb != bi) base_index[i] = nb;
  if (in.prop) in.prop[i] = prop8 ? prop8[i] : 0u;
}
__global__ void __launch_bounds__(256) unpack8_inbox_kernel(InboxView in, const uint64_t *meta, uint64_t *base_index,
                                                             const uint64_t *base_term, uint64_t gs, uint64_t G,
                                                             uint32_t R, const uint8_t *word, const uint8_t *prop8) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  unpack8_group(in, meta, base_index, base_term, gs, R, word, prop8, i);
}

// Compact commit drain: delta = committed - prev (saturated to 255), prev = committed.
__global__ void commit_delta_kernel(const uint64_t *committed, uint64_t *prev, uint8_t *delta, uint64_t G) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  const uint64_t c = committed[i], p = prev[i];
  const uint64_t d = c - p;
  delta[i] = (uint8_t)(d > 255 ? 255 : d);
  prev[i] = d > 255 ? p : c;  // a saturated group keeps its base until the host reads the full value
}

// ---- synthetic trace generation on the device (include/mrq_trace.h) -------------------------------------
__global__ void __launch_bounds__(256) gen_trace_kernel(InboxView in, StateView s, uint64_t gs, uint64_t G, uint32_t R,
                                                        uint64_t group_base, mrq_trace_params p, uint64_t tick) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  const Meta m = meta_unpack(s.meta[i]);
  mrq_trace_view v;
  v.term = s.term[i];
  v.last_index = s.last_index[i];
  v.last_term = s.last_term[i];
  v.committed = s.committed[i];
  v.role = m.role;
  v.lead = m.lead;
  v.self_id = m.self;
  v.votes = m.votes;
  for (uint32_t r = 0; r < R; ++r) {
    const mrq_trace_msg c = mrq_trace_cell(&p, tick, group_base + i, r, &v);
    const uint64_t o = (uint64_t)r * gs + i;
    in.type[o] = c.type;
    in.term[o] = c.term;
    in.index[o] = c.index;
    in.logterm[o] = c.logterm;
    in.commit[o] = c.commit;
  }
  in.prop[i] = mrq_trace_props(&p, tick, group_base + i, &v);
}

// ---- state export helpers ------------------------------------------------------------------------------------
__global__ void unpack_meta_kernel(const uint64_t *meta, uint64_t G, uint8_t *role, uint8_t *lead, uint8_t *self_id,
                                   uint64_t *vote, uint16_t *el, uint16_t *hb, uint16_t *rto, uint8_t *votes, uint64_t gs,
                                   uint32_t R) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  const Meta m = meta_unpack(meta[i]);
  role[i] = (uint8_t)m.role;
  lead[i] = (uint8_t)m.lead;
  self_id[i] = (uint8_t)m.self;
  vote[i] = m.vote;
  el[i] = (uint16_t)m.elapsed;
  hb[i] = (uint16_t)m.hb;
  rto[i] = (uint16_t)m.rto;
  for (uint32_t r = 0; r < R; ++r) votes[(uint64_t)r * gs + i] = (uint8_t)((m.votes >> (2 * r)) & 3u);
}

// Import: small-state columns -> meta.  The strict bit is recomputed from the imported columns
// (some match above lastIndex) by fix_strict_kernel afterwards.
__global__ void pack_meta_kernel(uint64_t *meta, uint64_t G, const uint8_t *role, const uint8_t *lead, const uint8_t *self_id,
                                 const uint64_t *vote, const uint16_t *el, const uint16_t *hb, const uint16_t *rto,
                                 const uint8_t *votes, uint64_t gs, uint32_t R) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  Meta m = meta_unpack(meta[i]);
  if (role) m.role = role[i];
  if (lead) m.lead = lead[i];
  if (self_id) m.self = self_id[i];
  if (vote) m.vote = (uint32_t)vote[i];
  if (el) m.elapsed = el[i];
  if (hb) m.hb = hb[i];
  if (rto) m.rto = rto[i];
  if (votes) {
    uint32_t w = 0;
    for (uint32_t r = 0; r < R; ++r) w |= (uint32_t)(votes[(uint64_t)r * gs + i] & 3u) << (2 * r);
    m.votes = w;
  }
  meta[i] = meta_pack(m);
}

__global__ void fix_strict_kernel(StateView s, uint64_t G, uint64_t gs, uint32_t R) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  Meta m = meta_unpack(s.meta[i]);
  uint32_t strict = 0;
  if (m.role == MRQ_ROLE_LEADER) {
    const uint64_t li = s.last_index[i];
    for (uint32_t r = 0; r < R; ++r) strict |= s.match[(uint64_t)r * gs + i] > li;
  }
  m.strict = strict;
  m.ltok = s.last_term[i] == s.term[i];
  s.meta[i] = meta_pack(m);
}

__global__ void init_state_kernel(StateView s, uint64_t G, uint64_t group_base, uint32_t R, uint32_t self_id, uint64_t seed,
                                  uint32_t election_tick) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  Meta m{};
  m.role = MRQ_ROLE_FOLLOWER;
  m.self = self_id ? self_id : (uint32_t)((group_base + i) % R) + 1u;
  m.rto = mrq_randomized_timeout(seed, group_base + i, 0, election_tick);  // newRaft(): becomeFollower -> reset()
  m.ltok = 1;  // term 0, empty log: lastTerm() == Term
  s.meta[i] = meta_pack(m);
  s.term_start[i] = kNoGate;
}

__global__ void export_next_kernel(const uint64_t *match, const uint64_t *term_start, uint64_t *next, uint64_t G, uint64_t gs,
                                   uint32_t R) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  const uint64_t ts = term_start[i];
  for (uint32_t r = 0; r < R; ++r) {
    const uint64_t mn = match[(uint64_t)r * gs + i] + 1;
    next[(uint64_t)r * G + i] = (ts != kNoGate && ts > mn) ? ts : mn;
  }
}

}  // namespace mrq
