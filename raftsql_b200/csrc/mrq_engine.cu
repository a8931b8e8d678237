// mrq_engine.cu — host side of the C-ABI (include/mrq.h): device state, launches, copies, NCCL/IPC.
//
// Replaces, for G groups at once, the part of the reference's raftNode that owns the raft.Node and
// drives it from one goroutine (reference raft.go:38-78 struct + constructor, :204-246 serveChannels).
// There is NO CPU fallback: without a CUDA device mrq_create fails with MRQ_E_NODEVICE.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <condition_variable>
#include <functional>
#include <algorithm>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_set>
#include <vector>

#include "mrq_kernels.cuh"

using namespace mrq;

namespace {

thread_local std::string g_create_error;

// ---- NCCL through dlopen: single-GPU use never touches it ---------------------------------------
struct NcclUniqueId { char internal[128]; };
typedef void *NcclComm;
struct NcclApi {
  void *lib = nullptr;
  int (*GetUniqueId)(NcclUniqueId *) = nullptr;
  int (*CommInitRank)(NcclComm *, int, NcclUniqueId, int) = nullptr;
  int (*AllGather)(const void *, void *, size_t, int, NcclComm, cudaStream_t) = nullptr;
  int (*CommDestroy)(NcclComm) = nullptr;
  const char *(*GetErrorString)(int) = nullptr;
  std::string err;
  bool load() {
    if (lib) return true;
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char *n : names) {
      lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (lib) break;
    }
    if (!lib) {
      const char *why = dlerror();  // one call: dlerror() clears the message it returns
      err = std::string("dlopen(libnccl.so.2) failed: ") + (why ? why : "?");
      return false;
    }
    GetUniqueId = (int (*)(NcclUniqueId *))dlsym(lib, "ncclGetUniqueId");
    CommInitRank = (int (*)(NcclComm *, int, NcclUniqueId, int))dlsym(lib, "ncclCommInitRank");
    AllGather = (int (*)(const void *, void *, size_t, int, NcclComm, cudaStream_t))dlsym(lib, "ncclAllGather");
    CommDestroy = (int (*)(NcclComm))dlsym(lib, "ncclCommDestroy");
    GetErrorString = (const char *(*)(int))dlsym(lib, "ncclGetErrorString");
    if (!GetUniqueId || !CommInitRank || !AllGather || !CommDestroy) {
      err = "libnccl is missing a required symbol";
      return false;
    }
    return true;
  }
};
NcclApi g_nccl;
constexpr int kNcclUint64 = 5;  // ncclDataType_t::ncclUint64

struct PackedStage {
  void *buf = nullptr;
  size_t bytes = 0;
  cudaEvent_t copied = nullptr, consumed = nullptr;
  bool used = false;
  // tick mode 3: the byte frame of this slot stays in the staging buffer and the tick reads it there
  const uint8_t *word8 = nullptr, *prop8 = nullptr;
  bool frame8 = false;  // a byte frame is waiting for its tick
  bool keep8 = false;   // MRQ_PACKED_KEEP: the frame stays valid after its tick (replayable sequences)
};

struct InboxBuf {
  uint8_t *type = nullptr;
  uint64_t *term = nullptr, *index = nullptr, *logterm = nullptr, *commit = nullptr;
  uint32_t *prop = nullptr;
  InboxView view() const { return InboxView{type, term, index, logterm, commit, prop}; }
};

}  // namespace

struct mrq_engine {
  mrq_config cfg;
  uint64_t G = 0, gs = 0;
  uint32_t R = 0;
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  StateView s{};
  std::vector<InboxBuf> inbox;
  Counters *ctr = nullptr;
  uint64_t *commit_prev = nullptr;  // commit-delta drain base
  uint8_t *delta = nullptr;
  uint64_t *gathered = nullptr;     // [world * G]
  uint64_t *pk_base_index = nullptr, *pk_base_term = nullptr;  // packed-inbox decode bases
  cudaEvent_t drain_done = nullptr;    // mrq_drain_commit_deltas / mrq_drain_wait
  cudaStream_t copy_stream = nullptr;  // H2D of packed inboxes, overlapped with the tick stream
  std::vector<PackedStage> pk_stage;   // one staging buffer per inbox slot
  uint32_t *slow_list = nullptr;    // [gs] groups left to the slow kernel this tick
  unsigned *slow_count = nullptr;   // [2] double-buffered list length
  uint32_t slow_parity = 0;
  uint64_t *tickbuf = nullptr;      // [2] device-resident tick number (current / next), see TickArgs
  uint32_t tick_parity = 0;
  bool gather_prime = false;        // next tick stores the FULL commit index of every group to the peers (not just its low byte)
  bool graphs_disabled = false;
  int graph_mode = 2;               // mrq_set_graph_mode: 0 never, 1 always, 2 auto (small shards only)
  int l2_policy = 1;                // mrq_set_l2_policy: keep state L2-resident, stream the inbox
  std::map<std::string, cudaGraphExec_t> graphs;  // mrq_tick_many: one executable graph per slot sequence
  int tick_mode = 0;                // 0 = fast + slow kernels, 1 = single general kernel
  uint64_t tick_no = 0;
  uint64_t launches = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // scratch for sparse posts
  void *scratch = nullptr;
  size_t scratch_bytes = 0;
  void *pinned = nullptr;
  size_t pinned_bytes = 0;
  // multi-GPU
  NcclComm comm = nullptr;
  uint32_t world = 1, rank = 0, comm_mode = 0;
  uint64_t *peer_gather[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool ipc_attached = false;
  int quorum_variant = 1;  // 0 = quad (4 groups/thread, 2 x LDG.128 per column), 1 = TMA bulk (fastest on H100), 2 = LDG.128
  // tick mode 4: compact state (16-bit offsets from a per-group base) + the byte inbox, four groups per thread
  CompactViewT<CompactOff> c{};
  bool compact_alloc = false;  // the compact columns exist
  bool compact_live = false;   // some groups may be compact-authoritative (wide columns stale for them)
  unsigned long long *slow_list64 = nullptr;
  std::vector<uint32_t *> out_slot;   // per inbox slot: that tick's out words (mrq_tick_many in mode 4)
  std::vector<uint8_t *> delta_slot;  // per inbox slot: that tick's commit advances
  uint32_t *last_out = nullptr;       // where the most recent tick wrote its out words (mrq_sync_out)
  uint8_t *last_delta = nullptr;      // ... and its commit advances (mrq_drain_tick_deltas)
  int write_through = 1;              // multi-tick launches: state columns written after every tick (1) or the last (0)
  uint64_t stage_gen = 0;             // bumps when a staging buffer moves: cached descriptor tables are keyed by it
  std::map<std::string, TickDesc *> desc_tables;
  // change feed (mrq_set_change_capacity): records the general tick appends, and their count since the last drain
  mrq_change *changes = nullptr;
  unsigned long long *change_count = nullptr;
  uint64_t change_cap = 0;
  std::vector<bool> slot_out_live;  // per inbox slot: out_slot / delta_slot hold a tick of the current group count
  bool gather_shared = false;       // mrq_comm_init / mrq_ipc_prepare sized the gather buffer for the peers
  std::string err;
};

namespace {

int fail(mrq_engine *e, int code, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (e)
    e->err = buf;
  else
    g_create_error = buf;
  return code;
}

#define CK(e, call)                                                                                       \
  do {                                                                                                    \
    cudaError_t _st = (call);                                                                             \
    if (_st != cudaSuccess)                                                                               \
      return fail((e), MRQ_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_st), __FILE__, __LINE__); \
  } while (0)

inline unsigned nblocks(uint64_t n, unsigned bs = 256) { return (unsigned)((n + bs - 1) / bs); }

// Launch with programmatic stream serialization (PDL): the grid may start occupying SMs while the previous
// kernel in the stream drains; the kernel itself waits (griddepcontrol.wait) before touching memory.
template <typename Arg>
cudaError_t launch_pdl(void (*kern)(Arg), unsigned grid, unsigned block, size_t smem, cudaStream_t st, const Arg &arg) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  static const bool no_pdl = getenv("MRQ_NO_PDL") != nullptr;  // development switch
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = no_pdl ? 0 : 1;
  return cudaLaunchKernelEx(&cfg, kern, arg);
}

template <typename T>
int dalloc(mrq_engine *e, T **p, size_t n) {
  CK(e, cudaMalloc((void **)p, n * sizeof(T)));
  CK(e, cudaMemsetAsync(*p, 0, n * sizeof(T), e->stream));
  return MRQ_OK;
}

int ensure_scratch(mrq_engine *e, size_t bytes) {
  if (bytes <= e->scratch_bytes) return MRQ_OK;
  if (e->scratch) {
    CK(e, cudaStreamSynchronize(e->stream));
    CK(e, cudaFree(e->scratch));
    e->scratch = nullptr;
    e->scratch_bytes = 0;
  }
  size_t want = bytes < (1u << 20) ? (1u << 20) : bytes;
  CK(e, cudaMalloc(&e->scratch, want));
  e->scratch_bytes = want;
  return MRQ_OK;
}

// strided column copy: host [rows][G] dense  <->  device [rows][gs]
int copy_in(mrq_engine *e, void *dev, const void *host, size_t elem, size_t rows) {
  if (!host) {
    CK(e, cudaMemsetAsync(dev, 0, rows * e->gs * elem, e->stream));
    return MRQ_OK;
  }
  CK(e, cudaMemcpy2DAsync(dev, e->gs * elem, host, e->G * elem, e->G * elem, rows, cudaMemcpyHostToDevice, e->stream));
  return MRQ_OK;
}
int copy_out(mrq_engine *e, void *host, const void *dev, size_t elem, size_t rows) {
  if (!host) return MRQ_OK;
  CK(e, cudaMemcpy2DAsync(host, e->G * elem, dev, e->gs * elem, e->G * elem, rows, cudaMemcpyDeviceToHost, e->stream));
  return MRQ_OK;
}

#define MRQ_DISPATCH_R(R, STMT)  \
  switch (R) {                   \
    case 1: { constexpr int kR = 1; STMT; } break; \
    case 2: { constexpr int kR = 2; STMT; } break; \
    case 3: { constexpr int kR = 3; STMT; } break; \
    case 4: { constexpr int kR = 4; STMT; } break; \
    case 5: { constexpr int kR = 5; STMT; } break; \
    case 6: { constexpr int kR = 6; STMT; } break; \
    case 7: { constexpr int kR = 7; STMT; } break; \
    case 8: { constexpr int kR = 8; STMT; } break; \
    default: break;              \
  }

int g_sm_count = 132;
// Graph replay pays off where the host's launch rate bounds the tick (the shards of a many-GPU job); a 1,048,576-group
// shard is kernel-bound and runs faster on plain PDL stream launches.
constexpr uint64_t kGraphAutoMaxGroups = 600000;


// ---- tick mode 4 plumbing ------------------------------------------------------------------------------------------
int ensure_compact_alloc(mrq_engine *e) {
  if (e->compact_alloc) return MRQ_OK;
  const size_t gs = e->gs;
  int r;
  if ((r = dalloc(e, &e->c.flag, gs))) return r;
  if ((r = dalloc(e, &e->c.commit, gs))) return r;
  if ((r = dalloc(e, &e->c.win, gs))) return r;
  if ((r = dalloc(e, &e->c.gate, gs))) return r;
  if ((r = dalloc(e, &e->c.iblo, gs))) return r;
  if ((r = dalloc(e, &e->c.match, gs * e->R))) return r;
  if ((r = dalloc(e, &e->c.ibase, gs))) return r;
  if ((r = dalloc(e, &e->c.clk, gs))) return r;
  if ((r = dalloc(e, &e->slow_list64, gs))) return r;
  e->compact_alloc = true;
  return MRQ_OK;
}

// Make the WIDE columns exact (compact -> wide for every compact group).  invalidate: the caller is about to change
// wide state, so the compact copies die (every group is re-compacted by the next mode-4 tick).
int ensure_wide(mrq_engine *e, bool invalidate) {
  if (!e->compact_live || e->G == 0) return MRQ_OK;
  materialise_all_kernel<<<nblocks(e->G), 256, 0, e->stream>>>(e->s, e->c, e->pk_base_index, e->gs, e->G, e->R, invalidate ? 1 : 0,
                                                               e->tick_no, e->cfg.election_tick, e->cfg.heartbeat_tick);
  CK(e, cudaGetLastError());
  e->launches++;
  if (invalidate) e->compact_live = false;
  return MRQ_OK;
}

int ensure_compact(mrq_engine *e) {
  if (e->compact_live || e->G == 0) return MRQ_OK;
  int r = ensure_compact_alloc(e);
  if (r) return r;
  compact_all_kernel<<<nblocks(e->G), 256, 0, e->stream>>>(e->s, e->c, e->pk_base_index, e->pk_base_term, e->gs, e->G, e->R, e->tick_no,
                                                           e->cfg.election_tick, e->cfg.heartbeat_tick);
  CK(e, cudaGetLastError());
  e->launches++;
  e->compact_live = true;
  return MRQ_OK;
}

// Rows [g0, G) become fresh groups (init_state_kernel): one launch, whatever their number.
int init_fresh_groups(mrq_engine *e, uint64_t g0) {
  if (g0 >= e->G) return MRQ_OK;
  const FreshRows f{e->commit_prev, e->pk_base_index, e->pk_base_term, e->c, e->compact_live ? 1 : 0};
  init_state_kernel<<<nblocks(e->G - g0), 256, 0, e->stream>>>(e->s, f, g0, e->G, e->gs, e->cfg.group_base, e->R, e->cfg.self_id,
                                                               e->cfg.seed, e->cfg.election_tick, e->cfg.heartbeat_tick, e->tick_no);
  CK(e, cudaGetLastError());
  e->launches++;
  return MRQ_OK;
}

void fill_tick_args(mrq_engine *e, TickArgs &a) {
  a.s = e->s;
  a.ctr = e->ctr;
  a.G = e->G;
  a.gs = e->gs;
  a.group_base = e->cfg.group_base;
  a.seed = e->cfg.seed;
  a.tick_cur = e->tickbuf + (e->tick_parity & 1u);
  a.tick_next = e->tickbuf + ((e->tick_parity + 1u) & 1u);
  a.election_tick = e->cfg.election_tick;
  a.heartbeat_tick = e->cfg.heartbeat_tick;
  a.world = (e->comm_mode == 1 && e->ipc_attached) ? e->world : 1;
  a.rank = e->rank;
  a.gather_prime = e->gather_prime ? 1u : 0u;
  a.l2_policy = e->l2_policy ? 1u : 0u;
  for (uint32_t p = 0; p < 8; ++p) {
    a.peer_full[p] = e->peer_gather[p];  // [world * G] full indices, then [world * G] low bytes (see TickArgs)
    a.peer_lo[p] = a.peer_full[p] ? reinterpret_cast<uint8_t *>(a.peer_full[p] + (size_t)e->world * e->G) : nullptr;
  }
  a.slow_list = e->slow_list;
  a.slow_count = e->slow_count + (e->slow_parity & 1u);
  a.slow_count_next = e->slow_count + ((e->slow_parity + 1u) & 1u);
  a.changes = e->changes;
  a.change_count = e->change_count;
  a.change_cap = e->change_cap;
}

// n ticks of mode 4 in ONE pair of launches: every slot holds a byte frame (mrq_post_inbox_packed, word_bits 8).
int launch_tick4(mrq_engine *e, const uint32_t *slots, uint32_t n) {
  // compact leaders' timers are phases against the tick number, which must not wrap within the compact representation
  if (n > UINT64_MAX - e->tick_no)
    return fail(e, MRQ_E_INVAL, "tick mode 4: tick number %llu + %u would wrap past 2^64 - 1 (rewind it with mrq_set_tick_count)",
                (unsigned long long)e->tick_no, n);
  int r = ensure_compact(e);
  if (r) return r;
  Tick4ArgsT<CompactOff> A{};
  fill_tick_args(e, A.t);
  A.c = e->c;
  A.base_index = e->pk_base_index;
  A.base_term = e->pk_base_term;
  A.nticks = n;
  A.write_through = e->write_through ? 1u : 0u;
  A.slow_list64 = e->slow_list64;
  auto desc_of = [&](uint32_t slot, bool per_slot_outputs, TickDesc *d) -> int {
    PackedStage &sg = e->pk_stage[slot];
    d->word8 = sg.word8;
    d->prop8 = sg.prop8;
    d->in = e->inbox[slot].view();
    if (per_slot_outputs) {
      if (e->out_slot.size() < e->inbox.size()) e->out_slot.resize(e->inbox.size(), nullptr);
      if (e->delta_slot.size() < e->inbox.size()) e->delta_slot.resize(e->inbox.size(), nullptr);
      int rr;
      if (!e->out_slot[slot] && (rr = dalloc(e, &e->out_slot[slot], e->gs))) return rr;
      if (!e->delta_slot[slot] && (rr = dalloc(e, &e->delta_slot[slot], e->gs))) return rr;
      d->out = e->out_slot[slot];
      d->delta = e->delta_slot[slot];
    } else {
      d->out = e->s.out;
      d->delta = e->delta;
    }
    return MRQ_OK;
  };
  if (n == 1) {
    if ((r = desc_of(slots[0], false, &A.d0))) return r;
    A.descs = nullptr;
    e->last_out = A.d0.out;
    e->last_delta = A.d0.delta;
  } else {
    std::string key((const char *)slots, (size_t)n * sizeof(uint32_t));
    key.append((const char *)&e->stage_gen, sizeof e->stage_gen);
    auto it = e->desc_tables.find(key);
    if (it == e->desc_tables.end()) {  // first use of this slot sequence: build and upload its descriptor table
      if (e->desc_tables.size() >= 64) {  // a host that never repeats a sequence must not grow the cache without bound
        CK(e, cudaStreamSynchronize(e->stream));  // (tables of launches still in flight)
        for (auto &kv : e->desc_tables) cudaFree(kv.second);
        e->desc_tables.clear();
      }
      std::vector<TickDesc> host(n);
      for (uint32_t k = 0; k < n; ++k)
        if ((r = desc_of(slots[k], true, &host[k]))) return r;
      TickDesc *dev = nullptr;
      CK(e, cudaMalloc((void **)&dev, n * sizeof(TickDesc)));
      CK(e, cudaMemcpyAsync(dev, host.data(), n * sizeof(TickDesc), cudaMemcpyHostToDevice, e->stream));
      CK(e, cudaStreamSynchronize(e->stream));  // `host` dies with this scope
      it = e->desc_tables.emplace(key, dev).first;
    }
    A.descs = it->second;
    A.d0 = TickDesc{};
    e->last_out = e->out_slot[slots[n - 1]];
    e->last_delta = e->delta_slot[slots[n - 1]];
  }
  const uint64_t quads = e->gs / 4;
  cudaError_t lst = cudaErrorInvalidValue;
  // Big shards: four groups per thread (128-bit column accesses, a quarter of the instructions per group).  Small shards
  // (a many-GPU job's): one group per thread — the GPU needs warps in flight more than it needs wide accesses.
  const char *gpt_env = getenv("MRQ_T4_GPT");  // development / test knob: force 1 or 4 groups per thread
  const int force_gpt = gpt_env ? atoi(gpt_env) : 0;
  // (one per thread only while the whole shard is resident at once: 7 CTAs of 128 threads per SM)
  const bool one_per_thread = force_gpt == 1 || (force_gpt != 4 && nblocks(e->gs, 128) <= 7u * (unsigned)g_sm_count);
  if (one_per_thread) {
    MRQ_DISPATCH_R(e->R, lst = launch_pdl(tick_fast1_kernel<kR>, nblocks(e->gs, 128), 128, 0, e->stream, A));
  } else {
    MRQ_DISPATCH_R(e->R, lst = launch_pdl(tick_fast4_kernel<kR, 128>, nblocks(quads, 128), 128, 0, e->stream, A));
  }
  CK(e, lst);
  unsigned nslow = (unsigned)g_sm_count * 6u;
  const unsigned nb1 = nblocks(e->G, kTickThreads);
  if (nslow > nb1) nslow = nb1;
  MRQ_DISPATCH_R(e->R, lst = launch_pdl(tick_slow4_kernel<kR>, nslow, kTickThreads, 0, e->stream, A));
  CK(e, lst);
  // host-side bookkeeping only once both launches are in the stream
  e->launches += 2;
  e->tick_parity ^= 1u;
  e->slow_parity ^= 1u;
  if (A.t.world > 1) e->gather_prime = false;
  e->tick_no += n;
  if (n > 1 && e->slot_out_live.size() < e->inbox.size()) e->slot_out_live.resize(e->inbox.size(), false);
  for (uint32_t k = 0; k < n; ++k) {
    PackedStage &sg = e->pk_stage[slots[k]];
    if (!sg.keep8) sg.frame8 = false;
    if (n > 1) e->slot_out_live[slots[k]] = true;
    CK(e, cudaEventRecord(sg.consumed, e->stream));  // only now may the next frame overwrite the staging buffer
  }
  return MRQ_OK;
}

bool slot_has_frame8(mrq_engine *e, uint32_t slot) { return slot < e->pk_stage.size() && e->pk_stage[slot].frame8; }

int launch_tick(mrq_engine *e, const InboxBuf *ib) {
  if (e->G == 0) {
    e->tick_no++;
    return MRQ_OK;
  }
  const size_t slot = ib ? (size_t)(ib - e->inbox.data()) : 0;
  if (e->tick_mode == 4) {
    if (ib && slot_has_frame8(e, (uint32_t)slot)) {
      const uint32_t s1 = (uint32_t)slot;
      int r = launch_tick4(e, &s1, 1);
      if (r) return r;
      if (e->world > 1 && e->comm_mode == 0 && e->comm) {  // per-tick ncclAllGather reads the wide committed column
        if ((r = ensure_wide(e, false))) return r;
        int st = g_nccl.AllGather(e->s.committed, e->gathered, (size_t)e->G, kNcclUint64, e->comm, e->stream);
        if (st != 0) return fail(e, MRQ_E_NCCL, "ncclAllGather failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(st) : "?");
      }
      return MRQ_OK;
    }
    // a wide inbox (or an idle tick) in mode 4: the general kernels work on the wide columns
    int r = ensure_wide(e, true);
    if (r) return r;
  }
  TickArgs a{};
  fill_tick_args(e, a);
  if (ib) a.in = ib->view();
  const unsigned nb = nblocks(e->G, kTickThreads);
  cudaError_t lst = cudaErrorInvalidValue;
  unsigned nlaunch = 0;
  bool flip_slow = false;
  if (e->tick_mode == 3 && ib && slot_has_frame8(e, (uint32_t)slot)) {
    // the tick on the byte form: the kernels read the frame where the copy left it (no unpack pass)
    PackedStage &sg = e->pk_stage[slot];
    Tick8Args a8{a, Inbox8{sg.word8, sg.prop8, e->pk_base_index, e->pk_base_term}};
    MRQ_DISPATCH_R(e->R, lst = launch_pdl(tick_fast8_kernel<kR>, nb, kTickThreads, 0, e->stream, a8));
    CK(e, lst);
    unsigned nslow = (unsigned)g_sm_count * 6u;
    if (nslow > nb) nslow = nb;
    MRQ_DISPATCH_R(e->R, lst = launch_pdl(tick_slow8_kernel<kR>, nslow, kTickThreads, 0, e->stream, a8));
    CK(e, lst);
    nlaunch = 2;
    flip_slow = true;
    if (!sg.keep8) sg.frame8 = false;
    CK(e, cudaEventRecord(sg.consumed, e->stream));  // only now may the next frame overwrite the staging buffer
  } else if (e->tick_mode == 1) {  // single launch, every group through the general path (differential testing)
    MRQ_DISPATCH_R(e->R, lst = launch_pdl(tick_general_kernel<kR>, nb, kTickThreads, 0, e->stream, a));
    CK(e, lst);
    nlaunch = 1;
  } else if (e->tick_mode == 2) {  // single launch: fast tick + in-CTA general path for the stragglers
    MRQ_DISPATCH_R(e->R, lst = launch_pdl(tick_fused_kernel<kR>, nb, kTickThreads, 0, e->stream, a));
    CK(e, lst);
    nlaunch = 1;
  } else {
    MRQ_DISPATCH_R(e->R, lst = launch_pdl(tick_fast_kernel<kR>, nb, kTickThreads, 0, e->stream, a));
    CK(e, lst);
    unsigned nslow = (unsigned)g_sm_count * 6u;
    if (nslow > nb) nslow = nb;
    MRQ_DISPATCH_R(e->R, lst = launch_pdl(tick_slow_kernel<kR>, nslow, kTickThreads, 0, e->stream, a));
    CK(e, lst);
    nlaunch = 2;
    flip_slow = true;
  }
  // the double-buffer parities move only once the launches are in the stream: a failed launch leaves the host's
  // bookkeeping in step with the device
  e->launches += nlaunch;
  e->tick_parity ^= 1u;
  if (flip_slow) e->slow_parity ^= 1u;
  if (a.world > 1) e->gather_prime = false;
  e->last_out = e->s.out;
  e->last_delta = nullptr;
  e->tick_no++;
  if (e->world > 1 && e->comm_mode == 0 && e->comm) {
    int st = g_nccl.AllGather(e->s.committed, e->gathered, (size_t)e->G, kNcclUint64, e->comm, e->stream);
    if (st != 0) return fail(e, MRQ_E_NCCL, "ncclAllGather failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(st) : "?");
  }
  return MRQ_OK;
}

constexpr int kTmaTile = 256;
constexpr int kTmaStages = 4;
constexpr int kQuadThreads = 128;

template <int R>
int launch_quorum_t(mrq_engine *e, const QuorumArgs &a0, int variant, cudaStream_t st, int sm_count) {
  QuorumArgs a = a0;
  uint64_t done = 0;
  if (variant == 1 && a.G >= (uint64_t)kTmaTile) {
    const uint64_t ntiles = a.G / kTmaTile;
    const size_t smem = (size_t)kTmaStages * (R + 2) * kTmaTile * 8 + kTmaStages * 8;
    auto kern = quorum_kernel_tma<R, kTmaTile, kTmaStages>;
    static bool attr_set[64] = {};  // the attribute is per device
    int dev = 0;
    CK(e, cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !attr_set[dev]) {
      CK(e, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      if (dev >= 0 && dev < 64) attr_set[dev] = true;
    }
    int per_sm = (int)((220 * 1024) / smem);
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 8) per_sm = 8;
    uint64_t grid = (uint64_t)sm_count * per_sm;
    if (grid > ntiles) grid = ntiles;
    QuorumArgs t = a;
    t.G = ntiles * kTmaTile;
    CK(e, launch_pdl(kern, (unsigned)grid, kTmaTile, smem, st, t));
    if (e) e->launches++;
    done = t.G;
  }
  if (done < a.G) {  // an LDG form (whole range, or the tail the tiled form left)
    QuorumArgs t = a;
    t.match = a.match + done;
    t.committed = a.committed + done;
    t.term_start = a.term_start + done;
    t.G = a.G - done;
    if (variant == 2) {
      const uint64_t pairs = (t.G + 1) / 2;
      CK(e, launch_pdl(quorum_kernel_ldg<R>, nblocks(pairs), 256, 0, st, t));
    } else {
      const uint64_t quads = (t.G + 3) / 4;
      CK(e, launch_pdl(quorum_kernel_quad<R, kQuadThreads>, nblocks(quads, kQuadThreads), kQuadThreads, 0, st, t));
    }
    if (e) e->launches++;
  }
  return MRQ_OK;
}


int launch_quorum(mrq_engine *e, const QuorumArgs &a, int variant) {
  int rc = MRQ_E_INVAL;
  MRQ_DISPATCH_R(e->R, rc = launch_quorum_t<kR>(e, a, variant, e->stream, g_sm_count));
  return rc;
}

int check_slot(mrq_engine *e, uint32_t slot) {
  if (!e) return MRQ_E_INVAL;
  if (slot >= e->inbox.size()) return fail(e, MRQ_E_INVAL, "inbox slot %u out of range (%zu slots)", slot, e->inbox.size());
  return MRQ_OK;
}

// a wide-form post (or a clear) supersedes a byte frame that was waiting for its tick in this slot (tick mode 3)
void drop_frame8(mrq_engine *e, uint32_t slot) {
  if (slot < e->pk_stage.size()) e->pk_stage[slot].frame8 = false;
}

}  // namespace

extern "C" {

uint32_t mrq_version(uint32_t *sm_arch) {
  if (sm_arch) *sm_arch = 90;
  return MRQ_ABI_VERSION;
}

void mrq_config_default(mrq_config *cfg) {
  if (!cfg) return;
  memset(cfg, 0, sizeof *cfg);
  cfg->abi_version = MRQ_ABI_VERSION;
  cfg->n_replicas = 3;
  cfg->election_tick = 10;  // reference raft.go:154
  cfg->heartbeat_tick = 1;  // reference raft.go:155
  cfg->inbox_slots = 2;
}

const char *mrq_last_error(const mrq_engine *e) { return e ? e->err.c_str() : g_create_error.c_str(); }

int mrq_create(const mrq_config *cfg, mrq_engine **out) {
  if (!cfg || !out) return fail(nullptr, MRQ_E_INVAL, "mrq_create: null argument");
  *out = nullptr;
  if (cfg->abi_version != MRQ_ABI_VERSION) return fail(nullptr, MRQ_E_INVAL, "abi_version %u != %u", cfg->abi_version, MRQ_ABI_VERSION);
  if (cfg->n_replicas < 1 || cfg->n_replicas > MRQ_MAX_REPLICAS)
    return fail(nullptr, MRQ_E_INVAL, "n_replicas %u outside 1..%u", cfg->n_replicas, MRQ_MAX_REPLICAS);
  if (cfg->self_id > cfg->n_replicas) return fail(nullptr, MRQ_E_INVAL, "self_id %u > n_replicas", cfg->self_id);
  if (cfg->election_tick < 1 || cfg->election_tick > 2047) return fail(nullptr, MRQ_E_INVAL, "election_tick outside 1..2047");
  if (cfg->heartbeat_tick < 1 || cfg->heartbeat_tick > 255) return fail(nullptr, MRQ_E_INVAL, "heartbeat_tick outside 1..255");
  if (cfg->n_groups >= (1ull << 32)) return fail(nullptr, MRQ_E_INVAL, "n_groups must be below 2^32 per engine (shard across engines)");
  int ndev = 0;
  cudaError_t st = cudaGetDeviceCount(&ndev);
  if (st != cudaSuccess || ndev == 0)
    return fail(nullptr, MRQ_E_NODEVICE, "no CUDA device (%s); this engine has no CPU fallback",
                st == cudaSuccess ? "device count 0" : cudaGetErrorString(st));
  if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, MRQ_E_INVAL, "device %d outside 0..%d", cfg->device, ndev - 1);
  mrq_engine *e = new (std::nothrow) mrq_engine();
  if (!e) return fail(nullptr, MRQ_E_NOMEM, "out of host memory");
  e->cfg = *cfg;
  e->G = cfg->n_groups;
  e->gs = ((e->G + 127) / 128) * 128;  // column stride: a multiple of the tick CTA size (kTickThreads)
  if (e->gs == 0) e->gs = 128;
  e->R = cfg->n_replicas;
  e->device = cfg->device;
  int rc = MRQ_OK;
  auto body = [&]() -> int {
    CK(e, cudaSetDevice(e->device));
    cudaDeviceProp prop;
    CK(e, cudaGetDeviceProperties(&prop, e->device));
    if (prop.major != 9 || prop.minor != 0)
      return fail(e, MRQ_E_NODEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", e->device, prop.major, prop.minor);
    g_sm_count = prop.multiProcessorCount;
    // Experiment knob (off unless set): the tick kernel's evict-last hints may be confined to the persisting-L2
    // carve-out; MRQ_L2_PERSIST_MB raises the device limit (capped at the device's persistingL2CacheMaxSize).
    if (const char *mb = getenv("MRQ_L2_PERSIST_MB")) {
      size_t want = (size_t)strtoull(mb, nullptr, 10) << 20;
      if (want > (size_t)prop.persistingL2CacheMaxSize) want = (size_t)prop.persistingL2CacheMaxSize;
      CK(e, cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want));
    }
    if (cfg->stream) {
      e->stream = (cudaStream_t)cfg->stream;
    } else {
      CK(e, cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
      e->own_stream = true;
    }
    CK(e, cudaEventCreate(&e->ev0));
    CK(e, cudaEventCreate(&e->ev1));
    const size_t gs = e->gs;
    int r;
    if ((r = dalloc(e, &e->s.term, gs))) return r;
    if ((r = dalloc(e, &e->s.meta, gs))) return r;
    if ((r = dalloc(e, &e->s.last_index, gs))) return r;
    if ((r = dalloc(e, &e->s.last_term, gs))) return r;
    if ((r = dalloc(e, &e->s.committed, gs))) return r;
    if ((r = dalloc(e, &e->s.term_start, gs))) return r;
    if ((r = dalloc(e, &e->s.match, gs * e->R))) return r;
    if ((r = dalloc(e, &e->s.out, gs))) return r;
    if ((r = dalloc(e, &e->ctr, kCtrShards))) return r;
    if ((r = dalloc(e, &e->commit_prev, gs))) return r;
    if ((r = dalloc(e, &e->delta, gs))) return r;
    if ((r = dalloc(e, &e->gathered, gs))) return r;
    if ((r = dalloc(e, &e->pk_base_index, gs))) return r;
    if ((r = dalloc(e, &e->pk_base_term, gs))) return r;
    if ((r = dalloc(e, &e->slow_list, gs))) return r;
    if ((r = dalloc(e, &e->slow_count, 2))) return r;
    if ((r = dalloc(e, &e->tickbuf, 2))) return r;
    uint32_t nslots = cfg->inbox_slots ? cfg->inbox_slots : 2;
    e->inbox.resize(nslots);
    for (auto &ib : e->inbox) {
      if ((r = dalloc(e, &ib.type, gs * e->R))) return r;
      if ((r = dalloc(e, &ib.term, gs * e->R))) return r;
      if ((r = dalloc(e, &ib.index, gs * e->R))) return r;
      if ((r = dalloc(e, &ib.logterm, gs * e->R))) return r;
      if ((r = dalloc(e, &ib.commit, gs * e->R))) return r;
      if ((r = dalloc(e, &ib.prop, gs))) return r;
    }
    if ((r = init_fresh_groups(e, 0))) return r;
    CK(e, cudaStreamSynchronize(e->stream));
    return MRQ_OK;
  };
  rc = body();
  if (rc != MRQ_OK) {
    g_create_error = e->err;
    mrq_destroy(e);
    return rc;
  }
  *out = e;
  return MRQ_OK;
}

void mrq_destroy(mrq_engine *e) {
  if (!e) return;
  cudaSetDevice(e->device);
  if (e->stream) cudaStreamSynchronize(e->stream);
  if (e->drain_done) cudaEventDestroy(e->drain_done);
  if (e->copy_stream) {
    cudaStreamSynchronize(e->copy_stream);
    cudaStreamDestroy(e->copy_stream);
  }
  for (auto &sg : e->pk_stage) {
    if (sg.buf) cudaFree(sg.buf);
    if (sg.copied) cudaEventDestroy(sg.copied);
    if (sg.consumed) cudaEventDestroy(sg.consumed);
  }
  if (e->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(e->comm);
  if (e->ipc_attached) {
    for (uint32_t p = 0; p < e->world; ++p)
      if (p != e->rank && e->peer_gather[p]) cudaIpcCloseMemHandle(e->peer_gather[p]);
  }
  void *ptrs[] = {e->s.term, e->s.meta, e->s.last_index, e->s.last_term, e->s.committed, e->s.term_start, e->s.match,
                  e->s.out, e->ctr, e->commit_prev, e->delta, e->gathered, e->scratch, e->pk_base_index, e->pk_base_term, e->slow_list, e->slow_count, e->tickbuf};
  for (auto &kv : e->graphs) cudaGraphExecDestroy(kv.second);
  for (auto &kv : e->desc_tables) cudaFree(kv.second);
  if (e->changes) cudaFree(e->changes);
  if (e->change_count) cudaFree(e->change_count);
  {
    void *cp[] = {e->c.flag, e->c.commit, e->c.win, e->c.gate, e->c.iblo, e->c.match, e->c.ibase, e->c.clk, e->slow_list64};
    for (void *p : cp)
      if (p) cudaFree(p);
    for (void *p : e->out_slot)
      if (p) cudaFree(p);
    for (void *p : e->delta_slot)
      if (p) cudaFree(p);
  }
  for (void *p : ptrs)
    if (p) cudaFree(p);
  for (auto &ib : e->inbox) {
    void *q[] = {ib.type, ib.term, ib.index, ib.logterm, ib.commit, ib.prop};
    for (void *p : q)
      if (p) cudaFree(p);
  }
  if (e->pinned) cudaFreeHost(e->pinned);
  if (e->ev0) cudaEventDestroy(e->ev0);
  if (e->ev1) cudaEventDestroy(e->ev1);
  if (e->own_stream && e->stream) cudaStreamDestroy(e->stream);
  delete e;
}

uint64_t mrq_tick_count(const mrq_engine *e) { return e ? e->tick_no : 0; }
int mrq_set_tick_count(mrq_engine *e, uint64_t t) {
  if (!e) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  // compact leaders keep their timers as phases against the tick number: bring them into meta before it moves
  int r = ensure_wide(e, true);
  if (r) return r;
  e->tick_no = t;
  // also normalise the double-buffer parities, so that a slot sequence replayed after a rewind hits the
  // same captured graph (mrq_tick_many keys its graphs by parity)
  e->tick_parity = 0;
  e->slow_parity = 0;
  CK(e, cudaMemcpyAsync(e->tickbuf, &e->tick_no, 8, cudaMemcpyHostToDevice, e->stream));
  CK(e, cudaMemsetAsync(e->slow_count, 0, 2 * sizeof(unsigned), e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}
void *mrq_stream(mrq_engine *e) { return e ? (void *)e->stream : nullptr; }

void *mrq_device_ptr(mrq_engine *e, int which) {
  if (!e) return nullptr;
  switch (which) {
    case MRQ_PTR_TERM: return e->s.term;
    case MRQ_PTR_META: return e->s.meta;
    case MRQ_PTR_LAST_INDEX: return e->s.last_index;
    case MRQ_PTR_LAST_TERM: return e->s.last_term;
    case MRQ_PTR_COMMITTED: return e->s.committed;
    case MRQ_PTR_TERM_START: return e->s.term_start;
    case MRQ_PTR_MATCH: return e->s.match;
    case MRQ_PTR_OUT: return e->s.out;
    case MRQ_PTR_GATHERED: return e->gathered;
    default: return nullptr;
  }
}

uint64_t mrq_group_stride(const mrq_engine *e) { return e ? e->gs : 0; }

}  // extern "C"

namespace {
// A device buffer sized by the group stride: `rows` rows of gs elements of `elem` bytes.  `keep`: the rows of the groups
// that survive a resize are copied into its replacement; every other buffer starts over zeroed, as mrq_create leaves it.
struct StrideBuf {
  void **at;
  size_t elem, rows;
  bool keep;
};
template <typename T>
StrideBuf stride_buf(T *&p, size_t rows, bool keep) {
  return StrideBuf{reinterpret_cast<void **>(&p), sizeof(T), rows, keep};
}

// Every buffer of the engine whose size follows the stride (scratch and staging are sized per call and follow alone).
std::vector<StrideBuf> stride_bufs(mrq_engine *e) {
  const size_t R = e->R;
  std::vector<StrideBuf> v = {
      stride_buf(e->s.term, 1, true),        stride_buf(e->s.meta, 1, true),          stride_buf(e->s.last_index, 1, true),
      stride_buf(e->s.last_term, 1, true),   stride_buf(e->s.committed, 1, true),     stride_buf(e->s.term_start, 1, true),
      stride_buf(e->s.match, R, true),       stride_buf(e->commit_prev, 1, true),     stride_buf(e->pk_base_index, 1, true),
      stride_buf(e->pk_base_term, 1, true),  stride_buf(e->s.out, 1, false),          stride_buf(e->delta, 1, false),
      stride_buf(e->gathered, 1, false),     stride_buf(e->slow_list, 1, false)};
  if (e->compact_alloc) {
    for (StrideBuf b : {stride_buf(e->c.flag, 1, true), stride_buf(e->c.commit, 1, true), stride_buf(e->c.win, 1, true),
                        stride_buf(e->c.gate, 1, true), stride_buf(e->c.iblo, 1, true), stride_buf(e->c.match, R, true),
                        stride_buf(e->c.ibase, 1, true), stride_buf(e->c.clk, 1, true), stride_buf(e->slow_list64, 1, false)})
      v.push_back(b);
  }
  for (auto &ib : e->inbox)
    for (StrideBuf b : {stride_buf(ib.type, R, false), stride_buf(ib.term, R, false), stride_buf(ib.index, R, false),
                        stride_buf(ib.logterm, R, false), stride_buf(ib.commit, R, false), stride_buf(ib.prop, 1, false)})
      v.push_back(b);
  for (auto &p : e->out_slot)
    if (p) v.push_back(stride_buf(p, 1, false));
  for (auto &p : e->delta_slot)
    if (p) v.push_back(stride_buf(p, 1, false));
  return v;
}

// Move every stride-sized buffer to stride `gs`, keeping the rows of the first `keep` groups.  All new buffers are
// allocated before any old one is freed, and the copies run on the device: a failure frees the new buffers only and
// leaves the engine as it was.
int restride(mrq_engine *e, uint64_t gs, uint64_t keep) {
  const std::vector<StrideBuf> bufs = stride_bufs(e);
  std::vector<void *> fresh(bufs.size(), nullptr);
  auto drop_fresh = [&]() {
    cudaStreamSynchronize(e->stream);
    for (void *p : fresh)
      if (p) cudaFree(p);
  };
  for (size_t k = 0; k < bufs.size(); ++k) {
    const size_t bytes = bufs[k].elem * bufs[k].rows * gs;
    if (cudaMalloc(&fresh[k], bytes) != cudaSuccess) {
      cudaGetLastError();
      fresh[k] = nullptr;
      drop_fresh();
      return fail(e, MRQ_E_NOMEM, "mrq_resize_groups: cannot allocate %zu bytes of device memory (the engine is unchanged)", bytes);
    }
  }
  for (size_t k = 0; k < bufs.size(); ++k) {
    const StrideBuf &b = bufs[k];
    cudaError_t st = cudaMemsetAsync(fresh[k], 0, b.elem * b.rows * gs, e->stream);
    if (st == cudaSuccess && b.keep && keep)
      st = cudaMemcpy2DAsync(fresh[k], gs * b.elem, *b.at, e->gs * b.elem, keep * b.elem, b.rows, cudaMemcpyDeviceToDevice, e->stream);
    if (st != cudaSuccess) {
      drop_fresh();
      return fail(e, MRQ_E_CUDA, "mrq_resize_groups: device copy failed: %s", cudaGetErrorString(st));
    }
  }
  const cudaError_t st = cudaStreamSynchronize(e->stream);
  if (st != cudaSuccess) {
    drop_fresh();
    return fail(e, MRQ_E_CUDA, "mrq_resize_groups: device copy failed: %s", cudaGetErrorString(st));
  }
  for (size_t k = 0; k < bufs.size(); ++k) {
    cudaFree(*bufs[k].at);
    *bufs[k].at = fresh[k];
  }
  e->gs = gs;
  // mode-4 descriptor tables hold output pointers, and staging buffers are laid out by the stride
  for (auto &kv : e->desc_tables) cudaFree(kv.second);
  e->desc_tables.clear();
  e->stage_gen++;
  return MRQ_OK;
}
}  // namespace

extern "C" {

int mrq_resize_groups(mrq_engine *e, uint64_t n_groups) {
  if (!e) return MRQ_E_INVAL;
  if (n_groups >= (1ull << 32)) return fail(e, MRQ_E_INVAL, "n_groups must be below 2^32 per engine (shard across engines)");
  if (e->comm || e->ipc_attached || e->gather_shared)
    return fail(e, MRQ_E_STATE, "mrq_resize_groups: the gather is shared with peers that own the same G (resize every rank's engine "
                                "by recreating it)");
  if (n_groups == e->G) return MRQ_OK;
  CK(e, cudaSetDevice(e->device));
  if (e->copy_stream) CK(e, cudaStreamSynchronize(e->copy_stream));  // a packed-inbox copy may still be filling a staging buffer
  CK(e, cudaStreamSynchronize(e->stream));
  const uint64_t old = e->G, keep = old < n_groups ? old : n_groups;
  uint64_t gs = ((n_groups + 127) / 128) * 128;  // as mrq_create: a multiple of the tick CTA size, at least one CTA
  if (gs == 0) gs = 128;
  int r;
  if (gs != e->gs) {
    if ((r = restride(e, gs, keep))) return r;
  } else {  // the buffers stay: clear what mrq_create leaves zeroed and the groups do not own
    CK(e, cudaMemsetAsync(e->s.out, 0, e->gs * sizeof(uint32_t), e->stream));
    CK(e, cudaMemsetAsync(e->delta, 0, e->gs, e->stream));
    for (auto &ib : e->inbox) {  // (mrq_clear_inbox)
      CK(e, cudaMemsetAsync(ib.type, 0, e->gs * e->R, e->stream));
      CK(e, cudaMemsetAsync(ib.prop, 0, e->gs * sizeof(uint32_t), e->stream));
    }
  }
  // Captured graphs hold G and the buffer addresses by value.  Waiting frames and the outputs of earlier ticks describe
  // the old group count: every slot starts over empty, as after mrq_create.
  for (auto &kv : e->graphs) cudaGraphExecDestroy(kv.second);
  e->graphs.clear();
  for (auto &sg : e->pk_stage) sg.frame8 = sg.keep8 = false;
  e->slot_out_live.assign(e->slot_out_live.size(), false);
  e->last_out = nullptr;
  e->last_delta = nullptr;
  e->G = n_groups;
  e->cfg.n_groups = n_groups;
  // While G == 0 no kernel runs to advance the device's tick number (TickArgs::tick_cur): bring it to the host's count,
  // which keys the groups' timeout draws from their first tick on.
  CK(e, cudaMemcpyAsync(e->tickbuf + (e->tick_parity & 1u), &e->tick_no, sizeof e->tick_no, cudaMemcpyHostToDevice, e->stream));
  if ((r = init_fresh_groups(e, old))) return r;
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

void *mrq_alloc_pinned(size_t bytes) {
  void *p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) return nullptr;
  return p;
}
void mrq_free_pinned(void *p) {
  if (p) cudaFreeHost(p);
}

// ---- state import / export ------------------------------------------------------------------------------
int mrq_export_state(mrq_engine *e, mrq_state *o) {
  if (!e || !o) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  const size_t gs = e->gs, G = e->G;
  if (G == 0) return MRQ_OK;
  {
    int rw = ensure_wide(e, false);
    if (rw) return rw;
  }
  // unpack meta into scratch columns: role, lead, self (u8), vote (u64), el, hb, rto (u16), votes (u8 [R][gs])
  const size_t need = gs * (3 + 8 + 6) + gs * e->R + 64;
  int r = ensure_scratch(e, need);
  if (r) return r;
  uint8_t *base = (uint8_t *)e->scratch;
  uint64_t *d_vote = (uint64_t *)base;
  uint16_t *d_el = (uint16_t *)(base + gs * 8), *d_hb = d_el + gs, *d_rto = d_hb + gs;
  uint8_t *d_role = base + gs * 14, *d_lead = d_role + gs, *d_self = d_lead + gs, *d_votes = d_self + gs;
  unpack_meta_kernel<<<nblocks(G), 256, 0, e->stream>>>(e->s.meta, G, d_role, d_lead, d_self, d_vote, d_el, d_hb, d_rto, d_votes, gs, e->R);
  CK(e, cudaGetLastError());
  e->launches++;
  if ((r = copy_out(e, o->term, e->s.term, 8, 1))) return r;
  if ((r = copy_out(e, o->vote, d_vote, 8, 1))) return r;
  if ((r = copy_out(e, o->committed, e->s.committed, 8, 1))) return r;
  if ((r = copy_out(e, o->last_index, e->s.last_index, 8, 1))) return r;
  if ((r = copy_out(e, o->last_term, e->s.last_term, 8, 1))) return r;
  if ((r = copy_out(e, o->term_start, e->s.term_start, 8, 1))) return r;
  if ((r = copy_out(e, o->match, e->s.match, 8, e->R))) return r;
  if ((r = copy_out(e, o->role, d_role, 1, 1))) return r;
  if ((r = copy_out(e, o->lead, d_lead, 1, 1))) return r;
  if ((r = copy_out(e, o->self_id, d_self, 1, 1))) return r;
  if ((r = copy_out(e, o->votes, d_votes, 1, e->R))) return r;
  if ((r = copy_out(e, o->election_elapsed, d_el, 2, 1))) return r;
  if ((r = copy_out(e, o->heartbeat_elapsed, d_hb, 2, 1))) return r;
  if ((r = copy_out(e, o->randomized_timeout, d_rto, 2, 1))) return r;
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

int mrq_import_state(mrq_engine *e, const mrq_state *in) {
  if (!e || !in) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  const size_t gs = e->gs, G = e->G;
  if (G == 0) return MRQ_OK;
  int r;
  if ((r = ensure_wide(e, true))) return r;  // partial imports overwrite some wide columns: the rest must be exact first
  auto put = [&](void *dev, const void *host, size_t elem, size_t rows) -> int {
    if (!host) return MRQ_OK;
    return copy_in(e, dev, host, elem, rows);
  };
  if ((r = put(e->s.term, in->term, 8, 1))) return r;
  if ((r = put(e->s.committed, in->committed, 8, 1))) return r;
  if ((r = put(e->s.last_index, in->last_index, 8, 1))) return r;
  if ((r = put(e->s.last_term, in->last_term, 8, 1))) return r;
  if ((r = put(e->s.term_start, in->term_start, 8, 1))) return r;
  if ((r = put(e->s.match, in->match, 8, e->R))) return r;
  const bool any_meta = in->role || in->lead || in->self_id || in->vote || in->votes || in->election_elapsed ||
                        in->heartbeat_elapsed || in->randomized_timeout;
  if (any_meta) {
    const size_t need = gs * (3 + 8 + 6) + gs * e->R + 64;
    if ((r = ensure_scratch(e, need))) return r;
    uint8_t *base = (uint8_t *)e->scratch;
    uint64_t *d_vote = (uint64_t *)base;
    uint16_t *d_el = (uint16_t *)(base + gs * 8), *d_hb = d_el + gs, *d_rto = d_hb + gs;
    uint8_t *d_role = base + gs * 14, *d_lead = d_role + gs, *d_self = d_lead + gs, *d_votes = d_self + gs;
    if ((r = put(d_vote, in->vote, 8, 1))) return r;
    if ((r = put(d_el, in->election_elapsed, 2, 1))) return r;
    if ((r = put(d_hb, in->heartbeat_elapsed, 2, 1))) return r;
    if ((r = put(d_rto, in->randomized_timeout, 2, 1))) return r;
    if ((r = put(d_role, in->role, 1, 1))) return r;
    if ((r = put(d_lead, in->lead, 1, 1))) return r;
    if ((r = put(d_self, in->self_id, 1, 1))) return r;
    if ((r = put(d_votes, in->votes, 1, e->R))) return r;
    pack_meta_kernel<<<nblocks(G), 256, 0, e->stream>>>(
        e->s.meta, G, in->role ? d_role : nullptr, in->lead ? d_lead : nullptr, in->self_id ? d_self : nullptr,
        in->vote ? d_vote : nullptr, in->election_elapsed ? d_el : nullptr, in->heartbeat_elapsed ? d_hb : nullptr,
        in->randomized_timeout ? d_rto : nullptr, in->votes ? d_votes : nullptr, gs, e->R);
    CK(e, cudaGetLastError());
    e->launches++;
  }
  fix_strict_kernel<<<nblocks(G), 256, 0, e->stream>>>(e->s, G, gs, e->R);
  CK(e, cudaGetLastError());
  e->launches++;
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

// ---- state of a list of groups ------------------------------------------------------------------------------
namespace {

int ensure_pinned(mrq_engine *e, size_t bytes) {
  if (bytes <= e->pinned_bytes) return MRQ_OK;
  if (e->pinned) {
    CK(e, cudaStreamSynchronize(e->stream));
    CK(e, cudaFreeHost(e->pinned));
    e->pinned = nullptr;
    e->pinned_bytes = 0;
  }
  const size_t want = bytes < (1u << 20) ? (1u << 20) : bytes;
  if (cudaHostAlloc(&e->pinned, want, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    e->pinned = nullptr;
    return fail(e, MRQ_E_NOMEM, "cannot allocate %zu bytes of page-locked staging", want);
  }
  e->pinned_bytes = want;
  return MRQ_OK;
}

// The columns of an n-row mrq_state, in GroupRows order, laid out in one staging block behind the n group ids: the
// block goes to / comes from the device in one copy, and the device pointers of the columns that are not NULL make
// the kernel's GroupRows (NULL columns get no room and stay NULL there).
struct RowsLayout {
  static constexpr int kCols = 14;
  void *host[kCols];
  size_t off[kCols], bytes[kCols];
  size_t cols_begin, total;
  RowsLayout(const mrq_state *st, uint64_t n, uint32_t R) {
    void *const h[kCols] = {st->term,  st->vote,    st->committed, st->last_index, st->last_term,        st->term_start,        st->match,
                            st->role,  st->lead,    st->self_id,   st->votes,      st->election_elapsed, st->heartbeat_elapsed, st->randomized_timeout};
    static const size_t elem[kCols] = {8, 8, 8, 8, 8, 8, 8, 1, 1, 1, 1, 2, 2, 2};
    static const bool per_replica[kCols] = {false, false, false, false, false, false, true, false, false, false, true, false, false, false};
    size_t at = ((n * 8 + 15) / 16) * 16;
    cols_begin = at;
    for (int k = 0; k < kCols; ++k) {
      host[k] = h[k];
      bytes[k] = h[k] ? elem[k] * n * (per_replica[k] ? R : 1u) : 0;
      off[k] = at;
      at += ((bytes[k] + 15) / 16) * 16;
    }
    total = at;
  }
  GroupRows rows(uint8_t *dev) const {
    auto p = [&](int k) -> void * { return host[k] ? dev + off[k] : nullptr; };
    return GroupRows{(uint64_t *)p(0), (uint64_t *)p(1), (uint64_t *)p(2), (uint64_t *)p(3), (uint64_t *)p(4),
                     (uint64_t *)p(5), (uint64_t *)p(6), (uint8_t *)p(7),  (uint8_t *)p(8),  (uint8_t *)p(9),
                     (uint8_t *)p(10), (uint16_t *)p(11), (uint16_t *)p(12), (uint16_t *)p(13)};
  }
};

// Shared argument checks of the group-list calls.  MRQ_OK with *skip set: nothing to do (n == 0, or G == 0).
int check_group_list(mrq_engine *e, const uint64_t *groups, uint64_t n, bool unique, bool *skip) {
  *skip = true;
  if (n == 0) return MRQ_OK;
  if (!groups) return fail(e, MRQ_E_INVAL, "null group list with n = %llu", (unsigned long long)n);
  if (e->G == 0) return MRQ_OK;
  for (uint64_t k = 0; k < n; ++k)
    if (groups[k] >= e->G)
      return fail(e, MRQ_E_INVAL, "group %llu (list entry %llu) out of range: G = %llu", (unsigned long long)groups[k], (unsigned long long)k,
                  (unsigned long long)e->G);
  if (unique) {  // one thread per listed group writes that group: a duplicate would race with itself
    std::vector<uint64_t> sorted(groups, groups + n);
    std::sort(sorted.begin(), sorted.end());
    const auto d = std::adjacent_find(sorted.begin(), sorted.end());
    if (d != sorted.end()) return fail(e, MRQ_E_INVAL, "group %llu is listed twice", (unsigned long long)*d);
  }
  *skip = false;
  return MRQ_OK;
}

}  // namespace

int mrq_export_groups(mrq_engine *e, const uint64_t *groups, uint64_t n, mrq_state *out) {
  if (!e || !out) return MRQ_E_INVAL;
  bool skip;
  int r = check_group_list(e, groups, n, false, &skip);
  if (r || skip) return r;
  CK(e, cudaSetDevice(e->device));
  const RowsLayout L(out, n, e->R);
  if ((r = ensure_scratch(e, L.total)) || (r = ensure_pinned(e, L.total))) return r;
  uint8_t *dev = (uint8_t *)e->scratch, *pin = (uint8_t *)e->pinned;
  memcpy(pin, groups, n * 8);
  CK(e, cudaMemcpyAsync(dev, pin, n * 8, cudaMemcpyHostToDevice, e->stream));
  const bool compact = e->compact_live;
  export_groups_kernel<<<nblocks(n), 256, 0, e->stream>>>(e->s, e->c, compact ? 1 : 0, e->gs, e->R, (const uint64_t *)dev, n, e->tick_no,
                                                          e->cfg.election_tick, e->cfg.heartbeat_tick, L.rows(dev));
  CK(e, cudaGetLastError());
  e->launches++;
  if (L.total > L.cols_begin)
    CK(e, cudaMemcpyAsync(pin + L.cols_begin, dev + L.cols_begin, L.total - L.cols_begin, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  for (int k = 0; k < RowsLayout::kCols; ++k)
    if (L.host[k]) memcpy(L.host[k], pin + L.off[k], L.bytes[k]);
  return MRQ_OK;
}

int mrq_import_groups(mrq_engine *e, const uint64_t *groups, uint64_t n, const mrq_state *in) {
  if (!e || !in) return MRQ_E_INVAL;
  bool skip;
  int r = check_group_list(e, groups, n, true, &skip);
  if (r || skip) return r;
  CK(e, cudaSetDevice(e->device));
  const RowsLayout L(in, n, e->R);
  if ((r = ensure_scratch(e, L.total)) || (r = ensure_pinned(e, L.total))) return r;
  uint8_t *dev = (uint8_t *)e->scratch, *pin = (uint8_t *)e->pinned;
  memcpy(pin, groups, n * 8);
  for (int k = 0; k < RowsLayout::kCols; ++k)
    if (L.host[k]) memcpy(pin + L.off[k], L.host[k], L.bytes[k]);
  CK(e, cudaMemcpyAsync(dev, pin, L.total, cudaMemcpyHostToDevice, e->stream));
  // With the compact state live the kernel materialises and re-compacts exactly the listed groups; every other group
  // keeps its compact copy, so the next mode-4 launch needs no compact_all_kernel.
  const bool compact = e->compact_live;
  import_groups_kernel<<<nblocks(n), 256, 0, e->stream>>>(e->s, e->c, compact ? 1 : 0, e->pk_base_index, e->pk_base_term, e->gs, e->R,
                                                          (const uint64_t *)dev, n, e->tick_no, e->cfg.election_tick,
                                                          e->cfg.heartbeat_tick, L.rows(dev));
  CK(e, cudaGetLastError());
  e->launches++;
  // The fused gather stores a group's full index only when its high bits move during a tick: an imported index has to
  // be republished in full, or the peers would stitch the old high bits onto its new low byte.
  if (in->committed && e->comm_mode == 1) e->gather_prime = true;
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

int mrq_export_next(mrq_engine *e, uint64_t *next_out) {
  if (!e || !next_out) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  if (e->G == 0) return MRQ_OK;
  int r = ensure_wide(e, false);
  if (r) return r;
  if ((r = ensure_scratch(e, e->G * e->R * 8))) return r;
  export_next_kernel<<<nblocks(e->G), 256, 0, e->stream>>>(e->s.match, e->s.term_start, (uint64_t *)e->scratch, e->G, e->gs, e->R);
  CK(e, cudaGetLastError());
  e->launches++;
  CK(e, cudaMemcpyAsync(next_out, e->scratch, e->G * e->R * 8, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

// ---- inbox ---------------------------------------------------------------------------------------------------
int mrq_clear_inbox(mrq_engine *e, uint32_t slot) {
  int r = check_slot(e, slot);
  if (r) return r;
  drop_frame8(e, slot);
  CK(e, cudaSetDevice(e->device));
  InboxBuf &ib = e->inbox[slot];
  CK(e, cudaMemsetAsync(ib.type, 0, e->gs * e->R, e->stream));
  CK(e, cudaMemsetAsync(ib.prop, 0, e->gs * 4, e->stream));
  return MRQ_OK;
}

int mrq_post_inbox_dense(mrq_engine *e, uint32_t slot, const mrq_inbox *in) {
  int r = check_slot(e, slot);
  if (r) return r;
  drop_frame8(e, slot);
  if (!in) return fail(e, MRQ_E_INVAL, "null inbox");
  CK(e, cudaSetDevice(e->device));
  if (e->G == 0) return MRQ_OK;
  InboxBuf &ib = e->inbox[slot];
  if ((r = copy_in(e, ib.type, in->type, 1, e->R))) return r;
  if ((r = copy_in(e, ib.term, in->term, 8, e->R))) return r;
  if ((r = copy_in(e, ib.index, in->index, 8, e->R))) return r;
  if ((r = copy_in(e, ib.logterm, in->logterm, 8, e->R))) return r;
  if ((r = copy_in(e, ib.commit, in->commit, 8, e->R))) return r;
  if ((r = copy_in(e, ib.prop, in->prop_count, 4, 1))) return r;
  return MRQ_OK;
}

int mrq_post_inbox_delta(mrq_engine *e, uint32_t slot, const mrq_msg *msgs, size_t n, int accumulate) {
  int r = check_slot(e, slot);
  if (r) return r;
  drop_frame8(e, slot);
  CK(e, cudaSetDevice(e->device));
  if (!accumulate && (r = mrq_clear_inbox(e, slot))) return r;
  if (n == 0) return MRQ_OK;
  if (!msgs) return fail(e, MRQ_E_INVAL, "null message list");
  // Several messages for one (from, group) slot: the LAST one in the list wins (include/mrq.h).  The scatter kernel
  // runs one unordered thread per message, so earlier duplicates are dropped here, on the host.
  std::vector<mrq_msg> uniq;
  {
    std::unordered_set<uint64_t> seen;
    seen.reserve(n * 2);
    bool dup = false;
    for (size_t k = n; k-- > 0;)
      if (!seen.insert(msgs[k].group * 16u + msgs[k].from).second) {
        dup = true;
        break;
      }
    if (dup) {
      seen.clear();
      uniq.reserve(n);
      for (size_t k = n; k-- > 0;)
        if (seen.insert(msgs[k].group * 16u + msgs[k].from).second) uniq.push_back(msgs[k]);
      msgs = uniq.data();
      n = uniq.size();
    }
  }
  if ((r = ensure_scratch(e, n * sizeof(mrq_msg)))) return r;
  CK(e, cudaMemcpyAsync(e->scratch, msgs, n * sizeof(mrq_msg), cudaMemcpyHostToDevice, e->stream));
  scatter_msgs_kernel<<<nblocks(n), 256, 0, e->stream>>>(e->inbox[slot].view(), e->gs, e->G, e->R, (const MsgRec *)e->scratch, n);
  CK(e, cudaGetLastError());
  e->launches++;
  // the staging buffer is reused by the next sparse post: the copy above must have consumed `msgs`
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

int mrq_post_inbox_packed(mrq_engine *e, uint32_t slot, const mrq_inbox_packed *in) {
  int r = check_slot(e, slot);
  if (r) return r;
  drop_frame8(e, slot);
  if (!in || !in->word) return fail(e, MRQ_E_INVAL, "null packed inbox");
  CK(e, cudaSetDevice(e->device));
  if (e->G == 0) return MRQ_OK;
  const uint32_t bits = in->word_bits ? in->word_bits : 32u;
  if (bits != 8u && bits != 16u && bits != 32u) return fail(e, MRQ_E_INVAL, "word_bits must be 8, 16 or 32");
  if (in->n_wide && !in->wide) return fail(e, MRQ_E_INVAL, "n_wide > 0 but wide == NULL");
  const size_t wsz = bits / 8;
  const size_t rows = bits == 8u ? e->R - 1u : e->R;  // the byte form leaves each group's own sender row out
  const size_t wbytes = ((e->gs * rows * wsz + 255) / 256) * 256, pbytes = ((e->gs + 255) / 256) * 256;
  const size_t xbytes = in->n_wide * sizeof(mrq_msg);
  // The copy runs on its own stream into a per-slot staging buffer, so the H2D of the NEXT tick's inbox
  // overlaps this tick's kernels and drain; events order copy -> unpack (main stream) -> reuse of the stage.
  if (e->pk_stage.size() < e->inbox.size()) e->pk_stage.resize(e->inbox.size());
  PackedStage &sg = e->pk_stage[slot];
  if (!e->copy_stream) CK(e, cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
  if (!sg.copied) {
    CK(e, cudaEventCreateWithFlags(&sg.copied, cudaEventDisableTiming));
    CK(e, cudaEventCreateWithFlags(&sg.consumed, cudaEventDisableTiming));
  }
  const size_t need = wbytes + pbytes + xbytes + 256;
  if (need > sg.bytes) {
    CK(e, cudaStreamSynchronize(e->stream));
    CK(e, cudaStreamSynchronize(e->copy_stream));
    if (sg.buf) CK(e, cudaFree(sg.buf));
    sg.buf = nullptr;
    sg.bytes = 0;
    CK(e, cudaMalloc(&sg.buf, need + (1u << 16)));
    sg.bytes = need + (1u << 16);
    sg.used = false;
    e->stage_gen++;  // descriptor tables cached by mrq_tick_many hold the old address
  }
  uint8_t *d_word = (uint8_t *)sg.buf;
  uint8_t *d_prop = d_word + wbytes;
  MsgRec *d_wide = (MsgRec *)(d_word + wbytes + pbytes);
  if (sg.used) CK(e, cudaStreamWaitEvent(e->copy_stream, sg.consumed, 0));
  // One frame, one copy, when the host laid it out the way the staging buffer is (rows without padding, the proposal
  // bytes right behind them): every async copy pays its own set-up on the link, and the link is this path's bound.
  const bool one_copy = rows && in->prop_count8 && e->gs == e->G && wbytes == e->G * rows * wsz &&
                        (const uint8_t *)in->prop_count8 == (const uint8_t *)in->word + wbytes;
  if (one_copy) {
    CK(e, cudaMemcpyAsync(d_word, in->word, wbytes + e->G, cudaMemcpyHostToDevice, e->copy_stream));
  } else {
    if (rows) CK(e, cudaMemcpy2DAsync(d_word, e->gs * wsz, in->word, e->G * wsz, e->G * wsz, rows, cudaMemcpyHostToDevice, e->copy_stream));
    if (in->prop_count8) CK(e, cudaMemcpyAsync(d_prop, in->prop_count8, e->G, cudaMemcpyHostToDevice, e->copy_stream));
  }
  if (in->n_wide) CK(e, cudaMemcpyAsync(d_wide, in->wide, xbytes, cudaMemcpyHostToDevice, e->copy_stream));
  CK(e, cudaEventRecord(sg.copied, e->copy_stream));
  CK(e, cudaStreamWaitEvent(e->stream, sg.copied, 0));
  if (bits == 32u) {
    unpack_inbox_kernel<<<nblocks(e->G), 256, 0, e->stream>>>(e->inbox[slot].view(), e->pk_base_index, e->pk_base_term, e->gs,
                                                            e->G, e->R, (const uint32_t *)d_word, in->prop_count8 ? d_prop : nullptr);
  } else if (bits == 8u && e->tick_mode >= 3) {
    // tick mode 3: no unpack pass — the tick kernels read the frame in the staging buffer (launch_tick records
    // `consumed` after them); only the escapes are scattered into the slot's wide columns, below
    sg.word8 = d_word;
    sg.prop8 = in->prop_count8 ? d_prop : nullptr;
    sg.frame8 = true;
    sg.keep8 = (in->reserved & MRQ_PACKED_KEEP) != 0;
    if (in->n_wide) {
      scatter_msgs_kernel<<<nblocks(in->n_wide), 256, 0, e->stream>>>(e->inbox[slot].view(), e->gs, e->G, e->R, d_wide, in->n_wide);
      CK(e, cudaGetLastError());
      e->launches++;
    }
    sg.used = true;
    return MRQ_OK;
  } else if (bits == 8u) {
    unpack8_inbox_kernel<<<nblocks(e->G), 256, 0, e->stream>>>(e->inbox[slot].view(), e->s.meta, e->pk_base_index, e->pk_base_term,
                                                             e->gs, e->G, e->R, d_word, in->prop_count8 ? d_prop : nullptr);
  } else {
    unpack16_inbox_kernel<<<nblocks(e->G), 256, 0, e->stream>>>(e->inbox[slot].view(), e->pk_base_index, e->pk_base_term, e->gs,
                                                              e->G, e->R, (const uint16_t *)d_word, in->prop_count8 ? d_prop : nullptr);
  }
  CK(e, cudaGetLastError());
  e->launches++;
  if (in->n_wide) {
    scatter_msgs_kernel<<<nblocks(in->n_wide), 256, 0, e->stream>>>(e->inbox[slot].view(), e->gs, e->G, e->R, d_wide, in->n_wide);
    CK(e, cudaGetLastError());
    e->launches++;
  }
  CK(e, cudaEventRecord(sg.consumed, e->stream));
  sg.used = true;
  return MRQ_OK;
}

int mrq_set_packed_base(mrq_engine *e, const uint64_t *base_index, const uint64_t *base_term) {
  if (!e) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  if (e->G == 0) return MRQ_OK;
  {
    int rw = ensure_wide(e, true);  // the window base is part of the compact representation (mode 4)
    if (rw) return rw;
  }
  if (base_index) CK(e, cudaMemcpyAsync(e->pk_base_index, base_index, e->G * 8, cudaMemcpyHostToDevice, e->stream));
  if (base_term) CK(e, cudaMemcpyAsync(e->pk_base_term, base_term, e->G * 8, cudaMemcpyHostToDevice, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

// ---- the byte form's host side: plain CPU code around the shared codec (include/mrq_packed8.h) ----------------
}  // extern "C"

namespace {
// Contiguous group ranges on a PERSISTENT pool of host threads: frames of a million groups are memory-bound host work
// (17 B of wide columns read per cell), so the builder scales with the cores the host gives it, and a live host builds
// one frame per tick — spawning threads per call would cost more than the frame.  MRQ_HOST_THREADS overrides the size.
extern "C" void mrqi_pack8_row(const uint8_t *ty, const uint64_t *tm, const uint64_t *ix, const uint64_t *bi, const uint64_t *bt,
                               uint64_t n, uint8_t *out);  // mrq_pack8_rows.cpp
extern "C" void mrqi_pack8_place(const uint8_t *b, const uint8_t *self, uint32_t r, uint64_t n, uint8_t *lo, uint8_t *hi, uint8_t *mn);
extern "C" int mrqi_pack8_marked(const uint8_t *b, uint64_t n);

class HostPool {
 public:
  ~HostPool() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      stop_ = true;
    }
    cv_.notify_all();
    for (auto &t : th_) t.join();
  }
  // f(chunk) for chunk = 0..n-1, on up to n threads (the caller's included); returns when all are done
  template <class F>
  void run(unsigned n, F f) {
    if (n <= 1) {
      if (n) f(0u);
      return;
    }
    std::lock_guard<std::mutex> serial(run_mu_);
    {
      std::lock_guard<std::mutex> lk(mu_);
      while (th_.size() + 1 < n) th_.emplace_back([this] { worker(); });
      job_ = [&f](unsigned c) { f(c); };
      njobs_ = n;
      next_ = 0;
      left_ = n;
      ++gen_;
    }
    cv_.notify_all();
    drain();
    std::unique_lock<std::mutex> lk(mu_);
    done_cv_.wait(lk, [this] { return left_ == 0; });
    job_ = nullptr;
  }
  std::vector<uint64_t> scratch;  // owned by whoever holds the pool inside run()'s caller (mrq_pack8 serialises itself)

 private:
  void drain() {
    for (;;) {
      unsigned c;
      {
        std::lock_guard<std::mutex> lk(mu_);
        if (next_ >= njobs_) return;
        c = next_++;
      }
      job_(c);
      {
        std::lock_guard<std::mutex> lk(mu_);
        if (--left_ == 0) done_cv_.notify_all();
      }
    }
  }
  void worker() {
    uint64_t seen = 0;
    for (;;) {
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return stop_ || gen_ != seen; });
        if (stop_) return;
        seen = gen_;
      }
      drain();
    }
  }
  std::mutex mu_, run_mu_;
  std::condition_variable cv_, done_cv_;
  std::vector<std::thread> th_;
  std::function<void(unsigned)> job_;
  unsigned njobs_ = 0, next_ = 0, left_ = 0;
  uint64_t gen_ = 0;
  bool stop_ = false;
};
HostPool &host_pool() {
  static HostPool *p = new HostPool();  // leaked on purpose: worker threads must not be joined from a static destructor
  return *p;
}
std::mutex g_pack_mu;

unsigned host_threads(uint64_t G) {
  unsigned hw = std::thread::hardware_concurrency();
  unsigned cap = 48;  // past a few dozen threads the frame builder is bound by host memory rather than cores; the cap
                      // was chosen on an earlier host and has not been re-tuned (tools/pack_probe.py times it)
  if (const char *s = getenv("MRQ_HOST_THREADS")) hw = cap = (unsigned)strtoul(s, nullptr, 10);
  if (hw < 1) hw = 1;
  const uint64_t by_size = G / 16384;  // below ~16k groups per thread the hand-off costs more than it saves
  if (by_size < hw) hw = (unsigned)(by_size < 1 ? 1 : by_size);
  return hw > cap ? cap : hw;
}
}  // namespace

extern "C" {

int mrq_pack8(const mrq_inbox *in, const uint8_t *self_id, uint64_t G, uint32_t R, uint64_t *base_index, const uint64_t *base_term,
              uint8_t *word_out, uint8_t *prop8_out, mrq_msg *wide_out, size_t wide_cap, size_t *n_wide) {
  if (!in || !in->type || !in->term || !in->index || !in->commit || !self_id || !base_index || !base_term || !n_wide)
    return fail(nullptr, MRQ_E_INVAL, "mrq_pack8: null argument");
  if (R < 1 || R > MRQ_MAX_REPLICAS) return fail(nullptr, MRQ_E_INVAL, "mrq_pack8: n_replicas %u outside 1..%u", R, MRQ_MAX_REPLICAS);
  if (R > 1 && !word_out) return fail(nullptr, MRQ_E_INVAL, "mrq_pack8: null word_out");
  const unsigned nt = host_threads(G);
  std::lock_guard<std::mutex> one_at_a_time(g_pack_mu);  // (the staging buffer below is shared)
  // One pass over the wide columns (they are the cost): bytes and proposal counts go straight to the output buffers;
  // escapes and the slid bases are staged and published only if everything fits, so a refused call leaves base_index —
  // the state that must stay in step with the device — untouched.  Only the columns a message's type needs are read.
  constexpr uint64_t kNone = ~0ull;
  std::vector<std::vector<mrq_msg>> esc(nt);
  std::vector<uint64_t> &slid = host_pool().scratch;
  if (slid.size() < G) slid.resize(G);
  std::vector<uint64_t> bad(nt, kNone);
  host_pool().run(nt, [&](unsigned c) {
    const uint64_t c0 = G * c / nt, c1 = G * (c + 1) / nt;
    // Row-major inside blocks of kBlk groups: each sender row is a straight streaming pass over its three columns
    // (type, then term / index / commit only where a message sits), the per-group window minimum lives in a block-sized
    // scratch that stays in L1.  The order of the escapes (by group, then by sender) is restored per block.
    constexpr uint64_t kBlk = 1024;
    uint8_t min_ack[kBlk], row_bytes[kBlk];
    std::vector<mrq_msg> blk_esc;
    for (uint64_t g0 = c0; g0 < c1; g0 += kBlk) {
      const uint64_t g1 = g0 + kBlk < c1 ? g0 + kBlk : c1;
      memset(min_ack, MRQ_P8_NO_ACK, sizeof min_ack);
      blk_esc.clear();
      for (uint32_t r = 0; r < R; ++r) {
        const uint8_t *ty = in->type + (uint64_t)r * G;
        const uint64_t *tm = in->term + (uint64_t)r * G, *ix = in->index + (uint64_t)r * G, *cm = in->commit + (uint64_t)r * G;
        // the common case for the whole row in one vectorised pass ...
        mrqi_pack8_row(ty + g0, tm + g0, ix + g0, base_index + g0, base_term + g0, g1 - g0, row_bytes);
        if (mrqi_pack8_marked(row_bytes, g1 - g0)) {  // ... the few marked cells re-encoded exactly, one by one
          for (uint64_t g = g0; g < g1; ++g) {
            if (row_bytes[g - g0] != MRQ_P8_ESCAPE) continue;
            const uint32_t self = self_id[g];
            if (r + 1u == self || self < 1u || self > R) continue;  // the group's own slot: nothing is ever stepped from there
            const uint8_t b = mrq_p8_encode(ty[g], tm[g], ix[g], cm[g], base_index[g], base_term[g]);
            row_bytes[g - g0] = b;
            if (b == MRQ_P8_ESCAPE) {
              mrq_msg m;
              memset(&m, 0, sizeof m);
              m.group = g;
              m.from = (uint8_t)(r + 1u);
              m.type = ty[g];
              m.term = tm[g];
              m.index = ix[g];
              m.logterm = in->logterm ? in->logterm[(uint64_t)r * G + g] : 0;
              m.commit = cm[g];
              blk_esc.push_back(m);
            }
          }
        }
        // ... and the row placed into the frame (row r or r - 1 by the group's own id) with byte-wide blends
        mrqi_pack8_place(row_bytes, self_id + g0, r, g1 - g0, r >= 1 ? word_out + (uint64_t)(r - 1u) * G + g0 : nullptr,
                         r + 1u < R ? word_out + (uint64_t)r * G + g0 : nullptr, min_ack);
      }
      if (!blk_esc.empty()) {  // rows were walked sender-major: put the block's escapes back in (group, sender) order
        std::stable_sort(blk_esc.begin(), blk_esc.end(), [](const mrq_msg &x, const mrq_msg &y) { return x.group < y.group; });
        esc[c].insert(esc[c].end(), blk_esc.begin(), blk_esc.end());
      }
      for (uint64_t g = g0; g < g1; ++g) slid[g] = mrq_p8_next_base(base_index[g], min_ack[g - g0]);
      if (prop8_out) {
        for (uint64_t g = g0; g < g1; ++g) {
          const uint32_t n = in->prop_count ? in->prop_count[g] : 0u;
          if (n > 255u && bad[c] == kNone) bad[c] = g;
          prop8_out[g] = (uint8_t)n;
        }
      }
    }
  });
  for (unsigned c = 0; c < nt; ++c)
    if (bad[c] != kNone)
      return fail(nullptr, MRQ_E_INVAL, "mrq_pack8: group %llu has %u proposals; the packed forms carry at most 255",
                  (unsigned long long)bad[c], in->prop_count[bad[c]]);
  size_t total = 0;
  for (unsigned c = 0; c < nt; ++c) total += esc[c].size();
  *n_wide = total;
  if (total > wide_cap || (total && !wide_out)) return fail(nullptr, MRQ_E_INVAL, "mrq_pack8: %zu escapes, room for %zu", total, wide_cap);
  size_t at = 0;
  for (unsigned c = 0; c < nt; ++c) {  // chunks are contiguous group ranges: the list stays in group order
    if (!esc[c].empty()) memcpy(wide_out + at, esc[c].data(), esc[c].size() * sizeof(mrq_msg));
    at += esc[c].size();
  }
  host_pool().run(nt, [&](unsigned c) {  // publish the slid window
    const uint64_t g0 = G * c / nt, g1 = G * (c + 1) / nt;
    if (g1 > g0) memcpy(base_index + g0, slid.data() + g0, (g1 - g0) * sizeof(uint64_t));
  });
  return MRQ_OK;
}

int mrq_unpack8(const uint8_t *word, const uint8_t *self_id, uint64_t G, uint32_t R, uint64_t *base_index, const uint64_t *base_term,
                const mrq_inbox_out *out) {
  if (!self_id || !base_index || !base_term || !out || !out->type || !out->term || !out->index || !out->commit)
    return fail(nullptr, MRQ_E_INVAL, "mrq_unpack8: null argument");
  if (R < 1 || R > MRQ_MAX_REPLICAS || (R > 1 && !word)) return fail(nullptr, MRQ_E_INVAL, "mrq_unpack8: bad arguments");
  for (uint64_t g = 0; g < G; ++g) {  // the body of unpack8_inbox_kernel, one group at a time
    const uint64_t bi = base_index[g], bt = base_term[g];
    uint32_t min_ack = MRQ_P8_NO_ACK;
    for (uint32_t r = 0; r < R; ++r) {
      const uint64_t o = (uint64_t)r * G + g;
      const uint32_t row = mrq_p8_row(r, self_id[g], R);
      if (row >= R - 1u) {
        out->type[o] = 0;
        continue;
      }
      const mrq_p8_cell c = mrq_p8_decode(word[(uint64_t)row * G + g], bi);
      out->type[o] = c.type;
      if (c.type == 0) continue;
      out->term[o] = bt;
      if (c.is_ack) {
        out->index[o] = c.value;
        min_ack = c.pay < min_ack ? c.pay : min_ack;
      } else if (c.is_hb) {
        out->commit[o] = c.value;
      } else {
        out->index[o] = 0;
      }
    }
    base_index[g] = mrq_p8_next_base(bi, min_ack);
  }
  return MRQ_OK;
}

int mrq_propose(mrq_engine *e, uint32_t slot, const uint64_t *groups, const uint32_t *counts, size_t n) {
  int r = check_slot(e, slot);
  if (r) return r;
  if (n == 0) return MRQ_OK;
  if (!groups || !counts) return fail(e, MRQ_E_INVAL, "null proposal list");
  CK(e, cudaSetDevice(e->device));
  if ((r = ensure_scratch(e, n * 12 + 64))) return r;
  uint64_t *d_g = (uint64_t *)e->scratch;
  uint32_t *d_c = (uint32_t *)((uint8_t *)e->scratch + n * 8);
  CK(e, cudaMemcpyAsync(d_g, groups, n * 8, cudaMemcpyHostToDevice, e->stream));
  CK(e, cudaMemcpyAsync(d_c, counts, n * 4, cudaMemcpyHostToDevice, e->stream));
  scatter_props_kernel<<<nblocks(n), 256, 0, e->stream>>>(e->inbox[slot].prop, e->G, d_g, d_c, n);
  CK(e, cudaGetLastError());
  e->launches++;
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

int mrq_read_inbox(mrq_engine *e, uint32_t slot, mrq_inbox_out *o) {
  int r = check_slot(e, slot);
  if (r) return r;
  if (!o) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  if (e->G == 0) return MRQ_OK;
  InboxBuf &ib = e->inbox[slot];
  if ((r = copy_out(e, o->type, ib.type, 1, e->R))) return r;
  if ((r = copy_out(e, o->term, ib.term, 8, e->R))) return r;
  if ((r = copy_out(e, o->index, ib.index, 8, e->R))) return r;
  if ((r = copy_out(e, o->logterm, ib.logterm, 8, e->R))) return r;
  if ((r = copy_out(e, o->commit, ib.commit, 8, e->R))) return r;
  if ((r = copy_out(e, o->prop_count, ib.prop, 4, 1))) return r;
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

int mrq_gen_trace(mrq_engine *e, uint32_t slot, const struct mrq_trace_params *p, uint64_t tick) {
  int r = check_slot(e, slot);
  if (r) return r;
  drop_frame8(e, slot);
  if (!p) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  if (e->G == 0) return MRQ_OK;
  if ((r = ensure_wide(e, false))) return r;
  gen_trace_kernel<<<nblocks(e->G), 256, 0, e->stream>>>(e->inbox[slot].view(), e->s, e->gs, e->G, e->R, e->cfg.group_base, *p, tick);
  CK(e, cudaGetLastError());
  e->launches++;
  return MRQ_OK;
}

// ---- hot path --------------------------------------------------------------------------------------------------
int mrq_tick(mrq_engine *e, uint32_t slot) {
  int r = check_slot(e, slot);
  if (r) return r;
  CK(e, cudaSetDevice(e->device));
  return launch_tick(e, &e->inbox[slot]);
}

// n ticks in one call.  The launch sequence for a given slot list is captured once into a CUDA graph (the
// tick number and the slow-list length live in device memory, double-buffered by tick parity, so a replay
// needs no per-launch host arguments) and replayed afterwards: the per-tick host cost drops from two
// cudaLaunchKernelEx calls to a fraction of one graph launch.
int mrq_tick_many(mrq_engine *e, const uint32_t *slots, uint32_t n) {
  if (!e) return MRQ_E_INVAL;
  if (n == 0) return MRQ_OK;
  if (!slots) return fail(e, MRQ_E_INVAL, "null slot list");
  for (uint32_t k = 0; k < n; ++k) {
    int r = check_slot(e, slots[k]);
    if (r) return r;
  }
  CK(e, cudaSetDevice(e->device));
  const bool nccl_gather = e->world > 1 && e->comm_mode == 0 && e->comm;
  if (e->tick_mode == 4 && e->G > 0 && !nccl_gather && e->graph_mode != 0) {
    // mode 4: the whole sequence in ONE pair of launches — every thread walks its four groups through the n frames
    // (state in registers from tick to tick), the general kernel finishes the groups that left the fast path
    bool all8 = true;
    for (uint32_t k = 0; k < n; ++k) all8 = all8 && slot_has_frame8(e, slots[k]);
    if (all8) {
      constexpr uint32_t kMaxBatch = kMaxTicksPerLaunch;
      for (uint32_t k = 0; k < n; k += kMaxBatch) {
        int r = launch_tick4(e, slots + k, n - k < kMaxBatch ? n - k : kMaxBatch);
        if (r) return r;
      }
      return MRQ_OK;
    }
  }
  // graph_mode: 0 never, 1 always, 2 (default) only for small shards, where the host's launch rate rather than
  // the kernels bounds the tick rate (kGraphAutoMaxGroups)
  const bool want_graph = e->graph_mode == 1 || (e->graph_mode == 2 && e->G <= kGraphAutoMaxGroups);
  const bool can_graph = want_graph && n >= 2 && !e->graphs_disabled && !nccl_gather && !e->gather_prime && e->G > 0 &&
                         e->tick_mode < 3;  // mode 3/4 ticks read per-post staging buffers: not replayable
  if (!can_graph) {
    for (uint32_t k = 0; k < n; ++k) {
      int r = launch_tick(e, &e->inbox[slots[k]]);
      if (r) return r;
    }
    return MRQ_OK;
  }
  std::string key((const char *)slots, (size_t)n * sizeof(uint32_t));
  key.push_back((char)('0' + (e->tick_parity & 1u)));
  key.push_back((char)('0' + (e->slow_parity & 1u)));
  key.push_back((char)('0' + e->tick_mode));
  key.push_back((char)('0' + ((e->comm_mode == 1 && e->ipc_attached) ? e->world : 1)));
  key.push_back((char)('0' + (e->l2_policy ? 1 : 0)));  // a kernel argument, so part of what was captured
  const uint64_t tick0 = e->tick_no, launches0 = e->launches;
  const uint32_t tp0 = e->tick_parity, sp0 = e->slow_parity;
  auto it = e->graphs.find(key);
  if (it == e->graphs.end()) {
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    bool ok = cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
    int rc = MRQ_OK;
    if (ok) {
      for (uint32_t k = 0; k < n && rc == MRQ_OK; ++k) rc = launch_tick(e, &e->inbox[slots[k]]);
      ok = cudaStreamEndCapture(e->stream, &graph) == cudaSuccess && rc == MRQ_OK && graph != nullptr;
    }
    // capture recorded the launches without running them: rewind the host-side bookkeeping
    const uint64_t per_tick = n ? (e->launches - launches0) / n : 0;
    e->tick_no = tick0;
    e->launches = launches0;
    e->tick_parity = tp0;
    e->slow_parity = sp0;
    if (ok) ok = cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess;
    if (graph) cudaGraphDestroy(graph);
    if (!ok) {  // no graph support for this sequence: fall back to plain launches from now on
      cudaGetLastError();
      e->graphs_disabled = true;
      return mrq_tick_many(e, slots, n);
    }
    (void)per_tick;
    it = e->graphs.emplace(key, exec).first;
  }
  CK(e, cudaGraphLaunch(it->second, e->stream));
  e->tick_no = tick0 + n;
  e->launches = launches0 + (uint64_t)n * (e->tick_mode == 0 ? 2u : 1u);
  if (n & 1u) {
    e->tick_parity = tp0 ^ 1u;
    if (e->tick_mode == 0) e->slow_parity = sp0 ^ 1u;
  }
  return MRQ_OK;
}

int mrq_tick_idle(mrq_engine *e, uint32_t n) {
  if (!e) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  for (uint32_t k = 0; k < n; ++k) {
    int r = launch_tick(e, nullptr);
    if (r) return r;
  }
  return MRQ_OK;
}

int mrq_quorum_commit(mrq_engine *e) {
  if (!e) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  if (e->G == 0) return MRQ_OK;
  {
    int rw = ensure_wide(e, true);
    if (rw) return rw;
  }
  QuorumArgs a{e->s.match, e->s.committed, e->s.term_start, e->ctr, e->G, e->gs};
  return launch_quorum(e, a, e->quorum_variant);
}

int mrq_set_l2_policy(mrq_engine *e, int on) {
  if (!e || on < 0 || on > 1) return MRQ_E_INVAL;
  e->l2_policy = on;
  return MRQ_OK;
}

int mrq_set_graph_mode(mrq_engine *e, int mode) {
  if (!e || mode < 0 || mode > 2) return MRQ_E_INVAL;
  e->graph_mode = mode;
  return MRQ_OK;
}

int mrq_set_tick_mode(mrq_engine *e, int mode) {
  if (!e || mode < 0 || mode > 4) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  if (e->tick_mode == 4 && mode != 4) {  // leaving compact state: the wide columns become the only truth again
    int r = ensure_wide(e, true);
    if (r) return r;
  }
  if (mode == 4) {
    int r = ensure_compact_alloc(e);
    if (r) return r;
  }
  e->tick_mode = mode;
  return MRQ_OK;
}

int mrq_set_quorum_variant(mrq_engine *e, int variant) {
  if (!e || variant < 0 || variant > 2) return MRQ_E_INVAL;
  e->quorum_variant = variant;
  return MRQ_OK;
}

int mrq_quorum_commit_ext(mrq_engine *e, const uint64_t *d_match, uint64_t *d_committed, const uint64_t *d_term_start,
                          uint64_t n_groups, uint64_t stride, int variant) {
  if (!e || !d_match || !d_committed || !d_term_start) return MRQ_E_INVAL;
  if (stride < n_groups || (stride & 3)) return fail(e, MRQ_E_INVAL, "stride must be a multiple of 4 and >= n_groups");
  // 16 bytes: the widest access of every form (128-bit loads / stores, and the source of a TMA bulk copy)
  if (((uintptr_t)d_match | (uintptr_t)d_committed | (uintptr_t)d_term_start) & 15)
    return fail(e, MRQ_E_INVAL, "device columns must be 16-byte aligned");
  if (variant < 0 || variant > 2) return fail(e, MRQ_E_INVAL, "variant outside 0..2");
  CK(e, cudaSetDevice(e->device));
  if (n_groups == 0) return MRQ_OK;
  QuorumArgs a{d_match, d_committed, d_term_start, nullptr, n_groups, stride};
  return launch_quorum(e, a, variant);
}

int mrq_match_update(mrq_engine *e, const uint64_t *groups, const uint8_t *from, const uint64_t *index, size_t n) {
  if (!e) return MRQ_E_INVAL;
  if (n == 0) return MRQ_OK;
  if (!groups || !from || !index) return fail(e, MRQ_E_INVAL, "null ack list");
  CK(e, cudaSetDevice(e->device));
  int r = ensure_wide(e, true);
  if (r) return r;
  if ((r = ensure_scratch(e, n * 17 + 64))) return r;
  uint64_t *d_g = (uint64_t *)e->scratch, *d_i = d_g + n;
  uint8_t *d_f = (uint8_t *)(d_i + n);
  CK(e, cudaMemcpyAsync(d_g, groups, n * 8, cudaMemcpyHostToDevice, e->stream));
  CK(e, cudaMemcpyAsync(d_i, index, n * 8, cudaMemcpyHostToDevice, e->stream));
  CK(e, cudaMemcpyAsync(d_f, from, n, cudaMemcpyHostToDevice, e->stream));
  match_update_kernel<<<nblocks(n), 256, 0, e->stream>>>(e->s.match, e->gs, e->G, e->R, d_g, d_f, d_i, n);
  CK(e, cudaGetLastError());
  e->launches++;
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

// ---- outputs ---------------------------------------------------------------------------------------------------
int mrq_synchronize(mrq_engine *e) {
  if (!e) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

int mrq_sync_commits(mrq_engine *e, uint64_t *committed_out, uint8_t *role_out, uint64_t *term_out) {
  if (!e) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  if (e->G == 0) return MRQ_OK;
  {
    int rw = ensure_wide(e, false);
    if (rw) return rw;
  }
  if (committed_out) {
    CK(e, cudaMemcpyAsync(committed_out, e->s.committed, e->G * 8, cudaMemcpyDeviceToHost, e->stream));
    // a full read rebases the compact drain: the next mrq_sync_commit_deltas counts from these values
    CK(e, cudaMemcpyAsync(e->commit_prev, e->s.committed, e->G * 8, cudaMemcpyDeviceToDevice, e->stream));
  }
  if (term_out) CK(e, cudaMemcpyAsync(term_out, e->s.term, e->G * 8, cudaMemcpyDeviceToHost, e->stream));
  if (role_out) {
    mrq_state st;
    memset(&st, 0, sizeof st);
    st.role = role_out;
    return mrq_export_state(e, &st);
  }
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

int mrq_sync_out(mrq_engine *e, uint32_t *out_words) {
  if (!e || !out_words) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  if (e->G) CK(e, cudaMemcpyAsync(out_words, e->last_out ? e->last_out : e->s.out, e->G * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

int mrq_sync_commit_deltas(mrq_engine *e, uint8_t *delta_out) {
  if (!e || !delta_out) return MRQ_E_INVAL;
  int r0 = MRQ_OK;
  CK(e, cudaSetDevice(e->device));
  if (e->G == 0) return MRQ_OK;
  {
    int rw = ensure_wide(e, false);
    if (rw) return rw;
  }
  if ((r0 = ensure_scratch(e, e->gs))) return r0;  // (e->delta holds the last mode-4 tick's own advances)
  commit_delta_kernel<<<nblocks(e->G), 256, 0, e->stream>>>(e->s.committed, e->commit_prev, (uint8_t *)e->scratch, e->G);
  CK(e, cudaGetLastError());
  e->launches++;
  CK(e, cudaMemcpyAsync(delta_out, e->scratch, e->G, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

int mrq_drain_commit_deltas(mrq_engine *e, uint8_t *delta_out_pinned) {
  if (!e || !delta_out_pinned) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  if (!e->drain_done) CK(e, cudaEventCreateWithFlags(&e->drain_done, cudaEventDisableTiming));
  if (e->G) {
    int rw = ensure_wide(e, false);
    if (rw) return rw;
    if ((rw = ensure_scratch(e, e->gs))) return rw;
    commit_delta_kernel<<<nblocks(e->G), 256, 0, e->stream>>>(e->s.committed, e->commit_prev, (uint8_t *)e->scratch, e->G);
    CK(e, cudaGetLastError());
    e->launches++;
    CK(e, cudaMemcpyAsync(delta_out_pinned, e->scratch, e->G, cudaMemcpyDeviceToHost, e->stream));
  }
  CK(e, cudaEventRecord(e->drain_done, e->stream));
  return MRQ_OK;
}

// Mode 4: the tick kernels write every group's commit advance of THAT tick (1 B, 255 = "read the index in full") next to
// the out word, so the per-tick drain is a plain copy of the last tick's bytes — no extra kernel, no extra pass.
int mrq_drain_tick_deltas(mrq_engine *e, uint8_t *delta_out_pinned) {
  if (!e || !delta_out_pinned) return MRQ_E_INVAL;
  if (!e->last_delta) return fail(e, MRQ_E_STATE, "mrq_drain_tick_deltas: the last tick was not a mode-4 tick on a byte frame");
  CK(e, cudaSetDevice(e->device));
  if (!e->drain_done) CK(e, cudaEventCreateWithFlags(&e->drain_done, cudaEventDisableTiming));
  if (e->G) CK(e, cudaMemcpyAsync(delta_out_pinned, e->last_delta, e->G, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaEventRecord(e->drain_done, e->stream));
  return MRQ_OK;
}

// The outputs of the tick that consumed inbox slot `slot` in the last mrq_tick_many of mode 4 (each tick of such a
// sequence writes its out words and commit advances to its slot's own buffers).  Blocking; NULL skips a column.
int mrq_sync_slot_outputs(mrq_engine *e, uint32_t slot, uint32_t *out_words, uint8_t *delta_out) {
  int r = check_slot(e, slot);
  if (r) return r;
  if (slot >= e->out_slot.size() || !e->out_slot[slot] || !e->delta_slot[slot] || slot >= e->slot_out_live.size() ||
      !e->slot_out_live[slot])
    return fail(e, MRQ_E_STATE, "slot %u was not part of a mode-4 mrq_tick_many sequence", slot);
  CK(e, cudaSetDevice(e->device));
  if (e->G && out_words) CK(e, cudaMemcpyAsync(out_words, e->out_slot[slot], e->G * 4, cudaMemcpyDeviceToHost, e->stream));
  if (e->G && delta_out) CK(e, cudaMemcpyAsync(delta_out, e->delta_slot[slot], e->G, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

int mrq_set_change_capacity(mrq_engine *e, uint64_t max_records) {
  if (!e) return MRQ_E_INVAL;
  if (max_records > (UINT64_MAX >> 6)) return fail(e, MRQ_E_INVAL, "change capacity %llu is too large", (unsigned long long)max_records);
  CK(e, cudaSetDevice(e->device));
  CK(e, cudaStreamSynchronize(e->stream));  // launches in flight may still append to the old buffer
  // Captured graphs (modes 0-3) hold the old feed arguments: a replay must not run with them, so they start over.  (The
  // mode-4 descriptor tables hold only frame and output pointers; the feed rides in the kernel arguments of every launch.)
  for (auto &kv : e->graphs) cudaGraphExecDestroy(kv.second);
  e->graphs.clear();
  if (max_records != 0 && max_records == e->change_cap) {  // same size: keep the buffer, discard what is pending
    CK(e, cudaMemsetAsync(e->change_count, 0, sizeof(unsigned long long), e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    return MRQ_OK;
  }
  if (e->changes) CK(e, cudaFree(e->changes));
  e->changes = nullptr;
  e->change_cap = 0;
  if (max_records == 0) return MRQ_OK;
  if (!e->change_count) {
    int r = dalloc(e, &e->change_count, 1);
    if (r) return r;
  }
  CK(e, cudaMalloc((void **)&e->changes, max_records * sizeof(mrq_change)));
  CK(e, cudaMemsetAsync(e->change_count, 0, sizeof(unsigned long long), e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  e->change_cap = max_records;
  return MRQ_OK;
}

int mrq_sync_changes(mrq_engine *e, mrq_change *out, uint64_t cap, uint64_t *n_out, uint64_t *lost) {
  if (!e || !n_out || !lost || (cap && !out)) return MRQ_E_INVAL;
  if (!e->changes) return fail(e, MRQ_E_STATE, "mrq_sync_changes: the change feed is off (mrq_set_change_capacity)");
  CK(e, cudaSetDevice(e->device));
  unsigned long long count = 0;
  CK(e, cudaMemcpyAsync(&count, e->change_count, sizeof count, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  const uint64_t n = count < e->change_cap ? count : e->change_cap;
  *n_out = n;
  if (cap < n) {
    *lost = 0;
    return fail(e, MRQ_E_INVAL, "mrq_sync_changes: %llu records pending, room for %llu", (unsigned long long)n, (unsigned long long)cap);
  }
  if (n) CK(e, cudaMemcpyAsync(out, e->changes, n * sizeof(mrq_change), cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaMemsetAsync(e->change_count, 0, sizeof(unsigned long long), e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  // warps append in whatever order they run: the host sorts the (sparse) list
  std::sort(out, out + n, [](const mrq_change &x, const mrq_change &y) { return x.tick != y.tick ? x.tick < y.tick : x.group < y.group; });
  *lost = count - n;
  return MRQ_OK;
}

int mrq_set_write_through(mrq_engine *e, int on) {
  if (!e || on < 0 || on > 1) return MRQ_E_INVAL;
  e->write_through = on;
  return MRQ_OK;
}

int mrq_drain_wait(mrq_engine *e) {
  if (!e) return MRQ_E_INVAL;
  if (!e->drain_done) return fail(e, MRQ_E_STATE, "mrq_drain_wait without mrq_drain_commit_deltas");
  CK(e, cudaSetDevice(e->device));
  CK(e, cudaEventSynchronize(e->drain_done));
  return MRQ_OK;
}

int mrq_get_counters(mrq_engine *e, mrq_counters *out) {
  if (!e || !out) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  Counters shards[kCtrShards];
  CK(e, cudaMemcpyAsync(shards, e->ctr, sizeof shards, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  Counters c{};
  for (int k = 0; k < kCtrShards; ++k) {
    c.campaigns += shards[k].campaigns;
    c.elections_won += shards[k].elections_won;
    c.step_downs += shards[k].step_downs;
    c.commits_advanced += shards[k].commits_advanced;
    c.votes_granted += shards[k].votes_granted;
    c.errors += shards[k].errors;
  }
  out->ticks = e->tick_no;
  out->kernel_launches = e->launches;
  out->campaigns = c.campaigns;
  out->elections_won = c.elections_won;
  out->step_downs = c.step_downs;
  out->commits_advanced = c.commits_advanced;
  out->votes_granted = c.votes_granted;
  out->errors = c.errors;
  return MRQ_OK;
}

int mrq_timer_start(mrq_engine *e) {
  if (!e) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  CK(e, cudaEventRecord(e->ev0, e->stream));
  return MRQ_OK;
}
int mrq_timer_stop(mrq_engine *e, float *ms) {
  if (!e || !ms) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  CK(e, cudaEventRecord(e->ev1, e->stream));
  CK(e, cudaEventSynchronize(e->ev1));
  CK(e, cudaEventElapsedTime(ms, e->ev0, e->ev1));
  return MRQ_OK;
}

// ---- multi-GPU -------------------------------------------------------------------------------------------------
int mrq_comm_unique_id(uint8_t id_out[MRQ_COMM_ID_BYTES]) {
  if (!id_out) return MRQ_E_INVAL;
  if (!g_nccl.load()) return fail(nullptr, MRQ_E_NCCL, "%s", g_nccl.err.c_str());
  NcclUniqueId id;
  int st = g_nccl.GetUniqueId(&id);
  if (st != 0) return fail(nullptr, MRQ_E_NCCL, "ncclGetUniqueId failed (%d)", st);
  static_assert(sizeof(NcclUniqueId) == MRQ_COMM_ID_BYTES, "id size");
  memcpy(id_out, &id, MRQ_COMM_ID_BYTES);
  return MRQ_OK;
}

static int ensure_gather(mrq_engine *e, uint32_t world) {
  // peers hold CUDA-IPC mappings of the current buffer and graphs hold its address: it cannot be replaced
  if (e->ipc_attached) return fail(e, MRQ_E_STATE, "the gather buffer is already shared with the peers (mrq_ipc_attach)");
  if (e->comm) return fail(e, MRQ_E_STATE, "a communicator is already attached to this engine");
  CK(e, cudaStreamSynchronize(e->stream));
  if (e->gathered) CK(e, cudaFree(e->gathered));
  e->gathered = nullptr;
  const size_t n = (size_t)world * (e->G ? e->G : 1);
  return dalloc(e, &e->gathered, n + (n + 7) / 8);  // n full indices + n low bytes (the peer-store layout); NCCL uses the first n
}

int mrq_comm_init(mrq_engine *e, const uint8_t id[MRQ_COMM_ID_BYTES], uint32_t rank, uint32_t world) {
  if (!e || !id || world < 1 || world > 8 || rank >= world) return fail(e, MRQ_E_INVAL, "bad communicator arguments");
  if (!g_nccl.load()) return fail(e, MRQ_E_NCCL, "%s", g_nccl.err.c_str());
  CK(e, cudaSetDevice(e->device));
  int r = ensure_gather(e, world);
  if (r) return r;
  NcclUniqueId uid;
  memcpy(&uid, id, MRQ_COMM_ID_BYTES);
  int st = g_nccl.CommInitRank(&e->comm, (int)world, uid, (int)rank);
  if (st != 0) return fail(e, MRQ_E_NCCL, "ncclCommInitRank failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(st) : "?");
  e->gather_shared = true;
  e->world = world;
  e->rank = rank;
  return MRQ_OK;
}

int mrq_comm_set_mode(mrq_engine *e, uint32_t mode) {
  if (!e || mode > 1) return MRQ_E_INVAL;
  if (mode == 1 && !e->ipc_attached) return fail(e, MRQ_E_STATE, "peer-store gather needs mrq_ipc_attach first");
  e->comm_mode = mode;
  if (mode == 1) e->gather_prime = true;  // (re)publish the full indices on the next tick
  return MRQ_OK;
}

int mrq_ipc_export(mrq_engine *e, uint8_t handle_out[MRQ_IPC_HANDLE_BYTES]) {
  if (!e || !handle_out) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  static_assert(sizeof(cudaIpcMemHandle_t) == MRQ_IPC_HANDLE_BYTES, "ipc handle size");
  cudaIpcMemHandle_t h;
  CK(e, cudaIpcGetMemHandle(&h, e->gathered));
  memcpy(handle_out, &h, sizeof h);
  return MRQ_OK;
}

int mrq_ipc_prepare(mrq_engine *e, uint32_t world) {
  if (!e || world < 1 || world > 8) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  int r = ensure_gather(e, world);
  if (r) return r;
  e->gather_shared = true;  // the buffer's handle may be exported from here on
  return MRQ_OK;
}

int mrq_ipc_attach(mrq_engine *e, const uint8_t *handles, uint32_t rank, uint32_t world) {
  if (!e || !handles || world < 1 || world > 8 || rank >= world) return fail(e, MRQ_E_INVAL, "bad ipc arguments");
  if (e->ipc_attached) return fail(e, MRQ_E_STATE, "mrq_ipc_attach called twice");
  CK(e, cudaSetDevice(e->device));
  for (uint32_t p = 0; p < world; ++p) {
    if (p == rank) {
      e->peer_gather[p] = e->gathered;
      continue;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + (size_t)p * MRQ_IPC_HANDLE_BYTES, sizeof h);
    void *ptr = nullptr;
    cudaError_t st = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
    if (st != cudaSuccess) {  // unmap what was opened so far: a failed attach leaves the engine unattached
      for (uint32_t q = 0; q < p; ++q)
        if (q != rank && e->peer_gather[q]) cudaIpcCloseMemHandle(e->peer_gather[q]);
      for (uint32_t q = 0; q < 8; ++q) e->peer_gather[q] = nullptr;
      return fail(e, MRQ_E_CUDA, "cudaIpcOpenMemHandle(rank %u) failed: %s", p, cudaGetErrorString(st));
    }
    e->peer_gather[p] = (uint64_t *)ptr;
  }
  e->world = world;
  e->rank = rank;
  e->ipc_attached = true;
  e->gather_prime = true;  // the first tick publishes the full index of every group
  return MRQ_OK;
}

int mrq_sync_gathered(mrq_engine *e, uint64_t *gathered_out) {
  if (!e || !gathered_out) return MRQ_E_INVAL;
  CK(e, cudaSetDevice(e->device));
  const size_t n = (size_t)e->world * e->G;
  if (e->comm_mode == 1 && e->ipc_attached) {
    // peer-store layout: full indices [n] (as of the last time anything above the low byte changed) then low bytes [n]
    std::vector<uint8_t> lo(n);
    CK(e, cudaMemcpyAsync(gathered_out, e->gathered, n * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(lo.data(), reinterpret_cast<const uint8_t *>(e->gathered + n), n, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    for (size_t k = 0; k < n; ++k) gathered_out[k] = (gathered_out[k] & ~0xFFull) | lo[k];
    return MRQ_OK;
  }
  CK(e, cudaMemcpyAsync(gathered_out, e->gathered, n * 8, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  return MRQ_OK;
}

}  // extern "C"
