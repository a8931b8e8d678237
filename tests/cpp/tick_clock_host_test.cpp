// tick_clock_host_test.cpp — tick mode 4 on the host in the library's form: 16-bit offset columns and clock-relative
// leader timers (c.clk).
//
// tick_host_test.cpp and tick_host16_test.cpp run the compact per-group functions of raftsql_b200/csrc/mrq_kernels.cuh
// with the timers in meta (c.clk null).  The library keeps a compact leader's electionElapsed and heartbeatElapsed as
// phases against the tick number instead: the hot step gets the "settled leader" test once per launch and a
// heartbeatElapsed countdown in registers, the cold step advances that countdown instead of meta, and materialise_group
// writes the real timers back into meta.  This file runs that form against the oracle, the way tick_fast4_kernel and
// tick_slow4_kernel run it: traces, message soups, the window-edge soup, ElectionTick and HeartbeatTick at their
// extremes, leaders imported with timers out of range, tick numbers near 2^32 and 2^64 - 1, a tick-count reset in the
// middle of a run, and the hot step switched off.  After every batch the timers materialise_group writes, and every
// other column, must equal the oracle's; a compact leader must never mark its meta word dirty.
//
// The harness around the compact columns (engine layout, oracle columns, comparison, trace presets) is
// tick_host_test.cpp's, included here with its main() renamed.
//
//   tick_clock_host_test               all cases;   exit code 0 and "tick_clock_host_test: ok" on success
#define main tick_host_test_main
#include "tick_host_test.cpp"
#undef main

namespace {

using W = uint16_t;

struct ClockHost {  // the library's compact columns: 16-bit offsets plus the timer phases
  uint64_t gs;
  uint32_t R;
  std::vector<uint8_t> flag;
  std::vector<W> commit, win, gate, match;
  std::vector<uint32_t> iblo, clk;
  std::vector<uint64_t> ibase;
  uint64_t fast_ticks = 0, slow_entries = 0, hot_ticks = 0, leader_ticks = 0;
  ClockHost(uint64_t gs_, uint32_t R_)
      : gs(gs_), R(R_), flag(gs_, 0), commit(gs_, 0), win(gs_, 0), gate(gs_, 0), match(gs_ * R_, 0), iblo(gs_, 0),
        clk(gs_, 0xA5A5A5A5u), ibase(gs_, 0) {}
  CompactViewT<W> view() {
    return CompactViewT<W>{flag.data(), commit.data(), win.data(), gate.data(), iblo.data(), match.data(), ibase.data(), clk.data()};
  }
  void invalidate() { std::fill(flag.begin(), flag.end(), 0); }
};

// what tick_fast4_kernel + tick_slow4_kernel do per group over one K-tick launch
template <int R>
void host_ticks_clk(HostEngine &e, ClockHost &ch, const TickArgs &a, std::vector<TickDesc> &descs, uint64_t *base_index,
                    const uint64_t *base_term, const char *where) {
  Tick4ArgsT<W> A{};
  A.t = a;
  A.c = ch.view();
  A.base_index = base_index;
  A.base_term = base_term;
  A.nticks = (uint32_t)descs.size();
  A.d0 = descs[0];
  A.descs = descs.size() > 1 ? descs.data() : nullptr;
  A.write_through = 1;
  const uint64_t tick0 = e.tick_no[0];
  const uint32_t et = a.election_tick, ht = a.heartbeat_tick;
  for (uint64_t i = 0; i < e.G; ++i) {
    CGroup<R> g;
    g.meta = e.meta[i];
    g.commit = ch.commit[i];
    g.win = ch.win[i];
    for (int r = 0; r < R; ++r) g.m[r] = ch.match[(uint64_t)r * e.gs + i];
    const uint32_t flag = ch.flag[i];
    const uint32_t gate = ch.gate[i];
    const bool settled = compact_settled(flag, g.meta);  // once per launch, as the kernels do
    const bool leader = (flag & CF_COMPACT) && meta_unpack(g.meta).role == MRQ_ROLE_LEADER;
    uint32_t hb = ht > 1u ? clk_value((ch.clk[i] >> 16) & 0xFFu, tick0, ht) & 0xFFu : 0u;
    uint32_t t = 0;
    bool slow = false;
    for (; t < A.nticks; ++t) {
      const TickDesc &d = descs[t];
      uint32_t wb[R > 1 ? R - 1 : 1] = {0};
      for (int j = 0; j < R - 1; ++j) wb[j] = d.word8[(uint64_t)j * e.gs + i];
      uint32_t o, adv, dirty;
      const uint32_t np = d.prop8 ? d.prop8[i] : 0u;
      slow = false;
      if (!hot_path || !compact_hot_step_clk<R, W>(g, settled, flag, wb, np, gate, ht, hb, 0, o, adv, dirty))
        slow = compact_step<R, W>(g, flag, wb, np, gate, et, ht, o, adv, dirty, &hb);
      else
        ++ch.hot_ticks;
      if (slow) break;
      if (leader && (dirty & CD_META)) {
        std::printf("FAIL %s tick %llu group %llu: a compact leader marked its meta word dirty\n", where,
                    (unsigned long long)(tick0 + t), (unsigned long long)i);
        ++failures;
      }
      if (hb > 0xFFu) {
        std::printf("FAIL %s tick %llu group %llu: heartbeat countdown %u outgrew its byte\n", where, (unsigned long long)(tick0 + t),
                    (unsigned long long)i, hb);
        ++failures;
      }
      d.out[i] = o;
      d.delta[i] = (uint8_t)(adv > 255u ? 255u : adv);
      ++ch.fast_ticks;
      ch.leader_ticks += leader;
    }
    e.meta[i] = g.meta;
    ch.commit[i] = (W)g.commit;
    ch.win[i] = (W)g.win;
    for (int r = 0; r < R; ++r) ch.match[(uint64_t)r * e.gs + i] = (W)g.m[r];
    if (slow) {
      slow_group_ticks_c<R>(A, i, t);
      ++ch.slow_entries;
    }
  }
  e.tick_no[0] += A.nticks;
}

void dispatch_ticks_clk(HostEngine &e, ClockHost &ch, const TickArgs &a, std::vector<TickDesc> &descs, uint64_t *bi, const uint64_t *bt,
                        const char *where) {
  switch (e.R) {
    case 1: host_ticks_clk<1>(e, ch, a, descs, bi, bt, where); break;
    case 2: host_ticks_clk<2>(e, ch, a, descs, bi, bt, where); break;
    case 3: host_ticks_clk<3>(e, ch, a, descs, bi, bt, where); break;
    case 4: host_ticks_clk<4>(e, ch, a, descs, bi, bt, where); break;
    case 5: host_ticks_clk<5>(e, ch, a, descs, bi, bt, where); break;
    case 6: host_ticks_clk<6>(e, ch, a, descs, bi, bt, where); break;
    case 7: host_ticks_clk<7>(e, ch, a, descs, bi, bt, where); break;
    case 8: host_ticks_clk<8>(e, ch, a, descs, bi, bt, where); break;
  }
}

struct Case {
  uint64_t G = 300;
  uint32_t R = 5, cfg = 5, K = 1;
  int T = 224, rebase_every = 32, also_rebase_at = -1;  // (a re-base once the cold start's elections are over)
  bool soup = false, edges = false;
  uint64_t big = 0;             // steady leaders whose indices sit this far up (0: the oracle's own start)
  bool wild_timers = false;     // (with big) leaders imported with electionElapsed >= ET or heartbeatElapsed >= HT
  uint32_t et = 10, ht = 1;
  uint64_t tick0 = 0;           // the tick number of the first tick
  int reset_at = -1;            // at this batch start the tick count is set to reset_to (mrq_set_tick_count)
  uint64_t reset_to = 0;
  const char *what = "";
};

// run_case_w of tick_host16_test.cpp with clock-relative timers: every batch is one launch of host_ticks_clk, and after
// it materialise_group at the current tick number must give the oracle's timers and state.
void run_case_clk(const Case &cs) {
  const uint64_t G = cs.G;
  const uint32_t R = cs.R, K = cs.K, et = cs.et, ht = cs.ht;
  char where[160];
  std::snprintf(where, sizeof where, "clock%s K=%u G=%llu R=%u %s=%u ET=%u HT=%u%s%s", cs.soup ? " soup" : "", K, (unsigned long long)G, R,
                cs.soup ? "seed" : "cfg", cs.cfg, et, ht, *cs.what ? " " : "", cs.what);
  const uint64_t seed = 0x5EEDC100ull + cs.cfg * 131 + R + et * 7 + ht;
  orc_engine *o = orc_create(G, R, 0, et, ht, seed, 0);
  HostEngine e(G, R);
  ClockHost ch(e.gs, R);
  OracleCols c(G, R);
  c.load(o);
  if (cs.big) {  // steady-state leaders (tick_host16_test's "far base" case), optionally with timers out of range
    uint64_t x = 7;
    auto rnd = [&]() { return x = mrq_mix64(x + 0x9E3779B97F4A7C15ull); };
    for (uint64_t g = 0; g < G; ++g) {
      const uint32_t self = (uint32_t)(g % R) + 1;
      c.self_id[g] = (uint8_t)self;
      c.role[g] = MRQ_ROLE_LEADER;
      c.lead[g] = (uint8_t)self;
      c.term[g] = 1 + rnd() % 8;
      c.vote[g] = self;
      c.last_index[g] = cs.big + rnd() % 40;
      c.last_term[g] = c.term[g];
      for (uint32_t r = 0; r < R; ++r) c.match[(uint64_t)r * G + g] = (g % 7 == 3 && r == (self % R)) ? 5 : c.last_index[g] - 1 - rnd() % 6;
      c.match[(uint64_t)(self - 1) * G + g] = c.last_index[g];
      c.committed[g] = c.last_index[g] - 8;
      c.term_start[g] = (g % 5 == 0) ? c.last_index[g] - 2 : c.committed[g] - 5;
      c.rto[g] = (uint16_t)(et + rnd() % et);
      c.el[g] = (uint16_t)(rnd() % et);
      c.hb[g] = (uint16_t)(rnd() % ht);
      if (cs.wild_timers) {
        if (g % 3 == 0) c.el[g] = (uint16_t)(et + rnd() % 64);  // at or above ElectionTick
        if (g % 4 == 1) c.hb[g] = (uint16_t)(ht + rnd() % (256 - ht));  // at or above HeartbeatTick (8 bits)
      }
    }
    orc_import(o, c.term.data(), c.vote.data(), c.committed.data(), c.last_index.data(), c.last_term.data(), c.term_start.data(),
               c.match.data(), c.role.data(), c.lead.data(), c.self_id.data(), nullptr, c.el.data(), c.hb.data(), c.rto.data());
    c.load(o);
  }
  import_from_oracle(e, c);
  e.tick_no[0] = cs.tick0;
  orc_set_tick_count(o, cs.tick0);
  mrq_trace_params p = preset(cs.soup ? 3 : cs.cfg);
  std::vector<uint8_t> type(G * R);
  std::vector<uint64_t> term(G * R), index(G * R), logterm(G * R), commit(G * R);
  std::vector<uint32_t> prop(G);
  std::vector<uint64_t> dev_base(e.gs, 0), enc_base(G, 0), base_term(e.gs, 0);
  std::vector<HostSlot> slots;
  for (uint32_t k = 0; k < K; ++k) slots.emplace_back(e.gs, R);
  std::vector<std::vector<uint32_t>> want_out(K, std::vector<uint32_t>(G));
  std::vector<std::vector<uint64_t>> want_commit(K + 1, std::vector<uint64_t>(G));
  static const uint8_t kTypes[] = {0, 0, 0, 3, 4, 4, 4, 4, 4, 5, 6, 6, 6, 8, 8, 9, 4 | 0x80, 6 | 0x80, 3 | 0x80};
  uint64_t x = seed * 77 + 5;
  auto rnd = [&]() { return x = mrq_mix64(x + 0x9E3779B97F4A7C15ull); };
  auto around = [](uint64_t v, int64_t d) -> uint64_t { return (d < 0 && v < (uint64_t)(-d)) ? 0 : v + (uint64_t)d; };
  bool bad = false;
  for (int t0 = 0; t0 < cs.T && !bad; t0 += (int)K) {
    const bool reset = t0 == cs.reset_at;
    if (t0 % cs.rebase_every == 0 || t0 == cs.also_rebase_at || reset) {  // mrq_set_packed_base / mrq_set_tick_count: ensure_wide(e, true)
      const TickArgs a0 = e.args(0, seed, et, ht, true);
      for (uint64_t g = 0; g < G; ++g) materialise_group(a0.s, ch.view(), dev_base.data(), e.gs, R, g, e.tick_no[0], et, ht);
      ch.invalidate();
      if (reset) {
        e.tick_no[0] = cs.reset_to;
        orc_set_tick_count(o, cs.reset_to);
      }
      c.load(o);
      for (uint64_t g = 0; g < G; ++g) {
        const uint64_t back = cs.soup ? 6 : 30;
        enc_base[g] = dev_base[g] = c.last_index[g] > back ? c.last_index[g] - back : 0;
        base_term[g] = c.term[g];
      }
    }
    c.load(o);
    want_commit[0] = c.committed;
    for (uint32_t k = 0; k < K; ++k) {
      HostSlot &s = slots[k];
      if (!cs.soup) {
        orc_gen_trace(o, &p, (uint64_t)(t0 + k), type.data(), term.data(), index.data(), logterm.data(), commit.data(), prop.data(), 1);
      } else {
        for (uint64_t g = 0; g < G; ++g) {
          for (uint32_t r = 0; r < R; ++r) {
            const uint64_t w = (uint64_t)r * G + g;
            uint8_t ty = kTypes[rnd() % sizeof kTypes];
            if (cs.edges) {  // compact-representable traffic aimed at the edges of the 64-entry window and of the log
              static const uint8_t kEdge[] = {4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 0, 0, 8, 9, 6, 4 | 0x80};
              ty = (rnd() % 16 == 0) ? kEdge[14 + rnd() % 6] : kEdge[rnd() % 14];
            }
            type[w] = ty;
            if ((ty & 0x0F) == 0) {
              term[w] = index[w] = logterm[w] = commit[w] = 0;
              continue;
            }
            const uint64_t u = rnd() % (cs.edges ? 4096 : 64);
            term[w] = around(c.term[g], u == 0 ? -2 : u == 1 ? -1 : u == 2 ? 1 : u == 3 ? 2 : 0);
            index[w] = around(c.last_index[g], (int64_t)(rnd() % 7) - 4);
            logterm[w] = around(c.last_term[g], (int64_t)(rnd() % 3) - 1);
            commit[w] = c.committed[g] + rnd() % 4;
            if (cs.edges) {
              const uint64_t wbase = enc_base[g], li = c.last_index[g];
              const uint64_t top = wbase + 63 < li ? wbase + 63 : li;
              switch (rnd() % 64) {
                case 0: index[w] = wbase + 64; break;
                case 1: index[w] = wbase ? wbase - 1 : 0; break;
                case 2: index[w] = (rnd() % 64 == 0) ? li + 1 : li; break;
                case 3: case 4: case 5: case 6: index[w] = wbase; break;
                case 7: case 8: case 9: case 10: index[w] = top; break;
                case 11: case 12: index[w] = li; break;
                default: index[w] = top > wbase ? wbase + rnd() % (top - wbase + 1) : wbase; break;
              }
              commit[w] = (rnd() % 4 == 0) ? wbase + rnd() % 64 : c.committed[g] + rnd() % 3;
              if (commit[w] > li) commit[w] = li;
            }
            if ((ty & 0x0F) == 3) {
              if (commit[w] > index[w]) commit[w] = index[w];
              if (index[w] == 0) logterm[w] = 0;
              if (logterm[w] > term[w]) logterm[w] = term[w];
            }
          }
          static const uint32_t kProps[] = {0, 0, 1, 4};
          prop[g] = kProps[rnd() % 4];
        }
      }
      std::fill(s.itype.begin(), s.itype.end(), 0xEE);
      for (uint64_t g = 0; g < G; ++g) {
        const uint32_t self = c.self_id[g];
        uint32_t min_ack = MRQ_P8_NO_ACK;
        for (uint32_t r = 0; r < R; ++r) {
          const uint32_t row = mrq_p8_row(r, self, R);
          if (row >= R - 1u) continue;
          const uint64_t w = (uint64_t)r * G + g, d = (uint64_t)r * e.gs + g;
          const uint8_t b = mrq_p8_encode(type[w], term[w], index[w], commit[w], enc_base[g], base_term[g]);
          s.word[(uint64_t)row * e.gs + g] = b;
          if (b == MRQ_P8_ESCAPE) {
            s.itype[d] = type[w];
            s.iterm[d] = term[w];
            s.iindex[d] = index[w];
            s.ilogterm[d] = logterm[w];
            s.icommit[d] = commit[w];
          } else if (b != 0 && (b & 3u) == 1u && (uint32_t)(b >> 2) < min_ack) {
            min_ack = b >> 2;
          }
        }
        enc_base[g] = mrq_p8_next_base(enc_base[g], min_ack);
        s.prop8[g] = (uint8_t)prop[g];
      }
      orc_tick(o, type.data(), term.data(), index.data(), logterm.data(), commit.data(), prop.data(), 1);
      c.load(o);
      want_out[k] = c.out;
      want_commit[k + 1] = c.committed;
    }
    const TickArgs a = e.args(0, seed, et, ht, true);
    std::vector<TickDesc> descs;
    for (uint32_t k = 0; k < K; ++k) descs.push_back(slots[k].desc());
    dispatch_ticks_clk(e, ch, a, descs, dev_base.data(), base_term.data(), where);
    if (e.tick_no[0] != orc_tick_count(o)) {
      std::printf("FAIL %s: tick number %llu, the oracle's %llu\n", where, (unsigned long long)e.tick_no[0],
                  (unsigned long long)orc_tick_count(o));
      ++failures;
      bad = true;
    }
    // ensure_wide(e, false): the real timers into meta, the compact state (and its phases) stays live
    for (uint64_t g = 0; g < G; ++g) materialise_group(a.s, ch.view(), dev_base.data(), e.gs, R, g, e.tick_no[0], et, ht);
    for (uint32_t k = 0; k < K && !bad; ++k)
      for (uint64_t g = 0; g < G; ++g) {
        const uint64_t adv = want_commit[k + 1][g] - want_commit[k][g];
        if (slots[k].out[g] != want_out[k][g] || slots[k].delta[g] != (adv > 255 ? 255 : adv)) {
          std::printf("FAIL %s tick %d group %llu: out %08x want %08x, commit advance %u want %llu\n", where, t0 + (int)k, (unsigned long long)g,
                      slots[k].out[g], want_out[k][g], slots[k].delta[g], (unsigned long long)adv);
          ++failures;
          bad = true;
          break;
        }
      }
    for (uint64_t g = 0; g < G && !bad; ++g)
      if (dev_base[g] != enc_base[g]) {
        std::printf("FAIL %s tick %d group %llu: device window %llu, frame builder's %llu\n", where, t0, (unsigned long long)g,
                    (unsigned long long)dev_base[g], (unsigned long long)enc_base[g]);
        ++failures;
        bad = true;
      }
    std::memcpy(e.out.data(), slots[K - 1].out.data(), e.gs * 4);
    if (!bad && !compare(e, c, where, (uint64_t)(t0 + K - 1))) bad = true;
  }
  uint64_t n_compact = 0;
  for (uint64_t g = 0; g < G; ++g) n_compact += ch.flag[g] & CF_COMPACT;
  std::printf("  %-62s %5d ticks  fast group-ticks %8llu (hot %8llu, compact leader %8llu)  general entries %7llu  compact now %llu/%llu\n",
              where, cs.T, (unsigned long long)ch.fast_ticks, (unsigned long long)ch.hot_ticks, (unsigned long long)ch.leader_ticks,
              (unsigned long long)ch.slow_entries, (unsigned long long)n_compact, (unsigned long long)G);
  if (!bad && !cs.soup && R > 1 && et > 2 && ch.fast_ticks < (uint64_t)cs.T * G / 4) {
    std::printf("FAIL %s: the compact fast path handled too little (%llu of %llu group-ticks)\n", where, (unsigned long long)ch.fast_ticks,
                (unsigned long long)((uint64_t)cs.T * G));
    ++failures;
  }
  if (!bad && cs.big && ch.leader_ticks == 0) {
    std::printf("FAIL %s: no compact leader ran on the fast path\n", where);
    ++failures;
  }
  orc_destroy(o);
}

}  // namespace

int main(int argc, char **) {
  const bool quick = argc > 1;  // any argument: the sanitizer build runs a smaller matrix
  const uint64_t q = quick ? 4 : 1;
  static_assert(sizeof(CompactOff) == sizeof(W), "the library's offset width is the one checked here");
  // the phase arithmetic itself, at the ends of the tick range
  for (uint64_t T : {0ull, 1ull, (1ull << 32) - 1, 1ull << 32, ~0ull - 1, ~0ull})
    for (uint32_t m : {1u, 2u, 3u, 10u, 255u, 2047u})
      for (uint32_t v = 0; v < m; v += 1 + m / 7) {
        const uint32_t p = clk_phase(v, T, m);
        if (p >= m || clk_value(p, T, m) != v || (T != ~0ull && clk_value(p, T + 1, m) != (v + 1) % m)) {
          std::printf("FAIL clk_phase/clk_value: v %u T %llu m %u -> p %u\n", v, (unsigned long long)T, m, p);
          ++failures;
        }
      }
  Case c;
  // traces: the steady trace, elections from a cold start, followers and heartbeats
  for (uint32_t R = 1; R <= 8; ++R) {
    c = Case{};
    c.G = 300 / q; c.R = R; c.cfg = 5; c.T = 224; c.rebase_every = 32; c.K = R % 2 ? 1 : 4;
    run_case_clk(c);
  }
  c = Case{}; c.G = 400 / q; c.cfg = 2; c.T = 300; c.rebase_every = 60; c.K = 5; run_case_clk(c);
  c = Case{}; c.G = 400 / q; c.R = 3; c.cfg = 6; c.T = 300; c.rebase_every = 30; c.K = 3; c.ht = 3; run_case_clk(c);
  c = Case{}; c.G = 400 / q; c.cfg = 3; c.T = 400; c.rebase_every = 1000; c.also_rebase_at = 64; c.K = 8; c.ht = 4; c.et = 7;
  run_case_clk(c);
  // ElectionTick and HeartbeatTick at their extremes
  for (uint32_t et : {1u, 2u, 2047u})
    for (uint32_t ht : {1u, 2u, 255u}) {
      c = Case{};
      c.G = 200 / q; c.cfg = et == 1 ? 2 : 3; c.T = 200; c.rebase_every = 64; c.also_rebase_at = 60; c.K = 6; c.et = et; c.ht = ht;
      run_case_clk(c);
    }
  // steady leaders imported with timers in range and out of range (el >= ET, hb >= HT): the latter stay wide for one tick
  for (uint32_t ht : {1u, 3u, 255u}) {
    c = Case{};
    c.G = 300 / q; c.cfg = 3; c.T = 240; c.rebase_every = 1000; c.K = 4; c.big = (1ull << 33) + 100; c.ht = ht; c.et = 9;
    run_case_clk(c);
    c.wild_timers = true; c.what = "imported timers out of range";
    run_case_clk(c);
  }
  // tick numbers around 2^32 and up to 2^64 - 1 (the last tick run is 2^64 - 2; the final count 2^64 - 1)
  for (uint32_t ht : {1u, 5u}) {
    c = Case{};
    c.G = 200 / q; c.cfg = 5; c.T = 240; c.rebase_every = 48; c.K = 8; c.et = 11; c.ht = ht;
    c.tick0 = (1ull << 32) - 100; c.what = "ticks across 2^32";
    run_case_clk(c);
    c.tick0 = ~0ull - 240; c.what = "ticks up to 2^64 - 1";
    run_case_clk(c);
    c.cfg = 3; c.big = 1ull << 20; c.wild_timers = true; c.tick0 = ~0ull - 240 - 7; c.K = 7; c.what = "leaders, ticks up to 2^64 - 1";
    run_case_clk(c);
  }
  // a tick-count reset in the middle of a run (backwards, then forwards past 2^32), compact state live at the time
  for (uint32_t ht : {1u, 3u}) {
    c = Case{};
    c.G = 300 / q; c.cfg = 3; c.T = 240; c.rebase_every = 1000; c.K = 5; c.et = 10; c.ht = ht; c.big = 1ull << 24;
    c.tick0 = 5000; c.reset_at = 120; c.reset_to = 17; c.what = "tick count reset";
    run_case_clk(c);
    c.reset_to = (1ull << 32) + 3; c.cfg = 5; c.big = 0; c.rebase_every = 40;
    run_case_clk(c);
  }
  // message soups and the window-edge soup
  for (uint32_t R : {2u, 3u, 5u, 8u}) {
    c = Case{};
    c.G = 120 / q + 8; c.R = R; c.cfg = 300 + R; c.T = 240; c.rebase_every = 8; c.K = R == 5 ? 4 : 1; c.soup = true; c.ht = R == 3 ? 2 : 1;
    run_case_clk(c);
  }
  for (uint32_t R : {2u, 3u, 5u, 8u}) {
    c = Case{};
    c.G = 160 / q + 8; c.R = R; c.cfg = 500 + R; c.T = 320; c.rebase_every = 16; c.K = R % 2 ? 1 : 4; c.soup = true; c.edges = true;
    c.big = 1ull << 22; c.ht = R == 5 ? 3 : 1;
    run_case_clk(c);
  }
  hot_path = false;  // the complete compact step alone
  c = Case{}; c.G = 300 / q; c.T = 224; c.K = 1; run_case_clk(c);
  c = Case{}; c.G = 300 / q; c.R = 3; c.cfg = 3; c.T = 300; c.rebase_every = 1000; c.also_rebase_at = 60; c.K = 4; c.ht = 3;
  run_case_clk(c);
  c = Case{}; c.G = 300 / q; c.cfg = 3; c.T = 240; c.rebase_every = 1000; c.K = 4; c.big = 1ull << 30; c.wild_timers = true; c.ht = 2;
  c.what = "imported timers out of range"; run_case_clk(c);
  hot_path = true;
  std::printf(failures ? "tick_clock_host_test: %d failure(s)\n" : "tick_clock_host_test: ok\n", failures);
  return failures ? 1 : 0;
}
