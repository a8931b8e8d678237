// tick_pair_clock_host_test.cpp — every case of tick_clock_host_test.cpp, run the way tick_fast4_kernel runs a launch:
// groups in pairs held as 16x2 pair words, a pair of settled leaders stepped by compact_hot_pair, a pair that declines
// unpacked into the per-group steps and repacked.  Traces, message soups, the window-edge soup, the timer extremes,
// imported timers, tick numbers near 2^32 and 2^64 - 1, the tick-count reset and the hot step switched off must all
// still equal the oracle.
//
// The cases, the oracle comparison and main() are tick_clock_host_test.cpp's, included unchanged; only its per-launch
// loop is replaced.  Its callers name it `host_ticks_clk<R>(...)`, while its definition is `host_ticks_clk(...)`:
// the function-like macro below renames that definition alone (a macro name followed by '<' is not an invocation), so
// the callers reach the pair-structured host_ticks_clk declared here.
//
//   tick_pair_clock_host_test          all cases;   exit code 0 and "tick_clock_host_test: ok" on success, then the
//                                                   number of group-ticks the pair step ran
#include <cstdint>
#include <cstdio>

namespace {
template <int R, class... A>
void host_ticks_clk(A &...args);  // the pair-structured launch, defined below
uint64_t pair_hot_ticks = 0;
struct PairReport {
  ~PairReport() { std::printf("  the pair step ran %llu group-ticks\n", (unsigned long long)pair_hot_ticks); }
} pair_report;
}  // namespace

#define host_ticks_clk(...) host_ticks_clk_per_group(__VA_ARGS__)
#include "tick_clock_host_test.cpp"
#undef host_ticks_clk

namespace {

// The launch structured as tick_fast4_kernel runs it: groups in pairs (2p, 2p + 1) held as 16x2 pair words, the
// bytes of a pair at lanes 0/1 or 2/3 of the quad's frame words.  A pair of settled leaders tries compact_hot_pair; a
// pair that declines unpacks and runs the per-group steps as tick_clock_host_test.cpp does, then repacks.
template <int R>
void host_ticks_pairs(HostEngine &e, ClockHost &ch, const TickArgs &a, std::vector<TickDesc> &descs, uint64_t *base_index,
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
  constexpr int NW = R > 1 ? R - 1 : 1;
  for (uint64_t i0 = 0; i0 < e.G; i0 += 2) {
    const int hi = (int)((i0 >> 1) & 1u);  // the pair's place in its quad
    uint64_t meta[2] = {0, 0};
    uint32_t flag[2] = {0, 0}, gate[2] = {0, 0}, hbw = 0, cm2 = 0, wn2 = 0, gt2 = 0, m2[R] = {0}, stopped = 0, settled = 0, t_slow[2] = {0, 0};
    bool leader[2] = {false, false};
    for (int h = 0; h < 2; ++h) {
      const uint64_t i = i0 + h;
      if (i >= e.G) {  // padding
        stopped |= 1u << h;
        continue;
      }
      meta[h] = e.meta[i];
      flag[h] = ch.flag[i];
      gate[h] = ch.gate[i];
      cm2 |= (uint32_t)ch.commit[i] << (16 * h);
      wn2 |= (uint32_t)ch.win[i] << (16 * h);
      for (int r = 0; r < R; ++r) m2[r] |= (uint32_t)ch.match[(uint64_t)r * e.gs + i] << (16 * h);
      settled |= compact_settled(flag[h], meta[h]) ? 1u << h : 0u;
      if (!(flag[h] & CF_GATE_OPEN)) gt2 |= gate[h] << (16 * h);
      leader[h] = (flag[h] & CF_COMPACT) && meta_unpack(meta[h]).role == MRQ_ROLE_LEADER;
      if (ht > 1u) hbw |= (clk_value((ch.clk[i] >> 16) & 0xFFu, tick0, ht) & 0xFFu) << (8 * h);
    }
    for (uint32_t t = 0; t < A.nticks && stopped != 3u; ++t) {
      const TickDesc &d = descs[t];
      uint32_t wq[NW] = {0}, pq = 0;
      for (int h = 0; h < 2; ++h) {
        if (i0 + h >= e.G) continue;
        const int sh = 8 * (2 * hi + h);
        for (int j = 0; j < R - 1; ++j) wq[j] |= (uint32_t)d.word8[(uint64_t)j * e.gs + i0 + h] << sh;
        pq |= (uint32_t)(d.prop8 ? d.prop8[i0 + h] : 0u) << sh;
      }
      uint32_t q2, o2, pd;
      if (hot_path && (settled & ~stopped) == 3u && compact_hot_pair<R>(cm2, wn2, m2, gt2, wq, pq, hi, q2, o2, pd)) {
        for (int h = 0; h < 2; ++h) {
          d.out[i0 + h] = ((o2 >> (16 * h)) & 0xFFFFu) | clk_heartbeat(ht, hbw, 8 * h);
          const uint32_t q = (q2 >> (16 * h)) & 0xFFFFu;
          d.delta[i0 + h] = (uint8_t)(q > 255u ? 255u : q);
        }
        ch.fast_ticks += 2;
        ch.hot_ticks += 2;
        ch.leader_ticks += 2;
        pair_hot_ticks += 2;
        continue;
      }
      for (int h = 0; h < 2; ++h) {
        if (stopped & (1u << h)) continue;
        const uint64_t i = i0 + h;
        CGroup<R> g;
        g.meta = meta[h];
        g.commit = (cm2 >> (16 * h)) & 0xFFFFu;
        g.win = (wn2 >> (16 * h)) & 0xFFFFu;
        for (int r = 0; r < R; ++r) g.m[r] = (m2[r] >> (16 * h)) & 0xFFFFu;
        uint32_t wb[NW] = {0};
        for (int j = 0; j < R - 1; ++j) wb[j] = (wq[j] >> (8 * (2 * hi + h))) & 0xFFu;
        const uint32_t np = (pq >> (8 * (2 * hi + h))) & 0xFFu;
        uint32_t o, adv, dirty;
        bool slow = false;
        if (!hot_path || !compact_hot_step_clk<R, W>(g, (settled >> h) & 1u, flag[h], wb, np, gate[h], ht, hbw, 8 * h, o, adv, dirty)) {
          uint32_t hb = (hbw >> (8 * h)) & 0xFFu;
          slow = compact_step<R, W>(g, flag[h], wb, np, gate[h], et, ht, o, adv, dirty, &hb);
          hbw = (hbw & ~(0xFFu << (8 * h))) | ((hb & 0xFFu) << (8 * h));
        } else {
          ++ch.hot_ticks;
        }
        if (slow) {  // (compact_step left g untouched)
          stopped |= 1u << h;
          t_slow[h] = t;
          continue;
        }
        if (leader[h] && (dirty & CD_META)) {
          std::printf("FAIL %s tick %llu group %llu: a compact leader marked its meta word dirty\n", where,
                      (unsigned long long)(tick0 + t), (unsigned long long)i);
          ++failures;
        }
        meta[h] = g.meta;
        cm2 = __byte_perm(cm2, g.commit, h ? 0x5410u : 0x3254u);
        wn2 = __byte_perm(wn2, g.win, h ? 0x5410u : 0x3254u);
        for (int r = 0; r < R; ++r) m2[r] = __byte_perm(m2[r], g.m[r], h ? 0x5410u : 0x3254u);
        d.out[i] = o;
        d.delta[i] = (uint8_t)(adv > 255u ? 255u : adv);
        ++ch.fast_ticks;
        ch.leader_ticks += leader[h];
      }
    }
    for (int h = 0; h < 2; ++h) {
      const uint64_t i = i0 + h;
      if (i >= e.G) continue;
      e.meta[i] = meta[h];
      ch.commit[i] = (W)(cm2 >> (16 * h));
      ch.win[i] = (W)(wn2 >> (16 * h));
      for (int r = 0; r < R; ++r) ch.match[(uint64_t)r * e.gs + i] = (W)(m2[r] >> (16 * h));
      if (stopped & (1u << h)) {
        slow_group_ticks_c<R>(A, i, t_slow[h]);
        ++ch.slow_entries;
      }
    }
  }
  e.tick_no[0] += A.nticks;
}


template <int R, class... A>
void host_ticks_clk(A &...args) {
  host_ticks_pairs<R>(args...);
}

}  // namespace
