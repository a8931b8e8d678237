// change_feed_host_test.cpp — the change feed of the tick (mrq_set_change_capacity / mrq_sync_changes), compiled for the
// host from the device source and checked against the oracle.
//
// The general tick appends one record per group whose term, vote, role or lead it moved.  Every tick below, the records
// must equal the diff of the oracle's exports before and after that tick, field for field (tick, term, term_start, vote,
// role, lead, what), and there must be exactly one per changed group.  The feed is emitted by the general path alone, so
// the design rests on one invariant, checked here on every group-tick: whenever a fast function accepts a group
// (fast_group_tick, fast_group_tick8, compact_hot_step_clk, compact_step), the group's term, vote, role and lead are
// what they were before.  (compact_hot_pair takes neither the meta word nor the term, so it cannot move them.)
//
// Paths: the wide inbox through fast + general (mode 0) and general only (mode 1), the byte form through
// fast_group_tick8 / general_group_tick8 (mode 3), and the compact path of mode 4 in 1..8-tick batches (the per-group
// compact steps, then slow_group_ticks_c from the first tick that needs the general path).  Traces: elections from a cold
// start (preset 2), lag + churn (5), and message soups.  The harness (engine layout, oracle columns, presets) is
// tick_host_test.cpp's, included with its main() renamed.
//
//   change_feed_host_test          all cases;   exit code 0 and "change_feed_host_test: ok" on success
#define main tick_host_test_main
#include "tick_host_test.cpp"
#undef main

#include <algorithm>

namespace {

using W = uint16_t;

uint64_t fast_accepts = 0, records_checked = 0;

// the device's record buffer and counter, in host memory
struct HostFeed {
  std::vector<mrq_change> buf;
  unsigned long long count = 0;
  explicit HostFeed(uint64_t cap) : buf(cap) {}
  void attach(TickArgs &a) {
    a.changes = buf.data();
    a.change_count = &count;
    a.change_cap = buf.size();
  }
  std::vector<mrq_change> drain(uint64_t &lost) {  // what mrq_sync_changes returns
    const uint64_t n = count < buf.size() ? count : buf.size();
    std::vector<mrq_change> v(buf.begin(), buf.begin() + n);
    std::sort(v.begin(), v.end(), [](const mrq_change &x, const mrq_change &y) { return x.tick != y.tick ? x.tick < y.tick : x.group < y.group; });
    lost = count - n;
    count = 0;
    return v;
  }
};

// the records one tick must produce: the diff of two oracle exports
void expect_diff(const OracleCols &b, const OracleCols &a, uint64_t G, uint64_t tick, std::vector<mrq_change> &want) {
  for (uint64_t g = 0; g < G; ++g) {
    const uint32_t what = (a.term[g] != b.term[g] ? MRQ_CHANGE_TERM : 0u) | (a.vote[g] != b.vote[g] ? MRQ_CHANGE_VOTE : 0u) |
                          (a.role[g] != b.role[g] ? MRQ_CHANGE_ROLE : 0u) | (a.lead[g] != b.lead[g] ? MRQ_CHANGE_LEAD : 0u);
    if (!what) continue;
    mrq_change c{};
    c.tick = tick;
    c.term = a.term[g];
    c.term_start = a.role[g] == MRQ_ROLE_LEADER ? a.term_start[g] : kNoGate;
    c.group = (uint32_t)g;
    c.vote = (uint8_t)a.vote[g];
    c.role = a.role[g];
    c.lead = a.lead[g];
    c.what = (uint8_t)what;
    want.push_back(c);
  }
}

bool same(const mrq_change &x, const mrq_change &y) {
  return x.tick == y.tick && x.term == y.term && x.term_start == y.term_start && x.group == y.group && x.vote == y.vote &&
         x.role == y.role && x.lead == y.lead && x.what == y.what;
}

bool check_records(HostFeed &f, const std::vector<mrq_change> &want, const char *where) {
  uint64_t lost = 0;
  const std::vector<mrq_change> got = f.drain(lost);
  bool ok = lost == 0 && got.size() == want.size();
  for (size_t k = 0; ok && k < got.size(); ++k) ok = same(got[k], want[k]);
  if (!ok) {
    size_t k = 0;
    while (k < got.size() && k < want.size() && same(got[k], want[k])) ++k;
    std::printf("FAIL %s: %zu records (lost %llu), want %zu; first difference at %zu", where, got.size(), (unsigned long long)lost, want.size(), k);
    for (const auto *v : {&got, &want})
      if (k < v->size()) {
        const mrq_change &c = (*v)[k];
        std::printf("\n     tick %llu group %u term %llu term_start %llx vote %u role %u lead %u what %x", (unsigned long long)c.tick, c.group,
                    (unsigned long long)c.term, (unsigned long long)c.term_start, c.vote, c.role, c.lead, c.what);
      }
    std::printf("\n");
    ++failures;
    return false;
  }
  records_checked += got.size();
  return true;
}

// a fast function accepted a group: its term, vote, role and lead must be what they were
bool unmoved(uint64_t term0, uint64_t meta0, uint64_t term1, uint64_t meta1, const char *fn, const char *where, uint64_t tick, uint64_t g) {
  ++fast_accepts;
  if (term0 == term1 && ((meta0 ^ meta1) & 0x3FFu) == 0) return true;
  std::printf("FAIL %s tick %llu group %llu: %s accepted the group and moved its term / vote / role / lead\n", where, (unsigned long long)tick,
              (unsigned long long)g, fn);
  ++failures;
  return false;
}

// one tick's inbox, [R][G]: a trace tick of preset `p`, or the message soup of tick_host_test.cpp's run_soup
struct Frame {
  std::vector<uint8_t> type;
  std::vector<uint64_t> term, index, logterm, commit;
  std::vector<uint32_t> prop;
  Frame(uint64_t G, uint32_t R) : type(G * R), term(G * R), index(G * R), logterm(G * R), commit(G * R), prop(G) {}
  void trace(orc_engine *o, const mrq_trace_params &p, uint64_t t) {
    orc_gen_trace(o, &p, t, type.data(), term.data(), index.data(), logterm.data(), commit.data(), prop.data(), 1);
  }
  void soup(const OracleCols &c, uint64_t G, uint32_t R, uint64_t &x) {
    static const uint8_t kTypes[] = {0, 0, 0, 3, 4, 4, 4, 5, 6, 6, 6, 6, 6, 8, 9, 4 | 0x80, 6 | 0x80, 3 | 0x80};
    auto rnd = [&]() { return x = mrq_mix64(x + 0x9E3779B97F4A7C15ull); };
    auto around = [](uint64_t v, int64_t d) -> uint64_t { return (d < 0 && v < (uint64_t)(-d)) ? 0 : v + (uint64_t)d; };
    for (uint64_t g = 0; g < G; ++g) {
      for (uint32_t r = 0; r < R; ++r) {
        const uint64_t w = (uint64_t)r * G + g;
        const uint8_t ty = kTypes[rnd() % sizeof kTypes];
        type[w] = ty;
        if ((ty & 0x0F) == 0) {
          term[w] = index[w] = logterm[w] = commit[w] = 0;
          continue;
        }
        const uint64_t u = rnd() % 64;
        term[w] = around(c.term[g], u == 0 ? -2 : u == 1 ? -1 : u == 2 ? 1 : u == 3 ? 2 : 0);
        index[w] = around(c.last_index[g], (int64_t)(rnd() % 7) - 3);
        logterm[w] = around(c.last_term[g], (int64_t)(rnd() % 3) - 1);
        commit[w] = c.committed[g] + rnd() % 4;
        if ((ty & 0x0F) == 3) {  // a host-resolved MsgApp reports a log (include/mrq.h)
          if (commit[w] > index[w]) commit[w] = index[w];
          if (index[w] == 0) logterm[w] = 0;
          if (logterm[w] > term[w]) logterm[w] = term[w];
        }
      }
      static const uint32_t kProps[] = {0, 0, 1, 4};
      prop[g] = kProps[rnd() % 4];
    }
  }
  void tick_oracle(orc_engine *o) { orc_tick(o, type.data(), term.data(), index.data(), logterm.data(), commit.data(), prop.data(), 1); }
};

// byte frame of `f` for the engine's groups (what mrq_pack8 builds), escapes into the wide slot columns; slides enc_base
void encode8(const Frame &f, const OracleCols &c, uint64_t G, uint32_t R, uint64_t gs, uint64_t *enc_base, const uint64_t *base_term,
             uint8_t *word, uint8_t *prop8, const InboxView &slot) {
  for (uint64_t g = 0; g < G; ++g) {
    uint32_t min_ack = MRQ_P8_NO_ACK;
    for (uint32_t r = 0; r < R; ++r) {
      const uint32_t row = mrq_p8_row(r, c.self_id[g], R);
      const uint64_t w = (uint64_t)r * G + g, d = (uint64_t)r * gs + g;
      slot.type[d] = 0xEE;  // poison: what the tick reads must come from the byte or the escape
      if (row >= R - 1u) continue;
      const uint8_t b = mrq_p8_encode(f.type[w], f.term[w], f.index[w], f.commit[w], enc_base[g], base_term[g]);
      word[(uint64_t)row * gs + g] = b;
      if (b == MRQ_P8_ESCAPE) {
        slot.type[d] = f.type[w];
        slot.term[d] = f.term[w];
        slot.index[d] = f.index[w];
        slot.logterm[d] = f.logterm[w];
        slot.commit[d] = f.commit[w];
      } else if ((b & 3u) == 1u && (uint32_t)(b >> 2) < min_ack) {
        min_ack = b >> 2;
      }
    }
    enc_base[g] = mrq_p8_next_base(enc_base[g], min_ack);
    prop8[g] = (uint8_t)f.prop[g];
  }
}

// ---- the wide and byte-form paths: mode 0 (fast + general), 1 (general only), 3 (the byte form) -----------------------
template <int R>
void feed_tick(HostEngine &e, const TickArgs &a, const Inbox8 *b, int mode, const char *where) {
  const uint64_t tick = e.tick_no[0];
  for (uint64_t i = 0; i < e.G; ++i) {
    if (mode == 1) {
      general_group_tick<R>(a, i);
      continue;
    }
    const uint64_t t0 = e.term[i], m0 = e.meta[i];
    bool slow = false;
    uint32_t ev = 0;
    if (b)
      fast_group_tick8<R>(a, *b, i, slow, ev);
    else
      fast_group_tick<R>(a, i, slow, ev);
    if (!slow)
      unmoved(t0, m0, e.term[i], e.meta[i], b ? "fast_group_tick8" : "fast_group_tick", where, tick, i);
    else if (b)
      general_group_tick8<R>(a, *b, i);
    else
      general_group_tick<R>(a, i);
  }
  e.tick_no[0] += 1;
}

void run_wide(uint64_t G, uint32_t R, uint32_t cfg, int T, int mode, bool soup) {
  char where[96];
  std::snprintf(where, sizeof where, "feed mode %d G=%llu R=%u %s", mode, (unsigned long long)G, R, soup ? "soup" : cfg == 2 ? "election" : "lag+churn");
  const uint64_t seed = 0xFEED0000ull + cfg * 131 + R;
  const uint32_t et = soup ? 5 : 10;
  orc_engine *o = orc_create(G, R, 0, et, 1, seed, 0);
  HostEngine e(G, R);
  OracleCols before(G, R), after(G, R);
  before.load(o);
  import_from_oracle(e, before);
  HostFeed feed(G * 4);
  const mrq_trace_params p = preset(cfg);
  Frame f(G, R);
  std::vector<uint8_t> word(e.gs * (R > 1 ? R - 1 : 1)), prop8(e.gs);
  std::vector<uint64_t> base_index(e.gs), base_term(e.gs);
  uint64_t x = seed * 77 + 5, n_records = 0;
  for (int t = 0; t < T; ++t) {
    if (soup)
      f.soup(before, G, R, x);
    else
      f.trace(o, p, (uint64_t)t);
    const bool idle = !soup && mode != 3 && (t % 17) == 16;  // now and then an idle tick (timers only)
    TickArgs a = e.args(0, seed, et, 1, !idle);
    feed.attach(a);
    if (!idle) {
      for (uint32_t r = 0; r < R; ++r) {
        std::memcpy(&e.itype[(uint64_t)r * e.gs], &f.type[(uint64_t)r * G], G);
        std::memcpy(&e.iterm[(uint64_t)r * e.gs], &f.term[(uint64_t)r * G], G * 8);
        std::memcpy(&e.iindex[(uint64_t)r * e.gs], &f.index[(uint64_t)r * G], G * 8);
        std::memcpy(&e.ilogterm[(uint64_t)r * e.gs], &f.logterm[(uint64_t)r * G], G * 8);
        std::memcpy(&e.icommit[(uint64_t)r * e.gs], &f.commit[(uint64_t)r * G], G * 8);
      }
      std::memcpy(e.iprop.data(), f.prop.data(), G * 4);
      f.tick_oracle(o);
    } else {
      orc_tick(o, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 1);
    }
    Inbox8 b8{word.data(), prop8.data(), base_index.data(), base_term.data()};
    if (mode == 3) {  // the byte form, re-based every tick
      std::vector<uint64_t> enc(e.gs);
      for (uint64_t g = 0; g < G; ++g) {
        enc[g] = base_index[g] = before.last_index[g] > 2 ? before.last_index[g] - 2 : 0;
        base_term[g] = before.term[g];
      }
      encode8(f, before, G, R, e.gs, enc.data(), base_term.data(), word.data(), prop8.data(), a.in);
      for (uint64_t g = 0; g < G; ++g) e.iprop[g] = 0xEEEEEEEEu;
    }
    switch (R) {
#define FEED_CASE(N) \
  case N: feed_tick<N>(e, a, mode == 3 ? &b8 : nullptr, mode, where); break;
      FEED_CASE(1) FEED_CASE(2) FEED_CASE(3) FEED_CASE(4) FEED_CASE(5) FEED_CASE(6) FEED_CASE(7) FEED_CASE(8)
#undef FEED_CASE
    }
    after.load(o);
    std::vector<mrq_change> want;
    expect_diff(before, after, G, (uint64_t)t, want);
    n_records += want.size();
    if (!check_records(feed, want, where) || !compare(e, after, where, (uint64_t)t)) break;
    std::swap(before, after);
  }
  std::printf("  %-44s %4d ticks  records %7llu\n", where, T, (unsigned long long)n_records);
  if (R > 1 && n_records < (uint64_t)G) {
    std::printf("FAIL %s: only %llu records: the case does not exercise the feed\n", where, (unsigned long long)n_records);
    ++failures;
  }
  orc_destroy(o);
}

// ---- the compact path of tick mode 4 (16-bit offsets, leader timers on the clock), K-tick batches ----------------------
struct ClockCols {
  std::vector<uint8_t> flag;
  std::vector<W> commit, win, gate, match;
  std::vector<uint32_t> iblo, clk;
  std::vector<uint64_t> ibase;
  ClockCols(uint64_t gs, uint32_t R) : flag(gs, 0), commit(gs), win(gs), gate(gs), match(gs * R), iblo(gs), clk(gs), ibase(gs) {}
  CompactViewT<W> view() {
    return CompactViewT<W>{flag.data(), commit.data(), win.data(), gate.data(), iblo.data(), match.data(), ibase.data(), clk.data()};
  }
};

template <int R>
void feed_ticks_c(HostEngine &e, ClockCols &ch, const TickArgs &a, std::vector<TickDesc> &descs, uint64_t *base_index,
                  const uint64_t *base_term, const char *where, uint64_t &slow_entries) {
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
    const uint32_t flag = ch.flag[i], gate = ch.gate[i];
    const bool settled = compact_settled(flag, g.meta);
    uint32_t hb = ht > 1u ? clk_value((ch.clk[i] >> 16) & 0xFFu, tick0, ht) & 0xFFu : 0u;
    uint32_t t = 0;
    bool slow = false;
    for (; t < A.nticks; ++t) {
      const TickDesc &d = descs[t];
      uint32_t wb[R > 1 ? R - 1 : 1] = {0};
      for (int j = 0; j < R - 1; ++j) wb[j] = d.word8[(uint64_t)j * e.gs + i];
      uint32_t o, adv, dirty;
      const uint32_t np = d.prop8 ? d.prop8[i] : 0u;
      const uint64_t m0 = g.meta;
      const char *fn = "compact_hot_step_clk";
      slow = false;
      if (!compact_hot_step_clk<R, W>(g, settled, flag, wb, np, gate, ht, hb, 0, o, adv, dirty)) {
        fn = "compact_step";
        slow = compact_step<R, W>(g, flag, wb, np, gate, et, ht, o, adv, dirty, &hb);
      }
      if (slow) break;
      unmoved(0, m0, 0, g.meta, fn, where, tick0 + t, i);  // (the term is not compact state: it stays wide and untouched)
      d.out[i] = o;
      d.delta[i] = (uint8_t)(adv > 255u ? 255u : adv);
    }
    e.meta[i] = g.meta;
    ch.commit[i] = (W)g.commit;
    ch.win[i] = (W)g.win;
    for (int r = 0; r < R; ++r) ch.match[(uint64_t)r * e.gs + i] = (W)g.m[r];
    if (slow) {
      slow_group_ticks_c<R>(A, i, t);
      ++slow_entries;
    }
  }
  e.tick_no[0] += A.nticks;
}

void run_compact(uint64_t G, uint32_t R, uint32_t cfg, int T, uint32_t K, bool soup, int rebase_every) {
  char where[96];
  std::snprintf(where, sizeof where, "feed compact K=%u G=%llu R=%u %s", K, (unsigned long long)G, R, soup ? "soup" : cfg == 2 ? "election" : "lag+churn");
  const uint64_t seed = 0xFEEDC000ull + cfg * 131 + R;
  const uint32_t et = soup ? 5 : 10;
  orc_engine *o = orc_create(G, R, 0, et, 1, seed, 0);
  HostEngine e(G, R);
  ClockCols ch(e.gs, R);
  OracleCols before(G, R), after(G, R);
  before.load(o);
  import_from_oracle(e, before);
  HostFeed feed(G * K * 4);
  const mrq_trace_params p = preset(cfg);
  Frame f(G, R);
  std::vector<uint64_t> dev_base(e.gs, 0), enc_base(G, 0), base_term(e.gs, 0);
  std::vector<HostSlot> slots;
  for (uint32_t k = 0; k < K; ++k) slots.emplace_back(e.gs, R);
  uint64_t x = seed * 77 + 5, n_records = 0, slow_entries = 0;
  bool bad = false;
  for (int t0 = 0; t0 < T && !bad; t0 += (int)K) {
    if (t0 % rebase_every == 0) {  // mrq_set_packed_base: the wide columns are made exact, the compact copies die
      const TickArgs a0 = e.args(0, seed, et, 1, true);
      for (uint64_t g = 0; g < G; ++g) materialise_group(a0.s, ch.view(), dev_base.data(), e.gs, R, g, e.tick_no[0], et, 1);
      std::fill(ch.flag.begin(), ch.flag.end(), 0);
      for (uint64_t g = 0; g < G; ++g) {
        const uint64_t back = soup ? 6 : 30;
        enc_base[g] = dev_base[g] = before.last_index[g] > back ? before.last_index[g] - back : 0;
        base_term[g] = before.term[g];
      }
    }
    std::vector<mrq_change> want;
    for (uint32_t k = 0; k < K; ++k) {  // K ticks: frames built as the oracle advances, one diff per tick
      HostSlot &s = slots[k];
      if (soup)
        f.soup(before, G, R, x);
      else
        f.trace(o, p, (uint64_t)(t0 + k));
      encode8(f, before, G, R, e.gs, enc_base.data(), base_term.data(), s.word.data(), s.prop8.data(), s.desc().in);
      f.tick_oracle(o);
      after.load(o);
      expect_diff(before, after, G, (uint64_t)(t0 + k), want);
      std::swap(before, after);
    }
    TickArgs a = e.args(0, seed, et, 1, true);
    feed.attach(a);
    std::vector<TickDesc> descs;
    for (uint32_t k = 0; k < K; ++k) descs.push_back(slots[k].desc());
    switch (R) {
#define FEED_CASE(N) \
  case N: feed_ticks_c<N>(e, ch, a, descs, dev_base.data(), base_term.data(), where, slow_entries); break;
      FEED_CASE(1) FEED_CASE(2) FEED_CASE(3) FEED_CASE(4) FEED_CASE(5) FEED_CASE(6) FEED_CASE(7) FEED_CASE(8)
#undef FEED_CASE
    }
    n_records += want.size();
    if (!check_records(feed, want, where)) bad = true;
    for (uint64_t g = 0; g < G; ++g) materialise_group(a.s, ch.view(), dev_base.data(), e.gs, R, g, e.tick_no[0], et, 1);
    std::memcpy(e.out.data(), slots[K - 1].out.data(), e.gs * 4);
    if (!bad && !compare(e, before, where, (uint64_t)(t0 + K - 1))) bad = true;
  }
  std::printf("  %-44s %4d ticks  records %7llu  general entries %7llu\n", where, T, (unsigned long long)n_records, (unsigned long long)slow_entries);
  if (R > 1 && n_records < (uint64_t)G) {
    std::printf("FAIL %s: only %llu records: the case does not exercise the feed\n", where, (unsigned long long)n_records);
    ++failures;
  }
  orc_destroy(o);
}

// A capacity below the change count: the first `cap` appended records are written (each one genuine), the rest counted.
void run_overflow() {
  const char *where = "feed overflow";
  const uint64_t G = 300;
  const uint32_t R = 5;
  orc_engine *o = orc_create(G, R, 0, 10, 1, 0xFEED0F10ull, 0);
  HostEngine e(G, R);
  OracleCols before(G, R), after(G, R);
  before.load(o);
  import_from_oracle(e, before);
  HostFeed feed(37);
  uint64_t total = 0;
  std::vector<mrq_change> want;
  for (int t = 0; t < 40; ++t) {  // idle ticks from term 0: every group campaigns when its timeout fires
    orc_tick(o, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 1);
    TickArgs a = e.args(0, 0xFEED0F10ull, 10, 1, false);
    feed.attach(a);
    feed_tick<5>(e, a, nullptr, 0, where);
    after.load(o);
    expect_diff(before, after, G, (uint64_t)t, want);
    std::swap(before, after);
  }
  total = want.size();
  uint64_t lost = 0;
  const std::vector<mrq_change> got = feed.drain(lost);
  bool ok = got.size() == 37 && lost == total - 37;
  for (const mrq_change &c : got) ok = ok && std::any_of(want.begin(), want.end(), [&](const mrq_change &w) { return same(w, c); });
  if (!ok || total <= 37) {
    std::printf("FAIL %s: %zu records, lost %llu, of %llu changes\n", where, got.size(), (unsigned long long)lost, (unsigned long long)total);
    ++failures;
  }
  std::printf("  %-44s %llu changes, capacity 37: lost %llu\n", where, (unsigned long long)total, (unsigned long long)lost);
  orc_destroy(o);
}

}  // namespace

int main(int argc, char **) {
  const bool quick = argc > 1;  // any argument: the sanitizer builds run a smaller matrix
  const uint64_t k = quick ? 3 : 1;
  for (uint32_t R = 1; R <= 8; ++R) {
    run_wide(240 / k, R, 2, 200, 0, false);  // elections from a cold start
    run_wide(200 / k, R, 5, 240, R % 2, false);  // lag + churn
    run_compact(200 / k, R, 5, 224, 1 + (R - 1) % 8, false, 32);  // batches of 1..8 ticks
  }
  for (uint32_t R : {2u, 3u, 5u, 8u}) {
    run_wide(120 / k + 8, R, 300 + R, 200, 0, true);  // message soups
    run_wide(120 / k + 8, R, 300 + R, 200, 3, true);
    run_compact(120 / k + 8, R, 300 + R, 200, R == 5 ? 4 : 1, true, 8);
  }
  for (uint32_t R : {3u, 5u, 7u}) {
    run_wide(200 / k, R, 5, 200, 3, false);
    run_compact(240 / k, R, 2, 240, 5, false, 60);
    run_compact(200 / k, R, 5, 240, 8, false, 40);
  }
  run_overflow();
  std::printf("  fast-path accepts checked: %llu   records checked: %llu\n", (unsigned long long)fast_accepts, (unsigned long long)records_checked);
  std::printf(failures ? "change_feed_host_test: %d failure(s)\n" : "change_feed_host_test: ok\n", failures);
  return failures ? 1 : 0;
}
