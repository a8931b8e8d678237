// group_state_host_test.cpp — the state of a list of groups (mrq_export_groups / mrq_import_groups), compiled for the host
// from the device source and checked against the oracle.
//
// export_group_row and import_group_row are the per-thread bodies of export_groups_kernel and import_groups_kernel.  Here
// they run over the engine's layout in host memory, in the library's form of tick mode 4 (16-bit offsets, leader timers on
// the clock), after traces (lag + churn, elections from a cold start) and message soups have driven the groups through
// the mode-4 per-group functions (compact_hot_step_clk, compact_step, then slow_group_ticks_c) into mixed states: compact
// leaders with clock phases, closed commit gates, far-behind followers, groups with flag 0, strict leaders.  Then:
//   - export rows for random lists with duplicates equal the rows of materialise_group over a copy of every group +
//     meta unpacked (what mrq_export_state returns), and no state or compact array changes by a single byte;
//   - after an import of rows (other groups' rows with their self ids, leaders with out-of-range timers, acks beyond
//     lastIndex, lastIndex beyond the 16-bit span), the compact arrays and wide columns of every untouched group are
//     byte-identical, and the ticks that follow equal the oracle fed the same rows through orc_import, after every batch
//     (state) and every tick (out words, commit advances).
// The harness (engine layout, oracle columns, presets) is tick_host_test.cpp's, included with its main() renamed.
//
//   group_state_host_test          all cases;   exit code 0 and "group_state_host_test: ok" on success
#define main tick_host_test_main
#include "tick_host_test.cpp"
#undef main

#include <algorithm>

namespace {

using W = uint16_t;

uint64_t rows_checked = 0, groups_imported = 0;
uint64_t seen_clock_leaders = 0, seen_flag0 = 0, seen_strict = 0, seen_closed_gate = 0;

struct ClockCols {  // the compact columns in the library's form
  std::vector<uint8_t> flag;
  std::vector<W> commit, win, gate, match;
  std::vector<uint32_t> iblo, clk;
  std::vector<uint64_t> ibase;
  ClockCols(uint64_t gs, uint32_t R) : flag(gs, 0), commit(gs), win(gs), gate(gs), match(gs * R), iblo(gs), clk(gs), ibase(gs) {}
  CompactViewT<W> view() {
    return CompactViewT<W>{flag.data(), commit.data(), win.data(), gate.data(), iblo.data(), match.data(), ibase.data(), clk.data()};
  }
  bool operator==(const ClockCols &o) const {
    return flag == o.flag && commit == o.commit && win == o.win && gate == o.gate && match == o.match && iblo == o.iblo && clk == o.clk &&
           ibase == o.ibase;
  }
};

// one tick's inbox, [R][G]: a trace tick, or a message soup around the current state
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

// byte frame of `f` (what mrq_pack8 builds), escapes into the wide slot columns; slides enc_base
void encode8(const Frame &f, const OracleCols &c, uint64_t G, uint32_t R, uint64_t gs, uint64_t *enc_base, const uint64_t *base_term,
             uint8_t *word, uint8_t *prop8, const InboxView &slot) {
  for (uint64_t g = 0; g < G; ++g) {
    uint32_t min_ack = MRQ_P8_NO_ACK;
    for (uint32_t r = 0; r < R; ++r) {
      const uint32_t row = mrq_p8_row(r, c.self_id[g], R);
      const uint64_t w = (uint64_t)r * G + g, d = (uint64_t)r * gs + g;
      slot.type[d] = 0xEE;
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

// one K-tick mode-4 launch, one "thread" per group: the compact steps, then the general path from the first tick that
// needs it (as the quad kernel + tick_slow4_kernel)
template <int R>
void ticks_c(HostEngine &e, ClockCols &ch, const TickArgs &a, std::vector<TickDesc> &descs, uint64_t *base_index, const uint64_t *base_term) {
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
      slow = false;
      if (!compact_hot_step_clk<R, W>(g, settled, flag, wb, np, gate, ht, hb, 0, o, adv, dirty))
        slow = compact_step<R, W>(g, flag, wb, np, gate, et, ht, o, adv, dirty, &hb);
      if (slow) break;
      d.out[i] = o;
      d.delta[i] = (uint8_t)(adv > 255u ? 255u : adv);
    }
    e.meta[i] = g.meta;
    ch.commit[i] = (W)g.commit;
    ch.win[i] = (W)g.win;
    for (int r = 0; r < R; ++r) ch.match[(uint64_t)r * e.gs + i] = (W)g.m[r];
    if (slow) slow_group_ticks_c<R>(A, i, t);
  }
  e.tick_no[0] += A.nticks;
}

struct Rows {  // n-row host columns, GroupRows layout
  std::vector<uint64_t> term, vote, committed, last_index, last_term, term_start, match;
  std::vector<uint8_t> role, lead, self_id, votes;
  std::vector<uint16_t> el, hb, rto;
  Rows(uint64_t n, uint32_t R)
      : term(n), vote(n), committed(n), last_index(n), last_term(n), term_start(n), match(n * R), role(n), lead(n), self_id(n),
        votes(n * R), el(n), hb(n), rto(n) {}
  GroupRows view() {
    return GroupRows{term.data(), vote.data(), committed.data(), last_index.data(), last_term.data(), term_start.data(), match.data(),
                     role.data(), lead.data(), self_id.data(), votes.data(), el.data(), hb.data(), rto.data()};
  }
};

struct Snapshot {  // every array the two calls could touch
  std::vector<uint64_t> term, meta, last_index, last_term, committed, term_start, match, base;
  ClockCols ch;
  Snapshot(const HostEngine &e, const ClockCols &c, const std::vector<uint64_t> &b)
      : term(e.term), meta(e.meta), last_index(e.last_index), last_term(e.last_term), committed(e.committed), term_start(e.term_start),
        match(e.match), base(b), ch(c) {}
};

bool fail_at(const char *where, const char *what, uint64_t g) {
  std::printf("FAIL %s: %s (group %llu)\n", where, what, (unsigned long long)g);
  ++failures;
  return false;
}

// export rows of a random list with duplicates against materialise_group over a copy of every group
bool check_export(HostEngine &e, ClockCols &ch, std::vector<uint64_t> &dev_base, uint32_t et, uint64_t &x, const char *where) {
  const uint64_t G = e.G, gs = e.gs;
  const uint32_t R = e.R;
  auto rnd = [&]() { return x = mrq_mix64(x + 0x9E3779B97F4A7C15ull); };
  const uint64_t n = 1 + rnd() % (2 * G);
  std::vector<uint64_t> groups(n);
  for (auto &g : groups) g = rnd() % G;
  groups[0] = 0;
  if (n > 1) groups[n - 1] = G - 1;
  if (n > 3) groups[2] = groups[1];
  const Snapshot before(e, ch, dev_base);
  const TickArgs a = e.args(0, 0, et, 1, false);
  Rows rows(n, R);
  const GroupRows o = rows.view();
  for (uint64_t k = 0; k < n; ++k) export_group_row(a.s, ch.view(), true, gs, R, groups[k], e.tick_no[0], et, 1, o, n, k);
  if (!(e.term == before.term && e.meta == before.meta && e.last_index == before.last_index &&
        e.last_term == before.last_term && e.committed == before.committed && e.term_start == before.term_start &&
        e.match == before.match && dev_base == before.base && ch == before.ch))
    return fail_at(where, "export_group_row changed engine state", 0);
  // what mrq_export_state returns: every group materialised (on a copy), meta unpacked
  HostEngine w = e;
  ClockCols wc = ch;
  std::vector<uint64_t> wb = dev_base;
  const TickArgs aw = w.args(0, 0, et, 1, false);
  for (uint64_t g = 0; g < G; ++g) materialise_group(aw.s, wc.view(), wb.data(), gs, R, g, e.tick_no[0], et, 1);
  for (uint64_t k = 0; k < n; ++k) {
    const uint64_t g = groups[k];
    const Meta m = meta_unpack(w.meta[g]);
    bool ok = rows.term[k] == w.term[g] && rows.vote[k] == m.vote && rows.committed[k] == w.committed[g] &&
              rows.last_index[k] == w.last_index[g] && rows.last_term[k] == w.last_term[g] && rows.term_start[k] == w.term_start[g] &&
              rows.role[k] == m.role && rows.lead[k] == m.lead && rows.self_id[k] == m.self && rows.el[k] == m.elapsed &&
              rows.hb[k] == m.hb && rows.rto[k] == m.rto;
    for (uint32_t r = 0; ok && r < R; ++r)
      ok = rows.match[(uint64_t)r * n + k] == w.match[(uint64_t)r * gs + g] && rows.votes[(uint64_t)r * n + k] == ((m.votes >> (2 * r)) & 3u);
    if (!ok) return fail_at(where, "export row differs from the materialised group", g);
    // what the mixed state holds
    const Meta mc = meta_unpack(e.meta[g]);
    if (ch.flag[g] & CF_COMPACT) {
      if (mc.role == MRQ_ROLE_LEADER) ++seen_clock_leaders;
      if (mc.role == MRQ_ROLE_LEADER && !(ch.flag[g] & CF_GATE_OPEN)) ++seen_closed_gate;
    } else {
      ++seen_flag0;
    }
    if (mc.strict) ++seen_strict;
  }
  rows_checked += n;
  return true;
}

// rows to import: the oracle's rows of the listed groups, perturbed
void make_rows(const OracleCols &c, uint64_t G, uint32_t R, uint32_t et, const std::vector<uint64_t> &groups, Rows &rows, uint64_t &x) {
  auto rnd = [&]() { return x = mrq_mix64(x + 0x9E3779B97F4A7C15ull); };
  const uint64_t n = groups.size();
  for (uint64_t k = 0; k < n; ++k) {
    const uint32_t sel = (uint32_t)(rnd() % 5);
    const uint64_t g = sel == 0 ? rnd() % G : groups[k];  // 0: another group's row, self id included (a slot reused)
    rows.term[k] = c.term[g];
    rows.vote[k] = c.vote[g];
    rows.committed[k] = c.committed[g];
    rows.last_index[k] = c.last_index[g];
    rows.last_term[k] = c.last_term[g];
    rows.term_start[k] = c.term_start[g];
    rows.role[k] = c.role[g];
    rows.lead[k] = c.lead[g];
    rows.self_id[k] = c.self_id[g];
    rows.el[k] = c.el[g];
    rows.hb[k] = c.hb[g];
    rows.rto[k] = c.rto[g];
    for (uint32_t r = 0; r < R; ++r) {
      rows.match[(uint64_t)r * n + k] = c.match[(uint64_t)r * G + g];
      rows.votes[(uint64_t)r * n + k] = c.votes[(uint64_t)r * G + g];
    }
    const bool leader = rows.role[k] == MRQ_ROLE_LEADER;
    const uint32_t self = rows.self_id[k];
    if (sel == 1 && leader) {  // timers out of range: the group stays wide until a general tick normalises them
      rows.el[k] = (uint16_t)(et + 3);
      rows.hb[k] = 2;
    } else if (sel == 2 && leader && R > 1) {  // an ack beyond lastIndex: strict
      rows.match[(uint64_t)(self % R) * n + k] = rows.last_index[k] + 2;
    } else if (sel == 3) {  // lastIndex beyond the 16-bit span of the offsets (the entries keep the last entry's term)
      rows.last_index[k] += 70000;
      if (leader) rows.match[(uint64_t)(self - 1) * n + k] = rows.last_index[k];
    }
  }
}

// import rows into a unique list; untouched groups must keep every byte; the oracle gets the same rows
bool do_import(HostEngine &e, ClockCols &ch, std::vector<uint64_t> &dev_base, const std::vector<uint64_t> &base_term, orc_engine *o,
               OracleCols &c, uint32_t et, uint64_t &x, const char *where) {
  const uint64_t G = e.G, gs = e.gs;
  const uint32_t R = e.R;
  auto rnd = [&]() { return x = mrq_mix64(x + 0x9E3779B97F4A7C15ull); };
  std::vector<uint64_t> groups;
  std::vector<uint8_t> listed(G, 0);
  for (uint64_t g = 0; g < G; ++g)
    if (g == 0 || g == G - 1 || rnd() % 4 == 0) groups.push_back(g);
  for (uint64_t k = groups.size(); k > 1; --k) std::swap(groups[k - 1], groups[rnd() % k]);  // any order
  for (uint64_t g : groups) listed[g] = 1;
  const uint64_t n = groups.size();
  Rows rows(n, R);
  make_rows(c, G, R, et, groups, rows, x);
  const Snapshot before(e, ch, dev_base);
  const TickArgs a = e.args(0, 0, et, 1, false);
  for (uint64_t k = 0; k < n; ++k)
    import_group_row(a.s, ch.view(), true, dev_base.data(), base_term.data(), gs, R, groups[k], e.tick_no[0], et, 1, rows.view(), n, k);
  for (uint64_t g = 0; g < G; ++g) {
    if (listed[g]) continue;
    bool same = e.term[g] == before.term[g] && e.meta[g] == before.meta[g] && e.last_index[g] == before.last_index[g] &&
                e.last_term[g] == before.last_term[g] && e.committed[g] == before.committed[g] && e.term_start[g] == before.term_start[g] &&
                dev_base[g] == before.base[g] && ch.flag[g] == before.ch.flag[g] && ch.commit[g] == before.ch.commit[g] &&
                ch.win[g] == before.ch.win[g] && ch.gate[g] == before.ch.gate[g] && ch.iblo[g] == before.ch.iblo[g] &&
                ch.clk[g] == before.ch.clk[g] && ch.ibase[g] == before.ch.ibase[g];
    for (uint32_t r = 0; same && r < R; ++r)
      same = e.match[(uint64_t)r * gs + g] == before.match[(uint64_t)r * gs + g] && ch.match[(uint64_t)r * gs + g] == before.ch.match[(uint64_t)r * gs + g];
    if (!same) return fail_at(where, "import_group_row touched a group that is not listed", g);
  }
  for (uint64_t k = 0; k < n; ++k) {  // the oracle: the same rows through import_state
    const uint64_t g = groups[k];
    c.term[g] = rows.term[k];
    c.vote[g] = rows.vote[k];
    c.committed[g] = rows.committed[k];
    c.last_index[g] = rows.last_index[k];
    c.last_term[g] = rows.last_term[k];
    c.term_start[g] = rows.term_start[k];
    c.role[g] = rows.role[k];
    c.lead[g] = rows.lead[k];
    c.self_id[g] = rows.self_id[k];
    c.el[g] = rows.el[k];
    c.hb[g] = rows.hb[k];
    c.rto[g] = rows.rto[k];
    for (uint32_t r = 0; r < R; ++r) {
      c.match[(uint64_t)r * G + g] = rows.match[(uint64_t)r * n + k];
      c.votes[(uint64_t)r * G + g] = rows.votes[(uint64_t)r * n + k];
    }
  }
  orc_import(o, c.term.data(), c.vote.data(), c.committed.data(), c.last_index.data(), c.last_term.data(), c.term_start.data(), c.match.data(),
             c.role.data(), c.lead.data(), c.self_id.data(), c.votes.data(), c.el.data(), c.hb.data(), c.rto.data());
  c.load(o);
  groups_imported += n;
  return true;
}

void run(uint64_t G, uint32_t R, uint32_t cfg, int T, uint32_t K, bool soup) {
  char where[96];
  std::snprintf(where, sizeof where, "groups K=%u G=%llu R=%u %s", K, (unsigned long long)G, R, soup ? "soup" : cfg == 2 ? "election" : "lag+churn");
  const uint64_t seed = 0x6E0E0000ull + cfg * 131 + R;
  const uint32_t et = soup ? 5 : 10;
  orc_engine *o = orc_create(G, R, 0, et, 1, seed, 0);
  HostEngine e(G, R);
  ClockCols ch(e.gs, R);
  OracleCols c(G, R);
  c.load(o);
  import_from_oracle(e, c);
  const mrq_trace_params p = preset(cfg);
  Frame f(G, R);
  std::vector<uint64_t> dev_base(e.gs, 0), enc_base(G, 0), base_term(e.gs, 0);
  std::vector<HostSlot> slots;
  for (uint32_t k = 0; k < K; ++k) slots.emplace_back(e.gs, R);
  uint64_t x = seed * 77 + 5;
  const int rebase_every = soup ? 8 * (int)K : 40 * (int)K;
  bool bad = false;
  for (int t0 = 0; t0 < T && !bad; t0 += (int)K) {
    if (t0 % rebase_every == 0) {  // mrq_set_packed_base: the wide columns are made exact, the compact copies die
      const TickArgs a0 = e.args(0, seed, et, 1, true);
      for (uint64_t g = 0; g < G; ++g) materialise_group(a0.s, ch.view(), dev_base.data(), e.gs, R, g, e.tick_no[0], et, 1);
      std::fill(ch.flag.begin(), ch.flag.end(), 0);
      for (uint64_t g = 0; g < G; ++g) {
        const uint64_t back = soup ? 6 : 30;
        enc_base[g] = dev_base[g] = c.last_index[g] > back ? c.last_index[g] - back : 0;
        base_term[g] = c.term[g];
      }
      // the first batch after a re-base compacts every group (compact_all_kernel)
      const TickArgs a1 = e.args(0, seed, et, 1, true);
      for (uint64_t g = 0; g < G; ++g) compact_group(a1.s, ch.view(), dev_base.data(), base_term.data(), e.gs, R, g, e.tick_no[0], et, 1);
    }
    const int phase = (t0 / (int)K) % 6;
    if (t0 > 0 && phase == 2 && !check_export(e, ch, dev_base, et, x, where)) bad = true;
    if (t0 > 0 && phase == 4 && !do_import(e, ch, dev_base, base_term, o, c, et, x, where)) bad = true;
    if (bad) break;
    std::vector<std::vector<uint32_t>> want_out;
    std::vector<std::vector<uint8_t>> want_adv;
    for (uint32_t k = 0; k < K; ++k) {
      HostSlot &s = slots[k];
      if (soup)
        f.soup(c, G, R, x);
      else
        f.trace(o, p, (uint64_t)(t0 + k));
      encode8(f, c, G, R, e.gs, enc_base.data(), base_term.data(), s.word.data(), s.prop8.data(), s.desc().in);
      const std::vector<uint64_t> c0 = c.committed;
      f.tick_oracle(o);
      c.load(o);
      want_out.push_back(c.out);
      std::vector<uint8_t> adv(G);
      for (uint64_t g = 0; g < G; ++g) adv[g] = (uint8_t)std::min<uint64_t>(c.committed[g] - c0[g], 255);
      want_adv.push_back(adv);
    }
    TickArgs a = e.args(0, seed, et, 1, true);
    std::vector<TickDesc> descs;
    for (uint32_t k = 0; k < K; ++k) descs.push_back(slots[k].desc());
    switch (R) {
#define TICK_CASE(N) \
  case N: ticks_c<N>(e, ch, a, descs, dev_base.data(), base_term.data()); break;
      TICK_CASE(1) TICK_CASE(2) TICK_CASE(3) TICK_CASE(4) TICK_CASE(5) TICK_CASE(6) TICK_CASE(7) TICK_CASE(8)
#undef TICK_CASE
    }
    for (uint32_t k = 0; k < K && !bad; ++k)
      for (uint64_t g = 0; g < G && !bad; ++g)
        if (slots[k].out[g] != want_out[k][g] || slots[k].delta[g] != want_adv[k][g]) {
          std::printf("FAIL %s tick %d group %llu: out %08x/%08x advance %u/%u\n", where, t0 + (int)k, (unsigned long long)g, slots[k].out[g],
                      want_out[k][g], slots[k].delta[g], want_adv[k][g]);
          ++failures;
          bad = true;
        }
    HostEngine w = e;  // the wide view, as an export sees it
    ClockCols wc = ch;
    std::vector<uint64_t> wb = dev_base;
    const TickArgs aw = w.args(0, seed, et, 1, true);
    for (uint64_t g = 0; g < G; ++g) materialise_group(aw.s, wc.view(), wb.data(), w.gs, R, g, w.tick_no[0], et, 1);
    std::memcpy(w.out.data(), slots[K - 1].out.data(), w.gs * 4);
    if (!bad && !compare(w, c, where, (uint64_t)(t0 + K - 1))) bad = true;
  }
  std::printf("  %-44s %4d ticks\n", where, T);
  orc_destroy(o);
}

}  // namespace

int main(int argc, char **) {
  const bool quick = argc > 1;  // any argument: the sanitizer builds run a smaller matrix
  const uint64_t k = quick ? 3 : 1;
  for (uint32_t R = 1; R <= 8; ++R) {
    run(200 / k + 3, R, 5, 240, 1 + (R - 1) % 4, false);  // lag + churn, batches of 1..4 ticks, a ragged G
    run(160 / k, R, 2, 120, 1 + R % 3, false);             // elections from a cold start
  }
  for (uint32_t R : {2u, 3u, 5u, 8u}) run(120 / k + 8, R, 300 + R, 160, R == 5 ? 4 : 1, true);  // message soups
  std::printf("  export rows checked: %llu   groups imported: %llu\n", (unsigned long long)rows_checked, (unsigned long long)groups_imported);
  std::printf("  exported from: compact leaders %llu (gate closed %llu), flag-0 groups %llu, strict leaders %llu\n",
              (unsigned long long)seen_clock_leaders, (unsigned long long)seen_closed_gate, (unsigned long long)seen_flag0,
              (unsigned long long)seen_strict);
  if (!seen_clock_leaders || !seen_flag0 || !seen_strict || !seen_closed_gate) {
    std::printf("FAIL: the traces did not reach every kind of state\n");
    ++failures;
  }
  std::printf(failures ? "group_state_host_test: %d failure(s)\n" : "group_state_host_test: ok\n", failures);
  return failures ? 1 : 0;
}
