// tick_host16_test.cpp — tick mode 4 on the host at the library's offset width: the compact columns as uint16_t.
//
// tick_host_test.cpp runs the compact per-group functions of raftsql_b200/csrc/mrq_kernels.cuh with 32-bit offset
// columns (the header's default width).  The library instantiates them with 16-bit columns (CompactOff), where the
// span an offset may reach is clamped to 0xFFFE, 0xFFFF marks a gate that is closed for good, and a group whose log
// outgrows the span is handed to the general path and re-based.  This file runs the same cases against the oracle with
// 16-bit columns: traces, message soups, the window-edge soup, a span small enough to re-base every few dozen ticks,
// and steady leaders whose logs grow past 2^16 entries from their base at the real span.
//
// The harness around the compact columns (engine layout, oracle columns, comparison, trace presets) is
// tick_host_test.cpp's, included here with its main() renamed.
//
//   tick_host16_test               all cases;   exit code 0 and "tick_host16_test: ok" on success
#define main tick_host_test_main
#include "tick_host_test.cpp"
#undef main

namespace {

template <typename Off>
struct CompactHostT {  // the compact columns at width Off (CompactHost of tick_host_test.cpp is the 32-bit one)
  uint64_t gs;
  uint32_t R;
  std::vector<uint8_t> flag;
  std::vector<Off> commit, win, gate, match;
  std::vector<uint32_t> iblo;
  std::vector<uint64_t> ibase;
  uint64_t fast_ticks = 0, slow_entries = 0, hot_ticks = 0, span_exits = 0;
  CompactHostT(uint64_t gs_, uint32_t R_) : gs(gs_), R(R_), flag(gs_, 0), commit(gs_, 0), win(gs_, 0), gate(gs_, 0), match(gs_ * R_, 0),
                                             iblo(gs_, 0), ibase(gs_, 0) {}
  CompactViewT<Off> view() {
    return CompactViewT<Off>{flag.data(), commit.data(), win.data(), gate.data(), iblo.data(), match.data(), ibase.data()};
  }
  void invalidate() { std::fill(flag.begin(), flag.end(), 0); }
};

// what tick_fast4_kernel + tick_slow4_kernel do per group over one K-tick launch, at width Off
template <int R, typename Off>
void host_ticks_w(HostEngine &e, CompactHostT<Off> &ch, const TickArgs &a, std::vector<TickDesc> &descs, uint64_t *base_index,
                  const uint64_t *base_term) {
  Tick4ArgsT<Off> A{};
  A.t = a;
  A.c = ch.view();
  A.base_index = base_index;
  A.base_term = base_term;
  A.nticks = (uint32_t)descs.size();
  A.d0 = descs[0];
  A.descs = descs.size() > 1 ? descs.data() : nullptr;
  A.write_through = 1;
  for (uint64_t i = 0; i < e.G; ++i) {
    CGroup<R> g;  // widened at the load, as the kernels do
    g.meta = e.meta[i];
    g.commit = ch.commit[i];
    g.win = ch.win[i];
    for (int r = 0; r < R; ++r) g.m[r] = ch.match[(uint64_t)r * e.gs + i];
    const uint32_t flag = ch.flag[i];
    const uint32_t gate = ch.gate[i];
    uint32_t t = 0, np = 0;
    bool slow = false;
    for (; t < A.nticks; ++t) {
      const TickDesc &d = descs[t];
      uint32_t wb[R > 1 ? R - 1 : 1] = {0};
      for (int j = 0; j < R - 1; ++j) wb[j] = d.word8[(uint64_t)j * e.gs + i];
      uint32_t o, adv, dirty;
      np = d.prop8 ? d.prop8[i] : 0u;
      slow = false;
      if (!hot_path || !compact_hot_step<R, Off>(g, flag, wb, np, gate, a.election_tick, a.heartbeat_tick, o, adv, dirty))
        slow = compact_step<R, Off>(g, flag, wb, np, gate, a.election_tick, a.heartbeat_tick, o, adv, dirty);
      else
        ++ch.hot_ticks;
      if (slow) break;
      d.out[i] = o;
      d.delta[i] = (uint8_t)(adv > 255u ? 255u : adv);
      ++ch.fast_ticks;
    }
    // narrowed at the store: whatever the fast path kept must fit the column
    const uint32_t top = (uint32_t)static_cast<Off>(~Off(0));
    bool fits = g.commit <= top && g.win <= top;
    for (int r = 0; r < R; ++r) fits = fits && g.m[r] <= top;
    if ((flag & CF_COMPACT) && !fits) {
      std::printf("FAIL group %llu: an offset outgrew the %u-bit column on the fast path\n", (unsigned long long)i, (unsigned)(8 * sizeof(Off)));
      ++failures;
    }
    e.meta[i] = g.meta;
    ch.commit[i] = (Off)g.commit;
    ch.win[i] = (Off)g.win;
    for (int r = 0; r < R; ++r) ch.match[(uint64_t)r * e.gs + i] = (Off)g.m[r];
    if (slow) {
      slow_group_ticks_c<R>(A, i, t);
      ++ch.slow_entries;
      ch.span_exits += (flag & CF_COMPACT) && g.m[R - 1] + np > compact_span<Off>();  // the log reached the end of the span
    }
  }
  e.tick_no[0] += A.nticks;
}

template <typename Off>
void dispatch_ticks_w(HostEngine &e, CompactHostT<Off> &ch, const TickArgs &a, std::vector<TickDesc> &descs, uint64_t *bi, const uint64_t *bt) {
  switch (e.R) {
    case 1: host_ticks_w<1>(e, ch, a, descs, bi, bt); break;
    case 2: host_ticks_w<2>(e, ch, a, descs, bi, bt); break;
    case 3: host_ticks_w<3>(e, ch, a, descs, bi, bt); break;
    case 4: host_ticks_w<4>(e, ch, a, descs, bi, bt); break;
    case 5: host_ticks_w<5>(e, ch, a, descs, bi, bt); break;
    case 6: host_ticks_w<6>(e, ch, a, descs, bi, bt); break;
    case 7: host_ticks_w<7>(e, ch, a, descs, bi, bt); break;
    case 8: host_ticks_w<8>(e, ch, a, descs, bi, bt); break;
  }
}

// run_case_c of tick_host_test.cpp at width Off, plus `max_prop` (0: the preset's) for logs that grow fast.
// Returns how often a group left the fast path because its log reached the end of the offset span.
template <typename Off>
uint64_t run_case_w(uint64_t G, uint32_t R, uint32_t cfg, int T, int rebase_every, uint32_t K, bool soup = false, uint64_t big = 0,
                    int also_rebase_at = -1, bool edges = false, uint32_t max_prop = 0) {
  char where[128];
  std::snprintf(where, sizeof where, "compact u%u%s K=%u G=%llu R=%u %s=%u%s", (unsigned)(8 * sizeof(Off)), soup ? " soup" : "", K,
                (unsigned long long)G, R, soup ? "seed" : "cfg", cfg, edges ? " window edges" : big ? " far base" : max_prop ? " long logs" : "");
  const uint64_t seed = 0x5EEDC000ull + cfg * 131 + R;
  const uint32_t et = soup ? 5 : 10;
  orc_engine *o = orc_create(G, R, 0, et, 1, seed, 0);
  HostEngine e(G, R);
  CompactHostT<Off> ch(e.gs, R);
  OracleCols c(G, R);
  c.load(o);
  if (big) {  // steady-state leaders whose indices sit `big` above a multiple of 2^32
    uint64_t x = 7;
    auto rnd = [&]() { return x = mrq_mix64(x + 0x9E3779B97F4A7C15ull); };
    for (uint64_t g = 0; g < G; ++g) {
      const uint32_t self = (uint32_t)(g % R) + 1;
      c.self_id[g] = (uint8_t)self;
      c.role[g] = MRQ_ROLE_LEADER;
      c.lead[g] = (uint8_t)self;
      c.term[g] = 1 + rnd() % 8;
      c.vote[g] = self;
      c.last_index[g] = big + rnd() % 40;
      c.last_term[g] = c.term[g];
      for (uint32_t r = 0; r < R; ++r) c.match[(uint64_t)r * G + g] = (g % 7 == 3 && r == (self % R)) ? 5 : c.last_index[g] - 1 - rnd() % 6;
      c.match[(uint64_t)(self - 1) * G + g] = c.last_index[g];
      c.committed[g] = c.last_index[g] - 8;
      c.term_start[g] = (g % 5 == 0) ? c.last_index[g] - 2 : c.committed[g] - 5;  // some gates still closed
      c.rto[g] = 10;
    }
    orc_import(o, c.term.data(), c.vote.data(), c.committed.data(), c.last_index.data(), c.last_term.data(), c.term_start.data(),
               c.match.data(), c.role.data(), c.lead.data(), c.self_id.data(), nullptr, nullptr, nullptr, c.rto.data());
    c.load(o);
  }
  import_from_oracle(e, c);
  mrq_trace_params p = preset(soup ? 3 : cfg);
  if (max_prop) p.max_prop = max_prop;
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
  uint64_t n_bytes = 0, n_escapes = 0;
  bool bad = false;
  for (int t0 = 0; t0 < T && !bad; t0 += (int)K) {
    if (t0 % rebase_every == 0 || t0 == also_rebase_at) {  // mrq_set_packed_base
      const TickArgs a0 = e.args(0, seed, et, 1, true);
      for (uint64_t g = 0; g < G; ++g) materialise_group(a0.s, ch.view(), dev_base.data(), e.gs, R, g);
      ch.invalidate();
      c.load(o);
      for (uint64_t g = 0; g < G; ++g) {
        const uint64_t back = soup ? 6 : 30;
        enc_base[g] = dev_base[g] = c.last_index[g] > back ? c.last_index[g] - back : 0;
        base_term[g] = c.term[g];
      }
    }
    c.load(o);
    want_commit[0] = c.committed;
    for (uint32_t k = 0; k < K; ++k) {
      HostSlot &s = slots[k];
      if (!soup) {
        orc_gen_trace(o, &p, (uint64_t)(t0 + k), type.data(), term.data(), index.data(), logterm.data(), commit.data(), prop.data(), 1);
      } else {
        for (uint64_t g = 0; g < G; ++g) {
          for (uint32_t r = 0; r < R; ++r) {
            const uint64_t w = (uint64_t)r * G + g;
            const uint8_t ty = kTypes[rnd() % sizeof kTypes];
            type[w] = ty;
            if ((ty & 0x0F) == 0) {
              term[w] = index[w] = logterm[w] = commit[w] = 0;
              continue;
            }
            const uint64_t u = rnd() % (edges ? 4096 : 64);
            term[w] = around(c.term[g], u == 0 ? -2 : u == 1 ? -1 : u == 2 ? 1 : u == 3 ? 2 : 0);
            index[w] = around(c.last_index[g], (int64_t)(rnd() % 7) - 4);
            logterm[w] = around(c.last_term[g], (int64_t)(rnd() % 3) - 1);
            commit[w] = c.committed[g] + rnd() % 4;
            if (edges) {  // compact-representable traffic aimed at the edges of the 64-entry window and of the log
              static const uint8_t kEdge[] = {4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 0, 0, 8, 9, 6, 4 | 0x80};
              const uint8_t t2 = (rnd() % 16 == 0) ? kEdge[14 + rnd() % 6] : kEdge[rnd() % 14];
              type[w] = t2;
              if ((t2 & 0x0F) == 0) {
                term[w] = index[w] = logterm[w] = commit[w] = 0;
                continue;
              }
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
            const uint8_t ty2 = type[w];
            if ((ty2 & 0x0F) == 3) {
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
            ++n_escapes;
          } else if (b != 0) {
            ++n_bytes;
            if ((b & 3u) == 1u && (uint32_t)(b >> 2) < min_ack) min_ack = b >> 2;
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
    const TickArgs a = e.args(0, seed, et, 1, true);
    std::vector<TickDesc> descs;
    for (uint32_t k = 0; k < K; ++k) descs.push_back(slots[k].desc());
    dispatch_ticks_w(e, ch, a, descs, dev_base.data(), base_term.data());
    for (uint64_t g = 0; g < G; ++g) materialise_group(a.s, ch.view(), dev_base.data(), e.gs, R, g);
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
  std::printf("  %-50s %5d ticks  bytes %8llu  escapes %7llu  fast group-ticks %8llu (hot %8llu)  general entries %7llu  span exits %5llu  "
              "compact now %llu/%llu\n",
              where, T, (unsigned long long)n_bytes, (unsigned long long)n_escapes, (unsigned long long)ch.fast_ticks,
              (unsigned long long)ch.hot_ticks, (unsigned long long)ch.slow_entries, (unsigned long long)ch.span_exits,
              (unsigned long long)n_compact, (unsigned long long)G);
  if (!bad && !soup && R > 1 && ch.fast_ticks < (uint64_t)T * G / 4) {
    std::printf("FAIL %s: the compact fast path handled too little (%llu of %llu group-ticks)\n", where, (unsigned long long)ch.fast_ticks,
                (unsigned long long)((uint64_t)T * G));
    ++failures;
  }
  orc_destroy(o);
  return ch.span_exits;
}

}  // namespace

int main(int argc, char **) {
  const bool quick = argc > 1;  // any argument: the sanitizer build runs a smaller matrix
  const uint64_t k = quick ? 4 : 1;
  using W = uint16_t;
  static_assert(sizeof(CompactOff) == sizeof(W), "the library's offset width is the one checked here");
  // the span at this width, whatever kCompactSpan allows
  if (compact_span<W>() != 0xFFFEu) {
    std::printf("FAIL compact_span<uint16_t>() = %u, want 0xFFFE\n", compact_span<W>());
    ++failures;
  }
  for (uint32_t R = 1; R <= 8; ++R) run_case_w<W>(300 / k, R, 5, 224, 32, R % 2 ? 1 : 4);
  run_case_w<W>(400 / k, 5, 2, 300, 60, 1);  // elections from a cold start
  run_case_w<W>(400 / k, 5, 2, 300, 60, 5);
  run_case_w<W>(400 / k, 3, 6, 300, 30, 3);  // follower / heartbeat heavy
  run_case_w<W>(400 / k, 5, 3, 400, 1000, 1, false, 0, 60);  // steady state: one base, then the window slides by itself
  run_case_w<W>(400 / k, 5, 3, 400, 1000, 8, false, 0, 64);
  run_case_w<W>(300 / k, 5, 3, 300, 1000, 4, false, (1ull << 33) + 100);  // 64-bit bases, far-behind followers, closed gates
  // Logs that outgrow 16 bits from their base at the real span: steady leaders proposing up to 20 entries a tick (as
  // many as the 64-entry ack window keeps up with), one frame-builder base for the whole run.  A leader reaches the end
  // of the span after ~6,500 ticks on the fast path and is re-based by the general path.
  if (run_case_w<W>(48 / k, 3, 3, 9000, 1 << 30, 8, false, 0, 64, false, 20) == 0) {
    std::printf("FAIL long logs: no group reached the end of the 16-bit span\n");
    ++failures;
  }
  kCompactSpan = 120;  // a tiny span: every group outgrows it every few dozen ticks
  run_case_w<W>(200 / k, 5, 3, 240, 1000, 4, false, (1ull << 31) - 300);
  run_case_w<W>(200 / k, 3, 5, 240, 40, 1);
  kCompactSpan = 0x7FFFFFFFu;
  for (uint32_t R : {2u, 3u, 5u, 8u}) run_case_w<W>(120 / k + 8, R, 300 + R, 240, 8, R == 5 ? 4 : 1, true);  // message soups
  for (uint32_t R : {2u, 3u, 4u, 5u, 7u, 8u}) run_case_w<W>(160 / k + 8, R, 500 + R, 320, 16, R % 2 ? 1 : 4, true, 1ull << 22, -1, true);
  hot_path = false;  // the complete compact step alone
  run_case_w<W>(300 / k, 5, 5, 224, 32, 1);
  run_case_w<W>(300 / k, 3, 3, 300, 1000, 4, false, 0, 60);
  hot_path = true;
  std::printf(failures ? "tick_host16_test: %d failure(s)\n" : "tick_host16_test: ok\n", failures);
  return failures ? 1 : 0;
}
