// resize_host_test.cpp — the fresh groups of mrq_resize_groups, compiled for the host from the device source.
//
// init_state_kernel is the one definition of a fresh group: mrq_create runs it over rows [0, G), a grow over rows
// [old G, new G).  Here its body runs over the engine's layout in host memory (one call per row: on the host the thread
// index is 0, so the first-row argument names the row).  For R = 1..8, the rotate rule and a fixed self id, group_base 0
// and a large one, and with tick mode 4's compact state live or not:
//   - "create": zeroed buffers, rows [0, G) initialised; every column equals a fresh oracle's export (orc_create with
//     the same configuration), meta field by field;
//   - "grow": buffers full of another run's bytes (the surviving groups below `old`, dropped groups in the padding),
//     rows [old, G) initialised; those rows equal create's in every wide column, the drain base and the packed bases,
//     and, with the compact state live, their compact columns equal what compact_group makes of create's rows at the same
//     tick (what the next mode-4 tick would otherwise have to do); every byte outside rows [old, G) is unchanged.
//
//   resize_host_test          all cases;   exit code 0 and "resize_host_test: ok" on success
#include "device_on_host.hpp"

#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../oracle/raft_oracle.h"
#include "../../raftsql_b200/csrc/mrq_kernels.cuh"

using namespace mrq;

namespace {

int failures = 0;
uint64_t rows_checked = 0;

#define CHECK(cond, ...)                          \
  do {                                            \
    if (!(cond)) {                                \
      if (failures++ < 20) {                      \
        std::printf("FAIL %s:%d: ", __FILE__, __LINE__); \
        std::printf(__VA_ARGS__);                 \
        std::printf("\n");                        \
      }                                           \
    }                                             \
  } while (0)

struct Cols {  // every buffer init_state_kernel writes, at stride gs
  uint64_t gs;
  uint32_t R;
  std::vector<uint64_t> term, meta, last_index, last_term, committed, term_start, match, commit_prev, base_index, base_term, ibase;
  std::vector<uint32_t> out, iblo, clk;
  std::vector<uint8_t> flag;
  std::vector<CompactOff> ccommit, win, gate, cmatch;
  Cols(uint64_t gs_, uint32_t R_)
      : gs(gs_), R(R_), term(gs), meta(gs), last_index(gs), last_term(gs), committed(gs), term_start(gs), match(gs * R), commit_prev(gs),
        base_index(gs), base_term(gs), ibase(gs), out(gs), iblo(gs), clk(gs), flag(gs), ccommit(gs), win(gs), gate(gs), cmatch(gs * R) {}
  StateView view() {
    return StateView{term.data(), meta.data(), last_index.data(), last_term.data(), committed.data(), term_start.data(), match.data(),
                     out.data()};
  }
  CompactViewT<CompactOff> cview() {
    return CompactViewT<CompactOff>{flag.data(), ccommit.data(), win.data(), gate.data(), iblo.data(), cmatch.data(), ibase.data(), clk.data()};
  }
  FreshRows fresh(bool compact) { return FreshRows{commit_prev.data(), base_index.data(), base_term.data(), cview(), compact ? 1 : 0}; }
  void scramble(uint64_t &x) {  // another run's bytes everywhere
    auto rnd = [&]() { return x = mrq_mix64(x + 0x9E3779B97F4A7C15ull); };
    for (auto *v : {&term, &meta, &last_index, &last_term, &committed, &term_start, &match, &commit_prev, &base_index, &base_term, &ibase})
      for (auto &e : *v) e = rnd();
    for (auto *v : {&out, &iblo, &clk})
      for (auto &e : *v) e = (uint32_t)rnd();
    for (auto &e : flag) e = (uint8_t)rnd();
    for (auto *v : {&ccommit, &win, &gate, &cmatch})
      for (auto &e : *v) e = (CompactOff)rnd();
  }
};

constexpr uint32_t kET = 10, kHT = 3;
constexpr uint64_t kSeed = 0x5EED5EEDull, kT = 987654321ull;

void run(uint64_t old_g, uint64_t new_g, uint32_t R, uint32_t self_id, uint64_t group_base, bool compact, uint64_t &x) {
  const uint64_t gs = std::max<uint64_t>(128, (new_g + 127) / 128 * 128);
  // create: zeroed buffers (cudaMemsetAsync in dalloc), then the kernel over rows [0, G); create never compacts
  Cols c(gs, R);
  for (uint64_t g = 0; g < new_g; ++g)
    init_state_kernel(c.view(), c.fresh(false), g, new_g, gs, group_base, R, self_id, kSeed, kET, kHT, kT);
  // ... equal to a fresh oracle
  orc_engine *o = orc_create(new_g, R, group_base, kET, kHT, kSeed, self_id);
  std::vector<uint64_t> ot(new_g), ov(new_g), oc(new_g), oli(new_g), olt(new_g), ots(new_g), om(new_g * R);
  std::vector<uint8_t> orole(new_g), olead(new_g), oself(new_g), ovotes(new_g * R);
  std::vector<uint16_t> oel(new_g), ohb(new_g), orto(new_g);
  orc_export(o, ot.data(), ov.data(), oc.data(), oli.data(), olt.data(), ots.data(), om.data(), orole.data(), olead.data(), oself.data(),
             ovotes.data(), oel.data(), ohb.data(), orto.data(), nullptr);
  orc_destroy(o);
  for (uint64_t g = 0; g < new_g; ++g) {
    const Meta m = meta_unpack(c.meta[g]);
    CHECK(c.term[g] == ot[g] && c.committed[g] == oc[g] && c.last_index[g] == oli[g] && c.last_term[g] == olt[g] && c.term_start[g] == ots[g],
          "R=%u self=%u base=%llu: created group %llu differs from the oracle's (wide columns)", R, self_id, (unsigned long long)group_base,
          (unsigned long long)g);
    uint32_t votes = 0;
    for (uint32_t r = 0; r < R; ++r) {
      CHECK(c.match[(uint64_t)r * gs + g] == om[(uint64_t)r * new_g + g], "R=%u: created group %llu match[%u]", R, (unsigned long long)g, r);
      votes |= (uint32_t)ovotes[(uint64_t)r * new_g + g] << (2 * r);
    }
    CHECK(m.role == orole[g] && m.lead == olead[g] && m.vote == ov[g] && m.self == oself[g] && m.elapsed == oel[g] && m.hb == ohb[g] &&
              m.rto == orto[g] && m.votes == votes && m.strict == 0 && m.ltok == 1,
          "R=%u self=%u base=%llu: created group %llu meta differs from the oracle's (self %u/%u rto %u/%u)", R, self_id,
          (unsigned long long)group_base, (unsigned long long)g, m.self, oself[g], m.rto, orto[g]);
  }
  // the compact form the next mode-4 tick would give create's rows (compact_all_kernel)
  Cols cc = c;
  if (compact)
    for (uint64_t g = 0; g < new_g; ++g) compact_group(cc.view(), cc.cview(), cc.base_index.data(), cc.base_term.data(), gs, R, g, kT, kET, kHT);

  // grow: another run's bytes everywhere, then the kernel over rows [old, G)
  Cols w(gs, R);
  w.scramble(x);
  const Cols before = w;
  for (uint64_t g = old_g; g < new_g; ++g)
    init_state_kernel(w.view(), w.fresh(compact), g, new_g, gs, group_base, R, self_id, kSeed, kET, kHT, kT);
  auto fresh_row = [&](uint64_t i) { return i >= old_g && i < new_g; };
  auto cmp_u64 = [&](const char *name, const std::vector<uint64_t> &want, const std::vector<uint64_t> &got, const std::vector<uint64_t> &was,
                     uint32_t rows) {
    for (uint32_t r = 0; r < rows; ++r)
      for (uint64_t i = 0; i < gs; ++i) {
        const uint64_t k = (uint64_t)r * gs + i;
        if (fresh_row(i))
          CHECK(got[k] == want[k], "R=%u self=%u base=%llu old=%llu new=%llu: %s of new group %llu (row %u) is %llx, create gives %llx", R,
                self_id, (unsigned long long)group_base, (unsigned long long)old_g, (unsigned long long)new_g, name, (unsigned long long)i, r,
                (unsigned long long)got[k], (unsigned long long)want[k]);
        else
          CHECK(got[k] == was[k], "R=%u old=%llu new=%llu: %s of group %llu (row %u) changed outside the new rows", R, (unsigned long long)old_g,
                (unsigned long long)new_g, name, (unsigned long long)i, r);
      }
  };
  cmp_u64("term", cc.term, w.term, before.term, 1);
  cmp_u64("meta", cc.meta, w.meta, before.meta, 1);
  cmp_u64("last_index", cc.last_index, w.last_index, before.last_index, 1);
  cmp_u64("last_term", cc.last_term, w.last_term, before.last_term, 1);
  cmp_u64("committed", cc.committed, w.committed, before.committed, 1);
  cmp_u64("term_start", cc.term_start, w.term_start, before.term_start, 1);
  cmp_u64("match", cc.match, w.match, before.match, R);
  cmp_u64("commit_prev", cc.commit_prev, w.commit_prev, before.commit_prev, 1);
  cmp_u64("base_index", cc.base_index, w.base_index, before.base_index, 1);
  cmp_u64("base_term", cc.base_term, w.base_term, before.base_term, 1);
  CHECK(w.out == before.out, "R=%u: the kernel wrote out words", R);
  // compact columns: create's compact form in the new rows with the compact state live, untouched otherwise
  for (uint64_t i = 0; i < gs; ++i) {
    const bool mine = compact && fresh_row(i);
    const Cols &want = mine ? cc : before;
    CHECK(w.flag[i] == want.flag[i] && w.ccommit[i] == want.ccommit[i] && w.win[i] == want.win[i] && w.gate[i] == want.gate[i] &&
              w.ibase[i] == want.ibase[i] && w.iblo[i] == want.iblo[i],
          "R=%u compact=%d old=%llu new=%llu: compact columns of group %llu (%s)", R, (int)compact, (unsigned long long)old_g,
          (unsigned long long)new_g, (unsigned long long)i, mine ? "new, differs from create's compact form" : "changed outside the new rows");
    CHECK(w.clk[i] == before.clk[i], "R=%u: clk of group %llu changed (fresh groups are followers)", R, (unsigned long long)i);
    for (uint32_t r = 0; r < R; ++r)
      CHECK(w.cmatch[(uint64_t)r * gs + i] == want.cmatch[(uint64_t)r * gs + i], "R=%u compact=%d: compact match row %u of group %llu", R,
            (int)compact, r, (unsigned long long)i);
    if (mine) CHECK(w.flag[i] & CF_COMPACT, "R=%u: new group %llu did not become compact", R, (unsigned long long)i);
  }
  rows_checked += new_g - old_g;
}

}  // namespace

int main() {
  uint64_t x = 0x12345;
  for (uint32_t R = 1; R <= 8; ++R)
    for (uint32_t self_id : {0u, (R + 1) / 2})
      for (uint64_t group_base : {0ull, 4000000007ull})
        for (bool compact : {false, true}) {
          run(0, 300, R, self_id, group_base, compact, x);    // 0 -> 300: every row fresh
          run(250, 300, R, self_id, group_base, compact, x);  // a grow within the stride
          run(100, 700, R, self_id, group_base, compact, x);  // across it
          run(383, 384, R, self_id, group_base, compact, x);  // one group, up to the stride
        }
  std::printf("  fresh rows checked: %llu\n", (unsigned long long)rows_checked);
  std::printf(failures ? "resize_host_test: %d failure(s)\n" : "resize_host_test: ok\n", failures);
  return failures ? 1 : 0;
}
