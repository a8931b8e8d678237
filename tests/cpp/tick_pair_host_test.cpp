// tick_pair_host_test.cpp — compact_hot_pair, the quad kernel's hot step for two groups in 16-bit lanes, against two
// calls of the scalar hot step compact_hot_step_clk on the same groups, compiled for the host.
//
// For R = 1..8, on random steady-state groups and on exhaustive sweeps over the edges — lastIndex and the window base at
// 0, 0xFEFF, 0xFF00, 0xFFBF, 0xFFC0 and 0xFFFE, every frame byte (every kind with every payload) in every row of either
// lane, proposal bytes 0 / 1 / 3 / 255, pairs with one lane eligible and one not, and lanes where nothing moved with
// the commit index below the quorum, with lanes whose commit gate is still closed (CF_GATE_OPEN clear, the gate
// anywhere around the quorum, or closed for good) mixed in throughout — the pair step must:
//   - accept exactly when both scalar steps accept and both lanes are inside the pair step's guards (lastIndex <=
//     0xFEFF, window base <= 0xFFBF, every Match after the acks <= lastIndex);
//   - when it accepts, leave both groups' state bit for bit as the scalar steps do, and give the same out words (with
//     the heartbeat the caller adds), commit advances, and the OR of the two dirty masks;
//   - when it declines, leave both groups untouched.
// The other pair's bytes of the quad's frame words are random and must not matter.
//
//   tick_pair_host_test               all cases;   exit code 0 and "tick_pair_host_test: ok" on success
#include "device_on_host.hpp"

#include <cstdio>
#include <cstdlib>

#include "../../raftsql_b200/csrc/mrq_kernels.cuh"

using namespace mrq;

namespace {

int failures = 0;
uint64_t n_checked = 0, n_accepted = 0;
uint64_t rng = 0x9A1Bu;
uint32_t rnd() {
  rng = rng * 6364136223846793005ull + 1442695040888963407ull;
  return (uint32_t)(rng >> 33);
}

template <int R>
struct Lane {  // one group of the pair and its frame bytes
  CGroup<R> g{};
  uint32_t wb[R > 1 ? R - 1 : 1] = {0};
  uint32_t np = 0;
  bool open = true;  // CF_GATE_OPEN
  uint32_t gate = 0;
};

constexpr uint32_t kEdges[] = {0u, 0xFEFFu, 0xFF00u, 0xFFBFu, 0xFFC0u, 0xFFFEu};

template <int R>
void check(const Lane<R> (&ln)[2], const int hi, const char *what) {
  constexpr int NW = R > 1 ? R - 1 : 1;
  ++n_checked;
  // the scalar reference: settled, HeartbeatTick 1
  CGroup<R> s[2] = {ln[0].g, ln[1].g};
  uint32_t so[2], sa[2], sd[2];
  bool want = true;
  for (int h = 0; h < 2; ++h) {
    uint32_t hbw = 0;
    const uint32_t flag = CF_COMPACT | CF_TERM_OK | (ln[h].open ? CF_GATE_OPEN : 0u);
    const bool acc = compact_hot_step_clk<R, uint16_t>(s[h], true, flag, ln[h].wb, ln[h].np, ln[h].gate, 1u, hbw, 0u, so[h], sa[h], sd[h]);
    const uint32_t li = ln[h].g.m[R - 1];
    want = want && acc && li <= 0xFEFFu && ln[h].g.win <= 0xFFBFu;
    for (int j = 0; j < R - 1; ++j) want = want && s[h].m[j] <= li;
  }
  // the pair: its bytes at lanes hi*2 + h of the quad's words, the other pair's bytes random
  uint32_t wq[NW], pq = 0;
  for (int j = 0; j < NW; ++j) {
    wq[j] = rnd();
    for (int h = 0; h < 2; ++h) {
      const int sh = 8 * (2 * hi + h);
      wq[j] = (wq[j] & ~(0xFFu << sh)) | ((R > 1 ? ln[h].wb[j] : 0u) << sh);
    }
  }
  pq = rnd();
  for (int h = 0; h < 2; ++h) {
    const int sh = 8 * (2 * hi + h);
    pq = (pq & ~(0xFFu << sh)) | (ln[h].np << sh);
  }
  auto pack = [&](uint32_t a, uint32_t b) { return (a & 0xFFFFu) | (b << 16); };
  uint32_t commit2 = pack(ln[0].g.commit, ln[1].g.commit), win2 = pack(ln[0].g.win, ln[1].g.win), m2[R];
  for (int r = 0; r < R; ++r) m2[r] = pack(ln[0].g.m[r], ln[1].g.m[r]);
  const uint32_t gate2 = pack(ln[0].open ? 0u : ln[0].gate, ln[1].open ? 0u : ln[1].gate);
  const uint32_t c0 = commit2, w0 = win2;
  uint32_t m0[R];
  for (int r = 0; r < R; ++r) m0[r] = m2[r];
  uint32_t q2 = 0xDEADBEEFu, out2 = 0xDEADBEEFu, dirty = 0xDEADBEEFu;
  const bool got = compact_hot_pair<R>(commit2, win2, m2, gate2, wq, pq, hi, q2, out2, dirty);
  bool ok = got == want;
  if (ok && !got) {
    ok = commit2 == c0 && win2 == w0;
    for (int r = 0; r < R; ++r) ok = ok && m2[r] == m0[r];
  } else if (ok) {
    ++n_accepted;
    for (int h = 0; h < 2; ++h) {
      const int sh = 16 * h;
      ok = ok && ((commit2 >> sh) & 0xFFFFu) == s[h].commit && ((win2 >> sh) & 0xFFFFu) == s[h].win;
      for (int r = 0; r < R; ++r) ok = ok && ((m2[r] >> sh) & 0xFFFFu) == s[h].m[r];
      ok = ok && (((out2 >> sh) & 0xFFFFu) | MRQ_OUT_BCAST_HEARTBEAT) == so[h] && ((q2 >> sh) & 0xFFFFu) == sa[h];
    }
    ok = ok && dirty == (sd[0] | sd[1]);
  }
  if (!ok) {
    if (failures < 20) {
      std::printf("FAIL R=%d %s (pair %d): pair %s, want %s\n", R, what, hi, got ? "accepted" : "declined", want ? "accept" : "decline");
      for (int h = 0; h < 2; ++h) {
        std::printf("  lane %d: commit %u win %u np %u gate %s %u m", h, ln[h].g.commit, ln[h].g.win, ln[h].np, ln[h].open ? "open" : "closed",
                    ln[h].gate);
        for (int r = 0; r < R; ++r) std::printf(" %u", ln[h].g.m[r]);
        std::printf("  bytes");
        for (int j = 0; j < R - 1; ++j) std::printf(" %02x", ln[h].wb[j]);
        std::printf("\n    scalar: commit %u win %u out %02x adv %u dirty %x m", s[h].commit, s[h].win, so[h], sa[h], sd[h]);
        for (int r = 0; r < R; ++r) std::printf(" %u", s[h].m[r]);
        std::printf("\n    pair:   commit %u win %u out %02x adv %u m", (commit2 >> 16 * h) & 0xFFFFu, (win2 >> 16 * h) & 0xFFFFu,
                    (out2 >> 16 * h) & 0xFFFFu, (q2 >> 16 * h) & 0xFFFFu);
        for (int r = 0; r < R; ++r) std::printf(" %u", (m2[r] >> 16 * h) & 0xFFFFu);
        std::printf("\n");
      }
      std::printf("  pair dirty %x\n", dirty);
    }
    ++failures;
  }
}

// a steady-state leader: lastIndex li, window base win, Matches a little behind, commit below them, acks around li
template <int R>
Lane<R> steady(uint32_t li, uint32_t win) {
  Lane<R> l;
  l.g.meta = 0;
  l.g.win = win;
  l.g.m[R - 1] = li;
  for (int j = 0; j < R - 1; ++j) {
    const uint32_t back = rnd() % 8 == 0 ? rnd() % 200 : rnd() % 12;
    l.g.m[j] = rnd() % 16 == 0 ? 0u : li - (back < li ? back : li);
  }
  const uint32_t cb = rnd() % 4 == 0 ? rnd() % 100 : rnd() % 16;
  l.g.commit = li - (cb < li ? cb : li);
  for (int j = 0; j < R - 1; ++j) {
    const uint32_t u = rnd() % 32;
    if (u < 8) {
      l.wb[j] = 0;  // no message
    } else if (u < 30) {  // an ack, mostly of something at or below lastIndex
      const uint32_t top = li > win ? li - win : 0u;
      const uint32_t pay = rnd() % 8 == 0 ? rnd() % 64 : (top < 63 ? top : 63) - rnd() % 4;
      l.wb[j] = ((pay & 63u) << 2) | 1u;
    } else {
      l.wb[j] = rnd() & 0xFFu;  // anything
    }
  }
  static const uint32_t kProps[] = {0, 0, 0, 1, 1, 2, 3, 255};
  l.np = kProps[rnd() % 8];
  l.open = rnd() % 4 != 0;  // (an open gate's c.gate is stale: anything)
  l.gate = rnd() % 8 == 0 ? 0xFFFFu : rnd() % 8 == 1 ? rnd() % 0x10000u : l.g.commit + rnd() % 24;
  if (l.gate > 0xFFFFu) l.gate = 0xFFFFu;
  return l;
}

template <int R>
void run() {
  Lane<R> ln[2];
  // random steady-state pairs, anywhere in the span
  for (int it = 0; it < 40000; ++it) {
    for (int h = 0; h < 2; ++h) {
      const uint32_t li = rnd() % 4 == 0 ? kEdges[rnd() % 6] - rnd() % 70 * (rnd() % 2) : 64 + rnd() % 0xFF00u;
      const uint32_t lic = li > 0xFFFEu ? 0xFFFEu : li;
      const uint32_t back = rnd() % 16 == 0 ? rnd() % 0x10000u : 16 + rnd() % 50;
      ln[h] = steady<R>(lic, rnd() % 8 == 0 ? kEdges[rnd() % 6] : lic - (back < lic ? back : lic));
    }
    check<R>(ln, it & 1, "random");
  }
  // lastIndex and the window base at the edges of the guards and of the span, every proposal byte class
  static const uint32_t kProps[] = {0u, 1u, 3u, 255u};
  for (uint32_t li : kEdges)
    for (uint32_t win : kEdges)
      for (uint32_t np : kProps)
        for (int other = 0; other < 3; ++other) {
          ln[0] = steady<R>(li, win > li ? li : win);
          ln[0].g.win = win;
          ln[0].np = np;
          ln[1] = other == 0 ? ln[0] : steady<R>(0x8000u + rnd() % 0x100u, 0x7FF0u);
          if (other == 2) std::swap(ln[0], ln[1]);
          check<R>(ln, other & 1, "edges");
        }
  // every frame byte in every row of either lane (every kind, every payload)
  if (R > 1)
    for (int h = 0; h < 2; ++h)
      for (int j = 0; j < R - 1; ++j)
        for (uint32_t b = 0; b < 256; ++b)
          for (int rep = 0; rep < 2; ++rep) {
            for (int x = 0; x < 2; ++x) ln[x] = steady<R>(100 + rnd() % 40, 60 + rnd() % 30);
            ln[h].wb[j] = b;
            check<R>(ln, (int)(b & 1), "every byte");
          }
  // one lane eligible, the other not (a heartbeat, a response, an ack beyond lastIndex, a lastIndex past the guard)
  for (int it = 0; it < 2000; ++it) {
    for (int x = 0; x < 2; ++x) ln[x] = steady<R>(5000 + rnd() % 100, 4960 + rnd() % 30);
    Lane<R> &bad = ln[it & 1];
    switch (it % 4) {
      case 0: if (R > 1) bad.wb[rnd() % (R > 1 ? R - 1 : 1)] = (rnd() % 64) << 2 | (2 + rnd() % 2); break;
      case 1: if (R > 1) bad.wb[0] = (63u << 2) | 1u, bad.g.win = bad.g.m[R - 1]; break;  // ack of win + 63 > lastIndex
      case 2: bad.g.m[R - 1] = 0xFF00u + rnd() % 0xFF, bad.g.win = bad.g.m[R - 1] - 40; break;
      default: bad.g.win = 0xFFC0u + rnd() % 0x3F; break;
    }
    check<R>(ln, (it >> 1) & 1, "one lane ineligible");
  }
  // nothing moved, the commit index below the quorum (as after an import): the commit must stay; and the same with
  // the other lane moving
  for (int it = 0; it < 2000; ++it) {
    for (int x = 0; x < 2; ++x) {
      ln[x] = steady<R>(3000 + rnd() % 100, 2990);
      for (int j = 0; j < R - 1; ++j) ln[x].g.m[j] = ln[x].g.m[R - 1] - rnd() % 4;
      ln[x].g.commit = ln[x].g.m[R - 1] - 40;
      for (int j = 0; j < R - 1; ++j) ln[x].wb[j] = rnd() % 2 ? 0u : 1u;  // no message, or an ack of the window base
      ln[x].np = 0;
    }
    if (it & 1) ln[1].np = 1 + rnd() % 3;
    check<R>(ln, (it >> 1) & 1, "nothing moved, commit below the quorum");
  }
}

}  // namespace

int main(int argc, char **) {
  (void)argc;
  run<1>();
  run<2>();
  run<3>();
  run<4>();
  run<5>();
  run<6>();
  run<7>();
  run<8>();
  std::printf("  %llu pairs checked, %llu accepted by the pair step\n", (unsigned long long)n_checked, (unsigned long long)n_accepted);
  if (n_accepted * 5 < n_checked) {
    std::printf("FAIL the pair step accepted too few pairs to mean much\n");
    ++failures;
  }
  std::printf(failures ? "tick_pair_host_test: %d failure(s)\n" : "tick_pair_host_test: ok\n", failures);
  return failures ? 1 : 0;
}
