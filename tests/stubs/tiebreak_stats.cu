// Host-side statistics of the supporting-surfel arrival key (csrc/sm_kernels.cuh) with the library's default
// parameters: how often the lower slot / the primary association wins, by where the two slots sit in the modelled
// launch. Printed as "name value" lines; tests/test_tiebreak_host.py compares them with what was measured on the
// reference (DESIGN.md section 4).
#include <cstdio>
#include <cstdlib>
#include <random>
#include "sm_handle.cuh"
using namespace smb;
namespace smb { int SetError(int c, const char*) { return c; } }

static u32 ModInverseHost(u32 a, u32 m) {
  long long t = 0, nt = 1, r = m, nr = a % m;
  while (nr) { long long q = r / nr; long long tmp = t - q * nt; t = nt; nt = tmp; tmp = r - q * nr; r = nr; nr = tmp; }
  if (t < 0) t += m;
  return (u32)t;
}

static TieBreak MakeDefault(u32 frame) {
  TieBreak t{};
  t.wave = kDefaultTieBreakWave; t.lane_shift = kDefaultTieBreakLaneShift; t.groups = t.wave >> t.lane_shift; t.wave_offset = 0;
  const unsigned long long prime = 2654435761ull;
  t.mul = (u32)(prime % t.groups); t.mul_inv = ModInverseHost(t.mul, t.groups);
  t.wave_reciprocal = ~0ull / t.wave; t.group_reciprocal = ~0ull / t.groups;
  t.add = tb_hash(frame * 0x9E3779B9u + 0x7F4A7C15u) % t.groups;
  t.salt = tb_hash(frame ^ 0x85EBCA6Bu);
  auto th = [](double f) { return (u32)(f * 4294967296.0); };
  t.early_threshold = th(kDefaultTieBreakEarlyFraction);
  t.index_order_threshold = th(kDefaultTieBreakIndexOrderFraction);
  t.early_threshold_later = th(kDefaultTieBreakEarlyFractionLater);
  t.early_threshold_second = th(kDefaultTieBreakEarlyFractionSecond);
  t.index_order_threshold_later = th(kDefaultTieBreakIndexOrderFractionLater);
  return t;
}

int main() {
  std::mt19937 rng(12345);
  const u32 W = kDefaultTieBreakWave;
  struct Case { const char* name; int wave; int kind; };   // kind 0: same warp, 1: same block other warp, 2: other block, 3: other wave
  const Case cases[] = {{"wave0_same_warp", 0, 0}, {"wave0_same_block", 0, 1}, {"wave0_other_block", 0, 2},
                        {"wave2_same_warp", 2, 0}, {"wave2_same_block", 2, 1}, {"wave2_other_block", 2, 2}, {"other_wave", 0, 3}};
  for (const Case& c : cases) {
    unsigned long long lower_wins = 0, n = 0;
    for (int trial = 0; trial < 200000; ++trial) {
      const TieBreak t = MakeDefault(4 + trial % 97);
      const u32 pixel = rng() % 307200u;
      u32 a, b;
      const u32 base = c.wave * W;
      if (c.kind == 0) { const u32 warp = rng() % (W / 32); a = base + warp * 32 + rng() % 32; do { b = base + warp * 32 + rng() % 32; } while (b == a); }
      else if (c.kind == 1) { const u32 block = rng() % (W / 1024); a = base + block * 1024 + rng() % 1024; do { b = base + block * 1024 + rng() % 1024; } while (b / 32 == a / 32); }
      else if (c.kind == 2) { a = base + rng() % W; do { b = base + rng() % W; } while (b / 1024 == a / 1024); }
      else { a = rng() % W; b = W + rng() % W; }
      const u32 lo = a < b ? a : b, hi = a < b ? b : a;
      lower_wins += tb_encode(t, lo, false, pixel) < tb_encode(t, hi, false, pixel);
      ++n;
    }
    printf("%s %.4f\n", c.name, (double)lower_wins / n);
  }
  // one primary and one secondary association in one wave: how often the secondary wins
  for (int wave = 0; wave < 3; ++wave) {
    unsigned long long secondary_wins = 0, n = 0;
    for (int trial = 0; trial < 400000; ++trial) {
      const TieBreak t = MakeDefault(4 + trial % 97);
      const u32 pixel = rng() % 307200u;
      const u32 p = wave * W + rng() % W, s = wave * W + rng() % W;
      if (p == s) continue;
      secondary_wins += tb_encode(t, s, true, pixel) < tb_encode(t, p, false, pixel);
      ++n;
    }
    printf("wave%d_secondary_wins %.4f\n", wave, (double)secondary_wins / n);
  }
  return 0;
}
