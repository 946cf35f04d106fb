// Exercises the per-utterance Harvest overload of include/world_b200.hpp: with one HarvestOption per utterance,
// every row must equal, bit for bit, what the reference-compatible single-utterance Harvest() gives that utterance
// with its own option (same kernels, N = 3 with three ranges vs N = 1).
#include <cmath>
#include <cstdio>
#include <vector>

#include "world_b200.hpp"

static std::vector<double> tone(int n, int fs, double f0, unsigned seed) {
  std::vector<double> x(n);
  unsigned s = seed;
  for (int i = 0; i < n; ++i) {
    s = s * 1664525u + 1013904223u;
    const double noise = ((s >> 8) / 16777216.0 - 0.5) * 0.01;
    double v = 0.0;
    for (int k = 1; k <= 8; ++k) v += std::sin(2.0 * 3.14159265358979323846 * f0 * k * i / fs) / k;
    x[i] = 0.2 * v + noise;
  }
  return x;
}

int main() {
  const int fs = 16000, n_utts = 3;
  const int lens[3] = {8000, 6400, 4000};
  const double f0s_true[3] = {120.0, 180.0, 240.0};
  std::vector<std::vector<double>> x(n_utts);
  const double *xs[3];
  for (int u = 0; u < n_utts; ++u) { x[u] = tone(lens[u], fs, f0s_true[u], 17u + u); xs[u] = x[u].data(); }

  std::vector<HarvestOption> per(n_utts);
  for (int u = 0; u < n_utts; ++u) InitializeHarvestOption(&per[u]);
  per[0].f0_floor = 40.0; per[0].f0_ceil = 1100.0;
  per[2].f0_floor = 100.0; per[2].f0_ceil = 600.0;
  int fl[3];
  std::vector<std::vector<double>> th(n_utts), fh(n_utts);
  double *thp[3], *fhp[3];
  for (int u = 0; u < n_utts; ++u) {
    fl[u] = GetSamplesForHarvest(fs, lens[u], per[u].frame_period);
    th[u].resize(fl[u]); fh[u].resize(fl[u]); thp[u] = th[u].data(); fhp[u] = fh[u].data();
  }
  const int rc = Harvest(xs, lens, n_utts, fs, per, thp, fhp);
  if (rc) { std::printf("FAIL: batched Harvest with per-utterance options returned %d\n", rc); return 1; }
  int bad = 0, voiced = 0;
  for (int u = 0; u < n_utts; ++u) {
    std::vector<double> t1(fl[u]), f1(fl[u]);
    Harvest(xs[u], lens[u], fs, &per[u], t1.data(), f1.data());
    for (int i = 0; i < fl[u]; ++i) {
      bad += (t1[i] != th[u][i]) + (f1[i] != fh[u][i]);
      voiced += f1[i] > 0;
    }
  }
  // a vector whose size is not n_utts is refused
  std::vector<HarvestOption> two(per.begin(), per.begin() + 2);
  if (Harvest(xs, lens, n_utts, fs, two, thp, fhp) != WORLD_B200_EINVAL) { std::printf("FAIL: size check\n"); return 1; }
  if (bad || voiced == 0) { std::printf("FAIL: %d mismatching values, %d voiced frames\n", bad, voiced); return 1; }
  std::printf("OK: per-utterance Harvest overload == single-utterance Harvest on %d utterances (%d voiced frames)\n",
              n_utts, voiced);
  return 0;
}
