// Exercises the per-utterance CheapTrick and D4C overloads of include/world_b200.hpp: with one option (and so one
// fft_size) per utterance, every row must equal, bit for bit, what the reference-compatible single-utterance
// CheapTrick() / D4C() give that utterance with its own option (N = 3 at three sizes vs N = 1).
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
  const double voice[3] = {45.0, 80.0, 150.0}, floor[3] = {40.0, 71.0, 100.0};
  std::vector<std::vector<double>> x(n_utts), t(n_utts), f(n_utts);
  const double *xs[3], *ts[3], *fs0[3];
  int fl[3];
  std::vector<CheapTrickOption> co(n_utts);
  std::vector<D4COption> dopt(n_utts);
  std::vector<int> sizes(n_utts);
  for (int u = 0; u < n_utts; ++u) {
    x[u] = tone(lens[u], fs, voice[u], 29u + u);
    fl[u] = lens[u] * 1000 / fs / 5 + 1;
    t[u].resize(fl[u]); f[u].resize(fl[u]);
    for (int i = 0; i < fl[u]; ++i) { t[u][i] = i * 0.005; f[u][i] = i < fl[u] * 4 / 5 ? voice[u] : 0.0; }
    xs[u] = x[u].data(); ts[u] = t[u].data(); fs0[u] = f[u].data();
    InitializeCheapTrickOption(fs, &co[u]);
    co[u].f0_floor = floor[u];
    co[u].fft_size = sizes[u] = GetFFTSizeForCheapTrick(fs, &co[u]);
    InitializeD4COption(&dopt[u]);
  }
  std::vector<std::vector<std::vector<double>>> sp(n_utts), ap(n_utts);
  std::vector<std::vector<double *>> spp(n_utts), app(n_utts);
  double **sps[3], **aps[3];
  for (int u = 0; u < n_utts; ++u) {
    const int bins = sizes[u] / 2 + 1;
    sp[u].assign(fl[u], std::vector<double>(bins)); ap[u].assign(fl[u], std::vector<double>(bins));
    for (int i = 0; i < fl[u]; ++i) { spp[u].push_back(sp[u][i].data()); app[u].push_back(ap[u][i].data()); }
    sps[u] = spp[u].data(); aps[u] = app[u].data();
  }
  int rc = CheapTrick(xs, lens, n_utts, fs, ts, fs0, fl, co, sps);
  if (!rc) rc = D4C(xs, lens, n_utts, fs, ts, fs0, fl, sizes, dopt, aps);
  if (rc) { std::printf("FAIL: per-utterance overloads returned %d\n", rc); return 1; }
  long bad = 0, values = 0;
  for (int u = 0; u < n_utts; ++u) {
    const int bins = sizes[u] / 2 + 1;
    std::vector<std::vector<double>> s1(fl[u], std::vector<double>(bins)), a1(fl[u], std::vector<double>(bins));
    std::vector<double *> s1p, a1p;
    for (int i = 0; i < fl[u]; ++i) { s1p.push_back(s1[i].data()); a1p.push_back(a1[i].data()); }
    CheapTrick(xs[u], lens[u], fs, ts[u], fs0[u], fl[u], &co[u], s1p.data());
    D4C(xs[u], lens[u], fs, ts[u], fs0[u], fl[u], sizes[u], &dopt[u], a1p.data());
    for (int i = 0; i < fl[u]; ++i)
      for (int k = 0; k < bins; ++k) {
        bad += (s1[i][k] != sp[u][i][k]) + (a1[i][k] != ap[u][i][k]);
        values += 2;
      }
  }
  // vectors whose size is not n_utts are refused
  std::vector<CheapTrickOption> two(co.begin(), co.begin() + 2);
  if (CheapTrick(xs, lens, n_utts, fs, ts, fs0, fl, two, sps) != WORLD_B200_EINVAL ||
      D4C(xs, lens, n_utts, fs, ts, fs0, fl, std::vector<int>(2, 1024), dopt, aps) != WORLD_B200_EINVAL) {
    std::printf("FAIL: size check\n");
    return 1;
  }
  if (bad || sizes[0] == sizes[2]) { std::printf("FAIL: %ld of %ld values differ\n", bad, values); return 1; }
  std::printf("OK: per-utterance CheapTrick / D4C overloads == single-utterance calls at fft_size %d / %d / %d (%ld values)\n",
              sizes[0], sizes[1], sizes[2], values);
  return 0;
}
