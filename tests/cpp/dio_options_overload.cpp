// Exercises the per-utterance DIO overload of include/world_b200.hpp: with one DioOption per utterance, every row
// must equal, bit for bit, what the reference-compatible single-utterance Dio() gives that utterance with its own
// option (same kernels, N = 3 with three band lists and two allowed_range values vs N = 1).  Utterance 1 has a
// vibrato and a tight allowed_range that decides some of its frames: the program checks that its row differs from
// the row at the default allowed_range, so the batched call must use each utterance's own value.
#include <cmath>
#include <cstdio>
#include <vector>

#include "world_b200.hpp"

// harmonic tone plus noise; vibrato: phase modulation of `vibrato` rad at 5 Hz
static std::vector<double> tone(int n, int fs, double f0, unsigned seed, double vibrato) {
  const double pi = 3.14159265358979323846;
  std::vector<double> x(n);
  unsigned s = seed;
  for (int i = 0; i < n; ++i) {
    s = s * 1664525u + 1013904223u;
    const double noise = ((s >> 8) / 16777216.0 - 0.5) * 0.01;
    double v = 0.0;
    const double ph = 2.0 * pi * f0 * i / fs + vibrato * std::sin(2.0 * pi * 5.0 * i / fs);
    for (int k = 1; k <= 8; ++k) v += std::sin(k * ph) / k;
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
  for (int u = 0; u < n_utts; ++u) {
    x[u] = tone(lens[u], fs, f0s_true[u], 17u + u, u == 1 ? 2.0 : 0.0);
    xs[u] = x[u].data();
  }

  std::vector<DioOption> per(n_utts);
  for (int u = 0; u < n_utts; ++u) InitializeDioOption(&per[u]);
  per[0].f0_floor = 40.0; per[0].f0_ceil = 1100.0;
  per[1].channels_in_octave = 3.0; per[1].allowed_range = 0.005;
  per[2].f0_floor = 100.0; per[2].f0_ceil = 600.0;
  int fl[3];
  std::vector<std::vector<double>> th(n_utts), fh(n_utts);
  double *thp[3], *fhp[3];
  for (int u = 0; u < n_utts; ++u) {
    fl[u] = GetSamplesForDIO(fs, lens[u], per[u].frame_period);
    th[u].resize(fl[u]); fh[u].resize(fl[u]); thp[u] = th[u].data(); fhp[u] = fh[u].data();
  }
  const int rc = Dio(xs, lens, n_utts, fs, per, thp, fhp);
  if (rc) { std::printf("FAIL: batched Dio with per-utterance options returned %d\n", rc); return 1; }
  int bad = 0, voiced = 0;
  for (int u = 0; u < n_utts; ++u) {
    std::vector<double> t1(fl[u]), f1(fl[u]);
    Dio(xs[u], lens[u], fs, &per[u], t1.data(), f1.data());
    for (int i = 0; i < fl[u]; ++i) {
      bad += (t1[i] != th[u][i]) + (f1[i] != fh[u][i]);
      voiced += f1[i] > 0;
    }
  }
  // utterance 1's allowed_range decides frames: its row at the default allowed_range differs
  {
    DioOption loose = per[1];
    loose.allowed_range = per[0].allowed_range;
    std::vector<double> t1(fl[1]), f1(fl[1]);
    Dio(xs[1], lens[1], fs, &loose, t1.data(), f1.data());
    int differ = 0;
    for (int i = 0; i < fl[1]; ++i) differ += f1[i] != fh[1][i];
    if (differ == 0) { std::printf("FAIL: utterance 1 does not depend on its allowed_range\n"); return 1; }
  }
  // a vector whose size is not n_utts is refused
  std::vector<DioOption> two(per.begin(), per.begin() + 2);
  if (Dio(xs, lens, n_utts, fs, two, thp, fhp) != WORLD_B200_EINVAL) { std::printf("FAIL: size check\n"); return 1; }
  if (bad || voiced == 0) { std::printf("FAIL: %d mismatching values, %d voiced frames\n", bad, voiced); return 1; }
  std::printf("OK: per-utterance Dio overload == single-utterance Dio on %d utterances (%d voiced frames)\n",
              n_utts, voiced);
  return 0;
}
