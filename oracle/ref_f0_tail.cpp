// Test-infrastructure only.  The reference's F0 decision stages -- everything Harvest does after its candidates are
// refined, and DIO's contour selection -- are file-static there, so the compiled reference does not export them.  This
// file pulls the reference's own translation units in from where they lie (-I$(REF)/src; no reference text is
// restated here) and exports C entry points that run those functions on caller-supplied candidate maps:
//
//   RefHarvestTail   RemoveUnreliableCandidates -> FixF0Contour -> SmoothF0Contour on 1 ms candidate rows
//   RefDioContour    GetBestF0Contour -> FixF0Contour on per-band candidate rows
//
// Built into _ref/libworld_ref_tail.so by the Makefile, with the reference's flags, where the reference tree exists.
//
// The headers come first, outside the namespaces, so that the two sources' own #include lines are no-ops there; the
// public functions they define (Harvest, Dio, ...) become namespace members that nothing calls, and the library
// functions they use (fft, decimate, ...) resolve to libworld_ref.so.
#include <math.h>
#include <stddef.h>

#include "world/common.h"
#include "world/constantnumbers.h"
#include "world/dio.h"
#include "world/fft.h"
#include "world/harvest.h"
#include "world/matlabfunctions.h"

namespace ref_harvest_tail {
#include "harvest.cpp"
}  // namespace ref_harvest_tail

namespace ref_dio_tail {
#include "dio.cpp"
}  // namespace ref_dio_tail

extern "C" {

// cand, score: [f0_length][max_candidates] row-major, number_of_candidates (= candidates per band crossing * 7) used
// per row.  Outputs (any may be null): the cleaned rows in the same layout, steps[5][f0_length] = SearchF0Base,
// FixStep1 .. FixStep4 called one by one with FixF0Contour's constants, contour = FixF0Contour itself (so
// steps[4] == contour pins those constants), f0 = the smoothed 1 ms contour.
void RefHarvestTail(const double *cand, const double *score, int f0_length, int number_of_candidates,
                    int max_candidates, double *out_cleaned_cand, double *out_cleaned_score, double *out_steps,
                    double *out_contour, double *out_f0) {
  using namespace ref_harvest_tail;
  double **c = new double *[f0_length], **s = new double *[f0_length];
  for (int i = 0; i < f0_length; ++i) {
    c[i] = new double[number_of_candidates];
    s[i] = new double[number_of_candidates];
    for (int j = 0; j < number_of_candidates; ++j) {
      c[i][j] = cand[(size_t)i * max_candidates + j];
      s[i][j] = score[(size_t)i * max_candidates + j];
    }
  }
  RemoveUnreliableCandidates(f0_length, number_of_candidates, c, s);
  for (int i = 0; i < f0_length; ++i)
    for (int j = 0; j < number_of_candidates; ++j) {
      if (out_cleaned_cand) out_cleaned_cand[(size_t)i * max_candidates + j] = c[i][j];
      if (out_cleaned_score) out_cleaned_score[(size_t)i * max_candidates + j] = s[i][j];
    }
  double *contour = new double[f0_length];
  FixF0Contour(c, s, f0_length, number_of_candidates, contour);
  if (out_steps) {
    double *t = out_steps;
    SearchF0Base(c, s, f0_length, number_of_candidates, t);
    FixStep1(t, f0_length, 0.008, t + f0_length);
    FixStep2(t + f0_length, f0_length, 6, t + 2 * (size_t)f0_length);
    FixStep3(t + 2 * (size_t)f0_length, f0_length, number_of_candidates, c, 0.18, s, t + 3 * (size_t)f0_length);
    FixStep4(t + 3 * (size_t)f0_length, f0_length, 9, t + 4 * (size_t)f0_length);
  }
  if (out_contour)
    for (int i = 0; i < f0_length; ++i) out_contour[i] = contour[i];
  if (out_f0) {
    for (int i = 0; i < f0_length; ++i) out_f0[i] = 0.0;   // as HarvestGeneralBody clears it first
    SmoothF0Contour(contour, f0_length, out_f0);
  }
  delete[] contour;
  for (int i = 0; i < f0_length; ++i) { delete[] c[i]; delete[] s[i]; }
  delete[] c;
  delete[] s;
}

// cand, score: [number_of_candidates][stride] (one row per band), f0_length frames used per row.  out_f0 is cleared
// first: the reference leaves it unwritten when f0_length <= voice_range_minimum.
void RefDioContour(double frame_period, int number_of_candidates, int fs, const double *cand, const double *score,
                   int stride, int f0_length, double f0_floor, double allowed_range, double *out_best,
                   double *out_f0) {
  using namespace ref_dio_tail;
  const double **c = new const double *[number_of_candidates], **s = new const double *[number_of_candidates];
  for (int b = 0; b < number_of_candidates; ++b) {
    c[b] = cand + (size_t)b * stride;
    s[b] = score + (size_t)b * stride;
  }
  double *best = new double[f0_length];
  GetBestF0Contour(f0_length, c, s, number_of_candidates, best);
  for (int i = 0; i < f0_length; ++i) out_f0[i] = 0.0;
  FixF0Contour(frame_period, number_of_candidates, fs, c, best, f0_length, f0_floor, allowed_range, out_f0);
  if (out_best)
    for (int i = 0; i < f0_length; ++i) out_best[i] = best[i];
  delete[] best;
  delete[] c;
  delete[] s;
}

}  // extern "C"
