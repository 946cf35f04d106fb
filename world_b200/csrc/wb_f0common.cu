// wb_f0common.cu -- kernels shared by DIO and Harvest (see wb_f0common.cuh for the design notes).
#include "wb_internal.h"
#include "wb_f0common.cuh"
#include <stdlib.h>

namespace wb {

WB_KERNEL(256, 3) fir_plain_kernel(FirParams p) {
  WB_DYN_SMEM(double, smem);
  const int tid = WB_TID, nth = WB_NTH;
  const int T = 2048, R = 8, G = T / R;
  const int u = blockIdx.y, n0 = blockIdx.x * T;
  const int qlen = p.base_len[u] + p.extra_len;
  if (n0 >= qlen) return;
  const int ntaps = p.ntaps;
  const int seg_len = T + ntaps - 1;
  const int seg_cap = seg_len + 16;
  double *seg = smem;
  double *hrev = seg + (seg_cap + (seg_cap >> 3) + 8);
  const double *in = p.in + (size_t)u * p.in_stride + p.in_origin;
  double *out = p.out + (size_t)u * p.out_stride + p.out_origin;
  for (int j = tid; j < ntaps + 8; j += nth) hrev[j] = j < ntaps ? __ldg(&p.taps_rev[j]) : 0.0;
  const int m0 = n0 - ntaps + 1;
  for (int i = tid; i < seg_len + 8; i += nth) seg[pad8(i)] = (i < seg_len) ? in[m0 + i] : 0.0;
  WB_SYNC();
  for (int g = tid; g < G; g += nth) {
    const int base = R * g;
    double acc[8], win[8];
#pragma unroll
    for (int r = 0; r < R; ++r) { acc[r] = 0.0; win[r] = seg[pad8(base + r)]; }
    for (int j0 = 0; j0 < ntaps; j0 += R) {
#pragma unroll
      for (int jj = 0; jj < R; ++jj) {
        const double hj = hrev[j0 + jj];
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] = fma(hj, win[(r + jj) & (R - 1)], acc[r]);
        win[jj] = seg[pad8(base + R + j0 + jj)];
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
      if (n0 + base + r < qlen) out[n0 + base + r] = acc[r];
  }
}

// ---------------------------------------------------------------------------------------------
// Event trains of one (utterance, band).  Fine edge positions e_j are appended to global lists
// (complete, for the rare look-back) and to shared-memory rings; every pair of consecutive edges
// defines the (location, interval) sample interp1 sees (matlabfunctions.cpp:157-176 through
// dio.cpp:357-393 / harvest.cpp:162-198):  x_j = (e_j + e_{j+1}) / 2 / afs,  y_j = afs / (e_{j+1} - e_j).
// x_j and y_j are evaluated ONCE per interval (same expressions as the reference) and kept in rings.
#ifndef WB_RING
#define WB_RING 256   // location / value rings per train; older intervals are recomputed from the global edge lists
#endif
#define WB_FCHUNK 256  // frames finalised per round (= WB_SWEEP_THREADS)
struct Trains {
  const double *g[4];   // global edge lists: history rings of `cap` entries (index modulo cap)
  double *xr, *yr;      // shared rings [4][WB_RING]: interval locations, interval values
  int cap;
  int ifrom[4];         // interval rings hold indices >= ifrom
  double afs;
};
// Edges are read back from global memory (L2): an edge ring in shared memory cost a CTA per SM.  A signal
// with far more crossings than the band frequency suggests (a loud out-of-band tone) wraps the ring; only a
// look-back beyond the last `cap` events -- one train silent for that long while another keeps firing --
// cannot be served; the sweep loop detects that case (status bit 4) before such a read can happen.
WB_DEV double edge_at(const Trains &T, int q, int i) {
  int s = i;
  while (s >= T.cap) s -= T.cap;   // wraps are rare and few: cheaper in registers than a division
  return T.g[q][s];
}
WB_DEV double loc_at(const Trains &T, int q, int j) {
  return j >= T.ifrom[q] ? T.xr[q * WB_RING + (j & (WB_RING - 1))] : (edge_at(T, q, j) + edge_at(T, q, j + 1)) / 2.0 / T.afs;
}
WB_DEV double val_at(const Trains &T, int q, int j) {
  return j >= T.ifrom[q] ? T.yr[q * WB_RING + (j & (WB_RING - 1))] : T.afs / (edge_at(T, q, j + 1) - edge_at(T, q, j));
}

// interp1 at time t given count = #{j : x_j <= t}: k = clamp(count, 1, n_int-1) picks the segment
WB_DEV double train_value(const Trains &T, int q, int count, int n_int, double t) {
  const int k = imin(n_int - 1, imax(1, count));
  const double x0 = loc_at(T, q, k - 1), x1 = loc_at(T, q, k);
  const double y0 = val_at(T, q, k - 1), y1 = val_at(T, q, k);
  const double s = (t - x0) / (x1 - x0);
  return y0 + s * (y1 - y0);
}

// smallest frame index i with t_i >= x, t_i = i * frame_period / 1000.0 (the reference's expression)
WB_DEV int first_frame_at_or_after(double x, double frame_period) {
  int g = (int)ceil(x * 1000.0 / frame_period);
  if (g < 0) g = 0;
  while (g > 0 && !((g - 1) * frame_period / 1000.0 < x)) --g;
  while (g * frame_period / 1000.0 < x) ++g;
  return g;
}

#ifdef WB_EMU
static inline void smem_add_u64(unsigned long long *p, unsigned long long v) { *p += v; }
#else
__device__ __forceinline__ void smem_add_u64(unsigned long long *p, unsigned long long v) { atomicAdd(p, v); }
#endif

// Exclusive scan of G packed counters (4 x 16 bit) held in shared memory, in place; adds the
// running totals in `carry` (also packed) and returns the new running total to every thread.
// CUDA path: requires blockDim.x == G (one counter per thread).
WB_DEV unsigned long long scan_packed(unsigned long long *c, int G, unsigned long long carry,
                                      unsigned long long *warp_tot /* >= 33 */) {
#ifdef WB_EMU
  (void)warp_tot;
  unsigned long long run = carry;
  for (int g = 0; g < G; ++g) { const unsigned long long v = c[g]; c[g] = run; run += v; }
  return run;
#else
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, nw = G >> 5;
  const unsigned long long v = c[tid];
  unsigned long long inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_tot[w] = inc;
  __syncthreads();
  unsigned long long base = carry, all = carry;
  for (int i = 0; i < nw; ++i) { const unsigned long long t = warp_tot[i]; if (i < w) base += t; all += t; }
  c[tid] = base + inc - v;
  __syncthreads();
  return all;
#endif
}

// One frame of one band from the four interpolated values (dio.cpp:441-465, 562-566 / harvest.cpp:240-254)
WB_DEV void sweep_store_candidate(const SweepParams &p, double v0, double v1, double v2, double v3, int i, double bf,
                                  double *cand, double *score) {
  double c = (v0 + v1 + v2 + v3) / 4.0, sc = 0.0;
  if (p.mode == 0) {
    sc = sqrt(((v0 - c) * (v0 - c) + (v1 - c) * (v1 - c) + (v2 - c) * (v2 - c) + (v3 - c) * (v3 - c)) / 3.0);
    if (c > bf || c < bf / 2.0 || c > p.f0_ceil || c < p.f0_floor) { c = 0.0; sc = 100000.0; }
  } else {
    if (c > bf * 1.1 || c < bf * 0.9 || c > p.f0_ceil || c < p.f0_floor) c = 0.0;
  }
  cand[i] = c;
  if (score) score[i] = sc / (c + kTiny);  // dio.cpp:562-566
}

// Finalises frames [f_begin, f_end): for every train the intervals still ahead of the frame cursor
// (indices lo_j .. ni-1) are binned by the first frame they precede-or-equal; a packed block scan
// turns the bins into per-frame interval counts, i.e. interp1's segment index, without any search.
// lo_j advances past the intervals consumed.  Block-cooperative; ends with a barrier.
WB_DEV void finalize_frames(const SweepParams &p, const Trains &T, int *lo_j, const int *ni, int f_begin, int f_end,
                            unsigned long long *marks, unsigned long long *orig, unsigned long long *scan_tmp,
                            double bf, double *cand, double *score) {
  const int tid = WB_TID, nth = WB_NTH;
  for (int c0 = f_begin; c0 < f_end; c0 += WB_FCHUNK) {
    const int c1 = imin(f_end, c0 + WB_FCHUNK);
    for (int i = tid; i < WB_FCHUNK; i += nth) marks[i] = 0ull;
    WB_SYNC();
    for (int q = 0; q < 4; ++q)
      for (int j = lo_j[q] + tid; j < ni[q]; j += nth) {
        int m = first_frame_at_or_after(loc_at(T, q, j), p.frame_period);
        if (m < c0) m = c0;
        if (m < c1) smem_add_u64(&marks[m - c0], 1ull << (16 * q));
      }
    WB_SYNC();
    for (int i = tid; i < WB_FCHUNK; i += nth) orig[i] = marks[i];
    WB_SYNC();
    const unsigned long long all = scan_packed(marks, WB_FCHUNK, 0ull, scan_tmp);
    for (int i = tid; i < c1 - c0; i += nth) {
      const unsigned long long inc = marks[i] + orig[i];
      const double t = (c0 + i) * p.frame_period / 1000.0;
      const double v0 = train_value(T, 0, lo_j[0] + (int)(inc & 0xffffull), ni[0], t);
      const double v1 = train_value(T, 1, lo_j[1] + (int)((inc >> 16) & 0xffffull), ni[1], t);
      const double v2 = train_value(T, 2, lo_j[2] + (int)((inc >> 32) & 0xffffull), ni[2], t);
      const double v3 = train_value(T, 3, lo_j[3] + (int)((inc >> 48) & 0xffffull), ni[3], t);
      sweep_store_candidate(p, v0, v1, v2, v3, c0 + i, bf, cand, score);
    }
    lo_j[0] += (int)(all & 0xffffull); lo_j[1] += (int)((all >> 16) & 0xffffull);
    lo_j[2] += (int)((all >> 32) & 0xffffull); lo_j[3] += (int)((all >> 48) & 0xffffull);
    WB_SYNC();
  }
}

// Bins N/2 - 1 and N/2 of the spectrum of the signal the band filters see, N = the reference's fft_size for
// this utterance (dio.cpp:590-592 / harvest.cpp:1164-1165, computed on the host).  The reference's spectral "mirroring" loop (dio.cpp:319-328, harvest.cpp:122-135) stores
// product bin i in slot N - i - 1 as well; for i = N/2 - 1 and N/2 those slots lie inside the half its c2r
// reads, so both bins end up as Q = Ys[N/2] * (Ys[N/2-1] * F[N/2-1]) instead of Ys[k] F[k].  What that adds to
// every band's filtered signal is a near-Nyquist ripple: negligible next to a real signal when the band's
// window is long, visible for the 4..12-tap windows of heavy decimation, and the ONLY thing left in digital
// silence -- where it gives the reference a zero crossing every sample or two, which is why it calls silence
// unvoiced instead of extrapolating the last interval.  band_sweep_ripple_kernel adds the same ripple (DIO
// always; Harvest only when its input is not decimated, the one case where exact zeros survive to this point).
//   exp(-j 2 pi (N/2 - 1) n / N) = (-1)^n exp(+j 2 pi n / N);  2 n / N is exact (N is a power of two).
WB_KERNEL(256, 2) nyquist_bins_kernel(NyquistParams p) {
  WB_SHARED double red[WB_RED_DOUBLES];
  const int tid = WB_TID, nth = WB_NTH, u = blockIdx.x;
  const int N = p.nfft[u];
  const int len = p.y_len[u] + 2 * p.c;
  const double *s = p.sig + (size_t)u * p.stride + p.origin;
  double a = 0.0, b = 0.0, d = 0.0;
  for (int q = tid; q < len; q += nth) {
    const int n = q - p.c;
    const double v = (n & 1) ? -s[q] : s[q];
    const double ang = 2.0 * n / N;
    a = fma(v, cospi(ang), a);
    b = fma(v, sinpi(ang), b);
    d += v;
  }
  block_sum2(a, b, red);
  d = block_sum(d, red);
  if (tid == 0) {
    double *o = p.nyq + 4 * (size_t)u;
    o[0] = a; o[1] = b; o[2] = d; o[3] = static_cast<double>(N);
  }
}


// kRipple = 1 adds the near-Nyquist ripple of the reference's spectral mirroring loop (nyquist_bins_kernel
// above); the default instantiation carries none of it.
template <int kRipple>
WB_DEV void sweep_body(const SweepParams &p, const int b, const int u) {
  WB_DYN_SMEM(double, smem);
  const int tid = WB_TID, nth = WB_NTH;
  const int T = WB_SWEEP_T, R = WB_SWEEP_R, G = T / R;
  const int ntaps = p.ntaps[b], shift = p.shift[b];
  const int seg_len = T + ntaps - 1;
  const int seg_cap = T + p.max_taps + 16;
  double *seg = smem;                                   // padded: pad8(seg_cap)
  double *hrev = seg + (seg_cap + (seg_cap >> 3) + 8);  // max_taps + 8
  double *st = hrev + (p.max_taps + 8);                 // T + 8: [0..1] carry, [2..T+2) this tile
  unsigned long long *cnt = reinterpret_cast<unsigned long long *>(st + (T + 8 + ((T + 8) >> 3) + 8));  // G + 40
  double *ring = reinterpret_cast<double *>(cnt + (G + 40));                                           // 2 * 4 * WB_RING
  unsigned long long *marks = reinterpret_cast<unsigned long long *>(ring + 8 * WB_RING);              // WB_FCHUNK
  unsigned long long *orig = marks + WB_FCHUNK;                                                        // WB_FCHUNK

  const int ylen = p.y_len[u];
  const double *sig = p.sig + (size_t)u * p.sig_stride + p.sig_origin;
  double *edges = p.edges + (size_t)u * p.edge_stride + (size_t)p.edge_off[b];
  const int cap = p.edge_cap[b];
  for (int j = tid; j < ntaps; j += nth) hrev[j] = __ldg(&p.taps_rev[p.tap_off[b] + j]);
  for (int j = ntaps + tid; j < ntaps + 8; j += nth) hrev[j] = 0.0;
  if (tid == 0) { st[0] = 0.0; st[1] = 0.0; }
  Trains tr;
  tr.xr = ring; tr.yr = ring + 4 * WB_RING; tr.afs = p.afs; tr.cap = cap;
  for (int q = 0; q < 4; ++q) { tr.g[q] = edges + (size_t)q * cap; tr.ifrom[q] = 0; }
  int ni[4] = {0, 0, 0, 0};   // intervals known so far per train (= max(0, events - 1))
  int tot[4] = {0, 0, 0, 0};  // running event counts per train (identical in every thread)
  int lo_j[4] = {0, 0, 0, 0}; // per train: intervals below this index lie before every unfinished frame
  int next_frame = 0;         // frames [0, next_frame) are done
  const int nf = p.n_frames[u];
  double *cand = p.cand + ((size_t)u * p.n_bands + b) * p.frame_stride;
  double *score = p.score ? p.score + ((size_t)u * p.n_bands + b) * p.frame_stride : nullptr;
  const double bf = p.boundary[b];
  WB_SYNC();
  // DIO: this band's window at bins N/2 - 1 and N/2, combined with the utterance's spectrum there into the
  // amplitudes of the ripple  (-1)^m (2 Re(dq e^{-j 2 pi m / N}) + dn) / N  at filtered-signal index m - shift
  double rip_a = 0.0, rip_b = 0.0, rip_d = 0.0, rot_c = 1.0, rot_s = 0.0, inv_half_n = 0.0;
  if (kRipple) {
    double *red = reinterpret_cast<double *>(cnt);   // idle until the event phase of the first tile
    const double *ny = p.nyq + 4 * (size_t)u;
    const double nf = ny[3];
    double f1r = 0.0, f1i = 0.0, f2 = 0.0;
    for (int k = tid; k < ntaps; k += nth) {
      const double w = hrev[ntaps - 1 - k];
      const double v = (k & 1) ? -w : w;
      const double ang = 2.0 * k / nf;
      f1r = fma(v, cospi(ang), f1r);
      f1i = fma(v, sinpi(ang), f1i);
      f2 += v;
    }
    block_sum2(f1r, f1i, red);
    f2 = block_sum(f2, red);
    const double p_re = ny[0] * f1r - ny[1] * f1i, p_im = ny[0] * f1i + ny[1] * f1r;   // Ys[N/2-1] F[N/2-1]
    rip_a = 2.0 * (ny[2] * p_re - p_re) / nf;
    rip_b = 2.0 * (ny[2] * p_im - p_im) / nf;
    rip_d = (ny[2] * p_re - ny[2] * f2) / nf;
    rot_c = cospi(2.0 / nf); rot_s = sinpi(2.0 / nf);
    inv_half_n = 2.0 / nf;
    WB_SYNC();
  }

  // Tile k produces outputs n0..n0+T-1 into st[2..]; events are detected for positions
  // i = n0-2 .. n0+T-3 (they need s[i], s[i+1], s[i+2]); the last two outputs carry over.
  for (int n0 = 0; n0 < ylen + 2; n0 += T) {
    const int m0 = n0 + shift - ntaps + 1;  // seg[i] = s(m0 + i)
    for (int i = tid; i < seg_len + 8; i += nth) seg[pad8(i)] = (i < seg_len) ? sig[m0 + i] : 0.0;
    WB_SYNC();
    for (int g = tid; g < G; g += nth) {
      const int base = R * g;
      double acc[WB_SWEEP_R], win[WB_SWEEP_R];
      // pad8(8 (g+1) + 8 it + jj) = 9 (g+1) + 9 it + jj: one running pointer, immediate offsets
      const double *sp = seg + 9 * (g + 1);
      const double *hp = hrev;
#pragma unroll
      for (int r = 0; r < R; ++r) { acc[r] = 0.0; win[r] = seg[9 * g + r]; }
      for (int j0 = 0; j0 < ntaps; j0 += R, sp += 9, hp += R) {
#pragma unroll
        for (int jj = 0; jj < R; ++jj) {
          const double hj = hp[jj];  // zero beyond ntaps
#pragma unroll
          for (int r = 0; r < R; ++r) acc[r] = fma(hj, win[(r + jj) & (R - 1)], acc[r]);
          win[jj] = sp[jj];
        }
      }
      if (kRipple) {
        const int m0 = n0 + base + shift;              // n0 and base are even: the parity of m is that of shift + r
        double c = cospi(inv_half_n * m0), sn = sinpi(inv_half_n * m0);
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const double ripple = fma(rip_a, c, fma(rip_b, sn, rip_d));
          acc[r] += ((shift + r) & 1) ? -ripple : ripple;
          const double c2 = fma(c, rot_c, -(sn * rot_s));
          sn = fma(sn, rot_c, c * rot_s);
          c = c2;
        }
      }
#pragma unroll
      for (int r = 0; r < R; ++r) st[pad8(2 + base + r)] = acc[r];
    }
    WB_SYNC();
    if (p.debug_skip >= 2) { WB_SYNC(); continue; }
    // train 0: s[i] > 0 >= s[i+1]   train 1: s[i] < 0 <= s[i+1]          (i >= 0, i+1 <= ylen-1)
    // train 2: d[i] > 0 >= d[i+1]   train 3: d[i] < 0 <= d[i+1], d[i] = s[i+1]-s[i]  (i+1 <= ylen-2)
    // Pass 1 marks events (bit 4 r + q of a per-group mask) and counts them; a packed scan gives
    // every group its offsets; pass 2 compacts the event POSITIONS into per-train lists (no
    // arithmetic); pass 3 walks the dense lists and evaluates the fine edge (one division per
    // event, all lanes busy) -- high bands have an event every few samples, so doing the division
    // inside the divergent per-position branches cost more than the FIR itself (r1h experiment).
    unsigned *emask = reinterpret_cast<unsigned *>(marks);  // G words (marks is idle here)
    int *elist = reinterpret_cast<int *>(seg);              // 4 x (T/2) positions (seg is idle after the FIR)
    for (int g = tid; g < G; g += nth) {
      unsigned long long c = 0ull;
      unsigned m = 0u;
      const int base = R * g;
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int i = n0 - 2 + base + r;
        const double a = st[pad8(base + r)], bb = st[pad8(base + r + 1)], cc = st[pad8(base + r + 2)];
        const double d0 = bb - a, d1 = cc - bb;
        if (i >= 0 && i + 1 <= ylen - 1) {
          if (0.0 < a && bb <= 0.0) { c += 1ull; m |= 1u << (4 * r); }
          if (a < 0.0 && 0.0 <= bb) { c += 1ull << 16; m |= 2u << (4 * r); }
        }
        if (i >= 0 && i + 1 <= ylen - 2) {
          if (0.0 < d0 && d1 <= 0.0) { c += 1ull << 32; m |= 4u << (4 * r); }
          if (d0 < 0.0 && 0.0 <= d1) { c += 1ull << 48; m |= 8u << (4 * r); }
        }
      }
      cnt[g] = c;
      emask[g] = m;
    }
    WB_SYNC();
    const unsigned long long tile_total = scan_packed(cnt, G, 0ull, cnt + G + 4);  // <= 2048 each: fits 16 bit
    int tcount[4];  // events of this tile
    for (int q = 0; q < 4; ++q) tcount[q] = (int)((tile_total >> (16 * q)) & 0xffffull);
    for (int g = tid; g < G; g += nth) {
      const unsigned long long o = cnt[g];
      int off[4] = {(int)(o & 0xffffull), (int)((o >> 16) & 0xffffull), (int)((o >> 32) & 0xffffull), (int)((o >> 48) & 0xffffull)};
      unsigned m = emask[g];
      while (m) {
#ifdef WB_EMU
        const int bit = __builtin_ctz(m);
#else
        const int bit = __ffs((int)m) - 1;
#endif
        m &= m - 1u;
        const int q = bit & 3, r = bit >> 2;
        elist[q * (T / 2) + off[q]] = R * g + r;  // position relative to n0 - 2
        ++off[q];
      }
    }
    WB_SYNC();
    for (int q = 0; q < 4; ++q) {
      for (int e = tid; e < tcount[q]; e += nth) {
        const int pos = elist[q * (T / 2) + e];
        const double a = st[pad8(pos)], bb = st[pad8(pos + 1)];
        double v;
        if (q < 2) {
          v = (double)(n0 - 2 + pos + 1) - a / (bb - a);
        } else {
          const double d0 = bb - a, d1 = st[pad8(pos + 2)] - bb;
          v = (double)(n0 - 2 + pos + 1) - d0 / (d1 - d0);
        }
        int o = tot[q] + e;
        while (o >= cap) o -= cap;
        edges[(size_t)q * cap + o] = v;
      }
    }
    tot[0] += (int)(tile_total & 0xffffull); tot[1] += (int)((tile_total >> 16) & 0xffffull);
    tot[2] += (int)((tile_total >> 32) & 0xffffull); tot[3] += (int)((tile_total >> 48) & 0xffffull);
    // unfinished frames still need the intervals from lo_j - 1 on: their edges must not have been overwritten
    if (tid == 0)
      for (int q = 0; q < 4; ++q)
        if (tot[q] - cap > imax(0, lo_j[q] - 1)) atomicOr_status(p.status, 4);
#ifndef WB_EMU
    __threadfence_block();
#endif
    WB_SYNC();
    if (tid == 0) { st[pad8(0)] = st[pad8(T)]; st[pad8(1)] = st[pad8(T + 1)]; }
    if (p.debug_skip >= 1) { WB_SYNC(); continue; }
    // ---- new intervals of this tile -> location / value rings
    bool can = true;
    for (int q = 0; q < 4; ++q) {
      const int n_new = imax(0, tot[q] - 1);
      const int from = imax(0, n_new - WB_RING);
      for (int j = imax(ni[q], from) + tid; j < n_new; j += nth) {
        const double e0 = edge_at(tr, q, j), e1 = edge_at(tr, q, j + 1);
        tr.xr[q * WB_RING + (j & (WB_RING - 1))] = (e0 + e1) / 2.0 / p.afs;
        tr.yr[q * WB_RING + (j & (WB_RING - 1))] = p.afs / (e1 - e0);
      }
      ni[q] = n_new;
      tr.ifrom[q] = from;
      if (n_new < 1) can = false;
    }
    WB_SYNC();
    // ---- streaming candidates: every frame whose time lies before the last complete interval of
    // all four trains can be interpolated now.
    if (can) {
      double t_safe = loc_at(tr, 0, ni[0] - 1);
      for (int q = 1; q < 4; ++q) t_safe = dmin(t_safe, loc_at(tr, q, ni[q] - 1));
      int i_safe = first_frame_at_or_after(t_safe, p.frame_period);  // frames below have t_i < t_safe
      if (i_safe > nf) i_safe = nf;
      if (i_safe > next_frame) {
        finalize_frames(p, tr, lo_j, ni, next_frame, i_safe, marks, orig, cnt + G + 4, bf, cand, score);
        next_frame = i_safe;
      }
    }
    WB_SYNC();
  }
  // ---- frames after the last complete interval (interp1 extrapolates from the last two samples)
  bool ok = true;
  for (int q = 0; q < 4; ++q) {
    const int n_int = tot[q] < 2 ? 0 : tot[q] - 1;  // ZeroCrossingEngine returns count-1 (0 if count<2)
    if (n_int - 2 <= 0) ok = false;                 // CheckEvent(n - 2), dio.cpp:475-484
  }
  if (ok) {
    finalize_frames(p, tr, lo_j, ni, next_frame, nf, marks, orig, cnt + G + 4, bf, cand, score);
  } else {
    for (int i = tid; i < nf; i += nth) {
      cand[i] = 0.0;
      if (score) score[i] = 100000.0 / (0.0 + kTiny);
    }
  }
}

WB_KERNEL(WB_SWEEP_THREADS, 3) band_sweep_kernel(SweepParams p) { sweep_body<0>(p, blockIdx.x, blockIdx.y); }          // Harvest on decimated input
WB_KERNEL(WB_SWEEP_THREADS, 3) band_sweep_ripple_kernel(SweepParams p) { sweep_body<1>(p, blockIdx.x, blockIdx.y); }   // DIO; Harvest at ratio 1
// the same streaming sweep over a device list of (utterance, band) pairs: bands whose complete edge lists did not fit
// (band_fir_events_kernel), i.e. far more zero crossings than the band frequency allows for -- usually none
WB_KERNEL(WB_SWEEP_THREADS, 3) band_sweep_list_kernel(SweepParams p) {
  const int n = *p.redo_count;
  for (int at = blockIdx.x; at < n; at += gridDim.x) {
    const int pair = p.redo_list[at];
    sweep_body<0>(p, pair % p.n_bands, pair / p.n_bands);
    WB_SYNC();
  }
}

// =============================================================================================
// Round 2: the Harvest sweep on decimated input as two kernels.
//
// band_sweep_kernel does everything for one (utterance, band) in one streaming pass: FIR tile, event detection,
// compaction, interval rings, frame finalisation -- fourteen block barriers per tile and a round trip of the fine
// edges through global memory, which leaves the FIR's FP64 pipe idle for much of the tile.
// Split:
//   band_fir_events_kernel  FIR (the same register tile, the same FMA order: bit-identical filtered samples) +
//                           the four event trains of every tile, fine edges appended to COMPLETE per-train lists
//                           in global memory (written once, never read back here).  Three block barriers per tile.
//                           The input segment of the next tile arrives by TMA (cp.async.bulk + mbarrier) while the
//                           current one is filtered: nine outputs per thread make consecutive threads 9 doubles
//                           apart -- conflict free without padding, so the segment is one contiguous bulk copy.
//   band_interp_kernel      edge lists -> intervals -> interp1 onto the frame grid, 256 frames per round; interval
//                           counts per frame by a fill (every interval owns the frames between its first frame and
//                           the next interval's), no search, no scan.
// A band whose lists overflow their capacity (far more crossings than its frequency allows for: a loud out-of-band
// tone) is left to the streaming kernel, whose history rings wrap instead (band_sweep_list_kernel).
#ifndef WB_EMU
WB_DEV unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
WB_DEV void mbar_init(unsigned long long *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
WB_DEV void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// 1-D TMA: `bytes` (multiple of 16) from global (16-byte aligned) to shared (16-byte aligned); completes on `bar`
WB_DEV void tma_load_1d(void *dst, const void *src, unsigned bytes, unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
WB_DEV void mbar_wait(unsigned long long *bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
#endif

// Warp-specialised: warps 0-3 (128 threads) only filter -- tile t+1 while warps 4-7 pick the events of tile t out of
// the other half of the double-buffered output tile.  The first version ran the two phases one after the other in
// all eight warps: the FP64 pipe idled through every event phase.
// Hand-over by named barriers (bar.arrive on one side, bar.sync on the other): full[2] filter -> events,
// empty[2] events -> filter; the input segments arrive by TMA on two mbarriers.
#define WB_FE_GROUP 128                      // threads per role
#define WB_FE_TILE (WB_FE_R * WB_FE_GROUP)   // outputs per tile
#ifndef WB_EMU
WB_DEV void bar_sync_named(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
WB_DEV void bar_arrive_named(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }
#endif

// acc[r] += h * w[r], r = 0..8, as ONE block of nine DFMAs in this order.  A DFMA reads three 64-bit operands; the
// register file delivers two per issue slot of the half-rate FP64 pipe, the third has to come from the operand-reuse
// cache, i.e. from the previous instruction's same slot.  Left to the scheduler, the nine FMAs of a tap were
// interleaved with those of other taps (few DFMAs carried a reuse flag); written as one block `h` stays in its slot
// for all nine.
WB_DEV void fe_fma9(double (&acc)[9], double h, double w0, double w1, double w2, double w3, double w4, double w5,
                    double w6, double w7, double w8) {
#ifdef WB_EMU
  acc[0] = fma(h, w0, acc[0]); acc[1] = fma(h, w1, acc[1]); acc[2] = fma(h, w2, acc[2]);
  acc[3] = fma(h, w3, acc[3]); acc[4] = fma(h, w4, acc[4]); acc[5] = fma(h, w5, acc[5]);
  acc[6] = fma(h, w6, acc[6]); acc[7] = fma(h, w7, acc[7]); acc[8] = fma(h, w8, acc[8]);
#else
  asm("fma.rn.f64 %0, %9, %10, %0;\n\t"
      "fma.rn.f64 %1, %9, %11, %1;\n\t"
      "fma.rn.f64 %2, %9, %12, %2;\n\t"
      "fma.rn.f64 %3, %9, %13, %3;\n\t"
      "fma.rn.f64 %4, %9, %14, %4;\n\t"
      "fma.rn.f64 %5, %9, %15, %5;\n\t"
      "fma.rn.f64 %6, %9, %16, %6;\n\t"
      "fma.rn.f64 %7, %9, %17, %7;\n\t"
      "fma.rn.f64 %8, %9, %18, %8;"
      : "+d"(acc[0]), "+d"(acc[1]), "+d"(acc[2]), "+d"(acc[3]), "+d"(acc[4]), "+d"(acc[5]), "+d"(acc[6]), "+d"(acc[7]),
        "+d"(acc[8])
      : "d"(h), "d"(w0), "d"(w1), "d"(w2), "d"(w3), "d"(w4), "d"(w5), "d"(w6), "d"(w7), "d"(w8));
#endif
}

// FIR of register group g (outputs 9 g .. 9 g + 8 of the tile): the same FMA order as band_sweep_kernel
WB_DEV void fe_fir_group(const double *seg, const double *hrev, int ntaps, int g, double *st) {
  const int R = WB_FE_R, base = R * g;
  double acc[WB_FE_R], win[WB_FE_R];
  const double *sp = seg + base + R;
  const double *hp = hrev;
#pragma unroll
  for (int r = 0; r < R; ++r) { acc[r] = 0.0; win[r] = seg[base + r]; }
  for (int j0 = 0; j0 < ntaps; j0 += R, sp += R, hp += R) {
#pragma unroll
    for (int jj = 0; jj < R; ++jj) {
      const double hj = hp[jj];
      fe_fma9(acc, hj, win[jj % 9], win[(jj + 1) % 9], win[(jj + 2) % 9], win[(jj + 3) % 9], win[(jj + 4) % 9],
              win[(jj + 5) % 9], win[(jj + 6) % 9], win[(jj + 7) % 9], win[(jj + 8) % 9]);
      win[jj] = sp[jj];
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) st[base + r] = acc[r];
}

// the 11 filtered samples group g looks at: positions pos = 9 g + r (relative to n0 - 2) need s[pos .. pos + 2];
// sample p of that axis is carry[p] for p < 2 (the last two outputs of the previous tile), st[p - 2] otherwise
WB_DEV void fe_load_group(const double *st, double c0, double c1, int g, double (&v)[WB_FE_R + 2]) {
  const int base = WB_FE_R * g;
#pragma unroll
  for (int k = 0; k < WB_FE_R + 2; ++k) {
    const int pp = base + k;
    v[k] = pp >= 2 ? st[pp - 2] : (pp == 0 ? c0 : c1);
  }
}

// sign tests on the bit pattern (integer pipe; DSETP would queue behind the filter's DFMAs on the FP64 pipe):
// v > 0 <=> pattern > 0 as a signed integer; v < 0 <=> sign bit set and not -0.0.  (NaN never occurs here.)
WB_DEV long long fe_bits(double v) {
#ifdef WB_EMU
  long long b; memcpy(&b, &v, 8); return b;
#else
  return __double_as_longlong(v);
#endif
}
WB_DEV bool fe_pos(long long b) { return b > 0; }
WB_DEV bool fe_neg(long long b) { return b < 0 && b != (long long)0x8000000000000000ull; }

// Events of group g: 4 flag bits per position (bit q = train q, position r at bits 4 r .. 4 r + 3) and the packed
// per-train counts.  `edge` = the tile touches the ends of the signal (positions before sample 0 / after the last
// pair are not events); interior tiles skip those tests.
WB_DEV unsigned long long fe_mask_group(const double (&v)[WB_FE_R + 2], int i0, int ylen, bool edge, unsigned long long *counts) {
  long long sb[WB_FE_R + 2], db[WB_FE_R + 1];
#pragma unroll
  for (int k = 0; k < WB_FE_R + 2; ++k) sb[k] = fe_bits(v[k]);
#pragma unroll
  for (int k = 0; k < WB_FE_R + 1; ++k) db[k] = fe_bits(v[k + 1] - v[k]);
  unsigned long long mask = 0ull, c = 0ull;
#pragma unroll
  for (int r = 0; r < WB_FE_R; ++r) {
    unsigned m = 0u;
    if (fe_pos(sb[r]) && !fe_pos(sb[r + 1])) m |= 1u;   // s[i] > 0 >= s[i+1]
    if (fe_neg(sb[r]) && !fe_neg(sb[r + 1])) m |= 2u;   // s[i] < 0 <= s[i+1]
    if (fe_pos(db[r]) && !fe_pos(db[r + 1])) m |= 4u;   // d[i] > 0 >= d[i+1]
    if (fe_neg(db[r]) && !fe_neg(db[r + 1])) m |= 8u;   // d[i] < 0 <= d[i+1]
    if (edge) {
      const int i = i0 + r;
      if (!(i >= 0 && i + 1 <= ylen - 1)) m &= ~3u;
      if (!(i >= 0 && i + 1 <= ylen - 2)) m &= ~12u;
    }
    mask |= (unsigned long long)m << (4 * r);
    c += (unsigned long long)(m & 1u) + ((unsigned long long)((m >> 1) & 1u) << 16) +
         ((unsigned long long)((m >> 2) & 1u) << 32) + ((unsigned long long)((m >> 3) & 1u) << 48);
  }
  *counts = c;
  return mask;
}

// fine edges of group g's events (one division per event), appended in position order at tot[q] + (offsets in o)
WB_DEV void fe_emit_group(const double (&v)[WB_FE_R + 2], unsigned long long mask, int i0, unsigned long long o,
                          const int (&tot)[4], double *edges, int cap) {
  int off[4] = {(int)(o & 0xffffull), (int)((o >> 16) & 0xffffull), (int)((o >> 32) & 0xffffull), (int)((o >> 48) & 0xffffull)};
  while (mask) {
#ifdef WB_EMU
    const int bit = __builtin_ctzll(mask);
#else
    const int bit = __ffsll((long long)mask) - 1;
#endif
    mask &= mask - 1ull;
    const int r = bit >> 2, q = bit & 3;
    double a = v[0], bb = v[1], cc = v[2];
#pragma unroll
    for (int k = 1; k < WB_FE_R; ++k)            // register array: select by comparison, not by a runtime index
      if (k == r) { a = v[k]; bb = v[k + 1]; cc = v[k + 2]; }
    double e;
    if (q < 2) {
      e = (double)(i0 + r + 1) - a / (bb - a);
    } else {
      const double d0 = bb - a, d1 = cc - bb;
      e = (double)(i0 + r + 1) - d0 / (d1 - d0);
    }
    const int at = tot[q] + off[q];
    ++off[q];
    if (at < cap) edges[(size_t)q * cap + at] = e;
  }
}

// A CTA takes a PAIR of bands -- band pr (long filter) and band n_bands - 1 - pr (short filter) -- and alternates
// between them tile by tile: filter work per tile varies 13x across bands while the event work is about constant,
// so a CTA with one band is either waiting for its filter warps or for its event warps; the pair sums are within
// 2x of each other and sit on the filter side.  Both bands read the same input segment (the long band's).
struct FeBand {
  int ntaps, seg_off, cap, band;   // seg_off: where this band's segment starts inside the pair's (long) segment
  double *edges;
};

WB_KERNEL(2 * WB_FE_GROUP, 3) band_fir_events_kernel(SweepParams p) {
  WB_DYN_SMEM(double, smem);
  const int pr = blockIdx.x, u = blockIdx.y;
  const int T = WB_FE_TILE, R = WB_FE_R, G = WB_FE_GROUP;
  const int segd = fe_seg_doubles(p.max_taps);
  double *segbuf[2] = {smem, smem + segd};
  const int hcap = ((p.max_taps + R - 1) / R) * R + R;
  double *hrev[2] = {smem + 2 * segd, smem + 2 * segd + hcap};
  double *stbuf[2] = {hrev[1] + hcap, hrev[1] + hcap + (T + 2)};
  unsigned long long *wtot = reinterpret_cast<unsigned long long *>(stbuf[1] + (T + 2));   // [2][4] warp totals
  unsigned long long *bars = wtot + 8;           // two mbarriers
  const int ylen = p.y_len[u];
  const size_t abs0 = (size_t)u * p.sig_stride + p.sig_origin;   // index of s(0) in p.sig
  const int n_tiles = (ylen + 2 + T - 1) / T;
  const int b_long = pr, b_short = p.n_bands - 1 - pr;
  const int nslot = b_short > b_long ? 2 : 1;    // the middle band of an odd count is alone
  FeBand fb[2];
  const int lead = p.shift[b_long] - p.ntaps[b_long] + 1;     // segment of tile t starts at s(t T + lead)
  for (int s = 0; s < nslot; ++s) {
    const int b = s == 0 ? b_long : b_short;
    fb[s].band = b; fb[s].ntaps = p.ntaps[b];
    fb[s].seg_off = (p.shift[b] - p.ntaps[b] + 1) - lead;     // >= 0: the short filter starts later and ends earlier
    fb[s].cap = p.edge_cap[b];
    fb[s].edges = p.edges + (size_t)u * p.edge_stride + (size_t)p.edge_off[b];
  }
  // seg[i] = s(n0 + lead + i), i < T + nt9 of the long band (beyond a filter's span its taps are zero; the signal
  // buffer is zero padded, so whatever lies there is finite)
  const int nt9_long = ((p.ntaps[b_long] + R - 1) / R) * R;
  const int seg_count = (T + nt9_long + 2) & ~1;
  int tot[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};   // events so far per band and train
#ifndef WB_EMU
  const int tid = threadIdx.x;
  for (int s = 0; s < nslot; ++s) {
    const int nt9 = ((fb[s].ntaps + R - 1) / R) * R;
    for (int j = tid; j < nt9 + R; j += blockDim.x)
      hrev[s][j] = j < fb[s].ntaps ? __ldg(&p.taps_rev[p.tap_off[fb[s].band] + j]) : 0.0;
  }
  if (tid == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid < G) {
    // ---------------------------------------------------------------- filter warps
    if (tid == 0 && n_tiles > 0) {
      const size_t a = abs0 + (size_t)lead;
      mbar_expect_tx(&bars[0], (unsigned)seg_count * 8u);
      tma_load_1d(segbuf[0], p.sig + (a & ~(size_t)1), (unsigned)seg_count * 8u, &bars[0]);
    }
    int item = 0;                                 // work item = (tile, band slot); its output half is item & 1
    for (int t = 0; t < n_tiles; ++t) {
      const size_t a0 = abs0 + (size_t)(t * T + lead);
      // every filter thread has left tile t-1 (bar 5 at its end), whose FIRs were the last readers of the other segment
      if (tid == 0 && t + 1 < n_tiles) {
        const size_t a1 = a0 + (size_t)T;
        mbar_expect_tx(&bars[(t + 1) & 1], (unsigned)seg_count * 8u);
        tma_load_1d(segbuf[(t + 1) & 1], p.sig + (a1 & ~(size_t)1), (unsigned)seg_count * 8u, &bars[(t + 1) & 1]);
      }
      mbar_wait(&bars[t & 1], (unsigned)((t >> 1) & 1));
      for (int s = 0; s < nslot; ++s, ++item) {
        if (item >= 2) bar_sync_named(3 + (item & 1), 2 * G);    // the event warps are done with this half (item - 2)
        fe_fir_group(segbuf[t & 1] + (a0 & 1) + fb[s].seg_off, hrev[s], fb[s].ntaps, tid, stbuf[item & 1]);
        __threadfence_block();
        bar_arrive_named(1 + (item & 1), 2 * G);                 // the item is ready
      }
      bar_sync_named(5, G);
    }
  } else {
    // ---------------------------------------------------------------- event warps
    const int ct = tid - G, lane = ct & 31, w = ct >> 5;
    // carry (the last two outputs of the band's previous tile): only group 0 reads it, and group 0 is this role's thread 0
    double c0[2] = {0.0, 0.0}, c1[2] = {0.0, 0.0};
    int item = 0;
    for (int t = 0; t < n_tiles; ++t) {
      const int n0 = t * T;
      const bool edge = n0 < 2 || n0 + T + 1 > ylen - 2;   // the tile reaches before sample 0 or past the last pair
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        if (s >= nslot) break;
        bar_sync_named(1 + (item & 1), 2 * G);
        const double *st = stbuf[item & 1];
        double v[WB_FE_R + 2];
        fe_load_group(st, c0[s], c1[s], ct, v);
        const int i0 = n0 - 2 + R * ct;
        unsigned long long c;
        const unsigned long long mask = fe_mask_group(v, i0, ylen, edge, &c);
        unsigned long long inc = c;
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned long long up = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= o) inc += up;
        }
        unsigned long long *wt = wtot + 4 * (item & 1);
        if (lane == 31) wt[w] = inc;
        bar_sync_named(6, G);
        unsigned long long basew = 0ull, all = 0ull;
#pragma unroll
        for (int k = 0; k < 4; ++k) { const unsigned long long x = wt[k]; if (k < w) basew += x; all += x; }
        fe_emit_group(v, mask, i0, basew + inc - c, tot[s], fb[s].edges, fb[s].cap);
        tot[s][0] += (int)(all & 0xffffull); tot[s][1] += (int)((all >> 16) & 0xffffull);
        tot[s][2] += (int)((all >> 32) & 0xffffull); tot[s][3] += (int)((all >> 48) & 0xffffull);
        if (ct == 0) { c0[s] = st[T - 2]; c1[s] = st[T - 1]; }
        __threadfence_block();
        bar_arrive_named(3 + (item & 1), 2 * G);                 // this half may be overwritten (item + 2)
        ++item;
      }
    }
    if (ct == 0) {
      for (int s = 0; s < nslot; ++s) {
        int *ec = p.ev_count + ((size_t)u * p.n_bands + fb[s].band) * 4;
        bool over = false;
        for (int q = 0; q < 4; ++q) { ec[q] = tot[s][q]; over = over || tot[s][q] > fb[s].cap; }
        if (over) {
          ec[0] = -1;
          p.redo_list[atomicAdd(p.redo_count, 1)] = u * p.n_bands + fb[s].band;
        }
      }
    }
  }
#else
  // one emulated thread: both roles, tile after tile, band after band
  for (int s = 0; s < nslot; ++s) {
    const int nt9 = ((fb[s].ntaps + R - 1) / R) * R;
    for (int j = 0; j < nt9 + R; ++j) hrev[s][j] = j < fb[s].ntaps ? p.taps_rev[p.tap_off[fb[s].band] + j] : 0.0;
  }
  double c0[2] = {0.0, 0.0}, c1[2] = {0.0, 0.0};
  for (int t = 0; t < n_tiles; ++t) {
    const int n0 = t * T;
    const size_t a0 = abs0 + (size_t)(n0 + lead);
    for (int i = 0; i < seg_count; ++i) segbuf[0][i] = p.sig[a0 + i];
    for (int s = 0; s < nslot; ++s) {
      double *st = stbuf[s];
      for (int g = 0; g < G; ++g) fe_fir_group(segbuf[0] + fb[s].seg_off, hrev[s], fb[s].ntaps, g, st);
      unsigned long long run = 0ull;
      for (int g = 0; g < G; ++g) {
        double v[WB_FE_R + 2];
        fe_load_group(st, c0[s], c1[s], g, v);
        const int i0 = n0 - 2 + R * g;
        unsigned long long c;
        const unsigned long long mask = fe_mask_group(v, i0, ylen, true, &c);
        fe_emit_group(v, mask, i0, run, tot[s], fb[s].edges, fb[s].cap);
        run += c;
      }
      tot[s][0] += (int)(run & 0xffffull); tot[s][1] += (int)((run >> 16) & 0xffffull);
      tot[s][2] += (int)((run >> 32) & 0xffffull); tot[s][3] += (int)((run >> 48) & 0xffffull);
      c0[s] = st[T - 2]; c1[s] = st[T - 1];
    }
  }
  for (int s = 0; s < nslot; ++s) {
    int *ec = p.ev_count + ((size_t)u * p.n_bands + fb[s].band) * 4;
    bool over = false;
    for (int q = 0; q < 4; ++q) { ec[q] = tot[s][q]; over = over || tot[s][q] > fb[s].cap; }
    if (over) {
      ec[0] = -1;
      p.redo_list[(*p.redo_count)++] = u * p.n_bands + fb[s].band;
    }
  }
#endif
}

// ---- edge lists -> candidates
// One CTA per (utterance, band); rounds of WB_IP_F frames, one frame per thread.  Per round and train a window of
// intervals starting two before the cursor (the intervals already behind the round) is loaded into shared memory --
// location x_j, value y_j and m_j = the first frame at or after x_j; its length follows the band (a 64 Hz band has
// ~16 intervals per 256 ms, an 880 Hz band ~225).  interp1's segment index for frame i is cursor + #{j : m_j <= i}:
// a binary search over the window's m.  A window that ends inside the round (far more crossings than the band
// frequency suggests) leaves its last frames to the next iteration of the same round.
#define WB_IP_F 256     // frames per round
#define WB_IP_W 256     // intervals per train and window (capacity)
struct IpTrain {        // one train of one band: complete edge list in global memory
  const double *e; int n_int; double afs;
};
WB_DEV double ip_loc(const IpTrain &T, int j) { return (T.e[j] + T.e[j + 1]) / 2.0 / T.afs; }     // dio.cpp:357-393
WB_DEV double ip_val(const IpTrain &T, int j) { return T.afs / (T.e[j + 1] - T.e[j]); }

// first_frame_at_or_after() with the two exact verifications (a multiplication and a division each) only when
// x * 1000 / frame_period lies within 1e-6 of an integer: otherwise t_g >= x > t_{g-1} hold with a margin ten
// orders of magnitude above the rounding of t_i = i * frame_period / 1000.0, and the quotient itself may come from
// a reciprocal.  Same result as the exact function in every case.
WB_DEV int first_frame_fast(double x, double frame_period, double frames_per_second) {
  const double r = x * frames_per_second;
  const double c = ceil(r);
  const double gap = c - r;
  if (gap > 1e-6 && gap < 1.0 - 1e-6 && r > 1.0 && r < 1e7) return (int)c;   // margin 1e-6 frames >> 3e-16 r
  return first_frame_at_or_after(x, frame_period);
}

WB_KERNEL(256, 4) band_interp_kernel(SweepParams p) {
  WB_SHARED double xw[4][WB_IP_W + 4], yw[4][WB_IP_W + 4];
  WB_SHARED unsigned long long marks[WB_IP_F + 40];   // per frame: intervals whose first frame it is, 4 x 16 bit; + scan scratch
  WB_SHARED unsigned long long orig[WB_IP_F];
  WB_SHARED int more_flag[2];   // "the last interval of a window still starts inside the round", per iteration parity
  const int tid = WB_TID, nth = WB_NTH;
  const int b = blockIdx.x, u = blockIdx.y;
  const int *ec = p.ev_count + ((size_t)u * p.n_bands + b) * 4;
  if (ec[0] < 0) return;   // lists overflowed: the streaming kernel redoes this band
  const int nf = p.n_frames[u];
  double *cand = p.cand + ((size_t)u * p.n_bands + b) * p.frame_stride;
  double *score = p.score ? p.score + ((size_t)u * p.n_bands + b) * p.frame_stride : nullptr;
  const double bf = p.boundary[b];
  const int cap = p.edge_cap[b];
  const double *edges = p.edges + (size_t)u * p.edge_stride + (size_t)p.edge_off[b];
  IpTrain tr[4];
  bool ok = true;
  for (int q = 0; q < 4; ++q) {
    tr[q].e = edges + (size_t)q * cap; tr[q].afs = p.afs;
    tr[q].n_int = ec[q] < 2 ? 0 : ec[q] - 1;        // ZeroCrossingEngine returns count-1 (0 if count<2)
    if (tr[q].n_int - 2 <= 0) ok = false;           // CheckEvent(n - 2), dio.cpp:475-484
  }
  if (!ok) {
    for (int i = tid; i < nf; i += nth) {
      cand[i] = 0.0;
      if (score) score[i] = 100000.0 / (0.0 + kTiny);
    }
    return;
  }
  // window length of this band: intervals expected per round (band frequency x round duration) + 65 %, at least 24
  int w_band = (int)(bf * 1.1 * (WB_IP_F * p.frame_period / 1000.0) * 1.65) + 24;
  if (w_band > WB_IP_W) w_band = WB_IP_W;
  const double fps = 1000.0 / p.frame_period;
  int cursor[4] = {0, 0, 0, 0};   // intervals whose first frame lies before the current round (identical in every thread)
  for (int c0 = 0; c0 < nf; c0 += WB_IP_F) {
    const int c1 = imin(nf, c0 + WB_IP_F);
    for (int i = tid; i < WB_IP_F; i += nth) marks[i] = 0ull;
    for (int i = tid; i < 2; i += nth) more_flag[i] = 0;
    int at[4] = {cursor[0], cursor[1], cursor[2], cursor[3]};   // first interval not yet examined in this round
    int wbase[4] = {0, 0, 0, 0}, wlen[4] = {0, 0, 0, 0};
    WB_SYNC();
    bool more = true;
    // One pass over the (train, interval) pairs of all four windows: the four trains' loads and divisions run side by
    // side instead of one latency chain after the other (otherwise the kernel waits at the barrier
    // behind the 20-60 loading threads of a low band).  The thread that loads a window's last interval tells
    // the CTA through more_flag[] whether that interval still starts inside the round; the flag of the next iteration
    // is cleared while this one's is read.
    for (int itn = 0; more; ++itn) {
      for (int q = 0; q < 4; ++q) {
        wbase[q] = imax(0, at[q] - 2);
        wlen[q] = imin(tr[q].n_int - wbase[q], at[q] - wbase[q] + w_band);
      }
      const int off1 = wlen[0], off2 = off1 + wlen[1], off3 = off2 + wlen[2], total = off3 + wlen[3];
      for (int j = tid; j < total; j += nth) {
        const int q = (j >= off1 ? 1 : 0) + (j >= off2 ? 1 : 0) + (j >= off3 ? 1 : 0);
        const int k = j - (q == 0 ? 0 : q == 1 ? off1 : q == 2 ? off2 : off3);
        const int wb = q == 0 ? wbase[0] : q == 1 ? wbase[1] : q == 2 ? wbase[2] : wbase[3];
        const int aq = q == 0 ? at[0] : q == 1 ? at[1] : q == 2 ? at[2] : at[3];
        const int wl = q == 0 ? wlen[0] : q == 1 ? wlen[1] : q == 2 ? wlen[2] : wlen[3];
        const int ni = q == 0 ? tr[0].n_int : q == 1 ? tr[1].n_int : q == 2 ? tr[2].n_int : tr[3].n_int;
        IpTrain T;
        T.e = edges + (size_t)q * cap; T.n_int = ni; T.afs = p.afs;
        const double x = ip_loc(T, wb + k);
        xw[q][k] = x; yw[q][k] = ip_val(T, wb + k);
        if (k >= aq - wb) {   // interval (wbase + k) is counted by every frame from its first frame on
          const int m = first_frame_fast(x, p.frame_period, fps);
          if (m < c1) {
            smem_add_u64(&marks[imax(m, c0) - c0], 1ull << (16 * q));
            if (k == wl - 1 && wb + wl < ni) more_flag[itn & 1] = 1;   // may be followed by more of them
          }
        }
      }
      WB_SYNC();
      more = more_flag[itn & 1] != 0;
      if (tid == 0) more_flag[(itn & 1) ^ 1] = 0;
      for (int q = 0; q < 4; ++q) at[q] = wbase[q] + wlen[q];
      if (more) WB_SYNC();   // the windows are rewritten
    }
    // inclusive counts per frame: exclusive scan + the frame's own marks
    for (int i = tid; i < WB_IP_F; i += nth) orig[i] = marks[i];
    WB_SYNC();
    const unsigned long long all = scan_packed(marks, WB_IP_F, 0ull, marks + WB_IP_F + 4);
    for (int i = c0 + tid; i < c1; i += nth) {
      const unsigned long long inc = marks[i - c0] + orig[i - c0];
      const double t = i * p.frame_period / 1000.0;
      double v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int cnt = cursor[q] + (int)((inc >> (16 * q)) & 0xffffull);
        const int k = imin(tr[q].n_int - 1, imax(1, cnt));   // interp1's segment (matlabfunctions.cpp:157-176)
        double x0, x1, y0, y1;
        const int w0 = k - 1 - wbase[q];
        if (w0 >= 0 && w0 + 1 < wlen[q]) {
          x0 = xw[q][w0]; x1 = xw[q][w0 + 1]; y0 = yw[q][w0]; y1 = yw[q][w0 + 1];
        } else {
          x0 = ip_loc(tr[q], k - 1); x1 = ip_loc(tr[q], k);
          y0 = ip_val(tr[q], k - 1); y1 = ip_val(tr[q], k);
        }
        const double s = (t - x0) / (x1 - x0);
        v[q] = y0 + s * (y1 - y0);
      }
      sweep_store_candidate(p, v[0], v[1], v[2], v[3], i, bf, cand, score);
    }
    cursor[0] += (int)(all & 0xffffull); cursor[1] += (int)((all >> 16) & 0xffffull);
    cursor[2] += (int)((all >> 32) & 0xffffull); cursor[3] += (int)((all >> 48) & 0xffffull);
    WB_SYNC();
  }
}

// extended input of decimate(): 9 mirrored samples on both sides of the edge-padded signal
WB_DEV double dec_ext(const double *__restrict__ x, int n, int lag, int nx, int i) {
#define WB_XIN(k) x[imin(n - 1, imax(0, (k) - lag))]
  if (i < 9) return 2 * WB_XIN(0) - WB_XIN(9 - i);
  if (i < 9 + nx) return WB_XIN(i - 9);
  return 2 * WB_XIN(nx - 1) - WB_XIN(nx - 2 - (i - (9 + nx)));
#undef WB_XIN
}

// pass 0: tmp[i] = forward IIR of ext;  pass 1: backward IIR over tmp, decimated into y
template <int kPass>
WB_KERNEL_PLAIN decimate_pass_kernel(DecimateParams p) {
  const int u = blockIdx.y;
  const int n = p.x_len[u];
  const int nx = n + 2 * p.lag, nt = nx + 18;
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long begin = g * WB_DEC_BLOCK;
  if (begin >= nt) return;
  const int end = (int)(begin + WB_DEC_BLOCK < nt ? begin + WB_DEC_BLOCK : nt);
  const int start = (int)(begin - WB_DEC_WARM > 0 ? begin - WB_DEC_WARM : 0);
  const double *x = p.x + (size_t)u * p.x_stride;
  double *tmp = p.tmp + (size_t)u * p.tmp_stride;
  double a[3], b[2];
  decimate_coefficients(p.ratio, a, b);
  double w0 = 0.0, w1 = 0.0, w2 = 0.0;
  if (kPass == 0) {
    for (int i = start; i < end; ++i) {
      const double wt = dec_ext(x, n, p.lag, nx, i) + a[0] * w0 + a[1] * w1 + a[2] * w2;
      if (i >= begin) tmp[i] = b[0] * wt + b[1] * w0 + b[1] * w1 + b[0] * w2;
      w2 = w1; w1 = w0; w0 = wt;
    }
  } else {
    // second filter runs over the reversed forward output; its result, reversed again, is tmp1 of
    // decimate(): final[j] with j = nt - 1 - i.  y[k] = final[nbeg + k r + 8]  (matlabfunctions.cpp:196-200)
    const int nout = (nx - 1) / p.ratio + 1;
    const int nbeg = p.ratio - p.ratio * nout + nx;
    const int n_out = p.n_out_mode == 0 ? 1 + n / p.ratio : static_cast<int>(ceil(static_cast<double>(n) / p.ratio));
    double *y = p.y + (size_t)u * p.y_stride + p.y_origin;
    for (int i = start; i < end; ++i) {
      const double wt = tmp[nt - 1 - i] + a[0] * w0 + a[1] * w1 + a[2] * w2;
      if (i >= begin) {
        const int j = nt - 1 - i - 8;          // = nbeg + k r  for a kept sample
        const int d = j - nbeg;
        if (d >= 0 && j < nx + 9 && d % p.ratio == 0) {
          const int k = d / p.ratio - p.first;
          if (k >= 0 && k < n_out) y[k] = b[0] * wt + b[1] * w0 + b[1] * w1 + b[0] * w2;
        }
      }
      w2 = w1; w1 = w0; w0 = wt;
    }
  }
}

void launch_decimate(Ctx *ctx, const DecimateParams &p, int max_x_len, unsigned n_utts) {
  const long long nt = (long long)max_x_len + 2 * p.lag + 18;
  const long long threads = (nt + WB_DEC_BLOCK - 1) / WB_DEC_BLOCK;
  const unsigned blocks = (unsigned)((threads + 63) / 64);
  WB_LAUNCH_FLAT(decimate_pass_kernel<0>, dim3(blocks, n_utts), 64, 0, ctx->stream, p);
  WB_LAUNCH_FLAT(decimate_pass_kernel<1>, dim3(blocks, n_utts), 64, 0, ctx->stream, p);
}

void launch_fir_plain(Ctx *ctx, const FirParams &p, unsigned tiles, unsigned n_utts) {
  const size_t smem = fir_plain_smem_bytes(p.ntaps);
#ifndef WB_EMU
  cudaFuncSetAttribute(fir_plain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
#endif
  WB_LAUNCH_COOP(fir_plain_kernel, dim3(tiles, n_utts), 256, smem, ctx->stream, p);
}

void launch_nyquist_bins(Ctx *ctx, const NyquistParams &p, unsigned n_utts) {
  WB_LAUNCH_COOP(nyquist_bins_kernel, dim3(n_utts), 256, 0, ctx->stream, p);
}

void launch_band_sweep(Ctx *ctx, const SweepParams &p_in, unsigned n_utts) {
  SweepParams p = p_in;
  p.debug_skip = 0;
  if (const char *e = getenv("WB_SWEEP_DEBUG")) p.debug_skip = atoi(e);
  const size_t smem = sweep_smem_bytes(p.max_taps);
  if (p.ripple) {
#ifndef WB_EMU
    cudaFuncSetAttribute(band_sweep_ripple_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
#endif
    WB_LAUNCH_COOP(band_sweep_ripple_kernel, dim3((unsigned)p.n_bands, n_utts), WB_SWEEP_THREADS, smem, ctx->stream, p);
  } else {
#ifndef WB_EMU
    cudaFuncSetAttribute(band_sweep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
#endif
    WB_LAUNCH_COOP(band_sweep_kernel, dim3((unsigned)p.n_bands, n_utts), WB_SWEEP_THREADS, smem, ctx->stream, p);
  }
}

void launch_band_sweep_split(Ctx *ctx, const SweepParams &p_in, unsigned n_utts) {
  SweepParams p = p_in;
  p.debug_skip = 0;
  const size_t smem_fe = fe_smem_bytes(p.max_taps), smem_sw = sweep_smem_bytes(p.max_taps);
#ifndef WB_EMU
  cudaFuncSetAttribute(band_fir_events_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_fe);
  cudaFuncSetAttribute(band_sweep_list_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sw);
#endif
  WB_LAUNCH_COOP(band_fir_events_kernel, dim3((unsigned)((p.n_bands + 1) / 2), n_utts), WB_SWEEP_THREADS, smem_fe, ctx->stream, p);
  WB_LAUNCH_COOP(band_interp_kernel, dim3((unsigned)p.n_bands, n_utts), 256, 0, ctx->stream, p);
  // bands whose edge lists overflowed (usually none): the streaming kernel with its history rings, over the list
  WB_LAUNCH_COOP(band_sweep_list_kernel, dim3((unsigned)(3 * ctx->sm_count)), WB_SWEEP_THREADS, smem_sw, ctx->stream, p);
}

}  // namespace wb
