// ground_lines.cuh -- ground lines (lmot_set_ground_lines, include/lmot.h): one channel's chain of ground lines over range, and the
// ground height of each of its 120 cells.  One function for the host (lmot_ground_lines_grid) and the device (ground.cu, phase 2 of
// ground_fused_lines_kernel): plain double arithmetic, left to right.  The library is built with -fmad=false and the host compiler
// targets baseline x86-64 (no FMA), so both evaluate every operation as written and agree bit for bit.
#pragma once
#include <cmath>
#include "lmot_internal.cuh"

namespace lmot {

struct GroundLinesSums {
  double n = 0, sr = 0, sz = 0, srr = 0, srz = 0, szz = 0;
  __host__ __device__ void add(double r, double z) { n = n + 1; sr = sr + r; sz = sz + z; srr = srr + r * r; srz = srz + r * z; szz = szz + z * z; }
  // fit(S): slope m, intercept c and the residual sum of squares
  __host__ __device__ void fit(double& m, double& c, double& sse) const {
    const double den = n * srr - sr * sr;
    m = (n * srz - sr * sz) / den;
    c = (sz - m * sr) / n;
    sse = szz - 2 * m * srz - 2 * c * sz + m * m * srr + 2 * m * c * sr + n * c * c;
  }
};

// one channel.  minz(b): the cell's min z (1000: empty); put(b, gz): the cell's ground height, called once per bin in bin order
template <class Src, class Dst>
__host__ __device__ inline void ground_lines_channel(const Src& minz, const Dst& put, double r_min, double r_max, double sensor_height,
                                                     double max_slope, double max_rmse, double max_step) {
  const double span = r_max - r_min;
  GroundLinesSums S;
  int first = 0;                       // S's first bin
  double r0 = 0, z0 = 0;               // S's point while n == 1
  bool have = false;                   // the channel has a line: (lm, lc) is its last
  int fill = 0;                        // first bin whose height is not written yet
  double lm = 0, lc = 0;
  for (int b = 0; b <= kNumBin; ++b) {
    const bool last = b == kNumBin;    // (one pass past bin 119 closes S)
    const float zf = last ? 1000.f : minz(b);
    if (!last && !(zf < 1000.f)) continue;
    const double r = last ? 0.0 : r_min + (b + 0.5) * span / 120;
    const double z = (double)zf;
    if (!last && S.n >= 2) {           // extend
      GroundLinesSums T = S;
      T.add(r, z);
      double m, c, sse;
      T.fit(m, c, sse);
      if (fabs(m) <= max_slope && sse <= T.n * max_rmse * max_rmse) { S = T; continue; }
    }
    if (S.n >= 2) {                    // close S: its line, and the cells the line before it now owns
      double m, c, sse;
      S.fit(m, c, sse);
      if (have) {
        for (int q = fill; q < first; ++q) put(q, (float)(lm * (r_min + (q + 0.5) * span / 120) + lc));
        fill = first;
      }
      have = true; lm = m; lc = c;
    }
    if (S.n >= 2) S = GroundLinesSums();
    if (last) break;
    for (;;) {                         // seed test
      bool pass = have ? fabs(z - (lm * r + lc)) <= max_step : fabs(z + sensor_height) <= max_slope * r + max_step;
      if (pass && S.n == 1) pass = fabs(z - z0) <= max_slope * (r - r0);
      if (pass) {
        if (S.n == 0) { first = b; r0 = r; z0 = z; }
        S.add(r, z);
        break;
      }
      if (S.n == 1) { S = GroundLinesSums(); continue; }   // drop the lone seed, test the point again
      break;                                               // drop the point
    }
  }
  if (have) for (int q = fill; q < kNumBin; ++q) put(q, (float)(lm * (r_min + (q + 0.5) * span / 120) + lc));
  else for (int q = 0; q < kNumBin; ++q) put(q, (float)(-sensor_height));
}

}  // namespace lmot
