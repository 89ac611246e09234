// polar_cell.cuh -- the exact point -> polar cell map of groundRemove, for the ground kernel (ground.cu) and for box heights from the
// local ground (boxfit_device.cuh, ground lines).  Internal linkage: every translation unit compiles its own copies.
#pragma once
#include "lmot_internal.cuh"
#include "exact_math.cuh"

namespace lmot {

namespace {

// ground_removal.cpp:46-64 (range filter) + :67-76 (getCellIndexFromPoints) + :89 (index guard), evaluated exactly as the
// reference does: IEEE sqrt and divisions, glibc's atan2f (fdlibm restatement, exact_math.cuh), the double add / divide.
// kClone: ground_fused_frame_kernel calls its own copy -- one shared non-inlined function would be compiled for the most general of its
// callers' arguments (a frame's entry of a parameter array) and change the code of the other kernels
template <int kClone = 0>
__device__ __noinline__ uint16_t polar_cell_exact(float x, float y, const GroundParams& p) {
  const float d = fsqrt(fadd(fmul(x, x), fmul(y, y)));
  if (d <= p.r_min || d >= p.r_max || d != d) return kNoCell;
  const float binP = fdiv(fsub(d, p.r_min), p.r_span);
  const float binF = floorf(fmul(binP, (float)kNumBin));
  if (!(binF >= 0.f && binF < (float)kNumBin)) return kNoCell;
  const float a = atan2f_fdlibm(y, x);
  const double chD = __ddiv_rn(__dadd_rn((double)a, 3.14159265358979323846), 6.28318530717958647692);
  const float chF = floorf(fmul((float)chD, (float)kNumChannel));
  if (!(chF >= 0.f && chF < (float)kNumChannel)) return kNoCell;
  return (uint16_t)((int)chF * kNumBin + (int)binF);
}

}  // namespace

}  // namespace lmot
