// deskew.cu -- sweep deskew (lmot_set_deskew / lmot_seq_set_deskew, include/lmot.h): every point of a frame moved to the frame's stamp
// from its own capture time and the stream's ego motion, before ground removal.  An opt-in pre-stage the reference does not have.
//
// The host builds one pose table per frame (deskew_table, in double, rounded to float once per entry) and stages it to the device on
// the slot's or bank's stream; deskew_points_kernel then streams the frame's points through it into the slot's float4 point buffer,
// which the detection stages read as they read an undeskewed frame.  One launch covers every deskewed frame of a submission: frame i
// owns the CTAs [cta0, cta0 + ctas), each of which loads the frame's 12 KB table into shared memory once.
#include <cmath>
#include "lmot_internal.cuh"

namespace lmot {

namespace {

constexpr int kDeskewThreads = 256;
constexpr int kDeskewPtsPerCta = 4 * kDeskewThreads;   // 4 points per thread: ~120 CTAs for a 120 k point frame

struct DeskewFrame {
  const float* in;          // n records of `stride` floats (x, y, z at 0..2, the time at time_field)
  float4* out;              // n points (x', y', z', 1)
  const float* table;       // [LMOT_DESKEW_SLICES][12] row-major 3x4 poses
  int n, stride, time_field, cta0;
  double time_scale, time_offset, t_min, h;
};
struct DeskewParams { DeskewFrame f[kMaxBatch]; int n_frames; };

__global__ void __launch_bounds__(kDeskewThreads)
deskew_points_kernel(const __grid_constant__ DeskewParams P) {
  __shared__ float s_tab[LMOT_DESKEW_SLICES * 12];
  int fi = 0;
  while (fi + 1 < P.n_frames && (int)blockIdx.x >= P.f[fi + 1].cta0) ++fi;
  const DeskewFrame& F = P.f[fi];
  {
    const float4* src = reinterpret_cast<const float4*>(F.table);
    float4* dst = reinterpret_cast<float4*>(s_tab);
    for (int i = threadIdx.x; i < LMOT_DESKEW_SLICES * 3; i += kDeskewThreads) dst[i] = src[i];
  }
  __syncthreads();
  const int ctas = (fi + 1 < P.n_frames ? P.f[fi + 1].cta0 : (int)gridDim.x) - F.cta0;
  const bool quad = F.stride == 4 && F.time_field == 3;
  for (int i = ((int)blockIdx.x - F.cta0) * kDeskewThreads + threadIdx.x; i < F.n; i += ctas * kDeskewThreads) {
    float x, y, z, t;
    if (quad) {
      const float4 q = reinterpret_cast<const float4*>(F.in)[i];
      x = q.x; y = q.y; z = q.z; t = q.w;
    } else {
      const float* p = F.in + (size_t)i * F.stride;
      x = p[0]; y = p[1]; z = p[2]; t = p[F.time_field];
    }
    // (the library is compiled with -fmad=false: neither line below is contracted)
    const double tau = (double)t * F.time_scale + F.time_offset;
    float4 o = make_float4(x, y, z, 1.f);
    if (isfinite(tau)) {
      const double q = floor((tau - F.t_min) / F.h);
      const int s = q < 0.0 ? 0 : (q > (double)(LMOT_DESKEW_SLICES - 1) ? LMOT_DESKEW_SLICES - 1 : (int)q);
      const float* d = s_tab + 12 * s;
      o.x = ((d[0] * x + d[1] * y) + d[2] * z) + d[3];
      o.y = ((d[4] * x + d[5] * y) + d[6] * z) + d[7];
      o.z = ((d[8] * x + d[9] * y) + d[10] * z) + d[11];
    }
    F.out[i] = o;
  }
}

}  // namespace

// T(tau) of the vehicle (moving along +x at v, turning about +z at omega) in its frame at the stamp, then M^-1 T M, in double
int deskew_table(const lmot_deskew& d, double v, double omega, const lmot_sensor* mount, float* out) {
  double M[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  if (mount) for (int i = 0; i < 12; ++i) M[i] = (double)mount->pose[i];
  double Mi[12];                     // [R^T | -R^T t]
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) Mi[4 * i + j] = M[4 * j + i];
    Mi[4 * i + 3] = -((M[i] * M[3] + M[4 + i] * M[7]) + M[8 + i] * M[11]);
  }
  const double h = (d.t_max - d.t_min) / (double)LMOT_DESKEW_SLICES;
  for (int s = 0; s < LMOT_DESKEW_SLICES; ++s) {
    const double tau = d.t_min + (s + 0.5) * h;
    const double th = omega * tau;
    const double c = std::cos(th), sn = std::sin(th);        // (once per slice: the host's table building is per-frame submission work)
    double tx, ty;
    if (std::fabs(omega) < 1e-9) { tx = v * tau; ty = 0.0; }
    else { tx = v * sn / omega; ty = v * (1.0 - c) / omega; }
    const double T[12] = {c, -sn, 0, tx, sn, c, 0, ty, 0, 0, 1, 0};
    double A[12], D[12];
    for (int pass = 0; pass < 2; ++pass) {       // A = T M, then D = M^-1 A; rows ((a0 b0j + a1 b1j) + a2 b2j) (+ a3 for column 3)
      const double* L = pass ? Mi : T;
      const double* R = pass ? A : M;
      double* X = pass ? D : A;
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 4; ++j) {
          double acc = (L[4 * i] * R[j] + L[4 * i + 1] * R[4 + j]) + L[4 * i + 2] * R[8 + j];
          if (j == 3) acc = acc + L[4 * i + 3];
          X[4 * i + j] = acc;
        }
    }
    for (int e = 0; e < 12; ++e) out[12 * s + e] = (float)D[e];
  }
  return LMOT_OK;
}

int deskew_launch(Ctx* c, cudaStream_t st, const DeskewJob* jobs, int n_jobs) {
  DeskewParams P{};
  int ctas = 0;
  P.n_frames = 0;
  for (int j = 0; j < n_jobs; ++j) {
    const DeskewJob& q = jobs[j];
    if (q.n <= 0) continue;
    DeskewFrame& f = P.f[P.n_frames++];
    f.in = q.in; f.out = q.out; f.table = q.table; f.n = q.n; f.stride = q.stride; f.time_field = q.d.time_field; f.cta0 = ctas;
    f.time_scale = q.d.time_scale; f.time_offset = q.d.time_offset; f.t_min = q.d.t_min;
    f.h = (q.d.t_max - q.d.t_min) / (double)LMOT_DESKEW_SLICES;
    ctas += (q.n + kDeskewPtsPerCta - 1) / kDeskewPtsPerCta;
  }
  if (ctas == 0) return LMOT_OK;
  deskew_points_kernel<<<ctas, kDeskewThreads, 0, st>>>(P);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

}  // namespace lmot
