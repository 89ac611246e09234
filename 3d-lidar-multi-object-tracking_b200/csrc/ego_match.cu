// ego_match.cu -- scan-matched ego motion (lmot_ego_estimate): a stream's planar motion between consecutive sweeps, on sm_90a.
//
// The definition is in include/lmot.h.  One synchronous call steps S streams (the own stream, or the sequences of lmot_seq_ego_estimate)
// with one launch per kernel on the context's matcher stream (blockIdx.z or blockIdx.y = stream):
//   ego_clear_kernel    the occupancy bitmap, the sub-cell minima and the stream's result row
//   ego_band_kernel     step 1 per point: band, window, one bit of the occupancy bitmap, atomicMin of the point index per sub-cell
//   ego_field_kernel    step 2 per cell: L from the 5 x 5 bits around it (the distance only matters up to 2), and |O|
//   ego_sample_kernel   step 3, one CTA per stream: a block scan over the sub-cells in raster order, every k-th occupied one kept
//   ego_coarse_kernel   step 4's coarse level: one CTA per (angle, 256 shifts).  The rotated base cells of every sample sit in shared
//                       memory; each thread sums its shift's bytes of the reference field.  A warp covers 32 consecutive kx of one ky, so
//                       for each sample it reads one or two 32-byte sectors of one field row: the grid^2-byte field stays in L2 (590 KB at
//                       the defaults) and neighbouring samples (raster order) hit the same lines.
//   ego_fine_kernel     the fine level: one CTA per fine angle, one thread per translation, around the coarse winner read on the device
// Both levels reduce to one 64-bit key per stream, score << 32 | ~(hypothesis index), with atomicMax: scores are integers, so the winner
// (ties to the first index) does not depend on the order CTAs finish in.  The angle tables (cos / sin in double with the host libm, rounded
// to float) are computed on the host for every angle either level can reach, so no host round trip separates the levels.
#include <climits>
#include <cmath>
#include <cstring>
#include "lmot_internal.cuh"

namespace lmot {

namespace {

constexpr int kEgoThreads = 256;
constexpr int kSampleThreads = 1024;

struct EgoRes {                        // one stream's device results of a call
  int n_used, n_occ, pad0, pad1;
  unsigned long long coarse, fine;
};

struct EgoJob {
  const float* pts; int n; int stride;
  int posed; float pose[12];
  int grid, ns, max_points, min_points;
  float H, cell, sub, z_min, z_max, rmin2, rmax2;
  double cell_d, yaw_step;
  unsigned* occ; int* sub_min; float2* samp;
  unsigned char* L_cur; const unsigned char* L_prev;
  int match, YH, SH, R;
  long long j0, k0x, k0y;
  const float2* tab_coarse;            // [2 YH + 1]: angle j0 - YH + a
  const float2* tab_fine;              // [2 YH R + 2 R + 1]: angle index R (j0 - YH) - R + i
  EgoRes* res;
};

struct EgoLaunch { int S; EgoJob job[kMaxBatch]; };

__device__ __forceinline__ bool ego_point(const EgoJob& J, int i, float& x, float& y) {
  const float* p = J.pts + (size_t)i * J.stride;
  float px = p[0], py = p[1], pz = p[2];
  if (J.posed) {
    const float* m = J.pose;
    const float qx = ((m[0] * px + m[1] * py) + m[2] * pz) + m[3];
    const float qy = ((m[4] * px + m[5] * py) + m[6] * pz) + m[7];
    const float qz = ((m[8] * px + m[9] * py) + m[10] * pz) + m[11];
    px = qx; py = qy; pz = qz;
  }
  x = px; y = py;
  if (!(isfinite(px) && isfinite(py) && isfinite(pz))) return false;
  if (!(pz >= J.z_min && pz <= J.z_max)) return false;
  const float r2 = px * px + py * py;
  return r2 >= J.rmin2 && r2 <= J.rmax2;
}

__global__ void __launch_bounds__(kEgoThreads) ego_clear_kernel(EgoLaunch P) {
  const EgoJob& J = P.job[blockIdx.y];
  const int words = J.grid * J.grid / 32, subs = J.ns * J.ns;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < words || i < subs; i += gridDim.x * blockDim.x) {
    if (i < words) J.occ[i] = 0u;
    if (i < subs) J.sub_min[i] = INT_MAX;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    J.res->n_used = 0; J.res->n_occ = 0;
    J.res->coarse = 0ull; J.res->fine = 0ull;
  }
}

__global__ void __launch_bounds__(kEgoThreads) ego_band_kernel(EgoLaunch P) {
  const EgoJob& J = P.job[blockIdx.y];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < J.n; i += gridDim.x * blockDim.x) {
    float x, y;
    if (!ego_point(J, i, x, y)) continue;
    const int ix = (int)floorf((x + J.H) / J.cell), iy = (int)floorf((y + J.H) / J.cell);
    if (ix < 0 || ix >= J.grid || iy < 0 || iy >= J.grid) continue;
    const int c = iy * J.grid + ix;
    atomicOr(&J.occ[c >> 5], 1u << (c & 31));
    const int sx = min((int)floorf((x + J.H) / J.sub), J.ns - 1), sy = min((int)floorf((y + J.H) / J.sub), J.ns - 1);
    atomicMin(&J.sub_min[sy * J.ns + sx], i);
  }
}

__device__ __forceinline__ bool occ_at(const unsigned* occ, int g, int x, int y) {
  if (x < 0 || x >= g || y < 0 || y >= g) return false;
  const int c = y * g + x;
  return occ[c >> 5] >> (c & 31) & 1u;
}

__global__ void __launch_bounds__(kEgoThreads) ego_field_kernel(EgoLaunch P) {
  const EgoJob& J = P.job[blockIdx.y];
  const int g = J.grid, cells = g * g;
  for (int base = blockIdx.x * blockDim.x; base < cells; base += gridDim.x * blockDim.x) {
    const int c = base + threadIdx.x;
    bool occupied = false;
    if (c < cells) {
      const int x = c % g, y = c / g;
      int d = 3;                       // Chebyshev distance to O, capped at 3
      for (int dy = -2; dy <= 2; ++dy)
        for (int dx = -2; dx <= 2; ++dx)
          if (occ_at(J.occ, g, x + dx, y + dy)) d = min(d, max(abs(dx), abs(dy)));
      J.L_cur[c] = (unsigned char)(3 - d);
      occupied = d == 0;
    }
    const unsigned b = __ballot_sync(0xffffffffu, occupied);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(&J.res->n_occ, __popc(b));
  }
}

__global__ void __launch_bounds__(kSampleThreads) ego_sample_kernel(EgoLaunch P) {
  const EgoJob& J = P.job[blockIdx.x];
  __shared__ int warp_sum[kSampleThreads / 32];
  __shared__ int total_s;
  const int subs = J.ns * J.ns;
  const int per = (subs + kSampleThreads - 1) / kSampleThreads;
  const int lo = min(subs, threadIdx.x * per), hi = min(subs, lo + per);
  int cnt = 0;
  for (int i = lo; i < hi; ++i) cnt += J.sub_min[i] != INT_MAX;
  // exclusive block scan of cnt
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int inc = cnt;
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) warp_sum[w] = inc;
  __syncthreads();
  if (w == 0) {
    int v = warp_sum[lane];
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
    warp_sum[lane] = v;                // inclusive over warps
    if (lane == 31) total_s = v;
  }
  __syncthreads();
  int rank = inc - cnt + (w > 0 ? warp_sum[w - 1] : 0);
  const int total = total_s;
  const int k = total > J.max_points ? (total + J.max_points - 1) / J.max_points : 1;
  for (int i = lo; i < hi; ++i) {
    const int p = J.sub_min[i];
    if (p == INT_MAX) continue;
    if (rank % k == 0) {
      float x, y;
      ego_point(J, p, x, y);
      J.samp[rank / k] = make_float2(x, y);
    }
    ++rank;
  }
  if (threadIdx.x == 0) J.res->n_used = (total + k - 1) / k;
}

__device__ __forceinline__ unsigned long long warp_max64(unsigned long long v) {
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long t = __shfl_xor_sync(0xffffffffu, v, o);
    v = t > v ? t : v;
  }
  return v;
}

// gridDim = (angles, shift blocks, S); blockIdx.x = a: angle j0 - YH + a; thread h of block y: shift index (ky - k0y + SH) * W + (kx - k0x + SH)
__global__ void __launch_bounds__(kEgoThreads) ego_coarse_kernel(EgoLaunch P) {
  const EgoJob& J = P.job[blockIdx.z];
  const int n = J.res->n_used;
  const int W = 2 * J.SH + 1;
  if (!J.match || n < J.min_points || (int)blockIdx.x > 2 * J.YH || (int)blockIdx.y * kEgoThreads >= W * W) return;
  extern __shared__ int2 base[];
  const float2 cs = J.tab_coarse[blockIdx.x];
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float2 p = J.samp[i];
    const float xr = cs.x * p.x - cs.y * p.y, yr = cs.y * p.x + cs.x * p.y;
    base[i] = make_int2((int)floorf((xr + J.H) / J.cell) + (int)(J.k0x - J.SH), (int)floorf((yr + J.H) / J.cell) + (int)(J.k0y - J.SH));
  }
  __syncthreads();
  const int h = blockIdx.y * kEgoThreads + threadIdx.x;
  const int ix = h % W, iy = h / W;
  const int g = J.grid;
  unsigned score = 0;
  if (h < W * W) {
    const unsigned char* __restrict__ L = J.L_prev;
    for (int i = 0; i < n; ++i) {
      const int cx = base[i].x + ix, cy = base[i].y + iy;
      if ((unsigned)cx < (unsigned)g && (unsigned)cy < (unsigned)g) score += __ldg(L + cy * g + cx);
    }
  }
  const unsigned idx = ((unsigned)blockIdx.x * W + ix) * W + iy;
  unsigned long long key = h < W * W ? ((unsigned long long)score << 32) | (0xffffffffu - idx) : 0ull;
  key = warp_max64(key);
  if ((threadIdx.x & 31) == 0 && key) atomicMax(&J.res->coarse, key);
}

// gridDim = (2 R + 1, 1, S); blockIdx.x = u + R; thread t: (ax, ay) = (t / (2R+1) - R, t % (2R+1) - R)
__global__ void __launch_bounds__(1024) ego_fine_kernel(EgoLaunch P) {
  const EgoJob& J = P.job[blockIdx.z];
  const int n = J.res->n_used;
  const int R = J.R, F = 2 * R + 1;
  if (!J.match || R < 2 || n < J.min_points || (int)blockIdx.x >= F) return;
  extern __shared__ float2 rot[];
  const int W = 2 * J.SH + 1;
  const unsigned cidx = 0xffffffffu - (unsigned)(J.res->coarse & 0xffffffffull);
  const int a = (int)(cidx / (unsigned)(W * W)), ix = (int)(cidx / (unsigned)W % (unsigned)W), iy = (int)(cidx % (unsigned)W);
  const long long k1x = J.k0x - J.SH + ix, k1y = J.k0y - J.SH + iy;
  const int u = (int)blockIdx.x - R;
  const float2 cs = J.tab_fine[R * a + u + R];
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float2 p = J.samp[i];
    rot[i] = make_float2(cs.x * p.x - cs.y * p.y, cs.y * p.x + cs.x * p.y);
  }
  __syncthreads();
  const int t = threadIdx.x;
  unsigned long long key = 0ull;
  if (t < F * F) {
    const int ax = t / F - R, ay = t % F - R;
    const float tx = (float)((double)(R * k1x + ax) * J.cell_d / (double)R);
    const float ty = (float)((double)(R * k1y + ay) * J.cell_d / (double)R);
    const int g = J.grid;
    const unsigned char* __restrict__ L = J.L_prev;
    unsigned score = 0;
    for (int i = 0; i < n; ++i) {
      const int cx = (int)floorf(((rot[i].x + tx) + J.H) / J.cell), cy = (int)floorf(((rot[i].y + ty) + J.H) / J.cell);
      if ((unsigned)cx < (unsigned)g && (unsigned)cy < (unsigned)g) score += __ldg(L + cy * g + cx);
    }
    const unsigned idx = ((unsigned)blockIdx.x * F + (unsigned)(ax + R)) * F + (unsigned)(ay + R);
    key = ((unsigned long long)score << 32) | (0xffffffffu - idx);
  }
  key = warp_max64(key);
  if ((threadIdx.x & 31) == 0 && key) atomicMax(&J.res->fine, key);
}

int sub_side(const lmot_ego_match& m) { return (int)ceil((double)m.grid * m.cell_m / m.sub_m) + 1; }

int grow(Ctx* c, void** p, size_t* cap, size_t need) {
  if (*cap >= need) return LMOT_OK;
  cudaFree(*p);
  *p = nullptr; *cap = 0;
  LMOT_CUDA(c, cudaMalloc(p, need));
  *cap = need;
  return LMOT_OK;
}

// the stream's device buffers for its current setting
int ego_ensure(Ctx* c, EgoMatch& e) {
  const lmot_ego_match& m = e.cfg;
  const size_t field = (size_t)m.grid * m.grid, subs = (size_t)sub_side(m) * sub_side(m);
  if (e.cap_field < field) {
    cudaFree(e.d_field[0]); cudaFree(e.d_field[1]); cudaFree(e.d_occ);
    e.d_field[0] = e.d_field[1] = nullptr; e.d_occ = nullptr; e.cap_field = 0;
    e.has_ref = false;                 // (a larger grid always follows a setting, which already dropped the reference)
    LMOT_CUDA(c, cudaMalloc(&e.d_field[0], field));
    LMOT_CUDA(c, cudaMalloc(&e.d_field[1], field));
    LMOT_CUDA(c, cudaMalloc(&e.d_occ, field / 8));
    e.cap_field = field;
  }
  size_t cap = e.cap_sub * sizeof(int);
  int rc = grow(c, (void**)&e.d_sub, &cap, subs * sizeof(int));
  if (rc) return rc;
  e.cap_sub = cap / sizeof(int);
  cap = e.cap_samp * sizeof(float2);
  rc = grow(c, (void**)&e.d_samp, &cap, (size_t)m.max_points * sizeof(float2));
  if (rc) return rc;
  e.cap_samp = cap / sizeof(float2);
  return LMOT_OK;
}

long long llround_or_zero(double v) { return std::isfinite(v) && fabs(v) < (double)(1 << 20) ? llround(v) : 0; }

}  // namespace

bool ego_match_valid(const lmot_ego_match& m) {
  const double d[] = {m.cell_m, m.z_min, m.z_max, m.r_min, m.r_max, m.sub_m, m.yaw_step, m.min_score_frac};
  for (double v : d) if (!std::isfinite(v)) return false;
  if (m.grid < 32 || m.grid > 1024 || m.grid % 32 != 0) return false;
  if (!(m.cell_m >= 0.01 && m.cell_m <= 10.0) || !((double)m.grid * m.cell_m <= 400.0)) return false;
  if (!(m.z_min < m.z_max) || !(m.r_min >= 0.0 && m.r_min < m.r_max && m.r_max <= 1000.0)) return false;
  if (!(m.sub_m > 0.0) || sub_side(m) > 1024) return false;
  if (m.max_points < 1 || m.max_points > 8192 || !(m.yaw_step > 0.0 && m.yaw_step <= 0.1)) return false;
  if (m.yaw_half < 0 || m.yaw_half > 180 || m.shift_half < 0 || m.shift_half > 127 || m.refine < 1 || m.refine > 15) return false;
  if (m.min_points < 1 || !(m.min_score_frac >= 0.0 && m.min_score_frac <= 1.0)) return false;
  return m.sensor >= -1 && m.sensor < kMaxBatch;
}

void ego_free(EgoMatch& e) {
  cudaFree(e.d_field[0]); cudaFree(e.d_field[1]); cudaFree(e.d_occ); cudaFree(e.d_sub); cudaFree(e.d_samp);
  e = EgoMatch{};
}

void ego_ctx_free(Ctx* c) {
  if (c->ego_stream) cudaStreamDestroy(c->ego_stream);
  if (c->ev_ego_in) cudaEventDestroy(c->ev_ego_in);
  cudaFree(c->d_ego_stage); cudaFree(c->d_ego_tab); cudaFree(c->d_ego_res);
  if (c->h_ego_tab) cudaFreeHost(c->h_ego_tab);
  if (c->h_ego_res) cudaFreeHost(c->h_ego_res);
  c->ego_stream = nullptr; c->ev_ego_in = nullptr; c->d_ego_stage = nullptr; c->d_ego_tab = nullptr; c->d_ego_res = nullptr;
  c->h_ego_tab = nullptr; c->h_ego_res = nullptr; c->ego_stage_bytes = 0; c->ego_tab_cap = 0;
}

int ego_estimate_run(Ctx* c, EgoMatch* const* q, const float* const* pts, const int* n, int stride, const double* ts,
                     const lmot_sensor* const* poses, int S, bool host, lmot_ego_out* const* out) {
  if (S <= 0) return LMOT_OK;
  if (!c->ego_stream) {
    LMOT_CUDA(c, cudaStreamCreateWithFlags(&c->ego_stream, cudaStreamNonBlocking));
    LMOT_CUDA(c, cudaEventCreateWithFlags(&c->ev_ego_in, cudaEventDisableTiming));
    LMOT_CUDA(c, cudaHostAlloc(&c->h_ego_res, kMaxBatch * sizeof(EgoRes), cudaHostAllocDefault));
    LMOT_CUDA(c, cudaMalloc(&c->d_ego_res, kMaxBatch * sizeof(EgoRes)));
  }
  cudaStream_t st = c->ego_stream;
  for (int i = 0; i < S; ++i) {
    const int rc = ego_ensure(c, *q[i]);
    if (rc) return rc;
  }
  // host frames: one staging buffer, frames back to back
  size_t off[kMaxBatch] = {}, tot = 0;
  if (host) {
    for (int i = 0; i < S; ++i) { off[i] = tot; tot += (size_t)n[i] * stride; }
    size_t cap = c->ego_stage_bytes;
    const int rc = grow(c, (void**)&c->d_ego_stage, &cap, std::max<size_t>(tot, 1) * sizeof(float));
    if (rc) return rc;
    c->ego_stage_bytes = cap;
  }
  // the step-4 plan of each stream, and its angle tables
  EgoLaunch L;
  memset(&L, 0, sizeof(L));
  L.S = S;
  double dt[kMaxBatch], prior[kMaxBatch][3];
  bool dt_ok[kMaxBatch];
  size_t tab_off[kMaxBatch], tab_n = 0;
  for (int i = 0; i < S; ++i) {
    const EgoMatch& e = *q[i];
    const lmot_ego_match& m = e.cfg;
    dt[i] = (ts[i] - e.ts) / 1e6;
    dt_ok[i] = e.has_ref && std::isfinite(dt[i]) && dt[i] > 0;
    for (int k = 0; k < 3; ++k) prior[i][k] = 0.0;
    if (dt_ok[i] && e.delta_ok) {
      const double r = dt[i] / e.dt;
      for (int k = 0; k < 3; ++k) prior[i][k] = e.delta[k] * r;
    }
    tab_off[i] = tab_n;
    if (dt_ok[i]) tab_n += (size_t)(2 * m.yaw_half + 1) + (size_t)(2 * m.yaw_half * m.refine + 2 * m.refine + 1);
  }
  if (tab_n > c->ego_tab_cap) {
    if (c->h_ego_tab) cudaFreeHost(c->h_ego_tab);
    cudaFree(c->d_ego_tab);
    c->h_ego_tab = nullptr; c->d_ego_tab = nullptr; c->ego_tab_cap = 0;
    LMOT_CUDA(c, cudaHostAlloc(&c->h_ego_tab, tab_n * sizeof(float2), cudaHostAllocDefault));
    LMOT_CUDA(c, cudaMalloc(&c->d_ego_tab, tab_n * sizeof(float2)));
    c->ego_tab_cap = tab_n;
  }
  int max_n = 1, max_grid = 32, max_subs = 1, max_ang = 1, max_w2 = 1, max_f = 1, max_pts = 1;
  EgoRes* d_res = (EgoRes*)c->d_ego_res;
  for (int i = 0; i < S; ++i) {
    EgoMatch& e = *q[i];
    const lmot_ego_match& m = e.cfg;
    EgoJob& J = L.job[i];
    J.pts = host ? c->d_ego_stage + off[i] : pts[i];
    J.n = n[i]; J.stride = stride;
    J.posed = poses[i] != nullptr;
    if (poses[i]) memcpy(J.pose, poses[i]->pose, sizeof(J.pose));
    J.grid = m.grid; J.ns = sub_side(m); J.max_points = m.max_points; J.min_points = m.min_points;
    J.H = (float)(m.grid * (double)m.cell_m * 0.5);
    J.cell = (float)m.cell_m; J.sub = (float)m.sub_m; J.z_min = (float)m.z_min; J.z_max = (float)m.z_max;
    const float rmin = (float)m.r_min, rmax = (float)m.r_max;
    J.rmin2 = rmin * rmin; J.rmax2 = rmax * rmax;
    J.cell_d = m.cell_m; J.yaw_step = m.yaw_step;
    J.occ = e.d_occ; J.sub_min = e.d_sub; J.samp = e.d_samp;
    J.L_cur = e.d_field[e.ref ^ 1]; J.L_prev = e.d_field[e.ref];
    J.match = dt_ok[i] ? 1 : 0;
    J.YH = m.yaw_half; J.SH = m.shift_half; J.R = m.refine;
    J.res = d_res + i;
    if (J.match) {
      J.j0 = llround_or_zero(prior[i][2] / m.yaw_step);
      J.k0x = llround_or_zero(prior[i][0] / m.cell_m);
      J.k0y = llround_or_zero(prior[i][1] / m.cell_m);
      float2* h = c->h_ego_tab + tab_off[i];
      const int na = 2 * m.yaw_half + 1, R = m.refine;
      for (int a = 0; a < na; ++a) {
        const double th = (double)(J.j0 - m.yaw_half + a) * m.yaw_step;
        h[a] = make_float2((float)cos(th), (float)sin(th));
      }
      const long long f0 = (long long)R * (J.j0 - m.yaw_half) - R;
      const int nf = 2 * m.yaw_half * R + 2 * R + 1;
      for (int t = 0; t < nf; ++t) {
        const double th = (double)(f0 + t) * m.yaw_step / R;
        h[na + t] = make_float2((float)cos(th), (float)sin(th));
      }
      J.tab_coarse = c->d_ego_tab + tab_off[i];
      J.tab_fine = c->d_ego_tab + tab_off[i] + na;
      max_ang = std::max(max_ang, na);
      max_w2 = std::max(max_w2, (2 * m.shift_half + 1) * (2 * m.shift_half + 1));
      max_f = std::max(max_f, 2 * R + 1);
      max_pts = std::max(max_pts, m.max_points);
    }
    max_n = std::max(max_n, n[i]);
    max_grid = std::max(max_grid, m.grid);
    max_subs = std::max(max_subs, J.ns * J.ns);
  }
  // the caller's frames: staged (host) or behind the caller stream's work (device)
  if (host) {
    for (int i = 0; i < S; ++i)
      if (n[i] > 0) LMOT_CUDA(c, cudaMemcpyAsync(c->d_ego_stage + off[i], pts[i], (size_t)n[i] * stride * sizeof(float), cudaMemcpyHostToDevice, st));
  } else {
    LMOT_CUDA(c, cudaEventRecord(c->ev_ego_in, c->stream));
    LMOT_CUDA(c, cudaStreamWaitEvent(st, c->ev_ego_in, 0));
  }
  if (tab_n) LMOT_CUDA(c, cudaMemcpyAsync(c->d_ego_tab, c->h_ego_tab, tab_n * sizeof(float2), cudaMemcpyHostToDevice, st));
  const int clear_blocks = std::min(1024, std::max((max_grid * max_grid / 32 + kEgoThreads - 1) / kEgoThreads, (max_subs + kEgoThreads - 1) / kEgoThreads));
  ego_clear_kernel<<<dim3(clear_blocks, S), kEgoThreads, 0, st>>>(L);
  ego_band_kernel<<<dim3(std::min(4096, (max_n + kEgoThreads - 1) / kEgoThreads), S), kEgoThreads, 0, st>>>(L);
  ego_field_kernel<<<dim3(std::min(4096, (max_grid * max_grid + kEgoThreads - 1) / kEgoThreads), S), kEgoThreads, 0, st>>>(L);
  ego_sample_kernel<<<S, kSampleThreads, 0, st>>>(L);
  bool any_match = false;
  for (int i = 0; i < S; ++i) any_match |= L.job[i].match != 0;
  if (any_match) {
    const size_t smem_c = (size_t)max_pts * sizeof(int2), smem_f = (size_t)max_pts * sizeof(float2);
    LMOT_CUDA(c, cudaFuncSetAttribute(ego_coarse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
    LMOT_CUDA(c, cudaFuncSetAttribute(ego_fine_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_f));
    ego_coarse_kernel<<<dim3(max_ang, (max_w2 + kEgoThreads - 1) / kEgoThreads, S), kEgoThreads, smem_c, st>>>(L);
    if (max_f >= 5) ego_fine_kernel<<<dim3(max_f, 1, S), std::max(32, (max_f * max_f + 31) / 32 * 32), smem_f, st>>>(L);
  }
  LMOT_CUDA(c, cudaGetLastError());
  LMOT_CUDA(c, cudaMemcpyAsync(c->h_ego_res, d_res, S * sizeof(EgoRes), cudaMemcpyDeviceToHost, st));
  LMOT_CUDA(c, cudaStreamSynchronize(st));
  // step 5 on the host
  const EgoRes* R = (const EgoRes*)c->h_ego_res;
  for (int i = 0; i < S; ++i) {
    EgoMatch& e = *q[i];
    const lmot_ego_match& m = e.cfg;
    const EgoJob& J = L.job[i];
    lmot_ego_out o;
    memset(&o, 0, sizeof(o));
    o.n_used = R[i].n_used;
    o.score_max = 3 * o.n_used;
    if (dt_ok[i]) {
      double d[3] = {prior[i][0], prior[i][1], prior[i][2]};
      bool good = false;
      if (o.n_used >= m.min_points) {
        const int W = 2 * m.shift_half + 1, Rf = m.refine;
        const unsigned cidx = 0xffffffffu - (unsigned)(R[i].coarse & 0xffffffffull);
        const long long j1 = J.j0 - m.yaw_half + cidx / (unsigned)(W * W);
        const long long k1x = J.k0x - m.shift_half + cidx / (unsigned)W % (unsigned)W, k1y = J.k0y - m.shift_half + cidx % (unsigned)W;
        double best[3];
        int score;
        if (Rf == 1) {
          score = (int)(R[i].coarse >> 32);
          best[0] = (double)k1x * m.cell_m; best[1] = (double)k1y * m.cell_m; best[2] = (double)j1 * m.yaw_step;
        } else {
          const int F = 2 * Rf + 1;
          const unsigned fidx = 0xffffffffu - (unsigned)(R[i].fine & 0xffffffffull);
          const int u = (int)(fidx / (unsigned)(F * F)) - Rf, ax = (int)(fidx / (unsigned)F % (unsigned)F) - Rf, ay = (int)(fidx % (unsigned)F) - Rf;
          score = (int)(R[i].fine >> 32);
          best[0] = (double)(Rf * k1x + ax) * m.cell_m / Rf;
          best[1] = (double)(Rf * k1y + ay) * m.cell_m / Rf;
          best[2] = (double)(Rf * j1 + u) * m.yaw_step / Rf;
        }
        o.score = score;
        o.n_ref = e.n_ref;
        if ((double)score >= m.min_score_frac * 3 * o.n_used) {
          good = true;
          for (int k = 0; k < 3; ++k) d[k] = best[k];
        }
      }
      o.ok = good;
      o.dx = d[0]; o.dy = d[1]; o.dtheta = d[2];
      o.v = (d[0] * cos(d[2]) + d[1] * sin(d[2])) / dt[i];
      e.yaw += d[2];
      for (int k = 0; k < 3; ++k) e.delta[k] = d[k];
      e.delta_ok = good;
      e.dt = dt[i];
    } else {
      e.delta[0] = e.delta[1] = e.delta[2] = 0; e.delta_ok = false; e.dt = 0;
    }
    o.yaw = e.yaw;
    e.ts = ts[i];
    e.has_ref = true;
    e.ref ^= 1;
    e.n_ref = R[i].n_occ;
    *out[i] = o;
  }
  return LMOT_OK;
}

}  // namespace lmot
