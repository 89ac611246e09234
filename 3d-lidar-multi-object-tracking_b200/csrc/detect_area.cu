// detect_area.cu -- detection areas (lmot_set_detect_area / lmot_seq_set_detect_area, include/lmot.h): the cell mask of every masked unit
// of a submission, from its stream's polygon rings, its pose and its clustering extent.  An opt-in filter the reference does not have.
//
// PNPOLY with the ray along +y: whether an edge straddles a cell depends only on the cell's bit-plane row xI, so a row's crossings yc are
// computed once, and cell (xI, yI) is inside iff an odd number of them satisfy cy(yI) < yc.  cy is non-decreasing in yI, so a crossing
// counts for the cells yI < k (k = the number of cells whose centre lies below it, found by bisection): it toggles bit k of the row's
// difference vector D, and inside(yI) = XOR of D[k] over k > yI, a suffix XOR over 251 bits.  That is O(250 x E) per unit instead of
// O(62,500 x E).  detect_area_kernel runs one CTA of 32 warps per unit, one warp per row at a time, with the 250 cell centres in
// shared memory; the host restatement (area_mask_host, behind
// lmot_detect_area_mask) evaluates the definition cell by cell with the same double expressions, and the library is built with
// -fmad=false, so the two agree bit for bit.
#include <cmath>
#include <cstring>
#include "lmot_internal.cuh"
#include "ccl_device.cuh"

namespace lmot {

namespace {

constexpr int kAreaThreads = 1024;

struct AreaParams { AreaJob j[kMaxBatch]; };

// the vertex in unit coordinates: dx = px - t0, dy = py - t1, u = r00*dx + r10*dy, w = r01*dx + r11*dy (pose widened from float)
__host__ __device__ __forceinline__ void area_uw(const float* m, double px, double py, double& u, double& w) {
  const double dx = px - (double)m[3], dy = py - (double)m[7];
  u = (double)m[0] * dx + (double)m[4] * dy;
  w = (double)m[1] * dx + (double)m[5] * dy;
}

__host__ __device__ __forceinline__ double area_centre(int i, double roi) { return ((double)i + 0.5) * roi / 250.0 - roi / 2.0; }

// the crossing of edge a -> b with the line u = cx (the caller checked that it straddles)
__host__ __device__ __forceinline__ double area_cross(double au, double aw, double bu, double bw, double cx) {
  return aw + (cx - au) * (bw - aw) / (bu - au);
}

__global__ void __launch_bounds__(kAreaThreads)
detect_area_kernel(const __grid_constant__ AreaParams P) {
  __shared__ double s_u[LMOT_AREA_MAX_VERTICES], s_w[LMOT_AREA_MAX_VERTICES];
  __shared__ unsigned short s_next[LMOT_AREA_MAX_VERTICES];
  __shared__ unsigned s_d[kAreaThreads / 32][kRowWords];
  __shared__ double s_c[kNumGrid];       // cell centres: the bisection's probes, and the rows' abscissae
  const AreaJob& J = P.j[blockIdx.x];
  const AreaBlock* __restrict__ A = J.a;
  const int nv = A->n_vertices, nr = A->n_rings;
  const double roi = (double)J.roi;
  for (int i = threadIdx.x; i < nv; i += kAreaThreads) area_uw(J.pose, A->xy[2 * i], A->xy[2 * i + 1], s_u[i], s_w[i]);
  if (threadIdx.x < kNumGrid) s_c[threadIdx.x] = area_centre(threadIdx.x, roi);
  if (threadIdx.x < 32) {            // the edge a -> next(a) of every vertex: rings closed implicitly
    for (int r = 0, v0 = 0; r < nr; v0 += A->ring_len[r], ++r) {
      const int len = A->ring_len[r];
      for (int e = threadIdx.x; e < len; e += 32) s_next[v0 + e] = (unsigned short)(v0 + (e + 1 < len ? e + 1 : 0));
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned* d = s_d[warp];
  if (lane < kRowWords) d[lane] = 0u;
  __syncthreads();
  const unsigned flip = A->keep_outside ? 0xFFFFFFFFu : 0u;
  for (int xI = warp; xI < kNumGrid; xI += kAreaThreads / 32) {
    const double cx = s_c[xI];
    for (int e = lane; e < nv; e += 32) {
      const double au = s_u[e], bu = s_u[s_next[e]];
      if ((au > cx) != (bu > cx)) {
        const double yc = area_cross(au, s_w[e], bu, s_w[s_next[e]], cx);
        int lo = 0, hi = kNumGrid;         // k = the first cell whose centre is not below yc
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (s_c[mid] < yc) lo = mid + 1; else hi = mid;
        }
        atomicXor(&d[lo >> 5], 1u << (lo & 31));
      }
    }
    __syncwarp();
    const unsigned dw = lane < kRowWords ? d[lane] : 0u;
    const unsigned par = __ballot_sync(0xFFFFFFFFu, __popc(dw) & 1);
    if (lane < kRowWords) {
      unsigned y = dw;                     // y bit b = XOR of dw's bits >= b
      y ^= y >> 1; y ^= y >> 2; y ^= y >> 4; y ^= y >> 8; y ^= y >> 16;
      const unsigned carry = (__popc(par >> (lane + 1)) & 1) ? 0xFFFFFFFFu : 0u;   // the words above
      unsigned m = ((y >> 1) ^ carry) ^ flip;
      if (lane == kRowWords - 1) m &= kLastWordMask;
      J.mask[xI * kRowWords + lane] = m;
      d[lane] = 0u;
    }
    __syncwarp();
  }
}

}  // namespace

bool area_valid(const lmot_area* a) {
  if (!a || a->n_rings == 0) return true;
  if (a->n_rings < 0 || a->n_rings > LMOT_AREA_MAX_RINGS || !a->ring_len || !a->xy) return false;
  if (a->keep_outside != 0 && a->keep_outside != 1) return false;
  long long nv = 0;
  for (int r = 0; r < a->n_rings; ++r) {
    if (a->ring_len[r] < 3) return false;
    nv += a->ring_len[r];
    if (nv > LMOT_AREA_MAX_VERTICES) return false;
  }
  for (long long i = 0; i < 2 * nv; ++i) if (!std::isfinite(a->xy[i])) return false;
  return true;
}

void area_copy(AreaBlock& dst, const lmot_area* a) {
  memset(&dst, 0, sizeof(dst));
  if (!a || a->n_rings == 0) return;
  dst.n_rings = a->n_rings;
  dst.keep_outside = a->keep_outside;
  for (int r = 0; r < a->n_rings; ++r) { dst.ring_len[r] = a->ring_len[r]; dst.n_vertices += a->ring_len[r]; }
  memcpy(dst.xy, a->xy, (size_t)dst.n_vertices * 2 * sizeof(double));
}

// the definition, cell by cell
void area_mask_host(const AreaBlock& a, const float* pose, float roi_f, unsigned* out) {
  static const float kIdentity[12] = {1.f, 0.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f, 1.f, 0.f};
  const float* m = pose ? pose : kIdentity;
  const double roi = (double)roi_f;
  const int nv = a.n_vertices;
  static thread_local double u[LMOT_AREA_MAX_VERTICES], w[LMOT_AREA_MAX_VERTICES];
  static thread_local int nxt[LMOT_AREA_MAX_VERTICES];
  for (int i = 0; i < nv; ++i) area_uw(m, a.xy[2 * i], a.xy[2 * i + 1], u[i], w[i]);
  for (int r = 0, v0 = 0; r < a.n_rings; v0 += a.ring_len[r], ++r)
    for (int e = 0; e < a.ring_len[r]; ++e) nxt[v0 + e] = v0 + (e + 1 < a.ring_len[r] ? e + 1 : 0);
  double yc[LMOT_AREA_MAX_VERTICES];
  memset(out, 0, kBitWords * sizeof(unsigned));
  for (int xI = 0; xI < kNumGrid; ++xI) {
    const double cx = area_centre(xI, roi);
    int nc = 0;
    for (int e = 0; e < nv; ++e)
      if ((u[e] > cx) != (u[nxt[e]] > cx)) yc[nc++] = area_cross(u[e], w[e], u[nxt[e]], w[nxt[e]], cx);
    for (int yI = 0; yI < kNumGrid; ++yI) {
      const double cy = area_centre(yI, roi);
      int odd = 0;
      for (int k = 0; k < nc; ++k) odd ^= (cy < yc[k]) ? 1 : 0;
      if ((odd != 0) != (a.keep_outside != 0)) out[xI * kRowWords + (yI >> 5)] |= 1u << (yI & 31);
    }
  }
}

int area_ensure(Ctx* c, Slot* s, int blocks) {
  if (!s->d_area_mask) LMOT_CUDA(c, cudaMalloc(&s->d_area_mask, kBitWords * sizeof(unsigned)));
  if (blocks > 0 && !s->d_area) LMOT_CUDA(c, cudaMalloc(&s->d_area, (size_t)blocks * sizeof(AreaBlock)));
  return LMOT_OK;
}

int area_launch(Ctx* c, cudaStream_t st, const AreaJob* jobs, int n_jobs) {
  if (n_jobs < 1 || n_jobs > kMaxBatch) return LMOT_ERR_INVALID;
  AreaParams P;
  memset(&P, 0, sizeof(P));
  for (int i = 0; i < n_jobs; ++i) P.j[i] = jobs[i];
  detect_area_kernel<<<n_jobs, kAreaThreads, 0, st>>>(P);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

}  // namespace lmot
