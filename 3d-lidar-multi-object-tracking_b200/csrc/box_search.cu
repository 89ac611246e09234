// box_search.cu -- box search (lmot_set_box_search, include/lmot.h): each cluster's rectangle from a search over yaw with the closeness
// criterion of Zhang et al. (IV 2017), in place of boxFitting's L-shape / minimum-area-rectangle fit (boxfit.cu B4).
//
// It reads what box fitting reads: the clusters' points gathered by the stable counting sort B1-B3 of boxfit.cu (sorted_pts, seg_start,
// seg_size), and it writes what box fitting writes: cl_ok / cl_box per cluster, then the accepted boxes in cluster-id order, the box
// count and the detection semaphore.  Everything behind it (concatenation, rig poses, global frame, tracker) is unchanged.
//   box_search_kernel   one CTA per cluster (grid-stride).  Warp w owns the angle groups w, w + 8, ... of kAnglesPerPass angles; its
//                       lanes stride the points, so each angle's four extremes and its score sum are warp reductions with no CTA barrier
//                       per angle.  Every score is an integer, so the sums and the argmax do not depend on which lane or warp saw which
//                       point.  The last CTA of a frame compacts the accepted boxes.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>
#include "lmot_internal.cuh"
#include "boxfit_device.cuh"

namespace lmot {

namespace {

constexpr int kSearchThreads = 256;
constexpr int kSearchWarps = kSearchThreads / 32;
// a cluster's (x, y) stay in shared memory up to this many points (32 KB); a larger cluster is read from global memory (L2) on each of
// its 2 A / kAnglesPerPass passes
constexpr int kSearchSmemPts = 4096;
constexpr int kAnglesPerPass = 4;      // angles one pass over the points projects: one load serves four
constexpr int kTabEntries = LMOT_BOX_SEARCH_MAX_ANGLES * (LMOT_BOX_SEARCH_MAX_ANGLES + 1) / 2;

// frame blockIdx.y's angle table (A entries (c_a, s_a)) and A
struct SearchFrames { const float2* tab[kMaxBatch]; int A[kMaxBatch]; };
static_assert(sizeof(FitBatch) + sizeof(BoxFrameParams) + sizeof(SearchFrames) + 16 <= 4096, "box_search_kernel: parameter block");
static_assert(LMOT_BOX_SEARCH_MAX_ANGLES <= 511, "the argmax key keeps 511 - a in 9 bits");

__device__ __forceinline__ float2 search_pt(bool smem, const float2* s_xy, const float4* __restrict__ seg, int j) {
  if (smem) return s_xy[j];
  const float4 q = __ldg(&seg[j]);
  return make_float2(q.x, q.y);
}

// kLines: each cluster's sensor_height from its unit's ground grid (ground lines, LF)
template <bool kLines>
__device__ __forceinline__ void box_search_body(const FitBatch& B, const BoxFrameParams& PF, const SearchFrames& S, const LinesFit* LF,
                                                int max_clusters, int max_boxes) {
  fit_pdl_trigger();
  fit_pdl_wait();                          // the kernel before it (scatter_kernel, or box fitting of the launch's other units) is complete
  const FitFrame& F = B.f[blockIdx.y];
  const BoxParams& P = PF.p[blockIdx.y];   // the unit's values, its sensor's height folded in
  const float2* __restrict__ tab = S.tab[blockIdx.y];
  const int A = S.A[blockIdx.y];
  const float4* __restrict__ sorted_pts = F.sorted_pts; const int* __restrict__ seg_start = F.seg_start; const int* __restrict__ seg_size = F.seg_size;
  int* __restrict__ counters = F.counters;
  float* __restrict__ cl_box = F.cl_box; uint8_t* __restrict__ cl_ok = F.cl_ok;
  float* __restrict__ boxes = F.boxes; int* __restrict__ done = F.done; int* __restrict__ det_sem = F.det_sem;
  __shared__ float2 s_xy[kSearchSmemPts];
  __shared__ float s_maxz[kSearchWarps];
  __shared__ unsigned long long s_key[kSearchWarps];
  __shared__ float s_ext[kSearchWarps][4];
  __shared__ int s_redi[kSearchWarps];
  __shared__ int s_src[kSearchThreads];    // compaction: cluster id of the j-th accepted box of the current batch
  __shared__ int s_flag;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int K = min(counters[CNT_NUM_CLUSTER], max_clusters);

  for (int k = blockIdx.x + 1; k <= K; k += gridDim.x) {
    const int n = seg_size[k];
    const float4* seg = sorted_pts + seg_start[k];
    if (tid == 0) cl_ok[k] = 0;
    if (n < P.min_points || n <= 0) continue;      // ruleBasedFilter's first test rejects it whatever the fit
    const bool smem = n <= kSearchSmemPts;

    // ---- maxZ (getBoundingBox's, from -99) and the points into shared memory
    float maxZ = -99.f;
    for (int j = tid; j < n; j += kSearchThreads) {
      const float4 q = __ldg(&seg[j]);
      if (smem) s_xy[j] = make_float2(q.x, q.y);
      if (q.z > maxZ) maxZ = q.z;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) maxZ = fmaxf(maxZ, __shfl_xor_sync(0xFFFFFFFFu, maxZ, o));
    if (lane == 0) s_maxz[warp] = maxZ;
    __syncthreads();
    maxZ = s_maxz[0];
    for (int w = 1; w < kSearchWarps; ++w) maxZ = fmaxf(maxZ, s_maxz[w]);
    float lsh = 0.f;                                                   // ground lines: the cluster's local ground
    if (kLines) lsh = lines_sensor_height(seg, n, *LF, P.sensor_height, s_key);

    // ---- this warp's angles: extremes of u and w, then the closeness sums; best key (S_a << 9) | (511 - a) with its extremes
    unsigned long long best = 0ull;
    float bext[4] = {0.f, 0.f, 0.f, 0.f};
    for (int a0 = warp * kAnglesPerPass; a0 < A; a0 += kSearchWarps * kAnglesPerPass) {
      float cs[kAnglesPerPass], sn[kAnglesPerPass];
      float umin[kAnglesPerPass], umax[kAnglesPerPass], wmin[kAnglesPerPass], wmax[kAnglesPerPass];
#pragma unroll
      for (int r = 0; r < kAnglesPerPass; ++r) {
        const float2 t = tab[a0 + r < A ? a0 + r : a0];
        cs[r] = t.x; sn[r] = t.y;
        umin[r] = FLT_MAX; umax[r] = -FLT_MAX; wmin[r] = FLT_MAX; wmax[r] = -FLT_MAX;
      }
      for (int j = lane; j < n; j += 32) {
        const float2 p = search_pt(smem, s_xy, seg, j);
#pragma unroll
        for (int r = 0; r < kAnglesPerPass; ++r) {
          const float u = p.x * cs[r] + p.y * sn[r], w = p.y * cs[r] - p.x * sn[r];    // (the library is built without contraction)
          umin[r] = fminf(umin[r], u); umax[r] = fmaxf(umax[r], u); wmin[r] = fminf(wmin[r], w); wmax[r] = fmaxf(wmax[r], w);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int r = 0; r < kAnglesPerPass; ++r) {
          umin[r] = fminf(umin[r], __shfl_xor_sync(0xFFFFFFFFu, umin[r], o)); umax[r] = fmaxf(umax[r], __shfl_xor_sync(0xFFFFFFFFu, umax[r], o));
          wmin[r] = fminf(wmin[r], __shfl_xor_sync(0xFFFFFFFFu, wmin[r], o)); wmax[r] = fmaxf(wmax[r], __shfl_xor_sync(0xFFFFFFFFu, wmax[r], o));
        }
      unsigned long long sum[kAnglesPerPass];
#pragma unroll
      for (int r = 0; r < kAnglesPerPass; ++r) sum[r] = 0ull;
      for (int j = lane; j < n; j += 32) {
        const float2 p = search_pt(smem, s_xy, seg, j);
#pragma unroll
        for (int r = 0; r < kAnglesPerPass; ++r) {
          const float u = p.x * cs[r] + p.y * sn[r], w = p.y * cs[r] - p.x * sn[r];
          const float d1 = fminf(umax[r] - u, u - umin[r]), d2 = fminf(wmax[r] - w, w - wmin[r]);
          const float d = fmaxf(fminf(d1, d2), 0.01f);
          sum[r] += (unsigned)(65536.0f / d);                     // IEEE division, truncated
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int r = 0; r < kAnglesPerPass; ++r) sum[r] += __shfl_xor_sync(0xFFFFFFFFu, sum[r], o);
#pragma unroll
      for (int r = 0; r < kAnglesPerPass; ++r) {
        const int a = a0 + r;
        const unsigned long long key = (sum[r] << 9) | (unsigned long long)(511 - a);
        if (a < A && key > best) { best = key; bext[0] = umin[r]; bext[1] = umax[r]; bext[2] = wmin[r]; bext[3] = wmax[r]; }
      }
    }
    if (lane == 0) { s_key[warp] = best; s_ext[warp][0] = bext[0]; s_ext[warp][1] = bext[1]; s_ext[warp][2] = bext[2]; s_ext[warp][3] = bext[3]; }
    __syncthreads();
    if (tid == 0) {
      int bw = 0;
      for (int w = 1; w < kSearchWarps; ++w) if (s_key[w] > s_key[bw]) bw = w;
      const int a = 511 - (int)(s_key[bw] & 511ull);
      const float2 t = tab[a];
      const float c = t.x, s = t.y;
      const float u0 = s_ext[bw][0], u1 = s_ext[bw][1], w0 = s_ext[bw][2], w1 = s_ext[bw][3];
      const float U[4] = {u0, u1, u1, u0}, W[4] = {w0, w0, w1, w1};
      float pc[4][2];
      for (int q = 0; q < 4; ++q) { pc[q][0] = U[q] * c - W[q] * s; pc[q][1] = U[q] * s + W[q] * c; }
      const bool ok = rule_filter(pc, maxZ, n, P, kLines ? lsh : P.sensor_height);
      cl_ok[k] = ok ? 1 : 0;
      if (ok) {
        float* b = cl_box + (size_t)k * 24;
        for (int h = 0; h < 2; ++h)
          for (int q = 0; q < 4; ++q) { b[(h * 4 + q) * 3] = pc[q][0]; b[(h * 4 + q) * 3 + 1] = pc[q][1]; b[(h * 4 + q) * 3 + 2] = h == 0 ? -(kLines ? lsh : P.sensor_height) : maxZ; }
      }
    }
    __syncthreads();                       // (s_xy, s_key and s_maxz are the next cluster's)
  }

  // ---- the last CTA of the frame compacts the accepted boxes in cluster-id order (box fitting's markers are not written: only the
  // stage entry point lmot_box_fit returns them, and it never searches)
  __threadfence();
  __syncthreads();
  if (tid == 0) s_flag = (atomicAdd(done, 1) == (int)gridDim.x - 1);
  __syncthreads();
  if (!s_flag) return;
  __threadfence();
  int carry = 0;
  for (int k0 = 1; k0 <= K; k0 += kSearchThreads) {
    const int k = k0 + tid;
    const int f = (k <= K) ? __ldcg((const unsigned char*)&cl_ok[k]) : 0;
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, f);
    if (lane == 0) s_redi[warp] = __popc(bal);
    __syncthreads();
    int wbase = 0, tot = 0;
    for (int w = 0; w < kSearchWarps; ++w) { if (w < warp) wbase += s_redi[w]; tot += s_redi[w]; }
    const int pos = carry + wbase + __popc(bal & ((1u << lane) - 1u));
    if (f && pos < max_boxes) s_src[pos - carry] = k;
    __syncthreads();
    const int nacc = min(tot, max_boxes - carry);
    for (int e = tid; e < nacc * 24; e += kSearchThreads) {
      const int j = e / 24, w = e - j * 24;
      boxes[(size_t)(carry + j) * 24 + w] = __ldcg(&cl_box[(size_t)s_src[j] * 24 + w]);
    }
    carry += tot;
    __syncthreads();
  }
  if (tid == 0) {
    if (carry > max_boxes) { counters[CNT_ERROR] = LMOT_ERR_CAPACITY; carry = max_boxes; }
    counters[CNT_N_BOXES] = carry;
  }
  if (det_sem) {                           // the unit's detection is complete (as box_fit_kernel posts it)
    __syncthreads();
    if (tid == 0) { __threadfence(); atomicAdd(det_sem, 1); }
  }
}

__global__ void __launch_bounds__(kSearchThreads)
box_search_kernel(const __grid_constant__ FitBatch B, const __grid_constant__ BoxFrameParams PF, const __grid_constant__ SearchFrames S,
                  int max_clusters, int max_boxes) {
  box_search_body<false>(B, PF, S, nullptr, max_clusters, max_boxes);
}

static_assert(sizeof(FitBatch) + sizeof(BoxFrameParams) + sizeof(SearchFrames) + sizeof(LinesFit) + 16 <= 4096,
              "box_search_lines_kernel: parameter block");
__global__ void __launch_bounds__(kSearchThreads)
box_search_lines_kernel(const __grid_constant__ FitBatch B, const __grid_constant__ BoxFrameParams PF, const __grid_constant__ SearchFrames S,
                        const __grid_constant__ LinesFit LG, int max_clusters, int max_boxes) {
  box_search_body<true>(B, PF, S, &LG, max_clusters, max_boxes);
}

}  // namespace

bool box_search_valid(const lmot_box_search& b) {
  return (b.on == 0 || b.on == 1) && b.n_angles >= 1 && b.n_angles <= LMOT_BOX_SEARCH_MAX_ANGLES;
}

void box_search_table(int A, float (*out)[2]) {
  for (int a = 0; a < A; ++a) {
    const double th = (M_PI / 2) * a / A;
    out[a][0] = (float)cos(th);
    out[a][1] = (float)sin(th);
  }
}

// every A's table, back to back (table A at A(A-1)/2): immutable, so ticks in flight and sequences with different A share it
int box_search_ensure(Ctx* c) {
  if (c->d_bs_tab) return LMOT_OK;
  std::vector<float> h((size_t)kTabEntries * 2);
  for (int A = 1; A <= LMOT_BOX_SEARCH_MAX_ANGLES; ++A)
    box_search_table(A, reinterpret_cast<float(*)[2]>(h.data() + (size_t)A * (A - 1)));
  float2* d = nullptr;
  LMOT_CUDA(c, cudaMalloc(&d, h.size() * sizeof(float)));
  if (cudaMemcpy(d, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
    cudaFree(d);
    return LMOT_ERR_CUDA;
  }
  c->d_bs_tab = d;
  return LMOT_OK;
}

int box_search_launch(Ctx* c, Slot* const* units, int n, const lmot_detect_params* det, const int* A, cudaStream_t st, bool post_sem, int gx,
                      bool pdl, const float* const* lines) {
  if (n < 1 || n > kMaxBatch || !c->d_bs_tab) return LMOT_ERR_STATE;
  FitBatch B;
  BoxFrameParams FP;
  SearchFrames S;
  LinesFit LG;
  memset(&FP, 0, sizeof(FP));
  memset(&S, 0, sizeof(S));
  memset(&LG, 0, sizeof(LG));
  for (int i = 0; i < n; ++i) {
    fit_frame_of(units[i], B.f[i], post_sem);
    FP.p[i] = box_params_of(det[i]);
    if (lines) lines_fit_of(det[i], lines[i], LG, i);
    S.tab[i] = c->d_bs_tab + (size_t)A[i] * (A[i] - 1) / 2;
    S.A[i] = A[i];
  }
  for (int i = n; i < kMaxBatch; ++i) B.f[i] = B.f[0];
  cudaLaunchAttribute at;
  at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at.val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(gx, n); cfg.blockDim = dim3(kSearchThreads); cfg.dynamicSmemBytes = 0; cfg.stream = st; cfg.attrs = &at; cfg.numAttrs = 1;
  if (lines) LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, box_search_lines_kernel, B, FP, S, LG, c->prm.max_clusters, c->prm.max_boxes));
  else LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, box_search_kernel, B, FP, S, c->prm.max_clusters, c->prm.max_boxes));
  return LMOT_OK;
}

}  // namespace lmot
