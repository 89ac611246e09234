// boxfit.cu -- per-cluster L-shape / minimum-area-rectangle box fitting on sm_90a.
//
// Replaces boxFitting (/root/reference/object_tracking/src/cluster/box_fitting.cpp:422-431):
//   getClusteredPoints (:46-72)   gather the elevated points of every cluster IN CLOUD ORDER
//   getBoundingBox (:212-418)     per cluster: pixelise @18 px/m around point #0, first-occurrence min/max
//                                 slope points, max z (:239-293); L-shape fit from 80 seeded random samples
//                                 (:296-356) or cv::minAreaRect (:358-365); ruleBasedFilter (:97-158);
//                                 8-corner box (:379-389); mark_cluster centroid + AABB (:161-209)
//
// The reference's results depend on the order of the points inside a cluster (point #0, first-occurrence
// ties, the random index picks the i-th point), so the gather is a STABLE counting sort by cluster id:
//   B1 tile_hist_kernel    per 1024-point tile: cluster id of each point (label grid lookup through the u16 cell
//                          id kept by clustering) + shared-memory histogram -> table[tile][cluster]
//   B2 seg_offsets_body    exclusive scan over tiles per cluster, then over clusters -> segment starts (run by B1's last CTA)
//   B3 scatter_kernel      stable in-tile ranks (warp match_any, warps in order) -> sorted point indices
//   B4 box_fit_kernel      one CTA per cluster (grid-stride), all of getBoundingBox; the last CTA to finish
//                          compacts the accepted boxes in cluster-id order (:355,365 skip rejected clusters).
//
// cv::minAreaRect is third-party arithmetic that is not in /root/reference: it is implemented as the exact
// integer contract documented in oracle/mar_contract.cpp / DESIGN.md (parity for that one call is UNPINNED
// against OpenCV itself, bit-exact against the contract).
#include <cfloat>
#include <climits>
#include <cstring>
#include <random>
#include <vector>
#include "lmot_internal.cuh"
#include "ccl_device.cuh"
#include "boxfit_device.cuh"

namespace lmot {

namespace {

constexpr int kTile = 1024;
constexpr int kFitThreadsFrame = 512;   // one CTA per cluster: the largest cluster IS the kernel of a single frame
constexpr int kFitThreadsBatch = 256;   // batched ticks hold ~8x the clusters: more, smaller CTAs per SM finish the union sooner
constexpr int kCols = 1800;        // pixel columns a cluster can span: offsetX-450 = picX-initPicX in [-899,899]
constexpr int kColShift = 899 - 450;
constexpr int kHullCap = 2048;

// ---------------------------------------------------------------------------------------------- B1
__device__ __forceinline__ void seg_offsets_body(const FitFrame& F, int max_clusters);

// kArea: a point whose cell is outside its unit's detection-area mask `area` gets cluster 0 -- dilation can label masked cells, and
// those hold no point of the masked cloud E_area
// kLayers: a layered unit (lt->slice set) takes each point's cluster from its slice and its column's run table (layers.cu) instead of the
// label grid; its slice byte already excludes points without a column or outside the detection area
template <bool kArea, bool kLayers = false>
__device__ __forceinline__ void tile_hist_body(const FitBatch& B, int max_clusters, const unsigned* __restrict__ area,
                                               const LayerTab* lt = nullptr) {
  extern __shared__ int s_hist[];
  fit_pdl_trigger();
  const FitFrame& F = B.f[blockIdx.y];
  const uint16_t* __restrict__ cart = F.cart; const int* __restrict__ label_grid = F.label_grid; const int* __restrict__ counters = F.counters;
  uint16_t* __restrict__ pcid = F.pcid; int* __restrict__ table = F.table;
  const int n = counters[CNT_N_ELEV];
  const int K = min(counters[CNT_NUM_CLUSTER], max_clusters);
  const int tile = blockIdx.x;
  if (tile * kTile < n) {
  for (int k = threadIdx.x; k <= K; k += kTile) s_hist[k] = 0;
  __syncthreads();
  const int i = tile * kTile + threadIdx.x;
  unsigned cid = 0;
  if (i < n) {
    const unsigned c = cart[i];
    if (kLayers && lt->slice) {
      const unsigned sl = __ldg(&lt->slice[i]);
      if (sl != 0xFFu) {
        const unsigned d = __ldg(&lt->cols[c]);
        if ((d >> sl) & 1u) cid = (unsigned)(-__ldg(&lt->lab[__ldg(&lt->base[c]) + __popc(piece_starts(d) & ((2u << sl) - 1u)) - 1]));
      }
    } else if (c != kNoCell && (!kArea || !area || area_kept(area, c))) {
      cid = (unsigned)__ldg(&label_grid[c]);
    }
    if (cid > (unsigned)K) cid = 0;                    // capacity overflow is reported by seg_offsets_kernel
    pcid[i] = (uint16_t)cid;
  }
  const unsigned grp = __match_any_sync(0xFFFFFFFFu, cid);
  if (cid != 0 && (threadIdx.x & 31) == __ffs(grp) - 1) atomicAdd(&s_hist[cid], __popc(grp));
  __syncthreads();
  int* row = table + (size_t)tile * (max_clusters + 1);
  for (int k = threadIdx.x; k <= K; k += kTile) row[k] = s_hist[k];
  }
  // B2 by the last CTA of the frame to get here (tiles past the end of the cloud count too)
  __shared__ int s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicInc(F.hist_ctr, gridDim.x - 1u) == gridDim.x - 1u) ? 1 : 0;
  __syncthreads();
  if (s_last) { __threadfence(); seg_offsets_body(F, max_clusters); }
}

__global__ void __launch_bounds__(kTile)
tile_hist_kernel(const __grid_constant__ FitBatch B, int max_clusters) { tile_hist_body<false>(B, max_clusters, nullptr); }

// detection areas: frame blockIdx.y's unit mask A.m[blockIdx.y] (nullptr: an unmasked unit of the same launch)
struct FitAreaMasks { const unsigned* m[kMaxBatch]; };

__global__ void __launch_bounds__(kTile)
tile_hist_area_kernel(const __grid_constant__ FitBatch B, int max_clusters, const __grid_constant__ FitAreaMasks A) {
  tile_hist_body<true>(B, max_clusters, A.m[blockIdx.y]);
}

// layered clustering: unit blockIdx.y's run tables (slice nullptr: a unit of the same launch clustered on its label grid) and area mask
struct FitLayers { LayerTab t[kMaxBatch]; };

__global__ void __launch_bounds__(kTile)
tile_hist_layers_kernel(const __grid_constant__ FitBatch B, int max_clusters, const __grid_constant__ FitAreaMasks A,
                        const __grid_constant__ FitLayers L) {
  tile_hist_body<true, true>(B, max_clusters, A.m[blockIdx.y], &L.t[blockIdx.y]);
}

// ---------------------------------------------------------------------------------------------- B2
// exclusive scan over tiles per cluster, then over clusters -> segment starts.  One CTA of 1,024 threads per frame: the LAST
// tile_hist CTA of the frame to finish runs it (no launch in between); seg_offsets_kernel wraps it for frames without points.
__device__ __forceinline__ void seg_offsets_body(const FitFrame& F, int max_clusters) {
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  int* __restrict__ table = F.table; int* counters = F.counters;
  int* __restrict__ seg_start = F.seg_start; int* __restrict__ seg_size = F.seg_size; int* __restrict__ done = F.done;
  const int n = counters[CNT_N_ELEV];
  int K = counters[CNT_NUM_CLUSTER];
  if (threadIdx.x == 0) {
    s_carry = 0;
    *done = 0;
    if (K > max_clusters) counters[CNT_ERROR] = LMOT_ERR_CAPACITY;
  }
  K = min(K, max_clusters);
  const int n_tiles = (n + kTile - 1) / kTile;
  const int stride = max_clusters + 1;
  __syncthreads();
  // P lanes per cluster (a power of two, aligned inside a warp): each takes a contiguous range of tiles, so that a frame of ~60 tiles
  // and ~100 clusters is ONE batch of independent loads per lane instead of four dependent batches on 100 of the 1,024 threads
  const int P = K <= 128 ? 8 : (K <= 256 ? 4 : (K <= 512 ? 2 : 1));
  const int per_round = 1024 / P;
  const int per = (n_tiles + P - 1) / P;                // tiles per lane
  for (int k0 = 1; k0 <= K; k0 += per_round) {
    const int k = k0 + (int)threadIdx.x / P, j = (int)threadIdx.x % P;
    const int t_beg = min(j * per, n_tiles), t_end = min(t_beg + per, n_tiles);
    const bool mine = k <= K;
    int v[16];
    int sum = 0;
    if (mine) {
      if (per <= 16) {
#pragma unroll
        for (int u = 0; u < 16; ++u) { v[u] = (t_beg + u < t_end) ? table[(size_t)(t_beg + u) * stride + k] : 0; }
#pragma unroll
        for (int u = 0; u < 16; ++u) sum += v[u];
      } else {
        for (int t0 = t_beg; t0 < t_end; t0 += 16) {
#pragma unroll
          for (int u = 0; u < 16; ++u) v[u] = (t0 + u < t_end) ? table[(size_t)(t0 + u) * stride + k] : 0;
#pragma unroll
          for (int u = 0; u < 16; ++u) sum += v[u];
        }
      }
    }
    // exclusive prefix of the lanes' sums inside the cluster's group of P lanes; the group total ends up on every lane
    int incl_l = sum;
    for (int o = 1; o < P; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, incl_l, o, P); if (j >= o) incl_l += t; }
    const int group_total = __shfl_sync(0xFFFFFFFFu, incl_l, P - 1, P);
    if (mine) {
      int run = incl_l - sum;
      if (per <= 16) {
#pragma unroll
        for (int u = 0; u < 16; ++u)
          if (t_beg + u < t_end) { table[(size_t)(t_beg + u) * stride + k] = run; run += v[u]; }
      } else {
        for (int t0 = t_beg; t0 < t_end; t0 += 16) {       // 16 independent loads in flight, then the dependent prefix
#pragma unroll
          for (int u = 0; u < 16; ++u) v[u] = (t0 + u < t_end) ? table[(size_t)(t0 + u) * stride + k] : 0;
#pragma unroll
          for (int u = 0; u < 16; ++u)
            if (t0 + u < t_end) { table[(size_t)(t0 + u) * stride + k] = run; run += v[u]; }
        }
      }
    }
    const int total = (mine && j == 0) ? group_total : 0;   // one lane per cluster carries its size into the scan over clusters
    // block exclusive scan of `total` (+ carry from previous chunks of 1024 clusters)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = total;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      const int v = s_warp[lane];
      int wi = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, wi, o); if (lane >= o) wi += t; }
      s_warp[lane] = wi - v;
    }
    __syncthreads();
    const int excl = s_carry + s_warp[warp] + incl - total;
    if (mine && j == 0) { seg_start[k] = excl; seg_size[k] = total; }
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = excl + total;
    __syncthreads();
  }
  if (threadIdx.x == 0) counters[CNT_N_CLUSTERED] = s_carry;
}

__global__ void __launch_bounds__(1024)
seg_offsets_kernel(const __grid_constant__ FitBatch B, int max_clusters) { seg_offsets_body(B.f[blockIdx.x], max_clusters); }

// ---------------------------------------------------------------------------------------------- B3
__global__ void __launch_bounds__(kTile)
scatter_kernel(const __grid_constant__ FitBatch B, int max_clusters) {
  extern __shared__ int s_cur[];
  fit_pdl_trigger();
  fit_pdl_wait();                          // tile_hist_kernel (+ the segment offsets of its last CTA) is complete
  const FitFrame& F = B.f[blockIdx.y];
  const uint16_t* __restrict__ pcid = F.pcid; const float4* __restrict__ elev = F.elev; const int* __restrict__ counters = F.counters;
  const int* __restrict__ table = F.table; const int* __restrict__ seg_start = F.seg_start; float4* __restrict__ sorted_pts = F.sorted_pts;
  const int n = counters[CNT_N_ELEV];
  const int K = min(counters[CNT_NUM_CLUSTER], max_clusters);
  const int tile = blockIdx.x;
  if (tile * kTile >= n) return;
  const int* row = table + (size_t)tile * (max_clusters + 1);
  for (int k = threadIdx.x + 1; k <= K; k += kTile) s_cur[k] = seg_start[k] + row[k];
  __syncthreads();
  const int i = tile * kTile + threadIdx.x;
  const unsigned cid = (i < n) ? pcid[i] : 0u;
  float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
  if (cid != 0) q = __ldg(&elev[i]);            // the point itself travels: box fitting then reads its cluster contiguously
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned grp = __match_any_sync(0xFFFFFFFFu, cid);
  const int leader = __ffs(grp) - 1;
  const int rank = __popc(grp & ((1u << lane) - 1u));
  // Ranks follow the cloud order: the warps' groups must take their segment ranges in warp order.  Every warp lists its groups
  // (cluster id, size); warp 0 then walks the 32 lists in order, one group per lane -- a warp's groups have distinct ids, so only
  // consecutive lists depend on each other.  (The warps taking turns behind 32 CTA barriers was most of this kernel's time.)
  __shared__ unsigned short s_gcid[kTile / 32][32];
  __shared__ unsigned char s_gcnt[kTile / 32][32], s_gn[kTile / 32];
  __shared__ int s_gbase[kTile / 32][32];
  const bool is_leader = cid != 0 && lane == leader;
  const unsigned lmask = __ballot_sync(0xFFFFFFFFu, is_leader);
  if (is_leader) {
    const int slot = __popc(lmask & ((1u << lane) - 1u));
    s_gcid[warp][slot] = (unsigned short)cid; s_gcnt[warp][slot] = (unsigned char)__popc(grp);
  }
  if (lane == 0) s_gn[warp] = (unsigned char)__popc(lmask);
  __syncthreads();
  if (warp == 0) {
    for (int w = 0; w < kTile / 32; ++w) {
      if (lane < (int)s_gn[w]) {
        const int c = s_gcid[w][lane];
        const int base = s_cur[c];
        s_cur[c] = base + (int)s_gcnt[w][lane];
        s_gbase[w][lane] = base;
      }
      __syncwarp();
    }
  }
  __syncthreads();
  if (cid != 0) sorted_pts[s_gbase[warp][__popc(lmask & ((1u << leader) - 1u))] + rank] = q;
}

// ---------------------------------------------------------------------------------------------- B4
__device__ __forceinline__ unsigned okey(float f) {   // order-preserving, -0 == +0
  if (f == 0.f) f = 0.f;
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

template <typename T, typename Op>
__device__ __forceinline__ T block_reduce(T v, Op op, T* s_buf) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
  __syncthreads();
  if (lane == 0) s_buf[warp] = v;
  __syncthreads();
  T r = s_buf[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) r = op(r, s_buf[w]);
  return r;
}

struct MinU64 { __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a < b ? a : b; } };
struct MaxU64 { __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a > b ? a : b; } };
struct MaxF { __device__ float operator()(float a, float b) const { return fmaxf(a, b); } };
struct MinF { __device__ float operator()(float a, float b) const { return fminf(a, b); } };
struct AddD { __device__ double operator()(double a, double b) const { return a + b; } };
struct MinI { __device__ int operator()(int a, int b) const { return a < b ? a : b; } };
struct MaxI { __device__ int operator()(int a, int b) const { return a > b ? a : b; } };


// kRig: sensor_height from the frame's FitFrame (a sensor rig, lmot_set_sensors) instead of P
template <int NT, bool kRig>
__global__ void __launch_bounds__(NT, 1024 / NT)     // <= 64 registers: 1,024 threads of box fitting per SM
box_fit_kernel(const __grid_constant__ FitBatch B, const __grid_constant__ BoxParams P,
               const unsigned long long* __restrict__ mt_raw, int n_raw, int max_clusters, int max_boxes) {
  constexpr bool kLines = false;
  const LinesFit* LF = nullptr;
  // box_fit_body.inc reads: B, P, NT, kRig, kLines, LF, mt_raw, n_raw, max_clusters, max_boxes
#include "box_fit_body.inc"
}

static_assert(sizeof(FitBatch) + sizeof(BoxFrameParams) + 32 <= 4096, "box_fit_frame_kernel: parameter block");

template <int NT>
__global__ void __launch_bounds__(NT, 1024 / NT)
box_fit_frame_kernel(const __grid_constant__ FitBatch B, const __grid_constant__ BoxFrameParams PF,
                     const unsigned long long* __restrict__ mt_raw, int n_raw, int max_clusters, int max_boxes) {
  constexpr bool kRig = false;                 // (the sensor's height is folded into the frame's entry)
  constexpr bool kLines = false;
  const LinesFit* LF = nullptr;
  const BoxParams& P = PF.p[blockIdx.y];
  // box_fit_body.inc reads: B, P, NT, kRig, kLines, LF, mt_raw, n_raw, max_clusters, max_boxes
#include "box_fit_body.inc"
}

// ground lines (lmot_set_ground_lines): box_fit_frame_kernel with each cluster's sensor_height from its unit's ground grid (a unit without
// one: its entry's, as box_fit_frame_kernel)
static_assert(sizeof(FitBatch) + sizeof(BoxFrameParams) + sizeof(LinesFit) + 32 <= 4096, "box_fit_lines_kernel: parameter block");

template <int NT>
__global__ void __launch_bounds__(NT, 1024 / NT)
box_fit_lines_kernel(const __grid_constant__ FitBatch B, const __grid_constant__ BoxFrameParams PF, const __grid_constant__ LinesFit LG,
                     const unsigned long long* __restrict__ mt_raw, int n_raw, int max_clusters, int max_boxes) {
  constexpr bool kRig = false;
  constexpr bool kLines = true;
  const LinesFit* LF = &LG;
  const BoxParams& P = PF.p[blockIdx.y];
  // box_fit_body.inc reads: B, P, NT, kRig, kLines, LF, mt_raw, n_raw, max_clusters, max_boxes
#include "box_fit_body.inc"
}

// one box (8 corners, 24 floats) moved by pose m
__device__ __forceinline__ void rig_apply_box(const float* m, float* b) {
#pragma unroll
  for (int c = 0; c < 8; ++c) rig_apply(m, b[3 * c], b[3 * c + 1], b[3 * c + 2]);
}

// batched submissions (one frame per sensor stream): the box lists of frames [f0, f0 + n_frames), concatenated in stream order, are ONE
// measurement list for the tracker (tracking/main.cpp:98-141 unpacks whatever the trackbox message holds; one immUkfJpdaf call per tick).
// kRig: frame f0 + w's boxes are moved into the vehicle frame by its sensor's pose R->m[f0 + w] on the way.  frame_counts row w = frame f0 + w.
template <bool kRig>
__device__ __forceinline__ void concat_boxes_body(const FitBatch& B, const RigPoses* R, int f0, int n_frames, int max_boxes, float* __restrict__ boxes,
                                                  int* __restrict__ counters, int* __restrict__ frame_counts, int* __restrict__ det_sem) {
  __shared__ int s_off[kMaxBatch + 1];
  __shared__ int s_fc[kMaxBatch][5];
  // thread f fetches frame f's five counters (independent loads: one L2 round trip for the whole tick; a single thread walking the
  // frames was 40 dependent round trips)
  if (threadIdx.x < n_frames) {
    const int f = threadIdx.x;
    int* fc = B.f[f0 + f].counters;
    const int ne = fc[CNT_N_ELEV], ng = fc[CNT_N_GROUND], nc = fc[CNT_NUM_CLUSTER], nb = fc[CNT_N_BOXES], er = fc[CNT_ERROR];
    s_fc[f][0] = ne; s_fc[f][1] = ng; s_fc[f][2] = nc; s_fc[f][3] = nb; s_fc[f][4] = er;
    frame_counts[4 * f] = ne; frame_counts[4 * f + 1] = ng; frame_counts[4 * f + 2] = nc; frame_counts[4 * f + 3] = nb;
    fc[CNT_ERROR] = 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0, err = 0, ne = 0, ng = 0, nc = 0;
    for (int f = 0; f < n_frames; ++f) {
      s_off[f] = acc;
      acc += s_fc[f][3];
      if (s_fc[f][4]) err = s_fc[f][4];
      ne += s_fc[f][0]; ng += s_fc[f][1]; nc += s_fc[f][2];
    }
    s_off[n_frames] = acc;
    if (acc > max_boxes) err = LMOT_ERR_CAPACITY;
    counters[CNT_N_BOXES] = acc < max_boxes ? acc : max_boxes;
    counters[CNT_ERROR] = err;
    // what the single-frame path reports per frame, summed over the tick (the tracker copies them into the result header)
    counters[CNT_N_ELEV] = ne; counters[CNT_N_GROUND] = ng; counters[CNT_NUM_CLUSTER] = nc;
  }
  __syncthreads();
  {
    // warp w copies frame w's list (96-byte boxes: six 16-byte words each, source and destination 16-byte aligned), four words per
    // lane in flight.  (One flat loop over all floats with a per-element frame search was 40 dependent L2 round trips.)
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (w < n_frames) {
      const int off = s_off[w], cnt = min(s_off[w + 1], max_boxes) - off;
      const uint4* src = reinterpret_cast<const uint4*>(B.f[f0 + w].boxes);
      uint4* dst = reinterpret_cast<uint4*>(boxes + (size_t)off * 24);
      if (!kRig) {
        const int nw = cnt > 0 ? cnt * 6 : 0;
        for (int e0 = lane; e0 < nw; e0 += 128) {
          uint4 v[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) { const int e = e0 + 32 * u; if (e < nw) v[u] = src[e]; }
#pragma unroll
          for (int u = 0; u < 4; ++u) { const int e = e0 + 32 * u; if (e < nw) dst[e] = v[u]; }
        }
      } else {
        // a whole box per lane: its six words in flight, then its eight corners through the pose
        const float* m = R->m[f0 + w];
        for (int j = lane; j < cnt; j += 32) {
          uint4 v[6];
#pragma unroll
          for (int u = 0; u < 6; ++u) v[u] = src[6 * j + u];
          float* b = reinterpret_cast<float*>(v);
          rig_apply_box(m, b);
#pragma unroll
          for (int u = 0; u < 6; ++u) dst[6 * j + u] = v[u];
        }
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();                // frame_counts lives in pinned host memory: the host reads it after the tick's completion event
    if (det_sem) atomicAdd(det_sem, 1);
  }
}

__global__ void __launch_bounds__(256)
concat_boxes_kernel(const __grid_constant__ FitBatch B, int n_frames, int max_boxes, float* __restrict__ boxes, int* __restrict__ counters,
                    int* __restrict__ frame_counts, int* __restrict__ det_sem) {
  concat_boxes_body<false>(B, nullptr, 0, n_frames, max_boxes, boxes, counters, frame_counts, det_sem);
}

__global__ void __launch_bounds__(256)
concat_boxes_rig_kernel(const __grid_constant__ FitBatch B, const __grid_constant__ RigPoses R, int n_frames, int max_boxes, float* __restrict__ boxes,
                        int* __restrict__ counters, int* __restrict__ frame_counts, int* __restrict__ det_sem) {
  concat_boxes_body<true>(B, &R, 0, n_frames, max_boxes, boxes, counters, frame_counts, det_sem);
}

// sequence ticks with sensor tables (lmot_seq_set_sensors): CTA k concatenates sequence k's frames [f0, f0 + n_frames) into the
// sequence's own measurement list.  A sequence with a table moves each box by its sensor's pose; a sequence without one has a single
// frame, copied unchanged.  det_sem: posted after the list is complete (nullptr with global_frame: boxes_to_global_seq_kernel posts it).
struct ConcatSeq { int f0, n_frames, rig; float* boxes; int* counters; int* frame_counts; int* det_sem; };
struct ConcatSeqParams { ConcatSeq s[kMaxBatch]; };

__global__ void __launch_bounds__(256)
concat_boxes_seq_kernel(const __grid_constant__ FitBatch B, const __grid_constant__ RigPoses R, const __grid_constant__ ConcatSeqParams P,
                        int max_boxes) {
  const ConcatSeq& q = P.s[blockIdx.x];
  if (q.rig) concat_boxes_body<true>(B, &R, q.f0, q.n_frames, max_boxes, q.boxes, q.counters, q.frame_counts, q.det_sem);
  else concat_boxes_body<false>(B, nullptr, q.f0, q.n_frames, max_boxes, q.boxes, q.counters, q.frame_counts, q.det_sem);
}

}  // namespace

int boxfit_alloc_shared(Ctx* c) {
  // raw mt19937_64(0) stream (box_fitting.cpp:303 re-seeds per cluster, so every cluster sees the same draws): LMOT_MAX_RAM_POINTS
  // draws and 64 spare ones for Lemire redraws (odds n / 2^64 each).  The first 256 values are the table's earlier extent.
  constexpr int kRaw = LMOT_MAX_RAM_POINTS + 64;
  std::mt19937_64 mt(0);
  std::vector<unsigned long long> raw(kRaw);
  for (int i = 0; i < kRaw; ++i) raw[i] = mt();
  c->n_mt_raw = kRaw;
  c->max_sort_tiles = (c->max_points + kTile - 1) / kTile;
  LMOT_CUDA(c, cudaMalloc(&c->d_mt_raw, kRaw * sizeof(unsigned long long)));
  LMOT_CUDA(c, cudaMemcpy(c->d_mt_raw, raw.data(), kRaw * sizeof(unsigned long long), cudaMemcpyHostToDevice));
  // tile_hist / scatter keep one int per cluster id in dynamic shared memory (lmot_create bounds max_clusters accordingly)
  const int sh = (c->prm.max_clusters + 1) * (int)sizeof(int);
  if (sh > 48 * 1024) {
    LMOT_CUDA(c, cudaFuncSetAttribute(tile_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, sh));
    LMOT_CUDA(c, cudaFuncSetAttribute(tile_hist_area_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, sh));
    LMOT_CUDA(c, cudaFuncSetAttribute(tile_hist_layers_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, sh));
    LMOT_CUDA(c, cudaFuncSetAttribute(scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, sh));
  }
  return LMOT_OK;
}

int boxfit_alloc(Ctx* c, Slot* s) {
  const size_t np = (size_t)c->max_points;
  const int K1 = c->prm.max_clusters + 1;
  LMOT_CUDA(c, cudaMalloc(&s->d_pcid, np * sizeof(uint16_t)));
  LMOT_CUDA(c, cudaMalloc(&s->d_table, (size_t)c->max_sort_tiles * K1 * sizeof(int)));
  LMOT_CUDA(c, cudaMalloc(&s->d_seg_start, K1 * sizeof(int)));
  LMOT_CUDA(c, cudaMalloc(&s->d_seg_size, K1 * sizeof(int)));
  LMOT_CUDA(c, cudaMalloc(&s->d_sorted_pts, np * sizeof(float4)));
  LMOT_CUDA(c, cudaMalloc(&s->d_cl_box, (size_t)K1 * 24 * sizeof(float)));
  LMOT_CUDA(c, cudaMalloc(&s->d_cl_marker, (size_t)K1 * 6 * sizeof(float)));
  LMOT_CUDA(c, cudaMalloc(&s->d_cl_ok, K1));
  LMOT_CUDA(c, cudaMalloc(&s->d_boxes, (size_t)c->prm.max_boxes * 24 * sizeof(float)));
  LMOT_CUDA(c, cudaMalloc(&s->d_boxes_g, (size_t)c->prm.max_boxes * 24 * sizeof(float)));
  LMOT_CUDA(c, cudaMalloc(&s->d_markers, (size_t)c->prm.max_boxes * 6 * sizeof(float)));
  LMOT_CUDA(c, cudaMalloc(&s->d_done, 2 * sizeof(int)));                 // [0] finished box_fit CTAs, [1] finished tile_hist CTAs
  LMOT_CUDA(c, cudaMemsetAsync(s->d_done, 0, 2 * sizeof(int), s->stream));
  LMOT_CUDA(c, cudaMalloc(&s->d_det_sem, sizeof(int)));
  LMOT_CUDA(c, cudaMemsetAsync(s->d_det_sem, 0, sizeof(int), s->stream));
  return LMOT_OK;
}

void boxfit_free(Slot* s) {
  cudaFree(s->d_pcid); cudaFree(s->d_table); cudaFree(s->d_seg_start); cudaFree(s->d_seg_size); cudaFree(s->d_sorted_pts);
  cudaFree(s->d_cl_box); cudaFree(s->d_cl_marker); cudaFree(s->d_cl_ok); cudaFree(s->d_boxes); cudaFree(s->d_boxes_g); cudaFree(s->d_markers);
  cudaFree(s->d_done); cudaFree(s->d_det_sem);
  cudaFree(s->d_obs_hull);                                      // obstacle footprints (obstacles.cu), allocated on first use
}

static void rig_poses_of(const lmot_sensor* rig, int n, RigPoses& R) {
  memset(&R, 0, sizeof(R));
  for (int i = 0; i < n; ++i) memcpy(R.m[i], rig[i].pose, sizeof(R.m[i]));
}


// inputs per frame: s->d_elev / CNT_N_ELEV, s->d_cart (from clustering), s->d_label_grid / CNT_NUM_CLUSTER.
// F > 1: one frame per sensor stream; the four kernels run over the union of the frames' clusters (blockIdx.y = frame).

int boxfit_launch_batch(Ctx* c, Slot* const* slots, int F, cudaStream_t st, const int* n_upper, bool post_sem, const lmot_sensor* rig,
                        const lmot_detect_params* det, const unsigned* const* area, const int* search, const float* const* lines,
                        const LayerTab* layers) {
  if (F < 1 || F > kMaxBatch) return LMOT_ERR_INVALID;
  const int K1 = c->prm.max_clusters + 1;
  int tiles = 0;
  for (int i = 0; i < F; ++i) { const int t = (n_upper[i] + kTile - 1) / kTile; if (t > tiles) tiles = t; }
  const size_t sh = (size_t)K1 * sizeof(int);
  FitBatch B;
  for (int i = 0; i < F; ++i) { fit_frame_of(slots[i], B.f[i], post_sem); if (rig) B.f[i].sensor_height = rig[i].sensor_height; }
  for (int i = F; i < kMaxBatch; ++i) B.f[i] = B.f[0];
  Slot* s0 = slots[0];
  bool masked = false;
  FitAreaMasks A{};
  for (int i = 0; area && i < F; ++i) { A.m[i] = area[i]; masked |= area[i] != nullptr; }
  if (tiles > 0 && layers) {
    FitLayers L{};
    for (int i = 0; i < F; ++i) L.t[i] = layers[i];
    tile_hist_layers_kernel<<<dim3(tiles, F), kTile, sh, st>>>(B, c->prm.max_clusters, A, L);
  } else if (tiles > 0 && masked) tile_hist_area_kernel<<<dim3(tiles, F), kTile, sh, st>>>(B, c->prm.max_clusters, A);
  else if (tiles > 0) tile_hist_kernel<<<dim3(tiles, F), kTile, sh, st>>>(B, c->prm.max_clusters);     // + segment offsets by its last CTA per frame
  else seg_offsets_kernel<<<F, 1024, 0, st>>>(B, c->prm.max_clusters);
  kernel_mark(c, s0, st);
  // scatter and box_fit as programmatic dependents of the kernel before them (timing mode records an event between the kernels,
  // which needs the ordinary full serialisation)
  cudaLaunchAttribute pdl;
  pdl.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  pdl.val.programmaticStreamSerializationAllowed = c->timing ? 0 : 1;
  const int max_clusters = c->prm.max_clusters;
  if (tiles > 0) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(tiles, F); cfg.blockDim = dim3(kTile); cfg.dynamicSmemBytes = sh; cfg.stream = st; cfg.attrs = &pdl; cfg.numAttrs = 1;
    LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, scatter_kernel, B, max_clusters));
    kernel_mark(c, s0, st);
  }
  const BoxParams P = box_params_of(detect_params_of(c->prm));
  // one CTA per cluster: a frame rarely holds more than a few hundred clusters, F frames share the grid
  const int gx = F == 1 ? c->fit_ctas : (c->fit_ctas / 2 > 8 ? c->fit_ctas / 2 : 8);
  // box search (box_search.cu): the searching units leave this launch for box_search_launch behind it; the others keep their kernel and
  // thread count, their frames (and own values) moved to the front of B in unit order
  // ground lines: every unit of the launch runs the per-unit variants, a unit with a grid measures its clusters from it
  Slot* su[kMaxBatch];
  lmot_detect_params sd[kMaxBatch];
  int sa[kMaxBatch], fi[kMaxBatch], ns = 0, nf = F;
  const float* sg[kMaxBatch];
  for (int i = 0; i < F; ++i) fi[i] = i;
  const lmot_detect_params base = detect_params_of(c->prm);
  if (search) {
    nf = 0;
    for (int i = 0; i < F; ++i) {
      if (search[i] > 0) {
        su[ns] = slots[i]; sa[ns] = search[i]; sg[ns] = lines ? lines[i] : nullptr;
        sd[ns] = det ? det[i] : base;
        if (!det && rig) sd[ns].sensor_height = rig[i].sensor_height;
        ++ns;
      } else {
        B.f[nf] = B.f[i]; fi[nf++] = i;
      }
    }
  }
  if (nf > 0) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(gx, nf); cfg.blockDim = dim3(F == 1 ? kFitThreadsFrame : kFitThreadsBatch); cfg.dynamicSmemBytes = 0; cfg.stream = st; cfg.attrs = &pdl; cfg.numAttrs = 1;
    const unsigned long long* mt = c->d_mt_raw;
    const int n_raw = c->n_mt_raw, max_boxes = c->prm.max_boxes;
    if (lines) {
      BoxFrameParams FP;
      LinesFit LG;
      memset(&FP, 0, sizeof(FP));
      memset(&LG, 0, sizeof(LG));
      for (int i = 0; i < nf; ++i) {
        lmot_detect_params d = det ? det[fi[i]] : base;
        if (!det && rig) d.sensor_height = rig[fi[i]].sensor_height;
        FP.p[i] = box_params_of(d);
        lines_fit_of(d, lines[fi[i]], LG, i);
      }
      if (F == 1) LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, box_fit_lines_kernel<kFitThreadsFrame>, B, FP, LG, mt, n_raw, max_clusters, max_boxes));
      else LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, box_fit_lines_kernel<kFitThreadsBatch>, B, FP, LG, mt, n_raw, max_clusters, max_boxes));
    } else if (det) {
      BoxFrameParams FP;
      memset(&FP, 0, sizeof(FP));
      for (int i = 0; i < nf; ++i) FP.p[i] = box_params_of(det[fi[i]]);
      if (F == 1) LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, box_fit_frame_kernel<kFitThreadsFrame>, B, FP, mt, n_raw, max_clusters, max_boxes));
      else LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, box_fit_frame_kernel<kFitThreadsBatch>, B, FP, mt, n_raw, max_clusters, max_boxes));
    } else if (rig) {
      if (F == 1) LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, box_fit_kernel<kFitThreadsFrame, true>, B, P, mt, n_raw, max_clusters, max_boxes));
      else LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, box_fit_kernel<kFitThreadsBatch, true>, B, P, mt, n_raw, max_clusters, max_boxes));
    } else {
      if (F == 1) LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, box_fit_kernel<kFitThreadsFrame, false>, B, P, mt, n_raw, max_clusters, max_boxes));
      else LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, box_fit_kernel<kFitThreadsBatch, false>, B, P, mt, n_raw, max_clusters, max_boxes));
    }
  }
  if (ns > 0) {
    int rc = box_search_launch(c, su, ns, sd, sa, st, post_sem, gx, !c->timing, lines ? sg : nullptr);
    if (rc) return rc;
  }
  kernel_mark(c, s0, st);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

// the frames' box lists concatenated in stream order -> d_boxes / counters of the batch (the tracker's measurement list)
// rig: frame i's boxes moved by sensor i's pose (vehicle frame)
int boxes_concat_launch(Ctx* c, Slot* const* slots, int F, cudaStream_t st, float* d_boxes, int* d_counters, int* d_frame_counts, int* det_sem,
                        const lmot_sensor* rig) {
  FitBatch B;
  for (int i = 0; i < F; ++i) fit_frame_of(slots[i], B.f[i], false);
  for (int i = F; i < kMaxBatch; ++i) B.f[i] = B.f[0];
  if (rig) {
    RigPoses R;
    rig_poses_of(rig, F, R);
    concat_boxes_rig_kernel<<<1, 256, 0, st>>>(B, R, F, c->prm.max_boxes, d_boxes, d_counters, d_frame_counts, det_sem);
  } else {
    concat_boxes_kernel<<<1, 256, 0, st>>>(B, F, c->prm.max_boxes, d_boxes, d_counters, d_frame_counts, det_sem);
  }
  kernel_mark(c, slots[0], st);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

// sequence ticks with sensor tables: sequence k's frames [f0[k], f0[k + 1]) of `slots` -> m[k]'s list and counters, per-frame counts into
// frame_counts[k] (device view of the tick's pinned block k).  rig: one entry per frame of the tick; sequence k's poses apply iff rig_on[k].
int boxes_concat_seq_launch(Ctx* c, Slot* const* slots, int S, const int* f0, const bool* rig_on, const lmot_sensor* rig, const SeqMeas* m,
                            int* const* frame_counts, bool post_sem, cudaStream_t st) {
  const int F = f0[S];
  if (S < 1 || F > kMaxBatch) return LMOT_ERR_INVALID;
  FitBatch B;
  for (int i = 0; i < F; ++i) fit_frame_of(slots[i], B.f[i], false);
  for (int i = F; i < kMaxBatch; ++i) B.f[i] = B.f[0];
  RigPoses R;
  rig_poses_of(rig, F, R);
  ConcatSeqParams P{};
  for (int k = 0; k < S; ++k)
    P.s[k] = ConcatSeq{f0[k], f0[k + 1] - f0[k], rig_on[k] ? 1 : 0, m[k].d_boxes, m[k].d_counters, frame_counts[k], post_sem ? m[k].d_det_sem : nullptr};
  concat_boxes_seq_kernel<<<S, 256, 0, st>>>(B, R, P, c->prm.max_boxes);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

// device box lists [f0, f0 + n_lists) of `src` (src.list(i): list i's boxes, src.count(i): its length clamped to its capacity) -> one
// contiguous list + the counter block the tracker reads (multi-GPU hand-over: the lists arrived by ncclAllGather; sequence ticks: one
// sequence's lists).  kRig: list f0 + l's boxes moved by pose R->m[f0 + l].  Optional outputs of sequence ticks: frame_counts row l =
// (0, 0, 0, list f0 + l's clamped length), det_sem posted once the list is complete.
// padded lists (one buffer, `cap` boxes per list)
struct PaddedLists {
  const float* lists; const int* counts; int cap;
  __device__ const float* list(int i) const { return lists + (size_t)i * cap * 24; }
  __device__ int count(int i) const { return min(max(counts[i], 0), cap); }
};
// a pointer and a length pointer per list (SeqLists in the parameter block)
struct PtrLists {
  const SeqLists* L;
  __device__ const float* list(int i) const { return L->lists[i]; }
  __device__ int count(int i) const { return min(max(*L->counts[i], 0), L->cap[i]); }
};

template <bool kRig, class Src>
__device__ __forceinline__ void pack_lists_body(const RigPoses* R, const Src& src, int f0, int n_lists, int max_boxes, float* __restrict__ boxes,
                                                int* __restrict__ counters, int* __restrict__ frame_counts = nullptr, int* __restrict__ det_sem = nullptr) {
  __shared__ int s_off[kMaxBatch + 1];
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int l = 0; l < n_lists; ++l) {
      s_off[l] = acc;
      const int n = src.count(f0 + l);
      acc += n;
      if (frame_counts) { frame_counts[4 * l] = 0; frame_counts[4 * l + 1] = 0; frame_counts[4 * l + 2] = 0; frame_counts[4 * l + 3] = n; }
    }
    s_off[n_lists] = acc;
    counters[CNT_N_BOXES] = acc < max_boxes ? acc : max_boxes;
    counters[CNT_ERROR] = acc > max_boxes ? (int)LMOT_ERR_CAPACITY : 0;
    counters[CNT_N_ELEV] = 0; counters[CNT_N_GROUND] = 0; counters[CNT_NUM_CLUSTER] = 0;
  }
  __syncthreads();
  for (int l = 0; l < n_lists; ++l) {
    const int off = s_off[l], cnt = min(s_off[l + 1], max_boxes) - off;
    const float* lst = src.list(f0 + l);
    if (!kRig) {
      for (int e = threadIdx.x; e < cnt * 24; e += 256) boxes[(size_t)off * 24 + e] = lst[e];
    } else {
      // a whole box per thread: its 24 floats in flight (the caller's lists need only 4-byte alignment), then the pose
      const float* m = R->m[f0 + l];
      for (int j = threadIdx.x; j < cnt; j += 256) {
        float b[24];
#pragma unroll
        for (int u = 0; u < 24; ++u) b[u] = lst[(size_t)j * 24 + u];
        rig_apply_box(m, b);
        float4* d = reinterpret_cast<float4*>(boxes + (size_t)(off + j) * 24);
#pragma unroll
        for (int u = 0; u < 6; ++u) d[u] = make_float4(b[4 * u], b[4 * u + 1], b[4 * u + 2], b[4 * u + 3]);
      }
    }
  }
  if (frame_counts || det_sem) {
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence_system();              // frame_counts lives in pinned host memory: the host reads it after the tick's completion event
      if (det_sem) atomicAdd(det_sem, 1);
    }
  }
}

__global__ void __launch_bounds__(256)
pack_lists_kernel(const float* __restrict__ lists, const int* __restrict__ counts, int n_lists, int cap, int max_boxes, float* __restrict__ boxes,
                  int* __restrict__ counters) {
  pack_lists_body<false>(nullptr, PaddedLists{lists, counts, cap}, 0, n_lists, max_boxes, boxes, counters);
}

__global__ void __launch_bounds__(256)
pack_lists_rig_kernel(const __grid_constant__ RigPoses R, const float* __restrict__ lists, const int* __restrict__ counts, int n_lists, int cap,
                      int max_boxes, float* __restrict__ boxes, int* __restrict__ counters) {
  pack_lists_body<true>(&R, PaddedLists{lists, counts, cap}, 0, n_lists, max_boxes, boxes, counters);
}

// LISTS entries of sequence ticks: CTA k packs position k's lists [f0, f0 + n_lists) of P.L into that sequence's own measurement list.  A
// sequence with a table moves each box by its sensor's pose; a sequence without one has a single list, copied unchanged.
// det_sem: posted after the list is complete (nullptr with global_frame: boxes_to_global_seq_kernel posts it).
struct PackSeq { int f0, n_lists, rig; float* boxes; int* counters; int* frame_counts; int* det_sem; };
struct PackSeqParams { PackSeq s[kMaxBatch]; SeqLists L; };

__global__ void __launch_bounds__(256)
pack_lists_seq_kernel(const __grid_constant__ RigPoses R, const __grid_constant__ PackSeqParams P, int max_boxes) {
  const PackSeq& q = P.s[blockIdx.x];
  const PtrLists src{&P.L};
  if (q.rig) pack_lists_body<true>(&R, src, q.f0, q.n_lists, max_boxes, q.boxes, q.counters, q.frame_counts, q.det_sem);
  else pack_lists_body<false>(nullptr, src, q.f0, q.n_lists, max_boxes, q.boxes, q.counters, q.frame_counts, q.det_sem);
}

int boxes_pack_lists_launch(Ctx* c, cudaStream_t st, const float* d_lists, const int* d_counts, int n_lists, int cap, float* d_boxes, int* d_counters,
                            const lmot_sensor* rig) {
  if (rig) {
    RigPoses R;
    rig_poses_of(rig, n_lists, R);
    pack_lists_rig_kernel<<<1, 256, 0, st>>>(R, d_lists, d_counts, n_lists, cap, c->prm.max_boxes, d_boxes, d_counters);
  } else {
    pack_lists_kernel<<<1, 256, 0, st>>>(d_lists, d_counts, n_lists, cap, c->prm.max_boxes, d_boxes, d_counters);
  }
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

// LISTS entries of sequence ticks: position k's lists [f0[k], f0[k + 1]) of L -> m[k]'s list and counters, per-list counts into
// frame_counts[k] (device view of that sequence's pinned result block).  rig: one entry per list; position k's poses apply iff rig_on[k].
int boxes_pack_lists_seq_launch(Ctx* c, cudaStream_t st, const SeqLists& L, int S, const int* f0, const bool* rig_on, const lmot_sensor* rig,
                                const SeqMeas* m, int* const* frame_counts, bool post_sem) {
  const int F = f0[S];
  if (S < 1 || F > kMaxBatch) return LMOT_ERR_INVALID;
  RigPoses R;
  rig_poses_of(rig, F, R);
  PackSeqParams P{};
  for (int k = 0; k < S; ++k)
    P.s[k] = PackSeq{f0[k], f0[k + 1] - f0[k], rig_on[k] ? 1 : 0, m[k].d_boxes, m[k].d_counters, frame_counts[k], post_sem ? m[k].d_det_sem : nullptr};
  P.L = L;
  pack_lists_seq_kernel<<<S, 256, 0, st>>>(R, P, c->prm.max_boxes);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

int boxfit_launch(Ctx* c, Slot* s, cudaStream_t st, int n_upper, bool post_sem, const unsigned* area, int search, const float* lines,
                  const LayerTab* layers) {
  Slot* sl[1] = {s};
  const int nu[1] = {n_upper};
  const unsigned* am[1] = {area};
  return boxfit_launch_batch(c, sl, 1, st, nu, post_sem, nullptr, nullptr, area ? am : nullptr, search > 0 ? &search : nullptr,
                             lines ? &lines : nullptr, layers);
}

}  // namespace lmot
