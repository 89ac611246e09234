// cluster.cu -- 2-D occupancy-grid connected-component clustering on sm_90a.
//
// Replaces componentClustering (/root/reference/object_tracking/src/cluster/component_clustering.cpp:260-268):
//   mapCartesianGrid (:28-225)  count points per 0.2 m cell of the 250x250 grid over +-25 m; every cell holding
//                               MORE THAN ONE point and its (clipped) 3x3 neighbourhood becomes occupied (-1)
//   findComponent/search (:228-257)  raster scan (x outer, y inner); each unlabelled occupied cell starts
//                               id = ++numCluster and a recursive 8-connected flood fill
//
// Design: the grid is 250 rows of 250 BITS (8 words per row, 8 KB in all), not 62,500 counters.
//   * "count > 1" needs no counter: two bit planes, `once` and `twice`.  A point sets its cell's bit in `once`; if it
//     was set already (or two points of one warp share the cell) it sets the bit in `twice`.  seed == twice.
//     (cart_mark(), called by ground_fused_kernel for every elevated point while it is still in registers, or by
//     cart_mark_kernel for the stand-alone entry point.)
//   * ccl_dense_kernel (ccl_device.cuh: the body is a device function, also called from the ground kernel's tail on the fused frame
//     path), ONE CTA per frame, everything in shared memory:
//       dilate3x3 on words  ->  "pieces" (maximal runs of 1-bits inside a word)  ->  a block-wide scan numbers the pieces in raster
//       order (dense ids; the smallest id of a component is its first piece in raster order)  ->  first parent = the smallest piece
//       a piece touches (plain stores: a forest, ids decrease upwards)  ->  pointer-jumping flatten  ->  the remaining adjacencies
//       (a piece touching several pieces above, or one above and one to the left) as union-find unions from a pair list  ->
//       flatten again  ->  id = 1 + rank of the root among the roots in id order.  The recursive fill labels components in the
//       order the raster scan first meets them, i.e. by their smallest linear index == smallest piece id: identical ids.
//       The 250x250 int label grid (the reference's only carrier of labels) is updated SPARSELY: cells occupied in the
//       previous frame are cleared, cells occupied now get their id (stores only where something is or was).
#include <climits>
#include "lmot_internal.cuh"
#include "exact_math.cuh"
#include "ccl_device.cuh"

namespace lmot {

namespace {

__global__ void __launch_bounds__(256)
cart_mark_kernel(const float4* __restrict__ elev, const int* __restrict__ counters, float roi, uint16_t* __restrict__ cart,
                 unsigned* __restrict__ once, unsigned* __restrict__ twice) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = counters[CNT_N_ELEV];
  if (blockIdx.x * blockDim.x >= n) return;      // whole block past the end (launch is sized for the input cloud)
  unsigned c = kNoCell;
  if (i < n) {
    const float4 q = __ldg(&elev[i]);
    c = cart_cell_of(q.x, q.y, roi, kNumGrid);
    cart[i] = (uint16_t)c;
  }
  cart_mark(c, once, twice);
}

__global__ void __launch_bounds__(256)
cart_cells_kernel(const float4* __restrict__ elev, const int* __restrict__ counters, float roi, uint16_t* __restrict__ cart) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < counters[CNT_N_ELEV]) { const float4 q = __ldg(&elev[i]); cart[i] = (uint16_t)cart_cell_of(q.x, q.y, roi, kNumGrid); }
}

__global__ void __launch_bounds__(kCclThreads, 1)
ccl_dense_kernel(const __grid_constant__ CclBatch B) {
  extern __shared__ __align__(16) unsigned char ccl_smem[];
  ccl_dense_body(B.f[blockIdx.x], ccl_smem);
}

// detection areas: frame blockIdx.x's seeds masked by its unit's cell mask (A.m[i], nullptr: an unmasked unit of the same launch)
struct AreaMasks { const unsigned* m[kMaxBatch]; };

__global__ void __launch_bounds__(kCclThreads, 1)
ccl_area_kernel(const __grid_constant__ CclBatch B, const __grid_constant__ AreaMasks A) {
  extern __shared__ __align__(16) unsigned char ccl_smem[];
  ccl_dense_body<true>(B.f[blockIdx.x], ccl_smem, A.m[blockIdx.x]);
}

// ---- the cluster node's side outputs (src/cluster/main.cpp:62-99), SURVEY.md §8(f)3 ------------------------------
//   makeClusteredCloud (component_clustering.cpp:308-335): every elevated point inside the ROI whose cell carries a label
//       becomes the CENTRE of its cell at z = -1, in cloud order
//   setObsMsg (:337-375): the same, but the function zeroes the cell in its by-value grid copy once it has emitted it, so
//       only the FIRST point (cloud order) of every labelled cell yields an obstacle, tagged with the cluster id
//   createCostMap (:425-454): 50 x 50 cells of 1 m, 15 per point (capped at 100) for points with z <= 0.1 outside the car's
//       4.5 x 2 m footprint; indices by double arithmetic and truncation toward zero exactly as written
// One CTA; two order-preserving compactions (ballot + carried offset per 1024-point tile).
constexpr int kCostW = 50, kCostH = 50;

// kArea: the points of cells outside the detection area's mask `area` are not part of the cloud (E_area): they are skipped
template <bool kArea>
__device__ __forceinline__ void cluster_outputs_body(const float4* __restrict__ elev, const uint16_t* __restrict__ cart, const int* __restrict__ counters,
                                                     const int* __restrict__ label_grid, float roi, int* __restrict__ first_idx,
                                                     float4* __restrict__ clustered, float4* __restrict__ obstacles, int* __restrict__ cost_map,
                                                     int* __restrict__ out_counts, const unsigned* __restrict__ area) {
  __shared__ int s_cost[kCostW * kCostH];
  __shared__ int s_warp[32], s_warp2[32];
  __shared__ int s_carry, s_carry2;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = counters[CNT_N_ELEV];
  const float grid_size = 0.2f;                                   // component_clustering.h:15
  for (int k = tid; k < kCostW * kCostH; k += 1024) s_cost[k] = 0;
  if (tid == 0) { s_carry = 0; s_carry2 = 0; }
  __syncthreads();
  // pass 1: first point of every labelled cell; cost map counts
  const double res = 1.0, cx = (kCostW / 2.0) * res - 0.0, cy = (kCostH / 2.0) * res - 25.0;   // g_resolution, g_offset_x/y (:15-20)
  for (int i = tid; i < n; i += 1024) {
    const unsigned cc = cart[i];
    if (kArea && !area_kept(area, cc)) continue;
    if (cc != kNoCell && label_grid[cc] != 0) atomicMin(&first_idx[cc], i);
    const float4 q = __ldg(&elev[i]);
    if (!((double)q.z > 0.1) && !(fabs((double)q.x) < 4.5 && fabs((double)q.y) < 2.0)) {
      const int gy = (int)(((double)q.x + cx) / res), gx = (int)(((double)q.y + cy) / res);
      if (!(gy < 0 || gy >= kCostW || gx < 0 || gx >= kCostH)) atomicAdd(&s_cost[kCostW * gx + gy], 1);
    }
  }
  __syncthreads();
  for (int k = tid; k < kCostW * kCostH; k += 1024) cost_map[k] = min(100, 15 * s_cost[k]);
  // pass 2: the two clouds, in cloud order
  for (int i0 = 0; i0 < n; i0 += 1024) {
    const int i = i0 + tid;
    int lab = 0, obs = 0;
    unsigned cc = kNoCell;
    if (i < n) {
      cc = cart[i];
      if (cc != kNoCell && (!kArea || area_kept(area, cc))) { lab = label_grid[cc]; obs = (lab != 0 && first_idx[cc] == i) ? 1 : 0; }
    }
    const unsigned bl = __ballot_sync(0xFFFFFFFFu, lab != 0), bo = __ballot_sync(0xFFFFFFFFu, obs);
    if (lane == 0) { s_warp[warp] = __popc(bl); s_warp2[warp] = __popc(bo); }
    __syncthreads();
    int wb = 0, tot = 0, wb2 = 0, tot2 = 0;
    for (int w = 0; w < 32; ++w) { if (w < warp) { wb += s_warp[w]; wb2 += s_warp2[w]; } tot += s_warp[w]; tot2 += s_warp2[w]; }
    if (lab != 0) {
      const int xI = (int)(cc / (unsigned)kNumGrid), yI = (int)(cc % (unsigned)kNumGrid);
      const float half = fdiv(roi, 2.f), hg = fdiv(grid_size, 2.f);
      const float ox = fadd(fsub(fmul(grid_size, (float)xI), half), hg), oy = fadd(fsub(fmul(grid_size, (float)yI), half), hg);
      clustered[s_carry + wb + __popc(bl & ((1u << lane) - 1u))] = make_float4(ox, oy, -1.f, 1.f);
      if (obs) {
        obstacles[s_carry2 + wb2 + __popc(bo & ((1u << lane) - 1u))] = make_float4(ox, oy, -1.f, (float)lab);
        first_idx[cc] = INT_MAX;                                   // scratch back to its rest state
      }
    }
    __syncthreads();
    if (tid == 0) { s_carry += tot; s_carry2 += tot2; }
    __syncthreads();
  }
  if (tid == 0) { out_counts[0] = s_carry; out_counts[1] = s_carry2; }
}

__global__ void __launch_bounds__(1024)
cluster_outputs_kernel(const float4* __restrict__ elev, const uint16_t* __restrict__ cart, const int* __restrict__ counters,
                       const int* __restrict__ label_grid, float roi, int* __restrict__ first_idx, float4* __restrict__ clustered,
                       float4* __restrict__ obstacles, int* __restrict__ cost_map, int* __restrict__ out_counts) {
  cluster_outputs_body<false>(elev, cart, counters, label_grid, roi, first_idx, clustered, obstacles, cost_map, out_counts, nullptr);
}

__global__ void __launch_bounds__(1024)
cluster_outputs_area_kernel(const float4* __restrict__ elev, const uint16_t* __restrict__ cart, const int* __restrict__ counters,
                            const int* __restrict__ label_grid, float roi, int* __restrict__ first_idx, float4* __restrict__ clustered,
                            float4* __restrict__ obstacles, int* __restrict__ cost_map, int* __restrict__ out_counts,
                            const unsigned* __restrict__ area) {
  cluster_outputs_body<true>(elev, cart, counters, label_grid, roi, first_idx, clustered, obstacles, cost_map, out_counts, area);
}

__global__ void fill_i32_kernel(int* p, int n, int v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

__global__ void zero_u32_kernel(unsigned* p, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = 0u;
}

}  // namespace

int cluster_alloc(Ctx* c, Slot* s) {
  const size_t np = (size_t)c->max_points;
  LMOT_CUDA(c, cudaMalloc(&s->d_cart, np * sizeof(uint16_t)));
  LMOT_CUDA(c, cudaMalloc(&s->d_cart_bits, 3 * kBitWords * sizeof(unsigned)));      // once | twice | occupancy of the previous frame
  LMOT_CUDA(c, cudaMalloc(&s->d_label_grid, kCartCells * sizeof(int)));
  LMOT_CUDA(c, cudaMemsetAsync(s->d_cart_bits, 0, 3 * kBitWords * sizeof(unsigned), s->stream));
  LMOT_CUDA(c, cudaMemsetAsync(s->d_label_grid, 0, kCartCells * sizeof(int), s->stream));
  s->label_grid_foreign = false;
  LMOT_CUDA(c, cudaFuncSetAttribute(ccl_dense_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDenseSmem));
  LMOT_CUDA(c, cudaFuncSetAttribute(ccl_area_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDenseSmem));
  return LMOT_OK;
}

void cluster_free(Slot* s) {
  cudaFree(s->d_cart); cudaFree(s->d_cart_bits); cudaFree(s->d_label_grid);
  cudaFree(s->d_first_idx); cudaFree(s->d_clustered); cudaFree(s->d_obstacles); cudaFree(s->d_cost_map);
  cudaFree(s->d_slice); cudaFree(s->d_colmask); cudaFree(s->d_layer_cols); cudaFree(s->d_layer_base); cudaFree(s->d_layer_lab);
}

// elevated cloud = s->d_elev with its length in d_counters[CNT_N_ELEV]; n_upper bounds that length on the host
int cluster_launch(Ctx* c, Slot* s, cudaStream_t st, int n_upper, bool counted, const unsigned* area) {
  unsigned* once = s->d_cart_bits, *twice = once + kBitWords;
  if (n_upper > 0 && !counted) {   // `counted`: ground_fused_kernel already marked the elevated points (fused frame path)
    cart_mark_kernel<<<(n_upper + 255) / 256, 256, 0, st>>>(s->d_elev, s->d_counters, c->prm.roi_m, s->d_cart, once, twice);
    kernel_mark(c, s, st);
  }
  Slot* sl[1] = {s};
  const unsigned* am[1] = {area};
  return ccl_launch_batch(c, sl, 1, st, area ? am : nullptr);
}

// connected components of F frames in one launch, one CTA per frame (the bit planes were marked by the ground kernel)
int ccl_launch_batch(Ctx* c, Slot* const* slots, int F, cudaStream_t st, const unsigned* const* area) {
  if (F < 1 || F > kMaxBatch) return LMOT_ERR_INVALID;
  CclBatch B;
  for (int i = 0; i < F; ++i) {
    Slot* s = slots[i];
    if (s->label_grid_foreign) {   // the caller uploaded its own label grid (lmot_box_fit): the sparse update needs a clean slate
      LMOT_CUDA(c, cudaMemsetAsync(s->d_label_grid, 0, kCartCells * sizeof(int), st));
      LMOT_CUDA(c, cudaMemsetAsync(s->d_cart_bits + 2 * kBitWords, 0, kBitWords * sizeof(unsigned), st));
      s->label_grid_foreign = false;
    }
    B.f[i].once = s->d_cart_bits; B.f[i].twice = s->d_cart_bits + kBitWords; B.f[i].prev_occ = s->d_cart_bits + 2 * kBitWords;
    B.f[i].out = s->d_label_grid; B.f[i].counters = s->d_counters;
  }
  for (int i = F; i < kMaxBatch; ++i) B.f[i] = B.f[0];
  bool masked = false;
  AreaMasks A{};
  for (int i = 0; area && i < F; ++i) { A.m[i] = area[i]; masked |= area[i] != nullptr; }
  if (masked) ccl_area_kernel<<<F, kCclThreads, kDenseSmem, st>>>(B, A);
  else ccl_dense_kernel<<<F, kCclThreads, kDenseSmem, st>>>(B);
  kernel_mark(c, slots[0], st);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

// side outputs of the cluster node for the slot's current elevated cloud + label grid; buffers are allocated on first use
int cluster_outputs_launch(Ctx* c, Slot* s, cudaStream_t st) {
  if (!s->d_first_idx) {
    LMOT_CUDA(c, cudaMalloc(&s->d_first_idx, kCartCells * sizeof(int)));
    LMOT_CUDA(c, cudaMalloc(&s->d_clustered, (size_t)c->max_points * sizeof(float4)));
    LMOT_CUDA(c, cudaMalloc(&s->d_obstacles, (size_t)kCartCells * sizeof(float4)));
    LMOT_CUDA(c, cudaMalloc(&s->d_cost_map, (kCostW * kCostH + 2) * sizeof(int)));
    fill_i32_kernel<<<(kCartCells + 255) / 256, 256, 0, st>>>(s->d_first_idx, kCartCells, INT_MAX);
  }
  if (s->area_last)
    cluster_outputs_area_kernel<<<1, 1024, 0, st>>>(s->d_elev, s->d_cart, s->d_counters, s->d_label_grid, c->prm.roi_m, s->d_first_idx,
                                                    s->d_clustered, s->d_obstacles, s->d_cost_map, s->d_cost_map + kCostW * kCostH,
                                                    s->d_area_mask);
  else
    cluster_outputs_kernel<<<1, 1024, 0, st>>>(s->d_elev, s->d_cart, s->d_counters, s->d_label_grid, c->prm.roi_m, s->d_first_idx,
                                               s->d_clustered, s->d_obstacles, s->d_cost_map, s->d_cost_map + kCostW * kCostH);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

int cluster_cells_only(Ctx* c, Slot* s, cudaStream_t st, int n_upper) {
  if (n_upper > 0)
    cart_cells_kernel<<<(n_upper + 255) / 256, 256, 0, st>>>(s->d_elev, s->d_counters, c->prm.roi_m, s->d_cart);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

}  // namespace lmot
