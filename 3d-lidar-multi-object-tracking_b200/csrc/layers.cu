// layers.cu -- layered clustering (lmot_set_layers): connected components over (x, y, height slice) on sm_90a.
//
// The definition is in include/lmot.h.  A unit's voxels are 62,500 columns of S <= 32 slices, one uint32 mask per column:
//   layer_mark_kernel  one launch for every layered unit of a submission: each point of E (its column is the cell clustering already
//                      keeps in d_cart) gets its slice byte, and ORs the slice bit into its column's mask (d_colmask, zero at rest)
//   ccl_layer_kernel   one CTA per unit, on global (L2-resident) arrays -- 62,500 column words do not fit in shared memory:
//     A  seeds: the `twice` bit plane AND the detection area, exactly ccl_area_kernel's; the once / twice planes are re-armed
//     B  the 2-D occupancy (seeds dilated 3x3) picks the columns that can hold a voxel
//     C  D(x, y) = the seed column masks of the 3x3 neighbourhood ORed, dilated vertically by g, clipped to S bits
//     D  nodes = the bit runs of D, dense ids by a block-wide scan in (x, y, bottom) order -- the smallest id of a component is its
//        smallest voxel in (x, y, s) order
//     E  union-find (root = smallest id, ccl_device.cuh) over every pair of touching runs of a column and its four earlier neighbour
//        columns; runs of one column never touch (maximal runs are one empty slice apart at least)
//     F  flatten, G  rank the roots (cluster ids, CNT_NUM_CLUSTER), H  every run gets -(its cluster id), I  column masks back to zero
//   The 2-D label grid and the previous-occupancy plane are left alone, so an unlayered frame on the slot later still updates the grid
//   sparsely and exactly.  Box fitting reads the run tables (boxfit.cu tile_hist_layers_kernel).
// With S = 1 every column is one run and the labelling is ccl_dense_kernel's: componentClustering.
#include <cmath>
#include <vector>
#include "lmot_internal.cuh"
#include "ccl_device.cuh"

namespace lmot {

namespace {

constexpr int kMaxRuns = 16;                       // runs of one 32-bit column mask
constexpr int kLayerNodes = kCartCells * kMaxRuns;  // 1,000,000

struct LayerMarkJob {
  const float4* elev; const uint16_t* cart; const int* counters; const unsigned* area;
  uint8_t* slice; unsigned* colmask;
  double sensor_height, z_min, slice_m;
  int S;
};
struct LayerMarkBatch { LayerMarkJob j[kMaxBatch]; };

struct LayerCclJob {
  unsigned* once; unsigned* twice; const unsigned* area; unsigned* colmask;
  unsigned* cols; int* base; int* lab; int* counters;
  int S, g;
};
struct LayerCclBatch { LayerCclJob j[kMaxBatch]; };

// steps 1-2 for unit blockIdx.y: the slice of every point with a column (in the area), and its column's mask
__global__ void __launch_bounds__(256)
layer_mark_kernel(const __grid_constant__ LayerMarkBatch B) {
  const LayerMarkJob& J = B.j[blockIdx.y];
  const int n = J.counters[CNT_N_ELEV];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned c = J.cart[i];
    uint8_t sl = 0xFF;
    if (c != kNoCell && (!J.area || area_kept(J.area, c))) {
      const double h = __dsub_rn(__dadd_rn((double)J.elev[i].z, J.sensor_height), J.z_min);
      const double q = floor(__ddiv_rn(h, J.slice_m));
      const int s = !(q >= 0.0) ? 0 : (q > (double)(J.S - 1) ? J.S - 1 : (int)q);
      sl = (uint8_t)s;
      atomicOr(&J.colmask[c], 1u << s);
    }
    J.slice[i] = sl;
  }
}

// exclusive block-wide scan of one int per thread (s_warp: 33 ints); returns the thread's offset, *total the sum
__device__ __forceinline__ int block_scan(int v, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= o) incl += t; }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    const int w = s_warp[lane];
    int wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, wi, o); if (lane >= o) wi += t; }
    s_warp[lane] = wi - w;
    if (lane == 31) s_warp[32] = wi;
  }
  __syncthreads();
  const int r = s_warp[warp] + incl - v;
  *total = s_warp[32];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(kCclThreads, 1)
ccl_layer_kernel(const __grid_constant__ LayerCclBatch B) {
  __shared__ unsigned s_seed[kBitWords];
  __shared__ unsigned s_any[kBitWords];
  __shared__ int s_warp[33];
  const LayerCclJob& J = B.j[blockIdx.x];
  const int tid = threadIdx.x;
  const int w0 = 2 * tid;
  const bool own = tid < kBitWords / 2;
  unsigned* __restrict__ cols = J.cols;
  int* __restrict__ base = J.base;
  volatile int* L = J.lab;
  // A: seeds, and every column a point may have marked; the bit planes are re-armed for the next frame
  if (own) {
    uint2 tw = __ldcg(reinterpret_cast<const uint2*>(J.twice) + tid);
    const uint2 on = __ldcg(reinterpret_cast<const uint2*>(J.once) + tid);
    s_any[w0] = on.x | tw.x; s_any[w0 + 1] = on.y | tw.y;
    if (J.area) { const uint2 am = __ldg(reinterpret_cast<const uint2*>(J.area) + tid); tw.x &= am.x; tw.y &= am.y; }
    s_seed[w0] = tw.x; s_seed[w0 + 1] = tw.y;
    reinterpret_cast<uint2*>(J.once)[tid] = make_uint2(0u, 0u);
    reinterpret_cast<uint2*>(J.twice)[tid] = make_uint2(0u, 0u);
  }
  __syncthreads();
  // B + C: the columns of the 2-D occupancy get D, every other column 0; runs per thread
  const unsigned smask = J.S >= 32 ? 0xFFFFFFFFu : ((1u << J.S) - 1u);
  unsigned occ[2] = {0u, 0u};
  int runs = 0;
  if (own) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int w = w0 + h, x = w >> 3, k = w & 7;
      unsigned o = hdil(s_seed + x * kRowWords, k);
      if (x > 0) o |= hdil(s_seed + (x - 1) * kRowWords, k);
      if (x < kNumGrid - 1) o |= hdil(s_seed + (x + 1) * kRowWords, k);
      if (k == kRowWords - 1) o &= kLastWordMask;
      occ[h] = o;
      for (int b = 0; b < 32 && 32 * k + b < kNumGrid; ++b) {
        const int y = 32 * k + b;
        unsigned d = 0u;
        if ((o >> b) & 1u) {
          for (int xx = max(x - 1, 0); xx <= min(x + 1, kNumGrid - 1); ++xx)
            for (int yy = max(y - 1, 0); yy <= min(y + 1, kNumGrid - 1); ++yy)
              if ((s_seed[xx * kRowWords + (yy >> 5)] >> (yy & 31)) & 1u) d |= __ldcg(&J.colmask[xx * kNumGrid + yy]);
          unsigned v = d;
          for (int e = 1; e <= J.g; ++e) v |= (d << e) | (d >> e);
          d = v & smask;
          runs += __popc(piece_starts(d));
        }
        cols[x * kNumGrid + y] = d;
      }
    }
  }
  // D: dense ids in (x, y, bottom) order; every run starts as its own root
  int P;
  int id = block_scan(runs, s_warp, &P);
  if (own) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int w = w0 + h, x = w >> 3, k = w & 7;
      unsigned o = occ[h];
      while (o) {
        const int b = __ffs(o) - 1;
        o &= o - 1u;
        const int col = x * kNumGrid + 32 * k + b;
        const int r = __popc(piece_starts(cols[col]));
        base[col] = id;
        for (int j = 0; j < r; ++j) L[id + j] = id + j;
        id += r;
      }
    }
  }
  if (tid == 0) base[kCartCells] = P;
  __syncthreads();
  // E: every run with the touching runs of the columns (x-1, y-1), (x-1, y), (x-1, y+1), (x, y-1)
  if (own) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int w = w0 + h, x = w >> 3, k = w & 7;
      unsigned o = occ[h];
      while (o) {
        const int b = __ffs(o) - 1;
        o &= o - 1u;
        const int y = 32 * k + b, col = x * kNumGrid + y;
        const unsigned m = cols[col];
        const int mybase = base[col];
        const int nb[4][2] = {{x - 1, y - 1}, {x - 1, y}, {x - 1, y + 1}, {x, y - 1}};
        for (int q = 0; q < 4; ++q) {
          const int nx = nb[q][0], ny = nb[q][1];
          if (nx < 0 || ny < 0 || ny >= kNumGrid) continue;
          const unsigned dn = cols[nx * kNumGrid + ny];
          if (!dn) continue;
          const int bn = base[nx * kNumGrid + ny];
          unsigned rest = m;
          int me = mybase;
          while (rest) {
            const int a = __ffs(rest) - 1;
            const unsigned t = ~(rest >> a);
            const int len = t ? __ffs(t) - 1 : 32;
            const unsigned pm = (len >= 32 ? 0xFFFFFFFFu : ((1u << len) - 1u)) << a;
            rest &= ~pm;
            unsigned touched = dn & (pm | (pm << 1) | (pm >> 1));
            while (touched) {
              const int p = 31 - __clz(touched);
              uf_union(L, J.lab, me, bn + piece_of(dn, p));
              const unsigned startbit = piece_starts(dn) & ((2u << p) - 1u);
              touched &= (1u << (31 - __clz(startbit))) - 1u;
            }
            ++me;
          }
        }
      }
    }
  }
  __syncthreads();
  // F: flatten (every run points at its root)
  for (int i = tid; i < P; i += kCclThreads) uf_compress(L, i);
  __syncthreads();
  // G: cluster id = 1 + rank of the root among the roots in id order; thread t ranks the ids [t*c, (t+1)*c)
  {
    const int c = (P + kCclThreads - 1) / kCclThreads;
    const int i0 = min(tid * c, P), i1 = min(i0 + c, P);
    int roots = 0;
    for (int i = i0; i < i1; ++i) roots += (L[i] == i) ? 1 : 0;
    int total;
    int rank = block_scan(roots, s_warp, &total);
    if (tid == 0) J.counters[CNT_NUM_CLUSTER] = total;
    for (int i = i0; i < i1; ++i) if (L[i] == i) L[i] = -(++rank);
  }
  __syncthreads();
  // H: every other run takes its root's -(id) (roots are negative now, and only a run's owner stores to it)
  for (int i = tid; i < P; i += kCclThreads) { const int r = L[i]; if (r >= 0) L[i] = L[r]; }
  // I: column masks back to rest (every column a point marked lies in once | twice)
  if (own) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int w = w0 + h;
      unsigned m = s_any[w];
      while (m) { const int b = __ffs(m) - 1; m &= m - 1u; J.colmask[(w >> 3) * kNumGrid + (w & 7) * 32 + b] = 0u; }
    }
  }
}

}  // namespace

bool layers_valid(const lmot_layers& l) {
  return (l.on == 0 || l.on == 1) && l.n_slices >= 1 && l.n_slices <= LMOT_MAX_SLICES && std::isfinite(l.slice_m) && l.slice_m > 0 &&
         std::isfinite(l.z_min) && l.gap_slices >= 0 && l.gap_slices <= l.n_slices - 1;
}

int layers_ensure(Ctx* c, Slot* s, cudaStream_t st) {
  if (s->d_layer_lab) return LMOT_OK;
  LMOT_CUDA(c, cudaMalloc(&s->d_slice, (size_t)c->max_points));
  LMOT_CUDA(c, cudaMalloc(&s->d_colmask, kCartCells * sizeof(unsigned)));
  LMOT_CUDA(c, cudaMemsetAsync(s->d_colmask, 0, kCartCells * sizeof(unsigned), st));
  LMOT_CUDA(c, cudaMalloc(&s->d_layer_cols, kCartCells * sizeof(unsigned)));
  LMOT_CUDA(c, cudaMalloc(&s->d_layer_base, (kCartCells + 1) * sizeof(int)));
  LMOT_CUDA(c, cudaMalloc(&s->d_layer_lab, (size_t)kLayerNodes * sizeof(int)));
  return LMOT_OK;
}

LayerTab layer_tab_of(const Slot* s) { return LayerTab{s->d_slice, s->d_layer_cols, s->d_layer_base, s->d_layer_lab}; }

int layers_launch(Ctx* c, cudaStream_t st, const LayerUnit* u, int n, Slot* mark) {
  if (n < 1 || n > kMaxBatch) return LMOT_ERR_INVALID;
  LayerMarkBatch M;
  LayerCclBatch C;
  int bound = 0;
  for (int i = 0; i < n; ++i) {
    Slot* s = u[i].s;
    M.j[i] = LayerMarkJob{s->d_elev, s->d_cart, s->d_counters, u[i].area, s->d_slice, s->d_colmask,
                          (double)u[i].sensor_height, u[i].cfg.z_min, u[i].cfg.slice_m, u[i].cfg.n_slices};
    C.j[i] = LayerCclJob{s->d_cart_bits, s->d_cart_bits + kBitWords, u[i].area, s->d_colmask, s->d_layer_cols, s->d_layer_base,
                         s->d_layer_lab, s->d_counters, u[i].cfg.n_slices, u[i].cfg.gap_slices};
    if (u[i].n_upper > bound) bound = u[i].n_upper;
  }
  for (int i = n; i < kMaxBatch; ++i) { M.j[i] = M.j[0]; C.j[i] = C.j[0]; }
  if (bound > 0) {
    const int bx = (bound + 255) / 256;
    layer_mark_kernel<<<dim3(bx, n), 256, 0, st>>>(M);
    kernel_mark(c, mark, st);
  }
  ccl_layer_kernel<<<n, kCclThreads, 0, st>>>(C);
  kernel_mark(c, mark, st);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

int layers_point_ids(Ctx* c, const Slot* s, int n, int32_t* ids) {
  if (n <= 0) return LMOT_OK;
  std::vector<uint16_t> cart(n);
  std::vector<uint8_t> slice(n);
  std::vector<unsigned> cols(kCartCells);
  std::vector<int> base(kCartCells + 1);
  LMOT_CUDA(c, cudaMemcpy(cart.data(), s->d_cart, (size_t)n * sizeof(uint16_t), cudaMemcpyDeviceToHost));
  LMOT_CUDA(c, cudaMemcpy(slice.data(), s->d_slice, (size_t)n, cudaMemcpyDeviceToHost));
  LMOT_CUDA(c, cudaMemcpy(cols.data(), s->d_layer_cols, kCartCells * sizeof(unsigned), cudaMemcpyDeviceToHost));
  LMOT_CUDA(c, cudaMemcpy(base.data(), s->d_layer_base, (kCartCells + 1) * sizeof(int), cudaMemcpyDeviceToHost));
  std::vector<int> lab(base[kCartCells] > 0 ? base[kCartCells] : 1);
  if (base[kCartCells] > 0)
    LMOT_CUDA(c, cudaMemcpy(lab.data(), s->d_layer_lab, (size_t)base[kCartCells] * sizeof(int), cudaMemcpyDeviceToHost));
  for (int i = 0; i < n; ++i) {
    ids[i] = 0;
    const unsigned sl = slice[i];
    if (sl == 0xFF) continue;
    const unsigned d = cols[cart[i]];
    if (!((d >> sl) & 1u)) continue;
    const unsigned starts = d & ~(d << 1);
    const unsigned below = sl == 31 ? 0xFFFFFFFFu : ((2u << sl) - 1u);
    ids[i] = -lab[base[cart[i]] + __builtin_popcount(starts & below) - 1];
  }
  return LMOT_OK;
}

}  // namespace lmot
