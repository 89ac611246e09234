// obstacles.cu -- obstacle footprints (lmot_set_obstacles): every cluster of a unit as a convex cell-footprint polygon, on sm_90a.
//
// The definition is in include/lmot.h.  One launch per submission, behind box fitting on the detection stream, over every unit whose
// stream has obstacles on (blockIdx.y = unit):
//   obstacles_kernel   one CTA per cluster (grid-stride over the unit's cluster count, read on the device).  The cluster's points are box
//                      fitting's gathered segment (d_sorted_pts / d_seg_start / d_seg_size, cloud order).  Each point's cell is
//                      cart_cell_of of its own x, y and the unit's ROI -- the function, the point and the ROI clustering stored in d_cart,
//                      so the same cell.  In shared memory: a 62,500-bit cell set (n_cells), per corner column u in [0, 250] the smallest
//                      and largest corner v of the cells touching it, and the z range.  Andrew's monotone chain then runs over at most
//                      2 x 251 column extremes, lower chain on one thread and upper chain on another, in integer arithmetic, and the
//                      hull goes to the slot's scratch (at most LMOT_OBSTACLE_MAX_HULL corners of one byte per coordinate).
//   its last CTA       per unit: one pass over the clusters in id order -- the box index is the rank of the cluster among box fitting's
//                      accepted clusters (d_cl_ok, the verdict the compaction used; the rule filter does not run again), the vertex
//                      offset the prefix of the hull sizes -- then every hull that fits the pool is written in metres.
// Headers and vertices are stored straight into the result's pinned, device-mapped obstacle block: no copy, and nothing is moved for a
// unit whose stream has obstacles off.
#include <climits>
#include <cstring>
#include <vector>
#include "lmot_internal.cuh"
#include "exact_math.cuh"

namespace lmot {

namespace {

constexpr int kObsThreads = 256;
constexpr int kHull = LMOT_OBSTACLE_MAX_HULL;
constexpr int kCellWords = (kCartCells + 31) / 32;     // 1,954
constexpr int kCornerCols = kNumGrid + 1;              // corners u = 0 .. 250
constexpr size_t kUnitHdrBytes = 16;                   // n_obstacles, n_vertices needed, 2 spare ints

static_assert(sizeof(lmot_obstacle) == 32, "lmot_obstacle layout");

struct ObsJob {
  const float4* sorted_pts; const int* seg_start; const int* seg_size; const int* counters; const uint8_t* cl_ok;
  int* hull_n; uchar2* hull; int* done;
  unsigned char* out;                                  // device view of the unit's part of the result's obstacle block
  float roi; int max_vertices;
};
struct ObsBatch { ObsJob j[kMaxBatch]; };

__device__ __forceinline__ unsigned zkey(float f) {   // order-preserving
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float zval(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }

// (b - a) x (c - a) of lattice points
__device__ __forceinline__ int cross3(short2 a, short2 b, short2 c) {
  return ((int)b.x - a.x) * ((int)c.y - a.y) - ((int)b.y - a.y) * ((int)c.x - a.x);
}

// one monotone chain: push p, popping while the last two points and p do not turn left (collinear corners are dropped)
__device__ __forceinline__ void chain_push(short2* h, int& n, short2 p) {
  while (n >= 2 && cross3(h[n - 2], h[n - 1], p) <= 0) --n;
  h[n++] = p;
}

// exclusive block scan of two ints (kObsThreads threads); totals to every thread
__device__ __forceinline__ void scan2(int a, int b, int& ea, int& eb, int& ta, int& tb, int2* s_w) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int ia = a, ib = b;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int xa = __shfl_up_sync(0xFFFFFFFFu, ia, o), xb = __shfl_up_sync(0xFFFFFFFFu, ib, o);
    if (lane >= o) { ia += xa; ib += xb; }
  }
  __syncthreads();
  if (lane == 31) s_w[warp] = make_int2(ia, ib);
  __syncthreads();
  int pa = 0, pb = 0;
  ta = 0; tb = 0;
  for (int w = 0; w < kObsThreads / 32; ++w) {
    const int2 v = s_w[w];
    if (w < warp) { pa += v.x; pb += v.y; }
    ta += v.x; tb += v.y;
  }
  ea = pa + ia - a; eb = pb + ib - b;
}

__global__ void __launch_bounds__(kObsThreads)
obstacles_kernel(const __grid_constant__ ObsBatch P, int max_clusters, int max_boxes) {
  const ObsJob& J = P.j[blockIdx.y];
  __shared__ unsigned s_cells[kCellWords];
  __shared__ int s_lo[kCornerCols], s_hi[kCornerCols];
  __shared__ short2 s_low[kCornerCols + 2], s_up[kCornerCols + 2];
  __shared__ int s_nlow, s_nup, s_ncells, s_umin, s_umax;
  __shared__ unsigned s_zmin, s_zmax;
  __shared__ int2 s_w[kObsThreads / 32];
  __shared__ int s_last;
  const int tid = threadIdx.x;
  const int K = min(J.counters[CNT_NUM_CLUSTER], max_clusters);
  lmot_obstacle* rows = reinterpret_cast<lmot_obstacle*>(J.out + kUnitHdrBytes);

  for (int k = blockIdx.x + 1; k <= K; k += gridDim.x) {
    const int n = J.seg_size[k];
    const float4* __restrict__ seg = J.sorted_pts + J.seg_start[k];
    for (int w = tid; w < kCellWords; w += kObsThreads) s_cells[w] = 0u;
    for (int u = tid; u < kCornerCols; u += kObsThreads) { s_lo[u] = INT_MAX; s_hi[u] = -1; }
    if (tid == 0) { s_ncells = 0; s_zmin = ~0u; s_zmax = 0u; s_umin = INT_MAX; s_umax = -1; }
    __syncthreads();
    unsigned zlo = ~0u, zhi = 0u;
    int fresh = 0, umin = INT_MAX, umax = -1;
    for (int j = tid; j < n; j += kObsThreads) {
      const float4 q = __ldg(&seg[j]);
      const unsigned kz = zkey(q.z);
      zlo = min(zlo, kz); zhi = max(zhi, kz);
      const unsigned c = cart_cell_of(q.x, q.y, J.roi, kNumGrid);
      if (c == kNoCell) continue;                      // (a clustered point always has its cell)
      const unsigned bit = 1u << (c & 31u);
      if (atomicOr(&s_cells[c >> 5], bit) & bit) continue;
      ++fresh;
      const int u = (int)(c / (unsigned)kNumGrid), v = (int)c - u * kNumGrid;
      atomicMin(&s_lo[u], v); atomicMin(&s_lo[u + 1], v);
      atomicMax(&s_hi[u], v + 1); atomicMax(&s_hi[u + 1], v + 1);
      umin = min(umin, u); umax = max(umax, u + 1);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      zlo = min(zlo, __shfl_xor_sync(0xFFFFFFFFu, zlo, o)); zhi = max(zhi, __shfl_xor_sync(0xFFFFFFFFu, zhi, o));
      fresh += __shfl_xor_sync(0xFFFFFFFFu, fresh, o);
      umin = min(umin, __shfl_xor_sync(0xFFFFFFFFu, umin, o)); umax = max(umax, __shfl_xor_sync(0xFFFFFFFFu, umax, o));
    }
    if ((tid & 31) == 0) {
      atomicMin(&s_zmin, zlo); atomicMax(&s_zmax, zhi); atomicAdd(&s_ncells, fresh);
      atomicMin(&s_umin, umin); atomicMax(&s_umax, umax);
    }
    __syncthreads();
    const int u0 = s_umin, u1 = s_umax;
    if (u1 >= 0) {
      // lower chain: column minima left to right, then the top of the last column; upper chain: column maxima right to left, then the
      // bottom of the first column.  Both start and end on the two extreme columns' corners, so hull = lower[:-1] + upper[:-1]
      if (tid == 0) {
        int nl = 0;
        for (int u = u0; u <= u1; ++u)
          if (s_hi[u] >= 0) chain_push(s_low, nl, make_short2((short)u, (short)s_lo[u]));
        chain_push(s_low, nl, make_short2((short)u1, (short)s_hi[u1]));
        s_nlow = nl;
      } else if (tid == 32) {
        int nu = 0;
        for (int u = u1; u >= u0; --u)
          if (s_hi[u] >= 0) chain_push(s_up, nu, make_short2((short)u, (short)s_hi[u]));
        chain_push(s_up, nu, make_short2((short)u0, (short)s_lo[u0]));
        s_nup = nu;
      }
    } else if (tid == 0) {
      s_nlow = 1; s_nup = 1;                           // no cell: no polygon
    }
    __syncthreads();
    const int nl = s_nlow - 1;
    const int m = min(nl + s_nup - 1, kHull);          // (<= 140 for every lattice polygon in [0, 250]^2: include/lmot.h)
    uchar2* __restrict__ hull = J.hull + (size_t)k * kHull;
    for (int j = tid; j < m; j += kObsThreads) {
      const short2 p = j < nl ? s_low[j] : s_up[j - nl];
      hull[j] = make_uchar2((unsigned char)p.x, (unsigned char)p.y);
    }
    if (tid == 0) {                                    // (box, vertex_offset and vertex_count: the last CTA's; no field is stored twice)
      J.hull_n[k] = m;
      lmot_obstacle* o = rows + (k - 1);
      o->cluster = k; o->n_points = n; o->n_cells = s_ncells;
      o->z_min = n > 0 ? zval(s_zmin) : 0.f; o->z_max = n > 0 ? zval(s_zmax) : 0.f;
    }
    __syncthreads();
  }

  // ---- the unit's last CTA: box indices, vertex offsets and the vertices themselves, in cluster-id order
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(J.done, 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (tid == 0) *J.done = 0;                           // re-armed for the next launch on this slot
  float2* __restrict__ xy = reinterpret_cast<float2*>(J.out + kUnitHdrBytes + (size_t)max_clusters * sizeof(lmot_obstacle));
  const double roi = (double)J.roi, half = __ddiv_rn(roi, 2.0);
  int carry_b = 0, carry_v = 0;
  for (int k0 = 1; k0 <= K; k0 += kObsThreads) {
    const int k = k0 + tid;
    const int ok = k <= K ? (int)__ldcg(&J.cl_ok[k]) : 0;
    const int hn = k <= K ? __ldcg(&J.hull_n[k]) : 0;
    int eb, ev, tb, tv;
    scan2(ok ? 1 : 0, hn, eb, ev, tb, tv, s_w);
    if (k <= K) {
      const int rank = carry_b + eb, off = carry_v + ev;
      const bool fits = (long long)off + hn <= (long long)J.max_vertices;
      rows[k - 1].box = (ok && rank < max_boxes) ? rank : -1;
      rows[k - 1].vertex_offset = off;
      rows[k - 1].vertex_count = fits ? hn : 0;
      if (fits) {
        const uchar2* __restrict__ hull = J.hull + (size_t)k * kHull;
        for (int j = 0; j < hn; ++j) {
          const uchar2 p = __ldcg(&hull[j]);
          xy[off + j] = make_float2((float)__dsub_rn(__ddiv_rn(__dmul_rn((double)p.x, roi), 250.0), half),
                                    (float)__dsub_rn(__ddiv_rn(__dmul_rn((double)p.y, roi), 250.0), half));
        }
      }
    }
    carry_b += tb; carry_v += tv;
  }
  if (tid == 0) {
    int* hdr = reinterpret_cast<int*>(J.out);
    hdr[0] = K; hdr[1] = carry_v; hdr[2] = 0; hdr[3] = 0;
    __threadfence_system();
  }
}

size_t hull_bytes(int max_clusters) { return (size_t)(max_clusters + 1) * (sizeof(int) + kHull * sizeof(uchar2)) + 16; }

size_t unit_bytes(int max_clusters, int cap_vertices) {
  return kUnitHdrBytes + (size_t)max_clusters * sizeof(lmot_obstacle) + (size_t)cap_vertices * sizeof(float2);
}

}  // namespace

bool obstacles_valid(const lmot_obstacles& o) {
  return (o.on == 0 || o.on == 1) && o.max_vertices >= LMOT_OBSTACLE_MAX_HULL && o.max_vertices <= (1 << 24);
}

int obstacles_ensure(Ctx* c, const ObsUnit* u, int n, cudaStream_t st) {
  for (int i = 0; i < n; ++i) {
    Slot* s = u[i].s;
    if (s->d_obs_hull) continue;
    const size_t b = hull_bytes(c->prm.max_clusters);
    LMOT_CUDA(c, cudaMalloc(&s->d_obs_hull, b));
    LMOT_CUDA(c, cudaMemsetAsync(s->d_obs_hull + b - 16, 0, 16, st));      // the last-CTA counter, zero at rest
  }
  for (int i = 0; i < n; ++i) {
    Result* r = u[i].r;
    bool first = true;
    for (int j = 0; j < i; ++j) first &= u[j].r != r;
    if (!first) continue;
    int units = 0, mv = 0;
    for (int j = 0; j < n; ++j)
      if (u[j].r == r) { units = u[j].slot + 1 > units ? u[j].slot + 1 : units; mv = u[j].max_vertices > mv ? u[j].max_vertices : mv; }
    if (!r->ev_obs) LMOT_CUDA(c, cudaEventCreateWithFlags(&r->ev_obs, cudaEventDisableTiming));
    if (r->obs_cap_units < units || r->obs_cap_vertices < mv) {       // grown, never shrunk
      const int cu = units > r->obs_cap_units ? units : r->obs_cap_units;
      const int cv = mv > r->obs_cap_vertices ? mv : r->obs_cap_vertices;
      if (r->obs_pending) LMOT_CUDA(c, cudaEventSynchronize(r->ev_obs));
      if (r->h_obs) cudaFreeHost(r->h_obs);
      r->h_obs = nullptr;
      r->obs_cap_units = 0; r->obs_cap_vertices = 0; r->obs_pending = false;
      LMOT_CUDA(c, cudaHostAlloc(&r->h_obs, (size_t)cu * unit_bytes(c->prm.max_clusters, cv), cudaHostAllocMapped));
      r->obs_cap_units = cu; r->obs_cap_vertices = cv;
    }
    // the block's previous obstacle kernel (a result dropped uncollected) is done before this one writes it
    if (r->obs_pending) LMOT_CUDA(c, cudaStreamWaitEvent(st, r->ev_obs, 0));
    r->obs_units = units;
  }
  for (int i = 0; i < n; ++i) u[i].r->obs_max_vertices[u[i].slot] = u[i].max_vertices;
  return LMOT_OK;
}

int obstacles_launch(Ctx* c, cudaStream_t st, const ObsUnit* u, int n, Slot* mark) {
  if (n < 1 || n > kMaxBatch) return LMOT_ERR_INVALID;
  const int MC = c->prm.max_clusters, K1 = MC + 1;
  ObsBatch B;
  memset(&B, 0, sizeof(B));
  for (int i = 0; i < n; ++i) {
    Slot* s = u[i].s;
    Result* r = u[i].r;
    unsigned char* d_blk = nullptr;
    LMOT_CUDA(c, cudaHostGetDevicePointer((void**)&d_blk, r->h_obs, 0));
    ObsJob& j = B.j[i];
    j.sorted_pts = s->d_sorted_pts; j.seg_start = s->d_seg_start; j.seg_size = s->d_seg_size; j.counters = s->d_counters; j.cl_ok = s->d_cl_ok;
    j.hull_n = reinterpret_cast<int*>(s->d_obs_hull);
    j.hull = reinterpret_cast<uchar2*>(s->d_obs_hull + (size_t)K1 * sizeof(int));
    j.done = reinterpret_cast<int*>(s->d_obs_hull + hull_bytes(MC) - 16);
    j.out = d_blk + (size_t)u[i].slot * unit_bytes(MC, r->obs_cap_vertices);
    j.roi = u[i].roi; j.max_vertices = u[i].max_vertices;
  }
  for (int i = n; i < kMaxBatch; ++i) B.j[i] = B.j[0];
  const int gx = n == 1 ? c->fit_ctas : (c->fit_ctas / 2 > 8 ? c->fit_ctas / 2 : 8);
  obstacles_kernel<<<dim3(gx, n), kObsThreads, 0, st>>>(B, MC, c->prm.max_boxes);
  kernel_mark(c, mark, st);
  LMOT_CUDA(c, cudaGetLastError());
  for (int i = 0; i < n; ++i) {
    bool first = true;
    for (int j = 0; j < i; ++j) first &= u[j].r != u[i].r;
    if (!first) continue;
    LMOT_CUDA(c, cudaEventRecord(u[i].r->ev_obs, st));
    u[i].r->obs_pending = true;
  }
  return LMOT_OK;
}

int obstacles_collect(Ctx* c, Result* r, ObsLast& dst) {
  dst.valid = false;
  dst.units = 0;
  if (r->obs_units <= 0) return LMOT_OK;
  LMOT_CUDA(c, cudaEventSynchronize(r->ev_obs));
  const int MC = c->prm.max_clusters;
  const size_t ub = unit_bytes(MC, r->obs_cap_vertices);
  for (int i = 0; i < r->obs_units; ++i) {
    const unsigned char* blk = r->h_obs + (size_t)i * ub;
    const int* hdr = reinterpret_cast<const int*>(blk);
    const int K = hdr[0], V = hdr[1], mv = r->obs_max_vertices[i];
    dst.n_obs[i] = K; dst.n_vert[i] = V; dst.max_vertices[i] = mv;
    const lmot_obstacle* rows = reinterpret_cast<const lmot_obstacle*>(blk + kUnitHdrBytes);
    dst.rows[i].assign(rows, rows + K);
    const float* xy = reinterpret_cast<const float*>(blk + kUnitHdrBytes + (size_t)MC * sizeof(lmot_obstacle));
    const int nv = V < mv ? V : mv;
    dst.xy[i].assign(xy, xy + 2 * (size_t)nv);
  }
  dst.units = r->obs_units;
  dst.valid = true;
  return LMOT_OK;
}

void obstacles_result_free(Result* r) {
  if (r->h_obs) cudaFreeHost(r->h_obs);
  if (r->ev_obs) cudaEventDestroy(r->ev_obs);
  r->h_obs = nullptr; r->ev_obs = nullptr;
  r->obs_cap_units = 0; r->obs_cap_vertices = 0; r->obs_units = 0; r->obs_pending = false;
}

}  // namespace lmot
