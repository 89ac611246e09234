// rig_merge.cu -- merging sensor rigs (lmot_set_rig_merge / lmot_seq_set_rig_merge): the sensors' elevated clouds of a tick, moved
// into the vehicle frame and concatenated in table order, become ONE cloud that is clustered and boxed once.
//
// Ground removal stays per sensor (the polar grid assumes rays from the cloud's origin and ground h_sensor below it: true only in the
// sensor's own frame).  rig_merge_kernel then does the merge, the 0.2 m cell of every merged point and the occupancy bit planes in one
// pass, so the CCL and box-fitting launches that follow treat a merge unit like any other frame.
#include "lmot_internal.cuh"
#include "exact_math.cuh"
#include "ccl_device.cuh"

namespace lmot {

namespace {

constexpr int kMergeThreads = 256;

// source i of the launch: a sensor's detection slot and its pose; it is sensor `rank` of merge unit `unit`
struct MergeSrc { const float4* elev; const int* counters; unsigned* bits; float m[12]; int unit, rank; };
// unit u: the merged cloud and its buffers; its sensors are sources [s0, s0 + ns); frame_counts: its rows of the result block
struct MergeDst { float4* elev; uint16_t* cart; unsigned* bits; int* counters; int* frame_counts; float roi; int s0, ns; };
struct MergeParams { MergeSrc s[kMaxBatch]; MergeDst u[kMaxBatch]; int max_points; };
static_assert(sizeof(MergeParams) <= 4096, "rig_merge_kernel: parameter block");

// grid (x: point blocks, y: source).  Thread i of source j's blocks moves point i of sensor j's elevated cloud to position
// off_j + i of its unit's cloud (off_j = the elevated points of the unit's earlier sensors); positions at or above max_points are cut.
__global__ void __launch_bounds__(kMergeThreads)
rig_merge_kernel(const __grid_constant__ MergeParams P) {
  const MergeSrc& S = P.s[blockIdx.y];
  const MergeDst& U = P.u[S.unit];
  // the sensor's `once` / `twice` planes back to their rest state: the ground kernel marked them, and no CCL runs on this sensor's frame
  // (ccl_dense_body re-arms only the frames it runs on)
  for (int w = blockIdx.x * kMergeThreads + threadIdx.x; w < 2 * kBitWords; w += gridDim.x * kMergeThreads) S.bits[w] = 0u;
  __shared__ int s_off, s_n;
  if (threadIdx.x == 0) {
    int off = 0;
    for (int i = U.s0; i < U.s0 + S.rank; ++i) off += P.s[i].counters[CNT_N_ELEV];
    s_off = off;
    s_n = S.counters[CNT_N_ELEV];
    if (blockIdx.x == 0 && S.rank == 0) {
      // the unit's counters (what clustering / box fitting read, and the concatenation sums) and the sensors' count rows
      int tot = 0, ng = 0;
      for (int r = 0; r < U.ns; ++r) {
        const int* fc = P.s[U.s0 + r].counters;
        const int e = fc[CNT_N_ELEV], g = fc[CNT_N_GROUND];
        tot += e; ng += g;
        U.frame_counts[4 * r] = e; U.frame_counts[4 * r + 1] = g; U.frame_counts[4 * r + 2] = 0; U.frame_counts[4 * r + 3] = 0;
      }
      U.counters[CNT_N_ELEV] = tot < P.max_points ? tot : P.max_points;
      U.counters[CNT_N_GROUND] = ng;
      U.counters[CNT_ERROR] = tot > P.max_points ? (int)LMOT_ERR_CAPACITY : 0;
    }
  }
  __syncthreads();
  const int n = s_n, off = s_off;
  if ((int)(blockIdx.x * kMergeThreads) >= n) return;          // whole block past the end (the grid is sized for the largest frame)
  const int i = blockIdx.x * kMergeThreads + threadIdx.x;
  unsigned c = kNoCell;
  if (i < n && off + i < P.max_points) {
    const float4 q = __ldg(&S.elev[i]);
    float x = q.x, y = q.y, z = q.z;
    rig_apply(S.m, x, y, z);
    U.elev[off + i] = make_float4(x, y, z, 1.f);
    c = cart_cell_of(x, y, U.roi, kNumGrid);
    U.cart[off + i] = (uint16_t)c;
  }
  cart_mark(c, U.bits, U.bits + kBitWords);
}

}  // namespace

// on failure the unit may be partly allocated: the caller frees it with merge_unit_destroy
int merge_unit_create(Ctx* c, Slot* u, int index) {
  u->index = index;
  u->stream = c->stream;               // (the allocators' memsets; the caller synchronises the device afterwards)
  int rc = LMOT_OK;
  if (cudaMalloc(&u->d_elev, (size_t)c->max_points * sizeof(float4)) != cudaSuccess ||
      cudaMalloc(&u->d_counters, CNT_COUNT * sizeof(int)) != cudaSuccess ||
      cudaMemsetAsync(u->d_counters, 0, CNT_COUNT * sizeof(int), c->stream) != cudaSuccess) {
    c->last_error = std::string("merge unit: ") + cudaGetErrorString(cudaGetLastError());
    rc = LMOT_ERR_CUDA;
  }
  if (rc == LMOT_OK) rc = cluster_alloc(c, u);
  if (rc == LMOT_OK) rc = boxfit_alloc(c, u);
  u->stream = nullptr;
  return rc;
}

bool merge_unit_ready(const Slot* u) {
  return u->d_elev && u->d_counters && u->d_cart && u->d_cart_bits && u->d_label_grid && u->d_pcid && u->d_table && u->d_seg_start &&
         u->d_seg_size && u->d_sorted_pts && u->d_cl_box && u->d_cl_marker && u->d_cl_ok && u->d_boxes && u->d_boxes_g && u->d_markers &&
         u->d_done && u->d_det_sem;
}

void merge_unit_destroy(Slot* u) {
  cudaFree(u->d_elev); cudaFree(u->d_counters);              // (cudaFree(nullptr) is a no-op: a partly created unit is fine)
  cudaFree(u->d_area_mask);
  cluster_free(u); boxfit_free(u);
  *u = Slot{};
}

int rig_merge_launch(Ctx* c, cudaStream_t st, Slot* const* src, const lmot_sensor* pose, const int* n_upper, int n_units, const int* s0,
                     Slot* const* units, int* const* frame_counts, const float* roi) {
  const int NS = s0[n_units];
  if (n_units < 1 || NS < 1 || NS > kMaxBatch) return LMOT_ERR_INVALID;
  MergeParams P;
  memset(&P, 0, sizeof(P));
  int blocks = 1;
  for (int u = 0; u < n_units; ++u) {
    Slot* d = units[u];
    P.u[u] = MergeDst{d->d_elev, d->d_cart, d->d_cart_bits, d->d_counters, frame_counts[u], roi[u], s0[u], s0[u + 1] - s0[u]};
    for (int i = s0[u]; i < s0[u + 1]; ++i) {
      MergeSrc& q = P.s[i];
      q.elev = src[i]->d_elev; q.counters = src[i]->d_counters; q.bits = src[i]->d_cart_bits;
      memcpy(q.m, pose[i].pose, sizeof(q.m));
      q.unit = u; q.rank = i - s0[u];
      const int b = (n_upper[i] + kMergeThreads - 1) / kMergeThreads;
      if (b > blocks) blocks = b;
    }
  }
  P.max_points = c->max_points;
  rig_merge_kernel<<<dim3(blocks, NS), kMergeThreads, 0, st>>>(P);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

}  // namespace lmot
