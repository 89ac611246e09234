// accumulate.cu -- sweep accumulation (lmot_set_accumulate): a frame is clustered and boxed together with the stream's last sweeps, each
// moved into the current sensor frame by the ego motion between the two stamps.
//
// The history is a ring of K = sweeps entries per detection unit on the device, one elevated cloud E_s each (a merge unit's: the merged
// vehicle-frame cloud).  accumulate_kernel runs between ground removal (and the rig merge) and clustering of a submission.  In one launch,
// for every accumulating unit, it copies the unit's own elevated cloud E_t into the ring entry the step owns, appends the earlier sweeps
// behind E_t in the unit's cloud (moved by their poses, with the clustering cell and occupancy bits of every
// appended point, as rig_merge_kernel does), and sets the count clustering and box fitting read to |E_acc|.  The ring holds K entries
// while a step reads at most K - 1: the entry being written is never one being read.
#include <cmath>
#include "lmot_internal.cuh"
#include "exact_math.cuh"
#include "ccl_device.cuh"

namespace lmot {

namespace {

constexpr int kAccThreads = 256;

struct AccParams {
  AccJob u[kMaxBatch];                 // blockIdx.z: the unit
  long long ring_stride;               // points per ring entry (max_points)
  int max_points;
};
static_assert(sizeof(AccParams) <= 4096, "accumulate_kernel: parameter block");

// grid (x: point blocks, y: 0 = copy E_t into the ring, 1 + j = sweep j, z: unit).  Sweep j of a unit starts at off_j = |E_t| + the
// lengths of its sweeps 0 .. j-1 and is used iff off_j + |E_s| <= max_points (the longest prefix of whole sweeps that fits).  The last of
// a unit's blocks to finish publishes its counts: nothing writes the counter the others read (CNT_N_ELEV: |E_t|) before every block of
// the unit has read it.
__global__ void __launch_bounds__(kAccThreads)
accumulate_kernel(const __grid_constant__ AccParams P) {
  __shared__ int s_n, s_off, s_fit, s_last;
  const AccJob& U = P.u[blockIdx.z];
  const int j = (int)blockIdx.y - 1;
  if (threadIdx.x == 0) {
    const int nt = U.counters[CNT_N_ELEV];
    int off = nt, n = nt, fit = 1;
    if (j >= U.n_sw) {
      n = 0; fit = 0;                  // (the grid is sized for the unit with the most candidates)
    } else if (j >= 0) {
      for (int i = 0; i < j; ++i) off += U.ring_n[U.entry[i]];
      n = U.ring_n[U.entry[j]];
      fit = off + n <= P.max_points;
    }
    s_n = n; s_off = off; s_fit = fit;
  }
  __syncthreads();
  const int n = s_n, off = s_off, i = blockIdx.x * kAccThreads + threadIdx.x;
  if (j < 0) {
    if (i < n) U.ring[U.w * P.ring_stride + i] = U.elev[i];
  } else if ((int)(blockIdx.x * kAccThreads) < n && s_fit) {      // (whole warps: cart_mark needs all 32 lanes)
    unsigned c = kNoCell;
    if (i < n) {
      const float4 q = U.ring[U.entry[j] * P.ring_stride + i];
      float x = q.x, y = q.y, z = q.z;
      rig_apply(U.m[j], x, y, z);
      U.elev[off + i] = make_float4(x, y, z, 1.f);
      c = cart_cell_of(x, y, U.roi, kNumGrid);
      U.cart[off + i] = (uint16_t)c;
    }
    cart_mark(c, U.bits, U.bits + kBitWords);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = atomicAdd(&U.counters[CNT_ACC_DONE], 1) == (int)(gridDim.x * gridDim.y) - 1;
  }
  __syncthreads();
  if (!s_last || threadIdx.x != 0) return;
  __threadfence();
  const int nt = U.counters[CNT_N_ELEV];
  int tot = nt, used = 0;
  for (; used < U.n_sw; ++used) {
    const int m = U.ring_n[U.entry[used]];
    if (tot + m > P.max_points) break;
    tot += m;
  }
  U.ring_n[U.w] = nt;
  U.counters[CNT_N_ELEV] = tot;
  U.counters[CNT_ACC_DONE] = 0;
  U.info[0] = tot; U.info[1] = used; U.info[2] = nt;
  __threadfence_system();              // info lives in pinned host memory: the host reads it after the step's completion event
}

}  // namespace

// step 2 of the definition (include/lmot.h), host libm, double, left to right.  4x4 products with the implicit row (0 0 0 1)
void accumulate_pose(const double fs[3], const double ft[3], const float* mount, float out[12]) {
  const double dy = ft[2] - fs[2];
  const double c = std::cos(dy), sn = std::sin(dy);
  const double tx = ft[0] - (c * fs[0] - sn * fs[1]);
  const double ty = ft[1] - (sn * fs[0] + c * fs[1]);
  const double A[4][4] = {{c, -sn, 0.0, tx}, {sn, c, 0.0, ty}, {0.0, 0.0, 1.0, 0.0}, {0.0, 0.0, 0.0, 1.0}};
  double M[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
  if (mount)
    for (int r = 0; r < 3; ++r)
      for (int k = 0; k < 4; ++k) M[r][k] = (double)mount[4 * r + k];
  double Mi[4][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 1}};
  for (int r = 0; r < 3; ++r) {
    for (int k = 0; k < 3; ++k) Mi[r][k] = M[k][r];
    Mi[r][3] = -((M[0][r] * M[0][3] + M[1][r] * M[1][3]) + M[2][r] * M[2][3]);
  }
  double P[4][4], D[4][4];
  for (int r = 0; r < 4; ++r)
    for (int k = 0; k < 4; ++k) P[r][k] = ((A[r][0] * M[0][k] + A[r][1] * M[1][k]) + A[r][2] * M[2][k]) + A[r][3] * M[3][k];
  for (int r = 0; r < 4; ++r)
    for (int k = 0; k < 4; ++k) D[r][k] = ((Mi[r][0] * P[0][k] + Mi[r][1] * P[1][k]) + Mi[r][2] * P[2][k]) + Mi[r][3] * P[3][k];
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 4; ++k) out[4 * r + k] = (float)D[r][k];
}

bool accumulate_valid(const lmot_accumulate& a) {
  return a.sweeps >= 1 && a.sweeps <= LMOT_MAX_SWEEPS && std::isfinite(a.max_age_s) && a.max_age_s > 0.0;
}

void accumulate_free(AccHist& h) {
  for (int u = 0; u < kMaxBatch; ++u) { cudaFree(h.d_ring[u]); cudaFree(h.d_ring_n[u]); h.d_ring[u] = nullptr; h.d_ring_n[u] = nullptr; }
  if (h.ev) cudaEventDestroy(h.ev);
  h.ev = nullptr; h.cap = 0; h.cap_units = 0; h.ev_live = false;
  h.forget();
  h.kind = -1; h.units = 0;
}

namespace {

// the rings for K entries of `units` units: all or nothing, after one device synchronisation (a smaller ring may still be read)
int accumulate_ensure(Ctx* c, AccHist& h, int K, int units) {
  if (h.cap >= K && h.cap_units >= units) return LMOT_OK;
  LMOT_CUDA(c, cudaDeviceSynchronize());
  const lmot_accumulate cfg = h.cfg;
  accumulate_free(h);
  h.cfg = cfg;
  bool ok = cudaEventCreateWithFlags(&h.ev, cudaEventDisableTiming) == cudaSuccess;
  for (int u = 0; ok && u < units; ++u)
    ok = cudaMalloc(&h.d_ring[u], (size_t)K * c->max_points * sizeof(float4)) == cudaSuccess &&
         cudaMalloc(&h.d_ring_n[u], K * sizeof(int)) == cudaSuccess && cudaMemset(h.d_ring_n[u], 0, K * sizeof(int)) == cudaSuccess;
  if (!ok) {
    c->last_error = std::string("sweep accumulation ring: ") + cudaGetErrorString(cudaGetLastError());
    accumulate_free(h);
    h.cfg = cfg;
    return LMOT_ERR_CUDA;
  }
  h.cap = K; h.cap_units = units;
  return LMOT_OK;
}

}  // namespace

int accumulate_step(Ctx* c, AccHist& h, int kind, int units, Slot* const* U, const lmot_sensor* pose, const float* roi, const int* n_upper,
                    const TrackerHost& th, double ts, double v, double yaw, Result* r, AccJob* jobs, int* fit_upper) {
  const int K = h.cfg.sweeps;
  int rc = accumulate_ensure(c, h, K, units);
  if (rc) return rc;
  if (h.kind != kind || h.units != units) { h.forget(); h.kind = kind; h.units = units; }
  TrackerHost peek = th;
  origin_points_fold(peek, ts, v, yaw);             // this step's fold, as the tracker launch will take it
  int nc = 0;
  long long sum[kMaxBatch];
  for (int u = 0; u < units; ++u) { sum[u] = n_upper[u]; jobs[u].bound = n_upper[u]; }
  int* info = nullptr;
  LMOT_CUDA(c, cudaHostGetDevicePointer((void**)&info, r->h_acc, 0));
  for (int j = 0; j < h.n; ++j) {
    const int e = (h.w - 1 - j + K) % K;
    const double age = (ts - h.ts[e]) / 1000000.0;
    if (!(age > 0.0 && age <= h.cfg.max_age_s)) break;
    r->acc_ts[nc] = h.ts[e];
    for (int u = 0; u < units; ++u) {
      accumulate_pose(h.fold[e], peek.fold, pose[u].pose, r->acc_pose[u][nc]);
      jobs[u].entry[nc] = e;
      memcpy(jobs[u].m[nc], r->acc_pose[u][nc], sizeof(jobs[u].m[nc]));
      sum[u] += h.n_upper[e][u];
      if (h.n_upper[e][u] > jobs[u].bound) jobs[u].bound = h.n_upper[e][u];
    }
    ++nc;
  }
  for (int u = 0; u < units; ++u) {
    AccJob& q = jobs[u];
    Slot* s = U[u];
    q.elev = s->d_elev; q.cart = s->d_cart; q.bits = s->d_cart_bits; q.counters = s->d_counters;
    q.ring = h.d_ring[u]; q.ring_n = h.d_ring_n[u]; q.info = info + 4 * u;
    q.roi = roi[u]; q.w = h.w; q.n_sw = nc;
    h.n_upper[h.w][u] = n_upper[u];
    fit_upper[u] = sum[u] < c->max_points ? (int)sum[u] : c->max_points;      // (may be n_upper itself)
  }
  r->acc_units = units;
  r->acc_cand = nc;
  h.ts[h.w] = ts;
  memcpy(h.fold[h.w], peek.fold, sizeof(h.fold[0]));
  h.w = (h.w + 1) % K;
  if (h.n < K - 1) ++h.n;
  return LMOT_OK;
}

int accumulate_launch(Ctx* c, cudaStream_t st, Slot* mark, const AccJob* jobs, int n_jobs, AccHist* const* hists, int nh) {
  if (n_jobs < 1 || n_jobs > kMaxBatch) return LMOT_ERR_INVALID;
  AccParams P;
  memset(&P, 0, sizeof(P));
  int ny = 1, nx = 1;
  for (int u = 0; u < n_jobs; ++u) {
    P.u[u] = jobs[u];
    if (1 + jobs[u].n_sw > ny) ny = 1 + jobs[u].n_sw;
    if (jobs[u].bound > nx) nx = jobs[u].bound;
  }
  P.ring_stride = c->max_points;
  P.max_points = c->max_points;
  for (int i = 0; i < nh; ++i)
    if (hists[i]->ev_live) LMOT_CUDA(c, cudaStreamWaitEvent(st, hists[i]->ev, 0));
  const int blocks = (nx + kAccThreads - 1) / kAccThreads;
  accumulate_kernel<<<dim3(blocks, ny, n_jobs), kAccThreads, 0, st>>>(P);
  kernel_mark(c, mark, st);
  LMOT_CUDA(c, cudaGetLastError());
  for (int i = 0; i < nh; ++i) { LMOT_CUDA(c, cudaEventRecord(hists[i]->ev, st)); hists[i]->ev_live = true; }
  return LMOT_OK;
}

}  // namespace lmot
