// api.cu -- the extern "C" boundary declared in include/lmot.h.  Host-side marshalling only: H2D/D2H copies,
// stream/event ordering of the frame pipeline and capacity checks; every algorithmic step is a CUDA kernel in
// ground.cu / cluster.cu / boxfit.cu / tracker.cu.  There is deliberately no CPU implementation of any stage here.
//
// Frame pipeline: a context owns `pipeline_depth` detection slots (own stream + own buffers each), one tracker stream
// and one publish stream.  Frame f runs ground -> cluster -> box on slot f % depth; the tracker chain (gate -> TA -> TB
// -> TC, tracker.cu) waits ON THE DEVICE for the slot's boxes and folds them into the track table; publish_kernel moves
// the frame's results (counts, boxes, per-track outputs) from their device block into the pinned, device-mapped host
// block of the result ring and releases the slot; the host only waits on an event.
#include <cmath>
#include <cstring>
#include <cstdint>
#include <cstdlib>
#include <new>
#include <chrono>
#include <vector>
#include "lmot_internal.cuh"
#include "exact_math.cuh"
#include "ground_lines.cuh"

using namespace lmot;

struct lmot_ctx {
  Ctx c;
};

namespace {

inline double now_ns() { return (double)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// gaussKernel(samples=3, sigma=1.0) exactly as gaus_blur.cpp:26-49 evaluates it (host libm, double)
void gauss_taps(double tap[3]) {
  const int samples = 3;
  const double sigma = 1.0;
  const double mean = samples / 2;  // integer division, = 1 (gaus_blur.cpp:28)
  double sum = 0.0;
  for (int x = 0; x < samples; ++x) {
    tap[x] = std::exp(-0.5 * (std::pow((x - mean) / sigma, 2.0))) / (2 * M_PI * sigma * sigma);
    sum += tap[x];
  }
  for (int x = 0; x < samples; ++x) tap[x] /= sum;
}

int upload_points(Ctx* c, Slot* s, cudaStream_t st, const float* points, int n, int stride, float4* d_dst) {
  if (n < 0 || (n > 0 && !points) || stride < 3) return LMOT_ERR_INVALID;
  if (n > c->max_points) return LMOT_ERR_CAPACITY;
  if (n == 0) return LMOT_OK;
  if (stride == 4) {
    LMOT_CUDA(c, cudaMemcpyAsync(d_dst, points, (size_t)n * 16, cudaMemcpyHostToDevice, st));
  } else {
    if (stride > 4) {  // wide host records: pack xyz on the host side of the copy
      std::vector<float> tmp((size_t)n * 3);
      for (int i = 0; i < n; ++i) { tmp[3*i] = points[(size_t)i*stride]; tmp[3*i+1] = points[(size_t)i*stride+1]; tmp[3*i+2] = points[(size_t)i*stride+2]; }
      LMOT_CUDA(c, cudaMemcpyAsync(s->d_stage_in, tmp.data(), (size_t)n * 12, cudaMemcpyHostToDevice, st));
      LMOT_CUDA(c, cudaStreamSynchronize(st));
      stride = 3;
    } else {
      LMOT_CUDA(c, cudaMemcpyAsync(s->d_stage_in, points, (size_t)n * stride * 4, cudaMemcpyHostToDevice, st));
    }
    int rc = ground_repack(c, st, s->d_stage_in, n, stride, d_dst);
    if (rc) return rc;
  }
  return LMOT_OK;
}

// ---- sweep deskew (deskew.cu; include/lmot.h): the frame's motion from the stream's fold, and the staging of frames and pose tables
constexpr int kDeskewTab = LMOT_DESKEW_SLICES * 12;            // floats of one pose table
constexpr size_t kDeskewTabBytes = kDeskewTab * sizeof(float);

// omega of the frame (ts, v, yaw) of the table whose host state is th: diffYaw and dt as the tracker launch's fold will take them
// (peeked on a copy); 0 on the table's first frame, for dt <= 0 and for anything not finite
double deskew_omega(const TrackerHost& th, double ts, double v, double yaw) {
  if (!th.init) return 0.0;
  TrackerHost peek = th;
  origin_points_fold(peek, ts, v, yaw);
  const double diffYaw = peek.egoYaw - peek.egoPreYaw;
  const double dt = (ts - th.timestamp) / 1000000.0;
  if (!std::isfinite(diffYaw) || !std::isfinite(dt) || !(dt > 0.0)) return 0.0;
  const double w = std::remainder(diffYaw, 2.0 * M_PI) / dt;
  return std::isfinite(w) ? w : 0.0;
}

// a host frame's records (stride floats each) -> slot s's raw device staging on st: d_stage_in for stride 4, d_stage_wide (grown to the
// largest frame seen; growing waits for the device once) for wider records
int deskew_stage_host(Ctx* c, Slot* s, cudaStream_t st, const float* points, int n, int stride, const float** d_raw) {
  *d_raw = nullptr;
  if (n == 0) return LMOT_OK;
  const size_t bytes = (size_t)n * stride * sizeof(float);
  float* dst = s->d_stage_in;
  if (stride > 4) {
    if (bytes > s->stage_wide_bytes) {
      LMOT_CUDA(c, cudaStreamSynchronize(st));       // (cudaFree waits for the device anyway: the old staging may still be read)
      cudaFree(s->d_stage_wide);
      s->d_stage_wide = nullptr; s->stage_wide_bytes = 0;
      LMOT_CUDA(c, cudaMalloc(&s->d_stage_wide, bytes));
      s->stage_wide_bytes = bytes;
    }
    dst = s->d_stage_wide;
  }
  LMOT_CUDA(c, cudaMemcpyAsync(dst, points, bytes, cudaMemcpyHostToDevice, st));
  *d_raw = dst;
  return LMOT_OK;
}

int fetch_counters(Ctx* c, Slot* s, cudaStream_t st) {
  LMOT_CUDA(c, cudaMemcpyAsync(s->h_counters, s->d_counters, CNT_COUNT * sizeof(int), cudaMemcpyDeviceToHost, st));
  LMOT_CUDA(c, cudaStreamSynchronize(st));
  return LMOT_OK;
}

// write a host-known count into the slot's device counter block (entry points that start mid-pipeline)
int set_counter(Ctx* c, Slot* s, cudaStream_t st, int which, int value) {
  s->h_set[which] = value;
  LMOT_CUDA(c, cudaMemcpyAsync(s->d_counters + which, s->h_set + which, sizeof(int), cudaMemcpyHostToDevice, st));
  return LMOT_OK;
}

int check_device_error(Ctx* c, Slot* s, cudaStream_t st) {
  const int e = s->h_counters[CNT_ERROR];
  if (e != 0) {
    set_counter(c, s, st, CNT_ERROR, 0);
    cudaStreamSynchronize(st);
    return e;
  }
  return LMOT_OK;
}

// wait until nothing of this context is running on the device and forget uncollected results
int drain(Ctx* c) {
  for (int i = 0; i < c->n_slots; ++i) LMOT_CUDA(c, cudaStreamSynchronize(c->slots[i].stream));
  for (int i = 0; i < c->n_bslots; ++i) LMOT_CUDA(c, cudaStreamSynchronize(c->bslots[i].stream));
  for (int b = 0; b < kBatchBanks; ++b) if (c->bank[b].stream) LMOT_CUDA(c, cudaStreamSynchronize(c->bank[b].stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->trk_stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->pub_stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < c->n_results; ++i) c->results[i].in_flight = false;
  c->n_in_flight = 0;
  c->res_oldest = c->res_next;
  return LMOT_OK;
}

// next detection slot of the ring (reuse is ordered on the device by the slot's ev_trk_done)
Slot* acquire_slot(Ctx* c) {
  Slot* s = &c->slots[c->next_slot];
  c->last_slot = c->next_slot;
  c->next_slot = (c->next_slot + 1) % c->n_slots;
  return s;
}

// next result block of the ring; `drop_oldest`: an uncollected result still sitting in it is dropped, otherwise the
// caller gets nullptr (ring full: collect first)
Result* acquire_result(Ctx* c, bool drop_oldest) {
  Result* r = &c->results[c->res_next];
  if (r->in_flight) {
    if (!drop_oldest) return nullptr;
    cudaEventSynchronize(r->ev_done);            // its kernels may still be writing the block
    r->in_flight = false;
    --c->n_in_flight;
    c->res_oldest = (c->res_next + 1) % c->n_results;
  }
  c->res_next = (c->res_next + 1) % c->n_results;
  c->last_res = r;
  r->merge_rows = 0;                             // only a merging batched tick sets it (batch_common): collect_result reads it
  r->acc_units = 0;                              // only an accumulating step sets it (accumulate_step)
  r->obs_units = 0;                              // only a step with obstacles on sets it (obstacles_ensure)
  return r;
}

// the tracker chain + publication of one tick: boxes / counters of `s` (a detection slot, or a batch bank) -> track table -> result block r
int submit_tracker(Ctx* c, Slot* s, Result* r, const float* d_boxes, const int* d_counters, double ts, double v, double yaw) {
  int rc;
  // the tracker waits for this tick's detection on the DEVICE (gate kernel), or on ev_det_done where that is not possible
  bool gated = false;
  if ((rc = tracker_launch(c, s, c->trk_stream, d_boxes, d_counters, ts, v, yaw, true, &gated))) return rc;
  if (gated) {
    // Nothing but kernels on the tracker stream (an event record between spawn_output_kernel and the next frame's gate
    // kernel would serialise the two launches): publish_kernel polls the device-side step count, and "the slot is free"
    // is recorded behind it on the publish stream -- a little later than strictly necessary, detection has the slack
    if ((rc = tracker_publish(c, r, c->pub_stream))) return rc;
    LMOT_CUDA(c, cudaEventRecord(r->ev_done, c->pub_stream));
    LMOT_CUDA(c, cudaEventRecord(s->ev_trk_done, c->pub_stream));
  } else {
    if (c->timing) cudaEventRecord(r->ev[4], c->trk_stream);
    LMOT_CUDA(c, cudaEventRecord(s->ev_trk_done, c->trk_stream));      // the slot is free: its boxes / counters were consumed
    LMOT_CUDA(c, cudaEventRecord(r->ev_tc, c->trk_stream));
    // device block -> pinned host block, off the tracker's sequential chain
    LMOT_CUDA(c, cudaStreamWaitEvent(c->pub_stream, r->ev_tc, 0));
    if ((rc = tracker_publish(c, r, c->pub_stream))) return rc;
    LMOT_CUDA(c, cudaEventRecord(r->ev_done, c->pub_stream));
  }
  return LMOT_OK;
}

// ground lines: the slot's ground grid, allocated on its first frame with lines on
int lines_ensure(Ctx* c, Slot* s) {
  if (!s->d_gz) LMOT_CUDA(c, cudaMalloc(&s->d_gz, kPolarCells * sizeof(float)));
  return LMOT_OK;
}

// ---- batched ticks: F sensor streams, one frame each, ONE track table (BASELINE.json configs[3]) -------------------------
// Their own detection slots (allocated on first use, two banks of F so that the detection of tick t+1 overlaps the tracker of
// tick t); a bank's kernels all run on its first slot's stream.  `bank` is a pseudo-slot: the concatenated box list, its
// counters, the detection semaphore and the events the tracker hand-over needs.
int slot_create(Ctx* c, Slot* s, int index);
void slot_destroy(Slot* s);

// the banks' pseudo-slots (once per context); the caller synchronises the device afterwards
int bank_ensure(Ctx* c) {
  for (int b = 0; b < kBatchBanks; ++b) {
    Slot* k = &c->bank[b];
    if (k->d_boxes) continue;
    k->index = 2000 + b;
    LMOT_CUDA(c, cudaMalloc(&k->d_boxes, (size_t)c->prm.max_boxes * 24 * sizeof(float)));
    LMOT_CUDA(c, cudaMalloc(&k->d_boxes_g, (size_t)c->prm.max_boxes * 24 * sizeof(float)));
    LMOT_CUDA(c, cudaMalloc(&k->d_counters, CNT_COUNT * sizeof(int)));
    LMOT_CUDA(c, cudaMemset(k->d_counters, 0, CNT_COUNT * sizeof(int)));
    LMOT_CUDA(c, cudaMalloc(&k->d_det_sem, sizeof(int)));
    LMOT_CUDA(c, cudaMemset(k->d_det_sem, 0, sizeof(int)));
    LMOT_CUDA(c, cudaMalloc(&k->d_deskew, kMaxBatch * kDeskewTabBytes));
    LMOT_CUDA(c, cudaMalloc(&k->d_area, kMaxBatch * sizeof(AreaBlock)));
    LMOT_CUDA(c, cudaEventCreateWithFlags(&k->ev_det_done, cudaEventDisableTiming));
    LMOT_CUDA(c, cudaEventCreateWithFlags(&k->ev_trk_done, cudaEventDisableTiming));
    LMOT_CUDA(c, cudaEventCreateWithFlags(&k->ev_fork, cudaEventDisableTiming));
    LMOT_CUDA(c, cudaEventRecord(k->ev_trk_done, c->stream));
    LMOT_CUDA(c, cudaEventRecord(k->ev_det_done, c->stream));
    LMOT_CUDA(c, cudaStreamCreateWithFlags(&k->stream, cudaStreamNonBlocking));
    k->res = &c->results[0];
  }
  return LMOT_OK;
}

int batch_ensure(Ctx* c, int F) {
  if (F <= c->batch_frames) return LMOT_OK;
  // (re)allocate for the larger batch: nothing of the old banks may be in flight
  for (int i = 0; i < c->n_bslots; ++i) LMOT_CUDA(c, cudaStreamSynchronize(c->bslots[i].stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->trk_stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->pub_stream));
  for (int i = c->n_bslots; i < kBatchBanks * F; ++i) {
    int rc = slot_create(c, &c->bslots[i], 1000 + i);
    if (rc) return rc;
    c->n_bslots = i + 1;
  }
  int rc = bank_ensure(c);
  if (rc) return rc;
  LMOT_CUDA(c, cudaDeviceSynchronize());
  c->batch_frames = F;
  return LMOT_OK;
}

void batch_destroy(Ctx* c) {
  for (int i = 0; i < c->n_bslots; ++i) slot_destroy(&c->bslots[i]);
  for (int b = 0; b < kBatchBanks; ++b) {
    Slot* k = &c->bank[b];
    cudaFree(k->d_boxes); cudaFree(k->d_boxes_g); cudaFree(k->d_counters); cudaFree(k->d_det_sem); cudaFree(k->d_deskew); cudaFree(k->d_area);
    if (k->ev_det_done) cudaEventDestroy(k->ev_det_done);
    if (k->ev_trk_done) cudaEventDestroy(k->ev_trk_done);
    if (k->ev_fork) cudaEventDestroy(k->ev_fork);
    if (k->stream) cudaStreamDestroy(k->stream);
  }
}

// the merge units of a merging stream (StreamCfg::merge_unit, one per bank), allocated on first use (one device synchronisation, as
// batch_ensure).  All or nothing: a failed allocation frees the whole set, so a later submission retries from scratch instead of finding
// a half-built one.
int merge_ensure(Ctx* c, Slot* units, int index) {
  bool ready = true;
  for (int b = 0; b < kBatchBanks; ++b) ready &= merge_unit_ready(&units[b]);
  if (ready) return LMOT_OK;
  int rc = LMOT_OK;
  for (int b = 0; b < kBatchBanks && rc == LMOT_OK; ++b)
    if (!merge_unit_ready(&units[b])) rc = merge_unit_create(c, &units[b], index + b);
  if (rc == LMOT_OK && cudaDeviceSynchronize() != cudaSuccess) rc = LMOT_ERR_CUDA;
  if (rc) {
    cudaDeviceSynchronize();           // (the allocators' memsets) before the buffers go back
    for (int b = 0; b < kBatchBanks; ++b) merge_unit_destroy(&units[b]);
  }
  return rc;
}

// ---- the detection front end: frames -> box-fitted units ---------------------------------------------------------------------------
// A submission's frames come in groups, one per stream: a single-stream frame (lmot_frame*, lmot_detect_dev) and a batched tick are one
// group (the context's own settings and fold), a sequence tick has one per FRAMES sequence.  Frame j of a group of sensors is its sensor
// j's; a single-stream frame ignores the stream's sensor table.
struct DetGroup {
  StreamCfg* cfg;                      // the stream's settings and merge units
  const TrackerHost* th;               // the fold the frames' motion is taken from (nullptr: frames without a stamp, never deskewed)
  const float* const* data;            // nf frames (host: stride floats per point; device: float4) of n[j] points
  const int* n;
  int nf;
  double ts, v, yaw;
  int* fc;                             // device view of the stream's per-frame counts in its result block (nullptr: none are written)
  Result* res = nullptr;               // the stream's result block (sweep accumulation: its candidates and count rows)
  bool sensors = false;                // the frames are the stream's sensors: its sensor table and merging apply
  bool tab() const { return sensors && cfg->n_sensors > 0; }
  bool merges() const { return sensors && cfg->merges(); }
};

// what the front end box-fitted, by group: group g's units are u[f0[g] .. f0[g + 1]) (its frames, or its merge unit), unit i with pose
// rig[i], which applies to its boxes iff rig_on[g]; the concatenation writes the group's count rows from fc[g] on
struct DetUnits {
  Slot* u[kMaxBatch];
  lmot_sensor rig[kMaxBatch];
  int f0[kMaxBatch + 1];
  bool rig_on[kMaxBatch];
  int* fc[kMaxBatch];
};

// G groups of frames on the consecutive detection slots fr[0 ..], in group order, all on stream st, for the staging slot's result block
// (stage->res).  The staging slot holds the deskew tables and area blocks the launches read and records the kernel events: a batch
// bank's pseudo-slot (bank b: its merge units), or a single-stream frame's own slot.  Staging (host frames uploaded, device frames read
// in place), deskew (tables into the pinned block h_dsk, one copy, one launch), ground removal, the merging groups' elevated clouds into
// their merge units, clustering, box fitting.  post_sem: every unit's last box-fitting CTA posts the unit's semaphore (nothing
// concatenates its list).
//   Ground removal gets the submission's pose table iff some group has a sensor table, box fitting iff some unit is an unmerged frame of
// such a group (a frame without a table: lmot_default_sensor); both get per-frame detection values iff some group has its own (sensor
// values folded in).  A merge unit is the vehicle's cloud: identity pose, the group's detection values without a sensor's, at most
// max_points points.  Clustering runs in the ground kernel's tail (fuse_ccl) unless a group masks, accumulates, layers or merges.  With
// one frame and nothing but the plain path on, these are the launches of the frame pipeline (F == 1 variants).
//   Detection areas: a group whose stream has one stages it into the pinned block h_area[i] (i-th masked group) -- one copy, one launch for
// every masked unit's cell mask (unit pose: the merge unit's identity, else U.rig); clustering then runs as its own launch, and the
// masked units cluster and box-fit through the masking kernel variants.
int detect_front(Ctx* c, Slot* stage, Slot* fr, cudaStream_t st, int b, const DetGroup* g, int G, int stride, bool host, float* h_dsk,
                 AreaBlock* h_area, bool post_sem, DetUnits& U) {
  int rc;
  Slot* sl[kMaxBatch];
  const float4* pp[kMaxBatch];
  int nn[kMaxBatch], F = 0, nj = 0;
  lmot_sensor rig[kMaxBatch];
  DeskewJob dj[kMaxBatch];
  bool rigged = false, own_det = false, merging = false;
  fr[0].res = stage->res;              // (kernel_mark)
  for (int d = 0; d < G; ++d) {
    const StreamCfg& q = *g[d].cfg;
    const bool tab = g[d].tab(), dsk = q.deskews(g[d].th != nullptr);
    rigged |= tab; own_det |= q.det_on; merging |= g[d].merges();
    const double om = dsk ? deskew_omega(*g[d].th, g[d].ts, g[d].v, g[d].yaw) : 0.0, vv = std::isfinite(g[d].v) ? g[d].v : 0.0;
    for (int j = 0; j < g[d].nf; ++j, ++F) {
      Slot* s = sl[F] = &fr[F];
      nn[F] = g[d].n[j];
      if (tab) rig[F] = q.sensors[j];
      else lmot_default_sensor(&c->prm, &rig[F]);
      pp[F] = s->d_points;
      if (dsk) {                       // the frame with its sensor's mount and its stream's fold
        const float* raw = g[d].data[j];
        if (host && (rc = deskew_stage_host(c, s, st, g[d].data[j], nn[F], stride, &raw))) return rc;
        deskew_table(q.deskew, vv, om, tab ? &q.sensors[j] : nullptr, h_dsk + (size_t)F * kDeskewTab);
        if (nn[F] > 0) dj[nj++] = DeskewJob{raw, s->d_points, stage->d_deskew + (size_t)F * kDeskewTab, nn[F], host ? stride : 4, q.deskew};
      } else if (host) {
        if ((rc = upload_points(c, s, st, g[d].data[j], nn[F], stride, s->d_points))) return rc;
      } else {
        pp[F] = reinterpret_cast<const float4*>(g[d].data[j]);
      }
    }
  }
  if (nj > 0) {                        // frame i's table at table i of the staging slot
    LMOT_CUDA(c, cudaMemcpyAsync(stage->d_deskew, h_dsk, (size_t)F * kDeskewTabBytes, cudaMemcpyHostToDevice, st));
    if ((rc = deskew_launch(c, st, dj, nj))) return rc;
  }
  // per-frame detection values and the units (copied into the launch parameters: later setting changes leave this tick alone)
  const lmot_detect_params base = detect_params_of(c->prm);
  lmot_detect_params det[kMaxBatch], udet[kMaxBatch];
  Slot* src[kMaxBatch];
  Slot* mu[kMaxBatch];
  lmot_sensor mpose[kMaxBatch];
  int mn[kMaxBatch], ms0[kMaxBatch + 1], *mfc[kMaxBatch], unn[kMaxBatch], nm = 0, nsrc = 0, nu = 0;
  float mroi[kMaxBatch];
  bool rig_fit = false;
  ms0[0] = 0;
  for (int d = 0, i0 = 0; d < G; i0 += g[d].nf, ++d) {
    StreamCfg& q = *g[d].cfg;
    const lmot_detect_params& vd = q.det_on ? q.det : base;
    if (own_det)
      for (int i = i0; i < i0 + g[d].nf; ++i) {
        det[i] = vd;
        if (g[d].tab()) {
          const lmot_sensor& s = rig[i];
          det[i].h_sensor = s.h_sensor; det[i].t_hmin = s.t_hmin; det[i].t_hmax = s.t_hmax; det[i].sensor_height = s.sensor_height;
        }
      }
    U.f0[d] = nu;
    U.rig_on[d] = g[d].tab() && !g[d].merges();
    U.fc[d] = g[d].fc;
    if (g[d].merges()) {
      long long tot = 0;
      for (int i = i0; i < i0 + g[d].nf; ++i) { src[nsrc] = sl[i]; mpose[nsrc] = rig[i]; mn[nsrc] = nn[i]; ++nsrc; tot += nn[i]; }
      mu[nm] = &q.merge_unit[b]; mfc[nm] = g[d].fc; mroi[nm] = vd.roi_m;
      ms0[++nm] = nsrc;
      U.u[nu] = mu[nm - 1];
      lmot_default_sensor(&c->prm, &U.rig[nu]);
      udet[nu] = vd;
      unn[nu] = (int)(tot < c->max_points ? tot : c->max_points);
      ++nu;
      U.fc[d] += 4 * g[d].nf;         // behind the sensors' rows, which rig_merge_kernel writes
    } else {
      for (int i = i0; i < i0 + g[d].nf; ++i) { U.u[nu] = sl[i]; U.rig[nu] = rig[i]; if (own_det) udet[nu] = det[i]; unn[nu] = nn[i]; ++nu; }
      rig_fit |= U.rig_on[d];
    }
  }
  U.f0[G] = nu;
  AreaJob aj[kMaxBatch];
  const unsigned* amask[kMaxBatch] = {};
  int na = 0, nblk = 0;
  for (int d = 0; d < G; ++d) {
    const StreamCfg& q = *g[d].cfg;
    if (!q.masked()) continue;
    if ((rc = area_ensure(c, stage, G))) return rc;        // (a bank's kMaxBatch blocks come with it: bank_ensure)
    h_area[nblk] = q.area;
    const float roi = (q.det_on ? q.det : base).roi_m;
    for (int i = U.f0[d]; i < U.f0[d + 1]; ++i) {
      if ((rc = area_ensure(c, U.u[i], 0))) return rc;
      aj[na] = AreaJob{stage->d_area + nblk, U.u[i]->d_area_mask, {}, roi};
      memcpy(aj[na++].pose, U.rig[i].pose, sizeof(aj[0].pose));
      amask[i] = U.u[i]->d_area_mask;
    }
    ++nblk;
  }
  if (nblk > 0) {
    LMOT_CUDA(c, cudaMemcpyAsync(stage->d_area, h_area, (size_t)nblk * sizeof(AreaBlock), cudaMemcpyHostToDevice, st));
    if ((rc = area_launch(c, st, aj, na))) return rc;
  }
  const unsigned* const* area = nblk > 0 ? amask : nullptr;
  // sweep accumulation: a group with a stamp whose stream accumulates -- its units' candidates and jobs (accumulate.cu), one launch for
  // every accumulating unit behind the ground kernel and the rig merge; clustering then runs as its own launch
  AccJob acj[kMaxBatch];
  AccHist* ach[kMaxBatch];
  int nacj = 0, nach = 0;
  for (int d = 0; d < G; ++d) {
    StreamCfg& q = *g[d].cfg;
    if (!g[d].th || !q.acc.on()) continue;
    const int u0 = U.f0[d], nu_d = U.f0[d + 1] - u0;
    const int kind = g[d].merges() ? ACC_MERGE : g[d].tab() ? ACC_RIG : ACC_FRAME;
    const float roi = (q.det_on ? q.det : base).roi_m;
    float rois[kMaxBatch];
    for (int i = 0; i < nu_d; ++i) rois[i] = roi;
    if ((rc = accumulate_step(c, q.acc, kind, nu_d, U.u + u0, U.rig + u0, rois, unn + u0, *g[d].th, g[d].ts, g[d].v, g[d].yaw, g[d].res,
                              acj + nacj, unn + u0))) return rc;
    nacj += nu_d;
    ach[nach++] = &q.acc;
  }
  // layered clustering: the units of a stream with layers on cluster in layers_launch (sensor_height: the unit's box-fitting value), the
  // others in ccl_launch_batch; box fitting reads the layered units' run tables
  LayerUnit lu[kMaxBatch];
  LayerTab ltab[kMaxBatch];
  Slot* cu[kMaxBatch];
  const unsigned* camask[kMaxBatch];
  int nl = 0, ncu = 0;
  bool layering = false;
  for (int d = 0; d < G; ++d) layering |= g[d].cfg->layers.on != 0;
  for (int d = 0; layering && d < G; ++d) {
    const StreamCfg& q = *g[d].cfg;
    for (int i = U.f0[d]; i < U.f0[d + 1]; ++i) {
      ltab[i] = LayerTab{};
      if (!q.layers.on) { cu[ncu] = U.u[i]; camask[ncu++] = amask[i]; continue; }
      if ((rc = layers_ensure(c, U.u[i], st))) return rc;
      lu[nl++] = LayerUnit{U.u[i], amask[i], q.layers, own_det ? udet[i].sensor_height : U.rig[i].sensor_height, unn[i]};
      ltab[i] = layer_tab_of(U.u[i]);
    }
  }
  const bool fuse = c->fuse_ccl && !merging && nblk == 0 && nacj == 0 && !layering;
  // ground lines: a frame whose stream has them on gets its slot's ground grid; its unit (an unmerged frame) measures boxes from it
  GroundLinesJob lj[kMaxBatch];
  const float* ugz[kMaxBatch] = {};
  bool lining = false;
  for (int d = 0, i0 = 0; d < G; i0 += g[d].nf, ++d) {
    const lmot_ground_lines* gl = g[d].cfg->lines_on();
    for (int i = i0; i < i0 + g[d].nf; ++i) {
      if (gl && (rc = lines_ensure(c, sl[i]))) return rc;
      lj[i] = GroundLinesJob{gl, sl[i]->d_gz};
    }
    if (gl && !g[d].merges())
      for (int i = U.f0[d]; i < U.f0[d + 1]; ++i) ugz[i] = U.u[i]->d_gz;
    lining |= gl != nullptr;
  }
  // box search: each unit takes its stream's setting (into the launch parameters, as the detection values)
  int usearch[kMaxBatch];
  bool searching = false;
  for (int d = 0; d < G; ++d)
    for (int i = U.f0[d]; i < U.f0[d + 1]; ++i) { usearch[i] = g[d].cfg->search_angles(); searching |= usearch[i] > 0; }
  Result* r = stage->res;
  if (c->timing) cudaEventRecord(r->ev[0], st);
  if ((rc = ground_launch_batch(c, sl, F, pp, nn, st, true, false, fuse, false, rigged ? rig : nullptr, own_det ? det : nullptr,
                                lining ? lj : nullptr))) return rc;
  if (c->timing) cudaEventRecord(r->ev[1], st);
  if (nm > 0 && (rc = rig_merge_launch(c, st, src, mpose, mn, nm, ms0, mu, mfc, mroi))) return rc;
  if (nacj > 0 && (rc = accumulate_launch(c, st, stage, acj, nacj, ach, nach))) return rc;
  if (!layering) {
    if (!fuse && (rc = ccl_launch_batch(c, U.u, nu, st, area))) return rc;
  } else {
    if ((rc = layers_launch(c, st, lu, nl, stage))) return rc;
    if (ncu > 0 && (rc = ccl_launch_batch(c, cu, ncu, st, area ? camask : nullptr))) return rc;
  }
  if (c->timing) cudaEventRecord(r->ev[2], st);
  if ((rc = boxfit_launch_batch(c, U.u, nu, st, unn, post_sem, rig_fit ? U.rig : nullptr, own_det ? udet : nullptr, area, searching ? usearch : nullptr,
                                lining ? ugz : nullptr, layering ? ltab : nullptr))) return rc;
  // obstacle footprints: every unit of a stream with obstacles on, in one launch behind box fitting, into its group's result block (unit
  // i - f0 of the group)
  ObsUnit ou[kMaxBatch];
  int no = 0;
  for (int d = 0; d < G; ++d) {
    const StreamCfg& q = *g[d].cfg;
    if (!q.obs.on) continue;
    const float roi = (q.det_on ? q.det : base).roi_m;
    for (int i = U.f0[d]; i < U.f0[d + 1]; ++i) ou[no++] = ObsUnit{U.u[i], roi, q.obs.max_vertices, g[d].res, i - U.f0[d]};
  }
  if (no > 0 && ((rc = obstacles_ensure(c, ou, no, st)) || (rc = obstacles_launch(c, st, ou, no, stage)))) return rc;
  return LMOT_OK;
}

// what the debug getters read of the most recent own-stream submission: its units' cell masks and layer tables, its frames' ground grids
// (none where the setting was off), and the units' area_last / layers_last (lmot_cluster_outputs, lmot_debug_label_grid)
void own_debug_note(Ctx* c, Slot* fr, int nf, const DetUnits& U) {
  const StreamCfg& q = c->own.cfg;
  const int nu = U.f0[1];
  c->n_area_dbg = q.masked() ? nu : 0;
  c->n_lay_dbg = q.layers.on ? nu : 0;
  c->n_gz_dbg = q.lines.on ? nf : 0;
  for (int i = 0; i < nu; ++i) {
    c->area_dbg[i] = U.u[i]->d_area_mask;
    c->lay_dbg[i] = U.u[i];
    U.u[i]->area_last = q.masked();
    U.u[i]->layers_last = q.layers.on != 0;
  }
  for (int i = 0; i < nf; ++i) c->gz_dbg[i] = fr[i].d_gz;
}

// the asynchronous single-stream frame: the detection front end on the frame's slot (its staging slot and only frame, on its stream),
// then the tracker on the tracker stream.  points: n host records of `stride` floats (host), or a device float4 frame
int submit(Ctx* c, Slot* s, Result* r, const float* points, int n, int stride, bool host, bool with_tracker, double ts, double v, double yaw) {
  int rc;
  struct Tail { Ctx* c; double t0; ~Tail() { c->host_ns[0] += now_ns() - t0; } } tail{c, now_ns()};
  s->res = r;
  r->n_kev = 0;
  r->batch_frames = 0;
  // the slot's previous boxes / counters must have been consumed by the tracker
  LMOT_CUDA(c, cudaStreamWaitEvent(s->stream, s->ev_trk_done, 0));
  const bool gf = with_tracker && c->prm.global_frame;
  const DetGroup g{&c->own.cfg, with_tracker ? &c->own.trk.th : nullptr, &points, &n, 1, ts, v, yaw, nullptr, r, false};
  DetUnits U;
  // with_tracker: the slot's last box-fitting CTA posts its detection semaphore (global_frame: boxes_to_global_kernel does)
  if ((rc = detect_front(c, s, s, s->stream, 0, &g, 1, stride, host, r->h_deskew, r->h_area, with_tracker && !gf, U))) return rc;
  own_debug_note(c, s, 1, U);
  if (gf && (rc = boxes_to_global_launch(c, s, s->stream, s->d_boxes, s->d_counters, ts, v, yaw, true))) return rc;
  if (c->timing) cudaEventRecord(r->ev[3], s->stream);
  LMOT_CUDA(c, cudaEventRecord(s->ev_det_done, s->stream));
  if (with_tracker) {
    if ((rc = submit_tracker(c, s, r, s->d_boxes, s->d_counters, ts, v, yaw))) return rc;
  } else {
    // no spawn_output_kernel will snapshot the counters / boxes: copy them before the slot is reused
    LMOT_CUDA(c, cudaMemcpyAsync(r->h_det, s->d_counters, CNT_COUNT * sizeof(int), cudaMemcpyDeviceToHost, s->stream));
    if ((rc = boxes_publish(c, s, r, s->stream))) return rc;
    LMOT_CUDA(c, cudaEventRecord(s->ev_trk_done, s->stream));
    LMOT_CUDA(c, cudaEventRecord(r->ev_done, s->stream));
  }
  r->has_tracks = with_tracker;
  if (!r->in_flight) { r->in_flight = true; ++c->n_in_flight; }
  return LMOT_OK;
}

// the IDs of a result being returned (lmot_track_ids): copied now, the block is reused by later submissions
void note_ids(Tracker& t, const Result* r) {
  const int T = r->h_hdr[HDR_N_TRACKS];
  t.ids_n = T;
  t.ids_rows = !r->ids;
  if (r->ids) t.ids_last.assign(r->h_ids, r->h_ids + T);
}

int copy_track_outputs(const Result* s, lmot_track_out* out) {
  const int T = s->h_hdr[HDR_N_TRACKS], nv = s->h_hdr[HDR_N_VIS];
  if (!out) return LMOT_OK;
  out->n_tracks = T; out->n_vis = nv;
  const int n = T < out->cap ? T : out->cap;
  const int nvc = nv < out->cap ? nv : out->cap;
  if (n > 0) {
    if (out->targets) memcpy(out->targets, s->h_targets, (size_t)n * 3 * sizeof(float));
    if (out->vandyaw) memcpy(out->vandyaw, s->h_vandyaw, (size_t)n * 2 * sizeof(double));
    if (out->track_manage) memcpy(out->track_manage, s->h_manage, (size_t)n * sizeof(int));
    if (out->is_static) memcpy(out->is_static, s->h_static, (size_t)n);
    if (out->is_vis) memcpy(out->is_vis, s->h_vis, (size_t)n);
  }
  if (nvc > 0 && out->vis_bb) memcpy(out->vis_bb, s->h_visbb, (size_t)nvc * 24 * sizeof(float));
  const bool wants = out->targets || out->vandyaw || out->track_manage || out->is_static || out->is_vis || out->vis_bb;
  return (wants && T > out->cap) ? LMOT_ERR_CAPACITY : LMOT_OK;      // a zero-initialised lmot_track_out asks for the counts only
}

// results of a finished frame from its pinned host block; `s`: the stream whose step the block holds
int collect_result(Ctx* c, Result* r, lmot_frame_out* out, Stream& s) {
  const double t0 = now_ns();
  LMOT_CUDA(c, cudaEventSynchronize(r->ev_done));
  const double t1 = now_ns();
  c->host_ns[1] += t1 - t0; c->host_ns[3] += 1;
  struct Tail { Ctx* c; double t1; ~Tail() { c->host_ns[2] += now_ns() - t1; } } tail{c, t1};
  if (c->timing && r->has_tracks) {
    for (int i = 0; i < 4; ++i) cudaEventElapsedTime(&c->stage_ms[i], r->ev[i], r->ev[i + 1]);
    c->n_kernel_ms = r->n_kev;
    for (int i = 0; i < r->n_kev; ++i) cudaEventElapsedTime(&c->kernel_ms[i], i == 0 ? r->ev[0] : r->kev[i - 1], r->kev[i]);
  }
  if (!r->has_tracks) {   // detect only: no kernel wrote the header
    r->h_hdr[HDR_N_ELEV] = r->h_det[CNT_N_ELEV]; r->h_hdr[HDR_N_GROUND] = r->h_det[CNT_N_GROUND];
    r->h_hdr[HDR_NUM_CLUSTER] = r->h_det[CNT_NUM_CLUSTER]; r->h_hdr[HDR_N_BOXES] = r->h_det[CNT_N_BOXES];
    r->h_hdr[HDR_N_TRACKS] = 0; r->h_hdr[HDR_N_VIS] = 0; r->h_hdr[HDR_ERROR] = r->h_det[CNT_ERROR]; r->h_hdr[HDR_WARN] = 0;
  }
  if (r->merge_rows > 0) {
    // merging rig: row 0 takes the merged cloud's num_cluster / n_boxes (written behind the sensors' rows); n_elevated is the sensors'
    // sum (the merged cloud's length is that, or max_points where it was cut)
    int* fc = r->h_frame_counts;
    const int F = r->merge_rows;
    fc[2] = fc[4 * F + 2]; fc[3] = fc[4 * F + 3];
    int ne = 0;
    for (int j = 0; j < F; ++j) ne += fc[4 * j];
    r->h_hdr[HDR_N_ELEV] = ne;
  }
  if (r->acc_units > 0 && r->merge_rows == 0) {
    // accumulating units: clustering counted E_acc, n_elevated is each frame's own (a merge unit's rows are the sensors' already)
    if (r->batch_frames > 0) {
      for (int u = 0; u < r->acc_units; ++u) {
        r->h_hdr[HDR_N_ELEV] -= r->h_frame_counts[4 * u] - r->h_acc[4 * u + 2];
        r->h_frame_counts[4 * u] = r->h_acc[4 * u + 2];
      }
    } else {
      r->h_hdr[HDR_N_ELEV] = r->h_acc[2];
    }
  }
  {                                                   // lmot_accumulate_info / lmot_seq_accumulate_info: what this result used
    lmot_accum_info& ai = s.acc_info;
    memset(&ai, 0, sizeof(ai));
    ai.n_units = r->acc_units;
    for (int u = 0; u < r->acc_units; ++u) {
      const int used = r->h_acc[4 * u + 1] < r->acc_cand ? r->h_acc[4 * u + 1] : r->acc_cand;
      ai.sweeps_used[u] = used;
      ai.n_points[u] = r->h_acc[4 * u];
      for (int j = 0; j < used; ++j) {
        ai.stamp_us[u][j] = r->acc_ts[j];
        memcpy(ai.pose[u][j], r->acc_pose[u][j], sizeof(ai.pose[u][j]));
      }
    }
  }
  {                                                   // lmot_obstacles_result / lmot_seq_obstacles_result: this result's footprints
    const int rc = obstacles_collect(c, r, s.obs_last);
    if (rc) return rc;
  }
  const int err = r->h_hdr[HDR_ERROR];
  const int warn = r->has_tracks ? r->h_hdr[HDR_WARN] : 0;
  if (r->has_tracks) {
    s.trk.last_n_act = r->h_hdr[HDR_N_ACT];
    note_ids(s.trk, r);
  }
  if (out) {
    out->n_elevated = r->h_hdr[HDR_N_ELEV]; out->n_ground = r->h_hdr[HDR_N_GROUND];
    out->num_cluster = r->h_hdr[HDR_NUM_CLUSTER]; out->n_boxes = r->h_hdr[HDR_N_BOXES];
    const int nb = out->n_boxes < out->max_boxes ? out->n_boxes : out->max_boxes;
    if (out->boxes && nb > 0) memcpy(out->boxes, r->h_boxes, (size_t)nb * 24 * sizeof(float));
    const int rc = copy_track_outputs(r, &out->tracks);
    if (rc && !err) return rc;
  }
  return err ? err : warn;      // warn > 0 (LMOT_WARN_*): the outputs are valid
}

int result_create(Ctx* c, Result* r) {
  const int TC = c->prm.max_tracks, MB = c->prm.max_boxes;
  const unsigned fl = cudaHostAllocMapped;
  LMOT_CUDA(c, cudaHostAlloc(&r->h_hdr, HDR_COUNT * sizeof(int) + 16, fl));
  memset(r->h_hdr, 0, HDR_COUNT * sizeof(int));
  LMOT_CUDA(c, cudaHostAlloc(&r->h_det, CNT_COUNT * sizeof(int), fl));
  memset(r->h_det, 0, CNT_COUNT * sizeof(int));
  LMOT_CUDA(c, cudaHostAlloc(&r->h_frame_counts, 4 * (kMaxBatch + 1) * sizeof(int), fl));   // + the merged cloud's row (merge_rows)
  memset(r->h_frame_counts, 0, 4 * (kMaxBatch + 1) * sizeof(int));
  LMOT_CUDA(c, cudaHostAlloc(&r->h_boxes, (size_t)MB * 24 * sizeof(float) + 16, fl));
  // + 16 bytes: spawn_output_kernel writes whole 16-byte words
  LMOT_CUDA(c, cudaHostAlloc(&r->h_targets, (size_t)TC * 3 * sizeof(float) + 16, fl));
  LMOT_CUDA(c, cudaHostAlloc(&r->h_vandyaw, (size_t)TC * 2 * sizeof(double) + 16, fl));
  LMOT_CUDA(c, cudaHostAlloc(&r->h_manage, (size_t)TC * sizeof(int) + 16, fl));
  LMOT_CUDA(c, cudaHostAlloc(&r->h_static, (size_t)TC + 16, fl));
  LMOT_CUDA(c, cudaHostAlloc(&r->h_vis, (size_t)TC + 16, fl));
  LMOT_CUDA(c, cudaHostAlloc(&r->h_visbb, (size_t)TC * 24 * sizeof(float) + 16, fl));
  LMOT_CUDA(c, cudaHostAlloc(&r->h_ids, ((size_t)TC + 2) * sizeof(long long), fl));
  LMOT_CUDA(c, cudaMalloc(&r->d_ids, ((size_t)TC + 2) * sizeof(long long)));
  {   // device copy of the block, one allocation, every array 256-byte aligned with 16 bytes of slack
    auto al = [](size_t b) { return (b + 16 + 255) & ~(size_t)255; };
    const size_t sz[8] = {al(HDR_COUNT * sizeof(int)), al((size_t)MB * 96), al((size_t)TC * 12), al((size_t)TC * 16), al((size_t)TC * 4),
                          al((size_t)TC), al((size_t)TC), al((size_t)TC * 96)};
    size_t tot = 0;
    for (size_t b : sz) tot += b;
    LMOT_CUDA(c, cudaMalloc(&r->d_block, tot));
    LMOT_CUDA(c, cudaMemsetAsync(r->d_block, 0, tot, c->stream));
    unsigned char* p = r->d_block;
    r->d_hdr = (int*)p; p += sz[0]; r->d_boxes = (float*)p; p += sz[1]; r->d_targets = (float*)p; p += sz[2];
    r->d_vandyaw = (double*)p; p += sz[3]; r->d_manage = (int*)p; p += sz[4]; r->d_static = p; p += sz[5]; r->d_vis = p; p += sz[6];
    r->d_visbb = (float*)p;
  }
  LMOT_CUDA(c, cudaEventCreateWithFlags(&r->ev_tc, cudaEventDisableTiming));
  LMOT_CUDA(c, cudaEventCreateWithFlags(&r->ev_done, cudaEventDisableTiming));
  LMOT_CUDA(c, cudaEventRecord(r->ev_done, c->stream));
  for (int i = 0; i < 5; ++i) LMOT_CUDA(c, cudaEventCreate(&r->ev[i]));
  for (int i = 0; i < kMaxKernelEvents; ++i) LMOT_CUDA(c, cudaEventCreate(&r->kev[i]));
  return LMOT_OK;
}

void result_destroy(Result* r) {
  if (r->h_hdr) cudaFreeHost(r->h_hdr);
  if (r->h_det) cudaFreeHost(r->h_det);
  if (r->h_frame_counts) cudaFreeHost(r->h_frame_counts);
  if (r->h_boxes) cudaFreeHost(r->h_boxes);
  if (r->h_targets) cudaFreeHost(r->h_targets);
  if (r->h_vandyaw) cudaFreeHost(r->h_vandyaw);
  if (r->h_manage) cudaFreeHost(r->h_manage);
  if (r->h_static) cudaFreeHost(r->h_static);
  if (r->h_vis) cudaFreeHost(r->h_vis);
  if (r->h_visbb) cudaFreeHost(r->h_visbb);
  if (r->h_ids) cudaFreeHost(r->h_ids);
  if (r->h_deskew) cudaFreeHost(r->h_deskew);
  if (r->h_area) cudaFreeHost(r->h_area);
  if (r->h_acc) cudaFreeHost(r->h_acc);
  obstacles_result_free(r);
  if (r->d_ids) cudaFree(r->d_ids);
  if (r->d_block) cudaFree(r->d_block);
  if (r->ev_tc) cudaEventDestroy(r->ev_tc);
  if (r->ev_done) cudaEventDestroy(r->ev_done);
  for (int i = 0; i < 5; ++i) if (r->ev[i]) cudaEventDestroy(r->ev[i]);
  for (int i = 0; i < kMaxKernelEvents; ++i) if (r->kev[i]) cudaEventDestroy(r->kev[i]);
}

// what a stream holds on the device and in pinned memory (track table, merge units, accumulation history), then its record back to the
// defaults
void stream_free(Stream& s) {
  tracker_free(s.trk);
  ego_free(s.ego);
  for (int b = 0; b < kBatchBanks; ++b) merge_unit_destroy(&s.cfg.merge_unit[b]);
  accumulate_free(s.cfg.acc);
  s = Stream{};
}

// ---- independent sequences (lmot_seq_*): S frame streams, one or more frames each per tick, S track tables ---------------------------
// Detection runs on the batch banks (batch_ensure).  Without sensor tables the box lists are NOT concatenated: a FRAMES sequence's tracker
// reads its detection slot's own list and counters (seq_tick_common's map).  With a table among the tick's FRAMES sequences,
// concat_boxes_seq_kernel concatenates each of their frames into that sequence's list on the bank (seq_meas) and the tracker reads those.
void seq_destroy(Ctx* c) {
  for (int k = 0; k < kMaxBatch; ++k) stream_free(c->seq[k]);
  for (int b = 0; b < kBatchBanks; ++b)
    for (int k = 0; k < kMaxBatch; ++k) {
      SeqMeas& m = c->seq_meas[b][k];
      cudaFree(m.d_boxes); cudaFree(m.d_boxes_g); cudaFree(m.d_counters); cudaFree(m.d_det_sem);
      m = SeqMeas{};
    }
  for (int b = 0; b < kBatchBanks; ++b) { cudaFree(c->seq_stage[b]); c->seq_stage[b] = nullptr; }
  for (int i = 0; i < c->seq_ring; ++i) {
    for (int k = 0; k < c->n_seq; ++k) result_destroy(&c->seq_ticks[i].blocks[k]);
    if (c->seq_ticks[i].h_deskew) cudaFreeHost(c->seq_ticks[i].h_deskew);
    if (c->seq_ticks[i].h_area) cudaFreeHost(c->seq_ticks[i].h_area);
  }
  delete[] c->seq_ticks;
  c->seq_ticks = nullptr; c->seq_last = nullptr; c->seq_stepped = 0;
  c->n_seq = 0; c->seq_ring = 0; c->seq_next = 0; c->seq_oldest = 0; c->seq_in_flight = 0;
}

// uncollected sequence ticks are dropped (after drain(): nothing is running)
void seq_forget(Ctx* c) {
  for (int i = 0; i < c->seq_ring; ++i) c->seq_ticks[i].in_flight = false;
  c->seq_in_flight = 0;
  c->seq_oldest = c->seq_next;
}

// The stream an entry point addresses: the context's own (k == kOwnStream, the lmot_X forms) or sequence k (the lmot_seq_X forms,
// 0 <= k < n_seq); nullptr for any other k and for a null context.  kOwnStream lies outside int: no k a caller passes names the own stream.
constexpr long long kOwnStream = -(1LL << 32);

Stream* stream_at(lmot_ctx* ctx, long long k) {
  if (!ctx) return nullptr;
  Ctx* c = &ctx->c;
  if (k == kOwnStream) return &c->own;
  return k >= 0 && k < c->n_seq ? &c->seq[k] : nullptr;
}

const Stream* stream_at(const lmot_ctx* ctx, long long k) { return stream_at(const_cast<lmot_ctx*>(ctx), k); }

// The pinned host blocks stream k's submissions stage from, at entry i of its ring (the setters that turn a feature on allocate them):
// deskew tables and detection-area blocks (area_blocks of them) of the own stream's result block i / of sequence tick i, and the
// accumulation count rows of the stream's result block there
struct RingPins { float** deskew; AreaBlock** area; int area_blocks; int** acc; };

int ring_size(const Ctx* c, long long k) { return k == kOwnStream ? c->n_results : c->seq_ring; }

RingPins ring_pins(Ctx* c, long long k, int i) {
  if (k == kOwnStream) {
    Result& r = c->results[i];
    return RingPins{&r.h_deskew, &r.h_area, 1, &r.h_acc};
  }
  SeqTick& t = c->seq_ticks[i];
  return RingPins{&t.h_deskew, &t.h_area, kMaxBatch, &t.blocks[k].h_acc};
}

// next tick of the sequence ring; `drop_oldest` as acquire_result
SeqTick* seq_acquire(Ctx* c, bool drop_oldest) {
  SeqTick* t = &c->seq_ticks[c->seq_next];
  if (t->in_flight) {
    if (!drop_oldest) return nullptr;
    cudaEventSynchronize(t->blocks[0].ev_done);
    t->in_flight = false;
    --c->seq_in_flight;
    c->seq_oldest = (c->seq_next + 1) % c->seq_ring;
  }
  c->seq_next = (c->seq_next + 1) % c->seq_ring;
  c->seq_last = t;
  return t;
}

// the tick's results: blocks[0].ev_done is recorded after the one publish launch that writes every stepped block.  A skipped sequence's
// block is stale (an earlier tick's step on this ring slot): its output, counts, IDs and last_n_act are left alone.
int seq_collect_tick(Ctx* c, SeqTick* t, lmot_seq_out* out) {
  LMOT_CUDA(c, cudaEventSynchronize(t->blocks[0].ev_done));
  int rc = LMOT_OK;
  if (out) out->n_seq = c->n_seq;
  c->seq_stepped = t->stepped;
  for (int k = 0; k < c->n_seq; ++k) {
    Stream& q = c->seq[k];
    if (!(t->stepped >> k & 1u)) { q.fc_n = 0; q.obs_last.valid = false; continue; }
    Result* b = &t->blocks[k];
    const int r = collect_result(c, b, out ? &out->seq[k] : nullptr, q);
    if (r < 0 ? (rc >= 0) : (rc == LMOT_OK)) rc = r;       // the first error, else the first warning
    // per-frame counts (lmot_seq_frame_counts): the concatenation / pack wrote them into the block; else the one frame's
    if (b->batch_frames > 0) {
      q.fc_n = b->batch_frames;
      memcpy(q.fc, b->h_frame_counts, (size_t)b->batch_frames * 4 * sizeof(int));
    } else {
      q.fc_n = 1;
      for (int j = 0; j < 4; ++j) q.fc[0][j] = b->h_hdr[HDR_N_ELEV + j];
    }
  }
  return rc;
}

int slot_create(Ctx* c, Slot* s, int index) {
  s->index = index;
  LMOT_CUDA(c, cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
  LMOT_CUDA(c, cudaEventCreateWithFlags(&s->ev_fork, cudaEventDisableTiming));
  LMOT_CUDA(c, cudaEventCreateWithFlags(&s->ev_det_done, cudaEventDisableTiming));
  LMOT_CUDA(c, cudaEventCreateWithFlags(&s->ev_trk_done, cudaEventDisableTiming));
  int rc = ground_alloc(c, s);
  if (rc == LMOT_OK) rc = cluster_alloc(c, s);
  if (rc == LMOT_OK) rc = boxfit_alloc(c, s);
  if (rc) return rc;
  LMOT_CUDA(c, cudaMalloc(&s->d_deskew, kDeskewTabBytes));
  LMOT_CUDA(c, cudaEventRecord(s->ev_trk_done, s->stream));   // "free" from the start
  LMOT_CUDA(c, cudaEventRecord(s->ev_det_done, s->stream));
  s->res = &c->results[0];
  return LMOT_OK;
}

void slot_destroy(Slot* s) {
  ground_free(s); cluster_free(s); boxfit_free(s);
  cudaFree(s->d_deskew); cudaFree(s->d_stage_wide); cudaFree(s->d_area_mask); cudaFree(s->d_area); cudaFree(s->d_gz);
  if (s->ev_fork) cudaEventDestroy(s->ev_fork);
  if (s->ev_det_done) cudaEventDestroy(s->ev_det_done);
  if (s->ev_trk_done) cudaEventDestroy(s->ev_trk_done);
  if (s->stream) cudaStreamDestroy(s->stream);
}

}  // namespace

extern "C" {

int lmot_default_params(lmot_params* p) {
  if (!p) return LMOT_ERR_INVALID;
  memset(p, 0, sizeof(*p));
  p->r_min = 3.4f; p->r_max = 120.f; p->t_hmin = -2.0f; p->t_hmax = -0.4f; p->t_hdiff = 0.4f; p->h_sensor = 2.f;
  p->ground_tolerance = 0.25;
  p->roi_m = 50.f;
  p->ram_points = 80; p->l_slope_dist = 1; p->l_num_points = 5; p->sensor_height = 2.f;
  p->t_height_min = 0.8f; p->t_height_max = 2.6f; p->t_width_min = 0.2f; p->t_width_max = 3.5f;
  p->t_len_min = 0.2f; p->t_len_max = 14.0f; p->t_area_max = 20.0f; p->t_ratio_min = 1.f; p->t_ratio_max = 8.0f;
  p->min_len_ratio = 3.0f; p->t_pt_per_m3 = 8.f; p->min_cluster_points = 30;
  p->rule_filter = LMOT_RULE_INTENDED;
  p->oracle_compat_first_frame = 1;
  p->max_points = 1 << 20; p->max_clusters = 4096; p->max_boxes = 1024; p->max_tracks = 8192;
  p->global_frame = 0;
  p->node_prefilter = 0; p->filter_z_min = -3.0f; p->filter_z_max = 1.0f;
  p->filter_x_min = -15.f; p->filter_x_max = 5.f; p->filter_y_min = -50.f; p->filter_y_max = 50.f;
  p->pipeline_depth = 8;   // detection takes 2-3x as long per frame as the tracker chain (H100: ~110 vs ~46 us): 8 frames in flight keep it ahead
  p->result_ring = 32;
  return LMOT_OK;
}

const char* lmot_strerror(int s) {
  switch (s) {
    case LMOT_OK: return "ok";
    case LMOT_ERR_INVALID: return "invalid argument";
    case LMOT_ERR_CUDA: return "CUDA error (no CPU fallback exists)";
    case LMOT_ERR_CAPACITY: return "capacity exceeded";
    case LMOT_ERR_STATE: return "invalid call sequence / not available";
    case LMOT_WARN_TRACK_TABLE_FULL: return "warning: track table full (max_tracks): unmatched boxes spawn no new track, existing tracks are still updated and reported";
    default: return "unknown status";
  }
}

const char* lmot_build_info(void) { return "liblmot sm_90a, nvcc " __DATE__ " -fmad=false"; }

int lmot_get_params(const lmot_ctx* ctx, lmot_params* out) {
  if (!ctx || !out) return LMOT_ERR_INVALID;
  *out = ctx->c.prm;
  return LMOT_OK;
}

const char* lmot_last_error(const lmot_ctx* ctx) { return ctx ? ctx->c.last_error.c_str() : ""; }

int lmot_create(lmot_ctx** out, const lmot_params* params, int device) {
  if (!out) return LMOT_ERR_INVALID;
  *out = nullptr;
  lmot_params p;
  if (params) p = *params; else lmot_default_params(&p);
  if (p.max_points <= 0 || p.max_clusters <= 0 || p.max_boxes <= 0 || p.max_tracks <= 0) return LMOT_ERR_INVALID;
  if (p.max_clusters > 50000 || p.max_boxes > 65535) return LMOT_ERR_INVALID;   // u16 cluster ids / box indices; one int per cluster id in the sort kernels' shared memory (<= 200 KB)
  if (p.pipeline_depth < 1) p.pipeline_depth = 1;
  if (p.pipeline_depth > kMaxSlots) p.pipeline_depth = kMaxSlots;
  if (p.result_ring < 1) p.result_ring = 1;
  if (p.result_ring > kMaxResults) p.result_ring = kMaxResults;
  // the frame pipeline uses up to 8 detection streams + tracker + publish stream per context; with the default of 8 hardware work
  // queues, streams alias and serialise each other.  Only effective if this process has not created its CUDA context yet.
  setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return LMOT_ERR_CUDA;
  if (cudaSetDevice(device) != cudaSuccess) return LMOT_ERR_CUDA;
  lmot_ctx* h = new (std::nothrow) lmot_ctx();
  if (!h) return LMOT_ERR_INVALID;
  Ctx* c = &h->c;
  c->prm = p;
  c->device = device;
  // grid-stride kernels are sized to the device: box fitting 2 CTAs per SM, the two wide tracker kernels 4 per SM
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) { delete h; return LMOT_ERR_CUDA; }
  c->fit_ctas = 2 * sms;
  c->trk_ctas = 4 * sms;
  c->max_points = p.max_points;
  c->n_slots = p.pipeline_depth;
  c->n_results = p.result_ring;
  {
    double tap[3];
    gauss_taps(tap);
    c->gp = ground_params_of(detect_params_of(p), tap);
  }
  if (const char* e = getenv("LMOT_COOP")) c->coop_launch = atoi(e) != 0;
  if (const char* e = getenv("LMOT_FUSE_CCL")) c->fuse_ccl = atoi(e) != 0;
  if (const char* e = getenv("LMOT_SPIN_LIMIT")) c->spin_limit = (unsigned)strtoul(e, nullptr, 0);   // 0: device-side waits never trap (debuggers, MPS)
  if (const char* e = getenv("LMOT_TRK_CTAS")) { const int v = atoi(e); if (v >= 8 && v <= 4096) c->trk_ctas = v; }     // tuning only
  if (const char* e = getenv("LMOT_TC_WIDE")) c->tc_force = atoi(e) != 0 ? 1 : 0;      // tests: pin spawn_output_kernel's variant (default: by active-track count)
  if (const char* e = getenv("LMOT_FIT_CTAS")) { const int v = atoi(e); if (v >= 8 && v <= 4096) c->fit_ctas = v; }
  if (const char* e = getenv("LMOT_ZERO_COPY")) c->zero_copy = atoi(e) != 0;
  if (const char* e = getenv("LMOT_GROUND_HALF")) c->ground_half_sms = atoi(e) != 0;
  if (const char* e = getenv("LMOT_PTS_PER_CTA")) { const int v = atoi(e); if (v >= 256 && v <= 16384) c->pts_per_cta = v; }
  int rc = LMOT_OK;
  // The tracker is the one sequential chain of the pipeline (frame f+1's tracker needs frame f's table): its CTAs get
  // the highest stream priority so they are never queued behind the detection kernels of later frames.
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  if (cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithPriority(&c->trk_stream, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
      cudaStreamCreateWithFlags(&c->pub_stream, cudaStreamNonBlocking) != cudaSuccess) { delete h; return LMOT_ERR_CUDA; }
  c->stream = c->own_stream;
  rc = boxfit_alloc_shared(c);
  for (int i = 0; i < c->n_results && rc == LMOT_OK; ++i) rc = result_create(c, &c->results[i]);
  for (int i = 0; i < c->n_slots && rc == LMOT_OK; ++i) rc = slot_create(c, &c->slots[i], i);
  c->last_res = &c->results[0];
  if (rc == LMOT_OK) rc = tracker_alloc(c, c->own.trk);
  if (rc == LMOT_OK) rc = (cudaDeviceSynchronize() == cudaSuccess) ? LMOT_OK : LMOT_ERR_CUDA;
  if (rc != LMOT_OK) { lmot_destroy(h); return rc; }
  *out = h;
  return LMOT_OK;
}

void lmot_destroy(lmot_ctx* ctx) {
  if (!ctx) return;
  Ctx* c = &ctx->c;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  ground_chain_forget(c->device, true);
  for (int i = 0; i < c->n_slots; ++i) slot_destroy(&c->slots[i]);
  batch_destroy(c);
  for (int i = 0; i < c->n_results; ++i) result_destroy(&c->results[i]);
  stream_free(c->own);
  seq_destroy(c);
  ego_ctx_free(c);
  cudaFree(c->d_mt_raw);
  cudaFree(c->d_bs_tab);
  if (c->ev_pred) cudaEventDestroy(c->ev_pred);
  if (c->ev_pred_in) cudaEventDestroy(c->ev_pred_in);
  cudaFree(c->d_pred_stage);
  if (c->h_pred_n) cudaFreeHost(c->h_pred_n);
  if (c->trk_stream) cudaStreamDestroy(c->trk_stream);
  if (c->pub_stream) cudaStreamDestroy(c->pub_stream);
  if (c->own_stream) cudaStreamDestroy(c->own_stream);
  delete ctx;
}

void* lmot_pinned_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  return p;
}

void lmot_pinned_free(void* p) { if (p) cudaFreeHost(p); }

int lmot_set_stream(lmot_ctx* ctx, void* s) {
  if (!ctx) return LMOT_ERR_INVALID;
  cudaSetDevice(ctx->c.device);
  ground_chain_forget(ctx->c.device, false);       // (the stream being replaced must still be valid, lmot.h)
  ctx->c.stream = s ? (cudaStream_t)s : ctx->c.own_stream;
  return LMOT_OK;
}

int lmot_sync(lmot_ctx* ctx) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  for (int i = 0; i < c->n_slots; ++i) LMOT_CUDA(c, cudaStreamSynchronize(c->slots[i].stream));
  for (int i = 0; i < c->n_bslots; ++i) LMOT_CUDA(c, cudaStreamSynchronize(c->bslots[i].stream));
  for (int b = 0; b < kBatchBanks; ++b) if (c->bank[b].stream) LMOT_CUDA(c, cudaStreamSynchronize(c->bank[b].stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->trk_stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->pub_stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->stream));
  return LMOT_OK;
}

// make the caller's stream wait for everything submitted so far (so CUDA events recorded on it bracket the work)
int lmot_flush(lmot_ctx* ctx) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  for (int i = 0; i < c->n_slots; ++i) {
    LMOT_CUDA(c, cudaStreamWaitEvent(c->stream, c->slots[i].ev_det_done, 0));
    LMOT_CUDA(c, cudaStreamWaitEvent(c->stream, c->slots[i].ev_trk_done, 0));
  }
  for (int b = 0; b < kBatchBanks && c->bank[b].ev_det_done; ++b) {      // (the banks exist once a batched or sequence tick ran)
    LMOT_CUDA(c, cudaStreamWaitEvent(c->stream, c->bank[b].ev_det_done, 0));
    LMOT_CUDA(c, cudaStreamWaitEvent(c->stream, c->bank[b].ev_trk_done, 0));
  }
  if (c->last_res && c->last_res->ev_done) LMOT_CUDA(c, cudaStreamWaitEvent(c->stream, c->last_res->ev_done, 0));   // publication is in order
  return LMOT_OK;
}

// ---------------------------------------------------------------------------------------------- stage entry points
int lmot_ground_remove_dev(lmot_ctx* ctx, const float* d_points, int n) {
  if (!ctx || n < 0 || (n > 0 && !d_points) || (reinterpret_cast<uintptr_t>(d_points) & 15u)) return LMOT_ERR_INVALID;   // cp.async.bulk: 16-byte aligned
  Ctx* c = &ctx->c;
  cudaSetDevice(c->device);
  if (n > c->max_points) return LMOT_ERR_CAPACITY;
  if (c->n_in_flight > 0) { int rc = drain(c); if (rc) return rc; }     // slot 0 may still be busy with a pipelined frame
  Slot* s = &c->slots[0];
  c->last_slot = 0;
  // (no label array, no debug grid: what the frame pipeline launches, minus the clustering bit planes)
  return ground_launch(c, s, c->stream, reinterpret_cast<const float4*>(d_points), n, false, false, false, true);
}

int lmot_ground_remove(lmot_ctx* ctx, const float* points, int n, int stride, uint8_t* labels, float* elevated,
                       int* n_elevated, float* ground, int* n_ground) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  cudaSetDevice(c->device);
  int rc = drain(c);
  if (rc) return rc;
  Slot* s = &c->slots[0];
  c->last_slot = 0;
  cudaStream_t st = c->stream;
  if ((rc = upload_points(c, s, st, points, n, stride, s->d_points))) return rc;
  if ((rc = ground_launch(c, s, st, s->d_points, n))) return rc;
  if ((rc = fetch_counters(c, s, st))) return rc;
  const int ne = s->h_counters[CNT_N_ELEV], ng = s->h_counters[CNT_N_GROUND];
  if (n_elevated) *n_elevated = ne;
  if (n_ground) *n_ground = ng;
  if (labels && n > 0) LMOT_CUDA(c, cudaMemcpyAsync(labels, s->d_labels, (size_t)n, cudaMemcpyDeviceToHost, st));
  if (elevated && ne > 0) LMOT_CUDA(c, cudaMemcpyAsync(elevated, s->d_elev, (size_t)ne * 16, cudaMemcpyDeviceToHost, st));
  if (ground && ng > 0) LMOT_CUDA(c, cudaMemcpyAsync(ground, s->d_ground, (size_t)ng * 16, cudaMemcpyDeviceToHost, st));
  LMOT_CUDA(c, cudaStreamSynchronize(st));
  return LMOT_OK;
}

int lmot_component_cluster(lmot_ctx* ctx, const float* elevated, int n, int stride, int32_t* grid, int* num_cluster) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  cudaSetDevice(c->device);
  int rc = drain(c);
  if (rc) return rc;
  Slot* s = &c->slots[0];
  c->last_slot = 0;
  cudaStream_t st = c->stream;
  if ((rc = upload_points(c, s, st, elevated, n, stride, s->d_elev))) return rc;
  if ((rc = set_counter(c, s, st, CNT_N_ELEV, n))) return rc;
  s->area_last = false;
  s->layers_last = false;
  c->n_lay_dbg = 0;
  if ((rc = cluster_launch(c, s, st, n))) return rc;
  if ((rc = fetch_counters(c, s, st))) return rc;
  if (num_cluster) *num_cluster = s->h_counters[CNT_NUM_CLUSTER];
  if (grid) {
    LMOT_CUDA(c, cudaMemcpyAsync(grid, s->d_label_grid, kCartCells * sizeof(int), cudaMemcpyDeviceToHost, st));
    LMOT_CUDA(c, cudaStreamSynchronize(st));
  }
  return LMOT_OK;
}

// the cluster node's side outputs for the elevated cloud + label grid of the most recent clustering of this context
int lmot_cluster_outputs(lmot_ctx* ctx, float* clustered, int cap_clustered, int* n_clustered, float* obstacles, int cap_obstacles,
                         int* n_obstacles, int32_t* cost_map) {
  if (!ctx || cap_clustered < 0 || cap_obstacles < 0) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  cudaSetDevice(c->device);
  int rc = lmot_sync(ctx);
  if (rc) return rc;
  Slot* s = &c->slots[c->last_slot];
  if (s->layers_last) return LMOT_ERR_STATE;           // the label grid does not name the layered clusters
  cudaStream_t st = c->stream;
  if ((rc = cluster_outputs_launch(c, s, st))) return rc;
  int cnt[2] = {0, 0};
  LMOT_CUDA(c, cudaMemcpyAsync(cnt, s->d_cost_map + 2500, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
  if (cost_map) LMOT_CUDA(c, cudaMemcpyAsync(cost_map, s->d_cost_map, 2500 * sizeof(int), cudaMemcpyDeviceToHost, st));
  LMOT_CUDA(c, cudaStreamSynchronize(st));
  if (n_clustered) *n_clustered = cnt[0];
  if (n_obstacles) *n_obstacles = cnt[1];
  const int nc = cnt[0] < cap_clustered ? cnt[0] : cap_clustered, no = cnt[1] < cap_obstacles ? cnt[1] : cap_obstacles;
  if (clustered && nc > 0) LMOT_CUDA(c, cudaMemcpyAsync(clustered, s->d_clustered, (size_t)nc * 16, cudaMemcpyDeviceToHost, st));
  if (obstacles && no > 0) LMOT_CUDA(c, cudaMemcpyAsync(obstacles, s->d_obstacles, (size_t)no * 16, cudaMemcpyDeviceToHost, st));
  LMOT_CUDA(c, cudaStreamSynchronize(st));
  return (cnt[0] > cap_clustered && clustered) || (cnt[1] > cap_obstacles && obstacles) ? LMOT_ERR_CAPACITY : LMOT_OK;
}

int lmot_debug_label_grid(lmot_ctx* ctx, int32_t* grid, int* num_cluster) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  int rc = lmot_sync(ctx);
  if (rc) return rc;
  Slot* s = &c->slots[c->last_slot];
  if (s->layers_last) return LMOT_ERR_STATE;
  if ((rc = fetch_counters(c, s, c->stream))) return rc;
  if (num_cluster) *num_cluster = s->h_counters[CNT_NUM_CLUSTER];
  if (grid) {
    LMOT_CUDA(c, cudaMemcpyAsync(grid, s->d_label_grid, kCartCells * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    LMOT_CUDA(c, cudaStreamSynchronize(c->stream));
  }
  return LMOT_OK;
}

int lmot_box_fit(lmot_ctx* ctx, const float* elevated, int n, int stride, const int32_t* grid, int num_cluster,
                 float* boxes, int max_boxes, int* n_boxes, float* markers) {
  if (!ctx || !grid || num_cluster < 0 || max_boxes < 0) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  cudaSetDevice(c->device);
  if (num_cluster > c->prm.max_clusters) return LMOT_ERR_CAPACITY;
  int rc = drain(c);
  if (rc) return rc;
  Slot* s = &c->slots[0];
  c->last_slot = 0;
  cudaStream_t st = c->stream;
  if ((rc = upload_points(c, s, st, elevated, n, stride, s->d_elev))) return rc;
  LMOT_CUDA(c, cudaMemcpyAsync(s->d_label_grid, grid, kCartCells * sizeof(int), cudaMemcpyHostToDevice, st));
  s->label_grid_foreign = true;
  s->area_last = false;
  s->layers_last = false;
  c->n_lay_dbg = 0;
  if ((rc = set_counter(c, s, st, CNT_N_ELEV, n))) return rc;
  if ((rc = set_counter(c, s, st, CNT_NUM_CLUSTER, num_cluster))) return rc;
  s->res = &c->results[0];
  s->res->n_kev = 0;
  if ((rc = cluster_cells_only(c, s, st, n))) return rc;
  if ((rc = boxfit_launch(c, s, st, n))) return rc;
  if ((rc = fetch_counters(c, s, st))) return rc;
  if ((rc = check_device_error(c, s, st))) return rc;
  const int nb = s->h_counters[CNT_N_BOXES];
  if (n_boxes) *n_boxes = nb;
  const int ncopy = nb < max_boxes ? nb : max_boxes;
  if (boxes && ncopy > 0) LMOT_CUDA(c, cudaMemcpyAsync(boxes, s->d_boxes, (size_t)ncopy * 24 * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (markers && ncopy > 0) LMOT_CUDA(c, cudaMemcpyAsync(markers, s->d_markers, (size_t)ncopy * 6 * sizeof(float), cudaMemcpyDeviceToHost, st));
  LMOT_CUDA(c, cudaStreamSynchronize(st));
  return nb > max_boxes ? LMOT_ERR_CAPACITY : LMOT_OK;
}

int lmot_track_step(lmot_ctx* ctx, const float* boxes, int m, double timestamp_us, double v_gps, double yaw_gps,
                    lmot_track_out* out) {
  if (!ctx || m < 0 || (m > 0 && !boxes)) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  cudaSetDevice(c->device);
  if (m > c->prm.max_boxes) return LMOT_ERR_CAPACITY;
  int rc = drain(c);
  if (rc) return rc;
  Slot* s = &c->slots[0];
  c->last_slot = 0;
  s->res = &c->results[0];
  c->last_res = s->res;
  s->res->n_kev = 0;
  cudaStream_t st = c->stream;
  if (m > 0) LMOT_CUDA(c, cudaMemcpyAsync(s->d_boxes, boxes, (size_t)m * 24 * sizeof(float), cudaMemcpyHostToDevice, st));
  if ((rc = set_counter(c, s, st, CNT_N_BOXES, m))) return rc;
  if (c->timing) cudaEventRecord(s->res->ev[3], st);
  if (c->prm.global_frame && (rc = boxes_to_global_launch(c, s, st, s->d_boxes, s->d_counters, timestamp_us, v_gps, yaw_gps, false))) return rc;
  if ((rc = tracker_launch(c, s, st, s->d_boxes, s->d_counters, timestamp_us, v_gps, yaw_gps))) return rc;
  if (c->timing) cudaEventRecord(s->res->ev[4], st);
  if ((rc = tracker_publish(c, s->res, st))) return rc;
  LMOT_CUDA(c, cudaStreamSynchronize(st));
  if (c->timing) {    // tracker stage only: stage_ms[3], kernel_ms[0..] = predict+gate, update, spawn/output
    c->stage_ms[0] = c->stage_ms[1] = c->stage_ms[2] = 0.f;
    cudaEventElapsedTime(&c->stage_ms[3], s->res->ev[3], s->res->ev[4]);
    c->n_kernel_ms = s->res->n_kev;
    for (int i = 0; i < s->res->n_kev; ++i) cudaEventElapsedTime(&c->kernel_ms[i], i == 0 ? s->res->ev[3] : s->res->kev[i - 1], s->res->kev[i]);
  }
  const int err = s->res->h_hdr[HDR_ERROR];
  c->own.trk.last_n_act = s->res->h_hdr[HDR_N_ACT];
  note_ids(c->own.trk, s->res);
  rc = copy_track_outputs(s->res, out);
  return err ? err : (rc ? rc : s->res->h_hdr[HDR_WARN]);
}

// ---------------------------------------------------------------------------------------------- frame pipeline
int lmot_detect_dev(lmot_ctx* ctx, const float* d_points, int n) {
  if (!ctx || n < 0 || (n > 0 && !d_points) || (reinterpret_cast<uintptr_t>(d_points) & 15u)) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  cudaSetDevice(c->device);
  if (n > c->max_points) return LMOT_ERR_CAPACITY;
  if (c->own.cfg.beyond_plain(false, false) && c->timing) return LMOT_ERR_STATE;
  Slot* s = acquire_slot(c);
  Result* r = acquire_result(c, true);
  LMOT_CUDA(c, cudaEventRecord(s->ev_fork, c->stream));
  LMOT_CUDA(c, cudaStreamWaitEvent(s->stream, s->ev_fork, 0));
  return submit(c, s, r, d_points, n, 4, false, false, 0, 0, 0);
}

int lmot_frame_dev(lmot_ctx* ctx, const float* d_points, int n, double timestamp_us, double v_gps, double yaw_gps) {
  if (!ctx || n < 0 || (n > 0 && !d_points) || (reinterpret_cast<uintptr_t>(d_points) & 15u)) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  if (c->own.cfg.beyond_plain(true, false) && c->timing) return LMOT_ERR_STATE;
  if (!c->own.cfg.deskew_fits(true, 4)) return LMOT_ERR_INVALID;     // device frames are float4: the time is the 4th float
  cudaSetDevice(c->device);
  if (n > c->max_points) return LMOT_ERR_CAPACITY;
  Slot* s = acquire_slot(c);
  Result* r = acquire_result(c, true);
  LMOT_CUDA(c, cudaEventRecord(s->ev_fork, c->stream));          // the caller's stream produced d_points
  LMOT_CUDA(c, cudaStreamWaitEvent(s->stream, s->ev_fork, 0));
  return submit(c, s, r, d_points, n, 4, false, true, timestamp_us, v_gps, yaw_gps);
}

int lmot_frame_submit(lmot_ctx* ctx, const float* points, int n, int stride, double timestamp_us, double v_gps, double yaw_gps) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  cudaSetDevice(c->device);
  if (c->own.cfg.beyond_plain(true, false) && c->timing) return LMOT_ERR_STATE;
  const bool dsk = c->own.cfg.deskews(true);
  if (dsk) {                           // (validated before anything is submitted: upload_points checks the rest without deskew)
    if (n < 0 || (n > 0 && !points) || !c->own.cfg.deskew_fits(true, stride)) return LMOT_ERR_INVALID;
    if (n > c->max_points) return LMOT_ERR_CAPACITY;
  }
  if (c->n_in_flight >= c->n_results) return LMOT_ERR_STATE;    // result ring full: collect first
  Slot* s = acquire_slot(c);
  Result* r = acquire_result(c, false);
  if (!r) return LMOT_ERR_STATE;
  // (End-to-end frames/s is bound by these copies -- one 1.9 MB copy per frame -- not by the tracker chain.  A copy stream of its
  // own changed nothing, two alternating ones made cudaMemcpyAsync
  // block the host.)
  // ZERO COPY (opt-in, LMOT_ZERO_COPY=1): a frame in page-locked host memory (lmot_pinned_alloc, cudaHostAlloc, cudaHostRegister) is
  // not copied; under unified addressing the ground kernel's bulk copies read it over PCIe straight into shared memory, so every
  // input byte crosses the link once and never touches HBM (possible whenever the launch keeps each CTA's chunk resident,
  // ground_reads_input_once).  Bit-identical results (tests/test_pipeline_gpu.py) -- but SM-issued reads over the link were
  // slower than the copy engine at this copy size.  Hence off by default.  The buffer must stay untouched until
  // the frame has been collected (the same contract as the asynchronous copy).
  if (!dsk && c->zero_copy && stride == 4 && n > 0 && n <= c->max_points && (reinterpret_cast<uintptr_t>(points) & 15u) == 0 && ground_reads_input_once(c, n)) {
    cudaPointerAttributes pa;
    if (cudaPointerGetAttributes(&pa, points) == cudaSuccess && pa.type == cudaMemoryTypeHost && pa.devicePointer)
      return submit(c, s, r, static_cast<const float*>(pa.devicePointer), n, 4, false, true, timestamp_us, v_gps, yaw_gps);
    cudaGetLastError();      // (pageable memory: not an error, take the copy path)
  }
  return submit(c, s, r, points, n, stride, true, true, timestamp_us, v_gps, yaw_gps);
}

int lmot_frame_collect(lmot_ctx* ctx, lmot_frame_out* out) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  if (c->n_in_flight <= 0) return LMOT_ERR_STATE;
  Result* r = &c->results[c->res_oldest];
  int guard = 0;
  while (!r->in_flight && guard++ < c->n_results) { c->res_oldest = (c->res_oldest + 1) % c->n_results; r = &c->results[c->res_oldest]; }
  if (!r->in_flight) return LMOT_ERR_STATE;
  const int rc = collect_result(c, r, out, c->own);
  r->in_flight = false;
  --c->n_in_flight;
  c->res_oldest = (c->res_oldest + 1) % c->n_results;
  return rc;
}

int lmot_frames_in_flight(lmot_ctx* ctx, int* n) {
  if (!ctx || !n) return LMOT_ERR_INVALID;
  *n = ctx->c.n_in_flight;
  return LMOT_OK;
}

// 1 if the oldest submitted frame has finished (lmot_frame_collect would not block), 0 if not, <0 on error
int lmot_frame_ready(lmot_ctx* ctx) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  if (c->n_in_flight <= 0) return 0;
  Result* r = &c->results[c->res_oldest];
  if (!r->in_flight) return 0;
  return cudaEventQuery(r->ev_done) == cudaSuccess ? 1 : 0;
}

// results of the MOST RECENT submission; older uncollected ones are dropped
int lmot_frame_fetch(lmot_ctx* ctx, lmot_frame_out* out) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  Result* r = c->last_res;
  const int rc = collect_result(c, r, out, c->own);
  for (int i = 0; i < c->n_results; ++i) c->results[i].in_flight = false;
  c->n_in_flight = 0;
  c->res_oldest = c->res_next;
  return rc;
}

int lmot_frame(lmot_ctx* ctx, const float* points, int n, int stride, double timestamp_us, double v_gps, double yaw_gps,
               lmot_frame_out* out) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  if (c->n_in_flight > 0) { int rc = drain(c); if (rc) return rc; }
  int rc = lmot_frame_submit(ctx, points, n, stride, timestamp_us, v_gps, yaw_gps);
  if (rc) return rc;
  return lmot_frame_collect(ctx, out);
}

// ---------------------------------------------------------------------------------------------- batched ticks
// one tick: F frames of the context's own stream -> the detection front end on the next bank -> concatenated boxes -> (optionally) the
// tracker.  A merging rig (lmot_set_rig_merge) concatenates the bank's merge unit, its boxes already in the vehicle frame.
static int batch_common(lmot_ctx* ctx, const float* const* points, const int* n, int n_frames, int stride, bool host, bool with_tracker,
                        double ts, double v, double yaw) {
  if (!ctx || !points || !n || n_frames < 1 || n_frames > kMaxBatch) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  StreamCfg& q = c->own.cfg;
  if (q.n_sensors > 0 && n_frames > q.n_sensors) return LMOT_ERR_INVALID;     // a frame without a sensor pose
  cudaSetDevice(c->device);
  for (int i = 0; i < n_frames; ++i) {
    if (n[i] < 0 || (n[i] > 0 && !points[i])) return LMOT_ERR_INVALID;
    if (n[i] > c->max_points) return LMOT_ERR_CAPACITY;
    if (!host && n[i] > 0 && (reinterpret_cast<uintptr_t>(points[i]) & 15u)) return LMOT_ERR_INVALID;   // bulk copies need 16-byte alignment
  }
  // (lmot_batch_detect_dev has no stamp: never deskewed, never accumulated)
  if (q.beyond_plain(with_tracker, true) && c->timing) return LMOT_ERR_STATE;
  if (!q.deskew_fits(with_tracker, stride)) return LMOT_ERR_INVALID;
  if (host && c->n_in_flight >= c->n_results) return LMOT_ERR_STATE;
  int rc = batch_ensure(c, n_frames);
  if (rc) return rc;
  if (q.merges() && (rc = merge_ensure(c, q.merge_unit, 3000))) return rc;
  Result* r = acquire_result(c, !host);
  if (!r) return LMOT_ERR_STATE;
  const int b = c->next_bank;
  c->next_bank = (c->next_bank + 1) % kBatchBanks;
  Slot* k = &c->bank[b];
  cudaStream_t st = c->bslots[b * c->batch_frames].stream;
  // the bank's previous tick must have been consumed by the tracker; device frames: ordered after the caller's stream
  LMOT_CUDA(c, cudaStreamWaitEvent(st, k->ev_trk_done, 0));
  if (!host) {
    LMOT_CUDA(c, cudaEventRecord(k->ev_fork, c->stream));
    LMOT_CUDA(c, cudaStreamWaitEvent(st, k->ev_fork, 0));
  }
  struct Tail { Ctx* c; double t0; ~Tail() { c->host_ns[0] += now_ns() - t0; } } tail{c, now_ns()};
  k->res = r;
  r->n_kev = 0;
  r->batch_frames = n_frames;
  r->merge_rows = q.merges() ? n_frames : 0;
  int* d_fc = nullptr;                       // the per-frame counts go straight into the result's pinned, device-mapped block
  LMOT_CUDA(c, cudaHostGetDevicePointer((void**)&d_fc, r->h_frame_counts, 0));
  const DetGroup grp{&q, with_tracker ? &c->own.trk.th : nullptr, points, n, n_frames, ts, v, yaw, d_fc, r, true};
  DetUnits U;
  Slot* fr = &c->bslots[b * c->batch_frames];
  if ((rc = detect_front(c, k, fr, st, b, &grp, 1, stride, host, r->h_deskew, r->h_area, false, U))) return rc;
  own_debug_note(c, fr, n_frames, U);
  const bool gf = with_tracker && c->prm.global_frame;
  if ((rc = boxes_concat_launch(c, U.u, U.f0[1], st, k->d_boxes, k->d_counters, U.fc[0], (with_tracker && !gf) ? k->d_det_sem : nullptr,
                                U.rig_on[0] ? U.rig : nullptr))) return rc;
  if (gf && (rc = boxes_to_global_launch(c, k, st, k->d_boxes, k->d_counters, ts, v, yaw, true))) return rc;
  if (c->timing) cudaEventRecord(r->ev[3], st);
  LMOT_CUDA(c, cudaEventRecord(k->ev_det_done, st));
  if (with_tracker) {
    if ((rc = submit_tracker(c, k, r, k->d_boxes, k->d_counters, ts, v, yaw))) return rc;
  } else {
    LMOT_CUDA(c, cudaMemcpyAsync(r->h_det, k->d_counters, CNT_COUNT * sizeof(int), cudaMemcpyDeviceToHost, st));
    if ((rc = boxes_publish(c, k, r, st))) return rc;
    LMOT_CUDA(c, cudaEventRecord(k->ev_trk_done, st));
    LMOT_CUDA(c, cudaEventRecord(r->ev_done, st));
  }
  r->has_tracks = with_tracker;
  if (!r->in_flight) { r->in_flight = true; ++c->n_in_flight; }
  return LMOT_OK;
}

int lmot_batch_submit(lmot_ctx* ctx, const float* const* points, const int* n, int n_frames, int stride_floats, double timestamp_us,
                      double v_gps, double yaw_gps) {
  return batch_common(ctx, points, n, n_frames, stride_floats, true, true, timestamp_us, v_gps, yaw_gps);
}

int lmot_batch_dev(lmot_ctx* ctx, const float* const* d_points, const int* n, int n_frames, double timestamp_us, double v_gps, double yaw_gps) {
  return batch_common(ctx, d_points, n, n_frames, 4, false, true, timestamp_us, v_gps, yaw_gps);
}

int lmot_batch_detect_dev(lmot_ctx* ctx, const float* const* d_points, const int* n, int n_frames) {
  return batch_common(ctx, d_points, n, n_frames, 4, false, false, 0, 0, 0);
}

// ground removal + connected components of F device frames in two launches on the CALLER's stream (bench.py times the
// ground_removal + CCL roofline of the batched configuration with it; results stay on the device)
int lmot_batch_ground_ccl_dev(lmot_ctx* ctx, const float* const* d_points, const int* n, int n_frames) {
  if (!ctx || !d_points || !n || n_frames < 1 || n_frames > kMaxBatch) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  const StreamCfg& q = c->own.cfg;
  if (q.n_sensors > 0 && n_frames > q.n_sensors) return LMOT_ERR_INVALID;
  cudaSetDevice(c->device);
  int rc = batch_ensure(c, n_frames);
  if (rc) return rc;
  if (c->n_in_flight > 0 && (rc = drain(c))) return rc;
  Slot* sl[kMaxBatch];
  const float4* pp[kMaxBatch];
  for (int i = 0; i < n_frames; ++i) {
    if (n[i] < 0 || n[i] > c->max_points || (n[i] > 0 && (!d_points[i] || (reinterpret_cast<uintptr_t>(d_points[i]) & 15u)))) return LMOT_ERR_INVALID;
    sl[i] = &c->bslots[i]; pp[i] = reinterpret_cast<const float4*>(d_points[i]);
  }
  sl[0]->res = &c->results[0];
  c->results[0].n_kev = 0;
  if ((rc = ground_launch_batch(c, sl, n_frames, pp, n, c->stream, true, false, c->fuse_ccl, c->fuse_ccl, q.n_sensors > 0 ? q.sensors : nullptr))) return rc;
  return c->fuse_ccl ? LMOT_OK : ccl_launch_batch(c, sl, n_frames, c->stream);
}

static int batch_fill(Ctx* c, Result* r, int rc0, lmot_batch_out* out, const lmot_frame_out& fo) {
  if (!out) return rc0;
  const int F = r->batch_frames;
  out->n_frames = F;
  for (int i = 0; i < kMaxBatch; ++i) {
    const bool in = i < F;
    out->n_elevated[i] = in ? r->h_frame_counts[4 * i] : 0; out->n_ground[i] = in ? r->h_frame_counts[4 * i + 1] : 0;
    out->num_cluster[i] = in ? r->h_frame_counts[4 * i + 2] : 0; out->n_boxes[i] = in ? r->h_frame_counts[4 * i + 3] : 0;
  }
  out->n_boxes_total = fo.n_boxes;
  out->tracks = fo.tracks;
  return rc0;
}

int lmot_batch_collect(lmot_ctx* ctx, lmot_batch_out* out) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  if (c->n_in_flight <= 0) return LMOT_ERR_STATE;
  Result* r = &c->results[c->res_oldest];
  int guard = 0;
  while (!r->in_flight && guard++ < c->n_results) { c->res_oldest = (c->res_oldest + 1) % c->n_results; r = &c->results[c->res_oldest]; }
  if (!r->in_flight) return LMOT_ERR_STATE;
  lmot_frame_out fo{};
  if (out) { fo.boxes = out->boxes; fo.max_boxes = out->max_boxes; fo.tracks = out->tracks; }
  const int rc = collect_result(c, r, out ? &fo : nullptr, c->own);
  r->in_flight = false;
  --c->n_in_flight;
  c->res_oldest = (c->res_oldest + 1) % c->n_results;
  return batch_fill(c, r, rc, out, fo);
}

int lmot_batch_fetch(lmot_ctx* ctx, lmot_batch_out* out) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  Result* r = c->last_res;
  lmot_frame_out fo{};
  if (out) { fo.boxes = out->boxes; fo.max_boxes = out->max_boxes; fo.tracks = out->tracks; }
  const int rc = collect_result(c, r, out ? &fo : nullptr, c->own);
  for (int i = 0; i < c->n_results; ++i) c->results[i].in_flight = false;
  c->n_in_flight = 0;
  c->res_oldest = c->res_next;
  return batch_fill(c, r, rc, out, fo);
}

int lmot_batch(lmot_ctx* ctx, const float* const* points, const int* n, int n_frames, int stride_floats, double timestamp_us, double v_gps,
               double yaw_gps, lmot_batch_out* out) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  if (c->n_in_flight > 0) { int rc = drain(c); if (rc) return rc; }
  int rc = lmot_batch_submit(ctx, points, n, n_frames, stride_floats, timestamp_us, v_gps, yaw_gps);
  if (rc) return rc;
  return lmot_batch_collect(ctx, out);
}

// ---------------------------------------------------------------------------------------------- independent sequences
static int seq_meas_alloc(Ctx* c, SeqMeas& m) {
  const size_t lb = (size_t)c->prm.max_boxes * 24 * sizeof(float);
  LMOT_CUDA(c, cudaMalloc(&m.d_boxes, lb));
  LMOT_CUDA(c, cudaMalloc(&m.d_boxes_g, lb));
  LMOT_CUDA(c, cudaMalloc(&m.d_counters, CNT_COUNT * sizeof(int)));
  LMOT_CUDA(c, cudaMemset(m.d_counters, 0, CNT_COUNT * sizeof(int)));
  LMOT_CUDA(c, cudaMalloc(&m.d_det_sem, sizeof(int)));
  LMOT_CUDA(c, cudaMemset(m.d_det_sem, 0, sizeof(int)));
  return LMOT_OK;
}

int lmot_seq_open(lmot_ctx* ctx, int n_seq, int ring) {
  if (!ctx || n_seq < 0 || n_seq > kMaxBatch || (n_seq > 0 && (ring < 1 || ring > kMaxResults))) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  cudaSetDevice(c->device);
  int rc = drain(c);
  if (rc) return rc;
  seq_destroy(c);
  if (n_seq == 0) return LMOT_OK;
  c->seq_ticks = new (std::nothrow) SeqTick[ring];
  if (!c->seq_ticks) return LMOT_ERR_INVALID;
  c->seq_ring = ring;
  c->n_seq = n_seq;                    // (set before the allocations: seq_destroy frees whatever was allocated on failure)
  for (int k = 0; k < n_seq && rc == LMOT_OK; ++k) rc = tracker_alloc(c, c->seq[k].trk);
  for (int b = 0; b < kBatchBanks && rc == LMOT_OK; ++b)         // (nothing is in flight: drained above)
    for (int k = 0; k < n_seq && rc == LMOT_OK; ++k) rc = seq_meas_alloc(c, c->seq_meas[b][k]);
  for (int b = 0; b < kBatchBanks && rc == LMOT_OK; ++b)
    if (cudaMalloc(&c->seq_stage[b], (size_t)kMaxBatch * c->prm.max_boxes * 24 * sizeof(float) + kMaxBatch * sizeof(int)) != cudaSuccess) rc = LMOT_ERR_CUDA;
  for (int i = 0; i < ring && rc == LMOT_OK; ++i)
    for (int k = 0; k < n_seq && rc == LMOT_OK; ++k) rc = result_create(c, &c->seq_ticks[i].blocks[k]);
  if (rc == LMOT_OK) rc = (cudaDeviceSynchronize() == cudaSuccess) ? LMOT_OK : LMOT_ERR_CUDA;
  if (rc) seq_destroy(c);
  return rc;
}

// ---- sequence ticks: one builder (seq_tick_common) for lmot_seq_tick_*, lmot_seq* (every entry FRAMES) and lmot_seq_track* (every entry
// LISTS).  A tick's entries say, per sequence, whether it steps this tick and from what: FRAMES entries go through the detection front
// end (detect_front, one group per sequence), LISTS entries through one pack launch; both fill the stepped sequences' measurement lists,
// and ONE tracker chain steps the stepped tables.  Every tick shares the ring and the bank alternation; each table folds its steps in
// submission order.
//
// The map: the stepped sequences, in sequence order, are the chain positions 0..S-1 (seq[pos] = sequence).  The FRAMES entries' frames
// are the detection slots in that order, the LISTS entries' lists the pack's lists in that order.  Every per-sequence array handed to a
// launch (measurement lists, ego values, rig poses, frame-count pointers, result blocks) is built through it.

// the set's layout: sequence k's sensors in table order, [f0[k], f0[k + 1]); one for a sequence without a table (lmot_seq_set_sensors
// keeps the total at or below kMaxBatch).  -> whether any sequence has a table
static bool seq_layout(const Ctx* c, int* f0, bool* rig_on) {
  bool rigged = false;
  f0[0] = 0;
  for (int k = 0; k < c->n_seq; ++k) {
    rig_on[k] = c->seq[k].cfg.n_sensors > 0;
    rigged |= rig_on[k];
    f0[k + 1] = f0[k] + (rig_on[k] ? c->seq[k].cfg.n_sensors : 1);
  }
  return rigged;
}

// LMOT_SEQ_RESTART: lmot_seq_tracker_reset's host state, and the table's counters cleared on the tracker stream ahead of the chain (in
// stream order: the table's earlier steps and predictions queued before come first).  act_valid = false: the chain rebuilds the active
// list (chain_prepare's `full` path) and seeds TC from this step's own block.
static void tracker_restart_host(Tracker& t) {
  t.th = TrackerHost();
  t.pred_ok = false;                   // no stamp to predict from until the next step or load
  t.act_valid = false;
  t.ids_identity = true;               // the spawn counter restarts at 0 (the retirement switch is kept)
}

// host form: frames with `stride` floats per point and host lists; device form (host = false): device frames (stride 4) and lists
static int seq_tick_common(lmot_ctx* ctx, const lmot_seq_entry* e, int n_seq, int stride, bool host) {
  if (!ctx || !e) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  if (c->n_seq == 0 || n_seq != c->n_seq) return LMOT_ERR_INVALID;
  if (c->timing) return LMOT_ERR_STATE;
  int f0[kMaxBatch + 1];
  bool rig_on[kMaxBatch];
  seq_layout(c, f0, rig_on);
  // validation: nothing is submitted unless the whole tick is valid
  int S = 0, F = 0, FL = 0;            // stepped sequences, detection frames, lists
  bool rigged = false;
  bool merge[kMaxBatch] = {};          // FRAMES sequences with a table and lmot_seq_set_rig_merge on: one merged cloud per sequence
  for (int k = 0; k < n_seq; ++k) {
    const lmot_seq_entry& q = e[k];
    const int nk = f0[k + 1] - f0[k];
    if (q.flags & ~LMOT_SEQ_RESTART) return LMOT_ERR_INVALID;
    if (q.kind == LMOT_SEQ_SKIP) { if (q.flags) return LMOT_ERR_INVALID; continue; }
    if (q.kind != LMOT_SEQ_FRAMES && q.kind != LMOT_SEQ_LISTS) return LMOT_ERR_INVALID;
    const bool dev_lists = !host && q.kind == LMOT_SEQ_LISTS;
    if (!q.data || (dev_lists ? (!q.d_counts || q.cap_per_list < 1) : !q.n)) return LMOT_ERR_INVALID;
    for (int j = 0; j < nk; ++j) {
      if (dev_lists) { if (!q.data[j]) return LMOT_ERR_INVALID; continue; }
      if (q.n[j] < 0 || (q.n[j] > 0 && !q.data[j])) return LMOT_ERR_INVALID;
      if (!host && q.kind == LMOT_SEQ_FRAMES && q.n[j] > 0 && (reinterpret_cast<uintptr_t>(q.data[j]) & 15u)) return LMOT_ERR_INVALID;   // bulk copies
    }
    if (q.kind == LMOT_SEQ_FRAMES && !c->seq[k].cfg.deskew_fits(true, host ? stride : 4)) return LMOT_ERR_INVALID;
    ++S;
    if (q.kind == LMOT_SEQ_FRAMES) { F += nk; rigged |= rig_on[k]; merge[k] = c->seq[k].cfg.merges(); }
    else FL += nk;
  }
  if (S == 0 || (host && F > 0 && stride < 3)) return LMOT_ERR_INVALID;
  for (int k = 0; k < n_seq; ++k) {
    const lmot_seq_entry& q = e[k];
    if (q.kind == LMOT_SEQ_SKIP || (!host && q.kind == LMOT_SEQ_LISTS)) continue;
    const int cap = q.kind == LMOT_SEQ_FRAMES ? c->max_points : c->prm.max_boxes;
    for (int j = 0; j < f0[k + 1] - f0[k]; ++j) if (q.n[j] > cap) return LMOT_ERR_CAPACITY;
  }
  if (host && c->seq_in_flight >= c->seq_ring) return LMOT_ERR_STATE;
  cudaSetDevice(c->device);
  int rc;
  if (F > 0) {
    if ((rc = batch_ensure(c, F))) return rc;
  } else if (!c->bank[0].stream) {     // a tracking tick needs the banks' events and streams, not their detection slots
    if ((rc = bank_ensure(c))) return rc;
    LMOT_CUDA(c, cudaDeviceSynchronize());
  }
  for (int k = 0; k < n_seq; ++k)
    if (merge[k] && (rc = merge_ensure(c, c->seq[k].cfg.merge_unit, 4000 + 16 * k))) return rc;
  // the tick's ring slot and bank; the front end runs on the bank's first detection slot's stream (on the bank's own stream when no
  // sequence sends frames), after the bank's previous tick has been consumed by the tracker
  SeqTick* t = seq_acquire(c, !host);
  if (!t) return LMOT_ERR_STATE;
  const int b = c->next_bank;
  c->next_bank = (c->next_bank + 1) % kBatchBanks;
  Slot* bk = &c->bank[b];
  cudaStream_t st = F > 0 ? c->bslots[b * c->batch_frames].stream : bk->stream;
  LMOT_CUDA(c, cudaStreamWaitEvent(st, bk->ev_trk_done, 0));
  if (!host) {                         // device data: ordered after the caller's stream
    LMOT_CUDA(c, cudaEventRecord(bk->ev_fork, c->stream));
    LMOT_CUDA(c, cudaStreamWaitEvent(st, bk->ev_fork, 0));
  }
  struct Tail { Ctx* c; double t0; ~Tail() { c->host_ns[0] += now_ns() - t0; } } tail{c, now_ns()};
  const bool gf = c->prm.global_frame != 0;
  // the map: chain position -> sequence, and per position its measurement list and ego values
  int seq[kMaxBatch];
  SeqMeas m[kMaxBatch];
  double ts[kMaxBatch], v[kMaxBatch], yaw[kMaxBatch];
  uint32_t stepped = 0;
  for (int k = 0, p = 0; k < n_seq; ++k) {
    if (e[k].kind == LMOT_SEQ_SKIP) continue;
    seq[p] = k; ts[p] = e[k].timestamp_us; v[p] = e[k].v_gps; yaw[p] = e[k].yaw_gps;
    ++p;
    stepped |= 1u << k;
    if (e[k].flags & LMOT_SEQ_RESTART) {
      c->seq[k].cfg.acc.forget();
      tracker_restart_host(c->seq[k].trk);
      LMOT_CUDA(c, cudaMemsetAsync(c->seq[k].trk.d_trk_counters, 0, CNT_COUNT * sizeof(int), c->trk_stream));
    }
    Result* r = &t->blocks[k];
    r->n_kev = 0; r->has_tracks = true;
    r->acc_units = 0;                  // (an accumulating FRAMES step sets it in detect_front)
    r->obs_units = 0;                  // (a FRAMES step with obstacles on sets it in detect_front)
    // > 0: the concatenation / pack writes the block's per-frame counts; 0: one frame, counts from the header
    r->batch_frames = (e[k].kind == LMOT_SEQ_LISTS || rigged) ? f0[k + 1] - f0[k] : 0;
    r->merge_rows = merge[k] ? f0[k + 1] - f0[k] : 0;
  }
  t->stepped = stepped;
  bk->res = &t->blocks[seq[0]];
  // the stepped sequences' measurement lists, by sequence (gathered by chain position below)
  SeqMeas mk[kMaxBatch];
  if (FL > 0) {
    // LISTS entries: host lists staged at list i * max_boxes boxes of the bank's staging buffer (16-byte aligned), their counts behind the
    // lists (the copies are ordered after the bank's previous tick, whose pack kernel was the last reader); device lists as they are
    const int MB = c->prm.max_boxes;
    float* stage = c->seq_stage[b];
    int* counts = reinterpret_cast<int*>(stage + (size_t)kMaxBatch * MB * 24);
    SeqLists L{};
    int lf0[kMaxBatch + 1], hn[kMaxBatch], fcount = 0, nl = 0;
    bool lrig[kMaxBatch];
    lmot_sensor rig[kMaxBatch];
    int* fc[kMaxBatch];
    SeqMeas lm[kMaxBatch];
    lf0[0] = 0;
    for (int k = 0; k < n_seq; ++k) {
      if (e[k].kind != LMOT_SEQ_LISTS) continue;
      for (int j = 0; j < f0[k + 1] - f0[k]; ++j, ++fcount) {
        const int i = fcount;
        if (host) {
          hn[i] = e[k].n[j];
          if (hn[i] > 0) LMOT_CUDA(c, cudaMemcpyAsync(stage + (size_t)i * MB * 24, e[k].data[j], (size_t)hn[i] * 24 * sizeof(float), cudaMemcpyHostToDevice, st));
          L.lists[i] = stage + (size_t)i * MB * 24; L.counts[i] = counts + i; L.cap[i] = MB;
        } else {
          L.lists[i] = e[k].data[j]; L.counts[i] = e[k].d_counts + j; L.cap[i] = e[k].cap_per_list;
        }
        if (rig_on[k]) rig[i] = c->seq[k].cfg.sensors[j];
        else lmot_default_sensor(&c->prm, &rig[i]);
      }
      lrig[nl] = rig_on[k];
      lm[nl] = mk[k] = c->seq_meas[b][k];
      LMOT_CUDA(c, cudaHostGetDevicePointer((void**)&fc[nl], t->blocks[k].h_frame_counts, 0));
      lf0[++nl] = fcount;
    }
    if (host) LMOT_CUDA(c, cudaMemcpyAsync(counts, hn, (size_t)FL * sizeof(int), cudaMemcpyHostToDevice, st));
    if ((rc = boxes_pack_lists_seq_launch(c, st, L, nl, lf0, lrig, rig, lm, fc, !gf))) return rc;
  }
  if (F > 0) {
    // FRAMES entries: one group per FRAMES sequence, in sequence order.  Without a table each frame's last box-fitting CTA (or, global_frame,
    // its boxes_to_global CTA) posts the semaphore of the frame's own list, which the tick's gate kernel polls; with one, each sequence's
    // frames are concatenated into its own list and that semaphore is polled
    DetGroup g[kMaxBatch];
    int gk[kMaxBatch], G = 0;
    for (int k = 0; k < n_seq; ++k) {
      if (e[k].kind != LMOT_SEQ_FRAMES) continue;
      int* fc = nullptr;
      if (rigged) LMOT_CUDA(c, cudaHostGetDevicePointer((void**)&fc, t->blocks[k].h_frame_counts, 0));
      gk[G] = k;
      g[G++] = DetGroup{&c->seq[k].cfg, &c->seq[k].trk.th, e[k].data, e[k].n, f0[k + 1] - f0[k], e[k].timestamp_us, e[k].v_gps, e[k].yaw_gps, fc, &t->blocks[k], true};
    }
    DetUnits U;
    if ((rc = detect_front(c, bk, &c->bslots[b * c->batch_frames], st, b, g, G, stride, host, t->h_deskew, t->h_area, !rigged && !gf, U)))
      return rc;
    SeqMeas dm[kMaxBatch];
    for (int d = 0; d < G; ++d) {
      const Slot* s = U.u[U.f0[d]];
      dm[d] = mk[gk[d]] = rigged ? c->seq_meas[b][gk[d]] : SeqMeas{s->d_boxes, s->d_boxes_g, s->d_counters, s->d_det_sem};
    }
    if (rigged && (rc = boxes_concat_seq_launch(c, U.u, G, U.f0, U.rig_on, U.rig, dm, U.fc, !gf, st))) return rc;
  }
  for (int p = 0; p < S; ++p) m[p] = mk[seq[p]];
  // the measurement lists (complete on `st`, or posting their semaphores there) -> global-frame step, ONE tracker chain for the stepped
  // tables, publication; the tick's events
  if (gf && (rc = seq_global_launch(c, seq, m, S, st, ts, v, yaw))) return rc;
  LMOT_CUDA(c, cudaEventRecord(bk->ev_det_done, st));
  if ((rc = seq_tracker_launch(c, seq, m, t, S, ts, v, yaw))) return rc;
  LMOT_CUDA(c, cudaEventRecord(t->blocks[0].ev_done, c->pub_stream));
  LMOT_CUDA(c, cudaEventRecord(bk->ev_trk_done, c->pub_stream));
  if (!t->in_flight) { t->in_flight = true; ++c->seq_in_flight; }
  return LMOT_OK;
}

// lmot_seq_submit / lmot_seq_dev: every sequence steps from its frames (points / n in the set's frame layout)
static int seq_frames_tick(lmot_ctx* ctx, const float* const* points, const int* n, int n_seq, int stride, bool host, const double* ts,
                           const double* v, const double* yaw) {
  if (!ctx || ctx->c.n_seq == 0 || n_seq != ctx->c.n_seq || !points || !n || !ts || !v || !yaw) return LMOT_ERR_INVALID;
  int f0[kMaxBatch + 1];
  bool rig_on[kMaxBatch];
  seq_layout(&ctx->c, f0, rig_on);
  lmot_seq_entry e[kMaxBatch];
  for (int k = 0; k < n_seq; ++k) e[k] = lmot_seq_entry{LMOT_SEQ_FRAMES, 0, ts[k], v[k], yaw[k], points + f0[k], n + f0[k], nullptr, 0};
  return seq_tick_common(ctx, e, n_seq, stride, host);
}

// lmot_seq_track_submit / lmot_seq_track_dev: every sequence steps from its lists (host lists boxes / m, or padded device lists d_lists /
// d_counts of cap boxes each, in the set's frame layout)
static int seq_lists_tick(lmot_ctx* ctx, const float* const* boxes, const int* m, const float* d_lists, const int* d_counts, int cap, int n_seq,
                          bool host, const double* ts, const double* v, const double* yaw) {
  if (!ctx || ctx->c.n_seq == 0 || n_seq != ctx->c.n_seq || !ts || !v || !yaw) return LMOT_ERR_INVALID;
  if (host ? (!boxes || !m) : (!d_lists || !d_counts || cap < 1)) return LMOT_ERR_INVALID;
  int f0[kMaxBatch + 1];
  bool rig_on[kMaxBatch];
  seq_layout(&ctx->c, f0, rig_on);
  const float* lp[kMaxBatch];
  for (int i = 0; !host && i < f0[n_seq]; ++i) lp[i] = d_lists + (size_t)i * cap * 24;
  lmot_seq_entry e[kMaxBatch];
  for (int k = 0; k < n_seq; ++k)
    e[k] = host ? lmot_seq_entry{LMOT_SEQ_LISTS, 0, ts[k], v[k], yaw[k], boxes + f0[k], m + f0[k], nullptr, 0}
                : lmot_seq_entry{LMOT_SEQ_LISTS, 0, ts[k], v[k], yaw[k], lp + f0[k], nullptr, d_counts + f0[k], cap};
  return seq_tick_common(ctx, e, n_seq, 0, host);
}

// uncollected ticks are dropped, as lmot_batch drops uncollected results
static int seq_drop_uncollected(Ctx* c) {
  if (c->seq_in_flight > 0) {
    LMOT_CUDA(c, cudaEventSynchronize(c->seq_last->blocks[0].ev_done));    // (ticks are published in submission order)
    seq_forget(c);
  }
  return LMOT_OK;
}

int lmot_seq_submit(lmot_ctx* ctx, const float* const* points, const int* n, int n_seq, int stride_floats, const double* timestamp_us,
                    const double* v_gps, const double* yaw_gps) {
  return seq_frames_tick(ctx, points, n, n_seq, stride_floats, true, timestamp_us, v_gps, yaw_gps);
}

int lmot_seq_dev(lmot_ctx* ctx, const float* const* d_points, const int* n, int n_seq, const double* timestamp_us, const double* v_gps,
                 const double* yaw_gps) {
  return seq_frames_tick(ctx, d_points, n, n_seq, 4, false, timestamp_us, v_gps, yaw_gps);
}

int lmot_seq_collect(lmot_ctx* ctx, lmot_seq_out* out) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  if (c->seq_in_flight <= 0) return LMOT_ERR_STATE;
  SeqTick* t = &c->seq_ticks[c->seq_oldest];
  int guard = 0;
  while (!t->in_flight && guard++ < c->seq_ring) { c->seq_oldest = (c->seq_oldest + 1) % c->seq_ring; t = &c->seq_ticks[c->seq_oldest]; }
  if (!t->in_flight) return LMOT_ERR_STATE;
  const int rc = seq_collect_tick(c, t, out);
  t->in_flight = false;
  --c->seq_in_flight;
  c->seq_oldest = (c->seq_oldest + 1) % c->seq_ring;
  return rc;
}

int lmot_seq_fetch(lmot_ctx* ctx, lmot_seq_out* out) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  if (!c->seq_last) return LMOT_ERR_STATE;
  const int rc = seq_collect_tick(c, c->seq_last, out);
  seq_forget(c);
  return rc;
}

int lmot_seq(lmot_ctx* ctx, const float* const* points, const int* n, int n_seq, int stride_floats, const double* timestamp_us,
             const double* v_gps, const double* yaw_gps, lmot_seq_out* out) {
  if (!ctx) return LMOT_ERR_INVALID;
  int rc = seq_drop_uncollected(&ctx->c);
  if (rc) return rc;
  rc = lmot_seq_submit(ctx, points, n, n_seq, stride_floats, timestamp_us, v_gps, yaw_gps);
  if (rc) return rc;
  return lmot_seq_collect(ctx, out);
}

int lmot_seq_track_submit(lmot_ctx* ctx, const float* const* boxes, const int* m, int n_seq, const double* timestamp_us, const double* v_gps,
                          const double* yaw_gps) {
  return seq_lists_tick(ctx, boxes, m, nullptr, nullptr, 0, n_seq, true, timestamp_us, v_gps, yaw_gps);
}

int lmot_seq_track_dev(lmot_ctx* ctx, const float* d_lists, const int* d_counts, int n_seq, int cap_per_list, const double* timestamp_us,
                       const double* v_gps, const double* yaw_gps) {
  return seq_lists_tick(ctx, nullptr, nullptr, d_lists, d_counts, cap_per_list, n_seq, false, timestamp_us, v_gps, yaw_gps);
}

int lmot_seq_track(lmot_ctx* ctx, const float* const* boxes, const int* m, int n_seq, const double* timestamp_us, const double* v_gps,
                   const double* yaw_gps, lmot_seq_out* out) {
  if (!ctx) return LMOT_ERR_INVALID;
  int rc = seq_drop_uncollected(&ctx->c);
  if (rc) return rc;
  rc = lmot_seq_track_submit(ctx, boxes, m, n_seq, timestamp_us, v_gps, yaw_gps);
  if (rc) return rc;
  return lmot_seq_collect(ctx, out);
}

int lmot_seq_tick_submit(lmot_ctx* ctx, const lmot_seq_entry* e, int n_seq, int stride_floats) {
  return seq_tick_common(ctx, e, n_seq, stride_floats, true);
}

int lmot_seq_tick_dev(lmot_ctx* ctx, const lmot_seq_entry* e, int n_seq) {
  return seq_tick_common(ctx, e, n_seq, 4, false);
}

int lmot_seq_tick(lmot_ctx* ctx, const lmot_seq_entry* e, int n_seq, int stride_floats, lmot_seq_out* out) {
  if (!ctx) return LMOT_ERR_INVALID;
  int rc = seq_drop_uncollected(&ctx->c);
  if (rc) return rc;
  rc = lmot_seq_tick_submit(ctx, e, n_seq, stride_floats);
  if (rc) return rc;
  return lmot_seq_collect(ctx, out);
}

int lmot_seq_stepped(const lmot_ctx* ctx, uint32_t* mask) {
  if (!ctx || !mask) return LMOT_ERR_INVALID;
  *mask = ctx->c.seq_stepped;
  return LMOT_OK;
}

// ---------------------------------------------------------------------------------------------- device-side hand-over (multi-GPU)
// Several sensor streams on several GPUs feeding ONE tracker (SURVEY.md §8e, host/shared_tracker.cpp): detection leaves its box
// list on the device, the lists travel rank to rank with NCCL, the owner folds them in WITHOUT a host bounce.
int lmot_detect_boxes_dev(lmot_ctx* ctx, const float** d_boxes, const int** d_n_boxes) {
  if (!ctx || !d_boxes || !d_n_boxes) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  Slot* s = &c->slots[c->last_slot];       // the slot of the most recent lmot_detect_dev / lmot_frame_dev
  *d_boxes = s->d_boxes;
  *d_n_boxes = s->d_counters + CNT_N_BOXES;
  return LMOT_OK;
}

int lmot_tracker_counters_dev(lmot_ctx* ctx, int** d_n_tracks) {
  if (!ctx || !d_n_tracks) return LMOT_ERR_INVALID;
  *d_n_tracks = ctx->c.own.trk.d_trk_counters + CNT_N_TRACKS;
  return LMOT_OK;
}

// n_lists box lists of capacity cap_per_list boxes each (d_lists[l * cap_per_list * 24], lengths d_counts[l], all DEVICE memory,
// ordered after the work queued on the caller stream) are concatenated in list order and folded into the track table as ONE
// immUkfJpdaf step.  Asynchronous on the caller stream; results with lmot_frame_fetch.
int lmot_track_step_lists_dev(lmot_ctx* ctx, const float* d_lists, const int* d_counts, int n_lists, int cap_per_list, double timestamp_us,
                              double v_gps, double yaw_gps) {
  if (!ctx || !d_lists || !d_counts || n_lists < 1 || n_lists > kMaxBatch || cap_per_list < 1) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  const StreamCfg& q = c->own.cfg;
  if (q.n_sensors > 0 && n_lists > q.n_sensors) return LMOT_ERR_INVALID;     // a list without a sensor pose
  cudaSetDevice(c->device);
  int rc = batch_ensure(c, 1);              // the bank's box buffer + counters are the tracker's input
  if (rc) return rc;
  Slot* k = &c->bank[0];                    // (ordering is the caller stream's; no host synchronisation here)
  Result* r = acquire_result(c, true);
  k->res = r;
  r->n_kev = 0; r->batch_frames = 0;
  cudaStream_t st = c->stream;
  if ((rc = boxes_pack_lists_launch(c, st, d_lists, d_counts, n_lists, cap_per_list, k->d_boxes, k->d_counters, q.n_sensors > 0 ? q.sensors : nullptr)))
    return rc;
  if (c->prm.global_frame && (rc = boxes_to_global_launch(c, k, st, k->d_boxes, k->d_counters, timestamp_us, v_gps, yaw_gps, false))) return rc;
  if ((rc = tracker_launch(c, k, st, k->d_boxes, k->d_counters, timestamp_us, v_gps, yaw_gps))) return rc;
  if ((rc = tracker_publish(c, r, st))) return rc;
  LMOT_CUDA(c, cudaEventRecord(r->ev_done, st));
  LMOT_CUDA(c, cudaEventRecord(k->ev_trk_done, st));
  LMOT_CUDA(c, cudaEventRecord(k->ev_det_done, st));
  r->has_tracks = true;
  if (!r->in_flight) { r->in_flight = true; ++c->n_in_flight; }
  return LMOT_OK;
}

// ---------------------------------------------------------------------------------------------- sensor rig
int lmot_default_sensor(const lmot_params* p, lmot_sensor* out) {
  if (!out) return LMOT_ERR_INVALID;
  lmot_params d;
  if (!p) { lmot_default_params(&d); p = &d; }
  memset(out, 0, sizeof(*out));
  out->pose[0] = out->pose[5] = out->pose[10] = 1.f;
  out->h_sensor = p->h_sensor; out->t_hmin = p->t_hmin; out->t_hmax = p->t_hmax; out->sensor_height = p->sensor_height;
  return LMOT_OK;
}

// a sensor table of n (0..kMaxBatch) entries: finite values, orthonormal rotations
static bool sensors_valid(const lmot_sensor* s, int n) {
  if (n < 0 || n > kMaxBatch || (n > 0 && !s)) return false;
  for (int k = 0; k < n; ++k) {
    const lmot_sensor& e = s[k];
    const float v[4] = {e.h_sensor, e.t_hmin, e.t_hmax, e.sensor_height};
    for (float x : e.pose) if (!std::isfinite(x)) return false;
    for (float x : v) if (!std::isfinite(x)) return false;
    for (int i = 0; i < 3; ++i)           // R^T R == I within 1e-5 per element (columns of the row-major 3x4)
      for (int j = 0; j < 3; ++j) {
        double d = 0.0;
        for (int r = 0; r < 3; ++r) d += (double)e.pose[4 * r + i] * (double)e.pose[4 * r + j];
        if (std::fabs(d - (i == j ? 1.0 : 0.0)) > 1e-5) return false;
      }
  }
  return true;
}

// a stream's sensor table, host state only: ticks already submitted carry their own copy in their launch parameters
static int sensors_set(Stream& q, const lmot_sensor* s, int n) {
  if (!sensors_valid(s, n)) return LMOT_ERR_INVALID;
  for (int k = 0; k < n; ++k) q.cfg.sensors[k] = s[k];
  q.cfg.n_sensors = n;
  return LMOT_OK;
}

static int sensors_get(const Stream* q, lmot_sensor* s, int cap, int* n) {
  if (!q || cap < 0 || (cap > 0 && !s)) return LMOT_ERR_INVALID;
  if (n) *n = q->cfg.n_sensors;
  for (int k = 0; k < q->cfg.n_sensors && k < cap; ++k) s[k] = q->cfg.sensors[k];
  return LMOT_OK;
}

int lmot_set_sensors(lmot_ctx* ctx, const lmot_sensor* s, int n) {
  Stream* q = stream_at(ctx, kOwnStream);
  if (!q) return LMOT_ERR_INVALID;
  q->cfg.acc.forget();                 // sweep accumulation: the history starts empty again (set or not)
  return sensors_set(*q, s, n);
}

int lmot_get_sensors(const lmot_ctx* ctx, lmot_sensor* s, int cap, int* n) { return sensors_get(stream_at(ctx, kOwnStream), s, cap, n); }

// sequence k's table: its frames of later ticks, in table order.  A tick's frames (one per sequence without a table) stay within kMaxBatch
int lmot_seq_set_sensors(lmot_ctx* ctx, int k, const lmot_sensor* s, int n) {
  Stream* q = stream_at(ctx, k);
  if (!q || !sensors_valid(s, n)) return LMOT_ERR_INVALID;
  q->cfg.acc.forget();                 // sweep accumulation: the history starts empty again (set or not)
  int frames = 0;
  for (int j = 0; j < ctx->c.n_seq; ++j) {
    const int nj = j == k ? n : ctx->c.seq[j].cfg.n_sensors;
    frames += nj > 0 ? nj : 1;
  }
  return frames > kMaxBatch ? LMOT_ERR_INVALID : sensors_set(*q, s, n);
}

int lmot_seq_get_sensors(const lmot_ctx* ctx, int k, lmot_sensor* s, int cap, int* n) { return sensors_get(stream_at(ctx, k), s, cap, n); }

// ---- merging rigs (rig_merge.cu).  The history is forgotten also when `on` is refused
static int rig_merge_set(Stream* q, int on) {
  if (!q) return LMOT_ERR_INVALID;
  q->cfg.acc.forget();
  if (on != 0 && on != 1) return LMOT_ERR_INVALID;
  q->cfg.rig_merge = on != 0;
  return LMOT_OK;
}

static int rig_merge_get(const Stream* q, int* on) {
  if (!q || !on) return LMOT_ERR_INVALID;
  *on = q->cfg.rig_merge ? 1 : 0;
  return LMOT_OK;
}

int lmot_set_rig_merge(lmot_ctx* ctx, int on) { return rig_merge_set(stream_at(ctx, kOwnStream), on); }
int lmot_get_rig_merge(const lmot_ctx* ctx, int* on) { return rig_merge_get(stream_at(ctx, kOwnStream), on); }
int lmot_seq_set_rig_merge(lmot_ctx* ctx, int k, int on) { return rig_merge_set(stream_at(ctx, k), on); }
int lmot_seq_get_rig_merge(const lmot_ctx* ctx, int k, int* on) { return rig_merge_get(stream_at(ctx, k), on); }

int lmot_seq_frame_counts(lmot_ctx* ctx, int k, int counts[LMOT_MAX_BATCH][4], int* n_frames) {
  const Stream* q = stream_at(ctx, k);
  if (!q || !counts) return LMOT_ERR_INVALID;
  if (n_frames) *n_frames = q->fc_n;
  for (int j = 0; j < q->fc_n; ++j)
    for (int i = 0; i < 4; ++i) counts[j][i] = q->fc[j][i];
  return LMOT_OK;
}

// ---------------------------------------------------------------------------------------------- tracker parameters
int lmot_default_tracker_params(lmot_tracker_params* p) {
  if (!p) return LMOT_ERR_INVALID;
  *p = tracker_params_defaults();
  return LMOT_OK;
}

static bool tracker_params_valid(const lmot_tracker_params& p) {
  const double pos[] = {p.gamma_g, p.std_a[0], p.std_a[1], p.std_a[2], p.std_yawdd[0], p.std_yawdd[1], p.std_yawdd[2], p.std_las_x,
                        p.std_las_y, p.p0_diag[0], p.p0_diag[1], p.p0_diag[2], p.p0_diag[3], p.p0_diag[4]};
  const double prob[] = {p.p_g, p.p_d, p.mode_prob0[0], p.mode_prob0[1], p.mode_prob0[2]};
  const double other[] = {p.distance_thres, p.bb_yaw_change_thres, p.second_init_v, p.static_dist};
  for (double v : pos) if (!std::isfinite(v) || !(v > 0)) return false;
  for (double v : prob) if (!std::isfinite(v) || !(v > 0 && v <= 1)) return false;
  for (double v : other) if (!std::isfinite(v)) return false;
  for (int j = 0; j < 3; ++j) {
    bool any = false;
    for (int i = 0; i < 3; ++i) {
      const double v = p.trans[i][j];
      if (!std::isfinite(v) || v < 0 || v > 1) return false;
      any |= v > 0;
    }
    if (!any) return false;
  }
  return p.lifetime_thres >= 0 && p.static_lifetime >= 0;
}

// host state only, as the sensor tables: submitted steps carry their own copy in their launch parameters
static int tracker_params_set(Stream* s, const lmot_tracker_params* p) {
  if (!s || (p && !tracker_params_valid(*p))) return LMOT_ERR_INVALID;
  const lmot_tracker_params d = tracker_params_defaults();
  Tracker& t = s->trk;
  t.prm = p ? *p : d;
  // field by field (a caller's struct may carry anything in its padding)
  const lmot_tracker_params& q = t.prm;
  bool same = q.gamma_g == d.gamma_g && q.p_g == d.p_g && q.p_d == d.p_d && q.distance_thres == d.distance_thres &&
              q.lifetime_thres == d.lifetime_thres && q.bb_yaw_change_thres == d.bb_yaw_change_thres && q.second_init_v == d.second_init_v &&
              q.static_lifetime == d.static_lifetime && q.static_dist == d.static_dist && q.std_las_x == d.std_las_x && q.std_las_y == d.std_las_y;
  for (int m = 0; m < 3; ++m) same = same && q.std_a[m] == d.std_a[m] && q.std_yawdd[m] == d.std_yawdd[m] && q.mode_prob0[m] == d.mode_prob0[m];
  for (int i = 0; i < 9; ++i) same = same && q.trans[i / 3][i % 3] == d.trans[i / 3][i % 3];
  for (int i = 0; i < 5; ++i) same = same && q.p0_diag[i] == d.p0_diag[i];
  t.tuned = !same;
  return LMOT_OK;
}

static int tracker_params_get(const Stream* s, lmot_tracker_params* p) {
  if (!s || !p) return LMOT_ERR_INVALID;
  *p = s->trk.prm;
  return LMOT_OK;
}

int lmot_set_tracker_params(lmot_ctx* ctx, const lmot_tracker_params* p) { return tracker_params_set(stream_at(ctx, kOwnStream), p); }
int lmot_get_tracker_params(const lmot_ctx* ctx, lmot_tracker_params* p) { return tracker_params_get(stream_at(ctx, kOwnStream), p); }
int lmot_seq_set_tracker_params(lmot_ctx* ctx, int k, const lmot_tracker_params* p) { return tracker_params_set(stream_at(ctx, k), p); }
int lmot_seq_get_tracker_params(const lmot_ctx* ctx, int k, lmot_tracker_params* p) { return tracker_params_get(stream_at(ctx, k), p); }

// ---------------------------------------------------------------------------------------------- detection parameters of a sequence
int lmot_default_detect_params(const lmot_params* p, lmot_detect_params* out) {
  if (!out) return LMOT_ERR_INVALID;
  lmot_params d;
  if (!p) { lmot_default_params(&d); p = &d; }
  *out = detect_params_of(*p);
  return LMOT_OK;
}

// What the kernels evaluate exactly.  The range window: the guarded fast path of the polar cell index (ground.cu polar_cell_fast) has
// an error in bin units that grows with r_max / (r_max - r_min) (DESIGN.md §6d); a window of at least r_max / 5 keeps it below half
// of the guard band.  ram_points: box fitting's table of mt19937_64 draws (boxfit.cu boxfit_alloc_shared).
static bool detect_params_valid(const lmot_detect_params& d) {
  const float f[] = {d.r_min, d.r_max, d.t_hmin, d.t_hmax, d.t_hdiff, d.h_sensor, d.filter_z_min, d.filter_z_max, d.filter_x_min,
                     d.filter_x_max, d.filter_y_min, d.filter_y_max, d.roi_m, d.sensor_height, d.t_height_min, d.t_height_max,
                     d.t_width_min, d.t_width_max, d.t_len_min, d.t_len_max, d.t_area_max, d.t_ratio_min, d.t_ratio_max, d.min_len_ratio,
                     d.t_pt_per_m3};
  for (float v : f) if (!std::isfinite(v)) return false;
  if (!std::isfinite(d.ground_tolerance)) return false;
  if (!(d.r_min >= 0.f) || !(d.r_max > d.r_min)) return false;
  if (!((double)d.r_max - (double)d.r_min >= (double)d.r_max / 5.0)) return false;
  if (!(d.roi_m > 0.f)) return false;
  if (d.rule_filter != LMOT_RULE_INTENDED && d.rule_filter != LMOT_RULE_GCC13_O2_COMPAT) return false;
  return d.ram_points >= 1 && d.ram_points <= LMOT_MAX_RAM_POINTS;
}

// host state only, as the sensor tables: submitted ticks carry their own copy in their launch parameters
int lmot_seq_set_detect_params(lmot_ctx* ctx, int k, const lmot_detect_params* p) {
  Stream* s = stream_at(ctx, k);
  if (!s || (p && !detect_params_valid(*p))) return LMOT_ERR_INVALID;
  s->cfg.det_on = p != nullptr;
  if (p) s->cfg.det = *p;
  return LMOT_OK;
}

int lmot_seq_get_detect_params(const lmot_ctx* ctx, int k, lmot_detect_params* p) {
  const Stream* s = stream_at(ctx, k);
  if (!s || !p) return LMOT_ERR_INVALID;
  *p = s->cfg.det_on ? s->cfg.det : detect_params_of(ctx->c.prm);
  return LMOT_OK;
}

// ---------------------------------------------------------------------------------------------- sweep deskew
int lmot_default_deskew(lmot_deskew* d) {
  if (!d) return LMOT_ERR_INVALID;
  *d = deskew_defaults();
  return LMOT_OK;
}

static bool deskew_valid(const lmot_deskew& d) {
  const double f[] = {d.time_scale, d.time_offset, d.t_min, d.t_max};
  for (double x : f) if (!std::isfinite(x)) return false;
  return d.t_min < d.t_max && d.t_max - d.t_min <= 1.0 && d.time_field >= 3;
}

// d (NULL: the defaults) validated; turning deskew on allocates the pinned table blocks of the stream's ring (once).  Host state only, as
// the sensor tables: submitted frames carry their own tables and launch parameters
static int deskew_set(lmot_ctx* ctx, long long k, const lmot_deskew* d) {
  Stream* s = stream_at(ctx, k);
  lmot_deskew v = d ? *d : deskew_defaults();
  if (!s || !deskew_valid(v)) return LMOT_ERR_INVALID;
  v.on = v.on ? 1 : 0;
  if (v.on) {
    Ctx* c = &ctx->c;
    cudaSetDevice(c->device);
    for (int i = 0; i < ring_size(c, k); ++i) {
      float** p = ring_pins(c, k, i).deskew;
      if (!*p) LMOT_CUDA(c, cudaHostAlloc((void**)p, kMaxBatch * kDeskewTabBytes, cudaHostAllocDefault));
    }
  }
  s->cfg.deskew = v;
  return LMOT_OK;
}

static int deskew_get(const Stream* s, lmot_deskew* d) {
  if (!s || !d) return LMOT_ERR_INVALID;
  *d = s->cfg.deskew;
  return LMOT_OK;
}

int lmot_set_deskew(lmot_ctx* ctx, const lmot_deskew* d) { return deskew_set(ctx, kOwnStream, d); }
int lmot_get_deskew(const lmot_ctx* ctx, lmot_deskew* d) { return deskew_get(stream_at(ctx, kOwnStream), d); }
int lmot_seq_set_deskew(lmot_ctx* ctx, int k, const lmot_deskew* d) { return deskew_set(ctx, k, d); }
int lmot_seq_get_deskew(const lmot_ctx* ctx, int k, lmot_deskew* d) { return deskew_get(stream_at(ctx, k), d); }

int lmot_deskew_table(const lmot_deskew* d, double v, double omega, const lmot_sensor* mount, float out[LMOT_DESKEW_SLICES][12]) {
  if (!d || !out || !deskew_valid(*d) || !std::isfinite(v) || !std::isfinite(omega) || (mount && !sensors_valid(mount, 1))) return LMOT_ERR_INVALID;
  return deskew_table(*d, v, omega, mount, &out[0][0]);
}

// ---- sweep accumulation (accumulate.cu).  Host state, as deskew: turning it on pins each result block's count block (once)
int lmot_default_accumulate(lmot_accumulate* a) {
  if (!a) return LMOT_ERR_INVALID;
  *a = accumulate_defaults();
  return LMOT_OK;
}

// a (NULL: the defaults) validated into the stream's setting; turning it on pins the count rows of the stream's result blocks (once).  The
// history starts empty again.
static int accumulate_set(lmot_ctx* ctx, long long k, const lmot_accumulate* a) {
  Stream* s = stream_at(ctx, k);
  const lmot_accumulate v = a ? *a : accumulate_defaults();
  if (!s || !accumulate_valid(v)) return LMOT_ERR_INVALID;
  if (v.sweeps > 1) {
    Ctx* c = &ctx->c;
    cudaSetDevice(c->device);
    for (int i = 0; i < ring_size(c, k); ++i) {
      int** p = ring_pins(c, k, i).acc;
      if (!*p) {
        LMOT_CUDA(c, cudaHostAlloc((void**)p, 4 * kMaxBatch * sizeof(int), cudaHostAllocMapped));
        memset(*p, 0, 4 * kMaxBatch * sizeof(int));
      }
    }
  }
  s->cfg.acc.cfg = v;
  s->cfg.acc.forget();                 // (the next accumulate launch is ordered behind every earlier one: entry 0 is free)
  return LMOT_OK;
}

static int accumulate_get(const Stream* s, lmot_accumulate* a) {
  if (!s || !a) return LMOT_ERR_INVALID;
  *a = s->cfg.acc.cfg;
  return LMOT_OK;
}

static int accumulate_info(const Stream* s, lmot_accum_info* out) {
  if (!s || !out) return LMOT_ERR_INVALID;
  *out = s->acc_info;
  return LMOT_OK;
}

int lmot_set_accumulate(lmot_ctx* ctx, const lmot_accumulate* a) { return accumulate_set(ctx, kOwnStream, a); }
int lmot_get_accumulate(const lmot_ctx* ctx, lmot_accumulate* a) { return accumulate_get(stream_at(ctx, kOwnStream), a); }
int lmot_seq_set_accumulate(lmot_ctx* ctx, int k, const lmot_accumulate* a) { return accumulate_set(ctx, k, a); }
int lmot_seq_get_accumulate(const lmot_ctx* ctx, int k, lmot_accumulate* a) { return accumulate_get(stream_at(ctx, k), a); }
int lmot_accumulate_info(lmot_ctx* ctx, lmot_accum_info* out) { return accumulate_info(stream_at(ctx, kOwnStream), out); }
int lmot_seq_accumulate_info(lmot_ctx* ctx, int k, lmot_accum_info* out) { return accumulate_info(stream_at(ctx, k), out); }

int lmot_accumulate_pose(const double fold_s[3], const double fold_t[3], const lmot_sensor* mount, float out[12]) {
  if (!fold_s || !fold_t || !out || (mount && !sensors_valid(mount, 1))) return LMOT_ERR_INVALID;
  accumulate_pose(fold_s, fold_t, mount ? mount->pose : nullptr, out);
  return LMOT_OK;
}

// ---- box search (box_search.cu).  Host state, as deskew: the launch parameters carry each unit's A; the first setter that turns it on
// uploads the angle tables
int lmot_default_box_search(lmot_box_search* b) {
  if (!b) return LMOT_ERR_INVALID;
  *b = box_search_defaults();
  return LMOT_OK;
}

static int box_search_set(lmot_ctx* ctx, long long k, const lmot_box_search* b) {
  Stream* s = stream_at(ctx, k);
  const lmot_box_search v = b ? *b : box_search_defaults();
  if (!s || !box_search_valid(v)) return LMOT_ERR_INVALID;
  if (v.on) {
    cudaSetDevice(ctx->c.device);
    const int rc = box_search_ensure(&ctx->c);
    if (rc) return rc;
  }
  s->cfg.search = v;
  return LMOT_OK;
}

static int box_search_get(const Stream* s, lmot_box_search* b) {
  if (!s || !b) return LMOT_ERR_INVALID;
  *b = s->cfg.search;
  return LMOT_OK;
}

int lmot_set_box_search(lmot_ctx* ctx, const lmot_box_search* b) { return box_search_set(ctx, kOwnStream, b); }
int lmot_get_box_search(const lmot_ctx* ctx, lmot_box_search* b) { return box_search_get(stream_at(ctx, kOwnStream), b); }
int lmot_seq_set_box_search(lmot_ctx* ctx, int k, const lmot_box_search* b) { return box_search_set(ctx, k, b); }
int lmot_seq_get_box_search(const lmot_ctx* ctx, int k, lmot_box_search* b) { return box_search_get(stream_at(ctx, k), b); }

// ---- scan-matched ego motion (ego_match.cu).  Synchronous calls on the context's matcher stream; the frame pipeline never reads it
int lmot_default_ego_match(lmot_ego_match* m) {
  if (!m) return LMOT_ERR_INVALID;
  *m = ego_match_defaults();
  return LMOT_OK;
}

static int ego_match_set(Stream* s, const lmot_ego_match* m) {
  const lmot_ego_match v = m ? *m : ego_match_defaults();
  if (!s || !ego_match_valid(v)) return LMOT_ERR_INVALID;
  s->ego.cfg = v;
  s->ego.reset();
  return LMOT_OK;
}

static int ego_match_get(const Stream* s, lmot_ego_match* m) {
  if (!s || !m) return LMOT_ERR_INVALID;
  *m = s->ego.cfg;
  return LMOT_OK;
}

static int ego_reset(Stream* s) {
  if (!s) return LMOT_ERR_INVALID;
  s->ego.reset();
  return LMOT_OK;
}

int lmot_set_ego_match(lmot_ctx* ctx, const lmot_ego_match* m) { return ego_match_set(stream_at(ctx, kOwnStream), m); }
int lmot_get_ego_match(const lmot_ctx* ctx, lmot_ego_match* m) { return ego_match_get(stream_at(ctx, kOwnStream), m); }
int lmot_seq_set_ego_match(lmot_ctx* ctx, int k, const lmot_ego_match* m) { return ego_match_set(stream_at(ctx, k), m); }
int lmot_seq_get_ego_match(const lmot_ctx* ctx, int k, lmot_ego_match* m) { return ego_match_get(stream_at(ctx, k), m); }
int lmot_ego_reset(lmot_ctx* ctx) { return ego_reset(stream_at(ctx, kOwnStream)); }
int lmot_seq_ego_reset(lmot_ctx* ctx, int k) { return ego_reset(stream_at(ctx, k)); }

// the own stream (k0 = kOwnStream, one frame) or every sequence whose frame is non-NULL: validate all, then one run over them
static int ego_estimate_common(lmot_ctx* ctx, long long k0, int n_seq, const float* const* pts, const int* n, int stride, const double* ts,
                               bool host, lmot_ego_out* out) {
  if (!ctx || !pts || !n || !ts || !out || stride < 3) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  if (k0 != kOwnStream && (c->n_seq == 0 || n_seq != c->n_seq)) return LMOT_ERR_INVALID;
  if (c->timing) return LMOT_ERR_STATE;
  EgoMatch* q[kMaxBatch];
  const float* p[kMaxBatch];
  int nn[kMaxBatch];
  double tt[kMaxBatch];
  const lmot_sensor* pose[kMaxBatch];
  lmot_ego_out* o[kMaxBatch];
  int S = 0;
  for (int i = 0; i < n_seq; ++i) {
    if (!pts[i]) continue;
    Stream* s = stream_at(ctx, k0 == kOwnStream ? k0 : i);
    const int j = s->ego.cfg.sensor;
    if (n[i] < 0 || (j >= 0 && j >= s->cfg.n_sensors)) return LMOT_ERR_INVALID;
    if (!host && ((uintptr_t)pts[i] & 15)) return LMOT_ERR_INVALID;
    q[S] = &s->ego; p[S] = pts[i]; nn[S] = n[i]; tt[S] = ts[i]; pose[S] = j >= 0 ? &s->cfg.sensors[j] : nullptr; o[S] = &out[i];
    ++S;
  }
  cudaSetDevice(c->device);
  return ego_estimate_run(c, q, p, nn, stride, tt, pose, S, host, o);
}

alignas(16) static const float kNoPoints[4] = {};   // an empty frame may come without data: never read

int lmot_ego_estimate(lmot_ctx* ctx, const float* points, int n, int stride_floats, double timestamp_us, lmot_ego_out* out) {
  if (!points && n == 0) points = kNoPoints;
  return ego_estimate_common(ctx, kOwnStream, 1, &points, &n, stride_floats, &timestamp_us, true, out);
}
int lmot_ego_estimate_dev(lmot_ctx* ctx, const float* d_points, int n, double timestamp_us, lmot_ego_out* out) {
  if (!d_points && n == 0) d_points = kNoPoints;
  return ego_estimate_common(ctx, kOwnStream, 1, &d_points, &n, 4, &timestamp_us, false, out);
}
int lmot_seq_ego_estimate(lmot_ctx* ctx, const float* const* points, const int* n, int n_seq, int stride_floats, const double* timestamp_us,
                          lmot_ego_out* out) {
  return ego_estimate_common(ctx, 0, n_seq, points, n, stride_floats, timestamp_us, true, out);
}
int lmot_seq_ego_estimate_dev(lmot_ctx* ctx, const float* const* d_points, const int* n, int n_seq, const double* timestamp_us,
                              lmot_ego_out* out) {
  return ego_estimate_common(ctx, 0, n_seq, d_points, n, 4, timestamp_us, false, out);
}

int lmot_box_search_angles(int n_angles, float out[][2]) {
  if (!out || n_angles < 1 || n_angles > LMOT_BOX_SEARCH_MAX_ANGLES) return LMOT_ERR_INVALID;
  box_search_table(n_angles, out);
  return LMOT_OK;
}

// ---- ground lines (ground_lines.cuh).  Host state, as box search: the launch parameters carry each frame's values
int lmot_default_ground_lines(lmot_ground_lines* g) {
  if (!g) return LMOT_ERR_INVALID;
  *g = ground_lines_defaults();
  return LMOT_OK;
}

static bool ground_lines_valid(const lmot_ground_lines& g) {
  return (g.on == 0 || g.on == 1) && std::isfinite(g.max_slope) && std::isfinite(g.max_rmse) && std::isfinite(g.max_step) &&
         g.max_slope > 0 && g.max_rmse > 0 && g.max_step > 0;
}

static int ground_lines_set(Stream* s, const lmot_ground_lines* g) {
  const lmot_ground_lines v = g ? *g : ground_lines_defaults();
  if (!s || !ground_lines_valid(v)) return LMOT_ERR_INVALID;
  s->cfg.lines = v;
  return LMOT_OK;
}

static int ground_lines_get(const Stream* s, lmot_ground_lines* g) {
  if (!s || !g) return LMOT_ERR_INVALID;
  *g = s->cfg.lines;
  return LMOT_OK;
}

int lmot_set_ground_lines(lmot_ctx* ctx, const lmot_ground_lines* g) { return ground_lines_set(stream_at(ctx, kOwnStream), g); }
int lmot_get_ground_lines(const lmot_ctx* ctx, lmot_ground_lines* g) { return ground_lines_get(stream_at(ctx, kOwnStream), g); }
int lmot_seq_set_ground_lines(lmot_ctx* ctx, int k, const lmot_ground_lines* g) { return ground_lines_set(stream_at(ctx, k), g); }
int lmot_seq_get_ground_lines(const lmot_ctx* ctx, int k, lmot_ground_lines* g) { return ground_lines_get(stream_at(ctx, k), g); }

int lmot_ground_lines_grid(const lmot_ground_lines* g, const float minz[LMOT_NUM_CHANNEL * LMOT_NUM_BIN], double r_min, double r_max,
                           double sensor_height, float gz[LMOT_NUM_CHANNEL * LMOT_NUM_BIN]) {
  if (!g || !minz || !gz || !ground_lines_valid(*g) || !std::isfinite(r_min) || !std::isfinite(r_max) || !std::isfinite(sensor_height) ||
      !(r_max > r_min))
    return LMOT_ERR_INVALID;
  struct Src { const float* z; float operator()(int b) const { return z[b]; } };
  struct Dst { float* o; void operator()(int b, float v) const { o[b] = v; } };
  for (int ch = 0; ch < kNumChannel; ++ch)
    ground_lines_channel(Src{minz + ch * kNumBin}, Dst{gz + ch * kNumBin}, r_min, r_max, sensor_height, g->max_slope, g->max_rmse, g->max_step);
  return LMOT_OK;
}

int lmot_debug_ground_lines(lmot_ctx* ctx, float* gz, int cap_units, int* n_units) {
  if (!ctx || cap_units < 0 || (cap_units > 0 && !gz)) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  int rc = lmot_sync(ctx);
  if (rc) return rc;
  if (n_units) *n_units = c->n_gz_dbg;
  const int n = c->n_gz_dbg < cap_units ? c->n_gz_dbg : cap_units;
  for (int i = 0; i < n; ++i)
    LMOT_CUDA(c, cudaMemcpy(gz + (size_t)i * kPolarCells, c->gz_dbg[i], kPolarCells * sizeof(float), cudaMemcpyDeviceToHost));
  return LMOT_OK;
}

// ---- layered clustering (layers.cu).  Host state, as ground lines: the launch parameters carry each unit's values
int lmot_default_layers(lmot_layers* l) {
  if (!l) return LMOT_ERR_INVALID;
  *l = layers_defaults();
  return LMOT_OK;
}

static int layers_set(Stream* s, const lmot_layers* l) {
  const lmot_layers v = l ? *l : layers_defaults();
  if (!s || !layers_valid(v)) return LMOT_ERR_INVALID;
  s->cfg.layers = v;
  return LMOT_OK;
}

static int layers_get(const Stream* s, lmot_layers* l) {
  if (!s || !l) return LMOT_ERR_INVALID;
  *l = s->cfg.layers;
  return LMOT_OK;
}

int lmot_set_layers(lmot_ctx* ctx, const lmot_layers* l) { return layers_set(stream_at(ctx, kOwnStream), l); }
int lmot_get_layers(const lmot_ctx* ctx, lmot_layers* l) { return layers_get(stream_at(ctx, kOwnStream), l); }
int lmot_seq_set_layers(lmot_ctx* ctx, int k, const lmot_layers* l) { return layers_set(stream_at(ctx, k), l); }
int lmot_seq_get_layers(const lmot_ctx* ctx, int k, lmot_layers* l) { return layers_get(stream_at(ctx, k), l); }

int lmot_debug_point_clusters(lmot_ctx* ctx, int32_t* ids, int cap, int* n_units, int n_points[LMOT_MAX_BATCH]) {
  if (!ctx || cap < 0 || (cap > 0 && !ids)) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  int rc = lmot_sync(ctx);
  if (rc) return rc;
  int n[kMaxBatch], tot = 0;
  for (int u = 0; u < c->n_lay_dbg; ++u) {
    LMOT_CUDA(c, cudaMemcpy(&n[u], c->lay_dbg[u]->d_counters + CNT_N_ELEV, sizeof(int), cudaMemcpyDeviceToHost));
    tot += n[u];
    if (n_points) n_points[u] = n[u];
  }
  if (n_units) *n_units = c->n_lay_dbg;
  if (tot > cap) return LMOT_ERR_CAPACITY;
  for (int u = 0, off = 0; u < c->n_lay_dbg; off += n[u], ++u)
    if ((rc = layers_point_ids(c, c->lay_dbg[u], n[u], ids + off))) return rc;
  return LMOT_OK;
}

// ---- obstacle footprints (obstacles.cu).  Host state, as layered clustering: the launch parameters carry each unit's values; results are
// read from the host copy collect_result took of the step most recently returned
int lmot_default_obstacles(lmot_obstacles* o) {
  if (!o) return LMOT_ERR_INVALID;
  *o = obstacles_defaults();
  return LMOT_OK;
}

static int obstacles_set(Stream* s, const lmot_obstacles* o) {
  const lmot_obstacles v = o ? *o : obstacles_defaults();
  if (!s || !obstacles_valid(v)) return LMOT_ERR_INVALID;
  s->cfg.obs = v;
  return LMOT_OK;
}

static int obstacles_get(const Stream* s, lmot_obstacles* o) {
  if (!s || !o) return LMOT_ERR_INVALID;
  *o = s->cfg.obs;
  return LMOT_OK;
}

static int obstacles_result(const Stream* s, int unit, lmot_obstacles_out* out) {
  if (!s || !out || out->cap_obstacles < 0 || out->cap_vertices < 0) return LMOT_ERR_INVALID;
  const ObsLast& L = s->obs_last;
  if (!L.valid) return LMOT_ERR_STATE;
  if (unit < 0 || unit >= L.units) return LMOT_ERR_INVALID;
  out->n_units = L.units;
  out->n_obstacles = L.n_obs[unit];
  out->n_vertices = L.n_vert[unit];
  const int K = L.n_obs[unit], nv = (int)(L.xy[unit].size() / 2);
  bool short_arr = false;
  if (out->obstacles) {
    const int m = K < out->cap_obstacles ? K : out->cap_obstacles;
    if (m > 0) memcpy(out->obstacles, L.rows[unit].data(), (size_t)m * sizeof(lmot_obstacle));
    short_arr |= K > out->cap_obstacles;
  }
  if (out->vertices) {
    const int m = nv < out->cap_vertices ? nv : out->cap_vertices;
    if (m > 0) memcpy(out->vertices, L.xy[unit].data(), (size_t)m * 2 * sizeof(float));
    short_arr |= nv > out->cap_vertices;
  }
  return (short_arr || L.n_vert[unit] > L.max_vertices[unit]) ? LMOT_ERR_CAPACITY : LMOT_OK;
}

int lmot_set_obstacles(lmot_ctx* ctx, const lmot_obstacles* o) { return obstacles_set(stream_at(ctx, kOwnStream), o); }
int lmot_get_obstacles(const lmot_ctx* ctx, lmot_obstacles* o) { return obstacles_get(stream_at(ctx, kOwnStream), o); }
int lmot_seq_set_obstacles(lmot_ctx* ctx, int k, const lmot_obstacles* o) { return obstacles_set(stream_at(ctx, k), o); }
int lmot_seq_get_obstacles(const lmot_ctx* ctx, int k, lmot_obstacles* o) { return obstacles_get(stream_at(ctx, k), o); }
int lmot_obstacles_result(lmot_ctx* ctx, int unit, lmot_obstacles_out* out) { return obstacles_result(stream_at(ctx, kOwnStream), unit, out); }
int lmot_seq_obstacles_result(lmot_ctx* ctx, int k, int unit, lmot_obstacles_out* out) { return obstacles_result(stream_at(ctx, k), unit, out); }

// ---- detection areas (detect_area.cu).  Host state only, as the sensor tables; setting one allocates the pinned staging blocks of the
// stream's ring (once)
static int area_set(lmot_ctx* ctx, long long k, const lmot_area* a) {
  Stream* s = stream_at(ctx, k);
  if (!s || !area_valid(a)) return LMOT_ERR_INVALID;
  if (a && a->n_rings > 0) {
    Ctx* c = &ctx->c;
    cudaSetDevice(c->device);
    for (int i = 0; i < ring_size(c, k); ++i) {
      const RingPins p = ring_pins(c, k, i);
      if (!*p.area) LMOT_CUDA(c, cudaHostAlloc((void**)p.area, (size_t)p.area_blocks * sizeof(AreaBlock), cudaHostAllocDefault));
    }
  }
  area_copy(s->cfg.area, a);
  return LMOT_OK;
}

static int area_get(const Stream* s, int* n_rings, int* ring_len, int cap_rings, int* n_vertices, double* xy, int cap_vertices,
                    int* keep_outside) {
  if (!s || cap_rings < 0 || cap_vertices < 0 || (cap_rings > 0 && !ring_len) || (cap_vertices > 0 && !xy)) return LMOT_ERR_INVALID;
  const AreaBlock& a = s->cfg.area;
  if (n_rings) *n_rings = a.n_rings;
  if (n_vertices) *n_vertices = a.n_vertices;
  if (keep_outside) *keep_outside = a.keep_outside;
  const int nr = a.n_rings < cap_rings ? a.n_rings : cap_rings, nv = a.n_vertices < cap_vertices ? a.n_vertices : cap_vertices;
  if (nr > 0) memcpy(ring_len, a.ring_len, (size_t)nr * sizeof(int));
  if (nv > 0) memcpy(xy, a.xy, (size_t)nv * 2 * sizeof(double));
  return LMOT_OK;
}

int lmot_set_detect_area(lmot_ctx* ctx, const lmot_area* area) { return area_set(ctx, kOwnStream, area); }

int lmot_get_detect_area(const lmot_ctx* ctx, int* n_rings, int* ring_len, int cap_rings, int* n_vertices, double* xy, int cap_vertices,
                         int* keep_outside) {
  return area_get(stream_at(ctx, kOwnStream), n_rings, ring_len, cap_rings, n_vertices, xy, cap_vertices, keep_outside);
}

int lmot_seq_set_detect_area(lmot_ctx* ctx, int k, const lmot_area* area) { return area_set(ctx, k, area); }

int lmot_seq_get_detect_area(const lmot_ctx* ctx, int k, int* n_rings, int* ring_len, int cap_rings, int* n_vertices, double* xy,
                             int cap_vertices, int* keep_outside) {
  return area_get(stream_at(ctx, k), n_rings, ring_len, cap_rings, n_vertices, xy, cap_vertices, keep_outside);
}

int lmot_detect_area_mask(const lmot_area* area, const lmot_sensor* mount, float roi_m, uint32_t out[LMOT_NUM_GRID * 8]) {
  if (!area || area->n_rings < 1 || !out || !area_valid(area) || !std::isfinite(roi_m) || !(roi_m > 0.f) ||
      (mount && !sensors_valid(mount, 1))) return LMOT_ERR_INVALID;
  AreaBlock* a = new (std::nothrow) AreaBlock;
  if (!a) return LMOT_ERR_INVALID;
  area_copy(*a, area);
  area_mask_host(*a, mount ? mount->pose : nullptr, roi_m, out);
  delete a;
  return LMOT_OK;
}

int lmot_debug_area_masks(lmot_ctx* ctx, uint32_t* out, int cap_units, int* n_units) {
  if (!ctx || cap_units < 0 || (cap_units > 0 && !out)) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  int rc = lmot_sync(ctx);
  if (rc) return rc;
  if (n_units) *n_units = c->n_area_dbg;
  const int n = c->n_area_dbg < cap_units ? c->n_area_dbg : cap_units;
  for (int i = 0; i < n; ++i)
    LMOT_CUDA(c, cudaMemcpy(out + (size_t)i * LMOT_NUM_GRID * 8, c->area_dbg[i], LMOT_NUM_GRID * 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  return LMOT_OK;
}

// after the table was received from another rank (NCCL broadcast into lmot_tracker_table's pointer, count already in the device
// counter lmot_tracker_counters_dev points at): rebuild the side arrays before the next step.  n = the count, as the host knows it.
int lmot_tracker_table_received(lmot_ctx* ctx, int n) {
  if (!ctx || n < 0 || n > ctx->c.prm.max_tracks) return LMOT_ERR_INVALID;
  Tracker& t = ctx->c.own.trk;
  t.h_trk_counters[CNT_N_TRACKS] = n;
  t.act_valid = false;
  t.ids_identity = true;
  t.last_trk_res = nullptr;
  return LMOT_OK;
}

int lmot_origin_points(lmot_ctx* ctx, double timestamp_us, double v_gps, double yaw_gps, double out6[6]) {
  if (!ctx || !out6) return LMOT_ERR_INVALID;
  TrackerHost h = ctx->c.own.trk.th;                   // peek: fold on a copy
  origin_points_fold(h, timestamp_us, v_gps, yaw_gps);
  out6[0] = h.egoPoint[0]; out6[1] = h.egoPoint[1]; out6[2] = h.egoPoint[2];
  out6[3] = h.egoPoint[0]; out6[4] = h.egoPoint[1]; out6[5] = h.egoPoint[2] + M_PI / 2;
  return LMOT_OK;
}

// ---------------------------------------------------------------------------------------------- tracker state
// The sequence forms of reset, load and set_ego also drop the uncollected sequence ticks: reset whatever its outcome, load and set_ego
// on success.  The own-stream forms never touch the sequence ring.
static int tracker_reset(lmot_ctx* ctx, long long k) {
  Stream* s = stream_at(ctx, k);
  if (!s) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  s->cfg.acc.forget();                 // sweep accumulation: the history starts empty again
  int rc = drain(c);
  if (rc) return rc;
  tracker_restart_host(s->trk);
  LMOT_CUDA(c, cudaMemsetAsync(s->trk.d_trk_counters, 0, CNT_COUNT * sizeof(int), c->stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->stream));
  return LMOT_OK;
}

int lmot_tracker_reset(lmot_ctx* ctx) { return tracker_reset(ctx, kOwnStream); }

int lmot_seq_tracker_reset(lmot_ctx* ctx, int k) {
  const int rc = tracker_reset(ctx, k);
  if (rc != LMOT_ERR_INVALID) seq_forget(&ctx->c);
  return rc;
}

static int fetch_trk_counters(Ctx* c, Tracker& t) {
  int rc = drain(c);
  if (rc) return rc;
  LMOT_CUDA(c, cudaMemcpyAsync(t.h_trk_counters, t.d_trk_counters, CNT_COUNT * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->stream));
  return LMOT_OK;
}

int lmot_tracker_num_tracks(lmot_ctx* ctx, int* n) {
  if (!ctx || !n) return LMOT_ERR_INVALID;
  Tracker& t = ctx->c.own.trk;
  int rc = fetch_trk_counters(&ctx->c, t);
  if (rc) return rc;
  *n = t.h_trk_counters[CNT_N_TRACKS];
  return LMOT_OK;
}

int lmot_tracker_table(lmot_ctx* ctx, void** dev_ptr, int* bytes_per_track, int* capacity) {
  if (!ctx) return LMOT_ERR_INVALID;
  if (dev_ptr) *dev_ptr = ctx->c.own.trk.d_tracks;
  if (bytes_per_track) *bytes_per_track = (int)sizeof(TrackState);
  if (capacity) *capacity = ctx->c.prm.max_tracks;
  return LMOT_OK;
}

int lmot_tracker_set_num_tracks(lmot_ctx* ctx, int n) {
  if (!ctx || n < 0 || n > ctx->c.prm.max_tracks) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  Tracker& t = c->own.trk;
  int rc = drain(c);
  if (rc) return rc;
  t.h_trk_counters[CNT_N_TRACKS] = n;
  t.act_valid = false;
  t.ids_identity = true;
  LMOT_CUDA(c, cudaMemcpyAsync(t.d_trk_counters + CNT_N_TRACKS, t.h_trk_counters + CNT_N_TRACKS, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->stream));
  return LMOT_OK;
}

// flat per-track dump, layout shared with oracle/ref_harness.cpp (documented in DESIGN.md)
enum { D_TRACKNUM = 0, D_LIFETIME = 1, D_STATIC = 2, D_VIS = 3, D_X = 4, D_P = 24, D_MODE = 124, D_ZPRED = 127, D_S = 133,
       D_K = 145, D_BESTYAW = 175, D_BBYAW = 176, D_BBAREA = 177, D_DISTINIT = 178, D_XMERGEYAW = 179, D_INITMEAS = 180,
       D_VELON = 182, D_VELO = 183, D_BBN = 186, D_BB = 187, D_BESTBBN = 211, D_BESTBB = 212, D_TOTAL = LMOT_TRACK_DUMP_DOUBLES };

static int tracker_dump(lmot_ctx* ctx, long long k, double* dumps, int cap, int* n_out) {
  Stream* s = stream_at(ctx, k);
  if (!s || cap < 0) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  Tracker& trk = s->trk;
  int rc = fetch_trk_counters(c, trk);
  if (rc) return rc;
  const int T = trk.h_trk_counters[CNT_N_TRACKS];
  if (n_out) *n_out = T;
  const int n = T < cap ? T : cap;
  if (n == 0 || !dumps) return LMOT_OK;
  std::vector<TrackState> h((size_t)n);
  LMOT_CUDA(c, cudaMemcpyAsync(h.data(), trk.d_tracks, (size_t)n * sizeof(TrackState), cudaMemcpyDeviceToHost, c->stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < n; ++i) {
    const TrackState& t = h[i];
    double* d = dumps + (size_t)i * D_TOTAL;
    memset(d, 0, sizeof(double) * D_TOTAL);
    d[D_TRACKNUM] = t.trackNum; d[D_LIFETIME] = t.lifetime; d[D_STATIC] = t.isStatic; d[D_VIS] = t.isVisBB;
    for (int m = 0; m < 4; ++m) { memcpy(d + D_X + 5 * m, t.x[m], 5 * sizeof(double)); memcpy(d + D_P + 25 * m, t.P[m], 25 * sizeof(double)); }
    for (int m = 0; m < 3; ++m) {
      d[D_MODE + m] = t.modeProb[m]; d[D_ZPRED + 2 * m] = t.zPred[m][0]; d[D_ZPRED + 2 * m + 1] = t.zPred[m][1];
      memcpy(d + D_S + 4 * m, t.S[m], 4 * sizeof(double)); memcpy(d + D_K + 10 * m, t.K[m], 10 * sizeof(double));
    }
    d[D_BESTYAW] = t.bestYaw; d[D_DISTINIT] = t.distFromInit; d[D_XMERGEYAW] = t.x_merge_yaw;
    d[D_INITMEAS] = t.initMeas[0]; d[D_INITMEAS + 1] = t.initMeas[1];
    d[D_VELON] = t.nVelo; for (int j = 0; j < t.nVelo && j < 3; ++j) d[D_VELO + j] = t.velo[j];
    d[D_BBN] = t.nBBox; for (int p = 0; p < t.nBBox && p < 8; ++p) for (int q = 0; q < 3; ++q) d[D_BB + 3 * p + q] = t.BBox[p][q];
    d[D_BESTBBN] = t.nBest; for (int p = 0; p < t.nBest && p < 8; ++p) for (int q = 0; q < 3; ++q) d[D_BESTBB + 3 * p + q] = t.bestBBox[p][q];
  }
  return T > cap ? LMOT_ERR_CAPACITY : LMOT_OK;
}

int lmot_tracker_dump(lmot_ctx* ctx, double* dumps, int cap, int* n_out) { return tracker_dump(ctx, kOwnStream, dumps, cap, n_out); }

int lmot_seq_tracker_dump(lmot_ctx* ctx, int k, double* dumps, int cap, int* n_out) { return tracker_dump(ctx, k, dumps, cap, n_out); }

// the history is forgotten before the arguments are validated
static int tracker_load(lmot_ctx* ctx, long long k, const double* dumps, int n, int init, double timestamp_us, double ego_velo,
                        double ego_yaw, double ego_pre_yaw, double ego_point_yaw) {
  Stream* s = stream_at(ctx, k);
  if (!s) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  Tracker& trk = s->trk;
  s->cfg.acc.forget();
  if (n < 0 || (n > 0 && !dumps)) return LMOT_ERR_INVALID;
  if (n > c->prm.max_tracks) return LMOT_ERR_CAPACITY;
  int rc = drain(c);
  if (rc) return rc;
  std::vector<TrackState> h((size_t)(n > 0 ? n : 1));
  for (int i = 0; i < n; ++i) {
    TrackState& t = h[i];
    memset(&t, 0, sizeof(t));
    const double* d = dumps + (size_t)i * D_TOTAL;
    t.trackNum = (int)d[D_TRACKNUM]; t.lifetime = (int)d[D_LIFETIME]; t.isStatic = d[D_STATIC] != 0; t.isVisBB = d[D_VIS] != 0;
    for (int m = 0; m < 4; ++m) { memcpy(t.x[m], d + D_X + 5 * m, 5 * sizeof(double)); memcpy(t.P[m], d + D_P + 25 * m, 25 * sizeof(double)); }
    for (int m = 0; m < 3; ++m) {
      t.modeProb[m] = d[D_MODE + m]; t.zPred[m][0] = d[D_ZPRED + 2 * m]; t.zPred[m][1] = d[D_ZPRED + 2 * m + 1];
      memcpy(t.S[m], d + D_S + 4 * m, 4 * sizeof(double)); memcpy(t.K[m], d + D_K + 10 * m, 10 * sizeof(double));
    }
    t.bestYaw = d[D_BESTYAW]; t.distFromInit = d[D_DISTINIT]; t.x_merge_yaw = d[D_XMERGEYAW];
    t.initMeas[0] = d[D_INITMEAS]; t.initMeas[1] = d[D_INITMEAS + 1];
    t.nVelo = (int)d[D_VELON]; for (int j = 0; j < t.nVelo && j < 3; ++j) t.velo[j] = d[D_VELO + j];
    t.nBBox = (int)d[D_BBN]; for (int p = 0; p < t.nBBox && p < 8; ++p) for (int q = 0; q < 3; ++q) t.BBox[p][q] = (float)d[D_BB + 3 * p + q];
    t.nBest = (int)d[D_BESTBBN]; for (int p = 0; p < t.nBest && p < 8; ++p) for (int q = 0; q < 3; ++q) t.bestBBox[p][q] = (float)d[D_BESTBB + 3 * p + q];
  }
  if (n > 0) LMOT_CUDA(c, cudaMemcpyAsync(trk.d_tracks, h.data(), (size_t)n * sizeof(TrackState), cudaMemcpyHostToDevice, c->stream));
  trk.h_trk_counters[CNT_N_TRACKS] = n;
  LMOT_CUDA(c, cudaMemsetAsync(trk.d_trk_counters, 0, CNT_COUNT * sizeof(int), c->stream));
  LMOT_CUDA(c, cudaMemcpyAsync(trk.d_trk_counters + CNT_N_TRACKS, trk.h_trk_counters + CNT_N_TRACKS, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->stream));
  trk.act_valid = false;
  trk.ids_identity = true;             // the loaded rows are numbered 0..n-1, the counter continues at n
  trk.th = TrackerHost();
  trk.th.init = init != 0; trk.th.timestamp = timestamp_us; trk.th.egoVelo = ego_velo; trk.th.egoYaw = ego_yaw;
  trk.th.egoPreYaw = ego_pre_yaw; trk.th.egoPoint[2] = ego_point_yaw;
  trk.pred_ok = true;                  // predictions start from timestamp_us
  // (like the oracle's ref_tracker_load, which clears egoDeltaHis_: the dead-reckoning fold restarts from (0, 0, -pi/2) and
  //  ego_point_yaw is only egoPoints_[0][2] until the next step recomputes it.  A checkpoint that must keep the accumulated ego
  //  pose restores it with lmot_tracker_set_ego.)
  return LMOT_OK;
}

int lmot_tracker_load(lmot_ctx* ctx, const double* dumps, int n, int init, double timestamp_us, double ego_velo,
                      double ego_yaw, double ego_pre_yaw, double ego_point_yaw) {
  return tracker_load(ctx, kOwnStream, dumps, n, init, timestamp_us, ego_velo, ego_yaw, ego_pre_yaw, ego_point_yaw);
}

int lmot_seq_tracker_load(lmot_ctx* ctx, int k, const double* dumps, int n, int init, double timestamp_us, double ego_velo, double ego_yaw,
                          double ego_pre_yaw, double ego_point_yaw) {
  const int rc = tracker_load(ctx, k, dumps, n, init, timestamp_us, ego_velo, ego_yaw, ego_pre_yaw, ego_point_yaw);
  if (rc == LMOT_OK) seq_forget(&ctx->c);
  return rc;
}

// the frame-level scalars of getOriginPoints / immUkfJpdaf (imm_ukf_jpda.cpp:19-24,56-58) incl. the accumulated dead-reckoning pose
static int tracker_get_ego(const Stream* s, double ego8[8]) {
  if (!s || !ego8) return LMOT_ERR_INVALID;
  const TrackerHost& h = s->trk.th;
  ego8[0] = h.init ? 1.0 : 0.0; ego8[1] = h.timestamp; ego8[2] = h.egoVelo; ego8[3] = h.egoYaw; ego8[4] = h.egoPreYaw;
  ego8[5] = h.fold[0]; ego8[6] = h.fold[1]; ego8[7] = h.fold[2];
  return LMOT_OK;
}

int lmot_tracker_get_ego(lmot_ctx* ctx, double ego8[8]) { return tracker_get_ego(stream_at(ctx, kOwnStream), ego8); }

int lmot_seq_tracker_get_ego(lmot_ctx* ctx, int k, double ego8[8]) { return tracker_get_ego(stream_at(ctx, k), ego8); }

static int tracker_set_ego(lmot_ctx* ctx, long long k, const double ego8[8]) {
  Stream* s = stream_at(ctx, k);
  if (!s || !ego8) return LMOT_ERR_INVALID;
  s->cfg.acc.forget();
  int rc = drain(&ctx->c);
  if (rc) return rc;
  TrackerHost& h = s->trk.th;
  h.init = ego8[0] != 0.0; h.timestamp = ego8[1]; h.egoVelo = ego8[2]; h.egoYaw = ego8[3]; h.egoPreYaw = ego8[4];
  h.fold[0] = ego8[5]; h.fold[1] = ego8[6]; h.fold[2] = ego8[7];
  h.egoPoint[0] = h.fold[0]; h.egoPoint[1] = h.fold[1]; h.egoPoint[2] = h.fold[2];
  return LMOT_OK;
}

int lmot_tracker_set_ego(lmot_ctx* ctx, const double ego8[8]) { return tracker_set_ego(ctx, kOwnStream, ego8); }

int lmot_seq_tracker_set_ego(lmot_ctx* ctx, int k, const double ego8[8]) {
  const int rc = tracker_set_ego(ctx, k, ego8);
  if (rc == LMOT_OK) seq_forget(&ctx->c);
  return rc;
}

// ---- track retirement and track IDs
static int track_retirement_set(Stream* s, int on) {
  if (!s) return LMOT_ERR_INVALID;
  s->trk.retire = on != 0;
  return LMOT_OK;
}

static int track_retirement_get(const Stream* s, int* on) {
  if (!s || !on) return LMOT_ERR_INVALID;
  *on = s->trk.retire ? 1 : 0;
  return LMOT_OK;
}

int lmot_set_track_retirement(lmot_ctx* ctx, int on) { return track_retirement_set(stream_at(ctx, kOwnStream), on); }
int lmot_get_track_retirement(const lmot_ctx* ctx, int* on) { return track_retirement_get(stream_at(ctx, kOwnStream), on); }
int lmot_seq_set_track_retirement(lmot_ctx* ctx, int k, int on) { return track_retirement_set(stream_at(ctx, k), on); }
int lmot_seq_get_track_retirement(const lmot_ctx* ctx, int k, int* on) { return track_retirement_get(stream_at(ctx, k), on); }

static int track_ids(const Stream* s, int64_t* ids, int cap, int* n) {
  if (!s || !n || cap < 0 || (cap > 0 && !ids)) return LMOT_ERR_INVALID;
  const Tracker& t = s->trk;
  if (t.ids_n < 0) return LMOT_ERR_STATE;
  *n = t.ids_n;
  const int m = t.ids_n < cap ? t.ids_n : cap;
  for (int i = 0; i < m; ++i) ids[i] = t.ids_rows ? (int64_t)i : (int64_t)t.ids_last[i];
  return LMOT_OK;
}

int lmot_track_ids(lmot_ctx* ctx, int64_t* ids, int cap, int* n) { return track_ids(stream_at(ctx, kOwnStream), ids, cap, n); }
int lmot_seq_track_ids(lmot_ctx* ctx, int k, int64_t* ids, int cap, int* n) { return track_ids(stream_at(ctx, k), ids, cap, n); }

// ---- track prediction (lmot_predict_tracks*; tracker.cu predict_launch)
static bool pred_out_valid(const lmot_pred_out& o) {
  return o.cap >= 0 && (o.cap == 0 || (o.ids && o.track_manage && o.flags && o.x && o.P && o.mode_prob));
}

// n_t in range, finite stamps, a table with a stamp, no stamp before it
static int pred_times_valid(const Tracker& t, const double* t_us, int n_t) {
  if (!t_us || n_t < 1 || n_t > LMOT_MAX_PRED_TIMES) return LMOT_ERR_INVALID;
  for (int j = 0; j < n_t; ++j) if (!std::isfinite(t_us[j])) return LMOT_ERR_INVALID;
  if (!t.pred_ok) return LMOT_ERR_STATE;
  for (int j = 0; j < n_t; ++j) if (t_us[j] < t.th.timestamp) return LMOT_ERR_INVALID;
  return LMOT_OK;
}

// the stream of the table's latest step (the prediction is ordered behind it there)
static cudaStream_t pred_stream_of(const Ctx* c, const Tracker& t) { return t.last_st ? t.last_st : c->trk_stream; }

// device outputs: the caller stream's earlier work on them comes first, and the caller stream waits for the prediction
static int predict_dev(Ctx* c, Tracker* const* tabs, int S, const double* t_us, int n_t, const lmot_pred_out* d_outs, int* const* d_n_rows,
                       cudaStream_t st) {
  if (st != c->stream) {
    if (!c->ev_pred_in) LMOT_CUDA(c, cudaEventCreateWithFlags(&c->ev_pred_in, cudaEventDisableTiming));
    LMOT_CUDA(c, cudaEventRecord(c->ev_pred_in, c->stream));
    LMOT_CUDA(c, cudaStreamWaitEvent(st, c->ev_pred_in, 0));
  }
  if (int rc = predict_launch(c, tabs, S, t_us, n_t, d_outs, d_n_rows, st)) return rc;
  if (st != c->stream) LMOT_CUDA(c, cudaStreamWaitEvent(c->stream, c->ev_pred, 0));
  return LMOT_OK;
}

// host outputs: the kernel writes a device staging area (grown to the largest request), then the rows that fit are copied out
static int predict_host(Ctx* c, Tracker& t, const double* t_us, int n_t, lmot_pred_out* out, cudaStream_t st) {
  if (!out || !pred_out_valid(*out)) return LMOT_ERR_INVALID;
  if (int rc = pred_times_valid(t, t_us, n_t)) return rc;
  const size_t cap = (size_t)out->cap, rows = (size_t)n_t * cap;
  auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t o_ids = 256, o_tm = o_ids + up(cap * 8), o_fl = o_tm + up(cap * 4), o_x = o_fl + up(rows), o_P = o_x + up(rows * 40),
               o_mp = o_P + up(rows * 200), o_gz = o_mp + up(rows * 24), o_gS = o_gz + up(rows * 16), bytes = o_gS + up(rows * 32);
  if (bytes > c->pred_stage_bytes) {
    cudaFree(c->d_pred_stage);           // (a host form has waited for its copies: nothing reads the old area)
    c->d_pred_stage = nullptr; c->pred_stage_bytes = 0;
    LMOT_CUDA(c, cudaMalloc(&c->d_pred_stage, bytes));
    c->pred_stage_bytes = bytes;
  }
  if (!c->h_pred_n) LMOT_CUDA(c, cudaHostAlloc(&c->h_pred_n, sizeof(int), cudaHostAllocDefault));
  unsigned char* b = c->d_pred_stage;
  lmot_pred_out d{out->cap, 0, reinterpret_cast<int64_t*>(b + o_ids), reinterpret_cast<int32_t*>(b + o_tm), b + o_fl,
                  reinterpret_cast<double*>(b + o_x), reinterpret_cast<double*>(b + o_P), reinterpret_cast<double*>(b + o_mp),
                  out->gate_z ? reinterpret_cast<double*>(b + o_gz) : nullptr, out->gate_S ? reinterpret_cast<double*>(b + o_gS) : nullptr};
  int* dn = reinterpret_cast<int*>(b);
  Tracker* tabs[1] = {&t};
  if (int rc = predict_launch(c, tabs, 1, t_us, n_t, &d, &dn, st)) return rc;
  LMOT_CUDA(c, cudaMemcpyAsync(c->h_pred_n, dn, sizeof(int), cudaMemcpyDeviceToHost, st));
  LMOT_CUDA(c, cudaEventRecord(c->ev_pred, st));
  LMOT_CUDA(c, cudaEventSynchronize(c->ev_pred));
  const int n = *c->h_pred_n;
  out->n_rows = n;
  const size_t m = (size_t)(n < out->cap ? n : out->cap);
  if (m > 0) {
    auto rows2d = [&](void* dst, const void* src, size_t k) {    // [n_t][cap][k] -> the first m rows of every time
      return cudaMemcpy2DAsync(dst, cap * k, src, cap * k, m * k, n_t, cudaMemcpyDeviceToHost, st);
    };
    LMOT_CUDA(c, cudaMemcpyAsync(out->ids, d.ids, m * 8, cudaMemcpyDeviceToHost, st));
    LMOT_CUDA(c, cudaMemcpyAsync(out->track_manage, d.track_manage, m * 4, cudaMemcpyDeviceToHost, st));
    LMOT_CUDA(c, rows2d(out->flags, d.flags, 1));
    LMOT_CUDA(c, rows2d(out->x, d.x, 40));
    LMOT_CUDA(c, rows2d(out->P, d.P, 200));
    LMOT_CUDA(c, rows2d(out->mode_prob, d.mode_prob, 24));
    if (out->gate_z) LMOT_CUDA(c, rows2d(out->gate_z, d.gate_z, 16));
    if (out->gate_S) LMOT_CUDA(c, rows2d(out->gate_S, d.gate_S, 32));
    LMOT_CUDA(c, cudaEventRecord(c->ev_pred, st));
    LMOT_CUDA(c, cudaEventSynchronize(c->ev_pred));
  }
  return n > out->cap ? LMOT_ERR_CAPACITY : LMOT_OK;
}

int lmot_predict_tracks(lmot_ctx* ctx, const double* t_us, int n_t, lmot_pred_out* out) {
  Stream* s = stream_at(ctx, kOwnStream);
  if (!s) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  cudaSetDevice(c->device);
  return predict_host(c, s->trk, t_us, n_t, out, pred_stream_of(c, s->trk));
}

int lmot_predict_tracks_dev(lmot_ctx* ctx, const double* t_us, int n_t, const lmot_pred_out* d_out, int* d_n_rows) {
  if (!ctx || !d_out || !pred_out_valid(*d_out)) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  Tracker* tabs[1] = {&c->own.trk};
  if (int rc = pred_times_valid(*tabs[0], t_us, n_t)) return rc;
  cudaSetDevice(c->device);
  return predict_dev(c, tabs, 1, t_us, n_t, d_out, &d_n_rows, pred_stream_of(c, *tabs[0]));
}

// a sequence's table on the tracker stream (behind the sequence ticks); refused in timing mode before the outputs are looked at
int lmot_seq_predict_tracks(lmot_ctx* ctx, int k, const double* t_us, int n_t, lmot_pred_out* out) {
  Stream* s = stream_at(ctx, k);
  if (!s) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  if (c->timing) return LMOT_ERR_STATE;
  cudaSetDevice(c->device);
  return predict_host(c, s->trk, t_us, n_t, out, c->trk_stream);
}

int lmot_seq_predict_tracks_dev(lmot_ctx* ctx, const double* t_us, int n_t, const lmot_pred_out* d_outs, int* d_n_rows) {
  if (!ctx || ctx->c.n_seq < 1 || !d_outs || !t_us || n_t < 1 || n_t > LMOT_MAX_PRED_TIMES) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  const int S = c->n_seq;
  for (int k = 0; k < S; ++k) if (!pred_out_valid(d_outs[k])) return LMOT_ERR_INVALID;
  if (c->timing) return LMOT_ERR_STATE;
  for (int k = 0; k < S; ++k) if (int rc = pred_times_valid(c->seq[k].trk, t_us + (size_t)k * n_t, n_t)) return rc;
  cudaSetDevice(c->device);
  Tracker* tabs[kMaxBatch];
  int* dn[kMaxBatch];
  for (int k = 0; k < S; ++k) { tabs[k] = &c->seq[k].trk; dn[k] = d_n_rows ? d_n_rows + k : nullptr; }
  return predict_dev(c, tabs, S, t_us, n_t, d_outs, dn, c->trk_stream);
}

// ---------------------------------------------------------------------------------------------- inspection
int lmot_debug_polar_grid(lmot_ctx* ctx, float* minz, float* height, float* smoothed, float* hdiff, float* hground,
                          uint8_t* isground) {
  if (!ctx) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  int rc = lmot_sync(ctx);
  if (rc) return rc;
  Slot* s = &c->slots[c->last_slot];
  cudaStream_t st = c->stream;
  // The fused kernel writes only what its phase 3 needs; the four intermediate grids are recomputed here from the launch's min-z
  // keys.  hGround / isGround are the fused kernel's own (stage entry points leave them in d_hg).
  if ((rc = ground_grids_debug(c, s, st))) return rc;
  const size_t b = kPolarCells * sizeof(float);
  if (minz) LMOT_CUDA(c, cudaMemcpyAsync(minz, s->d_minz, b, cudaMemcpyDeviceToHost, st));
  if (height) LMOT_CUDA(c, cudaMemcpyAsync(height, s->d_height, b, cudaMemcpyDeviceToHost, st));
  if (smoothed) LMOT_CUDA(c, cudaMemcpyAsync(smoothed, s->d_smoothed, b, cudaMemcpyDeviceToHost, st));
  if (hdiff) LMOT_CUDA(c, cudaMemcpyAsync(hdiff, s->d_hdiff, b, cudaMemcpyDeviceToHost, st));
  std::vector<float> hg, hu;
  if (hground || isground) {
    hg.resize(kPolarCells); hu.resize(kPolarCells);
    LMOT_CUDA(c, cudaMemcpyAsync(hg.data(), s->d_hg_dbg, b, cudaMemcpyDeviceToHost, st));
    LMOT_CUDA(c, cudaMemcpyAsync(hu.data(), s->d_hg, b, cudaMemcpyDeviceToHost, st));
  }
  LMOT_CUDA(c, cudaStreamSynchronize(st));
  for (int k = 0; k < kPolarCells && (hground || isground); ++k) {
    const float v = s->hg_valid ? hu[k] : hg[k];
    const bool g = !(std::isinf(v) && v < 0);
    if (hground) hground[k] = g ? v : 0.f;
    if (isground) isground[k] = g ? 1 : 0;
  }
  return LMOT_OK;
}

int lmot_debug_cell_index(lmot_ctx* ctx, int32_t* ch, int32_t* bin, int n) {
  if (!ctx || n < 0) return LMOT_ERR_INVALID;
  Ctx* c = &ctx->c;
  int rc = lmot_sync(ctx);
  if (rc) return rc;
  Slot* s = &c->slots[c->last_slot];
  if (n > s->cur_n) return LMOT_ERR_INVALID;
  std::vector<uint16_t> cell((size_t)n);
  if ((rc = ground_cells_debug(c, s, c->stream))) return rc;   // the fused kernel keeps the ids in shared memory: recompute them
  if (n) LMOT_CUDA(c, cudaMemcpyAsync(cell.data(), s->d_cell, (size_t)n * 2, cudaMemcpyDeviceToHost, c->stream));
  LMOT_CUDA(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < n; ++i) {
    if (cell[i] == kNoCell) { ch[i] = -1; bin[i] = -1; }
    else { ch[i] = cell[i] / kNumBin; bin[i] = cell[i] % kNumBin; }
  }
  return LMOT_OK;
}

int lmot_selftest_atan2f(const float* y, const float* x, int n, float* out) {
  if (n < 0 || (n > 0 && (!y || !x || !out))) return LMOT_ERR_INVALID;
  for (int i = 0; i < n; ++i) out[i] = atan2f_fdlibm(y[i], x[i]);
  return LMOT_OK;
}

int lmot_enable_timing(lmot_ctx* ctx, int on) {
  if (!ctx) return LMOT_ERR_INVALID;
  ctx->c.timing = on != 0;
  return LMOT_OK;
}

int lmot_last_kernel_ms(lmot_ctx* ctx, float* ms, int cap, int* n) {
  if (!ctx || !ms || !n) return LMOT_ERR_INVALID;
  *n = ctx->c.n_kernel_ms;
  for (int i = 0; i < ctx->c.n_kernel_ms && i < cap; ++i) ms[i] = ctx->c.kernel_ms[i];
  return LMOT_OK;
}

int lmot_debug_host_ns(lmot_ctx* ctx, double ns[4], int reset) {
  if (!ctx || !ns) return LMOT_ERR_INVALID;
  for (int i = 0; i < 4; ++i) { ns[i] = ctx->c.host_ns[i]; if (reset) ctx->c.host_ns[i] = 0; }
  return LMOT_OK;
}

int lmot_last_stage_ms(lmot_ctx* ctx, float ms[4]) {
  if (!ctx || !ms) return LMOT_ERR_INVALID;
  for (int i = 0; i < 4; ++i) ms[i] = ctx->c.stage_ms[i];
  return LMOT_OK;
}

}  // extern "C"
