// boxfit_device.cuh -- what box fitting (boxfit.cu) and box search (box_search.cu) share: a launch's per-frame buffers (FitBatch), the
// box-fitting values (BoxParams), ruleBasedFilter (rule_filter) and the programmatic-dependent-launch hooks.  Both translation units
// include it; everything here has internal linkage.
#pragma once
#include "lmot_internal.cuh"
#include "polar_cell.cuh"

namespace lmot {

namespace {

// Programmatic dependent launch inside a slot's detection stream: scatter behind tile_hist, box_fit behind scatter.  The dependent's
// CTAs become resident once EVERY CTA of the kernel before it has started (they all trigger at their first instruction) and wait there
// for it to finish -- its launch latency leaves the frame's critical path.  Deadlock-free next to the ground kernel's own barrier: a
// waiting CTA only ever waits for a grid that is completely resident and waits for nobody.  (Not used in front of tile_hist: its CTAs
// would hold SM slots for the duration of the ground kernel, slots the tracker chain needs.)
__device__ __forceinline__ void fit_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void fit_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------- B1
// One frame of a launch (blockIdx.y): every buffer the four kernels touch for it (the Slot's, see lmot_internal.cuh)
struct FitFrame {
  const uint16_t* cart; const int* label_grid; int* counters;
  uint16_t* pcid; int* table; int* seg_start; int* seg_size;
  const float4* elev; float4* sorted_pts;
  float* cl_box; float* cl_marker; uint8_t* cl_ok;
  float* boxes; float* markers; int* done; int* det_sem;
  unsigned* hist_ctr;      // atomicInc counter of finished tile_hist CTAs (wraps at the grid size: needs no reset)
  float sensor_height;     // box_fit_kernel<., true>: this frame's sensor's (lmot_set_sensors); unread otherwise
};
struct FitBatch { FitFrame f[kMaxBatch]; };

struct BoxParams {
  float roi, pic_scale, sensor_height;
  int ram_points, l_slope_dist, l_num_points, min_points, rule_mode;
  float t_height_min, t_height_max, t_width_min, t_width_max, t_len_min, t_len_max, t_area_max, t_ratio_min, t_ratio_max,
      min_len_ratio, t_pt_per_m3;
};

// ruleBasedFilter, box_fitting.cpp:97-158 (see lmot_rule_filter in lmot.h for the two modes)
__device__ bool rule_filter(const float pc[4][2], float maxZ, int n, const BoxParams& P, float sensor_height) {
  if (n < P.min_points) return false;
  const float x1 = pc[0][0], y1 = pc[0][1], x2 = pc[1][0], y2 = pc[1][1], x3 = pc[2][0], y3 = pc[2][1];
  const float dist1 = sqrtf((x1 - x2) * (x1 - x2) + (y1 - y2) * (y1 - y2));
  const float dist2 = sqrtf((x3 - x2) * (x3 - x2) + (y3 - y2) * (y3 - y2));
  float length, width;
  if (dist1 > dist2) { length = dist1; width = dist2; } else { length = dist2; width = dist1; }
  const float height = maxZ + sensor_height;
  const float area = dist1 * dist2;
  const float mass = area * height;
  const float ratio = length / width;
  if (height > P.t_height_min && height < P.t_height_max) {
    if (P.rule_mode == LMOT_RULE_GCC13_O2_COMPAT) return true;
    if (width > P.t_width_min && width < P.t_width_max)
      if (length > P.t_len_min && length < P.t_len_max)
        if (area < P.t_area_max)
          if ((float)n > mass * P.t_pt_per_m3) {
            if (length > P.min_len_ratio) { if (ratio > P.t_ratio_min && ratio < P.t_ratio_max) return true; }
            else return true;
          }
    return false;   // INTENDED: the reference falls off the end here (undefined behaviour)
  }
  return false;
}

// ground lines (lmot_set_ground_lines): unit blockIdx.y's ground grid (nullptr: flat, its BoxParams' sensor_height) and the range window of
// its polar cells
struct LinesFit { const float* gz[kMaxBatch]; float r_min[kMaxBatch], r_max[kMaxBatch], r_span[kMaxBatch]; };

// the sensor_height a cluster's box takes with ground lines: -gz of the polar cell of its lowest point (min z, ties to the first in cloud
// order), or the flat `sh` where that point is outside the window or the unit has no grid.  Every thread of the CTA calls it and gets the
// value; s_buf: one word per warp
__device__ __forceinline__ float lines_sensor_height(const float4* __restrict__ seg, int n, const LinesFit& L, float sh, unsigned long long* s_buf) {
  const float* __restrict__ gz = L.gz[blockIdx.y];
  if (!gz) return sh;
  unsigned long long key = ~0ull;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    float z = __ldg(&seg[j]).z;
    if (z == 0.f) z = 0.f;                               // -0 == +0
    const unsigned u = __float_as_uint(z);
    const unsigned long long k = ((unsigned long long)((u & 0x80000000u) ? ~u : (u | 0x80000000u)) << 32) | (unsigned)j;
    key = k < key ? k : key;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const unsigned long long v = __shfl_xor_sync(0xFFFFFFFFu, key, o); key = v < key ? v : key; }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_buf[threadIdx.x >> 5] = key;
  __syncthreads();
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { const unsigned long long v = s_buf[w]; key = v < key ? v : key; }
  key = s_buf[0] < key ? s_buf[0] : key;
  __syncthreads();                                       // (s_buf is the caller's again)
  const float4 q = __ldg(&seg[(unsigned)(key & 0xFFFFFFFFull)]);
  GroundParams p;
  p.r_min = L.r_min[blockIdx.y]; p.r_max = L.r_max[blockIdx.y]; p.r_span = L.r_span[blockIdx.y];
  const uint16_t cell = polar_cell_exact(q.x, q.y, p);
  return cell == kNoCell ? sh : -__ldg(&gz[cell]);
}

// sequence ticks with their own detection values (lmot_seq_set_detect_params): frame blockIdx.y's whole BoxParams -- ROI and picScale,
// L-shape gates, ram_points, min_points, rule mode and window, the sensor's height folded in on the host
struct BoxFrameParams { BoxParams p[kMaxBatch]; };

}  // namespace

static inline void fit_frame_of(const Slot* s, FitFrame& f, bool post_sem) {
  f.sensor_height = 0.f;
  f.cart = s->d_cart; f.label_grid = s->d_label_grid; f.counters = s->d_counters;
  f.pcid = s->d_pcid; f.table = s->d_table; f.seg_start = s->d_seg_start; f.seg_size = s->d_seg_size;
  f.elev = s->d_elev; f.sorted_pts = s->d_sorted_pts;
  f.cl_box = s->d_cl_box; f.cl_marker = s->d_cl_marker; f.cl_ok = s->d_cl_ok;
  f.boxes = s->d_boxes; f.markers = s->d_markers; f.done = s->d_done; f.det_sem = post_sem ? s->d_det_sem : nullptr;
  f.hist_ctr = reinterpret_cast<unsigned*>(s->d_done + 1);
}

// unit i's entry of a LinesFit: its ground grid gz (nullptr: flat) and the window of detection values d
static inline void lines_fit_of(const lmot_detect_params& d, const float* gz, LinesFit& L, int i) {
  L.gz[i] = gz;
  L.r_min[i] = d.r_min; L.r_max[i] = d.r_max;
  { volatile float span = d.r_max - d.r_min; L.r_span[i] = span; }      // as ground_params_of
}

// BoxParams of detection values d (the context's, or a frame's own)
static inline BoxParams box_params_of(const lmot_detect_params& p) {
  BoxParams P;
  P.roi = p.roi_m;
  { volatile float ps = 900 / p.roi_m; P.pic_scale = ps; }   // float picScale = 900/roiM (box_fitting.cpp:18)
  P.sensor_height = p.sensor_height; P.ram_points = p.ram_points; P.l_slope_dist = p.l_slope_dist;
  P.l_num_points = p.l_num_points; P.min_points = p.min_cluster_points; P.rule_mode = p.rule_filter;
  P.t_height_min = p.t_height_min; P.t_height_max = p.t_height_max; P.t_width_min = p.t_width_min; P.t_width_max = p.t_width_max;
  P.t_len_min = p.t_len_min; P.t_len_max = p.t_len_max; P.t_area_max = p.t_area_max; P.t_ratio_min = p.t_ratio_min;
  P.t_ratio_max = p.t_ratio_max; P.min_len_ratio = p.min_len_ratio; P.t_pt_per_m3 = p.t_pt_per_m3;
  return P;
}

}  // namespace lmot
