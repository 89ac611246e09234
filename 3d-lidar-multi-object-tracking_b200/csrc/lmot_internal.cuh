// lmot_internal.cuh -- context layout and launch prototypes shared by the stage translation units.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/lmot.h"

namespace lmot {

constexpr int kNumChannel = LMOT_NUM_CHANNEL;
constexpr int kNumBin = LMOT_NUM_BIN;
constexpr int kPolarCells = kNumChannel * kNumBin;  // 9600
constexpr int kNumGrid = LMOT_NUM_GRID;
constexpr int kCartCells = kNumGrid * kNumGrid;      // 62500
constexpr uint16_t kNoCell = 0xFFFFu;
constexpr uint16_t kPreFiltered = 0xFFFEu;           // removed by the ground node's pre-filters (never reaches groundRemove)
constexpr int kScanTile = 1024;                      // points per tile of the stable-partition scan
constexpr int kMaxBatch = 8;                         // frames (one per sensor stream) of one batched launch, lmot_batch_*

// device-side counters of one frame (one int each; written by kernels, read by later kernels and by fetch)
enum Counter {
  CNT_N_ELEV = 0, CNT_N_GROUND, CNT_NUM_CLUSTER, CNT_N_BOXES, CNT_N_CLUSTERED, CNT_ERROR, CNT_N_TRACKS, CNT_N_VIS,
  CNT_N_ACT,        // tracks the next frame has to visit (live, or dead with a stale isVisBB_ flag): length of d_act_list
  CNT_ACC_DONE = 14,   // accumulate_kernel's finished blocks (accumulate.cu), 0 at rest
  CNT_COUNT = 16
};

struct GroundParams {
  float r_min, r_max, t_hmin, t_hmax, t_hdiff, h_sensor;
  float r_span;          // r_max - r_min evaluated in float (ground_removal.cpp:71)
  float bin_scale;       // 120 / r_span: bins per metre of the guarded fast path (ground.cu polar_cell)
  int prefilter;         // the `ground` node's PassThrough(z) + ConditionalRemoval(x, y) in front of groundRemove
  float fz0, fz1, fx0, fx1, fy0, fy1;
  double tol;            // 0.25
  double tap[3];         // gaussKernel(3, 1.0) computed on the host with the host libm (gaus_blur.cpp:26-49)
};

// lmot_params' detection fields (lmot_default_detect_params)
inline lmot_detect_params detect_params_of(const lmot_params& p) {
  lmot_detect_params d;
  memset(&d, 0, sizeof(d));
  d.r_min = p.r_min; d.r_max = p.r_max; d.t_hmin = p.t_hmin; d.t_hmax = p.t_hmax; d.t_hdiff = p.t_hdiff; d.h_sensor = p.h_sensor;
  d.ground_tolerance = p.ground_tolerance;
  d.node_prefilter = p.node_prefilter;
  d.filter_z_min = p.filter_z_min; d.filter_z_max = p.filter_z_max; d.filter_x_min = p.filter_x_min; d.filter_x_max = p.filter_x_max;
  d.filter_y_min = p.filter_y_min; d.filter_y_max = p.filter_y_max;
  d.roi_m = p.roi_m;
  d.ram_points = p.ram_points; d.l_slope_dist = p.l_slope_dist; d.l_num_points = p.l_num_points; d.sensor_height = p.sensor_height;
  d.t_height_min = p.t_height_min; d.t_height_max = p.t_height_max; d.t_width_min = p.t_width_min; d.t_width_max = p.t_width_max;
  d.t_len_min = p.t_len_min; d.t_len_max = p.t_len_max; d.t_area_max = p.t_area_max; d.t_ratio_min = p.t_ratio_min;
  d.t_ratio_max = p.t_ratio_max; d.min_len_ratio = p.min_len_ratio; d.t_pt_per_m3 = p.t_pt_per_m3;
  d.min_cluster_points = p.min_cluster_points; d.rule_filter = p.rule_filter;
  return d;
}

// the ground kernel's parameter block of detection values d (lmot_create for the context, the sequence launches per frame: one
// evaluation of r_span / bin_scale for both, so equal values give equal bits).  tap: the Gaussian taps (gauss_taps, api.cu).
inline GroundParams ground_params_of(const lmot_detect_params& d, const double tap[3]) {
  GroundParams g;
  memset(&g, 0, sizeof(g));
  g.r_min = d.r_min; g.r_max = d.r_max; g.t_hmin = d.t_hmin; g.t_hmax = d.t_hmax; g.t_hdiff = d.t_hdiff; g.h_sensor = d.h_sensor;
  { volatile float span = d.r_max - d.r_min; g.r_span = span; }      // float, as ground_removal.cpp:71 evaluates it
  g.prefilter = d.node_prefilter ? 1 : 0;
  g.fz0 = d.filter_z_min; g.fz1 = d.filter_z_max; g.fx0 = d.filter_x_min; g.fx1 = d.filter_x_max; g.fy0 = d.filter_y_min; g.fy1 = d.filter_y_max;
  g.bin_scale = (float)((double)LMOT_NUM_BIN / (double)g.r_span);
  g.tol = d.ground_tolerance;
  for (int i = 0; i < 3; ++i) g.tap[i] = tap[i];
  return g;
}

// one track == one UKF object of the reference (ukf.h:15-263) + its trackNumVec_ entry; x/P index 0 = merge,
// 1 = cv, 2 = ctrv, 3 = rm.  Xsig_pred_* is transient (recomputed by every Prediction) and not stored.
struct TrackState {
  double x[4][5];
  double P[4][25];
  double modeProb[3];
  double zPred[3][2];
  double S[3][4];
  double K[3][10];
  double bestYaw, distFromInit, x_merge_yaw;
  double initMeas[2];
  double velo[3];
  float BBox[8][3];
  float bestBBox[8][3];
  int trackNum, lifetime, nVelo, nBBox, nBest;
  uint8_t isStatic, isVisBB;
};

// planar rigid transform, rows (m0 m1 . m2) / (m3 m4 . m5) of a 4x4 whose third row is (0 0 1 0): lmot_params.global_frame
struct Xf2 { int on = 0; float m[6] = {1.f, 0.f, 0.f, 0.f, 1.f, 0.f}; };

// sensor -> vehicle poses of a batched tick (lmot_set_sensors), copied into the launch parameters of the kernels that concatenate
// the tracker's measurement list: frame / list k uses m[k] (row-major 3x4 [R | t])
struct RigPoses { float m[kMaxBatch][12]; };

// frame-level scalars of imm_ukf_jpda.cpp:19-24,56-58 (host side: a handful of doubles per frame)
struct TrackerHost {
  bool init = false;
  double timestamp = 0, egoVelo = 0, egoYaw = 0, egoPreYaw = 0;
  double egoPoint[3] = {0, 0, 0};
  double fold[3] = {0, 0, -1.5707963267948966};
};

// A stream's detection area (lmot_set_detect_area / lmot_seq_set_detect_area) as it is staged: the host copy in StreamCfg, one block per
// masked stream in the pinned source of a submission (Result::h_area, SeqTick::h_area) and on the device (Slot::d_area).  n_rings 0: off.
struct AreaBlock {
  int n_rings, keep_outside, n_vertices, pad;
  int ring_len[LMOT_AREA_MAX_RINGS];
  double xy[2 * LMOT_AREA_MAX_VERTICES];
};

constexpr int kMaxKernelEvents = 20;

// Result block: where one frame's results land.  Pinned, device-mapped host memory written by the kernels themselves
// (box compaction, spawn_output_kernel) -- the stores ARE the D2H transfer; the host waits on ev_done and reads.
// The ring of result blocks is independent of the detection slots, so the host can run many frames ahead of the GPU.
struct Result {
  int* h_hdr = nullptr;                // [16] n_elev, n_ground, num_cluster, n_boxes, n_tracks, n_vis, error
  int* h_det = nullptr;                // [CNT_COUNT] raw detection counters (detect-only submissions)
  int* h_frame_counts = nullptr;       // [kMaxBatch + 1][4] batched ticks: n_elev, n_ground, num_cluster, n_boxes of every frame
  int batch_frames = 0;                // frames of the tick this block holds (0: a single-frame submission)
  float* h_boxes = nullptr;            // [max_boxes][24]
  float* h_targets = nullptr; double* h_vandyaw = nullptr; int* h_manage = nullptr;
  uint8_t* h_static = nullptr; uint8_t* h_vis = nullptr; float* h_visbb = nullptr;
  // device copy of the same block: written by spawn_output_kernel on the tracker stream, moved to the host block by
  // publish_kernel on the publish stream (off the tracker's sequential chain)
  unsigned char* d_block = nullptr;
  int* d_hdr = nullptr; float* d_boxes = nullptr; float* d_targets = nullptr; double* d_vandyaw = nullptr; int* d_manage = nullptr;
  uint8_t* d_static = nullptr; uint8_t* d_vis = nullptr; float* d_visbb = nullptr;
  cudaEvent_t ev_tc = nullptr;         // recorded on the tracker stream after spawn_output_kernel
  cudaEvent_t ev_done = nullptr;
  bool in_flight = false;              // submitted and not yet collected / dropped
  bool has_tracks = false;             // went through the tracker (frame) or not (detect only)
  Xf2 back;                            // global_frame: global -> sensor transform of this frame, applied by publish_kernel
  // track IDs (lmot_track_ids): written by the retire-capable TC (device) and moved to the host block by publish_ids_kernel
  long long* d_ids = nullptr;          // [max_tracks + 2]
  long long* h_ids = nullptr;          // [max_tracks + 2] pinned
  bool ids = false;                    // the step wrote ID rows; false: the IDs are the row indices
  // timing (lmot_enable_timing): stage boundaries and one event after every kernel
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t kev[kMaxKernelEvents] = {};
  int n_kev = 0;
  // deskew: pinned host source of the pose tables copied for this block's submission ([kMaxBatch][LMOT_DESKEW_SLICES * 12], allocated
  // by lmot_set_deskew).  Reusing a block means its previous submission has completed, so the copy from it has too.
  float* h_deskew = nullptr;
  // detection area: pinned host source of the context's area staged for this block's submission (one block, lmot_set_detect_area)
  AreaBlock* h_area = nullptr;
  // sweep accumulation (lmot_set_accumulate / lmot_seq_set_accumulate): h_acc = pinned, device-mapped [kMaxBatch][4] rows (n_points,
  // sweeps_used, n_elevated) of the stream's units written by accumulate_kernel (allocated by the setter); acc_units: the units this
  // block's step accumulated (0: none), with acc_cand candidate sweeps whose stamps and per-unit poses follow, newest first
  // (accumulate_kernel used the first h_acc[4 u + 1] of them for unit u)
  int* h_acc = nullptr;
  int acc_units = 0;
  int acc_cand = 0;
  double acc_ts[LMOT_MAX_SWEEPS - 1] = {};
  float acc_pose[kMaxBatch][LMOT_MAX_SWEEPS - 1][12] = {};
  // merging rig (lmot_set_rig_merge): the tick's sensors, 0 when it did not merge.  h_frame_counts rows 0..merge_rows-1 hold the
  // sensors' (n_elev, n_ground, 0, 0) from rig_merge_kernel, row merge_rows the merged cloud's row from the concatenation; collect
  // moves its num_cluster / n_boxes into row 0 (collect_result)
  int merge_rows = 0;
  // obstacle footprints (obstacles.cu): h_obs = pinned, device-mapped block of obs_cap_units units (ObsUnit layout, obs_cap_vertices
  // vertex pairs each), allocated by the first step that needs it; obs_units: the units this block's step reported (0: obstacles off),
  // ev_obs: recorded behind the obstacle kernel that wrote them
  unsigned char* h_obs = nullptr;
  int obs_cap_units = 0, obs_cap_vertices = 0;
  int obs_units = 0;
  int obs_max_vertices[kMaxBatch] = {};
  cudaEvent_t ev_obs = nullptr;
  bool obs_pending = false;            // an obstacle kernel was recorded into h_obs (the next writer or reallocation waits for ev_obs)
};

// Detection slot: every buffer the three detection stages (ground -> cluster -> box) touch for ONE frame, plus the
// stream they run on.  A context owns `pipeline_depth` slots so the detection stages of frame f+1.. run while the
// tracker (a sequential fold over frames, on its own stream) is still busy with frame f.
struct Slot {
  int index = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_fork = nullptr;       // recorded on the caller's stream: the frame's input is ready
  cudaEvent_t ev_det_done = nullptr;   // recorded on the slot stream after box fitting
  cudaEvent_t ev_trk_done = nullptr;   // recorded on the tracker stream when the tracker has consumed the slot

  // ---- frame input (host-buffer entry points copy here; *_dev entry points use the caller's pointer)
  float4* d_points = nullptr;
  float* d_stage_in = nullptr;         // raw staging for stride != 4 inputs
  float* d_stage_wide = nullptr;       // deskew: raw staging of host frames with stride > 4 (grown to the largest frame seen)
  size_t stage_wide_bytes = 0;
  float* d_deskew = nullptr;           // deskew pose tables: one on a frame slot, kMaxBatch on a bank pseudo-slot (written on its stream)
  const float4* cur_points = nullptr;
  int cur_n = 0;

  // ---- ground removal
  uint16_t* d_cell = nullptr;          // per point polar cell (ch*120+bin) or kNoCell
  unsigned* d_polar_key = nullptr;     // [2][9600] order-preserving uint key of min z; frame k uses grid k&1 and re-arms the other
  float* d_minz = nullptr;             // [9600] debug / parity
  float* d_height = nullptr;           // [9600]
  float* d_smoothed = nullptr;         // [9600]
  float* d_hdiff = nullptr;            // [9600]
  float* d_hg = nullptr;               // [9600] stage entry points: hGround of ground cells as the fused kernel evaluated it, -inf for non-ground cells
  bool hg_valid = false;               // the last launch wrote d_hg
  float* d_lim = nullptr;              // [9600] label limit of every cell (ground.cu label_limit): ground phase 2 -> phase 3
  float* d_hg_dbg = nullptr;           // [9600] the same grid recomputed as a whole by polar_grid_debug_kernel (allocated on first use)
  uint8_t* d_labels = nullptr;         // per point 0/1/2
  float4* d_elev = nullptr;            // compacted elevated cloud
  float4* d_ground = nullptr;          // compacted ground cloud
  unsigned long long* d_gdesc = nullptr;  // [2*CTAs] epoch-tagged per-CTA output counts of the fused ground kernel
  unsigned* d_gbar = nullptr;          // grid-barrier arrival counter of the fused ground kernel (never reset)
  unsigned bar_base = 0;               // host: arrivals of all earlier launches on this slot
  unsigned epoch = 0;                  // host: launches so far on this slot (tag of d_gdesc, parity of d_polar_key)
  int* d_counters = nullptr;           // [CNT_COUNT]
  int* h_counters = nullptr;           // pinned mirror
  int* h_set = nullptr;                // pinned staging for host-written counters

  // ---- clustering
  uint16_t* d_cart = nullptr;          // per elevated point cartesian cell (x*250+y) or kNoCell
  unsigned* d_cart_bits = nullptr;     // [3][2000] bit planes of the 250x250 grid (8 words per row): cells seen once | cells
                                       // seen more than once (re-armed by the CCL kernel) | occupancy of the previous frame
  int* d_label_grid = nullptr;         // [62500] final labels (0 = empty), x-major; updated sparsely from frame to frame
  // side outputs of the cluster node (allocated on first use by lmot_cluster_outputs)
  int* d_first_idx = nullptr;          // [62500] scratch: first point of each labelled cell, INT_MAX at rest
  float4* d_clustered = nullptr;       // makeClusteredCloud
  float4* d_obstacles = nullptr;       // setObsMsg: x, y, z, cluster id
  int* d_cost_map = nullptr;           // [2500] createCostMap, then the two output counts
  bool label_grid_foreign = false;     // the caller uploaded its own grid (lmot_box_fit): next clustering starts from zero

  // ---- box fitting
  uint16_t* d_pcid = nullptr;          // per elevated point cluster id (0 = none)
  int* d_table = nullptr;              // [tiles][max_clusters+1] tile histograms -> exclusive tile offsets
  int* d_seg_start = nullptr;          // [max_clusters+1] first slot of each cluster in d_sorted_idx
  int* d_seg_size = nullptr;           // [max_clusters+1] points per cluster
  float4* d_sorted_pts = nullptr;      // elevated points grouped by cluster, cloud order inside a cluster
  float* d_cl_box = nullptr;           // [max_clusters+1][24] per-cluster box (valid where d_cl_ok)
  float* d_cl_marker = nullptr;        // [max_clusters+1][6]
  uint8_t* d_cl_ok = nullptr;          // [max_clusters+1] rule filter verdict
  float* d_boxes = nullptr;            // [max_boxes][8][3] accepted boxes, cluster-id order
  float* d_boxes_g = nullptr;          // [max_boxes][8][3] the same list in the dead-reckoned global frame (lmot_params.global_frame)
  float* d_markers = nullptr;          // [max_boxes][6]
  int* d_done = nullptr;               // last-CTA-done counter
  int* d_det_sem = nullptr;            // semaphore: +1 by box_fit_kernel's last CTA (frame submissions), -1 by spawn_output_kernel

  // ---- detection area (detect_area.cu; allocated on the first masked submission that uses the slot)
  unsigned* d_area_mask = nullptr;     // [2000] cell mask of the unit this slot box-fits, in the bit-plane layout
  AreaBlock* d_area = nullptr;         // vertex staging: one block on a frame slot, kMaxBatch on a bank pseudo-slot
  bool area_last = false;              // the slot's most recent frame was masked (lmot_cluster_outputs)

  float* d_gz = nullptr;               // [9600] ground heights of the slot's latest frame with ground lines (allocated on first use)

  // ---- layered clustering (layers.cu; allocated on the first layered unit that uses the slot)
  uint8_t* d_slice = nullptr;          // per point of E its height slice, 0xFF: no column (or outside the detection area)
  unsigned* d_colmask = nullptr;       // [62500] slices seen per column (layer_mark_kernel), zero at rest
  unsigned* d_layer_cols = nullptr;    // [62500] occupied slices per column (the runs are the nodes), 0 for an empty column
  int* d_layer_base = nullptr;         // [62500 + 1] id of each occupied column's first run, then the number of runs
  int* d_layer_lab = nullptr;          // [62500 * 16] -(cluster id) of every run
  bool layers_last = false;            // the slot's most recent frame was layered (the label grid does not name its clusters)

  // ---- obstacle footprints (obstacles.cu; allocated on the first obstacle unit that uses the slot)
  unsigned char* d_obs_hull = nullptr; // [max_clusters + 1] hull size, then [max_clusters + 1][140] (u, v) corner bytes; + done counter

  struct Result* res = nullptr;       // result block of the frame currently (or last) processed on this slot
};

enum HostHdr { HDR_N_ELEV = 0, HDR_N_GROUND, HDR_NUM_CLUSTER, HDR_N_BOXES, HDR_N_TRACKS, HDR_N_VIS, HDR_ERROR, HDR_WARN, HDR_N_ACT, HDR_COUNT = 16 };

constexpr int kMaxSlots = 8;
constexpr int kBatchBanks = 2;                       // batched ticks: detection of tick t+1 overlaps the tracker of tick t
constexpr int kMaxResults = 64;

// lmot_default_tracker_params: the reference's constants (citations in include/lmot.h)
inline lmot_tracker_params tracker_params_defaults() {
  lmot_tracker_params p = {};
  p.gamma_g = 9.22; p.p_g = 0.99; p.p_d = 0.9;
  p.distance_thres = 99; p.lifetime_thres = 3;
  p.bb_yaw_change_thres = 0.2;
  p.second_init_v = 2;
  p.static_lifetime = 8; p.static_dist = 3.0;
  for (int m = 0; m < 3; ++m) { p.std_a[m] = (m == 2) ? 3 : 2; p.std_yawdd[m] = (m == 2) ? 3 : 2; }
  p.std_las_x = 0.15; p.std_las_y = 0.15;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) p.trans[i][j] = (i == j) ? 0.9 : 0.05;
  for (int m = 0; m < 3; ++m) p.mode_prob0[m] = 0.33;
  const double d[5] = {0.5, 0.5, 3, 10, 1};
  for (int i = 0; i < 5; ++i) p.p0_diag[i] = d[i];
  return p;
}

// One track table and everything the tracker chain carries from one step to the next.  The context's own tracker is one; every
// sequence of lmot_seq_* (an independent frame stream) is another.
struct Tracker {
  TrackerHost th;
  lmot_tracker_params prm = tracker_params_defaults();   // lmot_set_tracker_params / lmot_seq_set_tracker_params; read at submission
  bool tuned = false;                  // prm differs from the defaults: the chain runs the kernels that read it (tracker.cu)
  TrackState* d_tracks = nullptr;      // [max_tracks] append-only table, dead tracks keep their slot (without retirement)
  int* d_trk_counters = nullptr;       // [CNT_COUNT] CNT_N_TRACKS / CNT_N_VIS / CNT_ERROR of the track table
  int* h_trk_counters = nullptr;       // pinned mirror
  unsigned* d_gate = nullptr;          // [max_tracks][gate_words] chi-square gate bits per (track, box)
  unsigned* d_setter = nullptr;        // [max_tracks][gate_words] boxes this track marks as matched
  int* d_first_setter = nullptr;       // [max_boxes] lowest track index that matched the box (INT_MAX = unmatched)
  uint8_t* d_skip = nullptr;           // [max_tracks] track did not reach measurementValidation this frame
  int* d_new_num = nullptr;            // [max_tracks] mergeOverSegmentation: largest visible container index per live track
  int* d_live_list = nullptr;          // [max_tracks] scratch: indices of live tracks
  int* d_vis_list = nullptr;           // [max_tracks] scratch: indices of tracks with a visible box
  int* d_act_list = nullptr;           // [max_tracks] tracks to visit next frame (built by spawn_output_kernel)
  double4* d_pos = nullptr;            // [max_tracks] packed (x, y, yaw, -) of every track's merged state
  void* d_summary = nullptr;           // [max_tracks] ActSummary (tracker.cu): what TC needs of each active track, written by TB
  int* d_meas_n = nullptr;             // [max_tracks] TA -> TB: number of gated boxes of the track (-1: not provided)
  void* d_meas_ctr = nullptr;          // [max_tracks][32] double2: centre points of the first 32 gated boxes, box order
  unsigned* d_tc_seq = nullptr;        // tracker steps completed (counted by spawn_output_kernel, polled by publish_kernel)
  unsigned tc_launched = 0;            // host: tracker steps launched
  bool act_valid = false;              // false after the table was written from the host: rebuilt before the next step
  Result* last_trk_res = nullptr;      // result block of the previous tracker step (its device copy seeds the next one)
  int last_n_act = 0;                  // active tracks (live or visible) in the last result the host has read: picks spawn_output_kernel's variant
  // track retirement (lmot_set_track_retirement) and track IDs.  Read at submission (tracker.cu ret_prm)
  bool retire = false;                 // every step ends by removing the tracks with trackNum 0 (the retire-capable TC)
  bool ids_identity = true;            // every row's ID is its index: no retirement since the table's last reset / load / open
  long long* d_ids = nullptr;          // [max_tracks + 1] the ID of every row, then the table's spawn counter (retire-capable TC only)
  int ids_n = -1;                      // IDs of the result most recently returned for this table: count (-1: none yet) ...
  bool ids_rows = true;                // ... the row indices, or
  std::vector<long long> ids_last;     // ... these
  // track prediction (lmot_predict_tracks): the table's stamp th.timestamp is meaningful once it stepped or was loaded
  bool pred_ok = false;
  cudaStream_t last_st = nullptr;      // the stream of the table's latest submitted step (nullptr: none since open)
};

// what the tracker chain of a sequence tick reads for sequence k: its measurement list, the list in the dead-reckoned global frame
// (global_frame), its counter block and its detection semaphore.  Without sensor tables these are the buffers of the unit the detection
// front end (api.cu detect_front) box-fitted for it; with any table set, the bank's per-sequence lists (Ctx::seq_meas) that
// concat_boxes_seq_kernel fills.
struct SeqMeas { float* d_boxes = nullptr; float* d_boxes_g = nullptr; int* d_counters = nullptr; int* d_det_sem = nullptr; };

// the box lists of a sequence tick's LISTS entries, in tick order: list i at lists[i] (device), its length in the device int counts[i],
// clamped to [0, cap[i]] (api.cu seq_tick_common packs them; the staged host lists, or the caller's device lists)
struct SeqLists { const float* lists[kMaxBatch]; const int* counts[kMaxBatch]; int cap[kMaxBatch]; };

// one tick of lmot_seq_*: a result block per sequence; blocks[0].ev_done marks the whole tick published.  Only the stepped sequences'
// blocks are written: blocks[k] of a sequence the tick skipped still holds that sequence's step of an earlier tick on this ring slot.
struct SeqTick {
  Result blocks[kMaxBatch];
  uint32_t stepped = 0;                // bit k: sequence k stepped in this tick
  bool in_flight = false;
  float* h_deskew = nullptr;           // deskew: pinned host source of the tick's pose tables, as Result::h_deskew (lmot_seq_set_deskew)
  AreaBlock* h_area = nullptr;         // detection areas: [kMaxBatch] pinned blocks, as Result::h_area (lmot_seq_set_detect_area)
};

// lmot_default_deskew
inline lmot_deskew deskew_defaults() {
  lmot_deskew d;
  memset(&d, 0, sizeof(d));
  d.on = 0; d.time_field = 3; d.time_scale = 1.0; d.time_offset = 0.0; d.t_min = -0.1; d.t_max = 0.0;
  return d;
}

// lmot_default_box_search
inline lmot_box_search box_search_defaults() { lmot_box_search b; b.on = 0; b.n_angles = 90; return b; }

// lmot_default_ground_lines
inline lmot_ground_lines ground_lines_defaults() { lmot_ground_lines g; g.on = 0; g.max_slope = 0.3; g.max_rmse = 0.08; g.max_step = 0.3; return g; }

// lmot_default_obstacles
inline lmot_obstacles obstacles_defaults() { lmot_obstacles o; o.on = 0; o.max_vertices = 65536; return o; }

// lmot_default_layers
inline lmot_layers layers_defaults() { lmot_layers l; memset(&l, 0, sizeof(l)); l.on = 0; l.n_slices = 32; l.slice_m = 0.2; l.z_min = -0.5; l.gap_slices = 2; return l; }

// one frame of a launch with ground lines: its stream's setting (nullptr: off) and the grid of ground heights its lines go to
struct GroundLinesJob { const lmot_ground_lines* cfg; float* gz; };

// lmot_default_accumulate
inline lmot_accumulate accumulate_defaults() { lmot_accumulate a; memset(&a, 0, sizeof(a)); a.sweeps = 1; a.max_age_s = 0.5; return a; }

// One stream's sweep accumulation (accumulate.cu): the setting, and the history of its last sweeps per detection unit.  Unit u's ring
// entry e (of cap, allocated on the stream's first accumulating step for `units` units) holds E_s of the step that recorded it; the host
// keeps that step's stamp, fold and per-unit frame sizes (bounds on |E_s|).  The n valid entries are the ones written last before entry
// w, which the next step writes.  kind / units: the unit layout of the recorded steps (AccKind); a step with another layout starts empty.
enum AccKind { ACC_FRAME = 0, ACC_RIG = 1, ACC_MERGE = 2 };
struct AccHist {
  lmot_accumulate cfg = accumulate_defaults();
  float4* d_ring[kMaxBatch] = {};      // [cap][max_points] per unit
  int* d_ring_n[kMaxBatch] = {};       // [cap] |E_s| per unit (written by accumulate_kernel)
  int cap = 0, cap_units = 0;
  int n = 0, w = 0, kind = -1, units = 0;
  double ts[LMOT_MAX_SWEEPS] = {};
  double fold[LMOT_MAX_SWEEPS][3] = {};
  int n_upper[LMOT_MAX_SWEEPS][kMaxBatch] = {};
  cudaEvent_t ev = nullptr;            // recorded after the stream's latest accumulate launch (the next one waits for it)
  bool ev_live = false;
  bool on() const { return cfg.sweeps > 1; }
  void forget() { n = 0; w = 0; }
};

// One frame stream's detection-side settings: the context's own (lmot_set_sensors / _rig_merge / _deskew; batched ticks) and each
// sequence's (lmot_seq_set_*).  Host state read at submission: ticks already submitted carry their own copy in their launch parameters.
struct StreamCfg {
  int n_sensors = 0;                   // sensor table: sensor k = frame k of a tick; 0: every frame uses lmot_params' values
  lmot_sensor sensors[kMaxBatch] = {};
  // merging rig: with a table set, the sensors' elevated clouds are clustered and boxed as one vehicle-frame cloud in the bank's merge
  // unit (rig_merge.cu, allocated on the first merging submission)
  bool rig_merge = false;
  Slot merge_unit[kBatchBanks];
  // own detection values (lmot_seq_set_detect_params; the context's own stream has none): off = lmot_params' values.  A tick with any
  // of them on runs every frame through the per-frame kernel variants (ground.cu, boxfit.cu)
  bool det_on = false;
  lmot_detect_params det = {};
  lmot_deskew deskew = deskew_defaults();   // sweep deskew (deskew.cu)
  AreaBlock area = {};                      // detection area (detect_area.cu)
  AccHist acc;                              // sweep accumulation and its history (accumulate.cu)
  lmot_box_search search = box_search_defaults();   // box search (box_search.cu)
  lmot_ground_lines lines = ground_lines_defaults(); // ground lines (ground_lines.cuh)
  lmot_layers layers = layers_defaults();            // layered clustering (layers.cu)
  lmot_obstacles obs = obstacles_defaults();         // obstacle footprints (obstacles.cu)
  bool merges() const { return rig_merge && n_sensors > 0; }
  bool masked() const { return area.n_rings > 0; }
  int search_angles() const { return search.on ? search.n_angles : 0; }   // A of the stream's units, 0: boxFitting's fit
  const lmot_ground_lines* lines_on() const { return lines.on ? &lines : nullptr; }
  // a submission of the stream runs more than the plain detection path (timing mode times only that path).  stamped: it has a stamp
  // (deskew and accumulation apply); sensors: its frames are the stream's sensors (merging applies)
  bool beyond_plain(bool stamped, bool sensors) const {
    return masked() || search.on || lines.on || layers.on || obs.on || deskews(stamped) || (stamped && acc.on()) || (sensors && merges());
  }
  bool deskews(bool stamped) const { return stamped && deskew.on; }
  // records of `stride` floats hold the time field where the submission deskews them (device frames: stride 4)
  bool deskew_fits(bool stamped, int stride) const { return !deskews(stamped) || stride > deskew.time_field; }
};

// the obstacle footprints of one returned step, copied out of its result block (the block is reused by later submissions)
struct ObsLast {
  bool valid = false;                  // false: no step returned yet, or it ran with obstacles off
  int units = 0;
  int n_obs[kMaxBatch] = {}, n_vert[kMaxBatch] = {}, max_vertices[kMaxBatch] = {};
  std::vector<lmot_obstacle> rows[kMaxBatch];
  std::vector<float> xy[kMaxBatch];
};

// lmot_default_ego_match
inline lmot_ego_match ego_match_defaults() {
  lmot_ego_match m;
  memset(&m, 0, sizeof(m));
  m.grid = 768; m.cell_m = 0.1; m.z_min = -1.5; m.z_max = 0.5; m.r_min = 3.0; m.r_max = 38.0; m.sub_m = 0.4; m.max_points = 4096;
  m.yaw_step = 0.005; m.yaw_half = 30; m.shift_half = 30; m.refine = 5; m.min_points = 200; m.min_score_frac = 0.3; m.sensor = -1;
  return m;
}

// One stream's scan matcher (ego_match.cu): its setting, its state between calls and its device buffers (allocated on its first call,
// grown when a later setting needs more).  Fields d_field[ref] is the reference, d_field[ref ^ 1] the next call's field.
struct EgoMatch {
  lmot_ego_match cfg = ego_match_defaults();
  bool has_ref = false;
  double ts = 0, dt = 0;               // stamp of the reference; dt of the stored delta
  double delta[3] = {0, 0, 0};         // dx, dy, dth
  bool delta_ok = false;
  double yaw = 0;                      // Y
  int n_ref = 0;                       // occupied cells of the reference
  int ref = 0;
  unsigned char* d_field[2] = {nullptr, nullptr};
  unsigned* d_occ = nullptr;
  int* d_sub = nullptr;
  float2* d_samp = nullptr;
  size_t cap_field = 0, cap_sub = 0, cap_samp = 0;   // bytes of a field / entries of d_sub / entries of d_samp
  void reset() { has_ref = false; ts = 0; dt = 0; delta[0] = delta[1] = delta[2] = 0; delta_ok = false; yaw = 0; n_ref = 0; }
};

// One frame stream: the context's own (lmot_frame*, lmot_batch*, lmot_track_step*, lmot_tracker_*) or a sequence of lmot_seq_*.  Its
// settings, its track table, and what collect_result copied out of its most recently returned step.  Released by api.cu stream_free.
struct Stream {
  EgoMatch ego;                        // scan-matched ego motion (ego_match.cu): never read by the frame pipeline
  StreamCfg cfg;
  Tracker trk;
  lmot_accum_info acc_info = {};       // lmot_accumulate_info / lmot_seq_accumulate_info: what the step used
  ObsLast obs_last;                    // lmot_obstacles_result / lmot_seq_obstacles_result: its footprints
  int fc_n = 0;                        // lmot_seq_frame_counts: the frames of the sequence's step ...
  int fc[kMaxBatch][4] = {};           // ... and their n_elev, n_ground, num_cluster, n_boxes (host copies: the ring slot is reused)
};

struct Ctx {
  lmot_params prm;
  int device = 0;
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;       // the caller's stream: stage-by-stage entry points, fork/join of the pipeline
  std::string last_error;
  GroundParams gp;

  // ---- capacities
  int max_points = 0, max_sort_tiles = 0, fit_ctas = 0, n_mt_raw = 0;   // fit_ctas / trk_ctas: from the SM count (lmot_create)
  bool coop_launch = false;            // LMOT_COOP=1: cudaLaunchCooperativeKernel for the ground kernel (A/B diagnostics)
  int fused_max_ctas = 0;              // co-residency limit of the cooperative ground kernel on this device
  bool fuse_ccl = true;                // frame / batch path: clustering runs in the ground kernel's tail (LMOT_FUSE_CCL=0: separate launch, A/B)
  bool zero_copy = false;              // lmot_frame_submit: pinned host frames are read by the ground kernel directly (LMOT_ZERO_COPY=1; off: slower than the copy engine)
  bool ground_half_sms = true;         // frame pipeline: ground kernel on half of the SMs (ground.cu ground_launch; LMOT_GROUND_HALF=0 disables, A/B only)
  unsigned spin_limit = 1u << 24;      // polls after which a device-side wait traps instead of hanging the GPU (LMOT_SPIN_LIMIT, 0 = wait for ever)
  int pts_per_cta = 768;               // target chunk of the fused ground kernel (LMOT_PTS_PER_CTA overrides, tuning only)
  unsigned long long* d_mt_raw = nullptr;  // raw mt19937_64(0) outputs (shared, read only)
  float2* d_bs_tab = nullptr;          // box search: the angle tables of A = 1 .. LMOT_BOX_SEARCH_MAX_ANGLES, table A at A(A-1)/2 (read only)

  // ---- detection slots
  int n_slots = 1;
  Slot slots[kMaxSlots];
  int next_slot = 0;                   // slot of the next submission
  int last_slot = 0;                   // slot of the most recent submission (debug getters read it)
  // ---- batched ticks (lmot_batch_*): own detection slots, kBatchBanks x batch_frames, allocated on first use
  Slot bslots[kBatchBanks * kMaxBatch];
  int n_bslots = 0, batch_frames = 0, next_bank = 0;
  Slot bank[kBatchBanks];              // pseudo-slots: concatenated boxes + counters + semaphore + events of a bank, and the stream its
                                       // tracking-only sequence ticks (lmot_seq_track*) run on

  // ---- result ring
  int n_results = 1;
  Result results[kMaxResults];
  int res_next = 0, res_oldest = 0, n_in_flight = 0;
  Result* last_res = nullptr;

  // ---- the context's own stream: sensor k = frame k of a batched tick / list k of lmot_track_step_lists_dev; its settings apply to
  // lmot_frame* and batched ticks.  The sequences' records never apply to it, nor it to sequence ticks
  Stream own;

  // ---- tracker
  cudaStream_t trk_stream = nullptr;
  cudaStream_t pub_stream = nullptr;   // device -> host publication of finished frames
  int trk_ctas = 0, gate_words = 0;
  bool tc_wide = false;
  int tc_force = -1;           // LMOT_TC_WIDE: -1 by count, 0 / 1 pinned
  // ---- independent sequences (lmot_seq_*): one Stream each (its frames of a tick are its sensors in table order; no table: one frame),
  // a ring of ticks of n_seq result blocks; detection on the batch banks
  int n_seq = 0;
  Stream seq[kMaxBatch];
  SeqTick* seq_ticks = nullptr;        // [seq_ring]
  int seq_ring = 0, seq_next = 0, seq_oldest = 0, seq_in_flight = 0;
  SeqTick* seq_last = nullptr;         // most recent submission (lmot_seq_fetch)
  uint32_t seq_stepped = 0;            // lmot_seq_stepped: the stepped mask of the tick most recently returned
  bool seq_wide = false;               // spawn_output_kernel's variant of the sequence ticks (largest last_n_act of the stepped tables)
  SeqMeas seq_meas[kBatchBanks][kMaxBatch];    // per-sequence measurement lists of each batch bank, allocated by lmot_seq_open
  // staging of lmot_seq_track_submit's host lists, per bank: kMaxBatch lists of max_boxes boxes, then kMaxBatch counts (lmot_seq_open)
  float* seq_stage[kBatchBanks] = {};

  // ---- track prediction (lmot_predict_tracks*, tracker.cu predict_launch)
  bool pred_pending = false;           // a prediction was queued since the last tracker step: the next step's first kernel waits for it
  cudaStream_t pred_stream = nullptr;  // ... on this stream
  cudaEvent_t ev_pred = nullptr;       // recorded after every prediction (created on first use)
  cudaEvent_t ev_pred_in = nullptr;    // _dev forms on another stream: the caller stream's work so far (created on first use)
  unsigned char* d_pred_stage = nullptr;   // host forms: device staging of the outputs, grown to the largest request
  size_t pred_stage_bytes = 0;
  int* h_pred_n = nullptr;             // pinned: the staged row count

  // ---- lmot_debug_area_masks: the unit masks of the most recent own-stream submission (none: it was not masked)
  const unsigned* area_dbg[kMaxBatch] = {};
  int n_area_dbg = 0;
  // ---- lmot_debug_ground_lines: the ground grids of the most recent own-stream submission (none: its lines were off)
  const float* gz_dbg[kMaxBatch] = {};
  int n_gz_dbg = 0;
  // ---- lmot_debug_point_clusters: the units of the most recent own-stream submission (none: it was not layered)
  const Slot* lay_dbg[kMaxBatch] = {};
  int n_lay_dbg = 0;

  // ---- scan-matched ego motion (ego_match.cu): the matcher stream and what every call stages, created / grown on first use
  cudaStream_t ego_stream = nullptr;
  cudaEvent_t ev_ego_in = nullptr;     // _dev forms: the caller stream's work so far
  float* d_ego_stage = nullptr;        // host frames
  size_t ego_stage_bytes = 0;
  float2* h_ego_tab = nullptr;         // pinned angle tables of a call, and their device copy
  float2* d_ego_tab = nullptr;
  size_t ego_tab_cap = 0;              // entries
  void* h_ego_res = nullptr;           // pinned per-stream results of a call, and their device rows
  void* d_ego_res = nullptr;

  // ---- timing
  bool timing = false;
  float stage_ms[4] = {0, 0, 0, 0};
  float kernel_ms[kMaxKernelEvents] = {};
  int n_kernel_ms = 0;
  double host_ns[4] = {0, 0, 0, 0};    // accumulated host time: submit, collect: event wait, collect: copies, calls
};

// error helper: records the CUDA error text in the context and returns LMOT_ERR_CUDA
#define LMOT_CUDA(ctx, call)                                                                     \
  do {                                                                                           \
    cudaError_t e__ = (call);                                                                    \
    if (e__ != cudaSuccess) {                                                                    \
      (ctx)->last_error = std::string(#call) + ": " + cudaGetErrorString(e__);                   \
      return LMOT_ERR_CUDA;                                                                      \
    }                                                                                            \
  } while (0)

// timing mode only: mark the end of the kernel just launched on `st`
inline void kernel_mark(Ctx* c, Slot* s, cudaStream_t st) {
  if (c->timing && s->res && s->res->n_kev < kMaxKernelEvents) cudaEventRecord(s->res->kev[s->res->n_kev++], st);
}

#ifdef __CUDACC__
// mapCartesianGrid (component_clustering.cpp:38-47) + the "more than one point" test (:136) without a counter: bit planes
// `once` / `twice` of the 250x250 grid, 8 words per row.  c = x*250+y or 0xFFFF; ALL 32 lanes of the warp must call.
__device__ __forceinline__ void cart_mark(unsigned c, unsigned* __restrict__ once, unsigned* __restrict__ twice) {
  const unsigned grp = __match_any_sync(0xFFFFFFFFu, c);
  if (c != 0xFFFFu && (int)(threadIdx.x & 31) == __ffs(grp) - 1) {
    const unsigned x = c / (unsigned)kNumGrid, y = c - x * (unsigned)kNumGrid;
    const unsigned w = x * 8u + (y >> 5), bit = 1u << (y & 31u);
    if (__popc(grp) > 1) atomicOr(&twice[w], bit);
    else if (atomicOr(&once[w], bit) & bit) atomicOr(&twice[w], bit);
  }
}

// p' = [R | t] p (lmot_set_sensors): ((r0 x + r1 y) + r2 z) + t per row in float, no contraction -- pcl::transformPointCloud's
// evaluation with an Affine3f.  m = row-major 3x4.  (Boxes of a rig: boxfit.cu; points of a merging rig: rig_merge.cu)
__device__ __forceinline__ void rig_apply(const float* m, float& x, float& y, float& z) {
  const float ox = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], x), __fmul_rn(m[1], y)), __fmul_rn(m[2], z)), m[3]);
  const float oy = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[4], x), __fmul_rn(m[5], y)), __fmul_rn(m[6], z)), m[7]);
  const float oz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[8], x), __fmul_rn(m[9], y)), __fmul_rn(m[10], z)), m[11]);
  x = ox; y = oy; z = oz;
}
#endif

// ---- stage launchers (asynchronous on the given stream) -------------------------------------------------
int ground_alloc(Ctx* c, Slot* s);
void ground_free(Slot* s);
// pts: device float4 array of n points; fuse_count: also bin the elevated points into the slot's cartesian count grid
// want_labels: also write the per-point u8 label array (stage entry point); the frame pipeline skips it
// `chain`: stand-alone entry points -- nothing of the library follows on `st` before the next ground launch; consecutive launches on
// one stream then run as programmatic dependents without an event between them (ground.cu, GroundChain)
int ground_launch(Ctx* c, Slot* s, cudaStream_t st, const float4* pts, int n, bool fuse_count = false, bool want_labels = true, bool fuse_ccl = false, bool chain = false);
// rig (nullable): sensor i's h_sensor / t_hmin / t_hmax for frame i (lmot_set_sensors); nullptr: lmot_params' values for every frame
// det (nullable): frame i's own detection values (sensor values already folded in; lmot_seq_set_detect_params) -> the per-frame kernel
// variant; rig is then unused
// lines (nullable): frame i's ground lines (cfg nullptr: off) and the grid its lines go to -> ground_fused_lines_kernel, every frame with
// its own values (det, else lmot_params' with rig's folded in)
int ground_launch_batch(Ctx* c, Slot* const* slots, int F, const float4* const* pts, const int* n, cudaStream_t st, bool fuse_count, bool want_labels, bool fuse_ccl = false, bool chain = false, const lmot_sensor* rig = nullptr,
                        const lmot_detect_params* det = nullptr, const GroundLinesJob* lines = nullptr);
void ground_chain_forget(int device, bool device_idle);
int ground_cells_debug(Ctx* c, Slot* s, cudaStream_t st);
int ground_grids_debug(Ctx* c, Slot* s, cudaStream_t st);   // d_minz / d_height / d_smoothed / d_hdiff / d_hg_dbg from the last launch's keys
bool ground_reads_input_once(const Ctx* c, int n);
int ground_repack(Ctx* c, cudaStream_t st, const float* d_in, int n, int stride, float4* d_out);
int cluster_alloc(Ctx* c, Slot* s);
void cluster_free(Slot* s);
// area (nullable): unit i's cell mask (detect_area.cu), nullptr for an unmasked unit; any mask -> the masking kernel variants
int cluster_launch(Ctx* c, Slot* s, cudaStream_t st, int n_upper, bool counted = false, const unsigned* area = nullptr);
int ccl_launch_batch(Ctx* c, Slot* const* slots, int F, cudaStream_t st, const unsigned* const* area = nullptr);
int cluster_cells_only(Ctx* c, Slot* s, cudaStream_t st, int n_upper);
int cluster_outputs_launch(Ctx* c, Slot* s, cudaStream_t st);      // makeClusteredCloud / setObsMsg / createCostMap  // d_cart for a cloud whose label grid comes from the caller
int boxfit_alloc(Ctx* c, Slot* s);
int boxfit_alloc_shared(Ctx* c);
void boxfit_free(Slot* s);
// search: the frame's box search angle count A (0: boxFitting's fit)
// lines: the frame's ground grid (ground lines; nullptr: off)
// layers: the frame's layered run tables (nullptr: its label grid)
struct LayerTab;
int boxfit_launch(Ctx* c, Slot* s, cudaStream_t st, int n_upper, bool post_sem = false, const unsigned* area = nullptr, int search = 0,
                  const float* lines = nullptr, const LayerTab* layers = nullptr);
// rig (nullable): sensor i's sensor_height for frame i (box fitting) / sensor i's pose for list i (concatenation)
// det (nullable): frame i's own detection values, as ground_launch_batch's; rig is then unused
// area (nullable): as ccl_launch_batch's
// search (nullable): frame i's box search angle count A, 0: boxFitting's fit (box_search.cu fits the others)
// lines (nullable): unit i's ground grid, nullptr for a unit measured from the flat sensor_height; any -> every unit through the ground
// lines variants (box_fit_lines_kernel, box_search_lines_kernel)
// layers (nullable): unit i's run tables (slice nullptr: a unit clustered on the label grid); any -> tile_hist_layers_kernel
int boxfit_launch_batch(Ctx* c, Slot* const* slots, int F, cudaStream_t st, const int* n_upper, bool post_sem, const lmot_sensor* rig = nullptr,
                        const lmot_detect_params* det = nullptr, const unsigned* const* area = nullptr, const int* search = nullptr,
                        const float* const* lines = nullptr, const LayerTab* layers = nullptr);
// box search (box_search.cu): setting validation, the angle table of A (lmot_box_search_angles), and the device tables of every A
// (Ctx::d_bs_tab, uploaded once by the first setter that turns the search on)
bool box_search_valid(const lmot_box_search& b);
void box_search_table(int A, float (*out)[2]);
int box_search_ensure(Ctx* c);
// box search over n units (their Slots' box-fitting buffers): unit i with detection values det[i] (its sensor's height folded in) and A[i]
// angles, gx CTAs per unit, as a programmatic dependent of the kernel before it iff pdl
// lines (nullable): unit i's ground grid as boxfit_launch_batch's -> box_search_lines_kernel
int box_search_launch(Ctx* c, Slot* const* units, int n, const lmot_detect_params* det, const int* A, cudaStream_t st, bool post_sem, int gx,
                      bool pdl, const float* const* lines = nullptr);
int boxes_pack_lists_launch(Ctx* c, cudaStream_t st, const float* d_lists, const int* d_counts, int n_lists, int cap, float* d_boxes, int* d_counters,
                            const lmot_sensor* rig = nullptr);
int boxes_concat_launch(Ctx* c, Slot* const* slots, int F, cudaStream_t st, float* d_boxes, int* d_counters, int* d_frame_counts, int* det_sem,
                        const lmot_sensor* rig = nullptr);
void origin_points_fold(TrackerHost& h, double timestamp, double v_gps, double yaw_gps);
int tracker_alloc(Ctx* c, Tracker& t);
void tracker_free(Tracker& t);
// boxes: device float[M][8][3] with M in det_counters[CNT_N_BOXES]; results into the slot's pinned host block
int tracker_launch(Ctx* c, Slot* s, cudaStream_t st, const float* d_boxes, const int* det_counters, double timestamp, double v_gps,
                   double yaw_gps, bool gate = false, bool* gated = nullptr);   // gate: wait for the slot's detection semaphore on the device (tracker.cu)
int boxes_to_global_launch(Ctx* c, Slot* sl, cudaStream_t st, const float* d_boxes, const int* det_counters, double timestamp, double v_gps,
                           double yaw_gps, bool post_sem);
int tracker_publish(Ctx* c, Result* r, cudaStream_t st);            // device block of r -> pinned host block
// sequence ticks with sensor tables: sequence k's frames [f0[k], f0[k + 1]) of `slots` -> m[k] (boxfit.cu)
int boxes_concat_seq_launch(Ctx* c, Slot* const* slots, int S, const int* f0, const bool* rig_on, const lmot_sensor* rig, const SeqMeas* m,
                            int* const* frame_counts, bool post_sem, cudaStream_t st);
// LISTS entries of sequence ticks: position k's lists [f0[k], f0[k + 1]) of L -> m[k] (boxfit.cu)
int boxes_pack_lists_seq_launch(Ctx* c, cudaStream_t st, const SeqLists& L, int S, const int* f0, const bool* rig_on, const lmot_sensor* rig,
                                const SeqMeas* m, int* const* frame_counts, bool post_sem);
// sequence ticks over the S stepped sequences: chain position k is sequence seq[k]; measurement list m[k] and ego values ts / v / yaw[k]
// are indexed by position -> track table c->seq[seq[k]].trk -> tick->blocks[seq[k]] (tracker.cu)
int seq_global_launch(Ctx* c, const int* seq, const SeqMeas* m, int S, cudaStream_t st, const double* ts, const double* v, const double* yaw);
int seq_tracker_launch(Ctx* c, const int* seq, const SeqMeas* m, SeqTick* tick, int S, const double* ts, const double* v, const double* yaw);
// track prediction of S tables (1..kMaxBatch) at n_t times each (t_us[k * n_t + j]) into outs[k] (device arrays), row counts into
// d_n_rows[k] (nullable), on stream st behind the tables' latest steps; records c->ev_pred after the kernel (tracker.cu)
int predict_launch(Ctx* c, Tracker* const* tabs, int S, const double* t_us, int n_t, const lmot_pred_out* outs, int* const* d_n_rows,
                   cudaStream_t st);
int boxes_publish(Ctx* c, Slot* s, Result* r, cudaStream_t st);     // detection-only: slot box list -> pinned host block
// sweep deskew (deskew.cu): one frame's pose table (out: [LMOT_DESKEW_SLICES][12]; mount nullptr: identity), and one launch over the
// deskewed frames of a submission
struct DeskewJob { const float* in; float4* out; const float* table; int n, stride; lmot_deskew d; };
int deskew_table(const lmot_deskew& d, double v, double omega, const lmot_sensor* mount, float* out);
int deskew_launch(Ctx* c, cudaStream_t st, const DeskewJob* jobs, int n_jobs);
// merging rigs (rig_merge.cu).  A merge unit is a Slot with only the buffers clustering and box fitting of the merged cloud touch:
// d_elev (the merged cloud), d_counters, d_cart, bit planes, label grid and the box-fitting set.
int merge_unit_create(Ctx* c, Slot* u, int index);
bool merge_unit_ready(const Slot* u);  // every buffer of the unit allocated (merge_unit_create succeeded)
void merge_unit_destroy(Slot* u);      // frees whatever is allocated (also a partly created unit) and resets the slot
// one launch over every merging unit of a submission: unit u gathers the elevated clouds of sensor slots src[s0[u] .. s0[u + 1]) moved by
// their poses (pose[i] = sensor i's, in src order), writes its rows of the per-sensor counts to frame_counts[u] (device view of its
// result block) and marks its own bit planes; the sensor slots' bit planes are returned to rest.  n_upper[i]: source i's frame size
// (grid bound).  roi[u]: unit u's clustering ROI
int rig_merge_launch(Ctx* c, cudaStream_t st, Slot* const* src, const lmot_sensor* pose, const int* n_upper, int n_units, const int* s0,
                     Slot* const* units, int* const* frame_counts, const float* roi);
// detection areas (detect_area.cu).  area_valid: lmot_area's rules; area_copy: a valid area into its staging block (NULL: off)
bool area_valid(const lmot_area* a);
void area_copy(AreaBlock& dst, const lmot_area* a);
// lmot_detect_area_mask of a staged area: pose = row-major 3x4 (nullptr: identity), out = uint32[2000]
void area_mask_host(const AreaBlock& a, const float* pose, float roi, unsigned* out);
// the unit buffers a masked submission needs on slot s (its mask, and `blocks` vertex staging blocks when blocks > 0), allocated once
int area_ensure(Ctx* c, Slot* s, int blocks);
// one launch over the masked units of a submission: unit i's mask from its stream's staged block a, its pose and roi
struct AreaJob { const AreaBlock* a; unsigned* mask; float pose[12]; float roi; };
int area_launch(Ctx* c, cudaStream_t st, const AreaJob* jobs, int n_jobs);
// sweep accumulation (accumulate.cu).  accumulate_pose: lmot_accumulate_pose (mount: row-major 3x4, nullptr: identity)
void accumulate_pose(const double fold_s[3], const double fold_t[3], const float* mount, float out[12]);
bool accumulate_valid(const lmot_accumulate& a);
void accumulate_free(AccHist& h);
// one accumulating unit of a launch: its cloud (E_t in front), cells, bit planes and counters, its ring, its row of the result block
// (device view), its clustering ROI, and the step's candidates (ring entries and this unit's poses)
struct AccJob {
  float4* elev; uint16_t* cart; unsigned* bits; int* counters;
  float4* ring; int* ring_n; int* info;
  float roi; int w, n_sw;
  int bound;                           // host: bounds |E_t| and every candidate's length (the launch's point blocks)
  int entry[LMOT_MAX_SWEEPS - 1];
  float m[LMOT_MAX_SWEEPS - 1][12];
};
// the host side of one stream's accumulating step: `units` units of layout `kind` (U[i], pose[i], roi[i], frame-size bound n_upper[i])
// with the stream's fold th peeked at (ts, v, yaw).  Allocates the ring on first use, starts the history afresh on a new layout, picks
// the candidates into r (units r's rows from 0) and the jobs, raises fit_upper[i] to bound |E_acc| of unit i, records the step.
int accumulate_step(Ctx* c, AccHist& h, int kind, int units, Slot* const* U, const lmot_sensor* pose, const float* roi, const int* n_upper,
                    const TrackerHost& th, double ts, double v, double yaw, Result* r, AccJob* jobs, int* fit_upper);
// one launch over the jobs of a submission, behind each accumulating stream's previous launch (hists[0 .. nh)); records their events
int accumulate_launch(Ctx* c, cudaStream_t st, Slot* mark, const AccJob* jobs, int n_jobs, AccHist* const* hists, int nh);
// layered clustering (layers.cu).  What box fitting reads of a layered unit: each point's slice, and per column the occupied slices, the
// id of its first run and the cluster of every run (as -(id))
struct LayerTab { const uint8_t* slice; const unsigned* cols; const int* base; const int* lab; };
bool layers_valid(const lmot_layers& l);
int layers_ensure(Ctx* c, Slot* s, cudaStream_t st);   // the slot's layer buffers, allocated once (column masks zeroed on st)
LayerTab layer_tab_of(const Slot* s);
// one layered unit of a submission: its slot (cloud, cells, bit planes, counters, layer buffers), detection-area mask (nullable), setting,
// box-fitting sensor_height and a bound on |E|
struct LayerUnit { Slot* s; const unsigned* area; lmot_layers cfg; float sensor_height; int n_upper; };
// layer_mark_kernel over every unit, then ccl_layer_kernel with one CTA per unit
int layers_launch(Ctx* c, cudaStream_t st, const LayerUnit* u, int n, Slot* mark);
// step 6 on the host from the unit's device tables (synchronous): ids[i] for the n points of its cloud
int layers_point_ids(Ctx* c, const Slot* s, int n, int32_t* ids);
// obstacle footprints (obstacles.cu).  One unit of a submission: its slot (box-fitting buffers), clustering ROI, vertex pool, and where its
// footprints go: the result block r's unit `slot`
struct ObsUnit { Slot* s; float roi; int max_vertices; Result* r; int slot; };
bool obstacles_valid(const lmot_obstacles& o);
// the units' hull scratch and their blocks' pinned obstacle blocks (allocated or grown once; st: the stream the launch will run on)
int obstacles_ensure(Ctx* c, const ObsUnit* u, int n, cudaStream_t st);
// one launch over the n units behind box fitting on st; records each block's ev_obs
int obstacles_launch(Ctx* c, cudaStream_t st, const ObsUnit* u, int n, Slot* mark);
// the block's footprints into `dst` (waits for ev_obs); r->obs_units == 0: dst becomes invalid
int obstacles_collect(Ctx* c, Result* r, ObsLast& dst);
// scan-matched ego motion (ego_match.cu): setting validation, and one synchronous call over S streams q[i] with frame pts[i] of n[i]
// points of `stride` floats (host frames when host, else device frames ordered after the caller stream), stamp ts[i], poses[i] (nullable:
// the frame as given) -> out[i]
bool ego_match_valid(const lmot_ego_match& m);
int ego_estimate_run(Ctx* c, EgoMatch* const* q, const float* const* pts, const int* n, int stride, const double* ts,
                     const lmot_sensor* const* poses, int S, bool host, lmot_ego_out* const* out);
void ego_free(EgoMatch& e);
void ego_ctx_free(Ctx* c);
void obstacles_result_free(Result* r);

}  // namespace lmot
