/* lmot.h -- C ABI of the H100-native LiDAR multi-object-tracking hot path (liblmot.so).
 *
 * Drop-in boundary (SURVEY.md §8b).  The reference has no FFI; its boundary is four C++ free functions
 * called from the three ROS node callbacks.  Each entry point below replaces one of them:
 *
 *   lmot_ground_remove      <- groundRemove         object_tracking/include/ground_removal.h:62-64
 *                                                   (def. src/groundremove/ground_removal.cpp:177)
 *   lmot_component_cluster  <- componentClustering  object_tracking/include/component_clustering.h:20-22
 *                                                   (def. src/cluster/component_clustering.cpp:260)
 *   lmot_box_fit            <- boxFitting           object_tracking/include/box_fitting.h:34-36
 *                                                   (def. src/cluster/box_fitting.cpp:422)
 *   lmot_track_step         <- getOriginPoints + immUkfJpdaf
 *                                                   object_tracking/include/imm_ukf_jpda.h:15,19-22
 *                                                   (def. tracking/imm_ukf_jpda.cpp:74,704)
 *   lmot_frame              <- the four calls back to back, as object_tracking0/src/main.cpp:51-121 does in
 *                              one callback (device-resident between stages, one H2D and one D2H per frame)
 *
 * Conventions: plain pointers and sizes, caller-owned buffers, no C++/torch types.  Every function returns
 * LMOT_OK (0), a negative status (error), or a positive one (warning: the outputs are valid).  A context owns one CUDA device, one stream and all scratch memory;
 * it is NOT thread-safe (the reference's functions are non-re-entrant too); use one context per sensor stream.
 * There is no CPU fallback: without a usable CUDA device lmot_create fails with LMOT_ERR_CUDA.
 *
 * Point clouds are arrays of float with a caller-given stride in floats (3 = packed XYZ, 4 = XYZI or the
 * 16-byte pcl::PointXYZ layout the reference's PCL containers use).  Clouds RETURNED by the library are
 * always stride 4 (x, y, z, 1.0f) == pcl::PointXYZ, so a ROS shell can memcpy them into a PCL cloud.
 */
#ifndef LMOT_H
#define LMOT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LMOT_NUM_CHANNEL 80   /* ground_removal.h:16 */
#define LMOT_NUM_BIN 120      /* ground_removal.h:17 */
#define LMOT_NUM_GRID 250     /* component_clustering.h:13 */
#define LMOT_TRACK_DUMP_DOUBLES 236

typedef enum lmot_status {
  LMOT_OK = 0,
  LMOT_ERR_INVALID = -1,   /* bad argument */
  LMOT_ERR_CUDA = -2,      /* CUDA runtime/driver error, or no device (there is no CPU fallback) */
  LMOT_ERR_CAPACITY = -3,  /* input exceeds a capacity fixed at lmot_create (points, clusters, boxes, tracks) */
  LMOT_ERR_STATE = -4,     /* call sequence error (e.g. fetch before run) */
  /* positive = warning: the call did its work and every output is valid */
  LMOT_WARN_TRACK_TABLE_FULL = 1   /* the step's rows -- the rows the table held at its start plus this step's spawns -- would exceed
                                      max_tracks: boxes no track matched beyond that spawn no new track this frame; existing tracks are
                                      updated and reported as usual.  Without track retirement dead tracks keep their row (like the
                                      reference's targets_), so the table fills: at the default 8192 and ~3 spawns per frame that is
                                      ~4.5 min of a 10 Hz stream.  Turn retirement on (lmot_set_track_retirement: the table then holds
                                      the live tracks only), size max_tracks for the session (1.6 KB of device memory per track) or call
                                      lmot_tracker_reset between sequences. */
} lmot_status;

/* ruleBasedFilter (box_fitting.cpp:97-158) falls off its end without a return when a nested size check fails:
 * undefined behaviour.  INTENDED = fall-through means `false`; GCC13_O2_COMPAT = what g++ 13 -O2 makes of the
 * unmodified file (only the n>=30 test and the height window survive).  See SURVEY.md §8c. */
typedef enum lmot_rule_filter { LMOT_RULE_INTENDED = 0, LMOT_RULE_GCC13_O2_COMPAT = 1 } lmot_rule_filter;

/* Defaults (lmot_default_params) reproduce the reference's constants; citations are file:line under
 * /root/reference/object_tracking. */
typedef struct lmot_params {
  /* ground removal -- src/groundremove/ground_removal.cpp:24-33,239 */
  float r_min, r_max;        /* 3.4, 120 */
  float t_hmin, t_hmax;      /* -2.0, -0.4 */
  float t_hdiff;             /* 0.4 */
  float h_sensor;            /* 2.0 ("hSeonsor") */
  double ground_tolerance;   /* 0.25 */
  /* clustering -- src/cluster/component_clustering.cpp:11 */
  float roi_m;               /* 50 */
  /* box fitting -- src/cluster/box_fitting.cpp:18-44,100,308 */
  int ram_points;            /* 80 */
  int l_slope_dist;          /* 1 */
  int l_num_points;          /* 5 */
  float sensor_height;       /* 2 */
  float t_height_min, t_height_max;  /* 0.8, 2.6 */
  float t_width_min, t_width_max;    /* 0.2, 3.5 */
  float t_len_min, t_len_max;        /* 0.2, 14 */
  float t_area_max;          /* 20 */
  float t_ratio_min, t_ratio_max;    /* 1, 8 */
  float min_len_ratio;       /* 3 */
  float t_pt_per_m3;         /* 8 */
  int min_cluster_points;    /* 30 (box_fitting.cpp:100) */
  int rule_filter;           /* lmot_rule_filter, default LMOT_RULE_INTENDED */
  /* tracker -- tracking/imm_ukf_jpda.cpp:26-51,70 ; first-frame quirk :741-760 */
  int oracle_compat_first_frame; /* 1: first frame spawns ONE track from box #1 at the hard-coded (-1.5125,-8.975) */
  /* capacities (the reference's std::vectors grow without bound; fixed here, LMOT_ERR_CAPACITY when exceeded) */
  int max_points;            /* per frame, default 1<<20 */
  int max_clusters;          /* default 4096 (a 250x250 grid with 3x3 dilation cannot hold more) */
  int max_boxes;             /* default 1024 */
  int max_tracks;            /* rows of a track table: tracks ever created (dead ones keep their slot), or with track retirement
                                the live tracks plus one step's spawns; default 8192 */
  /* pre-filters of the reference's `ground` ROS node, applied BEFORE groundRemove (src/groundremove/main.cpp:56-89,104-112):
   * pcl::PassThrough on z (limits inclusive, non-finite points removed) then pcl::ConditionalRemoval x in (x_min,x_max) AND
   * y in (y_min,y_max) (strict).  Off by default: the hot path is groundRemove itself.  Fused into the first load. */
  int node_prefilter;        /* 0 */
  float filter_z_min, filter_z_max;   /* -3.0, 1.0  (ROS params filter_z_min / filter_z_max, main.cpp:147-148) */
  float filter_x_min, filter_x_max;   /* -15, 5     (main.cpp:68-71) */
  float filter_y_min, filter_y_max;   /* -50, 50    (main.cpp:73-76) */
  /* The `tracking` ROS node does not hand the boxes to immUkfJpdaf as they come: it moves them into a dead-reckoned "global" frame
   * first (pose of that frame in the sensor frame = egoPoints[0] of getOriginPoints, broadcast as tf velodyne -> global) and moves
   * targetPoints / visBBs back afterwards (tracking/main.cpp:76-83,142-158,182-195).  1: lmot_track_step / lmot_frame* / lmot_batch*
   * do the same on the device: boxes in, targets / vis_bb out stay in the SENSOR frame, the tracker state (and what lmot_tracker_dump
   * shows) is in the global frame.  0 (default): immUkfJpdaf as a function, boxes used as given.  The transform arithmetic is
   * pcl_ros::transformPointCloud's (float 4x4 from a double tf::Transform); tf and pcl_ros are not part of the reference tree.
   * With a sensor rig (lmot_set_sensors) the batched ticks first move each sensor's boxes into the vehicle frame with the same
   * evaluation, ((r00*x + r01*y) + r02*z) + t0 per row in float without contraction, and this step then runs on that list. */
  int global_frame;          /* 0 */
  /* frames in flight inside one context: detection stages of frame f+1.. overlap the tracker of frame f (1..8, default 4) */
  int pipeline_depth;
  /* result blocks (pinned host memory) = how many submitted frames may wait to be collected (1..64, default 32) */
  int result_ring;
} lmot_params;

typedef struct lmot_ctx lmot_ctx;

int lmot_default_params(lmot_params* p);
int lmot_create(lmot_ctx** out, const lmot_params* params, int device);
void lmot_destroy(lmot_ctx* ctx);
int lmot_get_params(const lmot_ctx* ctx, lmot_params* out);   /* the parameters the context runs with (capacities after clamping) */
const char* lmot_strerror(int status);
const char* lmot_last_error(const lmot_ctx* ctx); /* text of the last CUDA error seen by this context */
const char* lmot_build_info(void);

/* Caller stream (cudaStream_t passed as void*): stage-by-stage entry points run on it, and the frame pipeline forks from /
 * joins into it (lmot_frame_dev orders a frame after the work already queued on it; lmot_flush makes it wait for the
 * pipeline).  NULL restores the context's own stream -- the legacy default stream (handle 0) cannot be selected, create a
 * stream instead (CUDA events recorded on stream 0 are not ordered with the pipeline's non-blocking streams).  The stream being
 * replaced must still be valid at this call (the library may record an event on it), and a caller stream must be replaced
 * (or the context destroyed) before that stream is destroyed. */
int lmot_set_stream(lmot_ctx* ctx, void* cuda_stream);

/* Page-locked host memory for frames handed to lmot_frame / lmot_frame_submit (a pageable buffer makes the H2D copy
 * synchronous and half as fast).  A ROS node allocates its PointCloud2 staging buffer with this; NULL without a CUDA device. */
void* lmot_pinned_alloc(size_t bytes);
void lmot_pinned_free(void* p);

/* ---- stage entry points, HOST buffers (synchronous: H2D, kernels, D2H, stream sync) -------------------- */

/* groundRemove.  labels (nullable) gets one byte per input point: 0 = in neither output (range filter /
 * cell index out of range, ground_removal.cpp:54,233), 1 = ground, 2 = elevated.  With node_prefilter on, 0 = removed by
 * the node's pre-filters and 3 = survived them (i.e. belongs to the node's `aux_points` cloud, as 1 and 2 do) but in neither
 * output of groundRemove.  elevated / ground (nullable)
 * receive the order-preserving output clouds, stride 4 floats, capacity n points each. */
int lmot_ground_remove(lmot_ctx* ctx, const float* points, int n, int stride_floats, uint8_t* labels,
                       float* elevated, int* n_elevated, float* ground, int* n_ground);

/* componentClustering.  grid = int32[250*250], x-major like array<array<int,250>,250> (written entirely;
 * the caller's zero-initialisation at src/cluster/main.cpp:72-73 is implied). */
int lmot_component_cluster(lmot_ctx* ctx, const float* elevated, int n, int stride_floats, int32_t* grid,
                           int* num_cluster);

/* The cluster node's side outputs (src/cluster/main.cpp:62-99) for the elevated cloud and label grid of the most recent
 * lmot_component_cluster / lmot_frame of this context (synchronous; call it before submitting further frames):
 *   clustered  <- makeClusteredCloud  component_clustering.cpp:308-335   float[cap][4] (cell centre x, y, -1, 1), cloud order
 *   obstacles  <- setObsMsg           component_clustering.cpp:337-375   float[cap][4] (cell centre x, y, -1, cluster id):
 *                                      ONE obstacle per labelled cell that holds a point, in order of its first point
 *   cost_map   <- createCostMap       component_clustering.cpp:425-454   int32[50*50], row = y cell, column = x cell
 * all nullable; LMOT_ERR_CAPACITY if a requested list does not fit (the counts are still returned). */
int lmot_cluster_outputs(lmot_ctx* ctx, float* clustered, int cap_clustered, int* n_clustered, float* obstacles, int cap_obstacles,
                         int* n_obstacles, int32_t* cost_map);

/* boxFitting.  boxes = float[max_boxes*8*3] (4 bottom corners z=-sensor_height, then 4 top corners z=maxZ,
 * box_fitting.cpp:379-389), in cluster-id order.  markers (nullable) = float[max_boxes*6]: centroid xyz and
 * AABB extent xyz of the cluster (mark_cluster, box_fitting.cpp:161-209). */
int lmot_box_fit(lmot_ctx* ctx, const float* elevated, int n, int stride_floats, const int32_t* grid,
                 int num_cluster, float* boxes, int max_boxes, int* n_boxes, float* markers);

/* Outputs of immUkfJpdaf: one entry per track ever created (imm_ukf_jpda.cpp:995-1041).  All pointers are
 * caller-owned with capacity `cap` entries (vis_bb: cap boxes); nullable ones are skipped. */
typedef struct lmot_track_out {
  int cap;
  int n_tracks;        /* out */
  int n_vis;           /* out: number of boxes in vis_bb */
  float* targets;      /* [cap*3]  targetPoints (x, y, -1.73/2) */
  double* vandyaw;     /* [cap*2]  targetVandYaw (v, yaw + ego yaw) */
  int32_t* track_manage; /* [cap]  trackNumVec_ */
  uint8_t* is_static;  /* [cap] */
  uint8_t* is_vis;     /* [cap] */
  float* vis_bb;       /* [cap*8*3] boxes of the tracks with is_vis, in track order */
} lmot_track_out;

/* getOriginPoints(timestamp, v_gps, yaw_gps) then immUkfJpdaf(boxes, timestamp, ...).  timestamp in
 * microseconds (dt = (ts - ts_prev)/1e6, imm_ukf_jpda.cpp:807).  boxes = float[m*8*3]. */
int lmot_track_step(lmot_ctx* ctx, const float* boxes, int m, double timestamp_us, double v_gps, double yaw_gps,
                    lmot_track_out* out);

/* getOriginPoints (imm_ukf_jpda.cpp:74-172) on its own: what the ego origin points WOULD be for this frame, without
 * advancing the tracker (lmot_track_step / lmot_frame do the same fold internally).  out6 = {x, y, yaw, x, y, yaw+pi/2}. */
int lmot_origin_points(lmot_ctx* ctx, double timestamp_us, double v_gps, double yaw_gps, double out6[6]);

typedef struct lmot_frame_out {
  int n_elevated, n_ground, num_cluster, n_boxes; /* out */
  float* boxes;        /* nullable, [max_boxes*8*3] */
  int max_boxes;
  lmot_track_out tracks;
} lmot_frame_out;

/* The whole hot path on one frame: one H2D of the XYZI frame, four device-resident stages, one D2H. */
int lmot_frame(lmot_ctx* ctx, const float* points, int n, int stride_floats, double timestamp_us, double v_gps,
               double yaw_gps, lmot_frame_out* out);

/* ---- pipelined frames (asynchronous) ----------------------------------------------------------------------
 * A context keeps up to `pipeline_depth` frames in flight: the three detection stages of a frame run on one of
 * `pipeline_depth` internal streams (own buffers each) while the tracker -- a sequential fold over frames -- runs on
 * its own stream and consumes the box lists in submission order.  Results are identical to frame-at-a-time calls.
 *
 * lmot_frame_submit  : HOST frame (pinned memory recommended) -> H2D + all four stages, returns immediately.
 *                      LMOT_ERR_STATE if result_ring frames are already waiting to be collected (the result ring is
 *                      independent of pipeline_depth, so the host may run far ahead of the GPU).
 * lmot_frame_collect : blocks until the OLDEST submitted frame is done and returns its results
 *                      (the kernels wrote them into pinned host memory; no device copy is issued here).
 * lmot_frame_dev     : like submit, but the frame is already on the device (stride 4 floats, 16-byte aligned); ordered
 *                      after the work already queued on the context's caller stream (lmot_set_stream).  Uncollected
 *                      results older than result_ring submissions are dropped.
 * lmot_frame_fetch   : waits for everything submitted so far and returns the results of the MOST RECENT frame.
 * lmot_flush         : makes the caller stream wait (on the device, not the host) for everything submitted so far, so
 *                      that CUDA events recorded on the caller stream bracket the work. */
int lmot_frame_submit(lmot_ctx* ctx, const float* points, int n, int stride_floats, double timestamp_us, double v_gps,
                      double yaw_gps);
int lmot_frame_collect(lmot_ctx* ctx, lmot_frame_out* out);
int lmot_frames_in_flight(lmot_ctx* ctx, int* n);
/* 1 if lmot_frame_collect would return without waiting, 0 if the oldest frame is still running or nothing is in flight */
int lmot_frame_ready(lmot_ctx* ctx);
int lmot_frame_dev(lmot_ctx* ctx, const float* d_points, int n, double timestamp_us, double v_gps, double yaw_gps);
int lmot_frame_fetch(lmot_ctx* ctx, lmot_frame_out* out);
int lmot_flush(lmot_ctx* ctx);
int lmot_ground_remove_dev(lmot_ctx* ctx, const float* d_points, int n);
int lmot_detect_dev(lmot_ctx* ctx, const float* d_points, int n); /* ground + cluster + box, no tracker */
int lmot_sync(lmot_ctx* ctx);

/* ---- batched ticks: several sensor streams, ONE shared track table (BASELINE.json configs[3]) ------------------------------
 * One tick = one frame from each of n_frames (<= LMOT_MAX_BATCH) sensors.  Ground removal, clustering and box fitting of all
 * frames run as ONE launch per stage (CTA groups own frames); the frames' box lists, concatenated in stream order, are the
 * measurement list of ONE immUkfJpdaf step -- what the reference does when one tracking node receives the boxes of several
 * cluster nodes in one trackbox message (tracking/main.cpp:98-141,166; the monolithic callback object_tracking0/src/main.cpp:51-121
 * per stream).  Per-frame results are identical to lmot_ground_remove / lmot_component_cluster / lmot_box_fit on that frame, the
 * track outputs to lmot_track_step on the concatenation.  Submission / collection follow lmot_frame_submit / lmot_frame_collect
 * (same result ring; ticks and single frames may be mixed, the tracker folds them in submission order). */
#define LMOT_MAX_BATCH 8
typedef struct lmot_batch_out {
  int n_frames;                                   /* out */
  int n_elevated[LMOT_MAX_BATCH], n_ground[LMOT_MAX_BATCH], num_cluster[LMOT_MAX_BATCH], n_boxes[LMOT_MAX_BATCH];   /* out, per frame */
  int n_boxes_total;                              /* out: boxes in `boxes` (frame 0's first, then frame 1's, ...) */
  float* boxes;                                   /* nullable, [max_boxes*8*3] */
  int max_boxes;
  lmot_track_out tracks;
} lmot_batch_out;
int lmot_batch_submit(lmot_ctx* ctx, const float* const* points, const int* n, int n_frames, int stride_floats, double timestamp_us,
                      double v_gps, double yaw_gps);          /* HOST frames (pinned memory recommended) */
int lmot_batch_dev(lmot_ctx* ctx, const float* const* d_points, const int* n, int n_frames, double timestamp_us, double v_gps,
                   double yaw_gps);                           /* DEVICE frames, stride 4 floats, 16-byte aligned; ordered after the caller stream */
int lmot_batch_detect_dev(lmot_ctx* ctx, const float* const* d_points, const int* n, int n_frames);   /* no tracker step */
int lmot_batch_collect(lmot_ctx* ctx, lmot_batch_out* out);   /* oldest submitted tick */
int lmot_batch_fetch(lmot_ctx* ctx, lmot_batch_out* out);     /* most recent tick; older uncollected results are dropped */
int lmot_batch(lmot_ctx* ctx, const float* const* points, const int* n, int n_frames, int stride_floats, double timestamp_us,
               double v_gps, double yaw_gps, lmot_batch_out* out);   /* submit + collect */
/* ground removal + connected components only, two launches on the caller stream, results stay on the device (roofline measurement) */
int lmot_batch_ground_ccl_dev(lmot_ctx* ctx, const float* const* d_points, const int* n, int n_frames);

/* ---- sensor rig: where each sensor of a batched tick is mounted ------------------------------------------------------------------
 * Sensor k is frame k of a batched tick (lmot_batch, lmot_batch_submit, lmot_batch_dev, lmot_batch_detect_dev,
 * lmot_batch_ground_ccl_dev) and list k of lmot_track_step_lists_dev (rank k of lmot_shared_tick_dev in LMOT_SHARED_STREAMS mode;
 * in LMOT_SHARED_FRAMES mode every step is one list and uses sensor 0).  With sensors set:
 *   - frame k's ground removal uses sensor k's h_sensor / t_hmin / t_hmax and its box fitting sensor k's sensor_height in place of
 *     lmot_params' values: per-frame results equal lmot_ground_remove / lmot_box_fit on a context created with those four values;
 *   - where the tracker's measurement list is concatenated, every corner of list k's boxes is moved by sensor k's pose (sensor ->
 *     vehicle frame, row-major 3x4 [R | t]) as pcl::transformPointCloud evaluates it with an Affine3f, in float, without contraction:
 *         x' = ((r00*x + r01*y) + r02*z) + t0,  y' = ((r10*x + r11*y) + r12*z) + t1,  z' = ((r20*x + r21*y) + r22*z) + t2
 *     so the concatenated list, the tracker's input and lmot_batch_out.boxes are in the VEHICLE frame.  With global_frame = 1 the
 *     vehicle-frame list then takes the sensor -> global step of lmot_params.global_frame (the dead-reckoned ego pose is the
 *     vehicle's): two roundings in sequence, not one premultiplied matrix; targets and vis_bb come back in the vehicle frame.
 * The table is captured by value when a tick is submitted: ticks already in flight keep the table they were submitted with.  A tick or
 * list step with more frames than sensors is LMOT_ERR_INVALID while sensors are set.  Not affected: the stage entry points,
 * lmot_track_step, the single-stream lmot_frame* calls and sequence ticks (lmot_seq_*: each sequence has its own table,
 * lmot_seq_set_sensors).  Detections of one object by two sensors with overlapping fields of view stay two measurements (the reference
 * has no fusion step) unless the rig merges: lmot_set_rig_merge (below) clusters and boxes the sensors' elevated clouds as one. */
typedef struct lmot_sensor {
  float pose[12];                 /* sensor -> vehicle frame, row-major 3x4 [R | t]; R orthonormal (|R^T R - I| <= 1e-5 elementwise) */
  float h_sensor, t_hmin, t_hmax; /* ground removal: replace lmot_params' values for this sensor's frames */
  float sensor_height;            /* box fitting: likewise */
} lmot_sensor;
int lmot_default_sensor(const lmot_params* p, lmot_sensor* out);      /* identity pose + p's four values (p NULL: the defaults) */
/* n = 0 (s may be NULL): no sensors, every frame uses lmot_params.  LMOT_ERR_INVALID, table unchanged: n < 0, n > LMOT_MAX_BATCH,
 * a non-finite value, a rotation that is not orthonormal */
int lmot_set_sensors(lmot_ctx* ctx, const lmot_sensor* s, int n);
int lmot_get_sensors(const lmot_ctx* ctx, lmot_sensor* s, int cap, int* n);   /* *n = sensors set; copies min(n, cap) of them */

/* ---- merging rigs: the sensors' elevated clouds clustered and boxed together in the VEHICLE frame ----------------------------------------
 * With overlapping fields of view, separate detection gives an object seen by two sensors two boxes (two measurements, and a second track
 * where the tracker spawns one for every unmatched box), and cuts an object on the edge between two fields of view in two.  A rig with
 * merge on (off by default) and a table of F >= 1 sensors detects a tick as ONE cloud instead; a frame step of that rig gives, bit for bit:
 *   1. ground removal per sensor, exactly as without merge: frame j (deskewed first if deskew is on) with sensor j's h_sensor / t_hmin /
 *      t_hmax -> n_elevated[j], n_ground[j] and the order-preserving elevated cloud E_j in sensor j's frame;
 *   2. the merged cloud E = E_0' | E_1' | ... | E_{F-1}' in table order, E_j' = every point of E_j moved by sensor j's pose with the rig's
 *      arithmetic above (x' = ((r00*x + r01*y) + r02*z) + t0 and likewise y', z', in float without contraction), w = 1.  If |E| >
 *      max_points, E is cut at max_points in that order and the step's status is LMOT_ERR_CAPACITY; the cut step's results and later
 *      steps stay valid (the rule of an over-long list of lmot_seq_track_dev);
 *   3. componentClustering(E) with roi_m, boxFitting(E, grid, numCluster) with the box-fitting values of lmot_params, or of the sequence's
 *      lmot_detect_params if it has its own.  sensor_height is then the height of the VEHICLE frame's origin above the ground (box
 *      bottoms and the height test); no sensor's sensor_height is read;
 *   4. the boxes B, already in the vehicle frame, are the step's measurement list and lmot_batch_out.boxes (no pose applied again); with
 *      global_frame = 1 they take the global-frame step as a rig's list does.
 * That is: lmot_ground_remove(frame j) on a context created with sensor j's four values, for each j; the transform and concatenation
 * above; lmot_component_cluster(E) + lmot_box_fit(E, ...) + lmot_track_step(B) on a context with the step's parameters.
 * Counts: lmot_batch_out.n_elevated[j] / n_ground[j] per sensor; num_cluster[0] / n_boxes[0] the merged cloud's, the other entries 0;
 * n_boxes_total = |B|.  lmot_seq_frame_counts(k) gives the same rows, and out->seq[k] their sums.
 * Applies to the context's lmot_batch_submit / lmot_batch_dev / lmot_batch / lmot_batch_detect_dev while lmot_set_sensors holds a table,
 * and to the FRAMES steps of sequence k (lmot_seq*, lmot_seq_tick*) while lmot_seq_set_sensors(k) holds one.  Without a table the setting
 * has no effect and a tick runs exactly the launches it always did.  Never read by LISTS steps and lmot_seq_track*, the stage entry
 * points, lmot_frame*, lmot_track_step*, lmot_batch_ground_ccl_dev and lmot_shared_*.
 * Host state captured by value at submission, like the sensor tables: ticks in flight keep theirs.  lmot_seq_open turns it off for every
 * sequence; lmot_seq_tracker_reset / _load and LMOT_SEQ_RESTART keep it.
 * LMOT_ERR_INVALID, setting unchanged: on other than 0 or 1; k out of range or no open set.  LMOT_ERR_STATE, nothing submitted: a merging
 * submission in timing mode.
 * Memory: the first merging submission of the context allocates a merge unit per batch bank (2), and that of sequence k one per bank for
 * it, synchronising the device once: the merged cloud and the clustering / box-fitting buffers of one frame, 36 B x max_points +
 * 4 B x ceil(max_points / 1024) x (max_clusters + 1) + ~1 MB, about 55 MB at the default max_points and max_clusters: ~110 MB for the
 * context's rig and ~110 MB per merging sequence (~880 MB with all 8 merging).  All or nothing: a failed allocation frees both banks' units
 * and returns its error, and the next merging submission tries again.  Freed with the context (sequences: with the set). */
int lmot_set_rig_merge(lmot_ctx* ctx, int on);
int lmot_get_rig_merge(const lmot_ctx* ctx, int* on);
int lmot_seq_set_rig_merge(lmot_ctx* ctx, int k, int on);
int lmot_seq_get_rig_merge(const lmot_ctx* ctx, int k, int* on);

/* ---- independent sequences: up to LMOT_MAX_BATCH frame streams per tick, each with its OWN track table ---------------------------
 * A sequence is an independent frame stream (one vehicle, one replayed log): it has its own track table, its own getOriginPoints
 * state (timestamp, ego velocity and yaw, dead-reckoning fold, first-frame flag), its own global_frame pose and its own result block.
 * One tick carries one frame of each of the n_seq sequences (one per sensor for a sequence with a sensor table, at most LMOT_MAX_BATCH
 * frames in all).  Detection of all frames runs as the batched launches of lmot_batch_*, then ONE tracker chain steps all n_seq tables (one gate, TA, TB and TC launch per tick, whatever n_seq is).
 *
 * Sequence k of a tick gives bit for bit the results of a separate context created with the same lmot_params that receives sequence
 * k's frames through lmot_frame: the counts, the boxes (sensor frame), targets, vandyaw, trackManage, the static and visible flags,
 * vis_bb, the warning status and lmot_seq_tracker_dump (= that context's lmot_tracker_dump).  Sequences never interact, and the
 * context's own tracker (lmot_frame*, lmot_batch*, lmot_track_step*, lmot_tracker_*) is a separate table: sequence ticks and those
 * calls may be interleaved on one context without disturbing each other.  Timing mode (lmot_enable_timing) is not supported:
 * LMOT_ERR_STATE while it is on.
 *
 * Multi-sensor sequences (one vehicle with several LiDARs, or one LiDAR not mounted at lmot_params' height): lmot_seq_set_sensors(k)
 * gives sequence k its own sensor table, in lmot_set_sensors' format and with its rules.  Sequence k then has one frame per sensor in
 * every tick, and behaves bit for bit like a separate context with the same lmot_params and lmot_set_sensors(that table) that receives
 * those frames through lmot_batch: ground removal and box fitting with each sensor's thresholds, the frames' box lists concatenated in
 * table order and moved into the VEHICLE frame, one tracker step on that list.  out->seq[k] then follows lmot_batch_out's rules: the
 * counts are summed over its frames, boxes / n_boxes are the concatenated vehicle-frame list (LMOT_ERR_CAPACITY if it exceeds
 * max_boxes); lmot_seq_frame_counts gives the per-frame counts.  A sequence without a table keeps one frame per tick with lmot_params'
 * thresholds (its results stay those of lmot_frame), and with no table set a tick runs exactly the launches it always did.  The
 * context's own table (lmot_set_sensors) never applies to sequence ticks.
 *
 * lmot_seq_open(ctx, n_seq, ring): drains the context and replaces the set with n_seq (1..LMOT_MAX_BATCH) empty sequences, each at
 *   its first frame, and a ring of `ring` (1..64) ticks.  n_seq = 0 frees the set.  Memory: n_seq track tables (device, max_tracks x
 *   ~2.6 KB incl. side arrays at max_boxes 1024) plus ring x n_seq result blocks (each max_boxes x 96 B + max_tracks x 138 B of pinned host memory and
 *   the same again on the device), per sequence 2 x 2 x max_boxes x 96 B of device memory (a measurement list and its global-frame
 *   copy for each of the two detection banks), and 2 x 8 x max_boxes x 96 B of device memory (~1.5 MB at max_boxes 1024) staging the
 *   host lists of lmot_seq_track_submit -- size max_tracks and ring for it.  Reopening (or closing) also clears every sequence's sensor table.
 * lmot_seq_submit : HOST frames (stride in floats), LMOT_ERR_STATE if `ring` ticks wait to be collected.
 * lmot_seq_dev    : DEVICE frames (stride 4 floats, 16-byte aligned), ordered after the caller stream; a full ring drops the oldest tick.
 * points / n hold one entry per FRAME of the tick, in sequence order: sequence 0's frames (its sensors in table order, or its one
 * frame), then sequence 1's, and so on.  timestamp_us / v_gps / yaw_gps are arrays of n_seq (one per sequence): each sequence's dt
 * comes from its own previous stamp.  n[i] = 0 is an empty frame; that sequence's tracker still steps.  LMOT_ERR_INVALID: no open
 * set, n_seq of the call != the set's, null or misaligned pointers; LMOT_ERR_CAPACITY: a frame above max_points.
 * lmot_seq_collect: the OLDEST submitted tick (blocks until done); lmot_seq_fetch: the MOST RECENT one, older uncollected ticks are
 * dropped; lmot_seq: submit + collect.  out->seq[k] is an lmot_frame_out with the usual rules: caller-owned buffers and capacities; the
 * status is the first error of the tick's sequences, else its first warning.
 * lmot_seq_tracker_reset(k) drains first, like lmot_tracker_reset: the next tick is sequence k's first frame (with the
 * oracle_compat_first_frame quirk if that is on).  lmot_seq_tracker_dump uses lmot_tracker_dump's layout, lmot_seq_tracker_get_ego
 * lmot_tracker_get_ego's.  k out of range: LMOT_ERR_INVALID.
 * lmot_seq_set_sensors(k, s, n): sequence k's table; n = 0 (s may be NULL) removes it.  LMOT_ERR_INVALID, every table unchanged: k out
 *   of range (or no open set), lmot_set_sensors' rejections, or more than LMOT_MAX_BATCH frames per tick over the set (a sequence
 *   without a table counts one).  Host state only: submitted ticks keep the tables they were submitted with (copied into their launch
 *   parameters); lmot_seq_tracker_reset leaves the table alone.  lmot_seq_get_sensors reads it back as lmot_get_sensors does.
 * lmot_seq_frame_counts(k): (n_elevated, n_ground, num_cluster, n_boxes) of each of sequence k's frames in the tick most recently
 *   returned by lmot_seq_collect / lmot_seq_fetch / lmot_seq, and their number (0 before the first); a one-frame sequence's row equals
 *   out->seq[k]'s counts. */
typedef struct lmot_seq_out {
  int n_seq;                                      /* out */
  lmot_frame_out seq[LMOT_MAX_BATCH];             /* per sequence: caller sets boxes / max_boxes / tracks as for lmot_frame */
} lmot_seq_out;
int lmot_seq_open(lmot_ctx* ctx, int n_seq, int ring);
int lmot_seq_submit(lmot_ctx* ctx, const float* const* points, const int* n, int n_seq, int stride_floats, const double* timestamp_us,
                    const double* v_gps, const double* yaw_gps);
int lmot_seq_dev(lmot_ctx* ctx, const float* const* d_points, const int* n, int n_seq, const double* timestamp_us, const double* v_gps,
                 const double* yaw_gps);
int lmot_seq_collect(lmot_ctx* ctx, lmot_seq_out* out);
int lmot_seq_fetch(lmot_ctx* ctx, lmot_seq_out* out);
int lmot_seq(lmot_ctx* ctx, const float* const* points, const int* n, int n_seq, int stride_floats, const double* timestamp_us,
             const double* v_gps, const double* yaw_gps, lmot_seq_out* out);
int lmot_seq_tracker_reset(lmot_ctx* ctx, int k);
int lmot_seq_tracker_dump(lmot_ctx* ctx, int k, double* dumps, int cap, int* n);
int lmot_seq_tracker_get_ego(lmot_ctx* ctx, int k, double ego8[8]);
int lmot_seq_set_sensors(lmot_ctx* ctx, int k, const lmot_sensor* s, int n);
int lmot_seq_get_sensors(const lmot_ctx* ctx, int k, lmot_sensor* s, int cap, int* n);
int lmot_seq_frame_counts(lmot_ctx* ctx, int k, int counts[LMOT_MAX_BATCH][4], int* n_frames);

/* ---- tracking-only sequence ticks: each sequence's tracker fed with box lists from elsewhere (another detector, a detection log) -----
 * The sequence form of lmot_track_step: one tick carries the box lists of all n_seq sequences, and ONE tracker chain steps all tables
 * (no ground removal, clustering or box fitting runs).  Lists follow the frame layout of a detection tick: one list per sensor of a
 * sequence with a table (table order), one list for a sequence without one, in sequence order.  A box is float[8*3] as for
 * lmot_track_step; timestamp_us / v_gps / yaw_gps are arrays of n_seq as for lmot_seq_submit.
 *
 * Sequence k gives bit for bit what a separate context with the same lmot_params gives: without a table, lmot_track_step on its list;
 * with a table, lmot_set_sensors(that table) and lmot_track_step_lists_dev on its lists (each list's boxes moved into the VEHICLE
 * frame by its sensor's pose, as lmot_track_step_lists_dev does) -- targets, vandyaw, trackManage, static / visible flags, vis_bb,
 * the status and lmot_seq_tracker_dump, with global_frame 0 or 1.  out->seq[k]: boxes / n_boxes are the list that was tracked,
 * before the global-frame step (the caller's list, or the concatenated vehicle-frame list); n_elevated, n_ground and num_cluster are
 * 0; lmot_seq_frame_counts(k) gives one row (0, 0, 0, length) per list.  A sequence whose lists together exceed max_boxes reports
 * LMOT_ERR_CAPACITY at collect with its list cut at max_boxes, as its lmot_track_step_lists_dev twin does; the other sequences of the
 * tick are unaffected.
 *
 * Ticks use the ring of lmot_seq_*: lmot_seq_collect / lmot_seq_fetch, the same LMOT_ERR_STATE (host lists) and drop-oldest (device
 * lists) rules.  A set may mix detection ticks (lmot_seq*) and tracking ticks in any order; each table folds its steps in submission
 * order.  One lmot_seq* / lmot_seq_track* tick is all-detection or all-tracking and steps every sequence; lmot_seq_tick_* (below)
 * mixes the two kinds and steps any subset.
 * lmot_seq_track_submit: HOST lists boxes[i] of m[i] boxes.  LMOT_ERR_CAPACITY, nothing submitted: a list above max_boxes.  The
 *   lists and m are copied to a device staging buffer of the bank during the call (copies from pageable memory complete before the
 *   call returns; page-locked lists must stay untouched until lmot_flush has joined or the tick has been collected).
 * lmot_seq_track_dev: padded DEVICE lists as lmot_track_step_lists_dev takes them: list i at d_lists + i * cap_per_list * 24 floats
 *   (4-byte alignment suffices), its length in d_counts[i], clamped to [0, cap_per_list].  The tick is ordered after the work queued on
 *   the caller stream; the caller may overwrite the lists once lmot_flush has made its stream wait for the tick (or the tick has been
 *   collected), as for the frames of lmot_seq_dev.
 * lmot_seq_track: submit + collect, dropping uncollected ticks as lmot_seq does.
 * LMOT_ERR_INVALID: no open set, n_seq != the set's, null pointers, a negative m[i], cap_per_list < 1.  LMOT_ERR_STATE: timing mode.
 *
 * lmot_seq_tracker_load / lmot_seq_tracker_set_ego: lmot_tracker_load / lmot_tracker_set_ego applied to sequence k (same arguments
 * and rules; they drain first and drop uncollected sequence ticks, as lmot_seq_tracker_reset does).  k out of range: LMOT_ERR_INVALID;
 * n > max_tracks: LMOT_ERR_CAPACITY.  With lmot_seq_tracker_dump / lmot_seq_tracker_get_ego they move a sequence's checkpoint between
 * sequences and contexts (and to or from a context's own tracker). */
int lmot_seq_track_submit(lmot_ctx* ctx, const float* const* boxes, const int* m, int n_seq, const double* timestamp_us, const double* v_gps,
                          const double* yaw_gps);
int lmot_seq_track_dev(lmot_ctx* ctx, const float* d_lists, const int* d_counts, int n_seq, int cap_per_list, const double* timestamp_us,
                       const double* v_gps, const double* yaw_gps);
int lmot_seq_track(lmot_ctx* ctx, const float* const* boxes, const int* m, int n_seq, const double* timestamp_us, const double* v_gps,
                   const double* yaw_gps, lmot_seq_out* out);
int lmot_seq_tracker_load(lmot_ctx* ctx, int k, const double* dumps, int n, int init, double timestamp_us, double ego_velo,
                          double ego_yaw, double ego_pre_yaw, double ego_point_yaw);
int lmot_seq_tracker_set_ego(lmot_ctx* ctx, int k, const double ego8[8]);

/* ---- sequence ticks on each stream's own clock: any subset of the sequences, each from frames or box lists, restart in place ------
 * A tick describes each of the n_seq sequences with one lmot_seq_entry: LMOT_SEQ_SKIP (the sequence has no data this tick and does not
 * step), LMOT_SEQ_FRAMES (its frames: one per sensor of its table, or one without a table) or LMOT_SEQ_LISTS (its box lists, in the same
 * layout).  ONE tracker chain steps the stepped sequences' tables.  Streams at different rates, dropped frames, logs of different
 * lengths, and vehicles that send point clouds next to vehicles that send their own detector's boxes thus share one set and one chain.
 *
 * Equivalence: over any schedule of ticks, sequence k gives bit for bit what a separate context with the same lmot_params, tracker
 * parameters, retirement setting and detection parameters gives when it receives only sequence k's steps, in order, and nothing at
 * skipped ticks: a FRAMES step through lmot_frame (lmot_set_sensors(table) + lmot_batch with a table), a LISTS step through
 * lmot_track_step (lmot_track_step_lists_dev with the table).  This covers the counts, the boxes, every track output, the status,
 * lmot_seq_tracker_dump, lmot_seq_track_ids and lmot_seq_tracker_get_ego, with global_frame 0 or 1.  A sequence may switch kinds
 * from tick to tick.
 *
 * A skipped sequence is untouched: table, ego fold, stamp, first-frame flag, prediction stamp and IDs.  Its out->seq[k] is not written
 * (no count field, no caller buffer); lmot_seq_frame_counts(k) reports 0 frames for that tick; lmot_seq_track_ids(k) keeps the IDs of
 * its last returned step.  lmot_seq_stepped: bit k set iff sequence k stepped in the tick most recently returned by lmot_seq_collect /
 * lmot_seq_fetch / lmot_seq* (every bit of the set for lmot_seq* and lmot_seq_track* ticks).  The tick's status is the first error of
 * its stepped sequences, else their first warning.
 *
 * LMOT_SEQ_RESTART: the sequence first does what lmot_seq_tracker_reset(k) does -- empties its table, resets its ego state and
 * first-frame flag (the oracle_compat_first_frame quirk applies again), numbers its IDs from 0 -- then steps.  In stream order: nothing
 * is drained, other sequences' ticks stay in flight and their uncollected results are kept; a prediction queued before the tick sees the
 * old table.  Sensor tables, tracker and detection parameters and retirement are host state captured at submission, so a new stream on
 * sequence k is configured before its restarting tick without a drain.  lmot_seq_tracker_reset / _load / _set_ego still drain.
 *
 * Ticks use the ring of lmot_seq_* and mix freely with lmot_seq* and lmot_seq_track* ticks; each table folds its steps in submission
 * order.  lmot_seq_tick_submit: host data (frames with stride_floats, lists staged as lmot_seq_track_submit stages them);
 * LMOT_ERR_STATE when `ring` ticks wait to be collected.  lmot_seq_tick_dev: device data ordered after the caller stream (frames: stride
 * 4, 16-byte aligned; lists: data[j] of up to cap_per_list boxes, 4-byte alignment, lengths in the device ints d_counts[j] clamped to
 * [0, cap_per_list]); a full ring drops the oldest tick; a sequence whose lists together exceed max_boxes reports LMOT_ERR_CAPACITY at
 * collect with its list cut, the other sequences are unaffected.  lmot_seq_tick: submit + collect, dropping uncollected ticks as lmot_seq
 * does.  Timing mode: LMOT_ERR_STATE.
 * LMOT_ERR_INVALID, nothing submitted: no open set; n_seq != the set's; an unknown kind or flag bit; every entry SKIP; SKIP with
 * RESTART; a null data / n / d_counts where the kind needs it (a host frame or list of length > 0 needs its pointer, a device list
 * always); a negative count; cap_per_list < 1; a device frame that is not 16-byte aligned; a host FRAMES entry with stride_floats < 3.
 * LMOT_ERR_CAPACITY, nothing submitted: a frame above max_points, a host list above max_boxes. */
enum { LMOT_SEQ_SKIP = 0, LMOT_SEQ_FRAMES = 1, LMOT_SEQ_LISTS = 2 };
enum { LMOT_SEQ_RESTART = 1 };
typedef struct lmot_seq_entry {
  int kind;                    /* LMOT_SEQ_SKIP / _FRAMES / _LISTS */
  int flags;                   /* LMOT_SEQ_RESTART: the sequence starts over with this step */
  double timestamp_us, v_gps, yaw_gps;
  const float* const* data;    /* one per sensor of the sequence's table (one without a table): point arrays (FRAMES) or box lists (LISTS) */
  const int* n;                /* HOST ints: points per frame / boxes per list (dev form, LISTS: unused) */
  const int* d_counts;         /* dev form, LISTS only: DEVICE ints, list lengths */
  int cap_per_list;            /* dev form, LISTS only */
} lmot_seq_entry;
int lmot_seq_tick_submit(lmot_ctx* ctx, const lmot_seq_entry* e, int n_seq, int stride_floats);
int lmot_seq_tick_dev(lmot_ctx* ctx, const lmot_seq_entry* e, int n_seq);
int lmot_seq_tick(lmot_ctx* ctx, const lmot_seq_entry* e, int n_seq, int stride_floats, lmot_seq_out* out);
int lmot_seq_stepped(const lmot_ctx* ctx, uint32_t* mask);

/* ---- tracker parameters: the IMM-UKF-PDA noise, gating and track-management constants of one track table ------------------------
 * The defaults (lmot_default_tracker_params) are the reference's values; citations are file:line under object_tracking/tracking/.
 * A separate struct rather than fields of lmot_params, so that callers compiled against an older lmot_params keep working. */
typedef struct lmot_tracker_params {
  double gamma_g;              /* 9.22  chi-square gate, gammaG_ imm_ukf_jpda.cpp:26 (gate :230, PDA :263, likelihoods :374-388) */
  double p_g;                  /* 0.99  gate probability, pG_ :30 */
  double p_d;                  /* 0.9   detection probability, pD_ :34 */
  double distance_thres;       /* 99    box association distance (m), distanceThres_ :38 (associateBB :427-432) */
  int lifetime_thres;          /* 3     lifetime a track needs before a box is associated, lifeTimeThres_ :41 */
  double bb_yaw_change_thres;  /* 0.2   box yaw change (rad) below which the box is rotated, bbYawChangeThres_ :45 (updateBB :617-621) */
  double second_init_v;        /* 2     speed (m/s) of a track at its second initialisation, targetV :902 */
  int static_lifetime;         /* 8     lifetime above which a track may be flagged static, :1064 */
  double static_dist;          /* 3.0   distance (m) from the first position below which it is, distThres :1067 */
  double std_a[3];             /* 2, 2, 3  process noise, longitudinal acceleration (m/s^2) of CV, CTRV, RM: std_a_*_ ukf.cpp:68-70 */
  double std_yawdd[3];         /* 2, 2, 3  process noise, yaw acceleration (rad/s^2) of CV, CTRV, RM: std_*_yawdd_ ukf.cpp:71-73 */
  double std_las_x, std_las_y; /* 0.15, 0.15  lidar noise (m), std_laspx_ / std_laspy_ ukf.cpp:91-94 (R :841-842) */
  double trans[3][3];          /* IMM transition matrix, row i = p{i+1}_ (from model i to model j): 0.9 on the diagonal, 0.05 elsewhere,
                                  ukf.cpp:144-154 (MixingProbability :440-451) */
  double mode_prob0[3];        /* 0.33 each  initial mode probabilities of a new track, ukf.cpp:180-182 */
  double p0_diag[5];           /* 0.5, 0.5, 3, 10, 1  diagonal of a new track's covariance, P_merge_ ukf.cpp:275-279 */
} lmot_tracker_params;
/* Not parameters: the explosion guards (det > 10, P(4,4) > 1000, det(S) > 10), the mode-probability floor and the gate's S * 4, and
 * the UKF members gammaG_ / pD_ / pG_ (ukf.cpp:216-218: only UKF::PDAupdate reads them, which the tracker never calls).
 *
 * lmot_default_tracker_params(p): the defaults above.
 * lmot_set_tracker_params(ctx, p): the context's own track table (lmot_frame*, lmot_batch*, lmot_track_step, lmot_track_step_lists_dev,
 *   and through it the owner rank of lmot_shared_*).  p == NULL restores the defaults.  lmot_get_tracker_params reads them back.
 * lmot_seq_set_tracker_params(ctx, k, p) / lmot_seq_get_tracker_params: sequence k of the open set, for detection and tracking-only
 *   ticks alike.  lmot_seq_open (reopening the set) resets every sequence to the defaults; lmot_seq_tracker_reset / _load keep them.
 * Like the sensor tables, the parameters are host state captured by value when a step or tick is submitted: steps in flight keep the
 * values they were submitted with, and a change applies to every track of the table -- those that already exist included -- from the
 * next submitted step on.  (The reference fixes std_a, std_yawdd, the lidar noise and the transition matrix when a track's UKF is
 * constructed; a mid-run change here equals a reference whose constants are the new values, reloaded from lmot_tracker_dump.)
 * A table at the defaults runs the kernels it always ran; a tick in which any table has other values runs all of its tables through
 * kernels that read each table's values, with bit-identical results for the tables at the defaults.
 * LMOT_ERR_INVALID, parameters unchanged: a non-finite value; a standard deviation, gamma_g or p0_diag entry <= 0; p_g, p_d or a
 * mode_prob0 entry outside (0, 1]; a trans entry outside [0, 1] or a trans column that is all zero (the mixing divides by its weighted
 * sum); a negative lifetime_thres or static_lifetime; k out of range or no open set. */
int lmot_default_tracker_params(lmot_tracker_params* p);
int lmot_set_tracker_params(lmot_ctx* ctx, const lmot_tracker_params* p);
int lmot_get_tracker_params(const lmot_ctx* ctx, lmot_tracker_params* p);
int lmot_seq_set_tracker_params(lmot_ctx* ctx, int k, const lmot_tracker_params* p);
int lmot_seq_get_tracker_params(const lmot_ctx* ctx, int k, lmot_tracker_params* p);

/* ---- track retirement and track IDs: track a stream indefinitely ---------------------------------------------------------------------
 * By default a track table is append-only like the reference's targets_ / trackNumVec_: a dead track (trackManage 0) keeps its row and
 * is reported in every later frame, so a long stream fills max_tracks (LMOT_WARN_TRACK_TABLE_FULL) and every step costs more.
 * With retirement on, every step of the table ends by removing each track whose trackManage is 0; the remaining rows keep their
 * relative order and the next step's spawns are appended after them.  The results equal the reference with one extra operation after
 * every immUkfJpdaf: stably erase every i with trackNumVec_[i] == 0 from targets_ and trackNumVec_ (the ego state is not touched) --
 * the same trackManage, lifetime, static and visible flags, box and vis_bb rows bit for bit, UKF states to 1e-4 relative.
 *   Outputs: step f lists every row present during step f -- the rows retained after step f-1, then this step's spawns.  A track that
 *   dies in step f appears once with trackManage 0 (possibly visible) and is gone from step f+1.  lmot_tracker_num_tracks and
 *   lmot_tracker_dump (and the sequence forms) describe the retained table; the result's n_tracks is the number of its rows.
 *   max_tracks bounds the rows a step holds: the retained rows plus that step's spawns.
 *   The one deviation from the unbounded reference: mergeOverSegmentation (imm_ukf_jpda.cpp:682-695) tests every track, dead ones
 *   included, so there a visible box that contains the frozen position of a long-dead track promotes that visible track to 5.  Once
 *   the dead track is erased, that promotion does not happen.  Nothing else of the reference reads dead rows.
 * Track IDs.  Once rows move, a row index no longer names a track.  Every track has an int64 ID: the table's spawn counter at its
 *   spawn, 0, 1, 2, ... from the table's last reset / open / load (lmot_tracker_load numbers the loaded rows 0..n-1 and continues at n).
 *   A table that never retired has IDs equal to its row indices.
 * lmot_set_track_retirement(ctx, on) / lmot_get_track_retirement: the context's own table; lmot_seq_set_track_retirement(ctx, k, on) /
 *   lmot_seq_get_track_retirement: sequence k of the open set.  Off by default.  Host state captured by value when a step or tick is
 *   submitted, like the tracker parameters: steps in flight keep the setting they were submitted with.  lmot_seq_open turns it off for
 *   every sequence; lmot_tracker_reset / _load and lmot_seq_tracker_reset / _load keep it (and return the IDs to the row indices).
 *   A table that retired and is then switched off keeps numbering its tracks (its IDs stay right) until reset, load or reopen.
 * lmot_track_ids(ctx, ids, cap, n): the IDs of the rows of the result most recently returned for the context's own table (lmot_track_step,
 *   lmot_frame, lmot_frame_collect / _fetch, lmot_batch, lmot_batch_collect / _fetch, lmot_track_step_lists_dev), in the order of its
 *   outputs; *n = their number, min(*n, cap) are copied.  lmot_seq_track_ids(ctx, k, ...): sequence k of the tick most recently returned
 *   by lmot_seq_collect / lmot_seq_fetch / lmot_seq / lmot_seq_track.
 * LMOT_ERR_INVALID: k out of range, no open set, a null pointer (ids may be NULL when cap is 0).  LMOT_ERR_STATE: no result yet.
 * Not supported: retirement on a context driven by lmot_shared_tick_dev of liblmot_shared.so -- its receiving ranks hold no IDs. */
int lmot_set_track_retirement(lmot_ctx* ctx, int on);
int lmot_get_track_retirement(const lmot_ctx* ctx, int* on);
int lmot_seq_set_track_retirement(lmot_ctx* ctx, int k, int on);
int lmot_seq_get_track_retirement(const lmot_ctx* ctx, int k, int* on);
int lmot_track_ids(lmot_ctx* ctx, int64_t* ids, int cap, int* n);
int lmot_seq_track_ids(lmot_ctx* ctx, int k, int64_t* ids, int cap, int* n);

/* ---- track prediction: every track's IMM-UKF state, covariance and gate at caller-given later times ---------------------------------
 * For a track table, query time t (us, the clock of lmot_track_step) and row i, on a COPY of the track (the table is never modified):
 *   dt = (t - ts_last) / 1e6, ts_last = the stamp of the table's most recently SUBMITTED step, or the stamp given to lmot_tracker_load
 *   (computed as a step computes its dt, imm_ukf_jpda.cpp:807).
 *   trackManage 0: nothing is predicted, flag LMOT_PRED_DEAD.
 *   det(P_merge) > 10 || P_merge(4,4) > 1000 (the explosion guard, :828): nothing is predicted, flag LMOT_PRED_GUARD_P (a step would kill
 *   the track before predicting it).
 *   Otherwise ProcessIMMUKF(dt) (ukf.cpp:507-527: mixing, interaction, Prediction(dt, 0..2), UpdateLidar(0..2), which only sets zPred /
 *   S / K), findMaxZandS (imm_ukf_jpda.cpp:176), then PostProcessIMMUKF({1, 1, 1}) (ukf.cpp:529-535): the merge of a step that brings no
 *   information -- mode probabilities renormalised with the 1e-4 floor, merged mean and covariance, the yaw of the most probable model.
 *   Reported: x (x, y, v, yaw, yaw rate) and P (5x5, row-major) of the merge, the three mode probabilities, gate_z / gate_S = the
 *   max-det(S) model's predicted measurement and S (before the x4 of :844); flag LMOT_PRED_VALID, plus LMOT_PRED_GUARD_S if
 *   isnan(det(4 S)) || det(4 S) > 10 (:848: a step at t would kill the track).  dt = 0 is allowed: it is the mixed state, not the posterior.
 *   The values of rows that are not predicted are NaN.
 * Rows: the table as lmot_tracker_dump sees it, in that order, each with its int64 track ID (lmot_track_ids: the row index for a table
 * that never retired) and its trackManage.  Frame: the tracker's -- the dead-reckoned global frame with global_frame = 1, else the frame
 * the boxes came in (lmot_tracker_get_ego gives the pose).  Parameters: the table's current tracker parameters (std_a, std_yawdd, the lidar
 * noise and trans of lmot_set_tracker_params), the values the next submitted step would use.
 * Output layout (lmot_pred_out): ids / track_manage [cap]; flags [n_t][cap]; x [n_t][cap][5]; P [n_t][cap][25]; mode_prob [n_t][cap][3];
 * gate_z [n_t][cap][2]; gate_S [n_t][cap][4] (gate_z / gate_S nullable).  Rows beyond cap are not written; the row count is still
 * returned (n_rows / d_n_rows), and the host forms then return LMOT_ERR_CAPACITY.
 * lmot_predict_tracks(ctx, t_us, n_t, out): the context's own table, host outputs, out->n_rows = the row count.  Waits only for the
 *   prediction, which is ordered after the latest submitted step on the device; it does not drain the detection slots.
 * lmot_predict_tracks_dev(ctx, t_us, n_t, d_out, d_n_rows): the same into DEVICE arrays (d_out itself is a host struct), row count into
 *   the device int d_n_rows (nullable); asynchronous: the caller stream (lmot_set_stream) waits for it on the device.
 * lmot_seq_predict_tracks(ctx, k, t_us, n_t, out): sequence k of the open set, host outputs.
 * lmot_seq_predict_tracks_dev(ctx, t_us, n_t, d_outs, d_n_rows): every sequence in ONE launch; t_us [n_seq][n_t] (host), d_outs [n_seq]
 *   host structs of device arrays, d_n_rows [n_seq] device ints (nullable).
 * A prediction runs on the tracker chain's stream right behind the latest submitted step; the next step of the context then starts one
 * launch latency later (its first kernel waits for the prediction to finish).  Contexts that never predict run unchanged.
 * LMOT_ERR_INVALID: n_t outside [1, LMOT_MAX_PRED_TIMES], a non-finite t or t before ts_last, cap < 0, a required array null while
 * cap > 0, k out of range / no open set.  LMOT_ERR_STATE: the table has neither stepped nor been loaded since reset or open; the
 * sequence forms in timing mode. */
#define LMOT_MAX_PRED_TIMES 32
enum {
  LMOT_PRED_VALID = 1,     /* predicted */
  LMOT_PRED_DEAD = 2,      /* trackManage 0: not predicted */
  LMOT_PRED_GUARD_P = 4,   /* the P_merge explosion guard holds: not predicted */
  LMOT_PRED_GUARD_S = 8    /* predicted, but det(4 S) is NaN or > 10: a step at t would kill the track */
};
typedef struct lmot_pred_out {
  int cap;                 /* rows the arrays hold */
  int n_rows;              /* host forms: rows of the table (may exceed cap) */
  int64_t* ids;            /* [cap] */
  int32_t* track_manage;   /* [cap] */
  uint8_t* flags;          /* [n_t][cap] LMOT_PRED_* bits */
  double* x;               /* [n_t][cap][5] */
  double* P;               /* [n_t][cap][25] */
  double* mode_prob;       /* [n_t][cap][3] */
  double* gate_z;          /* [n_t][cap][2], nullable */
  double* gate_S;          /* [n_t][cap][4], nullable */
} lmot_pred_out;
int lmot_predict_tracks(lmot_ctx* ctx, const double* t_us, int n_t, lmot_pred_out* out);
int lmot_predict_tracks_dev(lmot_ctx* ctx, const double* t_us, int n_t, const lmot_pred_out* d_out, int* d_n_rows);
int lmot_seq_predict_tracks(lmot_ctx* ctx, int k, const double* t_us, int n_t, lmot_pred_out* out);
int lmot_seq_predict_tracks_dev(lmot_ctx* ctx, const double* t_us, int n_t, const lmot_pred_out* d_outs, int* d_n_rows);

/* ---- detection parameters of one sequence: ground removal, clustering ROI and box fitting ------------------------------------------
 * lmot_params' detection fields, as a separate struct (callers compiled against today's lmot_params keep working).  Defaults are
 * lmot_default_params' values; citations are file:line under object_tracking/src/. */
typedef struct lmot_detect_params {
  /* ground removal -- groundremove/ground_removal.cpp */
  float r_min, r_max;               /* 3.4, 120   range window, rMin / rMax :24-25 (filter :53, bin :71) */
  float t_hmin, t_hmax;             /* -2.0, -0.4 height clamp, tHmin / tHmax :27,29 (:194-196) */
  float t_hdiff;                    /* 0.4        hDiff threshold, tHDiff :32 */
  float h_sensor;                   /* 2.0        clamp value above t_hmax, hSeonsor :33 (:195) */
  double ground_tolerance;          /* 0.25       label margin above hGround, a literal at :239 */
  /* pre-filters of the `ground` node (groundremove/main.cpp:56-89,104-112), as lmot_params.node_prefilter */
  int node_prefilter;               /* 0 */
  float filter_z_min, filter_z_max; /* -3.0, 1.0 */
  float filter_x_min, filter_x_max; /* -15, 5 */
  float filter_y_min, filter_y_max; /* -50, 50 */
  /* clustering */
  float roi_m;                      /* 50         roiM cluster/component_clustering.cpp:11 (and box fitting's picScale = 900/roiM,
                                                  cluster/box_fitting.cpp:18) */
  /* box fitting -- cluster/box_fitting.cpp */
  int ram_points;                   /* 80         L-shape draws, ramPoints :19 (:314); 1..LMOT_MAX_RAM_POINTS */
  int l_slope_dist;                 /* 1          lSlopeDist :20 */
  int l_num_points;                 /* 5          lnumPoints :23 */
  float sensor_height;              /* 2          sensorHeight :26 */
  float t_height_min, t_height_max; /* 0.8, 2.6   tHeightMin / tHeightMax :28-29 */
  float t_width_min, t_width_max;   /* 0.2, 3.5   tWidthMin / tWidthMax :32-33 */
  float t_len_min, t_len_max;       /* 0.2, 14    tLenMin / tLenMax :34-35 */
  float t_area_max;                 /* 20         tAreaMax :36 */
  float t_ratio_min, t_ratio_max;   /* 1, 8       tRatioMin / tRatioMax :40-41 */
  float min_len_ratio;              /* 3          minLenRatio :43 */
  float t_pt_per_m3;                /* 8          tPtPerM3 :44 */
  int min_cluster_points;           /* 30         a literal at :100 (`numPoints < 30`) */
  int rule_filter;                  /* lmot_rule_filter, LMOT_RULE_INTENDED */
} lmot_detect_params;
/* box fitting evaluates the first LMOT_MAX_RAM_POINTS draws of the reference's mt19937_64(0) stream exactly; a Lemire redraw (odds
 * n / 2^64 per draw) needs one draw more, and the library's table covers those too */
#define LMOT_MAX_RAM_POINTS 1024
/* lmot_default_detect_params(p, out): p's detection fields (p NULL: lmot_default_params' values).
 * lmot_seq_set_detect_params(ctx, k, p): sequence k of the open set detects with p from the next submitted tick on.  Sequence k then
 *   gives bit for bit what a separate context gives that was created with the same lmot_params except that its detection fields are p:
 *   through lmot_frame for a sequence without a sensor table, through lmot_set_sensors(table) + lmot_batch for one with a table (the
 *   table's four mounting values still replace h_sensor / t_hmin / t_hmax / sensor_height of p for that sensor's frames).  p == NULL:
 *   the sequence follows lmot_params again.  lmot_seq_get_detect_params reads the values back (lmot_params' own while it follows them).
 * Like the sensor tables and tracker parameters, the values are host state captured by value when a tick is submitted: ticks in flight
 * keep theirs.  lmot_seq_open resets every sequence to lmot_params; lmot_seq_tracker_reset / _load keep them; tracking-only ticks
 * (lmot_seq_track*) do not read them.  A tick in which no sequence has its own values runs exactly the kernels it always ran; a tick in
 * which any has runs all of its frames through kernels that read each frame's values (bit-identical for sequences following lmot_params).
 * LMOT_ERR_INVALID, every sequence unchanged: no open set or k out of range; a non-finite value; r_min < 0 or r_max <= r_min; a range
 * window shorter than a fifth of r_max (r_max - r_min < r_max / 5: the guarded fast path of the polar cell index is only exact for
 * wider windows, DESIGN.md §6d); roi_m <= 0; rule_filter not an lmot_rule_filter; ram_points outside [1, LMOT_MAX_RAM_POINTS]. */
int lmot_default_detect_params(const lmot_params* p, lmot_detect_params* out);
int lmot_seq_set_detect_params(lmot_ctx* ctx, int k, const lmot_detect_params* p);
int lmot_seq_get_detect_params(const lmot_ctx* ctx, int k, lmot_detect_params* p);

/* ---- sweep deskew: every point of a frame moved to the frame's stamp from its own capture time and the stream's ego motion -----------
 * A spinning LiDAR takes a whole period (100 ms at 10 Hz) to sweep; on a moving vehicle the points of one frame are seen from different
 * poses, so static objects shift with their azimuth and an object on the sweep seam splits in two.  With deskew on, every frame is
 * first moved point by point into the vehicle's (sensor's) frame at the frame's timestamp; detection and tracking then run exactly as
 * on any other cloud.  The reference has no such step: deskew is opt-in, and with it off every launch and result is what it was.
 *
 * Definition.  Point i's time tau_i = (double)f[time_field] * time_scale + time_offset seconds relative to the frame's timestamp_us
 * (evaluated in double, without contraction).  The frame's motion is v = its v_gps and omega = remainder(diffYaw, 2 pi) / dt, with
 * diffYaw = egoYaw - egoPreYaw and dt = (ts - ts_prev) / 1e6 exactly as getOriginPoints' fold (lmot_origin_points) computes them for
 * this frame of this stream; omega = 0 on the stream's first frame (after create, lmot_tracker_reset / _load with init = 0,
 * lmot_seq_open, LMOT_SEQ_RESTART) and whenever dt <= 0 or a value is not finite (a non-finite v_gps gives v = 0).  The vehicle moves
 * along its +x axis and turns about +z, counter-clockwise positive; its pose at tau in its frame at the stamp is th = omega * tau,
 * tx = v * sin(th) / omega, ty = v * (1 - cos(th)) / omega (|omega| < 1e-9: tx = v * tau, ty = 0), rotation th about z.  The pose table
 * has LMOT_DESKEW_SLICES slices over [t_min, t_max): h = (t_max - t_min) / LMOT_DESKEW_SLICES, slice s at tau_s = t_min + (s + 0.5) h,
 * D_s = M^-1 T(tau_s) M built in double and rounded to float once per entry, M the sensor's mount pose (the rig table entry of the
 * frame's sensor, widened from float; identity without a table), M^-1 = [R^T | -R^T t].  lmot_deskew_table returns it (no device
 * needed).  Point i uses slice s = clamp(floor((tau_i - t_min) / h), 0, LMOT_DESKEW_SLICES - 1) and becomes, in float without
 * contraction, x' = ((d00*x + d01*y) + d02*z) + d03 (likewise y', z'), w = 1.  A point whose tau is not finite is passed unmoved.
 *
 * Equivalence (bit for bit): a context with deskew on given frame P through lmot_frame / lmot_frame_submit / lmot_frame_dev returns
 * what the same context with deskew off returns for the deskewed cloud P' (stride 4, same stamps and ego inputs): counts, boxes, every
 * track output, the status, the tracker dump; the elevated and ground clouds are those of P'.  lmot_batch_submit / lmot_batch_dev deskew each
 * sensor's frame with its own mount; sequences (lmot_seq_set_deskew) deskew the FRAMES steps of lmot_seq* / lmot_seq_tick* with their own
 * fold and sensor table, as a separate context with lmot_set_deskew would.  Node pre-filters, global_frame and retirement act on P'.
 *
 * The setting is host state captured by value at submission, as the sensor tables: frames in flight keep theirs.  lmot_seq_open turns
 * deskew off for every sequence; lmot_seq_tracker_reset / _load keep it; LISTS steps ignore it.  Not affected (no stamp, no ego): the
 * stage entry points (lmot_ground_remove, lmot_component_cluster, lmot_box_fit), lmot_detect_dev, lmot_batch_detect_dev,
 * lmot_batch_ground_ccl_dev, the tracking-only calls and lmot_shared_*.  With deskew on, LMOT_ZERO_COPY takes the copy path, and a host
 * frame with stride_floats > 4 is staged whole on the device (its staging grows once, synchronously, to the largest frame seen).
 *
 * Errors.  LMOT_ERR_INVALID from lmot_set_deskew / lmot_seq_set_deskew / lmot_deskew_table, setting unchanged: a non-finite value,
 * t_min >= t_max, t_max - t_min > 1 s, time_field < 3, k out of range (lmot_deskew_table: also non-finite v / omega, an invalid mount).
 * At submission, nothing submitted: LMOT_ERR_INVALID for a host frame with stride_floats <= time_field or a device frame while
 * time_field != 3; LMOT_ERR_STATE while timing mode (lmot_enable_timing) is on. */
#define LMOT_DESKEW_SLICES 256
typedef struct lmot_deskew {
  int on;                    /* 0 */
  int time_field;            /* 3: index of the float holding the point's time (device frames: must be 3, the 4th float) */
  double time_scale;         /* 1.0: tau = field * time_scale + time_offset, in seconds relative to the frame's timestamp_us */
  double time_offset;        /* 0.0 */
  double t_min, t_max;       /* -0.1, 0.0: the window the pose table covers (s); t_min < t_max, both finite, t_max - t_min <= 1 */
} lmot_deskew;
int lmot_default_deskew(lmot_deskew* d);
int lmot_set_deskew(lmot_ctx* ctx, const lmot_deskew* d);               /* d NULL: the defaults (off) */
int lmot_get_deskew(const lmot_ctx* ctx, lmot_deskew* d);
int lmot_seq_set_deskew(lmot_ctx* ctx, int k, const lmot_deskew* d);    /* sequence k of the open set; d NULL: the defaults (off) */
int lmot_seq_get_deskew(const lmot_ctx* ctx, int k, lmot_deskew* d);
/* the pose table of one frame: v, omega as above, mount NULL: identity */
int lmot_deskew_table(const lmot_deskew* d, double v, double omega, const lmot_sensor* mount, float out[LMOT_DESKEW_SLICES][12]);

/* ---- detection areas: cluster and box only the elevated points inside caller-given polygons -------------------------------------------
 * The detector is geometric: every elevated cluster that passes the rule filter becomes a box, and every unmatched box spawns a track --
 * poles, hedges, building corners, parked rows and the ego vehicle's own body included.  A detection area restricts clustering and box
 * fitting to a region of interest (a drivable-area polygon from a map, moved into the vehicle frame each tick) or, with keep_outside,
 * excludes zones from them, while ground removal still sees the whole frame.
 *
 * Definition.  An area is a set of closed polygon rings, vertices double (x, y) in metres in the VEHICLE frame (a stream without a sensor
 * table: the sensor frame).  For every unit of a FRAMES step of a stream with an area (a table-less frame, an unmerged rig frame, or a
 * merge unit):
 *   1. ground removal runs exactly as without an area: n_elevated, n_ground and both clouds are unchanged;
 *   2. the unit has a pose M = [R | t] (table-less frame and merge unit: identity; unmerged rig frame: sensor j's pose) and a clustering
 *      extent roi (lmot_params.roi_m, or the sequence's lmot_detect_params.roi_m).  Its cell mask is lmot_detect_area_mask(area, pose, roi):
 *      the 250 x 250 clustering grid in the bit-plane layout word x*8 + (y>>5), bit y&31 (bits above 250 in word 7 are 0).  All arithmetic
 *      is double, evaluated left to right without contraction; the pose is widened from float and only its xy block is used:
 *        vertex p in unit coordinates: dx = px - t0, dy = py - t1, u = r00*dx + r10*dy, w = r01*dx + r11*dy (identity: exactly (px, py));
 *        cell centre cx(xI) = ((double)xI + 0.5) * roi / 250.0 - roi / 2.0, cy(yI) likewise;
 *        PNPOLY with the ray along +y: an edge a -> b (rings closed implicitly) straddles row xI iff (a.u > cx) != (b.u > cx), and crosses it
 *        at yc = a.w + (cx - a.u) * (b.w - a.w) / (b.u - a.u); cell (xI, yI) is inside iff an odd number of straddling edges, over all
 *        rings, have cy(yI) < yc (even-odd: nested rings are holes, rectangles rasterise a raster);
 *        mask bit = inside != keep_outside;
 *   3. E_area = the points of the unit's elevated cloud whose clustering cell (componentClustering's float binning with the unit's roi)
 *      has its mask bit set, in cloud order;
 *   4. componentClustering(E_area) and boxFitting(E_area, grid, numCluster) with the unit's values; the tracker, global frame, retirement
 *      and the rest run as usual on those boxes.
 * That is the pipeline without an area with this filter between ground removal and clustering, bit for bit.
 *
 * Applies to lmot_frame / _submit / _dev and lmot_detect_dev (lmot_set_detect_area), lmot_batch* including lmot_batch_detect_dev (the
 * context's area), and the FRAMES steps of lmot_seq* / lmot_seq_tick* (lmot_seq_set_detect_area).  Never to the stage entry points,
 * lmot_batch_ground_ccl_dev, lmot_track_step*, LISTS steps and lmot_seq_track*.  lmot_cluster_outputs after a masked lmot_frame describes
 * E_area (makeClusteredCloud, setObsMsg and createCostMap on E_area).
 * Host state captured by value at submission, like the sensor tables: ticks in flight keep theirs, so a moving vehicle sets its polygons
 * before each submission.  lmot_seq_open turns every sequence's area off; lmot_seq_tracker_reset / _load and LMOT_SEQ_RESTART keep it.
 * The library copies the vertices.  NULL or n_rings = 0 turns the area off; a submission without an area runs exactly the launches it ran
 * before areas existed.  A masked submission clusters in a launch of its own instead of the ground kernel's tail.
 * Errors.  LMOT_ERR_INVALID, setting unchanged: n_rings outside [0, LMOT_AREA_MAX_RINGS], a ring with fewer than 3 vertices, more than
 * LMOT_AREA_MAX_VERTICES vertices in all, a non-finite vertex, keep_outside not 0 or 1, null pointers with n_rings > 0, k out of range or
 * no open set.  LMOT_ERR_STATE, nothing submitted: a masked submission in timing mode.
 * Memory: on the first masked submission, 8 KB of mask per detection slot, batch slot or merge unit it uses, and 16.3 KB of vertex staging
 * per stream, pinned per result-ring entry (sequence ticks: per ring tick and sequence) and on the device per slot or bank.  Freed with
 * the context.
 * lmot_detect_area_mask(area, mount, roi_m, out): the mask of step 2 on the host (no device needed), mount NULL: identity.
 * lmot_get_detect_area / lmot_seq_get_detect_area: the counts into *n_rings / *n_vertices / *keep_outside (each nullable), and as many
 * ring lengths and vertices as cap_rings / cap_vertices hold (ring_len / xy nullable when their capacity is 0).
 * lmot_debug_area_masks(ctx, out, cap_units, n_units): the device masks of the context's most recent own-stream submission (lmot_frame*,
 * lmot_detect_dev, lmot_batch*), one per unit in unit order, out = uint32[cap_units][LMOT_NUM_GRID * 8]; *n_units = 0 when it was not
 * masked.  Waits for the device. */
#define LMOT_AREA_MAX_RINGS 64
#define LMOT_AREA_MAX_VERTICES 1024
typedef struct lmot_area {
  int n_rings;
  const int* ring_len;         /* [n_rings] vertices of each ring, >= 3 */
  const double* xy;            /* [sum(ring_len)][2] vertices, ring after ring, metres in the vehicle frame */
  int keep_outside;            /* 0: keep the inside; 1: keep the outside (exclusion zones) */
} lmot_area;
int lmot_set_detect_area(lmot_ctx* ctx, const lmot_area* area);
int lmot_get_detect_area(const lmot_ctx* ctx, int* n_rings, int* ring_len, int cap_rings, int* n_vertices, double* xy, int cap_vertices,
                         int* keep_outside);
int lmot_seq_set_detect_area(lmot_ctx* ctx, int k, const lmot_area* area);
int lmot_seq_get_detect_area(const lmot_ctx* ctx, int k, int* n_rings, int* ring_len, int cap_rings, int* n_vertices, double* xy,
                             int cap_vertices, int* keep_outside);
int lmot_detect_area_mask(const lmot_area* area, const lmot_sensor* mount, float roi_m, uint32_t out[LMOT_NUM_GRID * 8]);
int lmot_debug_area_masks(lmot_ctx* ctx, uint32_t* out, int cap_units, int* n_units);

/* ---- sweep accumulation: cluster and box a frame together with the stream's last sweeps, moved into the current frame ----------------
 * The detector drops sparse objects where it counts points: componentClustering seeds only cells holding more than one point, and the
 * rule filter drops clusters under min_cluster_points or t_pt_per_m3.  On 16- and 32-beam sensors a car at 20 m or a pedestrian at 15 m
 * often stays under those counts.  Accumulation detects on the last K sweeps together, each moved by the ego motion between its stamp
 * and the current one.  Static objects register; moving objects smear by their speed times max_age_s at most.
 *
 * Definition.  A stream (the context's own: lmot_set_accumulate; sequence k: lmot_seq_set_accumulate) with sweeps = K > 1 keeps a
 * HISTORY per detection unit (a frame without a sensor table, an unmerged rig frame j, or a merge unit): the unit's cloud E_s (the
 * elevated cloud after deskew, before any detection-area mask; a merge unit's: the merged vehicle-frame cloud) of each of the stream's
 * last K-1 recorded steps, with that step's stamp ts_s and fold f_s = (x, y, yaw), the fold of the stream's track table after the
 * step's getOriginPoints (ego8[5..7] of lmot_tracker_get_ego / lmot_seq_tracker_get_ego read after the step).  Step t of a unit:
 *   1. ground removal, deskew and the rig merge are unchanged: n_elevated, n_ground and the clouds are what they are without it;
 *   2. the pose of an earlier step s, in double with the host libm, left to right, without contraction:
 *        c = cos(yaw_t - yaw_s), sn = sin(yaw_t - yaw_s), tx = x_t - (c*x_s - sn*y_s), ty = y_t - (sn*x_s + c*y_s),
 *        A = [[c, -sn, 0, tx], [sn, c, 0, ty], [0, 0, 1, 0]] (= G_t G_s^-1, G the global -> sensor pose of lmot_params.global_frame);
 *      D = M^-1 A M with M the unit pose as detection areas define it (a frame without a table and a merge unit: identity; unmerged
 *      rig frame j: sensor j's pose), M^-1 = [R^T | -R^T t] with
 *      -R^T t row r = -((R0r*t0 + R1r*t1) + R2r*t2), the pose widened from float.  Both products are 4x4 with the implicit last row
 *      (0 0 0 1), entry (r, k) = ((X[r][0]*Y[0][k] + X[r][1]*Y[1][k]) + X[r][2]*Y[2][k]) + X[r][3]*Y[3][k]; first P = A M, then
 *      D = M^-1 P; each entry of D's first three rows is rounded to float once.  lmot_accumulate_pose computes it;
 *   3. E_acc = E_t | D_1 E_s1 | D_2 E_s2 | ...: earlier steps newest first, each in its own cloud order, each point moved by the rig
 *      arithmetic of lmot_set_sensors (((d00*x + d01*y) + d02*z) + d03 per row, float, no contraction) with w = 1.  The steps used are
 *      the longest newest-first prefix of the history whose every entry has 0 < (ts_t - ts_s) / 1e6 <= max_age_s and fits WHOLE,
 *      together with E_t and every sweep before it, in max_points.  A sweep is never cut; leaving sweeps out is not an error;
 *   4. the detection area, if any, filters E_acc with the unit's mask exactly as it filters a plain frame; then componentClustering(E_acc)
 *      and boxFitting with the unit's values.  The tracker, global frame and retirement follow as usual on those boxes;
 *   5. E_t (not E_acc) joins the history; the oldest entry beyond K-1 leaves.
 * That is the pipeline without accumulation with this cloud between ground removal and clustering, bit for bit.
 *
 * Applies to lmot_frame / lmot_frame_submit / lmot_frame_dev, lmot_batch_submit / lmot_batch_dev / lmot_batch (every unit of the tick,
 * merged or not) and the FRAMES steps of lmot_seq* / lmot_seq_tick*.  Never to entry points without a stamp, which never touch the
 * history: the stage entry points, lmot_detect_dev, lmot_batch_detect_dev, lmot_batch_ground_ccl_dev, and lmot_shared_*.  LISTS steps,
 * lmot_track_step* and lmot_seq_track* advance the fold without recording, so older sweeps still get the motion made during them; SKIP
 * touches nothing.  lmot_cluster_outputs after an accumulating lmot_frame describes E_acc (intersected with the area).
 * The history starts empty again on the next submitted step after lmot_tracker_reset, _load or _set_ego (or their lmot_seq_ forms),
 * LMOT_SEQ_RESTART, lmot_seq_open, any call to lmot_set_accumulate, lmot_set_sensors or lmot_set_rig_merge (or their lmot_seq_ forms),
 * and, on the context's own stream, after a step whose units differ in number or kind from the previous accumulating step's (for example
 * an lmot_frame after a 2-sensor lmot_batch tick).  Deskew, detection-area and parameter changes keep it.  It holds coordinates: cells
 * are computed at use with the step's roi.
 * Submission.  The setting is host state captured by value at submission; frames in flight keep theirs.  Results depend neither on
 * pipeline_depth nor on host versus device frames: the accumulate launch of frame t waits for frame t-1's on the device (an event across
 * slot streams), so the ground kernels of consecutive frames still overlap and only this launch and the clustering behind it are
 * serialised; one launch covers every accumulating unit of a submission.  An accumulating submission clusters in a launch of its own
 * instead of the ground kernel's tail.  A submission without an accumulating stream runs exactly the launches, copies and memsets it ran
 * before accumulation existed.
 * Errors.  LMOT_ERR_INVALID, setting unchanged: sweeps outside [1, LMOT_MAX_SWEEPS], max_age_s not finite or <= 0, k out of range or
 * no open set.  LMOT_ERR_STATE, nothing submitted: an accumulating submission in timing mode.
 * Memory.  On a stream's first accumulating step, with one device synchronisation, all or nothing: per accumulating unit a ring of
 * sweeps x max_points x 16 B plus one int per entry (64 MB per unit at K = 4 and the default max_points); a larger K or more units later
 * reallocate it the same way.  The setters with sweeps > 1 pin 128 B per result-ring entry (sequences: per ring tick).  Freed with the
 * context; a sequence's with the set (lmot_seq_open, lmot_destroy).
 * lmot_accumulate_info / lmot_seq_accumulate_info: what the most recently RETURNED result of the own stream (lmot_frame*, lmot_batch*) /
 * of sequence k used, per unit in unit order (n_units = 0 when that result did not accumulate): the earlier sweeps in E_acc, |E_acc|
 * before the area mask, and each used sweep's stamp and pose D, newest first.  The counts travel in the result block: no extra
 * synchronisation at collect.
 * lmot_accumulate_pose(fold_s, fold_t, mount, out): step 2 on the host, no device needed; mount NULL: identity. */
#define LMOT_MAX_SWEEPS 8
typedef struct lmot_accumulate {
  int sweeps;                  /* 1 = off (default) .. LMOT_MAX_SWEEPS: this step's cloud plus up to sweeps-1 earlier ones */
  double max_age_s;            /* 0.5: an earlier sweep whose stamp is further back than this is not used */
} lmot_accumulate;
int lmot_default_accumulate(lmot_accumulate* a);
int lmot_set_accumulate(lmot_ctx* ctx, const lmot_accumulate* a);     /* NULL: the defaults (off) */
int lmot_get_accumulate(const lmot_ctx* ctx, lmot_accumulate* a);
typedef struct lmot_accum_info {
  int n_units;
  int sweeps_used[LMOT_MAX_BATCH];                            /* earlier sweeps in E_acc */
  int n_points[LMOT_MAX_BATCH];                               /* |E_acc| (before the area mask) */
  double stamp_us[LMOT_MAX_BATCH][LMOT_MAX_SWEEPS - 1];       /* ts_s of each used sweep, newest first */
  float pose[LMOT_MAX_BATCH][LMOT_MAX_SWEEPS - 1][12];        /* D of each used sweep, row-major 3x4 */
} lmot_accum_info;
int lmot_seq_set_accumulate(lmot_ctx* ctx, int k, const lmot_accumulate* a);
int lmot_seq_get_accumulate(const lmot_ctx* ctx, int k, lmot_accumulate* a);
int lmot_accumulate_info(lmot_ctx* ctx, lmot_accum_info* out);
int lmot_seq_accumulate_info(lmot_ctx* ctx, int k, lmot_accum_info* out);
int lmot_accumulate_pose(const double fold_s[3], const double fold_t[3], const lmot_sensor* mount, float out[12]);

/* ---- box search: fit each cluster's rectangle by a search over yaw with the closeness criterion -------------------------------------
 * boxFitting's fit (getBoundingBox: an L-shape from three points, or cv::minAreaRect on an 18 px/m image) depends on point order and on
 * random draws, and its L-shape is a parallelogram.  A car seen from one corner, the common case, often gets a rotated box.  Box search
 * fits the rectangle that best explains the points over A yaw angles in [0, pi/2) (Zhang et al., "Efficient L-Shape Fitting for Vehicle
 * Detection Using Laser Scanners", IV 2017, closeness criterion).
 *
 * Definition.  A stream (the context's own: lmot_set_box_search; sequence k: lmot_seq_set_box_search) with on = 1 and n_angles = A
 * replaces the fit of each cluster of each detection unit (a frame without a sensor table, an unmerged rig frame, or a merge unit; its
 * cloud is what reaches box fitting: after deskew, the rig merge, accumulation and the detection area).  Clustering, the gather of each
 * cluster's points, maxZ and the rule filter's first test (n >= min_cluster_points) are unchanged.  For a cluster of n points (x_i, y_i):
 *   1. angles: theta_a = (M_PI / 2) * a / A in double, left to right, a = 0 .. A-1; c_a = (float)cos(theta_a), s_a = (float)sin(theta_a)
 *      with the host libm, each rounded to float once.  lmot_box_search_angles returns the table;
 *   2. projections, float, no contraction: u_i = (x_i*c_a) + (y_i*s_a), w_i = (y_i*c_a) - (x_i*s_a); their minima and maxima;
 *   3. closeness, float: d1 = min(u_max - u_i, u_i - u_min), d2 = min(w_max - w_i, w_i - w_min), d = max(min(d1, d2), 0.01f); the
 *      point's score q_i = (uint32)(65536.0f / d) (correctly rounded division, truncated), at most 6,553,600; S_a = sum of q_i in uint64.
 *      Integer sums and min / max do not depend on order, so neither does the fit;
 *   4. a* = argmax S_a, ties to the smallest a;
 *   5. corners in (u, w): P0 = (u_min, w_min), P1 = (u_max, w_min), P2 = (u_max, w_max), P3 = (u_min, w_max), counter-clockwise; in the
 *      unit frame x = (u*c) - (w*s), y = (u*s) + (w*c), float, no contraction;
 *   6. ruleBasedFilter (lmot_rule_filter, both modes) on those corners with the unit's values, maxZ and n; an accepted cluster gives the
 *      usual 8-corner box: bottom z = -(the unit's sensor_height), top z = maxZ.  Boxes are in cluster-id order.
 * Everything behind box fitting runs as usual: concatenation, rig poses, global frame, tracker and retirement.
 *
 * Applies to lmot_frame / _submit / _dev, lmot_detect_dev, lmot_batch* including lmot_batch_detect_dev (every unit, merged or not) and
 * the FRAMES steps of lmot_seq* / lmot_seq_tick*.  Never to the stage entry points (lmot_box_fit stays the reference's boxFitting),
 * lmot_batch_ground_ccl_dev, LISTS steps, lmot_track_step*, lmot_seq_track* or lmot_shared_*.
 * Submission.  The setting is host state captured by value at submission; frames and ticks in flight keep theirs.  lmot_seq_open turns
 * it off for every sequence; lmot_seq_tracker_reset, _load and LMOT_SEQ_RESTART keep it.  A submission without a searching stream runs
 * exactly the launches, copies and memsets it ran before box search existed.
 * Errors.  LMOT_ERR_INVALID, setting unchanged: on not 0 / 1, n_angles outside [1, LMOT_BOX_SEARCH_MAX_ANGLES], k out of range or no
 * open set.  LMOT_ERR_STATE, nothing submitted: a searching submission in timing mode.
 * Memory.  The first setter that turns the search on uploads the angle tables of every A (520 KB of device memory, one synchronous copy),
 * freed with the context. */
#define LMOT_BOX_SEARCH_MAX_ANGLES 360
typedef struct lmot_box_search {
  int on;                      /* 0 (default): boxFitting's fit; 1: the search above */
  int n_angles;                /* A, 90: angle step (pi/2) / A */
} lmot_box_search;
int lmot_default_box_search(lmot_box_search* b);
int lmot_set_box_search(lmot_ctx* ctx, const lmot_box_search* b);          /* NULL: the defaults (off) */
int lmot_get_box_search(const lmot_ctx* ctx, lmot_box_search* b);
int lmot_seq_set_box_search(lmot_ctx* ctx, int k, const lmot_box_search* b);
int lmot_seq_get_box_search(const lmot_ctx* ctx, int k, lmot_box_search* b);
int lmot_box_search_angles(int n_angles, float out[][2]);                  /* step 1 on the host, no device needed: out[a] = (c_a, s_a) */

/* ---- ground lines: slope-following ground removal and box heights from the local ground ---------------------------------------------
 * groundRemove clamps each polar cell's min z into [t_hmin, t_hmax] and boxFitting measures a cluster's height from z = -sensor_height:
 * both assume the ground is the sensor frame's plane z = -sensor_height.  On a grade, under pitch, or with a sensor that is not mounted
 * level, objects uphill are too tall and objects downhill are labelled ground or too short.  Ground lines fit the ground of each of the
 * 80 channels as a chain of straight lines over range, and measure each cluster's height from the line under its lowest point.
 *
 * Definition.  A stream (the context's own: lmot_set_ground_lines; sequence k: lmot_seq_set_ground_lines) with on = 1: each frame of a
 * FRAMES step, with its unit values r_min, r_max, sensor_height and ground_tolerance (lmot_params', or the sequence's detection values; a
 * rig frame takes its sensor's sensor_height):
 *   1. phase 1 of ground removal is unchanged: the pre-filters, each point's polar cell (bit-exact) and minZ per cell (1000: empty);
 *   2. lines per channel: bins b = 0 .. 119 in order; a bin with minZ < 1000 is the prototype (r_b, z_b), r_b = r_min + (b + 0.5) *
 *      (r_max - r_min) / 120, z_b = (double)minZ.  Every operation is double, left to right, without contraction; the unit values are
 *      the float parameters widened to double (lmot_ground_lines_grid reproduces a frame when passed (double)p.r_min etc.).  S = (n, Sr, Sz, Srr,
 *      Srz, Szz) is the open point set; fit(S): den = n*Srr - Sr*Sr, m = (n*Srz - Sr*Sz) / den, c = (Sz - m*Sr) / n,
 *      sse = Szz - 2*m*Srz - 2*c*Sz + m*m*Srr + 2*m*c*Sr + n*c*c.  Closing S appends the line (first bin of S, m, c) of fit(S) if n >= 2,
 *      then empties S.  For each prototype:
 *        extend: if n >= 2, fit S plus the point; if |m| <= max_slope and sse <= n' * max_rmse * max_rmse (n' = n + 1) the point joins S,
 *          else S is closed and the point is a seed;
 *        seed test: with a line of the channel, |z - (m_last*r + c_last)| <= max_step; without one, |z + sensor_height| <= max_slope*r +
 *          max_step; with n == 1 also |z - z0| <= max_slope*(r - r0) ((r0, z0): S's point).  Pass: the point joins S.  Fail with n == 1:
 *          S is emptied and the seed test repeats for the point.  Fail with n == 0: the point is dropped.
 *      After bin 119, S is closed;
 *   3. ground height of a cell: gz(ch, b) = (float)(m*r_b + c) of the channel's last line whose first bin is <= b; none: its first line;
 *      a channel without lines: (float)(-sensor_height).  lmot_ground_lines_grid computes this grid on the host;
 *   4. labels: an in-window point is ground iff (double)z < (double)gz + ground_tolerance, elevated otherwise.  The median and outlier
 *      filters, t_hmin, t_hmax, h_sensor and t_hdiff are not read.  Both clouds keep the input order;
 *   5. box heights: each cluster's lowest point (min z, ties to the first in cloud order) gives g = gz of its polar cell, or
 *      -sensor_height when it lies outside the window.  The rule filter and the box's bottom corners use sensor_height := -g: the cluster
 *      gets what boxFitting gives it with sensorHeight = -g.  This holds for boxFitting's fit and for box search.  A merge unit
 *      (lmot_set_rig_merge) keeps the vehicle's flat sensor_height, because its cloud mixes sensor frames; its sensors' labels still
 *      come from their lines.
 * Applies to lmot_frame / _submit / _dev, lmot_detect_dev, lmot_batch* including lmot_batch_detect_dev, and the FRAMES steps of
 * lmot_seq* / lmot_seq_tick*.  Never to the stage entry points (they stay the reference), lmot_batch_ground_ccl_dev, LISTS steps,
 * lmot_track_step*, lmot_seq_track* or lmot_shared_*.
 * Submission.  Host state captured by value at submission; frames and ticks in flight keep theirs.  lmot_seq_open turns it off for every
 * sequence; lmot_seq_tracker_reset, _load and LMOT_SEQ_RESTART keep it.  A submission without a stream that has lines on runs exactly the
 * launches, copies and memsets it ran before ground lines existed.
 * Errors.  LMOT_ERR_INVALID, setting unchanged: on not 0 / 1, a value not finite, max_slope <= 0, max_rmse <= 0, max_step <= 0, k out of
 * range or no open set.  LMOT_ERR_STATE, nothing submitted: a submission with lines on in timing mode.
 * Memory.  Each detection slot that runs a frame with lines on allocates its 9,600-float ground grid once (38 KB).
 * lmot_debug_ground_lines(ctx, gz, cap_units, n_units): the device grids of the context's most recent own-stream submission, frame by
 * frame (9,600 floats each, cell ch * 120 + b); n_units = 0 when its lines were off.  Synchronises the device. */
typedef struct lmot_ground_lines {
  int on;                      /* 0 (default): groundRemove's polar grid and the flat sensor_height; 1: the lines above */
  double max_slope;            /* 0.3: largest |dz/dr| of a line, and the seed window's slope */
  double max_rmse;             /* 0.08 m: largest root-mean-square residual of a line */
  double max_step;             /* 0.3 m: largest step from the previous line (or the flat ground) to a seed */
} lmot_ground_lines;
int lmot_default_ground_lines(lmot_ground_lines* g);
int lmot_set_ground_lines(lmot_ctx* ctx, const lmot_ground_lines* g);     /* NULL: the defaults (off) */
int lmot_get_ground_lines(const lmot_ctx* ctx, lmot_ground_lines* g);
int lmot_seq_set_ground_lines(lmot_ctx* ctx, int k, const lmot_ground_lines* g);
int lmot_seq_get_ground_lines(const lmot_ctx* ctx, int k, lmot_ground_lines* g);
/* steps 2-3 on the host, no device needed (on is not read): minz[ch * 120 + b] -> gz[ch * 120 + b] */
int lmot_ground_lines_grid(const lmot_ground_lines* g, const float minz[LMOT_NUM_CHANNEL * LMOT_NUM_BIN], double r_min, double r_max,
                           double sensor_height, float gz[LMOT_NUM_CHANNEL * LMOT_NUM_BIN]);
int lmot_debug_ground_lines(lmot_ctx* ctx, float* gz, int cap_units, int* n_units);

/* ---- layered clustering: connected components over height slices ----------------------------------------------------------------------
 * componentClustering projects every elevated point onto the 250 x 250 grid and ignores z, so a car under a tree canopy, a pedestrian
 * under a shelter roof or a car under a sign gantry become one cluster with the structure above them; boxFitting then measures it to the
 * top of the canopy and the rule filter drops it.  Layered clustering labels connected components over (x, y, height slice) instead, so
 * that a vertical gap separates objects.
 *
 * Definition.  A stream (the context's own: lmot_set_layers; sequence k: lmot_seq_set_layers) with on = 1: each detection unit of a
 * FRAMES step (a frame without a sensor table, an unmerged rig frame, or a merge unit) with its cloud E (what reaches clustering: after
 * deskew, the rig merge, accumulation and the detection area), its clustering extent roi and its box-fitting sensor_height (lmot_params',
 * the sequence's own detection value, sensor j's for an unmerged rig frame, the vehicle's for a merge unit):
 *   1. column: the column (xI, yI) of a point is componentClustering's float binning with roi; points outside it have none.  N(x, y) is
 *      the number of points of E in the column;
 *   2. slice: in double, left to right, without contraction, h = ((double)z + (double)sensor_height) - z_min; s = floor(h / slice_m)
 *      clamped to [0, S - 1];
 *   3. seed voxels V = {(x, y, s(p)) : p in E, N(x, y) > 1} (the reference's "more than one point" rule, per column);
 *   4. occupied voxels O: every (x', y', s') inside the grid and inside [0, S) with |x' - x| <= 1, |y' - y| <= 1, |s' - s| <= g for some
 *      (x, y, s) in V;
 *   5. components: the connected parts of O under 26-adjacency (max(|dx|, |dy|, |ds|) = 1), numbered 1.. in the order of each
 *      component's smallest (x, y, s), x outermost; num_cluster is their number;
 *   6. cluster of a point: the id of the component holding (x, y, s(p)); 0 when that voxel is not in O or the point has no column;
 *   7. boxes: box fitting runs as it does without layers on each cluster's points in cloud order -- boxFitting's fit, box search,
 *      ground-line box heights, the rule filter in both modes, max_clusters and LMOT_ERR_CAPACITY -- and everything behind it
 *      (concatenation, poses, global frame, tracker, retirement) is unchanged.
 * With S = 1, step 5 is 8-connected labelling of the 3 x 3 dilation of the seed cells in raster order, i.e. componentClustering: S = 1
 * reproduces the unlayered pipeline bit for bit.  For any S a unit's boxes equal boxFitting(E_c, grid_c, 1) per cluster c (E_c: c's
 * points in cloud order, grid_c: their columns labelled 1), accepted boxes in id order.  Slices are measured from the flat
 * z = -sensor_height also with ground lines on.  Components do not depend on where the slices start except through the clamping at both
 * ends: two seeds closer than 2g + 2 slices join wherever slice 0 lies, unless clamping moves them together.
 * Applies to lmot_frame / _submit / _dev, lmot_detect_dev, lmot_batch* including lmot_batch_detect_dev, and the FRAMES steps of
 * lmot_seq* / lmot_seq_tick*.  Never to the stage entry points (lmot_component_cluster stays the reference), lmot_batch_ground_ccl_dev,
 * LISTS steps, lmot_track_step*, lmot_seq_track* or lmot_shared_*.
 * Submission.  Host state captured by value at submission; frames and ticks in flight keep theirs.  lmot_seq_open turns it off for every
 * sequence; lmot_seq_tracker_reset, _load and LMOT_SEQ_RESTART keep it.  A submission without a layered stream runs exactly the launches,
 * copies and memsets it ran before layered clustering existed.
 * Errors.  LMOT_ERR_INVALID, setting unchanged: on not 0 / 1, n_slices outside [1, LMOT_MAX_SLICES], slice_m not finite or <= 0, z_min
 * not finite, gap_slices outside [0, n_slices - 1], k out of range or no open set.  LMOT_ERR_STATE, nothing submitted: a layered
 * submission in timing mode.  LMOT_ERR_STATE from lmot_cluster_outputs and lmot_debug_label_grid after a layered own-stream frame: the
 * 2-D label grid does not name the layered clusters.
 * Memory.  Each detection slot or merge unit that runs a layered unit allocates, once, its column masks, run tables and a node table for
 * the worst case of 16 runs in each of the 62,500 columns: about 4.8 MB plus one byte per point of max_points.
 * lmot_debug_point_clusters(ctx, ids, cap, n_units, n_points): step 6's id of every point of E of every unit of the context's most recent
 * own-stream submission, unit after unit (n_points[u] points of unit u, in its cloud order); n_units = 0 when it was not layered.
 * LMOT_ERR_CAPACITY (nothing written) when the ids do not fit in cap.  Synchronises the device. */
#define LMOT_MAX_SLICES 32
typedef struct lmot_layers {
  int on;                      /* 0 (default): componentClustering's 2-D grid; 1: layered components (above) */
  int n_slices;                /* S = 32, 1 .. LMOT_MAX_SLICES */
  double slice_m;              /* 0.2: thickness of one slice, metres */
  double z_min;                /* -0.5: bottom of slice 0, metres above the unit's flat ground z = -sensor_height */
  int gap_slices;              /* g = 2, 0 .. S - 1: vertical reach of a seed (seeds with at most 2g empty slices between them join) */
} lmot_layers;
int lmot_default_layers(lmot_layers* l);
int lmot_set_layers(lmot_ctx* ctx, const lmot_layers* l);                  /* NULL: the defaults (off) */
int lmot_get_layers(const lmot_ctx* ctx, lmot_layers* l);
int lmot_seq_set_layers(lmot_ctx* ctx, int k, const lmot_layers* l);
int lmot_seq_get_layers(const lmot_ctx* ctx, int k, lmot_layers* l);
int lmot_debug_point_clusters(lmot_ctx* ctx, int32_t* ids, int cap, int* n_units, int n_points[LMOT_MAX_BATCH]);

/* ---- obstacle footprints: every cluster of a step as a convex polygon with its height range ----------------------------------------
 * Boxes and tracks only ever describe clusters the rule filter accepts (car- and pedestrian-shaped ones).  Trucks, buses, walls, hedges,
 * barriers and clusters below min_cluster_points leave no trace in them.  With obstacles on, every cluster of a step is also reported as
 * geometry, so that a planner sees whatever the filter drops.
 *
 * Definition.  A stream (the context's own: lmot_set_obstacles; sequence k: lmot_seq_set_obstacles) with on = 1: each detection unit of a
 * FRAMES step (a frame without a sensor table, an unmerged rig frame, or a merge unit -- the units of layered clustering and accumulation),
 * numbered from 0 in the step's frame order (a merging rig: its one merge unit):
 *   clusters    the clusters box fitting received for the unit, with their ids 1..K and in id order (K = min(num_cluster, max_clusters)):
 *               the 2-D label grid, the area-masked grid, layered point clusters, E_acc with accumulation, a merge unit's vehicle-frame
 *               cloud.  One obstacle per cluster, including clusters below min_cluster_points and clusters the rule filter rejects;
 *   cells       the clustering cells (u, v) of the unit's grid (u = floor(250 (x + roi/2) / roi) in componentClustering's float
 *               arithmetic, the same for v from y) holding at least one of the cluster's points: the point footprint, not the dilated
 *               label grid;
 *   footprint   the convex hull of every corner (u or u + 1, v or v + 1) of those cells.  Corners are lattice points, so the hull is exact
 *               in integer arithmetic.  Vertices counter-clockwise, starting at the corner with the smallest u, then the smallest v; no
 *               three consecutive vertices collinear; a single cell gives 4.  Vertex (u, v) is reported in metres as
 *               x = (float)((double)u * roi / 250.0 - roi / 2.0), y likewise from v, with the unit's own roi_m (a sequence's
 *               lmot_detect_params, else lmot_params').  The frame is the unit's cloud's: the sensor frame, or the vehicle frame for a
 *               merge unit.  (An unmerged rig frame's boxes are moved into the vehicle frame by its sensor's pose: apply the same pose.)
 *   z_min/max   float min and max of z over the cluster's points in the unit frame;
 *   box         the index, in the unit's own box list (lmot_frame_out.boxes; a batched or sequence unit's share of the concatenated list,
 *               in the unit's order), of the box this cluster produced, or -1 (no box: rejected, or cut by max_boxes).  A consumer that
 *               skips obstacles with box >= 0 never counts one object twice.
 * Vertex count.  No convex lattice polygon in [0, 250]^2 has more than LMOT_OBSTACLE_MAX_HULL = 140 vertices.  Its edge vectors are
 * multiples of distinct primitive vectors (a, b), and sum |a| = 2 width <= 500, sum |b| = 2 height <= 500, so sum (|a| + |b|) <= 1000.
 * There are 4 primitive vectors with |a| + |b| = 1 and 4 phi(m) with |a| + |b| = m >= 2.  Taking them by increasing m, all of m <= 10 cost
 * 868 for 128 vectors, and 132 buys at most 12 of the 40 with m = 11: at most 140 edges.  The bound is reached: all 128 vectors of
 * m <= 10 (width and height 217) plus +-(1,10), +-(10,1), +-(2,9), +-(9,2), +-(3,8), +-(8,3) (33 more each way) close to a polygon of
 * 140 vertices in [0, 250]^2.  No hull is ever truncated.
 * Setting.  lmot_obstacles { on, max_vertices }: max_vertices is each unit's vertex pool, LMOT_OBSTACLE_MAX_HULL .. 1 << 24 (65,536).
 * Vertex offsets run in cluster order; an obstacle whose vertices do not fit whole in the pool keeps its header, and gets the count 0.
 * Retrieval then returns LMOT_ERR_CAPACITY with the needed total in n_vertices, as lmot_cluster_outputs does.
 * Applies to lmot_frame / _submit / _dev, lmot_detect_dev, lmot_batch* and the FRAMES steps of lmot_seq* / lmot_seq_tick*.  Never to the
 * stage entry points (they have lmot_cluster_outputs), lmot_batch_ground_ccl_dev, LISTS steps, lmot_track_step* or lmot_seq_track*.
 * Submission.  Host state captured at submission; steps in flight keep theirs.  lmot_seq_open turns it off for every sequence;
 * lmot_seq_tracker_reset, _load and LMOT_SEQ_RESTART keep it.  A submission without a stream that has obstacles on runs exactly the
 * launches, copies and memsets it ran before obstacles existed.  One launch per submission covers every unit with obstacles on, behind
 * box fitting on the detection stream; its kernel writes the footprints straight into the result's pinned, device-mapped obstacle block.
 * Retrieval.  lmot_obstacles_result(ctx, unit, out) reads the result most recently returned for the own stream (lmot_frame,
 * lmot_frame_collect / _fetch, lmot_batch / _collect / _fetch); lmot_seq_obstacles_result(ctx, k, unit, out) sequence k's step of the
 * tick most recently returned.  They copy out->n_obstacles rows (cap_obstacles) and the pool's first n_vertices x/y pairs (cap_vertices
 * pairs); out->n_units is the step's unit count.  NULL arrays ask for the counts only.
 * Errors.  LMOT_ERR_INVALID, setting unchanged: on not 0 / 1, max_vertices out of range, k out of range or no open set; a unit outside
 * the step's units.  LMOT_ERR_STATE: an obstacle submission in timing mode (nothing submitted); retrieval without a returned result, or for
 * a result submitted with obstacles off (a LISTS step, a skipped sequence).  LMOT_ERR_CAPACITY: the pool overflowed (headers intact), or a
 * caller array is too small (the counts are still returned).
 * Memory.  Each detection slot or merge unit that runs an obstacle unit allocates, once, a hull scratch of (max_clusters + 1) x (4 + 2 x 140)
 * bytes plus 16 bytes (1.2 MB at the default max_clusters).  Each result block that receives one allocates, once per unit count and pool
 * size it needs, units x (32 B x max_clusters + 8 B x max_vertices + 16 B) of pinned host memory (0.64 MB per unit at the defaults);
 * the host keeps one copy of the most recently returned step per stream. */
#define LMOT_OBSTACLE_MAX_HULL 140
typedef struct lmot_obstacles {
  int on;                      /* 0 (default) / 1 */
  int max_vertices;            /* 65536: each unit's vertex pool, LMOT_OBSTACLE_MAX_HULL .. 1 << 24 */
} lmot_obstacles;
typedef struct lmot_obstacle {
  int cluster;                 /* cluster id, 1..K */
  int n_points, n_cells;
  int box;                     /* index in the unit's box list, or -1 */
  int vertex_offset, vertex_count;   /* into the unit's vertex array (pairs); count 0 when the pool overflowed */
  float z_min, z_max;
} lmot_obstacle;
typedef struct lmot_obstacles_out {
  lmot_obstacle* obstacles;    /* nullable, [cap_obstacles] */
  int cap_obstacles;
  float* vertices;             /* nullable, [cap_vertices][2] x, y metres */
  int cap_vertices;
  int n_units;                 /* out: the step's detection units */
  int n_obstacles;             /* out: K of the unit */
  int n_vertices;              /* out: vertices the unit's hulls need in all (pool overflow: more than max_vertices) */
} lmot_obstacles_out;
int lmot_default_obstacles(lmot_obstacles* o);
int lmot_set_obstacles(lmot_ctx* ctx, const lmot_obstacles* o);            /* NULL: the defaults (off) */
int lmot_get_obstacles(const lmot_ctx* ctx, lmot_obstacles* o);
int lmot_seq_set_obstacles(lmot_ctx* ctx, int k, const lmot_obstacles* o);
int lmot_seq_get_obstacles(const lmot_ctx* ctx, int k, lmot_obstacles* o);
int lmot_obstacles_result(lmot_ctx* ctx, int unit, lmot_obstacles_out* out);
int lmot_seq_obstacles_result(lmot_ctx* ctx, int k, int unit, lmot_obstacles_out* out);

/* ---- scan-matched ego motion: a stream's speed and yaw from consecutive sweeps, for rigs without GPS ---------------------------------
 * Every motion-aware part of the library (getOriginPoints' fold, global_frame, deskew, accumulation, the static flag) reads the ego motion
 * a caller passes as v_gps / yaw_gps.  A LiDAR-only rig has none.  The estimator matches each sweep against the previous one and returns
 * (v, yaw) in exactly the form lmot_frame* / lmot_seq* take: call it on a frame, then pass its v and yaw with that frame.  It is a separate,
 * synchronous call: the frame pipeline, the fold and the tracker are not touched by it.
 *
 * Definition.  A stream (the context's own: lmot_set_ego_match; sequence k: lmot_seq_set_ego_match) has the settings below and a matcher
 * state: the previous stamp, the previous frame's likelihood field L, the previous delta (dx, dy, dth), its dt and ok flag, and an
 * accumulated yaw Y.  H = (float)(grid * (double)cell_m * 0.5); float values below are the settings rounded to float once.  One call on
 * frame P with stamp ts:
 *   1. band: point p (moved first, with sensor = j, by sensor j's pose of the stream's table with the rig arithmetic of lmot_set_sensors:
 *      x' = ((r00*x + r01*y) + r02*z) + t0, likewise y', z', float without contraction) is used iff x, y, z are finite, z_min <= z <=
 *      z_max and r_min*r_min <= x*x + y*y <= r_max*r_max, in float without contraction.  Its cell is ((int)floorf((x + H) / cell_m),
 *      (int)floorf((y + H) / cell_m)); it is in the window iff both lie in [0, grid);
 *   2. field: O = the cells holding a window point; L[c] = 3 - min(3, Chebyshev distance from c to O), 0..3.  L becomes the stream's
 *      reference at the end of the call;
 *   3. sample: window points only; sub-cell (min((int)floorf((x + H) / sub_m), NS - 1), likewise y), NS = ceil(grid * cell_m / sub_m) + 1
 *      in double.  The lowest-index point of each occupied sub-cell, sub-cells in raster order (y outer); if more than max_points remain,
 *      every k-th of them from the first, k = ceil(count / max_points).  n_used points (x, y) remain;
 *   4. match, iff the stream has a reference, dt = (ts - ts_prev) / 1e6 is finite and > 0, and n_used >= min_points:
 *      prior: the previous delta times dt / dt_prev (double) if it was ok, else 0.  j0 = llround(prior_th / yaw_step), k0 =
 *      llround(prior_xy / cell_m) per axis (a quotient of 2^20 or more in magnitude: 0).  Coarse level: j in j0 +- yaw_half, kx, ky in k0 +- shift_half; cs = (float)cos(j * yaw_step),
 *      sn = (float)sin(j * yaw_step) in double with the host libm; xr = cs*x - sn*y, yr = sn*x + cs*y in float without contraction, base
 *      cell (bx, by) = floorf((xr + H) / cell_m), floorf((yr + H) / cell_m); score(j, kx, ky) = sum over the points of L_prev[bx + kx,
 *      by + ky], a cell outside the grid scoring 0.  Fine level (refine = R > 1) around the coarse winner (j1, k1): angles
 *      (double)(R*j1 + u) * yaw_step / R, translations t = (float)((double)(R*k1 + a) * cell_m / R) per axis, u, a in [-R, R]; cell =
 *      floorf(((xr + t) + H) / cell_m).  Both levels: the best score wins, ties to the first hypothesis in ascending (j, kx, ky) order
 *      ((u, ax, ay) for the fine one).  (dx, dy, dth) is the winner's lattice value in double: the pose of this frame's origin in the
 *      previous frame.  ok = (double)best >= min_score_frac * 3 * n_used.  Scores are integers: any reduction order gives the same result;
 *   5. outputs: ok: v = (dx*cos(dth) + dy*sin(dth)) / dt (getOriginPoints' own model: the displacement along the new heading), Y += dth.
 *      Not ok with dt valid (no match, or a weak one): the prior is reported as the delta, v and Y from it (constant velocity).  No valid
 *      dt (first call, after a reset, dt <= 0 or not finite): v = 0, dth = 0, ok = 0.  yaw = Y.  In every case the reference, the stamp
 *      and the delta (with its dt and ok) are then replaced.
 * The matched yaw starts at 0: the fold only reads its differences.
 * Settings.  Setting them (also to the same values) resets the stream's matcher state; so do lmot_ego_reset / lmot_seq_ego_reset and
 * lmot_seq_open (every sequence back to the defaults).  LMOT_ERR_INVALID, setting and state unchanged: a value not finite; grid outside
 * [32, 1024] or not a multiple of 32; cell_m outside [0.01, 10]; a window grid * cell_m above 400 m; z_min >= z_max; r_min < 0; r_min >=
 * r_max; r_max > 1000; sub_m <= 0 or NS > 1024; max_points outside [1, 8192]; yaw_step outside (0, 0.1]; yaw_half outside [0, 180];
 * shift_half outside [0, 127]; refine outside [1, 15]; min_points < 1; min_score_frac outside [0, 1]; sensor outside [-1, LMOT_MAX_BATCH);
 * k out of range or no open set.  No device is needed for the validation.
 * Estimation.  lmot_ego_estimate: a HOST frame of n points, stride floats each (>= 3).  lmot_ego_estimate_dev: a DEVICE frame (stride 4),
 * ordered after the caller stream.  lmot_seq_ego_estimate / _dev: one frame per sequence (n_seq entries = the open set's), every sequence
 * whose pointer is non-NULL stepped in one launch per kernel; a NULL entry leaves its sequence's state and out[k] untouched.  The calls run
 * on a matcher stream of the context and wait for their own work only: they never wait for, reorder or change frames and ticks in flight.
 * LMOT_ERR_INVALID: null arguments, n < 0, stride < 3, n_seq not the set's, sensor = j without a j-th sensor in the stream's table
 * (nothing is stepped).  LMOT_ERR_STATE: timing mode (lmot_enable_timing) is on.
 * Memory.  A stream's first call allocates two fields of grid^2 bytes, an occupancy bitmap of grid^2 / 8 bytes, NS^2 ints of sub-cells and
 * max_points x 8 bytes of samples (1.4 MB at the defaults); a later call whose settings need more reallocates them.  Per context: the
 * host-frame staging grows to the largest frame (sum of frames for the sequence form) seen, and the angle tables to (2 yaw_half + 1) +
 * (2 yaw_half refine + 2 refine + 1) float pairs per stream (3 KB at the defaults).  Freed with the context; a sequence's with the set. */
typedef struct lmot_ego_match {
  int grid;                    /* 768 cells per side, 32 .. 1024, a multiple of 32 */
  double cell_m;               /* 0.1 */
  double z_min, z_max;         /* -1.5, 0.5: the height band, stream frame (vehicle frame with sensor >= 0) */
  double r_min, r_max;         /* 3, 38: the range band */
  double sub_m;                /* 0.4: sampling sub-cell */
  int max_points;              /* 4096 */
  double yaw_step;             /* 0.005 rad */
  int yaw_half;                /* 30: coarse angles j0 +- yaw_half */
  int shift_half;              /* 30: coarse shifts k0 +- shift_half cells (+-3 m at the default cell) */
  int refine;                  /* 5: fine level at 1/refine of the coarse lattice; 1: none */
  int min_points;              /* 200: fewer sampled points: no match */
  double min_score_frac;       /* 0.3: ok iff best >= min_score_frac * 3 * n_used */
  int sensor;                  /* -1: the frame as given; j: sensor j's frame of the stream's table, moved into the vehicle frame */
} lmot_ego_match;
typedef struct lmot_ego_out {
  int ok;                      /* the match passed min_score_frac */
  int n_used;                  /* sampled points */
  int n_ref;                   /* occupied cells of the reference the match used (0: no match ran) */
  int score;                   /* the best score (0: no match ran) */
  int score_max;               /* 3 * n_used */
  double dx, dy, dtheta;       /* this frame's origin in the previous frame (m, m, rad) */
  double v;                    /* m/s: pass as v_gps */
  double yaw;                  /* rad, Y: pass as yaw_gps */
} lmot_ego_out;
int lmot_default_ego_match(lmot_ego_match* m);
int lmot_set_ego_match(lmot_ctx* ctx, const lmot_ego_match* m);            /* NULL: the defaults */
int lmot_get_ego_match(const lmot_ctx* ctx, lmot_ego_match* m);
int lmot_seq_set_ego_match(lmot_ctx* ctx, int k, const lmot_ego_match* m);
int lmot_seq_get_ego_match(const lmot_ctx* ctx, int k, lmot_ego_match* m);
int lmot_ego_reset(lmot_ctx* ctx);
int lmot_seq_ego_reset(lmot_ctx* ctx, int k);
int lmot_ego_estimate(lmot_ctx* ctx, const float* points, int n, int stride_floats, double timestamp_us, lmot_ego_out* out);
int lmot_ego_estimate_dev(lmot_ctx* ctx, const float* d_points, int n, double timestamp_us, lmot_ego_out* out);
int lmot_seq_ego_estimate(lmot_ctx* ctx, const float* const* points, const int* n, int n_seq, int stride_floats, const double* timestamp_us,
                          lmot_ego_out* out);
int lmot_seq_ego_estimate_dev(lmot_ctx* ctx, const float* const* d_points, const int* n, int n_seq, const double* timestamp_us,
                              lmot_ego_out* out);

/* ---- tracker state (checkpoint / teacher-forced parity tests) ------------------------------------------ */
int lmot_tracker_reset(lmot_ctx* ctx);
int lmot_tracker_num_tracks(lmot_ctx* ctx, int* n);
/* dumps = double[n*LMOT_TRACK_DUMP_DOUBLES], layout documented in DESIGN.md (same as oracle/ref_harness.cpp) */
int lmot_tracker_dump(lmot_ctx* ctx, double* dumps, int cap, int* n);
int lmot_tracker_load(lmot_ctx* ctx, const double* dumps, int n, int init, double timestamp_us, double ego_velo,
                      double ego_yaw, double ego_pre_yaw, double ego_point_yaw);
/* The frame-level state of getOriginPoints (imm_ukf_jpda.cpp:74-172), i.e. the other half of a checkpoint:
 * ego8 = {init, timestamp_us, egoVelo, egoYaw, egoPreYaw, x, y, yaw of the accumulated dead-reckoning pose}.
 * lmot_tracker_load restarts the dead reckoning at (0, 0, -pi/2) like the test oracle does; call lmot_tracker_set_ego AFTER it to
 * continue a sequence with a moving ego exactly where lmot_tracker_get_ego left it. */
int lmot_tracker_get_ego(lmot_ctx* ctx, double ego8[8]);
int lmot_tracker_set_ego(lmot_ctx* ctx, const double ego8[8]);

/* Device view of the track table for multi-GPU use (several sensor streams feeding ONE tracker, SURVEY.md §8e): the owner
 * rank broadcasts `bytes_per_track * n` bytes from *dev_ptr with NCCL, the other ranks receive into their own table and
 * then call lmot_tracker_set_num_tracks.  The pointer stays valid for the life of the context. */
int lmot_tracker_table(lmot_ctx* ctx, void** dev_ptr, int* bytes_per_track, int* capacity);
int lmot_tracker_set_num_tracks(lmot_ctx* ctx, int n);

/* ---- device-side hand-over for several GPUs feeding ONE tracker (SURVEY.md §8e; host/shared_tracker.cpp uses these with NCCL) ---
 * lmot_detect_boxes_dev      : device pointers to the box list (float[max_boxes*24]) and its length (int) of the most recent
 *                              lmot_detect_dev on this context -- the send buffers of the ncclAllGather
 * lmot_track_step_lists_dev  : n_lists (<= LMOT_MAX_BATCH) padded DEVICE box lists of cap_per_list boxes each, lengths in d_counts,
 *                              concatenated in list order -> ONE immUkfJpdaf step (imm_ukf_jpda.cpp:704), asynchronous on the caller
 *                              stream and ordered after the work already queued on it; results with lmot_frame_fetch
 * lmot_tracker_counters_dev  : device pointer to the number of tracks in the table (the count that travels with the table)
 * lmot_tracker_table_received: after an ncclBroadcast into lmot_tracker_table's pointer (and of the count): the table holds n tracks now */
int lmot_detect_boxes_dev(lmot_ctx* ctx, const float** d_boxes, const int** d_n_boxes);
int lmot_track_step_lists_dev(lmot_ctx* ctx, const float* d_lists, const int* d_counts, int n_lists, int cap_per_list, double timestamp_us,
                              double v_gps, double yaw_gps);
int lmot_tracker_counters_dev(lmot_ctx* ctx, int** d_n_tracks);
int lmot_tracker_table_received(lmot_ctx* ctx, int n);

/* ---- inspection of the last frame's device state (parity tests, debugging) ----------------------------- */
/* polar grid after ground removal: each float[80*120] / uint8[80*120], nullable */
int lmot_debug_polar_grid(lmot_ctx* ctx, float* minz, float* height, float* smoothed, float* hdiff, float* hground,
                          uint8_t* isground);
/* per-point polar cell of the last ground_remove: ch/bin int32[n]; -1/-1 for range-filtered points */
int lmot_debug_cell_index(lmot_ctx* ctx, int32_t* ch, int32_t* bin, int n);
/* label grid and per-elevated-point cluster id of the last clustering / box fitting */
int lmot_debug_label_grid(lmot_ctx* ctx, int32_t* grid, int* num_cluster);

/* host-side self test of the bit-exact atan2f restatement against the host libm (no GPU needed) */
int lmot_selftest_atan2f(const float* y, const float* x, int n, float* out);

/* Per-stage device time of the last lmot_frame / lmot_frame_dev in milliseconds (cudaEvent), for bench.py:
 * ms[0] ground, ms[1] cluster, ms[2] box, ms[3] tracker.  Only recorded after lmot_enable_timing(ctx,1). */
int lmot_enable_timing(lmot_ctx* ctx, int on);
int lmot_last_stage_ms(lmot_ctx* ctx, float ms[4]);
/* finer: device time between consecutive kernels of the last timed frame, in launch order (9 kernels: ground_fused,
 * ccl_bitmap, tile_hist, seg_offsets, scatter, box_fit, imm_predict_gate, imm_update, spawn_output) */
int lmot_last_kernel_ms(lmot_ctx* ctx, float* ms, int cap, int* n);
/* accumulated host-side nanoseconds inside the library: [0] submit (launch calls), [1] collect: waiting for the frame's
 * event, [2] collect: copying results out of the pinned block, [3] number of collects */
int lmot_debug_host_ns(lmot_ctx* ctx, double ns[4], int reset);

#ifdef __cplusplus
}
#endif
#endif /* LMOT_H */
