// frame_loop.cpp -- the per-frame loop a deployment runs around the C ABI (include/lmot.h), in the reference's host language.
//
// The reference's nodes are C++ callbacks that call groundRemove / componentClustering / boxFitting / immUkfJpdaf once per
// PointCloud2 message (src/groundremove/main.cpp:91-136, src/cluster/main.cpp:63-234, tracking/main.cpp:65-390).  This is
// the same loop over lmot_frame_submit / lmot_frame_collect with HOST buffers: every frame is copied host -> device from
// pinned memory inside lmot_frame_submit, and every frame's boxes and track outputs are read back by lmot_frame_collect.
// bench.py times its `e2e` figure with this binary (a Python loop around the same two calls adds interpreter and ctypes time
// to every frame).
//
// usage: frame_loop <frames.bin> <n_frames> <n_points> <warmup> <steps> [dt_us=100000] [windows=1] [in_flight=0]
//   frames.bin: n_frames x n_points x 4 float32 (XYZI).  n_frames >= warmup + windows * steps.
//   windows: the timed region (K steps, lmot_sync on both sides) is repeated that many times on consecutive frames;
//   in_flight: frames the host submits ahead of the results it has read back (0: 2 x pipeline_depth, at most result_ring - 1).
// prints one JSON line: wall time of every timed window, frames collected, host time inside submit / collect, per-frame latency
// (submit call -> its results copied out) percentiles, result sizes.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "lmot.h"

static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

int main(int argc, char** argv) {
  if (argc < 6) { fprintf(stderr, "usage: %s frames.bin n_frames n_points warmup steps [dt_us]\n", argv[0]); return 2; }
  const int nf = atoi(argv[2]), np = atoi(argv[3]), W = atoi(argv[4]), K = atoi(argv[5]);
  const double dt_us = argc > 6 ? atof(argv[6]) : 100000.0;
  const int R = argc > 7 ? std::max(1, atoi(argv[7])) : 1;
  const int want_depth = argc > 8 ? atoi(argv[8]) : 0;
  if (nf < W + R * K || np <= 0) { fprintf(stderr, "need n_frames >= warmup + windows * steps\n"); return 2; }
  const size_t frame_floats = (size_t)np * 4;
  float* frames = (float*)lmot_pinned_alloc((size_t)nf * frame_floats * sizeof(float));
  if (!frames) { fprintf(stderr, "pinned allocation failed (no CUDA device?)\n"); return 3; }
  FILE* fi = fopen(argv[1], "rb");
  if (!fi || fread(frames, sizeof(float), (size_t)nf * frame_floats, fi) != (size_t)nf * frame_floats) { fprintf(stderr, "cannot read %s\n", argv[1]); return 3; }
  fclose(fi);

  lmot_params prm;
  lmot_default_params(&prm);
  lmot_ctx* ctx = nullptr;
  int rc = lmot_create(&ctx, &prm, 0);
  if (rc) { fprintf(stderr, "lmot_create: %s\n", lmot_strerror(rc)); return 4; }

  const int cap = prm.max_tracks;
  std::vector<float> boxes((size_t)prm.max_boxes * 24), targets((size_t)cap * 3), visbb((size_t)cap * 24);
  std::vector<double> vandyaw((size_t)cap * 2);
  std::vector<int32_t> manage(cap);
  std::vector<uint8_t> is_static(cap), is_vis(cap);
  lmot_frame_out out;
  memset(&out, 0, sizeof(out));
  out.boxes = boxes.data(); out.max_boxes = prm.max_boxes;
  out.tracks.cap = cap; out.tracks.targets = targets.data(); out.tracks.vandyaw = vandyaw.data(); out.tracks.track_manage = manage.data();
  out.tracks.is_static = is_static.data(); out.tracks.is_vis = is_vis.data(); out.tracks.vis_bb = visbb.data();

  for (int i = 0; i < W; ++i)
    if ((rc = lmot_frame(ctx, frames + (size_t)i * frame_floats, np, 4, (i + 1) * dt_us, 0.0, 0.0, &out)) < 0) { fprintf(stderr, "lmot_frame: %s (%s)\n", lmot_strerror(rc), lmot_last_error(ctx)); return 5; }
  lmot_sync(ctx);

  int depth = want_depth > 0 ? want_depth : 2 * prm.pipeline_depth;       // frames the host may be ahead of the results it has read back
  if (depth > prm.result_ring - 1) depth = prm.result_ring - 1;
  int collected = 0;
  double t_submit = 0, t_collect = 0;
  long long sum_tracks = 0, sum_boxes = 0;
  std::vector<double> window_s(R), t_sub((size_t)R * K), lat;
  lat.reserve((size_t)R * K);
  for (int r = 0; r < R; ++r) {
    int in_flight = 0, next_done = W + r * K;
    lmot_sync(ctx);
    const double t0 = now_s();
    for (int i = W + r * K; i < W + (r + 1) * K; ++i) {
      if (in_flight == depth) {
        const double a = now_s();
        if ((rc = lmot_frame_collect(ctx, &out)) < 0) { fprintf(stderr, "collect: %s (%s)\n", lmot_strerror(rc), lmot_last_error(ctx)); return 6; }
        const double b = now_s();
        t_collect += b - a; ++collected; --in_flight; sum_tracks += out.tracks.n_tracks; sum_boxes += out.n_boxes;
        lat.push_back(b - t_sub[next_done - W]); ++next_done;
      }
      const double a = now_s();
      t_sub[i - W] = a;
      if ((rc = lmot_frame_submit(ctx, frames + (size_t)i * frame_floats, np, 4, (i + 1) * dt_us, 0.0, 0.0)) < 0) { fprintf(stderr, "submit: %s (%s)\n", lmot_strerror(rc), lmot_last_error(ctx)); return 6; }
      t_submit += now_s() - a; ++in_flight;
    }
    while (in_flight > 0) {
      const double a = now_s();
      if ((rc = lmot_frame_collect(ctx, &out)) < 0) { fprintf(stderr, "collect: %s (%s)\n", lmot_strerror(rc), lmot_last_error(ctx)); return 6; }
      const double b = now_s();
      t_collect += b - a; ++collected; --in_flight; sum_tracks += out.tracks.n_tracks; sum_boxes += out.n_boxes;
      lat.push_back(b - t_sub[next_done - W]); ++next_done;
    }
    lmot_sync(ctx);
    window_s[r] = now_s() - t0;
  }
  std::vector<double> ws = window_s;
  std::sort(ws.begin(), ws.end());
  const double e2e_s = ws[(R - 1) / 2];          // median window (lower median for even R)
  std::sort(lat.begin(), lat.end());
  const double lat_p50 = lat[lat.size() / 2], lat_p99 = lat[std::min(lat.size() - 1, (size_t)(0.99 * lat.size()))];
  int live = 0;
  for (int i = 0; i < out.tracks.n_tracks; ++i) live += manage[i] > 0;
  const long long d2h = 16 * 4 + (long long)out.n_boxes * 96 + (long long)out.tracks.n_tracks * (12 + 16 + 4 + 1 + 1) + (long long)out.tracks.n_vis * 96;
  printf("{\"e2e_s\": %.9f, \"windows\": %d, \"window_s\": [", e2e_s, R);
  for (int r = 0; r < R; ++r) printf("%s%.9f", r ? ", " : "", window_s[r]);
  printf("], \"frames\": %d, \"submit_us_per_frame\": %.3f, \"collect_us_per_frame\": %.3f, \"latency_us_p50\": %.2f, \"latency_us_p99\": %.2f, "
         "\"in_flight\": %d, \"tracks_last\": %d, "
         "\"live_tracks_last\": %d, \"boxes_last\": %d, \"vis_last\": %d, \"d2h_bytes_last\": %lld, \"sum_tracks\": %lld, \"sum_boxes\": %lld, "
         "\"h2d_bytes_per_frame\": %zu, \"pipeline_depth\": %d, \"result_ring\": %d}\n",
         collected, 1e6 * t_submit / ((double)R * K), 1e6 * t_collect / ((double)R * K), 1e6 * lat_p50, 1e6 * lat_p99, depth, out.tracks.n_tracks, live, out.n_boxes,
         out.tracks.n_vis, d2h, sum_tracks, sum_boxes, frame_floats * sizeof(float), prm.pipeline_depth, prm.result_ring);
  lmot_destroy(ctx);
  lmot_pinned_free(frames);
  return collected == R * K ? 0 : 7;
}
