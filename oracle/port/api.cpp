// TEST INFRASTRUCTURE ONLY -- C ABI of the plain-C++ restatement, same signatures as oracle/ref_harness.cpp
// (prefix port_ instead of ref_) so tests can swap one oracle for the other.  Inputs are double (the reference's values, exact in
// any wider type); what the reference computes in double -- the dump row, vandyaw, the prediction -- is returned as port::real.
#include <cstring>
#include <limits>
#include "port.h"

using namespace port;

static Tracker g_T;

enum { D_TRACKNUM = 0, D_LIFETIME = 1, D_STATIC = 2, D_VIS = 3, D_X = 4, D_P = 24, D_MODE = 124, D_ZPRED = 127, D_S = 133,
       D_K = 145, D_BESTYAW = 175, D_BBYAW = 176, D_BBAREA = 177, D_DISTINIT = 178, D_XMERGEYAW = 179, D_INITMEAS = 180,
       D_VELON = 182, D_VELO = 183, D_BBN = 186, D_BB = 187, D_BESTBBN = 211, D_BESTBB = 212, D_TOTAL = 236 };

static int g_rule_mode = 0;

extern "C" {

void port_set_rule_mode(int mode) { g_rule_mode = mode; }
int port_real_digits() { return std::numeric_limits<real>::digits; }   // mantissa bits of port::real: 53, or 64 for long double

void port_cell_index(const float* xy, int n, int stride, int* ch, int* bin) {
  for (int i = 0; i < n; ++i) cell_index(xy[(size_t)i * stride], xy[(size_t)i * stride + 1], ch[i], bin[i]);
}

void port_ground_remove(const float* xyz, int n, int stride, float* elev, int* n_elev, float* ground, int* n_ground) {
  std::vector<float> e, g;
  ground_remove(xyz, n, stride, e, g, nullptr);
  *n_elev = (int)e.size() / 3; *n_ground = (int)g.size() / 3;
  memcpy(elev, e.data(), e.size() * sizeof(float)); memcpy(ground, g.data(), g.size() * sizeof(float));
}

void port_polar_grid(const float* xyz, int n, int stride, float* minz, float* height, float* smoothed, float* hdiff,
                     float* hground, uint8_t* isground) {
  std::vector<float> e, g;
  GridDump d{minz, height, smoothed, hdiff, hground, isground};
  ground_remove(xyz, n, stride, e, g, &d);
}

void port_component_clustering(const float* xyz, int n, int stride, int32_t* grid, int* num_cluster) {
  int nc = 0;
  component_clustering(xyz, n, stride, grid, nc);
  *num_cluster = nc;
}

void port_box_fitting(const float* xyz, int n, int stride, const int32_t* grid, int num_cluster, int max_boxes, float* boxes,
                      int* n_boxes, float* markers) {
  std::vector<float> b, m;
  box_fitting(xyz, n, stride, grid, num_cluster, g_rule_mode, b, m);
  const int nb = (int)b.size() / 24;
  *n_boxes = nb;
  const int nc = nb < max_boxes ? nb : max_boxes;
  memcpy(boxes, b.data(), (size_t)nc * 24 * sizeof(float));
  if (markers) memcpy(markers, m.data(), (size_t)nc * 6 * sizeof(float));
}

void port_tracker_reset() { g_T = Tracker(); }
int port_tracker_num_tracks() { return (int)g_T.targets.size(); }

void port_tracker_step(const float* boxes, int m, double timestamp, double v_gps, double yaw_gps, int cap, float* targets,
                       real* vandyaw, int* track_manage, uint8_t* is_static, uint8_t* is_vis, float* vis_bb, int* n_vis,
                       int* n_tracks_out) {
  get_origin_points(g_T, timestamp, v_gps, yaw_gps);
  StepOut o;
  imm_ukf_jpdaf(g_T, boxes, m, timestamp, o);
  const int T = (int)o.track_manage.size();
  *n_tracks_out = T; *n_vis = (int)o.vis_bb.size() / 24;
  for (int i = 0; i < T && i < cap; ++i) {
    if (3 * i + 2 < (int)o.targets.size()) { targets[3*i] = o.targets[3*i]; targets[3*i+1] = o.targets[3*i+1]; targets[3*i+2] = o.targets[3*i+2]; }
    if (2 * i + 1 < (int)o.vandyaw.size()) { vandyaw[2*i] = o.vandyaw[2*i]; vandyaw[2*i+1] = o.vandyaw[2*i+1]; }
    track_manage[i] = o.track_manage[i];
    is_static[i] = i < (int)o.is_static.size() ? o.is_static[i] : 0;
    is_vis[i] = i < (int)o.is_vis.size() ? o.is_vis[i] : 0;
  }
  for (size_t k = 0; k < o.vis_bb.size() && k < (size_t)cap * 24; ++k) vis_bb[k] = o.vis_bb[k];
}

void port_tracker_dump(int i, real* d) {
  for (int k = 0; k < D_TOTAL; ++k) d[k] = 0;
  const Track& t = g_T.targets[i];
  d[D_TRACKNUM] = g_T.trackNum[i]; d[D_LIFETIME] = t.lifetime; d[D_STATIC] = t.isStatic; d[D_VIS] = t.isVisBB;
  for (int m = 0; m < 4; ++m) { memcpy(d + D_X + 5 * m, t.x[m], 5 * sizeof(real)); memcpy(d + D_P + 25 * m, t.P[m], 25 * sizeof(real)); }
  for (int m = 0; m < 3; ++m) {
    d[D_MODE + m] = t.modeProb[m]; d[D_ZPRED + 2 * m] = t.zPred[m][0]; d[D_ZPRED + 2 * m + 1] = t.zPred[m][1];
    memcpy(d + D_S + 4 * m, t.S[m], 4 * sizeof(real)); memcpy(d + D_K + 10 * m, t.K[m], 10 * sizeof(real));
  }
  d[D_BESTYAW] = t.bestYaw; d[D_BBYAW] = t.bb_yaw; d[D_BBAREA] = t.bb_area; d[D_DISTINIT] = t.distFromInit; d[D_XMERGEYAW] = t.x_merge_yaw;
  d[D_INITMEAS] = t.initMeas[0]; d[D_INITMEAS + 1] = t.initMeas[1];
  d[D_VELON] = t.nVelo; for (int k = 0; k < t.nVelo && k < 3; ++k) d[D_VELO + k] = t.velo[k];
  d[D_BBN] = t.nBBox; for (int p = 0; p < t.nBBox; ++p) for (int c = 0; c < 3; ++c) d[D_BB + 3 * p + c] = t.BBox[p][c];
  d[D_BESTBBN] = t.nBest; for (int p = 0; p < t.nBest; ++p) for (int c = 0; c < 3; ++c) d[D_BESTBB + 3 * p + c] = t.bestBBox[p][c];
}

void port_tracker_load(int n_tracks, const double* dumps, int init, double timestamp, double ego_velo, double ego_yaw,
                       double ego_pre_yaw, double ego_point_yaw) {
  g_T = Tracker();
  for (int i = 0; i < n_tracks; ++i) {
    const double* d = dumps + (size_t)i * D_TOTAL;
    Track t; memset(&t, 0, sizeof(t));
    t.lifetime = (int)d[D_LIFETIME]; t.isStatic = d[D_STATIC] != 0; t.isVisBB = d[D_VIS] != 0;
    for (int m = 0; m < 4; ++m) {
      for (int e = 0; e < 5; ++e) t.x[m][e] = d[D_X + 5 * m + e];
      for (int e = 0; e < 25; ++e) t.P[m][e] = d[D_P + 25 * m + e];
    }
    for (int m = 0; m < 3; ++m) {
      t.modeProb[m] = d[D_MODE + m]; t.zPred[m][0] = d[D_ZPRED + 2 * m]; t.zPred[m][1] = d[D_ZPRED + 2 * m + 1];
      for (int e = 0; e < 4; ++e) t.S[m][e] = d[D_S + 4 * m + e];
      for (int e = 0; e < 10; ++e) t.K[m][e] = d[D_K + 10 * m + e];
    }
    t.bestYaw = d[D_BESTYAW]; t.bb_yaw = d[D_BBYAW]; t.bb_area = d[D_BBAREA]; t.distFromInit = d[D_DISTINIT]; t.x_merge_yaw = d[D_XMERGEYAW];
    t.initMeas[0] = d[D_INITMEAS]; t.initMeas[1] = d[D_INITMEAS + 1];
    t.nVelo = (int)d[D_VELON]; for (int k = 0; k < t.nVelo && k < 3; ++k) t.velo[k] = d[D_VELO + k];
    t.nBBox = (int)d[D_BBN]; for (int p = 0; p < t.nBBox; ++p) for (int c = 0; c < 3; ++c) t.BBox[p][c] = (float)d[D_BB + 3 * p + c];
    t.nBest = (int)d[D_BESTBBN]; for (int p = 0; p < t.nBest; ++p) for (int c = 0; c < 3; ++c) t.bestBBox[p][c] = (float)d[D_BESTBB + 3 * p + c];
    g_T.targets.push_back(t); g_T.trackNum.push_back((int)d[D_TRACKNUM]);
  }
  g_T.init = init != 0; g_T.timestamp = timestamp; g_T.egoVelo = ego_velo; g_T.egoYaw = ego_yaw; g_T.egoPreYaw = ego_pre_yaw;
  g_T.egoPoint[0] = 0; g_T.egoPoint[1] = 0; g_T.egoPoint[2] = ego_point_yaw;
  g_T.fold[0] = 0; g_T.fold[1] = 0; g_T.fold[2] = -1.5707963267948966;
}

// ref_tracker_predict's signature and semantics (oracle/ref_predict.cpp), on the port's table
int port_tracker_predict(const double* t_us, int n_t, int cap, int* track_manage, unsigned char* flags, real* x, real* P, real* mode_prob,
                         real* gate_z, real* gate_S) {
  const int n = (int)g_T.targets.size();
  const int m = n < cap ? n : cap;
  const real nan = std::numeric_limits<real>::quiet_NaN();
  for (int i = 0; i < m; ++i) {
    track_manage[i] = g_T.trackNum[i];
    for (int j = 0; j < n_t; ++j) {
      const size_t row = (size_t)j * cap + i;
      for (int e = 0; e < 5; ++e) x[row * 5 + e] = nan;
      for (int e = 0; e < 25; ++e) P[row * 25 + e] = nan;
      for (int e = 0; e < 3; ++e) mode_prob[row * 3 + e] = nan;
      for (int e = 0; e < 2; ++e) gate_z[row * 2 + e] = nan;
      for (int e = 0; e < 4; ++e) gate_S[row * 4 + e] = nan;
      flags[row] = (unsigned char)predict_track(g_T, i, t_us[j], x + row * 5, P + row * 25, mode_prob + row * 3, gate_z + row * 2,
                                                gate_S + row * 4);
    }
  }
  return n;
}

}  // extern "C"
