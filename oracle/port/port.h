// TEST INFRASTRUCTURE ONLY -- shared declarations of the plain-C++ restatement (oracle/port/*.cpp).
#pragma once
#include <cstdint>
#include <vector>

// The tracker's floating type: every value the reference keeps in double.  double by default; the extended-precision build
// (-DPORT_REAL="long double", oracle/liboracle_port_hp.so) evaluates the same operations, in the same order and with the same
// double-rounded literal constants, with a 64-bit mantissa -- an oracle whose own error is far below the reference's.  Values the
// reference keeps in float (box corners, getBBoxYaw's atan2f) stay float in both builds.
#ifndef PORT_REAL
#define PORT_REAL double
#endif

namespace port {

typedef PORT_REAL real;

// one track == one UKF object of the reference (ukf.h:15-263); x/P index 0 = merge, 1 = cv, 2 = ctrv, 3 = rm
struct Track {
  real x[4][5];
  real P[4][25];
  real modeProb[3];
  real zPred[3][2];
  real S[3][4];
  real K[3][10];
  int lifetime;
  bool isStatic, isVisBB;
  float BBox[8][3]; int nBBox;
  float bestBBox[8][3]; int nBest;
  real bestYaw, bb_yaw, bb_area;
  real initMeas[2];
  real distFromInit;
  real x_merge_yaw;
  real velo[4]; int nVelo;
};

// file-scope globals of imm_ukf_jpda.cpp:19-24,56-58,66-70
struct Tracker {
  std::vector<Track> targets;
  std::vector<int> trackNum;
  bool init = false;
  real timestamp = 0, egoVelo = 0, egoYaw = 0, egoPreYaw = 0;
  real egoPoint[3] = {0, 0, 0};   // egoPoints_[0]
  real fold[3] = {0, 0, -1.5707963267948966};  // running (x, y, egoYaw) of getOriginPoints' replay
};

struct StepOut {
  std::vector<float> targets; std::vector<real> vandyaw; std::vector<int> track_manage;
  std::vector<uint8_t> is_static, is_vis; std::vector<float> vis_bb;
  void clear() { targets.clear(); vandyaw.clear(); track_manage.clear(); is_static.clear(); is_vis.clear(); vis_bb.clear(); }
};

struct GridDump { float *minz, *height, *smoothed, *hdiff, *hground; uint8_t* isground; };
void cell_index(float x, float y, int& chI, int& binI);
void ground_remove(const float* xyz, int n, int stride, std::vector<float>& elev, std::vector<float>& ground, GridDump* dump);
void component_clustering(const float* xyz, int n, int stride, int* grid, int& numCluster);
void box_fitting(const float* xyz, int n, int stride, const int* grid, int numCluster, int mode, std::vector<float>& boxes,
                 std::vector<float>& markers);
void ukf_initialize(Track& t, real zx, real zy);
void get_origin_points(Tracker& T, double timestamp, double v_gps, double yaw_gps);
void imm_ukf_jpdaf(Tracker& T, const float* boxes, int nb, double timestamp, StepOut& out);
// ref_tracker_predict (oracle/ref_predict.cpp) for row i at time t_us: flag 2 dead, 4 P guard, else 1 | (8 if the S guard fails);
// x [5], P [25], mode_prob [3], gate_z [2], gate_S [4] are written only when flag has bit 1.
int predict_track(const Tracker& T, int i, double t_us, real* x, real* P, real* mode_prob, real* gate_z, real* gate_S);

}  // namespace port
