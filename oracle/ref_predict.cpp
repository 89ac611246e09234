// TEST INFRASTRUCTURE ONLY -- track prediction on the reference's own track table (lmot_predict_tracks' oracle).
//
// Built by oracle/predict.mk into oracle/_ref/libref_predict_<mode>.so, one per reference library (intended, tunable), each linked
// against its libref_<mode>.so: loaded after that library, it resolves targets_ / trackNumVec_ / timestamp_ to the SAME instance the
// harness (ref_harness.cpp) steps.  No algorithm of the reference is restated here: every row is predicted on a COPY of its UKF by the
// reference's own functions -- ProcessIMMUKF(dt), findMaxZandS, PostProcessIMMUKF({1, 1, 1}) -- and the guards are immUkfJpdaf's
// expressions (imm_ukf_jpda.cpp:826-848).  The reference's table is never written.
#include <cmath>
#include <limits>
#include <vector>
#include "ukf.h"

// the track table and the stamp of the last step: externally linked globals of imm_ukf_jpda.cpp:20,57-58
extern std::vector<UKF> targets_;
extern std::vector<int> trackNumVec_;
extern double timestamp_;
void findMaxZandS(UKF target, Eigen::VectorXd& maxDetZ, Eigen::MatrixXd& maxDetS);   // imm_ukf_jpda.cpp:176

extern "C" {

// rows of the table at the n_t query times t_us (us): the outputs of include/lmot.h's track prediction in its layout -- track_manage
// [cap]; flags [n_t][cap] (1 valid, 2 dead, 4 P guard, 8 S guard); x [n_t][cap][5]; P [n_t][cap][25] row-major; mode_prob [n_t][cap][3];
// gate_z [n_t][cap][2]; gate_S [n_t][cap][4] row-major (before the x4).  Rows beyond cap are not written.  Returns the row count.
int ref_tracker_predict(const double* t_us, int n_t, int cap, int* track_manage, unsigned char* flags, double* x, double* P, double* mode_prob,
                        double* gate_z, double* gate_S) {
  const int n = (int)targets_.size();
  const int m = n < cap ? n : cap;
  const double nan = std::numeric_limits<double>::quiet_NaN();
  for (int i = 0; i < m; ++i) {
    track_manage[i] = trackNumVec_[i];
    int flag = 0;
    if (trackNumVec_[i] == 0) flag = 2;                                                                  // :826
    else if (targets_[i].P_merge_.determinant() > 10 || targets_[i].P_merge_(4, 4) > 1000) flag = 4;    // :828
    for (int j = 0; j < n_t; ++j) {
      const size_t row = (size_t)j * cap + i;
      for (int e = 0; e < 5; ++e) x[row * 5 + e] = nan;
      for (int e = 0; e < 25; ++e) P[row * 25 + e] = nan;
      for (int e = 0; e < 3; ++e) mode_prob[row * 3 + e] = nan;
      for (int e = 0; e < 2; ++e) gate_z[row * 2 + e] = nan;
      for (int e = 0; e < 4; ++e) gate_S[row * 4 + e] = nan;
      flags[row] = (unsigned char)flag;
      if (flag) continue;
      UKF u = targets_[i];
      const double dt = (t_us[j] - timestamp_) / 1000000.0;                                              // :807
      u.ProcessIMMUKF(dt);
      Eigen::VectorXd maxDetZ;
      Eigen::MatrixXd maxDetS;
      findMaxZandS(u, maxDetZ, maxDetS);
      const Eigen::MatrixXd S4 = maxDetS * 4;                                                            // :844-848
      const double detS = S4.determinant();
      u.PostProcessIMMUKF(std::vector<double>{1, 1, 1});
      flags[row] = (unsigned char)(1 | ((std::isnan(detS) || detS > 10) ? 8 : 0));
      for (int e = 0; e < 5; ++e) x[row * 5 + e] = u.x_merge_(e);
      for (int r = 0; r < 5; ++r) for (int c = 0; c < 5; ++c) P[row * 25 + r * 5 + c] = u.P_merge_(r, c);
      mode_prob[row * 3] = u.modeProbCV_; mode_prob[row * 3 + 1] = u.modeProbCTRV_; mode_prob[row * 3 + 2] = u.modeProbRM_;
      for (int e = 0; e < 2; ++e) gate_z[row * 2 + e] = maxDetZ(e);
      for (int r = 0; r < 2; ++r) for (int c = 0; c < 2; ++c) gate_S[row * 4 + r * 2 + c] = maxDetS(r, c);
    }
  }
  return n;
}

}  // extern "C"
