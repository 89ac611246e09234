// TEST INFRASTRUCTURE ONLY -- plain-C++ restatement ("port") of the reference IMM-UKF-PDA tracker.
//
// Restates /root/reference/object_tracking/tracking/ukf.cpp and tracking/imm_ukf_jpda.cpp with fixed-size
// arrays instead of Eigen::MatrixXd, one function per reference function, each citing the lines it follows.
// It is validated against the reference's own sources (oracle/_ref, tests/test_oracle_port.py) and then serves
// as the checker that travels to the GPU box.  It is never linked into liblmot.so.
//
// Numerics: same operation order as the reference where the reference's order is visible in its source; Eigen's
// internal kernels (gemv blocking, LU solve) are restated in textbook order, which differs from Eigen in the last
// ulp only (tests bound port-vs-reference at 1e-9 relative; the product bar is 1e-4).
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>
#include "port.h"

namespace port {

static const real kPi = M_PI;

// Literal constants and the constant expressions the reference folds at compile time keep their double-rounded values in every
// build; everything the reference computes at run time in double is computed in `real` (port.h).

// ---- small dense helpers ----------------------------------------------------------------------------------
// Eigen dynamic determinant(): partialPivLu().determinant() (OT0/src/Eigen/src/LU/Determinant.h:35-41,
// PartialPivLU.h:245-287): first-max partial pivoting, det = sign * prod(diag) in index order.
static real det_lu(const real* A, int n) {
  real lu[25];
  for (int i = 0; i < n * n; ++i) lu[i] = A[i];
  int sign = 1;
  for (int k = 0; k < n; ++k) {
    int piv = k; real big = std::fabs(lu[k * n + k]);
    for (int r = k + 1; r < n; ++r) { const real v = std::fabs(lu[r * n + k]); if (v > big) { big = v; piv = r; } }
    if (big != 0.0) {
      if (piv != k) { for (int c = 0; c < n; ++c) std::swap(lu[k * n + c], lu[piv * n + c]); sign = -sign; }
      for (int r = k + 1; r < n; ++r) lu[r * n + k] /= lu[k * n + k];
    }
    for (int r = k + 1; r < n; ++r)
      for (int c = k + 1; c < n; ++c) lu[r * n + c] -= lu[r * n + k] * lu[k * n + c];
  }
  real p = lu[0];
  for (int k = 1; k < n; ++k) p *= lu[k * n + k];
  return (real)sign * p;
}

// Eigen dynamic inverse() of a 2x2: partialPivLu().inverse() == solve(Identity) (LU/Inverse.h:22-27)
static void inv2_lu(const real* A, real* R) {
  real a00 = A[0], a01 = A[1], a10 = A[2], a11 = A[3];
  bool swap = std::fabs(a10) > std::fabs(a00);
  if (swap) { std::swap(a00, a10); std::swap(a01, a11); }
  const real l10 = a10 / a00;
  const real u11 = a11 - l10 * a01;
  for (int c = 0; c < 2; ++c) {
    real b0 = (c == 0) ? 1.0 : 0.0, b1 = (c == 1) ? 1.0 : 0.0;
    if (swap) std::swap(b0, b1);
    const real y1 = b1 - l10 * b0;
    const real x1 = y1 / u11;
    const real x0 = (b0 - a01 * x1) / a00;
    R[0 * 2 + c] = x0; R[1 * 2 + c] = x1;
  }
}

// Eigen LLT unblocked, lower (Cholesky/LLT.h:271-295) INCLUDING its early return on a non-positive pivot, which
// leaves the remaining columns unfactored; matrixL() then reads the lower triangle of that partial result and
// the reference never checks info().  L is n x n row-major; strictly-upper part zero.
static void llt_lower_partial(const real* A, int n, real* L) {
  for (int i = 0; i < n * n; ++i) L[i] = A[i];
  for (int k = 0; k < n; ++k) {
    real x = L[k * n + k];
    if (k > 0) { real s = L[k * n + 0] * L[k * n + 0]; for (int j = 1; j < k; ++j) s += L[k * n + j] * L[k * n + j]; x -= s; }
    if (x <= 0.0) break;
    x = std::sqrt(x);
    L[k * n + k] = x;
    for (int r = k + 1; r < n; ++r) {
      real acc = L[r * n + k];
      for (int j = 0; j < k; ++j) acc -= L[r * n + j] * L[k * n + j];
      L[r * n + k] = acc / x;
    }
  }
  for (int r = 0; r < n; ++r) for (int c = r + 1; c < n; ++c) L[r * n + c] = 0.0;
}

static inline void wrap_pi(real& a) {  // the reference's while loops (ukf.cpp:483-488 etc.)
  while (a > kPi) a -= 2. * kPi;
  while (a < -kPi) a += 2. * kPi;
}

// ---- UKF (ukf.cpp) ----------------------------------------------------------------------------------------
static const real kStdA[3] = {2, 2, 3};       // std_a_cv_, std_a_ctrv_, std_a_rm_      ukf.cpp:68-70
static const real kStdYawdd[3] = {2, 2, 3};   // std_cv_yawdd_, std_ctrv_yawdd_, std_rm_yawdd_  :71-73
static const real kStdLas = 0.15;             // std_laspx_/std_laspy_ :91-94
static const real kPmat[3][3] = {{0.9, 0.05, 0.05}, {0.05, 0.9, 0.05}, {0.05, 0.05, 0.9}};  // p1_,p2_,p3_ :144-154

void ukf_initialize(Track& t, real zx, real zy) {  // UKF::UKF ukf.cpp:20-249 + Initialize :257-322
  memset(&t, 0, sizeof(t));
  const real x0[5] = {zx, zy, 0, 0, 0.1};
  for (int m = 0; m < 4; ++m) {
    for (int i = 0; i < 5; ++i) t.x[m][i] = x0[i];
    const real d[5] = {0.5, 0.5, 3, 10, 1};
    for (int i = 0; i < 5; ++i) t.P[m][i * 5 + i] = d[i];
  }
  for (int m = 0; m < 3; ++m) {
    t.modeProb[m] = 0.33;
    t.zPred[m][0] = zx; t.zPred[m][1] = zy;
    t.S[m][0] = 1; t.S[m][3] = 1;
  }
}

// MixingProbability ukf.cpp:439-455 + Interaction :458-500.  Index 1..3 of x/P = cv, ctrv, rm (0 = merge).
static void mixing_interaction(Track& t) {
  real mu[3][3];  // mu[i][j] = modeMatchProb i->j
  for (int j = 0; j < 3; ++j) {
    const real sum = t.modeProb[0] * kPmat[0][j] + t.modeProb[1] * kPmat[1][j] + t.modeProb[2] * kPmat[2][j];
    for (int i = 0; i < 3; ++i) mu[i][j] = t.modeProb[i] * kPmat[i][j] / sum;
  }
  real xp[3][5], Pp[3][25];
  for (int i = 0; i < 3; ++i) { memcpy(xp[i], t.x[i + 1], sizeof(xp[i])); memcpy(Pp[i], t.P[i + 1], sizeof(Pp[i])); }
  for (int j = 0; j < 3; ++j) {
    real* x = t.x[j + 1];
    for (int e = 0; e < 5; ++e) x[e] = mu[0][j] * xp[0][e] + mu[1][j] * xp[1][e] + mu[2][j] * xp[2][e];
    x[3] = xp[j][3];  // yaw is not mixed (:471-473)
    wrap_pi(x[3]);
  }
  for (int j = 0; j < 3; ++j) {
    const real* x = t.x[j + 1];
    real* P = t.P[j + 1];
    for (int r = 0; r < 5; ++r)
      for (int c = 0; c < 5; ++c) {
        real acc = 0;
        for (int i = 0; i < 3; ++i) {
          const real term = mu[i][j] * (Pp[i][r * 5 + c] + (xp[i][r] - x[r]) * (xp[i][c] - x[c]));
          acc = (i == 0) ? term : acc + term;
        }
        P[r * 5 + c] = acc;
      }
  }
}

// Cv :564-588, Ctrv :539-563, randomMotion :589-606
static void motion(int model, const real* a, real dt, real* s) {
  const real p_x = a[0], p_y = a[1], v = a[2], yaw = a[3], yawd = a[4], nu_a = a[5], nu_yawdd = a[6];
  if (model == 2) { s[0] = p_x; s[1] = p_y; s[2] = v; s[3] = yaw; s[4] = yawd; return; }
  real px_p, py_p, yaw_p;
  if (model == 0) {
    px_p = p_x + v * std::cos(yaw) * dt;
    py_p = p_y + v * std::sin(yaw) * dt;
    yaw_p = yaw;
  } else {
    if (std::fabs(yawd) > 0.001) {
      px_p = p_x + v / yawd * (std::sin(yaw + yawd * dt) - std::sin(yaw));
      py_p = p_y + v / yawd * (std::cos(yaw) - std::cos(yaw + yawd * dt));
    } else {
      px_p = p_x + v * dt * std::cos(yaw);
      py_p = p_y + v * dt * std::sin(yaw);
    }
    yaw_p = yaw + yawd * dt;
  }
  real v_p = v, yawd_p = yawd;
  px_p = px_p + 0.5 * nu_a * dt * dt * std::cos(yaw);
  py_p = py_p + 0.5 * nu_a * dt * dt * std::sin(yaw);
  v_p = v_p + nu_a * dt;
  yaw_p = yaw_p + 0.5 * nu_yawdd * dt * dt;
  yawd_p = yawd_p + nu_yawdd * dt;
  s[0] = px_p; s[1] = py_p; s[2] = v_p; s[3] = yaw_p; s[4] = yawd_p;
}

static const real kLambdaAug = 3 - 7;  // lambda_aug_ = 3 - n_aug_ (:104-113)

// Prediction ukf.cpp:630-772 followed by UpdateLidar :778-902 for one model
static void predict_update(Track& t, int model, real dt) {
  real* x = t.x[model + 1];
  real* P = t.P[model + 1];
  real w[15];
  w[0] = kLambdaAug / (kLambdaAug + 7);
  for (int i = 1; i < 15; ++i) w[i] = 0.5 / (7 + kLambdaAug);
  // augmentation (:667-680)
  real x_aug[7], P_aug[49], L[49];
  for (int i = 0; i < 5; ++i) x_aug[i] = x[i];
  x_aug[5] = 0; x_aug[6] = 0;
  for (int i = 0; i < 49; ++i) P_aug[i] = 0;
  for (int r = 0; r < 5; ++r) for (int c = 0; c < 5; ++c) P_aug[r * 7 + c] = P[r * 5 + c];
  P_aug[5 * 7 + 5] = kStdA[model] * kStdA[model];
  P_aug[6 * 7 + 6] = kStdYawdd[model] * kStdYawdd[model];
  llt_lower_partial(P_aug, 7, L);
  real Xa[15][7];
  const real sq = std::sqrt(kLambdaAug + 7);
  for (int e = 0; e < 7; ++e) Xa[0][e] = x_aug[e];
  for (int i = 0; i < 7; ++i)
    for (int e = 0; e < 7; ++e) {
      Xa[i + 1][e] = x_aug[e] + sq * L[e * 7 + i];
      Xa[i + 8][e] = x_aug[e] - sq * L[e * 7 + i];
    }
  real Xs[15][5];
  for (int i = 0; i < 15; ++i) motion(model, Xa[i], dt, Xs[i]);
  // predicted mean / covariance (:737-755)
  for (int e = 0; e < 5; ++e) x[e] = 0;
  for (int i = 0; i < 15; ++i) for (int e = 0; e < 5; ++e) x[e] = x[e] + w[i] * Xs[i][e];
  wrap_pi(x[3]);
  for (int e = 0; e < 25; ++e) P[e] = 0;
  for (int i = 0; i < 15; ++i) {
    real d[5];
    for (int e = 0; e < 5; ++e) d[e] = Xs[i][e] - x[e];
    wrap_pi(d[3]);
    for (int r = 0; r < 5; ++r) for (int c = 0; c < 5; ++c) P[r * 5 + c] = P[r * 5 + c] + (w[i] * d[r]) * d[c];
  }
  // UpdateLidar (:805-870): measurement = (px, py)
  real zp[2] = {0, 0};
  for (int i = 0; i < 15; ++i) { zp[0] = zp[0] + w[i] * Xs[i][0]; zp[1] = zp[1] + w[i] * Xs[i][1]; }
  real S[4] = {0, 0, 0, 0};
  for (int i = 0; i < 15; ++i) {
    const real dz[2] = {Xs[i][0] - zp[0], Xs[i][1] - zp[1]};
    for (int r = 0; r < 2; ++r) for (int c = 0; c < 2; ++c) S[r * 2 + c] = S[r * 2 + c] + (w[i] * dz[r]) * dz[c];
  }
  S[0] = S[0] + kStdLas * kStdLas; S[1] = S[1] + 0; S[2] = S[2] + 0; S[3] = S[3] + kStdLas * kStdLas;
  real Tc[10];
  for (int e = 0; e < 10; ++e) Tc[e] = 0;
  for (int i = 0; i < 15; ++i) {
    const real dz[2] = {Xs[i][0] - zp[0], Xs[i][1] - zp[1]};
    for (int r = 0; r < 5; ++r) {
      const real xd = Xs[i][r] - x[r];
      for (int c = 0; c < 2; ++c) Tc[r * 2 + c] = Tc[r * 2 + c] + (w[i] * xd) * dz[c];
    }
  }
  real Si[4];
  inv2_lu(S, Si);
  for (int r = 0; r < 5; ++r)
    for (int c = 0; c < 2; ++c) t.K[model][r * 2 + c] = Tc[r * 2 + 0] * Si[0 * 2 + c] + Tc[r * 2 + 1] * Si[1 * 2 + c];
  t.zPred[model][0] = zp[0]; t.zPred[model][1] = zp[1];
  for (int e = 0; e < 4; ++e) t.S[model][e] = S[e];
}

static void process_imm_ukf(Track& t, real dt) {  // ProcessIMMUKF ukf.cpp:507-527
  mixing_interaction(t);
  for (int m = 0; m < 3; ++m) predict_update(t, m, dt);
}

// PostProcessIMMUKF :529-535 = UpdateModeProb :384-397 + MergeEstimationAndCovariance :419-437 (+UpdateYawWithHighProb :399-417)
static void post_process(Track& t, const real lam[3]) {
  real* mp = t.modeProb;
  const real sum = lam[0] * mp[0] + lam[1] * mp[1] + lam[2] * mp[2];
  mp[0] = (lam[0] * mp[0]) / sum; mp[1] = (lam[1] * mp[1]) / sum; mp[2] = (lam[2] * mp[2]) / sum;
  for (int m = 0; m < 3; ++m) if (std::fabs(mp[m]) < 0.0001) mp[m] = 0.0001;
  real* xm = t.x[0];
  for (int e = 0; e < 5; ++e) xm[e] = mp[0] * t.x[1][e] + mp[1] * t.x[2][e] + mp[2] * t.x[3][e];
  wrap_pi(xm[3]);
  if (mp[0] > mp[1]) t.x_merge_yaw = (mp[0] > mp[2]) ? t.x[1][3] : t.x[3][3];
  else               t.x_merge_yaw = (mp[1] > mp[2]) ? t.x[2][3] : t.x[3][3];
  xm[3] = t.x_merge_yaw;
  for (int r = 0; r < 5; ++r)
    for (int c = 0; c < 5; ++c) {
      real acc = 0;
      for (int m = 0; m < 3; ++m) {
        const real term = mp[m] * (t.P[m + 1][r * 5 + c] + (t.x[m + 1][r] - xm[r]) * (t.x[m + 1][c] - xm[c]));
        acc = (m == 0) ? term : acc + term;
      }
      t.P[0][r * 5 + c] = acc;
    }
}

// ---- imm_ukf_jpda.cpp ---------------------------------------------------------------------------------------
static const real gammaG = 9.22, pG = 0.99, pD = 0.9;      // :26-34
static const real distanceThres = 99; static const int lifeTimeThres = 3; static const real bbYawChangeThres = 0.2;  // :38-51

static int find_max_model(const Track& t) {   // findMaxZandS :176-203 (model index with the max det(S))
  const real cv = det_lu(t.S[0], 2), ctrv = det_lu(t.S[1], 2), rm = det_lu(t.S[2], 2);
  if (cv > ctrv) return (cv > rm) ? 0 : 2;
  return (ctrv > rm) ? 1 : 2;
}

struct Meas { real x, y; };
struct BBoxMeas { real v[10]; };

// getCpFromBbox :465-479 (float arithmetic inside S1/S2, real afterwards)
static void cp_from_bbox(const float b[][3], real& cx, real& cy) {
  const float p1x = b[0][0], p1y = b[0][1], p2x = b[1][0], p2y = b[1][1], p3x = b[2][0], p3y = b[2][1], p4x = b[3][0], p4y = b[3][1];
  const real S1 = ((p4x - p2x) * (p1y - p2y) - (p4y - p2y) * (p1x - p2x)) / 2;
  const real S2 = ((p4x - p2x) * (p2y - p3y) - (p4y - p2y) * (p2x - p3x)) / 2;
  cx = p1x + (p3x - p1x) * S1 / (S1 + S2);
  cy = p1y + (p3y - p1y) * S1 / (S1 + S2);
}

static real bbox_area(const float b[][3]) {   // getBboxArea :482-494 (abs(float))
  const float p1x = b[0][0], p1y = b[0][1], p2x = b[1][0], p2y = b[1][1], p3x = b[2][0], p3y = b[2][1], p4x = b[3][0], p4y = b[3][1];
  const real tri1 = 0.5 * std::fabs((float)((p1x - p3x) * (p2y - p3y) - (p2x - p3x) * (p1y - p3y)));
  const real tri2 = 0.5 * std::fabs((float)((p1x - p4x) * (p3y - p4y) - (p3x - p4x) * (p1y - p4y)));
  return tri1 + tri2;
}

static real bbox_yaw(const Track& t) {        // getBBoxYaw :535-563 (float sqrt / atan2f)
  const float p1x = t.BBox[0][0], p1y = t.BBox[0][1], p2x = t.BBox[1][0], p2y = t.BBox[1][1], p3x = t.BBox[2][0], p3y = t.BBox[2][1];
  const real dist1 = sqrtf((p1x - p2x) * (p1x - p2x) + (p1y - p2y) * (p1y - p2y));
  const real dist2 = sqrtf((p3x - p2x) * (p3x - p2x) + (p3y - p2y) * (p3y - p2y));
  real yaw;
  if (dist1 > dist2) yaw = atan2f(p1y - p2y, p1x - p2x);
  else yaw = atan2f(p3y - p2y, p3x - p2x);
  const real ukfYaw = t.x[0][3];
  const real diffYaw = std::fabs(yaw - ukfYaw);
  if (diffYaw < kPi * 0.5) return yaw;
  yaw += kPi;
  wrap_pi(yaw);
  return yaw;
}

static void update_box_yaw(Track& t, real cpx, real cpy, real dyaw, bool isVis) {   // updateBoxYaw :512-532
  float (*bb)[3] = isVis ? t.BBox : t.bestBBox;
  const int n = isVis ? t.nBBox : t.nBest;   // the reference loops over BBox_.size() and indexes either box
  (void)n;
  for (int i = 0; i < t.nBBox; ++i) {
    const real preX = bb[i][0], preY = bb[i][1];
    bb[i][0] = (float)(std::cos(dyaw) * (preX - cpx) - std::sin(dyaw) * (preY - cpy) + cpx);
    bb[i][1] = (float)(std::sin(dyaw) * (preX - cpx) + std::cos(dyaw) * (preY - cpy) + cpy);
  }
}

static void update_bb(Track& t) {   // updateBB :565-653
  if (!t.isVisBB) return;
  if (t.nBest == 0) {
    memcpy(t.bestBBox, t.BBox, sizeof(t.BBox)); t.nBest = t.nBBox;
    t.bestYaw = bbox_yaw(t);
    return;
  }
  real cpx, cpy, bcx, bcy;
  cp_from_bbox(t.BBox, cpx, cpy);
  cp_from_bbox(t.bestBBox, bcx, bcy);
  const real dtx = cpx - bcx, dty = cpy - bcy;
  const real yaw = bbox_yaw(t);
  const real area = bbox_area(t.BBox), bestArea = bbox_area(t.bestBBox);
  const real deltaArea = area - bestArea;
  if (deltaArea < 0) {   // updateVisBoxArea :496-510
    for (int i = 0; i < t.nBBox; ++i) {
      t.BBox[i][0] = (float)(t.bestBBox[i][0] + dtx);
      t.BBox[i][1] = (float)(t.bestBBox[i][1] + dty);
    }
  } else if (deltaArea > 0) {
    memcpy(t.bestBBox, t.BBox, sizeof(t.BBox)); t.nBest = t.nBBox;
  }
  const real currentYaw = bbox_yaw(t);
  const real DiffYaw = yaw - currentYaw;
  if (std::fabs(DiffYaw) > bbYawChangeThres) {
  } else if (std::fabs(DiffYaw) < bbYawChangeThres) {
    update_box_yaw(t, cpx, cpy, DiffYaw, true);
    update_box_yaw(t, cpx, cpy, DiffYaw, false);
    t.bestYaw = yaw;
  }
}

// associateBB :416-463 + getNearestEuclidBBox :396-413 (int minDist!)
static void associate_bb(int trackNum, const std::vector<BBoxMeas>& bboxVec, Track& t) {
  if (bboxVec.empty()) return;
  if (trackNum == 5 && t.lifetime > lifeTimeThres) {
    int minDist = 999, minInd = 0;
    const real px = t.x[0][0], py = t.x[0][1];
    for (size_t i = 0; i < bboxVec.size(); ++i) {
      const real mx = bboxVec[i].v[0], my = bboxVec[i].v[1];
      const real dist = std::sqrt((px - mx) * (px - mx) + (py - my) * (py - my));
      if (dist < minDist) { minDist = (int)dist; minInd = (int)i; }
    }
    if (minDist < distanceThres) {
      const real* nb = bboxVec[minInd].v;
      for (int i = 0; i < 2; ++i) {
        const real height = (i == 0) ? -1.73 : 0;
        for (int c = 0; c < 4; ++c) {
          t.BBox[i * 4 + c][0] = (float)nb[2 + 2 * c];
          t.BBox[i * 4 + c][1] = (float)nb[3 + 2 * c];
          t.BBox[i * 4 + c][2] = (float)height;
        }
      }
      t.nBBox = 8;
      t.isVisBB = true;
    }
  }
}

// measurementValidation :205-257
static void measurement_validation(const std::vector<std::vector<real>>& trackPoints, Track& t, bool secondInit, const real maxDetZ[2],
                                   const real maxDetS[4], std::vector<Meas>& measVec, std::vector<BBoxMeas>& bboxVec, std::vector<int>& matchingVec) {
  bool secondInitDone = false;
  real smallestNIS = 999;
  Meas smallest = {0, 0};
  real Si[4];
  for (size_t i = 0; i < trackPoints.size(); ++i) {
    const real x = trackPoints[i][0], y = trackPoints[i][1];
    const real d0 = x - maxDetZ[0], d1 = y - maxDetZ[1];
    inv2_lu(maxDetS, Si);
    const real nis = (d0 * Si[0] + d1 * Si[2]) * d0 + (d0 * Si[1] + d1 * Si[3]) * d1;
    if (nis < gammaG) {
      if (matchingVec[i] == 0) t.lifetime++;
      if (secondInit) {
        if (nis < smallestNIS) { smallestNIS = nis; smallest.x = x; smallest.y = y; matchingVec[i] = 1; secondInitDone = true; }
      } else {
        Meas m = {x, y}; measVec.push_back(m);
        BBoxMeas b; for (int k = 0; k < 10; ++k) b.v[k] = trackPoints[i][k];
        bboxVec.push_back(b);
        matchingVec[i] = 1;
      }
    }
  }
  if (secondInitDone) measVec.push_back(smallest);
}

// filterPDA :259-394
static void filter_pda(Track& t, const std::vector<Meas>& measVec, real lam[3]) {
  const real numMeas = (real)measVec.size();
  const real b = 2 * numMeas * (1 - pD * pG) / (gammaG * pD);
  real eSum[3] = {0, 0, 0};
  std::vector<real> e[3];
  std::vector<Meas> diff[3];
  real Si[3][4];
  for (int m = 0; m < 3; ++m) inv2_lu(t.S[m], Si[m]);
  for (size_t i = 0; i < measVec.size(); ++i)
    for (int m = 0; m < 3; ++m) {
      Meas d = {measVec[i].x - t.zPred[m][0], measVec[i].y - t.zPred[m][1]};
      diff[m].push_back(d);
      const real t0 = -0.5 * d.x, t1 = -0.5 * d.y;
      const real q = (t0 * Si[m][0] + t1 * Si[m][2]) * d.x + (t0 * Si[m][1] + t1 * Si[m][3]) * d.y;
      const real ev = std::exp(q);
      e[m].push_back(ev);
      eSum[m] += ev;
    }
  real betaZero[3];
  for (int m = 0; m < 3; ++m) betaZero[m] = b / (b + eSum[m]);
  real Vk;
  for (int m = 0; m < 3; ++m) {
    real sx[2] = {0, 0};
    std::vector<real> beta(measVec.size());
    for (size_t i = 0; i < measVec.size(); ++i) beta[i] = e[m][i] / (b + eSum[m]);
    for (size_t i = 0; i < measVec.size(); ++i) { sx[0] += beta[i] * diff[m][i].x; sx[1] += beta[i] * diff[m][i].y; }
    real sP[4] = {0, 0, 0, 0};
    for (size_t i = 0; i < measVec.size(); ++i) {
      const real d[2] = {diff[m][i].x, diff[m][i].y};
      for (int r = 0; r < 2; ++r) for (int c = 0; c < 2; ++c) sP[r * 2 + c] += ((beta[i] * d[r]) * d[c] - sx[r] * sx[c]);
    }
    real* x = t.x[m + 1];
    real* P = t.P[m + 1];
    const real* K = t.K[m];
    const real* S = t.S[m];
    for (int r = 0; r < 5; ++r) x[r] = x[r] + (K[r * 2] * sx[0] + K[r * 2 + 1] * sx[1]);
    wrap_pi(x[3]);
    // K S K^T and K sigmaP K^T
    real KS[10], KSK[25], KP[10], KPK[25];
    for (int r = 0; r < 5; ++r) for (int c = 0; c < 2; ++c) { KS[r * 2 + c] = K[r * 2] * S[c] + K[r * 2 + 1] * S[2 + c]; KP[r * 2 + c] = K[r * 2] * sP[c] + K[r * 2 + 1] * sP[2 + c]; }
    for (int r = 0; r < 5; ++r) for (int c = 0; c < 5; ++c) { KSK[r * 5 + c] = KS[r * 2] * K[c * 2] + KS[r * 2 + 1] * K[c * 2 + 1]; KPK[r * 5 + c] = KP[r * 2] * K[c * 2] + KP[r * 2 + 1] * K[c * 2 + 1]; }
    if (numMeas != 0) {
      for (int e2 = 0; e2 < 25; ++e2) P[e2] = betaZero[m] * P[e2] + (1 - betaZero[m]) * (P[e2] - KSK[e2]) + KPK[e2];
    } else {
      for (int e2 = 0; e2 < 25; ++e2) P[e2] = P[e2] - KSK[e2];
    }
  }
  const int mm = find_max_model(t);
  Vk = kPi * std::sqrt(gammaG * det_lu(t.S[mm], 2));
  for (int m = 0; m < 3; ++m) {
    if (numMeas != 0)
      lam[m] = (1 - pG * pD) / std::pow(Vk, numMeas) + pD * std::pow(Vk, 1 - numMeas) * eSum[m] / (numMeas * std::sqrt(2 * kPi * det_lu(t.S[m], 2)));
    else
      lam[m] = (1 - pG * pD) / std::pow(Vk, numMeas);
  }
}

static real intersect_coef(real v1x, real v1y, real v2x, real v2y, real px, real py, real cpx, real cpy) {  // :655-661
  return (((v1x - v2x) * (py - v1y) + (v1y - v2y) * (v1x - px)) * ((v1x - v2x) * (cpy - v1y) + (v1y - v2y) * (v1x - cpx)));
}

static void merge_over_segmentation(Tracker& T) {   // mergeOverSegmentation :666-700
  const size_t n = T.targets.size();
  for (size_t i = 0; i < n; ++i) {
    const Track& a = T.targets[i];
    if (!a.isVisBB) continue;
    const real v1x = a.BBox[0][0], v1y = a.BBox[0][1], v2x = a.BBox[1][0], v2y = a.BBox[1][1];
    const real v3x = a.BBox[2][0], v3y = a.BBox[2][1], v4x = a.BBox[3][0], v4y = a.BBox[3][1];
    const real cp1x = (v1x + v2x + v3x) / 3, cp1y = (v1y + v2y + v3y) / 3;
    const real cp2x = (v1x + v4x + v3x) / 3, cp2y = (v1y + v4y + v3y) / 3;
    for (size_t j = 0; j < n; ++j) {
      if (i == j) continue;
      const real px = T.targets[j].x[0][0], py = T.targets[j].x[0][1];
      const real c1 = intersect_coef(v1x, v1y, v2x, v2y, px, py, cp1x, cp1y);
      const real c2 = intersect_coef(v1x, v1y, v3x, v3y, px, py, cp1x, cp1y);
      const real c3 = intersect_coef(v3x, v3y, v2x, v2y, px, py, cp1x, cp1y);
      const real c4 = intersect_coef(v1x, v1y, v4x, v4y, px, py, cp2x, cp2y);
      const real c5 = intersect_coef(v1x, v1y, v3x, v3y, px, py, cp2x, cp2y);
      const real c6 = intersect_coef(v3x, v3y, v4x, v4y, px, py, cp2x, cp2y);
      if ((c1 > 0 && c2 > 0 && c3 > 0) || (c4 > 0 && c5 > 0 && c6 > 0)) { T.trackNum[i] = 5; T.trackNum[j] = 0; }
    }
  }
}

// getOriginPoints :74-172 -- the O(#frames) replay is a fold, restated incrementally (bit-identical: each step
// of the replay only uses the previous (x, y, egoYaw) and the i-th delta)
void get_origin_points(Tracker& T, double timestamp, double v_gps, double yaw_gps) {
  const real firstEgoYawOffset = (double)(-0.63035 - M_PI / 2);   // :70, a double global initialised by a constant expression
  const real dt = (timestamp - T.timestamp) / 1000000.0;
  T.egoVelo = v_gps;
  T.egoYaw = yaw_gps;
  T.egoYaw += firstEgoYawOffset;
  if (!T.init) {
    T.egoPoint[0] = 0; T.egoPoint[1] = 0; T.egoPoint[2] = T.egoYaw;
    T.fold[0] = 0; T.fold[1] = 0; T.fold[2] = -kPi / 2;
    return;
  }
  const real diffYaw = T.egoYaw - T.egoPreYaw;
  const real dX = dt * T.egoVelo * std::cos(diffYaw), dY = dt * T.egoVelo * std::sin(diffYaw);
  real x = T.fold[0], y = T.fold[1], egoYaw = T.fold[2];
  x -= dX; y -= dY;
  const real preX = x, preY = y;
  const real yaw = diffYaw * -1;
  egoYaw += yaw;
  x = std::cos(yaw) * preX - std::sin(yaw) * preY;
  y = std::sin(yaw) * preX + std::cos(yaw) * preY;
  T.fold[0] = x; T.fold[1] = y; T.fold[2] = egoYaw;
  T.egoPoint[0] = x; T.egoPoint[1] = y; T.egoPoint[2] = egoYaw;
}

// immUkfJpdaf :704-1112
void imm_ukf_jpdaf(Tracker& T, const float* boxes, int nb, double timestamp, StepOut& out) {
  std::vector<std::vector<real>> trackPoints;
  for (int i = 0; i < nb; ++i) {
    const float (*b)[3] = reinterpret_cast<const float (*)[3]>(boxes + (size_t)i * 24);
    real cx, cy;
    cp_from_bbox(b, cx, cy);
    std::vector<real> p;
    p.push_back(cx); p.push_back(cy);
    for (int c = 0; c < 4; ++c) { p.push_back(b[c][0]); p.push_back(b[c][1]); }
    trackPoints.push_back(p);
  }
  out.clear();
  if (!T.init) {   // :741-795
    for (size_t i = 0; i < trackPoints.size(); ++i) {
      if (i == 1) {
        const real px = -1.5125, py = -8.975;
        out.targets.push_back((float)px); out.targets.push_back((float)py); out.targets.push_back((float)(-1.73 / 2));
        out.vandyaw.push_back(0); out.vandyaw.push_back(0);
        out.is_static.push_back(0); out.is_vis.push_back(0);
        Track t; ukf_initialize(t, px, py);
        T.targets.push_back(t); T.trackNum.push_back(1);
      }
    }
    T.timestamp = timestamp;
    T.egoPreYaw = T.egoYaw;
    out.track_manage = T.trackNum;
    T.init = true;
    return;
  }
  std::vector<int> matchingVec(trackPoints.size());
  const real dt = (timestamp - T.timestamp) / 1000000.0;
  T.timestamp = timestamp;
  for (size_t i = 0; i < T.targets.size(); ++i) {   // :812-961
    Track& t = T.targets[i];
    t.isVisBB = false;
    if (T.trackNum[i] == 0) continue;
    if (det_lu(t.P[0], 5) > 10 || t.P[0][4 * 5 + 4] > 1000) { T.trackNum[i] = 0; continue; }
    std::vector<Meas> measVec; std::vector<BBoxMeas> bboxVec;
    real lam[3];
    process_imm_ukf(t, dt);
    const int mm = find_max_model(t);
    real maxDetZ[2] = {t.zPred[mm][0], t.zPred[mm][1]};
    real maxDetS[4];
    for (int e = 0; e < 4; ++e) maxDetS[e] = t.S[mm][e] * 4;
    const real detS = det_lu(maxDetS, 2);
    if (std::isnan(detS) || detS > 10) { T.trackNum[i] = 0; continue; }
    const bool secondInit = (T.trackNum[i] == 1);
    measurement_validation(trackPoints, t, secondInit, maxDetZ, maxDetS, measVec, bboxVec, matchingVec);
    associate_bb(T.trackNum[i], bboxVec, t);
    update_bb(t);
    if (secondInit) {   // :882-921
      if (measVec.size() == 0) { T.trackNum[i] = 0; continue; }
      t.initMeas[0] = t.x[0][0]; t.initMeas[1] = t.x[0][1];
      const real targetX = measVec[0].x, targetY = measVec[0].y;
      const real dX = targetX - t.x[0][0], dY = targetY - t.x[0][1];
      real targetYaw = std::atan2(dY, dX);
      const real targetV = 2;
      wrap_pi(targetYaw);
      for (int m = 0; m < 4; ++m) { t.x[m][0] = targetX; t.x[m][1] = targetY; t.x[m][2] = targetV; t.x[m][3] = targetYaw; }
      T.trackNum[i]++;
      continue;
    }
    int& tn = T.trackNum[i];   // :924-944
    if (measVec.size() > 0) {
      if (tn < 3) tn++;
      else if (tn == 3) tn = 5;
      else if (tn >= 5) tn = 5;
    } else {
      if (tn < 5) tn = 0;
      else if (tn >= 5 && tn < 10) tn++;
      else if ((tn = 10)) tn = 0;   // the reference's `=`-for-`==` at :941
    }
    if (tn == 0) continue;
    filter_pda(t, measVec, lam);
    post_process(t, lam);
    t.velo[t.nVelo++] = t.x[0][2];   // velo_history_ :955-959 (keeps the last three)
    if (t.nVelo == 4) { t.velo[0] = t.velo[1]; t.velo[1] = t.velo[2]; t.velo[2] = t.velo[3]; t.nVelo = 3; }
  }
  merge_over_segmentation(T);   // :968
  for (size_t i = 0; i < matchingVec.size(); ++i) {   // :972-989
    if (matchingVec[i] == 0) {
      Track t; ukf_initialize(t, trackPoints[i][0], trackPoints[i][1]);
      T.targets.push_back(t); T.trackNum.push_back(1);
    }
  }
  for (size_t i = 0; i < T.targets.size(); ++i) {   // :995-1041
    Track& t = T.targets[i];
    const real tx = t.x[0][0], ty = t.x[0][1];
    const real mx = t.initMeas[0], my = t.initMeas[1];
    t.distFromInit = std::sqrt((tx - mx) * (tx - mx) + (ty - my) * (ty - my));
    real tyaw = t.x[0][3];
    tyaw += T.egoPoint[2];
    wrap_pi(tyaw);
    out.targets.push_back((float)tx); out.targets.push_back((float)ty); out.targets.push_back((float)(-1.73 / 2));
    out.vandyaw.push_back(t.x[0][2]); out.vandyaw.push_back(tyaw);
    out.is_static.push_back(0);
    out.is_vis.push_back(t.isVisBB ? 1 : 0);
    if (t.isVisBB) for (int p = 0; p < 8; ++p) for (int c = 0; c < 3; ++c) out.vis_bb.push_back(t.BBox[p][c]);
  }
  for (size_t i = 0; i < T.trackNum.size(); ++i) {   // :1045-1081
    Track& t = T.targets[i];
    if (t.isStatic) { out.is_static[i] = 1; continue; }
    if (T.trackNum[i] == 5 && t.lifetime > 8) {
      const real distThres = 3.0;
      if ((t.distFromInit < distThres) && (t.modeProb[2] > t.modeProb[0] || t.modeProb[2] > t.modeProb[1])) {
        out.is_static[i] = 1; t.isStatic = true;
      }
    }
  }
  out.track_manage = T.trackNum;
  T.egoPreYaw = T.egoYaw;
}

// oracle/ref_predict.cpp's ref_tracker_predict for one row: immUkfJpdaf's guards (:826-848) and ProcessIMMUKF(dt), findMaxZandS,
// PostProcessIMMUKF({1, 1, 1}) on a copy of the row.  The table is not written.
int predict_track(const Tracker& T, int i, double t_us, real* x, real* P, real* mode_prob, real* gate_z, real* gate_S) {
  const Track& src = T.targets[i];
  if (T.trackNum[i] == 0) return 2;
  if (det_lu(src.P[0], 5) > 10 || src.P[0][4 * 5 + 4] > 1000) return 4;
  Track u = src;
  const real dt = (t_us - T.timestamp) / 1000000.0;
  process_imm_ukf(u, dt);
  const int mm = find_max_model(u);
  real S4[4];
  for (int e = 0; e < 4; ++e) S4[e] = u.S[mm][e] * 4;
  const real detS = det_lu(S4, 2);
  const real ones[3] = {1, 1, 1};
  post_process(u, ones);
  for (int e = 0; e < 5; ++e) x[e] = u.x[0][e];
  for (int e = 0; e < 25; ++e) P[e] = u.P[0][e];
  for (int m = 0; m < 3; ++m) mode_prob[m] = u.modeProb[m];
  for (int e = 0; e < 2; ++e) gate_z[e] = u.zPred[mm][e];
  for (int e = 0; e < 4; ++e) gate_S[e] = u.S[mm][e];
  return 1 | ((std::isnan(detS) || detS > 10) ? 8 : 0);
}

}  // namespace port
