// tracker.cu -- batched IMM-UKF-PDA tracker on sm_90a.
//
// Replaces immUkfJpdaf (/root/reference/object_tracking/tracking/imm_ukf_jpda.cpp:704-1112) and class UKF
// (tracking/ukf.cpp).  The reference walks its tracks sequentially; the only cross-track couplings are
//   (a) the shared matchingVec / lifetime_ bookkeeping of measurementValidation (:205-257),
//   (b) mergeOverSegmentation (:666-700), a last-writer-wins double loop, and
//   (c) append-order spawning of new tracks (:972-989),
// all deterministic functions of per-(track, box) predicates, so tracks run in parallel:
//
//   G  tracker_gate_kernel      one warp: waits (on the device) for this frame's detection stages, then lets TA's CTAs come.
//   TA imm_predict_gate_kernel  one CTA per active track, 3 warps = motion models CV/CTRV/RM: explosion guards (:826-831),
//                               IMM mixing + interaction (ukf.cpp:439-500), 7-dim augmented sigma points with Eigen's
//                               early-exit Cholesky (lane = sigma point), model propagation, weighted mean /
//                               covariance (lane = matrix element), lidar S / K (ukf.cpp:778-902); then the chi-square
//                               gate of every box against the max-det(S) model (:843-869) -> gate / setter bit
//                               rows, first_setter[box] = min track index (atomicMin), compact list of gated centres.
//   TB imm_update_kernel        one CTA per active track: warps 0-2 the PDA update of one model each (:259-394), warp 3
//                               lifetime_, measurement list, box association (:416-463), updateBB (:565-653), secondInit
//                               (:882-921); then warp 0: association likelihoods, track-number machine (:924-944), IMM
//                               mode-probability update and merge (ukf.cpp:384-437); 128-byte summary for TC.
//   TC spawn_output_kernel      one CTA: mergeOverSegmentation as "the last write of the reference's (i,j) loop" over
//                               (live x visible) and (visible x all) pairs, then spawn a UKF per unmatched box in box
//                               order, per-track outputs, static flag.  Fast path (<= 256 active tracks) from TB's
//                               summaries, general path from the records.
//   P  publish_kernel           device result block -> pinned host block, on its own stream (polls TC's step counter).
// G -> TA -> TB -> TC are programmatic dependent launches of one another (griddepcontrol); in steady state the tracker
// stream carries nothing else (DESIGN.md section 6).
//
// Each stage has one kernel per family, all from the stage's one body; chain_launch picks the family for a step of 1..8 tables:
//   the kernels above        the context's own table at the default parameters, not numbering its tracks (lmot_frame*, lmot_batch*,
//                            lmot_track_step*, lmot_shared_*);
//   *_seq_kernel             a sequence tick whose tables are all of that kind: one table per blockIdx.y (TA, TB) / blockIdx.x (TC);
//   *_seq_tuned_kernel       every other step, the own table's included (S = 1): each table's own parameters (DESIGN.md section 6c),
//                            and a TC whose track-retirement phase is on for each table that numbers its tracks (section 6e).
//
// All state is fp64 like the reference (Eigen::MatrixXd); this file is compiled with -fmad=false so that the
// operation sequence matches the x86-64 build of the reference except for libm (sin/cos/exp/pow/atan2 <= 2 ulp).
#include <cfloat>
#include <cstdlib>
#include <climits>
#include <type_traits>
#include <vector>
#include "lmot_internal.cuh"
#include "exact_math.cuh"

namespace lmot {

namespace {

constexpr double kPi = 3.14159265358979323846;
constexpr double gammaG = 9.22, pG = 0.99, pD = 0.9;   // imm_ukf_jpda.cpp:26-34
constexpr int lifeTimeThres = 3;                        // :42
constexpr double distanceThres = 99;                    // :38
constexpr double bbYawChangeThres = 0.2;                // :46

// ---- where the tracker's constants come from (lmot_tracker_params).  TA, TB and TC are templates on a parameter source: the
// Def* sources return the reference's constants as compile-time values (the kernels every table at the defaults runs); the Tun*
// sources read the stage's own slice of a table's parameters, which travels by value in the launch's parameter block.
struct TAPrm { double gamma_g, std_a[3], std_yawdd[3], std_las_x, std_las_y, trans[3][3]; };
struct TBPrm { double gamma_g, p_g, p_d, distance_thres, bb_yaw_change_thres, second_init_v; int lifetime_thres; };
struct TCPrm { double p0_diag[5], mode_prob0[3], static_dist; int static_lifetime; };

struct DefTA {
  __device__ static constexpr double gamma_g() { return gammaG; }
  __device__ static constexpr double std_a(int m) { return (m == 2) ? 3.0 : 2.0; }       // std_a_{cv,ctrv,rm}_ ukf.cpp:68-70
  __device__ static constexpr double std_yawdd(int m) { return (m == 2) ? 3.0 : 2.0; }   // std_*_yawdd_ :71-73
  __device__ static constexpr double r(int i) { return 0.15 * 0.15; }                   // std_laspx_ / std_laspy_ squared, :91-94
  __device__ static constexpr double trans(int i, int j) { return (i == j) ? 0.9 : 0.05; }   // p{i+1}_[j], :144-154
};
struct TunTA {
  const TAPrm& p;
  __device__ double gamma_g() const { return p.gamma_g; }
  __device__ double std_a(int m) const { return p.std_a[m]; }
  __device__ double std_yawdd(int m) const { return p.std_yawdd[m]; }
  __device__ double r(int i) const { return i == 0 ? p.std_las_x * p.std_las_x : p.std_las_y * p.std_las_y; }
  __device__ double trans(int i, int j) const { return p.trans[i][j]; }
};
struct DefTB {
  __device__ static constexpr double gamma_g() { return gammaG; }
  __device__ static constexpr double p_g() { return pG; }
  __device__ static constexpr double p_d() { return pD; }
  __device__ static constexpr double distance_thres() { return distanceThres; }
  __device__ static constexpr int lifetime_thres() { return lifeTimeThres; }
  __device__ static constexpr double second_init_v() { return 2; }                     // targetV, imm_ukf_jpda.cpp:902
};
struct TunTB {
  const TBPrm& p;
  __device__ double gamma_g() const { return p.gamma_g; }
  __device__ double p_g() const { return p.p_g; }
  __device__ double p_d() const { return p.p_d; }
  __device__ double distance_thres() const { return p.distance_thres; }
  __device__ int lifetime_thres() const { return p.lifetime_thres; }
  __device__ double second_init_v() const { return p.second_init_v; }
};
struct DefTC {
  __device__ static constexpr double mode_prob0(int m) { return 0.33; }                // ukf.cpp:180-182
  __device__ static constexpr int static_lifetime() { return 8; }                      // imm_ukf_jpda.cpp:1064
  __device__ static constexpr double static_dist() { return 3.0; }                     // :1067
};
struct TunTC {
  const TCPrm& p;
  __device__ double mode_prob0(int m) const { return p.mode_prob0[m]; }
  __device__ int static_lifetime() const { return p.static_lifetime; }
  __device__ double static_dist() const { return p.static_dist; }
};

// Programmatic dependent launch (sm_90+): the three kernels of the tracker chain are launched back to back on one stream.
// A kernel calls pdl_launch_dependents() at its start so that the NEXT kernel's CTAs may already become resident and run up to
// their pdl_wait(), which returns once the whole preceding grid has finished and its writes are visible -- the dependent
// kernel's launch latency leaves the sequential chain.  Both are no-ops for a kernel launched without the attribute.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ double wrap_pi(double a) {   // the reference's while loops; NaN falls through
  // (beyond 1e4 rad the reference's loop would need thousands of iterations -- millions for a diverged filter --
  //  so the bulk is removed in one step there; such a track is already past any parity claim)
  if (fabs(a) > 1.0e4) a -= 2. * kPi * rint(a / (2. * kPi));
  while (a > kPi) a -= 2. * kPi;
  while (a < -kPi) a += 2. * kPi;
  return a;
}

// a / b, bit-identical to IEEE division, but a zero numerator over a finite non-zero denominator (covariances are full of
// exact zeros) does not go through the slow-path subroutine of the software fp64 divide: 0 * b has the same signed zero
__device__ __forceinline__ double qdiv(double a, double b) {
  return (a == 0.0 && b != 0.0 && fabs(b) <= DBL_MAX) ? a * b : a / b;
}

// Eigen dynamic determinant() == partialPivLu().determinant() (first-max pivoting, product of the diagonal)
template <int N>
__device__ double det_lu(const double* A) {
  double lu[N * N];
#pragma unroll
  for (int i = 0; i < N * N; ++i) lu[i] = A[i];
  int sign = 1;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    int piv = k; double big = fabs(lu[k * N + k]);
#pragma unroll
    for (int r = k + 1; r < N; ++r) { const double v = fabs(lu[r * N + k]); if (v > big) { big = v; piv = r; } }
    if (big != 0.0) {
      if (piv != k) {
#pragma unroll
        for (int r = k + 1; r < N; ++r)
          if (r == piv) {
#pragma unroll
            for (int c = 0; c < N; ++c) { const double t = lu[k * N + c]; lu[k * N + c] = lu[r * N + c]; lu[r * N + c] = t; }
          }
        sign = -sign;
      }
#pragma unroll
      for (int r = k + 1; r < N; ++r) lu[r * N + k] = qdiv(lu[r * N + k], lu[k * N + k]);
    }
#pragma unroll
    for (int r = k + 1; r < N; ++r)
#pragma unroll
      for (int c = k + 1; c < N; ++c) lu[r * N + c] -= lu[r * N + k] * lu[k * N + c];
  }
  double p = lu[0];
#pragma unroll
  for (int k = 1; k < N; ++k) p *= lu[k * N + k];
  return (double)sign * p;
}

__device__ __forceinline__ double det2(const double* S) { return det_lu<2>(S); }


// Eigen dynamic inverse() of a 2x2 == partialPivLu().solve(Identity)
__device__ void inv2_lu(const double* A, double* R) {
  double a00 = A[0], a01 = A[1], a10 = A[2], a11 = A[3];
  const bool sw = fabs(a10) > fabs(a00);
  if (sw) { double t = a00; a00 = a10; a10 = t; t = a01; a01 = a11; a11 = t; }
  const double l10 = qdiv(a10, a00);
  const double u11 = a11 - l10 * a01;
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    double b0 = (c == 0) ? 1.0 : 0.0, b1 = (c == 1) ? 1.0 : 0.0;
    if (sw) { const double t = b0; b0 = b1; b1 = t; }
    const double y1 = b1 - l10 * b0;
    const double x1 = qdiv(y1, u11);
    const double x0 = qdiv(b0 - a01 * x1, a00);
    R[c] = x0; R[2 + c] = x1;
  }
}

// getCpFromBbox, imm_ukf_jpda.cpp:465-479: float arithmetic inside S1/S2, double afterwards
__device__ __forceinline__ void cp_from_corners(float p1x, float p1y, float p2x, float p2y, float p3x, float p3y, float p4x,
                                                float p4y, double& cx, double& cy) {
  const double S1 = ((p4x - p2x) * (p1y - p2y) - (p4y - p2y) * (p1x - p2x)) / 2;
  const double S2 = ((p4x - p2x) * (p2y - p3y) - (p4y - p2y) * (p2x - p3x)) / 2;
  cx = p1x + (p3x - p1x) * S1 / (S1 + S2);
  cy = p1y + (p3y - p1y) * S1 / (S1 + S2);
}
__device__ __forceinline__ void cp_from_box(const float* b, double& cx, double& cy) {   // b = 8x3 floats
  cp_from_corners(b[0], b[1], b[3], b[4], b[6], b[7], b[9], b[10], cx, cy);
}

// UKF::UKF + Initialize, ukf.cpp:20-322; d = P_merge_'s diagonal (:275-279), mp = the initial mode probabilities (:180-182)
__device__ __forceinline__ void ukf_init_body(TrackState& t, double zx, double zy, const double* d, const double* mp) {
  const double x0[5] = {zx, zy, 0, 0, 0.1};
  for (int m = 0; m < 4; ++m) {
    for (int i = 0; i < 5; ++i) t.x[m][i] = x0[i];
    for (int e = 0; e < 25; ++e) t.P[m][e] = 0;
    for (int i = 0; i < 5; ++i) t.P[m][i * 5 + i] = d[i];
  }
  for (int m = 0; m < 3; ++m) {
    t.modeProb[m] = mp[m];
    t.zPred[m][0] = zx; t.zPred[m][1] = zy;
    t.S[m][0] = 1; t.S[m][1] = 0; t.S[m][2] = 0; t.S[m][3] = 1;
    for (int e = 0; e < 10; ++e) t.K[m][e] = 0;
  }
  t.bestYaw = 0; t.distFromInit = 0; t.x_merge_yaw = 0; t.initMeas[0] = 0; t.initMeas[1] = 0;
  t.velo[0] = t.velo[1] = t.velo[2] = 0;
  for (int p = 0; p < 8; ++p) for (int c = 0; c < 3; ++c) { t.BBox[p][c] = 0; t.bestBBox[p][c] = 0; }
  t.trackNum = 1; t.lifetime = 0; t.nVelo = 0; t.nBBox = 0; t.nBest = 0; t.isStatic = 0; t.isVisBB = 0;
}
__device__ void ukf_initialize(TrackState& t, double zx, double zy) {
  const double d[5] = {0.5, 0.5, 3, 10, 1};
  const double mp[3] = {0.33, 0.33, 0.33};
  ukf_init_body(t, zx, zy, d, mp);
}
__device__ void ukf_initialize(TrackState& t, double zx, double zy, const TCPrm& p) { ukf_init_body(t, zx, zy, p.p0_diag, p.mode_prob0); }
__device__ __forceinline__ void ukf_initialize(TrackState& t, double zx, double zy, DefTC) { ukf_initialize(t, zx, zy); }
__device__ __forceinline__ void ukf_initialize(TrackState& t, double zx, double zy, TunTC s) { ukf_initialize(t, zx, zy, s.p); }

// ------------------------------------------------------------------------------------------------ gate
// The tracker of frame f+1 needs (a) the tracker of frame f (same stream) and (b) the detection stages of frame f+1 (another
// stream).  (b) as a stream-level event wait in front of TA costs a full launch latency on the sequential chain AFTER the
// previous spawn_output_kernel has drained, because an event wait cannot sit between two
// programmatically dependent launches.  Instead: box_fit_kernel's last CTA posts a per-slot semaphore, and this one-warp
// kernel -- launched as a programmatic dependent of the previous frame's spawn_output_kernel, so it is resident early --
// polls it, THEN lets TA's CTAs come (they hold SM resources, so they must not be resident while anything they wait for is
// still outside this stream: a ground kernel that needs every one of its CTAs co-resident could starve), then waits for the
// previous tracker step.  TA's own griddepcontrol.wait returns when this kernel has completed, i.e. when both (a) and (b) hold.
__device__ __forceinline__ void wait_det_sem(const int* det_sem, unsigned spin_limit) {
  unsigned spin = 0;
  int v;
  do {
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(det_sem) : "memory");
    if (spin_limit && ++spin > spin_limit) __trap();       // detection never finished (seconds): fail loudly instead of hanging the stream (0: wait for ever)
  } while (v < 1);
}

__global__ void __launch_bounds__(32)
tracker_gate_kernel(const int* __restrict__ det_sem, unsigned spin_limit) {
  if (threadIdx.x == 0) wait_det_sem(det_sem, spin_limit);
  __syncwarp();
  pdl_launch_dependents();
  // (no griddepcontrol.wait: this kernel may finish before the previous frame's spawn_output_kernel does.  TA's CTAs, resident from
  // here on, wait for that step through its completion counter -- one L2 poll after spawn_output_kernel's last store instead of two
  // grid-completion hops (TC -> this kernel -> TA).)
}

// Sequence ticks (lmot_seq_*): lane k waits for sequence k's detection (its slot's semaphore, posted by box fitting or by
// boxes_to_global_seq_kernel), so TA's CTAs are released only once every frame of the tick has its boxes.
struct GateSeq { const int* sem[kMaxBatch]; int n; };

__global__ void __launch_bounds__(32)
tracker_gate_seq_kernel(const __grid_constant__ GateSeq g, unsigned spin_limit) {
  if ((int)threadIdx.x < g.n) wait_det_sem(g.sem[threadIdx.x], spin_limit);
  __syncwarp();
  pdl_launch_dependents();
}

// ------------------------------------------------------------------------------------------------ TA
constexpr int kTAThreads = 128;     // warps 0-2: one motion model each; warp 3: explosion guard, then helps gating

struct TAShared {
  double xp[3][5];       // pre-interaction states of the three models
  double Pp[3][25];
  double L[3][49];       // per model: partial Cholesky factor of P_aug
  double Xs[3][15][5];   // per model: predicted sigma points
  double Pm[3][25];      // per model: mixed covariance
  double S[3][4], Tc[3][10], zp[3][2];
  double dyaw[3][15];    // per model: wrapped yaw residual of every sigma point against the predicted mean
  double detS[3];        // per model: det(S), computed by the model's own warp
  int flag;              // 0 run, 1 skip (dead track)
  int explode;           // det(P_merge) > 10 or P_merge(4,4) > 1000 (:828-831), computed by warp 3 while warps 0-2 predict
  unsigned gbits[16];    // gate bits of the (at most 16) 32-box chunks, for the compact measurement list handed to TB
};

__device__ __forceinline__ double bcast(double v, int src) { return __shfl_sync(0xFFFFFFFFu, v, src); }

// TA for one track table; the single-stream kernel and the sequence kernel (one table per blockIdx.y) share it.  P: DefTA / TunTA
template <class TP>
__device__ __forceinline__ void
imm_predict_gate_body(TrackState* __restrict__ tracks, const int* __restrict__ trk, const int* __restrict__ det, const float* __restrict__ boxes,
                      double dt, unsigned* __restrict__ gate, unsigned* __restrict__ setter, int* __restrict__ first_setter,
                      uint8_t* __restrict__ skip, int words, const int* __restrict__ act_list,
                      int* __restrict__ meas_n, double2* __restrict__ meas_ctr,
                      const unsigned* __restrict__ tc_seq, unsigned tc_want, unsigned spin_limit, const TP& P) {
  __shared__ TAShared sh;
  pdl_wait();                              // (gated launch: the gate kernel, hence this frame's detection, is complete)
  pdl_launch_dependents();                 // TB's CTAs may line up behind this grid
  // the previous tracker step: spawn_output_kernel counts itself complete (release) after its last store.  It is ONE resident CTA
  // that needs nothing more to finish, so spinning here cannot starve it (unlike a wait for detection, see tracker_gate_kernel).
  if (threadIdx.x == 0) {
    unsigned spin = 0, v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(tc_seq) : "memory");
      if (spin_limit && ++spin > spin_limit) __trap();
    } while ((int)(v - tc_want) < 0);
  }
  __syncthreads();
  const int tid = threadIdx.x, lane = tid & 31, model = tid >> 5;
  const int n_act = trk[CNT_N_ACT];
  const int M = det[CNT_N_BOXES];
  const double lambda_aug = 3 - 7;
  const double w0 = lambda_aug / (lambda_aug + 7), wi = 0.5 / (7 + lambda_aug);

  // Only the ACTIVE tracks are visited: live ones, plus dead ones whose isVisBB_ flag is still set from the frame they died
  // in (the reference clears it for every track at :814).  The table is append-only like targets_ -- dead tracks keep their
  // slot forever -- so walking all of it would put several tracks on one CTA once it outgrows the grid.
  for (int q = blockIdx.x; q < n_act; q += gridDim.x) {
    const int it = act_list[q];
    TrackState& t = tracks[it];
    __syncthreads();
    if (tid == 0) {
      t.isVisBB = 0;                                          // :814
      const int flag = (t.trackNum == 0) ? 1 : 0;             // :826
      sh.flag = flag;
      skip[it] = (uint8_t)flag;
    }
    // stage the pre-interaction states
    for (int e = tid; e < 15; e += kTAThreads) sh.xp[e / 5][e % 5] = t.x[1 + e / 5][e % 5];
    for (int e = tid; e < 75; e += kTAThreads) sh.Pp[e / 25][e % 25] = t.P[1 + e / 25][e % 25];
    const double mp0 = t.modeProb[0], mp1 = t.modeProb[1], mp2 = t.modeProb[2];
    __syncthreads();
    if (sh.flag) continue;
    // guard :828-831 on the side: the serial 5x5 LU no longer sits in front of the prediction
    if (tid == 96) sh.explode = (det_lu<5>(t.P[0]) > 10 || t.P[0][24] > 1000) ? 1 : 0;
    double x[5] = {0, 0, 0, 0, 0};
    double Pe = 0.0, zp0 = 0.0, zp1 = 0.0;
    double Si[4] = {0, 0, 0, 0};
    if (model < 3) {
#include "imm_mix.inc"
    __syncwarp();
#include "imm_propagate.inc"
    }   // model < 3
    __syncthreads();                      // the guard's verdict is in
    if (sh.explode) {
      if (tid == 0) { t.trackNum = 0; skip[it] = 1; }
      continue;
    }
    if (model < 3) {
    // write back: x_, P_, zPred, S, K
    if (lane < 5) t.x[1 + model][lane] = x[lane];
    if (lane < 25) t.P[1 + model][lane] = Pe;
    if (lane < 10) {
      const int r = lane >> 1, c = lane & 1;
      t.K[model][lane] = sh.Tc[model][r * 2] * Si[c] + sh.Tc[model][r * 2 + 1] * Si[2 + c];
    }
    if (lane < 4) t.S[model][lane] = sh.S[model][lane];
    if (lane == 0) { t.zPred[model][0] = zp0; t.zPred[model][1] = zp1; sh.zp[model][0] = zp0; sh.zp[model][1] = zp1; }
    }   // model < 3
    __syncthreads();

    // ---- findMaxZandS (:176-203), gate scale x4 and explosion guard (:843-851)
#include "imm_max_s.inc"
    const int trackNum = t.trackNum;
    __syncthreads();                      // everyone has read t.trackNum / sh before thread 0 may change it
    if (dead) {
      if (tid == 0) { t.trackNum = 0; skip[it] = 1; }
      continue;
    }
    const double z0 = sh.zp[mm][0], z1 = sh.zp[mm][1];
    inv2_lu(S4, Si);
    const bool secondInit = (trackNum == 1);
    // ---- measurementValidation (:205-257): gate bits for every box; warps take 32-box chunks round-robin
    const int nchunk = (M + 31) >> 5;
    if (!secondInit) {
      auto gate_chunk = [&](int ch, double& cx, double& cy, bool& g) -> unsigned {
        const int b = ch * 32 + lane;
        g = false; cx = 0; cy = 0;
        if (b < M) {
          cp_from_box(boxes + (size_t)b * 24, cx, cy);
          const double d0 = cx - z0, d1 = cy - z1;
          const double nis = (d0 * Si[0] + d1 * Si[2]) * d0 + (d0 * Si[1] + d1 * Si[3]) * d1;
          g = nis < P.gamma_g();
        }
        const unsigned bits = __ballot_sync(0xFFFFFFFFu, g);
        if (lane == 0) { gate[(size_t)it * words + ch] = bits; setter[(size_t)it * words + ch] = bits; }
        if (g) atomicMin(&first_setter[b], it);
        return bits;
      };
      // Up to 512 boxes (16 chunks, four per warp) the centre points of the gated boxes are also handed to TB as a compact list
      // in box order (meas_ctr[it][0..31], count in meas_n[it]): TB's model warps then start their update straight away instead
      // of re-deriving the list from the gate words (two dependent L2 round trips) and gathering the boxes (a third)
      constexpr int kCW = 4;
      const bool compact = nchunk <= 4 * kCW;
      double ccx[kCW], ccy[kCW];
      unsigned cb[kCW];
      bool cg[kCW];
#pragma unroll
      for (int ci = 0; ci < kCW; ++ci) {
        const int ch = model + 4 * ci;
        ccx[ci] = 0; ccy[ci] = 0; cb[ci] = 0; cg[ci] = false;
        if (ch < nchunk) {
          cb[ci] = gate_chunk(ch, ccx[ci], ccy[ci], cg[ci]);
          if (compact && lane == 0) sh.gbits[ch] = cb[ci];
        }
      }
      for (int ch = model + 4 * kCW; ch < nchunk; ch += 4) { double cx, cy; bool g; gate_chunk(ch, cx, cy, g); }
      if (compact) {
        __syncthreads();                  // (uniform: every thread of the CTA is in this branch)
        int total = 0;
        for (int c2 = 0; c2 < nchunk; ++c2) total += __popc(sh.gbits[c2]);
#pragma unroll
        for (int ci = 0; ci < kCW; ++ci) {
          const int ch = model + 4 * ci;
          if (ch < nchunk && cg[ci]) {
            int off = __popc(cb[ci] & ((1u << lane) - 1u));
            for (int c2 = 0; c2 < ch; ++c2) off += __popc(sh.gbits[c2]);
            if (off < 32) meas_ctr[(size_t)it * 32 + off] = make_double2(ccx[ci], ccy[ci]);
          }
        }
        if (tid == 0) meas_n[it] = total;
      } else if (tid == 0) meas_n[it] = -1;
    } else if (model == 0) {
      // secondInit (:238-246): every running minimum of the NIS marks its box; chunks in order with a carried minimum
      if (lane == 0) meas_n[it] = -1;
      double run = 999;
      for (int ch = 0; ch < nchunk; ++ch) {
        const int b = ch * 32 + lane;
        bool g = false;
        double nis = DBL_MAX;
        if (b < M) {
          double cx, cy;
          cp_from_box(boxes + (size_t)b * 24, cx, cy);
          const double d0 = cx - z0, d1 = cy - z1;
          nis = (d0 * Si[0] + d1 * Si[2]) * d0 + (d0 * Si[1] + d1 * Si[3]) * d1;
          g = nis < P.gamma_g();
        }
        const double v = g ? nis : DBL_MAX;
        double pm = v;     // inclusive prefix minimum over lanes
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const double u = __shfl_up_sync(0xFFFFFFFFu, pm, o); if (lane >= o) pm = fmin(pm, u); }
        double ex = __shfl_up_sync(0xFFFFFFFFu, pm, 1);
        if (lane == 0) ex = DBL_MAX;
        ex = fmin(ex, run);
        const bool s = g && (nis < ex);
        const unsigned gb = __ballot_sync(0xFFFFFFFFu, g), sb = __ballot_sync(0xFFFFFFFFu, s);
        if (lane == 0) { gate[(size_t)it * words + ch] = gb; setter[(size_t)it * words + ch] = sb; }
        if (s) atomicMin(&first_setter[b], it);
        run = fmin(run, __shfl_sync(0xFFFFFFFFu, pm, 31));
      }
    }
  }
}

__global__ void __launch_bounds__(kTAThreads, 4)     // <= 128 registers: a CTA (16 K registers) fits on an SM next to a ground-kernel CTA (47 K)
imm_predict_gate_kernel(TrackState* __restrict__ tracks, const int* __restrict__ trk, const int* __restrict__ det, const float* __restrict__ boxes,
                        double dt, unsigned* __restrict__ gate, unsigned* __restrict__ setter, int* __restrict__ first_setter,
                        uint8_t* __restrict__ skip, int words, const int* __restrict__ act_list,
                        int* __restrict__ meas_n, double2* __restrict__ meas_ctr,
                        const unsigned* __restrict__ tc_seq, unsigned tc_want, unsigned spin_limit) {
  imm_predict_gate_body(tracks, trk, det, boxes, dt, gate, setter, first_setter, skip, words, act_list, meas_n, meas_ctr, tc_seq, tc_want, spin_limit, DefTA{});
}

// Sequence ticks: one launch steps every sequence's table, sequence = blockIdx.y.  `run` = 0: the sequence is on its compat first
// frame, where the single-stream path launches neither TA nor TB (its CTAs leave at once; TC spawns the quirk's track).
struct TASeq {
  TrackState* tracks; const int* trk; const int* det; const float* boxes; double dt;
  unsigned* gate; unsigned* setter; int* first_setter; uint8_t* skip; const int* act_list;
  int* meas_n; double2* meas_ctr; const unsigned* tc_seq; unsigned tc_want; int run;
};
struct TASeqParams { TASeq s[kMaxBatch]; int words; unsigned spin_limit; };
static_assert(sizeof(TASeqParams) <= 4096, "kernel parameter block");
struct TASeqTunedParams { TASeqParams b; TAPrm tp[kMaxBatch]; };
static_assert(sizeof(TASeqTunedParams) <= 4096, "kernel parameter block");

__global__ void __launch_bounds__(kTAThreads, 4)
imm_predict_gate_seq_kernel(const __grid_constant__ TASeqParams p) {
  const TASeq& q = p.s[blockIdx.y];
  if (!q.run) return;
  imm_predict_gate_body(q.tracks, q.trk, q.det, q.boxes, q.dt, q.gate, q.setter, q.first_setter, q.skip, p.words, q.act_list, q.meas_n,
                        q.meas_ctr, q.tc_seq, q.tc_want, p.spin_limit, DefTA{});
}

// ... every other chain (a table with its own parameters, or one that numbers its tracks; the context's own table too, S = 1): every
// table of it, each with its own slice
__global__ void __launch_bounds__(kTAThreads, 4)
imm_predict_gate_seq_tuned_kernel(const __grid_constant__ TASeqTunedParams p) {
  const TASeq& q = p.b.s[blockIdx.y];
  if (!q.run) return;
  imm_predict_gate_body(q.tracks, q.trk, q.det, q.boxes, q.dt, q.gate, q.setter, q.first_setter, q.skip, p.b.words, q.act_list, q.meas_n,
                        q.meas_ctr, q.tc_seq, q.tc_want, p.b.spin_limit, TunTA{p.tp[blockIdx.y]});
}

// ------------------------------------------------------------------------------------------------ TB

// What TC needs of an active track, 128 bytes per entry of the active list, written by TB (which has the record staged in
// shared memory anyway) and read by TC with one coalesced load: TC's merge / spawn / output logic is a chain of dependent
// steps, and every step that fetched its operands from the 1.6 KB records was one more L2 round trip on the sequential chain.
struct __align__(16) ActSummary {
  double x, y, yaw, v;               // merged state x_merge_(0), (1), (3), (2)
  double initx, inity;               // initMeas
  double mp0, mp1, mp2;              // modeProb
  float bb[8];                       // BBox corners 0..3, (x, y)
  int k, trackNum, lifetime;
  unsigned char isStatic, isVis, pad[2];
  int pad2[2];
};
static_assert(sizeof(ActSummary) == 128, "ActSummary is copied as sixteen 8-byte words");
static_assert(sizeof(TrackState) % 8 == 0, "TrackState is copied as 8-byte words");
constexpr int kTrackWords = (int)(sizeof(TrackState) / 8);

// getBboxArea :482-494 (float arithmetic, abs(float))
__device__ double bbox_area(const float b[][3]) {
  const float p1x = b[0][0], p1y = b[0][1], p2x = b[1][0], p2y = b[1][1], p3x = b[2][0], p3y = b[2][1], p4x = b[3][0], p4y = b[3][1];
  const double tri1 = 0.5 * fabsf((p1x - p3x) * (p2y - p3y) - (p2x - p3x) * (p1y - p3y));
  const double tri2 = 0.5 * fabsf((p1x - p4x) * (p3y - p4y) - (p3x - p4x) * (p1y - p4y));
  return tri1 + tri2;
}

// getBBoxYaw :535-563 (float sqrt, float atan2 == host libm atan2f -> exact_math.cuh)
__device__ double bbox_yaw(const float b[][3], double ukfYaw) {
  const float p1x = b[0][0], p1y = b[0][1], p2x = b[1][0], p2y = b[1][1], p3x = b[2][0], p3y = b[2][1];
  const double dist1 = sqrtf((p1x - p2x) * (p1x - p2x) + (p1y - p2y) * (p1y - p2y));
  const double dist2 = sqrtf((p3x - p2x) * (p3x - p2x) + (p3y - p2y) * (p3y - p2y));
  double yaw;
  if (dist1 > dist2) yaw = atan2f_fdlibm(p1y - p2y, p1x - p2x);
  else yaw = atan2f_fdlibm(p3y - p2y, p3x - p2x);
  const double diffYaw = fabs(yaw - ukfYaw);
  if (diffYaw < kPi * 0.5) return yaw;
  yaw += kPi;
  return wrap_pi(yaw);
}

// updateBB :565-653, executed by the whole warp on the track staged in shared memory.  The reference's statements in its
// order; what is independent runs on different lanes: the two centre points and the two areas (lane 0: BBox, lane 1:
// bestBBox -- same code, different operand), the sixteen corner rotations (lane = corner).  getBBoxYaw of an UNCHANGED box
// (deltaArea >= 0) is the same pure function of the same operands as the first evaluation and is not repeated.
// thres = bbYawChangeThres_ (:617-621)
__device__ __forceinline__ void update_bb_warp_body(TrackState& t, int lane, double thres) {
  if (!t.isVisBB) return;
  if (t.nBest == 0) {
    const float v = (lane < 24) ? (&t.BBox[0][0])[lane] : 0.f;
    __syncwarp();
    if (lane < 24) (&t.bestBBox[0][0])[lane] = v;
    if (lane == 0) { t.nBest = t.nBBox; t.bestYaw = bbox_yaw(t.BBox, t.x[0][3]); }
    __syncwarp();
    return;
  }
  const float (*bbp)[3] = (lane == 1) ? t.bestBBox : t.BBox;
  double cx, cy;
  cp_from_corners(bbp[0][0], bbp[0][1], bbp[1][0], bbp[1][1], bbp[2][0], bbp[2][1], bbp[3][0], bbp[3][1], cx, cy);
  const double ar = bbox_area(bbp);
  const double cpx = __shfl_sync(0xFFFFFFFFu, cx, 0), cpy = __shfl_sync(0xFFFFFFFFu, cy, 0);
  const double bcx = __shfl_sync(0xFFFFFFFFu, cx, 1), bcy = __shfl_sync(0xFFFFFFFFu, cy, 1);
  const double dtx = cpx - bcx, dty = cpy - bcy;
  const double ukfYaw = t.x[0][3];
  const double yaw = bbox_yaw(t.BBox, ukfYaw);
  const double deltaArea = __shfl_sync(0xFFFFFFFFu, ar, 0) - __shfl_sync(0xFFFFFFFFu, ar, 1);
  const int nB = t.nBBox;
  __syncwarp();
  if (deltaArea < 0) {                         // updateVisBoxArea :496-510
    if (lane < nB) {
      t.BBox[lane][0] = (float)(t.bestBBox[lane][0] + dtx);
      t.BBox[lane][1] = (float)(t.bestBBox[lane][1] + dty);
    }
  } else if (deltaArea > 0) {
    const float v = (lane < 24) ? (&t.BBox[0][0])[lane] : 0.f;
    if (lane < 24) (&t.bestBBox[0][0])[lane] = v;
    if (lane == 0) t.nBest = nB;
  }
  __syncwarp();
  const double currentYaw = (deltaArea < 0) ? bbox_yaw(t.BBox, ukfYaw) : yaw;
  const double DiffYaw = yaw - currentYaw;
  if (fabs(DiffYaw) > thres) {
  } else if (fabs(DiffYaw) < thres) {
    const double cd = cos(DiffYaw), sd = sin(DiffYaw);
    // updateBoxYaw :512-532 on both boxes (n = nBBox for both, like the reference): lane < 8 -> BBox, 8 <= lane < 16 -> bestBBox
    const int i = lane & 7;
    if (lane < 16 && i < nB) {
      float (*bb)[3] = (lane < 8) ? t.BBox : t.bestBBox;
      const double preX = bb[i][0], preY = bb[i][1];
      bb[i][0] = (float)(cd * (preX - cpx) - sd * (preY - cpy) + cpx);
      bb[i][1] = (float)(sd * (preX - cpx) + cd * (preY - cpy) + cpy);
    }
    if (lane == 0) t.bestYaw = yaw;
  }
  __syncwarp();
}
__device__ void update_bb_warp(TrackState& t, int lane) { update_bb_warp_body(t, lane, bbYawChangeThres); }
__device__ void update_bb_warp(TrackState& t, int lane, double thres) { update_bb_warp_body(t, lane, thres); }
__device__ __forceinline__ void update_bb_warp(TrackState& t, int lane, DefTB) { update_bb_warp(t, lane); }
__device__ __forceinline__ void update_bb_warp(TrackState& t, int lane, TunTB s) { update_bb_warp(t, lane, s.p.bb_yaw_change_thres); }

constexpr int kTBThreads = 128;    // warps 0-2: PDA update of one motion model each; warp 3: box association + updateBB

struct TBShared {
  TrackState trk;                   // the track, staged (1.6 KB)
  ActSummary sum;
  double xnew[3][5];                // per model: updated state
  double Pnew[3][25];               // per model: updated covariance
  double eSum[3];
  int tn_out, life_out;             // trackNum / lifetime_ to store once every warp has read the old values
};

// One CTA per active track.  What the reference does one after the other for a track, and what does not depend on each other,
// runs on different warps: the PDA update of the three motion models (each its own S^-1, Gaussian kernels, beta weights,
// K nu, covariance update -- identical code, different model) on warps 0..2, measurement bookkeeping / box association /
// updateBB on warp 3; then warp 0 alone: association likelihoods, mode probabilities, merged estimate.  P: DefTB / TunTB
template <class TP>
__device__ __forceinline__ void
imm_update_body(TrackState* __restrict__ tracks, const int* __restrict__ trk, const int* __restrict__ det, const float* __restrict__ boxes,
                const unsigned* __restrict__ gate, const int* __restrict__ first_setter, const uint8_t* __restrict__ skip,
                int words, const int* __restrict__ act_list, ActSummary* __restrict__ summary,
                const int* __restrict__ meas_n, const double2* __restrict__ meas_ctr, const TP& P) {
  extern __shared__ unsigned short s_list[];              // indices of the gated boxes, in box order
  __shared__ TBShared sh;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  pdl_wait();                              // TA has finished (gate rows, first_setter, predicted states are visible)
  pdl_launch_dependents();                 // TC's CTA may line up behind this grid
  const int n_act = trk[CNT_N_ACT];
  const int M = det[CNT_N_BOXES];
  const int nchunk = (M + 31) >> 5;
  TrackState& t = sh.trk;

  for (int q = blockIdx.x; q < n_act; q += gridDim.x) {
    const int it = act_list[q];
    const bool skipped = skip[it] != 0;      // dead, or killed by TA's guards: no update, but TC still wants its summary
    // TA's compact measurement list (count, centre points of the first 32 gated boxes in box order): in flight together with
    // the staging loads below.  -1 / more than 32: derive the list from the gate words as before
    const int nm_ta = skipped ? -1 : meas_n[it];
    const double2 ctr_ta = skipped ? make_double2(0.0, 0.0) : meas_ctr[(size_t)it * 32 + lane];
    __syncthreads();                         // the previous track's readers are done with the shared copy
    // stage the whole track (1.6 KB) in shared memory with coalesced 8-byte loads: the update below touches almost
    // every field several times, and every one of those touches would otherwise be its own trip to L2 / HBM
    {
      const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&tracks[it]);
      unsigned long long* dst = reinterpret_cast<unsigned long long*>(&sh.trk);
      constexpr int kIt = (kTrackWords + kTBThreads - 1) / kTBThreads;
      unsigned long long v[kIt];                     // all loads in flight before the first store
#pragma unroll
      for (int u = 0; u < kIt; ++u) { const int w = tid + kTBThreads * u; v[u] = (w < kTrackWords) ? src[w] : 0ull; }
#pragma unroll
      for (int u = 0; u < kIt; ++u) { const int w = tid + kTBThreads * u; if (w < kTrackWords) dst[w] = v[u]; }
    }
    __syncthreads();
    bool pda = false;                        // CTA-uniform: the track reaches filterPDA
    int nmeas = 0, mm = 0;
    double numMeas = 0;
    if (!skipped) {
      const int trackNum0 = t.trackNum;
      const bool secondInit = (trackNum0 == 1);
      // ---- lifetime_ (:232): a gated box counts unless an earlier track already matched it.  Every warp derives the list for
      // itself (same loads, same values: no CTA barrier in front of the model warps)
      int life = 0;
      const bool quick = warp < 3 && !secondInit && nm_ta >= 0 && nm_ta <= 32;   // model warps: everything they need came from TA
      if (quick) nmeas = nm_ta;
      else
      for (int ch0 = 0; ch0 < nchunk; ch0 += 8) {      // eight chunks per batch: two round trips (gate words, then first_setter), not two per chunk
        unsigned g4[8]; int fs4[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) g4[u] = (ch0 + u < nchunk) ? gate[(size_t)it * words + ch0 + u] : 0u;
#pragma unroll
        for (int u = 0; u < 8; ++u) fs4[u] = ((g4[u] >> lane) & 1u) ? first_setter[(ch0 + u) * 32 + lane] : INT_MAX;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const unsigned g = g4[u];
          const int b = (ch0 + u) * 32 + lane;
          const bool cnt = ((g >> lane) & 1u) && (fs4[u] >= it);
          life += __popc(__ballot_sync(0xFFFFFFFFu, cnt));
          if ((g >> lane) & 1u) s_list[nmeas + __popc(g & ((1u << lane) - 1u))] = (unsigned short)b;   // (all warps store the same values)
          nmeas += __popc(g);
        }
      }
      __syncwarp();
      const int lifetime = t.lifetime + life;

      // measurement prediction used by the gate (same selection as TA)
      const double dcv = det2(t.S[0]), dctrv = det2(t.S[1]), drm = det2(t.S[2]);
      if (dcv > dctrv) mm = (dcv > drm) ? 0 : 2; else mm = (dctrv > drm) ? 1 : 2;

      if (secondInit) {                                   // :882-921, all of it on warp 3
        if (warp == 3) {
          // the last running minimum == first occurrence of the smallest NIS (:238-255)
          double S4[4], Si[4];
          for (int e = 0; e < 4; ++e) S4[e] = t.S[mm][e] * 4;
          inv2_lu(S4, Si);
          double best = DBL_MAX; int bi = INT_MAX; double bx = 0, by = 0;
          for (int k = lane; k < nmeas; k += 32) {
            double cx, cy;
            cp_from_box(boxes + (size_t)s_list[k] * 24, cx, cy);
            const double d0 = cx - t.zPred[mm][0], d1 = cy - t.zPred[mm][1];
            const double nis = (d0 * Si[0] + d1 * Si[2]) * d0 + (d0 * Si[1] + d1 * Si[3]) * d1;
            if (nis < best) { best = nis; bi = k; bx = cx; by = cy; }
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            const double ob = __shfl_xor_sync(0xFFFFFFFFu, best, o), ox = __shfl_xor_sync(0xFFFFFFFFu, bx, o), oy = __shfl_xor_sync(0xFFFFFFFFu, by, o);
            const int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, o);
            if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; bx = ox; by = oy; }
          }
          if (lane == 0) {
            sh.life_out = lifetime;
            if (nmeas == 0) sh.tn_out = 0;
            else {
              t.initMeas[0] = t.x[0][0]; t.initMeas[1] = t.x[0][1];
              const double dX = bx - t.x[0][0], dY = by - t.x[0][1];
              const double targetYaw = wrap_pi(atan2(dY, dX));
              for (int m = 0; m < 4; ++m) { t.x[m][0] = bx; t.x[m][1] = by; t.x[m][2] = P.second_init_v(); t.x[m][3] = targetYaw; }
              sh.tn_out = trackNum0 + 1;
            }
          }
        }
      } else {
        int tn = trackNum0;                               // :924-944 (measVec.size() == nmeas)
        if (nmeas > 0) {
          if (tn < 3) tn++;
          else if (tn == 3) tn = 5;
          else if (tn >= 5) tn = 5;
        } else {
          if (tn < 5) tn = 0;
          else if (tn >= 5 && tn < 10) tn++;
          else tn = 0;                                    // `else if (trackNum = 10) trackNum = 0` (:941)
        }
        pda = (tn != 0);
        numMeas = (double)nmeas;
        if (warp == 3) {
          // ---- associateBB (:416-463) + getNearestEuclidBBox (:396-413): int minDist => first box with the smallest
          // floor(distance)
          int isVis = 0;
          if (nmeas > 0 && trackNum0 == 5 && lifetime > P.lifetime_thres()) {
            const double px = t.x[0][0], py = t.x[0][1];
            long long key = LLONG_MAX;      // (floor(dist) << 32) | position
            for (int k = lane; k < nmeas; k += 32) {
              double cx, cy;
              cp_from_box(boxes + (size_t)s_list[k] * 24, cx, cy);
              const double dist = sqrt((px - cx) * (px - cx) + (py - cy) * (py - cy));
              if (dist < 999) { const long long kk = ((long long)(int)dist << 32) | (unsigned)k; key = key < kk ? key : kk; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) { const long long ok = __shfl_xor_sync(0xFFFFFFFFu, key, o); key = key < ok ? key : ok; }
            int minDist = 999, minInd = 0;
            if (key != LLONG_MAX) { minDist = (int)(key >> 32); minInd = (int)(key & 0xFFFFFFFFll); }
            if (minDist < P.distance_thres()) {
              const float* b = boxes + (size_t)s_list[minInd] * 24;
              if (lane < 8) {
                const int c = lane & 3;
                t.BBox[lane][0] = b[c * 3]; t.BBox[lane][1] = b[c * 3 + 1];
                t.BBox[lane][2] = (lane < 4) ? (float)-1.73 : 0.f;
              }
              isVis = 1;
            }
          }
          if (lane == 0) {
            sh.life_out = lifetime; sh.tn_out = tn;
            if (isVis) { t.isVisBB = 1; t.nBBox = 8; }
          }
          __syncwarp();
          update_bb_warp(t, lane, P);                       // :877 (reads x_merge_ before warp 0 replaces it below)
        } else if (pda) {
          // ---- filterPDA (:259-394) for model `warp`; scalars replicated on every lane
          const int m = warp;
          const double pD = P.p_d(), pG = P.p_g(), gammaG = P.gamma_g();
          const double bb = 2 * numMeas * (1 - pD * pG) / (gammaG * pD);
          // centre point of every gated box once (lane k <-> measurement k; beyond 32 measurements recomputed on the fly)
          double mcx = 0, mcy = 0;
          if (quick) { if (lane < nmeas) { mcx = ctr_ta.x; mcy = ctr_ta.y; } }
          else if (lane < nmeas) cp_from_box(boxes + (size_t)s_list[lane] * 24, mcx, mcy);
          double Si[4];
          inv2_lu(t.S[m], Si);
          const double zp0 = t.zPred[m][0], zp1 = t.zPred[m][1];
          // per-lane innovation and Gaussian kernel of "its" measurement
          const double ld0 = mcx - zp0, ld1 = mcy - zp1;
          double le = 0;
          if (lane < nmeas) { const double t0 = -0.5 * ld0, t1 = -0.5 * ld1; le = exp((t0 * Si[0] + t1 * Si[2]) * ld0 + (t0 * Si[1] + t1 * Si[3]) * ld1); }
          double es = 0, betaZero, sX0 = 0, sX1 = 0;
          double sP[4] = {0, 0, 0, 0};
          if (nmeas <= 32) {
            // lane k holds measurement k: the per-measurement factors (one fp64 division, the products) are computed by all
            // lanes at once; only the SUMS run over k in the reference's order (same operands, same operations, same bits)
            for (int k = 0; k < nmeas; ++k) es += __shfl_sync(0xFFFFFFFFu, le, k);
            betaZero = bb / (bb + es);
            const double beta = (lane < nmeas) ? le / (bb + es) : 0.0;
            const double p0 = beta * ld0, p1 = beta * ld1;
            for (int k = 0; k < nmeas; ++k) { sX0 += __shfl_sync(0xFFFFFFFFu, p0, k); sX1 += __shfl_sync(0xFFFFFFFFu, p1, k); }
            const double t00 = p0 * ld0 - sX0 * sX0, t01 = p0 * ld1 - sX0 * sX1, t10 = p1 * ld0 - sX1 * sX0, t11 = p1 * ld1 - sX1 * sX1;
            for (int k = 0; k < nmeas; ++k) {
              sP[0] += __shfl_sync(0xFFFFFFFFu, t00, k); sP[1] += __shfl_sync(0xFFFFFFFFu, t01, k);
              sP[2] += __shfl_sync(0xFFFFFFFFu, t10, k); sP[3] += __shfl_sync(0xFFFFFFFFu, t11, k);
            }
          } else {
            auto meas = [&](int k, double& d0, double& d1, double& e) {        // k is warp-uniform
              if (k < 32) { d0 = __shfl_sync(0xFFFFFFFFu, ld0, k); d1 = __shfl_sync(0xFFFFFFFFu, ld1, k); e = __shfl_sync(0xFFFFFFFFu, le, k); }
              else {
                double cx, cy;
                cp_from_box(boxes + (size_t)s_list[k] * 24, cx, cy);
                d0 = cx - zp0; d1 = cy - zp1;
                const double t0 = -0.5 * d0, t1 = -0.5 * d1;
                e = exp((t0 * Si[0] + t1 * Si[2]) * d0 + (t0 * Si[1] + t1 * Si[3]) * d1);
              }
            };
            for (int k = 0; k < nmeas; ++k) { double d0, d1, e; meas(k, d0, d1, e); es += e; }
            betaZero = bb / (bb + es);
            for (int k = 0; k < nmeas; ++k) {
              double d0, d1, e; meas(k, d0, d1, e);
              const double beta = e / (bb + es);
              sX0 += beta * d0; sX1 += beta * d1;
            }
            for (int k = 0; k < nmeas; ++k) {
              double d[2], e; meas(k, d[0], d[1], e);
              const double beta = e / (bb + es);
              const double sXv[2] = {sX0, sX1};
#pragma unroll
              for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int c = 0; c < 2; ++c) sP[r * 2 + c] += ((beta * d[r]) * d[c] - sXv[r] * sXv[c]);
            }
          }
          const double* K = t.K[m];
          const double* S = t.S[m];
          if (lane < 5) {
            double xr = t.x[1 + m][lane] + (K[lane * 2] * sX0 + K[lane * 2 + 1] * sX1);
            if (lane == 3) xr = wrap_pi(xr);
            sh.xnew[m][lane] = xr;
          }
          if (lane < 25) {
            const int r = lane / 5, c = lane % 5;
            const double KS0 = K[r * 2] * S[0] + K[r * 2 + 1] * S[2], KS1 = K[r * 2] * S[1] + K[r * 2 + 1] * S[3];
            const double KP0 = K[r * 2] * sP[0] + K[r * 2 + 1] * sP[2], KP1 = K[r * 2] * sP[1] + K[r * 2 + 1] * sP[3];
            const double KSK = KS0 * K[c * 2] + KS1 * K[c * 2 + 1], KPK = KP0 * K[c * 2] + KP1 * K[c * 2 + 1];
            const double P = t.P[1 + m][lane];
            double Pe;
            if (numMeas != 0) Pe = betaZero * P + (1 - betaZero) * (P - KSK) + KPK;
            else Pe = P - KSK;
            sh.Pnew[m][lane] = Pe;
          }
          if (lane == 0) sh.eSum[m] = es;
        }
      }
    }
    __syncthreads();
    if (!skipped && warp == 0) {
      if (pda) {
        const double pD = P.p_d(), pG = P.p_g(), gammaG = P.gamma_g();
        const double Vk = kPi * sqrt(gammaG * det2(t.S[mm]));     // S is untouched by the update, same max model
        double lam[3];
        {
          // the two pow() (same base, exponents numMeas and 1 - numMeas) on lanes 0 / 1, the three model terms on lanes 0..2: one
          // pass through pow / sqrt / the divisions instead of two and three
          const double ex = (lane == 1) ? 1 - numMeas : numMeas;
          const double pw = pow(Vk, ex);
          const double powN = __shfl_sync(0xFFFFFFFFu, pw, 0);
          const double pow1N = (numMeas != 0) ? __shfl_sync(0xFFFFFFFFu, pw, 1) : 0.0;
          const int ml = (lane < 3) ? lane : 0;
          const double em = sh.eSum[ml];
          double lv;
          if (numMeas != 0) lv = (1 - pG * pD) / powN + pD * pow1N * em / (numMeas * sqrt(2 * kPi * det2(t.S[ml])));
          else lv = (1 - pG * pD) / powN;
          lam[0] = __shfl_sync(0xFFFFFFFFu, lv, 0); lam[1] = __shfl_sync(0xFFFFFFFFu, lv, 1); lam[2] = __shfl_sync(0xFFFFFFFFu, lv, 2);
        }
        // ---- PostProcessIMMUKF: UpdateModeProb (ukf.cpp:384-397), MergeEstimationAndCovariance (:419-437)
        double mp[3] = {t.modeProb[0], t.modeProb[1], t.modeProb[2]};
#include "imm_merge.inc"
        if (lane < 25) {
#include "imm_merge_p.inc"
          t.P[0][lane] = a0 + a1 + a2;
          t.P[1][lane] = Pn0; t.P[2][lane] = Pn1; t.P[3][lane] = Pn2;
        }
        if (lane < 5) {
          const double xml = (lane == 0) ? xm[0] : (lane == 1) ? xm[1] : (lane == 2) ? xm[2] : (lane == 3) ? xm[3] : xm[4];
          t.x[0][lane] = xml; t.x[1][lane] = sh.xnew[0][lane]; t.x[2][lane] = sh.xnew[1][lane]; t.x[3][lane] = sh.xnew[2][lane];
        }
        if (lane == 0) {
          t.modeProb[0] = mp[0]; t.modeProb[1] = mp[1]; t.modeProb[2] = mp[2];
          t.x_merge_yaw = myaw;
          int nv = t.nVelo;                                 // velo_history_ :955-959
          if (nv == 3) { t.velo[0] = t.velo[1]; t.velo[1] = t.velo[2]; nv = 2; }
          t.velo[nv] = xm[2];
          t.nVelo = nv + 1;
        }
      }
      if (lane == 0) { t.trackNum = sh.tn_out; t.lifetime = sh.life_out; }
    }
    __syncthreads();
    if (!skipped) {
      const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&sh.trk);
      unsigned long long* dst = reinterpret_cast<unsigned long long*>(&tracks[it]);
      for (int w = tid; w < kTrackWords; w += kTBThreads) dst[w] = src[w];
    }
    if (warp == 0) {
      if (lane == 0) {
        ActSummary& a = sh.sum;
        a.x = t.x[0][0]; a.y = t.x[0][1]; a.yaw = t.x[0][3]; a.v = t.x[0][2];
        a.initx = t.initMeas[0]; a.inity = t.initMeas[1];
        a.mp0 = t.modeProb[0]; a.mp1 = t.modeProb[1]; a.mp2 = t.modeProb[2];
#pragma unroll
        for (int e = 0; e < 8; ++e) a.bb[e] = t.BBox[e >> 1][e & 1];
        a.k = it; a.trackNum = t.trackNum; a.lifetime = t.lifetime;
        a.isStatic = t.isStatic; a.isVis = t.isVisBB; a.pad[0] = a.pad[1] = 0; a.pad2[0] = a.pad2[1] = 0;
      }
      __syncwarp();
      if (lane < 16) reinterpret_cast<unsigned long long*>(&summary[q])[lane] = reinterpret_cast<const unsigned long long*>(&sh.sum)[lane];
    }
  }
}

__global__ void __launch_bounds__(kTBThreads)
imm_update_kernel(TrackState* __restrict__ tracks, const int* __restrict__ trk, const int* __restrict__ det, const float* __restrict__ boxes,
                  const unsigned* __restrict__ gate, const int* __restrict__ first_setter, const uint8_t* __restrict__ skip,
                  int words, const int* __restrict__ act_list, ActSummary* __restrict__ summary,
                  const int* __restrict__ meas_n, const double2* __restrict__ meas_ctr) {
  imm_update_body(tracks, trk, det, boxes, gate, first_setter, skip, words, act_list, summary, meas_n, meas_ctr, DefTB{});
}

// sequence ticks: sequence = blockIdx.y, `run` as for TA
struct TBSeq {
  TrackState* tracks; const int* trk; const int* det; const float* boxes; const unsigned* gate; const int* first_setter;
  const uint8_t* skip; const int* act_list; ActSummary* summary; const int* meas_n; const double2* meas_ctr; int run;
};
struct TBSeqParams { TBSeq s[kMaxBatch]; int words; };
static_assert(sizeof(TBSeqParams) <= 4096, "kernel parameter block");
struct TBSeqTunedParams { TBSeqParams b; TBPrm tp[kMaxBatch]; };
static_assert(sizeof(TBSeqTunedParams) <= 4096, "kernel parameter block");

__global__ void __launch_bounds__(kTBThreads)
imm_update_seq_kernel(const __grid_constant__ TBSeqParams p) {
  const TBSeq& q = p.s[blockIdx.y];
  if (!q.run) return;
  imm_update_body(q.tracks, q.trk, q.det, q.boxes, q.gate, q.first_setter, q.skip, p.words, q.act_list, q.summary, q.meas_n, q.meas_ctr, DefTB{});
}

// ... every other chain (as imm_predict_gate_seq_tuned_kernel's)
__global__ void __launch_bounds__(kTBThreads)
imm_update_seq_tuned_kernel(const __grid_constant__ TBSeqTunedParams p) {
  const TBSeq& q = p.b.s[blockIdx.y];
  if (!q.run) return;
  imm_update_body(q.tracks, q.trk, q.det, q.boxes, q.gate, q.first_setter, q.skip, p.b.words, q.act_list, q.summary, q.meas_n, q.meas_ctr,
                  TunTB{p.tp[blockIdx.y]});
}

// ------------------------------------------------------------------------------------------------ track prediction
// lmot_predict_tracks*: on a COPY of every row of 1..8 tables, at up to LMOT_MAX_PRED_TIMES query times: ProcessIMMUKF(dt), findMaxZandS,
// PostProcessIMMUKF({1, 1, 1}) (DESIGN.md section 6f).  Read-only: the table is never written.  One CTA per row (grid-stride over the
// table's row count, read on the device), table = blockIdx.y.  Warps 0-2 = the models CV / CTRV / RM, as in TA: the mixing, interaction
// and Cholesky of P_aug once per row (imm_mix.inc -- they do not depend on dt), then per query time the propagation, predicted mean /
// covariance and S (imm_propagate.inc) into one of two buffers.  Warp 3 works one time behind: findMaxZandS and the gate guard
// (imm_max_s.inc), TB's merge (imm_merge.inc, imm_merge_p.inc) and the outputs of time j - 1 while warps 0-2 predict time j.
// No polling of any kind: it never holds SMs that something outside its stream has to reach.
struct PredTab {
  const TrackState* tracks; const int* trk;
  const long long* ids;              // the rows' track IDs; nullptr: the row indices (a table that never retired)
  lmot_pred_out o; int* n_rows;      // device arrays; n_rows nullable
  TAPrm tp;
};
struct PredParams { PredTab s[kMaxBatch]; double dt[kMaxBatch][LMOT_MAX_PRED_TIMES]; int n_t; };
static_assert(sizeof(PredParams) <= 4096, "kernel parameter block");

struct PredBuf { double xnew[3][5], Pnew[3][25], S[3][4], zp[3][2], detS[3]; };   // the three models at one query time (TB's names)
struct PredShared {                  // TA's staging (TAShared's names: the shared bodies read them), two PredBufs, the row's verdict
  double xp[3][5];
  double Pp[3][25];
  double L[3][49];
  double Xs[3][15][5];
  double Pm[3][25];
  double S[3][4], Tc[3][10];
  double dyaw[3][15];
  double detS[3];
  PredBuf buf[2];
  int flag;                          // 0: predict; LMOT_PRED_DEAD / LMOT_PRED_GUARD_P: not predicted
};

__global__ void __launch_bounds__(kTAThreads, 4)     // <= 128 registers, like TA: fits on an SM next to a ground-kernel CTA
predict_tracks_kernel(const __grid_constant__ PredParams p) {
  __shared__ PredShared sh_all;
  PredShared& sh = sh_all;
  PredBuf* const bufs = sh_all.buf;
  pdl_wait();                              // the latest step (TC, its retire phase included) has completed
  const PredTab& q = p.s[blockIdx.y];
  const TunTA P{q.tp};
  const int tid = threadIdx.x, lane = tid & 31, model = tid >> 5;
  const int n_t = p.n_t, cap = q.o.cap;
  const int T = q.trk[CNT_N_TRACKS];
  if (blockIdx.x == 0 && tid == 0 && q.n_rows) *q.n_rows = T;
  const int n = T < cap ? T : cap;         // rows beyond cap are not written
  const double lambda_aug = 3 - 7;
  const double w0 = lambda_aug / (lambda_aug + 7), wi = 0.5 / (7 + lambda_aug);
  const double qnan = __longlong_as_double(0x7FF8000000000000ll);

  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const TrackState& t = q.tracks[i];
    __syncthreads();                       // the previous row's readers are done with the shared copy
    if (tid == 0) {
      const int tn = t.trackNum;
      sh.flag = (tn == 0) ? LMOT_PRED_DEAD : (det_lu<5>(t.P[0]) > 10 || t.P[0][24] > 1000) ? LMOT_PRED_GUARD_P : 0;   // :826, :828-831
      q.o.ids[i] = q.ids ? q.ids[i] : (long long)i;
      q.o.track_manage[i] = tn;
    }
    for (int e = tid; e < 15; e += kTAThreads) sh.xp[e / 5][e % 5] = t.x[1 + e / 5][e % 5];
    for (int e = tid; e < 75; e += kTAThreads) sh.Pp[e / 25][e % 25] = t.P[1 + e / 25][e % 25];
    const double mp0 = t.modeProb[0], mp1 = t.modeProb[1], mp2 = t.modeProb[2];
    __syncthreads();
    const int flag = sh.flag;
    if (flag) {                            // not predicted: the flag, and NaN for every value, at every time
      for (int e = tid; e < n_t * 40; e += kTAThreads) {
        const int j = e / 40, k = e % 40;
        const size_t row = (size_t)j * cap + i;
        if (k < 5) q.o.x[row * 5 + k] = qnan;
        else if (k < 30) q.o.P[row * 25 + (k - 5)] = qnan;
        else if (k < 33) q.o.mode_prob[row * 3 + (k - 30)] = qnan;
        else if (k < 35) { if (q.o.gate_z) q.o.gate_z[row * 2 + (k - 33)] = qnan; }
        else if (k < 39) { if (q.o.gate_S) q.o.gate_S[row * 4 + (k - 35)] = qnan; }
        else q.o.flags[row] = (uint8_t)flag;
      }
      continue;
    }
    double x[5] = {0, 0, 0, 0, 0};
    double Pe = 0.0, zp0 = 0.0, zp1 = 0.0;
    double Si[4] = {0, 0, 0, 0};
    double xi[5];                          // the mixed mean every query time starts from
    if (model < 3) {
#include "imm_mix.inc"
    __syncwarp();
    }
#pragma unroll
    for (int e = 0; e < 5; ++e) xi[e] = x[e];
    for (int j = 0; j <= n_t; ++j) {
      if (model < 3 && j < n_t) {
        const double dt = p.dt[blockIdx.y][j];
#pragma unroll
        for (int e = 0; e < 5; ++e) x[e] = xi[e];
        Pe = 0.0; zp0 = 0.0; zp1 = 0.0;
#include "imm_propagate.inc"
        PredBuf& b = bufs[j & 1];
        if (lane < 5) b.xnew[model][lane] = (lane == 0) ? x[0] : (lane == 1) ? x[1] : (lane == 2) ? x[2] : (lane == 3) ? x[3] : x[4];
        if (lane < 25) b.Pnew[model][lane] = Pe;
        if (lane < 4) b.S[model][lane] = sh.S[model][lane];
        if (lane == 0) { b.zp[model][0] = zp0; b.zp[model][1] = zp1; b.detS[model] = sh.detS[model]; }
      } else if (model == 3 && j > 0) {
        const PredBuf& sh = bufs[(j - 1) & 1];     // (the shared bodies read `sh`: here the buffer of time j - 1)
#include "imm_max_s.inc"
        double lam[3] = {1.0, 1.0, 1.0};           // PostProcessIMMUKF({1, 1, 1}): a step without information
        double mp[3] = {mp0, mp1, mp2};
#include "imm_merge.inc"
        const size_t row = (size_t)(j - 1) * cap + i;
        if (lane < 25) {
#include "imm_merge_p.inc"
          q.o.P[row * 25 + lane] = a0 + a1 + a2;
        }
        if (lane < 5) q.o.x[row * 5 + lane] = (lane == 0) ? xm[0] : (lane == 1) ? xm[1] : (lane == 2) ? xm[2] : (lane == 3) ? xm[3] : xm[4];
        if (lane < 3) q.o.mode_prob[row * 3 + lane] = (lane == 0) ? mp[0] : (lane == 1) ? mp[1] : mp[2];
        if (q.o.gate_z && lane < 2) q.o.gate_z[row * 2 + lane] = sh.zp[mm][lane];
        if (q.o.gate_S && lane < 4) q.o.gate_S[row * 4 + lane] = sh.S[mm][lane];
        if (lane == 0) q.o.flags[row] = (uint8_t)(LMOT_PRED_VALID | (dead ? LMOT_PRED_GUARD_S : 0));
      }
      __syncthreads();                     // buffer j is complete / buffer j - 1 is consumed
    }
  }
}

// ------------------------------------------------------------------------------------------------ TC: over-segmentation test
__device__ __forceinline__ double intersect_coef(double v1x, double v1y, double v2x, double v2y, double px, double py, double cpx, double cpy) {
  return (((v1x - v2x) * (py - v1y) + (v1y - v2y) * (v1x - px)) * ((v1x - v2x) * (cpy - v1y) + (v1y - v2y) * (v1x - cpx)));
}

// does the visible box with corners c[0..7] = (x1,y1,..,x4,y4) contain the position (px,py)?  (:670-696)
// ab = its axis-aligned bounds (min x, max x, min y, max y).  Cheap exact-safe rejection first: all three products of a
// triangle test are > 0 only for a point strictly inside that triangle (up to rounding of the cross products, ~1e-13 m
// here), hence inside the box's bounds.  The bounds are widened by 1 cm + 1e-9 of the coordinate, orders of magnitude
// beyond that rounding, so a rejected point fails the full test too; NaN coordinates are not rejected and fall through
// to it.  ~99 % of the (visible box, track) pairs stop here instead of running ~120 fp64 operations.
__device__ __forceinline__ bool overseg_cond(const float* c, const float* ab, double px, double py) {
  const double mg = 0.01 + 1.0e-9 * (fabs(px) + fabs(py));
  if (px < (double)ab[0] - mg || px > (double)ab[1] + mg || py < (double)ab[2] - mg || py > (double)ab[3] + mg) return false;
  const double v1x = c[0], v1y = c[1], v2x = c[2], v2y = c[3], v3x = c[4], v3y = c[5], v4x = c[6], v4y = c[7];
  const double cp1x = (v1x + v2x + v3x) / 3, cp1y = (v1y + v2y + v3y) / 3;
  const double cp2x = (v1x + v4x + v3x) / 3, cp2y = (v1y + v4y + v3y) / 3;
  const double c1 = intersect_coef(v1x, v1y, v2x, v2y, px, py, cp1x, cp1y);
  const double c2 = intersect_coef(v1x, v1y, v3x, v3y, px, py, cp1x, cp1y);
  const double c3 = intersect_coef(v3x, v3y, v2x, v2y, px, py, cp1x, cp1y);
  const double c4 = intersect_coef(v1x, v1y, v4x, v4y, px, py, cp2x, cp2y);
  const double c5 = intersect_coef(v1x, v1y, v3x, v3y, px, py, cp2x, cp2y);
  const double c6 = intersect_coef(v3x, v3y, v4x, v4y, px, py, cp2x, cp2y);
  return (c1 > 0 && c2 > 0 && c3 > 0) || (c4 > 0 && c5 > 0 && c6 > 0);
}

constexpr int kTCThreads = 256;      // ONE small CTA: 16 K registers, so it starts on any SM next to the resident detection kernels
                                     // instead of waiting for a whole SM to drain (a 1024-thread CTA needs the full register file)
constexpr int kTCWide = 512;         // the same kernel for scenes with 257..512 active tracks (multi-sensor ticks, dense traffic): the
                                     // fast path holds one active track per thread (chain_launch picks the variant from the last
                                     // active-track count the host has seen; either variant is correct for any count)
constexpr int kVisChunk = 128;       // visible boxes staged in shared memory per pass
constexpr int kCandCap = 1024;       // (box, track) pairs that pass the bounds pre-test, per pass (more: tested inline)

// ------------------------------------------------------------------------------------------------ TC2
// One frame's results.  spawn_output_kernel fills the DEVICE copy (the tracker is the sequential chain of the pipeline:
// nothing slow may sit on it); publish_kernel, on its own stream and off that chain, moves it into the pinned,
// device-mapped host block -- its stores are the D2H transfer, sized by the counts only the device knows.
struct OutPtrs {
  float* targets; double* vandyaw; int* track_manage; uint8_t* is_static; uint8_t* is_vis; float* vis_bb; int* hdr; float* boxes;
};

// Block-wide exclusive offsets of up to two 0/1 flags per thread (packed a | b << 16): ballot inside the warp, one shuffle scan
// of the 32 warp totals by warp 0.  s_w = int[33] scratch; returns (exclusive offset, block total), both packed the same way.
__device__ __forceinline__ void block_offsets(int a, int b, int* s_w, int& excl, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned ba = __ballot_sync(0xFFFFFFFFu, a), bb = __ballot_sync(0xFFFFFFFFu, b);
  if (lane == 0) s_w[warp] = __popc(ba) | (__popc(bb) << 16);
  __syncthreads();
  if (warp == 0) {
    const int c = lane < (int)(blockDim.x >> 5) ? s_w[lane] : 0;
    int inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (lane >= o) inc += u; }
    s_w[lane] = inc - c;
    if (lane == 31) s_w[32] = inc;
  }
  __syncthreads();
  const unsigned lt = (1u << lane) - 1u;
  excl = s_w[warp] + (__popc(ba & lt) | (__popc(bb & lt) << 16));
  total = s_w[32];
}

// per-track outputs of one track (:995-1041) + static flag (:1045-1081) into the frame's result block; returns isVisBB
template <class TP>
__device__ __forceinline__ int emit_track(TrackState& t, int i, double ego_yaw, const OutPtrs& o, double4* __restrict__ pos, const TP& P) {
  const double tx = t.x[0][0], ty = t.x[0][1];
  const double mx = t.initMeas[0], my = t.initMeas[1];
  t.distFromInit = sqrt((tx - mx) * (tx - mx) + (ty - my) * (ty - my));
  double tyaw = t.x[0][3];
  tyaw += ego_yaw;
  tyaw = wrap_pi(tyaw);
  o.targets[3 * i] = (float)tx; o.targets[3 * i + 1] = (float)ty; o.targets[3 * i + 2] = (float)(-1.73 / 2);
  o.vandyaw[2 * i] = t.x[0][2]; o.vandyaw[2 * i + 1] = tyaw;
  const int vis = t.isVisBB ? 1 : 0;
  o.is_vis[i] = (uint8_t)vis;
  int st = 0;
  if (t.isStatic) st = 1;
  else if (t.trackNum == 5 && t.lifetime > P.static_lifetime()) {
    if ((t.distFromInit < P.static_dist()) &&(t.modeProb[2] > t.modeProb[0] || t.modeProb[2] > t.modeProb[1])) { st = 1; t.isStatic = 1; }
  }
  o.is_static[i] = (uint8_t)st;
  o.track_manage[i] = t.trackNum;
  pos[i] = make_double4(tx, ty, t.x[0][3], 0.0);
  return vis;
}

// dst[0..n) = src[0..n) by the whole CTA, U loads in flight per thread before the first store.  (A plain
// `for (...) dst[e] = src[e]` over pointers the compiler cannot prove distinct is a chain of load -> store -> load round
// trips; on the one CTA of the tracker's sequential chain every one of them is on the critical path.)
template <int NT, typename T, int U>
__device__ __forceinline__ void cta_copy(T* dst, const T* src, int n) {
  for (int base = 0; base < n; base += NT * U) {
    T v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { const int e = base + u * NT + (int)threadIdx.x; if (e < n) v[u] = src[e]; }
#pragma unroll
    for (int u = 0; u < U; ++u) { const int e = base + u * NT + (int)threadIdx.x; if (e < n) dst[e] = v[u]; }
  }
}

// the two halves of cta_copy for the first U * NT items, so that the loads of SEVERAL arrays can be in flight together
template <int NT, typename T, int U>
__device__ __forceinline__ void cta_load(T (&v)[U], const T* src, int n) {
#pragma unroll
  for (int u = 0; u < U; ++u) { const int e = u * NT + (int)threadIdx.x; if (e < n) v[u] = src[e]; }
}
template <int NT, typename T, int U>
__device__ __forceinline__ void cta_store(T* dst, const T (&v)[U], int n) {
#pragma unroll
  for (int u = 0; u < U; ++u) { const int e = u * NT + (int)threadIdx.x; if (e < n) dst[e] = v[u]; }
}

// per-track outputs (:995-1041) + static flag (:1045-1081) from values instead of the record (the fast path of TC holds an
// active track's fields in registers); same statements as emit_track.  Returns the new isStatic.
template <class TP>
__device__ __forceinline__ int emit_values(int i, double tx, double ty, double yaw, double v, double mx, double my, double mp0, double mp1,
                                           double mp2, int trackNum, int lifetime, int isStatic, int vis, double ego_yaw, const OutPtrs& o,
                                           double4* __restrict__ pos, double& distFromInit, const TP& P) {
  distFromInit = sqrt((tx - mx) * (tx - mx) + (ty - my) * (ty - my));
  double tyaw = yaw;
  tyaw += ego_yaw;
  tyaw = wrap_pi(tyaw);
  o.targets[3 * i] = (float)tx; o.targets[3 * i + 1] = (float)ty; o.targets[3 * i + 2] = (float)(-1.73 / 2);
  o.vandyaw[2 * i] = v; o.vandyaw[2 * i + 1] = tyaw;
  o.is_vis[i] = (uint8_t)vis;
  int st = 0;
  if (isStatic) st = 1;
  else if (trackNum == 5 && lifetime > P.static_lifetime()) {
    if ((distFromInit < P.static_dist()) &&(mp2 > mp0 || mp2 > mp1)) st = 1;
  }
  o.is_static[i] = (uint8_t)st;
  o.track_manage[i] = trackNum;
  pos[i] = make_double4(tx, ty, yaw, 0.0);
  return st;
}


// TC, fast path: at most NT active tracks (thread q <-> entry q of the active list).  Everything the merge / spawn /
// output logic needs of an active track arrives in ONE coalesced load of TB's 128-byte summaries and stays in registers and
// shared memory; the 1.6 KB records are only written (trackNum / isStatic / distFromInit changes, new tracks), never waited
// for, except the 96-byte box of a visible track, whose load is in flight during the merge.  Same results as the general
// path below, statement for statement; see there for why mergeOverSegmentation reduces to imax / has5.
template <int NT>
struct TCFastShared {
  int w[33];
  int ncand, ncont, carry;
  int imax[NT];
  unsigned short cont[NT];             // (every active track sits in one thread: at most NT visible boxes)
  unsigned char h5[NT];
  int vid[NT];
  float bx[NT][8];
  float4 ab[NT];
  double px[NT], py[NT];
  float4 t4[NT];              // per active track: float position, pre-test margin, track index (bits; -1 = not live)
  unsigned cand[kCandCap];            // (visible slot << 16) | thread of the track
};

// a (visible box, track) pair passed the single-precision bounds pre-test: queue it for the exact test (one pair per thread
// later), or -- queue full -- test it here.  Not inlined: the callers' loops stay small, this is the rare path.
template <int NT>
__device__ __noinline__ void tc_candidate(TCFastShared<NT>& S, int v, int jt) {
  const int slot = atomicAdd(&S.ncand, 1);
  if (slot < kCandCap) S.cand[slot] = ((unsigned)v << 16) | (unsigned)jt;
  else if (overseg_cond(S.bx[v], reinterpret_cast<const float*>(&S.ab[v]), S.px[jt], S.py[jt])) atomicMax(&S.imax[jt], S.vid[v]);
}

template <int NT, class TP>
__device__ __forceinline__ void tc_fast(TCFastShared<NT>& S, TrackState* __restrict__ tracks, int* __restrict__ trk, int* __restrict__ det,
                                        const float* __restrict__ boxes, const float* __restrict__ boxes_pub, int* __restrict__ first_setter, double ego_yaw, int max_tracks,
                                        const OutPtrs& o, const OutPtrs& prev, int* __restrict__ act_list, double4* __restrict__ pos,
                                        const ActSummary* __restrict__ summary, int T0, int n_act0, int M, const TP& P) {
  const int tid = threadIdx.x, lane = tid & 31;
  const bool have = tid < n_act0;
  // ---- one round trip: the summaries, the previous result block, the spawn inputs
  ActSummary r;
  if (have) {
    const uint4* src = reinterpret_cast<const uint4*>(&summary[tid]);
    uint4* dst = reinterpret_cast<uint4*>(&r);
#pragma unroll
    for (int e = 0; e < 8; ++e) dst[e] = src[e];
  } else {
    r.k = -1; r.trackNum = 0; r.isVis = 0; r.isStatic = 0; r.lifetime = 0; r.x = r.y = r.yaw = r.v = 0; r.initx = r.inity = 0; r.mp0 = r.mp1 = r.mp2 = 0;
  }
  const bool cp = prev.targets != o.targets;
  // everything else this kernel reads that does not depend on the summaries: the frame's box list (it travels with the
  // results), the previous result block (dead tracks: unchanged), the packed yaw of every track, the spawn inputs.  ALL loads
  // are issued before the first store -- each load -> store pair behind another one was one more L2 round trip
  constexpr int UB = 4, UT = 4, UM = 2, UY = 4;
  const int nbx = M * 6, ntg = cp ? (T0 * 12 + 15) / 16 : 0, ntm = cp ? (T0 * 4 + 15) / 16 : 0, nsv = cp ? (T0 + 15) / 16 : 0;
  uint4 vbx[UB], vtg[UT], vtm[UM], vst[1], vvi[1];
  double pz[UY], pv[UY];
  cta_load<NT>(vbx, reinterpret_cast<const uint4*>(boxes_pub), nbx);     // (sensor-frame list; `boxes` is the tracker's input, in the global frame when lmot_params.global_frame is on)
  const int fs0 = (tid < M) ? first_setter[tid] : 0;            // first pass of the spawn loop below
  float bc[8] = {0, 0, 0, 0, 0, 0, 0, 0};                      // corners 0..3 (x, y) of this thread's box
  if (tid < M) {
    const float4* b4 = reinterpret_cast<const float4*>(boxes + (size_t)tid * 24);   // 96-byte boxes: 16-byte aligned
    const float4 q0 = b4[0], q1 = b4[1], q2 = b4[2];
    bc[0] = q0.x; bc[1] = q0.y; bc[2] = q0.w; bc[3] = q1.x; bc[4] = q1.z; bc[5] = q1.w; bc[6] = q2.y; bc[7] = q2.z;
  }
  int hdr_in[4] = {0, 0, 0, 0};
  if (tid == 0) { hdr_in[0] = det[CNT_N_ELEV]; hdr_in[1] = det[CNT_N_GROUND]; hdr_in[2] = det[CNT_NUM_CLUSTER]; hdr_in[3] = det[CNT_ERROR]; }
  cta_load<NT>(vtg, reinterpret_cast<const uint4*>(prev.targets), ntg);
  cta_load<NT>(vtm, reinterpret_cast<const uint4*>(prev.track_manage), ntm);
  cta_load<NT>(vst, reinterpret_cast<const uint4*>(prev.is_static), nsv);
  cta_load<NT>(vvi, reinterpret_cast<const uint4*>(prev.is_vis), nsv);
#pragma unroll
  for (int u = 0; u < UY; ++u) {
    const int e = u * NT + tid;
    pz[u] = 0; pv[u] = 0;
    if (e < T0) { pz[u] = pos[e].z; if (cp) pv[u] = prev.vandyaw[2 * e]; }
  }
  // ---- stores (and the rare remainders beyond the first batch of each array)
  cta_store<NT>(reinterpret_cast<uint4*>(o.boxes), vbx, nbx);
  if (nbx > UB * NT) cta_copy<NT, uint4, UB>(reinterpret_cast<uint4*>(o.boxes) + UB * NT, reinterpret_cast<const uint4*>(boxes_pub) + UB * NT, nbx - UB * NT);
  cta_store<NT>(reinterpret_cast<uint4*>(o.targets), vtg, ntg);
  if (ntg > UT * NT) cta_copy<NT, uint4, UT>(reinterpret_cast<uint4*>(o.targets) + UT * NT, reinterpret_cast<const uint4*>(prev.targets) + UT * NT, ntg - UT * NT);
  cta_store<NT>(reinterpret_cast<uint4*>(o.track_manage), vtm, ntm);
  if (ntm > UM * NT) cta_copy<NT, uint4, UM>(reinterpret_cast<uint4*>(o.track_manage) + UM * NT, reinterpret_cast<const uint4*>(prev.track_manage) + UM * NT, ntm - UM * NT);
  cta_store<NT>(reinterpret_cast<uint4*>(o.is_static), vst, nsv);
  cta_store<NT>(reinterpret_cast<uint4*>(o.is_vis), vvi, nsv);
  if (nsv > NT) {
    cta_copy<NT, uint4, 1>(reinterpret_cast<uint4*>(o.is_static) + NT, reinterpret_cast<const uint4*>(prev.is_static) + NT, nsv - NT);
    cta_copy<NT, uint4, 1>(reinterpret_cast<uint4*>(o.is_vis) + NT, reinterpret_cast<const uint4*>(prev.is_vis) + NT, nsv - NT);
  }
  // dead tracks: v unchanged, yaw re-offset by THIS frame's ego yaw (:1004-1008); active ones are re-emitted below
#pragma unroll
  for (int u = 0; u < UY; ++u) {
    const int e = u * NT + tid;
    if (e < T0) { if (cp) o.vandyaw[2 * e] = pv[u]; o.vandyaw[2 * e + 1] = wrap_pi(pz[u] + ego_yaw); }
  }
  for (int base = UY * NT; base < T0; base += NT * UY) {
    double qz[UY], qv[UY];
#pragma unroll
    for (int u = 0; u < UY; ++u) {
      const int e = base + u * NT + tid;
      qz[u] = 0; qv[u] = 0;
      if (e < T0) { qz[u] = pos[e].z; if (cp) qv[u] = prev.vandyaw[2 * e]; }
    }
#pragma unroll
    for (int u = 0; u < UY; ++u) {
      const int e = base + u * NT + tid;
      if (e < T0) { if (cp) o.vandyaw[2 * e] = qv[u]; o.vandyaw[2 * e + 1] = wrap_pi(qz[u] + ego_yaw); }
    }
  }
  const int vis = (have && r.isVis) ? 1 : 0;
  float2 vb[12];                                     // the visible track's whole box (8 x 3 floats) for the output list
  if (vis) {
    const float2* src = reinterpret_cast<const float2*>(&tracks[r.k].BBox[0][0]);
#pragma unroll
    for (int e = 0; e < 12; ++e) vb[e] = src[e];
  }
  if (have) pos[r.k] = make_double4(r.x, r.y, r.yaw, 0.0);     // pass B and the general path read positions from here
  S.px[tid] = r.x; S.py[tid] = r.y; S.imax[tid] = -1;
  {
    const float fx = (float)r.x, fy = (float)r.y;
    S.t4[tid] = make_float4(fx, fy, 0.011f + 2.0e-7f * (fabsf(fx) + fabsf(fy)), __int_as_float((have && r.trackNum != 0) ? r.k : -1));
  }
  if (tid == 0) { S.ncand = 0; S.ncont = 0; S.carry = 0; }

  // ---- visible boxes in track order (the active list is sorted by track index)
  int vslot, nv;
  block_offsets(vis, 0, S.w, vslot, nv);          // (its barriers also publish the shared arrays above)
  if (vis) {
#pragma unroll
    for (int e = 0; e < 8; ++e) S.bx[vslot][e] = r.bb[e];
    S.ab[vslot] = make_float4(fminf(fminf(r.bb[0], r.bb[2]), fminf(r.bb[4], r.bb[6])), fmaxf(fmaxf(r.bb[0], r.bb[2]), fmaxf(r.bb[4], r.bb[6])),
                              fminf(fminf(r.bb[1], r.bb[3]), fminf(r.bb[5], r.bb[7])), fmaxf(fmaxf(r.bb[1], r.bb[3]), fmaxf(r.bb[5], r.bb[7])));
    S.vid[vslot] = r.k; S.h5[vslot] = 0;
  }
  __syncthreads();

  // ---- mergeOverSegmentation, pass A: imax = largest visible box index containing this (live) track
  // (track x box) pairs spread over the whole CTA: a warp takes every 8th box (broadcast loads); its lanes hold the tracks
  // jt = lane, lane + 32, ... in REGISTERS for the whole loop, so an iteration is two independent shared-memory loads and
  // compares (the previous form was one dependent load chain per pair)
  {
    const int warp = tid >> 5;
    constexpr int kPerLane = NT / 32;
    constexpr int kGrp = 8;                                // tracks a lane holds at a time (the wide variant walks the boxes twice)
#pragma unroll 1
    for (int g = 0; g < kPerLane && g * 32 < n_act0; g += kGrp) {
      float4 tj[kGrp];
#pragma unroll
      for (int u = 0; u < kGrp; ++u) {
        const int jt = lane + 32 * (g + u);
        tj[u] = (jt < n_act0) ? S.t4[jt] : make_float4(0.f, 0.f, 0.f, __int_as_float(-1));
      }
      const int nu = ((n_act0 + 31) >> 5) - g;             // lanes-worth of tracks actually present in this group (uniform)
      for (int v = warp; v < nv; v += NT / 32) {
        const float4 ab = S.ab[v];
        const int vid = S.vid[v];
#pragma unroll
        for (int u = 0; u < kGrp; ++u) {
          if (u < nu) {
            const int kj = __float_as_int(tj[u].w);
            if (kj >= 0 && kj != vid && !(tj[u].x < ab.x - tj[u].z || tj[u].x > ab.y + tj[u].z || tj[u].y < ab.z - tj[u].z || tj[u].y > ab.w + tj[u].z))
              tc_candidate<NT>(S, v, lane + 32 * (g + u));
          }
        }
      }
    }
  }
  int imax = -1;
  __syncthreads();
  {
    const int ncand = min(S.ncand, kCandCap);
    for (int e = tid; e < ncand; e += NT) {      // the exact fp64 tests, one pair per thread
      const int v = (int)(S.cand[e] >> 16), jt = (int)(S.cand[e] & 0xFFFFu);
      if (overseg_cond(S.bx[v], reinterpret_cast<const float*>(&S.ab[v]), S.px[jt], S.py[jt])) atomicMax(&S.imax[jt], S.vid[v]);
    }
  }
  __syncthreads();
  imax = max(imax, S.imax[tid]);
  // ---- pass B: has5 for the rare visible box that sits inside another one, against EVERY track (dead ones included)
  if (vis && imax >= 0 && r.trackNum != 0) S.cont[atomicAdd(&S.ncont, 1)] = (unsigned short)vslot;
  __syncthreads();
  {
    const int ncont = S.ncont;
    for (int cidx = 0; cidx < ncont; ++cidx) {
      const int v = S.cont[cidx], k = S.vid[v];
      const float4 ab = S.ab[v];
      for (int j = tid; j < T0; j += NT) {
        const double4 pj = pos[j];
        const float px = (float)pj.x, py = (float)pj.y;
        const float mg = 0.011f + 2.0e-7f * (fabsf(px) + fabsf(py));
        if (j != k && !(px < ab.x - mg || px > ab.y + mg || py < ab.z - mg || py > ab.w + mg) &&
            overseg_cond(S.bx[v], reinterpret_cast<const float*>(&S.ab[v]), pj.x, pj.y)) S.h5[v] = 1;
      }
    }
    if (ncont > 0) __syncthreads();
  }
  int trackNum = r.trackNum;
  if (have && trackNum != 0 && nv > 0) {
    const bool has5 = vis && S.h5[vslot] != 0;
    if (imax >= 0 && (!has5 || imax > r.k)) trackNum = 0;
    else if (has5) trackNum = 5;
    if (trackNum != r.trackNum) tracks[r.k].trackNum = trackNum;
  }

  // ---- outputs of the active tracks, visible boxes in track order, the surviving part of the active list
  int act = 0;
  if (have) {
    double dfi;
    const int st = emit_values(r.k, r.x, r.y, r.yaw, r.v, r.initx, r.inity, r.mp0, r.mp1, r.mp2, trackNum, r.lifetime, r.isStatic, vis, ego_yaw, o, pos, dfi, P);
    tracks[r.k].distFromInit = dfi;
    if (st && !r.isStatic) tracks[r.k].isStatic = 1;
    act = (trackNum != 0 || vis) ? 1 : 0;
  }
  if (vis) {
    float2* dst = reinterpret_cast<float2*>(o.vis_bb + (size_t)vslot * 24);
#pragma unroll
    for (int e = 0; e < 12; ++e) dst[e] = vb[e];
  }
  int aex, atot;
  block_offsets(0, act, S.w, aex, atot);
  const int n_keep = atot >> 16;
  if (act) act_list[aex >> 16] = r.k;

  // ---- spawn one UKF per unmatched box, in box order (:972-989); the spawning thread also emits the new track
  for (int b0 = 0; b0 < M; b0 += NT) {
    const int b = b0 + tid;
    const int un = (b < M && (b0 == 0 ? fs0 : first_setter[b]) == INT_MAX) ? 1 : 0;
    int ex, tot;
    block_offsets(un, 0, S.w, ex, tot);
    const int p = T0 + S.carry + ex;
    if (un && p < max_tracks) {
      double cx, cy;
      if (b0 == 0) cp_from_corners(bc[0], bc[1], bc[2], bc[3], bc[4], bc[5], bc[6], bc[7], cx, cy);
      else cp_from_box(boxes + (size_t)b * 24, cx, cy);
      ukf_initialize(tracks[p], cx, cy, P);
      double dfi;
      emit_values(p, cx, cy, 0.0, 0.0, 0.0, 0.0, P.mode_prob0(0), P.mode_prob0(1), P.mode_prob0(2), 1, 0, 0, 0, ego_yaw, o, pos, dfi, P);
      tracks[p].distFromInit = dfi;
      act_list[n_keep + (p - T0)] = p;
    }
    if (b < M) first_setter[b] = INT_MAX;        // ready for the next frame
    __syncthreads();
    if (tid == 0) S.carry += tot;
    __syncthreads();
  }
  int T = T0 + S.carry;
  if (T > max_tracks) T = max_tracks;
  if (tid == 0) {
    trk[CNT_N_TRACKS] = T; trk[CNT_N_VIS] = nv; trk[CNT_N_ACT] = n_keep + (T - T0);
    o.hdr[HDR_N_ELEV] = hdr_in[0]; o.hdr[HDR_N_GROUND] = hdr_in[1]; o.hdr[HDR_NUM_CLUSTER] = hdr_in[2];
    o.hdr[HDR_N_BOXES] = M; o.hdr[HDR_N_TRACKS] = T; o.hdr[HDR_N_VIS] = nv; o.hdr[HDR_ERROR] = hdr_in[3];
    o.hdr[HDR_WARN] = (T0 + S.carry > max_tracks) ? (int)LMOT_WARN_TRACK_TABLE_FULL : 0;   // existing tracks' outputs stay valid: a warning, not an error
    o.hdr[HDR_N_ACT] = n_keep + (T - T0);
    det[CNT_ERROR] = 0;
  }
}

// ------------------------------------------------------------------------------------------------ TC: track retirement
// (lmot_set_track_retirement, DESIGN.md section 6e).  The retire-capable instantiations of TC end every step with this phase: after
// the step's outputs, before done_at_exit counts the step -- the next step's TA and publish_kernel poll that count, so neither ever
// sees a half-compacted table.  Per table of the launch:
//   on      the table numbers its tracks: this step's ID rows go into the result block (pre-compaction order, the order of its
//           outputs); the spawns take the next values of the table's spawn counter;
//   init    the table's IDs are still its row indices (no retirement since its last reset / load / open): derived from the rows;
//   retire  remove every row with trackNum 0.  The survivors move down in place, in order: their records, packed positions (d_pos)
//           and IDs; the active list becomes the identity over them.  A retained table has no dead rows, so TA / TB run unchanged.
struct RetPrm { long long* ids; long long* next; long long* out_ids; int* keep; int on, init, retire; };

// the default kernels: no phase at all
struct NoRetire {
  __device__ __forceinline__ void begin(const int*) {}
  __device__ __forceinline__ void end(bool, TrackState*, int*, const OutPtrs&, int*, double4*) {}
};

template <int NT>
__device__ __noinline__ void retire_phase(const RetPrm& p, int T0, TrackState* __restrict__ tracks, int* __restrict__ trk,
                                          const int* __restrict__ track_manage, int* __restrict__ act_list, double4* __restrict__ pos) {
  __shared__ int s_w[33];
  __shared__ int s_carry, s_first;
  const int tid = threadIdx.x;
  if (tid == 0) { s_carry = 0; s_first = INT_MAX; }
  __syncthreads();                               // (also: every record and output of this step is written)
  const int T = trk[CNT_N_TRACKS];
  const int n_new = T > T0 ? T - T0 : 0;
  const long long next = p.init ? (long long)T0 : *p.next;
  // ID rows; with retirement the stable in-place compaction of IDs and positions (a tile is read completely -- the barrier inside
  // block_offsets -- before anything at or below its range is written) and the list of kept rows
  for (int q0 = 0; q0 < T; q0 += NT) {
    const int i = q0 + tid;
    long long id = 0;
    int keep = 0;
    double4 ps = make_double4(0.0, 0.0, 0.0, 0.0);
    if (i < T) {
      id = (i >= T0) ? next + (i - T0) : (p.init ? (long long)i : p.ids[i]);
      p.out_ids[i] = id;
      keep = track_manage[i] != 0 ? 1 : 0;
      ps = pos[i];
    }
    if (!p.retire) {                             // (uniform) the table keeps its rows: only the spawns' IDs are new
      if (i < T && i >= T0) p.ids[i] = id;
      continue;
    }
    int ex, tot;
    block_offsets(keep, 0, s_w, ex, tot);
    if (keep) {
      const int d = s_carry + ex;
      p.ids[d] = id; pos[d] = ps; p.keep[d] = i; act_list[d] = d;
      if (d != i) atomicMin(&s_first, d);
    }
    __syncthreads();
    if (tid == 0) s_carry += tot;
    __syncthreads();
  }
  const int n = p.retire ? s_carry : T;
  if (p.retire) {
    // the records of the kept rows from the first moved one on, as one stream of words: dst word e <- src word keep[e / W] * W + e % W,
    // src >= dst throughout, so a chunk read completely before it is written never overwrites a word a later chunk still reads
    using Word = typename std::conditional<sizeof(TrackState) % 16 == 0, uint4, uint2>::type;
    constexpr int W = (int)(sizeof(TrackState) / sizeof(Word)), U = 4;
    static_assert(sizeof(TrackState) % sizeof(Word) == 0, "TrackState is a whole number of words");
    Word* rec = reinterpret_cast<Word*>(tracks);
    const int f = min(s_first, n);
    const int e1 = n * W;
    for (int base = f * W; base < e1; base += NT * U) {
      Word v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int e = base + u * NT + tid;
        if (e < e1) { const int d = e / W; v[u] = rec[(size_t)p.keep[d] * W + (e - d * W)]; }
      }
      __syncthreads();
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int e = base + u * NT + tid;
        if (e < e1) rec[e] = v[u];
      }
      __syncthreads();
    }
  }
  if (tid == 0) {
    *p.next = next + n_new;
    if (p.retire) { trk[CNT_N_TRACKS] = n; trk[CNT_N_ACT] = n; }
  }
}

template <int NT>
struct Retire {
  const RetPrm& p;
  int T0;
  __device__ __forceinline__ void begin(const int* trk) { T0 = trk[CNT_N_TRACKS]; }
  // fresh: the step rebuilt the table from nothing (the reference's first-call quirk): every row is a spawn
  __device__ __forceinline__ void end(bool fresh, TrackState* tracks, int* trk, const OutPtrs& o, int* act_list, double4* pos) {
    if (p.on) retire_phase<NT>(p, fresh ? 0 : T0, tracks, trk, o.track_manage, act_list, pos);
  }
};

// TC.  The track table only ever grows (dead tracks keep their slot, like targets_; retirement is the phase above), and the reference re-emits every track
// every frame.  Everything here that walks the table does so through coalesced side arrays; everything that touches the
// 1.6 KB TrackState records is limited to the ACTIVE tracks:
//   * the per-track outputs of a dead track never change, so the frame's result block starts as a copy of the previous
//     frame's block (device to device, 34 B per track, coalesced) and only active / new tracks are re-emitted;
//   * mergeOverSegmentation needs the position of EVERY track (dead ones included, like the reference), and the output yaw
//     of every track is its state's yaw plus THIS frame's ego yaw: `pos`, a packed (x, y, yaw) per track, refreshed for the
//     active tracks only.
// `full` (first step after the table was written from the host): everything is rebuilt from the records.
// P: DefTC / TunTC; R: NoRetire / Retire<NT>
template <int NT, class TP, class RH = NoRetire>
__device__ __forceinline__ void
spawn_output_body(TrackState* __restrict__ tracks, int* __restrict__ trk, int* __restrict__ det, const float* __restrict__ boxes,
                  const float* __restrict__ boxes_pub, int* __restrict__ first_setter, int* __restrict__ imax_arr, int* __restrict__ vis_list,
                  uint8_t* __restrict__ has5_arr, int first_frame, int compat_first, double ego_yaw, int max_tracks, const OutPtrs& o,
                  const OutPtrs& prev, int full, int* __restrict__ act_list, double4* __restrict__ pos, const ActSummary* __restrict__ summary,
                  int* __restrict__ det_sem, unsigned* __restrict__ tc_seq, const TP& P, RH R = RH{}) {
  pdl_launch_dependents();                 // the next frame's gate kernel may become resident
  pdl_wait();                              // TB has finished
  R.begin(trk);
  // every exit: this step's results are complete -> count it (release); publish_kernel, on its own stream, polls the count
  // instead of waiting for a stream event, so that nothing but kernels sits on the tracker stream
  struct Done { unsigned* p; __device__ ~Done() { __syncthreads(); if (threadIdx.x == 0) { __threadfence(); atomicAdd(p, 1u); } } } done_at_exit{tc_seq};
  if (det_sem && threadIdx.x == 0) atomicSub(det_sem, 1);     // this frame's detection results are being consumed (posted by box_fit_kernel)
  if (!full && !(first_frame && compat_first) && trk[CNT_N_ACT] <= NT) {
    extern __shared__ __align__(16) unsigned char tc_dyn[];          // sizeof(TCFastShared<NT>), tracker_launch
    TCFastShared<NT>& s_fast = *reinterpret_cast<TCFastShared<NT>*>(tc_dyn);
    const int M = det[CNT_N_BOXES];
    tc_fast<NT>(s_fast, tracks, trk, det, boxes, boxes_pub, first_setter, ego_yaw, max_tracks, o, prev, act_list, pos, summary, trk[CNT_N_TRACKS], trk[CNT_N_ACT], M, P);
    R.end(false, tracks, trk, o, act_list, pos);
    return;
  }
  __shared__ int s_w[33];
  __shared__ int s_carry, s_carry2, s_nvis, s_ncand, s_ncont;
  __shared__ unsigned char s_cont[kVisChunk];           // visible boxes that sit inside another visible box
  __shared__ __align__(16) float s_bx[kVisChunk][8];
  __shared__ __align__(16) float4 s_ab[kVisChunk];     // bounds of the box: min x, max x, min y, max y
  __shared__ int s_vid[kVisChunk];
  __shared__ unsigned char s_h5[kVisChunk];
  __shared__ unsigned s_cand[kCandCap];                 // (visible slot << 24) | track index
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int T0 = trk[CNT_N_TRACKS];
  const int n_act0 = trk[CNT_N_ACT];
  const int M = det[CNT_N_BOXES];
  if (tid == 0) { s_carry = 0; s_carry2 = 0; s_nvis = 0; }
  __syncthreads();

  if (first_frame && compat_first) {
    // :741-795 -- the first call spawns ONE track, from box #1, at a hard-coded position
    if (tid == 0) {
      int T = 0;
      if (M >= 2) {
        ukf_initialize(tracks[0], -1.5125, -8.975, P);
        o.targets[0] = (float)-1.5125; o.targets[1] = (float)-8.975; o.targets[2] = (float)(-1.73 / 2);
        o.vandyaw[0] = 0; o.vandyaw[1] = 0; o.is_static[0] = 0; o.is_vis[0] = 0; o.track_manage[0] = 1;
        pos[0] = make_double4(-1.5125, -8.975, 0.0, 0.0);
        T = 1;
      }
      trk[CNT_N_TRACKS] = T; trk[CNT_N_VIS] = 0; trk[CNT_N_ACT] = T; act_list[0] = 0;
      o.hdr[HDR_N_ELEV] = det[CNT_N_ELEV]; o.hdr[HDR_N_GROUND] = det[CNT_N_GROUND]; o.hdr[HDR_NUM_CLUSTER] = det[CNT_NUM_CLUSTER];
      o.hdr[HDR_N_BOXES] = M; o.hdr[HDR_N_TRACKS] = T; o.hdr[HDR_N_VIS] = 0; o.hdr[HDR_ERROR] = det[CNT_ERROR]; o.hdr[HDR_WARN] = 0; o.hdr[HDR_N_ACT] = T;
      det[CNT_ERROR] = 0;
    }
    for (int b = tid; b < M; b += NT) first_setter[b] = INT_MAX;
    for (int e = tid; e < M * 24; e += NT) o.boxes[e] = boxes_pub[e];
    R.end(true, tracks, trk, o, act_list, pos);
    return;
  }
  for (int e = tid; e < M * 24; e += NT) o.boxes[e] = boxes_pub[e];     // the frame's box list travels with its results

  // ---- start the frame's result block from the previous one (dead tracks: unchanged), refresh the positions of the
  // active tracks, collect the visible ones (a subset of the active list, which is sorted by track index)
  if (!full) {
    const bool cp = prev.targets != o.targets;   // same block (result_ring == 1, or the synchronous entry points): patch in place
    if (cp) {
      for (int e = tid; e < (T0 * 12 + 15) / 16; e += NT) reinterpret_cast<uint4*>(o.targets)[e] = reinterpret_cast<const uint4*>(prev.targets)[e];
      for (int e = tid; e < (T0 * 4 + 15) / 16; e += NT) reinterpret_cast<uint4*>(o.track_manage)[e] = reinterpret_cast<const uint4*>(prev.track_manage)[e];
      for (int e = tid; e < (T0 + 15) / 16; e += NT) {
        reinterpret_cast<uint4*>(o.is_static)[e] = reinterpret_cast<const uint4*>(prev.is_static)[e];
        reinterpret_cast<uint4*>(o.is_vis)[e] = reinterpret_cast<const uint4*>(prev.is_vis)[e];
      }
    }
    for (int e = tid; e < T0; e += NT) {      // v is the state's; the yaw is re-offset by THIS frame's ego yaw for every track (:1004-1008)
      if (cp) o.vandyaw[2 * e] = prev.vandyaw[2 * e];
      o.vandyaw[2 * e + 1] = wrap_pi(pos[e].z + ego_yaw);
    }
  }
  const int n_scan = full ? T0 : n_act0;       // entries to visit: the whole table, or the active list
  for (int q0 = 0; q0 < n_scan; q0 += NT) {
    const int q = q0 + tid;
    int vis = 0, k = 0;
    if (q < n_scan) {
      k = full ? q : act_list[q];
      const TrackState& t = tracks[k];
      pos[k] = make_double4(t.x[0][0], t.x[0][1], t.x[0][3], 0.0);
      vis = t.isVisBB ? 1 : 0;
    }
    int ex, tot;
    block_offsets(vis, 0, s_w, ex, tot);
    if (vis) vis_list[s_nvis + ex] = k;
    __syncthreads();
    if (tid == 0) s_nvis += tot;
    __syncthreads();
  }
  const int nv = s_nvis;

  // ---- mergeOverSegmentation (:666-700), folded into this kernel.  The sequential double loop writes trackNum[i]=5,
  // trackNum[j]=0 for every hit (i,j) with i visible ("box i contains the position of track j"); the value that survives at
  // index k is the write with the largest (i,j) key: 0 if some visible i > k contains k, else 5 if k (visible) contains
  // anybody, else unchanged.  Only LIVE k can change (0 -> 0 is a no-op), and a visible track already has trackNum 5 when it
  // gets here (associateBB requires 5, a validated measurement keeps it), so "k contains anybody" (has5) only matters for a
  // visible k that is itself inside another visible box.  Hence:
  //   pass A  imax[j] = largest visible i containing j, for the LIVE tracks j only (active list x visible boxes);
  //   pass B  has5[k] for the rare visible k with imax[k] >= 0: those alone are tested against EVERY track, dead ones
  //           included like the reference (positions from the packed array, coalesced).
  // Visible boxes + bounds are staged in shared memory; a single-precision bounds pre-test (the margin covers the rounding
  // of the position to float) selects the few pairs that get the exact fp64 test, queued so that they run one per THREAD.
  auto stage_boxes = [&](int v0, int nc) {
    for (int e = tid; e < nc * 8; e += NT) { const int v = e >> 3, q = e & 7; s_bx[v][q] = tracks[vis_list[v0 + v]].BBox[q >> 1][q & 1]; }
    if (tid == 0) { s_ncand = 0; s_ncont = 0; }
    __syncthreads();
    for (int v = tid; v < nc; v += NT) {
      const float* c = s_bx[v];
      s_ab[v] = make_float4(fminf(fminf(c[0], c[2]), fminf(c[4], c[6])), fmaxf(fmaxf(c[0], c[2]), fmaxf(c[4], c[6])),
                            fminf(fminf(c[1], c[3]), fminf(c[5], c[7])), fmaxf(fmaxf(c[1], c[3]), fmaxf(c[5], c[7])));
      s_vid[v] = vis_list[v0 + v]; s_h5[v] = 0;
    }
    __syncthreads();
  };
  if (nv > 0)
    for (int q = tid; q < n_scan; q += NT) imax_arr[full ? q : act_list[q]] = -1;
  __syncthreads();
  for (int v0 = 0; v0 < nv; v0 += kVisChunk) {                 // pass A
    const int nc = min(kVisChunk, nv - v0);
    stage_boxes(v0, nc);
    for (int q = tid; q < n_scan; q += NT) {
      const int j = full ? q : act_list[q];
      if (tracks[j].trackNum == 0) continue;                    // dead (stale-visible entry of the list): cannot change
      const double4 pj = pos[j];
      const float px = (float)pj.x, py = (float)pj.y;
      const float mg = 0.011f + 2.0e-7f * (fabsf(px) + fabsf(py));
      for (int v = 0; v < nc; ++v) {
        const float4 ab = s_ab[v];
        if (!(px < ab.x - mg || px > ab.y + mg || py < ab.z - mg || py > ab.w + mg) && s_vid[v] != j) {
          const int slot = atomicAdd(&s_ncand, 1);
          if (slot < kCandCap) s_cand[slot] = ((unsigned)v << 24) | (unsigned)j;
          else if (overseg_cond(s_bx[v], reinterpret_cast<const float*>(&s_ab[v]), pj.x, pj.y)) atomicMax(&imax_arr[j], s_vid[v]);
        }
      }
    }
    __syncthreads();
    const int ncand = min(s_ncand, kCandCap);
    for (int e = tid; e < ncand; e += NT) {
      const int v = (int)(s_cand[e] >> 24), j = (int)(s_cand[e] & 0xFFFFFFu);
      const double4 pj = pos[j];
      if (overseg_cond(s_bx[v], reinterpret_cast<const float*>(&s_ab[v]), pj.x, pj.y)) atomicMax(&imax_arr[j], s_vid[v]);
    }
    __syncthreads();
  }
  for (int v0 = 0; v0 < nv; v0 += kVisChunk) {                 // pass B
    const int nc = min(kVisChunk, nv - v0);
    if (nv > kVisChunk) stage_boxes(v0, nc);                    // otherwise the only chunk is still staged
    for (int v = tid; v < nc; v += NT)
      if (imax_arr[s_vid[v]] >= 0) s_cont[atomicAdd(&s_ncont, 1)] = (unsigned char)v;
    __syncthreads();
    const int ncont = s_ncont;
    for (int cidx = 0; cidx < ncont; ++cidx) {
      const int v = s_cont[cidx], k = s_vid[v];
      const float4 ab = s_ab[v];
      for (int j = tid; j < T0; j += NT) {
        const double4 pj = pos[j];
        const float px = (float)pj.x, py = (float)pj.y;
        const float mg = 0.011f + 2.0e-7f * (fabsf(px) + fabsf(py));
        if (j != k && !(px < ab.x - mg || px > ab.y + mg || py < ab.z - mg || py > ab.w + mg) &&
            overseg_cond(s_bx[v], reinterpret_cast<const float*>(&s_ab[v]), pj.x, pj.y)) s_h5[v] = 1;
      }
    }
    __syncthreads();
    for (int v = tid; v < nc; v += NT) has5_arr[s_vid[v]] = s_h5[v];
    __syncthreads();
  }
  if (nv > 0) {       // only live tracks can change (0 -> 0 is a no-op, 5 needs a visible, hence live, track)
    for (int q0 = 0; q0 < n_scan; q0 += NT) {
      const int q = q0 + tid;
      if (q < n_scan) {
        const int k = full ? q : act_list[q];
        if (tracks[k].trackNum != 0) {
          const int imax = imax_arr[k];
          const bool has5 = tracks[k].isVisBB && has5_arr[k] != 0;
          if (imax >= 0 && (!has5 || imax > k)) tracks[k].trackNum = 0;
          else if (has5) tracks[k].trackNum = 5;
        }
      }
    }
  }
  __syncthreads();

  // ---- spawn one UKF per unmatched box, in box order (:972-989)
  for (int b0 = 0; b0 < M; b0 += NT) {
    const int b = b0 + tid;
    const int un = (b < M && first_setter[b] == INT_MAX) ? 1 : 0;
    int ex, tot;
    block_offsets(un, 0, s_w, ex, tot);
    const int p = T0 + s_carry + ex;
    if (un && p < max_tracks) {
      double cx, cy;
      cp_from_box(boxes + (size_t)b * 24, cx, cy);
      ukf_initialize(tracks[p], cx, cy, P);
    }
    if (b < M) first_setter[b] = INT_MAX;        // ready for the next frame
    __syncthreads();
    if (tid == 0) s_carry += tot;
    __syncthreads();
  }
  int T = T0 + s_carry;
  const int table_full = (T > max_tracks) ? 1 : 0;      // boxes beyond the table's capacity spawn no track (warning; every existing track is still updated and emitted)
  if (T > max_tracks) T = max_tracks;
  __syncthreads();
  if (tid == 0) s_carry = 0;
  __syncthreads();

  // ---- outputs (:995-1081) of the active and the new tracks, visible boxes in track order, next frame's active list
  // (stable in-place compaction: a tile is read completely before anything at or below its range is written)
  const int n_new = T - T0;
  const int n_emit = n_scan + n_new;
  for (int q0 = 0; q0 < n_emit; q0 += NT) {
    const int q = q0 + tid;
    int vis = 0, act = 0, i = 0;
    if (q < n_emit) {
      i = (q < n_scan) ? (full ? q : act_list[q]) : T0 + (q - n_scan);
      TrackState& t = tracks[i];
      vis = emit_track(t, i, ego_yaw, o, pos, P);
      act = (t.trackNum != 0 || vis) ? 1 : 0;
    }
    int ex, tot;
    block_offsets(vis, act, s_w, ex, tot);
    if (act) act_list[s_carry2 + (ex >> 16)] = i;
    if (vis) {
      const int p = s_carry + (ex & 0xFFFF);
      const float2* src = reinterpret_cast<const float2*>(&tracks[i].BBox[0][0]);
      float2* dst = reinterpret_cast<float2*>(o.vis_bb + (size_t)p * 24);
#pragma unroll
      for (int e = 0; e < 12; ++e) dst[e] = src[e];
    }
    __syncthreads();
    if (tid == 0) { s_carry += tot & 0xFFFF; s_carry2 += tot >> 16; }
    __syncthreads();
  }
  if (tid == 0) {
    trk[CNT_N_TRACKS] = T; trk[CNT_N_VIS] = s_carry; trk[CNT_N_ACT] = s_carry2;
    o.hdr[HDR_N_ELEV] = det[CNT_N_ELEV]; o.hdr[HDR_N_GROUND] = det[CNT_N_GROUND]; o.hdr[HDR_NUM_CLUSTER] = det[CNT_NUM_CLUSTER];
    o.hdr[HDR_N_BOXES] = M; o.hdr[HDR_N_TRACKS] = T; o.hdr[HDR_N_VIS] = s_carry; o.hdr[HDR_ERROR] = det[CNT_ERROR];
    o.hdr[HDR_WARN] = table_full ? (int)LMOT_WARN_TRACK_TABLE_FULL : 0;
    o.hdr[HDR_N_ACT] = s_carry2;
    det[CNT_ERROR] = 0;
  }
  R.end(false, tracks, trk, o, act_list, pos);
}

template <int NT>
__global__ void __launch_bounds__(NT, NT == kTCThreads ? 2 : 1)
spawn_output_kernel(TrackState* __restrict__ tracks, int* __restrict__ trk, int* __restrict__ det, const float* __restrict__ boxes,
                    const float* __restrict__ boxes_pub, int* __restrict__ first_setter, int* __restrict__ imax_arr, int* __restrict__ vis_list,
                    uint8_t* __restrict__ has5_arr, int first_frame, int compat_first, double ego_yaw, int max_tracks, OutPtrs o,
                    OutPtrs prev, int full, int* __restrict__ act_list, double4* __restrict__ pos, const ActSummary* __restrict__ summary,
                    int* __restrict__ det_sem, unsigned* __restrict__ tc_seq) {
  spawn_output_body<NT>(tracks, trk, det, boxes, boxes_pub, first_setter, imax_arr, vis_list, has5_arr, first_frame, compat_first, ego_yaw,
                        max_tracks, o, prev, full, act_list, pos, summary, det_sem, tc_seq, DefTC{});
}

// sequence ticks: one CTA per sequence (blockIdx.x); each picks the fast or the general path from its own sequence's counts
struct TCSeq {
  TrackState* tracks; int* trk; int* det; const float* boxes; const float* boxes_pub; int* first_setter; int* imax_arr; int* vis_list;
  uint8_t* has5_arr; int* act_list; double4* pos; const ActSummary* summary; int* det_sem; unsigned* tc_seq;
  OutPtrs o, prev;
  double ego_yaw; int first_frame, full;
};
struct TCSeqParams { TCSeq s[kMaxBatch]; int compat_first, max_tracks; };
static_assert(sizeof(TCSeqParams) <= 4096, "kernel parameter block");

template <int NT>
__global__ void __launch_bounds__(NT, NT == kTCThreads ? 2 : 1)
spawn_output_seq_kernel(const __grid_constant__ TCSeqParams p) {
  const TCSeq& q = p.s[blockIdx.x];
  spawn_output_body<NT>(q.tracks, q.trk, q.det, q.boxes, q.boxes_pub, q.first_setter, q.imax_arr, q.vis_list, q.has5_arr, q.first_frame,
                        p.compat_first, q.ego_yaw, p.max_tracks, q.o, q.prev, q.full, q.act_list, q.pos, q.summary, q.det_sem, q.tc_seq, DefTC{});
}

// ... every other chain (as imm_predict_gate_seq_tuned_kernel's): each table with its own slice, and the retire-capable TC (track
// retirement / track IDs, lmot_set_track_retirement) with each table's own flags -- all off: no phase.  One TC on the tuned parameter
// source (bit-identical to the defaults at the default values, DESIGN.md section 6c) instead of a tuned and a retire variant.
// (the _seq block + a parameter slice per table, then a retire phase per table)
struct TCSeqPrmParams { TCSeqParams b; TCPrm tp[kMaxBatch]; };
struct TCSeqTunedParams { TCSeqPrmParams t; RetPrm rp[kMaxBatch]; };
static_assert(sizeof(TCSeqTunedParams) <= 4096, "kernel parameter block");

template <int NT>
__global__ void __launch_bounds__(NT, NT == kTCThreads ? 2 : 1)
spawn_output_seq_tuned_kernel(const __grid_constant__ TCSeqTunedParams p) {
  const TCSeq& q = p.t.b.s[blockIdx.x];
  spawn_output_body<NT>(q.tracks, q.trk, q.det, q.boxes, q.boxes_pub, q.first_setter, q.imax_arr, q.vis_list, q.has5_arr, q.first_frame,
                        p.t.b.compat_first, q.ego_yaw, p.t.b.max_tracks, q.o, q.prev, q.full, q.act_list, q.pos, q.summary, q.det_sem, q.tc_seq,
                        TunTC{p.t.tp[blockIdx.x]}, Retire<NT>{p.rp[blockIdx.x], 0});
}

// device copy of a frame's results -> pinned, device-mapped host block.  16 bytes per thread, consecutive threads ->
// consecutive addresses: every store instruction of a warp is four full 128-byte lines on the PCIe side.
__device__ __forceinline__ void copy16(void* dst, const void* src, size_t bytes, int tid, int nthreads) {
  const uint4* s = reinterpret_cast<const uint4*>(src);
  uint4* d = reinterpret_cast<uint4*>(dst);
  const size_t n16 = (bytes + 15) / 16;                 // the blocks have 16 bytes of slack
  for (size_t e = tid; e < n16; e += nthreads) d[e] = s[e];
}

// p' = M p as pcl::transformPointCloud evaluates it with the Eigen::Matrix4f pcl_ros builds from a tf::Transform: single
// precision, ((m0 x + m1 y) + m2 z) + m3 per row, no contraction.  Planar rigid transforms only: row 2 is (0, 0, 1, 0).
__device__ __forceinline__ void xf_apply(const Xf2& M, float x, float y, float z, float& ox, float& oy, float& oz) {
  ox = fadd(fadd(fadd(fmul(M.m[0], x), fmul(M.m[1], y)), fmul(0.f, z)), M.m[2]);
  oy = fadd(fadd(fadd(fmul(M.m[3], x), fmul(M.m[4], y)), fmul(0.f, z)), M.m[5]);
  oz = fadd(fadd(fadd(fmul(0.f, x), fmul(0.f, y)), fmul(1.f, z)), 0.f);
}

constexpr int kPubThreads = 128;    // small on purpose: it may sit on an SM polling while detection kernels need that SM's registers
__device__ __forceinline__ void
publish_body(const OutPtrs& d, const OutPtrs& h, const unsigned* __restrict__ tc_seq, unsigned want, unsigned spin_limit, const Xf2& back) {
  const int tid = threadIdx.x;
  if (tid == 0) {              // wait until `want` tracker steps have completed (spawn_output_kernel counts them)
    unsigned spin = 0, v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(tc_seq) : "memory");
      if (spin_limit && ++spin > spin_limit) __trap();
    } while ((int)(v - want) < 0);
  }
  __syncthreads();
  const int T = d.hdr[HDR_N_TRACKS], V = d.hdr[HDR_N_VIS], M = d.hdr[HDR_N_BOXES];
  copy16(h.boxes, d.boxes, (size_t)M * 96, tid, kPubThreads);
  if (!back.on) {
    copy16(h.targets, d.targets, (size_t)T * 12, tid, kPubThreads);
    copy16(h.vis_bb, d.vis_bb, (size_t)V * 96, tid, kPubThreads);
  } else {
    // global frame -> sensor frame for what the node publishes (tracking/main.cpp:182-195); the device block stays global:
    // the next step starts from it
    for (int i = tid; i < T; i += kPubThreads) xf_apply(back, d.targets[3 * i], d.targets[3 * i + 1], d.targets[3 * i + 2], h.targets[3 * i], h.targets[3 * i + 1], h.targets[3 * i + 2]);
    for (int i = tid; i < V * 8; i += kPubThreads) xf_apply(back, d.vis_bb[3 * i], d.vis_bb[3 * i + 1], d.vis_bb[3 * i + 2], h.vis_bb[3 * i], h.vis_bb[3 * i + 1], h.vis_bb[3 * i + 2]);
  }
  copy16(h.vandyaw, d.vandyaw, (size_t)T * 16, tid, kPubThreads);
  copy16(h.track_manage, d.track_manage, (size_t)T * 4, tid, kPubThreads);
  copy16(h.is_static, d.is_static, (size_t)T, tid, kPubThreads);
  copy16(h.is_vis, d.is_vis, (size_t)T, tid, kPubThreads);
  copy16(h.hdr, d.hdr, HDR_COUNT * sizeof(int), tid, kPubThreads);
}

__global__ void __launch_bounds__(kPubThreads)
publish_kernel(OutPtrs d, OutPtrs h, const unsigned* __restrict__ tc_seq, unsigned want, unsigned spin_limit, Xf2 back) {
  publish_body(d, h, tc_seq, want, spin_limit, back);
}

// sequence ticks: one CTA per sequence, each waits for its own sequence's step count
struct PubSeq { OutPtrs d, h; const unsigned* tc_seq; unsigned want; Xf2 back; };
struct PubSeqParams { PubSeq s[kMaxBatch]; unsigned spin_limit; };
static_assert(sizeof(PubSeqParams) <= 4096, "kernel parameter block");

__global__ void __launch_bounds__(kPubThreads)
publish_seq_kernel(const __grid_constant__ PubSeqParams p) {
  const PubSeq& q = p.s[blockIdx.x];
  publish_body(q.d, q.h, q.tc_seq, q.want, p.spin_limit, q.back);
}

// the ID rows of results whose table numbers its tracks (retire-capable TC): launched on the publish stream right behind the publish
// launch of the same step, which has waited for it; one CTA per result block (nullptr: the block's IDs are its row indices)
struct PubIds { const int* hdr; const long long* d_ids; long long* h_ids; };
struct PubIdsParams { PubIds s[kMaxBatch]; };

__global__ void __launch_bounds__(kPubThreads)
publish_ids_kernel(const __grid_constant__ PubIdsParams p) {
  const PubIds& q = p.s[blockIdx.x];
  if (q.d_ids) copy16(q.h_ids, q.d_ids, (size_t)q.hdr[HDR_N_TRACKS] * sizeof(long long), threadIdx.x, kPubThreads);
}

// lmot_params.global_frame: the frame's boxes (sensor frame) -> the dead-reckoned global frame the tracker works in
// (tracking/main.cpp:142-158: pcl_ros::transformPointCloud("/global", bBoxes[i], ...)).  One CTA; also takes over posting the
// detection semaphore from box fitting, because the tracker must not start before this list exists.
__device__ __forceinline__ void
boxes_to_global_body(const float* __restrict__ boxes, const int* __restrict__ det, float* __restrict__ boxes_g, const Xf2& fwd, int* __restrict__ det_sem) {
  const int M = det[CNT_N_BOXES];
  for (int i = threadIdx.x; i < M * 8; i += 256) xf_apply(fwd, boxes[3 * i], boxes[3 * i + 1], boxes[3 * i + 2], boxes_g[3 * i], boxes_g[3 * i + 1], boxes_g[3 * i + 2]);
  if (det_sem) {
    __syncthreads();
    if (threadIdx.x == 0) { __threadfence(); atomicAdd(det_sem, 1); }
  }
}

__global__ void __launch_bounds__(256)
boxes_to_global_kernel(const float* __restrict__ boxes, const int* __restrict__ det, float* __restrict__ boxes_g, Xf2 fwd, int* __restrict__ det_sem) {
  boxes_to_global_body(boxes, det, boxes_g, fwd, det_sem);
}

// sequence ticks: one CTA per sequence, each with its own ego pose; posts its sequence's slot semaphore
struct GlobalSeq { const float* boxes; const int* det; float* boxes_g; int* det_sem; Xf2 fwd; };
struct GlobalSeqParams { GlobalSeq s[kMaxBatch]; };

__global__ void __launch_bounds__(256)
boxes_to_global_seq_kernel(const __grid_constant__ GlobalSeqParams p) {
  const GlobalSeq& q = p.s[blockIdx.x];
  boxes_to_global_body(q.boxes, q.det, q.boxes_g, q.fwd, q.det_sem);
}

// detection-only submissions: the box list of the slot -> the result's host block
__global__ void __launch_bounds__(256)
publish_boxes_kernel(const float* __restrict__ d_boxes, const int* __restrict__ det, float* __restrict__ h_boxes) {
  copy16(h_boxes, d_boxes, (size_t)det[CNT_N_BOXES] * 96, threadIdx.x, 256);
}

// rebuilds the active-track list after the table was written from the host (load / reset / broadcast from another rank)
__global__ void build_active_kernel(const TrackState* __restrict__ tracks, int* __restrict__ trk, int* __restrict__ act_list) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < trk[CNT_N_TRACKS] && (tracks[k].trackNum != 0 || tracks[k].isVisBB)) act_list[atomicAdd(&trk[CNT_N_ACT], 1)] = k;
}

__global__ void fill_int_kernel(int* p, int n, int v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// each stage's slice of a table's parameters
TAPrm ta_prm(const lmot_tracker_params& p) {
  TAPrm a;
  a.gamma_g = p.gamma_g; a.std_las_x = p.std_las_x; a.std_las_y = p.std_las_y;
  for (int m = 0; m < 3; ++m) { a.std_a[m] = p.std_a[m]; a.std_yawdd[m] = p.std_yawdd[m]; }
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) a.trans[i][j] = p.trans[i][j];
  return a;
}
TBPrm tb_prm(const lmot_tracker_params& p) {
  return TBPrm{p.gamma_g, p.p_g, p.p_d, p.distance_thres, p.bb_yaw_change_thres, p.second_init_v, p.lifetime_thres};
}
// the retire phase's flags and arrays of table t for a step into result block r; r->ids: the step writes ID rows.  A table whose IDs
// are its row indices and that does not retire needs neither (the default kernels); after a retiring step its IDs stay the table's own
// until reset / load / reopen.
RetPrm ret_prm(const Ctx* c, Tracker& t, Result* r) {
  RetPrm a{t.d_ids, t.d_ids + c->prm.max_tracks, r->d_ids, t.d_live_list, 0, 0, 0};
  a.retire = t.retire ? 1 : 0;
  a.on = (t.retire || !t.ids_identity) ? 1 : 0;
  a.init = t.ids_identity ? 1 : 0;
  r->ids = a.on != 0;
  if (t.retire) t.ids_identity = false;
  return a;
}

TCPrm tc_prm(const lmot_tracker_params& p) {
  TCPrm a;
  for (int i = 0; i < 5; ++i) a.p0_diag[i] = p.p0_diag[i];
  for (int m = 0; m < 3; ++m) a.mode_prob0[m] = p.mode_prob0[m];
  a.static_dist = p.static_dist; a.static_lifetime = p.static_lifetime;
  return a;
}

}  // namespace

int tracker_alloc(Ctx* c, Tracker& t) {
  const int TC = c->prm.max_tracks, MB = c->prm.max_boxes;
  c->gate_words = (MB + 31) / 32;
  LMOT_CUDA(c, cudaMalloc(&t.d_tracks, (size_t)TC * sizeof(TrackState)));
  LMOT_CUDA(c, cudaMemsetAsync(t.d_tracks, 0, (size_t)TC * sizeof(TrackState), c->trk_stream));
  LMOT_CUDA(c, cudaMalloc(&t.d_trk_counters, CNT_COUNT * sizeof(int)));
  LMOT_CUDA(c, cudaMemsetAsync(t.d_trk_counters, 0, CNT_COUNT * sizeof(int), c->trk_stream));
  LMOT_CUDA(c, cudaHostAlloc(&t.h_trk_counters, CNT_COUNT * sizeof(int), cudaHostAllocDefault));
  LMOT_CUDA(c, cudaMalloc(&t.d_gate, (size_t)TC * c->gate_words * sizeof(unsigned)));
  LMOT_CUDA(c, cudaMalloc(&t.d_setter, (size_t)TC * c->gate_words * sizeof(unsigned)));
  LMOT_CUDA(c, cudaMalloc(&t.d_first_setter, (size_t)MB * sizeof(int)));
  LMOT_CUDA(c, cudaMalloc(&t.d_skip, TC));
  LMOT_CUDA(c, cudaMalloc(&t.d_new_num, (size_t)TC * sizeof(int)));
  LMOT_CUDA(c, cudaMalloc(&t.d_live_list, (size_t)TC * sizeof(int)));
  LMOT_CUDA(c, cudaMalloc(&t.d_vis_list, (size_t)TC * sizeof(int)));
  LMOT_CUDA(c, cudaMalloc(&t.d_act_list, (size_t)TC * sizeof(int)));
  LMOT_CUDA(c, cudaMalloc(&t.d_pos, (size_t)TC * sizeof(double4)));
  LMOT_CUDA(c, cudaMalloc(&t.d_summary, (size_t)TC * sizeof(ActSummary)));
  LMOT_CUDA(c, cudaMalloc(&t.d_meas_n, (size_t)TC * sizeof(int)));
  LMOT_CUDA(c, cudaMemsetAsync(t.d_meas_n, 0xFF, (size_t)TC * sizeof(int), c->trk_stream));
  LMOT_CUDA(c, cudaMalloc(&t.d_meas_ctr, (size_t)TC * 32 * sizeof(double2)));
  LMOT_CUDA(c, cudaMemsetAsync(t.d_meas_ctr, 0, (size_t)TC * 32 * sizeof(double2), c->trk_stream));
  LMOT_CUDA(c, cudaMalloc(&t.d_tc_seq, sizeof(unsigned)));
  LMOT_CUDA(c, cudaMemsetAsync(t.d_tc_seq, 0, sizeof(unsigned), c->trk_stream));
  LMOT_CUDA(c, cudaMalloc(&t.d_ids, ((size_t)TC + 1) * sizeof(long long)));
  t.tc_launched = 0;
  LMOT_CUDA(c, cudaMemsetAsync(t.d_pos, 0, (size_t)TC * sizeof(double4), c->trk_stream));
  t.last_trk_res = nullptr;
  t.act_valid = false;
  fill_int_kernel<<<(MB + 255) / 256, 256, 0, c->trk_stream>>>(t.d_first_setter, MB, INT_MAX);
  LMOT_CUDA(c, cudaGetLastError());
  const size_t sh = (size_t)c->gate_words * 32 * sizeof(unsigned short);
  LMOT_CUDA(c, cudaFuncSetAttribute(imm_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh));
  LMOT_CUDA(c, cudaFuncSetAttribute(spawn_output_kernel<kTCThreads>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TCFastShared<kTCThreads>)));
  LMOT_CUDA(c, cudaFuncSetAttribute(spawn_output_kernel<kTCWide>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TCFastShared<kTCWide>)));
  LMOT_CUDA(c, cudaFuncSetAttribute(imm_update_seq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh));
  LMOT_CUDA(c, cudaFuncSetAttribute(spawn_output_seq_kernel<kTCThreads>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TCFastShared<kTCThreads>)));
  LMOT_CUDA(c, cudaFuncSetAttribute(spawn_output_seq_kernel<kTCWide>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TCFastShared<kTCWide>)));
  LMOT_CUDA(c, cudaFuncSetAttribute(imm_update_seq_tuned_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh));
  LMOT_CUDA(c, cudaFuncSetAttribute(spawn_output_seq_tuned_kernel<kTCThreads>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TCFastShared<kTCThreads>)));
  LMOT_CUDA(c, cudaFuncSetAttribute(spawn_output_seq_tuned_kernel<kTCWide>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TCFastShared<kTCWide>)));
  t.last_n_act = 0;
  return LMOT_OK;
}

void tracker_free(Tracker& t) {
  cudaFree(t.d_tracks); cudaFree(t.d_trk_counters); cudaFree(t.d_gate); cudaFree(t.d_setter); cudaFree(t.d_first_setter);
  cudaFree(t.d_skip); cudaFree(t.d_new_num); cudaFree(t.d_live_list); cudaFree(t.d_vis_list); cudaFree(t.d_act_list); cudaFree(t.d_pos); cudaFree(t.d_summary); cudaFree(t.d_tc_seq); cudaFree(t.d_meas_n); cudaFree(t.d_meas_ctr);
  cudaFree(t.d_ids);
  if (t.h_trk_counters) cudaFreeHost(t.h_trk_counters);
  t = Tracker();
}

// getOriginPoints (imm_ukf_jpda.cpp:74-172) is scalar bookkeeping on three doubles per frame; it stays on the host.
// The reference replays its whole delta history every call; the replay is a left fold, so carrying (x, y, yaw) is
// bit-identical.
void origin_points_fold(TrackerHost& h, double timestamp, double v_gps, double yaw_gps) {
  const double firstEgoYawOffset = -0.63035 - M_PI / 2;
  const double dt = (timestamp - h.timestamp) / 1000000.0;
  h.egoVelo = v_gps;
  h.egoYaw = yaw_gps;
  h.egoYaw += firstEgoYawOffset;
  if (!h.init) {
    h.egoPoint[0] = 0; h.egoPoint[1] = 0; h.egoPoint[2] = h.egoYaw;
    h.fold[0] = 0; h.fold[1] = 0; h.fold[2] = -M_PI / 2;
    return;
  }
  const double diffYaw = h.egoYaw - h.egoPreYaw;
  const double dX = dt * h.egoVelo * cos(diffYaw), dY = dt * h.egoVelo * sin(diffYaw);
  double x = h.fold[0], y = h.fold[1], egoYaw = h.fold[2];
  x -= dX; y -= dY;
  const double preX = x, preY = y;
  const double yaw = diffYaw * -1;
  egoYaw += yaw;
  x = cos(yaw) * preX - sin(yaw) * preY;
  y = sin(yaw) * preX + cos(yaw) * preY;
  h.fold[0] = x; h.fold[1] = y; h.fold[2] = egoYaw;
  h.egoPoint[0] = x; h.egoPoint[1] = y; h.egoPoint[2] = egoYaw;
}

// boxes: device float[M][8][3] with M in det_counters[CNT_N_BOXES]; results into the DEVICE block of sl->res
// planar rigid transform of the "global" frame: pose (x, y, yaw) of `global` in the sensor frame, as the tracking node broadcasts it
// (tracking/main.cpp:76-83: setOrigin(egoPoints[0][0..1]), setRPY(0, 0, egoPoints[0][2])).  back: global -> sensor = that pose
// itself; fwd: sensor -> global = its inverse.  The 3x3 basis as tf::Matrix3x3::setRotation derives it from the quaternion
// tf::Quaternion::setRPY builds, the inverse as tf::Transform::inverse() (transpose, -(R^T t)), all in double, then narrowed to
// the Eigen::Matrix4f pcl_ros::transformPointCloud multiplies with.  (tf / pcl_ros are not in /root/reference: this arithmetic is
// the documented contract of this library, tests/test_global_frame_gpu.py restates it in numpy.)
void global_frame_xf(const double ego[3], Xf2* fwd, Xf2* back) {
  const double half = ego[2] * 0.5;
  const double qz = sin(half), qw = cos(half);        // setRPY(0, 0, yaw): x = y = 0
  const double d = qz * qz + qw * qw, s = 2.0 / d;
  const double zs = qz * s, wz = qw * zs, zz = qz * zs;
  const double r00 = 1.0 - zz, r01 = -wz, r10 = wz, r11 = 1.0 - zz;
  back->on = 1;
  back->m[0] = (float)r00; back->m[1] = (float)r01; back->m[2] = (float)ego[0];
  back->m[3] = (float)r10; back->m[4] = (float)r11; back->m[5] = (float)ego[1];
  // inverse: basis transposed, origin -(R^T t)
  const double tx = -(r00 * ego[0] + r10 * ego[1]), ty = -(r01 * ego[0] + r11 * ego[1]);
  fwd->on = 1;
  fwd->m[0] = (float)r00; fwd->m[1] = (float)r10; fwd->m[2] = (float)tx;
  fwd->m[3] = (float)r01; fwd->m[4] = (float)r11; fwd->m[5] = (float)ty;
}

// sensor-frame boxes of slot `sl` -> sl->d_boxes_g in the global frame of THIS frame's ego pose (peeked: tracker_launch folds it);
// post_sem: post the slot's detection semaphore afterwards (frame pipeline)
int boxes_to_global_launch(Ctx* c, Slot* sl, cudaStream_t st, const float* d_boxes, const int* det_counters, double timestamp, double v_gps,
                           double yaw_gps, bool post_sem) {
  TrackerHost peek = c->own.trk.th;
  origin_points_fold(peek, timestamp, v_gps, yaw_gps);
  Xf2 fwd, back;
  global_frame_xf(peek.egoPoint, &fwd, &back);
  boxes_to_global_kernel<<<1, 256, 0, st>>>(d_boxes, det_counters, sl->d_boxes_g, fwd, post_sem ? sl->d_det_sem : nullptr);
  kernel_mark(c, sl, st);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

// ---------------------------------------------------------------------------------------------- the tracker chain
// One step of 1 <= S <= 8 track tables: gate -> TA -> TB -> TC, as programmatic dependent launches on one stream.  The context's own
// table (tracker_launch) and the tables of a sequence tick (seq_tracker_launch) are prepared by chain_prepare and launched by
// chain_launch, which picks the kernel family (see the head of this file).
namespace {

// table k's slice of every parameter block (the default kernels take their arguments from slice 0); the _seq kernels take the
// `.b` blocks (`tc.t.b`), the _seq_tuned kernels the whole blocks
struct Chain {
  int S = 0;
  GateSeq g{};
  TASeqTunedParams ta{};
  TBSeqTunedParams tb{};
  TCSeqTunedParams tc{};
  PubSeqParams pub{};
  PubIdsParams ids{};
  bool tuned = false;          // some table has its own values ...
  bool ids_on = false;         // ... or numbers its tracks (RetPrm::on): the chain runs the _seq_tuned kernels
  int n_act_max = 0;           // the largest last_n_act of the tables: TC's width
  explicit Chain(const Ctx* c) {
    ta.b.words = tb.b.words = c->gate_words;
    ta.b.spin_limit = pub.spin_limit = c->spin_limit;
    tc.t.b.compat_first = c->prm.oracle_compat_first_frame ? 1 : 0;
    tc.t.b.max_tracks = c->prm.max_tracks;
  }
};

// table t's step on measurement list m (box list, counters, semaphore: nullptr for an ungated step) into result block r at the ego pose
// (ts, v, yaw) -> slot ch.S of the blocks.  Advances the table's host state; a table written from the host since its last step gets its
// active list rebuilt on `st` first.
int chain_prepare(Ctx* c, Tracker& t, const SeqMeas& m, Result* r, cudaStream_t st, double ts, double v, double yaw, Chain& ch) {
  const int k = ch.S++;
  const int first = t.th.init ? 0 : 1;
  const double dt = first ? 0.0 : (ts - t.th.timestamp) / 1000000.0;     // :807, from this table's own previous stamp
  origin_points_fold(t.th, ts, v, yaw);
  // global_frame: the tracker reads the list boxes_to_global_launch / seq_global_launch prepared, the results carry the sensor-frame list
  const bool gf = c->prm.global_frame != 0;
  if (gf) { Xf2 fwd; global_frame_xf(t.th.egoPoint, &fwd, &r->back); }
  else r->back.on = 0;
  const float* boxes = gf ? m.d_boxes_g : m.d_boxes;
  const int full = t.act_valid ? 0 : 1;   // the table was written from the host since its last step: rebuild the side arrays
  if (full) {
    LMOT_CUDA(c, cudaMemsetAsync(t.d_trk_counters + CNT_N_ACT, 0, sizeof(int), st));
    build_active_kernel<<<(c->prm.max_tracks + 255) / 256, 256, 0, st>>>(t.d_tracks, t.d_trk_counters, t.d_act_list);
    t.act_valid = true;
  }
  Result* pr = (full || !t.last_trk_res) ? r : t.last_trk_res;
  t.last_trk_res = r;
  const int run = (first && ch.tc.t.b.compat_first) ? 0 : 1;
  ActSummary* sum = reinterpret_cast<ActSummary*>(t.d_summary);
  double2* mc = reinterpret_cast<double2*>(t.d_meas_ctr);
  ch.g.sem[k] = m.d_det_sem;
  ch.ta.b.s[k] = TASeq{t.d_tracks, t.d_trk_counters, m.d_counters, boxes, dt, t.d_gate, t.d_setter, t.d_first_setter, t.d_skip, t.d_act_list,
                       t.d_meas_n, mc, t.d_tc_seq, t.tc_launched, run};
  ch.tb.b.s[k] = TBSeq{t.d_tracks, t.d_trk_counters, m.d_counters, boxes, t.d_gate, t.d_first_setter, t.d_skip, t.d_act_list, sum, t.d_meas_n, mc, run};
  OutPtrs o{r->d_targets, r->d_vandyaw, r->d_manage, r->d_static, r->d_vis, r->d_visbb, r->d_hdr, r->d_boxes};
  OutPtrs po{pr->d_targets, pr->d_vandyaw, pr->d_manage, pr->d_static, pr->d_vis, pr->d_visbb, pr->d_hdr, pr->d_boxes};
  ch.tc.t.b.s[k] = TCSeq{t.d_tracks, t.d_trk_counters, m.d_counters, boxes, m.d_boxes, t.d_first_setter, t.d_new_num, t.d_vis_list, t.d_skip,
                       t.d_act_list, t.d_pos, sum, m.d_det_sem, t.d_tc_seq, o, po, t.th.egoPoint[2], first, full};
  ch.ta.tp[k] = ta_prm(t.prm); ch.tb.tp[k] = tb_prm(t.prm); ch.tc.t.tp[k] = tc_prm(t.prm);
  ch.tuned |= t.tuned;
  ch.tc.rp[k] = ret_prm(c, t, r);
  if (ch.tc.rp[k].on) { ch.ids_on = true; ch.ids.s[k] = PubIds{r->d_hdr, r->d_ids, r->h_ids}; }
  ++t.tc_launched;
  OutPtrs h{r->h_targets, r->h_vandyaw, r->h_manage, r->h_static, r->h_vis, r->h_visbb, r->h_hdr, r->h_boxes};
  ch.pub.s[k] = PubSeq{o, h, t.d_tc_seq, t.tc_launched, r->back};
  if (t.last_n_act > ch.n_act_max) ch.n_act_max = t.last_n_act;
  t.th.timestamp = ts;
  t.th.egoPreYaw = t.th.egoYaw;
  t.th.init = true;
  t.pred_ok = true;
  t.last_st = st;
  return LMOT_OK;
}

enum class ChainGate { none, one, seq };   // tracker_gate_kernel on the one semaphore of slice 0, tracker_gate_seq_kernel on all S

// launches the prepared chain on `st`.  own: the context's own table (the single-table default kernels where the family is the
// default one; `tc_wide` holds TC's width) or a sequence tick (`seq_wide`).  gate: how the chain waits for its measurement lists on the
// device (none: the caller ordered the stream, or nothing to wait for); TA follows a gate kernel as its programmatic dependent.
// pdl: TB and TC as programmatic dependents (timing mode records an event between the kernels, which needs the ordinary full
// serialisation).  mark: the slot whose kernel_marks to record (nullptr: none).  ta_tb: false on the own table's compat first frame,
// where TC alone runs, fully serialised.
int chain_launch(Ctx* c, Chain& ch, cudaStream_t st, bool own, ChainGate gate, bool pdl, Slot* mark, bool ta_tb) {
  const int S = ch.S;
  const bool def = !ch.tuned && !ch.ids_on;
  cudaLaunchAttribute pa;
  pa.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  cudaLaunchConfig_t cfg = {};
  cfg.stream = st; cfg.attrs = &pa; cfg.numAttrs = 1;
  // a prediction queued since the last step reads the table this step writes, and TA waits for the previous TC, not for the grid in
  // front of the gate kernel: the step's first kernel runs fully serialised behind it (behind its event when it ran on another stream)
  const bool after_pred = c->pred_pending;
  c->pred_pending = false;
  if (after_pred && c->pred_stream != st) LMOT_CUDA(c, cudaStreamWaitEvent(st, c->ev_pred, 0));
  if (ta_tb) {
    pa.val.programmaticStreamSerializationAllowed = (gate != ChainGate::none && !after_pred) ? 1 : 0;
    cfg.gridDim = dim3(1); cfg.blockDim = dim3(32); cfg.dynamicSmemBytes = 0;
    if (gate == ChainGate::one) LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, tracker_gate_kernel, (const int*)ch.g.sem[0], c->spin_limit));
    if (gate == ChainGate::seq) { ch.g.n = S; LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, tracker_gate_seq_kernel, ch.g, c->spin_limit)); }
    pa.val.programmaticStreamSerializationAllowed = gate != ChainGate::none ? 1 : 0;      // TA: the gate kernel's programmatic dependent
    // the single-stream chain's CTA count, shared by the tables (grid-stride over each table's active tracks)
    cfg.gridDim = dim3((c->trk_ctas + S - 1) / S, S); cfg.blockDim = dim3(kTAThreads);
    const TASeq& a = ch.ta.b.s[0];
    if (own && def)
      LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, imm_predict_gate_kernel, a.tracks, a.trk, a.det, a.boxes, a.dt, a.gate, a.setter, a.first_setter, a.skip,
                                      ch.ta.b.words, a.act_list, a.meas_n, a.meas_ctr, a.tc_seq, a.tc_want, ch.ta.b.spin_limit));
    else if (def) LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, imm_predict_gate_seq_kernel, ch.ta.b));
    else LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, imm_predict_gate_seq_tuned_kernel, ch.ta));
    if (mark) kernel_mark(c, mark, st);
    pa.val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.blockDim = dim3(kTBThreads); cfg.dynamicSmemBytes = (size_t)c->gate_words * 32 * sizeof(unsigned short);
    const TBSeq& b = ch.tb.b.s[0];
    if (own && def)
      LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, imm_update_kernel, b.tracks, b.trk, b.det, b.boxes, b.gate, b.first_setter, b.skip, ch.tb.b.words,
                                      b.act_list, b.summary, b.meas_n, b.meas_ctr));
    else if (def) LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, imm_update_seq_kernel, ch.tb.b));
    else LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, imm_update_seq_tuned_kernel, ch.tb));
    if (mark) kernel_mark(c, mark, st);
  }
  pa.val.programmaticStreamSerializationAllowed = (pdl && ta_tb) ? 1 : 0;
  // TC's width: one active track per thread on the fast path.  The host only knows the active count of the last result it has read
  // (a few frames old inside the pipeline; the count moves by a handful per frame): switch early, with hysteresis.  A count above the
  // width runs the kernel's general path -- slower, same results.
  bool& wide_now = own ? c->tc_wide : c->seq_wide;
  if (ch.n_act_max > 208) wide_now = true;
  else if (ch.n_act_max < 144) wide_now = false;
  const bool wide = c->tc_force >= 0 ? c->tc_force != 0 : wide_now;
  cfg.gridDim = dim3(S); cfg.blockDim = dim3(wide ? kTCWide : kTCThreads);
  cfg.dynamicSmemBytes = wide ? sizeof(TCFastShared<kTCWide>) : sizeof(TCFastShared<kTCThreads>);
  const TCSeq& q = ch.tc.t.b.s[0];
  if (own && def)
    LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, wide ? spawn_output_kernel<kTCWide> : spawn_output_kernel<kTCThreads>, q.tracks, q.trk, q.det, q.boxes,
                                    q.boxes_pub, q.first_setter, q.imax_arr, q.vis_list, q.has5_arr, q.first_frame, ch.tc.t.b.compat_first, q.ego_yaw,
                                    ch.tc.t.b.max_tracks, q.o, q.prev, q.full, q.act_list, q.pos, q.summary, q.det_sem, q.tc_seq));
  else if (def) LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, wide ? spawn_output_seq_kernel<kTCWide> : spawn_output_seq_kernel<kTCThreads>, ch.tc.t.b));
  else LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, wide ? spawn_output_seq_tuned_kernel<kTCWide> : spawn_output_seq_tuned_kernel<kTCThreads>, ch.tc));
  if (mark) kernel_mark(c, mark, st);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

}  // namespace

int tracker_launch(Ctx* c, Slot* sl, cudaStream_t st, const float* d_boxes, const int* det_counters, double timestamp, double v_gps,
                   double yaw_gps, bool gate, bool* gated) {
  const bool compat_first = !c->own.trk.th.init && c->prm.oracle_compat_first_frame;   // the reference's first-frame quirk: TC alone
  // `gate` (frame submissions): the detection stages of this frame post sl->d_det_sem.  Either the gate kernel waits for it on
  // the device (see tracker_gate_kernel), or -- timing mode, the reference's first-frame quirk -- the stream waits for the event.
  const bool use_gate = gate && !c->timing && !compat_first;
  if (gate && !use_gate) LMOT_CUDA(c, cudaStreamWaitEvent(st, sl->ev_det_done, 0));
  if (gated) *gated = use_gate;
  Chain ch(c);
  const SeqMeas m{const_cast<float*>(d_boxes), sl->d_boxes_g, const_cast<int*>(det_counters), gate ? sl->d_det_sem : nullptr};
  if (int rc = chain_prepare(c, c->own.trk, m, sl->res, st, timestamp, v_gps, yaw_gps, ch)) return rc;
  return chain_launch(c, ch, st, true, use_gate ? ChainGate::one : ChainGate::none, !c->timing, sl, !compat_first);
}

// device block of `r` -> its pinned host block (asynchronous on st)
int tracker_publish(Ctx* c, Result* r, cudaStream_t st) {
  OutPtrs d{r->d_targets, r->d_vandyaw, r->d_manage, r->d_static, r->d_vis, r->d_visbb, r->d_hdr, r->d_boxes};
  OutPtrs h{r->h_targets, r->h_vandyaw, r->h_manage, r->h_static, r->h_vis, r->h_visbb, r->h_hdr, r->h_boxes};
  publish_kernel<<<1, kPubThreads, 0, st>>>(d, h, c->own.trk.d_tc_seq, c->own.trk.tc_launched, c->spin_limit, r->back);
  if (r->ids) {
    PubIdsParams p{};
    p.s[0] = PubIds{r->d_hdr, r->d_ids, r->h_ids};
    publish_ids_kernel<<<1, kPubThreads, 0, st>>>(p);
  }
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

int boxes_publish(Ctx* c, Slot* s, Result* r, cudaStream_t st) {
  publish_boxes_kernel<<<1, 256, 0, st>>>(s->d_boxes, s->d_counters, r->h_boxes);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

// ---------------------------------------------------------------------------------------------- sequence ticks (lmot_seq_*)
// Sequence k of a tick: measurement list m[k] (box list, counters, semaphore), track table c->seq[k].trk, result block tick->blocks[k].
// Every launch below covers all S sequences; per-sequence arguments travel in __grid_constant__ parameter blocks.

// global_frame: position k's sensor- (or vehicle-) frame boxes -> m[k].d_boxes_g with THIS tick's ego pose of sequence seq[k] (peeked:
// seq_tracker_launch folds it), posting m[k]'s detection semaphore
int seq_global_launch(Ctx* c, const int* seq, const SeqMeas* m, int S, cudaStream_t st, const double* ts, const double* v, const double* yaw) {
  GlobalSeqParams p{};
  for (int k = 0; k < S; ++k) {
    TrackerHost peek = c->seq[seq[k]].trk.th;
    origin_points_fold(peek, ts[k], v[k], yaw[k]);
    Xf2 back;
    global_frame_xf(peek.egoPoint, &p.s[k].fwd, &back);
    p.s[k].boxes = m[k].d_boxes; p.s[k].det = m[k].d_counters; p.s[k].boxes_g = m[k].d_boxes_g; p.s[k].det_sem = m[k].d_det_sem;
  }
  boxes_to_global_seq_kernel<<<S, 256, 0, st>>>(p);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

// gate -> TA -> TB -> TC once for the S stepped sequences on the tracker stream (chain_launch), then one publish launch on the publish
// stream.  The caller records the tick's events on the publish stream afterwards.
int seq_tracker_launch(Ctx* c, const int* seq, const SeqMeas* m, SeqTick* tick, int S, const double* ts, const double* v, const double* yaw) {
  Chain ch(c);
  for (int k = 0; k < S; ++k)
    if (int rc = chain_prepare(c, c->seq[seq[k]].trk, m[k], &tick->blocks[seq[k]], c->trk_stream, ts[k], v[k], yaw[k], ch)) return rc;
  if (int rc = chain_launch(c, ch, c->trk_stream, false, ChainGate::seq, true, nullptr, true)) return rc;
  publish_seq_kernel<<<S, kPubThreads, 0, c->pub_stream>>>(ch.pub);
  if (ch.ids_on) publish_ids_kernel<<<S, kPubThreads, 0, c->pub_stream>>>(ch.ids);
  LMOT_CUDA(c, cudaGetLastError());
  return LMOT_OK;
}

// ---------------------------------------------------------------------------------------------- track prediction (lmot_predict_tracks*)
// One launch for the S tables, on st behind their latest steps: a programmatic dependent of the step's TC, whose griddepcontrol.wait
// returns once TC (retire phase included) has completed.  The next chain_launch serialises its first kernel behind it (pred_pending).
int predict_launch(Ctx* c, Tracker* const* tabs, int S, const double* t_us, int n_t, const lmot_pred_out* outs, int* const* d_n_rows,
                   cudaStream_t st) {
  PredParams p{};
  p.n_t = n_t;
  for (int k = 0; k < S; ++k) {
    const Tracker& t = *tabs[k];
    p.s[k] = PredTab{t.d_tracks, t.d_trk_counters, t.ids_identity ? nullptr : t.d_ids, outs[k], d_n_rows ? d_n_rows[k] : nullptr, ta_prm(t.prm)};
    for (int j = 0; j < n_t; ++j) p.dt[k][j] = (t_us[k * n_t + j] - t.th.timestamp) / 1000000.0;     // as chain_prepare's dt (:807)
  }
  if (!c->ev_pred) LMOT_CUDA(c, cudaEventCreateWithFlags(&c->ev_pred, cudaEventDisableTiming));
  cudaLaunchAttribute pa;
  pa.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  pa.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.stream = st; cfg.attrs = &pa; cfg.numAttrs = 1;
  cfg.gridDim = dim3((c->trk_ctas + S - 1) / S, S); cfg.blockDim = dim3(kTAThreads);
  LMOT_CUDA(c, cudaLaunchKernelEx(&cfg, predict_tracks_kernel, p));
  LMOT_CUDA(c, cudaEventRecord(c->ev_pred, st));
  c->pred_pending = true;
  c->pred_stream = st;
  return LMOT_OK;
}

}  // namespace lmot
