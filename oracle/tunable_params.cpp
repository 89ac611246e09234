// TEST INFRASTRUCTURE ONLY -- linked into oracle/_ref/libref_tunable.so (oracle/tunable.mk), never into the product.
//
// The tracker constants of the reference that have no file-scope variable of their own, as exported globals with the reference's
// values.  The build-time copies of imm_ukf_jpda.cpp and ukf.cpp read these instead of their literals, so a test can move one
// (ctypes in_dll, oracle/ref_tunable.py) and compare the library's lmot_tracker_params with the reference's own arithmetic.
// gammaG_, pG_, pD_, distanceThres_, lifeTimeThres_ and bbYawChangeThres_ are the copy's own globals (their `const` removed).
extern "C" {
int lmot_tp_static_lifetime = 8;                      // imm_ukf_jpda.cpp:1064  lifetime_ > 8
double lmot_tp_static_dist = 3.0;                     // :1067  distThres = 3.0
double lmot_tp_second_init_v = 2;                     // :902   targetV = 2
double lmot_tp_std_a[3] = {2, 2, 3};                  // ukf.cpp:68-70  std_a_cv_, std_a_ctrv_, std_a_rm_
double lmot_tp_std_yawdd[3] = {2, 2, 3};              // :71-73  std_cv_yawdd_, std_ctrv_yawdd_, std_rm_yawdd_
double lmot_tp_std_las[2] = {0.15, 0.15};             // :91-94  std_laspx_, std_laspy_
double lmot_tp_trans[3][3] = {{0.9, 0.05, 0.05},      // :144-154  row i = p{i+1}_
                              {0.05, 0.9, 0.05},
                              {0.05, 0.05, 0.9}};
double lmot_tp_mode_prob0[3] = {0.33, 0.33, 0.33};    // :180-182  modeProbCV_, modeProbCTRV_, modeProbRM_
double lmot_tp_p0_diag[5] = {0.5, 0.5, 3, 10, 1};     // :275-279  P_merge_
}
