// TEST INFRASTRUCTURE ONLY -- linked into oracle/_ref/libref_detect_tunable.so (oracle/detect_tunable.mk), never into the product.
//
// The two detection values the reference writes as literals, as exported globals with the reference's values.  The build-time copies
// of ground_removal.cpp and box_fitting.cpp read these instead, so a test can move them (ctypes in_dll) and compare the library's
// lmot_detect_params.ground_tolerance / min_cluster_points with the reference's own arithmetic.  Every other detection value already
// is a mutable global of the reference (rMin, roiM, ramPoints, ...).
extern "C" {
double lmot_dp_ground_tolerance = 0.25;   // ground_removal.cpp:239  z < (hGround + 0.25)
int lmot_dp_min_cluster_points = 30;      // box_fitting.cpp:100      numPoints < 30
}
