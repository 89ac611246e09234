// TEST INFRASTRUCTURE ONLY -- the reference's side of box search (include/lmot.h, lmot_set_box_search).
//
// Built by oracle/box_search.mk into oracle/_ref/libref_box_search_<mode>.so, one per reference library (intended, o2), each linked
// against its libref_<mode>.so, so that it calls the instance the test process has loaded.  The search itself (steps 1-5) is restated
// once, in NumPy (tests/box_search_scenes.py); this helper only marshals flat arrays into the reference's own getClusteredPoints and
// ruleBasedFilter (box_fitting.cpp:46,97, both externally linked).  No algorithm is implemented in this file.
#include <cstdint>
#include <opencv2/opencv.hpp>
#include "box_fitting.h"

using namespace cv;

void getClusteredPoints(PointCloud<PointXYZ>::Ptr elevatedCloud, array<array<int, numGrid>, numGrid> cartesianData,
                        vector<PointCloud<PointXYZ>>& clusteredPoints);
bool ruleBasedFilter(vector<Point2f> pcPoints, float maxZ, int numPoints);
extern float sensorHeight;           // box_fitting.cpp:26

extern "C" {

// getClusteredPoints (box_fitting.cpp:46) on the elevated cloud xyz (n points, stride floats each) and the label grid: the clusters'
// points one after another, cluster 1 first, each in the reference's order -> pts [n][3]; cluster c holds pts[off[c - 1] .. off[c]).
// Returns the number of points written.
int ref_bs_clusters(const float* xyz, int n, int stride, const int32_t* grid, int num_cluster, float* pts, int* off) {
  PointCloud<PointXYZ>::Ptr cloud(new PointCloud<PointXYZ>());
  cloud->points.resize(n);
  for (int i = 0; i < n; ++i) { cloud->points[i].x = xyz[i * stride]; cloud->points[i].y = xyz[i * stride + 1]; cloud->points[i].z = xyz[i * stride + 2]; }
  static array<array<int, numGrid>, numGrid> cart;
  for (int x = 0; x < numGrid; ++x) for (int y = 0; y < numGrid; ++y) cart[x][y] = grid[x * numGrid + y];
  vector<PointCloud<PointXYZ>> cl(num_cluster);          // as boxFitting (box_fitting.cpp:425) sizes it
  getClusteredPoints(cloud, cart, cl);
  int m = 0;
  off[0] = 0;
  for (int c = 0; c < num_cluster; ++c) {
    for (size_t j = 0; j < cl[c].size(); ++j, ++m) { pts[3 * m] = cl[c][j].x; pts[3 * m + 1] = cl[c][j].y; pts[3 * m + 2] = cl[c][j].z; }
    off[c + 1] = m;
  }
  return m;
}

// ruleBasedFilter (box_fitting.cpp:97) on the four corners pc[4][2]
int ref_bs_rule(const float* pc, float max_z, int n_points) {
  vector<Point2f> v(4);
  for (int i = 0; i < 4; ++i) { v[i].x = pc[2 * i]; v[i].y = pc[2 * i + 1]; }
  return ruleBasedFilter(v, max_z, n_points) ? 1 : 0;
}

float ref_bs_sensor_height() { return sensorHeight; }

}  // extern "C"
