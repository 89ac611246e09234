// cluster_node.cpp -- `rosrun object_tracking cluster`, H100 edition (SURVEY.md §8(f)1).
//
// Same ROS surface as the reference's node (object_tracking/src/cluster/main.cpp:237-256): node "cluster", subscribes
// "none_ground_topic"; publishes "output" (clustered cloud), "realtime_cost_map" (nav_msgs/OccupancyGrid), "cluster_obs"
// (object_tracking/ObstacleList), "track_box" (object_tracking/trackbox), "cluster_ma" (cube markers) and
// "visualization_marker" (box edges).  componentClustering, boxFitting and the three side outputs are liblmot calls on the
// elevated cloud; this file only converts messages.  Needs ROS (catkin) and the package's generated message headers.
#include <ros/ros.h>
#include <nav_msgs/OccupancyGrid.h>
#include <sensor_msgs/PointCloud2.h>
#include <visualization_msgs/Marker.h>
#include <visualization_msgs/MarkerArray.h>
#include <object_tracking/ObstacleList.h>
#include <object_tracking/trackbox.h>
#include <vector>
#include "lmot.h"
#include "lmot_ros_codec.hpp"

namespace {
lmot_ctx* g_ctx = nullptr;
ros::Publisher g_pub_cloud, g_pub_cost, g_pub_obs, g_pub_boxes, g_pub_cubes, g_pub_edges;
std::vector<float> g_packed, g_clustered, g_obstacles, g_boxes, g_markers;
std::vector<int32_t> g_grid(LMOT_NUM_GRID * LMOT_NUM_GRID), g_cost(50 * 50);
constexpr int kMaxBoxes = 1024;

bool ok(int rc, const char* what) {
  if (rc == LMOT_OK) return true;
  ROS_ERROR_THROTTLE(1.0, "%s: %s (%s)", what, lmot_strerror(rc), lmot_last_error(g_ctx));
  return false;
}

void on_elevated(const sensor_msgs::PointCloud2ConstPtr& in) {
  const lmot_ros::XyzLayout L = lmot_ros::xyz_layout(*in);
  const float* pts = reinterpret_cast<const float*>(L.base);
  int stride = L.stride_floats();
  if (!L.zero_copy) { g_packed.resize((size_t)L.n * 4); lmot_ros::gather_xyz(L, g_packed.data(), 4); pts = g_packed.data(); stride = 4; }
  int num_cluster = 0;
  if (!ok(lmot_component_cluster(g_ctx, pts, L.n, stride, g_grid.data(), &num_cluster), "lmot_component_cluster")) return;

  // side outputs of the clustering (clustered cloud, obstacle list, cost map)
  const int cap = L.n > 0 ? L.n : 1;
  g_clustered.resize((size_t)cap * 4); g_obstacles.resize((size_t)LMOT_NUM_GRID * LMOT_NUM_GRID * 4);
  int n_cl = 0, n_ob = 0;
  if (!ok(lmot_cluster_outputs(g_ctx, g_clustered.data(), cap, &n_cl, g_obstacles.data(), LMOT_NUM_GRID * LMOT_NUM_GRID, &n_ob, g_cost.data()),
          "lmot_cluster_outputs")) return;
  sensor_msgs::PointCloud2 cloud;
  lmot_ros::fill_pointcloud2_xyz(cloud, g_clustered.data(), n_cl);
  cloud.header.frame_id = in->header.frame_id;
  nav_msgs::OccupancyGrid og;                                 // geometry: component_clustering.cpp:410-422 (50 x 50 cells of 1 m)
  og.header.frame_id = in->header.frame_id;
  og.info.resolution = 1.0; og.info.width = 50; og.info.height = 50;
  og.info.origin.position.x = -25.0; og.info.origin.position.y = 0.0; og.info.origin.position.z = -2.0;
  og.info.origin.orientation.w = 1.0;
  og.data.assign(g_cost.begin(), g_cost.end());
  object_tracking::ObstacleList obs;
  obs.header.frame_id = in->header.frame_id;
  obs.cellLength = 0.2f; obs.cellWidth = 0.2f;
  obs.obstacles.resize(n_ob);
  for (int i = 0; i < n_ob; ++i) {
    obs.obstacles[i].x = g_obstacles[4 * i]; obs.obstacles[i].y = g_obstacles[4 * i + 1]; obs.obstacles[i].z = g_obstacles[4 * i + 2];
    obs.obstacles[i].cluster = (int)g_obstacles[4 * i + 3];
  }
  g_pub_cost.publish(og);
  g_pub_obs.publish(obs);
  g_pub_cloud.publish(cloud);

  // boxes
  g_boxes.resize((size_t)kMaxBoxes * 24); g_markers.resize((size_t)kMaxBoxes * 6);
  int nb = 0;
  if (!ok(lmot_box_fit(g_ctx, pts, L.n, stride, g_grid.data(), num_cluster, g_boxes.data(), kMaxBoxes, &nb, g_markers.data()), "lmot_box_fit")) return;
  object_tracking::trackbox tb;
  tb.header = in->header;
  const int sent = lmot_ros::pack_trackbox(tb, g_boxes.data(), nb);
  if (sent < nb) ROS_WARN_THROTTLE(5.0, "track_box carries %d of %d boxes (uint8 box_num)", sent, nb);
  g_pub_boxes.publish(tb);

  visualization_msgs::MarkerArray cubes;                       // constants of the cube markers: box_fitting.cpp:170-207
  cubes.markers.resize(nb);
  for (int b = 0; b < nb; ++b) {
    visualization_msgs::Marker& m = cubes.markers[b];
    m.header.frame_id = "/velodyne"; m.header.stamp = ros::Time::now();
    m.ns = "cube"; m.id = b; m.type = visualization_msgs::Marker::CUBE; m.action = visualization_msgs::Marker::ADD;
    m.pose.position.x = g_markers[b * 6]; m.pose.position.y = g_markers[b * 6 + 1]; m.pose.position.z = g_markers[b * 6 + 2];
    m.pose.orientation.w = 1.0;
    m.scale.x = g_markers[b * 6 + 3]; m.scale.y = g_markers[b * 6 + 4]; m.scale.z = g_markers[b * 6 + 5];
    m.color.g = 1.0f; m.color.a = 0.5f;
    m.lifetime = ros::Duration(1.0);
  }
  g_pub_cubes.publish(cubes);
  visualization_msgs::Marker edges;
  edges.header.frame_id = "velodyne"; edges.header.stamp = ros::Time::now();
  edges.ns = "boxes"; edges.id = 0; edges.type = visualization_msgs::Marker::LINE_LIST; edges.action = visualization_msgs::Marker::ADD;
  edges.pose.orientation.w = 1.0; edges.scale.x = 0.1; edges.color.g = 1.0f; edges.color.a = 1.0f;
  for (int b = 0; b < nb; ++b) lmot_ros::box_edges(g_boxes.data() + (size_t)b * 24, edges.points);
  g_pub_edges.publish(edges);
}
}  // namespace

int main(int argc, char** argv) {
  ros::init(argc, argv, "cluster");
  ros::NodeHandle nh;
  lmot_params prm;
  lmot_default_params(&prm);
  prm.max_boxes = kMaxBoxes;
  int device = 0;
  nh.param<int>("cuda_device", device, 0);
  const int rc = lmot_create(&g_ctx, &prm, device);
  if (rc != LMOT_OK) { ROS_FATAL("lmot_create: %s -- this node has no CPU path", lmot_strerror(rc)); return 1; }
  g_pub_cloud = nh.advertise<sensor_msgs::PointCloud2>("output", 1);
  g_pub_edges = nh.advertise<visualization_msgs::Marker>("visualization_marker", 0);
  g_pub_cubes = nh.advertise<visualization_msgs::MarkerArray>("cluster_ma", 10);
  g_pub_cost = nh.advertise<nav_msgs::OccupancyGrid>("realtime_cost_map", 10);
  g_pub_obs = nh.advertise<object_tracking::ObstacleList>("cluster_obs", 10);
  g_pub_boxes = nh.advertise<object_tracking::trackbox>("track_box", 10);
  ros::Subscriber sub = nh.subscribe("none_ground_topic", 160, on_elevated);
  ros::spin();
  lmot_destroy(g_ctx);
  return 0;
}
