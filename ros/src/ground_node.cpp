// ground_node.cpp -- `rosrun object_tracking ground`, H100 edition (SURVEY.md §8(f)1).
//
// Same ROS surface as the reference's node (object_tracking/src/groundremove/main.cpp:139-157): node "ground", subscribes
// "velodyne_points" (sensor_msgs/PointCloud2, queue 160), parameters filter_z_min / filter_z_max (-3 / 1), publishes
// "ground_topic", "none_ground_topic" and "aux_points".  The callback hands the message buffer to liblmot: the node's
// PassThrough / ConditionalRemoval pre-filters and groundRemove run in ONE kernel on the GPU (lmot_params.node_prefilter),
// `aux_points` is rebuilt from the per-point labels.  Needs ROS (catkin); not built in the GPU image.
#include <ros/ros.h>
#include <sensor_msgs/PointCloud2.h>
#include <vector>
#include "lmot.h"
#include "lmot_ros_codec.hpp"

namespace {
lmot_ctx* g_ctx = nullptr;
ros::Publisher g_pub_ground, g_pub_elevated, g_pub_aux;
std::vector<float> g_packed, g_elev, g_ground, g_aux;
std::vector<uint8_t> g_labels;

void on_cloud(const sensor_msgs::PointCloud2ConstPtr& in) {
  const lmot_ros::XyzLayout L = lmot_ros::xyz_layout(*in);
  const float* pts = reinterpret_cast<const float*>(L.base);
  int stride = L.stride_floats();
  if (!L.zero_copy) {                       // exotic layouts only: gather x, y, z once
    g_packed.resize((size_t)L.n * 4);
    lmot_ros::gather_xyz(L, g_packed.data(), 4);
    pts = g_packed.data(); stride = 4;
  }
  const size_t cap = (size_t)(L.n > 0 ? L.n : 1);
  g_elev.resize(cap * 4); g_ground.resize(cap * 4); g_labels.resize(cap);
  int ne = 0, ng = 0;
  const int rc = lmot_ground_remove(g_ctx, pts, L.n, stride, g_labels.data(), g_elev.data(), &ne, g_ground.data(), &ng);
  if (rc != LMOT_OK) { ROS_ERROR_THROTTLE(1.0, "lmot_ground_remove: %s (%s)", lmot_strerror(rc), lmot_last_error(g_ctx)); return; }
  // aux_points = what survives the node's pre-filters = every point with a non-zero label, in cloud order
  g_aux.clear();
  for (int i = 0; i < L.n; ++i)
    if (g_labels[i]) { const float* p = pts + (size_t)i * stride; g_aux.insert(g_aux.end(), {p[0], p[1], p[2], 1.f}); }
  sensor_msgs::PointCloud2 aux, ground, elevated;
  lmot_ros::fill_pointcloud2_xyz(aux, g_aux.data(), (int)(g_aux.size() / 4));
  lmot_ros::fill_pointcloud2_xyz(ground, g_ground.data(), ng);
  lmot_ros::fill_pointcloud2_xyz(elevated, g_elev.data(), ne);
  aux.header = in->header;
  ground.header.frame_id = in->header.frame_id;          // the reference copies only the frame id onto its outputs
  elevated.header.frame_id = in->header.frame_id;
  g_pub_aux.publish(aux);
  g_pub_elevated.publish(elevated);
  g_pub_ground.publish(ground);
}
}  // namespace

int main(int argc, char** argv) {
  ros::init(argc, argv, "ground");
  ros::NodeHandle nh;
  lmot_params prm;
  lmot_default_params(&prm);
  prm.node_prefilter = 1;
  nh.param<float>("filter_z_max", prm.filter_z_max, 1.0f);
  nh.param<float>("filter_z_min", prm.filter_z_min, -3.0f);
  int device = 0;
  nh.param<int>("cuda_device", device, 0);
  const int rc = lmot_create(&g_ctx, &prm, device);
  if (rc != LMOT_OK) { ROS_FATAL("lmot_create: %s -- this node has no CPU path", lmot_strerror(rc)); return 1; }
  g_pub_ground = nh.advertise<sensor_msgs::PointCloud2>("ground_topic", 1);
  g_pub_elevated = nh.advertise<sensor_msgs::PointCloud2>("none_ground_topic", 1);
  g_pub_aux = nh.advertise<sensor_msgs::PointCloud2>("aux_points", 1);
  ros::Subscriber sub = nh.subscribe("velodyne_points", 160, on_cloud);
  ros::spin();
  lmot_destroy(g_ctx);
  return 0;
}
