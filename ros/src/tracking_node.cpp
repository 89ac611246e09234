// tracking_node.cpp -- `rosrun object_tracking tracking`, H100 edition (SURVEY.md §8(f)1).
//
// Same ROS surface as the reference's node (object_tracking/tracking/main.cpp:413-445): node "obj_track", subscribes
// "track_box" (object_tracking/trackbox) and "/gps/odom" (ego speed / yaw), publishes the track markers on
// "visualization_marker" (arrows, coloured points) and the visible boxes on "visualization_marker2".
// getOriginPoints + the tf round trip + immUkfJpdaf are ONE liblmot call: with lmot_params.global_frame = 1, lmot_track_step moves the
// boxes into the dead-reckoned "global" frame on the device before tracking and moves targets / visible boxes back afterwards,
// exactly where the reference calls pcl_ros::transformPointCloud (main.cpp:142-158,182-195); the UKF states, velocities,
// distFromInit and the static flag are therefore world-frame quantities as in the reference node.  The velodyne -> global transform
// is broadcast from lmot_origin_points like main.cpp:76-83 does from getOriginPoints.
// Timestamp: the reference node passes header.stamp.toSec() -- SECONDS -- to a tracker that divides by 1e6 (imm_ukf_jpda.cpp:807),
// i.e. the deployed reference runs with dt ~ 1e-7 s.  Default here = the same (drop-in for what is deployed); the private parameter
// ~stamp_in_microseconds:=true feeds the physically meaningful value instead.
// Track table: like the reference, dead tracks keep their row by default, so the table (kCap rows) fills after a few minutes of
// driving and new objects are no longer tracked.  ~retire_dead_tracks:=true turns track retirement on (lmot_set_track_retirement):
// dead tracks are removed after every step, the node can run indefinitely, and the arrow markers take their ids from the stable
// track IDs (lmot_track_ids) instead of the row index.
// Needs ROS (catkin) and the package's generated message headers.
#include <ros/ros.h>
#include <nav_msgs/Odometry.h>
#include <tf/transform_datatypes.h>
#include <tf/transform_broadcaster.h>
#include <visualization_msgs/Marker.h>
#include <object_tracking/trackbox.h>
#include <cmath>
#include <vector>
#include "lmot.h"
#include "lmot_ros_codec.hpp"

namespace {
lmot_ctx* g_ctx = nullptr;
ros::Publisher g_pub_markers, g_pub_boxes;
double g_v_gps = 0.0, g_yaw_gps = 0.0;
bool g_stamp_us = false;
bool g_retire = false;
constexpr int kCap = 8192;
std::vector<float> g_boxes, g_targets((size_t)kCap * 3), g_visbb((size_t)kCap * 24);
std::vector<double> g_vy((size_t)kCap * 2);
std::vector<int32_t> g_manage(kCap);
std::vector<uint8_t> g_static(kCap), g_vis(kCap);
std::vector<int64_t> g_ids(kCap);

void on_odom(const nav_msgs::Odometry& odom) {
  const auto& t = odom.twist.twist.linear;
  g_v_gps = std::sqrt(t.x * t.x + t.y * t.y);
  g_yaw_gps = tf::getYaw(odom.pose.pose.orientation);
}

visualization_msgs::Marker points_marker(int id, float r, float g, float b) {
  visualization_msgs::Marker m;
  m.header.frame_id = "velodyne"; m.header.stamp = ros::Time::now();
  m.ns = "points"; m.id = id; m.type = visualization_msgs::Marker::POINTS; m.action = visualization_msgs::Marker::ADD;
  m.pose.orientation.w = 1.0; m.scale.x = 0.5; m.scale.y = 0.5;
  m.color.r = r; m.color.g = g; m.color.b = b; m.color.a = 1.0f;
  return m;
}

void on_boxes(const object_tracking::trackbox& in) {
  const int m = lmot_ros::unpack_trackbox(in, g_boxes);
  lmot_track_out o{};
  o.cap = kCap; o.targets = g_targets.data(); o.vandyaw = g_vy.data(); o.track_manage = g_manage.data();
  o.is_static = g_static.data(); o.is_vis = g_vis.data(); o.vis_bb = g_visbb.data();
  const double stamp = g_stamp_us ? in.header.stamp.toSec() * 1.0e6 : in.header.stamp.toSec();      // main.cpp:72
  // tf velodyne -> global from this frame's ego pose (main.cpp:74-83); lmot_origin_points peeks, lmot_track_step folds the same values
  double ego[6];
  if (lmot_origin_points(g_ctx, stamp, g_v_gps, g_yaw_gps, ego) == LMOT_OK) {
    static tf::TransformBroadcaster br;
    tf::Transform transform;
    transform.setOrigin(tf::Vector3(ego[0], ego[1], 0.0));
    tf::Quaternion q;
    q.setRPY(0, 0, ego[2]);
    transform.setRotation(q);
    br.sendTransform(tf::StampedTransform(transform, in.header.stamp, "velodyne", "global"));
  }
  const int rc = lmot_track_step(g_ctx, g_boxes.data(), m, stamp, g_v_gps, g_yaw_gps, &o);
  if (rc < 0) { ROS_ERROR_THROTTLE(1.0, "lmot_track_step: %s (%s)", lmot_strerror(rc), lmot_last_error(g_ctx)); return; }
  if (rc > 0) ROS_WARN_THROTTLE(10.0, "lmot_track_step: %s", lmot_strerror(rc));      // e.g. track table full: outputs are valid, keep publishing
  int n_ids = 0;
  if (g_retire) lmot_track_ids(g_ctx, g_ids.data(), kCap, &n_ids);      // row i -> its track's ID (rows move once dead tracks are removed)

  // arrows: moving, visible, live tracks (speed = length, yaw = direction)
  for (int i = 0; i < o.n_tracks; ++i) {
    if (g_manage[i] == 0 || !g_vis[i] || g_static[i]) continue;
    visualization_msgs::Marker a;
    a.header.frame_id = "/velodyne"; a.header.stamp = ros::Time::now();
    a.ns = "arrows"; a.id = (g_retire && i < n_ids) ? (int)(g_ids[i] % 2147483647) : i; a.type = visualization_msgs::Marker::ARROW; a.action = visualization_msgs::Marker::ADD;
    a.lifetime = ros::Duration(0.1);
    a.pose.position.x = g_targets[3 * i]; a.pose.position.y = g_targets[3 * i + 1]; a.pose.position.z = -1.73 / 2;
    a.pose.orientation = tf::createQuaternionMsgFromYaw(g_vy[2 * i + 1]);
    a.scale.x = g_vy[2 * i]; a.scale.y = 0.1; a.scale.z = 0.1;
    a.color.g = 1.0f; a.color.a = 1.0f;
    g_pub_markers.publish(a);
  }
  // points: blue = static, yellow = tentative (< 5), green = mature (5), red = coasting (> 5)
  visualization_msgs::Marker yellow = points_marker(1, 1, 1, 0), green = points_marker(2, 0, 1, 0), red = points_marker(3, 1, 0, 0),
                             blue = points_marker(4, 0, 0, 1);
  for (int i = 0; i < o.n_tracks; ++i) {
    if (g_manage[i] == 0) continue;
    geometry_msgs::Point p;
    p.x = g_targets[3 * i]; p.y = g_targets[3 * i + 1]; p.z = -1.73 / 2;
    (g_static[i] ? blue : g_manage[i] < 5 ? yellow : g_manage[i] == 5 ? green : red).points.push_back(p);
  }
  g_pub_markers.publish(yellow); g_pub_markers.publish(green); g_pub_markers.publish(red); g_pub_markers.publish(blue);
  // boxes of the visible tracks
  visualization_msgs::Marker edges;
  edges.header.frame_id = "velodyne"; edges.header.stamp = ros::Time::now();
  edges.ns = "boxes"; edges.id = 0; edges.type = visualization_msgs::Marker::LINE_LIST; edges.action = visualization_msgs::Marker::ADD;
  edges.pose.orientation.w = 1.0; edges.scale.x = 0.1; edges.color.r = 1.0f; edges.color.a = 1.0f;
  for (int b = 0; b < o.n_vis; ++b) lmot_ros::box_edges(g_visbb.data() + (size_t)b * 24, edges.points);
  g_pub_boxes.publish(edges);
}
}  // namespace

int main(int argc, char** argv) {
  ros::init(argc, argv, "obj_track");
  ros::NodeHandle nh;
  lmot_params prm;
  lmot_default_params(&prm);
  prm.max_tracks = kCap;
  prm.global_frame = 1;          // track in the dead-reckoned global frame like the reference node (main.cpp:142-195)
  int device = 0;
  nh.param<int>("cuda_device", device, 0);
  ros::NodeHandle("~").param<bool>("stamp_in_microseconds", g_stamp_us, false);
  ros::NodeHandle("~").param<bool>("retire_dead_tracks", g_retire, false);      // false: the reference's append-only table (drop-in)
  const int rc = lmot_create(&g_ctx, &prm, device);
  if (rc != LMOT_OK) { ROS_FATAL("lmot_create: %s -- this node has no CPU path", lmot_strerror(rc)); return 1; }
  if (g_retire) lmot_set_track_retirement(g_ctx, 1);
  g_pub_markers = nh.advertise<visualization_msgs::Marker>("visualization_marker", 0);
  g_pub_boxes = nh.advertise<visualization_msgs::Marker>("visualization_marker2", 0);
  ros::Subscriber sub_boxes = nh.subscribe("track_box", 160, on_boxes);
  ros::Subscriber sub_odom = nh.subscribe("/gps/odom", 1000, on_odom);
  ros::spin();
  lmot_destroy(g_ctx);
  return 0;
}
