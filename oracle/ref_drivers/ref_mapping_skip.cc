// TEST INFRASTRUCTURE.  The driver of ref_mapping.cc (included whole: the reference's laserMapping.cpp against the stand-in
// headers, and every entry point of that driver) plus what a scan the odometry does not send to the mapper needs
// (mapping_skip_frame > 1, laserOdometry.cpp:570): an entry that delivers only its odometry message, and the pose
// laserOdometryHandler publishes for it on /aft_mapped_to_init_high_frec (laserMapping.cpp:197-229).
// Built into oracle/_ref/ by `make -C oracle -f ref_skip.mk`.
#include "ref_mapping.cc"

extern "C" {

// one odometry message without clouds: laserOdometryHandler publishes the high-frequency pose; process() finds no clouds and
// leaves, and the queued message is dropped by the next mapped frame (:239-240)
int ref_map_odometry_only(const double* q_wodom_curr, const double* t_wodom_curr, double stamp) {
  nav_msgs::Odometry od;
  od.header.stamp = ros::Time(stamp);
  od.pose.pose.orientation.x = q_wodom_curr[0]; od.pose.pose.orientation.y = q_wodom_curr[1];
  od.pose.pose.orientation.z = q_wodom_curr[2]; od.pose.pose.orientation.w = q_wodom_curr[3];
  od.pose.pose.position.x = t_wodom_curr[0]; od.pose.pose.position.y = t_wodom_curr[1]; od.pose.pose.position.z = t_wodom_curr[2];
  ros::Publisher("/laser_odom_to_init").publish(od);
  ros::spinOnce();
  try { process(); } catch (const ref_sync::FrameDone&) {}
  return 0;
}

// the pose published on /aft_mapped_to_init_high_frec ; returns the number of messages published so far
long ref_map_high_frec_pose(double* q, double* t) {
  ros::shim::Bus& b = ros::shim::Bus::get();
  auto it = b.last.find("/aft_mapped_to_init_high_frec");
  if (it == b.last.end()) return 0;
  const nav_msgs::Odometry& m = *std::static_pointer_cast<const nav_msgs::Odometry>(it->second);
  q[0] = m.pose.pose.orientation.x; q[1] = m.pose.pose.orientation.y; q[2] = m.pose.pose.orientation.z; q[3] = m.pose.pose.orientation.w;
  t[0] = m.pose.pose.position.x; t[1] = m.pose.pose.position.y; t[2] = m.pose.pose.position.z;
  return b.count["/aft_mapped_to_init_high_frec"];
}

}  // extern "C"
