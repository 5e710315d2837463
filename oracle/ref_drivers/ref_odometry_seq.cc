// TEST INFRASTRUCTURE.  The driver of ref_odometry.cc (included whole: the reference's laserOdometry.cpp against the stand-in
// headers, and every entry point of that driver) plus a sequence entry, for mapping_skip_frame > 1.  The per-scan entry
// ref_odom_process re-enters main() once per scan, so the loop-local frameCount (laserOdometry.cpp:217) restarts every time and
// the node publishes its clouds for every scan -- the mapping_skip_frame = 1 behaviour.  Here a whole sequence runs in ONE entry
// of main(), so frameCount counts the scans and :570 sends the clouds to the mapper only when frameCount % skipFrameNum == 0.
//   ref_odom_queue       publishes one scan's five clouds without running the loop;
//   ref_odom_run_queued  enters main() once with ros::ok() true for n turns.
// What each turn publishes is recorded by subscribers on the node's output topics: the bus delivers those messages at the next
// turn's ros::spinOnce() (and at the driver's own one after the last turn) in publication order, and every turn publishes
// /laser_odom_to_init (:521) before its clouds (:570-597).  Built into oracle/_ref/ by `make -C oracle -f ref_skip.mk`.
#include "ref_odometry.cc"
#include <vector>

namespace {
struct Turn {
  double pose[7];                  // /laser_odom_to_init: q x, y, z, w ; t
  std::vector<float> cloud[3];     // /laser_cloud_corner_last, /laser_cloud_surf_last, /velodyne_cloud_3
  bool clouds = false;             // the turn published the three clouds
};
std::vector<Turn> g_turns;
const char* const kTurnTopics[3] = {"/laser_cloud_corner_last", "/laser_cloud_surf_last", "/velodyne_cloud_3"};
}  // namespace

extern "C" {

void ref_odom_queue(const float* sharp, int n_sharp, const float* less_sharp, int n_less_sharp, const float* flat, int n_flat,
                    const float* less_flat, int n_less_flat, const float* full, int n_full, double stamp) {
  publish_cloud("/laser_cloud_sharp", sharp, n_sharp, stamp);
  publish_cloud("/laser_cloud_less_sharp", less_sharp, n_less_sharp, stamp);
  publish_cloud("/laser_cloud_flat", flat, n_flat, stamp);
  publish_cloud("/laser_cloud_less_flat", less_flat, n_less_flat, stamp);
  publish_cloud("/velodyne_cloud_2", full, n_full, stamp);
}

// runs n turns of the loop in one entry of main(); returns the number of turns recorded since ref_odom_init
int ref_odom_run_queued(int n) {
  ros::shim::Bus& b = ros::shim::Bus::get();
  auto& od = b.subscribers["/laser_odom_to_init"];
  od.clear();
  od.push_back([](const std::shared_ptr<const void>& p) {
    const nav_msgs::Odometry& m = *std::static_pointer_cast<const nav_msgs::Odometry>(p);
    Turn t;
    t.pose[0] = m.pose.pose.orientation.x; t.pose[1] = m.pose.pose.orientation.y; t.pose[2] = m.pose.pose.orientation.z;
    t.pose[3] = m.pose.pose.orientation.w;
    t.pose[4] = m.pose.pose.position.x; t.pose[5] = m.pose.pose.position.y; t.pose[6] = m.pose.pose.position.z;
    g_turns.push_back(t);
  });
  for (int w = 0; w < 3; ++w) {
    auto& s = b.subscribers[kTurnTopics[w]];
    s.clear();
    s.push_back([w](const std::shared_ptr<const void>& p) {
      if (g_turns.empty()) return;
      g_turns.back().cloud[w] = std::static_pointer_cast<const sensor_msgs::PointCloud2>(p)->xyzi;
      g_turns.back().clouds = true;
    });
  }
  b.ok_budget = n;
  int argc = 0;
  ref_laser_odometry_main(argc, nullptr);
  ros::spinOnce();   // the last turn's publications
  return (int)g_turns.size();
}

// turn i: the published odometry pose; returns 1 when the turn published the clouds for the mapper, 0 if not, -1 for no turn i
int ref_odom_turn(int i, double* pose7) {
  if (i < 0 || i >= (int)g_turns.size()) return -1;
  for (int k = 0; k < 7; ++k) pose7[k] = g_turns[i].pose[k];
  return g_turns[i].clouds ? 1 : 0;
}

// cloud `which` (0 corner_last, 1 surf_last, 2 full) that turn i published: number of points, up to cap of them into out
int ref_odom_turn_cloud(int i, int which, float* out, int cap) {
  if (i < 0 || i >= (int)g_turns.size() || which < 0 || which > 2) return -1;
  const std::vector<float>& v = g_turns[i].cloud[which];
  const int n = (int)(v.size() / 4);
  if (out) std::memcpy(out, v.data(), sizeof(float) * 4 * (size_t)(n < cap ? n : cap));
  return n;
}

}  // extern "C"
