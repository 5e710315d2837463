// TEST INFRASTRUCTURE.  The driver of ref_mapping.cc (included whole: the reference's laserMapping.cpp against the stand-in
// headers, and every entry point of that driver) plus read-back of the three clouds the node publishes per frame cadence:
// /laser_cloud_surround (laserMapping.cpp:806-821, every 5th frame), /laser_cloud_map (:823-836, every 20th frame) and
// /velodyne_cloud_registered (:838-848, every frame).  Built into oracle/_ref/ by `make -C oracle -f ref_clouds.mk`.
#include "ref_mapping.cc"

extern "C" {

// the last message published on `topic` (one of the three above): its size in *n, up to cap points of it into out (x, y, z,
// intensity); returns the number of messages published on the topic so far
long ref_map_published_cloud(const char* topic, float* out, int cap, int* n) {
  ros::shim::Bus& b = ros::shim::Bus::get();
  *n = 0;
  auto it = b.last.find(topic);
  if (it == b.last.end()) return 0;
  const sensor_msgs::PointCloud2& m = *std::static_pointer_cast<const sensor_msgs::PointCloud2>(it->second);
  *n = (int)(m.xyzi.size() / 4);
  for (int i = 0; i < *n && i < cap; ++i) for (int k = 0; k < 4; ++k) out[4 * i + k] = m.xyzi[4 * (size_t)i + k];
  return b.count[topic];
}

}  // extern "C"
