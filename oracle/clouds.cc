// ORACLE (test infrastructure) -- the restatements behind the clouds alaserMapping publishes (laserMapping.cpp:806-848), as a flat C
// interface for ctypes (oracle/pyclouds.py).  Built into oracle/libclouds.so by `make -C oracle -f clouds.mk libclouds.so`.
#include "oracle.h"

using namespace orc;

extern "C" {

// pointAssociateToMap (laserMapping.cpp:154-163) over a cloud: q_w_curr * p + t_w_curr in double in Eigen's operation order
// (x7 = parameters[7]: q x, y, z, w ; t), stored as float, intensity kept -- what /velodyne_cloud_registered carries (:838-848)
void orc_associate_to_map(const double x7[7], const float* in, int n, float* out) {
  const Quat q{x7[0], x7[1], x7[2], x7[3]};
  const Vec3 t{x7[4], x7[5], x7[6]};
  for (int i = 0; i < n; ++i) {
    const Vec3 w = rotate(q, Vec3{(double)in[4 * i], (double)in[4 * i + 1], (double)in[4 * i + 2]}) + t;
    out[4 * i] = (float)w.x; out[4 * i + 1] = (float)w.y; out[4 * i + 2] = (float)w.z; out[4 * i + 3] = in[4 * i + 3];
  }
}

}  // extern "C"
