/* aloam_io.h -- data formats either side of the registration path (SURVEY.md section 8 f-3).
 *
 * Host-side helpers only: nothing here touches the GPU, and nothing here is needed by aloam_b200.h.  They exist so
 * that real recordings can be replayed through aloam_scan_stream / aloam_scan_to_pose without ROS, PCL or OpenCV:
 *
 *   KITTI odometry velodyne scans   kittiHelper.cpp:25-35 (read_lidar_data), :140-151 (x, y, z, intensity as float32)
 *                                   -- the file layout IS the packed stride-4 layout of aloam_cloud_view
 *   KITTI ground-truth poses        kittiHelper.cpp:97-113 (12 numbers per line parsed with stof, i.e. through float;
 *                                   camera frame -> lidar frame with R_transform = [0 0 1; -1 0 0; 0 -1 0], :78-80)
 *   sensor_msgs/PointCloud2 payload of a pcl::PointCloud<pcl::PointXYZI> (what every A-LOAM topic carries,
 *                                   scanRegistration.cpp:413-441): 32-byte points, x@0 y@4 z@8 intensity@16
 *                                   -- the stride-8 layout of aloam_cloud_view
 */
#ifndef ALOAM_IO_H
#define ALOAM_IO_H
#ifdef __cplusplus
extern "C" {
#endif

/* number of points in a KITTI .bin scan (file size / 16, like `num_elements / 4` at kittiHelper.cpp:29,143) ; -1: cannot open */
long aloam_io_kitti_bin_points(const char* path);
/* reads at most `capacity_points` points as packed x,y,z,intensity ; returns the number read, -1: cannot open */
long aloam_io_read_kitti_bin(const char* path, float* xyzi, long capacity_points);
/* one line of a KITTI poses file -> row-major 3x4 ; every number goes through float like stof() at :106 ; 0 = ok */
int aloam_io_parse_kitti_pose(const char* line, double T[12]);
/* q = normalize(q_transform * Quaternion(R)), t = q_transform * T[:,3]   (kittiHelper.cpp:110-113) ; q is x,y,z,w */
void aloam_io_kitti_pose_to_lidar(const double T[12], double q[4], double t[3]);
/* the inverse direction for evaluation tools: a lidar-frame pose back to a KITTI row-major 3x4 (camera frame) */
void aloam_io_lidar_pose_to_kitti(const double q[4], const double t[3], double T[12]);

/* packed x,y,z,intensity -> PointCloud2 `data` of pcl::PointXYZI (point_step 32, padding zeroed) and back.  `unpack`
 * takes the field offsets of the message, so clouds whose fields sit elsewhere (e.g. a velodyne driver's
 * x,y,z,intensity,ring layout with point_step 22 or 32) can be read too. */
void aloam_io_pack_pointxyzi(const float* xyzi, long n, unsigned char* data32);
int aloam_io_unpack_points(const unsigned char* data, long n, int point_step, int off_x, int off_y, int off_z,
                           int off_intensity /* < 0: none, intensity = 0 */, float* xyzi);
/* PointCloud2 `data` of a driver cloud with a per-return ring field -> packed x,y,z,ring: the raw scan of
 * cfg.ring_source = ALOAM_RING_FIELD (float 3 = the ring id).  ring_type is the sensor_msgs/PointField datatype of the ring
 * field: 2 (UINT8) or 4 (UINT16), the types Velodyne (PointXYZIR: uint16 at byte 20 of 32) and Ouster drivers publish;
 * little-endian payloads.  Returns 0, or -1 for another ring_type or an offset whose field does not fit in point_step. */
int aloam_io_unpack_points_ring(const unsigned char* data, long n, int point_step, int off_x, int off_y, int off_z, int off_ring,
                                int ring_type, float* xyzr);

#ifdef __cplusplus
}
#endif
#endif
