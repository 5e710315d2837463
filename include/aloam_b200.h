/* aloam_b200.h -- C ABI of the H100-native A-LOAM per-scan registration hot path.
 *
 * The reference (HKUST-Aerial-Robotics/A-LOAM) has NO library / plugin / FFI boundary: the hot path is inline
 * code in three ROS node `main`s.  This header creates the boundary at exactly the seam between the node shells
 * (topic I/O, queues, publishing -- unchanged, stay in the ROS nodes) and the per-scan algorithms (replaced).
 * Each entry point names the reference code it replaces (file:line into the reference tree).  INTEGRATION.md
 * shows the call a maintainer adds at each site.
 *
 * Conventions
 *   - plain C99 types, no exceptions cross the boundary; every call returns 0 (ALOAM_OK) or a negative error.
 *   - points are 4 floats x,y,z,intensity (pcl::PointXYZI's meaningful fields, include/aloam_velodyne/common.h:43);
 *     `stride_floats` = 4 for packed arrays, 8 for PCL's 32-byte PointXYZI, so a pcl::PointCloud's storage can be
 *     passed without repacking.  intensity = scanID + 0.1*relTime exactly as scanRegistration.cpp:239.
 *   - quaternions are Eigen/Ceres parameter order x,y,z,w; poses are caller-owned in/out arrays exactly like
 *     para_q/para_t (laserOdometry.cpp:97-98) and parameters[7] (laserMapping.cpp:110).
 *   - inputs are borrowed for the duration of the call; output views point into ctx-owned pinned host memory and
 *     stay valid until the next call on the same ctx.  One ctx per calling thread (each reference node calls from
 *     exactly one thread); a ctx is not thread-safe; calls are synchronous.
 *   - soft conditions mirror the reference and are NOT errors: < 10 correspondences (laserOdometry.cpp:488-491)
 *     sets ALOAM_FLAG_FEW_CORRESPONDENCES; a thin map (corner <= 10 or surf <= 50, laserMapping.cpp:554,730-733)
 *     skips the optimisation, leaves the pose unchanged and sets ALOAM_FLAG_MAP_TOO_THIN.
 *   - there is NO CPU fallback: if the CUDA device or kernels are unavailable aloam_create fails.
 */
#ifndef ALOAM_B200_H_
#define ALOAM_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define ALOAM_OK 0
#define ALOAM_ERR_INVALID_ARG (-1)
#define ALOAM_ERR_UNSUPPORTED_SCANS (-2) /* scanRegistration.cpp:472-476: only 16, 32 or 64 scan lines under
                                            ALOAM_RING_ELEVATION; 1..64 under ALOAM_RING_FIELD (1..ALOAM_MAX_RINGS
                                            through aloam_create_wide) */
#define ALOAM_ERR_EMPTY_CLOUD (-3)       /* no point survives the NaN / minimum-range filter */
#define ALOAM_ERR_CAPACITY (-4)          /* more points than the ctx was created for */
#define ALOAM_ERR_CUDA (-5)
#define ALOAM_ERR_NO_DEVICE (-6)
#define ALOAM_ERR_RING_TOO_LARGE (-7)    /* a single ring holds more than ALOAM_MAX_RING_POINTS returns */
#define ALOAM_ERR_NOT_RING_MAJOR (-8)    /* "last" cloud with an int(intensity) outside 0..63 (0..127 in a context of
                                            aloam_create_wide with n_scans > 64) or two or more below an earlier
                                            point's: every scanRegistration output has int_i >= max_{j<i} int_j - 1, and the
                                            association's break tables rely on it (laserOdometry.cpp:310-361,400-455) */
#define ALOAM_ERR_STATE (-9)             /* call sequence error, e.g. register before set_last */
#define ALOAM_ERR_COMM (-10)
#define ALOAM_ERR_SNAPSHOT (-11)         /* snapshot malformed, of another format version, or taken under a configuration that
                                            changes results (aloam_lane_restore, aloam_snapshot_check) */

#define ALOAM_MAX_RING_POINTS 4096
#define ALOAM_MAX_RINGS 128   /* the most rings a context takes: through aloam_create_wide, ALOAM_RING_FIELD only */
#define ALOAM_MAX_BATCH 16
#define ALOAM_MAX_CUBE_POINTS 262144   /* 2^18: the most points one map cube holds with cube growth on (aloam_set_cube_growth) */

#define ALOAM_FLAG_FEW_CORRESPONDENCES 1
#define ALOAM_FLAG_MAP_TOO_THIN 2
#define ALOAM_FLAG_INITIALISED_ONLY 4 /* first frame: laserOdometry.cpp:267-271 */
#define ALOAM_FLAG_CUBE_OVERFLOW 8    /* map cube store: a cube was at its capacity (one slab of 16 k corner / 64 k surf points with
                                         cube growth off, its ceiling with growth on), no free run of slabs was left, the submap was
                                         truncated, or cubes were left out of the re-filter; see aloam_set_cube_growth */

typedef struct aloam_ctx aloam_ctx;

/* The constants of the hot path (SURVEY.md section 5 "config / flags").  aloam_default_config fills the values
 * of launch/aloam_velodyne_{VLP_16,HDL_32,HDL_64}.launch:3-13 for n_scans = 16 / 32 / 64. */
typedef struct aloam_config {
  int n_scans;           /* scan_line                       scanRegistration.cpp:466 */
  float minimum_range;   /* minimum_range                   scanRegistration.cpp:468 */
  float line_res;        /* mapping_line_resolution         laserMapping.cpp:902-906 */
  float plane_res;       /* mapping_plane_resolution */
  int outer_iters;       /* 2   laserOdometry.cpp:278, laserMapping.cpp:562; 1..4 */
  int inner_iters;       /* 4   options.max_num_iterations, laserOdometry.cpp:496, laserMapping.cpp:715; >= 0 */
  double huber;          /* 0.1 HuberLoss, laserOdometry.cpp:284, laserMapping.cpp:565; > 0.  huber, outer_iters and inner_iters
                            apply to both solves, scan-to-scan and scan-to-map (the reference hard-codes the same values in both
                            nodes); line_res and plane_res must be > 0 too */
  double dist_sq_thresh; /* 25  DISTANCE_SQ_THRESHOLD, laserOdometry.cpp:65; compared as the reference does, a float squared
                            distance against this double */
  double nearby_scan;    /* 2.5 NEARBY_SCAN, laserOdometry.cpp:66; >= 1, may be +inf (the ring-window walks never break) */
  int device;            /* CUDA device ordinal */
  int max_points;        /* capacity of one raw scan (reference: 400000 static arrays, scanRegistration.cpp:66-69); 1 .. 2^25 - 1
                            (2^24 - 1 above 64 rings, see aloam_create_wide): the association index packs a point's index and
                            ring into one int.  Larger values are ALOAM_ERR_INVALID_ARG */
  int max_map_points;    /* capacity of the uploaded submap, per cloud type (0 = mapping not used); at most 2^30, larger
                            values are rejected by aloam_create with ALOAM_ERR_INVALID_ARG */
  int max_batch;         /* trajectories a context can advance in lockstep (aloam_scan_stream_batch), or lanes of
                            aloam_scan_stream_lanes; 1..ALOAM_MAX_BATCH, default 1 */
  int distortion;        /* 0 (reference build) or 1: #define DISTORTION of laserOdometry.cpp:59 -- per-point interpolation ratio
                            s = (intensity - int(intensity)) / SCAN_PERIOD in TransformToStart (:113-118) and in the
                            residual blocks (:376-379, 470-473; slerp inside the functors, lidarFactor.hpp:27-33).
                            intensity = ring + 0.1 relTime is the reference's float: on rings 64..127 its fraction, and so s, is
                            quantised at 2^-17 instead of 2^-18, as scanRegistration.cpp's own float is */
  int max_ring_points;   /* capacity of one scan ring, multiple of 32, <= ALOAM_MAX_RING_POINTS (default).  Smaller rings take
                            less shared memory per ring CTA, so more of them are resident per SM (batched streams) */
  int mapping_skip_frame; /* mapping_skip_frame laserOdometry.cpp:191, launch/...:6 -- the mapped stream calls map every k-th scan
                            of a trajectory and give the others the high-frequency pose (see aloam_scan_stream_mapped).  Default 1
                            (every scan); 0 counts as 1 (zero-initialised tail of an older caller); < 0 is rejected by aloam_create */
  int ring_source;       /* where a raw return's ring id comes from (see below); 0 = ALOAM_RING_ELEVATION, the default and what a
                            zero-initialised tail of an older caller gets; any other value than 0 or 1 is ALOAM_ERR_INVALID_ARG */
} aloam_config;

/* Ring sources (aloam_config.ring_source).  Every entry point that takes a raw scan uses it: aloam_extract_features,
 * aloam_scan_to_pose(_device) and every stream call, device-resident raws included.
 *   ALOAM_RING_ELEVATION  the reference's elevation formula of the configured Velodyne (scanRegistration.cpp:166-205);
 *                         n_scans must be 16, 32 or 64.
 *   ALOAM_RING_FIELD      the sensor driver's ring: float 3 of every raw point (the 4th float, at stride 4 and 8 alike; the
 *                         reference never reads that slot of a raw scan).  n_scans may be 1..64, 1..128 through
 *                         aloam_create_wide.  After the NaN and
 *                         minimum-range filters a return's ring is w = float 3 when w is finite, integral and 0 <= w < n_scans;
 *                         any other w drops the return as an out-of-range formula id does (it does not count in the sweep walk
 *                         either, scanRegistration.cpp:174-175).  Everything after the ring binning is unchanged: the azimuth
 *                         walk, relTime, intensity = ring + 0.1 relTime, the per-ring features and voxel filter.
 *                         The ids must number the beams in elevation order, in either direction (Velodyne drivers put ring 0
 *                         at the lowest beam, Ouster drivers at the highest): the scan-to-scan association's NEARBY_SCAN
 *                         window assumes that neighbouring ids are neighbouring beams.  This is not checked.  A ring still
 *                         holds at most cfg.max_ring_points returns (ALOAM_ERR_RING_TOO_LARGE).
 * aloam_default_config(cfg, n) fills the VLP-16 / HDL-32 launch values for every n other than 64, and ring_source = 0: a caller
 * with another sensor sets n_scans, ring_source and, where its sensor needs them, minimum_range, line_res and plane_res. */
#define ALOAM_RING_ELEVATION 0
#define ALOAM_RING_FIELD 1

typedef struct aloam_cloud_view {
  const float* data;
  int n;
  int stride_floats; /* 4 or 8 */
} aloam_cloud_view;

typedef struct aloam_stats {
  int n_corner_corr, n_plane_corr; /* residual blocks built in the LAST outer iteration */
  int lm_iters;                    /* sum of trust-region iterations over the outer iterations */
  int accepted_steps;
  int flags;
  int termination[4];              /* per outer iteration: 0 max-iters 1 gradient 2 parameter 3 function 4 empty 5 failure */
  double init_cost, final_cost;    /* of the last outer iteration */
  float ms_total;                  /* device time of the call, CUDA events */
} aloam_stats;

void aloam_default_config(aloam_config* cfg, int n_scans);
int aloam_create(const aloam_config* cfg, aloam_ctx** out);
/* aloam_create_wide: everything aloam_create accepts, giving the same context, and also ring_source = ALOAM_RING_FIELD with
 * n_scans 65..ALOAM_MAX_RINGS (128-beam lidars: Ouster OS1/OS2-128, Velodyne VLS-128, Hesai Pandar128, RoboSense Ruby).
 * Elevation rings stay 16 / 32 / 64 (ALOAM_ERR_UNSUPPORTED_SCANS, as 0 or 129 driver rings), a ring source other than 0 or 1
 * stays ALOAM_ERR_INVALID_ARG.  With n_scans > 64:
 *   - the context's ring-indexed tables are 128 wide: an int(intensity) of 0..127 is a ring of aloam_odometry_set_last's
 *     clouds (ALOAM_ERR_NOT_RING_MAJOR above that);
 *   - cfg.max_points > 2^24 - 1 is ALOAM_ERR_INVALID_ARG: the association index packs a point's index into 24 bits, and
 *     index 2^24 - 1 on ring 127 would pack to INT_MAX, the search's "no candidate" word (2^25 - 1 at up to 64 rings);
 *   - every lane allocates 64 x (32 x (156 + max_ring_points) + 8 x (6 + ceil(max_points / 1024)) + 12 x 1040) bytes more
 *     than at 64 rings (64 more rings of: two staging sets of 12 + 120 + 24 + max_ring_points points, the ring-binning
 *     tables, and the twelve association indexes of 128 buckets): 9.7 MB per lane at max_ring_points = 4096 and
 *     max_points = 400000, 5.5 MB at 2048 (arithmetic, not a measurement);
 *   - 12 sharp and 24 flat query slots per ring: the fused paths' association covers 1536 + 3072 queries.
 * Snapshots of a 128-ring context restore only into a context with the same n_scans (ALOAM_ERR_SNAPSHOT elsewhere, every
 * context of aloam_create included).  Prior maps, relocalisation, recovery, cube growth, the registered sink and per-row
 * records do not depend on rings and work unchanged.  The recommended max_ring_points for a 128-beam sensor is in README.md. */
int aloam_create_wide(const aloam_config* cfg, aloam_ctx** out);
int aloam_destroy(aloam_ctx* ctx);
const char* aloam_strerror(int code);

/* ---- feature extraction: replaces scanRegistration.cpp:129-408 (body of laserCloudHandler between fromROSMsg
 * and the five toROSMsg/publish calls at :413-441).  raw = the PointXYZ cloud in arrival order. */
int aloam_extract_features(aloam_ctx* ctx, aloam_cloud_view raw, aloam_cloud_view* full,
                           aloam_cloud_view* sharp, aloam_cloud_view* less_sharp, aloam_cloud_view* flat,
                           aloam_cloud_view* less_flat);

/* ---- scan-to-scan odometry.
 * aloam_odometry_set_last replaces laserOdometry.cpp:554-568 (swap in the less-sharp / less-flat clouds and
 * rebuild kdtreeCornerLast / kdtreeSurfLast).  aloam_odometry_register replaces :274-502 (the two
 * association + ceres::Solve rounds); q_last_curr/t_last_curr are para_q/para_t, warm-started by the caller. */
int aloam_odometry_set_last(aloam_ctx* ctx, aloam_cloud_view corner_last, aloam_cloud_view surf_last);
int aloam_odometry_register(aloam_ctx* ctx, aloam_cloud_view sharp, aloam_cloud_view flat,
                            double q_last_curr[4], double t_last_curr[3], aloam_stats* stats);

/* ---- scan-to-map refinement.
 * aloam_map_upload replaces laserMapping.cpp:531-539 + :558-559 (the gathered 5x5x3-cube submap and the two
 * kd-tree builds).  aloam_mapping_register replaces :554-729; the stacks are the voxel-filtered current
 * corner / surf clouds of :542-550 (use aloam_voxel_filter for those), q_t_w_curr = parameters[7].
 * Input views of aloam_map_upload / aloam_odometry_* / aloam_mapping_* may point to host memory (pageable or pinned)
 * or to device memory: the copy kind is inferred from the address (unified virtual addressing). */
int aloam_map_upload(aloam_ctx* ctx, aloam_cloud_view corner_map, aloam_cloud_view surf_map);
int aloam_mapping_register(aloam_ctx* ctx, aloam_cloud_view corner_stack, aloam_cloud_view surf_stack,
                           double q_t_w_curr[7], aloam_stats* stats);
/* pcl::VoxelGrid<PointXYZI> with a cubic leaf: laserMapping.cpp:543-549 (scan stacks), scanRegistration.cpp:401-405 */
int aloam_voxel_filter(aloam_ctx* ctx, aloam_cloud_view in, float leaf, aloam_cloud_view* out);

/* ---- fused, device-resident pipeline (SURVEY.md 8f-2): one raw scan in, world pose out; the feature clouds
 * and the "last" clouds never leave the GPU.  Equivalent to extract_features -> odometry_register ->
 * pose integration (laserOdometry.cpp:504-505) -> odometry_set_last, with the reference's warm start.
 * First call only initialises (laserOdometry.cpp:267-271).  q_w_curr/t_w_curr are outputs. */
int aloam_scan_to_pose(aloam_ctx* ctx, aloam_cloud_view raw, double q_w_curr[4], double t_w_curr[3],
                       aloam_stats* stats);
/* same, raw scan already in device memory (4-float packed points); used for HBM-resident measurements */
int aloam_scan_to_pose_device(aloam_ctx* ctx, const float* d_raw_xyzi, int n, double q_w_curr[4],
                              double t_w_curr[3], aloam_stats* stats);
/* pipelined form for a sequence of scans: upload, ring binning, per-ring feature extraction, compaction + index build
 * and association + LM of consecutive scans overlap on five CUDA streams (the overlap the reference gets from its three
 * ROS processes); results identical to calling aloam_scan_to_pose once per scan, in any interleaving with it.  device_resident != 0: raws[k].data are device pointers (stride 4).
 * poses: n_scans x 7 doubles (q_w xyzw, t_w). */
int aloam_scan_stream(aloam_ctx* ctx, const aloam_cloud_view* raws, int n_scans, int device_resident, double* poses,
                      aloam_stats* stats_last);
/* batched form (BASELINE configs[4], SURVEY.md 8b "aloam_*_batch"): `batch` independent trajectories advance in lockstep and
 * SHARE every kernel launch (ring CTAs of all trajectories in one grid, one LM cluster per trajectory, ...), so one
 * context and one host thread fill the GPU.  raws: n_scans x batch views, scan-major (raws[k * batch + b] = scan k of
 * trajectory b); poses: n_scans x batch x 7 doubles in the same order; stats_last: `batch` entries or NULL.  Every
 * trajectory keeps the reference's warm-start chain (laserOdometry.cpp:97-98,504-505) and its result is bit-identical to
 * running it alone through aloam_scan_stream.  batch <= cfg.max_batch; all trajectories of a context share the frame
 * counter (the first scan of a fresh / reset context only initialises, laserOdometry.cpp:267-271). */
int aloam_scan_stream_batch(aloam_ctx* ctx, const aloam_cloud_view* raws, int n_scans, int batch, int device_resident,
                            double* poses, aloam_stats* stats_last);
/* the whole pipeline of the three reference nodes in one call (SURVEY.md 8 f-2): as aloam_scan_stream, and every scan's
 * less-sharp / less-flat clouds and odometry pose are handed ON THE DEVICE to the scan-to-map stage (one aloam_mapper_step
 * per scan, on its own stream, overlapping the odometry of the following scans) -- what the reference ships over
 * /laser_cloud_corner_last, /laser_cloud_surf_last and /laser_odom_to_init (laserOdometry.cpp:570-591 ->
 * laserMapping.cpp:278-288, 142-152).  odom_poses / map_poses: n_scans x 7 doubles (q xyzw, t): laser_odom_to_init and
 * aft_mapped_to_init.  Identical to calling aloam_scan_to_pose + aloam_mapper_step per scan; if any scan's mapper step would
 * have returned ALOAM_ERR_CAPACITY (a voxel index range beyond the sort key), the call fills both pose arrays and returns
 * ALOAM_ERR_CAPACITY.  Needs cfg.max_map_points > 0.
 * After aloam_comm_init (every rank fed the same scans) the scan-to-map stage is sharded: each rank keeps the whole cube store,
 * indexes and searches only its x-slabs of the gathered submap, and the ranks meet in the all-reduce of the normal equations;
 * all ranks return the same poses (equal to a single-GPU run to rounding of the summation order).
 * cfg.mapping_skip_frame = k (laserOdometry.cpp:191, 570-597; every launch file sets 1, the default): a trajectory's scans are
 * numbered from 0 at its START -- for this call and _mapped_batch the context's first scan after creation or
 * aloam_reset_odometry -- and the number carries over between calls.
 *   - scan j with j % k == 0 is MAPPED: its mapper frame is the one described above, and its map_poses row is the refined pose
 *     (/aft_mapped_to_init);
 *   - every other scan is SKIPPED: no mapper frame runs for it and the cube store does not change; its map_poses row is the
 *     high-frequency pose of laserMapping.cpp:197-229 (/aft_mapped_to_init_high_frec), q = q_wmap_wodom * q_wodom,
 *     t = q_wmap_wodom * t_wodom + t_wmap_wodom, with the T_wmap_wodom left by the trajectory's latest mapped scan, in the
 *     operation order of Eigen (bit-identical to aloam_mapper_debug_state's T composed on the host in that order).
 * So the map poses equal aloam_mapper_step run on exactly the mapped scans, with the composition for the others.  odom_poses,
 * stats_last, ALOAM_ERR_CAPACITY and ALOAM_FLAG_CUBE_OVERFLOW keep their meaning; the last two come from mapped scans only.  A
 * sharded job skips the same scans on every rank.  The reference's real-time drop of queued frames (laserMapping.cpp:299-303)
 * is not modelled: an offline stream maps every k-th scan, which is what the reference does whenever its mapper keeps up.
 * aloam_mapper_step does not count scans: a caller skips a frame by not calling it. */
int aloam_scan_stream_mapped(aloam_ctx* ctx, const aloam_cloud_view* raws, int n_scans, int device_resident, double* odom_poses,
                             double* map_poses, aloam_stats* stats_last);
/* aloam_scan_stream_mapped for `batch` independent trajectories ("lanes") in one context, laid out as aloam_scan_stream_batch:
 * raws n_scans x batch views, scan-major; odom_poses / map_poses n_scans x batch x 7 doubles each; stats_last `batch` entries
 * (odometry stats) or NULL.  The odometry of all lanes shares every launch, exactly as aloam_scan_stream_batch (its poses are
 * bit-identical to that call's), and so does the scan-to-map stage: one frame per scan covers every lane.  For every lane
 * b, odom_poses[:, b], map_poses[:, b] and the lane's cube store are bit-identical to running trajectory b alone through
 * aloam_scan_stream_mapped on a fresh context with the same config; batch = 1 IS that call.  State carries over between calls.
 * With cfg.mapping_skip_frame = k every lane maps its scans j % k == 0 (all lanes together, every k-th step) and gets the
 * high-frequency pose for the others, as aloam_scan_stream_mapped.
 * Lane 0's cube store is the one aloam_mapper_step uses; the stores of lanes 1 .. batch-1 are created on the first call that
 * uses them (on allocation failure ALOAM_ERR_CUDA, before any state changes).  Each lane owns its slab pool (1024 x (16 k +
 * 64 k) points x 16 B = 1.34 GB at the default caps), its re-filter sort buffers (75 x (16 k + 64 k) = 6.1 M keys, about
 * 200 MB) and registration buffers that scale with cfg.max_points and cfg.max_map_points (about 0.2 GB at 400 000 each):
 * about 1.75 GB per lane, 28 GB at 16 lanes (arithmetic, not measured).
 * Errors: ALOAM_ERR_INVALID_ARG when batch > cfg.max_batch, cfg.max_map_points <= 0 or map_poses is NULL; ALOAM_ERR_STATE
 * after aloam_comm_init with world > 1 (sharded mapping serves one trajectory); ALOAM_ERR_CAPACITY, after filling both pose
 * arrays, when a frame of any lane met a voxel index range beyond the sort key.  Any other failure drains the streams and
 * resets the odometry, as aloam_scan_stream does. */
int aloam_scan_stream_mapped_batch(aloam_ctx* ctx, const aloam_cloud_view* raws, int n_scans, int batch, int device_resident,
                                   double* odom_poses, double* map_poses, aloam_stats* stats_last);

/* Lane-scheduled streams: the `batch` lanes of a context run trajectories that start and end independently, so a server
 * replaying recordings of different lengths refills a lane as soon as its trajectory ends instead of waiting for the longest
 * one of a group.  lane_ops (n_scans x batch ints, scan-major like raws / odom_poses / map_poses) says per step and lane:
 *   ALOAM_LANE_START  the first scan of a new trajectory: the lane's odometry (and, mapped, its cube store) is reset first;
 *   ALOAM_LANE_SCAN   the next scan of the trajectory the lane runs;
 *   ALOAM_LANE_IDLE   no scan: the lane's trajectory, if any, has ended (its view is not read; its pose rows are NaN).
 * Lifecycle: START, then SCAN at every step, then IDLE until the next START (a START may also directly follow a SCAN).  An
 * IDLE step ends the trajectory; to pause one, save it with aloam_lane_save and resume it later with aloam_lane_restore, in
 * any lane of any context (below).  Lanes batch .. cfg.max_batch-1 are IDLE at every step of the call.
 * A START scan only initialises (laserOdometry.cpp:267-271): its odometry pose is the identity and, mapped, it is the first
 * mapper frame on a freshly reset cube store.
 * map_poses == NULL: odometry only, as aloam_scan_stream_batch; otherwise scan-to-map too, as aloam_scan_stream_mapped_batch
 * (needs cfg.max_map_points > 0).  A trajectory keeps the mode of the call that started it.
 * Results: for every trajectory, its odometry poses, its map poses and its final cube store are bit-identical to running it
 * alone through aloam_scan_stream (aloam_scan_stream_mapped) on a fresh context with the same config, whatever its lane,
 * its start step and the other lanes' schedules.  Each step packs its non-idle lanes into one set of launches; a step where
 * every lane is IDLE issues nothing.  Lane state carries over between calls, so a trajectory may span several calls.
 * cfg.mapping_skip_frame = k: a lane's scan index restarts at 0 with every START (a START is always mapped), and scan j of the
 * trajectory is mapped when j % k == 0, skipped (high-frequency pose, see aloam_scan_stream_mapped) otherwise.  A step packs
 * only its mapped lanes into the mapper frame; a step without one issues no frame, and one launch serves all its skipped lanes.
 * stats_last[b] (`batch` entries, or NULL): the odometry stats of lane b's last non-idle step of this call,
 * ALOAM_FLAG_INITIALISED_ONLY when that step was a START, all zero when the lane was idle all call.
 * Errors before any state changes: ALOAM_ERR_INVALID_ARG for an op outside {0, 1, 2}, batch > cfg.max_batch or map_poses
 * without cfg.max_map_points; ALOAM_ERR_STATE for a SCAN to a lane that is not running at that step (or that was started in
 * the other mode), and after aloam_comm_init with world > 1.  Any other failure (an empty or oversized scan included) drains
 * the streams and resets the odometry, after which no lane is running; ALOAM_ERR_CAPACITY keeps its meaning of
 * aloam_scan_stream_mapped_batch (pose arrays filled, lanes go on).
 * Once a context has run this call, aloam_scan_to_pose*, aloam_scan_stream, _batch, _mapped and _mapped_batch (the calls
 * driven by the context's shared frame counter) return ALOAM_ERR_STATE until aloam_reset_odometry, which also ends every lane. */
#define ALOAM_LANE_IDLE 0
#define ALOAM_LANE_SCAN 1
#define ALOAM_LANE_START 2
int aloam_scan_stream_lanes(aloam_ctx* ctx, const aloam_cloud_view* raws, const int* lane_ops, int n_scans, int batch,
                            int device_resident, double* odom_poses, double* map_poses, aloam_stats* stats_last);
int aloam_reset_odometry(aloam_ctx* ctx); /* forget pose, warm start and "last" clouds (all trajectories); ends every lane of
                                             aloam_scan_stream_lanes and allows the lockstep calls again; the next scan of
                                             every lane is scan 0 for cfg.mapping_skip_frame */

/* ---- lane snapshots: suspend a trajectory of aloam_scan_stream_lanes and resume it in any lane of any context, on any GPU, in
 * this process or a later one -- to time-slice more trajectories than a context has lanes, park a vehicle whose scans stop for a
 * while, move a trajectory to balance load, or survive a restart in the middle of a long recording.
 * aloam_lane_save writes the state later scans of `lane` depend on, as it stands after the last stream call (the call changes
 * nothing): its warm start and world pose, its "last" less-sharp / less-flat clouds, the index of its next scan and its mode,
 * and, mapped, its cube store.  out: device memory of the context's device (16-byte aligned), or host memory, pinned or pageable
 * (the copy kind is inferred from the address; the store's points go through the staging buffer of aloam_mapper_export).
 * *n_bytes is always set to the snapshot's size; out = NULL with capacity = 0 asks for the size only; capacity < *n_bytes
 * returns ALOAM_ERR_CAPACITY and writes nothing.  ALOAM_ERR_STATE unless the context runs lanes and `lane` is running.  (The
 * lockstep calls have no snapshots: aloam_scan_stream_lanes with batch 1 is the single-trajectory call.)  Size: 256 B + 16 B per
 * "last" point, and, mapped, 39 424 B + 16 B per map point.
 * aloam_lane_restore makes `lane` (0 <= lane < cfg.max_batch) run the saved trajectory: a lanes call that continues it with
 * ALOAM_LANE_SCAN, in the saved mode (map_poses set or not), gives exactly what the uninterrupted trajectory would have -- odometry
 * and map poses, stats, cube store, published and registered clouds.  blob: as `out` of aloam_lane_save, n_bytes its size
 * exactly.  It needs the configuration the snapshot was taken under in every field that can change a result: n_scans,
 * ring_source, minimum_range, outer_iters, inner_iters, huber, dist_sq_thresh, nearby_scan and distortion, and for a mapped snapshot also
 * line_res, plane_res, mapping_skip_frame, max_map_points and the slab capacities min(16384, max_points) / min(65536, max_points)
 * (floating-point fields compared bit for bit).  max_points beyond the slab capacities, max_batch, max_ring_points and device do
 * not count.  Errors: ALOAM_ERR_INVALID_ARG (bad lane or buffer: nothing changes), ALOAM_ERR_STATE on a rank of a sharded job or
 * an emulating context (nothing changes).  Otherwise the call first ends whatever the lane ran and puts the context in lanes
 * mode, as a START does (the lockstep calls are refused until aloam_reset_odometry); then it checks the whole snapshot on the
 * host before it writes anything to the device -- ALOAM_ERR_SNAPSHOT for a bad magic or version, a size that does not match the
 * sections, a cube_growth other than 0 or 1, a count above the cube's ceiling (the slab capacity when the snapshot's cube_growth
 * is 0, the largest run's capacity when it is 1), runs that need more than 1024 slabs of a type (one slab for a count up to the
 * slab capacity, else the next power of two of ceil(count / capacity); with growth off: more than 1024 cubes of a type holding a
 * slab), a payload that is not the sum of
 * the counts, a valid list of more than 125 entries or with an index outside 0 .. 4850, a non-finite warm start or world pose,
 * and for a mapped snapshot a non-finite T_wmap_wodom, a centre offset cen[a] outside -2^20 .. 2^20 (the range of
 * aloam_prior_map_build) or a map position T_wmap_wodom * world (translation) whose centre cube -- int((x + 25.0) / 50.0) + cen[a],
 * minus 1 when x + 25.0 < 0, refused when (x + 25.0) / 50.0 is not finite or lies beyond int -- is more than 16 cubes outside the
 * 21 x 21 x 11 buffer on an axis (below -16 or above 36 in i and j, above 26 in k: the next frame's ring-buffer shift runs one
 * step per cube beyond its edges, so a far or infinite position would never end it; after a mapped frame the centre cube is
 * 3 .. 17 (3 .. 7 in k), so a lane's own snapshot is refused only when the scans it skipped since then moved it more than
 * 950 m), or a configuration that differs --
 * ALOAM_ERR_CAPACITY when a "last" cloud exceeds cfg.max_points, ALOAM_ERR_NOT_RING_MAJOR when it is not ring-major (the check
 * of aloam_odometry_set_last).  It creates the lane's cube store if needed.  After any failure the lane is not running; no other
 * lane changes.  The restored lane takes the cube growth the snapshot records, not the context's (it is not a configuration field
 * that is compared).  Its runs are packed afresh (decreasing size, cube order within a size), so they can be smaller than those
 * of the uninterrupted lane, whose runs never shrink: the restored lane is bit-identical to the uninterrupted run while no run
 * allocation fails on either side.
 * aloam_snapshot_check runs the host checks of aloam_lane_restore on a snapshot in host memory without a context or a GPU (no
 * configuration is compared) and, when info is not NULL, describes it: format version, mode, n_scans, the index of its next scan,
 * its size, its map points and the world pose of its last scan.
 *
 * Snapshot format, version 1: little-endian, sections 16-byte aligned.
 *   1. header, 256 bytes:
 *        0 char magic[8] "ALOAMLS1"   8 int32 version (1)   12 int32 mapped (0 / 1)   16 int64 total_bytes
 *       24 int32 scan_index (the lane's next scan in its trajectory, >= 1)   28 int32 n_less_sharp   32 int32 n_less_flat
 *       configuration: 36 int32 n_scans   40 int32 distortion   44 int32 mapping_skip_frame   48 int32 outer_iters
 *       52 int32 inner_iters   56 float minimum_range   60 float line_res   64 float plane_res   68 int32 slab_cap[2]
 *       76 int32 max_map_points   80 double huber   88 double dist_sq_thresh   96 double nearby_scan
 *      104 double warm[7] (q_last_curr xyzw, t_last_curr: the next scan's warm start)   160 double world[7]
 *      216 int32 ring_source (0 or 1; snapshots written before the field existed hold 0 there, the elevation source)
 *      220 int32 cube_growth (0 or 1: the store's aloam_set_cube_growth setting; snapshots written before the field hold 0)   224 zero to 256
 *   2. at 256: n_less_sharp, then n_less_flat points of 4 floats (x, y, z, intensity) -- the lane's "last" clouds
 *   3. mapped snapshots only, at S = 256 + 16 (n_less_sharp + n_less_flat): the cube store
 *      S+0 int32 cen[3]   S+12 int32 n_valid (<= 125)   S+16 int32 valid[128] (unused entries 0)   S+528 int32 frames
 *      S+532 zero   S+536 double q_wmap_wodom[4]   S+568 double t_wmap_wodom[3]
 *      S+592 int32 count[2][4851]: points of corner (0) / surf (1) cube i; -1 = the cube holds no run (0 = a run, no points)
 *      S+39400 zero   S+39408 int64 n_points (the sum of the counts >= 0)   S+39416 zero
 *      S+39424 n_points points of 4 floats in ALOAM_EXPORT_MAP order: corner cube i, then surf cube i, for i = 0 .. 4850
 *   total_bytes = S, or S + 39424 + 16 n_points for a mapped snapshot.  Which slabs a cube held is not saved: only which cubes hold
 *   a run, and the points, change results.
 *
 * Snapshot format, version 2 -- a LOCALISING lane (aloam_lane_save_localising), which owns no cube store: the trajectory's state
 * is its odometry and its T_wmap_wodom, and it depends on a prior map the snapshot does not hold but names.
 *   1. the header of version 1 with version = 2, mapped = 0 and cube_growth = 0 (magic "ALOAMLS1"; the configuration fields as
 *      version 1 writes them)
 *   2. at 256: the "last" clouds, as version 1
 *   3. at S = 256 + 16 (n_less_sharp + n_less_flat), 128 bytes:
 *      S+0 double q_wmap_wodom[4]   S+32 double t_wmap_wodom[3] (the lane's T_wmap_wodom after its last registered scan and any
 *      recovery it adopted)   S+56 uint64 digest (aloam_prior_map_digest of the map)   S+64 int32 centre[3] (its centre offsets)
 *      S+76 zero   S+80 int64 map_points[2] (its corner / surf points)   S+96 zero to S+128
 *   total_bytes = S + 128.
 * aloam_lane_restore of a version-2 snapshot ends the lane first, as for version 1, then: ALOAM_ERR_STATE without a prior map (and,
 * as for version 1, on a rank of a sharded job or an emulating context); ALOAM_ERR_SNAPSHOT for the version-1 header checks, a size
 * other than S + 128, mapped or cube_growth not 0, a non-finite T_wmap_wodom or a zero quaternion, a centre offset outside
 * -2^20 .. 2^20, a negative point count, a map position T_wmap_wodom * world (translation) whose (x + 25.0) / 50.0 is not finite or
 * lies beyond int (or whose centre cube int((x + 25.0) / 50.0) + centre[a] does), cfg.max_map_points = 0, a configuration that
 * differs -- the odometry fields of version 1 and line_res, plane_res and mapping_skip_frame; the slab capacities and
 * max_map_points do not count --, and a map whose centre offsets, point counts or digest differ from the context's prior map.
 * ALOAM_ERR_CAPACITY / ALOAM_ERR_NOT_RING_MAJOR for the "last" clouds as for version 1; ALOAM_ERR_CUDA when the lane's locator cannot
 * be created (created if needed, as at a localising START).  On success the lane runs a localising trajectory at the saved scan
 * index, its frame state that of a fresh localising START with the saved T_wmap_wodom; a mapped lanes call that continues it with
 * ALOAM_LANE_SCAN gives exactly what the uninterrupted trajectory would have (odometry and map poses, row records and scores,
 * recovery, registered clouds).  The lane's arming is left alone, and aloam_prior_map_load / _build / _clear are refused while it
 * localises, as for any localising lane.  aloam_snapshot_check accepts a well-formed version-2 snapshot (info->version = 2,
 * mapped = 0, map_points = 0); aloam_prior_map_load refuses it with ALOAM_ERR_SNAPSHOT (it holds no store).
 * aloam_lane_save_localising writes the version-2 snapshot of a localising lane under the buffer rules of aloam_lane_save
 * (device, pinned or pageable memory; out = NULL with capacity = 0 for the size; ALOAM_ERR_CAPACITY).  ALOAM_ERR_STATE unless the
 * context runs lanes and `lane` runs a localising trajectory; aloam_lane_save of a localising lane stays ALOAM_ERR_STATE.  The
 * first save (or restore) against a map computes the map's digest (one launch over the map, one synchronisation).
 * aloam_snapshot_localise_info describes a version-2 snapshot in host memory without a context or a GPU, after the checks of
 * aloam_snapshot_check: t_wmap_wodom (q xyzw, t), the digest, centre offsets and point counts of its map (each output may be NULL).
 * ALOAM_ERR_SNAPSHOT for anything but a well-formed version-2 snapshot. */
typedef struct aloam_snapshot_info {
  int version, mapped, n_scans, scan_index;
  long long bytes, map_points;
  double world[7];
} aloam_snapshot_info;
int aloam_lane_save(aloam_ctx* ctx, int lane, void* out, long long capacity, long long* n_bytes);
int aloam_lane_save_localising(aloam_ctx* ctx, int lane, void* out, long long capacity, long long* n_bytes);
int aloam_lane_restore(aloam_ctx* ctx, int lane, const void* blob, long long n_bytes);
int aloam_snapshot_check(const void* host_blob, long long n_bytes, aloam_snapshot_info* info);
int aloam_snapshot_localise_info(const void* host_blob, long long n_bytes, double t_wmap_wodom[7], unsigned long long* digest, int centre[3],
                                 long long map_points[2]);

/* ---- localisation against a prior map: vehicles register their scans against ONE saved map that no frame changes.
 * aloam_prior_map_load makes the cube store of a MAPPED lane snapshot (format v1; blob in device, pinned or pageable memory, as
 * aloam_lane_restore) the prior map of the context.  Only the store section and the configuration are used: the snapshot's odometry
 * part and its T_wmap_wodom are ignored beyond the range checks on them.  The snapshot is checked on the host by the routine
 * aloam_lane_restore runs for a mapped snapshot, with its error codes (ALOAM_ERR_SNAPSHOT also for an unmapped snapshot), and nothing
 * on the device changes on failure.
 * The map is packed per cloud type and indexed once, with one hash grid over the WHOLE map (1.00001 m cells): it is not bounded by
 * cfg.max_map_points (no submap is gathered) but by the snapshot format (1024 slabs of a type, cubes up to the snapshot's ceiling:
 * a growth-on snapshot's cube may hold up to ALOAM_MAX_CUBE_POINTS) and by memory
 * (ALOAM_ERR_CUDA before any state changes): 32 B per point plus a table of 16 B x the power of two above 1.25 x the points of the
 * type.  Loading replaces an earlier prior map.  ALOAM_ERR_STATE while any lane is localising, on a rank of a sharded job and on an
 * emulating context.  aloam_prior_map_clear releases it (ALOAM_ERR_STATE while any lane is localising) and drops every arming;
 * aloam_destroy releases it too.
 * aloam_lane_localise arms `lane` (0 <= lane < cfg.max_batch): its next ALOAM_LANE_START in an aloam_scan_stream_lanes call with
 * map_poses begins a LOCALISING trajectory whose T_wmap_wodom starts at (q_init, t_init) -- the vehicle's pose in the map frame at
 * its first scan, i.e. the origin of its odometry frame -- instead of the identity.  That START consumes the arming;
 * aloam_reset_odometry and aloam_prior_map_clear drop it; a trajectory the lane runs before that START is not disturbed.
 * ALOAM_ERR_STATE without a prior map; ALOAM_ERR_INVALID_ARG for a bad lane, a NULL or non-finite pose or a zero quaternion (a
 * finite one is normalised).  There is no new lane op.
 * So a trajectory is in one of three modes, fixed at its START: odometry only, mapping, localising; one call advances mapping and
 * localising lanes side by side.  A localising frame is the mapper's frame (laserMapping.cpp:309-734) with two parts left out:
 *   - no ring-buffer shift (:323-507): the centre offsets are the prior map's and never change.  The centre cube is computed as at
 *     :312-321 and the 5 x 5 x 3 window of :512-531 is clipped to the buffer by that loop's own bounds test, in its order.  A
 *     vehicle that leaves the map sees a thin or empty window: ALOAM_FLAG_MAP_TOO_THIN, its pose the hand-off pose;
 *   - no insertion and no re-filter (:736-801): the map is never written, so every lane sees the same map whoever ran before.
 * Pose hand-off, the stack filters, the thin-map test on the window's points (corner > 10 and surf > 50), the association, the
 * two solves and transformUpdate are the mapping frame's.  While a mapping frame would neither shift nor exceed
 * cfg.max_map_points, a localising frame returns bit for bit the pose a mapping frame returns from the same store and T_wmap_wodom.
 * cfg.mapping_skip_frame applies as to mapping lanes (scan j registers when j % k == 0, the others get the high-frequency pose
 * from the lane's T_wmap_wodom); the registered sink serves localising rows like mapped rows; aloam_mapper_debug_state_lane answers
 * for a localising lane (centre = the prior map's, valid = the clipped window of its last frame, its T_wmap_wodom, totals = the prior
 * map's); aloam_mapper_export with lane = ALOAM_PRIOR_MAP and ALOAM_EXPORT_MAP exports the prior map (ALOAM_ERR_STATE without one).
 * Per-frame flags, stats and sizes of mapping and localising rows, and a prior-map inlier score of localising rows, come from
 * aloam_map_rows (per-row records, below) while recording is on.
 * A localising lane owns only what a frame writes, created at its first localising START (ALOAM_ERR_CUDA before any state changes):
 * its frame state, 5-NN records and residual blocks for 2 x cfg.max_points queries, the two filtered stacks and the stack filter's
 * sort buffers -- about 450 B per point of cfg.max_points, 0.18 GB at 400 000 and 27 MB at 60 000 (arithmetic from the buffer
 * sizes, not measured), against about 1.75 GB for a mapping lane -- and no cube store if the lane never maps.
 * A localising lane is suspended and resumed with aloam_lane_save_localising / aloam_lane_restore (snapshot format version 2,
 * above): its snapshot names the prior map by centre offsets, point counts and digest, and restores only against that map.
 * Limits, each ALOAM_ERR_STATE: aloam_lane_save of a localising lane (format version 1 has no section for it: use
 * aloam_lane_save_localising); sharded jobs.
 * The lockstep stream calls and aloam_mapper_step never localise.
 *
 * aloam_prior_map_build makes the prior map from two clouds in the MAP frame (the frame of aloam_lane_localise's q_init / t_init):
 * the points a cube store holds, e.g. the reference's laserCloudCornerArray / laserCloudSurfArray, the store clouds of one or more
 * snapshots moved into one frame, or a map built offline.  The clouds are aloam_cloud_views (stride 4 or 8, host memory pageable or
 * pinned, or device memory; the copy kind follows from the address).  centre = the ring buffer's centre offsets
 * (laserCloudCenWidth / Height / Depth), NULL for {10, 10, 5} (a fresh store's); it chooses which 1050 x 1050 x 550 m window of the
 * map frame the 21 x 21 x 11 cubes cover; |centre[a]| <= 2^20, else ALOAM_ERR_INVALID_ARG.
 *   - cube of a point, as the reference's insertion (laserMapping.cpp:741-757): int((x + 25.0) / 50.0) + centre, in double from the
 *     float coordinate, minus 1 when x + 25.0 < 0.  A point whose cube lies outside the buffer is dropped (:751-756), and so is one
 *     with a non-finite coordinate or with a (x + 25.0) / 50.0 beyond the range of int (undefined in the reference).  dropped[t]
 *     (may be NULL) = the points of type t (0 corner, 1 surf) dropped.
 *   - every cube of every type is voxel-filtered on its own (the re-filter of :787-801: cfg.line_res for corner cubes, cfg.plane_res
 *     for surf cubes) over its points in input order, with aloam_voxel_filter's semantics: the box is the cube's points, ties go by
 *     input index, centroids are float sums in sorted order, and a cube whose voxel index range overflows int is kept unfiltered in
 *     input order (PCL).  There is no key-width limit: every other cube is filtered.
 *   - the result is what aloam_prior_map_load makes of a store: per type the filtered cubes packed in cube order, points in voxel
 *     order, the same index, cube tags and ALOAM_EXPORT_MAP export, centre offsets = centre.  Nothing downstream tells the two apart.
 *   - limits: ALOAM_ERR_CAPACITY when a filtered cube holds more than 65536 points while the context's cube growth is off, more than
 *     ALOAM_MAX_CUBE_POINTS while it is on, or a cloud more than 2^30 points (or the two
 *     together more than 2^31 - 4097); nothing changes.  No bound on cubes per type or points per cube otherwise.  Memory: the map as
 *     for a load, plus about 42 B per input point of scratch that is freed before the call returns; ALOAM_ERR_CUDA when it fails.
 *   - state rules are aloam_prior_map_load's: ALOAM_ERR_STATE while any lane is localising, on a rank of a sharded job and on an
 *     emulating context; the new map is built beside the old one, which is replaced only on success; armings survive;
 *     aloam_prior_map_clear and aloam_destroy release it.  Two host synchronisations: one to learn the map's sizes, one at the end. */
/* aloam_prior_map_digest: a 64-bit digest of everything a localising frame reads of the context's prior map, which localising
 * snapshots (format version 2) carry to name their map.  Words w_k, each a 32-bit pattern zero-extended to 64 bits: the three centre
 * offsets; both types' cube-start tables cs[t][0 .. 4851] (cube i of type t holds the packed points cs[t][i] .. cs[t][i + 1] - 1;
 * corner table, then surf table); the corner points, then the surf points, 4 float bit patterns each (x, y, z, intensity), in the
 * packed cube order of the ALOAM_EXPORT_MAP export.  digest = sum over k of mix(k, w_k) mod 2^64, with
 *   mix(k, w) = f(k * 0x9E3779B97F4A7C15 ^ w) mod 2^64,  f(z) = splitmix64's finaliser:
 *   z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;  z = (z ^ (z >> 27)) * 0x94D049BB133111EB;  f = z ^ (z >> 31).
 * Maps loaded or built from the same store agree on it; a changed point bit, cube count or centre offset changes it (up to
 * collisions of a 64-bit sum).  Computed on the device by the first call that needs it (this call, or a localising save or
 * restore: one launch over the map and one synchronisation), then kept with the map; aloam_prior_map_load and _build issue no
 * digest launch.  ALOAM_ERR_STATE without a prior map. */
int aloam_prior_map_digest(aloam_ctx* ctx, unsigned long long* out);
#define ALOAM_PRIOR_MAP (-1)
int aloam_prior_map_load(aloam_ctx* ctx, const void* blob, long long n_bytes);
int aloam_prior_map_build(aloam_ctx* ctx, aloam_cloud_view corner_map, aloam_cloud_view surf_map, const int centre[3], long long dropped[2]);
int aloam_prior_map_clear(aloam_ctx* ctx);
int aloam_lane_localise(aloam_ctx* ctx, int lane, const double q_init[4], const double t_init[3]);

/* ---- extending a saved map in a later session: a MAPPING trajectory that starts on a copy of the prior map.
 * aloam_lane_map_on_prior arms `lane` (0 <= lane < cfg.max_batch): its next ALOAM_LANE_START in an aloam_scan_stream_lanes call with
 * map_poses begins a mapping trajectory (its rows are ALOAM_ROW_MAPPED; there is no new mode) whose cube store is, at that START, a
 * copy of the context's prior map and whose T_wmap_wodom is (q_init, t_init), normalised as aloam_lane_localise normalises it.  From
 * then on the lane is an ordinary mapping lane: it shifts the ring buffer, inserts and re-filters; aloam_lane_save,
 * aloam_mapper_export, the registered sink, aloam_map_rows and cfg.mapping_skip_frame work as for any mapping lane.  The prior map is
 * never written: to publish the extended map, save the lane and aloam_prior_map_load the snapshot, or export it and build from it.
 *   - the seeded store: the centre offsets are the prior map's; every cube the prior map holds points in gets a run of its type,
 *     packed as aloam_lane_restore packs a snapshot's store (with cube growth off one slab each: slabs 0, 1, 2, ... in cube order),
 *     the points in the prior map's per-cube order; cubes without points get no run; frames = 0 and the valid list is empty (the
 *     START frame computes it).  The lane takes the context's cube growth at that START.
 *   - equivalence: every row of the trajectory -- map pose, stats and flags -- and the final store are bit for bit those of
 *     aloam_mapper_step on a lane 0 restored (aloam_lane_restore) from a mapped snapshot that holds the prior map's store with
 *     T_wmap_wodom = the normalised init and frames = 0, driven with the same clouds and odometry poses (the START's odometry pose is
 *     the identity).  One exception: a cube the snapshot counts with 0 points (a slab, no points) has no slab in the seeded store,
 *     since the prior map keeps only counts.  Until a frame inserts into it, aloam_lane_save writes -1 for it where the restored
 *     lane writes 0, and the seeded lane's slab pool holds one more free slab of that type.  While the restored lane's pool is not
 *     exhausted nothing else differs; once it is, a new cube the restored lane must drop (ALOAM_FLAG_CUBE_OVERFLOW) can still take
 *     a slab on the seeded lane, and from that frame on its rows, points and poses may differ.  It is also the reference node
 *     (laserMapping.cpp) started with its cube arrays, centre offsets and q_wmap_wodom / t_wmap_wodom set that way.
 *   - errors, each with nothing armed: ALOAM_ERR_STATE without a prior map, on a rank of a sharded job and on an emulating context;
 *     ALOAM_ERR_INVALID_ARG for a bad lane, a NULL or non-finite pose, a zero quaternion, or an init position t_init whose centre
 *     cube (int((t + 25.0) / 50.0) + the prior map's centre offset, minus 1 below -25) lies more than 16 cubes outside the
 *     21 x 21 x 11 buffer on an axis -- the rule aloam_lane_restore applies to a snapshot's map position (the first frame's shift
 *     loop must end); ALOAM_ERR_CAPACITY when the prior map does not fit a lane's store under the context's cube growth at the time
 *     of the call.  Growth off: a cube with more points than the slab capacity of its type (min(16384, cfg.max_points) corner,
 *     min(65536, cfg.max_points) surf; a built map may hold up to 65536 corner points in a cube), or more than 1024 cubes of one
 *     type that hold points.  Growth on: a cube above its type's ceiling (the largest run's capacity), or runs that need more than
 *     1024 slabs of one type.
 *   - arming: a lane has one arming; aloam_lane_localise and aloam_lane_map_on_prior replace each other (the later call wins).  An
 *     odometry-only START does not consume it; aloam_reset_odometry drops it, and so do aloam_prior_map_load, aloam_prior_map_build
 *     and aloam_prior_map_clear when they succeed and every aloam_set_cube_growth call, since the fit was checked against the map
 *     and the setting of the time (aloam_lane_localise
 *     armings keep their rules).  After its START a seeded lane no longer depends on the prior map: loading, building or clearing a
 *     map between calls does not change it.
 *   - cost: arming allocates nothing and a stream call in which no seeded START runs issues exactly what it issued before.  A step
 *     with seeded STARTs issues 2 more launches on the mapper stream, for all of them together, before its mapping frame
 *     (k_store_seed_tables, k_store_seed_copy).  The lane's store is created as for any mapped START; the first call that seeds a
 *     store also creates cfg.max_batch export layouts of about 155 kB each on the device, kept until aloam_destroy. */
int aloam_lane_map_on_prior(aloam_ctx* ctx, int lane, const double q_init[4], const double t_init[3]);

/* ---- cube growth: map cubes that outgrow one slab, for dense lidars (OS1-64, HDL-64, VLP-32C, a VLP-16 at the default leaves).
 * The reference's cubes grow without bound; each cube of a lane store here holds a RUN of 2^k consecutive slabs of its type from
 * the lane's pool (1024 slabs per type, as before: store memory and re-filter buffers do not change).  With growth off (the
 * default) every run is one slab and the store is what it always was: a cube holds at most min(16384, max_points) corner /
 * min(65536, max_points) surf points and the rest is dropped (ALOAM_FLAG_CUBE_OVERFLOW).
 * aloam_set_cube_growth(ctx, on): on = 1 turns growth on, 0 off; anything else is ALOAM_ERR_INVALID_ARG.  It may be called at any
 * time between calls.  A lane takes the context's setting at each mapped START (a seeded START of aloam_lane_map_on_prior too);
 * lane 0 of the host API and the lockstep stream calls take it at aloam_mapper_reset and when a store is created; a running lane
 * keeps the setting it started with; a restored lane takes its snapshot's (header byte 220).  The call drops every
 * aloam_lane_map_on_prior arming (its fit was checked under the old setting).
 * With growth on:
 *   - runs: a run of 2^k slabs starts at a slab index that is a multiple of 2^k, so a cube's points lie contiguously.  The largest
 *     run is the largest power of two r with r x slab capacity <= ALOAM_MAX_CUBE_POINTS: 16 corner / 4 surf slabs at the default
 *     capacities.  A cube's first point takes one slab; when an insert would pass its run's capacity the cube moves to the smallest
 *     run that holds its new count (at most its ceiling), its points copied in order to the start of the new run, the old run freed
 *     once the insert has served every cube.  Points are appended in stack order: a cube's points are the reference's push_back
 *     order.  Which run a cube holds never changes a result, only whether a later allocation succeeds.  Runs never shrink while
 *     the cube stays in the buffer; a cube that scrolls out of the ring buffer frees its whole run.
 *   - the whole pool: when a type's largest run is all 1024 slabs (slab capacity <= 256 points, max_points <= 256), an insert
 *     grows a cube to at most 512 slabs, 512 x capacity points (131072 at 256): the new run is taken while the old one is still
 *     held, so the whole pool is never free for it.  The points beyond are dropped with ALOAM_FLAG_CUBE_OVERFLOW.  A restore or a
 *     seeded START can still give one cube the whole pool (up to ALOAM_MAX_CUBE_POINTS points).
 *   - allocation is deterministic: the lowest-address aligned free block, cubes served in the order of their first point in the
 *     frame's stack (so when the pool runs out, the new cubes that come first in the stack get runs).
 *   - drops: a point is dropped, with ALOAM_FLAG_CUBE_OVERFLOW, only when its cube already holds its ceiling or when no aligned free
 *     block of the needed size exists; the points dropped are those beyond the cube's current capacity, in stack order.
 *   - re-filter: the per-cube voxel filter of a frame sorts at most max(75 x (corner + surf slab capacity), 2 x max_points) points,
 *     as before.  The valid cubes go in, corner then surf, while their running total fits; the cubes from the first one that does
 *     not fit on stay unfiltered for that frame, and the frame raises ALOAM_FLAG_CUBE_OVERFLOW (error word bit 4).  This is the one
 *     way the store can differ from the reference without a drop.  With growth off every valid cube fits.
 * So with growth on a dense trajectory matches the reference until a cube passes the largest run's capacity (half of it where that
 * run is the whole pool) or the pool fragments.
 * Prior maps: a growth-on snapshot's cubes load (aloam_prior_map_load); aloam_prior_map_build accepts filtered cubes of up to
 * ALOAM_MAX_CUBE_POINTS while growth is on; aloam_lane_map_on_prior checks its fit under the setting at the time of the call. */
int aloam_set_cube_growth(aloam_ctx* ctx, int on);

/* ---- relocalisation: finding the map pose aloam_lane_localise needs, for a vehicle that boots on the map, a lane that lost
 * track or a recording that starts somewhere unknown.  aloam_prior_relocalise scores n_hyp pose hypotheses of ONE scan against
 * the context's prior map on the device and refines the `refine` best of them with a localising frame each.
 *   - inputs: less_sharp / less_flat = the scan's clouds in the sensor frame, as aloam_mapper_step and a localising frame take
 *     them.  hyps (host memory, n_hyp x 7 doubles q xyzw, t; 1 <= n_hyp <= 1 << 24): candidate T_wmap_wodom of a vehicle whose
 *     odometry frame starts at this scan, each checked and normalised as aloam_lane_localise does (a non-finite value or a zero
 *     quaternion: ALOAM_ERR_INVALID_ARG, and nothing runs).
 *   - scoring points: the frame's stack filters (cfg.line_res / cfg.plane_res) over the two clouds; per type, with n_t stack
 *     points and m = min(n_t, max_score_points), scoring point i < m is stack point floor(i * n_t / m) (64-bit integers).
 *   - score of a hypothesis: every scoring point is moved by pointAssociateToMap at the normalised hypothesis (the association's
 *     own float coordinates) and is an inlier when SOME map point of its type anywhere in the prior map (no cube window) lies at
 *     float ((dx*dx + dy*dy) + dz*dz) < inlier_sq.  The 27 grid cells around the point hold every such point (1.00001 m cells,
 *     inlier_sq <= 1).  score = inliers of both types, an integer independent of evaluation order.
 *   - selection: hypotheses ranked by (score descending, index ascending); the first `refine` = K go on.
 *   - refinement: each of the K runs one localising frame from T_wmap_wodom = its hypothesis and the identity odometry pose, all
 *     K in one batched frame.  out[r].pose is bit for bit the map pose of the START row of a lane armed with
 *     aloam_lane_localise(lane, hyps[out[r].hyp]) whose aloam_scan_stream_lanes START scan is this scan.  A thin window
 *     (ALOAM_FLAG_MAP_TOO_THIN in out[r].flags) leaves the pose at the hypothesis.  The refined pose is scored again
 *     (refined_score), and out is sorted by (refined_score descending, coarse rank ascending): out[0] is the answer.  Arm a lane
 *     with out[0].pose and START it on this scan or the next.
 *   - scores (may be NULL): the n_hyp coarse scores in hypothesis order.
 *   - errors, each before anything changes: ALOAM_ERR_STATE without a prior map, on a rank of a sharded job or on an emulating
 *     context; ALOAM_ERR_INVALID_ARG for NULL arguments, a bad cloud view, n_hyp out of range, or options outside
 *     0 < inlier_sq <= 1, max_score_points >= 1, 1 <= refine <= min(ALOAM_MAX_BATCH, n_hyp); ALOAM_ERR_CAPACITY for a cloud of
 *     more than cfg.max_points.  After a frame whose stack filter overflowed its key (as aloam_mapper_step) the outputs are
 *     written and the call returns ALOAM_ERR_CAPACITY.
 *   - synchronous; every lane, the prior map and the stream state are left as they were, so the call may run between any two
 *     stream calls.
 *   - memory, created on first use and kept until aloam_destroy: the K registration sets (a localising lane's, about 450 B per
 *     point of cfg.max_points each, created as calls need them), the two uploaded clouds (32 B per point of cfg.max_points), and
 *     60 B per hypothesis (the normalised hypotheses and their scores), grown to the largest call (arithmetic from the buffer
 *     sizes, not measured). */
typedef struct aloam_reloc_opts {
  float inlier_sq;        /* 0 < inlier_sq <= 1 (m^2) */
  int max_score_points;   /* per type, >= 1: how many stack points score each hypothesis */
  int refine;             /* K: the K best hypotheses are refined, 1 <= K <= min(ALOAM_MAX_BATCH, n_hyp) */
} aloam_reloc_opts;
typedef struct aloam_reloc_result {
  int hyp;                /* index into hyps */
  int score;              /* inliers at the hypothesis */
  int refined_score;      /* inliers at the refined pose */
  int flags;              /* ALOAM_FLAG_MAP_TOO_THIN when the refining frame saw a thin window (pose = the hypothesis) */
  double pose[7];         /* the refined map pose of this scan (q xyzw, t) */
} aloam_reloc_result;
int aloam_prior_relocalise(aloam_ctx* ctx, aloam_cloud_view less_sharp, aloam_cloud_view less_flat, const double* hyps, int n_hyp,
                           const aloam_reloc_opts* opts, int* scores, aloam_reloc_result* out);

/* TransformToEnd of laserOdometry.cpp:133-148 on a whole cloud: undistort every point to the sweep start with its own
 * interpolation ratio, then carry it to the sweep end with (q_last_curr, t_last_curr); the intensity keeps only the scan id.
 * (Dead code in the reference -- its call sites sit under `if (0)`, :533-552 -- provided because the DISTORTION build
 * is where it belongs.)  distortion != 0 uses the per-point ratio, 0 uses s = 1.  out: view into ctx-owned pinned memory. */
int aloam_transform_to_end(aloam_ctx* ctx, aloam_cloud_view in, const double q_last_curr[4], const double t_last_curr[3],
                           int distortion, aloam_cloud_view* out);

/* ---- fine-grained entry points (tests; or to keep Ceres in the loop) */
/* exact k-NN replacing pcl::KdTreeFLANN::nearestKSearch: which = 0 corner_last, 1 surf_last (laserOdometry.cpp:302,390),
 * 2 corner_map, 3 surf_map (laserMapping.cpp:582,648).  idx/sqdist: queries.n x k, ascending (dist, index). */
int aloam_knn(aloam_ctx* ctx, int which, aloam_cloud_view queries, int k, int* idx, float* sqdist);
/* association of laserOdometry.cpp:299-483 at pose (q,t): corner_corr n_sharp x 3 (a,b,valid), plane_corr n_flat x 4 (a,b,c,valid) */
int aloam_odometry_associate(aloam_ctx* ctx, aloam_cloud_view sharp, aloam_cloud_view flat, const double q[4],
                             const double t[3], int* corner_corr, int* plane_corr);
/* residual blocks are 11 doubles [type(0 edge,1 plane,2 plane-norm), cp(3), a(3), b(3), s]; for type 1 b is the unit
 * normal LidarPlaneFactor precomputes (lidarFactor.hpp:64-65), for type 2 a is the unit normal and s = negative_OA_dot_norm.
 * For types 0 and 1 s is the functor's interpolation ratio (1.0 in the reference build; any other value is evaluated with the
 * slerp of lidarFactor.hpp:27-33 and its analytic Jacobian.  The DISTORTION build makes s = frac(intensity) / 0.1, which lies
 * in (-2, 10): a return with relTime < 0 has int(intensity) = ring - 1 and s near 10, one on ring 0 has s < 0).  include/lidarFactor.hpp packs these records (PackBlock).
 * JtJ (6x6 row-major), Jtr (6) in the tangent [dtheta(3), dt(3)] with Huber(0.1) applied, cost = sum 0.5 rho. */
int aloam_normal_equations(aloam_ctx* ctx, const double* blocks, int n_blocks, const double x[7], double JtJ[36],
                           double Jtr[6], double* cost);
/* Ceres-equivalent trust-region solve on the device (replaces ceres::Solve at laserOdometry.cpp:494-499,
 * laserMapping.cpp:712-720).  trace: up to max_trace rows of 8 doubles, may be NULL. */
int aloam_solve(aloam_ctx* ctx, const double* blocks, int n_blocks, double x[7], double summary7[7], double* trace,
                int max_trace, int* trace_rows);
/* last extract_features call: per-point curvature (scanRegistration.cpp:262), label (:303,309,355), ring start/end */
int aloam_debug_features(aloam_ctx* ctx, float* curvature, int* label, int* scan_start, int* scan_end);

/* association + fits of laserMapping.cpp:577-687 at pose x (tests): fits = (n_corner + n_surf) x 14 doubles
 * [query, type (-1 rejected, 0 edge, 2 plane-norm), p0(3), p1(3), d, nn(5)], corner rows first.  A field a row does not reach
 * is NaN: a query without an accepted neighbourhood has only its type, one whose fit fails its type, query and nn. */
int aloam_mapping_associate(aloam_ctx* ctx, aloam_cloud_view corner_stack, aloam_cloud_view surf_stack,
                            const double x[7], double* fits);
/* association + fits against the prior map through the window that lane `lane`'s latest localising frame left (tests):
 * k_map_knn5_prior + k_map_fit at pose x; fits as aloam_mapping_associate, nn(5) = window offset + rank in the cube,
 * i.e. the index in the submap a mapping frame would gather from the same store.  ALOAM_ERR_STATE without a prior map or
 * when the lane has not run a localising frame against the current one. */
int aloam_debug_prior_associate(aloam_ctx* ctx, int lane, aloam_cloud_view corner_stack, aloam_cloud_view surf_stack,
                                const double x[7], double* fits);

/* ---- map cube store + the mapping loop around it (lane 0 of the mapper; the other lanes exist only for
 * aloam_scan_stream_mapped_batch) (laserMapping.cpp:74-108,142-163,309-550,736-801; SURVEY.md 8 f-1).
 * The 21 x 21 x 11 ring buffer of 50 m cubes lives in device memory: a pool of fixed-capacity slabs (1024 per cloud type,
 * 16 k corner / 64 k surf points each, 1.3 GB, created on first use) handed to cubes on their first insertion, one slab per cube
 * with cube growth off, a run of up to ALOAM_MAX_CUBE_POINTS points with growth on (aloam_set_cube_growth).
 * aloam_mapper_step is one frame of alaserMapping's process(), entirely on the device with one synchronisation at the end:
 * pose hand-off from the odometry (transformAssociateToMap), ring-buffer shift, gather of the <= 75 valid cubes (device
 * to device), stack filters at line_res / plane_res, optimisation against the gathered submap (skipped while it is thinner
 * than 10 corner / 50 surf points), transformUpdate, insertion of the registered stacks and per-cube VoxelGrid of the valid
 * cubes.  corner_last / surf_last are the less-sharp / less-flat clouds of the scan (what /laser_cloud_corner_last and
 * /laser_cloud_surf_last carry); the odometry pose is q_wodom_curr / t_wodom_curr; the refined pose is returned.
 * The call never fails half-way: a full cube, an exhausted pool, cubes beyond the re-filter's buffer (growth on) or a submap
 * beyond cfg.max_map_points drop (or leave unfiltered) the
 * overflow and set ALOAM_FLAG_CUBE_OVERFLOW in stats->flags of the frame where it happened (the flags of every frame
 * describe that frame only); argument errors are reported before any state changes.  A cube whose voxel index range does
 * not fit the sort key is kept unfiltered and the frame returns ALOAM_ERR_CAPACITY after completing (pose and store are
 * updated); the next frame starts clean.  cfg.max_map_points must be > 0. */
int aloam_mapper_reset(aloam_ctx* ctx);   /* creates lane 0 if needed; resets every lane that exists */
int aloam_mapper_step(aloam_ctx* ctx, aloam_cloud_view corner_last, aloam_cloud_view surf_last,
                      const double q_wodom_curr[4], const double t_wodom_curr[3], double q_w_curr[4], double t_w_curr[3],
                      aloam_stats* stats);
/* inspection (tests): ring-buffer centre offsets, valid cube indices of the last step (i + 21 j + 441 k), the map-to-
 * odometry transform, total stored points per type; and the points of one cube (which: 0 corner, 1 surf; host view,
 * valid until the next call) */
int aloam_mapper_debug_state(aloam_ctx* ctx, int centre[3], int* n_valid, int valid[125], double q_wmap_wodom[4],
                             double t_wmap_wodom[3], long long totals[2]);
int aloam_mapper_debug_cube(aloam_ctx* ctx, int which, int cube_index, aloam_cloud_view* out);
/* the same for lane `lane` of aloam_scan_stream_mapped_batch (0 <= lane < ALOAM_MAX_BATCH): ALOAM_ERR_STATE while that
 * lane's cube store does not exist.  aloam_mapper_debug_state / _cube are the lane-0 forms. */
int aloam_mapper_debug_state_lane(aloam_ctx* ctx, int lane, int centre[3], int* n_valid, int valid[125], double q_wmap_wodom[4],
                                  double t_wmap_wodom[3], long long totals[2]);
int aloam_mapper_debug_cube_lane(aloam_ctx* ctx, int lane, int which, int cube_index, aloam_cloud_view* out);
/* ---- the clouds the reference mapper publishes (laserMapping.cpp:806-848).
 * aloam_mapper_export copies the cube store of lane `lane` (0: aloam_mapper_step and the single-trajectory calls) out in the
 * reference's order, corner cube then surf cube of every cube:
 *   ALOAM_EXPORT_SURROUND  /laser_cloud_surround (:806-821): the valid cubes of the lane's last frame, in the order of
 *                          aloam_mapper_debug_state's valid list (laserCloudSurroundInd);
 *   ALOAM_EXPORT_MAP       /laser_cloud_map (:823-836): all 4851 cubes, i = 0 .. 4850.
 * out: 4 floats per point, device or host memory (pageable or pinned; the copy kind is inferred from the address).  A host
 * destination is filled through a device staging buffer of at most 4 M points (created on first use, released by aloam_destroy).
 * *n_out is always set to the size of the export; out = NULL with capacity = 0 asks for the size only.  capacity < *n_out
 * returns ALOAM_ERR_CAPACITY and writes nothing.  ALOAM_ERR_INVALID_ARG for a bad `what` or lane, ALOAM_ERR_STATE while the lane's
 * cube store does not exist.  The call reads the store as it is when it is made: after a stream call, the store of that call's
 * last frame.  The reference publishes the surround every 5th and the map every 20th frame (ROS control plane, not modelled):
 * a caller who wants that cadence ends its stream calls at those frames.  On a rank of a sharded job the store is the whole one
 * (it is replicated), so the export is the same on every rank. */
#define ALOAM_EXPORT_SURROUND 0
#define ALOAM_EXPORT_MAP 1
int aloam_mapper_export(aloam_ctx* ctx, int lane, int what, float* out, long long capacity, long long* n_out);
/* /velodyne_cloud_registered (:838-848) of the mapped streams.  While a sink is set, every MAPPED row (scan k, lane l) of
 * aloam_scan_stream_mapped, _mapped_batch and _lanes (with map_poses) -- the rows with j % cfg.mapping_skip_frame == 0 -- writes the
 * scan's ring-major full-resolution cloud (aloam_extract_features' `full`, intensity = ring + 0.1 relTime) moved into the world
 * frame by the row's refined pose exactly as pointAssociateToMap (:154-163: in double, stored as float, intensity kept).  With
 * cfg.distortion = 1 the cloud is not de-skewed first, as in the reference (its TransformToEnd of the full cloud is under if (0)).
 * data: device memory or page-locked host memory (written by the kernel through its device address), `capacity` points of 4
 * floats; pageable memory returns ALOAM_ERR_INVALID_ARG.  data = NULL turns the sink off (the default): the stream calls then
 * issue exactly what they issue without this feature.  The first set call allocates a stash of 4 ring-major clouds per lane
 * (4 x cfg.max_points x 16 B for each of cfg.max_batch lanes), kept until aloam_destroy.
 * Layout: every call writes from offset 0; row r = k * batch + l begins at the sum of raws[r'].n over the call's mapped rows
 * r' < r (a bound known before the call, since the ring-major cloud never holds more points than the raw scan) and holds
 * count = n_full points; the gaps are left untouched.  If that sum over all of the call's mapped rows exceeds `capacity`, the call
 * returns ALOAM_ERR_CAPACITY before any state changes.
 * aloam_registered_rows: begin / count of the `rows` = n_scans x batch rows of the last mapped stream call (skipped and idle rows,
 * and every row of a call made without a sink, have count 0).  ALOAM_ERR_STATE before any mapped stream call, ALOAM_ERR_INVALID_ARG
 * when `rows` is not that call's row count. */
int aloam_set_registered_sink(aloam_ctx* ctx, float* data, long long capacity);
int aloam_registered_rows(aloam_ctx* ctx, long long* begin, int* count, int rows);
/* ---- per-row records of the mapped stream calls: what every scan-to-map row of aloam_scan_stream_mapped, _mapped_batch and _lanes
 * (with map_poses) did -- its flags, stats and sizes, which the stream calls do not return, and for a localising row how many of
 * its scan's points still land on the prior map at the row's map pose.  A lane that drives off the map, locks onto a wrong pose
 * or overflows a cube slab shows in its own rows, so a caller can tell which lane to relocalise (aloam_prior_relocalise) and
 * which row made a call return ALOAM_ERR_CAPACITY.
 * aloam_set_map_rows(ctx, 1, inlier_sq, max_score_points) turns recording on from the next mapped stream call; on = 0 turns it
 * off (the default): the stream calls then issue exactly what they issue without this feature, same launches and copies.  The
 * first call that turns it on allocates a device row table of 4096 rows (kMaxStreamScans) and its pinned host copy, 200 B per
 * row each, kept until aloam_destroy; ALOAM_ERR_CUDA, with nothing changed, when that fails.  ALOAM_ERR_INVALID_ARG for on
 * outside {0, 1}, max_score_points < 0, or max_score_points > 0 with inlier_sq outside (0, 1] (the 27 cells of the 1.00001 m
 * grid hold every point that close, as for aloam_prior_relocalise); max_score_points = 0 records rows without scoring.
 * ALOAM_ERR_STATE on a rank of a sharded job and on an emulating context; aloam_comm_init and aloam_debug_shard_emulate with
 * world > 0 turn recording off.  Cost with recording on: one launch (k_map_rows) per frame, one more (k_inlier_score) per
 * localising frame when scoring, one device-to-host copy of the call's rows.
 * aloam_map_rows copies the `rows` = n_scans x batch rows of the last mapped stream call, scan-major like map_poses (it mirrors
 * aloam_registered_rows).  ALOAM_ERR_INVALID_ARG when out is NULL or `rows` is not that call's row count; ALOAM_ERR_STATE before
 * any mapped stream call, when that call ran with recording off, or when it failed with anything but ALOAM_ERR_CAPACITY or
 * ALOAM_ERR_COMM (after those two the rows are readable: they say which row was hit).
 * Rows:
 *   - ALOAM_ROW_MAPPED / ALOAM_ROW_LOCALISED: `stats` is exactly what aloam_mapper_step returns for that frame, ms_total = 0 -- a
 *     frame on a thin map (ALOAM_FLAG_MAP_TOO_THIN) has zeroed stats and only its flags, any other the stats of its outer_iters
 *     solves with ALOAM_FLAG_FEW_CORRESPONDENCES from the last; ALOAM_FLAG_CUBE_OVERFLOW from the frame's error word.
 *   - ALOAM_ROW_SKIPPED (cfg.mapping_skip_frame): zero stats, score = -1.  ALOAM_ROW_IDLE: kind only, every other field 0.
 *   - score (ALOAM_ROW_LOCALISED rows while max_score_points > 0, thin frames included): aloam_prior_relocalise's score at the row's
 *     map pose.  The scoring points are the frame's own filtered stacks: per type, with n_t stack points and m_t = min(n_t,
 *     max_score_points), scoring point i is stack point floor(i n_t / m_t); each is moved by pointAssociateToMap at the row's map
 *     pose and is an inlier when some prior-map point of its type, anywhere in the map, lies at float ((dx*dx + dy*dy) + dz*dz) <
 *     inlier_sq.  So for a lane armed with hyps[out[r].hyp] of an aloam_prior_relocalise call and STARTed on that call's scan, the
 *     START row's score equals out[r].refined_score when both run with the same inlier_sq and max_score_points.  A lane that keeps
 *     track scores near n_score; one that lost track scores far below it. */
#define ALOAM_ROW_IDLE 0        /* no scan at this step */
#define ALOAM_ROW_MAPPED 1      /* a mapping frame ran for the row */
#define ALOAM_ROW_LOCALISED 2   /* a localising frame against the prior map ran for the row */
#define ALOAM_ROW_SKIPPED 3     /* cfg.mapping_skip_frame: high-frequency pose, no frame */
typedef struct aloam_map_row {
  int kind;          /* ALOAM_ROW_* */
  int err;           /* the frame's error word: bit 0 voxel index range beyond the sort key (why the call returned ALOAM_ERR_CAPACITY),
                        bit 1 a cube at its capacity dropped points, bit 2 no free run of slabs, bit 3 submap truncated, bit 4
                        cubes left out of the re-filter (aloam_set_cube_growth) */
  int n_valid;       /* cubes in the frame's window */
  int n_sub[2];      /* corner / surf map points the frame registered against (the gathered submap, or a localising lane's window) */
  int n_stack[2];    /* the filtered corner / surf stacks */
  int score;         /* ALOAM_ROW_LOCALISED rows with scoring on: inliers at the row's map pose; otherwise -1 */
  int n_score;       /* scoring points behind `score` (m_corner + m_surf); 0 when not scored */
  aloam_stats stats; /* exactly what aloam_mapper_step returns for this frame, ms_total = 0 */
} aloam_map_row;
int aloam_set_map_rows(aloam_ctx* ctx, int on, float inlier_sq, int max_score_points);
int aloam_map_rows(aloam_ctx* ctx, aloam_map_row* out, int rows);
/* ---- recovery of localising lanes inside the mapped stream calls: when a localising row's score (above) falls below a threshold,
 * the same stream scores pose candidates around the row's map pose on the device and, when one is clearly better, re-seats the
 * lane's T_wmap_wodom.  The lane's next registered frame refines from there and its odometry goes on: no host round trip, no
 * relocalise call, no re-arming and no START.
 * aloam_set_recovery(ctx, 1, opts, deltas, n_delta) turns it on from the next mapped stream call; on = 0 turns it off (the default;
 * nothing else is read): the stream calls then issue exactly what they issue without this feature.  Recovery needs scoring rows
 * (aloam_set_map_rows with max_score_points > 0) and uses their inlier_sq and max_score_points; an aloam_set_map_rows call that
 * turns recording or scoring off turns recovery off too.
 *   - scope: ALOAM_ROW_LOCALISED rows (START rows included) of aloam_scan_stream_lanes with map_poses.  Mapping rows, skipped rows
 *     and odometry-only lanes are never touched.
 *   - trigger, per row: n_score > 0 and (float)score < opts->trigger_frac * (float)n_score (a float product).
 *   - candidates: the n_delta relative poses deltas[h] = (q_d, t_d), 7 doubles each, normalised at set time as aloam_lane_localise
 *     normalises.  With P = (q_P, t_P) the row's map pose, candidate h is q_h = normalise(q_d * q_P) (Eigen's product order,
 *     normalised as aloam_lane_localise does, all double) and t_h = t_P + t_d: headings turn about the sensor's position and offsets
 *     are in the map frame, as pose_grid(identity, 0, half, step, yaws) of the Python package lays them out.
 *   - scores: candidate h's score is aloam_prior_relocalise's coarse score of (q_d * q_P, t_P + t_d) for the row's scan, on the same
 *     scoring points as the row's score.  Candidates rank by (score descending, h ascending); `best` is the first.
 *   - adoption: when best_score > score and (float)best_score >= opts->accept_frac * (float)n_score, the lane's T_wmap_wodom becomes
 *     transformUpdate (laserMapping.cpp:148-152) at the best candidate with the row's odometry pose.  The row's map pose, its
 *     aloam_map_row and its registered cloud stay as the frame made them; the lane's next registered frame hands off from the
 *     adopted T, and skipped rows before it (cfg.mapping_skip_frame) compose with it.  The lane's odometry is untouched.
 *   - cost while on: four launches per localising frame, whether or not a row triggers (k_recover_cand, k_reloc_score,
 *     k_reloc_topk, k_recover_adopt), decided on the device without a host synchronisation; an untriggered row's CTAs leave at
 *     once.  A triggered row scores its n_delta candidates at max_score_points points per type.
 *   - buffers, created at set time and kept until aloam_destroy (a larger n_delta grows them): 16 lanes x n_delta candidates (56 B)
 *     and scores (4 B), and per lane the CTA key lists of one resident wave of k_reloc_score.
 *   - errors, each before anything changes: ALOAM_ERR_INVALID_ARG for on outside {0, 1}, n_delta outside 1 ... 65536, a NULL opts
 *     or deltas, a non-finite delta or a zero quaternion, fractions that are not finite or lie outside [0, 1]; ALOAM_ERR_STATE
 *     without scoring rows, on a rank of a sharded job and on an emulating context (aloam_comm_init and aloam_debug_shard_emulate
 *     with world > 0 turn recovery off); ALOAM_ERR_CUDA when the buffers cannot be allocated.
 * aloam_recovery_rows mirrors aloam_map_rows (same row count, scan-major order and state rules, readable after ALOAM_ERR_CAPACITY
 * and ALOAM_ERR_COMM): one aloam_recovery_row per row of the last mapped stream call.  Rows that are not localised, that did not
 * trigger, or of a call made with recovery off have triggered = adopted = 0, best = best_score = -1 and a zero pose.
 * aloam_debug_recovery_scores copies the n = n_delta candidate scores of lane `lane`'s latest triggered row of the last mapped
 * stream call: ALOAM_ERR_STATE when that call triggered no row of the lane (or recovery was set since), ALOAM_ERR_INVALID_ARG for
 * a bad lane, NULL scores or n != n_delta. */
typedef struct aloam_recovery_opts {
  float trigger_frac;  /* 0 <= . <= 1: a localising row triggers when n_score > 0 and (float)score < trigger_frac * (float)n_score */
  float accept_frac;   /* 0 <= . <= 1: the best candidate is adopted when best_score > score and (float)best_score >= accept_frac * (float)n_score */
} aloam_recovery_opts;
int aloam_set_recovery(aloam_ctx* ctx, int on, const aloam_recovery_opts* opts, const double* deltas, int n_delta);
typedef struct aloam_recovery_row {
  int triggered;     /* the row's score met the trigger and its candidates were scored */
  int best;          /* index into deltas of the best candidate, -1 when not triggered */
  int best_score;    /* its score, -1 when not triggered */
  int adopted;       /* the lane's T_wmap_wodom was re-seated after this row */
  double pose[7];    /* the best candidate's map pose (q xyzw, t); zeros when not triggered */
} aloam_recovery_row;
int aloam_recovery_rows(aloam_ctx* ctx, aloam_recovery_row* out, int rows);
int aloam_debug_recovery_scores(aloam_ctx* ctx, int lane, int* scores, int n);
/* ---- place recognition: the Scan Context descriptor (G. Kim and A. Kim, "Scan Context: Egocentric Spatial Descriptor for Place
 * Recognition within 3D Point Cloud Map", IROS 2018), for loop candidates of mapping lanes and for relocalisation without a pose guess.
 * Search is the paper's exact definition: brute force over every keyframe and every column shift (no ring-key tree).
 * Descriptor of a scan: its less_sharp then less_flat clouds in the sensor frame (as aloam_mapper_step takes them).  For every point
 * (float x, y, z), float operations without contraction:
 *   r = sqrtf(x*x + y*y); the point is skipped unless r < max_range;  ring = min(19, (int)((r * 20.0f) / max_range));
 *   a = atan2f(y, x) (glibc's float atan2f), a = a + 6.28318548f when a < 0;  sector = min(59, (int)((a * 60.0f) / 6.28318548f));
 *   v = z + z_offset.  Bin (ring, sector) holds the maximum v of its points in the total order of IEEE bit patterns (-0 < +0, so
 *   the result does not depend on point order); an empty bin holds +0.0f.  Storage is ring-major: bin (r, s) at r * 60 + s.
 * Distance, in double, one IEEE operation at a time (no FMA), sums in ascending index order:
 *   column norm n[c] = sqrt(sum_r d[r][c]^2);  for a shift s visit c = 0 .. 59 with c' = (c + s) mod 60, skip the column when
 *   n_q[c] == 0 or n_d[c'] == 0, else dot = sum_r q[r][c] * d[r][c'], sim += dot / (n_q[c] * n_d[c']), cnt += 1;
 *   dist(s) = cnt ? 1 - sim / cnt : 1.0;  D = min_s dist(s), the smallest s on ties: the match's `shift`.
 *   Heading: q_query ~ q_keyframe * Rz(shift * 2 pi / 60).  Matches rank by (D ascending, keyframe index ascending).
 * Keyframe record, ALOAM_PLACE_RECORD_BYTES, little-endian: 0 double pose[7] (the row's map pose, q xyzw, t)  56 int32 scan_index
 * (the row's scan j in its trajectory)  60 int32 lane  64 float max_range  68 float z_offset  72 zero  80 float desc[1200].
 * Records concatenate: keyframes of several lanes or sessions form one database by appending.
 *
 * aloam_set_place(ctx, on, opts): opts->max_range and opts->z_offset are the descriptor parameters of every call below (80 and 2.0
 * before any call).  on = 1 records keyframes in the mapped stream calls from the next call on, on = 0 stops.  Every call clears
 * every lane's keyframe table.  Errors, with nothing changed: ALOAM_ERR_INVALID_ARG for on outside {0, 1}, a NULL opts, non-finite
 * values, max_range <= 0, keyframe_gap < 0, exclude_recent < 0 or max_keyframes outside 1 .. 65536; ALOAM_ERR_STATE on a rank of a
 * sharded job or an emulating context (aloam_comm_init and aloam_debug_shard_emulate turn recording off); ALOAM_ERR_CUDA when the
 * tables cannot be allocated.
 * Recording: ALOAM_ROW_MAPPED rows of aloam_scan_stream_mapped, _mapped_batch and _lanes (seeded aloam_lane_map_on_prior lanes
 * included); skipped rows, localising rows, odometry-only lanes and aloam_mapper_step record nothing.  A mapped row is a keyframe
 * when its lane's table is empty or when (dx*dx + dy*dy) + dz*dz (double) between the row's map translation and the lane's last
 * keyframe's is >= keyframe_gap^2: its record is appended to the lane's table, then it is queried against the lane's keyframes
 * 0 .. n - 1 - exclude_recent (n: its own index); the best match is the row's loop candidate.  A full table records nothing and
 * sets the row's `full`.  A lane's table is cleared by every mapping START (seeded STARTs included), aloam_reset_odometry and
 * aloam_lane_restore (keyframes are not part of snapshots).  All of it is decided on the device without a host synchronisation:
 * 3 launches per mapping frame (k_place_gate, k_place_dist, k_place_best) and one device-to-host copy of the call's place rows.
 * With recording off the stream calls issue exactly what they issue without this feature.
 * aloam_place_rows mirrors aloam_map_rows: the same row count, scan-major order, state rules, and readability after
 * ALOAM_ERR_CAPACITY / ALOAM_ERR_COMM (ALOAM_ERR_STATE when the last mapped call ran with recording off).  Fields are -1 / -1.0
 * where there is none; `full` is 0 or 1.
 * aloam_place_keyframes exports lane `lane`'s records to device, pinned or pageable memory, with the size rules of
 * aloam_mapper_export counted in records: *n_out is always set; out = NULL with capacity = 0 asks for the size; capacity < *n_out is
 * ALOAM_ERR_CAPACITY and writes nothing.  ALOAM_ERR_INVALID_ARG for a bad lane, ALOAM_ERR_STATE before recording was ever turned on.
 * aloam_place_db_load replaces the context's database with n_records records (host or device memory), checked on the device before
 * anything changes: ALOAM_ERR_INVALID_ARG when a record's max_range / z_offset differ bit for bit from the context's, a pose or
 * descriptor value is not finite, or n_records is outside 1 .. 2^20.  Column norms are computed on load.  aloam_place_db_clear
 * releases it.
 * aloam_place_describe: the descriptor of one scan into desc (host or device memory); ALOAM_ERR_CAPACITY above cfg.max_points.
 * aloam_place_query: n_query descriptors (n_query x 1200 floats, host or device memory) against the database; out = n_query x k
 * matches, the k best per query in rank order.  ALOAM_ERR_STATE without a database; ALOAM_ERR_INVALID_ARG unless
 * 1 <= k <= min(ALOAM_PLACE_MAX_K, M) and n_query >= 1.
 * Memory, arithmetic from the buffer sizes: recording on allocates max_keyframes x (4880 + 480) B for each of cfg.max_batch lanes and
 * a 4096-row place-row table (24 B per row, device and pinned), kept until aloam_destroy (a larger max_keyframes replaces them); the
 * database M x 5360 B; aloam_place_describe two staging clouds of 16 B x cfg.max_points; aloam_place_query the queries (4.8 kB each)
 * and 12 B per (query, keyframe) pair of up to 2^24 pairs at a time. */
#define ALOAM_PLACE_RINGS 20
#define ALOAM_PLACE_SECTORS 60
#define ALOAM_PLACE_MAX_K 64
#define ALOAM_PLACE_RECORD_BYTES 4880
typedef struct aloam_place_opts {
  float max_range;      /* > 0 (m): points at r >= max_range are skipped; default 80 */
  float z_offset;       /* added to z before the maximum; default 2.0 */
  double keyframe_gap;  /* >= 0 (m): the least distance from the lane's last keyframe to a new one */
  int exclude_recent;   /* >= 0: the newest keyframes a loop query leaves out */
  int max_keyframes;    /* 1 .. 65536: the capacity of each lane's table */
} aloam_place_opts;
typedef struct aloam_place_row {
  int keyframe;         /* the row's index in its lane's table, -1 when it is not a keyframe */
  int loop;             /* the best match among the lane's older keyframes, -1 when none */
  int shift;            /* its column shift, -1 when none */
  int full;             /* 1 when the row would have been a keyframe but the table was full */
  double distance;      /* its distance, -1.0 when none */
} aloam_place_row;
typedef struct aloam_place_match {
  int keyframe;         /* index into the database */
  int shift;
  double distance;
} aloam_place_match;
int aloam_set_place(aloam_ctx* ctx, int on, const aloam_place_opts* opts);
int aloam_place_rows(aloam_ctx* ctx, aloam_place_row* out, int rows);
int aloam_place_keyframes(aloam_ctx* ctx, int lane, void* out, long long capacity, long long* n_out);
int aloam_place_db_load(aloam_ctx* ctx, const void* records, int n_records);
int aloam_place_db_clear(aloam_ctx* ctx);
int aloam_place_describe(aloam_ctx* ctx, aloam_cloud_view less_sharp, aloam_cloud_view less_flat, float* desc);
int aloam_place_query(aloam_ctx* ctx, const float* descs, int n_query, int k, aloam_place_match* out);

/* ---- loop verification: the geometric half of loop closure (the registration step SC-A-LOAM runs after Scan Context detection).
 * A place row's loop candidate is a hypothesis; verification registers the query keyframe against a submap made of the candidate's
 * neighbouring keyframes and returns the refined pose, its inlier score and the relative-pose constraint a pose-graph optimiser takes.
 *
 * aloam_set_loops(ctx, on, opts): needs place recording on (aloam_set_place; ALOAM_ERR_STATE otherwise) and clears every lane's
 * keyframe table.  aloam_set_place turns loops off.  While loops are on:
 *   Keyframe clouds: every keyframe a mapping row appends also stores its frame's filtered corner and surf stacks in the sensor
 *   frame (the clouds the frame registered, aloam_map_row.n_stack points each).  Per type, with n stack points and
 *   m = min(n, cloud_points), stored point i is stack point floor(i * n / m) (64-bit integers): the relocaliser's scoring-point
 *   rule.  Clouds are cleared with their table (a mapping START, aloam_reset_odometry, aloam_lane_restore, aloam_set_place,
 *   aloam_set_loops); neither they nor keyframes are part of snapshots.
 *   Verification of (lane, query q, candidate c, shift s), n the lane's keyframe count and e = exclude_recent: it requires q < n
 *   and 0 <= c <= q - 1 - e.
 *     window W = [max(0, c - window), min(c + window, q - 1 - e)]: the keyframes the loop query itself searched, so the current
 *       pass through the place never enters the submap;
 *     submap, per type: the concatenation over k in W (ascending) of keyframe k's stored cloud in stored order, every point moved by
 *       pointAssociateToMap at record k's pose (double, stored as float, intensity kept -- the rule of the registered clouds);
 *     initial pose: q0 = q_c * (0, 0, sz, cz) written as (x cz + y sz, y cz - x sz, z cz + w sz, w cz - z sz) with
 *       (sz, cz) = (sin, cos)(a / 2), a = ((s * 2.0) * pi) / 60 (the C library's sin / cos on the host), then normalised as
 *       aloam_lane_localise normalises (|q|^2 summed in index order, q / sqrt); t0 = t_c.  aloam_loop_verify takes `init` instead
 *       when it is not NULL (normalised the same way; `shift` is ignored and the row's shift is -1);
 *     registration: with <= 10 corner or <= 50 surf submap points no round runs, the pose stays the initial pose and the row is
 *       flagged ALOAM_FLAG_MAP_TOO_THIN.  Otherwise outer_iters rounds of the mapper's association and solve run with the query
 *       keyframe's stored clouds as the stacks.  The result is, bit for bit, what a context of the same configuration with
 *       outer_iters = 1 computes with one aloam_map_upload of the submap and outer_iters successive aloam_mapping_register calls
 *       from the initial pose: the pose and the last call's stats (ms_total = 0);
 *     score: the relocaliser's inlier rule -- a stored point of the query keyframe moved by `pose` is an inlier when a submap point
 *       of its type lies at float ((dx*dx + dy*dy) + dz*dz) < inlier_sq.  An integer count; there is no accept threshold, the caller
 *       judges score / n_score;
 *     constraint: rel = T_c^-1 * pose in Eigen's operation order, (q_c.conjugate() * q, q_c.conjugate() * (t - t_c)).
 *   In the stream: every ALOAM_ROW_MAPPED keyframe row of aloam_scan_stream_mapped, _mapped_batch and _lanes whose place row has
 *   loop >= 0 and distance <= max_distance (double compare) is verified at its own step on the mapper stream with (its lane, its
 *   keyframe, its loop, its shift), without a host synchronisation.  Launches per mapping frame: 1 (k_loop_keep); when some record
 *   can have a candidate (the bound place recognition uses to size its query), 8 + 3 outer_iters more (k_loop_gather, k_grid_setup,
 *   the 4 index-build launches, outer_iters x (k_map_knn5, k_map_fit, k_lm_solve), k_inlier_score, k_loop_finish); one device-to-host
 *   copy of the loop rows per call.  With loops off the stream calls issue exactly what they issue without this feature.
 * aloam_loop_rows mirrors aloam_place_rows: the same row count, scan-major order, state rules, and readability after
 * ALOAM_ERR_CAPACITY / ALOAM_ERR_COMM (ALOAM_ERR_STATE when the last mapped call ran with loops off).  Fields are -1 / 0 where a row
 * was not verified.
 * aloam_loop_verify runs one verification on the context's stream and synchronises once; ALOAM_ERR_STATE while loops are off.
 * aloam_place_keyframe_cloud exports keyframe `keyframe` of lane `lane`: corner points then surf points, 4 floats each, to device,
 * pinned or pageable memory with the size rules of aloam_place_keyframes counted in points (n_out[0], n_out[1] always set).
 * ALOAM_ERR_INVALID_ARG for a bad lane or a keyframe outside the lane's table, ALOAM_ERR_STATE while loops are off.
 * Errors, each leaving nothing changed: ALOAM_ERR_INVALID_ARG for on outside {0, 1}, a NULL or out-of-range option, a bad lane,
 * query, cand or shift (0 .. 59), a non-finite init or a zero quaternion; ALOAM_ERR_CAPACITY when (2 window + 1) x cloud_points >
 * cfg.max_map_points (the submap bound, so no frame truncates a submap); ALOAM_ERR_STATE on a rank of a sharded job or an emulating
 * context (aloam_comm_init and aloam_debug_shard_emulate turn loops off), for aloam_loop_verify while loops are off and for
 * aloam_loop_rows after a call made with loops off; ALOAM_ERR_CUDA when the buffers cannot be allocated.
 * Memory, per lane of cfg.max_batch lanes, with K = the place table's max_keyframes, P = cloud_points, B = (2 window + 1) P and
 * S = the power of two >= 1.25 B (at least 1024): the cloud pool K x 2 x P x 16 B + K x 8 B; the registration set 2 x (S x 16 B +
 * B x 16 B) grids, 2P x 80 B neighbours, 2P x 96 B residual blocks, 2P x 16 B query stacks and 4 solve summaries; the two submap
 * buffers 2 x B x 16 B; plus a 4096-row loop-row table (device and pinned). */
typedef struct aloam_loop_opts {
  double max_distance;  /* >= 0: a keyframe row whose place-row distance is <= this (double compare) is verified */
  int window;           /* 0 .. 64: keyframes on each side of the candidate that form its submap */
  int cloud_points;     /* 1 .. cfg.max_points: per type, the most points a keyframe keeps of its frame's filtered stack */
  int outer_iters;      /* 1 .. 16: association + solve rounds of a verification */
  float inlier_sq;      /* 0 < . <= 1 (m^2): the relocaliser's inlier rule, for the score */
} aloam_loop_opts;
typedef struct aloam_loop_row {
  int query, cand;      /* the row's keyframe and its candidate; -1 when the row was not verified */
  int verified;         /* 1 when verification ran */
  int shift;            /* the place row's shift used for the initial heading; -1 when not verified */
  int n_sub[2];         /* corner / surf points of the candidate submap */
  int score, n_score;   /* inliers of the query keyframe's stored points at `pose`, out of n_score (its stored corner + surf) */
  aloam_stats stats;    /* the last round's stats as aloam_mapping_register returns them, ms_total = 0; MAP_TOO_THIN for a thin submap */
  double pose[7];       /* the query keyframe's refined pose in the map frame of the candidate's submap (q xyzw, t) */
  double rel[7];        /* the constraint: that pose in the candidate keyframe's frame, T_cand^-1 * pose */
} aloam_loop_row;
int aloam_set_loops(aloam_ctx* ctx, int on, const aloam_loop_opts* opts);
int aloam_loop_rows(aloam_ctx* ctx, aloam_loop_row* out, int rows);
int aloam_loop_verify(aloam_ctx* ctx, int lane, int query, int cand, int shift, const double init[7], aloam_loop_row* out);
int aloam_place_keyframe_cloud(aloam_ctx* ctx, int lane, int keyframe, float* out, long long capacity, long long n_out[2]);

/* the segmented VoxelGrid of the mapper (tests): n_segs clouds, each with its own cubic leaf, filtered by one pass with
 * idx_bits voxel-index bits in the 32-bit sort key (the segments go in windows of 2^(32 - idx_bits) when they do not fit
 * beside the index), exactly as the per-cube re-filter runs.  out: room for the sum of segs[s].n points; segment s is
 * written at its input offset (the sum of the sizes before it), out_counts[s] points.  err: bit 0 = a segment's index range
 * needed more than idx_bits bits (that segment is returned unchanged).  n_segs > 160 or more points than the mapper's sort
 * buffers hold: ALOAM_ERR_CAPACITY.  Creates the cube store if needed; never changes its state. */
int aloam_debug_seg_voxel_filter(aloam_ctx* ctx, const aloam_cloud_view* segs, const float* leaves, int n_segs, int idx_bits,
                                 float* out, int* out_counts, int* err);

/* ---- multi-GPU scan-to-map (one process per GPU).  Rank 0 creates the 128-byte id and ships it to the others;
 * after aloam_comm_init each rank uploads only ITS shard of the submap (x-slabs of aloam_shard_slab_cells() cells of
 * 1.00001 m, owner = slab mod world, plus one cell of halo) and aloam_mapping_register fits only the stack points
 * whose cell the rank owns; the ranks meet in one ncclAllReduce of the 6x6 / 6x1 normal equations per evaluation and
 * return the identical pose.  On the peer-memory exchange a peer that does not answer within about 2 s makes
 * aloam_mapping_register, aloam_mapper_step and aloam_scan_stream_mapped return ALOAM_ERR_COMM (after writing the pose). */
int aloam_comm_unique_id(char out128[128]);
int aloam_comm_init(aloam_ctx* ctx, int rank, int world, const char id128[128]);
int aloam_shard_slab_cells(void);
/* as aloam_map_upload, for a rank that holds the WHOLE submap (host or device memory): the rank's shard -- its x-slabs plus the
 * one-cell halo -- is cut out on the device (stable compaction), then indexed.  cfg.max_map_points must hold the shard: a larger
 * shard returns ALOAM_ERR_CAPACITY and leaves the context without a map (aloam_mapping_register returns ALOAM_ERR_STATE). */
int aloam_map_upload_sharded(aloam_ctx* ctx, aloam_cloud_view corner_map, aloam_cloud_view surf_map);
/* 1 when the ranks exchange the normal equations through NVLink peer memory INSIDE the LM kernel (one launch per solve; CUDA IPC
 * mailboxes set up by aloam_comm_init), 0 when they use ncclAllReduce between per-evaluation kernels (no peer access, or the
 * environment variable ALOAM_NO_PEER is set -- kept for A/B measurements). */
int aloam_comm_uses_peer_memory(aloam_ctx* ctx);
/* Test hook: one context behaves as rank `rank` of `world` without a communicator, so the sharded path can be checked on one
 * GPU.  aloam_map_upload_sharded cuts this rank's shard, the index build counts its owned points, the 5-NN rejects queries in
 * cells it does not own, and aloam_mapping_register / aloam_mapper_step / aloam_scan_stream_mapped run the sharded frame.  The
 * all-reduces become loopbacks: the global map size is this rank's owned count, and the LM exchange is `exchange`:
 *   0  k_lm_solve on this rank's blocks (the single-GPU solve);
 *   1  per evaluation k_lm_eval_shard, a device copy of the 32 sums in place of ncclAllReduce, k_lm_tr_shard;
 *   2  k_lm_solve_x with a one-rank peer mailbox (aloam_comm_uses_peer_memory returns 1).
 * With exchange 1 or 2, aloam_solve also goes through that exchange.  world = 0 ends the emulation; a change of rank or world
 * drops the uploaded map.  poison_peer_err = 1 (exchange 2) makes the next call start with the mailbox's error word set, as
 * after a peer timeout.  What stays unchecked on one GPU: the NVLink / IPC transport, the tag order across ranks and
 * ncclAllReduce itself.  ALOAM_ERR_STATE on a context with a communicator (and aloam_comm_init on an emulating context), and
 * aloam_scan_stream_mapped_batch / aloam_scan_stream_lanes return it while emulating. */
int aloam_debug_shard_emulate(aloam_ctx* ctx, int rank, int world, int exchange, int poison_peer_err);
/* points indexed by the last aloam_map_upload(_sharded) (kept: this rank's shard) and the submap size the thin-map test of
 * aloam_mapping_register sees (global: summed over the ranks); ALOAM_ERR_STATE without a map */
int aloam_debug_map_sizes(aloam_ctx* ctx, int kept[2], int global[2]);

/* ---- measurement hooks (bench.py): per-kernel CUDA-event timing on the ctx stream, and a launch counter */
int aloam_profile_enable(aloam_ctx* ctx, int on);
int aloam_profile_read(aloam_ctx* ctx, double* ms_sum, long long* count, const char** names, int capacity);
long long aloam_launch_count(aloam_ctx* ctx);
int aloam_debug_lm_cycles(aloam_ctx* ctx, long long* out, int outer_iters); /* SM cycles: [solve, evaluation passes] per outer iteration */

#ifdef __cplusplus
}
#endif
#endif /* ALOAM_B200_H_ */
