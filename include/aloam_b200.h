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
#define ALOAM_ERR_UNSUPPORTED_SCANS (-2) /* scanRegistration.cpp:472-476: only 16, 32 or 64 scan lines */
#define ALOAM_ERR_EMPTY_CLOUD (-3)       /* no point survives the NaN / minimum-range filter */
#define ALOAM_ERR_CAPACITY (-4)          /* more points than the ctx was created for */
#define ALOAM_ERR_CUDA (-5)
#define ALOAM_ERR_NO_DEVICE (-6)
#define ALOAM_ERR_RING_TOO_LARGE (-7)    /* a single ring holds more than ALOAM_MAX_RING_POINTS returns */
#define ALOAM_ERR_NOT_RING_MAJOR (-8)    /* "last" cloud with an int(intensity) outside 0..63 or two or more below an earlier
                                            point's: every scanRegistration output has int_i >= max_{j<i} int_j - 1, and the
                                            association's break tables rely on it (laserOdometry.cpp:310-361,400-455) */
#define ALOAM_ERR_STATE (-9)             /* call sequence error, e.g. register before set_last */
#define ALOAM_ERR_COMM (-10)
#define ALOAM_ERR_SNAPSHOT (-11)         /* snapshot malformed, of another format version, or taken under a configuration that
                                            changes results (aloam_lane_restore, aloam_snapshot_check) */

#define ALOAM_MAX_RING_POINTS 4096
#define ALOAM_MAX_BATCH 16

#define ALOAM_FLAG_FEW_CORRESPONDENCES 1
#define ALOAM_FLAG_MAP_TOO_THIN 2
#define ALOAM_FLAG_INITIALISED_ONLY 4 /* first frame: laserOdometry.cpp:267-271 */
#define ALOAM_FLAG_CUBE_OVERFLOW 8    /* map cube store: a cube slab (16 k corner / 64 k surf points) or the slab pool was full; the overflow was dropped */

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
  int max_points;        /* capacity of one raw scan (reference: 400000 static arrays, scanRegistration.cpp:66-69) */
  int max_map_points;    /* capacity of the uploaded submap, per cloud type (0 = mapping not used); at most 2^30, larger
                            values are rejected by aloam_create with ALOAM_ERR_INVALID_ARG */
  int max_batch;         /* trajectories a context can advance in lockstep (aloam_scan_stream_batch), or lanes of
                            aloam_scan_stream_lanes; 1..ALOAM_MAX_BATCH, default 1 */
  int distortion;        /* 0 (reference build) or 1: #define DISTORTION of laserOdometry.cpp:59 -- per-point interpolation ratio
                            s = (intensity - int(intensity)) / SCAN_PERIOD in TransformToStart (:113-118) and in the
                            residual blocks (:376-379, 470-473; slerp inside the functors, lidarFactor.hpp:27-33) */
  int max_ring_points;   /* capacity of one scan ring, multiple of 32, <= ALOAM_MAX_RING_POINTS (default).  Smaller rings take
                            less shared memory per ring CTA, so more of them are resident per SM (batched streams) */
  int mapping_skip_frame; /* mapping_skip_frame laserOdometry.cpp:191, launch/...:6 -- the mapped stream calls map every k-th scan
                            of a trajectory and give the others the high-frequency pose (see aloam_scan_stream_mapped).  Default 1
                            (every scan); 0 counts as 1 (zero-initialised tail of an older caller); < 0 is rejected by aloam_create */
} aloam_config;

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
 * minimum_range, outer_iters, inner_iters, huber, dist_sq_thresh, nearby_scan and distortion, and for a mapped snapshot also
 * line_res, plane_res, mapping_skip_frame, max_map_points and the slab capacities min(16384, max_points) / min(65536, max_points)
 * (floating-point fields compared bit for bit).  max_points beyond the slab capacities, max_batch, max_ring_points and device do
 * not count.  Errors: ALOAM_ERR_INVALID_ARG (bad lane or buffer: nothing changes), ALOAM_ERR_STATE on a rank of a sharded job or
 * an emulating context (nothing changes).  Otherwise the call first ends whatever the lane ran and puts the context in lanes
 * mode, as a START does (the lockstep calls are refused until aloam_reset_odometry); then it checks the whole snapshot on the
 * host before it writes anything to the device -- ALOAM_ERR_SNAPSHOT for a bad magic or version, a size that does not match the
 * sections, a count above the slab capacity, more than 1024 cubes of a type holding a slab, a payload that is not the sum of
 * the counts, a valid list of more than 125 entries or with an index outside 0 .. 4850, or a configuration that differs --
 * ALOAM_ERR_CAPACITY when a "last" cloud exceeds cfg.max_points, ALOAM_ERR_NOT_RING_MAJOR when it is not ring-major (the check
 * of aloam_odometry_set_last).  It creates the lane's cube store if needed.  After any failure the lane is not running; no other
 * lane changes.
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
 *      104 double warm[7] (q_last_curr xyzw, t_last_curr: the next scan's warm start)   160 double world[7]   216 zero to 256
 *   2. at 256: n_less_sharp, then n_less_flat points of 4 floats (x, y, z, intensity) -- the lane's "last" clouds
 *   3. mapped snapshots only, at S = 256 + 16 (n_less_sharp + n_less_flat): the cube store
 *      S+0 int32 cen[3]   S+12 int32 n_valid (<= 125)   S+16 int32 valid[128] (unused entries 0)   S+528 int32 frames
 *      S+532 zero   S+536 double q_wmap_wodom[4]   S+568 double t_wmap_wodom[3]
 *      S+592 int32 count[2][4851]: points of corner (0) / surf (1) cube i; -1 = the cube holds no slab (0 = a slab, no points)
 *      S+39400 zero   S+39408 int64 n_points (the sum of the counts >= 0)   S+39416 zero
 *      S+39424 n_points points of 4 floats in ALOAM_EXPORT_MAP order: corner cube i, then surf cube i, for i = 0 .. 4850
 *   total_bytes = S, or S + 39424 + 16 n_points for a mapped snapshot.  Which slab a cube held is not saved: only which cubes hold
 *   one, and the points, change results. */
typedef struct aloam_snapshot_info {
  int version, mapped, n_scans, scan_index;
  long long bytes, map_points;
  double world[7];
} aloam_snapshot_info;
int aloam_lane_save(aloam_ctx* ctx, int lane, void* out, long long capacity, long long* n_bytes);
int aloam_lane_restore(aloam_ctx* ctx, int lane, const void* blob, long long n_bytes);
int aloam_snapshot_check(const void* host_blob, long long n_bytes, aloam_snapshot_info* info);

/* ---- localisation against a prior map: vehicles register their scans against ONE saved map that no frame changes.
 * aloam_prior_map_load makes the cube store of a MAPPED lane snapshot (format v1; blob in device, pinned or pageable memory, as
 * aloam_lane_restore) the prior map of the context.  Only the store section and the configuration are used: the snapshot's odometry
 * part and its T_wmap_wodom are ignored.  The snapshot is checked on the host by the routine aloam_lane_restore runs for a mapped
 * snapshot, with its error codes (ALOAM_ERR_SNAPSHOT also for an unmapped snapshot), and nothing on the device changes on failure.
 * The map is packed per cloud type and indexed once, with one hash grid over the WHOLE map (1.00001 m cells): it is not bounded by
 * cfg.max_map_points (no submap is gathered) but by the snapshot format (1024 cubes of a type x the slab capacity) and by memory
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
 * Per-frame flags are not returned by the stream calls (as for mapping lanes).
 * A localising lane owns only what a frame writes, created at its first localising START (ALOAM_ERR_CUDA before any state changes):
 * its frame state, 5-NN records and residual blocks for 2 x cfg.max_points queries, the two filtered stacks and the stack filter's
 * sort buffers -- about 450 B per point of cfg.max_points, 0.18 GB at 400 000 and 27 MB at 60 000 (arithmetic from the buffer
 * sizes, not measured), against about 1.75 GB for a mapping lane -- and no cube store if the lane never maps.
 * Limits, each ALOAM_ERR_STATE: aloam_lane_save of a localising lane (snapshot format v1 has no section for it); sharded jobs.
 * The lockstep stream calls and aloam_mapper_step never localise. */
#define ALOAM_PRIOR_MAP (-1)
int aloam_prior_map_load(aloam_ctx* ctx, const void* blob, long long n_bytes);
int aloam_prior_map_clear(aloam_ctx* ctx);
int aloam_lane_localise(aloam_ctx* ctx, int lane, const double q_init[4], const double t_init[3]);

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
 * 16 k corner / 64 k surf points each, 1.3 GB, created on first use) handed to cubes on their first insertion.
 * aloam_mapper_step is one frame of alaserMapping's process(), entirely on the device with one synchronisation at the end:
 * pose hand-off from the odometry (transformAssociateToMap), ring-buffer shift, gather of the <= 75 valid cubes (device
 * to device), stack filters at line_res / plane_res, optimisation against the gathered submap (skipped while it is thinner
 * than 10 corner / 50 surf points), transformUpdate, insertion of the registered stacks and per-cube VoxelGrid of the valid
 * cubes.  corner_last / surf_last are the less-sharp / less-flat clouds of the scan (what /laser_cloud_corner_last and
 * /laser_cloud_surf_last carry); the odometry pose is q_wodom_curr / t_wodom_curr; the refined pose is returned.
 * The call never fails half-way: a full cube slab, an exhausted pool or a submap beyond cfg.max_map_points drop the
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
