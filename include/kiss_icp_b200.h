/* kiss_icp_b200.h — C-ABI of the CUDA (H100, sm_90a) KISS-ICP registration hot path.
 *
 * This is the drop-in boundary: one entry point per function the reference's language
 * bindings reach on this path (python/kiss_icp/pybind/kiss_icp_pybind.cpp:48-144 and the C++
 * surface used by ros/src/OdometryServer.cpp:80,162,165,222). Each declaration cites the
 * reference interface it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - plain pointers + sizes, no C++/torch types; every call returns a kb_status (0 = ok) and
 *     never throws or aborts across the ABI; kb_last_error() gives a thread-local message.
 *   - point clouds are dense double[n][3] (== std::vector<Eigen::Vector3d>::data(), 24 B stride)
 *   - rigid transforms are 4x4 ROW-MAJOR double[16] (numpy layout). Eigen/Sophus callers pass
 *     T.matrix().transpose().data() or copy (Eigen default is column-major).
 *   - a matrix that is not in SE(3) returns KB_ERR_NOT_SE3 where Sophus would SOPHUS_ENSURE
 *     (abort) in the reference (kiss_icp_pybind.cpp:68,84,99,117).
 *   - "host" entry points take HOST buffers and do the H2D/D2H copies themselves;
 *     "_dev" entry points take DEVICE pointers resident in HBM on the handle's device.
 *   - handles are not thread-safe (same as the reference objects); distinct handles may be
 *     used from distinct threads / on distinct GPUs concurrently.
 *   - there is NO CPU fallback: every compute entry point fails with KB_ERR_NO_DEVICE when no
 *     CUDA device is present.
 */
#ifndef KISS_ICP_B200_H
#define KISS_ICP_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum kb_status {
    KB_OK = 0,
    KB_ERR_INVALID_ARG = 1,
    KB_ERR_NOT_SE3 = 2,      /* Sophus SE3d(Matrix4d) would have ENSURE-failed */
    KB_ERR_OUT_OF_RANGE = 3, /* timestamps.at(idx) would have thrown (core/Preprocessing.cpp:76-77) */
    KB_ERR_CUDA = 4,
    KB_ERR_CAPACITY = 5, /* caller buffer too small; *n_out holds the required count */
    KB_ERR_NO_DEVICE = 6
} kb_status;

typedef struct kb_map kb_map;                   /* kiss_icp::VoxelHashMap            */
typedef struct kb_registration kb_registration; /* kiss_icp::Registration            */
typedef struct kb_preprocessor kb_preprocessor; /* kiss_icp::Preprocessor            */
typedef struct kb_threshold kb_threshold;       /* kiss_icp::AdaptiveThreshold       */
typedef struct kb_pipeline kb_pipeline;         /* kiss_icp::pipeline::KissICP       */

/* ---- library -------------------------------------------------------------------------- */
const char *kb_last_error(void);
const char *kb_version(void);
/* number of visible CUDA devices (0 when none: every compute call then returns KB_ERR_NO_DEVICE) */
int kb_device_count(void);
/* device used by handles created afterwards on the calling thread (default 0) */
int kb_set_device(int device);
/* run the handle-less calls (kb_voxel_down_sample, kb_preprocess ...) and handles created
 * afterwards on this CUDA stream (a cudaStream_t; NULL = the library's own stream) */
int kb_set_stream(void *cuda_stream);
/* persistent-grid size (thread blocks) used by the cooperative kernels; 0 = one per SM */
int kb_set_grid_blocks(int blocks);

/* ---- kiss_icp::VoxelHashMap (cpp/kiss_icp/core/VoxelHashMap.hpp:38-57) ------------------ */
/* VoxelHashMap(double voxel_size, double max_distance, unsigned max_points_per_voxel); pybind
 * `_VoxelHashMap(voxel_size, max_distance, max_points_per_voxel)` kiss_icp_pybind.cpp:54-57 */
int kb_map_create(double voxel_size, double max_distance, unsigned max_points_per_voxel, kb_map **out);
int kb_map_destroy(kb_map *map);
/* Clear() VoxelHashMap.hpp:44 / `_clear` */
int kb_map_clear(kb_map *map);
/* Empty() VoxelHashMap.hpp:45 / `_empty` */
int kb_map_empty(const kb_map *map, int *out_is_empty);
/* Update(points, origin) VoxelHashMap.cpp:83-87 / `_update(points, origin)` */
int kb_map_update_origin(kb_map *map, const double *xyz, size_t n, const double origin[3]);
/* Update(points, pose) VoxelHashMap.cpp:89-95 / `_update(points, pose)` */
int kb_map_update_pose(kb_map *map, const double *xyz, size_t n, const double pose[16]);
/* AddPoints VoxelHashMap.cpp:97-119 / `_add_points` */
int kb_map_add_points(kb_map *map, const double *xyz, size_t n);
/* RemovePointsFarFromLocation VoxelHashMap.cpp:121-132 / `_remove_far_away_points` */
int kb_map_remove_far(kb_map *map, const double origin[3]);
/* Pointcloud() VoxelHashMap.cpp:72-81 / `_point_cloud`. Two-call: pass capacity 0 to query
 * *n_out. Per-voxel point order is the reference's (insertion order); the order of VOXELS is
 * ascending (x,y,z) instead of the reference's hash-table iteration order (documented in
 * DESIGN.md: that order is an artefact of robin_map history and feeds nothing on this path). */
int kb_map_pointcloud(const kb_map *map, double *out_xyz, size_t capacity, size_t *n_out);
int kb_map_num_points(const kb_map *map, size_t *out);
int kb_map_num_voxels(const kb_map *map, size_t *out);
/* per-voxel dump (checkpoint / parity tests): voxels int[nv][3] ascending, counts int[nv],
 * points double[np][3] concatenated in per-voxel insertion order */
int kb_map_dump(const kb_map *map, int *voxels, int *counts, double *points, size_t voxel_capacity,
                size_t point_capacity, size_t *n_voxels, size_t *n_points);
/* GetClosestNeighbor VoxelHashMap.cpp:46-70, batched over n queries (the reference calls it
 * from a TBB parallel_for, Registration.cpp:66-76). out_points double[n][3], out_dist
 * double[n]; a miss returns (0,0,0), DBL_MAX like VoxelHashMap.cpp:51-52. */
int kb_map_closest_neighbors(const kb_map *map, const double *queries, size_t n, double *out_points,
                             double *out_dist);
int kb_map_closest_neighbors_dev(const kb_map *map, const double *d_queries, size_t n, double *d_out_points,
                                 double *d_out_dist);
/* rebuild the table at load factor <= 0.5 without tombstones (smallest power-of-two capacity): shrinks the
 * address range the point blocks are scattered over — for query-heavy phases on a static map */
int kb_map_compact(kb_map *map);
/* public data members voxel_size_, max_distance_, max_points_per_voxel_ VoxelHashMap.hpp:53-55 */
int kb_map_params(const kb_map *map, double *voxel_size, double *max_distance, unsigned *max_points_per_voxel);
/* ALGORITHMIC bytes of kb_map_closest_neighbors_dev for these n queries on this map: sum over
 * queries of 24 + 27*16 + 24*candidates + 32 (SURVEY.md 8d), candidates counted on the device
 * by an instrumented (untimed) pass. */
int kb_map_query_bytes_dev(const kb_map *map, const double *d_queries, size_t n, double *bytes);
/* kb_map_closest_neighbors_dev is asynchronous on the map's stream; this waits for it */
int kb_map_sync(const kb_map *map);

/* ---- kiss_icp::Registration (cpp/kiss_icp/core/Registration.hpp:33-45) ------------------ */
/* Registration(int max_num_iteration, double convergence_criterion, int max_num_threads);
 * max_num_threads is accepted and ignored (it sizes the TBB pool in the reference). */
int kb_registration_create(int max_num_iterations, double convergence_criterion, int max_num_threads,
                           kb_registration **out);
int kb_registration_destroy(kb_registration *reg);
/* AlignPointsToMap(frame, voxel_map, initial_guess, max_correspondence_distance, kernel_scale)
 * Registration.cpp:138-167 / `_align_points_to_map` kiss_icp_pybind.cpp:94-106 */
int kb_registration_align_points_to_map(kb_registration *reg, const double *xyz, size_t n, const kb_map *map,
                                        const double initial_guess[16], double max_correspondence_distance,
                                        double kernel_scale, double out_pose[16]);
/* number of ICP iterations the last call ran (diagnostic; no reference counterpart) */
int kb_registration_last_iterations(const kb_registration *reg, int *out);
/* one DataAssociation + BuildLinearSystem pass (Registration.cpp:60-121) on points already in
 * the map frame: JTJ double[36] row-major (full symmetric), JTr double[6], correspondences */
int kb_registration_build_system(kb_registration *reg, const double *xyz, size_t n, const kb_map *map,
                                 double max_correspondence_distance, double kernel_scale, double JTJ[36],
                                 double JTr[6], int *n_correspondences);
/* B independent AlignPointsToMap problems against one map (Registration.cpp:138-167 each) in one call; no reference
 * counterpart (its Python layer loops). Hypothesis b aligns xyz[offset[b] .. offset[b] + count[b]) from
 * initial_guesses[b] (row-major 4x4) with max_correspondence_distance[b] and kernel_scale[b]. Ranges may overlap or
 * repeat, so one cloud can be tried from many guesses without copying it. Out: poses[b][16], iterations[b], and
 * inliers[b] (may be NULL): the n_correspondences kb_registration_build_system reports for the source mapped by
 * poses[b]. Each hypothesis gives, bit for bit, the pose and iteration count of kb_registration_align_points_to_map
 * on it alone; the hypotheses run side by side on teams of CTAs of one launch. Every argument is checked before any
 * work starts: KB_ERR_NOT_SE3 for a guess that is not in SE(3), KB_ERR_INVALID_ARG for a range outside
 * [0, n_points) or a NULL pointer; on error no output is written. B = 0 does nothing. The host form leaves
 * kb_registration_last_iterations at iterations[B - 1], like a loop of single calls. */
int kb_registration_align_batch(kb_registration *reg, const double *xyz, size_t n_points, const size_t *offset,
                                const size_t *count, size_t B, const kb_map *map, const double *initial_guesses,
                                const double *max_correspondence_distance, const double *kernel_scale, double *poses,
                                int *iterations, int *inliers);
/* same with every array (points, ranges, guesses, scalars, outputs) in device memory on the map's device. The ranges,
 * guesses and scalars are read back first (one small synchronous copy: the launch is planned on the host); the
 * alignment itself is asynchronous on the map's stream (kb_map_sync). kb_registration_last_iterations is unchanged. */
int kb_registration_align_batch_dev(kb_registration *reg, const double *d_xyz, size_t n_points, const size_t *d_offset,
                                    const size_t *d_count, size_t B, const kb_map *map, const double *d_initial_guesses,
                                    const double *d_max_correspondence_distance, const double *d_kernel_scale,
                                    double *d_poses, int *d_iterations, int *d_inliers);

/* ---- kiss_icp::Preprocessor (cpp/kiss_icp/core/Preprocessing.hpp:32-45) ----------------- */
int kb_preprocessor_create(double max_range, double min_range, int deskew, int max_num_threads,
                           kb_preprocessor **out);
int kb_preprocessor_destroy(kb_preprocessor *pre);
/* Preprocess(frame, timestamps, relative_motion) Preprocessing.cpp:55-95 / `_preprocess`.
 * out_xyz double[capacity][3]; *n_out = points kept (order preserved). */
int kb_preprocessor_preprocess(kb_preprocessor *pre, const double *xyz, size_t n, const double *timestamps,
                               size_t n_timestamps, const double relative_motion[16], double *out_xyz,
                               size_t capacity, size_t *n_out);

/* ---- kiss_icp::AdaptiveThreshold (cpp/kiss_icp/core/Threshold.hpp:29-47) ---------------- */
int kb_threshold_create(double initial_threshold, double min_motion_threshold, double max_range,
                        kb_threshold **out);
int kb_threshold_destroy(kb_threshold *th);
/* ComputeThreshold() Threshold.hpp:38 / `_compute_threshold` */
int kb_threshold_compute(const kb_threshold *th, double *out_sigma);
/* UpdateModelDeviation(SE3) Threshold.cpp:38-49 / `_update_model_deviation` */
int kb_threshold_update_model_deviation(kb_threshold *th, const double model_deviation[16]);

/* ---- kiss_icp::VoxelDownsample (cpp/kiss_icp/core/VoxelUtils.cpp:7-21) ------------------ */
/* `_voxel_down_sample(frame, voxel_size)` kiss_icp_pybind.cpp:123. Output ORDER is the
 * reference's (robin_map iteration order) — it is result-affecting downstream. */
int kb_voxel_down_sample(const double *xyz, size_t n, double voxel_size, double *out_xyz, size_t capacity,
                         size_t *n_out);

/* ---- `_correct_kitti_scan(frame)` (python/kiss_icp/pybind/kiss_icp_pybind.cpp:127-138) ---- */
/* The KITTI loader's per-point intrinsic correction (datasets/kitti.py:44-48,68): every point is rotated by
 * 0.205 deg about normalized(pt x e_z). out_xyz may alias xyz. The _dev form works on device buffers and is
 * asynchronous on the calling thread's stream (kb_set_stream), so it chains into kb_pipeline_register_frame_dev. */
int kb_correct_kitti_scan(const double *xyz, size_t n, double *out_xyz);
int kb_correct_kitti_scan_dev(const double *d_xyz, size_t n, double *d_out_xyz);

/* ---- kiss_icp::pipeline::KissICP (cpp/kiss_icp/pipeline/KissICP.hpp:36-96) -------------- */
/* KISSConfig KissICP.hpp:36-54, field for field */
typedef struct kb_config {
    double voxel_size;           /* 1.0   */
    double max_range;            /* 100.0 */
    double min_range;            /* 0.0   */
    int max_points_per_voxel;    /* 20    */
    double min_motion_th;        /* 0.1   */
    double initial_threshold;    /* 2.0   */
    int max_num_iterations;      /* 500   */
    double convergence_criterion; /* 1e-4 */
    int max_num_threads;         /* 0 (ignored on the GPU) */
    int deskew;                  /* 1     */
} kb_config;
void kb_config_default(kb_config *cfg);

int kb_pipeline_create(const kb_config *cfg, kb_pipeline **out);
int kb_pipeline_destroy(kb_pipeline *p);
/* RegisterFrame(frame, timestamps) KissICP.cpp:35-68. The two clouds the reference returns by
 * value (preprocessed_frame, source) stay on the device; fetch them with
 * kb_pipeline_last_clouds only when wanted (ROS publishes them only for debugging,
 * ros/src/OdometryServer.cpp:168-172). */
int kb_pipeline_register_frame(kb_pipeline *p, const double *xyz, size_t n, const double *timestamps,
                               size_t n_timestamps);
/* same with a float32 frame float[n][3] (KITTI .bin / PointCloud2 payloads are float32 and the reference widens
 * them on the host: python/kiss_icp/datasets/kitti.py:66, ros/src/Utils.hpp:198-208). Half the H2D bytes; the
 * exact float->double widening happens on the device, so results equal the f64 call on the widened array. */
int kb_pipeline_register_frame_f32(kb_pipeline *p, const float *xyz, size_t n, const double *timestamps,
                                   size_t n_timestamps);
/* same, frame (and stamps) already resident in HBM on the pipeline's device */
int kb_pipeline_register_frame_dev(kb_pipeline *p, const double *d_xyz, size_t n, const double *d_timestamps,
                                   size_t n_timestamps);
/* A whole sequence: the loop `for frame in dataset: RegisterFrame(frame, stamps)` of
 * python/kiss_icp/pipeline.py:106-112 as one call. Poses, motion model, threshold and map never leave the device
 * between frames, so the frames are QUEUED: frame k+1 is copied to the device while frame k is registered and
 * results are read back behind the queue (depth 3). Results are identical to `count` blocking calls.
 * xyz[k] is frame k in the given layout, timestamps / n_timestamps may be NULL (no stamps at all);
 * poses_out, if not NULL, receives the `count` row-major poses. An invalid frame (e.g. too few stamps) stops the
 * sequence with the error the blocking call would give, after the frames before it were registered. Host buffers
 * may be pageable (staged through pinned memory) or pinned (copied directly). */
enum kb_frame_layout { KB_FRAMES_HOST_F64 = 0, KB_FRAMES_HOST_F32 = 1, KB_FRAMES_DEVICE_F64 = 2 };
int kb_pipeline_register_frames(kb_pipeline *p, const void *const *xyz, const size_t *n,
                                const double *const *timestamps, const size_t *n_timestamps, size_t count,
                                int layout, double *poses_out);
/* how many frames were vetoed by the kernel (voxel table sized too optimistically), grown for and replayed */
int kb_pipeline_grow_retries(const kb_pipeline *p, unsigned long long *out);
/* sizes / contents of the (preprocessed_frame, source) tuple of the last RegisterFrame */
int kb_pipeline_last_cloud_sizes(const kb_pipeline *p, size_t *n_preprocessed, size_t *n_source);
int kb_pipeline_last_clouds(const kb_pipeline *p, double *preprocessed_xyz, size_t cap_preprocessed,
                            double *source_xyz, size_t cap_source);
/* Voxelize(frame) KissICP.cpp:70-75 -> (source, frame_downsample) */
int kb_pipeline_voxelize(kb_pipeline *p, const double *xyz, size_t n, double *source_xyz, size_t cap_source,
                         size_t *n_source, double *downsample_xyz, size_t cap_downsample, size_t *n_downsample);
/* pose() / delta() KissICP.hpp:81-85 (getters and setters) */
int kb_pipeline_pose(const kb_pipeline *p, double out[16]);
int kb_pipeline_delta(const kb_pipeline *p, double out[16]);
int kb_pipeline_set_pose(kb_pipeline *p, const double pose[16]);
int kb_pipeline_set_delta(kb_pipeline *p, const double delta[16]);
/* VoxelMap() KissICP.hpp:78-79 — borrowed handle, owned by the pipeline */
kb_map *kb_pipeline_voxel_map(kb_pipeline *p);
/* LocalMap() KissICP.hpp:76 == kb_map_pointcloud(kb_pipeline_voxel_map(p), ...) */
/* diagnostics: adaptive threshold sigma used by / ICP iterations of the last RegisterFrame */
int kb_pipeline_last_sigma(const kb_pipeline *p, double *out);
int kb_pipeline_last_iterations(const kb_pipeline *p, int *out);
/* adaptive_threshold_.ComputeThreshold() of the pipeline's own estimator (Threshold.hpp:38):
 * the sigma the NEXT RegisterFrame will use */
int kb_pipeline_threshold(const kb_pipeline *p, double *out_sigma);
/* (profiling and diagnostic entry points: kiss_icp_b200_debug.h) */
/* kernels launched by this pipeline so far (bench "gpu_launches") */
int kb_pipeline_launch_count(const kb_pipeline *p, unsigned long long *out);

/* ---- checkpoint / restore ----------------------------------------------------------------
 * The reference leaves a sequence's whole state public: the map (VoxelHashMap::map_,
 * cpp/kiss_icp/core/VoxelHashMap.hpp:56), pose() / delta() as mutable Sophus::SE3d&
 * (cpp/kiss_icp/pipeline/KissICP.hpp:79-95) and AdaptiveThreshold::model_sse_ / num_samples_
 * (cpp/kiss_icp/core/Threshold.hpp:44-46). These calls read and write the same state, exactly.
 * A pipeline's map is restored with kb_map_load(kb_pipeline_voxel_map(p), ...); there is no
 * blob format, callers compose the calls they need. */
/* Replace the map's contents. Layout = kb_map_dump's: voxels int[n_voxels][3] in any order,
 * counts int[n_voxels], points double[n_points][3] concatenated per voxel in insertion order.
 * Synchronous: all or nothing. KB_ERR_INVALID_ARG (map, counters and capacity unchanged) for a
 * duplicate voxel, a count outside [1, max_points_per_voxel], n_points != sum of counts, a
 * non-finite coordinate, or a point whose voxel (the hot path's own FP64 voxel function) is not
 * the voxel it is listed under. The _dev form takes device pointers on the map's device. */
int kb_map_load(kb_map *map, const int *voxels, const int *counts, const double *points, size_t n_voxels,
                size_t n_points);
int kb_map_load_dev(kb_map *map, const int *d_voxels, const int *d_counts, const double *d_points, size_t n_voxels,
                    size_t n_points);
/* the pipeline's exact state; SE(3) elements in Sophus::SE3d::params() order {qx,qy,qz,qw,tx,ty,tz} */
typedef struct kb_pipeline_state {
    double pose[7];
    double delta[7];
    double model_sse;
    int num_samples;
} kb_pipeline_state;
int kb_pipeline_get_state(const kb_pipeline *p, kb_pipeline_state *out);
/* Stores the values bit for bit (no renormalisation: get -> set -> get is the identity) and drops
 * any prefetched frame. KB_ERR_INVALID_ARG for a non-finite value, num_samples < 1 or
 * model_sse < 0; KB_ERR_NOT_SE3 for a quaternion whose squared norm is not within 1e-10 of 1. */
int kb_pipeline_set_state(kb_pipeline *p, const kb_pipeline_state *s);
/* the stand-alone AdaptiveThreshold's model_sse_ / num_samples_ (same checks as above) */
int kb_threshold_get_state(const kb_threshold *th, double *model_sse, int *num_samples);
int kb_threshold_set_state(kb_threshold *th, double model_sse, int num_samples);

/* ---- localization in a fixed prior map ----------------------------------------------------
 * No reference counterpart. A localizer registers every frame with RegisterFrame (KissICP.cpp:35-68) without the map
 * update (:61, local_map_.Update) against a prior map that it never writes, and reports how well each frame fits. */
/* The fit of one frame at its final pose, with that frame's (3 sigma, sigma): n_correspondences = source points whose
 * nearest map neighbour is closer than 3 sigma (what kb_registration_build_system counts for the source mapped by the
 * pose), n_source = source points, sum_sq_residual = sum of |r|^2 over the correspondences (unweighted), JTJ = the
 * Geman-McClure-weighted J^T W J of kb_registration_build_system for the same input, row-major, symmetric: the
 * information matrix of the pose. Bit-identical from run to run for a given grid size (kb_set_grid_blocks). */
typedef struct kb_fit {
    int n_correspondences, n_source;
    double sum_sq_residual;
    double JTJ[36];
} kb_fit;
/* A pipeline that localizes in `prior` instead of building a map. The prior must be on the pipeline's device (the
 * calling thread's, kb_set_device) and have cfg's voxel_size and max_points_per_voxel, else KB_ERR_INVALID_ARG; its
 * max_distance does not matter (nothing is evicted). A pipeline's own map (kb_pipeline_voxel_map of an odometry
 * pipeline) cannot be a prior. Waits once for the work queued on the prior. The localizer allocates no voxel table;
 * kb_pipeline_voxel_map returns the prior, borrowed. While localizers exist, every call that would change or free the
 * prior (kb_map_clear, _update_origin, _update_pose, _add_points, _remove_far, _compact, _load[_dev], _destroy) fails
 * with KB_ERR_INVALID_ARG and changes nothing; read-only calls keep working. Several localizers, on any host threads,
 * may share one prior. kb_pipeline_destroy of a localizer waits for its own streams before it releases the prior.
 * Every other kb_pipeline_* call works as on an odometry pipeline; set_pose seeds the track (e.g. from a
 * kb_registration_align_batch relocalization). */
int kb_pipeline_create_localizer(const kb_config *cfg, const kb_map *prior, kb_pipeline **out);
/* localizers reading the map (0: it may be changed) */
int kb_map_readers(const kb_map *map, int *out);
/* the fit of the last frame (all zero before the first); KB_ERR_INVALID_ARG on an odometry pipeline without fit
 * reporting (kb_pipeline_set_fit_reporting) */
int kb_pipeline_last_fit(const kb_pipeline *p, kb_fit *out);
/* kb_pipeline_register_frames with one fit per frame in fits_out[count] (may be NULL), read behind the queue like
 * the poses. Same poses as kb_pipeline_register_frames. A non-NULL fits_out on an odometry pipeline without fit
 * reporting is KB_ERR_INVALID_ARG. */
int kb_pipeline_register_frames_fit(kb_pipeline *p, const void *const *xyz, const size_t *n,
                                    const double *const *timestamps, const size_t *n_timestamps, size_t count,
                                    int layout, double *poses_out, kb_fit *fits_out);
/* Fit reporting of an odometry pipeline (off when it is created). With it on, every registered frame also gets a kb_fit,
 * defined as a localizer's, against the pipeline's own map as that frame's ICP saw it: before the frame's
 * local_map_.Update (KissICP.cpp:61), which would put the scan's own points in the map. kb_pipeline_last_fit and
 * kb_pipeline_register_frames_fit then work as on a localizer. A frame vetoed for table capacity gets the fit of its
 * replay. Poses, iterations, the threshold state and the map are bit for bit those of reporting off; the frames run a
 * kernel of their own, which costs one more grid barrier and the fit pass per frame. Enabling allocates the fit buffers
 * and resets the last fit to zeros (KB_ERR_CUDA if that fails; reporting stays off), enabling it again is a no-op;
 * disabling releases them. A localizer always reports: enabled = 1 is a no-op, 0 is KB_ERR_INVALID_ARG.
 * KB_ERR_INVALID_ARG for p == NULL. */
int kb_pipeline_set_fit_reporting(kb_pipeline *p, int enabled);
/* *out = 1 if the pipeline reports fits (a localizer, or fit reporting on), else 0; KB_ERR_INVALID_ARG for NULL */
int kb_pipeline_fit_reporting(const kb_pipeline *p, int *out);

/* ---- plane constraints: which directions a registration pins down ---------------------------
 * No reference counterpart. For every correspondence of the fit (source point p = pose * s, nearest map neighbour q
 * closer than max_correspondence_distance) whose voxel (q's own) holds m >= 3 points: the voxel's mean and covariance
 * C (1/m), n = a unit eigenvector of C's smallest eigenvalue l0 (l0 <= l1 <= l2), planarity a = (l1 - l0) / l2 (0 when
 * l2 = 0), residual e = n.(p - q) and Jacobian J = [n^T, (p x n)^T] in the tangent order (translation, rotation) of
 * kb_fit.JTJ. The information matrix is a sum of rank-one terms a J^T J: a direction no plane faces has no
 * information. Bit-identical from run to run for a given grid size (kb_set_grid_blocks). */
typedef struct kb_constraints {
    int n_planes;                   /* correspondences whose map voxel holds >= 3 points                */
    double weight_sum;              /* sum of planarity weights a_i                                     */
    double sum_sq_plane_residual;   /* sum a_i e_i^2                                                    */
    double information[36];         /* sum a_i J_i^T J_i, row-major, symmetric, (translation, rotation) */
} kb_constraints;
/* one source (host xyz[n][3]) at one pose against a map. Read-only: allowed while localizers hold the map.
 * KB_ERR_INVALID_ARG for a NULL argument, KB_ERR_NOT_SE3 for a pose outside SE(3); n = 0 or an empty map gives zeros. */
int kb_registration_constraints(kb_registration *reg, const double *xyz, size_t n, const kb_map *map,
                                const double pose[16], double max_correspondence_distance, kb_constraints *out);
/* Plane-constraint reporting (off when a pipeline is created): every registered frame also gets a kb_constraints, of
 * the fit's correspondences (3 sigma at the final pose, against the map the fit is against: for odometry, before the
 * frame's own update). Needs a pipeline that reports fits (a localizer, or kb_pipeline_set_fit_reporting on), else
 * KB_ERR_INVALID_ARG and nothing changes. Enabling allocates its buffers and zeroes the last result, enabling again is a
 * no-op, 0 releases them. While it is on, kb_pipeline_set_fit_reporting(p, 0) is KB_ERR_INVALID_ARG. Poses, fits and
 * the map are bit for bit those of reporting off; the frames run a kernel of their own. */
int kb_pipeline_set_constraint_reporting(kb_pipeline *p, int enabled);
/* the plane constraints of the last frame (zeros before the first); KB_ERR_INVALID_ARG when reporting is off */
int kb_pipeline_last_constraints(const kb_pipeline *p, kb_constraints *out);
/* kb_pipeline_register_frames_fit with one kb_constraints per frame in constraints_out[count] (may be NULL; non-NULL
 * without constraint reporting is KB_ERR_INVALID_ARG). A frame vetoed for table capacity gets its replay's. */
int kb_pipeline_register_frames_constraints(kb_pipeline *p, const void *const *xyz, const size_t *n,
                                            const double *const *timestamps, const size_t *n_timestamps, size_t count,
                                            int layout, double *poses_out, kb_fit *fits_out, kb_constraints *constraints_out);

/* ---- degeneracy-aware ICP: hold the prediction along directions a scan does not constrain ----------------
 * No reference counterpart. In a tunnel, a corridor or open ground with one wall, point-to-point ICP has no information
 * along the free axis and drags the pose toward the previous scan's ring pattern. With a degeneracy ratio rho in
 * (0, 1), every frame first runs the plane pass of kb_registration_constraints at its initial guess G = last_pose *
 * last_delta with the frame's own 3 sigma, but with the lever about the guess's position c = G.t:
 * J_c = [n^T, ((p - c) x n)^T], H_c = sum a J_c^T J_c (= A^T H A, A = [[I, [c]x], [0, I]]). Its translation block and
 * its rotation block are eigen-decomposed separately (3x3 Jacobi, ascending); in each block an axis with
 * l_k < rho * l_max is held, except that nothing is held in a block with l_max <= 0 or in a frame without a plane term.
 * P = blockdiag(V_t M_t V_t^T, V_r M_r V_r^T), M = 0 on held axes and 1 elsewhere. Every ICP step dx (tangent order
 * translation, rotation, about the map origin) becomes A P A^-1 dx before Exp and before the convergence test, so
 * held directions keep the prediction (the constant-velocity model). A frame that holds nothing runs the plain ICP
 * loop: its result is bit for bit that of rho = 0. No pipeline state is added: checkpoints are unchanged.
 * Recommended: rho = 0.02 (both synthetic test streams, which are well conditioned, stay above it in both blocks;
 * DESIGN.md section 4.16). The frames run a kernel of their own with one more pass and grid barrier before ICP. */
typedef struct kb_degeneracy {
    int n_planes;                       /* plane terms of the pass at the guess (0: nothing held)                 */
    double weight_sum;                  /* sum of their planarity weights                                         */
    double translation_eigenvalues[3];  /* of H_c[:3, :3], ascending                                              */
    double translation_axes[9];         /* row-major, column k = unit axis of eigenvalue k (sign arbitrary)       */
    double rotation_eigenvalues[3];     /* of H_c[3:, 3:], ascending                                              */
    double rotation_axes[9];            /* likewise, rotation axes through c                                      */
    int translation_held[3];            /* 1: axis k was held                                                     */
    int rotation_held[3];
} kb_degeneracy;
/* Set the degeneracy ratio (0 when a pipeline is created: off). ratio > 0 needs a pipeline that reports fits (a
 * localizer, or kb_pipeline_set_fit_reporting on), else KB_ERR_INVALID_ARG. NaN, negative and >= 1 values are
 * KB_ERR_INVALID_ARG. On error nothing changes. A ratio > 0 allocates the per-frame results (zeroed; KB_ERR_CUDA if
 * that fails, and the mode stays off), changing it keeps them, 0 releases them. While it is on,
 * kb_pipeline_set_fit_reporting(p, 0) is KB_ERR_INVALID_ARG. */
int kb_pipeline_set_degeneracy_ratio(kb_pipeline *p, double ratio);
/* the pipeline's degeneracy ratio (0: off); KB_ERR_INVALID_ARG for NULL */
int kb_pipeline_degeneracy_ratio(const kb_pipeline *p, double *out);
/* the degeneracy result of the last frame (zeros before the first); KB_ERR_INVALID_ARG when the mode is off */
int kb_pipeline_last_degeneracy(const kb_pipeline *p, kb_degeneracy *out);
/* kb_pipeline_register_frames_constraints with one kb_degeneracy per frame in degeneracy_out[count] (may be NULL;
 * non-NULL with the mode off is KB_ERR_INVALID_ARG), read behind the queue like the fits. A frame vetoed for table
 * capacity gets its replay's. */
int kb_pipeline_register_frames_degeneracy(kb_pipeline *p, const void *const *xyz, const size_t *n,
                                           const double *const *timestamps, const size_t *n_timestamps, size_t count,
                                           int layout, double *poses_out, kb_fit *fits_out, kb_constraints *constraints_out,
                                           kb_degeneracy *degeneracy_out);

/* ---- sampled motion: deskew and predict a scan from IMU or wheel-odometry samples --------------------------
 * No reference counterpart (DESIGN.md section 4.17). The pipeline's own motion model is KISS-ICP's constant velocity:
 * the previous frame's last_delta deskews the next scan and predicts its pose. A kb_motion replaces it for one frame
 * with the LiDAR's measured trajectory T(t), sampled at times[k]:
 *   T(t) = T_k Exp(tau xi_k), k the interval [t_k, t_k+1] holding t, tau = t - t_k, xi_k = Log(T_k^-1 T_k+1) / (t_k+1 - t_k)
 * (= T_k Exp(alpha Log(T_k^-1 T_k+1)), alpha = tau / (t_k+1 - t_k)). Before t_0 and after t_m-1 the first and the last
 * interval are extrapolated.
 * Deskew (cfg.deskew on and the frame has stamps): point p with stamp s becomes T(end_time)^-1 T(s + stamp_offset) p, and
 * the range crop follows as without a kb_motion. A NaN stamp makes a NaN point, which the crop drops. Constant stamps
 * are valid. Without stamps, or with cfg.deskew = 0, the points are used as they are.
 * Prediction: when the previous frame was registered with a kb_motion whose end_time (kb_pipeline_motion_time) lies in
 * [t_0, t_m-1] of this frame's samples, the initial guess is last_pose * T(prev)^-1 T(end_time); otherwise it is the
 * constant-velocity guess last_pose * last_delta. The model deviation of the adaptive threshold is guess^-1 new_pose,
 * last_delta after the frame is last_pose^-1 new_pose and the degeneracy pass is taken at this guess, as always. */
#define KB_MOTION_MAX_SAMPLES 65536
typedef struct kb_motion {
    const double *times;  /* [m], strictly increasing, finite, in the sample clock                           */
    const double *poses;  /* [m][16] row-major SE(3): the LiDAR's pose at times[k] in any fixed frame        */
    size_t m;             /* 2 <= m <= KB_MOTION_MAX_SAMPLES; 0 in a frame of kb_pipeline_register_frames_motion:
                             no kb_motion for that frame                                                      */
    double stamp_offset;  /* added to every point stamp to put it on the sample clock (per-scan stamps)      */
    double end_time;      /* sample-clock time the scan's pose refers to; its points are deskewed to it      */
} kb_motion;
/* Host only (works without a device). KB_ERR_INVALID_ARG for a NULL motion, times or poses, m outside
 * [2, KB_MOTION_MAX_SAMPLES], times that are not finite or not strictly increasing, consecutive samples whose relative
 * rotation is within 1e-6 rad of pi or more (where Log is not unique), a non-finite stamp_offset or end_time;
 * KB_ERR_NOT_SE3 for a pose outside SE(3). */
int kb_motion_check(const kb_motion *motion);
/* kb_pipeline_register_frames_degeneracy with a kb_motion per frame: motion[count] may be NULL (none at all), and a frame
 * whose motion has m == 0 has none. Every motion is checked (kb_motion_check) before any device work; on error nothing is
 * registered. A frame with a kb_motion does not depend on the previous frame's result, so, like a frame without stamps,
 * its front end (deskew, crop, downsampling) may run in the launch of the frame before it. A frame vetoed for table
 * capacity and replayed keeps its prediction. Outputs as kb_pipeline_register_frames_degeneracy. */
int kb_pipeline_register_frames_motion(kb_pipeline *p, const void *const *xyz, const size_t *n,
                                       const double *const *timestamps, const size_t *n_timestamps,
                                       const kb_motion *motion, size_t count, int layout, double *poses_out,
                                       kb_fit *fits_out, kb_constraints *constraints_out, kb_degeneracy *degeneracy_out);
/* the end_time of the last frame registered, if it had a kb_motion, else NaN (also for a new pipeline). Part of a
 * checkpoint next to kb_pipeline_state: set it back with kb_pipeline_set_motion_time (NaN: none; +-inf is
 * KB_ERR_INVALID_ARG). */
int kb_pipeline_motion_time(const kb_pipeline *p, double *out);
int kb_pipeline_set_motion_time(kb_pipeline *p, double end_time);
/* The deskew of one frame alone: out[k] = T(end_time)^-1 T(timestamps[k] + stamp_offset) xyz[k], no crop. Without
 * stamps (n_timestamps == 0) out = xyz. KB_ERR_OUT_OF_RANGE for 0 < n_timestamps < n, the checks of kb_motion_check
 * otherwise. Synchronous; out may alias xyz. */
int kb_deskew_motion(const double *xyz, size_t n, const double *timestamps, size_t n_timestamps, const kb_motion *motion,
                     double *out);

/* ---- multi-LiDAR rigs: per-sensor extrinsics, range crops and clocks, merged on the device ------------------------
 * No reference counterpart (DESIGN.md section 4.18). A rig is 1 <= S <= KB_RIG_MAX_SENSORS sensors mounted on a base
 * (the vehicle). Sensor i has an extrinsic E_i (base <- sensor), a range crop (min_range_i, max_range_i) and, per frame,
 * a stamp_offset_i that puts its point stamps on the common clock. A rig frame is S point arrays (and S stamp arrays:
 * either every sensor with points has stamps or none has; a mix is KB_ERR_INVALID_ARG, a sensor without points may
 * have none either way). Its merged frame is:
 *   order   the sensors' points concatenated in sensor order, each sensor's in its own order (the downsample keeps the
 *           first point per voxel);
 *   crop    point p of sensor i is kept iff min_range_i < |p| < max_range_i in the sensor frame; a point that is not
 *           becomes NaN (the frame's own crop drops it), its stamp is kept. A sensor with min_range 0 and max_range
 *           +inf has no crop: its points pass as they are;
 *   to base q = E_i p (an identity E_i passes the point without arithmetic);
 *   stamps  s + stamp_offset_i.
 * Then, with deskewing on and stamps given: without a kb_motion the merged frame and merged stamps are registered as a
 * stamped frame (constant velocity: stamps normalised over the union's [min, max], deskewed to its end by last_delta,
 * exactly KISS-ICP on the concatenated base-frame cloud); with a kb_motion (the BASE's poses) a point becomes
 * T(end_time)^-1 T(s + stamp_offset_i + motion.stamp_offset) E_i p and the frame is registered without stamps. The
 * frame's own crop (cfg.min_range / max_range, about the base origin) applies afterwards. Poses, last_delta, the map,
 * fits, constraints and degeneracy refer to the base; the preprocessed cloud of kb_pipeline_last_clouds is the merged
 * base-frame cloud. */
#define KB_RIG_MAX_SENSORS 16
typedef struct kb_sensor {
    double extrinsic[16];        /* row-major SE(3), base <- sensor                             */
    double min_range, max_range; /* 0 <= min_range < max_range (+inf allowed), in the sensor frame */
} kb_sensor;
/* Host only (works without a device). KB_ERR_INVALID_ARG for NULL sensors, n_sensors outside [1, KB_RIG_MAX_SENSORS],
 * a NaN, negative or infinite min_range, a NaN max_range or min_range >= max_range; KB_ERR_NOT_SE3 for an extrinsic
 * outside SE(3). */
int kb_rig_check(const kb_sensor *sensors, size_t n_sensors);
/* kb_pipeline_register_frames_motion for rig frames: frame k is xyz[k S + i], n[k S + i] (i < S) in the layout, stamps
 * timestamps / n_timestamps likewise (both may be NULL: no stamps at all), stamp_offsets[k S + i] (NULL: all 0, each
 * finite), motion as kb_pipeline_register_frames_motion (NULL or [count], m == 0: none). The merged frame must hold
 * fewer than 2^30 points. The rig and every motion are checked before any device work (on error nothing is
 * registered); an invalid frame stops the sequence after the frames before it were registered. Rig frames with stamps
 * and without a kb_motion depend on the previous frame's result and are not prefetched; the others are. Outputs as
 * kb_pipeline_register_frames_degeneracy. */
int kb_pipeline_register_rig_frames(kb_pipeline *p, const kb_sensor *sensors, size_t n_sensors, const void *const *xyz,
                                    const size_t *n, const double *const *timestamps, const size_t *n_timestamps,
                                    const double *stamp_offsets, const kb_motion *motion, size_t count, int layout,
                                    double *poses_out, kb_fit *fits_out, kb_constraints *constraints_out,
                                    kb_degeneracy *degeneracy_out);
/* The merge of one rig frame alone (host float64 arrays, synchronous): xyz_out[N][3] (N the sum of n) receives the
 * merged base-frame points, deskewed along the motion when motion is not NULL and the frame has stamps, no frame
 * crop; timestamps_out[N] (may be NULL) the merged stamps s + stamp_offset_i, when the frame has stamps. Checks of
 * kb_rig_check, kb_motion_check and of the stamps as kb_pipeline_register_rig_frames. */
int kb_merge_rig(const kb_sensor *sensors, size_t n_sensors, const double *const *xyz, const size_t *n,
                 const double *const *timestamps, const size_t *n_timestamps, const double *stamp_offsets,
                 const kb_motion *motion, double *xyz_out, double *timestamps_out);
/* Extrinsic calibration of a rig from a recorded run (DESIGN.md section 4.19). Given a map in the world frame, the base
 * poses T_k (world <- base) of K frames and, per frame k and sensor j, a scan p in the sensor frame without stamps, every
 * refined sensor j (refine[j] = 1; refine NULL: all) minimises over E_j
 *   sum_k sum_i rho(|T_k E_j p - q|),  q the nearest map point of T_k E_j p, kept when closer than
 *   max_correspondence_distance, rho KISS-ICP's Geman-McClure (w = kernel_scale^2 / (kernel_scale + |r|^2)^2).
 * A point counts only if min_range_j < |p| < max_range_j (strict; a non-finite point fails). Each iteration builds,
 * per refined sensor, KISS-ICP's system with source p and target (T_k E_j)^-1 q, solves it as the ICP loop does and
 * sets E_j <- E_j Exp(dx), tangent (translation, rotation) along the sensor's own axes. Sensors are independent: each
 * stops at |dx| < convergence_criterion or after max_iterations. A sensor without correspondences keeps its extrinsic.
 * At the returned extrinsics one more pass gives each refined sensor its kb_fit (n_source: points that passed the crop;
 * JTJ in the sensor tangent) and its kb_constraints over the same correspondences, J = [n_s^T, (p x n_s)^T] with the
 * voxel normal rotated into the sensor frame, n_s = (R_k R_j)^T n. A sensor that is not refined is not read: its
 * extrinsic comes back bit for bit and its report is zeros. A refined extrinsic that no step moved comes back bit for
 * bit too.
 * frames: xyz[k S + j], n[k S + j] in `layout` (device frames on the map's device are read in place). Synchronous;
 * only reads the map (allowed while localizers hold it). Bit-identical from run to run for a given grid size
 * (kb_set_grid_blocks). Every argument is checked before any device is looked for, and on error nothing is written:
 * KB_ERR_INVALID_ARG for a NULL argument (an array of a refined sensor with points included), a refine entry other
 * than 0 or 1, an option that is NaN or out of range, a layout that is none of kb_frame_layout, or 2^31 or more points
 * of the refined sensors in all; the checks of kb_rig_check; KB_ERR_NOT_SE3 for a pose outside SE(3). K = 0, or no
 * refined sensor, returns the extrinsics and zero reports without device work. KB_ERR_CUDA when a device allocation
 * fails. */
typedef struct kb_rig_calibration_options {
    double max_correspondence_distance;  /* > 0, finite                                      */
    double kernel_scale;                 /* > 0, finite                                      */
    int    max_iterations;               /* >= 0; 0: only the report at the given extrinsics */
    double convergence_criterion;        /* >= 0, finite                                     */
} kb_rig_calibration_options;
typedef struct kb_sensor_calibration {
    int iterations, converged;
    kb_fit fit;                  /* at the returned extrinsic, sensor tangent          */
    kb_constraints constraints;  /* same correspondences, sensor tangent, lever = p    */
} kb_sensor_calibration;
int kb_calibrate_rig(const kb_map *map, const double *poses /* [K][16] */, size_t K,
                     const kb_sensor *sensors, size_t n_sensors, const int *refine /* [S], NULL: all */,
                     const void *const *xyz /* [K S] */, const size_t *n /* [K S] */, int layout,
                     const kb_rig_calibration_options *opt,
                     double *extrinsics_out /* [S][16] */, kb_sensor_calibration *report_out /* [S] */);
/* Clock-offset and extrinsic calibration of a rig from a recorded run with per-point stamps (DESIGN.md section 4.20).
 * The base moves along one trajectory over the whole run, T(t) = T_i Exp((t - t_i) xi_i) (the kb_motion's samples,
 * world <- base; end_time is ignored). Point p of frame k, sensor j, with stamp s is at trajectory-clock time
 *   t = s + stamp_offsets[k S + j] + o_j + trajectory->stamp_offset
 * (the stamp offsets of all frames on one clock, e.g. each sweep's start time), o_j the sensor's unknown clock offset,
 * and at m = T(t) E_j p in the world. Every processed sensor (refine[j] or refine_time[j]) minimises
 *   sum rho(|m - q|),  q the nearest map point of m, kept when closer than max_correspondence_distance, rho as in
 *   kb_calibrate_rig,
 * over E_j <- E_j Exp(dx) (refine[j]) and o_j <- o_j + do (refine_time[j]). Per correspondence, in the sensor
 * coordinates of kb_calibrate_rig (source p, target q_s = (T(t) E_j)^-1 q), the extrinsic columns are KISS-ICP's
 * J = [I, -[p]x] and the time column J_o = R_j^T (v_i + w_i x E_j p), (v_i, w_i) = xi_i of the point's interval.
 * The 7x7 system [H_ee h; h^T H_oo] [dx; do] = -[g_e; g_o] is solved by a Schur complement on the offset: H_ee (the
 * ICP loop's 6x6 rule) is solved for -g_e and for h, s = H_oo - h^T H_ee^-1 h, do = -(g_o + h^T H_ee^-1 g_e) / s,
 * dx = H_ee^-1 (-g_e - h do). The offset is held (do = 0, and dx is exactly kb_calibrate_rig's step on the same sums)
 * when the sensor's offset is not refined, H_oo is 0, or s <= KB_CLOCK_HOLD_RATIO H_oo (the offset is confounded with
 * the extrinsic). With only the offset refined, do = -g_o / H_oo under the same rule. Without motion (xi = 0, which
 * two bit-identical consecutive samples give exactly) J_o is 0 and the offset comes back bit for bit. A sensor stops
 * when every unknown it refines moved less than its criterion (|dx| < convergence_criterion, |do| <
 * time_convergence_criterion) or after max_iterations. A point counts if it passes its sensor's crop and its stamp is
 * finite. At the returned values one more pass reports, per processed sensor, the kb_fit and kb_constraints of
 * kb_calibrate_rig, time_row = (H_oe, H_oo) and time_schur = s (0: the run does not pin the offset).
 * Frames: xyz[k S + j], n[k S + j] in `layout`; timestamps[k S + j] (n_timestamps[k S + j] == n[k S + j]) are host
 * float64 in every layout: the host reads them to bound each frame's interval search. stamp_offsets NULL: all 0;
 * time_offsets NULL: all 0. Sensors that neither flag selects are not read: their extrinsics and offsets come back
 * bit for bit and their reports are zeros. Synchronous, reads the map only (allowed while localizers hold it),
 * bit-identical from run to run for a given grid size (kb_set_grid_blocks). Every argument is checked before any
 * device is looked for, and on error nothing is written: the checks of kb_calibrate_rig (without poses), and
 * KB_ERR_INVALID_ARG for a refine_time entry other than 0 or 1, a processed sensor's frame with points but NULL stamps
 * or n_timestamps != n, a non-finite stamp offset or time offset of a processed sensor, or a time_convergence_criterion
 * that is NaN, negative or infinite; the checks of kb_motion_check on the trajectory. K = 0, or no processed sensor,
 * returns the values as given and zero reports without device work. */
#define KB_CLOCK_HOLD_RATIO 1e-10
typedef struct kb_rig_clock_calibration_options {
    double max_correspondence_distance;  /* > 0, finite                                    */
    double kernel_scale;                 /* > 0, finite                                    */
    int    max_iterations;               /* >= 0; 0: only the report at the given values   */
    double convergence_criterion;        /* >= 0, finite; of |dx|                          */
    double time_convergence_criterion;   /* >= 0, finite; of |do| [s]                      */
} kb_rig_clock_calibration_options;
typedef struct kb_sensor_clock_calibration {
    int iterations, converged;
    kb_fit fit;                  /* at the returned values, sensor tangent                               */
    kb_constraints constraints;  /* same correspondences, sensor tangent, lever = p                      */
    double time_row[7];          /* (H_oe[6], H_oo) at the returned values                               */
    double time_schur;           /* s = H_oo - H_oe H_ee^-1 H_eo: the offset's information with E_j free */
} kb_sensor_clock_calibration;
int kb_calibrate_rig_clocks(const kb_map *map, const kb_motion *trajectory, const kb_sensor *sensors, size_t n_sensors,
                            const int *refine /* [S], NULL: all */, const int *refine_time /* [S], NULL: all */,
                            const double *time_offsets /* [S], NULL: all 0 */,
                            const void *const *xyz /* [K S] */, const size_t *n /* [K S] */,
                            const double *const *timestamps /* [K S] */, const size_t *n_timestamps /* [K S] */,
                            const double *stamp_offsets /* [K S], NULL: all 0 */, size_t K, int layout,
                            const kb_rig_clock_calibration_options *opt, double *extrinsics_out /* [S][16] */,
                            double *time_offsets_out /* [S] */, kb_sensor_clock_calibration *report_out /* [S] */);

/* ---- relocalization: a global pose search in a bounded region ----------------------------
 * No reference counterpart. Finds a scan's pose in a map without an initial pose: every hypothesis of a grid in x, y
 * and yaw around a centre is scored on the device, the best peaks are refined with kb_registration_align_batch, and
 * the winner is the refined candidate with the most inliers. Whether to accept it is the caller's decision. */
/* The grid: Nx = 2 half_cells_x + 1, Ny = 2 half_cells_y + 1, H = n_yaw Nx Ny <= 2^24 hypotheses. Hypothesis
 * h = (k Ny + (j + half_cells_y)) Nx + (i + half_cells_x), i in [-half_cells_x, half_cells_x], j likewise, k in [0, n_yaw):
 *   yaw_k = (k - n_yaw / 2) yaw_step (integer division), R_h = Rz(yaw_k) R_c with Rz = [c -s 0; s c 0; 0 0 1] from
 *   std::cos / std::sin and R_h[r][c] = (Rz[r][0] R_c[0][c] + Rz[r][1] R_c[1][c]) + Rz[r][2] R_c[2][c],
 *   t_h = (t_c.x + i step, t_c.y + j step, t_c.z).
 * z, roll and pitch come from the centre. The yaw axis is a full circle when |n_yaw yaw_step - 2 pi| < 1e-9.
 * max_correspondence_distance and kernel_scale are those of the refinement (kb_registration_align_points_to_map). */
typedef struct kb_reloc_search {
    double center[16];              /* row-major SE(3) */
    int half_cells_x, half_cells_y; /* >= 0 */
    double step;                    /* metres between grid positions, > 0 */
    int n_yaw;                      /* >= 1 */
    double yaw_step;                /* radians, > 0 */
    int top_k;                      /* peaks refined, 1..256 */
    double max_correspondence_distance, kernel_scale;
} kb_reloc_search;
/* The hypotheses kb_relocalize scores, in order h, as row-major poses[H][16]. Two-call like kb_map_pointcloud: *n_out = H;
 * poses NULL or cap 0 only queries it, cap < H is KB_ERR_CAPACITY. Host only (works without a device).
 * KB_ERR_INVALID_ARG for a field outside its range, H > 2^24 or a non-finite centre translation, KB_ERR_NOT_SE3 for a
 * centre rotation that is not in SO(3). */
int kb_reloc_hypotheses(const kb_reloc_search *search, double *poses, size_t cap, size_t *n_out);
typedef struct kb_reloc_result {
    double pose[16];  /* the winner, refined, row-major */
    int inliers, iterations, rank; /* its inliers, ICP iterations and index among the candidates */
    int n_source;
    int n_hypotheses, n_peaks, n_candidates;
    double runner_up_pose[16];     /* all zero when there is no runner-up */
    int runner_up_inliers;         /* -1 when there is no runner-up */
} kb_reloc_result;
/* Relocalize the source xyz[n] in map within `search`:
 *   1. score_h = source points q whose voxel point_to_voxel(R_h p_q + t_h) the map holds, each component computed as
 *      ((R0 x + R1 y) + R2 z) + t0 (one device launch on the map's stream, integer counts: deterministic);
 *   2. peaks: h is a peak when no neighbour (i +- 1, j +- 1, k +- 1; k wraps on a full circle; no padding at the edges)
 *      has a higher score, or the same score and a smaller h;
 *   3. candidates: the peaks by (score descending, h ascending), the first top_k;
 *   4. refinement: kb_registration_align_batch of the source from every candidate with the search's thresholds, inliers
 *      on: each refined pose, iteration count and inlier count is bit for bit that call's. Uses reg's
 *      max_num_iterations and convergence criterion; kb_registration_last_iterations is unchanged;
 *   5. winner: the most inliers, ties to the lower rank. Runner-up: the best other candidate (same order) whose refined
 *      pose is farther from the winner's than 2 step in xy or 2 yaw_step in rotation angle.
 * candidates (double[top_k][16], the coarse poses), candidate_scores (int[top_k]) and scores (int[H], in order h) may each
 * be NULL; the first n_candidates entries are written. Host buffers. Only reads the map: allowed while localizers hold it.
 * Every argument is checked before any work, and on error nothing is written: KB_ERR_INVALID_ARG for a NULL pointer,
 * n = 0, an empty map, the limits of kb_reloc_hypotheses, or a hypothesis under which a source point's voxel coordinate
 * would not fit in an int (checked from |t_h| and the largest |p|); KB_ERR_NOT_SE3 for the centre. Handles exist only
 * where a device does: without one the call returns KB_ERR_NO_DEVICE once the arguments that need no handle (search,
 * source, out) have passed. */
int kb_relocalize(kb_registration *reg, const double *xyz, size_t n, const kb_map *map, const kb_reloc_search *search,
                  kb_reloc_result *out, double *candidates, int *candidate_scores, int *scores);

/* ---- place recognition: relocalization without any pose, loop-closure candidates -----------------------------
 * No reference counterpart. A database holds the Scan Context descriptor (Kim & Kim, IROS 2018) of a cloud at each
 * keyframe pose of a mapping run. A query cloud is compared with every entry at every cyclic shift on the device; the
 * best entries, rotated by their shift, are initial guesses for kb_registration_align_batch.
 * Parameters: 1 <= n_rings <= 64, 3 <= n_sectors <= 720, n_rings n_sectors <= 4096, max_radius finite and > 0, z_offset
 * finite (defaults 20, 60, 80.0, 2.0).
 * Descriptor D[r][k] of a cloud in its sensor frame (bit for bit; the device rounds like the host, without FMA):
 *   a point with x = y = 0 is skipped; d2 = x*x + y*y;
 *   ring r: b_r <= d2 < b_{r+1} with b_i = (i * (max_radius / n_rings))^2 for i < n_rings and b_{n_rings} =
 *     max_radius * max_radius (computed on the host); a point with d2 >= b_{n_rings} is skipped;
 *   sector k: u_k x p >= 0 and u_{k+1} x p < 0 with u x p = u.x*y - u.y*x, u_k = (cos t_k, sin t_k) from std::cos /
 *     std::sin on the host, t_k = -pi + k * (2 pi / n_sectors), u_{n_sectors} = u_0. Exactly one k passes for every point
 *     (a point no k passes, possible only for subnormal x and y, is skipped);
 *   D[r][k] = max(0, the largest z + z_offset of the cell's points); an empty cell is 0.
 * Distance of a query Q to an entry C: norm_k = sqrt(sum_r D[r][k]^2) (ring order); column k is nonempty when norm_k > 0,
 *   its unit column is D[.][k] / norm_k (zeros when empty). For shift s in [0, n_sectors):
 *   dot_k = sum_r q[r][k] c[r][(k + s) mod n_sectors] (ring order, from 0), S_s = sum_k dot_k (k order, from 0),
 *   m_s = the k where both columns are nonempty, d_s = 1 - S_s / m_s (1 when m_s = 0).
 *   The entry's distance is min_s d_s, its shift the smallest s attaining it.
 * Heading: shift s means the query's column k matches the entry's column k + s: a cloud rotated by Rz(j D), D = 2 pi /
 *   n_sectors, against the unrotated one gives s = (n_sectors - j) mod n_sectors. The query's pose guess from entry i is
 *   T_i Rz(s D), Rz = [c -s 0; s c 0; 0 0 1] from std::cos / std::sin of yaw = s D:
 *   guess[r][c] = (T_i[r][0] Rz[0][c] + T_i[r][1] Rz[1][c]) + T_i[r][2] Rz[2][c] for c < 3, guess[r][3] = T_i[r][3].
 * Candidates: the searched entries by (distance ascending, entry ascending); walking that order an entry is taken unless
 *   its keyframe's xy is closer than `separation` to a candidate already taken (0 takes everything); at most top_k
 *   (1..256). max_entry < 0 searches every entry, otherwise entries [0, min(max_entry, N)) (a loop-closure query:
 *   only entries older than the recent ones); an empty range is KB_ERR_INVALID_ARG.
 * Every argument that needs no handle is checked first; without a device the calls then return KB_ERR_NO_DEVICE. A
 * non-finite point is KB_ERR_INVALID_ARG, a pose outside SE(3) KB_ERR_NOT_SE3. On error nothing is written. */
typedef struct kb_place_params {
    int n_rings, n_sectors;
    double max_radius, z_offset;
} kb_place_params;
void kb_place_params_default(kb_place_params *p); /* 20, 60, 80.0, 2.0; needs no device */
typedef struct kb_place_db kb_place_db;
/* a database on the calling thread's device (kb_set_device) */
int kb_place_db_create(const kb_place_params *p, kb_place_db **out);
int kb_place_db_destroy(kb_place_db *db);
int kb_place_db_size(const kb_place_db *db, size_t *out);
/* the descriptor of xyz[n] into out[n_rings][n_sectors]; nothing is added. n = 0 gives zeros. */
int kb_place_descriptor(kb_place_db *db, const double *xyz, size_t n, double *out);
/* append the descriptor of xyz[n] (the cloud in its sensor frame) with the keyframe pose (row-major SE(3)); *index (may
 * be NULL) = its entry. At most 2^24 entries. Earlier entries are unchanged when the storage grows. */
int kb_place_db_add(kb_place_db *db, const double *xyz, size_t n, const double pose[16], size_t *index);
/* two-call like kb_map_pointcloud: *n_out = N; descriptors (double[N][n_rings][n_sectors]) and poses (double[N][16])
 * both NULL or cap 0 only query it; cap < N is KB_ERR_CAPACITY, with *n_out = N written (the one output written on that
 * error) and nothing else. Either array may be NULL when cap >= N. */
int kb_place_db_dump(const kb_place_db *db, double *descriptors, double *poses, size_t cap, size_t *n_out);
/* replace the entries by n dumped ones, all or nothing: KB_ERR_INVALID_ARG for a negative or non-finite descriptor value
 * or n > 2^24, KB_ERR_NOT_SE3 for a pose outside SE(3); the database is unchanged on error */
int kb_place_db_load(kb_place_db *db, const double *descriptors, const double *poses, size_t n);
typedef struct kb_place_match {
    int entry, shift;
    double yaw, distance; /* yaw = shift 2 pi / n_sectors */
    double guess[16];     /* T_entry Rz(yaw), row-major */
} kb_place_match;
/* the candidates of the query cloud xyz[n] into out[top_k], *n_out = their count. entry_distances / entry_shifts (may be
 * NULL) receive every searched entry's distance and shift, in entry order. */
int kb_place_query(kb_place_db *db, const double *xyz, size_t n, int max_entry, double separation, int top_k,
                   kb_place_match *out, size_t *n_out, double *entry_distances, int *entry_shifts);
typedef struct kb_place_match_report {
    size_t queries, entries; /* Q, and the entries of db */
    size_t pairs;            /* (query, entry) pairs searched: the sum of the queries' ranges */
    size_t fallbacks;        /* queries whose walk read back their whole row */
    size_t chunks;           /* device passes: the queries are split so that a chunk's pairs stay within a fixed budget */
} kb_place_match_report;
/* Every entry of `queries` (Q of them, its unit columns and masks; `queries` may be db itself) as a query of db:
 * out[q][top_k] and n_out[q] are, bit for bit, the matches kb_place_query gives for the cloud entry q was added from
 * (entry, shift, yaw, distance, guess), with the same max_entry, separation and top_k. max_entry (int[Q], may be NULL:
 * every entry): max_entry[q] < 0 searches every entry, otherwise [0, min(max_entry[q], N)); an empty range gives
 * n_out[q] = 0 (unlike kb_place_query, it fails no call). Q = 0 does nothing.
 * On the device every (query, entry) pair's distance and shift are computed as kb_place_query computes them, and each
 * query's pairs are sorted by (distance, entry); the first 8 top_k of them (all, when fewer) are read back and walked
 * as kb_place_query walks its entries. A query whose walk uses them up with fewer than top_k matches while entries
 * remain reads back its whole row and walks that (report->fallbacks). report (may be NULL) receives the counts.
 * KB_ERR_INVALID_ARG for top_k outside [1, 256], a separation that is negative or not finite, NULL out, n_out, db or
 * queries, databases of different place parameters or on different devices; every check is made before any device
 * work, and on error nothing is written. */
int kb_place_db_match(kb_place_db *db, const kb_place_db *queries, const int *max_entry, double separation, int top_k,
                      kb_place_match *out, int *n_out, kb_place_match_report *report);
typedef struct kb_place_search {
    int top_k, max_entry;   /* as kb_place_query */
    double separation;      /* metres, >= 0: of the candidate walk and of the runner-up */
    double max_correspondence_distance, kernel_scale; /* of the refinement */
} kb_place_search;
typedef struct kb_place_result {
    double pose[16];  /* the winner, refined, row-major */
    int inliers, iterations, rank; /* its inliers, ICP iterations and index among the candidates */
    int n_source, n_entries, n_candidates;  /* source points, entries searched, candidates refined */
    double runner_up_pose[16];  /* all zero when there is no runner-up */
    int runner_up_inliers;      /* -1 when there is none */
} kb_place_result;
/* Relocalize without any pose: the candidates of the descriptor cloud desc_xyz[n_desc] (kb_place_query with s's top_k,
 * max_entry and separation), then kb_registration_align_batch of the source src_xyz[n_src] from every candidate's guess
 * with s's thresholds, inliers on: each refined pose, iteration count and inlier count is bit for bit that call's.
 * Winner: the most inliers, ties to the lower rank. Runner-up: the best other candidate whose refined pose is farther
 * from the winner's than `separation` in xy or 2 sector widths in rotation angle (the rule of kb_relocalize).
 * candidates (kb_place_match[top_k], may be NULL) receives the first n_candidates matches. db, map and reg must be on
 * one device. Only reads the map: allowed while localizers hold it. KB_ERR_INVALID_ARG as kb_place_query, for n_src = 0
 * and for an empty map. */
int kb_place_relocalize(kb_registration *reg, kb_place_db *db, const double *desc_xyz, size_t n_desc,
                        const double *src_xyz, size_t n_src, const kb_map *map, const kb_place_search *s,
                        kb_place_result *out, kb_place_match *candidates);

/* ---- pose graph: loop closure --------------------------------------------------------------------------------------
 * No reference counterpart. Nodes are poses T_i (row-major SE(3)); a fixed node does not move. An edge
 * e = (i, j, Z, Omega, c) has the residual r_e = Log(Z^-1 T_i^-1 T_j) in R^6, in the tangent order (translation,
 * rotation) of the library, s_e = r_e^T Omega r_e, and the cost F = 1/2 (sum_e rho_e(s_e) + sum_p rho_p(s_p)) with
 * rho(s) = s for c = 0 and the Cauchy loss rho(s) = c^2 log(1 + s / c^2) for c > 0; w_e = rho'(s_e).
 * A prior p is a unary factor on one node k, with its own Omega and Cauchy scale c, s_p = r_p^T Omega r_p and
 * w_p = rho'(s_p) as for edges. Two kinds (kb_pose_graph_add_pose_prior, kb_pose_graph_add_position_prior):
 *   pose prior (k, Z, Omega 6x6, c): r_p = Log(Z^-1 T_k), dr/dd_k = J_r^-1(r_p);
 *   position prior (k, p, lever arm l in the body frame, Omega 3x3 in the world frame, c): r_p = R_k l + t_k - p in
 *   R^3, dr/dd_k = [R_k, -R_k [l]x], e.g. a GNSS antenna l away from the body origin.
 * A prior adds only to its node's diagonal block and gradient, after the node's edges (and nothing on a fixed node, whose
 * prior adds a constant to F). The gauge: every connected component of free nodes must hold a fixed node or a node with
 * a prior, so a graph with priors needs no fixed node. Position priors fix a component's rotation only through at least
 * 3 non-collinear antenna positions; on fewer, the damped steps still solve, but kb_pose_graph_marginals reports H as
 * not positive definite. A graph without priors computes exactly what it computed before priors existed.
 * kb_pose_graph_optimize moves the free nodes by right perturbation, T_i <- T_i Exp(d_i), with Levenberg-Marquardt on
 * IRLS weights and exact Jacobians (dr/dd_j = J_r^-1(r), dr/dd_i = -J_r^-1(r) Ad(T_j^-1 T_i)):
 *   H = sum J^T w Omega J, g = sum J^T w Omega r over the free nodes (edges, then priors); (H + lambda diag H) d = -g
 *   is solved by PCG
 *   preconditioned by the exact inverse of M, the block-tridiagonal part of the damped system (the edges with
 *   |i - j| = 1 in full, every other edge's two diagonal blocks, the damping), which block cyclic reduction factors once
 *   per step. PCG stops at |r_k| <= cg_tolerance |g| or after max_cg_iterations.
 *   An accepted step (lower F) divides lambda by 10, a rejected one (including a non-finite F) multiplies it by 10.
 *   Stop: an accepted step lowers F by at most function_tolerance F; max |d| <= parameter_tolerance; lambda > 1e12; or
 *   max_iterations steps (accepted and rejected both count).
 * One cooperative launch per call, on the graph's device and stream. The results are bit-identical from run to run for a
 * given grid size (kb_set_grid_blocks caps it at optimize time): every sum is formed in a fixed order.
 * The graph lives on the host. Its device buffers are allocated at the first optimize on the device and stream the
 * creating thread had selected (kb_set_device / kb_set_stream), kept for later calls and released by destroy. Nodes and
 * edges may be added after an optimize; the next one starts from the current poses.
 * Every argument is checked before any work and nothing is written on error: KB_ERR_NOT_SE3 for a pose or measurement
 * outside SE(3) (non-finite included); KB_ERR_INVALID_ARG for a NULL argument, i == j, a node that does not exist,
 * information that is not exactly symmetric, not finite or not positive definite, a negative or non-finite
 * robust_scale, more than 2^22 nodes, 2^24 edges or 2^24 priors, a non-finite prior position or lever arm, options out
 * of range, and at optimize a free node that no path of edges connects to a fixed node or a prior. Without a device,
 * optimize returns KB_ERR_NO_DEVICE after these checks. */
typedef struct kb_pose_graph kb_pose_graph;
int kb_pose_graph_create(kb_pose_graph **out); /* host-side; needs no device */
int kb_pose_graph_destroy(kb_pose_graph *g);
/* *index (may be NULL) = the new node's index */
int kb_pose_graph_add_node(kb_pose_graph *g, const double pose[16], int fixed, size_t *index);
/* information: row-major 6x6 in the tangent order; robust_scale: c (0 = squared loss). *index may be NULL. */
int kb_pose_graph_add_edge(kb_pose_graph *g, size_t i, size_t j, const double measurement[16],
                           const double information[36], double robust_scale, size_t *index);
/* Priors of both kinds share one index space, in the order they are added; *index (may be NULL) = the new prior's.
 * pose: row-major SE(3) Z; information: row-major 6x6 in the tangent order; robust_scale: c (0 = squared loss). */
int kb_pose_graph_add_pose_prior(kb_pose_graph *g, size_t k, const double pose[16], const double information[36],
                                 double robust_scale, size_t *index);
/* position: p in the world frame; lever_arm: l in node k's body frame; information: row-major 3x3 in the world frame */
int kb_pose_graph_add_position_prior(kb_pose_graph *g, size_t k, const double position[3], const double lever_arm[3],
                                     const double information[9], double robust_scale, size_t *index);
int kb_pose_graph_num_priors(const kb_pose_graph *g, size_t *n);
/* s_p and w_p of every prior at the graph's current poses; host-side, needs no device. Two-call: *n_out = P; chi2 and
 * weight (double[P], either may be NULL) both NULL or cap 0 only queries it, cap < P is KB_ERR_CAPACITY (with *n_out) */
int kb_pose_graph_prior_chi2(const kb_pose_graph *g, double *chi2, double *weight, size_t cap, size_t *n_out);
int kb_pose_graph_size(const kb_pose_graph *g, size_t *n_nodes, size_t *n_edges);
/* two-call: *n_out = N; poses (double[N][16]) NULL or cap 0 only queries it, cap < N is KB_ERR_CAPACITY (with *n_out) */
int kb_pose_graph_poses(const kb_pose_graph *g, double *poses, size_t cap, size_t *n_out);
typedef struct kb_pose_graph_options {
    int max_iterations;          /* [0, 10^6] */
    double function_tolerance;   /* >= 0 */
    double parameter_tolerance;  /* >= 0 */
    double initial_lambda;       /* (0, 1e12] */
    int max_cg_iterations;       /* [1, 10^6] */
    double cg_tolerance;         /* [0, 1) */
} kb_pose_graph_options;
/* 100, 1e-12, 1e-10, 1e-4, 100, 1e-10; needs no device */
void kb_pose_graph_options_default(kb_pose_graph_options *o);
enum { KB_PG_FUNCTION_TOLERANCE = 0, KB_PG_PARAMETER_TOLERANCE = 1, KB_PG_MAX_ITERATIONS = 2, KB_PG_NO_DECREASE = 3 };
typedef struct kb_pose_graph_report {
    int iterations, accepted, cg_iterations; /* LM steps (accepted and rejected), accepted ones, PCG iterations in all */
    int termination;                         /* KB_PG_* */
    double initial_cost, final_cost, lambda; /* F at the start and at the returned poses, the last lambda */
} kb_pose_graph_report;
/* o may be NULL (the defaults). edge_chi2 / edge_weight (double[E], may be NULL) receive s_e and w_e at the returned
 * poses. */
int kb_pose_graph_optimize(kb_pose_graph *g, const kb_pose_graph_options *o, kb_pose_graph_report *out,
                           double *edge_chi2, double *edge_weight);
/* The same problem and the same Levenberg-Marquardt as kb_pose_graph_optimize (cost, IRLS weights, exact Jacobians,
 * right perturbation, lambda schedule, the four stopping rules and their order, fixed nodes returned bit for bit), with
 * every step solved exactly: (H + lambda diag H) d = -g by P L L^T P^T, the sparse block Cholesky factorization of
 * kb_pose_graph_marginals applied to the damped system (its symbolic analysis; damping changes only diagonal blocks),
 * then a forward and a backward block substitution. A pivot that is not positive and finite rejects the step like a
 * non-finite F (lambda x 10); it is not an error. Each step is one factorization; report.iterations counts them and
 * report.cg_iterations is 0. max_cg_iterations and cg_tolerance are checked as by kb_pose_graph_optimize and otherwise
 * ignored.
 * Where it pays: on graphs with loops, whose edges reach far back in node index, PCG's block-tridiagonal preconditioner
 * covers little of H and a step takes many PCG iterations; the exact step takes one factorization. On a pure chain PCG
 * is exact in one iteration and needs fewer grid barriers.
 * One cooperative launch per call. The results are bit-identical from run to run and for every grid size: the factor
 * and the solves are formed in a fixed order, and the cost is summed over fixed chunks of factors (the edges, then the
 * priors), then the chunks in index order. The symbolic analysis stays cached for the graph's size; the numeric factor the call leaves behind is of
 * the damped system, so the next kb_pose_graph_marginals factors H again at the new poses. kb_debug_pose_graph_ms
 * times this call's launch as it times kb_pose_graph_optimize's.
 * Checked before any work, in the order of kb_pose_graph_optimize and with its codes, writing nothing on error; in
 * addition KB_ERR_INVALID_ARG for a graph whose factorization needs more than 2^30 block updates (as the marginals).
 * Without a device, KB_ERR_NO_DEVICE after these checks. */
int kb_pose_graph_optimize_direct(kb_pose_graph *g, const kb_pose_graph_options *o, kb_pose_graph_report *out,
                                  double *edge_chi2, double *edge_weight);

/* ---- pose graph: marginal covariances -------------------------------------------------------------------------------
 * How well each pose is known, at the graph's current poses (as added, or as the last optimize left them):
 *   H = sum_e J_e^T w_e Omega_e J_e over the free nodes, with the optimizer's exact Jacobians
 *   (dr/dd_j = J_r^-1(r), dr/dd_i = -J_r^-1(r) Ad(T_j^-1 T_i)) and w_e = rho'(s_e) at those poses; no damping. An edge
 *   with one fixed node adds only the free node's diagonal block, an edge between two fixed nodes nothing; parallel
 *   edges between one pair add up in ascending edge order. Priors add J^T w Omega J to their free node's diagonal
 *   block, after its edges.
 *   Sigma = H^-1, in the tangent space of the right perturbation T_k Exp(d_k), order (translation, rotation). A fixed
 *   node's rows and columns are exactly 0.
 * Sigma is the Gauss-Newton (Laplace) approximation at those poses. It is not rescaled by the residuals: Omega is taken
 * as the measurement's true information.
 * Method: H = P L L^T P^T, a sparse block Cholesky factorization with a nested-dissection order P (George), computed on
 * the device (one cooperative launch); Sigma_ij = sum_m X_i[m]^T X_j[m] with X_k = L^-1 P^T E_k, which is non-zero only
 * on the elimination-tree path from k's column to its root, summed over the common part of the two paths (Sigma_ij = 0
 * when the two lie in different trees). Every value is formed by one thread in a fixed order: the results are
 * bit-identical from run to run and for every grid size, and a diagonal block is exactly symmetric.
 * The symbolic analysis is cached for the graph's size, the numeric factor until the next add_node, add_edge,
 * add_*_prior or optimize; neither changes what optimize computes.
 * Checked before any device work, writing nothing on error: KB_ERR_INVALID_ARG for NULL with n > 0, a node that does
 * not exist, a free node that no path of edges connects to a fixed node or a prior, and (after the factorization) an H
 * that is not positive definite at the current poses; then KB_ERR_NO_DEVICE without a device. n == 0 does nothing. */
/* cov: double[n][36], the row-major 6x6 Sigma_kk of each nodes[t] */
int kb_pose_graph_marginals(kb_pose_graph *g, const size_t *nodes, size_t n, double *cov);
/* pairs: size_t[n][2]; cov: double[n][144], the row-major 12x12 [[Sigma_ii, Sigma_ij], [Sigma_ji, Sigma_jj]] of each
 * pair (any pair: i == j, and nodes that share no edge) */
int kb_pose_graph_joint_marginals(kb_pose_graph *g, const size_t *pairs, size_t n, double *cov);
struct kb_pose_graph_factor_info {
    size_t free_nodes;
    size_t h_blocks;      /* 6x6 blocks of H's lower triangle, diagonal included */
    size_t l_blocks;      /* 6x6 blocks of L, diagonal included */
    size_t etree_height;  /* columns on the longest leaf-to-root path of the elimination tree */
    double flops;         /* of one numeric factorization: 2*6^3 per block update, 6^3 per block solve, 6^3/3 per pivot */
};
/* the symbolic analysis of the graph as it is now; host-side, needs no device (the struct shares the function's
 * name: C and C++ refer to it as struct kb_pose_graph_factor_info) */
int kb_pose_graph_factor_info(kb_pose_graph *g, struct kb_pose_graph_factor_info *out);

/* ---- pose graph: adjustment to the planes of the map ----------------------------------------------------------------
 * No reference counterpart. After loop closure the graph fits its edges, but each edge summarises a pair of keyframes by
 * one measurement; this call aligns every keyframe's points with the planes the other keyframes' points form.
 * Inputs: the graph's N nodes T_k and, per node, a cloud P_k of n_k >= 0 points p in the node's body frame, the clouds
 * concatenated in node order: xyz[offsets[k] .. offsets[k + 1]) (offsets[N + 1], offsets[0] = 0, offsets[N] = n_points).
 * Parameters: voxel size s, min_points m, planarity rho, point sigma [m], Cauchy scale c (in units of sigma; 0: squared
 * loss), rounds R, round_tolerance.
 * A round:
 *   1. Planes from the others. Every point goes to the world frame at the current poses, q = T_k p, and into the voxel
 *      floor(q / s) (the map's point_to_voxel). For each pair (voxel v, node k) of a free node k with points in v, the
 *      points of v from all other nodes (fixed ones included) give the pair's plane, leave-one-out so that a keyframe is
 *      never pulled toward itself: the pair counts when there are at least m of them and the eigenvalues of their
 *      covariance (1/count) satisfy lambda_0 <= rho lambda_1 with lambda_1 > 0; its plane is n = the unit eigenvector of
 *      lambda_0 and d = n^T c_bar (c_bar their mean). The moments are summed about the voxel's centre, per voxel and
 *      per (voxel, node), and the leave-one-out moments are (the voxel's) - (the node's own).
 *   2. Terms. Each point p of a free node k in a planar pair (v, k): r = n^T (T_k p) - d, s = r^2 / sigma^2, the cost
 *      1/2 rho_c(s) (the edges' loss), the IRLS weight w = rho_c'(s), dr/dd_k = n^T R_k [I | -[p]x] (the graph's right
 *      perturbation and tangent order). F = F_graph (edges and priors, unchanged) + 1/2 sum_points rho_c(s).
 *   3. Levenberg-Marquardt with the planes held: kb_pose_graph_optimize_direct's loop and exact solve (options as
 *      there), where H_kk gains sum J^T (w / sigma^2) J and g_k gains sum J^T (w / sigma^2) r, the damping is lambda diag
 *      of the whole block, and every cost includes the plane terms. The plane terms touch diagonal blocks only, so the
 *      symbolic analysis of the marginals is reused as it is.
 * The rounds stop after R, when a round moves no node by more than round_tolerance (max |Log(T_before^-1 T_after)| over
 * the free nodes, the largest component), or after a round without a planar pair: that round was exactly
 * kb_pose_graph_optimize_direct (same poses and report, bit for bit), and another would only repeat it.
 * The poses are written back into the graph as optimize writes them (fixed nodes untouched). The edges, priors and
 * marginals keep their meaning: kb_pose_graph_marginals afterwards is of the graph's edges and priors alone, at the new
 * poses (the cached factor is dropped).
 * Determinism: no floating-point atomics; every sum is formed in a fixed order (a voxel's points are sorted stably by
 * voxel key and summed per node in input order, the nodes in index order; the terms over fixed chunks of a node's
 * points, folded in chunk order). The results are bit-identical from run to run and for every kb_set_grid_blocks.
 * The points are uploaded once per call into buffers the graph owns; they grow as needed and are released by destroy.
 * Checked before any device work, writing nothing on error (KB_ERR_INVALID_ARG): NULL g, p, or xyz / offsets where
 * needed; a non-finite coordinate; offsets that do not rise monotonically from 0 to n_points, or n_points >= 2^31; a
 * point whose voxel coordinate at the current poses lies outside [-2^19, 2^19) (half the packed key's range, so that
 * the rounds cannot leave it); parameters out of range (below); the options as kb_pose_graph_optimize; the gauge as
 * kb_pose_graph_optimize (plane terms do not connect nodes); rounds_out with rounds_cap < p->rounds; a graph whose
 * factorization needs more than 2^30 block updates. Then KB_ERR_NO_DEVICE without a device. */
typedef struct kb_plane_adjust_params {
    double voxel_size;       /* s > 0 */
    int min_points;          /* m >= 3 */
    double planarity;        /* rho in [0, 1] */
    double sigma;            /* > 0 [m] */
    double robust_scale;     /* c >= 0 (units of sigma) */
    int rounds;              /* R in [1, 1000] */
    double round_tolerance;  /* >= 0 */
} kb_plane_adjust_params;
/* voxel_size s, min_points 5, planarity 0.1, sigma 0.2 s, robust_scale 3, rounds 20, round_tolerance 1e-4 (DESIGN.md
 * §4.21 has the measurements behind them); needs no device */
void kb_plane_adjust_params_default(kb_plane_adjust_params *p, double voxel_size);
typedef struct kb_plane_round {
    unsigned long long planar_pairs;     /* (voxel, free node) pairs with a plane */
    unsigned long long points_used;      /* points with a plane */
    double initial_cost, final_cost;     /* F (graph + planes) at the round's start and end, with its planes */
    double final_plane_cost;             /* the plane part of final_cost */
    int iterations, accepted;            /* LM steps, accepted steps */
    int termination;                     /* KB_PG_* */
    double max_change;                   /* max |Log(T_before^-1 T_after)| over the nodes */
} kb_plane_round;
typedef struct kb_plane_adjust_report {
    int rounds;                          /* rounds run */
    int converged;                       /* 1: stopped by round_tolerance or a round without a planar pair */
    double initial_cost, final_cost;     /* of the first round's start and the last round's end */
} kb_plane_adjust_report;
/* report (may be NULL); rounds_out (kb_plane_round[rounds_cap], may be NULL) receives each round's record; node_rms and
 * node_points (double[N] / unsigned long long[N], may be NULL) receive each node's RMS point-to-plane residual [m] and
 * points with a plane at the returned poses with the last round's planes (0 and 0 for a node without any). o may be
 * NULL (the defaults). */
int kb_pose_graph_adjust_planes(kb_pose_graph *g, const double *xyz, size_t n_points, const size_t *offsets,
                                const kb_plane_adjust_params *p, const kb_pose_graph_options *o,
                                kb_plane_adjust_report *report, kb_plane_round *rounds_out, size_t rounds_cap,
                                double *node_rms, unsigned long long *node_points);

/* ---- free space: removing moving objects from a map ----------------------------------------------------------------
 * No reference counterpart. A map keeps everything the sensor ever hit, including a car that drove past or was parked
 * and left. The scans of a run that saw through such a place are evidence that it is free; this call counts that
 * evidence for every map point and removes the points it outweighs.
 * Inputs: a map and S scans; scan s is points p in its sensor frame and a pose T_s (world <- sensor, row-major SE(3)).
 * Rays: each point gives a ray from o = t_s to e = T_s p, computed exactly as kb_map_update_pose transforms points (the
 *   same device function); L = |e - o|, d = (e - o) / L, each component divided by L.
 * Planes: a voxel is planar when it holds m >= 3 points and its planarity a >= min_planarity, with the mean, the
 *   covariance C (1/m), n (the unit eigenvector of C's smallest eigenvalue) and a = (l1 - l0) / l2 (0 when l2 = 0) of the
 *   plane constraints above.
 * Passes, per map point m: a ray passes m when all of these hold (rays with L = 0 pass nothing):
 *   1. u = (m - o).d lies in [0, L - end_margin];
 *   2. r = |m - o - u d| <= pass_radius;
 *   3. if m's voxel is planar, |n.d| >= sin(min_incidence).
 *   Rule 3 keeps the ground and walls: a ray that ends on m's own plane at least end_margin beyond m, at an angle alpha to
 *   that plane, has r >= end_margin sin(alpha) at m. So when sin(min_incidence) > pass_radius / end_margin, a planar
 *   surface is never passed by the rays that graze it; only rays steeper than min_incidence can pass its points, and
 *   those end far from it. The defaults meet this condition with a factor of 2 for noise.
 * Hits, per map voxel V: the rays whose endpoint e falls in V (the hot path's FP64 point_to_voxel; a zero-length ray
 *   too). Hits protect thin static objects (poles, box edges): rays skim past their edges, but every scan that sees them
 *   ends many rays in their voxels.
 * Removed: a map point m is removed when passes(m) >= min_passes and passes(m) >= ratio * hits(V(m)) (in double).
 * Parameters are checked on the host before any device call: KB_ERR_INVALID_ARG for a non-finite value,
 * pass_radius <= 0, end_margin < 0, min_incidence outside [0, pi/2], min_planarity outside [0, 1], min_passes = 0 or
 * ratio < 0. */
typedef struct kb_free_space_params {
    double pass_radius;    /* epsilon [m] */
    double end_margin;     /* delta [m] */
    double min_incidence;  /* theta_min [rad] */
    double min_planarity;  /* a_min */
    unsigned min_passes;
    double ratio;
} kb_free_space_params;
/* pass_radius 0.1 v, end_margin 2.0 v, min_incidence asin(2 pass_radius / end_margin), min_planarity 0.3, min_passes 20,
 * ratio 0.1 for voxel size v (chosen from measurements: DESIGN.md §4.13); needs no device */
void kb_free_space_params_default(kb_free_space_params *p, double voxel_size);
typedef struct kb_free_space_report {
    unsigned long long rays, scans;                   /* the input */
    unsigned long long points, voxels;                /* of the map */
    unsigned long long points_removed, voxels_removed; /* voxels that lose every point */
    unsigned long long ray_point_tests;               /* (ray, point) pairs the counting tested exactly */
} kb_free_space_report;
/* Count the free-space evidence of scans xyz[offset[s] .. offset[s + 1]) at poses[s][16] (s < n_scans) for map.
 * passes (unsigned[kb_map_num_points]) and hits (unsigned[kb_map_num_voxels]) may each be NULL; both are in dump order
 * (kb_map_dump: voxels ascending, points in per-voxel insertion order). out, when not NULL, receives the kept points
 * through kb_map_load_dev's path, in per-voxel insertion order; voxels that lose every point disappear. out must be
 * another map with map's voxel_size and max_points_per_voxel, on map's device, that no localizer reads; else
 * KB_ERR_INVALID_ARG and nothing changes. report may be NULL.
 * map is only read: the call works while localizers read it. Device memory is bounded by the map and the largest chunk
 * of scans (up to 2^22 rays, or one larger scan), not by n_scans. The counts are integers: they do not depend on
 * kb_set_grid_blocks, the ray bin size, the order of the scans or how they are split over calls (two calls over a
 * split of the scans sum to one call's counts).
 * Every argument is checked before any work and nothing is written on error: KB_ERR_INVALID_ARG for the parameters
 * above, NULL p, NULL xyz / offset / poses where needed, an offset that is not a non-decreasing partition of
 * [0, n_points], a non-finite point, an endpoint whose voxel coordinate would not fit in an int, or n_points >= 2^32;
 * KB_ERR_NOT_SE3 for a pose outside SE(3). Without a device the call then returns KB_ERR_NO_DEVICE; a NULL map is
 * KB_ERR_INVALID_ARG after that. */
int kb_map_free_space(const kb_map *map, const double *xyz, size_t n_points, const size_t *offset, size_t n_scans,
                      const double *poses, const kb_free_space_params *p, unsigned *passes, unsigned *hits, kb_map *out,
                      kb_free_space_report *report);

#ifdef __cplusplus
}
#endif
#endif /* KISS_ICP_B200_H */
