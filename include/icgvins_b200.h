/*
 * icgvins_b200.h -- C ABI of libicgvins_b200.so: H100-native (sm_90a) replacements for the two compute hot paths
 * of i2Nav-WHU/IC-GVINS.  Plain pointers and sizes only; no C++ / torch / OpenCV / Ceres types cross this boundary.
 *
 * Every entry point names the reference interface it replaces (paths relative to the reference checkout,
 * IG/ = ic_gvins/ic_gvins/).  The reference has no FFI of its own: the seams are direct library calls into
 * OpenCV (front end) and Ceres (window solve); INTEGRATION.md shows the shim a maintainer adds at each call site.
 *
 * Conventions
 *   - All functions return 0 on success, a negative ICG_E* code on failure (no exceptions, no aborts).
 *   - "host" pointers are ordinary process memory; "dev" pointers are CUDA device memory of the handle's device.
 *   - A handle is bound to one CUDA device and one stream and is NOT re-entrant (the reference calls each seam
 *     from a single thread: tracking thread IG/ic_gvins.cc:535, optimization thread IG/ic_gvins.cc:434-448).
 *   - Points are interleaved float (x, y) pairs == std::vector<cv::Point2f>::data().
 *   - There is NO CPU fallback: without a CUDA device every create() fails with ICG_ENODEVICE.
 */
#ifndef ICGVINS_B200_H
#define ICGVINS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ICG_OK 0
#define ICG_EINVAL (-1)     /* bad argument */
#define ICG_ENODEVICE (-2)  /* no usable CUDA device / driver */
#define ICG_ECUDA (-3)      /* CUDA runtime error (see icg_last_error) */
#define ICG_EUNSUPPORTED (-4) /* parameter combination the sm_90a kernels are not built for */
#define ICG_ENOMEM (-5)

#define ICG_OPTFLOW_USE_INITIAL_FLOW 4 /* == cv::OPTFLOW_USE_INITIAL_FLOW */

const char *icg_last_error(void);
int icg_version(void);
/* number of kernels launched by this library in this process since load / last reset (bench "gpu_launches") */
uint64_t icg_launch_count(void);
void icg_launch_count_reset(void);

/* ===================================================================================================== *
 *  Path A: pyramidal KLT front end
 * ===================================================================================================== */
typedef struct icg_klt icg_klt;

/*
 * Create a tracker for width x height u8 images.  n_slots device-resident image slots (each holds a 4-level
 * pyramid, levels 0..3 as cv::buildOpticalFlowPyramid(img, winSize 21, maxLevel 3) produces them);
 * max_points = largest n of one call.  stream may be NULL (handle creates its own) or a cudaStream_t.
 */
int icg_klt_create(icg_klt **h, int width, int height, int n_slots, int max_points, int device, void *stream);
void icg_klt_destroy(icg_klt *h);

/*
 * Drop-in for cv::calcOpticalFlowPyrLK as the reference calls it (IG/tracking/tracking.cc:385,390,487,493):
 *   cv::calcOpticalFlowPyrLK(prev, next, prevPts, nextPts, status, err, Size(win,win), max_level,
 *                            TermCriteria(COUNT+EPS, max_iter, eps), flags)
 * Host buffers, synchronous.  next_xy is in/out (initial flow when flags has ICG_OPTFLOW_USE_INITIAL_FLOW).
 * err may be NULL (the reference never reads it).  Only win == 21 and max_level <= 3 are built
 * (the values at all four call sites); anything else returns ICG_EUNSUPPORTED.
 * Pyramids are cached per image content (the reference passes the same two images to 4 calls per frame).
 */
int icg_klt_calc_optical_flow_pyr_lk(icg_klt *h, const uint8_t *prev, const uint8_t *next, int stride,
                                     const float *prev_xy, float *next_xy, uint8_t *status, float *err, int n,
                                     int win, int max_level, int max_iter, double eps, int flags);

/*
 * Fused replacement for the forward LK + backward LK + gate block (IG/tracking/tracking.cc:385-403 and :487-506):
 *   status[k] = st_fwd && st_bwd && !isOnBorder(fwd) && ptsDistance(bwd, prev) < 0.5
 * next_xy in: predicted positions, out: forward result.  back_xy (may be NULL) receives the backward result.
 */
int icg_klt_track_fb(icg_klt *h, const uint8_t *prev, const uint8_t *next, int stride, const float *prev_xy,
                     float *next_xy, float *back_xy, uint8_t *status, int n);

/* ---- device-resident / batched API (throughput mode: many independent streams per GPU) ---- */

/* async H2D of one frame into slot's level 0 (host memory should be pinned for overlap) + pyramid build */
int icg_klt_upload(icg_klt *h, int slot, const uint8_t *host_img, int stride);
/* async H2D of one frame into slot's level 0 only (no pyramid build; pair with icg_klt_build_pyramids) */
int icg_klt_upload_level0(icg_klt *h, int slot, const uint8_t *host_img, int stride);
/* async H2D of `count` frames into the level-0 planes of slots [first_slot, first_slot + count) in one call (throughput mode: one new frame
 * of every stream per step): linear DMA copies into a device staging buffer + one scatter kernel; no pyramid build
 * (pair with icg_klt_build_pyramids).  host_imgs[k] should be pinned. */
int icg_klt_upload_batch(icg_klt *h, int first_slot, int count, const uint8_t *const *host_imgs, int stride);
/* synchronous D2H of one pyramid level of a slot into a host buffer of row stride `stride` (parity tests) */
int icg_klt_download_level(icg_klt *h, int slot, int level, uint8_t *host_img, int stride);
/* device pointer + pitch of a slot's level-0 plane, so a producer on the same device can write frames in place */
int icg_klt_slot_level0(icg_klt *h, int slot, void **dev_ptr, int *pitch);
/* device pointer + pitch + size of level `level` (read-back for parity tests) */
int icg_klt_slot_level(icg_klt *h, int slot, int level, void **dev_ptr, int *pitch, int *w, int *hgt);
/* build levels 1..3 for slots [first, first+count) from their level-0 planes (one launch) */
int icg_klt_build_pyramids(icg_klt *h, int first_slot, int count);
/*
 * Batched forward+backward tracking of n_total points, all arrays in DEVICE memory:
 *   slots[2k], slots[2k+1] = (prev slot, next slot) of point k;  prev_xy/init_xy/fwd_xy/bwd_xy: float2 per point.
 * Asynchronous on the handle's stream.  mode 0: forward only (status = raw LK status);
 * mode 1: fused forward+backward+gates (as icg_klt_track_fb).  Tracks on the pyramid levels cv::buildOpticalFlowPyramid(winSize 21,
 * maxLevel 3) builds for the handle's size: it stops at the first level whose width or height is <= 21 (e.g. 320x168: 3 levels, 32x32: 1).
 */
int icg_klt_track_batch_dev(icg_klt *h, int n_total, const int32_t *dev_slots, const float *dev_prev_xy,
                            const float *dev_init_xy, float *dev_fwd_xy, float *dev_bwd_xy, uint8_t *dev_status,
                            int mode);
int icg_klt_sync(icg_klt *h);

/* ----- camera model of path A (SURVEY 8a row A6): HOST functions by design (<= 300 points per frame, FP64) ----- */
typedef struct icg_camera {
    double fx, fy, cx, cy, skew; /* intrinsic_(0,0), (1,1), (0,2), (1,2), (0,1)   (IG/tracking/camera.cc:29-33) */
    double k1, k2, p1, p2, k3;   /* distortion_ in OpenCV order                    (:35-39) */
} icg_camera;
/* Camera::undistortPoints (IG/tracking/camera.cc:72-74) == cv::undistortPoints(pts, pts, K, D, Mat(), K); in place on n (x, y) floats */
int icg_camera_undistort_points(const icg_camera *c, float *pts_xy, int n);
/* Camera::distortPoints / distortPoint (:76-104): pixel2cam -> radtan -> cam2pixel, in place */
int icg_camera_distort_points(const icg_camera *c, float *pts_xy, int n);
/* Camera::distortCameraPoint (:106-120) for n camera-frame points (x, y, z) -> distorted pixels */
int icg_camera_distort_camera_points(const icg_camera *c, const double *pc_xyz, float *px_xy, int n);
/* Camera::pixel2cam (:126-130): pixels -> normalised camera points (x, y, 1) */
int icg_camera_pixel2cam(const icg_camera *c, const float *px_xy, double *cam_xyz, int n);
/* Camera::world2pixel (:144-146) = cam2pixel(R^T (pw - t)); R9 row-major body/camera attitude, t3 its position */
int icg_camera_world2pixel(const icg_camera *c, const double *R9, const double *t3, const double *pw_xyz, float *px_xy, int n);

/* Drop-in for cv::findFundamentalMat(pts1, pts2, cv::FM_RANSAC, threshold, confidence, status) as Tracking::trackReferenceFrame calls it
 * (IG/tracking/tracking.cc:547, maxIters = 1000): status[i] = 1 for the inliers of the best 7-point model; F9 (row-major, may be NULL)
 * receives that model.  HOST function in this round (<= 300 pairs, serially adaptive loop); the inlier mask is identical to OpenCV's
 * (tests/golden/fundamental_golden.npz).  n >= 15 as at the call site. */
int icg_find_fundamental_mat_ransac(const float *pts1_xy, const float *pts2_xy, int n, double threshold, double confidence, int max_iters,
                                    uint8_t *status, double *F9);

/* Tracking::triangulatePoint (IG/tracking/tracking.cc:796-808) for n point pairs: Tcw0 = n x (3 x 4 row-major T_c_w of the reference frames),
 * Tcw1 = the current frame's, pc0 / pc1 = normalised camera coordinates (x, y); pw = dehomogenised null vector of the 4 x 4 design matrix.
 * Host function. */
int icg_triangulate_points(const double *Tcw0, const double *Tcw1, const double *pc0_xy, const double *pc1_xy, int n, double *pw_xyz);

/* Tracking::calculateHistigram (IG/tracking/tracking.cc:88-104): the brightness statistic of the histogram gate in
 * Tracking::preprocessing (:115-133).  Host function (one pass over the frame). */
int icg_tracking_histogram(const uint8_t *img, int width, int height, int stride, double *out);

/* ----- SURVEY 8f ranks 2-4 on the DEVICE (csrc/geom.cu): the same functions as the host entry points above / icg_imu_preintegrate below, batched as
 * CUDA kernels (one __host__ __device__ definition of the arithmetic, csrc/geom_core.cuh).  Host buffers in / out, synchronous. ----- */
typedef struct icg_geom icg_geom;
int icg_geom_create(icg_geom **h, int device, void *stream);
void icg_geom_destroy(icg_geom *h);
/* Camera::undistortPoints / distortPoints (IG/tracking/camera.cc:72-104), thread per point, any n */
int icg_geom_undistort_points(icg_geom *h, const icg_camera *c, float *pts_xy, int n);
int icg_geom_distort_points(icg_geom *h, const icg_camera *c, float *pts_xy, int n);
/* cv::findFundamentalMat(FM_RANSAC) (IG/tracking/tracking.cc:547) on the device: a batch of one of icg_geom_find_fundamental_mat_ransac_batch
 * below (rounds of subsets drawn from the cv::RNG stream, solved and scored in parallel, OpenCV's serial acceptance rule and adaptive iteration
 * bound replayed per round).  Same inlier mask as icg_find_fundamental_mat_ransac / OpenCV. */
int icg_geom_find_fundamental_mat_ransac(icg_geom *h, const float *pts1_xy, const float *pts2_xy, int n, double threshold, double confidence, int max_iters,
                                         uint8_t *status, double *F9);
/* Tracking::triangulatePoint (IG/tracking/tracking.cc:796-808), thread per pair */
int icg_geom_triangulate_points(icg_geom *h, const double *Tcw0, const double *Tcw1, const double *pc0_xy, const double *pc1_xy, int n, double *pw_xyz);
/* icg_imu_preintegrate for n_intervals intervals at once (doReintegration over a window, IG/ic_gvins.cc:1680-1695; throughput mode): state16 is
 * n_intervals x 16, imu the concatenated sample rows, imu_off[k] .. imu_off[k+1] the rows of interval k (row imu_off[k] = the sample at its start);
 * iewn3 / gravity3 / noise5 shared; iewn3 == NULL: PreintegrationNormal.  blobs_out n_intervals x ICG_IMU_BLOB_DOUBLES, end_states10 may be NULL. */
int icg_geom_imu_preintegrate_batch(icg_geom *h, int n_intervals, const double *state16, const double *iewn3, const double *gravity3, const double *noise5,
                                    const double *imu, const int32_t *imu_off, double *blobs_out, double *end_states10);

/* Batched device version for S point sets (cv::findFundamentalMat(FM_RANSAC) per set, as icg_find_fundamental_mat_ransac: a fresh
 * cv::RNG(-1) per set, the subsets in stream order with the collinearity re-draws, 7-point models, OpenCV's serial acceptance rule and
 * adaptive iteration bound; n < 15 or no drawable subset: all-zero mask).  Set s = pairs set_off[s] .. set_off[s + 1] of the DEVICE arrays
 * dev_pts1_xy / dev_pts2_xy; set_off (n_sets + 1), threshold and confidence (n_sets each, NULL = 3 / 0.99) are HOST arrays.  Outputs in DEVICE
 * memory: dev_mask (one u8 per pair, at the pair's index), dev_n_inliers (n_sets), dev_F9 (9 per set, may be NULL), dev_stats (3 per set, may
 * be NULL: subsets drawn, clock64 cycles spent drawing them, cycles of the whole set).  One CTA per set; asynchronous on the handle's stream.
 * icg_geom_find_fundamental_mat_ransac is a batch of one. */
int icg_geom_find_fundamental_mat_ransac_batch(icg_geom *h, int n_sets, const int32_t *set_off, const float *dev_pts1_xy, const float *dev_pts2_xy,
                                               const double *threshold, const double *confidence, int max_iters, uint8_t *dev_mask,
                                               int32_t *dev_n_inliers, double *dev_F9, long long *dev_stats);

/* ----- Tracking::trackMappoint (IG/tracking/tracking.cc:351-455) + Tracking::trackReferenceFrame (:457-574) on the KLT handle (csrc/track.cu) ----- */
/* Per-stream parameters.  Attitudes are camera-to-world rotations (Pose::R), row-major. */
typedef struct icg_track_frame {
    int32_t prev_slot, cur_slot; /* KLT slots of frame_pre_ / frame_cur_ (pyramids built) */
    icg_camera camera;
    double R_pre[9], R_cur[9], R_ref[9]; /* frame_pre_, predicted frame_cur_, frame_ref_ */
    double t_cur[3];                     /* predicted frame_cur_ position (world2pixel, :367) */
    double dt;                           /* frame_cur_->stamp() - frame_pre_->stamp() (:429, :528) */
    int64_t ref_id;                      /* frame_ref_->id() (:536, :912) */
    double fm_threshold;                 /* reprojection_error_std_ (:548) */
} icg_track_frame;
/* Map-point list (trackMappoint; the previous frame's map-point features in list order).  Inputs per point: prev_xy = distortedKeyPoint()
 * (pts2d_map), prev_undis_xy = keyPoint() (pts2d_map_undis), pw = mappoint->pos(), ref_kp_xy = keyPoint() of the same map point's feature in
 * frame_ref_ or NaN when it has none.  Outputs per INPUT point: fwd_xy (LK forward position), fwd_undis_xy (its undistortion), keep (the
 * gate).  Outputs compacted in list order within the stream's segment: cur_xy (pts2d_matched), cur_undis_xy, velocity (2 doubles),
 * src (index of the survivor in the stream's input list, for reducing mappoint_matched_ / mappoint_type). */
typedef struct icg_track_map {
    const float *prev_xy, *prev_undis_xy;
    const double *pw;
    const float *ref_kp_xy;
    float *fwd_xy, *fwd_undis_xy;
    uint8_t *keep;
    float *cur_xy, *cur_undis_xy;
    double *velocity;
    int32_t *src;
} icg_track_map;
/* Reference list (trackReferenceFrame).  Inputs per point: new_xy = pts2d_new_, ref_xy = pts2d_ref_, ref_frame_id = pts2d_ref_frame_[k]->id(),
 * velocity_ref = velocity_ref_ (2 doubles).  Outputs per INPUT point: fwd_xy, fwd_undis_xy, keep (LK gate && RANSAC inlier).  Compacted within
 * the stream's segment: cur_xy (pts2d_cur_, the next pts2d_new_), cur_undis_xy, velocity (velocity_cur_), ref_out_xy, ref_frame_id_out,
 * velocity_ref_out (velocity_ref_ with the :536-538 rule applied), src. */
typedef struct icg_track_ref {
    const float *new_xy, *ref_xy;
    const int64_t *ref_frame_id;
    const double *velocity_ref;
    float *fwd_xy, *fwd_undis_xy;
    uint8_t *keep;
    float *cur_xy, *cur_undis_xy;
    double *velocity;
    float *ref_out_xy;
    int64_t *ref_frame_id_out;
    double *velocity_ref_out;
    int32_t *src;
} icg_track_ref;
/*
 * Both steps for n_streams streams in one asynchronous call on the KLT handle's stream:
 *   prediction   map: distortPoints(world2pixel(pw, pose_cur)) (:367, :378); ref: undistort(new) -> pixel2cam -> R_cur^T R_pre . ->
 *                distortCameraPoint, float cast included (:465-479)
 *   LK + gate    one forward+backward batch over both lists of all streams (icg_klt_track_batch_dev mode 1; :385-403, :487-506)
 *   compaction   stable, in list order (reduceVector, :404-408, :507-511)
 *   velocities   (pixel2cam(undistort(cur)) - pixel2cam(prev_undis)) / dt (:429-434, :527-533); velocity_ref = velocity_cur where
 *                ref_frame_id > ref_id (:536-538)
 *   parallax     map: mean keyPointParallax(ref_kp, cur_undis, R_ref, R_cur) over the survivors with a ref_kp (:873-905, :450);
 *                ref: over undistort(ref) of the survivors with ref_frame_id == ref_id, BEFORE the RANSAC (:541-544);
 *                keyPointParallax = |(R_cur^T R_ref pc0).xy - pc1.xy| (fx + fy) / 2 (:861-871).  Both sums run in list order; the
 *                reference iterates an std::unordered_map (frame.h:80), whose order is implementation-defined.
 *   RANSAC       findFundamentalMat(new_undis, cur_undis, FM_RANSAC, fm_threshold, 0.99), maxIters 1000, when >= 15 ref points survive
 *                the gate, then the second compaction (:546-555)
 * map_off / ref_off: HOST arrays of n_streams + 1 (starting at 0): stream s owns points off[s] .. off[s + 1] of its list; the lists' pointers
 * are DEVICE pointers (a list with no points may be NULL).  n_map + n_ref <= the handle's max_points.  Outputs (DEVICE): dev_n_out[2 s] /
 * [2 s + 1] = compacted map / ref count; dev_parallax[2 s] / [2 s + 1] = parallax_map_ / parallax_ref_ (the mean), dev_parallax_n likewise
 * = their counts, -1 when the reference returns before computing it and keeps the previous value (empty input list :372-375, :459-462;
 * ref list emptied by the gate :513-517); a map list emptied by the gate gives 0 / 0 (:416-417).
 * The per-input fwd_undis_xy (map list, the `feat` list of featuresDetection :598) and fwd_xy (ref list, `new` :602) with their keep flags
 * feed icg_detect_features_dev with the same offsets and no host round trip.  Scratch is allocated on first use (ICG_ENOMEM on failure).
 */
int icg_klt_track_frames_dev(icg_klt *h, int n_streams, const icg_track_frame *params, const int32_t *map_off, const icg_track_map *map,
                             const int32_t *ref_off, const icg_track_ref *ref, int32_t *dev_n_out, double *dev_parallax, int32_t *dev_parallax_n);
/* The same for one stream from HOST buffers (every pointer of map / ref is a host pointer; n_out / parallax / parallax_n: 2 each, host);
 * synchronous.  A thin wrapper over the launch sequence of icg_klt_track_frames_dev. */
int icg_klt_track_frame(icg_klt *h, const icg_track_frame *params, int n_map, const icg_track_map *map, int n_ref, const icg_track_ref *ref,
                        int32_t *n_out, double *parallax, int32_t *parallax_n);

/* ----- Tracking::triangulation (IG/tracking/tracking.cc:690-798) on the KLT handle (csrc/track.cu) ----- */
/* Per-stream parameters.  Attitudes are camera-to-world rotations (Pose::R), row-major, as in icg_track_frame. */
typedef struct icg_tri_frame {
    icg_camera camera;
    double R_cur[9], t_cur[3];     /* frame_cur_->pose() (:699) */
    int64_t cur_id, ref_id;        /* frame_cur_->id(), frame_ref_->id() (:723) */
    int32_t window_normal;         /* map_->isWindowNormal() (:733) */
    int32_t triangulate;           /* the host's keyframe decision (:215-217); 0: the stream is left untouched, kept = -1 */
    double reprojection_error_std; /* reprojection_error_std_ (isGoodToTrack, :813-829) */
} icg_tri_frame;
/* A frame a point of the stream can name as pts2d_ref_frame_[k]: its id, pose (Pose::R row-major, Pose::t) and whether
 * map_->isKeyFrameInMap(frame) holds (:733). */
typedef struct icg_tri_keyframe {
    int64_t id;
    double R[9], t[3];
    int32_t in_map;
} icg_tri_keyframe;
/* The reference list as icg_klt_track_frames_dev leaves it (the same pointers can be passed).  ref_out_xy = pts2d_ref_, ref_frame_id_out =
 * pts2d_ref_frame_[k]->id(), cur_xy = pts2d_cur_, velocity_ref_out = velocity_ref_ (2 doubles): compacted IN PLACE in list order by the
 * status of :788-791 (reduceVector).  velocity = velocity_cur_ (2 doubles), read only (:791 does not reduce it).  src: the input index of
 * every kept point. */
typedef struct icg_tri_list {
    float *ref_out_xy;
    int64_t *ref_frame_id_out;
    float *cur_xy;
    double *velocity_ref_out;
    const double *velocity;
    int32_t *src;
} icg_tri_list;
/* The new map points in creation order (MapPoint ids are issued in this order, mappoint.cc:45-49; :761-784): pw (3 doubles), depth =
 * world2cam(pw, frame_ref->pose()).z with MapPoint's clamp (outside [1, 200] -> 10, mappoint.cc:39-42), the reference feature
 * (ref_undis_xy = undistort(pts2d_ref_[k]), ref_xy = pts2d_ref_[k], velocity_ref = velocity_ref_[k] (2 doubles), ref_frame_id), the current
 * feature (cur_undis_xy, cur_xy = pts2d_cur_[k], velocity_cur = velocity_cur_[k] (2 doubles)) and src = the point's input index. */
typedef struct icg_tri_new {
    double *pw, *depth;
    float *ref_undis_xy, *ref_xy, *cur_undis_xy, *cur_xy;
    double *velocity_cur, *velocity_ref;
    int64_t *ref_frame_id;
    int32_t *src;
} icg_tri_new;
/*
 * Tracking::triangulation for n_streams streams in one asynchronous call on the KLT handle's stream (stream-ordered after
 * icg_klt_track_frames_dev).  Per point k, in list order:
 *   reset      ref_frame_id > ref_id: ref_frame_id := cur_id, ref_xy := cur_xy, kept; velocity_ref untouched (:723-730)
 *   outtime    window_normal && !in_map(ref frame): dropped (:733-737)
 *   parallax   keyPointParallax(undistort(ref), undistort(cur), ref frame pose, pose_cur) < 10 (TRACK_MIN_PARALLAX, tracking.h:114): kept (:740-745)
 *   triangulate pw = triangulatePoint(Tcw(ref frame), Tcw(pose_cur), pixel2cam(ref_undis), pixel2cam(cur_undis)), Tcw = [R^T | -R^T t] (:747-753, :851-859)
 *   outlier    unless isGoodToTrack(ref_undis, pose_ref, pw, 1, 3) && isGoodToTrack(cur_undis, pose_cur, pw, 1, 3): 1 < z < 600 and
 *              |world2pixel(pw) - pp| <= reprojection_error_std, the difference taken in float (camera.cc:153-157): dropped (:756-760, :813-829)
 *   succeeded  dropped from the list, written to `out` as a new map point (:761-784)
 * kf_off (n_streams + 1, starting at 0) and kf: HOST CSR of each stream's frames, at most 64 per stream with distinct ids (ICG_EINVAL
 * otherwise).  Every ref_frame_id <= ref_id in a stream's live list must be in its table (frames that left the map with in_map = 0),
 * otherwise the stream reports -2 and nothing of it is written.  ref_off (HOST, n_streams + 1): stream s owns list entries ref_off[s] ..
 * ref_off[s + 1] and writes its new points from out index ref_off[s].  The live count of stream s is read ON THE DEVICE from
 * dev_n_in[s * n_in_stride] (icg_klt_track_frames_dev's dev_n_out + 1 with stride 2 chains both calls without a host sync); dev_n_in NULL:
 * the segment length; a count outside [0, segment] gives -2.  dev_counts (DEVICE, 5 int32 per stream): kept (-1: the reference's
 * `return false` for an empty list, and streams with triangulate == 0; -2: see above), succeeded, outlier, reset, outtime (:795).
 * Parameters, offsets and tables are staged through the handle's pinned buffer; list and out pointers are DEVICE pointers.
 */
int icg_klt_triangulate_dev(icg_klt *h, int n_streams, const icg_tri_frame *params, const int32_t *kf_off, const icg_tri_keyframe *kf,
                            const int32_t *ref_off, const int32_t *dev_n_in, int n_in_stride, const icg_tri_list *list, const icg_tri_new *out,
                            int32_t *dev_counts);
/* The same for one stream from HOST buffers (n points, n_kf table entries; out needs room for n points; counts: 5 int32, host);
 * synchronous.  A thin wrapper over the launch of icg_klt_triangulate_dev.  n <= the handle's max_points. */
int icg_klt_triangulate(icg_klt *h, const icg_tri_frame *params, int n_kf, const icg_tri_keyframe *kf, int n, const icg_tri_list *list,
                        const icg_tri_new *out, int32_t *counts);

/* ----- pre-pass of path A: cv::CLAHE (IG/tracking/tracking.cc:62 createCLAHE(3.0, Size(21, 21)); :141 clahe_->apply(img, img)) ----- */
typedef struct icg_clahe icg_clahe;
int icg_clahe_create(icg_clahe **h, int width, int height, int tiles_x, int tiles_y, double clip_limit, int device, void *stream);
void icg_clahe_destroy(icg_clahe *h);
/* Drop-in for cv::CLAHE::apply(src, dst) on 8-bit single-channel host buffers (dst may alias src): H2D, per-tile LUTs, bilinear LUT
 * interpolation, D2H; synchronous.  Bit-exact with OpenCV (tests/golden/clahe_golden.npz). */
int icg_clahe_apply(icg_clahe *h, const uint8_t *src, int src_stride, uint8_t *dst, int dst_stride);
/* Device-resident variant (asynchronous on the handle's stream): src / dst are device pointers, e.g. the level-0 plane of a KLT slot
 * (icg_klt_slot_level0) so that upload -> CLAHE -> pyramid -> track never leaves HBM; dst may alias src. */
int icg_clahe_apply_dev(icg_clahe *h, const uint8_t *dev_src, int src_pitch, uint8_t *dev_dst, int dst_pitch);
/* Frame-batched device-resident variant: n_frames frames (frame f at dev_src + f * src_frame_stride, written to dev_dst + f * dst_frame_stride;
 * in place allowed) in one launch pair.  hist_out (host, n_frames doubles, may be NULL): Tracking::calculateHistigram of every RAW frame
 * (IG/tracking/tracking.cc:88-104), accumulated by the LUT pass at no extra read of the frame -- the statistic of the histogram gate in
 * Tracking::preprocessing (:115-133).  With hist_out the call synchronises (the host decides whether to skip the frame); without, it is asynchronous. */
int icg_clahe_apply_batch_dev(icg_clahe *h, int n_frames, const uint8_t *dev_src, int src_pitch, size_t src_frame_stride, uint8_t *dev_dst, int dst_pitch,
                              size_t dst_frame_stride, double *hist_out);
int icg_clahe_sync(icg_clahe *h);

/* ----- detection leg of path A: Tracking::featuresDetection (IG/tracking/tracking.cc:576-688) ----- */
typedef struct icg_rect {
    int32_t x, y, w, h;
} icg_rect;
typedef struct icg_detect icg_detect;
/* width x height frames; up to max_blocks ROIs per call, each at most max_roi_pixels pixels, at most
 * max_corners_per_block corners returned per block. */
int icg_detect_create(icg_detect **h, int width, int height, int max_blocks, int max_corners_per_block, int max_roi_pixels, int device, void *stream);
void icg_detect_destroy(icg_detect *h);
/*
 * The body of the tbb::parallel_for over blocks (IG/tracking/tracking.cc:627-656) for all blocks in one call:
 *   cv::goodFeaturesToTrack(frame(roi), out, max_corners[b], quality, min_distance, mask(roi))          (:647)
 *   cv::cornerSubPix(frame(roi), out, Size(5,5), Size(-1,-1), TermCriteria(COUNT+EPS, 20, 0.01))        (:651, when do_subpix)
 * with C++ ROI semantics (the derivative of a block reads the frame beyond the block edge).  img / mask are full frames
 * (mask may be NULL == all 255).  out_xy: n_blocks x max_corners_per_block x 2 floats, block-LOCAL coordinates in
 * OpenCV's order (strength descending, ties by address descending); out_n: corners per block.  Host buffers, synchronous.
 * A single ROI covering the frame reproduces the stand-alone cv::goodFeaturesToTrack / cv::cornerSubPix calls.
 */
int icg_detect_blocks(icg_detect *h, const uint8_t *img, const uint8_t *mask, int stride, int n_blocks, const icg_rect *rois,
                      const int32_t *max_corners, double quality, double min_distance, int do_subpix, float *out_xy, int32_t *out_n);
/* The same for n_frames DEVICE-resident frames in one call (throughput mode / the keyframe path of many streams): frame f starts at
 * dev_img + f * frame_stride (row pitch `pitch` bytes; e.g. the level-0 planes of consecutive KLT slots, icg_klt_slot_level0), dev_mask (NULL or the
 * same geometry) likewise; the n_blocks ROIs apply to every frame; max_corners is n_frames x n_blocks (or NULL); outputs are host arrays of
 * n_frames x n_blocks (x cap x 2).  The handle's max_blocks must cover n_frames * n_blocks. */
int icg_detect_blocks_dev(icg_detect *h, int n_frames, const uint8_t *dev_img, int pitch, size_t frame_stride, const uint8_t *dev_mask, int n_blocks,
                          const icg_rect *rois, const int32_t *max_corners, double quality, double min_distance, int do_subpix, float *out_xy,
                          int32_t *out_n);
/*
 * Tracking::featuresDetection (IG/tracking/tracking.cc:576-685) up to the append into the reference's lists, driven by the point lists:
 *   gate (:579-582): |feat| + n_ref > max_features - 5 -> the frame is not detected, *out_n = -1 (the caller keeps its lists);
 *   counts (:591-606): every feat point (undistorted keyPoint(), :598) and every new point (pts2d_new_, distorted, :602) goes into block
 *     int(y / (float) bh) * cols + int(x / (float) bw) (a col == cols aliases into the next row's first block; indices outside the grid are
 *     dropped); block k asks for quota - count[k] corners (:629) and is skipped when that is <= 0;
 *   mask (:609-620, when ismask): 255, and 0 on the disc of radius min_dist around cvRound of every point, clipped to the frame;
 *   goodFeaturesToTrack(quality 0.01, min_dist) + cornerSubPix per block as icg_detect_blocks (:627-656), then the shift to frame
 *     coordinates (float) (col * bw) + x (:669-675).
 * The grid is Tracking::Tracking's (:66-85): cols = lround(W / 200.0), rows = lround(H / 200.0), bw = W / cols, bh = H / rows,
 * quota = lround(max_features / (double) (cols * rows)), min_dist = (int) round(200 / sqrt(quota * 1.5)).  ICG_EINVAL when quota exceeds the
 * handle's max_corners_per_block, the frames' blocks exceed max_blocks, a block exceeds max_roi_pixels or the offsets are not monotone.
 * Host buffers, one frame, synchronous.  out_xy: cols * rows * quota x 2 floats (frame coordinates, block order, OpenCV's order within a block);
 * *out_n = the number of corners, -1 when the gate skipped the frame.  n_ref < 0 stands for n_new.
 */
int icg_detect_features(icg_detect *h, const uint8_t *img, int stride, const float *feat_xy, int n_feat, const float *new_xy, int n_new,
                        int n_ref, int ismask, int max_features, float *out_xy, int32_t *out_n);
/* The same for n_frames DEVICE-resident frames in one call (geometry as icg_detect_blocks_dev).  Point lists in DEVICE memory: frame f's feat
 * points are dev_feat_xy[feat_off[f] .. feat_off[f + 1]), its new points likewise; feat_off / new_off are HOST arrays of n_frames + 1.
 * dev_feat_status / dev_new_status: DEVICE u8 per point or NULL; a point with status 0 is neither counted nor masked, so the LK status of
 * icg_klt_track_batch_dev can be passed without compacting.  n_ref: HOST, n_frames, or NULL = the number of valid points of the frame's new
 * list.  ismask: HOST, n_frames (NULL = all set).  Outputs in DEVICE memory: frame f's corners at dev_out_xy + f * cols * rows * quota * 2,
 * dev_out_n[f] as *out_n above, or -2 when an internal capacity was exceeded.  Asynchronous on the handle's stream.  The first call allocates
 * one pitch x height mask plane per frame the handle's max_blocks allows (ICG_ENOMEM if that fails). */
int icg_detect_features_dev(icg_detect *h, int n_frames, const uint8_t *dev_img, int pitch, size_t frame_stride,
                            const float *dev_feat_xy, const uint8_t *dev_feat_status, const int32_t *feat_off,
                            const float *dev_new_xy, const uint8_t *dev_new_status, const int32_t *new_off,
                            const int32_t *n_ref, const uint8_t *ismask, int max_features, float *dev_out_xy, int32_t *dev_out_n);
/* device pointer + row pitch of frame f's occupancy mask as the last icg_detect_features[_dev] call built it (parity tests); the mask of a
 * frame the gate skipped is not written */
int icg_detect_mask_dev(icg_detect *h, int frame, void **dev_ptr, int *pitch);
/* Drop-in for cv::cornerSubPix(img, corners, Size(5,5), Size(-1,-1), (COUNT+EPS, 20, 0.01)) on the whole frame; corners in/out */
int icg_corner_subpix(icg_detect *h, const uint8_t *img, int stride, float *corners_xy, int n);

/* ===================================================================================================== *
 *  Path B: sliding-window factor-graph solve
 * ===================================================================================================== */
/*
 * One window problem == what GVINS::gvinsOptimization hands to Ceres (IG/ic_gvins.cc:1130-1239, 1697-1909):
 *   parameter blocks  statedatalist_[k].pose[7] = (p, q_xyzw), .mix[9] = (v, bg, ba)      (IG/preintegration/integration_state.h:53-66)
 *                     extrinsic_[8] = (t_bc, q_bc xyzw, td)                                 (IG/ic_gvins.cc:1736-1756)
 *                     invdepthlist_ values, one per landmark                                (IG/ic_gvins.cc:1727)
 *   residual blocks   ReprojectionFactor(pose_ref, pose_obs, extrinsic, invdepth, td) + HuberLoss(1.0)   (:1826-1831)
 *                     PreintegrationFactor(pose_k, mix_k, pose_k+1, mix_k+1)                              (:1870-1872)
 *                     ImuErrorFactor(mix_last), ImuPosePriorFactor(pose_0), ImuMixPriorFactor(mix_0)       (:1877-1887)
 *                     GnssFactor(pose_node) + HuberLoss(1.0) in the first pass                             (:1896-1903)
 *                     MarginalizationFactor(remained blocks)                                               (:1158-1161)
 * All arrays are caller-owned host memory; pose/mix/ext/invdepth are updated in place by the solve
 * (as Ceres mutates the reference's parameter arrays in place).
 */
#define ICG_IMU_BLOB_DOUBLES 480
/* IMU preintegration blob (doubles): [0] delta_time, [1..3] delta p, [4..6] delta v, [7..10] delta q (x,y,z,w),
 * [11..13] bg, [14..16] ba (linearisation biases), [17..19] gravity, [20..22] iewn,
 * [23] S0 = sum_i dt_i, [24..26] S1 = sum_i dt_i * pn_i   (the two moments of pn_ that
 *      PreintegrationEarth::evaluate's position-compensation loop needs, IG/preintegration/preintegration_earth.cc:55-59),
 * [27..251] jacobian_ 15x15 row-major, [252..476] covariance_ 15x15 row-major,
 * [477] factor form: 0 = PreintegrationEarth (IG/preintegration/preintegration_earth.cc), 1 = PreintegrationNormal
 *       (preintegration_normal.cc, `iswithearth: false`: iewn = 0, S0 = S1 = 0), [478..479] reserved. */
typedef struct icg_ba_problem {
    int32_t K, L, F;
    double *pose;     /* K*7 in/out */
    double *mix;      /* K*9 in/out */
    double *ext;      /* 8   in/out */
    double *invdepth; /* L   in/out */
    int32_t ext_const, td_const; /* SetParameterBlockConstant (IG/ic_gvins.cc:1750,1758) */
    const int32_t *f_lm, *f_ref, *f_obs; /* F each: landmark, reference node, observing node */
    const double *f_const;               /* F*14: pts0[3] pts1[3] vel0[3] vel1[3] td0 td1 */
    const uint8_t *f_active;             /* F, or NULL == all active (RemoveResidualBlock, IG/ic_gvins.cc:1291) */
    double reproj_std;
    int32_t reproj_huber;
    int32_t n_imu;
    const double *imu_blob; /* n_imu * ICG_IMU_BLOB_DOUBLES; factor k joins node k and k+1 */
    int32_t has_imu_error;
    int32_t has_pose_prior;
    const double *pose_prior, *pose_prior_std; /* 7, 6 */
    int32_t has_mix_prior;
    const double *mix_prior, *mix_prior_std; /* 9, 9 */
    int32_t n_gnss;
    const int32_t *gnss_node;
    const double *gnss_blh, *gnss_std; /* n_gnss*3 each */
    double lever[3];
    int32_t gnss_huber;
    int32_t marg_r, marg_nblocks;                    /* 0 == no prior */
    const int32_t *marg_block_type, *marg_block_node; /* type 0 pose(node) 1 mix(node) 2 extrinsic 3 td */
    const double *marg_x0, *marg_J0, *marg_e0;        /* concatenated x0 (global sizes), J0 row-major r x r, e0 */
} icg_ba_problem;

typedef struct icg_ba_summary {
    int32_t iterations;           /* LM iterations executed */
    int32_t num_successful_steps; /* ceres::Solver::Summary::num_successful_steps (IG/ic_gvins.cc:1186) */
    int32_t termination;          /* 0 NO_CONVERGENCE (max iterations), 1 CONVERGENCE, 2 FAILURE */
    int32_t reserved;
    double initial_cost, final_cost, final_radius;
} icg_ba_summary;

/* B3 (host side, as in the reference: fusion thread, IG/ic_gvins.cc:917-919): IMU preintegration propagation
 * PreintegrationEarth::resetState/integrationProcess/updateJacobianAndCovariance (IG/preintegration/preintegration_earth.cc:205-338).
 * state16 = p[3] q_xyzw[4] v[3] bg[3] ba[3] at the interval start; noise5 = gyr_arw, acc_vrw, gyr_bias_std, acc_bias_std, corr_time;
 * imu = n rows of (dt, dtheta[3], dvel[3]), row 0 being the sample at the interval start.  Writes the factor blob and the
 * mechanised end state (p, q_xyzw, v).  Sequential recurrence; runs on the calling host thread.
 * iewn3 == NULL selects PreintegrationNormal (PreintegrationBase::integration + PreintegrationNormal::updateJacobianAndCovariance,
 * IG/preintegration/preintegration_base.cc:39-70, preintegration_normal.cc:195-232). */
int icg_imu_preintegrate(const double *state16, const double *iewn3, const double *gravity3, const double *noise5, const double *imu,
                         int n, double *blob_out, double *end_state10);

typedef struct icg_ba icg_ba;
/*
 * Solver for batches of up to max_windows windows of at most max_K nodes / max_L landmarks / max_F reprojection
 * factors each (throughput mode: one window per independent stream).  stream may be NULL.
 */
int icg_ba_create(icg_ba **h, int max_windows, int max_K, int max_L, int max_F, int max_gnss, int max_marg_r, int device,
                  void *stream);
void icg_ba_destroy(icg_ba *h);
/*
 * Drop-in for `ceres::Solver::Solve(options, &problem, &summary)` with LEVENBERG_MARQUARDT + DENSE_SCHUR
 * (IG/ic_gvins.cc:1143-1146, 1183, 1217) on n_windows independent problems at once.  Parameters are updated in place.
 */
int icg_ba_solve(icg_ba *h, int n_windows, const icg_ba_problem *problems, int max_num_iterations, icg_ba_summary *summaries);
/* The three stages of icg_ba_solve, exposed for device-resident operation (throughput mode / benchmarking):
 *   upload   : pack + H2D of n problems (what AddParameterBlock / AddResidualBlock build, IG/ic_gvins.cc:1697-1909)
 *   run      : enqueue max_num_iterations LM iterations, asynchronously on the handle's stream; restart != 0 first restores
 *              the parameters that were uploaded (re-solve the same problems)
 *   download : D2H of the parameters into the problems' arrays (problems may be NULL) + summaries; synchronises. */
int icg_ba_upload(icg_ba *h, int n_windows, const icg_ba_problem *problems);
int icg_ba_run(icg_ba *h, int max_num_iterations, int restart);
int icg_ba_download(icg_ba *h, int n_windows, const icg_ba_problem *problems, icg_ba_summary *summaries);
/*
 * Drop-in for the body of GVINS::gvinsOptimization (IG/ic_gvins.cc:1130-1239) on n_windows problems:
 *   Solve(max_num_iterations = N/4) with HuberLoss on GNSS + reprojection         (:1183)
 *   gnssOutlierCullingByChi2 (chi2 > 7.815 -> std *= sqrt(chi2/7.815))            (:1241-1267)
 *   removeReprojectionFactorsByChi2(5.991)                                        (:1269-1297)
 *   GNSS factors re-added without loss, Solve(max_num_iterations = N - N/4)       (:1202-1217)
 * entirely on the device (no host round trip between the passes).  Parameters are updated in place; the problems'
 * f_active (must be non-NULL to receive the removals) and gnss_std arrays are updated in place too, as the reference mutates
 * `gnss->std` and removes residual blocks.  summaries: 2 per window (pass 1, pass 2), may be NULL.
 * culled: 2 ints per window (reprojection factors removed, GNSS fixes re-weighted), may be NULL.
 * icg_ba_run_gvins is the asynchronous device-only stage for problems already uploaded.
 */
int icg_ba_gvins_optimization(icg_ba *h, int n_windows, const icg_ba_problem *problems, int num_iterations, icg_ba_summary *summaries,
                              int32_t *culled);
int icg_ba_run_gvins(icg_ba *h, int num_iterations, int restart);
/* The same call split in two so that a caller driving several handles (streams) can overlap them: _begin packs, uploads and
 * enqueues (asynchronous on the handle's stream), _end synchronises and writes the results back. */
int icg_ba_gvins_optimization_begin(icg_ba *h, int n_windows, const icg_ba_problem *problems, int num_iterations);
int icg_ba_gvins_optimization_end(icg_ba *h, int n_windows, const icg_ba_problem *problems, icg_ba_summary *summaries, int32_t *culled);
int icg_ba_sync(icg_ba *h);
/*
 * Drop-in for `MarginalizationInfo::marginalization()` as GVINS::gvinsMarginalization drives it (IG/ic_gvins.cc:1412-1640,
 * IG/factors/marginalization_info.h:73-253): for each window, the num_marg oldest nodes (pose + mix) and the inverse depths of the
 * landmarks anchored in them are marginalized out of [previous prior, GNSS at those nodes, preintegration factors 0..num_marg-1,
 * first-window pose / mix priors, reprojection factors of those landmarks] (no loss functions, every Jacobian, as
 * ResidualBlockInfo::Evaluate does), linearised at the parameter values in `problems`.  Output: the new prior in the layout
 * icg_ba_problem.marg_* consumes -- remained blocks (node indices already shifted by num_marg), x0 = remainedBlockData(),
 * J0 = linearizedJacobians() (r x r row-major, rows in ascending eigenvalue order), e0 = linearizedResiduals() -- plus, optionally,
 * the Schur complement itself (Hp, bp).  Arrays are caller-allocated: block_type/block_node 2K+2 ints, x0 16K+8, J0/Hp rcap*rcap,
 * e0/bp rcap doubles with rcap >= 15*(K - num_marg) + 7.  Column order inside the marginalized / remained groups is
 * [pose_k, mix_k ascending k | landmarks ascending] / [pose_k, mix_k (touched blocks only) | ext | td]; the reference's order is that of
 * an unordered_map (implementation-defined) and only permutes rows / columns.
 * Sizes: the device workspace follows the batch (its largest m and m + r), not the handle's max_K / max_L, so any handle marginalizes,
 * cfg-4 windows (max_K = 20, max_L = 2000) included.  A window whose m or r exceeds 512 rows (the largest eigensolver) returns
 * ICG_EUNSUPPORTED naming the window, before anything runs on the device.  Landmark-sharded handles return ICG_EUNSUPPORTED here (the
 * resident forms below run on them).  The next
 * window consumes the prior through icg_ba_problem.marg_r <= max_marg_r: a window of K nodes can need 15 (K - 1) + 7 rows (292 at K = 20).
 */
typedef struct icg_ba_prior {
    int32_t m, r, nblocks;            /* out: marginalizedSize(), remainedSize(), number of remained blocks */
    int32_t rcap;                     /* in: capacity of J0 / e0 / Hp / bp */
    int32_t *block_type, *block_node; /* out */
    double *x0, *J0, *e0;             /* out */
    double *Hp, *bp;                  /* out, may be NULL */
} icg_ba_prior;
int icg_ba_marginalize(icg_ba *h, int n_windows, const icg_ba_problem *problems, const int32_t *num_marg, icg_ba_prior *out);
/* The same on the windows the handle already holds: gvinsMarginalization runs right after gvinsOptimization on the same window
 * (IG/ic_gvins.cc:560-567 -> 1412), so after icg_ba_gvins_optimization[_end] / icg_ba_solve the device copy already has the optimised
 * parameters, the culled factor set and the re-weighted GNSS sigmas; nothing is packed or uploaded again.  `problems` must be the array
 * of that solve (n_windows equal to the uploaded count; read for the factor structure and x0 only).
 * Landmark-sharded handle (world > 1): a COLLECTIVE call.  Every rank calls with its shard problems (what it uploaded) and the same
 * num_marg; each window must list its factors landmark by landmark (f_lm non-decreasing, as the reference builds them), which is checked
 * before anything is launched.  Every rank exports the rows of its factors with f_ref < num_marg; the owner of window w (rank w mod world)
 * gathers them over peer memory in rank order and forms the prior with the single-GPU kernels: out[w] is bit-for-bit what an unsharded
 * handle holding the same values produces.  out[w] is filled on the owner only; on every other rank out[w].m = r = nblocks = 0 and its
 * arrays are not written.  No resident prior is kept for a slide (both slides remain unavailable on sharded handles).  A rank that
 * rejects its arguments leaves its peers to the bounded flag waits: they return ICG_ECUDA (icg_ba_shard_error).
 * Memory: each rank's export region (max_windows x max_F x 128 bytes, allocated by icg_ba_shard_export), and on an owner a second handle
 * the gathered windows are marginalized in (ceil(max_windows / world) windows, this handle's max_K / max_gnss / max_marg_r, 1.25 x the
 * largest gathered window's landmarks and factors; created on the first call, grown when a batch needs more).  Buffers a call outgrows
 * are freed by icg_ba_shard_leave, the next icg_ba_shard_export or icg_ba_destroy. */
int icg_ba_marginalize_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const int32_t *num_marg, icg_ba_prior *out);
/*
 * The rest of GVINS::gvinsOptimization after the second Solve (IG/ic_gvins.cc:1232-1236), on the windows the handle holds:
 *   updateParametersFromOptimizer (:1299-1389)
 *     td_b_c = ext[7] when estimate_td;  when estimate_ext: R = toRotationMatrix(Quaterniond(ext[6], ext[3..5]).normalized()), t = ext[0..2],
 *     dt = |t - t_bc|, dr = |Quaterniond(R R_bc^T).vec()| 180 / pi; (R, t) replaces (R_bc, t_bc) unless dt > 1 || dr > 5
 *     node k: R_c = R(q_k normalised) R_bc, t_c = p_k + R(q_k) t_bc (MISC::stateToCameraPose with the gated extrinsic, misc.cc:102-108)
 *     landmark l: depth = 1 / invdepth (no clamp), pw = R_c(ref) (pixel2cam(ref_kp) depth) + t_c(ref)
 *   gvinsOutlierCulling (:1035-1128), per landmark, its observations in list order:
 *     an observation fails unless isGoodToTrack(kp, pose, pw, 3.0): 1 < z < 200 and |float(world2pixel) - kp| <= 3 std (a NaN or infinite
 *     depth fails); a failing observation is a feature outlier; if it is in the landmark's reference node the landmark is an outlier
 *     (reason 1) and the walk stops there.  Then, whatever the walk did: fewer than two passing observations -> reason 2, otherwise
 *     mean of their errors (summed in list order) > std -> reason 3.
 * Arithmetic: fixed-order sums without FMA; parity with Eigen's products and its Quaterniond(Matrix3d) is not pinned.
 * The caller gathers, per landmark, the observations the culling visits (mappoint->observations() in that order, skipping features that
 * are already outliers and frames that are not keyframes in the map; the reference observation included, the factors the chi-square
 * pass removed included).  Every keyframe in the map has a time node (addNewKeyFrameTimeNode, IG/ic_gvins.cc:724-752), so every
 * observation names a node.  Landmarks are in the problem's order (the order of invdepth); outputs are in that order too.
 */
typedef struct icg_ba_cull_window {
    /* in */
    double R_bc[9], t_bc[3], td_bc;    /* pose_b_c_ (R row-major) and td_b_c_ before the update */
    int32_t estimate_ext, estimate_td; /* optimize_estimate_extrinsic_, optimize_estimate_td_ */
    const int32_t *lm_ref_node;        /* L: node of mappoint->referenceFrame() */
    const float *lm_ref_kp;            /* L x 2: mappoint->referenceKeypoint() */
    const int32_t *obs_off;            /* L + 1, obs_off[0] = 0: landmark l owns observations obs_off[l] .. obs_off[l + 1] */
    const int32_t *obs_node;           /* node of the observing keyframe (every keyframe in the map has one) */
    const float *obs_kp;               /* x 2: feat->keyPoint() */
    const int32_t *obs_factor;         /* reprojection factor (problem row) of the observation, -1 for none (the reference observation);
                                          read by icg_ba_marginalize_resident_culled only, may be NULL for the culling */
    /* out */
    double R_bc_out[9], t_bc_out[3], td_bc_out; /* pose_b_c_ / td_b_c_ after the update */
    int32_t ext_accepted;              /* 1: the estimate replaced pose_b_c_, 0: the 1 m / 5 deg gate rejected it, -1: estimate_ext is 0 */
    double *cam_pose;                  /* K x 12: frame->pose() of every node, R row-major | t */
    double *lm_pw, *lm_depth;          /* L x 3, L: mappoint->pos(), the depth of updateDepth */
    uint8_t *lm_outlier;               /* L: bit 0 reason 1, bit 1 reason 2, bit 2 reason 3 (0: kept) */
    uint8_t *obs_outlier;              /* per observation: feat->setOutlier(true) (observations after a reason-1 stop stay 0) */
    int32_t counts[5];                 /* outliers_[0], outliers_[1], num1, num2, num3 as the reference counts them (a landmark with reason 1
                                          and reason 2 or 3 counts twice in outliers_[0]) */
} icg_ba_cull_window;
/* One CTA per window; the observation lists go up in one copy through pinned staging and the outputs come back in one copy; synchronous.
 * `problems` is the array of the solve (n_windows equal to the uploaded count; K and L are read).  The handle's state (parameters,
 * factor activity, GNSS sigmas) is not changed.
 * Landmark-sharded handle (world > 1): a collective call.  Every rank passes its shard problems and, per window, the observation lists of
 * its own landmarks in shard order.  cam_pose, the extrinsic outputs and td_bc_out come from the replicated camera side and are the same on
 * every rank; lm_pw, lm_depth, lm_outlier and obs_outlier cover the caller's shard; counts are the window's totals on every rank (summed
 * over the ranks through the peer-memory exchange buffer). */
int icg_ba_update_and_cull_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const icg_camera *cam, double reprojection_error_std,
                                    icg_ba_cull_window *io);
/* icg_ba_marginalize_resident on the map after the culling: reprojection factor f of a landmark anchored in a removed node is marginalized
 * iff its landmark is not a culling outlier, neither its observation nor the landmark's reference observation is a feature outlier, and
 * node_in_map[w][f_obs[f]] is set (the keyframes gvinsRemoveAllSecondNewFrame left in the map, IG/ic_gvins.cc:1391-1410): the factor set
 * gvinsMarginalization builds (:1558-1609).  The chi-square activity plays no part (removeReprojectionFactorsByChi2 never marks a feature).
 * culled: the io array of icg_ba_update_and_cull_resident after that call (obs_factor must be set); node_in_map: K bytes per window.  The
 * handle's factor activity is not changed.  On a landmark-sharded handle: collective, as icg_ba_marginalize_resident; each rank passes its
 * own `culled` array (its shard's landmarks, obs_factor naming its shard's factors) and the same node_in_map. */
int icg_ba_marginalize_resident_culled(icg_ba *h, int n_windows, const icg_ba_problem *problems, const int32_t *num_marg,
                                       const icg_ba_cull_window *culled, const uint8_t *const *node_in_map, icg_ba_prior *out);
/*
 * GVINS::doReintegration (IG/ic_gvins.cc:1680-1695), which gvinsOptimization runs after the second Solve while the window is not full
 * (:1223-1227), on the IMU factors the handle holds.  For factor k of a window (joining nodes k and k + 1):
 *   state    stateFromData(statedatalist_[k]): node k's resident pose with q normalised (q / sqrt(x^2 + y^2 + z^2 + w^2), summed in that
 *            order; parity with Eigen's norm reduction is not pinned) and mix (v, bg, ba), i.e. the values the last solve left
 *   gate     |blob.bg - mix.bg| > 6 noise5[2] or |blob.ba - mix.ba| > 6 noise5[3] (blob[11..16] = deltaState().bg / ba; strict; each norm
 *            the sqrt of the fixed-order sum of squares)
 *   replay   reintegration(state): the whole imu_buffer_ from the new state with the factor's own form (blob[477]) and gravity
 *            (blob[17..19]); the Earth form recomputes iewn = Earth::iewn(station3, p_k) (resetState, preintegration_earth.cc:305-324),
 *            the Normal form keeps iewn = 0.  station3 is parameters_->station, which the reference never assigns: make_shared value-
 *            initialises it (IG/ic_gvins.cc:91), so a faithful caller passes (0, 0, 0).
 * A status-1 factor's blob and square-root information are replaced on the device, so every later icg_ba_marginalize_resident[_culled]
 * and icg_ba_run[_gvins](restart = 1) sees the reintegrated factor, as the reference's next Evaluate does; the square-root information is
 * the one icg_ba_upload computes (same code, same result bit for bit).  Parameters, factor activity and GNSS sigmas are not changed.
 * One warp per factor; the rows go up in one copy through pinned staging, and the statuses, end states and reintegrated blobs come back
 * (unchanged blobs do not).  Synchronous.  `problems` is the array of the solve (n_windows equal to the uploaded count; K and n_imu are
 * read).  ICG_EINVAL before anything is launched when imu_off is not increasing by at least one row per factor; ICG_EINVAL after the call,
 * naming the first such factor, when a reintegrated covariance is not positive definite (status -1: that factor is kept, every other one
 * is processed).  ICG_EUNSUPPORTED on a landmark-sharded handle: its group calls icg_ba_shard_reintegrate_resident.
 */
typedef struct icg_ba_reint_window {
    /* in */
    int32_t reintegrate;    /* 0: the window is left alone (the reference reintegrates only while !map_->isMaximumKeframes(), :1223) */
    const double *imu;      /* rows (dt, dtheta[3], dvel[3]) of every factor's interval (imu_buffer_ of preintegrationlist_[k]) */
    const int32_t *imu_off; /* n_imu + 1: factor k = rows imu_off[k] .. imu_off[k + 1] - 1, row imu_off[k] = imu0 (the sample at its start) */
    /* out */
    int8_t *status;         /* n_imu: 1 reintegrated, 0 gate closed, -1 reintegrated covariance not positive definite (factor NOT replaced) */
    double *blob_out;       /* n_imu x ICG_IMU_BLOB_DOUBLES: written where status == 1 only */
    double *end_state10;    /* n_imu x 10 or NULL: currentState() p, q_xyzw, v after the replay, where status != 0 (addNewTimeNode reads the
                               last one, :923) */
    int32_t count;          /* cnt of :1689: factors whose gate opened (0 for windows left alone) */
} icg_ba_reint_window;
int icg_ba_reintegrate_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const double *noise5, const double *station3,
                                icg_ba_reint_window *io);
/*
 * The next keyframe's windows from the ones the handle holds, without re-uploading what the device already has.  GVINS rebuilds the problem
 * every keyframe (IG/ic_gvins.cc:1130-1239, 1697-1837); between two windows most of it carries over: node states (the values the solve left),
 * inverse depths (through depth = 1 / invdepth and back: rho' = 1.0 / (1.0 / rho)), reprojection factor constants, IMU blobs (reintegrated
 * ones included) with their square-root information, GNSS fixes with their re-weighted std, and the prior gvinsMarginalization just built.
 * `next` is the next window exactly as icg_ba_upload would take it; per window, `carry` names for every row of next its source row in the old
 * window, or -1 for a row read from next (a NULL map: no row of that kind is carried).  Carried value rows of next are not read.  The structure
 * (indices, f_active -- NULL: all active --, sizes, flags, ext, lever, first-window priors, the prior's block tables and x0) is read from next.
 * prior_from_marg = 1: the prior is the one the last icg_ba_marginalize_resident[_culled] call left for this window (it must be the last
 * marginalization on the handle, over the same n_windows, with no upload or slide since, and next.marg_r / marg_nblocks must be its r / nblocks);
 * 0: next.marg_J0 / marg_e0.  H0 = J0^T J0, b0 = J0^T e0, c0 = e0.e0 are formed on the device in icg_ba_upload's summation order.
 * Afterwards the handle is indistinguishable from one that called icg_ba_upload(next) with the carried values filled in: icg_ba_run[_gvins]
 * (restart included), icg_ba_download / icg_ba_gvins_optimization_end(next) and the resident calls give the same bits.  Every check (map ranges
 * against the old window, the upload's checks of next, a new blob's positive-definite covariance, the prior's origin) runs before the device is
 * written; a rejected call (ICG_EINVAL with a message) leaves the handle as it was.  n_windows must equal the uploaded count.  Asynchronous on the
 * handle's stream.  ICG_EUNSUPPORTED on a landmark-sharded handle: its group calls icg_ba_shard_slide_resident.
 */
typedef struct icg_ba_slide_window {
    const int32_t *node_src;  /* next.K: old node whose pose / mix carries over, or -1 (next.pose / next.mix row) */
    const int32_t *lm_src;    /* next.L: old landmark whose inverse depth carries over as 1.0 / (1.0 / rho), or -1 (next.invdepth) */
    const int32_t *f_src;     /* next.F: old reprojection factor whose 14 constants carry over, or -1 (next.f_const row) */
    const int32_t *imu_src;   /* next.n_imu: old IMU factor whose blob and square-root information carry over, or -1 (next.imu_blob row) */
    const int32_t *gnss_src;  /* next.n_gnss: old GNSS fix whose blh and current (re-weighted) std carry over, or -1 (next rows) */
    int32_t prior_from_marg;  /* 1: the prior the last icg_ba_marginalize_resident[_culled] call computed for this window;
                                 0: next.marg_* (J0 / e0 uploaded, H0 / b0 / c0 formed on the device) */
} icg_ba_slide_window;
int icg_ba_slide_resident(icg_ba *h, int n_windows, const icg_ba_problem *next, const icg_ba_slide_window *carry);
/*
 * icg_ba_slide_resident whose new IMU factors, new node states and aligned GNSS fixes are computed on the device from the states the handle
 * holds, instead of being preintegrated on the host and read from `next`: the host halves of the time-node edits between two solves,
 *   GVINS::addNewTimeNode (IG/ic_gvins.cc:897-928)        a new factor from the last node's state (NODE), the new node = its currentState();
 *   GVINS::removeUnusedTimeNode (:754-789)                 a merged factor: the first interval's start state replayed over the first interval's
 *                                                         rows followed by the second's without its first row (ROW);
 *   GVINS::insertNewGnssTimeNode (:791-888)                a fix moved onto a node, blh -= v dt / blh += v dt (alignment); or a node inserted at
 *                                                         the fix and the later nodes re-created, each interval from the state the previous
 *                                                         one propagated (NODE, then CHAIN).
 * Per window, only rows that `carry` marks -1 (or whose carry map is NULL) are read.  For an integrated factor k (joining new nodes k, k + 1):
 *   start  NODE i (>= 0): old node i's resident pose (q normalised as icg_ba_reintegrate_resident normalises it) and mix;  ICG_SLIDE_CHAIN:
 *          stateFromData(stateToData(currentState())) of factor k - 1 of the same window, which must be integrated too;  ICG_SLIDE_ROW:
 *          state16 row k as given (p, q_xyzw, v, bg, ba; not normalised)
 *   form   normal[k] (NULL: all PreintegrationEarth) and gravity3 row k; the Earth form takes iewn = Earth::iewn(station3, start p) as resetState
 *          does (preintegration_earth.cc:305-324), the Normal form iewn = 0
 *   rows   imu rows imu_off[k] .. imu_off[k + 1] - 1 (dt, dtheta[3], dvel[3]), row imu_off[k] the sample at the interval's start; at least one
 * Its blob and square-root information become new factor k's, as icg_ba_slide_resident would read them from next.imu_blob (the blob is
 * icg_imu_preintegrate's from the same start state, bit for bit).  A flagged new node j takes pose = (p, q) and mix = (v, bg, ba) of
 * stateToData(currentState()) of integrated factor j - 1 (bg, ba: its start state's).  An aligned new GNSS fix g takes
 * blh = next.gnss_blh[g] + dt v(old node), each component rounded on its own (blh - v |dt| bit for bit for dt < 0); its std is next's (the
 * caller applies the reference's x 1.2).  One warp per window walks the window's integrated factors in order.
 * Every check of icg_ba_slide_resident and of these arrays (sources and nodes in range, CHAIN after an integrated factor, offsets, flags)
 * runs before the device is written.  The integration then runs into the slide's staging, the call synchronises and, when an integrated
 * covariance is not positive definite, returns ICG_EINVAL naming the first such factor (window order, then factor order) with the handle as it
 * was; the outputs are written either way.  Otherwise the call goes on as icg_ba_slide_resident does (asynchronous from there).
 * ICG_EUNSUPPORTED on a landmark-sharded handle: its group calls icg_ba_shard_slide_integrate_resident.
 */
#define ICG_SLIDE_CHAIN (-2)
#define ICG_SLIDE_ROW (-3)
typedef struct icg_ba_slide_integrate {
    /* in: per new IMU factor (next.n_imu entries) */
    const int32_t *imu_from;      /* NULL: nothing integrated in this window.  -1: next.imu_blob row; i >= 0: NODE i; ICG_SLIDE_CHAIN; ICG_SLIDE_ROW */
    const double *state16;        /* n_imu x 16: the ICG_SLIDE_ROW start states (other rows not read; NULL when there is none) */
    const double *gravity3;       /* n_imu x 3 */
    const uint8_t *normal;        /* n_imu: 1 PreintegrationNormal, 0 PreintegrationEarth; NULL: all Earth */
    const double *imu;            /* rows (dt, dtheta[3], dvel[3]) */
    const int32_t *imu_off;       /* n_imu + 1 */
    /* in: per new node (next.K entries), NULL: none */
    const uint8_t *node_from_imu; /* 1: the node is currentState() of integrated factor j - 1 */
    /* in: per new GNSS fix (next.n_gnss entries), NULL: none */
    const int32_t *gnss_node;     /* -1: next.gnss_blh as given; i >= 0: aligned by old node i's velocity */
    const double *gnss_dt;        /* signed dt of the alignment (the reference's -dt for a fix moved back onto node index - 1) */
    /* out, each may be NULL */
    int8_t *status;               /* n_imu: 1 integrated, 0 not integrated, -1 integrated covariance not positive definite */
    double *blob_out;             /* n_imu x ICG_IMU_BLOB_DOUBLES: written where status != 0 */
    double *end_state10;          /* n_imu x 10: currentState() p, q_xyzw, v where status != 0 */
} icg_ba_slide_integrate;
int icg_ba_slide_integrate_resident(icg_ba *h, int n_windows, const icg_ba_problem *next, const icg_ba_slide_window *carry,
                                    const icg_ba_slide_integrate *integ, const double *noise5, const double *station3);
/*
 * icg_ba_slide_integrate_resident (integ NULL: icg_ba_slide_resident) whose vision rows are built on the device: GVINS::addReprojectionParameters
 * + addReprojectionFactors (IG/ic_gvins.cc:1697-1837) on the map after the culling and Map::removeKeyFrame(frame, true) (tracking/map.cc:89-125,
 * called at :1675), from the culled window the handle holds and the new keyframes' observations.  next.L, F, invdepth, f_lm / f_ref / f_obs /
 * f_const, f_active and carry.lm_src / f_src are NOT read: the call builds them.  Everything else of next and carry keeps its meaning.
 * The old window is the one the handle holds; the culling outcome is the last icg_ba_update_and_cull_resident on this handle, which must still be
 * current (no upload or slide since, the same n_windows): the handle keeps its landmark and observation flags on the device for this call.
 * Landmarks of the next window:
 *   carried first, in old order: landmark l is carried when it is not a culling outlier, its reference node (the culling's lm_ref_node) is
 *     >= num_marg, set in node_in_map and kept by carry.node_src, and its inverse depth 1.0 / (1.0 / rho) is not NaN (a NaN drops it and is counted
 *     in nan_dropped and flagged in nan_flags: the caller marks the map point an outlier); a 0 becomes 1 / 10 (MapPoint::DEFAULT_DEPTH): its
 *     row is then staged (lm_src -1) and lm_origin still names the old landmark;
 *   then the new map points in creation order, invdepth = 1.0 / depth under the same two rules.
 * Factors, landmark by landmark (f_lm non-decreasing):
 *   the landmark's surviving old factors in old order: the culling lists the factor's observation (obs_factor) and did not mark it an outlier,
 *     and its observing node is usable as above (the reference node never observes: the reference skips it).  The chi-square pass's removals
 *     come back: every factor of the next window is active;
 *   then its new observations in node order: pts0 / vel0 / td0 from the landmark's reference row, pts1 = pixel2cam(undis_xy) (geom_core, as
 *     icg_camera_pixel2cam), vel1 = (vx, vy, 0),
 *     td1 = node_td[node].  An observation of a landmark that is not carried, or in its reference node, is skipped;
 *   a new map point: one factor from its reference node (frame table) to cur_node, pts = pixel2cam of the two keypoints, vel = (v, 0), td from
 *     node_td; none when the two nodes are the same.
 * Reference rows.  The handle keeps every landmark's reference row (pts0, vel0, td0 = pixel2cam(referenceKeypoint()), the reference feature's
 * velocity, the reference frame's timeDelay()), so that a landmark whose factors were all dropped can still take a new observation:
 * icg_ba_upload sets it from the landmark's first factor (unknown, NaN, for a landmark uploaded without factors), every slide carries it with
 * the landmark (a landmark that carry.lm_src names keeps its old row; a new one takes its first factor's), and this call writes a new map
 * point's from its reference keypoint, velocity and node_td.  A new observation of a landmark whose row is unknown is ICG_EINVAL.
 * The reference's order is unordered_map iteration (implementation-defined); this order is fixed and only permutes rows.
 * One CTA per window builds the structure on the device; the counts, the integer structure, the new invdepth rows and the new factors' constants
 * come back in one copy (one synchronisation), and the call goes on as icg_ba_slide_integrate_resident with that window, every check included.
 * A rejected call (ICG_EINVAL: max_L / max_F exceeded, a reference frame id missing from the table, a node, landmark or source index out of
 * range, a count outside its list, two observations of one landmark in one node) leaves the handle as it was.  Afterwards the handle cannot be
 * told apart from one that called icg_ba_slide_integrate_resident with the same next whose vision rows were built on the host by these rules.
 * ICG_EUNSUPPORTED on a landmark-sharded handle: its group calls icg_ba_shard_slide_vision_resident.
 */
typedef struct icg_ba_slide_vision {
    /* in: the old window */
    int32_t num_marg;
    const uint8_t *node_in_map;  /* old K: isKeyFrameInMap after gvinsRemoveAllSecondNewFrame */
    const int32_t *obs_factor;   /* the culling's observations (its obs_off order): factor of each, -1 for none */
    /* in: the new keyframes */
    icg_camera cam;
    const double *node_td;       /* next.K: frame->timeDelay() */
    int32_t cur_node;            /* next-window node of the current frame */
    int32_t n_frames;            /* <= 64 */
    const int64_t *frame_id;     /* HOST n_frames: frame id -> */
    const int32_t *frame_node;   /* HOST n_frames:   next-window node */
    /* tracked map-point observations (DEVICE): k < count (*dev_n when dev_n is not NULL, else n_obs; a count outside [0, n_obs] is an error),
       j = obs_src ? obs_src[k] : k (< n_in): landmark obs_lm[j] (old landmark, -1: not in the window), node obs_node[j] (NULL: cur_node),
       undis_xy[2 k] (feat->keyPoint()), vel[2 k]; icg_klt_track_frames_dev's compacted map list plugs in with obs_src = its src and
       dev_n = dev_n_out + 2 s */
    int32_t n_obs, n_in;
    const int32_t *dev_n, *obs_src, *obs_lm, *obs_node;
    const float *obs_undis_xy;
    const double *obs_vel;
    /* new map points (DEVICE, icg_tri_new's arrays at the stream's offset): count *dev_new_n (dev_counts + 5 s + 1) or n_new */
    int32_t n_new;
    const int32_t *dev_new_n;
    const double *new_depth, *new_vel_ref, *new_vel_cur;
    const float *new_ref_undis_xy, *new_cur_undis_xy;
    const int64_t *new_ref_frame_id;
    /* out */
    int32_t L, F, nan_dropped;
    int32_t *lm_src, *f_src, *f_lm, *f_ref, *f_obs; /* HOST, each may be NULL: max_L / max_F entries (lm_src / f_src as carry takes them) */
    int32_t *lm_origin;                             /* HOST or NULL: max_L, every next landmark's origin: old landmark l, or -(j + 1) for new point j */
    uint8_t *nan_flags;                             /* HOST or NULL: old L + n_new, 1 where the landmark / new point was dropped for a NaN inverse
                                                       depth (the caller sets that MapPoint an outlier, IG/ic_gvins.cc:1720-1724) */
    double *invdepth;                               /* HOST or NULL: max_L, the landmarks' inverse depths (carried ones as the slide computes them) */
    double *f_const;                                /* HOST or NULL: max_F x 14, the rows of the new factors (f_src = -1); carried rows are not written */
} icg_ba_slide_vision;
int icg_ba_slide_vision_resident(icg_ba *h, int n_windows, const icg_ba_problem *next, const icg_ba_slide_window *carry,
                                 const icg_ba_slide_integrate *integ, const double *noise5, const double *station3, icg_ba_slide_vision *vis);
/*
 * The reintegration and the two slides on a landmark-sharded handle (world > 1): doReintegration (IG/ic_gvins.cc:1680-1695) and the time-node
 * edits and next window of gvinsOptimization (:754-928, 1697-1837), as icg_ba_reintegrate_resident, icg_ba_slide_resident and
 * icg_ba_slide_integrate_resident describe them, with the same structs.  Each is a COLLECTIVE call: every rank of the group calls it with its
 * own shard problems, the same number of times.  On a handle outside a shard group (world == 1) each returns ICG_EINVAL naming its plain call.
 *   Replicated / shard-local.  node_src, imu_src, gnss_src, prior_from_marg, the camera-side rows read from `next` (new pose / mix rows, new
 *     blobs, new GNSS rows, gnss_node, the prior's block tables and x0, marg_J0 / marg_e0 when prior_from_marg = 0), noise5, station3, every
 *     `integ` array and every icg_ba_reint_window must be the same on every rank.  lm_src and f_src name rows of the same rank's old shard (a
 *     landmark never changes rank across a slide); new landmarks go to whichever rank the caller puts them on.  Every next shard lists its
 *     factors landmark by landmark (f_lm non-decreasing), as the next sharded marginalization requires; a shard may be empty (L = 0).
 *   Redundant integration.  The reintegration and the slide's integration run on every rank from its replicated states with the same
 *     inputs, so every rank writes the same blobs, square-root information and node rows bit for bit; nothing is exchanged for them.
 *   The prior on its owner.  prior_from_marg = 1: the owner of window w (rank w mod world) forms H0 / b0 / c0 on the device from the J0 / e0
 *     that the last icg_ba_marginalize_resident[_culled] of the group left in the owner's gather handle.  That call must be the last
 *     marginalization of the handle, a sharded resident one over the same n_windows with no upload or slide since, and the owner checks
 *     next.marg_r / marg_nblocks against it.  The other ranks write zeros into that window's prior rows: nothing reads them there
 *     (ba_lin_cam and ba_cost_cam evaluate the prior factor under the owner gate of the camera-only factors, and the sharded marginalization's
 *     ba_marg_fill copies the prior from the owner's own handle).  prior_from_marg = 0: every rank forms it from next.marg_J0 / marg_e0, as
 *     icg_ba_upload does.
 *   Agreement before any write.  Each rank runs every check of the plain call, the ones above and its owner checks, then joins one integer
 *     exchange of the group: its verdict and a 31-bit fingerprint of its camera-side arguments.  When any rank rejected, or the fingerprints
 *     differ, EVERY rank returns ICG_EINVAL with its handle as it was, naming the rejecting rank or saying that the ranks' camera sides differ
 *     (a rejecting rank keeps its own message; a failed allocation or CUDA call before the agreement is a rejection like any other).
 *     The integrating slide exchanges its positive-definiteness outcome once more before the device is written.  A rank's own argument error therefore never leaves its peers to the bounded waits of the exchange; only a rank
 *     that does not make the call does.  The sharded slide synchronises for the agreement (the plain slide stays asynchronous).
 *   Contract.  After icg_ba_shard_slide[_integrate]_resident the group cannot be told apart from one whose ranks each called icg_ba_upload on
 *     their next shards with the carried values filled in -- blobs as icg_imu_preintegrate gives them from the same start states, and the
 *     owner's J0 / e0 as the prior --, for every later call (icg_ba_run_gvins with restart, icg_ba_gvins_optimization_end, the sharded
 *     culling and marginalizations, the next sharded slide), except for the non-owners' prior rows, which nothing reads.
 */
int icg_ba_shard_reintegrate_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const double *noise5, const double *station3,
                                      icg_ba_reint_window *io);
int icg_ba_shard_slide_resident(icg_ba *h, int n_windows, const icg_ba_problem *next, const icg_ba_slide_window *carry);
int icg_ba_shard_slide_integrate_resident(icg_ba *h, int n_windows, const icg_ba_problem *next, const icg_ba_slide_window *carry,
                                          const icg_ba_slide_integrate *integ, const double *noise5, const double *station3);
/*
 * icg_ba_slide_vision_resident on a landmark-sharded handle: each rank builds its own next shard's landmarks and reprojection factors on the
 * device, from its own old shard and its own culling, then slides as icg_ba_shard_slide[_integrate]_resident (integ NULL or not), with every
 * rule above.  A COLLECTIVE call, with the structs of the plain call.
 *   What each rank passes.  Its own next shard problems and carry maps; next.L, F, f_* and carry.lm_src / f_src are built, not read.
 *     vis[w].obs_factor is the table the rank's own sharded culling took (shard_cull_inputs' obs_factor); vis[w].obs_lm names rows of the
 *     rank's own OLD shard, -1 for a map point the rank does not hold.  The lists are otherwise the same on every rank (the same tracked
 *     observations, the same new map points), and every device array must be readable from the rank's own device.
 *   Old landmarks.  A carried landmark stays on the rank that held it; each rank applies the plain call's rules to its shard: the carry rule,
 *     the surviving factors, the new observations in node order.
 *   New map points.  New point j of window w (creation order) goes to rank (j + w) mod world.  The rule is fixed: the count lives on the
 *     device, so the caller could not place points itself without a host round trip.
 *   Order.  Each rank's next shard holds its carried landmarks in old shard order, then its new points in creation order; factors landmark
 *     by landmark.  The next whole window written rank-major is exactly what icg_ba_slide_vision_resident builds from the merged old window,
 *     reordered rank-major (new points by the rule above, a carried landmark staged for a zero depth -- lm_src -1, lm_origin >= 0 -- on its
 *     old rank).
 *   Outputs, per rank.  L, F, nan_dropped of the rank's shard; lm_src / f_src local to the shard, as carry takes them; lm_origin: the old
 *     shard-local landmark, or -(j + 1) for global new point j; nan_flags: the old shard's L entries, then all n_new entries, a new point
 *     flagged on its own rank only (OR the ranks together).
 *   Agreement.  Each rank folds num_marg, node_in_map, cam, node_td, cur_node, the frame table, n_obs / n_new and the observation and
 *     new-point counts its build read on the device into the fingerprint of the slide's one agreement.  One rejection on any rank (capacity
 *     on the rank that received the new points, no current culling, every build error of the plain call) or a fingerprint mismatch makes
 *     EVERY rank return ICG_EINVAL with its handle as it was.  On a handle outside a shard group: ICG_EINVAL naming
 *     icg_ba_slide_vision_resident.
 */
int icg_ba_shard_slide_vision_resident(icg_ba *h, int n_windows, const icg_ba_problem *next, const icg_ba_slide_window *carry,
                                       const icg_ba_slide_integrate *integ, const double *noise5, const double *station3,
                                       icg_ba_slide_vision *vis);
/*
 * Landmark sharding of the window solve across the GPUs of one box (SURVEY.md 8e), over PEER MEMORY (transport "p2p"): every process
 * (one per GPU) uploads the same camera-side problem but only ITS landmarks and their reprojection factors; window w of the batch is
 * owned by rank w mod world.  Every rank STORES its packed reduction operand straight into the owner's inbox over NVLink; the owner sums
 * the `world` slots in rank order while assembling the reduced camera system (the reduction is fused into the consumer, no collective
 * kernel), solves it on a thread-block cluster and stores the camera step into every rank's step buffer; a 5-scalar all-to-all closes
 * the attempt.  Camera-only factors (IMU, GNSS, priors) are evaluated by the window's owner.  Three release/acquire flag
 * synchronisations per LM attempt, no host round trip, deterministic (fixed summation order, independent of arrival order).
 *   icg_ba_shard_export : allocates this rank's exchange buffer for a group of `world` ranks (<= 8, one box) and writes the
 *                         ICG_SHARD_BLOB_BYTES blob the other ranks need (CUDA IPC handle + process-local pointer);
 *   icg_ba_shard_connect: blobs = world x ICG_SHARD_BLOB_BYTES in rank order (the caller gathers them, e.g. torch.distributed
 *                         all_gather_object); handles living in the same process are connected by pointer (peer access enabled);
 *   icg_ba_shard_error  : non-zero if a flag wait timed out (a rank did not enqueue the same sequence);
 *   icg_ba_shard_leave  : releases the group's exchange buffers and returns the handle to the pipeline its window size selects on this
 *                         GPU alone (the fused single-GPU pipeline, or the split pipeline when the reduced system does not fit one CTA).
 * All ranks must create their handles with the same max_windows and max_K and call the solve entry points with the same arguments.
 */
#define ICG_SHARD_BLOB_BYTES 128
int icg_ba_shard_export(icg_ba *h, int rank, int world, uint8_t *blob);
int icg_ba_shard_connect(icg_ba *h, const uint8_t *blobs);
int icg_ba_shard_error(icg_ba *h);
int icg_ba_shard_leave(icg_ba *h);
/* Problem::EvaluateResidualBlock(id, false, &cost, NULL, NULL) for every reprojection / GNSS block
 * (the two chi-square passes, IG/ic_gvins.cc:1251,1278): cost = 0.5 |r|^2 without the loss function. */
int icg_ba_residual_costs(icg_ba *h, const icg_ba_problem *problem, double *reproj_cost /* F */, double *gnss_cost /* n_gnss */);
/* Single-factor evaluation with the Ceres CostFunction::Evaluate contract (IG/factors/reprojection_factor.h:55):
 * residuals[2]; jacobians row-major 2x7, 2x7, 2x7, 2x1, 2x1 (any may be NULL).  Computed on the device. */
int icg_ba_reproj_evaluate(icg_ba *h, const double *pose0, const double *pose1, const double *ext, const double *invdepth,
                           const double *td, const double *f_const14, double std, double *residuals, double **jacobians);
/* The same factor in the node-frame form ba_lin_vis and ba_cost run: R = toRotationMatrix(q) of both poses and the extrinsic (node_frame),
 * R^T in place of each quaternion inverse (reproj_eval_frames).  Same arguments and outputs as icg_ba_reproj_evaluate. */
int icg_ba_reproj_evaluate_frames(icg_ba *h, const double *pose0, const double *pose1, const double *ext, const double *invdepth,
                                  const double *td, const double *f_const14, double std, double *residuals, double **jacobians);
/* PreintegrationFactor::Evaluate (IG/preintegration/preintegration_factor.h:45): residuals[15], jacobians 15x7,15x9,15x7,15x9 */
int icg_ba_imu_evaluate(icg_ba *h, const double *imu_blob, const double *pose0, const double *mix0, const double *pose1,
                        const double *mix1, double *residuals, double **jacobians);

/* The remaining CostFunction::Evaluate seams of the window graph (same contract: residuals, then one row-major Jacobian per parameter
 * block with its GLOBAL size, any may be NULL; computed on the device):
 *   GnssFactor::Evaluate            (IG/factors/gnss_factor.h:43-71)                 residuals[3], jacobians[0] 3x7
 *   ImuPosePriorFactor::Evaluate    (IG/preintegration/imu_pose_prior_factor.h:42-68) residuals[6], jacobians[0] 6x7
 *   ImuMixPriorFactor::Evaluate     (IG/preintegration/imu_mix_prior_factor.h:40-75)  residuals[9], jacobians[0] 9x9
 *   ImuErrorFactor::Evaluate        (IG/preintegration/imu_error_factor.h:45-91)      residuals[6], jacobians[0] 6x9
 *   MarginalizationFactor::Evaluate (IG/factors/marginalization_factor.h:47-101)      residuals[r], jacobians[b] r x (7 | 9 | 7 | 1);
 *       parameters[b] = the current value of remained block b (block_type as in icg_ba_problem.marg_block_type), x0 / J0 / e0 the prior. */
int icg_ba_gnss_evaluate(icg_ba *h, const double *pose, const double *blh, const double *std3, const double *lever, double *residuals,
                         double **jacobians);
int icg_ba_pose_prior_evaluate(icg_ba *h, const double *pose, const double *prior7, const double *std6, double *residuals, double **jacobians);
int icg_ba_mix_prior_evaluate(icg_ba *h, const double *mix, const double *prior9, const double *std9, double *residuals, double **jacobians);
int icg_ba_imu_error_evaluate(icg_ba *h, const double *mix, double *residuals, double **jacobians);
int icg_ba_marg_factor_evaluate(icg_ba *h, int r, int nblocks, const int32_t *block_type, const double *const *parameters, const double *x0,
                                const double *J0, const double *e0, double *residuals, double **jacobians);

/* ===================================================================================================== *
 *  INS windows: the per-stream IMU recurrence that gives every frame its prior camera pose
 * ===================================================================================================== */
/* One handle holds max_streams INS windows (GVINS::ins_window_, IG/ic_gvins.h), each a ring of `capacity` entries on the device.  An entry
 * is one IMU row (time, dt, dtheta[3], dvel[3]) and the state after it (time, p[3], q_xyzw[4], v[3], bg[3], ba[3]).  The handle mirrors each
 * stream's count, last sample time and "mechanized" flag on the host, so every check of icg_ins_push runs before the device is written.
 * A stream is "mechanized" from its first icg_ins_redo or icg_ins_gins_initialize with status 1 on (GVINS::gvinsInitialization followed
 * by the redo at IG/ic_gvins.cc:301-306 and :683); before that its pushes take runFusion's initialization path.
 * capacity is in [1000, 65536]: 1000 = MAXIMUM_INS_NUMBER (IG/ic_gvins.h:124), the most an unmechanized window holds; up to 65537 entries the
 * binary search of getInsWindowIndex (misc.cc:30-65) ends within the 16 halvings its `counts++ > 15` cap allows, so the cap never triggers. */
typedef struct icg_ins icg_ins;
typedef struct icg_ins_config { /* integration_config_ (IG/ic_gvins.cc:99-106, 675-678), one per stream */
    int32_t with_earth;         /* iswithearth: the Earth form of insMechanization (Coriolis, gravity, Earth rotation) or the Normal form */
    double gravity[3];          /* (0, 0, g) */
    double iewn[3];             /* Earth::iewn(origin, p) set at initialization; unused when with_earth == 0 */
} icg_ins_config;
int icg_ins_create(icg_ins **h, int max_streams, int capacity, int device, void *stream);
void icg_ins_destroy(icg_ins *h);
/* runFusion's per-sample step (IG/ic_gvins.cc:249-293) for streams 0 .. n_streams-1: rows off[s] .. off[s+1]-1 of imu (HOST, 8 doubles per
 * row: time, dt, dtheta[3], dvel[3]) belong to stream s, cfg (HOST) holds n_streams configurations.
 *   mechanized stream: each row is insMechanization(imu_pre = the window's last row, imu_cur = the row) (misc.cc:151-206) from the window's
 *                      last state, and the state is stored with the row (:284-286);
 *   otherwise:         the row is appended with a zero state and the window keeps its newest 1000 rows (:288-293).
 * The reference redoes instead of mechanizing the one sample that arrives while isoptimized_ is set (:272-280).  A push followed by
 * icg_ins_redo gives the same window, because the redo rewrites every state from its index on.
 * ICG_EINVAL, before anything is launched and with every window unchanged: a row time not greater than the stream's previous one, or a
 * mechanized stream that would exceed capacity (the reference's window only shrinks at a redo).  Asynchronous. */
int icg_ins_push(icg_ins *h, int n_streams, const icg_ins_config *cfg, const int32_t *off, const double *imu);
/* redoInsMechanization (misc.cc:208-261) of streams 0 .. n_streams-1 from state17 (HOST, n x 17: time, p, q_xyzw, v, bg, ba =
 * statedatalist_.back(); q is normalised as stateFromData does, preintegration_base.cc:115-125).  redo (HOST, n; NULL: all) selects streams.
 * The window is re-mechanized from getInsWindowIndex(state time) with isNeedInterpolation's four cases (:229-242; MINIMUM_TIME_INTERVAL =
 * 1e-4), then index - reserved entries are dropped from the front when index >= reserved (:253-260; the reference's reserved_ins_num_ is 2,
 * IG/ic_gvins.cc:82).  status (HOST, n): 1 redone, 0 not selected, -1 index == 0 (the reference logs and leaves the window unchanged).
 * Synchronous. */
int icg_ins_redo(icg_ins *h, int n_streams, const icg_ins_config *cfg, const uint8_t *redo, const double *state17, int reserved, int8_t *status);
/* GVINS::gvinsInitialization (IG/ic_gvins.cc:584-692), which the fusion thread retries at every GNSS epoch while a stream is initializing
 * (:297-312), for the selected streams of 0 .. n_streams-1.  in (HOST, n) holds the members it reads; cfg (HOST, n) is read and, for the
 * streams that initialize, receives gravity = (0, 0, g) and, in the Earth form, iewn = Earth::iewn(origin, p) (:675-678).
 *   1 the rows with last_time < t < gnss_time (both strict, :592-598); fewer than 20: status -2.  A time of 0: status -1.
 *   2 MISC::detectZeroVelocity (misc.cc:363-415) on them, sums in row order; at zero velocity bg = mean(dtheta) rate, roll = -asin(fb_y / g),
 *     pitch = asin(fb_x / g) go to the stream's slots, which then has a zero-velocity detection, and the status is -3 (:648-650).
 *   3 heading: the dual-antenna yaw when last_yaw_valid, else atan2 of the GNSS displacement (|d| < 0.5 m: status -4), with roll = 0 and pitch
 *     from the displacement when the stream has had no zero-velocity detection.
 *   4 state17[0] = (last_time, last_blh - q antlever, q = euler2quaternion(initatt), v = 0, bg, ba = 0) and constructPrior (:1911-1936:
 *     gyroscope bias std 3 noise5[2] after a zero-velocity detection, else 7200 deg/h; accelerometer bias std 20000 mGal).
 *   5 the redo of icg_ins_redo from state17[0] with `reserved`; the stream becomes mechanized.
 *   6 addNewGnssTimeNode's factor (:889-928): getImuSeriesFromTo(last_time, gnss_time) (misc.cc:307-361) on the redone window, preintegrated
 *     from state17[0] with noise5 / station3 as icg_ba_slide_integrate_resident forms a new node's factor; state17[1] = its end state at
 *     gnss_time.  The reference then sets isoptimized_ (:302-306): its next IMU sample redoes the window again from state17[1]
 *     (:272-280), which the caller binds as icg_ins_push followed by icg_ins_redo with state17[1].
 * Status -5: the window cannot serve the redo and the series (getInsWindowIndex == 0 at either end, or an empty series).  It is decided
 * before anything is written, so the window, the mechanized flag and the slots stay as they were; the reference logs and indexes an empty
 * series there instead.  The slots (bg, initatt, has_zero_velocity) are the reference's function statics, which every GVINS object of a
 * process shares: with one GVINS per process, one set per stream is the equivalent.  icg_ins_create zeroes them.
 * ICG_EINVAL, with every stream unchanged: bad arguments, a bad configuration, or a selected stream that is already mechanized.  sel (HOST,
 * n; NULL: all).  noise5 (HOST) = gyr_arw, acc_vrw, gyr_bias_std, acc_bias_std, corr_time; station3 (HOST) = parameters_->station.
 * out (HOST, n): every stream's slots; the rest for status 1 only.  Synchronous. */
typedef struct icg_gins_init { /* per stream: the GVINS members gvinsInitialization reads */
    double gnss_time, gnss_blh[3], gnss_std[3]; /* gnss_, blh local (Earth::global2local in addNewGnss, IG/ic_gvins.cc:199-220) */
    double last_time, last_blh[3], last_std[3]; /* last_gnss_ */
    int32_t last_yaw_valid;                     /* last_gnss_.isyawvalid (dual antenna) */
    double last_yaw;                            /* last_gnss_.yaw */
    double origin_blh[3];                       /* integration_config_.origin (the Earth form's iewn) */
    double gravity;                             /* integration_parameters_->gravity = Earth::gravity(origin) */
    double antlever[3], imudatarate;
} icg_gins_init;
typedef struct icg_gins_init_out {
    int32_t status;            /* 1 initialized; 0 not selected; -1 .. -5 as above */
    int32_t has_zero_velocity; /* the slot after the call */
    double bg[3], initatt[3];  /* the slots after the call */
    double state17[2 * 17];    /* statedatalist_[0] (last_time) and [1] (gnss_time) */
    double pose_prior[7], pose_prior_std[6], mix_prior[9], mix_prior_std[9]; /* constructPrior */
    double imu_blob[ICG_IMU_BLOB_DOUBLES];                                   /* the first GNSS time node's factor */
    int32_t n_series;          /* rows of its series */
} icg_gins_init_out;
int icg_ins_gins_initialize(icg_ins *h, int n_streams, icg_ins_config *cfg, const uint8_t *sel, const icg_gins_init *in, const double *noise5,
                            const double *station3, int reserved, icg_gins_init_out *out);
/* getCameraPoseFromInsWindow (misc.cc:67-108; called at IG/ic_gvins.cc:527-533) of streams 0 .. n_streams-1 at stamp[s] = frame->stamp()
 * + td (HOST), with pose_b_c (HOST, n x 12: R row-major, t).  dev_pose (DEVICE, n x 12): Pose::R row-major, Pose::t, as icg_track_frame
 * takes them.  host_pose (HOST or NULL: then the call is asynchronous and nothing is copied back) receives the same values.  found (HOST when
 * host_pose is given, else DEVICE, or NULL): 1 interpolated, 0 outside the window (the back state's pose, the reference's `false`), -1 the
 * window was never mechanized (pose not written). */
int icg_ins_camera_pose(icg_ins *h, int n_streams, const double *stamp, const double *pose_b_c, double *dev_pose, double *host_pose,
                        int32_t *found);
/* One stream's window, oldest first (tests, and the navigation output of ins_window_.back(), IG/ic_gvins.cc:382-389): *count receives the
 * window's size, the first min(count, cap) entries go to imu8 (HOST, cap x 8) and state17 (HOST, cap x 17).  Synchronous. */
int icg_ins_window(icg_ins *h, int stream, int cap, int32_t *count, double *imu8, double *state17);
int icg_ins_sync(icg_ins *h);

/* ===================================================================================================== *
 *  Every IMU factor's samples on the device: the window solver's sample store, filled from the INS windows
 * ===================================================================================================== */
/*
 * The reference keeps each factor's imu_buffer_ (PreintegrationBase) from the moment its interval is cut, MISC::getImuSeriesFromTo (misc.cc:
 * 307-361) on ins_window_, for two later readers: the merge of removeUnusedTimeNode (IG/ic_gvins.cc:754-789) and doReintegration (:1680-1695).
 * An icg_ba handle keeps the same rows on the device, per resident window and factor, so that a caller whose samples live in icg_ins windows
 * needs no host copy of them.  The store is filled only by the two calls below that cut from the INS windows; icg_ba_upload and every other
 * slide replace the factors and leave the handle without samples (bookkeeping only).  A call builds the next store in a second buffer and
 * swaps only when it commits, so a rejected call leaves the store as it was.
 * The series cut is getImuSeriesFromTo(start, end) exactly (both getInsWindowIndex, the four isNeedInterpolation cases at each end with
 * MINIMUM_TIME_INTERVAL = 1e-4, imuInterpolation's split, the middle rows), on the window as the INS handle holds it when the call runs.  An
 * interval the window cannot serve -- getInsWindowIndex 0 at either end, or an empty series, the rule of icg_ins_gins_initialize's status -5
 * -- is refused.
 * Ordering.  The solver's stream waits for an event recorded on the INS handle's stream (pushes and redos queued before the call are seen), and
 * each call synchronises before it returns, so a later icg_ins_push / icg_ins_redo cannot overwrite rows it reads.  The two handles must be on
 * one device.  Every check (streams in range and mechanized, node_time increasing, merge_src in range with both sources holding samples, the
 * NULL rows) runs before anything is written; a rejected call leaves the handle, its store and the INS windows as they were.
 * Landmark-sharded handles: ICG_EUNSUPPORTED for all four calls.
 */
typedef struct icg_ba_ins_cut {
    int32_t stream;          /* the window's INS stream */
    const double *node_time; /* next.K: timelist_; factor k is getImuSeriesFromTo(node_time[k], node_time[k + 1]) */
} icg_ba_ins_cut;
/* Seeds the store of n_windows (the uploaded count) resident windows: every IMU factor k of window w from cut[w].  Call it right after the
 * upload of a window whose INS window still covers the window's span.  After icg_ins_gins_initialize and the upload of the K = 2 GINS window
 * (gvinsInitializationOptimization), that is before the next icg_ins_redo, which prunes the first interval out of the INS window.  Synchronous. */
int icg_ba_imu_samples_from_ins(icg_ba *h, icg_ins *ins, int n_windows, const icg_ba_ins_cut *cut);
/* icg_ba_slide_integrate_resident (vis NULL) or icg_ba_slide_vision_resident (vis given, its vision build exactly) whose integrated factors'
 * rows come from the device.  Per new IMU factor k of window w:
 *   NODE / ICG_SLIDE_CHAIN     getImuSeriesFromTo(node_time[k], node_time[k + 1]) cut from INS stream `stream` (addNewTimeNode, :897-928;
 *                              the re-created tail of insertNewGnssTimeNode, :791-888);
 *   ICG_SLIDE_ROW              old factor merge_src[k]'s stored rows, then old factor merge_src[k] + 1's without its first row
 *                              (removeUnusedTimeNode's addNewImu loop);
 *   carried (imu_src >= 0)     its stored rows carry over (none when the handle holds no samples);
 *   read from next.imu_blob    no samples.
 * Everything after the rows is icg_ba_slide_integrate_resident's path, on the same kernels; the handle is bit for bit the one that call leaves
 * when it is given the same rows from the host.  integ.imu / imu_off must be NULL; its other fields keep their meaning.  An interval the INS
 * window cannot serve: ICG_EINVAL naming the window and factor, integ.status -2 there (0 elsewhere), and the handle, its store and the INS
 * windows as they were.  Order of the checks: the call's own (streams, node_time, merge_src, the NULL rows) run first, then the cut (into
 * staging only, one launch and one synchronisation), then every check of icg_ba_slide_integrate_resident / icg_ba_slide_vision_resident;
 * so an interval the window cannot serve is reported ahead of those, and a call they reject has run the cut.  Nothing the handle, its store
 * or the INS windows hold is written before every check has passed.  Synchronous. */
typedef struct icg_ba_slide_ins {
    icg_ba_slide_integrate integ; /* imu / imu_off NULL */
    int32_t stream;               /* the window's INS stream (read when a factor is cut) */
    const double *node_time;      /* next.K: the next window's timelist_ (read when a factor is cut) */
    const int32_t *merge_src;     /* next.n_imu: read for ICG_SLIDE_ROW factors */
    int32_t *n_rows;              /* out, next.n_imu or NULL: every new factor's stored rows, -1 for none */
} icg_ba_slide_ins;
int icg_ba_slide_ins_resident(icg_ba *h, icg_ins *ins, int n_windows, const icg_ba_problem *next, const icg_ba_slide_window *carry,
                              const icg_ba_slide_ins *io, const double *noise5, const double *station3, icg_ba_slide_vision *vis);
/* icg_ba_reintegrate_resident with every factor's rows from the store: io[w].imu / imu_off must be NULL.  The same gate, replay and
 * replacement on the same kernel; a window with reintegrate = 1 that holds a factor without samples is refused before any launch, as is a
 * handle without a store.  The stored rows do not change (the reference's imu_buffer_ does not either).  Synchronous. */
int icg_ba_reintegrate_stored_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const double *noise5, const double *station3,
                                       icg_ba_reint_window *io);
/* Download of one resident window's stored rows (HOST): off (n_imu + 1): factor k's first row in rows, or -1 for a factor without samples;
 * off[n_imu] = the window's rows.  A factor's rows run to the next non-negative offset.  The first min(total, cap_rows) rows go to rows
 * (cap_rows x 7).  Synchronous. */
int icg_ba_imu_samples(icg_ba *h, int window, int cap_rows, int32_t *off, double *rows);

#ifdef __cplusplus
}
#endif
#endif /* ICGVINS_B200_H */
