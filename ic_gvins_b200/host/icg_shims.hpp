// icg_shims.hpp -- header-only C++ shims that keep the reference's call signatures and forward to the C ABI
// (include/icgvins_b200.h).  A maintainer includes this in IG/tracking/tracking.cc and IG/ic_gvins.cc; see INTEGRATION.md.
//
// When OpenCV headers are present the shims take cv:: types; otherwise (this image has no OpenCV C++ headers) minimal
// stand-ins with the same data layout are used so that the header still compiles and can be unit-tested.
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/icgvins_b200.h"

#if __has_include(<opencv2/core.hpp>)
#include <opencv2/core.hpp>
namespace icg_b200 {
using Point2f = cv::Point2f;
using Mat = cv::Mat;
using Size = cv::Size;
using TermCriteria = cv::TermCriteria;
inline const uint8_t *mat_data(const Mat &m) { return m.data; }
inline int mat_stride(const Mat &m) { return (int) m.step; }
inline int mat_cols(const Mat &m) { return m.cols; }
inline int mat_rows(const Mat &m) { return m.rows; }
}  // namespace icg_b200
#else
namespace icg_b200 {
struct Point2f {
    float x, y;
};
struct Size {
    int width, height;
    Size(int w = 0, int h = 0) : width(w), height(h) {}
};
struct TermCriteria {
    enum { COUNT = 1, EPS = 2 };
    int type, maxCount;
    double epsilon;
    TermCriteria(int t = 3, int c = 30, double e = 0.01) : type(t), maxCount(c), epsilon(e) {}
};
struct Mat {  // 8-bit single channel view
    const uint8_t *data;
    int rows, cols, step;
};
inline const uint8_t *mat_data(const Mat &m) { return m.data; }
inline int mat_stride(const Mat &m) { return m.step; }
inline int mat_cols(const Mat &m) { return m.cols; }
inline int mat_rows(const Mat &m) { return m.rows; }
}  // namespace icg_b200
#endif

namespace icg_b200 {

inline void check(int rc, const char *what) {
    if (rc != ICG_OK) throw std::runtime_error(std::string(what) + ": " + icg_last_error());
}

// One tracker per Tracking object (single tracking thread, IG/ic_gvins.cc:535).
class KltContext {
public:
    KltContext(int width, int height, int max_points = 4096, int device = 0) { check(icg_klt_create(&h_, width, height, 4, max_points, device, nullptr), "icg_klt_create"); }
    ~KltContext() { icg_klt_destroy(h_); }
    KltContext(const KltContext &) = delete;
    KltContext &operator=(const KltContext &) = delete;

    // cv::calcOpticalFlowPyrLK(prev, next, prevPts, nextPts, status, err, winSize, maxLevel, criteria, flags)
    // exactly as called at IG/tracking/tracking.cc:385,390,487,493.
    void calcOpticalFlowPyrLK(const Mat &prev, const Mat &next, const std::vector<Point2f> &prevPts, std::vector<Point2f> &nextPts,
                              std::vector<uint8_t> &status, std::vector<float> &err, Size winSize, int maxLevel, TermCriteria criteria, int flags) {
        const int n = (int) prevPts.size();
        if (!(flags & ICG_OPTFLOW_USE_INITIAL_FLOW)) nextPts = prevPts;
        nextPts.resize(n);
        status.resize(n);
        err.resize(n);
        // OpenCV's defaults for a criterion the type leaves out: 30 iterations, epsilon 0.01
        const int max_iter = (criteria.type & 1) ? criteria.maxCount : 30;
        const double eps = (criteria.type & 2) ? criteria.epsilon : 0.01;
        check(icg_klt_calc_optical_flow_pyr_lk(h_, mat_data(prev), mat_data(next), mat_stride(prev), reinterpret_cast<const float *>(prevPts.data()),
                                               reinterpret_cast<float *>(nextPts.data()), status.data(), err.data(), n, winSize.width, maxLevel, max_iter, eps,
                                               flags),
              "icg_klt_calc_optical_flow_pyr_lk");
    }

    // The whole forward + backward + gate block of Tracking::trackMappoint (IG/tracking/tracking.cc:385-403):
    // status[k] = st_fwd && st_bwd && !isOnBorder(fwd) && ptsDistance(bwd, prev) < 0.5
    void trackForwardBackward(const Mat &prev, const Mat &next, const std::vector<Point2f> &prevPts, std::vector<Point2f> &nextPts, std::vector<uint8_t> &status) {
        const int n = (int) prevPts.size();
        nextPts.resize(n);
        status.resize(n);
        check(icg_klt_track_fb(h_, mat_data(prev), mat_data(next), mat_stride(prev), reinterpret_cast<const float *>(prevPts.data()),
                               reinterpret_cast<float *>(nextPts.data()), nullptr, status.data(), n),
              "icg_klt_track_fb");
    }

    // Tracking::trackMappoint (IG/tracking/tracking.cc:351-455) from the prediction to the parallax, one call (icg_klt_track_frame with an
    // empty reference list).  Inputs in the order :357-370 gathers them: pts2d_map (distortedKeyPoint), pts2d_map_undis (keyPoint),
    // pw_xyz (mappoint->pos(), 3 doubles per point), ref_kp (the map point's keyPoint() in frame_ref_, NaN when it has none).  p: poses,
    // camera, dt (prev_slot / cur_slot are set here: the two frames are uploaded into slots 0 and 1).  Outputs: pts2d_matched /
    // pts2d_matched_undis / velocity_xy (2 doubles per point) of the survivors, src = their input indices (reduce mappoint_matched_ and
    // mappoint_type with it).  parallax_map / parallax_map_counts are updated as :416-417 and :450 do and left alone when the reference
    // returns before (:372-375).  Returns the reference's return value.
    bool trackMappoint(const Mat &pre, const Mat &cur, icg_track_frame p, const std::vector<Point2f> &pts2d_map, const std::vector<Point2f> &pts2d_map_undis,
                       const std::vector<double> &pw_xyz, const std::vector<Point2f> &ref_kp, std::vector<Point2f> &pts2d_matched,
                       std::vector<Point2f> &pts2d_matched_undis, std::vector<double> &velocity_xy, std::vector<int32_t> &src, double &parallax_map,
                       int &parallax_map_counts) {
        const int n = (int) pts2d_map.size();
        upload(pre, cur, p);
        std::vector<Point2f> fwd(n), fwd_undis(n);
        std::vector<uint8_t> keep(n);
        pts2d_matched.resize(n), pts2d_matched_undis.resize(n), velocity_xy.resize(2 * (size_t) n), src.resize(n);
        icg_track_map m{reinterpret_cast<const float *>(pts2d_map.data()), reinterpret_cast<const float *>(pts2d_map_undis.data()), pw_xyz.data(),
                        reinterpret_cast<const float *>(ref_kp.data()), reinterpret_cast<float *>(fwd.data()), reinterpret_cast<float *>(fwd_undis.data()),
                        keep.data(), reinterpret_cast<float *>(pts2d_matched.data()), reinterpret_cast<float *>(pts2d_matched_undis.data()), velocity_xy.data(),
                        src.data()};
        int32_t n_out[2];
        double par[2];
        int32_t par_n[2];
        check(icg_klt_track_frame(h_, &p, n, &m, 0, nullptr, n_out, par, par_n), "icg_klt_track_frame");
        pts2d_matched.resize(n_out[0]), pts2d_matched_undis.resize(n_out[0]), velocity_xy.resize(2 * (size_t) n_out[0]), src.resize(n_out[0]);
        if (par_n[0] >= 0) parallax_map = par[0], parallax_map_counts = par_n[0];
        return n_out[0] > 0;
    }

    // Tracking::trackReferenceFrame (IG/tracking/tracking.cc:457-574), one call (icg_klt_track_frame with an empty map list).  pts2d_new,
    // pts2d_ref, ref_frame_id (pts2d_ref_frame_[k]->id()) and velocity_ref (2 doubles per point) are reduced in place as :507-511 and
    // :550-554 reduce them, and pts2d_new becomes pts2d_cur_ (:569); src = the input index of every survivor (reduce pts2d_ref_frame_ with it);
    // velocity_cur (2 doubles per point) = velocity_cur_.  parallax_ref / parallax_ref_counts are left alone when the reference returns before
    // computing them (:459-462, :513-517).  Returns the reference's return value.  One corner differs: when the RANSAC rejects every survivor,
    // the reference returns at :557-561 with pts2d_new_ still the gate-reduced list; here pts2d_new comes back empty like pts2d_ref.
    bool trackReferenceFrame(const Mat &pre, const Mat &cur, icg_track_frame p, std::vector<Point2f> &pts2d_new, std::vector<Point2f> &pts2d_ref,
                             std::vector<int64_t> &ref_frame_id, std::vector<double> &velocity_ref, std::vector<double> &velocity_cur, std::vector<int32_t> &src,
                             double &parallax_ref, int &parallax_ref_counts) {
        const int n = (int) pts2d_new.size();
        upload(pre, cur, p);
        std::vector<Point2f> fwd(n), fwd_undis(n), cur_pts(n), cur_undis(n), ref_out(n);
        std::vector<uint8_t> keep(n);
        std::vector<int64_t> id_out(n);
        std::vector<double> vref_out(2 * (size_t) n);
        velocity_cur.resize(2 * (size_t) n), src.resize(n);
        icg_track_ref r{reinterpret_cast<const float *>(pts2d_new.data()), reinterpret_cast<const float *>(pts2d_ref.data()), ref_frame_id.data(),
                        velocity_ref.data(), reinterpret_cast<float *>(fwd.data()), reinterpret_cast<float *>(fwd_undis.data()), keep.data(),
                        reinterpret_cast<float *>(cur_pts.data()), reinterpret_cast<float *>(cur_undis.data()), velocity_cur.data(),
                        reinterpret_cast<float *>(ref_out.data()), id_out.data(), vref_out.data(), src.data()};
        int32_t n_out[2];
        double par[2];
        int32_t par_n[2];
        check(icg_klt_track_frame(h_, &p, 0, nullptr, n, &r, n_out, par, par_n), "icg_klt_track_frame");
        const int k = n_out[1];
        cur_pts.resize(k), ref_out.resize(k), id_out.resize(k), vref_out.resize(2 * (size_t) k), velocity_cur.resize(2 * (size_t) k), src.resize(k);
        pts2d_new.swap(cur_pts), pts2d_ref.swap(ref_out), ref_frame_id.swap(id_out), velocity_ref.swap(vref_out);
        if (par_n[1] >= 0) parallax_ref = par[1], parallax_ref_counts = par_n[1];
        return k > 0;
    }

    // One new map point of Tracking::triangulation (IG/tracking/tracking.cc:761-784): what MapPoint::createMapPoint and the two
    // Feature::createFeature calls take.  depth already carries MapPoint's clamp (mappoint.cc:39-42); src = the point's index in the input list.
    struct NewMapPoint {
        double pw[3], depth;
        Point2f ref_undis, ref, cur_undis, cur;
        double velocity_cur[2], velocity_ref[2];
        int64_t ref_frame_id;
        int32_t src;
    };

    // Tracking::triangulation (IG/tracking/tracking.cc:690-798), one call (icg_klt_triangulate).  frames: every frame pts2d_ref_frame_ can
    // name with id <= frame_ref_->id(), with its pose and map_->isKeyFrameInMap (at most 64).  pts2d_ref, ref_frame_id (pts2d_ref_frame_[k]->id()),
    // pts2d_cur and velocity_ref (2 doubles per point) are reduced in place as :788-791 reduces them; pts2d_new becomes pts2d_cur (:793);
    // src = the input index of every kept point (reduce pts2d_ref_frame_ with it).  velocity_cur (2 doubles per point) is read only.  points
    // receives the new map points in creation order: create the MapPoint / Feature objects in this order.  counts (may be NULL): kept,
    // succeeded, outlier, reset, outtime (:795).  Returns the reference's return value.
    bool triangulation(const icg_tri_frame &p, const std::vector<icg_tri_keyframe> &frames, std::vector<Point2f> &pts2d_ref, std::vector<int64_t> &ref_frame_id,
                       std::vector<Point2f> &pts2d_cur, std::vector<double> &velocity_ref, const std::vector<double> &velocity_cur, std::vector<Point2f> &pts2d_new,
                       std::vector<int32_t> &src, std::vector<NewMapPoint> &points, int32_t *counts = nullptr) {
        const int n = (int) pts2d_cur.size();
        const size_t N = n > 0 ? n : 1;
        src.resize(N);
        std::vector<double> pw(3 * N), depth(N), vcur(2 * N), vref(2 * N);
        std::vector<Point2f> ru(N), rp(N), cu(N), cp(N);
        std::vector<int64_t> fid(N);
        std::vector<int32_t> nsrc(N);
        icg_tri_list l{reinterpret_cast<float *>(pts2d_ref.data()), ref_frame_id.data(), reinterpret_cast<float *>(pts2d_cur.data()), velocity_ref.data(),
                       velocity_cur.data(), src.data()};
        icg_tri_new o{pw.data(), depth.data(), reinterpret_cast<float *>(ru.data()), reinterpret_cast<float *>(rp.data()), reinterpret_cast<float *>(cu.data()),
                      reinterpret_cast<float *>(cp.data()), vcur.data(), vref.data(), fid.data(), nsrc.data()};
        int32_t c[5];
        check(icg_klt_triangulate(h_, &p, (int) frames.size(), frames.data(), n, &l, &o, c), "icg_klt_triangulate");
        if (c[0] == -2) throw std::runtime_error("KltContext::triangulation: a reference frame of the list is missing from `frames`");
        if (counts)
            for (int k = 0; k < 5; k++) counts[k] = c[k];
        points.clear();
        src.resize(c[0] >= 0 ? c[0] : 0);
        if (c[0] < 0) return false;  // :692-694 (or triangulate == 0): nothing changes
        const int k = c[0];
        pts2d_ref.resize(k), ref_frame_id.resize(k), pts2d_cur.resize(k), velocity_ref.resize(2 * (size_t) k);
        pts2d_new = pts2d_cur;
        for (int m = 0; m < c[1]; m++) {
            NewMapPoint q;
            for (int d = 0; d < 3; d++) q.pw[d] = pw[3 * (size_t) m + d];
            q.depth = depth[m], q.ref_undis = ru[m], q.ref = rp[m], q.cur_undis = cu[m], q.cur = cp[m];
            q.velocity_cur[0] = vcur[2 * (size_t) m], q.velocity_cur[1] = vcur[2 * (size_t) m + 1];
            q.velocity_ref[0] = vref[2 * (size_t) m], q.velocity_ref[1] = vref[2 * (size_t) m + 1];
            q.ref_frame_id = fid[m], q.src = nsrc[m];
            points.push_back(q);
        }
        return true;
    }

private:
    void upload(const Mat &pre, const Mat &cur, icg_track_frame &p) {
        check(icg_klt_upload(h_, 0, mat_data(pre), mat_stride(pre)), "icg_klt_upload");
        check(icg_klt_upload(h_, 1, mat_data(cur), mat_stride(cur)), "icg_klt_upload");
        p.prev_slot = 0, p.cur_slot = 1;
    }
    icg_klt *h_ = nullptr;
};

// The window solve seam: what GVINS::gvinsOptimization hands to ceres::Solver::Solve (IG/ic_gvins.cc:1130-1239).
// Any max_K / max_L marginalizes (a block beyond 512 rows throws ICG_EUNSUPPORTED); to consume its own prior the handle needs
// max_marg_r >= 15 (max_K - 1) + 7, e.g. 292 for a 20-keyframe window.
// ins_window_ of GVINS (IG/ic_gvins.cc:249-293) for a set of streams on the device: the per-sample mechanization, the post-solve redo
// (MISC::redoInsMechanization), the prior camera pose and gvinsInitialization (see the icg_ins_* calls).  WindowSolver cuts its factors' IMU
// series out of these windows (imuSamplesFromIns, the INS form of slideWindow).
class InsWindows {
public:
    explicit InsWindows(int max_streams, int capacity = 1000, int device = 0) {
        check(icg_ins_create(&h_, max_streams, capacity, device, nullptr), "icg_ins_create");
    }
    ~InsWindows() { icg_ins_destroy(h_); }
    InsWindows(const InsWindows &) = delete;
    InsWindows &operator=(const InsWindows &) = delete;

    // runFusion's IMU step: rows (time, dt, dtheta[3], dvel[3]) of stream s are imu[off[s] .. off[s + 1])
    void push(int n_streams, const icg_ins_config *cfg, const int32_t *off, const double *imu) {
        check(icg_ins_push(h_, n_streams, cfg, off, imu), "icg_ins_push");
    }
    // redoInsMechanization from state17 (n x 17) of the streams redo selects (nullptr: all); status per stream (1, 0, -1)
    void redo(int n_streams, const icg_ins_config *cfg, const uint8_t *redo, const double *state17, int reserved, int8_t *status) {
        check(icg_ins_redo(h_, n_streams, cfg, redo, state17, reserved, status), "icg_ins_redo");
    }
    // getCameraPoseFromInsWindow at stamp[s] (see icg_ins_camera_pose)
    void cameraPose(int n_streams, const double *stamp, const double *pose_b_c, double *dev_pose, double *host_pose, int32_t *found) {
        check(icg_ins_camera_pose(h_, n_streams, stamp, pose_b_c, dev_pose, host_pose, found), "icg_ins_camera_pose");
    }
    // gvinsInitialization of the selected streams (see icg_ins_gins_initialize)
    void ginsInitialize(int n_streams, icg_ins_config *cfg, const uint8_t *sel, const icg_gins_init *in, const double noise5[5],
                        const double station[3], int reserved, icg_gins_init_out *out) {
        check(icg_ins_gins_initialize(h_, n_streams, cfg, sel, in, noise5, station, reserved, out), "icg_ins_gins_initialize");
    }
    // one stream's window, oldest first: rows (count x 8) and states (count x 17)
    void window(int stream, std::vector<double> &imu8, std::vector<double> &state17) {
        int32_t count = 0;
        check(icg_ins_window(h_, stream, 0, &count, nullptr, nullptr), "icg_ins_window");
        imu8.resize(8 * (size_t) count), state17.resize(17 * (size_t) count);
        check(icg_ins_window(h_, stream, count, &count, imu8.data(), state17.data()), "icg_ins_window");
    }
    icg_ins *handle() const { return h_; }

private:
    icg_ins *h_ = nullptr;
};

class WindowSolver {
public:
    WindowSolver(int max_K, int max_L, int max_F, int max_gnss = 16, int max_marg_r = 160, int device = 0) {
        check(icg_ba_create(&h_, 1, max_K, max_L, max_F, max_gnss, max_marg_r, device, nullptr), "icg_ba_create");
    }
    ~WindowSolver() { icg_ba_destroy(h_); }
    WindowSolver(const WindowSolver &) = delete;
    WindowSolver &operator=(const WindowSolver &) = delete;

    // solver.Solve(options, &problem, &summary) with options.max_num_iterations = max_iter
    icg_ba_summary Solve(const icg_ba_problem &problem, int max_iter) {
        icg_ba_summary s{};
        check(icg_ba_solve(h_, 1, &problem, max_iter, &s), "icg_ba_solve");
        return s;
    }
    // the two-pass body of gvinsOptimization (first N/4, chi2 culling, then N - N/4 iterations); out[0], out[1] = pass summaries
    void gvinsOptimization(const icg_ba_problem &problem, int num_iterations, icg_ba_summary out[2], int32_t culled[2]) {
        check(icg_ba_gvins_optimization(h_, 1, &problem, num_iterations, out, culled), "icg_ba_gvins_optimization");
    }

    // marginalization_info->marginalization() as GVINS::gvinsMarginalization drives it (IG/ic_gvins.cc:1412-1640): the prior that
    // replaces last_marginalization_info_ / last_marginalization_parameter_blocks_.  Vectors are sized here.
    struct Prior {
        int m = 0, r = 0;
        std::vector<int32_t> block_type, block_node;  // remainedBlock*: type 0 pose 1 mix 2 extrinsic 3 td; node index after the removal
        std::vector<double> x0, J0, e0;               // remainedBlockData(), linearizedJacobians() (r x r row-major), linearizedResiduals()
    };
    Prior marginalization(const icg_ba_problem &problem, int num_marg, bool after_solve = false) {  // after_solve: the window this solver just optimised (no re-upload)
        return marginalize(problem, num_marg, [&](const int32_t *nm, icg_ba_prior *o) {
            return after_solve ? icg_ba_marginalize_resident(h_, 1, &problem, nm, o) : icg_ba_marginalize(h_, 1, &problem, nm, o);
        });
    }
    // The same on the window this solver just optimised, with the factor set of the map after updateAndCull (IG/ic_gvins.cc:1558-1609):
    // culled = that call's io (obs_factor set), node_in_map = K flags, 0 for the keyframes gvinsRemoveAllSecondNewFrame took out of the map.
    // Both resident forms also run on a landmark-sharded handle: every rank calls with its shard, and the prior is returned on the window's
    // owner (rank w mod world) only.  Elsewhere m = r = 0, block_type / block_node / J0 / e0 come back empty and x0 keeps its capacity
    // unwritten, as for any prior (icgvins_b200.h, icg_ba_marginalize_resident).
    Prior marginalization(const icg_ba_problem &problem, int num_marg, const icg_ba_cull_window &culled, const uint8_t *node_in_map) {
        return marginalize(problem, num_marg, [&](const int32_t *nm, icg_ba_prior *o) {
            return icg_ba_marginalize_resident_culled(h_, 1, &problem, nm, &culled, &node_in_map, o);
        });
    }
    // The same after updateAndCullBuilt, with the factor set and the column map built on the device (icg_ba_marginalize_built): problem needs
    // its camera side only (f_lm / f_ref / f_obs / f_active / invdepth may be NULL), node_in_map = K flags.  Single-GPU solvers only.
    Prior marginalizeBuilt(const icg_ba_problem &problem, int num_marg, const uint8_t *node_in_map) {
        return marginalize(problem, num_marg, [&](const int32_t *nm, icg_ba_prior *o) { return icg_ba_marginalize_built(h_, 1, &problem, nm, &node_in_map, o); });
    }

    // updateParametersFromOptimizer + gvinsOutlierCulling (IG/ic_gvins.cc:1232-1236) on the window this solver just optimised: io carries the
    // observation lists the caller gathered and receives pose_b_c_ / td_b_c_, every node's frame->pose(), every landmark's pos() / depth and
    // the outlier flags (see icg_ba_cull_window); the caller applies them to its object graph.  On a landmark-sharded handle every rank passes
    // its shard and its landmarks' observation lists; the counts are the window's totals on every rank, the landmark outputs its shard's.
    void updateAndCull(const icg_ba_problem &problem, const icg_camera &camera, double reprojection_error_std, icg_ba_cull_window &io) {
        check(icg_ba_update_and_cull_resident(h_, 1, &problem, &camera, reprojection_error_std, &io), "icg_ba_update_and_cull_resident");
    }
    // The same on the observation lists the last slideVision built on the device (icg_ba_update_and_cull_built): io's list inputs stay NULL,
    // its outputs are updateAndCull's with obs_outlier indexed by the built list, and `lists` (may be null; each array may be NULL) receives
    // that list, so that the caller maps each flag to its Feature through (landmark, obs_node).  marginalization(problem, num_marg, io,
    // node_in_map) and the next slideVision (vision.obs_factor NULL) then use the culling's own lists.  Single-GPU solvers only.
    void updateAndCullBuilt(const icg_ba_problem &problem, const icg_camera &camera, double reprojection_error_std, icg_ba_cull_window &io,
                            icg_ba_cull_lists *lists = nullptr) {
        check(icg_ba_update_and_cull_built(h_, 1, &problem, &camera, reprojection_error_std, &io, lists), "icg_ba_update_and_cull_built");
    }
    // updateAndCullBuilt on a landmark-sharded solver, a collective call of its group (icg_ba_shard_update_and_cull_built): every rank passes
    // its shard problem and the same extrinsic inputs, and culls on the lists its last sharded slideVision built; the outputs are
    // updateAndCull's on a shard, `lists` the rank's shard-local lists.  A rejection on any rank throws on every rank, no solver changed.
    void shardUpdateAndCullBuilt(const icg_ba_problem &problem, const icg_camera &camera, double reprojection_error_std, icg_ba_cull_window &io,
                                 icg_ba_cull_lists *lists = nullptr) {
        check(icg_ba_shard_update_and_cull_built(h_, 1, &problem, &camera, reprojection_error_std, &io, lists), "icg_ba_shard_update_and_cull_built");
    }

    // GVINS::doReintegration (IG/ic_gvins.cc:1680-1695) on the window this solver just optimised, as gvinsOptimization calls it while the
    // window is not full (:1223-1227).  imu = the rows (dt, dtheta[3], dvel[3]) of every factor's imu_buffer_, imu_off = n_imu + 1 offsets
    // into them; noise5 = gyr_arw, acc_vrw, gyr_bias_std, acc_bias_std, corr_time; station = parameters_->station ((0, 0, 0) in the
    // reference).  blobs (n_imu x ICG_IMU_BLOB_DOUBLES) is updated in place where status == 1 (the solver holds the same factors from then on);
    // end_states (n_imu x 10, may be NULL) receives currentState() of every reintegrated factor.  Returns cnt (the factors whose gate opened).
    int doReintegration(const icg_ba_problem &problem, const double noise5[5], const double station[3], const std::vector<double> &imu,
                        const std::vector<int32_t> &imu_off, std::vector<int8_t> &status, std::vector<double> &blobs,
                        std::vector<double> *end_states = nullptr) {
        const size_t m = problem.n_imu > 0 ? (size_t) problem.n_imu : 0;
        status.assign(m, 0);
        blobs.resize(m * ICG_IMU_BLOB_DOUBLES);
        if (end_states) end_states->assign(10 * m, 0.0);
        icg_ba_reint_window io{};
        io.reintegrate = 1, io.imu = imu.data(), io.imu_off = imu_off.data(), io.status = status.data(), io.blob_out = blobs.data();
        io.end_state10 = end_states ? end_states->data() : nullptr;
        if (m > 0 && imu_off.size() != m + 1) throw std::runtime_error("WindowSolver::doReintegration: imu_off needs n_imu + 1 entries");
        check(icg_ba_reintegrate_resident(h_, 1, &problem, noise5, station, &io), "icg_ba_reintegrate_resident");
        return io.count;
    }

    // The next gvinsOptimization's problem (IG/ic_gvins.cc:1130-1239, 1697-1837) from the window this solver holds, without re-uploading what
    // carries over.  next = the problem as Solve would take it; carry = per row of next its row in the old window or -1 (an empty vector: none
    // of that kind carries): node_src from timelist_ before and after gvinsMarginalization / removeUnusedTimeNode, lm_src from the old
    // invdepthlist_ keys (a re-anchored map point is -1), f_src by (map point, observing keyframe), imu_src by preintegrationlist_ element (a
    // merged factor is -1), gnss_src by gnsslist_ element.  prior_from_marginalization: the prior is the one marginalization(..., culled, ...)
    // or marginalization(..., true) just built on this solver.  Then gvinsOptimizationResident(next, ...) solves it.
    struct Carry {
        std::vector<int32_t> node_src, lm_src, f_src, imu_src, gnss_src;
    };
    void slideWindow(const icg_ba_problem &next, const Carry &carry, bool prior_from_marginalization) {
        icg_ba_slide_window c = carryStruct(next, carry);
        c.prior_from_marg = prior_from_marginalization ? 1 : 0;
        check(icg_ba_slide_resident(h_, 1, &next, &c), "icg_ba_slide_resident");
    }
    // The same, with the new factors, node states and aligned GNSS fixes that `integrate` names computed on the device from the states this
    // solver holds, in place of the host parts of addNewTimeNode, removeUnusedTimeNode and insertNewGnssTimeNode (IG/ic_gvins.cc:754-928):
    // see icg_ba_slide_integrate. Its outputs (status, blob_out, end_state10) are written as that struct names them.
    void slideWindow(const icg_ba_problem &next, const Carry &carry, bool prior_from_marginalization, icg_ba_slide_integrate &integrate,
                     const double noise5[5], const double station[3]) {
        icg_ba_slide_window c = carryStruct(next, carry);
        c.prior_from_marg = prior_from_marginalization ? 1 : 0;
        check(icg_ba_slide_integrate_resident(h_, 1, &next, &c, &integrate, noise5, station), "icg_ba_slide_integrate_resident");
    }
    // The same again with the vision half built on the device in place of addReprojectionParameters + addReprojectionFactors
    // (IG/ic_gvins.cc:1697-1837): see icg_ba_slide_vision.  carry.lm_src / f_src and next's vision rows are not read; integrate may be null
    // (no IMU row integrated).  The last updateAndCull on this solver must be current.  On return next.L / F and, where `vision` names
    // output arrays, next's invdepth / f_lm / f_ref / f_obs / f_const point at them (f_active all active), so gvinsOptimizationResident(next)
    // writes the solved inverse depths there; vision.lm_origin / nan_flags say which MapPoint each row is and which ones to set outliers.
    void slideVision(icg_ba_problem &next, const Carry &carry, bool prior_from_marginalization, icg_ba_slide_vision &vision,
                     icg_ba_slide_integrate *integrate = nullptr, const double noise5[5] = nullptr, const double station[3] = nullptr) {
        icg_ba_slide_window c = carryStruct(next, Carry{carry.node_src, {}, {}, carry.imu_src, carry.gnss_src});
        c.prior_from_marg = prior_from_marginalization ? 1 : 0;
        check(icg_ba_slide_vision_resident(h_, 1, &next, &c, integrate, noise5, station, &vision), "icg_ba_slide_vision_resident");
        next.L = vision.L, next.F = vision.F, next.f_active = nullptr;
        if (vision.invdepth) next.invdepth = vision.invdepth;
        if (vision.f_lm) next.f_lm = vision.f_lm;
        if (vision.f_ref) next.f_ref = vision.f_ref;
        if (vision.f_obs) next.f_obs = vision.f_obs;
        if (vision.f_const) next.f_const = vision.f_const;
    }
    // Every IMU factor's imu_buffer_ kept on the device, cut from `ins` (icg_ba_imu_samples_from_ins): factor k of the window this solver
    // holds is getImuSeriesFromTo(timelist[k], timelist[k + 1]) of stream `stream`.  Right after the upload of a window whose INS window still
    // covers it (the GINS window of gvinsInitializationOptimization: before the next redo).
    void imuSamplesFromIns(InsWindows &ins, int32_t stream, const std::vector<double> &timelist) {
        const icg_ba_ins_cut cut = {stream, timelist.data()};
        check(icg_ba_imu_samples_from_ins(h_, ins.handle(), 1, &cut), "icg_ba_imu_samples_from_ins");
    }
    // slideWindow(next, carry, prior, integrate, ...) whose integrated factors' rows come from the device (icg_ba_slide_ins_resident): NODE
    // and ICG_SLIDE_CHAIN factors cut from stream `stream` of `ins` over the next timelist_ (next.K times), ICG_SLIDE_ROW factor k merged
    // from stored factors merge_src[k] and merge_src[k] + 1 (an empty vector: no ROW factor), carried factors keep their rows.
    // integrate.imu / imu_off must be null.  n_rows (optional): every new factor's stored rows, -1 for none.
    void slideWindow(const icg_ba_problem &next, const Carry &carry, bool prior_from_marginalization, icg_ba_slide_integrate &integrate,
                     InsWindows &ins, int32_t stream, const std::vector<double> &timelist, const std::vector<int32_t> &merge_src,
                     const double noise5[5], const double station[3], std::vector<int32_t> *n_rows = nullptr) {
        icg_ba_slide_window c = carryStruct(next, carry);
        c.prior_from_marg = prior_from_marginalization ? 1 : 0;
        if (timelist.size() != (size_t) (next.K > 0 ? next.K : 0)) throw std::runtime_error("WindowSolver::slideWindow: timelist needs next.K times");
        icg_ba_slide_ins io{};
        io.integ = integrate, io.stream = stream, io.node_time = timelist.data(), io.merge_src = merge_src.empty() ? nullptr : merge_src.data();
        if (n_rows) n_rows->assign(next.n_imu > 0 ? next.n_imu : 0, -1), io.n_rows = n_rows->data();
        check(icg_ba_slide_ins_resident(h_, ins.handle(), 1, &next, &c, &io, noise5, station, nullptr), "icg_ba_slide_ins_resident");
    }
    // doReintegration from the stored rows (icg_ba_reintegrate_stored_resident): as the other doReintegration, without the host's rows
    int doReintegration(const icg_ba_problem &problem, const double noise5[5], const double station[3], std::vector<int8_t> &status,
                        std::vector<double> &blobs, std::vector<double> *end_states = nullptr) {
        const size_t m = problem.n_imu > 0 ? (size_t) problem.n_imu : 0;
        status.assign(m, 0);
        blobs.resize(m * ICG_IMU_BLOB_DOUBLES);
        if (end_states) end_states->assign(10 * m, 0.0);
        icg_ba_reint_window io{};
        io.reintegrate = 1, io.status = status.data(), io.blob_out = blobs.data(), io.end_state10 = end_states ? end_states->data() : nullptr;
        check(icg_ba_reintegrate_stored_resident(h_, 1, &problem, noise5, station, &io), "icg_ba_reintegrate_stored_resident");
        return io.count;
    }
    // the stored rows of the window (icg_ba_imu_samples): off (n_imu + 1; -1 for a factor without samples) and rows (7 per row)
    void imuSamples(int n_imu, std::vector<int32_t> &off, std::vector<double> &rows) {
        off.assign((size_t) n_imu + 1, 0);
        check(icg_ba_imu_samples(h_, 0, 0, off.data(), nullptr), "icg_ba_imu_samples");
        rows.resize(7 * (size_t) off[n_imu]);
        check(icg_ba_imu_samples(h_, 0, off[n_imu], off.data(), rows.data()), "icg_ba_imu_samples");
    }
    // the two-pass body of gvinsOptimization on the window slideWindow left (nothing is uploaded); results as gvinsOptimization gives them
    void gvinsOptimizationResident(const icg_ba_problem &next, int num_iterations, icg_ba_summary out[2], int32_t culled[2]) {
        check(icg_ba_run_gvins(h_, num_iterations, 0), "icg_ba_run_gvins");
        check(icg_ba_gvins_optimization_end(h_, 1, &next, out, culled), "icg_ba_gvins_optimization_end");
    }

private:
    static icg_ba_slide_window carryStruct(const icg_ba_problem &next, const Carry &carry) {
        auto ptr = [](const std::vector<int32_t> &v, int32_t n, const char *what) -> const int32_t * {
            if (v.empty()) return nullptr;
            if (v.size() != (size_t) (n > 0 ? n : 0)) throw std::runtime_error(std::string("WindowSolver::slideWindow: ") + what + " needs one entry per row of next");
            return v.data();
        };
        icg_ba_slide_window c{};
        c.node_src = ptr(carry.node_src, next.K, "node_src"), c.lm_src = ptr(carry.lm_src, next.L, "lm_src"), c.f_src = ptr(carry.f_src, next.F, "f_src");
        c.imu_src = ptr(carry.imu_src, next.n_imu, "imu_src"), c.gnss_src = ptr(carry.gnss_src, next.n_gnss, "gnss_src");
        return c;
    }
    template <typename Call>
    Prior marginalize(const icg_ba_problem &problem, int num_marg, Call call) {
        Prior P;
        const int rcap = 15 * problem.K + 7;
        P.block_type.resize(2 * problem.K + 2), P.block_node.resize(2 * problem.K + 2);
        P.x0.resize(16 * problem.K + 8), P.J0.resize((size_t) rcap * rcap), P.e0.resize(rcap);
        icg_ba_prior o{};
        o.rcap = rcap, o.block_type = P.block_type.data(), o.block_node = P.block_node.data(), o.x0 = P.x0.data(), o.J0 = P.J0.data(), o.e0 = P.e0.data();
        const int32_t nm = num_marg;
        check(call(&nm, &o), "icg_ba_marginalize");
        P.m = o.m, P.r = o.r;
        P.block_type.resize(o.nblocks), P.block_node.resize(o.nblocks);
        P.J0.resize((size_t) o.r * o.r), P.e0.resize(o.r);
        return P;
    }

    icg_ba *h_ = nullptr;
};

// Camera (IG/tracking/camera.cc): the point-wise model functions Tracking calls (host code in the library)
class CameraModel {
public:
    explicit CameraModel(const icg_camera &c) : c_(c) {}
    void undistortPoints(std::vector<Point2f> &pts) const { check(icg_camera_undistort_points(&c_, reinterpret_cast<float *>(pts.data()), (int) pts.size()), "icg_camera_undistort_points"); }
    void distortPoints(std::vector<Point2f> &pts) const { check(icg_camera_distort_points(&c_, reinterpret_cast<float *>(pts.data()), (int) pts.size()), "icg_camera_distort_points"); }
    Point2f distortCameraPoint(const double pc[3]) const {
        Point2f out{};
        check(icg_camera_distort_camera_points(&c_, pc, reinterpret_cast<float *>(&out), 1), "icg_camera_distort_camera_points");
        return out;
    }

private:
    icg_camera c_;
};

// cv::Ptr<cv::CLAHE> clahe_ = cv::createCLAHE(3.0, cv::Size(21, 21)) (IG/tracking/tracking.cc:62); clahe_->apply(img, img) (:141)
class Clahe {
public:
    Clahe(int width, int height, double clipLimit = 3.0, Size tileGridSize = Size(21, 21), int device = 0) {
        check(icg_clahe_create(&h_, width, height, tileGridSize.width, tileGridSize.height, clipLimit, device, nullptr), "icg_clahe_create");
    }
    ~Clahe() { icg_clahe_destroy(h_); }
    Clahe(const Clahe &) = delete;
    Clahe &operator=(const Clahe &) = delete;
    // apply(src, dst) on 8-bit single-channel images; dst may be src
    void apply(const uint8_t *src, int src_step, uint8_t *dst, int dst_step) { check(icg_clahe_apply(h_, src, src_step, dst, dst_step), "icg_clahe_apply"); }

private:
    icg_clahe *h_ = nullptr;
};

// Tracking::featuresDetection (IG/tracking/tracking.cc:576-688): the tbb::parallel_for body (:627-656) for all blocks in one call, or the
// whole detection step driven by the point lists.
class BlockDetector {
public:
    BlockDetector(int width, int height, int max_blocks, int max_corners_per_block, int max_roi_pixels, int device = 0)
        : cap_(max_corners_per_block), max_blocks_(max_blocks) {
        check(icg_detect_create(&h_, width, height, max_blocks, max_corners_per_block, max_roi_pixels, device, nullptr), "icg_detect_create");
    }
    ~BlockDetector() { icg_detect_destroy(h_); }
    BlockDetector(const BlockDetector &) = delete;
    BlockDetector &operator=(const BlockDetector &) = delete;

    // goodFeaturesToTrack(frame(roi), out, max_corners[b], quality, min_distance, mask(roi)) + cornerSubPix(...) per block;
    // features[b] holds block-local coordinates in OpenCV's order
    void detect(const Mat &frame, const Mat *mask, const std::vector<icg_rect> &rois, const std::vector<int32_t> &max_corners, double quality,
                double min_distance, std::vector<std::vector<Point2f>> &features) {
        const int nb = (int) rois.size();
        std::vector<float> xy((size_t) nb * cap_ * 2);
        std::vector<int32_t> cnt(nb);
        check(icg_detect_blocks(h_, mat_data(frame), mask ? mat_data(*mask) : nullptr, mat_stride(frame), nb, rois.data(), max_corners.data(), quality,
                                min_distance, 1, xy.data(), cnt.data()),
              "icg_detect_blocks");
        features.assign(nb, {});
        for (int b = 0; b < nb; b++)
            for (int k = 0; k < cnt[b]; k++) features[b].push_back(Point2f{xy[((size_t) b * cap_ + k) * 2], xy[((size_t) b * cap_ + k) * 2 + 1]});
    }

    // Tracking::featuresDetection(frame, ismask) (IG/tracking/tracking.cc:576-685) up to the append into the reference's lists:
    // keypoints = the frame's features' keyPoint() (undistorted), pts2d_new = pts2d_new_, n_ref = pts2d_ref_.size().  Returns the new
    // corners in frame coordinates, in the order :669-685 appends them.  *skipped is set when the gate of :579-582 returned before
    // detection; the caller then leaves its lists as they are (an empty result with *skipped false means nothing was found).
    std::vector<Point2f> featuresDetection(const Mat &frame, const std::vector<Point2f> &keypoints, const std::vector<Point2f> &pts2d_new, int n_ref,
                                           bool ismask, int max_features, bool *skipped = nullptr) {
        std::vector<float> xy((size_t) max_blocks_ * cap_ * 2);
        int32_t n = 0;
        check(icg_detect_features(h_, mat_data(frame), mat_stride(frame), reinterpret_cast<const float *>(keypoints.data()), (int) keypoints.size(),
                                  reinterpret_cast<const float *>(pts2d_new.data()), (int) pts2d_new.size(), n_ref, ismask ? 1 : 0, max_features, xy.data(),
                                  &n),
              "icg_detect_features");
        if (skipped) *skipped = n < 0;
        std::vector<Point2f> out;
        for (int k = 0; k < n; k++) out.push_back(Point2f{xy[2 * (size_t) k], xy[2 * (size_t) k + 1]});
        return out;
    }

private:
    icg_detect *h_ = nullptr;
    int cap_, max_blocks_;
};

}  // namespace icg_b200
