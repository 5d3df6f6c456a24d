// track.cu -- Tracking::trackMappoint (IG/tracking/tracking.cc:351-455) and Tracking::trackReferenceFrame (:457-574) for B streams on the
// KLT handle: from the predicted pose to the compacted point lists, pixel velocities and the two parallax figures checkKeyFrameSate reads
// (:263-307), with no host round trip.  Launch sequence of icg_klt_track_frames_dev (all on the handle's stream):
//
//   track_predict    thread / point of both lists: the initial flow the reference computes from the poses
//                      map list: distortPoints(world2pixel(pw, pose_cur))                                             (:367, :378)
//                      ref list: undistortPoints(new) -> pixel2cam -> R_cur^T R_pre . -> distortCameraPoint (float cast) (:465-479)
//   klt_track_kernel ONE launch (icg_klt_track_batch_dev, mode 1) over both lists of all streams: forward + backward LK and the gate
//                    st_f && st_b && !isOnBorder && ptsDistance < 0.5                                                 (:385-403, :487-506)
//   track_post       CTA / stream: stable compaction (ballot + block prefix, reduceVector :404-408, :507-511), undistortPoints of the
//                    survivors, velocities (pixel2cam(cur_undis) - pixel2cam(prev_undis)) / dt (:429-434, :527-533), the velocity_ref
//                    rule (ref_frame_id > ref_id -> velocity_cur, :536-538), parallaxFromReferenceMapPoints (:873-905) and
//                    parallaxFromReferenceKeyPoints over undistort(ref) (:541-544, before RANSAC)
//   geom_ransac_batch_kernel  findFundamentalMat(new_undis, cur_undis, FM_RANSAC, threshold, 0.99), maxIters 1000 (:546-548), on the
//                    survivors of every reference list (sets with fewer than 15 survivors are not applied, :547)
//   track_compact    CTA / stream: in-place stable compaction of ref, cur, ref_frame_id, velocity_cur, velocity_ref by the inlier mask
//                    (:550-554) for the lists with >= 15 survivors; the per-input keep flag of an outlier is cleared
//
// Early returns of the reference, reported through the parallax count: an empty input list leaves parallax_map_ / parallax_ref_ as they
// were (:372-375, :459-462) -> count -1; a reference list the LK gate empties returns before the parallax (:513-517) -> -1; a map list the
// LK gate empties sets parallax_map_ = parallax_map_counts_ = 0 (:410-419) -> 0.
//
// Documented difference: both parallax sums run in LIST order.  The reference iterates frame_ref_->features(), an std::unordered_map
// (frame.h:80) whose order is implementation-defined, so its sum has no defined order to reproduce (as the marginalization ordering in
// INTEGRATION.md).  Matrix products (R_cur^T R_pre, R_cur^T R_ref, world2cam) are fixed-order sums without FMA (geom_core.cuh, -fmad=false);
// parity with Eigen's product is not pinned.
#include <float.h>
#include <math.h>
#include <string.h>

#include "common.cuh"
#include "geom_core.cuh"
#include "klt_handle.cuh"

namespace icg {

constexpr int TRK_THREADS = 256;  // track_post / track_compact: one CTA per stream, chunks of 256 points

struct TrackScratch {
    int cap_streams = 0;
    icg_track_frame *d_par = nullptr;  // n_streams
    int32_t *d_moff = nullptr, *d_roff = nullptr;  // n_streams + 1 each
    double *d_thr = nullptr;                       // n_streams: fundamental threshold of each stream's RANSAC
    int32_t *d_n1 = nullptr, *d_ninl = nullptr;    // n_streams: LK survivors of the ref list, RANSAC inliers
    uint8_t *h_stage = nullptr;                    // pinned: params | moff | roff
    size_t stage_bytes = 0;
    cudaEvent_t stage_ev = nullptr;
    bool stage_pending = false;
    // per point (handle's max_points): undistorted new points of the ref-list survivors (RANSAC input), the inlier mask
    float *d_nu = nullptr;
    uint8_t *d_rmask = nullptr;
    // device copies of the single-stream host call (icg_klt_track_frame)
    uint8_t *d_host = nullptr;
    // triangulation (icg_klt_triangulate_dev): params | kf_off | ref_off | kf staged as one blob (pinned + its device copy, fenced by stage_ev),
    // and the device copies of the single-stream host call (icg_klt_triangulate)
    uint8_t *h_tri = nullptr, *d_tri = nullptr;
    size_t tri_bytes = 0;
    uint8_t *d_tri_host = nullptr;
};

void track_scratch_free(TrackScratch *t) {
    if (!t) return;
    cudaFree(t->d_par), cudaFree(t->d_moff), cudaFree(t->d_roff), cudaFree(t->d_thr), cudaFree(t->d_n1), cudaFree(t->d_ninl);
    cudaFree(t->d_nu), cudaFree(t->d_rmask);
    if (t->d_host) cudaFree(t->d_host);
    if (t->d_tri) cudaFree(t->d_tri);
    if (t->d_tri_host) cudaFree(t->d_tri_host);
    if (t->h_tri) cudaFreeHost(t->h_tri);
    if (t->h_stage) cudaFreeHost(t->h_stage);
    if (t->stage_ev) cudaEventDestroy(t->stage_ev);
    delete t;
}

__device__ __forceinline__ int find_stream(const int32_t *off, int n_streams, int i) {  // the s with off[s] <= i < off[s + 1]
    int lo = 0, hi = n_streams - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

struct TrackArgs {
    int n_streams, n_map, n_ref;  // n_map / n_ref: total points of each list
    const icg_track_frame *par;
    const int32_t *moff, *roff;
    icg_track_map map;
    icg_track_ref ref;
    // the KLT batch: map points at [0, n_map), ref points at [n_map, n_map + n_ref)
    int32_t *slots;
    float2 *prev, *init, *fwd;
    const uint8_t *status;
    double *thr;
    int32_t *n1, *ninl;
    float *nu;
    const uint8_t *rmask;
    int32_t *n_out, *par_n;
    double *parallax;
};

__global__ void __launch_bounds__(128) track_predict_kernel(TrackArgs A) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g < A.n_streams) A.thr[g] = A.par[g].fm_threshold;
    if (g >= A.n_map + A.n_ref) return;
    const bool is_map = g < A.n_map;
    const int i = is_map ? g : g - A.n_map;
    const int s = find_stream(is_map ? A.moff : A.roff, A.n_streams, i);
    const icg_track_frame &P = A.par[s];
    float2 prev, init;
    if (is_map) {
        prev = ((const float2 *) A.map.prev_xy)[i];
        float px[2];
        gc::world2pixel(P.camera, P.R_cur, P.t_cur, A.map.pw + 3 * (size_t) i, px[0], px[1]);  // tracking.cc:367
        gc::distort_point(P.camera, px);                                                      // :378
        init = make_float2(px[0], px[1]);
    } else {
        prev = ((const float2 *) A.ref.new_xy)[i];
        double Rcp[9], x, y, X, Y, Z;
        gc::rt_mul(P.R_cur, P.R_pre, Rcp);  // :465
        float p[2] = {prev.x, prev.y};
        gc::undistort_point(P.camera, p);  // :468-469
        gc::pixel2cam(P.camera, p[0], p[1], x, y);
        gc::mat_vec(Rcp, x, y, 1.0, X, Y, Z);  // :473-474
        gc::distort_camera_point(P.camera, X, Y, Z, init.x, init.y);  // :477
    }
    A.slots[2 * g] = P.prev_slot, A.slots[2 * g + 1] = P.cur_slot;
    A.prev[g] = prev, A.init[g] = init;
}

// block-wide stable compaction index: returns the number of set flags before this thread in the chunk; *total = flags in the chunk
__device__ __forceinline__ int block_prefix(bool f, int *s_warp, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned b = __ballot_sync(0xffffffffu, f);
    if (lane == 0) s_warp[warp] = __popc(b);
    __syncthreads();
    int before = 0, tot = 0;
    for (int w = 0; w < TRK_THREADS / 32; w++) {
        const int c = s_warp[w];
        before += w < warp ? c : 0;
        tot += c;
    }
    __syncthreads();
    *total = tot;
    return before + __popc(b & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(TRK_THREADS) track_post_kernel(TrackArgs A) {
    __shared__ int s_warp[TRK_THREADS / 32];
    __shared__ double s_val[TRK_THREADS];
    __shared__ uint8_t s_has[TRK_THREADS];
    const int s = blockIdx.x, tid = threadIdx.x;
    const icg_track_frame &P = A.par[s];
    const icg_camera &cam = P.camera;
    double Rcr[9];
    gc::rt_mul(P.R_cur, P.R_ref, Rcr);  // keyPointParallax: pose1.R^T pose0.R with pose0 = frame_ref_, pose1 = frame_cur_ (:867)
    // ---------------------------------------------------------------- map list (trackMappoint)
    {
        const int base = A.moff[s], n = A.moff[s + 1] - base;
        int kept = 0, cnt = 0;
        double sum = 0;
        for (int c = 0; c < n; c += TRK_THREADS) {
            const int li = c + tid, i = base + li;
            const bool valid = li < n;
            bool keep = false, has = false;
            float2 f = make_float2(0.f, 0.f), u = f;
            if (valid) {
                keep = A.status[i] != 0;
                f = A.fwd[i];
                float p[2] = {f.x, f.y};
                gc::undistort_point(cam, p);  // :422-423
                u = make_float2(p[0], p[1]);
                ((float2 *) A.map.fwd_xy)[i] = f, ((float2 *) A.map.fwd_undis_xy)[i] = u, A.map.keep[i] = keep;
            }
            int tot;
            const int j = base + kept + block_prefix(keep, s_warp, &tot);
            double v = 0;
            if (keep) {
                const float2 m = ((const float2 *) A.map.prev_undis_xy)[i];
                double x1, y1, x0, y0;
                gc::pixel2cam(cam, u.x, u.y, x1, y1);
                gc::pixel2cam(cam, m.x, m.y, x0, y0);
                ((float2 *) A.map.cur_xy)[j] = f, ((float2 *) A.map.cur_undis_xy)[j] = u;
                A.map.velocity[2 * (size_t) j] = (x1 - x0) / P.dt, A.map.velocity[2 * (size_t) j + 1] = (y1 - y0) / P.dt;  // :434
                A.map.src[j] = li;
                const float2 r = ((const float2 *) A.map.ref_kp_xy)[i];
                has = !isnan(r.x) && !isnan(r.y);
                if (has) v = gc::key_point_parallax(cam, Rcr, r.x, r.y, u.x, u.y);  // :892-893
            }
            s_val[tid] = v, s_has[tid] = has;
            __syncthreads();
            if (tid == 0)
                for (int t = 0; t < TRK_THREADS; t++)
                    if (s_has[t]) sum += s_val[t], cnt++;  // list order
            __syncthreads();
            kept += tot;
        }
        if (tid == 0) {
            A.n_out[2 * s] = kept;
            A.parallax[2 * s] = n == 0 ? 0.0 : (cnt ? sum / cnt : 0.0);
            A.par_n[2 * s] = n == 0 ? -1 : cnt;  // :372-375 (-1: keep), :416-417 (kept == 0: 0)
        }
    }
    // ---------------------------------------------------------------- reference list (trackReferenceFrame, up to the RANSAC)
    {
        const int base = A.roff[s], n = A.roff[s + 1] - base;
        int kept = 0, cnt = 0;
        double sum = 0;
        for (int c = 0; c < n; c += TRK_THREADS) {
            const int li = c + tid, i = base + li;
            const bool valid = li < n;
            bool keep = false, has = false;
            float2 f = make_float2(0.f, 0.f), u = f;
            if (valid) {
                keep = A.status[A.n_map + i] != 0;
                f = A.fwd[A.n_map + i];
                float p[2] = {f.x, f.y};
                gc::undistort_point(cam, p);  // :524
                u = make_float2(p[0], p[1]);
                ((float2 *) A.ref.fwd_xy)[i] = f, ((float2 *) A.ref.fwd_undis_xy)[i] = u, A.ref.keep[i] = keep;
            }
            int tot;
            const int j = base + kept + block_prefix(keep, s_warp, &tot);
            double v = 0;
            if (keep) {
                const float2 nw = ((const float2 *) A.ref.new_xy)[i];
                float q[2] = {nw.x, nw.y};
                gc::undistort_point(cam, q);  // :523
                double x1, y1, x0, y0;
                gc::pixel2cam(cam, u.x, u.y, x1, y1);
                gc::pixel2cam(cam, q[0], q[1], x0, y0);
                const double vx = (x1 - x0) / P.dt, vy = (y1 - y0) / P.dt;  // :531
                const int64_t fid = A.ref.ref_frame_id[i];
                ((float2 *) A.nu)[j] = make_float2(q[0], q[1]);
                ((float2 *) A.ref.cur_xy)[j] = f, ((float2 *) A.ref.cur_undis_xy)[j] = u;
                A.ref.velocity[2 * (size_t) j] = vx, A.ref.velocity[2 * (size_t) j + 1] = vy;
                const float2 rp = ((const float2 *) A.ref.ref_xy)[i];
                ((float2 *) A.ref.ref_out_xy)[j] = rp;
                A.ref.ref_frame_id_out[j] = fid;
                const bool newer = fid > P.ref_id;  // :536-538
                A.ref.velocity_ref_out[2 * (size_t) j] = newer ? vx : A.ref.velocity_ref[2 * (size_t) i];
                A.ref.velocity_ref_out[2 * (size_t) j + 1] = newer ? vy : A.ref.velocity_ref[2 * (size_t) i + 1];
                A.ref.src[j] = li;
                has = fid == P.ref_id;  // parallaxFromReferenceKeyPoints (:911-915)
                if (has) {
                    float r[2] = {rp.x, rp.y};
                    gc::undistort_point(cam, r);  // :542-543
                    v = gc::key_point_parallax(cam, Rcr, r[0], r[1], u.x, u.y);
                }
            }
            s_val[tid] = v, s_has[tid] = has;
            __syncthreads();
            if (tid == 0)
                for (int t = 0; t < TRK_THREADS; t++)
                    if (s_has[t]) sum += s_val[t], cnt++;
            __syncthreads();
            kept += tot;
        }
        if (tid == 0) {
            A.n1[s] = kept;
            A.n_out[2 * s + 1] = kept;
            A.parallax[2 * s + 1] = kept == 0 ? 0.0 : (cnt ? sum / cnt : 0.0);
            A.par_n[2 * s + 1] = kept == 0 ? -1 : cnt;  // :459-462, :513-517 (-1: keep)
        }
    }
}

// reduceVector by the RANSAC status (:550-554), in place: a chunk is read completely before any of it is written, and its writes land at or
// before its own first index (the compacted prefix only grows), so no unread element is overwritten
__global__ void __launch_bounds__(TRK_THREADS) track_compact_kernel(TrackArgs A) {
    __shared__ int s_warp[TRK_THREADS / 32];
    const int s = blockIdx.x, tid = threadIdx.x;
    const int base = A.roff[s], n = A.n1[s];
    if (n < 15) return;  // :547
    int kept = 0;
    for (int c = 0; c < n; c += TRK_THREADS) {
        const int j = base + c + tid;
        const bool valid = c + tid < n;
        const bool in = valid && A.rmask[j] != 0;
        float2 cur, cu, rp;
        double v0 = 0, v1 = 0, r0 = 0, r1 = 0;
        int64_t fid = 0;
        int src = 0;
        if (valid) {
            cur = ((float2 *) A.ref.cur_xy)[j], cu = ((float2 *) A.ref.cur_undis_xy)[j], rp = ((float2 *) A.ref.ref_out_xy)[j];
            v0 = A.ref.velocity[2 * (size_t) j], v1 = A.ref.velocity[2 * (size_t) j + 1];
            r0 = A.ref.velocity_ref_out[2 * (size_t) j], r1 = A.ref.velocity_ref_out[2 * (size_t) j + 1];
            fid = A.ref.ref_frame_id_out[j], src = A.ref.src[j];
            if (!in) A.ref.keep[base + src] = 0;
        }
        int tot;
        const int o = base + kept + block_prefix(in, s_warp, &tot);  // contains the barriers that order the reads before the writes
        if (in) {
            ((float2 *) A.ref.cur_xy)[o] = cur, ((float2 *) A.ref.cur_undis_xy)[o] = cu, ((float2 *) A.ref.ref_out_xy)[o] = rp;
            A.ref.velocity[2 * (size_t) o] = v0, A.ref.velocity[2 * (size_t) o + 1] = v1;
            A.ref.velocity_ref_out[2 * (size_t) o] = r0, A.ref.velocity_ref_out[2 * (size_t) o + 1] = r1;
            A.ref.ref_frame_id_out[o] = fid, A.ref.src[o] = src;
        }
        __syncthreads();
        kept += tot;
    }
    if (tid == 0) A.n_out[2 * s + 1] = kept;
}

// ------------------------------------------------------------------------------------------------ Tracking::triangulation (:690-798)
constexpr int TRI_MAX_KF = 64;             // table entries per stream
constexpr double TRI_MIN_PARALLAX = 10.0;  // TRACK_MIN_PARALLAX (tracking.h:114)

struct TriKf {             // one table entry with the products the points need, computed once per CTA
    double Rck[9];         // R_cur^T R_kf: keyPointParallax with pose0 = the point's reference frame, pose1 = frame_cur_ (:741)
    double T[12];          // pose2Tcw(pose_kf) (:749)
    double R[9], t[3];     // pose_kf for world2cam (isGoodToTrack and the depth, :756, :765)
    int64_t id;
    int in_map;
};

struct TriArgs {
    const icg_tri_frame *par;
    const int32_t *koff, *roff;
    const icg_tri_keyframe *kf;
    const int32_t *n_in;
    int n_in_stride;
    icg_tri_list list;
    icg_tri_new out;
    int32_t *counts;
};

// CTA / stream: table -> shared memory, id check over the live list, then chunks of 256 points: thread per point for rules 2-8, two stable
// block-prefix compactions (kept: in place, as track_compact_kernel; new: into out from the segment start)
__global__ void __launch_bounds__(TRK_THREADS, 1) tri_kernel(TriArgs A) {
    __shared__ TriKf s_kf[TRI_MAX_KF];
    __shared__ double s_T1[12];
    __shared__ int s_warp[TRK_THREADS / 32];
    __shared__ int s_cnt[3];  // outlier, reset, outtime
    const int s = blockIdx.x, tid = threadIdx.x;
    const icg_tri_frame &P = A.par[s];
    const icg_camera &cam = P.camera;
    int32_t *cnt = A.counts + 5 * (size_t) s;
    const int base = A.roff[s], seg = A.roff[s + 1] - base;
    if (!P.triangulate) {  // not a keyframe of this stream: untouched
        if (tid == 0) cnt[0] = -1, cnt[1] = cnt[2] = cnt[3] = cnt[4] = 0;
        return;
    }
    const int n = A.n_in ? A.n_in[(size_t) s * A.n_in_stride] : seg;
    if (n < 0 || n > seg || n == 0) {  // n == 0: pts2d_cur_.empty() -> return false (:692-694)
        if (tid == 0) cnt[0] = n == 0 ? -1 : -2, cnt[1] = cnt[2] = cnt[3] = cnt[4] = 0;
        return;
    }
    const int k0 = A.koff[s], nk = A.koff[s + 1] - k0;
    for (int e = tid; e < nk; e += TRK_THREADS) {
        const icg_tri_keyframe &K = A.kf[k0 + e];
        TriKf &E = s_kf[e];
        gc::rt_mul(P.R_cur, K.R, E.Rck);
        gc::pose_tcw(K.R, K.t, E.T);
        for (int q = 0; q < 9; q++) E.R[q] = K.R[q];
        for (int q = 0; q < 3; q++) E.t[q] = K.t[q];
        E.id = K.id, E.in_map = K.in_map;
    }
    if (tid == 0) {
        gc::pose_tcw(P.R_cur, P.t_cur, s_T1);
        s_cnt[0] = s_cnt[1] = s_cnt[2] = 0;
    }
    __syncthreads();
    auto find = [&](int64_t id) {
        for (int e = 0; e < nk; e++)
            if (s_kf[e].id == id) return e;
        return -1;
    };
    // every frame a point can name must be in the table; checked before anything is written (the compaction is in place)
    bool miss = false;
    for (int li = tid; li < n; li += TRK_THREADS) {
        const int64_t fid = A.list.ref_frame_id_out[base + li];
        miss = miss || (fid <= P.ref_id && find(fid) < 0);
    }
    if (__syncthreads_or(miss)) {
        if (tid == 0) cnt[0] = -2, cnt[1] = cnt[2] = cnt[3] = cnt[4] = 0;
        return;
    }
    int kept = 0, made = 0;
    for (int c = 0; c < n; c += TRK_THREADS) {
        const int li = c + tid, i = base + li;
        const bool valid = li < n;
        bool keep = false, made_pt = false;
        float2 rp = make_float2(0.f, 0.f), cp = rp, ru = rp, cu = rp;
        int64_t fid = 0;
        double vr0 = 0, vr1 = 0, pw[3] = {0, 0, 0}, depth = 0;
        if (valid) {
            rp = ((const float2 *) A.list.ref_out_xy)[i], cp = ((const float2 *) A.list.cur_xy)[i];
            fid = A.list.ref_frame_id_out[i];
            vr0 = A.list.velocity_ref_out[2 * (size_t) i], vr1 = A.list.velocity_ref_out[2 * (size_t) i + 1];
            float r[2] = {rp.x, rp.y}, q[2] = {cp.x, cp.y};
            gc::undistort_point(cam, r);  // :708-713
            gc::undistort_point(cam, q);
            ru = make_float2(r[0], r[1]), cu = make_float2(q[0], q[1]);
            if (fid > P.ref_id) {  // :723-730, before the window test
                keep = true;
                rp = cp, fid = P.cur_id;
                atomicAdd(&s_cnt[1], 1);
            } else {
                const TriKf &E = s_kf[find(fid)];
                if (P.window_normal && !E.in_map) {  // :733-737
                    atomicAdd(&s_cnt[2], 1);
                } else if (gc::key_point_parallax(cam, E.Rck, ru.x, ru.y, cu.x, cu.y) < TRI_MIN_PARALLAX) {  // :740-745
                    keep = true;
                } else {
                    double pc0[2], pc1[2];
                    gc::pixel2cam(cam, ru.x, ru.y, pc0[0], pc0[1]);  // :750-751
                    gc::pixel2cam(cam, cu.x, cu.y, pc1[0], pc1[1]);
                    gc::triangulate_point(E.T, s_T1, pc0, pc1, pw);  // :753
                    if (gc::good_to_track(cam, ru.x, ru.y, E.R, E.t, pw, P.reprojection_error_std) &&
                        gc::good_to_track(cam, cu.x, cu.y, P.R_cur, P.t_cur, pw, P.reprojection_error_std)) {  // :756-760
                        double x, y;
                        gc::world2cam(E.R, E.t, pw, x, y, depth);  // :764-765
                        if (depth < 1.0 || depth > 200.0) depth = 10.0;  // MapPoint's constructor (mappoint.cc:39-42)
                        made_pt = true;
                    } else {
                        atomicAdd(&s_cnt[0], 1);
                    }
                }
            }
        }
        int tot_k, tot_m;
        const int j = base + kept + block_prefix(keep, s_warp, &tot_k);  // contains the barriers that order the reads before the writes
        const int o = base + made + block_prefix(made_pt, s_warp, &tot_m);
        if (keep) {  // reduceVector (:788-791)
            ((float2 *) A.list.ref_out_xy)[j] = rp, ((float2 *) A.list.cur_xy)[j] = cp;
            A.list.ref_frame_id_out[j] = fid;
            A.list.velocity_ref_out[2 * (size_t) j] = vr0, A.list.velocity_ref_out[2 * (size_t) j + 1] = vr1;
            A.list.src[j] = li;
        }
        if (made_pt) {  // :761-784
            const icg_tri_new &O = A.out;
            O.pw[3 * (size_t) o] = pw[0], O.pw[3 * (size_t) o + 1] = pw[1], O.pw[3 * (size_t) o + 2] = pw[2];
            O.depth[o] = depth;
            ((float2 *) O.ref_undis_xy)[o] = ru, ((float2 *) O.ref_xy)[o] = rp;
            ((float2 *) O.cur_undis_xy)[o] = cu, ((float2 *) O.cur_xy)[o] = cp;
            O.velocity_cur[2 * (size_t) o] = A.list.velocity[2 * (size_t) i], O.velocity_cur[2 * (size_t) o + 1] = A.list.velocity[2 * (size_t) i + 1];
            O.velocity_ref[2 * (size_t) o] = vr0, O.velocity_ref[2 * (size_t) o + 1] = vr1;
            O.ref_frame_id[o] = fid, O.src[o] = li;
        }
        kept += tot_k, made += tot_m;
    }
    __syncthreads();
    if (tid == 0) cnt[0] = kept, cnt[1] = made, cnt[2] = s_cnt[0], cnt[3] = s_cnt[1], cnt[4] = s_cnt[2];
}

}  // namespace icg

using namespace icg;

namespace {

bool bad_lists(const char *who, int n_streams, const int32_t *off, bool has_ptrs, int *total) {
    if (off[0] != 0) {
        set_error("%s: offsets must start at 0", who);
        return true;
    }
    for (int s = 0; s < n_streams; s++)
        if (off[s + 1] < off[s]) {
            set_error("%s: offsets are not monotone at stream %d", who, s);
            return true;
        }
    *total = off[n_streams];
    if (*total > 0 && !has_ptrs) {
        set_error("%s: NULL list pointer", who);
        return true;
    }
    return false;
}
bool map_ptrs(const icg_track_map *m) {
    return m && m->prev_xy && m->prev_undis_xy && m->pw && m->ref_kp_xy && m->fwd_xy && m->fwd_undis_xy && m->keep && m->cur_xy && m->cur_undis_xy &&
           m->velocity && m->src;
}
bool ref_ptrs(const icg_track_ref *r) {
    return r && r->new_xy && r->ref_xy && r->ref_frame_id && r->velocity_ref && r->fwd_xy && r->fwd_undis_xy && r->keep && r->cur_xy &&
           r->cur_undis_xy && r->velocity && r->ref_out_xy && r->ref_frame_id_out && r->velocity_ref_out && r->src;
}

int track_reserve(icg_klt *h, int n_streams) {
    if (!h->track) {
        h->track = new TrackScratch();
        TrackScratch &t = *h->track;
        if (cudaMalloc(&t.d_nu, sizeof(float) * 2 * (size_t) h->max_pts) != cudaSuccess || cudaMalloc(&t.d_rmask, (size_t) h->max_pts) != cudaSuccess ||
            cudaEventCreateWithFlags(&t.stage_ev, cudaEventDisableTiming) != cudaSuccess) {
            track_scratch_free(h->track);
            h->track = nullptr;
            set_error("icg_klt_track_frames_dev: scratch allocation failed");
            return ICG_ENOMEM;
        }
    }
    TrackScratch &t = *h->track;
    if (t.cap_streams >= n_streams) return ICG_OK;
    ICG_CUDA(cudaStreamSynchronize(h->stream));  // the old buffers may still be read by an enqueued call
    cudaFree(t.d_par), cudaFree(t.d_moff), cudaFree(t.d_roff), cudaFree(t.d_thr), cudaFree(t.d_n1), cudaFree(t.d_ninl);
    if (t.h_stage) cudaFreeHost(t.h_stage);
    t.d_par = nullptr, t.d_moff = t.d_roff = t.d_n1 = t.d_ninl = nullptr, t.d_thr = nullptr, t.h_stage = nullptr, t.cap_streams = 0;
    t.stage_pending = false;
    const size_t S = n_streams;
    t.stage_bytes = sizeof(icg_track_frame) * S + 8 * (S + 1);
    if (cudaMalloc(&t.d_par, sizeof(icg_track_frame) * S) != cudaSuccess || cudaMalloc(&t.d_moff, 4 * (S + 1)) != cudaSuccess ||
        cudaMalloc(&t.d_roff, 4 * (S + 1)) != cudaSuccess || cudaMalloc(&t.d_thr, 8 * S) != cudaSuccess || cudaMalloc(&t.d_n1, 4 * S) != cudaSuccess ||
        cudaMalloc(&t.d_ninl, 4 * S) != cudaSuccess || cudaMallocHost(&t.h_stage, t.stage_bytes) != cudaSuccess) {
        set_error("icg_klt_track_frames_dev: scratch allocation for %d streams failed", n_streams);
        return ICG_ENOMEM;
    }
    t.cap_streams = n_streams;
    return ICG_OK;
}

// the whole launch sequence; every pointer of m / r is a device pointer
int track_launch(icg_klt *h, const char *who, int n_streams, const icg_track_frame *params, const int32_t *map_off, const icg_track_map *m,
                 const int32_t *ref_off, const icg_track_ref *r, int32_t *dev_n_out, double *dev_parallax, int32_t *dev_parallax_n) {
    if (!h || n_streams < 1 || !params || !map_off || !ref_off || !dev_n_out || !dev_parallax || !dev_parallax_n) {
        set_error("%s: bad arguments", who);
        return ICG_EINVAL;
    }
    int n_map, n_ref;
    if (bad_lists(who, n_streams, map_off, map_ptrs(m), &n_map) || bad_lists(who, n_streams, ref_off, ref_ptrs(r), &n_ref)) return ICG_EINVAL;
    if (n_map + n_ref > h->max_pts) {
        set_error("%s: %d points exceed max_points=%d of the handle", who, n_map + n_ref, h->max_pts);
        return ICG_EINVAL;
    }
    for (int s = 0; s < n_streams; s++) {
        const icg_track_frame &P = params[s];
        if (P.prev_slot < 0 || P.prev_slot >= h->n_slots || P.cur_slot < 0 || P.cur_slot >= h->n_slots || !(P.camera.fx != 0.0) || !(P.camera.fy != 0.0)) {
            set_error("%s: bad slot or camera in stream %d", who, s);
            return ICG_EINVAL;
        }
    }
    ICG_CUDA(cudaSetDevice(h->device));
    int rc = track_reserve(h, n_streams);
    if (rc != ICG_OK) return rc;
    TrackScratch &t = *h->track;
    if (t.stage_pending) ICG_CUDA(cudaEventSynchronize(t.stage_ev));
    t.stage_pending = false;
    const size_t S = n_streams, pb = sizeof(icg_track_frame) * S;
    memcpy(t.h_stage, params, pb);
    memcpy(t.h_stage + pb, map_off, 4 * (S + 1));
    memcpy(t.h_stage + pb + 4 * (S + 1), ref_off, 4 * (S + 1));
    ICG_CUDA(cudaMemcpyAsync(t.d_par, t.h_stage, pb, cudaMemcpyHostToDevice, h->stream));
    ICG_CUDA(cudaMemcpyAsync(t.d_moff, t.h_stage + pb, 4 * (S + 1), cudaMemcpyHostToDevice, h->stream));
    ICG_CUDA(cudaMemcpyAsync(t.d_roff, t.h_stage + pb + 4 * (S + 1), 4 * (S + 1), cudaMemcpyHostToDevice, h->stream));
    ICG_CUDA(cudaEventRecord(t.stage_ev, h->stream));
    t.stage_pending = true;

    static const icg_track_map no_map = {};
    static const icg_track_ref no_ref = {};
    TrackArgs A;
    A.n_streams = n_streams, A.n_map = n_map, A.n_ref = n_ref;
    A.par = t.d_par, A.moff = t.d_moff, A.roff = t.d_roff;
    A.map = m ? *m : no_map, A.ref = r ? *r : no_ref;
    // the KLT batch lives in the handle's scratch of the host-pointer API (max_points entries; stream-ordered with the synchronous calls)
    A.slots = h->d_slots, A.prev = (float2 *) h->d_prev, A.init = (float2 *) h->d_init, A.fwd = (float2 *) h->d_fwd, A.status = h->d_status;
    A.thr = t.d_thr, A.n1 = t.d_n1, A.ninl = t.d_ninl, A.nu = t.d_nu, A.rmask = t.d_rmask;
    A.n_out = dev_n_out, A.par_n = dev_parallax_n, A.parallax = dev_parallax;
    const int n_pred = n_map + n_ref > n_streams ? n_map + n_ref : n_streams;
    track_predict_kernel<<<(n_pred + 127) / 128, 128, 0, h->stream>>>(A);
    ICG_CHECK_LAUNCH();
    count_launch();
    rc = icg_klt_track_batch_dev(h, n_map + n_ref, h->d_slots, h->d_prev, h->d_init, h->d_fwd, h->d_bwd, h->d_status, 1);
    if (rc != ICG_OK) return rc;
    track_post_kernel<<<n_streams, TRK_THREADS, 0, h->stream>>>(A);
    ICG_CHECK_LAUNCH();
    count_launch();
    if (n_ref > 0) {
        RansacBatch B;
        B.off = t.d_roff, B.n = t.d_n1, B.p1 = t.d_nu, B.p2 = r->cur_undis_xy, B.thr = t.d_thr, B.conf = nullptr, B.max_iters = 1000;
        B.mask = t.d_rmask, B.n_inliers = t.d_ninl, B.F = nullptr, B.stats = nullptr;
        rc = ransac_batch_launch(h->stream, n_streams, B);
        if (rc != ICG_OK) return rc;
        track_compact_kernel<<<n_streams, TRK_THREADS, 0, h->stream>>>(A);
        ICG_CHECK_LAUNCH();
        count_launch();
    }
    return ICG_OK;
}

bool tri_list_ptrs(const icg_tri_list *l) { return l && l->ref_out_xy && l->ref_frame_id_out && l->cur_xy && l->velocity_ref_out && l->velocity && l->src; }
bool tri_new_ptrs(const icg_tri_new *o) {
    return o && o->pw && o->depth && o->ref_undis_xy && o->ref_xy && o->cur_undis_xy && o->cur_xy && o->velocity_cur && o->velocity_ref && o->ref_frame_id &&
           o->src;
}

// the triangulation launch; every pointer of list / out and dev_n_in / dev_counts are device pointers
int tri_launch(icg_klt *h, const char *who, int n_streams, const icg_tri_frame *params, const int32_t *kf_off, const icg_tri_keyframe *kf,
               const int32_t *ref_off, const int32_t *dev_n_in, int n_in_stride, const icg_tri_list *list, const icg_tri_new *out, int32_t *dev_counts) {
    if (!h || n_streams < 1 || !params || !kf_off || !ref_off || !dev_counts || (dev_n_in && n_in_stride < 1)) {
        set_error("%s: bad arguments", who);
        return ICG_EINVAL;
    }
    int n_kf, n_pts;
    if (bad_lists(who, n_streams, kf_off, kf != nullptr, &n_kf)) return ICG_EINVAL;
    if (bad_lists(who, n_streams, ref_off, tri_list_ptrs(list) && tri_new_ptrs(out), &n_pts)) return ICG_EINVAL;
    for (int s = 0; s < n_streams; s++) {
        const icg_tri_frame &P = params[s];
        if (!(P.camera.fx != 0.0) || !(P.camera.fy != 0.0)) {
            set_error("%s: bad camera in stream %d", who, s);
            return ICG_EINVAL;
        }
        const int k0 = kf_off[s], nk = kf_off[s + 1] - k0;
        if (nk > TRI_MAX_KF) {
            set_error("%s: %d keyframes in stream %d exceed %d", who, nk, s, TRI_MAX_KF);
            return ICG_EINVAL;
        }
        for (int a = 0; a < nk; a++)
            for (int b = 0; b < a; b++)
                if (kf[k0 + a].id == kf[k0 + b].id) {
                    set_error("%s: duplicate keyframe id %lld in stream %d", who, (long long) kf[k0 + a].id, s);
                    return ICG_EINVAL;
                }
    }
    ICG_CUDA(cudaSetDevice(h->device));
    int rc = track_reserve(h, 1);  // creates the handle's scratch (stage event) on first use
    if (rc != ICG_OK) return rc;
    TrackScratch &t = *h->track;
    const size_t S = n_streams, pb = (sizeof(icg_tri_frame) * S + 15) & ~(size_t) 15, ob = (4 * (S + 1) + 15) & ~(size_t) 15;
    const size_t bytes = pb + 2 * ob + sizeof(icg_tri_keyframe) * (size_t) n_kf;
    if (t.stage_pending) ICG_CUDA(cudaEventSynchronize(t.stage_ev));
    t.stage_pending = false;
    if (t.tri_bytes < bytes) {
        ICG_CUDA(cudaStreamSynchronize(h->stream));  // the old device blob may still be read by an enqueued call
        if (t.h_tri) cudaFreeHost(t.h_tri);
        if (t.d_tri) cudaFree(t.d_tri);
        t.h_tri = t.d_tri = nullptr, t.tri_bytes = 0;
        if (cudaMallocHost(&t.h_tri, bytes) != cudaSuccess || cudaMalloc(&t.d_tri, bytes) != cudaSuccess) {
            set_error("%s: staging allocation of %zu bytes failed", who, bytes);
            return ICG_ENOMEM;
        }
        t.tri_bytes = bytes;
    }
    memcpy(t.h_tri, params, sizeof(icg_tri_frame) * S);
    memcpy(t.h_tri + pb, kf_off, 4 * (S + 1));
    memcpy(t.h_tri + pb + ob, ref_off, 4 * (S + 1));
    if (n_kf) memcpy(t.h_tri + pb + 2 * ob, kf, sizeof(icg_tri_keyframe) * (size_t) n_kf);
    ICG_CUDA(cudaMemcpyAsync(t.d_tri, t.h_tri, bytes, cudaMemcpyHostToDevice, h->stream));
    ICG_CUDA(cudaEventRecord(t.stage_ev, h->stream));
    t.stage_pending = true;

    static const icg_tri_list no_list = {};
    static const icg_tri_new no_new = {};
    TriArgs A;
    A.par = (const icg_tri_frame *) t.d_tri, A.koff = (const int32_t *) (t.d_tri + pb), A.roff = (const int32_t *) (t.d_tri + pb + ob);
    A.kf = (const icg_tri_keyframe *) (t.d_tri + pb + 2 * ob);
    A.n_in = dev_n_in, A.n_in_stride = n_in_stride;
    A.list = n_pts ? *list : no_list, A.out = n_pts ? *out : no_new;
    A.counts = dev_counts;
    tri_kernel<<<n_streams, TRK_THREADS, 0, h->stream>>>(A);
    ICG_CHECK_LAUNCH();
    count_launch();
    return ICG_OK;
}

}  // namespace

extern "C" {

int icg_klt_triangulate_dev(icg_klt *h, int n_streams, const icg_tri_frame *params, const int32_t *kf_off, const icg_tri_keyframe *kf,
                            const int32_t *ref_off, const int32_t *dev_n_in, int n_in_stride, const icg_tri_list *list, const icg_tri_new *out,
                            int32_t *dev_counts) {
    return tri_launch(h, "icg_klt_triangulate_dev", n_streams, params, kf_off, kf, ref_off, dev_n_in, n_in_stride, list, out, dev_counts);
}

int icg_klt_triangulate(icg_klt *h, const icg_tri_frame *params, int n_kf, const icg_tri_keyframe *kf, int n, const icg_tri_list *list,
                        const icg_tri_new *out, int32_t *counts) {
    const char *who = "icg_klt_triangulate";
    if (!h || !params || n_kf < 0 || (n_kf > 0 && !kf) || n < 0 || !counts || (n > 0 && (!tri_list_ptrs(list) || !tri_new_ptrs(out)))) {
        set_error("%s: bad arguments", who);
        return ICG_EINVAL;
    }
    if (n > h->max_pts) {
        set_error("%s: %d points exceed max_points=%d of the handle", who, n, h->max_pts);
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    int rc = track_reserve(h, 1);
    if (rc != ICG_OK) return rc;
    TrackScratch &t = *h->track;
    // device copies, max_points entries each: list 60 bytes / point, out 108, + the 5 counts
    const size_t P = h->max_pts;
    if (!t.d_tri_host && cudaMalloc(&t.d_tri_host, P * 168 + 32) != cudaSuccess) {
        t.d_tri_host = nullptr;
        set_error("%s: scratch allocation failed", who);
        return ICG_ENOMEM;
    }
    uint8_t *q = t.d_tri_host;
    auto take = [&](size_t bytes) {
        uint8_t *p = q;
        q += bytes;
        return p;
    };
    icg_tri_list dl;
    icg_tri_new dn;
    dl.ref_frame_id_out = (int64_t *) take(8 * P), dl.velocity_ref_out = (double *) take(16 * P), dl.velocity = (const double *) take(16 * P);
    dn.pw = (double *) take(24 * P), dn.depth = (double *) take(8 * P), dn.velocity_cur = (double *) take(16 * P), dn.velocity_ref = (double *) take(16 * P);
    dn.ref_frame_id = (int64_t *) take(8 * P);
    dl.ref_out_xy = (float *) take(8 * P), dl.cur_xy = (float *) take(8 * P);
    dn.ref_undis_xy = (float *) take(8 * P), dn.ref_xy = (float *) take(8 * P), dn.cur_undis_xy = (float *) take(8 * P), dn.cur_xy = (float *) take(8 * P);
    dl.src = (int32_t *) take(4 * P), dn.src = (int32_t *) take(4 * P);
    int32_t *d_cnt = (int32_t *) take(32);
    auto h2d = [&](const void *dst, const void *src, size_t bytes) -> int {
        if (bytes) ICG_CUDA(cudaMemcpyAsync((void *) dst, src, bytes, cudaMemcpyHostToDevice, h->stream));
        return ICG_OK;
    };
    auto d2h = [&](void *dst, const void *src, size_t bytes) -> int {
        if (bytes) ICG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, h->stream));
        return ICG_OK;
    };
    const size_t N = n;
    if (N && ((rc = h2d(dl.ref_out_xy, list->ref_out_xy, 8 * N)) || (rc = h2d(dl.ref_frame_id_out, list->ref_frame_id_out, 8 * N)) ||
              (rc = h2d(dl.cur_xy, list->cur_xy, 8 * N)) || (rc = h2d(dl.velocity_ref_out, list->velocity_ref_out, 16 * N)) ||
              (rc = h2d(dl.velocity, list->velocity, 16 * N))))
        return rc;
    const int32_t koff[2] = {0, n_kf}, roff[2] = {0, n};
    rc = tri_launch(h, who, 1, params, koff, kf, roff, nullptr, 1, &dl, &dn, d_cnt);
    if (rc != ICG_OK) return rc;
    if ((rc = d2h(counts, d_cnt, 20))) return rc;
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    const size_t K = counts[0] > 0 ? counts[0] : 0, M = counts[0] >= 0 ? counts[1] : 0;
    if (K && ((rc = d2h(list->ref_out_xy, dl.ref_out_xy, 8 * K)) || (rc = d2h(list->ref_frame_id_out, dl.ref_frame_id_out, 8 * K)) ||
              (rc = d2h(list->cur_xy, dl.cur_xy, 8 * K)) || (rc = d2h(list->velocity_ref_out, dl.velocity_ref_out, 16 * K)) ||
              (rc = d2h(list->src, dl.src, 4 * K))))
        return rc;
    if (M && ((rc = d2h(out->pw, dn.pw, 24 * M)) || (rc = d2h(out->depth, dn.depth, 8 * M)) || (rc = d2h(out->ref_undis_xy, dn.ref_undis_xy, 8 * M)) ||
              (rc = d2h(out->ref_xy, dn.ref_xy, 8 * M)) || (rc = d2h(out->cur_undis_xy, dn.cur_undis_xy, 8 * M)) ||
              (rc = d2h(out->cur_xy, dn.cur_xy, 8 * M)) || (rc = d2h(out->velocity_cur, dn.velocity_cur, 16 * M)) ||
              (rc = d2h(out->velocity_ref, dn.velocity_ref, 16 * M)) || (rc = d2h(out->ref_frame_id, dn.ref_frame_id, 8 * M)) ||
              (rc = d2h(out->src, dn.src, 4 * M))))
        return rc;
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    return ICG_OK;
}


int icg_klt_track_frames_dev(icg_klt *h, int n_streams, const icg_track_frame *params, const int32_t *map_off, const icg_track_map *map,
                             const int32_t *ref_off, const icg_track_ref *ref, int32_t *dev_n_out, double *dev_parallax, int32_t *dev_parallax_n) {
    return track_launch(h, "icg_klt_track_frames_dev", n_streams, params, map_off, map, ref_off, ref, dev_n_out, dev_parallax, dev_parallax_n);
}

int icg_klt_track_frame(icg_klt *h, const icg_track_frame *params, int n_map, const icg_track_map *map, int n_ref, const icg_track_ref *ref,
                        int32_t *n_out, double *parallax, int32_t *parallax_n) {
    const char *who = "icg_klt_track_frame";
    if (!h || !params || n_map < 0 || n_ref < 0 || !n_out || !parallax || !parallax_n || (n_map > 0 && !map_ptrs(map)) || (n_ref > 0 && !ref_ptrs(ref))) {
        set_error("%s: bad arguments", who);
        return ICG_EINVAL;
    }
    if (n_map + n_ref > h->max_pts) {
        set_error("%s: %d points exceed max_points=%d of the handle", who, n_map + n_ref, h->max_pts);
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    int rc = track_reserve(h, 1);
    if (rc != ICG_OK) return rc;
    TrackScratch &t = *h->track;
    // device copies of both lists, max_points entries each: map 101 bytes / point, ref 125, + the 6 result scalars
    const size_t P = h->max_pts;
    const size_t map_b = P * 101, ref_b = P * 125;
    if (!t.d_host && cudaMalloc(&t.d_host, map_b + ref_b + 64) != cudaSuccess) {
        t.d_host = nullptr;
        set_error("%s: scratch allocation failed", who);
        return ICG_ENOMEM;
    }
    uint8_t *q = t.d_host;
    auto take = [&](size_t bytes) {
        uint8_t *p = q;
        q += bytes;
        return p;
    };
    // 8-byte arrays of both lists first, then the 4-byte ones, then the 1-byte ones: every array stays aligned for any max_points
    icg_track_map dm;
    icg_track_ref dr;
    dm.pw = (const double *) take(24 * P), dm.velocity = (double *) take(16 * P);
    dm.prev_xy = (const float *) take(8 * P), dm.prev_undis_xy = (const float *) take(8 * P), dm.ref_kp_xy = (const float *) take(8 * P);
    dm.fwd_xy = (float *) take(8 * P), dm.fwd_undis_xy = (float *) take(8 * P), dm.cur_xy = (float *) take(8 * P), dm.cur_undis_xy = (float *) take(8 * P);
    dr.ref_frame_id = (const int64_t *) take(8 * P), dr.velocity_ref = (const double *) take(16 * P), dr.velocity = (double *) take(16 * P);
    dr.ref_frame_id_out = (int64_t *) take(8 * P), dr.velocity_ref_out = (double *) take(16 * P);
    dr.new_xy = (const float *) take(8 * P), dr.ref_xy = (const float *) take(8 * P), dr.fwd_xy = (float *) take(8 * P), dr.fwd_undis_xy = (float *) take(8 * P);
    dr.cur_xy = (float *) take(8 * P), dr.cur_undis_xy = (float *) take(8 * P), dr.ref_out_xy = (float *) take(8 * P);
    double *d_par = (double *) take(16);
    int32_t *d_n = (int32_t *) take(8), *d_pn = (int32_t *) take(8);
    dm.src = (int32_t *) take(4 * P), dr.src = (int32_t *) take(4 * P);
    dm.keep = take(P), dr.keep = take(P);
    auto h2d = [&](const void *dst, const void *src, size_t bytes) -> int {
        if (bytes) ICG_CUDA(cudaMemcpyAsync((void *) dst, src, bytes, cudaMemcpyHostToDevice, h->stream));
        return ICG_OK;
    };
    auto d2h = [&](void *dst, const void *src, size_t bytes) -> int {
        if (bytes) ICG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, h->stream));
        return ICG_OK;
    };
    const size_t M = n_map, R = n_ref;
    if (M) {
        if ((rc = h2d(dm.prev_xy, map->prev_xy, 8 * M)) || (rc = h2d(dm.prev_undis_xy, map->prev_undis_xy, 8 * M)) || (rc = h2d(dm.pw, map->pw, 24 * M)) ||
            (rc = h2d(dm.ref_kp_xy, map->ref_kp_xy, 8 * M)))
            return rc;
    }
    if (R) {
        if ((rc = h2d(dr.new_xy, ref->new_xy, 8 * R)) || (rc = h2d(dr.ref_xy, ref->ref_xy, 8 * R)) || (rc = h2d(dr.ref_frame_id, ref->ref_frame_id, 8 * R)) ||
            (rc = h2d(dr.velocity_ref, ref->velocity_ref, 16 * R)))
            return rc;
    }
    const int32_t moff[2] = {0, n_map}, roff[2] = {0, n_ref};
    rc = track_launch(h, who, 1, params, moff, &dm, roff, &dr, d_n, d_par, d_pn);
    if (rc != ICG_OK) return rc;
    if (M) {
        if ((rc = d2h(map->fwd_xy, dm.fwd_xy, 8 * M)) || (rc = d2h(map->fwd_undis_xy, dm.fwd_undis_xy, 8 * M)) || (rc = d2h(map->keep, dm.keep, M)) ||
            (rc = d2h(map->cur_xy, dm.cur_xy, 8 * M)) || (rc = d2h(map->cur_undis_xy, dm.cur_undis_xy, 8 * M)) || (rc = d2h(map->velocity, dm.velocity, 16 * M)) ||
            (rc = d2h(map->src, dm.src, 4 * M)))
            return rc;
    }
    if (R) {
        if ((rc = d2h(ref->fwd_xy, dr.fwd_xy, 8 * R)) || (rc = d2h(ref->fwd_undis_xy, dr.fwd_undis_xy, 8 * R)) || (rc = d2h(ref->keep, dr.keep, R)) ||
            (rc = d2h(ref->cur_xy, dr.cur_xy, 8 * R)) || (rc = d2h(ref->cur_undis_xy, dr.cur_undis_xy, 8 * R)) || (rc = d2h(ref->velocity, dr.velocity, 16 * R)) ||
            (rc = d2h(ref->ref_out_xy, dr.ref_out_xy, 8 * R)) || (rc = d2h(ref->ref_frame_id_out, dr.ref_frame_id_out, 8 * R)) ||
            (rc = d2h(ref->velocity_ref_out, dr.velocity_ref_out, 16 * R)) || (rc = d2h(ref->src, dr.src, 4 * R)))
            return rc;
    }
    if ((rc = d2h(n_out, d_n, 8)) || (rc = d2h(parallax, d_par, 16)) || (rc = d2h(parallax_n, d_pn, 8))) return rc;
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    return ICG_OK;
}

}  // extern "C"
