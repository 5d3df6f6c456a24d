// geom.cu -- SURVEY.md 8f ranks 2-4 on the device: the point-wise geometry of the front end and the IMU propagation, batched.
//
//   icg_geom_undistort_points / icg_geom_distort_points   Camera::undistortPoints / distortPoints (IG/tracking/camera.cc:72-104), thread / point
//   icg_geom_find_fundamental_mat_ransac[_batch]           cv::findFundamentalMat(FM_RANSAC) of Tracking::trackReferenceFrame (tracking.cc:547)
//        on S point sets, a cluster of CTAs or one CTA per set (geom_ransac_batch_kernel): rounds of subsets (one per thread) of the set's cv::RNG stream, drawn serially by
//        one thread, solved (thread / subset: 7-point null space + cubic) and scored (warp / model) in parallel, then OpenCV's serial
//        acceptance rule and adaptive iteration bound replayed on the round's counts; the next round is drawn only while the bound is not
//        reached.  The unbatched entry is a batch of one; track.cu runs the same kernel on the reference-list survivors
//   icg_geom_triangulate_points                            Tracking::triangulatePoint (tracking.cc:796-808), thread / pair (4 x 4 one-sided Jacobi)
//   icg_geom_imu_preintegrate_batch                        PreintegrationEarth / Normal propagation (preintegration_earth.cc:205-303) of many
//        intervals at once (doReintegration, IG/ic_gvins.cc:1680-1695; throughput mode): warp / interval (preint.cu)
//
// The arithmetic is the host code of camera.cu / fundamental.cu / ba.cu compiled for the device (shared __host__ __device__ cores in
// geom_core.cuh), -fmad=false: same operation order, IEEE double; only libm calls (sin, cos, acos, pow, log) differ in the last ulp.
#include <float.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include <cooperative_groups.h>

#include "common.cuh"
#include "geom_core.cuh"
#include "preint.cuh"

namespace icg {

namespace cg = cooperative_groups;

__global__ void geom_undistort_kernel(icg_camera c, float *pts, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) gc::undistort_point(c, pts + 2 * (size_t) i);
}
__global__ void geom_distort_kernel(icg_camera c, float *pts, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) gc::distort_point(c, pts + 2 * (size_t) i);
}

// cv::findFundamentalMat(FM_RANSAC) of S point sets, one cluster of CL CTAs (RS_CTA threads each) per set, in rounds of CL * RS_CTA subsets:
// thread 0 of CTA 0 draws the next subsets of the set's cv::RNG(-1) stream (RANSACPointSetRegistrator::getSubset, collinearity re-draws
// included; the draw is the serial part), one thread per subset solves its 7-point models, each warp scores its CTA's models against all
// pairs, then thread 0 of CTA 0 replays OpenCV's serial acceptance on the round's counts (read over distributed shared memory) in iteration
// order -- strictly better than the best so far and than 6, iteration bound updated after every improvement (RANSACPointSetRegistrator::run,
// ptsetreg.cpp).  The next round is drawn only while the bound is not reached, so the work stops near the adaptive bound.  n < 15 or no
// drawable first subset: all-zero mask, 0 inliers.  A round costs about one 7-point solve (a serial chain of FP64 divisions and square roots
// in the Jacobi sweeps) per SM, so a few sets spread their rounds after the first over a cluster of SMs (CL = RS_CLUSTER: 1 000 iterations in
// 3 rounds) and large batches use one CTA per set (CL = 1).
template <int CL>
__global__ void __launch_bounds__(RS_CTA) geom_ransac_batch_kernel(RansacBatch B) {
    constexpr int R = CL * RS_CTA;  // subsets per round
    __shared__ int s_idx[R * 7], s_nm[RS_CTA], s_good[RS_CTA * 3];
    __shared__ double s_F[RS_CTA * 27], s_best[9];
    __shared__ int s_drawn, s_stop, s_max_good;
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = CL > 1 ? (int) cluster.block_rank() : 0;
    auto cl_sync = [&]() {
        if (CL > 1) cluster.sync();
        else __syncthreads();
    };
    auto at0 = [&](auto *p) { return CL > 1 ? cluster.map_shared_rank(p, 0) : p; };  // CTA 0's copy
    const int set = blockIdx.x / CL, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int base = B.off[set], n = B.n ? B.n[set] : B.off[set + 1] - base;
    const float *p1 = B.p1 + 2 * (size_t) base, *p2 = B.p2 + 2 * (size_t) base;
    double thr = B.thr ? B.thr[set] : 3.0, conf = B.conf ? B.conf[set] : 0.99;
    if (thr <= 0) thr = 3;
    if (conf < DBL_EPSILON || conf > 1 - DBL_EPSILON) conf = 0.99;
    const long long t_start = clock64();
    long long t_draw = 0;
    int drawn_total = 0;
    gc::CvRng rng;  // used by thread 0 of CTA 0 only
    int niters = B.max_iters, max_good = 0, iter0 = 0;
    bool fail = false;  // the last draw found no subset
    const bool lead = rank == 0 && tid == 0;
    if (tid == 0) s_max_good = 0;
    if (n >= 15) {
        const int *idx0 = at0(s_idx);
        const int *drawn0 = at0(&s_drawn), *stop0 = at0(&s_stop);
        for (;;) {
            if (lead) {
                const long long t0 = clock64();
                // the first round stays at one CTA's worth: its serial draw is short, and it usually reaches the adaptive bound
                const int cap = iter0 == 0 ? RS_CTA : R;
                int d = 0;
                while (d < cap && iter0 + d < niters) {
                    if (!gc::draw_subset(rng, p1, p2, n, s_idx + 7 * d)) {
                        fail = true;
                        break;
                    }
                    d++;
                }
                t_draw += clock64() - t0;
                drawn_total += d;
                s_drawn = d;
            }
            cl_sync();
            const int drawn = *drawn0, mine = min(max(drawn - rank * RS_CTA, 0), RS_CTA);  // this CTA's subsets: rank * RS_CTA + [0, mine)
            if (tid < mine) {
                float ms1[14], ms2[14];
                for (int i = 0; i < 7; i++) {
                    const int v = idx0[7 * (rank * RS_CTA + tid) + i];
                    ms1[2 * i] = p1[2 * v], ms1[2 * i + 1] = p1[2 * v + 1], ms2[2 * i] = p2[2 * v], ms2[2 * i + 1] = p2[2 * v + 1];
                }
                double Fm[3][9];
                const int nm = gc::run_7point(ms1, ms2, Fm);
                s_nm[tid] = nm;
                for (int k = 0; k < 3; k++)
                    for (int e = 0; e < 9; e++) s_F[(tid * 3 + k) * 9 + e] = (k < nm && nm > 0) ? Fm[k][e] : 0.0;
            }
            __syncthreads();
            for (int m = warp; m < 3 * mine; m += RS_CTA / 32) {
                const int it = m / 3, k = m - 3 * it;
                int cnt = 0;
                if (k < s_nm[it])
                    for (int i = lane; i < n; i += 32) cnt += gc::is_inlier(p1, p2, i, s_F + (size_t) m * 9, thr) ? 1 : 0;
                for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
                if (lane == 0) s_good[m] = cnt;
            }
            cl_sync();
            if (lead) {
                for (int it = 0; it < drawn && iter0 + it < niters; it++) {
                    const int r = it / RS_CTA, j = it - r * RS_CTA;
                    const int *nm_r = CL > 1 ? cluster.map_shared_rank(s_nm, r) : s_nm, *good_r = CL > 1 ? cluster.map_shared_rank(s_good, r) : s_good;
                    const double *F_r = CL > 1 ? cluster.map_shared_rank(s_F, r) : s_F;
                    const int nm = nm_r[j];
                    for (int k = 0; k < nm; k++) {
                        const int g = good_r[3 * j + k];
                        if (g > (max_good > 6 ? max_good : 6)) {
                            for (int e = 0; e < 9; e++) s_best[e] = F_r[(3 * j + k) * 9 + e];
                            max_good = g;
                            niters = gc::update_num_iters(conf, (double) (n - g) / n, 7, niters);
                        }
                    }
                }
                iter0 += drawn;
                s_max_good = max_good;
                s_stop = fail || drawn == 0 || iter0 >= niters;  // read by all after the barrier below, rewritten only after the next round's second
            }
            cl_sync();
            if (*stop0) break;
        }
    }
    cl_sync();  // n < 15: CTA 0's s_max_good is initialised and every CTA of the cluster has started before it is read
    const int good = *at0(&s_max_good);
    double best[9];
    const double *b0 = at0(s_best);
    for (int e = 0; e < 9; e++) best[e] = good > 0 ? b0[e] : 0.0;
    for (int i = rank * RS_CTA + tid; i < (n > 0 ? n : 0); i += R) B.mask[base + i] = good > 0 && gc::is_inlier(p1, p2, i, best, thr) ? 1 : 0;
    if (lead) {
        B.n_inliers[set] = good;
        if (B.F) for (int e = 0; e < 9; e++) B.F[9 * (size_t) set + e] = best[e];
        if (B.stats) {
            B.stats[3 * (size_t) set] = drawn_total;
            B.stats[3 * (size_t) set + 1] = t_draw;
            B.stats[3 * (size_t) set + 2] = clock64() - t_start;
        }
    }
    cl_sync();  // CTA 0's shared memory stays alive until every CTA of the cluster has read it
}

int ransac_batch_launch(cudaStream_t st, int n_sets, const RansacBatch &B) {
    if (n_sets <= 0) return ICG_OK;
    int dev = 0, n_sm = 0;
    ICG_CUDA(cudaGetDevice(&dev));
    ICG_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    if (n_sets * RS_CLUSTER <= 4 * n_sm) {  // few sets: one cluster of SMs per set
        cudaLaunchConfig_t cfg = {};
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = RS_CLUSTER, attr[0].val.clusterDim.y = 1, attr[0].val.clusterDim.z = 1;
        cfg.gridDim = dim3(n_sets * RS_CLUSTER), cfg.blockDim = dim3(RS_CTA), cfg.dynamicSmemBytes = 0, cfg.stream = st;
        cfg.attrs = attr, cfg.numAttrs = 1;
        ICG_CUDA(cudaLaunchKernelEx(&cfg, geom_ransac_batch_kernel<RS_CLUSTER>, B));
    } else {
        geom_ransac_batch_kernel<1><<<n_sets, RS_CTA, 0, st>>>(B);
    }
    ICG_CHECK_LAUNCH();
    count_launch();
    return ICG_OK;
}

__global__ void geom_triangulate_kernel(const double *Tcw0, const double *Tcw1, const double *pc0, const double *pc1, int n, double *pw) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) gc::triangulate_point(Tcw0 + 12 * (size_t) i, Tcw1, pc0 + 2 * (size_t) i, pc1 + 2 * (size_t) i, pw + 3 * (size_t) i);
}

}  // namespace icg

using namespace icg;

struct icg_geom {
    int device;
    cudaStream_t stream;
    bool own_stream;
    uint8_t *d_buf = nullptr, *h_buf = nullptr;  // one device + one pinned scratch arena, grown on demand
    size_t d_bytes = 0, h_bytes = 0;
    // per-set parameters of the asynchronous batched RANSAC: their H2D copy completes at stage_ev, the next call waits for it
    uint8_t *d_b = nullptr, *h_b = nullptr;
    size_t b_bytes = 0;
    cudaEvent_t stage_ev = nullptr;
    bool stage_pending = false;
};

static int geom_reserve(icg_geom *h, size_t bytes) {
    bytes = (bytes + 255) & ~(size_t) 255;
    if (h->d_bytes >= bytes) return ICG_OK;
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    if (h->d_buf) cudaFree(h->d_buf);
    if (h->h_buf) cudaFreeHost(h->h_buf);
    h->d_buf = h->h_buf = nullptr, h->d_bytes = h->h_bytes = 0;
    if (cudaMalloc(&h->d_buf, bytes) != cudaSuccess || cudaMallocHost(&h->h_buf, bytes) != cudaSuccess) {
        set_error("icg_geom: scratch allocation of %zu bytes failed", bytes);
        return ICG_ENOMEM;
    }
    h->d_bytes = h->h_bytes = bytes;
    return ICG_OK;
}

extern "C" {

int icg_geom_create(icg_geom **out, int device, void *stream) {
    if (!out) {
        set_error("icg_geom_create: bad arguments");
        return ICG_EINVAL;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        set_error("icg_geom_create: no CUDA device (this library has no CPU fallback)");
        return ICG_ENODEVICE;
    }
    if (device < 0 || device >= ndev) {
        set_error("icg_geom_create: device %d out of range", device);
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    ICG_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error("icg_geom_create: device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor);
        return ICG_ENODEVICE;
    }
    icg_geom *h = new icg_geom();
    h->device = device, h->own_stream = stream == nullptr;
    if (stream) {
        h->stream = (cudaStream_t) stream;
    } else if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete h;
        set_error("icg_geom_create: stream creation failed");
        return ICG_ECUDA;
    }
    *out = h;
    return ICG_OK;
}

void icg_geom_destroy(icg_geom *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    if (h->d_buf) cudaFree(h->d_buf);
    if (h->h_buf) cudaFreeHost(h->h_buf);
    if (h->d_b) cudaFree(h->d_b);
    if (h->h_b) cudaFreeHost(h->h_b);
    if (h->stage_ev) cudaEventDestroy(h->stage_ev);
    if (h->own_stream) cudaStreamDestroy(h->stream);
    delete h;
}

static int geom_points(icg_geom *h, const icg_camera *c, float *pts_xy, int n, int undistort) {
    if (!h || !c || (!pts_xy && n > 0) || n < 0 || !(c->fx != 0.0) || !(c->fy != 0.0)) {
        set_error("icg_geom_%s_points: bad arguments", undistort ? "undistort" : "distort");
        return ICG_EINVAL;
    }
    if (n == 0) return ICG_OK;
    ICG_CUDA(cudaSetDevice(h->device));
    int rc = geom_reserve(h, sizeof(float) * 2 * (size_t) n);
    if (rc != ICG_OK) return rc;
    memcpy(h->h_buf, pts_xy, sizeof(float) * 2 * (size_t) n);
    ICG_CUDA(cudaMemcpyAsync(h->d_buf, h->h_buf, sizeof(float) * 2 * (size_t) n, cudaMemcpyHostToDevice, h->stream));
    if (undistort)
        geom_undistort_kernel<<<(n + 127) / 128, 128, 0, h->stream>>>(*c, (float *) h->d_buf, n);
    else
        geom_distort_kernel<<<(n + 127) / 128, 128, 0, h->stream>>>(*c, (float *) h->d_buf, n);
    ICG_CHECK_LAUNCH();
    count_launch();
    ICG_CUDA(cudaMemcpyAsync(h->h_buf, h->d_buf, sizeof(float) * 2 * (size_t) n, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    memcpy(pts_xy, h->h_buf, sizeof(float) * 2 * (size_t) n);
    return ICG_OK;
}
int icg_geom_undistort_points(icg_geom *h, const icg_camera *c, float *pts_xy, int n) { return geom_points(h, c, pts_xy, n, 1); }
int icg_geom_distort_points(icg_geom *h, const icg_camera *c, float *pts_xy, int n) { return geom_points(h, c, pts_xy, n, 0); }

int icg_geom_find_fundamental_mat_ransac(icg_geom *h, const float *pts1_xy, const float *pts2_xy, int n, double threshold, double confidence, int max_iters,
                                         uint8_t *status, double *F9) {
    if (!h || !pts1_xy || !pts2_xy || !status || n < 0 || max_iters < 1) {
        set_error("icg_geom_find_fundamental_mat_ransac: bad arguments");
        return ICG_EINVAL;
    }
    if (n < 15) {
        set_error("icg_geom_find_fundamental_mat_ransac: needs at least 15 point pairs (got %d)", n);
        return ICG_EUNSUPPORTED;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    // a batch of one set on the synchronous arena: [p1 | p2 | off[2] thr conf | n_inliers | F | mask]
    const size_t N = n, o_p2 = 8 * N, o_off = (o_p2 + 8 * N + 15) & ~(size_t) 15, o_thr = o_off + 16, o_conf = o_thr + 8, o_ni = o_conf + 8;
    const size_t o_F = o_ni + 8, o_mask = o_F + 72, total = o_mask + N;
    int rc = geom_reserve(h, total);
    if (rc != ICG_OK) return rc;
    memcpy(h->h_buf, pts1_xy, 8 * N), memcpy(h->h_buf + o_p2, pts2_xy, 8 * N);
    const int off[2] = {0, n};
    memcpy(h->h_buf + o_off, off, sizeof(off)), memcpy(h->h_buf + o_thr, &threshold, 8), memcpy(h->h_buf + o_conf, &confidence, 8);
    ICG_CUDA(cudaMemcpyAsync(h->d_buf, h->h_buf, o_ni, cudaMemcpyHostToDevice, h->stream));
    RansacBatch B;
    B.off = (const int *) (h->d_buf + o_off), B.n = nullptr;
    B.p1 = (const float *) h->d_buf, B.p2 = (const float *) (h->d_buf + o_p2);
    B.thr = (const double *) (h->d_buf + o_thr), B.conf = (const double *) (h->d_buf + o_conf);
    B.max_iters = max_iters;
    B.mask = h->d_buf + o_mask, B.n_inliers = (int *) (h->d_buf + o_ni), B.F = (double *) (h->d_buf + o_F), B.stats = nullptr;
    rc = ransac_batch_launch(h->stream, 1, B);
    if (rc != ICG_OK) return rc;
    ICG_CUDA(cudaMemcpyAsync(h->h_buf + o_F, h->d_buf + o_F, total - o_F, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    memcpy(status, h->h_buf + o_mask, N);
    if (F9) memcpy(F9, h->h_buf + o_F, 72);
    return ICG_OK;
}

int icg_geom_find_fundamental_mat_ransac_batch(icg_geom *h, int n_sets, const int32_t *set_off, const float *dev_pts1_xy, const float *dev_pts2_xy,
                                               const double *threshold, const double *confidence, int max_iters, uint8_t *dev_mask,
                                               int32_t *dev_n_inliers, double *dev_F9, long long *dev_stats) {
    if (!h || n_sets < 0 || (n_sets > 0 && (!set_off || !dev_mask || !dev_n_inliers)) || max_iters < 1) {
        set_error("icg_geom_find_fundamental_mat_ransac_batch: bad arguments");
        return ICG_EINVAL;
    }
    if (n_sets == 0) return ICG_OK;
    for (int s = 0; s < n_sets; s++)
        if (set_off[s] < 0 || set_off[s + 1] < set_off[s]) {
            set_error("icg_geom_find_fundamental_mat_ransac_batch: set_off is not monotone at set %d", s);
            return ICG_EINVAL;
        }
    if (set_off[n_sets] > 0 && (!dev_pts1_xy || !dev_pts2_xy)) {
        set_error("icg_geom_find_fundamental_mat_ransac_batch: NULL point arrays");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    // [off (n_sets + 1) | thr (n_sets) | conf (n_sets)] through the batch's own pinned / device buffers, fenced by stage_ev (the call is asynchronous)
    const size_t S = n_sets, o_thr = (4 * (S + 1) + 7) & ~(size_t) 7, o_conf = o_thr + 8 * S, total = o_conf + 8 * S;
    if (h->stage_pending) ICG_CUDA(cudaEventSynchronize(h->stage_ev));
    h->stage_pending = false;
    if (h->b_bytes < total) {
        ICG_CUDA(cudaStreamSynchronize(h->stream));
        if (h->d_b) cudaFree(h->d_b);
        if (h->h_b) cudaFreeHost(h->h_b);
        h->d_b = h->h_b = nullptr, h->b_bytes = 0;
        if (cudaMalloc(&h->d_b, total) != cudaSuccess || cudaMallocHost(&h->h_b, total) != cudaSuccess) {
            set_error("icg_geom_find_fundamental_mat_ransac_batch: staging allocation of %zu bytes failed", total);
            return ICG_ENOMEM;
        }
        h->b_bytes = total;
    }
    if (!h->stage_ev) ICG_CUDA(cudaEventCreateWithFlags(&h->stage_ev, cudaEventDisableTiming));
    memcpy(h->h_b, set_off, 4 * (S + 1));
    for (size_t s = 0; s < S; s++) {
        ((double *) (h->h_b + o_thr))[s] = threshold ? threshold[s] : 3.0;
        ((double *) (h->h_b + o_conf))[s] = confidence ? confidence[s] : 0.99;
    }
    ICG_CUDA(cudaMemcpyAsync(h->d_b, h->h_b, total, cudaMemcpyHostToDevice, h->stream));
    ICG_CUDA(cudaEventRecord(h->stage_ev, h->stream));
    h->stage_pending = true;
    RansacBatch B;
    B.off = (const int *) h->d_b, B.n = nullptr, B.p1 = dev_pts1_xy, B.p2 = dev_pts2_xy;
    B.thr = (const double *) (h->d_b + o_thr), B.conf = (const double *) (h->d_b + o_conf), B.max_iters = max_iters;
    B.mask = dev_mask, B.n_inliers = dev_n_inliers, B.F = dev_F9, B.stats = dev_stats;
    return ransac_batch_launch(h->stream, n_sets, B);
}

int icg_geom_triangulate_points(icg_geom *h, const double *Tcw0, const double *Tcw1, const double *pc0_xy, const double *pc1_xy, int n, double *pw_xyz) {
    if (!h || n < 0 || ((!Tcw0 || !Tcw1 || !pc0_xy || !pc1_xy || !pw_xyz) && n > 0)) {
        set_error("icg_geom_triangulate_points: bad arguments");
        return ICG_EINVAL;
    }
    if (n == 0) return ICG_OK;
    ICG_CUDA(cudaSetDevice(h->device));
    const size_t N = n, o_T0 = 0, o_T1 = o_T0 + 96 * N, o_c0 = o_T1 + 96, o_c1 = o_c0 + 16 * N, o_pw = o_c1 + 16 * N, total = o_pw + 24 * N;
    int rc = geom_reserve(h, total);
    if (rc != ICG_OK) return rc;
    memcpy(h->h_buf + o_T0, Tcw0, 96 * N), memcpy(h->h_buf + o_T1, Tcw1, 96), memcpy(h->h_buf + o_c0, pc0_xy, 16 * N), memcpy(h->h_buf + o_c1, pc1_xy, 16 * N);
    ICG_CUDA(cudaMemcpyAsync(h->d_buf, h->h_buf, o_pw, cudaMemcpyHostToDevice, h->stream));
    geom_triangulate_kernel<<<(n + 63) / 64, 64, 0, h->stream>>>((const double *) (h->d_buf + o_T0), (const double *) (h->d_buf + o_T1),
                                                                (const double *) (h->d_buf + o_c0), (const double *) (h->d_buf + o_c1), n,
                                                                (double *) (h->d_buf + o_pw));
    ICG_CHECK_LAUNCH();
    count_launch();
    ICG_CUDA(cudaMemcpyAsync(h->h_buf + o_pw, h->d_buf + o_pw, 24 * N, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    memcpy(pw_xyz, h->h_buf + o_pw, 24 * N);
    return ICG_OK;
}

int icg_geom_imu_preintegrate_batch(icg_geom *h, int n_intervals, const double *state16, const double *iewn3, const double *gravity3, const double *noise5,
                                    const double *imu, const int32_t *imu_off, double *blobs_out, double *end_states10) {
    if (!h || n_intervals < 1 || !state16 || !gravity3 || !noise5 || !imu || !imu_off || !blobs_out) {
        set_error("icg_geom_imu_preintegrate_batch: bad arguments");
        return ICG_EINVAL;
    }
    for (int k = 0; k < n_intervals; k++)
        if (imu_off[k + 1] - imu_off[k] < 1 || imu_off[k] < 0) {
            set_error("icg_geom_imu_preintegrate_batch: interval %d has no samples", k);
            return ICG_EINVAL;
        }
    ICG_CUDA(cudaSetDevice(h->device));
    const size_t NI = n_intervals, ns = imu_off[n_intervals];
    const size_t o_st = 0, o_iw = o_st + 128 * NI, o_g = o_iw + 24, o_nz = o_g + 24, o_imu = o_nz + 40, o_off = o_imu + 56 * ns;
    const size_t o_blob = (o_off + 4 * (NI + 1) + 15) & ~(size_t) 15, o_end = o_blob + sizeof(double) * ICG_IMU_BLOB_DOUBLES * NI, total = o_end + 80 * NI;
    int rc = geom_reserve(h, total);
    if (rc != ICG_OK) return rc;
    memcpy(h->h_buf + o_st, state16, 128 * NI);
    if (iewn3) memcpy(h->h_buf + o_iw, iewn3, 24);
    memcpy(h->h_buf + o_g, gravity3, 24), memcpy(h->h_buf + o_nz, noise5, 40), memcpy(h->h_buf + o_imu, imu, 56 * ns), memcpy(h->h_buf + o_off, imu_off, 4 * (NI + 1));
    ICG_CUDA(cudaMemcpyAsync(h->d_buf, h->h_buf, o_blob, cudaMemcpyHostToDevice, h->stream));
    PreintBatch a;
    a.n = n_intervals, a.state16 = (const double *) (h->d_buf + o_st), a.iewn3 = iewn3 ? (const double *) (h->d_buf + o_iw) : nullptr;
    a.gravity3 = (const double *) (h->d_buf + o_g), a.noise5 = (const double *) (h->d_buf + o_nz), a.imu = (const double *) (h->d_buf + o_imu);
    a.off = (const int *) (h->d_buf + o_off), a.blobs = (double *) (h->d_buf + o_blob), a.ends = (double *) (h->d_buf + o_end);
    ICG_CUDA(preint_batch_launch(a, h->stream));
    count_launch();
    ICG_CUDA(cudaMemcpyAsync(h->h_buf + o_blob, h->d_buf + o_blob, total - o_blob, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    memcpy(blobs_out, h->h_buf + o_blob, sizeof(double) * ICG_IMU_BLOB_DOUBLES * NI);
    if (end_states10) memcpy(end_states10, h->h_buf + o_end, 80 * NI);
    return ICG_OK;
}

}  // extern "C"
