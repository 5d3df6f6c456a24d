// fundamental.cu -- SURVEY.md 8f rank 3: the fundamental-matrix outlier gate of the front end and two-view triangulation, HOST entry points
// (the serial reference loop: the iteration bound shrinks as better models are found, the subsets come from one cv::RNG stream).  The
// arithmetic lives in geom_core.cuh; geom.cu runs the same cores on the device (rounds of subsets solved and scored in parallel, the serial
// acceptance rule replayed on each round's counts).
//
// Replaces cv::findFundamentalMat(pts_new_undis, pts_cur_undis, cv::FM_RANSAC, reprojection_error_std_, 0.99, status)
// (IG/tracking/tracking.cc:547; only `status` is consumed, :549-553).  OpenCV is an un-vendored dependency of the reference; its
// algorithm (calib3d fundam.cpp / ptsetreg.cpp) is restated here and pinned against cv2 4.13.0 by tests/golden/fundamental_golden.npz:
// identical inlier masks.
#include <float.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "geom_core.cuh"

using namespace icg;

namespace {
using gc::CvRng;
using gc::run_7point;
using gc::update_num_iters;
// FMEstimatorCallback::computeError + findInliers (ptsetreg.cpp) over all pairs
int find_inliers(const float *m1, const float *m2, int count, const double *F, double thresh, uint8_t *mask) {
    int good = 0;
    for (int i = 0; i < count; i++) good += mask[i] = gc::is_inlier(m1, m2, i, F, thresh) ? 1 : 0;
    return good;
}
}  // namespace

extern "C" {

int icg_find_fundamental_mat_ransac(const float *pts1_xy, const float *pts2_xy, int n, double threshold, double confidence, int max_iters,
                                    uint8_t *status, double *F9) {
    if (!pts1_xy || !pts2_xy || !status || n < 0 || max_iters < 1) {
        set_error("icg_find_fundamental_mat_ransac: bad arguments");
        return ICG_EINVAL;
    }
    if (n < 15) {  // cv::findFundamentalMat switches to other estimators below 15 points; the reference only calls it with >= 15 (tracking.cc:546)
        set_error("icg_find_fundamental_mat_ransac: needs at least 15 point pairs (got %d)", n);
        return ICG_EUNSUPPORTED;
    }
    if (threshold <= 0) threshold = 3;
    if (confidence < DBL_EPSILON || confidence > 1 - DBL_EPSILON) confidence = 0.99;
    CvRng rng;
    std::vector<uint8_t> mask(n), best(n, 0);
    double bestF[9] = {0};
    int niters = max_iters, max_good = 0;
    float ms1[14], ms2[14];
    for (int iter = 0; iter < niters; iter++) {
        // RANSACPointSetRegistrator::getSubset: 7 distinct indices, the subset redrawn while either image has collinear points
        int idx[7];
        const bool found = gc::draw_subset(rng, pts1_xy, pts2_xy, n, idx);
        for (int i = 0; i < 7 && found; i++) {
            ms1[2 * i] = pts1_xy[2 * idx[i]], ms1[2 * i + 1] = pts1_xy[2 * idx[i] + 1];
            ms2[2 * i] = pts2_xy[2 * idx[i]], ms2[2 * i + 1] = pts2_xy[2 * idx[i] + 1];
        }
        if (!found) {
            if (iter == 0) {
                memset(status, 0, n);
                if (F9) memset(F9, 0, sizeof(double) * 9);
                return ICG_OK;
            }
            break;
        }
        double F[3][9];
        const int nmodels = run_7point(ms1, ms2, F);
        if (nmodels <= 0) continue;
        for (int k = 0; k < nmodels; k++) {
            const int good = find_inliers(pts1_xy, pts2_xy, n, F[k], threshold, mask.data());
            if (good > std::max(max_good, 6)) {
                std::swap(mask, best);
                memcpy(bestF, F[k], sizeof(bestF));
                max_good = good;
                niters = update_num_iters(confidence, (double) (n - good) / n, 7, niters);
            }
        }
    }
    memcpy(status, best.data(), n);
    if (F9) memcpy(F9, bestF, sizeof(bestF));
    return ICG_OK;
}

// Tracking::triangulatePoint (IG/tracking/tracking.cc:796-808) for n point pairs: rows of the 4 x 4 design matrix
//   pc0.x * P0.row(2) - P0.row(0),  pc0.y * P0.row(2) - P0.row(1),  pc1.x * P1.row(2) - P1.row(0),  pc1.y * P1.row(2) - P1.row(1)
// (P = T_c_w, 3 x 4 row-major), pw = right singular vector of the smallest singular value, dehomogenised (scale / sign invariant, so any
// accurate SVD gives the reference's Eigen::JacobiSVD result up to rounding).  Host function: <= 300 pairs, the caller interleaves it
// with map bookkeeping (:715-789).
int icg_triangulate_points(const double *Tcw0 /* n x 12 */, const double *Tcw1 /* 12 */, const double *pc0_xy, const double *pc1_xy, int n,
                           double *pw_xyz) {
    if ((!Tcw0 || !Tcw1 || !pc0_xy || !pc1_xy || !pw_xyz) && n > 0) {
        set_error("icg_triangulate_points: bad arguments");
        return ICG_EINVAL;
    }
    for (int i = 0; i < n; i++) gc::triangulate_point(Tcw0 + 12 * (size_t) i, Tcw1, pc0_xy + 2 * (size_t) i, pc1_xy + 2 * (size_t) i, pw_xyz + 3 * (size_t) i);
    return ICG_OK;
}

}  // extern "C"
