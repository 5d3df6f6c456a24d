// camera.cu -- SURVEY.md 8a row A6: the radtan camera model of the front end, HOST entry points (<= 300 points per frame, FP64, called from the
// tracking thread between the GPU stages; SURVEY: "small; stays host").  The arithmetic lives in geom_core.cuh (__host__ __device__), which
// geom.cu also runs as batched kernels; compiled into the same library so that the Tracking shims find every call behind one C ABI.
//
// Replaces Camera::undistortPoints / distortPoints / distortPoint / distortCameraPoint / pixel2cam / cam2pixel / world2pixel
// (IG/tracking/camera.cc:72-146).  undistortPoints forwards to cv::undistortPoints(pts, pts, K, D, Mat(), K) in the reference
// (:72-74); OpenCV is un-vendored, its algorithm (calib3d/undistort: five fixed-point iterations, skew ignored when normalising, P = K
// applied with its skew) is restated here and pinned against cv2 4.13.0 by tests/golden/camera_golden.npz -- float outputs bit-identical.
#include <math.h>

#include "common.cuh"
#include "geom_core.cuh"

using namespace icg;

namespace {
using gc::pixel2cam;
inline bool bad(const icg_camera *c, const void *p, int n, const char *who) {
    if (!c || (!p && n > 0) || n < 0 || !(c->fx != 0.0) || !(c->fy != 0.0)) {
        set_error("%s: bad arguments", who);
        return true;
    }
    return false;
}
}  // namespace

extern "C" {

int icg_camera_undistort_points(const icg_camera *c, float *pts_xy, int n) {
    if (bad(c, pts_xy, n, "icg_camera_undistort_points")) return ICG_EINVAL;
    for (int i = 0; i < n; i++) gc::undistort_point(*c, pts_xy + 2 * (size_t) i);  // one definition for host and device (geom_core.cuh)
    return ICG_OK;
}

int icg_camera_distort_points(const icg_camera *c, float *pts_xy, int n) {
    if (bad(c, pts_xy, n, "icg_camera_distort_points")) return ICG_EINVAL;
    for (int i = 0; i < n; i++) gc::distort_point(*c, pts_xy + 2 * (size_t) i);
    return ICG_OK;
}

int icg_camera_distort_camera_points(const icg_camera *c, const double *pc_xyz, float *px_xy, int n) {
    if (bad(c, pc_xyz, n, "icg_camera_distort_camera_points") || !px_xy) return ICG_EINVAL;
    for (int i = 0; i < n; i++) gc::distort_camera_point(*c, pc_xyz[3 * i], pc_xyz[3 * i + 1], pc_xyz[3 * i + 2], px_xy[2 * i], px_xy[2 * i + 1]);
    return ICG_OK;
}

int icg_camera_pixel2cam(const icg_camera *c, const float *px_xy, double *cam_xyz, int n) {
    if (bad(c, px_xy, n, "icg_camera_pixel2cam") || !cam_xyz) return ICG_EINVAL;
    for (int i = 0; i < n; i++) {
        pixel2cam(*c, px_xy[2 * i], px_xy[2 * i + 1], cam_xyz[3 * i], cam_xyz[3 * i + 1]);
        cam_xyz[3 * i + 2] = 1.0;
    }
    return ICG_OK;
}

int icg_camera_world2pixel(const icg_camera *c, const double *R9, const double *t3, const double *pw_xyz, float *px_xy, int n) {
    if (bad(c, pw_xyz, n, "icg_camera_world2pixel") || !R9 || !t3 || !px_xy) return ICG_EINVAL;
    for (int i = 0; i < n; i++) gc::world2pixel(*c, R9, t3, pw_xyz + 3 * (size_t) i, px_xy[2 * i], px_xy[2 * i + 1]);
    return ICG_OK;
}

// Tracking::calculateHistigram (IG/tracking/tracking.cc:88-104): cv::calcHist (256 uniform bins, float counts) then
// sum_k hist[k] * (float) k / 256.0 in double, divided by cols * rows -- the brightness gate of Tracking::preprocessing (:115-133).
int icg_tracking_histogram(const uint8_t *img, int width, int height, int stride, double *out) {
    if (!img || !out || width < 1 || height < 1 || stride < width) {
        set_error("icg_tracking_histogram: bad arguments");
        return ICG_EINVAL;
    }
    unsigned cnt[256] = {0};
    for (int y = 0; y < height; y++) {
        const uint8_t *r = img + (size_t) y * stride;
        for (int x = 0; x < width; x++) cnt[r[x]]++;
    }
    double hist = 0;
    for (int k = 0; k < 256; k++) {
        const float prod = (float) cnt[k] * (float) k;  // float x float, as histogram.at<float>(k) * (float) k
        hist += (double) prod / 256.0;
    }
    *out = hist / (double) (width * height);  // hist /= (image.cols * image.rows): int product
    return ICG_OK;
}

}  // extern "C"
