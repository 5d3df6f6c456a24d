// geom_core.cuh -- __host__ __device__ cores of the point-wise front-end geometry and of the IMU propagation, shared by the host entry
// points (camera.cu, fundamental.cu, ba.cu: icg_camera_*, icg_find_fundamental_mat_ransac, icg_triangulate_points, icg_imu_preintegrate)
// and by their batched device versions (geom.cu).  One definition of the arithmetic -> host and device results agree to the last ulp of
// the libm calls.  References as in the callers (IG/ = ic_gvins/ic_gvins/).
#pragma once
#include <float.h>
#include <math.h>
#include <stdint.h>

#include "../../include/icgvins_b200.h"
#include "ba_math.cuh"

namespace icg {
namespace gc {

#define GC_HD __host__ __device__ inline

// ------------------------------------------------------------------------------------------------ camera model (IG/tracking/camera.cc)
GC_HD void pixel2cam(const icg_camera &c, double u, double v, double &x, double &y) {  // camera.cc:126-130
    y = (v - c.cy) / c.fy;
    x = (u - c.cx - c.skew * y) / c.fx;
}
GC_HD void cam2pixel(const icg_camera &c, double x, double y, double z, float &u, float &v) {  // camera.cc:132-134
    u = (float) ((c.fx * x + c.skew * y) / z + c.cx);
    v = (float) (c.fy * y / z + c.cy);
}
GC_HD void distort_xy(const icg_camera &c, double x, double y, double &xd, double &yd) {  // camera.cc:79-86
    const double r2 = x * x + y * y;
    const double rr = (1 + c.k1 * r2 + c.k2 * r2 * r2 + c.k3 * r2 * r2 * r2);
    xd = x * rr + 2 * c.p1 * x * y + c.p2 * (r2 + 2 * x * x);
    yd = y * rr + c.p1 * (r2 + 2 * y * y) + 2 * c.p2 * x * y;
}
// cv::undistortPoints(pts, pts, K, D, Mat(), K) on one point (calib3d: five fixed-point iterations, skew ignored when normalising, P = K)
GC_HD void undistort_point(const icg_camera &c, float *p) {
    const double ifx = 1.0 / c.fx, ify = 1.0 / c.fy;
    double x = ((double) p[0] - c.cx) * ifx, y = ((double) p[1] - c.cy) * ify;
    const double x0 = x, y0 = y;
    for (int j = 0; j < 5; j++) {
        const double r2 = x * x + y * y;
        const double icdist = 1.0 / (1 + ((c.k3 * r2 + c.k2) * r2 + c.k1) * r2);
        if (icdist < 0) {
            x = x0, y = y0;
            break;
        }
        const double dx = 2 * c.p1 * x * y + c.p2 * (r2 + 2 * x * x), dy = c.p1 * (r2 + 2 * y * y) + 2 * c.p2 * x * y;
        x = (x0 - dx) * icdist;
        y = (y0 - dy) * icdist;
    }
    p[0] = (float) (c.fx * x + c.skew * y + c.cx);
    p[1] = (float) (c.fy * y + c.cy);
}
GC_HD void distort_point(const icg_camera &c, float *p) {  // Camera::distortPoint (camera.cc:88-104)
    double x, y, xd, yd;
    pixel2cam(c, p[0], p[1], x, y);
    distort_xy(c, x, y, xd, yd);
    cam2pixel(c, xd, yd, 1.0, p[0], p[1]);
}
// Camera::distortCameraPoint (camera.cc:104-117): normalise by z, radtan, the distorted coordinates pass through float (:112-113), cam2pixel
GC_HD void distort_camera_point(const icg_camera &c, double X, double Y, double Z, float &u, float &v) {
    const double x = X / Z, y = Y / Z;
    double xd, yd;
    distort_xy(c, x, y, xd, yd);
    cam2pixel(c, (double) (float) xd, (double) (float) yd, 1.0, u, v);
}
// Camera::world2cam (camera.cc:145-147): R^T (pw - t), R9 row-major; the products as fixed-order sums (no FMA: the callers build with -fmad=false)
GC_HD void world2cam(const double *R9, const double *t3, const double *pw, double &x, double &y, double &z) {
    const double d0 = pw[0] - t3[0], d1 = pw[1] - t3[1], d2 = pw[2] - t3[2];
    x = R9[0] * d0 + R9[3] * d1 + R9[6] * d2;
    y = R9[1] * d0 + R9[4] * d1 + R9[7] * d2;
    z = R9[2] * d0 + R9[5] * d1 + R9[8] * d2;
}
// Camera::world2pixel (camera.cc:141-143) = cam2pixel(world2cam(pw, pose))
GC_HD void world2pixel(const icg_camera &c, const double *R9, const double *t3, const double *pw, float &u, float &v) {
    double x, y, z;
    world2cam(R9, t3, pw, x, y, z);
    cam2pixel(c, x, y, z, u, v);
}
// M = A^T B for row-major 3 x 3 A, B (R_cur^T R_pre of tracking.cc:465, pose1.R^T pose0.R of :867): M(i,j) = sum_k A(k,i) B(k,j), k ascending
GC_HD void rt_mul(const double *A, const double *B, double *M) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) M[3 * i + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
}
// M v for row-major 3 x 3 M, fixed-order sums
GC_HD void mat_vec(const double *M, double x, double y, double z, double &ox, double &oy, double &oz) {
    ox = M[0] * x + M[1] * y + M[2] * z;
    oy = M[3] * x + M[4] * y + M[5] * z;
    oz = M[6] * x + M[7] * y + M[8] * z;
}
// Tracking::keyPointParallax (tracking.cc:861-871) with Rc1c0 = pose1.R^T pose0.R precomputed (rt_mul):
//   |(Rc1c0 pixel2cam(pp0)).xy - pixel2cam(pp1).xy| * focalLength(),  focalLength() = (fx + fy) * 0.5 (camera.h:82-84)
GC_HD double key_point_parallax(const icg_camera &c, const double *Rc1c0, float u0, float v0, float u1, float v1) {
    double x0, y0, x1, y1, px, py, pz;
    pixel2cam(c, u0, v0, x0, y0);
    pixel2cam(c, u1, v1, x1, y1);
    mat_vec(Rc1c0, x0, y0, 1.0, px, py, pz);
    const double dx = px - x1, dy = py - y1;
    return sqrt(dx * dx + dy * dy) * ((c.fx + c.fy) * 0.5);
}

// ------------------------------------------------------------------------------------------------ cv::findFundamentalMat(FM_RANSAC)
struct CvRng {  // cv::RNG: multiply-with-carry, CV_RNG_COEFF = 4164903690
    uint64_t state;
    GC_HD explicit CvRng(uint64_t s = 0xffffffffffffffffull) : state(s ? s : 0xffffffffffffffffull) {}
    GC_HD unsigned next() {
        state = (uint64_t) (unsigned) state * 4164903690u + (unsigned) (state >> 32);
        return (unsigned) state;
    }
    GC_HD int uniform(int a, int b) { return a == b ? a : (int) (next() % (unsigned) (b - a) + a); }
};
// haveCollinearPoints (fundam.cpp): the LAST of `count` points against every pair of earlier ones
GC_HD bool collinear_last(const float *p, int count) {
    const int i = count - 1;
    for (int j = 0; j < i; j++) {
        const double dx1 = p[2 * j] - p[2 * i], dy1 = p[2 * j + 1] - p[2 * i + 1];
        for (int k = 0; k < j; k++) {
            const double dx2 = p[2 * k] - p[2 * i], dy2 = p[2 * k + 1] - p[2 * i + 1];
            if (fabs(dx2 * dy1 - dy2 * dx1) <= FLT_EPSILON * (fabs(dx1) + fabs(dy1) + fabs(dx2) + fabs(dy2))) return true;
        }
    }
    return false;
}
// RANSACPointSetRegistrator::getSubset: 7 distinct indices, redrawn while either image has collinear points (<= 10000 attempts)
GC_HD bool draw_subset(CvRng &rng, const float *p1, const float *p2, int n, int *idx) {
    float ms1[14], ms2[14];
    for (int attempts = 0; attempts < 10000; attempts++) {
        for (int i = 0; i < 7; i++) {
            int v;
            bool dup;
            do {
                v = rng.uniform(0, n);
                dup = false;
                for (int j = 0; j < i; j++) dup = dup || idx[j] == v;
            } while (dup);
            idx[i] = v;
            ms1[2 * i] = p1[2 * v], ms1[2 * i + 1] = p1[2 * v + 1], ms2[2 * i] = p2[2 * v], ms2[2 * i + 1] = p2[2 * v + 1];
        }
        if (collinear_last(ms1, 7) || collinear_last(ms2, 7)) continue;
        return true;
    }
    return false;
}
// cv::solveCubic: c[0] x^3 + c[1] x^2 + c[2] x + c[3] = 0, real roots in OpenCV's order
GC_HD int solve_cubic(const double c[4], double r[3]) {
    const double PI = 3.14159265358979323846;
    double a0 = c[0], a1 = c[1], a2 = c[2], a3 = c[3];
    if (a0 == 0) {
        if (a1 == 0) {
            if (a2 == 0) return a3 == 0 ? -1 : 0;
            r[0] = -a3 / a2;
            return 1;
        }
        double d = a2 * a2 - 4 * a1 * a3;
        if (d >= 0) {
            d = sqrt(d);
            const double q1 = (-a2 + d) * 0.5, q2 = (a2 + d) * -0.5;
            if (fabs(q1) > fabs(q2)) {
                r[0] = q1 / a1;
                r[1] = a3 / q1;
            } else {
                r[0] = q2 / a1;
                r[1] = a3 / q2;
            }
            return d > 0 ? 2 : 1;
        }
        return 0;
    }
    a0 = 1. / a0;
    a1 *= a0, a2 *= a0, a3 *= a0;
    const double Q = (a1 * a1 - 3 * a2) * (1. / 9), R = (2 * a1 * a1 * a1 - 9 * a1 * a2 + 27 * a3) * (1. / 54), Qcubed = Q * Q * Q;
    double d = Qcubed - R * R;
    if (d > 0) {
        const double theta = acos(R / sqrt(Qcubed)), sqrtQ = sqrt(Q), t0 = -2 * sqrtQ, t1 = theta * (1. / 3), t2 = a1 * (1. / 3);
        r[0] = t0 * cos(t1) - t2;
        r[1] = t0 * cos(t1 + (2. * PI / 3)) - t2;
        r[2] = t0 * cos(t1 + (4. * PI / 3)) - t2;
        return 3;
    }
    if (d == 0) {
        if (R >= 0) {
            r[0] = -2 * pow(R, 1. / 3) - a1 / 3;
            r[1] = pow(R, 1. / 3) - a1 / 3;
        } else {
            r[0] = 2 * pow(-R, 1. / 3) - a1 / 3;
            r[1] = -pow(-R, 1. / 3) - a1 / 3;
        }
        return 2;
    }
    d = sqrt(-d);
    double e = pow(d + fabs(R), 1. / 3);
    if (R > 0) e = -e;
    r[0] = (e + Q / e) - a1 * (1. / 3);
    return 1;
}
// right null space of the 7 x 9 system: one-sided (Hestenes) Jacobi on the columns of A; the two columns of V whose A-images have the
// smallest norms span it.  f1 = v7, f2 = v8 in the descending-singular-value order of cv::SVDecomp.
GC_HD void null_space_7x9(const double a[7 * 9], double f1[9], double f2[9]) {
    double G[9][7], V[9][9];
    for (int c = 0; c < 9; c++) {
        for (int r = 0; r < 7; r++) G[c][r] = a[r * 9 + c];
        for (int r = 0; r < 9; r++) V[c][r] = r == c ? 1.0 : 0.0;
    }
    for (int sweep = 0; sweep < 60; sweep++) {
        bool rotated = false;
        for (int p = 0; p < 8; p++)
            for (int q = p + 1; q < 9; q++) {
                double al = 0, be = 0, ga = 0;
                for (int r = 0; r < 7; r++) al += G[p][r] * G[p][r], be += G[q][r] * G[q][r], ga += G[p][r] * G[q][r];
                if (ga == 0.0 || fabs(ga) <= 1e-16 * sqrt(al * be)) continue;
                rotated = true;
                const double zeta = (be - al) / (2.0 * ga);
                const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
                for (int r = 0; r < 7; r++) {
                    const double x = G[p][r], y = G[q][r];
                    G[p][r] = cs * x - sn * y, G[q][r] = sn * x + cs * y;
                }
                for (int r = 0; r < 9; r++) {
                    const double x = V[p][r], y = V[q][r];
                    V[p][r] = cs * x - sn * y, V[q][r] = sn * x + cs * y;
                }
            }
        if (!rotated) break;
    }
    int order[9];
    double nrm[9];
    for (int c = 0; c < 9; c++) {
        order[c] = c, nrm[c] = 0;
        for (int r = 0; r < 7; r++) nrm[c] += G[c][r] * G[c][r];
    }
    for (int i = 1; i < 9; i++) {  // stable insertion sort, descending norm (== std::stable_sort with nrm[x] > nrm[y])
        const int oi = order[i];
        int j = i - 1;
        while (j >= 0 && nrm[order[j]] < nrm[oi]) order[j + 1] = order[j], j--;
        order[j + 1] = oi;
    }
    for (int r = 0; r < 9; r++) f1[r] = V[order[7]][r], f2[r] = V[order[8]][r];
}
// run7Point (fundam.cpp): up to three fundamental matrices through seven correspondences
GC_HD int run_7point(const float *m1, const float *m2, double F[3][9]) {
    double a[7 * 9], f1[9], f2[9], c[4], r[3] = {0, 0, 0};
    for (int i = 0; i < 7; i++) {
        const double x0 = m1[2 * i], y0 = m1[2 * i + 1], x1 = m2[2 * i], y1 = m2[2 * i + 1];
        double *row = a + i * 9;
        row[0] = x1 * x0, row[1] = x1 * y0, row[2] = x1, row[3] = y1 * x0, row[4] = y1 * y0, row[5] = y1, row[6] = x0, row[7] = y0, row[8] = 1;
    }
    null_space_7x9(a, f1, f2);
    for (int i = 0; i < 9; i++) f1[i] -= f2[i];
    double t0 = f2[4] * f2[8] - f2[5] * f2[7], t1 = f2[3] * f2[8] - f2[5] * f2[6], t2 = f2[3] * f2[7] - f2[4] * f2[6];
    c[3] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2;
    c[2] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2 - f1[3] * (f2[1] * f2[8] - f2[2] * f2[7]) + f1[4] * (f2[0] * f2[8] - f2[2] * f2[6]) -
           f1[5] * (f2[0] * f2[7] - f2[1] * f2[6]) + f1[6] * (f2[1] * f2[5] - f2[2] * f2[4]) - f1[7] * (f2[0] * f2[5] - f2[2] * f2[3]) +
           f1[8] * (f2[0] * f2[4] - f2[1] * f2[3]);
    t0 = f1[4] * f1[8] - f1[5] * f1[7], t1 = f1[3] * f1[8] - f1[5] * f1[6], t2 = f1[3] * f1[7] - f1[4] * f1[6];
    c[0] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2;
    c[1] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2 - f2[3] * (f1[1] * f1[8] - f1[2] * f1[7]) + f2[4] * (f1[0] * f1[8] - f1[2] * f1[6]) -
           f2[5] * (f1[0] * f1[7] - f1[1] * f1[6]) + f2[6] * (f1[1] * f1[5] - f1[2] * f1[4]) - f2[7] * (f1[0] * f1[5] - f1[2] * f1[3]) +
           f2[8] * (f1[0] * f1[4] - f1[1] * f1[3]);
    const int n = solve_cubic(c, r);
    if (n < 1 || n > 3) return n;
    for (int k = 0; k < n; k++) {
        double lambda = r[k], mu = 1.;
        const double s = f1[8] * r[k] + f2[8];
        if (fabs(s) > DBL_EPSILON) {  // normalise so that F(3,3) == 1
            mu = 1. / s;
            lambda *= mu;
            F[k][8] = 1.;
        } else {
            F[k][8] = 0.;
        }
        for (int i = 0; i < 8; i++) F[k][i] = f1[i] * lambda + f2[i] * mu;
    }
    return n;
}
// FMEstimatorCallback::computeError + findInliers (ptsetreg.cpp) for pair i: err = max(d1^2 s1, d2^2 s2) rounded to float <= thresh^2
GC_HD bool is_inlier(const float *m1, const float *m2, int i, const double *F, double thresh) {
    const float t = (float) (thresh * thresh);
    const double x1 = m1[2 * i], y1 = m1[2 * i + 1], x2 = m2[2 * i], y2 = m2[2 * i + 1];
    double a = F[0] * x1 + F[1] * y1 + F[2], b = F[3] * x1 + F[4] * y1 + F[5], c = F[6] * x1 + F[7] * y1 + F[8];
    const double s2 = 1. / (a * a + b * b), d2 = x2 * a + y2 * b + c;
    a = F[0] * x2 + F[3] * y2 + F[6], b = F[1] * x2 + F[4] * y2 + F[7], c = F[2] * x2 + F[5] * y2 + F[8];
    const double s1 = 1. / (a * a + b * b), d1 = x1 * a + y1 * b + c;
    const double e1 = d1 * d1 * s1, e2 = d2 * d2 * s2;
    const float err = (float) (e1 > e2 ? e1 : e2);  // std::max(a, b): b unless a > b... max(a, b) = (a < b) ? b : a
    return err <= t;
}
GC_HD int update_num_iters(double p, double ep, int model_points, int max_iters) {  // RANSACUpdateNumIters (ptsetreg.cpp)
    p = p < 0. ? 0. : p > 1. ? 1. : p, ep = ep < 0. ? 0. : ep > 1. ? 1. : ep;
    double num = 1. - p > DBL_MIN ? 1. - p : DBL_MIN, denom = 1. - pow(1. - ep, model_points);
    if (denom < DBL_MIN) return 0;
    num = log(num), denom = log(denom);
    return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : (int) lrint(num / denom);
}

// ------------------------------------------------------------------------------------------------ Tracking::triangulatePoint (tracking.cc:796-808)
// rows of the 4 x 4 design matrix: pc0.x P0.row(2) - P0.row(0), pc0.y P0.row(2) - P0.row(1), pc1.x P1.row(2) - P1.row(0), pc1.y P1.row(2) - P1.row(1)
// (P = T_c_w, 3 x 4 row-major); pw = right singular vector of the smallest singular value (one-sided Jacobi), dehomogenised
GC_HD void triangulate_point(const double *P0, const double *P1, const double *pc0, const double *pc1, double *pw) {
    double G[4][4], V[4][4];
    for (int c = 0; c < 4; c++) {
        G[c][0] = pc0[0] * P0[8 + c] - P0[c];
        G[c][1] = pc0[1] * P0[8 + c] - P0[4 + c];
        G[c][2] = pc1[0] * P1[8 + c] - P1[c];
        G[c][3] = pc1[1] * P1[8 + c] - P1[4 + c];
        for (int r = 0; r < 4; r++) V[c][r] = r == c ? 1.0 : 0.0;
    }
    for (int sweep = 0; sweep < 60; sweep++) {
        bool rotated = false;
        for (int p = 0; p < 3; p++)
            for (int q = p + 1; q < 4; q++) {
                double al = 0, be = 0, ga = 0;
                for (int r = 0; r < 4; r++) al += G[p][r] * G[p][r], be += G[q][r] * G[q][r], ga += G[p][r] * G[q][r];
                if (ga == 0.0 || fabs(ga) <= 1e-16 * sqrt(al * be)) continue;
                rotated = true;
                const double zeta = (be - al) / (2.0 * ga);
                const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
                for (int r = 0; r < 4; r++) {
                    const double x = G[p][r], y = G[q][r];
                    G[p][r] = cs * x - sn * y, G[q][r] = sn * x + cs * y;
                    const double vx = V[p][r], vy = V[q][r];
                    V[p][r] = cs * vx - sn * vy, V[q][r] = sn * vx + cs * vy;
                }
            }
        if (!rotated) break;
    }
    int best = 0;
    double bn = 1e300;
    for (int c = 0; c < 4; c++) {
        double nn = 0;
        for (int r = 0; r < 4; r++) nn += G[c][r] * G[c][r];
        if (nn < bn) bn = nn, best = c;
    }
    for (int k = 0; k < 3; k++) pw[k] = V[best][k] / V[best][3];
}
// Tracking::pose2Tcw (tracking.cc:851-859), top 3 rows: T = [R^T | -R^T t], 3 x 4 row-major; -R^T t as the fixed-order sum of world2cam
GC_HD void pose_tcw(const double *R9, const double *t3, double *T12) {
    for (int i = 0; i < 3; i++) {
        T12[4 * i] = R9[i], T12[4 * i + 1] = R9[3 + i], T12[4 * i + 2] = R9[6 + i];
        T12[4 * i + 3] = -(R9[i] * t3[0] + R9[3 + i] * t3[1] + R9[6 + i] * t3[2]);
    }
}
// Tracking::isGoodToTrack(pp, pose, pw, 1.0, 3.0) (tracking.cc:813-829): isGoodDepth(z, 3) = 1 < z < 200 * 3 (:247-249, mappoint.h:52-53),
// then |reprojectionError(pose, pw, pp)| <= std (camera.cc:153-157: world2pixel returns a cv::Point2f, so each difference is float - float)
GC_HD bool good_to_track(const icg_camera &c, float u, float v, const double *R9, const double *t3, const double *pw, double std) {
    double x, y, z;
    world2cam(R9, t3, pw, x, y, z);
    if (!(z > 1.0 && z < 200.0 * 3.0)) return false;
    float pu, pv;
    cam2pixel(c, x, y, z, pu, pv);
    const float ex = pu - u, ey = pv - v;
    const double dx = ex, dy = ey;
    return !(sqrt(dx * dx + dy * dy) > std * 1.0);
}
// Tracking::isGoodToTrack(pp, pose, pw, scale, depth_scale): 1 < z < 200 * depth_scale, then |reprojectionError| <= std * scale.  err receives
// the error when the depth passes (gvinsOutlierCulling sums it, IG/ic_gvins.cc:1066-1081).  Every test keeps the reference's sense: a NaN
// depth fails.
GC_HD bool good_to_track_scaled(const icg_camera &c, float u, float v, const double *R9, const double *t3, const double *pw, double std, double scale,
                                double depth_scale, double &err) {
    double x, y, z;
    world2cam(R9, t3, pw, x, y, z);
    if (!(z > 1.0 && z < 200.0 * depth_scale)) return false;
    float pu, pv;
    cam2pixel(c, x, y, z, pu, pv);
    const float ex = pu - u, ey = pv - v;
    const double dx = ex, dy = ey;
    err = sqrt(dx * dx + dy * dy);
    return !(err > std * scale);
}

// ------------------------------------------------------------------------------------------------ IMU preintegration propagation
// PreintegrationEarth::resetState / integrationProcess / updateJacobianAndCovariance (IG/preintegration/preintegration_earth.cc:205-338) or, with
// iewn3 == NULL, PreintegrationNormal (PreintegrationBase::integration, preintegration_base.cc:39-70 + preintegration_normal.cc:195-232).
// state16 = p[3] q_xyzw[4] v[3] bg[3] ba[3]; noise5 = gyr_arw, acc_vrw, gyr_bias_std, acc_bias_std, corr_time; imu = n rows (dt, dtheta[3], dvel[3]).
// The scalar recurrence is split into preint_begin / preint_sample / preint_head so that the warp-per-interval kernel (preint.cu) runs the
// same code on every lane; preintegrate_core below is the sequential whole.
struct PreintScalar {  // the mechanised state, the preintegrated deltas and the interval constants
    bam::V3 cur_p, cur_v, bg, ba, iewn, grav, dp, dv, s1;
    bam::Q cur_q, q0, dq;
    double delta_time, s0;
    bool normal;
};
GC_HD void preint_begin(PreintScalar &S, const double *state16, const double *iewn3, const double *gravity3) {
    using namespace bam;
    S.normal = iewn3 == nullptr;
    S.cur_p = mk(state16[0], state16[1], state16[2]), S.cur_v = mk(state16[7], state16[8], state16[9]);
    S.cur_q = mkq(state16[6], state16[3], state16[4], state16[5]);
    S.q0 = S.cur_q;
    S.bg = mk(state16[10], state16[11], state16[12]), S.ba = mk(state16[13], state16[14], state16[15]);
    S.iewn = S.normal ? mk(0, 0, 0) : mk(iewn3[0], iewn3[1], iewn3[2]), S.grav = mk(gravity3[0], gravity3[1], gravity3[2]);
    S.dp = mk(0, 0, 0), S.dv = mk(0, 0, 0);
    S.dq = mkq(1, 0, 0, 0);
    S.delta_time = 0, S.s0 = 0;
    S.s1 = mk(0, 0, 0);
}
// setNoiseMatrix (preintegration_earth.cc:326-334): the diagonal of noise_
GC_HD void preint_noise(const double *noise5, double *noise) {
    const double corr = noise5[4];
    for (int k = 0; k < 3; k++) {
        noise[k] = noise5[0] * noise5[0], noise[3 + k] = noise5[1] * noise5[1];
        noise[6 + k] = 2 * noise5[2] * noise5[2] / corr, noise[9 + k] = 2 * noise5[3] * noise5[3] / corr;
    }
}
// ---- insMechanization (IG/misc.cc:151-206), the state part that integrationProcess shares with it, in two pieces so that a warp can form
// the state-independent part of many samples at once (ins.cu) and one lane run the dependent chain.  iswithscale is false in the reference
// (IG/ic_gvins.cc:100), so the scale factors have no code path.
// Bias compensation and the two-sample corrections (misc.cc:154-176 = compensationBias, preintegration_base.cc:84-90, + integrationProcess).
// Rows pr = imu_pre, cu = imu_cur as (dt, dtheta[3], dvel[3]).
GC_HD void ins_increments(const double *pr, const double *cu, bam::V3 bg, bam::V3 ba, bam::V3 &cth, bam::V3 &cvl, bam::V3 &dvfb, bam::V3 &dtheta) {
    using namespace bam;
    const double dt = cu[0];
    V3 pth = mk(pr[1], pr[2], pr[3]) - pr[0] * bg, pvl = mk(pr[4], pr[5], pr[6]) - pr[0] * ba;
    cth = mk(cu[1], cu[2], cu[3]) - dt * bg, cvl = mk(cu[4], cu[5], cu[6]) - dt * ba;
    dvfb = cvl + 0.5 * cross(cth, cvl) + (1.0 / 12.0) * (cross(pth, cvl) + cross(pvl, cth));
    dtheta = cth + (1.0 / 12.0) * cross(pth, cth);
}
// The state update (misc.cc:178-205): qth = rotvec2q(dtheta); qnn = rotvec2q(-(dt iewn)), read in the Earth form (earth) only.
GC_HD void ins_mechanize_step(bam::V3 &p, bam::Q &q, bam::V3 &v, bam::V3 dvfb, bam::Q qth, bam::Q qnn, double dt, bam::V3 grav, bam::V3 iewn,
                              bool earth) {
    using namespace bam;
    if (earth) {
        V3 dv_cor_g = dt * (grav - 2.0 * cross(iewn, v));
        V3 dvel = mul(scale(0.5, add(ident(), qmat(qnn))), mul(qmat(q), dvfb)) + dv_cor_g;
        p = p + dt * v + (0.5 * dt) * dvel;
        v = v + dvel;
        q = qnormalized(qmul(qmul(qnn, q), qth));
    } else {
        V3 dvel = mul(qmat(q), dvfb) + dt * grav;
        p = p + dt * v + (0.5 * dt) * dvel;
        v = v + dvel;
        q = qnormalized(qmul(q, qth));
    }
}

// one sample (rows pr = imu_pre, cu = imu_cur): integrationProcess up to the covariance update; returns what phi and gt are built from
GC_HD void preint_sample(PreintScalar &S, const double *pr, const double *cu, double &dt_out, bam::V3 &cth_out, bam::V3 &cvl_out, bam::M3 &cbb0) {
    using namespace bam;
    const double dt = cu[0];
    const V3 iewn = S.iewn;
    V3 cth, cvl, dvfb, dtheta;
    ins_increments(pr, cu, S.bg, S.ba, cth, cvl, dvfb, dtheta);
    S.delta_time += dt;
    const Q qth = rotvec2q(dtheta);
    if (!S.normal) {
        Q qnn = rotvec2q(-(dt * iewn));
        ins_mechanize_step(S.cur_p, S.cur_q, S.cur_v, dvfb, qth, qnn, dt, S.grav, iewn, true);
        S.s0 += dt;
        S.s1 = S.s1 + dt * S.cur_p;
        V3 dnn = -((S.delta_time - 0.5 * dt) * iewn);
        V3 dvel = mul(qmat(qmul(qmul(qmul(qinv(S.q0), rotvec2q(dnn)), S.q0), S.dq)), dvfb);
        S.dp = S.dp + dt * S.dv + (0.5 * dt) * dvel;
        S.dv = S.dv + dvel;
        S.dq = qnormalized(qmul(S.dq, qth));
        cbb0 = neg(qmat(qmul(qmul(qmul(qinv(S.q0), rotvec2q(-(S.delta_time * iewn))), S.q0), S.dq)));
    } else {
        ins_mechanize_step(S.cur_p, S.cur_q, S.cur_v, dvfb, qth, qth, dt, S.grav, iewn, false);
        V3 dvel = mul(qmat(S.dq), dvfb);
        S.dp = S.dp + dt * S.dv + (0.5 * dt) * dvel;
        S.dv = S.dv + dvel;
        S.dq = qnormalized(qmul(S.dq, qth));
        // phi(3,6) = -R(dq) [dvel]x, phi(3,12) = -R(dq) dt; gt(3,3) = R(dq), gt(6,0) = +I (preintegration_normal.cc:207-225): with a diagonal
        // noise matrix G = gt noise gt^T does not see the sign of a column block of gt, so the Earth form below with cbb0 = -R(dq) is the same
        cbb0 = neg(qmat(S.dq));
    }
    dt_out = dt, cth_out = cth, cvl_out = cvl;
}
// the blob's scalar part ([0..26], [477..479]) and the end state; jacobian_ / covariance_ ([27..476]) are the caller's
GC_HD void preint_head(const PreintScalar &S, const double *state16, const double *gravity3, double *blob, double *end_state10) {
    blob[0] = S.delta_time;
    blob[1] = S.dp.x, blob[2] = S.dp.y, blob[3] = S.dp.z, blob[4] = S.dv.x, blob[5] = S.dv.y, blob[6] = S.dv.z;
    blob[7] = S.dq.x, blob[8] = S.dq.y, blob[9] = S.dq.z, blob[10] = S.dq.w;
    for (int k = 0; k < 3; k++) blob[11 + k] = state16[10 + k], blob[14 + k] = state16[13 + k], blob[17 + k] = gravity3[k];
    blob[20] = S.iewn.x, blob[21] = S.iewn.y, blob[22] = S.iewn.z;
    blob[23] = S.s0, blob[24] = S.s1.x, blob[25] = S.s1.y, blob[26] = S.s1.z;
    blob[477] = S.normal ? 1.0 : 0.0, blob[478] = 0, blob[479] = 0;
    if (end_state10) {
        end_state10[0] = S.cur_p.x, end_state10[1] = S.cur_p.y, end_state10[2] = S.cur_p.z;
        end_state10[3] = S.cur_q.x, end_state10[4] = S.cur_q.y, end_state10[5] = S.cur_q.z, end_state10[6] = S.cur_q.w;
        end_state10[7] = S.cur_v.x, end_state10[8] = S.cur_v.y, end_state10[9] = S.cur_v.z;
    }
}
GC_HD void preintegrate_core(const double *state16, const double *iewn3, const double *gravity3, const double *noise5, const double *imu, int n, double *blob,
                             double *end_state10) {
    using namespace bam;
    PreintScalar S;
    preint_begin(S, state16, iewn3, gravity3);
    const double corr = noise5[4];
    double noise[12];
    preint_noise(noise5, noise);
    double jac[225], cov[225];
    for (int i = 0; i < 225; i++) jac[i] = 0, cov[i] = 0;
    for (int i = 0; i < 15; i++) jac[i * 15 + i] = 1;
    for (int s = 1; s < n; s++) {
        double dt;
        V3 cth, cvl;
        M3 cbb0;
        preint_sample(S, imu + 7 * (size_t) (s - 1), imu + 7 * (size_t) s, dt, cth, cvl, cbb0);
        // updateJacobianAndCovariance: phi = I + F dt; the non-trivial blocks are applied directly (phi is sparse)
        double phi[225], gt[180];
        for (int i = 0; i < 225; i++) phi[i] = 0;
        for (int i = 0; i < 180; i++) gt[i] = 0;
        auto put = [](double *M, int nc, int r0, int c0, const M3 &m) {
            for (int i = 0; i < 3; i++)
                for (int j = 0; j < 3; j++) M[(r0 + i) * nc + c0 + j] = m.m[3 * i + j];
        };
        put(phi, 15, 0, 0, ident());
        put(phi, 15, 0, 3, scale(dt, ident()));
        put(phi, 15, 3, 3, ident());
        put(phi, 15, 3, 6, mul(cbb0, skew(cvl)));
        put(phi, 15, 3, 12, scale(dt, cbb0));
        put(phi, 15, 6, 6, sub(ident(), skew(cth)));
        put(phi, 15, 6, 9, scale(-dt, ident()));
        put(phi, 15, 9, 9, scale(1 - dt / corr, ident()));
        put(phi, 15, 12, 12, scale(1 - dt / corr, ident()));
        double tmp[225];
        for (int i = 0; i < 15; i++)
            for (int j = 0; j < 15; j++) {
                double a = 0;
                for (int k = 0; k < 15; k++) a += phi[i * 15 + k] * jac[k * 15 + j];
                tmp[i * 15 + j] = a;
            }
        for (int i = 0; i < 225; i++) jac[i] = tmp[i];
        put(gt, 12, 3, 3, cbb0);
        put(gt, 12, 6, 0, neg(ident()));
        put(gt, 12, 9, 6, ident());
        put(gt, 12, 12, 9, ident());
        double G[225], pg[225], pc[225];
        for (int i = 0; i < 15; i++)
            for (int j = 0; j < 15; j++) {
                double a = 0;
                for (int k = 0; k < 12; k++) a += gt[i * 12 + k] * noise[k] * gt[j * 12 + k];
                G[i * 15 + j] = a;
            }
        for (int i = 0; i < 15; i++)
            for (int j = 0; j < 15; j++) {
                double a = 0, c = 0;
                for (int k = 0; k < 15; k++) a += phi[i * 15 + k] * G[k * 15 + j], c += phi[i * 15 + k] * cov[k * 15 + j];
                pg[i * 15 + j] = a, pc[i * 15 + j] = c;
            }
        for (int i = 0; i < 15; i++)
            for (int j = 0; j < 15; j++) {
                double a = 0, gpt = 0;
                for (int k = 0; k < 15; k++) a += pc[i * 15 + k] * phi[j * 15 + k], gpt += G[i * 15 + k] * phi[j * 15 + k];
                tmp[i * 15 + j] = a + 0.5 * dt * (pg[i * 15 + j] + gpt);
            }
        for (int i = 0; i < 225; i++) cov[i] = tmp[i];
    }
    preint_head(S, state16, gravity3, blob, end_state10);
    for (int i = 0; i < 225; i++) blob[27 + i] = jac[i], blob[252 + i] = cov[i];
}

// ------------------------------------------------------------------------------------------------ Earth::iewn(origin, local) (IG/common/earth.h:120-237)
// iewn at local2global(origin, local): ecef1 = blh2ecef(origin) + cne(origin) local, then ecef2blh's fixed-point loop on the latitude
// (do ... while (|h - h2| > 1e-4)) and iewn(lat) = (wie cos lat, 0, -wie sin lat).  The WGS84 constants are the reference's.
GC_HD bam::V3 earth_iewn(const double *origin_blh, bam::V3 local) {
    const double WIE = 7.2921151467E-5, RA = 6378137.0000000000, E1 = 0.0066943799901413156;
    const double lat0 = origin_blh[0], lon0 = origin_blh[1], h0 = origin_blh[2];
    const double sinlat = sin(lat0), sinlon = sin(lon0), coslat = cos(lat0), coslon = cos(lon0);
    const double rn0 = RA / sqrt(1.0 - E1 * sinlat * sinlat), rnh = rn0 + h0;  // RN(lat), blh2ecef
    const double e0x = rnh * coslat * coslon, e0y = rnh * coslat * sinlon, e0z = (rnh - rn0 * E1) * sinlat;
    const double c00 = -sinlat * coslon, c01 = -sinlon, c02 = -coslat * coslon;  // cne(origin), row-major
    const double c10 = -sinlat * sinlon, c11 = coslon, c12 = -coslat * sinlon;
    const double c20 = coslat, c21 = 0, c22 = -sinlat;
    const double x = e0x + (c00 * local.x + c01 * local.y + c02 * local.z);
    const double y = e0y + (c10 * local.x + c11 * local.y + c12 * local.z);
    const double z = e0z + (c20 * local.x + c21 * local.y + c22 * local.z);
    const double p = sqrt(x * x + y * y);
    double lat = atan(z / (p * (1.0 - E1))), h = 0, h2;
    do {
        h2 = h;
        const double sl = sin(lat), rn = RA / sqrt(1.0 - E1 * sl * sl);
        h = p / cos(lat) - rn;
        lat = atan(z / (p * (1.0 - E1 * rn / (rn + h))));
    } while (fabs(h - h2) > 1.0e-4);
    return bam::mk(WIE * cos(lat), 0, -WIE * sin(lat));
}

// ------------------------------------------------------------------------------------------------ IMU factor square-root information
// U = LLT(cov^-1).matrixL().transpose() (IG/preintegration/preintegration_earth.cc:39-40): Gauss-Jordan inverse with partial pivoting,
// symmetrised, Cholesky.  One definition for the upload (host) and the reintegration kernel (device, -fmad=false): the host build has no
// FMA contraction either, so both give the same U for the same covariance.  work: 675 doubles (copy of cov | inverse | L).  Returns false
// (U untouched) when the covariance is singular or its inverse not positive definite.
GC_HD bool imu_sqrt_info(const double *cov, double *U, double *work) {
    const int n = 15;
    double *a = work, *Ai = work + 225, *Lm = work + 450;
    for (int i = 0; i < n * n; i++) a[i] = cov[i], Ai[i] = 0;
    for (int i = 0; i < n; i++) Ai[i * n + i] = 1;
    for (int c = 0; c < n; c++) {
        int p = c;
        for (int r = c + 1; r < n; r++)
            if (fabs(a[r * n + c]) > fabs(a[p * n + c])) p = r;
        if (a[p * n + c] == 0) return false;
        if (p != c)
            for (int k = 0; k < n; k++) {
                double t = a[c * n + k];
                a[c * n + k] = a[p * n + k], a[p * n + k] = t;
                t = Ai[c * n + k], Ai[c * n + k] = Ai[p * n + k], Ai[p * n + k] = t;
            }
        const double d = a[c * n + c];
        for (int k = 0; k < n; k++) a[c * n + k] /= d, Ai[c * n + k] /= d;
        for (int r = 0; r < n; r++) {
            if (r == c) continue;
            const double f = a[r * n + c];
            if (f == 0) continue;
            for (int k = 0; k < n; k++) a[r * n + k] -= f * a[c * n + k], Ai[r * n + k] -= f * Ai[c * n + k];
        }
    }
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) Lm[i * n + j] = 0.5 * (Ai[i * n + j] + Ai[j * n + i]);
    for (int j = 0; j < n; j++) {
        double d = Lm[j * n + j];
        for (int k = 0; k < j; k++) d -= Lm[j * n + k] * Lm[j * n + k];
        if (!(d > 0)) return false;
        d = sqrt(d);
        Lm[j * n + j] = d;
        for (int i = j + 1; i < n; i++) {
            double s = Lm[i * n + j];
            for (int k = 0; k < j; k++) s -= Lm[i * n + k] * Lm[j * n + k];
            Lm[i * n + j] = s / d;
        }
    }
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) U[i * n + j] = j >= i ? Lm[j * n + i] : 0.0;
    return true;
}

}  // namespace gc

// ------------------------------------------------------------------------------------------------ batched device RANSAC (geom.cu)
constexpr int RS_CTA = 64;      // subsets solved and scored per CTA and round == threads per CTA
constexpr int RS_CLUSTER = 8;  // CTAs per set when the batch is small (64, then 8 x 64 subsets per round: 1 000 iterations in 3 rounds)
struct RansacBatch {          // all DEVICE pointers; set s = pairs off[s] .. off[s] + n[s] (n == NULL: off[s + 1] - off[s])
    const int *off, *n;
    const float *p1, *p2;
    const double *thr, *conf;  // per set; NULL = 3 / 0.99
    int max_iters;
    uint8_t *mask;             // per pair, at the pair's index
    int *n_inliers;            // per set
    double *F;                 // 9 per set, may be NULL
    long long *stats;          // 3 per set (subsets drawn, clock64 cycles of the draw, of the whole CTA), may be NULL
};
int ransac_batch_launch(cudaStream_t st, int n_sets, const RansacBatch &B);

}  // namespace icg
