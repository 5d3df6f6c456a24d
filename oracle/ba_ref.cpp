// oracle/ba_ref.cpp -- see ba_ref.hpp.  TEST INFRASTRUCTURE ONLY (tests/, __graft_entry__.smoke(), bench cpu_baseline).
#include "ba_ref.hpp"

#include <algorithm>
#include <cfloat>
#include <cstdio>
#include <limits>
#include <thread>

namespace icgo {

// ===================================================================================== PoseParameterization::Plus
void pose_plus(const double *x, const double *delta, double *out) {
    // pose_parameterization.h:34-49: p = _p + dp; q = (_q * dq).normalized(), dq = rotvec2quaternion(delta+3)
    Q q  = {x[6], x[3], x[4], x[5]};
    Q dq = rotvec2quaternion({delta[3], delta[4], delta[5]});
    Q r  = q_normalized(q * dq);
    out[0] = x[0] + delta[0];
    out[1] = x[1] + delta[1];
    out[2] = x[2] + delta[2];
    out[3] = r.x;
    out[4] = r.y;
    out[5] = r.z;
    out[6] = r.w;
}

static inline void set_block(double *J, int ncols, int r0, int c0, const M3 &m) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) J[(r0 + i) * ncols + c0 + j] = m(i, j);
}

// ===================================================================================== ReprojectionFactor
bool ReprojectionFactor::Evaluate(double const *const *parameters, double *residuals, double **jacobians) const {
    // reprojection_factor.h:55-147
    V3 p0 = pose_p(parameters[0]);
    Q q0  = pose_q(parameters[0]);
    V3 p1 = pose_p(parameters[1]);
    Q q1  = pose_q(parameters[1]);
    V3 tic = pose_p(parameters[2]);
    Q qic  = pose_q(parameters[2]);
    double id0 = parameters[3][0];
    double td  = parameters[4][0];

    V3 pts_0_td = pts0 - (td - td0) * vel0;
    V3 pts_1_td = pts1 - (td - td1) * vel1;

    V3 pts_c_0 = pts_0_td / id0;
    V3 pts_b_0 = q_rotate(qic, pts_c_0) + tic;
    V3 pts_n   = q_rotate(q0, pts_b_0) + p0;
    V3 pts_b_1 = q_rotate(q_inverse(q1), pts_n - p1);
    V3 pts_1   = q_rotate(q_inverse(qic), pts_b_1 - tic);

    double d1  = pts_1.z;
    double si  = 1.0 / std_;
    residuals[0] = si * (pts_1.x / d1 - pts_1_td.x);
    residuals[1] = si * (pts_1.y / d1 - pts_1_td.y);

    if (jacobians) {
        M3 cb0n = q_matrix(q0);
        M3 cnb1 = transpose(q_matrix(q1));
        M3 cbc  = transpose(q_matrix(qic));
        // reduce (2x3) = sqrt_info * [1/d1 0 -x/d1^2; 0 1/d1 -y/d1^2]
        double red[6] = {si * (1.0 / d1), 0, si * (-pts_1.x / (d1 * d1)), 0, si * (1.0 / d1), si * (-pts_1.y / (d1 * d1))};
        auto reduce_mul = [&](const M3 &a, double *out, int ncols, int c0) {
            for (int r = 0; r < 2; r++)
                for (int c = 0; c < 3; c++) out[r * ncols + c0 + c] = red[3 * r] * a(0, c) + red[3 * r + 1] * a(1, c) + red[3 * r + 2] * a(2, c);
        };
        auto reduce_vec = [&](V3 v, double *o0, double *o1) {
            *o0 = red[0] * v.x + red[1] * v.y + red[2] * v.z;
            *o1 = red[3] * v.x + red[4] * v.y + red[5] * v.z;
        };
        if (jacobians[0]) {
            double *J = jacobians[0];
            M3 a = cbc * cnb1;
            M3 b = -(cbc * cnb1 * cb0n * skew(pts_b_0));
            reduce_mul(a, J, 7, 0);
            reduce_mul(b, J, 7, 3);
            J[6] = J[13] = 0;
        }
        if (jacobians[1]) {
            double *J = jacobians[1];
            M3 a = -(cbc * cnb1);
            M3 b = cbc * skew(pts_b_1);
            reduce_mul(a, J, 7, 0);
            reduce_mul(b, J, 7, 3);
            J[6] = J[13] = 0;
        }
        if (jacobians[2]) {
            double *J = jacobians[2];
            M3 a     = cbc * (cnb1 * cb0n - m3_identity());
            M3 tmp_r = cbc * cnb1 * cb0n * transpose(cbc);
            M3 b     = -(tmp_r * skew(pts_c_0)) + skew(tmp_r * pts_c_0) + skew(cbc * (cnb1 * (cb0n * tic + p0 - p1) - tic));
            reduce_mul(a, J, 7, 0);
            reduce_mul(b, J, 7, 3);
            J[6] = J[13] = 0;
        }
        if (jacobians[3]) {
            M3 t = cbc * cnb1 * cb0n * transpose(cbc);
            V3 v = (t * pts_0_td) / (id0 * id0);
            double a, b;
            reduce_vec(v, &a, &b);
            jacobians[3][0] = -a;
            jacobians[3][1] = -b;
        }
        if (jacobians[4]) {
            M3 t = cbc * cnb1 * cb0n * transpose(cbc);
            V3 v = (t * vel0) / id0;
            double a, b;
            reduce_vec(v, &a, &b);
            jacobians[4][0] = -a + si * vel1.x;
            jacobians[4][1] = -b + si * vel1.y;
        }
    }
    return true;
}

// ===================================================================================== GnssFactor
bool GnssFactor::Evaluate(double const *const *parameters, double *residuals, double **jacobians) const {
    // gnss_factor.h:43-71
    V3 p = pose_p(parameters[0]);
    Q q  = pose_q(parameters[0]);
    M3 R = q_matrix(q);
    V3 e = p + R * lever - blh;
    double si[3] = {1.0 / std_.x, 1.0 / std_.y, 1.0 / std_.z};
    residuals[0] = si[0] * e.x;
    residuals[1] = si[1] * e.y;
    residuals[2] = si[2] * e.z;
    if (jacobians && jacobians[0]) {
        double *J = jacobians[0];
        std::memset(J, 0, sizeof(double) * 21);
        M3 b = -(R * skew(lever));
        for (int r = 0; r < 3; r++) {
            J[r * 7 + r] = si[r];
            for (int c = 0; c < 3; c++) J[r * 7 + 3 + c] = si[r] * b(r, c);
        }
    }
    return true;
}

// ===================================================================================== small dense helpers
// inverse by Gauss-Jordan with partial pivoting (Eigen's MatrixXd::inverse() is PartialPivLU based)
static bool invert(const double *A, double *Ainv, int n) {
    std::vector<double> a(A, A + n * n);
    for (int i = 0; i < n * n; i++) Ainv[i] = 0;
    for (int i = 0; i < n; i++) Ainv[i * n + i] = 1;
    for (int c = 0; c < n; c++) {
        int piv = c;
        double best = std::fabs(a[c * n + c]);
        for (int r = c + 1; r < n; r++)
            if (std::fabs(a[r * n + c]) > best) best = std::fabs(a[r * n + c]), piv = r;
        if (best == 0) return false;
        if (piv != c)
            for (int k = 0; k < n; k++) std::swap(a[c * n + k], a[piv * n + k]), std::swap(Ainv[c * n + k], Ainv[piv * n + k]);
        double d = a[c * n + c];
        for (int k = 0; k < n; k++) a[c * n + k] /= d, Ainv[c * n + k] /= d;
        for (int r = 0; r < n; r++) {
            if (r == c) continue;
            double f = a[r * n + c];
            if (f == 0) continue;
            for (int k = 0; k < n; k++) a[r * n + k] -= f * a[c * n + k], Ainv[r * n + k] -= f * Ainv[c * n + k];
        }
    }
    return true;
}
// lower Cholesky A = L L^T in place on the lower triangle; returns false if not positive definite
static bool cholesky_lower(double *A, int n) {
    for (int j = 0; j < n; j++) {
        double d = A[j * n + j];
        for (int k = 0; k < j; k++) d -= A[j * n + k] * A[j * n + k];
        if (!(d > 0)) return false;
        d = std::sqrt(d);
        A[j * n + j] = d;
        for (int i = j + 1; i < n; i++) {
            double s = A[i * n + j];
            for (int k = 0; k < j; k++) s -= A[i * n + k] * A[j * n + k];
            A[i * n + j] = s / d;
        }
    }
    return true;
}
// sqrt_information_ = LLT(covariance_.inverse()).matrixL().transpose()  (preintegration_earth.cc:39-40): upper U
void imu_sqrt_information(const double *cov, double *U /*15x15 row-major*/) {
    double inv[225], L[225];
    invert(cov, inv, 15);
    for (int i = 0; i < 15; i++)
        for (int j = 0; j < 15; j++) L[i * 15 + j] = 0.5 * (inv[i * 15 + j] + inv[j * 15 + i]);  // LLT reads one triangle
    cholesky_lower(L, 15);
    for (int i = 0; i < 15; i++)
        for (int j = 0; j < 15; j++) U[i * 15 + j] = (j >= i) ? L[j * 15 + i] : 0.0;
}

// ===================================================================================== PreintegrationFactor
// PreintegrationNormal::evaluate + residualJacobianPose0/Pose1/Mix0/Mix1 (preintegration/preintegration_normal.cc:38-142): no Earth
// rotation terms, and the attitude residual is 2 (corrected_q^-1 q0^-1 q1).vec() (the inverse ordering of the Earth form)
static bool evaluate_normal(const Preintegration &P, double const *const *parameters, double *residuals, double **jacobians) {
    V3 p0 = pose_p(parameters[0]);
    Q q0  = pose_q(parameters[0]);
    V3 v0{parameters[1][0], parameters[1][1], parameters[1][2]}, bg0{parameters[1][3], parameters[1][4], parameters[1][5]},
        ba0{parameters[1][6], parameters[1][7], parameters[1][8]};
    V3 p1 = pose_p(parameters[2]);
    Q q1  = pose_q(parameters[2]);
    V3 v1{parameters[3][0], parameters[3][1], parameters[3][2]}, bg1{parameters[3][3], parameters[3][4], parameters[3][5]},
        ba1{parameters[3][6], parameters[3][7], parameters[3][8]};
    double U[225];
    imu_sqrt_information(P.covariance, U);
    auto blk = [&](int r, int c) {
        M3 m;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) m(i, j) = P.jacobian[(r + i) * 15 + c + j];
        return m;
    };
    M3 dp_dbg = blk(0, 9), dp_dba = blk(0, 12), dv_dbg = blk(3, 9), dv_dba = blk(3, 12), dq_dbg = blk(6, 9);
    V3 dbg = bg0 - P.bg, dba = ba0 - P.ba;
    const double dt = P.delta_time;
    V3 corrected_p = P.dp + dp_dba * dba + dp_dbg * dbg;
    V3 corrected_v = P.dv + dv_dba * dba + dv_dbg * dbg;
    Q corrected_q  = P.dq * rotvec2quaternion(dq_dbg * dbg);
    Q q0i = q_inverse(q0);
    M3 c0 = q_matrix(q0i);
    V3 dpn = p1 - p0 - v0 * dt - 0.5 * P.gravity * dt * dt;
    V3 dvn = v1 - v0 - P.gravity * dt;
    double r[15];
    V3 rp = q_rotate(q0i, dpn) - corrected_p, rv = q_rotate(q0i, dvn) - corrected_v;
    V3 rq = 2.0 * vec(q_inverse(corrected_q) * q0i * q1), rbg = bg1 - bg0, rba = ba1 - ba0;
    r[0] = rp.x, r[1] = rp.y, r[2] = rp.z, r[3] = rv.x, r[4] = rv.y, r[5] = rv.z, r[6] = rq.x, r[7] = rq.y, r[8] = rq.z;
    r[9] = rbg.x, r[10] = rbg.y, r[11] = rbg.z, r[12] = rba.x, r[13] = rba.y, r[14] = rba.z;
    for (int i = 0; i < 15; i++) {
        double s = 0;
        for (int k = 0; k < 15; k++) s += U[i * 15 + k] * r[k];
        residuals[i] = s;
    }
    if (!jacobians) return true;
    auto whiten = [&](const double *Jraw, int ncols, double *out) {
        for (int i = 0; i < 15; i++)
            for (int c = 0; c < ncols; c++) {
                double s = 0;
                for (int k = 0; k < 15; k++) s += U[i * 15 + k] * Jraw[k * ncols + c];
                out[i * ncols + c] = s;
            }
    };
    // bottom-right 3x3 of quaternionleft(a) * quaternionright(b) (rotation.h:103-119): -a_v b_v^T + L_br(a) R_br(b)
    auto lr_br = [&](Q a, Q b) {
        V3 av = vec(a), bv = vec(b);
        M3 lr = qleft_br(a) * qright_br(b), m;
        const double x[3] = {av.x, av.y, av.z}, y[3] = {bv.x, bv.y, bv.z};
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) m(i, j) = -x[i] * y[j] + lr(i, j);
        return m;
    };
    if (jacobians[0]) {  // residualJacobianPose0 (:77-97)
        double J[15 * 7] = {0};
        set_block(J, 7, 0, 0, -c0);
        set_block(J, 7, 0, 3, skew(q_rotate(q0i, dpn)));
        set_block(J, 7, 3, 3, skew(q_rotate(q0i, dvn)));
        set_block(J, 7, 6, 3, -lr_br(q_inverse(q1) * q0, corrected_q));
        whiten(J, 7, jacobians[0]);
    }
    if (jacobians[1]) {  // residualJacobianMix0 (:113-140)
        double J[15 * 9] = {0};
        set_block(J, 9, 0, 0, -dt * c0);
        set_block(J, 9, 0, 3, -dp_dbg);
        set_block(J, 9, 0, 6, -dp_dba);
        set_block(J, 9, 3, 0, -c0);
        set_block(J, 9, 3, 3, -dv_dbg);
        set_block(J, 9, 3, 6, -dv_dba);
        set_block(J, 9, 6, 3, -(qleft_br(q_inverse(q1) * q0 * P.dq) * dq_dbg));
        set_block(J, 9, 9, 3, -m3_identity());
        set_block(J, 9, 12, 6, -m3_identity());
        whiten(J, 9, jacobians[1]);
    }
    if (jacobians[2]) {  // residualJacobianPose1 (:99-111)
        double J[15 * 7] = {0};
        set_block(J, 7, 0, 0, c0);
        set_block(J, 7, 6, 3, qleft_br(q_inverse(corrected_q) * q0i * q1));
        whiten(J, 7, jacobians[2]);
    }
    if (jacobians[3]) {  // residualJacobianMix1 (:142-153)
        double J[15 * 9] = {0};
        set_block(J, 9, 3, 0, c0);
        set_block(J, 9, 9, 3, m3_identity());
        set_block(J, 9, 12, 6, m3_identity());
        whiten(J, 9, jacobians[3]);
    }
    return true;
}

bool PreintegrationFactor::Evaluate(double const *const *parameters, double *residuals, double **jacobians) const {
    const Preintegration &P = *pre;
    // constructState (preintegration_earth.cc:186-203)
    V3 p0 = pose_p(parameters[0]);
    Q q0  = pose_q(parameters[0]);
    V3 v0{parameters[1][0], parameters[1][1], parameters[1][2]}, bg0{parameters[1][3], parameters[1][4], parameters[1][5]},
        ba0{parameters[1][6], parameters[1][7], parameters[1][8]};
    V3 p1 = pose_p(parameters[2]);
    Q q1  = pose_q(parameters[2]);
    V3 v1{parameters[3][0], parameters[3][1], parameters[3][2]}, bg1{parameters[3][3], parameters[3][4], parameters[3][5]},
        ba1{parameters[3][6], parameters[3][7], parameters[3][8]};

    if (P.normal) return evaluate_normal(P, parameters, residuals, jacobians);
    // evaluate (preintegration_earth.cc:37-90)
    double U[225];
    imu_sqrt_information(P.covariance, U);
    auto blk = [&](int r, int c) {
        M3 m;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) m(i, j) = P.jacobian[(r + i) * 15 + c + j];
        return m;
    };
    M3 dp_dbg = blk(0, 9), dp_dba = blk(0, 12), dv_dbg = blk(3, 9), dv_dba = blk(3, 12), dq_dbg = blk(6, 9);
    V3 dbg = bg0 - P.bg, dba = ba0 - P.ba;
    M3 iewn_skew = skew(P.iewn);
    V3 p_cor{0, 0, 0};
    for (size_t i = 0; i + 3 < P.pn.size(); i += 4) p_cor = p_cor + (V3{P.pn[i + 1], P.pn[i + 2], P.pn[i + 3]} - p0) * P.pn[i];
    p_cor    = 2.0 * (iewn_skew * p_cor);
    V3 v_cor = 2.0 * (iewn_skew * (p1 - p0));
    double dt = P.delta_time;
    V3 dnn   = -(P.iewn * dt);
    Q qnn    = rotvec2quaternion(dnn);
    V3 dpn   = p1 - p0 - v0 * dt - 0.5 * P.gravity * dt * dt + p_cor;
    V3 dvn   = v1 - v0 - P.gravity * dt + v_cor;
    V3 corrected_p = P.dp + dp_dba * dba + dp_dbg * dbg;
    V3 corrected_v = P.dv + dv_dba * dba + dv_dbg * dbg;
    Q corrected_q  = P.dq * rotvec2quaternion(dq_dbg * dbg);
    Q qnb0   = q_inverse(q0);
    M3 cnb0  = q_matrix(qnb0);
    Q qb0b1  = q_inverse(q1) * qnn * q0;

    double r[15];
    V3 rp = cnb0 * dpn - corrected_p, rv = cnb0 * dvn - corrected_v, rq = 2.0 * vec(qb0b1 * corrected_q), rbg = bg1 - bg0, rba = ba1 - ba0;
    r[0] = rp.x, r[1] = rp.y, r[2] = rp.z, r[3] = rv.x, r[4] = rv.y, r[5] = rv.z, r[6] = rq.x, r[7] = rq.y, r[8] = rq.z;
    r[9] = rbg.x, r[10] = rbg.y, r[11] = rbg.z, r[12] = rba.x, r[13] = rba.y, r[14] = rba.z;
    for (int i = 0; i < 15; i++) {
        double s = 0;
        for (int k = 0; k < 15; k++) s += U[i * 15 + k] * r[k];
        residuals[i] = s;
    }
    if (!jacobians) return true;
    auto whiten = [&](const double *Jraw, int ncols, double *out) {
        for (int i = 0; i < 15; i++)
            for (int c = 0; c < ncols; c++) {
                double s = 0;
                for (int k = 0; k < 15; k++) s += U[i * 15 + k] * Jraw[k * ncols + c];
                out[i * ncols + c] = s;
            }
    };
    if (jacobians[0]) {  // residualJacobianPose0 (:92-111)
        double J[15 * 7] = {0};
        set_block(J, 7, 0, 0, -cnb0 - 2.0 * (cnb0 * iewn_skew) * dt);
        set_block(J, 7, 0, 3, skew(cnb0 * dpn));
        set_block(J, 7, 3, 0, -2.0 * (cnb0 * iewn_skew));
        set_block(J, 7, 3, 3, skew(cnb0 * dvn));
        // (quaternionleft(qb0b1) * quaternionright(corrected_q)).bottomRightCorner<3,3>()
        {
            V3 a = vec(qb0b1), b = vec(corrected_q);
            M3 la = qleft_br(qb0b1), rb = qright_br(corrected_q), m;
            // full 4x4 product bottom-right = a * (-b^T) + la * rb   (row 1..3 of left: [a | la], col 1..3 of right: [-b^T ; rb])
            double av[3] = {a.x, a.y, a.z}, bv[3] = {b.x, b.y, b.z};
            M3 lr = la * rb;
            for (int i = 0; i < 3; i++)
                for (int j = 0; j < 3; j++) m(i, j) = -av[i] * bv[j] + lr(i, j);
            set_block(J, 7, 6, 3, m);
        }
        whiten(J, 7, jacobians[0]);
    }
    if (jacobians[1]) {  // residualJacobianMix0 (:127-154)
        double J[15 * 9] = {0};
        set_block(J, 9, 0, 0, -dt * cnb0);
        set_block(J, 9, 0, 3, -dp_dbg);
        set_block(J, 9, 0, 6, -dp_dba);
        set_block(J, 9, 3, 0, -cnb0);
        set_block(J, 9, 3, 3, -dv_dbg);
        set_block(J, 9, 3, 6, -dv_dba);
        set_block(J, 9, 6, 3, qleft_br(qb0b1 * P.dq) * dq_dbg);
        set_block(J, 9, 9, 3, -m3_identity());
        set_block(J, 9, 12, 6, -m3_identity());
        whiten(J, 9, jacobians[1]);
    }
    if (jacobians[2]) {  // residualJacobianPose1 (:113-125)
        double J[15 * 7] = {0};
        set_block(J, 7, 0, 0, cnb0);
        set_block(J, 7, 3, 0, 2.0 * (cnb0 * iewn_skew));
        set_block(J, 7, 6, 3, -qright_br(qb0b1 * corrected_q));
        whiten(J, 7, jacobians[2]);
    }
    if (jacobians[3]) {  // residualJacobianMix1 (:156-168)
        double J[15 * 9] = {0};
        set_block(J, 9, 3, 0, cnb0);
        set_block(J, 9, 9, 3, m3_identity());
        set_block(J, 9, 12, 6, m3_identity());
        whiten(J, 9, jacobians[3]);
    }
    return true;
}

// ===================================================================================== small IMU factors
bool ImuErrorFactor::Evaluate(double const *const *parameters, double *residuals, double **jacobians) const {
    // imu_error_factor.h:45-91
    const double GB = 7200 / 3600.0 * M_PI / 180.0, AB = 2.0e4 * 1.0e-5;
    for (int k = 0; k < 3; k++) {
        residuals[k]     = parameters[0][k + 3] / GB;
        residuals[k + 3] = parameters[0][k + 6] / AB;
    }
    if (jacobians && jacobians[0]) {
        std::memset(jacobians[0], 0, sizeof(double) * 54);
        for (int k = 0; k < 3; k++) {
            jacobians[0][k * 9 + k + 3]       = 1.0 / GB;
            jacobians[0][(k + 3) * 9 + k + 6] = 1.0 / AB;
        }
    }
    return true;
}

bool ImuPosePriorFactor::Evaluate(double const *const *parameters, double *residuals, double **jacobians) const {
    // imu_pose_prior_factor.h:42-68
    for (int k = 0; k < 3; k++) residuals[k] = parameters[0][k] - pose[k];
    Q q_p = pose_q(pose), q = pose_q(parameters[0]);
    Q dq  = q_inverse(q) * q_p;
    V3 a  = 2.0 * vec(dq);
    residuals[3] = a.x, residuals[4] = a.y, residuals[5] = a.z;
    for (int k = 0; k < 6; k++) residuals[k] *= sqrt_info[k];
    if (jacobians && jacobians[0]) {
        double *J = jacobians[0];
        std::memset(J, 0, sizeof(double) * 42);
        M3 b = -qright_br(dq);
        for (int r = 0; r < 3; r++) {
            J[r * 7 + r] = sqrt_info[r];
            for (int c = 0; c < 3; c++) J[(3 + r) * 7 + 3 + c] = sqrt_info[3 + r] * b(r, c);
        }
    }
    return true;
}

bool ImuMixPriorFactor::Evaluate(double const *const *parameters, double *residuals, double **jacobians) const {
    // imu_mix_prior_factor.h:40-75
    for (int k = 0; k < 9; k++) residuals[k] = (parameters[0][k] - mix[k]) / mix_std[k];
    if (jacobians && jacobians[0]) {
        std::memset(jacobians[0], 0, sizeof(double) * 81);
        for (int k = 0; k < 9; k++) jacobians[0][k * 9 + k] = 1.0 / mix_std[k];
    }
    return true;
}

bool MarginalizationFactor::Evaluate(double const *const *parameters, double *residuals, double **jacobians) const {
    // marginalization_factor.h:47-101
    std::vector<double> dx(r, 0.0);
    int off = 0;
    for (size_t i = 0; i < block_size.size(); i++) {
        int size = block_size[i], index = block_index[i];
        const double *x = parameters[i], *xl = &x0[off];
        if (size == 7) {
            Q dq = q_inverse(pose_q(xl)) * pose_q(x);
            for (int k = 0; k < 3; k++) dx[index + k] = x[k] - xl[k];
            V3 a = 2.0 * vec(dq);
            if (dq.w < 0) a = -a;
            dx[index + 3] = a.x, dx[index + 4] = a.y, dx[index + 5] = a.z;
        } else {
            for (int k = 0; k < size; k++) dx[index + k] = x[k] - xl[k];
        }
        off += size;
    }
    for (int i = 0; i < r; i++) {
        double s = e0[i];
        for (int k = 0; k < r; k++) s += J0[(size_t) i * r + k] * dx[k];
        residuals[i] = s;
    }
    if (jacobians) {
        for (size_t b = 0; b < block_size.size(); b++) {
            if (!jacobians[b]) continue;
            int size = block_size[b], index = block_index[b], local = size == 7 ? 6 : size;
            for (int i = 0; i < r; i++)
                for (int c = 0; c < size; c++) jacobians[b][(size_t) i * size + c] = c < local ? J0[(size_t) i * r + index + c] : 0.0;
        }
    }
    return true;
}

// ===================================================================================== IMU propagation (B3)
static void mat15_mul(const double *A, const double *B, double *C) {
    for (int i = 0; i < 15; i++)
        for (int j = 0; j < 15; j++) {
            double s = 0;
            for (int k = 0; k < 15; k++) s += A[i * 15 + k] * B[k * 15 + j];
            C[i * 15 + j] = s;
        }
}

// covariance_ = phi covariance_ phi^T + 0.5 dt (phi G + G phi^T), G = gt noise_ gt^T  (preintegration_earth.cc:296-302, _normal.cc:226-231)
static void propagate_covariance(Preintegration &P, const double *phi, const double *gt, double dt) {
    // G = gt * noise * gt^T (15x15)
    double gn[15 * 12], G[225];
    for (int i = 0; i < 15; i++)
        for (int j = 0; j < 12; j++) {
            double s = 0;
            for (int k = 0; k < 12; k++) s += gt[i * 12 + k] * P.noise[k * 12 + j];
            gn[i * 12 + j] = s;
        }
    for (int i = 0; i < 15; i++)
        for (int j = 0; j < 15; j++) {
            double s = 0;
            for (int k = 0; k < 12; k++) s += gn[i * 12 + k] * gt[j * 12 + k];
            G[i * 15 + j] = s;
        }
    double pg[225], cov2[225], pc[225];
    mat15_mul(phi, G, pg);  // phi * G
    // Qk = 0.5 dt (phi G + G phi^T)
    mat15_mul(phi, P.covariance, pc);
    for (int i = 0; i < 15; i++)
        for (int j = 0; j < 15; j++) {
            double s = 0;
            for (int k = 0; k < 15; k++) s += pc[i * 15 + k] * phi[j * 15 + k];
            double gpt = 0;
            for (int k = 0; k < 15; k++) gpt += G[i * 15 + k] * phi[j * 15 + k];
            cov2[i * 15 + j] = s + 0.5 * dt * (pg[i * 15 + j] + gpt);
        }
    std::memcpy(P.covariance, cov2, sizeof(cov2));
}

void preint_reset(Preintegration &P, V3 p, Q q, V3 v, V3 bg, V3 ba, V3 iewn, V3 gravity, double gyr_arw, double acc_vrw, double gyr_bias_std,
                  double acc_bias_std, double corr_time) {
    // resetState (preintegration_earth.cc:305-324) + setNoiseMatrix (:326-334)
    P.delta_time = 0;
    P.dp = {0, 0, 0};
    P.dv = {0, 0, 0};
    P.dq = {1, 0, 0, 0};
    P.bg = bg;
    P.ba = ba;
    for (int i = 0; i < 225; i++) P.jacobian[i] = 0, P.covariance[i] = 0;
    for (int i = 0; i < 15; i++) P.jacobian[i * 15 + i] = 1;
    P.q0 = q;
    P.cur_p = p, P.cur_q = q, P.cur_v = v;
    P.iewn = iewn;
    P.gravity = gravity;
    P.pn.clear();
    P.corr_time = corr_time;
    for (int i = 0; i < 144; i++) P.noise[i] = 0;
    for (int k = 0; k < 3; k++) {
        P.noise[(k) * 12 + k]         = gyr_arw * gyr_arw;
        P.noise[(3 + k) * 12 + 3 + k] = acc_vrw * acc_vrw;
        P.noise[(6 + k) * 12 + 6 + k] = 2 * gyr_bias_std * gyr_bias_std / corr_time;
        P.noise[(9 + k) * 12 + 9 + k] = 2 * acc_bias_std * acc_bias_std / corr_time;
    }
}

void preint_add_imu(Preintegration &P, const double *pre_raw, const double *cur_raw) {
    // compensationBias (preintegration_base.cc:84-90)
    auto comp = [&](const double *imu, double &dt, V3 &dth, V3 &dvl) {
        dt  = imu[0];
        dth = V3{imu[1], imu[2], imu[3]} - dt * P.bg;
        dvl = V3{imu[4], imu[5], imu[6]} - dt * P.ba;
    };
    double dtp, dt;
    V3 pth, pvl, cth, cvl;
    comp(pre_raw, dtp, pth, pvl);
    comp(cur_raw, dt, cth, cvl);
    if (P.normal) {
        // PreintegrationBase::integration (preintegration_base.cc:39-70) + PreintegrationNormal::updateJacobianAndCovariance
        // (preintegration_normal.cc:195-232)
        P.delta_time += dt;
        V3 dvfb = cvl + 0.5 * cross(cth, cvl) + (1.0 / 12.0) * (cross(pth, cvl) + cross(pvl, cth));
        V3 dvel = q_matrix(P.cur_q) * dvfb + P.gravity * dt;
        P.cur_p = P.cur_p + dt * P.cur_v + 0.5 * dt * dvel;
        P.cur_v = P.cur_v + dvel;
        V3 dtheta = cth + (1.0 / 12.0) * cross(pth, cth);
        P.cur_q = q_normalized(P.cur_q * rotvec2quaternion(dtheta));
        dvel = q_matrix(P.dq) * dvfb;
        P.dp = P.dp + dt * P.dv + 0.5 * dt * dvel;
        P.dv = P.dv + dvel;
        P.dq = q_normalized(P.dq * rotvec2quaternion(dtheta));
        double phi[225] = {0};
        M3 Rdq = q_matrix(P.dq);
        set_block(phi, 15, 0, 0, m3_identity());
        set_block(phi, 15, 0, 3, dt * m3_identity());
        set_block(phi, 15, 3, 3, m3_identity());
        set_block(phi, 15, 3, 6, -(Rdq * skew(cvl)));
        set_block(phi, 15, 3, 12, -dt * Rdq);
        set_block(phi, 15, 6, 6, m3_identity() - skew(cth));
        set_block(phi, 15, 6, 9, -dt * m3_identity());
        set_block(phi, 15, 9, 9, (1 - dt / P.corr_time) * m3_identity());
        set_block(phi, 15, 12, 12, (1 - dt / P.corr_time) * m3_identity());
        double tmp[225];
        mat15_mul(phi, P.jacobian, tmp);
        std::memcpy(P.jacobian, tmp, sizeof(tmp));
        double gt[15 * 12] = {0};
        set_block(gt, 12, 3, 3, Rdq);
        set_block(gt, 12, 6, 0, m3_identity());
        set_block(gt, 12, 9, 6, m3_identity());
        set_block(gt, 12, 12, 9, m3_identity());
        propagate_covariance(P, phi, gt, dt);
        return;
    }
    // integrationProcess (preintegration_earth.cc:205-260)
    P.delta_time += dt;
    V3 dvfb     = cvl + 0.5 * cross(cth, cvl) + (1.0 / 12.0) * (cross(pth, cvl) + cross(pvl, cth));
    V3 dv_cor_g = (P.gravity - 2.0 * cross(P.iewn, P.cur_v)) * dt;
    V3 dnn      = -(P.iewn * dt);
    Q qnn       = rotvec2quaternion(dnn);
    V3 dvel     = (0.5 * (m3_identity() + q_matrix(qnn))) * (q_matrix(P.cur_q) * dvfb) + dv_cor_g;
    P.cur_p     = P.cur_p + dt * P.cur_v + 0.5 * dt * dvel;
    P.cur_v     = P.cur_v + dvel;
    P.pn.push_back(dt);
    P.pn.push_back(P.cur_p.x);
    P.pn.push_back(P.cur_p.y);
    P.pn.push_back(P.cur_p.z);
    V3 dtheta = cth + (1.0 / 12.0) * cross(pth, cth);
    P.cur_q   = q_normalized(qnn * P.cur_q * rotvec2quaternion(dtheta));
    dnn       = -((P.delta_time - 0.5 * dt) * P.iewn);
    dvel      = q_matrix(q_inverse(P.q0) * rotvec2quaternion(dnn) * P.q0 * P.dq) * dvfb;
    P.dp      = P.dp + dt * P.dv + 0.5 * dt * dvel;
    P.dv      = P.dv + dvel;
    P.dq      = q_normalized(P.dq * rotvec2quaternion(dtheta));
    // updateJacobianAndCovariance (:266-303)
    double phi[225] = {0};
    dnn     = -(P.iewn * P.delta_time);
    M3 cbb0 = -q_matrix(q_inverse(P.q0) * rotvec2quaternion(dnn) * P.q0 * P.dq);
    auto setb = [&](double *M, int nc, int r, int c, const M3 &m) { set_block(M, nc, r, c, m); };
    setb(phi, 15, 0, 0, m3_identity());
    setb(phi, 15, 0, 3, dt * m3_identity());
    setb(phi, 15, 3, 3, m3_identity());
    setb(phi, 15, 3, 6, cbb0 * skew(cvl));
    setb(phi, 15, 3, 12, dt * cbb0);
    setb(phi, 15, 6, 6, m3_identity() - skew(cth));
    setb(phi, 15, 6, 9, -dt * m3_identity());
    setb(phi, 15, 9, 9, (1 - dt / P.corr_time) * m3_identity());
    setb(phi, 15, 12, 12, (1 - dt / P.corr_time) * m3_identity());
    double tmp[225];
    mat15_mul(phi, P.jacobian, tmp);
    std::memcpy(P.jacobian, tmp, sizeof(tmp));
    double gt[15 * 12] = {0};
    setb(gt, 12, 3, 3, cbb0);
    setb(gt, 12, 6, 0, -m3_identity());
    setb(gt, 12, 9, 6, m3_identity());
    setb(gt, 12, 12, 9, m3_identity());
    propagate_covariance(P, phi, gt, dt);
}

// ===================================================================================== residual blocks + Ceres-style evaluation
namespace {

struct Block {  // parameter block
    double *data;
    int gsize, lsize;
    bool is_pose, constant;
    int col;  // column offset in the reduced program (local coordinates); -1 if constant
};
struct Residual {
    const CostFunction *cost;
    bool huber;
    std::vector<int> blocks;
    bool active = true;
};

struct Program {
    std::vector<Block> blocks;
    std::vector<Residual> residuals;
    int n_cam = 0, n_lm = 0, lm_block0 = 0;  // landmark blocks are [lm_block0, lm_block0 + n_lm)
    std::vector<const CostFunction *> owned;
    ~Program() {
        for (auto *c : owned) delete c;
    }
};

// HuberLoss(1.0)::Evaluate (Ceres loss_function.cc)
inline void huber(double s, double rho[3]) {
    const double a = 1.0, b = 1.0;
    if (s > b) {
        const double r = std::sqrt(s);
        rho[0] = 2.0 * a * r - b;
        rho[1] = std::max(std::numeric_limits<double>::min(), a / r);
        rho[2] = -rho[1] / (2.0 * s);
    } else {
        rho[0] = s, rho[1] = 1.0, rho[2] = 0.0;
    }
}

// The loss as the solver applies it to one residual block: no loss, cost = 0.5 |r|^2; HuberLoss(1.0), cost = 0.5 rho(|r|^2) and the
// Corrector (ceres corrector.cc; the reference's own copy: factors/residual_block_info.h:59-87) on the residuals and on every non-null
// global Jacobian J[i] (nres x gsize[i], row-major).
void apply_loss(bool hub, int nres, double *r, int nb, double *const *J, const int *gsize, double &cost) {
    double sq = 0;
    for (int k = 0; k < nres; k++) sq += r[k] * r[k];
    if (!hub) {
        cost = 0.5 * sq;
        return;
    }
    double rho[3];
    huber(sq, rho);
    cost = 0.5 * rho[0];
    const double sqrt_rho1 = std::sqrt(rho[1]);
    double residual_scaling, alpha_sq_norm;
    if (sq == 0.0 || rho[2] <= 0.0) {
        residual_scaling = sqrt_rho1;
        alpha_sq_norm    = 0.0;
    } else {
        const double D     = 1.0 + 2.0 * sq * rho[2] / rho[1];
        const double alpha = 1.0 - std::sqrt(D);
        residual_scaling   = sqrt_rho1 / (1 - alpha);
        alpha_sq_norm      = alpha / sq;
    }
    for (int i = 0; J && i < nb; i++) {
        if (!J[i]) continue;
        const int gs = gsize[i];
        if (alpha_sq_norm == 0.0) {
            for (int e = 0; e < nres * gs; e++) J[i][e] *= sqrt_rho1;
        } else {
            for (int c = 0; c < gs; c++) {
                double rtj = 0;
                for (int k = 0; k < nres; k++) rtj += r[k] * J[i][(size_t) k * gs + c];
                for (int k = 0; k < nres; k++) J[i][(size_t) k * gs + c] = sqrt_rho1 * (J[i][(size_t) k * gs + c] - alpha_sq_norm * r[k] * rtj);
            }
        }
    }
    for (int k = 0; k < nres; k++) r[k] *= residual_scaling;
}

struct EvalBlock {  // one residual block's corrected residuals + local Jacobians
    int nres;
    std::vector<double> r;
    std::vector<std::vector<double>> J;  // per parameter block: nres x lsize (empty if constant)
    double cost;
};

void evaluate_block(const Program &P, const Residual &R, bool want_jac, EvalBlock &E, const std::vector<double *> *override_data = nullptr) {
    const int nres = R.cost->num_residuals();
    E.nres = nres;
    E.r.assign(nres, 0.0);
    const int nb = (int) R.blocks.size();
    // scratch reused across calls (per thread): the evaluation runs ~3 000 times per LM iteration, allocation must stay out of it
    static thread_local std::vector<const double *> params;
    static thread_local std::vector<std::vector<double>> Jg;
    static thread_local std::vector<double *> jp;
    params.assign(nb, nullptr);
    jp.assign(nb, nullptr);
    if ((int) Jg.size() < nb) Jg.resize(nb);
    for (int i = 0; i < nb; i++) {
        const Block &B = P.blocks[R.blocks[i]];
        params[i]      = override_data ? (*override_data)[R.blocks[i]] : B.data;
        if (want_jac && !B.constant) {
            Jg[i].assign((size_t) nres * B.gsize, 0.0);
            jp[i] = Jg[i].data();
        }
    }
    R.cost->Evaluate(params.data(), E.r.data(), want_jac ? jp.data() : nullptr);
    static thread_local std::vector<int> gs;
    gs.resize(nb);
    for (int i = 0; i < nb; i++) gs[i] = P.blocks[R.blocks[i]].gsize;
    apply_loss(R.huber, nres, E.r.data(), nb, want_jac ? jp.data() : nullptr, gs.data(), E.cost);
    if (want_jac) {
        E.J.resize(nb);
        for (int i = 0; i < nb; i++) {
            if (!jp[i]) {
                E.J[i].clear();
                continue;
            }
            const Block &B = P.blocks[R.blocks[i]];
            // local parameterization: J_local = J_global * [I6; 0] for poses (pose_parameterization.h:51-57), identity otherwise
            E.J[i].assign((size_t) nres * B.lsize, 0.0);
            for (int k = 0; k < nres; k++)
                for (int c = 0; c < B.lsize; c++) E.J[i][(size_t) k * B.lsize + c] = Jg[i][(size_t) k * B.gsize + c];
        }
    }
}

void build_program(WindowProblem &W, Program &P) {
    const int K = W.K, L = W.L;
    P.blocks.clear();
    for (int k = 0; k < K; k++) {
        P.blocks.push_back({&W.pose[7 * k], 7, 6, true, false, 0});
        P.blocks.push_back({&W.mix[9 * k], 9, 9, false, false, 0});
    }
    P.blocks.push_back({W.ext, 7, 6, true, W.ext_const, 0});
    P.blocks.push_back({&W.ext[7], 1, 1, false, W.td_const, 0});
    P.lm_block0 = (int) P.blocks.size();
    P.n_lm      = L;
    for (int l = 0; l < L; l++) P.blocks.push_back({&W.invdepth[l], 1, 1, false, false, 0});
    int col = 0;
    for (int b = 0; b < P.lm_block0; b++) {
        if (P.blocks[b].constant) {
            P.blocks[b].col = -1;
        } else {
            P.blocks[b].col = col;
            col += P.blocks[b].lsize;
        }
    }
    P.n_cam = col;
    for (int l = 0; l < L; l++) P.blocks[P.lm_block0 + l].col = col + l;

    auto add = [&](const CostFunction *c, bool own, bool hub, std::vector<int> blocks) {
        if (own) P.owned.push_back(c);
        P.residuals.push_back({c, hub, std::move(blocks), true});
    };
    // order of insertion follows gvinsOptimization (ic_gvins.cc:1158-1173): prior, GNSS, IMU, reprojection
    if (W.has_marg) {
        std::vector<int> bl;
        for (size_t i = 0; i < W.marg_block_type.size(); i++) {
            int t = W.marg_block_type[i], nd = W.marg_block_node[i];
            bl.push_back(t == 0 ? 2 * nd : t == 1 ? 2 * nd + 1 : t == 2 ? 2 * K : 2 * K + 1);
        }
        add(&W.marg, false, false, bl);
    }
    for (size_t g = 0; g < W.gnss_node.size(); g++)
        add(new GnssFactor({W.gnss_blh[3 * g], W.gnss_blh[3 * g + 1], W.gnss_blh[3 * g + 2]}, {W.gnss_std[3 * g], W.gnss_std[3 * g + 1], W.gnss_std[3 * g + 2]},
                           W.lever),
            true, W.gnss_huber, {2 * W.gnss_node[g]});
    for (size_t k = 0; k < W.preint.size(); k++) add(new PreintegrationFactor(&W.preint[k]), true, false, {2 * (int) k, 2 * (int) k + 1, 2 * (int) k + 2, 2 * (int) k + 3});
    if (W.has_imu_error) add(new ImuErrorFactor(), true, false, {2 * (int) W.preint.size() + 1});
    if (W.has_pose_prior) add(&W.pose_prior, false, false, {0});
    if (W.has_mix_prior) add(&W.mix_prior, false, false, {1});
    const int F = (int) W.f_lm.size();
    for (int f = 0; f < F; f++) {
        if (!W.f_active.empty() && !W.f_active[f]) continue;
        const double *c = &W.f_const[14 * f];
        add(new ReprojectionFactor({c[0], c[1], c[2]}, {c[3], c[4], c[5]}, {c[6], c[7], c[8]}, {c[9], c[10], c[11]}, c[12], c[13], W.reproj_std), true,
            W.reproj_huber, {2 * W.f_ref[f], 2 * W.f_obs[f], 2 * K, P.lm_block0 + W.f_lm[f], 2 * K + 1});
    }
}

// evaluate everything at the current (or candidate) point
double evaluate_all(const Program &P, bool want_jac, std::vector<EvalBlock> &E, const std::vector<double *> *cand, int num_threads) {
    const int nr = (int) P.residuals.size();
    E.resize(nr);
    auto work = [&](int t0, int t1) {
        for (int i = t0; i < t1; i++) evaluate_block(P, P.residuals[i], want_jac, E[i], cand);
    };
    if (num_threads <= 1 || nr < 64) {
        work(0, nr);
    } else {
        std::vector<std::thread> th;
        int per = (nr + num_threads - 1) / num_threads;
        for (int t = 0; t < num_threads; t++) th.emplace_back(work, std::min(nr, t * per), std::min(nr, (t + 1) * per));
        for (auto &t : th) t.join();
    }
    double cost = 0;
    for (int i = 0; i < nr; i++) cost += E[i].cost;
    return cost;
}

}  // namespace

// ===================================================================================== Solver::Solve (LM + DENSE_SCHUR)
SolveSummary solve(WindowProblem &W, int max_num_iterations, int num_threads) {
    // Ceres defaults left untouched by the reference (ic_gvins.cc:1143-1146)
    const double initial_radius = 1e4, max_radius = 1e16, min_radius = 1e-32, min_relative_decrease = 1e-3;
    const double min_lm_diag = 1e-6, max_lm_diag = 1e32;
    const double function_tolerance = 1e-6, gradient_tolerance = 1e-10, parameter_tolerance = 1e-8;
    const int max_consecutive_invalid = 5;

    Program P;
    build_program(W, P);
    const int nc = P.n_cam, L = P.n_lm, n = nc + L;
    SolveSummary S;

    auto x_norm = [&]() {
        double s = 0;
        for (const Block &B : P.blocks)
            if (!B.constant)
                for (int i = 0; i < B.gsize; i++) s += B.data[i] * B.data[i];
        return std::sqrt(s);
    };

    std::vector<EvalBlock> E;
    double x_cost = evaluate_all(P, true, E, nullptr, num_threads);
    S.initial_cost = x_cost;
    // which landmark blocks actually appear (Ceres removes unused parameter blocks from the reduced program)
    std::vector<double> scale(n, 1.0), grad(n, 0.0), colsq(n, 0.0);
    auto accumulate = [&](bool first) {
        std::fill(grad.begin(), grad.end(), 0.0);
        std::fill(colsq.begin(), colsq.end(), 0.0);
        for (size_t i = 0; i < E.size(); i++) {
            const Residual &R = P.residuals[i];
            for (size_t b = 0; b < R.blocks.size(); b++) {
                const Block &B = P.blocks[R.blocks[b]];
                if (B.constant) continue;
                const auto &J = E[i].J[b];
                for (int c = 0; c < B.lsize; c++) {
                    double g = 0, s2 = 0;
                    for (int k = 0; k < E[i].nres; k++) {
                        double v = J[(size_t) k * B.lsize + c];
                        g += v * E[i].r[k];
                        s2 += v * v;
                    }
                    grad[B.col + c] += g;
                    colsq[B.col + c] += s2;
                }
            }
        }
        if (first)
            for (int i = 0; i < n; i++) scale[i] = 1.0 / (1.0 + std::sqrt(colsq[i]));  // jacobi_scaling (once, iteration 0)
    };
    accumulate(true);
    double gmax = 0;
    for (int i = 0; i < n; i++) gmax = std::max(gmax, std::fabs(grad[i]));
    double xn = x_norm();
    if (gmax <= gradient_tolerance) {
        S.termination = 1;
        S.final_cost  = x_cost;
        return S;
    }

    double radius = initial_radius, decrease_factor = 2.0;
    int invalid = 0;
    bool last_successful = true;
    std::vector<double> Hcc, Wm, hl, gl, gc, diag(n), step(n), delta(n);
    std::vector<double> cand_store;
    std::vector<double *> cand(P.blocks.size());
    {
        size_t tot = 0;
        for (const Block &B : P.blocks) tot += B.gsize;
        cand_store.resize(tot);
        size_t o = 0;
        for (size_t b = 0; b < P.blocks.size(); b++) {
            cand[b] = &cand_store[o];
            o += P.blocks[b].gsize;
        }
    }
    bool need_assemble = true;

    for (int iter = 1;; iter++) {
        // FinalizeIterationAndCheckIfMinimizerCanContinue
        if (iter - 1 >= max_num_iterations) {
            S.termination = 0;
            break;
        }
        if (last_successful && gmax <= gradient_tolerance) {
            S.termination = 1;
            break;
        }
        if (last_successful && radius <= min_radius) {
            S.termination = 1;
            break;
        }
        S.iterations = iter;

        if (need_assemble) {
            // normal equations of the scaled Jacobian J' = J diag(scale): camera block dense, landmark block diagonal
            Hcc.assign((size_t) nc * nc, 0.0);
            Wm.assign((size_t) nc * L, 0.0);
            hl.assign(L, 0.0);
            gl.assign(L, 0.0);
            gc.assign(nc, 0.0);
            for (size_t i = 0; i < E.size(); i++) {
                const Residual &R = P.residuals[i];
                const int nres    = E[i].nres;
                for (size_t a = 0; a < R.blocks.size(); a++) {
                    const Block &A = P.blocks[R.blocks[a]];
                    if (A.constant) continue;
                    const auto &JA  = E[i].J[a];
                    const bool a_lm = R.blocks[a] >= P.lm_block0;
                    for (int ca = 0; ca < A.lsize; ca++) {
                        const double sa = scale[A.col + ca];
                        double g = 0;
                        for (int k = 0; k < nres; k++) g += JA[(size_t) k * A.lsize + ca] * E[i].r[k];
                        g *= sa;
                        if (a_lm)
                            gl[A.col - nc] += g;
                        else
                            gc[A.col + ca] += g;
                        for (size_t b = 0; b < R.blocks.size(); b++) {
                            const Block &B = P.blocks[R.blocks[b]];
                            if (B.constant) continue;
                            const bool b_lm = R.blocks[b] >= P.lm_block0;
                            const auto &JB  = E[i].J[b];
                            for (int cb = 0; cb < B.lsize; cb++) {
                                double s = 0;
                                for (int k = 0; k < nres; k++) s += JA[(size_t) k * A.lsize + ca] * JB[(size_t) k * B.lsize + cb];
                                s *= sa * scale[B.col + cb];
                                if (!a_lm && !b_lm)
                                    Hcc[(size_t) (A.col + ca) * nc + B.col + cb] += s;
                                else if (!a_lm && b_lm)
                                    Wm[(size_t) (A.col + ca) * L + (B.col - nc)] += s;
                                else if (a_lm && b_lm)
                                    hl[A.col - nc] += s;
                            }
                        }
                    }
                }
            }
            // LM diagonal source: diag(J'^T J')
            for (int i = 0; i < nc; i++) diag[i] = Hcc[(size_t) i * nc + i];
            for (int l = 0; l < L; l++) diag[nc + l] = hl[l];
            need_assemble = false;
        }
        // LevenbergMarquardtStrategy::ComputeStep: D^2 = clamp(diag) / radius
        std::vector<double> D2(n);
        for (int i = 0; i < n; i++) D2[i] = std::min(std::max(diag[i], min_lm_diag), max_lm_diag) / radius;
        // Schur complement on the landmark (e) blocks, dense Cholesky of the reduced camera system
        std::vector<double> Sred(Hcc), rhs(nc);
        for (int i = 0; i < nc; i++) {
            Sred[(size_t) i * nc + i] += D2[i];
            rhs[i] = -gc[i];
        }
        std::vector<double> hinv(L, 0.0);
        for (int l = 0; l < L; l++) {
            double h = hl[l] + D2[nc + l];
            hinv[l]  = 1.0 / h;
        }
        // only camera columns that couple to some landmark have a non-zero row in W (the mix blocks never do): restricting the
        // Schur update to them skips exact zeros only -- same values, as Ceres' block-sparse Schur eliminator does structurally
        std::vector<int> nzrow;
        for (int i = 0; i < nc; i++) {
            const double *wi = &Wm[(size_t) i * L];
            bool any = false;
            for (int l = 0; l < L && !any; l++) any = wi[l] != 0.0;
            if (any) nzrow.push_back(i);
        }
        for (size_t ii = 0; ii < nzrow.size(); ii++) {
            const int i = nzrow[ii];
            const double *wi = &Wm[(size_t) i * L];
            double s = 0;
            for (int l = 0; l < L; l++) s += wi[l] * hinv[l] * (-gl[l]);
            rhs[i] -= s;
            for (size_t jj = ii; jj < nzrow.size(); jj++) {
                const int j = nzrow[jj];
                const double *wj = &Wm[(size_t) j * L];
                double t = 0;
                for (int l = 0; l < L; l++) t += wi[l] * hinv[l] * wj[l];
                Sred[(size_t) i * nc + j] -= t;
                if (j != i) Sred[(size_t) j * nc + i] -= t;
            }
        }
        bool ok = cholesky_lower(Sred.data(), nc);
        bool step_valid = false;
        double model_cost_change = 0;
        if (ok) {
            // solve L L^T y = rhs
            std::vector<double> y(rhs);
            for (int i = 0; i < nc; i++) {
                double s = y[i];
                for (int k = 0; k < i; k++) s -= Sred[(size_t) i * nc + k] * y[k];
                y[i] = s / Sred[(size_t) i * nc + i];
            }
            for (int i = nc - 1; i >= 0; i--) {
                double s = y[i];
                for (int k = i + 1; k < nc; k++) s -= Sred[(size_t) k * nc + i] * y[k];
                y[i] = s / Sred[(size_t) i * nc + i];
            }
            for (int i = 0; i < nc; i++) step[i] = y[i];
            // back-substitution of the landmarks
            for (int l = 0; l < L; l++) {
                double s = -gl[l];
                for (int i = 0; i < nc; i++) s -= Wm[(size_t) i * L + l] * step[i];
                step[nc + l] = s * hinv[l];
            }
            bool finite = true;
            for (int i = 0; i < n; i++) finite = finite && std::isfinite(step[i]);
            if (finite) {
                // model_cost_change = -(J' step)^T (r + J' step / 2)   (TrustRegionMinimizer::ComputeTrustRegionStep)
                double mcc = 0;
                for (size_t i = 0; i < E.size(); i++) {
                    const Residual &R = P.residuals[i];
                    for (int k = 0; k < E[i].nres; k++) {
                        double m = 0;
                        for (size_t b = 0; b < R.blocks.size(); b++) {
                            const Block &B = P.blocks[R.blocks[b]];
                            if (B.constant) continue;
                            for (int c = 0; c < B.lsize; c++) m += E[i].J[b][(size_t) k * B.lsize + c] * scale[B.col + c] * step[B.col + c];
                        }
                        mcc -= m * (E[i].r[k] + m / 2.0);
                    }
                }
                model_cost_change = mcc;
                step_valid        = mcc > 0.0;
            }
        }
        if (!step_valid) {
            // HandleInvalidStep + LevenbergMarquardtStrategy::StepIsInvalid
            if (++invalid >= max_consecutive_invalid) {
                S.termination = 2;
                break;
            }
            radius *= 0.5;
            last_successful = false;
            continue;
        }
        invalid = 0;
        for (int i = 0; i < n; i++) delta[i] = step[i] * scale[i];
        // candidate point
        for (size_t b = 0; b < P.blocks.size(); b++) {
            const Block &B = P.blocks[b];
            if (B.constant) {
                std::memcpy(cand[b], B.data, sizeof(double) * B.gsize);
            } else if (B.is_pose) {
                pose_plus(B.data, &delta[B.col], cand[b]);
            } else {
                for (int i = 0; i < B.gsize; i++) cand[b][i] = B.data[i] + delta[B.col + i];
            }
        }
        std::vector<EvalBlock> Ec;
        double cand_cost = evaluate_all(P, false, Ec, &cand, num_threads);
        // ParameterToleranceReached
        double step_norm = 0;
        for (size_t b = 0; b < P.blocks.size(); b++)
            if (!P.blocks[b].constant)
                for (int i = 0; i < P.blocks[b].gsize; i++) {
                    double d = P.blocks[b].data[i] - cand[b][i];
                    step_norm += d * d;
                }
        step_norm = std::sqrt(step_norm);
        if (step_norm <= parameter_tolerance * (xn + parameter_tolerance)) {
            S.termination = 1;
            break;
        }
        // FunctionToleranceReached
        double cost_change = x_cost - cand_cost;
        if (std::fabs(cost_change) <= function_tolerance * x_cost) {
            S.termination = 1;
            break;
        }
        double relative_decrease = cost_change / model_cost_change;
        if (relative_decrease > min_relative_decrease) {
            // HandleSuccessfulStep
            for (size_t b = 0; b < P.blocks.size(); b++)
                if (!P.blocks[b].constant) std::memcpy(P.blocks[b].data, cand[b], sizeof(double) * P.blocks[b].gsize);
            xn     = x_norm();
            x_cost = evaluate_all(P, true, E, nullptr, num_threads);
            accumulate(false);
            gmax = 0;
            for (int i = 0; i < n; i++) gmax = std::max(gmax, std::fabs(grad[i]));
            need_assemble = true;
            S.num_successful_steps++;
            // LevenbergMarquardtStrategy::StepAccepted
            radius          = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * relative_decrease - 1.0, 3));
            radius          = std::min(max_radius, radius);
            decrease_factor = 2.0;
            last_successful = true;
        } else {
            // StepRejected
            radius          = radius / decrease_factor;
            decrease_factor *= 2.0;
            last_successful = false;
        }
    }
    S.final_cost   = x_cost;
    S.final_radius = radius;
    return S;
}

void reproj_costs(const WindowProblem &Wc, std::vector<double> &cost) {
    WindowProblem &W = const_cast<WindowProblem &>(Wc);
    const int F = (int) W.f_lm.size();
    cost.assign(F, 0.0);
    for (int f = 0; f < F; f++) {
        const double *c = &W.f_const[14 * f];
        ReprojectionFactor fac({c[0], c[1], c[2]}, {c[3], c[4], c[5]}, {c[6], c[7], c[8]}, {c[9], c[10], c[11]}, c[12], c[13], W.reproj_std);
        const double *params[5] = {&W.pose[7 * W.f_ref[f]], &W.pose[7 * W.f_obs[f]], W.ext, &W.invdepth[W.f_lm[f]], &W.ext[7]};
        double r[2];
        fac.Evaluate(params, r, nullptr);
        double sq = r[0] * r[0] + r[1] * r[1];
        // EvaluateResidualBlock(id, apply_loss_function=false, &cost, ...): cost = 0.5 |r|^2 (ic_gvins.cc:1278)
        cost[f] = 0.5 * sq;
    }
}

void gnss_costs(const WindowProblem &Wc, std::vector<double> &cost) {
    WindowProblem &W = const_cast<WindowProblem &>(Wc);
    const int G = (int) W.gnss_node.size();
    cost.assign(G, 0.0);
    for (int g = 0; g < G; g++) {
        GnssFactor fac({W.gnss_blh[3 * g], W.gnss_blh[3 * g + 1], W.gnss_blh[3 * g + 2]}, {W.gnss_std[3 * g], W.gnss_std[3 * g + 1], W.gnss_std[3 * g + 2]}, W.lever);
        const double *params[1] = {&W.pose[7 * W.gnss_node[g]]};
        double r[3];
        fac.Evaluate(params, r, nullptr);
        cost[g] = 0.5 * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    }
}


// ===================================================================================== sliding-window marginalization (B10)
// Restates GVINS::gvinsMarginalization (ic_gvins/ic_gvins/ic_gvins.cc:1412-1640) + MarginalizationInfo
// (ic_gvins/ic_gvins/factors/marginalization_info.h:73-253) + ResidualBlockInfo::Evaluate (residual_block_info.h:45-91).
// Eigen::SelfAdjointEigenSolver is un-vendored; a cyclic two-sided Jacobi eigensolver stands in for it (same decomposition up
// to rounding; the decomposition is pinned against numpy.linalg.eigh in tests/test_oracle_marg.py).
void sym_eig_jacobi(std::vector<double> &A, int n, std::vector<double> &evals, std::vector<double> &V) {
    // A: n x n row-major symmetric (destroyed); V columns = eigenvectors
    V.assign((size_t) n * n, 0.0);
    for (int i = 0; i < n; i++) V[(size_t) i * n + i] = 1.0;
    for (int sweep = 0; sweep < 60; sweep++) {
        double off = 0, diag = 0;
        for (int i = 0; i < n; i++)
            for (int j = 0; j < n; j++) (i == j ? diag : off) += A[(size_t) i * n + j] * A[(size_t) i * n + j];
        if (off <= 1e-60 || off <= 1e-34 * diag) break;
        for (int p = 0; p < n - 1; p++)
            for (int q = p + 1; q < n; q++) {
                const double apq = A[(size_t) p * n + q];
                if (apq == 0.0) continue;
                const double app = A[(size_t) p * n + p], aqq = A[(size_t) q * n + q];
                const double theta = (aqq - app) / (2.0 * apq);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
                const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < n; k++) {  // columns p, q
                    const double akp = A[(size_t) k * n + p], akq = A[(size_t) k * n + q];
                    A[(size_t) k * n + p] = c * akp - s * akq;
                    A[(size_t) k * n + q] = s * akp + c * akq;
                }
                for (int k = 0; k < n; k++) {  // rows p, q
                    const double apk = A[(size_t) p * n + k], aqk = A[(size_t) q * n + k];
                    A[(size_t) p * n + k] = c * apk - s * aqk;
                    A[(size_t) q * n + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < n; k++) {
                    const double vkp = V[(size_t) k * n + p], vkq = V[(size_t) k * n + q];
                    V[(size_t) k * n + p] = c * vkp - s * vkq;
                    V[(size_t) k * n + q] = s * vkp + c * vkq;
                }
            }
    }
    evals.resize(n);
    for (int i = 0; i < n; i++) evals[i] = A[(size_t) i * n + i];
}

void marginalize(WindowProblem &W, int num_marg, MargOut &out) {
    const double EPS = 1e-8;  // MarginalizationInfo::EPS (marginalization_info.h:256)
    const int K = W.K, L = W.L, F = (int) W.f_lm.size();
    // ---- parameter blocks (ids in the order of ic_gvins.cc:1438-1476; no block is constant here: ResidualBlockInfo asks
    //      the cost functions for every Jacobian, residual_block_info.h:49-57)
    Program P;
    for (int k = 0; k < K; k++) {
        P.blocks.push_back({&W.pose[7 * k], 7, 6, true, false, 0});
        P.blocks.push_back({&W.mix[9 * k], 9, 9, false, false, 0});
    }
    P.blocks.push_back({W.ext, 7, 6, true, false, 0});
    P.blocks.push_back({&W.ext[7], 1, 1, false, false, 0});
    P.lm_block0 = (int) P.blocks.size();
    for (int l = 0; l < L; l++) P.blocks.push_back({&W.invdepth[l], 1, 1, false, false, 0});
    const int NB = (int) P.blocks.size();
    std::vector<char> is_marg(NB, 0), touched(NB, 0);
    auto add = [&](const CostFunction *c, bool own, std::vector<int> blocks, std::vector<int> marg_idx) {
        if (own) P.owned.push_back(c);
        for (int b : blocks) touched[b] = 1;
        for (int i : marg_idx) is_marg[blocks[i]] = 1;
        P.residuals.push_back({c, false /* loss_function == nullptr everywhere, ic_gvins.cc:1499,1510,1532,1543,1605 */, std::move(blocks), true});
    };
    // the previous prior (ic_gvins.cc:1485-1501)
    if (W.has_marg) {
        std::vector<int> bl, mi;
        for (size_t i = 0; i < W.marg_block_type.size(); i++) {
            const int t = W.marg_block_type[i], nd = W.marg_block_node[i];
            bl.push_back(t == 0 ? 2 * nd : t == 1 ? 2 * nd + 1 : t == 2 ? 2 * K : 2 * K + 1);
            if ((t == 0 || t == 1) && nd < num_marg) mi.push_back((int) i);
        }
        add(&W.marg, false, bl, mi);
    }
    // GNSS factors at the removed nodes (:1505-1516)
    for (size_t g = 0; g < W.gnss_node.size(); g++)
        if (W.gnss_node[g] < num_marg)
            add(new GnssFactor({W.gnss_blh[3 * g], W.gnss_blh[3 * g + 1], W.gnss_blh[3 * g + 2]}, {W.gnss_std[3 * g], W.gnss_std[3 * g + 1], W.gnss_std[3 * g + 2]},
                               W.lever),
                true, {2 * W.gnss_node[g]}, {0});
    // preintegration factors (:1520-1538)
    for (int k = 0; k < num_marg && k < (int) W.preint.size(); k++)
        add(new PreintegrationFactor(&W.preint[k]), true, {2 * k, 2 * k + 1, 2 * k + 2, 2 * k + 3},
            k == num_marg - 1 ? std::vector<int>{0, 1} : std::vector<int>{0, 1, 2, 3});
    // first-window priors (:1542-1554)
    if (W.has_pose_prior) add(&W.pose_prior, false, {0}, {0});
    if (W.has_mix_prior) add(&W.mix_prior, false, {1}, {0});
    // reprojection factors of the landmarks anchored in the oldest keyframe (:1559-1611)
    for (int f = 0; f < F; f++) {
        if (!W.f_active.empty() && !W.f_active[f]) continue;
        if (W.f_ref[f] >= num_marg) continue;
        const double *c = &W.f_const[14 * f];
        add(new ReprojectionFactor({c[0], c[1], c[2]}, {c[3], c[4], c[5]}, {c[6], c[7], c[8]}, {c[9], c[10], c[11]}, c[12], c[13], W.reproj_std), true,
            {2 * W.f_ref[f], 2 * W.f_obs[f], 2 * K, P.lm_block0 + W.f_lm[f], 2 * K + 1}, {0, 3});
    }
    // ---- updateParameterBlocksIndex (marginalization_info.h:228-251): marginalized blocks first.  The reference iterates
    //      unordered_maps, so the order inside each group is implementation-defined; it only permutes rows / columns.  Here:
    //      marginalized = [pose_k, mix_k (k < num_marg), landmarks ascending]; remained = [pose_k, mix_k (k >= num_marg), ext, td].
    std::vector<int> col(NB, -1);
    int idx = 0;
    for (int b = 0; b < NB; b++)
        if (touched[b] && is_marg[b]) col[b] = idx, idx += P.blocks[b].lsize;
    const int m = idx;
    out.block_type.clear(), out.block_node.clear(), out.x0.clear();
    for (int b = 0; b < NB; b++)
        if (touched[b] && !is_marg[b]) {
            col[b] = idx, idx += P.blocks[b].lsize;
            const int t = b < 2 * K ? (b & 1) : b == 2 * K ? 2 : 3;
            out.block_type.push_back(t);
            out.block_node.push_back(b < 2 * K ? b / 2 - num_marg : 0);  // node index in the window AFTER the removal
            for (int k = 0; k < P.blocks[b].gsize; k++) out.x0.push_back(P.blocks[b].data[k]);  // preMarginalization copies the data (:270-283)
        }
    const int n0 = idx, r = n0 - m;
    out.m = m, out.r = r;
    if (m == 0) return;
    // ---- preMarginalization + constructEquation (:195-226, 253-285)
    std::vector<double> H0((size_t) n0 * n0, 0.0), b0(n0, 0.0);
    for (const Residual &R : P.residuals) {
        EvalBlock E;
        evaluate_block(P, R, true, E);
        const int nb = (int) R.blocks.size();
        for (int i = 0; i < nb; i++) {
            const int row0 = col[R.blocks[i]], rows = P.blocks[R.blocks[i]].lsize;
            for (int j = i; j < nb; j++) {
                const int col0 = col[R.blocks[j]], cols = P.blocks[R.blocks[j]].lsize;
                for (int a = 0; a < rows; a++)
                    for (int b = 0; b < cols; b++) {
                        double s = 0;
                        for (int k = 0; k < E.nres; k++) s += E.J[i][(size_t) k * rows + a] * E.J[j][(size_t) k * cols + b];
                        H0[(size_t) (row0 + a) * n0 + col0 + b] += s;
                        if (i != j) H0[(size_t) (col0 + b) * n0 + row0 + a] = H0[(size_t) (row0 + a) * n0 + col0 + b];
                    }
            }
            for (int a = 0; a < rows; a++) {
                double s = 0;
                for (int k = 0; k < E.nres; k++) s += E.J[i][(size_t) k * rows + a] * E.r[k];
                b0[row0 + a] -= s;
            }
        }
    }
    // ---- schurElimination (:170-193)
    std::vector<double> Hmm((size_t) m * m), ev, V;
    for (int i = 0; i < m; i++)
        for (int j = 0; j < m; j++) Hmm[(size_t) i * m + j] = 0.5 * (H0[(size_t) i * n0 + j] + H0[(size_t) j * n0 + i]);
    sym_eig_jacobi(Hmm, m, ev, V);
    std::vector<double> Hinv((size_t) m * m, 0.0);
    for (int k = 0; k < m; k++) {
        if (!(ev[k] > EPS)) continue;
        const double inv = 1.0 / ev[k];
        for (int i = 0; i < m; i++)
            for (int j = 0; j < m; j++) Hinv[(size_t) i * m + j] += V[(size_t) i * m + k] * inv * V[(size_t) j * m + k];
    }
    std::vector<double> T((size_t) r * m, 0.0);  // Hrm * Hmm^-1
    for (int i = 0; i < r; i++)
        for (int j = 0; j < m; j++) {
            double s = 0;
            for (int k = 0; k < m; k++) s += H0[(size_t) (m + i) * n0 + k] * Hinv[(size_t) k * m + j];
            T[(size_t) i * m + j] = s;
        }
    out.Hp.assign((size_t) r * r, 0.0), out.bp.assign(r, 0.0);
    for (int i = 0; i < r; i++) {
        for (int j = 0; j < r; j++) {
            double s = 0;
            for (int k = 0; k < m; k++) s += T[(size_t) i * m + k] * H0[(size_t) k * n0 + m + j];
            out.Hp[(size_t) i * r + j] = H0[(size_t) (m + i) * n0 + m + j] - s;
        }
        double s = 0;
        for (int k = 0; k < m; k++) s += T[(size_t) i * m + k] * b0[k];
        out.bp[i] = b0[m + i] - s;
    }
    // ---- linearization (:153-168)
    std::vector<double> Hp = out.Hp, S, V2;
    sym_eig_jacobi(Hp, r, S, V2);
    out.J0.assign((size_t) r * r, 0.0), out.e0.assign(r, 0.0);
    for (int k = 0; k < r; k++) {
        const double s = S[k] > EPS ? S[k] : 0.0, sinv = S[k] > EPS ? 1.0 / S[k] : 0.0;
        const double ss = std::sqrt(s), ssi = std::sqrt(sinv);
        double d = 0;
        for (int j = 0; j < r; j++) {
            out.J0[(size_t) k * r + j] = ss * V2[(size_t) j * r + k];
            d += V2[(size_t) j * r + k] * -out.bp[j];
        }
        out.e0[k] = ssi * d;
    }
}

}  // namespace icgo

// ===================================================================================== C API (ctypes) over the public problem struct
#include "../include/icgvins_b200.h"
using namespace icgo;

static void blob_to_preint(const double *b, const double *pn, int npn, Preintegration &P) {
    P.delta_time = b[0];
    P.dp = {b[1], b[2], b[3]};
    P.dv = {b[4], b[5], b[6]};
    P.dq = {b[10], b[7], b[8], b[9]};
    P.bg = {b[11], b[12], b[13]};
    P.ba = {b[14], b[15], b[16]};
    P.gravity = {b[17], b[18], b[19]};
    P.iewn    = {b[20], b[21], b[22]};
    std::memcpy(P.jacobian, b + 27, sizeof(double) * 225);
    std::memcpy(P.covariance, b + 252, sizeof(double) * 225);
    P.normal = b[477] != 0.0;
    P.pn.assign(pn, pn + 4 * (size_t) npn);
}

static void preint_to_blob(const Preintegration &P, double *b) {
    std::memset(b, 0, sizeof(double) * ICG_IMU_BLOB_DOUBLES);
    b[0] = P.delta_time;
    b[1] = P.dp.x, b[2] = P.dp.y, b[3] = P.dp.z, b[4] = P.dv.x, b[5] = P.dv.y, b[6] = P.dv.z;
    b[7] = P.dq.x, b[8] = P.dq.y, b[9] = P.dq.z, b[10] = P.dq.w;
    b[11] = P.bg.x, b[12] = P.bg.y, b[13] = P.bg.z, b[14] = P.ba.x, b[15] = P.ba.y, b[16] = P.ba.z;
    b[17] = P.gravity.x, b[18] = P.gravity.y, b[19] = P.gravity.z, b[20] = P.iewn.x, b[21] = P.iewn.y, b[22] = P.iewn.z;
    double s0 = 0, s1[3] = {0, 0, 0};
    for (size_t i = 0; i + 3 < P.pn.size(); i += 4) {
        s0 += P.pn[i];
        for (int k = 0; k < 3; k++) s1[k] += P.pn[i] * P.pn[i + 1 + k];
    }
    b[23] = s0, b[24] = s1[0], b[25] = s1[1], b[26] = s1[2];
    std::memcpy(b + 27, P.jacobian, sizeof(double) * 225);
    std::memcpy(b + 252, P.covariance, sizeof(double) * 225);
    b[477] = P.normal ? 1.0 : 0.0;
}

static void to_window(const icg_ba_problem *p, const double *pn, const int32_t *pn_off, WindowProblem &W) {
    W.K = p->K, W.L = p->L;
    W.pose.assign(p->pose, p->pose + 7 * p->K);
    W.mix.assign(p->mix, p->mix + 9 * p->K);
    std::memcpy(W.ext, p->ext, sizeof(double) * 8);
    W.invdepth.assign(p->invdepth, p->invdepth + p->L);
    W.ext_const = p->ext_const != 0, W.td_const = p->td_const != 0;
    W.f_lm.assign(p->f_lm, p->f_lm + p->F);
    W.f_ref.assign(p->f_ref, p->f_ref + p->F);
    W.f_obs.assign(p->f_obs, p->f_obs + p->F);
    W.f_const.assign(p->f_const, p->f_const + 14 * (size_t) p->F);
    if (p->f_active) W.f_active.assign(p->f_active, p->f_active + p->F);
    W.reproj_std = p->reproj_std, W.reproj_huber = p->reproj_huber != 0;
    W.preint.resize(p->n_imu);
    for (int k = 0; k < p->n_imu; k++)
        blob_to_preint(p->imu_blob + (size_t) k * ICG_IMU_BLOB_DOUBLES, pn + 4 * (size_t) pn_off[k], pn_off[k + 1] - pn_off[k], W.preint[k]);
    W.has_imu_error = p->has_imu_error != 0;
    W.has_pose_prior = p->has_pose_prior != 0;
    if (W.has_pose_prior) {
        std::memcpy(W.pose_prior.pose, p->pose_prior, sizeof(double) * 7);
        for (int k = 0; k < 6; k++) W.pose_prior.sqrt_info[k] = 1.0 / p->pose_prior_std[k];
    }
    W.has_mix_prior = p->has_mix_prior != 0;
    if (W.has_mix_prior) {
        std::memcpy(W.mix_prior.mix, p->mix_prior, sizeof(double) * 9);
        std::memcpy(W.mix_prior.mix_std, p->mix_prior_std, sizeof(double) * 9);
    }
    W.gnss_node.assign(p->gnss_node, p->gnss_node + p->n_gnss);
    W.gnss_blh.assign(p->gnss_blh, p->gnss_blh + 3 * p->n_gnss);
    W.gnss_std.assign(p->gnss_std, p->gnss_std + 3 * p->n_gnss);
    W.lever = {p->lever[0], p->lever[1], p->lever[2]};
    W.gnss_huber = p->gnss_huber != 0;
    W.has_marg = p->marg_r > 0;
    if (W.has_marg) {
        W.marg.r = p->marg_r;
        W.marg_block_type.assign(p->marg_block_type, p->marg_block_type + p->marg_nblocks);
        W.marg_block_node.assign(p->marg_block_node, p->marg_block_node + p->marg_nblocks);
        int col = 0, tot = 0;
        for (int i = 0; i < p->marg_nblocks; i++) {
            int t = p->marg_block_type[i], gs = t == 0 ? 7 : t == 1 ? 9 : t == 2 ? 7 : 1, ls = gs == 7 ? 6 : gs;
            W.marg.block_size.push_back(gs);
            W.marg.block_index.push_back(col);
            col += ls;
            tot += gs;
        }
        W.marg.x0.assign(p->marg_x0, p->marg_x0 + tot);
        W.marg.J0.assign(p->marg_J0, p->marg_J0 + (size_t) p->marg_r * p->marg_r);
        W.marg.e0.assign(p->marg_e0, p->marg_e0 + p->marg_r);
    }
}

extern "C" {

int icgo_ba_solve(const icg_ba_problem *p, const double *pn, const int32_t *pn_off, int max_iter, int num_threads, icg_ba_summary *out) {
    WindowProblem W;
    to_window(p, pn, pn_off, W);
    SolveSummary S = solve(W, max_iter, num_threads);
    std::memcpy(p->pose, W.pose.data(), sizeof(double) * 7 * p->K);
    std::memcpy(p->mix, W.mix.data(), sizeof(double) * 9 * p->K);
    std::memcpy(p->ext, W.ext, sizeof(double) * 8);
    std::memcpy(p->invdepth, W.invdepth.data(), sizeof(double) * p->L);
    if (out) {
        out->iterations = S.iterations, out->num_successful_steps = S.num_successful_steps, out->termination = S.termination;
        out->initial_cost = S.initial_cost, out->final_cost = S.final_cost, out->final_radius = S.final_radius;
    }
    return 0;
}

int icgo_ba_residual_costs(const icg_ba_problem *p, double *reproj_cost, double *gnss_cost) {
    WindowProblem W;
    int32_t zero[64] = {0};
    std::vector<int32_t> off(p->n_imu + 1, 0);
    (void) zero;
    icg_ba_problem q = *p;
    q.n_imu = 0;  // IMU blobs are irrelevant for these costs
    to_window(&q, nullptr, off.data(), W);
    std::vector<double> c;
    if (reproj_cost) {
        reproj_costs(W, c);
        std::memcpy(reproj_cost, c.data(), sizeof(double) * c.size());
    }
    if (gnss_cost) {
        gnss_costs(W, c);
        std::memcpy(gnss_cost, c.data(), sizeof(double) * c.size());
    }
    return 0;
}

// Build one preintegration from raw IMU samples (n x 7: dt, dtheta[3], dvel[3]); state = p[3] q_xyzw[4] v[3] bg[3] ba[3].
// noise = gyr_arw, acc_vrw, gyr_bias_std, acc_bias_std, corr_time.  Outputs the blob, the pn list (n-1 x 4) and the
// mechanised end state (p q v) so a generator can chain intervals.
int icgo_preintegrate(const double *state16, const double *iewn, const double *gravity, const double *noise5, const double *imu, int n,
                      double *blob, double *pn_out, double *end_state10) {
    Preintegration P;
    const V3 iw = iewn ? V3{iewn[0], iewn[1], iewn[2]} : V3{0, 0, 0};
    preint_reset(P, {state16[0], state16[1], state16[2]}, {state16[6], state16[3], state16[4], state16[5]}, {state16[7], state16[8], state16[9]},
                 {state16[10], state16[11], state16[12]}, {state16[13], state16[14], state16[15]}, iw,
                 {gravity[0], gravity[1], gravity[2]}, noise5[0], noise5[1], noise5[2], noise5[3], noise5[4]);
    P.normal = iewn == nullptr;  // iswithearth: false -> PreintegrationNormal (preintegration.h factory)
    for (int i = 1; i < n; i++) preint_add_imu(P, imu + 7 * (size_t) (i - 1), imu + 7 * (size_t) i);
    preint_to_blob(P, blob);
    if (pn_out) std::memcpy(pn_out, P.pn.data(), sizeof(double) * P.pn.size());
    if (end_state10) {
        end_state10[0] = P.cur_p.x, end_state10[1] = P.cur_p.y, end_state10[2] = P.cur_p.z;
        end_state10[3] = P.cur_q.x, end_state10[4] = P.cur_q.y, end_state10[5] = P.cur_q.z, end_state10[6] = P.cur_q.w;
        end_state10[7] = P.cur_v.x, end_state10[8] = P.cur_v.y, end_state10[9] = P.cur_v.z;
    }
    return (int) P.pn.size() / 4;
}

int icgo_reproj_eval(const double *pose0, const double *pose1, const double *ext, const double *invdepth, const double *td, const double *c,
                     double std_, double *r, double **J) {
    ReprojectionFactor f({c[0], c[1], c[2]}, {c[3], c[4], c[5]}, {c[6], c[7], c[8]}, {c[9], c[10], c[11]}, c[12], c[13], std_);
    const double *params[5] = {pose0, pose1, ext, invdepth, td};
    f.Evaluate(params, r, J);
    return 0;
}

int icgo_imu_eval(const double *blob, const double *pn, int npn, const double *pose0, const double *mix0, const double *pose1, const double *mix1,
                  double *r, double **J) {
    Preintegration P;
    blob_to_preint(blob, pn, npn, P);
    PreintegrationFactor f(&P);
    const double *params[4] = {pose0, mix0, pose1, mix1};
    f.Evaluate(params, r, J);
    return 0;
}

int icgo_gnss_eval(const double *pose, const double *blh, const double *std3, const double *lever, double *r, double *J) {
    GnssFactor f({blh[0], blh[1], blh[2]}, {std3[0], std3[1], std3[2]}, {lever[0], lever[1], lever[2]});
    const double *params[1] = {pose};
    double *Jp[1] = {J};
    f.Evaluate(params, r, J ? Jp : nullptr);
    return 0;
}

// The same factors with the loss the solver applies (huber = 0: none), through apply_loss: corrected residuals and global Jacobians, and
// the block's cost (evaluate_block's arithmetic)
int icgo_reproj_eval_loss(const double *pose0, const double *pose1, const double *ext, const double *invdepth, const double *td, const double *c,
                          double std_, int huber, double *r, double **J, double *cost) {
    icgo_reproj_eval(pose0, pose1, ext, invdepth, td, c, std_, r, J);
    const int gs[5] = {7, 7, 7, 1, 1};
    apply_loss(huber != 0, 2, r, 5, J, gs, *cost);
    return 0;
}

int icgo_gnss_eval_loss(const double *pose, const double *blh, const double *std3, const double *lever, int huber, double *r, double *J, double *cost) {
    icgo_gnss_eval(pose, blh, std3, lever, r, J);
    const int gs[1] = {7};
    double *Jp[1] = {J};
    apply_loss(huber != 0, 3, r, 1, J ? Jp : nullptr, gs, *cost);
    return 0;
}

int icgo_pose_prior_eval(const double *pose, const double *prior7, const double *std6, double *r, double *J) {
    ImuPosePriorFactor f;
    std::memcpy(f.pose, prior7, sizeof(double) * 7);
    for (int k = 0; k < 6; k++) f.sqrt_info[k] = 1.0 / std6[k];
    const double *params[1] = {pose};
    double *Jp[1] = {J};
    f.Evaluate(params, r, J ? Jp : nullptr);
    return 0;
}

// MarginalizationInfo::marginalization on the window held by `p` (num_marg oldest nodes + the landmarks anchored there).
// Outputs are sized by the caller for r <= 15*K+7: block list, x0, J0 (r x r row-major), e0, Hp, bp.  Returns r (0: nothing to do).
int icgo_ba_marginalize(const icg_ba_problem *p, const double *pn, const int32_t *pn_off, int num_marg, int32_t *m_out, int32_t *nblocks_out,
                        int32_t *block_type, int32_t *block_node, double *x0, double *J0, double *e0, double *Hp, double *bp) {
    WindowProblem W;
    to_window(p, pn, pn_off, W);
    MargOut M;
    marginalize(W, num_marg, M);
    if (m_out) *m_out = M.m;
    if (nblocks_out) *nblocks_out = (int32_t) M.block_type.size();
    for (size_t i = 0; i < M.block_type.size(); i++) block_type[i] = M.block_type[i], block_node[i] = M.block_node[i];
    std::memcpy(x0, M.x0.data(), sizeof(double) * M.x0.size());
    if (M.m > 0) {
        std::memcpy(J0, M.J0.data(), sizeof(double) * M.J0.size());
        std::memcpy(e0, M.e0.data(), sizeof(double) * M.e0.size());
        if (Hp) std::memcpy(Hp, M.Hp.data(), sizeof(double) * M.Hp.size());
        if (bp) std::memcpy(bp, M.bp.data(), sizeof(double) * M.bp.size());
    }
    return M.r;
}

// symmetric eigendecomposition used by the marginalization restatement (checked against numpy.linalg.eigh in the tests)
void icgo_sym_eig(const double *A, int n, double *evals, double *V) {
    std::vector<double> a(A, A + (size_t) n * n), e, v;
    sym_eig_jacobi(a, n, e, v);
    std::memcpy(evals, e.data(), sizeof(double) * n);
    std::memcpy(V, v.data(), sizeof(double) * (size_t) n * n);
}

void icgo_pose_plus(const double *x, const double *delta, double *out) { pose_plus(x, delta, out); }

}  // extern "C"
