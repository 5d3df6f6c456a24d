// ba_math.cuh -- FP64 device/host algebra + the factor arithmetic of IC-GVINS' sliding-window graph.
// Every function cites the reference code it restates (IG/ = ic_gvins/ic_gvins/).  Written from the reference
// formulas for this library (it shares no code with oracle/).
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace icg {
namespace bam {

#define BAM_HD __host__ __device__ __forceinline__

struct V3 {
    double x, y, z;
};
BAM_HD V3 mk(double x, double y, double z) { return V3{x, y, z}; }
BAM_HD V3 operator+(V3 a, V3 b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
BAM_HD V3 operator-(V3 a, V3 b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
BAM_HD V3 operator-(V3 a) { return mk(-a.x, -a.y, -a.z); }
BAM_HD V3 operator*(double s, V3 a) { return mk(s * a.x, s * a.y, s * a.z); }
BAM_HD V3 operator*(V3 a, double s) { return mk(s * a.x, s * a.y, s * a.z); }
BAM_HD V3 operator/(V3 a, double s) { return mk(a.x / s, a.y / s, a.z / s); }
BAM_HD double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
BAM_HD V3 cross(V3 a, V3 b) { return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }

struct M3 {
    double m[9];
};
BAM_HD M3 ident() {
    M3 r;
    r.m[0] = 1, r.m[1] = 0, r.m[2] = 0, r.m[3] = 0, r.m[4] = 1, r.m[5] = 0, r.m[6] = 0, r.m[7] = 0, r.m[8] = 1;
    return r;
}
BAM_HD M3 mul(const M3 &a, const M3 &b) {
    M3 r;
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) r.m[3 * i + j] = a.m[3 * i] * b.m[j] + a.m[3 * i + 1] * b.m[3 + j] + a.m[3 * i + 2] * b.m[6 + j];
    return r;
}
BAM_HD V3 mul(const M3 &a, V3 v) {
    return mk(a.m[0] * v.x + a.m[1] * v.y + a.m[2] * v.z, a.m[3] * v.x + a.m[4] * v.y + a.m[5] * v.z, a.m[6] * v.x + a.m[7] * v.y + a.m[8] * v.z);
}
BAM_HD M3 scale(double s, const M3 &a) {
    M3 r;
#pragma unroll
    for (int i = 0; i < 9; i++) r.m[i] = s * a.m[i];
    return r;
}
BAM_HD M3 add(const M3 &a, const M3 &b) {
    M3 r;
#pragma unroll
    for (int i = 0; i < 9; i++) r.m[i] = a.m[i] + b.m[i];
    return r;
}
BAM_HD M3 sub(const M3 &a, const M3 &b) {
    M3 r;
#pragma unroll
    for (int i = 0; i < 9; i++) r.m[i] = a.m[i] - b.m[i];
    return r;
}
BAM_HD M3 neg(const M3 &a) { return scale(-1.0, a); }
BAM_HD M3 tr(const M3 &a) {
    M3 r;
    r.m[0] = a.m[0], r.m[1] = a.m[3], r.m[2] = a.m[6], r.m[3] = a.m[1], r.m[4] = a.m[4], r.m[5] = a.m[7], r.m[6] = a.m[2], r.m[7] = a.m[5], r.m[8] = a.m[8];
    return r;
}
// Rotation::skewSymmetric (IG/common/rotation.h:97-101)
BAM_HD M3 skew(V3 v) {
    M3 r;
    r.m[0] = 0, r.m[1] = -v.z, r.m[2] = v.y, r.m[3] = v.z, r.m[4] = 0, r.m[5] = -v.x, r.m[6] = -v.y, r.m[7] = v.x, r.m[8] = 0;
    return r;
}

struct Q {
    double w, x, y, z;
};  // Eigen::Quaterniond(w, x, y, z)
BAM_HD Q mkq(double w, double x, double y, double z) { return Q{w, x, y, z}; }
BAM_HD V3 qv(Q q) { return mk(q.x, q.y, q.z); }
BAM_HD Q qmul(Q a, Q b) {
    return mkq(a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
               a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x);
}
BAM_HD Q qinv(Q q) {  // Eigen inverse(): conjugate / squaredNorm
    double n2 = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
    return mkq(q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2);
}
BAM_HD Q qinv_r(Q q) {  // the same with ONE reciprocal (hot kernels: a quotient becomes a product with 1 / |q|^2, <= 1.5 ulp apart)
    const double i2 = 1.0 / (q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    return mkq(q.w * i2, -q.x * i2, -q.y * i2, -q.z * i2);
}
BAM_HD Q qnormalized(Q q) {
    double n = sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    return mkq(q.w / n, q.x / n, q.y / n, q.z / n);
}
BAM_HD M3 qmat(Q q) {  // Eigen toRotationMatrix()
    double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    M3 r;
    r.m[0] = 1 - (tyy + tzz), r.m[1] = txy - twz, r.m[2] = txz + twy;
    r.m[3] = txy + twz, r.m[4] = 1 - (txx + tzz), r.m[5] = tyz - twx;
    r.m[6] = txz - twy, r.m[7] = tyz + twx, r.m[8] = 1 - (txx + tyy);
    return r;
}
BAM_HD V3 qrot(Q q, V3 v) {  // Eigen q * v
    V3 uv = cross(qv(q), v);
    uv = uv + uv;
    return v + q.w * uv + cross(qv(q), uv);
}
// Rotation::rotvec2quaternion (IG/common/rotation.h:72-76)
BAM_HD Q rotvec2q(V3 rv) {
    double a = sqrt(dot(rv, rv));
    V3 ax = a > 0 ? rv / a : rv;
    double s = sin(0.5 * a), c = cos(0.5 * a);
    return mkq(c, s * ax.x, s * ax.y, s * ax.z);
}
// bottom-right 3x3 of Rotation::quaternionleft / quaternionright (IG/common/rotation.h:103-119)
BAM_HD M3 qleft_br(Q q) { return add(scale(q.w, ident()), skew(qv(q))); }
BAM_HD M3 qright_br(Q q) { return sub(scale(q.w, ident()), skew(qv(q))); }

BAM_HD V3 pose_p(const double *p) { return mk(p[0], p[1], p[2]); }
BAM_HD Q pose_q(const double *p) { return mkq(p[6], p[3], p[4], p[5]); }

// PoseParameterization::Plus (IG/factors/pose_parameterization.h:34-49)
BAM_HD void pose_plus(const double *x, const double *d, double *o) {
    Q r = qnormalized(qmul(pose_q(x), rotvec2q(mk(d[3], d[4], d[5]))));
    o[0] = x[0] + d[0], o[1] = x[1] + d[1], o[2] = x[2] + d[2];
    o[3] = r.x, o[4] = r.y, o[5] = r.z, o[6] = r.w;
}

// HuberLoss(1.0) + Corrector (Ceres loss_function.cc / corrector.cc; the reference's own copy IG/factors/residual_block_info.h:59-87).
// For Huber rho'' <= 0 always, so the correction reduces to scaling residuals and Jacobians by sqrt(rho').
BAM_HD void huber(double sq, double &cost, double &scale) {
    if (sq > 1.0) {
        double r = sqrt(sq);
        double rho1 = fmax(2.2250738585072014e-308, 1.0 / r);
        cost = 0.5 * (2.0 * r - 1.0);
        scale = sqrt(rho1);
    } else {
        cost = 0.5 * sq;
        scale = 1.0;
    }
}

// ReprojectionFactor::Evaluate (IG/factors/reprojection_factor.h:55-147).  c = pts0[3] pts1[3] vel0[3] vel1[3] td0 td1.
// Jacobians in LOCAL coordinates: Ji, Jj, Je are 2x6 row-major (the 7th global column is zero and dropped by
// PoseParameterization::ComputeJacobian), Jr, Jt are 2x1.  want_j = false computes residuals only.
BAM_HD void reproj_eval(const double *pi, const double *pj, const double *ext, double id0, double td, const double *c, double sinv, bool want_j,
                        double *r, double *Ji, double *Jj, double *Je, double *Jr, double *Jt) {
    V3 p0 = pose_p(pi), p1 = pose_p(pj), tic = pose_p(ext);
    Q q0 = pose_q(pi), q1 = pose_q(pj), qic = pose_q(ext);
    V3 pts0 = mk(c[0], c[1], c[2]), pts1 = mk(c[3], c[4], c[5]), vel0 = mk(c[6], c[7], c[8]), vel1 = mk(c[9], c[10], c[11]);
    // FP64 division is ~20 instructions on this part and the reference's form has 15 of them per factor (x / depth, the Eigen inverse() of two
    // quaternions = conjugate / squaredNorm per component, two projections, the reduce matrix): one reciprocal per distinct divisor instead
    // (4 divisions); each quotient differs from the divided form by at most 1.5 ulp, inside the per-entry first-order rounding bound that
    // tests/test_factor_edges_gpu.py holds this function to.
    V3 pts_0_td = pts0 - (td - c[12]) * vel0;
    V3 pts_1_td = pts1 - (td - c[13]) * vel1;
    const double inv_id0 = 1.0 / id0;
    V3 pts_c_0 = inv_id0 * pts_0_td;
    V3 pts_b_0 = qrot(qic, pts_c_0) + tic;
    V3 pts_n = qrot(q0, pts_b_0) + p0;
    V3 pts_b_1 = qrot(qinv_r(q1), pts_n - p1);
    V3 pts_1 = qrot(qinv_r(qic), pts_b_1 - tic);
    const double d1 = pts_1.z, inv_d = 1.0 / d1;
    r[0] = sinv * (pts_1.x * inv_d - pts_1_td.x);
    r[1] = sinv * (pts_1.y * inv_d - pts_1_td.y);
    if (!want_j) return;
    // Jacobians (reprojection_factor.h:84-144), evaluated row by row instead of as 3x3 matrix products: with r = a row of the 2x3
    // reduce matrix and R0 = R(q0), R1 = R(q1), Ric = R(q_ic) (so cb0n = R0, cnb1 = R1^T, cbc = Ric^T) every Jacobian row is a chain
    // of matrix-VECTOR products   a1 = r^T cbc = Ric r,  a2 = a1^T cnb1 = R1 a1,  a3 = a2^T cb0n = R0^T a2,  a4 = a3^T cbc^T = Ric^T a3
    // and cross products (a^T [p]x = (a x p)^T).  Same algebra as the reference's matrix form, ~3x fewer flops and far fewer live
    // registers; the sum of the two skew terms of the extrinsic-rotation block is [tmp_r pts_c_0 + lever]x = [pts_1]x.
    const M3 R0 = qmat(q0), R1 = qmat(q1), Ric = qmat(qic);
    const double redr[2][3] = {{sinv * inv_d, 0.0, sinv * (-pts_1.x * (inv_d * inv_d))}, {0.0, sinv * inv_d, sinv * (-pts_1.y * (inv_d * inv_d))}};
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {
        const V3 r3 = mk(redr[rr][0], redr[rr][1], redr[rr][2]);
        const V3 a1 = mul(Ric, r3);
        const V3 a2 = mul(R1, a1);
        const V3 a3 = mul(tr(R0), a2);
        const V3 a4 = mul(tr(Ric), a3);
        const V3 ji_rot = cross(pts_b_0, a3);  // -(a3 x pts_b_0)
        const V3 jj_rot = cross(a1, pts_b_1);
        const V3 je_pos = a3 - a1;
        const V3 je_rot = cross(pts_c_0, a4) + cross(r3, pts_1);  // -(a4 x pts_c_0) + (r x pts_1)
        double *ji = Ji + 6 * rr, *jj = Jj + 6 * rr, *je = Je + 6 * rr;
        ji[0] = a2.x, ji[1] = a2.y, ji[2] = a2.z, ji[3] = ji_rot.x, ji[4] = ji_rot.y, ji[5] = ji_rot.z;
        jj[0] = -a2.x, jj[1] = -a2.y, jj[2] = -a2.z, jj[3] = jj_rot.x, jj[4] = jj_rot.y, jj[5] = jj_rot.z;
        je[0] = je_pos.x, je[1] = je_pos.y, je[2] = je_pos.z, je[3] = je_rot.x, je[4] = je_rot.y, je[5] = je_rot.z;
        Jr[rr] = -dot(a4, pts_0_td) * (inv_id0 * inv_id0);
        Jt[rr] = -dot(a4, vel0) * inv_id0 + sinv * (rr == 0 ? vel1.x : vel1.y);
    }
}

// The same factor over pre-computed NODE FRAMES (hot kernels: ba_lin_vis, ba_cost).  Every factor of a window rotates with the matrices of
// its reference node, its observing node and the extrinsic -- K + 1 distinct rotations per window against ~2700 factors -- so the CTA
// builds them once (node_frame: R = toRotationMatrix(q) row-major | p) and the factor does matrix-vector products: four of them replace the
// reference's quaternion sandwich products and the two quaternion inverses, and the Jacobian rows use the same matrices.  For the unit
// quaternions PoseParameterization::Plus maintains, q v q^-1 = R(q) v and q^-1 v q = R(q)^T v up to rounding (tests/test_factor_edges_gpu.py
// holds this form, through icg_ba_reproj_evaluate_frames, to a high-precision restatement of the reference's quaternion form entry by entry
// at a first-order rounding bound, with quaternions up to 4 ulp per component off the unit sphere).  About 40 % fewer FP64 instructions per
// factor than reproj_eval.
constexpr int NODE_FRAME_LD = 13;  // 9 + 3, padded to an odd length (shared-memory banks)
BAM_HD void node_frame(const double *pose7, double *F) {
    const M3 R = qmat(pose_q(pose7));
#pragma unroll
    for (int i = 0; i < 9; i++) F[i] = R.m[i];
    F[9] = pose7[0], F[10] = pose7[1], F[11] = pose7[2];
}
BAM_HD V3 mulT(const M3 &a, V3 v) {  // a^T v
    return mk(a.m[0] * v.x + a.m[3] * v.y + a.m[6] * v.z, a.m[1] * v.x + a.m[4] * v.y + a.m[7] * v.z, a.m[2] * v.x + a.m[5] * v.y + a.m[8] * v.z);
}
BAM_HD void reproj_eval_frames(const double *Fi, const double *Fj, const double *Fe, double id0, double td, const double *c, double sinv, bool want_j,
                               double *r, double *Ji, double *Jj, double *Je, double *Jr, double *Jt) {
    M3 R0, R1, Ric;
#pragma unroll
    for (int i = 0; i < 9; i++) R0.m[i] = Fi[i], R1.m[i] = Fj[i], Ric.m[i] = Fe[i];
    const V3 p0 = mk(Fi[9], Fi[10], Fi[11]), p1 = mk(Fj[9], Fj[10], Fj[11]), tic = mk(Fe[9], Fe[10], Fe[11]);
    V3 pts0 = mk(c[0], c[1], c[2]), pts1 = mk(c[3], c[4], c[5]), vel0 = mk(c[6], c[7], c[8]), vel1 = mk(c[9], c[10], c[11]);
    V3 pts_0_td = pts0 - (td - c[12]) * vel0;
    V3 pts_1_td = pts1 - (td - c[13]) * vel1;
    const double inv_id0 = 1.0 / id0;
    V3 pts_c_0 = inv_id0 * pts_0_td;
    V3 pts_b_0 = mul(Ric, pts_c_0) + tic;
    V3 pts_n = mul(R0, pts_b_0) + p0;
    V3 pts_b_1 = mulT(R1, pts_n - p1);
    V3 pts_1 = mulT(Ric, pts_b_1 - tic);
    const double d1 = pts_1.z, inv_d = 1.0 / d1;
    r[0] = sinv * (pts_1.x * inv_d - pts_1_td.x);
    r[1] = sinv * (pts_1.y * inv_d - pts_1_td.y);
    if (!want_j) return;
    const double redr[2][3] = {{sinv * inv_d, 0.0, sinv * (-pts_1.x * (inv_d * inv_d))}, {0.0, sinv * inv_d, sinv * (-pts_1.y * (inv_d * inv_d))}};
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {  // same row-by-row chain as reproj_eval
        const V3 r3 = mk(redr[rr][0], redr[rr][1], redr[rr][2]);
        const V3 a1 = mul(Ric, r3);
        const V3 a2 = mul(R1, a1);
        const V3 a3 = mulT(R0, a2);
        const V3 a4 = mulT(Ric, a3);
        const V3 ji_rot = cross(pts_b_0, a3);
        const V3 jj_rot = cross(a1, pts_b_1);
        const V3 je_pos = a3 - a1;
        const V3 je_rot = cross(pts_c_0, a4) + cross(r3, pts_1);
        double *ji = Ji + 6 * rr, *jj = Jj + 6 * rr, *je = Je + 6 * rr;
        ji[0] = a2.x, ji[1] = a2.y, ji[2] = a2.z, ji[3] = ji_rot.x, ji[4] = ji_rot.y, ji[5] = ji_rot.z;
        jj[0] = -a2.x, jj[1] = -a2.y, jj[2] = -a2.z, jj[3] = jj_rot.x, jj[4] = jj_rot.y, jj[5] = jj_rot.z;
        je[0] = je_pos.x, je[1] = je_pos.y, je[2] = je_pos.z, je[3] = je_rot.x, je[4] = je_rot.y, je[5] = je_rot.z;
        Jr[rr] = -dot(a4, pts_0_td) * (inv_id0 * inv_id0);
        Jt[rr] = -dot(a4, vel0) * inv_id0 + sinv * (rr == 0 ? vel1.x : vel1.y);
    }
}

// GnssFactor::Evaluate (IG/factors/gnss_factor.h:43-71); J local 3x6 row-major
BAM_HD void gnss_eval(const double *pose, const double *blh, const double *std3, const double *lever, bool want_j, double *r, double *J) {
    V3 p = pose_p(pose);
    M3 R = qmat(pose_q(pose));
    V3 lv = mk(lever[0], lever[1], lever[2]);
    V3 e = p + mul(R, lv) - mk(blh[0], blh[1], blh[2]);
    double si[3] = {1.0 / std3[0], 1.0 / std3[1], 1.0 / std3[2]};
    r[0] = si[0] * e.x, r[1] = si[1] * e.y, r[2] = si[2] * e.z;
    if (!want_j) return;
    M3 b = neg(mul(R, skew(lv)));
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            J[i * 6 + j] = (i == j) ? si[i] : 0.0;
            J[i * 6 + 3 + j] = si[i] * b.m[3 * i + j];
        }
}

// ImuPosePriorFactor::Evaluate (IG/preintegration/imu_pose_prior_factor.h:42-68); sinfo = 1/std; J local 6x6
BAM_HD void pose_prior_eval(const double *pose, const double *prior, const double *sinfo, bool want_j, double *r, double *J) {
    for (int k = 0; k < 3; k++) r[k] = sinfo[k] * (pose[k] - prior[k]);
    Q dq = qmul(qinv(pose_q(pose)), pose_q(prior));
    V3 a = 2.0 * qv(dq);
    r[3] = sinfo[3] * a.x, r[4] = sinfo[4] * a.y, r[5] = sinfo[5] * a.z;
    if (!want_j) return;
    M3 b = neg(qright_br(dq));
    for (int i = 0; i < 36; i++) J[i] = 0;
    for (int i = 0; i < 3; i++) {
        J[i * 6 + i] = sinfo[i];
        for (int j = 0; j < 3; j++) J[(3 + i) * 6 + 3 + j] = sinfo[3 + i] * b.m[3 * i + j];
    }
}

// IMU blob layout (include/icgvins_b200.h)
constexpr int IB_DT = 0, IB_DP = 1, IB_DV = 4, IB_DQ = 7, IB_BG = 11, IB_BA = 14, IB_G = 17, IB_IEWN = 20, IB_S0 = 23, IB_S1 = 24, IB_JAC = 27,
              IB_COV = 252, IB_MODE = 477;  // mode 0: PreintegrationEarth, 1: PreintegrationNormal

// PreintegrationEarth::evaluate (IG/preintegration/preintegration_earth.cc:37-90): UNWHITENED residual (15) and the
// intermediates the Jacobian methods read (dpn, dvn, qb0b1, corrected_q: `:61-72`).
struct ImuMid {
    V3 dpn, dvn;
    Q qb0b1, corrected_q;
    M3 cnb0;
};
// mode_slot: where the mode word sits in `b` (IB_MODE in a full blob; callers that stage only the head of the blob pass their own slot)
BAM_HD void imu_residual_raw(const double *b, const double *pose0, const double *mix0, const double *pose1, const double *mix1, double *r, ImuMid &M,
                             int mode_slot = IB_MODE) {
    V3 p0 = pose_p(pose0), p1 = pose_p(pose1);
    Q q0 = pose_q(pose0), q1 = pose_q(pose1);
    V3 v0 = mk(mix0[0], mix0[1], mix0[2]), bg0 = mk(mix0[3], mix0[4], mix0[5]), ba0 = mk(mix0[6], mix0[7], mix0[8]);
    V3 v1 = mk(mix1[0], mix1[1], mix1[2]), bg1 = mk(mix1[3], mix1[4], mix1[5]), ba1 = mk(mix1[6], mix1[7], mix1[8]);
    const double *Jc = b + IB_JAC;
    auto blk = [&](int r0, int c0) {
        M3 m;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) m.m[3 * i + j] = Jc[(r0 + i) * 15 + c0 + j];
        return m;
    };
    M3 dp_dbg = blk(0, 9), dp_dba = blk(0, 12), dv_dbg = blk(3, 9), dv_dba = blk(3, 12), dq_dbg = blk(6, 9);
    V3 dbg = bg0 - mk(b[IB_BG], b[IB_BG + 1], b[IB_BG + 2]);
    V3 dba = ba0 - mk(b[IB_BA], b[IB_BA + 1], b[IB_BA + 2]);
    V3 iewn = mk(b[IB_IEWN], b[IB_IEWN + 1], b[IB_IEWN + 2]), grav = mk(b[IB_G], b[IB_G + 1], b[IB_G + 2]);
    M3 isk = skew(iewn);
    double dt = b[IB_DT];
    // p_cor = 2 iewn_skew sum_i (pn_i - p0) dt_i = 2 iewn_skew (S1 - p0 S0)   (:55-59, algebraically regrouped)
    V3 p_cor = 2.0 * mul(isk, mk(b[IB_S1], b[IB_S1 + 1], b[IB_S1 + 2]) - b[IB_S0] * p0);
    V3 v_cor = 2.0 * mul(isk, p1 - p0);
    Q qnn = rotvec2q(-(dt * iewn));
    M.dpn = p1 - p0 - dt * v0 - (0.5 * dt * dt) * grav + p_cor;
    M.dvn = v1 - v0 - dt * grav + v_cor;
    V3 corrected_p = mk(b[IB_DP], b[IB_DP + 1], b[IB_DP + 2]) + mul(dp_dba, dba) + mul(dp_dbg, dbg);
    V3 corrected_v = mk(b[IB_DV], b[IB_DV + 1], b[IB_DV + 2]) + mul(dv_dba, dba) + mul(dv_dbg, dbg);
    Q dq = mkq(b[IB_DQ + 3], b[IB_DQ], b[IB_DQ + 1], b[IB_DQ + 2]);
    M.corrected_q = qmul(dq, rotvec2q(mul(dq_dbg, dbg)));
    M.cnb0 = qmat(qinv(q0));
    M.qb0b1 = qmul(qmul(qinv(q1), qnn), q0);
    V3 rp = mul(M.cnb0, M.dpn) - corrected_p, rv = mul(M.cnb0, M.dvn) - corrected_v, rq = 2.0 * qv(qmul(M.qb0b1, M.corrected_q));
    if (b[mode_slot] != 0.0) {
        // PreintegrationNormal::evaluate (IG/preintegration/preintegration_normal.cc:38-75): iewn = 0 in the blob, so dpn / dvn / cnb0 above
        // are already its terms; the attitude residual is 2 (corrected_q^-1 q0^-1 q1).vec().  M.qb0b1 carries q1^-1 q0 for the Jacobians.
        rq = 2.0 * qv(qmul(qmul(qinv(M.corrected_q), qinv(q0)), q1));
    }
    V3 rbg = bg1 - bg0, rba = ba1 - ba0;
    r[0] = rp.x, r[1] = rp.y, r[2] = rp.z, r[3] = rv.x, r[4] = rv.y, r[5] = rv.z, r[6] = rq.x, r[7] = rq.y, r[8] = rq.z;
    r[9] = rbg.x, r[10] = rbg.y, r[11] = rbg.z, r[12] = rba.x, r[13] = rba.y, r[14] = rba.z;
}

// Unwhitened IMU Jacobian in LOCAL coordinates, 15 x 30 row-major, columns [pose0 6 | mix0 9 | pose1 6 | mix1 9]
// (residualJacobianPose0/Mix0/Pose1/Mix1, IG/preintegration/preintegration_earth.cc:92-164).
BAM_HD void imu_jacobian_raw(const double *b, const ImuMid &M, double *J /* 450, zero-initialised by the caller */, int mode_slot = IB_MODE) {
    const double *Jc = b + IB_JAC;
    auto blk = [&](int r0, int c0) {
        M3 m;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) m.m[3 * i + j] = Jc[(r0 + i) * 15 + c0 + j];
        return m;
    };
    auto put = [&](int r0, int c0, const M3 &m) {
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) J[(r0 + i) * 30 + c0 + j] = m.m[3 * i + j];
    };
    M3 dp_dbg = blk(0, 9), dp_dba = blk(0, 12), dv_dbg = blk(3, 9), dv_dba = blk(3, 12), dq_dbg = blk(6, 9);
    V3 iewn = mk(b[IB_IEWN], b[IB_IEWN + 1], b[IB_IEWN + 2]);
    M3 isk = skew(iewn);
    double dt = b[IB_DT];
    Q dq = mkq(b[IB_DQ + 3], b[IB_DQ], b[IB_DQ + 1], b[IB_DQ + 2]);
    M3 cnb0_isk = mul(M.cnb0, isk);
    // pose0 (:92-111)
    put(0, 0, sub(neg(M.cnb0), scale(2.0 * dt, cnb0_isk)));
    put(0, 3, skew(mul(M.cnb0, M.dpn)));
    put(3, 0, scale(-2.0, cnb0_isk));
    put(3, 3, skew(mul(M.cnb0, M.dvn)));
    {
        // (quaternionleft(qb0b1) * quaternionright(corrected_q)).bottomRightCorner<3,3>() = -a b^T + L_br(a) R_br(b)
        V3 a = qv(M.qb0b1), bb = qv(M.corrected_q);
        M3 lr = mul(qleft_br(M.qb0b1), qright_br(M.corrected_q));
        double av[3] = {a.x, a.y, a.z}, bv[3] = {bb.x, bb.y, bb.z};
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) J[(6 + i) * 30 + 3 + j] = -av[i] * bv[j] + lr.m[3 * i + j];
    }
    // mix0 (:127-154) at column offset 6
    put(0, 6, scale(-dt, M.cnb0));
    put(0, 9, neg(dp_dbg));
    put(0, 12, neg(dp_dba));
    put(3, 6, neg(M.cnb0));
    put(3, 9, neg(dv_dbg));
    put(3, 12, neg(dv_dba));
    put(6, 9, mul(qleft_br(qmul(M.qb0b1, dq)), dq_dbg));
    put(9, 9, neg(ident()));
    put(12, 12, neg(ident()));
    // pose1 (:113-125) at column offset 15
    put(0, 15, M.cnb0);
    put(3, 15, scale(2.0, cnb0_isk));
    put(6, 18, neg(qright_br(qmul(M.qb0b1, M.corrected_q))));
    // mix1 (:156-168) at column offset 21
    put(3, 21, M.cnb0);
    put(9, 24, ident());
    put(12, 27, ident());
    if (b[mode_slot] != 0.0) {
        // PreintegrationNormal::residualJacobianPose0/Pose1/Mix0 (preintegration_normal.cc:77-140): only the attitude rows differ from the
        // Earth form evaluated with iewn = 0 (M.qb0b1 = q1^-1 q0):
        //   pose0 (6,3) = -(quaternionleft(q1^-1 q0) quaternionright(corrected_q)).bottomRight
        //   pose1 (6,3) =  quaternionleft(corrected_q^-1 q0^-1 q1).bottomRight
        //   mix0  (6,3) = -quaternionleft(q1^-1 q0 dq).bottomRight dq_dbg
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) J[(6 + i) * 30 + 3 + j] = -J[(6 + i) * 30 + 3 + j];
        put(6, 18, qleft_br(qmul(qinv(M.corrected_q), qinv(M.qb0b1))));
        put(6, 9, neg(mul(qleft_br(qmul(M.qb0b1, dq)), dq_dbg)));
    }
}

}  // namespace bam
}  // namespace icg
