// ba_cull.cu -- updateParametersFromOptimizer + gvinsOutlierCulling (IG/ic_gvins.cc:1299-1389, 1035-1128) for B windows: one CTA per window.
//   thread 0        : the extrinsic / td update with its 1 m / 5 deg gate (:1306-1347)
//   thread per node : frame->pose() = MISC::stateToCameraPose(state, pose_b_c) with the gated extrinsic (:1351-1360)
//   thread per landmark (landmarks in chunks of the CTA): pw and depth from the optimised inverse depth (:1364-1388), then the walk over the
//                   landmark's observations in list order on the same thread, so that the error sum keeps the reference's order (:1058-1113)
//   block reduction : the five counters of :1085-1124
// Built with -fmad=false: every product and sum below is the fixed-order, uncontracted sequence tests/post_solve_oracle.py restates.
#include <math.h>

#include "ba_cull.cuh"
#include "geom_core.cuh"

namespace icg {
namespace {

// Eigen::Quaterniond::toRotationMatrix (Eigen/src/Geometry/Quaternion.h) for q = (x, y, z, w), row-major
__device__ void quat_to_rot(double x, double y, double z, double w, double *R) {
    const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1.0 - (tyy + tzz), R[1] = txy - twz, R[2] = txz + twy;
    R[3] = txy + twz, R[4] = 1.0 - (txx + tzz), R[5] = tyz - twx;
    R[6] = txz - twy, R[7] = tyz + twx, R[8] = 1.0 - (txx + tyy);
}
// R(q / |q|), |q| = sqrt(x^2 + y^2 + z^2 + w^2) summed in that order (Quaterniond::normalized; Eigen's own reduction order is not pinned)
__device__ void unit_quat_to_rot(const double *q_xyzw, double *R) {
    const double x = q_xyzw[0], y = q_xyzw[1], z = q_xyzw[2], w = q_xyzw[3];
    const double n = sqrt(x * x + y * y + z * z + w * w);
    quat_to_rot(x / n, y / n, z / n, w / n, R);
}
// |Quaterniond(M).vec()| with Eigen's branch structure for the matrix -> quaternion conversion
__device__ double quat_vec_norm(const double *M) {
    double q[4];  // x, y, z, w
    double t = M[0] + M[4] + M[8];
    if (t > 0.0) {
        t = sqrt(t + 1.0);
        q[3] = 0.5 * t;
        t = 0.5 / t;
        q[0] = (M[7] - M[5]) * t, q[1] = (M[2] - M[6]) * t, q[2] = (M[3] - M[1]) * t;
    } else {
        int i = 0;
        if (M[4] > M[0]) i = 1;
        if (M[8] > M[4 * i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = sqrt(M[4 * i] - M[4 * j] - M[4 * k] + 1.0);
        q[i] = 0.5 * t;
        t = 0.5 / t;
        q[3] = (M[3 * k + j] - M[3 * j + k]) * t;
        q[j] = (M[3 * j + i] + M[3 * i + j]) * t;
        q[k] = (M[3 * k + i] + M[3 * i + k]) * t;
    }
    return sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
}

__global__ void __launch_bounds__(CULL_THREADS) ba_update_cull(CullArgs a) {
    __shared__ double s_pose[CULL_MAX_NODES][12];  // camera pose of every node: R row-major | t
    __shared__ double s_bc[12];                    // the gated extrinsic
    __shared__ int s_cnt[5];
    const int w = blockIdx.x, tid = threadIdx.x;
    const CullWin &W = a.win[w];
    CullOut &O = a.out[w];
    if (tid == 0) {
        const double *ext = a.ext + (size_t) w * 8;
        for (int i = 0; i < 9; i++) s_bc[i] = W.R_bc[i];
        for (int i = 0; i < 3; i++) s_bc[9 + i] = W.t_bc[i];
        int accepted = -1;
        if (W.estimate_ext) {
            double R[9], M[9];
            unit_quat_to_rot(ext + 3, R);
            const double d0 = ext[0] - W.t_bc[0], d1 = ext[1] - W.t_bc[1], d2 = ext[2] - W.t_bc[2];
            const double dt = sqrt(d0 * d0 + d1 * d1 + d2 * d2);
            for (int i = 0; i < 3; i++)  // R R_bc^T
                for (int j = 0; j < 3; j++) M[3 * i + j] = R[3 * i] * W.R_bc[3 * j] + R[3 * i + 1] * W.R_bc[3 * j + 1] + R[3 * i + 2] * W.R_bc[3 * j + 2];
            const double dr = quat_vec_norm(M) * (180.0 / M_PI);
            accepted = (dt > 1.0) || (dr > 5.0) ? 0 : 1;
            if (accepted) {
                for (int i = 0; i < 9; i++) s_bc[i] = R[i];
                for (int i = 0; i < 3; i++) s_bc[9 + i] = ext[i];
            }
        }
        for (int i = 0; i < 9; i++) O.R_bc[i] = s_bc[i];
        for (int i = 0; i < 3; i++) O.t_bc[i] = s_bc[9 + i];
        O.td_bc = W.estimate_td ? ext[7] : W.td_bc;
        O.ext_accepted = accepted;
        for (int i = 0; i < 5; i++) s_cnt[i] = 0;
    }
    __syncthreads();
    if (tid < W.K) {
        const double *p = a.pose + (size_t) w * a.pose_stride + 7 * tid;
        double Rq[9];
        unit_quat_to_rot(p + 3, Rq);
        double *P = s_pose[tid];
        for (int i = 0; i < 3; i++) {
            for (int j = 0; j < 3; j++) P[3 * i + j] = Rq[3 * i] * s_bc[j] + Rq[3 * i + 1] * s_bc[3 + j] + Rq[3 * i + 2] * s_bc[6 + j];
            P[9 + i] = p[i] + (Rq[3 * i] * s_bc[9] + Rq[3 * i + 1] * s_bc[10] + Rq[3 * i + 2] * s_bc[11]);
        }
        double *o = a.cam_pose + (size_t) (W.node0 + tid) * 12;
        for (int i = 0; i < 12; i++) o[i] = P[i];
    }
    __syncthreads();
    int cnt[5] = {0, 0, 0, 0, 0};
    const int *off = a.obs_off + W.off0;
    for (int l = tid; l < W.L; l += CULL_THREADS) {
        const int g = W.lm0 + l, ref = a.lm_ref_node[g];
        const double *P = s_pose[ref];
        double x, y;
        gc::pixel2cam(a.cam, a.lm_ref_kp[2 * g], a.lm_ref_kp[2 * g + 1], x, y);
        const double depth = 1.0 / a.rho[(size_t) w * a.rho_stride + l];
        const double c0 = x * depth, c1 = y * depth, c2 = 1.0 * depth;
        double pw[3];
        for (int i = 0; i < 3; i++) pw[i] = (P[3 * i] * c0 + P[3 * i + 1] * c1 + P[3 * i + 2] * c2) + P[9 + i];
        a.lm_pw[3 * (size_t) g] = pw[0], a.lm_pw[3 * (size_t) g + 1] = pw[1], a.lm_pw[3 * (size_t) g + 2] = pw[2];
        a.lm_depth[g] = depth;
        double sum = 0.0;
        int n_good = 0, reason = 0;
        const int ob = W.obs0 + off[l], oe = W.obs0 + off[l + 1];
        int o = ob;
        for (; o < oe; o++) {
            const int k = a.obs_node[o];
            double err = 0.0;
            if (gc::good_to_track_scaled(a.cam, a.obs_kp[2 * (size_t) o], a.obs_kp[2 * (size_t) o + 1], s_pose[k], s_pose[k] + 9, pw, a.std, 3.0, 1.0,
                                         err)) {
                a.obs_outlier[o] = 0;
                sum += err;
                n_good++;
            } else {
                a.obs_outlier[o] = 1;
                if (k == ref) {  // the reference observation: the landmark goes, the walk stops (:1085-1091)
                    reason |= 1, cnt[0]++, cnt[2]++;
                    o++;
                    break;
                }
                cnt[1]++;
            }
        }
        for (; o < oe; o++) a.obs_outlier[o] = 0;
        if (n_good < 2)
            reason |= 2, cnt[0]++, cnt[3]++;
        else if (sum / (double) n_good > a.std)
            reason |= 4, cnt[0]++, cnt[4]++;
        a.lm_outlier[g] = (uint8_t) reason;
    }
#pragma unroll
    for (int i = 0; i < 5; i++) {
        const int v = __reduce_add_sync(0xffffffffu, cnt[i]);
        if ((tid & 31) == 0 && v) atomicAdd(&s_cnt[i], v);  // integer sums: exact in any order
    }
    __syncthreads();
    if (tid < 5) O.counts[tid] = s_cnt[tid];
}

}  // namespace

cudaError_t preload_update_cull() {
    cudaFuncAttributes attr;
    return cudaFuncGetAttributes(&attr, ba_update_cull);
}

cudaError_t launch_update_cull(const CullArgs &a, int n_windows, cudaStream_t stream) {
    ba_update_cull<<<n_windows, CULL_THREADS, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace icg
