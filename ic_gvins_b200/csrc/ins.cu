// ins.cu -- device INS windows for B streams: runFusion's per-sample mechanization (IG/ic_gvins.cc:249-293), the post-solve redo
// (MISC::redoInsMechanization, IG/misc.cc:208-261) and each frame's prior camera pose (MISC::getCameraPoseFromInsWindow, misc.cc:67-108).
// GVINS::gvinsInitialization (IG/ic_gvins.cc:584-692) starts a stream from its window: the kernel below up to the redo, preint.cu for the
// first GNSS node's factor.
//
// Layout: stream s owns rows imu[s][capacity][8] (time, dt, dtheta[3], dvel[3]) and states st[s][capacity][17] (time, p, q_xyzw, v, bg, ba),
// a ring whose head and count live in the host mirror and reach the kernels through the per-call job table.
//
// Kernel shape (push and redo): one warp per stream.  The lanes form the state-independent part of 32 samples at a time -- bias compensation,
// dvfb, dtheta, rotvec2q(dtheta) and qnn, which depends on dt only (gc::ins_increments) -- and lane 0 then runs the dependent q / v / p chain
// (gc::ins_mechanize_step).  The biases are constant along a window (insMechanization never changes them), so each precomputed value is the
// number the sequential code forms, whichever lane made it.  Built with -fmad=false: the operation order of geom_core.cuh, IEEE double; only
// sin / cos / sqrt / atan2 may differ from a host libm in the last ulp.
#include <string.h>

#include <vector>

#include "common.cuh"
#include "geom_core.cuh"
#include "ins_handle.cuh"
#include "preint.cuh"

using namespace icg;
using namespace icg::bam;

namespace {

constexpr int INS_ROW = 8, INS_ST = 17;
constexpr int INS_INIT_KEEP = 1000;    // MAXIMUM_INS_NUMBER (IG/ic_gvins.h:124)
constexpr int INS_MAX_CAPACITY = 65536;
constexpr double INS_MIN_DT = 0.0001;  // MISC::MINIMUM_TIME_INTERVAL (IG/misc.h:72)
constexpr int INS_WARPS = 4;           // streams per CTA

struct InsJob {                // one stream of one call
    double grav[3], iewn[3];
    int32_t head, count, n;    // ring head and size before the call; rows pushed
    int32_t off, skip;         // first row of the stream in the call's rows; leading rows the initialization path drops unwritten
    int32_t mech, earth, sel;  // mechanized; Earth form; selected (redo)
};

__device__ __forceinline__ int ring(const InsJob &J, int cap, int i) { return (J.head + i) % cap; }

// MISC::getInsWindowIndex (misc.cc:30-65): the first entry whose row time is greater than t; 0 when t is before the front, at or after the
// back, or (never, for capacity <= 65536) when the search runs past its cap
__device__ int window_index(const double *I, const InsJob &J, int cap, double t) {
    if (J.count == 0 || I[INS_ROW * ring(J, cap, 0)] > t || I[INS_ROW * ring(J, cap, J.count - 1)] <= t) return 0;
    int index = 0, sta = 0, end = J.count, counts = 0;
    while (true) {
        const int mid = (sta + end) / 2;
        const double first = I[INS_ROW * ring(J, cap, mid - 1)], second = I[INS_ROW * ring(J, cap, mid)];
        if (first <= t && t < second) {
            index = mid;
            break;
        } else if (first > t) {
            end = mid;
        } else if (second <= t) {
            sta = mid;
        }
        if (counts++ > 15) break;
    }
    return index;
}

__device__ __forceinline__ void put_state(double *x, double time, V3 p, Q q, V3 v, V3 bg, V3 ba) {
    x[0] = time, x[1] = p.x, x[2] = p.y, x[3] = p.z, x[4] = q.x, x[5] = q.y, x[6] = q.z, x[7] = q.w, x[8] = v.x, x[9] = v.y, x[10] = v.z;
    x[11] = bg.x, x[12] = bg.y, x[13] = bg.z, x[14] = ba.x, x[15] = ba.y, x[16] = ba.z;
}

// Mechanize entries first .. count-1 of a window from (p, q, v), which lane 0 holds: the row before entry first is `carry` (a row in
// (dt, dtheta, dvel) form), every later one the window's previous row.  Each state is stored with its row's time.
__device__ void mechanize_run(double (*sh)[12], const InsJob &J, int cap, const double *I, double *X, int first, const double *carry, V3 bg,
                              V3 ba, V3 &p, Q &q, V3 &v) {
    const int lane = threadIdx.x & 31;
    const V3 grav = mk(J.grav[0], J.grav[1], J.grav[2]), iewn = mk(J.iewn[0], J.iewn[1], J.iewn[2]);
    for (int base = first; base < J.count; base += 32) {
        const int k = base + lane;
        if (k < J.count) {
            const double *cu = I + INS_ROW * ring(J, cap, k) + 1;
            const double *pr = k == first ? carry : I + INS_ROW * ring(J, cap, k - 1) + 1;
            V3 cth, cvl, dvfb, dtheta;
            gc::ins_increments(pr, cu, bg, ba, cth, cvl, dvfb, dtheta);
            const double dt = cu[0];
            const Q qth = rotvec2q(dtheta), qnn = J.earth ? rotvec2q(-(dt * iewn)) : mkq(1, 0, 0, 0);
            double *o = sh[lane];
            o[0] = dvfb.x, o[1] = dvfb.y, o[2] = dvfb.z, o[3] = qth.w, o[4] = qth.x, o[5] = qth.y, o[6] = qth.z;
            o[7] = qnn.w, o[8] = qnn.x, o[9] = qnn.y, o[10] = qnn.z, o[11] = dt;
        }
        __syncwarp();
        if (lane == 0) {
            const int m = min(32, J.count - base);
            for (int j = 0; j < m; j++) {
                const double *o = sh[j];
                gc::ins_mechanize_step(p, q, v, mk(o[0], o[1], o[2]), mkq(o[3], o[4], o[5], o[6]), mkq(o[7], o[8], o[9], o[10]), o[11], grav, iewn,
                                       J.earth != 0);
                const int slot = ring(J, cap, base + j);
                put_state(X + INS_ST * slot, I[INS_ROW * slot], p, q, v, bg, ba);
            }
        }
        __syncwarp();
    }
}

// runFusion's IMU step for one stream per warp.  J.count is the size AFTER the push (the host adds the rows); the new rows are entries
// J.count - (n - skip) ..  J.count - 1.
__global__ void __launch_bounds__(32 * INS_WARPS) ins_push_kernel(int n_streams, int cap, const InsJob *jobs, const double *rows, double *imu,
                                                                 double *st) {
    __shared__ double sh[INS_WARPS][32][12];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, s = blockIdx.x * INS_WARPS + w;
    if (s >= n_streams) return;
    const InsJob J = jobs[s];
    const int n_new = J.n - J.skip;
    if (n_new == 0) return;
    double *I = imu + (size_t) s * cap * INS_ROW, *X = st + (size_t) s * cap * INS_ST;
    const double *R = rows + (size_t) (J.off + J.skip) * INS_ROW;
    const int e0 = J.count - n_new;
    for (int k = lane; k < n_new; k += 32) {
        const int slot = ring(J, cap, e0 + k);
        for (int c = 0; c < INS_ROW; c++) I[INS_ROW * slot + c] = R[INS_ROW * k + c];
        if (!J.mech)
            for (int c = 0; c < INS_ST; c++) X[INS_ST * slot + c] = 0.0;
    }
    if (!J.mech) return;
    __syncwarp();
    // a mechanized window is never empty (its first redo left at least one entry), so entry e0 - 1 holds the last state and imu_pre
    const double *last = X + INS_ST * ring(J, cap, e0 - 1);
    const V3 bg = mk(last[11], last[12], last[13]), ba = mk(last[14], last[15], last[16]);
    V3 p = mk(last[1], last[2], last[3]), v = mk(last[8], last[9], last[10]);
    Q q = mkq(last[7], last[4], last[5], last[6]);
    mechanize_run(sh[w], J, cap, I, X, e0, I + INS_ROW * ring(J, cap, e0 - 1) + 1, bg, ba, p, q, v);
}

// MISC::isNeedInterpolation (misc.cc:263-286) of time t between rows imu0 and imu1
__device__ __forceinline__ int need_interpolation(const double *imu0, const double *imu1, double t) {
    if (imu0[0] < t && imu1[0] > t) return t - imu0[0] < INS_MIN_DT ? -1 : imu1[0] - t < INS_MIN_DT ? 1 : 2;
    return 0;
}

// MISC::imuInterpolation(row, first, second, t) (misc.cc:288-305): row split at t into first (up to t) and second (from t); second may not
// alias row
__device__ __forceinline__ void imu_interpolation(const double *row, double t, double *first, double *second) {
    const double scale = (row[0] - t) / row[1];
    first[0] = t, first[1] = row[1] - (row[0] - t);
    for (int k = 2; k < INS_ROW; k++) first[k] = row[k] * (1 - scale);
    second[0] = row[0], second[1] = row[0] - t;
    for (int k = 2; k < INS_ROW; k++) second[k] = row[k] * scale;
}

// redoInsMechanization of one window by one warp from u (state17); returns getInsWindowIndex (0: nothing written).  carry: 8 doubles of
// shared memory.
__device__ int redo_window(double (*sh)[12], double *carry, const InsJob &J, int cap, double *I, double *X, const double *u) {
    const int lane = threadIdx.x & 31;
    const double t = u[0];
    int index = 0;
    if (lane == 0) index = window_index(I, J, cap, t);
    index = __shfl_sync(0xffffffffu, index, 0);
    if (index == 0) return 0;
    // stateFromData (preintegration_base.cc:115-125)
    V3 p = mk(u[1], u[2], u[3]), v = mk(u[8], u[9], u[10]);
    Q q = qnormalized(mkq(u[7], u[4], u[5], u[6]));
    const V3 bg = mk(u[11], u[12], u[13]), ba = mk(u[14], u[15], u[16]);
    if (lane == 0) {
        const int s1 = ring(J, cap, index);
        const double *imu0 = I + INS_ROW * ring(J, cap, index - 1), *imu1 = I + INS_ROW * s1;
        double *c = carry;
        for (int k = 0; k < INS_ROW; k++) c[k] = imu1[k];
        const int isneed = need_interpolation(imu0, imu1, t);
        const V3 grav = mk(J.grav[0], J.grav[1], J.grav[2]), iewn = mk(J.iewn[0], J.iewn[1], J.iewn[2]);
        double a[INS_ROW];
        const double *pre = imu0;
        if (isneed == 2) {  // imuInterpolation(imu1, imu0, imu1, t): imu0 := the first part, imu1 := the second
            imu_interpolation(imu1, t, a, c);
            pre = a;
        }
        if (isneed == -1 || isneed == 2) {
            V3 cth, cvl, dvfb, dtheta;
            gc::ins_increments(pre + 1, c + 1, bg, ba, cth, cvl, dvfb, dtheta);
            gc::ins_mechanize_step(p, q, v, dvfb, rotvec2q(dtheta), J.earth ? rotvec2q(-(c[1] * iewn)) : mkq(1, 0, 0, 0), c[1], grav, iewn,
                                   J.earth != 0);
            put_state(X + INS_ST * s1, c[0], p, q, v, bg, ba);
        } else if (isneed == 1) {
            put_state(X + INS_ST * s1, imu1[0], p, q, v, bg, ba);
        }
        // isneed == 0: the state time equals row index - 1's; nothing is stored at index and the loop integrates on from it (:245-251)
    }
    __syncwarp();
    mechanize_run(sh, J, cap, I, X, index + 1, carry + 1, bg, ba, p, q, v);
    return index;
}

// redoInsMechanization for one stream per warp; out[2 s] = status (1 / -1), out[2 s + 1] = index
__global__ void __launch_bounds__(32 * INS_WARPS) ins_redo_kernel(int n_streams, int cap, const InsJob *jobs, const double *state17, double *imu,
                                                                 double *st, int32_t *out) {
    __shared__ double sh[INS_WARPS][32][12];
    __shared__ double carry[INS_WARPS][8];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, s = blockIdx.x * INS_WARPS + w;
    if (s >= n_streams) return;
    const InsJob J = jobs[s];
    if (!J.sel) return;
    double *I = imu + (size_t) s * cap * INS_ROW, *X = st + (size_t) s * cap * INS_ST;
    const int index = redo_window(sh[w], carry[w], J, cap, I, X, state17 + (size_t) INS_ST * s);
    if (lane == 0) out[2 * s] = index == 0 ? -1 : 1, out[2 * s + 1] = index;
}

// ---- gvinsInitialization (IG/ic_gvins.cc:584-692), one stream per warp
constexpr int INS_SERIES_MAX = INS_INIT_KEEP + 2;  // getImuSeriesFromTo over an unmechanized window: at most its rows + 2
constexpr double ZV_GYR = 0.002, ZV_ACC = 0.1;     // MISC::ZERO_VELOCITY_GYR / ACC_THRESHOLD (IG/misc.h:75-76)
constexpr double MIN_ALIGN_VELOCITY = 0.5;         // GVINS::MINMUM_ALIGN_VELOCITY (IG/ic_gvins.h:128)

struct GinsOut {  // device outputs of one call, per stream
    int32_t *status, *n_series, *zv, *index;
    double *slot6;    // bg[3], initatt[3]
    double *state17;  // statedatalist_[0]
    double *iewn;     // Earth::iewn(origin, p)
};

__device__ __forceinline__ void series_row(double *dst, const double *row8) {  // (time, dt, ..) -> the preintegration's (dt, ..)
    for (int k = 1; k < INS_ROW; k++) dst[k - 1] = row8[k];
}

// MISC::getImuSeriesFromTo(start, end) (misc.cc:307-361) of window J in two halves.  series_ends, on one lane: both indices, the
// isNeedInterpolation cases at each end with imuInterpolation's split, written to ser (rows of 7); n = 0 when the window cannot serve the
// interval (getInsWindowIndex 0 at either end, or an empty series).  series_middle, on the warp: the middle rows (:337-340) between them.
// The last row's time becomes `end` (:357-358); the rows carry no time, and the preintegration does not read it.
struct SeriesCut {
    int n, m0, nm, nh;  // rows; first middle entry, middle rows, rows before them
};

__device__ SeriesCut series_ends(const double *I, const InsJob &J, int cap, double start, double end, double *ser) {
    SeriesCut c = {0, 0, 0, 0};
    const int is = window_index(I, J, cap, start), ie = window_index(I, J, cap, end);
    if (!is || !ie) return c;
    const double *a0 = I + INS_ROW * ring(J, cap, is - 1), *a1 = I + INS_ROW * ring(J, cap, is);
    const double *b0 = I + INS_ROW * ring(J, cap, ie - 1), *b1 = I + INS_ROW * ring(J, cap, ie);
    double part[INS_ROW], rest[INS_ROW];
    const int sa = need_interpolation(a0, a1, start);
    if (sa == -1) {
        series_row(ser, a0), series_row(ser + 7, a1), c.nh = 2;
    } else if (sa == 1) {
        series_row(ser, a1), c.nh = 1;
    } else if (sa == 2) {
        imu_interpolation(a1, start, part, rest);
        series_row(ser, part), series_row(ser + 7, rest), c.nh = 2;
    }
    c.m0 = is + 1, c.nm = ie - 1 - c.m0 > 0 ? ie - 1 - c.m0 : 0;
    double *tail = ser + 7 * (c.nh + c.nm);
    int nt = 0;
    const int sb = need_interpolation(b0, b1, end);
    if (sb == -1) {
        series_row(tail, b0), nt = 1;
    } else if (sb == 1) {
        series_row(tail, b0), series_row(tail + 7, b1), nt = 2;
    } else if (sb == 2) {
        imu_interpolation(b1, end, part, rest);
        series_row(tail, b0), series_row(tail + 7, part), nt = 2;
    }
    c.n = c.nh + c.nm + nt;
    return c;
}

__device__ __forceinline__ void series_middle(const double *I, const InsJob &J, int cap, const SeriesCut &c, double *ser) {
    for (int k = threadIdx.x & 31; k < c.nm; k += 32) series_row(ser + 7 * (c.nh + k), I + INS_ROW * ring(J, cap, c.m0 + k));
}

// the series of each (stream, start, end) job, one warp per job (ins_handle.cuh)
__global__ void __launch_bounds__(32 * INS_WARPS) ins_cut_kernel(int n_jobs, int cap, const InsCutJob *jobs, const double *imu, double *rows,
                                                                int32_t *n_rows, int32_t *status) {
    const int lane = threadIdx.x & 31, j = blockIdx.x * INS_WARPS + (threadIdx.x >> 5);
    if (j >= n_jobs) return;
    const InsCutJob q = jobs[j];
    InsJob J = {};
    J.head = q.head, J.count = q.count;
    const double *I = imu + (size_t) q.stream * cap * INS_ROW;
    double *ser = rows + 7 * (size_t) q.out;
    SeriesCut c = {0, 0, 0, 0};
    if (lane == 0) c = series_ends(I, J, cap, q.t0, q.t1, ser);
    c.n = __shfl_sync(0xffffffffu, c.n, 0), c.m0 = __shfl_sync(0xffffffffu, c.m0, 0);
    c.nm = __shfl_sync(0xffffffffu, c.nm, 0), c.nh = __shfl_sync(0xffffffffu, c.nh, 0);
    if (c.n > 0) series_middle(I, J, cap, c, ser);
    if (lane == 0) n_rows[j] = c.n, status[j] = c.n > 0 ? 1 : -5;
}

// gvinsInitialization up to and including the redo; series (INS_SERIES_MAX x 7 per stream) receives getImuSeriesFromTo(last_time,
// gnss_time) of the window the redo leaves.  The series only reads rows, which the redo does not change, so it and every status are decided
// before the window is written.
__global__ void __launch_bounds__(32 * INS_WARPS) ins_gins_init_kernel(int n_streams, int cap, int reserved, const InsJob *jobs,
                                                                      const icg_gins_init *in, const double *slot6, const int32_t *zv,
                                                                      double *imu, double *st, double *series, GinsOut out) {
    __shared__ double sh[INS_WARPS][32][12];
    __shared__ double carry[INS_WARPS][8];
    __shared__ double u[INS_WARPS][INS_ST];
    __shared__ int info[INS_WARPS][5];  // status, first middle row, middle rows, rows before them, rows the redo drops
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, s = blockIdx.x * INS_WARPS + w;
    if (s >= n_streams) return;
    InsJob J = jobs[s];
    if (!J.sel) return;
    const icg_gins_init &G = in[s];
    double *I = imu + (size_t) s * cap * INS_ROW, *X = st + (size_t) s * cap * INS_ST, *ser = series + (size_t) s * INS_SERIES_MAX * 7;
    if (lane == 0) {
        double bg[3], att[3];
        for (int k = 0; k < 3; k++) bg[k] = slot6[6 * s + k], att[k] = slot6[6 * s + 3 + k];
        int hzv = zv[s], status = 0, n_ser = 0, m0 = 0, nm = 0, nh = 0, drop = 0;
        InsJob J2 = J;
        if (G.gnss_time == 0 || G.last_time == 0) {
            status = -1;
        } else {
            // the zero-velocity buffer (:592-598) and MISC::detectZeroVelocity (misc.cc:363-415), sums in row order
            int n = 0;
            double avg[6] = {0, 0, 0, 0, 0, 0}, sum[6] = {0, 0, 0, 0, 0, 0};
            for (int e = 0; e < J.count; e++) {
                const double *r = I + INS_ROW * ring(J, cap, e);
                if (r[0] > G.last_time && r[0] < G.gnss_time) {
                    n++;
                    for (int k = 0; k < 6; k++) avg[k] += r[2 + k];
                }
            }
            if (n < 20) {
                status = -2;
            } else {
                const double inv = 1.0 / (double) n;
                for (int k = 0; k < 6; k++) avg[k] *= inv;
                for (int e = 0; e < J.count; e++) {
                    const double *r = I + INS_ROW * ring(J, cap, e);
                    if (r[0] > G.last_time && r[0] < G.gnss_time)
                        for (int k = 0; k < 6; k++) sum[k] += (r[2 + k] - avg[k]) * (r[2 + k] - avg[k]);
                }
                bool zero = true;
                for (int k = 0; k < 6; k++) zero = zero && sqrt(sum[k] * inv) * G.imudatarate < (k < 3 ? ZV_GYR : ZV_ACC);
                if (zero) {  // gyroscope biases and levelling (:611-626), then `return false` (:648-650)
                    for (int k = 0; k < 3; k++) bg[k] = avg[k] * G.imudatarate;
                    const double fx = avg[3] * G.imudatarate, fy = avg[4] * G.imudatarate;
                    att[0] = -asin(fy / G.gravity), att[1] = asin(fx / G.gravity);
                    hzv = 1, status = -3;
                } else if (G.last_yaw_valid) {
                    att[2] = G.last_yaw;
                } else {
                    const double vx = G.gnss_blh[0] - G.last_blh[0], vy = G.gnss_blh[1] - G.last_blh[1], vz = G.gnss_blh[2] - G.last_blh[2];
                    if (sqrt(vx * vx + vy * vy + vz * vz) < MIN_ALIGN_VELOCITY) {
                        status = -4;
                    } else {
                        if (!hzv) att[0] = 0, att[1] = atan(-vz / sqrt(vx * vx + vy * vy));
                        att[2] = atan2(vy, vx);
                    }
                }
            }
        }
        if (status == 0) {
            // the redo's index and pruning (misc.cc:212, 253-260), then getImuSeriesFromTo's indices on the pruned window (misc.cc:307-316)
            const int index = window_index(I, J, cap, G.last_time);
            drop = index >= reserved ? index - reserved : 0;
            J2.head = (J.head + drop) % cap, J2.count = J.count - drop;
            if (index) {
                const SeriesCut c = series_ends(I, J2, cap, G.last_time, G.gnss_time, ser);
                n_ser = c.n, m0 = c.m0, nm = c.nm, nh = c.nh;
            }
            status = n_ser > 0 ? 1 : -5;
        }
        if (status == 1) {
            // the initial state (:652-668): q = euler2quaternion(initatt) = AngleAxis(yaw, Z) AngleAxis(pitch, Y) AngleAxis(roll, X)
            const Q qz = mkq(cos(0.5 * att[2]), 0, 0, sin(0.5 * att[2])), qy = mkq(cos(0.5 * att[1]), 0, sin(0.5 * att[1]), 0);
            const Q qx = mkq(cos(0.5 * att[0]), sin(0.5 * att[0]), 0, 0), q = qmul(qmul(qz, qy), qx);
            const V3 p = mk(G.last_blh[0], G.last_blh[1], G.last_blh[2]) - qrot(q, mk(G.antlever[0], G.antlever[1], G.antlever[2]));
            put_state(u[w], G.last_time, p, q, mk(0, 0, 0), mk(bg[0], bg[1], bg[2]), mk(0, 0, 0));
            for (int k = 0; k < INS_ST; k++) out.state17[INS_ST * s + k] = u[w][k];
            // integration_config_.gravity / iewn (:675-678)
            const V3 iw = J.earth ? gc::earth_iewn(G.origin_blh, p) : mk(J.iewn[0], J.iewn[1], J.iewn[2]);
            out.iewn[3 * s] = iw.x, out.iewn[3 * s + 1] = iw.y, out.iewn[3 * s + 2] = iw.z;
        }
        out.status[s] = status, out.n_series[s] = n_ser, out.zv[s] = hzv;
        for (int k = 0; k < 3; k++) out.slot6[6 * s + k] = bg[k], out.slot6[6 * s + 3 + k] = att[k];
        info[w][0] = status, info[w][1] = m0, info[w][2] = nm, info[w][3] = nh, info[w][4] = drop;
    }
    __syncwarp();
    if (info[w][0] != 1) return;
    const SeriesCut c = {0, info[w][1], info[w][2], info[w][3]};
    InsJob J2 = J;
    J2.head = (J.head + info[w][4]) % cap, J2.count = J.count - info[w][4];
    series_middle(I, J2, cap, c, ser);  // on the pruned window
    // the redo of :682-683 from that state, with integration_config_ as it now is
    J.grav[0] = 0, J.grav[1] = 0, J.grav[2] = G.gravity;
    if (J.earth)
        for (int k = 0; k < 3; k++) J.iewn[k] = out.iewn[3 * s + k];
    const int index = redo_window(sh[w], carry[w], J, cap, I, X, u[w]);
    if (lane == 0) out.index[s] = index;
}

// Rotation::quaternion2vector (IG/common/rotation.h:78-81) through Eigen's AngleAxis(quaternion): n = |vec|; n != 0: angle 2 atan2(n, |w|),
// axis +-vec / n by the sign of w; otherwise angle 0, axis (1, 0, 0) [ext, unpinned: Eigen is not part of this build]
__device__ V3 quat2rotvec(Q q) {
    const double n = sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
    if (n == 0) return mk(0, 0, 0);
    const double angle = 2 * atan2(n, fabs(q.w));
    const V3 axis = q.w < 0 ? mk(-q.x, -q.y, -q.z) / n : mk(q.x, q.y, q.z) / n;
    return angle * axis;
}

// getCameraPoseFromInsWindow, one stream per thread: statePoseInterpolation (misc.cc:85-100, the STATES' times) and stateToCameraPose
// (:102-108)
__global__ void ins_pose_kernel(int n_streams, int cap, const InsJob *jobs, const double *stamp, const double *pose_b_c, const double *imu,
                                const double *st, double *pose, int32_t *found) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_streams) return;
    const InsJob J = jobs[s];
    if (!J.mech) {
        found[s] = -1;
        return;
    }
    const double *I = imu + (size_t) s * cap * INS_ROW, *X = st + (size_t) s * cap * INS_ST;
    const double t = stamp[s];
    const int index = window_index(I, J, cap, t);
    V3 p;
    Q q;
    if (index > 0) {
        const double *x0 = X + INS_ST * ring(J, cap, index - 1), *x1 = X + INS_ST * ring(J, cap, index);
        const V3 p0 = mk(x0[1], x0[2], x0[3]), p1 = mk(x1[1], x1[2], x1[3]);
        const Q q0 = mkq(x0[7], x0[4], x0[5], x0[6]), q1 = mkq(x1[7], x1[4], x1[5], x1[6]);
        const V3 dp = p1 - p0;
        const double scale = (t - x0[0]) / (x1[0] - x0[0]);
        const Q dq = rotvec2q(quat2rotvec(qmul(qinv(q1), q0)) * scale);
        p = p0 + dp * scale;
        q = qnormalized(qmul(q0, qinv(dq)));
    } else {
        const double *x = X + INS_ST * ring(J, cap, J.count - 1);
        p = mk(x[1], x[2], x[3]), q = mkq(x[7], x[4], x[5], x[6]);
    }
    const double *bc = pose_b_c + 12 * (size_t) s;
    M3 Rbc;
    for (int k = 0; k < 9; k++) Rbc.m[k] = bc[k];
    const M3 R = qmat(q), Rc = mul(R, Rbc);
    const V3 tc = p + mul(R, mk(bc[9], bc[10], bc[11]));
    double *o = pose + 12 * (size_t) s;
    for (int k = 0; k < 9; k++) o[k] = Rc.m[k];
    o[9] = tc.x, o[10] = tc.y, o[11] = tc.z;
    found[s] = index > 0 ? 1 : 0;
}

}  // namespace

cudaError_t icg::ins_cut_launch(const icg_ins *h, int n_jobs, const InsCutJob *jobs, double *rows, int32_t *n_rows, int32_t *status,
                                cudaStream_t stream) {
    if (n_jobs <= 0) return cudaSuccess;
    ins_cut_kernel<<<(n_jobs + INS_WARPS - 1) / INS_WARPS, 32 * INS_WARPS, 0, stream>>>(n_jobs, h->capacity, jobs, h->d_imu, rows, n_rows, status);
    count_launch();
    return cudaGetLastError();
}

static int ins_stage(icg_ins *h, size_t bytes) {
    if (h->stage_pending) ICG_CUDA(cudaEventSynchronize(h->stage_ev));
    h->stage_pending = false;
    if (h->stage_bytes >= bytes) return ICG_OK;
    bytes = ((bytes + 4095) & ~(size_t) 4095) * 2;
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    if (h->d_stage) cudaFree(h->d_stage);
    if (h->h_stage) cudaFreeHost(h->h_stage);
    h->d_stage = h->h_stage = nullptr, h->stage_bytes = 0;
    if (cudaMalloc(&h->d_stage, bytes) != cudaSuccess || cudaMallocHost(&h->h_stage, bytes) != cudaSuccess) {
        set_error("icg_ins: staging allocation of %zu bytes failed", bytes);
        return ICG_ENOMEM;
    }
    h->stage_bytes = bytes;
    return ICG_OK;
}

static int ins_fence(icg_ins *h) {
    ICG_CUDA(cudaEventRecord(h->stage_ev, h->stream));
    h->stage_pending = true;
    return ICG_OK;
}

static bool ins_cfg_ok(const icg_ins_config &c) { return c.with_earth == 0 || c.with_earth == 1; }

static void ins_job(const icg_ins *h, int s, const icg_ins_config *cfg, InsJob &J) {
    memset(&J, 0, sizeof(J));
    if (cfg) {
        for (int k = 0; k < 3; k++) J.grav[k] = cfg->gravity[k], J.iewn[k] = cfg->with_earth ? cfg->iewn[k] : 0.0;
        J.earth = cfg->with_earth;
    }
    J.head = h->head[s], J.count = h->count[s], J.mech = h->mech[s];
}

extern "C" {

int icg_ins_create(icg_ins **out, int max_streams, int capacity, int device, void *stream) {
    if (!out || max_streams < 1 || capacity < INS_INIT_KEEP || capacity > INS_MAX_CAPACITY) {
        set_error("icg_ins_create: bad arguments (max_streams >= 1, capacity in [%d, %d])", INS_INIT_KEEP, INS_MAX_CAPACITY);
        return ICG_EINVAL;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        set_error("icg_ins_create: no CUDA device (this library has no CPU fallback)");
        return ICG_ENODEVICE;
    }
    if (device < 0 || device >= ndev) {
        set_error("icg_ins_create: device %d out of range", device);
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    ICG_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error("icg_ins_create: device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor);
        return ICG_ENODEVICE;
    }
    icg_ins *h = new icg_ins();
    h->device = device, h->max_streams = max_streams, h->capacity = capacity, h->own_stream = stream == nullptr;
    h->head.assign(max_streams, 0), h->count.assign(max_streams, 0), h->mech.assign(max_streams, 0), h->seen.assign(max_streams, 0);
    h->last_time.assign(max_streams, 0.0);
    h->init_slot6.assign(6 * (size_t) max_streams, 0.0), h->init_zv.assign(max_streams, 0);
    const size_t entries = (size_t) max_streams * capacity;
    bool ok = true;
    if (stream)
        h->stream = (cudaStream_t) stream;
    else
        ok = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) == cudaSuccess;
    if (!ok) h->own_stream = false;
    ok = ok && cudaEventCreateWithFlags(&h->stage_ev, cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaMalloc(&h->d_imu, sizeof(double) * INS_ROW * entries) == cudaSuccess;
    ok = ok && cudaMalloc(&h->d_st, sizeof(double) * INS_ST * entries) == cudaSuccess;
    ok = ok && cudaMemsetAsync(h->d_imu, 0, sizeof(double) * INS_ROW * entries, h->stream) == cudaSuccess;
    ok = ok && cudaMemsetAsync(h->d_st, 0, sizeof(double) * INS_ST * entries, h->stream) == cudaSuccess;
    if (!ok) {
        icg_ins_destroy(h);
        set_error("icg_ins_create: allocation of %d x %d window entries failed", max_streams, capacity);
        return ICG_ENOMEM;
    }
    *out = h;
    return ICG_OK;
}

void icg_ins_destroy(icg_ins *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->d_imu) cudaFree(h->d_imu);
    if (h->d_st) cudaFree(h->d_st);
    if (h->d_series) cudaFree(h->d_series);
    if (h->d_stage) cudaFree(h->d_stage);
    if (h->h_stage) cudaFreeHost(h->h_stage);
    if (h->stage_ev) cudaEventDestroy(h->stage_ev);
    if (h->own_stream) cudaStreamDestroy(h->stream);
    delete h;
}

int icg_ins_push(icg_ins *h, int n_streams, const icg_ins_config *cfg, const int32_t *off, const double *imu) {
    if (!h || n_streams < 0 || n_streams > h->max_streams || (n_streams > 0 && (!cfg || !off))) {
        set_error("icg_ins_push: bad arguments");
        return ICG_EINVAL;
    }
    if (n_streams == 0) return ICG_OK;
    if (off[0] < 0 || (!imu && off[n_streams] > off[0])) {
        set_error("icg_ins_push: bad row offsets");
        return ICG_EINVAL;
    }
    for (int s = 0; s < n_streams; s++) {
        if (off[s + 1] < off[s] || !ins_cfg_ok(cfg[s])) {
            set_error("icg_ins_push: stream %d: bad row offsets or configuration", s);
            return ICG_EINVAL;
        }
        const int n = off[s + 1] - off[s];
        double prev = h->last_time[s];
        bool have = h->seen[s];
        for (int k = 0; k < n; k++) {
            const double t = imu[INS_ROW * ((size_t) off[s] + k)];
            if (!(t == t) || (have && !(t > prev))) {
                set_error("icg_ins_push: stream %d row %d: time %.17g is not greater than the previous sample's %.17g", s, k, t, prev);
                return ICG_EINVAL;
            }
            prev = t, have = true;
        }
        if (h->mech[s] && (int64_t) h->count[s] + n > h->capacity) {
            set_error("icg_ins_push: stream %d: %d + %d rows exceed the window capacity %d (no redo has pruned it)", s, h->count[s], n, h->capacity);
            return ICG_EINVAL;
        }
    }
    ICG_CUDA(cudaSetDevice(h->device));
    const size_t rows = (size_t) (off[n_streams] - off[0]);
    const size_t o_rows = (sizeof(InsJob) * n_streams + 255) & ~(size_t) 255, total = o_rows + sizeof(double) * INS_ROW * rows;
    int rc = ins_stage(h, total);
    if (rc != ICG_OK) return rc;
    InsJob *jobs = (InsJob *) h->h_stage;
    for (int s = 0; s < n_streams; s++) {
        InsJob &J = jobs[s];
        ins_job(h, s, cfg + s, J);
        const int n = off[s + 1] - off[s];
        J.n = n, J.off = off[s] - off[0];
        if (h->mech[s]) {
            J.count += n;
        } else {  // initialization path: the window keeps its newest 1000 rows
            J.skip = n > INS_INIT_KEEP ? n - INS_INIT_KEEP : 0;
            const int total_n = h->count[s] + n, keep = total_n < INS_INIT_KEEP ? total_n : INS_INIT_KEEP;
            h->head[s] = (h->head[s] + total_n - keep) % h->capacity;
            J.count = keep, J.head = h->head[s];
        }
        h->count[s] = J.count;
        if (n > 0) h->last_time[s] = imu[INS_ROW * ((size_t) off[s + 1] - 1)], h->seen[s] = 1;
    }
    if (rows) memcpy(h->h_stage + o_rows, imu + INS_ROW * (size_t) off[0], sizeof(double) * INS_ROW * rows);
    ICG_CUDA(cudaMemcpyAsync(h->d_stage, h->h_stage, total, cudaMemcpyHostToDevice, h->stream));
    rc = ins_fence(h);
    if (rc != ICG_OK) return rc;
    ins_push_kernel<<<(n_streams + INS_WARPS - 1) / INS_WARPS, 32 * INS_WARPS, 0, h->stream>>>(
        n_streams, h->capacity, (const InsJob *) h->d_stage, (const double *) (h->d_stage + o_rows), h->d_imu, h->d_st);
    ICG_CHECK_LAUNCH();
    count_launch();
    return ICG_OK;
}

int icg_ins_redo(icg_ins *h, int n_streams, const icg_ins_config *cfg, const uint8_t *redo, const double *state17, int reserved, int8_t *status) {
    if (!h || n_streams < 0 || n_streams > h->max_streams || reserved < 0 || (n_streams > 0 && (!cfg || !state17 || !status))) {
        set_error("icg_ins_redo: bad arguments");
        return ICG_EINVAL;
    }
    for (int s = 0; s < n_streams; s++)
        if ((!redo || redo[s]) && !ins_cfg_ok(cfg[s])) {
            set_error("icg_ins_redo: stream %d: bad configuration", s);
            return ICG_EINVAL;
        }
    if (n_streams == 0) return ICG_OK;
    ICG_CUDA(cudaSetDevice(h->device));
    const size_t o_st = (sizeof(InsJob) * n_streams + 255) & ~(size_t) 255, o_out = o_st + sizeof(double) * INS_ST * n_streams;
    const size_t total = o_out + sizeof(int32_t) * 2 * n_streams;
    int rc = ins_stage(h, total);
    if (rc != ICG_OK) return rc;
    InsJob *jobs = (InsJob *) h->h_stage;
    for (int s = 0; s < n_streams; s++) ins_job(h, s, cfg + s, jobs[s]), jobs[s].sel = !redo || redo[s];
    memcpy(h->h_stage + o_st, state17, sizeof(double) * INS_ST * n_streams);
    ICG_CUDA(cudaMemcpyAsync(h->d_stage, h->h_stage, o_out, cudaMemcpyHostToDevice, h->stream));
    ins_redo_kernel<<<(n_streams + INS_WARPS - 1) / INS_WARPS, 32 * INS_WARPS, 0, h->stream>>>(
        n_streams, h->capacity, (const InsJob *) h->d_stage, (const double *) (h->d_stage + o_st), h->d_imu, h->d_st,
        (int32_t *) (h->d_stage + o_out));
    ICG_CHECK_LAUNCH();
    count_launch();
    ICG_CUDA(cudaMemcpyAsync(h->h_stage + o_out, h->d_stage + o_out, sizeof(int32_t) * 2 * n_streams, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    const int32_t *res = (const int32_t *) (h->h_stage + o_out);
    for (int s = 0; s < n_streams; s++) {
        status[s] = 0;
        if (!jobs[s].sel) continue;
        status[s] = (int8_t) res[2 * s];
        if (res[2 * s] != 1) continue;
        const int index = res[2 * s + 1];
        h->mech[s] = 1;
        if (index >= reserved) {  // pop_front of the expired entries (misc.cc:253-260)
            h->head[s] = (h->head[s] + index - reserved) % h->capacity;
            h->count[s] -= index - reserved;
        }
    }
    return ICG_OK;
}

int icg_ins_gins_initialize(icg_ins *h, int n_streams, icg_ins_config *cfg, const uint8_t *sel, const icg_gins_init *in, const double *noise5,
                            const double *station3, int reserved, icg_gins_init_out *out) {
    if (!h || n_streams < 0 || n_streams > h->max_streams || reserved < 0 ||
        (n_streams > 0 && (!cfg || !in || !noise5 || !station3 || !out))) {
        set_error("icg_ins_gins_initialize: bad arguments");
        return ICG_EINVAL;
    }
    for (int s = 0; s < n_streams; s++) {
        if (sel && !sel[s]) continue;
        if (!ins_cfg_ok(cfg[s])) {
            set_error("icg_ins_gins_initialize: stream %d: bad configuration", s);
            return ICG_EINVAL;
        }
        if (h->mech[s]) {
            set_error("icg_ins_gins_initialize: stream %d is already mechanized (initialized)", s);
            return ICG_EINVAL;
        }
    }
    if (n_streams == 0) return ICG_OK;
    ICG_CUDA(cudaSetDevice(h->device));
    if (!h->d_series && cudaMalloc(&h->d_series, sizeof(double) * 7 * INS_SERIES_MAX * (size_t) h->max_streams) != cudaSuccess) {
        set_error("icg_ins_gins_initialize: allocation of the series buffer failed");
        return ICG_ENOMEM;
    }
    const size_t n = (size_t) n_streams;
    auto al = [](size_t b) { return (b + 255) & ~(size_t) 255; };
    // [jobs | in | slot6 | zv | earth | gravity]  ->  [status | n_series | zv | index | slot6 | state17 | iewn | blob | ends]
    const size_t o_in = al(sizeof(InsJob) * n), o_slot = o_in + al(sizeof(icg_gins_init) * n), o_zv = o_slot + al(sizeof(double) * 6 * n);
    const size_t o_earth = o_zv + al(sizeof(int32_t) * n), o_grav = o_earth + al(sizeof(int32_t) * n), o_out = o_grav + al(sizeof(double) * n);
    const size_t o_status = o_out, o_nser = o_status + al(sizeof(int32_t) * n), o_ozv = o_nser + al(sizeof(int32_t) * n);
    const size_t o_index = o_ozv + al(sizeof(int32_t) * n), o_oslot = o_index + al(sizeof(int32_t) * n);
    const size_t o_st = o_oslot + al(sizeof(double) * 6 * n), o_iewn = o_st + al(sizeof(double) * INS_ST * n);
    const size_t o_blob = o_iewn + al(sizeof(double) * 3 * n), o_ends = o_blob + al(sizeof(double) * ICG_IMU_BLOB_DOUBLES * n);
    const size_t total = o_ends + al(sizeof(double) * 10 * n);
    int rc = ins_stage(h, total);
    if (rc != ICG_OK) return rc;
    uint8_t *hs = h->h_stage, *ds = h->d_stage;
    InsJob *jobs = (InsJob *) hs;
    int32_t *earth = (int32_t *) (hs + o_earth);
    double *grav = (double *) (hs + o_grav);
    for (int s = 0; s < n_streams; s++) {
        ins_job(h, s, cfg + s, jobs[s]), jobs[s].sel = !sel || sel[s];
        earth[s] = cfg[s].with_earth, grav[s] = in[s].gravity;
    }
    memcpy(hs + o_in, in, sizeof(icg_gins_init) * n);
    memcpy(hs + o_slot, h->init_slot6.data(), sizeof(double) * 6 * n);
    memcpy(hs + o_zv, h->init_zv.data(), sizeof(int32_t) * n);
    memset(hs + o_out, 0, total - o_out);
    ICG_CUDA(cudaMemcpyAsync(ds, hs, total, cudaMemcpyHostToDevice, h->stream));
    GinsOut go;
    go.status = (int32_t *) (ds + o_status), go.n_series = (int32_t *) (ds + o_nser), go.zv = (int32_t *) (ds + o_ozv);
    go.index = (int32_t *) (ds + o_index), go.slot6 = (double *) (ds + o_oslot), go.state17 = (double *) (ds + o_st);
    go.iewn = (double *) (ds + o_iewn);
    ins_gins_init_kernel<<<(n_streams + INS_WARPS - 1) / INS_WARPS, 32 * INS_WARPS, 0, h->stream>>>(
        n_streams, h->capacity, reserved, (const InsJob *) ds, (const icg_gins_init *) (ds + o_in), (const double *) (ds + o_slot),
        (const int32_t *) (ds + o_zv), h->d_imu, h->d_st, h->d_series, go);
    ICG_CHECK_LAUNCH();
    count_launch();
    PreintGins pg;
    pg.n = n_streams, pg.status = go.status, pg.state17 = go.state17, pg.gravity = (const double *) (ds + o_grav);
    pg.earth = (const int32_t *) (ds + o_earth), pg.imu = h->d_series, pg.nrow = go.n_series, pg.max_rows = INS_SERIES_MAX;
    for (int k = 0; k < 5; k++) pg.noise5[k] = noise5[k];
    for (int k = 0; k < 3; k++) pg.station[k] = station3[k];
    pg.blob = (double *) (ds + o_blob), pg.ends = (double *) (ds + o_ends);
    ICG_CUDA(preint_gins_launch(pg, h->stream));
    count_launch();
    ICG_CUDA(cudaMemcpyAsync(hs + o_out, ds + o_out, total - o_out, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    const int32_t *status = (const int32_t *) (hs + o_status), *nser = (const int32_t *) (hs + o_nser), *ozv = (const int32_t *) (hs + o_ozv);
    const int32_t *index = (const int32_t *) (hs + o_index);
    const double *oslot = (const double *) (hs + o_oslot), *ost = (const double *) (hs + o_st), *oiewn = (const double *) (hs + o_iewn);
    const double *oblob = (const double *) (hs + o_blob), *oends = (const double *) (hs + o_ends);
    const double D2R = M_PI / 180.0, att_std = 0.5 * D2R;  // constructPrior (IG/ic_gvins.cc:1911-1936)
    for (int s = 0; s < n_streams; s++) {
        icg_gins_init_out &o = out[s];
        memset(&o, 0, sizeof(o));
        const int st = jobs[s].sel ? status[s] : 0;
        o.status = st;
        if (st == -3 || st == 1) {  // the slots change: levelling at zero velocity, the heading (and pitch) at initialization
            memcpy(&h->init_slot6[6 * s], oslot + 6 * s, sizeof(double) * 6);
            h->init_zv[s] = ozv[s];
        }
        o.has_zero_velocity = h->init_zv[s];
        memcpy(o.bg, &h->init_slot6[6 * s], sizeof(double) * 3), memcpy(o.initatt, &h->init_slot6[6 * s + 3], sizeof(double) * 3);
        if (st != 1) continue;
        h->mech[s] = 1;
        if (index[s] >= reserved) {  // the redo's pop_front (misc.cc:253-260)
            h->head[s] = (h->head[s] + index[s] - reserved) % h->capacity;
            h->count[s] -= index[s] - reserved;
        }
        cfg[s].gravity[0] = 0, cfg[s].gravity[1] = 0, cfg[s].gravity[2] = in[s].gravity;
        if (cfg[s].with_earth) memcpy(cfg[s].iewn, oiewn + 3 * s, sizeof(double) * 3);
        const double *x0 = ost + INS_ST * s, *e = oends + 10 * s;
        double *x1 = o.state17 + INS_ST;
        memcpy(o.state17, x0, sizeof(double) * INS_ST);
        // currentState() at gnss_time (:923-924): the propagated p, q, v and the start state's biases
        x1[0] = in[s].gnss_time;
        memcpy(x1 + 1, e, sizeof(double) * 10);
        memcpy(x1 + 11, x0 + 11, sizeof(double) * 6);
        memcpy(o.pose_prior, x0 + 1, sizeof(double) * 7), memcpy(o.mix_prior, x0 + 8, sizeof(double) * 9);
        const double bg_std = h->init_zv[s] ? noise5[2] * 3 : 7200 * D2R / 3600;  // GYROSCOPE_BIAS_PRIOR_STD (IG/ic_gvins.h:140)
        for (int k = 0; k < 3; k++) {
            o.pose_prior_std[k] = 0.1, o.pose_prior_std[3 + k] = att_std;
            o.mix_prior_std[k] = 0.1, o.mix_prior_std[3 + k] = bg_std, o.mix_prior_std[6 + k] = 20000 * 1.0e-5;  // ACCELEROMETER_BIAS_PRIOR_STD
        }
        o.pose_prior_std[5] = att_std * 3;
        memcpy(o.imu_blob, oblob + (size_t) ICG_IMU_BLOB_DOUBLES * s, sizeof(double) * ICG_IMU_BLOB_DOUBLES);
        o.n_series = nser[s];
    }
    return ICG_OK;
}

int icg_ins_camera_pose(icg_ins *h, int n_streams, const double *stamp, const double *pose_b_c, double *dev_pose, double *host_pose,
                        int32_t *found) {
    if (!h || n_streams < 0 || n_streams > h->max_streams || (n_streams > 0 && (!stamp || !pose_b_c || !dev_pose))) {
        set_error("icg_ins_camera_pose: bad arguments");
        return ICG_EINVAL;
    }
    if (n_streams == 0) return ICG_OK;
    ICG_CUDA(cudaSetDevice(h->device));
    const size_t o_in = (sizeof(InsJob) * n_streams + 255) & ~(size_t) 255, o_found = o_in + sizeof(double) * 13 * n_streams;
    const size_t total = o_found + sizeof(int32_t) * n_streams;
    int rc = ins_stage(h, total);
    if (rc != ICG_OK) return rc;
    InsJob *jobs = (InsJob *) h->h_stage;
    for (int s = 0; s < n_streams; s++) ins_job(h, s, nullptr, jobs[s]);
    double *in = (double *) (h->h_stage + o_in);
    memcpy(in, stamp, sizeof(double) * n_streams);
    memcpy(in + n_streams, pose_b_c, sizeof(double) * 12 * n_streams);
    ICG_CUDA(cudaMemcpyAsync(h->d_stage, h->h_stage, o_found, cudaMemcpyHostToDevice, h->stream));
    const double *d_in = (const double *) (h->d_stage + o_in);
    int32_t *d_found = (int32_t *) (h->d_stage + o_found);
    ins_pose_kernel<<<(n_streams + 127) / 128, 128, 0, h->stream>>>(n_streams, h->capacity, (const InsJob *) h->d_stage, d_in, d_in + n_streams,
                                                                    h->d_imu, h->d_st, dev_pose, d_found);
    ICG_CHECK_LAUNCH();
    count_launch();
    if (host_pose) {
        ICG_CUDA(cudaMemcpyAsync(h->h_stage + o_in, dev_pose, sizeof(double) * 12 * n_streams, cudaMemcpyDeviceToHost, h->stream));
        ICG_CUDA(cudaMemcpyAsync(h->h_stage + o_found, d_found, sizeof(int32_t) * n_streams, cudaMemcpyDeviceToHost, h->stream));
        ICG_CUDA(cudaStreamSynchronize(h->stream));
        memcpy(host_pose, h->h_stage + o_in, sizeof(double) * 12 * n_streams);
        if (found) memcpy(found, h->h_stage + o_found, sizeof(int32_t) * n_streams);
        return ICG_OK;
    }
    if (found) ICG_CUDA(cudaMemcpyAsync(found, d_found, sizeof(int32_t) * n_streams, cudaMemcpyDeviceToDevice, h->stream));
    return ins_fence(h);
}

int icg_ins_window(icg_ins *h, int stream, int cap, int32_t *count, double *imu8, double *state17) {
    if (!h || stream < 0 || stream >= h->max_streams || cap < 0 || !count || (cap > 0 && (!imu8 || !state17))) {
        set_error("icg_ins_window: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    const int n = h->count[stream] < cap ? h->count[stream] : cap, head = h->head[stream];
    *count = h->count[stream];
    const int n1 = n < h->capacity - head ? n : h->capacity - head;  // entries before the ring wraps
    const size_t base = (size_t) stream * h->capacity;
    const struct { double *dst; const double *src; int w; } parts[2] = {{imu8, h->d_imu, INS_ROW}, {state17, h->d_st, INS_ST}};
    for (const auto &P : parts) {
        if (n1 > 0)
            ICG_CUDA(cudaMemcpyAsync(P.dst, P.src + P.w * (base + head), sizeof(double) * P.w * n1, cudaMemcpyDeviceToHost, h->stream));
        if (n > n1)
            ICG_CUDA(cudaMemcpyAsync(P.dst + P.w * (size_t) n1, P.src + P.w * base, sizeof(double) * P.w * (n - n1), cudaMemcpyDeviceToHost, h->stream));
    }
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    return ICG_OK;
}

int icg_ins_sync(icg_ins *h) {
    if (!h) {
        set_error("icg_ins_sync: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    return ICG_OK;
}

}  // extern "C"
