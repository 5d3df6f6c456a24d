// ins.cu -- device INS windows for B streams: runFusion's per-sample mechanization (IG/ic_gvins.cc:249-293), the post-solve redo
// (MISC::redoInsMechanization, IG/misc.cc:208-261) and each frame's prior camera pose (MISC::getCameraPoseFromInsWindow, misc.cc:67-108).
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
    const double *u = state17 + (size_t) INS_ST * s;
    const double t = u[0];
    int index = 0;
    if (lane == 0) index = window_index(I, J, cap, t);
    index = __shfl_sync(0xffffffffu, index, 0);
    if (lane == 0) out[2 * s] = index == 0 ? -1 : 1, out[2 * s + 1] = index;
    if (index == 0) return;
    // stateFromData (preintegration_base.cc:115-125)
    V3 p = mk(u[1], u[2], u[3]), v = mk(u[8], u[9], u[10]);
    Q q = qnormalized(mkq(u[7], u[4], u[5], u[6]));
    const V3 bg = mk(u[11], u[12], u[13]), ba = mk(u[14], u[15], u[16]);
    if (lane == 0) {
        const int s1 = ring(J, cap, index);
        const double *imu0 = I + INS_ROW * ring(J, cap, index - 1), *imu1 = I + INS_ROW * s1;
        double *c = carry[w];
        for (int k = 0; k < INS_ROW; k++) c[k] = imu1[k];
        // isNeedInterpolation (misc.cc:263-286)
        int isneed = 0;
        if (imu0[0] < t && imu1[0] > t) isneed = t - imu0[0] < INS_MIN_DT ? -1 : imu1[0] - t < INS_MIN_DT ? 1 : 2;
        const V3 grav = mk(J.grav[0], J.grav[1], J.grav[2]), iewn = mk(J.iewn[0], J.iewn[1], J.iewn[2]);
        double a[INS_ROW];
        const double *pre = imu0;
        if (isneed == 2) {  // imuInterpolation(imu1, imu0, imu1, t) (misc.cc:288-305): imu0 := the first part, imu1 := the second
            const double scale = (imu1[0] - t) / imu1[1];
            a[0] = t, a[1] = imu1[1] - (imu1[0] - t);
            for (int k = 2; k < INS_ROW; k++) a[k] = imu1[k] * (1 - scale);
            c[0] = imu1[0], c[1] = imu1[0] - t;
            for (int k = 2; k < INS_ROW; k++) c[k] = imu1[k] * scale;
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
    mechanize_run(sh[w], J, cap, I, X, index + 1, carry[w] + 1, bg, ba, p, q, v);
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

struct icg_ins {
    int device, max_streams, capacity;
    cudaStream_t stream;
    bool own_stream;
    double *d_imu = nullptr, *d_st = nullptr;
    // the host mirror
    std::vector<int32_t> head, count;
    std::vector<uint8_t> mech, seen;
    std::vector<double> last_time;
    // per-call staging [jobs | doubles | ints], pinned and device, grown on demand; the asynchronous calls' copies complete at stage_ev
    uint8_t *h_stage = nullptr, *d_stage = nullptr;
    size_t stage_bytes = 0;
    cudaEvent_t stage_ev = nullptr;
    bool stage_pending = false;
};

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
