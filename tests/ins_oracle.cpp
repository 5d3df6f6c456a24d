// ins_oracle.cpp -- CPU restatement of IC-GVINS' INS window (TEST INFRASTRUCTURE ONLY; shares no code with ic_gvins_b200/).
// MISC::insMechanization, redoInsMechanization, getInsWindowIndex, isNeedInterpolation, imuInterpolation, statePoseInterpolation and
// stateToCameraPose (IG/misc.cc), and runFusion's per-sample window step (IG/ic_gvins.cc:249-293), on std::deque storage as the reference
// keeps ins_window_.  Quaternions follow Eigen's Quaterniond conventions (Hamilton product, toRotationMatrix, inverse() = conjugate /
// squaredNorm); AngleAxis(quaternion) as Eigen states it [ext, unpinned].  Built by tests/ins_oracle.py.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <deque>
#include <utility>
#include <vector>

namespace {

struct V {
    double x, y, z;
};
V operator+(V a, V b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
V operator-(V a, V b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
V operator*(double s, V a) { return {s * a.x, s * a.y, s * a.z}; }
V operator*(V a, double s) { return {a.x * s, a.y * s, a.z * s}; }
V operator/(V a, double s) { return {a.x / s, a.y / s, a.z / s}; }
V crs(V a, V b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
double nrm(V a) { return sqrt(a.x * a.x + a.y * a.y + a.z * a.z); }

struct M {
    double a[3][3];
};
V mv(const M &m, V v) {
    return {m.a[0][0] * v.x + m.a[0][1] * v.y + m.a[0][2] * v.z, m.a[1][0] * v.x + m.a[1][1] * v.y + m.a[1][2] * v.z,
            m.a[2][0] * v.x + m.a[2][1] * v.y + m.a[2][2] * v.z};
}
M mm(const M &l, const M &r) {
    M o;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) o.a[i][j] = l.a[i][0] * r.a[0][j] + l.a[i][1] * r.a[1][j] + l.a[i][2] * r.a[2][j];
    return o;
}

struct Qd {
    double w, x, y, z;
};
Qd qprod(Qd a, Qd b) {
    return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}
Qd qinverse(Qd q) {
    const double n2 = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
    return {q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2};
}
Qd qnorm(Qd q) {
    const double n = sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    return {q.w / n, q.x / n, q.y / n, q.z / n};
}
M rot(Qd q) {
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z, twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    M r = {{{1 - (tyy + tzz), txy - twz, txz + twy}, {txy + twz, 1 - (txx + tzz), tyz - twx}, {txz - twy, tyz + twx, 1 - (txx + tyy)}}};
    return r;
}
// Rotation::rotvec2quaternion (IG/common/rotation.h:72-76): Quaterniond(AngleAxisd(|rv|, rv.normalized()))
Qd rotvec2quaternion(V rv) {
    const double angle = nrm(rv);
    const V ax = angle > 0 ? rv / angle : rv;
    const double s = sin(0.5 * angle);
    return {cos(0.5 * angle), s * ax.x, s * ax.y, s * ax.z};
}
// Rotation::quaternion2vector (rotation.h:78-81) = AngleAxisd(q).angle() * axis()
V quaternion2vector(Qd q) {
    const double n = sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
    double angle = 0;
    V axis = {1, 0, 0};
    if (n != 0) {
        angle = 2 * atan2(n, fabs(q.w));
        axis = q.w < 0 ? V{-q.x, -q.y, -q.z} / n : V{q.x, q.y, q.z} / n;
    }
    return angle * axis;
}

struct IMU {
    double time, dt;
    V dtheta, dvel;
};
struct State {
    double time;
    V p;
    Qd q;
    V v, bg, ba;
};
struct Config {
    bool earth;
    V gravity, iewn;
};
using Window = std::deque<std::pair<IMU, State>>;
constexpr double MINIMUM_TIME_INTERVAL = 0.0001;
constexpr size_t MAXIMUM_INS_NUMBER = 1000;

IMU imu_of(const double *r) { return {r[0], r[1], {r[2], r[3], r[4]}, {r[5], r[6], r[7]}}; }
void imu_out(const IMU &m, double *r) {
    const double v[8] = {m.time, m.dt, m.dtheta.x, m.dtheta.y, m.dtheta.z, m.dvel.x, m.dvel.y, m.dvel.z};
    memcpy(r, v, sizeof(v));
}
State state_of(const double *x) { return {x[0], {x[1], x[2], x[3]}, {x[7], x[4], x[5], x[6]}, {x[8], x[9], x[10]}, {x[11], x[12], x[13]}, {x[14], x[15], x[16]}}; }
void state_out(const State &s, double *x) {
    const double v[17] = {s.time, s.p.x, s.p.y, s.p.z, s.q.x, s.q.y, s.q.z, s.q.w, s.v.x, s.v.y, s.v.z, s.bg.x, s.bg.y, s.bg.z, s.ba.x, s.ba.y, s.ba.z};
    memcpy(x, v, sizeof(v));
}
Config config_of(const double *c) { return {c[0] != 0, {c[1], c[2], c[3]}, {c[4], c[5], c[6]}}; }

// MISC::insMechanization (misc.cc:151-206), iswithscale == false
void insMechanization(const Config &config, const IMU &imu_pre, const IMU &imu_cur, State &state) {
    const V cth = imu_cur.dtheta - imu_cur.dt * state.bg, cvl = imu_cur.dvel - imu_cur.dt * state.ba;
    const V pth = imu_pre.dtheta - imu_pre.dt * state.bg, pvl = imu_pre.dvel - imu_pre.dt * state.ba;
    const double dt = imu_cur.dt;
    state.time = imu_cur.time;
    const V dvfb = cvl + 0.5 * crs(cth, cvl) + 1.0 / 12.0 * (crs(pth, cvl) + crs(pvl, cth));
    const V dtheta = cth + 1.0 / 12.0 * crs(pth, cth);
    V dvel;
    if (config.earth) {
        const V dv_cor_g = (config.gravity - 2.0 * crs(config.iewn, state.v)) * dt;
        const Qd qnn = rotvec2quaternion(V{0, 0, 0} - config.iewn * dt);
        const M Rn = rot(qnn);
        M half;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) half.a[i][j] = 0.5 * ((i == j ? 1.0 : 0.0) + Rn.a[i][j]);
        dvel = mv(mm(half, rot(state.q)), dvfb) + dv_cor_g;  // Eigen's left-to-right product
        state.q = qnorm(qprod(qprod(qnn, state.q), rotvec2quaternion(dtheta)));
    } else {
        dvel = mv(rot(state.q), dvfb) + config.gravity * dt;
        state.q = qnorm(qprod(state.q, rotvec2quaternion(dtheta)));
    }
    state.p = state.p + (dt * state.v + 0.5 * dt * dvel);  // p += ...
    state.v = state.v + dvel;
}

// MISC::getInsWindowIndex (misc.cc:30-65)
size_t getInsWindowIndex(const Window &window, double time) {
    if (window.empty() || window.front().first.time > time || window.back().first.time <= time) return 0;
    size_t index = 0, sta = 0, end = window.size();
    int counts = 0;
    while (true) {
        const size_t mid = (sta + end) / 2;
        const double first = window[mid - 1].first.time, second = window[mid].first.time;
        if (first <= time && time < second) {
            index = mid;
            break;
        } else if (first > time) {
            end = mid;
        } else if (second <= time) {
            sta = mid;
        }
        if (counts++ > 15) break;
    }
    return index;
}

// MISC::isNeedInterpolation (misc.cc:263-286)
int isNeedInterpolation(const IMU &imu0, const IMU &imu1, double mid) {
    if (imu0.time < mid && imu1.time > mid) {
        if (mid - imu0.time < MINIMUM_TIME_INTERVAL) return -1;
        if (imu1.time - mid < MINIMUM_TIME_INTERVAL) return 1;
        return 2;
    }
    return 0;
}

// MISC::imuInterpolation (misc.cc:288-305); imu01 may alias imu11
void imuInterpolation(const IMU &imu01, IMU &imu00, IMU &imu11, double mid) {
    const double scale = (imu01.time - mid) / imu01.dt;
    const IMU buff = imu01;
    imu00.time = mid;
    imu00.dt = buff.dt - (buff.time - mid);
    imu00.dtheta = buff.dtheta * (1 - scale);
    imu00.dvel = buff.dvel * (1 - scale);
    imu11.time = buff.time;
    imu11.dt = buff.time - mid;
    imu11.dtheta = buff.dtheta * scale;
    imu11.dvel = buff.dvel * scale;
}

// MISC::redoInsMechanization (misc.cc:208-261); returns index
size_t redoInsMechanization(const Config &config, const State &updated_state, size_t reserved, Window &w) {
    State state = updated_state;
    const size_t index = getInsWindowIndex(w, state.time);
    if (index == 0) return 0;
    IMU imu0 = w[index - 1].first, imu1 = w[index].first;
    const int isneed = isNeedInterpolation(imu0, imu1, state.time);
    if (isneed == -1) {
        insMechanization(config, imu0, imu1, state);
        w[index].second = state;
    } else if (isneed == 1) {
        state.time = imu1.time;
        w[index].second = state;
    } else if (isneed == 2) {
        imuInterpolation(imu1, imu0, imu1, state.time);
        insMechanization(config, imu0, imu1, state);
        w[index].second = state;
    }
    for (size_t k = index + 1; k < w.size(); k++) {
        imu0 = imu1;
        imu1 = w[k].first;
        insMechanization(config, imu0, imu1, state);
        w[k].second = state;
    }
    if (index >= reserved)
        for (size_t k = 0; k < index - reserved; k++) w.pop_front();
    return index;
}

// MISC::statePoseInterpolation (misc.cc:85-100)
void statePoseInterpolation(const State &state0, const State &state1, double midtime, State &state) {
    const V dp = state1.p - state0.p;
    Qd dq = qprod(qinverse(state1.q), state0.q);
    V rvec = quaternion2vector(dq);
    const double scale = (midtime - state0.time) / (state1.time - state0.time);
    rvec = rvec * scale;
    dq = rotvec2quaternion(rvec);
    state.p = state0.p + dp * scale;
    state.q = qnorm(qprod(state0.q, qinverse(dq)));
}

// MISC::stateToCameraPose (misc.cc:102-108); pose = R row-major, t
void stateToCameraPose(const State &state, const double *pose_b_c, double *pose) {
    M Rbc;
    for (int i = 0; i < 9; i++) Rbc.a[i / 3][i % 3] = pose_b_c[i];
    const M R = rot(state.q);
    const V t = state.p + mv(R, V{pose_b_c[9], pose_b_c[10], pose_b_c[11]});
    const M Rc = mm(R, Rbc);
    for (int i = 0; i < 9; i++) pose[i] = Rc.a[i / 3][i % 3];
    pose[9] = t.x, pose[10] = t.y, pose[11] = t.z;
}

// MISC::getCameraPoseFromInsWindow (misc.cc:67-83)
bool getCameraPoseFromInsWindow(const Window &w, const double *pose_b_c, double time, double *pose) {
    const size_t index = getInsWindowIndex(w, time);
    if (index > 0) {
        State state = w[index].second;
        statePoseInterpolation(w[index - 1].second, w[index].second, time, state);
        stateToCameraPose(state, pose_b_c, pose);
        return true;
    }
    stateToCameraPose(w.back().second, pose_b_c, pose);
    return false;
}

struct Ins {
    int capacity;
    std::vector<Window> w;
    std::vector<char> mech, seen;
    std::vector<double> last;
};

}  // namespace

extern "C" {

void *icgo_ins_new(int n_streams, int capacity) {
    Ins *h = new Ins();
    h->capacity = capacity;
    h->w.resize(n_streams), h->mech.assign(n_streams, 0), h->seen.assign(n_streams, 0), h->last.assign(n_streams, 0.0);
    return h;
}
void icgo_ins_free(void *p) { delete (Ins *) p; }

// runFusion's IMU step (IG/ic_gvins.cc:249-293) per row.  cfg7 per stream: with_earth, gravity[3], iewn[3].  Returns -1 (nothing changed)
// for a non-increasing time or a mechanized window that would exceed the capacity.
int icgo_ins_push(void *p, int n_streams, const double *cfg7, const int32_t *off, const double *imu8) {
    Ins *h = (Ins *) p;
    for (int s = 0; s < n_streams; s++) {
        double prev = h->last[s];
        bool have = h->seen[s];
        for (int k = off[s]; k < off[s + 1]; k++) {
            if (have && !(imu8[8 * k] > prev)) return -1;
            prev = imu8[8 * k], have = true;
        }
        if (h->mech[s] && h->w[s].size() + (size_t) (off[s + 1] - off[s]) > (size_t) h->capacity) return -1;
    }
    for (int s = 0; s < n_streams; s++) {
        const Config config = config_of(cfg7 + 7 * s);
        Window &w = h->w[s];
        for (int k = off[s]; k < off[s + 1]; k++) {
            const IMU imu_cur = imu_of(imu8 + 8 * k);
            State state{};
            if (!w.empty()) state = w.back().second;
            const IMU imu_pre = w.empty() ? imu_cur : w.back().first;
            w.emplace_back(imu_cur, State{});
            if (h->mech[s]) {
                insMechanization(config, imu_pre, imu_cur, state);
                w.back().second = state;
            } else if (w.size() > MAXIMUM_INS_NUMBER) {
                w.pop_front();
            }
            h->last[s] = imu_cur.time, h->seen[s] = 1;
        }
    }
    return 0;
}

// redoInsMechanization per selected stream (redo NULL: all); status 1 / 0 / -1 as icg_ins_redo
void icgo_ins_redo(void *p, int n_streams, const double *cfg7, const uint8_t *redo, const double *state17, int reserved, int8_t *status) {
    Ins *h = (Ins *) p;
    for (int s = 0; s < n_streams; s++) {
        status[s] = 0;
        if (redo && !redo[s]) continue;
        State st = state_of(state17 + 17 * s);
        st.q = qnorm(st.q);  // stateFromData (preintegration_base.cc:115-125)
        const size_t index = redoInsMechanization(config_of(cfg7 + 7 * s), st, (size_t) reserved, h->w[s]);
        status[s] = index == 0 ? -1 : 1;
        if (index) h->mech[s] = 1;
    }
}

// getCameraPoseFromInsWindow per stream; found 1 / 0 / -1 as icg_ins_camera_pose
void icgo_ins_camera_pose(void *p, int n_streams, const double *stamp, const double *pose_b_c, double *pose, int32_t *found) {
    Ins *h = (Ins *) p;
    for (int s = 0; s < n_streams; s++) {
        if (!h->mech[s]) {
            found[s] = -1;
            continue;
        }
        found[s] = getCameraPoseFromInsWindow(h->w[s], pose_b_c + 12 * s, stamp[s], pose + 12 * s) ? 1 : 0;
    }
}

int icgo_ins_window(void *p, int stream, int cap, double *imu8, double *state17) {
    const Window &w = ((Ins *) p)->w[stream];
    for (size_t k = 0; k < w.size() && k < (size_t) cap; k++) imu_out(w[k].first, imu8 + 8 * k), state_out(w[k].second, state17 + 17 * k);
    return (int) w.size();
}

// one insMechanization step on state17 (in / out)
void icgo_ins_mechanize(const double *cfg7, const double *imu_pre8, const double *imu_cur8, double *state17) {
    State st = state_of(state17);
    insMechanization(config_of(cfg7), imu_of(imu_pre8), imu_of(imu_cur8), st);
    state_out(st, state17);
}

int icgo_ins_window_index(int n, const double *times, double t) {
    Window w(n);
    for (int k = 0; k < n; k++) w[k].first.time = times[k];
    return (int) getInsWindowIndex(w, t);
}

int icgo_ins_need_interpolation(double t0, double t1, double mid) {
    IMU a{}, b{};
    a.time = t0, b.time = t1;
    return isNeedInterpolation(a, b, mid);
}

void icgo_ins_interpolate(const double *imu8, double mid, double *first8, double *second8) {
    IMU a{}, b = imu_of(imu8);
    imuInterpolation(b, a, b, mid);
    imu_out(a, first8), imu_out(b, second8);
}

void icgo_ins_pose_interpolate(const double *state0, const double *state1, double mid, const double *pose_b_c, double *pose) {
    State s{};
    statePoseInterpolation(state_of(state0), state_of(state1), mid, s);
    stateToCameraPose(s, pose_b_c, pose);
}

}  // extern "C"
