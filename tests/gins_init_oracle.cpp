// gins_init_oracle.cpp -- CPU restatement of IC-GVINS' GNSS/INS initialization (TEST INFRASTRUCTURE ONLY; shares no code with ic_gvins_b200/).
// GVINS::gvinsInitialization (IG/ic_gvins.cc:584-692), MISC::detectZeroVelocity (IG/misc.cc:363-415), GVINS::constructPrior
// (ic_gvins.cc:1911-1936), MISC::getImuSeriesFromTo (misc.cc:307-361) and Earth::iewn(origin, local) (IG/common/earth.h:117-237), on the
// std::deque windows of tests/ins_oracle.cpp, which this file includes.  The preintegration of the series is left to the BA oracle
// (oracle/ba_ref.cpp), which the tests call on the series and the state this file returns.  Built by tests/gins_init_oracle.py.
#include "ins_oracle.cpp"

namespace {

constexpr double ZERO_VELOCITY_GYR_THRESHOLD = 0.002, ZERO_VELOCITY_ACC_THRESHOLD = 0.1;  // IG/misc.h:75-76
constexpr double MINMUM_ALIGN_VELOCITY = 0.5;                                             // IG/ic_gvins.h:128
const double D2R = M_PI / 180.0;
const double GYROSCOPE_BIAS_PRIOR_STD = 7200 * D2R / 3600, ACCELEROMETER_BIAS_PRIOR_STD = 20000 * 1.0e-5;  // IG/ic_gvins.h:140-141

// MISC::detectZeroVelocity
bool detectZeroVelocity(const std::vector<IMU> &buf, double rate, double *average) {
    const double size = (double) buf.size(), size_invert = 1.0 / size;
    double sum[6] = {0, 0, 0, 0, 0, 0};
    for (int k = 0; k < 6; k++) average[k] = 0;
    for (const IMU &m : buf) {
        average[0] += m.dtheta.x, average[1] += m.dtheta.y, average[2] += m.dtheta.z;
        average[3] += m.dvel.x, average[4] += m.dvel.y, average[5] += m.dvel.z;
    }
    for (int k = 0; k < 6; k++) average[k] *= size_invert;
    for (const IMU &m : buf) {
        const double v[6] = {m.dtheta.x, m.dtheta.y, m.dtheta.z, m.dvel.x, m.dvel.y, m.dvel.z};
        for (int k = 0; k < 6; k++) sum[k] += (v[k] - average[k]) * (v[k] - average[k]);
    }
    bool zero = true;
    for (int k = 0; k < 6; k++) zero = zero && sqrt(sum[k] * size_invert) * rate < (k < 3 ? ZERO_VELOCITY_GYR_THRESHOLD : ZERO_VELOCITY_ACC_THRESHOLD);
    return zero;
}

// MISC::getImuSeriesFromTo; false where the reference logs (both indices 0) or would index outside the window (either index 0, or an
// empty series), which the product reports as status -5
bool getImuSeriesFromTo(const Window &w, double start, double end, std::vector<IMU> &series) {
    const size_t is = getInsWindowIndex(w, start), ie = getInsWindowIndex(w, end);
    series.clear();
    if (is == 0 || ie == 0) return false;
    IMU imu0 = w[is - 1].first, imu1 = w[is].first, imu{};
    int isneed = isNeedInterpolation(imu0, imu1, start);
    if (isneed == -1) {
        series.push_back(imu0), series.push_back(imu1);
    } else if (isneed == 1) {
        series.push_back(imu1);
    } else if (isneed == 2) {
        imuInterpolation(imu1, imu, imu1, start);
        series.push_back(imu), series.push_back(imu1);
    }
    for (size_t k = is + 1; k + 1 < ie; k++) series.push_back(w[k].first);  // k < ie - 1
    imu0 = w[ie - 1].first, imu1 = w[ie].first;
    isneed = isNeedInterpolation(imu0, imu1, end);
    if (isneed == -1) {
        series.push_back(imu0);
    } else if (isneed == 1) {
        series.push_back(imu0), series.push_back(imu1);
    } else if (isneed == 2) {
        series.push_back(imu0);
        imuInterpolation(imu1, imu, imu1, end);
        series.push_back(imu);
    }
    if (series.empty()) return false;
    series.back().time = end;
    return true;
}

// Earth::iewn(origin, local) = iewn(local2global(origin, local)[0]): blh2ecef, cne, ecef2blh's latitude loop
V earthIewn(const double *origin, V local) {
    const double WGS84_WIE = 7.2921151467E-5, WGS84_RA = 6378137.0000000000, WGS84_E1 = 0.0066943799901413156;
    auto RN = [&](double lat) {
        const double s = sin(lat);
        return WGS84_RA / sqrt(1.0 - WGS84_E1 * s * s);
    };
    const double sinlat = sin(origin[0]), sinlon = sin(origin[1]), coslat = cos(origin[0]), coslon = cos(origin[1]);
    const double rn = RN(origin[0]), rnh = rn + origin[2];
    const V ecef0 = {rnh * coslat * coslon, rnh * coslat * sinlon, (rnh - rn * WGS84_E1) * sinlat};
    const M cn0e = {{{-sinlat * coslon, -sinlon, -coslat * coslon}, {-sinlat * sinlon, coslon, -coslat * sinlon}, {coslat, 0, -sinlat}}};
    const V e = ecef0 + mv(cn0e, local);
    const double p = sqrt(e.x * e.x + e.y * e.y);
    double lat = atan(e.z / (p * (1.0 - WGS84_E1))), h = 0, h2;
    do {
        h2 = h;
        const double r = RN(lat);
        h = p / cos(lat) - r;
        lat = atan(e.z / (p * (1.0 - WGS84_E1 * r / (r + h))));
    } while (fabs(h - h2) > 1.0e-4);
    return {WGS84_WIE * cos(lat), 0, -WGS84_WIE * sin(lat)};
}

// Rotation::euler2quaternion (IG/common/rotation.h:90-94): AngleAxis(yaw, Z) * AngleAxis(pitch, Y) * AngleAxis(roll, X)
Qd euler2quaternion(const double *e) {
    const Qd qz = {cos(0.5 * e[2]), 0, 0, sin(0.5 * e[2])}, qy = {cos(0.5 * e[1]), 0, sin(0.5 * e[1]), 0}, qx = {cos(0.5 * e[0]), sin(0.5 * e[0]), 0, 0};
    return qprod(qprod(qz, qy), qx);
}

// Eigen's q * v (_transformVector)
V qrotate(Qd q, V v) {
    const V qv = {q.x, q.y, q.z};
    V uv = crs(qv, v);
    uv = uv + uv;
    return v + q.w * uv + crs(qv, uv);
}

}  // namespace

extern "C" {

// gvinsInitialization for each selected stream (sel NULL: all) of the oracle's windows p.  in24 per stream: gnss_time, gnss_blh[3],
// last_time, last_blh[3], last_yaw_valid, last_yaw, origin[3], gravity, antlever[3], imudatarate, 6 unused.  cfg7 (in / out) as
// tests/ins_oracle.cpp's.  slot7 (in / out) per stream: bg[3], initatt[3], has_zero_velocity -- the reference's function statics.
// Per stream out: status (1, 0, -1 .. -5 as icg_ins_gins_initialize), state17 (statedatalist_[0]), priors31 (pose 7 | pose std 6 | mix 9 |
// mix std 9), series8 (max_series x 8 rows, time column included) and n_series.  gyr_bias_std = integration_parameters_->gyr_bias_std.
void icgo_gins_initialize(void *p, int n_streams, double *cfg7, const uint8_t *sel, const double *in24, double gyr_bias_std, int reserved,
                          double *slot7, int32_t *status, double *state17, double *priors31, int max_series, double *series8, int32_t *n_series) {
    Ins *h = (Ins *) p;
    for (int s = 0; s < n_streams; s++) {
        status[s] = 0, n_series[s] = 0;
        if (sel && !sel[s]) continue;
        const double *g = in24 + 24 * s;
        const double gnss_time = g[0], last_time = g[4], gravity = g[13], rate = g[17];
        const V gnss_blh = {g[1], g[2], g[3]}, last_blh = {g[5], g[6], g[7]}, antlever = {g[14], g[15], g[16]};
        double *bg = slot7 + 7 * s, *initatt = bg + 3;
        Window &w = h->w[s];
        if (gnss_time == 0 || last_time == 0) {
            status[s] = -1;
            continue;
        }
        std::vector<IMU> imu_buff;
        for (const auto &ins : w)
            if (ins.first.time > last_time && ins.first.time < gnss_time) imu_buff.push_back(ins.first);
        if (imu_buff.size() < 20) {
            status[s] = -2;
            continue;
        }
        double average[6];
        if (detectZeroVelocity(imu_buff, rate, average)) {
            for (int k = 0; k < 3; k++) bg[k] = average[k] * rate;
            const double fb[3] = {average[3] * rate, average[4] * rate, average[5] * rate};
            initatt[0] = -asin(fb[1] / gravity), initatt[1] = asin(fb[0] / gravity);
            slot7[7 * s + 6] = 1;
            status[s] = -3;
            continue;
        }
        double att[3] = {initatt[0], initatt[1], initatt[2]};
        if (g[8] != 0) {
            att[2] = g[9];
        } else {
            const V vel = gnss_blh - last_blh;
            if (nrm(vel) < MINMUM_ALIGN_VELOCITY) {
                status[s] = -4;
                continue;
            }
            if (slot7[7 * s + 6] == 0) att[0] = 0, att[1] = atan(-vel.z / sqrt(vel.x * vel.x + vel.y * vel.y));
            att[2] = atan2(vel.y, vel.x);
        }
        // the window after the redo must serve the series: try both on a copy first (status -5 leaves everything as it was)
        const Qd q = euler2quaternion(att);
        State st{last_time, last_blh - qrotate(q, antlever), q, {0, 0, 0}, {bg[0], bg[1], bg[2]}, {0, 0, 0}};
        Config config = config_of(cfg7 + 7 * s);
        config.gravity = {0, 0, gravity};
        if (config.earth) config.iewn = earthIewn(g + 10, st.p);
        Window redone = w;
        State from = st;
        from.q = qnorm(from.q);  // stateFromData (preintegration_base.cc:115-125)
        std::vector<IMU> series;
        if (redoInsMechanization(config, from, (size_t) reserved, redone) == 0 || !getImuSeriesFromTo(redone, last_time, gnss_time, series)) {
            status[s] = -5;
            continue;
        }
        w.swap(redone);
        h->mech[s] = 1;
        for (int k = 0; k < 3; k++) initatt[k] = att[k];
        double *c = cfg7 + 7 * s;
        c[1] = config.gravity.x, c[2] = config.gravity.y, c[3] = config.gravity.z;
        if (config.earth) c[4] = config.iewn.x, c[5] = config.iewn.y, c[6] = config.iewn.z;
        state_out(st, state17 + 17 * s);
        // constructPrior(is_has_zero_velocity)
        double *pr = priors31 + 31 * s;
        const double att_std = 0.5 * D2R, bg_std = slot7[7 * s + 6] != 0 ? gyr_bias_std * 3 : GYROSCOPE_BIAS_PRIOR_STD;
        memcpy(pr, state17 + 17 * s + 1, sizeof(double) * 7), memcpy(pr + 13, state17 + 17 * s + 8, sizeof(double) * 9);
        for (int k = 0; k < 3; k++) {
            pr[7 + k] = 0.1, pr[10 + k] = att_std;
            pr[22 + k] = 0.1, pr[25 + k] = bg_std, pr[28 + k] = ACCELEROMETER_BIAS_PRIOR_STD;
        }
        pr[12] = att_std * 3;
        status[s] = 1;
        n_series[s] = (int32_t) series.size();
        for (size_t k = 0; k < series.size() && (int) k < max_series; k++) imu_out(series[k], series8 + 8 * ((size_t) max_series * s + k));
    }
}

void icgo_earth_iewn(const double *origin3, const double *local3, double *iewn3) {
    const V v = earthIewn(origin3, V{local3[0], local3[1], local3[2]});
    iewn3[0] = v.x, iewn3[1] = v.y, iewn3[2] = v.z;
}

void icgo_euler2quaternion(const double *euler3, double *q_xyzw) {
    const Qd q = euler2quaternion(euler3);
    q_xyzw[0] = q.x, q_xyzw[1] = q.y, q_xyzw[2] = q.z, q_xyzw[3] = q.w;
}

}  // extern "C"
