// ins_series_oracle.cpp -- MISC::getImuSeriesFromTo (IG/misc.cc:307-361) of the CPU restatement (tests/gins_init_oracle.cpp, which this
// file includes with tests/ins_oracle.cpp) on any interval of an oracle window (TEST INFRASTRUCTURE ONLY).  Built by tests/ins_series_oracle.py.
#include "gins_init_oracle.cpp"

extern "C" {

// the series of stream `stream` from start to end: rows (time, dt, dtheta[3], dvel[3]) into series8 (max rows); returns its row count, or -1
// where the product refuses the interval (either window index 0, or an empty series)
int icgo_imu_series(void *p, int stream, double start, double end, int max, double *series8) {
    std::vector<IMU> series;
    if (!getImuSeriesFromTo(((Ins *) p)->w[stream], start, end, series)) return -1;
    for (size_t k = 0; k < series.size() && (int) k < max; k++) imu_out(series[k], series8 + 8 * k);
    return (int) series.size();
}

}  // extern "C"
