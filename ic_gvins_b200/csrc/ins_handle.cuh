// ins_handle.cuh -- the INS window handle (ins.cu) as the window solve's sample store (ba_keyframe.cu) reads it: the rings, the host mirror
// of their heads and sizes, the handle's stream, and the series cut MISC::getImuSeriesFromTo (IG/misc.cc:307-361) over (stream, start, end)
// jobs.  Internal: the C ABI exposes no cut of its own.
#pragma once
#include <stdint.h>

#include <vector>

#include "common.cuh"

struct icg_ins {
    int device, max_streams, capacity;
    cudaStream_t stream;
    bool own_stream;
    double *d_imu = nullptr, *d_st = nullptr;  // stream s: rows imu[s][capacity][8] (time, dt, dtheta[3], dvel[3]), states st[s][capacity][17]
    // the host mirror: ring head and size per stream, mechanized (its first redo or initialization has run)
    std::vector<int32_t> head, count;
    std::vector<uint8_t> mech, seen;
    std::vector<double> last_time;
    // gvinsInitialization's function statics, one set per stream: bg[3], initatt[3]; is_has_zero_velocity
    std::vector<double> init_slot6;
    std::vector<int32_t> init_zv;
    double *d_series = nullptr;  // max_streams x INS_SERIES_MAX x 7, the first GNSS interval's rows (allocated by the first initialization)
    // per-call staging [jobs | doubles | ints], pinned and device, grown on demand; the asynchronous calls' copies complete at stage_ev
    uint8_t *h_stage = nullptr, *d_stage = nullptr;
    size_t stage_bytes = 0;
    cudaEvent_t stage_ev = nullptr;
    bool stage_pending = false;
};

namespace icg {

// getImuSeriesFromTo(t0, t1) of one stream's window as the host mirror has it now (head, count), written as rows (dt, dtheta[3], dvel[3])
// from row `out` of the caller's buffer.  The series has at most count + 2 rows.
struct InsCutJob {
    double t0, t1;
    int32_t stream, head, count, out;
};
// one warp per job; per job n_rows (the series' rows) and status (1, or -5: getInsWindowIndex is 0 at either end, or the series is empty --
// the rule of icg_ins_gins_initialize's status -5).  Every pointer is a device pointer of the INS handle's device.
cudaError_t ins_cut_launch(const icg_ins *h, int n_jobs, const InsCutJob *jobs, double *rows, int32_t *n_rows, int32_t *status, cudaStream_t stream);

}  // namespace icg
