// ba.cu -- Path B: batched sliding-window factor-graph solve on sm_90a.
//
// Replaces `ceres::Solver::Solve` (LEVENBERG_MARQUARDT + DENSE_SCHUR, IG/ic_gvins.cc:1143-1146,1183,1217) and the
// per-factor `CostFunction::Evaluate` calls Ceres drives (IG/factors/*.h, IG/preintegration/*.h) for MANY independent
// windows at once (throughput mode: one window per stream).  Ceres is an un-vendored dependency of the reference; the
// trust-region loop restated here follows its published algorithm and the defaults the reference leaves untouched.
//
// Device-resident LM: the host only enqueues a fixed kernel sequence per iteration; every decision (step validity,
// accept/reject, radius update, convergence) is taken on the device in per-window LM state.
//
// Per window: n = 15K+7 camera-side columns laid out [pose_0..pose_{K-1} (6 each) | extrinsic 6 | td 1 | mix_0..mix_{K-1} (9 each)];
// the vision factors only touch the first NCV = 6K+7 ("vision columns").  Landmarks (inverse depths) are eliminated:
//   lin_vis    : CTA / run of landmarks of one reference node: thread / reprojection factor -> residual, local Jacobians, Huber
//                correction -> record in shared memory; per (reference node, observing node) pair the 20x20 Gram matrix of the run's
//                records on the FP64 tensor cores (DMMA.8x8x4), summed over the node's runs in run order;
//                lanes / landmark -> h_l, g_l and the dense coupling row w_l (A_W, landmark-major)
//   schur_dmma : cluster of 4 CTAs / window: sum_l phi_l w_l w_l^T with phi_l = s_l^2 / (s_l^2 h_l + D_l^2) on the FP64 tensor cores, one
//                landmark split per CTA, the partials summed over DSMEM; epilogue: one-writer-per-entry gather of the pair Gram matrices
//                into the vision part of H_cc and g_c -> Hs = H_c + H_vis - Schur term and the solve's vision vectors (or the split
//                pipeline's export payload)
//   lin_cam    : one CTA / window (second stream, beside the vision chain) -> IMU preintegration, GNSS, bias, prior and
//                marginalization factors -> H_c, g_c
//   solve      : one CTA / window -> Jacobi scaling, LM diagonal, S = s(H - Schur)s + D^2, packed Cholesky in shared memory
//                (panel updates on DMMA), triangular solves, landmark back-substitution, model cost change, candidate x (+) delta
//   single GPU : lin_vis + lin_cam at the candidate, into the window's second linearisation buffer (its costs are the candidate cost)
//   cost       : candidate cost (all factors, residuals only) of the split pipeline;   accept : Ceres step acceptance + radius update
//   ba_marg.cuh: sliding-window marginalization (MarginalizationInfo) on the same device-resident linearisation
#include <cooperative_groups.h>
#include <unistd.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <functional>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include "ba_cull.cuh"
#include "ba_slide.cuh"
#include "ba_vision.cuh"
#include "preint.cuh"
#include "ba_math.cuh"
#include "common.cuh"
#include "geom_core.cuh"

namespace icg {
using namespace bam;
namespace cg = cooperative_groups;

constexpr int BA_SPLIT_W = 4;   // row splits of the Schur SYRK = CTAs of its cluster (partials summed in fixed order -> deterministic)
constexpr int BA_CHOL_NB = 8;   // Cholesky block width
constexpr int BA_MARG_MAXB = 72;  // remained blocks of a prior: <= 2 max_K + 2 = 66 at max_K = 32 (table stride)
constexpr int BA_MAX_NODES = 32;  // icg_ba_create: max_K <= 32

struct BaCaps {
    int NW, K, L, F, G, R;     // capacities
    int NCV, N, NS, NCA, RJ, LP, NVB;  // derived strides: NCV = 6K+7, N = 15K+7, NS = N padded, NCA = roundup4(NCV+1), RJ = 2F padded, LP = L padded
    int GQ;                            // Gram partials per window: one per (lin_vis run, observing node) <= min(F, runs x (K - 1))
};

struct WinDims {  // per-window actual sizes
    int K, L, F, n_imu, n_gnss, marg_r, marg_nb;
    int ext_const, td_const, reproj_huber, gnss_huber, has_imu_error, has_pose_prior, has_mix_prior;
    double reproj_sinv;
};

struct LmState {
    double radius, decrease_factor, x_cost, x_norm, cand_cost, model_cost_change, step_norm, gmax, initial_cost;
    double cost_cam[2];  // camera-only cost of each linearisation buffer
    int iter, n_success, n_invalid, done, need_lin, last_success, first, step_valid, fresh_lin, max_iter, chol_ok;
    int lin_buf;  // linearisation buffer that holds the linearisation at x (the other one receives the candidate's)
};

// Exchange state of the split pipeline (ba_split.cuh): one buffer per rank holding the inbox of reduction operands, the step broadcast, the
// scalar exchange and the epoch flags; `peer[r]` is rank r's buffer as mapped into this process (peer memory, CUDA IPC or same process)
struct ShardDev {
    int split;                 // 1: the split pipeline drives this handle (large systems and / or landmark shards)
    int PK, BS, RV;            // packed partial length, step-broadcast stride, reduced-vector stride (doubles)
    double *peer[8];
    size_t off_inbox, off_bcast, off_scal, off_flagA, off_flagB, off_flagC;  // offsets in doubles, identical on every rank
    size_t off_flagX, off_post, off_exp;  // the post-solve exchanges of a shard group (ba_split.cuh); off_exp: sized by this rank's max_F
    double *redv;              // [NW][RV] owner-side reduced vectors: diag H_vis | g_vis | W phi g_l | cost, sum rho^2, max |g_l|
    int *err;                  // device error word (flag wait timed out)
    double *slm;               // [NW][STEP_SLICES][8] partial sums of ba_step_lm's landmark slices
    int *slm_cnt;              // [NW] slices arrived (resets itself)
};

struct BaDev {  // device pointers (flat, capacity-strided by window)
    ShardDev S;
    WinDims *dims;
    LmState *st;
    double *pose, *mix, *ext, *rho;          // current parameters
    double *pose_c, *mix_c, *ext_c, *rho_c;  // candidate
    double *pose_0, *mix_0, *ext_0, *rho_0;  // initial copy (for re-running the same problem: bench)
    uint8_t *f_active_0;                     // pristine copies of what the two-pass protocol mutates (restart re-solves the UPLOADED problem)
    double *gnss_std_0;
    uint8_t *f_active;                       // by factor id
    // landmark POSITIONS: the window's landmarks ordered by reference node, stable by id (landmarks without factors last); record slots
    // follow that order.  Arrays indexed by landmark id (rho, h_l, g_l, scale_l, A_W rows) keep the id.
    int *lm_off;  // CSR offsets of the factor records by landmark position
    int *lm_perm; // [NW][L] landmark id at each position
    int *vb_lm0;  // [NW][NVB] first landmark position of every lin_vis run (whole landmarks of ONE reference node, <= 128 factors); last entry = run count
    int *ref_nrun;       // [NW][K] lin_vis runs per reference node
    int *f_meta_s;       // per record slot: (landmark, reference node, observing node, factor id)
    double *f_const_s;   // per record slot: the factor's 14 constants (copy of f_const in slot order)
    int *vis_ord;        // per record slot: the run's slots ordered by observing node (stable): run-local slot | Gram partial index << 8
    int *part_off, *pair_ro, *npairs;  // (reference node, observing node) pairs: CSR offsets of their Gram partials (in run order), (ref << 8 | obs), count
    double *gpart;       // [NW][GQ][210] Gram partial of one (run, observing node): packed upper 20x20
    int *vis_cnt;        // [NW][K] lin_vis runs of the reference node arrived (the last one resets it)
    // Linearisation buffers: everything a linearisation writes and a later iteration reads comes in two copies, selected per window by
    // LmState::lin_buf through the lin_* helpers below.  The single-GPU pipeline linearises the candidate into the copy the window is not
    // using and flips lin_buf when ba_accept takes the step; the split pipeline never flips it and has copy 0 only.
    double *Mp[2];         // per-pair 20x20 Gram matrices (upper, 210 entries)
    double *AW[2];         // Schur SYRK input
    double *costf[2];      // per-factor cost
    double *hl[2], *gl[2];
    double *Hc[2], *gc[2];
    double *scale_l, *scale_c;
    double *Hs;  // H_c + vision Gram - Schur term (lower triangle, ld NS): the operand ba_solve scales and factorises
    double *visv;  // [NW][3 NCV] diag H_vis | g_vis | W phi g_l (window NCV): ba_solve's other operands (single GPU)
    double *imu_blob, *imu_U;
    int *gnss_node;
    double *gnss_blh, *gnss_std, *lever;
    double *pose_prior, *pose_prior_sinfo, *mix_prior, *mix_prior_std;
    int *marg_type, *marg_node;
    double *marg_x0, *marg_H0, *marg_b0, *marg_c0;
    double *cost_part;  // [NW][ncost_blocks]
    double *red2;       // [NW][4]: model cost change, step norm^2, non-finite count of the step (+ the split pipeline's fourth exchanged partial)
    int rank, world;    // landmark shard of this process (camera-only terms are counted on rank 0 only)
    double *step_c, *step_l;
    double *Sglobal;    // fallback Cholesky workspace when the packed system does not fit shared memory
    unsigned long long *clk;  // ICG_BA_PROFILE: SM-clock totals of ba_solve's phases for window 0 (nullptr otherwise)
};

// window w's part of linearisation buffer b
__device__ __forceinline__ double *lin_Mp(const BaCaps &C, const BaDev &D, int b, int w) { return D.Mp[b] + (size_t) w * C.K * (C.K - 1) * 210; }
__device__ __forceinline__ double *lin_AW(const BaCaps &C, const BaDev &D, int b, int w) { return D.AW[b] + (size_t) w * C.LP * C.NCA; }
__device__ __forceinline__ double *lin_costf(const BaCaps &C, const BaDev &D, int b, int w) { return D.costf[b] + (size_t) w * C.F; }
__device__ __forceinline__ double *lin_hl(const BaCaps &C, const BaDev &D, int b, int w) { return D.hl[b] + (size_t) w * C.L; }
__device__ __forceinline__ double *lin_gl(const BaCaps &C, const BaDev &D, int b, int w) { return D.gl[b] + (size_t) w * C.L; }
__device__ __forceinline__ double *lin_Hc(const BaCaps &C, const BaDev &D, int b, int w) { return D.Hc[b] + (size_t) w * C.NS * C.NS; }
__device__ __forceinline__ double *lin_gc(const BaCaps &C, const BaDev &D, int b, int w) { return D.gc[b] + (size_t) w * C.NS; }

__device__ __forceinline__ int col_pose(int k) { return 6 * k; }
__device__ __forceinline__ int col_ext(int K) { return 6 * K; }
__device__ __forceinline__ int col_td(int K) { return 6 * K + 6; }
__device__ __forceinline__ int col_mix(int K, int k) { return 6 * K + 7 + 9 * k; }

// ------------------------------------------------------------------------------------------------ lin_vis (+ landmark rows)
__device__ __forceinline__ int jc_off(int a) { return a < 18 ? (a / 6) * 12 + (a % 6) : 36 + 2 * (a - 18); }  // row 0 offset in a record
__device__ __forceinline__ int jc_row1(int a) { return a < 18 ? 6 : 1; }                                           // + this for row 1
__device__ __forceinline__ int tri20(int la, int lb) {  // index of (la <= lb) in the packed upper 20x20
    return la * 20 - la * (la - 1) / 2 + (lb - la);
}
__device__ __forceinline__ void dmma884(double &c0, double &c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
// One CTA linearises a run of WHOLE landmarks of ONE reference node (<= 128 reprojection factors; the host packs the runs at upload).
//  phase 1: thread / factor, in record slot order -> residual, local Jacobians, Huber correction -> 40-double record
//           [Ji 12 | Jj 12 | Je 12 | Jt 2 | r 2] + [j_rho 2 | observing node | reference node], staged in shared memory;
//  phase 2: the Gram matrices of the run.  Within a (reference node, observing node) pair every factor has the same 19 camera-side columns
//           [ref pose 6 | obs pose 6 | extrinsic 6 | td 1] (+ the residual as a 20th column), so the pair's contribution is the dense
//           20x20 Gram matrix X^T X of its stacked 2x20 rows: one warp per observing node of the run, 4 rows (2 factors) per DMMA.8x8x4
//           k-step.  With the m8n8k4 fragment layout (A: lane -> (row lane/4, k lane%4); B: lane -> (k lane%4, col lane/4)) the A and
//           B operands of X^T X are the SAME register: lane loads X[k = lane%4][8 t + lane/4] for the three column tiles t and issues
//           the six upper-triangular tile products.  The packed result is the run's partial of that pair (D.gpart);
//  phase 3: eight lanes per landmark reduce its records, straight from shared memory, to h_l, g_l and the coupling row
//           w_l[c] = sum_f J_f[:, c]^T j_rho,f of A_W (landmark-major [l][NCA]: zeroed, then the <= 13 + 6 n_obs non-zeros).  All
//           factors of a landmark share the reference node, the extrinsic and td (accumulated); each observing node appears once
//           (written directly; icg_ba_upload checks it);
//  phase 4: the last run of the reference node to arrive (arrival counter) sums the node's partials of every pair in run order -> Mp.
//           No floating-point atomics: the result does not depend on which CTA arrives last, nor on the other windows of the batch.
// The Jacobians never leave the SM: per factor only the cost is stored.
// at_cand = 0: at x (windows that need a linearisation) into buffer lin_buf; at_cand = 1: at the candidate of a valid step into buffer
// 1 - lin_buf (its per-factor costs are the candidate cost ba_accept tests).
constexpr int LV_LD = 45;  // shared-memory record row: 44 doubles padded to an odd length (conflict-free)
constexpr size_t LV_SMEM = sizeof(double) * (128 * LV_LD + (BA_MAX_NODES + 1) * NODE_FRAME_LD);  // records + node frames (49.5 KB: dynamic, opted in at create)
__global__ void __launch_bounds__(128, 4) ba_lin_vis(BaCaps C, BaDev D, int at_cand) {
    extern __shared__ double lv_sm[];
    __shared__ int s_ord[128], s_gbeg[BA_MAX_NODES], s_gend[BA_MAX_NODES], s_last, s_p0, s_np;
    double (*s_rec)[LV_LD] = (double (*)[LV_LD]) lv_sm;
    double (*s_frame)[NODE_FRAME_LD] = (double (*)[NODE_FRAME_LD]) (lv_sm + 128 * LV_LD);
    const int w = blockIdx.y;
    const LmState &st = D.st[w];
    if (st.done || !(at_cand ? st.step_valid : st.need_lin)) return;
    const int b = at_cand ? 1 - st.lin_buf : st.lin_buf;
    const double *pose = at_cand ? D.pose_c : D.pose, *xext = at_cand ? D.ext_c : D.ext, *rho = at_cand ? D.rho_c : D.rho;
    const int *vb = D.vb_lm0 + (size_t) w * C.NVB;
    if ((int) blockIdx.x >= vb[C.NVB - 1]) return;  // last entry = number of runs of this window
    const WinDims dm = D.dims[w];
    const int tid = threadIdx.x;
    const int *off = D.lm_off + (size_t) w * (C.L + 1);
    const int pA = vb[blockIdx.x], pB = vb[blockIdx.x + 1];  // landmark positions of the run
    const int s0 = off[pA], nslot = off[pB] - s0;
    // ---- phase 0: the window's K + 1 node frames (rotation matrix | position of every pose and of the extrinsic), once per CTA
    if (tid <= dm.K) node_frame(tid < dm.K ? pose + ((size_t) w * C.K + tid) * 7 : xext + (size_t) w * 8, s_frame[tid]);
    if (tid < BA_MAX_NODES) s_gbeg[tid] = s_gend[tid] = 0;
    if (tid == 0) s_np = 0;
    __syncthreads();
    // ---- phase 1
    if (tid < nslot) {
        const int q = s0 + tid;
        double r[2], Ji[12], Jj[12], Je[12], Jr[2], Jt[2], cost = 0;
        const int4 meta = ((const int4 *) D.f_meta_s)[(size_t) w * C.F + q];  // (landmark, reference node, observing node, factor id)
        const int i = meta.y, j = meta.z, f = meta.w;
        if (D.f_active[(size_t) w * C.F + f] != 0) {
            const double *ext = xext + (size_t) w * 8;
            reproj_eval_frames(s_frame[i], s_frame[j], s_frame[dm.K], rho[(size_t) w * C.L + meta.x], ext[7],
                               D.f_const_s + ((size_t) w * C.F + q) * 14, dm.reproj_sinv, true, r, Ji, Jj, Je, Jr, Jt);
            if (dm.ext_const)
                for (int k = 0; k < 12; k++) Je[k] = 0;
            if (dm.td_const) Jt[0] = Jt[1] = 0;
            double sq = r[0] * r[0] + r[1] * r[1], sc = 1.0;
            if (dm.reproj_huber)
                huber(sq, cost, sc);
            else
                cost = 0.5 * sq;
            if (sc != 1.0) {
                for (int k = 0; k < 12; k++) Ji[k] *= sc, Jj[k] *= sc, Je[k] *= sc;
                Jr[0] *= sc, Jr[1] *= sc, Jt[0] *= sc, Jt[1] *= sc, r[0] *= sc, r[1] *= sc;
            }
        } else {
            for (int k = 0; k < 12; k++) Ji[k] = Jj[k] = Je[k] = 0;
            Jr[0] = Jr[1] = Jt[0] = Jt[1] = r[0] = r[1] = 0;
        }
        lin_costf(C, D, b, w)[f] = cost;
        double *sr = s_rec[tid];
#pragma unroll
        for (int k = 0; k < 12; k++) sr[k] = Ji[k], sr[12 + k] = Jj[k], sr[24 + k] = Je[k];
        sr[36] = Jt[0], sr[37] = Jt[1], sr[38] = r[0], sr[39] = r[1];
        sr[40] = Jr[0], sr[41] = Jr[1], sr[42] = (double) j, sr[43] = (double) i;
    }
    __syncthreads();
    // ---- phase 2
    const int lane = tid & 31, warp = tid >> 5;
    if (nslot > 0) {
        if (tid < nslot) {  // slots [s_gbeg[o], s_gend[o]) of s_ord observe from node o
            const int *ord = D.vis_ord + (size_t) w * C.F + s0;
            const int v = ord[tid], ob = (int) s_rec[v & 255][42];
            s_ord[tid] = v;
            if (tid == 0 || (int) s_rec[ord[tid - 1] & 255][42] != ob) s_gbeg[ob] = tid;
            if (tid == nslot - 1 || (int) s_rec[ord[tid + 1] & 255][42] != ob) s_gend[ob] = tid + 1;
        }
        __syncthreads();
        const int kk = lane & 3, g = lane >> 2;  // k index inside the step (factor kk/2, residual row kk%2), column inside the tile
        int o[3];
#pragma unroll
        for (int t = 0; t < 3; t++) {
            const int a = 8 * t + g;
            o[t] = a < 20 ? jc_off(a) + (kk & 1) * jc_row1(a) : -1;
        }
        for (int ob = warp; ob < dm.K; ob += 4) {
            const int beg = s_gbeg[ob], end = s_gend[ob];
            if (beg == end) continue;
            double c00[2] = {0, 0}, c01[2] = {0, 0}, c02[2] = {0, 0}, c11[2] = {0, 0}, c12[2] = {0, 0}, c22[2] = {0, 0};
            constexpr int UNR = 2;  // k-steps in flight (4 factors)
            for (int base = beg; base < end; base += 2 * UNR) {
                double x[UNR][3];
#pragma unroll
                for (int u = 0; u < UNR; u++) {
                    const int q = base + 2 * u + (kk >> 1);
                    const bool ok = q < end;
                    const double *rec = s_rec[ok ? s_ord[q] & 255 : 0];
#pragma unroll
                    for (int t = 0; t < 3; t++) x[u][t] = (ok && o[t] >= 0) ? rec[o[t]] : 0.0;
                }
#pragma unroll
                for (int u = 0; u < UNR; u++) {
                    dmma884(c00[0], c00[1], x[u][0], x[u][0]);
                    dmma884(c01[0], c01[1], x[u][0], x[u][1]);
                    dmma884(c02[0], c02[1], x[u][0], x[u][2]);
                    dmma884(c11[0], c11[1], x[u][1], x[u][1]);
                    dmma884(c12[0], c12[1], x[u][1], x[u][2]);
                    dmma884(c22[0], c22[1], x[u][2], x[u][2]);
                }
            }
            // C fragment: lane holds (row lane/4, cols 2 (lane%4) + {0,1}) of each 8x8 tile
            double *pp = D.gpart + ((size_t) w * C.GQ + (s_ord[beg] >> 8)) * 210;
            auto put = [&](int ti, int tj, const double *c) {
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int la = 8 * ti + g, lb = 8 * tj + 2 * kk + e;
                    if (la <= lb && lb < 20) pp[tri20(la, lb)] = c[e];
                }
            };
            put(0, 0, c00), put(0, 1, c01), put(0, 2, c02), put(1, 1, c11), put(1, 2, c12), put(2, 2, c22);
        }
        __threadfence();  // the partials are visible device-wide before this run is counted (phase 4)
    }
    // ---- phase 3
    const int *perm = D.lm_perm + (size_t) w * C.L;
    const int K = dm.K, NCV = 6 * K + 7, NCA = 4 * ((NCV + 1 + 3) / 4);
    const int grp = tid >> 3, sl = tid & 7;
    int o0[3], o1[3];
#pragma unroll
    for (int t = 0; t < 3; t++) {
        const int c = sl + 8 * t;  // 0..23; 19 -> residual pair (g_l); 20 -> h_l from j_rho; > 20 unused
        o0[t] = c < 19 ? jc_off(c) : 38, o1[t] = c < 19 ? o0[t] + jc_row1(c) : 39;
    }
    for (int pl = pA + grp; pl < pB; pl += 16) {
        const int l = perm[pl], f0 = off[pl] - s0, nf = off[pl + 1] - off[pl];
        double *row = lin_AW(C, D, b, w) + (size_t) l * C.NCA;
        for (int c = sl; c < NCA; c += 8) row[c] = 0.0;
        __syncwarp(0xffu << (tid & 24));  // the landmark's eight lanes: zeros land before the values
        double acc[3] = {0, 0, 0};
        for (int q = 0; q < nf; q++) {
            const double *rec = s_rec[f0 + q];
            const double r0 = rec[40], r1 = rec[41];
            const int ob = (int) rec[42];
#pragma unroll
            for (int t = 0; t < 3; t++) {
                const int c = sl + 8 * t;
                if (c == 20) {
                    acc[t] += r0 * r0 + r1 * r1;
                } else if (c < 20) {
                    const double v = rec[o0[t]] * r0 + rec[o1[t]] * r1;
                    if (c >= 6 && c < 12)
                        row[col_pose(ob) + c - 6] = v;
                    else
                        acc[t] += v;
                }
            }
        }
        const int ref = nf > 0 ? (int) s_rec[f0][43] : 0;
#pragma unroll
        for (int t = 0; t < 3; t++) {
            const int c = sl + 8 * t;
            if (nf > 0) {
                if (c < 6) row[col_pose(ref) + c] = acc[t];
                else if (c >= 12 && c < 18) row[col_ext(K) + c - 12] = acc[t];
                else if (c == 18) row[col_td(K)] = acc[t];
            }
            if (c == 19) {
                row[NCV] = acc[t];
                lin_gl(C, D, b, w)[l] = acc[t];
            } else if (c == 20) {
                lin_hl(C, D, b, w)[l] = acc[t];
                if (st.first) D.scale_l[(size_t) w * C.L + l] = 1.0 / (1.0 + sqrt(acc[t]));  // jacobi_scaling, once (iteration 0)
            }
        }
    }
    // ---- phase 4
    if (nslot == 0) return;  // a run of landmarks without factors: no pair
    const int rn = (int) s_rec[0][43];
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(D.vis_cnt + (size_t) w * C.K + rn, 1) == D.ref_nrun[(size_t) w * C.K + rn] - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (tid == 0) D.vis_cnt[(size_t) w * C.K + rn] = 0;
    const int PM = C.K * (C.K - 1), P = D.npairs[w];
    const int *pro = D.pair_ro + (size_t) w * PM, *poff = D.part_off + (size_t) w * (PM + 1);
    for (int p = tid; p < P; p += 128)  // the node's pairs are consecutive (pairs are ordered by reference node)
        if ((pro[p] >> 8) == rn) {
            atomicAdd(&s_np, 1);
            if (p == 0 || (pro[p - 1] >> 8) != rn) s_p0 = p;
        }
    __syncthreads();
    const double *part = D.gpart + (size_t) w * C.GQ * 210;
    double *Mp = lin_Mp(C, D, b, w);
    for (int p = s_p0 + warp; p < s_p0 + s_np; p += 4) {  // warp / pair: the 7 entries of a lane in flight together
        const int k0 = poff[p], k1 = poff[p + 1];
        double acc[7];
#pragma unroll
        for (int j = 0; j < 7; j++) acc[j] = lane + 32 * j < 210 ? __ldcg(part + (size_t) k0 * 210 + lane + 32 * j) : 0.0;
        for (int k = k0 + 1; k < k1; k++) {
            double v[7];
#pragma unroll
            for (int j = 0; j < 7; j++) v[j] = lane + 32 * j < 210 ? __ldcg(part + (size_t) k * 210 + lane + 32 * j) : 0.0;
#pragma unroll
            for (int j = 0; j < 7; j++) acc[j] += v[j];
        }
#pragma unroll
        for (int j = 0; j < 7; j++)
            if (lane + 32 * j < 210) Mp[(size_t) p * 210 + lane + 32 * j] = acc[j];
    }
}

// ------------------------------------------------------------------------------------------------ pair_gram: vision part of H_cc, g_c
// ba_lin_vis leaves one packed 20x20 Gram matrix per (reference node, observing node) pair in Mp; the epilogue of ba_schur_dmma gathers
// them (thread / output entry) into the symmetric (NCV+1)^2 matrix [H_vis g_vis; g_vis^T r^T r].  No atomics: every output has one writer.

// gather of one entry (A <= B) of the symmetric (NCV+1)^2 matrix [H_vis g_vis; g_vis^T r^T r] from the per-pair Gram matrices: the groups
// that touch both of its blocks
__device__ __forceinline__ void gram2_slots(const BaCaps &C, const BaDev &D, int w, int K, short *s_slot) {
    const int PM = C.K * (C.K - 1), P = D.npairs[w];
    const int *pro = D.pair_ro + (size_t) w * PM;
    for (int e = threadIdx.x; e < K * K; e += blockDim.x) s_slot[e] = -1;
    __syncthreads();
    for (int p = threadIdx.x; p < P; p += blockDim.x) s_slot[(pro[p] >> 8) * K + (pro[p] & 255)] = (short) p;
    __syncthreads();
}
__device__ __forceinline__ double gram2_entry(const BaCaps &C, const BaDev &D, int buf, int w, int K, const short *s_slot, int A, int B) {
    const int P = D.npairs[w];
    const double *Mp = lin_Mp(C, D, buf, w);
    const int bA = A < 6 * K ? A / 6 : K, bB = B < 6 * K ? B / 6 : K;
    const int a = A - 6 * bA, b = B - 6 * bB;  // offsets inside the block (global block: 0..7 = ext 6, td, residual)
    const int ga = 12 + a, gb = 12 + b;          // local column of a global-block column
    double sum = 0;
    if (bA == K) {  // (global, global): every group
        // up to K (K - 1) groups: sixteen loads in flight and four partial sums in a fixed order, group p into sum p mod 4 (these 36 entries
        // are the tail of the epilogue: a serial sum is 90 dependent L2 round trips)
        const int idx = tri20(ga, gb);
        double s4[4] = {0, 0, 0, 0};
        int p = 0;
        for (; p + 16 <= P; p += 16) {
            double v[16];
#pragma unroll
            for (int u = 0; u < 16; u++) v[u] = Mp[(size_t) (p + u) * 210 + idx];
#pragma unroll
            for (int u = 0; u < 16; u++) s4[u & 3] += v[u];
        }
        for (; p < P; p++) s4[p & 3] += Mp[(size_t) p * 210 + idx];
        sum = (s4[0] + s4[1]) + (s4[2] + s4[3]);
    } else if (bB == K || bB == bA) {  // (pose, global) or the pose's diagonal block
        const int i1 = tri20(a, bB == K ? gb : b), i2 = tri20(6 + a, bB == K ? gb : 6 + b);
        // 16 loads in flight; same summation order as a serial loop (a missing pair or o >= K adds +0.0, which leaves a sum that started
        // at +0.0 unchanged)
        for (int o0 = 0; o0 < K; o0 += 8) {
            double v1[8], v2[8];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int o = o0 + u;
                const int p1 = o < K ? s_slot[bA * K + o] : -1, p2 = o < K ? s_slot[o * K + bA] : -1;  // bA as reference node / as observing node
                v1[u] = p1 >= 0 ? Mp[(size_t) p1 * 210 + i1] : 0.0;
                v2[u] = p2 >= 0 ? Mp[(size_t) p2 * 210 + i2] : 0.0;
            }
#pragma unroll
            for (int u = 0; u < 8; u++) sum += v1[u], sum += v2[u];
        }
    } else {  // two different poses: the (bA -> bB) and (bB -> bA) groups
        const int p1 = s_slot[bA * K + bB], p2 = s_slot[bB * K + bA];
        if (p1 >= 0) sum += Mp[(size_t) p1 * 210 + tri20(a, 6 + b)];
        if (p2 >= 0) sum += Mp[(size_t) p2 * 210 + tri20(b, 6 + a)];
    }
    return sum;
}

// ------------------------------------------------------------------------------------------------ Schur term + reduced camera system
__device__ __forceinline__ double block_sum(double v, double *s_red);
__device__ __forceinline__ double block_max(double v, double *s_red);
__device__ __forceinline__ double *x_inbox(const BaDev &D, int peer, int w, int from);  // ba_split.cuh
__device__ __forceinline__ int tri_idx(int A, int B, int ncv);

// Entry (A <= B <= NCV) of the vision Gram matrix (cj, gathered here from Mp) and of the Schur term (cw): stores what the solve of the
// pipeline that drives the handle reads.
//   single GPU (fused pipeline): Hs = H_c + (cj - cw) on the vision rows (lower triangle) and D.visv = [diag H_vis | g_vis | W phi g_l];
//   split pipeline: [tri(H_vis - Schur) | diag H_vis | g_vis | W phi g_l] straight into the owner's inbox (P2P stores; ba_signal publishes
//                   them, the owner's ba_reduce sums the ranks).
__device__ __forceinline__ void schur_store(const BaCaps &C, const BaDev &D, int buf, int w, int K, const short *s_slot, int A, int B, double cw) {
    const int NCV = 6 * K + 7;
    if (A == NCV) return;  // the r^T r corner: no solve reads it
    const size_t e = (size_t) w * C.NS * C.NS + (size_t) B * C.NS + A;
    const double hc = !D.S.split && B < NCV ? lin_Hc(C, D, buf, w)[(size_t) B * C.NS + A] : 0.0;  // in flight during the gather
    const double cj = gram2_entry(C, D, buf, w, K, s_slot, A, B);
    if (D.S.split) {
        double *P = x_inbox(D, w % D.world, w, D.rank);
        const int TRI = NCV * (NCV + 1) / 2;
        if (B < NCV) {
            P[tri_idx(A, B, NCV)] = cj - cw;
            if (A == B) P[TRI + A] = cj;
        } else {
            P[TRI + NCV + A] = cj;       // g_vis
            P[TRI + 2 * NCV + A] = cw;   // W phi g_l
        }
    } else {
        double *V = D.visv + (size_t) w * 3 * C.NCV;
        if (B < NCV) {
            D.Hs[e] = hc + (cj - cw);
            if (A == B) V[A] = cj;
        } else {
            V[NCV + A] = cj, V[2 * NCV + A] = cw;
        }
    }
}

// the scalars of the split payload: vision cost, sum rho^2 and max |g_l| over this rank's factors and landmarks (one CTA)
__device__ __forceinline__ void schur_scalars(const BaCaps &C, const BaDev &D, int w, const WinDims &dm, double *s_red) {
    const int tid = threadIdx.x;
    double c = 0, q = 0, gm = 0;
    const double *costf = lin_costf(C, D, 0, w), *gl = lin_gl(C, D, 0, w);  // the split pipeline uses buffer 0 only
    for (int f = tid; f < dm.F; f += 256) c += costf[f];
    for (int l = tid; l < dm.L; l += 256) {
        const double r = D.rho[(size_t) w * C.L + l];
        q += r * r;
        gm = fmax(gm, fabs(gl[l]));
    }
    c = block_sum(c, s_red);
    q = block_sum(q, s_red);
    gm = block_max(gm, s_red);
    if (tid != 0) return;
    const int NCV = 6 * dm.K + 7, TRI = NCV * (NCV + 1) / 2;
    double *P = x_inbox(D, w % D.world, w, D.rank);
    P[TRI + 3 * NCV] = c, P[TRI + 3 * NCV + 1] = q, P[TRI + 3 * NCV + 2] = gm;
}

// Schur SYRK on the FP64 tensor cores: the sum over the window's landmarks of phi_l w_l w_l^T, with
// phi_l = s_l^2 / (s_l^2 h_l + clamp(s_l^2 h_l) / radius) the LM-damped landmark pivot.  DMMA.8x8x4 with k = 4 landmarks per step; as in
// ba_lin_vis's Gram phase the A and B fragments of X^T X share one layout: lane reads A_W[l0 + lane%4][8 t + lane/4].  The CTA stages its
// landmark rows (and phi) in shared memory once per pass -- leading dimension = 8 mod 16 doubles, so a fragment read is the minimal
// two wavefronts -- and every warp accumulates two 16x16 super-tiles (2x2 DMMA tiles each) of the upper triangle per pass.
// One thread-block CLUSTER of BA_SPLIT_W CTAs per window: CTA k accumulates the partial of landmark split k.  After each pass (16
// super-tiles) every CTA puts its partials in shared memory over its staging rows, which the pass no longer needs; after a cluster barrier
// each CTA owns a quarter of the pass's super-tiles, sums the BA_SPLIT_W partials of an entry over DSMEM in split order starting from 0.0
// (deterministic) and hands the entry to schur_store.  The partials never leave the cluster.
constexpr int SCHUR_RCH = 80;  // landmark rows staged per chunk (multiple of 4)
constexpr int SCHUR_PASS = 16;  // super-tiles per pass
__global__ void __cluster_dims__(BA_SPLIT_W, 1, 1) __launch_bounds__(256) ba_schur_dmma(BaCaps C, BaDev D, int ld) {
    extern __shared__ double sA[];  // [SCHUR_RCH][ld] rows, then phi[SCHUR_RCH]; between passes: [SCHUR_PASS][256] partials
    __shared__ short s_slot[32 * 32];
    __shared__ double s_red[40];
    cg::cluster_group cluster = cg::this_cluster();
    const int w = blockIdx.y, split = blockIdx.x;  // cluster rank = split
    const LmState &st = D.st[w];
    if (st.done) return;  // per window: the whole cluster leaves
    const WinDims dm = D.dims[w];
    const int NCV = 6 * dm.K + 7, NCA = 4 * ((NCV + 1 + 3) / 4);
    const int T2 = (NCA + 15) / 16, nsuper = T2 * (T2 + 1) / 2;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, kk = lane & 3;
    double *sphi = sA + (size_t) SCHUR_RCH * ld;
    const int b = st.lin_buf;
    const double *A = lin_AW(C, D, b, w), *hl = lin_hl(C, D, b, w);
    const double radius = st.radius;
    const int nsteps = (dm.L + 3) / 4;
    const int r_beg = 4 * (int) ((long long) nsteps * split / BA_SPLIT_W), r_end = min(dm.L, 4 * (int) ((long long) nsteps * (split + 1) / BA_SPLIT_W));
    const int npass = (nsuper + SCHUR_PASS - 1) / SCHUR_PASS;
    gram2_slots(C, D, w, dm.K, s_slot);
    for (int pass = 0; pass < npass; pass++) {
        if (pass > 0) cluster.barrier_wait();  // the peers have read this CTA's partials of the previous pass: its staging rows are free
        int si[2], sj[2];
        bool on[2];
#pragma unroll
        for (int h2 = 0; h2 < 2; h2++) {
            const int su = (2 * pass + h2) * 8 + warp;
            on[h2] = su < nsuper;
            int a = 0, e = on[h2] ? su : 0;
            while (e >= T2 - a) e -= T2 - a, a++;
            si[h2] = a, sj[h2] = a + e;
        }
        double acc[2][4][2];
#pragma unroll
        for (int h2 = 0; h2 < 2; h2++)
#pragma unroll
            for (int q = 0; q < 4; q++) acc[h2][q][0] = acc[h2][q][1] = 0;
        for (int r0 = r_beg; r0 < r_end; r0 += SCHUR_RCH) {
            const int nr = min(SCHUR_RCH, r_end - r0), nr4 = (nr + 3) & ~3;
            __syncthreads();
            for (int rb = warp; rb < nr4; rb += 8 * 4) {  // warp stages rows rb, rb + 8, rb + 16, rb + 24: 4 rows x 3 column chunks in flight
                double v[4][3];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int rr = rb + 8 * u;
#pragma unroll
                    for (int cchunk = 0; cchunk < 3; cchunk++) {
                        const int c = lane + 32 * cchunk;
                        v[u][cchunk] = (rr < nr && c < NCA) ? A[(size_t) (r0 + rr) * C.NCA + c] : 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int rr = rb + 8 * u;
#pragma unroll
                    for (int cchunk = 0; cchunk < 3; cchunk++) {
                        const int c = lane + 32 * cchunk;
                        if (rr < nr4 && c < ld) sA[(size_t) rr * ld + c] = v[u][cchunk];
                    }
                }
                for (int c = lane + 96; c < ld; c += 32)  // wider rows (K > 12): remaining columns
                    for (int u = 0; u < 4; u++) {
                        const int rr = rb + 8 * u;
                        if (rr < nr4) sA[(size_t) rr * ld + c] = (rr < nr && c < NCA) ? A[(size_t) (r0 + rr) * C.NCA + c] : 0.0;
                    }
            }
            for (int rr = tid; rr < nr4; rr += 256) {
                double ph = 0;
                if (rr < nr) {
                    const int l = r0 + rr;
                    const double sl = D.scale_l[(size_t) w * C.L + l], hs = sl * sl * hl[l];
                    ph = sl * sl / (hs + fmin(fmax(hs, 1e-6), 1e32) / radius);
                }
                sphi[rr] = ph;
            }
            __syncthreads();
            for (int ks = 0; ks < nr4 / 4; ks++) {
                const double *row = sA + (size_t) (4 * ks + kk) * ld;
                const double ph = sphi[4 * ks + kk];
#pragma unroll
                for (int h2 = 0; h2 < 2; h2++) {
                    if (!on[h2]) continue;
                    const double xb0 = row[16 * sj[h2] + g], xb1 = row[16 * sj[h2] + 8 + g];
                    const double a0 = row[16 * si[h2] + g] * ph, a1 = row[16 * si[h2] + 8 + g] * ph;
                    dmma884(acc[h2][0][0], acc[h2][0][1], a0, xb0);
                    dmma884(acc[h2][1][0], acc[h2][1][1], a0, xb1);
                    dmma884(acc[h2][2][0], acc[h2][2][1], a1, xb0);
                    dmma884(acc[h2][3][0], acc[h2][3][1], a1, xb1);
                }
            }
        }
        __syncthreads();  // every warp is done with the staged rows
        // super-tile (2 pass + h2) * 8 + warp -> slot h2 * 8 + warp, in C-fragment order: position 64 q + 32 e + lane holds (row g, col
        // 2 kk + e) of DMMA tile q (conflict-free stores, and reads below)
#pragma unroll
        for (int h2 = 0; h2 < 2; h2++) {
            if (!on[h2]) continue;
#pragma unroll
            for (int q = 0; q < 4; q++)
#pragma unroll
                for (int e = 0; e < 2; e++) sA[(h2 * 8 + warp) * 256 + 64 * q + 32 * e + lane] = acc[h2][q][e];
        }
        cluster.sync();  // every split's partials of this pass are in place
        // CTA `split` owns slots split, split + 4, ...; thread tid owns position tid of each
        const int nslot = min(SCHUR_PASS, nsuper - SCHUR_PASS * pass);
        double cw[SCHUR_PASS / BA_SPLIT_W];
#pragma unroll
        for (int j = 0; j < SCHUR_PASS / BA_SPLIT_W; j++) {
            const int sl = split + BA_SPLIT_W * j;
            double p[BA_SPLIT_W];
#pragma unroll
            for (int k = 0; k < BA_SPLIT_W; k++) p[k] = sl < nslot ? cluster.map_shared_rank(sA, k)[sl * 256 + tid] : 0.0;
            cw[j] = 0;
#pragma unroll
            for (int k = 0; k < BA_SPLIT_W; k++) cw[j] += p[k];
        }
        cluster.barrier_arrive();  // done reading the peers (the matching wait comes before this CTA's shared memory is reused or released)
        const int q = tid >> 6, r_in = 8 * (q >> 1) + ((tid & 31) >> 2), c_in = 8 * (q & 1) + 2 * (tid & 3) + ((tid >> 5) & 1);
#pragma unroll
        for (int j = 0; j < SCHUR_PASS / BA_SPLIT_W; j++) {
            const int sl = split + BA_SPLIT_W * j;
            if (sl >= nslot) break;
            int a = 0, e = SCHUR_PASS * pass + sl;
            while (e >= T2 - a) e -= T2 - a, a++;
            const int r = 16 * a + r_in, cc = 16 * (a + e) + c_in;
            if (r <= cc && cc <= NCV) schur_store(C, D, b, w, dm.K, s_slot, r, cc, cw[j]);
        }
    }
    if (split == 0 && D.S.split) schur_scalars(C, D, w, dm, s_red);
    cluster.barrier_wait();  // no CTA leaves while a peer may still read its shared memory
}

// ------------------------------------------------------------------------------------------------ camera-only factors
constexpr double IMU_GB_STD = 7200 / 3600.0 * 3.14159265358979323846 / 180.0;  // IG/preintegration/imu_error_factor.h:89-91
constexpr double IMU_AB_STD = 2.0e4 * 1.0e-5;

// one warp evaluates one IMU factor: whitened residual rw[15] and (optionally) whitened local Jacobian Jw[15x30] in shared memory
__device__ void imu_factor_warp(const double *blob, const double *U, const double *pose0, const double *mix0, const double *pose1,
                                const double *mix1, bool want_j, double *rw, double *Jw, int lane) {
    __shared__ ImuMid s_mid[16];
    double *raw_r = rw + 15;  // scratch behind rw (caller provides 30 doubles)
    const int wslot = (threadIdx.x >> 5) & 15;
    if (want_j)
        for (int e = lane; e < 450; e += 32) Jw[e] = 0;
    __syncwarp();
    if (lane == 0) {
        ImuMid M;
        imu_residual_raw(blob, pose0, mix0, pose1, mix1, raw_r, M);
        if (want_j) imu_jacobian_raw(blob, M, Jw);
        s_mid[wslot] = M;
    }
    __syncwarp();
    // whitening by the upper-triangular sqrt information: out[i] = sum_{k >= i} U[i][k] in[k]  (in place, rows ascending)
    if (want_j && lane < 30) {
        for (int i = 0; i < 15; i++) {
            double s = 0;
            for (int k = i; k < 15; k++) s += U[i * 15 + k] * Jw[k * 30 + lane];
            Jw[i * 30 + lane] = s;
        }
    }
    if (lane < 15) {
        double s = 0;
        for (int k = lane; k < 15; k++) s += U[lane * 15 + k] * raw_r[k];
        rw[lane] = s;
    }
    __syncwarp();
}

// marginalization prior (IG/factors/marginalization_factor.h:47-101): dx of every remained block
__device__ void marg_dx(const BaCaps &C, const BaDev &D, int w, const WinDims &dm, const double *pose, const double *mix, const double *ext, double *dx,
                        int *colmap, int tid, int nthreads) {
    const int *type = D.marg_type + (size_t) w * BA_MARG_MAXB, *node = D.marg_node + (size_t) w * BA_MARG_MAXB;
    const double *x0 = D.marg_x0 + (size_t) w * BA_MARG_MAXB * 9;
    if (tid == 0) {
        int col = 0, xo = 0;
        for (int b = 0; b < dm.marg_nb; b++) {
            int t = type[b], nd = node[b];
            if (t == 0 || t == 2) {
                const double *x = t == 0 ? pose + nd * 7 : ext;
                const double *xl = x0 + xo;
                Q dq = qmul(qinv(pose_q(xl)), pose_q(x));
                V3 a = 2.0 * qv(dq);
                if (dq.w < 0) a = -a;
                for (int k = 0; k < 3; k++) dx[col + k] = x[k] - xl[k];
                dx[col + 3] = a.x, dx[col + 4] = a.y, dx[col + 5] = a.z;
                int base = t == 0 ? col_pose(nd) : col_ext(dm.K);
                for (int k = 0; k < 6; k++) colmap[col + k] = (t == 2 && dm.ext_const) ? -1 : base + k;
                col += 6, xo += 7;
            } else if (t == 1) {
                for (int k = 0; k < 9; k++) dx[col + k] = mix[nd * 9 + k] - x0[xo + k], colmap[col + k] = col_mix(dm.K, nd) + k;
                col += 9, xo += 9;
            } else {
                dx[col] = ext[7] - x0[xo];
                colmap[col] = dm.td_const ? -1 : col_td(dm.K);
                col += 1, xo += 1;
            }
        }
    }
}

// cost of all camera-only factors at (pose, mix, ext); optionally the linearisation (H_c, g_c of buffer b).  One CTA (256 threads).
// smem: per IMU factor 30 + 450 doubles; GNSS 3 + 18 each; misc.
// x += v on a global accumulator whose value the thread does not need back: one fire-and-forget reduction at the L2 (RED.ADD.F64) instead of a
// load -> add -> store chain (a dependent L2 round trip per entry: measured 50 k of ba_lin_cam's 123 k cycles in the IMU block accumulation).
// Every entry has ONE writer per phase and the phases are separated by block barriers, so the summation order is fixed (deterministic).
__device__ __forceinline__ void red_add(double *p, double v) { asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory"); }

__device__ double cam_factors(const BaCaps &C, const BaDev &D, int w, const WinDims &dm, const double *pose, const double *mix, const double *ext,
                              bool lin, int b, double *smem) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const int K = dm.K, N = 15 * K + 7;
    double *Hc = lin_Hc(C, D, b, w), *gc = lin_gc(C, D, b, w);
    double *s_imu = smem;                              // n_imu * 480
    double *s_gnss = s_imu + (size_t) C.K * 480;       // G * 24 : r[3] J[18] cost scale
    double *s_misc = s_gnss + (size_t) C.G * 24;       // pose prior r[6] J[36] | mix prior r[9] | marg dx[R] y[R] | costs
    double *s_pp = s_misc, *s_mp = s_misc + 48, *s_dx = s_mp + 16, *s_y = s_dx + C.R, *s_cost = s_y + C.R;
    int *s_colmap = (int *) (s_cost + 8);
    __shared__ double s_total;
#ifdef ICG_BA_PHASE_CLOCKS
    unsigned long long cclk = D.clk ? clock64() : 0ull;  // profiling build: phase clocks of the linearising call, window 0
#define CAM_CLK(k)                                                 \
    if (D.clk && lin && w == 0 && tid == 0) {                      \
        const unsigned long long t_ = clock64();                   \
        atomicAdd(&D.clk[16 + (k)], t_ - cclk), atomicAdd(&D.clk[24 + (k)], 1ull); \
        cclk = t_;                                                 \
    }
#else
#define CAM_CLK(k)
#endif
    // ---- phase 1: evaluate
    for (int k = warp; k < dm.n_imu; k += nwarps)
        imu_factor_warp(D.imu_blob + ((size_t) w * C.K + k) * ICG_IMU_BLOB_DOUBLES, D.imu_U + ((size_t) w * C.K + k) * 225, pose + k * 7, mix + k * 9,
                        pose + (k + 1) * 7, mix + (k + 1) * 9, lin, s_imu + (size_t) k * 480, s_imu + (size_t) k * 480 + 30, lane);
    if (tid < dm.n_gnss) {
        const int nd = D.gnss_node[(size_t) w * C.G + tid];
        double *o = s_gnss + tid * 24;
        gnss_eval(pose + nd * 7, D.gnss_blh + ((size_t) w * C.G + tid) * 3, D.gnss_std + ((size_t) w * C.G + tid) * 3, D.lever + (size_t) w * 3, lin, o, o + 3);
        double sq = o[0] * o[0] + o[1] * o[1] + o[2] * o[2], cost, sc = 1.0;
        if (dm.gnss_huber)
            huber(sq, cost, sc);
        else
            cost = 0.5 * sq;
        if (sc != 1.0) {
            for (int e = 0; e < 3; e++) o[e] *= sc;
            if (lin)
                for (int e = 0; e < 18; e++) o[3 + e] *= sc;
        }
        o[21] = cost;
    }
    if (tid == 64 && dm.has_pose_prior) pose_prior_eval(pose, D.pose_prior + (size_t) w * 7, D.pose_prior_sinfo + (size_t) w * 6, lin, s_pp, s_pp + 6);
    if (tid == 96 && dm.has_mix_prior)
        for (int k = 0; k < 9; k++) s_mp[k] = (mix[k] - D.mix_prior[(size_t) w * 9 + k]) / D.mix_prior_std[(size_t) w * 9 + k];
    if (dm.marg_r > 0) marg_dx(C, D, w, dm, pose, mix, ext, s_dx, s_colmap, tid, blockDim.x);
    __syncthreads();
    CAM_CLK(0)  // factor evaluation
    const double *H0 = D.marg_H0 + (size_t) w * C.R * C.R, *b0 = D.marg_b0 + (size_t) w * C.R;
    if (dm.marg_r > 0) {
        for (int i = tid; i < dm.marg_r; i += blockDim.x) {
            double s = 0;
            for (int k = 0; k < dm.marg_r; k++) s += H0[(size_t) i * dm.marg_r + k] * s_dx[k];
            s_y[i] = s;
        }
    }
    __syncthreads();
    // ---- cost (single thread, fixed order -> deterministic)
    if (tid == 0) {
        double c = 0;
        for (int k = 0; k < dm.n_imu; k++) {
            const double *r = s_imu + (size_t) k * 480;
            double sq = 0;
            for (int e = 0; e < 15; e++) sq += r[e] * r[e];
            c += 0.5 * sq;
        }
        for (int g = 0; g < dm.n_gnss; g++) c += s_gnss[g * 24 + 21];
        if (dm.has_imu_error) {
            const double *m = mix + dm.n_imu * 9;
            double sq = 0;
            for (int e = 0; e < 3; e++) sq += (m[3 + e] / IMU_GB_STD) * (m[3 + e] / IMU_GB_STD) + (m[6 + e] / IMU_AB_STD) * (m[6 + e] / IMU_AB_STD);
            c += 0.5 * sq;
        }
        if (dm.has_pose_prior) {
            double sq = 0;
            for (int e = 0; e < 6; e++) sq += s_pp[e] * s_pp[e];
            c += 0.5 * sq;
        }
        if (dm.has_mix_prior) {
            double sq = 0;
            for (int e = 0; e < 9; e++) sq += s_mp[e] * s_mp[e];
            c += 0.5 * sq;
        }
        if (dm.marg_r > 0) {
            // 0.5 |e0 + J0 dx|^2 = 0.5 (e0.e0 + 2 b0.dx + dx.H0.dx)
            double q = D.marg_c0[w];
            for (int i = 0; i < dm.marg_r; i++) q += (2.0 * b0[i] + s_y[i]) * s_dx[i];
            c += 0.5 * q;
        }
        s_total = c;
    }
    if (!lin) {
        __syncthreads();
        return s_total;
    }
    CAM_CLK(1)  // prior product + cost
    // ---- phase 2: H_c = sum J^T J, g_c = sum J^T r   (every entry has exactly one writer per round -> deterministic)
    for (int e = tid; e < N * C.NS; e += blockDim.x) Hc[e] = 0;
    for (int e = tid; e < N; e += blockDim.x) gc[e] = 0;
    __syncthreads();
    CAM_CLK(2)  // zero H_c
    if (dm.marg_r > 0) {
        const int r = dm.marg_r;
        for (int e = tid; e < r * r; e += blockDim.x) {
            int i = e / r, j = e - i * r;
            int ci = s_colmap[i], cj = s_colmap[j];
            if (ci >= 0 && cj >= 0) Hc[(size_t) ci * C.NS + cj] = H0[e];
        }
        for (int i = tid; i < r; i += blockDim.x)
            if (s_colmap[i] >= 0) gc[s_colmap[i]] = b0[i] + s_y[i];
    }
    __syncthreads();
    CAM_CLK(3)  // prior blocks
    for (int parity = 0; parity < 2; parity++) {  // IMU factors k and k+2 touch disjoint nodes
        const int nf = (dm.n_imu - parity + 1) / 2;
        for (int e = tid; e < nf * 930; e += blockDim.x) {
            const int k = parity + 2 * (e / 930), q = e % 930;
            const double *rw = s_imu + (size_t) k * 480, *Jw = rw + 30;
            auto gcol = [&](int c) { return c < 6 ? col_pose(k) + c : c < 15 ? col_mix(K, k) + c - 6 : c < 21 ? col_pose(k + 1) + c - 15 : col_mix(K, k + 1) + c - 21; };
            if (q < 900) {
                int a = q / 30, b = q - a * 30;
                double s = 0;
                for (int m = 0; m < 15; m++) s += Jw[m * 30 + a] * Jw[m * 30 + b];
                red_add(&Hc[(size_t) gcol(a) * C.NS + gcol(b)], s);
            } else {
                int a = q - 900;
                double s = 0;
                for (int m = 0; m < 15; m++) s += Jw[m * 30 + a] * rw[m];
                red_add(&gc[gcol(a)], s);
            }
        }
        __syncthreads();
    }
    CAM_CLK(4)  // IMU J^T J
    // pose-diagonal blocks: GNSS + pose prior; mix-diagonal: bias-magnitude factor + mix prior
    for (int e = tid; e < K * 42; e += blockDim.x) {
        const int k = e / 42, q = e % 42;
        double s = 0;
        if (q < 36) {
            const int a = q / 6, b = q % 6;
            for (int g = 0; g < dm.n_gnss; g++)
                if (D.gnss_node[(size_t) w * C.G + g] == k) {
                    const double *J = s_gnss + g * 24 + 3;
                    s += J[a] * J[b] + J[6 + a] * J[6 + b] + J[12 + a] * J[12 + b];
                }
            if (k == 0 && dm.has_pose_prior)
                for (int m = 0; m < 6; m++) s += s_pp[6 + m * 6 + a] * s_pp[6 + m * 6 + b];
            red_add(&Hc[(size_t) (col_pose(k) + a) * C.NS + col_pose(k) + b], s);
        } else {
            const int a = q - 36;
            for (int g = 0; g < dm.n_gnss; g++)
                if (D.gnss_node[(size_t) w * C.G + g] == k) {
                    const double *o = s_gnss + g * 24;
                    s += o[3 + a] * o[0] + o[9 + a] * o[1] + o[15 + a] * o[2];
                }
            if (k == 0 && dm.has_pose_prior)
                for (int m = 0; m < 6; m++) s += s_pp[6 + m * 6 + a] * s_pp[m];
            red_add(&gc[col_pose(k) + a], s);
        }
    }
    if (tid < 9) {
        if (dm.has_imu_error && tid >= 3) {
            const int k = dm.n_imu;
            const double sd = tid < 6 ? IMU_GB_STD : IMU_AB_STD;
            Hc[(size_t) (col_mix(K, k) + tid) * C.NS + col_mix(K, k) + tid] += 1.0 / (sd * sd);
            gc[col_mix(K, k) + tid] += mix[k * 9 + tid] / (sd * sd);
        }
    }
    __syncthreads();
    if (tid < 9 && dm.has_mix_prior) {
        const double sd = D.mix_prior_std[(size_t) w * 9 + tid];
        Hc[(size_t) (col_mix(K, 0) + tid) * C.NS + col_mix(K, 0) + tid] += 1.0 / (sd * sd);
        gc[col_mix(K, 0) + tid] += s_mp[tid] / sd;
    }
    __syncthreads();
    CAM_CLK(5)  // GNSS / prior diagonal blocks
#undef CAM_CLK
    return s_total;
}

constexpr int CAM_THREADS = 320;  // 10 warps: the K - 1 = 9 IMU factors of a 10-node window are evaluated in one round (warp per factor)
// at_cand: as ba_lin_vis
__global__ void __launch_bounds__(CAM_THREADS) ba_lin_cam(BaCaps C, BaDev D, int at_cand) {
    extern __shared__ double smem[];
    const int w = blockIdx.x;
    LmState &st = D.st[w];
    if (st.done || !(at_cand ? st.step_valid : st.need_lin)) return;
    if (D.S.split && (w % D.world) != D.rank) return;  // split pipeline: the window's owner handles the camera-only factors
    const WinDims dm = D.dims[w];
    const int b = at_cand ? 1 - st.lin_buf : st.lin_buf;
    const double *pose = at_cand ? D.pose_c : D.pose, *mix = at_cand ? D.mix_c : D.mix, *ext = at_cand ? D.ext_c : D.ext;
    double c = cam_factors(C, D, w, dm, pose + (size_t) w * C.K * 7, mix + (size_t) w * C.K * 9, ext + (size_t) w * 8, true, b, smem);
    if (threadIdx.x == 0) st.cost_cam[b] = c;
}

// ------------------------------------------------------------------------------------------------ solve (one CTA per window)
constexpr int SOLVE_THREADS = 256;  // 2 CTAs (windows) per SM: 107 KB shared memory and <= 128 registers each

__device__ __forceinline__ double block_sum(double v, double *s_red) {
    // deterministic block reduction (fixed tree)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    double t = 0;
    if (tid == 0) {
        for (int k = 0; k < (int) (blockDim.x >> 5); k++) t += s_red[k];
        s_red[32] = t;
    }
    __syncthreads();
    return s_red[32];
}
__device__ __forceinline__ double block_max(double v, double *s_red) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, o));
    __syncthreads();
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    if (tid == 0) {
        double t = 0;
        for (int k = 0; k < (int) (blockDim.x >> 5); k++) t = fmax(t, s_red[k]);
        s_red[32] = t;
    }
    __syncthreads();
    return s_red[32];
}

__global__ void __launch_bounds__(SOLVE_THREADS, 2) ba_solve(BaCaps C, BaDev D) {
    extern __shared__ double sm[];
    const int w = blockIdx.x, tid = threadIdx.x;
    LmState &st = D.st[w];
    if (st.done) return;
    // phase clocks (profiling BUILD only, -DICG_BA_PHASE_CLOCKS: the instrumentation perturbs register allocation): thread 0 of window 0 adds
    // the SM cycles since the previous mark
#ifdef ICG_BA_PHASE_CLOCKS
    unsigned long long clk_prev = D.clk ? clock64() : 0ull;
#define SOLVE_CLK(k)                                              \
    if (D.clk && w == 0 && tid == 0) {                            \
        const unsigned long long t_ = clock64();                  \
        atomicAdd(&D.clk[k], t_ - clk_prev), atomicAdd(&D.clk[8 + (k)], 1ull); \
        clk_prev = t_;                                            \
    }
#define SOLVE_CLK_NOW() (D.clk ? clock64() : 0ull)
#define SOLVE_CLK_ADD(k, t0)                                      \
    if (D.clk && w == 0 && tid == 0) atomicAdd(&D.clk[k], clock64() - (t0)), atomicAdd(&D.clk[8 + (k)], 1ull);
#else
#define SOLVE_CLK(k)
#define SOLVE_CLK_NOW() 0ull
#define SOLVE_CLK_ADD(k, t0)
#endif
    const WinDims dm = D.dims[w];
    const int K = dm.K, L = dm.L, NCV = 6 * K + 7, N = 15 * K + 7;
    const int f_first = st.first, f_fresh = st.fresh_lin, f_last = st.last_success, f_iter = st.iter;
    const double f_gmax_old = st.gmax;
    (void) f_gmax_old;
    // shared layout: vectors first, packed matrix last
    double *s_red = sm;                 // 40
    double *s_scale = s_red + 40;       // N
    double *s_g = s_scale + C.NS;       // N   full camera gradient (unscaled)
    double *s_rhs = s_g + C.NS;         // N   -> step' (scaled space)
    double *s_d2 = s_rhs + C.NS;        // N
    double *s_diag = s_d2 + C.NS;       // N   Cholesky diagonal
    // packed lower triangle, N + 1 rows, ALWAYS in shared memory (systems that do not fit are driven by the split pipeline, ba_solve_cam): a
    // pointer that could also be global made every access a generic LD / ST (longer latency, long-scoreboard tracked)
    double *S = s_diag + C.NS;
    const int b = st.lin_buf;
    const double *Hc = lin_Hc(C, D, b, w), *gcam = lin_gc(C, D, b, w), *Hs = D.Hs + (size_t) w * C.NS * C.NS;
    // Vision vectors [diag H_vis | g_vis | W phi g_l] (a < NCV), as ba_schur_dmma's epilogue wrote them.
    const double *V = D.visv + (size_t) (3 * C.NCV) * w;
    if (tid == 0 && st.need_lin) st.need_lin = 0;      // the linearisation kernels of this iteration have run (stream order)
    double *scale_c = D.scale_c + (size_t) w * C.NS;
    const double *hl = lin_hl(C, D, b, w), *gl = lin_gl(C, D, b, w), *scale_l = D.scale_l + (size_t) w * C.L;

    // ---- after a fresh linearisation: total cost, gradient, (first time) Jacobi scaling
    for (int a = tid; a < N; a += SOLVE_THREADS) {
        double g = gcam[a];
        if (a < NCV) g += V[NCV + a];
        s_g[a] = g;
        if (f_first) {
            double h = Hc[(size_t) a * C.NS + a] + (a < NCV ? V[a] : 0.0);
            scale_c[a] = 1.0 / (1.0 + sqrt(h));
        }
    }
    __syncthreads();
    for (int a = tid; a < N; a += SOLVE_THREADS) s_scale[a] = scale_c[a];
    double gmax_now = st.gmax;
    if (f_fresh) {
        double cs = 0, gq = 0;
        const double *costf = lin_costf(C, D, b, w);
        for (int f = tid; f < dm.F; f += SOLVE_THREADS) cs += costf[f];
        for (int l = tid; l < L; l += SOLVE_THREADS) gq = fmax(gq, fabs(gl[l]));
        const double c = block_sum(cs, s_red), gml = block_max(gq, s_red);
        double gm = 0;
        for (int a = tid; a < N; a += SOLVE_THREADS) gm = fmax(gm, fabs(s_g[a]));
        gm = fmax(block_max(gm, s_red), gml);
        gmax_now = gm;
        if (tid == 0) {
            st.x_cost = c + st.cost_cam[b];
            st.gmax = gm;
            if (f_first) st.initial_cost = st.x_cost;
            st.fresh_lin = 0;
        }
        __syncthreads();
    }
    if (f_first) {
        __syncthreads();
        if (tid == 0) st.first = 0;
    }
    // ---- TrustRegionMinimizer::FinalizeIterationAndCheckIfMinimizerCanContinue
    {
        int term = 0;
        if (f_iter >= st.max_iter) term = 1;                                    // NO_CONVERGENCE
        else if (f_last && gmax_now <= 1e-10) term = 2;                         // gradient tolerance
        else if (f_last && st.radius <= 1e-32) term = 2;                        // min trust region radius
        if (term) {
            __syncthreads();
            if (tid == 0) st.done = term, st.step_valid = 0;
            return;
        }
    }
    __syncthreads();
    if (tid == 0) st.iter++;
    const double radius = st.radius;
    SOLVE_CLK(0)  // gradient, cost, termination tests

    // ---- assemble S' = s (H - Schur) s + D^2 (packed lower), rhs' = -s (g - W phi g_l)
    // The reduced camera matrix (Hs, row i contiguous) goes global -> packed shared rows with 8-byte cp.async: every element of
    // the lower triangle is in flight at once (one L2 round trip for the whole matrix instead of one per row and warp), the vector part below
    // overlaps the copy, and the Jacobi scaling + LM diagonal are applied in place afterwards.
    constexpr bool async_fill = true;
    if (async_fill) {
        for (int i = tid >> 5; i < N; i += SOLVE_THREADS / 32) {
            const double *src = (i < NCV ? Hs : Hc) + (size_t) i * C.NS;
            const unsigned dst = (unsigned) __cvta_generic_to_shared(S + i * (i + 1) / 2);
            for (int j = tid & 31; j <= i; j += 32)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst + 8u * j), "l"(src + j) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    for (int a = tid; a < N; a += SOLVE_THREADS) {
        double h = Hc[(size_t) a * C.NS + a] + (a < NCV ? V[a] : 0.0);
        double hs = s_scale[a] * s_scale[a] * h;
        s_d2[a] = fmin(fmax(hs, 1e-6), 1e32) / radius;
        double gw = a < NCV ? V[2 * NCV + a] : 0.0;
        s_rhs[a] = -s_scale[a] * (s_g[a] - gw);
    }
    if (async_fill) asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
    if (async_fill) {
        for (int i = tid >> 5; i < N; i += SOLVE_THREADS / 32) {
            double *row = S + i * (i + 1) / 2;
            const double si = s_scale[i];
            for (int j = tid & 31; j <= i; j += 32) {
                double v = si * s_scale[j] * row[j];
                if (i == j) v += s_d2[i];
                row[j] = v;
            }
        }
    } else {
        for (int i = tid >> 5; i < N; i += SOLVE_THREADS / 32) {
            // one warp per row; all global loads of the row are issued before the first store (memory-level parallelism)
            constexpr int MAXQ = 16;  // N <= 512
            double hv[MAXQ];
            const int nq = i / 32 + 1;
#pragma unroll
            for (int q = 0; q < MAXQ; q++) {
                const int j = (tid & 31) + 32 * q;
                hv[q] = 0;
                if (q < nq && j <= i) hv[q] = (i < NCV ? Hs : Hc)[(size_t) i * C.NS + j];  // Hs: H_c + vision Gram - Schur (vision rows); row i contiguous
            }
#pragma unroll
            for (int q = 0; q < MAXQ; q++) {
                const int j = (tid & 31) + 32 * q;
                if (q < nq && j <= i) {
                    double v = s_scale[i] * s_scale[j] * hv[q];
                    if (i == j) v += s_d2[i];
                    S[i * (i + 1) / 2 + j] = v;
                }
            }
        }
    }
    // augmented row N = rhs': the factorisation then leaves y = L^-1 rhs' in it (forward substitution for free)
    for (int a = tid; a < N; a += SOLVE_THREADS) S[N * (N + 1) / 2 + a] = s_rhs[a];
    __syncthreads();
    SOLVE_CLK(1)  // assembly
    // ---- blocked left-looking Cholesky on the packed lower triangle (two barriers per 8 columns); failure -> invalid step.
    // Per panel J (columns J0 .. J0 + 7):
    //   (1) panel update with all previous columns on the FP64 tensor cores, S[J0:, J0:J0+8] -= L[J0:, :J0] L[J0:J0+8, :J0]^T, one warp per
    //       8-row tile (A fragment = L[i0 + g][k0 + kk], B fragment = L[J0 + g][k0 + kk], DMMA.8x8x4, J0 % 8 == 0).  WARP 0 takes the
    //       diagonal tile alone and FACTORS it straight away (in registers: the 8-column pivot chain, ~8 x (DFMA + rsqrt + DMUL) = 600 cycles of
    //       pure latency) while warps 1..7 are still updating the tiles below -- the chain hides behind their tensor-core work.  (The
    //       previous version let every thread factor the block redundantly to save a barrier: measured, a barrier costs ~30 cycles here,
    //       the redundant factorisation ~3 000 issue slots per panel -- 58 % of the kernel.)
    //   (2) barrier; every row below the block (and the augmented rhs row) is solved against the factored block by its own thread; barrier.
    // 1/sqrt(d) comes from rsqrt (one dependent op per column instead of sqrt + divide); the row solve multiplies by it.
    __shared__ int s_fail;
    if (tid == 0) s_fail = 0;
    __syncthreads();
    const int NR = N + 1;
    for (int J0 = 0; J0 < N; J0 += BA_CHOL_NB) {
        const int nb = min(BA_CHOL_NB, N - J0);
        const int lane = tid & 31, warp = tid >> 5, g = lane >> 2, kk = lane & 3;
        const int ntile = (NR - J0 + 7) / 8;
        const unsigned long long pc0 = SOLVE_CLK_NOW();  // profiling: warp 0's own work / the row-solve phase of this panel
        (void) pc0;
        const int cb = J0 + g;                                     // row of L that is the B operand's column
        const double *rb = S + (cb < NR ? cb * (cb + 1) / 2 : 0);
        const bool okb = cb < NR;
        if (warp == 0) {
            if (J0 > 0) {  // diagonal tile: rows J0 + g; four accumulator chains over the k range
                const double *ra = rb;
                double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                int k0 = 0;
                for (; k0 + 16 <= J0; k0 += 16) {
                    const double x0 = okb ? ra[k0 + kk] : 0.0, x1 = okb ? ra[k0 + 4 + kk] : 0.0, x2 = okb ? ra[k0 + 8 + kk] : 0.0, x3 = okb ? ra[k0 + 12 + kk] : 0.0;
                    dmma884(acc[0], acc[1], x0, x0);
                    dmma884(acc[2], acc[3], x1, x1);
                    dmma884(acc[4], acc[5], x2, x2);
                    dmma884(acc[6], acc[7], x3, x3);
                }
                for (; k0 + 8 <= J0; k0 += 8) {
                    const double x0 = okb ? ra[k0 + kk] : 0.0, x1 = okb ? ra[k0 + 4 + kk] : 0.0;
                    dmma884(acc[0], acc[1], x0, x0);
                    dmma884(acc[2], acc[3], x1, x1);
                }
                const double c0 = (acc[0] + acc[2]) + (acc[4] + acc[6]), c1 = (acc[1] + acc[3]) + (acc[5] + acc[7]);
                const int i = J0 + g;
                if (i < NR) {
                    const int ca = J0 + 2 * kk;
                    if (ca < J0 + nb && ca <= i) S[i * (i + 1) / 2 + ca] -= c0;
                    if (ca + 1 < J0 + nb && ca + 1 <= i) S[i * (i + 1) / 2 + ca + 1] -= c1;
                }
                __syncwarp();
            }
            // factor the nb x nb diagonal block: every lane of warp 0 runs the same register code on broadcast loads (no divergence, no
            // shuffles on the chain); lane a writes row a of L_JJ and its pivot reciprocal back
            double Ld[BA_CHOL_NB][BA_CHOL_NB], dinv[BA_CHOL_NB];
            bool bad = false;
#pragma unroll
            for (int a = 0; a < BA_CHOL_NB; a++)
#pragma unroll
                for (int b = 0; b < BA_CHOL_NB; b++) Ld[a][b] = (a < nb && b <= a) ? S[(J0 + a) * (J0 + a + 1) / 2 + J0 + b] : (a == b ? 1.0 : 0.0);
#pragma unroll
            for (int j = 0; j < BA_CHOL_NB; j++) {
                double d = Ld[j][j];
#pragma unroll
                for (int k = 0; k < j; k++) d -= Ld[j][k] * Ld[j][k];
                if (!(d > 0.0) || !isfinite(d)) bad = true;
                const double di = rsqrt(d);
                dinv[j] = di;
                Ld[j][j] = d * di;
#pragma unroll
                for (int a = j + 1; a < BA_CHOL_NB; a++) {
                    double sum = Ld[a][j];
#pragma unroll
                    for (int k = 0; k < j; k++) sum -= Ld[a][k] * Ld[j][k];
                    Ld[a][j] = sum * di;
                }
            }
            __syncwarp();  // every lane has read the unfactored block
            if (bad && lane == 0) s_fail = 1;
#pragma unroll
            for (int a2 = 0; a2 < BA_CHOL_NB; a2++) {
                // every lane holds the whole factor: entry (a2, b) is stored by ONE lane under a predicate -- statically indexed registers and no
                // divergent code.  ("lane a writes row a" was compiled into a switch on the lane, eight serial paths, several times slower in
                // ba_solve_cam_dsm's phase clocks than this form.)
                double *ri = S + (J0 + a2) * (J0 + a2 + 1) / 2 + J0;
#pragma unroll
                for (int b = 0; b <= a2; b++)
                    if (lane == ((a2 * 8 + b) & 31) && a2 < nb) ri[b] = Ld[a2][b];
                if (lane == 8 + a2 && a2 < nb) s_diag[J0 + a2] = dinv[a2];
            }
            SOLVE_CLK_ADD(6, pc0)
        } else if (J0 > 0 && warp != 4) {
            // tiles 1 .. ntile-1 over warps 1, 2, 3, 5, 6, 7, up to four row tiles per warp in flight (they share the B fragment): N = 157 gives
            // <= 19 such tiles, so the whole panel update is ONE round of the k loop, and eight independent DMMA chains hide the tensor-pipe
            // latency.  Warp 4 sits out: it shares warp 0's scheduler and FP64 pipe (warp id mod 4), and every DMMA holds that pipe for 16
            // cycles -- measured, warp 0's 130-operation pivot chain took 3 600 cycles per panel queuing behind warp 4's tiles.
            constexpr int TPW = 4, NWARP = 6;
            const int wslot = warp < 4 ? warp - 1 : warp - 2;  // 0..5
            for (int t0 = 1 + wslot; t0 < ntile; t0 += TPW * NWARP) {
                const double *ra[TPW];
                bool oka[TPW];
                double acc[TPW][4];
#pragma unroll
                for (int u = 0; u < TPW; u++) {
                    const int ia = J0 + 8 * (t0 + u * NWARP) + g;
                    oka[u] = (t0 + u * NWARP) < ntile && ia < NR;
                    ra[u] = S + (oka[u] ? ia * (ia + 1) / 2 : 0);
                    acc[u][0] = acc[u][1] = acc[u][2] = acc[u][3] = 0;
                }
                for (int k0 = 0; k0 + 8 <= J0; k0 += 8) {
                    const double b0 = okb ? rb[k0 + kk] : 0.0, b1 = okb ? rb[k0 + 4 + kk] : 0.0;
                    double a0[TPW], a1[TPW];
#pragma unroll
                    for (int u = 0; u < TPW; u++) a0[u] = oka[u] ? ra[u][k0 + kk] : 0.0, a1[u] = oka[u] ? ra[u][k0 + 4 + kk] : 0.0;
#pragma unroll
                    for (int u = 0; u < TPW; u++) {
                        dmma884(acc[u][0], acc[u][1], a0[u], b0);
                        dmma884(acc[u][2], acc[u][3], a1[u], b1);
                    }
                }
#pragma unroll
                for (int u = 0; u < TPW; u++) {
                    const double c0 = acc[u][0] + acc[u][2], c1 = acc[u][1] + acc[u][3];
                    const int i = J0 + 8 * (t0 + u * NWARP) + g;
                    if (oka[u]) {
                        const int ca = J0 + 2 * kk;
                        if (ca < J0 + nb && ca <= i) S[i * (i + 1) / 2 + ca] -= c0;
                        if (ca + 1 < J0 + nb && ca + 1 <= i) S[i * (i + 1) / 2 + ca + 1] -= c1;
                    }
                }
            }
        }
        __syncthreads();
        const unsigned long long pc1 = SOLVE_CLK_NOW();
        (void) pc1;
        if (s_fail) break;
        // rows below the block (incl. the augmented rhs row): solve against the factored block, one row per thread.  L_JJ and the pivot
        // reciprocals are read from shared memory as the chain needs them (every thread reads the same address: broadcast, off the
        // dependent chain) instead of being staged in 36 + 8 registers
        for (int i = J0 + nb + tid; i < NR; i += SOLVE_THREADS) {
            double *ri = S + i * (i + 1) / 2 + J0;
            double x[BA_CHOL_NB];
#pragma unroll
            for (int c = 0; c < BA_CHOL_NB; c++) x[c] = c < nb ? ri[c] : 0.0;
#pragma unroll
            for (int c = 0; c < BA_CHOL_NB; c++) {
                if (c < nb) {
                    const double *lc = S + (J0 + c) * (J0 + c + 1) / 2 + J0;
                    double sum = x[c];
#pragma unroll
                    for (int k = 0; k < c; k++) sum -= x[k] * lc[k];
                    x[c] = sum * s_diag[J0 + c];
                }
            }
#pragma unroll
            for (int c = 0; c < BA_CHOL_NB; c++)
                if (c < nb) ri[c] = x[c];
        }
        __syncthreads();
        SOLVE_CLK_ADD(7, pc1)
    }
    __syncthreads();
    bool valid = !s_fail;
    SOLVE_CLK(2)  // Cholesky
    // ---- backward substitution L^T x = y, blocked by the factorisation's 8-column panels, last panel first:
    //   (a) warp 0 solves the panel's 8 x 8 triangle L_JJ^T x_J = y_J in registers (every lane the same code on broadcast loads; the
    //       dependent chain is 8 x (DFMA + DMUL));
    //   (b) barrier; every thread i < J0 applies the panel to its own entry, y_i -= sum_c L[J0 + c][i] x_{J0 + c} -- row J0 + c of the
    //       packed triangle is contiguous in i, so the reads are coalesced; barrier.
    // Same operations in the same order as a column-by-column substitution (c descending), on 256 threads instead of one warp:
    // measured 185 cycles per COLUMN for the single-warp form (29 k cycles at N = 157), about 400 cycles per PANEL for this one.
    if (valid) {
        double *y = S + N * (N + 1) / 2;
        const int lane = tid & 31;
        for (int J0 = ((N - 1) / BA_CHOL_NB) * BA_CHOL_NB; J0 >= 0; J0 -= BA_CHOL_NB) {
            const int nb = min(BA_CHOL_NB, N - J0);
            if (tid < 32) {
                double x[BA_CHOL_NB];
#pragma unroll
                for (int c = BA_CHOL_NB - 1; c >= 0; c--) {
                    x[c] = 0.0;
                    if (c < nb) {
                        double sum = y[J0 + c];
#pragma unroll
                        for (int k = BA_CHOL_NB - 1; k > c; k--)
                            if (k < nb) sum -= S[(J0 + k) * (J0 + k + 1) / 2 + J0 + c] * x[k];
                        x[c] = sum * s_diag[J0 + c];
                    }
                }
#pragma unroll
                for (int c = 0; c < BA_CHOL_NB; c++)
                    if (c == lane && c < nb) s_rhs[J0 + c] = x[c];
            }
            __syncthreads();
            for (int i = tid; i < J0; i += SOLVE_THREADS) {
                double acc = y[i];
#pragma unroll
                for (int c = BA_CHOL_NB - 1; c >= 0; c--)
                    if (c < nb) acc -= S[(J0 + c) * (J0 + c + 1) / 2 + i] * s_rhs[J0 + c];
                y[i] = acc;
            }
            __syncthreads();
        }
    }
    __syncthreads();
    SOLVE_CLK(3)  // camera back-substitution
    // ---- landmark back-substitution + model cost change  (-1/2 step'.g' + 1/2 step'.D^2 step', exact identity of
    //      Ceres' -(J' step)^T (r + J' step / 2) for the damped normal-equation solution)
    double *step_l = D.step_l + (size_t) w * C.L;
    const double *AW = lin_AW(C, D, b, w);  // landmark-major
    double part = 0;
    bool finite = true;
    double *R2 = D.red2 + (size_t) w * 4;
    if (!valid) {
        // Cholesky breakdown: the step is invalid; ba_accept applies HandleInvalidStep
        if (tid == 0) {
            st.chol_ok = 0, st.step_valid = 0;
            R2[0] = 0, R2[1] = 0, R2[2] = 1;
        }
        return;
    }
    for (int a = tid; a < N; a += SOLVE_THREADS) {
        double sp = s_rhs[a];
        finite = finite && isfinite(sp);
        part += -0.5 * sp * (s_scale[a] * s_g[a]) + 0.5 * s_d2[a] * sp * sp;
    }
    // landmark back-substitution: one warp per landmark, the coupling row is read coalesced (two landmarks in flight per warp)
    double *s_sx = s_diag;  // s_diag is dead after the back-substitution: scaled camera step s_c * step'_c
    __syncthreads();
    for (int a = tid; a < NCV; a += SOLVE_THREADS) s_sx[a] = s_scale[a] * s_rhs[a];
    __syncthreads();
    {
        const int lane = tid & 31, warp = tid >> 5;
        constexpr int LB = 8;  // landmarks in flight per warp (the coupling rows come from L2: 24 loads per lane outstanding)
        // after the transposing reduction below, lane holds the dot product of landmark l0 + lu; its per-landmark scalars are loaded at the top
        // of the round, together with the coupling rows (one L2 round trip per round instead of two)
        const int lu = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
        for (int l0 = LB * warp; l0 < L; l0 += LB * (SOLVE_THREADS / 32)) {
            const int l = l0 + lu;
            const bool lok = l < L;
            const double sl = lok ? scale_l[l] : 0.0, hh = lok ? hl[l] : 0.0, gg = lok ? gl[l] : 0.0;
            double d[LB];
#pragma unroll
            for (int u = 0; u < LB; u++) d[u] = 0;
            for (int c = lane; c < NCV; c += 32) {
                const double sx = s_sx[c];
#pragma unroll
                for (int u = 0; u < LB; u++) d[u] += (l0 + u < L ? AW[(size_t) (l0 + u) * C.NCA + c] : 0.0) * sx;
            }
            const double hs = sl * sl * hh, d2 = fmin(fmax(hs, 1e-6), 1e32) / radius, den = hs + d2, sg = sl * gg;
            // transposing butterfly: 8 values x 32 lanes -> 1 value per lane in 4 + 2 + 1 + 1 + 1 exchanges (a plain butterfly needs 8 x 5)
            double e4[4], e2[2];
            {
                const bool hi = lane & 16;
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const double keep = hi ? d[u + 4] : d[u], send = hi ? d[u] : d[u + 4];
                    e4[u] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
                }
            }
            {
                const bool hi = lane & 8;
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    const double keep = hi ? e4[u + 2] : e4[u], send = hi ? e4[u] : e4[u + 2];
                    e2[u] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
                }
            }
            double mine;
            {
                const bool hi = lane & 4;
                const double keep = hi ? e2[1] : e2[0], send = hi ? e2[0] : e2[1];
                mine = keep + __shfl_xor_sync(0xffffffffu, send, 4);
            }
            mine += __shfl_xor_sync(0xffffffffu, mine, 2);
            mine += __shfl_xor_sync(0xffffffffu, mine, 1);
            if ((lane & 3) == 0 && lok) {
                double sp = (-sg - sl * mine) / den;
                finite = finite && isfinite(sp);
                step_l[l] = sp;
                part += -0.5 * sp * sg + 0.5 * d2 * sp * sp;
            }
        }
    }
    __syncthreads();
    SOLVE_CLK(4)  // landmark back-substitution
    const double mcc = block_sum(part, s_red);
    const double nfin = block_sum(finite ? 0.0 : 1.0, s_red);
    // ---- candidate point x (+) delta, delta = step' * scale; |x - x_cand|^2 over active blocks
    const double *pose = D.pose + (size_t) w * C.K * 7, *mix = D.mix + (size_t) w * C.K * 9, *ext = D.ext + (size_t) w * 8, *rho = D.rho + (size_t) w * C.L;
    double *pose_c = D.pose_c + (size_t) w * C.K * 7, *mix_c = D.mix_c + (size_t) w * C.K * 9, *ext_c = D.ext_c + (size_t) w * 8, *rho_c = D.rho_c + (size_t) w * C.L;
    double sn = 0;
    for (int k = tid; k <= K; k += SOLVE_THREADS) {  // K poses + the extrinsic
        const bool is_ext = (k == K);
        const double *x = is_ext ? ext : pose + k * 7;
        double *xc = is_ext ? ext_c : pose_c + k * 7;
        if (is_ext && dm.ext_const) {
            for (int e = 0; e < 7; e++) xc[e] = x[e];
        } else {
            const int c0 = is_ext ? col_ext(K) : col_pose(k);
            double d[6];
            for (int e = 0; e < 6; e++) d[e] = s_rhs[c0 + e] * s_scale[c0 + e];
            pose_plus(x, d, xc);
            for (int e = 0; e < 7; e++) sn += (x[e] - xc[e]) * (x[e] - xc[e]);
        }
    }
    for (int e = tid; e < K * 9; e += SOLVE_THREADS) {
        int k = e / 9, q = e - 9 * k, c = col_mix(K, k) + q;
        double v = mix[e] + s_rhs[c] * s_scale[c];
        mix_c[e] = v;
        sn += (mix[e] - v) * (mix[e] - v);
    }
    if (tid == 0) {
        if (dm.td_const) {
            ext_c[7] = ext[7];
        } else {
            double v = ext[7] + s_rhs[col_td(K)] * s_scale[col_td(K)];
            ext_c[7] = v;
            sn += (ext[7] - v) * (ext[7] - v);
        }
    }
    for (int l = tid; l < L; l += SOLVE_THREADS) {
        double v = rho[l] + step_l[l] * scale_l[l];
        rho_c[l] = v;
        sn += (rho[l] - v) * (rho[l] - v);
    }
    sn = block_sum(sn, s_red);
    if (tid == 0) {
        st.chol_ok = 1, st.step_valid = 1;  // provisional: ba_accept validates with the reduced model cost change
        R2[0] = mcc, R2[1] = sn, R2[2] = nfin;
    }
    SOLVE_CLK(5)  // candidate point, reductions
#undef SOLVE_CLK
#undef SOLVE_CLK_NOW
#undef SOLVE_CLK_ADD
}

// ------------------------------------------------------------------------------------------------ candidate cost (split pipeline)
// The single-GPU pipeline takes the candidate cost from the linearisation at the candidate instead (ba_accept).
// camera-only factors at the candidate point (one CTA per window; runs beside the vision blocks on the handle's second stream)
__global__ void __launch_bounds__(CAM_THREADS) ba_cost_cam(BaCaps C, BaDev D, int nblk_vis) {
    extern __shared__ double smem[];
    const int w = blockIdx.x;
    const LmState &st = D.st[w];
    if (st.done || !st.step_valid) return;
    if (D.S.split && (w % D.world) != D.rank) return;
    const WinDims dm = D.dims[w];
    double c = cam_factors(C, D, w, dm, D.pose_c + (size_t) w * C.K * 7, D.mix_c + (size_t) w * C.K * 9, D.ext_c + (size_t) w * 8, false, 0, smem);
    if (threadIdx.x == 0) D.cost_part[(size_t) w * (nblk_vis + 1) + nblk_vis] = c;
}
__global__ void __launch_bounds__(256) ba_cost(BaCaps C, BaDev D, int nblk_vis) {
    __shared__ double s_red[40];
    const int w = blockIdx.y;
    const LmState &st = D.st[w];
    if (st.done || !st.step_valid) return;
    const WinDims dm = D.dims[w];
    const double *pose = D.pose_c + (size_t) w * C.K * 7, *ext = D.ext_c + (size_t) w * 8, *rho = D.rho_c + (size_t) w * C.L;
    double *part = D.cost_part + (size_t) w * (nblk_vis + 1);
    const int q = blockIdx.x * 256 + threadIdx.x;  // record slot (landmark-CSR order): the slot-ordered copies are the only factor data on the device
    __shared__ double s_frame[BA_MAX_NODES + 1][NODE_FRAME_LD];  // node frames of the candidate point (see ba_lin_vis)
    if ((int) threadIdx.x <= dm.K) node_frame((int) threadIdx.x < dm.K ? pose + threadIdx.x * 7 : ext, s_frame[threadIdx.x]);
    __syncthreads();
    double cost = 0;
    int4 meta = make_int4(0, 0, 0, 0);
    if (q < dm.F) meta = ((const int4 *) D.f_meta_s)[(size_t) w * C.F + q];  // (landmark, reference node, observing node, factor id)
    if (q < dm.F && D.f_active[(size_t) w * C.F + meta.w]) {
        double r[2];
        reproj_eval_frames(s_frame[meta.y], s_frame[meta.z], s_frame[dm.K], rho[meta.x], ext[7], D.f_const_s + ((size_t) w * C.F + q) * 14, dm.reproj_sinv,
                           false, r, nullptr, nullptr, nullptr, nullptr, nullptr);
        double sq = r[0] * r[0] + r[1] * r[1], sc;
        if (dm.reproj_huber)
            huber(sq, cost, sc);
        else
            cost = 0.5 * sq;
    }
    cost = block_sum(cost, s_red);
    if (threadIdx.x == 0) part[blockIdx.x] = cost;
}

// ------------------------------------------------------------------------------------------------ accept / reject
__global__ void __launch_bounds__(128) ba_accept(BaCaps C, BaDev D) {
    __shared__ int s_accept;
    __shared__ double s_camsq, s_rhosq;
    __shared__ double s_red[40];
    const int w = blockIdx.x, tid = threadIdx.x;
    LmState &st = D.st[w];
    if (st.done) return;
    const WinDims dm = D.dims[w];
    const double *R2 = D.red2 + (size_t) w * 4;
    // |x|^2 of the camera-side blocks and of the landmarks
    {
        const double *pose = D.pose + (size_t) w * C.K * 7, *mix = D.mix + (size_t) w * C.K * 9, *ext = D.ext + (size_t) w * 8;
        double s = 0;
        for (int e = tid; e < dm.K * 7; e += 128) s += pose[e] * pose[e];
        for (int e = tid; e < dm.K * 9; e += 128) s += mix[e] * mix[e];
        if (tid < 7 && !dm.ext_const) s += ext[tid] * ext[tid];
        if (tid == 7 && !dm.td_const) s += ext[7] * ext[7];
        s = block_sum(s, s_red);
        double q = 0;  // |rho|^2
        for (int l = tid; l < dm.L; l += 128) q += D.rho[(size_t) w * C.L + l] * D.rho[(size_t) w * C.L + l];
        q = block_sum(q, s_red);
        if (tid == 0) s_camsq = s, s_rhosq = q;
    }
    // The candidate cost from the linearisation at the candidate (buffer 1 - lin_buf), summed in ba_cost's order -- per 256 record slots
    // block_sum's tree (warp k sums slots [32 k, 32 k + 32) of the block, then the eight warp sums in order), the blocks in order, then the
    // camera-only cost -- so that every decision below matches the sum of ba_cost's partials bit for bit.
    // s_warp (dynamic, 8 per 256 slots): the sums of the 32-slot groups; warp k of this CTA reduces groups k, k + 4, ... with no barrier in
    // between, so that the loads of several groups are in flight together.
    extern __shared__ double s_warp[];
    const int lane = tid & 31, warp = tid >> 5, ngrp = (dm.F + 31) / 32;
    if (st.step_valid) {
        const double *costf = lin_costf(C, D, 1 - st.lin_buf, w);
        const int4 *meta = (const int4 *) D.f_meta_s + (size_t) w * C.F;  // (landmark, reference node, observing node, factor id) per slot
#pragma unroll 4
        for (int g = warp; g < ngrp; g += 4) {
            const int q = 32 * g + lane;
            double v = q < dm.F ? costf[meta[q].w] : 0.0;  // lin_vis leaves 0 for an inactive factor
            for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
            if (lane == 0) s_warp[g] = v;
        }
    }
    __syncthreads();
    if (tid == 0) {
        s_accept = 0;
        const double mcc = R2[0], sn = R2[1], nfin = R2[2];
        double cand = 0;
        if (st.step_valid) {
            for (int g0 = 0; g0 < ngrp; g0 += 8) {
                double t = 0;
                for (int k = 0; k < 8; k++) t += g0 + k < ngrp ? s_warp[g0 + k] : 0.0;
                cand += t;
            }
            cand += st.cost_cam[1 - st.lin_buf];
        }
        if (!st.chol_ok || nfin != 0.0 || !(mcc > 0.0)) {
            // HandleInvalidStep + LevenbergMarquardtStrategy::StepIsInvalid
            st.step_valid = 0;
            st.n_invalid++;
            if (st.n_invalid >= 5) st.done = 3;  // FAILURE
            st.radius *= 0.5;
            st.last_success = 0;
        } else {
            st.n_invalid = 0;
            st.model_cost_change = mcc;
            st.step_norm = sqrt(sn);
            st.x_norm = sqrt(s_camsq + s_rhosq);
            st.cand_cost = cand;
            // ParameterToleranceReached / FunctionToleranceReached (Ceres trust_region_minimizer.cc)
            if (st.step_norm <= 1e-8 * (st.x_norm + 1e-8)) {
                st.done = 2;
            } else if (fabs(st.x_cost - cand) <= 1e-6 * st.x_cost) {
                st.done = 2;
            } else {
                const double rel = (st.x_cost - cand) / mcc;
                if (rel > 1e-3) {
                    s_accept = 1;
                    st.n_success++;
                    // LevenbergMarquardtStrategy::StepAccepted
                    double t = 2.0 * rel - 1.0;
                    st.radius = fmin(1e16, st.radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
                    st.decrease_factor = 2.0;
                    st.last_success = 1;
                    st.fresh_lin = 1;
                    st.lin_buf ^= 1;  // the candidate's linearisation is now the one at x
                } else {
                    // StepRejected
                    st.radius = st.radius / st.decrease_factor;
                    st.decrease_factor *= 2.0;
                    st.last_success = 0;
                    st.need_lin = 0;
                }
            }
        }
    }
    __syncthreads();
    if (!s_accept) return;
    double *pose = D.pose + (size_t) w * C.K * 7, *mix = D.mix + (size_t) w * C.K * 9, *ext = D.ext + (size_t) w * 8, *rho = D.rho + (size_t) w * C.L;
    const double *pose_c = D.pose_c + (size_t) w * C.K * 7, *mix_c = D.mix_c + (size_t) w * C.K * 9, *ext_c = D.ext_c + (size_t) w * 8, *rho_c = D.rho_c + (size_t) w * C.L;
    for (int e = tid; e < dm.K * 7; e += 128) pose[e] = pose_c[e];
    for (int e = tid; e < dm.K * 9; e += 128) mix[e] = mix_c[e];
    if (tid < 8) ext[tid] = ext_c[tid];
    for (int e = tid; e < dm.L; e += 128) rho[e] = rho_c[e];
}

// ------------------------------------------------------------------------------------------------ LM state reset (device side)
__global__ void ba_reset_state(BaDev D, LmState *save, int n, int max_iter) {
    int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n) return;
    if (save) save[w] = D.st[w];
    LmState st;
    memset(&st, 0, sizeof(st));
    st.radius = 1e4, st.decrease_factor = 2.0;  // Ceres initial_trust_region_radius
    st.need_lin = 1, st.fresh_lin = 1, st.first = 1, st.last_success = 1, st.max_iter = max_iter;
    D.st[w] = st;
}

// The outlier pass between the two solves of GVINS::gvinsOptimization (IG/ic_gvins.cc:1196-1207):
//   gnssOutlierCullingByChi2 (:1241-1267): chi2 = 2 cost > 7.815 -> std *= sqrt(chi2 / 7.815)
//   removeReprojectionFactorsByChi2 (:1269-1297): chi2 = 2 cost > 5.991 -> RemoveResidualBlock
//   GNSS factors re-added without loss function (:1202-1207)
__global__ void __launch_bounds__(128) ba_chi2_cull(BaCaps C, BaDev D, int *counters) {
    const int w = blockIdx.y;
    WinDims &dm = D.dims[w];
    const int t = blockIdx.x * 128 + threadIdx.x;
    const double *pose = D.pose + (size_t) w * C.K * 7, *ext = D.ext + (size_t) w * 8, *rho = D.rho + (size_t) w * C.L;
    int4 meta = make_int4(0, 0, 0, 0);
    if (t < dm.F) meta = ((const int4 *) D.f_meta_s)[(size_t) w * C.F + t];  // record slot t
    if (t < dm.F && D.f_active[(size_t) w * C.F + meta.w]) {
        double r[2];
        reproj_eval(pose + meta.y * 7, pose + meta.z * 7, ext, rho[meta.x], ext[7], D.f_const_s + ((size_t) w * C.F + t) * 14, dm.reproj_sinv, false, r, nullptr,
                    nullptr, nullptr, nullptr, nullptr);
        if ((r[0] * r[0] + r[1] * r[1]) > 5.991) {
            D.f_active[(size_t) w * C.F + meta.w] = 0;
            atomicAdd(&counters[2 * w], 1);
        }
    }
    if (t < dm.n_gnss) {
        double r[3];
        double *sd = D.gnss_std + ((size_t) w * C.G + t) * 3;
        gnss_eval(pose + D.gnss_node[(size_t) w * C.G + t] * 7, D.gnss_blh + ((size_t) w * C.G + t) * 3, sd, D.lever + (size_t) w * 3, false, r, nullptr);
        double chi2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
        if (chi2 > 7.815) {
            double sc = sqrt(chi2 / 7.815);
            sd[0] *= sc, sd[1] *= sc, sd[2] *= sc;
            atomicAdd(&counters[2 * w + 1], 1);
        }
    }
}
__global__ void ba_set_gnss_huber(BaDev D, int n, int v) {
    int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w < n) D.dims[w].gnss_huber = v;
}

// ------------------------------------------------------------------------------------------------ utility kernels
__global__ void ba_residual_costs_kernel(BaCaps C, BaDev D, double *reproj_cost, double *gnss_cost) {
    const int w = 0;
    const WinDims dm = D.dims[w];
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const double *pose = D.pose, *ext = D.ext, *rho = D.rho;
    if (t < dm.F) {
        double r[2];
        const int4 meta = ((const int4 *) D.f_meta_s)[t];  // record slot t -> (landmark, reference node, observing node, factor id)
        reproj_eval(pose + meta.y * 7, pose + meta.z * 7, ext, rho[meta.x], ext[7], D.f_const_s + (size_t) t * 14, dm.reproj_sinv, false, r, nullptr, nullptr,
                    nullptr, nullptr, nullptr);
        reproj_cost[meta.w] = 0.5 * (r[0] * r[0] + r[1] * r[1]);  // EvaluateResidualBlock(id, false, &cost, ...) (IG/ic_gvins.cc:1278)
    }
    if (t < dm.n_gnss) {
        double r[3];
        gnss_eval(pose + D.gnss_node[t] * 7, D.gnss_blh + t * 3, D.gnss_std + t * 3, D.lever, false, r, nullptr);
        gnss_cost[t] = 0.5 * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    }
}

__global__ void ba_reproj_eval_kernel(const double *in /* 7+7+8+1+1+14+1 */, double *out /* 2 + 14+14+14+2+2 */) {
    double r[2], Ji[12], Jj[12], Je[12], Jr[2], Jt[2];
    reproj_eval(in, in + 7, in + 14, in[22], in[23], in + 24, 1.0 / in[38], true, r, Ji, Jj, Je, Jr, Jt);
    out[0] = r[0], out[1] = r[1];
    double *o = out + 2;
    const double *src[3] = {Ji, Jj, Je};
    for (int b = 0; b < 3; b++)
        for (int rr = 0; rr < 2; rr++) {
            for (int c = 0; c < 6; c++) o[b * 14 + rr * 7 + c] = src[b][rr * 6 + c];
            o[b * 14 + rr * 7 + 6] = 0.0;  // the quaternion-w column of the global Jacobian is zero (reprojection_factor.h:103,114,131)
        }
    o[42] = Jr[0], o[43] = Jr[1], o[44] = Jt[0], o[45] = Jt[1];
}

__global__ void ba_imu_eval_kernel(const double *blob, const double *U, const double *x /* 7 9 7 9 */, double *out /* 15 + 450 */) {
    __shared__ double s_buf[480];
    imu_factor_warp(blob, U, x, x + 7, x + 16, x + 23, true, s_buf, s_buf + 30, threadIdx.x);
    for (int e = threadIdx.x; e < 15; e += 32) out[e] = s_buf[e];
    for (int e = threadIdx.x; e < 450; e += 32) out[15 + e] = s_buf[30 + e];
}

// GnssFactor / ImuPosePriorFactor / ImuMixPriorFactor / ImuErrorFactor (kind 0..3), one thread; in / out layouts in the callers below
__global__ void ba_small_factor_eval_kernel(int kind, const double *in, double *out) {
    if (kind == 0) {         // in: pose7 blh3 std3 lever3 -> r[3], J local 3x6
        gnss_eval(in, in + 7, in + 10, in + 13, true, out, out + 3);
    } else if (kind == 1) {  // in: pose7 prior7 sinfo6 -> r[6], J local 6x6
        pose_prior_eval(in, in + 7, in + 14, true, out, out + 6);
    } else if (kind == 2) {  // in: mix9 prior9 std9 -> r[9], diag J[9]   (ImuMixPriorFactor, imu_mix_prior_factor.h:40-75)
        for (int k = 0; k < 9; k++) out[k] = (in[k] - in[9 + k]) / in[18 + k], out[9 + k] = 1.0 / in[18 + k];
    } else {                 // in: mix9 -> r[6], diag J[6]                (ImuErrorFactor, imu_error_factor.h:45-91)
        for (int k = 0; k < 3; k++) {
            out[k] = in[3 + k] / IMU_GB_STD, out[3 + k] = in[6 + k] / IMU_AB_STD;
            out[6 + k] = 1.0 / IMU_GB_STD, out[9 + k] = 1.0 / IMU_AB_STD;
        }
    }
}

// MarginalizationFactor::Evaluate (IG/factors/marginalization_factor.h:47-101): e = e0 + J0 dx with dx the local difference of every
// remained block to its linearisation point (quaternion blocks: 2 vec(q0^-1 q), sign-fixed).  One CTA; thread per residual row.
// in: [r, nb, types[nb], x (global sizes, concatenated), x0 (same), e0[r], J0[r*r]] as doubles; out: residuals[r]
__global__ void ba_marg_factor_eval_kernel(const double *in, double *out) {
    extern __shared__ double s_dx[];
    const int r = (int) in[0], nb = (int) in[1];
    const double *types = in + 2;
    int tot = 0;
    for (int b = 0; b < nb; b++) tot += ((int) types[b] == 1) ? 9 : ((int) types[b] == 3) ? 1 : 7;
    const double *x = types + nb, *x0 = x + tot, *e0 = x0 + tot, *J0 = e0 + r;
    if (threadIdx.x == 0) {
        int col = 0, xo = 0;
        for (int b = 0; b < nb; b++) {
            const int t = (int) types[b];
            if (t == 0 || t == 2) {
                Q dq = qmul(qinv(pose_q(x0 + xo)), pose_q(x + xo));
                V3 a = 2.0 * qv(dq);
                if (dq.w < 0) a = -a;
                for (int k = 0; k < 3; k++) s_dx[col + k] = x[xo + k] - x0[xo + k];
                s_dx[col + 3] = a.x, s_dx[col + 4] = a.y, s_dx[col + 5] = a.z;
                col += 6, xo += 7;
            } else {
                const int g = t == 1 ? 9 : 1;
                for (int k = 0; k < g; k++) s_dx[col + k] = x[xo + k] - x0[xo + k];
                col += g, xo += g;
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < r; i += blockDim.x) {
        double sum = e0[i];
        for (int k = 0; k < r; k++) sum += J0[(size_t) i * r + k] * s_dx[k];
        out[i] = sum;
    }
}

}  // namespace icg

#include "ba_split.cuh"
#include "ba_marg.cuh"

// ======================================================================================================= host side
using namespace icg;

namespace {
// ---- IMU sqrt information  U = LLT(cov^-1).matrixL().transpose(): the shared core of geom_core.cuh, so that the reintegration kernel
//      (preint.cu) writes the same U into the handle as the upload
bool host_imu_sqrt_info(const double *cov, double *U) {
    double work[675];
    return gc::imu_sqrt_info(cov, U, work);
}

template <typename T>
struct HostDev {  // pinned host staging + device array
    T *h = nullptr, *d = nullptr;
    size_t n = 0;
    int alloc(size_t count) {
        n = count;
        if (cudaMallocHost(&h, sizeof(T) * count) != cudaSuccess) return ICG_ENOMEM;
        if (cudaMalloc(&d, sizeof(T) * count) != cudaSuccess) return ICG_ENOMEM;
        memset(h, 0, sizeof(T) * count);
        return ICG_OK;
    }
    void release() {
        if (h) cudaFreeHost(h);
        if (d) cudaFree(d);
        h = d = nullptr;
    }
    cudaError_t up(cudaStream_t s, size_t count = 0) { return cudaMemcpyAsync(d, h, sizeof(T) * (count ? count : n), cudaMemcpyHostToDevice, s); }
    cudaError_t down(cudaStream_t s, size_t count = 0) { return cudaMemcpyAsync(h, d, sizeof(T) * (count ? count : n), cudaMemcpyDeviceToHost, s); }
};
}  // namespace

struct icg_ba {
    BaCaps C;
    BaDev D;
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t stream_cam = nullptr;  // the camera-only factors are linearised concurrently with the vision chain
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    bool own_stream = false;
    int nblk_vis = 0;
    int cur_windows = 0;
    size_t smem_cam, smem_solve, smem_schur;
    int ld_schur;
    int use_global_S;
    HostDev<WinDims> dims;
    HostDev<LmState> st;
    HostDev<double> pose, mix, ext, rho, imu_blob, imu_U, gnss_blh, gnss_std, lever, pose_prior, pose_prior_sinfo, mix_prior, mix_prior_std, marg_x0,
        marg_H0, marg_b0, marg_c0;
    HostDev<int> f_meta_s, vb_lm0, ref_nrun;  // lm_fidx: host-side packing helper only (record slot -> factor id)
    HostDev<double> f_const_s;
    HostDev<int> lm_off, lm_perm, lm_fidx, gnss_node, marg_type, marg_node, part_off, pair_ro, vis_ord, npairs;
    HostDev<uint8_t> f_active;
    std::vector<void *> dev_only;
    HostDev<double> scratch;  // single-factor evaluation
    HostDev<LmState> st_save;   // pass-1 LM state of the two-pass protocol
    HostDev<int> cull_counters; // per window: reprojection factors removed, GNSS fixes re-weighted
    // split pipeline (ba_split.cuh): exchange buffer of this rank, peers' buffers opened through CUDA IPC, epoch counter of the flags
    double *xbuf = nullptr;
    size_t xbuf_doubles = 0;
    int x_world = 0;
    void *ipc_opened[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    unsigned long long epoch = 0;
    size_t smem_solve_cam = 0, smem_step_lm = 0;
    bool solve_cam_dsm = false;      // the packed system fits the cluster's shared memory: ba_solve_cam_dsm (max_K <= 23)
    size_t smem_solve_cam_dsm = 0;
    // in-situ stage timing (ICG_BA_PROFILE=1): events between the kernels of the LM sequence on the main stream, read back in
    // icg_ba_sync / icg_ba_download and printed by icg_ba_destroy (warm caches, real launch gaps -- unlike an ncu replay)
    bool prof = false;
    std::vector<cudaEvent_t> prof_ev;
    std::vector<int> prof_tag;
    size_t prof_used = 0;
    int prof_skip = 1;  // LM sequences to discard first (lazy module loading puts a one-off multi-ms cost on every kernel's first launch)
    double prof_ms[16] = {0};
    long prof_cnt[16] = {0};
    // marginalization workspace (allocated on the first icg_ba_marginalize call).  The parts sized by the marginalized block (H0, b0, G1,
    // V1, lam1, Z) follow the largest batch seen so far: marg_nw windows at the strides M.n0cap / M.mcap, grown on demand
    bool marg_ready = false;
    MargDev M{};
    int marg_nw = 0;
    int marg_cluster_ok = -1;  // -1 not checked yet; 1: an 8-CTA marg_jacobi_cluster with its largest shared memory can be scheduled
    HostDev<int> marg_map;
    HostDev<double> marg_oJ0, marg_oe0, marg_oHp, marg_obp;
    HostDev<uint8_t> marg_fmask;  // factor set of icg_ba_marginalize_resident_culled (ba_lin_vis reads it in place of f_active)
    // post-solve update + culling: one pinned staging buffer and its device twin, [inputs | outputs], grown on demand
    unsigned char *cull_h = nullptr, *cull_d = nullptr;
    size_t cull_cap = 0;
    // the last culling, while it is current (icg_ba_slide_vision_resident reads its flags from the staging above): its window count (0: none;
    // an upload, a slide or a sharded culling clears it), every window's slices and observation count, the staging offsets of its arrays
    int cull_res_n = 0;
    std::vector<CullWin> cull_res_win;
    std::vector<int> cull_res_nobs;
    size_t cull_res_ref = 0, cull_res_off = 0, cull_res_lmo = 0, cull_res_obso = 0;
    // icg_ba_slide_vision_resident: pinned staging and its device twin, grown on demand
    unsigned char *vis_h = nullptr, *vis_d = nullptr;
    size_t vis_cap = 0;
    // reintegration of the resident IMU factors: the same arrangement, its own buffers
    unsigned char *reint_h = nullptr, *reint_d = nullptr;
    size_t reint_cap = 0;
    // the last resident marginalization, while its workspace (marg_oJ0 / marg_oe0) is the prior of the windows the handle holds: its window
    // count (0: none; an upload, a slide or another marginalization clears it) and every window's m, r and number of remained blocks.
    // marg_res_sharded: it was the sharded resident marginalization of a shard group; the prior of window w is then in the workspace of mx_h
    // (slot (w - rank) / world) on its owner, and m = r = nblocks = 0 is kept for the windows another rank owns
    int marg_res_n = 0;
    bool marg_res_sharded = false;
    std::vector<int> marg_res_m, marg_res_r, marg_res_nb;
    // icg_ba_slide_resident: pinned staging and its device twin (grown on demand), the copy of the old value rows, the second f_const_s buffer
    unsigned char *slide_h = nullptr, *slide_d = nullptr;
    size_t slide_cap = 0;
    double *slide_old = nullptr, *fc_alt = nullptr;
    // every landmark's reference row pts0[3] | vel0[3] | td0 (NaN: unknown), 7 doubles at w L + l, and the buffer the next slide writes: set by
    // icg_ba_upload from the landmark's first factor, carried by every slide, read by icg_ba_slide_vision_resident
    double *lm_ref = nullptr, *lm_ref_alt = nullptr;
    cudaEvent_t slide_ev = nullptr;  // recorded after the staging's H2D
    // post-solve calls of a shard group (world > 1): integer exchanges so far (slot parity), epoch of the last marginalization export, the
    // exchange's device word, the export's slot lists, the owner's gathered rows with their tables, and the handle the owner uploads its
    // gathered windows to (created on first use, recreated when a batch needs more landmarks, factors or windows)
    unsigned long long xs_calls = 0, exp_epoch = 0;
    HostDev<int> xs_v, mx_sel, mx_row;
    HostDev<long long> mx_heads, mx_idx;
    double *mx_rows = nullptr;
    size_t mx_rows_cap = 0;
    icg_ba *mx_h = nullptr;
    // buffers a shard group's call outgrew.  Freeing synchronises the device, and between handles of one process that would wait for a
    // peer's kernel spinning on this rank's flags: they are freed when the group is left or the handle destroyed
    std::vector<void *> retired_d, retired_h;
    std::vector<icg_ba *> retired_mx;
};

extern "C" {
static void prof_collect(icg_ba *h);
static void prof_print(icg_ba *h);
}

static int dmalloc(icg_ba *h, double **p, size_t n) {
    if (cudaMalloc(p, sizeof(double) * n) != cudaSuccess) {
        set_error("icg_ba_create: cudaMalloc of %zu doubles failed", n);
        return ICG_ENOMEM;
    }
    cudaMemsetAsync(*p, 0, sizeof(double) * n, h->stream);
    h->dev_only.push_back(*p);
    return ICG_OK;
}

// CTA size of the camera-only factor kernels (ba_lin_cam, ba_cost_cam).  160 threads x 168 registers leave room for two ba_lin_vis CTAs on
// the SM (320 threads take 82 % of the register file: nothing else fits beside them).  With four or more landmark shards the owner's
// camera-only kernels are on the attempt's critical path (the vision kernels shrink with the shard -- 410 us at one rank, ~100 at four --,
// the per-window IMU chain of ~118 us does not): all 10 warps, two rounds of IMU factors at K = 20 instead of four.
static int cam_threads(const icg_ba *h) { return h->D.world >= 4 ? CAM_THREADS : 160; }

extern "C" {
static int split_setup(icg_ba *h, int rank, int world);
static void split_release(icg_ba *h);

int icg_imu_preintegrate(const double *state16, const double *iewn3, const double *gravity3, const double *noise5, const double *imu, int n, double *blob,
                         double *end_state10) {
    // PreintegrationEarth: resetState (:305-324), setNoiseMatrix (:326-334), integrationProcess (:205-260),
    // updateJacobianAndCovariance (:266-303) of IG/preintegration/preintegration_earth.cc.  Host code (sequential recurrence).
    // iewn3 == NULL selects PreintegrationNormal (`iswithearth: false`, IG/preintegration/preintegration_normal.cc:155-232 +
    // PreintegrationBase::integration, preintegration_base.cc:39-70): no Earth-rotation / Coriolis terms; the blob is tagged (blob[477] = 1)
    // so that the factor evaluates PreintegrationNormal::evaluate.
    if (!state16 || !gravity3 || !noise5 || !imu || !blob || n < 1) {
        set_error("icg_imu_preintegrate: bad arguments");
        return ICG_EINVAL;
    }
    gc::preintegrate_core(state16, iewn3, gravity3, noise5, imu, n, blob, end_state10);  // one definition for host and device (geom_core.cuh)
    return ICG_OK;
}

static int ba_create_body(icg_ba *h, int max_windows, int max_K, int max_L, int max_F, int max_gnss, int max_marg_r, void *stream);

int icg_ba_create(icg_ba **out, int max_windows, int max_K, int max_L, int max_F, int max_gnss, int max_marg_r, int device, void *stream) {
    if (!out || max_windows < 1 || max_K < 2 || max_K > 32 || max_L < 0 || max_F < 0 || max_gnss < 0 || max_marg_r < 0) {
        set_error("icg_ba_create: bad arguments");
        return ICG_EINVAL;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        set_error("icg_ba_create: no CUDA device (this library has no CPU fallback)");
        return ICG_ENODEVICE;
    }
    if (device < 0 || device >= ndev) {
        set_error("icg_ba_create: device %d out of range", device);
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    ICG_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error("icg_ba_create: device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor);
        return ICG_ENODEVICE;
    }
    icg_ba *h = new icg_ba();
    h->device = device;
    const int rc_init = ba_create_body(h, max_windows, max_K, max_L, max_F, max_gnss, max_marg_r, stream);
    if (rc_init != ICG_OK) {  // every failure path releases what was already allocated (streams, events, pinned + device memory)
        icg_ba_destroy(h);
        return rc_init;
    }
    *out = h;
    return ICG_OK;
}

static int ba_create_body(icg_ba *h, int max_windows, int max_K, int max_L, int max_F, int max_gnss, int max_marg_r, void *stream) {
    if (stream) {
        h->stream = (cudaStream_t) stream;
    } else {
        ICG_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        h->own_stream = true;
    }
    {   // the forked camera-factor kernels are one latency-bound CTA per window: give them priority so that they are placed before the
        // wide vision kernels fill the SMs (otherwise they start late and then contend with the Schur / Gram kernels)
        int prio_lo = 0, prio_hi = 0;
        ICG_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
        ICG_CUDA(cudaStreamCreateWithPriority(&h->stream_cam, cudaStreamNonBlocking, prio_hi));
    }
    ICG_CUDA(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    ICG_CUDA(cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming));
    h->prof = getenv("ICG_BA_PROFILE") != nullptr;
    if (h->prof) {
        double *ck = nullptr;
        if (dmalloc(h, &ck, 48) != ICG_OK) return ICG_ENOMEM;
        h->D.clk = (unsigned long long *) ck;
    }
    if (getenv("ICG_BA_PROFILE_SKIP")) h->prof_skip = atoi(getenv("ICG_BA_PROFILE_SKIP"));
    BaCaps &C = h->C;
    max_L = std::max(1, max_L), max_F = std::max(1, max_F);  // capacities stay >= 1; windows without landmarks (first keyframes, IG/ic_gvins.cc:1698) are accepted
    C.NW = max_windows, C.K = max_K, C.L = max_L, C.F = max_F, C.G = std::max(1, max_gnss), C.R = std::max(1, max_marg_r);
    C.NCV = 6 * max_K + 7, C.N = 15 * max_K + 7, C.NS = (C.N + 3) & ~3, C.NCA = 4 * ((C.NCV + 1 + 3) / 4);
    C.RJ = (2 * max_F + 31) & ~31, C.LP = (max_L + 31) & ~31;
    // worst case: every run is cut short by one landmark's K - 1 factors, plus one more run per reference node (runs never span two)
    C.NVB = (max_F + 127 - max_K) / (128 - max_K) + max_L / 128 + 4 + max_K;
    C.GQ = std::max(1, std::min(max_F, (C.NVB - 2) * (max_K - 1)));  // a partial holds >= 1 factor; a run observes from <= K - 1 nodes
    h->nblk_vis = (max_F + 255) / 256;
    const size_t NW = max_windows;
#define HD(field, count)                                                       \
    if (h->field.alloc(count) != ICG_OK) {                                     \
        set_error("icg_ba_create: allocation of " #field " failed");           \
        return ICG_ENOMEM;                                                     \
    }
    HD(dims, NW) HD(st, NW) HD(pose, NW * C.K * 7) HD(mix, NW * C.K * 9) HD(ext, NW * 8) HD(rho, NW * C.L)
    HD(imu_blob, NW * C.K * ICG_IMU_BLOB_DOUBLES) HD(imu_U, NW * C.K * 225) HD(gnss_blh, NW * C.G * 3) HD(gnss_std, NW * C.G * 3) HD(lever, NW * 3)
    HD(pose_prior, NW * 7) HD(pose_prior_sinfo, NW * 6) HD(mix_prior, NW * 9) HD(mix_prior_std, NW * 9) HD(marg_x0, NW * BA_MARG_MAXB * 9)
    HD(marg_H0, NW * C.R * C.R) HD(marg_b0, NW * C.R) HD(marg_c0, NW)
    HD(lm_off, NW * (C.L + 1)) HD(lm_perm, NW * C.L) HD(lm_fidx, NW * C.F) HD(gnss_node, NW * C.G) HD(marg_type, NW * BA_MARG_MAXB) HD(marg_node, NW * BA_MARG_MAXB) HD(f_active, NW * C.F)
    HD(scratch, 1024) HD(st_save, NW) HD(cull_counters, 2 * NW) HD(f_meta_s, NW * C.F * 4) HD(vb_lm0, NW * C.NVB) HD(ref_nrun, NW * C.K) HD(f_const_s, NW * C.F * 14)
    HD(part_off, NW * ((size_t) C.K * (C.K - 1) + 1)) HD(pair_ro, NW * (size_t) C.K * (C.K - 1)) HD(vis_ord, NW * C.F) HD(npairs, NW)
#undef HD
    // the LM state is otherwise written only when a run starts: zero it, so that a marginalization on a handle that has not solved yet reads
    // linearisation buffer 0 (the one every handle has) rather than whatever the allocation held
    ICG_CUDA(cudaMemsetAsync(h->st.d, 0, sizeof(LmState) * NW, h->stream));
    BaDev &D = h->D;
    D.rank = 0, D.world = 1;
    D.dims = h->dims.d, D.st = h->st.d, D.pose = h->pose.d, D.mix = h->mix.d, D.ext = h->ext.d, D.rho = h->rho.d;
    D.f_active = h->f_active.d;
    D.part_off = h->part_off.d, D.pair_ro = h->pair_ro.d, D.vis_ord = h->vis_ord.d, D.npairs = h->npairs.d;
    D.f_meta_s = h->f_meta_s.d, D.vb_lm0 = h->vb_lm0.d, D.ref_nrun = h->ref_nrun.d, D.f_const_s = h->f_const_s.d;
    D.lm_off = h->lm_off.d, D.lm_perm = h->lm_perm.d, D.imu_blob = h->imu_blob.d, D.imu_U = h->imu_U.d;
    D.gnss_node = h->gnss_node.d, D.gnss_blh = h->gnss_blh.d, D.gnss_std = h->gnss_std.d, D.lever = h->lever.d;
    D.pose_prior = h->pose_prior.d, D.pose_prior_sinfo = h->pose_prior_sinfo.d, D.mix_prior = h->mix_prior.d, D.mix_prior_std = h->mix_prior_std.d;
    D.marg_type = h->marg_type.d, D.marg_node = h->marg_node.d, D.marg_x0 = h->marg_x0.d, D.marg_H0 = h->marg_H0.d, D.marg_b0 = h->marg_b0.d, D.marg_c0 = h->marg_c0.d;
    int rc = ICG_OK;
#define DM(field, count) \
    if (rc == ICG_OK) rc = dmalloc(h, &D.field, count);
    DM(pose_c, NW * C.K * 7) DM(mix_c, NW * C.K * 9) DM(ext_c, NW * 8) DM(rho_c, NW * C.L)
    DM(pose_0, NW * C.K * 7) DM(mix_0, NW * C.K * 9) DM(ext_0, NW * 8) DM(rho_0, NW * C.L)
    DM(AW[0], NW * C.NCA * C.LP) DM(Mp[0], NW * (size_t) C.K * (C.K - 1) * 210) DM(visv, NW * 3 * C.NCV)
    DM(gpart, NW * (size_t) C.GQ * 210) DM(costf[0], NW * C.F) DM(hl[0], NW * C.L) DM(gl[0], NW * C.L) DM(scale_l, NW * C.L) DM(scale_c, NW * C.NS)
    DM(Hc[0], NW * C.NS * C.NS) DM(gc[0], NW * C.NS) DM(Hs, NW * C.NS * C.NS) DM(cost_part, NW * (h->nblk_vis + 1)) DM(red2, NW * 4) DM(step_c, NW * C.NS) DM(step_l, NW * C.L)
#undef DM
    if (rc == ICG_OK) rc = dmalloc(h, &D.gnss_std_0, NW * C.G * 3);
    if (rc == ICG_OK) {
        double *cnt = nullptr;
        rc = dmalloc(h, &cnt, (NW * C.K + 1) / 2);  // zeroed: the arrival counters start at 0 and every lin_vis launch leaves them at 0
        D.vis_cnt = (int *) cnt;
    }
    if (rc == ICG_OK) {
        double *fa0 = nullptr;
        rc = dmalloc(h, &fa0, (NW * C.F + 7) / 8 + 1);
        D.f_active_0 = (uint8_t *) fa0;
    }
    if (rc == ICG_OK) rc = dmalloc(h, &h->lm_ref, NW * C.L * 7);
    if (rc == ICG_OK) rc = dmalloc(h, &h->lm_ref_alt, NW * C.L * 7);
    if (rc != ICG_OK) return rc;
    // shared-memory budgets
    h->smem_cam = sizeof(double) * ((size_t) C.K * 480 + (size_t) C.G * 24 + 48 + 16 + 2 * (size_t) C.R + 8) + sizeof(int) * (size_t) C.R + 64;
    size_t vec = sizeof(double) * (40 + 5 * (size_t) C.NS);
    size_t packed = sizeof(double) * ((size_t) (C.N + 1) * (C.N + 2) / 2);
    h->use_global_S = (vec + packed > 220 * 1024) ? 1 : 0;
    h->smem_solve = vec + (h->use_global_S ? 0 : packed);
    D.Sglobal = nullptr;
    memset(&D.S, 0, sizeof(D.S));
    if (h->use_global_S) {  // the reduced system does not fit one CTA: the split pipeline (cluster solve, S in L2) drives this handle
        rc = split_setup(h, 0, 1);
        if (rc != ICG_OK) return rc;
    } else {
        ICG_CUDA(raise_dynamic_smem((const void *) ba_solve, (size_t) (h->smem_solve)));
    }
    h->ld_schur = 16 * ((C.NCA + 15) / 16) + 8;  // = 8 mod 16 doubles: conflict-free fragment reads
    h->smem_schur = sizeof(double) * std::max((size_t) SCHUR_RCH * h->ld_schur + SCHUR_RCH, (size_t) SCHUR_PASS * 256);  // staging | one pass's partials
    ICG_CUDA(raise_dynamic_smem((const void *) ba_schur_dmma, (size_t) (h->smem_schur)));
    ICG_CUDA(cudaFuncSetAttribute(ba_schur_dmma, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    ICG_CUDA(raise_dynamic_smem((const void *) ba_lin_cam, (size_t) (h->smem_cam)));
    ICG_CUDA(raise_dynamic_smem((const void *) ba_cost_cam, (size_t) (h->smem_cam)));
    ICG_CUDA(raise_dynamic_smem((const void *) ba_lin_vis, LV_SMEM));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    h->cur_windows = 0;
    return ICG_OK;
}

void icg_ba_destroy(icg_ba *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    prof_collect(h);
    prof_print(h);
    for (cudaEvent_t e : h->prof_ev) cudaEventDestroy(e);
    h->dims.release(), h->st.release(), h->pose.release(), h->mix.release(), h->ext.release(), h->rho.release();
    h->imu_blob.release(), h->imu_U.release(), h->gnss_blh.release(), h->gnss_std.release(), h->lever.release(), h->pose_prior.release();
    h->pose_prior_sinfo.release(), h->mix_prior.release(), h->mix_prior_std.release(), h->marg_x0.release(), h->marg_H0.release(), h->marg_b0.release();
    h->marg_c0.release(), h->lm_off.release(), h->lm_perm.release(), h->lm_fidx.release(), h->gnss_node.release();
    h->f_meta_s.release(), h->vb_lm0.release(), h->ref_nrun.release(), h->f_const_s.release(), h->marg_type.release(), h->marg_node.release(), h->f_active.release(), h->scratch.release(), h->st_save.release(), h->cull_counters.release(), h->part_off.release(), h->pair_ro.release(), h->vis_ord.release(), h->npairs.release();
    split_release(h);
    if (h->mx_h) icg_ba_destroy(h->mx_h);
    h->xs_v.release(), h->mx_sel.release(), h->mx_row.release(), h->mx_heads.release(), h->mx_idx.release();
    if (h->mx_rows) cudaFree(h->mx_rows);
    if (h->marg_ready) h->marg_map.release(), h->marg_oJ0.release(), h->marg_oe0.release(), h->marg_oHp.release(), h->marg_obp.release(), h->marg_fmask.release();
    for (double *p : {h->M.H0, h->M.b0, h->M.G1, h->M.V1, h->M.lam1, h->M.Z})
        if (p) cudaFree(p);
    if (h->cull_h) cudaFreeHost(h->cull_h);
    if (h->cull_d) cudaFree(h->cull_d);
    if (h->reint_h) cudaFreeHost(h->reint_h);
    if (h->reint_d) cudaFree(h->reint_d);
    if (h->slide_h) cudaFreeHost(h->slide_h);
    if (h->slide_d) cudaFree(h->slide_d);
    if (h->vis_h) cudaFreeHost(h->vis_h);
    if (h->vis_d) cudaFree(h->vis_d);
    if (h->slide_old) cudaFree(h->slide_old);
    if (h->fc_alt) cudaFree(h->fc_alt);
    if (h->slide_ev) cudaEventDestroy(h->slide_ev);
    for (void *p : h->dev_only) cudaFree(p);
    if (h->stream_cam) cudaStreamSynchronize(h->stream_cam), cudaStreamDestroy(h->stream_cam);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->ev_join) cudaEventDestroy(h->ev_join);
    if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

// Every landmark's reference row (pts0, vel0, td0 of its factors' constants) into out: the old row of the landmark a slide carries (win / map:
// the slide's staging), otherwise its first factor's (record slot order), otherwise NaN.  One thread per landmark position, blockIdx.y = window.
__global__ void ba_lm_ref_fill(const WinDims *dims, const SlideWin *win, const int *map, const double *old, const double *fc, const int *lm_off,
                               const int *lm_perm, double *out, int Lc, int Fc) {
    const int w = blockIdx.y, L = dims[w].L;
    const size_t wL = (size_t) w * Lc;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < L; p += gridDim.x * blockDim.x) {
        const int l = lm_perm[wL + p], m = win ? map[win[w].lm_map + l] : -1;
        const int q0 = lm_off[(size_t) w * (Lc + 1) + p], q1 = lm_off[(size_t) w * (Lc + 1) + p + 1];
        double *r = out + (wL + l) * 7;
        if (m >= 0) {
            for (int c = 0; c < 7; c++) r[c] = old[(wL + m) * 7 + c];
        } else if (q1 > q0) {
            const double *f = fc + ((size_t) w * Fc + q0) * 14;
            r[0] = f[0], r[1] = f[1], r[2] = f[2], r[3] = f[6], r[4] = f[7], r[5] = f[8], r[6] = f[12];
        } else {
            for (int c = 0; c < 7; c++) r[c] = __longlong_as_double(0x7ff8000000000000LL);
        }
    }
}

static cudaError_t launch_lm_ref_fill(icg_ba *h, int n, const SlideWin *win, const int *map, const double *old, double *out) {
    const int gx = std::max(1, std::min(8, (h->C.L + 255) / 256));
    ba_lm_ref_fill<<<dim3(gx, n), 256, 0, h->stream>>>(h->D.dims, win, map, old, h->D.f_const_s, h->D.lm_off, h->D.lm_perm, out, h->C.L, h->C.F);
    count_launch();
    return cudaGetLastError();
}

// Packing of one window into the pinned staging arrays (host side of the seam: what AddParameterBlock / AddResidualBlock do in
// IG/ic_gvins.cc:1697-1909).  The structure part (validation, dims, landmark positions, CSR, lin_vis runs, pairs, vis_ord, GNSS nodes, the
// prior's block tables, factor activity, lever and first-window priors) is always packed; values = true adds the value part (parameters, factor
// constants, IMU blobs and U, GNSS fixes, the prior's H0 / b0 / c0), which icg_ba_slide_resident gathers on the device instead.
#define PK_FAIL(code, ...)                          \
    do {                                            \
        char eb_[512];                              \
        snprintf(eb_, sizeof(eb_), __VA_ARGS__);    \
        err = eb_;                                  \
        return code;                                \
    } while (0)
static int pack_window(icg_ba *h, int w, const icg_ba_problem &p, bool values, std::string &err) {
        const BaCaps &C = h->C;
        if (p.K < 2 || p.K > C.K || p.L < 0 || p.L > C.L || p.F < 0 || p.F > C.F || p.n_imu < 0 || p.n_imu > p.K - 1 || p.n_gnss < 0 || p.n_gnss > C.G ||
            p.marg_r < 0 || p.marg_r > C.R || p.marg_nblocks < 0 || p.marg_nblocks > 2 * C.K + 2 || !p.pose || !p.mix || !p.ext || (p.L > 0 && !p.invdepth) ||
            (p.F > 0 && (!p.f_lm || !p.f_ref || !p.f_obs || !p.f_const))) {
            PK_FAIL(ICG_EINVAL, "icg_ba_upload: window %d exceeds the handle's capacity or has null parameter arrays (K=%d L=%d F=%d gnss=%d marg_r=%d)", w, p.K, p.L, p.F,
                      p.n_gnss, p.marg_r);
        }
        WinDims &d = h->dims.h[w];
        d.K = p.K, d.L = p.L, d.F = p.F, d.n_imu = p.n_imu, d.n_gnss = p.n_gnss, d.marg_r = p.marg_r, d.marg_nb = p.marg_nblocks;
        d.ext_const = p.ext_const != 0, d.td_const = p.td_const != 0, d.reproj_huber = p.reproj_huber != 0, d.gnss_huber = p.gnss_huber != 0;
        d.has_imu_error = p.has_imu_error != 0, d.has_pose_prior = p.has_pose_prior != 0, d.has_mix_prior = p.has_mix_prior != 0;
        d.reproj_sinv = 1.0 / p.reproj_std;
        if (values) {
            memcpy(h->pose.h + (size_t) w * C.K * 7, p.pose, sizeof(double) * 7 * p.K);
            memcpy(h->mix.h + (size_t) w * C.K * 9, p.mix, sizeof(double) * 9 * p.K);
        }
        memcpy(h->ext.h + (size_t) w * 8, p.ext, sizeof(double) * 8);
        if (values && p.L > 0) memcpy(h->rho.h + (size_t) w * C.L, p.invdepth, sizeof(double) * p.L);
        for (int f = 0; f < p.F; f++) {
            if (p.f_lm[f] < 0 || p.f_lm[f] >= p.L || p.f_ref[f] < 0 || p.f_ref[f] >= p.K || p.f_obs[f] < 0 || p.f_obs[f] >= p.K || p.f_ref[f] == p.f_obs[f]) {
                PK_FAIL(ICG_EINVAL, "icg_ba_upload: window %d factor %d has invalid indices", w, f);
            }
        }
        std::vector<int> refof(p.L, -1);  // reference node of every landmark (-1: no factor)
        {   // a map point has one reference frame and at most one observation per keyframe (IG/ic_gvins.cc:1777-1834): lin_lm relies on it
            std::vector<unsigned> seen((size_t) p.L, 0u);
            for (int f = 0; f < p.F; f++) {
                const int l = p.f_lm[f];
                if (refof[l] < 0) refof[l] = p.f_ref[f];
                if (refof[l] != p.f_ref[f] || (seen[l] >> p.f_obs[f]) & 1u) {
                    PK_FAIL(ICG_EINVAL, "icg_ba_upload: window %d factor %d: landmark %d has two reference nodes or two observations in node %d", w, f, l, p.f_obs[f]);
                }
                seen[l] |= 1u << p.f_obs[f];
            }
        }
        if (p.f_active)
            memcpy(h->f_active.h + (size_t) w * C.F, p.f_active, p.F);
        else
            memset(h->f_active.h + (size_t) w * C.F, 1, p.F);
        // landmark positions: ordered by reference node, stable by id, landmarks without factors last
        int *perm = h->lm_perm.h + (size_t) w * C.L;
        std::vector<int> pos_of(p.L);
        {
            std::vector<int> kcur(p.K + 2, 0);
            for (int l = 0; l < p.L; l++) kcur[(refof[l] < 0 ? p.K : refof[l]) + 1]++;
            for (int k = 0; k <= p.K; k++) kcur[k + 1] += kcur[k];
            for (int l = 0; l < p.L; l++) pos_of[l] = kcur[refof[l] < 0 ? p.K : refof[l]]++, perm[pos_of[l]] = l;
        }
        // CSR by landmark position: the record slots
        int *off = h->lm_off.h + (size_t) w * (C.L + 1), *fidx = h->lm_fidx.h + (size_t) w * C.F;
        for (int l = 0; l <= p.L; l++) off[l] = 0;
        for (int f = 0; f < p.F; f++) off[pos_of[p.f_lm[f]] + 1]++;
        for (int l = 0; l < p.L; l++) off[l + 1] += off[l];
        int *vbh = h->vb_lm0.h + (size_t) w * C.NVB, *meta = h->f_meta_s.h + (size_t) w * C.F * 4;
        int nrun = 0;
        {
            std::vector<int> cur(off, off + p.L);
            for (int f = 0; f < p.F; f++) fidx[cur[pos_of[p.f_lm[f]]]++] = f;
            // lin_vis runs: greedy packing of whole landmarks of one reference node into <= 128 record slots
            int *nrun_of = h->ref_nrun.h + (size_t) w * C.K;
            for (int k = 0; k < C.K; k++) nrun_of[k] = 0;
            int l0 = 0;
            while (l0 < p.L) {
                const int ref = refof[perm[l0]];
                int l1 = l0;
                while (l1 < p.L && refof[perm[l1]] == ref && off[l1 + 1] - off[l0] <= 128) l1++;
                if (l1 == l0 || nrun >= C.NVB - 2) PK_FAIL(ICG_EINVAL, "icg_ba_upload: window %d: landmark %d has more than 128 factors or the run table overflows", w, perm[l0]);
                if (ref >= 0) nrun_of[ref]++;
                vbh[nrun++] = l0;
                l0 = l1;
            }
            vbh[nrun] = p.L;
            vbh[C.NVB - 1] = nrun;
            double *fcs = h->f_const_s.h + (size_t) w * C.F * 14;
            for (int q = 0; q < p.F; q++) {
                const int f = fidx[q];
                meta[4 * q] = p.f_lm[f], meta[4 * q + 1] = p.f_ref[f], meta[4 * q + 2] = p.f_obs[f], meta[4 * q + 3] = f;
                if (values) memcpy(fcs + (size_t) q * 14, p.f_const + (size_t) f * 14, sizeof(double) * 14);
            }
        }
        // (reference node, observing node) pairs and their Gram partials: one per (run, observing node of the run), numbered pair by pair
        // and, within a pair, in run order (the order ba_lin_vis sums them in); every run's slots ordered by observing node (stable)
        {
            const int PM = C.K * (C.K - 1);
            int *poff = h->part_off.h + (size_t) w * (PM + 1), *pro = h->pair_ro.h + (size_t) w * PM, *ord = h->vis_ord.h + (size_t) w * C.F;
            std::vector<int> slot((size_t) p.K * p.K, -1);
            for (int f = 0; f < p.F; f++) slot[(size_t) p.f_ref[f] * p.K + p.f_obs[f]] = 0;
            int P = 0;
            for (int key = 0; key < p.K * p.K; key++)
                if (slot[key] == 0) slot[key] = P, pro[P++] = ((key / p.K) << 8) | (key % p.K);
            std::vector<int> npart(P, 0);
            for (int r = 0; r < nrun; r++) {
                unsigned seen = 0u;
                for (int q = off[vbh[r]]; q < off[vbh[r + 1]]; q++) seen |= 1u << meta[4 * q + 2];
                for (int k = 0; k < p.K; k++)
                    if ((seen >> k) & 1u) npart[slot[(size_t) refof[perm[vbh[r]]] * p.K + k]]++;
            }
            poff[0] = 0;
            for (int i = 0; i < P; i++) poff[i + 1] = poff[i] + npart[i];
            std::vector<int> cur(poff, poff + P), start(p.K), pidx(p.K);
            for (int r = 0; r < nrun; r++) {
                const int a = off[vbh[r]], b = off[vbh[r + 1]];
                if (a == b) continue;
                const int ref = meta[4 * a + 1];
                std::fill(start.begin(), start.end(), 0);
                for (int q = a; q < b; q++) start[meta[4 * q + 2]]++;
                for (int k = 0, t = 0; k < p.K; k++) {
                    const int c = start[k];
                    start[k] = t, t += c;
                    if (c) pidx[k] = cur[slot[(size_t) ref * p.K + k]]++;
                }
                for (int q = a; q < b; q++) {
                    const int k = meta[4 * q + 2];
                    ord[a + start[k]++] = (q - a) | (pidx[k] << 8);
                }
            }
            h->npairs.h[w] = P;
        }
        for (int k = 0; values && k < p.n_imu; k++) {
            const double *b = p.imu_blob + (size_t) k * ICG_IMU_BLOB_DOUBLES;
            memcpy(h->imu_blob.h + ((size_t) w * C.K + k) * ICG_IMU_BLOB_DOUBLES, b, sizeof(double) * ICG_IMU_BLOB_DOUBLES);
            if (!host_imu_sqrt_info(b + 252, h->imu_U.h + ((size_t) w * C.K + k) * 225)) {
                PK_FAIL(ICG_EINVAL, "icg_ba_upload: window %d IMU factor %d has a non positive-definite covariance", w, k);
            }
        }
        for (int g = 0; g < p.n_gnss; g++) {
            if (p.gnss_node[g] < 0 || p.gnss_node[g] >= p.K) {
                PK_FAIL(ICG_EINVAL, "icg_ba_upload: window %d GNSS factor %d has an invalid node", w, g);
            }
            h->gnss_node.h[(size_t) w * C.G + g] = p.gnss_node[g];
        }
        if (values && p.n_gnss) {
            memcpy(h->gnss_blh.h + (size_t) w * C.G * 3, p.gnss_blh, sizeof(double) * 3 * p.n_gnss);
            memcpy(h->gnss_std.h + (size_t) w * C.G * 3, p.gnss_std, sizeof(double) * 3 * p.n_gnss);
        }
        memcpy(h->lever.h + (size_t) w * 3, p.lever, sizeof(double) * 3);
        if (p.has_pose_prior) {
            memcpy(h->pose_prior.h + (size_t) w * 7, p.pose_prior, sizeof(double) * 7);
            for (int k = 0; k < 6; k++) h->pose_prior_sinfo.h[(size_t) w * 6 + k] = 1.0 / p.pose_prior_std[k];
        }
        if (p.has_mix_prior) {
            memcpy(h->mix_prior.h + (size_t) w * 9, p.mix_prior, sizeof(double) * 9);
            memcpy(h->mix_prior_std.h + (size_t) w * 9, p.mix_prior_std, sizeof(double) * 9);
        }
        if (p.marg_r > 0) {
            // the prior is linear: H0 = J0^T J0, b0 = J0^T e0, c0 = e0.e0 are constant over the solve (marginalization_factor.h:79-81)
            const int r = p.marg_r;
            int tot = 0, cols = 0;
            for (int b = 0; b < p.marg_nblocks; b++) {
                int t = p.marg_block_type[b];
                if (t < 0 || t > 3 || ((t == 0 || t == 1) && (p.marg_block_node[b] < 0 || p.marg_block_node[b] >= p.K))) {
                    PK_FAIL(ICG_EINVAL, "icg_ba_upload: window %d marginalization block %d invalid", w, b);
                }
                tot += (t == 0 || t == 2) ? 7 : t == 1 ? 9 : 1;
                cols += (t == 0 || t == 2) ? 6 : t == 1 ? 9 : 1;
                h->marg_type.h[(size_t) w * BA_MARG_MAXB + b] = t;
                h->marg_node.h[(size_t) w * BA_MARG_MAXB + b] = p.marg_block_node[b];
            }
            if (cols != r || tot > BA_MARG_MAXB * 9) {
                PK_FAIL(ICG_EINVAL, "icg_ba_upload: window %d marginalization prior size mismatch (blocks give %d columns, marg_r=%d)", w, cols, r);
            }
            memcpy(h->marg_x0.h + (size_t) w * BA_MARG_MAXB * 9, p.marg_x0, sizeof(double) * tot);
            if (!values) return ICG_OK;
            double *H0 = h->marg_H0.h + (size_t) w * C.R * C.R, *b0 = h->marg_b0.h + (size_t) w * C.R;
            for (int i = 0; i < r; i++) {
                for (int j = i; j < r; j++) {
                    double s = 0;
                    for (int k = 0; k < r; k++) s += p.marg_J0[(size_t) k * r + i] * p.marg_J0[(size_t) k * r + j];
                    H0[(size_t) i * r + j] = H0[(size_t) j * r + i] = s;
                }
                double s = 0;
                for (int k = 0; k < r; k++) s += p.marg_J0[(size_t) k * r + i] * p.marg_e0[k];
                b0[i] = s;
            }
            double c0 = 0;
            for (int k = 0; k < r; k++) c0 += p.marg_e0[k] * p.marg_e0[k];
            h->marg_c0.h[w] = c0;
        }
            return ICG_OK;
}
#undef PK_FAIL

// pack_window over n windows.  Per-window packing is independent (disjoint slices of the pinned staging arrays): spread it over a few host
// threads -- it is memcpy-bound (about 0.4 MB per cfg-3 window) and sits inside the end-to-end path of every keyframe
static int pack_windows(icg_ba *h, int n, const icg_ba_problem *P, bool values) {
    const int nthreads = std::max(1, std::min({n / 4, 16, (int) std::thread::hardware_concurrency()}));
    std::vector<int> rcs(nthreads, ICG_OK);
    std::vector<std::string> errs(nthreads);
    auto worker = [&](int t) {
        for (int w = t; w < n; w += nthreads) {
            const int rc = pack_window(h, w, P[w], values, errs[t]);
            if (rc != ICG_OK) {
                rcs[t] = rc;
                return;
            }
        }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < nthreads; t++) th.emplace_back(worker, t);
    worker(0);
    for (auto &x : th) x.join();
    for (int t = 0; t < nthreads; t++)
        if (rcs[t] != ICG_OK) {
            set_error("%s", errs[t].c_str());
            return rcs[t];
        }
    return ICG_OK;
}

// H2D of the structure part of n packed windows only (the arrays are capacity-strided by window; a partially filled handle moves a prefix)
static int upload_structure(icg_ba *h, int n) {
    const BaCaps &C = h->C;
    cudaStream_t s = h->stream;
    const size_t nn = (size_t) n, PM = (size_t) C.K * (C.K - 1);
#define UP(field, stride) ICG_CUDA(h->field.up(s, nn * (size_t) (stride)))
    UP(dims, 1); UP(ext, 8);
    UP(f_active, C.F);  // factor constants and indices travel once, in record-slot order (f_meta_s / f_const_s)
    UP(f_meta_s, C.F * 4); UP(vb_lm0, C.NVB); UP(lm_off, C.L + 1); UP(lm_perm, C.L); UP(ref_nrun, C.K); UP(part_off, PM + 1); UP(pair_ro, PM); UP(vis_ord, C.F);
    UP(npairs, 1); UP(gnss_node, C.G); UP(lever, 3);
    UP(pose_prior, 7); UP(pose_prior_sinfo, 6); UP(mix_prior, 9); UP(mix_prior_std, 9);
    UP(marg_type, BA_MARG_MAXB); UP(marg_node, BA_MARG_MAXB); UP(marg_x0, BA_MARG_MAXB * 9);
#undef UP
    return ICG_OK;
}

// keep a pristine copy of the parameters and of what the two-pass protocol mutates (icg_ba_run(restart=1) re-solves the same problems: bench /
// repeated solves)
static int keep_pristine(icg_ba *h, int n) {
    const BaCaps &C = h->C;
    const BaDev &D = h->D;
    cudaStream_t s = h->stream;
    ICG_CUDA(cudaMemcpyAsync(D.pose_0, D.pose, sizeof(double) * (size_t) n * C.K * 7, cudaMemcpyDeviceToDevice, s));
    ICG_CUDA(cudaMemcpyAsync(D.mix_0, D.mix, sizeof(double) * (size_t) n * C.K * 9, cudaMemcpyDeviceToDevice, s));
    ICG_CUDA(cudaMemcpyAsync(D.ext_0, D.ext, sizeof(double) * (size_t) n * 8, cudaMemcpyDeviceToDevice, s));
    ICG_CUDA(cudaMemcpyAsync(D.rho_0, D.rho, sizeof(double) * (size_t) n * C.L, cudaMemcpyDeviceToDevice, s));
    ICG_CUDA(cudaMemcpyAsync(D.f_active_0, D.f_active, (size_t) n * C.F, cudaMemcpyDeviceToDevice, s));
    ICG_CUDA(cudaMemcpyAsync(D.gnss_std_0, D.gnss_std, sizeof(double) * (size_t) n * C.G * 3, cudaMemcpyDeviceToDevice, s));
    return ICG_OK;
}

// pack + upload n problems
int icg_ba_upload(icg_ba *h, int n, const icg_ba_problem *P) {
    if (!h || !P || n < 1 || n > h->C.NW) {
        set_error("icg_ba_upload: bad arguments (n=%d, capacity %d)", n, h ? h->C.NW : 0);
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    const BaCaps &C = h->C;
    h->marg_res_n = 0;  // the marginalization workspace no longer belongs to the windows the handle holds
    h->cull_res_n = 0;
    int rc = pack_windows(h, n, P, true);
    if (rc != ICG_OK) return rc;
    rc = upload_structure(h, n);
    if (rc != ICG_OK) return rc;
    cudaStream_t s = h->stream;
    const size_t nn = (size_t) n;
#define UP(field, stride) ICG_CUDA(h->field.up(s, nn * (size_t) (stride)))
    UP(pose, C.K * 7); UP(mix, C.K * 9); UP(rho, C.L); UP(f_const_s, C.F * 14); UP(imu_blob, C.K * ICG_IMU_BLOB_DOUBLES); UP(imu_U, C.K * 225);
    UP(gnss_blh, C.G * 3); UP(gnss_std, C.G * 3); UP(marg_H0, (size_t) C.R * C.R); UP(marg_b0, C.R); UP(marg_c0, 1);
#undef UP
    ICG_CUDA(launch_lm_ref_fill(h, n, nullptr, nullptr, nullptr, h->lm_ref));
    rc = keep_pristine(h, n);
    if (rc != ICG_OK) return rc;
    h->cur_windows = n;
    return ICG_OK;
}

// ---- in-situ stage timing
static const char *PROF_NAMES[16] = {"(gap/other)", "lin_vis", "lin_lm", "lin at candidate", "","schur_dmma (+ epilogue)", "join lin_cam + lin_done",
                                     "signal", "solve", "cost (+cost_cam)", "exchange", "accept", "reduce", "join gram chain", "step_lm", ""};
static void prof_mark(icg_ba *h, int tag) {
    if (!h->prof) return;
    if (h->prof_used == h->prof_ev.size()) {
        cudaEvent_t e;
        cudaEventCreate(&e);
        h->prof_ev.push_back(e);
        h->prof_tag.push_back(0);
    }
    h->prof_tag[h->prof_used] = tag;
    cudaEventRecord(h->prof_ev[h->prof_used++], h->stream);
}
static void prof_collect(icg_ba *h) {  // call after the stream has been synchronised
    if (!h->prof) return;
    if (h->prof_used && h->prof_skip > 0) {
        h->prof_skip--;
        h->prof_used = 0;
        return;
    }
    for (size_t i = 1; i < h->prof_used; i++) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, h->prof_ev[i - 1], h->prof_ev[i]) == cudaSuccess) {
            h->prof_ms[h->prof_tag[i]] += ms;
            h->prof_cnt[h->prof_tag[i]]++;
        }
    }
    h->prof_used = 0;
}
static void prof_print(icg_ba *h) {
    if (!h->prof) return;
    double tot = 0;
    for (int t = 0; t < 16; t++) tot += h->prof_ms[t];
    fprintf(stderr, "[icg_ba profile] handle %p, %d windows: stage totals over all recorded LM sequences (ms, mean us, share)\n", (void *) h, h->cur_windows);
    for (int t = 0; t < 16; t++)
        if (h->prof_cnt[t])
            fprintf(stderr, "  %-28s %9.3f ms  %8.1f us  %5.1f %%\n", PROF_NAMES[t], h->prof_ms[t], 1e3 * h->prof_ms[t] / h->prof_cnt[t], 100.0 * h->prof_ms[t] / tot);
    if (h->D.clk) {
        unsigned long long ck[48];
        if (cudaMemcpy(ck, h->D.clk, sizeof(ck), cudaMemcpyDeviceToHost) == cudaSuccess) {
            static const char *cn[6] = {"factor evaluation", "prior product + cost", "zero H_c", "prior blocks", "IMU J^T J", "GNSS / prior diagonals"};
            fprintf(stderr, "[icg_ba profile] ba_lin_cam phases of window 0 (SM cycles per call, mean):\n");
            for (int k = 0; k < 6; k++)
                if (ck[24 + k]) fprintf(stderr, "  %-28s %9.0f cycles\n", cn[k], (double) ck[16 + k] / (double) ck[24 + k]);
            if (h->D.S.split) {
                static const char *sn_l2[6] = {"per panel: stage B operand", "per panel: warp 0 tile + factor", "per panel: tiles + barrier 1", "per panel: row solve + barrier 2", "whole factorisation", ""};
                static const char *sn_dsm[6] = {"assembly", "per panel: warp 0 tile + factor", "per panel: until block barrier", "per panel: row solve + cl. barrier", "whole factorisation", "backward substitution"};
                const char **sn = h->solve_cam_dsm ? sn_dsm : sn_l2;
                fprintf(stderr, "[icg_ba profile] %s phases of window 0 (SM cycles, mean):\n", h->solve_cam_dsm ? "ba_solve_cam_dsm" : "ba_solve_cam");
                for (int k = 0; k < 6; k++)
                    if (ck[8 + k]) fprintf(stderr, "  %-34s %9.0f cycles\n", sn[k], (double) ck[k] / (double) ck[8 + k]);
                static const char *sn2[5] = {"(unused)", "(unused)", "per panel: warp 0 diagonal-tile update", "per panel: warp 0 loads + 8x8 factorisation", "per panel: warp 0 write-back"};
                for (int k = 0; k < 5 && h->solve_cam_dsm; k++)
                    if (ck[40 + k]) fprintf(stderr, "  %-50s %9.0f cycles\n", sn2[k], (double) ck[32 + k] / (double) ck[40 + k]);
            }
            static const char *nm[8] = {"gradient / cost / tests", "assembly", "Cholesky", "camera back-substitution", "landmark back-substitution", "candidate + reductions",
                                        "  per panel: warp 0 tile+factor", "  per panel: row solve phase"};
            if (!h->D.S.split) fprintf(stderr, "[icg_ba profile] ba_solve phases of window 0 (SM cycles per call, mean):\n");
            for (int k = 0; k < 8 && !h->D.S.split; k++)
                if (ck[8 + k]) fprintf(stderr, "  %-28s %9.0f cycles\n", nm[k], (double) ck[k] / (double) ck[8 + k]);
        }
    }
}

static int enqueue_lm_split(icg_ba *h, int max_num_iterations);

// The second linearisation buffer (BaDev::Mp etc.), allocated on the first LM sequence of the single-GPU pipeline: handles that the split
// pipeline drives never linearise a candidate and do not pay for it (~80 MB for 148 windows at K = 10, L = 300).
static int alloc_lin_buf2(icg_ba *h) {
    BaDev &D = h->D;
    if (D.Mp[1]) return ICG_OK;
    const BaCaps &C = h->C;
    const size_t NW = C.NW;
    int rc = ICG_OK;
#define DM(field, count) \
    if (rc == ICG_OK) rc = dmalloc(h, &D.field, count);
    DM(AW[1], NW * C.NCA * C.LP) DM(Mp[1], NW * (size_t) C.K * (C.K - 1) * 210) DM(costf[1], NW * C.F) DM(hl[1], NW * C.L) DM(gl[1], NW * C.L)
    DM(Hc[1], NW * C.NS * C.NS) DM(gc[1], NW * C.NS)
#undef DM
    return rc;
}

static int enqueue_lm(icg_ba *h, int max_num_iterations) {
    if (h->D.S.split) return enqueue_lm_split(h, max_num_iterations);
    int rc = alloc_lin_buf2(h);
    if (rc != ICG_OK) return rc;
    const BaCaps &C = h->C;
    const BaDev &D = h->D;
    const int n = h->cur_windows;
    cudaStream_t s = h->stream;
    const dim3 g_vis(C.NVB - 2, n);
    // Linearisation at x (iteration 0) + (max_iter) x [schur syrk, solve, linearisation at the candidate, accept]; one extra schur + solve
    // performs the final termination bookkeeping.  The linearisation at the candidate goes into the window's other buffer: its per-factor
    // costs are the candidate cost ba_accept tests, and an accepted step flips the buffers instead of linearising again at the new x; a
    // rejected one leaves the linearisation at x untouched.
    // the linearisation (at x or at the candidate); the camera-only factors are joined before the next kernel reads H_c
    auto enqueue_lin = [&](int at_cand) -> int {
        // fork: IMU / GNSS / prior factors (one latency-bound CTA per window) run beside the vision chain -- forked ahead of ba_lin_vis, so
        // that the two overlap (measured against a fork behind it with in-kernel phase clocks, ICG_BA_PROFILE)
        ICG_CUDA(cudaEventRecord(h->ev_fork, s));
        ICG_CUDA(cudaStreamWaitEvent(h->stream_cam, h->ev_fork, 0));
        ba_lin_cam<<<n, cam_threads(h), h->smem_cam, h->stream_cam>>>(C, D, at_cand);
        ICG_CUDA(cudaEventRecord(h->ev_join, h->stream_cam));
        prof_mark(h, 0);
        ba_lin_vis<<<g_vis, 128, LV_SMEM, s>>>(C, D, at_cand);
        prof_mark(h, at_cand ? 3 : 1);
        // (measured: one fused launch or two streams are both slower -- the Schur CTAs' shared memory throttles the latency-bound
        //  Gram warps when they share SMs)
        ICG_CUDA(cudaStreamWaitEvent(s, h->ev_join, 0));
        prof_mark(h, at_cand ? 3 : 6);
        count_launch(2);
        return ICG_OK;
    };
    rc = enqueue_lin(0);
    if (rc != ICG_OK) return rc;
    for (int it = 0; it <= max_num_iterations; it++) {
        ba_schur_dmma<<<dim3(BA_SPLIT_W, n), 256, h->smem_schur, s>>>(C, D, h->ld_schur);
        prof_mark(h, 5);
        ba_solve<<<n, SOLVE_THREADS, h->smem_solve, s>>>(C, D);
        prof_mark(h, 8);
        count_launch(2);
        if (it == max_num_iterations) break;
        rc = enqueue_lin(1);
        if (rc != ICG_OK) return rc;
        ba_accept<<<n, 128, sizeof(double) * 8 * h->nblk_vis, s>>>(C, D);  // one double per 32 record slots
        prof_mark(h, 11);
        count_launch();
    }
    ICG_CHECK_LAUNCH();
    return ICG_OK;
}

// ---- split pipeline: host side
// a buffer outgrown by a call: freed now on a single rank, kept until the group is left in a shard group (icg_ba::retired_d)
static void retire(icg_ba *h, void *d, void *hp) {
    if (h->D.world > 1) {
        if (d) h->retired_d.push_back(d);
        if (hp) h->retired_h.push_back(hp);
        return;
    }
    if (d) cudaFree(d);
    if (hp) cudaFreeHost(hp);
}

static void split_release(icg_ba *h) {
    if (h->stream) cudaStreamSynchronize(h->stream);
    for (void *p : h->retired_d) cudaFree(p);
    for (void *p : h->retired_h) cudaFreeHost(p);
    for (icg_ba *m : h->retired_mx) icg_ba_destroy(m);
    h->retired_d.clear(), h->retired_h.clear(), h->retired_mx.clear();
    for (int r = 0; r < 8; r++)
        if (h->ipc_opened[r]) cudaIpcCloseMemHandle(h->ipc_opened[r]), h->ipc_opened[r] = nullptr;
    if (h->xbuf) cudaFree(h->xbuf), h->xbuf = nullptr;
    if (h->D.S.redv) cudaFree(h->D.S.redv), h->D.S.redv = nullptr;
    if (h->D.S.err) cudaFree(h->D.S.err), h->D.S.err = nullptr;
    if (h->D.S.slm) cudaFree(h->D.S.slm), h->D.S.slm = nullptr;
    if (h->D.S.slm_cnt) cudaFree(h->D.S.slm_cnt), h->D.S.slm_cnt = nullptr;
    if (h->D.Sglobal) cudaFree(h->D.Sglobal), h->D.Sglobal = nullptr;
    h->D.S.split = 0;
}

// Under lazy module loading (the CUDA 12 default) a kernel is loaded at its first launch, and the load waits for the kernels running in the
// context.  Ranks driven by one process share the context: a rank's first launch of a kernel would wait for a peer's kernel that spins on
// this very rank's flags, until the bounded wait gives up.  A group therefore loads every kernel its calls launch when it is set up.
static int preload_group_kernels() {
    const void *k[] = {(const void *) ba_accept, (const void *) ba_accept_split, (const void *) ba_chi2_cull, (const void *) ba_cost, (const void *) ba_cost_cam,
                       (const void *) ba_exchange, (const void *) ba_lin_cam, (const void *) ba_lin_vis, (const void *) ba_marg_export, (const void *) ba_marg_fill,
                       (const void *) ba_marg_gather, (const void *) ba_marg_heads, (const void *) ba_reduce, (const void *) ba_reset_state,
                       (const void *) ba_schur_dmma, (const void *) ba_set_gnss_huber, (const void *) ba_signal, (const void *) ba_solve, (const void *) ba_solve_cam,
                       (const void *) ba_solve_cam_dsm, (const void *) ba_step_lm, (const void *) ba_xflag, (const void *) ba_xsum, (const void *) marg_assemble,
                       (const void *) marg_finish, (const void *) marg_jacobi, (const void *) marg_jacobi_cluster, (const void *) marg_jacobi_cta,
                       (const void *) marg_jacobi_pair, (const void *) marg_prepare, (const void *) marg_schur};
    cudaFuncAttributes a;
    for (const void *f : k) ICG_CUDA(cudaFuncGetAttributes(&a, f));
    ICG_CUDA(preload_update_cull());
    ICG_CUDA(preload_slide());
    ICG_CUDA(preload_preint_resident());
    return ICG_OK;
}

// (re)allocate the exchange buffer of this rank for a group of `world` ranks and switch the handle to the split pipeline.  The layout
// depends only on (max_windows, max_K, world), so every rank computes the same offsets.
static int split_setup(icg_ba *h, int rank, int world) {
    if (world < 1 || world > 8 || rank < 0 || rank >= world) {
        set_error("split pipeline: rank %d / world %d out of range (<= 8 GPUs of one box)", rank, world);
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    split_release(h);
    const BaCaps &C = h->C;
    ShardDev &S = h->D.S;
    const size_t NW = C.NW, G = world;
    const size_t TRI = (size_t) C.NCV * (C.NCV + 1) / 2;
    S.PK = (int) ((TRI + 3 * (size_t) C.NCV + 4 + 3) & ~(size_t) 3);
    S.BS = (SPLIT_HDR + C.NS + 3) & ~3;
    S.RV = (3 * C.NCV + 4 + 3) & ~3;
    const size_t NWo = (NW + G - 1) / G;
    size_t off = 0;
    S.off_inbox = off, off += NWo * G * S.PK;
    S.off_bcast = off, off += NW * S.BS;
    S.off_scal = off, off += NW * G * SPLIT_SCAL;
    S.off_flagA = off, off += 8;
    S.off_flagB = off, off += (NW + 3) & ~(size_t) 3;
    S.off_flagC = off, off += (NW * G + 3) & ~(size_t) 3;
    S.off_flagX = off, off += 3 * 8;
    S.off_post = off, off += 2 * NW * G * SPLIT_SCAL;
    S.off_exp = off;  // the part every rank lays out alike ends here; the export region follows at this rank's own max_F
    if (world > 1) off += 2 * NW + NW * (size_t) C.F * MEXP_ROW;
    h->xbuf_doubles = off;
    h->xs_calls = 0, h->exp_epoch = 0;
    if (world > 1) {
        const int rc = preload_group_kernels();
        if (rc != ICG_OK) return rc;
        if (!h->xs_v.d && h->xs_v.alloc(16) != ICG_OK) {
            set_error("split pipeline: allocation of the exchange word failed");
            return ICG_ENOMEM;
        }
    }
    if (cudaMalloc(&h->xbuf, sizeof(double) * off) != cudaSuccess || cudaMalloc(&S.redv, sizeof(double) * NW * S.RV) != cudaSuccess ||
        cudaMalloc(&S.err, sizeof(int) * 4) != cudaSuccess || cudaMalloc(&S.slm, sizeof(double) * NW * STEP_SLICES * 8) != cudaSuccess ||
        cudaMalloc(&S.slm_cnt, sizeof(int) * NW) != cudaSuccess ||
        cudaMalloc(&h->D.Sglobal, sizeof(double) * NWo * split_S_stride(C)) != cudaSuccess) {
        set_error("split pipeline: allocation of the exchange buffers failed (%zu doubles)", off);
        return ICG_ENOMEM;
    }
    ICG_CUDA(cudaMemset(h->xbuf, 0, sizeof(double) * off));
    ICG_CUDA(cudaMemset(S.redv, 0, sizeof(double) * NW * S.RV));
    ICG_CUDA(cudaMemset(S.err, 0, sizeof(int) * 4));
    ICG_CUDA(cudaMemset(S.slm, 0, sizeof(double) * NW * STEP_SLICES * 8));
    ICG_CUDA(cudaMemset(S.slm_cnt, 0, sizeof(int) * NW));
    for (int r = 0; r < 8; r++) S.peer[r] = nullptr;
    S.peer[rank] = h->xbuf;
    S.split = 1;
    h->D.rank = rank, h->D.world = world;
    h->x_world = world;
    h->epoch = 0;
    {   // ba_solve_cam: vectors + the larger of the back-substitution staging and [B rows | 8 x 8 hand-over]
        const size_t ldbp = ((size_t) (C.N + 15) / 16) * 16 + 8;
        const size_t bs = (size_t) SPLIT_BS_ROWS * (C.NS + 1), base = 8 * ldbp + 64;
        h->smem_solve_cam = sizeof(double) * (40 + 4 * (size_t) C.NS + std::max(bs, base));
    }
    h->smem_step_lm = sizeof(double) * (40 + (size_t) C.NS);
    h->smem_solve_cam_dsm = sizeof(double) * dsm_smem_doubles(C);
    // the shared-memory form wherever it fits, max_K <= 23 (the assembly stages <= 11 chunks of 32 columns per row); ba_solve_cam beyond
    h->solve_cam_dsm = h->smem_solve_cam_dsm <= 227 * 1024 && C.N <= 32 * 11;
    if (h->solve_cam_dsm) ICG_CUDA(raise_dynamic_smem((const void *) ba_solve_cam_dsm, h->smem_solve_cam_dsm));
    ICG_CUDA(raise_dynamic_smem((const void *) ba_solve_cam, (size_t) (h->smem_solve_cam)));
    ICG_CUDA(cudaFuncSetAttribute(ba_solve_cam, cudaFuncAttributeNonPortableClusterSizeAllowed, 0));
    ICG_CUDA(raise_dynamic_smem((const void *) ba_step_lm, (size_t) (h->smem_step_lm)));
    return ICG_OK;
}

static int launch_solve_cam(icg_ba *h, int n, unsigned long long epoch) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned) (n * SPLIT_CLUSTER)), cfg.blockDim = dim3(SOLVE_THREADS);
    cfg.dynamicSmemBytes = h->solve_cam_dsm ? h->smem_solve_cam_dsm : h->smem_solve_cam, cfg.stream = h->stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = SPLIT_CLUSTER, at[0].val.clusterDim.y = 1, at[0].val.clusterDim.z = 1;
    cfg.attrs = at, cfg.numAttrs = 1;
    if (h->solve_cam_dsm) ICG_CUDA(cudaLaunchKernelEx(&cfg, ba_solve_cam_dsm, h->C, h->D, epoch));
    else ICG_CUDA(cudaLaunchKernelEx(&cfg, ba_solve_cam, h->C, h->D, epoch));
    return ICG_OK;
}

// One LM sequence of the split pipeline (see ba_split.cuh).  Window w of a sharded group is solved by rank w mod world; the solve kernel
// is launched over all windows and the clusters of windows owned elsewhere return at once.
static int enqueue_lm_split(icg_ba *h, int max_num_iterations) {
    const BaCaps &C = h->C;
    const BaDev &D = h->D;
    const int n = h->cur_windows;
    cudaStream_t s = h->stream;
    for (int r = 0; r < D.world; r++)
        if (!D.S.peer[r]) {
            set_error("landmark-sharded solve: peer %d is not connected (icg_ba_shard_connect)", r);
            return ICG_EINVAL;
        }
    const dim3 g_vis(C.NVB - 2, n), g_cost(h->nblk_vis, n), g_nn(((C.NCV + 1) * (C.NCV + 1) + 255) / 256, n);
    for (int it = 0; it <= max_num_iterations; it++) {
        const unsigned long long epoch = ++h->epoch;
        ICG_CUDA(cudaEventRecord(h->ev_fork, s));
        ICG_CUDA(cudaStreamWaitEvent(h->stream_cam, h->ev_fork, 0));
        ba_lin_cam<<<n, cam_threads(h), h->smem_cam, h->stream_cam>>>(C, D, 0);
        ICG_CUDA(cudaEventRecord(h->ev_join, h->stream_cam));
        prof_mark(h, 0);
        ba_lin_vis<<<g_vis, 128, LV_SMEM, s>>>(C, D, 0);
        prof_mark(h, 1);
        ba_schur_dmma<<<dim3(BA_SPLIT_W, n), 256, h->smem_schur, s>>>(C, D, h->ld_schur);  // + the export into the owner's inbox
        prof_mark(h, 5);
        ba_signal<<<1, 32, 0, s>>>(D, epoch);
        prof_mark(h, 7);
        ICG_CUDA(cudaStreamWaitEvent(s, h->ev_join, 0));
        prof_mark(h, 6);
        ba_reduce<<<g_nn, 256, 0, s>>>(C, D, epoch);
        prof_mark(h, 12);
        int rc = launch_solve_cam(h, n, epoch);
        if (rc != ICG_OK) return rc;
        prof_mark(h, 8);
        ba_step_lm<<<dim3(n, STEP_SLICES), SOLVE_THREADS, h->smem_step_lm, s>>>(C, D, epoch);
        prof_mark(h, 14);
        count_launch(7);
        if (it == max_num_iterations) break;
        ICG_CUDA(cudaEventRecord(h->ev_fork, s));
        ICG_CUDA(cudaStreamWaitEvent(h->stream_cam, h->ev_fork, 0));
        ba_cost_cam<<<n, cam_threads(h), h->smem_cam, h->stream_cam>>>(C, D, h->nblk_vis);
        ICG_CUDA(cudaEventRecord(h->ev_join, h->stream_cam));
        ba_cost<<<g_cost, 256, 0, s>>>(C, D, h->nblk_vis);
        ICG_CUDA(cudaStreamWaitEvent(s, h->ev_join, 0));
        prof_mark(h, 9);
        ba_exchange<<<(n + 63) / 64, 64, 0, s>>>(C, D, n, h->nblk_vis, epoch);
        prof_mark(h, 10);
        ba_accept_split<<<n, 128, 0, s>>>(C, D, epoch);
        prof_mark(h, 11);
        count_launch(4);
    }
    ICG_CHECK_LAUNCH();
    return ICG_OK;
}

static int restore_params(icg_ba *h) {
    const BaCaps &C = h->C;
    const BaDev &D = h->D;
    const int n = h->cur_windows;
    cudaStream_t s = h->stream;
    ICG_CUDA(cudaMemcpyAsync(D.pose, D.pose_0, sizeof(double) * (size_t) n * C.K * 7, cudaMemcpyDeviceToDevice, s));
    ICG_CUDA(cudaMemcpyAsync(D.mix, D.mix_0, sizeof(double) * (size_t) n * C.K * 9, cudaMemcpyDeviceToDevice, s));
    ICG_CUDA(cudaMemcpyAsync(D.ext, D.ext_0, sizeof(double) * (size_t) n * 8, cudaMemcpyDeviceToDevice, s));
    ICG_CUDA(cudaMemcpyAsync(D.rho, D.rho_0, sizeof(double) * (size_t) n * C.L, cudaMemcpyDeviceToDevice, s));
    // problem data the two-pass protocol mutates: factor activity, GNSS std (device-side pristine copies: the pinned staging buffers
    // receive the culled / re-weighted results in icg_ba_gvins_optimization_end), GNSS loss flag
    ICG_CUDA(cudaMemcpyAsync(D.f_active, D.f_active_0, (size_t) n * C.F, cudaMemcpyDeviceToDevice, s));
    ICG_CUDA(cudaMemcpyAsync(D.gnss_std, D.gnss_std_0, sizeof(double) * (size_t) n * C.G * 3, cudaMemcpyDeviceToDevice, s));
    ICG_CUDA(h->dims.up(s, n));
    return ICG_OK;
}

// enqueue the LM iterations for the uploaded problems (asynchronous; device-resident decisions)
int icg_ba_run(icg_ba *h, int max_num_iterations, int restart) {
    if (!h || h->cur_windows < 1 || max_num_iterations < 0) {
        set_error("icg_ba_run: no problems uploaded");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    const int n = h->cur_windows;
    if (restart) {
        int rc = restore_params(h);
        if (rc != ICG_OK) return rc;
    }
    ba_reset_state<<<(n + 127) / 128, 128, 0, h->stream>>>(h->D, nullptr, n, max_num_iterations);
    count_launch();
    return enqueue_lm(h, max_num_iterations);
}

// GVINS::gvinsOptimization (IG/ic_gvins.cc:1130-1239) entirely on the stream: pass 1 (N/4 iterations, Huber on GNSS),
// chi-square culling, pass 2 (N - N/4 iterations, GNSS without loss).  No host round trip between the passes.
int icg_ba_run_gvins(icg_ba *h, int num_iterations, int restart) {
    if (!h || h->cur_windows < 1 || num_iterations < 1) {
        set_error("icg_ba_run_gvins: no problems uploaded");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    const BaCaps &C = h->C;
    const int n = h->cur_windows;
    const int first = num_iterations / 4, second = num_iterations - first;  // IG/ic_gvins.cc:1131-1132
    if (restart) {
        int rc = restore_params(h);
        if (rc != ICG_OK) return rc;
    }
    cudaStream_t s = h->stream;
    ba_set_gnss_huber<<<(n + 127) / 128, 128, 0, s>>>(h->D, n, 1);
    ba_reset_state<<<(n + 127) / 128, 128, 0, s>>>(h->D, nullptr, n, first);
    count_launch(2);
    int rc = enqueue_lm(h, first);
    if (rc != ICG_OK) return rc;
    ICG_CUDA(cudaMemsetAsync(h->cull_counters.d, 0, sizeof(int) * 2 * (size_t) n, s));
    const dim3 g_cull((std::max(C.F, C.G) + 127) / 128, n);
    ba_chi2_cull<<<g_cull, 128, 0, s>>>(C, h->D, h->cull_counters.d);
    ba_set_gnss_huber<<<(n + 127) / 128, 128, 0, s>>>(h->D, n, 0);
    ba_reset_state<<<(n + 127) / 128, 128, 0, s>>>(h->D, h->st_save.d, n, second);
    count_launch(3);
    return enqueue_lm(h, second);
}

int icg_ba_download(icg_ba *h, int n, const icg_ba_problem *P, icg_ba_summary *summaries) {
    if (!h || n < 1 || n > h->cur_windows) {
        set_error("icg_ba_download: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    const BaCaps &C = h->C;
    cudaStream_t s = h->stream;
    ICG_CUDA(h->pose.down(s, (size_t) n * C.K * 7)); ICG_CUDA(h->mix.down(s, (size_t) n * C.K * 9)); ICG_CUDA(h->ext.down(s, (size_t) n * 8));
    ICG_CUDA(h->rho.down(s, (size_t) n * C.L)); ICG_CUDA(h->st.down(s, n));
    ICG_CUDA(cudaStreamSynchronize(s));
    if (h->D.S.split && icg_ba_shard_error(h) != 0) {
        set_error("icg_ba_download: a peer exchange of the split pipeline timed out (a rank of the shard group did not run the same sequence)");
        return ICG_ECUDA;
    }
    for (int w = 0; w < n; w++) {
        if (P) {
            const icg_ba_problem &p = P[w];
            memcpy(p.pose, h->pose.h + (size_t) w * C.K * 7, sizeof(double) * 7 * p.K);
            memcpy(p.mix, h->mix.h + (size_t) w * C.K * 9, sizeof(double) * 9 * p.K);
            memcpy(p.ext, h->ext.h + (size_t) w * 8, sizeof(double) * 8);
            if (p.L > 0) memcpy(p.invdepth, h->rho.h + (size_t) w * C.L, sizeof(double) * p.L);
        }
        if (summaries) {
            const LmState &st = h->st.h[w];
            icg_ba_summary &o = summaries[w];
            o.iterations = st.iter, o.num_successful_steps = st.n_success;
            o.termination = st.done == 2 ? 1 : st.done == 3 ? 2 : 0;
            o.reserved = 0;
            o.initial_cost = st.initial_cost, o.final_cost = st.x_cost, o.final_radius = st.radius;
        }
    }
    return ICG_OK;
}

int icg_ba_solve(icg_ba *h, int n_windows, const icg_ba_problem *problems, int max_num_iterations, icg_ba_summary *summaries) {
    int rc = icg_ba_upload(h, n_windows, problems);
    if (rc != ICG_OK) return rc;
    rc = icg_ba_run(h, max_num_iterations, 0);
    if (rc != ICG_OK) return rc;
    return icg_ba_download(h, n_windows, problems, summaries);
}

static void fill_summary(const LmState &st, icg_ba_summary &o) {
    o.iterations = st.iter, o.num_successful_steps = st.n_success;
    o.termination = st.done == 2 ? 1 : st.done == 3 ? 2 : 0;
    o.reserved = 0;
    o.initial_cost = st.initial_cost, o.final_cost = st.x_cost, o.final_radius = st.radius;
}

int icg_ba_gvins_optimization_begin(icg_ba *h, int n_windows, const icg_ba_problem *problems, int num_iterations) {
    int rc = icg_ba_upload(h, n_windows, problems);
    if (rc != ICG_OK) return rc;
    return icg_ba_run_gvins(h, num_iterations, 0);
}

int icg_ba_gvins_optimization_end(icg_ba *h, int n_windows, const icg_ba_problem *problems, icg_ba_summary *summaries, int32_t *culled) {
    if (!h || !problems || n_windows < 1 || n_windows > h->cur_windows) {
        set_error("icg_ba_gvins_optimization_end: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    const BaCaps &C = h->C;
    cudaStream_t s = h->stream;
    ICG_CUDA(h->st_save.down(s, n_windows));
    ICG_CUDA(h->cull_counters.down(s, 2 * (size_t) n_windows));
    ICG_CUDA(h->f_active.down(s, (size_t) n_windows * C.F));
    ICG_CUDA(h->gnss_std.down(s, (size_t) n_windows * C.G * 3));
    std::vector<icg_ba_summary> second(n_windows);
    int rc = icg_ba_download(h, n_windows, problems, second.data());
    if (rc != ICG_OK) return rc;
    for (int w = 0; w < n_windows; w++) {
        const icg_ba_problem &p = problems[w];
        // the reference mutates gnss->std in place and removes residual blocks from the problem: mirror both
        if (p.f_active) memcpy(const_cast<uint8_t *>(p.f_active), h->f_active.h + (size_t) w * C.F, p.F);
        if (p.n_gnss) memcpy(const_cast<double *>(p.gnss_std), h->gnss_std.h + (size_t) w * C.G * 3, sizeof(double) * 3 * p.n_gnss);
        if (summaries) {
            fill_summary(h->st_save.h[w], summaries[2 * w]);
            summaries[2 * w + 1] = second[w];
        }
        if (culled) culled[2 * w] = h->cull_counters.h[2 * w], culled[2 * w + 1] = h->cull_counters.h[2 * w + 1];
    }
    return ICG_OK;
}

int icg_ba_gvins_optimization(icg_ba *h, int n_windows, const icg_ba_problem *problems, int num_iterations, icg_ba_summary *summaries,
                              int32_t *culled) {
    int rc = icg_ba_gvins_optimization_begin(h, n_windows, problems, num_iterations);
    if (rc != ICG_OK) return rc;
    return icg_ba_gvins_optimization_end(h, n_windows, problems, summaries, culled);
}

// ---- marginalization (B10)
constexpr int MARG_MAXN = 512;  // rows of the largest block an eigensolver takes (marg_jacobi: RPL = 16 rows per lane)

// The parts of the workspace that do not depend on the batch: the structure map, the outputs (rcap = N per window), the Jacobi workspace
// of Hp (n = r <= N) and the saved flags
static int marg_alloc(icg_ba *h) {
    if (h->marg_ready) return ICG_OK;
    const BaCaps &C = h->C;
    MargDev &M = h->M;
    const size_t NW = C.NW;
    M.rcap = C.N, M.mcap = 0, M.n0cap = 0;
    M.map_stride = MARG_MAP_HDR + 2 * C.K + C.L;
    if (h->marg_map.alloc(NW * M.map_stride) != ICG_OK || h->marg_oJ0.alloc(NW * (size_t) M.rcap * M.rcap) != ICG_OK || h->marg_oe0.alloc(NW * M.rcap) != ICG_OK ||
        h->marg_oHp.alloc(NW * (size_t) M.rcap * M.rcap) != ICG_OK || h->marg_obp.alloc(NW * M.rcap) != ICG_OK || h->marg_fmask.alloc(NW * C.F) != ICG_OK) {
        set_error("icg_ba_marginalize: workspace allocation failed");
        return ICG_ENOMEM;
    }
    M.map = h->marg_map.d, M.J0 = h->marg_oJ0.d, M.e0 = h->marg_oe0.d, M.Hp = h->marg_oHp.d, M.bp = h->marg_obp.d;
    int rc = ICG_OK;
    double *fl = nullptr;
#define DM(ptr, count) \
    if (rc == ICG_OK) rc = dmalloc(h, &ptr, count);
    DM(M.G2, NW * (size_t) M.rcap * M.rcap) DM(M.V2, NW * (size_t) M.rcap * M.rcap) DM(M.lam2, NW * M.rcap) DM(fl, NW * 2)
#undef DM
    if (rc != ICG_OK) return rc;
    M.flags = (int *) fl;
    const size_t smem = sizeof(double) * (8 * 480 + 2 * (size_t) C.R) + sizeof(int) * (size_t) C.R + 64;
    ICG_CUDA(raise_dynamic_smem((const void *) marg_assemble, (size_t) (smem)));
    h->marg_ready = true;
    return ICG_OK;
}

// The parts sized by the marginalized block: H0 / b0 (n0 = m + r), G1 / V1 / lam1 (m), Z (m (rcap + 1)) for n windows.  They grow to the
// batch's maxima when a batch needs more than the last allocation (strides only: the kernels index window w's slot by them and touch the
// n0^2 / m^2 leading entries, so the results do not depend on them).
static int marg_grow(icg_ba *h, int n, int max_m, int max_n0) {
    MargDev &M = h->M;
    if (n <= h->marg_nw && max_m <= M.mcap && max_n0 <= M.n0cap) return ICG_OK;
    const int nw = std::max(n, h->marg_nw), mcap = std::max(max_m, M.mcap), n0cap = std::max(max_n0, M.n0cap);
    ICG_CUDA(cudaStreamSynchronize(h->stream));  // earlier launches on the handle's stream may still read the old buffers
    for (double **p : {&M.H0, &M.b0, &M.G1, &M.V1, &M.lam1, &M.Z}) {
        if (*p) cudaFree(*p);
        *p = nullptr;
    }
    h->marg_nw = 0, M.mcap = 0, M.n0cap = 0;
    const size_t NW = nw;
    const size_t count[6] = {NW * n0cap * n0cap, NW * n0cap, NW * mcap * mcap, NW * mcap * mcap, NW * mcap, NW * mcap * (M.rcap + 1)};
    double **ptr[6] = {&M.H0, &M.b0, &M.G1, &M.V1, &M.lam1, &M.Z};
    for (int k = 0; k < 6; k++) {
        if (cudaMalloc(ptr[k], sizeof(double) * std::max<size_t>(1, count[k])) != cudaSuccess) {
            *ptr[k] = nullptr;
            set_error("icg_ba_marginalize: workspace allocation of %zu doubles failed (%d windows, m <= %d, m + r <= %d)", count[k], nw, mcap, n0cap);
            return ICG_ENOMEM;
        }
        ICG_CUDA(cudaMemsetAsync(*ptr[k], 0, sizeof(double) * std::max<size_t>(1, count[k]), h->stream));
    }
    h->marg_nw = nw, M.mcap = mcap, M.n0cap = n0cap;
    return ICG_OK;
}

// fmask (resident only, may be NULL): per window, the factor set to marginalize in place of the problem's activity (F bytes each); it reaches
// ba_lin_vis through a copy of the device view, so the handle's own f_active is never written.
// agree (may be NULL): called once the structure is known, with {largest m, largest r, 1 if a window is rejected} of this batch; it returns
// the values the eigensolver kernels are chosen by (the owner of a shard group's windows takes the group's maxima, so that it runs the
// kernels an unsharded handle holding the whole batch runs).  It is called on the rejection path too, so that no peer is left waiting.
static int marginalize_body(icg_ba *h, int n_windows, const icg_ba_problem *problems, const int32_t *num_marg, icg_ba_prior *out, bool resident,
                            const uint8_t *const *fmask = nullptr, const std::function<int(int *)> *agree = nullptr) {
    if (!h || !problems || !num_marg || !out || n_windows < 1 || n_windows > h->C.NW) {
        set_error("icg_ba_marginalize: bad arguments");
        return ICG_EINVAL;
    }
    if (h->D.world > 1) {
        set_error("icg_ba_marginalize: not available on a landmark-sharded handle (icg_ba_shard_leave first)");
        return ICG_EUNSUPPORTED;
    }
    int rc = ICG_OK;
    h->marg_res_n = 0;  // the workspace is about to be overwritten: it is the resident prior again only if this call is resident and succeeds
    if (resident) {
        // the windows of the last upload / solve are still on the device (parameters at their optimised values, factor activity and GNSS
        // weights as the two-pass solve left them): `problems` is read for the structure and for x0 only
        if (h->cur_windows != n_windows) {
            set_error("icg_ba_marginalize_resident: the handle holds %d uploaded windows, the call names %d", h->cur_windows, n_windows);
            return ICG_EINVAL;
        }
        ICG_CUDA(cudaSetDevice(h->device));
    } else {
        rc = icg_ba_upload(h, n_windows, problems);
        if (rc != ICG_OK) return rc;
    }
    rc = marg_alloc(h);
    if (rc != ICG_OK) return rc;
    const BaCaps &C = h->C;
    MargDev &M = h->M;
    const int n = n_windows;
    // ---- updateParameterBlocksIndex (marginalization_info.h:228-251) on the host: structure only.  The reference iterates
    //      unordered_maps (implementation-defined order inside each group); here: marginalized = [pose_k, mix_k (k < num_marg),
    //      landmarks ascending], remained = [pose_k, mix_k (k >= num_marg, only blocks some factor touches), ext, td].
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = problems[w];
        const int nm = num_marg[w];
        icg_ba_prior &o = out[w];
        if (nm < 1 || nm >= p.K || !o.block_type || !o.block_node || !o.x0 || !o.J0 || !o.e0 || o.rcap < 15 * (p.K - nm) + 7) {
            set_error("icg_ba_marginalize: window %d: num_marg=%d out of range or output arrays missing / too small (rcap=%d)", w, nm, o.rcap);
            return ICG_EINVAL;
        }
        int *map = h->marg_map.h + (size_t) w * M.map_stride;
        int *pose_col = map + MARG_MAP_HDR, *mix_col = pose_col + C.K, *lm_col = mix_col + C.K;
        std::vector<char> tp(p.K, 0), tm(p.K, 0), tl(p.L, 0);
        const uint8_t *act = fmask ? fmask[w] : p.f_active;
        if (fmask) memcpy(h->marg_fmask.h + (size_t) w * C.F, act, p.F);
        bool any_vis = false;
        for (int f = 0; f < p.F; f++) {
            if ((act && !act[f]) || p.f_ref[f] >= nm) continue;
            tl[p.f_lm[f]] = 1, tp[p.f_obs[f]] = 1, any_vis = true;
        }
        bool has_ext = any_vis, has_td = any_vis;
        // a block exists in the marginalization problem only if some factor touches it (MarginalizationInfo::addResidualBlockInfo,
        // marginalization_info.h:103-121): removed nodes without any factor get no columns
        for (int f = 0; f < p.F; f++)
            if (!(act && !act[f]) && p.f_ref[f] < nm) tp[p.f_ref[f]] = 1;
        for (int k = 0; k < nm && k < p.n_imu; k++) tp[k] = tm[k] = tp[k + 1] = tm[k + 1] = 1;  // factor k joins node k and node k + 1
        for (int g = 0; g < p.n_gnss; g++)
            if (p.gnss_node[g] < nm) tp[p.gnss_node[g]] = 1;
        if (p.has_pose_prior) tp[0] = 1;
        if (p.has_mix_prior) tm[0] = 1;
        for (int b = 0; b < p.marg_nblocks && p.marg_r > 0; b++) {
            const int t = p.marg_block_type[b], nd = p.marg_block_node[b];
            if (t == 0) tp[nd] = 1;
            else if (t == 1) tm[nd] = 1;
            else if (t == 2) has_ext = true;
            else has_td = true;
        }
        int idx = 0;
        for (int k = 0; k < C.K; k++) pose_col[k] = mix_col[k] = -1;
        for (int k = 0; k < nm; k++) {
            if (tp[k]) pose_col[k] = idx, idx += 6;
            if (tm[k]) mix_col[k] = idx, idx += 9;
        }
        for (int l = 0; l < C.L; l++) lm_col[l] = -1;
        for (int l = 0; l < p.L; l++)
            if (tl[l]) lm_col[l] = idx++;
        const int m = idx;
        int nb = 0, xo = 0;
        for (int k = nm; k < p.K; k++) {
            if (tp[k]) pose_col[k] = idx, idx += 6, o.block_type[nb] = 0, o.block_node[nb++] = k - nm, xo += 7;
            if (tm[k]) mix_col[k] = idx, idx += 9, o.block_type[nb] = 1, o.block_node[nb++] = k - nm, xo += 9;
        }
        int ext_col = -1, td_col = -1;
        if (has_ext) ext_col = idx, idx += 6, o.block_type[nb] = 2, o.block_node[nb++] = 0, xo += 7;
        if (has_td) td_col = idx, idx += 1, o.block_type[nb] = 3, o.block_node[nb++] = 0, xo += 1;
        // a reprojection factor always carries ext and td columns; give them (unused) columns when only camera factors exist
        if (ext_col < 0) ext_col = 0;
        if (td_col < 0) td_col = 0;
        map[0] = m, map[1] = idx - m, map[2] = idx, map[3] = nm, map[4] = ext_col, map[5] = td_col, map[6] = map[7] = 0;
        o.m = m, o.r = idx - m, o.nblocks = nb;
        // checked before anything is launched: a rejected call leaves the device state of the handle as it was
        if (m > MARG_MAXN || idx - m > MARG_MAXN) {
            if (agree) {
                int mx[3] = {0, 0, 1};
                (*agree)(mx);
            }
            set_error("icg_ba_marginalize: window %d: %s=%d exceeds the %d rows of the largest eigensolver kernel", w, m > MARG_MAXN ? "m" : "r",
                      m > MARG_MAXN ? m : idx - m, MARG_MAXN);
            return ICG_EUNSUPPORTED;
        }
    }
    int max_m = 0, max_r = 0, max_n0 = 0;
    for (int w = 0; w < n; w++) max_m = std::max(max_m, out[w].m), max_r = std::max(max_r, out[w].r), max_n0 = std::max(max_n0, out[w].m + out[w].r);
    int sel_m = max_m, sel_r = max_r;  // what the eigensolver kernels are chosen by
    if (agree) {
        int mx[3] = {max_m, max_r, 0};
        rc = (*agree)(mx);
        if (rc != ICG_OK) return rc;
        if (mx[2]) {
            set_error("icg_ba_marginalize_resident: a window owned by another rank of the shard group was rejected (see that rank's error)");
            return ICG_EUNSUPPORTED;
        }
        sel_m = mx[0], sel_r = mx[1];
    }
    rc = marg_grow(h, n, max_m, max_n0);
    if (rc != ICG_OK) return rc;
    cudaStream_t s = h->stream;
    if (h->marg_cluster_ok < 0) {  // once per handle: can an 8-CTA marg_jacobi_cluster with the largest shared-memory slices be placed at all?
        const size_t csm = marg_cluster_smem(MARG_CLUSTER_MAXN);
        ICG_CUDA(raise_dynamic_smem((const void *) marg_jacobi_cluster, csm));
        cudaLaunchConfig_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.gridDim = dim3(MARG_CLUSTER_CTAS), cfg.blockDim = dim3(MARG_CLUSTER_THREADS), cfg.dynamicSmemBytes = csm, cfg.stream = s;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = MARG_CLUSTER_CTAS, at[0].val.clusterDim.y = 1, at[0].val.clusterDim.z = 1;
        cfg.attrs = at, cfg.numAttrs = 1;
        int nclusters = 0;
        h->marg_cluster_ok = cudaOccupancyMaxActiveClusters(&nclusters, marg_jacobi_cluster, &cfg) == cudaSuccess && nclusters > 0 ? 1 : 0;
        cudaGetLastError();  // a refused query is an answer (the global kernel takes those blocks), not an error of this call
    }
    ICG_CUDA(h->marg_map.up(s, (size_t) n * M.map_stride));
    BaDev D = h->D;
    if (fmask) {
        ICG_CUDA(h->marg_fmask.up(s, (size_t) n * C.F));
        D.f_active = h->marg_fmask.d;
    }
    const size_t smem = sizeof(double) * (8 * 480 + 2 * (size_t) C.R) + sizeof(int) * (size_t) C.R + 64;
    marg_prepare<<<(n + 127) / 128, 128, 0, s>>>(D, M, n, 0);
    ba_lin_vis<<<dim3(C.NVB - 2, n), 128, LV_SMEM, s>>>(C, D, 0);
    marg_assemble<<<n, 256, smem, s>>>(C, D, M);
    // eigendecompositions: one kernel per stage serves the whole batch, chosen by the batch's largest block --
    //   n <= MARG_CTA_MAXN: one CTA;  n <= MARG_PAIR_MAXN: cluster pair;  n <= MARG_CLUSTER_MAXN: 8-CTA cluster;  otherwise: global memory.
    // ICG_MARG_GLOBAL_JACOBI forces the global kernel, ICG_MARG_PAIR_JACOBI skips the one-CTA kernel, ICG_MARG_CLUSTER_JACOBI takes the
    // 8-CTA cluster for any n it supports.
    auto jacobi = [&](int which, int nmax) -> int {
        const bool cluster_ok = nmax <= MARG_CLUSTER_MAXN && h->marg_cluster_ok == 1;
        if (cluster_ok && !getenv("ICG_MARG_GLOBAL_JACOBI") && (getenv("ICG_MARG_CLUSTER_JACOBI") || nmax > MARG_PAIR_MAXN)) {
            const size_t smem = marg_cluster_smem(nmax);
            cudaLaunchConfig_t cfg;
            memset(&cfg, 0, sizeof(cfg));
            cfg.gridDim = dim3((unsigned) (MARG_CLUSTER_CTAS * n)), cfg.blockDim = dim3(MARG_CLUSTER_THREADS), cfg.dynamicSmemBytes = smem, cfg.stream = s;
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeClusterDimension;
            at[0].val.clusterDim.x = MARG_CLUSTER_CTAS, at[0].val.clusterDim.y = 1, at[0].val.clusterDim.z = 1;
            cfg.attrs = at, cfg.numAttrs = 1;
            ICG_CUDA(cudaLaunchKernelEx(&cfg, marg_jacobi_cluster, M, which));
        } else if (nmax <= MARG_CTA_MAXN && !getenv("ICG_MARG_GLOBAL_JACOBI") && !getenv("ICG_MARG_PAIR_JACOBI")) {
            const size_t smem = sizeof(double) * 2 * (size_t) nmax * nmax;
            ICG_CUDA(raise_dynamic_smem((const void *) marg_jacobi_cta, smem));
            marg_jacobi_cta<<<n, MARG_CTA_THREADS, smem, s>>>(M, which);
        } else if (nmax <= MARG_PAIR_MAXN && !getenv("ICG_MARG_GLOBAL_JACOBI")) {
            const size_t smem = sizeof(double) * ((size_t) nmax * nmax + 2 * (size_t) (nmax + 2));
            cudaLaunchConfig_t cfg;
            memset(&cfg, 0, sizeof(cfg));
            cfg.gridDim = dim3((unsigned) (2 * n)), cfg.blockDim = dim3(MARG_THREADS), cfg.dynamicSmemBytes = smem, cfg.stream = s;
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeClusterDimension;
            at[0].val.clusterDim.x = 2, at[0].val.clusterDim.y = 1, at[0].val.clusterDim.z = 1;
            cfg.attrs = at, cfg.numAttrs = 1;
            ICG_CUDA(raise_dynamic_smem((const void *) marg_jacobi_pair, (size_t) (smem)));
            ICG_CUDA(cudaLaunchKernelEx(&cfg, marg_jacobi_pair, M, which));
        } else {
            marg_jacobi<<<n, MARG_THREADS, 0, s>>>(M, which);
        }
        return ICG_OK;
    };
    rc = jacobi(0, sel_m);
    if (rc != ICG_OK) return rc;
    marg_schur<<<n, MARG_THREADS, 0, s>>>(M);
    rc = jacobi(1, sel_r);
    if (rc != ICG_OK) return rc;
    marg_finish<<<n, MARG_THREADS, 0, s>>>(M);
    marg_prepare<<<(n + 127) / 128, 128, 0, s>>>(D, M, n, 1);
    ICG_CHECK_LAUNCH();
    count_launch(9);
    // D2H: every window's r x r result sits at the start of its rcap^2 slot -- move the used prefix of each slot only (one strided copy)
    {
        const size_t pitch = sizeof(double) * (size_t) M.rcap * M.rcap, used = sizeof(double) * (size_t) max_r * max_r;
        bool want_Hp = false;
        for (int w = 0; w < n; w++) want_Hp = want_Hp || out[w].Hp != nullptr;
        if (used) ICG_CUDA(cudaMemcpy2DAsync(h->marg_oJ0.h, pitch, h->marg_oJ0.d, pitch, used, (size_t) n, cudaMemcpyDeviceToHost, s));
        ICG_CUDA(h->marg_oe0.down(s, (size_t) n * M.rcap));
        if (want_Hp && used) ICG_CUDA(cudaMemcpy2DAsync(h->marg_oHp.h, pitch, h->marg_oHp.d, pitch, used, (size_t) n, cudaMemcpyDeviceToHost, s));
        ICG_CUDA(h->marg_obp.down(s, (size_t) n * M.rcap));
    }
    ICG_CUDA(cudaStreamSynchronize(s));
    auto write_back = [&](int w) {
        const icg_ba_problem &p = problems[w];
        icg_ba_prior &o = out[w];
        const int nm = num_marg[w], r = o.r;
        // preMarginalization copies the parameter data of every block: x0 of the remained blocks (marginalization_info.h:270-283)
        int xo = 0;
        for (int b = 0; b < o.nblocks; b++) {
            const int t = o.block_type[b], nd = o.block_node[b] + nm;
            const double *src = t == 0 ? p.pose + 7 * nd : t == 1 ? p.mix + 9 * nd : t == 2 ? p.ext : p.ext + 7;
            const int gs = t == 1 ? 9 : t == 3 ? 1 : 7;
            memcpy(o.x0 + xo, src, sizeof(double) * gs);
            xo += gs;
        }
        if (o.m <= 0) return;
        memcpy(o.J0, h->marg_oJ0.h + (size_t) w * M.rcap * M.rcap, sizeof(double) * (size_t) r * r);
        memcpy(o.e0, h->marg_oe0.h + (size_t) w * M.rcap, sizeof(double) * r);
        if (o.Hp) memcpy(o.Hp, h->marg_oHp.h + (size_t) w * M.rcap * M.rcap, sizeof(double) * (size_t) r * r);
        if (o.bp) memcpy(o.bp, h->marg_obp.h + (size_t) w * M.rcap, sizeof(double) * r);
    };
    {   // the copies into the caller's arrays are memcpy-bound (r^2 doubles per window): a few host threads, like the packing of icg_ba_upload
        const int nthreads = std::max(1, std::min({n / 8, 8, (int) std::thread::hardware_concurrency()}));
        auto worker = [&](int t) {
            for (int w = t; w < n; w += nthreads) write_back(w);
        };
        std::vector<std::thread> th;
        for (int t = 1; t < nthreads; t++) th.emplace_back(worker, t);
        worker(0);
        for (auto &x : th) x.join();
    }
    if (resident) {  // icg_ba_slide_resident(prior_from_marg = 1) takes this prior from the workspace
        h->marg_res_m.resize(n), h->marg_res_r.resize(n), h->marg_res_nb.resize(n);
        for (int w = 0; w < n; w++) h->marg_res_m[w] = out[w].m, h->marg_res_r[w] = out[w].r, h->marg_res_nb[w] = out[w].nblocks;
        h->marg_res_n = n, h->marg_res_sharded = false;
    }
    return ICG_OK;
}

int icg_ba_marginalize(icg_ba *h, int n_windows, const icg_ba_problem *problems, const int32_t *num_marg, icg_ba_prior *out) {
    return marginalize_body(h, n_windows, problems, num_marg, out, false);
}

// ---- post-solve calls of a landmark-sharded group (world > 1, ba_split.cuh)
extern "C++" {
template <typename T>
static int hd_reserve(icg_ba *h, HostDev<T> &b, size_t count) {
    if (b.d && b.n >= count) return ICG_OK;
    retire(h, b.d, b.h);  // earlier launches may still use the old buffers
    b.d = b.h = nullptr, b.n = 0;
    if (b.alloc(std::max<size_t>(16, count + count / 4)) != ICG_OK) {
        set_error("landmark-sharded post-solve call: staging allocation of %zu elements failed", count);
        return ICG_ENOMEM;
    }
    return ICG_OK;
}
}

static int shard_timed_out(icg_ba *h, const char *what) {
    if (icg_ba_shard_error(h) == 0) return ICG_OK;
    set_error("%s: a peer exchange of the shard group timed out (a rank did not make the same call)", what);
    return ICG_ECUDA;
}

// enqueue the group's integer exchange of v (device; see ba_xsum)
static int shard_xsum(icg_ba *h, int *v, int stride, int n, int nv, int op) {
    const unsigned long long epoch = ++h->epoch;
    const int par = (int) (h->xs_calls++ & 1);
    ba_xsum<<<1, 256, 0, h->stream>>>(h->C, h->D, v, stride, n, nv, op, par, epoch);
    ICG_CHECK_LAUNCH();
    count_launch();
    return ICG_OK;
}

// the group's maxima of three host integers (fn: the calling entry point, for the timeout's message)
static int shard_xmax(icg_ba *h, int *v3, const char *fn) {
    int rc = hd_reserve(h, h->xs_v, 8);
    if (rc != ICG_OK) return rc;
    memcpy(h->xs_v.h, v3, 3 * sizeof(int));
    ICG_CUDA(h->xs_v.up(h->stream, 3));
    rc = shard_xsum(h, h->xs_v.d, 3, 1, 3, 1);
    if (rc != ICG_OK) return rc;
    ICG_CUDA(h->xs_v.down(h->stream, 3));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    rc = shard_timed_out(h, fn);
    if (rc != ICG_OK) return rc;
    memcpy(v3, h->xs_v.h, 3 * sizeof(int));
    return ICG_OK;
}

// 31-bit fingerprint of the arguments a collective call requires to be the same on every rank (FNV-1a over 64-bit words)
extern "C++" {
struct ArgPrint {
    uint64_t v = 1469598103934665603ull;
    void bytes(const void *p, size_t n) {
        const unsigned char *c = (const unsigned char *) p;
        size_t i = 0;
        for (uint64_t x; i + 8 <= n; i += 8) memcpy(&x, c + i, 8), v = (v ^ x) * 1099511628211ull;
        for (; i < n; i++) v = (v ^ c[i]) * 1099511628211ull;
    }
    template <typename T>
    void arr(const T *p, long long count) {
        if (p && count > 0) bytes(p, sizeof(T) * (size_t) count);
    }
    void num(long long x) { bytes(&x, sizeof(x)); }
    int get() const { return (int) ((v ^ (v >> 31) ^ (v >> 62)) & 0x7fffffff); }
};
}

// The agreement of a collective call before any rank writes its device: one exchange of (rejecting rank + 1, +fp, -fp).  ICG_OK when no rank
// rejected and every rank passed the same fingerprint fp; otherwise ICG_EINVAL on every rank (a rejecting rank keeps its own message).
static int shard_agree(icg_ba *h, bool rejected, int fp, const char *fn) {
    int mx[3] = {rejected ? h->D.rank + 1 : 0, rejected ? 0 : fp, rejected ? 0 : -fp};
    const int rc = shard_xmax(h, mx, fn);
    if (rc != ICG_OK || rejected) return rc != ICG_OK ? rc : ICG_EINVAL;
    if (mx[0]) {
        set_error("%s: rank %d of the shard group rejected the call (see that rank's error); no rank changed its handle", fn, mx[0] - 1);
        return ICG_EINVAL;
    }
    if (mx[1] != -mx[2]) {
        set_error("%s: the ranks' camera sides differ (node, IMU and GNSS rows and maps, the prior's source and the integration's inputs must be "
                  "the same on every rank); no rank changed its handle", fn);
        return ICG_EINVAL;
    }
    return ICG_OK;
}

// The resident marginalization on a landmark-sharded handle, a collective call: every rank exports the rows of its factors with
// f_ref < num_marg (ba_marg_export); the owner of window w (w mod world) gathers the world exports of w in rank order -- global landmark
// order, since the landmarks are block-partitioned and each rank lists its factors landmark by landmark --, packs the gathered windows' integer
// structure into a handle of its own (nothing of their values goes through the host: ba_marg_fill copies the gathered rows and the shard
// handle's resident camera side on the device), and runs the single-GPU marginalization there.  That handle packs the
// gathered window exactly as an unsharded handle packs the marginalized part of the whole window (runs, Gram partials and pairs of the
// reference nodes < num_marg depend on those landmarks only), so the prior is the unsharded one, bit for bit.
static int marginalize_sharded(icg_ba *h, int n, const icg_ba_problem *problems, const int32_t *num_marg, icg_ba_prior *out, const uint8_t *const *fmask,
                               const char *fn) {
    const BaCaps &C = h->C;
    const int G = h->D.world, R = h->D.rank;
    if (!problems || !num_marg || !out || n < 1 || n > C.NW) {
        set_error("%s: bad arguments", fn);
        return ICG_EINVAL;
    }
    if (h->cur_windows != n) {
        set_error("%s: the handle holds %d uploaded windows, the call names %d", fn, h->cur_windows, n);
        return ICG_EINVAL;
    }
    for (int r = 0; r < G; r++)
        if (!h->D.S.peer[r]) {
            set_error("%s: peer %d is not connected (icg_ba_shard_connect)", fn, r);
            return ICG_EINVAL;
        }
    // every check before anything is launched: a rank that returns here leaves its peers to the bounded waits
    size_t n_sel = 0;
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = problems[w];
        const WinDims &d = h->dims.h[w];
        const icg_ba_prior &o = out[w];
        if (p.K != d.K || p.L != d.L || p.F != d.F || (p.F > 0 && (!p.f_lm || !p.f_ref || !p.f_obs))) {
            set_error("%s: window %d does not describe the uploaded shard (K=%d L=%d F=%d)", fn, w, p.K, p.L, p.F);
            return ICG_EINVAL;
        }
        if (num_marg[w] < 1 || num_marg[w] >= p.K || !o.block_type || !o.block_node || !o.x0 || !o.J0 || !o.e0 || o.rcap < 15 * (p.K - num_marg[w]) + 7) {
            set_error("%s: window %d: num_marg=%d out of range or output arrays missing / too small (rcap=%d)", fn, w, num_marg[w], o.rcap);
            return ICG_EINVAL;
        }
        for (int f = 0; f < p.F; f++) {
            if (f > 0 && p.f_lm[f] < p.f_lm[f - 1]) {
                set_error("%s: window %d factor %d: a landmark-sharded window must list its factors landmark by landmark (f_lm non-decreasing)", fn, w, f);
                return ICG_EINVAL;
            }
            n_sel += p.f_ref[f] < num_marg[w];
        }
    }
    ICG_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    int rc = marg_alloc(h);  // marg_fmask: the culled factor set the export reads
    if (rc != ICG_OK) return rc;
    if ((rc = hd_reserve(h, h->mx_sel, n_sel + n + 1)) != ICG_OK) return rc;
    int *sel = h->mx_sel.h, *sel_off = sel + n_sel;
    {   // the record slots of the exported factors, in factor order (the inverse of the packing's slot -> factor table)
        size_t at = 0;
        std::vector<int> slot_of;
        for (int w = 0; w < n; w++) {
            const icg_ba_problem &p = problems[w];
            slot_of.assign(p.F, 0);
            const int *fidx = h->lm_fidx.h + (size_t) w * C.F;
            for (int q = 0; q < p.F; q++) slot_of[fidx[q]] = q;
            sel_off[w] = (int) at;
            for (int f = 0; f < p.F; f++)
                if (p.f_ref[f] < num_marg[w]) sel[at++] = slot_of[f];
            if (fmask) memcpy(h->marg_fmask.h + (size_t) w * C.F, fmask[w], p.F);
        }
        sel_off[n] = (int) at;
    }
    ICG_CUDA(h->mx_sel.up(s, n_sel + n + 1));
    if (fmask) ICG_CUDA(h->marg_fmask.up(s, (size_t) n * C.F));
    const unsigned long long epoch = ++h->epoch;
    ba_marg_export<<<n, 128, 0, s>>>(C, h->D, h->mx_sel.d, h->mx_sel.d + n_sel, fmask ? h->marg_fmask.d : nullptr, h->exp_epoch);
    ba_xflag<<<1, 32, 0, s>>>(h->D, XF_EXPORT, epoch);
    h->exp_epoch = epoch;
    count_launch(2);
    const int n_own = R < n ? (n - R + G - 1) / G : 0;
    std::vector<int> row0(n_own + 1, 0);
    if (n_own > 0) {
        if ((rc = hd_reserve(h, h->mx_heads, 2 * (size_t) n_own * G)) != ICG_OK) return rc;
        ba_marg_heads<<<1, 256, 0, s>>>(C, h->D, n_own, h->mx_heads.d, epoch);
        ICG_CUDA(h->mx_heads.down(s, 2 * (size_t) n_own * G));
        ICG_CUDA(cudaStreamSynchronize(s));
        if ((rc = shard_timed_out(h, fn)) != ICG_OK) return rc;
        if ((rc = hd_reserve(h, h->mx_row, (size_t) n_own * G + n_own + 1)) != ICG_OK) return rc;
        size_t tot = 0;
        for (int e = 0; e < n_own * G; e++) {
            if (e % G == 0) row0[e / G] = (int) tot;
            h->mx_row.h[e] = (int) tot;
            tot += (size_t) h->mx_heads.h[2 * e + 1];
        }
        row0[n_own] = (int) tot;
        if (tot > (size_t) INT32_MAX / MEXP_ROW) {
            set_error("%s: %zu gathered factors exceed the gather buffer's index range", fn, tot);
            return ICG_EINVAL;
        }
        if (tot * MEXP_ROW > h->mx_rows_cap) {
            retire(h, h->mx_rows, nullptr), h->mx_rows = nullptr;
            h->mx_rows_cap = 0;
            const size_t cap = (tot + tot / 4) * MEXP_ROW;
            if (cudaMalloc(&h->mx_rows, sizeof(double) * cap) != cudaSuccess) {
                set_error("%s: gather buffer allocation of %zu doubles failed", fn, cap);
                return ICG_ENOMEM;
            }
            h->mx_rows_cap = cap;
        }
        if ((rc = hd_reserve(h, h->mx_idx, std::max<size_t>(1, tot))) != ICG_OK) return rc;
        memcpy(h->mx_row.h + (size_t) n_own * G, row0.data(), sizeof(int) * (n_own + 1));
        ICG_CUDA(h->mx_row.up(s, (size_t) n_own * G + n_own + 1));
        ba_marg_gather<<<dim3(n_own, G), 256, 0, s>>>(C, h->D, h->mx_heads.d, h->mx_row.d, h->mx_rows);
        count_launch(2);
        if (tot) ICG_CUDA(cudaMemcpy2DAsync(h->mx_idx.h, sizeof(long long), h->mx_rows, sizeof(double) * MEXP_ROW, sizeof(long long), tot, cudaMemcpyDeviceToHost, s));
    }
    ba_xflag<<<1, 32, 0, s>>>(h->D, XF_DONE, epoch);  // this rank's reads of the exports are enqueued: the exporters may reuse their regions
    ICG_CHECK_LAUNCH();
    count_launch();
    for (int w = 0; w < n; w++)
        if (w % G != R) out[w].m = out[w].r = out[w].nblocks = 0;
    h->marg_res_n = 0;  // the workspace is about to be overwritten: the sharded slide's prior again only if this call succeeds
    // on success: the record icg_ba_shard_slide[_integrate]_resident checks (every rank: a sharded resident marginalization of these n
    // windows; the owner: each owned window's m, r, nblocks)
    auto record = [&]() {
        h->marg_res_m.assign(n, 0), h->marg_res_r.assign(n, 0), h->marg_res_nb.assign(n, 0);
        for (int w = R; w < n; w += G) h->marg_res_m[w] = out[w].m, h->marg_res_r[w] = out[w].r, h->marg_res_nb[w] = out[w].nblocks;
        h->marg_res_n = n, h->marg_res_sharded = true;
        return ICG_OK;
    };
    if (n_own == 0) {
        int mx[3] = {0, 0, 0};
        rc = shard_xmax(h, mx, fn);
        if (rc != ICG_OK) return rc;
        if (mx[2]) {
            set_error("%s: a window owned by another rank of the shard group was rejected (see that rank's error)", fn);
            return ICG_EUNSUPPORTED;
        }
        return record();
    }
    ICG_CUDA(cudaStreamSynchronize(s));
    if ((rc = shard_timed_out(h, fn)) != ICG_OK) return rc;
    // the gathered windows, structure on the host (values follow on the device): landmarks renumbered densely in (rank, shard landmark) order
    std::vector<icg_ba_problem> gp(n_own);
    std::vector<std::vector<int32_t>> g_lm(n_own), g_ref(n_own), g_obs(n_own);
    std::vector<std::vector<uint8_t>> g_act(n_own);
    int max_L = 1, max_F = 1;
    for (int j = 0; j < n_own; j++) {
        const int w = R + j * G, F = row0[j + 1] - row0[j];
        const icg_ba_problem &p = problems[w];
        g_lm[j].resize(F), g_ref[j].resize(F), g_obs[j].resize(F), g_act[j].resize(F);
        int L = 0, last_r = -1, last_l = -1;
        for (int r = 0, i = 0; r < G; r++)
            for (long long k = 0; k < h->mx_heads.h[2 * ((size_t) j * G + r) + 1]; k++, i++) {
                const unsigned long long x = (unsigned long long) h->mx_idx.h[row0[j] + i];
                const int l = (int) (x & 0xffffffffu), hi = (int) (x >> 32), ref = hi & 255, obs = (hi >> 8) & 255;
                if (r != last_r || l != last_l) L++, last_r = r, last_l = l;
                if (ref >= num_marg[w] || obs >= p.K) {
                    set_error("%s: window %d: gathered factor %d names nodes %d / %d (the ranks' windows differ)", fn, w, i, ref, obs);
                    int mx[3] = {0, 0, 1};
                    shard_xmax(h, mx, fn);
                    return ICG_EINVAL;
                }
                g_lm[j][i] = L - 1, g_ref[j][i] = ref, g_obs[j][i] = obs, g_act[j][i] = (uint8_t) ((hi >> 16) & 1);
            }
        icg_ba_problem &q = gp[j];
        q = p;
        q.L = L, q.F = F;
        q.f_lm = g_lm[j].data(), q.f_ref = g_ref[j].data(), q.f_obs = g_obs[j].data(), q.f_active = g_act[j].data();
        max_L = std::max(max_L, L), max_F = std::max(max_F, F);
    }
    double unread = 0;  // the structure-only packing checks these pointers but reads no value: ba_marg_fill writes them on the device
    for (auto &q : gp) q.invdepth = &unread, q.f_const = &unread;
    icg_ba *&mh = h->mx_h;
    if (mh && (mh->C.NW < n_own || mh->C.L < max_L || mh->C.F < max_F)) {
        max_L = std::max(max_L, mh->C.L), max_F = std::max(max_F, mh->C.F);
        h->retired_mx.push_back(mh), mh = nullptr;
    }
    if (!mh) {
        const int nw = std::max(n_own, (C.NW + G - 1) / G);
        rc = icg_ba_create(&mh, nw, C.K, max_L + max_L / 4, max_F + max_F / 4, C.G, C.R, h->device, (void *) s);
        if (rc != ICG_OK) {
            mh = nullptr;
            int mx[3] = {0, 0, 1};
            shard_xmax(h, mx, fn);
            return rc;
        }
    }
    // structure only (landmark positions, record slots, lin_vis runs, Gram partials, pairs; the small camera-side tables): the same packing
    // icg_ba_upload does, so the sums match an unsharded handle's.  Every value comes from the device: the gathered rows, and the shard
    // handle's resident camera side (parameters, IMU blobs and square-root information, GNSS, the carried prior's normal equations).
    rc = pack_windows(mh, n_own, gp.data(), false);
    if (rc == ICG_OK) rc = upload_structure(mh, n_own);
    if (rc == ICG_OK) {
        mh->cur_windows = n_own, mh->marg_res_n = 0;
        ICG_CUDA(mh->lm_fidx.up(s, (size_t) n_own * mh->C.F));
        ba_marg_fill<<<n_own, 128, 0, s>>>(mh->C, mh->D, C, h->D, h->mx_rows, h->mx_row.d + (size_t) n_own * G, mh->lm_fidx.d);
        ICG_CHECK_LAUNCH();
        count_launch();
    } else {
        int mx[3] = {0, 0, 1};
        shard_xmax(h, mx, fn);
        return rc;
    }
    std::vector<int32_t> nm(n_own);
    std::vector<icg_ba_prior> po(n_own);
    for (int j = 0; j < n_own; j++) nm[j] = num_marg[R + j * G], po[j] = out[R + j * G];
    const std::function<int(int *)> agree = [h, fn](int *mx) { return shard_xmax(h, mx, fn); };
    rc = marginalize_body(mh, n_own, gp.data(), nm.data(), po.data(), true, nullptr, &agree);
    for (int j = 0; j < n_own; j++) out[R + j * G].m = po[j].m, out[R + j * G].r = po[j].r, out[R + j * G].nblocks = po[j].nblocks;
    return rc == ICG_OK ? record() : rc;
}

int icg_ba_marginalize_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const int32_t *num_marg, icg_ba_prior *out) {
    if (h && h->D.world > 1) return marginalize_sharded(h, n_windows, problems, num_marg, out, nullptr, "icg_ba_marginalize_resident");
    return marginalize_body(h, n_windows, problems, num_marg, out, true);
}

// ---- post-solve map update + outlier culling (ba_cull.cu)
static int resident_single_rank(icg_ba *h, int n_windows, const icg_ba_problem *problems, const char *what, bool sharded_ok = false) {
    if (!h || !problems || n_windows < 1) {
        set_error("%s: bad arguments", what);
        return ICG_EINVAL;
    }
    if (h->D.world > 1 && !sharded_ok) {  // the reintegration and the slides: their collective forms are icg_ba_shard_*
        set_error("%s: not available on a landmark-sharded handle (the group calls icg_ba_shard_%s; or icg_ba_shard_leave first)", what, what + 7);
        return ICG_EUNSUPPORTED;
    }
    if (h->cur_windows != n_windows) {
        set_error("%s: the handle holds %d uploaded windows, the call names %d", what, h->cur_windows, n_windows);
        return ICG_EINVAL;
    }
    return ICG_OK;
}

int icg_ba_update_and_cull_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const icg_camera *cam, double reprojection_error_std,
                                    icg_ba_cull_window *io) {
    int rc = resident_single_rank(h, n_windows, problems, "icg_ba_update_and_cull_resident", true);
    if (rc != ICG_OK) return rc;
    if (!cam || !io) {
        set_error("icg_ba_update_and_cull_resident: bad arguments");
        return ICG_EINVAL;
    }
    const BaCaps &C = h->C;
    const int n = n_windows;
    // layout of the staging buffer: inputs [windows | lm_ref_node | obs_off | obs_node | lm_ref_kp | obs_kp], then outputs
    // [windows | cam_pose | lm_pw | lm_depth | lm_outlier | obs_outlier], every array 16-byte aligned
    std::vector<CullWin> win(n);
    size_t nL = 0, nO = 0, nK = 0;
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = problems[w];
        const icg_ba_cull_window &c = io[w];
        if (p.K < 2 || p.K > C.K || p.L < 0 || p.L > C.L || !c.cam_pose ||
            (p.L > 0 && (!c.lm_ref_node || !c.lm_ref_kp || !c.obs_off || !c.lm_pw || !c.lm_depth || !c.lm_outlier))) {
            set_error("icg_ba_update_and_cull_resident: window %d: sizes out of range or arrays missing", w);
            return ICG_EINVAL;
        }
        const int no = p.L > 0 ? c.obs_off[p.L] : 0;
        if (p.L > 0 && (c.obs_off[0] != 0 || no < 0 || no > INT32_MAX - (int64_t) nO || (no > 0 && (!c.obs_node || !c.obs_kp || !c.obs_outlier)))) {
            set_error("icg_ba_update_and_cull_resident: window %d: obs_off must start at 0 and observation arrays must be given", w);
            return ICG_EINVAL;
        }
        for (int l = 0; l < p.L; l++) {
            if (c.obs_off[l + 1] < c.obs_off[l] || c.lm_ref_node[l] < 0 || c.lm_ref_node[l] >= p.K) {
                set_error("icg_ba_update_and_cull_resident: window %d landmark %d: obs_off not monotone or reference node out of range", w, l);
                return ICG_EINVAL;
            }
        }
        for (int o = 0; o < no; o++)
            if (c.obs_node[o] < 0 || c.obs_node[o] >= p.K) {
                set_error("icg_ba_update_and_cull_resident: window %d observation %d: node %d out of range", w, o, c.obs_node[o]);
                return ICG_EINVAL;
            }
        CullWin &W = win[w];
        memcpy(W.R_bc, c.R_bc, sizeof(W.R_bc)), memcpy(W.t_bc, c.t_bc, sizeof(W.t_bc));
        W.td_bc = c.td_bc, W.K = p.K, W.L = p.L, W.estimate_ext = c.estimate_ext != 0, W.estimate_td = c.estimate_td != 0;
        W.lm0 = (int) nL, W.off0 = (int) (nL + w), W.obs0 = (int) nO, W.node0 = (int) nK;
        nL += p.L, nO += no, nK += p.K;
    }
    auto al = [](size_t b) { return (b + 15) & ~(size_t) 15; };
    size_t at = 0;
    auto take = [&](size_t bytes) {
        const size_t o = at;
        at += al(bytes);
        return o;
    };
    const size_t i_win = take(sizeof(CullWin) * n), i_ref = take(4 * nL), i_off = take(4 * (nL + n)), i_node = take(4 * nO), i_rkp = take(8 * nL),
                 i_kp = take(8 * nO);
    const size_t in_bytes = at;
    const size_t o_win = take(sizeof(CullOut) * n), o_pose = take(96 * nK), o_pw = take(24 * nL), o_depth = take(8 * nL), o_lmo = take(nL), o_obso = take(nO);
    const size_t out_bytes = at - in_bytes;
    h->cull_res_n = 0;  // the staging is rewritten (or replaced) from here
    ICG_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    if (at > h->cull_cap) {
        ICG_CUDA(cudaStreamSynchronize(s));
        retire(h, h->cull_d, h->cull_h), h->cull_h = nullptr, h->cull_d = nullptr;
        h->cull_cap = 0;
        const size_t cap = at + at / 4;
        if (cudaMallocHost(&h->cull_h, cap) != cudaSuccess || cudaMalloc(&h->cull_d, cap) != cudaSuccess) {
            set_error("icg_ba_update_and_cull_resident: staging allocation of %zu bytes failed", cap);
            return ICG_ENOMEM;
        }
        h->cull_cap = cap;
    }
    unsigned char *H = h->cull_h, *Dv = h->cull_d;
    memcpy(H + i_win, win.data(), sizeof(CullWin) * n);
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = problems[w];
        const icg_ba_cull_window &c = io[w];
        const CullWin &W = win[w];
        if (p.L == 0) {
            ((int *) (H + i_off))[W.off0] = 0;
            continue;
        }
        const int no = c.obs_off[p.L];
        memcpy(H + i_ref + 4 * (size_t) W.lm0, c.lm_ref_node, 4 * (size_t) p.L);
        memcpy(H + i_off + 4 * (size_t) W.off0, c.obs_off, 4 * ((size_t) p.L + 1));
        memcpy(H + i_rkp + 8 * (size_t) W.lm0, c.lm_ref_kp, 8 * (size_t) p.L);
        if (no > 0) memcpy(H + i_node + 4 * (size_t) W.obs0, c.obs_node, 4 * (size_t) no), memcpy(H + i_kp + 8 * (size_t) W.obs0, c.obs_kp, 8 * (size_t) no);
    }
    ICG_CUDA(cudaMemcpyAsync(Dv, H, in_bytes, cudaMemcpyHostToDevice, s));
    CullArgs a;
    a.cam = *cam, a.std = reprojection_error_std;
    a.pose = h->D.pose, a.ext = h->D.ext, a.rho = h->D.rho, a.pose_stride = C.K * 7, a.rho_stride = C.L;
    a.win = (const CullWin *) (Dv + i_win), a.lm_ref_node = (const int *) (Dv + i_ref), a.obs_off = (const int *) (Dv + i_off);
    a.obs_node = (const int *) (Dv + i_node), a.lm_ref_kp = (const float *) (Dv + i_rkp), a.obs_kp = (const float *) (Dv + i_kp);
    a.out = (CullOut *) (Dv + o_win), a.cam_pose = (double *) (Dv + o_pose), a.lm_pw = (double *) (Dv + o_pw), a.lm_depth = (double *) (Dv + o_depth);
    a.lm_outlier = Dv + o_lmo, a.obs_outlier = Dv + o_obso;
    ICG_CUDA(launch_update_cull(a, n, s));
    count_launch();
    if (h->D.world > 1) {  // landmark shards: every rank's counters become the window's totals (the other outputs are the camera side or its shard's)
        rc = shard_xsum(h, (int *) (Dv + o_win + offsetof(CullOut, counts)), (int) (sizeof(CullOut) / sizeof(int)), n, 5, 0);
        if (rc != ICG_OK) return rc;
    }
    ICG_CUDA(cudaMemcpyAsync(H + in_bytes, Dv + in_bytes, out_bytes, cudaMemcpyDeviceToHost, s));
    ICG_CUDA(cudaStreamSynchronize(s));
    if (h->D.world > 1 && (rc = shard_timed_out(h, "icg_ba_update_and_cull_resident")) != ICG_OK) return rc;
    if (h->D.world == 1) {
        h->cull_res_n = n, h->cull_res_win = win, h->cull_res_nobs.resize(n);
        for (int w = 0; w < n; w++) h->cull_res_nobs[w] = problems[w].L > 0 ? io[w].obs_off[problems[w].L] : 0;
        h->cull_res_ref = i_ref, h->cull_res_off = i_off, h->cull_res_lmo = o_lmo, h->cull_res_obso = o_obso;
    }
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = problems[w];
        icg_ba_cull_window &c = io[w];
        const CullWin &W = win[w];
        const CullOut &O = ((const CullOut *) (H + o_win))[w];
        memcpy(c.R_bc_out, O.R_bc, sizeof(c.R_bc_out)), memcpy(c.t_bc_out, O.t_bc, sizeof(c.t_bc_out));
        c.td_bc_out = O.td_bc, c.ext_accepted = O.ext_accepted;
        memcpy(c.counts, O.counts, sizeof(c.counts));
        memcpy(c.cam_pose, H + o_pose + 96 * (size_t) W.node0, 96 * (size_t) p.K);
        if (p.L == 0) continue;
        const int no = c.obs_off[p.L];
        memcpy(c.lm_pw, H + o_pw + 24 * (size_t) W.lm0, 24 * (size_t) p.L);
        memcpy(c.lm_depth, H + o_depth + 8 * (size_t) W.lm0, 8 * (size_t) p.L);
        memcpy(c.lm_outlier, H + o_lmo + W.lm0, p.L);
        if (no > 0) memcpy(c.obs_outlier, H + o_obso + W.obs0, no);
    }
    return ICG_OK;
}

// ---- doReintegration (IG/ic_gvins.cc:1680-1695) on the resident IMU factors (preint.cu)
// sharded (icg_ba_shard_reintegrate_resident): every rank runs the same reintegration on its replicated states, after the group agreed
static int reint_body(icg_ba *h, int n_windows, const icg_ba_problem *problems, const double *noise5, const double *station3, icg_ba_reint_window *io,
                      const char *fn, bool sharded) {
    const int n = n_windows;
    // validation first: nothing is launched on bad input
    size_t n_items = 0, n_rows = 0;
    auto validate = [&]() -> int {
        int rc = resident_single_rank(h, n_windows, problems, fn, sharded);
        if (rc != ICG_OK) return rc;
        if (!noise5 || !station3 || !io) {
            set_error("%s: bad arguments", fn);
            return ICG_EINVAL;
        }
        for (int w = 0; w < n; w++) {
            const icg_ba_problem &p = problems[w];
            const icg_ba_reint_window &c = io[w];
            if (p.K < 2 || p.K > h->C.K || p.n_imu < 0 || p.n_imu > p.K - 1) {
                set_error("%s: window %d: sizes out of range", fn, w);
                return ICG_EINVAL;
            }
            if (!c.reintegrate || p.n_imu == 0) continue;
            if (!c.imu || !c.imu_off || !c.status || !c.blob_out) {
                set_error("%s: window %d: arrays missing", fn, w);
                return ICG_EINVAL;
            }
            if (c.imu_off[0] < 0) {
                set_error("%s: window %d: imu_off[0] is negative", fn, w);
                return ICG_EINVAL;
            }
            for (int k = 0; k < p.n_imu; k++)
                if (c.imu_off[k + 1] - c.imu_off[k] < 1) {
                    set_error("%s: window %d factor %d: imu_off must give every interval at least one row", fn, w, k);
                    return ICG_EINVAL;
                }
            n_items += p.n_imu, n_rows += (size_t) (c.imu_off[p.n_imu] - c.imu_off[0]);
        }
        if (n_items > INT32_MAX / 8 || n_rows > INT32_MAX / 8) {
            set_error("%s: too many factors or IMU rows in one call", fn);
            return ICG_EINVAL;
        }
        return ICG_OK;
    };
    int rc = validate();
    if (sharded) {  // every argument is camera side: the sizes, the flags, the rows, noise and station
        ArgPrint fp;
        fp.num(n);
        for (int w = 0; rc == ICG_OK && w < n; w++) {
            const icg_ba_problem &p = problems[w];
            const icg_ba_reint_window &c = io[w];
            const bool on = c.reintegrate && p.n_imu > 0;
            fp.num(p.K), fp.num(p.n_imu), fp.num(on);
            if (!on) continue;
            fp.arr(c.imu_off, p.n_imu + 1);
            fp.arr(c.imu + 7 * (size_t) c.imu_off[0], 7LL * (c.imu_off[p.n_imu] - c.imu_off[0]));
        }
        if (rc == ICG_OK) fp.arr(noise5, 5), fp.arr(station3, 3);
        rc = shard_agree(h, rc != ICG_OK, fp.get(), fn);
    }
    if (rc != ICG_OK) return rc;
    const BaCaps &C = h->C;
    for (int w = 0; w < n; w++) io[w].count = 0;
    if (n_items == 0) return ICG_OK;
    // staging: inputs [items | rows | counter (0)] go up in one copy; [counter | status | ends | out_item] come back in one copy, then the
    // status-1 blobs, compacted on the device
    auto al = [](size_t b) { return (b + 15) & ~(size_t) 15; };
    size_t at = 0;
    auto take = [&](size_t bytes) {
        const size_t o = at;
        at += al(bytes);
        return o;
    };
    const size_t i_item = take(sizeof(ReintItem) * n_items), i_rows = take(56 * n_rows), o_cnt = take(sizeof(int));
    const size_t o_status = take(n_items), o_ends = take(80 * n_items), o_item = take(4 * n_items), o_blob = take(sizeof(double) * ICG_IMU_BLOB_DOUBLES * n_items);
    ICG_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    if (at > h->reint_cap) {
        ICG_CUDA(cudaStreamSynchronize(s));
        retire(h, h->reint_d, h->reint_h);  // a shard group keeps it: freeing would wait for a peer's kernel
        h->reint_h = nullptr, h->reint_d = nullptr;
        h->reint_cap = 0;
        const size_t cap = at + at / 4;
        if (cudaMallocHost(&h->reint_h, cap) != cudaSuccess || cudaMalloc(&h->reint_d, cap) != cudaSuccess) {
            set_error("%s: staging allocation of %zu bytes failed", fn, cap);
            return ICG_ENOMEM;
        }
        h->reint_cap = cap;
    }
    unsigned char *H = h->reint_h, *Dv = h->reint_d;
    ReintItem *items = (ReintItem *) (H + i_item);
    std::vector<int> first(n, -1);  // first item of each reintegrated window
    {
        size_t it = 0, row = 0;
        for (int w = 0; w < n; w++) {
            const icg_ba_problem &p = problems[w];
            const icg_ba_reint_window &c = io[w];
            if (!c.reintegrate || p.n_imu == 0) continue;
            first[w] = (int) it;
            const int r0 = c.imu_off[0], nr = c.imu_off[p.n_imu] - r0;
            memcpy(H + i_rows + 56 * row, c.imu + 7 * (size_t) r0, 56 * (size_t) nr);
            for (int k = 0; k < p.n_imu; k++, it++)
                items[it] = ReintItem{w, k, (int) row + c.imu_off[k] - r0, c.imu_off[k + 1] - c.imu_off[k]};
            row += nr;
        }
    }
    *(int *) (H + o_cnt) = 0;
    ICG_CUDA(cudaMemcpyAsync(Dv, H, o_status, cudaMemcpyHostToDevice, s));
    PreintResident a;
    a.n = (int) n_items, a.item = (const ReintItem *) (Dv + i_item), a.imu = (const double *) (Dv + i_rows);
    a.pose = h->D.pose, a.mix = h->D.mix, a.blob = h->D.imu_blob, a.U = h->D.imu_U, a.K = C.K;
    for (int k = 0; k < 5; k++) a.noise5[k] = noise5[k];
    for (int k = 0; k < 3; k++) a.station[k] = station3[k];
    a.status = (int8_t *) (Dv + o_status), a.ends = (double *) (Dv + o_ends), a.out_blob = (double *) (Dv + o_blob), a.out_item = (int *) (Dv + o_item);
    a.counter = (int *) (Dv + o_cnt);
    ICG_CUDA(preint_resident_launch(a, s));
    count_launch();
    ICG_CUDA(cudaMemcpyAsync(H + o_cnt, Dv + o_cnt, o_blob - o_cnt, cudaMemcpyDeviceToHost, s));
    ICG_CUDA(cudaStreamSynchronize(s));
    const int n_done = *(const int *) (H + o_cnt);
    if (n_done < 0 || (size_t) n_done > n_items) {
        set_error("%s: inconsistent completion count %d", fn, n_done);
        return ICG_ECUDA;
    }
    if (n_done > 0) {
        ICG_CUDA(cudaMemcpyAsync(H + o_blob, Dv + o_blob, sizeof(double) * ICG_IMU_BLOB_DOUBLES * (size_t) n_done, cudaMemcpyDeviceToHost, s));
        ICG_CUDA(cudaStreamSynchronize(s));
    }
    const int8_t *st = (const int8_t *) (H + o_status);
    const double *ends = (const double *) (H + o_ends);
    for (int q = 0; q < n_done; q++) {
        const ReintItem &it = items[((const int *) (H + o_item))[q]];
        memcpy(io[it.win].blob_out + (size_t) ICG_IMU_BLOB_DOUBLES * it.fac, H + o_blob + sizeof(double) * ICG_IMU_BLOB_DOUBLES * (size_t) q,
               sizeof(double) * ICG_IMU_BLOB_DOUBLES);
    }
    int bad_w = -1, bad_k = -1;
    for (int w = 0; w < n; w++) {
        if (first[w] < 0) continue;
        icg_ba_reint_window &c = io[w];
        for (int k = 0; k < problems[w].n_imu; k++) {
            const int q = first[w] + k;
            c.status[k] = st[q];
            if (st[q] != 0) {
                c.count++;
                if (c.end_state10) memcpy(c.end_state10 + 10 * (size_t) k, ends + 10 * (size_t) q, 80);
            }
            if (st[q] < 0 && bad_w < 0) bad_w = w, bad_k = k;
        }
    }
    if (bad_w >= 0) {
        set_error("%s: window %d IMU factor %d: the reintegrated covariance is not positive definite (the factor was kept)", fn, bad_w, bad_k);
        return ICG_EINVAL;
    }
    return ICG_OK;
}

int icg_ba_reintegrate_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const double *noise5, const double *station3,
                                icg_ba_reint_window *io) {
    return reint_body(h, n_windows, problems, noise5, station3, io, "icg_ba_reintegrate_resident", false);
}

// a collective call of a shard group: the entry points below take the sharded form of their plain counterpart's body
static int shard_group_only(icg_ba *h, const char *fn, const char *plain) {
    if (!h) {
        set_error("%s: bad arguments", fn);
        return ICG_EINVAL;
    }
    if (h->D.world < 2) {
        set_error("%s: the handle is not in a landmark-shard group (call %s)", fn, plain);
        return ICG_EINVAL;
    }
    return ICG_OK;
}

int icg_ba_shard_reintegrate_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const double *noise5, const double *station3,
                                      icg_ba_reint_window *io) {
    const char *fn = "icg_ba_shard_reintegrate_resident";
    const int rc = shard_group_only(h, fn, "icg_ba_reintegrate_resident");
    return rc != ICG_OK ? rc : reint_body(h, n_windows, problems, noise5, station3, io, fn, true);
}

int icg_ba_marginalize_resident_culled(icg_ba *h, int n_windows, const icg_ba_problem *problems, const int32_t *num_marg,
                                       const icg_ba_cull_window *culled, const uint8_t *const *node_in_map, icg_ba_prior *out) {
    int rc = resident_single_rank(h, n_windows, problems, "icg_ba_marginalize_resident_culled", true);
    if (rc != ICG_OK) return rc;
    if (!culled || !node_in_map) {
        set_error("icg_ba_marginalize_resident_culled: bad arguments");
        return ICG_EINVAL;
    }
    // the factor set of gvinsMarginalization (IG/ic_gvins.cc:1558-1609) from the culling's flags: on the host, beside the structure loop
    // of marginalize_body, which reads the factor set on the host as well
    std::vector<std::vector<uint8_t>> masks(n_windows);
    std::vector<const uint8_t *> mp(n_windows);
    for (int w = 0; w < n_windows; w++) {
        const icg_ba_problem &p = problems[w];
        const icg_ba_cull_window &c = culled[w];
        if (!node_in_map[w] || (p.L > 0 && (!c.lm_ref_node || !c.obs_off || !c.lm_outlier)) || p.K > h->C.K || p.L > h->C.L || p.F > h->C.F ||
            (p.L > 0 && c.obs_off[p.L] > 0 && (!c.obs_node || !c.obs_factor || !c.obs_outlier))) {
            set_error("icg_ba_marginalize_resident_culled: window %d: arrays missing", w);
            return ICG_EINVAL;
        }
        std::vector<uint8_t> &m = masks[w];
        m.assign(p.F, 1);
        std::vector<uint8_t> lm_bad(p.L, 0);
        for (int l = 0; l < p.L; l++) {
            lm_bad[l] = c.lm_outlier[l] != 0;
            for (int o = c.obs_off[l]; o < c.obs_off[l + 1]; o++) {
                const int f = c.obs_factor[o], k = c.obs_node[o];
                if (f < -1 || f >= p.F || (f >= 0 && (p.f_lm[f] != l || p.f_obs[f] != k))) {
                    set_error("icg_ba_marginalize_resident_culled: window %d landmark %d: observation %d names factor %d of another landmark or node", w, l, o, f);
                    return ICG_EINVAL;
                }
                if (!c.obs_outlier[o]) continue;
                if (k == c.lm_ref_node[l]) lm_bad[l] = 1;
                if (f >= 0) m[f] = 0;
            }
        }
        for (int f = 0; f < p.F; f++)
            if (lm_bad[p.f_lm[f]] || !node_in_map[w][p.f_obs[f]]) m[f] = 0;
        mp[w] = m.data();
    }
    if (h->D.world > 1) return marginalize_sharded(h, n_windows, problems, num_marg, out, mp.data(), "icg_ba_marginalize_resident_culled");
    return marginalize_body(h, n_windows, problems, num_marg, out, true, mp.data());
}

// ---- the next keyframe's windows from the resident ones (ba_slide.cu): the structure is packed on the host as icg_ba_upload packs it, the
//      values of the carried rows never leave the device.  With `integ`, the new factors, node rows and aligned fixes it names are computed on
//      the device (preint.cu) into the staged value rows before the gather reads them.
//
// sharded (icg_ba_shard_slide[_integrate]_resident, a collective call): the same checks, plus landmark-by-landmark factor lists and the owner's
// check of its own prior; then one agreement of the group (shard_agree: every rank's verdict and a fingerprint of the camera side) before any
// rank writes its device, and with `integ` a second one on the integration's outcome.  A rank that rejects joins the agreement all the same
// (fail below), so its peers never wait for it.  The owner of window w forms its prior from the workspace of mx_h; the other ranks get zeros.
// lm_ref_built: icg_ba_slide_vision_resident has written the next windows' reference rows into lm_ref_alt already
static int slide_body(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry, const icg_ba_slide_integrate *integ,
                      const double *noise5, const double *station3, const char *fn, bool sharded, bool lm_ref_built = false) {
    bool joined = false;  // sharded: this rank has joined the agreement of the call
    std::vector<WinDims> old_dims;
    std::vector<std::vector<int>> old_slot;
    // a rejected call leaves the handle as it was: the packing below rewrites the host tables later calls read (dims, which restore_params
    // uploads, and the slot table of the next slide), so they go back on failure; nothing reaches the device before every check has passed
    auto fail = [&](int code) {
        if (!old_dims.empty()) {
            memcpy(h->dims.h, old_dims.data(), sizeof(WinDims) * n);
            for (int w = 0; w < n; w++) {
                int *fidx = h->lm_fidx.h + (size_t) w * h->C.F;
                for (int f = 0; f < old_dims[w].F; f++) fidx[old_slot[w][f]] = f;
            }
        }
        // sharded: a rank that rejects before the agreement joins it with its rejection, and returns ICG_EINVAL as its peers do (its own
        // message says why); only a failed exchange (a peer did not make the call) returns that error instead
        if (sharded && !joined) joined = true, code = shard_agree(h, true, 0, fn);
        return code;
    };
    // a CUDA error before the agreement is this rank's rejection like any other
    auto cuda_fail = [&](cudaError_t e, const char *what) {
        set_error("%s: %s failed: %s", fn, what, cudaGetErrorString(e));
        return fail(ICG_ECUDA);
    };
    int rc = resident_single_rank(h, n, next, fn, sharded);
    if (rc != ICG_OK) return fail(rc);
    if (!carry || (integ && (!noise5 || !station3))) {
        set_error("%s: bad arguments", fn);
        return fail(ICG_EINVAL);
    }
    if (cudaError_t e = cudaSetDevice(h->device)) return cuda_fail(e, "cudaSetDevice");
    const BaCaps &C = h->C;
    const size_t NW = C.NW;
    const int G = h->D.world, R = h->D.rank;
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = next[w];
        if (sharded)
            for (int f = 1; p.f_lm && f < p.F; f++)
                if (p.f_lm[f] < p.f_lm[f - 1]) {
                    set_error("%s: window %d factor %d: a landmark-sharded window must list its factors landmark by landmark (f_lm non-decreasing)", fn, w, f);
                    return fail(ICG_EINVAL);
                }
        if (!carry[w].prior_from_marg) continue;
        if (h->marg_res_n != n || h->marg_res_sharded != sharded) {
            set_error("%s: window %d takes its prior from the marginalization, but no %sresident marginalization of these %d windows "
                      "ran since the last upload or slide", fn, w, sharded ? "sharded " : "", n);
            return fail(ICG_EINVAL);
        }
        if (sharded && w % G != R) continue;  // the owner holds the window's m, r and nblocks
        if (h->marg_res_m[w] <= 0 || p.marg_r != h->marg_res_r[w] || p.marg_nblocks != h->marg_res_nb[w]) {
            set_error("%s: window %d: marg_r=%d / marg_nblocks=%d, but the resident marginalization left m=%d, r=%d / nblocks=%d", fn, w,
                      p.marg_r, p.marg_nblocks, h->marg_res_m[w], h->marg_res_r[w], h->marg_res_nb[w]);
            return fail(ICG_EINVAL);
        }
    }
    // the device buffers of the first slide: the old value rows at the handle's strides, the second f_const_s
    const size_t o_mix = NW * C.K * 7, o_rho = o_mix + NW * C.K * 9, o_blob = o_rho + NW * C.L, o_U = o_blob + NW * C.K * ICG_IMU_BLOB_DOUBLES,
                 o_blh = o_U + NW * C.K * 225, o_std = o_blh + NW * C.G * 3, n_old = o_std + NW * C.G * 3;
    if (!h->slide_old && (cudaMalloc(&h->slide_old, sizeof(double) * n_old) != cudaSuccess ||
                          cudaMalloc(&h->fc_alt, sizeof(double) * NW * C.F * 14) != cudaSuccess)) {
        if (h->slide_old) cudaFree(h->slide_old), h->slide_old = nullptr;
        set_error("%s: allocation of the slide buffers failed", fn);
        return fail(ICG_ENOMEM);
    }
    // the old windows: sizes, and every factor's record slot (the inverse of the last packing's slot -> factor table)
    old_dims.assign(h->dims.h, h->dims.h + n);
    old_slot.resize(n);
    for (int w = 0; w < n; w++) {
        old_slot[w].resize(old_dims[w].F);
        const int *fidx = h->lm_fidx.h + (size_t) w * C.F;
        for (int q = 0; q < old_dims[w].F; q++) old_slot[w][fidx[q]] = q;
    }
    rc = pack_windows(h, n, next, false);
    if (rc != ICG_OK) return fail(rc);
    // the maps: range checks, sizes of the staging
    std::vector<SlideWin> wins(n);
    std::vector<size_t> vbase(n);  // first staged value of each window
    size_t n_map = 0, n_val = 0;
    int max_elems = 0, max_r = 0;
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = next[w];
        const icg_ba_slide_window &c = carry[w];
        const WinDims &od = old_dims[w];
        const int32_t *maps[5] = {c.node_src, c.lm_src, c.f_src, c.imu_src, c.gnss_src};
        const int cnt[5] = {p.K, p.L, p.F, p.n_imu, p.n_gnss}, lim[5] = {od.K, od.L, od.F, od.n_imu, od.n_gnss}, width[5] = {SLIDE_NODE, 1, 14, SLIDE_IMU, SLIDE_GNSS};
        static const char *names[5] = {"node_src", "lm_src", "f_src", "imu_src", "gnss_src"};
        vbase[w] = n_val;
        for (int t = 0; t < 5; t++)
            for (int i = 0; maps[t] && i < cnt[t]; i++) {
                if (maps[t][i] < -1 || maps[t][i] >= lim[t]) {
                    set_error("%s: window %d: %s[%d] = %d is out of range of the old window (%d)", fn, w, names[t], i, maps[t][i], lim[t]);
                    return fail(ICG_EINVAL);
                }
                if (maps[t][i] >= 0) continue;
                n_val += width[t];
            }
        for (int t = 0; t < 5; t++)
            if (!maps[t]) n_val += (size_t) width[t] * cnt[t];
        SlideWin &W = wins[w];
        W.K = p.K, W.L = p.L, W.F = p.F, W.n_imu = p.n_imu, W.n_gnss = p.n_gnss;
        W.node_map = (int) n_map, W.lm_map = W.node_map + p.K, W.slot_map = W.lm_map + p.L, W.imu_map = W.slot_map + p.F, W.gnss_map = W.imu_map + p.n_imu;
        n_map = (size_t) W.gnss_map + p.n_gnss;
        W.r = p.marg_r, W.from_marg = c.prior_from_marg != 0, W.j0 = W.e0 = 0;
        W.slot = !sharded ? w : w % G == R ? (w - R) / G : -1;
        if (W.r > 0 && !W.from_marg) n_val += (size_t) W.r * W.r + W.r;
        max_elems = std::max(max_elems, SLIDE_NODE * p.K + p.L + 14 * p.F + SLIDE_IMU * p.n_imu + SLIDE_GNSS * p.n_gnss);
        max_r = std::max(max_r, W.r);
    }
    // the integration's arrays (only rows the carry maps leave to next are read): every check before anything is staged
    std::vector<std::vector<int>> item_of(integ ? n : 0);  // per window and new factor: its item, or -1
    std::vector<int> iwin_of(integ ? n : 0, -1);           // per window: its entry of iwins, or -1
    std::vector<SlideIntWin> iwins;                         // the windows with device work, one warp each
    std::vector<size_t> row_base(integ ? n : 0), state_base(integ ? n : 0);
    size_t n_item = 0, n_align = 0, n_row = 0, n_state = 0;
    bool want_blob = false;
    for (int w = 0; integ && w < n; w++) {
        const icg_ba_problem &p = next[w];
        const icg_ba_slide_window &c = carry[w];
        const icg_ba_slide_integrate &g = integ[w];
        const int oK = old_dims[w].K;
        std::vector<int> &io = item_of[w];
        io.assign(p.n_imu, -1);
        const size_t item0 = n_item, align0 = n_align;
        row_base[w] = n_row, state_base[w] = n_state;
        for (int k = 0; g.imu_from && k < p.n_imu; k++) {
            const int src = g.imu_from[k];
            if ((c.imu_src && c.imu_src[k] >= 0) || src == -1) continue;
            if (src >= oK || (src < 0 && src != ICG_SLIDE_CHAIN && src != ICG_SLIDE_ROW)) {
                set_error("%s: window %d: imu_from[%d] = %d is out of range of the old window (%d)", fn, w, k, src, oK);
                return fail(ICG_EINVAL);
            }
            if (src == ICG_SLIDE_CHAIN && (k == 0 || io[k - 1] < 0)) {
                set_error("%s: window %d: imu_from[%d] is ICG_SLIDE_CHAIN, but no integrated factor precedes it", fn, w, k);
                return fail(ICG_EINVAL);
            }
            if (!g.gravity3 || !g.imu || !g.imu_off || (src == ICG_SLIDE_ROW && !g.state16)) {
                set_error("%s: window %d: arrays missing", fn, w);
                return fail(ICG_EINVAL);
            }
            if (g.imu_off[k] < 0 || (long long) g.imu_off[k + 1] - g.imu_off[k] < 1) {
                set_error("%s: window %d factor %d: imu_off must give every integrated interval at least one row", fn, w, k);
                return fail(ICG_EINVAL);
            }
            io[k] = (int) n_item++;
            n_row += (size_t) (g.imu_off[k + 1] - g.imu_off[k]);
            n_state += src == ICG_SLIDE_ROW;
        }
        for (int j = 0; g.node_from_imu && j < p.K; j++) {
            if ((c.node_src && c.node_src[j] >= 0) || !g.node_from_imu[j]) continue;
            if (j == 0 || j - 1 >= p.n_imu || io[j - 1] < 0) {
                set_error("%s: window %d: node_from_imu[%d] is set, but factor %d is not integrated", fn, w, j, j - 1);
                return fail(ICG_EINVAL);
            }
        }
        for (int q = 0; g.gnss_node && q < p.n_gnss; q++) {
            if ((c.gnss_src && c.gnss_src[q] >= 0) || g.gnss_node[q] == -1) continue;
            if (g.gnss_node[q] < -1 || g.gnss_node[q] >= oK) {
                set_error("%s: window %d: gnss_node[%d] = %d is out of range of the old window (%d)", fn, w, q, g.gnss_node[q], oK);
                return fail(ICG_EINVAL);
            }
            if (!g.gnss_dt) {
                set_error("%s: window %d: arrays missing", fn, w);
                return fail(ICG_EINVAL);
            }
            n_align++;
        }
        if (n_item == item0 && n_align == align0) continue;
        iwin_of[w] = (int) iwins.size();
        iwins.push_back(SlideIntWin{w, (int) item0, (int) (n_item - item0), (int) align0, (int) (n_align - align0)});
        want_blob = want_blob || (g.blob_out && n_item > item0);
    }
    if (n_val >= (size_t) INT32_MAX || n_map >= (size_t) INT32_MAX || n_row >= (size_t) INT32_MAX / 8 || n_item >= (size_t) INT32_MAX / 8) {
        set_error("%s: too many new value rows in one call", fn);
        return fail(ICG_EINVAL);
    }
    // staging: [windows | maps | new value rows] in one pinned buffer, one H2D; with device work also [its windows | items | alignments |
    // IMU rows | ICG_SLIDE_ROW states] (up to in_end) and the outputs that come back, [status | end states | blobs]
    auto al = [](size_t b) { return (b + 15) & ~(size_t) 15; };
    const size_t b_map = al(sizeof(SlideWin) * n), b_val = b_map + al(sizeof(int) * n_map);
    size_t total = b_val + sizeof(double) * n_val;
    auto take = [&](size_t bytes) {
        const size_t o = al(total);
        total = o + bytes;
        return o;
    };
    size_t b_iw = 0, b_item = 0, b_align = 0, b_rows = 0, b_state = 0, b_status = 0, b_ends = 0, b_blob = 0;
    if (!iwins.empty()) {
        b_iw = take(sizeof(SlideIntWin) * iwins.size()), b_item = take(sizeof(SlideItem) * n_item), b_align = take(sizeof(SlideAlign) * n_align);
        b_rows = take(56 * n_row), b_state = take(128 * n_state);
    }
    const size_t in_end = total;
    if (!iwins.empty()) {
        b_status = take(n_item), b_ends = take(80 * n_item);
        if (want_blob) b_blob = take(sizeof(double) * ICG_IMU_BLOB_DOUBLES * n_item);
    }
    cudaStream_t s = h->stream;
    if (total > h->slide_cap) {
        if (cudaError_t e = cudaStreamSynchronize(s)) return cuda_fail(e, "cudaStreamSynchronize");  // an earlier slide's copy may read the old buffer
        retire(h, h->slide_d, h->slide_h);    // a shard group keeps it: freeing would wait for a peer's kernel
        h->slide_h = nullptr, h->slide_d = nullptr;
        h->slide_cap = 0;
        const size_t cap = total + total / 4;
        if (cudaMallocHost(&h->slide_h, cap) != cudaSuccess || cudaMalloc(&h->slide_d, cap) != cudaSuccess) {
            set_error("%s: staging allocation of %zu bytes failed", fn, cap);
            return fail(ICG_ENOMEM);
        }
        h->slide_cap = cap;
    } else if (h->slide_ev) {
        // the previous slide's H2D has left the pinned buffer before it is rewritten
        if (cudaError_t e = cudaEventSynchronize(h->slide_ev)) return cuda_fail(e, "cudaEventSynchronize");
    }
    if (!h->slide_ev)
        if (cudaError_t e = cudaEventCreateWithFlags(&h->slide_ev, cudaEventDisableTiming)) return cuda_fail(e, "cudaEventCreateWithFlags");
    int *map = (int *) (h->slide_h + b_map);
    double *val = (double *) (h->slide_h + b_val);
    SlideItem *items = (SlideItem *) (h->slide_h + b_item);
    SlideAlign *aligns = (SlideAlign *) (h->slide_h + b_align);
    double *rows = (double *) (h->slide_h + b_rows), *states = (double *) (h->slide_h + b_state);
    // per window: its slices of the maps, the values and the integration's inputs are disjoint, so the windows are staged on a few host
    // threads, as pack_windows packs them (the square-root information of every new blob is a 15 x 15 factorisation).  A row the device
    // computes gets its value slot here and is written there.
    auto stage_window = [&](int w, std::string &err) -> int {
        const icg_ba_problem &p = next[w];
        const icg_ba_slide_window &c = carry[w];
        const icg_ba_slide_integrate *g = integ && iwin_of[w] >= 0 ? &integ[w] : nullptr;
        SlideWin &W = wins[w];
        int vo = (int) vbase[w];
        auto stage = [&](const double *src, int count) {
            const int at = vo;
            memcpy(val + vo, src, sizeof(double) * count);
            vo += count;
            return -(at + 1);
        };
        std::vector<int> node_at(g ? p.K + 1 : 0, -1);  // value offset of a node row the device writes
        for (int k = 0; k < p.K; k++) {
            if (c.node_src && c.node_src[k] >= 0) {
                map[W.node_map + k] = c.node_src[k];
                continue;
            }
            if (g && g->node_from_imu && g->node_from_imu[k]) {
                node_at[k] = vo, map[W.node_map + k] = -(vo + 1), vo += SLIDE_NODE;
                continue;
            }
            map[W.node_map + k] = stage(p.pose + 7 * (size_t) k, 7);
            stage(p.mix + 9 * (size_t) k, 9);
        }
        for (int l = 0; l < p.L; l++) map[W.lm_map + l] = c.lm_src && c.lm_src[l] >= 0 ? c.lm_src[l] : stage(p.invdepth + l, 1);
        const int *fidx = h->lm_fidx.h + (size_t) w * C.F;  // the new packing's slot -> factor table
        for (int q = 0; q < p.F; q++) {
            const int f = fidx[q];
            map[W.slot_map + q] = c.f_src && c.f_src[f] >= 0 ? old_slot[w][c.f_src[f]] : stage(p.f_const + 14 * (size_t) f, 14);
        }
        size_t row_at = g ? row_base[w] : 0, state_at = g ? state_base[w] : 0;
        for (int k = 0; k < p.n_imu; k++) {
            if (c.imu_src && c.imu_src[k] >= 0) {
                map[W.imu_map + k] = c.imu_src[k];
                continue;
            }
            if (g && item_of[w][k] >= 0) {
                SlideItem &it = items[item_of[w][k]];
                const int r0 = g->imu_off[k], nr = g->imu_off[k + 1] - r0;
                it.src = g->imu_from[k], it.row0 = (int) row_at, it.nrow = nr, it.state = -1, it.blob = vo, it.node = node_at[k + 1];
                it.normal = g->normal && g->normal[k] ? 1 : 0;
                for (int i = 0; i < 3; i++) it.grav[i] = g->gravity3[3 * (size_t) k + i];
                memcpy(rows + 7 * row_at, g->imu + 7 * (size_t) r0, 56 * (size_t) nr);
                row_at += nr;
                if (it.src == ICG_SLIDE_ROW) {
                    memcpy(states + 16 * state_at, g->state16 + 16 * (size_t) k, 128);
                    it.state = (int) (16 * state_at++);
                }
                map[W.imu_map + k] = -(vo + 1), vo += SLIDE_IMU;
                continue;
            }
            const double *b = p.imu_blob + (size_t) k * ICG_IMU_BLOB_DOUBLES;
            map[W.imu_map + k] = stage(b, ICG_IMU_BLOB_DOUBLES);
            if (!host_imu_sqrt_info(b + 252, val + vo)) {
                char eb[256];
                snprintf(eb, sizeof(eb), "%s: window %d IMU factor %d has a non positive-definite covariance", fn, w, k);
                err = eb;
                return ICG_EINVAL;
            }
            vo += 225;
        }
        int align_at = g ? iwins[iwin_of[w]].align0 : 0;
        for (int q = 0; q < p.n_gnss; q++) {
            if (c.gnss_src && c.gnss_src[q] >= 0) {
                map[W.gnss_map + q] = c.gnss_src[q];
                continue;
            }
            map[W.gnss_map + q] = stage(p.gnss_blh + 3 * (size_t) q, 3);
            stage(p.gnss_std + 3 * (size_t) q, 3);
            if (g && g->gnss_node && g->gnss_node[q] >= 0) aligns[align_at++] = SlideAlign{-(map[W.gnss_map + q] + 1), g->gnss_node[q], g->gnss_dt[q]};
        }
        if (W.r > 0 && !W.from_marg) {
            W.j0 = -(stage(p.marg_J0, W.r * W.r) + 1);
            W.e0 = -(stage(p.marg_e0, W.r) + 1);
        }
        return ICG_OK;
    };
    {
        const int nthreads = std::max(1, std::min({n / 4, 16, (int) std::thread::hardware_concurrency()}));
        std::vector<int> rcs(nthreads, ICG_OK);
        std::vector<std::string> errs(nthreads);
        auto worker = [&](int t) {
            for (int w = t; w < n && rcs[t] == ICG_OK; w += nthreads) rcs[t] = stage_window(w, errs[t]);
        };
        std::vector<std::thread> th;
        for (int t = 1; t < nthreads; t++) th.emplace_back(worker, t);
        worker(0);
        for (auto &x : th) x.join();
        for (int t = 0; t < nthreads; t++)
            if (rcs[t] != ICG_OK) {
                set_error("%s", errs[t].c_str());
                return fail(rcs[t]);
            }
    }
    if (sharded) {
        ArgPrint fp;
        fp.num(n);
        if (integ) fp.arr(noise5, 5), fp.arr(station3, 3);
        for (int w = 0; w < n; w++) {
            const icg_ba_problem &p = next[w];
            const icg_ba_slide_window &c = carry[w];
            const icg_ba_slide_integrate *g = integ ? &integ[w] : nullptr;
            fp.num(p.K), fp.num(p.n_imu), fp.num(p.n_gnss), fp.num(c.prior_from_marg), fp.num(p.marg_r), fp.num(p.marg_nblocks);
            // the flags and camera-side values the structure packing reads from next
            fp.arr(p.ext, 8), fp.num(p.ext_const), fp.num(p.td_const), fp.arr(&p.reproj_std, 1), fp.num(p.reproj_huber), fp.num(p.gnss_huber);
            fp.num(p.has_imu_error), fp.arr(p.lever, 3), fp.num(p.has_pose_prior), fp.num(p.has_mix_prior);
            if (p.has_pose_prior) fp.arr(p.pose_prior, 7), fp.arr(p.pose_prior_std, 6);
            if (p.has_mix_prior) fp.arr(p.mix_prior, 9), fp.arr(p.mix_prior_std, 9);
            fp.num(!c.node_src), fp.num(!c.imu_src), fp.num(!c.gnss_src);
            fp.arr(c.node_src, p.K), fp.arr(c.imu_src, p.n_imu), fp.arr(c.gnss_src, p.n_gnss), fp.arr(p.gnss_node, p.n_gnss);
            for (int k = 0; k < p.K; k++) {
                if (c.node_src && c.node_src[k] >= 0) continue;
                if (g && g->node_from_imu && g->node_from_imu[k]) fp.num(-1);
                else fp.arr(p.pose + 7 * (size_t) k, 7), fp.arr(p.mix + 9 * (size_t) k, 9);
            }
            for (int k = 0; k < p.n_imu; k++) {
                if (c.imu_src && c.imu_src[k] >= 0) continue;
                const int q = g ? item_of[w][k] : -1;
                if (q < 0) {
                    fp.arr(p.imu_blob + (size_t) k * ICG_IMU_BLOB_DOUBLES, ICG_IMU_BLOB_DOUBLES);
                    continue;
                }
                fp.num(g->imu_from[k]), fp.arr(g->gravity3 + 3 * (size_t) k, 3), fp.num(g->normal && g->normal[k]);
                fp.arr(g->imu + 7 * (size_t) g->imu_off[k], 7LL * (g->imu_off[k + 1] - g->imu_off[k]));
                if (g->imu_from[k] == ICG_SLIDE_ROW) fp.arr(g->state16 + 16 * (size_t) k, 16);
            }
            for (int q = 0; q < p.n_gnss; q++) {
                if (c.gnss_src && c.gnss_src[q] >= 0) continue;
                fp.arr(p.gnss_blh + 3 * (size_t) q, 3), fp.arr(p.gnss_std + 3 * (size_t) q, 3);
                if (g && g->gnss_node) fp.num(g->gnss_node[q]), fp.arr(g->gnss_node[q] >= 0 ? g->gnss_dt + q : nullptr, 1);
            }
            if (p.marg_r > 0) {
                long long nx = 0;
                for (int b = 0; p.marg_block_type && b < p.marg_nblocks; b++) nx += p.marg_block_type[b] == 1 ? 9 : p.marg_block_type[b] == 3 ? 1 : 7;
                fp.arr(p.marg_block_type, p.marg_nblocks), fp.arr(p.marg_block_node, p.marg_nblocks), fp.arr(p.marg_x0, nx);
                if (!c.prior_from_marg) fp.arr(p.marg_J0, (long long) p.marg_r * p.marg_r), fp.arr(p.marg_e0, p.marg_r);
            }
        }
        joined = true;
        if ((rc = shard_agree(h, false, fp.get(), fn)) != ICG_OK) return fail(rc);
    }
    memcpy(h->slide_h, wins.data(), sizeof(SlideWin) * n);
    if (integ) {
        // the device work writes the staging only; a covariance that is not positive definite is known after it, so the call waits for it.
        // Sharded: the ranks integrate the same rows from the same states; the outcome is agreed on all the same before the device is written
        int irc = ICG_OK;
        if (!iwins.empty()) {
            memcpy(h->slide_h + b_iw, iwins.data(), sizeof(SlideIntWin) * iwins.size());
            PreintSlide a;
            a.n = (int) iwins.size(), a.win = (const SlideIntWin *) (h->slide_d + b_iw), a.item = (const SlideItem *) (h->slide_d + b_item);
            a.align = (const SlideAlign *) (h->slide_d + b_align), a.imu = (const double *) (h->slide_d + b_rows);
            a.state = (const double *) (h->slide_d + b_state), a.pose = h->D.pose, a.mix = h->D.mix, a.K = C.K, a.val = (double *) (h->slide_d + b_val);
            for (int k = 0; k < 5; k++) a.noise5[k] = noise5[k];
            for (int k = 0; k < 3; k++) a.station[k] = station3[k];
            a.status = (int8_t *) (h->slide_d + b_status), a.ends = (double *) (h->slide_d + b_ends);
            a.out_blob = want_blob ? (double *) (h->slide_d + b_blob) : nullptr;
            cudaError_t e = cudaMemcpyAsync(h->slide_d, h->slide_h, in_end, cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = preint_slide_launch(a, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(h->slide_h + b_status, h->slide_d + b_status, total - b_status, cudaMemcpyDeviceToHost, s);
            if (e == cudaSuccess) e = cudaStreamSynchronize(s);
            if (e != cudaSuccess) {
                set_error("%s: the integration on the device failed: %s", fn, cudaGetErrorString(e));
                irc = ICG_ECUDA;
            }
            count_launch();
        }
        const int8_t *st = (const int8_t *) (h->slide_h + b_status);
        const double *ends = (const double *) (h->slide_h + b_ends), *blobs = (const double *) (h->slide_h + b_blob);
        int bad_w = -1, bad_k = -1;
        for (int w = 0; irc == ICG_OK && w < n; w++) {
            const icg_ba_slide_integrate &g = integ[w];
            for (int k = 0; k < next[w].n_imu; k++) {
                const int q = item_of[w][k];
                if (g.status) g.status[k] = q >= 0 ? st[q] : 0;
                if (q < 0) continue;
                if (g.end_state10) memcpy(g.end_state10 + 10 * (size_t) k, ends + 10 * (size_t) q, 80);
                if (g.blob_out) memcpy(g.blob_out + (size_t) ICG_IMU_BLOB_DOUBLES * k, blobs + (size_t) ICG_IMU_BLOB_DOUBLES * q, 8 * ICG_IMU_BLOB_DOUBLES);
                if (st[q] < 0 && bad_w < 0) bad_w = w, bad_k = k;
            }
        }
        if (bad_w >= 0) {
            set_error("%s: window %d IMU factor %d: the integrated covariance is not positive definite", fn, bad_w, bad_k);
            irc = ICG_EINVAL;
        }
        if (sharded) irc = shard_agree(h, irc != ICG_OK, 0, fn);  // a rank's own rejection or a peer's: ICG_EINVAL on every rank
        if (irc != ICG_OK) return fail(irc);
    }
    // every check has passed: from here on the device is written
    h->marg_res_n = 0;
    h->cull_res_n = 0;
    if (iwins.empty()) ICG_CUDA(cudaMemcpyAsync(h->slide_d, h->slide_h, in_end, cudaMemcpyHostToDevice, s));
    ICG_CUDA(cudaEventRecord(h->slide_ev, s));
    rc = upload_structure(h, n);
    if (rc != ICG_OK) return rc;
    BaDev &D = h->D;
    double *old = h->slide_old;
    const size_t nn = (size_t) n;
    auto d2d = [&](double *dst, const double *src, size_t count) { return cudaMemcpyAsync(dst, src, sizeof(double) * count, cudaMemcpyDeviceToDevice, s); };
    ICG_CUDA(d2d(old, D.pose, nn * C.K * 7));
    ICG_CUDA(d2d(old + o_mix, D.mix, nn * C.K * 9));
    ICG_CUDA(d2d(old + o_rho, D.rho, nn * C.L));
    ICG_CUDA(d2d(old + o_blob, D.imu_blob, nn * C.K * ICG_IMU_BLOB_DOUBLES));
    ICG_CUDA(d2d(old + o_U, D.imu_U, nn * C.K * 225));
    ICG_CUDA(d2d(old + o_blh, D.gnss_blh, nn * C.G * 3));
    ICG_CUDA(d2d(old + o_std, D.gnss_std, nn * C.G * 3));
    SlideArgs a;
    a.win = (const SlideWin *) h->slide_d, a.map = (const int *) (h->slide_d + b_map), a.val = (const double *) (h->slide_d + b_val);
    a.K = C.K, a.L = C.L, a.F = C.F, a.G = C.G, a.R = C.R;
    a.old_pose = old, a.old_mix = old + o_mix, a.old_rho = old + o_rho, a.old_fc = D.f_const_s, a.old_blob = old + o_blob, a.old_U = old + o_U;
    a.old_blh = old + o_blh, a.old_std = old + o_std;
    a.pose = D.pose, a.mix = D.mix, a.rho = D.rho, a.fc = h->fc_alt, a.blob = D.imu_blob, a.U = D.imu_U, a.blh = D.gnss_blh, a.std = D.gnss_std;
    const icg_ba *mw = sharded ? h->mx_h : h;  // the marginalization's workspace (sharded: the owner's gather handle; none on a rank owning no window)
    a.mJ0 = mw ? mw->M.J0 : nullptr, a.me0 = mw ? mw->M.e0 : nullptr, a.mrcap = mw ? mw->M.rcap : 0;
    a.H0 = D.marg_H0, a.b0 = D.marg_b0, a.c0 = D.marg_c0;
    ICG_CUDA(launch_slide(a, n, max_elems, max_r, s));
    count_launch(2);
    std::swap(h->f_const_s.d, h->fc_alt);  // the gathered record constants become the handle's
    D.f_const_s = h->f_const_s.d;
    if (!lm_ref_built) ICG_CUDA(launch_lm_ref_fill(h, n, a.win, a.map, h->lm_ref, h->lm_ref_alt));
    std::swap(h->lm_ref, h->lm_ref_alt);
    rc = keep_pristine(h, n);
    if (rc != ICG_OK) return rc;
    h->cur_windows = n;
    return ICG_OK;
}

int icg_ba_slide_resident(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry) {
    return slide_body(h, n, next, carry, nullptr, nullptr, nullptr, "icg_ba_slide_resident", false);
}

int icg_ba_slide_integrate_resident(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry, const icg_ba_slide_integrate *integ,
                                    const double *noise5, const double *station3) {
    if (!integ) {
        set_error("icg_ba_slide_integrate_resident: bad arguments");
        return ICG_EINVAL;
    }
    return slide_body(h, n, next, carry, integ, noise5, station3, "icg_ba_slide_integrate_resident", false);
}

// the vision half of the next windows built on the device (ba_vision.cu), then the slide of those windows
int icg_ba_slide_vision_resident(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry, const icg_ba_slide_integrate *integ,
                                 const double *noise5, const double *station3, icg_ba_slide_vision *vis) {
    static const char *fn = "icg_ba_slide_vision_resident";
    if (h && h->D.world > 1) {
        set_error("%s: not available on a landmark-sharded handle", fn);
        return ICG_EUNSUPPORTED;
    }
    int rc = resident_single_rank(h, n, next, fn);
    if (rc != ICG_OK) return rc;
    if (!carry || !vis || (integ && (!noise5 || !station3))) {
        set_error("%s: bad arguments", fn);
        return ICG_EINVAL;
    }
    if (h->cull_res_n != n) {
        set_error("%s: no culling of these %d windows is current (icg_ba_update_and_cull_resident, with no upload or slide since)", fn, n);
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    const BaCaps &C = h->C;
    std::vector<VisWin> wins(n);
    size_t n_ofac = 0, n_lm = 0, n_f = 0, n_nf = 0, n_scr = 0;
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = next[w];
        const icg_ba_slide_vision &v = vis[w];
        const WinDims &od = h->dims.h[w];
        const CullWin &cw = h->cull_res_win[w];
        const int nco = h->cull_res_nobs[w];
        bool bad = p.K < 2 || p.K > C.K || v.num_marg < 0 || v.num_marg > od.K || !v.node_in_map || !v.node_td || v.cur_node < 0 || v.cur_node >= p.K ||
                   v.n_frames < 0 || v.n_frames > VIS_MAX_FRAMES || (v.n_frames > 0 && (!v.frame_id || !v.frame_node)) || v.n_obs < 0 || v.n_new < 0 ||
                   (v.obs_src && v.n_in < 0) || (v.n_obs > 0 && (!v.obs_lm || !v.obs_undis_xy || !v.obs_vel)) ||
                   (v.n_new > 0 && (!v.new_depth || !v.new_vel_ref || !v.new_vel_cur || !v.new_ref_undis_xy || !v.new_cur_undis_xy || !v.new_ref_frame_id)) ||
                   (nco > 0 && !v.obs_factor) || cw.K != od.K || cw.L != od.L;
        for (int e = 0; !bad && e < v.n_frames; e++) bad = v.frame_node[e] < 0 || v.frame_node[e] >= p.K;
        if (bad) {
            set_error("%s: window %d: arguments out of range or arrays missing", fn, w);
            return ICG_EINVAL;
        }
        VisWin &W = wins[w];
        memset(&W, 0, sizeof(W));
        W.cam = v.cam;
        memcpy(W.node_td, v.node_td, sizeof(double) * p.K);
        memset(W.onode, -1, sizeof(W.onode));
        const int32_t *ns = carry[w].node_src;
        for (int j = 0; ns && j < p.K; j++)
            if (ns[j] >= v.num_marg && ns[j] < od.K && v.node_in_map[ns[j]]) W.onode[ns[j]] = (int8_t) j;
        for (int e = 0; e < v.n_frames; e++) W.frame_id[e] = v.frame_id[e], W.frame_node[e] = v.frame_node[e];
        W.oK = od.K, W.oL = od.L, W.oF = od.F, W.nK = p.K, W.n_frames = v.n_frames, W.cur_node = v.cur_node;
        W.cull_lm0 = cw.lm0, W.cull_off0 = cw.off0, W.cull_obs0 = cw.obs0, W.n_cull_obs = nco, W.obs_factor0 = (int) n_ofac;
        W.n_obs = v.n_obs, W.n_in = v.obs_src ? v.n_in : v.n_obs, W.dev_n = v.dev_n, W.src = v.obs_src, W.obs_node = v.obs_node, W.obs_lm = v.obs_lm;
        W.obs_xy = v.obs_undis_xy, W.obs_vel = v.obs_vel;
        W.n_new = v.n_new, W.dev_new_n = v.dev_new_n, W.new_depth = v.new_depth, W.new_vel_ref = v.new_vel_ref, W.new_vel_cur = v.new_vel_cur;
        W.new_ref_xy = v.new_ref_undis_xy, W.new_cur_xy = v.new_cur_undis_xy, W.new_ref_frame = v.new_ref_frame_id;
        W.lm_out = (int) n_lm, W.f_out = (int) n_f, W.nf_out = (int) n_nf, W.scr = (int) n_scr;
        n_ofac += nco, n_lm += (size_t) od.L + v.n_new, n_f += (size_t) od.F + v.n_obs + v.n_new, n_nf += (size_t) v.n_obs + v.n_new;
        n_scr += (size_t) od.F + 3 * (size_t) od.L + 5 * ((size_t) od.L + v.n_new) + v.n_new;  // ba_vision_build's scratch
        if (n_ofac >= INT32_MAX / 2 || n_f >= INT32_MAX / 16 || n_scr >= INT32_MAX / 2) {
            set_error("%s: too many rows in one call", fn);
            return ICG_EINVAL;
        }
    }
    // staging: inputs [windows | obs_factor], outputs [counts | lm_src | lm_org | f_lm | f_ref | f_obs | f_src | invdepth | new factor rows |
    // NaN flags], then the kernel's scratch (never copied)
    auto al = [](size_t b) { return (b + 15) & ~(size_t) 15; };
    size_t at = 0;
    auto take = [&](size_t bytes) {
        const size_t o = at;
        at += al(bytes);
        return o;
    };
    const size_t b_win = take(sizeof(VisWin) * n), b_ofac = take(4 * n_ofac), in_end = at;
    const size_t b_cnt = take(4 * VIS_COUNTS * (size_t) n), b_lms = take(4 * n_lm), b_org = take(4 * n_lm), b_flm = take(4 * n_f), b_fref = take(4 * n_f), b_fobs = take(4 * n_f),
                 b_fsrc = take(4 * n_f), b_invd = take(8 * n_lm), b_fnew = take(112 * n_nf), b_nan = take(n_lm), out_end = at, b_scr = take(4 * n_scr);
    cudaStream_t s = h->stream;
    if (at > h->vis_cap) {
        ICG_CUDA(cudaStreamSynchronize(s));
        if (h->vis_h) cudaFreeHost(h->vis_h);
        if (h->vis_d) cudaFree(h->vis_d);
        h->vis_h = nullptr, h->vis_d = nullptr, h->vis_cap = 0;
        const size_t cap = at + at / 4;
        if (cudaMallocHost(&h->vis_h, cap) != cudaSuccess || cudaMalloc(&h->vis_d, cap) != cudaSuccess) {
            set_error("%s: staging allocation of %zu bytes failed", fn, cap);
            return ICG_ENOMEM;
        }
        h->vis_cap = cap;
    }
    unsigned char *H = h->vis_h, *Dv = h->vis_d;
    memcpy(H + b_win, wins.data(), sizeof(VisWin) * n);
    for (int w = 0; w < n; w++)
        if (wins[w].n_cull_obs > 0) memcpy(H + b_ofac + 4 * (size_t) wins[w].obs_factor0, vis[w].obs_factor, 4 * (size_t) wins[w].n_cull_obs);
    ICG_CUDA(cudaMemcpyAsync(Dv, H, in_end, cudaMemcpyHostToDevice, s));
    VisArgs a;
    a.win = (const VisWin *) (Dv + b_win), a.K = C.K, a.L = C.L, a.F = C.F;
    a.rho = h->D.rho, a.lm_ref = h->lm_ref, a.lm_ref_next = h->lm_ref_alt, a.f_meta_s = h->D.f_meta_s, a.lm_off = h->D.lm_off, a.lm_perm = h->D.lm_perm;
    a.lm_ref_node = (const int *) (h->cull_d + h->cull_res_ref), a.obs_off = (const int *) (h->cull_d + h->cull_res_off);
    a.lm_outlier = h->cull_d + h->cull_res_lmo, a.obs_outlier = h->cull_d + h->cull_res_obso, a.obs_factor = (const int *) (Dv + b_ofac);
    a.counts = (int *) (Dv + b_cnt), a.lm_src = (int *) (Dv + b_lms), a.lm_org = (int *) (Dv + b_org), a.lm_nan = Dv + b_nan, a.f_lm = (int *) (Dv + b_flm), a.f_ref = (int *) (Dv + b_fref);
    a.f_obs = (int *) (Dv + b_fobs), a.f_src = (int *) (Dv + b_fsrc), a.invdepth = (double *) (Dv + b_invd), a.f_new = (double *) (Dv + b_fnew);
    a.scratch = (int *) (Dv + b_scr);
    ICG_CUDA(cudaMemsetAsync(Dv + b_cnt, 0, 4 * VIS_COUNTS * (size_t) n, s));
    ICG_CUDA(launch_vision(a, n, s));
    count_launch();
    ICG_CUDA(cudaMemcpyAsync(H + b_cnt, Dv + b_cnt, out_end - b_cnt, cudaMemcpyDeviceToHost, s));
    ICG_CUDA(cudaStreamSynchronize(s));
    // the built windows: every check, then the slide of next with these vision rows
    static const char *what[] = {"", "obs_factor names no factor of the old window", "a device count is outside its list", "obs_src is out of range",
                                 "a node is out of range", "obs_lm is out of range", "two observations of one landmark in one node",
                                 "a reference frame id is not in the frame table", "a landmark whose reference row is unknown takes a new observation"};
    std::vector<icg_ba_problem> nx(next, next + n);
    std::vector<icg_ba_slide_window> cr(carry, carry + n);
    std::vector<std::unique_ptr<double[]>> fc_tmp(n);
    const int *cnt = (const int *) (H + b_cnt);
    for (int w = 0; w < n; w++) {
        const int *c = cnt + VIS_COUNTS * w;
        if (c[3] != 0) {
            set_error("%s: window %d: %s (entry %d)", fn, w, c[3] > 0 && c[3] <= VIS_EROW ? what[c[3]] : "?", c[4]);
            return ICG_EINVAL;
        }
        if (c[0] > C.L || c[1] > C.F) {
            set_error("%s: window %d: the next window has %d landmarks and %d factors, the handle holds %d / %d", fn, w, c[0], c[1], C.L, C.F);
            return ICG_EINVAL;
        }
    }
    for (int w = 0; w < n; w++) {
        const int *c = cnt + VIS_COUNTS * w;
        const VisWin &W = wins[w];
        icg_ba_slide_vision &v = vis[w];
        icg_ba_problem &p = nx[w];
        const int L = c[0], F = c[1];
        int *lm_src = (int *) (H + b_lms) + W.lm_out, *f_src = (int *) (H + b_fsrc) + W.f_out;
        p.L = L, p.F = F, p.invdepth = (double *) (H + b_invd) + W.lm_out, p.f_active = nullptr;
        p.f_lm = (int *) (H + b_flm) + W.f_out, p.f_ref = (int *) (H + b_fref) + W.f_out, p.f_obs = (int *) (H + b_fobs) + W.f_out;
        double *fc = v.f_const;
        if (!fc) fc_tmp[w].reset(new double[14 * (size_t) std::max(F, 1)]), fc = fc_tmp[w].get();
        const double *rows = (const double *) (H + b_fnew) + 14 * (size_t) W.nf_out;
        for (int f = 0, t = 0; f < F; f++)
            if (f_src[f] < 0) memcpy(fc + 14 * (size_t) f, rows + 14 * (size_t) t++, 112);
        p.f_const = fc;
        cr[w].lm_src = lm_src, cr[w].f_src = f_src;
        v.L = L, v.F = F, v.nan_dropped = c[5];
        if (v.lm_src) memcpy(v.lm_src, lm_src, 4 * (size_t) L);
        if (v.lm_origin) memcpy(v.lm_origin, (int *) (H + b_org) + W.lm_out, 4 * (size_t) L);
        if (v.nan_flags) memcpy(v.nan_flags, H + b_nan + W.lm_out, (size_t) W.oL + W.n_new);
        if (v.f_src) memcpy(v.f_src, f_src, 4 * (size_t) F);
        if (v.f_lm) memcpy(v.f_lm, p.f_lm, 4 * (size_t) F);
        if (v.f_ref) memcpy(v.f_ref, p.f_ref, 4 * (size_t) F);
        if (v.f_obs) memcpy(v.f_obs, p.f_obs, 4 * (size_t) F);
        if (v.invdepth) memcpy(v.invdepth, p.invdepth, 8 * (size_t) L);
    }
    return slide_body(h, n, nx.data(), cr.data(), integ, noise5, station3, fn, false, true);
}

int icg_ba_shard_slide_resident(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry) {
    const char *fn = "icg_ba_shard_slide_resident";
    const int rc = shard_group_only(h, fn, "icg_ba_slide_resident");
    return rc != ICG_OK ? rc : slide_body(h, n, next, carry, nullptr, nullptr, nullptr, fn, true);
}

int icg_ba_shard_slide_integrate_resident(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry,
                                          const icg_ba_slide_integrate *integ, const double *noise5, const double *station3) {
    const char *fn = "icg_ba_shard_slide_integrate_resident";
    int rc = shard_group_only(h, fn, "icg_ba_slide_integrate_resident");
    if (rc != ICG_OK) return rc;
    if (!integ) {  // still a collective call: the rank joins the agreement with its rejection
        set_error("%s: bad arguments", fn);
        shard_agree(h, true, 0, fn);
        return ICG_EINVAL;
    }
    return slide_body(h, n, next, carry, integ, noise5, station3, fn, true);
}

// ---- landmark shards over peer memory (transport "p2p")
struct ShardBlob {  // what a rank publishes to the others (ICG_SHARD_BLOB_BYTES)
    uint64_t magic, pid, ptr, doubles;  // doubles: the part of the exchange buffer every rank lays out alike (the export region is per rank)
    int32_t rank, world, device, pad;
    cudaIpcMemHandle_t ipc;
};
static_assert(sizeof(ShardBlob) <= ICG_SHARD_BLOB_BYTES, "ShardBlob size");

int icg_ba_shard_export(icg_ba *h, int rank, int world, uint8_t *blob) {
    if (!h || !blob) {
        set_error("icg_ba_shard_export: bad arguments");
        return ICG_EINVAL;
    }
    int rc = split_setup(h, rank, world);
    if (rc != ICG_OK) return rc;
    ShardBlob b;
    memset(&b, 0, sizeof(b));
    b.magic = 0x49434753484152ull, b.pid = (uint64_t) getpid(), b.ptr = (uint64_t) (uintptr_t) h->xbuf, b.doubles = h->D.S.off_exp;
    b.rank = rank, b.world = world, b.device = h->device;
    if (world > 1) ICG_CUDA(cudaIpcGetMemHandle(&b.ipc, h->xbuf));
    memset(blob, 0, ICG_SHARD_BLOB_BYTES);
    memcpy(blob, &b, sizeof(b));
    return ICG_OK;
}

int icg_ba_shard_connect(icg_ba *h, const uint8_t *blobs) {
    if (!h || !blobs || !h->D.S.split) {
        set_error("icg_ba_shard_connect: call icg_ba_shard_export first");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    const int world = h->D.world, rank = h->D.rank;
    for (int r = 0; r < world; r++) {
        ShardBlob b;
        memcpy(&b, blobs + (size_t) r * ICG_SHARD_BLOB_BYTES, sizeof(b));
        if (b.magic != 0x49434753484152ull || b.rank != r || b.world != world || b.doubles != h->D.S.off_exp) {
            set_error("icg_ba_shard_connect: blob %d does not describe rank %d of %d with the same window capacity", r, r, world);
            return ICG_EINVAL;
        }
        if (r == rank) continue;
        if (b.pid == (uint64_t) getpid()) {  // same process (several handles driven by one host process): plain device pointers
            if (b.device != h->device) {
                int can = 0;
                ICG_CUDA(cudaDeviceCanAccessPeer(&can, h->device, b.device));
                if (!can) {
                    set_error("icg_ba_shard_connect: device %d cannot access device %d", h->device, b.device);
                    return ICG_EUNSUPPORTED;
                }
                cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) ICG_CUDA(e);
                cudaGetLastError();
            }
            h->D.S.peer[r] = (double *) (uintptr_t) b.ptr;
        } else {  // one process per GPU: map the peer's buffer through CUDA IPC (NVLink peer memory)
            void *p = nullptr;
            ICG_CUDA(cudaIpcOpenMemHandle(&p, b.ipc, cudaIpcMemLazyEnablePeerAccess));
            h->ipc_opened[r] = p;
            h->D.S.peer[r] = (double *) p;
        }
    }
    return ICG_OK;
}

// Leave the peer-memory shard group: the exchange buffers and the peers' mappings are released and the handle returns to the pipeline
// its window size selects, on this GPU alone -- the fused single-GPU pipeline, or the split pipeline for systems that do not fit one CTA.
int icg_ba_shard_leave(icg_ba *h) {
    if (!h) {
        set_error("icg_ba_shard_leave: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    if (h->use_global_S) {
        if (h->x_world > 1) {
            const int rc = split_setup(h, 0, 1);
            if (rc != ICG_OK) return rc;
        }
    } else {
        split_release(h);
    }
    h->D.rank = 0, h->D.world = 1;
    return ICG_OK;
}

int icg_ba_shard_error(icg_ba *h) {
    if (!h || !h->D.S.split) return 0;
    int e = 0;
    cudaSetDevice(h->device);
    if (cudaMemcpy(&e, h->D.S.err, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return e;
}

int icg_ba_sync(icg_ba *h) {
    if (!h) return ICG_EINVAL;
    ICG_CUDA(cudaSetDevice(h->device));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    prof_collect(h);
    return ICG_OK;
}

int icg_ba_residual_costs(icg_ba *h, const icg_ba_problem *problem, double *reproj_cost, double *gnss_cost) {
    if (!h || !problem) {
        set_error("icg_ba_residual_costs: bad arguments");
        return ICG_EINVAL;
    }
    int rc = icg_ba_upload(h, 1, problem);
    if (rc != ICG_OK) return rc;
    const int F = problem->F, G = problem->n_gnss;
    double *d_out;
    ICG_CUDA(cudaMalloc(&d_out, sizeof(double) * (size_t) (F + G + 1)));
    const int nthreads = std::max(F, G);
    if (nthreads > 0) {
        ba_residual_costs_kernel<<<(nthreads + 127) / 128, 128, 0, h->stream>>>(h->C, h->D, d_out, d_out + F);
        count_launch();
    }
    std::vector<double> host(F + G + 1);
    ICG_CUDA(cudaMemcpyAsync(host.data(), d_out, sizeof(double) * (size_t) (F + G), cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    cudaFree(d_out);
    if (reproj_cost) memcpy(reproj_cost, host.data(), sizeof(double) * F);
    if (gnss_cost) memcpy(gnss_cost, host.data() + F, sizeof(double) * G);
    return ICG_OK;
}

int icg_ba_reproj_evaluate(icg_ba *h, const double *pose0, const double *pose1, const double *ext, const double *invdepth, const double *td,
                           const double *c14, double std_, double *residuals, double **jacobians) {
    if (!h || !pose0 || !pose1 || !ext || !invdepth || !td || !c14 || !residuals) {
        set_error("icg_ba_reproj_evaluate: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    double *in = h->scratch.h;
    memcpy(in, pose0, 56), memcpy(in + 7, pose1, 56), memcpy(in + 14, ext, 56);
    in[21] = 0, in[22] = *invdepth, in[23] = *td;
    memcpy(in + 24, c14, 112);
    in[38] = std_;
    ICG_CUDA(cudaMemcpyAsync(h->scratch.d, in, sizeof(double) * 40, cudaMemcpyHostToDevice, h->stream));
    ba_reproj_eval_kernel<<<1, 1, 0, h->stream>>>(h->scratch.d, h->scratch.d + 64);
    count_launch();
    ICG_CUDA(cudaMemcpyAsync(h->scratch.h + 64, h->scratch.d + 64, sizeof(double) * 48, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    const double *o = h->scratch.h + 64;
    residuals[0] = o[0], residuals[1] = o[1];
    if (jacobians) {
        for (int b = 0; b < 3; b++)
            if (jacobians[b]) memcpy(jacobians[b], o + 2 + 14 * b, sizeof(double) * 14);
        if (jacobians[3]) jacobians[3][0] = o[44], jacobians[3][1] = o[45];
        if (jacobians[4]) jacobians[4][0] = o[46], jacobians[4][1] = o[47];
    }
    return ICG_OK;
}

int icg_ba_imu_evaluate(icg_ba *h, const double *blob, const double *pose0, const double *mix0, const double *pose1, const double *mix1,
                        double *residuals, double **jacobians) {
    if (!h || !blob || !pose0 || !mix0 || !pose1 || !mix1 || !residuals) {
        set_error("icg_ba_imu_evaluate: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    double *in = h->scratch.h;
    memcpy(in, pose0, 56), memcpy(in + 7, mix0, 72), memcpy(in + 16, pose1, 56), memcpy(in + 23, mix1, 72);
    if (!host_imu_sqrt_info(blob + 252, in + 32)) {
        set_error("icg_ba_imu_evaluate: covariance is not positive definite");
        return ICG_EINVAL;
    }
    double *d_blob;
    ICG_CUDA(cudaMalloc(&d_blob, sizeof(double) * (ICG_IMU_BLOB_DOUBLES + 480)));
    ICG_CUDA(cudaMemcpyAsync(d_blob, blob, sizeof(double) * ICG_IMU_BLOB_DOUBLES, cudaMemcpyHostToDevice, h->stream));
    ICG_CUDA(cudaMemcpyAsync(h->scratch.d, in, sizeof(double) * (32 + 225), cudaMemcpyHostToDevice, h->stream));
    ba_imu_eval_kernel<<<1, 32, 0, h->stream>>>(d_blob, h->scratch.d + 32, h->scratch.d, d_blob + ICG_IMU_BLOB_DOUBLES);
    count_launch();
    std::vector<double> out(465);
    ICG_CUDA(cudaMemcpyAsync(out.data(), d_blob + ICG_IMU_BLOB_DOUBLES, sizeof(double) * 465, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    cudaFree(d_blob);
    memcpy(residuals, out.data(), sizeof(double) * 15);
    if (jacobians) {
        // local 15x30 [pose0 6 | mix0 9 | pose1 6 | mix1 9] -> global row-major 15x7, 15x9, 15x7, 15x9
        const double *J = out.data() + 15;
        const int c0[4] = {0, 6, 15, 21}, ls[4] = {6, 9, 6, 9}, gs[4] = {7, 9, 7, 9};
        for (int b = 0; b < 4; b++) {
            if (!jacobians[b]) continue;
            for (int r = 0; r < 15; r++)
                for (int c = 0; c < gs[b]; c++) jacobians[b][r * gs[b] + c] = c < ls[b] ? J[r * 30 + c0[b] + c] : 0.0;
        }
    }
    return ICG_OK;
}

// host helper of the small single-factor seams: upload `nin` doubles, run, download `nout` doubles (through the handle's scratch buffers)
static int small_factor_eval(icg_ba *h, int kind, const double *in, int nin, double *out, int nout) {
    ICG_CUDA(cudaSetDevice(h->device));
    memcpy(h->scratch.h, in, sizeof(double) * nin);
    ICG_CUDA(cudaMemcpyAsync(h->scratch.d, h->scratch.h, sizeof(double) * nin, cudaMemcpyHostToDevice, h->stream));
    ba_small_factor_eval_kernel<<<1, 1, 0, h->stream>>>(kind, h->scratch.d, h->scratch.d + 128);
    count_launch();
    ICG_CUDA(cudaMemcpyAsync(h->scratch.h + 128, h->scratch.d + 128, sizeof(double) * nout, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    memcpy(out, h->scratch.h + 128, sizeof(double) * nout);
    return ICG_OK;
}

int icg_ba_gnss_evaluate(icg_ba *h, const double *pose, const double *blh, const double *std3, const double *lever, double *residuals, double **jacobians) {
    if (!h || !pose || !blh || !std3 || !lever || !residuals) {
        set_error("icg_ba_gnss_evaluate: bad arguments");
        return ICG_EINVAL;
    }
    double in[16], out[21];
    memcpy(in, pose, 56), memcpy(in + 7, blh, 24), memcpy(in + 10, std3, 24), memcpy(in + 13, lever, 24);
    int rc = small_factor_eval(h, 0, in, 16, out, 21);
    if (rc != ICG_OK) return rc;
    memcpy(residuals, out, 24);
    if (jacobians && jacobians[0])  // global 3x7 row-major; the quaternion-w column is zero (gnss_factor.h:60-68)
        for (int r = 0; r < 3; r++)
            for (int c = 0; c < 7; c++) jacobians[0][r * 7 + c] = c < 6 ? out[3 + r * 6 + c] : 0.0;
    return ICG_OK;
}

int icg_ba_pose_prior_evaluate(icg_ba *h, const double *pose, const double *prior7, const double *std6, double *residuals, double **jacobians) {
    if (!h || !pose || !prior7 || !std6 || !residuals) {
        set_error("icg_ba_pose_prior_evaluate: bad arguments");
        return ICG_EINVAL;
    }
    double in[20], out[42];
    memcpy(in, pose, 56), memcpy(in + 7, prior7, 56);
    for (int k = 0; k < 6; k++) in[14 + k] = 1.0 / std6[k];
    int rc = small_factor_eval(h, 1, in, 20, out, 42);
    if (rc != ICG_OK) return rc;
    memcpy(residuals, out, 48);
    if (jacobians && jacobians[0])
        for (int r = 0; r < 6; r++)
            for (int c = 0; c < 7; c++) jacobians[0][r * 7 + c] = c < 6 ? out[6 + r * 6 + c] : 0.0;
    return ICG_OK;
}

int icg_ba_mix_prior_evaluate(icg_ba *h, const double *mix, const double *prior9, const double *std9, double *residuals, double **jacobians) {
    if (!h || !mix || !prior9 || !std9 || !residuals) {
        set_error("icg_ba_mix_prior_evaluate: bad arguments");
        return ICG_EINVAL;
    }
    double in[27], out[18];
    memcpy(in, mix, 72), memcpy(in + 9, prior9, 72), memcpy(in + 18, std9, 72);
    int rc = small_factor_eval(h, 2, in, 27, out, 18);
    if (rc != ICG_OK) return rc;
    memcpy(residuals, out, 72);
    if (jacobians && jacobians[0]) {
        memset(jacobians[0], 0, sizeof(double) * 81);
        for (int k = 0; k < 9; k++) jacobians[0][k * 9 + k] = out[9 + k];
    }
    return ICG_OK;
}

int icg_ba_imu_error_evaluate(icg_ba *h, const double *mix, double *residuals, double **jacobians) {
    if (!h || !mix || !residuals) {
        set_error("icg_ba_imu_error_evaluate: bad arguments");
        return ICG_EINVAL;
    }
    double out[12];
    int rc = small_factor_eval(h, 3, mix, 9, out, 12);
    if (rc != ICG_OK) return rc;
    memcpy(residuals, out, 48);
    if (jacobians && jacobians[0]) {  // 6x9: rows 0..2 on bg (columns 3..5), rows 3..5 on ba (columns 6..8)
        memset(jacobians[0], 0, sizeof(double) * 54);
        for (int k = 0; k < 3; k++) jacobians[0][k * 9 + 3 + k] = out[6 + k], jacobians[0][(3 + k) * 9 + 6 + k] = out[9 + k];
    }
    return ICG_OK;
}

int icg_ba_marg_factor_evaluate(icg_ba *h, int r, int nblocks, const int32_t *block_type, const double *const *parameters, const double *x0,
                                const double *J0, const double *e0, double *residuals, double **jacobians) {
    if (!h || r < 1 || nblocks < 1 || !block_type || !parameters || !x0 || !J0 || !e0 || !residuals) {
        set_error("icg_ba_marg_factor_evaluate: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    int tot = 0, cols = 0;
    for (int b = 0; b < nblocks; b++) {
        const int t = block_type[b];
        if (t < 0 || t > 3 || !parameters[b]) {
            set_error("icg_ba_marg_factor_evaluate: block %d invalid", b);
            return ICG_EINVAL;
        }
        tot += t == 1 ? 9 : t == 3 ? 1 : 7, cols += t == 1 ? 9 : t == 3 ? 1 : 6;
    }
    if (cols != r) {
        set_error("icg_ba_marg_factor_evaluate: the blocks give %d local columns, r = %d", cols, r);
        return ICG_EINVAL;
    }
    const size_t nin = 2 + (size_t) nblocks + 2 * (size_t) tot + r + (size_t) r * r;
    std::vector<double> in(nin);
    in[0] = r, in[1] = nblocks;
    for (int b = 0; b < nblocks; b++) in[2 + b] = block_type[b];
    double *px = in.data() + 2 + nblocks;
    int xo = 0;
    for (int b = 0; b < nblocks; b++) {
        const int g = block_type[b] == 1 ? 9 : block_type[b] == 3 ? 1 : 7;
        memcpy(px + xo, parameters[b], sizeof(double) * g);
        xo += g;
    }
    memcpy(px + tot, x0, sizeof(double) * tot);
    memcpy(px + 2 * tot, e0, sizeof(double) * r);
    memcpy(px + 2 * tot + r, J0, sizeof(double) * (size_t) r * r);
    double *d = nullptr;
    ICG_CUDA(cudaMalloc(&d, sizeof(double) * (nin + r)));
    ICG_CUDA(cudaMemcpyAsync(d, in.data(), sizeof(double) * nin, cudaMemcpyHostToDevice, h->stream));
    ba_marg_factor_eval_kernel<<<1, 256, sizeof(double) * r, h->stream>>>(d, d + nin);
    count_launch();
    ICG_CUDA(cudaMemcpyAsync(residuals, d + nin, sizeof(double) * r, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    cudaFree(d);
    if (jacobians) {  // the factor is linear: d e / d (block b) = J0[:, columns of b], quaternion-w column zero (marginalization_factor.h:84-97)
        int col = 0;
        for (int b = 0; b < nblocks; b++) {
            const int t = block_type[b], g = t == 1 ? 9 : t == 3 ? 1 : 7, l = t == 1 ? 9 : t == 3 ? 1 : 6;
            if (jacobians[b])
                for (int i = 0; i < r; i++)
                    for (int c = 0; c < g; c++) jacobians[b][(size_t) i * g + c] = c < l ? J0[(size_t) i * r + col + c] : 0.0;
            col += l;
        }
    }
    return ICG_OK;
}

}  // extern "C"
