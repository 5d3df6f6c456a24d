// ba_dev.cuh -- what the host side of the window solve (ba_handle.cu, ba_keyframe.cu) shares with its kernels (ba.cu, ba_split.cuh,
// ba_marg.cuh): the device view of a handle, the launch constants and shared-memory sizes the host reads, and the kernels it launches.
#pragma once
#include "ba_math.cuh"
#include "ba_slide.cuh"
#include "common.cuh"

namespace icg {

constexpr int BA_SPLIT_W = 4;   // row splits of the Schur SYRK = CTAs of its cluster (partials summed in fixed order -> deterministic)
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
    // LmState::lin_buf through the lin_* helpers of ba.cu.  The single-GPU pipeline linearises the candidate into the copy the window is not
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

constexpr int LV_LD = 45;  // shared-memory record row: 44 doubles padded to an odd length (conflict-free)
constexpr size_t LV_SMEM = sizeof(double) * (128 * LV_LD + (BA_MAX_NODES + 1) * bam::NODE_FRAME_LD);  // records + node frames (49.5 KB: dynamic, opted in at create)
constexpr int SCHUR_RCH = 80;  // landmark rows staged per chunk (multiple of 4)
constexpr int SCHUR_PASS = 16;  // super-tiles per pass
constexpr int CAM_THREADS = 320;  // 10 warps: the K - 1 = 9 IMU factors of a 10-node window are evaluated in one round (warp per factor)
constexpr int SOLVE_THREADS = 256;  // 2 CTAs (windows) per SM: 107 KB shared memory and <= 128 registers each

// ---- split pipeline (ba_split.cuh)
constexpr int SPLIT_CLUSTER = 4;      // CTAs per window in ba_solve_cam
constexpr int SPLIT_HDR = 16;         // header doubles of the step broadcast
constexpr int SPLIT_SCAL = 8;         // doubles per (window, rank) slot of the scalar exchange
constexpr int SPLIT_BS_ROWS = 32;     // rows per block of the blocked back-substitution
constexpr int STEP_SLICES = 4;        // CTAs (landmark slices) per window of ba_step_lm
constexpr int MEXP_ROW = 16;  // [landmark | f_ref, f_obs, active (int64 bits)] | inverse depth | f_const[14]
enum { XF_SUM = 0, XF_EXPORT = 1, XF_DONE = 2 };

__host__ __device__ inline size_t split_S_stride(const BaCaps &C) { return (size_t) (C.N + 1) * (C.N + 2) / 2 + (size_t) C.NS; }

constexpr int DSM_CL = 4;
static_assert(SOLVE_THREADS == 256 && DSM_CL == SPLIT_CLUSTER, "ba_solve_cam_dsm: warp r assembles row r of a tile row; one launch geometry for both forms");
__host__ __device__ constexpr int dsm_ntiles(int NR) { return (NR + 7) / 8; }
__host__ inline size_t dsm_smem_doubles(const BaCaps &C) {
    const int nt = dsm_ntiles(C.N + 1);
    int mx = 0;
    for (int cr = 0; cr < DSM_CL; cr++) {
        int s = 0;
        for (int T = cr; T < nt; T += DSM_CL) s += T;
        mx = s > mx ? s : mx;
    }
    return 40 + 8 * (size_t) nt * 8 + 64 + 8 + 8 * DSM_CL + 8 + 8 + (size_t) nt * 64 * 3 + (size_t) mx * 64;
}

// ---- marginalization (ba_marg.cuh)
constexpr int MARG_THREADS = 512;
constexpr int MARG_MAP_HDR = 8;    // [m, r, n0, num_marg, ext_col, td_col, -, -] then pose_col[K], mix_col[K], lm_col[L]

struct MargDev {
    int *map;        // [NW][MARG_MAP_HDR + 2*K + L]
    int map_stride;
    double *H0, *b0; // [NW][n0cap^2], [NW][n0cap]
    double *G1, *V1; // [NW][mcap^2] each: Jacobi workspace of Hmm
    double *G2, *V2; // [NW][rcap^2] each: Jacobi workspace of Hp
    double *lam1, *lam2;  // eigenvalues
    double *Z;       // [NW][mcap * (rcap + 1)]
    double *Hp, *bp; // [NW][rcap^2], [NW][rcap]
    double *J0, *e0; // outputs
    int *flags;      // [NW][4] saved dims flags
    int n0cap, mcap, rcap;
};

// marg_select_built (icg_ba_marginalize_built): the factor set and the column map from the built culling, on the device.  MargSelWin: one
// window as the host stages it (the built lists' slices, num_marg, node_in_map and the camera side's touched blocks); out: per window
// MARG_SEL_HDR + 2 max_K ints [m, r, nblocks, invalid observations, -, -, -, -] then the remained blocks, type | node << 2 each
constexpr int MARG_SEL_HDR = 8;
constexpr int MARG_SEL_THREADS = 256;
struct MargSelWin {
    int lm0, off0, obs0, num_marg;  // CullWin's slices of the built lists and the culling's flags
    int ext, td;                    // the previous prior's block table names ext / td
    uint8_t tp[BA_MAX_NODES], tm[BA_MAX_NODES];  // pose / mix blocks the camera-side factors touch
    uint8_t in_map[BA_MAX_NODES];                // node_in_map
};
struct MargSelArgs {
    const MargSelWin *win;
    const int *ref, *off, *node, *fac;  // the built lists (CullSrc)
    const uint8_t *lm_outlier, *obs_outlier;
    uint8_t *fmask;  // [NW][F] the factor set, by factor id
    int *ftab;       // [NW][F] scratch: landmark * BA_MAX_NODES + observing node, by factor id
    int *out;        // [n][MARG_SEL_HDR + 2 K]
};

constexpr int MARG_PAIR_MAXN = 160;  // 160^2 doubles = 204.8 KB per CTA
constexpr int MARG_CTA_MAXN = 118;     // 2 * 118^2 doubles = 222.8 KB
constexpr int MARG_CTA_THREADS = 512;  // 64 pair slots >= MARG_CTA_MAXN / 2
constexpr int MARG_CLUSTER_MAXN = 320;
constexpr int MARG_CLUSTER_CTAS = 8;                       // portable maximum cluster size
constexpr int MARG_CLUSTER_THREADS = 640;                  // 160 four-lane groups: one per pair of a step at n = 320
constexpr int MARG_CLUSTER_SLOT = 3 * (MARG_CLUSTER_MAXN / 2);  // (al, be, ga) per pair
__host__ __device__ constexpr int marg_cluster_rows(int n) { return (n + MARG_CLUSTER_CTAS - 1) / MARG_CLUSTER_CTAS; }
__host__ __device__ constexpr size_t marg_cluster_smem(int n) {
    return sizeof(double) * (2 * (size_t) marg_cluster_rows(n) * n + 2 * (size_t) MARG_CLUSTER_SLOT);
}

// ---- the kernels the host launches (defined in ba.cu, ba_split.cuh and ba_marg.cuh, with their launch bounds)
__global__ void ba_lin_vis(BaCaps C, BaDev D, int at_cand);
__global__ void ba_schur_dmma(BaCaps C, BaDev D, int ld);
__global__ void ba_lin_cam(BaCaps C, BaDev D, int at_cand);
__global__ void ba_solve(BaCaps C, BaDev D);
__global__ void ba_cost_cam(BaCaps C, BaDev D, int nblk_vis);
__global__ void ba_cost(BaCaps C, BaDev D, int nblk_vis);
__global__ void ba_accept(BaCaps C, BaDev D);
__global__ void ba_reset_state(BaDev D, LmState *save, int n, int max_iter);
__global__ void ba_chi2_cull(BaCaps C, BaDev D, int *counters);
__global__ void ba_set_gnss_huber(BaDev D, int n, int v);
__global__ void ba_residual_costs_kernel(BaCaps C, BaDev D, double *reproj_cost, double *gnss_cost);
__global__ void ba_reproj_eval_kernel(const double *in, double *out, int frames);
__global__ void ba_imu_eval_kernel(const double *blob, const double *U, const double *x, double *out);
__global__ void ba_small_factor_eval_kernel(int kind, const double *in, double *out);
__global__ void ba_marg_factor_eval_kernel(const double *in, double *out);
__global__ void ba_lm_ref_fill(const WinDims *dims, const SlideWin *win, const int *map, const double *old, const double *fc, const int *lm_off,
                               const int *lm_perm, double *out, int Lc, int Fc);

__global__ void ba_signal(BaDev D, unsigned long long epoch);
__global__ void ba_reduce(BaCaps C, BaDev D, unsigned long long epoch);
__global__ void ba_solve_cam(BaCaps C, BaDev D, unsigned long long epoch);
__global__ void ba_solve_cam_dsm(BaCaps C, BaDev D, unsigned long long epoch);
__global__ void ba_step_lm(BaCaps C, BaDev D, unsigned long long epoch);
__global__ void ba_exchange(BaCaps C, BaDev D, int n, int nblk_vis, unsigned long long epoch);
__global__ void ba_accept_split(BaCaps C, BaDev D, unsigned long long epoch);
__global__ void ba_xflag(BaDev D, int kind, unsigned long long epoch);
__global__ void ba_xsum(BaCaps C, BaDev D, int *v, int stride, int n, int nv, int op, int par, unsigned long long epoch);
__global__ void ba_marg_export(BaCaps C, BaDev D, const int *sel, const int *sel_off, const uint8_t *fmask, unsigned long long prev);
__global__ void ba_marg_heads(BaCaps C, BaDev D, int n_own, long long *heads, unsigned long long epoch);
__global__ void ba_marg_gather(BaCaps C, BaDev D, const long long *heads, const int *dst_row, double *dst);
__global__ void ba_marg_fill(BaCaps Cm, BaDev Dm, BaCaps C, BaDev D, const double *rows, const int *row0, const int *fidx);

__global__ void marg_prepare(BaDev D, MargDev M, int n, int restore);
__global__ void marg_select_built(BaCaps C, BaDev D, MargDev M, MargSelArgs a);
__global__ void marg_assemble(BaCaps C, BaDev D, MargDev M);
__global__ void marg_jacobi(MargDev M, int which);
__global__ void marg_jacobi_pair(MargDev M, int which);
__global__ void marg_jacobi_cta(MargDev M, int which);
__global__ void marg_jacobi_cluster(MargDev M, int which);
__global__ void marg_schur(MargDev M);
__global__ void marg_finish(MargDev M);

}  // namespace icg
