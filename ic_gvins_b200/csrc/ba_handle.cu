// ba_handle.cu -- host side of the window solve (ba.cu): the handle's lifecycle, the packing and upload of the windows, the LM sequences of the
// fused single-GPU pipeline and of the split pipeline (ba_split.cuh), the shard group's plumbing, and the single-factor evaluations.  The
// resident keyframe cycle that runs on the same handle is ba_keyframe.cu.
#include <unistd.h>

#include <string>
#include <thread>

#include "ba_handle.cuh"
#include "preint.cuh"

using namespace icg;

int dmalloc(icg_ba *h, double **p, size_t n) {
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

// ---- split pipeline: host side
// a buffer outgrown by a call: freed now on a single rank, kept until the group is left in a shard group (icg_ba::retired_d)
void retire(icg_ba *h, void *d, void *hp) {
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

cudaError_t launch_lm_ref_fill(icg_ba *h, int n, const SlideWin *win, const int *map, const double *old, double *out) {
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
int pack_windows(icg_ba *h, int n, const icg_ba_problem *P, bool values) {
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
int upload_structure(icg_ba *h, int n) {
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
int keep_pristine(icg_ba *h, int n) {
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

static int launch_solve_cam(icg_ba *h, int n, unsigned long long epoch) {
    const ClusterLaunch L((unsigned) (n * SPLIT_CLUSTER), SOLVE_THREADS, h->solve_cam_dsm ? h->smem_solve_cam_dsm : h->smem_solve_cam, h->stream,
                          SPLIT_CLUSTER);
    if (h->solve_cam_dsm) ICG_CUDA(cudaLaunchKernelEx(&L.cfg, ba_solve_cam_dsm, h->C, h->D, epoch));
    else ICG_CUDA(cudaLaunchKernelEx(&L.cfg, ba_solve_cam, h->C, h->D, epoch));
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

static void fill_summary(const LmState &st, icg_ba_summary &o) {
    o.iterations = st.iter, o.num_successful_steps = st.n_success;
    o.termination = st.done == 2 ? 1 : st.done == 3 ? 2 : 0;
    o.reserved = 0;
    o.initial_cost = st.initial_cost, o.final_cost = st.x_cost, o.final_radius = st.radius;
}

int shard_timed_out(icg_ba *h, const char *what) {
    if (icg_ba_shard_error(h) == 0) return ICG_OK;
    set_error("%s: a peer exchange of the shard group timed out (a rank did not make the same call)", what);
    return ICG_ECUDA;
}

// enqueue the group's integer exchange of v (device; see ba_xsum)
int shard_xsum(icg_ba *h, int *v, int stride, int n, int nv, int op) {
    const unsigned long long epoch = ++h->epoch;
    const int par = (int) (h->xs_calls++ & 1);
    ba_xsum<<<1, 256, 0, h->stream>>>(h->C, h->D, v, stride, n, nv, op, par, epoch);
    ICG_CHECK_LAUNCH();
    count_launch();
    return ICG_OK;
}

// the group's maxima of three host integers (fn: the calling entry point, for the timeout's message)
int shard_xmax(icg_ba *h, int *v3, const char *fn) {
    int rc = hd_reserve(h, h->xs_v, 8, fn);
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

// The agreement of a collective call before any rank writes its device: one exchange of (rejecting rank + 1, +fp, -fp).  ICG_OK when no rank
// rejected and every rank passed the same fingerprint fp; otherwise ICG_EINVAL on every rank (a rejecting rank keeps its own message).
int shard_agree(icg_ba *h, bool rejected, int fp, const char *fn) {
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

// ---- landmark shards over peer memory (transport "p2p")
struct ShardBlob {  // what a rank publishes to the others (ICG_SHARD_BLOB_BYTES)
    uint64_t magic, pid, ptr, doubles;  // doubles: the part of the exchange buffer every rank lays out alike (the export region is per rank)
    int32_t rank, world, device, pad;
    cudaIpcMemHandle_t ipc;
};
static_assert(sizeof(ShardBlob) <= ICG_SHARD_BLOB_BYTES, "ShardBlob size");

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

extern "C" {

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

void icg_ba_destroy(icg_ba *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    prof_collect(h);
    prof_print(h);
    for (cudaEvent_t e : h->prof_ev) cudaEventDestroy(e);
    split_release(h);
    if (h->mx_h) icg_ba_destroy(h->mx_h);
    if (h->mx_rows) cudaFree(h->mx_rows);
    for (double *p : {h->M.H0, h->M.b0, h->M.G1, h->M.V1, h->M.lam1, h->M.Z})
        if (p) cudaFree(p);
    if (h->slide_old) cudaFree(h->slide_old);
    for (double *p : {h->store_d[0], h->store_d[1], h->cut_rows})
        if (p) cudaFree(p);
    if (h->ins_ev) cudaEventDestroy(h->ins_ev);
    if (h->fc_alt) cudaFree(h->fc_alt);
    if (h->slide_ev) cudaEventDestroy(h->slide_ev);
    for (void *p : h->dev_only) cudaFree(p);
    if (h->stream_cam) cudaStreamSynchronize(h->stream_cam), cudaStreamDestroy(h->stream_cam);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->ev_join) cudaEventDestroy(h->ev_join);
    if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
    delete h;  // the HostDev members release themselves
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
    h->store_valid = false;  // the IMU factors are next's now, without samples
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
        if (summaries) fill_summary(h->st.h[w], summaries[w]);
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

static int reproj_evaluate(icg_ba *h, const char *name, int frames, const double *pose0, const double *pose1, const double *ext, const double *invdepth,
                           const double *td, const double *c14, double std_, double *residuals, double **jacobians) {
    if (!h || !pose0 || !pose1 || !ext || !invdepth || !td || !c14 || !residuals) {
        set_error("%s: bad arguments", name);
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    double *in = h->scratch.h;
    memcpy(in, pose0, 56), memcpy(in + 7, pose1, 56), memcpy(in + 14, ext, 56);
    in[21] = 0, in[22] = *invdepth, in[23] = *td;
    memcpy(in + 24, c14, 112);
    in[38] = std_;
    ICG_CUDA(cudaMemcpyAsync(h->scratch.d, in, sizeof(double) * 40, cudaMemcpyHostToDevice, h->stream));
    ba_reproj_eval_kernel<<<1, 1, 0, h->stream>>>(h->scratch.d, h->scratch.d + 64, frames);
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

int icg_ba_reproj_evaluate(icg_ba *h, const double *pose0, const double *pose1, const double *ext, const double *invdepth, const double *td,
                           const double *c14, double std_, double *residuals, double **jacobians) {
    return reproj_evaluate(h, "icg_ba_reproj_evaluate", 0, pose0, pose1, ext, invdepth, td, c14, std_, residuals, jacobians);
}

int icg_ba_reproj_evaluate_frames(icg_ba *h, const double *pose0, const double *pose1, const double *ext, const double *invdepth, const double *td,
                                  const double *c14, double std_, double *residuals, double **jacobians) {
    return reproj_evaluate(h, "icg_ba_reproj_evaluate_frames", 1, pose0, pose1, ext, invdepth, td, c14, std_, residuals, jacobians);
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
