// ba_lm.cuh -- the trust-region policy of the window solve, stated once for both device pipelines: the single-GPU one (ba_schur_dmma,
// ba_solve, ba_accept in ba.cu) and the split one (ba_solve_cam / ba_solve_cam_dsm, ba_step_lm, ba_accept_split in ba_split.cuh).  The policy
// is Ceres' TrustRegionMinimizer (trust_region_minimizer.cc) with the LevenbergMarquardtStrategy (levenberg_marquardt_strategy.cc), at the
// options the reference leaves at their defaults.  Included by ba.cu; the decisions live in the per-window LmState.
#pragma once

namespace icg {

// LevenbergMarquardtStrategy::ComputeStep: the LM diagonal D^2 of a column whose Jacobi-scaled Hessian diagonal is hs, clamped to
// [min_lm_diagonal, max_lm_diagonal] = [1e-6, 1e32], over the trust-region radius
__device__ __forceinline__ double lm_d2(double hs, double radius) { return fmin(fmax(hs, 1e-6), 1e32) / radius; }

// TrustRegionMinimizer::FinalizeIterationAndCheckIfMinimizerCanContinue: 0 continues, 1 is NO_CONVERGENCE (max_num_iterations reached),
// 2 is convergence after a successful step (gradient_tolerance on max |g|, min_trust_region_radius).  radius is a reference so that a caller
// may pass the LmState field: it is then read only where the chain reaches it.
__device__ __forceinline__ int lm_term(int iter, int max_iter, int last_success, double gmax, const double &radius) {
    int term = 0;
    if (iter >= max_iter) term = 1;
    else if (last_success && gmax <= 1e-10) term = 2;
    else if (last_success && radius <= 1e-32) term = 2;
    return term;
}

// The commit at the start of an iteration: the cost and max |g| at x, the initial cost (the cost at x of the first iteration), the
// linearisation at x consumed, then the termination or the next iteration.  Every rank of a shard group commits the same values (the owner
// from its solve, the others from its step header), so their LM states stay identical.  ba_solve commits the same fields in stages.
__device__ __forceinline__ void lm_begin(LmState &st, double x_cost, double gmax, double initial_cost, int term) {
    st.x_cost = x_cost, st.gmax = gmax, st.initial_cost = initial_cost;
    st.fresh_lin = 0, st.first = 0, st.need_lin = 0;
    if (term) st.done = term, st.step_valid = 0;
    else st.iter = st.iter + 1;
}

// The step decision, from the step's model cost change mcc, |x - x_cand|^2 (sn), its count of non-finite entries (nfin), |x|^2 (x_sq) and the
// cost at the candidate (cand):
//  - HandleInvalidStep + LevenbergMarquardtStrategy::StepIsInvalid: a failed factorisation, a non-finite step or mcc <= 0 halves the radius;
//    the fifth in a row is FAILURE;
//  - ParameterToleranceReached / FunctionToleranceReached: convergence;
//  - LevenbergMarquardtStrategy::StepAccepted (relative decrease > 1e-3): the radius grows, x needs a fresh cost and gradient;
//  - StepRejected: the radius shrinks, the linearisation at x is kept.
// Returns whether the step is accepted: the caller then copies the candidate into x and says where the linearisation at the new x comes from.
__device__ __forceinline__ bool lm_decide(LmState &st, double mcc, double sn, double nfin, double x_sq, double cand) {
    if (!st.chol_ok || nfin != 0.0 || !(mcc > 0.0)) {
        st.step_valid = 0;
        st.n_invalid++;
        if (st.n_invalid >= 5) st.done = 3;  // FAILURE
        st.radius *= 0.5;
        st.last_success = 0;
        return false;
    }
    st.n_invalid = 0;
    st.model_cost_change = mcc;
    st.step_norm = sqrt(sn);
    st.x_norm = sqrt(x_sq);
    st.cand_cost = cand;
    if (st.step_norm <= 1e-8 * (st.x_norm + 1e-8)) {
        st.done = 2;
    } else if (fabs(st.x_cost - cand) <= 1e-6 * st.x_cost) {
        st.done = 2;
    } else {
        const double rel = (st.x_cost - cand) / mcc;
        if (rel > 1e-3) {
            st.n_success++;
            const double t = 2.0 * rel - 1.0;
            st.radius = fmin(1e16, st.radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
            st.decrease_factor = 2.0;
            st.last_success = 1;
            st.fresh_lin = 1;
            return true;
        }
        st.radius = st.radius / st.decrease_factor;
        st.decrease_factor *= 2.0;
        st.last_success = 0;
        st.need_lin = 0;
    }
    return false;
}

// |x|^2 of window w's camera-side blocks (a constant extrinsic or td left out), summed over the 128 threads of an accept kernel
__device__ __forceinline__ double lm_cam_sq(const BaCaps &C, const BaDev &D, int w, const WinDims &dm, double *s_red) {
    const int tid = threadIdx.x;
    const double *pose = D.pose + (size_t) w * C.K * 7, *mix = D.mix + (size_t) w * C.K * 9, *ext = D.ext + (size_t) w * 8;
    double s = 0;
    for (int e = tid; e < dm.K * 7; e += 128) s += pose[e] * pose[e];
    for (int e = tid; e < dm.K * 9; e += 128) s += mix[e] * mix[e];
    if (tid < 7 && !dm.ext_const) s += ext[tid] * ext[tid];
    if (tid == 7 && !dm.td_const) s += ext[7] * ext[7];
    return block_sum(s, s_red);
}

// an accepted step: x <- x_cand, camera blocks and landmarks (128 threads)
__device__ __forceinline__ void lm_take_cand(const BaCaps &C, const BaDev &D, int w, const WinDims &dm) {
    const int tid = threadIdx.x;
    double *pose = D.pose + (size_t) w * C.K * 7, *mix = D.mix + (size_t) w * C.K * 9, *ext = D.ext + (size_t) w * 8, *rho = D.rho + (size_t) w * C.L;
    const double *pose_c = D.pose_c + (size_t) w * C.K * 7, *mix_c = D.mix_c + (size_t) w * C.K * 9, *ext_c = D.ext_c + (size_t) w * 8, *rho_c = D.rho_c + (size_t) w * C.L;
    for (int e = tid; e < dm.K * 7; e += 128) pose[e] = pose_c[e];
    for (int e = tid; e < dm.K * 9; e += 128) mix[e] = mix_c[e];
    if (tid < 8) ext[tid] = ext_c[tid];
    for (int e = tid; e < dm.L; e += 128) rho[e] = rho_c[e];
}

}  // namespace icg
