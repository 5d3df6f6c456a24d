// klt.cu -- Path A: pyramid build + pyramidal Lucas-Kanade tracker for sm_90a.
//
// Replaces cv::calcOpticalFlowPyrLK as called from IG/tracking/tracking.cc:385,390,487,493 (OpenCV is an
// un-vendored dependency of the reference; the arithmetic restated here is specified in SURVEY.md Appendix A.1-A.3
// and pinned by oracle/klt_ref.c + tests/golden/klt_golden.npz).
//
// Design (GPU-first, not a translation of OpenCV's row-parallel CPU code):
//   * pyramids live in HBM as [slot][row][pitch] u8 planes per level; one 3-D TMA descriptor per level.
//   * one warp tracks one point through all levels (forward, then backward): the 21x21 template (I, Ix, Iy) lives in registers
//     (two 7-pixel horizontal runs per lane), the 48x32 search window of the second image is staged into shared memory by TMA
//     (cp.async.bulk.tensor.3d, mbarrier completion) and re-centred only when the track leaves it; the template comes from ONE exact
//     Q14 interpolation grid per level (interpolate first, differentiate second: no derivative image ever touches HBM); the bilinear
//     taps of a run are dp2a on packed bytes (aligned 32-bit shared-memory loads + funnel shifts, not byte loads); the 2x2 normal
//     equations are reduced with REDUX (exact integer sums, one rounding).
//   * compile with -fmad=false: the float sequence of the reference library must not be contracted.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "klt_handle.cuh"

namespace icg {

struct KltArgs {
    KltLevel lv[KLT_LEVELS];
    int n_total;
    int n_levels;  // maxLevel + 1
    int max_iter;
    int mode;      // 0 forward only, 1 forward+backward+gates
    int use_initial_flow;
    int check_final;  // level-0 epilogue status check (OpenCV does it only when err is requested)
    double eps2;
    double min_eig_thr;
    float img_w, img_h;  // level-0 size for the border gate
    const int32_t *slots;
    const float2 *prev_xy;
    const float2 *init_xy;
    float2 *fwd_xy;
    float2 *bwd_xy;
    uint8_t *status;
    float *err;
};

__device__ __forceinline__ int reflect101(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) p = p < 0 ? -p : 2 * (len - 1) - p;
    return p;
}

// ------------------------------------------------------------------------------------------------ pyrDown
// cv::pyrDown (SURVEY A.1): dst(y,x) = (sum_{i,j} k_i k_j src(2y+i, 2x+j) + 128) >> 8, k = [1 4 6 4 1], reflect-101.
// One thread per FOUR horizontally adjacent output pixels: a source row contributes the 11 bytes [8t-2, 8t+8], fetched as four aligned
// 32-bit words from 8t-4; the row filter of each output is one dp4a (weights 1 4 6 4 on a funnel-shifted 4-byte window) plus the fifth tap.
// HBM-bound in bytes (W*H in, W*H/4 out per level); the packed form keeps it off the issue limit.
__device__ __forceinline__ void pd_row4(const uint8_t *__restrict__ r, int t, int h[4]) {
    const unsigned *wp = (const unsigned *) (r + 8 * t - 4);  // 4-byte aligned: row starts are 16-byte aligned
    const unsigned w0 = wp[0], w1 = wp[1], w2 = wp[2], w3 = wp[3];
    const unsigned K = 0x04060401u;  // bytes (1, 4, 6, 4)
    h[0] = (int) __dp4a(__funnelshift_r(w0, w1, 16), K, w1 >> 16 & 0xFFu);  // columns 8t-2 .. 8t+1, + 8t+2
    h[1] = (int) __dp4a(w1, K, w2 & 0xFFu);                                 // 8t .. 8t+3, + 8t+4
    h[2] = (int) __dp4a(__funnelshift_r(w1, w2, 16), K, w2 >> 16 & 0xFFu);  // 8t+2 .. 8t+5, + 8t+6
    h[3] = (int) __dp4a(w2, K, w3 & 0xFFu);                                 // 8t+4 .. 8t+7, + 8t+8
}
__device__ __forceinline__ int pd_scalar(const uint8_t *__restrict__ src, int sW, int sH, int spitch, int x, int y) {
    const int kk[5] = {1, 4, 6, 4, 1};
    const int x0 = 2 * x - 2, y0 = 2 * y - 2;
    int s = 0;
    for (int j = 0; j < 5; j++) {
        const uint8_t *r = src + (size_t) reflect101(y0 + j, sH) * spitch;
        int rs = 0;
        for (int i = 0; i < 5; i++) rs += kk[i] * r[reflect101(x0 + i, sW)];
        s += kk[j] * rs;
    }
    return (s + 128) >> 8;
}
__global__ void __launch_bounds__(256) pyr_down_kernel(const uint8_t *__restrict__ src, int sW, int sH, int spitch, size_t s_slot,
                                                       uint8_t *__restrict__ dst, int dW, int dH, int dpitch, size_t d_slot,
                                                       int first_slot) {
    const int slot = first_slot + blockIdx.z;
    src += (size_t) slot * s_slot + (size_t) KLT_PAD * spitch + KLT_PAD;  // interiors of the padded planes
    dst += (size_t) slot * d_slot + (size_t) KLT_PAD * dpitch + KLT_PAD;
    const int t = blockIdx.x * 64 + (threadIdx.x & 63), y = blockIdx.y * 4 + (threadIdx.x >> 6);
    const int x = 4 * t;
    if (x >= dW || y >= dH) return;
    const int y0 = 2 * y - 2;
    uint8_t *drow = dst + (size_t) y * dpitch;
    // the source plane's reflect-101 padding is already filled (icg_klt_build_pyramids pads a level before it reduces it), and reflect-101 is
    // cv::pyrDown's border rule: border outputs take the packed path too, reading into the padding.  (With the scalar border path, every warp
    // that held an edge thread -- 2 of 5 at level 1, all of them at level 3 -- ran both paths and the kernel was issue-bound.)
    if (x + 3 < dW) {
        const uint8_t *r = src + (size_t) y0 * spitch;
        int h0[4], h1[4], h2[4], h3[4], h4[4];
        pd_row4(r, t, h0);
        pd_row4(r + spitch, t, h1);
        pd_row4(r + 2 * (size_t) spitch, t, h2);
        pd_row4(r + 3 * (size_t) spitch, t, h3);
        pd_row4(r + 4 * (size_t) spitch, t, h4);
        unsigned out = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int v = (h0[j] + 4 * h1[j] + 6 * h2[j] + 4 * h3[j] + h4[j] + 128) >> 8;
            out |= (unsigned) v << (8 * j);
        }
        *(unsigned *) (drow + x) = out;
    } else {
        for (int j = 0; j < 4; j++)
            if (x + j < dW) drow[x + j] = (uint8_t) pd_scalar(src, sW, sH, spitch, x + j, y);
    }
}

// Fill the reflect-101 padding of all levels of a range of slots (OpenCV pads its pyramid the same way, lkpyramid.cpp).
// One thread writes one aligned 16-byte chunk: whole rows for the PAD rows above / below, the two 48-byte side strips otherwise.
struct PadArgs {
    uint8_t *base[KLT_LEVELS];
    int W[KLT_LEVELS], H[KLT_LEVELS], pitch[KLT_LEVELS];
    size_t slot_stride[KLT_LEVELS];
    int off[KLT_LEVELS + 1];  // prefix sums of the per-level chunk counts
    int first_slot;
};
__host__ __device__ inline int pad_chunks(int W, int H) {
    const int row_chunks = (W + 2 * KLT_PAD + 15) / 16;
    return 2 * KLT_PAD * row_chunks + H * 7;  // side strips: 3 chunks left, 4 chunks from the 16-byte boundary at or below PAD + W
}
__global__ void __launch_bounds__(256) pad_fill_kernel(PadArgs P) {
    const int slot = P.first_slot + blockIdx.y;
    const int total = P.off[KLT_LEVELS];
    for (int g = blockIdx.x * 256 + threadIdx.x; g < total; g += gridDim.x * 256) {
        int level = 0;
        while (g >= P.off[level + 1]) level++;
        int e = g - P.off[level];
        const int W = P.W[level], H = P.H[level], pitch = P.pitch[level];
        const int row_chunks = (W + 2 * KLT_PAD + 15) / 16, side_chunks = 7;
        uint8_t *plane = P.base[level] + (size_t) slot * P.slot_stride[level];
        int yo, xo;  // padded coordinates of the chunk's first byte
        if (e < 2 * KLT_PAD * row_chunks) {
            yo = e / row_chunks, xo = 16 * (e - yo * row_chunks);
            if (yo >= KLT_PAD) yo += H;
        } else {
            e -= 2 * KLT_PAD * row_chunks;
            yo = KLT_PAD + e / side_chunks;
            const int c = e % side_chunks;
            // left strip: chunks 0..2; right strip: 4 chunks from the 16-byte boundary at or below PAD + W (in-image bytes it
            // covers are rewritten with their own values)
            xo = c < 3 ? 16 * c : ((KLT_PAD + W) & ~15) + 16 * (c - 3);
        }
        const uint8_t *srow = plane + (size_t) (reflect101(yo - KLT_PAD, H) + KLT_PAD) * pitch + KLT_PAD;  // interior of the source row
        union {
            uint4 v;
            uint8_t b[16];
        } u;
        const int lx = xo - KLT_PAD;  // logical x of the first byte
        if (lx >= 0 && lx + 16 <= W && (((size_t) (srow + lx)) & 15) == 0) {
            u.v = *(const uint4 *) (srow + lx);  // interior columns of a pad row: straight aligned copy
        } else {
#pragma unroll
            for (int k = 0; k < 16; k++) u.b[k] = srow[reflect101(lx + k, W)];
        }
        if (xo + 16 <= pitch) *(uint4 *) (plane + (size_t) yo * pitch + xo) = u.v;
    }
}

// Scatter `count` linearly staged W x H frames into the level-0 planes of consecutive slots (16-byte chunks; HBM-bound, W * H in + out per
// frame).  The H2D copies that feed it are LINEAR (full-rate DMA); a strided cudaMemcpy2D into the padded planes runs well below that.
__global__ void __launch_bounds__(256) klt_unpack_level0_kernel(const uint8_t *__restrict__ stage, uint8_t *__restrict__ plane0, int W, int H, int pitch,
                                                                size_t slot_stride, int first_slot) {
    const int slot = first_slot + blockIdx.z;
    const uint8_t *src = stage + (size_t) blockIdx.z * W * H;
    uint8_t *dst = plane0 + (size_t) slot * slot_stride + (size_t) KLT_PAD * pitch + KLT_PAD;
    const int chunks = (W + 15) / 16;
    const int y = blockIdx.y, c = blockIdx.x * 256 + threadIdx.x;
    if (c >= chunks || y >= H) return;
    const uint8_t *sp = src + (size_t) y * W + 16 * c;
    uint8_t *dp = dst + (size_t) y * pitch + 16 * c;
    if (16 * c + 16 <= W && ((((size_t) sp) | ((size_t) dp)) & 15) == 0) {
        *(uint4 *) dp = *(const uint4 *) sp;
    } else {
        for (int k = 0; k < 16 && 16 * c + k < W; k++) dp[k] = sp[k];
    }
}

// ------------------------------------------------------------------------------------------------ LK tracker
// The staged windows are addressed by 32-bit SHARED-space addresses and read with ld.shared (no generic loads, no generic <-> shared
// conversions, and the per-warp bases stay in three registers instead of being re-derived from threadIdx inside the loops: an instruction profile of
// the earlier form showed a noticeable share of such re-materialisations and generic loads).
struct WarpSmem {
    uint32_t iw;    // 48x24 template window, origin ((ipx-1) & ~15, ipy-1)
    uint32_t jw;    // 48x32 search window, origin (jx0 (16-aligned), jy0)
    uint32_t pg;    // 26 x 24 ints: Q14 bilinear grid P (23 rows) + 3 zero rows (interior windows) or 22 x 22 packed Scharr taps (border windows)
    uint32_t bar_i, bar_j;  // mbarriers: template window, search window
    uint32_t phase_i, phase_j;
};
__device__ __forceinline__ unsigned lds_u32(uint32_t a) {
    unsigned v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ int lds_s32(uint32_t a) { return (int) lds_u32(a); }
__device__ __forceinline__ unsigned lds_u8(uint32_t a) {
    unsigned v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_v4(uint32_t a, int x, int y, int z, int w) {
    asm volatile("st.shared.v4.s32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ void sts_s32(uint32_t a, int x) { asm volatile("st.shared.s32 [%0], %1;" ::"r"(a), "r"(x) : "memory"); }
// mbarrier / TMA wrappers on shared-space addresses
__device__ __forceinline__ void mbar_expect_tx_a(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP_A:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_A;\n"
        "bra WAIT_LOOP_A;\n"
        "DONE_A:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d_a(uint32_t smem_dst, const CUtensorMap *map, int c0, int c1, int c2, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(smem_dst),
                 "l"((uint64_t) map), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
                 : "memory");
}

// Box origin for a window whose top-left pixel is (px, py): `margin` pixels of slack on the low side, x aligned to 16 bytes (TMA).
__device__ __forceinline__ void box_origin(int px, int py, int margin, int &bx, int &by) {
    bx = (px - margin) & ~15;
    by = py - margin;
}

__device__ __forceinline__ void bilinear_weights(float a, float b, int &iw00, int &iw01, int &iw10, int &iw11) {
    iw00 = __float2int_rn((1.f - a) * (1.f - b) * 16384.f);
    iw01 = __float2int_rn(a * (1.f - b) * 16384.f);
    iw10 = __float2int_rn((1.f - a) * b * 16384.f);
    iw11 = 16384 - iw00 - iw01 - iw10;
}

__device__ __forceinline__ float warp_sum_exact(int v) {
    // exact sum of 32 int32 values (two REDUX on 16-bit halves, recombined exactly in int64), rounded ONCE to f32
    int lo = v & 0xFFFF, hi = v >> 16;
    int slo = __reduce_add_sync(0xffffffffu, lo);
    int shi = __reduce_add_sync(0xffffffffu, hi);
    return (float) ((long long) shi * 65536LL + (long long) slo);  // exact 64-bit integer, one rounding (int64 -> f32, RN)
}

// ---- packed-byte bilinear taps ------------------------------------------------------------------------------------------------
// dp2a with signed 16-bit weights (iw11 = 16384 - iw00 - iw01 - iw10 can be -1 after rounding) and unsigned bytes:
//   d = c + a.h0 * b.byte[0|2] + a.h1 * b.byte[1|3]
__device__ __forceinline__ int dp2a_lo_su(int a, unsigned b, int c) {
    int d;
    asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ int dp2a_hi_su(int a, unsigned b, int c) {
    int d;
    asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
// The 21x21 window is cut into 63 horizontal runs of 7 pixels (3 per row); lane owns runs `lane` and `lane + 32` (lane 31: one run).
// A run's 8 + 8 tap bytes (two rows) are fetched as aligned 32-bit words and re-aligned with funnel shifts, then every pixel's four taps
// are two dp2a on packed byte pairs: ~4 instructions per pixel instead of 4 byte loads + 4 multiply-adds.
__device__ __forceinline__ int pack_w(int lo, int hi) { return (int) (((unsigned) lo & 0xFFFFu) | ((unsigned) hi << 16)); }
struct RunBytes {
    unsigned e0, e1, o0, o1;  // even stream: bytes 0..3 | 4..7;  odd stream (shifted by one byte): bytes 1..4 | 5..7
};
__device__ __forceinline__ RunBytes run_bytes(uint32_t wa, int m8) {  // wa: 4-byte aligned shared address of the word holding the run's first byte
    const unsigned w0 = lds_u32(wa), w1 = lds_u32(wa + 4), w2 = lds_u32(wa + 8);
    RunBytes r;
    r.e0 = __funnelshift_r(w0, w1, m8);
    r.e1 = __funnelshift_r(w1, w2, m8);
    r.o0 = __funnelshift_r(r.e0, r.e1, 8);
    r.o1 = r.e1 >> 8;
    return r;
}
// v[i] = c0 + sum of the four Q14-weighted taps of pixel i of the run (i = 0..6, or 0..7 with N8); wt = iw00 | iw01 << 16, wb = iw10 | iw11 << 16
template <int NPIX>
__device__ __forceinline__ void run_taps(const RunBytes &t, const RunBytes &b, int wt, int wb, int c0, int *v) {
    v[0] = dp2a_lo_su(wb, b.e0, dp2a_lo_su(wt, t.e0, c0));
    v[1] = dp2a_lo_su(wb, b.o0, dp2a_lo_su(wt, t.o0, c0));
    v[2] = dp2a_hi_su(wb, b.e0, dp2a_hi_su(wt, t.e0, c0));
    v[3] = dp2a_hi_su(wb, b.o0, dp2a_hi_su(wt, t.o0, c0));
    v[4] = dp2a_lo_su(wb, b.e1, dp2a_lo_su(wt, t.e1, c0));
    v[5] = dp2a_lo_su(wb, b.o1, dp2a_lo_su(wt, t.o1, c0));
    v[6] = dp2a_hi_su(wb, b.e1, dp2a_hi_su(wt, t.e1, c0));
    if (NPIX == 8) v[7] = 0;  // pixel 7 needs byte 8: handled by the caller
}

// the same with a per-pixel accumulator start c0[i] (the iteration: c0 = 2^8 - 512 I folds the "- I" of the difference into the taps)
template <int NPIX>
__device__ __forceinline__ void run_taps_c(const RunBytes &t, const RunBytes &b, int wt, int wb, const int *c0, int *v) {
    v[0] = dp2a_lo_su(wb, b.e0, dp2a_lo_su(wt, t.e0, c0[0]));
    v[1] = dp2a_lo_su(wb, b.o0, dp2a_lo_su(wt, t.o0, c0[1]));
    v[2] = dp2a_hi_su(wb, b.e0, dp2a_hi_su(wt, t.e0, c0[2]));
    v[3] = dp2a_hi_su(wb, b.o0, dp2a_hi_su(wt, t.o0, c0[3]));
    v[4] = dp2a_lo_su(wb, b.e1, dp2a_lo_su(wt, t.e1, c0[4]));
    v[5] = dp2a_lo_su(wb, b.o1, dp2a_lo_su(wt, t.o1, c0[5]));
    v[6] = dp2a_hi_su(wb, b.e1, dp2a_hi_su(wt, t.e1, c0[6]));
}

// Track one point from image slot sI to image slot sJ through all levels.  All lanes hold identical scalars.
__device__ __forceinline__ void lk_track_point(const KltMaps &maps, const KltArgs &A, WarpSmem &S, int lane, int sI, int sJ,
                                               float2 prev, float2 init, bool check_final, float2 &out, int &status,
                                               float *err_out) {
    // lane's template pixels: runs rA = lane and rB = lane + 32 of the 63 seven-pixel runs; register k = 7 * run + i <-> pixel
    // (x0 + i, y) of that run.  Lane 31 has no second run: its slots k = 7..13 carry I = G = 0.
    const int yA = lane / 3, xA = 7 * (lane - 3 * yA);
    const bool validB = lane < 31;
    const int rB = validB ? lane + 32 : 62;
    const int yB = rB / 3, xB = 7 * (rB - 3 * yB);
    const int offA = yA * KLT_BOXW + xA, offB = yB * KLT_BOXW + xB;  // byte offset of the run's first tap inside a staged window
    const float half = 10.f;
    const float FLT_SCALE = 1.f / (1 << 20);
    status = 1;
    float err_val = 0.f;
    float2 nextPt = make_float2(0.f, 0.f);
    const int maxLevel = A.n_levels - 1;
    bool i_pending = false;  // a template-window TMA for the upcoming level is in flight

    for (int level = maxLevel; level >= 0; level--) {
        const KltLevel &L = A.lv[level];
        const float scale = __int_as_float((127 - level) << 23);  // 2^-level, exact (OpenCV: (float) (1. / (1 << level)))
        float px = prev.x * scale, py = prev.y * scale;
        if (level == maxLevel) {
            if (A.use_initial_flow) {
                nextPt.x = init.x * scale;
                nextPt.y = init.y * scale;
            } else {
                nextPt.x = px;
                nextPt.y = py;
            }
        } else {
            nextPt.x = nextPt.x * 2.f;
            nextPt.y = nextPt.y * 2.f;
        }
        px -= half;
        py -= half;
        const int ipx = __float2int_rd(px), ipy = __float2int_rd(py);
        if (ipx < -KLT_WIN || ipx >= L.W || ipy < -KLT_WIN || ipy >= L.H) {
            if (level == 0) status = 0;
            continue;
        }
        float nx = nextPt.x - half, ny = nextPt.y - half;
        int inx = __float2int_rd(nx), iny = __float2int_rd(ny);
        const bool j_ok = !(inx < -KLT_WIN || inx >= L.W || iny < -KLT_WIN || iny >= L.H);
        int jx0, jy0, ix0, iy0;
        box_origin(inx, iny, KLT_MARGIN, jx0, jy0);
        box_origin(ipx - 1, ipy - 1, 0, ix0, iy0);  // template window: 21 + 1 (bilinear) + 2 (Scharr)
        const int oxI = ipx - 1 - ix0 + (ipy - 1 - iy0) * KLT_BOXW;        // byte offset of pixel (ipx-1, ipy-1) inside the staged window
        // all 24x24 template taps inside the image <=> OpenCV's zero derivative border is never touched
        const bool t_in = ipx - 1 >= 0 && ipy - 1 >= 0 && ipx + 23 <= L.W && ipy + 23 <= L.H;

        // ---- stage the windows with TMA: the template window may already be in flight (prefetched by the previous level)
        __syncwarp();
        if (lane == 0) {
            fence_proxy_async();
            if (!i_pending) {
                mbar_expect_tx_a(S.bar_i, KLT_BOXW * KLT_BOXH_I);
                tma_load_3d_a(S.iw, &maps.mi[level], ix0 + KLT_PAD, iy0 + KLT_PAD, sI, S.bar_i);
            }
            if (j_ok) {
                mbar_expect_tx_a(S.bar_j, KLT_BOXW * KLT_BOXH_J);
                tma_load_3d_a(S.jw, &maps.mj[level], jx0 + KLT_PAD, jy0 + KLT_PAD, sJ, S.bar_j);
            }
        }
        i_pending = false;
        mbar_wait_a(S.bar_i, S.phase_i);
        S.phase_i ^= 1;

        float a = px - (float) ipx, b = py - (float) ipy;
        int iw00, iw01, iw10, iw11;
        bilinear_weights(a, b, iw00, iw01, iw10, iw11);
        int Ireg[KLT_PXL], Gxr[KLT_PXL], Gyr[KLT_PXL];
        int sA11 = 0, sA12 = 0, sA22 = 0;
        if (t_in) {
            // ---- interpolate first, differentiate second.  Scharr is linear and OpenCV rounds only AFTER interpolating, so
            //      sum_taps w * Ix(tap) == Scharr_x(P) with P = sum_taps w * I(tap) (exact Q14 integers, |.| < 2^27):
            //      one 23x23 grid gives I, Ix and Iy of the whole 21x21 template.
            // P grid (23 x 23, pitch 24): lane = (column run cr of 8, row group rg of 3 rows), 24 lanes; the bottom tap row of one grid
            // row is the top tap row of the next, so 4 byte rows are fetched for 3 grid rows
            const int wt = pack_w(iw00, iw01), wb = pack_w(iw10, iw11);
            if (lane < 24) {
                const int cr = lane % 3, rg = lane / 3;
                const uint32_t bp = S.iw + oxI + (3 * rg) * KLT_BOXW + 8 * cr;  // the windows are 128-byte aligned: alignment of bp = that of the offset
                const int m8 = (int) (bp & 3u) * 8;
                const uint32_t wa = bp & ~3u;
                RunBytes top = run_bytes(wa, m8);
                unsigned tb8 = lds_u8(bp + 8);  // 9th byte: right tap of grid column 7 of the run
#pragma unroll
                for (int rr = 0; rr < 3; rr++) {
                    const int gy = 3 * rg + rr;
                    const RunBytes bot = run_bytes(wa + (rr + 1) * KLT_BOXW, m8);
                    const unsigned bb8 = lds_u8(bp + (rr + 1) * KLT_BOXW + 8);
                    int v[8];
                    run_taps<8>(top, bot, wt, wb, 0, v);
                    v[7] = (int) (top.o1 >> 16 & 0xFF) * iw00 + (int) tb8 * iw01 + (int) (bot.o1 >> 16 & 0xFF) * iw10 + (int) bb8 * iw11;
                    if (gy < 23) {
                        const uint32_t dst = S.pg + 4 * (gy * 24 + 8 * cr);
                        sts_v4(dst, v[0], v[1], v[2], v[3]);
                        sts_v4(dst + 16, v[4], v[5], v[6], v[7]);
                    }
                    top = bot, tb8 = bb8;
                }
            }
            __syncwarp();
            // template of the lane's two runs: separable Scharr on the grid (column sums c_j shared along the run)
#pragma unroll
            for (int run = 0; run < 2; run++) {
                // lane 31 has no second run: it reads the three zero rows (23..25) instead
                const uint32_t pp = S.pg + 4 * (run ? (validB ? yB * 24 + xB : 23 * 24) : yA * 24 + xA);
                int P1[9], c[9], d[9];
#pragma unroll
                for (int j = 0; j < 9; j++) {
                    const int p0 = lds_s32(pp + 4 * j), p2 = lds_s32(pp + 4 * (48 + j));
                    P1[j] = lds_s32(pp + 4 * (24 + j));
                    c[j] = 3 * (p0 + p2) + 10 * P1[j];  // vertical smoothing (3 10 3): Ix = c[i + 2] - c[i]
                    d[j] = p2 - p0;                     // vertical difference:        Iy = 3 (d[i] + d[i + 2]) + 10 d[i + 1]
                }
#pragma unroll
                for (int i = 0; i < 7; i++) {
                    const int ival = (P1[i + 1] + (1 << 8)) >> 9;
                    const int ixv = (c[i + 2] - c[i] + (1 << 13)) >> 14;
                    const int iyv = (3 * (d[i] + d[i + 2]) + 10 * d[i + 1] + (1 << 13)) >> 14;
                    // the iteration needs (v - 512 I) only: keep c0 = 2^8 - (I << 9), the dp2a accumulator start ((v - 512 I) >> 9 == (v >> 9) - I)
                    Ireg[7 * run + i] = (1 << 8) - (ival << 9), Gxr[7 * run + i] = ixv, Gyr[7 * run + i] = iyv;
                    sA11 += ixv * ixv;
                    sA12 += ixv * iyv;
                    sA22 += iyv * iyv;
                }
            }
        } else {
            // ---- window touches the image border: Scharr taps first (zero outside the image: OpenCV pads derivI with zeros)
            for (int i = lane; i < 22 * 22; i += 32) {
                int dy = i / 22, dx = i - dy * 22;
                const uint32_t r0 = S.iw + dy * KLT_BOXW + dx + oxI, r1 = r0 + KLT_BOXW, r2 = r1 + KLT_BOXW;
                const int a00 = (int) lds_u8(r0), a01 = (int) lds_u8(r0 + 1), a02 = (int) lds_u8(r0 + 2);
                const int a10 = (int) lds_u8(r1), a12 = (int) lds_u8(r1 + 2);
                const int a20 = (int) lds_u8(r2), a21 = (int) lds_u8(r2 + 1), a22 = (int) lds_u8(r2 + 2);
                int t0m = 3 * (a00 + a20) + 10 * a10;
                int t0p = 3 * (a02 + a22) + 10 * a12;
                int t1m = a20 - a00, t1c = a21 - a01, t1p = a22 - a02;
                int gx = t0p - t0m, gy = 3 * (t1m + t1p) + 10 * t1c;
                int X = ipx + dx, Y = ipy + dy;
                if (X < 0 || X >= L.W || Y < 0 || Y >= L.H) gx = gy = 0;
                sts_s32(S.pg + 4 * i, (gx & 0xFFFF) | (gy << 16));
            }
            __syncwarp();
#pragma unroll
            for (int k = 0; k < KLT_PXL; k++) {
                const int run = k / 7, i = k - 7 * run;
                if (run == 0 || validB) {
                    const int y = run ? yB : yA, x = (run ? xB : xA) + i;
                    const uint32_t sp = S.iw + (y + 1) * KLT_BOXW + x + 1 + oxI;
                    int ival = ((int) lds_u8(sp) * iw00 + (int) lds_u8(sp + 1) * iw01 + (int) lds_u8(sp + KLT_BOXW) * iw10 + (int) lds_u8(sp + KLT_BOXW + 1) * iw11 +
                                (1 << 8)) >> 9;
                    const uint32_t d = S.pg + 4 * (y * 22 + x);
                    int d00 = lds_s32(d), d01 = lds_s32(d + 4), d10 = lds_s32(d + 88), d11 = lds_s32(d + 92);
                    int ixv = ((short) d00 * iw00 + (short) d01 * iw01 + (short) d10 * iw10 + (short) d11 * iw11 + (1 << 13)) >> 14;
                    int iyv = ((d00 >> 16) * iw00 + (d01 >> 16) * iw01 + (d10 >> 16) * iw10 + (d11 >> 16) * iw11 + (1 << 13)) >> 14;
                    Ireg[k] = (1 << 8) - (ival << 9);
                    Gxr[k] = ixv, Gyr[k] = iyv;
                    sA11 += ixv * ixv;
                    sA12 += ixv * iyv;
                    sA22 += iyv * iyv;
                } else {
                    Ireg[k] = 0;
                    Gxr[k] = Gyr[k] = 0;
                }
            }
        }
        // ---- the template now lives in registers: prefetch the NEXT level's template window while this level iterates
        if (level > 0) {
            const KltLevel &Ln = A.lv[level - 1];
            const float sn = __int_as_float((127 - (level - 1)) << 23);
            const int npx = __float2int_rd(prev.x * sn - half), npy = __float2int_rd(prev.y * sn - half);
            if (!(npx < -KLT_WIN || npx >= Ln.W || npy < -KLT_WIN || npy >= Ln.H)) {
                int nx0, ny0;
                box_origin(npx - 1, npy - 1, 0, nx0, ny0);
                __syncwarp();  // every lane is done reading the template window
                if (lane == 0) {
                    fence_proxy_async();
                    mbar_expect_tx_a(S.bar_i, KLT_BOXW * KLT_BOXH_I);
                    tma_load_3d_a(S.iw, &maps.mi[level - 1], nx0 + KLT_PAD, ny0 + KLT_PAD, sI, S.bar_i);
                }
                i_pending = true;
            }
        }
        if (j_ok) {
            mbar_wait_a(S.bar_j, S.phase_j);
            S.phase_j ^= 1;
        }
        // per-lane partials fit int32 (14 * 4080^2 < 2^28); the warp total needs 64 bits
        const float A11 = warp_sum_exact(sA11) * FLT_SCALE;
        const float A12 = warp_sum_exact(sA12) * FLT_SCALE;
        const float A22 = warp_sum_exact(sA22) * FLT_SCALE;
        float D = A11 * A22 - A12 * A12;
        const float minEig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / (float) (2 * KLT_WIN * KLT_WIN);
        if ((double) minEig < A.min_eig_thr || D < 1.192092896e-07f) {
            if (level == 0) status = 0;
            continue;
        }
        D = 1.f / D;

        float pdx = 0.f, pdy = 0.f;
        for (int j = 0; j < A.max_iter; j++) {
            inx = __float2int_rd(nx);
            iny = __float2int_rd(ny);
            if (inx < -KLT_WIN || inx >= L.W || iny < -KLT_WIN || iny >= L.H) {
                if (level == 0) status = 0;
                break;
            }
            int ox = inx - jx0, oy = iny - jy0;
            if (ox < 0 || ox > KLT_BOXW - 22 || oy < 0 || oy > KLT_BOXH_J - 22) {
                // the track left the staged window: re-centre it
                box_origin(inx, iny, KLT_MARGIN, jx0, jy0);
                __syncwarp();
                if (lane == 0) {
                    fence_proxy_async();
                    mbar_expect_tx_a(S.bar_j, KLT_BOXW * KLT_BOXH_J);
                    tma_load_3d_a(S.jw, &maps.mj[level], jx0 + KLT_PAD, jy0 + KLT_PAD, sJ, S.bar_j);
                }
                mbar_wait_a(S.bar_j, S.phase_j);
                S.phase_j ^= 1;
                ox = inx - jx0;
                oy = iny - jy0;
            }
            a = nx - (float) inx;
            b = ny - (float) iny;
            bilinear_weights(a, b, iw00, iw01, iw10, iw11);
            const uint32_t jb = S.jw + oy * KLT_BOXW + ox;
            const int wt = pack_w(iw00, iw01), wb = pack_w(iw10, iw11);
            int sb1 = 0, sb2 = 0;
#pragma unroll
            for (int run = 0; run < 2; run++) {
                const uint32_t bp = jb + (run ? offB : offA);
                const int m8 = (int) (bp & 3u) * 8;
                const RunBytes top = run_bytes(bp & ~3u, m8), bot = run_bytes((bp & ~3u) + KLT_BOXW, m8);
                int v[7];
                run_taps_c<7>(top, bot, wt, wb, &Ireg[7 * run], v);  // accumulator start = 2^8 - 512 I: v >> 9 is J - I
#pragma unroll
                for (int i = 0; i < 7; i++) {
                    const int diff = v[i] >> 9;  // dead slots: G = 0
                    sb1 += diff * Gxr[7 * run + i];
                    sb2 += diff * Gyr[7 * run + i];
                }
            }
            const float b1 = warp_sum_exact(sb1) * FLT_SCALE;
            const float b2 = warp_sum_exact(sb2) * FLT_SCALE;
            const float dx = (A12 * b2 - A22 * b1) * D;
            const float dy = (A12 * b1 - A11 * b2) * D;
            nx += dx;
            ny += dy;
            nextPt.x = nx + half;
            nextPt.y = ny + half;
            if ((double) dx * (double) dx + (double) dy * (double) dy <= A.eps2) break;
            // OpenCV compares the float sums with the double 0.01; for a float x, |x| < 0.01 (double) <=> |x| <= 0.01f, because
            // 0.01f = 0.0099999997765 is the largest float below 0.01
            if (j > 0 && fabsf(dx + pdx) <= 0.01f && fabsf(dy + pdy) <= 0.01f) {
                nextPt.x -= dx * 0.5f;
                nextPt.y -= dy * 0.5f;
                break;
            }
            pdx = dx;
            pdy = dy;
        }

        if (level == 0 && status && check_final) {
            // lkpyramid.cpp level-0 epilogue: the final window origin must still be inside [-win, cols) x [-win, rows)
            float fx = nextPt.x - half, fy = nextPt.y - half;
            int fix = __float2int_rd(fx), fiy = __float2int_rd(fy);
            if (fix < -KLT_WIN || fix >= L.W || fiy < -KLT_WIN || fiy >= L.H) {
                status = 0;
            } else if (err_out != nullptr) {
                int ox = fix - jx0, oy = fiy - jy0;
                if (ox < 0 || ox > KLT_BOXW - 22 || oy < 0 || oy > KLT_BOXH_J - 22) {
                    box_origin(fix, fiy, KLT_MARGIN, jx0, jy0);
                    __syncwarp();
                    if (lane == 0) {
                        fence_proxy_async();
                        mbar_expect_tx_a(S.bar_j, KLT_BOXW * KLT_BOXH_J);
                        tma_load_3d_a(S.jw, &maps.mj[level], jx0 + KLT_PAD, jy0 + KLT_PAD, sJ, S.bar_j);
                    }
                    mbar_wait_a(S.bar_j, S.phase_j);
                    S.phase_j ^= 1;
                    ox = fix - jx0;
                    oy = fiy - jy0;
                }
                a = fx - (float) fix;
                b = fy - (float) fiy;
                bilinear_weights(a, b, iw00, iw01, iw10, iw11);
                const uint32_t jb = S.jw + oy * KLT_BOXW + ox;
                const int wt = pack_w(iw00, iw01), wb = pack_w(iw10, iw11);
                int se = 0;
#pragma unroll
                for (int run = 0; run < 2; run++) {
                    if (run == 1 && !validB) continue;
                    const uint32_t bp = jb + (run ? offB : offA);
                    const int m8 = (int) (bp & 3u) * 8;
                    const RunBytes top = run_bytes(bp & ~3u, m8), bot = run_bytes((bp & ~3u) + KLT_BOXW, m8);
                    int v[7];
                    run_taps_c<7>(top, bot, wt, wb, &Ireg[7 * run], v);
#pragma unroll
                    for (int i = 0; i < 7; i++) se += abs(v[i] >> 9);
                }
                err_val = warp_sum_exact(se) * 1.f / (float) (32 * KLT_WIN * KLT_WIN);
            }
        }
    }
    out = nextPt;
    if (err_out != nullptr) *err_out = status ? err_val : 0.f;
}

// held to 4 resident CTAs per SM (<= 128 registers, no spills): measured faster than the 5-CTA bound, whose register cap (<= 102) costs
// more instructions
__global__ void __launch_bounds__(KLT_WPB * 32, 4) klt_track_kernel(const __grid_constant__ KltMaps maps, const KltArgs A) {
    __shared__ __align__(128) uint8_t s_iw[KLT_WPB][KLT_BOXW * KLT_BOXH_I];
    __shared__ __align__(128) uint8_t s_jw[KLT_WPB][KLT_BOXW * KLT_BOXH_J];
    __shared__ __align__(16) int s_pg[KLT_WPB][26 * 24];
    __shared__ __align__(8) uint64_t s_bar[KLT_WPB][2];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int task = blockIdx.x * KLT_WPB + warp;
    if (lane == 0) {
        mbar_init(&s_bar[warp][0], 1);
        mbar_init(&s_bar[warp][1], 1);
        fence_mbar_init();
    }
    __syncwarp();
    if (task >= A.n_total) return;

    WarpSmem S;
    S.iw    = smem_u32(s_iw[warp]);
    S.jw    = smem_u32(s_jw[warp]);
    S.pg    = smem_u32(s_pg[warp]);
    S.bar_i = smem_u32(&s_bar[warp][0]);
    S.bar_j = smem_u32(&s_bar[warp][1]);
    // rows 23..25 of the grid stay zero for the whole kernel (the grid writes rows 0..22, the border path entries 0..483): lane 31's second
    // (dead) run reads them, so its I = Ix = Iy = 0 without any select
    for (int e = lane; e < 72; e += 32) sts_s32(S.pg + 4 * (23 * 24 + e), 0);
    __syncwarp();
    S.phase_i = S.phase_j = 0;

    const int sP = A.slots[2 * task], sN = A.slots[2 * task + 1];
    const float2 prev = A.prev_xy[task];
    const float2 init = A.init_xy[task];

    // direction 0: forward (prev slot -> next slot); direction 1 (mode 1 only): backward with
    // prevPts = forward result and initial flow = the original points (IG/tracking/tracking.cc:390-393).
    float2 fwd = make_float2(0.f, 0.f), bwd = make_float2(0.f, 0.f);
    int st = 0, st2 = 0;
    float err_v = 0.f;
    const int ndir = A.mode == 0 ? 1 : 2;
#pragma unroll 1
    for (int dir = 0; dir < ndir; dir++) {
        float2 o;
        int s;
        lk_track_point(maps, A, S, lane, dir == 0 ? sP : sN, dir == 0 ? sN : sP, dir == 0 ? prev : fwd, dir == 0 ? init : prev,
                       dir == 0 ? (A.check_final != 0) : true, o, s, (dir == 0 && A.err) ? &err_v : nullptr);
        if (dir == 0) {
            fwd = o;
            st  = s;
        } else {
            bwd = o;
            st2 = s;
        }
    }
    if (lane != 0) return;
    if (A.mode == 0) {
        A.fwd_xy[task] = fwd;
        A.status[task] = (uint8_t) st;
        if (A.err) A.err[task] = err_v;
        return;
    }
    // gates (tracking.cc:396-403): isOnBorder (tracking.cc:847-849, double compare) and ptsDistance (841-845)
    bool on_border = (double) fwd.x < 5.0 || (double) fwd.y < 5.0 || (double) fwd.x > ((double) A.img_w - 5.0) ||
                     (double) fwd.y > ((double) A.img_h - 5.0);
    double ddx = (double) (bwd.x - prev.x), ddy = (double) (bwd.y - prev.y);
    double dist = sqrt(ddx * ddx + ddy * ddy);
    A.fwd_xy[task] = fwd;
    if (A.bwd_xy) A.bwd_xy[task] = bwd;
    A.status[task] = (uint8_t) ((st && st2 && !on_border && dist < 0.5) ? 1 : 0);
}

}  // namespace icg

// ======================================================================================================= C ABI
using namespace icg;

static uint64_t hash_image(const uint8_t *p, int W, int H, int stride) {
    // 64-bit multiply-fold hash over the full image (a false cache hit would be a correctness bug)
    uint64_t h = 0x9E3779B97F4A7C15ull ^ ((uint64_t) W << 32) ^ (uint64_t) H;
    for (int y = 0; y < H; y++) {
        const uint8_t *r = p + (size_t) y * stride;
        int x = 0;
        for (; x + 8 <= W; x += 8) {
            uint64_t v;
            memcpy(&v, r + x, 8);
            h = (h ^ v) * 0xFF51AFD7ED558CCDull;
            h ^= h >> 29;
        }
        for (; x < W; x++) {
            h = (h ^ r[x]) * 0xC4CEB9FE1A85EC53ull;
            h ^= h >> 31;
        }
    }
    return h ? h : 1;
}

extern "C" {

int icg_klt_create(icg_klt **out, int width, int height, int n_slots, int max_points, int device, void *stream) {
    if (!out || width < 32 || height < 32 || n_slots < 2 || max_points < 1) {
        set_error("icg_klt_create: bad arguments");
        return ICG_EINVAL;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        set_error("icg_klt_create: no CUDA device (this library has no CPU fallback)");
        return ICG_ENODEVICE;
    }
    if (device < 0 || device >= ndev) {
        set_error("icg_klt_create: device %d out of range (%d devices)", device, ndev);
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    ICG_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error("icg_klt_create: device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor);
        return ICG_ENODEVICE;
    }
    icg_klt *h = new icg_klt();
    h->W = width;
    h->H = height;
    h->n_slots = n_slots;
    h->max_pts = max_points;
    h->device = device;
    h->own_stream = (stream == nullptr);
    if (stream)
        h->stream = (cudaStream_t) stream;
    else
        ICG_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    int w = width, hh = height;
    for (int l = 0; l < KLT_LEVELS; l++) {
        if (l > 0) {
            w = (w + 1) / 2;
            hh = (hh + 1) / 2;
        }
        int pitch = (w + 2 * KLT_PAD + 15) & ~15;
        size_t slot_stride = (size_t) pitch * (hh + 2 * KLT_PAD);
        ICG_CUDA(cudaMalloc(&h->planes[l], slot_stride * n_slots));
        ICG_CUDA(cudaMemsetAsync(h->planes[l], 0, slot_stride * n_slots, h->stream));
        h->lv[l] = KltLevel{h->planes[l], w, hh, pitch, slot_stride};
        // cv::buildOpticalFlowPyramid stops at the first level that is not larger than the window
        if (l == 0 || (h->n_levels == l && w > KLT_WIN && hh > KLT_WIN)) h->n_levels = l + 1;
        int rc = encode_tensor_map_u8_3d(&h->maps.mj[l], h->planes[l], (uint64_t) (w + 2 * KLT_PAD), (uint64_t) (hh + 2 * KLT_PAD), (uint64_t) n_slots,
                                         (uint64_t) pitch, (uint64_t) slot_stride, KLT_BOXW, KLT_BOXH_J, 1);
        if (rc != ICG_OK) return rc;
        rc = encode_tensor_map_u8_3d(&h->maps.mi[l], h->planes[l], (uint64_t) (w + 2 * KLT_PAD), (uint64_t) (hh + 2 * KLT_PAD), (uint64_t) n_slots,
                                     (uint64_t) pitch, (uint64_t) slot_stride, KLT_BOXW, KLT_BOXH_I, 1);
        if (rc != ICG_OK) return rc;
    }
    ICG_CUDA(cudaMalloc(&h->d_slots, sizeof(int32_t) * 2 * max_points));
    ICG_CUDA(cudaMalloc(&h->d_prev, sizeof(float) * 2 * max_points));
    ICG_CUDA(cudaMalloc(&h->d_init, sizeof(float) * 2 * max_points));
    ICG_CUDA(cudaMalloc(&h->d_fwd, sizeof(float) * 2 * max_points));
    ICG_CUDA(cudaMalloc(&h->d_bwd, sizeof(float) * 2 * max_points));
    ICG_CUDA(cudaMalloc(&h->d_err, sizeof(float) * max_points));
    ICG_CUDA(cudaMalloc(&h->d_status, max_points));
    h->h_stage_bytes = (size_t) max_points * (2 * 4 + 8 * 4 + 4 + 1) + 64;
    ICG_CUDA(cudaMallocHost(&h->h_stage, h->h_stage_bytes));
    h->slot_hash.assign(n_slots, 0);
    h->slot_age.assign(n_slots, 0);
    h->age = 0;
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    *out = h;
    return ICG_OK;
}

void icg_klt_destroy(icg_klt *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    for (int l = 0; l < KLT_LEVELS; l++) cudaFree(h->planes[l]);
    cudaFree(h->d_slots);
    cudaFree(h->d_prev);
    cudaFree(h->d_init);
    cudaFree(h->d_fwd);
    cudaFree(h->d_bwd);
    cudaFree(h->d_err);
    cudaFree(h->d_status);
    cudaFreeHost(h->h_stage);
    if (h->d_upstage) cudaFree(h->d_upstage);
    track_scratch_free(h->track);
    if (h->own_stream) cudaStreamDestroy(h->stream);
    delete h;
}

int icg_klt_slot_level(icg_klt *h, int slot, int level, void **dev_ptr, int *pitch, int *w, int *hgt) {
    if (!h || slot < 0 || slot >= h->n_slots || level < 0 || level >= KLT_LEVELS) {
        set_error("icg_klt_slot_level: bad arguments");
        return ICG_EINVAL;
    }
    if (dev_ptr) *dev_ptr = h->planes[level] + (size_t) slot * h->lv[level].slot_stride + (size_t) KLT_PAD * h->lv[level].pitch + KLT_PAD;
    if (pitch) *pitch = h->lv[level].pitch;
    if (w) *w = h->lv[level].W;
    if (hgt) *hgt = h->lv[level].H;
    return ICG_OK;
}

int icg_klt_slot_level0(icg_klt *h, int slot, void **dev_ptr, int *pitch) { return icg_klt_slot_level(h, slot, 0, dev_ptr, pitch, nullptr, nullptr); }

int icg_klt_build_pyramids(icg_klt *h, int first_slot, int count) {
    if (!h || first_slot < 0 || count < 1 || first_slot + count > h->n_slots) {
        set_error("icg_klt_build_pyramids: bad slot range");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    // a producer may have written these level-0 planes in place (icg_klt_slot_level0): the host API's content cache must not hit on them
    for (int sl = first_slot; sl < first_slot + count; sl++) h->slot_hash[sl] = 0;
    // level by level: pad level l - 1 (reflect-101), then reduce it -- the reduction reads its border taps from the padding
    auto pad_level = [&](int lv) -> int {
        PadArgs P;
        for (int l = 0; l < KLT_LEVELS; l++) {
            P.base[l] = h->planes[l], P.W[l] = h->lv[l].W, P.H[l] = h->lv[l].H, P.pitch[l] = h->lv[l].pitch, P.slot_stride[l] = h->lv[l].slot_stride;
        }
        P.first_slot = first_slot;
        P.off[0] = 0;
        for (int l = 0; l < KLT_LEVELS; l++) P.off[l + 1] = P.off[l] + (l == lv ? pad_chunks(h->lv[l].W, h->lv[l].H) : 0);
        pad_fill_kernel<<<dim3((P.off[KLT_LEVELS] + 255) / 256, count), 256, 0, h->stream>>>(P);
        ICG_CHECK_LAUNCH();
        count_launch();
        return ICG_OK;
    };
    for (int l = 1; l < KLT_LEVELS; l++) {
        const KltLevel &s = h->lv[l - 1], &d = h->lv[l];
        int rc = pad_level(l - 1);
        if (rc != ICG_OK) return rc;
        dim3 grid((d.W + 255) / 256, (d.H + 3) / 4, count);
        pyr_down_kernel<<<grid, 256, 0, h->stream>>>(s.base, s.W, s.H, s.pitch, s.slot_stride, h->planes[l], d.W, d.H, d.pitch,
                                                     d.slot_stride, first_slot);
        ICG_CHECK_LAUNCH();
        count_launch();
    }
    {
        int rc = pad_level(KLT_LEVELS - 1);
        if (rc != ICG_OK) return rc;
    }
    return ICG_OK;
}

int icg_klt_upload_level0(icg_klt *h, int slot, const uint8_t *host_img, int stride) {
    if (!h || !host_img || slot < 0 || slot >= h->n_slots || stride < h->W) {
        set_error("icg_klt_upload: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    ICG_CUDA(cudaMemcpy2DAsync(h->planes[0] + (size_t) slot * h->lv[0].slot_stride + (size_t) KLT_PAD * h->lv[0].pitch + KLT_PAD, h->lv[0].pitch, host_img, stride,
                               h->W, h->H, cudaMemcpyHostToDevice, h->stream));
    h->slot_hash[slot] = 0;
    return ICG_OK;
}

int icg_klt_upload_batch(icg_klt *h, int first_slot, int count, const uint8_t *const *host_imgs, int stride) {
    if (!h || !host_imgs || first_slot < 0 || count < 1 || first_slot + count > h->n_slots || stride < h->W) {
        set_error("icg_klt_upload_batch: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    const size_t fb = (size_t) h->W * h->H;
    if (h->d_upstage_bytes < fb * count) {
        ICG_CUDA(cudaStreamSynchronize(h->stream));
        if (h->d_upstage) cudaFree(h->d_upstage);
        h->d_upstage = nullptr, h->d_upstage_bytes = 0;
        if (cudaMalloc(&h->d_upstage, fb * count) != cudaSuccess) {
            set_error("icg_klt_upload_batch: staging allocation of %zu bytes failed", fb * count);
            return ICG_ENOMEM;
        }
        h->d_upstage_bytes = fb * count;
    }
    for (int k = 0; k < count; k++) {
        if (!host_imgs[k]) {
            set_error("icg_klt_upload_batch: frame %d is NULL", k);
            return ICG_EINVAL;
        }
        if (stride == h->W) {  // one linear copy per frame
            ICG_CUDA(cudaMemcpyAsync(h->d_upstage + fb * k, host_imgs[k], fb, cudaMemcpyHostToDevice, h->stream));
        } else {
            ICG_CUDA(cudaMemcpy2DAsync(h->d_upstage + fb * k, h->W, host_imgs[k], stride, h->W, h->H, cudaMemcpyHostToDevice, h->stream));
        }
        h->slot_hash[first_slot + k] = 0;
    }
    const dim3 grid(((h->W + 15) / 16 + 255) / 256, h->H, count);
    klt_unpack_level0_kernel<<<grid, 256, 0, h->stream>>>(h->d_upstage, h->planes[0], h->W, h->H, h->lv[0].pitch, h->lv[0].slot_stride, first_slot);
    ICG_CHECK_LAUNCH();
    count_launch();
    return ICG_OK;
}

int icg_klt_upload(icg_klt *h, int slot, const uint8_t *host_img, int stride) {
    int rc = icg_klt_upload_level0(h, slot, host_img, stride);
    if (rc != ICG_OK) return rc;
    return icg_klt_build_pyramids(h, slot, 1);
}

int icg_klt_download_level(icg_klt *h, int slot, int level, uint8_t *host_img, int stride) {
    if (!h || !host_img || slot < 0 || slot >= h->n_slots || level < 0 || level >= KLT_LEVELS || stride < h->lv[level].W) {
        set_error("icg_klt_download_level: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    const KltLevel &L = h->lv[level];
    ICG_CUDA(cudaMemcpy2DAsync(host_img, stride, h->planes[level] + (size_t) slot * L.slot_stride + (size_t) KLT_PAD * L.pitch + KLT_PAD, L.pitch, L.W, L.H,
                               cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    return ICG_OK;
}

static int launch_track(icg_klt *h, int n_total, const int32_t *d_slots, const float *d_prev, const float *d_init, float *d_fwd,
                        float *d_bwd, uint8_t *d_status, float *d_err, int mode, int n_levels, int max_iter, double eps, int flags,
                        int check_final) {
    KltArgs A;
    for (int l = 0; l < KLT_LEVELS; l++) A.lv[l] = h->lv[l];
    A.n_total = n_total;
    A.n_levels = n_levels;
    if (max_iter < 0) max_iter = 0;
    if (max_iter > 100) max_iter = 100;
    if (eps < 0) eps = 0;
    if (eps > 10) eps = 10;
    A.max_iter = max_iter;
    A.mode = mode;
    A.use_initial_flow = (flags & ICG_OPTFLOW_USE_INITIAL_FLOW) ? 1 : 0;
    A.check_final = check_final;
    A.eps2 = eps * eps;
    A.min_eig_thr = 1e-4;
    A.img_w = (float) h->W;
    A.img_h = (float) h->H;
    A.slots = d_slots;
    A.prev_xy = (const float2 *) d_prev;
    A.init_xy = (const float2 *) d_init;
    A.fwd_xy = (float2 *) d_fwd;
    A.bwd_xy = (float2 *) d_bwd;
    A.status = d_status;
    A.err = d_err;
    int grid = (n_total + KLT_WPB - 1) / KLT_WPB;
    klt_track_kernel<<<grid, KLT_WPB * 32, 0, h->stream>>>(h->maps, A);
    ICG_CHECK_LAUNCH();
    count_launch();
    return ICG_OK;
}

int icg_klt_track_batch_dev(icg_klt *h, int n_total, const int32_t *dev_slots, const float *dev_prev_xy, const float *dev_init_xy,
                            float *dev_fwd_xy, float *dev_bwd_xy, uint8_t *dev_status, int mode) {
    if (!h || n_total < 0 || !dev_slots || !dev_prev_xy || !dev_init_xy || !dev_fwd_xy || !dev_status || (mode != 0 && mode != 1)) {
        set_error("icg_klt_track_batch_dev: bad arguments");
        return ICG_EINVAL;
    }
    if (n_total == 0) return ICG_OK;
    ICG_CUDA(cudaSetDevice(h->device));
    // reference parameters (IG/tracking/tracking.cc:385-393): maxLevel 3, (COUNT+EPS, 30, 0.01), USE_INITIAL_FLOW, err requested;
    // tracked on the levels cv2 builds for this size (fewer than 4 when a level would not be larger than the window)
    return launch_track(h, n_total, dev_slots, dev_prev_xy, dev_init_xy, dev_fwd_xy, dev_bwd_xy, dev_status, nullptr, mode, h->n_levels,
                        30, 0.01, ICG_OPTFLOW_USE_INITIAL_FLOW, 1);
}

int icg_klt_sync(icg_klt *h) {
    if (!h) return ICG_EINVAL;
    ICG_CUDA(cudaSetDevice(h->device));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    return ICG_OK;
}

// find (or create) the slot holding this host image; never evicts `keep`
static int slot_for_image(icg_klt *h, const uint8_t *img, int stride, int keep, int *slot_out) {
    uint64_t hv = hash_image(img, h->W, h->H, stride);
    h->age++;
    int victim = -1;
    uint64_t oldest = ~0ull;
    for (int s = 0; s < h->n_slots; s++) {
        if (h->slot_hash[s] == hv) {
            h->slot_age[s] = h->age;
            *slot_out = s;
            return ICG_OK;
        }
        if (s != keep && h->slot_age[s] < oldest) {
            oldest = h->slot_age[s];
            victim = s;
        }
    }
    int rc = icg_klt_upload(h, victim, img, stride);
    if (rc != ICG_OK) return rc;
    h->slot_hash[victim] = hv;
    h->slot_age[victim] = h->age;
    *slot_out = victim;
    return ICG_OK;
}

static int host_track(icg_klt *h, const uint8_t *prev, const uint8_t *next, int stride, const float *prev_xy, float *next_xy,
                      float *back_xy, uint8_t *status, float *err, int n, int mode, int n_levels, int max_iter, double eps, int flags) {
    if (!h || !prev || !next || !prev_xy || !next_xy || !status || n < 0 || stride < h->W) {
        set_error("klt host call: bad arguments");
        return ICG_EINVAL;
    }
    if (n > h->max_pts) {
        set_error("klt host call: n=%d exceeds max_points=%d of the handle", n, h->max_pts);
        return ICG_EINVAL;
    }
    if (n == 0) return ICG_OK;
    ICG_CUDA(cudaSetDevice(h->device));
    int sp, sn;
    int rc = slot_for_image(h, prev, stride, -1, &sp);
    if (rc != ICG_OK) return rc;
    rc = slot_for_image(h, next, stride, sp, &sn);
    if (rc != ICG_OK) return rc;
    // pack inputs into the pinned stage: [slots int2*n][prev float2*n][init float2*n]
    int32_t *hs = (int32_t *) h->h_stage;
    float *hp = (float *) (hs + 2 * n);
    float *hi = hp + 2 * n;
    for (int k = 0; k < n; k++) {
        hs[2 * k] = sp;
        hs[2 * k + 1] = sn;
    }
    memcpy(hp, prev_xy, sizeof(float) * 2 * n);
    if (flags & ICG_OPTFLOW_USE_INITIAL_FLOW)
        memcpy(hi, next_xy, sizeof(float) * 2 * n);
    else
        memcpy(hi, prev_xy, sizeof(float) * 2 * n);
    ICG_CUDA(cudaMemcpyAsync(h->d_slots, hs, sizeof(int32_t) * 2 * n, cudaMemcpyHostToDevice, h->stream));
    ICG_CUDA(cudaMemcpyAsync(h->d_prev, hp, sizeof(float) * 2 * n, cudaMemcpyHostToDevice, h->stream));
    ICG_CUDA(cudaMemcpyAsync(h->d_init, hi, sizeof(float) * 2 * n, cudaMemcpyHostToDevice, h->stream));
    rc = launch_track(h, n, h->d_slots, h->d_prev, h->d_init, h->d_fwd, h->d_bwd, h->d_status, (err && mode == 0) ? h->d_err : nullptr, mode,
                      n_levels, max_iter, eps, flags, (mode == 1 || err != nullptr) ? 1 : 0);
    if (rc != ICG_OK) return rc;
    float *of = (float *) h->h_stage;
    float *ob = of + 2 * n;
    float *oe = ob + 2 * n;
    uint8_t *os = (uint8_t *) (oe + n);
    ICG_CUDA(cudaMemcpyAsync(of, h->d_fwd, sizeof(float) * 2 * n, cudaMemcpyDeviceToHost, h->stream));
    if (mode == 1) ICG_CUDA(cudaMemcpyAsync(ob, h->d_bwd, sizeof(float) * 2 * n, cudaMemcpyDeviceToHost, h->stream));
    if (err && mode == 0) ICG_CUDA(cudaMemcpyAsync(oe, h->d_err, sizeof(float) * n, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaMemcpyAsync(os, h->d_status, n, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    memcpy(next_xy, of, sizeof(float) * 2 * n);
    if (mode == 1 && back_xy) memcpy(back_xy, ob, sizeof(float) * 2 * n);
    if (err) {
        if (mode == 0)
            memcpy(err, oe, sizeof(float) * n);
        else
            memset(err, 0, sizeof(float) * n);
    }
    memcpy(status, os, n);
    return ICG_OK;
}

int icg_klt_calc_optical_flow_pyr_lk(icg_klt *h, const uint8_t *prev, const uint8_t *next, int stride, const float *prev_xy,
                                     float *next_xy, uint8_t *status, float *err, int n, int win, int max_level, int max_iter,
                                     double eps, int flags) {
    if (win != KLT_WIN || max_level < 0 || max_level > KLT_LEVELS - 1) {
        set_error("calcOpticalFlowPyrLK: only winSize 21 and maxLevel 0..3 are built (got win=%d maxLevel=%d)", win, max_level);
        return ICG_EUNSUPPORTED;
    }
    if (!h) return ICG_EINVAL;
    const int n_levels = h->n_levels < max_level + 1 ? h->n_levels : max_level + 1;
    return host_track(h, prev, next, stride, prev_xy, next_xy, nullptr, status, err, n, 0, n_levels, max_iter, eps, flags);
}

int icg_klt_track_fb(icg_klt *h, const uint8_t *prev, const uint8_t *next, int stride, const float *prev_xy, float *next_xy,
                     float *back_xy, uint8_t *status, int n) {
    if (!h) return ICG_EINVAL;
    return host_track(h, prev, next, stride, prev_xy, next_xy, back_xy, status, nullptr, n, 1, h->n_levels, 30, 0.01,
                      ICG_OPTFLOW_USE_INITIAL_FLOW);
}

}  // extern "C"
