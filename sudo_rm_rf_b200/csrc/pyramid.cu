// The depthwise pyramid of a U-ConvBlock in ONE pass over the projection output.
//
// Reference: UConvBlock.forward, improved_sudormrf.py:205-216 (GC: groupcomm_sudormrf_v2.py:405-418):
//     u   = PReLU(GLN(proj(x)))
//     z_0 = dw5_s1(u),  z_d = dw5_s2(GLN(z_{d-1}))      d = 1 .. D-1
//     m   = sum_d up_{2^d}(GLN(z_d))
// Every GLN needs statistics over a whole sample, so kernel-per-level was a chain of D + 1 global passes
// (dw_0 .. dw_{D-1}, merge) in which the small levels ran at 0.35 - 0.63 of the HBM roofline.
//
// Observation: only u is non-linear.  For d >= 1 the level input GLN(z_{d-1}) = A z_{d-1} + B is AFFINE per
// (sample, channel), and the depthwise convolution is linear, so
//     z_d[t] = alpha_d * R_d[t] + kappa_d(t),      R_d = dw_s2_raw(R_{d-1}),  R_0 = z_0
// where R_d is the chain of RAW convolutions (no bias, no normalisation) and kappa_d(t) is a per-(sample, channel)
// constant except at the positions whose window touches the zero padding (t = 0, 1 and t = L_d - 1).  The chain of
// raw convolutions needs NO statistics, so one kernel (`dw_pyramid_kernel`) reads y once, keeps a row of every level in
// shared memory and writes z_0, R_1 .. R_{D-1} plus, per (row, level): sum R, sum R^2, R[0], R[1], R[L_d - 1].
// From those a tiny kernel (`pyramid_solve_kernel`, one CTA per sample) reproduces every GlobLN exactly:
//     sum z_d   = sum_c alpha sum R + sum_t kappa(t)
//     sum z_d^2 = sum_c alpha^2 sum R^2 + 2 alpha sum_t R kappa + sum_t kappa^2
// and emits, per (sample, channel), the coefficients of the merge, which is again affine in the raw tensors:
//     m[t] = sum_d P_d R_d[t >> d] + Q(t),   Q(t) = Q_int + edge corrections at t >> d in {0, 1, L_d - 1}.
// `merge_pyramid_kernel` evaluates that (and accumulates the statistics of m for final_norm).
// Written out, z_0 and R_d are 1.94 tensors of y's size (D = 5) that the merge reads straight back.  The forward
// therefore runs the fused stage instead (`launch_pyramid_fused`): dw_pyramid_kernel<.., kPyrStats> reads y and keeps
// only the statistics, the solve runs, and dw_pyramid_kernel<.., kPyrMerge> reads y again, rebuilds the same chain
// with the same instructions and evaluates the merge from the registers that hold a lane's 16 positions of every
// level.  Traffic per block at the benchmark shape: y twice + m = 0.63 GB instead of y + 2 x levels + m = 1.23 GB,
// still 3 launches instead of D + 1.  Shapes outside the fast path (D < 4, rows longer than the shared-memory budget,
// L_d < 6) keep the per-level kernels in levels.cu.
#include <cstring>
#include <type_traits>
#include "common.cuh"

namespace sdr {

constexpr int kPyrMaxDepth = kMaxDepthApi;
constexpr int kRowStat = 5;                 // sum R, sum R^2, R[0], R[1], R[L_d - 1]
// merge coefficient table per (sample, channel): [P_0 P_1 P_2 P_3 | Q_int P_4 .. P_{D-1} | (dq0, dq1, dqr) for d = 1 .. D-1],
// padded to a multiple of 4 floats (the merge reads the first 8 as two float4)
__host__ __device__ constexpr int pyr_table_width(int D) { return (4 * D - 2 + 3) & ~3; }
__host__ __device__ constexpr int pyr_p_index(int D, int d) { return d < 4 ? d : d + 1; }      // P_d
__host__ __device__ constexpr int pyr_q_index() { return 4; }                                   // Q_int
__host__ __device__ constexpr int pyr_dq_index(int D, int d) { return D + 1 + 3 * (d - 1); }   // dq0 of level d

struct PyrArgs {
    const float* y;                 // projection output [rows][L] (raw)
    NormIn nin;                     // its GlobLN (+PReLU): statistics per sample, gamma/beta per channel
    const float* w[kPyrMaxDepth];   // depthwise taps of level d: [C][5]
    const float* bias0;             // bias of level 0: [C]
    float* z[kPyrMaxDepth];         // z[0] = z_0 (raw, with bias), z[d] = R_d (raw convolution chain)
    double* stats0;                 // per-sample (sum, sumsq) of z_0
    double* rowstats;               // [samples][D - 1][C][kRowStat]: a (sample, level) block is contiguous for the solve
    const float* table;             // kPyrMerge: the solve's merge coefficients [rows][pyr_table_width(D)]
    float* m;                       // kPyrMerge: the merged output [rows][L]; may be y itself
    double* stats_m;                // kPyrMerge: per-sample (sum, sumsq) of m
    int D, C, L, rows;
};

// What one pass of dw_pyramid_kernel leaves in HBM.  kPyrLevels: z_0, R_1 .. R_{D-1}, their row statistics and the
// statistics of z_0 (read by sdr_merge_pyramid).  The fused stage runs two passes over y instead and never writes the
// levels: kPyrStats keeps only the statistics, the solve turns them into the merge table, and kPyrMerge rebuilds the
// same pyramid bit for bit and evaluates the merge from the registers that hold it (m and its statistics).
enum PyrMode : int { kPyrLevels = 0, kPyrStats = 1, kPyrMerge = 2 };

// One CTA per row, one WARP per 512-position window of the row, the whole pyramid of the window in REGISTERS:
// lane l owns 16 consecutive positions of level 0 (its u, z_0), 8 of R_1, 4 of R_2, 2 of R_3, 1 of R_4 (and, for
// D = 6, every second lane one of R_5); the two-left / one-right halo of every stride-2 level comes from the
// neighbouring lanes by shuffle.  No shared-memory staging, no barrier between levels (the first version kept rows in
// shared memory with a barrier per level and was instruction-bound: 8.9 k warp instructions per row, 73 % issue
// utilisation in ncu; this formulation needs about a third).  Windows overlap: a window's first 2^D (32, or 64 for
// D = 6) and last 32 level-0 positions only feed the halos of the deeper levels, each window stores and counts the
// 448 (416) positions in between, so every output is produced exactly once from exact inputs.
constexpr int kWin = 512;                   // level-0 positions per warp window
template <int D> struct PyrGeom {
    static constexpr int kLeft = 2 << (D - 1);          // two inexact entries at the left of the deepest level (whole lanes)
    static constexpr int kRight = D <= 5 ? 16 : 32;     // one inexact entry at the right
    static constexpr int kStep = kWin - kLeft - kRight; // valid positions per window: 480 / 464 / 416, multiples of 2^(D-1)
};

// Sums NV per-lane values over the warp with NV + NV/2 + ... shuffles instead of 5 NV: at every butterfly step a lane
// keeps one half of its values (adding the partner's copies) and hands the other half over.  Afterwards v[0] of lane
// `l` is the warp total of value warp_multi_owner<NV>(l).
// value index whose warp total ends in v[0] of `lane` after warp_multi_sum<NV> (-1: a replica), NV = 2 D = 8 / 10 / 12
// (derived by simulating the butterfly; checked by test_depthwise_pyramid's statistics)
template <int NV> __device__ __forceinline__ int warp_multi_owner(int lane) {
    if (NV == 8) return (lane & 3) == 0 ? lane >> 2 : -1;
    if (NV == 10) {
        switch (lane) {
            case 0: return 0; case 4: return 1; case 8: return 2; case 12: return 3; case 2: return 4;
            case 16: return 5; case 20: return 6; case 24: return 7; case 28: return 8; case 18: return 9;
            default: return -1;
        }
    }
    switch (lane) {   // NV == 12
        case 0: return 0; case 4: return 1; case 2: return 2; case 8: return 3; case 12: return 4; case 10: return 5;
        case 16: return 6; case 20: return 7; case 18: return 8; case 24: return 9; case 28: return 10; case 26: return 11;
        default: return -1;
    }
}
template <int NV>
__device__ __forceinline__ void warp_multi_sum(float (&v)[NV], int lane) {
    // step widths: 16, 8, 4, 2, 1 ; n = number of live values
    int n = NV;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const bool up = (lane & off) != 0;
        const int half = n / 2;                         // pairs (i, i + half) are split between the two partner lanes
#pragma unroll
        for (int i = 0; i < NV / 2; ++i) {
            if (i < half) {
                const float keep = up ? v[i + half] : v[i];
                const float send = up ? v[i] : v[i + half];
                v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
            }
        }
        if (n & 1) {                                    // odd one out: plain butterfly, stays replicated
            v[half] = v[n - 1] + __shfl_xor_sync(0xffffffffu, v[n - 1], off);
        }
        n = half + (n & 1);
    }
}
__device__ __forceinline__ uint32_t pyr_smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void pyr_mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(pyr_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void pyr_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(pyr_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void pyr_mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = pyr_smem_u32(bar);
    uint32_t done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    } while (!done);
}
__device__ __forceinline__ void pyr_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(pyr_smem_u32(dst)), "l"(src), "r"(bytes), "r"(pyr_smem_u32(bar)) : "memory");
}

// Persistent CTAs: rows blockIdx.x, + gridDim.x, ...  The NEXT row's y arrives by 1-D bulk TMA into the other half of
// a double buffer and its per-row parameters by 4-byte cp.async while the current row is computed, so no thread ever
// waits on a global load (one CTA per row with plain loads measured 1.7 us per row and SM: launch-to-first-use
// latency of y, of the 28 parameters and of the fp64 statistics in every CTA).  One barrier per row.
#ifndef SDR_PYR_MINB
#define SDR_PYR_MINB 6                  // resident CTAs per SM the <= 256-thread instantiation is compiled for
#endif
#ifndef SDR_PYR_STATS_MINB
#define SDR_PYR_STATS_MINB 5            // the same for kPyrStats (at 6, 40 registers, the per-channel-slope D = 6 one spills)
#endif
#ifndef SDR_PYR_MERGE_MINB
#define SDR_PYR_MERGE_MINB 4            // the same for kPyrMerge, which holds every level of its 16 positions live at once
#endif                                  // (64 registers; at 5 it spills)
// PC: one PReLU slope per channel (the original model's nn.PReLU(C), sudormrf.py:33): a row is one channel, so the
// slope simply travels with the row's other parameters; the shared-slope instantiations are unchanged.
template <int D, int MAXT, int MINB, bool PC, int MODE = kPyrLevels>
__global__ void __launch_bounds__(MAXT, MINB)
dw_pyramid_kernel(const PyrArgs a) {
    static_assert(D >= 4 && D <= 6, "register pyramid: levels 0..3 by lane chunks, 4 per lane, 5 per lane pair");
    constexpr int S = PyrGeom<D>::kStep, ML = PyrGeom<D>::kLeft;
    constexpr bool kMerge = MODE == kPyrMerge;
    constexpr int NP = 5 * D + 3 + (PC ? 1 : 0);            // per-row parameters ...
    constexpr int TW = pyr_table_width(D);                  // ... followed, for the merge, by the row's table
    extern __shared__ __align__(16) float pyr_smem[];       // [2][L + 8]: raw rows of y with 4 floats of slack on either side
    __shared__ float s_par[2][NP + (kMerge ? TW : 0)];      // taps of every level, bias_0, gamma_y, beta_y (one row ahead) [, slope] [, table]
    __shared__ float s_part[2][32][kMerge ? 1 : 2 * D];
    __shared__ double s_mst[2][32][kMerge ? 2 : 1];         // kPyrMerge: per-warp (sum, sumsq) of m
    __shared__ __align__(8) uint64_t s_bar[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int L = a.L;
    const int LB = L + 8;
    float2* s_mr = reinterpret_cast<float2*>(pyr_smem + 2 * (size_t)LB);   // [samples] (mean, rstd) of y
    const int samples = a.rows / a.C;
    const uint32_t row_bytes = (uint32_t)L * sizeof(float);
    const bool act = a.nin.prelu != nullptr;
    float slope = (act && !PC) ? __ldg(a.nin.prelu) : 1.f;
    bool sle1 = slope <= 1.f;

    auto stage_params = [&](int row, int slot) {
        for (int i = tid; i < NP + (kMerge ? TW : 0); i += blockDim.x) {
            const int c = row % a.C;
            const float* src;
            if (kMerge && i >= NP) src = a.table + (size_t)row * TW + (i - NP);
            else if (i < 5 * D) src = a.w[i / 5] + c * 5 + (i % 5);
            else if (i == 5 * D) src = a.bias0 + c;
            else if (i == 5 * D + 1) src = a.nin.stats ? a.nin.gamma + c : a.bias0 + c;
            else if (PC && i == 5 * D + 3) src = act ? a.nin.prelu + c : a.bias0 + c;
            else src = a.nin.stats ? a.nin.beta + c : a.bias0 + c;
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(pyr_smem_u32(&s_par[slot][i])), "l"(src) : "memory");
        }
    };
    for (int sidx = tid; sidx < samples; sidx += blockDim.x) {
        const SampleNorm sn = sample_norm(a.nin, sidx);
        s_mr[sidx] = make_float2(sn.mean, sn.rstd);
    }
    if (tid < 8) {                                          // the slack around both row buffers reads as zero
        pyr_smem[tid < 4 ? tid : L + tid] = 0.f;
        pyr_smem[LB + (tid < 4 ? tid : L + tid)] = 0.f;
    }
    if (tid == 0) {
        pyr_mbar_init(&s_bar[0], 1);
        pyr_mbar_init(&s_bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        if ((int)blockIdx.x < a.rows) {
            pyr_mbar_expect_tx(&s_bar[0], row_bytes);
            pyr_bulk_g2s(pyr_smem + 4, a.y + (size_t)blockIdx.x * L, row_bytes, &s_bar[0]);
        }
    }
    if ((int)blockIdx.x < a.rows) stage_params(blockIdx.x, 0);
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();

    const int w0 = warp * S - ML;
    const int g0 = w0 + 16 * lane;
    const bool inrow = g0 >= 0 && g0 < L;                   // L % 16 == 0: a chunk is entirely inside or outside the row
    const bool valid = inrow && g0 >= warp * S && g0 < (warp + 1) * S;   // stored and counted by this window
    const bool in_l = g0 - 2 >= 0 && g0 - 2 < L, in_r = g0 + 16 >= 0 && g0 + 16 < L;

    uint32_t it = 0;
#pragma unroll 1
    for (int row = blockIdx.x; row < a.rows; row += gridDim.x, ++it) {
    const int sample = row / a.C;
    const int cur = it & 1;
    if (tid == 0) {
        const int nxt = row + gridDim.x;
        if (nxt < a.rows) {
            pyr_mbar_expect_tx(&s_bar[cur ^ 1], row_bytes);
            pyr_bulk_g2s(pyr_smem + (size_t)(cur ^ 1) * LB + 4, a.y + (size_t)nxt * L, row_bytes, &s_bar[cur ^ 1]);
        }
    }
    if (row + (int)gridDim.x < a.rows) stage_params(row + gridDim.x, cur ^ 1);
    const float* par = s_par[cur];
    float na = 1.f, nb = 0.f;
    if (a.nin.stats) { const float2 mr = s_mr[sample]; na = par[5 * D + 1] * mr.y; nb = fmaf(-mr.x, na, par[5 * D + 2]); }
    if constexpr (PC) { if (act) { slope = par[5 * D + 3]; sle1 = slope <= 1.f; } }      // this row's (channel's) own slope
    pyr_mbar_wait(&s_bar[cur], (it >> 1) & 1);

    // y[g0-2 .. g0+17] from the row buffer (index 4 + position), then u = PReLU(GLN(y)), 0 outside the row
    float u[20];
#pragma unroll
    for (int i = 0; i < 20; ++i) u[i] = 0.f;
    {
        const float* yb = pyr_smem + (size_t)cur * LB + 4;
        if (inrow) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float4 v = *reinterpret_cast<const float4*>(yb + g0 + 4 * k);
                u[2 + 4 * k] = v.x; u[3 + 4 * k] = v.y; u[4 + 4 * k] = v.z; u[5 + 4 * k] = v.w;
            }
        }
        if (in_l) { const float2 h = *reinterpret_cast<const float2*>(yb + g0 - 2); u[0] = h.x; u[1] = h.y; }
        if (in_r) { const float2 h = *reinterpret_cast<const float2*>(yb + g0 + 16); u[18] = h.x; u[19] = h.y; }
    }
    // (uniform branches: the slope's side of 1 and the row-edge lanes are decided once, not per element)
    if (!act) {
#pragma unroll
        for (int i = 0; i < 20; ++i) u[i] = fmaf(u[i], na, nb);
    } else if (sle1) {
#pragma unroll
        for (int i = 0; i < 20; ++i) { const float t = fmaf(u[i], na, nb); u[i] = fmaxf(t, t * slope); }
    } else {
#pragma unroll
        for (int i = 0; i < 20; ++i) { const float t = fmaf(u[i], na, nb); u[i] = fminf(t, t * slope); }
    }
    if (!(inrow && in_l && in_r)) {                         // zero padding applies to u (not to y): exactly 0 outside the row
        if (!in_l) { u[0] = 0.f; u[1] = 0.f; }
        if (!in_r) { u[18] = 0.f; u[19] = 0.f; }
        if (!inrow) {
#pragma unroll
            for (int i = 2; i < 18; ++i) u[i] = 0.f;
        }
    }

    float part[2 * D];
#pragma unroll
    for (int i = 0; i < 2 * D; ++i) part[i] = 0.f;
    const int c_row = row - sample * a.C;
    double* rs = a.rowstats + ((size_t)sample * (D - 1) * a.C + c_row) * kRowStat;   // level 1; level d at + (d - 1) * rsl
    const size_t rsl = (size_t)a.C * kRowStat;

    // ---- level 0 ----
    float z0[16];
    {
        const float w0_ = par[0], w1_ = par[1], w2_ = par[2], w3_ = par[3], w4_ = par[4], b0 = par[5 * D];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            float acc = fmaf(w0_, u[i], b0);
            acc = fmaf(w1_, u[i + 1], acc);
            acc = fmaf(w2_, u[i + 2], acc);
            acc = fmaf(w3_, u[i + 3], acc);
            acc = fmaf(w4_, u[i + 4], acc);
            z0[i] = acc;
        }
        if (!inrow) {                                       // zero padding of level 1's input
#pragma unroll
            for (int i = 0; i < 16; ++i) z0[i] = 0.f;
        }
        if (valid && !kMerge) {
            if constexpr (MODE == kPyrLevels) {
                float* zr = a.z[0] + (size_t)row * L + g0;
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    *reinterpret_cast<float4*>(zr + 4 * k) = make_float4(z0[4 * k], z0[4 * k + 1], z0[4 * k + 2], z0[4 * k + 3]);
            }
#pragma unroll
            for (int i = 0; i < 16; ++i) { part[0] += z0[i]; part[1] = fmaf(z0[i], z0[i], part[1]); }
        }
    }
    // one stride-2 level held as N = 16 >> d values per lane, from the 2N values of the level above
    auto level = [&](auto n_tag, const float* prev, float* cur, int d) {
        constexpr int N = decltype(n_tag)::value;
        const float hl0 = __shfl_up_sync(0xffffffffu, prev[2 * N - 2], 1), hl1 = __shfl_up_sync(0xffffffffu, prev[2 * N - 1], 1);
        const float hr = __shfl_down_sync(0xffffffffu, prev[0], 1);
        float v[2 * N + 3];
        v[0] = hl0; v[1] = hl1; v[2 * N + 2] = hr;          // (the window's end lanes compute inexact, never-stored entries)
#pragma unroll
        for (int i = 0; i < 2 * N; ++i) v[2 + i] = prev[i];
        const float* w = par + 5 * d;
        const float w0_ = w[0], w1_ = w[1], w2_ = w[2], w3_ = w[3], w4_ = w[4];
#pragma unroll
        for (int i = 0; i < N; ++i) {
            float acc = w0_ * v[2 * i];
            acc = fmaf(w1_, v[2 * i + 1], acc);
            acc = fmaf(w2_, v[2 * i + 2], acc);
            acc = fmaf(w3_, v[2 * i + 3], acc);
            acc = fmaf(w4_, v[2 * i + 4], acc);
            cur[i] = acc;
        }
        if (!inrow) {
#pragma unroll
            for (int i = 0; i < N; ++i) cur[i] = 0.f;
        }
        if (valid && !kMerge) {
            if constexpr (MODE == kPyrLevels) {
                const int Ld = L >> d;
                float* rr = a.z[d] + (size_t)row * Ld + (g0 >> d);
                if constexpr (N >= 4) {
#pragma unroll
                    for (int k = 0; k < N / 4; ++k)
                        *reinterpret_cast<float4*>(rr + 4 * k) = make_float4(cur[4 * k], cur[4 * k + 1], cur[4 * k + 2], cur[4 * k + 3]);
                } else if constexpr (N == 2) {
                    *reinterpret_cast<float2*>(rr) = make_float2(cur[0], cur[1]);
                } else {
                    rr[0] = cur[0];
                }
            }
#pragma unroll
            for (int i = 0; i < N; ++i) { part[2 * d] += cur[i]; part[2 * d + 1] = fmaf(cur[i], cur[i], part[2 * d + 1]); }
            if constexpr (N >= 2) {
                if (g0 == 0) { rs[(d - 1) * rsl + 2] = (double)cur[0]; rs[(d - 1) * rsl + 3] = (double)cur[1]; }
            } else {
                if (g0 == 0) rs[(d - 1) * rsl + 2] = (double)cur[0];
                if (g0 == 16) rs[(d - 1) * rsl + 3] = (double)cur[0];
            }
            if (g0 + 16 == L) rs[(d - 1) * rsl + 4] = (double)cur[N - 1];
        }
    };
    float r1[8], r2[4], r3[2], r4[1], r5 = 0.f;
    level(std::integral_constant<int, 8>{}, z0, r1, 1);
    level(std::integral_constant<int, 4>{}, r1, r2, 2);
    level(std::integral_constant<int, 2>{}, r2, r3, 3);
    if constexpr (D >= 5) level(std::integral_constant<int, 1>{}, r3, r4, 4);
    if constexpr (D == 6) {
        // level 5: one entry per lane pair (32 level-0 positions), held by the even lane: R_5[e] from R_4 of lanes 2e-2 .. 2e+2
        const float m2 = __shfl_up_sync(0xffffffffu, r4[0], 2), m1 = __shfl_up_sync(0xffffffffu, r4[0], 1);
        const float p1 = __shfl_down_sync(0xffffffffu, r4[0], 1), p2 = __shfl_down_sync(0xffffffffu, r4[0], 2);
        const float* w = par + 25;
        float acc = w[0] * m2;
        acc = fmaf(w[1], m1, acc);
        acc = fmaf(w[2], r4[0], acc);
        acc = fmaf(w[3], p1, acc);
        acc = fmaf(w[4], p2, acc);
        if constexpr (kMerge) {
            r5 = __shfl_sync(0xffffffffu, acc, lane & ~1);  // the odd lane's 16 outputs read the same entry
        } else if (valid && (lane & 1) == 0) {              // S and the window origin are multiples of 32: the pair is valid together
            if constexpr (MODE == kPyrLevels) a.z[5][(size_t)row * (L >> 5) + (g0 >> 5)] = acc;
            part[10] += acc;
            part[11] = fmaf(acc, acc, part[11]);
            if (g0 == 0) rs[4 * rsl + 2] = (double)acc;
            if (g0 == 32) rs[4 * rsl + 3] = (double)acc;
            if (g0 + 32 == L) rs[4 * rsl + 4] = (double)acc;
        }
    }

    // ---- kPyrMerge: m[t] = sum_d P_d R_d[t >> d] + Q(t) over the lane's 16 positions, in merge_pyramid_kernel's order
    // (coarse to fine, then the edge corrections), so m is bitwise what the level-writing pair computes ----
    StatAcc macc;
    if constexpr (kMerge) {
        if (valid) {
            const float* tb = par + NP;
            const int q = g0 >> 4, QR = L >> 4;
            const int left_runs = (2 << (D - 1)) >> 4, right_runs = ((1 << (D - 1)) + 15) >> 4;
            float base = tb[pyr_q_index()];
            if constexpr (D > 4) base = fmaf(r4[0], tb[pyr_p_index(D, 4)], base);
            if constexpr (D > 5) base = fmaf(r5, tb[pyr_p_index(D, 5)], base);
            const float p0 = tb[pyr_p_index(D, 0)], p1 = tb[pyr_p_index(D, 1)];
            const float p2 = tb[pyr_p_index(D, 2)], p3 = tb[pyr_p_index(D, 3)];
            float s3[2], s2[4], s1[8], o[16];
            s3[0] = fmaf(r3[0], p3, base); s3[1] = fmaf(r3[1], p3, base);
#pragma unroll
            for (int i = 0; i < 4; ++i) s2[i] = fmaf(r2[i], p2, s3[i >> 1]);
#pragma unroll
            for (int i = 0; i < 8; ++i) s1[i] = fmaf(r1[i], p1, s2[i >> 1]);
#pragma unroll
            for (int i = 0; i < 16; ++i) o[i] = fmaf(z0[i], p0, s1[i >> 1]);
            if (q < left_runs || q >= QR - right_runs) {
#pragma unroll 1
                for (int d = 1; d < D; ++d) {
                    const float dq0 = tb[pyr_dq_index(D, d)], dq1 = tb[pyr_dq_index(D, d) + 1], dqr = tb[pyr_dq_index(D, d) + 2];
                    const int last = (L >> d) - 1;
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const int idx = (16 * q + i) >> d;
                        o[i] += idx == 0 ? dq0 : (idx == 1 ? dq1 : 0.f);
                        o[i] += idx == last ? dqr : 0.f;
                    }
                }
            }
            float* mr = a.m + (size_t)row * L + g0;         // (in place over y: this row is already in shared memory)
#pragma unroll
            for (int k = 0; k < 4; ++k)
                *reinterpret_cast<float4*>(mr + 4 * k) = make_float4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]);
            macc.add_run(o);
        }
    }

    // ---- row sums of every level, or of m (s_part / s_mst alternate between rows: one barrier per row) ----
    if constexpr (kMerge) {
        const double ms = warp_sum_f64(macc.s), mq = warp_sum_f64(macc.q);
        if (lane == 0) { s_mst[cur][warp][0] = ms; s_mst[cur][warp][1] = mq; }
    } else {
        warp_multi_sum<2 * D>(part, lane);
        const int own = warp_multi_owner<2 * D>(lane);
        if (own >= 0) s_part[cur][warp][own] = part[0];
    }
    asm volatile("cp.async.wait_all;" ::: "memory");        // the next row's parameters (issued at the top of this row)
    __syncthreads();
    if constexpr (kMerge) {
        if (tid < 2) {
            const int nw = blockDim.x >> 5;
            double tot = 0.0;
            for (int wv = 0; wv < nw; ++wv) tot += s_mst[cur][wv][tid];
            atomicAdd(a.stats_m + 2 * (size_t)sample + tid, tot);
        }
    } else if (tid < 2 * D) {
        const int nw = blockDim.x >> 5;
        double tot = 0.0;
        for (int wv = 0; wv < nw; ++wv) tot += (double)s_part[cur][wv][tid];
        if (tid < 2) atomicAdd(a.stats0 + 2 * (size_t)sample + tid, tot);
        else rs[(size_t)(tid / 2 - 1) * rsl + (tid & 1)] = tot;
    }
    }   // rows
}

// ---------------------------------------------------------------------------
// solve: one CTA per sample walks the levels, reproducing every GlobLN from the row statistics
// ---------------------------------------------------------------------------
struct SolveArgs {
    const double* stats0;           // per-sample (sum, sumsq) of z_0
    const double* rowstats;         // [samples][D - 1][C][kRowStat]
    const float* gamma[kPyrMaxDepth];   // GlobLN of level d's OUTPUT (spp_dw[d].norm)
    const float* beta[kPyrMaxDepth];
    const float* w[kPyrMaxDepth];       // taps of level d
    const float* bias[kPyrMaxDepth];    // bias of level d
    float* table;                   // [rows][pyr_table_width(D)]
    int D, C, L;
};

constexpr int kSolveThreads = 256;
constexpr int kSolveKC = 2;                 // channels per thread: C <= 512 (wider layers take the per-level kernels)

// Everything a level needs is loaded one level ahead into registers (row statistics of level d + 1, and the norm /
// tap parameters used after level d's reduction), so a level costs its arithmetic and two barriers instead of three
// dependent L2 round trips (22.7 us per launch in the first version, as much as 12 % of the pyramid itself).
__global__ void __launch_bounds__(kSolveThreads)
pyramid_solve_kernel(const SolveArgs a) {
    __shared__ double s_red[2][kSolveThreads / 32];
    __shared__ double s_mean, s_rstd;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int sample = blockIdx.x;
    const int D = a.D, C = a.C;
    const int TW = pyr_table_width(D);

    auto block_norm = [&](double sz, double sq, double count) {   // all threads call; result in s_mean / s_rstd
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { sz += __shfl_xor_sync(0xffffffffu, sz, o); sq += __shfl_xor_sync(0xffffffffu, sq, o); }
        if (lane == 0) { s_red[0][warp] = sz; s_red[1][warp] = sq; }
        __syncthreads();
        if (tid == 0) {
            double ts = 0.0, tq = 0.0;
            for (int wv = 0; wv < kSolveThreads / 32; ++wv) { ts += s_red[0][wv]; tq += s_red[1][wv]; }
            const double mu = ts / count;
            double var = tq / count - mu * mu;
            var = var < 0.0 ? 0.0 : var;
            s_mean = mu;
            s_rstd = 1.0 / sqrt(var + (double)kGlnEps);
        }
        __syncthreads();
    };
    struct After { float g, be, w[5], bias; };              // used after level d's reduction: gamma_d, beta_d, taps / bias of level d + 1
    auto load_after = [&](int d, int c) -> After {
        After r;
        r.g = __ldg(a.gamma[d] + c); r.be = __ldg(a.beta[d] + c);
        if (d + 1 < D) {
            const float* w = a.w[d + 1] + c * 5;
#pragma unroll
            for (int j = 0; j < 5; ++j) r.w[j] = __ldg(w + j);
            r.bias = __ldg(a.bias[d + 1] + c);
        } else {
#pragma unroll
            for (int j = 0; j < 5; ++j) r.w[j] = 0.f;
            r.bias = 0.f;
        }
        return r;
    };
    struct Rs { double v[kRowStat]; };
    auto load_rs = [&](int d, int c) -> Rs {                  // row statistics of level d (d >= 1)
        Rs r;
        const double* p = a.rowstats + (((size_t)sample * (D - 1) + (d - 1)) * C + c) * kRowStat;
#pragma unroll
        for (int k = 0; k < kRowStat; ++k) r.v[k] = p[k];
        return r;
    };

    // per-channel state: alpha, k0, k1, kint, kr of the level about to be reduced, and the Q accumulator
    double al[kSolveKC], k0[kSolveKC], k1[kSolveKC], ki[kSolveKC], kr[kSolveKC], qa[kSolveKC];
    Rs rs[kSolveKC];
    After af[kSolveKC];
#pragma unroll
    for (int k = 0; k < kSolveKC; ++k) {
        const int c = tid + k * kSolveThreads;
        if (c < C) { af[k] = load_after(0, c); rs[k] = load_rs(1, c); }
    }
    if (tid == 0) {                                         // level 0: statistics measured directly
        const double cnt = (double)C * a.L;
        const double mu = a.stats0[2 * (size_t)sample] / cnt;
        double var = a.stats0[2 * (size_t)sample + 1] / cnt - mu * mu;
        var = var < 0.0 ? 0.0 : var;
        s_mean = mu;
        s_rstd = 1.0 / sqrt(var + (double)kGlnEps);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kSolveKC; ++k) {
        const int c = tid + k * kSolveThreads;
        if (c < C) {
            const double A0 = (double)af[k].g * s_rstd;
            const double B0 = (double)af[k].be - s_mean * A0;
            a.table[((size_t)sample * C + c) * TW + pyr_p_index(D, 0)] = (float)A0;
            // z_1 = alpha R_1 + kappa_1(t):  alpha = A0, kappa = B0 * (sum of in-bounds taps of level 1) + bias_1
            const double w0 = af[k].w[0], w1 = af[k].w[1], w2 = af[k].w[2], w3 = af[k].w[3], w4 = af[k].w[4];
            const double b1 = af[k].bias;
            al[k] = A0;
            k0[k] = B0 * (w2 + w3 + w4) + b1;               // t = 0: taps 0, 1 fall on the padding
            ki[k] = B0 * (w0 + w1 + w2 + w3 + w4) + b1;     // interior
            k1[k] = ki[k];                                  // t = 1 is interior at level 1
            kr[k] = B0 * (w0 + w1 + w2 + w3) + b1;          // t = L_1 - 1: tap 4 falls on the padding
            qa[k] = B0;                                     // sum_d (A_d kint_d + B_d), kint_0 = 0
        }
    }

    for (int d = 1; d < D; ++d) {
        const int Ld = a.L >> d;
        double sz = 0.0, sq = 0.0;
        Rs rn[kSolveKC];
#pragma unroll
        for (int k = 0; k < kSolveKC; ++k) {
            const int c = tid + k * kSolveThreads;
            if (c < C) {
                af[k] = load_after(d, c);                   // consumed after the reduction below
                if (d + 1 < D) rn[k] = load_rs(d + 1, c);   // consumed in the next iteration
                const double sR = rs[k].v[0], sR2 = rs[k].v[1], R0 = rs[k].v[2], R1 = rs[k].v[3], Rl = rs[k].v[4];
                sz += al[k] * sR + (double)(Ld - 3) * ki[k] + k0[k] + k1[k] + kr[k];
                sq += al[k] * al[k] * sR2
                      + 2.0 * al[k] * (ki[k] * sR + (k0[k] - ki[k]) * R0 + (k1[k] - ki[k]) * R1 + (kr[k] - ki[k]) * Rl)
                      + (double)(Ld - 3) * ki[k] * ki[k] + k0[k] * k0[k] + k1[k] * k1[k] + kr[k] * kr[k];
            }
        }
        block_norm(sz, sq, (double)C * Ld);
#pragma unroll
        for (int k = 0; k < kSolveKC; ++k) {
            const int c = tid + k * kSolveThreads;
            if (c < C) {
                const double Ad = (double)af[k].g * s_rstd;
                const double Bd = (double)af[k].be - s_mean * Ad;
                float* tb = a.table + ((size_t)sample * C + c) * TW;
                tb[pyr_p_index(D, d)] = (float)(Ad * al[k]);
                tb[pyr_dq_index(D, d) + 0] = (float)(Ad * (k0[k] - ki[k]));
                tb[pyr_dq_index(D, d) + 1] = (float)(Ad * (k1[k] - ki[k]));
                tb[pyr_dq_index(D, d) + 2] = (float)(Ad * (kr[k] - ki[k]));
                qa[k] += Ad * ki[k] + Bd;
                if (d + 1 < D) {                            // z_{d+1} = (Ad alpha) R_{d+1} + Ad conv(kappa_d) + Bd S(t) + bias
                    const double w0 = af[k].w[0], w1 = af[k].w[1], w2 = af[k].w[2], w3 = af[k].w[3], w4 = af[k].w[4];
                    const double bn = af[k].bias;
                    const double S = w0 + w1 + w2 + w3 + w4;
                    const double c0 = w2 * k0[k] + w3 * k1[k] + w4 * ki[k];              // window -2 .. 2
                    const double c1 = w0 * k0[k] + w1 * k1[k] + (w2 + w3 + w4) * ki[k];  // window 0 .. 4
                    const double ci = S * ki[k];
                    const double cr = (w0 + w1 + w2) * ki[k] + w3 * kr[k];               // window L_d - 4 .. L_d
                    al[k] = Ad * al[k];
                    k0[k] = Ad * c0 + Bd * (w2 + w3 + w4) + bn;
                    k1[k] = Ad * c1 + Bd * S + bn;
                    ki[k] = Ad * ci + Bd * S + bn;
                    kr[k] = Ad * cr + Bd * (w0 + w1 + w2 + w3) + bn;
                    rs[k] = rn[k];
                }
            }
        }
        // (block_norm's first barrier of the next level orders the reads of s_mean / s_rstd above before they are rewritten)
    }
#pragma unroll
    for (int k = 0; k < kSolveKC; ++k) {
        const int c = tid + k * kSolveThreads;
        if (c < C) a.table[((size_t)sample * C + c) * TW + pyr_q_index()] = (float)qa[k];
    }
}

// ---------------------------------------------------------------------------
// merge: m[t] = sum_d P_d R_d[t >> d] + Q(t); 16 outputs per thread, coarse to fine; + statistics of m
// requires D >= 4 and L % 16 == 0
// ---------------------------------------------------------------------------
struct MergePyrArgs {
    const float* z[kPyrMaxDepth];
    const float* table;
    int D, C, L;
};
#ifndef SDR_MP_THREADS
#define SDR_MP_THREADS 128
#endif
#ifndef SDR_MP_ITEMS
#define SDR_MP_ITEMS 4                 // runs of 16 outputs per thread (1 / 2 / 4 on one box: 116.2 / 108.7 / 104.7 us at cfg 2; 256 threads x 1: 130.9)
#endif
constexpr int kMpThreads = SDR_MP_THREADS;
constexpr int kMpItems = SDR_MP_ITEMS;

__global__ void __launch_bounds__(kMpThreads)
merge_pyramid_kernel(const MergePyrArgs a, float* __restrict__ m, double* __restrict__ stats_out, int chunks_per_sample) {
    __shared__ double s_red[64];
    const int sample = blockIdx.x / chunks_per_sample;
    const int chunk = blockIdx.x - sample * chunks_per_sample;
    const int L = a.L, D = a.D, C = a.C;
    const int QR = L >> 4;
    const int items = C * QR;
    const int TW = pyr_table_width(D);
    const int left_runs = (2 << (D - 1)) >> 4;            // runs whose positions satisfy t >> d < 2 for some d: t < 2^D
    const int right_runs = ((1 << (D - 1)) + 15) >> 4;    // t >> d == L_d - 1 for some d: t >= L - 2^(D-1)
    StatAcc acc;
#pragma unroll
    for (int iti = 0; iti < kMpItems; ++iti) {
        const int item = (chunk * kMpItems + iti) * kMpThreads + threadIdx.x;
        if (item < items) {
            const int c = item / QR;
            const int q = item - c * QR;
            const size_t row = (size_t)sample * C + c;
            const float* z0 = a.z[0] + row * L + 16 * q;
            const float4 v00 = ldg4(z0), v01 = ldg4(z0 + 4), v02 = ldg4(z0 + 8), v03 = ldg4(z0 + 12);
            const float* z1 = a.z[1] + row * (L >> 1) + 8 * q;
            const float4 v10 = ldg4(z1), v11 = ldg4(z1 + 4);
            const float4 v2 = ldg4(a.z[2] + row * (L >> 2) + 4 * q);
            const float2 v3 = __ldg(reinterpret_cast<const float2*>(a.z[3] + row * (L >> 3) + 2 * q));
            const float* tb = a.table + row * TW;
            const float4 pp = ldg4(tb), qq = ldg4(tb + 4);     // P_0..P_3 | Q_int, P_4, P_5, P_6
            float base = qq.x;                                 // Q_int + the levels that are constant over the run
            if (D > 4) base = fmaf(__ldg(a.z[4] + row * (L >> 4) + q), qq.y, base);
            if (D > 5) base = fmaf(__ldg(a.z[5] + row * (L >> 5) + (q >> 1)), qq.z, base);
            const float p0 = pp.x, p1 = pp.y, p2 = pp.z, p3 = pp.w;
            float s3[2], s2[4], s1[8], o[16];
            s3[0] = fmaf(v3.x, p3, base); s3[1] = fmaf(v3.y, p3, base);
            const float z2v[4] = {v2.x, v2.y, v2.z, v2.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) s2[i] = fmaf(z2v[i], p2, s3[i >> 1]);
            const float z1v[8] = {v10.x, v10.y, v10.z, v10.w, v11.x, v11.y, v11.z, v11.w};
#pragma unroll
            for (int i = 0; i < 8; ++i) s1[i] = fmaf(z1v[i], p1, s2[i >> 1]);
            const float z0v[16] = {v00.x, v00.y, v00.z, v00.w, v01.x, v01.y, v01.z, v01.w,
                                   v02.x, v02.y, v02.z, v02.w, v03.x, v03.y, v03.z, v03.w};
#pragma unroll
            for (int i = 0; i < 16; ++i) o[i] = fmaf(z0v[i], p0, s1[i >> 1]);
            if (q < left_runs || q >= QR - right_runs) {   // rows' ends: the padding of a level reaches these positions
                // (kept inline: as a __noinline__ helper taking o[] by reference the run lived in local memory: 120 -> 165 us)
#pragma unroll 1
                for (int d = 1; d < D; ++d) {
                    const float dq0 = __ldg(tb + pyr_dq_index(D, d)), dq1 = __ldg(tb + pyr_dq_index(D, d) + 1);
                    const float dqr = __ldg(tb + pyr_dq_index(D, d) + 2);
                    const int last = (L >> d) - 1;
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const int idx = (16 * q + i) >> d;
                        o[i] += idx == 0 ? dq0 : (idx == 1 ? dq1 : 0.f);
                        o[i] += idx == last ? dqr : 0.f;
                    }
                }
            }
            float* mr = m + row * L + 16 * q;
#pragma unroll
            for (int i = 0; i < 4; ++i)
                *reinterpret_cast<float4*>(mr + 4 * i) = make_float4(o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
            acc.add_run(o);
        }
    }
    block_stats_atomic(acc, stats_out, sample, s_red);
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
constexpr int kPyrMaxSamples = 4096;                           // per-sample (mean, rstd) table in shared memory: 32 KB at most
static int pyramid_windows(int D, int L) {                     // warps per row
    const int step = D == 4 ? PyrGeom<4>::kStep : (D == 5 ? PyrGeom<5>::kStep : PyrGeom<6>::kStep);
    return (L + step - 1) / step;
}
// The one predicate for "the one-pass pyramid takes this block": the forward's plan (scratch and launch count), the
// scratch size of the stage entry and both launchers all ask it, so they cannot disagree about a shape.
bool pyramid_eligible(int D, int samples, int C, int L) {
    if (D < 4 || D > 6 || C <= 0 || C > kSolveKC * kSolveThreads) return false;   // levels 0..3 by lane chunks, 4 per lane, 5 per lane pair
    if (samples > kPyrMaxSamples) return false;                // per-sample (mean, rstd) of y in shared memory
    if (L % 16 != 0 || (L % (1 << (D - 1))) != 0) return false;
    if ((L >> (D - 1)) < 6) return false;                      // the edge bookkeeping assumes 2 + 1 distinct edge positions
    return pyramid_windows(D, L) <= 32;                        // one CTA (<= 1024 threads) per row
}
size_t pyramid_rowstats_bytes(int samples, int C, int D) { return (size_t)samples * C * (D - 1) * kRowStat * sizeof(double); }
size_t pyramid_table_bytes(int samples, int C, int D) { return (size_t)samples * C * pyr_table_width(D) * sizeof(float); }

// The arguments of the pyramid pass and of the solve, shared by both launchers.  z: the level outputs (kPyrLevels),
// or null.
static int pyramid_args(const float* y, const NormIn& nin, const float* const* w5, const float* const* bias,
                        const float* const* gamma, const float* const* beta, float* const* z, double* stats0,
                        double* rowstats, float* table, int D, int samples, int C, int L, PyrArgs& a, SolveArgs& s) {
    if (!pyramid_eligible(D, samples, C, L)) return SDR_ERR_UNSUPPORTED;
    if (!y || !stats0 || !rowstats || !table || samples <= 0) return SDR_ERR_BAD_ARGUMENT;
    uintptr_t al = reinterpret_cast<uintptr_t>(y);
    for (int d = 0; d < D; ++d) {
        if (!w5[d] || !bias[d] || !gamma[d] || !beta[d] || (z && !z[d])) return SDR_ERR_BAD_ARGUMENT;
        if (z) al |= reinterpret_cast<uintptr_t>(z[d]);
    }
    if (al % 16 != 0) return SDR_ERR_UNSUPPORTED;
    const long long rows = (long long)samples * C;
    if (rows > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    memset(&a, 0, sizeof(a));
    a.y = y; a.nin = nin; a.bias0 = bias[0]; a.stats0 = stats0; a.rowstats = rowstats;
    a.D = D; a.C = C; a.L = L; a.rows = (int)rows;
    memset(&s, 0, sizeof(s));
    s.stats0 = stats0; s.rowstats = rowstats; s.table = table; s.D = D; s.C = C; s.L = L;
    for (int d = 0; d < D; ++d) {
        a.w[d] = w5[d]; a.z[d] = z ? z[d] : nullptr;
        s.gamma[d] = gamma[d]; s.beta[d] = beta[d]; s.w[d] = w5[d]; s.bias[d] = bias[d];
    }
    return SDR_OK;
}

// One pass of dw_pyramid_kernel on persistent CTAs: exactly as many as are resident at once.
template <typename K>
static int launch_pyramid_pass(K kern, const PyrArgs& a, int samples, cudaStream_t st) {
    const int threads = 32 * pyramid_windows(a.D, a.L);
    const size_t smem = (2 * (size_t)(a.L + 8)) * sizeof(float) + (size_t)samples * sizeof(float2);
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return SDR_ERR_CUDA;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return SDR_ERR_CUDA;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem) != cudaSuccess || per_sm < 1) {
        cudaGetLastError();
        per_sm = 1;
    }
    long long grid = (long long)sms * per_sm;
    if (grid > a.rows) grid = a.rows;
    kern<<<(unsigned)grid, threads, smem, st>>>(a);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

// y [samples][C][L] -> z[0] = z_0, z[d] = R_d, table (merge coefficients).  stats0: zeroed slot for the statistics of z_0.
int launch_pyramid(const float* y, const NormIn& nin, const float* const* w5, const float* const* bias,
                   const float* const* gamma, const float* const* beta, float* const* z, double* stats0,
                   double* rowstats, float* table, int D, int samples, int C, int L, cudaStream_t st) {
    if (!z) return SDR_ERR_BAD_ARGUMENT;
    PyrArgs a;
    SolveArgs s;
    int rc = pyramid_args(y, nin, w5, bias, gamma, beta, z, stats0, rowstats, table, D, samples, C, L, a, s);
    if (rc != SDR_OK) return rc;
    const int threads = 32 * pyramid_windows(D, L);
    auto launch = [&](auto kern) -> int { return launch_pyramid_pass(kern, a, samples, st); };
    if (nin.prelu && nin.prelu_pc) {
        if (threads <= 256)
            rc = D == 4 ? launch(dw_pyramid_kernel<4, 256, SDR_PYR_MINB, true>)
                        : (D == 5 ? launch(dw_pyramid_kernel<5, 256, SDR_PYR_MINB, true>) : launch(dw_pyramid_kernel<6, 256, SDR_PYR_MINB, true>));
        else
            rc = D == 4 ? launch(dw_pyramid_kernel<4, 1024, 1, true>)
                        : (D == 5 ? launch(dw_pyramid_kernel<5, 1024, 1, true>) : launch(dw_pyramid_kernel<6, 1024, 1, true>));
    } else if (threads <= 256)      // rows up to 7-8 windows (L <= 3712 / 3328): compiled for several resident CTAs per SM
        rc = D == 4 ? launch(dw_pyramid_kernel<4, 256, SDR_PYR_MINB, false>)
                    : (D == 5 ? launch(dw_pyramid_kernel<5, 256, SDR_PYR_MINB, false>) : launch(dw_pyramid_kernel<6, 256, SDR_PYR_MINB, false>));
    else
        rc = D == 4 ? launch(dw_pyramid_kernel<4, 1024, 1, false>)
                    : (D == 5 ? launch(dw_pyramid_kernel<5, 1024, 1, false>) : launch(dw_pyramid_kernel<6, 1024, 1, false>));
    if (rc != SDR_OK) return rc;
    pyramid_solve_kernel<<<(unsigned)samples, kSolveThreads, 0, st>>>(s);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

// One pass of the fused stage (M = kPyrStats or kPyrMerge), with the instantiation the row length and slope call for.
template <int M>
static int launch_fused_pass(const PyrArgs& a, bool pc, int samples, cudaStream_t st) {
    constexpr int MB = M == kPyrMerge ? SDR_PYR_MERGE_MINB : SDR_PYR_STATS_MINB;
    const int D = a.D, threads = 32 * pyramid_windows(a.D, a.L);
    auto launch = [&](auto kern) -> int { return launch_pyramid_pass(kern, a, samples, st); };
    if (pc) {
        if (threads <= 256)
            return D == 4 ? launch(dw_pyramid_kernel<4, 256, MB, true, M>)
                          : (D == 5 ? launch(dw_pyramid_kernel<5, 256, MB, true, M>) : launch(dw_pyramid_kernel<6, 256, MB, true, M>));
        return D == 4 ? launch(dw_pyramid_kernel<4, 1024, 1, true, M>)
                      : (D == 5 ? launch(dw_pyramid_kernel<5, 1024, 1, true, M>) : launch(dw_pyramid_kernel<6, 1024, 1, true, M>));
    }
    if (threads <= 256)
        return D == 4 ? launch(dw_pyramid_kernel<4, 256, MB, false, M>)
                      : (D == 5 ? launch(dw_pyramid_kernel<5, 256, MB, false, M>) : launch(dw_pyramid_kernel<6, 256, MB, false, M>));
    return D == 4 ? launch(dw_pyramid_kernel<4, 1024, 1, false, M>)
                  : (D == 5 ? launch(dw_pyramid_kernel<5, 1024, 1, false, M>) : launch(dw_pyramid_kernel<6, 1024, 1, false, M>));
}

// The whole depthwise stage without the levels in HBM: statistics pass over y, solve, merge pass over y.
// y [samples][C][L] -> m [samples][C][L] (m == y or disjoint), stats_m.  stats0 / stats_m: zeroed slots.
int launch_pyramid_fused(const float* y, const NormIn& nin, const float* const* w5, const float* const* bias,
                         const float* const* gamma, const float* const* beta, float* m, double* stats0, double* stats_m,
                         double* rowstats, float* table, int D, int samples, int C, int L, cudaStream_t st) {
    PyrArgs a;
    SolveArgs s;
    int rc = pyramid_args(y, nin, w5, bias, gamma, beta, nullptr, stats0, rowstats, table, D, samples, C, L, a, s);
    if (rc != SDR_OK) return rc;
    if (!m || !stats_m) return SDR_ERR_BAD_ARGUMENT;
    const size_t n = (size_t)samples * C * L;
    if (m != y && m < y + n && y < m + n) return SDR_ERR_BAD_ARGUMENT;   // a row's m would overwrite rows not yet read
    if (reinterpret_cast<uintptr_t>(m) % 16 != 0) return SDR_ERR_UNSUPPORTED;
    const bool pc = nin.prelu && nin.prelu_pc;
    if ((rc = launch_fused_pass<kPyrStats>(a, pc, samples, st)) != SDR_OK) return rc;
    pyramid_solve_kernel<<<(unsigned)samples, kSolveThreads, 0, st>>>(s);
    if (cudaGetLastError() != cudaSuccess) return SDR_ERR_CUDA;
    a.table = table; a.m = m; a.stats_m = stats_m;
    return launch_fused_pass<kPyrMerge>(a, pc, samples, st);
}

int launch_merge_pyramid(const float* const* z, const float* table, int D, float* m, double* stats_out,
                         int samples, int C, int L, cudaStream_t st) {
    if (!pyramid_eligible(D, samples, C, L)) return SDR_ERR_UNSUPPORTED;
    MergePyrArgs a;
    memset(&a, 0, sizeof(a));
    a.table = table; a.D = D; a.C = C; a.L = L;
    uintptr_t al = reinterpret_cast<uintptr_t>(m);
    for (int d = 0; d < D; ++d) { a.z[d] = z[d]; al |= reinterpret_cast<uintptr_t>(z[d]); }
    if (al % 16 != 0) return SDR_ERR_UNSUPPORTED;
    const long long items = (long long)C * (L / 16);
    const int per_cta = kMpThreads * kMpItems;
    const int chunks = (int)((items + per_cta - 1) / per_cta);
    const long long grid = (long long)chunks * samples;
    if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    merge_pyramid_kernel<<<(unsigned)grid, kMpThreads, 0, st>>>(a, m, stats_out, chunks);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

}  // namespace sdr
