// 1x1 Conv1d as a batched GEMM, fp32 FFMA path (exact-parity path; also the
// path for the small / odd channel counts that cannot fill a wgmma tile).
//
//   y[s, m, l] = sum_k W[m, k] * f(x[s, k, l]) + bias[m]  (+ residual[s, m, l])
//   f = deferred GlobLN (+PReLU) of the producer, applied while the activation
//       tile is staged into shared memory.
//
// Replaces (reference file:line)
//   bottleneck        improved_sudormrf.py:256-259,292   f = GlobLN (ln, :255,291)
//   proj_1x1.conv     improved_sudormrf.py:174,205       f = identity
//   res_conv (+skip)  improved_sudormrf.py:196,220       f = GlobLN+PReLU (final_norm :195,218)
//   mask_net          improved_sudormrf.py:268-269,295-298  f = PReLU, epilogue relu()*encoder
//   decoder (as GEMM) improved_sudormrf.py:272-279,300   frames = Wd^T . masked
#include "common.cuh"

namespace sdr {

struct PwArgs {
    const float* x;
    NormIn nin;
    const float* W;
    const float* bias;
    const float* residual;
    const float* gate;
    int gate_channels;
    float* y;
    double* stats_out;
    int M, K, L;
    int l_tiles;
    int epilogue;      // 0 plain, 1 relu(y) * gate
    // small-channel kernel only (GroupComm, groupcomm_sudormrf_v2.py:381-383,411): the operand is
    // x + GlobLN(pre_add) (the TAC residual + norm), which is also written to pre_out (the block's skip connection)
    const float* pre_add;
    NormIn pre_norm;
    float* pre_out;
};

constexpr int kPwThreads = 256;
constexpr int kBN = 128;
constexpr int kBK = 16;

template <int BM, bool VEC>
__global__ void __launch_bounds__(kPwThreads, 2)
pw_gemm_kernel(const PwArgs a) {
    constexpr int TM = BM / 16;
    constexpr int AS = BM + 4;                       // padded row stride of the W tile
    constexpr int WPT = BM * kBK / kPwThreads;       // W elements per thread per k-tile
    __shared__ __align__(16) float As[2][kBK][AS];
    __shared__ __align__(16) float Bs[2][kBK][kBN];
    __shared__ SampleNorm s_norm;
    __shared__ float s_red[64];

    const int tid = threadIdx.x;
    const int sample = blockIdx.x / a.l_tiles;
    const int l0 = (blockIdx.x - sample * a.l_tiles) * kBN;
    const int m0 = blockIdx.y * BM;
    if (tid == 0) s_norm = sample_norm(a.nin, sample);
    __syncthreads();
    const SampleNorm sn = s_norm;

    const int tx = tid & 15, ty = tid >> 4;
    const float* xs = a.x + (size_t)sample * a.K * a.L;

    // staging coordinates
    const int xk = tid >> 5;            // 0..7 (+8)
    const int xl = (tid & 31) * 4;      // 0..124
    const int wk = tid & 15;            // k within tile (lanes along k: coalesced W rows)
    const int wm = tid >> 4;            // 0..15, + 16*i

    float acc[TM][8];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    float wreg[WPT];
    float4 xreg[2];

    auto load_tiles = [&](int k0) {
#pragma unroll
        for (int i = 0; i < WPT; ++i) {
            const int m = m0 + wm + 16 * i, k = k0 + wk;
            wreg[i] = (m < a.M && k < a.K) ? __ldg(a.W + (size_t)m * a.K + k) : 0.f;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int k = k0 + xk + 8 * h;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k < a.K) {
                const ChanNorm cn = chan_norm(a.nin, sn, k);
                const float* p = xs + (size_t)k * a.L + l0 + xl;
                if (VEC) {
                    if (l0 + xl < a.L) {
                        v = ldg4(p);
                        v.x = apply_norm(cn, v.x); v.y = apply_norm(cn, v.y);
                        v.z = apply_norm(cn, v.z); v.w = apply_norm(cn, v.w);
                    }
                } else {
                    if (l0 + xl + 0 < a.L) v.x = apply_norm(cn, __ldg(p + 0));
                    if (l0 + xl + 1 < a.L) v.y = apply_norm(cn, __ldg(p + 1));
                    if (l0 + xl + 2 < a.L) v.z = apply_norm(cn, __ldg(p + 2));
                    if (l0 + xl + 3 < a.L) v.w = apply_norm(cn, __ldg(p + 3));
                }
            }
            xreg[h] = v;
        }
    };
    auto store_tiles = [&](int buf) {
#pragma unroll
        for (int i = 0; i < WPT; ++i) As[buf][wk][wm + 16 * i] = wreg[i];
#pragma unroll
        for (int h = 0; h < 2; ++h)
            *reinterpret_cast<float4*>(&Bs[buf][xk + 8 * h][xl]) = xreg[h];
    };

    const int nk = (a.K + kBK - 1) / kBK;
    load_tiles(0);
    store_tiles(0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int cur = kt & 1;
        if (kt + 1 < nk) load_tiles((kt + 1) * kBK);
#pragma unroll
        for (int k = 0; k < kBK; ++k) {
            float af[TM];
            if constexpr (BM == 128) {
                const float4 a0 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 4]);
                const float4 a1 = *reinterpret_cast<const float4*>(&As[cur][k][64 + ty * 4]);
                af[0] = a0.x; af[1] = a0.y; af[2] = a0.z; af[3] = a0.w;
                af[4] = a1.x; af[5] = a1.y; af[6] = a1.z; af[7] = a1.w;
            } else if constexpr (BM == 64) {
                const float4 a0 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 4]);
                af[0] = a0.x; af[1] = a0.y; af[2] = a0.z; af[3] = a0.w;
            } else {
                const float2 a0 = *reinterpret_cast<const float2*>(&As[cur][k][ty * 2]);
                af[0] = a0.x; af[1] = a0.y;
            }
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[cur][k][64 + tx * 4]);
            const float bf[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(af[i], bf[j], acc[i][j]);
        }
        if (kt + 1 < nk) store_tiles(cur ^ 1);
        __syncthreads();
    }

    // ---- epilogue: bias, residual, gate, store, statistics ----
    float st_s = 0.f, st_q = 0.f;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        int mr;
        if (BM == 128) mr = (i < 4) ? ty * 4 + i : 64 + ty * 4 + (i - 4);
        else if (BM == 64) mr = ty * 4 + i;
        else mr = ty * 2 + i;
        const int m = m0 + mr;
        if (m >= a.M) continue;
        const float b = a.bias ? __ldg(a.bias + m) : 0.f;
        const size_t row = ((size_t)sample * a.M + m) * a.L;
        const float* grow = (a.epilogue == 1)
            ? a.gate + ((size_t)sample * a.gate_channels + (m % a.gate_channels)) * a.L : nullptr;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int l = l0 + h * 64 + tx * 4;
            float o[4] = {acc[i][4 * h + 0] + b, acc[i][4 * h + 1] + b,
                          acc[i][4 * h + 2] + b, acc[i][4 * h + 3] + b};
            if (VEC) {
                if (l < a.L) {
                    if (a.residual) {
                        const float4 r = *reinterpret_cast<const float4*>(a.residual + row + l);  // plain load: may alias y (in-place skip)
                        o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w;
                    }
                    if (a.epilogue == 1) {
                        const float4 g = ldg4(grow + l);
                        o[0] = fmaxf(o[0], 0.f) * g.x; o[1] = fmaxf(o[1], 0.f) * g.y;
                        o[2] = fmaxf(o[2], 0.f) * g.z; o[3] = fmaxf(o[3], 0.f) * g.w;
                    }
                    *reinterpret_cast<float4*>(a.y + row + l) = make_float4(o[0], o[1], o[2], o[3]);
#pragma unroll
                    for (int e = 0; e < 4; ++e) { st_s += o[e]; st_q = fmaf(o[e], o[e], st_q); }
                }
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    if (l + e < a.L) {
                        float v = o[e];
                        if (a.residual) v += a.residual[row + l + e];
                        if (a.epilogue == 1) v = fmaxf(v, 0.f) * __ldg(grow + l + e);
                        a.y[row + l + e] = v;
                        st_s += v; st_q = fmaf(v, v, st_q);
                    }
                }
            }
        }
    }
    if (a.stats_out) block_stats_atomic(st_s, st_q, a.stats_out, sample, s_red);
}


// ---------------------------------------------------------------------------
// Small-channel variant (group-communication blocks: 16 -> 32 and 32 -> 16 channels per
// group, groupcomm_sudormrf_v2.py:401-403).  The op is pure streaming (AI ~ 4 FLOP/B), so the
// tiled GEMM above wastes its tile; here a thread owns 4 consecutive positions x 16 output
// channels: per input channel ONE float4 load (lanes = consecutive position quads -> 512 B per
// warp), 64 FMAs against 16 weights broadcast from shared memory, float4 stores.
// Requires K <= 64, L % 4 == 0.
// ---------------------------------------------------------------------------
#ifndef SDR_PW_TILE
#define SDR_PW_TILE 1                  // 1: shapes the tile-staged kernel takes (M <= 32, K <= 32) run on it; 0: pw_small_kernel (A/B builds)
#endif
constexpr int kSmMaxThreads = 256;
constexpr int kSmMT = 16;          // output channels per thread (8 per thread, 5 CTAs per SM, measured slower: res_conv shape 72 -> 88 us)
constexpr int kSmKT = 8;           // input rows whose loads are issued together (8 x 16 B in flight per thread)
constexpr int kSmMaxK = 64;

// The launch list of the GroupComm model (profiles/r02_groupcomm.md) had this kernel at 0.34 of the HBM roofline: the
// block size did not divide the 800 position quads of a row (a quarter of the threads idle) and only 4 loads per thread
// were in flight.  Now: block size chosen by the launcher to divide the row, loads batched 8 rows at a time.
template <bool PRE>                     // PRE: operand = x + GlobLN(pre_add), written to pre_out (GroupComm proj_1x1)
__global__ void __launch_bounds__(kSmMaxThreads, 2)
pw_small_kernel(const PwArgs a, int chunks_per_sample) {
    constexpr int KT = PRE ? kSmKT / 2 : kSmKT;            // rows per batch: 4 + 4 loads in flight with the second operand
    __shared__ __align__(16) float sW[kSmMaxK][kSmMT];     // [k][m]
    __shared__ float2 sAB[kSmMaxK];                         // folded norm: y = x*a + b
    __shared__ float2 sPre[kSmMaxK];                        // folded norm of the pre-add operand
    __shared__ float sBias[kSmMT];
    __shared__ float s_red[64];
    const int tid = threadIdx.x, nthr = blockDim.x;
    const int sample = blockIdx.x / chunks_per_sample;
    const int chunk = blockIdx.x - sample * chunks_per_sample;
    const int m0 = blockIdx.y * kSmMT;
    for (int i = tid; i < a.K * kSmMT; i += nthr) {
        const int k = i / kSmMT, m = i - k * kSmMT;
        sW[k][m] = (m0 + m < a.M) ? __ldg(a.W + (size_t)(m0 + m) * a.K + k) : 0.f;
    }
    if (tid < kSmMT) sBias[tid] = (a.bias && m0 + tid < a.M) ? __ldg(a.bias + m0 + tid) : 0.f;
    if (tid < a.K) {
        float aa = 1.f, bb = 0.f;
        if (a.nin.stats) {
            const SampleNorm sn = sample_norm(a.nin, sample);
            aa = __ldg(a.nin.gamma + tid) * sn.rstd;
            bb = fmaf(-sn.mean, aa, __ldg(a.nin.beta + tid));
        }
        sAB[tid] = make_float2(aa, bb);
        float pa = 1.f, pb = 0.f;
        if (PRE && a.pre_norm.stats) {
            const SampleNorm sn = sample_norm(a.pre_norm, sample);
            pa = __ldg(a.pre_norm.gamma + tid) * sn.rstd;
            pb = fmaf(-sn.mean, pa, __ldg(a.pre_norm.beta + tid));
        }
        sPre[tid] = make_float2(pa, pb);
    }
    const bool act = a.nin.prelu != nullptr;
    const float slope = act ? __ldg(a.nin.prelu) : 1.f;
    __syncthreads();

    const int QR = a.L >> 2;
    const int q = chunk * nthr + tid;
    float st_s = 0.f, st_q = 0.f;
    if (q < QR) {
        const float* xp = a.x + (size_t)sample * a.K * a.L + 4 * q;
        float acc[kSmMT][4];
#pragma unroll
        for (int m = 0; m < kSmMT; ++m) { acc[m][0] = acc[m][1] = acc[m][2] = acc[m][3] = sBias[m]; }
#pragma unroll 1
        for (int k0 = 0; k0 < a.K; k0 += KT) {
            float4 v[KT];
#pragma unroll
            for (int j = 0; j < KT; ++j)                       // all loads of the batch first
                v[j] = (k0 + j < a.K) ? ldg4(xp + (size_t)(k0 + j) * a.L) : make_float4(0.f, 0.f, 0.f, 0.f);
            if constexpr (PRE) {                               // operand = x + GlobLN(pre_add); kept for the skip connection
                const float* pp = a.pre_add + (size_t)sample * a.K * a.L + 4 * q;
                float4 w[KT];
#pragma unroll
                for (int j = 0; j < KT; ++j)
                    w[j] = (k0 + j < a.K) ? ldg4(pp + (size_t)(k0 + j) * a.L) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int j = 0; j < KT; ++j) {
                    if (k0 + j < a.K) {
                        const float2 pn = sPre[k0 + j];
                        v[j].x += fmaf(w[j].x, pn.x, pn.y); v[j].y += fmaf(w[j].y, pn.x, pn.y);
                        v[j].z += fmaf(w[j].z, pn.x, pn.y); v[j].w += fmaf(w[j].w, pn.x, pn.y);
                        if (blockIdx.y == 0)
                            *reinterpret_cast<float4*>(a.pre_out + ((size_t)sample * a.K + k0 + j) * a.L + 4 * q) = v[j];
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < KT; ++j) {
                if (k0 + j < a.K) {
                    const float2 ab = sAB[k0 + j];
                    float4 x = v[j];
                    x.x = fmaf(x.x, ab.x, ab.y); x.y = fmaf(x.y, ab.x, ab.y);
                    x.z = fmaf(x.z, ab.x, ab.y); x.w = fmaf(x.w, ab.x, ab.y);
                    if (act) {
                        x.x = x.x >= 0.f ? x.x : x.x * slope; x.y = x.y >= 0.f ? x.y : x.y * slope;
                        x.z = x.z >= 0.f ? x.z : x.z * slope; x.w = x.w >= 0.f ? x.w : x.w * slope;
                    }
#pragma unroll
                    for (int m4 = 0; m4 < kSmMT / 4; ++m4) {
                        const float4 w = *reinterpret_cast<const float4*>(&sW[k0 + j][m4 * 4]);
                        const float ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            acc[m4 * 4 + u][0] = fmaf(ww[u], x.x, acc[m4 * 4 + u][0]);
                            acc[m4 * 4 + u][1] = fmaf(ww[u], x.y, acc[m4 * 4 + u][1]);
                            acc[m4 * 4 + u][2] = fmaf(ww[u], x.z, acc[m4 * 4 + u][2]);
                            acc[m4 * 4 + u][3] = fmaf(ww[u], x.w, acc[m4 * 4 + u][3]);
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int m = 0; m < kSmMT; ++m) {
            if (m0 + m < a.M) {
                const size_t idx = ((size_t)sample * a.M + m0 + m) * a.L + 4 * q;
                float o[4] = {acc[m][0], acc[m][1], acc[m][2], acc[m][3]};
                if (a.residual) {
                    const float4 r = *reinterpret_cast<const float4*>(a.residual + idx);   // may alias y
                    o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w;
                }
                if (a.epilogue == 1) {
                    const float4 g = ldg4(a.gate + ((size_t)sample * a.gate_channels + ((m0 + m) % a.gate_channels)) * a.L + 4 * q);
                    o[0] = fmaxf(o[0], 0.f) * g.x; o[1] = fmaxf(o[1], 0.f) * g.y;
                    o[2] = fmaxf(o[2], 0.f) * g.z; o[3] = fmaxf(o[3], 0.f) * g.w;
                }
                *reinterpret_cast<float4*>(a.y + idx) = make_float4(o[0], o[1], o[2], o[3]);
#pragma unroll
                for (int e = 0; e < 4; ++e) { st_s += o[e]; st_q = fmaf(o[e], o[e], st_q); }
            }
        }
    }
    if (a.stats_out) block_stats_atomic(st_s, st_q, a.stats_out, sample, s_red);
}

// ---------------------------------------------------------------------------
// Tile-staged variant of the small-channel kernel (the GroupComm production geometry: 16 -> 32 and 32 -> 16 channels).
// ncu of pw_small_kernel at cfg 4 (profiles/r02b_kernels.md): 124-126 registers -> 15 warps per SM, issue-active
// 36-46 %, long-scoreboard the top stall, and the two blockIdx.y halves of the 32-output conv re-read their inputs
// from DRAM (209 MB read for 105 MB of operands): load and FFMA phases of a thread run back to back and there are too
// few warps to overlap them.  Here the loads leave the registers: a CTA owns P positions of one sample, thread 0 issues
// ONE bulk TMA copy per input row ([K (+K) rows][P] fp32, up to 40 KB in flight per CTA) while the other threads stage
// the weights; every thread then owns 2 positions x ALL output channels (inputs by LDS.64, weights by broadcast LDS.128,
// 2*MT accumulators), so nothing is read twice and 4 CTAs per SM overlap each other's copy, FFMA and store phases.
// ---------------------------------------------------------------------------
constexpr int kStMaxRows = 64;         // input rows staged per CTA (K, or 2K with the pre-add operand)
constexpr int kStMaxK = 32;

__device__ __forceinline__ uint32_t st_smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

constexpr int kStThreads = 160;        // block size bound (the launcher picks 128 or 160)
#ifndef SDR_ST_MINB32
#define SDR_ST_MINB32 3                // resident CTAs per SM the 32-outputs-per-thread instantiations are compiled for (4: 96 registers
#endif                                 // with 300 B of spills, 77 us against 69 us at the cfg-4 proj shape)
#ifndef SDR_ST_MINB16
#define SDR_ST_MINB16 4                // ... and the 16-outputs-per-thread ones (4 / 5 / 6: 62.8 / 64.8 / 66.4 us at the cfg-4 res_conv shape)
#endif
// (A persistent version with a double buffer - the next tile's copy in flight during the FFMA loop, 2 CTAs per SM by
//  shared memory - measured 92 / 73 us against 69 / 63 us for one tile per CTA: profiles/r02b_kernels.md.)
template <bool PRE, int MT>
__global__ void __launch_bounds__(kStThreads, MT == 32 ? SDR_ST_MINB32 : SDR_ST_MINB16)
pw_tile_kernel(const PwArgs a, int tiles_per_sample, int P) {
    extern __shared__ __align__(16) float st_buf[];        // [rows][P]
    __shared__ __align__(16) float sW[kStMaxK][MT];        // [k][m]
    __shared__ float2 sAB[kStMaxK];                         // folded norm of the operand: y = x*a + b
    __shared__ float2 sPre[kStMaxK];                        // folded norm of the pre-add operand
    __shared__ float sBias[MT];
    __shared__ float s_red[64];
    __shared__ __align__(8) uint64_t s_bar;
    const int tid = threadIdx.x, nthr = blockDim.x;
    const int sample = blockIdx.x / tiles_per_sample;
    const int p0 = (blockIdx.x - sample * tiles_per_sample) * P;
    const int np = min(P, a.L - p0);                        // positions of this tile (a multiple of 4)
    const int rows = PRE ? 2 * a.K : a.K;
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(st_smem_u32(&s_bar)), "r"(1) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const uint32_t bytes = (uint32_t)np * sizeof(float);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(st_smem_u32(&s_bar)), "r"(bytes * (uint32_t)rows) : "memory");
        for (int r = 0; r < rows; ++r) {
            const float* src = (PRE && r >= a.K) ? a.pre_add + ((size_t)sample * a.K + (r - a.K)) * a.L + p0
                                                 : a.x + ((size_t)sample * a.K + r) * a.L + p0;
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(st_smem_u32(st_buf + (size_t)r * P)), "l"(src), "r"(bytes), "r"(st_smem_u32(&s_bar)) : "memory");
        }
    }
    for (int i = tid; i < a.K * MT; i += nthr) {
        const int k = i / MT, m = i - k * MT;
        sW[k][m] = (m < a.M) ? __ldg(a.W + (size_t)m * a.K + k) : 0.f;
    }
    if (tid < MT) sBias[tid] = (a.bias && tid < a.M) ? __ldg(a.bias + tid) : 0.f;
    if (tid < a.K) {
        float aa = 1.f, bb = 0.f;
        if (a.nin.stats) {
            const SampleNorm sn = sample_norm(a.nin, sample);
            aa = __ldg(a.nin.gamma + tid) * sn.rstd;
            bb = fmaf(-sn.mean, aa, __ldg(a.nin.beta + tid));
        }
        sAB[tid] = make_float2(aa, bb);
        float pa = 1.f, pb = 0.f;
        if (PRE && a.pre_norm.stats) {
            const SampleNorm sn = sample_norm(a.pre_norm, sample);
            pa = __ldg(a.pre_norm.gamma + tid) * sn.rstd;
            pb = fmaf(-sn.mean, pa, __ldg(a.pre_norm.beta + tid));
        }
        sPre[tid] = make_float2(pa, pb);
    }
    const bool act = a.nin.prelu != nullptr;
    const float slope = act ? __ldg(a.nin.prelu) : 1.f;
    __syncthreads();                                        // tables + the initialised barrier are visible
    {
        const uint32_t addr = st_smem_u32(&s_bar);
        uint32_t done;
        do {
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                         : "=r"(done) : "r"(addr), "r"(0) : "memory");
        } while (!done);
    }
    const int t2 = 2 * tid;                                 // this thread's 2 positions inside the tile
    float st_s = 0.f, st_q = 0.f;
    if (t2 < np) {
        float acc[MT][2];
#pragma unroll
        for (int m = 0; m < MT; ++m) { acc[m][0] = sBias[m]; acc[m][1] = sBias[m]; }
        const size_t gpos = (size_t)p0 + t2;
        const size_t obase = (size_t)sample * a.M * a.L + gpos;
        // 16 outputs per thread (every res_conv of a GroupComm block): the skip-connection rows are fetched BEFORE the
        // FFMA loop and consumed after it (ncu: the epilogue's adds sat on the long scoreboard of these loads).
        // They may alias y: every element is read by the thread that writes it.
        float2 rpre[MT == 16 ? 16 : 1];
        if constexpr (MT == 16) {
            if (a.residual) {
#pragma unroll
                for (int m = 0; m < 16; ++m)
                    rpre[m] = (m < a.M) ? *reinterpret_cast<const float2*>(a.residual + obase + (size_t)m * a.L)
                                        : make_float2(0.f, 0.f);
            }
        }
        // row cursors bumped per input channel (the compiler re-derived the 64-bit global address of every pre_out row)
        const float* xs = st_buf + t2;
        const float* os = st_buf + (size_t)a.K * P + t2;
        float* pre_p = PRE ? a.pre_out + (size_t)sample * a.K * a.L + gpos : nullptr;
#pragma unroll 2
        for (int k = 0; k < a.K; ++k) {
            float2 v = *reinterpret_cast<const float2*>(xs);
            xs += P;
            if constexpr (PRE) {                            // operand = x + GlobLN(pre_add); kept for the skip connection
                const float2 w = *reinterpret_cast<const float2*>(os);
                os += P;
                const float2 pn = sPre[k];
                v.x += fmaf(w.x, pn.x, pn.y); v.y += fmaf(w.y, pn.x, pn.y);
                *reinterpret_cast<float2*>(pre_p) = v;
                pre_p += a.L;
            }
            if constexpr (!PRE) {                           // (the pre-add operand is never normalised again: launch_pointwise_small_preadd)
                const float2 ab = sAB[k];
                v.x = fmaf(v.x, ab.x, ab.y); v.y = fmaf(v.y, ab.x, ab.y);
                if (act) { v.x = v.x >= 0.f ? v.x : v.x * slope; v.y = v.y >= 0.f ? v.y : v.y * slope; }
            }
#pragma unroll
            for (int m4 = 0; m4 < MT / 4; ++m4) {
                const float4 w = *reinterpret_cast<const float4*>(&sW[k][m4 * 4]);
                acc[m4 * 4 + 0][0] = fmaf(w.x, v.x, acc[m4 * 4 + 0][0]); acc[m4 * 4 + 0][1] = fmaf(w.x, v.y, acc[m4 * 4 + 0][1]);
                acc[m4 * 4 + 1][0] = fmaf(w.y, v.x, acc[m4 * 4 + 1][0]); acc[m4 * 4 + 1][1] = fmaf(w.y, v.y, acc[m4 * 4 + 1][1]);
                acc[m4 * 4 + 2][0] = fmaf(w.z, v.x, acc[m4 * 4 + 2][0]); acc[m4 * 4 + 2][1] = fmaf(w.z, v.y, acc[m4 * 4 + 2][1]);
                acc[m4 * 4 + 3][0] = fmaf(w.w, v.x, acc[m4 * 4 + 3][0]); acc[m4 * 4 + 3][1] = fmaf(w.w, v.y, acc[m4 * 4 + 3][1]);
            }
        }
        if constexpr (MT == 16) {
            if (a.residual) {
#pragma unroll
                for (int m = 0; m < 16; ++m) { acc[m][0] += rpre[m].x; acc[m][1] += rpre[m].y; }
            }
        }
        const bool want_stats = a.stats_out != nullptr;
        if (a.M == MT && (MT == 16 || !a.residual)) {       // every row real, nothing left to add: pointer-bumped stores
            float* yp = a.y + obase;
#pragma unroll
            for (int m = 0; m < MT; ++m) {
                *reinterpret_cast<float2*>(yp) = make_float2(acc[m][0], acc[m][1]);
                yp += a.L;
                if (want_stats) {
                    st_s += acc[m][0] + acc[m][1];
                    st_q = fmaf(acc[m][0], acc[m][0], st_q); st_q = fmaf(acc[m][1], acc[m][1], st_q);
                }
            }
        } else {
#pragma unroll
        for (int m8 = 0; m8 < MT; m8 += 8) {               // 8 output rows at a time: the residual loads of a group in flight together
            if (MT != 16 && a.residual) {                   // may alias y: every element is read by the thread that writes it
                float2 r[8];
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    r[j] = (m8 + j < a.M) ? *reinterpret_cast<const float2*>(a.residual + obase + (size_t)(m8 + j) * a.L)
                                          : make_float2(0.f, 0.f);
#pragma unroll
                for (int j = 0; j < 8; ++j) { acc[m8 + j][0] += r[j].x; acc[m8 + j][1] += r[j].y; }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int m = m8 + j;
                if (m < a.M) {
                    *reinterpret_cast<float2*>(a.y + obase + (size_t)m * a.L) = make_float2(acc[m][0], acc[m][1]);
                    st_s += acc[m][0] + acc[m][1];
                    st_q = fmaf(acc[m][0], acc[m][0], st_q); st_q = fmaf(acc[m][1], acc[m][1], st_q);
                }
            }
        }
        }
    }
    if (a.stats_out) block_stats_atomic(st_s, st_q, a.stats_out, sample, s_red);
}

// Tile geometry of pw_tile_kernel: threads = the multiple of 32 in [128, 256] that wastes the fewest threads on rows of
// L / 2 position pairs; P = 2 * threads positions per CTA.  false: the shape is not taken (the caller uses pw_small_kernel).
static bool tile_shape(int M, int K, int rows, int L, int epilogue, bool aligned, int* threads_out) {
    if (!aligned || (L % 4) != 0 || epilogue != 0 || M > 32 || K > kStMaxK || rows > kStMaxRows) return false;
    int best = kStThreads;
    long long best_waste = -1;
    const int pairs = L / 2;
    for (int t = kStThreads; t >= 128; t -= 32) {
        const long long waste = (long long)((pairs + t - 1) / t) * t - pairs;
        if (best_waste < 0 || waste < best_waste) { best = t; best_waste = waste; }
    }
    if ((size_t)rows * 2 * best * sizeof(float) > 160 * 1024) return false;
    *threads_out = best;
    return true;
}

template <bool PRE>
static int launch_tile(const PwArgs& a, int samples, int threads, cudaStream_t st) {
    const int P = 2 * threads;
    const int tiles = (a.L + P - 1) / P;
    const long long gx = (long long)tiles * samples;
    if (gx > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    const int rows = PRE ? 2 * a.K : a.K;
    const size_t smem = (size_t)rows * P * sizeof(float);
    auto go = [&](auto kern) -> int {
        if (smem > 40 * 1024 &&
            cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            cudaGetLastError();
            return SDR_ERR_CUDA;
        }
        kern<<<(unsigned)gx, threads, smem, st>>>(a, tiles, P);
        return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
    };
    return a.M <= 16 ? go(pw_tile_kernel<PRE, 16>) : go(pw_tile_kernel<PRE, 32>);
}

// block size for rows of `quads` position quads: the multiple of 32 in [128, 256] that wastes the fewest threads
static int small_block_threads(int quads) {
    int best = kSmMaxThreads;
    long long best_waste = -1;
    for (int t = kSmMaxThreads; t >= 128; t -= 32) {
        const long long waste = (long long)((quads + t - 1) / t) * t - quads;
        if (best_waste < 0 || waste < best_waste) { best = t; best_waste = waste; }
    }
    return best;
}

template <int BM>
static int launch_bm(const PwArgs& a, int samples, bool vec, cudaStream_t st) {
    const long long gx = (long long)a.l_tiles * samples;
    const int gy = (a.M + BM - 1) / BM;
    if (gx > 0x7fffffffLL || gy > 65535) return SDR_ERR_UNSUPPORTED;
    dim3 grid((unsigned)gx, (unsigned)gy);
    if (vec) pw_gemm_kernel<BM, true><<<grid, kPwThreads, 0, st>>>(a);
    else     pw_gemm_kernel<BM, false><<<grid, kPwThreads, 0, st>>>(a);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

int launch_pointwise_ffma(const float* x, const NormIn& nin, const float* W, const float* bias,
                          const float* residual, const float* gate, int gate_channels,
                          float* y, double* stats_out, int samples, int M, int K, int L,
                          int epilogue, cudaStream_t st) {
    if (samples <= 0 || M <= 0 || K <= 0 || L <= 0) return SDR_ERR_BAD_ARGUMENT;
    if (epilogue == 1 && (!gate || gate_channels <= 0)) return SDR_ERR_BAD_ARGUMENT;
    PwArgs a;
    a.x = x; a.nin = nin; a.W = W; a.bias = bias; a.residual = residual; a.gate = gate;
    a.gate_channels = gate_channels; a.y = y; a.stats_out = stats_out;
    a.M = M; a.K = K; a.L = L; a.l_tiles = (L + kBN - 1) / kBN; a.epilogue = epilogue;
    a.pre_add = nullptr; a.pre_norm = NormIn{nullptr, nullptr, nullptr, nullptr, 1.0}; a.pre_out = nullptr;
    uintptr_t al = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y);
    if (residual) al |= reinterpret_cast<uintptr_t>(residual);
    if (gate) al |= reinterpret_cast<uintptr_t>(gate);
    const bool vec = (L % 4 == 0) && (al % 16 == 0);
    if (vec && K <= kSmMaxK && M <= 64 && !nin.prelu_pc) {   // streaming small-channel kernels (one shared PReLU slope)
        int tt = 0;
        if (SDR_PW_TILE && tile_shape(M, K, K, L, epilogue, true, &tt)) return launch_tile<false>(a, samples, tt, st);
        const int threads = small_block_threads(L / 4);
        const int chunks = (L / 4 + threads - 1) / threads;
        const long long gx = (long long)chunks * samples;
        if (gx > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
        dim3 grid((unsigned)gx, (unsigned)((M + kSmMT - 1) / kSmMT));
        pw_small_kernel<false><<<grid, threads, 0, st>>>(a, chunks);
        return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
    }
    if (M > 64) return launch_bm<128>(a, samples, vec, st);
    if (M > 32) return launch_bm<64>(a, samples, vec, st);
    return launch_bm<32>(a, samples, vec, st);
}

// 1x1 conv of x + GlobLN(pre_add) for the small-channel (GroupComm) blocks; xt_out receives x + GlobLN(pre_add).
// SDR_ERR_UNSUPPORTED when the streaming kernel cannot take the shape (the caller then materialises xt first).
int launch_pointwise_small_preadd(const float* x, const float* pre_add, const NormIn& pre_norm, float* xt_out,
                                  const float* W, const float* bias, float* y, double* stats_out,
                                  int samples, int M, int K, int L, cudaStream_t st) {
    if (samples <= 0 || M <= 0 || K <= 0 || L <= 0 || !x || !pre_add || !xt_out || !W || !y) return SDR_ERR_BAD_ARGUMENT;
    const uintptr_t al = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) |
                         reinterpret_cast<uintptr_t>(pre_add) | reinterpret_cast<uintptr_t>(xt_out);
    if ((L % 4) != 0 || (al % 16) != 0 || K > kSmMaxK || M > 64) return SDR_ERR_UNSUPPORTED;
    PwArgs a;
    a.x = x; a.nin = NormIn{nullptr, nullptr, nullptr, nullptr, 1.0}; a.W = W; a.bias = bias; a.residual = nullptr;
    a.gate = nullptr; a.gate_channels = 0; a.y = y; a.stats_out = stats_out;
    a.M = M; a.K = K; a.L = L; a.l_tiles = (L + kBN - 1) / kBN; a.epilogue = 0;
    a.pre_add = pre_add; a.pre_norm = pre_norm; a.pre_out = xt_out;
    {
        int tt = 0;
        if (SDR_PW_TILE && tile_shape(M, K, 2 * K, L, 0, true, &tt)) return launch_tile<true>(a, samples, tt, st);
    }
    const int threads = small_block_threads(L / 4);
    const int chunks = (L / 4 + threads - 1) / threads;
    const long long gx = (long long)chunks * samples;
    if (gx > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    dim3 grid((unsigned)gx, (unsigned)((M + kSmMT - 1) / kSmMT));
    pw_small_kernel<true><<<grid, threads, 0, st>>>(a, chunks);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

}  // namespace sdr
