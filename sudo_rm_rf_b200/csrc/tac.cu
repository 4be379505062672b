// Transform-average-concatenate for the group-communication model.
//
// Reference: groupcomm_sudormrf_v2.py:343-384 (class TAC) and :405-418
// (GC_UConvBlock.forward).  For every (b, t) column, with x_g the n = Co/G
// channels of group g and H = 3n:
//     h_g = PReLU(W1 x_g + b1)                       TAC_input   (:366-367)
//     q   = PReLU(W2 mean_g(h_g) + b2)               TAC_mean    (:369-375)
//     o_g = PReLU(W3 [h_g ; q] + b3)                 TAC_output  (:376-378)
//     out = x + GlobLN_{(n,L) per (b,g)}(o)          TAC_norm    (:381-383)
// The reference materialises three permuted copies and a concat; here a CTA
// keeps the whole column block on chip: thread = (t, g), lanes along t so that
// every global access is a coalesced 128 B row segment, weights are broadcast
// from shared memory, and the mean over groups is a shared-memory reduction.
// The kernel stores o RAW plus per-(b,g) statistics; tac_apply then writes
// x + GlobLN(o) which is both the U-ConvBlock input and its residual.
#include <cuda_bf16.h>
#include "common.cuh"
#include "launchers.cuh"

namespace sdr {

struct TacParams {
    const float *W1, *b1, *a1, *W2, *b2, *a2, *W3, *b3, *a3;
};

template <int NPG>
__global__ void __launch_bounds__(512)
tac_kernel(const float* __restrict__ x, TacParams p, float* __restrict__ o,
           double* __restrict__ stats, int G, int L, int t_tiles) {
    constexpr int H = 3 * NPG;
    extern __shared__ __align__(16) float sm[];
    float* sW1 = sm;                      // [H][NPG]
    float* sb1 = sW1 + H * NPG;           // [H]
    float* sW2 = sb1 + H;                 // [H][H]
    float* sb2 = sW2 + H * H;             // [H]
    float* sW3 = sb2 + H;                 // [NPG][2H]
    float* sb3 = sW3 + NPG * 2 * H;       // [NPG]  (padded to 4)
    float* sMean = sb3 + ((NPG + 3) & ~3);// [H][32]
    float* sQ = sMean + H * 32;           // [H][32]
    float* sU = sQ + H * 32;              // [NPG][32]
    float* sS = sU + NPG * 32;            // [NPG][G][32]   reduction scratch

    const int tid = threadIdx.x, nthr = blockDim.x;
    const int lane = tid & 31, g = tid >> 5;
    const int b = blockIdx.x / t_tiles;
    const int t = (blockIdx.x - b * t_tiles) * 32 + lane;
    const bool valid = t < L;

    for (int i = tid; i < H * NPG; i += nthr) sW1[i] = __ldg(p.W1 + i);
    for (int i = tid; i < H; i += nthr) { sb1[i] = __ldg(p.b1 + i); sb2[i] = __ldg(p.b2 + i); }
    for (int i = tid; i < H * H; i += nthr) sW2[i] = __ldg(p.W2 + i);
    for (int i = tid; i < NPG * 2 * H; i += nthr) sW3[i] = __ldg(p.W3 + i);
    for (int i = tid; i < NPG; i += nthr) sb3[i] = __ldg(p.b3 + i);
    const float a1 = __ldg(p.a1), a2 = __ldg(p.a2), a3 = __ldg(p.a3);

    // 1. this thread's group column
    float xv[NPG];
    const size_t rowbase = ((size_t)b * G + g) * NPG;
#pragma unroll
    for (int i = 0; i < NPG; ++i) xv[i] = valid ? __ldg(x + (rowbase + i) * L + t) : 0.f;
    __syncthreads();

    // 2. h_g = PReLU(W1 x_g + b1)
    float h[H];
#pragma unroll
    for (int j = 0; j < H; ++j) {
        float acc = sb1[j];
#pragma unroll
        for (int i = 0; i < NPG; i += 4) {
            const float4 w = *reinterpret_cast<const float4*>(sW1 + j * NPG + i);
            acc = fmaf(w.x, xv[i], acc); acc = fmaf(w.y, xv[i + 1], acc);
            acc = fmaf(w.z, xv[i + 2], acc); acc = fmaf(w.w, xv[i + 3], acc);
        }
        h[j] = acc >= 0.f ? acc : acc * a1;
    }

    // 3. mean over groups, NPG hidden units at a time
    const float invG = 1.0f / (float)G;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int jj = 0; jj < NPG; ++jj) sS[(jj * G + g) * 32 + lane] = h[c * NPG + jj];
        __syncthreads();
        for (int jj = g; jj < NPG; jj += G) {
            float s = 0.f;
            for (int gg = 0; gg < G; ++gg) s += sS[(jj * G + gg) * 32 + lane];
            sMean[(c * NPG + jj) * 32 + lane] = s * invG;
        }
        __syncthreads();
    }

    // 4. q = PReLU(W2 mean + b2): hidden units dealt round-robin over the G warps
    for (int j = g; j < H; j += G) {
        float acc = sb2[j];
        for (int k = 0; k < H; k += 4) {
            const float4 w = *reinterpret_cast<const float4*>(sW2 + j * H + k);
            acc = fmaf(w.x, sMean[(k + 0) * 32 + lane], acc);
            acc = fmaf(w.y, sMean[(k + 1) * 32 + lane], acc);
            acc = fmaf(w.z, sMean[(k + 2) * 32 + lane], acc);
            acc = fmaf(w.w, sMean[(k + 3) * 32 + lane], acc);
        }
        sQ[j * 32 + lane] = acc >= 0.f ? acc : acc * a2;
    }
    __syncthreads();

    // 5. the q half of TAC_output is shared by all groups: u = W3[:, H:] q
    for (int i = g; i < NPG; i += G) {
        float acc = 0.f;
        for (int j = 0; j < H; j += 4) {
            const float4 w = *reinterpret_cast<const float4*>(sW3 + i * 2 * H + H + j);
            acc = fmaf(w.x, sQ[(j + 0) * 32 + lane], acc);
            acc = fmaf(w.y, sQ[(j + 1) * 32 + lane], acc);
            acc = fmaf(w.z, sQ[(j + 2) * 32 + lane], acc);
            acc = fmaf(w.w, sQ[(j + 3) * 32 + lane], acc);
        }
        sU[i * 32 + lane] = acc;
    }
    __syncthreads();

    // 6. o_g = PReLU(W3[:, :H] h_g + u + b3), raw store + per-(b,g) statistics
    float st_s = 0.f, st_q = 0.f;
#pragma unroll
    for (int i = 0; i < NPG; ++i) {
        float acc = sb3[i] + sU[i * 32 + lane];
#pragma unroll
        for (int j = 0; j < H; j += 4) {
            const float4 w = *reinterpret_cast<const float4*>(sW3 + i * 2 * H + j);
            acc = fmaf(w.x, h[j], acc); acc = fmaf(w.y, h[j + 1], acc);
            acc = fmaf(w.z, h[j + 2], acc); acc = fmaf(w.w, h[j + 3], acc);
        }
        const float v = acc >= 0.f ? acc : acc * a3;
        if (valid) {
            o[(rowbase + i) * L + t] = v;
            st_s += v; st_q = fmaf(v, v, st_q);
        }
    }
    const double ds = warp_sum_f64((double)st_s);
    const double dq = warp_sum_f64((double)st_q);
    if (lane == 0) {
        atomicAdd(stats + 2 * ((size_t)b * G + g), ds);
        atomicAdd(stats + 2 * ((size_t)b * G + g) + 1, dq);
    }
}

// ---------------------------------------------------------------------------
// Tensor-core TAC for 16 channels per group (the published GroupComm models: Co = 256, G = 16).
//
// The FFMA kernel above ran at 0.19 of the HBM roofline (173 us for 210 MB at the benchmark shape): 27.6 k MACs per
// time column on the FP32 pipe.  The three linear maps are small GEMMs over positions, so here a WARP owns 16
// consecutive positions of one batch element and walks the groups with warp-level MMAs (mma.sync m16n8k16, bf16
// operands split hi/lo in three products like the wgmma GEMM, fp32 accumulate):
//   pass 1, per group g:  h_g[16 x 48] = PReLU(X_g[16 x 16] W1^T + b1), accumulated into the group mean (registers)
//   once:                 q = PReLU(mean W2^T + b2),   u = q W3[:, 48:]^T + b3
//   pass 2, per group g:  h_g again (X_g is re-read from L1/L2; keeping 16 groups of h would take 384 registers),
//                         o_g = PReLU(h_g W3[:, :48]^T + u) -> raw store + per-(b, g) statistics
// The accumulator fragment of one GEMM is the A fragment of the next (rows = positions, two adjacent n-tiles = one
// k-tile), so nothing goes through shared memory between the three layers.  Weights are split and laid out in
// fragment order in shared memory once per CTA.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// (x, y) -> packed bf16x2 hi (truncation) and lo (RN of the exact remainder); x in the low half
__device__ __forceinline__ void split_pair(float x, float y, uint32_t& hi, uint32_t& lo) {
    const uint32_t hx = __float_as_uint(x) & 0xffff0000u, hy = __float_as_uint(y) & 0xffff0000u;
    hi = __byte_perm(hx, hy, 0x7632);
    const __nv_bfloat162 l = __floats2bfloat162_rn(x - __uint_as_float(hx), y - __uint_as_float(hy));
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
// d += A B with A = ah + al, B = bh + bl (the al * bl term is dropped: 2^-16 relative)
__device__ __forceinline__ void mma3(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                     uint32_t bh0, uint32_t bh1, uint32_t bl0, uint32_t bl1) {
    mma_16816(d, ah, bh0, bh1);
    mma_16816(d, al, bh0, bh1);
    mma_16816(d, ah, bl0, bl1);
}
// accumulator fragments of two adjacent n-tiles -> hi / lo A fragments of one k-tile
__device__ __forceinline__ void acc_to_a(const float (&d0)[4], const float (&d1)[4], uint32_t (&ah)[4], uint32_t (&al)[4]) {
    split_pair(d0[0], d0[1], ah[0], al[0]);        // row r,     cols 2c, 2c+1
    split_pair(d0[2], d0[3], ah[1], al[1]);        // row r + 8
    split_pair(d1[0], d1[1], ah[2], al[2]);        // row r,     cols 8 + 2c, ...
    split_pair(d1[2], d1[3], ah[3], al[3]);        // row r + 8
}

constexpr int kTacWarps = 8;
constexpr int kTacH = 48;

// B fragments of W^T for (k-tile kt, n-tile nt): [kt][nt][reg 0..1][hi, lo][lane]
struct TacFrags {
    uint32_t w1[1][6][2][2][32];       // TAC_input  [48][16]
    uint32_t w2[3][6][2][2][32];       // TAC_mean   [48][48]
    uint32_t w3[6][2][2][2][32];       // TAC_output [16][96]: k-tiles 0..2 = h part, 3..5 = q part
    float b1[kTacH], b2[kTacH], b3[16];
};

constexpr int kTacMinB = 2;           // resident CTAs per SM tac_mma16_kernel is compiled (and its persistent grid sized) for
__global__ void __launch_bounds__(32 * kTacWarps, kTacMinB)
tac_mma16_kernel(const float* __restrict__ x, TacParams p, float* __restrict__ o, double* __restrict__ stats,
                 int G, int L, int tiles_per_b, int total_tiles) {
    extern __shared__ __align__(16) uint8_t tac_smem[];
    TacFrags& F = *reinterpret_cast<TacFrags*>(tac_smem);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // ---- weights -> fragment order ----
    auto build = [&](uint32_t* dst, const float* W, int KT, int NT, int ldw) {    // W[n][k], row length ldw
        const int total = KT * NT * 2 * 32;
        for (int i = tid; i < total; i += blockDim.x) {
            const int ln = i & 31, reg = (i >> 5) & 1, nt = (i >> 6) % NT, kt = (i >> 6) / NT;
            const int k = kt * 16 + (ln & 3) * 2 + reg * 8, n = nt * 8 + (ln >> 2);
            uint32_t hi, lo;
            split_pair(__ldg(W + (size_t)n * ldw + k), __ldg(W + (size_t)n * ldw + k + 1), hi, lo);
            uint32_t* q = dst + (((size_t)(kt * NT + nt) * 2 + reg) * 2) * 32 + ln;
            q[0] = hi;
            q[32] = lo;
        }
    };
    build(&F.w1[0][0][0][0][0], p.W1, 1, 6, 16);
    build(&F.w2[0][0][0][0][0], p.W2, 3, 6, kTacH);
    build(&F.w3[0][0][0][0][0], p.W3, 6, 2, 2 * kTacH);
    for (int i = tid; i < kTacH; i += blockDim.x) { F.b1[i] = __ldg(p.b1 + i); F.b2[i] = __ldg(p.b2 + i); }
    if (tid < 16) F.b3[tid] = __ldg(p.b3 + tid);
    const float a1 = __ldg(p.a1), a2 = __ldg(p.a2), a3 = __ldg(p.a3);
    __syncthreads();

    const int r = lane >> 2, cq = (lane & 3) * 2;
    // TAC_input is used twice for every group: keep its fragments in registers (the h half of TAC_output is read from
    // shared memory where it is used: with it in registers too the kernel needed 168 registers = one CTA per SM)
    uint32_t w1h[6][2], w1l[6][2];
#pragma unroll
    for (int nt = 0; nt < 6; ++nt)
#pragma unroll
        for (int rg = 0; rg < 2; ++rg) { w1h[nt][rg] = F.w1[0][nt][rg][0][lane]; w1l[nt][rg] = F.w1[0][nt][rg][1][lane]; }
    const float invG = 1.0f / (float)G;
    const size_t Ls = (size_t)L;

    for (int tile = blockIdx.x * kTacWarps + warp; tile < total_tiles; tile += gridDim.x * kTacWarps) {
        const int b = tile / tiles_per_b;
        const int t0 = (tile - b * tiles_per_b) * 16;
        const bool v0 = t0 + r < L, v1 = t0 + r + 8 < L;
        // A fragments of X_g: rows = positions t0 + r (+8), k = channel cq (+1, +8, +9)
        auto load_x = [&](int g, uint32_t (&ah)[4], uint32_t (&al)[4]) {
            const float* xr = x + (((size_t)b * G + g) * 16 + cq) * Ls + t0 + r;
            const float x00 = v0 ? __ldg(xr) : 0.f,            x01 = v0 ? __ldg(xr + Ls) : 0.f;
            const float x10 = v1 ? __ldg(xr + 8) : 0.f,        x11 = v1 ? __ldg(xr + Ls + 8) : 0.f;
            const float x20 = v0 ? __ldg(xr + 8 * Ls) : 0.f,   x21 = v0 ? __ldg(xr + 9 * Ls) : 0.f;
            const float x30 = v1 ? __ldg(xr + 8 * Ls + 8) : 0.f, x31 = v1 ? __ldg(xr + 9 * Ls + 8) : 0.f;
            split_pair(x00, x01, ah[0], al[0]);
            split_pair(x10, x11, ah[1], al[1]);
            split_pair(x20, x21, ah[2], al[2]);
            split_pair(x30, x31, ah[3], al[3]);
        };
        // h_g = PReLU(X_g W1^T + b1) as 6 accumulator fragments
        auto hidden = [&](const uint32_t (&ah)[4], const uint32_t (&al)[4], float (&h)[6][4]) {
#pragma unroll
            for (int nt = 0; nt < 6; ++nt) {
                const float bb0 = F.b1[nt * 8 + cq], bb1 = F.b1[nt * 8 + cq + 1];
                h[nt][0] = bb0; h[nt][1] = bb1; h[nt][2] = bb0; h[nt][3] = bb1;
                mma3(h[nt], ah, al, w1h[nt][0], w1h[nt][1], w1l[nt][0], w1l[nt][1]);
#pragma unroll
                for (int e = 0; e < 4; ++e) h[nt][e] = h[nt][e] >= 0.f ? h[nt][e] : h[nt][e] * a1;
            }
        };

        // ---- pass 1: mean over groups of h_g ----
        float msum[6][4];
#pragma unroll
        for (int nt = 0; nt < 6; ++nt) { msum[nt][0] = msum[nt][1] = msum[nt][2] = msum[nt][3] = 0.f; }
#pragma unroll 1
        for (int g = 0; g < G; ++g) {
            uint32_t ah[4], al[4];
            float h[6][4];
            load_x(g, ah, al);
            hidden(ah, al, h);
#pragma unroll
            for (int nt = 0; nt < 6; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) msum[nt][e] += h[nt][e];
        }
#pragma unroll
        for (int nt = 0; nt < 6; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) msum[nt][e] *= invG;

        // ---- q = PReLU(mean W2^T + b2);  u = q W3[:, 48:]^T + b3 ----
        float u[2][4];
        {
            uint32_t mh[3][4], ml[3][4];
#pragma unroll
            for (int kt = 0; kt < 3; ++kt) acc_to_a(msum[2 * kt], msum[2 * kt + 1], mh[kt], ml[kt]);
            float q[6][4];
#pragma unroll
            for (int nt = 0; nt < 6; ++nt) {
                const float bb0 = F.b2[nt * 8 + cq], bb1 = F.b2[nt * 8 + cq + 1];
                q[nt][0] = bb0; q[nt][1] = bb1; q[nt][2] = bb0; q[nt][3] = bb1;
#pragma unroll
                for (int kt = 0; kt < 3; ++kt)
                    mma3(q[nt], mh[kt], ml[kt], F.w2[kt][nt][0][0][lane], F.w2[kt][nt][1][0][lane],
                         F.w2[kt][nt][0][1][lane], F.w2[kt][nt][1][1][lane]);
#pragma unroll
                for (int e = 0; e < 4; ++e) q[nt][e] = q[nt][e] >= 0.f ? q[nt][e] : q[nt][e] * a2;
            }
            uint32_t qh[3][4], ql[3][4];
#pragma unroll
            for (int kt = 0; kt < 3; ++kt) acc_to_a(q[2 * kt], q[2 * kt + 1], qh[kt], ql[kt]);
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) {
                const float bb0 = F.b3[nt * 8 + cq], bb1 = F.b3[nt * 8 + cq + 1];
                u[nt][0] = bb0; u[nt][1] = bb1; u[nt][2] = bb0; u[nt][3] = bb1;
#pragma unroll
                for (int kt = 0; kt < 3; ++kt)
                    mma3(u[nt], qh[kt], ql[kt], F.w3[3 + kt][nt][0][0][lane], F.w3[3 + kt][nt][1][0][lane],
                         F.w3[3 + kt][nt][0][1][lane], F.w3[3 + kt][nt][1][1][lane]);
            }
        }

        // ---- pass 2: o_g = PReLU(h_g W3[:, :48]^T + u), raw store + per-(b, g) statistics ----
#pragma unroll 1
        for (int g = 0; g < G; ++g) {
            uint32_t ah[4], al[4];
            float h[6][4];
            load_x(g, ah, al);
            hidden(ah, al, h);
            uint32_t hh[3][4], hl[3][4];
#pragma unroll
            for (int kt = 0; kt < 3; ++kt) acc_to_a(h[2 * kt], h[2 * kt + 1], hh[kt], hl[kt]);
            float st_s = 0.f, st_q = 0.f;
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) {
                float od[4] = {u[nt][0], u[nt][1], u[nt][2], u[nt][3]};
#pragma unroll
                for (int kt = 0; kt < 3; ++kt)
                    mma3(od, hh[kt], hl[kt], F.w3[kt][nt][0][0][lane], F.w3[kt][nt][1][0][lane],
                         F.w3[kt][nt][0][1][lane], F.w3[kt][nt][1][1][lane]);
#pragma unroll
                for (int e = 0; e < 4; ++e) od[e] = od[e] >= 0.f ? od[e] : od[e] * a3;
                float* orow = o + (((size_t)b * G + g) * 16 + nt * 8 + cq) * Ls + t0 + r;     // (channel nt*8 + cq, position t0 + r)
                if (v0) { orow[0] = od[0]; orow[Ls] = od[1]; st_s += od[0] + od[1]; st_q = fmaf(od[0], od[0], fmaf(od[1], od[1], st_q)); }
                if (v1) { orow[8] = od[2]; orow[Ls + 8] = od[3]; st_s += od[2] + od[3]; st_q = fmaf(od[2], od[2], fmaf(od[3], od[3], st_q)); }
            }
            const double ds = warp_sum_f64((double)st_s);
            const double dq = warp_sum_f64((double)st_q);
            if (lane == 0) {
                atomicAdd(stats + 2 * ((size_t)b * G + g), ds);
                atomicAdd(stats + 2 * ((size_t)b * G + g) + 1, dq);
            }
        }
    }
}

static int launch_tac_mma16(const float* x, const TacParams& p, float* o, double* stats, int B, int G, int L, cudaStream_t st) {
    const int tiles_per_b = (L + 15) / 16;
    const long long total = (long long)tiles_per_b * B;
    if (total > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    const int sms = sm_count();
    if (sms <= 0) return SDR_ERR_CUDA;
    long long grid = (total + kTacWarps - 1) / kTacWarps;
    if (grid > (long long)kTacMinB * sms) grid = (long long)kTacMinB * sms;                   // warps loop over tiles; the weight fragments are built once per CTA
    return launch(tac_mma16_kernel, (unsigned)grid, 32 * kTacWarps, sizeof(TacFrags), st, x, p, o, stats, G, L,
                  tiles_per_b, (int)total);
}

template <int NPG>
static int launch_tac_n(const float* x, const TacParams& p, float* o, double* stats,
                        int B, int G, int L, cudaStream_t st) {
    constexpr int H = 3 * NPG;
    const size_t floats = (size_t)H * NPG + H + (size_t)H * H + H + (size_t)NPG * 2 * H +
                          ((NPG + 3) & ~3) + 2 * (size_t)H * 32 + (size_t)NPG * 32 +
                          (size_t)NPG * G * 32;
    const size_t smem = floats * sizeof(float);
    if (smem > 220 * 1024) return SDR_ERR_UNSUPPORTED;
    const int t_tiles = (L + 31) / 32;
    const long long grid = (long long)t_tiles * B;
    if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    return launch(tac_kernel<NPG>, (unsigned)grid, 32 * G, smem, st, x, p, o, stats, G, L, t_tiles);
}

int launch_tac(const float* x, const float* const* params, float* o, double* stats,
               int B, int G, int n, int L, cudaStream_t st) {
    if (B <= 0 || G <= 0 || n <= 0 || L <= 0 || !params) return SDR_ERR_BAD_ARGUMENT;
    if (G > 16) return SDR_ERR_UNSUPPORTED;      // CTA = 32*G threads
    TacParams p{params[0], params[1], params[2], params[3], params[4],
                params[5], params[6], params[7], params[8]};
    switch (n) {
        case 4:  return launch_tac_n<4>(x, p, o, stats, B, G, L, st);
        case 8:  return launch_tac_n<8>(x, p, o, stats, B, G, L, st);
        case 16: return launch_tac_mma16(x, p, o, stats, B, G, L, st);      // tensor cores (any G <= 16)
        case 32: return launch_tac_n<32>(x, p, o, stats, B, G, L, st);
        default: return SDR_ERR_UNSUPPORTED;     // channels per group must be 4, 8, 16 or 32
    }
}

// out[bg, i, t] = x[bg, i, t] + GlobLN_{bg}(o)[bg, i, t]   (groupcomm_sudormrf_v2.py:381-383)
__global__ void __launch_bounds__(256)
tac_apply_kernel(const float* __restrict__ x, const float* __restrict__ o, NormIn nin,
                 float* __restrict__ out, int n, int L, int chunks_per_sample) {
    __shared__ SampleNorm s_norm;
    const int sample = blockIdx.x / chunks_per_sample;       // sample = b*G + g
    const int chunk = blockIdx.x - sample * chunks_per_sample;
    if (threadIdx.x == 0) s_norm = sample_norm(nin, sample);
    __syncthreads();
    const SampleNorm sn = s_norm;
    const int items = n * L;
    const size_t base = (size_t)sample * items;
    for (int it = 0; it < 4; ++it) {
        const int item = (chunk * 4 + it) * 256 + threadIdx.x;
        if (item < items) {
            const ChanNorm cn = chan_norm(nin, sn, item / L);
            out[base + item] = __ldg(x + base + item) + apply_norm(cn, __ldg(o + base + item));
        }
    }
}

int launch_tac_apply(const float* x, const float* o, const NormIn& nin, float* out,
                     int samples, int n, int L, cudaStream_t st) {
    const long long items = (long long)n * L;
    if (items > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;                // the kernel counts a sample's items in int
    const int chunks = (int)((items + 1023) / 1024);
    const long long grid = (long long)chunks * samples;
    if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    return launch(tac_apply_kernel, (unsigned)grid, 256, 0, st, x, o, nin, out, n, L, chunks);
}

}  // namespace sdr
