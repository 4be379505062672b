// Depthwise stage of the causal U-ConvBlock (causal_improved_sudormrf_v3.py:57-118) in ONE pass.
//
// The causal block has no normalisation layers, so every level is a local function of its input:
//   o_0 = PReLU_0(dw_0(PReLU_p(y)))                      stride 1        (:106)
//   o_d = PReLU_d(dw_d(o_{d-1}))            d = 1..D-1,  stride 2        (:109-111)
//   m[t] = sum_d o_d[t >> d]                             nearest upsampling + adds   (:114-116)
// with dw_d the 21-tap depthwise filter under the causal mask (ScaledWSConv1d.get_weight, :21-27): the last 10
// taps are zero, so out[p] = b + sum_{j=0..10} w[j] * in[stride * p - 10 + j], in[] zero for negative indices
// (the symmetric padding only ever reaches the left edge: stride * p <= L_in - 1).
//
// One CTA owns a window of W output positions of one (sample, channel) row.  The halo is on the left only:
// level d is computed from (t0 >> d) - h_d with h_{D-1} = 0, h_{d-1} = 2 h_d + 12 (10 taps of history, rounded
// so that every level's buffer starts on a float4 boundary); y is read from t0 - h_0 - 12.  All levels live in
// shared memory; each thread produces four consecutive outputs of a level from 4-5 LDS.128 of its input; the
// merge reads every level once and stores float4.  HBM traffic: y once (+ halo, from L2) and m once,
// 8 B per (row, position) against the 5 round trips of a level-by-level schedule.
#include "common.cuh"
#include "launchers.cuh"

namespace sdr {

constexpr int kCzThreads = 256;      // upper bound; the host picks the block size (a multiple of 32) that leaves the fewest idle lanes
constexpr int kCzWindow = 4096;      // positions per CTA (upper bound; the host balances the windows of a row).  ncu of the
                                     // 2 x 1600-position windows of a 3200-position row with 256 threads (profiles/r02b_kernels.md):
                                     // 421 / 209 / 103 / 50 quads per level against 256 lanes = 66 % of the issued lanes useful,
                                     // barrier the second stall reason; a whole row per CTA with 160 threads: 800 / 400 / 200 / 100
                                     // quads = 5 / 2.5 / 1.25 / 0.6 passes (90 %), no halo, 6 CTAs per SM
constexpr int kCzTaps = 11;          // taps that survive the causal mask of a 21-tap filter
constexpr int kCzFilter = 21;
constexpr int kCzSlack = 8;          // floats of slack after every level buffer (the last, ragged quad of a level)

struct CausalPyrArgs {
    const float* y;                  // [rows][L] raw proj_1x1 output (bias included)
    float* m;                        // [rows][L] merged output
    const float* slope_in;           // proj_1x1.act.weight
    const float* w[kMaxDepthApi];    // spp_dw[d].conv.weight [C][1][21] (reference layout; taps 0..10 are read)
    const float* b[kMaxDepthApi];    // spp_dw[d].conv.bias   [C]
    const float* slope[kMaxDepthApi];// spp_dw[d].act.weight
    int D, C, L, W, tiles;           // W: window (multiple of 4 << (D-1)); tiles per row
    int h[kMaxDepthApi];             // left halo of level d, in level-d positions
    int off[kMaxDepthApi];           // float offset of level d's buffer in shared memory (y's buffer is at 0)
};

__global__ void __launch_bounds__(kCzThreads)
causal_pyramid_kernel(const CausalPyrArgs a) {
    extern __shared__ __align__(16) float smem[];
    // (Staging the 13 parameters of every level in 512 B of static shared memory instead of 13 __ldg per level and thread
    //  measured 222 us against 199 us: the extra bytes cost the sixth resident CTA, profiles/r02b_kernels.md.)
    const int tid = threadIdx.x, nthr = blockDim.x;
    const long long row = blockIdx.x / a.tiles;
    const int tile = (int)(blockIdx.x - row * a.tiles);
    const int c = (int)(row % a.C);
    const int t0 = tile * a.W;
    const int Wt = min(a.W, a.L - t0);
    const int D = a.D;

    // ---- y window -> shared memory, PReLU of proj_1x1 applied on the way (zero left of the row: the conv's padding)
    {
        const float sp = __ldg(a.slope_in);
        const bool sp1 = sp <= 1.f;
        const int hy = a.h[0] + 12;
        const int nq = (Wt + hy) >> 2;
        const float* src = a.y + row * a.L;
        const int g0 = t0 - hy;                         // multiple of 4
        for (int q = tid; q < nq; q += nthr) {
            const int g = g0 + 4 * q;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (g >= 0) {
                v = ldg4(src + g);
                v.x = prelu2(v.x, sp, sp1); v.y = prelu2(v.y, sp, sp1); v.z = prelu2(v.z, sp, sp1); v.w = prelu2(v.w, sp, sp1);
            }
            *reinterpret_cast<float4*>(smem + 4 * q) = v;
        }
    }
    __syncthreads();

    // ---- levels (unrolled over the compile-time bound so that the per-level fields of the argument struct are read
    // from constant parameter space instead of a local copy)
#pragma unroll
    for (int d = 0; d < kMaxDepthApi; ++d) {
        if (d >= D) continue;                           // uniform across the CTA: the barriers below stay matched
        float w[kCzTaps];
        const float* wp = a.w[d] + (size_t)c * kCzFilter;
#pragma unroll
        for (int j = 0; j < kCzTaps; ++j) w[j] = __ldg(wp + j);
        const float bias = __ldg(a.b[d] + c);
        const float sl = __ldg(a.slope[d]);
        const bool sl1 = sl <= 1.f;
        const float* in = d == 0 ? smem : smem + a.off[d - 1];
        float* out = smem + a.off[d];
        const int n = (Wt >> d) + a.h[d];               // outputs of this level in the window (halo included)
        const int org = (t0 >> d) - a.h[d];             // global index of out[0]
        const int nq = (n + 3) >> 2;
        if (d == 0) {
            for (int q = tid; q < nq; q += nthr) {
                if (org + 4 * q + 3 < 0) {                   // left of the row (first window's halo): the padding zeros
                    *reinterpret_cast<float4*>(out + 4 * q) = make_float4(0.f, 0.f, 0.f, 0.f);
                    continue;
                }
                float x[16];
#pragma unroll
                for (int v = 0; v < 4; ++v) {
                    const float4 f = *reinterpret_cast<const float4*>(in + 4 * q + 4 * v);
                    x[4 * v] = f.x; x[4 * v + 1] = f.y; x[4 * v + 2] = f.z; x[4 * v + 3] = f.w;
                }
                float o[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    float acc = bias;
#pragma unroll
                    for (int j = 0; j < kCzTaps; ++j) acc = fmaf(w[j], x[u + 2 + j], acc);
                    o[u] = prelu2(acc, sl, sl1);            // (org is a multiple of 4: a quad is entirely left of the row, skipped above, or inside)
                }
                *reinterpret_cast<float4*>(out + 4 * q) = make_float4(o[0], o[1], o[2], o[3]);
            }
        } else {
            for (int q = tid; q < nq; q += nthr) {
                if (org + 4 * q + 3 < 0) {
                    *reinterpret_cast<float4*>(out + 4 * q) = make_float4(0.f, 0.f, 0.f, 0.f);
                    continue;
                }
                float x[20];
#pragma unroll
                for (int v = 0; v < 5; ++v) {
                    const float4 f = *reinterpret_cast<const float4*>(in + 8 * q + 4 * v);
                    x[4 * v] = f.x; x[4 * v + 1] = f.y; x[4 * v + 2] = f.z; x[4 * v + 3] = f.w;
                }
                float o[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    float acc = bias;
#pragma unroll
                    for (int j = 0; j < kCzTaps; ++j) acc = fmaf(w[j], x[2 * u + 2 + j], acc);
                    o[u] = prelu2(acc, sl, sl1);            // (org is a multiple of 4: a quad is entirely left of the row, skipped above, or inside)
                }
                *reinterpret_cast<float4*>(out + 4 * q) = make_float4(o[0], o[1], o[2], o[3]);
            }
        }
        __syncthreads();
    }

    // ---- merge: m[t] = sum_d o_d[t >> d], four positions per thread
    {
        float* dst = a.m + row * a.L + t0;
        for (int q = tid; q < (Wt >> 2); q += nthr) {
            const int t = 4 * q;                         // relative to t0 (t0 is a multiple of 4 << (D-1))
            float4 v = *reinterpret_cast<const float4*>(smem + a.off[0] + a.h[0] + t);
            if (D > 1) {
                const float* o1 = smem + a.off[1] + a.h[1] + (t >> 1);
                const float p = o1[0], r = o1[1];
                v.x += p; v.y += p; v.z += r; v.w += r;
                float deep = 0.f;
#pragma unroll
                for (int d = 2; d < kMaxDepthApi; ++d)
                    if (d < D) deep += smem[a.off[d] + a.h[d] + (t >> d)];
                v.x += deep; v.y += deep; v.z += deep; v.w += deep;
            }
            *reinterpret_cast<float4*>(dst + t) = v;
        }
    }
}

// Shapes the one-pass kernel takes: float4 rows and a length that halves exactly D times (every padded length
// of the model does: pad_to_appropriate_length rounds to hop * 2^D samples, :213-224).
bool causal_pyramid_eligible(int D, int L) {
    return D >= 1 && D <= kMaxDepthApi && L > 0 && (L % 4) == 0 && (L % (1 << D)) == 0;
}

int launch_causal_pyramid(const float* y, const float* slope_in, const float* const* w, const float* const* b,
                          const float* const* slope, float* m, int D, int samples, int C, int L, cudaStream_t st) {
    if (!y || !m || !slope_in || !w || !b || !slope || samples <= 0 || C <= 0) return SDR_ERR_BAD_ARGUMENT;
    if (!causal_pyramid_eligible(D, L)) return SDR_ERR_UNSUPPORTED;
    CausalPyrArgs a;
    a.y = y; a.m = m; a.slope_in = slope_in; a.D = D; a.C = C; a.L = L;
    for (int d = 0; d < kMaxDepthApi; ++d) {
        a.w[d] = d < D ? w[d] : nullptr; a.b[d] = d < D ? b[d] : nullptr; a.slope[d] = d < D ? slope[d] : nullptr;
        a.h[d] = 0; a.off[d] = 0;
    }
    const int gran = D == 1 ? 4 : 4 << (D - 1);        // a window start must be a float4 boundary at every level
    const int tiles = ceil_div(L, kCzWindow);
    a.W = ceil_div(ceil_div(L, tiles), gran) * gran;
    a.tiles = ceil_div(L, a.W);
    for (int d = D - 2; d >= 0; --d) a.h[d] = 2 * a.h[d + 1] + 12;
    size_t cur = (size_t)a.W + a.h[0] + 12 + kCzSlack;   // y's buffer
    for (int d = 0; d < D; ++d) {
        a.off[d] = (int)cur;
        cur += (size_t)(((a.W >> d) + a.h[d] + 3) & ~3) + kCzSlack;
    }
    const size_t smem = cur * sizeof(float);
    if (smem > 200 * 1024) return SDR_ERR_UNSUPPORTED;
    const long long grid = (long long)samples * C * a.tiles;
    if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    // block size: measured at the default model's rows (L = 3200, D = 4, one window per row, 6 CTAs per SM by shared
    // memory): 128 / 160 / 192 / 224 / 256 threads = 206 / 192 / 187 / 193 / 196 us; short windows take fewer threads
    int threads = 192;
    while (threads > 128 && (a.W >> 2) < threads) threads -= 32;
    return launch(causal_pyramid_kernel, (unsigned)grid, threads, smem, st, a);
}

// ---------------------------------------------------------------------------
// pack-time helpers of the causal model
// ---------------------------------------------------------------------------
// encoder.weight [rows][src_taps] -> [rows][dst_taps]: the taps the causal mask keeps (:21-27)
__global__ void take_taps_kernel(const float* __restrict__ src, float* __restrict__ dst, long long rows,
                                 int src_taps, int dst_taps) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * dst_taps) return;
    const long long r = i / dst_taps;
    const int j = (int)(i - r * dst_taps);
    dst[i] = src[r * src_taps + j];
}

// res_conv(x) * skipinit_gain * alpha (:118) == (gain * W) x + gain * b: the gain is folded into the packed weights
__global__ void scale_by_scalar_kernel(const float* __restrict__ src, const float* __restrict__ gain,
                                       float* __restrict__ dst, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i] * __ldg(gain);
}

int launch_take_taps(const float* src, float* dst, long long rows, int src_taps, int dst_taps, cudaStream_t st) {
    const long long n = rows * dst_taps;
    return launch(take_taps_kernel, (unsigned)((n + 255) / 256), 256, 0, st, src, dst, rows, src_taps, dst_taps);
}

int launch_scale_by_scalar(const float* src, const float* gain, float* dst, long long n, cudaStream_t st) {
    return launch(scale_by_scalar_kernel, (unsigned)((n + 255) / 256), 256, 0, st, src, gain, dst, n);
}

}  // namespace sdr
