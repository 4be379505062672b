// Shared device helpers for the SuDoRM-RF sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/sudormrf_b200.h"

namespace sdr {

constexpr int kMaxDepthApi = 8;   // deepest upsampling_depth the kernels take
constexpr float kGlnEps = 1e-8f;   // improved_sudormrf.py:47  (var + 1e-8).sqrt()

// Deferred GlobLN (+PReLU) applied while loading a producer's raw output.
// Device-side copy of sdr_norm_in (same fields, kept POD so it can be passed by
// value as a kernel argument).
struct NormIn {
    const double* stats;
    const float* gamma;
    const float* beta;
    const float* prelu;
    double count;
    int prelu_pc;          // 1: one PReLU slope per channel (the original model, sudormrf.py:33,71); 0: one shared slope
};

__host__ inline NormIn make_norm(const sdr_norm_in* n) {
    NormIn r{nullptr, nullptr, nullptr, nullptr, 1.0, 0};
    if (n) {
        r.stats = n->stats; r.gamma = n->gamma; r.beta = n->beta; r.prelu = n->prelu; r.count = n->count;
        r.prelu_pc = n->prelu_per_channel != 0;
    }
    return r;
}

// Per-sample normalisation scalars, computed from the fp64 (sum, sumsq).
struct SampleNorm {
    float mean;
    float rstd;
};

__device__ __forceinline__ SampleNorm sample_norm(const NormIn& n, int sample) {
    SampleNorm s{0.f, 1.f};
    if (n.stats) {
        const double sum = n.stats[2 * (size_t)sample];
        const double sq = n.stats[2 * (size_t)sample + 1];
        const double mu = sum / n.count;
        double var = sq / n.count - mu * mu;      // biased variance, as the reference
        var = var < 0.0 ? 0.0 : var;
        s.mean = (float)mu;
        s.rstd = (float)(1.0 / sqrt(var + (double)kGlnEps));
    }
    return s;
}

// Per-(sample, channel) affine: y = (x - mean) * a + b, then PReLU.
struct ChanNorm {
    float mean, a, b, slope;
    bool act;
};

__device__ __forceinline__ ChanNorm chan_norm(const NormIn& n, const SampleNorm& s, int c) {
    ChanNorm r;
    r.mean = s.mean;
    r.a = 1.f; r.b = 0.f;
    if (n.stats) { r.a = __ldg(n.gamma + c) * s.rstd; r.b = __ldg(n.beta + c); }
    r.act = n.prelu != nullptr;
    r.slope = r.act ? __ldg(n.prelu + (n.prelu_pc ? c : 0)) : 1.f;
    return r;
}

__device__ __forceinline__ float apply_norm(const ChanNorm& c, float x) {
    float y = fmaf(x - c.mean, c.a, c.b);
    return (y >= 0.f) ? y : y * c.slope;          // slope == 1 when no activation
}

// The same GlobLN with the mean folded into the shift: y = x * a + b, a = gamma * rstd, b = beta - mean * a (one fmaf
// per element; no PReLU fields).  ChanNorm subtracts the mean first and FoldedNorm folds it in, so the two round
// differently and are NOT interchangeable: each kernel keeps the one it was validated with.
struct FoldedNorm { float a, b; };
__device__ __forceinline__ FoldedNorm fold_norm(const NormIn& n, const SampleNorm& s, int c) {
    FoldedNorm f{1.f, 0.f};
    if (n.stats) { f.a = __ldg(n.gamma + c) * s.rstd; f.b = fmaf(-s.mean, f.a, __ldg(n.beta + c)); }
    return f;
}

// ReLU as torch.relu: NaN stays NaN (fmaxf(NaN, 0) would be 0 and hide a corrupt mixture).  max.NaN is fmaxf's one
// instruction with NaN propagation, so every other value, signed zeros included, comes out as fmaxf(v, 0) does.
__device__ __forceinline__ float relu(float v) {
    float r;
    asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(r) : "f"(v));
    return r;
}

// PReLU in two instructions: max(v, s*v) for s <= 1, min otherwise (the caller decides the slope's side of 1 once)
__device__ __forceinline__ float prelu2(float v, float s, bool s_le1) {
    const float t = v * s;
    return s_le1 ? fmaxf(v, t) : fminf(v, t);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Per-thread (sum, sumsq) of a producer's output.  The squares of a sample offset by r standard deviations are about
// r^2 times its variance, and the variance is what survives sumsq/n - mean^2, so a long fp32 chain loses it: values are
// summed in fp32 over a short run (at most 16 outputs, add_run) and the runs in fp64.
struct StatAcc {
    double s = 0.0, q = 0.0;
    __device__ __forceinline__ void add(float v) { s += (double)v; q = fma((double)v, (double)v, q); }
    __device__ __forceinline__ void add_run(float rs, float rq) { s += (double)rs; q += (double)rq; }
    template <int N> __device__ __forceinline__ void add_run(const float (&o)[N]) {
        float rs = 0.f, rq = 0.f;
#pragma unroll
        for (int i = 0; i < N; ++i) { rs += o[i]; rq = fmaf(o[i], o[i], rq); }
        add_run(rs, rq);
    }
};

// Block-wide (sum, sumsq) -> one fp64 atomic pair per CTA on stats[2*sample], reduced in fp64 from the thread up.
// All threads of the block must call it.  `red` is >= 2*32 doubles of shared memory.
__device__ __forceinline__ void block_stats_atomic(const StatAcc& acc, double* stats, int sample, double* red) {
    const double s = warp_sum_f64(acc.s);
    const double q = warp_sum_f64(acc.q);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nwarps = (blockDim.x + 31) >> 5;
    if (lane == 0) { red[warp] = s; red[32 + warp] = q; }
    __syncthreads();
    if (warp == 0) {
        const double ds = warp_sum_f64((lane < nwarps) ? red[lane] : 0.0);
        const double dq = warp_sum_f64((lane < nwarps) ? red[32 + lane] : 0.0);
        if (lane == 0) {
            atomicAdd(stats + 2 * (size_t)sample, ds);
            atomicAdd(stats + 2 * (size_t)sample + 1, dq);
        }
    }
}

__device__ __forceinline__ float4 ldg4(const float* p) {
    return __ldg(reinterpret_cast<const float4*>(p));
}

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// CTAs per item of the fp64 reductions over time that end in per-(item, chunk) sums (the SDR Gram pass, the mixture
// consistency backward): one per 4096 samples, 1..64.
inline int gram_chunks(long long T) {
    const long long c = (T + 4095) / 4096;
    return (int)(c < 1 ? 1 : (c > 64 ? 64 : c));
}

// Grid of an elementwise pass of 256-thread CTAs over `rows` rows of T samples: x tiles of 1024 samples (1..4096) and
// y rows (at most 65535); the kernel strides over the time and the rows beyond the grid.
inline dim3 row_tiled_grid(long long rows, long long T) {
    long long gx = (T + 256 * 4 - 1) / (256 * 4);
    gx = gx < 1 ? 1 : (gx > 4096 ? 4096 : gx);
    return dim3((unsigned)gx, (unsigned)(rows < 65535 ? rows : 65535));
}

}  // namespace sdr
