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

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Block-wide (sum, sumsq) -> one fp64 atomic pair per CTA on stats[2*sample].
// All threads of the block must call it.  `red` is >= 2*32 floats of shared memory.
__device__ __forceinline__ void block_stats_atomic(float s, float q, double* stats, int sample,
                                                   float* red) {
    s = warp_sum(s);
    q = warp_sum(q);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nwarps = (blockDim.x + 31) >> 5;
    if (lane == 0) { red[warp] = s; red[32 + warp] = q; }
    __syncthreads();
    if (warp == 0) {
        double ds = (lane < nwarps) ? (double)red[lane] : 0.0;
        double dq = (lane < nwarps) ? (double)red[32 + lane] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            ds += __shfl_xor_sync(0xffffffffu, ds, o);
            dq += __shfl_xor_sync(0xffffffffu, dq, o);
        }
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

}  // namespace sdr
