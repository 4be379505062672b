// U-ConvBlock level kernels (HBM-bound): depthwise k=5 stride 1|2 with the
// producer's GlobLN(+PReLU) applied on load, and the multi-resolution merge.
//
// Reference semantics:
//   DilatedConvNorm  improved_sudormrf.py:138-159  (Conv1d k=5, pad 2, groups=C, then GlobLN)
//   UConvBlock.forward level loops  improved_sudormrf.py:206-216
// Each kernel stores its RAW result once and accumulates the (sum, sumsq) of
// that result per sample in fp64 so the consumer can normalise while loading.
#include "common.cuh"
#include "launchers.cuh"

namespace sdr {

constexpr int kDwThreads = 256;
constexpr int kDwItems = 2;        // output quads per thread

// ---------------------------------------------------------------------------
// depthwise, vector path: one item = 4 consecutive outputs of one (sample, c) row
// requires Lout % 4 == 0 (then Lin % 4 == 0 as well).
// ---------------------------------------------------------------------------
template <int STRIDE>
__global__ void __launch_bounds__(kDwThreads)
dw5_vec_kernel(const float* __restrict__ x, NormIn nin,
               const float* __restrict__ w5, const float* __restrict__ bias,
               float* __restrict__ y, double* __restrict__ stats_out,
               int C, int Lin, int Lout, int chunks_per_sample) {
    __shared__ SampleNorm s_norm;
    __shared__ double s_red[64];
    const int sample = blockIdx.x / chunks_per_sample;
    const int chunk = blockIdx.x - sample * chunks_per_sample;
    if (threadIdx.x == 0) s_norm = sample_norm(nin, sample);
    __syncthreads();
    const SampleNorm sn = s_norm;

    const int QR = Lout >> 2;                 // quads per row
    const int items = C * QR;                 // per sample
    const float* xs = x + (size_t)sample * C * Lin;
    float* ys = y + (size_t)sample * C * Lout;

    StatAcc acc;
#pragma unroll
    for (int it = 0; it < kDwItems; ++it) {
        const int item = (chunk * kDwItems + it) * kDwThreads + threadIdx.x;
        if (item < items) {
            const int c = item / QR;
            const int q = item - c * QR;
            const ChanNorm cn = chan_norm(nin, sn, c);
            const float* xr = xs + (size_t)c * Lin;
            float w[5];
#pragma unroll
            for (int j = 0; j < 5; ++j) w[j] = __ldg(w5 + c * 5 + j);
            const float b = __ldg(bias + c);
            float o[4];
            if (STRIDE == 1) {
                // window v[0..7] = positions 4q-2 .. 4q+5
                float v[8];
                const float4 m = ldg4(xr + 4 * q);
                v[2] = apply_norm(cn, m.x); v[3] = apply_norm(cn, m.y);
                v[4] = apply_norm(cn, m.z); v[5] = apply_norm(cn, m.w);
                if (q > 0) {
                    const float2 l = __ldg(reinterpret_cast<const float2*>(xr + 4 * q - 2));
                    v[0] = apply_norm(cn, l.x); v[1] = apply_norm(cn, l.y);
                } else { v[0] = 0.f; v[1] = 0.f; }
                if (q < QR - 1) {
                    const float2 r = __ldg(reinterpret_cast<const float2*>(xr + 4 * q + 4));
                    v[6] = apply_norm(cn, r.x); v[7] = apply_norm(cn, r.y);
                } else { v[6] = 0.f; v[7] = 0.f; }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    float a = b;
#pragma unroll
                    for (int j = 0; j < 5; ++j) a = fmaf(w[j], v[i + j], a);
                    o[i] = a;
                }
            } else {
                // outputs 4q..4q+3 read inputs 8q-2 .. 8q+8 ; window v[0..10]
                float v[11];
                const float4 m0 = ldg4(xr + 8 * q);
                const float4 m1 = ldg4(xr + 8 * q + 4);
                v[2] = apply_norm(cn, m0.x); v[3] = apply_norm(cn, m0.y);
                v[4] = apply_norm(cn, m0.z); v[5] = apply_norm(cn, m0.w);
                v[6] = apply_norm(cn, m1.x); v[7] = apply_norm(cn, m1.y);
                v[8] = apply_norm(cn, m1.z); v[9] = apply_norm(cn, m1.w);
                if (q > 0) {
                    const float2 l = __ldg(reinterpret_cast<const float2*>(xr + 8 * q - 2));
                    v[0] = apply_norm(cn, l.x); v[1] = apply_norm(cn, l.y);
                } else { v[0] = 0.f; v[1] = 0.f; }
                v[10] = (8 * q + 8 < Lin) ? apply_norm(cn, __ldg(xr + 8 * q + 8)) : 0.f;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    float a = b;
#pragma unroll
                    for (int j = 0; j < 5; ++j) a = fmaf(w[j], v[2 * i + j], a);
                    o[i] = a;
                }
            }
            *reinterpret_cast<float4*>(ys + (size_t)c * Lout + 4 * q) = make_float4(o[0], o[1], o[2], o[3]);
            acc.add_run(o);
        }
    }
    block_stats_atomic(acc, stats_out, sample, s_red);
}

// scalar fallback (any Lin/Lout): one output element per thread-iteration
__global__ void __launch_bounds__(kDwThreads)
dw5_scalar_kernel(const float* __restrict__ x, NormIn nin,
                  const float* __restrict__ w5, const float* __restrict__ bias,
                  float* __restrict__ y, double* __restrict__ stats_out,
                  int C, int Lin, int Lout, int stride, int chunks_per_sample) {
    __shared__ SampleNorm s_norm;
    __shared__ double s_red[64];
    const int sample = blockIdx.x / chunks_per_sample;
    const int chunk = blockIdx.x - sample * chunks_per_sample;
    if (threadIdx.x == 0) s_norm = sample_norm(nin, sample);
    __syncthreads();
    const SampleNorm sn = s_norm;
    const int items = C * Lout;
    const float* xs = x + (size_t)sample * C * Lin;
    float* ys = y + (size_t)sample * C * Lout;
    StatAcc acc;
    for (int it = 0; it < 4; ++it) {
        const int item = (chunk * 4 + it) * kDwThreads + threadIdx.x;
        if (item < items) {
            const int c = item / Lout;
            const int t = item - c * Lout;
            const ChanNorm cn = chan_norm(nin, sn, c);
            float a = __ldg(bias + c);
#pragma unroll
            for (int j = 0; j < 5; ++j) {
                const int p = t * stride + j - 2;
                if (p >= 0 && p < Lin)
                    a = fmaf(__ldg(w5 + c * 5 + j), apply_norm(cn, __ldg(xs + (size_t)c * Lin + p)), a);
            }
            ys[(size_t)c * Lout + t] = a;
            acc.add(a);
        }
    }
    block_stats_atomic(acc, stats_out, sample, s_red);
}

// ---------------------------------------------------------------------------
// merge: m[c,t] = sum_d norm_d(z_d)[c, t >> d]   (closed form of the
// upsample(scale 2, nearest)+add chain, improved_sudormrf.py:214-216)
// ---------------------------------------------------------------------------
constexpr int kMaxDepth = kMaxDepthApi;
struct MergeArgs {
    const float* z[kMaxDepth];
    NormIn n[kMaxDepth];
    int depth;
};

constexpr int kMgThreads = 256;
constexpr int kMgItems = 2;

// vector path: L % 4 == 0 and L % 2^(depth-1) == 0
__global__ void __launch_bounds__(kMgThreads)
merge_vec_kernel(MergeArgs a, float* __restrict__ m, double* __restrict__ stats_out,
                 int C, int L, int chunks_per_sample) {
    __shared__ SampleNorm s_norm[kMaxDepth];
    __shared__ double s_red[64];
    const int sample = blockIdx.x / chunks_per_sample;
    const int chunk = blockIdx.x - sample * chunks_per_sample;
    if (threadIdx.x < a.depth) s_norm[threadIdx.x] = sample_norm(a.n[threadIdx.x], sample);
    __syncthreads();

    const int QR = L >> 2;
    const int items = C * QR;
    StatAcc acc;
#pragma unroll
    for (int it = 0; it < kMgItems; ++it) {
        const int item = (chunk * kMgItems + it) * kMgThreads + threadIdx.x;
        if (item < items) {
            const int c = item / QR;
            const int q = item - c * QR;
            const size_t row = (size_t)sample * C + c;
            float o[4];
            {
                const ChanNorm cn = chan_norm(a.n[0], s_norm[0], c);
                const float4 v = ldg4(a.z[0] + row * L + 4 * q);
                o[0] = apply_norm(cn, v.x); o[1] = apply_norm(cn, v.y);
                o[2] = apply_norm(cn, v.z); o[3] = apply_norm(cn, v.w);
            }
            if (a.depth > 1) {
                const ChanNorm cn = chan_norm(a.n[1], s_norm[1], c);
                const float2 v = __ldg(reinterpret_cast<const float2*>(a.z[1] + row * (L >> 1) + 2 * q));
                const float v0 = apply_norm(cn, v.x), v1 = apply_norm(cn, v.y);
                o[0] += v0; o[1] += v0; o[2] += v1; o[3] += v1;
            }
            for (int d = 2; d < a.depth; ++d) {
                const ChanNorm cn = chan_norm(a.n[d], s_norm[d], c);
                const float v = apply_norm(cn, __ldg(a.z[d] + row * (L >> d) + (q >> (d - 2))));
                o[0] += v; o[1] += v; o[2] += v; o[3] += v;
            }
            *reinterpret_cast<float4*>(m + row * L + 4 * q) = make_float4(o[0], o[1], o[2], o[3]);
            acc.add_run(o);
        }
    }
    block_stats_atomic(acc, stats_out, sample, s_red);
}

__global__ void __launch_bounds__(kMgThreads)
merge_scalar_kernel(MergeArgs a, float* __restrict__ m, double* __restrict__ stats_out,
                    int C, int L, int chunks_per_sample) {
    __shared__ SampleNorm s_norm[kMaxDepth];
    __shared__ double s_red[64];
    const int sample = blockIdx.x / chunks_per_sample;
    const int chunk = blockIdx.x - sample * chunks_per_sample;
    if (threadIdx.x < a.depth) s_norm[threadIdx.x] = sample_norm(a.n[threadIdx.x], sample);
    __syncthreads();
    const int items = C * L;
    StatAcc acc;
    for (int it = 0; it < 4; ++it) {
        const int item = (chunk * 4 + it) * kMgThreads + threadIdx.x;
        if (item < items) {
            const int c = item / L;
            const int t = item - c * L;
            const size_t row = (size_t)sample * C + c;
            float o = 0.f;
            for (int d = 0; d < a.depth; ++d) {
                const ChanNorm cn = chan_norm(a.n[d], s_norm[d], c);
                o += apply_norm(cn, __ldg(a.z[d] + row * (L >> d) + (t >> d)));
            }
            m[row * L + t] = o;
            acc.add(o);
        }
    }
    block_stats_atomic(acc, stats_out, sample, s_red);
}


// ---------------------------------------------------------------------------
// Wide paths (the ones the benchmark shapes take).  The narrow kernels above were
// instruction-issue bound (ncu: issue-active 70-80 %, DRAM 40-58 %): per output
// they paid ~30 instructions of parameter loads, index division and a 5-op
// normalise+PReLU.  Here a thread owns a run of 8 (depthwise) or 16 (merge)
// consecutive outputs of one row, the GlobLN mean is folded into the shift
// (y = x*a + b, a = gamma*rstd, b = beta - mean*a) and PReLU is 2 ops
// (t = y*slope; y = slope <= 1 ? max(y,t) : min(y,t)), so the kernels sit on the
// HBM roofline instead of the issue roofline.
// ---------------------------------------------------------------------------
template <bool ACT>
__device__ __forceinline__ float norm_act(float x, const FoldedNorm& f, float slope, bool slope_le1) {
    const float y = fmaf(x, f.a, f.b);
    return ACT ? prelu2(y, slope, slope_le1) : y;
}

// 128 threads x 4 runs (2 for the merge).  Every byte of these kernels is touched once, but the L1-bypass hints
// (ld.global.nc.L1::no_allocate + st.global.cs) measured slower on the stride-2 levels, so the accesses are plain.
constexpr int kDw8Threads = 128;
constexpr int kDw8Items = 4;         // runs of 8 outputs per thread

// requires Lout % 8 == 0
template <int STRIDE, bool ACT>
__global__ void __launch_bounds__(kDw8Threads)
dw5_wide_kernel(const float* __restrict__ x, NormIn nin,
                const float* __restrict__ w5, const float* __restrict__ bias,
                float* __restrict__ y, double* __restrict__ stats_out,
                int C, int Lin, int Lout, int chunks_per_sample) {
    __shared__ SampleNorm s_norm;
    __shared__ double s_red[64];
    const int sample = blockIdx.x / chunks_per_sample;
    const int chunk = blockIdx.x - sample * chunks_per_sample;
    if (threadIdx.x == 0) s_norm = sample_norm(nin, sample);
    const float slope = ACT ? __ldg(nin.prelu) : 1.f;
    const bool sle1 = slope <= 1.f;
    __syncthreads();
    const SampleNorm sn = s_norm;

    const int QR = Lout >> 3;                 // runs per row
    const int items = C * QR;                 // per sample
    const float* xs = x + (size_t)sample * C * Lin;
    float* ys = y + (size_t)sample * C * Lout;
    StatAcc acc;
#pragma unroll
    for (int it = 0; it < kDw8Items; ++it) {
        const int item = (chunk * kDw8Items + it) * kDw8Threads + threadIdx.x;
        if (item < items) {
            const int c = item / QR;
            const int q = item - c * QR;
            const FoldedNorm f = fold_norm(nin, sn, c);
            float w[5];
#pragma unroll
            for (int j = 0; j < 5; ++j) w[j] = __ldg(w5 + c * 5 + j);
            const float b = __ldg(bias + c);
            float o[8];
            if (STRIDE == 1) {
                const float* xr = xs + (size_t)c * Lin + 8 * q;       // window v[0..11] = positions 8q-2 .. 8q+9
                float v[12];
                const float4 m0 = ldg4(xr), m1 = ldg4(xr + 4);
                float2 l = make_float2(0.f, 0.f), r = make_float2(0.f, 0.f);
                const bool hl = q > 0, hr = q < QR - 1;
                if (hl) l = __ldg(reinterpret_cast<const float2*>(xr - 2));
                if (hr) r = __ldg(reinterpret_cast<const float2*>(xr + 8));
                v[0] = hl ? norm_act<ACT>(l.x, f, slope, sle1) : 0.f;
                v[1] = hl ? norm_act<ACT>(l.y, f, slope, sle1) : 0.f;
                v[2] = norm_act<ACT>(m0.x, f, slope, sle1); v[3] = norm_act<ACT>(m0.y, f, slope, sle1);
                v[4] = norm_act<ACT>(m0.z, f, slope, sle1); v[5] = norm_act<ACT>(m0.w, f, slope, sle1);
                v[6] = norm_act<ACT>(m1.x, f, slope, sle1); v[7] = norm_act<ACT>(m1.y, f, slope, sle1);
                v[8] = norm_act<ACT>(m1.z, f, slope, sle1); v[9] = norm_act<ACT>(m1.w, f, slope, sle1);
                v[10] = hr ? norm_act<ACT>(r.x, f, slope, sle1) : 0.f;
                v[11] = hr ? norm_act<ACT>(r.y, f, slope, sle1) : 0.f;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    float a = b;
#pragma unroll
                    for (int j = 0; j < 5; ++j) a = fmaf(w[j], v[i + j], a);
                    o[i] = a;
                }
            } else {
                const float* xr = xs + (size_t)c * Lin + 16 * q;      // window v[0..18] = positions 16q-2 .. 16q+16
                float v[19];
                const float4 m0 = ldg4(xr), m1 = ldg4(xr + 4), m2 = ldg4(xr + 8), m3 = ldg4(xr + 12);
                float2 l = make_float2(0.f, 0.f);
                float r = 0.f;
                const bool hl = q > 0, hr = 16 * q + 16 < Lin;
                if (hl) l = __ldg(reinterpret_cast<const float2*>(xr - 2));
                if (hr) r = __ldg(xr + 16);
                v[0] = hl ? norm_act<ACT>(l.x, f, slope, sle1) : 0.f;
                v[1] = hl ? norm_act<ACT>(l.y, f, slope, sle1) : 0.f;
                const float mm[16] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w,
                                      m2.x, m2.y, m2.z, m2.w, m3.x, m3.y, m3.z, m3.w};
#pragma unroll
                for (int i = 0; i < 16; ++i) v[2 + i] = norm_act<ACT>(mm[i], f, slope, sle1);
                v[18] = hr ? norm_act<ACT>(r, f, slope, sle1) : 0.f;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    float a = b;
#pragma unroll
                    for (int j = 0; j < 5; ++j) a = fmaf(w[j], v[2 * i + j], a);
                    o[i] = a;
                }
            }
            float* yr = ys + (size_t)c * Lout + 8 * q;
            *reinterpret_cast<float4*>(yr) = make_float4(o[0], o[1], o[2], o[3]);
            *reinterpret_cast<float4*>(yr + 4) = make_float4(o[4], o[5], o[6], o[7]);
            acc.add_run(o);
        }
    }
    block_stats_atomic(acc, stats_out, sample, s_red);
}


// merge, 16 outputs per thread, coarse-to-fine: s_d[i] = z_d[i]*a_d + (b_d + s_{d+1}[i>>1])
// requires depth >= 4 and L % 16 == 0
constexpr int kMg16Threads = 128;
constexpr int kMg16Items = 2;
__global__ void __launch_bounds__(kMg16Threads)
merge_wide_kernel(MergeArgs a, float* __restrict__ m, double* __restrict__ stats_out,
                  int C, int L, int chunks_per_sample) {
    __shared__ SampleNorm s_norm[kMaxDepth];
    __shared__ double s_red[64];
    const int sample = blockIdx.x / chunks_per_sample;
    const int chunk = blockIdx.x - sample * chunks_per_sample;
    if (threadIdx.x < a.depth) s_norm[threadIdx.x] = sample_norm(a.n[threadIdx.x], sample);
    __syncthreads();
    const int QR = L >> 4;
    const int items = C * QR;
    StatAcc acc;
#pragma unroll
    for (int iti = 0; iti < kMg16Items; ++iti) {
      const int item = (chunk * kMg16Items + iti) * kMg16Threads + threadIdx.x;
      if (item < items) {
        const int c = item / QR;
        const int q = item - c * QR;
        const size_t row = (size_t)sample * C + c;
        // issue every load of this run first
        const float* z0 = a.z[0] + row * L + 16 * q;
        const float4 v00 = ldg4(z0), v01 = ldg4(z0 + 4), v02 = ldg4(z0 + 8), v03 = ldg4(z0 + 12);
        const float* z1 = a.z[1] + row * (L >> 1) + 8 * q;
        const float4 v10 = ldg4(z1), v11 = ldg4(z1 + 4);
        const float4 v2 = ldg4(a.z[2] + row * (L >> 2) + 4 * q);
        const float2 v3 = __ldg(reinterpret_cast<const float2*>(a.z[3] + row * (L >> 3) + 2 * q));
        float base = 0.f;                      // levels >= 4 are constant over the run
        for (int d = 4; d < a.depth; ++d) {
            const FoldedNorm f = fold_norm(a.n[d], s_norm[d], c);
            base += fmaf(__ldg(a.z[d] + row * (L >> d) + (q >> (d - 4))), f.a, f.b);
        }
        const FoldedNorm f3 = fold_norm(a.n[3], s_norm[3], c);
        const FoldedNorm f2 = fold_norm(a.n[2], s_norm[2], c);
        const FoldedNorm f1 = fold_norm(a.n[1], s_norm[1], c);
        const FoldedNorm f0 = fold_norm(a.n[0], s_norm[0], c);
        float s3[2], s2[4], s1[8], o[16];
        const float c3 = f3.b + base;
        s3[0] = fmaf(v3.x, f3.a, c3); s3[1] = fmaf(v3.y, f3.a, c3);
        const float z2v[4] = {v2.x, v2.y, v2.z, v2.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) s2[i] = fmaf(z2v[i], f2.a, f2.b + s3[i >> 1]);
        const float z1v[8] = {v10.x, v10.y, v10.z, v10.w, v11.x, v11.y, v11.z, v11.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) s1[i] = fmaf(z1v[i], f1.a, f1.b + s2[i >> 1]);
        const float z0v[16] = {v00.x, v00.y, v00.z, v00.w, v01.x, v01.y, v01.z, v01.w,
                               v02.x, v02.y, v02.z, v02.w, v03.x, v03.y, v03.z, v03.w};
#pragma unroll
        for (int i = 0; i < 16; ++i) o[i] = fmaf(z0v[i], f0.a, f0.b + s1[i >> 1]);
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
// host launchers
// ---------------------------------------------------------------------------
int launch_depthwise(const float* x, const NormIn& nin, const float* w5, const float* bias,
                     float* y, double* stats_out, int samples, int C, int Lin, int stride,
                     cudaStream_t st) {
    if (samples <= 0 || C <= 0 || Lin <= 0 || (stride != 1 && stride != 2)) return SDR_ERR_BAD_ARGUMENT;
    if ((long long)C * Lin > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;   // the kernels count a sample's items in int
    const int Lout = (Lin + 4 - 5) / stride + 1;
    const bool vec = (Lout % 4 == 0) && (stride == 1 || Lin == 2 * Lout) &&
                     ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) % 16 == 0);
    if (vec && (Lout % 8 == 0) && !nin.prelu_pc) {   // (per-channel PReLU slopes, the original model: dw5_vec_kernel reads them per channel)
        const long long items = (long long)C * (Lout / 8);
        const int per_cta = kDw8Threads * kDw8Items;
        const int chunks = (int)((items + per_cta - 1) / per_cta);
        const long long grid = (long long)chunks * samples;
        if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
        const bool act = nin.prelu != nullptr;
        const auto kern = stride == 1 ? (act ? dw5_wide_kernel<1, true> : dw5_wide_kernel<1, false>)
                                      : (act ? dw5_wide_kernel<2, true> : dw5_wide_kernel<2, false>);
        return launch(kern, (unsigned)grid, kDw8Threads, 0, st, x, nin, w5, bias, y, stats_out, C, Lin, Lout, chunks);
    } else if (vec) {
        const long long items = (long long)C * (Lout / 4);
        const int chunks = (int)((items + kDwThreads * kDwItems - 1) / (kDwThreads * kDwItems));
        const long long grid = (long long)chunks * samples;
        if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
        return launch(stride == 1 ? dw5_vec_kernel<1> : dw5_vec_kernel<2>, (unsigned)grid, kDwThreads, 0, st, x, nin,
                      w5, bias, y, stats_out, C, Lin, Lout, chunks);
    } else {
        const long long items = (long long)C * Lout;
        const int chunks = (int)((items + kDwThreads * 4 - 1) / (kDwThreads * 4));
        const long long grid = (long long)chunks * samples;
        if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
        return launch(dw5_scalar_kernel, (unsigned)grid, kDwThreads, 0, st, x, nin, w5, bias, y, stats_out, C, Lin,
                      Lout, stride, chunks);
    }
}

int launch_merge(const float* const* z, const NormIn* nins, int depth, float* m, double* stats_out,
                 int samples, int C, int L, cudaStream_t st) {
    if (depth < 1 || depth > kMaxDepth) return SDR_ERR_UNSUPPORTED;
    if (samples <= 0 || C <= 0 || L <= 0 || (L % (1 << (depth - 1))) != 0) return SDR_ERR_BAD_ARGUMENT;
    if ((long long)C * L > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;     // the kernels count a sample's items in int
    MergeArgs a;
    a.depth = depth;
    bool aligned = reinterpret_cast<uintptr_t>(m) % 16 == 0;
    for (int d = 0; d < kMaxDepth; ++d) {
        a.z[d] = d < depth ? z[d] : nullptr;
        a.n[d] = d < depth ? nins[d] : NormIn{nullptr, nullptr, nullptr, nullptr, 1.0};
        if (d < depth) aligned = aligned && reinterpret_cast<uintptr_t>(z[d]) % 16 == 0;
    }
    // vector path: rows of level 0 are float4-aligned, rows of level 1 float2-aligned
    const bool vec = aligned && (L % 4 == 0);
    if (vec && depth >= 4 && (L % 16 == 0)) {
        const long long items = (long long)C * (L / 16);
        const int per_cta = kMg16Threads * kMg16Items;
        const int chunks = (int)((items + per_cta - 1) / per_cta);
        const long long grid = (long long)chunks * samples;
        if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
        return launch(merge_wide_kernel, (unsigned)grid, kMg16Threads, 0, st, a, m, stats_out, C, L, chunks);
    } else if (vec) {
        const long long items = (long long)C * (L / 4);
        const int chunks = (int)((items + kMgThreads * kMgItems - 1) / (kMgThreads * kMgItems));
        const long long grid = (long long)chunks * samples;
        if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
        return launch(merge_vec_kernel, (unsigned)grid, kMgThreads, 0, st, a, m, stats_out, C, L, chunks);
    } else {
        const long long items = (long long)C * L;
        const int chunks = (int)((items + kMgThreads * 4 - 1) / (kMgThreads * 4));
        const long long grid = (long long)chunks * samples;
        if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
        return launch(merge_scalar_kernel, (unsigned)grid, kMgThreads, 0, st, a, m, stats_out, C, L, chunks);
    }
}

}  // namespace sdr
