// Stages that only the ORIGINAL SuDoRM-RF has (sudo_rm_rf/dnn/models/sudormrf.py, variant 3 of the C-ABI).
//
// Everything else of that model runs on the kernels of the improved model: GroupNorm(1, C, eps=1e-8)
// (sudormrf.py:32,56,70,117) is the arithmetic of GlobLN (statistics over (C, L) per sample, biased variance, eps
// inside the square root), so it is deferred the same way (producer: raw output + fp64 (sum, sumsq); consumer: applied
// on load); the per-channel PReLU (nn.PReLU(C), :33,71) rides on the same operand loads with one slope per channel
// (NormIn::prelu_pc).  What is new:
//   * the tail of a UBlock, :184-186:  out = PReLU_c(GN_ma(GN_e(conv_1x1_exp(..)) + x)).  Two normalisations in a row
//     need two sets of statistics, so one element-wise pass forms u = GN_e(e) + x (x itself read through the previous
//     block's deferred module_act) and accumulates the statistics of u; module_act is then applied by u's consumers.
//   * the masks, :239-242,284-289: an (N+1) x 1 Conv2d over the basis axis is a dense [S*N, N] Toeplitz matrix per
//     source, i.e. one more 1x1-conv GEMM on the tensor-core kernel (the matrix is expanded once at pack time);
//     softmax over the sources (sigmoid for one source) times the encoder output is one element-wise pass.
//   * the grouped ConvTranspose1d decoder, :245-252: block-diagonal weights for the same frames GEMM + overlap-add.
#include "common.cuh"
#include "launchers.cuh"

namespace sdr {

// ---------------------------------------------------------------------------
// x <- GN_e(e) + f(x)  (+ statistics of the new x), in place
// ---------------------------------------------------------------------------
constexpr int kRnThreads = 256;
constexpr int kRnItems = 4;            // float4 quads (or scalars) per thread

template <bool VEC>
__global__ void __launch_bounds__(kRnThreads)
residual_norm_kernel(const float* __restrict__ e, NormIn fe, float* x, NormIn fx, double* __restrict__ stats_out,
                     int C, int L, int chunks_per_sample) {
    __shared__ SampleNorm s_n[2];
    __shared__ double s_red[64];
    const int sample = blockIdx.x / chunks_per_sample;
    const int chunk = blockIdx.x - sample * chunks_per_sample;
    if (threadIdx.x == 0) { s_n[0] = sample_norm(fe, sample); s_n[1] = sample_norm(fx, sample); }
    __syncthreads();
    const SampleNorm ne = s_n[0], nx = s_n[1];
    const size_t base = (size_t)sample * C * L;
    const int items = VEC ? (C * L) >> 2 : C * L;
    StatAcc acc;
#pragma unroll
    for (int it = 0; it < kRnItems; ++it) {
        const int item = (chunk * kRnItems + it) * kRnThreads + threadIdx.x;
        if (item < items) {
            if (VEC) {                                     // L % 4 == 0: a quad lies inside one channel row
                const int idx = item << 2;
                const int c = idx / L;
                const ChanNorm ce = chan_norm(fe, ne, c), cx = chan_norm(fx, nx, c);
                const float4 v = ldg4(e + base + idx);
                const float4 r = *reinterpret_cast<const float4*>(x + base + idx);
                float4 o;
                o.x = apply_norm(ce, v.x) + apply_norm(cx, r.x);
                o.y = apply_norm(ce, v.y) + apply_norm(cx, r.y);
                o.z = apply_norm(ce, v.z) + apply_norm(cx, r.z);
                o.w = apply_norm(ce, v.w) + apply_norm(cx, r.w);
                *reinterpret_cast<float4*>(x + base + idx) = o;
                acc.add_run((o.x + o.y) + (o.z + o.w), fmaf(o.x, o.x, fmaf(o.y, o.y, fmaf(o.z, o.z, o.w * o.w))));
            } else {
                const int c = item / L;
                const ChanNorm ce = chan_norm(fe, ne, c), cx = chan_norm(fx, nx, c);
                const float o = apply_norm(ce, __ldg(e + base + item)) + apply_norm(cx, x[base + item]);
                x[base + item] = o;
                acc.add(o);
            }
        }
    }
    block_stats_atomic(acc, stats_out, sample, s_red);
}

int launch_residual_norm(const float* e, const NormIn& fe, float* x, const NormIn& fx, double* stats_out,
                         int samples, int C, int L, cudaStream_t st) {
    if (!e || !x || !stats_out || samples <= 0 || C <= 0 || L <= 0) return SDR_ERR_BAD_ARGUMENT;
    if ((long long)C * L > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    const bool vec = (L % 4 == 0) && ((reinterpret_cast<uintptr_t>(e) | reinterpret_cast<uintptr_t>(x)) % 16 == 0);
    const long long items = vec ? ((long long)C * L) >> 2 : (long long)C * L;
    const int per_cta = kRnThreads * kRnItems;
    const long long chunks = (items + per_cta - 1) / per_cta;
    const long long grid = chunks * samples;
    if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    return launch(vec ? residual_norm_kernel<true> : residual_norm_kernel<false>, (unsigned)grid, kRnThreads, 0, st, e,
                  fe, x, fx, stats_out, C, L, (int)chunks);
}

// ---------------------------------------------------------------------------
// masks: out[b,s,n,l] = softmax_s(logits[b,s,n,l]) * enc[b,n,l]   (sigmoid when S == 1), sudormrf.py:285-289
// ---------------------------------------------------------------------------
constexpr int kSgMaxSrc = 16;

template <bool VEC>
__device__ __forceinline__ void sg_load(const float* p, float (&v)[4]) {
    if (VEC) { const float4 t = *reinterpret_cast<const float4*>(p); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
    else { v[0] = *p; v[1] = v[2] = v[3] = 0.f; }
}
template <bool VEC>
__device__ __forceinline__ void sg_store(float* p, const float (&v)[4]) {
    if (VEC) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    else *p = v[0];
}

// one thread: all S sources of 4 (VEC) or 1 positions; reads complete before the first write, so out may alias logits.
// SS: compile-time source count (2, 3, 4: the loops unroll to exactly S loads / exps / stores, ~40 registers); 0 = any S
// up to kSgMaxSrc (the first version, every S through 16 predicated copies: 92 registers, 557 instructions per warp,
// 433 us for the 1.05 GB of the default model's masks, profiles/r02b_kernels.md).
template <bool VEC, int SS>
__device__ __forceinline__ void softmax_gate_item(const float* logits, const float* __restrict__ enc, float* out,
                                                  int S_rt, long long NL, int b, long long i) {
    constexpr int W = VEC ? 4 : 1;
    constexpr int SMAX = SS ? SS : kSgMaxSrc;
    const int S = SS ? SS : S_rt;
    const float* lp = logits + (size_t)b * S * NL + i;
    float* op = out + (size_t)b * S * NL + i;
    float g[4];
    sg_load<VEC>(enc + (size_t)b * NL + i, g);
    if (S == 1) {                                           // torch.sigmoid (sudormrf.py:285-286)
        float v[4];
        sg_load<VEC>(lp, v);
#pragma unroll
        for (int u = 0; u < W; ++u) v[u] = g[u] / (1.f + expf(-v[u]));
        sg_store<VEC>(op, v);
        return;
    }
    float v[SMAX][4];
    float mx[4], sum[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) { mx[u] = -INFINITY; sum[u] = 0.f; }
#pragma unroll
    for (int s = 0; s < SMAX; ++s) {
        if (s < S) {
            sg_load<VEC>(lp + (size_t)s * NL, v[s]);
#pragma unroll
            for (int u = 0; u < W; ++u) mx[u] = fmaxf(mx[u], v[s][u]);
        }
    }
#pragma unroll
    for (int s = 0; s < SMAX; ++s) {
        if (s < S) {
#pragma unroll
            for (int u = 0; u < W; ++u) { v[s][u] = expf(v[s][u] - mx[u]); sum[u] += v[s][u]; }
        }
    }
#pragma unroll
    for (int u = 0; u < W; ++u) g[u] = g[u] / sum[u];
#pragma unroll
    for (int s = 0; s < SMAX; ++s) {
        if (s < S) {
#pragma unroll
            for (int u = 0; u < W; ++u) v[s][u] *= g[u];
            sg_store<VEC>(op + (size_t)s * NL, v[s]);
        }
    }
}

// grid.y is capped at 65535; each CTA row strides over the batch
template <bool VEC, int SS>
__global__ void __launch_bounds__(256)
softmax_gate_kernel(const float* logits, const float* __restrict__ enc, float* out, int B, int S_rt, long long NL) {
    const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * (VEC ? 4 : 1);
    if (i >= NL) return;
    for (long long b = blockIdx.y; b < B; b += gridDim.y)      // long long: b + gridDim.y may pass INT_MAX
        softmax_gate_item<VEC, SS>(logits, enc, out, S_rt, NL, (int)b, i);
}

template <bool VEC>
static auto softmax_gate_for(int S) {
    switch (S) {
        case 2: return softmax_gate_kernel<VEC, 2>;
        case 3: return softmax_gate_kernel<VEC, 3>;
        case 4: return softmax_gate_kernel<VEC, 4>;
        default: return softmax_gate_kernel<VEC, 0>;
    }
}

int launch_softmax_gate(const float* logits, const float* enc, float* out, int B, int S, int N, int L, cudaStream_t st) {
    if (!logits || !enc || !out || B <= 0 || S <= 0 || N <= 0 || L <= 0) return SDR_ERR_BAD_ARGUMENT;
    if (S > kSgMaxSrc) return SDR_ERR_UNSUPPORTED;
    const long long NL = (long long)N * L;
    const bool vec = (NL % 4 == 0) &&
                     ((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(enc) | reinterpret_cast<uintptr_t>(out)) % 16 == 0);
    const long long threads = vec ? NL / 4 : NL;
    const long long gx = (threads + 255) / 256;
    if (gx > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    dim3 grid((unsigned)gx, (unsigned)(B < 65535 ? B : 65535));
    return launch(vec ? softmax_gate_for<true>(S) : softmax_gate_for<false>(S), grid, 256, 0, st, logits, enc, out, B,
                  S, NL);
}

// ---------------------------------------------------------------------------
// pack-time expansions
// ---------------------------------------------------------------------------
// m = nn.Conv2d(1, S, (N + 1, 1), padding=(N - N / 2, 0)) on x[:, None] (sudormrf.py:239-242,284):
//   logits[s, n, l] = bias[s] + sum_j w[s, j] * xpad[n + j, l],  xpad[r] = x[r - pad],  pad = N - N / 2
//   = sum_c W[s*N + n, c] * x[c, l] + bias[s]   with   W[s*N + n, c] = w[s, c - n + pad]  (0 <= c - n + pad <= N)
__global__ void toeplitz_mask_kernel(const float* __restrict__ w, const float* __restrict__ bias,
                                     float* __restrict__ W, float* __restrict__ brow, int S, int N) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)S * N * N;
    if (i < (long long)S * N) brow[i] = __ldg(bias + i / N);
    if (i >= total) return;
    const int c = (int)(i % N);
    const int row = (int)(i / N);
    const int s = row / N, n = row - s * N;
    const int j = c - n + (N - N / 2);
    W[i] = (j >= 0 && j <= N) ? __ldg(w + (size_t)s * (N + 1) + j) : 0.f;
}

int launch_toeplitz_mask(const float* w, const float* bias, float* W, float* brow, int S, int N, cudaStream_t st) {
    if (!w || !bias || !W || !brow || S <= 0 || N <= 0) return SDR_ERR_BAD_ARGUMENT;
    const long long total = (long long)S * N * N;
    return launch(toeplitz_mask_kernel, (unsigned)((total + 255) / 256), 256, 0, st, w, bias, W, brow, S, N);
}

// decoder = nn.ConvTranspose1d(S*N, S, K, groups=S) (sudormrf.py:245-252): weight [S*N][1][K]; source s only sees its
// own N masked channels.  As the frames GEMM operand [S*K][S*N] (row s'*K + j, column s*N + n): block diagonal.
__global__ void grouped_decoder_kernel(const float* __restrict__ w, float* __restrict__ wt, int S, int N, int K) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long C = (long long)S * N;
    if (i >= C * S * K) return;
    const int col = (int)(i % C);
    const int row = (int)(i / C);
    const int sp = row / K, j = row - sp * K;
    const int s = col / N;
    wt[i] = (s == sp) ? __ldg(w + (size_t)col * K + j) : 0.f;
}

int launch_grouped_decoder(const float* w, float* wt, int S, int N, int K, cudaStream_t st) {
    if (!w || !wt || S <= 0 || N <= 0 || K <= 0) return SDR_ERR_BAD_ARGUMENT;
    const long long total = (long long)S * N * S * K;
    return launch(grouped_decoder_kernel, (unsigned)((total + 255) / 256), 256, 0, st, w, wt, S, N, K);
}

}  // namespace sdr
