// Front end (encoder) and back end (overlap-add of decoder frames, crop,
// mixture consistency).
//
// Reference semantics:
//   pad_to_appropriate_length   improved_sudormrf.py:303-314 (zeros to Tp; folded into the
//                               load predicate here: no padded copy is ever materialised)
//   encoder                     improved_sudormrf.py:247-251,286  Conv1d(A,N,K,stride=K/2,pad=K/2)
//                               (original model, sudormrf.py:212-218,269: the same Conv1d with a bias, then ReLU;
//                                its ConvTranspose1d decoder, :245-252, has one bias per source)
//   decoder                     improved_sudormrf.py:272-279,300  ConvTranspose1d(...,stride=K/2,
//                               padding=K/2, output_padding=K/2-1)  -> length hop*L
//   remove_trailing_zeros       improved_sudormrf.py:316-318      crop to T
//   mixture_consistency.apply   mixture_consistency.py:14-36
#include "common.cuh"
#include "launchers.cuh"

namespace sdr {

// ---------------------------------------------------------------------------
// encoder: enc[b,n,t] = sum_a sum_j w[n,a,j] * wav[b,a, hop*t + j - pad]
// CTA = 128 positions x kEncNB basis functions; the waveform chunk and the
// weight slab sit in shared memory; each thread owns one position and walks the
// basis functions four at a time (weights read as broadcast float4).
// ---------------------------------------------------------------------------
constexpr int kEncThreads = 128;
constexpr int kEncNB = 64;

__global__ void __launch_bounds__(kEncThreads)
encoder_kernel(const float* __restrict__ wav, const float* __restrict__ weight, const float* __restrict__ bias,
               float* __restrict__ enc, double* __restrict__ stats,
               int A, long long T, int N, int K, int L, int t_tiles, int pad, int relu_out) {
    extern __shared__ __align__(16) float smem[];
    __shared__ double s_red[64];
    const int hop = K / 2;
    const int span = hop * (kEncThreads - 1) + K;        // samples needed by 128 positions
    float* s_x = smem;                                     // [A][span]
    float* s_w = smem + ((A * span + 3) & ~3);             // [A*K][kEncNB]  (n fastest)

    const int b = blockIdx.x / t_tiles;
    const int t0 = (blockIdx.x - b * t_tiles) * kEncThreads;
    const int n0 = blockIdx.y * kEncNB;
    const int tid = threadIdx.x;

    const long long base = (long long)hop * t0 - pad;      // first sample index of the chunk (pad = hop; 2 * hop for the causal model)
    for (int i = tid; i < A * span; i += kEncThreads) {
        const int a = i / span, p = i - a * span;
        const long long g = base + p;
        s_x[i] = (g >= 0 && g < T) ? __ldg(wav + ((size_t)b * A + a) * T + g) : 0.f;
    }
    for (int i = tid; i < A * K * kEncNB; i += kEncThreads) {
        const int n = i % kEncNB, aj = i / kEncNB;         // aj = a*K + j
        s_w[i] = (n0 + n < N) ? __ldg(weight + (size_t)(n0 + n) * A * K + aj) : 0.f;
    }
    __syncthreads();

    const int t = t0 + tid;
    StatAcc acc;
    const int AK = A * K;
    for (int nn = 0; nn < kEncNB; nn += 4) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        for (int a = 0; a < A; ++a) {
            const float* xr = s_x + a * span + hop * tid;
            const float* wr = s_w + (size_t)a * K * kEncNB + nn;
            for (int j = 0; j < K; ++j) {
                const float xv = xr[j];
                const float4 w = *reinterpret_cast<const float4*>(wr + j * kEncNB);
                a0 = fmaf(w.x, xv, a0); a1 = fmaf(w.y, xv, a1);
                a2 = fmaf(w.z, xv, a2); a3 = fmaf(w.w, xv, a3);
            }
        }
        (void)AK;
        if (t < L) {
            float o[4] = {a0, a1, a2, a3};
            float rs = 0.f, rq = 0.f;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int n = n0 + nn + e;
                if (n < N) {
                    if (bias) o[e] += __ldg(bias + n);
                    if (relu_out) o[e] = relu(o[e]);
                    enc[((size_t)b * N + n) * L + t] = o[e];
                    rs += o[e]; rq = fmaf(o[e], o[e], rq);
                }
            }
            acc.add_run(rs, rq);
        }
    }
    if (stats) block_stats_atomic(acc, stats, b, s_red);
}

// Dynamic shared memory of one CTA: the waveform chunk of every audio channel and the [A*K][kEncNB] weight slab.
static size_t encoder_smem_bytes(int A, int K) {
    const int span = (K / 2) * (kEncThreads - 1) + K;
    return (size_t)(((A * span + 3) & ~3) + A * K * kEncNB) * sizeof(float);
}

// Whether the FFMA encoder can take A audio channels and K taps (its CTA would need more than 200 KB otherwise).
bool encoder_ffma_fits(int A, int K) { return encoder_smem_bytes(A, K) <= 200 * 1024; }

int launch_encoder(const float* wav, const float* weight, const float* bias, int relu, float* enc, double* stats,
                   int B, int A, long long T, int N, int K, int L, int pad, cudaStream_t st) {
    if (B <= 0 || A <= 0 || T <= 0 || N <= 0 || K < 3 || L <= 0) return SDR_ERR_BAD_ARGUMENT;
    if (!encoder_ffma_fits(A, K)) return SDR_ERR_UNSUPPORTED;
    const size_t smem = encoder_smem_bytes(A, K);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(encoder_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return SDR_ERR_CUDA;
    }
    const int t_tiles = (L + kEncThreads - 1) / kEncThreads;
    const long long gx = (long long)t_tiles * B;
    if (gx > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    dim3 grid((unsigned)gx, (unsigned)((N + kEncNB - 1) / kEncNB));
    encoder_kernel<<<grid, kEncThreads, smem, st>>>(wav, weight, bias, enc, stats, A, T, N, K, L, t_tiles, pad, relu);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

// ---------------------------------------------------------------------------
// overlap-add: frames[b, sa*K + j, t] (= sum_c Wd[c,sa,j] masked[b,c,t]) ->
// out[b, sa, tau] = sum over (t, j) with hop*t + j - hop == tau, tau < T;
// optional uniform mixture consistency (needs all sources of a tau in one thread).
// ---------------------------------------------------------------------------
constexpr int kMaxSrc = 16;

__global__ void __launch_bounds__(256)
overlap_add_kernel(const float* __restrict__ frames, const float* __restrict__ mix, const float* __restrict__ bias,
                   const float2* __restrict__ rescale, float* __restrict__ out, int B, int SA, int K, int L, long long T) {
    const int hop = K / 2;
    const long long tau = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (tau >= T) return;
    // j = tau + hop - hop*t in [0, K)  ->  t in [ceil((tau+hop-K+1)/hop), floor((tau+hop)/hop)]
    const long long thi = (tau + hop) / hop;
    long long tlo = tau + hop - (K - 1);
    tlo = tlo <= 0 ? 0 : (tlo + hop - 1) / hop;
    // grid.y is capped at 65535; each CTA row strides over the batch
    for (long long b = blockIdx.y; b < B; b += gridDim.y) {   // long long: b + gridDim.y may pass INT_MAX
        float est[kMaxSrc];
        float sum = 0.f;
        // separate(): undo the per-utterance input normalisation, est * std + mean (README.md:109), before the
        // mixture-consistency projection, which the README applies to the rescaled estimates (README.md:113-114)
        const float2 rs = rescale ? rescale[b] : make_float2(0.f, 1.f);
        for (int s = 0; s < SA; ++s) {
            float acc = 0.f;
            for (long long t = tlo; t <= thi && t < L; ++t) {
                const int j = (int)(tau + hop - hop * t);
                acc += __ldg(frames + ((size_t)b * SA * K + (size_t)s * K + j) * L + t);
            }
            if (bias) acc += __ldg(bias + s);            // decoder bias of the original model (one per source)
            if (rescale) acc = __fadd_rn(__fmul_rn(acc, rs.y), rs.x);
            est[s] = acc;
            sum += acc;
        }
        float corr = 0.f;
        if (mix) corr = (__ldg(mix + (size_t)b * T + tau) - sum) * (1.0f / SA);   // mixture_consistency.py:29-35
        for (int s = 0; s < SA; ++s) out[((size_t)b * SA + s) * T + tau] = est[s] + corr;
    }
}

int launch_overlap_add(const float* frames, const float* mix, const float* bias, const float2* rescale, float* out,
                       int B, int SA, int K, int L, long long T, cudaStream_t st) {
    if (B <= 0 || SA <= 0 || K < 3 || L <= 0 || T <= 0) return SDR_ERR_BAD_ARGUMENT;
    if (SA > kMaxSrc) return SDR_ERR_UNSUPPORTED;
    dim3 grid((unsigned)((T + 255) / 256), (unsigned)(B < 65535 ? B : 65535));
    overlap_add_kernel<<<grid, 256, 0, st>>>(frames, mix, bias, rescale, out, B, SA, K, L, T);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

// ---------------------------------------------------------------------------
// standalone mixture consistency (mixture_consistency.py:14-36)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
mc_power_kernel(const float* __restrict__ est, double* __restrict__ power, int rows, long long T) {
    // power[b*S+s] += sum_t est^2   (grid.y = min(B*S, 65535), striding over the rows)
    __shared__ float red[32];
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {    // long long: r + gridDim.y may pass INT_MAX
        const size_t row = r;
        float q = 0.f;
        for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < T;
             t += (long long)gridDim.x * blockDim.x) {
            const float v = __ldg(est + row * T + t);
            q = fmaf(v, v, q);
        }
        q = warp_sum(q);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = q;
        __syncthreads();
        if (threadIdx.x < 32) {
            double d = threadIdx.x < (blockDim.x >> 5) ? (double)red[threadIdx.x] : 0.0;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
            if (threadIdx.x == 0) atomicAdd(power + row, d);
        }
        __syncthreads();                                   // red is reused by the next row
    }
}

__global__ void __launch_bounds__(256)
mc_apply_kernel(const float* __restrict__ est, const float* __restrict__ mix,
                const double* __restrict__ power, float* __restrict__ out, int B, int S, long long T) {
    const long long tau = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (tau >= T) return;
    for (long long b = blockIdx.y; b < B; b += gridDim.y) {   // long long: b + gridDim.y may pass INT_MAX
        float sum = 0.f;
        for (int s = 0; s < S; ++s) sum += __ldg(est + ((size_t)b * S + s) * T + tau);
        const float resid = __ldg(mix + (size_t)b * T + tau) - sum;
        float wsum = 0.f;
        if (power) {
            for (int s = 0; s < S; ++s) wsum += (float)(power[(size_t)b * S + s] / (double)T);
        }
        for (int s = 0; s < S; ++s) {
            float w;
            if (power) {
                const float mw = (float)(power[(size_t)b * S + s] / (double)T);  // mean(est^2, -1)
                w = mw / (wsum + 1e-9f);                                          // mixture_consistency.py:27-28
            } else {
                w = 1.0f / S;
            }
            const size_t i = ((size_t)b * S + s) * T + tau;
            out[i] = __ldg(est + i) + w * resid;
        }
    }
}

int launch_mixture_consistency(const float* est, const float* mix, float* out, int B, int S,
                               long long T, int weights_type, void* scratch, cudaStream_t st) {
    if (B <= 0 || S <= 0 || T <= 0 || !est || !mix || !out) return SDR_ERR_BAD_ARGUMENT;
    if ((long long)B * S > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;   // rows are indexed in int
    double* power = nullptr;
    if (weights_type == 1) {
        if (!scratch) return SDR_ERR_BAD_ARGUMENT;
        power = static_cast<double*>(scratch);
        const int rows = B * S;
        if (cudaMemsetAsync(power, 0, sizeof(double) * rows, st) != cudaSuccess) return SDR_ERR_CUDA;
        int gx = (int)((T + 256 * 8 - 1) / (256 * 8));
        if (gx < 1) gx = 1;
        mc_power_kernel<<<dim3((unsigned)gx, (unsigned)(rows < 65535 ? rows : 65535)), 256, 0, st>>>(est, power, rows, T);
    } else if (weights_type != 0) {
        return SDR_ERR_BAD_ARGUMENT;
    }
    dim3 grid((unsigned)((T + 255) / 256), (unsigned)(B < 65535 ? B : 65535));
    mc_apply_kernel<<<grid, 256, 0, st>>>(est, mix, power, out, B, S, T);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

// ---------------------------------------------------------------------------
// backward of the projection.  With r = mix - sum_s est_s and g = dL/dout:
//   uniform: d est_k = g_k - (1/S) sum_s g_s,                  d mix = (1/S) sum_s g_s
//   magsq:   P_s = mean_t est_s^2, Q = sum_s P_s + 1e-9, w_s = P_s / Q, c_s = <g_s, r>,
//            d est_k = g_k - sum_s w_s g_s + alpha_k est_k,    d mix = sum_s w_s g_s,
//            alpha_k = (2 / T) (c_k / Q - sum_s c_s P_s / Q^2)
// magsq: mc_bwd_partials_kernel writes (sum est_s^2, c_s) per (row, chunk) in fp64, mc_bwd_coef_kernel adds the
// chunks in index order and forms (w_s, alpha_s).  No atomics, so a backward is bitwise reproducible.
// ---------------------------------------------------------------------------
static int mc_bwd_chunks(long long T) {
    long long c = (T + 4095) / 4096;
    return (int)(c < 1 ? 1 : (c > 64 ? 64 : c));
}

size_t mc_backward_scratch_bytes(int B, int S, long long T, int weights_type) {
    if (B <= 0 || S <= 0 || T <= 0 || weights_type != 1) return 0;
    return sizeof(double) * 2 * (size_t)B * S * (mc_bwd_chunks(T) + 1);
}

// grid = rows * chunks (rows = B * S); part[row][chunk] = (sum est^2, <g, r>) over the chunk
__global__ void __launch_bounds__(256)
mc_bwd_partials_kernel(const float* __restrict__ est, const float* __restrict__ mix, const float* __restrict__ g,
                       double2* __restrict__ part, int S, long long T, int chunks) {
    __shared__ double red[2][8];
    const long long row = blockIdx.x / chunks;
    const int chunk = (int)(blockIdx.x - row * chunks);
    const long long b = row / S;
    const long long per = (T + chunks - 1) / chunks;
    const long long t0 = (long long)chunk * per;
    const long long t1 = t0 + per < T ? t0 + per : T;
    const float* eb = est + (size_t)b * S * T;
    const float* er = est + (size_t)row * T;
    const float* gr = g + (size_t)row * T;
    double p = 0.0, c = 0.0;
    for (long long t = t0 + threadIdx.x; t < t1; t += 256) {
        float sum = 0.f;
        for (int s = 0; s < S; ++s) sum += __ldg(eb + (size_t)s * T + t);
        const double r = (double)(__ldg(mix + (size_t)b * T + t) - sum);      // the residual as the forward forms it
        const double e = (double)__ldg(er + t);
        p = fma(e, e, p);
        c = fma((double)__ldg(gr + t), r, c);
    }
    p = warp_sum_f64(p);
    c = warp_sum_f64(c);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { red[0][warp] = p; red[1][warp] = c; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double tp = 0.0, tc = 0.0;
        for (int w = 0; w < 8; ++w) { tp += red[0][w]; tc += red[1][w]; }
        part[blockIdx.x] = make_double2(tp, tc);
    }
}

// one thread per item: coef[b * S + s] = (w_s, alpha_s)
__global__ void __launch_bounds__(256)
mc_bwd_coef_kernel(const double2* __restrict__ part, double2* __restrict__ coef, int B, int S, long long T, int chunks) {
    for (long long b = blockIdx.x * 256LL + threadIdx.x; b < B; b += (long long)gridDim.x * 256) {
        double q = 0.0, cp = 0.0;
        for (int s = 0; s < S; ++s) {
            double ps = 0.0, cs = 0.0;
            const double2* pr = part + ((size_t)b * S + s) * chunks;
            for (int k = 0; k < chunks; ++k) { ps += pr[k].x; cs += pr[k].y; }
            ps /= (double)T;                                      // P_s = mean_t est_s^2
            coef[(size_t)b * S + s] = make_double2(ps, cs);
            q += ps;
            cp += cs * ps;
        }
        q += 1e-9;
        for (int s = 0; s < S; ++s) {
            const double2 v = coef[(size_t)b * S + s];
            coef[(size_t)b * S + s] = make_double2(v.x / q, 2.0 / (double)T * (v.y / q - cp / (q * q)));
        }
    }
}

// grid (T tiles, min(B, 65535)): gsum = sum_s w_s g_s; d est_k = g_k - gsum + alpha_k est_k; d mix = gsum.
// magsq runs in fp64: a dominant source has w close to 1, and g_k - w_k g_k would cancel in fp32.
__global__ void __launch_bounds__(256)
mc_bwd_apply_kernel(const float* __restrict__ est, const float* __restrict__ g, const double2* __restrict__ coef,
                    float* __restrict__ grad_est, float* __restrict__ grad_mix, int B, int S, long long T) {
    const long long tau = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (tau >= T) return;
    for (long long b = blockIdx.y; b < B; b += gridDim.y) {
        const float* gb = g + (size_t)b * S * T + tau;
        if (coef) {
            const double2* cb = coef + (size_t)b * S;
            double gsum = 0.0;
            for (int s = 0; s < S; ++s) gsum = fma(cb[s].x, (double)__ldg(gb + (size_t)s * T), gsum);
            for (int s = 0; s < S; ++s) {
                const size_t i = ((size_t)b * S + s) * T + tau;
                grad_est[i] = (float)(fma(cb[s].y, (double)__ldg(est + i), (double)__ldg(g + i) - gsum));
            }
            if (grad_mix) grad_mix[(size_t)b * T + tau] = (float)gsum;
        } else {
            float gsum = 0.f;
            for (int s = 0; s < S; ++s) gsum += __ldg(gb + (size_t)s * T);
            gsum *= 1.0f / S;
            for (int s = 0; s < S; ++s) {
                const size_t i = ((size_t)b * S + s) * T + tau;
                grad_est[i] = __ldg(g + i) - gsum;
            }
            if (grad_mix) grad_mix[(size_t)b * T + tau] = gsum;
        }
    }
}

int launch_mixture_consistency_backward(const float* est, const float* mix, const float* grad_out, float* grad_est,
                                        float* grad_mix, int B, int S, long long T, int weights_type, void* scratch,
                                        cudaStream_t st) {
    if (B <= 0 || S <= 0 || T <= 0 || !est || !grad_out || !grad_est) return SDR_ERR_BAD_ARGUMENT;
    if (weights_type != 0 && weights_type != 1) return SDR_ERR_BAD_ARGUMENT;
    if ((long long)B * S > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    double2* coef = nullptr;
    if (weights_type == 1) {
        if (!mix || !scratch) return SDR_ERR_BAD_ARGUMENT;
        const int chunks = mc_bwd_chunks(T);
        const long long rows = (long long)B * S, grid = rows * chunks;
        if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
        double2* part = static_cast<double2*>(scratch);
        coef = part + (size_t)grid;
        mc_bwd_partials_kernel<<<(unsigned)grid, 256, 0, st>>>(est, mix, grad_out, part, S, T, chunks);
        const long long cb = (B + 255) / 256;
        mc_bwd_coef_kernel<<<(unsigned)(cb < 4096 ? cb : 4096), 256, 0, st>>>(part, coef, B, S, T, chunks);
    }
    dim3 grid((unsigned)((T + 255) / 256), (unsigned)(B < 65535 ? B : 65535));
    mc_bwd_apply_kernel<<<grid, 256, 0, st>>>(est, grad_out, coef, grad_est, grad_mix, B, S, T);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

}  // namespace sdr
