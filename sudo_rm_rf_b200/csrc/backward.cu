// Backward kernels of the improved SuDoRM-RF (variant 0): weight-gradient GEMM, GlobLN / PReLU backward (reduce +
// apply), depthwise backward, mask backward, frame gather and weight transposes.  api.cu orders them.
//
// Every gradient that is a reduction over (sample, position) is summed in a fixed order: per-CTA partials (fp32 over
// at most kWgChunk positions, or fp64 block sums) go to the workspace and a second pass adds them up in fp64, one
// output per thread, in index order.  No atomics touch a gradient, so a backward is bitwise reproducible.
#include "common.cuh"
#include "launchers.cuh"

namespace sdr {

constexpr int kBwThreads = 256;
constexpr int kWgTile = 64;       // wgrad CTA tile: 64 output rows x 64 output columns
constexpr int kWgStep = 16;       // positions per shared-memory stage
constexpr int kWgChunk = 512;     // positions one CTA reduces before its partial goes to the workspace

// Block-wide fp64 sums of NV per-thread values, returned in every thread.  All threads of the block must call it.
template <int NV>
__device__ __forceinline__ void block_sum_f64(double (&v)[NV], double* red /* >= 32 * NV */) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const double s = warp_sum_f64(v[i]);
        if (lane == 0) red[i * 32 + warp] = s;
    }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const double s = warp_sum_f64(lane < nwarps ? red[i * 32 + lane] : 0.0);
            if (lane == 0) red[i * 32] = s;
        }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = red[i * 32];
    __syncthreads();
}

// ---------------------------------------------------------------------------
// weight gradient of a 1x1 convolution: dW[m][k] = sum_{b,t} dY[b][m][t] * f(X[b][k][t]), db[m] = sum dY
// ---------------------------------------------------------------------------
// One CTA per (64 x 64 output tile, sample, chunk of kWgChunk positions); its fp32 tile goes to part[p] with
// p = sample * nchunk + chunk, laid out [M*K] followed by the bias partial [M] (written by the column-0 CTAs).
// The grid is one-dimensional, column tile fastest, then row tile, then p, so that samples * nchunk may exceed the
// 65535 a grid's y and z dimensions allow.
__global__ void __launch_bounds__(kBwThreads)
wgrad_partial_kernel(const float* __restrict__ dY, const float* __restrict__ X, NormIn nin, float* __restrict__ part,
                     int M, int K, int L, int nchunk, int ktiles, int mtiles, int with_bias) {
    __shared__ float As[kWgStep][kWgTile + 4];
    __shared__ float Bs[kWgStep][kWgTile + 4];
    __shared__ ChanNorm cns[kWgTile];
    const int kti = blockIdx.x % ktiles, mti = (blockIdx.x / ktiles) % mtiles;
    const int kt = kti * kWgTile, mt = mti * kWgTile;
    const int p = blockIdx.x / (ktiles * mtiles), b = p / nchunk, chunk = p % nchunk;
    const int t0 = chunk * kWgChunk, t1 = min(L, t0 + kWgChunk);
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    if (tid < kWgTile) {
        const SampleNorm sn = sample_norm(nin, b);
        cns[tid] = chan_norm(nin, sn, kt + tid < K ? kt + tid : 0);
    }
    __syncthreads();
    const bool bias_cta = with_bias && kti == 0;
    float acc[4][4] = {};
    float bacc = 0.f;
    for (int t = t0; t < t1; t += kWgStep) {
        for (int e = tid; e < kWgTile * kWgStep; e += kBwThreads) {
            const int r = e / kWgStep, tt = e % kWgStep;
            const bool in = t + tt < t1;
            const int m = mt + r, k = kt + r;
            As[tt][r] = (in && m < M) ? __ldg(dY + ((size_t)b * M + m) * L + t + tt) : 0.f;
            Bs[tt][r] = (in && k < K) ? apply_norm(cns[r], __ldg(X + ((size_t)b * K + k) * L + t + tt)) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int tt = 0; tt < kWgStep; ++tt) {
            float a[4], x[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { a[i] = As[tt][ty * 4 + i]; x[i] = Bs[tt][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], x[j], acc[i][j]);
        }
        if (bias_cta && tid < kWgTile)
#pragma unroll
            for (int tt = 0; tt < kWgStep; ++tt) bacc += As[tt][tid];
        __syncthreads();
    }
    float* o = part + (size_t)p * ((size_t)M * K + M);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = mt + ty * 4 + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = kt + tx * 4 + j;
            if (k < K) o[(size_t)m * K + k] = acc[i][j];
        }
    }
    if (bias_cta && tid < kWgTile && mt + tid < M) o[(size_t)M * K + mt + tid] = bacc;
}

// dW (and db) = the partials summed over p in fp64, in order.
__global__ void __launch_bounds__(kBwThreads)
wgrad_reduce_kernel(const float* __restrict__ part, int P, long long MK, long long stride, long long n,
                    float* __restrict__ dW, float* __restrict__ db) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    for (int q = 0; q < P; ++q) s += (double)part[(size_t)q * stride + i];
    if (i < MK) dW[i] = (float)s;
    else db[i - MK] = (float)s;
}

static int wgrad_chunks(int L) { return (L + kWgChunk - 1) / kWgChunk; }

size_t wgrad_scratch_bytes(int samples, int M, int K, int L) {
    return (size_t)samples * wgrad_chunks(L) * ((size_t)M * K + M) * sizeof(float);
}

int launch_wgrad(const float* dY, const float* X, const NormIn& nin, float* dW, float* db, float* scratch,
                 int samples, int M, int K, int L, cudaStream_t st) {
    if (!dY || !X || !dW || !scratch || samples <= 0 || M <= 0 || K <= 0 || L <= 0) return SDR_ERR_BAD_ARGUMENT;
    const int nchunk = wgrad_chunks(L);
    const long long P = (long long)samples * nchunk;
    const int ktiles = (K + kWgTile - 1) / kWgTile, mtiles = (M + kWgTile - 1) / kWgTile;
    const long long ctas = P * ktiles * mtiles;
    if (ctas > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    if (const int rc = launch(wgrad_partial_kernel, (unsigned)ctas, kBwThreads, 0, st, dY, X, nin, scratch, M, K, L,
                              nchunk, ktiles, mtiles, db ? 1 : 0))
        return rc;
    const long long MK = (long long)M * K, n = MK + (db ? M : 0);
    // the partial stride is M*K + M whether or not the bias is reduced
    return launch(wgrad_reduce_kernel, (unsigned)((n + kBwThreads - 1) / kBwThreads), kBwThreads, 0, st, scratch,
                  (int)P, MK, MK + M, n, dW, db);
}

// ---------------------------------------------------------------------------
// GlobLN (+ shared-slope PReLU) backward, or the PReLU alone when nin.stats is null
// ---------------------------------------------------------------------------
// v = gamma * xhat + beta (v = x without statistics), p = PReLU(v); given dp:
//   dv = dp * (v > 0 ? 1 : a),  da = sum dp * (v > 0 ? 0 : v),  dgamma_c = sum dv * xhat,  dbeta_c = sum dv,
//   dx = rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = gamma * dv, means over the sample's (C, L).
// Reduce: one CTA per (sample, channel) row writes the row's (sum dv, sum dv * xhat, sum da) in fp64.
struct NormBwdTerms { float dv, pre; bool neg; };

__device__ __forceinline__ NormBwdTerms norm_bwd_terms(const ChanNorm& cn, float x, float dp) {
    NormBwdTerms r;
    r.pre = fmaf(x - cn.mean, cn.a, cn.b);
    r.neg = cn.act && !(r.pre > 0.f);          // nn.PReLU: the slope applies at 0 as well
    r.dv = r.neg ? dp * cn.slope : dp;
    return r;
}

__global__ void __launch_bounds__(kBwThreads)
norm_bwd_reduce_kernel(const float* __restrict__ x, NormIn nin, const float* dp, double* __restrict__ part, int C,
                       int L) {
    __shared__ double red[32 * 3];
    const int row = blockIdx.x, b = row / C, c = row % C;
    const SampleNorm sn = sample_norm(nin, b);
    const ChanNorm cn = chan_norm(nin, sn, c);
    const float* xr = x + (size_t)row * L;
    const float* gr = dp + (size_t)row * L;
    double v[3] = {0.0, 0.0, 0.0};
    for (int t = threadIdx.x; t < L; t += blockDim.x) {
        const float xv = __ldg(xr + t), g = gr[t];
        const NormBwdTerms q = norm_bwd_terms(cn, xv, g);
        if (q.neg) v[2] += (double)g * (double)q.pre;
        v[0] += (double)q.dv;
        v[1] += (double)q.dv * (double)((xv - sn.mean) * sn.rstd);
    }
    block_sum_f64(v, red);
    if (threadIdx.x == 0) {
        part[(size_t)row * 3 + 0] = v[0];
        part[(size_t)row * 3 + 1] = v[1];
        part[(size_t)row * 3 + 2] = v[2];
    }
}

// Apply: out = dx (or out += dx).  Every CTA sums its sample's row terms itself (fixed order); the sample-0 CTAs also
// write dgamma / dbeta of their channel, and the (0, 0) CTA the PReLU slope gradient.  out may alias dp.
__global__ void __launch_bounds__(kBwThreads)
norm_bwd_apply_kernel(const float* __restrict__ x, NormIn nin, const float* dp, const double* __restrict__ part,
                      float* out, int accumulate, float* __restrict__ g_gamma, float* __restrict__ g_beta,
                      float* __restrict__ g_slope, int B, int C, int L) {
    __shared__ double red[32 * 2];
    const int row = blockIdx.x, b = row / C, c = row % C;
    const bool norm = nin.stats != nullptr;
    const SampleNorm sn = sample_norm(nin, b);
    const ChanNorm cn = chan_norm(nin, sn, c);
    double sg = 0.0, sgx = 0.0;
    if (norm) {
        double v[2] = {0.0, 0.0};
        for (int k = threadIdx.x; k < C; k += blockDim.x) {
            const double gm = (double)__ldg(nin.gamma + k);
            v[0] += gm * part[((size_t)b * C + k) * 3 + 0];
            v[1] += gm * part[((size_t)b * C + k) * 3 + 1];
        }
        block_sum_f64(v, red);
        sg = v[0]; sgx = v[1];
    }
    if (b == 0) {
        if (norm && (g_gamma || g_beta)) {
            double v[2] = {0.0, 0.0};
            for (int s = threadIdx.x; s < B; s += blockDim.x) {
                v[0] += part[((size_t)s * C + c) * 3 + 1];
                v[1] += part[((size_t)s * C + c) * 3 + 0];
            }
            block_sum_f64(v, red);
            if (threadIdx.x == 0) {
                if (g_gamma) g_gamma[c] = (float)v[0];
                if (g_beta) g_beta[c] = (float)v[1];
            }
        }
        if (c == 0 && cn.act && g_slope) {
            double v[1] = {0.0};
            for (long long r = threadIdx.x; r < (long long)B * C; r += blockDim.x) v[0] += part[(size_t)r * 3 + 2];
            block_sum_f64(v, red);
            if (threadIdx.x == 0) g_slope[0] = (float)v[0];
        }
    }
    const float mg = (float)(sg / nin.count), mgx = (float)(sgx / nin.count);
    const float gamma = norm ? __ldg(nin.gamma + c) : 1.f;
    const float* xr = x + (size_t)row * L;
    const float* gr = dp + (size_t)row * L;
    float* orow = out + (size_t)row * L;
    for (int t = threadIdx.x; t < L; t += blockDim.x) {
        const float xv = __ldg(xr + t);
        const NormBwdTerms q = norm_bwd_terms(cn, xv, gr[t]);
        float r = q.dv;
        if (norm) {
            const float xh = (xv - sn.mean) * sn.rstd;
            r = sn.rstd * (gamma * q.dv - mg - xh * mgx);
        }
        orow[t] = accumulate ? orow[t] + r : r;
    }
}

size_t norm_bwd_scratch_bytes(int samples, int C) { return (size_t)samples * C * 3 * sizeof(double); }

int launch_norm_bwd(const float* x, const NormIn& nin, const float* dp, float* out, int accumulate, float* g_gamma,
                    float* g_beta, float* g_slope, double* scratch, int samples, int C, int L, cudaStream_t st) {
    if (!x || !dp || !out || !scratch || samples <= 0 || C <= 0 || L <= 0) return SDR_ERR_BAD_ARGUMENT;
    if (nin.prelu_pc) return SDR_ERR_UNSUPPORTED;            // the improved model's PReLUs share one slope
    if (nin.stats && (!nin.gamma || !nin.beta)) return SDR_ERR_BAD_ARGUMENT;
    const long long rows = (long long)samples * C;
    if (rows > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    if (const int rc = launch(norm_bwd_reduce_kernel, (unsigned)rows, kBwThreads, 0, st, x, nin, dp, scratch, C, L))
        return rc;
    return launch(norm_bwd_apply_kernel, (unsigned)rows, kBwThreads, 0, st, x, nin, dp, scratch, out, accumulate,
                  g_gamma, g_beta, g_slope, samples, C, L);
}

// ---------------------------------------------------------------------------
// depthwise 5-tap convolution backward (padding 2, stride 1 or 2), with the merge's pooling folded in
// ---------------------------------------------------------------------------
// z[t'] = bias + sum_j w[j] * f(x[s t' + j - 2]) (zero outside [0, Lin)).  One CTA per (sample, channel) row:
//   din[tau] = sum_j w[j] dz[(tau + 2 - j) / s]  +  sum_{i < P} pool[P tau + i]          (dz and pool optional)
//   row partials of dw[j] = sum dz[t'] f(x[s t' + j - 2]) and db = sum dz                  (when part is given)
__global__ void __launch_bounds__(kBwThreads)
dw_bwd_kernel(const float* __restrict__ dz, const float* __restrict__ x, NormIn nin, const float* __restrict__ w5,
              const float* __restrict__ pool, int P, float* __restrict__ din, double* __restrict__ part, int C, int Lin,
              int stride) {
    __shared__ double red[32 * 6];
    const int row = blockIdx.x, b = row / C, c = row % C;
    const int Lout = stride == 1 ? Lin : Lin / 2;
    const float* dzr = dz ? dz + (size_t)row * Lout : nullptr;
    float w[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    if (dzr)
#pragma unroll
        for (int j = 0; j < 5; ++j) w[j] = __ldg(w5 + (size_t)c * 5 + j);
    const float* pr = pool ? pool + (size_t)row * Lin * P : nullptr;
    for (int tau = threadIdx.x; tau < Lin; tau += blockDim.x) {
        float acc = 0.f;
        if (dzr) {
#pragma unroll
            for (int j = 0; j < 5; ++j) {
                const int q = tau + 2 - j;
                if (q < 0 || (stride == 2 && (q & 1))) continue;
                const int tp = q / stride;
                if (tp < Lout) acc = fmaf(w[j], dzr[tp], acc);
            }
        }
        if (pr)
            for (int i = 0; i < P; ++i) acc += pr[(size_t)tau * P + i];
        din[(size_t)row * Lin + tau] = acc;
    }
    if (!dzr || !part) return;
    const ChanNorm cn = chan_norm(nin, sample_norm(nin, b), c);
    const float* xr = x + (size_t)row * Lin;
    double v[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int tp = threadIdx.x; tp < Lout; tp += blockDim.x) {
        const float g = dzr[tp];
        v[5] += (double)g;
#pragma unroll
        for (int j = 0; j < 5; ++j) {
            const int q = stride * tp + j - 2;
            if (q >= 0 && q < Lin) v[j] += (double)g * (double)apply_norm(cn, __ldg(xr + q));
        }
    }
    block_sum_f64(v, red);
    if (threadIdx.x < 6) part[(size_t)row * 6 + threadIdx.x] = v[threadIdx.x];
}

// dw[c][j] = sum_b part[b][c][j], db[c] = sum_b part[b][c][5], in sample order.
__global__ void __launch_bounds__(kBwThreads)
dw_finish_kernel(const double* __restrict__ part, float* __restrict__ gw, float* __restrict__ gb, int B, int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C * 6) return;
    const int c = i / 6, k = i % 6;
    double s = 0.0;
    for (int b = 0; b < B; ++b) s += part[((size_t)b * C + c) * 6 + k];
    if (k < 5) gw[(size_t)c * 5 + k] = (float)s;
    else gb[c] = (float)s;
}

size_t dw_bwd_scratch_bytes(int samples, int C) { return (size_t)samples * C * 6 * sizeof(double); }

// Pooling alone (dz null): din[tau] = sum_{i < P} pool[P tau + i].
int launch_dw_bwd(const float* dz, const float* x, const NormIn& nin, const float* w5, const float* pool, int P,
                  float* din, float* gw, float* gb, double* scratch, int samples, int C, int Lin, int stride,
                  cudaStream_t st) {
    if (!din || samples <= 0 || C <= 0 || Lin <= 0 || (stride != 1 && stride != 2)) return SDR_ERR_BAD_ARGUMENT;
    if (stride == 2 && (Lin % 2)) return SDR_ERR_BAD_ARGUMENT;
    if (!dz && !pool) return SDR_ERR_BAD_ARGUMENT;
    if (dz && (!x || !w5 || !gw || !gb || !scratch)) return SDR_ERR_BAD_ARGUMENT;
    if (pool && P < 1) return SDR_ERR_BAD_ARGUMENT;
    if (nin.prelu_pc) return SDR_ERR_UNSUPPORTED;
    const long long rows = (long long)samples * C;
    if (rows > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    const int rc = launch(dw_bwd_kernel, (unsigned)rows, kBwThreads, 0, st, dz, x, nin, w5, pool, pool ? P : 0, din,
                          dz ? scratch : nullptr, C, Lin, stride);
    if (rc != SDR_OK || !dz) return rc;
    return launch(dw_finish_kernel, (unsigned)((C * 6 + kBwThreads - 1) / kBwThreads), kBwThreads, 0, st, scratch, gw,
                  gb, samples, C);
}

// ---------------------------------------------------------------------------
// mask: masked = relu(mlog) * e (recompute) and its backward
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kBwThreads)
mask_apply_kernel(const float* __restrict__ mlog, const float* __restrict__ e, float* __restrict__ masked, int S,
                  int N, int L, long long total) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const long long NL = (long long)N * L;
    const long long b = i / (S * NL), r = i % NL;
    masked[i] = relu(mlog[i]) * __ldg(e + b * NL + r);
}

// dmlog = dmasked * e * [mlog > 0] (in place over dmasked), de = sum_s dmasked * relu(mlog).
__global__ void __launch_bounds__(kBwThreads)
mask_bwd_kernel(const float* __restrict__ mlog, const float* __restrict__ e, float* __restrict__ dmasked,
                float* __restrict__ de, int S, int N, int L, long long total) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const long long NL = (long long)N * L;
    const long long b = i / NL, r = i % NL;
    const float ev = __ldg(e + i);
    float acc = 0.f;
    for (int s = 0; s < S; ++s) {
        const size_t o = (size_t)(b * S + s) * NL + r;
        const float ml = mlog[o], g = dmasked[o];
        const bool on = ml > 0.f;
        if (on) acc = fmaf(g, ml, acc);
        dmasked[o] = on ? g * ev : 0.f;
    }
    de[i] = acc;
}

int launch_mask_apply(const float* mlog, const float* e, float* masked, int B, int S, int N, int L, cudaStream_t st) {
    if (!mlog || !e || !masked || B <= 0 || S <= 0 || N <= 0 || L <= 0) return SDR_ERR_BAD_ARGUMENT;
    const long long total = (long long)B * S * N * L;
    return launch(mask_apply_kernel, (unsigned)((total + kBwThreads - 1) / kBwThreads), kBwThreads, 0, st, mlog, e,
                  masked, S, N, L, total);
}

int launch_mask_bwd(const float* mlog, const float* e, float* dmasked, float* de, int B, int S, int N, int L,
                    cudaStream_t st) {
    if (!mlog || !e || !dmasked || !de || B <= 0 || S <= 0 || N <= 0 || L <= 0) return SDR_ERR_BAD_ARGUMENT;
    const long long total = (long long)B * N * L;
    return launch(mask_bwd_kernel, (unsigned)((total + kBwThreads - 1) / kBwThreads), kBwThreads, 0, st, mlog, e,
                  dmasked, de, S, N, L, total);
}

// ---------------------------------------------------------------------------
// frame gather: frames[b][s K + j][t] = wav[b][s][hop t + j - hop], zero outside [0, T)
// ---------------------------------------------------------------------------
// The decoder's crop + overlap-add read backwards (wav = dOut), and the encoder's input windows (wav = mixture, SA = 1).
__global__ void __launch_bounds__(kBwThreads)
frame_gather_kernel(const float* __restrict__ wav, float* __restrict__ frames, int SA, int K, int L, long long T,
                    long long total) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int hop = K / 2;
    const long long t = i % L, r = (i / L) % ((long long)SA * K), b = i / ((long long)L * SA * K);
    const long long s = r / K, j = r % K;
    const long long tau = hop * t + j - hop;
    frames[i] = (tau >= 0 && tau < T) ? __ldg(wav + (b * SA + s) * T + tau) : 0.f;
}

int launch_frame_gather(const float* wav, float* frames, int B, int SA, int K, int L, long long T, cudaStream_t st) {
    if (!wav || !frames || B <= 0 || SA <= 0 || K < 3 || (K % 2) == 0 || L <= 0 || T <= 0) return SDR_ERR_BAD_ARGUMENT;
    const long long total = (long long)B * SA * K * L;
    const long long grid = (total + kBwThreads - 1) / kBwThreads;
    if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    return launch(frame_gather_kernel, (unsigned)grid, kBwThreads, 0, st, wav, frames, SA, K, L, T, total);
}

// ---------------------------------------------------------------------------
// [R][C] -> [C][R]: the transposed weights the input-gradient GEMMs read
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kBwThreads)
transpose_kernel(const float* __restrict__ w, float* __restrict__ wt, int R, int C) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)R * C) return;
    const int r = (int)(i / C), c = (int)(i % C);
    wt[(size_t)c * R + r] = __ldg(w + i);
}

int launch_transpose(const float* w, float* wt, int R, int C, cudaStream_t st) {
    if (!w || !wt || R <= 0 || C <= 0) return SDR_ERR_BAD_ARGUMENT;
    const long long n = (long long)R * C;
    return launch(transpose_kernel, (unsigned)((n + kBwThreads - 1) / kBwThreads), kBwThreads, 0, st, w, wt, R, C);
}

}  // namespace sdr
