// Steps either side of the forward (SURVEY.md 8f rows 1 and 2):
//   * per-utterance normalisation before the model and the rescale after it
//     (reference README.md:100-109: std is torch's unbiased std over time,
//      input = (x - mean) / (std + 1e-9), output = est * std + mean);
//   * permutation-invariant SI-SDR(i) evaluation of a batch of estimates
//     (reference dnn/losses/sisdr.py:66-194, class PermInvariantSISDR).
// Both are tiny HBM-streaming reductions next to the forward (a few MB per batch);
// they exist so that `separate()` and the validation metric never leave the device.
#include "common.cuh"
#include "launchers.cuh"

namespace sdr {

// ---------------------------------------------------------------------------
// utterance moments: sums[row] = (sum_t x, sum_t x^2), fp64
// grid = rows * chunks, 256 threads; the caller zeroes `sums`.
// Rows are T apart; with `lengths` (ragged batch, zero-padded to T) only the first
// lengths[row] samples of a row are the utterance.
// ---------------------------------------------------------------------------
__device__ __forceinline__ long long row_length(const long long* lengths, int row, long long T) {
    if (!lengths) return T;
    const long long n = lengths[row];
    return n < 0 ? 0 : (n > T ? T : n);
}

__global__ void __launch_bounds__(256)
row_moments_kernel(const float* __restrict__ x, double* __restrict__ sums, long long T, int chunks,
                   const long long* __restrict__ lengths) {
    __shared__ double red[2][8];
    const int row = blockIdx.x / chunks, chunk = blockIdx.x - row * chunks;
    const long long Tr = row_length(lengths, row, T);
    const long long per = (Tr + chunks - 1) / chunks;
    const long long t0 = (long long)chunk * per;
    const long long t1 = t0 + per < Tr ? t0 + per : Tr;
    const float* xr = x + (size_t)row * T;
    double s = 0.0, q = 0.0;
    for (long long t = t0 + threadIdx.x; t < t1; t += 256) {
        const double v = (double)__ldg(xr + t);
        s += v;
        q = fma(v, v, q);
    }
    s = warp_sum_f64(s);
    q = warp_sum_f64(q);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { red[0][warp] = s; red[1][warp] = q; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double ts = 0.0, tq = 0.0;
        for (int w = 0; w < 8; ++w) { ts += red[0][w]; tq += red[1][w]; }
        atomicAdd(sums + 2 * (size_t)row, ts);
        atomicAdd(sums + 2 * (size_t)row + 1, tq);
    }
}

// (mean, unbiased std) per row as fp32, the precision the reference carries them in
__global__ void row_mean_std_kernel(const double* __restrict__ sums, float2* __restrict__ ms, int rows, long long T,
                                    const long long* __restrict__ lengths) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const double n = (double)row_length(lengths, r, T);
    const double s = sums[2 * (size_t)r], q = sums[2 * (size_t)r + 1];
    const double mean = s / n;
    double var = (q - s * mean) / (n - 1.0);          // torch.std default: Bessel's correction (T == 1 -> NaN, as torch)
    if (var < 0.0) var = 0.0;
    ms[r] = make_float2((float)mean, (float)sqrt(var));
}

// y = (x - mean) / (std + 1e-9)      (README.md:103)
__global__ void __launch_bounds__(256)
normalize_rows_kernel(const float* __restrict__ x, const float2* __restrict__ ms, float* __restrict__ y, int rows,
                      long long T, const long long* __restrict__ lengths) {
    for (long long row = blockIdx.y; row < rows; row += gridDim.y) {   // grid.y is capped at 65535; row + gridDim.y
                                                                       // may pass INT_MAX
        const float2 m = ms[row];
        const float den = m.y + 1e-9f;
        const size_t base = (size_t)row * T;
        const long long Tr = row_length(lengths, row, T);      // beyond the utterance: the zero padding stays zero
        for (long long t = (long long)blockIdx.x * 256 + threadIdx.x; t < T; t += (long long)gridDim.x * 256)
            y[base + t] = t < Tr ? (__ldg(x + base + t) - m.x) / den : 0.f;
    }
}

int launch_utterance_stats(const float* wav, double* sums, float2* mean_std, int rows, long long T,
                           const long long* lengths, cudaStream_t st) {
    if (!wav || !sums || !mean_std || rows <= 0 || T <= 0) return SDR_ERR_BAD_ARGUMENT;
    if (cudaMemsetAsync(sums, 0, sizeof(double) * 2 * rows, st) != cudaSuccess) return SDR_ERR_CUDA;
    int chunks = (int)((T + 8191) / 8192);
    if (chunks < 1) chunks = 1;
    if (chunks > 64) chunks = 64;
    const long long grid = (long long)rows * chunks;
    if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    row_moments_kernel<<<(unsigned)grid, 256, 0, st>>>(wav, sums, T, chunks, lengths);
    row_mean_std_kernel<<<(rows + 127) / 128, 128, 0, st>>>(sums, mean_std, rows, T, lengths);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

int launch_normalize_rows(const float* wav, const float2* mean_std, float* out, int rows, long long T,
                          const long long* lengths, cudaStream_t st) {
    if (!wav || !mean_std || !out || rows <= 0 || T <= 0) return SDR_ERR_BAD_ARGUMENT;
    long long gx = (T + 256 * 4 - 1) / (256 * 4);
    if (gx < 1) gx = 1;
    if (gx > 4096) gx = 4096;
    normalize_rows_kernel<<<dim3((unsigned)gx, (unsigned)(rows < 65535 ? rows : 65535)), 256, 0, st>>>(
        wav, mean_std, out, rows, T, lengths);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

// ---------------------------------------------------------------------------
// permutation-invariant SI-SDR (sisdr.py:66-194)
//
// Everything the metric needs is an inner product over time, so ONE pass gathers, per
// batch item, the sums of the 2S+1 signals (estimates e_i, targets t_j, mixture m) and
// the products <e_i,t_j>, <t_j,t_j>, <e_i,e_i>, <m,t_j>, <m,m> in fp64; a second,
// single-block kernel removes the means (zero_mean, sisdr.py:104-111), forms
//     alpha = <e,t> / (<t,t> + eps),  |s_t|^2 = alpha^2 <t,t>,
//     |e_t|^2 = <e,e> - 2 alpha <e,t> + alpha^2 <t,t>
//     sisnr   = 10 log10(|s_t|^2 / (|e_t|^2 + eps))                  (sisdr.py:117-125)
// for every (estimate, target) pair, averages over sources for each permutation
// (itertools.permutations order), keeps the best (sisdr.py:139-141) and, for SI-SDRi,
// subtracts the BATCH mean of the mixture's own sisnr (sisdr.py:143-148).
// Layout of acc[b]: [0,V) sums; then ET[S*S] (i*S+j), TT[S], EE[S], MT[S], MM.
// ---------------------------------------------------------------------------
template <int S> struct PitLayout {
    static constexpr int V = 2 * S + 1;
    static constexpr int ET = V, TT = ET + S * S, EE = TT + S, MT = EE + S, MM = MT + S, N = MM + 1;
};

template <int S>
__global__ void __launch_bounds__(256)
pit_gram_kernel(const float* __restrict__ est, const float* __restrict__ tgt, const float* __restrict__ mix,
                double* __restrict__ acc, long long T, int chunks) {
    using P = PitLayout<S>;
    __shared__ double red[8][P::N];
    const int b = blockIdx.x / chunks, chunk = blockIdx.x - b * chunks;
    const long long per = (T + chunks - 1) / chunks;
    const long long t0 = (long long)chunk * per;
    const long long t1 = t0 + per < T ? t0 + per : T;
    double a[P::N];
#pragma unroll
    for (int i = 0; i < P::N; ++i) a[i] = 0.0;
    const float* eb = est + (size_t)b * S * T;
    const float* tb = tgt + (size_t)b * S * T;
    const float* mb = mix ? mix + (size_t)b * T : nullptr;
    for (long long t = t0 + threadIdx.x; t < t1; t += 256) {
        double e[S], g[S];
#pragma unroll
        for (int i = 0; i < S; ++i) { e[i] = (double)__ldg(eb + (size_t)i * T + t); g[i] = (double)__ldg(tb + (size_t)i * T + t); }
        const double m = mb ? (double)__ldg(mb + t) : 0.0;
#pragma unroll
        for (int i = 0; i < S; ++i) {
            a[i] += e[i];
            a[S + i] += g[i];
            a[P::TT + i] = fma(g[i], g[i], a[P::TT + i]);
            a[P::EE + i] = fma(e[i], e[i], a[P::EE + i]);
            a[P::MT + i] = fma(m, g[i], a[P::MT + i]);
#pragma unroll
            for (int j = 0; j < S; ++j) a[P::ET + i * S + j] = fma(e[i], g[j], a[P::ET + i * S + j]);
        }
        a[2 * S] += m;
        a[P::MM] = fma(m, m, a[P::MM]);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < P::N; ++i) {
        const double v = warp_sum_f64(a[i]);
        if (lane == 0) red[warp][i] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < P::N; i += 256) {
        double v = 0.0;
        for (int w = 0; w < 8; ++w) v += red[w][i];
        atomicAdd(acc + (size_t)b * P::N + i, v);
    }
}

// A mean-removed energy sum(x^2) - n * mean^2 can round to a few ulp below zero (a constant row under zero_mean);
// the energy it stands for is never negative.  NaN passes through.
__device__ __forceinline__ double clamp_energy(double v) { return v < 0.0 ? 0.0 : v; }

// torch.max's selection over candidates in order: the first NaN wins and is kept, otherwise the first maximum.
__device__ __forceinline__ bool takes_max(double m, double best, int idx) {
    return idx == 0 || (!isnan(best) && (isnan(m) || m > best));
}

__device__ __forceinline__ double sisnr_from_dots(double et, double tt, double ee, double eps) {
    const double alpha = et / (tt + eps);
    const double st = alpha * alpha * tt;
    double er = ee - 2.0 * alpha * et + st;
    if (er < 0.0) er = 0.0;
    return 10.0 * log10(st / (er + eps));
}

// one block; thread-strided over the batch.  best[b], perm[b] (index in itertools.permutations order)
template <int S>
__global__ void __launch_bounds__(256)
pit_finalize_kernel(const double* __restrict__ acc, float* __restrict__ best, int* __restrict__ perm,
                    int B, long long T, int zero_mean, int improvement, double eps) {
    using P = PitLayout<S>;
    __shared__ double red[8];
    __shared__ double s_base;
    const double n = (double)T;
    double base_sum = 0.0;
    for (int b = threadIdx.x; b < B; b += 256) {
        const double* a = acc + (size_t)b * P::N;
        double me[S], mt[S], mm = 0.0;
#pragma unroll
        for (int i = 0; i < S; ++i) { me[i] = zero_mean ? a[i] / n : 0.0; mt[i] = zero_mean ? a[S + i] / n : 0.0; }
        if (zero_mean) mm = a[2 * S] / n;
        double tt[S], ee[S], sn[S][S];
#pragma unroll
        for (int j = 0; j < S; ++j) tt[j] = clamp_energy(a[P::TT + j] - n * mt[j] * mt[j]);
#pragma unroll
        for (int i = 0; i < S; ++i) ee[i] = clamp_energy(a[P::EE + i] - n * me[i] * me[i]);
#pragma unroll
        for (int i = 0; i < S; ++i)
#pragma unroll
            for (int j = 0; j < S; ++j)
                sn[i][j] = sisnr_from_dots(a[P::ET + i * S + j] - n * me[i] * mt[j], tt[j], ee[i], eps);
        // permutations in lexicographic order (itertools.permutations(range(S))): perm p maps target j -> estimate p[j]
        double bestv = 0.0;
        int besti = 0, idx = 0;
        int p[S];
#pragma unroll
        for (int i = 0; i < S; ++i) p[i] = i;
        while (true) {
            double m = 0.0;
            for (int j = 0; j < S; ++j) m += sn[p[j]][j];
            m /= (double)S;
            if (takes_max(m, bestv, idx)) { bestv = m; besti = idx; }
            ++idx;
            // next lexicographic permutation
            int k = S - 2;
            while (k >= 0 && p[k] > p[k + 1]) --k;
            if (k < 0) break;
            int l = S - 1;
            while (p[l] < p[k]) --l;
            int tmp = p[k]; p[k] = p[l]; p[l] = tmp;
            for (int lo = k + 1, hi = S - 1; lo < hi; ++lo, --hi) { tmp = p[lo]; p[lo] = p[hi]; p[hi] = tmp; }
        }
        best[b] = (float)bestv;
        perm[b] = besti;
        if (improvement) {
            const double em = clamp_energy(a[P::MM] - n * mm * mm);
            for (int j = 0; j < S; ++j)
                base_sum += sisnr_from_dots(a[P::MT + j] - n * mm * mt[j], tt[j], em, eps);
        }
    }
    if (!improvement) return;
    base_sum = warp_sum_f64(base_sum);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = base_sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += red[w];
        s_base = t / ((double)B * S);              // base_sisdr.mean(): over the whole batch (sisdr.py:148)
    }
    __syncthreads();
    const double base = s_base;
    for (int b = threadIdx.x; b < B; b += 256) best[b] = (float)((double)best[b] - base);
}

template <int S>
static int launch_pit_s(const float* est, const float* tgt, const float* mix, float* best, int* perm,
                        int B, long long T, int zero_mean, int improvement, double eps, double* acc, cudaStream_t st) {
    using P = PitLayout<S>;
    if (cudaMemsetAsync(acc, 0, sizeof(double) * P::N * B, st) != cudaSuccess) return SDR_ERR_CUDA;
    int chunks = (int)((T + 4095) / 4096);
    if (chunks < 1) chunks = 1;
    if (chunks > 64) chunks = 64;
    const long long grid = (long long)B * chunks;
    if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    pit_gram_kernel<S><<<(unsigned)grid, 256, 0, st>>>(est, tgt, mix, acc, T, chunks);
    pit_finalize_kernel<S><<<1, 256, 0, st>>>(acc, best, perm, B, T, zero_mean, improvement, eps);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

// ---------------------------------------------------------------------------
// pairwise negative SNR / SI-SDR / SD-SDR (sisdr.py:372-457, PairwiseNegSDR): out[b, i, j] = -sdr(estimate i, target j),
// from the same one-pass fp64 Gram as the PIT metric.  With d = <e_i, t_j>, tt = <t_j, t_j>, ee = <e_i, e_i>
// (means removed when zero_mean) and c = d / (tt + 1e-8):
//     sisdr:  |proj|^2 = c^2 tt,  |noise|^2 = ee - 2 c d + c^2 tt
//     sdsdr:  |proj|^2 = c^2 tt,  |noise|^2 = ee - 2 d + tt
//     snr:    |proj|^2 = tt,      |noise|^2 = ee - 2 d + tt
//     sdr = |proj|^2 / (|noise|^2 + 1e-8);  take_log: 10 log10(sdr + 1e-8)
// ---------------------------------------------------------------------------
template <int S>
__global__ void __launch_bounds__(256)
pairwise_finalize_kernel(const double* __restrict__ acc, float* __restrict__ out, int B, long long T,
                         int sdr_type, int zero_mean, int take_log) {
    using P = PitLayout<S>;
    const double n = (double)T;
    for (int b = blockIdx.x * 256 + threadIdx.x; b < B; b += gridDim.x * 256) {
        const double* a = acc + (size_t)b * P::N;
        double me[S], mt[S];
#pragma unroll
        for (int i = 0; i < S; ++i) { me[i] = zero_mean ? a[i] / n : 0.0; mt[i] = zero_mean ? a[S + i] / n : 0.0; }
#pragma unroll
        for (int i = 0; i < S; ++i) {
            const double ee = clamp_energy(a[P::EE + i] - n * me[i] * me[i]);
#pragma unroll
            for (int j = 0; j < S; ++j) {
                const double tt = clamp_energy(a[P::TT + j] - n * mt[j] * mt[j]);
                const double d = a[P::ET + i * S + j] - n * me[i] * mt[j];
                const double c = d / (tt + 1e-8);
                const double proj = sdr_type == 0 ? tt : c * c * tt;                       // 0 snr, 1 sisdr, 2 sdsdr
                double noise = sdr_type == 1 ? ee - 2.0 * c * d + c * c * tt : ee - 2.0 * d + tt;
                if (sdr_type != 1 && isinf(ee) && isfinite(tt)) noise = ee;    // |e - t|^2 with an inf in e: inf - inf above
                if (noise < 0.0) noise = 0.0;
                double v = proj / (noise + 1e-8);
                if (take_log) v = 10.0 * log10(v + 1e-8);
                out[((size_t)b * S + i) * S + j] = (float)(-v);
            }
        }
    }
}

template <int S>
static int launch_pairwise_s(const float* est, const float* tgt, float* out, int B, long long T, int sdr_type,
                             int zero_mean, int take_log, double* acc, cudaStream_t st) {
    using P = PitLayout<S>;
    if (cudaMemsetAsync(acc, 0, sizeof(double) * P::N * B, st) != cudaSuccess) return SDR_ERR_CUDA;
    int chunks = (int)((T + 4095) / 4096);
    if (chunks < 1) chunks = 1;
    if (chunks > 64) chunks = 64;
    const long long grid = (long long)B * chunks;
    if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    pit_gram_kernel<S><<<(unsigned)grid, 256, 0, st>>>(est, tgt, nullptr, acc, T, chunks);
    pairwise_finalize_kernel<S><<<(unsigned)((B + 255) / 256), 256, 0, st>>>(acc, out, B, T, sdr_type, zero_mean, take_log);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

int launch_pairwise_neg_sdr(const float* est, const float* tgt, float* out, int B, int S, long long T, int sdr_type,
                            int zero_mean, int take_log, void* scratch, cudaStream_t st) {
    if (!est || !tgt || !out || !scratch || B <= 0 || T <= 0 || sdr_type < 0 || sdr_type > 2) return SDR_ERR_BAD_ARGUMENT;
    double* acc = static_cast<double*>(scratch);
    switch (S) {
        case 1: return launch_pairwise_s<1>(est, tgt, out, B, T, sdr_type, zero_mean, take_log, acc, st);
        case 2: return launch_pairwise_s<2>(est, tgt, out, B, T, sdr_type, zero_mean, take_log, acc, st);
        case 3: return launch_pairwise_s<3>(est, tgt, out, B, T, sdr_type, zero_mean, take_log, acc, st);
        case 4: return launch_pairwise_s<4>(est, tgt, out, B, T, sdr_type, zero_mean, take_log, acc, st);
        default: return SDR_ERR_UNSUPPORTED;
    }
}

// ---------------------------------------------------------------------------
// StabilizedPermInvSISDRMetric (sisdr.py:460-591), the validation metric of run_fuss_separation.py:111-131:
// SE estimated sources against SA <= SE actual ones,
//     rho^2 = <e,t>^2 / (<e,e> <t,t> + eps),  sisnr = 10 log10((rho^2 + eps) / (1 - rho^2 + eps))    (:508-515)
// best source-mean over the assignments itertools.permutations(range(SE), r=SA) (:490-492,526-533); for the
// improvement the mixture is the SUM of the (mean-removed) targets (:535-541), so its inner products are sums of the
// target Gram <t_j, t_k>, which this pass therefore keeps in full.  single_source (:576-577): the `rows` estimate rows
// of an item are summed on load and scored as one source.
// Layout of acc[b]: sums e[SE], t[SA]; ET[SE*SA] (i*SA+j); EE[SE]; TT[SA*SA].
// ---------------------------------------------------------------------------
template <int SE, int SA> struct StabLayout {
    static constexpr int V = SE + SA;
    static constexpr int ET = V, EE = ET + SE * SA, TT = EE + SE, N = TT + SA * SA;
};

template <int SE, int SA>
__global__ void __launch_bounds__(256)
stab_gram_kernel(const float* __restrict__ est, const float* __restrict__ tgt, double* __restrict__ acc,
                 long long T, int chunks, int rows) {
    using P = StabLayout<SE, SA>;
    __shared__ double red[8][P::N];
    const int b = blockIdx.x / chunks, chunk = blockIdx.x - b * chunks;
    const long long per = (T + chunks - 1) / chunks;
    const long long t0 = (long long)chunk * per;
    const long long t1 = t0 + per < T ? t0 + per : T;
    double a[P::N];
#pragma unroll
    for (int i = 0; i < P::N; ++i) a[i] = 0.0;
    const float* eb = est + (size_t)b * rows * T;
    const float* tb = tgt + (size_t)b * SA * T;
    for (long long t = t0 + threadIdx.x; t < t1; t += 256) {
        double e[SE], g[SA];
        if (SE == 1 && rows > 1) {                         // single_source: the estimates are summed first (fp32, as torch.sum)
            float sum = 0.f;
            for (int r = 0; r < rows; ++r) sum += __ldg(eb + (size_t)r * T + t);
            e[0] = (double)sum;
        } else {
#pragma unroll
            for (int i = 0; i < SE; ++i) e[i] = (double)__ldg(eb + (size_t)i * T + t);
        }
#pragma unroll
        for (int j = 0; j < SA; ++j) g[j] = (double)__ldg(tb + (size_t)j * T + t);
#pragma unroll
        for (int i = 0; i < SE; ++i) {
            a[i] += e[i];
            a[P::EE + i] = fma(e[i], e[i], a[P::EE + i]);
#pragma unroll
            for (int j = 0; j < SA; ++j) a[P::ET + i * SA + j] = fma(e[i], g[j], a[P::ET + i * SA + j]);
        }
#pragma unroll
        for (int j = 0; j < SA; ++j) {
            a[SE + j] += g[j];
#pragma unroll
            for (int k = 0; k < SA; ++k) a[P::TT + j * SA + k] = fma(g[j], g[k], a[P::TT + j * SA + k]);
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < P::N; ++i) {
        const double v = warp_sum_f64(a[i]);
        if (lane == 0) red[warp][i] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < P::N; i += 256) {
        double v = 0.0;
        for (int w = 0; w < 8; ++w) v += red[w][i];
        atomicAdd(acc + (size_t)b * P::N + i, v);
    }
}

__device__ __forceinline__ double stab_sisnr(double et, double ee, double tt, double eps) {
    double rho = et * et / (ee * tt + eps);
    if (rho > 1.0) rho = 1.0;          // a squared correlation; rounding of the Gram form can push it past 1 (then NaN)
    return 10.0 * log10((rho + eps) / (1.0 - rho + eps));
}

// one block; thread-strided over the batch.  best[b], perm[b] (index in itertools.permutations(range(SE), r=SA) order)
template <int SE, int SA>
__global__ void __launch_bounds__(256)
stab_finalize_kernel(const double* __restrict__ acc, float* __restrict__ best, int* __restrict__ perm,
                     int B, long long T, int zero_mean, int improvement, double eps) {
    using P = StabLayout<SE, SA>;
    __shared__ double red[8];
    __shared__ double s_base;
    const double n = (double)T;
    double base_sum = 0.0;
    for (int b = threadIdx.x; b < B; b += 256) {
        const double* a = acc + (size_t)b * P::N;
        double me[SE], mt[SA];
#pragma unroll
        for (int i = 0; i < SE; ++i) me[i] = zero_mean ? a[i] / n : 0.0;
#pragma unroll
        for (int j = 0; j < SA; ++j) mt[j] = zero_mean ? a[SE + j] / n : 0.0;
        double tt[SA][SA], sn[SE][SA];
#pragma unroll
        for (int j = 0; j < SA; ++j)
#pragma unroll
            for (int k = 0; k < SA; ++k) tt[j][k] = a[P::TT + j * SA + k] - n * mt[j] * mt[k];
#pragma unroll
        for (int j = 0; j < SA; ++j) tt[j][j] = clamp_energy(tt[j][j]);
#pragma unroll
        for (int i = 0; i < SE; ++i) {
            const double ee = clamp_energy(a[P::EE + i] - n * me[i] * me[i]);
#pragma unroll
            for (int j = 0; j < SA; ++j)
                sn[i][j] = stab_sisnr(a[P::ET + i * SA + j] - n * me[i] * mt[j], ee, tt[j][j], eps);
        }
        // assignments p[0..SA) of distinct estimates, lexicographic (= itertools.permutations(range(SE), r=SA))
        double bestv = 0.0;
        int besti = 0, idx = 0;
        int total = 1;
#pragma unroll
        for (int j = 0; j < SA; ++j) total *= SE;
        for (int code = 0; code < total; ++code) {
            int p[SA], c = code;
            bool ok = true;
#pragma unroll
            for (int j = SA - 1; j >= 0; --j) { p[j] = c % SE; c /= SE; }      // p[0] is the most significant digit
#pragma unroll
            for (int j = 0; j < SA; ++j)
#pragma unroll
                for (int k = 0; k < SA; ++k) if (k < j && p[k] == p[j]) ok = false;
            if (!ok) continue;
            double m = 0.0;
#pragma unroll
            for (int j = 0; j < SA; ++j) {
                double v = 0.0;
#pragma unroll
                for (int i = 0; i < SE; ++i) if (p[j] == i) v = sn[i][j];
                m += v;
            }
            m /= (double)SA;
            if (takes_max(m, bestv, idx)) { bestv = m; besti = idx; }
            ++idx;
        }
        best[b] = (float)bestv;
        perm[b] = besti;
        if (improvement) {                                  // mixture = sum of the targets
            double mm = 0.0;
#pragma unroll
            for (int j = 0; j < SA; ++j)
#pragma unroll
                for (int k = 0; k < SA; ++k) mm += tt[j][k];
            mm = clamp_energy(mm);
#pragma unroll
            for (int j = 0; j < SA; ++j) {
                double mtj = 0.0;
#pragma unroll
                for (int k = 0; k < SA; ++k) mtj += tt[k][j];
                base_sum += stab_sisnr(mtj, mm, tt[j][j], eps);
            }
        }
    }
    if (!improvement) return;
    base_sum = warp_sum_f64(base_sum);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = base_sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += red[w];
        s_base = t / ((double)B * SA);             // base_sisdr.mean(): over the whole batch (sisdr.py:541)
    }
    __syncthreads();
    const double base = s_base;
    for (int b = threadIdx.x; b < B; b += 256) best[b] = (float)((double)best[b] - base);
}

template <int SE, int SA>
static int launch_stab(const float* est, const float* tgt, float* best, int* perm, int B, int rows, long long T,
                       int zero_mean, int improvement, double eps, double* acc, cudaStream_t st) {
    using P = StabLayout<SE, SA>;
    if (cudaMemsetAsync(acc, 0, sizeof(double) * P::N * B, st) != cudaSuccess) return SDR_ERR_CUDA;
    int chunks = (int)((T + 4095) / 4096);
    if (chunks < 1) chunks = 1;
    if (chunks > 64) chunks = 64;
    const long long grid = (long long)B * chunks;
    if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    stab_gram_kernel<SE, SA><<<(unsigned)grid, 256, 0, st>>>(est, tgt, acc, T, chunks, rows);
    stab_finalize_kernel<SE, SA><<<1, 256, 0, st>>>(acc, best, perm, B, T, zero_mean, improvement, eps);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

size_t stabilized_sisdr_scratch_bytes(int B, int n_est, int n_act) {
    if (B <= 0 || n_est < 1 || n_est > 4 || n_act < 1 || n_act > n_est) return 0;
    return sizeof(double) * (size_t)B * (n_est + n_act + n_est * n_act + n_est + n_act * n_act);
}

int launch_stabilized_sisdr(const float* est, const float* tgt, float* best, int* perm, int B, int rows, int n_est,
                            int n_act, long long T, int zero_mean, int improvement, double eps, void* scratch,
                            cudaStream_t st) {
    if (!est || !tgt || !best || !perm || !scratch || B <= 0 || T <= 0 || rows < 1) return SDR_ERR_BAD_ARGUMENT;
    if (rows != n_est && n_est != 1) return SDR_ERR_BAD_ARGUMENT;          // summing the rows is the single_source mode
    if (!stabilized_sisdr_scratch_bytes(B, n_est, n_act)) return SDR_ERR_UNSUPPORTED;
    double* acc = static_cast<double*>(scratch);
#define SDR_STAB(E, A) if (n_est == E && n_act == A) \
        return launch_stab<E, A>(est, tgt, best, perm, B, rows, T, zero_mean, improvement, eps, acc, st);
    SDR_STAB(1, 1) SDR_STAB(2, 1) SDR_STAB(2, 2) SDR_STAB(3, 1) SDR_STAB(3, 2) SDR_STAB(3, 3)
    SDR_STAB(4, 1) SDR_STAB(4, 2) SDR_STAB(4, 3) SDR_STAB(4, 4)
#undef SDR_STAB
    return SDR_ERR_UNSUPPORTED;
}

size_t pit_sisdr_scratch_bytes(int B, int S) {
    if (B <= 0 || S < 1 || S > 4) return 0;
    const int V = 2 * S + 1;
    return sizeof(double) * (size_t)B * (V + S * S + 3 * S + 1);
}

int launch_pit_sisdr(const float* est, const float* tgt, const float* mix, float* best, int* perm,
                     int B, int S, long long T, int zero_mean, int improvement, double eps,
                     void* scratch, cudaStream_t st) {
    if (!est || !tgt || !best || !perm || !scratch || B <= 0 || T <= 0) return SDR_ERR_BAD_ARGUMENT;
    if (improvement && !mix) return SDR_ERR_BAD_ARGUMENT;
    double* acc = static_cast<double*>(scratch);
    switch (S) {
        case 1: return launch_pit_s<1>(est, tgt, mix, best, perm, B, T, zero_mean, improvement, eps, acc, st);
        case 2: return launch_pit_s<2>(est, tgt, mix, best, perm, B, T, zero_mean, improvement, eps, acc, st);
        case 3: return launch_pit_s<3>(est, tgt, mix, best, perm, B, T, zero_mean, improvement, eps, acc, st);
        case 4: return launch_pit_s<4>(est, tgt, mix, best, perm, B, T, zero_mean, improvement, eps, acc, st);
        default: return SDR_ERR_UNSUPPORTED;     // S! permutations are enumerated per item; 4 sources = 24
    }
}

}  // namespace sdr
