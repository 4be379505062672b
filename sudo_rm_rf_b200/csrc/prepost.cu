// Steps either side of the forward (SURVEY.md 8f rows 1 and 2):
//   * per-utterance normalisation before the model and the rescale after it
//     (reference README.md:100-109: std is torch's unbiased std over time,
//      input = (x - mean) / (std + 1e-9), output = est * std + mean);
//   * the runners' SI-SDR / SNR metrics and losses (reference dnn/losses/sisdr.py and snr.py): PermInvariantSISDR,
//     PairwiseNegSDR (evaluation and autograd), StabilizedPermInvSISDRMetric and PermInvariantSNRwithZeroRefs.
// Every metric and loss is one fp64 Gram pass over time per batch item (gram_kernel), a finalize kernel that reads
// the sums through GramSums and, for the permutation-invariant ones, one assignment search (best_assignment).
// All are tiny HBM-streaming reductions next to the forward (a few MB per batch); they exist so that `separate()`,
// the validation metrics and the training losses never leave the device.
#include "assign.cuh"
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
    if (const int rc = cuda_status(cudaMemsetAsync(sums, 0, sizeof(double) * 2 * rows, st))) return rc;
    int chunks = (int)((T + 8191) / 8192);
    if (chunks < 1) chunks = 1;
    if (chunks > 64) chunks = 64;
    const long long grid = (long long)rows * chunks;
    if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    if (const int rc = launch(row_moments_kernel, (unsigned)grid, 256, 0, st, wav, sums, T, chunks, lengths)) return rc;
    return launch(row_mean_std_kernel, (rows + 127) / 128, 128, 0, st, sums, mean_std, rows, T, lengths);
}

int launch_normalize_rows(const float* wav, const float2* mean_std, float* out, int rows, long long T,
                          const long long* lengths, cudaStream_t st) {
    if (!wav || !mean_std || !out || rows <= 0 || T <= 0) return SDR_ERR_BAD_ARGUMENT;
    return launch(normalize_rows_kernel, row_tiled_grid(rows, T), 256, 0, st, wav, mean_std, out, rows, T, lengths);
}

// ---------------------------------------------------------------------------
// The fp64 Gram pass every metric and loss below starts from.  Per batch item, one pass over time gathers the sums and
// inner products of SE estimate rows e_i and SA target rows t_j.  Layout of one item's N doubles:
//     sums e[R] (R = SE, plus the extra row with kMix), t[SA];  ET[R*SA] = <e_i, t_j> (i*SA+j);  EE[R] = <e_i, e_i>;
//     TT = <t_j, t_k>: the full [SA*SA] block with kFull, else only its diagonal [SA].
// With kMix, estimate row SE is an extra row read from its own pointer (the mixture of the PIT metric, whose SI-SDRi
// baseline needs <m, t_j>, <m, m> and sum m): GramLayout<S, S, false, true> is the PIT metric's S^2 + 5S + 2 doubles.
// ---------------------------------------------------------------------------
template <int SE_, int SA_, bool kFull_, bool kMix_> struct GramLayout {
    static constexpr int SE = SE_, SA = SA_;
    static constexpr bool kFull = kFull_, kMix = kMix_;
    static constexpr int R = SE + (kMix ? 1 : 0);
    static constexpr int ET = R + SA, EE = ET + R * SA, TT = EE + R, N = TT + (kFull ? SA * SA : SA);
};

// grid = B * chunks CTAs of 256 threads, each over one chunk of one item's time axis.  Rows are T apart; an item has
// `rows` estimate rows (SE except in single_source, where SE == 1 and the rows are summed on load and scored as one
// source), SA target rows and, with kMix, one extra row.  kOrdered: each CTA writes its chunk's sums to
// acc[blockIdx.x] (layout [b][chunk][N]) and the reader adds the chunks in index order, so the result is bitwise
// reproducible; otherwise it adds them to acc[b] atomically.
template <class L, bool kOrdered>
__global__ void __launch_bounds__(256)
gram_kernel(const float* __restrict__ est, const float* __restrict__ tgt, const float* __restrict__ extra,
            double* __restrict__ acc, long long T, int chunks, int rows) {
    constexpr int SE = L::SE, SA = L::SA, R = L::R;
    __shared__ double red[8][L::N];
    const int b = blockIdx.x / chunks, chunk = blockIdx.x - b * chunks;
    const long long per = (T + chunks - 1) / chunks;
    const long long t0 = (long long)chunk * per;
    const long long t1 = t0 + per < T ? t0 + per : T;
    double a[L::N];
#pragma unroll
    for (int i = 0; i < L::N; ++i) a[i] = 0.0;
    // Only the stabilised metric's items (full layout) can have more rows than SE; elsewhere the stride is known at
    // compile time, which saves the diagonal passes registers.
    const float* eb = est + (size_t)b * (L::kFull ? rows : SE) * T;
    const float* tb = tgt + (size_t)b * SA * T;
    const float* xb = extra ? extra + (size_t)b * T : nullptr;
    for (long long t = t0 + threadIdx.x; t < t1; t += 256) {
        double e[R], g[SA];                                // SA <= SE: estimate row i is loaded with target row i
#pragma unroll
        for (int i = 0; i < SE; ++i) {
            if (SE == 1 && rows > 1) {                     // single_source: the estimates are summed first (fp32, as torch.sum)
                float sum = 0.f;
                for (int r = 0; r < rows; ++r) sum += __ldg(eb + (size_t)r * T + t);
                e[0] = (double)sum;
            } else {
                e[i] = (double)__ldg(eb + (size_t)i * T + t);
            }
            if (i < SA) g[i] = (double)__ldg(tb + (size_t)i * T + t);
        }
        if constexpr (L::kMix) e[SE] = xb ? (double)__ldg(xb + t) : 0.0;
#pragma unroll
        for (int i = 0; i < R; ++i) {
            a[i] += e[i];
            a[L::EE + i] = fma(e[i], e[i], a[L::EE + i]);
#pragma unroll
            for (int j = 0; j < SA; ++j) a[L::ET + i * SA + j] = fma(e[i], g[j], a[L::ET + i * SA + j]);
        }
#pragma unroll
        for (int j = 0; j < SA; ++j) {
            a[R + j] += g[j];
            if constexpr (L::kFull) {
#pragma unroll
                for (int k = 0; k < SA; ++k) a[L::TT + j * SA + k] = fma(g[j], g[k], a[L::TT + j * SA + k]);
            } else {
                a[L::TT + j] = fma(g[j], g[j], a[L::TT + j]);
            }
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < L::N; ++i) {
        const double v = warp_sum_f64(a[i]);
        if (lane == 0) red[warp][i] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < L::N; i += 256) {
        double v = 0.0;
        for (int w = 0; w < 8; ++w) v += red[w][i];
        if (kOrdered) acc[(size_t)blockIdx.x * L::N + i] = v;
        else atomicAdd(acc + (size_t)b * L::N + i, v);
    }
}

// Launches the Gram pass of layout L into `acc`; the atomic mode zeroes its B * N sums first.
template <class L, bool kOrdered>
static int launch_gram(const float* est, const float* tgt, const float* extra, int rows, int B, long long T,
                       double* acc, cudaStream_t st) {
    if (!kOrdered)
        if (const int rc = cuda_status(cudaMemsetAsync(acc, 0, sizeof(double) * L::N * B, st))) return rc;
    const int chunks = gram_chunks(T);
    const long long grid = (long long)B * chunks;
    if (grid > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    return launch(gram_kernel<L, kOrdered>, (unsigned)grid, 256, 0, st, est, tgt, extra, acc, T, chunks, rows);
}

// A mean-removed energy sum(x^2) - n * mean^2 can round to a few ulp below zero (a constant row under zero_mean);
// the energy it stands for is never negative.  NaN passes through.
__device__ __forceinline__ double clamp_energy(double v) { return v < 0.0 ? 0.0 : v; }

// One item's Gram sums, read back: `chunks` partial sums per item ([b][chunk][N], added in chunk order; the atomic
// mode's one sum per item is chunks = 1), with the row means removed under zero_mean (sisdr.py:104-111).
template <class L> struct GramSums {
    double a[L::N], me[L::R], mt[L::SA], n;
    __device__ __forceinline__ GramSums(const double* acc, int chunks, long long b, long long T, int zero_mean)
        : n((double)T) {
#pragma unroll
        for (int i = 0; i < L::N; ++i) a[i] = 0.0;
        for (int c = 0; c < chunks; ++c) {
            const double* pc = acc + ((size_t)b * chunks + c) * L::N;
#pragma unroll
            for (int i = 0; i < L::N; ++i) a[i] += pc[i];
        }
#pragma unroll
        for (int i = 0; i < L::R; ++i) me[i] = zero_mean ? a[i] / n : 0.0;
#pragma unroll
        for (int j = 0; j < L::SA; ++j) mt[j] = zero_mean ? a[L::R + j] / n : 0.0;
    }
    // <e_i, t_j>
    __device__ __forceinline__ double et(int i, int j) const { return a[L::ET + i * L::SA + j] - n * me[i] * mt[j]; }
    // clamped <e_i, e_i>
    __device__ __forceinline__ double ee(int i) const { return clamp_energy(a[L::EE + i] - n * me[i] * me[i]); }
    // <t_j, t_k> as summed, not clamped (full layout)
    __device__ __forceinline__ double tt(int j, int k) const {
        static_assert(L::kFull, "the diagonal layout keeps only the target energies");
        return a[L::TT + j * L::SA + k] - n * mt[j] * mt[k];
    }
    // clamped <t_j, t_j>
    __device__ __forceinline__ double td(int j) const {
        return clamp_energy(a[L::TT + (L::kFull ? j * L::SA + j : j)] - n * mt[j] * mt[j]);
    }
};

// SI-SDRi: best[b] -= the batch mean of the mixture's own scores (base_sisdr.mean() over the whole batch,
// sisdr.py:148 and :541).  One block of 256 threads; base_sum is the sum over this thread's items, count the number of
// scores in the batch.
__device__ void subtract_batch_baseline(float* best, int B, double base_sum, double count) {
    __shared__ double red[8];
    __shared__ double s_base;
    base_sum = warp_sum_f64(base_sum);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = base_sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += red[w];
        s_base = t / count;
    }
    __syncthreads();
    const double base = s_base;
    for (int b = threadIdx.x; b < B; b += 256) best[b] = (float)((double)best[b] - base);
}

// ---------------------------------------------------------------------------
// permutation-invariant SI-SDR (sisdr.py:66-194).  From the diagonal Gram with the mixture row, per item:
//     alpha = <e,t> / (<t,t> + eps),  |s_t|^2 = alpha^2 <t,t>,
//     |e_t|^2 = <e,e> - 2 alpha <e,t> + alpha^2 <t,t>
//     sisnr   = 10 log10(|s_t|^2 / (|e_t|^2 + eps))                  (sisdr.py:117-125)
// for every (estimate, target) pair, the best source mean over the permutations (sisdr.py:139-141) and, for SI-SDRi,
// minus the BATCH mean of the mixture's own sisnr (sisdr.py:143-148).
// ---------------------------------------------------------------------------
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
    double base_sum = 0.0;
    for (int b = threadIdx.x; b < B; b += 256) {
        const GramSums<GramLayout<S, S, false, true>> g(acc, 1, b, T, zero_mean);
        double sn[S][S];
#pragma unroll
        for (int i = 0; i < S; ++i)
#pragma unroll
            for (int j = 0; j < S; ++j) sn[i][j] = sisnr_from_dots(g.et(i, j), g.td(j), g.ee(i), eps);
        int besti, p[S];
        best[b] = (float)best_assignment<S, S>([&](const int* q) {
            double m = 0.0;
            for (int j = 0; j < S; ++j) m = __dadd_rn(m, sn[q[j]][j]);
            return m / (double)S;
        }, besti, p);
        perm[b] = besti;
        if (improvement)                                    // the mixture is estimate row S
            for (int j = 0; j < S; ++j) base_sum += sisnr_from_dots(g.et(S, j), g.td(j), g.ee(S), eps);
    }
    if (improvement) subtract_batch_baseline(best, B, base_sum, (double)B * S);
}

// ---------------------------------------------------------------------------
// pairwise negative SNR / SI-SDR / SD-SDR (sisdr.py:372-457, PairwiseNegSDR): out[b, i, j] = -sdr(estimate i, target j).
// With d = <e_i, t_j>, tt = <t_j, t_j>, ee = <e_i, e_i> (means removed when zero_mean) and c = d / (tt + 1e-8):
//     sisdr:  |proj|^2 = c^2 tt,  |noise|^2 = ee - 2 c d + c^2 tt
//     sdsdr:  |proj|^2 = c^2 tt,  |noise|^2 = ee - 2 d + tt
//     snr:    |proj|^2 = tt,      |noise|^2 = ee - 2 d + tt
//     sdr = |proj|^2 / (|noise|^2 + 1e-8);  take_log: 10 log10(sdr + 1e-8)
// Evaluation reads the atomic diagonal Gram (S^2 + 4S doubles, within sdr_pit_sisdr_scratch_bytes).  Under autograd
// (the training loss of run_improved_sudormrf.py:64-66 through PITLossWrapper) the forward reads the ordered full Gram
// that the SNR loss below also runs, and the same finalize writes, per entry, the three coefficients of
//     d out[b, i, j] / d e_i = alpha_ij (e'_i - k_ij t'_j) + beta_ij t'_j
// where e' = e - mu_e and t' = t - mu_t (the row means under zero_mean, else 0; the mean removal's own derivative
// subtracts the mean of this gradient, which is zero) and e'_i - k_ij t'_j is the noise vector: k = c for sisdr, 1 for
// sdsdr and snr.  With E = tt + 1e-8, P = |proj|^2, Q = |noise|^2 + 1e-8 and r = P / Q:
//     dr/de = (dP/de - r dQ/de) / Q,  dQ/de = 2 noise + q t',  dP/de = p t'
//     sisdr:  p = 2 c tt / E,  q = -2 c 1e-8 / E   (<noise, t'> = c 1e-8; c depends on e)
//     sdsdr:  p = 2 c tt / E,  q = 0
//     snr:    p = 0,           q = 0
// out = -r, or -10 log10(r + 1e-8) with take_log, so alpha = s 2 r / Q and beta = -s (p - r q) / Q with s = 1, or
// 10 / (ln 10 (r + 1e-8)).  Written on the noise vector, the two terms do not cancel each other: with an estimate
// equal to its target, alpha is ~1e16 and the noise exactly 0.  coef[b] = [alpha, k, beta per (i, j)][mu_e S][mu_t S],
// fp64.  pairwise_backward_kernel is one elementwise pass:
//     grad_e_i[t] = sum_j g_ij (alpha_ij (e'_i[t] - k_ij t'_j[t]) + beta_ij t'_j[t]).
// ---------------------------------------------------------------------------
struct PairTerms { double c, proj, q; };        // c, |proj|^2 and |noise|^2 + 1e-8 of one (estimate, target) pair

__device__ __forceinline__ PairTerms pairwise_terms(double d, double tt, double ee, int sdr_type) {
    const double c = d / (tt + 1e-8);
    const double proj = sdr_type == 0 ? tt : c * c * tt;                                // 0 snr, 1 sisdr, 2 sdsdr
    double noise = sdr_type == 1 ? ee - 2.0 * c * d + c * c * tt : ee - 2.0 * d + tt;
    if (sdr_type != 1 && isinf(ee) && isfinite(tt)) noise = ee;            // |e - t|^2 with an inf in e: inf - inf above
    if (noise < 0.0) noise = 0.0;
    return {c, proj, noise + 1e-8};
}

// out[b] and, when coef is non-null, the backward coefficients coef[b]
template <int S, bool kFull>
__global__ void __launch_bounds__(256)
pairwise_finalize_kernel(const double* __restrict__ acc, int chunks, float* __restrict__ out, double* __restrict__ coef,
                         int B, long long T, int sdr_type, int zero_mean, int take_log) {
    for (long long b = blockIdx.x * 256LL + threadIdx.x; b < B; b += (long long)gridDim.x * 256) {
        const GramSums<GramLayout<S, S, kFull, false>> g(acc, chunks, b, T, zero_mean);
        double* cb = coef ? coef + (size_t)b * (3 * S * S + 2 * S) : nullptr;
#pragma unroll
        for (int i = 0; i < S; ++i) {
            const double ee = g.ee(i);
#pragma unroll
            for (int j = 0; j < S; ++j) {
                const double tt = g.td(j);
                const PairTerms p = pairwise_terms(g.et(i, j), tt, ee, sdr_type);
                const double r = p.proj / p.q;
                out[((size_t)b * S + i) * S + j] = (float)(-(take_log ? 10.0 * log10(r + 1e-8) : r));
                if (!cb) continue;
                const double E = tt + 1e-8;
                const double dp = sdr_type == 0 ? 0.0 : 2.0 * p.c * tt / E;
                const double dq = sdr_type == 1 ? -2.0 * p.c * 1e-8 / E : 0.0;
                const double s = take_log ? 10.0 / (2.302585092994045684 * (r + 1e-8)) : 1.0;
                double* cij = cb + 3 * (i * S + j);
                cij[0] = s * 2.0 * r / p.q;
                cij[1] = sdr_type == 1 ? p.c : 1.0;
                cij[2] = -s * (dp - r * dq) / p.q;
            }
        }
        if (cb)
#pragma unroll
            for (int i = 0; i < S; ++i) { cb[3 * S * S + i] = g.me[i]; cb[3 * S * S + S + i] = g.mt[i]; }
    }
}

// grid row_tiled_grid(B S, T); est, tgt and grad rows are T apart
template <int S>
__global__ void __launch_bounds__(256)
pairwise_backward_kernel(const float* __restrict__ est, const float* __restrict__ tgt, const double* __restrict__ coef,
                         const float* __restrict__ grad_out, float* __restrict__ grad, int B, long long T) {
    const long long rows = (long long)B * S;
    for (long long row = blockIdx.y; row < rows; row += gridDim.y) {
        const long long b = row / S;
        const int i = (int)(row - b * S);
        const double* cb = coef + (size_t)b * (3 * S * S + 2 * S);
        const float* go = grad_out + (size_t)row * S;
        double al[S], k[S], be[S], mt[S];
#pragma unroll
        for (int j = 0; j < S; ++j) {
            const double g = (double)__ldg(go + j);
            const double* cij = cb + 3 * (i * S + j);
            al[j] = g * cij[0];
            k[j] = cij[1];
            be[j] = g * cij[2];
            mt[j] = cb[3 * S * S + S + j];
        }
        const double mi = cb[3 * S * S + i];
        const float* er = est + (size_t)row * T;
        const float* tb = tgt + (size_t)b * S * T;
        float* gr = grad + (size_t)row * T;
        for (long long t = (long long)blockIdx.x * 256 + threadIdx.x; t < T; t += (long long)gridDim.x * 256) {
            const double e = (double)__ldg(er + t) - mi;
            double v = 0.0;
#pragma unroll
            for (int j = 0; j < S; ++j) {
                const double tj = (double)__ldg(tb + (size_t)j * T + t) - mt[j];
                v = fma(al[j], fma(-k[j], tj, e), v);                   // the noise e' - k t', then its weight
                v = fma(be[j], tj, v);
            }
            gr[t] = (float)v;
        }
    }
}

// ---------------------------------------------------------------------------
// StabilizedPermInvSISDRMetric (sisdr.py:460-591), the validation metric of run_fuss_separation.py:111-131:
// SE estimated sources against SA <= SE actual ones,
//     rho^2 = <e,t>^2 / (<e,e> <t,t> + eps),  sisnr = 10 log10((rho^2 + eps) / (1 - rho^2 + eps))    (:508-515)
// best source-mean over the assignments itertools.permutations(range(SE), r=SA) (:490-492,526-533); for the
// improvement the mixture is the SUM of the (mean-removed) targets (:535-541), so its inner products are sums of the
// target Gram <t_j, t_k>, which this metric therefore reads in full.  single_source (:576-577): the `rows` estimate
// rows of an item are summed on load and scored as one source.
// ---------------------------------------------------------------------------
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
    double base_sum = 0.0;
    for (int b = threadIdx.x; b < B; b += 256) {
        const GramSums<GramLayout<SE, SA, true, false>> g(acc, 1, b, T, zero_mean);
        double sn[SE][SA];
#pragma unroll
        for (int i = 0; i < SE; ++i)
#pragma unroll
            for (int j = 0; j < SA; ++j) sn[i][j] = stab_sisnr(g.et(i, j), g.ee(i), g.td(j), eps);
        int besti, p[SA];
        best[b] = (float)best_assignment<SE, SA>([&](const int* q) {
            double m = 0.0;
            for (int j = 0; j < SA; ++j) m = __dadd_rn(m, sn[q[j]][j]);
            return m / (double)SA;
        }, besti, p);
        perm[b] = besti;
        if (improvement) {                                  // mixture = sum of the targets, their energies clamped
            double tt[SA][SA], mm = 0.0;
#pragma unroll
            for (int j = 0; j < SA; ++j)
#pragma unroll
                for (int k = 0; k < SA; ++k) mm += tt[j][k] = j == k ? g.td(j) : g.tt(j, k);
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
    if (improvement) subtract_batch_baseline(best, B, base_sum, (double)B * SA);
}

// ---------------------------------------------------------------------------
// PermInvariantSNRwithZeroRefs (dnn/losses/snr.py:13-142), the training loss of run_fuss_separation.py:257-259.
// The ordered full Gram holds every term: with means removed under zero_mean,
//     tt_k = ||t_k||^2,  mixture power mp = sum_jk <t_j, t_k> = ||sum_j t_j||^2,
//     active_k = 10 log10(tt_k / (mp + eps)) >= threshold,  stab_k = 1e-3 (active_k ? tt_k : mp),
//     nom_k = tt_k + eps,  den_ik = ||e_i - t_k||^2 + stab_k + eps = ee_i - 2 <e_i, t_k> + tt_k + stab_k + eps,
//     score(p) = num_active * sum_k 10 a_k log10(nom_k / den_{p[k] k} + eps)                    (:86-109)
// best over itertools.permutations(range(S)) by torch.max's rule.  For the backward, coef[b] holds per estimate row
// i = p*[k]: dscore/d den * 2 = -20 a_k num_active / ln10 * nom_k / (den^2 (nom_k / den + eps)), the target k it
// is matched to, and the row means of estimates and targets (zero under !zero_mean):  [coef S][k S][me S][mt S].
// ---------------------------------------------------------------------------
template <int S>
__global__ void __launch_bounds__(256)
snr_zero_refs_finalize_kernel(const double* __restrict__ part, int chunks, float* __restrict__ value,
                              int* __restrict__ perm, double* __restrict__ coef, int B, long long T, int zero_mean,
                              double threshold, double eps) {
    for (long long b = blockIdx.x * 256LL + threadIdx.x; b < B; b += (long long)gridDim.x * 256) {
        const GramSums<GramLayout<S, S, true, false>> g(part, chunks, b, T, zero_mean);
        double mp = 0.0;                                    // the raw entries, the diagonal unclamped
#pragma unroll
        for (int j = 0; j < S; ++j)
#pragma unroll
            for (int k = 0; k < S; ++k) mp += g.tt(j, k);
        mp = clamp_energy(mp);
        double tt[S], act[S], nom[S], stab[S];
        int num_active = 0;
#pragma unroll
        for (int k = 0; k < S; ++k) {
            tt[k] = g.td(k);
            const bool on = 10.0 * log10(tt[k] / (mp + eps)) >= threshold;        // NaN: inactive, as Tensor.ge
            act[k] = on ? 1.0 : 0.0;
            num_active += on ? 1 : 0;
            nom[k] = tt[k] + eps;
            stab[k] = 1e-3 * (on ? tt[k] : mp);
        }
        double den[S][S], sc[S][S];
#pragma unroll
        for (int i = 0; i < S; ++i) {
            const double ee = g.ee(i);
#pragma unroll
            for (int k = 0; k < S; ++k) {
                double err = ee - 2.0 * g.et(i, k) + tt[k];
                if (isinf(ee) && isfinite(tt[k])) err = ee;              // ||e - t||^2 with an inf in e: inf - inf above
                err = clamp_energy(err);
                den[i][k] = err + stab[k] + eps;
                sc[i][k] = 10.0 * act[k] * log10(nom[k] / den[i][k] + eps);
            }
        }
        int besti, bp[S];
        value[b] = (float)best_assignment<S, S>([&](const int* q) {
            double m = 0.0;
            for (int k = 0; k < S; ++k) m = __dadd_rn(m, sc[q[k]][k]);
            return m * (double)num_active;
        }, besti, bp);
        perm[b] = besti;
        double* cb = coef + (size_t)b * 4 * S;
        for (int k = 0; k < S; ++k) {
            double d = 0.0, nk = 0.0, ak = 0.0;
#pragma unroll
            for (int i = 0; i < S; ++i) if (bp[k] == i) d = den[i][k];
#pragma unroll
            for (int j = 0; j < S; ++j) if (j == k) { nk = nom[j]; ak = act[j]; }
            const int i = bp[k];
            cb[i] = -20.0 * ak * (double)num_active / 2.302585092994045684 * nk / (d * d * (nk / d + eps));
            cb[S + i] = (double)k;
        }
#pragma unroll
        for (int i = 0; i < S; ++i) { cb[2 * S + i] = g.me[i]; cb[3 * S + i] = g.mt[i]; }
    }
}

// grad[b][i][t] = g[b] coef_i ((e_i - me_i) - (t_k - mt_k)) for t < T, 0 for T <= t < Tg (rows Tg apart); est and tgt
// rows are T apart.  grid row_tiled_grid(B S, Tg).
__global__ void __launch_bounds__(256)
snr_zero_refs_backward_kernel(const float* __restrict__ est, const float* __restrict__ tgt,
                              const double* __restrict__ coef, const float* __restrict__ grad_value,
                              float* __restrict__ grad, int B, int S, long long T, long long Tg) {
    const long long rows = (long long)B * S;
    for (long long row = blockIdx.y; row < rows; row += gridDim.y) {
        const long long b = row / S;
        const int i = (int)(row - b * S);
        const double* cb = coef + (size_t)b * 4 * S;
        const int k = (int)cb[S + i];
        const double c = cb[i] * (double)__ldg(grad_value + b);
        const double mi = cb[2 * S + i], mk = cb[3 * S + k];
        const float* er = est + (size_t)row * T;
        const float* tr = tgt + ((size_t)b * S + k) * T;
        float* gr = grad + (size_t)row * Tg;
        for (long long t = (long long)blockIdx.x * 256 + threadIdx.x; t < Tg; t += (long long)gridDim.x * 256)
            gr[t] = t < T ? (float)(c * (((double)__ldg(er + t) - mi) - ((double)__ldg(tr + t) - mk))) : 0.f;
    }
}

}  // namespace sdr

using namespace sdr;

#pragma GCC visibility push(default)
extern "C" {

size_t sdr_pit_sisdr_scratch_bytes(int B, int S) {
    if (B <= 0 || S < 1 || S > 4) return 0;
    const int V = 2 * S + 1;
    return sizeof(double) * (size_t)B * (V + S * S + 3 * S + 1);
}

int sdr_pit_sisdr(const float* est, const float* tgt, const float* mix, float* best, int32_t* perm, int B, int S,
                  int64_t T, int zero_mean, int improvement, double eps, void* scratch, sdr_stream stream) {
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!est || !tgt || !best || !perm || !scratch || reinterpret_cast<uintptr_t>(scratch) % 8 || B <= 0 || T <= 0)
        return SDR_ERR_BAD_ARGUMENT;
    if (improvement && !mix) return SDR_ERR_BAD_ARGUMENT;
    double* acc = static_cast<double*>(scratch);
    return with_sources(S, [&](auto s) {
        constexpr int n = decltype(s)::value;
        if (const int e = launch_gram<GramLayout<n, n, false, true>, false>(est, tgt, mix, n, B, T, acc, st)) return e;
        return launch(pit_finalize_kernel<n>, 1, 256, 0, st, acc, best, perm, B, T, zero_mean, improvement, eps);
    });
}

int sdr_pairwise_neg_sdr(const float* est, const float* tgt, float* out, int B, int S, int64_t T, int sdr_type,
                         int zero_mean, int take_log, void* scratch, sdr_stream stream) {
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!est || !tgt || !out || !scratch || reinterpret_cast<uintptr_t>(scratch) % 8 || B <= 0 || T <= 0 ||
        sdr_type < 0 || sdr_type > 2)
        return SDR_ERR_BAD_ARGUMENT;
    double* acc = static_cast<double*>(scratch);
    return with_sources(S, [&](auto s) {
        constexpr int n = decltype(s)::value;
        if (const int e = launch_gram<GramLayout<n, n, false, false>, false>(est, tgt, nullptr, n, B, T, acc, st))
            return e;
        return launch(pairwise_finalize_kernel<n, false>, item_blocks(B), 256, 0, st, acc, 1, out, nullptr, B, T,
                      sdr_type, zero_mean, take_log);
    });
}

size_t sdr_pairwise_neg_sdr_train_scratch_bytes(int B, int S, int64_t T) {
    return sdr_snr_zero_refs_scratch_bytes(B, S, T);
}

size_t sdr_pairwise_neg_sdr_coef_bytes(int B, int S) {
    if (B <= 0 || S < 1 || S > 4) return 0;
    return sizeof(double) * (size_t)B * (3 * S * S + 2 * S);
}

int sdr_pairwise_neg_sdr_train(const float* est, const float* tgt, float* out, void* coef, int B, int S, int64_t T,
                               int sdr_type, int zero_mean, int take_log, void* scratch, sdr_stream stream) {
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!est || !tgt || !out || !coef || !scratch || reinterpret_cast<uintptr_t>(scratch) % 8 ||
        reinterpret_cast<uintptr_t>(coef) % 8 || B <= 0 || T <= 0 || sdr_type < 0 || sdr_type > 2)
        return SDR_ERR_BAD_ARGUMENT;
    double* part = static_cast<double*>(scratch);
    return with_sources(S, [&](auto s) {
        constexpr int n = decltype(s)::value;
        if (const int e = launch_gram<GramLayout<n, n, true, false>, true>(est, tgt, nullptr, n, B, T, part, st))
            return e;
        return launch(pairwise_finalize_kernel<n, true>, item_blocks(B), 256, 0, st, part, gram_chunks(T), out,
                      static_cast<double*>(coef), B, T, sdr_type, zero_mean, take_log);
    });
}

int sdr_pairwise_neg_sdr_backward(const float* est, const float* tgt, const void* coef, const float* grad_out,
                                  float* grad, int B, int S, int64_t T, sdr_stream stream) {
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!est || !tgt || !coef || reinterpret_cast<uintptr_t>(coef) % 8 || !grad_out || !grad || B <= 0 || T <= 0)
        return SDR_ERR_BAD_ARGUMENT;
    return with_sources(S, [&](auto s) {
        constexpr int n = decltype(s)::value;
        return launch(pairwise_backward_kernel<n>, row_tiled_grid((long long)B * n, T), 256, 0, st, est, tgt,
                      static_cast<const double*>(coef), grad_out, grad, B, T);
    });
}

size_t sdr_stabilized_sisdr_scratch_bytes(int B, int n_est, int n_act) {
    if (B <= 0 || n_est < 1 || n_est > 4 || n_act < 1 || n_act > n_est) return 0;
    return sizeof(double) * (size_t)B * (n_est + n_act + n_est * n_act + n_est + n_act * n_act);
}

int sdr_stabilized_sisdr(const float* est, const float* tgt, float* best, int32_t* perm, int B, int rows, int n_est,
                         int n_act, int64_t T, int zero_mean, int improvement, double eps, void* scratch,
                         sdr_stream stream) {
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!est || !tgt || !best || !perm || !scratch || reinterpret_cast<uintptr_t>(scratch) % 8 || B <= 0 || T <= 0 ||
        rows < 1)
        return SDR_ERR_BAD_ARGUMENT;
    if (rows != n_est && n_est != 1) return SDR_ERR_BAD_ARGUMENT;          // summing the rows is the single_source mode
    if (!sdr_stabilized_sisdr_scratch_bytes(B, n_est, n_act)) return SDR_ERR_UNSUPPORTED;
    double* acc = static_cast<double*>(scratch);
    return with_sources(n_est, [&](auto se) {
        return with_sources(n_act, [&](auto sa) -> int {
            constexpr int E = decltype(se)::value, A = decltype(sa)::value;
            if constexpr (A > E) {
                return SDR_ERR_UNSUPPORTED;
            } else {
                if (const int e = launch_gram<GramLayout<E, A, true, false>, false>(est, tgt, nullptr, rows, B, T,
                                                                                   acc, st))
                    return e;
                return launch(stab_finalize_kernel<E, A>, 1, 256, 0, st, acc, best, perm, B, T, zero_mean, improvement,
                              eps);
            }
        });
    });
}

size_t sdr_snr_zero_refs_scratch_bytes(int B, int S, int64_t T) {
    if (B <= 0 || S < 1 || S > 4 || T <= 0) return 0;
    return sizeof(double) * (size_t)B * gram_chunks(T) * (2 * S + 2 * S * S + S);
}

size_t sdr_snr_zero_refs_coef_bytes(int B, int S) {
    if (B <= 0 || S < 1 || S > 4) return 0;
    return sizeof(double) * (size_t)B * 4 * S;
}

int sdr_snr_zero_refs(const float* est, const float* tgt, float* value, int32_t* perm, void* coef, int B, int S,
                      int64_t T, int zero_mean, double threshold, double eps, void* scratch, sdr_stream stream) {
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!est || !tgt || !value || !perm || !coef || !scratch || reinterpret_cast<uintptr_t>(scratch) % 8 ||
        reinterpret_cast<uintptr_t>(coef) % 8 || B <= 0 || T <= 0)
        return SDR_ERR_BAD_ARGUMENT;
    double* part = static_cast<double*>(scratch);
    return with_sources(S, [&](auto s) {
        constexpr int n = decltype(s)::value;
        if (const int e = launch_gram<GramLayout<n, n, true, false>, true>(est, tgt, nullptr, n, B, T, part, st))
            return e;
        return launch(snr_zero_refs_finalize_kernel<n>, item_blocks(B), 256, 0, st, part, gram_chunks(T), value, perm,
                      static_cast<double*>(coef), B, T, zero_mean, threshold, eps);
    });
}

int sdr_snr_zero_refs_backward(const float* est, const float* tgt, const void* coef, const float* grad_value,
                               float* grad, int B, int S, int64_t T, int64_t Tg, sdr_stream stream) {
    if (!est || !tgt || !coef || reinterpret_cast<uintptr_t>(coef) % 8 || !grad_value || !grad || B <= 0 || T <= 0 ||
        Tg < T)
        return SDR_ERR_BAD_ARGUMENT;
    if (S < 1 || S > 4) return SDR_ERR_UNSUPPORTED;
    return launch(snr_zero_refs_backward_kernel, row_tiled_grid((long long)B * S, Tg), 256, 0,
                  static_cast<cudaStream_t>(stream), est, tgt, static_cast<const double*>(coef), grad_value, grad, B,
                  S, T, Tg);
}

}  // extern "C"
#pragma GCC visibility pop
