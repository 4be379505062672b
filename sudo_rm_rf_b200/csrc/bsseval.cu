// BSS-eval v3 source criteria (mir_eval.separation.bss_eval_sources, the `sdr`, `sir` and `sar` of asteroid's
// get_metrics that the reference's evaluation scripts report).  Per item, with references s_1..s_S, an estimate e and
// F-tap distortion filters, in R^(T+F-1):
//     P_j e   = projection of e onto span{s_j[t - l], l < F},  P_all e = projection onto all S F delayed references
//     SDR = 10 log10(|P_j e|^2 / |e - P_j e|^2),  SIR = 10 log10(|P_j e|^2 / |P_all e - P_j e|^2),
//     SAR = 10 log10(|P_all e|^2 / |e - P_all e|^2)
// for every (estimate, reference) pair, then the assignment of estimates to references with the largest mean SIR.
// Four kernels:
//   bss_corr_kernel    lagged fp64 correlations  X_ar[k] = sum_t a[t] r[t + k], k < F, of every reference row a with
//                      every row r (references, estimates, mixture): the normal equations' block-Toeplitz matrix
//                      (r a reference) and right-hand sides (r an estimate).  Per-chunk partials, no atomics.
//   bss_solve_kernel   one CTA per (item, system): the joint system (S x S blocks) or one reference's own F x F
//                      Toeplitz system, each shared by every estimate, by block Levinson (Whittle-Wiggins-Robinson)
//                      with generalised inverses, so a rank-deficient reference set still gives the projection.
//   bss_energy_kernel  the projections as FIR filters of the references and the five energies of each estimate,
//                      formed from the filtered signals rather than as |e|^2 - c.D, which cancels at high SDR/SAR.
//   bss_final_kernel   the criteria, the permutation search (best_assignment on the mean SIR) and the outputs.
// The correlation and energy kernels read their items through a BssItems view: a whole [S, T] item of a contiguous
// batch (sdr_bss_eval) or one window of a recording, read in place (sdr_bss_eval_framewise).
//
// Source images (mir_eval.separation.bss_eval_images, sdr_bss_eval_images): source j is an image s_j of C channel rows
// and so is estimate i, R = S C rows each.  P_j projects each channel of e_i onto the F delays of all C rows of s_j,
// P_all onto all R F delayed rows, and energies sum over channels:
//     SDR = 10 log10(|s_j|^2 / |e_i - s_j|^2),         ISR = 10 log10(|s_j|^2 / |P_j e_i - s_j|^2),
//     SIR = 10 log10(|P_j e_i|^2 / |P_all e_i - P_j e_i|^2),  SAR = 10 log10(|P_all e_i|^2 / |e_i - P_all e_i|^2)
// The same four kernels with the reference rows grouped by source (template parameter C): the joint system has R
// blocks and source j's own system its C rows.  The sources are the instance C = 1 without the images' two extra
// energies, and compute what they computed before images existed.
//
// BSS-eval v4 (museval's, sdr_bss_eval_v4): the image criteria with the filters solved once per recording, from the
// correlations of its whole length (bss_corr_kernel in fixed track chunks, bss_fold_kernel adding them in chunk order),
// tested by bss_track_check_kernel, and applied to each window's reference slice by bss_energy_kernel.
#include <type_traits>

#include "assign.cuh"
#include "launchers.cuh"

namespace sdr {

constexpr int kBssCorrTile = 512;       // samples staged per correlation step; one thread per lag, so F <= 512
constexpr int kBssEnergyTile = 256;     // output samples per energy step, one per thread
constexpr int kBssMaxF = 512;
// A prediction-error pivot at or below this (the references scaled to unit energy) marks a delayed reference that the
// earlier ones already span: its generalised inverse drops it.  Exact dependences (equal, scaled or delayed copies)
// leave pivots of rounding size, ~1e-14 after 512 steps.
constexpr double kBssPivotTol = 1e-10;
// Framewise scoring runs its windows through one scratch in launches of at most this many items, so the scratch does
// not grow with the recording (a window's scratch is at most 16 correlation chunks: 2.6 MB at S = 4, F = 512).
constexpr long long kBssFramewiseItems = 128;

__host__ __device__ inline int bss_corr_chunks(long long T) {
    const long long c = (T + 4095) / 4096;
    return (int)(c < 1 ? 1 : (c > 16 ? 16 : c));
}
__host__ __device__ inline int bss_energy_chunks(long long T, int F) { return bss_corr_chunks(T + F - 1); }

// A row can be scored when its energy is positive and finite: an all-zero row, or one holding a NaN or an infinity
// (whose energy is NaN or inf), gives its item NaN and perm -1 rather than a NaN score and an arbitrary assignment.
__device__ __forceinline__ bool bss_scorable(double energy) { return energy > 0.0 && energy < (double)INFINITY; }

// An orthogonal projection p of e leaves a residual orthogonal to it: |p|^2 + |e - p|^2 = |e|^2.  The recursion on the
// normal equations loses that when the delays are nearly, but not numerically, dependent (several band-limited
// references with deep stop bands: G's condition number near 1 / eps, and the prediction-error matrices lose
// definiteness).  Its scores are then those of no projection, so the item is reported NaN.  Where the recursion
// holds, the defect stays below 1e-3 of |e|^2 (a few 1e-4 next to dropped delays, rounding elsewhere).
constexpr double kBssProjectionDefect = 1e-2;
__device__ __forceinline__ bool bss_is_projection(double p2, double r2, double e2) {
    return fabs(p2 + r2 - e2) <= kBssProjectionDefect * e2;
}

// Energies per estimate row (bss_energy_kernel's layout): 3 S + 3, 2 S more for source images, and S more for v4
__host__ __device__ constexpr int bss_energy_count(int S, bool images, bool v4 = false) {
    return 3 * S + 3 + (images ? 2 * S : 0) + (v4 ? S : 0);
}

// Estimate row e's energies come from projections: the joint one and every own one.
template <int S, int NV>
__device__ __forceinline__ bool bss_projections_hold(const double (&en)[NV]) {
    bool ok = bss_is_projection(en[3 * S], en[3 * S + 1], en[3 * S + 2]);
#pragma unroll
    for (int j = 0; j < S; ++j) ok = ok && bss_is_projection(en[j], en[S + j], en[3 * S + 2]);
    return ok;
}

// Scratch carve-up for R = S C reference rows, sized for R estimate rows plus the mixture's whether or not it is
// given, and NV energies per estimate row.  Doubles:
//   part  [B][chunks][R][2R+1][F]   correlation partials (rows: R references, then the NE estimate rows)
//   rj    [B][F][R][R]              the joint system's normalised blocks
//   rt    [B][S][F][C][C]           each source's own normalised blocks
//   eref  [B][R]                    reference row energies
//   cj    [B][R+1][R][F]            joint filters per estimate row
//   ct    [B][R+1][R][F]            own-source filters per estimate row
//   epart [B][echunks][R+1][NV]     energy partials
struct BssScratch {
    double *part, *rj, *rt, *eref, *cj, *ct, *epart;
    size_t bytes;
    BssScratch(void* base, int B, int S, int C, long long T, int F, int NV) {
        const size_t b = (size_t)B, s = (size_t)S, c = (size_t)C, r = s * c, f = (size_t)F, ne = r + 1;
        size_t off = 0;
        double* p = static_cast<double*>(base);
        auto take = [&](size_t n) { double* q = p ? p + off : nullptr; off += n; return q; };
        part = take(b * bss_corr_chunks(T) * r * (r + ne) * f);
        rj = take(b * f * r * r);
        rt = take(b * s * f * c * c);
        eref = take(b * r);
        cj = take(b * ne * r * f);
        ct = take(b * ne * r * f);
        epart = take(b * bss_energy_chunks(T, F) * ne * (size_t)NV);
        bytes = off * sizeof(double);
    }
};

// Row r of item b, S reference rows per item: references 0..S-1, estimates S..2S-1, the mixture 2S.  Source images
// pass S = R: reference row j C + c is channel c of image j.
__device__ __forceinline__ const float* bss_row(const float* ref, const float* est, const float* mix, int S,
                                                long long b, int r, long long T) {
    if (r < S) return ref + ((size_t)b * S + r) * T;
    if (r < 2 * S) return est + ((size_t)b * S + (r - S)) * T;
    return mix + (size_t)b * T;
}

// The items of a launch as views of the inputs, whose rows are T samples apart.  Item i is window k = (first + i) %
// nwin of recording b = (first + i) / nwin, which is n = lengths[b] samples long (T without lengths).  The recording
// has (n - W + H) / H windows, window k covering [k H, k H + W), when that is at least 2 (n >= W + H); otherwise it
// is one item, the whole recording (mir_eval's fallback).  A column past the recording's windows, a length outside
// [1, T] and a fallback shorter than min_len get length 0: nothing is read, the reference energies are zero and the
// item is reported NaN with perm -1.  sdr_bss_eval's items are the view W = H = T, nwin = 1, where every recording
// falls back: item b is the whole of recording b.
struct BssItems {
    long long T, W, H, nwin, first, min_len;
    const long long* lengths;
    // -> the item's first sample within its recording's rows; b its recording, len its length
    __device__ __forceinline__ long long span(long long i, long long& b, long long& len) const {
        const long long g = first + i;
        b = g / nwin;
        const long long k = g - b * nwin;
        const long long n = lengths ? lengths[b] : T;
        len = 0;
        if (n < 1 || n > T) return 0;
        if (n - W < H) {
            if (k == 0 && n >= min_len) len = n;
            return 0;
        }
        if (k < (n - W) / H + 1) len = W;
        return k * H;
    }
    // BSS-eval v4's windows (museval): (n - W) / H + 1 of them when n >= W and none otherwise, with no whole-recording
    // fallback; a recording shorter than min_len has none either.
    __device__ __forceinline__ long long window(long long i, long long& b, long long& len) const {
        const long long g = first + i;
        b = g / nwin;
        const long long k = g - b * nwin;
        const long long n = lengths ? lengths[b] : T;
        len = 0;
        if (n < W || n < min_len || n > T) return 0;
        if (k < (n - W) / H + 1) len = W;
        return k * H;
    }
};

// The correlation kernel's chunk policy is the type of its last argument.  An int (the item entries): `chunks` per
// item in the launch, the item cut into its own bss_corr_chunks(length) chunks, so its partials are those of the item
// scored alone; the launch's chunks past them are written as zeros, which leave the reader's chunk-order sums unchanged.
__device__ __forceinline__ int bss_chunk_count(int chunks) { return chunks; }
__device__ __forceinline__ void bss_chunk_range(int, long long T, int chunk, long long& t0, long long& t1) {
    const int own = bss_corr_chunks(T);
    const long long per = (T + own - 1) / own;
    t0 = chunk < own ? (long long)chunk * per : T;
    t1 = t0 + per < T ? t0 + per : T;
}

// BSS-eval v4's whole-recording correlations: chunks of kBssTrackChunk samples at fixed positions in the recording, a
// launch taking chunks [c0, c0 + n) of every recording.  Each chunk's partials also hold the estimate rows' energies
// |e|^2 over the chunk, after its correlations.  bss_fold_kernel adds them in chunk order, so a recording's sums depend
// on its own length only: not on the batch, nor on how many chunks a launch takes.
constexpr long long kBssTrackChunk = 8192;
struct BssTrackChunks {
    int n;
    long long c0;
};
__device__ __forceinline__ int bss_chunk_count(const BssTrackChunks& c) { return c.n; }
__device__ __forceinline__ void bss_chunk_range(const BssTrackChunks& c, long long T, int chunk, long long& t0,
                                                long long& t1) {
    const long long s = (c.c0 + chunk) * kBssTrackChunk;
    t0 = s < T ? s : T;
    t1 = t0 + kBssTrackChunk < T ? t0 + kBssTrackChunk : T;
}
// Doubles per chunk partial: the correlations of S reference rows with NB rows, and for v4 the NE estimate energies
__host__ __device__ constexpr size_t bss_partial_size(int S, int NE, int F, bool track) {
    return (size_t)S * (S + NE) * F + (track ? NE : 0);
}

// grid = items * chunks, kBssCorrTile threads; smem [NB][kBssCorrTile + F - 1] doubles.  S counts reference rows (R
// for source images).
template <int S, int NE, class Chunks>
__global__ void __launch_bounds__(kBssCorrTile)
bss_corr_kernel(const float* __restrict__ ref, const float* __restrict__ est, const float* __restrict__ mix,
                double* __restrict__ part, BssItems items, int F, Chunks chunks) {
    constexpr int NB = S + NE;
    constexpr bool kTrack = std::is_same<Chunks, BssTrackChunks>::value;
    extern __shared__ double sm[];
    const int nc = bss_chunk_count(chunks);
    const long long it = blockIdx.x / nc;
    const int chunk = (int)(blockIdx.x - it * nc);
    long long b, T;
    const long long off = items.span(it, b, T);
    long long t0, t1;
    bss_chunk_range(chunks, T, chunk, t0, t1);
    const int W = kBssCorrTile + F - 1;
    double ee[kTrack ? NE : 1];
#pragma unroll
    for (int e = 0; e < (kTrack ? NE : 1); ++e) ee[e] = 0.0;
    const int k = threadIdx.x;
    double acc[S][NB];
#pragma unroll
    for (int i = 0; i < S; ++i)
#pragma unroll
        for (int r = 0; r < NB; ++r) acc[i][r] = 0.0;
    for (long long tt = t0; tt < t1; tt += kBssCorrTile) {
        const int n = (int)(t1 - tt < kBssCorrTile ? t1 - tt : kBssCorrTile);
        __syncthreads();
        for (int idx = threadIdx.x; idx < NB * W; idx += kBssCorrTile) {
            const int r = idx / W, q = idx - r * W;
            const long long t = tt + q;               // the halo reaches into the next chunk: zero only past T
            sm[idx] = (q < n + F - 1 && t < T) ? (double)__ldg(bss_row(ref, est, mix, S, b, r, items.T) + off + t)
                                               : 0.0;
        }
        __syncthreads();
        if (k < F) {
            for (int q = 0; q < n; ++q) {
                double a[S], v[NB];
#pragma unroll
                for (int i = 0; i < S; ++i) a[i] = sm[i * W + q];
#pragma unroll
                for (int r = 0; r < NB; ++r) v[r] = sm[r * W + q + k];
#pragma unroll
                for (int i = 0; i < S; ++i)
#pragma unroll
                    for (int r = 0; r < NB; ++r) acc[i][r] = fma(a[i], v[r], acc[i][r]);
            }
        }
        if constexpr (kTrack) {                       // sample q of the tile: one per thread
            if (k < n) {
#pragma unroll
                for (int e = 0; e < NE; ++e) {
                    const double v = sm[(S + e) * W + k];
                    ee[e] = fma(v, v, ee[e]);
                }
            }
        }
    }
    double* const pc = kTrack ? part + ((size_t)it * nc + chunk) * bss_partial_size(S, NE, F, true)
                              : part + ((size_t)it * nc + chunk) * S * NB * F;
    if (k < F) {
#pragma unroll
        for (int i = 0; i < S; ++i)
#pragma unroll
            for (int r = 0; r < NB; ++r) pc[((size_t)i * NB + r) * F + k] = acc[i][r];
    }
    if constexpr (kTrack) {                           // the energies, reduced in a fixed order
        __shared__ double red[kBssCorrTile / 32][NE];
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
        for (int e = 0; e < NE; ++e) {
            const double s = warp_sum_f64(ee[e]);
            if (lane == 0) red[warp][e] = s;
        }
        __syncthreads();
        if (threadIdx.x < NE) {
            double s = 0.0;
            for (int w = 0; w < kBssCorrTile / 32; ++w) s += red[w][threadIdx.x];
            pc[(size_t)S * NB * F + threadIdx.x] = s;
        }
    }
}

// v4: adds a launch's chunk partials (n per recording, the chunks from c0 on) to each recording's running totals,
// correlations tot [B][csize] and estimate energies etot [B][NE], in chunk order, starting from zero at c0 = 0.  Chunks past a recording's length are skipped, so
// its totals are the same whatever the batch.  One thread per (recording, double of the partial).
__global__ void __launch_bounds__(256)
bss_fold_kernel(const double* __restrict__ part, double* __restrict__ tot, double* __restrict__ etot, BssItems items,
                int B, long long csize, int NE, BssTrackChunks chunks) {
    const long long size = csize + NE;
    const long long idx = blockIdx.x * 256LL + threadIdx.x;
    if (idx >= B * size) return;
    const long long b = idx / size, i = idx - b * size;
    long long rb, len;
    items.span(b, rb, len);
    double* dst = i < csize ? tot + b * csize + i : etot + b * NE + (i - csize);
    double s = chunks.c0 == 0 ? 0.0 : *dst;
    for (int c = 0; c < chunks.n; ++c)
        if ((chunks.c0 + c) * kBssTrackChunk < len) s += part[((size_t)b * chunks.n + c) * size + i];
    *dst = s;
}

// One item's lagged correlations X_ar[k], its chunk partials added in chunk order.
template <int S, int NB> struct BssCorr {
    const double* p;
    int chunks, F;
    __device__ __forceinline__ double operator()(int a, int r, int k) const {
        double v = 0.0;
        for (int c = 0; c < chunks; ++c) v += p[(((size_t)c * S + a) * NB + r) * F + k];
        return v;
    }
};

// Generalised inverse of a symmetric positive semi-definite M x M matrix by the sweep operator: pivots at or below
// kBssPivotTol are not swept and their rows and columns of the result are zero, so P G P = P whenever the dropped
// pivots are (numerically) zero Schur complements.
template <int M>
__device__ void bss_ginv(const double (&P)[M][M], double (&G)[M][M]) {
    double W[M][M];
    bool kept[M];
#pragma unroll
    for (int i = 0; i < M; ++i)
#pragma unroll
        for (int j = 0; j < M; ++j) W[i][j] = P[i][j];
#pragma unroll
    for (int p = 0; p < M; ++p) {
        const double d = W[p][p];
        kept[p] = d > kBssPivotTol;
        if (!kept[p]) continue;
#pragma unroll
        for (int i = 0; i < M; ++i)
#pragma unroll
            for (int j = 0; j < M; ++j)
                if (i != p && j != p) W[i][j] -= W[i][p] * W[p][j] / d;
#pragma unroll
        for (int i = 0; i < M; ++i)
            if (i != p) { W[i][p] /= d; W[p][i] /= d; }
        W[p][p] = -1.0 / d;
    }
#pragma unroll
    for (int i = 0; i < M; ++i)
#pragma unroll
        for (int j = 0; j < M; ++j) G[i][j] = kept[i] && kept[j] ? -W[i][j] : 0.0;
}

// Block Levinson for G c_e = D_e, e < NE, where G[(r,l),(q,m)] = R_{l-m}[r][q], R_k[r][q] = X_{ch r, ch q}[k] (and
// R_{-k} = R_k^T), D_e[(r,l)] = X_{ch r, estimate e}[l], over the M reference channels ch[].  The system is solved
// in unit-energy coordinates (row and column r scaled by 1/sqrt(E_ch r)).  Forward predictors A, backward predictors
// kept reversed (Brev_n[m] = B_n[n - m], so that the thread owning lag k reads and writes A[k] and Brev[n + 1 - k]
// only) and the solutions x_e grow by one lag per step; the step's two inner products are block reductions in a fixed
// order and its M x M algebra runs on thread 0.  Writes coef[e][ch r][l] = c_e[(r, l)].
template <int M, int NE, int S, int NB>
__device__ void bss_levinson(const BssCorr<S, NB>& cr, const int (&ch)[M], const double* sE, double* Rg,
                             double* coef, int F, double* smem) {
    constexpr int MM = M * M, NV = MM + NE * M;
    __shared__ double red[8][NV];
    __shared__ double sKf[MM], sKb[MM], sg[NE * M], srhs[NE * M];
    // A zero-energy channel of a non-silent source image is dropped, not normalised: its rows and columns of the
    // system are zero, so every pivot of it is dropped, and its filters are zero (mir_eval's lstsq fallback).
    double inv[M];
#pragma unroll
    for (int r = 0; r < M; ++r) inv[r] = sE[ch[r]] > 0.0 ? 1.0 / sqrt(sE[ch[r]]) : 0.0;
    for (int idx = threadIdx.x; idx < F * MM; idx += blockDim.x) {
        const int k = idx / MM, r = (idx / M) % M, q = idx % M;
        Rg[idx] = cr(ch[r], ch[q], k) * inv[r] * inv[q];
    }
    double* A = smem;
    double* Br = A + (size_t)F * MM;
    double* x = Br + (size_t)F * MM;
    for (int idx = threadIdx.x; idx < F * MM; idx += blockDim.x) {
        const int r = (idx / M) % M, q = idx % M;
        A[idx] = idx < MM && r == q ? 1.0 : 0.0;
        Br[idx] = A[idx];
    }
    for (int idx = threadIdx.x; idx < F * NE * M; idx += blockDim.x) x[idx] = 0.0;
    if (threadIdx.x < NE * M) {
        const int e = threadIdx.x / M, r = threadIdx.x % M;
        srhs[threadIdx.x] = cr(ch[r], S + e, 0) * inv[r];
    }
    __syncthreads();                                    // Rg (global, written by this CTA) and the smem state
    double Pf[M][M], Pb[M][M], Pbi[M][M];               // thread 0's
    if (threadIdx.x == 0) {
#pragma unroll
        for (int r = 0; r < M; ++r)
#pragma unroll
            for (int q = 0; q < M; ++q) Pf[r][q] = Pb[r][q] = Rg[r * M + q];
        bss_ginv<M>(Pb, Pbi);
        for (int e = 0; e < NE; ++e)
#pragma unroll
            for (int r = 0; r < M; ++r) {
                double v = 0.0;
#pragma unroll
                for (int q = 0; q < M; ++q) v += Pbi[r][q] * srhs[e * M + q];
                x[e * M + r] = v;
            }
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int n = 0; n + 1 < F; ++n) {
        // Delta = sum_k R_{n+1-k} A[k],  eps_e = sum_k R_{n+1-k} x_e[k]
        double v[NV];
#pragma unroll
        for (int i = 0; i < NV; ++i) v[i] = 0.0;
        for (int k = threadIdx.x; k <= n; k += blockDim.x) {
            const double* R = Rg + (size_t)(n + 1 - k) * MM;
            double Rl[MM];
#pragma unroll
            for (int i = 0; i < MM; ++i) Rl[i] = R[i];
            const double* a = A + (size_t)k * MM;
            const double* xk = x + (size_t)k * NE * M;
#pragma unroll
            for (int r = 0; r < M; ++r)
#pragma unroll
                for (int q = 0; q < M; ++q) {
#pragma unroll
                    for (int c = 0; c < M; ++c) v[r * M + c] = fma(Rl[r * M + q], a[q * M + c], v[r * M + c]);
#pragma unroll
                    for (int e = 0; e < NE; ++e) v[MM + e * M + r] = fma(Rl[r * M + q], xk[e * M + q], v[MM + e * M + r]);
                }
        }
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const double s = warp_sum_f64(v[i]);
            if (lane == 0) red[warp][i] = s;
        }
        if (threadIdx.x < NE * M) {
            const int e = threadIdx.x / M, r = threadIdx.x % M;
            srhs[threadIdx.x] = cr(ch[r], S + e, n + 1) * inv[r];
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            double D[M][M], Pfi[M][M], Kf[M][M], Kb[M][M], eps[NE * M];
#pragma unroll
            for (int i = 0; i < NV; ++i) {
                double s = 0.0;
                for (int w = 0; w < nwarps; ++w) s += red[w][i];
                if (i < MM) D[i / M][i % M] = s;
                else eps[i - MM] = s;
            }
            bss_ginv<M>(Pf, Pfi);
#pragma unroll
            for (int r = 0; r < M; ++r)
#pragma unroll
                for (int c = 0; c < M; ++c) {
                    double f = 0.0, g = 0.0;
#pragma unroll
                    for (int q = 0; q < M; ++q) {
                        f += Pbi[r][q] * D[q][c];               // Kf = Pb^- Delta
                        g += Pfi[r][q] * D[c][q];               // Kb = Pf^- Delta^T
                    }
                    Kf[r][c] = f;
                    Kb[r][c] = g;
                }
            double nPf[M][M], nPb[M][M];
#pragma unroll
            for (int r = 0; r < M; ++r)
#pragma unroll
                for (int c = 0; c < M; ++c) {
                    double f = Pf[r][c], g = Pb[r][c];
#pragma unroll
                    for (int q = 0; q < M; ++q) {
                        f -= D[q][r] * Kf[q][c];                // Pf - Delta^T Kf
                        g -= D[r][q] * Kb[q][c];                // Pb - Delta Kb
                    }
                    nPf[r][c] = f;
                    nPb[r][c] = g;
                }
#pragma unroll
            for (int r = 0; r < M; ++r)
#pragma unroll
                for (int c = 0; c < M; ++c) {
                    Pf[r][c] = 0.5 * (nPf[r][c] + nPf[c][r]);
                    Pb[r][c] = 0.5 * (nPb[r][c] + nPb[c][r]);
                    sKf[r * M + c] = Kf[r][c];
                    sKb[r * M + c] = Kb[r][c];
                }
            bss_ginv<M>(Pb, Pbi);
            for (int e = 0; e < NE; ++e)
#pragma unroll
                for (int r = 0; r < M; ++r) {
                    double g = 0.0;
#pragma unroll
                    for (int q = 0; q < M; ++q) g += Pbi[r][q] * (srhs[e * M + q] - eps[e * M + q]);
                    sg[e * M + r] = g;
                }
        }
        __syncthreads();
        // A[k] -= Brev[n+1-k] Kf,  Brev[n+1-k] -= A[k] Kb,  x_e[k] += B_{n+1}[k] g_e
        for (int k = threadIdx.x; k <= n + 1; k += blockDim.x) {
            double* a = A + (size_t)k * MM;
            double* br = Br + (size_t)(n + 1 - k) * MM;
            double ao[MM], bo[MM];
#pragma unroll
            for (int i = 0; i < MM; ++i) { ao[i] = a[i]; bo[i] = br[i]; }
#pragma unroll
            for (int r = 0; r < M; ++r)
#pragma unroll
                for (int c = 0; c < M; ++c) {
                    double na = ao[r * M + c], nb = bo[r * M + c];
#pragma unroll
                    for (int q = 0; q < M; ++q) {
                        na = fma(-bo[r * M + q], sKf[q * M + c], na);
                        nb = fma(-ao[r * M + q], sKb[q * M + c], nb);
                    }
                    a[r * M + c] = na;
                    br[r * M + c] = nb;
                }
            double* xk = x + (size_t)k * NE * M;
            for (int e = 0; e < NE; ++e)
#pragma unroll
                for (int r = 0; r < M; ++r) {
                    double s = xk[e * M + r];
#pragma unroll
                    for (int q = 0; q < M; ++q) s = fma(br[r * M + q], sg[e * M + q], s);
                    xk[e * M + r] = s;
                }
        }
        __syncthreads();
    }
    for (int idx = threadIdx.x; idx < NE * M * F; idx += blockDim.x) {
        const int e = idx / (M * F), r = (idx / F) % M, l = idx % F;
        coef[((size_t)e * S + ch[r]) * F + l] = x[((size_t)l * NE + e) * M + r] * inv[r];
    }
}

// Source j's energy, its C rows' summed in channel order (the row's own for C = 1)
template <int C>
__device__ __forceinline__ double bss_image_energy(const double* rows, int j) {
    double e = rows[j * C];
#pragma unroll
    for (int c = 1; c < C; ++c) e += rows[j * C + c];
    return e;
}

// grid = B (S + 1): system 0 of an item is the joint one over all R = S C reference rows, system 1 + j source j's own
// over its C rows.  256 threads.
template <int S, int NE, int C = 1>
__global__ void __launch_bounds__(256)
bss_solve_kernel(const double* __restrict__ part, int chunks, double* __restrict__ rj, double* __restrict__ rt,
                 double* __restrict__ eref, double* __restrict__ cj, double* __restrict__ ct, int F) {
    constexpr int R = S * C, NB = R + NE;
    extern __shared__ double smem[];
    __shared__ double sE[R];
    const long long b = blockIdx.x / (S + 1);
    const int sys = (int)(blockIdx.x - b * (S + 1));
    const BssCorr<R, NB> cr{part + (size_t)b * chunks * R * NB * F, chunks, F};
    if (threadIdx.x < R) sE[threadIdx.x] = cr(threadIdx.x, threadIdx.x, 0);
    __syncthreads();
    bool silent = false;
#pragma unroll
    for (int i = 0; i < S; ++i) silent = silent || !bss_scorable(bss_image_energy<C>(sE, i));
    if (sys == 0 && threadIdx.x < R) eref[(size_t)b * R + threadIdx.x] = sE[threadIdx.x];
    double* out = (sys == 0 ? cj : ct) + (size_t)b * (R + 1) * R * F;
    if (silent) {                                       // the item's outputs are NaN; its filters are set to zero
        for (int idx = threadIdx.x; idx < NE * R * F; idx += blockDim.x) {
            const int r = (idx / F) % R;
            if (sys == 0 || r / C == sys - 1) out[idx] = 0.0;
        }
        return;
    }
    if (sys == 0) {
        int ch[R];
#pragma unroll
        for (int i = 0; i < R; ++i) ch[i] = i;
        bss_levinson<R, NE>(cr, ch, sE, rj + (size_t)b * F * R * R, out, F, smem);
    } else {
        int ch[C];
#pragma unroll
        for (int c = 0; c < C; ++c) ch[c] = (sys - 1) * C + c;
        bss_levinson<C, NE>(cr, ch, sE, rt + ((size_t)b * S + sys - 1) * F * C * C, out, F, smem);
    }
}

// grid = items * echunks, kBssEnergyTile threads; smem: reference rows [R][kBssEnergyTile + F - 1], filters
// [2][R][F], R = S C.  Over t < T + F - 1 (T the item's length), estimate row e's projections pa = sum_r cj_e,r * s_r
// and pt_j = sum_c ct_e,jC+c * s_jC+c and the energies
//     [0, S)  |pt_j|^2,   [S, 2S)  |e - pt_j|^2,   [2S, 3S)  |pa - pt_j|^2,   3S |pa|^2,   3S+1 |e - pa|^2,   3S+2 |e|^2
// and for source images (IMG), with s_j the row of reference j in e's channel (e mod C):
//     [3S+3, 4S+3)  |pt_j - s_j|^2,   [4S+3, 5S+3)  |e - s_j|^2
// and for BSS-eval v4 (V4, with IMG), whose items are museval's windows (BssItems::window) filtered by their
// recording's whole-track filters (cj, ct indexed by recording), the window's own reference energies
//     [5S+3, 6S+3)  |s_j|^2
// Chunked as bss_corr_kernel: the item's own bss_energy_chunks, zero partials past them.
template <int S, int NE, int C = 1, bool IMG = false, bool V4 = false>
__global__ void __launch_bounds__(kBssEnergyTile)
bss_energy_kernel(const float* __restrict__ ref, const float* __restrict__ est, const float* __restrict__ mix,
                  const double* __restrict__ cj, const double* __restrict__ ct, double* __restrict__ epart,
                  BssItems items, int F, int chunks) {
    constexpr int R = S * C, NV = bss_energy_count(S, IMG, V4);
    static_assert(!V4 || IMG, "v4 scores source images");
    extern __shared__ double sm[];
    __shared__ double red[kBssEnergyTile / 32][NV];
    const int W = kBssEnergyTile + F - 1;
    double* sref = sm;                                  // [R][W]: s_r[tt - F + 1 + q]
    double* sj = sref + (size_t)R * W;                  // [R][F]
    double* st = sj + (size_t)R * F;                    // [R][F]
    const long long it = blockIdx.x / chunks;
    const int chunk = (int)(blockIdx.x - it * chunks);
    long long b, T;
    const long long off = V4 ? items.window(it, b, T) : items.span(it, b, T);
    const long long fi = V4 ? b : it;                   // whose filters
    const int own = bss_energy_chunks(T, F);
    const long long L = T + F - 1;
    const long long per = (L + own - 1) / own;
    const long long t0 = chunk < own ? (long long)chunk * per : L;
    const long long t1 = t0 + per < L ? t0 + per : L;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int e = 0; e < NE; ++e) {
        const float* er = bss_row(ref, est, mix, R, b, R + e, items.T) + off;
        __syncthreads();
        for (int idx = threadIdx.x; idx < R * F; idx += kBssEnergyTile) {
            sj[idx] = cj[((size_t)fi * (R + 1) + e) * R * F + idx];
            st[idx] = ct[((size_t)fi * (R + 1) + e) * R * F + idx];
        }
        double acc[NV];
#pragma unroll
        for (int i = 0; i < NV; ++i) acc[i] = 0.0;
        for (long long tt = t0; tt < t1; tt += kBssEnergyTile) {
            __syncthreads();
            for (int idx = threadIdx.x; idx < R * W; idx += kBssEnergyTile) {
                const int i = idx / W, q = idx - i * W;
                const long long t = tt - (F - 1) + q;
                sref[idx] = t >= 0 && t < T ? (double)__ldg(ref + ((size_t)b * R + i) * items.T + off + t) : 0.0;
            }
            __syncthreads();
            const long long t = tt + threadIdx.x;
            if (t < t1) {
                double pa = 0.0, pt[S];
#pragma unroll
                for (int j = 0; j < S; ++j) {
                    double p = 0.0;
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        const int i = j * C + c;
                        const double* s = sref + (size_t)i * W + threadIdx.x + F - 1;
                        for (int l = 0; l < F; ++l) {
                            const double v = s[-l];
                            pa = fma(sj[i * F + l], v, pa);
                            p = fma(st[i * F + l], v, p);
                        }
                    }
                    pt[j] = p;
                }
                const double ev = t < T ? (double)__ldg(er + t) : 0.0;
#pragma unroll
                for (int j = 0; j < S; ++j) {
                    acc[j] = fma(pt[j], pt[j], acc[j]);
                    acc[S + j] = fma(ev - pt[j], ev - pt[j], acc[S + j]);
                    acc[2 * S + j] = fma(pa - pt[j], pa - pt[j], acc[2 * S + j]);
                }
                acc[3 * S] = fma(pa, pa, acc[3 * S]);
                acc[3 * S + 1] = fma(ev - pa, ev - pa, acc[3 * S + 1]);
                acc[3 * S + 2] = fma(ev, ev, acc[3 * S + 2]);
                if constexpr (IMG) {
                    const int c = e % C;
#pragma unroll
                    for (int j = 0; j < S; ++j) {
                        const double sv = sref[(size_t)(j * C + c) * W + threadIdx.x + F - 1];   // s_jC+c[t]
                        acc[3 * S + 3 + j] = fma(pt[j] - sv, pt[j] - sv, acc[3 * S + 3 + j]);
                        acc[4 * S + 3 + j] = fma(ev - sv, ev - sv, acc[4 * S + 3 + j]);
                        if constexpr (V4) acc[5 * S + 3 + j] = fma(sv, sv, acc[5 * S + 3 + j]);
                    }
                }
            }
        }
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const double s = warp_sum_f64(acc[i]);
            if (lane == 0) red[warp][i] = s;
        }
        __syncthreads();
        if (threadIdx.x < NV) {
            double s = 0.0;
            for (int w = 0; w < kBssEnergyTile / 32; ++w) s += red[w][threadIdx.x];
            epart[(((size_t)it * chunks + chunk) * (R + 1) + e) * NV + threadIdx.x] = s;
        }
    }
}

// mir_eval's _safe_db: a zero denominator is +inf
__device__ __forceinline__ double bss_db(double num, double den) {
    return den == 0.0 ? (double)INFINITY : 10.0 * log10(num / den);
}

// one thread per item.  sdr/sir/sar/perm [B][S] for the estimates (perm[j]: the estimate given reference j); with the
// mixture (NE == S + 1), msdr/msir/msar [B][S]: the mixture scored as the estimate of every reference.  Source images
// (IMG) sum each estimate image's rows' energies over its C channels, in channel order, and also write isr [B][S].
// BSS-eval v4 (V4, with IMG; eref unused) takes |s_j|^2 from the window's own energies and tests no projection per
// window, where whole-track filters give none: bss_track_check_kernel has tested the recording and set the filters of
// a recording that failed, or held a silent or non-finite row, to NaN, which makes its windows' energies NaN.
template <int S, int NE, int C = 1, bool IMG = false, bool V4 = false>
__global__ void __launch_bounds__(256)
bss_final_kernel(const double* __restrict__ epart, const double* __restrict__ eref, int chunks, double* __restrict__ sdr,
                 double* __restrict__ isr, double* __restrict__ sir, double* __restrict__ sar, int* __restrict__ perm,
                 double* __restrict__ msdr, double* __restrict__ msir, double* __restrict__ msar, int B,
                 int compute_permutation) {
    constexpr int R = S * C, NV = bss_energy_count(S, IMG, V4);
    constexpr int NI = IMG ? S : NE;                    // scored estimates: images, or rows (with the mixture's)
    for (long long b = blockIdx.x * 256LL + threadIdx.x; b < B; b += (long long)gridDim.x * 256) {
        double en[NE][NV];
#pragma unroll
        for (int e = 0; e < NE; ++e)
#pragma unroll
            for (int i = 0; i < NV; ++i) en[e][i] = 0.0;
        for (int c = 0; c < chunks; ++c) {
            const double* pc = epart + ((size_t)b * chunks + c) * (R + 1) * NV;
#pragma unroll
            for (int e = 0; e < NE; ++e)
#pragma unroll
                for (int i = 0; i < NV; ++i) en[e][i] += pc[e * NV + i];
        }
        double wref[S];                                 // v4: the window's reference image energies
        if constexpr (V4) {
#pragma unroll
            for (int j = 0; j < S; ++j) {
                wref[j] = en[0][5 * S + 3 + j];
#pragma unroll
                for (int c = 1; c < C; ++c) wref[j] += en[c][5 * S + 3 + j];
            }
        }
        const double* er = V4 ? nullptr : eref + (size_t)b * R;
        bool silent_ref = false;
#pragma unroll
        for (int i = 0; i < S; ++i)
            silent_ref = silent_ref || !bss_scorable(V4 ? wref[i] : bss_image_energy<C>(er, i));
        bool silent = silent_ref;
#pragma unroll
        for (int e = 0; e < S; ++e) {
            double e2 = en[e * C][3 * S + 2];
            bool held = V4 || bss_projections_hold<S>(en[e * C]);
#pragma unroll
            for (int c = 1; c < C; ++c) {
                e2 += en[e * C + c][3 * S + 2];
                held = held && (V4 || bss_projections_hold<S>(en[e * C + c]));
            }
            if constexpr (V4) {                         // NaN filters: a recording that cannot be scored
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    held = held && en[e * C + c][3 * S] < (double)INFINITY;
#pragma unroll
                    for (int j = 0; j < S; ++j) held = held && en[e * C + c][j] < (double)INFINITY;
                }
            }
            silent = silent || !bss_scorable(e2) || !held;
        }
        double d[NI][S], i_[NI][S], a[NI][S], g[IMG ? S : 1][S];
        if constexpr (!IMG) {
#pragma unroll
            for (int e = 0; e < NE; ++e)
#pragma unroll
                for (int j = 0; j < S; ++j) {
                    d[e][j] = bss_db(en[e][j], en[e][S + j]);
                    i_[e][j] = bss_db(en[e][j], en[e][2 * S + j]);
                    a[e][j] = bss_db(en[e][3 * S], en[e][3 * S + 1]);
                }
        } else {
#pragma unroll
            for (int e = 0; e < S; ++e)
#pragma unroll
                for (int j = 0; j < S; ++j) {
                    // |P_j e|^2, |P_all e - P_j e|^2, |P_all e|^2, |e - P_all e|^2, |P_j e - s_j|^2, |e - s_j|^2
                    double pj = 0.0, in = 0.0, pa = 0.0, ar = 0.0, sp = 0.0, dd = 0.0;
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        const double* v = en[e * C + c];
                        pj += v[j];
                        in += v[2 * S + j];
                        pa += v[3 * S];
                        ar += v[3 * S + 1];
                        sp += v[3 * S + 3 + j];
                        dd += v[4 * S + 3 + j];
                    }
                    const double sj = V4 ? wref[j] : bss_image_energy<C>(er, j);
                    d[e][j] = bss_db(sj, dd);
                    g[e][j] = bss_db(sj, sp);
                    i_[e][j] = bss_db(pj, in);
                    a[e][j] = bss_db(pa, ar);
                }
        }
        int p[S];
#pragma unroll
        for (int j = 0; j < S; ++j) p[j] = j;
        if (compute_permutation) {
            int besti;
            best_assignment<S, S>([&](const int* q) {
                double m = 0.0;
                for (int j = 0; j < S; ++j) m = __dadd_rn(m, i_[q[j]][j]);
                return m / (double)S;
            }, besti, p);
        }
        const double nan = __longlong_as_double(0x7ff8000000000000LL);
#pragma unroll
        for (int j = 0; j < S; ++j) {
            double dj = 0.0, ij = 0.0, aj = 0.0, gj = 0.0;
#pragma unroll
            for (int e = 0; e < S; ++e)
                if (p[j] == e) {
                    dj = d[e][j]; ij = i_[e][j]; aj = a[e][j];
                    if constexpr (IMG) gj = g[e][j];
                }
            const size_t o = (size_t)b * S + j;
            sdr[o] = silent ? nan : dj;
            sir[o] = silent ? nan : ij;
            sar[o] = silent ? nan : aj;
            if constexpr (IMG) isr[o] = silent ? nan : gj;
            if (perm) perm[o] = silent ? -1 : p[j];
            if constexpr (NI > S) {
                const bool ms = silent_ref || !bss_scorable(en[S][3 * S + 2]) || !bss_projections_hold<S>(en[S]);
                msdr[o] = ms ? nan : d[S][j];
                msir[o] = ms ? nan : i_[S][j];
                msar[o] = ms ? nan : a[S][j];
            }
        }
    }
}

// BSS-eval v4: tests each recording's whole-track filters.  grid = B (S + 1), the solve's systems; 256 threads; smem
// [M][M][F] + [M][F] doubles for the system's M rows.  Estimate row e's filters c solve G c = D_e, so for a projection
// c^T G c = c^T D_e = |P e|^2 over the whole track, and 2 |c^T G c - c^T D_e| is the defect |p|^2 + |e - p|^2 - |e|^2
// that bss_final_kernel bounds per item for the other entries, here formed from the recording's correlations.  A
// system that fails it for any estimate row, and every system of a recording with a silent or non-finite reference or
// estimate image, has its filters set to NaN, which makes each of the recording's windows NaN.
template <int S, int C>
__global__ void __launch_bounds__(256)
bss_track_check_kernel(const double* __restrict__ tot, const double* __restrict__ etot,
                       const double* __restrict__ eref, double* __restrict__ cj, double* __restrict__ ct, int F) {
    constexpr int R = S * C, NE = R, NB = R + NE;
    extern __shared__ double smem[];
    __shared__ double red[8][2];
    __shared__ int held;
    const long long b = blockIdx.x / (S + 1);
    const int sys = (int)(blockIdx.x - b * (S + 1));
    const int M = sys == 0 ? R : C, r0 = sys == 0 ? 0 : (sys - 1) * C;
    const BssCorr<R, NB> cr{tot + (size_t)b * R * NB * F, 1, F};
    const double* ee = etot + (size_t)b * NE;         // |e|^2 of each estimate row over the track
    double* sg = smem;                                  // sg[(r M + q) F + k] = X_{r0+r, r0+q}[k]
    double* sc = sg + (size_t)M * M * F;                // the filters of one estimate row
    bool ok = true;
#pragma unroll
    for (int i = 0; i < S; ++i)
        ok = ok && bss_scorable(bss_image_energy<C>(eref + (size_t)b * R, i)) && bss_scorable(bss_image_energy<C>(ee, i));
    for (int idx = threadIdx.x; idx < M * M * F; idx += blockDim.x) {
        const int r = idx / (M * F), q = (idx / F) % M, k = idx % F;
        sg[idx] = cr(r0 + r, r0 + q, k);
    }
    double* fil = (sys == 0 ? cj : ct) + (size_t)b * (R + 1) * R * F;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int e = 0; e < NE && ok; ++e) {                // ok is the same in every thread
        __syncthreads();
        for (int idx = threadIdx.x; idx < M * F; idx += blockDim.x)
            sc[idx] = fil[((size_t)e * R + r0 + idx / F) * F + idx % F];
        __syncthreads();
        double cgc = 0.0, cd = 0.0;
        for (int idx = threadIdx.x; idx < M * F; idx += blockDim.x) {
            const int r = idx / F, l = idx % F;
            double g = 0.0;                             // (G c)[(r, l)]
            for (int q = 0; q < M; ++q) {
                const double* xrq = sg + ((size_t)r * M + q) * F;
                const double* xqr = sg + ((size_t)q * M + r) * F;
                const double* cq = sc + (size_t)q * F;
                for (int m = 0; m <= l; ++m) g = fma(xrq[l - m], cq[m], g);
                for (int m = l + 1; m < F; ++m) g = fma(xqr[m - l], cq[m], g);
            }
            cgc = fma(sc[idx], g, cgc);
            cd = fma(sc[idx], cr(r0 + r, R + e, l), cd);
        }
        cgc = warp_sum_f64(cgc);
        cd = warp_sum_f64(cd);
        if (lane == 0) { red[warp][0] = cgc; red[warp][1] = cd; }
        __syncthreads();
        if (threadIdx.x == 0) {
            double a = 0.0, d = 0.0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { a += red[w][0]; d += red[w][1]; }
            held = 2.0 * fabs(a - d) <= kBssProjectionDefect * ee[e];
        }
        __syncthreads();
        ok = held != 0;
    }
    if (ok) return;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    for (int idx = threadIdx.x; idx < NE * R * F; idx += blockDim.x) {
        const int r = (idx / F) % R;
        if (sys == 0 || r / C == sys - 1) fil[idx] = nan;
    }
}

// Scores n items of the view in launches of at most cap items, all through one scratch sized for cap items of at most
// L samples: the launches follow each other on the stream with no host synchronisation between them, so a call can
// be captured in a CUDA graph.  Item i's outputs are [i][S].  Source images are <S, S C, C, true>.
template <int S, int NE, int C = 1, bool IMG = false>
static int bss_eval_launch(const float* ref, const float* est, const float* mix, double* sdr, double* isr,
                           double* sir, double* sar, int* perm, double* msdr, double* msir, double* msar,
                           BssItems items, long long n, long long cap, long long L, int F, int compute_permutation,
                           void* scratch, cudaStream_t st) {
    constexpr int R = S * C;
    const int m = (int)(n < cap ? n : cap);
    const BssScratch s(scratch, m, S, C, L, F, bss_energy_count(S, IMG));
    const int cc = bss_corr_chunks(L), ec = bss_energy_chunks(L, F);
    if ((long long)m * cc > 0x7fffffffLL || (long long)m * (S + 1) > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    const size_t corr_smem = sizeof(double) * (R + NE) * (kBssCorrTile + F - 1);
    const size_t solve_smem = sizeof(double) * (size_t)F * (2 * R * R + NE * R);
    const size_t energy_smem = sizeof(double) * (size_t)R * (kBssEnergyTile + F - 1 + 2 * F);
    for (long long first = 0; first < n; first += m) {
        const int k = (int)(n - first < m ? n - first : m);
        const size_t o = (size_t)first * S;
        items.first = first;
        int e;
        if ((e = launch(bss_corr_kernel<R, NE, int>, (unsigned)((long long)k * cc), kBssCorrTile, corr_smem, st, ref, est,
                        mix, s.part, items, F, cc)))
            return e;
        if ((e = launch(bss_solve_kernel<S, NE, C>, (unsigned)((long long)k * (S + 1)), 256, solve_smem, st, s.part,
                        cc, s.rj, s.rt, s.eref, s.cj, s.ct, F)))
            return e;
        if ((e = launch(bss_energy_kernel<S, NE, C, IMG>, (unsigned)((long long)k * ec), kBssEnergyTile, energy_smem,
                        st, ref, est, mix, s.cj, s.ct, s.epart, items, F, ec)))
            return e;
        if ((e = launch(bss_final_kernel<S, NE, C, IMG>, item_blocks(k), 256, 0, st, s.epart, s.eref, ec, sdr + o,
                        isr ? isr + o : nullptr, sir + o, sar + o, perm ? perm + o : nullptr,
                        msdr ? msdr + o : nullptr, msir ? msir + o : nullptr, msar ? msar + o : nullptr, k,
                        compute_permutation)))
            return e;
    }
    return SDR_OK;
}

// Null or misaligned buffers, shared by every entry
static bool bss_buffers_ok(const float* ref, const float* est, const float* mix, const double* sdr, const double* sir,
                           const double* sar, const double* msdr, const double* msir, const double* msar,
                           const void* scratch) {
    if (!ref || !est || !sdr || !sir || !sar || !scratch || reinterpret_cast<uintptr_t>(scratch) % 8) return false;
    return !mix || (msdr && msir && msar);
}

static int bss_dispatch(const float* ref, const float* est, const float* mix, double* sdr, double* sir, double* sar,
                        int* perm, double* msdr, double* msir, double* msar, int S, const BssItems& items, long long n,
                        long long cap, long long L, int F, int compute_permutation, void* scratch, cudaStream_t st) {
    return with_sources(S, [&](auto s) {
        constexpr int c = decltype(s)::value;
        return mix ? bss_eval_launch<c, c + 1>(ref, est, mix, sdr, nullptr, sir, sar, perm, msdr, msir, msar, items, n,
                                               cap, L, F, compute_permutation, scratch, st)
                   : bss_eval_launch<c, c>(ref, est, nullptr, sdr, nullptr, sir, sar, perm, nullptr, nullptr, nullptr,
                                           items, n, cap, L, F, compute_permutation, scratch, st);
    });
}

// The source-image kernels are instantiated for S C <= 4: the joint system's shared memory, (2 R^2 + E R) F doubles
// at R = E = S C, is 192 KiB at R = 4 and F = 512.
// Calls run(std::integral_constant<int, S>(), std::integral_constant<int, C>()) for the instantiated (S, C).
template <class Fn> static int with_images(int S, int C, const Fn& run) {
    using I1 = std::integral_constant<int, 1>;
    using I2 = std::integral_constant<int, 2>;
    if (C == 1) return with_sources(S, [&](auto s) { return run(s, I1()); });
    if (S == 1 && C == 2) return run(I1(), I2());
    if (S == 1 && C == 3) return run(I1(), std::integral_constant<int, 3>());
    if (S == 1 && C == 4) return run(I1(), std::integral_constant<int, 4>());
    if (S == 2 && C == 2) return run(I2(), I2());
    return SDR_ERR_UNSUPPORTED;
}

static int bss_images_dispatch(const float* ref, const float* est, double* sdr, double* isr, double* sir, double* sar,
                               int* perm, int S, int C, const BssItems& items, long long n, long long cap, long long L,
                               int F, int compute_permutation, void* scratch, cudaStream_t st) {
    return with_images(S, C, [&](auto s, auto c) {
        constexpr int S_ = decltype(s)::value, C_ = decltype(c)::value;
        return bss_eval_launch<S_, S_ * C_, C_, true>(ref, est, nullptr, sdr, isr, sir, sar, perm, nullptr, nullptr,
                                                      nullptr, items, n, cap, L, F, compute_permutation, scratch, st);
    });
}

// sdr_bss_eval (mix null) and sdr_bss_eval_mixture: item b is the whole of recording b, all in one launch sequence
static int bss_eval(const float* ref, const float* est, const float* mix, double* sdr, double* sir, double* sar,
                    int* perm, double* msdr, double* msir, double* msar, int B, int S, long long T, int F,
                    int compute_permutation, void* scratch, cudaStream_t st) {
    if (!bss_buffers_ok(ref, est, mix, sdr, sir, sar, msdr, msir, msar, scratch)) return SDR_ERR_BAD_ARGUMENT;
    if (!sdr_bss_eval_scratch_bytes(B, S, T, F)) return B <= 0 || T <= 0 ? SDR_ERR_BAD_ARGUMENT : SDR_ERR_UNSUPPORTED;
    const BssItems whole{T, T, T, 1, 0, 0, nullptr};
    return bss_dispatch(ref, est, mix, sdr, sir, sar, perm, msdr, msir, msar, S, whole, B, B, T, F,
                        compute_permutation, scratch, st);
}

// mir_eval's window count, floor((T - W + H) / H), and one column (the whole-item fallback) when that is below 2:
// when T < W + H
static long long bss_window_count(long long T, long long W, long long H) {
    return T - W < H ? 1 : (T - W) / H + 1;
}

// The longest item a framewise call can score: W, or a fallback recording, which is shorter than W + H
static long long bss_framewise_span(long long T, long long W, long long H) {
    return W > T || H - 1 > T - W ? T : W + H - 1;
}

// The scratch of B whole items of S sources of C rows (0: unsupported).  S F delayed references in R^(T+F-1), R = S C:
// more than the dimensions (T < (R - 1) F + 1) makes the joint system singular by construction, where the recursion's
// rounding no longer separates dependent pivots from independent ones.
static size_t bss_scratch_bytes(int B, int S, int C, long long T, int F, bool images) {
    if (B <= 0 || S < 1 || S > 4 || C < 1 || S * C > 4 || T <= 0 || F < 1 || F > kBssMaxF) return 0;
    if ((long long)S * C * F > T + F - 1) return 0;
    return BssScratch(nullptr, B, S, C, T, F, bss_energy_count(S, images)).bytes;
}

// The scratch of a framewise call: at most kBssFramewiseItems items of the longest length one can have (0: unsupported)
static size_t bss_framewise_scratch_bytes(int B, int S, int C, long long T, long long W, long long H, int F,
                                          bool images) {
    if (B <= 0 || S < 1 || S > 4 || C < 1 || S * C > 4 || T <= 0 || W <= 0 || H <= 0 || F < 1 || F > kBssMaxF)
        return 0;
    const long long len = T - W < H ? T : W;               // the length of every item, or of the fallback's
    if ((long long)S * C * F > len + F - 1) return 0;
    const long long nwin = bss_window_count(T, W, H);
    if (nwin > INT64_MAX / S / B) return 0;
    const long long n = (long long)B * nwin;
    return BssScratch(nullptr, (int)(n < kBssFramewiseItems ? n : kBssFramewiseItems), S, C,
                      bss_framewise_span(T, W, H), F, bss_energy_count(S, images)).bytes;
}

// BSS-eval v4's correlation launches take at most this many CTAs' chunks (kBssTrackChunk samples each) across the
// batch, at least one chunk per recording: about four waves of the correlation kernel on an H100, so one recording
// fills the GPU while the launch partials stay bounded (69 MB at R = 4, F = 512).
constexpr long long kBssTrackBlocks = 512;

static long long bss_track_chunks(long long T) { return (T + kBssTrackChunk - 1) / kBssTrackChunk; }

// Chunks per recording in one v4 correlation launch
static int bss_track_launch_chunks(int B, long long T) {
    const long long g = kBssTrackBlocks / B < 1 ? 1 : kBssTrackBlocks / B, total = bss_track_chunks(T);
    return (int)(g < total ? g : total);
}

// museval's window count: floor((T - W + H) / H) for T >= W
static long long bss_v4_window_count(long long T, long long W, long long H) { return (T - W) / H + 1; }

// BSS-eval v4's scratch for B recordings of R = S C rows and n windows.  Doubles:
//   part  [B][G][R 2R F + R]   one correlation launch's chunk partials (G chunks per recording)
//   tot   [B][R][2R][F]        each recording's correlations over its whole length
//   etot  [B][R]               its estimate rows' energies
//   rj, rt, eref, cj, ct       the solve's, per recording (as BssScratch with the mixture's row)
//   epart [m][echunks][R+1][NV]  the energy partials of a launch of m <= kBssFramewiseItems windows of W samples
struct BssV4Scratch {
    double *part, *tot, *etot, *rj, *rt, *eref, *cj, *ct, *epart;
    int G;
    size_t bytes;
    BssV4Scratch(void* base, int B, int S, int C, long long T, long long W, long long n, int F) {
        const size_t b = (size_t)B, s = (size_t)S, c = (size_t)C, r = s * c, f = (size_t)F, ne = r + 1;
        const size_t m = (size_t)(n < kBssFramewiseItems ? n : kBssFramewiseItems);
        G = bss_track_launch_chunks(B, T);
        size_t off = 0;
        double* p = static_cast<double*>(base);
        auto take = [&](size_t k) { double* q = p ? p + off : nullptr; off += k; return q; };
        part = take(b * G * bss_partial_size((int)r, (int)r, F, true));
        tot = take(b * r * 2 * r * f);
        etot = take(b * r);
        rj = take(b * f * r * r);
        rt = take(b * s * f * c * c);
        eref = take(b * r);
        cj = take(b * ne * r * f);
        ct = take(b * ne * r * f);
        epart = take(m * bss_energy_chunks(W, F) * ne * (size_t)bss_energy_count(S, true, true));
        bytes = off * sizeof(double);
    }
};

static size_t bss_v4_scratch_bytes(int B, int S, int C, long long T, long long W, long long H, int F) {
    if (B <= 0 || S < 1 || S > 4 || C < 1 || S * C > 4 || T <= 0 || W <= 0 || H <= 0 || F < 1 || F > kBssMaxF)
        return 0;
    if (T < W || (long long)S * C * F > T + F - 1) return 0;     // no window, or no recording that can be solved
    const long long nwin = bss_v4_window_count(T, W, H);
    if (nwin > INT64_MAX / S / B) return 0;
    return BssV4Scratch(nullptr, B, S, C, T, W, (long long)B * nwin, F).bytes;
}

// Correlations over each whole recording in launches of G chunks per recording, each folded into the running totals;
// one solve and one filter check per recording; then the windows, in launches of at most kBssFramewiseItems through
// one scratch.  Nothing synchronises with the host.
template <int S, int C>
static int bss_v4_launch(const float* ref, const float* est, const long long* lengths, double* sdr, double* isr,
                         double* sir, double* sar, int* perm, int B, long long T, long long W, long long H, int F,
                         int compute_permutation, void* scratch, cudaStream_t st) {
    constexpr int R = S * C, NE = R;
    const long long nwin = bss_v4_window_count(T, W, H), n = (long long)B * nwin;
    const BssV4Scratch s(scratch, B, S, C, T, W, n, F);
    const long long min_len = (long long)(R - 1) * F + 1;
    const size_t psize = bss_partial_size(R, NE, F, true);
    const long long fold_blocks = ((long long)B * psize + 255) / 256;
    const int ec = bss_energy_chunks(W, F);
    const int m = (int)(n < kBssFramewiseItems ? n : kBssFramewiseItems);
    if ((long long)B * s.G > 0x7fffffffLL || (long long)B * (S + 1) > 0x7fffffffLL || fold_blocks > 0x7fffffffLL ||
        (long long)m * ec > 0x7fffffffLL)
        return SDR_ERR_UNSUPPORTED;
    const size_t corr_smem = sizeof(double) * (R + NE) * (kBssCorrTile + F - 1);
    const size_t solve_smem = sizeof(double) * (size_t)F * (2 * R * R + NE * R);
    const size_t check_smem = sizeof(double) * (size_t)F * (R * R + R);
    const size_t energy_smem = sizeof(double) * (size_t)R * (kBssEnergyTile + F - 1 + 2 * F);
    const BssItems whole{T, T, T, 1, 0, min_len, lengths};
    const long long total = bss_track_chunks(T);
    int e;
    for (long long c0 = 0; c0 < total; c0 += s.G) {
        const BssTrackChunks ch{(int)(total - c0 < s.G ? total - c0 : s.G), c0};
        if ((e = launch(bss_corr_kernel<R, NE, BssTrackChunks>, (unsigned)((long long)B * ch.n), kBssCorrTile,
                        corr_smem, st, ref, est, nullptr, s.part, whole, F, ch)))
            return e;
        if ((e = launch(bss_fold_kernel, (unsigned)fold_blocks, 256, 0, st, s.part, s.tot, s.etot, whole, B,
                        (long long)R * 2 * R * F, NE, ch)))
            return e;
    }
    if ((e = launch(bss_solve_kernel<S, NE, C>, (unsigned)(B * (S + 1)), 256, solve_smem, st, s.tot, 1, s.rj, s.rt,
                    s.eref, s.cj, s.ct, F)))
        return e;
    if ((e = launch(bss_track_check_kernel<S, C>, (unsigned)(B * (S + 1)), 256, check_smem, st, s.tot, s.etot,
                    s.eref, s.cj, s.ct, F)))
        return e;
    BssItems win{T, W, H, nwin, 0, min_len, lengths};
    for (long long first = 0; first < n; first += m) {
        const int k = (int)(n - first < m ? n - first : m);
        const size_t o = (size_t)first * S;
        win.first = first;
        if ((e = launch(bss_energy_kernel<S, NE, C, true, true>, (unsigned)((long long)k * ec), kBssEnergyTile,
                        energy_smem, st, ref, est, nullptr, s.cj, s.ct, s.epart, win, F, ec)))
            return e;
        if ((e = launch(bss_final_kernel<S, NE, C, true, true>, item_blocks(k), 256, 0, st, s.epart, nullptr, ec,
                        sdr + o, isr + o, sir + o, sar + o, perm ? perm + o : nullptr, nullptr, nullptr, nullptr, k,
                        compute_permutation)))
            return e;
    }
    return SDR_OK;
}

}  // namespace sdr

using namespace sdr;

#pragma GCC visibility push(default)
extern "C" {

size_t sdr_bss_eval_scratch_bytes(int B, int S, int64_t T, int F) { return bss_scratch_bytes(B, S, 1, T, F, false); }

int sdr_bss_eval(const float* reference, const float* estimate, double* sdr, double* sir, double* sar,
                 int32_t* perm_or_null, int B, int S, int64_t T, int F, int compute_permutation, void* scratch,
                 sdr_stream stream) {
    return bss_eval(reference, estimate, nullptr, sdr, sir, sar, perm_or_null, nullptr, nullptr, nullptr, B, S, T, F,
                    compute_permutation, scratch, static_cast<cudaStream_t>(stream));
}

int sdr_bss_eval_mixture(const float* reference, const float* estimate, const float* mixture, double* sdr,
                         double* sir, double* sar, int32_t* perm_or_null, double* mix_sdr, double* mix_sir,
                         double* mix_sar, int B, int S, int64_t T, int F, int compute_permutation, void* scratch,
                         sdr_stream stream) {
    if (!mixture) return SDR_ERR_BAD_ARGUMENT;
    return bss_eval(reference, estimate, mixture, sdr, sir, sar, perm_or_null, mix_sdr, mix_sir, mix_sar, B, S, T, F,
                    compute_permutation, scratch, static_cast<cudaStream_t>(stream));
}

size_t sdr_bss_eval_framewise_scratch_bytes(int B, int S, int64_t T, int64_t W, int64_t H, int F) {
    return bss_framewise_scratch_bytes(B, S, 1, T, W, H, F, false);
}

int sdr_bss_eval_framewise(const float* reference, const float* estimate, const float* mixture_or_null,
                           const int64_t* lengths_or_null, double* sdr, double* sir, double* sar,
                           int32_t* perm_or_null, double* mix_sdr, double* mix_sir, double* mix_sar, int B, int S,
                           int64_t T, int64_t W, int64_t H, int F, int compute_permutation, void* scratch,
                           sdr_stream stream) {
    const float* mix = mixture_or_null;
    if (!bss_buffers_ok(reference, estimate, mix, sdr, sir, sar, mix_sdr, mix_sir, mix_sar, scratch) ||
        reinterpret_cast<uintptr_t>(lengths_or_null) % 8)
        return SDR_ERR_BAD_ARGUMENT;
    if (!sdr_bss_eval_framewise_scratch_bytes(B, S, T, W, H, F))
        return B <= 0 || T <= 0 || W <= 0 || H <= 0 ? SDR_ERR_BAD_ARGUMENT : SDR_ERR_UNSUPPORTED;
    const long long nwin = bss_window_count(T, W, H);
    const BssItems items{T, W, H, nwin, 0, (long long)(S - 1) * F + 1,
                         reinterpret_cast<const long long*>(lengths_or_null)};
    return bss_dispatch(reference, estimate, mix, sdr, sir, sar, perm_or_null, mix ? mix_sdr : nullptr,
                        mix ? mix_sir : nullptr, mix ? mix_sar : nullptr, S, items, (long long)B * nwin,
                        kBssFramewiseItems, bss_framewise_span(T, W, H), F, compute_permutation, scratch,
                        static_cast<cudaStream_t>(stream));
}

size_t sdr_bss_eval_images_scratch_bytes(int B, int S, int C, int64_t T, int F) {
    return bss_scratch_bytes(B, S, C, T, F, true);
}

int sdr_bss_eval_images(const float* reference, const float* estimate, double* sdr, double* isr, double* sir,
                        double* sar, int32_t* perm_or_null, int B, int S, int C, int64_t T, int F,
                        int compute_permutation, void* scratch, sdr_stream stream) {
    if (!isr || !bss_buffers_ok(reference, estimate, nullptr, sdr, sir, sar, nullptr, nullptr, nullptr, scratch))
        return SDR_ERR_BAD_ARGUMENT;
    if (!sdr_bss_eval_images_scratch_bytes(B, S, C, T, F))
        return B <= 0 || T <= 0 ? SDR_ERR_BAD_ARGUMENT : SDR_ERR_UNSUPPORTED;
    const BssItems whole{T, T, T, 1, 0, 0, nullptr};
    return bss_images_dispatch(reference, estimate, sdr, isr, sir, sar, perm_or_null, S, C, whole, B, B, T, F,
                               compute_permutation, scratch, static_cast<cudaStream_t>(stream));
}

size_t sdr_bss_eval_images_framewise_scratch_bytes(int B, int S, int C, int64_t T, int64_t W, int64_t H, int F) {
    return bss_framewise_scratch_bytes(B, S, C, T, W, H, F, true);
}

int sdr_bss_eval_images_framewise(const float* reference, const float* estimate, const int64_t* lengths_or_null,
                                  double* sdr, double* isr, double* sir, double* sar, int32_t* perm_or_null, int B,
                                  int S, int C, int64_t T, int64_t W, int64_t H, int F, int compute_permutation,
                                  void* scratch, sdr_stream stream) {
    if (!isr || !bss_buffers_ok(reference, estimate, nullptr, sdr, sir, sar, nullptr, nullptr, nullptr, scratch) ||
        reinterpret_cast<uintptr_t>(lengths_or_null) % 8)
        return SDR_ERR_BAD_ARGUMENT;
    if (!sdr_bss_eval_images_framewise_scratch_bytes(B, S, C, T, W, H, F))
        return B <= 0 || T <= 0 || W <= 0 || H <= 0 ? SDR_ERR_BAD_ARGUMENT : SDR_ERR_UNSUPPORTED;
    const long long nwin = bss_window_count(T, W, H);
    const BssItems items{T, W, H, nwin, 0, (long long)(S * C - 1) * F + 1,
                         reinterpret_cast<const long long*>(lengths_or_null)};
    return bss_images_dispatch(reference, estimate, sdr, isr, sir, sar, perm_or_null, S, C, items,
                               (long long)B * nwin, kBssFramewiseItems, bss_framewise_span(T, W, H), F,
                               compute_permutation, scratch, static_cast<cudaStream_t>(stream));
}

size_t sdr_bss_eval_v4_scratch_bytes(int B, int S, int C, int64_t T, int64_t W, int64_t H, int F) {
    return bss_v4_scratch_bytes(B, S, C, T, W, H, F);
}

int sdr_bss_eval_v4(const float* reference, const float* estimate, const int64_t* lengths_or_null, double* sdr,
                    double* isr, double* sir, double* sar, int32_t* perm_or_null, int B, int S, int C, int64_t T,
                    int64_t W, int64_t H, int F, int compute_permutation, void* scratch, sdr_stream stream) {
    if (!isr || !bss_buffers_ok(reference, estimate, nullptr, sdr, sir, sar, nullptr, nullptr, nullptr, scratch) ||
        reinterpret_cast<uintptr_t>(lengths_or_null) % 8)
        return SDR_ERR_BAD_ARGUMENT;
    if (!sdr_bss_eval_v4_scratch_bytes(B, S, C, T, W, H, F))
        return B <= 0 || T <= 0 || W <= 0 || H <= 0 ? SDR_ERR_BAD_ARGUMENT : SDR_ERR_UNSUPPORTED;
    return with_images(S, C, [&](auto s, auto c) {
        return bss_v4_launch<decltype(s)::value, decltype(c)::value>(
            reference, estimate, reinterpret_cast<const long long*>(lengths_or_null), sdr, isr, sir, sar,
            perm_or_null, B, T, W, H, F, compute_permutation, scratch, static_cast<cudaStream_t>(stream));
    });
}

}  // extern "C"
#pragma GCC visibility pop
