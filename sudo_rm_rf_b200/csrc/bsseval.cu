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

// Estimate row e's energies (bss_energy_kernel's layout) come from projections: the joint one and every own one.
template <int S>
__device__ __forceinline__ bool bss_projections_hold(const double (&en)[3 * S + 3]) {
    bool ok = bss_is_projection(en[3 * S], en[3 * S + 1], en[3 * S + 2]);
#pragma unroll
    for (int j = 0; j < S; ++j) ok = ok && bss_is_projection(en[j], en[S + j], en[3 * S + 2]);
    return ok;
}

// Scratch carve-up, sized for S estimates plus the mixture whether or not it is given.  Doubles:
//   part  [B][chunks][S][2S+1][F]   correlation partials (rows: S references, then the NE estimate rows)
//   rj    [B][F][S][S]              the joint system's normalised blocks
//   rt    [B][S][F]                 each reference's normalised autocorrelation
//   eref  [B][S]                    reference energies
//   cj    [B][S+1][S][F]            joint filters per estimate row
//   ct    [B][S+1][S][F]            own-reference filters per estimate row
//   epart [B][echunks][S+1][3S+3]   energy partials
struct BssScratch {
    double *part, *rj, *rt, *eref, *cj, *ct, *epart;
    size_t bytes;
    BssScratch(void* base, int B, int S, long long T, int F) {
        const size_t b = (size_t)B, s = (size_t)S, f = (size_t)F, ne = s + 1;
        size_t off = 0;
        double* p = static_cast<double*>(base);
        auto take = [&](size_t n) { double* r = p ? p + off : nullptr; off += n; return r; };
        part = take(b * bss_corr_chunks(T) * s * (s + ne) * f);
        rj = take(b * f * s * s);
        rt = take(b * s * f);
        eref = take(b * s);
        cj = take(b * ne * s * f);
        ct = take(b * ne * s * f);
        epart = take(b * bss_energy_chunks(T, F) * ne * (3 * s + 3));
        bytes = off * sizeof(double);
    }
};

// Row r of item b: references 0..S-1, estimates S..2S-1, the mixture 2S.
__device__ __forceinline__ const float* bss_row(const float* ref, const float* est, const float* mix, int S,
                                                long long b, int r, long long T) {
    if (r < S) return ref + ((size_t)b * S + r) * T;
    if (r < 2 * S) return est + ((size_t)b * S + (r - S)) * T;
    return mix + (size_t)b * T;
}

// grid = B * chunks, kBssCorrTile threads; smem [NB][kBssCorrTile + F - 1] doubles
template <int S, int NE>
__global__ void __launch_bounds__(kBssCorrTile)
bss_corr_kernel(const float* __restrict__ ref, const float* __restrict__ est, const float* __restrict__ mix,
                double* __restrict__ part, long long T, int F, int chunks) {
    constexpr int NB = S + NE;
    extern __shared__ double sm[];
    const long long b = blockIdx.x / chunks;
    const int chunk = (int)(blockIdx.x - b * chunks);
    const long long per = (T + chunks - 1) / chunks;
    const long long t0 = (long long)chunk * per;
    const long long t1 = t0 + per < T ? t0 + per : T;
    const int W = kBssCorrTile + F - 1;
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
            sm[idx] = (q < n + F - 1 && t < T) ? (double)__ldg(bss_row(ref, est, mix, S, b, r, T) + t) : 0.0;
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
    }
    if (k < F) {
        double* pc = part + ((size_t)b * chunks + chunk) * S * NB * F;
#pragma unroll
        for (int i = 0; i < S; ++i)
#pragma unroll
            for (int r = 0; r < NB; ++r) pc[((size_t)i * NB + r) * F + k] = acc[i][r];
    }
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
    double inv[M];
#pragma unroll
    for (int r = 0; r < M; ++r) inv[r] = 1.0 / sqrt(sE[ch[r]]);
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

// grid = B (S + 1): system 0 of an item is the joint one, system 1 + j reference j's own.  256 threads.
template <int S, int NE>
__global__ void __launch_bounds__(256)
bss_solve_kernel(const double* __restrict__ part, int chunks, double* __restrict__ rj, double* __restrict__ rt,
                 double* __restrict__ eref, double* __restrict__ cj, double* __restrict__ ct, int F) {
    constexpr int NB = S + NE;
    extern __shared__ double smem[];
    __shared__ double sE[S];
    const long long b = blockIdx.x / (S + 1);
    const int sys = (int)(blockIdx.x - b * (S + 1));
    const BssCorr<S, NB> cr{part + (size_t)b * chunks * S * NB * F, chunks, F};
    if (threadIdx.x < S) sE[threadIdx.x] = cr(threadIdx.x, threadIdx.x, 0);
    __syncthreads();
    bool silent = false;
#pragma unroll
    for (int i = 0; i < S; ++i) silent = silent || !bss_scorable(sE[i]);
    if (sys == 0 && threadIdx.x < S) eref[(size_t)b * S + threadIdx.x] = sE[threadIdx.x];
    double* out = (sys == 0 ? cj : ct) + (size_t)b * (S + 1) * S * F;
    if (silent) {                                       // the item's outputs are NaN; its filters are set to zero
        for (int idx = threadIdx.x; idx < NE * S * F; idx += blockDim.x) {
            const int e = idx / (S * F), r = (idx / F) % S;
            if (sys == 0 || r == sys - 1) out[idx] = 0.0;
        }
        return;
    }
    if (sys == 0) {
        int ch[S];
#pragma unroll
        for (int i = 0; i < S; ++i) ch[i] = i;
        bss_levinson<S, NE>(cr, ch, sE, rj + (size_t)b * F * S * S, out, F, smem);
    } else {
        const int ch[1] = {sys - 1};
        bss_levinson<1, NE>(cr, ch, sE, rt + ((size_t)b * S + sys - 1) * F, out, F, smem);
    }
}

// grid = B * echunks, kBssEnergyTile threads; smem: references [S][kBssEnergyTile + F - 1], filters [2][S][F].
// Over t < T + F - 1, estimate row e's projections pa = sum_i cj_e,i * s_i and pt_j = ct_e,j * s_j and the energies
//     [0, S)  |pt_j|^2,   [S, 2S)  |e - pt_j|^2,   [2S, 3S)  |pa - pt_j|^2,   3S |pa|^2,   3S+1 |e - pa|^2,   3S+2 |e|^2
template <int S, int NE>
__global__ void __launch_bounds__(kBssEnergyTile)
bss_energy_kernel(const float* __restrict__ ref, const float* __restrict__ est, const float* __restrict__ mix,
                  const double* __restrict__ cj, const double* __restrict__ ct, double* __restrict__ epart,
                  long long T, int F, int chunks) {
    constexpr int NV = 3 * S + 3;
    extern __shared__ double sm[];
    __shared__ double red[kBssEnergyTile / 32][NV];
    const int W = kBssEnergyTile + F - 1;
    double* sref = sm;                                  // [S][W]: s_i[tt - F + 1 + q]
    double* sj = sref + (size_t)S * W;                  // [S][F]
    double* st = sj + (size_t)S * F;                    // [S][F]
    const long long b = blockIdx.x / chunks;
    const int chunk = (int)(blockIdx.x - b * chunks);
    const long long L = T + F - 1;
    const long long per = (L + chunks - 1) / chunks;
    const long long t0 = (long long)chunk * per;
    const long long t1 = t0 + per < L ? t0 + per : L;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int e = 0; e < NE; ++e) {
        const float* er = bss_row(ref, est, mix, S, b, S + e, T);
        __syncthreads();
        for (int idx = threadIdx.x; idx < S * F; idx += kBssEnergyTile) {
            sj[idx] = cj[((size_t)b * (S + 1) + e) * S * F + idx];
            st[idx] = ct[((size_t)b * (S + 1) + e) * S * F + idx];
        }
        double acc[NV];
#pragma unroll
        for (int i = 0; i < NV; ++i) acc[i] = 0.0;
        for (long long tt = t0; tt < t1; tt += kBssEnergyTile) {
            __syncthreads();
            for (int idx = threadIdx.x; idx < S * W; idx += kBssEnergyTile) {
                const int i = idx / W, q = idx - i * W;
                const long long t = tt - (F - 1) + q;
                sref[idx] = t >= 0 && t < T ? (double)__ldg(ref + ((size_t)b * S + i) * T + t) : 0.0;
            }
            __syncthreads();
            const long long t = tt + threadIdx.x;
            if (t < t1) {
                double pa = 0.0, pt[S];
#pragma unroll
                for (int i = 0; i < S; ++i) {
                    const double* s = sref + (size_t)i * W + threadIdx.x + F - 1;
                    double p = 0.0;
                    for (int l = 0; l < F; ++l) {
                        const double v = s[-l];
                        pa = fma(sj[i * F + l], v, pa);
                        p = fma(st[i * F + l], v, p);
                    }
                    pt[i] = p;
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
            epart[(((size_t)b * chunks + chunk) * (S + 1) + e) * NV + threadIdx.x] = s;
        }
    }
}

// mir_eval's _safe_db: a zero denominator is +inf
__device__ __forceinline__ double bss_db(double num, double den) {
    return den == 0.0 ? (double)INFINITY : 10.0 * log10(num / den);
}

// one thread per item.  sdr/sir/sar/perm [B][S] for the estimates (perm[j]: the estimate given reference j); with the
// mixture (NE == S + 1), msdr/msir/msar [B][S]: the mixture scored as the estimate of every reference.
template <int S, int NE>
__global__ void __launch_bounds__(256)
bss_final_kernel(const double* __restrict__ epart, const double* __restrict__ eref, int chunks, double* __restrict__ sdr,
                 double* __restrict__ sir, double* __restrict__ sar, int* __restrict__ perm, double* __restrict__ msdr,
                 double* __restrict__ msir, double* __restrict__ msar, int B, int compute_permutation) {
    constexpr int NV = 3 * S + 3;
    for (long long b = blockIdx.x * 256LL + threadIdx.x; b < B; b += (long long)gridDim.x * 256) {
        double en[NE][NV];
#pragma unroll
        for (int e = 0; e < NE; ++e)
#pragma unroll
            for (int i = 0; i < NV; ++i) en[e][i] = 0.0;
        for (int c = 0; c < chunks; ++c) {
            const double* pc = epart + ((size_t)b * chunks + c) * (S + 1) * NV;
#pragma unroll
            for (int e = 0; e < NE; ++e)
#pragma unroll
                for (int i = 0; i < NV; ++i) en[e][i] += pc[e * NV + i];
        }
        bool silent_ref = false;
#pragma unroll
        for (int i = 0; i < S; ++i) silent_ref = silent_ref || !bss_scorable(eref[(size_t)b * S + i]);
        bool silent = silent_ref;
#pragma unroll
        for (int e = 0; e < S; ++e)
            silent = silent || !bss_scorable(en[e][3 * S + 2]) || !bss_projections_hold<S>(en[e]);
        double d[NE][S], i_[NE][S], a[NE][S];
#pragma unroll
        for (int e = 0; e < NE; ++e)
#pragma unroll
            for (int j = 0; j < S; ++j) {
                d[e][j] = bss_db(en[e][j], en[e][S + j]);
                i_[e][j] = bss_db(en[e][j], en[e][2 * S + j]);
                a[e][j] = bss_db(en[e][3 * S], en[e][3 * S + 1]);
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
            double dj = 0.0, ij = 0.0, aj = 0.0;
#pragma unroll
            for (int e = 0; e < S; ++e)
                if (p[j] == e) { dj = d[e][j]; ij = i_[e][j]; aj = a[e][j]; }
            const size_t o = (size_t)b * S + j;
            sdr[o] = silent ? nan : dj;
            sir[o] = silent ? nan : ij;
            sar[o] = silent ? nan : aj;
            if (perm) perm[o] = silent ? -1 : p[j];
            if constexpr (NE > S) {
                const bool ms = silent_ref || !bss_scorable(en[S][3 * S + 2]) || !bss_projections_hold<S>(en[S]);
                msdr[o] = ms ? nan : d[S][j];
                msir[o] = ms ? nan : i_[S][j];
                msar[o] = ms ? nan : a[S][j];
            }
        }
    }
}

template <int S, int NE>
static int bss_eval_launch(const float* ref, const float* est, const float* mix, double* sdr, double* sir,
                           double* sar, int* perm, double* msdr, double* msir, double* msar, int B, long long T, int F,
                           int compute_permutation, void* scratch, cudaStream_t st) {
    const BssScratch s(scratch, B, S, T, F);
    const int cc = bss_corr_chunks(T), ec = bss_energy_chunks(T, F);
    if ((long long)B * cc > 0x7fffffffLL || (long long)B * (S + 1) > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    const size_t corr_smem = sizeof(double) * (S + NE) * (kBssCorrTile + F - 1);
    const size_t solve_smem = sizeof(double) * (size_t)F * (2 * S * S + NE * S);
    const size_t energy_smem = sizeof(double) * (size_t)S * (kBssEnergyTile + F - 1 + 2 * F);
    int e;
    if ((e = launch(bss_corr_kernel<S, NE>, (unsigned)((long long)B * cc), kBssCorrTile, corr_smem, st, ref, est, mix,
                    s.part, T, F, cc)))
        return e;
    if ((e = launch(bss_solve_kernel<S, NE>, (unsigned)((long long)B * (S + 1)), 256, solve_smem, st, s.part, cc, s.rj,
                    s.rt, s.eref, s.cj, s.ct, F)))
        return e;
    if ((e = launch(bss_energy_kernel<S, NE>, (unsigned)((long long)B * ec), kBssEnergyTile, energy_smem, st, ref, est,
                    mix, s.cj, s.ct, s.epart, T, F, ec)))
        return e;
    return launch(bss_final_kernel<S, NE>, item_blocks(B), 256, 0, st, s.epart, s.eref, ec, sdr, sir, sar, perm, msdr,
                  msir, msar, B, compute_permutation);
}

// sdr_bss_eval (mix null) and sdr_bss_eval_mixture
static int bss_eval(const float* ref, const float* est, const float* mix, double* sdr, double* sir, double* sar,
                    int* perm, double* msdr, double* msir, double* msar, int B, int S, long long T, int F,
                    int compute_permutation, void* scratch, cudaStream_t st) {
    if (!ref || !est || !sdr || !sir || !sar || !scratch || reinterpret_cast<uintptr_t>(scratch) % 8)
        return SDR_ERR_BAD_ARGUMENT;
    if (mix && (!msdr || !msir || !msar)) return SDR_ERR_BAD_ARGUMENT;
    if (!sdr_bss_eval_scratch_bytes(B, S, T, F)) return B <= 0 || T <= 0 ? SDR_ERR_BAD_ARGUMENT : SDR_ERR_UNSUPPORTED;
    return with_sources(S, [&](auto s) {
        constexpr int n = decltype(s)::value;
        return mix ? bss_eval_launch<n, n + 1>(ref, est, mix, sdr, sir, sar, perm, msdr, msir, msar, B, T, F,
                                               compute_permutation, scratch, st)
                   : bss_eval_launch<n, n>(ref, est, nullptr, sdr, sir, sar, perm, nullptr, nullptr, nullptr, B, T, F,
                                           compute_permutation, scratch, st);
    });
}

}  // namespace sdr

using namespace sdr;

#pragma GCC visibility push(default)
extern "C" {

size_t sdr_bss_eval_scratch_bytes(int B, int S, int64_t T, int F) {
    if (B <= 0 || S < 1 || S > 4 || T <= 0 || F < 1 || F > kBssMaxF) return 0;
    // S F delayed references in R^(T+F-1): more than the dimensions (T < (S-1) F + 1) makes the joint system singular
    // by construction, where the recursion's rounding no longer separates dependent pivots from independent ones
    if ((long long)S * F > T + F - 1) return 0;
    return BssScratch(nullptr, B, S, T, F).bytes;
}

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

}  // extern "C"
#pragma GCC visibility pop
