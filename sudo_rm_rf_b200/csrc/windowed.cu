// Windowed separation of long recordings (DESIGN.md section 7e): windows of W samples every H samples
// (W/2 <= H < W, so only neighbouring windows overlap), separated in batches by the whole-model entries, each
// window's sources put in the order of the window before it and cross-faded.  Per batch of windows k0 .. k0+M-1:
//   window_gather_kernel    the windows of every recording into the batch [B][M][A][W], zeros past T
//   window_align_kernel     per (recording, window k >= 1): the centred fp64 correlations C_k[i][j] of window k-1's
//                           sources i with window k's sources j over their overlap, and rho_k, the first best
//                           assignment in itertools order (the identity when C_k is not finite)
//   window_scan_kernel      per recording: pi_k = rho_k o pi_{k-1}, from the carried pi of window k0-1
//   window_ola_kernel       the output samples the batch finalises, [k0 H, min((k0+M) H, T)), the permutations
//                           applied on read and overlaps cross-faded
//   window_carry_kernel     window k0+M-1's raw estimate kept for the next batch
// No atomics and fixed-order reductions: bitwise reproducible, and independent of how the windows are batched.
#include "assign.cuh"
#include "launch.cuh"
#include "launchers.cuh"

namespace sdr {

constexpr int kWinThreads = 256;
constexpr long long kWinMaxW = 1LL << 24;     // the cross-fade's (j + 1) / (W - H + 1) is exact in fp32 below this

// The batching of one call: K windows over T samples.
struct WindowPlan {
    bool ok = false;
    long long K = 0;
    WindowPlan(long long T, long long W, long long H) {
        if (T <= 0 || W < 2 || W > kWinMaxW || 2 * H < W || H >= W) return;
        K = T <= W ? 1 : 1 + (T - W + H - 1) / H;
        ok = true;
    }
};

// The carry between two batches: pi of the batch's last window [B][S] (int32), then its raw estimate [B][S A][W].
struct WindowCarry {
    int* pi;
    float* est;
    size_t bytes;
    WindowCarry(void* base, int B, int S, int A, long long W) {
        char* c = static_cast<char*>(base);
        const size_t pi_bytes = ((size_t)B * S * 4 + 255) / 256 * 256;
        pi = reinterpret_cast<int*>(c);
        est = reinterpret_cast<float*>(c ? c + pi_bytes : nullptr);
        bytes = pi_bytes + (size_t)B * S * A * W * 4;
    }
};

// Merge scratch: rho [B][M][S], then pis [B][M+1][S] (pis[b][m] = pi of window k0+m-1), int32.
struct WindowScratch {
    int *rho, *pis;
    size_t bytes;
    WindowScratch(void* base, int B, int S, int M) {
        int* c = static_cast<int*>(base);
        rho = c;
        pis = c ? c + (size_t)B * M * S : nullptr;
        bytes = ((size_t)B * M * S + (size_t)B * (M + 1) * S) * 4;
    }
};

__global__ void __launch_bounds__(kWinThreads)
window_gather_kernel(const float* __restrict__ x, float* __restrict__ batch, long long rows, int M, int A, long long T,
                     long long W, long long H, long long k0) {
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {       // r = (b M + m) A + a
        const long long a = r % A, bm = r / A, m = bm % M, b = bm / M;
        const long long start = (k0 + m) * H;
        const float* src = x + (b * A + a) * T;
        float* dst = batch + r * W;
        for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < W;
             t += (long long)gridDim.x * blockDim.x)
            dst[t] = start + t < T ? src[start + t] : 0.f;
    }
}

// Sums each of the N per-thread values over the CTA: warp shuffles, then the warps in index order.  Every thread gets
// the sums.  `red` holds kWinThreads / 32 * N doubles.
template <int N>
__device__ __forceinline__ void block_sums(double (&v)[N], double* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const double s = warp_sum_f64(v[i]);
        if (lane == 0) red[warp * N + i] = s;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < N; ++i) {
        double s = 0.0;
        for (int w = 0; w < kWinThreads / 32; ++w) s += red[w * N + i];
        v[i] = s;
    }
    __syncthreads();
}

// One CTA per (recording b, window k0 + m).  p = window k-1's rows at H .. H + O - 1, c = window k's rows at 0 .. O-1;
// per channel a, the means over the overlap, then the centred cross products, summed over a in order.
template <int S>
__global__ void __launch_bounds__(kWinThreads)
window_align_kernel(const float* __restrict__ est, const float* __restrict__ carry_est, int* __restrict__ rho, int B,
                    int M, int A, long long T, long long W, long long H, long long k0) {
    __shared__ double red[kWinThreads / 32 * S * S];
    const long long bm = blockIdx.x;
    const long long b = bm / M, m = bm % M, k = k0 + m;
    int* out = rho + bm * S;
    if (k == 0 || S == 1) {        // pi_0 is the identity; one source has nothing to search
        if (threadIdx.x < S) out[threadIdx.x] = threadIdx.x;
        return;
    }
    const long long SA = (long long)S * A;
    const long long O = min(W - H, T - k * H);
    const float* prev = (m == 0 ? carry_est + b * SA * W : est + (bm - 1) * SA * W) + H;
    const float* cur = est + bm * SA * W;
    double C[S][S];
#pragma unroll
    for (int i = 0; i < S; ++i)
#pragma unroll
        for (int j = 0; j < S; ++j) C[i][j] = 0.0;
    for (int a = 0; a < A; ++a) {
        double mean[2 * S];
#pragma unroll
        for (int i = 0; i < 2 * S; ++i) mean[i] = 0.0;
        for (long long t = threadIdx.x; t < O; t += kWinThreads) {
#pragma unroll
            for (int i = 0; i < S; ++i) {
                mean[i] += (double)prev[(i * A + a) * W + t];
                mean[S + i] += (double)cur[(i * A + a) * W + t];
            }
        }
        block_sums(mean, red);
#pragma unroll
        for (int i = 0; i < 2 * S; ++i) mean[i] /= (double)O;
        double acc[S * S];
#pragma unroll
        for (int i = 0; i < S * S; ++i) acc[i] = 0.0;
        for (long long t = threadIdx.x; t < O; t += kWinThreads) {
            double pc[S], cc[S];
#pragma unroll
            for (int i = 0; i < S; ++i) {
                pc[i] = (double)prev[(i * A + a) * W + t] - mean[i];
                cc[i] = (double)cur[(i * A + a) * W + t] - mean[S + i];
            }
#pragma unroll
            for (int i = 0; i < S; ++i)
#pragma unroll
                for (int j = 0; j < S; ++j) acc[i * S + j] = fma(pc[i], cc[j], acc[i * S + j]);
        }
        block_sums(acc, red);
#pragma unroll
        for (int i = 0; i < S; ++i)
#pragma unroll
            for (int j = 0; j < S; ++j) C[i][j] += acc[i * S + j];
    }
    if (threadIdx.x != 0) return;
    bool finite = true;
#pragma unroll
    for (int i = 0; i < S; ++i)
#pragma unroll
        for (int j = 0; j < S; ++j) finite = finite && isfinite(C[i][j]);
    int p[S];
#pragma unroll
    for (int i = 0; i < S; ++i) p[i] = i;
    if (finite) {
        int idx = 0;
        best_assignment<S, S>(
            [&](const int (&q)[S]) {
                double s = C[0][q[0]];
#pragma unroll
                for (int i = 1; i < S; ++i) s = __dadd_rn(s, C[i][q[i]]);
                return s;
            },
            idx, p);
    }
#pragma unroll
    for (int i = 0; i < S; ++i) out[i] = p[i];
}

// One thread per recording: pi_{k0-1} (the identity before window 0) composed with rho_k0 .. rho_{k0+M-1}.
__global__ void window_scan_kernel(const int* __restrict__ rho, int* __restrict__ pis, int* __restrict__ carry_pi,
                                   int* __restrict__ perm, int B, int S, int M, long long K, long long k0) {
    const long long b = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (b >= B) return;
    int pi[4];
    for (int s = 0; s < S; ++s) pi[s] = k0 == 0 ? s : carry_pi[b * S + s];
    for (int s = 0; s < S; ++s) pis[b * (M + 1) * S + s] = pi[s];
    for (int m = 0; m < M; ++m) {
        const int* r = rho + (b * M + m) * S;
        for (int s = 0; s < S; ++s) pi[s] = r[pi[s]];
        for (int s = 0; s < S; ++s) pis[(b * (M + 1) + m + 1) * S + s] = pi[s];
        if (perm)
            for (int s = 0; s < S; ++s) perm[(b * K + k0 + m) * S + s] = pi[s];
    }
    for (int s = 0; s < S; ++s) carry_pi[b * S + s] = pi[s];
}

// The cross-fade of overlap sample j (0 <= j < W - H): the weights 1 - r and r sum to one, so it needs no division by
// their sum.  tests/windowed_oracle.py computes the same fp32 operations.
__device__ __forceinline__ float window_fade(float prev, float cur, long long j, long long overlap) {
    const float r = __fdiv_rn((float)(j + 1), (float)(overlap + 1));
    return __fadd_rn(__fmul_rn(__fsub_rn(1.f, r), prev), __fmul_rn(r, cur));
}

// Row r = (b, s, a) of the output over [t0, t1): sample t takes window k = min(t / H, K - 1) (its latest window) and,
// when t also lies in window k - 1, the cross-fade of the two; source s of window k is raw source pi_k(s).
__global__ void __launch_bounds__(kWinThreads)
window_ola_kernel(const float* __restrict__ est, const float* __restrict__ carry_est, const int* __restrict__ pis,
                  float* __restrict__ out, long long rows, int S, int A, int M, long long T, long long W, long long H,
                  long long K, long long k0, long long t0, long long t1) {
    const long long SA = (long long)S * A;
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {
        const long long a = r % A, s = (r / A) % S, b = r / SA;
        const int* pb = pis + b * (M + 1) * S;
        for (long long t = t0 + blockIdx.x * (long long)blockDim.x + threadIdx.x; t < t1;
             t += (long long)gridDim.x * blockDim.x) {
            const long long k = min(t / H, K - 1), j = t - k * H, m = k - k0;
            const float c = est[((b * M + m) * SA + (long long)pb[(m + 1) * S + s] * A + a) * W + j];
            float v = c;
            if (k > 0 && j < W - H) {
                const long long row = (long long)pb[m * S + s] * A + a;
                const float p = m == 0 ? carry_est[(b * SA + row) * W + H + j]
                                       : est[((b * M + m - 1) * SA + row) * W + H + j];
                v = window_fade(p, c, j, W - H);
            }
            out[r * T + t] = v;
        }
    }
}

__global__ void __launch_bounds__(kWinThreads)
window_carry_kernel(const float* __restrict__ est, float* __restrict__ carry_est, long long rows, long long SA, int M,
                    long long W) {
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {       // r = b SA + row
        const float* src = est + ((r / SA * M + M - 1) * SA + r % SA) * W;
        for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < W;
             t += (long long)gridDim.x * blockDim.x)
            carry_est[r * W + t] = src[t];
    }
}

long long window_count(long long T, long long W, long long H) {
    const WindowPlan g(T, W, H);
    return g.ok ? g.K : 0;
}

size_t window_carry_bytes(int B, int S, int A, long long W) {
    if (B <= 0 || S <= 0 || S > 4 || A <= 0 || W < 2 || W > kWinMaxW) return 0;
    return WindowCarry(nullptr, B, S, A, W).bytes;
}

size_t window_merge_scratch_bytes(int B, int S, int M) {
    if (B <= 0 || S <= 0 || S > 4 || M <= 0) return 0;
    return WindowScratch(nullptr, B, S, M).bytes;
}

int launch_window_gather(const float* x, float* batch, int B, int A, long long T, long long W, long long H,
                         long long k0, int M, cudaStream_t st) {
    if (!x || !batch) return SDR_ERR_BAD_ARGUMENT;
    const WindowPlan g(T, W, H);
    if (!g.ok || B <= 0 || A <= 0 || M <= 0 || k0 < 0 || k0 + M > g.K) return SDR_ERR_BAD_ARGUMENT;
    const long long rows = (long long)B * M * A;
    return launch(window_gather_kernel, row_tiled_grid(rows, W), kWinThreads, 0, st, x, batch, rows, M, A, T, W, H,
                  k0);
}

int launch_window_merge(const float* est, void* carry, int* perm, float* out, int B, int S, int A, long long T,
                        long long W, long long H, long long k0, int M, void* scratch, cudaStream_t st) {
    if (!est || !carry || !out || !scratch) return SDR_ERR_BAD_ARGUMENT;
    if (reinterpret_cast<uintptr_t>(carry) % 256 || reinterpret_cast<uintptr_t>(scratch) % 8)
        return SDR_ERR_BAD_ARGUMENT;
    if (S > 4) return SDR_ERR_UNSUPPORTED;
    const WindowPlan g(T, W, H);
    if (!g.ok || B <= 0 || S <= 0 || A <= 0 || M <= 0 || k0 < 0 || k0 + M > g.K) return SDR_ERR_BAD_ARGUMENT;
    const WindowCarry c(carry, B, S, A, W);
    const WindowScratch s(scratch, B, S, M);
    int e = with_sources(S, [&](auto sc) {
        return launch(window_align_kernel<decltype(sc)::value>, (unsigned)((long long)B * M), kWinThreads, 0, st, est,
                      c.est, s.rho, B, M, A, T, W, H, k0);
    });
    if (e) return e;
    if ((e = launch(window_scan_kernel, (unsigned)((B + 127) / 128), 128, 0, st, s.rho, s.pis, c.pi, perm, B, S, M,
                    g.K, k0)))
        return e;
    const long long t0 = k0 * H, t1 = k0 + M == g.K ? T : (k0 + M) * H;
    const long long rows = (long long)B * S * A;
    if ((e = launch(window_ola_kernel, row_tiled_grid(rows, t1 - t0), kWinThreads, 0, st, est, c.est, s.pis, out,
                    rows, S, A, M, T, W, H, g.K, k0, t0, t1)))
        return e;
    return launch(window_carry_kernel, row_tiled_grid(rows, W), kWinThreads, 0, st, est, c.est, rows,
                  (long long)S * A, M, W);
}

}  // namespace sdr
