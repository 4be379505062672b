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
//
// A windowed stream (DESIGN.md section 7f) runs the same align / scan / overlap-add / carry kernels on each step's
// q = C / H windows, with every slot's own window origin read from its counter on the device (WinOrigin), and its
// output origin at the step's first output sample.  Its state per slot is the carry, the last H input samples and
// the counter c (c H samples received since the slot's reset):
//   window_stream_gather_kernel   windows c-1 .. c+q-2 out of [history | chunk] into [B][q][A][W] (zeros below 0)
//   window_stream_history_kernel  the chunk's last H samples become the history
//
// A corpus of recordings of different lengths (DESIGN.md section 7i) shares window batches: slot m of a batch holds
// global window g0 + m, window k of the recording whose descriptor it finds (RaggedOrigin).  The align and scan
// kernels take that origin in place of WinOrigin; window_gather_ragged_kernel and window_ola_ragged_kernel gather and
// overlap-add per slot, the latter through the same window_value as window_ola_kernel.
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

// A stream's state: the carry, then the history [B][A][H] fp32, then the window counters [B] (int64), each region
// starting on a 256-byte boundary.
struct WindowStreamState {
    WindowCarry carry;
    float* hist;
    long long* count;
    size_t hist_off, count_off, bytes;
    WindowStreamState(void* base, int B, int S, int A, long long W, long long H) : carry(base, B, S, A, W) {
        char* c = static_cast<char*>(base);
        hist_off = (carry.bytes + 255) / 256 * 256;         // every region 256-byte aligned (the counters are int64)
        count_off = hist_off + ((size_t)B * A * H * 4 + 255) / 256 * 256;
        bytes = count_off + (size_t)B * 8;
        hist = reinterpret_cast<float*>(c ? c + hist_off : nullptr);
        count = reinterpret_cast<long long*>(c ? c + count_off : nullptr);
    }
};

__host__ __device__ __forceinline__ long long win_count(long long T, long long W, long long H) {
    return T <= W ? 1 : 1 + (T - W + H - 1) / H;
}

// Where a batch lies in each recording: windows k0 .. k0+M-1 of a recording of T samples.  The offline merge gives
// every recording the same k0 and T.  A stream reads each slot's counter c: k0 = c + dk and T = c H + dT.
// at(b, m, k, T): window m of recording b's batch is its window k, of a recording of T samples; false when the slot
// holds no window (never, here).  perm_row: the row of perm [B][K][S] that window takes.
struct WinOrigin {
    const long long* count;
    long long k0, T;
    __device__ __forceinline__ long long first(long long b) const { return count ? count[b] + k0 : k0; }
    __device__ __forceinline__ long long length(long long b, long long H) const {
        return count ? count[b] * H + T : T;
    }
    __device__ __forceinline__ bool at(long long b, long long m, long long H, long long& k, long long& t) const {
        k = first(b) + m;
        t = length(b, H);
        return true;
    }
    __device__ __forceinline__ long long perm_row(long long b, long long m, long long K) const {
        return b * K + first(b) + m;
    }
};
constexpr long long kWinUnbounded = 1LL << 62;   // a stream step's T: every window it merges overlaps in full

// A corpus of recordings of different lengths (DESIGN.md section 7i): recording r's first sample per channel in the
// flat buffers (its mixture [A][T] at A off, its output [S A][T] at S A off), its length T and its first global window
// g, ascending in r.  The layout of the C-ABI's int64 descriptor [R][3].
struct WinRec {
    long long off, T, g;
};

// A ragged batch (B = 1): slot m holds global window g0 + m, window k = g0 + m - g of the last recording whose first
// window g is at or below it.  A slot past the corpus's last window holds none.
struct RaggedOrigin {
    const WinRec* desc;
    int R;
    long long g0, W, H;
    __device__ __forceinline__ bool slot(long long m, WinRec& d, long long& k) const {
        const long long g = g0 + m;
        int lo = 0, hi = R - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (desc[mid].g <= g) lo = mid; else hi = mid - 1;
        }
        d = desc[lo];
        k = g - d.g;
        return k >= 0 && k < win_count(d.T, W, H);
    }
    __device__ __forceinline__ bool at(long long, long long m, long long, long long& k, long long& t) const {
        WinRec d;
        const bool ok = slot(m, d, k);
        t = d.T;
        return ok;
    }
    __device__ __forceinline__ long long perm_row(long long, long long m, long long) const { return g0 + m; }
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

// One CTA per (recording b, window k0 + m), or per slot m of a ragged batch.  p = window k-1's rows at H .. H + O - 1,
// c = window k's rows at 0 .. O-1; per channel a, the means over the overlap, then the centred cross products, summed
// over a in order.
template <int S, class Org>
__global__ void __launch_bounds__(kWinThreads)
window_align_kernel(const float* __restrict__ est, const float* __restrict__ carry_est, int* __restrict__ rho, int B,
                    int M, int A, long long W, long long H, Org org) {
    __shared__ double red[kWinThreads / 32 * S * S];
    const long long bm = blockIdx.x;
    const long long b = bm / M, m = bm % M;
    long long k, T;
    const bool valid = org.at(b, m, H, k, T);
    int* out = rho + bm * S;
    // pi_0 is the identity; one source has nothing to search; a stream's window below 0 or past its last is never read
    if (!valid || k <= 0 || k >= win_count(T, W, H) || S == 1) {
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

// One thread per recording (one for a ragged batch): pi_{k0-1} (the identity before window 0) composed with
// rho_k0 .. rho_{k0+M-1}; the composition restarts from the identity at every recording's window 0.  carry_out
// (null: left as it is) receives the last; it may be carry_in.
template <class Org>
__global__ void window_scan_kernel(const int* __restrict__ rho, int* __restrict__ pis, const int* carry_in,
                                   int* carry_out, int* __restrict__ perm, int B, int S, int M, long long K, long long H,
                                   Org org) {
    const long long b = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (b >= B) return;
    long long k, T;
    bool valid = org.at(b, 0, H, k, T);
    int pi[4];
    for (int s = 0; s < S; ++s) pi[s] = !valid || k <= 0 ? s : carry_in[b * S + s];
    for (int s = 0; s < S; ++s) pis[b * (M + 1) * S + s] = pi[s];
    for (int m = 0; m < M; ++m) {
        valid = org.at(b, m, H, k, T);
        if (!valid || k <= 0)
            for (int s = 0; s < S; ++s) pi[s] = s;
        const int* r = rho + (b * M + m) * S;
        for (int s = 0; s < S; ++s) pi[s] = r[pi[s]];
        for (int s = 0; s < S; ++s) pis[(b * (M + 1) + m + 1) * S + s] = pi[s];
        if (perm && valid)
            for (int s = 0; s < S; ++s) perm[org.perm_row(b, m, K) * S + s] = pi[s];
    }
    if (carry_out)
        for (int s = 0; s < S; ++s) carry_out[b * S + s] = pi[s];
}

// The cross-fade of overlap sample j (0 <= j < W - H): the weights 1 - r and r sum to one, so it needs no division by
// their sum.  tests/windowed_oracle.py computes the same fp32 operations.
__device__ __forceinline__ float window_fade(float prev, float cur, long long j, long long overlap) {
    const float r = __fdiv_rn((float)(j + 1), (float)(overlap + 1));
    return __fadd_rn(__fmul_rn(__fsub_rn(1.f, r), prev), __fmul_rn(r, cur));
}

// Sample j of window k's output source s, channel a: raw source pi_k(s) of `cur` and, inside overlap k (k > 0 and
// j < W - H), its cross-fade with raw source pi_{k-1}(s) of `prev` at H + j.  cur, prev: estimates [S A][W].
__device__ __forceinline__ float window_value(const float* cur, const float* prev, const int* pi_cur,
                                              const int* pi_prev, long long s, long long a, long long A, long long j,
                                              bool overlap, long long W, long long H) {
    const float c = cur[((long long)pi_cur[s] * A + a) * W + j];
    if (!overlap) return c;
    const float p = prev[((long long)pi_prev[s] * A + a) * W + H + j];
    return window_fade(p, c, j, W - H);
}

// Row r = (b, s, a) of the output over samples t = k0 H + u, 0 <= u < len: t takes window k = min(t / H, K - 1) (its
// latest window) and, when t also lies in window k - 1, the cross-fade of the two; source s of window k is raw source
// pi_k(s), and window k0 - 1 is the carry.  Sample t goes to out[r ld + o0 + u].  A stream's samples below 0 are 0,
// and `single` (a stream's flush, null otherwise) holds the whole-recording estimate [B][S A][len] of a slot that is
// one window long and starts at window 0.
__global__ void __launch_bounds__(kWinThreads)
window_ola_kernel(const float* __restrict__ est, const float* __restrict__ carry_est, const int* __restrict__ pis,
                  const float* __restrict__ single, float* __restrict__ out, long long rows, int S, int A, int M,
                  long long W, long long H, WinOrigin org, long long len, long long ld, long long o0) {
    const long long SA = (long long)S * A;
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {
        const long long a = r % A, s = (r / A) % S, b = r / SA;
        const long long k0 = org.first(b), T = org.length(b, H), K = win_count(T, W, H);
        const int* pb = pis + b * (M + 1) * S;
        const float* raw = est + b * M * SA * W;             // window k0 + m of recording b (m = -1: the carry)
        const float* car = carry_est + b * SA * W;
        for (long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x; u < len;
             u += (long long)gridDim.x * blockDim.x) {
            const long long k = min(k0 + u / H, K - 1), j = k0 * H + u - k * H, m = k - k0;
            float v = 0.f;
            if (single && k0 == 0 && T <= W) {
                v = single[r * len + u];
            } else if (k >= 0) {
                // an overlap lies in window k0 or later: m >= 0 wherever `prev` is read
                v = window_value(m < 0 ? car : raw + m * SA * W, m <= 0 ? car : raw + (m - 1) * SA * W,
                                 pb + (m + 1) * S, pb + max(m, 0LL) * S, s, a, A, j, k > 0 && j < W - H, W, H);
            }
            out[r * ld + o0 + u] = v;
        }
    }
}

// Also advances a stream's counters (null: none) by `advance` windows, after every kernel that reads them.
__global__ void __launch_bounds__(kWinThreads)
window_carry_kernel(const float* __restrict__ est, float* __restrict__ carry_est, long long rows, long long SA, int M,
                    long long W, long long* __restrict__ count, long long advance) {
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {       // r = b SA + row
        const float* src = est + ((r / SA * M + M - 1) * SA + r % SA) * W;
        for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < W;
             t += (long long)gridDim.x * blockDim.x)
            carry_est[r * W + t] = src[t];
        if (count && r % SA == 0 && blockIdx.x == 0 && threadIdx.x == 0) count[r / SA] += advance;
    }
}

// Window m of slot b's step is window c - 1 + m, samples [m H, m H + W) of [history (H) | chunk (C)]; zeros below
// window 0.  chunk = null (C = 0, q = 1): the flush's window, the history followed by zeros.
__global__ void __launch_bounds__(kWinThreads)
window_stream_gather_kernel(const float* __restrict__ hist, const float* __restrict__ chunk,
                            const long long* __restrict__ count, float* __restrict__ batch, long long rows, int q,
                            int A, long long C, long long W, long long H) {
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {       // r = (b q + m) A + a
        const long long a = r % A, bm = r / A, m = bm % q, b = bm / q;
        const bool valid = count[b] - 1 + m >= 0;
        const float* h = hist + (b * A + a) * H;
        const float* x = chunk ? chunk + (b * A + a) * C : nullptr;
        float* dst = batch + r * W;
        for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < W;
             t += (long long)gridDim.x * blockDim.x) {
            const long long p = m * H + t;
            dst[t] = !valid ? 0.f : p < H ? h[p] : x && p - H < C ? x[p - H] : 0.f;
        }
    }
}

__global__ void __launch_bounds__(kWinThreads)
window_stream_history_kernel(const float* __restrict__ chunk, float* __restrict__ hist, long long rows, long long C,
                             long long H) {
    for (long long r = blockIdx.y; r < rows; r += gridDim.y)         // r = b A + a
        for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < H;
             t += (long long)gridDim.x * blockDim.x)
            hist[r * H + t] = chunk[r * C + C - H + t];
}

// Align, scan and overlap-add windows org.first(b) .. + M - 1 of every recording.  `single` non-null: a stream's flush,
// which leaves the carry as it is.  Otherwise the carry receives the batch's last window and a stream's counters
// (null for the offline merge) advance by `advance`.
static int merge_stages(const float* est, const WindowCarry& c, const float* single, int* perm, float* out, int B,
                        int S, int A, long long W, long long H, int M, WinOrigin org, long long K, long long len,
                        long long ld, long long o0, void* scratch, long long* count, long long advance,
                        cudaStream_t st) {
    const WindowScratch s(scratch, B, S, M);
    int e = with_sources(S, [&](auto sc) {
        return launch(window_align_kernel<decltype(sc)::value, WinOrigin>, (unsigned)((long long)B * M), kWinThreads,
                      0, st, est, c.est, s.rho, B, M, A, W, H, org);
    });
    if (e) return e;
    if ((e = launch(window_scan_kernel<WinOrigin>, (unsigned)((B + 127) / 128), 128, 0, st, s.rho, s.pis, c.pi,
                    single ? nullptr : c.pi, perm, B, S, M, K, H, org)))
        return e;
    const long long rows = (long long)B * S * A;
    if ((e = launch(window_ola_kernel, row_tiled_grid(rows, len), kWinThreads, 0, st, est, c.est, s.pis, single, out,
                    rows, S, A, M, W, H, org, len, ld, o0)))
        return e;
    if (single) return SDR_OK;
    return launch(window_carry_kernel, row_tiled_grid(rows, W), kWinThreads, 0, st, est, c.est, rows,
                  (long long)S * A, M, W, count, advance);
}

// ---- a corpus of recordings in shared window batches (DESIGN.md section 7i) -------------------------------------

// Row (m, a) of the batch [M][A][W]: window k of slot m's recording, zeros past its T and for a slot past the corpus.
__global__ void __launch_bounds__(kWinThreads)
window_gather_ragged_kernel(const float* __restrict__ x, float* __restrict__ batch, long long rows, int A, long long W,
                            RaggedOrigin org) {
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {       // r = m A + a
        const long long a = r % A, m = r / A;
        WinRec d;
        long long k;
        const bool valid = org.slot(m, d, k);
        const long long start = k * org.H;
        const float* src = x + (A * d.off + a * d.T);
        float* dst = batch + r * W;
        for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < W;
             t += (long long)gridDim.x * blockDim.x)
            dst[t] = valid && start + t < d.T ? src[start + t] : 0.f;
    }
}

// Row (m, s, a) of a ragged batch: the samples slot m's window k finalises, [k H, (k + 1) H), or up to T in its
// recording's last window, each as window_ola_kernel computes it; slot m - 1 (the carry for m = 0) is window k - 1
// wherever k > 0.  Sample t of row s A + a of recording r goes to out[S A off + (s A + a) T + t].
__global__ void __launch_bounds__(kWinThreads)
window_ola_ragged_kernel(const float* __restrict__ est, const float* __restrict__ carry_est,
                         const int* __restrict__ pis, float* __restrict__ out, long long rows, int S, int A,
                         RaggedOrigin org) {
    const long long SA = (long long)S * A, W = org.W, H = org.H;
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {       // r = (m S + s) A + a
        const long long a = r % A, s = (r / A) % S, m = r / SA;
        WinRec d;
        long long k;
        if (!org.slot(m, d, k)) continue;
        const long long len = k == win_count(d.T, W, H) - 1 ? d.T - k * H : H;
        const float* cur = est + m * SA * W;
        const float* prev = m == 0 ? carry_est : cur - SA * W;
        float* dst = out + (SA * d.off + (s * A + a) * d.T + k * H);
        for (long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x; u < len;
             u += (long long)gridDim.x * blockDim.x)
            dst[u] = window_value(cur, prev, pis + (m + 1) * S, pis + m * S, s, a, A, u, k > 0 && u < W - H, W, H);
    }
}

// ---- windowed stream (DESIGN.md section 7f) ----------------------------------------------------------------------

// SDR_OK, or the refusal of a bad shape (more than 4 sources: unsupported) or of a state off a 256-byte boundary.
static int stream_refusal(const void* state, int B, int S, int A, long long W, long long H) {
    if (!(B > 0 && S > 0 && S <= 4 && A > 0 && WindowPlan(W + 1, W, H).ok))
        return S > 4 ? SDR_ERR_UNSUPPORTED : SDR_ERR_BAD_ARGUMENT;
    return reinterpret_cast<uintptr_t>(state) % 256 ? SDR_ERR_BAD_ARGUMENT : SDR_OK;
}

// Zeroes the whole state (neither slots nor mask given) or each chosen slot's pi, carried estimate, history and
// counter.  The counter alone decides what a step reads; the rest is zeroed for hygiene.
static int reset_stream(void* state, int B, int S, int A, long long W, long long H, const int* slots, int n,
                        const unsigned char* mask, cudaStream_t st) {
    if (const int e = stream_refusal(state, B, S, A, W, H)) return e;
    const WindowStreamState ss(state, B, S, A, W, H);
    if (!slots && !mask) return cuda_status(cudaMemsetAsync(state, 0, ss.bytes, st));
    return reset_slots({{ss.carry.pi, (size_t)S * 4}, {ss.carry.est, (size_t)S * A * W * 4},
                        {ss.hist, (size_t)A * H * 4}, {ss.count, 8}},
                       B, slots, n, mask, st);
}

}  // namespace sdr

using namespace sdr;

#pragma GCC visibility push(default)
extern "C" {

int64_t sdr_window_count(int64_t T, int64_t W, int64_t H) {
    const WindowPlan g(T, W, H);
    return g.ok ? g.K : 0;
}

size_t sdr_window_carry_bytes(int B, int S, int A, int64_t W) {
    if (B <= 0 || S <= 0 || S > 4 || A <= 0 || W < 2 || W > kWinMaxW) return 0;
    return WindowCarry(nullptr, B, S, A, W).bytes;
}

size_t sdr_window_merge_scratch_bytes(int B, int S, int M) {
    if (B <= 0 || S <= 0 || S > 4 || M <= 0) return 0;
    return WindowScratch(nullptr, B, S, M).bytes;
}

int sdr_window_gather(const float* x, float* batch, int B, int A, int64_t T, int64_t W, int64_t H, int64_t k0, int M,
                      sdr_stream stream) {
    if (!x || !batch) return SDR_ERR_BAD_ARGUMENT;
    const WindowPlan g(T, W, H);
    if (!g.ok || B <= 0 || A <= 0 || M <= 0 || k0 < 0 || k0 + M > g.K) return SDR_ERR_BAD_ARGUMENT;
    const long long rows = (long long)B * M * A;
    return launch(window_gather_kernel, row_tiled_grid(rows, W), kWinThreads, 0, static_cast<cudaStream_t>(stream), x,
                  batch, rows, M, A, T, W, H, k0);
}

int sdr_window_merge(const float* est, void* carry, int32_t* perm, float* out, int B, int S, int A, int64_t T,
                     int64_t W, int64_t H, int64_t k0, int M, void* scratch, sdr_stream stream) {
    if (!est || !carry || !out || !scratch) return SDR_ERR_BAD_ARGUMENT;
    if (reinterpret_cast<uintptr_t>(carry) % 256 || reinterpret_cast<uintptr_t>(scratch) % 8)
        return SDR_ERR_BAD_ARGUMENT;
    if (S > 4) return SDR_ERR_UNSUPPORTED;
    const WindowPlan g(T, W, H);
    if (!g.ok || B <= 0 || S <= 0 || A <= 0 || M <= 0 || k0 < 0 || k0 + M > g.K) return SDR_ERR_BAD_ARGUMENT;
    const WindowCarry c(carry, B, S, A, W);
    const long long t0 = k0 * H, t1 = k0 + M == g.K ? T : (k0 + M) * H;
    return merge_stages(est, c, nullptr, perm, out, B, S, A, W, H, M, WinOrigin{nullptr, k0, T}, g.K, t1 - t0, T, t0,
                        scratch, nullptr, 0, static_cast<cudaStream_t>(stream));
}

size_t sdr_window_ragged_carry_bytes(int S, int A, int64_t W) { return sdr_window_carry_bytes(1, S, A, W); }

size_t sdr_window_ragged_scratch_bytes(int S, int M) { return sdr_window_merge_scratch_bytes(1, S, M); }

int sdr_window_gather_ragged(const float* x, const int64_t* desc, int R, int A, int64_t W, int64_t H, int64_t g0,
                             int M, float* batch, sdr_stream stream) {
    if (!x || !desc || !batch || reinterpret_cast<uintptr_t>(desc) % 8) return SDR_ERR_BAD_ARGUMENT;
    if (!WindowPlan(W + 1, W, H).ok || R <= 0 || A <= 0 || M <= 0 || g0 < 0) return SDR_ERR_BAD_ARGUMENT;
    const RaggedOrigin org{reinterpret_cast<const WinRec*>(desc), R, g0, W, H};
    const long long rows = (long long)M * A;
    return launch(window_gather_ragged_kernel, row_tiled_grid(rows, W), kWinThreads, 0,
                  static_cast<cudaStream_t>(stream), x, batch, rows, A, W, org);
}

int sdr_window_merge_ragged(const float* est, const int64_t* desc, int R, void* carry, int32_t* perm, float* out,
                            int S, int A, int64_t W, int64_t H, int64_t g0, int M, void* scratch, sdr_stream stream) {
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!est || !desc || !carry || !out || !scratch) return SDR_ERR_BAD_ARGUMENT;
    if (reinterpret_cast<uintptr_t>(carry) % 256 || reinterpret_cast<uintptr_t>(scratch) % 8 ||
        reinterpret_cast<uintptr_t>(desc) % 8)
        return SDR_ERR_BAD_ARGUMENT;
    if (S > 4) return SDR_ERR_UNSUPPORTED;
    if (!WindowPlan(W + 1, W, H).ok || R <= 0 || S <= 0 || A <= 0 || M <= 0 || g0 < 0) return SDR_ERR_BAD_ARGUMENT;
    const RaggedOrigin org{reinterpret_cast<const WinRec*>(desc), R, g0, W, H};
    const WindowCarry c(carry, 1, S, A, W);
    const WindowScratch s(scratch, 1, S, M);
    // the stages of merge_stages with B = 1, each slot's window and recording looked up in the descriptors
    int e = with_sources(S, [&](auto sc) {
        return launch(window_align_kernel<decltype(sc)::value, RaggedOrigin>, (unsigned)M, kWinThreads, 0, st, est,
                      c.est, s.rho, 1, M, A, W, H, org);
    });
    if (e) return e;
    if ((e = launch(window_scan_kernel<RaggedOrigin>, 1u, 128, 0, st, s.rho, s.pis, c.pi, c.pi, perm, 1, S, M, 0LL, H,
                    org)))
        return e;
    const long long rows = (long long)M * S * A;
    if ((e = launch(window_ola_ragged_kernel, row_tiled_grid(rows, W), kWinThreads, 0, st, est, c.est, s.pis, out,
                    rows, S, A, org)))
        return e;
    return launch(window_carry_kernel, row_tiled_grid((long long)S * A, W), kWinThreads, 0, st, est, c.est,
                  (long long)S * A, (long long)S * A, M, W, nullptr, 0LL);
}

size_t sdr_window_stream_state_bytes(int B, int S, int A, int64_t W, int64_t H) {
    if (stream_refusal(nullptr, B, S, A, W, H)) return 0;
    return WindowStreamState(nullptr, B, S, A, W, H).bytes;
}

int sdr_window_stream_reset(void* state, int B, int S, int A, int64_t W, int64_t H, const int32_t* slots, int n,
                            sdr_stream stream) {
    if (!state || (slots && n < 0)) return SDR_ERR_BAD_ARGUMENT;
    return reset_stream(state, B, S, A, W, H, slots, n, nullptr, static_cast<cudaStream_t>(stream));
}

// sdr_window_stream_reset of the slots whose mask[b] is set, the mask read on the device.
int sdr_window_stream_reset_masked(void* state, int B, int S, int A, int64_t W, int64_t H, const uint8_t* mask,
                                   sdr_stream stream) {
    if (!state || !mask) return SDR_ERR_BAD_ARGUMENT;
    return reset_stream(state, B, S, A, W, H, nullptr, 0, mask, static_cast<cudaStream_t>(stream));
}

// C = 0 with chunk null: the flush's window [B][A][W]; nothing in the state changes.
int sdr_window_stream_gather(void* state, const float* chunk, float* batch, int B, int S, int A, int64_t C, int64_t W,
                             int64_t H, sdr_stream stream) {
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!state || !batch || (!chunk && C != 0)) return SDR_ERR_BAD_ARGUMENT;
    if (const int e = stream_refusal(state, B, S, A, W, H)) return e;
    if (chunk && (C <= 0 || C % H)) return SDR_ERR_BAD_ARGUMENT;
    const WindowStreamState ss(state, B, S, A, W, H);
    const int q = chunk ? (int)(C / H) : 1;
    const long long rows = (long long)B * q * A;
    int e = launch(window_stream_gather_kernel, row_tiled_grid(rows, W), kWinThreads, 0, st, ss.hist, chunk, ss.count,
                   batch, rows, q, A, C, W, H);
    if (e || !chunk) return e;
    return launch(window_stream_history_kernel, row_tiled_grid((long long)B * A, H), kWinThreads, 0, st, chunk,
                  ss.hist, (long long)B * A, C, H);
}

size_t sdr_window_stream_merge_scratch_bytes(int B, int S, int64_t C, int64_t H) {
    if (B <= 0 || S <= 0 || S > 4 || H <= 0 || C <= 0 || C % H || C / H > (1 << 30)) return 0;
    return WindowScratch(nullptr, B, S, (int)(C / H)).bytes;
}

int sdr_window_stream_merge(const float* est, void* state, float* out, int B, int S, int A, int64_t C, int64_t W,
                            int64_t H, void* scratch, sdr_stream stream) {
    if (!est || !state || !out || !scratch) return SDR_ERR_BAD_ARGUMENT;
    if (const int e = stream_refusal(state, B, S, A, W, H)) return e;
    if (sdr_window_stream_merge_scratch_bytes(B, S, C, H) == 0 || reinterpret_cast<uintptr_t>(scratch) % 8)
        return SDR_ERR_BAD_ARGUMENT;
    WindowStreamState ss(state, B, S, A, W, H);
    const int q = (int)(C / H);
    return merge_stages(est, ss.carry, nullptr, nullptr, out, B, S, A, W, H, q, WinOrigin{ss.count, -1, kWinUnbounded},
                        kWinUnbounded, C, C, 0, scratch, ss.count, q, static_cast<cudaStream_t>(stream));
}

size_t sdr_window_stream_flush_scratch_bytes(int B, int S) { return sdr_window_merge_scratch_bytes(B, S, 1); }

int sdr_window_stream_flush(const float* single, const float* est, const void* state, float* out, int B, int S, int A,
                            int64_t W, int64_t H, void* scratch, sdr_stream stream) {
    if (!single || !state || !out || !scratch || (!est && W < 2 * H)) return SDR_ERR_BAD_ARGUMENT;
    if (const int e = stream_refusal(state, B, S, A, W, H)) return e;
    if (reinterpret_cast<uintptr_t>(scratch) % 8) return SDR_ERR_BAD_ARGUMENT;
    // the state is only read: the carry's pi is not written when `single` is given
    WindowStreamState ss(const_cast<void*>(state), B, S, A, W, H);
    return merge_stages(est, ss.carry, single, nullptr, out, B, S, A, W, H, 1, WinOrigin{ss.count, -1, 0}, 0, H, H, 0,
                        scratch, nullptr, 0, static_cast<cudaStream_t>(stream));
}

int sdr_window_stream_launch_count(int B, int S, int A, int64_t C, int64_t W, int64_t H) {
    if (const int e = stream_refusal(nullptr, B, S, A, W, H)) return e;
    if (sdr_window_stream_merge_scratch_bytes(B, S, C, H) == 0) return SDR_ERR_BAD_ARGUMENT;
    return 6;          // gather, history; align, scan, overlap-add, carry (the forward between them not counted)
}

}  // extern "C"
#pragma GCC visibility pop
