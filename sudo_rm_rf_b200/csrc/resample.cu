// scipy.signal.resample_poly(x, up, down) with its defaults (window=('kaiser', 5.0), padtype='constant') on every row
// of x [rows][T] fp32.  With up / down reduced to p / q and L = 10 max(p, q):
//   h = firwin(2L + 1, 1 / max(p, q), window=('kaiser', 5.0)) * p  (the windowed sinc normalised to sum 1, times p),
//   out[i] = sum_t h[i q + L - t p] x[t] over the taps inside [0, 2L], i < ceil(T p / q),
// summed in fp64 in ascending t and rounded once to fp32.  The order is fixed, so an output is bitwise independent of
// the batch, the grid and the tiling.  p == q is a copy.  Three kernels, no atomics, no host synchronisation:
//   resample_taps_kernel       the filter's taps before normalisation, one per thread
//   resample_normalise_kernel  one CTA: their sum in a fixed order, then h / sum * p
//   resample_poly_kernel       per tile of 256 consecutive outputs of one row, one per thread: the tile's input span
//                              staged in shared memory as fp64 in chunks, the filter too when it fits
#include <algorithm>
#include <numeric>
#include "launchers.cuh"
#include "resample.cuh"

namespace sdr {

constexpr int kResampleMaxRatio = 4096;          // largest reduced max(p, q): 11.025 <-> 192 kHz is 147 / 2560
constexpr double kResampleBeta = 5.0;            // resample_poly's default window ('kaiser', 5.0)
constexpr int kResampleThreads = 256;            // outputs per tile, one per thread
constexpr int kResampleChunk = 2048;             // input samples staged per pass
constexpr int kResampleSmemTaps = 12288;         // filters up to this many taps (max(p, q) <= 614) are staged too
constexpr long long kResampleMaxT = 1LL << 40;

struct ResamplePlan {
    bool ok = false;
    int p = 1, q = 1, L = 0;
    ResamplePlan(int up, int down) {
        if (up < 1 || down < 1) return;
        const int g = std::gcd(up, down);
        p = up / g;
        q = down / g;
        const int mx = std::max(p, q);
        if (mx > kResampleMaxRatio) return;
        L = 10 * mx;
        ok = true;
    }
    size_t scratch_bytes() const { return (2 * (size_t)L + 1) * sizeof(double); }
};

__global__ void __launch_bounds__(256) resample_taps_kernel(double* __restrict__ h, int L, int mx) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i <= 2 * L) h[i] = kaiser_sinc_tap(i, L, mx, kResampleBeta, resample_i0(kResampleBeta), 2.0);
}

__global__ void __launch_bounds__(1024) resample_normalise_kernel(double* __restrict__ h, int L, int p) {
    __shared__ double red[32];
    __shared__ double total;
    const int taps = 2 * L + 1;
    double part = 0.0;
    for (int i = threadIdx.x; i < taps; i += 1024) part += h[i];
    part = warp_sum_f64(part);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < 32; ++w) s += red[w];
        total = s;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < taps; i += 1024) h[i] = h[i] / total * (double)p;
}

// One tile: outputs [i0, i0 + count) of row `row`, c = i0 q + L = cbq p + cbr, reading input samples [lo, hi].
struct ResampleTile {
    long long row, i0, cbq, lo, hi;
    int cbr, count;
};

// A persistent grid strides over the rows x tiles.  Thread k of a tile computes output i0 + k over its support in
// ascending t, chunk by chunk of the staged span; dynamic shared memory holds the chunk and, with kSmemFilter, h.
template <bool kSmemFilter>
__global__ void __launch_bounds__(kResampleThreads)
resample_poly_kernel(const float* __restrict__ x, float* __restrict__ out, const double* __restrict__ h,
                     long long rows, long long T, long long n, int p, int q, int L) {
    extern __shared__ double smem[];
    __shared__ ResampleTile tile;
    double* xs = smem;
    double* hs = smem + kResampleChunk;
    if (kSmemFilter)
        for (int k = threadIdx.x; k <= 2 * L; k += kResampleThreads) hs[k] = h[k];
    const long long tiles = (n + kResampleThreads - 1) / kResampleThreads;
    for (long long w = blockIdx.x; w < rows * tiles; w += gridDim.x) {
        __syncthreads();                                    // the last tile's reads of xs and `tile` are done
        if (threadIdx.x == 0) {
            ResampleTile tl;
            tl.row = w / tiles;
            tl.i0 = (w - tl.row * tiles) * kResampleThreads;
            tl.count = (int)std::min((long long)kResampleThreads, n - tl.i0);
            const long long cb = tl.i0 * q + L;
            tl.cbq = cb / p;
            tl.cbr = (int)(cb - tl.cbq * p);
            const int v = tl.cbr + (tl.count - 1) * q;
            tl.lo = resample_support(tl.cbq, tl.cbr, p, L, T).t0;
            tl.hi = resample_support(tl.cbq + v / p, v % p, p, L, T).t1;
            tile = tl;
        }
        __syncthreads();
        const ResampleTile tl = tile;
        const int v = tl.cbr + (int)threadIdx.x * q;        // < p + 255 q: 32-bit
        const ResampleSupport s = resample_support(tl.cbq + v / p, v % p, p, L, T);
        const bool active = (int)threadIdx.x < tl.count;
        const float* xr = x + tl.row * T;
        double acc = 0.0;
        for (long long c0 = tl.lo; c0 <= tl.hi; c0 += kResampleChunk) {
            const int m = (int)std::min((long long)kResampleChunk, tl.hi - c0 + 1);
            if (c0 != tl.lo) __syncthreads();
            for (int j = threadIdx.x; j < m; j += kResampleThreads) xs[j] = (double)__ldg(xr + c0 + j);
            __syncthreads();
            const long long a = std::max(s.t0, c0), b = std::min(s.t1, c0 + m - 1);
            if (active && a <= b) {
                int k = s.r + (int)(s.cp - a) * p;               // tap of sample a; one p lower per sample
                const double* xp = xs + (a - c0);
                const int cnt = (int)(b - a + 1);
#pragma unroll 4
                for (int j = 0; j < cnt; ++j, k -= p) acc = fma(kSmemFilter ? hs[k] : __ldg(h + k), xp[j], acc);
            }
        }
        if (active) out[tl.row * n + tl.i0 + threadIdx.x] = (float)acc;
    }
}

size_t resample_poly_scratch_bytes(int up, int down) {
    const ResamplePlan g(up, down);
    return g.ok ? g.scratch_bytes() : 0;
}

int launch_resample_poly(const float* x, float* out, long long rows, long long T, int up, int down, void* scratch,
                         size_t scratch_bytes, cudaStream_t st) {
    if (!x || !out || !scratch || reinterpret_cast<uintptr_t>(scratch) % 8) return SDR_ERR_BAD_ARGUMENT;
    if (rows < 1 || T < 1 || T > kResampleMaxT || rows > (1LL << 62) / (T * 4096)) return SDR_ERR_BAD_ARGUMENT;
    const ResamplePlan g(up, down);
    if (!g.ok) return up < 1 || down < 1 ? SDR_ERR_BAD_ARGUMENT : SDR_ERR_UNSUPPORTED;
    if (scratch_bytes < g.scratch_bytes()) return SDR_ERR_WORKSPACE;
    if (g.p == g.q)
        return cuda_status(cudaMemcpyAsync(out, x, (size_t)(rows * T) * sizeof(float), cudaMemcpyDeviceToDevice, st));
    double* h = static_cast<double*>(scratch);
    const int taps = 2 * g.L + 1;
    int e;
    if ((e = launch(resample_taps_kernel, (unsigned)((taps + 255) / 256), 256, 0, st, h, g.L, std::max(g.p, g.q))))
        return e;
    if ((e = launch(resample_normalise_kernel, 1, 1024, 0, st, h, g.L, g.p))) return e;
    const long long n = resampled_length(T, g.p, g.q);
    const bool smem_filter = taps <= kResampleSmemTaps;
    const size_t smem = (kResampleChunk + (smem_filter ? taps : 0)) * sizeof(double);
    auto kern = smem_filter ? resample_poly_kernel<true> : resample_poly_kernel<false>;
    if ((e = allow_dynamic_smem(reinterpret_cast<const void*>(kern), smem))) return e;
    int per_sm = 0;
    if ((e = cuda_status(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kResampleThreads, smem))))
        return e;
    const long long work = rows * ((n + kResampleThreads - 1) / kResampleThreads);
    const long long grid = std::min(work, (long long)std::max(per_sm, 1) * std::max(sm_count(), 1));
    return launch(kern, (unsigned)grid, kResampleThreads, smem, st, x, out, h, rows, T, n, g.p, g.q, g.L);
}

}  // namespace sdr
