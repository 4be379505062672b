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
// The streaming resampler (section 7h below) runs the same tiles over each slot's [history | chunk]:
//   resample_stream_kernel          a step's or a flush's outputs, and a step's next history
//   resample_stream_advance_kernel  the step counters, once every read of them is done
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
constexpr int kResampleStreamMaxSlots = 65535;

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

// One tile's sums: thread k's output over its support s (when `active`) in ascending t, the tile's input span
// [lo, hi] staged chunk by chunk in xs as fp64 by load(t), the taps from hs (kSmemFilter) or h.  Every thread of the CTA
// calls it: the staging is shared.
template <bool kSmemFilter, class Load>
__device__ __forceinline__ double resample_tile_sum(const ResampleSupport& s, bool active, long long lo, long long hi,
                                                    Load load, const double* __restrict__ h, const double* hs,
                                                    double* xs, int p) {
    double acc = 0.0;
    for (long long c0 = lo; c0 <= hi; c0 += kResampleChunk) {
        const int m = (int)std::min((long long)kResampleChunk, hi - c0 + 1);
        if (c0 != lo) __syncthreads();
        for (int j = threadIdx.x; j < m; j += kResampleThreads) xs[j] = (double)load(c0 + j);
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
    return acc;
}

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
        const double acc = resample_tile_sum<kSmemFilter>(s, active, tl.lo, tl.hi,
                                                          [xr](long long t) { return __ldg(xr + t); }, h, hs, xs, p);
        if (active) out[tl.row * n + tl.i0 + threadIdx.x] = (float)acc;
    }
}

// ---- streaming resampler (DESIGN.md section 7h) ------------------------------------------------------------------
// Per slot, s = `lead` zeros then everything received since the reset, and r = resample_poly(s).  Step j (the slot's
// counter) writes r[j P - delay + i], i < P = C p / q (zeros below 0), summed exactly as resample_poly_kernel sums
// them, from the virtual row V = [history | chunk]: V[k] is s[lead + j C - Hs + k].  Every output of a step has its
// whole support in V (delay >= floor((L - lead p) / q)), and V's first sample lies at or below the first support.
// The history of step j is read from buffer j & 1 and the next one written to the other, so one launch reads the old
// history and writes the new; a second launch advances the counters once every read is done.

static long long floor_div(long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

struct ResampleStreamPlan {
    int err = SDR_ERR_BAD_ARGUMENT;
    int p = 1, q = 1, L = 0;
    long long P = 0, Hs = 0;
    size_t count_off = 0, hist_off = 0, bytes = 0;
    ResampleStreamPlan(int B, int rows, long long C, int up, int down, long long delay, long long lead) {
        const ResamplePlan g(up, down);
        if (up < 1 || down < 1) return;
        if (!g.ok || g.p == g.q) {
            err = SDR_ERR_UNSUPPORTED;
            return;
        }
        p = g.p, q = g.q, L = g.L;
        if (B < 1 || B > kResampleStreamMaxSlots || rows < 1 || C < 1 || C > kResampleMaxT || C % q) return;
        if (lead < 0 || lead > kResampleMaxT || delay > kResampleMaxT) return;
        if (delay < min_delay(L, p, q, lead)) return;
        P = C / q * p;
        Hs = lead + floor_div(delay * q + L, p) + 1;
        const long long R = (long long)B * rows, widest = std::max(std::max(C, P), Hs);
        if (widest > (1LL << 62) / (2 * R * 4096)) return;
        count_off = ((2 * (size_t)L + 1) * sizeof(double) + 255) / 256 * 256;
        hist_off = count_off + ((size_t)B * sizeof(long long) + 255) / 256 * 256;
        bytes = hist_off + 2 * (size_t)R * Hs * sizeof(float);
        err = SDR_OK;
    }
    static long long min_delay(int L, int p, int q, long long lead) { return floor_div(L - lead * p, q); }
};

struct ResampleStreamTile {
    long long row, i0, o0, base, len, lo, hi;
    const float* hist;
    const float* x;
    int count;
    bool zero;
};

// Outputs [0, n) of every row of the B x rows, from [history | x] (x: Tx samples per row; zero[slot] set: read as
// zeros).  hist_out non-null: a step, which also writes V[Tx, Tx + Hs) as the next history.
template <bool kSmemFilter>
__global__ void __launch_bounds__(kResampleThreads)
resample_stream_kernel(const float* hist, float* hist_out, const long long* __restrict__ count,
                       const float* __restrict__ x, const unsigned char* __restrict__ zero, float* __restrict__ out,
                       const double* __restrict__ h, int rows, long long R, long long Hs, long long Tx, long long C,
                       long long n, long long P, long long delay, long long lead, int p, int q, int L) {
    extern __shared__ double smem[];
    __shared__ ResampleStreamTile tile;
    double* xs = smem;
    double* hs = smem + kResampleChunk;
    if (kSmemFilter)
        for (int k = threadIdx.x; k <= 2 * L; k += kResampleThreads) hs[k] = h[k];
    const long long tiles = (n + kResampleThreads - 1) / kResampleThreads;
    for (long long w = blockIdx.x; w < R * tiles; w += gridDim.x) {
        __syncthreads();                                    // the last tile's reads of xs and `tile` are done
        if (threadIdx.x == 0) {
            ResampleStreamTile tl;
            tl.row = w / tiles;
            tl.i0 = (w - tl.row * tiles) * kResampleThreads;
            tl.count = (int)std::min((long long)kResampleThreads, n - tl.i0);
            const long long slot = tl.row / rows, j = count[slot];
            tl.o0 = j * P - delay + tl.i0;
            tl.base = lead + j * C - Hs;
            tl.len = lead + j * C + Tx;
            tl.hist = hist + ((j & 1) * R + tl.row) * Hs;
            tl.x = x ? x + tl.row * Tx : nullptr;
            tl.zero = zero && zero[slot];
            const long long a = std::max(tl.o0, 0LL), b = tl.o0 + tl.count - 1;
            tl.lo = 0;
            tl.hi = -1;
            if (a <= b) {
                const long long ca = a * q + L, cb = b * q + L;
                tl.lo = resample_support(ca / p, (int)(ca % p), p, L, tl.len).t0;
                tl.hi = resample_support(cb / p, (int)(cb % p), p, L, tl.len).t1;
            }
            tile = tl;
        }
        __syncthreads();
        const ResampleStreamTile tl = tile;
        const long long o = tl.o0 + threadIdx.x, c = std::max(o, 0LL) * q + L;
        const ResampleSupport s = resample_support(c / p, (int)(c % p), p, L, tl.len);
        const bool active = (int)threadIdx.x < tl.count && o >= 0;
        const long long base = tl.base;
        const float* hr = tl.hist;
        const float* xr = tl.x;
        const bool zr = tl.zero;
        const double acc = resample_tile_sum<kSmemFilter>(
            s, active, tl.lo, tl.hi,
            [=](long long t) {
                const long long k = t - base;
                return k < Hs ? hr[k] : (zr ? 0.f : __ldg(xr + (k - Hs)));
            },
            h, hs, xs, p);
        if ((int)threadIdx.x < tl.count) out[tl.row * n + tl.i0 + threadIdx.x] = active ? (float)acc : 0.f;
    }
    if (!hist_out) return;
    for (long long e = (long long)blockIdx.x * kResampleThreads + threadIdx.x; e < R * Hs;
         e += (long long)gridDim.x * kResampleThreads) {
        const long long row = e / Hs, k = e - row * Hs + Tx, slot = row / rows, j = count[slot];
        const float v = k < Hs ? hist[((j & 1) * R + row) * Hs + k]
                               : (zero && zero[slot] ? 0.f : __ldg(x + row * Tx + (k - Hs)));
        hist_out[(((j + 1) & 1) * R + row) * Hs + (e - row * Hs)] = v;
    }
}

__global__ void resample_stream_advance_kernel(long long* __restrict__ count, int B) {
    const int b = blockIdx.x * 256 + threadIdx.x;
    if (b < B) count[b] += 1;
}

// The refusals of every streaming entry in order: the plan's, a null state or !args_ok, a small state, a misaligned one.
static int stream_refusal(const ResampleStreamPlan& g, const void* state, bool args_ok, size_t state_bytes) {
    if (g.err) return g.err;
    if (!state || !args_ok) return SDR_ERR_BAD_ARGUMENT;
    if (state_bytes < g.bytes) return SDR_ERR_WORKSPACE;
    return reinterpret_cast<uintptr_t>(state) % 256 ? SDR_ERR_BAD_ARGUMENT : SDR_OK;
}

static long long resample_stream_flush_length(int p, int q, long long delay, long long lead, long long tail_len) {
    return resampled_length(lead + tail_len, p, q) + delay;
}

// A step (tail_len < 0: x is the chunk of C samples) or a flush (x is the tail of tail_len samples, maybe null when
// tail_len is 0).
static int resample_stream_run(const ResampleStreamPlan& g, void* state, const float* x, long long tail_len,
                               const unsigned char* zero, float* out, int B, int rows, long long C, long long delay,
                               long long lead, cudaStream_t st) {
    char* base = static_cast<char*>(state);
    const double* h = reinterpret_cast<const double*>(base);
    long long* count = reinterpret_cast<long long*>(base + g.count_off);
    float* hist = reinterpret_cast<float*>(base + g.hist_off);
    const bool step = tail_len < 0;
    const long long Tx = step ? C : tail_len;
    const long long n = step ? g.P : resample_stream_flush_length(g.p, g.q, delay, lead, tail_len);
    const long long R = (long long)B * rows;
    const int taps = 2 * g.L + 1;
    const bool smem_filter = taps <= kResampleSmemTaps;
    const size_t smem = (kResampleChunk + (smem_filter ? taps : 0)) * sizeof(double);
    auto kern = smem_filter ? resample_stream_kernel<true> : resample_stream_kernel<false>;
    int e;
    if ((e = allow_dynamic_smem(reinterpret_cast<const void*>(kern), smem))) return e;
    int per_sm = 0;
    if ((e = cuda_status(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kResampleThreads, smem))))
        return e;
    const long long work = std::max(R * ((n + kResampleThreads - 1) / kResampleThreads),
                                    step ? (R * g.Hs + kResampleThreads - 1) / kResampleThreads : 0LL);
    if (work == 0) return SDR_OK;
    const long long grid = std::min(work, (long long)std::max(per_sm, 1) * std::max(sm_count(), 1));
    if ((e = launch(kern, (unsigned)grid, kResampleThreads, smem, st, hist, step ? hist : nullptr, count, x, zero, out,
                    h, rows, R, g.Hs, Tx, C, n, g.P, delay, lead, g.p, g.q, g.L)))
        return e;
    if (!step) return SDR_OK;
    return launch(resample_stream_advance_kernel, (unsigned)((B + 255) / 256), 256, 0, st, count, B);
}

}  // namespace sdr

using namespace sdr;

#pragma GCC visibility push(default)
extern "C" {

size_t sdr_resample_poly_scratch_bytes(int up, int down) {
    const ResamplePlan g(up, down);
    return g.ok ? g.scratch_bytes() : 0;
}

int sdr_resample_poly(const float* x, float* out, int64_t rows, int64_t T, int up, int down, void* scratch,
                      size_t scratch_bytes, sdr_stream stream) {
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
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

size_t sdr_resample_stream_state_bytes(int B, int rows, int64_t C, int up, int down, int64_t delay, int64_t lead) {
    const ResampleStreamPlan g(B, rows, C, up, down, delay, lead);
    return g.err == SDR_OK ? g.bytes : 0;
}

int sdr_resample_stream_reset(void* state, size_t state_bytes, int B, int rows, int64_t C, int up, int down,
                              int64_t delay, int64_t lead, const int32_t* slots, int n, sdr_stream stream) {
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const ResampleStreamPlan g(B, rows, C, up, down, delay, lead);
    if (const int e = stream_refusal(g, state, !(slots && n < 0), state_bytes)) return e;
    char* base = static_cast<char*>(state);
    long long* count = reinterpret_cast<long long*>(base + g.count_off);
    float* hist = reinterpret_cast<float*>(base + g.hist_off);
    if (!slots) {                                 // the whole state: the filter, the counters and both histories
        double* h = reinterpret_cast<double*>(base);
        int e;
        if ((e = launch(resample_taps_kernel, (unsigned)((2 * g.L + 1 + 255) / 256), 256, 0, st, h, g.L,
                        std::max(g.p, g.q))))
            return e;
        if ((e = launch(resample_normalise_kernel, 1, 1024, 0, st, h, g.L, g.p))) return e;
        return cuda_status(cudaMemsetAsync(count, 0, g.bytes - g.count_off, st));
    }
    const size_t slot = (size_t)rows * g.Hs * sizeof(float);        // one slot's rows of one history buffer
    return reset_slots({{count, sizeof(long long)}, {hist, slot}, {hist + (long long)B * rows * g.Hs, slot}}, B, slots,
                       n, nullptr, st);
}

int sdr_resample_stream_step(void* state, size_t state_bytes, const float* chunk, const uint8_t* zero, float* out,
                             int B, int rows, int64_t C, int up, int down, int64_t delay, int64_t lead,
                             sdr_stream stream) {
    const ResampleStreamPlan g(B, rows, C, up, down, delay, lead);
    if (const int e = stream_refusal(g, state, chunk && out, state_bytes)) return e;
    return resample_stream_run(g, state, chunk, -1, zero, out, B, rows, C, delay, lead,
                               static_cast<cudaStream_t>(stream));
}

int sdr_resample_stream_flush(const void* state, size_t state_bytes, const float* tail, int64_t tail_len,
                              const uint8_t* zero, float* out, int B, int rows, int64_t C, int up, int down,
                              int64_t delay, int64_t lead, sdr_stream stream) {
    const ResampleStreamPlan g(B, rows, C, up, down, delay, lead);
    const bool args_ok = out && tail_len >= 0 && tail_len <= kResampleMaxT && (tail || tail_len == 0);
    if (const int e = stream_refusal(g, state, args_ok, state_bytes)) return e;
    // the state is only read: no history is written and the counters do not move
    return resample_stream_run(g, const_cast<void*>(state), tail, tail_len, zero, out, B, rows, C, delay, lead,
                               static_cast<cudaStream_t>(stream));
}

}  // extern "C"
#pragma GCC visibility pop
