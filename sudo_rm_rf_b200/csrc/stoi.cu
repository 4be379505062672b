// Short-time objective intelligibility (STOI; Taal et al., IEEE TASLP 2011) as pystoi 0.3.3's
// stoi(x, y, fs_sig, extended=False) computes it, the `stoi` of asteroid's get_metrics.  Per (clean x, processed y):
//   1. both resampled to 10 kHz by Octave's resample (a Kaiser-windowed sinc, scipy's resample_poly alignment);
//   2. the 256-sample Hann frames (hop 128) of x more than 40 dB below x's loudest frame dropped from x and y, the
//      kept frames overlap-added back;
//   3. Hann-windowed 256-sample frames (hop 128) of the result, a 512-point FFT, 15 third-octave band magnitudes;
//   4. for every 30-frame segment and band: y scaled to x's norm, clipped at x (1 + 10^(15/20)), both centred and
//      normalised, their inner product; d = the mean over segments and bands (1e-5 below 30 frames).
// Everything after the fp32 inputs is fp64.  Five kernels, no atomics (bitwise reproducible), no host synchronisation:
//   stoi_filter_kernel    the resampling filter, on the device so a call holds no host-to-device copy
//   stoi_resample_kernel  polyphase resampling of every reference, estimate and mixture row
//   stoi_mask_kernel      per reference row: frame energies, the silent-frame mask, the kept frames compacted in order
//   stoi_spectra_kernel   per (row, spectral frame), one warp: the frame rebuilt from kept frames j-1, j and j+1 (the
//                         overlap-added signal is never stored), the FFT in shared memory, the 15 band magnitudes
//   stoi_segment_kernel   per (item, source): the segment correlations of the estimate and of the mixture, d
#include <math_constants.h>
#include <cmath>
#include <numeric>
#include "launchers.cuh"
#include "resample.cuh"

namespace sdr {

constexpr int kStoiFs = 10000;
constexpr int kStoiFrame = 256, kStoiHop = 128, kStoiFft = 512, kStoiBands = 15, kStoiSeg = 30;
// Largest reduced max(p, q) of the resampling ratio 10000 / fs: 441 takes 44.1 and 22.05 kHz (a 31947-tap filter).
constexpr int kStoiMaxRatio = 441;
constexpr double kStoiEps = 2.220446049250313e-16;       // np.finfo(float).eps
constexpr int kStoiValid = 8;                            // flags: the item's length lies in [1, T]

// pystoi's thirdoct(10000, 512, 15, 150): band i covers FFT bins [lo, hi)
__constant__ int kStoiBandLo[kStoiBands] = {7, 9, 11, 14, 17, 22, 27, 34, 43, 55, 69, 87, 109, 138, 174};
__constant__ int kStoiBandHi[kStoiBands] = {9, 11, 14, 17, 22, 27, 34, 43, 55, 69, 87, 109, 138, 174, 219};

// The geometry of one call: the resampling ratio p / q, the filter's half length L (taps 2L + 1), the longest
// resampled row Tn, its analysis-frame count F0 and spectral-frame count M.
struct StoiPlan {
    bool ok = false;
    int p = 1, q = 1, L = 0;
    long long Tn = 0, F0 = 0, M = 0;
    StoiPlan(int B, int S, long long T, int fs) {
        if (B <= 0 || S <= 0 || T <= 0 || fs < 1000 || T > (1LL << 40)) return;
        if ((long long)B * S > 0x7fffffffLL / 3) return;            // 3 B S tob rows are counted in int
        const int g = std::gcd(kStoiFs, fs);
        p = kStoiFs / g;
        q = fs / g;
        const int mx = p > q ? p : q;
        if (mx > kStoiMaxRatio) return;
        // pystoi's _resample_window_oct, operation for operation: L = ceil((60 - 8) / (28.714 roll-off))
        if (p != q) L = (int)std::ceil((60.0 - 8.0) / (28.714 * ((1.0 / (2 * (double)mx)) / 10)));
        Tn = (T * p + q - 1) / q;
        F0 = Tn > kStoiFrame ? (Tn - kStoiFrame + kStoiHop - 1) / kStoiHop : 0;
        M = F0 > 1 ? F0 - 1 : 0;
        ok = true;
    }
};

// Scratch carve-up.  Doubles: h [2L+1], sig [2R + B][Tn] (references, estimates, mixtures resampled), energy [R][F0],
// tob [3R][15][M] (band magnitudes of references, estimates, the mixture under each reference's mask); then ints:
// kept [R][F0] (kept frame indices), count [R], flags [R] (bit 0 reference finite, 1 estimate finite, 2 mixture
// finite, 3 valid length).
struct StoiScratch {
    double *h, *sig, *energy, *tob;
    int *kept, *count, *flags;
    size_t bytes;
    StoiScratch(void* base, const StoiPlan& g, int B, int S) {
        const size_t R = (size_t)B * S;
        char* c = static_cast<char*>(base);
        size_t off = 0;
        auto take = [&](size_t n, size_t elem) { void* r = c ? c + off : nullptr; off += n * elem; return r; };
        h = static_cast<double*>(take(2 * (size_t)g.L + 1, 8));
        sig = static_cast<double*>(take((2 * R + B) * (size_t)g.Tn, 8));
        energy = static_cast<double*>(take(R * (size_t)g.F0, 8));
        tob = static_cast<double*>(take(3 * R * kStoiBands * (size_t)g.M, 8));
        kept = static_cast<int*>(take(R * (size_t)g.F0, 4));
        count = static_cast<int*>(take(R, 4));
        flags = static_cast<int*>(take(R, 4));
        bytes = off;
    }
};

// np.hanning(258)[1:-1][k] = 0.5 + 0.5 cos(pi (2k - 255) / 257)
__device__ __forceinline__ double stoi_hann(int k) { return 0.5 + 0.5 * cospi((2.0 * k - 255.0) / 257.0); }

// One CTA of 256 threads.  h[t + L] = kaiser(2L+1, 0.1102 (60 - 8.7))[t + L] * 2 p cutoff sinc(2 cutoff t),
// cutoff = 1 / (2 max(p, q)), then h / sum(h) * p: pystoi's window normalised to sum 1, times resample_poly's gain p.
// p == q (10 kHz input): h = [1], the identity.
__global__ void __launch_bounds__(256) stoi_filter_kernel(double* __restrict__ h, int p, int q, int L) {
    __shared__ double red[8];
    __shared__ double total;
    if (L == 0) {
        if (threadIdx.x == 0) h[0] = 1.0;
        return;
    }
    const int taps = 2 * L + 1;
    const double beta = 0.1102 * (60.0 - 8.7);
    const double i0b = resample_i0(beta);
    double part = 0.0;
    for (int i = threadIdx.x; i < taps; i += 256) {
        const double v = kaiser_sinc_tap(i, L, p > q ? p : q, beta, i0b, 2.0 * p);
        h[i] = v;
        part += v;
    }
    part = warp_sum_f64(part);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < 8; ++w) s += red[w];
        total = s;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < taps; i += 256) h[i] = h[i] / total * (double)p;
}

// Row r of the resampled signals: references [0, R), estimates [R, 2R), mixtures [2R, 2R + B).  Item b's rows are
// scored over their first lengths[b] samples; out[i] = sum_t h[i q + L - t p] x[t] over 0 <= t < len, i < ceil(len p / q)
// (scipy's upfirdn with resample_poly's padding and alignment).  Nothing is written for an invalid length.
__global__ void __launch_bounds__(256)
stoi_resample_kernel(const float* __restrict__ ref, const float* __restrict__ est, const float* __restrict__ mix,
                     const long long* __restrict__ lengths, const double* __restrict__ h, double* __restrict__ sig,
                     int S, long long R, long long rows, long long T, long long Tn, int p, int q, int L) {
    for (long long row = blockIdx.y; row < rows; row += gridDim.y) {
        long long b;
        const float* x;
        if (row < R) { b = row / S; x = ref + row * T; }
        else if (row < 2 * R) { b = (row - R) / S; x = est + (row - R) * T; }
        else { b = row - 2 * R; x = mix + b * T; }
        const long long len = lengths ? lengths[b] : T;
        if (len < 1 || len > T) continue;
        const long long n = resampled_length(len, p, q);
        double* out = sig + row * Tn;
        for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += gridDim.x * 256LL) {
            const long long c = i * q + L;
            const ResampleSupport s = resample_support(c / p, (int)(c % p), p, L, len);
            double acc = 0.0;
            for (long long t = s.t0; t <= s.t1; ++t) acc = fma(__ldg(h + (c - t * p)), (double)__ldg(x + t), acc);
            out[i] = acc;
        }
    }
}

// One CTA of 512 threads per reference row r (item b = r / S).  Frames f < F0 = ceil((n - 256) / 128) of the
// resampled row (n samples), energy 20 log10(|w x_f| + eps); frame f is kept when (max - 40 - energy_f) < 0.  The kept
// indices are compacted in order by a block scan.  Also the row's flags: its length valid, and reference row r,
// estimate row r and mixture row b finite over that length.
__global__ void __launch_bounds__(512)
stoi_mask_kernel(const float* __restrict__ ref, const float* __restrict__ est, const float* __restrict__ mix,
                 const long long* __restrict__ lengths, const double* __restrict__ sig, double* __restrict__ energy,
                 int* __restrict__ kept, int* __restrict__ count, int* __restrict__ flags, int S, long long T,
                 long long Tn, long long F0max, int p, int q) {
    __shared__ double win[kStoiFrame];
    __shared__ double red[16];
    __shared__ int wcount[16];
    __shared__ int base;
    const long long r = blockIdx.x;
    const long long b = r / S;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long len = lengths ? lengths[b] : T;
    if (len < 1 || len > T) {
        if (threadIdx.x == 0) { count[r] = 0; flags[r] = 0; }
        return;
    }
    bool rf = true, ef = true, mf = true;
    for (long long t = threadIdx.x; t < len; t += 512) {
        rf = rf && isfinite(__ldg(ref + r * T + t));
        ef = ef && isfinite(__ldg(est + r * T + t));
        if (mix) mf = mf && isfinite(__ldg(mix + b * T + t));
    }
    rf = __syncthreads_and(rf);
    ef = __syncthreads_and(ef);
    mf = __syncthreads_and(mf);
    for (int k = threadIdx.x; k < kStoiFrame; k += 512) win[k] = stoi_hann(k);
    if (threadIdx.x == 0) base = 0;
    __syncthreads();
    const long long n = resampled_length(len, p, q);
    const long long F0 = n > kStoiFrame ? (n - kStoiFrame + kStoiHop - 1) / kStoiHop : 0;
    const double* x = sig + r * Tn;
    double* e = energy + r * F0max;
    double mx = -INFINITY;
    for (long long f = threadIdx.x; f < F0; f += 512) {
        const double* xf = x + f * kStoiHop;
        double s = 0.0;
        for (int k = 0; k < kStoiFrame; ++k) {
            const double v = win[k] * xf[k];
            s = fma(v, v, s);
        }
        const double en = 20.0 * log10(sqrt(s) + kStoiEps);
        e[f] = en;
        mx = fmax(mx, en);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = red[0];
    for (int w = 1; w < 16; ++w) mx = fmax(mx, red[w]);
    int* kr = kept + r * F0max;
    for (long long tile = 0; tile < F0; tile += 512) {
        const long long f = tile + threadIdx.x;
        const bool keep = f < F0 && (mx - 40.0 - e[f]) < 0.0;
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) wcount[warp] = __popc(bal);
        __syncthreads();
        int off = base;
        for (int w = 0; w < warp; ++w) off += wcount[w];
        if (keep) kr[off + __popc(bal & ((1u << lane) - 1u))] = (int)f;
        __syncthreads();
        if (threadIdx.x == 0) for (int w = 0; w < 16; ++w) base += wcount[w];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        count[r] = base;
        flags[r] = kStoiValid | (rf ? 1 : 0) | (ef ? 2 : 0) | (mf ? 4 : 0);
    }
}

// 128 threads, one warp per (tob row, spectral frame j).  Tob row q: kind q / R (0 reference, 1 estimate, 2 the
// mixture) under reference r = q % R's mask, whose K kept frames give M = K - 1 spectral frames.  Frame j of the
// overlap-added signal is [kept_{j-1}[128:] + kept_j[:128], kept_j[128:] + kept_{j+1}[:128]] (kept_{-1} = 0), Hann
// windowed and zero-padded to 512; a radix-2 FFT in shared memory; tob[q][band][j] = sqrt(sum |X_k|^2 over the band).
__global__ void __launch_bounds__(128)
stoi_spectra_kernel(const double* __restrict__ sig, const int* __restrict__ kept, const int* __restrict__ count,
                    const int* __restrict__ flags, double* __restrict__ tob, int S, long long R, long long nrows,
                    long long Tn, long long F0max, long long Mmax) {
    __shared__ double2 buf[4][kStoiFft];
    __shared__ double2 tw[kStoiFft / 2];
    __shared__ double win[kStoiFrame];
    for (int k = threadIdx.x; k < kStoiFft / 2; k += 128) {
        double s, c;
        sincospi((double)k / (kStoiFft / 2), &s, &c);
        tw[k] = make_double2(c, -s);                                   // exp(-2 pi i k / 512)
    }
    for (int k = threadIdx.x; k < kStoiFrame; k += 128) win[k] = stoi_hann(k);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double2* a = buf[warp];
    const long long groups = (Mmax + 3) / 4;
    for (long long wi = blockIdx.x; wi < nrows * groups; wi += gridDim.x) {
        const long long qrow = wi / groups;
        const long long j = (wi - qrow * groups) * 4 + warp;
        const long long r = qrow % R;
        const int kind = (int)(qrow / R);
        if (!(flags[r] & kStoiValid) || j >= (long long)count[r] - 1) continue;
        const long long srow = kind == 0 ? r : kind == 1 ? R + r : 2 * R + r / S;
        const double* x = sig + srow * Tn;
        const int* kr = kept + r * F0max;
        const long long k0 = j > 0 ? kr[j - 1] : -1, k1 = kr[j], k2 = kr[j + 1];
        for (int t = lane; t < kStoiFrame; t += 32) {
            double v;
            if (t < kStoiHop) {
                v = win[t] * x[k1 * kStoiHop + t];
                if (k0 >= 0) v = win[t + kStoiHop] * x[k0 * kStoiHop + t + kStoiHop] + v;
            } else {
                v = win[t] * x[k1 * kStoiHop + t] + win[t - kStoiHop] * x[k2 * kStoiHop + t - kStoiHop];
            }
            a[__brev(t) >> 23] = make_double2(win[t] * v, 0.0);
            a[__brev(t + kStoiFrame) >> 23] = make_double2(0.0, 0.0);
        }
        __syncwarp();
        for (int len = 2, step = kStoiFft / 2; len <= kStoiFft; len <<= 1, step >>= 1) {
            const int half = len >> 1;
            for (int bf = lane; bf < kStoiFft / 2; bf += 32) {
                const int pos = bf & (half - 1);
                const int i0 = (bf - pos) * 2 + pos, i1 = i0 + half;
                const double2 w = tw[pos * step], u = a[i0], v = a[i1];
                const double2 m = make_double2(v.x * w.x - v.y * w.y, v.x * w.y + v.y * w.x);
                a[i0] = make_double2(u.x + m.x, u.y + m.y);
                a[i1] = make_double2(u.x - m.x, u.y - m.y);
            }
            __syncwarp();
        }
        if (lane < kStoiBands) {
            double s = 0.0;
            for (int k = kStoiBandLo[lane]; k < kStoiBandHi[lane]; ++k) s = fma(a[k].x, a[k].x, fma(a[k].y, a[k].y, s));
            tob[(qrow * kStoiBands + lane) * Mmax + j] = sqrt(s);
        }
        __syncwarp();
    }
}

// One segment's correlation: x, y the band's 30 magnitudes of the reference and of the scored signal (stride 1).
__device__ __forceinline__ double stoi_segment(const double* __restrict__ xs, const double* __restrict__ ys,
                                               double clip1) {
    double x[kStoiSeg], y[kStoiSeg];
    double nx = 0.0, ny = 0.0;
#pragma unroll
    for (int k = 0; k < kStoiSeg; ++k) {
        x[k] = xs[k];
        y[k] = ys[k];
        nx = fma(x[k], x[k], nx);
        ny = fma(y[k], y[k], ny);
    }
    const double alpha = sqrt(nx) / (sqrt(ny) + kStoiEps);
    double my = 0.0, mx = 0.0;
#pragma unroll
    for (int k = 0; k < kStoiSeg; ++k) {
        y[k] = fmin(y[k] * alpha, x[k] * clip1);
        my += y[k];
        mx += x[k];
    }
    my /= kStoiSeg;
    mx /= kStoiSeg;
    double vy = 0.0, vx = 0.0;
#pragma unroll
    for (int k = 0; k < kStoiSeg; ++k) {
        y[k] -= my;
        x[k] -= mx;
        vy = fma(y[k], y[k], vy);
        vx = fma(x[k], x[k], vx);
    }
    const double dy = sqrt(vy) + kStoiEps, dx = sqrt(vx) + kStoiEps;
    double c = 0.0;
#pragma unroll
    for (int k = 0; k < kStoiSeg; ++k) c = fma(y[k] / dy, x[k] / dx, c);
    return c;
}

// One CTA of 256 threads per (item, source) r: d of the estimate and, with the mixture, of the mixture under reference
// r, summed over (band, segment) in a fixed order.  Fewer than 30 spectral frames: 1e-5.  An invalid length, or a
// non-finite sample in the reference or the scored signal: NaN.
__global__ void __launch_bounds__(256)
stoi_segment_kernel(const double* __restrict__ tob, const int* __restrict__ count, const int* __restrict__ flags,
                    double* __restrict__ out, double* __restrict__ mout, long long R, long long Mmax, double clip1) {
    __shared__ double red[2][8];
    const long long r = blockIdx.x;
    const int fl = flags[r];
    const long long M = (long long)count[r] - 1;
    const double* xt = tob + r * kStoiBands * Mmax;
    const double* yt = tob + (R + r) * kStoiBands * Mmax;
    const double* mt = tob + (2 * R + r) * kStoiBands * Mmax;
    const long long J = M - (kStoiSeg - 1);
    double ad = 0.0, am = 0.0;
    if ((fl & kStoiValid) && M >= kStoiSeg) {
        for (long long n = threadIdx.x; n < J * kStoiBands; n += 256) {
            const long long band = n / J, m = n - band * J;
            const long long o = band * Mmax + m;
            ad += stoi_segment(xt + o, yt + o, clip1);
            if (mout) am += stoi_segment(xt + o, mt + o, clip1);
        }
    }
    ad = warp_sum_f64(ad);
    am = warp_sum_f64(am);
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = ad; red[1][threadIdx.x >> 5] = am; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double sd = 0.0, sm = 0.0;
        for (int w = 0; w < 8; ++w) { sd += red[0][w]; sm += red[1][w]; }
        const double nan = __longlong_as_double(0x7ff8000000000000LL);
        const bool valid = fl & kStoiValid;
        const double n = (double)(J * kStoiBands);
        const double d = M < kStoiSeg ? 1e-5 : sd / n;
        const double dm = M < kStoiSeg ? 1e-5 : sm / n;
        out[r] = valid && (fl & 1) && (fl & 2) ? d : nan;
        if (mout) mout[r] = valid && (fl & 1) && (fl & 4) ? dm : nan;
    }
}

}  // namespace sdr

using namespace sdr;

#pragma GCC visibility push(default)
extern "C" {

size_t sdr_stoi_scratch_bytes(int B, int S, int64_t T, int fs) {
    const StoiPlan g(B, S, T, fs);
    return g.ok ? StoiScratch(nullptr, g, B, S).bytes : 0;
}

int sdr_stoi(const float* ref, const float* est, const float* mix, const int64_t* lengths_or_null, double* out,
             double* mout, int B, int S, int64_t T, int fs, void* scratch, sdr_stream stream) {
    const long long* lengths = reinterpret_cast<const long long*>(lengths_or_null);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!ref || !est || !out || !scratch || reinterpret_cast<uintptr_t>(scratch) % 8 || (mix && !mout))
        return SDR_ERR_BAD_ARGUMENT;
    const StoiPlan g(B, S, T, fs);
    if (!g.ok) return B <= 0 || S <= 0 || T <= 0 ? SDR_ERR_BAD_ARGUMENT : SDR_ERR_UNSUPPORTED;
    const StoiScratch s(scratch, g, B, S);
    const long long R = (long long)B * S;
    const long long rows = 2 * R + (mix ? B : 0);
    const long long nrows = (mix ? 3 : 2) * R;
    const double clip1 = 1.0 + std::pow(10.0, 15.0 / 20.0);
    const long long chunks = (g.Tn + 255) / 256;
    const dim3 rgrid((unsigned)(chunks < 65535 ? chunks : 65535), (unsigned)(rows < 65535 ? rows : 65535));
    const long long sw = nrows * ((g.M + 3) / 4);
    const unsigned sgrid = (unsigned)(sw < 1 ? 1 : (sw < (1LL << 20) ? sw : (1LL << 20)));
    int e;
    if ((e = launch(stoi_filter_kernel, 1, 256, 0, st, s.h, g.p, g.q, g.L))) return e;
    if ((e = launch(stoi_resample_kernel, rgrid, 256, 0, st, ref, est, mix, lengths, s.h, s.sig, S, R, rows, T, g.Tn,
                    g.p, g.q, g.L)))
        return e;
    if ((e = launch(stoi_mask_kernel, (unsigned)R, 512, 0, st, ref, est, mix, lengths, s.sig, s.energy, s.kept,
                    s.count, s.flags, S, T, g.Tn, g.F0, g.p, g.q)))
        return e;
    if ((e = launch(stoi_spectra_kernel, sgrid, 128, 0, st, s.sig, s.kept, s.count, s.flags, s.tob, S, R, nrows, g.Tn,
                    g.F0, g.M)))
        return e;
    return launch(stoi_segment_kernel, (unsigned)R, 256, 0, st, s.tob, s.count, s.flags, out, mout, R, g.M, clip1);
}

}  // extern "C"
#pragma GCC visibility pop
