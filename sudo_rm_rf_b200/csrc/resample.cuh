// Device code shared by the polyphase resamplers of stoi.cu (Octave's filter, into 10 kHz) and resample.cu (scipy's
// resample_poly): the Kaiser-windowed sinc tap and the support arithmetic of resample_poly's alignment.
#pragma once
#include <math_constants.h>

namespace sdr {

// Resampled length ceil(len p / q).
__host__ __device__ __forceinline__ long long resampled_length(long long len, int p, int q) {
    return (len * p + q - 1) / q;
}

// The modified Bessel function I0 by its power series sum ((x/2)^k / k!)^2, to full precision for x <= 6.
__device__ inline double resample_i0(double x) {
    const double q = 0.25 * x * x;
    double term = 1.0, sum = 1.0;
    for (int k = 1; k < 64 && term > 1e-18 * sum; ++k) {
        term *= q / ((double)k * k);
        sum += term;
    }
    return sum;
}

// Tap i of the 2L + 1 (L >= 1) of a Kaiser-windowed lowpass with cutoff c = 1 / (2 mx) cycles per sample, before
// normalisation: kaiser(2L+1, beta)[i] * gain c sinc(2 c (i - L)), with i0b = I0(beta).
__device__ __forceinline__ double kaiser_sinc_tap(int i, int L, int mx, double beta, double i0b, double gain) {
    const int t = i - L;
    const double cutoff = 1.0 / (2.0 * (double)mx);
    const double a = 2.0 * cutoff * t;
    const double sinc = t == 0 ? 1.0 : sinpi(a) / (CUDART_PI * a);
    const double r = (double)(i - L) / (double)L;
    return resample_i0(beta * sqrt(1.0 - r * r)) / i0b * (gain * cutoff * sinc);
}

// Output i of a signal of len samples upsampled by p, filtered by h[0, 2L] and downsampled by q with
// resample_poly's alignment: out[i] = sum h[c - t p] x[t] over the input samples t0 <= t <= t1 whose tap lies in
// [0, 2L], c = i q + L.  With c = cp p + r (0 <= r < p, r <= 2L), sample t takes tap
// h[r + (cp - t) p].
struct ResampleSupport {
    long long cp, t0, t1;
    int r;
};
__device__ __forceinline__ ResampleSupport resample_support(long long cp, int r, int p, int L, long long len) {
    ResampleSupport s;
    s.cp = cp;
    s.r = r;
    const long long k = (2 * L - r) / p;                     // taps r, r + p, .., r + k p
    s.t0 = cp > k ? cp - k : 0;
    s.t1 = cp < len - 1 ? cp : len - 1;
    return s;
}

}  // namespace sdr
