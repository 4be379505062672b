// The permutation search and source-count dispatch shared by the metrics (prepost.cu) and BSS-eval (bsseval.cu).
#pragma once
#include <type_traits>

#include "common.cuh"

namespace sdr {

// torch.max's selection over candidates in order: the first NaN wins and is kept, otherwise the first maximum.
// np.argmax picks the same one.
__device__ __forceinline__ bool takes_max(double m, double best, int idx) {
    return idx == 0 || (!isnan(best) && (isnan(m) || m > best));
}

// itertools.permutations(range(SE), r=SA) as a compile-time table: assignment p gives target j the estimate p[j].
// Counting in base SE with p[0] as the most significant digit and keeping the codes whose digits are distinct lists
// them in itertools' (lexicographic) order.
template <int SE, int SA> struct Assignments {
    static constexpr int count() {
        int n = 1;
        for (int j = 0; j < SA; ++j) n *= SE - j;
        return n;
    }
    int p[count()][SA];
    constexpr Assignments() : p() {
        int codes = 1, n = 0;
        for (int j = 0; j < SA; ++j) codes *= SE;
        for (int code = 0; code < codes; ++code) {
            int d[SA] = {}, c = code;
            bool distinct = true;
            for (int j = SA - 1; j >= 0; --j) { d[j] = c % SE; c /= SE; }
            for (int j = 0; j < SA; ++j)
                for (int k = 0; k < j; ++k) distinct = distinct && d[k] != d[j];
            if (!distinct) continue;
            for (int j = 0; j < SA; ++j) p[n][j] = d[j];
            ++n;
        }
    }
};

// Keeps torch.max's pick of score(p) over the assignments in itertools order and returns that score; best_idx gets
// its index in that order and best_p the assignment.  Unrolled, so every p[j] is a constant and the caller's scores
// stay in registers; a score that sums them adds with __dadd_rn, which keeps each product out of a fused
// multiply-add and the sum in the separate roundings of the reference's torch sum.
template <int SE, int SA, class Score>
__device__ __forceinline__ double best_assignment(const Score& score, int& best_idx, int (&best_p)[SA]) {
    constexpr Assignments<SE, SA> kAll;
    double best = 0.0;
#pragma unroll
    for (int idx = 0; idx < Assignments<SE, SA>::count(); ++idx) {
        const double m = score(kAll.p[idx]);
        if (takes_max(m, best, idx)) {
            best = m;
            best_idx = idx;
#pragma unroll
            for (int j = 0; j < SA; ++j) best_p[j] = kAll.p[idx][j];
        }
    }
    return best;
}

// Calls f(std::integral_constant<int, n>()) for the source counts 1..4 the kernels are instantiated for.
template <class F> static int with_sources(int n, const F& f) {
    if (n == 1) return f(std::integral_constant<int, 1>());
    if (n == 2) return f(std::integral_constant<int, 2>());
    if (n == 3) return f(std::integral_constant<int, 3>());
    if (n == 4) return f(std::integral_constant<int, 4>());
    return SDR_ERR_UNSUPPORTED;       // the searches enumerate up to S! assignments per item; 4 sources = 24
}

// Blocks of 256 threads for a finalize kernel that strides over the batch, one item per thread.
static inline unsigned item_blocks(int B) {
    const long long fb = ((long long)B + 255) / 256;
    return (unsigned)(fb < 4096 ? fb : 4096);
}

}  // namespace sdr
