// Chunk-by-chunk streaming of the causal model (causal_improved_sudormrf_v3.py): the kernels a step adds to the GEMMs.
//
// The causal model has no normalisation layers, so a chunk can be run exactly from a small carried state per slot:
//   waveform context  [A][2*hop]          the last 2*hop input samples: encoder frame f reads samples
//                                         hop*f - 2*hop .. hop*f (the causal mask keeps k of its 2k-1 taps)
//   decoder carry     [S*A][hop+1]        partial overlap-add sums of the samples the next chunk's frames still reach
//   level histories   [U][D][10][Ci]      the last 10 inputs of every depthwise level, at that level's rate
// Every activation of a step is [channels][B*F] with columns (slot, frame), F = C / hop frames per slot; the 1x1
// convolutions are one GEMM each over all columns.  Chunks start on multiples of 2^(D-1) frames, so every level's
// chunk starts on an integer position of that level.  All state starts at zero, the reference's zero padding.
#include "common.cuh"
#include "launchers.cuh"

namespace sdr {

constexpr int kStMaxF = 4096;        // frames per slot and step the stream stage takes
constexpr int kStHist = 10;          // history per level: a level-d output p reads inputs stride*p - 10 .. stride*p
constexpr int kStTaps = 11;          // taps that survive the causal mask of a 21-tap filter
constexpr int kStFilter = 21;
constexpr int kStThreads = 128;
constexpr int kStMaxRows = 32;       // channels per CTA (a power of two, so a thread keeps one channel: kStThreads % R == 0)
constexpr int kStSmemSmall = 48 * 1024;
constexpr int kStSmemMax = 64 * 1024;

// ---------------------------------------------------------------------------
// framing: the encoder's operand [Kr][B*F], row a*k + j of column (b, f) = sample hop*f + j - 2*hop of slot b's
// audio channel a (negative indices from the context); rows A*k .. Kr-1 are zeros (the tensor-core image pads the
// taps to a whole k-block).  The context is only read here; the overlap-add kernel advances it.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
stream_frame_kernel(const float* __restrict__ chunk, const float* __restrict__ state, long long slot_stride,
                    float* __restrict__ framed, int A, int k, int Kr, int F, int BF, long long C) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)Kr * BF) return;
    const int r = (int)(i / BF), col = (int)(i - (long long)r * BF);
    float v = 0.f;
    if (r < A * k) {
        const int hop = k / 2;
        const int a = r / k, j = r - a * k;
        const int b = col / F, f = col - b * F;
        const long long s = (long long)hop * f + j - 2 * hop;
        v = s < 0 ? __ldg(state + b * slot_stride + a * 2 * hop + 2 * hop + s)
                  : __ldg(chunk + ((size_t)b * A + a) * C + s);
    }
    framed[i] = v;
}

int launch_stream_frame(const float* chunk, const float* state, long long slot_stride, float* framed, int B, int A,
                        int k, int Kr, int F, long long C, cudaStream_t st) {
    const long long n = (long long)Kr * B * F;
    return launch(stream_frame_kernel, (unsigned)((n + 255) / 256), 256, 0, st, chunk, state, slot_stride, framed, A,
                  k, Kr, F, B * F, C);
}

// ---------------------------------------------------------------------------
// stream stage of the causal U-ConvBlock: the D levels of causal_pyramid_kernel (causal.cu) over one chunk, with the
// history of every level in front of its input.  One CTA owns R channels of one slot; every buffer is
// [position][channel] in shared memory:
//   X_d  level d's input: 10 history values, then F (d = 0) or F >> (d-1) new ones, PReLU applied (PReLU_p(y) for
//        d = 0, o_{d-1} for d >= 1);  level d < D-1 writes its output into X_{d+1} after the history
//   O    level D-1's output (F >> (D-1) positions)
// Taps, fmaf order and PReLU are those of causal_pyramid_kernel, so m is bitwise what the one-pass kernel computes
// over the concatenated chunks.  R = 32 for short chunks (history and y reads are whole lines); long chunks take
// fewer channels per CTA, down to one, so that the buffers fit in shared memory.
// ---------------------------------------------------------------------------
struct StreamStageArgs {
    const float* y;                  // [C][B*F] raw proj_1x1 output
    float* m;                        // [C][B*F] merged output
    float* hist;                     // slot 0's [D][10][C] histories; slot b at hist + b * hist_stride
    long long hist_stride;
    const float* slope_in;
    const float* w[kMaxDepthApi];
    const float* b[kMaxDepthApi];
    const float* slope[kMaxDepthApi];
    int D, C, B, F, R;
    int xoff[kMaxDepthApi];          // first position of X_d in shared memory (times R: float offset)
    int ooff;
};

__host__ __device__ __forceinline__ int st_nin(int d, int F) { return d == 0 ? F : F >> (d - 1); }

__global__ void __launch_bounds__(kStThreads)
causal_stream_kernel(const StreamStageArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, nthr = blockDim.x;
    const int R = a.R, D = a.D, F = a.F;
    const int slot = blockIdx.y;
    const int c0 = blockIdx.x * R;
    const int nr = min(R, a.C - c0);
    const long long BF = (long long)a.B * F;
    float* hb = a.hist + slot * a.hist_stride;

    // ---- histories -> X_d[0, 10)
#pragma unroll
    for (int d = 0; d < kMaxDepthApi; ++d) {
        if (d >= D) continue;
        for (int i = tid; i < kStHist * R; i += nthr) {
            const int row = i % R, j = i / R;
            if (row < nr) smem[(a.xoff[d] + j) * R + row] = hb[((size_t)d * kStHist + j) * a.C + c0 + row];
        }
    }
    // ---- y -> X_0[10, 10 + F), PReLU of proj_1x1 on the way
    {
        const float sp = __ldg(a.slope_in);
        const bool sp1 = sp <= 1.f;
        const int nq = F >> 2;
        for (int i = tid; i < R * nq; i += nthr) {
            const int row = i / nq, q = i - row * nq;
            if (row >= nr) continue;
            const float4 v = ldg4(a.y + (size_t)(c0 + row) * BF + (size_t)slot * F + 4 * q);
            float* dst = smem + (a.xoff[0] + kStHist + 4 * q) * R + row;
            dst[0] = prelu2(v.x, sp, sp1); dst[R] = prelu2(v.y, sp, sp1);
            dst[2 * R] = prelu2(v.z, sp, sp1); dst[3 * R] = prelu2(v.w, sp, sp1);
        }
    }
    __syncthreads();

    // ---- levels (R divides the thread count: a thread keeps one channel, and its taps, for the whole level)
    const int row = tid % R;
    const int c = c0 + row;
#pragma unroll
    for (int d = 0; d < kMaxDepthApi; ++d) {
        if (d >= D) continue;                           // uniform across the CTA: the barriers stay matched
        float w[kStTaps];
        float bias = 0.f, sl = 1.f;
        if (row < nr) {
            const float* wp = a.w[d] + (size_t)c * kStFilter;
#pragma unroll
            for (int j = 0; j < kStTaps; ++j) w[j] = __ldg(wp + j);
            bias = __ldg(a.b[d] + c);
            sl = __ldg(a.slope[d]);
        }
        const bool sl1 = sl <= 1.f;
        const int stride = d == 0 ? 1 : 2;
        const float* in = smem + a.xoff[d] * R + row;
        float* out = smem + (d + 1 < D ? a.xoff[d + 1] + kStHist : a.ooff) * R + row;
        const int n = F >> d;
        if (row < nr) {
            for (int p = tid / R; p < n; p += nthr / R) {
                const float* x = in + stride * p * R;
                float acc = bias;
#pragma unroll
                for (int j = 0; j < kStTaps; ++j) acc = fmaf(w[j], x[j * R], acc);
                out[p * R] = prelu2(acc, sl, sl1);
            }
        }
        __syncthreads();
    }

    // ---- new histories: the last 10 entries of every X_d
#pragma unroll
    for (int d = 0; d < kMaxDepthApi; ++d) {
        if (d >= D) continue;
        const int nin = st_nin(d, F);
        for (int i = tid; i < kStHist * R; i += nthr) {
            const int r = i % R, j = i / R;
            if (r < nr) hb[((size_t)d * kStHist + j) * a.C + c0 + r] = smem[(a.xoff[d] + nin + j) * R + r];
        }
    }

    // ---- merge m[t] = sum_d o_d[t >> d] (causal_pyramid_kernel's order), four positions per thread
    {
        const int nq = F >> 2;
        for (int i = tid; i < R * nq; i += nthr) {
            const int r = i / nq, q = i - r * nq;
            if (r >= nr) continue;
            auto lvl = [&](int d, int p) -> float {
                return smem[((d + 1 < D ? a.xoff[d + 1] + kStHist : a.ooff) + p) * R + r];
            };
            const int t = 4 * q;
            float4 v = make_float4(lvl(0, t), lvl(0, t + 1), lvl(0, t + 2), lvl(0, t + 3));
            if (D > 1) {
                const float p = lvl(1, t >> 1), s = lvl(1, (t >> 1) + 1);
                v.x += p; v.y += p; v.z += s; v.w += s;
                float deep = 0.f;
#pragma unroll
                for (int d = 2; d < kMaxDepthApi; ++d)
                    if (d < D) deep += lvl(d, t >> d);
                v.x += deep; v.y += deep; v.z += deep; v.w += deep;
            }
            *reinterpret_cast<float4*>(a.m + (size_t)(c0 + r) * BF + (size_t)slot * F + t) = v;
        }
    }
}

// Chunk lengths the stream stage takes: whole float4 rows, an integer position at every level, the buffers of one
// channel within shared memory.
bool causal_stream_eligible(int D, int F) {
    return D >= 1 && D <= kMaxDepthApi && F >= 4 && F <= kStMaxF && (F % 4) == 0 && (F % (1 << (D - 1))) == 0;
}

int launch_causal_stream(const float* y, const float* slope_in, const float* const* w, const float* const* b,
                         const float* const* slope, float* hist, long long hist_stride, float* m, int D, int B, int C,
                         int F, cudaStream_t st) {
    if (!y || !m || !hist || !slope_in || !w || !b || !slope || B <= 0 || C <= 0) return SDR_ERR_BAD_ARGUMENT;
    if (!causal_stream_eligible(D, F) || B > 65535) return SDR_ERR_UNSUPPORTED;
    if ((long long)B * F > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(m)) % 16) return SDR_ERR_UNSUPPORTED;
    StreamStageArgs a;
    a.y = y; a.m = m; a.hist = hist; a.hist_stride = hist_stride; a.slope_in = slope_in;
    a.D = D; a.C = C; a.B = B; a.F = F;
    int pos = 0;
    for (int d = 0; d < kMaxDepthApi; ++d) {
        a.w[d] = d < D ? w[d] : nullptr; a.b[d] = d < D ? b[d] : nullptr; a.slope[d] = d < D ? slope[d] : nullptr;
        a.xoff[d] = 0;
        if (d < D) { a.xoff[d] = pos; pos += kStHist + st_nin(d, F); }
    }
    a.ooff = pos;
    pos += F >> (D - 1);
    int R = kStMaxRows;
    while (R > 1 && (size_t)R * pos * sizeof(float) > kStSmemSmall) R >>= 1;
    const size_t smem = (size_t)R * pos * sizeof(float);
    if (smem > kStSmemMax) return SDR_ERR_UNSUPPORTED;
    a.R = R;
    return launch(causal_stream_kernel, dim3((unsigned)ceil_div(C, R), (unsigned)B), kStThreads, smem, st, a);
}

// ---------------------------------------------------------------------------
// overlap-add of one step: frames [SA*k][B*F] (row s*k + j, column (b, f)) -> out[b][s][p], p in [0, C), which is the
// model's output sample c*C - hop + p.  Frame f of the chunk reaches p = hop*f + j, j in [0, k); p <= hop also holds
// the carry of the earlier frames, p >= C goes to the new carry.  Frames are added in ascending order onto the carry,
// as overlap_add_kernel adds them.  Optionally the uniform mixture-consistency projection against the mixture
// delayed by hop (mono).  Block 0 of a slot owns every access to the slot's carry and context: it reads the carry
// (p <= hop) and the old context (p < hop) before it writes the new ones, so no other CTA sees them half-updated.
// ---------------------------------------------------------------------------
constexpr int kOlaThreads = 256;
constexpr int kStMaxSrc = 16;

__device__ __forceinline__ float ola_sum(const float* __restrict__ frames, int s, int k, int hop, int F, long long BF,
                                         int col0, int p, float acc) {
    int flo = p - (k - 1);
    flo = flo <= 0 ? 0 : (flo + hop - 1) / hop;
    const int fhi = min(p / hop, F - 1);
    for (int f = flo; f <= fhi; ++f) acc += __ldg(frames + (size_t)(s * k + p - hop * f) * BF + col0 + f);
    return acc;
}

__global__ void __launch_bounds__(kOlaThreads)
stream_ola_kernel(const float* __restrict__ frames, const float* __restrict__ chunk, float* __restrict__ state,
                  long long slot_stride, long long carry_off, float* __restrict__ out, int SA, int A, int k, int F,
                  int B, long long C, int mc) {
    const int hop = k / 2;
    const int b = blockIdx.y, tid = threadIdx.x;
    const long long BF = (long long)B * F;
    const int col0 = b * F;
    float* ctx = state + b * slot_stride;                 // [A][2*hop]
    float* carry = ctx + carry_off;                       // [SA][hop+1], then the started flag
    float est[kStMaxSrc];
    if (blockIdx.x > 0) {
        const long long p = hop + 1 + (long long)(blockIdx.x - 1) * kOlaThreads + tid;
        if (p >= C) return;
        float sum = 0.f;
        for (int s = 0; s < SA; ++s) { est[s] = ola_sum(frames, s, k, hop, F, BF, col0, (int)p, 0.f); sum += est[s]; }
        float corr = 0.f;
        if (mc) corr = (__ldg(chunk + (size_t)b * C + p - hop) - sum) * (1.0f / SA);   // mixture_consistency.py:29-35
        for (int s = 0; s < SA; ++s) out[((size_t)b * SA + s) * C + p] = est[s] + corr;
        return;
    }
    // block 0: head p = tid in [0, hop] (carry + frames), tail q = tid - hop - 1 in [0, hop] (new carry)
    const bool head = tid <= hop, tail = !head && tid <= 2 * hop + 1;
    // the first step of a slot: p < hop precede the stream (the reference crops them), written as zeros
    const bool before_start = tid < hop && carry[SA * (hop + 1)] == 0.f;
    float corr = 0.f;
    if (head) {
        float sum = 0.f;
        for (int s = 0; s < SA; ++s) { est[s] = ola_sum(frames, s, k, hop, F, BF, col0, tid, carry[s * (hop + 1) + tid]); sum += est[s]; }
        if (mc) {
            const float mix = tid < hop ? ctx[hop + tid] : __ldg(chunk + (size_t)b * C);
            corr = (mix - sum) * (1.0f / SA);
        }
    } else if (tail) {
        const int q = tid - hop - 1;
        for (int s = 0; s < SA; ++s) est[s] = ola_sum(frames, s, k, hop, F, BF, col0, (int)C + q, 0.f);
    }
    __syncthreads();
    if (head) {
        for (int s = 0; s < SA; ++s) out[((size_t)b * SA + s) * C + tid] = before_start ? 0.f : est[s] + corr;
    } else if (tail) {
        const int q = tid - hop - 1;
        for (int s = 0; s < SA; ++s) carry[s * (hop + 1) + q] = est[s];
    }
    if (tid == 0) carry[SA * (hop + 1)] = 1.f;
    for (int i = tid; i < A * 2 * hop; i += kOlaThreads) {
        const int aa = i / (2 * hop), j = i - aa * 2 * hop;
        ctx[i] = __ldg(chunk + ((size_t)b * A + aa) * C + C - 2 * hop + j);
    }
}

int launch_stream_ola(const float* frames, const float* chunk, float* state, long long slot_stride, long long carry_off,
                      float* out, int B, int SA, int A, int k, int F, long long C, int mc, cudaStream_t st) {
    const int hop = k / 2;
    if (SA > kStMaxSrc || 2 * hop + 2 > kOlaThreads || B > 65535 || C <= hop) return SDR_ERR_UNSUPPORTED;
    dim3 grid((unsigned)(1 + (C - hop - 1 + kOlaThreads - 1) / kOlaThreads), (unsigned)B);
    return launch(stream_ola_kernel, grid, kOlaThreads, 0, st, frames, chunk, state, slot_stride, carry_off, out, SA, A,
                  k, F, B, C, mc);
}

// The pending tail: the model's output samples n*C - hop .. n*C - 1 are the carry (no later frame reaches them once
// the stream ends), with the mixture-consistency projection against the context's last hop samples.  State unchanged.
__global__ void stream_flush_kernel(const float* __restrict__ state, long long slot_stride, long long carry_off,
                                    float* __restrict__ tail, int SA, int hop, int B, int mc) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * hop) return;
    const int b = (int)(i / hop), p = (int)(i - (long long)b * hop);
    const float* ctx = state + b * slot_stride;
    const float* carry = ctx + carry_off;
    float est[kStMaxSrc];
    float sum = 0.f;
    for (int s = 0; s < SA; ++s) { est[s] = carry[s * (hop + 1) + p]; sum += est[s]; }
    const float corr = mc ? (ctx[hop + p] - sum) * (1.0f / SA) : 0.f;
    for (int s = 0; s < SA; ++s) tail[((size_t)b * SA + s) * hop + p] = est[s] + corr;
}

int launch_stream_flush(const float* state, long long slot_stride, long long carry_off, float* tail, int B, int SA,
                        int hop, int mc, cudaStream_t st) {
    if (SA > kStMaxSrc) return SDR_ERR_UNSUPPORTED;
    const long long n = (long long)B * hop;
    return launch(stream_flush_kernel, (unsigned)((n + 255) / 256), 256, 0, st, state, slot_stride, carry_off, tail, SA,
                  hop, B, mc);
}

// Zeroes the slot_bytes (a multiple of 4) of every slot b < B of `base` whose mask[b] is set: a reset whose slots are
// chosen on the device, so that a captured graph can run it.
__global__ void zero_masked_slots_kernel(unsigned* __restrict__ base, long long words, long long total,
                                         const unsigned char* __restrict__ mask) {
    for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < total; e += (long long)gridDim.x * 256)
        if (mask[e / words]) base[e] = 0u;
}

static int launch_zero_masked_slots(void* base, int B, size_t slot_bytes, const unsigned char* mask, cudaStream_t st) {
    if (!base || !mask || B <= 0 || slot_bytes % 4 || reinterpret_cast<uintptr_t>(base) % 4) return SDR_ERR_BAD_ARGUMENT;
    const long long words = (long long)(slot_bytes / 4), total = words * B;
    if (total == 0) return SDR_OK;
    const long long grid = std::min((total + 255) / 256, (long long)std::max(sm_count(), 1) * 8);
    return launch(zero_masked_slots_kernel, (unsigned)grid, 256, 0, st, static_cast<unsigned*>(base), words, total,
                  mask);
}

// Zeroes slot b of every region for the n slots listed on the host (all checked before the first memset) or the slots
// whose mask[b] is set (one launch per region); exactly one of `slots` and `mask` is given.
int reset_slots(std::initializer_list<SlotRegion> regions, int B, const int* slots, int n, const unsigned char* mask,
                cudaStream_t st) {
    if (mask) {
        for (const SlotRegion& r : regions)
            if (const int e = launch_zero_masked_slots(r.base, B, r.slot_bytes, mask, st)) return e;
        return SDR_OK;
    }
    for (int i = 0; i < n; ++i)
        if (slots[i] < 0 || slots[i] >= B) return SDR_ERR_BAD_ARGUMENT;
    for (int i = 0; i < n; ++i)
        for (const SlotRegion& r : regions)
            if (const int e = cuda_status(cudaMemsetAsync(static_cast<char*>(r.base) + (size_t)slots[i] * r.slot_bytes,
                                                          0, r.slot_bytes, st)))
                return e;
    return SDR_OK;
}

}  // namespace sdr
