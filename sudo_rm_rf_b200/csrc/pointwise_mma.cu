// 1x1 Conv1d on the Hopper tensor cores (wgmma, TMA, mbarrier), sm_90a.
//
//   y[s, m, l] = sum_k W[m, k] * f(x[s, k, l]) + bias[m]   (+ residual | relu()*gate)
//
// GEMM view per tile: D[128 positions, 128 channels] = A[128, K] * B[128, K]^T with
//   A = f(x) tile, produced on the fly: the activation tile cannot be TMA'd
//       straight into the MMA because the producer's deferred GlobLN(+PReLU)
//       has to be applied first.  A TMA warp lands the raw fp32 tile in shared
//       memory; 8 transform warps apply the per-channel affine (+PReLU), split
//       the fp32 value into bf16 hi + bf16 lo, and store both into the MN-major
//       SWIZZLE_128B shared-memory layout the wgmma descriptors expect.
//   B = weights, pre-split into bf16 hi/lo and pre-swizzled at pack time, so a
//       k-block is ONE TMA box of a contiguous image.
//   D = fp32 accumulator in registers: two consumer warpgroups, each owning 64
//       positions x 128 channels (64 registers per thread), issue the wgmmas
//       and run the epilogue.  Persistent CTAs, one per SM; the transform and
//       TMA warps run ahead into the free stages while the consumers drain.
// Precision: x*w ~= xh*wh + xl*wh + xh*wl (3 bf16 MMAs, fp32 accumulate): the
// dropped terms are O(2^-16) relative, i.e. fp32-grade for the 1e-3 parity
// budget, where a single bf16 (5e-3) or tf32 (7e-4) pass is not (SURVEY §7).
//
// Replaces (reference file:line): bottleneck improved_sudormrf.py:256-259,292;
// proj_1x1.conv :174,205; res_conv(+skip) :196,220; mask_net :268-269,295-298.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>
#include <cuda.h>
#include <cuda_bf16.h>
#include "common.cuh"

namespace sdr {

constexpr int kTileM = 128;            // positions per CTA tile (2 consumer warpgroups x wgmma M = 64)
constexpr int kTileN = 128;            // output channels per tile (wgmma N); 64 fp32 accumulator registers per thread
constexpr int kBlockK = 64;            // channels per k-block = one 128 B swizzle row of bf16
constexpr int kStages = 2;             // A (transformed activations) and B (weights) stages share one full/empty barrier ring
constexpr int kRawStages = 2;          // fp32 [64 channels][128 positions] tiles landed by TMA, read once by the transform warps
constexpr int kRawStageBytes = kTileM * kBlockK * 4;         // 32 KB
constexpr int kAHalf = kTileM * 128;   // 16 KB: bf16 [128 rows][64 k]
constexpr int kBHalf = kTileN * 128;   // 16 KB: bf16 [128 weight rows][64 k]
constexpr int kAStageBytes = 2 * kAHalf;                     // 32 KB: hi + lo
constexpr int kBStageBytes = 2 * kBHalf;                     // 32 KB: hi + lo
// Warp roles: [0, 8) the two consumer warpgroups (wgmma + epilogue), [8, 16) operand transform, 16 weight TMA,
// 17 raw activation TMA.
constexpr int kConsWarps = 8, kProdWarp0 = 8, kProdWarps = 8, kTmaWarp = 16, kRawWarp = 17;
constexpr int kMmaThreads = 32 * (kRawWarp + 1);             // 576
constexpr int kProdThreads = 32 * kProdWarps;                // 256
constexpr int kProdElems = kTileM * kBlockK / kProdThreads;  // 32 = 8 channels x 4 positions per thread and k-block
static_assert(kProdWarps == 8 && kProdElems == 32, "one transform warp per 8-channel k-group, 4 positions per lane");

struct MmaArgs {
    const float* x;
    NormIn nin;
    const float* bias;
    const float* residual;
    const float* gate;
    int gate_channels;
    float* y;
    double* stats_out;
    int M, K, L;
    int l_tiles, n_tiles;
    int num_tiles;        // n_tiles * samples * l_tiles; tile t covers channel tile t % n_tiles of position tile t / n_tiles
    int epilogue;
    // window mode (encoder Conv1d as a GEMM without im2col): operand element (position p, k = a*win_k + j)
    // is wav[sample, a, win_hop * p + j - win_pad] (zero outside [0, win_T)); x = wav, K = padded taps
    int win_k;            // 0 = normal pointwise mode
    int win_hop, win_pad, win_a;
    long long win_T;
};

// ---------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    } while (!done);
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// global -> shared tensor (TMA) loads; out-of-range elements arrive as zeros
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// wgmma shared-memory matrix descriptor (cute/arch/mma_sm90_desc.hpp documents the bit layout): start address >> 4
// in [0,14), leading byte offset >> 4 in [16,30), stride byte offset >> 4 in [32,46), layout type 1 (SWIZZLE_128B)
// in [62,64).  Stage bases are 1024 B aligned, so the base offset field stays 0.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// A operand, MN-major (positions contiguous).  Canonical layout in 16 B units ((8,n),(8,k)):((1,LBO),(8,SBO)): a 128 B
// row holds 64 consecutive positions of one k; 8 k-rows form a 1024 B atom (16 B chunk index XOR k%8); LBO = byte
// stride between 64-wide position blocks (one per consumer warpgroup), SBO = byte stride between groups of 8 k.
constexpr uint32_t kALbo = 1024;       // A tile: [8 k-groups][2 position blocks][8 k rows][128 B]
constexpr uint32_t kASbo = 2048;
// B operand, K-major: 128 B per weight row, 8-row groups 1024 B apart (LBO unused for swizzled K-major, canonical 16 B).
constexpr uint32_t kBLbo = 16, kBSbo = 1024;

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T for the executing warpgroup; A MN-major (imm-trans-a = 1), B K-major.
// Thread t of the warpgroup holds d[i] at row 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2),
// column 8 * (i / 4) + 2 * (t % 4) + i % 2.
__device__ __forceinline__ void wgmma_bf16_m64n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
        "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, "
        "%45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}

// ---------------------------------------------------------------------------
// weight packing: W[M][K] fp32 -> per (n_tile, k_block) a contiguous image of 2 x kTileN rows x 128 B
// [hi: the tile's weight rows | lo: the same rows], rows swizzled exactly as they must sit in shared memory
// (16 B chunk index XOR row % 8), so a k-block is ONE TMA box of [2 * kTileN][128 B].
// ---------------------------------------------------------------------------
__global__ void pack_weight_mma_kernel(const float* __restrict__ W, uint8_t* __restrict__ out,
                                       int M, int Mpad, int Kreal, int K) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one 16 B chunk (8 k) per thread
    const long long chunks = (long long)Mpad * K / 8;
    if (i >= chunks) return;
    const int kc = (int)(i % (K / 8));        // chunk index along K
    const int m = (int)(i / (K / 8));
    const int kb = kc / 8, c = kc % 8;
    const int nt = m / kTileN, r = m % kTileN;
    const int KB = K / kBlockK;
    uint8_t* img = out + ((size_t)nt * KB + kb) * kBStageBytes;
    const size_t off = (size_t)(r >> 3) * 1024 + (size_t)(r & 7) * 128 + (size_t)((c ^ (r & 7)) << 4);
    __nv_bfloat16 hi[8], lo[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const int k = kc * 8 + e;                                          // rows >= M, taps >= Kreal: zero padding
        const float v = (m < M && k < Kreal) ? W[(size_t)m * Kreal + k] : 0.f;
        hi[e] = __float2bfloat16_rn(v);
        lo[e] = __float2bfloat16_rn(v - __bfloat162float(hi[e]));
    }
    *reinterpret_cast<uint4*>(img + off) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(img + kBHalf + off) = *reinterpret_cast<const uint4*>(lo);
}

// ---------------------------------------------------------------------------
// the GEMM kernel
// ---------------------------------------------------------------------------
struct TileCoord { int sample, l0, n0; };
// Consecutive tiles share a position tile (the CTAs working on its channel tiles read the same activations from L2).
__device__ __forceinline__ TileCoord decode_tile(const MmaArgs& a, int tile) {
    TileCoord t;
    const int pos = tile / a.n_tiles;
    t.n0 = (tile - pos * a.n_tiles) * kTileN;
    t.sample = pos / a.l_tiles;
    t.l0 = (pos - t.sample * a.l_tiles) * kTileM;
    return t;
}

// Compile-time specialisation keeps the hot loops small.
//   WINDOW: encoder mode (strided waveform windows as the A operand)
//   ACT:    PReLU in the operand transform: 0 none, 1 one shared slope (nn.PReLU()), 2 one slope per input
//           channel (nn.PReLU(C) of the original model, sudormrf.py:33,71; shared -> shared transform loop only)
//   MODE:   epilogue 0 = bias only, 1 = + residual (may alias y: every element is read by the thread that writes it),
//           2 = ReLU * gate
//   STATS:  accumulate (sum, sumsq) of the output
template <bool WINDOW, int ACT, int MODE, bool STATS>
__global__ void __launch_bounds__(kMmaThreads, 1)
pw_mma_kernel(const MmaArgs a, const __grid_constant__ CUtensorMap wmap,      // wmap: packed weights as [rows][128 B]
              const __grid_constant__ CUtensorMap xmap) {                     // xmap: activations [samples][K][L], box [64][128]
    // 2 x (32 KB A stage + 32 KB B stage) + 2 x 32 KB raw tiles + 4 KB of tables + barriers (of the 227 KB an sm_90
    // CTA can own).  SWIZZLE_128B needs the stage bases 1024 B aligned; the launch reserves 1 KB to align by hand.
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* a_base = smem;                                                  // kStages x 32 KB
    uint8_t* b_base = smem + kStages * kAStageBytes;                         // kStages x 32 KB
    uint8_t* r_base = b_base + kStages * kBStageBytes;                       // kRawStages x 32 KB
    // warp-private tables (no CTA-level barrier in the steady state): per transform warp the (scale, shift) of its
    // channels, double-buffered
    float2* s_ab = reinterpret_cast<float2*>(r_base + kRawStages * kRawStageBytes);   // [kProdWarps][64]
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_ab + kProdWarps * 64);
    //   full_bar:   the 8 transform warps + the weight TMA thread (with the weights' tx bytes); waited on by the consumers
    //   empty_bar:  the 8 consumer warps once their wgmmas reading the stage have retired
    //   rfull_bar:  raw tile landed (TMA tx bytes); rempty_bar: all 8 transform warps hold it in registers
    uint64_t* full_bar = bars;                       // [kStages]
    uint64_t* empty_bar = full_bar + kStages;        // [kStages]
    uint64_t* rfull_bar = empty_bar + kStages;       // [kRawStages]
    uint64_t* rempty_bar = rfull_bar + kRawStages;   // [kRawStages]

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int KB = a.K / kBlockK;
    const int tile0 = (int)blockIdx.x;               // tiles of this CTA: tile0, tile0 + tstep, ...
    const int tstep = (int)gridDim.x;

    if (warp == kTmaWarp && lane == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], kProdWarps + 1); mbar_init(&empty_bar[s], kConsWarps); }
        for (int s = 0; s < kRawStages; ++s) { mbar_init(&rfull_bar[s], 1); mbar_init(&rempty_bar[s], kProdWarps); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp >= kProdWarp0 && warp < kProdWarp0 + kProdWarps) {
        // ===================== A-operand transform producers =====================
        // Warp w owns the 8 channels of k-group w of every k-block; lane i owns positions 4i..4i+3.
        // Per channel a thread reads one float4, applies the folded normalisation (+PReLU), splits bf16 hi/lo,
        // and does two conflict-free 8-byte stores into the MN-major SWIZZLE_128B tile (row = channel, 64
        // positions per 128 B row).
        const int pw = warp - kProdWarp0;          // k-group (8 channels) of this warp
        const int p4 = lane * 4;                   // first of this lane's 4 positions in the tile
        const bool has_norm = a.nin.stats != nullptr;
        const float slope = ACT == 1 ? __ldg(a.nin.prelu) : 1.f;
        const bool slope_le1 = slope <= 1.f;
        float2* const my_tab = s_ab + pw * 64;     // this warp's [2][8] (scale, shift) table (lane e < 8); ACT == 2: the
                                                   // channels' PReLU slopes in entries [16, 32) of the same 64-entry slice
        static_assert(!(WINDOW && ACT != 0), "the encoder's window operand has no activation");
        const double inv_count = 1.0 / a.nin.count;
        // byte offset of (channel row e = 0, this lane's positions) inside an A half tile
        const uint32_t lane_off = (uint32_t)pw * kASbo + (uint32_t)(lane >> 4) * kALbo + (uint32_t)(lane & 1) * 8;
        const uint32_t lane_chunk = (uint32_t)((lane & 15) >> 1);

        struct Cur { int tile, kb; TileCoord tc; };
        auto advance = [&](Cur& c) {              // next (tile, k-block) of this CTA; tile >= num_tiles == end
            if (++c.kb == KB) {
                c.kb = 0;
                c.tile += tstep;
                if (c.tile < a.num_tiles) c.tc = decode_tile(a, c.tile);
            }
        };
        struct Aux { float g, b; double s0, s1; float sl; };
        auto load_aux = [&](const Cur& c) -> Aux {   // lane e: gamma/beta of channel e of this warp's k-group
            Aux x{1.f, 0.f, 0.0, 1.0, 1.f};
            if constexpr (ACT == 2) {
                if (c.tile < a.num_tiles) x.sl = __ldg(a.nin.prelu + c.kb * kBlockK + pw * 8 + (lane & 7));
            }
            if (has_norm && c.tile < a.num_tiles) {
                const int k = c.kb * kBlockK + pw * 8 + (lane & 7);
                x.g = __ldg(a.nin.gamma + k);
                x.b = __ldg(a.nin.beta + k);
                if (c.kb == 0) {                   // new tile: its sample's (sum, sumsq)
                    x.s0 = a.nin.stats[2 * (size_t)c.tc.sample];
                    x.s1 = a.nin.stats[2 * (size_t)c.tc.sample + 1];
                }
            }
            return x;
        };
        // one stage's 8 channel rows (4 positions each) -> folded affine (+PReLU) -> bf16 hi/lo into A stage `stage`
        auto store_rows = [&](const float4 (&v)[8], const float2 (&abv)[8], const float (&slv)[ACT == 2 ? 8 : 1],
                              int stage) {
            uint8_t* a_hi = a_base + (size_t)stage * kAStageBytes;
            uint8_t* a_lo = a_hi + kAHalf;
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float2 ab = abv[e];
                float y[4] = {fmaf(v[e].x, ab.x, ab.y), fmaf(v[e].y, ab.x, ab.y),
                              fmaf(v[e].z, ab.x, ab.y), fmaf(v[e].w, ab.x, ab.y)};
                if constexpr (ACT == 1) {      // PReLU in 2 ops: max(y, s*y) for s <= 1, min otherwise
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const float t = y[u] * slope;
                        y[u] = slope_le1 ? fmaxf(y[u], t) : fminf(y[u], t);
                    }
                } else if constexpr (ACT == 2) {   // this channel's own slope (either side of 1, either sign)
                    const float sl = slv[ACT == 2 ? e : 0];
#pragma unroll
                    for (int u = 0; u < 4; ++u) y[u] = y[u] >= 0.f ? y[u] : y[u] * sl;
                }
                // hi = top 16 bits (truncation), lo = bf16(y - hi): y - hi is exact in fp32, so
                // |y - hi - lo| <= 2^-9 |y - hi| <= 2^-16 |y|
                uint32_t hb[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) hb[u] = __float_as_uint(y[u]) & 0xffff0000u;
                const uint32_t h01 = __byte_perm(hb[0], hb[1], 0x7632), h23 = __byte_perm(hb[2], hb[3], 0x7632);
                const __nv_bfloat162 l01 = __floats2bfloat162_rn(y[0] - __uint_as_float(hb[0]), y[1] - __uint_as_float(hb[1]));
                const __nv_bfloat162 l23 = __floats2bfloat162_rn(y[2] - __uint_as_float(hb[2]), y[3] - __uint_as_float(hb[3]));
                const uint32_t off = lane_off + (uint32_t)e * 128 + ((lane_chunk ^ (uint32_t)e) << 4);
                *reinterpret_cast<uint2*>(a_hi + off) = make_uint2(h01, h23);
                *reinterpret_cast<uint2*>(a_lo + off) = make_uint2(*reinterpret_cast<const uint32_t*>(&l01),
                                                                    *reinterpret_cast<const uint32_t*>(&l23));
            }
            fence_proxy_async_smem();          // generic-proxy stores -> visible to the tensor core (async proxy)
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[stage]);
        };

        Cur c;
        c.tile = tile0; c.kb = 0;
        if (c.tile < a.num_tiles) {
            c.tc = decode_tile(a, c.tile);
            Aux aux = load_aux(c);
            uint32_t it = 0;
            int stage = 0, rs = 0;
            uint32_t phase = 0, rphase = 0;    // parities of the ring passes
            float mean = 0.f, rstd = 1.f;      // of the current tile's sample
            const uint32_t raw_lane = (uint32_t)(pw * 8) * 512u + (uint32_t)lane * 16u;
#pragma unroll 1
            while (c.tile < a.num_tiles) {
                Cur n = c;
                advance(n);                    // next step (n.tile >= num_tiles: none)
                {                              // y = x * aa + bb  ==  gamma * (x - mean) * rstd + beta
                    float aa = 1.f, bb = 0.f;
                    if (has_norm) {
                        if (c.kb == 0) {
                            const double mu = aux.s0 * inv_count;
                            double var = aux.s1 * inv_count - mu * mu;
                            var = var < 0.0 ? 0.0 : var;
                            mean = (float)mu;
                            rstd = rsqrtf((float)var + kGlnEps);
                        }
                        aa = aux.g * rstd;
                        bb = aux.b - mean * aa;
                    }
                    if (lane < 8) {
                        my_tab[(it & 1) * 8 + lane] = make_float2(aa, bb);
                        if constexpr (ACT == 2) my_tab[16 + (it & 1) * 8 + lane] = make_float2(aux.sl, 0.f);
                    }
                    aux = load_aux(n);
                }
                __syncwarp();                  // table visible to the warp (reuse is ordered by the next __syncwarp)
                const float2* tab = my_tab + (it & 1) * 8;
                float2 abv[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) abv[e] = tab[e];
                float slv[ACT == 2 ? 8 : 1] = {1.f};
                if constexpr (ACT == 2) {
#pragma unroll
                    for (int e = 0; e < 8; ++e) slv[e] = tab[16 + e].x;
                }
                float4 v[8];
                if constexpr (WINDOW) {        // encoder: strided analysis windows of the waveform, gathered directly
                    const int l = c.tc.l0 + p4;
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                        const int k = c.kb * kBlockK + pw * 8 + e;
                        const int ch = k / a.win_k, j = k - ch * a.win_k;
                        float vv[4];
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            const long long t = (long long)a.win_hop * (l + u) + j - a.win_pad;
                            vv[u] = (l + u < a.L && ch < a.win_a && t >= 0 && t < a.win_T)
                                        ? __ldg(a.x + ((size_t)c.tc.sample * a.win_a + ch) * a.win_T + t) : 0.f;
                        }
                        v[e] = make_float4(vv[0], vv[1], vv[2], vv[3]);
                    }
                } else {                       // the raw tile of this k-block, landed by the raw loader's TMA
                    mbar_wait(&rfull_bar[rs], rphase);
                    const uint8_t* rp = r_base + (size_t)rs * kRawStageBytes + raw_lane;
#pragma unroll
                    for (int e = 0; e < 8; ++e) v[e] = *reinterpret_cast<const float4*>(rp + e * 512);
                    __syncwarp();              // every lane holds its quads: the slot may be refilled
                    if (lane == 0) mbar_arrive(&rempty_bar[rs]);
                    if (++rs == kRawStages) { rs = 0; rphase ^= 1; }
                }
                mbar_wait(&empty_bar[stage], phase ^ 1);
                store_rows(v, abv, slv, stage);
                ++it;
                if (++stage == kStages) { stage = 0; phase ^= 1; }
                c = n;
            }
        }
    } else if (warp == kRawWarp) {
        // ===================== raw activation tiles: TMA producer =====================
        if (lane == 0 && !WINDOW) {
            int rs = 0;
            uint32_t rphase = 0;
            for (int tile = tile0; tile < a.num_tiles; tile += tstep) {
                const TileCoord tc = decode_tile(a, tile);
                for (int kb = 0; kb < KB; ++kb) {
                    mbar_wait(&rempty_bar[rs], rphase ^ 1);
                    mbar_arrive_expect_tx(&rfull_bar[rs], kRawStageBytes);
                    tma_load_3d(r_base + (size_t)rs * kRawStageBytes, &xmap, &rfull_bar[rs], tc.l0, kb * kBlockK, tc.sample);
                    if (++rs == kRawStages) { rs = 0; rphase ^= 1; }
                }
            }
        }
        __syncwarp();
    } else if (warp == kTmaWarp) {
        // ===================== B-operand (weights) TMA producer =====================
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = tile0; tile < a.num_tiles; tile += tstep) {
                const int nt = tile % a.n_tiles;
                for (int kb = 0; kb < KB; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&full_bar[stage], kBStageBytes);
                    tma_load_2d(b_base + (size_t)stage * kBStageBytes, &wmap, &full_bar[stage], 0, (nt * KB + kb) * 2 * kTileN);
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                }
            }
        }
        __syncwarp();
    } else if (warp < kConsWarps) {
        // ===================== consumers: wgmma main loop + epilogue from registers =====================
        const int wg = warp >> 2;                  // position block [64 wg, 64 wg + 64) of the tile
        const int wr = warp & 3;                   // 16-row slice of the warpgroup's block
        const size_t Ls = (size_t)a.L;
        const bool relu_out = WINDOW && a.epilogue == 2;       // window mode only: ReLU on the way out
        int stage = 0;
        uint32_t phase = 0;
        float acc[64];
#pragma unroll 1
        for (int tile = tile0; tile < a.num_tiles; tile += tstep) {
            const TileCoord tc = decode_tile(a, tile);
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = 0.f;
#pragma unroll 1
            for (int kb = 0; kb < KB; ++kb) {
                mbar_wait(&full_bar[stage], phase);   // A transformed, B landed
                const uint32_t sa_hi = smem_u32(a_base + (size_t)stage * kAStageBytes) + (uint32_t)wg * kALbo;
                const uint32_t sa_lo = sa_hi + kAHalf;
                const uint32_t sb_hi = smem_u32(b_base + (size_t)stage * kBStageBytes);
                const uint32_t sb_lo = sb_hi + kBHalf;
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < kBlockK / 16; ++ks) {
                    // A is MN-major: a K=16 step spans two 8-channel groups (2 * SBO bytes apart)
                    const uint64_t dah = gmma_desc_sw128(sa_hi + ks * 2 * kASbo, kALbo, kASbo);
                    const uint64_t dal = gmma_desc_sw128(sa_lo + ks * 2 * kASbo, kALbo, kASbo);
                    const uint64_t dbh = gmma_desc_sw128(sb_hi + ks * 32, kBLbo, kBSbo);
                    const uint64_t dbl = gmma_desc_sw128(sb_lo + ks * 32, kBLbo, kBSbo);
                    wgmma_bf16_m64n128(acc, dah, dbh, (kb | ks) != 0 ? 1u : 0u);
                    wgmma_bf16_m64n128(acc, dal, dbh, 1u);
                    wgmma_bf16_m64n128(acc, dah, dbl, 1u);
                }
                wgmma_commit();
                wgmma_wait_all();
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[stage]);   // this warp's reads of the stage have retired
                if (++stage == kStages) { stage = 0; phase ^= 1; }
            }
            // epilogue: lane owns positions p and p + 8, and channel pairs 8 j + 2 (lane % 4) + {0, 1}
            const int l = tc.l0 + wg * 64 + wr * 16 + (lane >> 2);
            const int ch0 = tc.n0 + 2 * (lane & 3);
            float st_s = 0.f, st_q = 0.f;
            const size_t gate_row0 = MODE == 2 ? (size_t)tc.sample * a.gate_channels + (tc.n0 % a.gate_channels) - tc.n0 : 0;
#pragma unroll
            for (int i = 0; i < 64; ++i) {
                const int m = ch0 + 8 * (i >> 2) + (i & 1);
                const int p = l + 8 * ((i >> 1) & 1);
                if (m < a.M && p < a.L) {
                    float o = acc[i] + (a.bias ? __ldg(a.bias + m) : 0.f);
                    const size_t idx = ((size_t)tc.sample * a.M + m) * Ls + p;
                    if (MODE == 1) o += a.residual[idx];           // plain load: may alias y
                    if (MODE == 2) o = fmaxf(o, 0.f) * __ldg(a.gate + (gate_row0 + m) * Ls + p);
                    if constexpr (WINDOW) { if (relu_out) o = fmaxf(o, 0.f); }   // the original model's encoder (sudormrf.py:212-218)
                    a.y[idx] = o;
                    if (STATS) { st_s += o; st_q = fmaf(o, o, st_q); }
                }
            }
            if (STATS) {
                st_s = warp_sum(st_s);
                st_q = warp_sum(st_q);
                if (lane == 0) {
                    atomicAdd(a.stats_out + 2 * (size_t)tc.sample, (double)st_s);
                    atomicAdd(a.stats_out + 2 * (size_t)tc.sample + 1, (double)st_q);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
static inline int mma_pad_m(int M) { return (M + kTileN - 1) / kTileN * kTileN; }

// Output-channel counts that are not a multiple of 128 are zero-padded (decoder: 2*21 = 42 rows);
// the reduction dimension must fill whole 64-channel k-blocks.
bool pointwise_mma_eligible(int M, int K) {
    return M >= 32 && K >= kBlockK && (K % kBlockK) == 0;
}

size_t pointwise_mma_packed_bytes(int M, int K) {
    if (!pointwise_mma_eligible(M, K)) return 0;
    return (size_t)mma_pad_m(M) * K * 4;          // bf16 hi + bf16 lo per (padded) weight
}

int pack_pointwise_mma(const float* W, int M, int K, void* packed, cudaStream_t st) {
    if (!pointwise_mma_eligible(M, K)) return SDR_ERR_UNSUPPORTED;
    const int Mpad = mma_pad_m(M);
    const long long chunks = (long long)Mpad * K / 8;
    pack_weight_mma_kernel<<<(unsigned)((chunks + 255) / 256), 256, 0, st>>>(
        W, static_cast<uint8_t*>(packed), M, Mpad, K, K);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

constexpr size_t kMmaSmemBytes = 1024 + (size_t)kStages * (kAStageBytes + kBStageBytes) +
                                 (size_t)kRawStages * kRawStageBytes + kProdWarps * 64 * sizeof(float2) +
                                 (2 * kStages + 2 * kRawStages) * sizeof(uint64_t);
static_assert(kMmaSmemBytes <= 232448, "exceeds the 227 KB a CTA may own on sm_90");

// cuTensorMapEncodeTiled is a pure host-side encoder; it is fetched through the runtime so that the library
// carries no link-time dependency on libcuda.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = [] {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            ptr = nullptr;
        return reinterpret_cast<EncodeTiledFn>(ptr);
    }();
    return fn;
}

// Tensor map of a packed weight buffer seen as [rows][128 B]: one box = the 2 x kTileN rows (hi | lo) of one
// (n_tile, k_block) image, already in shared-memory order (no TMA swizzle).
static int make_weight_map(CUtensorMap* tm, const void* wpk, size_t bytes) {
    memset(tm, 0, sizeof(*tm));
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) return SDR_ERR_CUDA;
    const cuuint64_t dims[2] = {32, (cuuint64_t)(bytes / 128)};
    const cuuint64_t strides[1] = {128};
    const cuuint32_t box[2] = {32, (cuuint32_t)(2 * kTileN)};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(wpk), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? SDR_OK : SDR_ERR_UNSUPPORTED;
}

// Tensor map of the activations [samples][K][L] with a [1][64][128] box: one raw k-block tile
// (positions beyond L arrive as zeros: ragged last tiles need no special case).
static int make_act_map(CUtensorMap* tm, const float* x, int samples, int K, int L) {
    memset(tm, 0, sizeof(*tm));
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) return SDR_ERR_CUDA;
    const cuuint64_t dims[3] = {(cuuint64_t)L, (cuuint64_t)K, (cuuint64_t)samples};
    const cuuint64_t strides[2] = {(cuuint64_t)L * 4, (cuuint64_t)L * K * 4};
    const cuuint32_t box[3] = {(cuuint32_t)kTileM, (cuuint32_t)kBlockK, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(x), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? SDR_OK : SDR_ERR_UNSUPPORTED;
}

// Persistent launch: one CTA per SM (the shared-memory footprint allows no second), never more than there are tiles.
// (All instantiations share one function-pointer type, so the per-kernel state is keyed by the pointer, not by Kern.)
struct MmaLaunchInfo { const void* fn; int dev; int sms; };
static std::mutex g_launch_mutex;
static std::vector<MmaLaunchInfo> g_launch_info;

template <typename Kern>
static int launch_persistent(Kern kern, const MmaArgs& a, const CUtensorMap& wmap, const CUtensorMap& xmap,
                             cudaStream_t st) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return SDR_ERR_CUDA;
    int sms = 0;
    {
        std::lock_guard<std::mutex> lock(g_launch_mutex);
        for (const MmaLaunchInfo& e : g_launch_info)
            if (e.fn == reinterpret_cast<const void*>(kern) && e.dev == dev) { sms = e.sms; break; }
        if (sms == 0) {                           // first launch of this kernel on this device
            if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMmaSmemBytes) != cudaSuccess) {
                cudaGetLastError();
                return SDR_ERR_CUDA;
            }
            if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) return SDR_ERR_CUDA;
            g_launch_info.push_back(MmaLaunchInfo{reinterpret_cast<const void*>(kern), dev, sms});
        }
    }
    const int grid = a.num_tiles < sms ? a.num_tiles : sms;
    kern<<<grid, kMmaThreads, kMmaSmemBytes, st>>>(a, wmap, xmap);
    if (cudaGetLastError() != cudaSuccess) return SDR_ERR_CUDA;
    return SDR_OK;
}

int launch_pointwise_mma(const float* x, const NormIn& nin, const void* wpk, const float* bias,
                         const float* residual, const float* gate, int gate_channels,
                         float* y, double* stats_out, int samples, int M, int K, int L,
                         int epilogue, cudaStream_t st) {
    if (!pointwise_mma_eligible(M, K) || (L % 4) != 0 || (reinterpret_cast<uintptr_t>(x) % 16) != 0)
        return SDR_ERR_UNSUPPORTED;                      // TMA rows of the activations: 16 B aligned
    if (samples <= 0 || L <= 0 || !x || !wpk || !y) return SDR_ERR_BAD_ARGUMENT;
    if (epilogue == 1 && (!gate || gate_channels <= 0)) return SDR_ERR_BAD_ARGUMENT;
    if (epilogue == 1 && (gate_channels % kTileN) != 0) return SDR_ERR_UNSUPPORTED;
    if (reinterpret_cast<uintptr_t>(wpk) % 16) return SDR_ERR_BAD_ARGUMENT;
    MmaArgs a;
    a.x = x; a.nin = nin; a.bias = bias; a.residual = residual;
    a.gate = gate; a.gate_channels = gate_channels; a.y = y; a.stats_out = stats_out;
    a.M = M; a.K = K; a.L = L; a.epilogue = epilogue;
    a.win_k = 0; a.win_hop = 0; a.win_pad = 0; a.win_a = 0; a.win_T = 0;
    a.n_tiles = mma_pad_m(M) / kTileN;
    a.l_tiles = (L + kTileM - 1) / kTileM;
    const long long tiles = (long long)samples * a.l_tiles * a.n_tiles;
    if (tiles > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    a.num_tiles = (int)tiles;
    const int act = nin.prelu ? (nin.prelu_pc ? 2 : 1) : 0;
    const int mode = epilogue == 1 ? 2 : (residual ? 1 : 0);
    const bool stats = stats_out != nullptr;
    CUtensorMap wmap, xmap;
    if (int rc = make_weight_map(&wmap, wpk, pointwise_mma_packed_bytes(M, K))) return rc;
    if (int rc = make_act_map(&xmap, x, samples, K, L)) return rc;
#define SDR_MMA_CASE(A, MD, ST)                                                                                   \
    if (act == A && mode == MD && stats == ST) return launch_persistent(pw_mma_kernel<false, A, MD, ST>, a, wmap, xmap, st);
    SDR_MMA_CASE(0, 0, false) SDR_MMA_CASE(0, 0, true)
    SDR_MMA_CASE(1, 0, false) SDR_MMA_CASE(1, 0, true)
    SDR_MMA_CASE(0, 1, false) SDR_MMA_CASE(0, 1, true)
    SDR_MMA_CASE(1, 1, false) SDR_MMA_CASE(1, 1, true)
    SDR_MMA_CASE(0, 2, false) SDR_MMA_CASE(0, 2, true)
    SDR_MMA_CASE(1, 2, false) SDR_MMA_CASE(1, 2, true)
    SDR_MMA_CASE(2, 0, false) SDR_MMA_CASE(2, 0, true)      // the original model: proj_1x1 / conv_1x1_exp / mask front
#undef SDR_MMA_CASE
    return SDR_ERR_UNSUPPORTED;
}

// ---- encoder on the same kernel (window mode) ----
static inline int enc_kpad(int A, int Kk) { return (A * Kk + kBlockK - 1) / kBlockK * kBlockK; }

size_t encoder_mma_packed_bytes(int N, int A, int Kk) {
    if (N < 32 || A < 1 || Kk < 3) return 0;
    return (size_t)mma_pad_m(N) * enc_kpad(A, Kk) * 4;
}

int pack_encoder_mma(const float* W, int N, int A, int Kk, void* packed, cudaStream_t st) {
    if (!encoder_mma_packed_bytes(N, A, Kk)) return SDR_ERR_UNSUPPORTED;
    const int Mpad = mma_pad_m(N), K = enc_kpad(A, Kk);
    const long long chunks = (long long)Mpad * K / 8;
    pack_weight_mma_kernel<<<(unsigned)((chunks + 255) / 256), 256, 0, st>>>(
        W, static_cast<uint8_t*>(packed), N, Mpad, A * Kk, K);
    return cudaGetLastError() == cudaSuccess ? SDR_OK : SDR_ERR_CUDA;
}

int launch_encoder_mma(const float* wav, const void* wpk, const float* bias, int relu, float* enc, double* stats,
                       int B, int A, long long T, int N, int Kk, int L, int pad, cudaStream_t st) {
    if (!encoder_mma_packed_bytes(N, A, Kk)) return SDR_ERR_UNSUPPORTED;
    if (B <= 0 || T <= 0 || L <= 0 || !wav || !wpk || !enc) return SDR_ERR_BAD_ARGUMENT;
    MmaArgs a;
    a.x = wav; a.nin = NormIn{nullptr, nullptr, nullptr, nullptr, 1.0};
    a.bias = bias; a.residual = nullptr; a.gate = nullptr;
    a.gate_channels = 0; a.y = enc; a.stats_out = stats;
    a.M = N; a.K = enc_kpad(A, Kk); a.L = L; a.epilogue = relu ? 2 : 0;      // (window kernels read it as "ReLU on the way out")
    a.win_k = Kk; a.win_hop = Kk / 2; a.win_pad = pad; a.win_a = A; a.win_T = T;   // pad = hop; 2 * hop for the causal model
    a.n_tiles = mma_pad_m(N) / kTileN;
    a.l_tiles = (L + kTileM - 1) / kTileM;
    const long long tiles = (long long)B * a.l_tiles * a.n_tiles;
    if (tiles > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    a.num_tiles = (int)tiles;
    CUtensorMap wmap, xmap;
    if (int rc = make_weight_map(&wmap, wpk, encoder_mma_packed_bytes(N, A, Kk))) return rc;
    memset(&xmap, 0, sizeof(xmap));               // window mode gathers the waveform itself
    if (stats) return launch_persistent(pw_mma_kernel<true, 0, 0, true>, a, wmap, xmap, st);
    return launch_persistent(pw_mma_kernel<true, 0, 0, false>, a, wmap, xmap, st);
}

}  // namespace sdr
