// 1x1 Conv1d on the Hopper tensor cores (wgmma, TMA, mbarrier), sm_90a.
//
//   y[s, m, l] = sum_k W[m, k] * f(x[s, k, l]) + bias[m]   (+ residual | relu()*gate)
//
// GEMM view per tile: D[128 positions, 128 channels] = A[128, K] * B[128, K]^T with
//   A = f(x) tile, produced on the fly: the activation tile cannot be TMA'd
//       straight into the MMA because the producer's deferred GlobLN(+PReLU)
//       has to be applied first.  A TMA warp lands the raw fp32 k-block in shared
//       memory together with a table of its channels' folded (scale, shift); the
//       consumer warpgroups read their A fragments from it, apply the affine
//       (+PReLU), split each fp32 value into bf16 hi + bf16 lo and hand both to the
//       tensor cores from registers.
//   B = weights, pre-split into bf16 hi/lo and pre-swizzled at pack time, so a
//       k-block is ONE TMA box of a contiguous image.
//   D = fp32 accumulator in registers: two consumer warpgroups, each owning 64
//       positions x 128 channels (64 registers per thread), transform their A,
//       issue the wgmmas and run the epilogue.  Persistent CTAs, one per SM; the
//       TMA warps run ahead into the free stages while the consumers drain.
//   Epilogue: through four 16 KB shared-memory slots, one per quarter of the tile
//       (one warpgroup's 64 positions x 64 channels).  The residual / gate quarter
//       arrives there by TMA while the tile's main loop runs, the warpgroup combines
//       it with its accumulators in place and goes straight on; a store warp stores
//       the quarter to y by TMA and refills the slot with the next tile's quarter.
// Precision: x*w ~= xh*wh + xl*wh + xh*wl (3 bf16 MMAs, fp32 accumulate): the
// dropped terms are O(2^-16) relative, i.e. fp32-grade for the 1e-3 parity
// budget, where a single bf16 (5e-3) or tf32 (7e-4) pass is not (SURVEY §7).
//
// Replaces (reference file:line): bottleneck improved_sudormrf.py:256-259,292;
// proj_1x1.conv :174,205; res_conv(+skip) :196,220; mask_net :268-269,295-298.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cuda.h>
#include <cuda_bf16.h>
#include "common.cuh"
#include "sm90.cuh"
#include "launchers.cuh"

namespace sdr {

constexpr int kTileM = 128;            // positions per CTA tile (2 consumer warpgroups x wgmma M = 64)
constexpr int kTileN = 128;            // output channels per tile (wgmma N); 64 fp32 accumulator registers per thread
constexpr int kBlockK = 64;            // channels per k-block = one 128 B swizzle row of bf16
constexpr int kStages = 3;             // weight stages: one is released a k-block after its wgmmas were issued
constexpr int kRawStages = 2;          // fp32 activation k-blocks, released once the consumers hold them in registers
// Raw k-blocks and epilogue slots share one box format: fp32 [64 channels][32 positions], 128 B rows, SWIZZLE_128B
// (16 B chunk index XOR channel % 8), which keeps the A-fragment and accumulator-fragment accesses conflict-free.
constexpr int kBoxL = 32;
constexpr int kBoxBytes = 64 * kBoxL * 4;                    // 8 KB
constexpr int kRawStageBytes = kTileM / kBoxL * kBoxBytes;   // 32 KB: the k-block's 128 positions as 4 boxes
constexpr int kBHalf = kTileN * 128;   // 16 KB: bf16 [128 weight rows][64 k]
constexpr int kBStageBytes = 2 * kBHalf;                     // 32 KB: hi + lo
constexpr int kSlotBytes = 2 * kBoxBytes;                    // 16 KB: a quarter of the tile, 64 channels x 64 positions
constexpr int kSlots = 4;                                    // slot 2 wg + h: warpgroup wg's channel half h
// Warp roles: [0, 8) the two consumer warpgroups (operand transform, wgmma, epilogue), 8 weight TMA, 9 raw activation
// TMA, 10 epilogue stores and residual / gate refills; in window mode warps 9 and 10 instead gather the waveform
// windows into the raw ring (and the consumers copy their output out themselves).
constexpr int kConsWarps = 8, kTmaWarp = 8, kRawWarp = 9, kStoreWarp = 10, kGatherWarps = 2;
constexpr int kMmaThreads = 32 * (kStoreWarp + 1);   // 352: 11 warps, still at most 3 on one SM sub-partition
static_assert(kRawWarp + kGatherWarps == kStoreWarp + 1, "window mode's gather warps take the raw and store warps' places");

struct MmaArgs {
    const float* x;
    NormIn nin;
    const float* bias;    // residual, gate and (outside window mode) y are read and written through tensor maps
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
// PTX wrappers with this file as their only user (the shared ones: sm90.cuh)
// ---------------------------------------------------------------------------
// global -> shared tensor (TMA) loads; out-of-range elements arrive as zeros
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// shared -> global tensor (TMA) store; out-of-range elements are not written
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tm, const void* smem_src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(tm), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the committed stores have finished reading shared memory / have completed
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
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
// B operand, K-major: 128 B per weight row, 8-row groups 1024 B apart (LBO unused for swizzled K-major, canonical 16 B).
constexpr uint32_t kBLbo = 16, kBSbo = 1024;

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T for the executing warpgroup; A from registers, B K-major in shared memory.
// Thread t of the warpgroup holds a[j] (two bf16, the lower k in the low half) at row 16 * (t / 32) + (t % 32) / 4 +
// 8 * (j % 2), k 2 * (t % 4) + 8 * (j / 2) + {0, 1}, and d[i] at row 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2),
// column 8 * (i / 4) + 2 * (t % 4) + i % 2.
__device__ __forceinline__ void wgmma_bf16_m64n128_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc,
                                                      uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
        "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, "
        "%45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
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

// The consumers issue a k-block as kGroups wgmma groups of kGroupSteps k-steps each and double-buffer the A fragments
// per group: 64 accumulators + 2 x 16 fragment registers.  (Whole k-blocks would take 2 x 32 and spill: 11 warps put
// 3 on one SM sub-partition, which caps a thread at 168 registers.)
constexpr int kGroupSteps = 2;
constexpr int kGroups = kBlockK / 16 / kGroupSteps;
static_assert(kGroups == 2, "group g of every k-block uses fragment buffer g");
// A operand of one group for one thread: per k-step the m64k16 register fragments of bf16 hi and bf16 lo.
struct AFrag { uint32_t hi[kGroupSteps][4], lo[kGroupSteps][4]; };

// Compile-time specialisation keeps the hot loops small.
//   WINDOW: encoder mode (strided waveform windows as the A operand)
//   ACT:    PReLU in the operand transform: 0 none, 1 one shared slope (nn.PReLU()), 2 one slope per input
//           channel (nn.PReLU(C) of the original model, sudormrf.py:33,71)
//   MODE:   epilogue 0 = bias only, 1 = + residual (may alias y: a tile's residual is loaded before its output is
//           stored), 2 = ReLU * gate
//   STATS:  accumulate (sum, sumsq) of the output
template <bool WINDOW, int ACT, int MODE, bool STATS>
__global__ void __launch_bounds__(kMmaThreads, 1)
pw_mma_kernel(const MmaArgs a, const __grid_constant__ CUtensorMap wmap,      // wmap: packed weights as [rows][128 B]
              const __grid_constant__ CUtensorMap xmap,                       // xmap: activations [samples][K][L], box [64][32]
              const __grid_constant__ CUtensorMap emap,                       // emap: residual (MODE 1) or gate (MODE 2)
              const __grid_constant__ CUtensorMap ymap) {                     // ymap: output (not in window mode)
    static_assert(!(WINDOW && ACT != 0), "the encoder's window operand has no activation");
    // 2 x 32 KB raw k-blocks + 3 x 32 KB weight stages + 4 x 16 KB epilogue slots + 1.5 KB of tables + barriers (of
    // the 227 KB an sm_90 CTA can own).  SWIZZLE_128B needs the stage and slot bases 1024 B aligned; the launch
    // reserves 1 KB to align by hand.
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* r_base = smem;                                                  // kRawStages x 32 KB
    uint8_t* b_base = r_base + kRawStages * kRawStageBytes;                  // kStages x 32 KB
    uint8_t* slots = b_base + kStages * kBStageBytes;                        // kSlots x 16 KB
    // per raw stage, its 64 channels' folded (scale, shift) and (ACT 2) PReLU slopes, written by the raw TMA warp
    float2* s_ab = reinterpret_cast<float2*>(slots + kSlots * kSlotBytes);   // [kRawStages][64]
    float* s_sl = reinterpret_cast<float*>(s_ab + kRawStages * kBlockK);     // [kRawStages][64]
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_sl + kRawStages * kBlockK);
    //   full_bar:   weight stage landed (TMA tx bytes); empty_bar: the 8 consumer warps' wgmmas reading it have retired
    //   rfull_bar:  raw k-block ready: the TMA thread's arrival with the tx bytes and the raw warp's once the stage's
    //               table is written (window mode: one arrival per gather warp)
    //   rempty_bar: the 8 consumer warps hold the raw k-block's values in registers
    //   slot_bar:   per slot: the previous quarter's store has read it and, in MODE 1 / 2, it holds the quarter's
    //               residual / gate (TMA tx bytes); the store warp's arrival
    //   slot_full:  per slot: the owning warpgroup's 4 warps have written the combined quarter (not in window mode)
    uint64_t* full_bar = bars;                       // [kStages]
    uint64_t* empty_bar = full_bar + kStages;        // [kStages]
    uint64_t* rfull_bar = empty_bar + kStages;       // [kRawStages]
    uint64_t* rempty_bar = rfull_bar + kRawStages;   // [kRawStages]
    uint64_t* slot_bar = rempty_bar + kRawStages;    // [kSlots]
    uint64_t* slot_full = slot_bar + kSlots;         // [kSlots]

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int KB = a.K / kBlockK;
    const int tile0 = (int)blockIdx.x;               // tiles of this CTA: tile0, tile0 + tstep, ...
    const int tstep = (int)gridDim.x;

    if (warp == kTmaWarp && lane == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsWarps); }
        for (int s = 0; s < kRawStages; ++s) {
            mbar_init(&rfull_bar[s], WINDOW ? kGatherWarps : 2);
            mbar_init(&rempty_bar[s], kConsWarps);
        }
        for (int s = 0; s < kSlots; ++s) { mbar_init(&slot_bar[s], 1); mbar_init(&slot_full[s], kConsWarps / 2); }
        fence_barrier_init();
    }
    __syncthreads();

    if (WINDOW ? warp >= kRawWarp : warp == kRawWarp) {
        int rs = 0;
        uint32_t rphase = 0;
        if constexpr (WINDOW) {
            // ===================== window gather: strided waveform windows -> raw ring =====================
            // Warp g writes channels [32 g, 32 g + 32) of every k-block, 16 at a time, in the raw TMA's box layout;
            // lane = position within a box, so each row write is one conflict-free 128 B store.
            constexpr int kGatherCh = kBlockK / kGatherWarps;
            const int c0 = (warp - kRawWarp) * kGatherCh;
#pragma unroll 1
            for (int tile = tile0; tile < a.num_tiles; tile += tstep) {
                const TileCoord tc = decode_tile(a, tile);
#pragma unroll 1
                for (int kb = 0; kb < KB; ++kb) {
                    uint8_t* rp = r_base + (size_t)rs * kRawStageBytes + (lane & 3) * 4;
#pragma unroll
                    for (int i0 = 0; i0 < kGatherCh; i0 += 16) {
                        float v[16][kTileM / kBoxL];
#pragma unroll
                        for (int i = 0; i < 16; ++i) {
                            const int k = kb * kBlockK + c0 + i0 + i;
                            const int ch = k / a.win_k, j = k - ch * a.win_k;
                            const float* src = a.x + ((size_t)tc.sample * a.win_a + ch) * a.win_T;
#pragma unroll
                            for (int b = 0; b < kTileM / kBoxL; ++b) {
                                const int l = tc.l0 + b * kBoxL + lane;
                                const long long t = (long long)a.win_hop * l + j - a.win_pad;
                                v[i][b] = (l < a.L && ch < a.win_a && t >= 0 && t < a.win_T) ? __ldg(src + t) : 0.f;
                            }
                        }
                        if (i0 == 0) mbar_wait(&rempty_bar[rs], rphase ^ 1);
#pragma unroll
                        for (int i = 0; i < 16; ++i) {
                            const int c = c0 + i0 + i;
#pragma unroll
                            for (int b = 0; b < kTileM / kBoxL; ++b)
                                *reinterpret_cast<float*>(rp + b * kBoxBytes + c * 128 + (((lane >> 2) ^ (c & 7)) << 4)) = v[i][b];
                        }
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&rfull_bar[rs]);
                    if (++rs == kRawStages) { rs = 0; rphase ^= 1; }
                }
            }
        } else {
            // ===================== raw activation k-blocks: TMA + the channels' folded affine =====================
            // y = x * aa + bb  ==  gamma * (x - mean) * rstd + beta; lane e computes channels 2 e and 2 e + 1.
            const bool has_norm = a.nin.stats != nullptr;
            const double inv_count = 1.0 / a.nin.count;
#pragma unroll 1
            for (int tile = tile0; tile < a.num_tiles; tile += tstep) {
                const TileCoord tc = decode_tile(a, tile);
                float mean = 0.f, rstd = 1.f;          // of the tile's sample
                if (has_norm) {
                    const double mu = a.nin.stats[2 * (size_t)tc.sample] * inv_count;
                    double var = a.nin.stats[2 * (size_t)tc.sample + 1] * inv_count - mu * mu;
                    var = var < 0.0 ? 0.0 : var;
                    mean = (float)mu;
                    rstd = rsqrtf((float)var + kGlnEps);
                }
#pragma unroll 1
                for (int kb = 0; kb < KB; ++kb) {
                    const int k = kb * kBlockK + 2 * lane;
                    float g[2] = {1.f, 1.f}, be[2] = {0.f, 0.f}, sl[2] = {1.f, 1.f};
                    if (has_norm) {
                        g[0] = __ldg(a.nin.gamma + k); g[1] = __ldg(a.nin.gamma + k + 1);
                        be[0] = __ldg(a.nin.beta + k); be[1] = __ldg(a.nin.beta + k + 1);
                    }
                    if constexpr (ACT == 2) { sl[0] = __ldg(a.nin.prelu + k); sl[1] = __ldg(a.nin.prelu + k + 1); }
                    mbar_wait(&rempty_bar[rs], rphase ^ 1);
                    if (lane == 0) {
                        mbar_arrive_expect_tx(&rfull_bar[rs], kRawStageBytes);
                        for (int b = 0; b < kTileM / kBoxL; ++b)
                            tma_load_3d(r_base + (size_t)rs * kRawStageBytes + b * kBoxBytes, &xmap, &rfull_bar[rs],
                                        tc.l0 + b * kBoxL, kb * kBlockK, tc.sample);
                    }
                    float aa[2] = {1.f, 1.f}, bb[2] = {0.f, 0.f};
                    if (has_norm) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) { aa[e] = g[e] * rstd; bb[e] = be[e] - mean * aa[e]; }
                    }
                    *reinterpret_cast<float4*>(s_ab + rs * kBlockK + 2 * lane) = make_float4(aa[0], bb[0], aa[1], bb[1]);
                    if constexpr (ACT == 2) *reinterpret_cast<float2*>(s_sl + rs * kBlockK + 2 * lane) = make_float2(sl[0], sl[1]);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&rfull_bar[rs]);
                    if (++rs == kRawStages) { rs = 0; rphase ^= 1; }
                }
            }
        }
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
    } else if (warp == kStoreWarp) {
        // ===================== epilogue stores + residual / gate refills (not in window mode) =====================
        // Slot 2 wg + h holds warpgroup wg's channel half h.  The warp walks the consumers' tiles and slots in their
        // order; once a quarter's store has read its slot it loads the same quarter of the CTA's next tile (MODE 1 /
        // 2) or only arrives (MODE 0), so all four residual / gate quarters land while that tile's main loop runs.
        // The in-place skip stays correct: a tile's region is touched by its own CTA only, and this thread refills a
        // slot only after its store has read it.
        if constexpr (!WINDOW) {
            if (lane == 0) {
                auto fill_slot = [&](int tile, int s) {
                    if constexpr (MODE == 0) {
                        mbar_arrive(&slot_bar[s]);
                    } else {
                        const TileCoord t = decode_tile(a, tile);
                        const int c0 = t.l0 + 64 * (s >> 1);
                        const int c1 = (MODE == 1 ? t.n0 : t.n0 % a.gate_channels) + 64 * (s & 1);
                        uint8_t* const dst = slots + (size_t)s * kSlotBytes;
                        mbar_arrive_expect_tx(&slot_bar[s], kSlotBytes);
                        tma_load_3d(dst, &emap, &slot_bar[s], c0, c1, t.sample);
                        tma_load_3d(dst + kBoxBytes, &emap, &slot_bar[s], c0 + kBoxL, c1, t.sample);
                    }
                };
                for (int s = 0; s < kSlots; ++s) fill_slot(tile0, s);
                uint32_t phase = 0;
#pragma unroll 1
                for (int tile = tile0; tile < a.num_tiles; tile += tstep) {
                    const TileCoord tc = decode_tile(a, tile);
#pragma unroll 1
                    for (int i = 0; i < kSlots; ++i) {
                        const int h = i >> 1, wg = i & 1, s = 2 * wg + h;   // both warpgroups' half 0, then half 1
                        uint8_t* const slot = slots + (size_t)s * kSlotBytes;
                        const int c0 = tc.l0 + 64 * wg, c1 = tc.n0 + 64 * h;
                        mbar_wait(&slot_full[s], phase);
                        tma_store_3d(&ymap, slot, c0, c1, tc.sample);
                        tma_store_3d(&ymap, slot + kBoxBytes, c0 + kBoxL, c1, tc.sample);
                        bulk_commit();
                        bulk_wait_read_all();
                        if (tile + tstep < a.num_tiles) fill_slot(tile + tstep, s);
                    }
                    phase ^= 1;
                }
                bulk_wait_all();                   // the last stores have completed
            }
            __syncwarp();
        }
    } else {
        // ===================== consumers: operand transform + wgmma main loop + epilogue =====================
        const int wg = warp >> 2;                  // position block [64 wg, 64 wg + 64) of the tile
        const int wr = warp & 3;                   // 16-row slice of the warpgroup's block
        const int q = lane & 3;
        const bool relu_out = WINDOW && a.epilogue == 2;       // window mode only: ReLU on the way out
        const float slope = ACT == 1 ? __ldg(a.nin.prelu) : 1.f;
        const bool slope_le1 = slope <= 1.f;
        // The lane's A-fragment and accumulator elements sit in box 2 wg + wr / 2 of a raw stage or box wr / 2 of a
        // slot, at channel row c = 2 (lane % 4) + v % 2 (+ 8 j) and position pp = 16 (wr % 2) + lane / 4 + 8 (v / 2);
        // the swizzled byte offset of (c, pp) is 128 c + 16 ((pp / 4) ^ (c % 8)) + 4 (pp % 4) = boff[v] + 1024 j.
        uint32_t boff[4];
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const uint32_t c = 2 * q + (v & 1), pp = 16 * (wr & 1) + (lane >> 2) + 8 * (v >> 1);
            boff[v] = c * 128 + (((pp >> 2) ^ c) << 4) + (pp & 3) * 4;
        }
        const uint32_t raw_box = (uint32_t)(2 * wg + (wr >> 1)) * kBoxBytes;
        // Each warpgroup owns slots 2 wg (channels 0-63 of the tile) and 2 wg + 1 (64-127).
        uint8_t* const my_slots = slots + (size_t)(2 * wg) * kSlotBytes;

        int rs = 0, stage = 0, prev_stage = 0;
        uint32_t rphase = 0, phase = 0, slot_phase = 0;
        // Group g of the current raw k-block -> folded affine (+PReLU) -> A fragments of bf16 hi (truncation) and lo
        // (bf16(y - hi)): y - hi is exact in fp32, so |y - hi - lo| <= 2^-9 |y - hi| <= 2^-16 |y|.  The last group
        // releases the raw stage.
        auto transform = [&](AFrag& f, int g) {
            if (g == 0) mbar_wait(&rfull_bar[rs], rphase);
            const uint8_t* rp = r_base + (size_t)rs * kRawStageBytes + raw_box;
            const float2* tab = s_ab + rs * kBlockK + 2 * q;
            const float* tsl = s_sl + rs * kBlockK + 2 * q;
#pragma unroll
            for (int s = 0; s < kGroupSteps; ++s) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {      // channels 16 ks + 8 h + 2 q + {0, 1}: fragment registers 2 h, 2 h + 1
                    const int c = 16 * (g * kGroupSteps + s) + 8 * h;
                    float4 ab = make_float4(1.f, 0.f, 1.f, 0.f);
                    float2 sl = make_float2(1.f, 1.f);
                    if constexpr (!WINDOW) ab = *reinterpret_cast<const float4*>(tab + c);
                    if constexpr (ACT == 2) sl = *reinterpret_cast<const float2*>(tsl + c);
#pragma unroll
                    for (int ph = 0; ph < 2; ++ph) {   // positions + 8 ph
                        float y[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const float x = *reinterpret_cast<const float*>(rp + boff[e + 2 * ph] + c * 128);
                            y[e] = WINDOW ? x : fmaf(x, e ? ab.z : ab.x, e ? ab.w : ab.y);
                            if constexpr (ACT == 1) {
                                y[e] = prelu2(y[e], slope, slope_le1);
                            } else if constexpr (ACT == 2) {   // this channel's own slope (either side of 1, either sign)
                                y[e] = y[e] >= 0.f ? y[e] : y[e] * (e ? sl.y : sl.x);
                            }
                        }
                        const uint32_t h0 = __float_as_uint(y[0]) & 0xffff0000u, h1 = __float_as_uint(y[1]) & 0xffff0000u;
                        const __nv_bfloat162 lo = __floats2bfloat162_rn(y[0] - __uint_as_float(h0), y[1] - __uint_as_float(h1));
                        f.hi[s][2 * h + ph] = __byte_perm(h0, h1, 0x7632);
                        f.lo[s][2 * h + ph] = *reinterpret_cast<const uint32_t*>(&lo);
                    }
                }
            }
            if (g == kGroups - 1) {
                __syncwarp();                      // every lane holds its values: the raw stage may be refilled
                if (lane == 0) mbar_arrive(&rempty_bar[rs]);
                if (++rs == kRawStages) { rs = 0; rphase ^= 1; }
            }
        };
        float acc[64];
        // Group g of k-block kb: 3 products per k-step (xh*wh, xl*wh, xh*wl) with A from `cur`.  Once the previous
        // group's wgmmas have retired (fragment buffer `nxt` is free, and at g == 0 the previous k-block's weight
        // stage), the next group is transformed into `nxt` while these run.
        auto mma_group = [&](int kb, int g, const AFrag& cur, AFrag& nxt) {
            if (g == 0) mbar_wait(&full_bar[stage], phase);
            const uint32_t sb_hi = smem_u32(b_base + (size_t)stage * kBStageBytes);
            const uint32_t sb_lo = sb_hi + kBHalf;
            wgmma_fence();                         // cur's registers were written by the transform
#pragma unroll
            for (int s = 0; s < kGroupSteps; ++s) {
                const int ks = g * kGroupSteps + s;
                const uint64_t dbh = gmma_desc_sw128(sb_hi + ks * 32, kBLbo, kBSbo);
                const uint64_t dbl = gmma_desc_sw128(sb_lo + ks * 32, kBLbo, kBSbo);
                wgmma_bf16_m64n128_rs(acc, cur.hi[s], dbh, (kb | ks) != 0 ? 1u : 0u);
                wgmma_bf16_m64n128_rs(acc, cur.lo[s], dbh, 1u);
                wgmma_bf16_m64n128_rs(acc, cur.hi[s], dbl, 1u);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (g == 0 && kb > 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
            }
            if (g == kGroups - 1) {
                prev_stage = stage;
                if (++stage == kStages) { stage = 0; phase ^= 1; }
                if (kb + 1 < KB) transform(nxt, 0);
            } else {
                transform(nxt, g + 1);
            }
        };
        AFrag fa, fb;
#pragma unroll 1
        for (int tile = tile0; tile < a.num_tiles; tile += tstep) {
            const TileCoord tc = decode_tile(a, tile);
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = 0.f;
            transform(fa, 0);
#pragma unroll 1
            for (int kb = 0; kb < KB; ++kb) {
                mma_group(kb, 0, fa, fb);
                mma_group(kb, 1, fb, fa);
            }
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);   // the last k-block's wgmmas have retired
            // epilogue, one channel half h (accumulators [32 h, 32 h + 32), slot 2 wg + h) at a time: lane owns
            // positions pp and pp + 8 of its warp's 32-position box, and channel pairs 8 j + 2 (lane % 4) + {0, 1} of
            // the half; accumulator u of the half sits at boff[u % 4] + 1024 (u / 4) of the box.
            const int prem = a.L - (tc.l0 + wg * 64 + 32 * (wr >> 1) + 16 * (wr & 1) + (lane >> 2));   // positions left
            StatAcc st;
            float rs_ = 0.f, rq = 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                uint8_t* const slot = my_slots + (size_t)h * kSlotBytes;
                uint8_t* const box = slot + (wr >> 1) * kBoxBytes;
                const int m0 = tc.n0 + 64 * h + 2 * q;
                const int mrem = a.M - m0;             // channels left from this lane's first one
                if constexpr (!WINDOW) mbar_wait(&slot_bar[2 * wg + h], slot_phase);
#pragma unroll
                for (int j = 0; j < 8; ++j) {          // channels m0 + 8 j + {0, 1}
                    float bv[2];
#pragma unroll
                    for (int b = 0; b < 2; ++b) bv[b] = (a.bias && 8 * j + b < mrem) ? __ldg(a.bias + m0 + 8 * j + b) : 0.f;
#pragma unroll
                    for (int v = 0; v < 4; ++v) {
                        const int u = 4 * j + v, i = 32 * h + u;
                        float* e = reinterpret_cast<float*>(box + boff[v] + 1024 * j);
                        float o = acc[i] + bv[v & 1];
                        if (MODE == 1) o += *e;
                        if (MODE == 2) o = relu(o) * *e;
                        if constexpr (WINDOW) { if (relu_out) o = relu(o); }   // the original model's encoder (sudormrf.py:212-218)
                        *e = o;
                        if (STATS && 8 * j + (v & 1) < mrem && 8 * (v >> 1) < prem) { rs_ += o; rq = fmaf(o, o, rq); }
                        if (STATS && (i & 15) == 15) { st.add_run(rs_, rq); rs_ = rq = 0.f; }   // fp32 runs of 16 (StatAcc)
                    }
                }
                if constexpr (WINDOW) {
                    // the encoder's frame count is arbitrary, so its rows need not be 16 B aligned for TMA: the
                    // warpgroup copies the quarter out, one 128 B row segment per warp instruction; the second
                    // barrier frees the slot for the next tile
                    named_bar_sync(1 + wg, 128);
#pragma unroll 4
                    for (int r = wr; r < 64; r += 4) {
                        const int m = tc.n0 + 64 * h + r;
#pragma unroll
                        for (int half = 0; half < 2; ++half) {
                            const int p = tc.l0 + wg * 64 + half * kBoxL + lane;
                            const float v = *reinterpret_cast<const float*>(
                                slot + half * kBoxBytes + r * 128 + (((lane >> 2) ^ (r & 7)) << 4) + (lane & 3) * 4);
                            if (m < a.M && p < a.L) a.y[((size_t)tc.sample * a.M + m) * a.L + p] = v;
                        }
                    }
                    named_bar_sync(1 + wg, 128);
                } else {
                    fence_proxy_async_smem();          // generic-proxy stores -> visible to the store warp's TMA store
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&slot_full[2 * wg + h]);
                }
            }
            slot_phase ^= 1;
            if (STATS) {
                const double ds = warp_sum_f64(st.s), dq = warp_sum_f64(st.q);
                if (lane == 0) {
                    atomicAdd(a.stats_out + 2 * (size_t)tc.sample, ds);
                    atomicAdd(a.stats_out + 2 * (size_t)tc.sample + 1, dq);
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
static bool pointwise_mma_eligible(int M, int K) {
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
    return launch(pack_weight_mma_kernel, (unsigned)((chunks + 255) / 256), 256, 0, st, W,
                  static_cast<uint8_t*>(packed), M, Mpad, K, K);
}

constexpr size_t kMmaSmemBytes = 1024 + (size_t)kRawStages * kRawStageBytes + (size_t)kStages * kBStageBytes +
                                 (size_t)kSlots * kSlotBytes + kRawStages * kBlockK * (sizeof(float2) + sizeof(float)) +
                                 (2 * kStages + 2 * kRawStages + 2 * kSlots) * sizeof(uint64_t);
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
        if (cuda_status(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres)) ||
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

// Tensor map of an fp32 activation tensor [samples][C][L] with a [1][64][32] box, SWIZZLE_128B: a quarter of a raw
// k-block (activations) or half of an epilogue slot (residual, gate, y).  Loads fill positions beyond L and channels
// beyond C with zeros and stores skip them: ragged last tiles need no special case.
static int make_act_map(CUtensorMap* tm, const float* x, int samples, int C, int L) {
    memset(tm, 0, sizeof(*tm));
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) return SDR_ERR_CUDA;
    const cuuint64_t dims[3] = {(cuuint64_t)L, (cuuint64_t)C, (cuuint64_t)samples};
    const cuuint64_t strides[2] = {(cuuint64_t)L * 4, (cuuint64_t)L * C * 4};
    const cuuint32_t box[3] = {(cuuint32_t)kBoxL, 64, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(x), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? SDR_OK : SDR_ERR_UNSUPPORTED;
}
static_assert(kBlockK == 64 && kTileN == 2 * 64, "activation boxes are 64 channels: one k-block, half a channel tile");

// Persistent launch: one CTA per SM (the shared-memory footprint allows no second), never more than there are tiles.
template <typename Kern>
static int launch_persistent(Kern kern, const MmaArgs& a, const CUtensorMap& wmap, const CUtensorMap& xmap,
                             const CUtensorMap& emap, const CUtensorMap& ymap, cudaStream_t st) {
    const int sms = sm_count();
    if (sms <= 0) return SDR_ERR_CUDA;
    return launch(kern, a.num_tiles < sms ? a.num_tiles : sms, kMmaThreads, kMmaSmemBytes, st, a, wmap, xmap, emap,
                  ymap);
}

int launch_pointwise_mma(const float* x, const NormIn& nin, const void* wpk, const float* bias,
                         const float* residual, const float* gate, int gate_channels,
                         float* y, double* stats_out, int samples, int M, int K, int L,
                         int epilogue, cudaStream_t st) {
    auto misaligned = [](const float* p) { return (reinterpret_cast<uintptr_t>(p) % 16) != 0; };
    if (!pointwise_mma_eligible(M, K) || (L % 4) != 0 || misaligned(x) || misaligned(y) ||
        (epilogue != 1 && misaligned(residual)) || (epilogue == 1 && misaligned(gate)))
        return SDR_ERR_UNSUPPORTED;                      // TMA rows of the activations and outputs: 16 B aligned
    if (samples <= 0 || L <= 0 || !x || !wpk || !y) return SDR_ERR_BAD_ARGUMENT;
    if (epilogue == 1 && (!gate || gate_channels <= 0)) return SDR_ERR_BAD_ARGUMENT;
    if (epilogue == 1 && (gate_channels % kTileN) != 0) return SDR_ERR_UNSUPPORTED;
    if (reinterpret_cast<uintptr_t>(wpk) % 16) return SDR_ERR_BAD_ARGUMENT;
    MmaArgs a;
    a.x = x; a.nin = nin; a.bias = bias;
    a.gate_channels = gate_channels; a.y = y; a.stats_out = stats_out;
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
    CUtensorMap wmap, xmap, emap, ymap;
    if (int rc = make_weight_map(&wmap, wpk, pointwise_mma_packed_bytes(M, K))) return rc;
    if (int rc = make_act_map(&xmap, x, samples, K, L)) return rc;
    if (int rc = make_act_map(&ymap, y, samples, M, L)) return rc;
    memset(&emap, 0, sizeof(emap));
    if (mode == 1)
        if (int rc = make_act_map(&emap, residual, samples, M, L)) return rc;
    if (mode == 2)
        if (int rc = make_act_map(&emap, gate, samples, gate_channels, L)) return rc;
#define SDR_MMA_CASE(A, MD, ST)                                                                                   \
    if (act == A && mode == MD && stats == ST)                                                                    \
        return launch_persistent(pw_mma_kernel<false, A, MD, ST>, a, wmap, xmap, emap, ymap, st);
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
    return launch(pack_weight_mma_kernel, (unsigned)((chunks + 255) / 256), 256, 0, st, W,
                  static_cast<uint8_t*>(packed), N, Mpad, A * Kk, K);
}

int launch_encoder_mma(const float* wav, const void* wpk, const float* bias, int relu, float* enc, double* stats,
                       int B, int A, long long T, int N, int Kk, int L, int pad, cudaStream_t st) {
    if (!encoder_mma_packed_bytes(N, A, Kk)) return SDR_ERR_UNSUPPORTED;
    if (B <= 0 || T <= 0 || L <= 0 || !wav || !wpk || !enc) return SDR_ERR_BAD_ARGUMENT;
    MmaArgs a;
    a.x = wav; a.nin = NormIn{nullptr, nullptr, nullptr, nullptr, 1.0};
    a.bias = bias;
    a.gate_channels = 0; a.y = enc; a.stats_out = stats;
    a.M = N; a.K = enc_kpad(A, Kk); a.L = L; a.epilogue = relu ? 2 : 0;      // (window kernels read it as "ReLU on the way out")
    a.win_k = Kk; a.win_hop = Kk / 2; a.win_pad = pad; a.win_a = A; a.win_T = T;   // pad = hop; 2 * hop for the causal model
    a.n_tiles = mma_pad_m(N) / kTileN;
    a.l_tiles = (L + kTileM - 1) / kTileM;
    const long long tiles = (long long)B * a.l_tiles * a.n_tiles;
    if (tiles > 0x7fffffffLL) return SDR_ERR_UNSUPPORTED;
    a.num_tiles = (int)tiles;
    CUtensorMap wmap, none;
    if (int rc = make_weight_map(&wmap, wpk, encoder_mma_packed_bytes(N, A, Kk))) return rc;
    memset(&none, 0, sizeof(none));               // window mode gathers the waveform and writes enc itself
    if (stats) return launch_persistent(pw_mma_kernel<true, 0, 0, true>, a, wmap, none, none, none, st);
    return launch_persistent(pw_mma_kernel<true, 0, 0, false>, a, wmap, none, none, none, st);
}

}  // namespace sdr
