// C-ABI of the H100-native SuDoRM-RF forward (see include/sudormrf_b200.h):
// parameter layout (reference state_dict order), weight packing, workspace
// planning and the forward orchestration that enqueues every kernel on the
// caller's stream.
#include <vector>
#include <cstring>
#include "common.cuh"

#define SDR_TRY(expr) do { int _e = (expr); if (_e != SDR_OK) return _e; } while (0)

namespace sdr {

// kernel launchers (levels.cu, pointwise.cu, frontback.cu, tac.cu)
int launch_depthwise(const float*, const NormIn&, const float*, const float*, float*, double*, int, int, int, int, cudaStream_t);
int launch_merge(const float* const*, const NormIn*, int, float*, double*, int, int, int, cudaStream_t);
// depthwise pyramid in one pass (pyramid.cu)
bool pyramid_eligible(int D, int samples, int C, int L);
size_t pyramid_rowstats_bytes(int samples, int C, int D);
size_t pyramid_table_bytes(int samples, int C, int D);
int launch_pyramid(const float*, const NormIn&, const float* const*, const float* const*, const float* const*,
                   const float* const*, float* const*, double*, double*, float*, int, int, int, int, cudaStream_t);
int launch_merge_pyramid(const float* const*, const float*, int, float*, double*, int, int, int, cudaStream_t);
int launch_pyramid_fused(const float*, const NormIn&, const float* const*, const float* const*, const float* const*,
                         const float* const*, float*, double*, double*, double*, float*, int, int, int, int, cudaStream_t);
int launch_pointwise_ffma(const float*, const NormIn&, const float*, const float*, const float*, const float*, int,
                          float*, double*, int, int, int, int, int, cudaStream_t);
int launch_encoder(const float*, const float*, const float*, int, float*, double*, int, int, long long, int, int, int, int, cudaStream_t);
int launch_overlap_add(const float*, const float*, const float*, const float2*, float*, int, int, int, int, long long, cudaStream_t);
int launch_mixture_consistency(const float*, const float*, float*, int, int, long long, int, void*, cudaStream_t);
int launch_tac(const float*, const float* const*, float*, double*, int, int, int, int, cudaStream_t);
int launch_tac_apply(const float*, const float*, const NormIn&, float*, int, int, int, cudaStream_t);
bool preadd_eligible(int M, int K, int L);
int launch_pointwise_small_preadd(const float*, const float*, const NormIn&, float*, const float*, const float*, float*,
                                  double*, int, int, int, int, cudaStream_t);
// causal model (causal.cu)
bool causal_pyramid_eligible(int D, int L);
int launch_causal_pyramid(const float*, const float*, const float* const*, const float* const*, const float* const*, float*,
                          int, int, int, int, cudaStream_t);
int launch_take_taps(const float*, float*, long long, int, int, cudaStream_t);
int launch_scale_by_scalar(const float*, const float*, float*, long long, cudaStream_t);
// original model (original.cu)
int launch_residual_norm(const float*, const NormIn&, float*, const NormIn&, double*, int, int, int, cudaStream_t);
int launch_softmax_gate(const float*, const float*, float*, int, int, int, int, cudaStream_t);
int launch_toeplitz_mask(const float*, const float*, float*, float*, int, int, cudaStream_t);
int launch_grouped_decoder(const float*, float*, int, int, int, cudaStream_t);
// pre/post steps (prepost.cu)
int launch_utterance_stats(const float*, double*, float2*, int, long long, const long long*, cudaStream_t);
int launch_normalize_rows(const float*, const float2*, float*, int, long long, const long long*, cudaStream_t);
size_t pit_sisdr_scratch_bytes(int B, int S);
size_t stabilized_sisdr_scratch_bytes(int B, int n_est, int n_act);
int launch_stabilized_sisdr(const float*, const float*, float*, int*, int, int, int, int, long long, int, int, double, void*,
                            cudaStream_t);
int launch_pairwise_neg_sdr(const float*, const float*, float*, int, int, long long, int, int, int, void*, cudaStream_t);
int launch_pit_sisdr(const float*, const float*, const float*, float*, int*, int, int, long long, int, int, double,
                     void*, cudaStream_t);
// tensor-core path (pointwise_mma.cu)
bool pointwise_mma_eligible(int M, int K);
size_t pointwise_mma_packed_bytes(int M, int K);
int pack_pointwise_mma(const float* W, int M, int K, void* packed, cudaStream_t);
int launch_pointwise_mma(const float*, const NormIn&, const void*, const float*, const float*, const float*, int,
                         float*, double*, int, int, int, int, int, cudaStream_t);

size_t encoder_mma_packed_bytes(int N, int A, int Kk);
int pack_encoder_mma(const float* W, int N, int A, int Kk, void* packed, cudaStream_t);
int launch_encoder_mma(const float*, const void*, const float*, int, float*, double*, int, int, long long, int, int, int, int, cudaStream_t);

// One 1x1 convolution with the weight at pk + w_off: tensor cores when its image was packed (pk_off != 0, the channel
// counts fill a wgmma tile), FFMA otherwise.
static int pointwise(const float* x, const NormIn& nin, const float* pk, size_t w_off, size_t pk_off, const float* bias,
                     const float* residual, const float* gate, int gate_channels, float* y, double* stats,
                     int samples, int M, int K, int L, int epilogue, cudaStream_t st) {
    if (pk_off && (L % 4) == 0)    // the tensor-core kernel loads activations as float4
        return launch_pointwise_mma(x, nin, pk + pk_off, bias, residual, gate, gate_channels, y, stats,
                                    samples, M, K, L, epilogue, st);
    return launch_pointwise_ffma(x, nin, pk + w_off, bias, residual, gate, gate_channels, y, stats,
                                 samples, M, K, L, epilogue, st);
}

// ---------------------------------------------------------------------------
// parameter layout: offsets (in floats) of every tensor inside the packed buffer
// ---------------------------------------------------------------------------
// What the improved / GroupComm block and the original block share: proj_1x1 (conv, norm, PReLU), spp_dw[d]
// (depthwise conv, norm) and final_norm (norm, PReLU), so one depthwise stage takes either.
struct NormBlockOff {
    size_t proj_w, proj_b, proj_g, proj_be, proj_a;
    size_t dw_w[kMaxDepthApi], dw_b[kMaxDepthApi], dw_g[kMaxDepthApi], dw_be[kMaxDepthApi];
    size_t fn_g, fn_be, fn_a;
    size_t proj_pk;               // tensor-core image (0 = not eligible -> FFMA kernel)
};
struct UBlockOff : NormBlockOff {
    size_t res_w, res_b, res_pk;
};
// sudormrf.py:134-162: proj_1x1 (conv, GroupNorm, PReLU(Ci)), spp_dw[d] (depthwise conv, GroupNorm), conv_1x1_exp (conv,
// GroupNorm), final_norm (GroupNorm, PReLU(Ci)), module_act (GroupNorm, PReLU(Co)), in state_dict order
struct OrigBlockOff : NormBlockOff {
    size_t exp_w, exp_b, exp_g, exp_be;
    size_t ma_g, ma_be, ma_a;
    size_t exp_pk;
};
struct TacOff { size_t p[9]; size_t g, be; };
// causal_improved_sudormrf_v3.py:71-96: one scalar gain, proj (conv + PReLU), D x (21-tap depthwise + PReLU), res_conv
struct CausalBlockOff {
    size_t gain, proj_w, proj_b, proj_a;
    size_t dw_w[kMaxDepthApi], dw_b[kMaxDepthApi], dw_a[kMaxDepthApi];
    size_t res_w, res_b;
    size_t res_wg, res_bg;        // derived: gain * res_conv.{weight,bias}
    size_t proj_pk, res_pk;
};
// the bf16 hi/lo, pre-swizzled tensor-core image at dst of the [M][K] 1x1 weight at src
struct PackedImage { size_t src; int M, K; size_t dst; };

struct Layout {
    bool ok = false;
    int A, N, Co, Ci, U, D, K, S, G, hop;
    int cob, cib;                 // channels seen by one U-ConvBlock (Co/G, Ci/G for groupcomm)
    bool gc;
    bool causal = false;          // variant 2: CausalSuDORMRF
    bool orig = false;            // variant 3: the original SuDORMRF (sudormrf.py)
    std::vector<OrigBlockOff> ob;
    size_t enc_b = 0, rs_w = 0, rs_b = 0, m_w = 0, m_b = 0, dec_b = 0;   // orig: encoder bias, reshape_before_masks, m, decoder bias
    size_t toep_w = 0, toep_b = 0, rs_pk = 0;                            // orig, derived: [S*N][N] mask matrix + its row bias
    std::vector<CausalBlockOff> cb;
    size_t mask_nl = 0;           // causal: mask_nl_class.weight (PReLU on the masks)
    size_t enc_wc = 0;            // causal: derived [N][A][K], the encoder taps the causal mask keeps
    size_t enc_w = 0, ln_g = 0, ln_be = 0, bn_w = 0, bn_b = 0, mask_a = 0, mask_w = 0, mask_b = 0, dec_w = 0;
    size_t dec_wt = 0;            // derived: decoder weight as [S*A*K, S*A*N]
    size_t bn_pk = 0, mask_pk = 0, dec_pk = 0;   // tensor-core images of the 1x1 weights (0 = not eligible)
    size_t enc_pk = 0, enc_src = 0;              // encoder window image (0 = not eligible) and the [N][A][K] weight behind it
    std::vector<UBlockOff> ub;
    std::vector<TacOff> tac;
    std::vector<PackedImage> images;  // every 1x1 image, in reservation order
    std::vector<size_t> off, numel;   // per state_dict entry
    size_t total = 0;             // floats
};

static Layout make_layout(const sdr_config* c) {
    Layout l;
    if (!c) return l;
    l.gc = c->variant == 1;
    l.causal = c->variant == 2;
    l.orig = c->variant == 3;
    if (c->variant < 0 || c->variant > 3) return l;
    l.A = (l.gc || l.causal) ? c->in_audio_channels : 1;
    l.N = c->enc_num_basis; l.Co = c->out_channels; l.Ci = c->in_channels;
    l.U = c->num_blocks; l.D = c->upsampling_depth; l.K = c->enc_kernel_size;
    l.S = c->num_sources; l.G = l.gc ? c->group_size : 1;
    l.hop = l.K / 2;
    if (l.A < 1 || l.N < 1 || l.Co < 1 || l.Ci < 1 || l.U < 0 || l.S < 1 || l.G < 1) return l;
    if (l.D < 1 || l.D > kMaxDepthApi) return l;
    if (l.K < 3 || (l.K % 2) == 0) return l;          // hop-size arithmetic needs an odd filter (groupcomm_sudormrf_v2.py:255-258)
    if (l.S * l.A > 16) return l;
    if (l.gc && (l.Co % l.G || l.Ci % l.G)) return l;
    l.cob = l.Co / l.G; l.cib = l.Ci / l.G;
    if (l.orig && (l.N % 2)) return l;   // (N+1) x 1 mask conv with padding N - N/2 returns N rows only for an even N (sudormrf.py:239-242,289)

    size_t cur = 0;
    auto derived = [&](size_t n) { const size_t o = cur; cur += (n + 3) & ~(size_t)3; return o; };   // made by sdr_pack_weights
    auto add = [&](size_t n) { l.off.push_back(cur); l.numel.push_back(n); return derived(n); };      // state_dict entry
    auto begin_images = [&] { cur = (cur + 63) & ~(size_t)63; };   // 256 B alignment for the bulk-TMA images
    auto image = [&](size_t src, int M, int K) -> size_t {
        const size_t b = pointwise_mma_packed_bytes(M, K);
        if (!b) return 0;
        l.images.push_back(PackedImage{src, M, K, cur});
        cur += b / sizeof(float);
        return l.images.back().dst;
    };
    auto proj_and_levels = [&](NormBlockOff& u, size_t slopes) {   // proj_1x1 and spp_dw: cib channels
        u.proj_w = add((size_t)l.cib * l.cob); u.proj_b = add(l.cib);
        u.proj_g = add(l.cib); u.proj_be = add(l.cib); u.proj_a = add(slopes);
        for (int d = 0; d < l.D; ++d) {
            u.dw_w[d] = add((size_t)l.cib * 5); u.dw_b[d] = add(l.cib);
            u.dw_g[d] = add(l.cib); u.dw_be[d] = add(l.cib);
        }
    };
    if (l.orig) {
        // state_dict order of the original SuDORMRF (sudormrf.py:211-252; block :134-162) without ln_mask_in (:253, unused)
        l.enc_w = add((size_t)l.N * l.K); l.enc_b = add(l.N);
        l.ln_g = add(l.N); l.ln_be = add(l.N);
        l.bn_w = add((size_t)l.Co * l.N); l.bn_b = add(l.Co);                      // l1
        for (int i = 0; i < l.U; ++i) {
            OrigBlockOff u;
            proj_and_levels(u, l.Ci);
            u.exp_w = add((size_t)l.Co * l.Ci); u.exp_b = add(l.Co); u.exp_g = add(l.Co); u.exp_be = add(l.Co);
            u.fn_g = add(l.Ci); u.fn_be = add(l.Ci); u.fn_a = add(l.Ci);
            u.ma_g = add(l.Co); u.ma_be = add(l.Co); u.ma_a = add(l.Co);
            l.ob.push_back(u);
        }
        if (l.Co != l.N) { l.rs_w = add((size_t)l.N * l.Co); l.rs_b = add(l.N); }   // :233-236
        l.m_w = add((size_t)l.S * (l.N + 1)); l.m_b = add(l.S);
        l.dec_w = add((size_t)l.S * l.N * l.K); l.dec_b = add(l.S);
        l.toep_w = derived((size_t)l.S * l.N * l.N);
        l.toep_b = derived((size_t)l.S * l.N);
        l.dec_wt = derived((size_t)l.S * l.K * l.S * l.N);
        begin_images();
        l.bn_pk = image(l.bn_w, l.Co, l.N);
        for (OrigBlockOff& u : l.ob) {
            u.proj_pk = image(u.proj_w, l.Ci, l.Co);
            u.exp_pk = image(u.exp_w, l.Co, l.Ci);
        }
        if (l.rs_w) l.rs_pk = image(l.rs_w, l.N, l.Co);
        l.mask_pk = image(l.toep_w, l.S * l.N, l.N);
    } else if (l.causal) {
        // state_dict order of CausalSuDORMRF (causal_improved_sudormrf_v3.py:146-189; block :71-96)
        l.enc_w = add((size_t)l.N * l.A * (2 * l.K - 1));
        l.bn_w = add((size_t)l.Co * l.N); l.bn_b = add(l.Co);
        for (int i = 0; i < l.U; ++i) {
            CausalBlockOff u;
            u.gain = add(1);
            u.proj_w = add((size_t)l.Ci * l.Co); u.proj_b = add(l.Ci); u.proj_a = add(1);
            for (int d = 0; d < l.D; ++d) { u.dw_w[d] = add((size_t)l.Ci * 21); u.dw_b[d] = add(l.Ci); u.dw_a[d] = add(1); }
            u.res_w = add((size_t)l.Co * l.Ci); u.res_b = add(l.Co);
            l.cb.push_back(u);
        }
        l.mask_a = add(1);
        l.mask_w = add((size_t)l.S * l.N * l.A * l.Co); l.mask_b = add((size_t)l.S * l.N * l.A);
        l.dec_w = add((size_t)l.N * l.S * l.A * l.S * l.A * l.K);
        l.mask_nl = add(1);
        l.dec_wt = derived((size_t)l.S * l.A * l.K * l.S * l.A * l.N);
        l.enc_wc = derived((size_t)l.N * l.A * l.K);
        for (CausalBlockOff& u : l.cb) {
            u.res_wg = derived((size_t)l.Co * l.Ci);
            u.res_bg = derived(l.Co);
        }
        begin_images();
        l.bn_pk = image(l.bn_w, l.Co, l.N);
        for (CausalBlockOff& u : l.cb) {
            u.proj_pk = image(u.proj_w, l.Ci, l.Co);
            u.res_pk = image(u.res_wg, l.Co, l.Ci);
        }
        l.mask_pk = image(l.mask_w, l.S * l.A * l.N, l.Co);
    } else {
        l.enc_w = add((size_t)l.N * l.A * l.K);
        l.ln_g = add(l.N); l.ln_be = add(l.N);
        l.bn_w = add((size_t)l.Co * l.N); l.bn_b = add(l.Co);
        for (int i = 0; i < l.U; ++i) {
            if (l.gc) {
                TacOff t;
                const size_t n = l.cob, H = 3 * (size_t)l.cob;
                t.p[0] = add(H * n); t.p[1] = add(H); t.p[2] = add(1);
                t.p[3] = add(H * H); t.p[4] = add(H); t.p[5] = add(1);
                t.p[6] = add(n * 2 * H); t.p[7] = add(n); t.p[8] = add(1);
                t.g = add(n); t.be = add(n);
                l.tac.push_back(t);
            }
            UBlockOff u;
            proj_and_levels(u, 1);
            u.fn_g = add(l.cib); u.fn_be = add(l.cib); u.fn_a = add(1);
            u.res_w = add((size_t)l.cob * l.cib); u.res_b = add(l.cob);
            l.ub.push_back(u);
        }
        l.mask_a = add(1);
        l.mask_w = add((size_t)l.S * l.N * l.A * l.Co); l.mask_b = add((size_t)l.S * l.N * l.A);
        l.dec_w = add((size_t)l.N * l.S * l.A * l.S * l.A * l.K);
        l.dec_wt = derived((size_t)l.S * l.A * l.K * l.S * l.A * l.N);
        begin_images();
        l.bn_pk = image(l.bn_w, l.Co, l.N);
        for (UBlockOff& u : l.ub) {
            u.proj_pk = image(u.proj_w, l.cib, l.cob);
            u.res_pk = image(u.res_w, l.cob, l.cib);
        }
        // the gated epilogue needs an output tile (128/256 channels) to stay inside one source's N basis rows
        if (l.N % 256 == 0) l.mask_pk = image(l.mask_w, l.S * l.A * l.N, l.Co);
    }
    l.dec_pk = image(l.dec_wt, l.S * l.A * l.K, l.S * l.A * l.N);
    // the original model's biased encoder + ReLU runs the same window kernel with bias / ReLU on the way out
    l.enc_src = l.causal ? l.enc_wc : l.enc_w;
    const size_t enc_bytes = encoder_mma_packed_bytes(l.N, l.A, l.K);
    l.enc_pk = enc_bytes ? cur : 0;
    cur += enc_bytes / sizeof(float);
    l.total = cur;
    l.ok = true;
    return l;
}

static long long gcd_ll(long long a, long long b) { while (b) { const long long t = a % b; a = b; b = t; } return a; }

static long long padded_len(const Layout& l, long long T) {
    if (l.orig) {                                          // sudormrf.py:206-209,283-293: multiples of lcm(hop, 2^D), no minimum
        const long long p2 = 1LL << l.D;
        const long long q = (long long)l.hop * p2 / gcd_ll(l.hop, p2);
        return T % q ? T + q - T % q : T;
    }
    const long long q = (long long)l.hop << l.D;          // improved_sudormrf.py:244
    if (T < q) return q;
    return (T + q - 1) / q * q;
}

// decoder.weight [C=S*A*N][SA][K]  ->  [SA*K][C]
__global__ void transpose_decoder_kernel(const float* __restrict__ w, float* __restrict__ wt,
                                         int C, int SAK) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)C * SAK) return;
    const int c = (int)(i % C), r = (int)(i / C);
    wt[i] = w[(size_t)c * SAK + r];
}

// ---------------------------------------------------------------------------
// workspace plan: every choice that changes which kernels a forward runs is made here, once
// ---------------------------------------------------------------------------
struct Plan {
    long long Tp; int L; int samples;          // samples = B (improved) or B*G
    int block_slots;                           // statistics slots per block; slot 0 holds the encoder output's
    int slots; size_t stats_doubles;
    size_t o_stats, o_e, o_x, o_xt, o_o, o_y, o_z[kMaxDepthApi], o_masked, o_frames, total;  // bytes
    bool pyramid;                              // the depthwise pyramid runs as one pass (pyramid.cu)
    bool tac_folded;                           // GroupComm: tac_apply rides on proj_1x1's operand load (pointwise.cu)
    size_t o_rowstats, o_table;

    double* stats(char* ws) const { return reinterpret_cast<double*>(ws + o_stats); }
    // statistics slot k of block i
    double* slot(char* ws, int i, int k) const { return stats(ws) + (1 + (size_t)i * block_slots + k) * samples * 2; }
    float* buf(char* ws, size_t o) const { return reinterpret_cast<float*>(ws + o); }
};

static Plan make_plan(const Layout& l, int B, long long T) {
    Plan p;
    p.Tp = padded_len(l, T);
    p.L = (int)(p.Tp / l.hop);
    p.samples = B * l.G;
    // improved: proj, D levels, merge; GroupComm: + TAC; original: + conv_1x1_exp, + residual; causal: no statistics
    p.block_slots = l.causal ? 0 : l.D + 2 + (l.gc ? 1 : 0) + (l.orig ? 2 : 0);
    p.slots = 1 + l.U * p.block_slots;
    p.stats_doubles = (size_t)p.slots * p.samples * 2;
    size_t cur = 0;
    auto seg = [&](size_t bytes) { size_t o = cur; cur += (bytes + 255) & ~(size_t)255; return o; };
    const size_t BL = (size_t)B * p.L * sizeof(float);
    p.o_stats = seg(p.stats_doubles * sizeof(double));
    p.o_e = seg(BL * l.N);
    p.o_x = seg(BL * l.Co);
    p.o_xt = (l.gc || l.orig) ? seg(BL * l.Co) : 0;                       // orig: conv_1x1_exp output
    p.o_o = l.gc ? seg(BL * l.Co) : ((l.orig && l.rs_w) ? seg(BL * l.N) : 0);   // orig: reshape_before_masks output
    p.o_y = seg(BL * l.Ci);
    for (int d = 0; d < kMaxDepthApi; ++d) p.o_z[d] = (d < l.D && !(l.causal && d > 0)) ? seg((BL * l.Ci) >> d) : 0;
    p.pyramid = !l.causal && pyramid_eligible(l.D, p.samples, l.cib, p.L);
    // proj_1x1 weights of every block have one shape, so they share one tensor-core eligibility
    p.tac_folded = l.gc && l.U > 0 && !l.ub[0].proj_pk && preadd_eligible(l.cib, l.cob, p.L);
    p.o_rowstats = p.pyramid ? seg(pyramid_rowstats_bytes(p.samples, l.cib, l.D)) : 0;
    p.o_table = p.pyramid ? seg(pyramid_table_bytes(p.samples, l.cib, l.D)) : 0;
    p.o_masked = seg(BL * l.S * l.A * l.N);
    p.o_frames = seg(BL * l.S * l.A * l.K);
    p.total = cur;
    return p;
}

// Kernels one forward enqueues, from the plan's choices.
static int launch_count(const Layout& l, const Plan& p) {
    // encoder + bottleneck + U * (proj + levels + merge + res [+ tac (+ tac_apply unless it is folded into proj)])
    // + mask + decoder GEMM + overlap-add; levels = pyramid + solve when the plan takes the one-pass path, else D launches
    if (l.causal) return 2 + 3 * l.U + 3;      // encoder, bottleneck, U x (proj, depthwise pyramid, res), mask, decoder, overlap-add
    const int levels = p.pyramid ? 2 : l.D;
    if (l.orig)                                // encoder, l1, U x (proj, levels, merge, exp, residual-norm), [reshape], mask GEMM, softmax-gate, decoder, overlap-add
        return 2 + l.U * (levels + 4) + (l.rs_w ? 1 : 0) + 4;
    return 2 + l.U * (levels + 3 + (l.gc ? (p.tac_folded ? 1 : 2) : 0)) + 3;
}

// The encoder window kernel (+ statistics unless `stats` is null): tensor cores when its image was packed, FFMA
// otherwise.  The original model's encoder carries a bias and a ReLU; the causal one reads one hop further into the
// past (left padding 2 * hop: 2k-1 taps of which the causal mask keeps the first k).
static int encoder(const Layout& l, const float* pk, const float* mixture, float* e, double* stats, int B, long long T,
                   int L, cudaStream_t st) {
    const float* bias = l.orig ? pk + l.enc_b : nullptr;
    const int relu = l.orig ? 1 : 0, pad = l.causal ? 2 * l.hop : l.hop;
    if (l.enc_pk)
        return launch_encoder_mma(mixture, pk + l.enc_pk, bias, relu, e, stats, B, l.A, T, l.N, l.K, L, pad, st);
    return launch_encoder(mixture, pk + l.enc_src, bias, relu, e, stats, B, l.A, T, l.N, l.K, L, pad, st);
}

// The decoder GEMM (frames = Wd^T masked, `nin` applied on load) and the overlap-add / crop / per-source bias /
// mixture consistency / rescale into out.
static int decoder_tail(const Layout& l, const Plan& p, const float* pk, const NormIn& nin, const float* bias,
                        const float* mixture, int apply_mc, const float2* rescale, float* out, int B, long long T,
                        char* ws, cudaStream_t st) {
    const int SA = l.S * l.A;
    float* frames = p.buf(ws, p.o_frames);
    SDR_TRY(pointwise(p.buf(ws, p.o_masked), nin, pk, l.dec_wt, l.dec_pk, nullptr, nullptr, nullptr, 0,
                      frames, nullptr, B, SA * l.K, SA * l.N, p.L, 0, st));
    return launch_overlap_add(frames, apply_mc ? mixture : nullptr, bias, rescale, out, B, SA, l.K, p.L, T, st);
}

// spp_dw and the merge of block i (improved_sudormrf.py / sudormrf.py UBlock): y holds the raw proj_1x1 output with its
// statistics in slot 0, read through GlobLN + PReLU (one slope per channel for the original model); the merge m
// replaces it in y with its statistics in slot D + 1.  When the plan takes the pyramid, two passes over y (row
// statistics of the raw convolution chain, every GlobLN solved from them, then the chain rebuilt and merged as an
// affine combination of the raw levels), with no level in HBM; else level by level.
static int depthwise_stage(const Layout& l, const Plan& p, const NormBlockOff& u, int i, int prelu_pc, const float* pk,
                           char* ws, cudaStream_t st) {
    const int L = p.L, D = l.D, ns = p.samples, C = l.cib;
    float* y = p.buf(ws, p.o_y);
    float* z[kMaxDepthApi];
    const float* zc[kMaxDepthApi];
    for (int d = 0; d < D; ++d) zc[d] = z[d] = p.buf(ws, p.o_z[d]);
    const NormIn n0{p.slot(ws, i, 0), pk + u.proj_g, pk + u.proj_be, pk + u.proj_a, (double)C * L, prelu_pc};
    if (p.pyramid) {
        const float *pw[kMaxDepthApi], *pb[kMaxDepthApi], *pg[kMaxDepthApi], *pbe[kMaxDepthApi];
        for (int d = 0; d < D; ++d) { pw[d] = pk + u.dw_w[d]; pb[d] = pk + u.dw_b[d]; pg[d] = pk + u.dw_g[d]; pbe[d] = pk + u.dw_be[d]; }
        return launch_pyramid_fused(y, n0, pw, pb, pg, pbe, y, p.slot(ws, i, 1), p.slot(ws, i, D + 1),
                                    reinterpret_cast<double*>(ws + p.o_rowstats), p.buf(ws, p.o_table), D, ns, C, L, st);
    }
    SDR_TRY(launch_depthwise(y, n0, pk + u.dw_w[0], pk + u.dw_b[0], z[0], p.slot(ws, i, 1), ns, C, L, 1, st));
    for (int d = 1; d < D; ++d) {
        const NormIn nd{p.slot(ws, i, d), pk + u.dw_g[d - 1], pk + u.dw_be[d - 1], nullptr, (double)C * (L >> (d - 1)), 0};
        SDR_TRY(launch_depthwise(z[d - 1], nd, pk + u.dw_w[d], pk + u.dw_b[d], z[d], p.slot(ws, i, 1 + d),
                                 ns, C, L >> (d - 1), 2, st));
    }
    NormIn nm[kMaxDepthApi];
    for (int d = 0; d < D; ++d)
        nm[d] = NormIn{p.slot(ws, i, 1 + d), pk + u.dw_g[d], pk + u.dw_be[d], nullptr, (double)C * (L >> d), 0};
    return launch_merge(zc, nm, D, y, p.slot(ws, i, D + 1), ns, C, L, st);
}

// CausalSuDORMRF.forward (causal_improved_sudormrf_v3.py:191-211): no normalisation anywhere, so nothing is deferred
// except the PReLUs, which ride on the consumers' operand loads.
static int forward_causal(const Layout& l, const Plan& p, const float* pk, const float* mixture, float* out,
                          int B, long long T, int apply_mc, char* ws, cudaStream_t st, const float2* rescale) {
    const int L = p.L, D = l.D;
    float* e = p.buf(ws, p.o_e);
    float* x = p.buf(ws, p.o_x);
    float* y = p.buf(ws, p.o_y);
    float* m = p.buf(ws, p.o_z[0]);
    const NormIn none{nullptr, nullptr, nullptr, nullptr, 1.0, 0};
    SDR_TRY(encoder(l, pk, mixture, e, nullptr, B, T, L, st));                                    // :194
    SDR_TRY(pointwise(e, none, pk, l.bn_w, l.bn_pk, pk + l.bn_b, nullptr, nullptr, 0,
                      x, nullptr, B, l.Co, l.N, L, 0, st));                                       // :199
    for (const CausalBlockOff& u : l.cb) {
        SDR_TRY(pointwise(x, none, pk, u.proj_w, u.proj_pk, pk + u.proj_b, nullptr, nullptr, 0,
                          y, nullptr, B, l.Ci, l.Co, L, 0, st));                                  // :105 (PReLU deferred)
        const float *w[kMaxDepthApi], *b[kMaxDepthApi], *a[kMaxDepthApi];
        for (int d = 0; d < D; ++d) { w[d] = pk + u.dw_w[d]; b[d] = pk + u.dw_b[d]; a[d] = pk + u.dw_a[d]; }
        SDR_TRY(launch_causal_pyramid(y, pk + u.proj_a, w, b, a, m, D, B, l.Ci, L, st));          // :106-116
        SDR_TRY(pointwise(m, none, pk, u.res_wg, u.res_pk, pk + u.res_bg, x, nullptr, 0,
                          x, nullptr, B, l.Co, l.Ci, L, 0, st));                                  // :118
    }
    const NormIn pm{nullptr, nullptr, nullptr, pk + l.mask_a, 1.0, 0};                            // :202 PReLU -> 1x1
    SDR_TRY(pointwise(x, pm, pk, l.mask_w, l.mask_pk, pk + l.mask_b, nullptr, nullptr, 0,
                      p.buf(ws, p.o_masked), nullptr, B, l.S * l.A * l.N, l.Co, L, 0, st));
    const NormIn pn{nullptr, nullptr, nullptr, pk + l.mask_nl, 1.0, 0};                           // :206 PReLU, :209 decoder
    return decoder_tail(l, p, pk, pn, nullptr, mixture, apply_mc, rescale, out, B, T, ws, st);
}

// The original SuDORMRF.forward (sudormrf.py:266-292; UBlock.forward :164-186).
static int forward_original(const Layout& l, const Plan& p, const float* pk, const float* mixture, float* out,
                            int B, long long T, int apply_mc, char* ws, cudaStream_t st, const float2* rescale) {
    const int L = p.L, D = l.D, Co = l.Co, Ci = l.Ci, N = l.N, S = l.S;
    float* e = p.buf(ws, p.o_e);
    float* x = p.buf(ws, p.o_x);
    float* ex = p.buf(ws, p.o_xt);
    float* y = p.buf(ws, p.o_y);
    float* masked = p.buf(ws, p.o_masked);
    const NormIn none{nullptr, nullptr, nullptr, nullptr, 1.0, 0};
    if (cudaMemsetAsync(p.stats(ws), 0, p.stats_doubles * sizeof(double), st) != cudaSuccess) return SDR_ERR_CUDA;

    // front end (:268-276): biased encoder + ReLU (+stats), ln folded into l1's operand load
    SDR_TRY(encoder(l, pk, mixture, e, p.stats(ws), B, T, L, st));
    {
        NormIn ln{p.stats(ws), pk + l.ln_g, pk + l.ln_be, nullptr, (double)N * L, 0};
        SDR_TRY(pointwise(e, ln, pk, l.bn_w, l.bn_pk, pk + l.bn_b, nullptr, nullptr, 0, x, nullptr, B, Co, N, L, 0, st));
    }
    // x holds u_i = GN(conv_1x1_exp(..)) + block input (raw); the block output PReLU_c(GN_ma(u_i)) is applied by its readers
    NormIn xin = none;
    for (int i = 0; i < l.U; ++i) {
        const OrigBlockOff& u = l.ob[i];
        SDR_TRY(pointwise(x, xin, pk, u.proj_w, u.proj_pk, pk + u.proj_b, nullptr, nullptr, 0,
                          y, p.slot(ws, i, 0), B, Ci, Co, L, 0, st));                                // :171
        SDR_TRY(depthwise_stage(l, p, u, i, 1, pk, ws, st));                                         // :172-182, m in y
        {                                                                                            // :184 conv_1x1_exp.conv
            NormIn nf{p.slot(ws, i, D + 1), pk + u.fn_g, pk + u.fn_be, pk + u.fn_a, (double)Ci * L, 1};
            SDR_TRY(pointwise(y, nf, pk, u.exp_w, u.exp_pk, pk + u.exp_b, nullptr, nullptr, 0,
                              ex, p.slot(ws, i, D + 2), B, Co, Ci, L, 0, st));
        }
        {                                                                                            // :184 .norm, :186 + x
            NormIn ne{p.slot(ws, i, D + 2), pk + u.exp_g, pk + u.exp_be, nullptr, (double)Co * L, 0};
            SDR_TRY(launch_residual_norm(ex, ne, x, xin, p.slot(ws, i, D + 3), B, Co, L, st));
        }
        xin = NormIn{p.slot(ws, i, D + 3), pk + u.ma_g, pk + u.ma_be, pk + u.ma_a, (double)Co * L, 1};   // :186 module_act
    }
    const float* mask_in = x;                              // input of the mask convolution and how to read it
    NormIn mnin = xin;
    if (l.rs_w) {                                                                                     // :279-281
        float* r = p.buf(ws, p.o_o);
        SDR_TRY(pointwise(x, xin, pk, l.rs_w, l.rs_pk, pk + l.rs_b, nullptr, nullptr, 0, r, nullptr, B, N, Co, L, 0, st));
        mask_in = r; mnin = none;
    }
    SDR_TRY(pointwise(mask_in, mnin, pk, l.toep_w, l.mask_pk, pk + l.toep_b, nullptr, nullptr, 0,
                      masked, nullptr, B, S * N, N, L, 0, st));                                       // :284
    SDR_TRY(launch_softmax_gate(masked, e, masked, B, S, N, L, st));                                  // :285-289
    return decoder_tail(l, p, pk, none, pk + l.dec_b, mixture, apply_mc, rescale, out, B, T, ws, st);   // :291
}

static int forward_impl(const Layout& l, const Plan& p, const float* pk, const float* mixture, float* out,
                        int B, long long T, int apply_mc, char* ws, cudaStream_t st,
                        const float2* rescale = nullptr) {
    // mixture_consistency.apply (mixture_consistency.py:14-36) sums the estimates over dim 1 and broadcasts against a
    // [B, 1, T] mixture: it is only defined for mono models; refuse instead of silently skipping the projection
    if (apply_mc && l.A != 1) return SDR_ERR_UNSUPPORTED;
    if (l.causal) return forward_causal(l, p, pk, mixture, out, B, T, apply_mc, ws, st, rescale);
    if (l.orig) return forward_original(l, p, pk, mixture, out, B, T, apply_mc, ws, st, rescale);
    const int L = p.L, D = l.D;
    float* e = p.buf(ws, p.o_e);
    float* x = p.buf(ws, p.o_x);
    float* xt = l.gc ? p.buf(ws, p.o_xt) : nullptr;
    float* o = l.gc ? p.buf(ws, p.o_o) : nullptr;
    float* y = p.buf(ws, p.o_y);
    const NormIn none{nullptr, nullptr, nullptr, nullptr, 1.0, 0};

    if (cudaMemsetAsync(p.stats(ws), 0, p.stats_doubles * sizeof(double), st) != cudaSuccess) return SDR_ERR_CUDA;

    // front end: encoder (+stats), ln folded into the bottleneck's operand load
    SDR_TRY(encoder(l, pk, mixture, e, p.stats(ws), B, T, L, st));
    {
        NormIn ln{p.stats(ws), pk + l.ln_g, pk + l.ln_be, nullptr, (double)l.N * L, 0};
        SDR_TRY(pointwise(e, ln, pk, l.bn_w, l.bn_pk, pk + l.bn_b, nullptr, nullptr, 0, x, nullptr, B, l.Co, l.N, L, 0, st));
    }
    // separation module
    const int ns = p.samples, cob = l.cob, cib = l.cib;
    for (int i = 0; i < l.U; ++i) {
        const UBlockOff& u = l.ub[i];
        const float* bin = x;                       // block input == residual
        if (l.gc) {
            const TacOff& tc = l.tac[i];
            const float* tp[9];
            for (int k = 0; k < 9; ++k) tp[k] = pk + tc.p[k];
            double* st_tac = p.slot(ws, i, D + 2);
            SDR_TRY(launch_tac(x, tp, o, st_tac, B, l.G, cob, L, st));
            NormIn tn{st_tac, pk + tc.g, pk + tc.be, nullptr, (double)cob * L, 0};
            bin = xt;
            // xt = x + GlobLN(o) is formed inside proj_1x1's operand load (and written once for the skip connection)
            // when the plan folds it; otherwise it is materialised first
            if (p.tac_folded)
                SDR_TRY(launch_pointwise_small_preadd(x, o, tn, xt, pk + u.proj_w, pk + u.proj_b, y, p.slot(ws, i, 0),
                                                      ns, cib, cob, L, st));
            else
                SDR_TRY(launch_tac_apply(x, o, tn, xt, ns, cob, L, st));
        }
        // proj_1x1: raw + stats
        if (!p.tac_folded)
            SDR_TRY(pointwise(bin, none, pk, u.proj_w, u.proj_pk, pk + u.proj_b, nullptr, nullptr, 0,
                              y, p.slot(ws, i, 0), ns, cib, cob, L, 0, st));
        SDR_TRY(depthwise_stage(l, p, u, i, 0, pk, ws, st));              // m reuses y's storage
        // res_conv + skip
        {
            NormIn nf{p.slot(ws, i, D + 1), pk + u.fn_g, pk + u.fn_be, pk + u.fn_a, (double)cib * L, 0};
            SDR_TRY(pointwise(y, nf, pk, u.res_w, u.res_pk, pk + u.res_b, bin, nullptr, 0, x, nullptr, ns, cob, cib, L, 0, st));
        }
    }
    // mask: PReLU -> 1x1 -> ReLU -> * encoder output
    {
        NormIn pm{nullptr, nullptr, nullptr, pk + l.mask_a, 1.0, 0};
        SDR_TRY(pointwise(x, pm, pk, l.mask_w, l.mask_pk, pk + l.mask_b, nullptr, e, l.N,
                          p.buf(ws, p.o_masked), nullptr, B, l.S * l.A * l.N, l.Co, L, 1, st));
    }
    // decoder: frames = Wd^T masked, then overlap-add / crop / mixture consistency
    return decoder_tail(l, p, pk, none, nullptr, mixture, apply_mc, rescale, out, B, T, ws, st);
}

}  // namespace sdr

// ===========================================================================
// extern "C" surface
// ===========================================================================
using namespace sdr;

#pragma GCC visibility push(default)
extern "C" {

int sdr_abi_version(void) { return SDR_ABI_VERSION; }

const char* sdr_error_string(int code) {
    switch (code) {
        case SDR_OK: return "ok";
        case SDR_ERR_BAD_CONFIG: return "bad model configuration";
        case SDR_ERR_BAD_ARGUMENT: return "bad argument";
        case SDR_ERR_WORKSPACE: return "workspace or packed-weight buffer too small";
        case SDR_ERR_CUDA: return "CUDA call or kernel launch failed";
        case SDR_ERR_UNSUPPORTED: return "configuration not supported by the sm_90a kernels";
        default: return "unknown error";
    }
}

int sdr_num_params(const sdr_config* cfg) {
    const Layout l = make_layout(cfg);
    return l.ok ? (int)l.off.size() : SDR_ERR_BAD_CONFIG;
}

int64_t sdr_param_numel(const sdr_config* cfg, int index) {
    const Layout l = make_layout(cfg);
    if (!l.ok) return SDR_ERR_BAD_CONFIG;
    if (index < 0 || index >= (int)l.numel.size()) return SDR_ERR_BAD_ARGUMENT;
    return (int64_t)l.numel[index];
}

int64_t sdr_padded_length(const sdr_config* cfg, int64_t T) {
    const Layout l = make_layout(cfg);
    if (!l.ok) return SDR_ERR_BAD_CONFIG;
    if (T <= 0) return SDR_ERR_BAD_ARGUMENT;
    return padded_len(l, T);
}

size_t sdr_packed_weight_bytes(const sdr_config* cfg) {
    const Layout l = make_layout(cfg);
    return l.ok ? l.total * sizeof(float) : 0;
}

int sdr_pack_weights(const sdr_config* cfg, const float* const* params, int n_params,
                     void* packed, size_t packed_bytes, sdr_stream stream) {
    const Layout l = make_layout(cfg);
    if (!l.ok) return SDR_ERR_BAD_CONFIG;
    if (!params || !packed || n_params != (int)l.off.size()) return SDR_ERR_BAD_ARGUMENT;
    if (packed_bytes < l.total * sizeof(float)) return SDR_ERR_WORKSPACE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* pk = static_cast<float*>(packed);
    if (cudaMemsetAsync(pk, 0, l.total * sizeof(float), st) != cudaSuccess) return SDR_ERR_CUDA;
    for (size_t i = 0; i < l.off.size(); ++i) {
        if (!params[i]) return SDR_ERR_BAD_ARGUMENT;
        if (cudaMemcpyAsync(pk + l.off[i], params[i], l.numel[i] * sizeof(float),
                            cudaMemcpyDeviceToDevice, st) != cudaSuccess) return SDR_ERR_CUDA;
    }
    // the derived regions, then the images (some are packed from a derived region): all in stream order
    if (l.orig) {
        SDR_TRY(launch_toeplitz_mask(pk + l.m_w, pk + l.m_b, pk + l.toep_w, pk + l.toep_b, l.S, l.N, st));
        SDR_TRY(launch_grouped_decoder(pk + l.dec_w, pk + l.dec_wt, l.S, l.N, l.K, st));
    } else {
        const int C = l.S * l.A * l.N, SAK = l.S * l.A * l.K;
        const long long n = (long long)C * SAK;
        transpose_decoder_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(pk + l.dec_w, pk + l.dec_wt, C, SAK);
        if (cudaGetLastError() != cudaSuccess) return SDR_ERR_CUDA;
    }
    if (l.causal) {
        SDR_TRY(launch_take_taps(pk + l.enc_w, pk + l.enc_wc, (long long)l.N * l.A, 2 * l.K - 1, l.K, st));
        for (const CausalBlockOff& u : l.cb) {
            SDR_TRY(launch_scale_by_scalar(pk + u.res_w, pk + u.gain, pk + u.res_wg, (long long)l.Co * l.Ci, st));
            SDR_TRY(launch_scale_by_scalar(pk + u.res_b, pk + u.gain, pk + u.res_bg, l.Co, st));
        }
    }
    for (const PackedImage& im : l.images) SDR_TRY(pack_pointwise_mma(pk + im.src, im.M, im.K, pk + im.dst, st));
    if (l.enc_pk) SDR_TRY(pack_encoder_mma(pk + l.enc_src, l.N, l.A, l.K, pk + l.enc_pk, st));
    return SDR_OK;
}

size_t sdr_workspace_bytes(const sdr_config* cfg, int B, int64_t T) {
    const Layout l = make_layout(cfg);
    if (!l.ok || B <= 0 || T <= 0) return 0;
    return make_plan(l, B, T).total;
}

static int check_forward_args(const Layout& l, int B, int64_t T) {
    if (!l.ok) return SDR_ERR_BAD_CONFIG;
    if (B <= 0 || T <= 0) return SDR_ERR_BAD_ARGUMENT;
    if (l.gc) {
        const int n = l.cob;
        if (!(n == 4 || n == 8 || n == 16 || n == 32) || l.G > 16) return SDR_ERR_UNSUPPORTED;
    }
    if (padded_len(l, T) / l.hop > 0x3fffffffLL) return SDR_ERR_UNSUPPORTED;
    if (l.causal && !causal_pyramid_eligible(l.D, (int)(padded_len(l, T) / l.hop))) return SDR_ERR_UNSUPPORTED;
    // original model: lcm(hop, 2^D) padding makes L a multiple of 2^D / gcd(hop, 2^D); the D - 1 stride-2 levels need
    // exact halvings (the reference's up-sample + add fails otherwise, sudormrf.py:180-182)
    if (l.orig && ((padded_len(l, T) / l.hop) % (1LL << (l.D - 1))) != 0) return SDR_ERR_UNSUPPORTED;
    return SDR_OK;
}

int sdr_forward(const sdr_config* cfg, const void* packed, const float* mixture, float* out,
                int B, int64_t T, int apply_mixture_consistency,
                void* workspace, size_t workspace_bytes, sdr_stream stream) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_forward_args(l, B, T));
    if (!packed || !mixture || !out || !workspace) return SDR_ERR_BAD_ARGUMENT;
    const Plan p = make_plan(l, B, T);
    if (workspace_bytes < p.total) return SDR_ERR_WORKSPACE;
    if (reinterpret_cast<uintptr_t>(workspace) % 256 || reinterpret_cast<uintptr_t>(packed) % 16)
        return SDR_ERR_BAD_ARGUMENT;
    return forward_impl(l, p, static_cast<const float*>(packed), mixture, out, B, T,
                        apply_mixture_consistency, static_cast<char*>(workspace),
                        static_cast<cudaStream_t>(stream));
}

int sdr_forward_launch_count(const sdr_config* cfg) {          // at the reference's 4 s @ 8 kHz length
    const Layout l = make_layout(cfg);
    if (!l.ok) return SDR_ERR_BAD_CONFIG;
    return launch_count(l, make_plan(l, 1, 32000));
}

int sdr_forward_launch_count_at(const sdr_config* cfg, int64_t T) {
    return sdr_forward_launch_count_for(cfg, 1, T);
}

int sdr_forward_launch_count_for(const sdr_config* cfg, int B, int64_t T) {
    const Layout l = make_layout(cfg);
    if (!l.ok || B <= 0 || T <= 0) return SDR_ERR_BAD_CONFIG;
    return launch_count(l, make_plan(l, B, T));
}

// Byte offsets of the buffers either side of the forward.  sdr_forward_host stages the mixture at 0 and the estimates
// at `est` of its device buffer (`staging` bytes); sdr_separate appends the normalised mixture, the per-row sums (at
// `sums`) and the per-row (mean, std) (at `ms`) to the forward's workspace (`separate` bytes past its end).
struct IoOffsets { size_t est, staging, sums, ms, separate; };
static IoOffsets io_offsets(const Layout& l, int B, long long T) {
    auto seg = [](size_t bytes) { return (bytes + 255) & ~(size_t)255; };
    IoOffsets o;
    o.est = o.sums = seg((size_t)B * l.A * T * sizeof(float));
    o.staging = o.est + seg((size_t)B * l.S * l.A * T * sizeof(float));
    o.ms = o.sums + seg((size_t)B * 2 * sizeof(double));
    o.separate = o.ms + seg((size_t)B * sizeof(float2));
    return o;
}

size_t sdr_host_staging_bytes(const sdr_config* cfg, int B, int64_t T) {
    const Layout l = make_layout(cfg);
    if (!l.ok || B <= 0 || T <= 0) return 0;
    return io_offsets(l, B, T).staging;
}

int sdr_forward_host(const sdr_config* cfg, const void* packed, const float* host_mixture,
                     float* host_out, int B, int64_t T, int apply_mixture_consistency,
                     void* dev_io, size_t dev_io_bytes, void* workspace, size_t workspace_bytes,
                     sdr_stream stream) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_forward_args(l, B, T));
    if (!host_mixture || !host_out || !dev_io) return SDR_ERR_BAD_ARGUMENT;
    const IoOffsets io = io_offsets(l, B, T);
    if (dev_io_bytes < io.staging) return SDR_ERR_WORKSPACE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t in_bytes = (size_t)B * l.A * T * sizeof(float);
    const size_t out_bytes = (size_t)B * l.S * l.A * T * sizeof(float);
    float* d_in = static_cast<float*>(dev_io);
    float* d_out = reinterpret_cast<float*>(static_cast<char*>(dev_io) + io.est);
    if (cudaMemcpyAsync(d_in, host_mixture, in_bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) return SDR_ERR_CUDA;
    SDR_TRY(sdr_forward(cfg, packed, d_in, d_out, B, T, apply_mixture_consistency, workspace, workspace_bytes, stream));
    if (cudaMemcpyAsync(host_out, d_out, out_bytes, cudaMemcpyDeviceToHost, st) != cudaSuccess) return SDR_ERR_CUDA;
    return SDR_OK;
}

int sdr_mixture_consistency(const float* est, const float* mix, float* out, int B, int S, int64_t T,
                            int weights_type, void* scratch, sdr_stream stream) {
    return launch_mixture_consistency(est, mix, out, B, S, T, weights_type, scratch,
                                      static_cast<cudaStream_t>(stream));
}

int sdr_encoder(const float* wav, const float* weight, float* enc, double* stats,
                int B, int A, int64_t T, int N, int K, int L, sdr_stream stream) {
    if (!wav || !weight || !enc || !stats) return SDR_ERR_BAD_ARGUMENT;
    if (K % 2 == 0) return SDR_ERR_BAD_CONFIG;
    return launch_encoder(wav, weight, nullptr, 0, enc, stats, B, A, T, N, K, L, K / 2, static_cast<cudaStream_t>(stream));
}

size_t sdr_encoder_mma_packed_bytes(int N, int A, int K) { return encoder_mma_packed_bytes(N, A, K); }

int sdr_encoder_mma_pack(const float* weight, int N, int A, int K, void* packed, sdr_stream stream) {
    if (!weight || !packed) return SDR_ERR_BAD_ARGUMENT;
    if (K % 2 == 0) return SDR_ERR_BAD_CONFIG;
    return pack_encoder_mma(weight, N, A, K, packed, static_cast<cudaStream_t>(stream));
}

int sdr_encoder_mma(const float* wav, const void* packed_w, float* enc, double* stats,
                    int B, int A, int64_t T, int N, int K, int L, sdr_stream stream) {
    if (K % 2 == 0) return SDR_ERR_BAD_CONFIG;
    return launch_encoder_mma(wav, packed_w, nullptr, 0, enc, stats, B, A, T, N, K, L, K / 2, static_cast<cudaStream_t>(stream));
}

int sdr_encoder_ex(const float* wav, const float* weight, const float* bias_or_null, int relu, int pad, float* enc,
                   double* stats_or_null, int B, int A, int64_t T, int N, int K, int L, sdr_stream stream) {
    if (!wav || !weight || !enc || pad < 0) return SDR_ERR_BAD_ARGUMENT;
    if (K % 2 == 0) return SDR_ERR_BAD_CONFIG;
    return launch_encoder(wav, weight, bias_or_null, relu, enc, stats_or_null, B, A, T, N, K, L, pad,
                          static_cast<cudaStream_t>(stream));
}

int sdr_encoder_mma_ex(const float* wav, const void* packed_w, const float* bias_or_null, int relu, int pad, float* enc,
                       double* stats_or_null, int B, int A, int64_t T, int N, int K, int L, sdr_stream stream) {
    if (pad < 0) return SDR_ERR_BAD_ARGUMENT;
    if (K % 2 == 0) return SDR_ERR_BAD_CONFIG;
    return launch_encoder_mma(wav, packed_w, bias_or_null, relu, enc, stats_or_null, B, A, T, N, K, L, pad,
                              static_cast<cudaStream_t>(stream));
}

int sdr_pointwise(const float* x, const sdr_norm_in* fin, const float* W, const float* bias,
                  const float* residual, const float* gate, int gate_channels, float* y,
                  double* stats_out, int samples, int M, int Kc, int L, int epilogue, sdr_stream stream) {
    if (!x || !W || !y) return SDR_ERR_BAD_ARGUMENT;
    return launch_pointwise_ffma(x, make_norm(fin), W, bias, residual, gate, gate_channels, y, stats_out,
                                 samples, M, Kc, L, epilogue, static_cast<cudaStream_t>(stream));
}

size_t sdr_pointwise_mma_packed_bytes(int M, int Kc) { return pointwise_mma_packed_bytes(M, Kc); }

int sdr_pointwise_mma_pack(const float* W, int M, int Kc, void* packed, sdr_stream stream) {
    if (!W || !packed) return SDR_ERR_BAD_ARGUMENT;
    return pack_pointwise_mma(W, M, Kc, packed, static_cast<cudaStream_t>(stream));
}

int sdr_pointwise_mma(const float* x, const sdr_norm_in* fin, const void* packed_w, const float* bias,
                      const float* residual, const float* gate, int gate_channels, float* y,
                      double* stats_out, int samples, int M, int Kc, int L, int epilogue, sdr_stream stream) {
    return launch_pointwise_mma(x, make_norm(fin), packed_w, bias, residual, gate, gate_channels, y, stats_out,
                                samples, M, Kc, L, epilogue, static_cast<cudaStream_t>(stream));
}

int sdr_depthwise(const float* x, const sdr_norm_in* fin, const float* w5, const float* bias,
                  float* y, double* stats_out, int samples, int C, int Lin, int stride, sdr_stream stream) {
    if (!x || !w5 || !bias || !y || !stats_out) return SDR_ERR_BAD_ARGUMENT;
    if (stride == 2 && (Lin % 2)) return SDR_ERR_BAD_ARGUMENT;
    return launch_depthwise(x, make_norm(fin), w5, bias, y, stats_out, samples, C, Lin, stride,
                            static_cast<cudaStream_t>(stream));
}

static size_t pyr_table_offset(int samples, int C, int D) {
    return (pyramid_rowstats_bytes(samples, C, D) + 255) & ~(size_t)255;
}

size_t sdr_pyramid_scratch_bytes(int samples, int C, int D, int L) {
    if (samples <= 0 || !pyramid_eligible(D, samples, C, L)) return 0;
    return pyr_table_offset(samples, C, D) + pyramid_table_bytes(samples, C, D);
}

int sdr_depthwise_pyramid(const float* y, const sdr_norm_in* fin, const float* const* w5, const float* const* bias,
                          const float* const* gamma, const float* const* beta, float* const* z, double* stats0,
                          void* scratch, int D, int samples, int C, int L, sdr_stream stream) {
    if (!y || !w5 || !bias || !gamma || !beta || !z || !stats0 || !scratch) return SDR_ERR_BAD_ARGUMENT;
    if (!pyramid_eligible(D, samples, C, L)) return SDR_ERR_UNSUPPORTED;
    char* sc = static_cast<char*>(scratch);
    return launch_pyramid(y, make_norm(fin), w5, bias, gamma, beta, z, stats0, reinterpret_cast<double*>(sc),
                          reinterpret_cast<float*>(sc + pyr_table_offset(samples, C, D)), D, samples, C, L,
                          static_cast<cudaStream_t>(stream));
}

int sdr_merge_pyramid(const float* const* z, const void* scratch, int D, float* m, double* stats_out,
                      int samples, int C, int L, sdr_stream stream) {
    if (!z || !scratch || !m || !stats_out) return SDR_ERR_BAD_ARGUMENT;
    if (!pyramid_eligible(D, samples, C, L)) return SDR_ERR_UNSUPPORTED;
    const char* sc = static_cast<const char*>(scratch);
    return launch_merge_pyramid(z, reinterpret_cast<const float*>(sc + pyr_table_offset(samples, C, D)), D, m, stats_out,
                                samples, C, L, static_cast<cudaStream_t>(stream));
}

int sdr_depthwise_pyramid_fused(const float* y, const sdr_norm_in* fin, const float* const* w5, const float* const* bias,
                                const float* const* gamma, const float* const* beta, float* m, double* stats0,
                                double* stats_m, void* scratch, int D, int samples, int C, int L, sdr_stream stream) {
    if (!y || !w5 || !bias || !gamma || !beta || !m || !stats0 || !stats_m || !scratch) return SDR_ERR_BAD_ARGUMENT;
    if (!pyramid_eligible(D, samples, C, L)) return SDR_ERR_UNSUPPORTED;
    char* sc = static_cast<char*>(scratch);
    return launch_pyramid_fused(y, make_norm(fin), w5, bias, gamma, beta, m, stats0, stats_m, reinterpret_cast<double*>(sc),
                                reinterpret_cast<float*>(sc + pyr_table_offset(samples, C, D)), D, samples, C, L,
                                static_cast<cudaStream_t>(stream));
}

int sdr_causal_pyramid(const float* y, const float* slope_in, const float* const* w21, const float* const* bias,
                       const float* const* slope, float* m, int D, int samples, int C, int L, sdr_stream stream) {
    return launch_causal_pyramid(y, slope_in, w21, bias, slope, m, D, samples, C, L, static_cast<cudaStream_t>(stream));
}

int sdr_merge(const float* const* z, const sdr_norm_in* fins, int depth, float* m, double* stats_out,
              int samples, int C, int L, sdr_stream stream) {
    if (!z || !fins || !m || !stats_out || depth < 1 || depth > kMaxDepthApi) return SDR_ERR_BAD_ARGUMENT;
    NormIn n[kMaxDepthApi];
    for (int d = 0; d < depth; ++d) n[d] = make_norm(fins + d);
    return launch_merge(z, n, depth, m, stats_out, samples, C, L, static_cast<cudaStream_t>(stream));
}

int sdr_tac(const float* x, const float* const* params, float* o, double* stats_out,
            int B, int G, int n, int L, sdr_stream stream) {
    if (!x || !params || !o || !stats_out) return SDR_ERR_BAD_ARGUMENT;
    return launch_tac(x, params, o, stats_out, B, G, n, L, static_cast<cudaStream_t>(stream));
}

int sdr_tac_apply(const float* x, const float* o, const sdr_norm_in* norm, float* out, int samples, int n, int L,
                  sdr_stream stream) {
    if (!x || !o || !norm || !norm->stats || !norm->gamma || !norm->beta || !out) return SDR_ERR_BAD_ARGUMENT;
    if (samples <= 0 || n <= 0 || L <= 0) return SDR_ERR_BAD_ARGUMENT;
    return launch_tac_apply(x, o, make_norm(norm), out, samples, n, L, static_cast<cudaStream_t>(stream));
}

int sdr_pointwise_preadd(const float* x, const float* pre_add, const sdr_norm_in* pre_norm, float* xt_out,
                         const float* W, const float* bias, float* y, double* stats_out,
                         int samples, int M, int Kc, int L, sdr_stream stream) {
    if (!pre_norm) return SDR_ERR_BAD_ARGUMENT;
    return launch_pointwise_small_preadd(x, pre_add, make_norm(pre_norm), xt_out, W, bias, y, stats_out,
                                         samples, M, Kc, L, static_cast<cudaStream_t>(stream));
}

int sdr_overlap_add(const float* frames, const float* mix_or_null, float* out, int B, int SA, int K,
                    int L, int64_t T, sdr_stream stream) {
    if (!frames || !out) return SDR_ERR_BAD_ARGUMENT;
    if (K % 2 == 0) return SDR_ERR_BAD_CONFIG;
    return launch_overlap_add(frames, mix_or_null, nullptr, nullptr, out, B, SA, K, L, T, static_cast<cudaStream_t>(stream));
}

int sdr_residual_norm(const float* e, const sdr_norm_in* fe, float* x, const sdr_norm_in* fx, double* stats_out,
                      int samples, int C, int L, sdr_stream stream) {
    return launch_residual_norm(e, make_norm(fe), x, make_norm(fx), stats_out, samples, C, L,
                                static_cast<cudaStream_t>(stream));
}

int sdr_softmax_gate(const float* logits, const float* enc, float* out, int B, int S, int N, int L, sdr_stream stream) {
    return launch_softmax_gate(logits, enc, out, B, S, N, L, static_cast<cudaStream_t>(stream));
}

// ---- steps either side of the forward (SURVEY 8f) ----

int sdr_utterance_stats(const float* wav, float* mean_std, int rows, int64_t T, void* scratch, sdr_stream stream) {
    if (!scratch || reinterpret_cast<uintptr_t>(scratch) % 8 || reinterpret_cast<uintptr_t>(mean_std) % 8)
        return SDR_ERR_BAD_ARGUMENT;
    return launch_utterance_stats(wav, static_cast<double*>(scratch), reinterpret_cast<float2*>(mean_std), rows, T,
                                  nullptr, static_cast<cudaStream_t>(stream));
}

size_t sdr_separate_workspace_bytes(const sdr_config* cfg, int B, int64_t T) {
    const Layout l = make_layout(cfg);
    if (!l.ok || B <= 0 || T <= 0) return 0;
    return make_plan(l, B, T).total + io_offsets(l, B, T).separate;
}

static int separate_impl(const sdr_config* cfg, const void* packed, const float* wav, const int64_t* lengths,
                         float* out, int B, int64_t T, int apply_mixture_consistency, int rescale,
                         void* workspace, size_t workspace_bytes, sdr_stream stream) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_forward_args(l, B, T));
    if (l.A != 1) return SDR_ERR_UNSUPPORTED;            // the README recipe is written for mono mixtures
    if (!packed || !wav || !out || !workspace) return SDR_ERR_BAD_ARGUMENT;
    const Plan p = make_plan(l, B, T);
    const IoOffsets io = io_offsets(l, B, T);
    if (workspace_bytes < p.total + io.separate) return SDR_ERR_WORKSPACE;
    if (reinterpret_cast<uintptr_t>(workspace) % 256 || reinterpret_cast<uintptr_t>(packed) % 16)
        return SDR_ERR_BAD_ARGUMENT;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    char* extra = ws + p.total;
    float* norm = reinterpret_cast<float*>(extra);
    double* sums = reinterpret_cast<double*>(extra + io.sums);
    float2* ms = reinterpret_cast<float2*>(extra + io.ms);
    const long long* len = reinterpret_cast<const long long*>(lengths);
    SDR_TRY(launch_utterance_stats(wav, sums, ms, B, T, len, st));               // README.md:101-102
    SDR_TRY(launch_normalize_rows(wav, ms, norm, B, T, len, st));                // README.md:103
    return forward_impl(l, p, static_cast<const float*>(packed), norm, out, B, T,   // README.md:106,109,113-114
                        apply_mixture_consistency, ws, st, rescale ? ms : nullptr);
}

int sdr_separate(const sdr_config* cfg, const void* packed, const float* wav, float* out,
                 int B, int64_t T, int apply_mixture_consistency,
                 void* workspace, size_t workspace_bytes, sdr_stream stream) {
    return separate_impl(cfg, packed, wav, nullptr, out, B, T, apply_mixture_consistency, 1,
                         workspace, workspace_bytes, stream);
}

int sdr_separate_ragged(const sdr_config* cfg, const void* packed, const float* wav, const int64_t* lengths,
                        float* out, int B, int64_t T, int apply_mixture_consistency, int rescale,
                        void* workspace, size_t workspace_bytes, sdr_stream stream) {
    const Layout l = make_layout(cfg);
    if (!l.ok) return SDR_ERR_BAD_CONFIG;
    if (!lengths) return SDR_ERR_BAD_ARGUMENT;
    if (T <= 0 || padded_len(l, T) != T) return SDR_ERR_BAD_ARGUMENT;   // the bucket width is a padded length
    return separate_impl(cfg, packed, wav, lengths, out, B, T, apply_mixture_consistency, rescale,
                         workspace, workspace_bytes, stream);
}

int sdr_pairwise_neg_sdr(const float* est, const float* target, float* out, int B, int S, int64_t T, int sdr_type,
                         int zero_mean, int take_log, void* scratch, sdr_stream stream) {
    return launch_pairwise_neg_sdr(est, target, out, B, S, T, sdr_type, zero_mean, take_log, scratch,
                                   static_cast<cudaStream_t>(stream));
}

size_t sdr_pit_sisdr_scratch_bytes(int B, int S) { return pit_sisdr_scratch_bytes(B, S); }

int sdr_pit_sisdr(const float* est, const float* target, const float* mixture_or_null, float* best, int32_t* perm_index,
                  int B, int S, int64_t T, int zero_mean, int improvement, double eps,
                  void* scratch, sdr_stream stream) {
    if (scratch && reinterpret_cast<uintptr_t>(scratch) % 8) return SDR_ERR_BAD_ARGUMENT;
    return launch_pit_sisdr(est, target, mixture_or_null, best, perm_index, B, S, T, zero_mean, improvement, eps,
                            scratch, static_cast<cudaStream_t>(stream));
}

size_t sdr_stabilized_sisdr_scratch_bytes(int B, int n_est, int n_act) { return stabilized_sisdr_scratch_bytes(B, n_est, n_act); }

int sdr_stabilized_sisdr(const float* est, const float* target, float* best, int32_t* perm_index, int B, int est_rows,
                         int n_est, int n_act, int64_t T, int zero_mean, int improvement, double eps,
                         void* scratch, sdr_stream stream) {
    if (scratch && reinterpret_cast<uintptr_t>(scratch) % 8) return SDR_ERR_BAD_ARGUMENT;
    return launch_stabilized_sisdr(est, target, best, perm_index, B, est_rows, n_est, n_act, T, zero_mean, improvement, eps,
                                   scratch, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
#pragma GCC visibility pop
