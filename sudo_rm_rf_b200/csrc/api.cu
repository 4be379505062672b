// C-ABI of the H100-native SuDoRM-RF forward (see include/sudormrf_b200.h):
// parameter layout (reference state_dict order), weight packing, workspace
// planning and the forward orchestration that enqueues every kernel on the
// caller's stream.
#include <algorithm>
#include <vector>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include "common.cuh"
#include "launchers.cuh"

#define SDR_TRY(expr) do { int _e = (expr); if (_e != SDR_OK) return _e; } while (0)

namespace sdr {

static const NormIn kNoNorm{nullptr, nullptr, nullptr, nullptr, 1.0, 0};   // operand read as stored

// ---------------------------------------------------------------------------
// parameter layout: offsets (in floats) of every tensor inside the packed buffer
// ---------------------------------------------------------------------------
// A tensor of the packed buffer: its offset there and, for a state_dict entry, its offset in the flat gradient buffer
// of sdr_backward.  It converts to the packed offset (0 = absent), so `pk + p` addresses the tensor.
struct Param {
    size_t off = 0, grad = 0;
    operator size_t() const { return off; }
};
// One 1x1 convolution: [M][K] weight w, bias b (absent when 0) and the bf16 hi/lo, pre-swizzled tensor-core image of w
// at pk (0 = the channel counts do not fill a wgmma tile -> FFMA kernel).
struct Conv1x1 { Param w, b; size_t pk = 0; int M = 0, K = 0; };

// What the improved / GroupComm block and the original block share: proj_1x1 (conv, norm, PReLU), spp_dw[d]
// (depthwise conv, norm) and final_norm (norm, PReLU), so one depthwise stage takes either.
struct NormBlockOff {
    Conv1x1 proj;
    Param proj_g, proj_be, proj_a;
    Param dw_w[kMaxDepthApi], dw_b[kMaxDepthApi], dw_g[kMaxDepthApi], dw_be[kMaxDepthApi];
    Param fn_g, fn_be, fn_a;
};
struct UBlockOff : NormBlockOff { Conv1x1 res; };
// sudormrf.py:134-162: proj_1x1 (conv, GroupNorm, PReLU(Ci)), spp_dw[d] (depthwise conv, GroupNorm), conv_1x1_exp (conv,
// GroupNorm), final_norm (GroupNorm, PReLU(Ci)), module_act (GroupNorm, PReLU(Co)), in state_dict order
struct OrigBlockOff : NormBlockOff {
    Conv1x1 exp;
    Param exp_g, exp_be;
    Param ma_g, ma_be, ma_a;
};
struct TacOff { Param p[9]; Param g, be; };
// causal_improved_sudormrf_v3.py:71-96: one scalar gain, proj (conv + PReLU), D x (21-tap depthwise + PReLU), res_conv
struct CausalBlockOff {
    Param gain;
    Conv1x1 proj;
    Param proj_a;
    Param dw_w[kMaxDepthApi], dw_b[kMaxDepthApi], dw_a[kMaxDepthApi];
    Conv1x1 res;
    Conv1x1 res_g;                // derived: gain * res_conv.{weight,bias}, the one the forward runs
};

// A state_dict entry: its offset in the packed buffer, its element count and its key, printf(blk, i) + printf(name, d)
// + leaf, from string literals, the block i and the level d: nothing is formatted until sdr_param_name asks.
struct Entry { size_t off, numel; const char *blk, *name, *leaf; int i, d; };

struct Layout {
    bool ok = false;
    int A, N, Co, Ci, U, D, K, S, G, hop;
    int cob, cib;                 // channels seen by one U-ConvBlock (Co/G, Ci/G for groupcomm)
    bool gc;
    bool causal = false;          // variant 2: CausalSuDORMRF
    bool orig = false;            // variant 3: the original SuDORMRF (sudormrf.py)
    std::vector<OrigBlockOff> ob;
    Param enc_b, m_w, m_b, dec_b; // orig: encoder bias, m, decoder bias
    Conv1x1 rs;                   // orig: reshape_before_masks (absent when Co == N)
    std::vector<CausalBlockOff> cb;
    Param mask_nl;                // causal: mask_nl_class.weight (PReLU on the masks)
    size_t enc_wc = 0;            // causal: derived [N][A][K], the encoder taps the causal mask keeps
    Param enc_w, ln_g, ln_be, mask_a, dec_w;
    Conv1x1 bn;                   // bottleneck (orig: l1)
    Conv1x1 mask;                 // mask 1x1 (orig: derived [S*N][N] Toeplitz matrix of the m convolution + row bias)
    Conv1x1 dec;                  // derived: decoder weight as [S*A*K][S*A*N], no bias
    size_t enc_pk = 0, enc_src = 0;              // encoder window image (0 = not eligible) and the [N][A][K] weight behind it
    std::vector<UBlockOff> ub;
    std::vector<TacOff> tac;
    std::vector<Conv1x1> images;  // every 1x1 convolution with a tensor-core image, in reservation order
    std::vector<Entry> entries;   // per state_dict entry, in state_dict order
    size_t total = 0;             // floats
};

// Epilogue of a 1x1 convolution beyond its bias (pointwise.cu): residual add, gate by `gate_channels` rows of `gate`,
// and the epilogue mode.
struct Epi { const float* residual = nullptr; const float* gate = nullptr; int gate_channels = 0, mode = 0; };

// y = conv(x read through nin) (+ statistics unless `stats` is null): tensor cores when its image was packed, FFMA
// otherwise.
static int gemm(const float* pk, const Conv1x1& c, const float* x, const NormIn& nin, float* y, double* stats,
                int samples, int L, cudaStream_t st, const Epi& epi = {}) {
    const float* bias = c.b ? pk + c.b : nullptr;
    if (c.pk && (L % 4) == 0)    // the tensor-core kernel loads activations as float4
        return launch_pointwise_mma(x, nin, pk + c.pk, bias, epi.residual, epi.gate, epi.gate_channels, y, stats,
                                    samples, c.M, c.K, L, epi.mode, st);
    return launch_pointwise_ffma(x, nin, pk + c.w, bias, epi.residual, epi.gate, epi.gate_channels, y, stats,
                                 samples, c.M, c.K, L, epi.mode, st);
}

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

    size_t cur = 0, grad = 0;
    const char* blk = ""; int bi = 0;     // key prefix of the entries being added ("sm.%d." ...) and its block index
    auto derived = [&](size_t n) { const size_t o = cur; cur += (n + 3) & ~(size_t)3; return Param{o}; };   // made by sdr_pack_weights
    auto add = [&](size_t n, const char* name, const char* leaf = "", int d = 0) {                          // state_dict entry
        l.entries.push_back({cur, n, blk, name, leaf, bi, d});
        const Param p{derived(n).off, grad};
        grad += n;
        return p;
    };
    auto conv = [&](int M, int K, const char* name) {
        Conv1x1 c; c.M = M; c.K = K; c.w = add((size_t)M * K, name, "weight"); c.b = add(M, name, "bias"); return c;
    };
    auto begin_images = [&] { cur = (cur + 63) & ~(size_t)63; };   // 256 B alignment for the bulk-TMA images
    auto image = [&](Conv1x1& c) {
        const size_t b = pointwise_mma_packed_bytes(c.M, c.K);
        if (!b) return;
        c.pk = cur;
        cur += b / sizeof(float);
        l.images.push_back(c);
    };
    // proj_1x1 and spp_dw: cib channels; norms' affine parameters `g`, `be` (GlobLN: gamma, beta; GroupNorm: weight, bias)
    auto proj_and_levels = [&](NormBlockOff& u, size_t slopes, const char* g, const char* be) {
        u.proj = conv(l.cib, l.cob, "proj_1x1.conv.");
        u.proj_g = add(l.cib, "proj_1x1.norm.", g); u.proj_be = add(l.cib, "proj_1x1.norm.", be);
        u.proj_a = add(slopes, "proj_1x1.act.weight");
        for (int d = 0; d < l.D; ++d) {
            u.dw_w[d] = add((size_t)l.cib * 5, "spp_dw.%d.conv.", "weight", d); u.dw_b[d] = add(l.cib, "spp_dw.%d.conv.", "bias", d);
            u.dw_g[d] = add(l.cib, "spp_dw.%d.norm.", g, d); u.dw_be[d] = add(l.cib, "spp_dw.%d.norm.", be, d);
        }
    };
    const int SA = l.S * l.A;
    if (l.orig) {
        // state_dict order of the original SuDORMRF (sudormrf.py:211-252; block :134-162) without ln_mask_in (:253, unused)
        l.enc_w = add((size_t)l.N * l.K, "encoder.0.weight"); l.enc_b = add(l.N, "encoder.0.bias");
        l.ln_g = add(l.N, "ln.weight"); l.ln_be = add(l.N, "ln.bias");
        l.bn = conv(l.Co, l.N, "l1.");
        for (int i = 0; i < l.U; ++i) {
            OrigBlockOff u; blk = "sm.%d."; bi = i;
            proj_and_levels(u, l.Ci, "weight", "bias");
            u.exp = conv(l.Co, l.Ci, "conv_1x1_exp.conv.");
            u.exp_g = add(l.Co, "conv_1x1_exp.norm.weight"); u.exp_be = add(l.Co, "conv_1x1_exp.norm.bias");
            u.fn_g = add(l.Ci, "final_norm.norm.weight"); u.fn_be = add(l.Ci, "final_norm.norm.bias"); u.fn_a = add(l.Ci, "final_norm.act.weight");
            u.ma_g = add(l.Co, "module_act.norm.weight"); u.ma_be = add(l.Co, "module_act.norm.bias"); u.ma_a = add(l.Co, "module_act.act.weight");
            l.ob.push_back(u);
        }
        blk = "";
        if (l.Co != l.N) l.rs = conv(l.N, l.Co, "reshape_before_masks.");        // :233-236
        l.m_w = add((size_t)l.S * (l.N + 1), "m.weight"); l.m_b = add(l.S, "m.bias");
        l.dec_w = add((size_t)l.S * l.N * l.K, "decoder.weight"); l.dec_b = add(l.S, "decoder.bias");
        l.mask.M = l.S * l.N; l.mask.K = l.N;
        l.mask.w = derived((size_t)l.mask.M * l.mask.K);
        l.mask.b = derived(l.mask.M);
    } else if (l.causal) {
        // state_dict order of CausalSuDORMRF (causal_improved_sudormrf_v3.py:146-189; block :71-96)
        l.enc_w = add((size_t)l.N * l.A * (2 * l.K - 1), "encoder.weight");
        l.bn = conv(l.Co, l.N, "bottleneck.");
        for (int i = 0; i < l.U; ++i) {
            CausalBlockOff u; blk = "sm.%d."; bi = i;
            u.gain = add(1, "skipinit_gain");
            u.proj = conv(l.Ci, l.Co, "proj_1x1.conv."); u.proj_a = add(1, "proj_1x1.act.weight");
            for (int d = 0; d < l.D; ++d) {
                u.dw_w[d] = add((size_t)l.Ci * 21, "spp_dw.%d.conv.", "weight", d); u.dw_b[d] = add(l.Ci, "spp_dw.%d.conv.", "bias", d);
                u.dw_a[d] = add(1, "spp_dw.%d.act.weight", "", d);
            }
            u.res = conv(l.Co, l.Ci, "res_conv.");
            l.cb.push_back(u);
        }
        blk = "";
        l.mask_a = add(1, "mask_net.0.weight");
        l.mask = conv(SA * l.N, l.Co, "mask_net.1.");
        l.dec_w = add((size_t)l.N * SA * SA * l.K, "decoder.weight");
        l.mask_nl = add(1, "mask_nl_class.weight");
    } else {
        // state_dict order of SuDORMRF (improved_sudormrf.py:247-281,170-196) and GroupCommSudoRmRf (groupcomm_sudormrf_v2.py:347-354,401-403)
        l.enc_w = add((size_t)l.N * l.A * l.K, "encoder.weight");
        l.ln_g = add(l.N, "ln.gamma"); l.ln_be = add(l.N, "ln.beta");
        l.bn = conv(l.Co, l.N, "bottleneck.");
        for (int i = 0; i < l.U; ++i) {
            bi = i;
            if (l.gc) {
                TacOff t; blk = "sm.%d.TAC.";
                const size_t n = l.cob, H = 3 * (size_t)l.cob;
                t.p[0] = add(H * n, "TAC_input.0.weight"); t.p[1] = add(H, "TAC_input.0.bias"); t.p[2] = add(1, "TAC_input.1.weight");
                t.p[3] = add(H * H, "TAC_mean.0.weight"); t.p[4] = add(H, "TAC_mean.0.bias"); t.p[5] = add(1, "TAC_mean.1.weight");
                t.p[6] = add(n * 2 * H, "TAC_output.0.weight"); t.p[7] = add(n, "TAC_output.0.bias"); t.p[8] = add(1, "TAC_output.1.weight");
                t.g = add(n, "TAC_norm.gamma"); t.be = add(n, "TAC_norm.beta");
                l.tac.push_back(t);
            }
            UBlockOff u; blk = l.gc ? "sm.%d.UBlock." : "sm.%d.";
            proj_and_levels(u, 1, "gamma", "beta");
            u.fn_g = add(l.cib, "final_norm.norm.gamma"); u.fn_be = add(l.cib, "final_norm.norm.beta"); u.fn_a = add(1, "final_norm.act.weight");
            u.res = conv(l.cob, l.cib, "res_conv.");
            l.ub.push_back(u);
        }
        blk = "";
        l.mask_a = add(1, "mask_net.0.weight");
        l.mask = conv(SA * l.N, l.Co, "mask_net.1.");
        l.dec_w = add((size_t)l.N * SA * SA * l.K, "decoder.weight");
    }
    l.dec.M = SA * l.K; l.dec.K = SA * l.N;
    l.dec.w = derived((size_t)l.dec.M * l.dec.K);
    if (l.causal) {
        l.enc_wc = derived((size_t)l.N * l.A * l.K);
        for (CausalBlockOff& u : l.cb) {
            u.res_g.M = l.Co; u.res_g.K = l.Ci;
            u.res_g.w = derived((size_t)l.Co * l.Ci);
            u.res_g.b = derived(l.Co);
        }
    }
    begin_images();
    image(l.bn);
    for (OrigBlockOff& u : l.ob) { image(u.proj); image(u.exp); }
    for (CausalBlockOff& u : l.cb) { image(u.proj); image(u.res_g); }
    for (UBlockOff& u : l.ub) { image(u.proj); image(u.res); }
    if (l.rs.w) image(l.rs);
    // improved / GroupComm: the gated epilogue needs an output tile (128/256 channels) to stay inside one source's N
    // basis rows
    if (l.orig || l.causal || l.N % 256 == 0) image(l.mask);
    image(l.dec);
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

// Byte offsets of 256-byte aligned segments, handed out in order; `total` bytes hold them all.
struct Segments {
    size_t total = 0;
    size_t take(size_t bytes) { const size_t o = total; total += (bytes + 255) & ~(size_t)255; return o; }
    float* buf(char* ws, size_t o) const { return reinterpret_cast<float*>(ws + o); }
};

// ---------------------------------------------------------------------------
// workspace plan: every choice that changes which kernels a forward runs is made here, once
// ---------------------------------------------------------------------------
struct Plan : Segments {
    long long Tp; int L; int samples;          // samples = B (improved) or B*G
    int block_slots;                           // statistics slots per block; slot 0 holds the encoder output's
    int slots; size_t stats_doubles;
    size_t o_stats, o_e, o_x, o_xt, o_o, o_y, o_z[kMaxDepthApi], o_masked, o_frames;  // bytes
    bool pyramid;                              // the depthwise pyramid runs as one pass (pyramid.cu)
    bool tac_folded;                           // GroupComm: tac_apply rides on proj_1x1's operand load (pointwise.cu)
    size_t o_rowstats, o_table;

    double* stats(char* ws) const { return reinterpret_cast<double*>(ws + o_stats); }
    // statistics slot k of block i
    double* slot(char* ws, int i, int k) const { return stats(ws) + (1 + (size_t)i * block_slots + k) * samples * 2; }
};

// Counts the kernels hold in int: samples = B * G in the plan and every launcher, and the items of one sample (channels
// x frames) in the depthwise, merge, TAC-apply and residual-norm kernels.  A forward past either is refused.
static bool counts_fit(const Layout& l, int B, long long T) {
    const long long C = std::max(std::max(l.cib, l.cob), l.N);
    return (long long)B * l.G <= 0x7fffffffLL && C * (padded_len(l, T) / l.hop) <= 0x7fffffffLL;
}

static Plan make_plan(const Layout& l, int B, long long T) {
    Plan p;
    p.Tp = padded_len(l, T);
    p.L = (int)(p.Tp / l.hop);
    p.samples = B * l.G;
    // improved: proj, D levels, merge; GroupComm: + TAC; original: + conv_1x1_exp, + residual; causal: no statistics
    p.block_slots = l.causal ? 0 : l.D + 2 + (l.gc ? 1 : 0) + (l.orig ? 2 : 0);
    p.slots = 1 + l.U * p.block_slots;
    p.stats_doubles = (size_t)p.slots * p.samples * 2;
    const size_t BL = (size_t)B * p.L * sizeof(float);
    p.o_stats = p.take(p.stats_doubles * sizeof(double));
    p.o_e = p.take(BL * l.N);
    p.o_x = p.take(BL * l.Co);
    p.o_xt = (l.gc || l.orig) ? p.take(BL * l.Co) : 0;                       // orig: conv_1x1_exp output
    p.o_o = l.gc ? p.take(BL * l.Co) : ((l.orig && l.rs.w) ? p.take(BL * l.N) : 0);   // orig: reshape_before_masks output
    p.o_y = p.take(BL * l.Ci);
    for (int d = 0; d < kMaxDepthApi; ++d) p.o_z[d] = (d < l.D && !(l.causal && d > 0)) ? p.take((BL * l.Ci) >> d) : 0;
    p.pyramid = !l.causal && pyramid_eligible(l.D, p.samples, l.cib, p.L);
    // proj_1x1 weights of every block have one shape, so they share one tensor-core eligibility
    p.tac_folded = l.gc && l.U > 0 && !l.ub[0].proj.pk && preadd_eligible(l.cib, l.cob, p.L);
    p.o_rowstats = p.pyramid ? p.take(pyramid_rowstats_bytes(p.samples, l.cib, l.D)) : 0;
    p.o_table = p.pyramid ? p.take(pyramid_table_bytes(p.samples, l.cib, l.D)) : 0;
    p.o_masked = p.take(BL * l.S * l.A * l.N);
    p.o_frames = p.take(BL * l.S * l.A * l.K);
    return p;
}

// Kernels one forward enqueues, from the plan's choices.
static int launch_count(const Layout& l, const Plan& p) {
    // encoder + bottleneck + U * (proj + levels + merge + res [+ tac (+ tac_apply unless it is folded into proj)])
    // + mask + decoder GEMM + overlap-add; levels = pyramid + solve when the plan takes the one-pass path, else D launches
    if (l.causal) return 2 + 3 * l.U + 3;      // encoder, bottleneck, U x (proj, depthwise pyramid, res), mask, decoder, overlap-add
    const int levels = p.pyramid ? 2 : l.D;
    if (l.orig)                                // encoder, l1, U x (proj, levels, merge, exp, residual-norm), [reshape], mask GEMM, softmax-gate, decoder, overlap-add
        return 2 + l.U * (levels + 4) + (l.rs.w ? 1 : 0) + 4;
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
    float* frames = p.buf(ws, p.o_frames);
    SDR_TRY(gemm(pk, l.dec, p.buf(ws, p.o_masked), nin, frames, nullptr, B, p.L, st));
    return launch_overlap_add(frames, apply_mc ? mixture : nullptr, bias, rescale, out, B, l.S * l.A, l.K, p.L, T, st);
}

// The front end of the models with statistics: the statistics cleared, the encoder into e (+ its statistics in slot 0)
// and the bottleneck (original model: l1) into x with ln folded into its operand load.
static int front_end(const Layout& l, const Plan& p, const float* pk, const float* mixture, int B, long long T,
                     char* ws, cudaStream_t st) {
    SDR_TRY(cuda_status(cudaMemsetAsync(p.stats(ws), 0, p.stats_doubles * sizeof(double), st)));
    float* e = p.buf(ws, p.o_e);
    SDR_TRY(encoder(l, pk, mixture, e, p.stats(ws), B, T, p.L, st));
    const NormIn ln{p.stats(ws), pk + l.ln_g, pk + l.ln_be, nullptr, (double)l.N * p.L, 0};
    return gemm(pk, l.bn, e, ln, p.buf(ws, p.o_x), nullptr, B, p.L, st);
}

// spp_dw level by level and the merge (levels.cu): y, read through n0, into the levels z[0..D-1], merged into m.
// Statistics slot k is s0 + k * samples * 2: level d's in slot 1 + d, the merge's in slot D + 1.  nl receives how each
// level is read (its GlobLN).
static int depthwise_levels(const NormBlockOff& u, const float* pk, int D, const float* y, const NormIn& n0,
                            float* const* z, float* m, double* s0, NormIn* nl, int samples, int C, int L,
                            cudaStream_t st) {
    auto slot = [&](int k) { return s0 + (size_t)k * samples * 2; };
    for (int d = 0; d < D; ++d)
        nl[d] = NormIn{slot(1 + d), pk + u.dw_g[d], pk + u.dw_be[d], nullptr, (double)C * (L >> d), 0};
    SDR_TRY(launch_depthwise(y, n0, pk + u.dw_w[0], pk + u.dw_b[0], z[0], slot(1), samples, C, L, 1, st));
    for (int d = 1; d < D; ++d)
        SDR_TRY(launch_depthwise(z[d - 1], nl[d - 1], pk + u.dw_w[d], pk + u.dw_b[d], z[d], slot(1 + d),
                                 samples, C, L >> (d - 1), 2, st));
    return launch_merge(z, nl, D, m, slot(D + 1), samples, C, L, st);
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
    const NormIn n0{p.slot(ws, i, 0), pk + u.proj_g, pk + u.proj_be, pk + u.proj_a, (double)C * L, prelu_pc};
    if (p.pyramid) {
        const float *pw[kMaxDepthApi], *pb[kMaxDepthApi], *pg[kMaxDepthApi], *pbe[kMaxDepthApi];
        for (int d = 0; d < D; ++d) { pw[d] = pk + u.dw_w[d]; pb[d] = pk + u.dw_b[d]; pg[d] = pk + u.dw_g[d]; pbe[d] = pk + u.dw_be[d]; }
        return launch_pyramid_fused(y, n0, pw, pb, pg, pbe, y, p.slot(ws, i, 1), p.slot(ws, i, D + 1),
                                    reinterpret_cast<double*>(ws + p.o_rowstats), p.buf(ws, p.o_table), D, ns, C, L, st);
    }
    float* z[kMaxDepthApi];
    for (int d = 0; d < D; ++d) z[d] = p.buf(ws, p.o_z[d]);
    NormIn nl[kMaxDepthApi];
    return depthwise_levels(u, pk, D, y, n0, z, y, p.slot(ws, i, 0), nl, ns, C, L, st);
}

// What CausalSuDORMRF.forward (causal_improved_sudormrf_v3.py:191-211) and a stream step share, from the encoder output
// e to the decoder's frames: the bottleneck, U x (proj, the depthwise stage into m, res_conv with the gain folded in and
// the skip in place), the mask 1x1 and the decoder GEMM.  No normalisation anywhere, so nothing is deferred except the
// PReLUs, which ride on the consumers' operand loads.  The GEMMs see [samples][channels][L]; the depthwise stage sees B
// rows of Lb frames, and continues each row from its level histories in the stream state `hist` (rows `row` floats
// apart) when that is given.
static int causal_body(const Layout& l, const float* pk, const float* e, float* x, float* y, float* m, float* masked,
                       float* frames, int samples, int L, int B, int Lb, float* hist, long long row, cudaStream_t st) {
    const int D = l.D;
    SDR_TRY(gemm(pk, l.bn, e, kNoNorm, x, nullptr, samples, L, st));                              // :199
    for (int i = 0; i < l.U; ++i) {
        const CausalBlockOff& u = l.cb[i];
        SDR_TRY(gemm(pk, u.proj, x, kNoNorm, y, nullptr, samples, L, st));                        // :105 (PReLU deferred)
        const float *w[kMaxDepthApi], *b[kMaxDepthApi], *a[kMaxDepthApi];
        for (int d = 0; d < D; ++d) { w[d] = pk + u.dw_w[d]; b[d] = pk + u.dw_b[d]; a[d] = pk + u.dw_a[d]; }
        if (hist)                                                                                 // :106-116
            SDR_TRY(launch_causal_stream(y, pk + u.proj_a, w, b, a, hist + (size_t)i * D * 10 * l.Ci, row, m,
                                         D, B, l.Ci, Lb, st));
        else
            SDR_TRY(launch_causal_pyramid(y, pk + u.proj_a, w, b, a, m, D, B, l.Ci, Lb, st));
        SDR_TRY(gemm(pk, u.res_g, m, kNoNorm, x, nullptr, samples, L, st, {x}));                  // :118
    }
    const NormIn pm{nullptr, nullptr, nullptr, pk + l.mask_a, 1.0, 0};                            // :202 PReLU -> 1x1
    SDR_TRY(gemm(pk, l.mask, x, pm, masked, nullptr, samples, L, st));
    const NormIn pn{nullptr, nullptr, nullptr, pk + l.mask_nl, 1.0, 0};                           // :206 PReLU, :209 decoder
    return gemm(pk, l.dec, masked, pn, frames, nullptr, samples, L, st);
}

static int forward_causal(const Layout& l, const Plan& p, const float* pk, const float* mixture, float* out,
                          int B, long long T, int apply_mc, char* ws, cudaStream_t st, const float2* rescale) {
    float* e = p.buf(ws, p.o_e);
    float* frames = p.buf(ws, p.o_frames);
    SDR_TRY(encoder(l, pk, mixture, e, nullptr, B, T, p.L, st));                                  // :194
    SDR_TRY(causal_body(l, pk, e, p.buf(ws, p.o_x), p.buf(ws, p.o_y), p.buf(ws, p.o_z[0]), p.buf(ws, p.o_masked),
                        frames, B, p.L, B, p.L, nullptr, 0, st));
    return launch_overlap_add(frames, apply_mc ? mixture : nullptr, nullptr, rescale, out, B, l.S * l.A, l.K, p.L, T, st);
}

// ---------------------------------------------------------------------------
// streaming of the causal model (stream.cu): state layout, step plan and orchestration
// ---------------------------------------------------------------------------
// Chunk granule: a multiple of 4 frames (float4 rows) that starts every level's chunk on an integer position.
static long long stream_granule(const Layout& l) {
    return (long long)l.hop * (1 << (l.D - 1) > 4 ? 1 << (l.D - 1) : 4);
}

// Per-slot state, in floats: waveform context [A][2 hop], decoder carry [S*A][hop + 1], a flag set by the slot's
// first step, level histories [U][D][10][Ci]; slots are 256 B apart so that a slot's state is one contiguous range.
struct StreamState { size_t ctx, carry, hist, slot; };
static StreamState stream_state(const Layout& l) {
    StreamState s;
    s.ctx = 0;
    s.carry = (size_t)l.A * 2 * l.hop;
    s.hist = (s.carry + (size_t)l.S * l.A * (l.hop + 1) + 1 + 3) & ~(size_t)3;
    s.slot = (s.hist + (size_t)l.U * l.D * 10 * l.Ci + 63) & ~(size_t)63;
    return s;
}

// Workspace of one step: every activation is [channels][B*F] with columns (slot, frame).
struct StreamPlan : Segments {
    int F, BF, Kr;                             // Kr: rows of the encoder operand (taps padded to a k-block for the image)
    size_t o_framed, o_e, o_x, o_y, o_m, o_masked, o_frames;   // bytes
};
static StreamPlan make_stream_plan(const Layout& l, int B, long long C) {
    StreamPlan p;
    p.F = (int)(C / l.hop);
    p.BF = B * p.F;
    p.Kr = l.enc_pk ? (l.A * l.K + 63) / 64 * 64 : l.A * l.K;
    auto rows = [&](size_t n) { return p.take(n * p.BF * sizeof(float)); };
    p.o_framed = rows(p.Kr);
    p.o_e = rows(l.N);
    p.o_x = rows(l.Co);
    p.o_y = rows(l.Ci);
    p.o_m = rows(l.Ci);
    p.o_masked = rows((size_t)l.S * l.A * l.N);
    p.o_frames = rows((size_t)l.S * l.A * l.K);
    return p;
}

static int check_stream_config(const Layout& l) {
    if (!l.ok) return SDR_ERR_BAD_CONFIG;
    if (!l.causal) return SDR_ERR_UNSUPPORTED;         // GlobLN / GroupNorm statistics span the whole clip
    if (2 * l.hop + 2 > 256) return SDR_ERR_UNSUPPORTED;
    return SDR_OK;
}

static int check_stream_args(const Layout& l, int B, long long C) {
    SDR_TRY(check_stream_config(l));
    if (B <= 0 || B > 65535 || C <= 0) return SDR_ERR_BAD_ARGUMENT;
    if (C % stream_granule(l)) return SDR_ERR_UNSUPPORTED;
    const long long F = C / l.hop;
    if (!causal_stream_eligible(l.D, (int)(F < 0x7fffffffLL ? F : 0)) || (long long)B * F > 0x7fffffffLL)
        return SDR_ERR_UNSUPPORTED;
    return SDR_OK;
}

// One step: framing, encoder, bottleneck, U x (proj, stream stage, res_conv), mask, decoder, overlap-add.
static int stream_step(const Layout& l, const StreamPlan& p, const float* pk, float* state, const float* chunk,
                       float* out, int B, long long C, int apply_mc, char* ws, cudaStream_t st) {
    const StreamState ss = stream_state(l);
    float* framed = p.buf(ws, p.o_framed);
    float* e = p.buf(ws, p.o_e);
    float* frames = p.buf(ws, p.o_frames);
    SDR_TRY(launch_stream_frame(chunk, state, (long long)ss.slot, framed, B, l.A, l.K, p.Kr, p.F, C, st));
    if (l.enc_pk)                                      // the window encoder's image is a plain [N][Kr] GEMM image
        SDR_TRY(launch_pointwise_mma(framed, kNoNorm, pk + l.enc_pk, nullptr, nullptr, nullptr, 0, e, nullptr,
                                     1, l.N, p.Kr, p.BF, 0, st));
    else
        SDR_TRY(launch_pointwise_ffma(framed, kNoNorm, pk + l.enc_src, nullptr, nullptr, nullptr, 0, e, nullptr,
                                      1, l.N, l.A * l.K, p.BF, 0, st));
    SDR_TRY(causal_body(l, pk, e, p.buf(ws, p.o_x), p.buf(ws, p.o_y), p.buf(ws, p.o_m), p.buf(ws, p.o_masked), frames,
                        1, p.BF, B, p.F, state + ss.hist, (long long)ss.slot, st));
    return launch_stream_ola(frames, chunk, state, (long long)ss.slot, (long long)ss.carry, out, B, l.S * l.A, l.A, l.K,
                             p.F, C, apply_mc, st);
}

// The original SuDORMRF.forward (sudormrf.py:266-292; UBlock.forward :164-186).
static int forward_original(const Layout& l, const Plan& p, const float* pk, const float* mixture, float* out,
                            int B, long long T, int apply_mc, char* ws, cudaStream_t st, const float2* rescale) {
    const int L = p.L, D = l.D, Co = l.Co, Ci = l.Ci;
    float* e = p.buf(ws, p.o_e);
    float* x = p.buf(ws, p.o_x);
    float* ex = p.buf(ws, p.o_xt);
    float* y = p.buf(ws, p.o_y);
    float* masked = p.buf(ws, p.o_masked);
    SDR_TRY(front_end(l, p, pk, mixture, B, T, ws, st));                // :268-276: the encoder has a bias and a ReLU
    // x holds u_i = GN(conv_1x1_exp(..)) + block input (raw); the block output PReLU_c(GN_ma(u_i)) is applied by its readers
    NormIn xin = kNoNorm;
    for (int i = 0; i < l.U; ++i) {
        const OrigBlockOff& u = l.ob[i];
        SDR_TRY(gemm(pk, u.proj, x, xin, y, p.slot(ws, i, 0), B, L, st));                           // :171
        SDR_TRY(depthwise_stage(l, p, u, i, 1, pk, ws, st));                                         // :172-182, m in y
        const NormIn nf{p.slot(ws, i, D + 1), pk + u.fn_g, pk + u.fn_be, pk + u.fn_a, (double)Ci * L, 1};
        SDR_TRY(gemm(pk, u.exp, y, nf, ex, p.slot(ws, i, D + 2), B, L, st));                         // :184 conv_1x1_exp.conv
        const NormIn ne{p.slot(ws, i, D + 2), pk + u.exp_g, pk + u.exp_be, nullptr, (double)Co * L, 0};
        SDR_TRY(launch_residual_norm(ex, ne, x, xin, p.slot(ws, i, D + 3), B, Co, L, st));            // :184 .norm, :186 + x
        xin = NormIn{p.slot(ws, i, D + 3), pk + u.ma_g, pk + u.ma_be, pk + u.ma_a, (double)Co * L, 1};   // :186 module_act
    }
    const float* mask_in = x;                              // input of the mask convolution and how to read it
    NormIn mnin = xin;
    if (l.rs.w) {                                                                                     // :279-281
        float* r = p.buf(ws, p.o_o);
        SDR_TRY(gemm(pk, l.rs, x, xin, r, nullptr, B, L, st));
        mask_in = r; mnin = kNoNorm;
    }
    SDR_TRY(gemm(pk, l.mask, mask_in, mnin, masked, nullptr, B, L, st));                              // :284
    SDR_TRY(launch_softmax_gate(masked, e, masked, B, l.S, l.N, L, st));                              // :285-289
    return decoder_tail(l, p, pk, kNoNorm, pk + l.dec_b, mixture, apply_mc, rescale, out, B, T, ws, st);   // :291
}

// What a training forward keeps for the backward (improved model): the forward's statistics slots, the raw encoder
// output e and every block input x_0..x_U (x_U feeds the mask), each segment 256-byte aligned.
struct Saved : Segments {
    size_t o_stats, o_e, o_x, x_stride;
    const float* x(const char* s, int i) const { return reinterpret_cast<const float*>(s + o_x + (size_t)i * x_stride); }
};
static Saved saved_layout(const Layout& l, const Plan& p, int B) {
    Saved s;
    const size_t BL = (size_t)B * p.L * sizeof(float);
    s.o_stats = s.take(p.stats_doubles * sizeof(double));
    s.o_e = s.take(BL * l.N);
    s.x_stride = (BL * l.Co + 255) & ~(size_t)255;
    s.o_x = s.take(s.x_stride * (l.U + 1));
    return s;
}

static int copy_d2d(void* dst, const void* src, size_t bytes, cudaStream_t st) {
    return cuda_status(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st));
}

// `save` (improved model only, else null): the training forward's copy of what saved_layout lists.
static int forward_impl(const Layout& l, const Plan& p, const float* pk, const float* mixture, float* out,
                        int B, long long T, int apply_mc, char* ws, cudaStream_t st,
                        const float2* rescale = nullptr, char* save = nullptr) {
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
    SDR_TRY(front_end(l, p, pk, mixture, B, T, ws, st));
    const Saved sv = save ? saved_layout(l, p, B) : Saved{};
    const size_t xbytes = (size_t)B * L * l.Co * sizeof(float);
    if (save) SDR_TRY(copy_d2d(save + sv.o_x, x, xbytes, st));
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
                SDR_TRY(launch_pointwise_small_preadd(x, o, tn, xt, pk + u.proj.w, pk + u.proj.b, y, p.slot(ws, i, 0),
                                                      ns, u.proj.M, u.proj.K, L, st));
            else
                SDR_TRY(launch_tac_apply(x, o, tn, xt, ns, cob, L, st));
        }
        // proj_1x1: raw + stats
        if (!p.tac_folded) SDR_TRY(gemm(pk, u.proj, bin, kNoNorm, y, p.slot(ws, i, 0), ns, L, st));
        SDR_TRY(depthwise_stage(l, p, u, i, 0, pk, ws, st));              // m reuses y's storage
        // res_conv + skip
        const NormIn nf{p.slot(ws, i, D + 1), pk + u.fn_g, pk + u.fn_be, pk + u.fn_a, (double)cib * L, 0};
        SDR_TRY(gemm(pk, u.res, y, nf, x, nullptr, ns, L, st, {bin}));
        if (save) SDR_TRY(copy_d2d(save + sv.o_x + (size_t)(i + 1) * sv.x_stride, x, xbytes, st));
    }
    if (save) {
        SDR_TRY(copy_d2d(save + sv.o_e, e, (size_t)B * L * l.N * sizeof(float), st));
        SDR_TRY(copy_d2d(save + sv.o_stats, p.stats(ws), p.stats_doubles * sizeof(double), st));
    }
    // mask: PReLU -> 1x1 -> ReLU -> * encoder output
    const NormIn pm{nullptr, nullptr, nullptr, pk + l.mask_a, 1.0, 0};
    SDR_TRY(gemm(pk, l.mask, x, pm, p.buf(ws, p.o_masked), nullptr, B, L, st, {nullptr, e, l.N, 1}));
    // decoder: frames = Wd^T masked, then overlap-add / crop / mixture consistency
    return decoder_tail(l, p, pk, kNoNorm, nullptr, mixture, apply_mc, rescale, out, B, T, ws, st);
}

// ---------------------------------------------------------------------------
// backward of the improved model: workspace plan and orchestration
// ---------------------------------------------------------------------------
// Transposed 1x1 weights for the input-gradient GEMMs, one block's recomputed tensors and their statistics, the
// gradient buffers, and the scratch of the fixed-order reductions.  Every activation buffer is [B][channels][L].
struct BwdPlan : Segments {
    size_t o_wt_mask, o_wt_bn, o_wt_p, o_wt_r, wt_block;    // wt_p / wt_r: per block, wt_block bytes apart
    size_t o_stats, o_dx, o_y, o_m, o_z[kMaxDepthApi], o_dn[kMaxDepthApi], o_dp;
    size_t o_mlog, o_dmask, o_frames, o_de, o_dq, o_win;
    size_t o_npart, o_dwpart, o_wpart;
};

static BwdPlan make_bwd_plan(const Layout& l, const Plan& p, int B) {
    BwdPlan b;
    const size_t F = sizeof(float), BL = (size_t)B * p.L * F;
    const int L = p.L, Co = l.Co, Ci = l.Ci, N = l.N, SN = l.S * l.N, SK = l.S * l.K;
    b.o_wt_mask = b.take((size_t)l.mask.M * l.mask.K * F);
    b.o_wt_bn = b.take((size_t)l.bn.M * l.bn.K * F);
    b.wt_block = ((size_t)Co * Ci * F + 255) & ~(size_t)255;
    b.o_wt_p = b.take(b.wt_block * l.U);
    b.o_wt_r = b.take(b.wt_block * l.U);
    b.o_stats = b.take((size_t)(l.D + 2) * B * 2 * sizeof(double));
    b.o_dx = b.take(BL * Co);
    b.o_y = b.take(BL * Ci);
    b.o_m = b.take(BL * Ci);
    for (int d = 0; d < kMaxDepthApi; ++d) b.o_z[d] = d < l.D ? b.take((BL * Ci) >> d) : 0;
    for (int d = 0; d < kMaxDepthApi; ++d) b.o_dn[d] = d < l.D ? b.take((BL * Ci) >> d) : 0;
    b.o_dp = b.take(BL * Ci);
    b.o_mlog = b.take(BL * SN);
    b.o_dmask = b.take(BL * SN);
    b.o_frames = b.take(BL * SK);
    b.o_de = b.take(BL * N);
    b.o_dq = b.take(BL * (Co > N ? Co : N));
    b.o_win = b.take(BL * l.K);
    const int cmax = Ci > Co ? (Ci > N ? Ci : N) : (Co > N ? Co : N);
    b.o_npart = b.take(norm_bwd_scratch_bytes(B, cmax));
    b.o_dwpart = b.take(dw_bwd_scratch_bytes(B, Ci));
    // every weight-gradient GEMM the backward runs: decoder (on its [S*N][S*K] weight), mask, res_conv and proj_1x1
    // (stated here: with U = 0 there is no block to read them from), bottleneck, encoder
    const int shapes[6][2] = {{l.dec.K, l.dec.M}, {l.mask.M, l.mask.K}, {Co, Ci}, {Ci, Co}, {l.bn.M, l.bn.K}, {N, l.K}};
    size_t wp = 0;
    for (const auto& s : shapes) { const size_t w = wgrad_scratch_bytes(B, s[0], s[1], L); wp = w > wp ? w : wp; }
    b.o_wpart = b.take(wp);
    return b;
}

// Kernels one backward enqueues: transposes (2 + 2U), mask and decoder (12), per block (12 + 5D, + 1 pooling launch
// when D > 1), bottleneck, ln and encoder (8).
static int bwd_launch_count(const Layout& l) {
    return 2 + 2 * l.U + 12 + l.U * (12 + 5 * l.D + (l.D > 1 ? 1 : 0)) + 8;
}

// grads: flat fp32, state_dict order, each tensor sdr_param_numel floats.  Written, never accumulated.
static int backward_impl(const Layout& l, const Plan& p, const BwdPlan& bp, const float* pk, const float* mixture,
                         const char* saved, const float* gout, float* grads, int B, long long T, char* ws,
                         cudaStream_t st) {
    const int L = p.L, D = l.D, N = l.N, Ci = l.Ci, S = l.S, K = l.K;
    const Saved sv = saved_layout(l, p, B);
    const float* e = reinterpret_cast<const float*>(saved + sv.o_e);
    const double* fstats = reinterpret_cast<const double*>(saved + sv.o_stats);   // slot 0: the encoder output's
    auto G = [&](const Param& t) { return grads + t.grad; };
    double* nsc = reinterpret_cast<double*>(ws + bp.o_npart);
    double* dsc = reinterpret_cast<double*>(ws + bp.o_dwpart);
    float* wsc = bp.buf(ws, bp.o_wpart);
    float* wt_mask = bp.buf(ws, bp.o_wt_mask);
    float* wt_bn = bp.buf(ws, bp.o_wt_bn);
    auto wt_p = [&](int i) { return bp.buf(ws, bp.o_wt_p + (size_t)i * bp.wt_block); };
    auto wt_r = [&](int i) { return bp.buf(ws, bp.o_wt_r + (size_t)i * bp.wt_block); };
    // W^T ([K][M]) of a 1x1 convolution into wt, for its input-gradient GEMM
    auto transpose = [&](const Conv1x1& c, float* wt) { return launch_transpose(pk + c.w, wt, c.M, c.K, st); };
    // input gradient on FFMA: dx = W^T dy (+ acc unless null), W^T read from wt
    auto dgrad = [&](const Conv1x1& c, const float* wt, const float* dy, const float* acc, float* dx) {
        return launch_pointwise_ffma(dy, kNoNorm, wt, nullptr, acc, nullptr, 0, dx, nullptr, B, c.K, c.M, L, 0, st);
    };
    // weight and bias gradients of a 1x1 convolution whose input x was read through nin
    auto wgrad = [&](const Conv1x1& c, const float* dy, const float* x, const NormIn& nin) {
        return launch_wgrad(dy, x, nin, G(c.w), G(c.b), wsc, B, c.M, c.K, L, st);
    };
    SDR_TRY(transpose(l.mask, wt_mask));
    SDR_TRY(transpose(l.bn, wt_bn));
    for (int i = 0; i < l.U; ++i) {
        SDR_TRY(transpose(l.ub[i].proj, wt_p(i)));
        SDR_TRY(transpose(l.ub[i].res, wt_r(i)));
    }
    float* dx = bp.buf(ws, bp.o_dx);
    float* mlog = bp.buf(ws, bp.o_mlog);
    float* dmask = bp.buf(ws, bp.o_dmask);
    float* frames = bp.buf(ws, bp.o_frames);
    float* de = bp.buf(ws, bp.o_de);
    float* dq = bp.buf(ws, bp.o_dq);

    // mask and decoder: mlog = W_m PReLU_m(x_U) + b_m, masked = relu(mlog) * e, frames = Wd^T masked, crop + overlap-add
    const float* xU = sv.x(saved, l.U);
    const NormIn pm{nullptr, nullptr, nullptr, pk + l.mask_a, 1.0, 0};
    SDR_TRY(launch_pointwise_ffma(xU, pm, pk + l.mask.w, pk + l.mask.b, nullptr, nullptr, 0, mlog, nullptr,
                                  B, l.mask.M, l.mask.K, L, 0, st));   // fp32: the ReLU mask bits follow the logits closely
    SDR_TRY(launch_mask_apply(mlog, e, dmask, B, S, N, L, st));                    // dmask holds masked for now
    SDR_TRY(launch_frame_gather(gout, frames, B, S, K, L, T, st));                 // dF
    // decoder.weight [S*N][S][K] is the transpose of l.dec
    SDR_TRY(launch_wgrad(dmask, frames, kNoNorm, G(l.dec_w), nullptr, wsc, B, l.dec.K, l.dec.M, L, st));
    SDR_TRY(dgrad(l.dec, pk + l.dec_w, frames, nullptr, dmask));                   // dmasked = Wd dF
    SDR_TRY(launch_mask_bwd(mlog, e, dmask, de, B, S, N, L, st));                  // dmlog (in dmask), de
    SDR_TRY(wgrad(l.mask, dmask, xU, pm));
    SDR_TRY(dgrad(l.mask, wt_mask, dmask, nullptr, dq));                           // W_m^T dmlog
    SDR_TRY(launch_norm_bwd(xU, pm, dq, dx, 0, nullptr, nullptr, G(l.mask_a), nsc, B, l.Co, L, st));   // dx_U

    // U-ConvBlocks, last to first: recompute from x_i, then backward; dx carries the residual stream's gradient
    double* bst = reinterpret_cast<double*>(ws + bp.o_stats);
    auto slot = [&](int k) { return bst + (size_t)k * B * 2; };
    float* y = bp.buf(ws, bp.o_y);
    float* m = bp.buf(ws, bp.o_m);
    float* dp = bp.buf(ws, bp.o_dp);
    float* z[kMaxDepthApi];
    float* dn[kMaxDepthApi];
    for (int d = 0; d < D; ++d) { z[d] = bp.buf(ws, bp.o_z[d]); dn[d] = bp.buf(ws, bp.o_dn[d]); }
    for (int i = l.U - 1; i >= 0; --i) {
        const UBlockOff& u = l.ub[i];
        const float* xi = sv.x(saved, i);
        SDR_TRY(cuda_status(cudaMemsetAsync(bst, 0, (size_t)(D + 2) * B * 2 * sizeof(double), st)));
        SDR_TRY(gemm(pk, u.proj, xi, kNoNorm, y, slot(0), B, L, st));
        const NormIn n0{slot(0), pk + u.proj_g, pk + u.proj_be, pk + u.proj_a, (double)Ci * L, 0};
        NormIn nl[kMaxDepthApi];
        SDR_TRY(depthwise_levels(u, pk, D, y, n0, z, m, slot(0), nl, B, Ci, L, st));
        const NormIn nf{slot(D + 1), pk + u.fn_g, pk + u.fn_be, pk + u.fn_a, (double)Ci * L, 0};

        // out = W_r PReLU_f(GLN_f(m)) + b_r + x
        SDR_TRY(wgrad(u.res, dx, m, nf));
        SDR_TRY(dgrad(u.res, wt_r(i), dx, nullptr, dp));
        SDR_TRY(launch_norm_bwd(m, nf, dp, dp, 0, G(u.fn_g), G(u.fn_be), G(u.fn_a), nsc, B, Ci, L, st));   // dm
        // m[t] = sum_d n_d[t >> d]: the deepest level's gradient is dm pooled; the others get theirs from the
        // depthwise backward of the level below them
        const float* up = dp;
        if (D > 1) {
            SDR_TRY(launch_dw_bwd(nullptr, nullptr, kNoNorm, nullptr, dp, 1 << (D - 1), dn[D - 1], nullptr, nullptr,
                                  nullptr, B, Ci, L >> (D - 1), 2, st));
            up = dn[D - 1];
        }
        for (int d = D - 1; d >= 0; --d) {
            const int Ld = L >> d;
            SDR_TRY(launch_norm_bwd(z[d], nl[d], up, dn[d], 0, G(u.dw_g[d]), G(u.dw_be[d]), nullptr, nsc,
                                    B, Ci, Ld, st));                               // dz_d
            if (d > 0)      // dn_{d-1} = pool(dm) + dw_d^T dz_d
                SDR_TRY(launch_dw_bwd(dn[d], z[d - 1], nl[d - 1], pk + u.dw_w[d], dp, 1 << (d - 1), dn[d - 1],
                                      G(u.dw_w[d]), G(u.dw_b[d]), dsc, B, Ci, L >> (d - 1), 2, st));
            else            // gradient of PReLU_p(GLN_p(y)), over dm (no longer needed)
                SDR_TRY(launch_dw_bwd(dn[0], y, n0, pk + u.dw_w[0], nullptr, 0, dp, G(u.dw_w[0]), G(u.dw_b[0]), dsc,
                                      B, Ci, L, 1, st));
            up = d > 0 ? dn[d - 1] : nullptr;
        }
        SDR_TRY(launch_norm_bwd(y, n0, dp, dp, 0, G(u.proj_g), G(u.proj_be), G(u.proj_a), nsc, B, Ci, L, st));   // dy
        SDR_TRY(wgrad(u.proj, dp, xi, kNoNorm));
        SDR_TRY(dgrad(u.proj, wt_p(i), dp, dx, dx));                               // dx += W_p^T dy
    }

    // x_0 = W_bn GLN_ln(e) + b_bn; e = encoder(mixture)
    const NormIn ln{fstats, pk + l.ln_g, pk + l.ln_be, nullptr, (double)N * L, 0};
    SDR_TRY(wgrad(l.bn, dx, e, ln));
    SDR_TRY(dgrad(l.bn, wt_bn, dx, nullptr, dq));
    SDR_TRY(launch_norm_bwd(e, ln, dq, de, 1, G(l.ln_g), G(l.ln_be), nullptr, nsc, B, N, L, st));   // de += GLN bwd
    float* win = bp.buf(ws, bp.o_win);
    SDR_TRY(launch_frame_gather(mixture, win, B, 1, K, L, T, st));                 // the encoder's input windows
    return launch_wgrad(de, win, kNoNorm, G(l.enc_w), nullptr, wsc, B, N, K, L, st);
}

// A buffer handed to an entry that enqueues a whole model: `align` bytes of alignment, and at least `need` bytes where
// the caller says it has `bytes`.
struct Buf { const void* ptr; size_t align = 1, bytes = 0, need = 0; };
// Refuses a null buffer first, then one that is too small, then one that is misaligned.
static int check_buffers(std::initializer_list<Buf> bufs) {
    for (const Buf& b : bufs) if (!b.ptr) return SDR_ERR_BAD_ARGUMENT;
    for (const Buf& b : bufs) if (b.bytes < b.need) return SDR_ERR_WORKSPACE;
    for (const Buf& b : bufs) if (reinterpret_cast<uintptr_t>(b.ptr) % b.align) return SDR_ERR_BAD_ARGUMENT;
    return SDR_OK;
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
    return l.ok ? (int)l.entries.size() : SDR_ERR_BAD_CONFIG;
}

int64_t sdr_param_numel(const sdr_config* cfg, int index) {
    const Layout l = make_layout(cfg);
    if (!l.ok) return SDR_ERR_BAD_CONFIG;
    if (index < 0 || index >= (int)l.entries.size()) return SDR_ERR_BAD_ARGUMENT;
    return (int64_t)l.entries[index].numel;
}

int64_t sdr_param_name(const sdr_config* cfg, int index, char* buf, size_t buf_bytes) {
    const Layout l = make_layout(cfg);
    if (!l.ok) return SDR_ERR_BAD_CONFIG;
    if (index < 0 || index >= (int)l.entries.size() || (!buf && buf_bytes)) return SDR_ERR_BAD_ARGUMENT;
    const Entry& e = l.entries[index];
    char name[96];              // the longest key, "sm.<int>.UBlock.spp_dw.<d>.norm.gamma", takes 41 bytes
    int n = snprintf(name, sizeof(name), e.blk, e.i);
    n += snprintf(name + n, sizeof(name) - n, e.name, e.d);
    n += snprintf(name + n, sizeof(name) - n, "%s", e.leaf);
    if (buf && buf_bytes <= (size_t)n) return SDR_ERR_WORKSPACE;
    if (buf) memcpy(buf, name, (size_t)n + 1);
    return n;
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
    if (!params || n_params != (int)l.entries.size()) return SDR_ERR_BAD_ARGUMENT;
    SDR_TRY(check_buffers({{packed, 16, packed_bytes, l.total * sizeof(float)}}));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* pk = static_cast<float*>(packed);
    SDR_TRY(cuda_status(cudaMemsetAsync(pk, 0, l.total * sizeof(float), st)));
    for (size_t i = 0; i < l.entries.size(); ++i) {
        if (!params[i]) return SDR_ERR_BAD_ARGUMENT;
        SDR_TRY(copy_d2d(pk + l.entries[i].off, params[i], l.entries[i].numel * sizeof(float), st));
    }
    // the derived regions, then the images (some are packed from a derived region): all in stream order
    if (l.orig) {
        SDR_TRY(launch_toeplitz_mask(pk + l.m_w, pk + l.m_b, pk + l.mask.w, pk + l.mask.b, l.S, l.N, st));
        SDR_TRY(launch_grouped_decoder(pk + l.dec_w, pk + l.dec.w, l.S, l.N, l.K, st));
    } else {
        // decoder.weight [C][SA][K] -> [SA*K][C]
        SDR_TRY(launch_transpose(pk + l.dec_w, pk + l.dec.w, l.dec.K, l.dec.M, st));
    }
    if (l.causal) {
        SDR_TRY(launch_take_taps(pk + l.enc_w, pk + l.enc_wc, (long long)l.N * l.A, 2 * l.K - 1, l.K, st));
        for (const CausalBlockOff& u : l.cb) {
            SDR_TRY(launch_scale_by_scalar(pk + u.res.w, pk + u.gain, pk + u.res_g.w, (long long)u.res.M * u.res.K, st));
            SDR_TRY(launch_scale_by_scalar(pk + u.res.b, pk + u.gain, pk + u.res_g.b, u.res.M, st));
        }
    }
    for (const Conv1x1& c : l.images) SDR_TRY(pack_pointwise_mma(pk + c.w, c.M, c.K, pk + c.pk, st));
    if (l.enc_pk) SDR_TRY(pack_encoder_mma(pk + l.enc_src, l.N, l.A, l.K, pk + l.enc_pk, st));
    return SDR_OK;
}

size_t sdr_workspace_bytes(const sdr_config* cfg, int B, int64_t T) {
    const Layout l = make_layout(cfg);
    if (!l.ok || B <= 0 || T <= 0 || !counts_fit(l, B, T)) return 0;
    return make_plan(l, B, T).total;
}

static int check_forward_args(const Layout& l, int B, int64_t T) {
    if (!l.ok) return SDR_ERR_BAD_CONFIG;
    if (B <= 0 || T <= 0) return SDR_ERR_BAD_ARGUMENT;
    if (!counts_fit(l, B, T)) return SDR_ERR_UNSUPPORTED;
    if (l.gc) {
        const int n = l.cob;
        if (!(n == 4 || n == 8 || n == 16 || n == 32) || l.G > 16) return SDR_ERR_UNSUPPORTED;
    }
    if (padded_len(l, T) / l.hop > 0x3fffffffLL) return SDR_ERR_UNSUPPORTED;
    // the FFMA encoder (no tensor-core image: N < 32) holds A audio channels x K taps in one CTA's shared memory
    if (!l.enc_pk && !encoder_ffma_fits(l.A, l.K)) return SDR_ERR_UNSUPPORTED;
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
    const Plan p = make_plan(l, B, T);
    SDR_TRY(check_buffers({{packed, 16}, {mixture}, {out}, {workspace, 256, workspace_bytes, p.total}}));
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
    if (!counts_fit(l, B, T)) return SDR_ERR_UNSUPPORTED;
    return launch_count(l, make_plan(l, B, T));
}

// ---- training of the improved model: forward that keeps what the backward needs, and the backward ----

static int check_train_args(const Layout& l, int B, int64_t T) {
    if (!l.ok) return SDR_ERR_BAD_CONFIG;
    if (l.gc || l.causal || l.orig) return SDR_ERR_UNSUPPORTED;     // improved model only
    return check_forward_args(l, B, T);
}

size_t sdr_train_saved_bytes(const sdr_config* cfg, int B, int64_t T) {
    const Layout l = make_layout(cfg);
    if (check_train_args(l, B, T) != SDR_OK) return 0;
    return saved_layout(l, make_plan(l, B, T), B).total;
}

size_t sdr_backward_workspace_bytes(const sdr_config* cfg, int B, int64_t T) {
    const Layout l = make_layout(cfg);
    if (check_train_args(l, B, T) != SDR_OK) return 0;
    return make_bwd_plan(l, make_plan(l, B, T), B).total;
}

int sdr_forward_train(const sdr_config* cfg, const void* packed, const float* mixture, float* out, int B, int64_t T,
                      void* saved, size_t saved_bytes, void* ws, size_t ws_bytes, sdr_stream stream) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_train_args(l, B, T));
    const Plan p = make_plan(l, B, T);
    SDR_TRY(check_buffers({{packed, 16}, {mixture}, {out}, {saved, 256, saved_bytes, saved_layout(l, p, B).total},
                           {ws, 256, ws_bytes, p.total}}));
    return forward_impl(l, p, static_cast<const float*>(packed), mixture, out, B, T, 0, static_cast<char*>(ws),
                        static_cast<cudaStream_t>(stream), nullptr, static_cast<char*>(saved));
}

int sdr_backward(const sdr_config* cfg, const void* packed, const float* mixture, const void* saved,
                 const float* grad_out, float* grad_params, int B, int64_t T, void* ws, size_t ws_bytes,
                 sdr_stream stream) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_train_args(l, B, T));
    const Plan p = make_plan(l, B, T);
    const BwdPlan bp = make_bwd_plan(l, p, B);
    SDR_TRY(check_buffers({{packed, 16}, {mixture}, {saved, 256}, {grad_out}, {grad_params},
                           {ws, 256, ws_bytes, bp.total}}));
    return backward_impl(l, p, bp, static_cast<const float*>(packed), mixture, static_cast<const char*>(saved),
                         grad_out, grad_params, B, T, static_cast<char*>(ws), static_cast<cudaStream_t>(stream));
}

int sdr_backward_launch_count(const sdr_config* cfg, int B, int64_t T) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_train_args(l, B, T));
    return bwd_launch_count(l);
}

// stage entries of the backward kernels
size_t sdr_pointwise_wgrad_scratch_bytes(int samples, int M, int Kc, int L) {
    if (samples <= 0 || M <= 0 || Kc <= 0 || L <= 0) return 0;
    return wgrad_scratch_bytes(samples, M, Kc, L);
}

int sdr_pointwise_wgrad(const float* dy, const float* x, const sdr_norm_in* fin, float* dw, float* db_or_null,
                        void* scratch, int samples, int M, int Kc, int L, sdr_stream stream) {
    return launch_wgrad(dy, x, make_norm(fin), dw, db_or_null, static_cast<float*>(scratch), samples, M, Kc, L,
                        static_cast<cudaStream_t>(stream));
}

size_t sdr_norm_act_backward_scratch_bytes(int samples, int C) {
    return samples > 0 && C > 0 ? norm_bwd_scratch_bytes(samples, C) : 0;
}

int sdr_norm_act_backward(const float* x, const sdr_norm_in* fin, const float* dp, float* dx, int accumulate,
                          float* dgamma, float* dbeta, float* dslope, void* scratch, int samples, int C, int L,
                          sdr_stream stream) {
    if (scratch && reinterpret_cast<uintptr_t>(scratch) % 8) return SDR_ERR_BAD_ARGUMENT;
    return launch_norm_bwd(x, make_norm(fin), dp, dx, accumulate, dgamma, dbeta, dslope, static_cast<double*>(scratch),
                           samples, C, L, static_cast<cudaStream_t>(stream));
}

size_t sdr_depthwise_backward_scratch_bytes(int samples, int C) {
    return samples > 0 && C > 0 ? dw_bwd_scratch_bytes(samples, C) : 0;
}

int sdr_depthwise_backward(const float* dz, const float* x, const sdr_norm_in* fin, const float* w5,
                           const float* pool_or_null, int pool_factor, float* dx, float* dw5, float* dbias,
                           void* scratch, int samples, int C, int Lin, int stride, sdr_stream stream) {
    if (scratch && reinterpret_cast<uintptr_t>(scratch) % 8) return SDR_ERR_BAD_ARGUMENT;
    return launch_dw_bwd(dz, x, make_norm(fin), w5, pool_or_null, pool_factor, dx, dw5, dbias,
                         static_cast<double*>(scratch), samples, C, Lin, stride, static_cast<cudaStream_t>(stream));
}

int sdr_mask_backward(const float* mlog, const float* enc, float* dmasked, float* denc, int B, int S, int N, int L,
                      sdr_stream stream) {
    return launch_mask_bwd(mlog, enc, dmasked, denc, B, S, N, L, static_cast<cudaStream_t>(stream));
}

int sdr_overlap_add_backward(const float* grad_out, float* grad_frames, int B, int SA, int K, int L, int64_t T,
                             sdr_stream stream) {
    return launch_frame_gather(grad_out, grad_frames, B, SA, K, L, T, static_cast<cudaStream_t>(stream));
}

size_t sdr_encoder_wgrad_scratch_bytes(int B, int N, int K, int L) {
    if (B <= 0 || N <= 0 || K <= 0 || L <= 0) return 0;
    return (((size_t)B * K * L * sizeof(float) + 255) & ~(size_t)255) + wgrad_scratch_bytes(B, N, K, L);
}

int sdr_encoder_wgrad(const float* denc, const float* wav, float* dw, void* scratch, int B, int N, int K, int L,
                      int64_t T, sdr_stream stream) {
    if (!scratch || reinterpret_cast<uintptr_t>(scratch) % 16) return SDR_ERR_BAD_ARGUMENT;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* win = static_cast<float*>(scratch);
    float* part = reinterpret_cast<float*>(static_cast<char*>(scratch) +
                                           (((size_t)B * K * L * sizeof(float) + 255) & ~(size_t)255));
    SDR_TRY(launch_frame_gather(wav, win, B, 1, K, L, T, st));
    return launch_wgrad(denc, win, kNoNorm, dw, nullptr, part, B, N, K, L, st);
}

// ---- streaming of the causal model ----

int64_t sdr_stream_granule(const sdr_config* cfg) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_stream_config(l));
    return stream_granule(l);
}

size_t sdr_stream_state_bytes(const sdr_config* cfg, int B) {
    const Layout l = make_layout(cfg);
    if (check_stream_config(l) != SDR_OK || B <= 0) return 0;
    return (size_t)B * stream_state(l).slot * sizeof(float);
}

size_t sdr_stream_workspace_bytes(const sdr_config* cfg, int B, int64_t C) {
    const Layout l = make_layout(cfg);
    if (check_stream_args(l, B, C) != SDR_OK) return 0;
    return make_stream_plan(l, B, C).total;
}

int sdr_stream_launch_count(const sdr_config* cfg, int B, int64_t C) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_stream_args(l, B, C));
    return 3 * l.U + 6;                // framing, encoder, bottleneck, U x (proj, stream stage, res), mask, decoder, overlap-add
}

int sdr_stream_reset(const sdr_config* cfg, void* state, int B, const int32_t* host_slots_or_null, int n,
                     sdr_stream stream) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_stream_config(l));
    if (B <= 0 || (host_slots_or_null && n < 0)) return SDR_ERR_BAD_ARGUMENT;
    SDR_TRY(check_buffers({{state, 16}}));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t slot = stream_state(l).slot * sizeof(float);
    if (!host_slots_or_null)
        return cuda_status(cudaMemsetAsync(state, 0, (size_t)B * slot, st));
    return reset_slots({{state, slot}}, B, host_slots_or_null, n, nullptr, st);
}

int sdr_stream_reset_masked(const sdr_config* cfg, void* state, int B, const uint8_t* mask, sdr_stream stream) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_stream_config(l));
    if (B <= 0) return SDR_ERR_BAD_ARGUMENT;
    SDR_TRY(check_buffers({{state, 16}, {mask}}));
    return reset_slots({{state, stream_state(l).slot * sizeof(float)}}, B, nullptr, 0, mask,
                       static_cast<cudaStream_t>(stream));
}

int sdr_stream_step(const sdr_config* cfg, const void* packed, void* state, const float* chunk, float* out, int B,
                    int64_t C, int apply_mixture_consistency, void* ws, size_t ws_bytes, sdr_stream stream) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_stream_args(l, B, C));
    if (apply_mixture_consistency && l.A != 1) return SDR_ERR_UNSUPPORTED;
    const StreamPlan p = make_stream_plan(l, B, C);
    SDR_TRY(check_buffers({{packed, 16}, {state, 16}, {chunk}, {out}, {ws, 256, ws_bytes, p.total}}));
    return stream_step(l, p, static_cast<const float*>(packed), static_cast<float*>(state), chunk, out, B, C,
                       apply_mixture_consistency, static_cast<char*>(ws), static_cast<cudaStream_t>(stream));
}

int sdr_stream_flush(const sdr_config* cfg, void* state, float* tail, int B, int apply_mixture_consistency,
                     sdr_stream stream) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_stream_config(l));
    if (apply_mixture_consistency && l.A != 1) return SDR_ERR_UNSUPPORTED;
    if (B <= 0) return SDR_ERR_BAD_ARGUMENT;
    SDR_TRY(check_buffers({{state, 16}, {tail}}));
    const StreamState ss = stream_state(l);
    return launch_stream_flush(static_cast<const float*>(state), (long long)ss.slot, (long long)ss.carry, tail, B,
                               l.S * l.A, l.hop, apply_mixture_consistency, static_cast<cudaStream_t>(stream));
}

int sdr_causal_stream_stage(const float* y, const float* slope_in, const float* const* w21, const float* const* bias,
                            const float* const* slope, float* history, float* m, int D, int B, int C, int F,
                            sdr_stream stream) {
    if (D < 1 || D > kMaxDepthApi) return SDR_ERR_UNSUPPORTED;
    return launch_causal_stream(y, slope_in, w21, bias, slope, history, (long long)D * 10 * C, m, D, B, C, F,
                                static_cast<cudaStream_t>(stream));
}

// Byte offsets of the buffers either side of the forward.  sdr_forward_host stages the mixture at 0 and the estimates
// at `est` of its device buffer (`staging` bytes); sdr_separate appends the normalised mixture, the per-row sums (at
// `sums`) and the per-row (mean, std) (at `ms`) to the forward's workspace (`separate` bytes past its end).
struct IoOffsets { size_t est, staging, sums, ms, separate; };
static IoOffsets io_offsets(const Layout& l, int B, long long T) {
    const size_t mixture = (size_t)B * l.A * T * sizeof(float);
    IoOffsets o;
    Segments staging, extra;
    staging.take(mixture);
    o.est = staging.take((size_t)B * l.S * l.A * T * sizeof(float));
    o.staging = staging.total;
    extra.take(mixture);
    o.sums = extra.take((size_t)B * 2 * sizeof(double));
    o.ms = extra.take((size_t)B * sizeof(float2));
    o.separate = extra.total;
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
    const IoOffsets io = io_offsets(l, B, T);
    // every buffer before the first copy is enqueued, the forward's workspace included
    SDR_TRY(check_buffers({{packed, 16}, {host_mixture}, {host_out}, {dev_io, 256, dev_io_bytes, io.staging},
                           {workspace, 256, workspace_bytes, make_plan(l, B, T).total}}));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t in_bytes = (size_t)B * l.A * T * sizeof(float);
    const size_t out_bytes = (size_t)B * l.S * l.A * T * sizeof(float);
    float* d_in = static_cast<float*>(dev_io);
    float* d_out = reinterpret_cast<float*>(static_cast<char*>(dev_io) + io.est);
    SDR_TRY(cuda_status(cudaMemcpyAsync(d_in, host_mixture, in_bytes, cudaMemcpyHostToDevice, st)));
    SDR_TRY(sdr_forward(cfg, packed, d_in, d_out, B, T, apply_mixture_consistency, workspace, workspace_bytes, stream));
    return cuda_status(cudaMemcpyAsync(host_out, d_out, out_bytes, cudaMemcpyDeviceToHost, st));
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
    if (!l.ok || B <= 0 || T <= 0 || !counts_fit(l, B, T)) return 0;
    return make_plan(l, B, T).total + io_offsets(l, B, T).separate;
}

static int separate_impl(const sdr_config* cfg, const void* packed, const float* wav, const int64_t* lengths,
                         float* out, int B, int64_t T, int apply_mixture_consistency, int rescale,
                         void* workspace, size_t workspace_bytes, sdr_stream stream) {
    const Layout l = make_layout(cfg);
    SDR_TRY(check_forward_args(l, B, T));
    if (l.A != 1) return SDR_ERR_UNSUPPORTED;            // the README recipe is written for mono mixtures
    const Plan p = make_plan(l, B, T);
    const IoOffsets io = io_offsets(l, B, T);
    SDR_TRY(check_buffers({{packed, 16}, {wav}, {out}, {workspace, 256, workspace_bytes, p.total + io.separate}}));
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

}  // extern "C"
#pragma GCC visibility pop
