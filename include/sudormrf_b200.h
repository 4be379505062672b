/*
 * sudormrf_b200.h — C ABI of the H100-native SuDoRM-RF forward path.
 *
 * The reference (etzinis/sudo_rm_rf) has no native/FFI layer: its boundary is
 * the Python nn.Module contract.  This header is the C-ABI that sits UNDER the
 * Python mirror of that contract (sudo_rm_rf_b200/improved_sudormrf.py etc.);
 * each entry point names the reference interface it replaces (file:line in
 * /root/reference).  Plain pointers and sizes only; no torch types.
 *
 * Ownership: the caller owns every byte (parameters, packed weights,
 * workspace, inputs, outputs are caller-allocated device buffers); the library
 * never allocates or frees device memory and keeps no mutable global state
 * beyond one-time cudaFuncSetAttribute calls.  All work is enqueued on the
 * stream passed in; nothing synchronises.  Fully re-entrant (nn.DataParallel
 * calls forward from one host thread per device).
 *
 * Caller-owned buffers (tests/test_gpu_scratch.py runs every entry on exactly-sized, guarded buffers filled with
 * NaN and with 1e30 patterns):
 *   - Contents on entry are ignored for every workspace and scratch buffer, `saved` of sdr_forward_train, the device
 *     staging buffer of sdr_forward_host, the packed buffer of sdr_pack_weights and every output: a result depends on
 *     the weights and the inputs only, whatever an earlier call of any shape or variant left behind.  Every element
 *     of an output is written.  Nothing outside the stated sizes is read or written, and inputs are not modified.
 *   - Required on entry: the stream state reset by sdr_stream_reset before a slot's first step; the statistics
 *     slots of the per-stage entries zeroed (they are accumulated into: a pre-loaded `stats0` / `stats_m` of the
 *     pyramid entries comes back as pre-load + sums); the padding of a ragged batch zero (sdr_separate_ragged).
 *   - Size: the byte count the matching size query returns suffices exactly.
 *   - Alignment: 256 bytes for workspaces, `saved` and the staging buffer; 16 bytes for the packed weights and the
 *     stream state; 8 bytes for the scratch of the metrics.
 *   - The whole-model entries (sdr_pack_weights, sdr_forward, sdr_forward_host, sdr_separate, sdr_separate_ragged,
 *     sdr_stream_reset / _step / _flush, sdr_forward_train, sdr_backward) refuse a null, too small
 *     (SDR_ERR_WORKSPACE) or misaligned (SDR_ERR_BAD_ARGUMENT) buffer before anything is enqueued.
 *   - Non-finite inputs are neither refused nor sanitised: a NaN or inf in mixture (slot, utterance) j changes no
 *     other mixture's output, and makes j's output non-finite where the reference's is (DESIGN.md section 2).
 *
 * Errors: integer return codes, 0 = OK, negative = failure (see
 * sdr_error_string).  No C++ exceptions cross the ABI.
 */
#ifndef SUDORMRF_B200_H
#define SUDORMRF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SDR_ABI_VERSION 2

/* return codes */
#define SDR_OK                 0
#define SDR_ERR_BAD_CONFIG    -1   /* constructor arguments the kernels cannot run */
#define SDR_ERR_BAD_ARGUMENT  -2   /* null pointer, wrong count, B/T <= 0 ... */
#define SDR_ERR_WORKSPACE     -3   /* workspace / packed buffer too small */
#define SDR_ERR_CUDA          -4   /* a CUDA call or launch failed */
#define SDR_ERR_UNSUPPORTED   -5   /* valid for the reference, not implemented here */

/* Constructor arguments of the reference models:
 *   improved_sudormrf.py:224-231   SuDORMRF.__init__
 *   groupcomm_sudormrf_v2.py:232-241 GroupCommSudoRmRf.__init__
 *   causal_improved_sudormrf_v3.py:121-129 CausalSuDORMRF.__init__
 *   sudormrf.py:186-193 SuDORMRF.__init__ (the original model)             */
typedef struct {
    int32_t variant;            /* 0 = improved SuDORMRF, 1 = GroupCommSudoRmRf, 2 = CausalSuDORMRF,
                                   3 = the original SuDORMRF (sudormrf.py) */
    int32_t in_audio_channels;  /* 1 for improved */
    int32_t out_channels;
    int32_t in_channels;
    int32_t num_blocks;
    int32_t upsampling_depth;
    int32_t enc_kernel_size;
    int32_t enc_num_basis;
    int32_t num_sources;
    int32_t group_size;         /* ignored for improved */
} sdr_config;

typedef void* sdr_stream;       /* a cudaStream_t (CUstream); NULL = legacy default stream */

int         sdr_abi_version(void);
const char* sdr_error_string(int code);

/* Number of parameter tensors in the reference's state_dict() order
 * (improved_sudormrf.py:247-281, :170-196; groupcomm_sudormrf_v2.py:262-299,
 * :347-354, :401-403; causal_improved_sudormrf_v3.py:146-189, :71-96) and the
 * element count of parameter i.  For the causal model the caller passes
 * skipinit_gain already multiplied by the block's alpha and proj_1x1's weight
 * divided by its beta (both 1.0 in the reference's constructor, :165-174).
 * Original model (variant 3, sudormrf.py:211-264, :134-162): every state_dict
 * entry in order EXCEPT the trailing ln_mask_in.{weight,bias}, which forward
 * never reads (:264).                                                         */
int     sdr_num_params(const sdr_config* cfg);
int64_t sdr_param_numel(const sdr_config* cfg, int index);
/* The state_dict key of parameter i, e.g. "sm.3.spp_dw.2.norm.gamma": the
 * library names every entry it packs, with the same exception (the original
 * model's ln_mask_in.{weight,bias} has no index).  Returns the key's length
 * without the terminating NUL, and writes the key with its NUL when buf_bytes
 * exceeds that length.  buf = NULL with buf_bytes = 0 is a size query.
 * SDR_ERR_BAD_CONFIG for a bad config; SDR_ERR_BAD_ARGUMENT for an index
 * outside [0, sdr_num_params) or a NULL buf with buf_bytes > 0;
 * SDR_ERR_WORKSPACE, writing nothing, for a non-NULL buf that is too small.    */
int64_t sdr_param_name(const sdr_config* cfg, int index, char* buf, size_t buf_bytes);

/* Padded length rule of pad_to_appropriate_length (improved_sudormrf.py:303-310;
 * variant 3: sudormrf.py:206-209,283-293, multiples of lcm(hop, 2^depth)).     */
int64_t sdr_padded_length(const sdr_config* cfg, int64_t T);

/* Packed weights: one flat device buffer holding every parameter plus derived
 * layouts (decoder weight as a [S*K, S*N] matrix, ...).  A single buffer so the
 * multi-GPU driver can broadcast it with ONE ncclBroadcast.  Replaces the
 * per-forward module replication of nn.DataParallel
 * (run_improved_sudormrf.py:118).                                            */
size_t sdr_packed_weight_bytes(const sdr_config* cfg);
int    sdr_pack_weights(const sdr_config* cfg,
                        const float* const* params, /* host array of n device pointers, state_dict order, fp32 contiguous */
                        int n_params,
                        void* packed, size_t packed_bytes, sdr_stream stream);

/* Caller-allocated scratch for a forward at batch B, length T (all
 * intermediates + the GlobLN statistics).  The forward, the separate() recipe and
 * sdr_mixture_consistency take any B whose buffers fit; no kernel's grid limits the
 * batch.  Refused (this query then returns 0, the launch count and the forward
 * SDR_ERR_UNSUPPORTED): B * group_size > 2^31 - 1, and more than 2^31 - 1
 * channels x frames in one GlobLN sample; the kernels count both in int.     */
size_t sdr_workspace_bytes(const sdr_config* cfg, int B, int64_t T);

/* SuDORMRF.forward (improved_sudormrf.py:283-301) /
 * GroupCommSudoRmRf.forward (groupcomm_sudormrf_v2.py:302-322) /
 * CausalSuDORMRF.forward (causal_improved_sudormrf_v3.py:191-211) /
 * the original SuDORMRF.forward (sudormrf.py:266-292), optionally
 * followed by mixture_consistency.apply(..., 'uniform')
 * (mixture_consistency.py:14-36; only when in_audio_channels == 1).
 *   mixture: device [B, in_audio_channels, T] fp32 contiguous
 *   out:     device [B, num_sources*in_audio_channels, T] fp32 contiguous   */
int sdr_forward(const sdr_config* cfg, const void* packed,
                const float* mixture, float* out, int B, int64_t T,
                int apply_mixture_consistency,
                void* workspace, size_t workspace_bytes, sdr_stream stream);

/* Number of kernels one sdr_forward of B mixtures of T samples enqueues (the benchmark's gpu_launches claim).  The
 * depthwise levels of a block run as one pass or level by level depending on the padded length and, through the
 * pyramid's per-sample table, on the number of GlobLN samples (B, or B * group_size for GroupComm).
 * sdr_forward_launch_count is the count for B = 1, T = 32000; sdr_forward_launch_count_at for B = 1 at any T.  */
int sdr_forward_launch_count(const sdr_config* cfg);
int sdr_forward_launch_count_at(const sdr_config* cfg, int64_t T);
int sdr_forward_launch_count_for(const sdr_config* cfg, int B, int64_t T);

/* Same call with HOST buffers (pinned for real asynchrony): H2D copy of the
 * mixture, forward, D2H copy of the estimates, all on `stream`.  `dev_io` is a
 * device staging buffer of sdr_host_staging_bytes().  This is the end-to-end
 * entry the benchmark's `e2e` figure times.                                  */
size_t sdr_host_staging_bytes(const sdr_config* cfg, int B, int64_t T);
int sdr_forward_host(const sdr_config* cfg, const void* packed,
                     const float* host_mixture, float* host_out, int B, int64_t T,
                     int apply_mixture_consistency,
                     void* dev_io, size_t dev_io_bytes,
                     void* workspace, size_t workspace_bytes, sdr_stream stream);

/* ---- streaming of the causal model (variant 2) ---------------------------
 * CausalSuDORMRF has no normalisation layers, so it can run chunk by chunk with
 * a small carried state per slot and produce what model(x) produces on the
 * concatenation, delayed by hop = enc_kernel_size / 2 samples:
 *   cat(step(x_0) .. step(x_{n-1}))[..., hop:] == model(x)[..., :n*C - hop]
 *   flush() == model(x)[..., n*C - hop : n*C]      when n*C % (hop * 2^depth) == 0
 * (otherwise the reference's zero padding adds one more frame, and only the
 * first identity holds).  The first hop samples of the first step are zeros.
 *
 * Granule G = hop * max(4, 2^(depth-1)) samples; a chunk C is a multiple of G
 * of at most 4096 * hop samples.  The state ([B] slots; layout private, slots
 * contiguous) and the step workspace are caller-allocated device buffers; the
 * state must be zeroed by sdr_stream_reset before the first step.  Nothing
 * synchronises, and a step can be captured in a CUDA graph.  Variants other
 * than 2 and chunks that are not a multiple of G return SDR_ERR_UNSUPPORTED.  */
int64_t sdr_stream_granule(const sdr_config* cfg);
size_t  sdr_stream_state_bytes(const sdr_config* cfg, int B);
size_t  sdr_stream_workspace_bytes(const sdr_config* cfg, int B, int64_t C);
/* 3 * num_blocks + 6 kernels per step */
int     sdr_stream_launch_count(const sdr_config* cfg, int B, int64_t C);
/* zero every slot (host_slots_or_null = NULL) or the n slots listed (host array) */
int     sdr_stream_reset(const sdr_config* cfg, void* state, int B, const int32_t* host_slots_or_null, int n,
                         sdr_stream stream);
/* chunk [B, A, C] -> out [B, S*A, C]: the model's output samples c*C - hop .. (c+1)*C - hop - 1 of the c-th step;
 * apply_mixture_consistency: the uniform projection against the mixture delayed by hop (mono models only)      */
/* sdr_stream_reset of the slots b < B whose mask[b] (device memory, uint8) is nonzero: the same bytes, with the slots
 * chosen on the device, so that a captured graph can reset them */
int     sdr_stream_reset_masked(const sdr_config* cfg, void* state, int B, const uint8_t* mask, sdr_stream stream);
int     sdr_stream_step(const sdr_config* cfg, const void* packed, void* state, const float* chunk, float* out,
                        int B, int64_t C, int apply_mixture_consistency, void* ws, size_t ws_bytes, sdr_stream stream);
/* tail [B, S*A, hop]: the pending overlap-add sums; the state is left as it is */
int     sdr_stream_flush(const sdr_config* cfg, void* state, float* tail, int B, int apply_mixture_consistency,
                         sdr_stream stream);
/* The stream stage of one causal U-ConvBlock: the depthwise pyramid of sdr_causal_pyramid over one chunk of F
 * frames per slot, with the last 10 inputs of every level carried in history [B][D][10][C] (zero to start).
 * y, m [C][B*F] (columns slot-major); m is bitwise what sdr_causal_pyramid computes over the concatenated chunks.
 * F % 4 == 0, F % 2^(D-1) == 0 and F <= 4096, else SDR_ERR_UNSUPPORTED.                                      */
int     sdr_causal_stream_stage(const float* y, const float* slope_in, const float* const* w21,
                                const float* const* bias, const float* const* slope, float* history, float* m,
                                int D, int B, int C, int F, sdr_stream stream);

/* mixture_consistency.apply (mixture_consistency.py:14-36).
 * weights_type: 0 = 'uniform', 1 = 'magsq'.  est/out [B,S,T], mix [B,1,T].
 * `scratch` (device, >= B*S doubles) is only used by 'magsq'.               */
int sdr_mixture_consistency(const float* est, const float* mix, float* out,
                            int B, int S, int64_t T, int weights_type,
                            void* scratch, sdr_stream stream);

/* Backward of sdr_mixture_consistency: grad_out [B,S,T] -> grad_est [B,S,T] and, unless NULL, grad_mix [B,1,T].
 * 'uniform' (0) needs neither `mix` nor scratch; 'magsq' (1) reads `mix` and needs
 * sdr_mixture_consistency_backward_scratch_bytes(B, S, T, 1) bytes of 16-byte aligned scratch (0 for 'uniform').
 * Its reductions are fp64 per-chunk partials added in index order: bitwise reproducible, no synchronisation.    */
size_t sdr_mixture_consistency_backward_scratch_bytes(int B, int S, int64_t T, int weights_type);
int sdr_mixture_consistency_backward(const float* est, const float* mix, const float* grad_out, float* grad_est,
                                     float* grad_mix_or_null, int B, int S, int64_t T, int weights_type,
                                     void* scratch, sdr_stream stream);

/* ---- per-stage entry points (stage-level parity tests; same kernels the
 *      forward launches).  "Deferred GlobLN": a producer stores its RAW output
 *      and accumulates per-sample (sum, sum of squares) in fp64 into `stats`
 *      ([samples][2] doubles, zero-initialised by the caller); the consumer
 *      applies gamma*(x-mean)*rstd+beta (+PReLU) while loading.
 *      GlobLN = improved_sudormrf.py:30-47.                                  */

/* description of a deferred normalisation applied to an input while loading */
typedef struct {
    const double* stats;   /* [samples][2] or NULL = no normalisation */
    const float*  gamma;   /* [C] */
    const float*  beta;    /* [C] */
    const float*  prelu;   /* 1 element ([C] when prelu_per_channel), or NULL = no activation */
    double        count;   /* elements per sample the statistics were taken over */
    int32_t       prelu_per_channel;   /* 0: nn.PReLU() (one shared slope); 1: nn.PReLU(C) (sudormrf.py:33,71) */
} sdr_norm_in;

/* nn.Conv1d(A, N, k, stride=k/2, padding=k/2, bias=False) on the zero-padded
 * waveform (improved_sudormrf.py:247-251,286,303-314).
 * wav [B,A,T] -> enc [B,N,L] (L = padded_length/hop), stats over (N,L).      */
int sdr_encoder(const float* wav, const float* weight, float* enc, double* stats,
                int B, int A, int64_t T, int N, int K, int L, sdr_stream stream);

/* The same encoder on the tensor cores: the wgmma GEMM kernel with a "window" operand producer
 * (A[position, tap] = wav[hop*position + tap - pad], built in registers: no im2col in HBM); the
 * weight is converted once to pre-swizzled bf16 hi/lo images (taps zero-padded to 64).  N >= 32. */
size_t sdr_encoder_mma_packed_bytes(int N, int A, int K);
int sdr_encoder_mma_pack(const float* weight, int N, int A, int K, void* packed, sdr_stream stream);
int sdr_encoder_mma(const float* wav, const void* packed_w, float* enc, double* stats,
                    int B, int A, int64_t T, int N, int K, int L, sdr_stream stream);

/* Both encoders with every mode the model forwards use:
 *   enc[b,n,p] = act(sum_{a,j} w[n,a,j] * wav[b,a, hop*p + j - pad] + bias[n]), zero outside [0, T),
 * hop = K/2; pad = hop (improved / groupcomm / original models), 2*hop (the causal model's encoder,
 * causal_improved_sudormrf_v3.py:194); bias NULL = none; relu != 0: act = ReLU (the original model,
 * sudormrf.py:212-218,269), else identity; stats NULL = no statistics, else (sum, sumsq) of the final output.
 * sdr_encoder_mma_ex takes the image of sdr_encoder_mma_pack in place of the weight.                     */
int sdr_encoder_ex(const float* wav, const float* weight, const float* bias_or_null, int relu, int pad,
                   float* enc, double* stats_or_null, int B, int A, int64_t T, int N, int K, int L, sdr_stream stream);
int sdr_encoder_mma_ex(const float* wav, const void* packed_w, const float* bias_or_null, int relu, int pad,
                       float* enc, double* stats_or_null, int B, int A, int64_t T, int N, int K, int L,
                       sdr_stream stream);

/* 1x1 Conv1d as a GEMM: y[b,m,l] = sum_k W[m,k] f(x[b,k,l]) + bias[m]
 * (+ residual[b,m,l]); f = deferred norm/PReLU.  epilogue 0: plain,
 * 1: relu(y) * gate[b, m % gate_channels, l] (mask path, improved_sudormrf.py:296-298).
 * Replaces bottleneck / proj_1x1.conv / res_conv / mask_net.1 (+decoder GEMM). */
int sdr_pointwise(const float* x, const sdr_norm_in* fin, const float* W, const float* bias,
                  const float* residual, const float* gate, int gate_channels,
                  float* y, double* stats_out,
                  int samples, int M, int Kc, int L, int epilogue, sdr_stream stream);

/* Tensor-core (wgmma, bf16x3 split, fp32 accumulate) variant of sdr_pointwise for
 * channel counts that fill a tile: M % 128 == 0 and Kc % 64 == 0.  The weight is
 * first converted to pre-swizzled bf16 hi/lo shared-memory images (bulk-TMA source);
 * sdr_pointwise_mma_packed_bytes returns 0 when the shape is not eligible.           */
size_t sdr_pointwise_mma_packed_bytes(int M, int Kc);
int sdr_pointwise_mma_pack(const float* W, int M, int Kc, void* packed, sdr_stream stream);
int sdr_pointwise_mma(const float* x, const sdr_norm_in* fin, const void* packed_w, const float* bias,
                      const float* residual, const float* gate, int gate_channels,
                      float* y, double* stats_out,
                      int samples, int M, int Kc, int L, int epilogue, sdr_stream stream);

/* depthwise Conv1d(k=5, padding=2, stride 1|2, groups=C) on the deferred-normalised
 * input (improved_sudormrf.py:178-189,206-211).  x [samples,C,Lin] ->
 * y [samples,C,Lout] raw + stats.                                            */
int sdr_depthwise(const float* x, const sdr_norm_in* fin, const float* w5, const float* bias,
                  float* y, double* stats_out,
                  int samples, int C, int Lin, int stride, sdr_stream stream);

/* The whole depthwise pyramid of a U-ConvBlock (improved_sudormrf.py:205-216) in one pass over the projection
 * output y [samples,C,L] (fin: its GlobLN + PReLU).  Levels d >= 1 are affine in their inputs, so the kernel
 * chains RAW stride-2 convolutions without waiting for any statistics: z[0] receives level 0's output, z[d]
 * (d >= 1) the raw chain R_d [samples,C,L>>d]; a second small kernel reproduces every level's GlobLN from row
 * statistics and leaves the coefficients of the merge in `scratch` (sdr_pyramid_scratch_bytes; 0 = shape not
 * eligible: D < 4, L % 16, L >> (D-1) < 6, rows too long for shared memory, or more than 4096 samples -> use
 * sdr_depthwise / sdr_merge; both pyramid entries then return SDR_ERR_UNSUPPORTED).
 * w5[d] [C][5], bias[d] [C]: level d's depthwise conv; gamma[d] / beta[d] [C]: spp_dw[d].norm.
 * stats0: zeroed (sum, sumsq) slot per sample for level 0's output.
 * sdr_merge_pyramid then writes m[c,t] = sum_d GLN_d(z_d)[c, t>>d] (+ its statistics), reading z and scratch. */
size_t sdr_pyramid_scratch_bytes(int samples, int C, int D, int L);
int sdr_depthwise_pyramid(const float* y, const sdr_norm_in* fin, const float* const* w5, const float* const* bias,
                          const float* const* gamma, const float* const* beta, float* const* z, double* stats0,
                          void* scratch, int D, int samples, int C, int L, sdr_stream stream);
int sdr_merge_pyramid(const float* const* z, const void* scratch, int D, float* m, double* stats_out,
                      int samples, int C, int L, sdr_stream stream);
/* The same stage without the levels in HBM (what the forward runs): one pass over y keeps only the row statistics,
 * the solve fills `scratch`, and a second pass over y rebuilds the raw chain and writes the merge m [samples,C,L]
 * (+ its statistics in stats_m, a zeroed slot) from registers.  m is bitwise what sdr_depthwise_pyramid +
 * sdr_merge_pyramid compute.  m may be y itself (the forward merges in place); otherwise it must not overlap y.
 * Same eligibility and scratch as sdr_depthwise_pyramid. */
int sdr_depthwise_pyramid_fused(const float* y, const sdr_norm_in* fin, const float* const* w5, const float* const* bias,
                                const float* const* gamma, const float* const* beta, float* m, double* stats0,
                                double* stats_m, void* scratch, int D, int samples, int C, int L, sdr_stream stream);

/* The depthwise stage of the causal U-ConvBlock (causal_improved_sudormrf_v3.py:106-116) in one pass: PReLU of
 * proj_1x1 on load (slope_in), D levels of [causally masked 21-tap depthwise conv (stride 1, then 2) + bias + PReLU]
 * kept in shared memory, nearest up-sampling and adds, m[c,t] = sum_d o_d[c, t>>d].  No normalisation layers exist
 * in this block, so nothing crosses CTAs.  y, m [samples,C,L]; w21[d] [C][1][21] in the reference's layout (the 10
 * taps the causal mask zeroes, :21-27, are not read); bias[d] [C]; slope_in, slope[d]: one float each.
 * L % 4 == 0 and L % 2^D == 0 (every padded length is), else SDR_ERR_UNSUPPORTED.                              */
int sdr_causal_pyramid(const float* y, const float* slope_in, const float* const* w21, const float* const* bias,
                       const float* const* slope, float* m, int D, int samples, int C, int L, sdr_stream stream);

/* nearest x2 up-sampling + skip adds, closed form
 * m[c,t] = sum_d norm_d(z_d)[c, t>>d] (improved_sudormrf.py:214-216).        */
int sdr_merge(const float* const* z, const sdr_norm_in* fins, int depth,
              float* m, double* stats_out, int samples, int C, int L, sdr_stream stream);

/* TAC (groupcomm_sudormrf_v2.py:356-384) up to (not including) its GlobLN:
 * x [B,G,n,L] -> o [B,G,n,L] raw + stats per (b,g).  params = the 9 TAC
 * tensors before TAC_norm, state_dict order.                                 */
int sdr_tac(const float* x, const float* const* params, float* o, double* stats_out,
            int B, int G, int n, int L, sdr_stream stream);

/* TAC's residual + norm (groupcomm_sudormrf_v2.py:381-383): out = x + GlobLN(o) per sample, with
 * x, o, out [samples,n,L] (samples = B*G) and norm = the statistics of sdr_tac + TAC_norm's gamma / beta.   */
int sdr_tac_apply(const float* x, const float* o, const sdr_norm_in* norm, float* out, int samples, int n, int L,
                  sdr_stream stream);

/* GroupComm proj_1x1 with TAC's residual + norm fused into its operand load:
 *   xt_out = x + GlobLN(pre_add),  y = W xt_out + bias (+ (sum, sumsq) of y into stats_out unless NULL)
 * x, pre_add, xt_out [samples,Kc,L]; y [samples,M,L]; pre_norm as for sdr_tac_apply.  SDR_ERR_UNSUPPORTED
 * when the small-channel kernels cannot take the shape (L % 4, unaligned pointers, Kc > 64 or M > 64): the
 * forward then runs sdr_tac_apply and sdr_pointwise.                                                        */
int sdr_pointwise_preadd(const float* x, const float* pre_add, const sdr_norm_in* pre_norm, float* xt_out,
                         const float* W, const float* bias, float* y, double* stats_out,
                         int samples, int M, int Kc, int L, sdr_stream stream);

/* ConvTranspose1d overlap-add + crop (+ uniform mixture consistency):
 * frames [B, SA*K, L] -> out [B, SA, T] (improved_sudormrf.py:272-279,300-301). */
int sdr_overlap_add(const float* frames, const float* mix_or_null, float* out,
                    int B, int SA, int K, int L, int64_t T, sdr_stream stream);

/* ---- stages that only the original model has (sudormrf.py) ---------------- */

/* Tail of the original UBlock (sudormrf.py:184-186) up to the statistics module_act needs:
 *   x[b,c,l] <- GN_e(e)[b,c,l] + f(x[b,c,l])      in place, (sum, sumsq) of the new x into stats_out
 * e [samples,C,L]: raw conv_1x1_exp.conv output, fe its GroupNorm (stats + weight/bias, no activation);
 * fx: how the block input is read: NULL stats = plain tensor (first block), else module_act of the previous
 * block (GroupNorm + per-channel PReLU) applied on load.                                                   */
int sdr_residual_norm(const float* e, const sdr_norm_in* fe, float* x, const sdr_norm_in* fx, double* stats_out,
                      int samples, int C, int L, sdr_stream stream);

/* Masks of the original model (sudormrf.py:285-289): logits [B,S,N,L] (the (N+1)x1 Conv2d output) ->
 * softmax over the S sources (sigmoid when S == 1) times the encoder output enc [B,N,L]; in place is allowed. */
int sdr_softmax_gate(const float* logits, const float* enc, float* out, int B, int S, int N, int L, sdr_stream stream);

/* ---- the steps either side of the forward (SURVEY.md 8f rows 1-2) -------- */

/* Per-row (mean, unbiased std) of a waveform batch: wav [rows, T] ->
 * mean_std [rows][2] fp32 (README.md:101-102: `x.mean(-1)`, `x.std(-1)`).
 * scratch: rows * 2 doubles of device memory.                                */
int sdr_utterance_stats(const float* wav, float* mean_std, int rows, int64_t T,
                        void* scratch, sdr_stream stream);

/* The README inference recipe as ONE call (README.md:100-114):
 *   m, s = wav.mean(-1), wav.std(-1);  x = (wav - m) / (s + 1e-9)
 *   est  = model(x.unsqueeze(1)) * s + m
 *   [est = mixture_consistency.apply(est, x.unsqueeze(1))]      (uniform)
 * wav [B,1,T] -> out [B,S,T].  Mono models only (in_audio_channels == 1).
 * Workspace: sdr_separate_workspace_bytes (forward workspace + the
 * normalised copy of the batch).                                             */
size_t sdr_separate_workspace_bytes(const sdr_config* cfg, int B, int64_t T);
int sdr_separate(const sdr_config* cfg, const void* packed, const float* wav, float* out,
                 int B, int64_t T, int apply_mixture_consistency,
                 void* workspace, size_t workspace_bytes, sdr_stream stream);

/* The same recipe for a RAGGED batch: B utterances of different lengths that
 * share one padded length T (a multiple of hop * 2^depth, sdr_padded_length),
 * stored zero-padded as wav [B,1,T]; lengths[b] (device, int64) = true length.
 * Statistics use the first lengths[b] samples only, the padding stays zero,
 * i.e. every row is computed exactly as the reference computes that utterance
 * alone (improved_sudormrf.py:303-318 pads it to the same T).  rescale = 0
 * skips `est * std + mean` (utils/simple_whamr_evaluation.py:141-148 evaluates
 * the normalised estimates).  out [B,S,T]: row b is valid up to lengths[b].   */
int sdr_separate_ragged(const sdr_config* cfg, const void* packed, const float* wav,
                        const int64_t* lengths, float* out, int B, int64_t T,
                        int apply_mixture_consistency, int rescale,
                        void* workspace, size_t workspace_bytes, sdr_stream stream);

/* Permutation-invariant SI-SDR of a batch (dnn/losses/sisdr.py:66-194,
 * PermInvariantSISDR.forward with return_individual_results=True,
 * backward_loss=False): est, target [B,S,T], mixture [B,1,T] (needed only for
 * improvement != 0) -> best[b] = max over permutations of the source-mean
 * SI-SNR (minus the batch-mean SI-SNR of the mixture when improvement != 0),
 * perm_index[b] = index of that permutation in itertools.permutations(range(S))
 * order.  1 <= S <= 4.  eps as in the reference's forward (default 1e-9).     */
/* Pairwise negative SNR / SI-SDR / SD-SDR of a batch (dnn/losses/sisdr.py:372-457, PairwiseNegSDR.forward):
 * out[b, i, j] = -sdr(estimate i, target j), [B, S, S] fp32; sdr_type 0 = "snr", 1 = "sisdr", 2 = "sdsdr".
 * One fp64 Gram pass + a finalize kernel; scratch: sdr_pit_sisdr_scratch_bytes(B, S).  1 <= S <= 4.        */
int sdr_pairwise_neg_sdr(const float* est, const float* target, float* out, int B, int S, int64_t T, int sdr_type,
                         int zero_mean, int take_log, void* scratch, sdr_stream stream);

/* The same [B, S, S] output for training (PairwiseNegSDR under autograd, the loss of run_improved_sudormrf.py:64-66
 * through PITLossWrapper): also writes into `coef` (sdr_pairwise_neg_sdr_coef_bytes(B, S), 8-byte aligned) the fp64
 * coefficients of d out / d est that sdr_pairwise_neg_sdr_backward reads.  Scratch:
 * sdr_pairwise_neg_sdr_train_scratch_bytes(B, S, T), per-chunk fp64 Gram partials added in index order.  1 <= S <= 4.
 * sdr_pairwise_neg_sdr_backward: grad_out [B,S,S] = dL/d out -> grad_est [B,S,T].  No call synchronises; a forward
 * and a backward are bitwise reproducible.                                                                          */
size_t sdr_pairwise_neg_sdr_train_scratch_bytes(int B, int S, int64_t T);
size_t sdr_pairwise_neg_sdr_coef_bytes(int B, int S);
int sdr_pairwise_neg_sdr_train(const float* est, const float* target, float* out, void* coef, int B, int S,
                               int64_t T, int sdr_type, int zero_mean, int take_log, void* scratch, sdr_stream stream);
int sdr_pairwise_neg_sdr_backward(const float* est, const float* target, const void* coef, const float* grad_out,
                                  float* grad_est, int B, int S, int64_t T, sdr_stream stream);

size_t sdr_pit_sisdr_scratch_bytes(int B, int S);
int sdr_pit_sisdr(const float* est, const float* target, const float* mixture_or_null,
                  float* best, int32_t* perm_index, int B, int S, int64_t T,
                  int zero_mean, int improvement, double eps,
                  void* scratch, sdr_stream stream);

/* StabilizedPermInvSISDRMetric.forward (dnn/losses/sisdr.py:460-591; backward_loss=False,
 * return_individual_results=True), the validation metric of run_fuss_separation.py:111-131: n_est estimated sources
 * scored against n_act <= n_est actual ones with the stabilised SI-SNR
 *     rho^2 = <e,t>^2 / (<e,e><t,t> + eps),  10 log10((rho^2 + eps) / (1 - rho^2 + eps)),
 * best[b] = max over itertools.permutations(range(n_est), r=n_act) of the source mean (minus, for improvement != 0,
 * the batch mean of the same figure for the mixture = sum of the targets), perm_index[b] = index of that assignment.
 * est [B, est_rows, T], target [B, n_act, T]; est_rows == n_est, or est_rows > n_est == 1: single_source mode, the
 * rows are summed first (:576-577).  1 <= n_act <= n_est <= 4.  eps as in the reference's forward (1e-9).            */
size_t sdr_stabilized_sisdr_scratch_bytes(int B, int n_est, int n_act);
int sdr_stabilized_sisdr(const float* est, const float* target, float* best, int32_t* perm_index,
                         int B, int est_rows, int n_est, int n_act, int64_t T,
                         int zero_mean, int improvement, double eps, void* scratch, sdr_stream stream);

/* PermInvariantSNRwithZeroRefs.forward (dnn/losses/snr.py:13-142; backward_loss=False, return_individual_results=True),
 * the training loss of run_fuss_separation.py:257-259: est, target [B,S,T] (already cropped to one length) ->
 * value[b] = max over itertools.permutations(range(S)) of num_active * sum_k 10 a_k log10(nom_k / den_k + eps),
 * perm_index[b] = index of that permutation (torch.max's rule: the first NaN, else the first maximum).  Also writes
 * into `coef` (sdr_snr_zero_refs_coef_bytes(B, S), 8-byte aligned) what sdr_snr_zero_refs_backward reads.  Scratch:
 * sdr_snr_zero_refs_scratch_bytes(B, S, T), per-chunk fp64 Gram partials added in index order.  1 <= S <= 4.
 * sdr_snr_zero_refs_backward: grad_value [B] = dL/d value -> grad_est [B,S,T_grad] (rows T_grad >= T apart, zero
 * past T).  No call synchronises; a forward and a backward are bitwise reproducible.                                */
size_t sdr_snr_zero_refs_scratch_bytes(int B, int S, int64_t T);
size_t sdr_snr_zero_refs_coef_bytes(int B, int S);
int sdr_snr_zero_refs(const float* est, const float* target, float* value, int32_t* perm_index, void* coef,
                      int B, int S, int64_t T, int zero_mean, double inactivity_threshold, double eps,
                      void* scratch, sdr_stream stream);
int sdr_snr_zero_refs_backward(const float* est, const float* target, const void* coef, const float* grad_value,
                               float* grad_est, int B, int S, int64_t T, int64_t T_grad, sdr_stream stream);

/* BSS-eval v3 source criteria (mir_eval.separation.bss_eval_sources, the sdr / sir / sar of asteroid's get_metrics):
 * reference, estimate [B,S,T] -> sdr, sir, sar [B,S] fp64 in dB and perm [B,S] (perm[b][j] = the estimate scored
 * against reference j).  Per item, with F-tap distortion filters (mir_eval: 512), in R^(T+F-1), P_j e the projection
 * of e onto the F delays of reference j and P_all e onto the delays of every reference:
 *     SDR = 10 log10(|P_j e|^2 / |e - P_j e|^2),  SIR = 10 log10(|P_j e|^2 / |P_all e - P_j e|^2),
 *     SAR = 10 log10(|P_all e|^2 / |e - P_all e|^2)     (a zero denominator: +inf).
 * compute_permutation != 0 scores every (estimate, reference) pair and takes the assignment with the largest mean SIR
 * (the first in itertools.permutations order); else estimate j is scored against reference j.  An item with an
 * all-zero reference or estimate row gets NaN in every output and perm -1.  perm_or_null may be NULL.  The outputs
 * are bitwise reproducible; no call synchronises.  1 <= S <= 4, 1 <= F <= 512, T >= (S - 1) F + 1 (no more delayed
 * references than dimensions: for S = 1 any T >= 1); scratch:
 * sdr_bss_eval_scratch_bytes(B, S, T, F) (0: unsupported arguments), 8-byte aligned.
 * sdr_bss_eval_mixture also scores mixture [B,1,T] as the estimate of every reference into mix_sdr, mix_sir,
 * mix_sar [B,S] (NaN where the mixture or a reference is silent), from the same reference correlations and solves. */
size_t sdr_bss_eval_scratch_bytes(int B, int S, int64_t T, int F);
int sdr_bss_eval(const float* reference, const float* estimate, double* sdr, double* sir, double* sar,
                 int32_t* perm_or_null, int B, int S, int64_t T, int F, int compute_permutation, void* scratch,
                 sdr_stream stream);
int sdr_bss_eval_mixture(const float* reference, const float* estimate, const float* mixture, double* sdr,
                         double* sir, double* sar, int32_t* perm_or_null, double* mix_sdr, double* mix_sir,
                         double* mix_sar, int B, int S, int64_t T, int F, int compute_permutation, void* scratch,
                         sdr_stream stream);

/* Framewise BSS-eval (mir_eval.separation.bss_eval_sources_framewise): reference, estimate [B,S,T] scored in windows
 * of W samples every H samples, each window exactly as sdr_bss_eval scores that slice (its own permutation search)
 * -> sdr, sir, sar [B,nwin,S] fp64 and perm [B,nwin,S], nwin = floor((T - W + H) / H), window k covering
 * [k H, k H + W).  When that count is below 2 (T < W + H), nwin = 1 and the column is the whole item (mir_eval's
 * fallback).  The windows are read in place: nothing is copied, and the scratch,
 * sdr_bss_eval_framewise_scratch_bytes(B, S, T, W, H, F) (0: unsupported arguments, 8-byte aligned), holds at most
 * 128 windows whatever T is; more windows run in successive launches on the stream.  A window with an all-zero
 * reference or estimate row, or one holding a NaN or an infinity, gets NaN and perm -1; windows that do not contain
 * it are unaffected.  lengths_or_null (device [B], 8-byte aligned) gives recording b its own length n_b, read on the
 * device: its window count follows from n_b as above (with the same fallback), its columns past that count are NaN
 * with perm -1, and nothing past n_b is read.  A length outside [1, T], and a fallback recording shorter than
 * (S - 1) F + 1, give NaN and perm -1 in every column.  1 <= S <= 4, 1 <= F <= 512, and W >= (S - 1) F + 1
 * (T >= (S - 1) F + 1 when the fallback applies).  mixture_or_null [B,1,T] is also scored as the estimate of every
 * reference into mix_sdr, mix_sir, mix_sar [B,nwin,S], as sdr_bss_eval_mixture scores it.  perm may be NULL.
 * Bitwise reproducible; no call synchronises.                                                                        */
size_t sdr_bss_eval_framewise_scratch_bytes(int B, int S, int64_t T, int64_t W, int64_t H, int F);
int sdr_bss_eval_framewise(const float* reference, const float* estimate, const float* mixture_or_null,
                           const int64_t* lengths_or_null, double* sdr, double* sir, double* sar,
                           int32_t* perm_or_null, double* mix_sdr, double* mix_sir, double* mix_sar, int B, int S,
                           int64_t T, int64_t W, int64_t H, int F, int compute_permutation, void* scratch,
                           sdr_stream stream);

/* BSS-eval of source images (mir_eval.separation.bss_eval_images), the multichannel criteria: reference, estimate
 * [B,S,C,T] (S images of C channel rows, each row contiguous in time) -> sdr, isr, sir, sar [B,S] fp64 in dB and perm
 * [B,S].  Per item, in R^(T+F-1) per channel, P_j e_i projects each channel of e_i onto the F delays of all C channels
 * of s_j and P_all e_i onto all S C F delayed reference channels; energies sum over channels:
 *     SDR = 10 log10(|s_j|^2 / |e_i - s_j|^2),             ISR = 10 log10(|s_j|^2 / |P_j e_i - s_j|^2),
 *     SIR = 10 log10(|P_j e_i|^2 / |P_all e_i - P_j e_i|^2),  SAR = 10 log10(|P_all e_i|^2 / |e_i - P_all e_i|^2)
 * (a zero denominator: +inf).  compute_permutation and perm as sdr_bss_eval (the largest mean SIR).  For C = 1, SIR
 * and SAR are sdr_bss_eval's.  An all-zero channel of a non-silent image is dropped from its systems (the projection
 * onto the other channels); an item with an all-zero reference or estimate image, or one holding a NaN or an
 * infinity, gets NaN in every output and perm -1.  1 <= S C <= 4, 1 <= F <= 512, T >= (S C - 1) F + 1; scratch:
 * sdr_bss_eval_images_scratch_bytes(B, S, C, T, F) (0: unsupported arguments), 8-byte aligned.  perm_or_null may be
 * NULL.  Bitwise reproducible; no call synchronises.
 * sdr_bss_eval_images_framewise scores [B,S,C,T] in windows as sdr_bss_eval_framewise does (the same window count,
 * fallback, lengths_or_null and NaN columns; at most 128 windows per scratch) -> sdr, isr, sir, sar, perm
 * [B,nwin,S], each column exactly sdr_bss_eval_images of its window.  W >= (S C - 1) F + 1 (T when the fallback
 * applies). */
size_t sdr_bss_eval_images_scratch_bytes(int B, int S, int C, int64_t T, int F);
int sdr_bss_eval_images(const float* reference, const float* estimate, double* sdr, double* isr, double* sir,
                        double* sar, int32_t* perm_or_null, int B, int S, int C, int64_t T, int F,
                        int compute_permutation, void* scratch, sdr_stream stream);
size_t sdr_bss_eval_images_framewise_scratch_bytes(int B, int S, int C, int64_t T, int64_t W, int64_t H, int F);
int sdr_bss_eval_images_framewise(const float* reference, const float* estimate, const int64_t* lengths_or_null,
                                  double* sdr, double* isr, double* sir, double* sar, int32_t* perm_or_null, int B,
                                  int S, int C, int64_t T, int64_t W, int64_t H, int F, int compute_permutation,
                                  void* scratch, sdr_stream stream);
/* BSS-eval v4 (museval.evaluate(..., mode='v4'), the SiSEC 2018 / MUSDB18 criteria): reference, estimate [B,S,C,T]
 * as sdr_bss_eval_images -> sdr, isr, sir, sar, perm [B,nwin,S], nwin = (T - W) / H + 1.  The distortion filters are
 * solved once per recording from the correlations of its whole length (those sdr_bss_eval_images computes on it);
 * window k, [k H, k H + W), then filters its own reference slice (zero outside the window) with them, and its
 * criteria are sdr_bss_eval_images' formulas on the window's slices and energies.  No whole-recording fallback.  A
 * window with an all-zero reference or estimate image is NaN with perm -1; a NaN or an infinity anywhere in a
 * recording, or whole-track filters that are no projection, make every window of that recording NaN with perm -1.
 * lengths_or_null [B] (read on the device): recording b is its first lengths[b] samples, with its own filters and
 * (n - W) / H + 1 windows; columns past them, and every column of a recording with n < W, n < (S C - 1) F + 1 or n
 * outside [1, T], are NaN with perm -1.  1 <= S C <= 4, 1 <= F <= 512, T >= W and T >= (S C - 1) F + 1; scratch:
 * sdr_bss_eval_v4_scratch_bytes (0: unsupported arguments), 8-byte aligned, bounded in T once T passes 512 chunks of
 * 8192 samples per recording.  Bitwise reproducible, a recording's columns the same in any batch; no call
 * synchronises. */
size_t sdr_bss_eval_v4_scratch_bytes(int B, int S, int C, int64_t T, int64_t W, int64_t H, int F);
int sdr_bss_eval_v4(const float* reference, const float* estimate, const int64_t* lengths_or_null, double* sdr,
                    double* isr, double* sir, double* sar, int32_t* perm_or_null, int B, int S, int C, int64_t T,
                    int64_t W, int64_t H, int F, int compute_permutation, void* scratch, sdr_stream stream);

/* STOI (pystoi 0.3.3's stoi(x, y, fs_sig, extended=False), the stoi of asteroid's get_metrics): reference and
 * estimate [B,S,T], mixture_or_null [B,T] -> stoi [B,S] fp64 (estimate j scored against reference j) and, with the
 * mixture, mix_stoi [B,S] (the mixture scored against every reference).  Rows are resampled from fs to 10 kHz as
 * Octave's resample does (scipy resample_poly alignment), frames more than 40 dB below the reference's loudest are
 * dropped from both signals, and the 30-frame segment correlations of the 15 third-octave band magnitudes are
 * averaged; fewer than 30 spectral frames (including rows of at most 256 samples after resampling) give 1e-5.
 * lengths_or_null (device [B]) scores item b over its first lengths[b] samples and reads nothing past them; a length
 * outside [1, T] gives NaN in the item's outputs.  A NaN or infinity in reference j or estimate j gives stoi[b][j]
 * NaN, in reference j or the mixture mix_stoi[b][j] NaN; nothing else changes.  Any integer fs >= 1000 whose reduced
 * ratio 10000 / fs has max(p, q) <= 441 (44.1 and 22.05 kHz included).  fp64 after the inputs, no atomics: bitwise
 * reproducible; no call synchronises or allocates.  Scratch: sdr_stoi_scratch_bytes(B, S, T, fs) (0: unsupported
 * arguments), 8-byte aligned. */
size_t sdr_stoi_scratch_bytes(int B, int S, int64_t T, int fs);
int sdr_stoi(const float* reference, const float* estimate, const float* mixture_or_null,
             const int64_t* lengths_or_null, double* stoi, double* mix_stoi_or_null, int B, int S, int64_t T, int fs,
             void* scratch, sdr_stream stream);

/* ---- polyphase resampling (DESIGN.md section 7g) ---------------------------
 * scipy.signal.resample_poly(x, up, down) with its defaults (window=('kaiser', 5.0), padtype='constant') on every row
 * of x [rows][T] fp32 -> out [rows][ceil(T p / q)] fp32, up / down reduced to p / q by their gcd.  The filter is
 * firwin(2L + 1, 1 / max(p, q), window=('kaiser', 5.0)) * p with L = 10 max(p, q), designed on the device into
 * scratch; out[i] = sum_t h[i q + L - t p] x[t] over the taps inside [0, 2L], summed in fp64 in ascending t and
 * rounded once, so every row is bitwise independent of the others and of rows.  A NaN or infinity in x[t] makes
 * exactly the outputs whose support holds t non-finite.  p == q copies x.  up, down >= 1 and max(p, q) <= 4096 (else
 * 0 / SDR_ERR_UNSUPPORTED; up or down < 1: SDR_ERR_BAD_ARGUMENT), rows >= 1, 1 <= T <= 2^40.  Scratch:
 * sdr_resample_poly_scratch_bytes(up, down) = 8 (20 max(p, q) + 1), 8-byte aligned; a null, misaligned
 * (SDR_ERR_BAD_ARGUMENT) or smaller (SDR_ERR_WORKSPACE) scratch is refused before anything is enqueued.  x and out
 * must not overlap.  No call synchronises or allocates: a call can be captured in a CUDA graph. */
size_t sdr_resample_poly_scratch_bytes(int up, int down);
int    sdr_resample_poly(const float* x, float* out, int64_t rows, int64_t T, int up, int down, void* scratch,
                         size_t scratch_bytes, sdr_stream stream);

/* ---- streaming resampler (DESIGN.md section 7h) ----------------------------
 * resample_poly chunk by chunk for B independent slots of `rows` rows.  With up / down reduced to p / q (p != q,
 * max(p, q) <= 4096) and L = 10 max(p, q), per slot let s be `lead` zeros followed by everything the slot received
 * since its reset and r = resample_poly(s) as sdr_resample_poly computes it.  Step j since the reset takes chunk
 * [B][rows][C] (C a positive multiple of q) and writes out [B][rows][C p / q] = samples [j C p / q - delay,
 * (j + 1) C p / q - delay) of r, zeros below index 0.  The flush takes tail_or_null [B][rows][tail_len] (any
 * tail_len >= 0) and writes out [B][rows][ceil((lead + tail_len) p / q) + delay] = the rest of r with s extended by
 * the tail, up to ceil(len(s) p / q); it leaves the state as it was.  Every value is bitwise sdr_resample_poly's on
 * the concatenation: the same filter, each output summed in fp64 by fma in ascending input index over the same
 * support and rounded once.  delay >= floor((L - lead p) / q) (the smallest delay at which every output of a step has
 * its whole support received), 0 <= lead <= 2^40, 1 <= B <= 65535, rows >= 1.  zero_slots_or_null (device, uint8
 * [B]): the chunk or tail of a slot whose byte is nonzero is read as zeros.
 * State: sdr_resample_stream_state_bytes(...), 256-byte aligned: the filter [2L + 1] fp64, the step counters [B]
 * int64 and two histories [2][B][rows][Hs] fp32, Hs = lead + floor((delay q + L) / p) + 1, each region on a 256-byte
 * boundary (0 bytes for arguments the entries refuse).  sdr_resample_stream_reset with host_slots_or_null = NULL
 * designs the filter and zeroes every slot; with n slots listed in host memory it zeroes those slots' counters and
 * histories.  A step is two launches (the outputs and the next history, then the counters), the flush one.  Every
 * entry refuses a null (SDR_ERR_BAD_ARGUMENT), small (SDR_ERR_WORKSPACE) or misaligned (SDR_ERR_BAD_ARGUMENT) state
 * and arguments out of range (SDR_ERR_BAD_ARGUMENT; p == q or max(p, q) > 4096: SDR_ERR_UNSUPPORTED) before anything
 * is enqueued.  No atomics and no synchronisation: a step with fixed buffers can be captured in a CUDA graph. */
size_t sdr_resample_stream_state_bytes(int B, int rows, int64_t C, int up, int down, int64_t delay, int64_t lead);
int    sdr_resample_stream_reset(void* state, size_t state_bytes, int B, int rows, int64_t C, int up, int down,
                                 int64_t delay, int64_t lead, const int32_t* host_slots_or_null, int n,
                                 sdr_stream stream);
int    sdr_resample_stream_step(void* state, size_t state_bytes, const float* chunk, const uint8_t* zero_slots_or_null,
                                float* out, int B, int rows, int64_t C, int up, int down, int64_t delay, int64_t lead,
                                sdr_stream stream);
int    sdr_resample_stream_flush(const void* state, size_t state_bytes, const float* tail_or_null, int64_t tail_len,
                                 const uint8_t* zero_slots_or_null, float* out, int B, int rows, int64_t C, int up,
                                 int down, int64_t delay, int64_t lead, sdr_stream stream);

/* ---- windowed separation of long recordings (DESIGN.md section 7e) ---------
 * A recording of T samples is cut into K = sdr_window_count(T, W, H) windows (1 when T <= W, else
 * 1 + ceil((T - W) / H)); window k covers samples [k H, k H + W), zeros at T and beyond.  W/2 <= H < W and
 * 2 <= W <= 2^24; sdr_window_count returns 0 for anything else.  Windows are processed in batches k0 .. k0+M-1 in
 * increasing k0, without gaps:
 *   sdr_window_gather copies them out of mixture [B][A][T] into batch [B][M][A][W];
 *   the caller separates the batch ([B M, A, W] through sdr_forward or sdr_separate) into estimates
 *   [B][M][S A][W];
 *   sdr_window_merge aligns and overlap-adds them.  For each window k >= 1 of the batch it takes
 *   C_k[i][j] = sum_a sum_t (p_ia - mean p_ia)(c_ja - mean c_ja) in fp64 over the overlap [k H, (k-1) H + W) below T
 *   (p: window k-1's source i, c: window k's source j, rows s A + a), and rho_k, the first maximum of
 *   sum_i C_k[i][rho(i)] over the permutations in itertools order (the identity when C_k is not finite).  With
 *   pi_0 = id and pi_k(s) = rho_k(pi_{k-1}(s)), output source s of window k is its raw source pi_k(s).  It writes out
 *   [B][S A][T] over [k0 H, (k0 + M) H), or up to T in the last batch: a sample in one window takes that window's
 *   value, sample k H + j of overlap k takes (1 - r) prev + r cur in fp32 with r = (j + 1) / (W - H + 1).
 *   perm_or_null [B][K][S] receives pi_k of the batch's windows.
 * carry (sdr_window_carry_bytes(B, S, A, W), 256-byte aligned) holds pi and the raw estimate of the batch's last
 * window for the next batch: ignored when k0 = 0, else it must hold what the merge of the previous batch left.
 * Scratch: sdr_window_merge_scratch_bytes(B, S, M), 8-byte aligned.  1 <= S <= 4 (else 0 / SDR_ERR_UNSUPPORTED).
 * A NaN or infinity in one recording changes no other recording's output.  No atomics, fixed-order reductions and
 * no synchronisation: given the same estimates the output is bitwise independent of the batch sizes M. */
int64_t sdr_window_count(int64_t T, int64_t W, int64_t H);
size_t  sdr_window_carry_bytes(int B, int S, int A, int64_t W);
size_t  sdr_window_merge_scratch_bytes(int B, int S, int M);
int     sdr_window_gather(const float* mixture, float* batch, int B, int A, int64_t T, int64_t W, int64_t H,
                          int64_t k0, int M, sdr_stream stream);
int     sdr_window_merge(const float* estimates, void* carry, int32_t* perm_or_null, float* out, int B, int S, int A,
                         int64_t T, int64_t W, int64_t H, int64_t k0, int M, void* scratch, sdr_stream stream);

/* ---- a corpus of recordings of different lengths in shared window batches (DESIGN.md section 7i) ----
 * R recordings, each longer than W, laid out back to back: recording r's mixture [A][T_r] starts at element A off_r of
 * the flat mixture and its output [S A][T_r] at element S A off_r of the flat output.  desc (device memory, int64,
 * 8-byte aligned) is [R][3]: (off_r, T_r, g_r), g_r = the sum of K_s = sdr_window_count(T_s, W, H) over s < r, the
 * first global window of recording r.  Global window g = g_r + k is window k of recording r.  Batches are the global
 * windows g0 .. g0+M-1, in increasing g0 without gaps, g0 + M at most the corpus's window count:
 *   sdr_window_gather_ragged copies them into batch [M][A][W], zeros past each T_r;
 *   the caller separates the batch into estimates [M][S A][W];
 *   sdr_window_merge_ragged aligns and overlap-adds each window exactly as sdr_window_merge does for its recording
 *   alone with B = 1 (pi restarts at the identity at every recording's window 0): window k < K_r - 1 writes samples
 *   [k H, (k + 1) H) of its recording, the last one [k H, T_r).  perm_or_null [G][S] (G the corpus's window count)
 *   receives pi of global window g in row g.
 * carry (sdr_window_ragged_carry_bytes(S, A, W) = sdr_window_carry_bytes(1, S, A, W), 256-byte aligned) holds the
 * batch's last window for the next batch, read only when that batch's first window is not its recording's window 0.
 * Scratch: sdr_window_ragged_scratch_bytes(S, M), 8-byte aligned.  1 <= S <= 4 (else 0 / SDR_ERR_UNSUPPORTED).
 * Given the same estimates, the output is bitwise independent of M and bitwise sdr_window_merge's on each recording
 * alone. */
size_t  sdr_window_ragged_carry_bytes(int S, int A, int64_t W);
size_t  sdr_window_ragged_scratch_bytes(int S, int M);
int     sdr_window_gather_ragged(const float* mixture, const int64_t* desc, int R, int A, int64_t W, int64_t H,
                                 int64_t g0, int M, float* batch, sdr_stream stream);
int     sdr_window_merge_ragged(const float* estimates, const int64_t* desc, int R, void* carry, int32_t* perm_or_null,
                                float* out, int S, int A, int64_t W, int64_t H, int64_t g0, int M, void* scratch,
                                sdr_stream stream);

/* ---- windowed stream (DESIGN.md section 7f) --------------------------------
 * separate_long's windows, taken step by step for B independent slots.  With q = C / H (C a positive multiple of
 * H) and n = j C the samples a slot has received since its reset, a step's output [B][S A][C] is samples
 * [n - H, n + C - H) of the windowed separation of the slot's input up to n + C (zeros below 0), and the flush's
 * [B][S A][H] is samples [n - H, n) of the separation up to n.  Per step:
 *   sdr_window_stream_gather copies windows c-1 .. c+q-2 of each slot (c = n / H, the slot's window counter; the
 *   window below 0 of a slot's first step is all zeros) out of its history and chunk [B][A][C] into batch
 *   [B][q][A][W], and makes the chunk's last H samples the history;
 *   the caller separates the batch ([B q, A, W] through sdr_forward or sdr_separate) into estimates [B][q][S A][W];
 *   sdr_window_stream_merge aligns, scans and overlap-adds them as sdr_window_merge does, with each slot's own window
 *   origin, into out [B][S A][C], keeps the carry and advances the counters by q.
 * Flush: sdr_window_stream_gather with chunk_or_null = NULL and C = 0 writes the window that starts at n - H, the
 * history followed by zeros, into batch [B][A][W]; the caller separates it (needed when W < 2 H) and, as `single`
 * [B][S A][H], the history alone (the whole recording of a slot with n = H); sdr_window_stream_flush picks per slot
 * on the device: zeros (n = 0), single (n = H), else the carry and, when W < 2 H, the flush window.  Neither the
 * flush gather nor the flush changes the state.
 * State: sdr_window_stream_state_bytes(B, S, A, W, H), 256-byte aligned: the carry of sdr_window_carry_bytes, the
 * history [B][A][H] fp32 and the counters [B] int64, each starting on a 256-byte boundary.  sdr_window_stream_reset zeroes it (all
 * slots, or the n listed in host memory) before a slot's first step.  Scratch: sdr_window_stream_merge_scratch_bytes
 * (B, S, C, H) and sdr_window_stream_flush_scratch_bytes(B, S), 8-byte aligned.  1 <= S <= 4, W/2 <= H < W,
 * W <= 2^24 (else 0 / SDR_ERR_UNSUPPORTED for S, SDR_ERR_BAD_ARGUMENT otherwise).  sdr_window_stream_launch_count is
 * the number of kernels a step's gather and merge launch.  No atomics, fixed-order reductions and no
 * synchronisation: a step can be captured in a CUDA graph, and given the same window estimates its output is
 * bitwise sdr_window_merge's. */
size_t sdr_window_stream_state_bytes(int B, int S, int A, int64_t W, int64_t H);
int    sdr_window_stream_reset(void* state, int B, int S, int A, int64_t W, int64_t H,
                               const int32_t* host_slots_or_null, int n, sdr_stream stream);
/* sdr_window_stream_reset of the slots b < B whose mask[b] (device memory, uint8) is nonzero, chosen on the device */
int    sdr_window_stream_reset_masked(void* state, int B, int S, int A, int64_t W, int64_t H, const uint8_t* mask,
                                      sdr_stream stream);
int    sdr_window_stream_gather(void* state, const float* chunk_or_null, float* batch, int B, int S, int A, int64_t C,
                                int64_t W, int64_t H, sdr_stream stream);
size_t sdr_window_stream_merge_scratch_bytes(int B, int S, int64_t C, int64_t H);
int    sdr_window_stream_merge(const float* estimates, void* state, float* out, int B, int S, int A, int64_t C,
                               int64_t W, int64_t H, void* scratch, sdr_stream stream);
size_t sdr_window_stream_flush_scratch_bytes(int B, int S);
int    sdr_window_stream_flush(const float* single, const float* estimates_or_null, const void* state, float* out,
                               int B, int S, int A, int64_t W, int64_t H, void* scratch, sdr_stream stream);
int    sdr_window_stream_launch_count(int B, int S, int A, int64_t C, int64_t W, int64_t H);

/* ---- training of the improved model (variant 0) ---------------------------
 * sdr_forward_train runs sdr_forward's kernels (same plan, pyramid choice and GEMMs, no mixture consistency) and
 * also copies into `saved` what the backward recomputes from: the statistics slots, the raw encoder output and every
 * U-ConvBlock input x_0..x_U, each segment 256-byte aligned (4 B L ((U+1) Co + N) bytes plus the statistics).
 * sdr_backward takes dL/d(estimates) [B, S, T] and WRITES (never accumulates) the gradient of every parameter into
 * grad_params: flat fp32, state_dict order, sdr_param_numel(i) floats each, no padding.  Every gradient reduction
 * runs in a fixed order (no atomics), so a backward is bitwise reproducible.  The gradient with respect to the
 * mixture is not computed.  Neither call synchronises or allocates; `saved` and the workspaces are 256-byte aligned.
 * Any other variant: 0 bytes / SDR_ERR_UNSUPPORTED.                                                                  */
size_t sdr_train_saved_bytes(const sdr_config* cfg, int B, int64_t T);
size_t sdr_backward_workspace_bytes(const sdr_config* cfg, int B, int64_t T);
int    sdr_forward_train(const sdr_config* cfg, const void* packed, const float* mixture, float* out, int B, int64_t T,
                         void* saved, size_t saved_bytes, void* ws, size_t ws_bytes, sdr_stream stream);
int    sdr_backward(const sdr_config* cfg, const void* packed, const float* mixture, const void* saved,
                    const float* grad_out, float* grad_params, int B, int64_t T, void* ws, size_t ws_bytes,
                    sdr_stream stream);
/* kernels one sdr_backward enqueues (memsets not counted): 22 + U (14 + 5 D + [D > 1]) */
int    sdr_backward_launch_count(const sdr_config* cfg, int B, int64_t T);

/* stage entries of the backward kernels (activations [samples][channels][L]) */
/* dW[m][k] = sum_{b,t} dy[b][m][t] f(x[b][k][t]) (f: the deferred GlobLN / PReLU of `fin`, NULL = identity),
 * db[m] = sum dy; per-CTA fp32 partials over <= 512 positions in `scratch`, summed in fp64 in order */
size_t sdr_pointwise_wgrad_scratch_bytes(int samples, int M, int Kc, int L);
int    sdr_pointwise_wgrad(const float* dy, const float* x, const sdr_norm_in* fin, float* dw, float* db_or_null,
                           void* scratch, int samples, int M, int Kc, int L, sdr_stream stream);
/* backward of p = PReLU(GlobLN(x)) (fin->stats set) or p = PReLU(x) (fin->stats NULL): dx (or dx += when
 * accumulate), dgamma / dbeta [C], dslope [1] (each may be NULL); one shared slope only */
size_t sdr_norm_act_backward_scratch_bytes(int samples, int C);
int    sdr_norm_act_backward(const float* x, const sdr_norm_in* fin, const float* dp, float* dx, int accumulate,
                             float* dgamma, float* dbeta, float* dslope, void* scratch, int samples, int C, int L,
                             sdr_stream stream);
/* backward of z = dw5(f(x)) (padding 2, stride 1 or 2, Lin even for stride 2): dx[tau] = (dw^T dz)[tau] +
 * sum_{i < pool_factor} pool[pool_factor tau + i] (dz or pool may be NULL), dw5 [C][5] and dbias [C] */
size_t sdr_depthwise_backward_scratch_bytes(int samples, int C);
int    sdr_depthwise_backward(const float* dz, const float* x, const sdr_norm_in* fin, const float* w5,
                              const float* pool_or_null, int pool_factor, float* dx, float* dw5, float* dbias,
                              void* scratch, int samples, int C, int Lin, int stride, sdr_stream stream);
/* masked = relu(mlog) * enc: dmasked [B][S*N][L] becomes dmlog in place, denc [B][N][L] = sum_s dmasked relu(mlog) */
int    sdr_mask_backward(const float* mlog, const float* enc, float* dmasked, float* denc, int B, int S, int N, int L,
                         sdr_stream stream);
/* crop + overlap-add read backwards: grad_frames[b][s K + j][t] = grad_out[b][s][hop t + j - hop] (0 outside [0,T)) */
int    sdr_overlap_add_backward(const float* grad_out, float* grad_frames, int B, int SA, int K, int L, int64_t T,
                                sdr_stream stream);
/* dW[n][j] = sum_{b,t} denc[b][n][t] wav[b][hop t + j - hop] (mono, 0 outside [0, T)) */
size_t sdr_encoder_wgrad_scratch_bytes(int B, int N, int K, int L);
int    sdr_encoder_wgrad(const float* denc, const float* wav, float* dw, void* scratch, int B, int N, int K, int L,
                         int64_t T, sdr_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* SUDORMRF_B200_H */
