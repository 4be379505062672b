// The host launchers and eligibility predicates that api.cu's model code calls, by defining file.  api.cu and every
// file that defines one of them include this header, so a definition that drifts from its declaration is a compile or
// link error (the library is linked with undefined symbols refused) instead of a failure at load time.  Every launcher
// enqueues its kernels through launch.cuh.
// A C-ABI entry whose work no model code shares (mixture consistency, the metrics, resampling, windowed separation and
// the pyramid stage entries) is defined in the file that implements it instead, inside that file's one extern "C"
// block: there the public header's declaration makes a drifting definition a compile error the same way.
#pragma once
#include <initializer_list>
#include "launch.cuh"

namespace sdr {

// per-level depthwise and merge (levels.cu)
int launch_depthwise(const float* x, const NormIn& nin, const float* w5, const float* bias,
                     float* y, double* stats_out, int samples, int C, int Lin, int stride,
                     cudaStream_t st);
int launch_merge(const float* const* z, const NormIn* nins, int depth, float* m, double* stats_out,
                 int samples, int C, int L, cudaStream_t st);

// depthwise pyramid in one pass (pyramid.cu)
bool pyramid_eligible(int D, int samples, int C, int L);
size_t pyramid_rowstats_bytes(int samples, int C, int D);
size_t pyramid_table_bytes(int samples, int C, int D);
int launch_pyramid_fused(const float* y, const NormIn& nin, const float* const* w5, const float* const* bias,
                         const float* const* gamma, const float* const* beta, float* m, double* stats0, double* stats_m,
                         double* rowstats, float* table, int D, int samples, int C, int L, cudaStream_t st);

// 1x1 convolutions, FFMA path (pointwise.cu)
int launch_pointwise_ffma(const float* x, const NormIn& nin, const float* W, const float* bias,
                          const float* residual, const float* gate, int gate_channels,
                          float* y, double* stats_out, int samples, int M, int K, int L,
                          int epilogue, cudaStream_t st);
bool preadd_eligible(int M, int K, int L);
int launch_pointwise_small_preadd(const float* x, const float* pre_add, const NormIn& pre_norm, float* xt_out,
                                  const float* W, const float* bias, float* y, double* stats_out,
                                  int samples, int M, int K, int L, cudaStream_t st);

// encoder and overlap-add (frontback.cu)
bool encoder_ffma_fits(int A, int K);
int launch_encoder(const float* wav, const float* weight, const float* bias, int relu, float* enc, double* stats,
                   int B, int A, long long T, int N, int K, int L, int pad, cudaStream_t st);
int launch_overlap_add(const float* frames, const float* mix, const float* bias, const float2* rescale, float* out,
                       int B, int SA, int K, int L, long long T, cudaStream_t st);

// transform-average-concatenate of the GroupComm blocks (tac.cu)
int launch_tac(const float* x, const float* const* params, float* o, double* stats,
               int B, int G, int n, int L, cudaStream_t st);
int launch_tac_apply(const float* x, const float* o, const NormIn& nin, float* out,
                     int samples, int n, int L, cudaStream_t st);

// causal model (causal.cu)
bool causal_pyramid_eligible(int D, int L);
int launch_causal_pyramid(const float* y, const float* slope_in, const float* const* w, const float* const* b,
                          const float* const* slope, float* m, int D, int samples, int C, int L, cudaStream_t st);
int launch_take_taps(const float* src, float* dst, long long rows, int src_taps, int dst_taps, cudaStream_t st);
int launch_scale_by_scalar(const float* src, const float* gain, float* dst, long long n, cudaStream_t st);

// streaming of the causal model (stream.cu)
int launch_stream_frame(const float* chunk, const float* state, long long slot_stride, float* framed, int B, int A,
                        int k, int Kr, int F, long long C, cudaStream_t st);
bool causal_stream_eligible(int D, int F);
int launch_causal_stream(const float* y, const float* slope_in, const float* const* w, const float* const* b,
                         const float* const* slope, float* hist, long long hist_stride, float* m, int D, int B, int C,
                         int F, cudaStream_t st);
int launch_stream_ola(const float* frames, const float* chunk, float* state, long long slot_stride, long long carry_off,
                      float* out, int B, int SA, int A, int k, int F, long long C, int mc, cudaStream_t st);
// slot b of a region is [base + b * slot_bytes, base + (b + 1) * slot_bytes)
struct SlotRegion { void* base; size_t slot_bytes; };
int reset_slots(std::initializer_list<SlotRegion> regions, int B, const int* slots, int n, const unsigned char* mask,
                cudaStream_t st);
int launch_stream_flush(const float* state, long long slot_stride, long long carry_off, float* tail, int B, int SA,
                        int hop, int mc, cudaStream_t st);

// original model (original.cu)
int launch_residual_norm(const float* e, const NormIn& fe, float* x, const NormIn& fx, double* stats_out,
                         int samples, int C, int L, cudaStream_t st);
int launch_softmax_gate(const float* logits, const float* enc, float* out, int B, int S, int N, int L, cudaStream_t st);
int launch_toeplitz_mask(const float* w, const float* bias, float* W, float* brow, int S, int N, cudaStream_t st);
int launch_grouped_decoder(const float* w, float* wt, int S, int N, int K, cudaStream_t st);

// pre/post steps (prepost.cu)
int launch_utterance_stats(const float* wav, double* sums, float2* mean_std, int rows, long long T,
                           const long long* lengths, cudaStream_t st);
int launch_normalize_rows(const float* wav, const float2* mean_std, float* out, int rows, long long T,
                          const long long* lengths, cudaStream_t st);

// tensor-core path (pointwise_mma.cu)
size_t pointwise_mma_packed_bytes(int M, int K);
int pack_pointwise_mma(const float* W, int M, int K, void* packed, cudaStream_t st);
int launch_pointwise_mma(const float* x, const NormIn& nin, const void* wpk, const float* bias,
                         const float* residual, const float* gate, int gate_channels,
                         float* y, double* stats_out, int samples, int M, int K, int L,
                         int epilogue, cudaStream_t st);
size_t encoder_mma_packed_bytes(int N, int A, int Kk);
int pack_encoder_mma(const float* W, int N, int A, int Kk, void* packed, cudaStream_t st);
int launch_encoder_mma(const float* wav, const void* wpk, const float* bias, int relu, float* enc, double* stats,
                       int B, int A, long long T, int N, int Kk, int L, int pad, cudaStream_t st);

// backward of the improved model (backward.cu)
size_t wgrad_scratch_bytes(int samples, int M, int K, int L);
int launch_wgrad(const float* dY, const float* X, const NormIn& nin, float* dW, float* db, float* scratch,
                 int samples, int M, int K, int L, cudaStream_t st);
size_t norm_bwd_scratch_bytes(int samples, int C);
int launch_norm_bwd(const float* x, const NormIn& nin, const float* dp, float* out, int accumulate, float* g_gamma,
                    float* g_beta, float* g_slope, double* scratch, int samples, int C, int L, cudaStream_t st);
size_t dw_bwd_scratch_bytes(int samples, int C);
int launch_dw_bwd(const float* dz, const float* x, const NormIn& nin, const float* w5, const float* pool, int P,
                  float* din, float* gw, float* gb, double* scratch, int samples, int C, int Lin, int stride,
                  cudaStream_t st);
int launch_mask_apply(const float* mlog, const float* e, float* masked, int B, int S, int N, int L, cudaStream_t st);
int launch_mask_bwd(const float* mlog, const float* e, float* dmasked, float* de, int B, int S, int N, int L,
                    cudaStream_t st);
int launch_frame_gather(const float* wav, float* frames, int B, int SA, int K, int L, long long T, cudaStream_t st);
int launch_transpose(const float* w, float* wt, int R, int C, cudaStream_t st);

}  // namespace sdr
