/*
 * audiomuse_b200_debug.h -- debug / probe entry points, built into libaudiomuse_b200_debug.so (the product library
 * libaudiomuse_b200.so does not export them).  Test infrastructure and tuning probes only.
 */
#ifndef AUDIOMUSE_B200_DEBUG_H
#define AUDIOMUSE_B200_DEBUG_H

#include "audiomuse_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* debug: wgmma GEMM vs a CUDA-core reference on seeded operands (tests/test_gpu_gemm.py) */
AM_API int am_selftest_gemm(int M, int N, int K, int flags, double* max_abs_diff);
/* debug: device time (CUDA events, mean of `iters` launches after one warm-up) of the wgmma GEMM
 * on seeded bf16 operands, bf16 output, no epilogue terms: the tensor-pipe ceiling of this kernel */
AM_API int am_bench_gemm(int M, int N, int K, int iters, double* ms_per_launch);
/* debug: issue rate of one fp16x2 / pack / permute instruction kind (op 0 HFMA2, 1 HFMA2 immediate, 2 HFMA2.SAT,
 * 3 HMNMX2 pair, 4 PRMT, 5 F2FP pack + add, 6 HFMA2 + PRMT) with `warps` warps per SM: cycles per warp-instruction
 * per SM sub-partition */
AM_API int am_probe_pipe(int op, int warps, int iters, double* cycles_per_warp_instr_per_smsp);
/* debug: one inverted-residual block [1x1 expand + bias + ReLU6] -> 3x3 depthwise (pad 1, stride) + bias + ReLU6 ->
 * 1x1 project + bias [+ X], on host operands (bf16 as raw uint16, NHWC activations): X [B, H, W, cin_p],
 * W1 [cmid_p, cin_p] + b1 [cmid_p] (NULL without an expansion, then cin_p == cmid_p), wd [9, cmid_p] + bd [cmid_p],
 * W2 [cout_p, cmid_p] + b2 [cout_p] -> Y [B, Ho, Wo, cout_p].  Allocates, uploads, runs, synchronises, downloads.
 *   path 0: the fused kernel as the encoder plans it; a block it rejects is an error and launches nothing.
 *           *info = the ring depth of the plan.
 *   path 1: layer by layer through the encoder's GEMM and depthwise dispatch; *info = the depthwise kernel (0 strip,
 *           1 row, 2 fp32 generic).  E_out [B, H, W, cmid_p] and D_out [B, Ho, Wo, cmid_p] (may be NULL) receive the
 *           expanded and depthwise tensors.
 *   path 2: the fused kernel's plan only, on the host (no device, no operand is read: they may be NULL);
 *           *info = the output rows (time) of its tiles, 8 or 16 (tiles are 8 columns wide).  A block it rejects is
 *           an error. */
AM_API int am_debug_block(int path, int B, int H, int W, int cin_p, int cmid_p, int cout_p, int stride, int has_expand,
                          int residual, const uint16_t* X, const uint16_t* W1, const float* b1, const float* wd,
                          const float* bd, const uint16_t* W2, const float* b2, uint16_t* Y, uint16_t* E_out,
                          uint16_t* D_out, int* info);
/* debug: one k-means Lloyd step on a named path, with the operands of am_kmeans_plan_step plus the rows X_dev [N, d]
 * and k; synchronises before it returns.
 *   path 0: the tensor-core step; a shape it does not take is an error.
 *   path 1: the exact CUDA-core step. */
AM_API int am_debug_kmeans_step(int path, const float* X_dev, int64_t N, int d, int k, const float* centers_dev,
                                int32_t* labels_dev, float* sums_dev, float* counts_dev, float* inertia_dev,
                                float* dist_dev, void* stream);

/* debug: the encoder's execution plan for windows of T frames.  counts[4] = steps, late_step (the first step of the
 * late phase), layers, head ops.  The arrays may be NULL; else, sized from counts:
 *   steps  [n_steps, 9]:  kind (kStepStem .. kStepSqueezeExcite), first, last layer, in H, in W, out H, out W, cout_p,
 *                         starts_block
 *   layers [n_layers, 18]: type, cin, cout, kh, kw, stride, pad_t, pad_b, pad_l, pad_r, act, gate_act, cmid,
 *                         h_is_time, residual, block_start, cin_p, cout_p
 *   head   [n_head, 8]:   kind, a, b, dst, K, N (the width it writes), act, stride;  head_eps [n_head, 2]: eps, eps2 */
#define AM_TRACE_STEP_INTS 9
#define AM_TRACE_LAYER_INTS 18
#define AM_TRACE_HEAD_INTS 8
AM_API int am_debug_encoder_plan(am_model* m, int T, int* counts, int* steps, int* layers, int* head, float* head_eps);
/* debug: one forward pass of B windows of the host log-mel [B, n_mels, T] through the encoder's own dispatch, traced.
 * steps_out: every step's output in plan order, each raw bf16 NHWC [B, out H, out W, cout_p] (padded channels
 * included); head_out: every head op's result in program order, each f32 [B, N] (op 0: the pooling); emb [B, emb]:
 * the embedding, as am_clap_embed computes it.  Synchronises before it returns. */
AM_API int am_debug_encoder_trace(am_model* m, const float* mel, int B, int T, uint16_t* steps_out, float* head_out,
                                  float* emb);

#ifdef __cplusplus
}
#endif
#endif /* AUDIOMUSE_B200_DEBUG_H */
