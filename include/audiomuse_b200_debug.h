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

#ifdef __cplusplus
}
#endif
#endif /* AUDIOMUSE_B200_DEBUG_H */
