// wgmma GEMM engine of the Matryoshka denoising path (sm_90a only).
//
// One kernel template covers every dense contraction of the nested U-Net forward and backward:
//   * Linear / 1x1 conv forward, dgrad, wgrad            (reference: nn.Linear / nn.Conv2d 1x1 calls,
//     ml_mdm/models/unet.py:206,219,260-271,605-626,763)
//   * 3x3 conv forward / dgrad as an implicit GEMM over NHWC pixel patches, the nine taps being nine
//     shifted TMA boxes with hardware zero fill for the padding (unet.py:199,210,515,525,632,751;
//     nested_unet.py:110,121), and 3x3 wgrad with pixels as the contraction dimension
//   * attention QK^T / PV and their backward contractions (unet.py:276-294)
//
// Operands are fp16 in HBM, staged by TMA into 128B-swizzled shared memory through an mbarrier pipeline, multiplied
// by wgmma (two consumer warpgroups of 64 x N x 16 instructions, N <= 256) with fp32 accumulators in registers, and
// drained by a fused epilogue (alpha, bias, residual add, GELU, fp32/fp16 stores, split-K atomics), from the registers
// or, in the persistent kernel, from a shared-memory staging tile on warps of its own.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <utility>
#include <vector>

#include "mdm_b200.h"

namespace mdm {

enum GemmKind : int {
  GEMM_PLAIN = 0,       // A, B are (batched) matrices
  GEMM_CONV = 1,        // A = NHWC activation walked as pixel patches with tap shifts; B = packed weights
  GEMM_CONV_WGRAD = 2,  // A = dY patches, B = shifted X patches, contraction over pixels
};

enum GemmAct : int { ACT_NONE = 0, ACT_GELU = 1 };

using TmapSpec = mdm_tmap_spec;      // see include/mdm_b200.h
using GemmParams = mdm_gemm_params;  // see include/mdm_b200.h

// Host launcher. a_mn / b_mn select MN-major (transposed) operands. b_lo / a_lo (optional): second fp16 planes of B and
// of a K-major A, laid out exactly like them; the kernel then computes A B + A B_lo + A_lo B. Returns cudaError_t as int.
int launch_gemm(const TmapSpec& A, const TmapSpec& B, int a_mn, int b_mn, const GemmParams& p,
                cudaStream_t stream, const void* b_lo = nullptr, const void* a_lo = nullptr);

// Counts kernel launches issued by this library (bench.py reports it as gpu_launches).
extern unsigned long long g_launch_count;
extern int g_sm_reserve;  // mdm_set_sm_reserve: SMs the persistent GEMM grid leaves free for collectives
extern bool g_profile;
extern std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_profile_events;
extern std::vector<mdm_gemm_params> g_profile_params;
extern std::vector<int> g_profile_majors;
extern std::vector<int> g_profile_planes;  // PL_BLO | PL_ALO of each profiled launch

}  // namespace mdm
