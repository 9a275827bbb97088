// Pieces shared by the two fused attention kernels (attention.cu: spatial self + cross attention of the denoiser;
// token_attention.cu: masked self-attention over text tokens): shared-memory descriptors of 128B-swizzled
// [rows][64 fp16] k-blocks, accumulator-fragment helpers and the TMA view of one head of a [rows][slots * d] tensor.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ptx.cuh"

namespace mdm {
namespace attn {

constexpr int KB_BYTES = 128 * 128;  // one [128 rows][64 fp16] k-block / slab

__device__ __forceinline__ uint64_t desc_k(uint32_t base, int k16) {  // K-major, 16-element step k16
  return ptx::make_smem_desc_sw128(base + k16 * 32, 16, 1024);
}
__device__ __forceinline__ uint64_t desc_mn(uint32_t base, int k16, uint32_t slab_bytes) {  // MN-major
  return ptx::make_smem_desc_sw128(base + k16 * 2048, slab_bytes, 1024);
}

// Accumulator fragment of a 64 x N wgmma in one thread: element e = 4 j + 2 h + u holds row
// (warp % 4) * 16 + lane / 4 + 8 h and column 8 j + 2 (lane % 4) + u of the warpgroup's 64-row block.
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
// the 16-column k step t of a 64 x N accumulator as the A operand (four fp16x2 registers) of the next wgmma
__device__ __forceinline__ void frag_a(const float* v, int t, uint32_t* a) {
  a[0] = pack_half2(v[8 * t + 0], v[8 * t + 1]);
  a[1] = pack_half2(v[8 * t + 2], v[8 * t + 3]);
  a[2] = pack_half2(v[8 * t + 4], v[8 * t + 5]);
  a[3] = pack_half2(v[8 * t + 6], v[8 * t + 7]);
}
// row reductions over the four threads (lane % 4) that share an accumulator row
__device__ __forceinline__ float quad_max(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
__device__ __forceinline__ float quad_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}

// 4-D fp16 view (inner d, rows, slots, batch), box {64, box_rows, 1, 1}, 128B swizzle; elements outside the view
// (columns >= d, rows >= rows) arrive as zeros
void head_map(CUtensorMap* m, const void* ptr, int d, int rows, long long row_stride, int slots, long long slot_stride,
              int batch, long long batch_stride, int box_rows = 128);
// out[r][c] = half(in[r][c]) for c < C, rows with stride ld_out (C % 4 == 0)
void cast_rows_f16(const float* in, __half* out, long long rows, int C, int ld_out, cudaStream_t st);

}  // namespace attn
}  // namespace mdm
