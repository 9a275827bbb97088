// wgmma / TMA / mbarrier GEMM engine (see gemm_tc.cuh for the role of this kernel in the path).
#include "gemm_tc.cuh"

#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <climits>
#include <cstring>
#include <set>
#include <utility>
#include <vector>

#include "gemm_epi.cuh"
#include "ptx.cuh"

namespace mdm {

unsigned long long g_launch_count = 0;
int g_sm_reserve = 0;

// Optional per-launch timing of this kernel (bench.py's roofline leg): CUDA events on the launching
// stream around every launch while enabled.
bool g_profile = false;
std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_profile_events;
std::vector<GemmParams> g_profile_params;  // parallel to g_profile_events
std::vector<int> g_profile_majors;
std::vector<int> g_profile_planes;

using namespace ptx;

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // fp16 elements (K-major) or rows (MN-major) per pipeline stage
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;
constexpr int SLAB_BYTES = 64 * 64 * 2;  // one 64(k) x 64(mn) MN-major slab
constexpr int MAX_STAGES = 8;
constexpr int SMEM_LIMIT = 226 * 1024;  // dynamic shared memory; with the static barriers within H100's 227 KB a block

// warpgroup 0: TMA producer (one thread) and, staged, the epilogue warps (1-3); warpgroups 1 and 2: wgmma consumers, 64
// tile rows each, and the in-register epilogue
constexpr int NUM_THREADS = 384;
constexpr int RASTER_N = 8;   // column tiles per band of the persistent kernel's tile order

// Epilogue of one pair of adjacent columns (c, c + 1) of tile row r: alpha, bias, residual, GELU', then the stores.
__device__ __forceinline__ void epi_pair(const GemmParams& p, long long row_off, int col0, float v0, float v1,
                                         float alpha) {
  if (col0 >= p.N) return;
  const bool two = col0 + 1 < p.N;
  v0 *= alpha;
  v1 *= alpha;
  if (p.bias != nullptr) {
    v0 += __ldg(p.bias + col0);
    if (two) v1 += __ldg(p.bias + col0 + 1);
  }
  const long long off = row_off + col0;
  if (p.residual != nullptr) {
    v0 += __ldg(p.residual + off);
    if (two) v1 += __ldg(p.residual + off + 1);
  }
  if (p.gelu_grad_src != nullptr) {
    const __half* gp = reinterpret_cast<const __half*>(p.gelu_grad_src) + off;
    v0 *= gelu_grad(__half2float(gp[0]));
    if (two) v1 *= gelu_grad(__half2float(gp[1]));
  }
  if (p.atomic) {
    atomicAdd(p.out_f32 + off, v0);
    if (two) atomicAdd(p.out_f32 + off + 1, v1);
    return;
  }
  if (p.out_f32 != nullptr) {
    float* o = p.out_f32 + off;
    if (two && (reinterpret_cast<uintptr_t>(o) & 7) == 0) {
      *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
    } else {
      o[0] = v0;
      if (two) o[1] = v1;
    }
  }
  __half* outs[2] = {reinterpret_cast<__half*>(p.out_f16), reinterpret_cast<__half*>(p.out_act_f16)};
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    if (outs[t] == nullptr) continue;
    float a0 = v0, a1 = v1;
    if (t == 1 && p.act == ACT_GELU) {
      a0 = gelu_erf(v0);
      a1 = gelu_erf(v1);
    }
    __half* o = outs[t] + off;
    if (two && (reinterpret_cast<uintptr_t>(o) & 3) == 0) {
      *reinterpret_cast<__half2*>(o) = __floats2half2_rn(a0, a1);
    } else {
      o[0] = __float2half_rn(a0);
      if (two) o[1] = __float2half_rn(a1);
    }
  }
}

// Operand planes a kernel multiplies besides A x B: the lo plane of B (weights) and the lo plane of a K-major A.
constexpr int PL_BLO = 1;
constexpr int PL_ALO = 2;

// Stage layout of the plain and conv modes: A | B | B lo plane (PL_BLO) | A lo plane (PL_ALO).
template <bool B_MN, int BN, int PL>
struct StageLayout {
  static constexpr int nb_alloc = B_MN ? ((BN + 63) / 64) * 64 : BN;
  static constexpr int b_bytes = nb_alloc * 128;  // one B plane
  static constexpr int b_lo_off = A_STAGE_BYTES + b_bytes;
  static constexpr int a_lo_off = A_STAGE_BYTES + b_bytes * ((PL & PL_BLO) ? 2 : 1);
  static constexpr int bytes = a_lo_off + ((PL & PL_ALO) ? A_STAGE_BYTES : 0);
};

// TMA loads of k block kb of the plain and conv modes into the stage at sA (producer thread).
template <bool A_MN, bool B_MN, int BN, int PL>
__device__ __forceinline__ void load_stage(const GemmParams& p, const CUtensorMap* tmA, const CUtensorMap* tmB,
                                           const CUtensorMap* tmBlo, const CUtensorMap* tmAlo, uint8_t* sA,
                                           uint64_t* bar, int kb, int m0, int n0, int z1, int z2, int img, int th,
                                           int tw) {
  using S = StageLayout<B_MN, BN, PL>;
  constexpr int nslab_b = S::nb_alloc / 64;
  uint8_t* sB = sA + A_STAGE_BYTES;
  if (p.kind == GEMM_PLAIN) {
    const int az1 = p.a_use_z ? z1 + p.a_z1_off : 0;
    const int az2 = p.a_use_z ? z2 : 0;
    const int bz1 = p.b_use_z ? z1 + p.b_z1_off : 0;
    const int bz2 = p.b_use_z ? z2 : 0;
    if (!A_MN) {
      tma_load_4d(sA, tmA, bar, kb * BLOCK_K, m0, az1, az2);
      if (PL & PL_ALO) tma_load_4d(sA + S::a_lo_off, tmAlo, bar, kb * BLOCK_K, m0, az1, az2);
    } else {
      tma_load_4d(sA, tmA, bar, m0, kb * BLOCK_K, az1, az2);
      tma_load_4d(sA + SLAB_BYTES, tmA, bar, m0 + 64, kb * BLOCK_K, az1, az2);
    }
#pragma unroll
    for (int pl = 0; pl <= ((PL & PL_BLO) ? 1 : 0); ++pl) {
      const CUtensorMap* mb = pl ? tmBlo : tmB;
      uint8_t* sBp = sB + pl * S::b_bytes;
      if (!B_MN) {
        tma_load_4d(sBp, mb, bar, kb * BLOCK_K, n0, bz1, bz2);
      } else {
        for (int s = 0; s < nslab_b; ++s)
          tma_load_4d(sBp + s * SLAB_BYTES, mb, bar, n0 + 64 * s, kb * BLOCK_K, bz1, bz2);
      }
    }
  } else {  // GEMM_CONV
    const int tap = kb / p.kblocks_c;
    const int cb = kb - tap * p.kblocks_c;
    const int kh = (p.taps == 9) ? tap / 3 : 1;
    const int kw = (p.taps == 9) ? tap % 3 : 1;
    tma_load_4d(sA, tmA, bar, cb * BLOCK_K, tw * p.PW + kw - 1, th * p.PH + kh - 1, img);
    if (PL & PL_ALO) tma_load_4d(sA + S::a_lo_off, tmAlo, bar, cb * BLOCK_K, tw * p.PW + kw - 1, th * p.PH + kh - 1, img);
    const int wt = p.flip ? (p.taps - 1 - tap) : tap;
#pragma unroll
    for (int pl = 0; pl <= ((PL & PL_BLO) ? 1 : 0); ++pl) {
      const CUtensorMap* mb = pl ? tmBlo : tmB;
      uint8_t* sBp = sB + pl * S::b_bytes;
      if (!B_MN) {
        tma_load_4d(sBp, mb, bar, cb * BLOCK_K, n0, tap, 0);
      } else {
        for (int s = 0; s < nslab_b; ++s)
          tma_load_4d(sBp + s * SLAB_BYTES, mb, bar, n0 + 64 * s, cb * BLOCK_K, wt, 0);
      }
    }
  }
}

// The wgmmas of k16 step k of a plain / conv stage for 64 tile rows, in the order every output element sums them:
// A x B, then A x B lo, then A lo x B. a_rows / a_lo_rows: those rows of the A planes in the stage.
template <bool A_MN, bool B_MN, int BN, int PL>
__device__ __forceinline__ void mma_k16(float* acc, uint32_t a_rows, uint32_t a_lo_rows, uint32_t b_base,
                                        uint32_t b_lo_base, int k, uint32_t scale_d) {
  const uint64_t adesc = A_MN ? make_smem_desc_sw128(a_rows + k * 2048, SLAB_BYTES, 1024)
                              : make_smem_desc_sw128(a_rows + k * 32, 16, 1024);
  const uint64_t bdesc = B_MN ? make_smem_desc_sw128(b_base + k * 2048, SLAB_BYTES, 1024)
                              : make_smem_desc_sw128(b_base + k * 32, 16, 1024);
  Wgmma<BN>::template ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc, scale_d);
  if constexpr ((PL & PL_BLO) != 0) {
    const uint64_t bdesc_lo = B_MN ? make_smem_desc_sw128(b_lo_base + k * 2048, SLAB_BYTES, 1024)
                                   : make_smem_desc_sw128(b_lo_base + k * 32, 16, 1024);
    Wgmma<BN>::template ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc_lo, 1u);
  }
  if constexpr (!A_MN && (PL & PL_ALO) != 0) {
    Wgmma<BN>::template ss<0, B_MN ? 1 : 0>(acc, make_smem_desc_sw128(a_lo_rows + k * 32, 16, 1024), bdesc, 1u);
  }
}

// Output tile of a linear tile index of the plain and conv modes (tiles ordered m fastest, then n, then z).
struct TileCoord {
  int m0, n0, z1, z2, img, th, tw, kb_begin, kb_end;
};
__device__ __forceinline__ TileCoord tile_coord(const GemmParams& p, int m_tile, int n_tile, int z, int bn) {
  TileCoord c;
  const int split = z % p.nsplit;
  z /= p.nsplit;
  c.z1 = z % p.nz1;
  c.z2 = z / p.nz1;
  const int per = (p.num_kblocks + p.nsplit - 1) / p.nsplit;
  c.kb_begin = split * per;
  c.kb_end = min(p.num_kblocks, c.kb_begin + per);
  c.m0 = m_tile * BLOCK_M;
  c.n0 = n_tile * bn;
  c.img = c.th = c.tw = 0;
  if (p.kind == GEMM_CONV) {
    c.tw = m_tile % p.tiles_w;
    const int t = m_tile / p.tiles_w;
    c.th = t % p.tiles_h;
    c.img = t / p.tiles_h;
  }
  return c;
}

// Epilogue of 64 tile rows (r0 .. r0 + 63) from the accumulators of one m64 wgmma.
template <int BN>
__device__ __forceinline__ void store_rows(const GemmParams& p, const float* acc, const TileCoord& c, int r0,
                                           float alpha) {
  const int lane = threadIdx.x & 31;
  const int wq = (threadIdx.x >> 5) & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + wq * 16 + (lane >> 2) + 8 * h;  // tile row of accumulator elements 4j + 2h + {0, 1}
    bool valid;
    long long row_off;
    if (p.kind == GEMM_CONV) {
      const int ph = r / p.PW;
      const int pw = r - ph * p.PW;
      const int hh = c.th * p.PH + ph;
      const int ww = c.tw * p.PW + pw;
      valid = (hh < p.H) && (ww < p.W) && (c.img < p.nimg);
      row_off = (static_cast<long long>(c.img * p.H + hh) * p.W + ww) * p.ldc;
    } else {
      const int row = c.m0 + r;
      valid = row < p.M;
      row_off = static_cast<long long>(row) * p.ldc + static_cast<long long>(c.z1) * p.c_z1_stride +
                static_cast<long long>(c.z2) * p.c_z2_stride;
    }
    if (!valid) continue;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
      epi_pair(p, row_off, c.n0 + j * 8 + (lane & 3) * 2, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], alpha);
  }
}

__device__ __forceinline__ float epi_alpha(const GemmParams& p) {
  return p.alpha_dev != nullptr ? p.alpha * __ldg(p.alpha_dev) : p.alpha;
}

// Staged epilogue of the persistent kernel: the consumers park their raw accumulators in a shared-memory tile and go
// on to the next tile's MMAs while warps 1-3 of warpgroup 0 (idle otherwise: one thread issues the TMA loads) run the
// epilogue from there.
constexpr int EPI_THREADS = 96;
constexpr int EPI_ROWS = 8;  // rows each epilogue thread has in flight: 96 x 8 x 16 B = 12 KB of residual loads per SM
// Row stride of the staging tile: BN + STAGE_PAD floats. The pad spreads a half-warp's float2 fragment stores over all
// 32 banks (a 512 B row stride would put them 8-way on the same banks).
constexpr int STAGE_PAD = 8;

// Raw accumulators of 64 tile rows (r0 .. r0 + 63) of one m64 wgmma into the staging tile.
template <int BN>
__device__ __forceinline__ void stage_rows(float* stg, const float* acc, int r0) {
  const int lane = threadIdx.x & 31;
  const int wq = (threadIdx.x >> 5) & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float* row = stg + (r0 + wq * 16 + (lane >> 2) + 8 * h) * (BN + STAGE_PAD) + (lane & 3) * 2;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
      *reinterpret_cast<float2*>(row + j * 8) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
  }
}

// Epilogue of one staged tile by epilogue thread et (0 .. 95). Each thread owns one quad of 4 adjacent columns (96 is
// a multiple of every BN / 4) and walks the tile's rows, so a warp's loads and stores cover whole row segments and the
// bias is read once per tile. The arithmetic is epi_pair's, operation by operation (alpha, bias, residual, then the
// stores); the explicitly rounded mul / adds keep v * alpha + bias unfused, as epi_pair compiles. The launcher keeps
// GELU and GELU' epilogues on the in-register path, so there are none here (out_act_f16 receives a copy of out_f16).
// vec: every output / operand row is 16 B (fp32) or 8 B (fp16) aligned at each column quad.
template <int BN>
__device__ __forceinline__ void epilogue_staged(const GemmParams& p, const float* stg, const TileCoord& c, int et,
                                                float alpha, bool vec) {
  constexpr int QPR = BN / 4;            // column quads per row
  constexpr int RPP = EPI_THREADS / QPR;  // rows per pass of the 96 threads
  const int q = et % QPR;
  const int col0 = c.n0 + 4 * q;
  if (col0 >= p.N) return;
  const int ncol = min(4, p.N - col0);
  const bool full = vec && ncol == 4;
  float bias[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) bias[e] = (p.bias != nullptr && e < ncol) ? __ldg(p.bias + col0 + e) : 0.f;
  __half* o16[2] = {reinterpret_cast<__half*>(p.out_f16), reinterpret_cast<__half*>(p.out_act_f16)};

  for (int rb = et / QPR; rb < BLOCK_M; rb += RPP * EPI_ROWS) {
    long long off[EPI_ROWS];
    float v[EPI_ROWS][4];
    // output offsets (-1: row outside the output) and the staged accumulators
#pragma unroll
    for (int u = 0; u < EPI_ROWS; ++u) {
      const int r = rb + u * RPP;
      off[u] = -1;
      if (r < BLOCK_M) {
        const float4 a = *reinterpret_cast<const float4*>(stg + r * (BN + STAGE_PAD) + 4 * q);
        v[u][0] = a.x;
        v[u][1] = a.y;
        v[u][2] = a.z;
        v[u][3] = a.w;
        if (p.kind == GEMM_CONV) {
          const int ph = r / p.PW;
          const int pw = r - ph * p.PW;
          const int hh = c.th * p.PH + ph;
          const int ww = c.tw * p.PW + pw;
          if (hh < p.H && ww < p.W && c.img < p.nimg)
            off[u] = (static_cast<long long>(c.img * p.H + hh) * p.W + ww) * p.ldc + col0;
        } else if (c.m0 + r < p.M) {
          off[u] = static_cast<long long>(c.m0 + r) * p.ldc + static_cast<long long>(c.z1) * p.c_z1_stride +
                   static_cast<long long>(c.z2) * p.c_z2_stride + col0;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < EPI_ROWS; ++u)
#pragma unroll
      for (int e = 0; e < 4; ++e) v[u][e] = __fmul_rn(v[u][e], alpha);
    if (p.bias != nullptr) {
#pragma unroll
      for (int u = 0; u < EPI_ROWS; ++u)
#pragma unroll
        for (int e = 0; e < 4; ++e) v[u][e] = __fadd_rn(v[u][e], bias[e]);
    }
    if (p.residual != nullptr) {
      // all rows' loads first, so EPI_ROWS of them are in flight
      float res[EPI_ROWS][4];
#pragma unroll
      for (int u = 0; u < EPI_ROWS; ++u) {
        if (off[u] < 0) continue;
        if (full) {
          const float4 x = __ldg(reinterpret_cast<const float4*>(p.residual + off[u]));
          res[u][0] = x.x;
          res[u][1] = x.y;
          res[u][2] = x.z;
          res[u][3] = x.w;
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e) res[u][e] = e < ncol ? __ldg(p.residual + off[u] + e) : 0.f;
        }
      }
#pragma unroll
      for (int u = 0; u < EPI_ROWS; ++u)
#pragma unroll
        for (int e = 0; e < 4; ++e) v[u][e] = __fadd_rn(v[u][e], res[u][e]);
    }
#pragma unroll
    for (int u = 0; u < EPI_ROWS; ++u) {
      if (off[u] < 0) continue;
      if (p.out_f32 != nullptr) {
        float* o = p.out_f32 + off[u];
        if (full) {
          *reinterpret_cast<float4*>(o) = make_float4(v[u][0], v[u][1], v[u][2], v[u][3]);
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (e < ncol) o[e] = v[u][e];
        }
      }
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        if (o16[t] == nullptr) continue;
        const float* a = v[u];
        __half* o = o16[t] + off[u];
        if (full) {
          const __half2 h01 = __floats2half2_rn(a[0], a[1]);
          const __half2 h23 = __floats2half2_rn(a[2], a[3]);
          uint2 x;
          x.x = *reinterpret_cast<const uint32_t*>(&h01);
          x.y = *reinterpret_cast<const uint32_t*>(&h23);
          *reinterpret_cast<uint2*>(o) = x;
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (e < ncol) o[e] = __float2half_rn(a[e]);
        }
      }
    }
  }
}

// TMA epilogue of the persistent kernel (p.epi_tma = 1). The staging tile is a row of 128-row panels, 32 columns each,
// in the 128B (fp32) or 64B (fp16) swizzle of a 32-column TMA box, so one box loads or stores a whole panel and the
// consumers' fragment accesses stay free of bank conflicts. An epilogue touches fp32 planes (residual, out_f32) or fp16
// ones (GELU' source, out_f16, out_act_f16), never both (the launcher's rule): the fp32 plane fills the staging tile;
// fp16 plane 0 (GELU' source, then out_f16) its first half and fp16 plane 1 (out_act_f16) its second.
// Plain mode only (see epi_tma_maps): the tensor maps view each epilogue buffer as (N, M, z1, z2).
struct EpiMaps {
  CUtensorMap src;   // residual (fp32) or GELU' source (fp16)
  CUtensorMap o32;   // out_f32
  CUtensorMap o16;   // out_f16
  CUtensorMap oact;  // out_act_f16
};
constexpr int EPI_PANEL = 32;                       // columns per panel
constexpr int EPI_PANEL_F32 = BLOCK_M * EPI_PANEL * 4;  // bytes of one fp32 panel
constexpr int EPI_PANEL_F16 = BLOCK_M * EPI_PANEL * 2;

// byte offsets of element (r, c) of the staging tile, c even (the pair c, c + 1 is contiguous)
__device__ __forceinline__ uint32_t epi_off_f32(int r, int c) {
  const int cc = c & 31;
  return (c >> 5) * EPI_PANEL_F32 + r * 128 + ((((cc >> 2) ^ r) & 7) << 4) + (cc & 3) * 4;
}
template <int BN>
__device__ __forceinline__ uint32_t epi_off_f16(int plane, int r, int c) {
  const int cc = c & 31;
  return plane * (BN / EPI_PANEL) * EPI_PANEL_F16 + (c >> 5) * EPI_PANEL_F16 + r * 64 +
         ((((cc >> 3) ^ (r >> 1)) & 3) << 4) + (cc & 7) * 2;
}

// The consumers' part of the TMA epilogue for 64 tile rows (r0 .. r0 + 63): epi_pair's arithmetic on the accumulators,
// operation by operation (explicitly rounded, so v * alpha + bias stays unfused as epi_pair compiles), with the
// residual or GELU' source read from the staging tile where the epilogue thread's TMA load left it, and the results
// written back over it for the TMA stores. Every element is read and written by the same thread. Rows and columns
// outside the output compute on zero fill and are never stored.
template <int BN>
__device__ __forceinline__ void fold_rows(const GemmParams& p, uint8_t* stg, const float* acc, int n0, int r0,
                                          float alpha) {
  const int lane = threadIdx.x & 31;
  const int wq = (threadIdx.x >> 5) & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + wq * 16 + (lane >> 2) + 8 * h;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = j * 8 + (lane & 3) * 2;
      const int col = n0 + c;
      float v0 = __fmul_rn(acc[4 * j + 2 * h], alpha);
      float v1 = __fmul_rn(acc[4 * j + 2 * h + 1], alpha);
      if (p.bias != nullptr) {
        v0 = __fadd_rn(v0, col < p.N ? __ldg(p.bias + col) : 0.f);
        v1 = __fadd_rn(v1, col + 1 < p.N ? __ldg(p.bias + col + 1) : 0.f);
      }
      float2* s32 = reinterpret_cast<float2*>(stg + epi_off_f32(r, c));
      __half2* s16 = reinterpret_cast<__half2*>(stg + epi_off_f16<BN>(0, r, c));
      if (p.residual != nullptr) {
        const float2 x = *s32;
        v0 = __fadd_rn(v0, x.x);
        v1 = __fadd_rn(v1, x.y);
      }
      if (p.gelu_grad_src != nullptr) {
        const float2 x = __half22float2(*s16);
        v0 = __fmul_rn(v0, gelu_grad(x.x));
        v1 = __fmul_rn(v1, gelu_grad(x.y));
      }
      if (p.out_f32 != nullptr) *s32 = make_float2(v0, v1);
      if (p.out_f16 != nullptr) *s16 = __floats2half2_rn(v0, v1);
      if (p.out_act_f16 != nullptr) {
        const bool g = p.act == ACT_GELU;
        *reinterpret_cast<__half2*>(stg + epi_off_f16<BN>(1, r, c)) =
            __floats2half2_rn(g ? gelu_erf(v0) : v0, g ? gelu_erf(v1) : v1);
      }
    }
  }
}

// TMA coordinates of panel j of a tile (see EpiMaps)
__device__ __forceinline__ void epi_coords(const TileCoord& c, int j, int* x) {
  x[0] = c.n0 + j * EPI_PANEL;
  x[1] = c.m0;
  x[2] = c.z1;
  x[3] = c.z2;
}

// The epilogue thread's TMA load of a tile's residual / GELU' source into the staging tile, completing on bar (which
// it arrives on, with or without a source).
template <int BN>
__device__ __forceinline__ void epi_load_source(const GemmParams& p, const EpiMaps& em, uint8_t* stg, uint64_t* bar,
                                                const TileCoord& c) {
  const bool f32 = p.residual != nullptr;
  if (!f32 && p.gelu_grad_src == nullptr) {
    mbar_arrive(bar);
    return;
  }
  const int panel = f32 ? EPI_PANEL_F32 : EPI_PANEL_F16;
  mbar_expect_tx(bar, static_cast<uint32_t>((BN / EPI_PANEL) * panel));
#pragma unroll
  for (int j = 0; j < BN / EPI_PANEL; ++j) {
    int x[4];
    epi_coords(c, j, x);
    tma_load_4d(stg + j * panel, &em.src, bar, x[0], x[1], x[2], x[3]);
  }
}

// The epilogue thread's TMA stores of a folded tile.
template <int BN>
__device__ __forceinline__ void epi_store_tile(const GemmParams& p, const EpiMaps& em, const uint8_t* stg,
                                               const TileCoord& c) {
#pragma unroll
  for (int j = 0; j < BN / EPI_PANEL; ++j) {
    int x[4];
    epi_coords(c, j, x);
    if (p.out_f32 != nullptr) tma_store_4d(&em.o32, stg + j * EPI_PANEL_F32, x[0], x[1], x[2], x[3]);
    if (p.out_f16 != nullptr) tma_store_4d(&em.o16, stg + j * EPI_PANEL_F16, x[0], x[1], x[2], x[3]);
    if (p.out_act_f16 != nullptr)
      tma_store_4d(&em.oact, stg + ((BN / EPI_PANEL) + j) * EPI_PANEL_F16, x[0], x[1], x[2], x[3]);
  }
  bulk_commit();
}

// One output tile per CTA: the weight gradients (MN-major A: plain MN x MN with split-K, 3x3 wgrad with tall stages).
template <bool B_MN, int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmBlo, const __grid_constant__ CUtensorMap tmAlo,
               const __grid_constant__ EpiMaps em, const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[MAX_STAGES];
  __shared__ __align__(8) uint64_t empty_bar[MAX_STAGES];

  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  const int wg = threadIdx.x >> 7;

  using S = StageLayout<B_MN, BN, 0>;
  // weight gradients of narrow layers: kf x 64 pixel rows per stage, and a single A slab when M <= 64
  const int kf = (p.kind == GEMM_CONV_WGRAD && p.kfactor > 1) ? p.kfactor : 1;
  const int slab_bytes = SLAB_BYTES * kf;
  const int a_slabs = (kf > 1 && p.M <= 64) ? 1 : 2;
  const int a_stage_bytes = kf > 1 ? a_slabs * slab_bytes : A_STAGE_BYTES;
  const int stage_bytes = kf > 1 ? a_stage_bytes + S::nb_alloc * 128 * kf : S::bytes;
  const int nstages = p.num_stages;

  const TileCoord c = tile_coord(p, blockIdx.x, blockIdx.y, blockIdx.z, BN);
  const int nkb = c.kb_end - c.kb_begin;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < nstages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // =========================== TMA producer ===========================
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int i = 0; i < nkb; ++i) {
        const int kb = c.kb_begin + i;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sA = smem + stage * stage_bytes;
        uint64_t* bar = &full_bar[stage];
        mbar_expect_tx(bar, static_cast<uint32_t>(stage_bytes));
        if (p.kind != GEMM_CONV_WGRAD) {
          load_stage<true, B_MN, BN, 0>(p, &tmA, &tmB, &tmBlo, &tmAlo, sA, bar, kb, c.m0, c.n0, c.z1, c.z2, c.img,
                                         c.th, c.tw);
        } else {  // k block = one patch of 64 * kf pixels
          uint8_t* sB = sA + a_stage_bytes;
          const int ptw = kb % p.tiles_w;
          const int t = kb / p.tiles_w;
          const int pth = t % p.tiles_h;
          const int pimg = t / p.tiles_h;
          const int kh = (p.taps == 9) ? c.z1 / 3 : 1;
          const int kw = (p.taps == 9) ? c.z1 % 3 : 1;
          tma_load_4d(sA, &tmA, bar, c.m0, ptw * p.PW, pth * p.PH, pimg);
          if (a_slabs == 2) tma_load_4d(sA + slab_bytes, &tmA, bar, c.m0 + 64, ptw * p.PW, pth * p.PH, pimg);
          for (int s = 0; s < S::nb_alloc / 64; ++s)
            tma_load_4d(sB + s * slab_bytes, &tmB, bar, c.n0 + 64 * s, ptw * p.PW + kw - 1, pth * p.PH + kh - 1,
                        pimg);
        }
        if (++stage == nstages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // =========================== wgmma consumers ===========================
  reg_alloc<232>();
  const int cw = wg - 1;  // this warpgroup's 64 rows of the tile
  const int lane = threadIdx.x & 31;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  {
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int i = 0; i < nkb; ++i) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_base = smem_u32(smem + stage * stage_bytes);
      const uint32_t b_base = a_base + a_stage_bytes;
      fence_regs<BN / 2>(acc);
      if constexpr (B_MN) {
        // kf * 64 pixel rows x 64 columns per MN-major slab (64 rows outside the 3x3 wgrad). With one A slab
        // (M <= 64) the second warpgroup re-reads the first slab: its rows (64..127) are never stored.
        const uint32_t a_wg = a_base + (a_slabs == 2 ? cw * slab_bytes : 0);
        wgmma_arrive();
        for (int k = 0; k < 4 * kf; ++k) {
          const uint64_t adesc = make_smem_desc_sw128(a_wg + k * 2048, static_cast<uint32_t>(slab_bytes), 1024);
          const uint64_t bdesc = make_smem_desc_sw128(b_base + k * 2048, static_cast<uint32_t>(slab_bytes), 1024);
          Wgmma<BN>::template ss<1, 1>(acc, adesc, bdesc, (i > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
      } else {
        const uint32_t a_wg = a_base + cw * SLAB_BYTES;
        wgmma_arrive();
#pragma unroll
        for (int k = 0; k < BLOCK_K / 16; ++k)
          mma_k16<true, false, BN, 0>(acc, a_wg, 0, b_base, 0, k, (i > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
      }
      // the previous stage's MMAs have retired once at most this stage's group is in flight: free that slot
      wgmma_wait<1>();
      fence_regs<BN / 2>(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == nstages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    fence_regs<BN / 2>(acc);
  }

  // =========================== epilogue ===========================
  store_rows<BN>(p, acc, c, cw * 64, epi_alpha(p));
}

// Persistent schedule of the weight products (plain K x K, plain K x MN, 3x3 conv forward / data gradient; K-major A).
// Each CTA walks tiles blockIdx.x + i * gridDim.x, and the producer streams the k blocks of all its tiles through one
// stage ring, so the next tile's stages load while the last one is drained. Both consumer warpgroups work on every
// tile, 64 rows each, as in the one-tile kernel. (Consumers taking alternate whole tiles, one in its epilogue while
// the other issues MMAs, measured slower: at 128 accumulators per thread the epilogue of a whole tile on one
// warpgroup took more than twice as long.)
// p.epi_op = 1 (staged epilogue, BN <= 128): after a tile's last MMA the consumers wait until the staging tile behind
// the stage ring is free, store their raw accumulators there, arrive on staged_full and start the next tile; warps 1-3
// of warpgroup 0 walk the same tile sequence, run each tile's epilogue from the staging tile and arrive on
// staged_free. The epilogue then overlaps the next tile's MMAs instead of holding up the tensor cores.
// p.epi_tma = 1 (with p.epi_op = 1): the TMA epilogue (see EpiMaps): one epilogue thread loads each tile's residual /
// GELU' source into the staging tile during its MMAs and stores the consumers' results from there by TMA.
// p.epi_op = 0: the consumers run the epilogue from their registers after the mainloop.
template <bool B_MN, int BN, int PL>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_persistent_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const __grid_constant__ CUtensorMap tmBlo, const __grid_constant__ CUtensorMap tmAlo,
                       const __grid_constant__ EpiMaps em, const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[MAX_STAGES];
  __shared__ __align__(8) uint64_t empty_bar[MAX_STAGES];
  __shared__ __align__(8) uint64_t staged_full, staged_free;

  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  const int wg = threadIdx.x >> 7;
  using S = StageLayout<B_MN, BN, PL>;
  const bool staged = BN <= 128 && p.epi_op == 1;
  const bool tma_epi = staged && p.epi_tma == 1 && BN % EPI_PANEL == 0;
  const int nstages = p.num_stages;
  const int m_tiles = p.kind == GEMM_CONV ? p.nimg * p.tiles_h * p.tiles_w : (p.M + BLOCK_M - 1) / BLOCK_M;
  const int n_tiles = (p.N + BN - 1) / BN;
  const int num_tiles = m_tiles * n_tiles * p.nz1 * p.nz2 * p.nsplit;
  // Tile order: bands of RASTER_N column tiles; within a band the band's columns fastest, then m. The CTAs resident at
  // one time then cover ~132 / RASTER_N row tiles x RASTER_N column tiles, so A is read from HBM once per band instead
  // of once per column tile. Each output element's sum is the same in any tile order.
  auto coord = [&](int t) {
    const int per_z = m_tiles * n_tiles;
    const int z = t / per_z;
    const int r = t - z * per_z;
    const int band = r / (m_tiles * RASTER_N);
    const int in_band = r - band * (m_tiles * RASTER_N);
    const int width = min(RASTER_N, n_tiles - band * RASTER_N);
    return tile_coord(p, in_band / width, band * RASTER_N + in_band % width, z, BN);
  };

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    if (PL & PL_BLO) prefetch_tmap(&tmBlo);
    if (PL & PL_ALO) prefetch_tmap(&tmAlo);
    for (int s = 0; s < nstages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    mbar_init(&staged_full, 256);  // every consumer thread
    mbar_init(&staged_free, tma_epi ? 1 : EPI_THREADS);
    fence_barrier_init();
  }
  __syncthreads();
  uint8_t* stg = smem + nstages * S::bytes;

  if (wg == 0) {
    // =========================== TMA producer ===========================
    auto produce = [&] {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const TileCoord c = coord(t);
        for (int kb = c.kb_begin; kb < c.kb_end; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sA = smem + stage * S::bytes;
          uint64_t* bar = &full_bar[stage];
          mbar_expect_tx(bar, static_cast<uint32_t>(S::bytes));
          load_stage<false, B_MN, BN, PL>(p, &tmA, &tmB, &tmBlo, &tmAlo, sA, bar, kb, c.m0, c.n0, c.z1, c.z2, c.img,
                                          c.th, c.tw);
          if (++stage == nstages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    };
    // (each branch keeps its own register budget: code after a join would be compiled for the smaller one)
    if (!staged) {
      reg_dealloc<40>();
      if (threadIdx.x == 0) produce();
    } else if constexpr (BN <= 128) {
      reg_dealloc<152>();
      if (threadIdx.x == 0) {
        produce();
      } else if (tma_epi) {
        // =========================== epilogue thread (TMA) ===========================
        // Phase i of staged_free completes when tile i's source is in the staging tile (at once without a source) and
        // the stores of tile i - 1 have read it; tile i + 1's source load is issued as soon as tile i's stores have
        // read the staging tile, so it lands while the consumers run tile i + 1's MMAs.
        if (threadIdx.x == 32) {
          if (p.residual != nullptr || p.gelu_grad_src != nullptr) prefetch_tmap(&em.src);
          uint32_t sphase = 0;
          if (blockIdx.x < num_tiles) epi_load_source<BN>(p, em, stg, &staged_free, coord(blockIdx.x));
          for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
            mbar_wait(&staged_full, sphase);
            sphase ^= 1;
            epi_store_tile<BN>(p, em, stg, coord(t));
            bulk_wait_read();
            if (t + static_cast<int>(gridDim.x) < num_tiles)
              epi_load_source<BN>(p, em, stg, &staged_free, coord(t + gridDim.x));
          }
          bulk_wait_all();
        }
      } else if (threadIdx.x >= 32) {
        // =========================== epilogue warps (staged) ===========================
        const float alpha = epi_alpha(p);
        const bool vec = ((p.ldc | p.c_z1_stride | p.c_z2_stride) & 3) == 0 &&
                         ((reinterpret_cast<uintptr_t>(p.out_f32) | reinterpret_cast<uintptr_t>(p.residual)) & 15) == 0 &&
                         ((reinterpret_cast<uintptr_t>(p.out_f16) | reinterpret_cast<uintptr_t>(p.out_act_f16)) & 7) == 0;
        uint32_t sphase = 0;
        for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
          const TileCoord c = coord(t);
          mbar_wait(&staged_full, sphase);
          epilogue_staged<BN>(p, reinterpret_cast<const float*>(stg), c, threadIdx.x - 32, alpha, vec);
          mbar_arrive(&staged_free);
          sphase ^= 1;
        }
      }
    }
    return;
  }

  // =========================== wgmma consumers ===========================
  if (staged) {
    reg_alloc<168>();
  } else {
    reg_alloc<232>();
  }
  const int cw = wg - 1;  // this warpgroup's 64 rows of every tile
  const int lane = threadIdx.x & 31;
  const float alpha = epi_alpha(p);
  float acc[BN / 2];
  int stage = 0;
  uint32_t phase = 0;
  uint32_t sphase = 0;
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    const TileCoord c = coord(t);
    int prev = -1;
    for (int i = c.kb_begin; i < c.kb_end; ++i) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_base = smem_u32(smem + stage * S::bytes);
      fence_regs<BN / 2>(acc);
      wgmma_arrive();
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k)
        mma_k16<false, B_MN, BN, PL>(acc, a_base + cw * 64 * 128, a_base + S::a_lo_off + cw * 64 * 128,
                                     a_base + A_STAGE_BYTES, a_base + S::b_lo_off, k,
                                     (i > c.kb_begin || k > 0) ? 1u : 0u);
      wgmma_commit();
      // the previous stage's MMAs have retired once at most this stage's group is in flight: free that slot
      wgmma_wait<1>();
      fence_regs<BN / 2>(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == nstages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    fence_regs<BN / 2>(acc);
    if (lane == 0) mbar_arrive(&empty_bar[prev]);
    if constexpr (BN <= 128) {
      if (tma_epi) {
        mbar_wait(&staged_free, sphase);  // this tile's source has landed, the previous tile's stores have read it
        fold_rows<BN>(p, stg, acc, c.n0, cw * 64, alpha);
        fence_proxy_async();  // before the TMA stores read the results
        mbar_arrive(&staged_full);
        sphase ^= 1;
        continue;
      }
      if (staged) {
        mbar_wait(&staged_free, sphase ^ 1);  // the epilogue warps are done with the previous tile
        stage_rows<BN>(reinterpret_cast<float*>(stg), acc, cw * 64);
        mbar_arrive(&staged_full);
        sphase ^= 1;
        continue;
      }
    }
    // =========================== epilogue (the producer already loads the next tile) ===========================
    store_rows<BN>(p, acc, c, cw * 64, alpha);
  }
}

// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int encode_tmap(CUtensorMap* out, const TmapSpec& s, bool f32 = false) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return -1;
  cuuint64_t gdim[4], gstr[3];
  cuuint32_t box[4], estr[4] = {1, 1, 1, 1};
  for (int i = 0; i < 4; ++i) {
    gdim[i] = s.dims[i];
    box[i] = s.box[i];
  }
  for (int i = 0; i < 3; ++i) gstr[i] = s.strides[i + 1] * (f32 ? 4 : 2);  // bytes
  CUresult r = fn(out, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(s.ptr), gdim, gstr, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr,
            "[mdm_b200] cuTensorMapEncodeTiled failed (%d): ptr=%p dims=(%llu,%llu,%llu,%llu) "
            "strides=(%llu,%llu,%llu,%llu) box=(%u,%u,%u,%u)\n",
            static_cast<int>(r), s.ptr, (unsigned long long)s.dims[0], (unsigned long long)s.dims[1],
            (unsigned long long)s.dims[2], (unsigned long long)s.dims[3],
            (unsigned long long)s.strides[0], (unsigned long long)s.strides[1],
            (unsigned long long)s.strides[2], (unsigned long long)s.strides[3], s.box[0], s.box[1],
            s.box[2], s.box[3]);
    return -2;
  }
  return 0;
}

// Tensor map of an epilogue buffer (see EpiMaps): dims / strides (elements) of dims 1-3, a 32-column panel box,
// zero fill outside the tensor on loads, clipping on stores.
int encode_epi_map(CUtensorMap* out, const void* ptr, bool f32, const uint64_t* dims, const uint64_t* strides,
                   const uint32_t* box) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return -1;
  const int esz = f32 ? 4 : 2;
  cuuint64_t gdim[4], gstr[3];
  cuuint32_t bx[4], estr[4] = {1, 1, 1, 1};
  for (int i = 0; i < 4; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
  }
  for (int i = 0; i < 3; ++i) gstr[i] = strides[i] * esz;
  CUresult r = fn(out, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr),
                  gdim, gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  f32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -2;
}

constexpr int TMA_EPI_MAX_KBLOCKS = 8;  // see launch_gemm

// Whether the TMA epilogue can serve p (tile width already rounded), and if so its tensor maps.
bool epi_tma_maps(const GemmParams& p, EpiMaps* em) {
  const bool uses32 = p.residual != nullptr || p.out_f32 != nullptr;
  const bool uses16 = p.gelu_grad_src != nullptr || p.out_f16 != nullptr || p.out_act_f16 != nullptr;
  // (3x3 convs have at least nine k blocks and no GELU, so none qualifies: conv64.fwd measured 10 % slower)
  if (p.kind != GEMM_PLAIN || uses32 == uses16 || p.atomic || p.block_n % EPI_PANEL != 0 || p.block_n > 128)
    return false;
  const long long esz = uses32 ? 4 : 2;
  const void* bufs[] = {p.residual, p.out_f32, p.gelu_grad_src, p.out_f16, p.out_act_f16};
  for (const void* b : bufs)
    if ((reinterpret_cast<uintptr_t>(b) & 15) != 0) return false;
  uint64_t dims[4], str[3];
  const uint32_t box[4] = {EPI_PANEL, BLOCK_M, 1, 1};
  if (p.ldc < p.N || p.N < 1 || p.M < 1) return false;
  // a batch dimension of one is never stepped: any valid stride will do
  const long long z1 = p.nz1 > 1 ? p.c_z1_stride : p.ldc * p.M;
  const long long z2 = p.nz2 > 1 ? p.c_z2_stride : z1 * p.nz1;
  if (z1 <= 0 || z2 <= 0) return false;
  const long long s[3] = {p.ldc, z1, z2};
  const long long d[4] = {p.N, p.M, p.nz1, p.nz2};
  for (int i = 0; i < 4; ++i) dims[i] = static_cast<uint64_t>(d[i]);
  for (int i = 0; i < 3; ++i) str[i] = static_cast<uint64_t>(s[i]);
  for (int i = 0; i < 3; ++i)
    if ((str[i] * esz) % 16 != 0 || str[i] * esz >= (1ull << 40)) return false;
  const void* src = uses32 ? static_cast<const void*>(p.residual) : p.gelu_grad_src;
  if (src != nullptr && encode_epi_map(&em->src, src, uses32, dims, str, box) != 0) return false;
  if (p.out_f32 != nullptr && encode_epi_map(&em->o32, p.out_f32, true, dims, str, box) != 0) return false;
  if (p.out_f16 != nullptr && encode_epi_map(&em->o16, p.out_f16, false, dims, str, box) != 0) return false;
  if (p.out_act_f16 != nullptr && encode_epi_map(&em->oact, p.out_act_f16, false, dims, str, box) != 0) return false;
  return true;
}

using GemmKernel = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, EpiMaps, GemmParams);

// majors (profile record): bit 1 = MN-major A, bit 0 = MN-major B, bit 2 = persistent kernel, bit 3 = staged epilogue,
// bit 4 = TMA epilogue
int launch_impl(GemmKernel k, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmBlo,
                const CUtensorMap& tmAlo, const EpiMaps& em, const GemmParams& p, int majors, int planes, dim3 grid,
                size_t smem, cudaStream_t stream) {
  static std::set<GemmKernel> attr_set;
  if (attr_set.count(k) == 0) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
    if (e != cudaSuccess) return static_cast<int>(e);
    attr_set.insert(k);
  }
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (g_profile) {
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    cudaEventRecord(e0, stream);
  }
  k<<<grid, NUM_THREADS, smem, stream>>>(tmA, tmB, tmBlo, tmAlo, em, p);
  if (g_profile) {
    cudaEventRecord(e1, stream);
    g_profile_events.emplace_back(e0, e1);
    g_profile_params.push_back(p);
    g_profile_majors.push_back(majors);
    g_profile_planes.push_back(planes);
  }
  ++g_launch_count;
  return static_cast<int>(cudaGetLastError());
}

// Kernel instance of (A_MN, B_MN, tile width, planes); nullptr for a combination the engine never launches.
template <bool B_MN, int BN>
GemmKernel persistent_kernel(int planes) {
  switch (planes) {
    case 0: return gemm_persistent_kernel<B_MN, BN, 0>;
    case PL_BLO: return gemm_persistent_kernel<B_MN, BN, PL_BLO>;
    case PL_ALO: return gemm_persistent_kernel<B_MN, BN, PL_ALO>;
    default: return gemm_persistent_kernel<B_MN, BN, PL_BLO | PL_ALO>;
  }
}
template <bool B_MN>
GemmKernel pick_kernel(bool persistent, int bn, int planes) {
  if (persistent) {
    switch (bn) {
      case 16: return persistent_kernel<B_MN, 16>(planes);
      case 32: return persistent_kernel<B_MN, 32>(planes);
      case 48: return persistent_kernel<B_MN, 48>(planes);
      case 64: return persistent_kernel<B_MN, 64>(planes);
      case 96: return persistent_kernel<B_MN, 96>(planes);
      case 128: return persistent_kernel<B_MN, 128>(planes);
      case 192: return persistent_kernel<B_MN, 192>(planes);
      default: return persistent_kernel<B_MN, 256>(planes);
    }
  }
  if (planes != 0) return nullptr;  // MN-major A (weight gradients) carries no lo planes
  switch (bn) {
    case 16: return gemm_tc_kernel<B_MN, 16>;
    case 32: return gemm_tc_kernel<B_MN, 32>;
    case 48: return gemm_tc_kernel<B_MN, 48>;
    case 64: return gemm_tc_kernel<B_MN, 64>;
    case 96: return gemm_tc_kernel<B_MN, 96>;
    case 128: return gemm_tc_kernel<B_MN, 128>;
    case 192: return gemm_tc_kernel<B_MN, 192>;
    default: return gemm_tc_kernel<B_MN, 256>;
  }
}

// The tile widths the kernel is instantiated for; a requested width runs on the next one up (the extra
// columns are outside the output and never stored).
int tile_width(int block_n) {
  const int widths[] = {16, 32, 48, 64, 96, 128, 192, 256};
  for (int w : widths)
    if (block_n <= w) return w;
  return 256;
}

}  // namespace

int launch_gemm(const TmapSpec& A, const TmapSpec& Bin, int a_mn, int b_mn, const GemmParams& pin,
                cudaStream_t stream, const void* b_lo, const void* a_lo) {
  GemmParams p = pin;
  if (p.block_n < 16 || p.block_n > 256 || (p.block_n % 16) != 0) return -10;
  if (p.nz1 < 1) p.nz1 = 1;
  if (p.nz2 < 1) p.nz2 = 1;
  if (p.nsplit < 1) p.nsplit = 1;
  if (p.num_kblocks < 1) return -11;
  if (p.nsplit > p.num_kblocks) p.nsplit = p.num_kblocks;
  // every split must own at least one k block
  while (p.nsplit > 1 && (p.nsplit - 1) * ((p.num_kblocks + p.nsplit - 1) / p.nsplit) >= p.num_kblocks)
    --p.nsplit;
  if (p.atomic == 0 && p.nsplit != 1) return -12;
  if (p.atomic && (p.out_f16 != nullptr || p.out_act_f16 != nullptr || p.out_f32 == nullptr)) return -16;

  p.block_n = tile_width(p.block_n);
  TmapSpec B = Bin;
  if (!b_mn) B.box[1] = static_cast<uint32_t>(p.block_n);  // K-major B: one box of block_n rows per stage
  alignas(64) CUtensorMap tmA, tmB;
  if (encode_tmap(&tmA, A) != 0) return -20;
  if (encode_tmap(&tmB, B) != 0) return -21;
  // the lo plane of a split B (weights): same geometry, its own base address (weight GEMMs: plain or 3x3 conv)
  const int b_split = (b_lo != nullptr && p.kind != GEMM_CONV_WGRAD) ? 1 : 0;
  alignas(64) CUtensorMap tmBlo = tmB;
  if (b_split) {
    TmapSpec Blo = B;
    Blo.ptr = b_lo;
    if (encode_tmap(&tmBlo, Blo) != 0) return -23;
  }
  const int a_split = (a_lo != nullptr && !a_mn && p.kind != GEMM_CONV_WGRAD) ? 1 : 0;
  alignas(64) CUtensorMap tmAlo = tmA;
  if (a_split) {
    TmapSpec Alo = A;
    Alo.ptr = a_lo;
    if (encode_tmap(&tmAlo, Alo) != 0) return -24;
  }

  if (p.kind != GEMM_CONV_WGRAD || p.kfactor < 1) p.kfactor = 1;
  const int kf = p.kfactor;
  if (kf > 1 && (!a_mn || !b_mn || p.PW * p.PH != 64 * kf || kf > 4)) return -15;
  if (p.kind == GEMM_CONV_WGRAD && !a_mn) return -15;  // dY patches are MN-major
  int m_tiles;
  if (p.kind == GEMM_CONV) {
    m_tiles = p.nimg * p.tiles_h * p.tiles_w;
  } else {
    m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  }
  const int n_tiles = (p.N + p.block_n - 1) / p.block_n;

  const int nb_alloc = b_mn ? ((p.block_n + 63) / 64) * 64 : p.block_n;
  const int stage_bytes =
      kf > 1 ? ((p.M <= 64 ? 1 : 2) + nb_alloc / 64) * SLAB_BYTES * kf : A_STAGE_BYTES * (1 + a_split) + nb_alloc * 128 * (1 + b_split);
  // one CTA per SM (384 threads at the consumers' register budget): the whole shared memory goes to the pipeline,
  // less the staging tile of a staged epilogue
  const int per = (p.num_kblocks + p.nsplit - 1) / p.nsplit;
  auto ring = [&](int reserved) { return std::min({(SMEM_LIMIT - 1024 - reserved) / stage_bytes, MAX_STAGES, per}); };
  int stages = ring(0);
  if (stages < 1) return -13;

  // The weight products (K-major A: linears, 1x1 and 3x3 convs forward and data gradient) run persistent; weight
  // gradients (MN-major A: split-K with fp32 atomics, 3x3 wgrad with tall stages) keep one tile per CTA.
  const bool persistent = !a_mn;
  // Staged epilogue (gemm_persistent_kernel) for tiles up to 128 columns, where the staging tile still leaves a ring
  // of three stages (or every k block of a short contraction): with two, the producer can no longer load a stage ahead
  // of the two the consumers hold, and the MMAs wait on TMA. Epilogues that evaluate the erf-GELU or its derivative
  // per element keep the in-register path: on three warps that arithmetic outlasts the next tile's mainloop (the FFN
  // up-projection and its data gradient ran up to 32 % slower staged on an H100). Split-K atomics keep it too.
  // The TMA epilogue (staged, with the residual / GELU' source loaded into the staging tile and the results stored by
  // TMA; see EpiMaps) where its tensor maps can describe the epilogue buffers, for GELU / GELU' epilogues and for
  // contractions of at most TMA_EPI_MAX_KBLOCKS k blocks. Measured on an H100 (tests/profile_gemm_epilogue.py): the FFN
  // up-projection and its GELU' data gradient ran 20-39 % faster, with GELU / GELU' on the consumers; K = 512
  // products 11-13 % faster; but K >= 768 products without GELU 3-15 % slower than the staged path below (the
  // consumers' fold does not explain it; the cause is not found), so those keep it. Its unpadded staging tile is
  // smaller, so it too keeps three stages.
  const bool gelu_math = (p.act == ACT_GELU && p.out_act_f16 != nullptr) || p.gelu_grad_src != nullptr;
  alignas(64) EpiMaps em;
  memset(&em, 0, sizeof(em));
  const int staging_tma = BLOCK_M * p.block_n * 4;
  const bool tma = persistent && (gelu_math || per <= TMA_EPI_MAX_KBLOCKS) && ring(staging_tma) >= std::min(3, per) &&
                   epi_tma_maps(p, &em);
  const int staging = tma ? staging_tma : BLOCK_M * (p.block_n + STAGE_PAD) * 4;
  const bool staged =
      tma || (persistent && p.block_n <= 128 && !p.atomic && !gelu_math && ring(staging) >= std::min(3, per));
  if (staged) stages = ring(staging);
  p.num_stages = stages;
  const size_t smem = static_cast<size_t>(stages) * stage_bytes + 1024 + (staged ? staging : 0);
  p.epi_tma = tma ? 1 : 0;
  p.epi_op = staged ? 1 : 0;
  p.cluster = 1;
  p.pair = 0;

  const int planes = (b_split ? PL_BLO : 0) | (a_split ? PL_ALO : 0);
  GemmKernel k = b_mn ? pick_kernel<true>(persistent, p.block_n, planes) : pick_kernel<false>(persistent, p.block_n, planes);
  if (k == nullptr) return -17;
  const int majors = (a_mn ? 2 : 0) | (b_mn ? 1 : 0) | (persistent ? 4 : 0) | (staged ? 8 : 0) | (tma ? 16 : 0);
  const long long tiles = static_cast<long long>(m_tiles) * n_tiles * p.nz1 * p.nz2 * p.nsplit;
  if (persistent) {
    if (tiles > INT_MAX) return -14;
    static const int num_sms = [] {
      int dev = 0, n = 0;
      cudaGetDevice(&dev);
      cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
      return n;
    }();
    const long long ctas = std::min<long long>(tiles, std::max(1, num_sms - g_sm_reserve));
    return launch_impl(k, tmA, tmB, tmBlo, tmAlo, em, p, majors, planes, dim3(static_cast<unsigned>(ctas)), smem, stream);
  }
  dim3 grid(m_tiles, n_tiles, p.nz1 * p.nz2 * p.nsplit);
  if (grid.y > 65535 || grid.z > 65535) return -14;
  return launch_impl(k, tmA, tmB, tmBlo, tmAlo, em, p, majors, planes, grid, smem, stream);
}

}  // namespace mdm
