// Fused masked self-attention over text tokens: the SelfAttention1D of the lm_head layers (reference
// models/unet.py:316-388) on a qkv16 [B*T][3D] tensor laid out like the spatial one (q | k | v thirds, 8 heads of
// d = D/8 columns each), with an optional key mask [B][T]:
//   o = softmax((q / d^1/4) (k / d^1/4)^T, masked keys -> -inf) v
// Head widths up to 256 (d a multiple of 8); the hot shape is d = 256 with T <= 128 tokens, one key tile.
//
// Forward: one CTA per (128 queries, head, sample), two warpgroups of 64 query rows. Q, one 128-key chunk of K and
// of V are staged by TMA (3 x 64 KB at d = 256). S = Q K^T (over all of d) goes to registers; P is formed there and
// fed as the register A operand of O = P V, which runs per 128-column half of d so that O never takes more than 64
// fp32 registers. With one key chunk P is computed once and serves both halves; with several chunks a first pass
// finds the row maxima and every half recomputes S (P = 2^(s - m) unnormalised, O divided by the row sum at the end).
// Backward: one CTA per (128 keys, head, sample), looping over 64-query tiles: P^T and dS^T = P^T (dP^T - D) alpha in
// registers, dV += P^T dO and dK += dS^T Q for one 128-column half of d at a time (the query loop runs once per half),
// dQ = dS K from dS^T in shared memory, added to an fp32 buffer by atomics in the first half's loop.
// A sample whose keys are all masked has no softmax (the reference gives NaN): its outputs and gradients are zero.
#include <math.h>

#include <type_traits>

#include "attn_common.cuh"
#include "engine.cuh"
#include "mdm_b200.h"
#include "ptx.cuh"

namespace mdm {
using namespace ptx;
using namespace attn;

namespace {

constexpr int THREADS = 256;        // two warpgroups
constexpr int TILE = 128;           // queries per forward CTA, keys per chunk / per backward CTA
constexpr int QT = 64;              // queries per backward tile
constexpr int QB_BYTES = QT * 128;  // one [64 rows][64 fp16] k-block

struct TokParams {
  int T, d, heads, D;
  float alpha;        // 1/sqrt(d)
  float alpha_log2e;  // alpha * log2(e)
  const float* mask;  // [B][T] key mask or null
  __half* o16;        // [B*T][D]
  float* stats;       // [B][heads][T][2] = (row max of s * alpha * log2 e, 1/l)
  const float* Dterm; // [B][heads][T]
  float* dq32;        // [B*T][D], accumulated atomically (zero on entry)
  __half* dqkv16;     // [B*T][3D]
};

// DN: the head width rounded up to 16 (to 256 above 128); the products with d columns run in halves of ON columns
template <int DN>
struct Shape {
  static constexpr int KBK = (DN + 63) / 64;       // 64-wide k-blocks of d
  static constexpr int ON = DN > 128 ? 128 : DN;   // columns per half
  static constexpr int NH = DN / ON;               // halves
  static constexpr size_t FWD_SMEM = 3ull * KBK * KB_BYTES + 1024;
  static constexpr size_t BWD_SMEM = 2ull * KBK * KB_BYTES + 2ull * KBK * QB_BYTES + KB_BYTES + 1024;
};

// ------------------------------------------------------------------------------------------ forward
template <int DN>
__global__ void __launch_bounds__(THREADS, 1)
tok_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQKV, const TokParams p) {
  using Sh = Shape<DN>;
  constexpr int KBK = Sh::KBK, ON = Sh::ON, NH = Sh::NH;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t q_bar, kv_bar;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int hd = blockIdx.y, b = blockIdx.z;
  const int q0 = blockIdx.x * TILE;
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + KBK * KB_BYTES;
  uint8_t* sV = sK + KBK * KB_BYTES;

  if (tid == 0) {
    prefetch_tmap(&tmQKV);
    mbar_init(&q_bar, 1);
    mbar_init(&kv_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  const int nchunks = (p.T + TILE - 1) / TILE;
  const bool single = nchunks == 1;
  // K (+ V) chunk loads, one buffer: with several chunks items 0 .. nchunks - 1 are the max pass (K only), then every
  // half walks the chunks again with V
  auto issue = [&](int i) {
    const bool with_v = single || i >= nchunks;
    const int key0 = (i % nchunks) * TILE;
    mbar_expect_tx(&kv_bar, (with_v ? 2 : 1) * KBK * KB_BYTES);
    for (int kb = 0; kb < KBK; ++kb) {
      tma_load_4d(sK + kb * KB_BYTES, &tmQKV, &kv_bar, kb * 64, key0, p.heads + hd, b);
      if (with_v) tma_load_4d(sV + kb * KB_BYTES, &tmQKV, &kv_bar, kb * 64, key0, 2 * p.heads + hd, b);
    }
  };
  if (tid == 0) {
    mbar_expect_tx(&q_bar, KBK * KB_BYTES);
    for (int kb = 0; kb < KBK; ++kb) tma_load_4d(sQ + kb * KB_BYTES, &tmQKV, &q_bar, kb * 64, q0, hd, b);
    issue(0);
  }
  mbar_wait(&q_bar, 0);

  const uint32_t qa = smem_u32(sQ) + wg * 64 * 128, ka = smem_u32(sK), va = smem_u32(sV);
  const int col_l = 2 * (lane & 3);
  const float* mk = p.mask != nullptr ? p.mask + static_cast<long long>(b) * p.T : nullptr;
  float m2[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float v[TILE / 2];
  int item = 0;
  uint32_t phase = 0;
  // S of the chunk in flight into v (masked and out-of-range keys -inf); the buffer is refilled once both
  // warpgroups are done with the previous item
  auto scores = [&](int c) {
    if (item > 0) {
      __syncthreads();
      if (tid == 0) issue(item);
    }
    ++item;
    mbar_wait(&kv_bar, phase);
    phase ^= 1;
    fence_regs<TILE / 2>(v);
    wgmma_arrive();
#pragma unroll
    for (int kb = 0; kb < KBK; ++kb)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        Wgmma<TILE>::ss<0, 0>(v, desc_k(qa + kb * KB_BYTES, k), desc_k(ka + kb * KB_BYTES, k), (kb | k) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<TILE / 2>(v);
    const int key0 = c * TILE;
    if (key0 + TILE > p.T || mk != nullptr) {
#pragma unroll
      for (int e = 0; e < TILE / 2; ++e) {
        const int key = key0 + 8 * (e >> 2) + col_l + (e & 1);
        const bool ok = key < p.T && (mk == nullptr || mk[key] != 0.f);
        v[e] = ok ? v[e] : -INFINITY;
      }
    }
  };
  // running row maximum, in units of log2 (alpha > 0: the maximum commutes with the scaling)
  auto row_max = [&]() {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float cm = -INFINITY;
#pragma unroll
      for (int j = 0; j < TILE / 8; ++j) cm = fmaxf(cm, fmaxf(v[4 * j + 2 * h], v[4 * j + 2 * h + 1]));
      m2[h] = fmaxf(m2[h], quad_max(cm) * p.alpha_log2e);
    }
  };
  // v <- 2^(s alpha log2e - m) (0 for masked keys); the row sums are added to l when asked
  auto exponentiate = [&](bool sum_rows) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float mref = m2[h] > -INFINITY ? m2[h] : 0.f;
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < TILE / 8; ++j)
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          float& x = v[4 * j + 2 * h + u];
          x = ex2_approx(fmaf(x, p.alpha_log2e, -mref));
          sum += x;
        }
      sum = quad_sum(sum);
      if (sum_rows) l[h] += sum;
    }
  };

  if (single) {
    scores(0);
    row_max();
    exponentiate(true);
#pragma unroll
    for (int e = 0; e < TILE / 2; ++e) {
      const float il = l[(e >> 1) & 1];
      v[e] *= il > 0.f ? 1.0f / il : 0.f;
    }
  } else {
    for (int c = 0; c < nchunks; ++c) {
      scores(c);
      row_max();
    }
  }
  for (int half = 0; half < NH; ++half) {
    float o[ON / 2];
#pragma unroll
    for (int i = 0; i < ON / 2; ++i) o[i] = 0.f;
    for (int c = 0; c < nchunks; ++c) {
      if (!single) {
        scores(c);
        exponentiate(half == 0);  // P stays unnormalised (<= 1); O is divided by l below
      }
      fence_regs<ON / 2>(o);
      wgmma_arrive();
#pragma unroll
      for (int t = 0; t < TILE / 16; ++t) {  // 128 keys = 8 x 16
        uint32_t a[4];
        frag_a(v, t, a);
        Wgmma<ON>::template rs<1>(o, a, desc_mn(va + half * 2 * KB_BYTES, t, KB_BYTES), (c | t) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<ON / 2>(o);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = q0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
      if (q >= p.T) continue;
      const float os = single ? 1.f : (l[h] > 0.f ? 1.0f / l[h] : 0.f);
      __half* dst = p.o16 + (static_cast<long long>(b) * p.T + q) * p.D + hd * p.d + half * ON;
#pragma unroll
      for (int j = 0; j < ON / 8; ++j) {
        const int col = 8 * j + col_l;
        if (half * ON + col < p.d)
          *reinterpret_cast<__half2*>(dst + col) = __floats2half2_rn(o[4 * j + 2 * h] * os, o[4 * j + 2 * h + 1] * os);
      }
    }
  }
  if (p.stats != nullptr && (lane & 3) == 0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = q0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
      if (q >= p.T) continue;
      float* st = p.stats + ((static_cast<long long>(b) * p.heads + hd) * p.T + q) * 2;
      st[0] = m2[h];
      st[1] = l[h] > 0.f ? 1.0f / l[h] : 0.f;
    }
  }
}

// ------------------------------------------------------------------------------------------ backward
// D[b][h][q] = sum_c dO[q][h d + c] * O[q][h d + c], one warp per token row
__global__ void tok_attn_bwd_prep_kernel(const __half* __restrict__ dO, const __half* __restrict__ o16,
                                         float* __restrict__ Dterm, int T, int D, int heads, int d, long long rows) {
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const long long b = row / T;
  const int q = static_cast<int>(row - b * T);
  for (int hd = 0; hd < heads; ++hd) {
    float s = 0.f;
    for (int c = lane; c < d; c += 32) {
      const long long o = row * D + hd * d + c;
      s += __half2float(dO[o]) * __half2float(o16[o]);
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) Dterm[(b * heads + hd) * T + q] = s;
  }
}

// Warpgroup g owns keys 64 g .. 64 g + 63 of the CTA's 128: S^T = K Q^T and dP^T = V dO^T for a 64-query tile in
// registers, P^T and dS^T formed in place and fed as register A operands to dV += P^T dO and dK += dS^T Q. dQ = dS K
// reads dS^T from shared memory: with two halves warpgroup g takes column half g over all 128 keys, with one half
// it takes its own 64 keys over all columns (both add into dq32).
template <int DN>
__global__ void __launch_bounds__(THREADS, 1)
tok_attn_bwd_kernel(const __grid_constant__ CUtensorMap tmKV, const __grid_constant__ CUtensorMap tmQ,
                    const __grid_constant__ CUtensorMap tmDO, const TokParams p) {
  using Sh = Shape<DN>;
  constexpr int KBK = Sh::KBK, ON = Sh::ON, NH = Sh::NH;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t kv_bar, qd_bar;
  __shared__ float s_m2[QT], s_il[QT], s_nD[QT];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int hd = blockIdx.y, b = blockIdx.z;
  const int key0 = blockIdx.x * TILE;
  uint8_t* sK = smem;
  uint8_t* sV = sK + KBK * KB_BYTES;
  uint8_t* sQ = sV + KBK * KB_BYTES;
  uint8_t* sDO = sQ + KBK * QB_BYTES;
  uint8_t* sDS = sDO + KBK * QB_BYTES;  // dS^T: [128 keys][64 queries], 128B-swizzled

  if (tid == 0) {
    prefetch_tmap(&tmKV);
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmDO);
    mbar_init(&kv_bar, 1);
    mbar_init(&qd_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto load_qd = [&](int q0) {
    mbar_expect_tx(&qd_bar, 2 * KBK * QB_BYTES);
    for (int kb = 0; kb < KBK; ++kb) {
      tma_load_4d(sQ + kb * QB_BYTES, &tmQ, &qd_bar, kb * 64, q0, hd, b);
      tma_load_4d(sDO + kb * QB_BYTES, &tmDO, &qd_bar, kb * 64, q0, hd, b);
    }
  };
  if (tid == 0) {
    mbar_expect_tx(&kv_bar, 2 * KBK * KB_BYTES);
    for (int kb = 0; kb < KBK; ++kb) {
      tma_load_4d(sK + kb * KB_BYTES, &tmKV, &kv_bar, kb * 64, key0, p.heads + hd, b);
      tma_load_4d(sV + kb * KB_BYTES, &tmKV, &kv_bar, kb * 64, key0, 2 * p.heads + hd, b);
    }
    load_qd(0);
  }
  const float* mk = p.mask != nullptr ? p.mask + static_cast<long long>(b) * p.T : nullptr;
  const int col_l = 2 * (lane & 3);
  const int krow = wg * 64 + wq * 16 + (lane >> 2);  // tile-local key of accumulator rows h = 0 (+ 8 for h = 1)
  bool kok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int key = key0 + krow + 8 * h;
    kok[h] = key < p.T && (mk == nullptr || mk[key] != 0.f);
  }
  const uint32_t ka = smem_u32(sK), va = smem_u32(sV), qa = smem_u32(sQ), da = smem_u32(sDO), sa = smem_u32(sDS);
  mbar_wait(&kv_bar, 0);
  uint32_t qd_phase = 0;
  const int nq = (p.T + QT - 1) / QT;
  const long long bh = static_cast<long long>(b) * p.heads + hd;
  for (int half = 0; half < NH; ++half) {
    float dv[ON / 2], dk[ON / 2];
#pragma unroll
    for (int i = 0; i < ON / 2; ++i) dv[i] = dk[i] = 0.f;
    for (int it = 0; it < nq; ++it) {
      const int q0 = it * QT;
      if (tid < QT) {
        const int q = q0 + tid;
        float m2 = 0.f, inv_l = 0.f, Dq = 0.f;
        if (q < p.T) {
          m2 = p.stats[(bh * p.T + q) * 2];
          inv_l = p.stats[(bh * p.T + q) * 2 + 1];
          Dq = p.Dterm[bh * p.T + q];
        }
        if (!(inv_l > 0.f)) {  // row outside the sequence or fully masked: P = 0 without inf arithmetic
          inv_l = 0.f;
          m2 = 0.f;
        }
        s_m2[tid] = m2;
        s_il[tid] = inv_l;
        s_nD[tid] = -Dq * p.alpha;
      }
      __syncthreads();
      mbar_wait(&qd_bar, qd_phase);
      qd_phase ^= 1;
      float s[QT / 2], dp[QT / 2];
      fence_regs<QT / 2>(s);
      fence_regs<QT / 2>(dp);
      wgmma_arrive();
#pragma unroll
      for (int kb = 0; kb < KBK; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          Wgmma<QT>::ss<0, 0>(s, desc_k(ka + kb * KB_BYTES + wg * 64 * 128, k), desc_k(qa + kb * QB_BYTES, k),
                              (kb | k) ? 1u : 0u);
          Wgmma<QT>::ss<0, 0>(dp, desc_k(va + kb * KB_BYTES + wg * 64 * 128, k), desc_k(da + kb * QB_BYTES, k),
                              (kb | k) ? 1u : 0u);
        }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<QT / 2>(s);
      fence_regs<QT / 2>(dp);
#pragma unroll
      for (int e = 0; e < QT / 2; ++e) {
        const int ql = 8 * (e >> 2) + col_l + (e & 1);  // tile-local query (column)
        float pe = ex2_approx(fmaf(s[e], p.alpha_log2e, -s_m2[ql])) * s_il[ql];
        pe = kok[(e >> 1) & 1] ? pe : 0.f;
        s[e] = pe;                                     // P^T
        dp[e] = pe * fmaf(dp[e], p.alpha, s_nD[ql]);  // dS^T = P^T (dP^T - D) / sqrt(d)
      }
      if (half == 0) {  // dS^T into shared memory for dQ
#pragma unroll
        for (int e = 0; e < QT / 2; e += 2) {
          const int kr = krow + 8 * ((e >> 1) & 1);
          const int qc = 8 * (e >> 2) + col_l;
          uint8_t* dst = sDS + kr * 128 + ((((qc >> 3) ^ (kr & 7))) << 4) + (qc & 7) * 2;
          *reinterpret_cast<uint32_t*>(dst) = pack_half2(dp[e], dp[e + 1]);
        }
      }
      fence_regs<ON / 2>(dv);
      fence_regs<ON / 2>(dk);
      wgmma_arrive();
#pragma unroll
      for (int t = 0; t < QT / 16; ++t) {  // contraction over the tile's 64 queries
        uint32_t a[4];
        const uint32_t scale = (it | t) ? 1u : 0u;
        frag_a(s, t, a);
        Wgmma<ON>::template rs<1>(dv, a, make_smem_desc_sw128(da + half * 2 * QB_BYTES + t * 2048, QB_BYTES, 1024), scale);
        frag_a(dp, t, a);
        Wgmma<ON>::template rs<1>(dk, a, make_smem_desc_sw128(qa + half * 2 * QB_BYTES + t * 2048, QB_BYTES, 1024), scale);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<ON / 2>(dv);
      fence_regs<ON / 2>(dk);
      if (half == 0) {
        fence_proxy_async();  // dS^T stores -> visible to wgmma
        __syncthreads();
        // dQ[q][c] = sum_k dS[q][k] K[k][c]  (A = dS, MN-major in the dS^T tile; B = K, MN-major)
        constexpr int KSTEPS = NH == 2 ? TILE / 16 : 64 / 16;
        const uint32_t a_base = NH == 2 ? sa : sa + wg * 64 * 128;
        const uint32_t b_base = NH == 2 ? ka + wg * 2 * KB_BYTES : ka + wg * 64 * 128;
        const int c_off = NH == 2 ? wg * ON : 0;
        float dq[ON / 2];
        fence_regs<ON / 2>(dq);
        wgmma_arrive();
#pragma unroll
        for (int t = 0; t < KSTEPS; ++t)
          Wgmma<ON>::template ss<1, 1>(dq, make_smem_desc_sw128(a_base + t * 2048, KB_BYTES, 1024),
                                       desc_mn(b_base, t, KB_BYTES), t ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs<ON / 2>(dq);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int q = q0 + wq * 16 + (lane >> 2) + 8 * h;
          if (q >= p.T) continue;
          float* dst = p.dq32 + (static_cast<long long>(b) * p.T + q) * p.D + hd * p.d + c_off;
#pragma unroll
          for (int j = 0; j < ON / 8; ++j) {
            const int col = 8 * j + col_l;
            if (c_off + col < p.d) {
              atomicAdd(dst + col, dq[4 * j + 2 * h]);
              atomicAdd(dst + col + 1, dq[4 * j + 2 * h + 1]);
            }
          }
        }
      }
      __syncthreads();  // Q / dO / dS^T and the row statistics are rewritten for the next tile
      if (tid == 0 && (half + 1 < NH || it + 1 < nq)) load_qd(it + 1 < nq ? (it + 1) * QT : 0);
    }
    // dK, dV of this key tile, columns of this half
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int key = key0 + krow + 8 * h;
      if (key >= p.T) continue;
      __half* base = p.dqkv16 + (static_cast<long long>(b) * p.T + key) * 3 * p.D + hd * p.d + half * ON;
#pragma unroll
      for (int j = 0; j < ON / 8; ++j) {
        const int col = 8 * j + col_l;
        if (half * ON + col < p.d) {
          *reinterpret_cast<__half2*>(base + p.D + col) = __floats2half2_rn(dk[4 * j + 2 * h], dk[4 * j + 2 * h + 1]);
          *reinterpret_cast<__half2*>(base + 2 * p.D + col) = __floats2half2_rn(dv[4 * j + 2 * h], dv[4 * j + 2 * h + 1]);
        }
      }
    }
  }
}

// Calls f(std::integral_constant<int, DN>): the head width rounded up to 16, and to 256 above 128.
template <typename F>
void with_token_width(int d, F&& f) {
  switch ((d + 15) / 16) {
    case 1: f(std::integral_constant<int, 16>()); break;
    case 2: f(std::integral_constant<int, 32>()); break;
    case 3: f(std::integral_constant<int, 48>()); break;
    case 4: f(std::integral_constant<int, 64>()); break;
    case 5: f(std::integral_constant<int, 80>()); break;
    case 6: f(std::integral_constant<int, 96>()); break;
    case 7: f(std::integral_constant<int, 112>()); break;
    case 8: f(std::integral_constant<int, 128>()); break;
    default: f(std::integral_constant<int, 256>()); break;
  }
}

TokParams make_params(const float* mask, int T, int D, int heads) {
  const int d = D / heads;
  MDM_CHECK(heads > 0 && D % heads == 0 && d % 8 == 0 && d >= 8 && d <= 256,
            "token attention: head width must be a multiple of 8 in [8, 256]");
  MDM_CHECK(T >= 1, "token attention: no tokens");
  TokParams p{};
  p.T = T; p.d = d; p.heads = heads; p.D = D;
  p.alpha = 1.0f / sqrtf(static_cast<float>(d));
  p.alpha_log2e = p.alpha * 1.4426950408889634f;
  p.mask = mask;
  return p;
}

}  // namespace

// ------------------------------------------------------------------------------------------ host API
void token_attention_forward(const __half* qkv, const float* mask, int B, int T, int D, int heads, __half* o16,
                             float* stats, cudaStream_t st) {
  TokParams p = make_params(mask, T, D, heads);
  p.o16 = o16;
  p.stats = stats;
  alignas(64) CUtensorMap mq;
  head_map(&mq, qkv, p.d, T, 3ll * D, 3 * heads, p.d, B, static_cast<long long>(T) * 3 * D);
  dim3 grid((T + TILE - 1) / TILE, heads, B);
  with_token_width(p.d, [&](auto dn) {
    constexpr int DN = decltype(dn)::value;
    constexpr size_t smem = Shape<DN>::FWD_SMEM;
    static bool attr = false;
    if (!attr) {
      MDM_CUDA(cudaFuncSetAttribute(tok_attn_fwd_kernel<DN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      attr = true;
    }
    tok_attn_fwd_kernel<DN><<<grid, THREADS, smem, st>>>(mq, p);
  });
  ++g_launch_count;
  MDM_CUDA(cudaGetLastError());
}

void token_attention_backward(const __half* qkv, const float* mask, const __half* dO, const __half* o16,
                              const float* stats, int B, int T, int D, int heads, float* Dterm, float* dq32,
                              __half* dqkv16, cudaStream_t st) {
  TokParams p = make_params(mask, T, D, heads);
  p.stats = const_cast<float*>(stats);
  p.Dterm = Dterm; p.dq32 = dq32; p.dqkv16 = dqkv16;
  const long long rows = static_cast<long long>(B) * T;
  tok_attn_bwd_prep_kernel<<<static_cast<unsigned>((rows + 7) / 8), 256, 0, st>>>(dO, o16, Dterm, T, D, heads, p.d,
                                                                                  rows);
  ++g_launch_count;
  MDM_CUDA(cudaMemsetAsync(dq32, 0, sizeof(float) * rows * D, st));
  alignas(64) CUtensorMap mkv, mq, mdo;
  head_map(&mkv, qkv, p.d, T, 3ll * D, 3 * heads, p.d, B, static_cast<long long>(T) * 3 * D);
  head_map(&mq, qkv, p.d, T, 3ll * D, 3 * heads, p.d, B, static_cast<long long>(T) * 3 * D, QT);
  head_map(&mdo, dO, p.d, T, D, heads, p.d, B, static_cast<long long>(T) * D, QT);
  dim3 grid((T + TILE - 1) / TILE, heads, B);
  with_token_width(p.d, [&](auto dn) {
    constexpr int DN = decltype(dn)::value;
    constexpr size_t smem = Shape<DN>::BWD_SMEM;
    static bool attr = false;
    if (!attr) {
      MDM_CUDA(cudaFuncSetAttribute(tok_attn_bwd_kernel<DN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      attr = true;
    }
    tok_attn_bwd_kernel<DN><<<grid, THREADS, smem, st>>>(mkv, mq, mdo, p);
  });
  ++g_launch_count;
  MDM_CUDA(cudaGetLastError());
  // dQ: fp32 accumulator -> fp16 into the q third of dqkv
  cast_rows_f16(dq32, dqkv16, rows, D, 3 * D, st);
}

}  // namespace mdm

// ------------------------------------------------------------------------------------------ C ABI (tests)
#define MDM_TRY(...)                  \
  try {                               \
    __VA_ARGS__;                      \
    return 0;                         \
  } catch (const std::exception& e) { \
    mdm::set_error("%s", e.what());   \
    return -1;                        \
  }

extern "C" {

int mdm_op_token_attention_fwd(const void* qkv16, const float* mask, int B, int T, int D, int heads, void* o16,
                               float* stats, mdm_stream_t stream) {
  MDM_TRY(mdm::token_attention_forward(static_cast<const __half*>(qkv16), mask, B, T, D, heads,
                                       static_cast<__half*>(o16), stats, static_cast<cudaStream_t>(stream)))
}

int mdm_op_token_attention_bwd(const void* qkv16, const float* mask, const void* dO16, const void* o16,
                               const float* stats, int B, int T, int D, int heads, float* Dterm, float* dq32,
                               void* dqkv16, mdm_stream_t stream) {
  MDM_TRY(mdm::token_attention_backward(static_cast<const __half*>(qkv16), mask, static_cast<const __half*>(dO16),
                                        static_cast<const __half*>(o16), stats, B, T, D, heads, Dterm, dq32,
                                        static_cast<__half*>(dqkv16), static_cast<cudaStream_t>(stream)))
}
}
