// Fused attention for the denoiser's SelfAttention blocks (reference models/unet.py:276-313):
//   h = softmax(q k^T / sqrt(d)) v  +  softmax(q k_c^T / sqrt(d)) v_c        (two independent softmaxes)
// with q,k,v = channel thirds of the qkv 1x1 conv, k_c,v_c = halves of kv_cond(LayerNorm(cond)),
// 8 heads of d = C/8 channels, optional token mask on the cross branch.
//
// Forward: one CTA per (128 queries, head, sample). Scores never leave the SM: S = Q K^T by
// wgmma into registers, exact two-pass softmax (pass A: row max / sum over all key chunks,
// pass B: recompute S, P = exp2(..)/l in fp16 registers, O += P V on the tensor core).
// Backward: one CTA per (128 keys, head, sample) looping over query tiles: recomputes P from the
// saved row statistics, dV += P^T dO, dP = dO V^T, dS = P (dP - D) alpha, dK += dS^T Q, dQ += dS K
// (fp32 atomics). All five products are wgmma on operands staged by TMA; P^T and dS^T feed the
// next products straight from registers, and dS^T is written once to smem for dQ.
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

constexpr int AT_THREADS = 256;   // forward: two warpgroups, 64 queries each
constexpr int BWD_THREADS = 256;  // backward: two warpgroups, 64 keys each
constexpr int TILE = 128;           // queries per CTA (fwd) / keys per CTA (bwd); key chunk size

struct AttnParams {
  int T, S, d, heads, B;
  int kblocks;        // ceil(d / 64)
  float alpha_log2e;  // (1/sqrt(d)) * log2(e)
  float alpha;
  const float* mask;  // [B][S] or null (cross branch)
  // forward outputs
  __half* h16;        // [B*T][C] summed output
  __half* oself16;    // [B*T][C] self branch only (training) or null
  float* stats;       // [B][heads][2 branches][T][2] = (m2, 1/l)
  int C;
  // backward
  const float* Dterm;  // [B][heads][2][T]
  float* dq32;         // [B*T][C] fp32, accumulated atomically (zero on entry)
  __half* dqkv16;      // [B*T][3C]: dK at +C, dV at +2C
  __half* dkv16;       // [B*S][2C]: dKc at +0, dVc at +C
};

// ------------------------------------------------------------------------------------------ forward
// Two warpgroups, 64 query rows each. S (64 x 128 keys) and O (64 x DN) live in registers; P goes from the S
// registers straight into the A operand of O += P V.
template <int DN>
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmQKVv,
                const __grid_constant__ CUtensorMap tmKV, const __grid_constant__ CUtensorMap tmKVv,
                const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t q_bar, kv_bar[2];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int qt = blockIdx.x, hd = blockIdx.y, b = blockIdx.z;
  const int q0 = qt * TILE;
  const int kbk = p.kblocks;
  const int stage_bytes = 2 * kbk * KB_BYTES;  // K then V
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + kbk * KB_BYTES;

  if (tid == 0) {
    prefetch_tmap(&tmQKV);
    prefetch_tmap(&tmQKVv);
    prefetch_tmap(&tmKV);
    prefetch_tmap(&tmKVv);
    mbar_init(&q_bar, 1);
    mbar_init(&kv_bar[0], 1);
    mbar_init(&kv_bar[1], 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (tid == 0) {
    mbar_expect_tx(&q_bar, kbk * KB_BYTES);
    for (int kb = 0; kb < kbk; ++kb) tma_load_4d(sQ + kb * KB_BYTES, &tmQKV, &q_bar, kb * 64, q0, hd, b);
  }
  uint32_t kv_phase[2] = {0, 0};
  bool o_started = false;

  // K / V chunk loads form one queue across passes and branches (two stages), so the first chunk of
  // the next pass or branch is already in flight while the current one finishes.
  const int nself = (p.T + TILE - 1) / TILE;
  const int ncross = p.S > 0 ? (p.S + TILE - 1) / TILE : 0;
  const int self_p0 = nself > 1 ? nself : 0;  // statistics-pass items of the self branch
  const int items_self = self_p0 + nself;
  const int cross_p0 = ncross > 1 ? ncross : 0;
  const int n_items = items_self + cross_p0 + ncross;
  auto issue_item = [&](int i) {
    const bool cross = i >= items_self;
    const int k = cross ? i - items_self : i;
    const int p0 = cross ? cross_p0 : self_p0;
    const bool with_v = k >= p0;
    const int key0 = (with_v ? k - p0 : k) * TILE;
    const int st = i & 1;
    uint8_t* dst = sKV + st * stage_bytes;
    mbar_expect_tx(&kv_bar[st], (with_v ? 2 : 1) * kbk * KB_BYTES);
    for (int kb = 0; kb < kbk; ++kb) {
      if (!cross) tma_load_4d(dst + kb * KB_BYTES, &tmQKV, &kv_bar[st], kb * 64, key0, p.heads + hd, b);
      else tma_load_4d(dst + kb * KB_BYTES, &tmKV, &kv_bar[st], kb * 64, key0, hd, b);
    }
    if (with_v) {
      for (int sl = 0; sl < kbk; ++sl) {
        if (!cross) tma_load_4d(dst + (kbk + sl) * KB_BYTES, &tmQKVv, &kv_bar[st], sl * 64, key0, 2 * p.heads + hd, b);
        else tma_load_4d(dst + (kbk + sl) * KB_BYTES, &tmKVv, &kv_bar[st], sl * 64, key0, p.heads + hd, b);
      }
    }
  };
  int item = 0;  // queue position of the chunk being consumed
  if (tid == 0 && n_items > 0) issue_item(0);
  mbar_wait(&q_bar, 0);

  const uint32_t qa = smem_u32(sQ) + wg * 64 * 128;  // this warpgroup's 64 query rows
  const int col_l = 2 * (lane & 3);
  float o[DN / 2];
#pragma unroll
  for (int i = 0; i < DN / 2; ++i) o[i] = 0.f;

  for (int branch = 0; branch < 2; ++branch) {
    const bool cross = branch == 1;
    const int nkeys = cross ? p.S : p.T;
    if (nkeys <= 0) continue;
    const int nchunks = (nkeys + TILE - 1) / TILE;
    const float* mk = (cross && p.mask != nullptr) ? p.mask + static_cast<long long>(b) * p.S : nullptr;
    float m2[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};  // rows h = 0, 1 of this thread
    // Self branch over several chunks: pass 0 finds the row maximum only, pass 1 uses unnormalised
    // P = 2^(s - m) (one exponential per score), and O is divided by l afterwards.
    const bool deferred = branch == 0 && nchunks > 1;
    // pass 0: statistics (skipped when a single chunk holds the whole row), pass 1: P and O += P V
    for (int pass = (nchunks > 1 ? 0 : 1); pass < 2; ++pass) {
      for (int c = 0; c < nchunks; ++c, ++item) {
        const int st = item & 1;
        uint8_t* sK = sKV + st * stage_bytes;
        uint8_t* sV = sK + kbk * KB_BYTES;
        // the other stage was released by the barrier that ended the previous item
        if (tid == 0 && item + 1 < n_items) issue_item(item + 1);
        mbar_wait(&kv_bar[st], kv_phase[st]);
        kv_phase[st] ^= 1;
        float v[TILE / 2];
        {
          const uint32_t ka = smem_u32(sK);
          fence_regs<TILE / 2>(v);
          wgmma_arrive();
          for (int kb = 0; kb < kbk; ++kb)
#pragma unroll
            for (int k = 0; k < 4; ++k)
              Wgmma<TILE>::ss<0, 0>(v, desc_k(qa + kb * KB_BYTES, k), desc_k(ka + kb * KB_BYTES, k), (kb | k) ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<0>();
          fence_regs<TILE / 2>(v);
        }
        const int key0 = c * TILE;
        const bool tail = key0 + TILE > nkeys;
        if (tail || mk != nullptr) {
#pragma unroll
          for (int e = 0; e < TILE / 2; ++e) {
            const int key = key0 + 8 * (e >> 2) + col_l + (e & 1);
            const bool ok = key < nkeys && (mk == nullptr || mk[key] != 0.f);
            v[e] = ok ? v[e] : -INFINITY;
          }
        }
        if (pass == 0 || nchunks == 1) {  // running row maximum (alpha > 0: max commutes with the scaling)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float cm = -INFINITY;
#pragma unroll
            for (int j = 0; j < TILE / 8; ++j) cm = fmaxf(cm, fmaxf(v[4 * j + 2 * h], v[4 * j + 2 * h + 1]));
            cm = quad_max(cm) * p.alpha_log2e;
            if (pass == 0 && !deferred) {  // (uniform: the quad shuffles below need every lane)
              // several cross chunks: the sum is needed before P can be formed, so pass 0 carries it too
              const float mn = fmaxf(m2[h], cm);
              const float mref = mn > -INFINITY ? mn : 0.f;
              float sum = 0.f;
#pragma unroll
              for (int j = 0; j < TILE / 8; ++j)
                sum += ex2_approx(fmaf(v[4 * j + 2 * h], p.alpha_log2e, -mref)) +
                       ex2_approx(fmaf(v[4 * j + 2 * h + 1], p.alpha_log2e, -mref));
              sum = quad_sum(sum);
              if (cm > -INFINITY) l[h] = l[h] * (m2[h] > -INFINITY ? ex2_approx(m2[h] - mn) : 0.f) + sum;
            }
            m2[h] = fmaxf(m2[h], cm);
          }
        }
        if (pass == 1) {
          float pscale[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float mref = m2[h] > -INFINITY ? m2[h] : 0.f;
            float sum = 0.f;
#pragma unroll
            for (int j = 0; j < TILE / 8; ++j)
#pragma unroll
              for (int u = 0; u < 2; ++u) {
                float& x = v[4 * j + 2 * h + u];
                x = ex2_approx(fmaf(x, p.alpha_log2e, -mref));  // 2^-inf = 0 for masked keys
                sum += x;
              }
            if (deferred || nchunks == 1) l[h] += quad_sum(sum);
            // deferred: P stays unnormalised (<= 1) and O is divided by l once after the branch
            pscale[h] = deferred ? 1.f : (l[h] > 0.f ? 1.0f / l[h] : 0.f);
          }
#pragma unroll
          for (int e = 0; e < TILE / 2; ++e) v[e] *= pscale[(e >> 1) & 1];
          const uint32_t va = smem_u32(sV);
          fence_regs<DN / 2>(o);
          wgmma_arrive();
#pragma unroll
          for (int t = 0; t < TILE / 16; ++t) {  // 128 keys = 8 x 16
            uint32_t a[4];
            frag_a(v, t, a);
            Wgmma<DN>::template rs<1>(o, a, desc_mn(va, t, KB_BYTES), (o_started || t) ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          fence_regs<DN / 2>(o);
          o_started = true;
        }
        __syncthreads();  // both warpgroups are done with this stage: it may be refilled
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = q0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
      // row statistics for the backward pass
      if (p.stats != nullptr && q < p.T && (lane & 3) == 0) {
        float* st = p.stats + ((((static_cast<long long>(b) * p.heads + hd) * 2 + branch) * p.T) + q) * 2;
        st[0] = m2[h];
        st[1] = l[h] > 0.f ? 1.0f / l[h] : 0.f;
      }
      if (branch == 0) {
        // self-branch output alone (the backward needs rowsum(dO * O_branch) per branch); a deferred
        // normalisation is applied here so the cross branch accumulates on top of it
        const float oscale = deferred ? (l[h] > 0.f ? 1.0f / l[h] : 0.f) : 1.f;
#pragma unroll
        for (int j = 0; j < DN / 8; ++j) {
          o[4 * j + 2 * h] *= oscale;
          o[4 * j + 2 * h + 1] *= oscale;
        }
        if (p.oself16 != nullptr && q < p.T) {
          __half* dst = p.oself16 + (static_cast<long long>(b) * p.T + q) * p.C + hd * p.d;
#pragma unroll
          for (int j = 0; j < DN / 8; ++j) {
            const int col = 8 * j + col_l;
            if (col < p.d) *reinterpret_cast<__half2*>(dst + col) = __floats2half2_rn(o[4 * j + 2 * h], o[4 * j + 2 * h + 1]);
          }
        }
      }
    }
  }
  // final output
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
    if (q >= p.T) continue;
    __half* dst = p.h16 + (static_cast<long long>(b) * p.T + q) * p.C + hd * p.d;
#pragma unroll
    for (int j = 0; j < DN / 8; ++j) {
      const int col = 8 * j + col_l;
      if (col < p.d) *reinterpret_cast<__half2*>(dst + col) = __floats2half2_rn(o[4 * j + 2 * h], o[4 * j + 2 * h + 1]);
    }
  }
}

// ------------------------------------------------------------------------------------------ backward
// D[b][h][branch][q] = sum_c dO[q][c] * O_branch[q][c]  with O_cross = h - O_self
__global__ void attn_bwd_prep_kernel(const __half* __restrict__ dO, const __half* __restrict__ h16,
                                     const __half* __restrict__ oself16, float* __restrict__ Dterm, int T, int C,
                                     int heads, int d, long long rows) {
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const long long b = row / T;
  const int q = static_cast<int>(row - b * T);
  for (int hd = 0; hd < heads; ++hd) {
    float s0 = 0.f, s1 = 0.f;
    for (int c = lane; c < d; c += 32) {
      const long long o = row * C + hd * d + c;
      const float g = __half2float(dO[o]);
      const float os = oself16 != nullptr ? __half2float(oself16[o]) : __half2float(h16[o]);
      const float oc = __half2float(h16[o]) - os;
      s0 += g * os;
      s1 += g * oc;
    }
    for (int o = 16; o > 0; o >>= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, o);
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    }
    if (lane == 0) {
      Dterm[((b * heads + hd) * 2 + 0) * T + q] = s0;
      Dterm[((b * heads + hd) * 2 + 1) * T + q] = s1;
    }
  }
}

// One CTA per (128 keys, head, sample), looping over 128-query tiles in two 64-query halves. Warpgroup g owns keys
// 64 g .. 64 g + 63: it computes S^T = K Q^T and dP^T = V dO^T for its keys (registers), forms P^T and
// dS^T = P^T (dP^T - D) alpha in place and feeds them as register A operands to dV += P^T dO and dK += dS^T Q
// (accumulated in registers over all query tiles). dS^T also goes to shared memory, from which
// dQ = dS K (warpgroup g: queries 64 g ..) is computed per query tile and added to the fp32 dQ by atomics.
template <int DN>
__global__ void __launch_bounds__(BWD_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmKV,
                const __grid_constant__ CUtensorMap tmDO, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t kv_bar, qd_bar;
  __shared__ float s_m2[TILE], s_il[TILE], s_nD[TILE];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int hd = blockIdx.y, b = blockIdx.z;
  const int n_self = (p.T + TILE - 1) / TILE;
  const bool cross = static_cast<int>(blockIdx.x) >= n_self;
  const int jt = cross ? blockIdx.x - n_self : blockIdx.x;
  const int key0 = jt * TILE;
  const int nkeys = cross ? p.S : p.T;
  const int branch = cross ? 1 : 0;
  const int kbk = p.kblocks;
  uint8_t* sK = smem;
  uint8_t* sV = sK + kbk * KB_BYTES;
  uint8_t* sQ = sV + kbk * KB_BYTES;
  uint8_t* sDO = sQ + kbk * KB_BYTES;
  uint8_t* sDS = sDO + kbk * KB_BYTES;  // dS^T: [2 query halves][128 keys][64 queries], 128B-swizzled

  if (tid == 0) {
    prefetch_tmap(&tmQKV);
    prefetch_tmap(&tmKV);
    prefetch_tmap(&tmDO);
    mbar_init(&kv_bar, 1);
    mbar_init(&qd_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto load_qd = [&](int q0) {
    mbar_expect_tx(&qd_bar, 2 * kbk * KB_BYTES);
    for (int kb = 0; kb < kbk; ++kb) {
      tma_load_4d(sQ + kb * KB_BYTES, &tmQKV, &qd_bar, kb * 64, q0, hd, b);
      tma_load_4d(sDO + kb * KB_BYTES, &tmDO, &qd_bar, kb * 64, q0, hd, b);
    }
  };
  if (tid == 0) {
    mbar_expect_tx(&kv_bar, 2 * kbk * KB_BYTES);
    for (int kb = 0; kb < kbk; ++kb) {
      if (!cross) {
        tma_load_4d(sK + kb * KB_BYTES, &tmQKV, &kv_bar, kb * 64, key0, p.heads + hd, b);
        tma_load_4d(sV + kb * KB_BYTES, &tmQKV, &kv_bar, kb * 64, key0, 2 * p.heads + hd, b);
      } else {
        tma_load_4d(sK + kb * KB_BYTES, &tmKV, &kv_bar, kb * 64, key0, hd, b);
        tma_load_4d(sV + kb * KB_BYTES, &tmKV, &kv_bar, kb * 64, key0, p.heads + hd, b);
      }
    }
    load_qd(0);
  }
  const float* mk = (cross && p.mask != nullptr) ? p.mask + static_cast<long long>(b) * p.S : nullptr;
  const int col_l = 2 * (lane & 3);
  const int krow = wg * 64 + wq * 16 + (lane >> 2);  // tile-local key of accumulator rows h = 0 (+ 8 for h = 1)
  bool kok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int key = key0 + krow + 8 * h;
    kok[h] = key < nkeys && (mk == nullptr || mk[key] != 0.f);
  }
  const uint32_t ka = smem_u32(sK), va = smem_u32(sV), qa = smem_u32(sQ), da = smem_u32(sDO), sa = smem_u32(sDS);
  float dv[DN / 2], dk[DN / 2];
#pragma unroll
  for (int i = 0; i < DN / 2; ++i) dv[i] = dk[i] = 0.f;
  mbar_wait(&kv_bar, 0);
  uint32_t qd_phase = 0;
  const int nq = (p.T + TILE - 1) / TILE;
  for (int it = 0; it < nq; ++it) {
    const int q0 = it * TILE;
    if (tid < TILE) {
      const int q = q0 + tid;
      float m2 = 0.f, inv_l = 0.f, Dq = 0.f;
      if (q < p.T) {
        const float* st = p.stats + ((((static_cast<long long>(b) * p.heads + hd) * 2 + branch) * p.T) + q) * 2;
        m2 = st[0];
        inv_l = st[1];
        Dq = p.Dterm[((static_cast<long long>(b) * p.heads + hd) * 2 + branch) * p.T + q];
      }
      if (!(inv_l > 0.f)) {  // row outside the tile or fully masked: P = 0 without inf arithmetic
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
#pragma unroll 1
    for (int half = 0; half < 2; ++half) {
      const uint32_t qoff = half * 64 * 128;  // this half's 64 query rows in the Q / dO slabs
      float s[32], dp[32];
      fence_regs<32>(s);
      fence_regs<32>(dp);
      wgmma_arrive();
      for (int kb = 0; kb < kbk; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          Wgmma<64>::ss<0, 0>(s, desc_k(ka + kb * KB_BYTES + wg * 64 * 128, k), desc_k(qa + kb * KB_BYTES + qoff, k),
                              (kb | k) ? 1u : 0u);
          Wgmma<64>::ss<0, 0>(dp, desc_k(va + kb * KB_BYTES + wg * 64 * 128, k), desc_k(da + kb * KB_BYTES + qoff, k),
                              (kb | k) ? 1u : 0u);
        }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<32>(s);
      fence_regs<32>(dp);
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        const int ql = half * 64 + 8 * (e >> 2) + col_l + (e & 1);  // tile-local query (column)
        float pe = ex2_approx(fmaf(s[e], p.alpha_log2e, -s_m2[ql])) * s_il[ql];
        pe = kok[(e >> 1) & 1] ? pe : 0.f;
        s[e] = pe;                                 // P^T
        dp[e] = pe * fmaf(dp[e], p.alpha, s_nD[ql]);  // dS^T = P^T (dP^T - D) / sqrt(d)
      }
      // dS^T into shared memory for dQ
#pragma unroll
      for (int e = 0; e < 32; e += 2) {
        const int kr = krow + 8 * ((e >> 1) & 1);
        const int qc = 8 * (e >> 2) + col_l;
        uint8_t* dst = sDS + half * KB_BYTES + kr * 128 + ((((qc >> 3) ^ (kr & 7))) << 4) + (qc & 7) * 2;
        *reinterpret_cast<uint32_t*>(dst) = pack_half2(dp[e], dp[e + 1]);
      }
      fence_regs<DN / 2>(dv);
      fence_regs<DN / 2>(dk);
      wgmma_arrive();
#pragma unroll
      for (int t = 0; t < 4; ++t) {  // contraction over this half's 64 queries
        uint32_t a[4];
        const uint32_t scale = (it | half | t) ? 1u : 0u;
        frag_a(s, t, a);
        Wgmma<DN>::template rs<1>(dv, a, make_smem_desc_sw128(da + qoff + t * 2048, KB_BYTES, 1024), scale);
        frag_a(dp, t, a);
        Wgmma<DN>::template rs<1>(dk, a, make_smem_desc_sw128(qa + qoff + t * 2048, KB_BYTES, 1024), scale);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<DN / 2>(dv);
      fence_regs<DN / 2>(dk);
    }
    fence_proxy_async();  // dS^T stores -> visible to wgmma
    __syncthreads();      // every read of Q / dO is done and dS^T is complete
    if (tid == 0 && it + 1 < nq) load_qd((it + 1) * TILE);
    {
      // dQ[q][d] = dS K for queries 64 wg .. (A = dS, MN-major in the dS^T tile; B = K, MN-major)
      float dq[DN / 2];
      fence_regs<DN / 2>(dq);
      wgmma_arrive();
#pragma unroll
      for (int t = 0; t < TILE / 16; ++t)
        Wgmma<DN>::template ss<1, 1>(dq, make_smem_desc_sw128(sa + wg * KB_BYTES + t * 2048, KB_BYTES, 1024),
                            desc_mn(ka, t, KB_BYTES), t ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<DN / 2>(dq);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int q = q0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
        if (q >= p.T) continue;
        float* dst = p.dq32 + (static_cast<long long>(b) * p.T + q) * p.C + hd * p.d;
#pragma unroll
        for (int j = 0; j < DN / 8; ++j) {
          const int col = 8 * j + col_l;
          if (col < p.d) {
            atomicAdd(dst + col, dq[4 * j + 2 * h]);
            atomicAdd(dst + col + 1, dq[4 * j + 2 * h + 1]);
          }
        }
      }
    }
    __syncthreads();  // dS^T and the row statistics are rewritten by the next tile
  }
  // dK, dV of this key tile
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int key = key0 + krow + 8 * h;
    if (key >= nkeys) continue;
    __half *dkp, *dvp;
    if (!cross) {
      __half* base = p.dqkv16 + (static_cast<long long>(b) * p.T + key) * 3 * p.C + hd * p.d;
      dkp = base + p.C;
      dvp = base + 2 * p.C;
    } else {
      __half* base = p.dkv16 + (static_cast<long long>(b) * p.S + key) * 2 * p.C + hd * p.d;
      dkp = base;
      dvp = base + p.C;
    }
#pragma unroll
    for (int j = 0; j < DN / 8; ++j) {
      const int col = 8 * j + col_l;
      if (col < p.d) {
        *reinterpret_cast<__half2*>(dkp + col) = __floats2half2_rn(dk[4 * j + 2 * h], dk[4 * j + 2 * h + 1]);
        *reinterpret_cast<__half2*>(dvp + col) = __floats2half2_rn(dv[4 * j + 2 * h], dv[4 * j + 2 * h + 1]);
      }
    }
  }
}

__global__ void cast_strided_kernel(const float* __restrict__ in, __half* __restrict__ out, long long rows, int C,
                                    int ld_out) {
  const long long total = rows * (C / 4);
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total; i += gs) {
    const long long r = i / (C / 4);
    const int c = static_cast<int>(i - r * (C / 4)) * 4;
    const float4 v = *reinterpret_cast<const float4*>(in + r * C + c);
    __half2 a = __floats2half2_rn(v.x, v.y), bq = __floats2half2_rn(v.z, v.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&a);
    o.y = *reinterpret_cast<uint32_t*>(&bq);
    *reinterpret_cast<uint2*>(out + r * ld_out + c) = o;
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* q = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &q, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(q);
  }
  return fn;
}

// Calls f(std::integral_constant<int, DN>) with DN = the head dimension rounded up to 16 (the wgmma N of the
// products with d columns).
template <typename F>
void with_head_width(int d, F&& f) {
  switch ((d + 15) / 16) {
    case 1: f(std::integral_constant<int, 16>()); break;
    case 2: f(std::integral_constant<int, 32>()); break;
    case 3: f(std::integral_constant<int, 48>()); break;
    case 4: f(std::integral_constant<int, 64>()); break;
    case 5: f(std::integral_constant<int, 80>()); break;
    case 6: f(std::integral_constant<int, 96>()); break;
    case 7: f(std::integral_constant<int, 112>()); break;
    default: f(std::integral_constant<int, 128>()); break;
  }
}

}  // namespace

void attn::head_map(CUtensorMap* m, const void* ptr, int d, int rows, long long row_stride, int slots,
                    long long slot_stride, int batch, long long batch_stride, int box_rows) {
  EncodeTiledFn fn = encode_fn();
  MDM_CHECK(fn != nullptr, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(d), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(slots),
                        static_cast<cuuint64_t>(batch)};
  cuuint64_t str[3] = {static_cast<cuuint64_t>(row_stride) * 2, static_cast<cuuint64_t>(slot_stride) * 2,
                       static_cast<cuuint64_t>(batch_stride) * 2};
  cuuint32_t box[4] = {64, static_cast<cuuint32_t>(box_rows), 1, 1}, es[4] = {1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, str, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  MDM_CHECK(r == CUDA_SUCCESS, "attention tensor map encode failed");
}

void attn::cast_rows_f16(const float* in, __half* out, long long rows, int C, int ld_out, cudaStream_t st) {
  cast_strided_kernel<<<132 * 8, 256, 0, st>>>(in, out, rows, C, ld_out);
  ++g_launch_count;
}

// ------------------------------------------------------------------------------------------ host API
void attention_forward(const __half* qkv, const __half* kv, const float* mask, int B, int T, int S, int C, int heads,
                       __half* h16, __half* oself16, float* stats, cudaStream_t st) {
  const int d = C / heads;
  MDM_CHECK(d % 8 == 0 && d <= 128, "head dim must be a multiple of 8 and <= 128");
  AttnParams p{};
  p.T = T; p.S = kv != nullptr ? S : 0; p.d = d; p.heads = heads; p.B = B; p.C = C;
  p.kblocks = (d + 63) / 64;
  p.alpha = 1.0f / sqrtf(static_cast<float>(d));
  p.alpha_log2e = p.alpha * 1.4426950408889634f;
  p.mask = mask;
  p.h16 = h16; p.oself16 = oself16; p.stats = stats;
  alignas(64) CUtensorMap mq, mqv, mk, mkv;
  head_map(&mq, qkv, d, T, 3ll * C, 3 * heads, d, B, static_cast<long long>(T) * 3 * C);
  mqv = mq;
  if (kv != nullptr) head_map(&mk, kv, d, S, 2ll * C, 2 * heads, d, B, static_cast<long long>(S) * 2 * C);
  else mk = mq;
  mkv = mk;
  const int kbk = p.kblocks;
  const size_t smem = static_cast<size_t>(kbk) * KB_BYTES + 2 * (2 * kbk * KB_BYTES) + 1024;
  dim3 grid((T + TILE - 1) / TILE, heads, B);
  with_head_width(d, [&](auto dn) {
    constexpr int DN = decltype(dn)::value;
    static bool attr = false;
    if (!attr) {
      MDM_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<DN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      attr = true;
    }
    attn_fwd_kernel<DN><<<grid, AT_THREADS, smem, st>>>(mq, mqv, mk, mkv, p);
  });
  ++g_launch_count;
  MDM_CUDA(cudaGetLastError());
}

void attention_backward(const __half* qkv, const __half* kv, const float* mask, const __half* dO, const __half* h16,
                        const __half* oself16, const float* stats, int B, int T, int S, int C, int heads,
                        float* Dterm, float* dq32, __half* dqkv16, __half* dkv16, cudaStream_t st) {
  const int d = C / heads;
  AttnParams p{};
  p.T = T; p.S = kv != nullptr ? S : 0; p.d = d; p.heads = heads; p.B = B; p.C = C;
  p.kblocks = (d + 63) / 64;
  p.alpha = 1.0f / sqrtf(static_cast<float>(d));
  p.alpha_log2e = p.alpha * 1.4426950408889634f;
  p.mask = mask;
  p.stats = const_cast<float*>(stats);
  p.Dterm = Dterm; p.dq32 = dq32; p.dqkv16 = dqkv16; p.dkv16 = dkv16;
  const long long rows = static_cast<long long>(B) * T;
  attn_bwd_prep_kernel<<<static_cast<unsigned>((rows + 7) / 8), 256, 0, st>>>(dO, h16, oself16, Dterm, T, C, heads, d, rows);
  ++g_launch_count;
  MDM_CUDA(cudaMemsetAsync(dq32, 0, sizeof(float) * rows * C, st));
  alignas(64) CUtensorMap mq, mk, mdo;
  head_map(&mq, qkv, d, T, 3ll * C, 3 * heads, d, B, static_cast<long long>(T) * 3 * C);
  if (kv != nullptr) head_map(&mk, kv, d, S, 2ll * C, 2 * heads, d, B, static_cast<long long>(S) * 2 * C);
  else mk = mq;
  head_map(&mdo, dO, d, T, C, heads, d, B, static_cast<long long>(T) * C);
  const int kbk = p.kblocks;
  const size_t smem = static_cast<size_t>(4 * kbk + 2) * KB_BYTES + 1024;
  const int n_self = (T + TILE - 1) / TILE, n_cross = p.S > 0 ? (p.S + TILE - 1) / TILE : 0;
  dim3 grid(n_self + n_cross, heads, B);
  with_head_width(d, [&](auto dn) {
    constexpr int DN = decltype(dn)::value;
    static bool attr = false;
    if (!attr) {
      MDM_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<DN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      attr = true;
    }
    attn_bwd_kernel<DN><<<grid, BWD_THREADS, smem, st>>>(mq, mk, mdo, p);
  });
  ++g_launch_count;
  MDM_CUDA(cudaGetLastError());
  // dQ: fp32 accumulator -> fp16 into the q third of dqkv
  cast_rows_f16(dq32, dqkv16, rows, C, 3 * C, st);
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

int mdm_op_attention_fwd(const void* qkv16, const void* kv16, const float* mask, int B, int T, int S, int C, int heads,
                         void* h16, void* oself16, float* stats, mdm_stream_t stream) {
  MDM_TRY(mdm::attention_forward(static_cast<const __half*>(qkv16), static_cast<const __half*>(kv16), mask, B, T, S, C,
                                 heads, static_cast<__half*>(h16), static_cast<__half*>(oself16), stats,
                                 static_cast<cudaStream_t>(stream)))
}

int mdm_op_attention_bwd(const void* qkv16, const void* kv16, const float* mask, const void* dO16, const void* h16,
                         const void* oself16, const float* stats, int B, int T, int S, int C, int heads, float* Dterm,
                         float* dq32, void* dqkv16, void* dkv16, mdm_stream_t stream) {
  MDM_TRY(mdm::attention_backward(static_cast<const __half*>(qkv16), static_cast<const __half*>(kv16), mask,
                                  static_cast<const __half*>(dO16), static_cast<const __half*>(h16),
                                  static_cast<const __half*>(oself16), stats, B, T, S, C, heads, Dterm, dq32,
                                  static_cast<__half*>(dqkv16), static_cast<__half*>(dkv16),
                                  static_cast<cudaStream_t>(stream)))
}
}
