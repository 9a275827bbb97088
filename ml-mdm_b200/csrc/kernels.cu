// Streaming (HBM-bound) kernels of the denoising path. See kernels.cuh for the contracts.
#include <stdexcept>

#include "kernels.cuh"

#include <curand_philox4x32_x.h>  // Philox4x32-10 of curand_kernel.h, header only
#include <math.h>

#include <algorithm>
#include <utility>
#include <vector>

#include "gemm_tc.cuh"  // g_launch_count

namespace mdm {
namespace {

constexpr int TPB = 256;
constexpr int NL_MAX = 6;  // float4 channel lanes per thread (C <= 4 * TPB * NL_MAX)
constexpr float GN_EPS = 1e-5f;

#define MDM_LAUNCHED() (++g_launch_count)

__host__ __device__ inline long long cdiv(long long a, long long b) { return (a + b - 1) / b; }

// Thread -> (channel lane, pixel sub-slot) mapping shared by the per-channel streaming kernels.
// C/4 float4 "lanes" per pixel. When lanes <= TPB several pixels are processed per pass.
struct LaneMap {
  int lanes, ppi, t_lane, stride, sub;
  bool active;
};
__device__ __forceinline__ LaneMap lane_map(int C) {
  LaneMap m;
  m.lanes = C >> 2;
  if (m.lanes <= TPB) {
    m.ppi = TPB / m.lanes;
    m.t_lane = threadIdx.x % m.lanes;
    m.sub = threadIdx.x / m.lanes;
    m.active = m.sub < m.ppi;
    m.stride = m.lanes;  // only j == 0 is in range
  } else {
    m.ppi = 1;
    m.t_lane = threadIdx.x;
    m.sub = 0;
    m.active = true;
    m.stride = TPB;
  }
  return m;
}

__device__ __forceinline__ float4 ld_src(const Src2& s, long long pix, int c) {
  if (c < s.c0) return __ldg(reinterpret_cast<const float4*>(s.p0 + pix * s.c0 + c));
  return __ldg(reinterpret_cast<const float4*>(s.p1 + pix * s.c1 + (c - s.c0)));
}

// gradient operand stored as fp32 or fp16
template <bool F16>
__device__ __forceinline__ float4 ld_dy(const void* dy, long long off) {
  if (F16) {
    const uint2 raw = __ldg(reinterpret_cast<const uint2*>(static_cast<const __half*>(dy) + off));
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&raw.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
    return make_float4(a.x, a.y, b.x, b.y);
  }
  return __ldg(reinterpret_cast<const float4*>(static_cast<const float*>(dy) + off));
}

// sigmoid on the SFU: rcp(1 + 2^(-x log2 e)); saturates cleanly (2^+inf -> rcp(inf) = 0, 2^-inf -> 1)
__device__ __forceinline__ float sigmoidf_(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return r;
}
// pixels handled per loop trip of the GroupNorm streaming kernels: all their loads are issued before the
// first use, which is what keeps enough bytes in flight at the 25-40 % occupancy these kernels run at
template <int NL>
struct PixUnroll {
  static constexpr int U = NL == 1 ? 4 : (NL == 2 ? 2 : 1);
};
__device__ __forceinline__ float siluf_(float x) { return x * sigmoidf_(x); }
__device__ __forceinline__ float silu_grad(float x) {
  const float s = sigmoidf_(x);
  return s * (1.0f + x * (1.0f - s));
}

__device__ __forceinline__ void st_half4(__half* p, float a, float b, float c, float d) {
  __half2 lo = __floats2half2_rn(a, b), hi = __floats2half2_rn(c, d);
  uint2 v;
  v.x = *reinterpret_cast<uint32_t*>(&lo);
  v.y = *reinterpret_cast<uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(p) = v;
}
// the second fp16 plane of st_half4's values: what rounding them to fp16 left behind
__device__ __forceinline__ float f16_rest(float a) { return a - __half2float(__float2half_rn(a)); }
__device__ __forceinline__ void st_half4_lo(__half* p, float a, float b, float c, float d) {
  st_half4(p, f16_rest(a), f16_rest(b), f16_rest(c), f16_rest(d));
}

// Dropout (kernels.cuh) as the kernels see it: one Philox4x32-10 call gives the four factors of a float4 channel lane.
struct DropK {
  const unsigned long long* seed;
  uint32_t stream;
  uint32_t thresh;  // keep when the Philox word >= ceil(p * 2^32)
  float scale;      // 1/(1-p); 0 when p == 1
};
DropK drop_k(const Dropout& d) {
  DropK k{d.seed, d.stream, 0u, 0.f};
  if (d.p >= 1.f) {
    k.thresh = 0xffffffffu;
  } else {
    k.thresh = static_cast<uint32_t>(std::min(ceil(static_cast<double>(d.p) * 4294967296.0), 4294967295.0));
    k.scale = static_cast<float>(1.0 / (1.0 - static_cast<double>(d.p)));
  }
  return k;
}
// factors of elements 4q .. 4q+3
__device__ __forceinline__ float4 drop_factors(unsigned long long seed, uint32_t stream, uint32_t thresh, float scale,
                                               long long q) {
  const uint4 r = curand_Philox4x32_10(
      make_uint4(static_cast<uint32_t>(q), static_cast<uint32_t>(static_cast<unsigned long long>(q) >> 32), stream, 0u),
      make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32)));
  return make_float4(r.x >= thresh ? scale : 0.f, r.y >= thresh ? scale : 0.f, r.z >= thresh ? scale : 0.f,
                     r.w >= thresh ? scale : 0.f);
}
__device__ __forceinline__ float4 drop_factors(const DropK& d, unsigned long long seed, long long q) {
  return drop_factors(seed, d.stream, d.thresh, d.scale, q);
}
template <bool DROP>
__device__ __forceinline__ unsigned long long drop_seed(const DropK& d) {
  return DROP ? __ldg(d.seed) : 0ull;
}


// Sum per-thread float4 accumulators over the pixel sub-slots that share a channel lane (lane_map: when C/4 <= TPB a
// CTA walks TPB / lanes pixels at once), so that ONE thread per channel lane issues the global atomics. Without it a
// 32-channel tensor has 32 sub-slots x every CTA hammering the same 32 addresses (on the 1024-px level of
// cc12m_1024x1024 the atomics serialise the whole kernel).
// Every thread of the block must call this (it synchronises); afterwards the sums live in the threads with sub == 0.
template <int K>
__device__ __forceinline__ void reduce_over_subs(float4 (&v)[K], const LaneMap& m, float4* red) {
  if (m.ppi <= 1) return;  // block-uniform
#pragma unroll
  for (int k = 0; k < K; ++k) {
    red[threadIdx.x] = m.active ? v[k] : make_float4(0, 0, 0, 0);
    __syncthreads();
    if (m.active && m.sub == 0) {
      float4 s = red[m.t_lane];
      for (int i = 1; i < m.ppi; ++i) {
        const float4 o = red[m.t_lane + i * m.lanes];
        s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w;
      }
      v[k] = s;
    }
    __syncthreads();
  }
}

inline int pixel_chunks(int N, int HW, int ppi_hint, int per_sm = 8) {
  long long want = cdiv(per_sm * 132, N);
  // at least ~32 pixel passes per CTA: every CTA pays a prologue (per-channel coefficients) and ends with atomics onto
  // the same few addresses -- at 16x16 pixels and batch 16, 74 CTAs per sample made gn_stats ten times its data time
  long long maxc = std::max<long long>(1, HW / (32ll * (ppi_hint > 0 ? ppi_hint : 1)));
  if (want > maxc) want = maxc;
  if (want < 1) want = 1;
  if (want > 65535) want = 65535;
  return static_cast<int>(want);
}
#define MDM_DISPATCH_NL(C, ...)                    \
  do {                                            \
    const int lanes__ = (C) / 4;                  \
    if (lanes__ <= TPB) {                         \
      constexpr int NL = 1;                       \
      __VA_ARGS__;                                \
    } else if (lanes__ <= 2 * TPB) {              \
      constexpr int NL = 2;                       \
      __VA_ARGS__;                                \
    } else {                                      \
      constexpr int NL = NL_MAX;                  \
      __VA_ARGS__;                                \
    }                                             \
  } while (0)

inline int host_ppi(int C) {
  int lanes = C / 4;
  return lanes <= TPB ? TPB / lanes : 1;
}


// ------------------------------------------------------------------ bulk-copy staged streaming
// The GroupNorm backward kernels were latency-bound (low occupancy at ~80 registers, most warp cycles waiting on
// global loads): the loads in flight lived in registers. Here one thread feeds a ring of
// shared-memory stages with cp.async.bulk (the TMA engine, 1-D), so the bytes in flight no longer cost registers:
// every CTA keeps STAGES x ~24-36 KB outstanding, the 256 threads read their float4 lanes from shared memory.
constexpr int RS_STAGES = 3;

__device__ __forceinline__ uint32_t rs_smem(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void rs_bar_init(uint64_t* bar) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(rs_smem(bar)));
}
__device__ __forceinline__ void rs_expect(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(rs_smem(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void rs_copy(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   rs_smem(dst)),
               "l"(src), "r"(bytes), "r"(rs_smem(bar))
               : "memory");
}
__device__ __forceinline__ void rs_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  const long long t0 = clock64();
  while (true) {
    asm volatile(
        "{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok)
        : "r"(rs_smem(bar)), "r"(parity)
        : "memory");
    if (ok) return;
    if (clock64() - t0 > 4000000000LL) __trap();  // a protocol bug must not hang the GPU box
  }
}

// Stage layout: [x source 0: pix * c0 fp32][x source 1: pix * c1 fp32][dy: pix * C (fp16 | fp32)]
struct RowStage {
  const float* x0;
  const float* x1;
  const uint8_t* dy;
};
struct RowStream {
  uint8_t* base;
  uint64_t* full;  // [RS_STAGES]
  int stage_bytes, x0_bytes_pp, x1_bytes_pp, dy_bytes_pp, pix;  // bytes per pixel of each part, pixels per chunk
  __device__ __forceinline__ RowStage stage(int s) const {
    uint8_t* b = base + static_cast<size_t>(s) * stage_bytes;
    RowStage r;
    r.x0 = reinterpret_cast<const float*>(b);
    r.x1 = reinterpret_cast<const float*>(b + static_cast<size_t>(pix) * x0_bytes_pp);
    r.dy = b + static_cast<size_t>(pix) * (x0_bytes_pp + x1_bytes_pp);
    return r;
  }
  // one thread: fetch pixels [pix0, pix0 + np) of sample-major tensors into stage s
  __device__ __forceinline__ void issue(int s, const Src2& x, const void* dy, long long pix0, int np) const {
    uint8_t* b = base + static_cast<size_t>(s) * stage_bytes;
    const uint32_t b0 = static_cast<uint32_t>(np) * x0_bytes_pp, b1 = static_cast<uint32_t>(np) * x1_bytes_pp,
                   b2 = static_cast<uint32_t>(np) * dy_bytes_pp;
    rs_expect(&full[s], b0 + b1 + b2);
    rs_copy(b, reinterpret_cast<const uint8_t*>(x.p0) + pix0 * x0_bytes_pp, b0, &full[s]);
    if (b1 > 0)
      rs_copy(b + static_cast<size_t>(pix) * x0_bytes_pp, reinterpret_cast<const uint8_t*>(x.p1) + pix0 * x1_bytes_pp, b1,
              &full[s]);
    if (b2 > 0)
      rs_copy(b + static_cast<size_t>(pix) * (x0_bytes_pp + x1_bytes_pp), static_cast<const uint8_t*>(dy) + pix0 * dy_bytes_pp,
              b2, &full[s]);
  }
};
__device__ __forceinline__ float4 rs_ld_x(const RowStage& st, const Src2& x, int pl, int c) {
  if (c < x.c0) return *reinterpret_cast<const float4*>(st.x0 + static_cast<size_t>(pl) * x.c0 + c);
  return *reinterpret_cast<const float4*>(st.x1 + static_cast<size_t>(pl) * x.c1 + (c - x.c0));
}
template <bool F16>
__device__ __forceinline__ float4 rs_ld_dy(const RowStage& st, int C, int pl, int c) {
  if (F16) {
    const uint2 raw = *reinterpret_cast<const uint2*>(st.dy + (static_cast<size_t>(pl) * C + c) * 2);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&raw.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
    return make_float4(a.x, a.y, b.x, b.y);
  }
  return *reinterpret_cast<const float4*>(st.dy + (static_cast<size_t>(pl) * C + c) * 4);
}
// host: pixels per chunk (a multiple of the CTA's pixels-per-pass) for ~16 KB of x per stage, and the stage size
inline void rs_geometry(int C, int dy_esz, int* pix, int* stage_bytes) {
  const int ppi = host_ppi(C);
  int px = std::max(1, 16384 / (C * 4));
  px = std::max(ppi, px / ppi * ppi);
  *pix = px;
  *stage_bytes = (px * C * (4 + dy_esz) + 127) / 128 * 128;
}

// ------------------------------------------------------------------ GroupNorm statistics
template <int NL>
__global__ void __launch_bounds__(TPB) gn_stats_kernel(Src2 x, int HW, int G, float* __restrict__ sums) {
  const int C = x.c0 + x.c1;
  const int cpg = C / G;
  const LaneMap m = lane_map(C);
  const int n = blockIdx.y;
  const int per = static_cast<int>(cdiv(HW, gridDim.x));
  const int p_begin = blockIdx.x * per;
  const int p_end = min(HW, p_begin + per);
  float4 s[NL], q[NL];
#pragma unroll
  for (int j = 0; j < NL; ++j) {
    s[j] = make_float4(0, 0, 0, 0);
    q[j] = make_float4(0, 0, 0, 0);
  }
  if (m.active) {
    constexpr int U = PixUnroll<NL>::U;
    for (int p = p_begin + m.sub; p < p_end; p += U * m.ppi) {
      float4 vv[U][NL];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int pu = p + u * m.ppi;
        const long long pix = static_cast<long long>(n) * HW + pu;
#pragma unroll
        for (int j = 0; j < NL; ++j) {
          const int l = m.t_lane + j * m.stride;
          vv[u][j] = (l < m.lanes && pu < p_end) ? ld_src(x, pix, 4 * l) : make_float4(0, 0, 0, 0);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
#pragma unroll
        for (int j = 0; j < NL; ++j) {
          const float4 v = vv[u][j];  // zeros where out of range
          s[j].x += v.x; s[j].y += v.y; s[j].z += v.z; s[j].w += v.w;
          q[j].x += v.x * v.x; q[j].y += v.y * v.y; q[j].z += v.z * v.z; q[j].w += v.w * v.w;
        }
      }
    }
  }
  __shared__ float gs[128], gq[128];
  for (int i = threadIdx.x; i < G; i += TPB) {
    gs[i] = 0.f;
    gq[i] = 0.f;
  }
  __syncthreads();
  if (m.active) {
#pragma unroll
    for (int j = 0; j < NL; ++j) {
      const int l = m.t_lane + j * m.stride;
      if (l < m.lanes) {
        const int c = 4 * l;
        const float sv[4] = {s[j].x, s[j].y, s[j].z, s[j].w};
        const float qv[4] = {q[j].x, q[j].y, q[j].z, q[j].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          atomicAdd(&gs[(c + k) / cpg], sv[k]);
          atomicAdd(&gq[(c + k) / cpg], qv[k]);
        }
      }
    }
  }
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += TPB) {
    atomicAdd(&sums[(static_cast<long long>(n) * G + g) * 2 + 0], gs[g]);
    atomicAdd(&sums[(static_cast<long long>(n) * G + g) * 2 + 1], gq[g]);
  }
}

// Per-thread GroupNorm coefficients of its channel lanes: xhat = x*rs + (-mean*rs); u = xhat*ga + be
// with ga = gamma*(1+ta), be = beta*(1+ta)+tb.
template <int NL>
struct GnCoef {
  float4 rs[NL], nm[NL], ga[NL], be[NL];
};
template <int NL>
__device__ __forceinline__ void gn_coefs(GnCoef<NL>& k, const LaneMap& m, int n, int C, int G, int HW,
                                         const float* sums, const float* gamma, const float* beta,
                                         const float* film, int film_ld, int film_off) {
  const int cpg = C / G;
  const float inv_cnt = 1.0f / (static_cast<float>(HW) * cpg);
#pragma unroll
  for (int j = 0; j < NL; ++j) {
    const int l = m.t_lane + j * m.stride;
    if (l < m.lanes) {
      float rs[4], nm[4], ga[4], be[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = 4 * l + e;
        const int g = c / cpg;
        const float su = __ldg(sums + (static_cast<long long>(n) * G + g) * 2);
        const float sq = __ldg(sums + (static_cast<long long>(n) * G + g) * 2 + 1);
        const float mean = su * inv_cnt;
        const float var = fmaxf(sq * inv_cnt - mean * mean, 0.f);
        const float r = rsqrtf(var + GN_EPS);
        rs[e] = r;
        nm[e] = -mean * r;
        float gm = __ldg(gamma + c), bt = __ldg(beta + c);
        if (film != nullptr) {
          const float ta = __ldg(film + static_cast<long long>(n) * film_ld + film_off + c);
          const float tb = __ldg(film + static_cast<long long>(n) * film_ld + film_off + C + c);
          gm = gm * (1.f + ta);
          bt = bt * (1.f + ta) + tb;
        }
        ga[e] = gm;
        be[e] = bt;
      }
      k.rs[j] = make_float4(rs[0], rs[1], rs[2], rs[3]);
      k.nm[j] = make_float4(nm[0], nm[1], nm[2], nm[3]);
      k.ga[j] = make_float4(ga[0], ga[1], ga[2], ga[3]);
      k.be[j] = make_float4(be[0], be[1], be[2], be[3]);
    }
  }
}

template <int NL, bool DROP>
__global__ void __launch_bounds__(TPB)
gn_apply_kernel(Src2 x, int HW, int G, const float* __restrict__ sums, const float* __restrict__ gamma,
                const float* __restrict__ beta, const float* __restrict__ film, int film_ld, int film_off,
                int silu, __half* __restrict__ y16, __half* __restrict__ raw16, DropK drop) {
  const int C = x.c0 + x.c1;
  const LaneMap m = lane_map(C);
  const int n = blockIdx.y;
  const int per = static_cast<int>(cdiv(HW, gridDim.x));
  const int p_begin = blockIdx.x * per;
  const int p_end = min(HW, p_begin + per);
  if (!m.active) return;
  const unsigned long long seed = drop_seed<DROP>(drop);
  GnCoef<NL> k;
  gn_coefs(k, m, n, C, G, HW, sums, gamma, beta, film, film_ld, film_off);
  constexpr int U = PixUnroll<NL>::U;
  for (int p0 = p_begin + m.sub; p0 < p_end; p0 += U * m.ppi) {
    float4 vv[U][NL];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int pu = p0 + u * m.ppi;
#pragma unroll
      for (int j = 0; j < NL; ++j) {
        const int l = m.t_lane + j * m.stride;
        if (l < m.lanes && pu < p_end) vv[u][j] = ld_src(x, static_cast<long long>(n) * HW + pu, 4 * l);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
    const int p = p0 + u * m.ppi;
    if (p >= p_end) break;
    const long long pix = static_cast<long long>(n) * HW + p;
#pragma unroll
    for (int j = 0; j < NL; ++j) {
      const int l = m.t_lane + j * m.stride;
      if (l < m.lanes) {
        const float4 v = vv[u][j];
        float u0 = (v.x * k.rs[j].x + k.nm[j].x) * k.ga[j].x + k.be[j].x;
        float u1 = (v.y * k.rs[j].y + k.nm[j].y) * k.ga[j].y + k.be[j].y;
        float u2 = (v.z * k.rs[j].z + k.nm[j].z) * k.ga[j].z + k.be[j].z;
        float u3 = (v.w * k.rs[j].w + k.nm[j].w) * k.ga[j].w + k.be[j].w;
        if (silu) {
          u0 = siluf_(u0); u1 = siluf_(u1); u2 = siluf_(u2); u3 = siluf_(u3);
        }
        if (DROP) {
          const float4 f = drop_factors(drop, seed, pix * m.lanes + l);
          u0 *= f.x; u1 *= f.y; u2 *= f.z; u3 *= f.w;
        }
        st_half4(y16 + pix * C + 4 * l, u0, u1, u2, u3);
        if (raw16 != nullptr) st_half4(raw16 + pix * C + 4 * l, v.x, v.y, v.z, v.w);
      }
    }
    }
  }
}

template <int NL, bool DY16, bool DROP>
__global__ void __launch_bounds__(TPB)
gn_bwd_reduce_kernel(Src2 x, const void* __restrict__ dy, int HW, int G, const float* __restrict__ sums,
                     const float* __restrict__ gamma, const float* __restrict__ beta,
                     const float* __restrict__ film, int film_ld, int film_off, int silu,
                     float* __restrict__ ab, DropK drop) {
  const int C = x.c0 + x.c1;
  const LaneMap m = lane_map(C);
  const int n = blockIdx.y;
  const int per = static_cast<int>(cdiv(HW, gridDim.x));
  const int p_begin = blockIdx.x * per;
  const int p_end = min(HW, p_begin + per);
  __shared__ float4 red[TPB];
  const unsigned long long seed = drop_seed<DROP>(drop);
  GnCoef<NL> k;
  if (m.active) gn_coefs(k, m, n, C, G, HW, sums, gamma, beta, film, film_ld, film_off);
  float4 A[NL], Bq[NL];
#pragma unroll
  for (int j = 0; j < NL; ++j) {
    A[j] = make_float4(0, 0, 0, 0);
    Bq[j] = make_float4(0, 0, 0, 0);
  }
  constexpr int U = PixUnroll<NL>::U;
  for (int p0 = p_begin + m.sub; m.active && p0 < p_end; p0 += U * m.ppi) {
    float4 vv[U][NL], dd[U][NL];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int pu = p0 + u * m.ppi;
      const long long pix = static_cast<long long>(n) * HW + pu;
#pragma unroll
      for (int j = 0; j < NL; ++j) {
        const int l = m.t_lane + j * m.stride;
        if (l < m.lanes && pu < p_end) {
          vv[u][j] = ld_src(x, pix, 4 * l);
          dd[u][j] = ld_dy<DY16>(dy, pix * C + 4 * l);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (p0 + u * m.ppi >= p_end) break;
#pragma unroll
      for (int j = 0; j < NL; ++j) {
        const int l = m.t_lane + j * m.stride;
        if (l < m.lanes) {
          const float4 v = vv[u][j];
          float4 d = dd[u][j];
          if (DROP) {
            const float4 f = drop_factors(drop, seed, (static_cast<long long>(n) * HW + p0 + u * m.ppi) * m.lanes + l);
            d.x *= f.x; d.y *= f.y; d.z *= f.z; d.w *= f.w;
          }
          const float xh[4] = {v.x * k.rs[j].x + k.nm[j].x, v.y * k.rs[j].y + k.nm[j].y,
                               v.z * k.rs[j].z + k.nm[j].z, v.w * k.rs[j].w + k.nm[j].w};
          const float ga[4] = {k.ga[j].x, k.ga[j].y, k.ga[j].z, k.ga[j].w};
          const float be[4] = {k.be[j].x, k.be[j].y, k.be[j].z, k.be[j].w};
          float du[4] = {d.x, d.y, d.z, d.w};
          if (silu) {
#pragma unroll
            for (int e = 0; e < 4; ++e) du[e] *= silu_grad(xh[e] * ga[e] + be[e]);
          }
          A[j].x += du[0]; A[j].y += du[1]; A[j].z += du[2]; A[j].w += du[3];
          Bq[j].x += du[0] * xh[0]; Bq[j].y += du[1] * xh[1]; Bq[j].z += du[2] * xh[2]; Bq[j].w += du[3] * xh[3];
        }
      }
    }
  }
  reduce_over_subs(A, m, red);
  reduce_over_subs(Bq, m, red);
  if (!m.active || (m.ppi > 1 && m.sub != 0)) return;
#pragma unroll
  for (int j = 0; j < NL; ++j) {
    const int l = m.t_lane + j * m.stride;
    if (l < m.lanes) {
      float* o = ab + (static_cast<long long>(n) * C + 4 * l) * 2;
      atomicAdd(o + 0, A[j].x); atomicAdd(o + 1, Bq[j].x);
      atomicAdd(o + 2, A[j].y); atomicAdd(o + 3, Bq[j].y);
      atomicAdd(o + 4, A[j].z); atomicAdd(o + 5, Bq[j].z);
      atomicAdd(o + 6, A[j].w); atomicAdd(o + 7, Bq[j].w);
    }
  }
}


template <int NL, bool DY16, bool DROP>
__global__ void __launch_bounds__(TPB)
gn_bwd_reduce_staged_kernel(Src2 x, const void* __restrict__ dy, int HW, int G, const float* __restrict__ sums,
                            const float* __restrict__ gamma, const float* __restrict__ beta,
                            const float* __restrict__ film, int film_ld, int film_off, int silu,
                            float* __restrict__ ab, int pix, int stage_bytes, DropK drop) {
  extern __shared__ __align__(128) uint8_t rs_mem[];
  __shared__ __align__(8) uint64_t full[RS_STAGES];
  __shared__ float4 red[TPB];
  const int C = x.c0 + x.c1;
  const LaneMap m = lane_map(C);
  const int n = blockIdx.y;
  const int per = static_cast<int>(cdiv(cdiv(HW, gridDim.x), pix)) * pix;  // whole chunks per CTA
  const int p_begin = blockIdx.x * per;
  const int p_end = min(HW, p_begin + per);
  const int nchunks = p_end > p_begin ? static_cast<int>(cdiv(p_end - p_begin, pix)) : 0;
  RowStream rs{rs_mem, full, stage_bytes, x.c0 * 4, x.c1 * 4, C * (DY16 ? 2 : 4), pix};
  if (threadIdx.x == 0) {
    for (int s = 0; s < RS_STAGES; ++s) rs_bar_init(&full[s]);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const long long base_pix = static_cast<long long>(n) * HW;
  if (threadIdx.x == 0)
    for (int it = 0; it < RS_STAGES && it < nchunks; ++it)
      rs.issue(it, x, dy, base_pix + p_begin + it * pix, min(pix, p_end - p_begin - it * pix));
  GnCoef<NL> k;
  if (m.active) gn_coefs(k, m, n, C, G, HW, sums, gamma, beta, film, film_ld, film_off);
  const unsigned long long seed = drop_seed<DROP>(drop);
  float4 A[NL], Bq[NL];
#pragma unroll
  for (int j = 0; j < NL; ++j) {
    A[j] = make_float4(0, 0, 0, 0);
    Bq[j] = make_float4(0, 0, 0, 0);
  }
  for (int it = 0; it < nchunks; ++it) {
    const int s = it % RS_STAGES;
    rs_wait(&full[s], static_cast<uint32_t>(it / RS_STAGES) & 1u);
    const RowStage st = rs.stage(s);
    const int np = min(pix, p_end - p_begin - it * pix);
    if (m.active) {
      for (int pl = m.sub; pl < np; pl += m.ppi) {
#pragma unroll
        for (int j = 0; j < NL; ++j) {
          const int l = m.t_lane + j * m.stride;
          if (l < m.lanes) {
            const float4 v = rs_ld_x(st, x, pl, 4 * l);
            float4 d = rs_ld_dy<DY16>(st, C, pl, 4 * l);
            if (DROP) {
              const float4 f = drop_factors(drop, seed, (base_pix + p_begin + it * pix + pl) * m.lanes + l);
              d.x *= f.x; d.y *= f.y; d.z *= f.z; d.w *= f.w;
            }
            const float xh[4] = {v.x * k.rs[j].x + k.nm[j].x, v.y * k.rs[j].y + k.nm[j].y,
                                 v.z * k.rs[j].z + k.nm[j].z, v.w * k.rs[j].w + k.nm[j].w};
            const float ga[4] = {k.ga[j].x, k.ga[j].y, k.ga[j].z, k.ga[j].w};
            const float be[4] = {k.be[j].x, k.be[j].y, k.be[j].z, k.be[j].w};
            float du[4] = {d.x, d.y, d.z, d.w};
            if (silu) {
#pragma unroll
              for (int e = 0; e < 4; ++e) du[e] *= silu_grad(xh[e] * ga[e] + be[e]);
            }
            A[j].x += du[0]; A[j].y += du[1]; A[j].z += du[2]; A[j].w += du[3];
            Bq[j].x += du[0] * xh[0]; Bq[j].y += du[1] * xh[1]; Bq[j].z += du[2] * xh[2]; Bq[j].w += du[3] * xh[3];
          }
        }
      }
    }
    __syncthreads();  // every thread is done with stage s
    if (threadIdx.x == 0 && it + RS_STAGES < nchunks)
      rs.issue(s, x, dy, base_pix + p_begin + (it + RS_STAGES) * pix, min(pix, p_end - p_begin - (it + RS_STAGES) * pix));
  }
  reduce_over_subs(A, m, red);
  reduce_over_subs(Bq, m, red);
  if (!m.active || (m.ppi > 1 && m.sub != 0)) return;
#pragma unroll
  for (int j = 0; j < NL; ++j) {
    const int l = m.t_lane + j * m.stride;
    if (l < m.lanes) {
      float* o = ab + (static_cast<long long>(n) * C + 4 * l) * 2;
      atomicAdd(o + 0, A[j].x); atomicAdd(o + 1, Bq[j].x);
      atomicAdd(o + 2, A[j].y); atomicAdd(o + 3, Bq[j].y);
      atomicAdd(o + 4, A[j].z); atomicAdd(o + 5, Bq[j].z);
      atomicAdd(o + 6, A[j].w); atomicAdd(o + 7, Bq[j].w);
    }
  }
}

__global__ void gn_bwd_finalize_kernel(int C, int G, int HW, const float* __restrict__ ab,
                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                       const float* __restrict__ film, int film_ld, int film_off,
                                       float* __restrict__ pg, float* __restrict__ dgamma,
                                       float* __restrict__ dbeta, float* __restrict__ dfilm,
                                       const float* __restrict__ inv_scale) {
  const int n = blockIdx.x;
  const int cpg = C / G;
  __shared__ float p1[128], p2[128];
  for (int i = threadIdx.x; i < G; i += blockDim.x) {
    p1[i] = 0.f;
    p2[i] = 0.f;
  }
  __syncthreads();
  const float inv = inv_scale != nullptr ? __ldg(inv_scale) : 1.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float A = ab[(static_cast<long long>(n) * C + c) * 2];
    const float B = ab[(static_cast<long long>(n) * C + c) * 2 + 1];
    const float gm = gamma[c], bt = beta[c];
    float f = 1.f;
    if (film != nullptr) {
      f = 1.f + film[static_cast<long long>(n) * film_ld + film_off + c];
      if (dfilm != nullptr) {
        dfilm[static_cast<long long>(n) * 2 * C + c] = gm * B + bt * A;
        dfilm[static_cast<long long>(n) * 2 * C + C + c] = A;
      }
    }
    atomicAdd(&p1[c / cpg], gm * f * A);
    atomicAdd(&p2[c / cpg], gm * f * B);
    atomicAdd(&dgamma[c], inv * f * B);
    atomicAdd(&dbeta[c], inv * f * A);
  }
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    pg[(static_cast<long long>(n) * G + g) * 2 + 0] = p1[g];
    pg[(static_cast<long long>(n) * G + g) * 2 + 1] = p2[g];
  }
}

template <int NL, bool DY16, bool DROP>
__global__ void __launch_bounds__(TPB)
gn_bwd_apply_kernel(Src2 x, const void* __restrict__ dy, int HW, int G, const float* __restrict__ sums,
                    const float* __restrict__ gamma, const float* __restrict__ beta,
                    const float* __restrict__ film, int film_ld, int film_off, int silu,
                    const float* __restrict__ pg, const float* __restrict__ extra, Dst2 dst, DropK drop) {
  const int C = x.c0 + x.c1;
  const int cpg = C / G;
  const LaneMap m = lane_map(C);
  const int n = blockIdx.y;
  const int per = static_cast<int>(cdiv(HW, gridDim.x));
  const int p_begin = blockIdx.x * per;
  const int p_end = min(HW, p_begin + per);
  __shared__ float4 red[TPB];
  const unsigned long long seed = drop_seed<DROP>(drop);
  GnCoef<NL> k;
  if (m.active) gn_coefs(k, m, n, C, G, HW, sums, gamma, beta, film, film_ld, film_off);
  float4 csum[NL];
#pragma unroll
  for (int j = 0; j < NL; ++j) csum[j] = make_float4(0, 0, 0, 0);
  // per-channel group terms P1/m, P2/m and gamma' (already includes 1+ta)
  float4 q1[NL], q2[NL];
  const float inv_m = 1.0f / (static_cast<float>(HW) * cpg);
#pragma unroll
  for (int j = 0; j < NL; ++j) {
    const int l = m.t_lane + j * m.stride;
    if (m.active && l < m.lanes) {
      float a[4], b[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int g = (4 * l + e) / cpg;
        a[e] = __ldg(pg + (static_cast<long long>(n) * G + g) * 2) * inv_m;
        b[e] = __ldg(pg + (static_cast<long long>(n) * G + g) * 2 + 1) * inv_m;
      }
      q1[j] = make_float4(a[0], a[1], a[2], a[3]);
      q2[j] = make_float4(b[0], b[1], b[2], b[3]);
    }
  }
  constexpr int U = NL == 1 ? 2 : 1;  // measured: 4 pixels per trip costs this kernel a resident CTA (92 regs)
  for (int p0 = p_begin + m.sub; m.active && p0 < p_end; p0 += U * m.ppi) {
    float4 vv[U][NL], dd[U][NL];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int pu = p0 + u * m.ppi;
      const long long pixu = static_cast<long long>(n) * HW + pu;
#pragma unroll
      for (int j = 0; j < NL; ++j) {
        const int l = m.t_lane + j * m.stride;
        if (l < m.lanes && pu < p_end) {
          vv[u][j] = ld_src(x, pixu, 4 * l);
          dd[u][j] = ld_dy<DY16>(dy, pixu * C + 4 * l);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
    const int p = p0 + u * m.ppi;
    if (p >= p_end) break;
    const long long pix = static_cast<long long>(n) * HW + p;
#pragma unroll
    for (int j = 0; j < NL; ++j) {
      const int l = m.t_lane + j * m.stride;
      if (l < m.lanes) {
        const int c = 4 * l;
        const float4 v = vv[u][j];
        float4 d = dd[u][j];
        if (DROP) {
          const float4 f = drop_factors(drop, seed, pix * m.lanes + l);
          d.x *= f.x; d.y *= f.y; d.z *= f.z; d.w *= f.w;
        }
        const float xh[4] = {v.x * k.rs[j].x + k.nm[j].x, v.y * k.rs[j].y + k.nm[j].y,
                             v.z * k.rs[j].z + k.nm[j].z, v.w * k.rs[j].w + k.nm[j].w};
        const float ga[4] = {k.ga[j].x, k.ga[j].y, k.ga[j].z, k.ga[j].w};
        const float be[4] = {k.be[j].x, k.be[j].y, k.be[j].z, k.be[j].w};
        const float rs[4] = {k.rs[j].x, k.rs[j].y, k.rs[j].z, k.rs[j].w};
        const float a1[4] = {q1[j].x, q1[j].y, q1[j].z, q1[j].w};
        const float a2[4] = {q2[j].x, q2[j].y, q2[j].z, q2[j].w};
        float du[4] = {d.x, d.y, d.z, d.w};
        float r[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (silu) du[e] *= silu_grad(xh[e] * ga[e] + be[e]);
          r[e] = rs[e] * (du[e] * ga[e] - a1[e] - xh[e] * a2[e]);
        }
        if (extra != nullptr) {
          const float4 ex = __ldg(reinterpret_cast<const float4*>(extra + pix * C + c));
          r[0] += ex.x; r[1] += ex.y; r[2] += ex.z; r[3] += ex.w;
        }
        if (dst.h16 != nullptr) {  // single consumer: fp16 operand for the next GEMM + bias-gradient column sums
          st_half4(dst.h16 + pix * C + c, r[0], r[1], r[2], r[3]);
          if (dst.h16lo != nullptr) st_half4_lo(dst.h16lo + pix * C + c, r[0], r[1], r[2], r[3]);
          csum[j].x += r[0]; csum[j].y += r[1]; csum[j].z += r[2]; csum[j].w += r[3];
          continue;
        }
        float* o;
        int acc;
        if (c < dst.c0) {
          o = dst.p0 + pix * dst.c0 + c;
          acc = dst.acc0;
        } else {
          o = dst.p1 + pix * dst.c1 + (c - dst.c0);
          acc = dst.acc1;
        }
        float4 outv = make_float4(r[0], r[1], r[2], r[3]);
        if (acc) {
          const float4 old = *reinterpret_cast<const float4*>(o);
          outv.x += old.x; outv.y += old.y; outv.z += old.z; outv.w += old.w;
        }
        *reinterpret_cast<float4*>(o) = outv;
      }
    }
    }
  }
  if (dst.h16 != nullptr && dst.colsum != nullptr) {  // kernel-argument condition: uniform over the block
    reduce_over_subs(csum, m, red);
    if (!m.active || (m.ppi > 1 && m.sub != 0)) return;
    const float inv = dst.inv_scale != nullptr ? __ldg(dst.inv_scale) : 1.f;
#pragma unroll
    for (int j = 0; j < NL; ++j) {
      const int l = m.t_lane + j * m.stride;
      if (l < m.lanes) {
        atomicAdd(dst.colsum + 4 * l + 0, inv * csum[j].x);
        atomicAdd(dst.colsum + 4 * l + 1, inv * csum[j].y);
        atomicAdd(dst.colsum + 4 * l + 2, inv * csum[j].z);
        atomicAdd(dst.colsum + 4 * l + 3, inv * csum[j].w);
      }
    }
  }
}


template <int NL, bool DY16, bool DROP>
__global__ void __launch_bounds__(TPB)
gn_bwd_apply_staged_kernel(Src2 x, const void* __restrict__ dy, int HW, int G, const float* __restrict__ sums,
                           const float* __restrict__ gamma, const float* __restrict__ beta,
                           const float* __restrict__ film, int film_ld, int film_off, int silu,
                           const float* __restrict__ pg, const float* __restrict__ extra, Dst2 dst, int pix,
                           int stage_bytes, DropK drop) {
  extern __shared__ __align__(128) uint8_t rs_mem[];
  __shared__ __align__(8) uint64_t full[RS_STAGES];
  __shared__ float4 red[TPB];
  const int C = x.c0 + x.c1;
  const int cpg = C / G;
  const LaneMap m = lane_map(C);
  const int n = blockIdx.y;
  const int per = static_cast<int>(cdiv(cdiv(HW, gridDim.x), pix)) * pix;
  const int p_begin = blockIdx.x * per;
  const int p_end = min(HW, p_begin + per);
  const int nchunks = p_end > p_begin ? static_cast<int>(cdiv(p_end - p_begin, pix)) : 0;
  RowStream rs{rs_mem, full, stage_bytes, x.c0 * 4, x.c1 * 4, C * (DY16 ? 2 : 4), pix};
  if (threadIdx.x == 0) {
    for (int s = 0; s < RS_STAGES; ++s) rs_bar_init(&full[s]);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const long long base_pix = static_cast<long long>(n) * HW;
  if (threadIdx.x == 0)
    for (int it = 0; it < RS_STAGES && it < nchunks; ++it)
      rs.issue(it, x, dy, base_pix + p_begin + it * pix, min(pix, p_end - p_begin - it * pix));
  GnCoef<NL> k;
  if (m.active) gn_coefs(k, m, n, C, G, HW, sums, gamma, beta, film, film_ld, film_off);
  const unsigned long long seed = drop_seed<DROP>(drop);
  float4 csum[NL], q1[NL], q2[NL];
  const float inv_m = 1.0f / (static_cast<float>(HW) * cpg);
#pragma unroll
  for (int j = 0; j < NL; ++j) {
    csum[j] = make_float4(0, 0, 0, 0);
    const int l = m.t_lane + j * m.stride;
    if (m.active && l < m.lanes) {
      float a[4], b[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int g = (4 * l + e) / cpg;
        a[e] = __ldg(pg + (static_cast<long long>(n) * G + g) * 2) * inv_m;
        b[e] = __ldg(pg + (static_cast<long long>(n) * G + g) * 2 + 1) * inv_m;
      }
      q1[j] = make_float4(a[0], a[1], a[2], a[3]);
      q2[j] = make_float4(b[0], b[1], b[2], b[3]);
    }
  }
  for (int it = 0; it < nchunks; ++it) {
    const int s = it % RS_STAGES;
    rs_wait(&full[s], static_cast<uint32_t>(it / RS_STAGES) & 1u);
    const RowStage st = rs.stage(s);
    const int np = min(pix, p_end - p_begin - it * pix);
    if (m.active) {
      for (int pl = m.sub; pl < np; pl += m.ppi) {
        const long long gpix = base_pix + p_begin + it * pix + pl;
#pragma unroll
        for (int j = 0; j < NL; ++j) {
          const int l = m.t_lane + j * m.stride;
          if (l < m.lanes) {
            const int c = 4 * l;
            const float4 v = rs_ld_x(st, x, pl, c);
            float4 d = rs_ld_dy<DY16>(st, C, pl, c);
            if (DROP) {
              const float4 f = drop_factors(drop, seed, gpix * m.lanes + l);
              d.x *= f.x; d.y *= f.y; d.z *= f.z; d.w *= f.w;
            }
            const float xh[4] = {v.x * k.rs[j].x + k.nm[j].x, v.y * k.rs[j].y + k.nm[j].y,
                                 v.z * k.rs[j].z + k.nm[j].z, v.w * k.rs[j].w + k.nm[j].w};
            const float ga[4] = {k.ga[j].x, k.ga[j].y, k.ga[j].z, k.ga[j].w};
            const float be[4] = {k.be[j].x, k.be[j].y, k.be[j].z, k.be[j].w};
            const float rsd[4] = {k.rs[j].x, k.rs[j].y, k.rs[j].z, k.rs[j].w};
            const float a1[4] = {q1[j].x, q1[j].y, q1[j].z, q1[j].w};
            const float a2[4] = {q2[j].x, q2[j].y, q2[j].z, q2[j].w};
            float du[4] = {d.x, d.y, d.z, d.w};
            float r[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              if (silu) du[e] *= silu_grad(xh[e] * ga[e] + be[e]);
              r[e] = rsd[e] * (du[e] * ga[e] - a1[e] - xh[e] * a2[e]);
            }
            if (extra != nullptr) {
              const float4 ex = __ldg(reinterpret_cast<const float4*>(extra + gpix * C + c));
              r[0] += ex.x; r[1] += ex.y; r[2] += ex.z; r[3] += ex.w;
            }
            if (dst.h16 != nullptr) {
              st_half4(dst.h16 + gpix * C + c, r[0], r[1], r[2], r[3]);
              if (dst.h16lo != nullptr) st_half4_lo(dst.h16lo + gpix * C + c, r[0], r[1], r[2], r[3]);
              csum[j].x += r[0]; csum[j].y += r[1]; csum[j].z += r[2]; csum[j].w += r[3];
              continue;
            }
            float* o;
            int acc;
            if (c < dst.c0) {
              o = dst.p0 + gpix * dst.c0 + c;
              acc = dst.acc0;
            } else {
              o = dst.p1 + gpix * dst.c1 + (c - dst.c0);
              acc = dst.acc1;
            }
            float4 outv = make_float4(r[0], r[1], r[2], r[3]);
            if (acc) {
              const float4 old = *reinterpret_cast<const float4*>(o);
              outv.x += old.x; outv.y += old.y; outv.z += old.z; outv.w += old.w;
            }
            *reinterpret_cast<float4*>(o) = outv;
          }
        }
      }
    }
    __syncthreads();
    if (threadIdx.x == 0 && it + RS_STAGES < nchunks)
      rs.issue(s, x, dy, base_pix + p_begin + (it + RS_STAGES) * pix, min(pix, p_end - p_begin - (it + RS_STAGES) * pix));
  }
  if (dst.h16 != nullptr && dst.colsum != nullptr) {
    reduce_over_subs(csum, m, red);
    if (!m.active || (m.ppi > 1 && m.sub != 0)) return;
    const float inv = dst.inv_scale != nullptr ? __ldg(dst.inv_scale) : 1.f;
#pragma unroll
    for (int j = 0; j < NL; ++j) {
      const int l = m.t_lane + j * m.stride;
      if (l < m.lanes) {
        atomicAdd(dst.colsum + 4 * l + 0, inv * csum[j].x);
        atomicAdd(dst.colsum + 4 * l + 1, inv * csum[j].y);
        atomicAdd(dst.colsum + 4 * l + 2, inv * csum[j].z);
        atomicAdd(dst.colsum + 4 * l + 3, inv * csum[j].w);
      }
    }
  }
}

// ------------------------------------------------------------------ casts and column sums
template <bool IN_F16>
__global__ void __launch_bounds__(TPB)
cast_colsum_kernel(const void* __restrict__ in_, __half* __restrict__ out16, long long rows, int C,
                   float* __restrict__ colsum, const float* __restrict__ inv_scale) {
  // blockIdx.y: tile of up to 4*TPB channels (one float4 lane per thread); blockIdx.x: row chunk
  const int c0 = blockIdx.y * (4 * TPB);
  const int Ct = min(C - c0, 4 * TPB);
  const LaneMap m = lane_map(Ct);
  const long long per = cdiv(rows, gridDim.x);
  const long long r_begin = blockIdx.x * per;
  const long long r_end = min(rows, r_begin + per);
  __shared__ float4 red[TPB];
  float4 s = make_float4(0, 0, 0, 0);
  const int c = c0 + 4 * m.t_lane;
  constexpr int U = 4;  // rows per trip: all loads issued before the first use
  for (long long r = r_begin + m.sub; m.active && r < r_end; r += U * m.ppi) {
    float4 v[U];
    uint2 raw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long rr = r + static_cast<long long>(u) * m.ppi;
      v[u] = make_float4(0, 0, 0, 0);
      raw[u] = make_uint2(0, 0);
      if (rr < r_end) {
        if (IN_F16) raw[u] = __ldg(reinterpret_cast<const uint2*>(static_cast<const __half*>(in_) + rr * C + c));
        else v[u] = __ldg(reinterpret_cast<const float4*>(static_cast<const float*>(in_) + rr * C + c));
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long rr = r + static_cast<long long>(u) * m.ppi;
      if (IN_F16) {
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&raw[u].x));
        const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&raw[u].y));
        v[u] = make_float4(a.x, a.y, b.x, b.y);
      } else if (out16 != nullptr && rr < r_end) {
        st_half4(out16 + rr * C + c, v[u].x, v[u].y, v[u].z, v[u].w);
      }
      s.x += v[u].x; s.y += v[u].y; s.z += v[u].z; s.w += v[u].w;
    }
  }
  if (colsum == nullptr) return;
  {
    float4 sv[1] = {s};
    reduce_over_subs(sv, m, red);
    s = sv[0];
  }
  if (!m.active || (m.ppi > 1 && m.sub != 0)) return;
  const float inv = inv_scale != nullptr ? __ldg(inv_scale) : 1.f;
  atomicAdd(colsum + c + 0, inv * s.x);
  atomicAdd(colsum + c + 1, inv * s.y);
  atomicAdd(colsum + c + 2, inv * s.z);
  atomicAdd(colsum + c + 3, inv * s.w);
}


// staged fp32 -> fp16 cast + column sums (single channel tile: C <= 4 * TPB)
__global__ void __launch_bounds__(TPB)
cast_colsum_staged_kernel(const float* __restrict__ in, __half* __restrict__ out16, long long rows, int C,
                          float* __restrict__ colsum, const float* __restrict__ inv_scale, int pix, int stage_bytes) {
  extern __shared__ __align__(128) uint8_t rs_mem[];
  __shared__ __align__(8) uint64_t full[RS_STAGES];
  __shared__ float4 red[TPB];
  const LaneMap m = lane_map(C);
  const long long per = cdiv(cdiv(rows, static_cast<long long>(gridDim.x)), pix) * pix;
  const long long r_begin = blockIdx.x * per;
  const long long r_end = min(rows, r_begin + per);
  const int nchunks = r_end > r_begin ? static_cast<int>(cdiv(r_end - r_begin, pix)) : 0;
  const Src2 x{in, nullptr, C, 0};
  RowStream rs{rs_mem, full, stage_bytes, C * 4, 0, 0, pix};
  if (threadIdx.x == 0) {
    for (int s = 0; s < RS_STAGES; ++s) rs_bar_init(&full[s]);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int it = 0; it < RS_STAGES && it < nchunks; ++it)
      rs.issue(it, x, nullptr, r_begin + static_cast<long long>(it) * pix,
               static_cast<int>(min(static_cast<long long>(pix), r_end - r_begin - static_cast<long long>(it) * pix)));
  float4 sacc = make_float4(0, 0, 0, 0);
  const int c = 4 * m.t_lane;
  for (int it = 0; it < nchunks; ++it) {
    const int s = it % RS_STAGES;
    rs_wait(&full[s], static_cast<uint32_t>(it / RS_STAGES) & 1u);
    const RowStage st = rs.stage(s);
    const long long r0 = r_begin + static_cast<long long>(it) * pix;
    const int np = static_cast<int>(min(static_cast<long long>(pix), r_end - r0));
    if (m.active) {
      for (int pl = m.sub; pl < np; pl += m.ppi) {
        const float4 v = *reinterpret_cast<const float4*>(st.x0 + static_cast<size_t>(pl) * C + c);
        if (out16 != nullptr) st_half4(out16 + (r0 + pl) * C + c, v.x, v.y, v.z, v.w);
        sacc.x += v.x; sacc.y += v.y; sacc.z += v.z; sacc.w += v.w;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0 && it + RS_STAGES < nchunks)
      rs.issue(s, x, nullptr, r_begin + static_cast<long long>(it + RS_STAGES) * pix,
               static_cast<int>(min(static_cast<long long>(pix), r_end - r_begin - static_cast<long long>(it + RS_STAGES) * pix)));
  }
  if (colsum == nullptr) return;
  {
    float4 sv[1] = {sacc};
    reduce_over_subs(sv, m, red);
    sacc = sv[0];
  }
  if (!m.active || (m.ppi > 1 && m.sub != 0)) return;
  const float inv = inv_scale != nullptr ? __ldg(inv_scale) : 1.f;
  atomicAdd(colsum + c + 0, inv * sacc.x);
  atomicAdd(colsum + c + 1, inv * sacc.y);
  atomicAdd(colsum + c + 2, inv * sacc.z);
  atomicAdd(colsum + c + 3, inv * sacc.w);
}

// staged GroupNorm (+FiLM, +SiLU) apply
template <int NL, bool DROP>
__global__ void __launch_bounds__(TPB)
gn_apply_staged_kernel(Src2 x, int HW, int G, const float* __restrict__ sums, const float* __restrict__ gamma,
                       const float* __restrict__ beta, const float* __restrict__ film, int film_ld, int film_off,
                       int silu, __half* __restrict__ y16, __half* __restrict__ raw16, int pix, int stage_bytes,
                       DropK drop) {
  extern __shared__ __align__(128) uint8_t rs_mem[];
  __shared__ __align__(8) uint64_t full[RS_STAGES];
  const int C = x.c0 + x.c1;
  const LaneMap m = lane_map(C);
  const int n = blockIdx.y;
  const int per = static_cast<int>(cdiv(cdiv(HW, gridDim.x), pix)) * pix;
  const int p_begin = blockIdx.x * per;
  const int p_end = min(HW, p_begin + per);
  const int nchunks = p_end > p_begin ? static_cast<int>(cdiv(p_end - p_begin, pix)) : 0;
  RowStream rs{rs_mem, full, stage_bytes, x.c0 * 4, x.c1 * 4, 0, pix};
  if (threadIdx.x == 0) {
    for (int s = 0; s < RS_STAGES; ++s) rs_bar_init(&full[s]);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const long long base_pix = static_cast<long long>(n) * HW;
  if (threadIdx.x == 0)
    for (int it = 0; it < RS_STAGES && it < nchunks; ++it)
      rs.issue(it, x, nullptr, base_pix + p_begin + it * pix, min(pix, p_end - p_begin - it * pix));
  GnCoef<NL> k;
  if (m.active) gn_coefs(k, m, n, C, G, HW, sums, gamma, beta, film, film_ld, film_off);
  const unsigned long long seed = drop_seed<DROP>(drop);
  for (int it = 0; it < nchunks; ++it) {
    const int s = it % RS_STAGES;
    rs_wait(&full[s], static_cast<uint32_t>(it / RS_STAGES) & 1u);
    const RowStage st = rs.stage(s);
    const int np = min(pix, p_end - p_begin - it * pix);
    if (m.active) {
      for (int pl = m.sub; pl < np; pl += m.ppi) {
        const long long gpix = base_pix + p_begin + it * pix + pl;
#pragma unroll
        for (int j = 0; j < NL; ++j) {
          const int l = m.t_lane + j * m.stride;
          if (l < m.lanes) {
            const float4 v = rs_ld_x(st, x, pl, 4 * l);
            float u0 = (v.x * k.rs[j].x + k.nm[j].x) * k.ga[j].x + k.be[j].x;
            float u1 = (v.y * k.rs[j].y + k.nm[j].y) * k.ga[j].y + k.be[j].y;
            float u2 = (v.z * k.rs[j].z + k.nm[j].z) * k.ga[j].z + k.be[j].z;
            float u3 = (v.w * k.rs[j].w + k.nm[j].w) * k.ga[j].w + k.be[j].w;
            if (silu) {
              u0 = siluf_(u0); u1 = siluf_(u1); u2 = siluf_(u2); u3 = siluf_(u3);
            }
            if (DROP) {
              const float4 f = drop_factors(drop, seed, gpix * m.lanes + l);
              u0 *= f.x; u1 *= f.y; u2 *= f.z; u3 *= f.w;
            }
            st_half4(y16 + gpix * C + 4 * l, u0, u1, u2, u3);
            if (raw16 != nullptr) st_half4(raw16 + gpix * C + 4 * l, v.x, v.y, v.z, v.w);
          }
        }
      }
    }
    __syncthreads();
    if (threadIdx.x == 0 && it + RS_STAGES < nchunks)
      rs.issue(s, x, nullptr, base_pix + p_begin + (it + RS_STAGES) * pix, min(pix, p_end - p_begin - (it + RS_STAGES) * pix));
  }
}


__global__ void dropout_set_seed_kernel(unsigned long long* slot, unsigned long long seed) { *slot = seed; }

__global__ void __launch_bounds__(TPB)
dropout_mask_kernel(unsigned long long seed, uint32_t stream, uint32_t thresh, float scale, long long n,
                    float* __restrict__ out) {
  const long long nq = cdiv(n, 4);
  for (long long q = blockIdx.x * static_cast<long long>(TPB) + threadIdx.x; q < nq;
       q += static_cast<long long>(gridDim.x) * TPB) {
    const float4 f = drop_factors(seed, stream, thresh, scale, q);
    const float fv[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (4 * q + e < n) out[4 * q + e] = fv[e];
  }
}

// Column sums of an fp16 matrix (bias gradients of the linear layers): 8 channels (one 16-byte load) per thread and
// 8 rows in flight per trip. The generic cast_colsum path moved 8 bytes per load, far below the HBM rate on the
// (rows x 3072) FFN / qkv gradients.
__global__ void __launch_bounds__(TPB)
colsum_f16_wide_kernel(const __half* __restrict__ in, long long rows, int C, float* __restrict__ colsum,
                       const float* __restrict__ inv_scale) {
  __shared__ float4 red[TPB];
  const int c0 = blockIdx.y * (8 * TPB);
  const int Ct = min(C - c0, 8 * TPB);
  const int lanes = Ct >> 3;
  int ppi, t_lane, sub;
  bool active;
  if (lanes <= TPB) {
    ppi = TPB / lanes;
    t_lane = threadIdx.x % lanes;
    sub = threadIdx.x / lanes;
    active = sub < ppi;
  } else {
    ppi = 1; t_lane = threadIdx.x; sub = 0; active = true;
  }
  const long long per = cdiv(rows, gridDim.x);
  const long long r_begin = blockIdx.x * per;
  const long long r_end = min(rows, r_begin + per);
  const int c = c0 + 8 * t_lane;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  constexpr int U = 8;
  if (active) {
    for (long long r = r_begin + sub; r < r_end; r += static_cast<long long>(U) * ppi) {
      uint4 raw[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long rr = r + static_cast<long long>(u) * ppi;
        raw[u] = rr < r_end ? __ldg(reinterpret_cast<const uint4*>(in + rr * C + c)) : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const __half2* h = reinterpret_cast<const __half2*>(&raw[u]);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 f = __half22float2(h[q]);
          acc[2 * q] += f.x;
          acc[2 * q + 1] += f.y;
        }
      }
    }
  }
  // sum over the row sub-slots of the CTA, then one atomic per channel
  for (int half_i = 0; half_i < 2; ++half_i) {
    if (ppi > 1) {
      red[threadIdx.x] = active ? make_float4(acc[4 * half_i], acc[4 * half_i + 1], acc[4 * half_i + 2], acc[4 * half_i + 3])
                                : make_float4(0, 0, 0, 0);
      __syncthreads();
      if (active && sub == 0) {
        float4 sm = red[t_lane];
        for (int i = 1; i < ppi; ++i) {
          const float4 o = red[t_lane + i * lanes];
          sm.x += o.x; sm.y += o.y; sm.z += o.z; sm.w += o.w;
        }
        acc[4 * half_i] = sm.x; acc[4 * half_i + 1] = sm.y; acc[4 * half_i + 2] = sm.z; acc[4 * half_i + 3] = sm.w;
      }
      __syncthreads();
    }
  }
  if (!active || (ppi > 1 && sub != 0)) return;
  const float inv = inv_scale != nullptr ? __ldg(inv_scale) : 1.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) atomicAdd(colsum + c + e, inv * acc[e]);
}

__global__ void cast_f32_to_f16_kernel(const float* __restrict__ in, __half* __restrict__ out, long long n) {
  long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 4;
  for (; i + 3 < n; i += stride) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(in + i));
    st_half4(out + i, v.x, v.y, v.z, v.w);
  }
  if (i < n) {
    for (long long k = i; k < n && k < i + 4; ++k) out[k] = __float2half_rn(in[k]);
  }
}

// out[r][:] = half(in[r][:] * rowscale[r])  (T5 features times their 0/1 token mask, language_models/factory.py:101)
__global__ void cast_rowscale_f16_kernel(const float* __restrict__ in, const float* __restrict__ rowscale,
                                         __half* __restrict__ out, long long rows, int D) {
  const int per_row = D / 4;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x, total = rows * per_row;
  for (; i < total; i += stride) {
    const long long r = i / per_row;
    const float m = __ldg(rowscale + r);
    const float4 v = __ldg(reinterpret_cast<const float4*>(in) + i);
    st_half4(out + 4 * i, v.x * m, v.y * m, v.z * m, v.w * m);
  }
}

__global__ void add_f32_kernel(float* __restrict__ dst, const float* __restrict__ a,
                               const float* __restrict__ b, long long n) {
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) dst[i] = a[i] + b[i];
}
__global__ void axpy_f32_kernel(float* __restrict__ dst, const float* __restrict__ a, float alpha,
                                long long n, int acc) {
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) dst[i] = (acc ? dst[i] : 0.f) + alpha * a[i];
}
__global__ void scale_f32_kernel(float* __restrict__ dst, const float* __restrict__ a, const float* __restrict__ s,
                                 long long n) {
  const float f = *s;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) dst[i] = f * a[i];
}

// ------------------------------------------------------------------ softmax (warp per row)
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ scores, __half* __restrict__ P16, long long rows, int S, int ld,
                    const float* __restrict__ mask, long long rows_per_batch) {
  const int lane = threadIdx.x & 31;
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* s = scores + row * ld;
  const float* mk = mask != nullptr ? mask + (row / rows_per_batch) * S : nullptr;
  float mx = -INFINITY;
  for (int i = lane; i < S; i += 32) {
    float v = s[i];
    if (mk != nullptr && mk[i] == 0.f) v = -INFINITY;
    mx = fmaxf(mx, v);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int i = lane; i < S; i += 32) {
    float v = s[i];
    if (mk != nullptr && mk[i] == 0.f) v = -INFINITY;
    sum += expf(v - mx);
  }
  sum = warp_sum(sum);
  const float inv = 1.0f / sum;
  __half* o = P16 + row * ld;
  for (int i = lane; i < S; i += 32) {
    float v = s[i];
    if (mk != nullptr && mk[i] == 0.f) v = -INFINITY;
    o[i] = __float2half_rn(expf(v - mx) * inv);
  }
}

__global__ void __launch_bounds__(256)
softmax_bwd_rows_kernel(const __half* __restrict__ P16, const float* __restrict__ dP,
                        __half* __restrict__ dS16, long long rows, int S, int ld, float scale) {
  const int lane = threadIdx.x & 31;
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const __half* p = P16 + row * ld;
  const float* d = dP + row * ld;
  float dot = 0.f;
  for (int i = lane; i < S; i += 32) dot += __half2float(p[i]) * d[i];
  dot = warp_sum(dot);
  __half* o = dS16 + row * ld;
  for (int i = lane; i < S; i += 32) o[i] = __float2half_rn(__half2float(p[i]) * (d[i] - dot) * scale);
}

// ------------------------------------------------------------------ LayerNorm (block per row)
__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float t = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.f;
  if (w == 0) {
    t = warp_sum(t);
    if (l == 0) sh[0] = t;
  }
  __syncthreads();
  return sh[0];
}

__global__ void __launch_bounds__(256)
layernorm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                     __half* __restrict__ y16, float* __restrict__ stats, int D) {
  __shared__ float sh[32];
  const long long row = blockIdx.x;
  const float* xr = x + row * D;
  float s = 0.f;
  for (int i = threadIdx.x; i < D; i += blockDim.x) s += xr[i];
  const float mean = block_sum(s, sh) / D;
  float q = 0.f;
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    const float d = xr[i] - mean;
    q += d * d;
  }
  const float var = block_sum(q, sh) / D;
  const float rstd = rsqrtf(var + 1e-5f);
  if (threadIdx.x == 0) {
    stats[row * 2] = mean;
    stats[row * 2 + 1] = rstd;
  }
  for (int i = threadIdx.x; i < D; i += blockDim.x)
    y16[row * D + i] = __float2half_rn(w != nullptr ? (xr[i] - mean) * rstd * w[i] + b[i] : (xr[i] - mean) * rstd);
}

constexpr int LN_ROWS = 16;
constexpr int LN_COLS = 8;  // columns per thread => D <= 256 * 8
__global__ void __launch_bounds__(256)
layernorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ stats,
                     const float* __restrict__ dy, float* __restrict__ dx, int acc_dx,
                     float* __restrict__ dw, float* __restrict__ db, const float* __restrict__ inv_scale,
                     long long rows, int D) {
  __shared__ float sh[32];
  const long long r0 = static_cast<long long>(blockIdx.x) * LN_ROWS;
  float aw[LN_COLS], abias[LN_COLS], wv[LN_COLS];
#pragma unroll
  for (int j = 0; j < LN_COLS; ++j) {
    aw[j] = 0.f;
    abias[j] = 0.f;
    const int i = threadIdx.x + j * 256;
    wv[j] = i < D ? (w != nullptr ? w[i] : 1.f) : 0.f;
  }
  for (int rr = 0; rr < LN_ROWS; ++rr) {
    const long long row = r0 + rr;
    if (row >= rows) break;  // uniform across the block
    const float mean = stats[row * 2], rstd = stats[row * 2 + 1];
    float xh[LN_COLS], g[LN_COLS];
    float c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int j = 0; j < LN_COLS; ++j) {
      const int i = threadIdx.x + j * 256;
      xh[j] = 0.f;
      g[j] = 0.f;
      if (i < D) {
        xh[j] = (x[row * D + i] - mean) * rstd;
        const float d = dy[row * D + i];
        g[j] = d * wv[j];
        aw[j] += d * xh[j];
        abias[j] += d;
        c1 += g[j];
        c2 += g[j] * xh[j];
      }
    }
    c1 = block_sum(c1, sh) / D;
    c2 = block_sum(c2, sh) / D;
#pragma unroll
    for (int j = 0; j < LN_COLS; ++j) {
      const int i = threadIdx.x + j * 256;
      if (i < D) {
        const float v = rstd * (g[j] - c1 - xh[j] * c2);
        float* o = dx + row * D + i;
        *o = acc_dx ? (*o + v) : v;
      }
    }
  }
  if (dw == nullptr) return;
  const float inv = inv_scale != nullptr ? __ldg(inv_scale) : 1.f;
#pragma unroll
  for (int j = 0; j < LN_COLS; ++j) {
    const int i = threadIdx.x + j * 256;
    if (i < D) {
      atomicAdd(dw + i, inv * aw[j]);
      atomicAdd(db + i, inv * abias[j]);
    }
  }
}

// ---- LayerNorm affine folded into the following Linear (cross-attention kv_cond, unet.py:263-264,304):
//   kv = Linear(LN(x)) = xhat (W diag(w))^T + (W b + bias)
__global__ void fold_ln_weight_kernel(const float* __restrict__ W, const float* __restrict__ w, __half* __restrict__ out,
                                      __half* __restrict__ lo, long long rows, int D) {
  const long long total = rows * D;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total; i += gs) {
    const float v = W[i] * w[i % D];
    const __half h = __float2half_rn(v);
    out[i] = h;
    if (lo != nullptr) lo[i] = __float2half_rn(v - __half2float(h));
  }
}
// out = in - fp16(in): what rounding a weight to fp16 leaves behind (its second fp16 plane)
__global__ void f16_residual_kernel(const float* __restrict__ in, float* __restrict__ out, long long n) {
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < n; i += gs) out[i] = in[i] - __half2float(__float2half_rn(in[i]));
}
__global__ void fold_ln_bias_kernel(const float* __restrict__ W, const float* __restrict__ b, const float* __restrict__ bias,
                                    float* __restrict__ out, int rows, int D) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float s = 0.f;
  for (int j = lane; j < D; j += 32) s += W[static_cast<long long>(row) * D + j] * b[j];
  s = warp_sum(s);
  if (lane == 0) out[row] = s + bias[row];
}
// gradients back through the fold. dWf: fp32 [rows][D] gradient of the folded weight (already unscaled),
// dbf: [rows] gradient of the folded bias (unscaled).
//   dW[i][j] += dWf[i][j] w[j] + dbf[i] b[j];  dw[j] += sum_i dWf[i][j] W[i][j];  db[j] += sum_i dbf[i] W[i][j]
__global__ void unfold_ln_grads_kernel(const float* __restrict__ dWf, const float* __restrict__ dbf,
                                       const float* __restrict__ W, const float* __restrict__ w,
                                       const float* __restrict__ b, float* __restrict__ dW,
                                       float* __restrict__ dw, float* __restrict__ db, int rows, int D) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= D) return;
  const int r0 = blockIdx.y * 64;
  const int r1 = min(rows, r0 + 64);
  const float wj = w[j], bj = b[j];
  float a = 0.f, c = 0.f;
  for (int i = r0; i < r1; ++i) {
    const long long o = static_cast<long long>(i) * D + j;
    const float g = dWf[o];
    const float Wij = W[o];
    if (dW != nullptr) dW[o] += g * wj + dbf[i] * bj;
    a += g * Wij;
    c += dbf[i] * Wij;
  }
  if (dw != nullptr) atomicAdd(dw + j, a);
  if (db != nullptr) atomicAdd(db + j, c);
}

// ------------------------------------------------------------------ embeddings / activations
// grid.y: the key (1 for the time embedding). sinf/cosf, not the fast intrinsics: micro arguments reach ~1e3 rad.
__global__ void sinusoid_embed_kernel(const long long* __restrict__ times, MicroKeys micro,
                                      const float* __restrict__ freq, int B, int half, long long key_stride,
                                      __half* __restrict__ e16) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * half) return;
  const int b = idx / half, i = idx - b * half, k = blockIdx.y;
  float v;
  if (times != nullptr) {
    v = static_cast<float>(times[b]);
  } else {
    const float d = micro.defaults[k];
    v = micro.values[k] != nullptr ? micro.values[k][b] : d;
    v = (micro.scale_mask >> k) & 1u ? fminf(v / d, 1.0f) * d : v * 1000.0f;
  }
  const float w = freq[i];
  const float a = v * w;
  __half* e = e16 + k * key_stride + static_cast<long long>(b) * 2 * half;
  e[i] = __float2half_rn(sinf(a));
  e[half + i] = __float2half_rn(cosf(a));
}

__global__ void silu_f16_kernel(const float* __restrict__ x, __half* __restrict__ y, long long n) {
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) y[i] = __float2half_rn(siluf_(x[i]));
}
__global__ void silu_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                float* __restrict__ dx, long long n, int acc) {
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) {
    const float v = dy[i] * silu_grad(x[i]);
    dx[i] = acc ? dx[i] + v : v;
  }
}
__global__ void gelu_bwd_kernel(const __half* __restrict__ u16, const float* __restrict__ dg,
                                __half* __restrict__ du16, long long n) {
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) {
    const float u = __half2float(u16[i]);
    const float cdf = 0.5f * (1.0f + erff(u * 0.70710678118654752440f));
    const float pdf = 0.39894228040143267794f * expf(-0.5f * u * u);
    du16[i] = __float2half_rn(dg[i] * (cdf + u * pdf));
  }
}

__global__ void masked_mean_kernel(const float* __restrict__ x, const float* __restrict__ mask,
                                   float* __restrict__ y, __half* __restrict__ y16, int S, int D) {
  const int b = blockIdx.y;
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  float s = 0.f, cnt = 0.f;
  for (int t = 0; t < S; ++t) {
    const float mk = mask != nullptr ? mask[static_cast<long long>(b) * S + t] : 1.f;
    s += mk * x[(static_cast<long long>(b) * S + t) * D + d];
    cnt += mk;
  }
  const float v = s / cnt;
  y[static_cast<long long>(b) * D + d] = v;
  if (y16 != nullptr) y16[static_cast<long long>(b) * D + d] = __float2half_rn(v);
}
__global__ void masked_mean_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ mask,
                                       float* __restrict__ dx, int acc, int S, int D) {
  const int b = blockIdx.z, t = blockIdx.y;
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  float cnt = 0.f;
  for (int i = 0; i < S; ++i) cnt += mask != nullptr ? mask[static_cast<long long>(b) * S + i] : 1.f;
  const float mk = mask != nullptr ? mask[static_cast<long long>(b) * S + t] : 1.f;
  const float v = mk * dy[static_cast<long long>(b) * D + d] / cnt;
  float* o = dx + (static_cast<long long>(b) * S + t) * D + d;
  *o = acc ? (*o + v) : v;
}

// ------------------------------------------------------------------ conv helpers
__global__ void im2col3x3_kernel(const float* __restrict__ x, __half* __restrict__ col, int N, int H, int W,
                                 int C, int stride, int Ho, int Wo) {
  const int lanes = C >> 2;
  const long long total = static_cast<long long>(N) * Ho * Wo * 9 * lanes;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total; i += gs) {
    const int l = static_cast<int>(i % lanes);
    long long t = i / lanes;
    const int tap = static_cast<int>(t % 9);
    t /= 9;
    const int wo = static_cast<int>(t % Wo);
    t /= Wo;
    const int ho = static_cast<int>(t % Ho);
    const int n = static_cast<int>(t / Ho);
    const int h = ho * stride + tap / 3 - 1;
    const int w = wo * stride + tap % 3 - 1;
    float4 v = make_float4(0, 0, 0, 0);
    if (h >= 0 && h < H && w >= 0 && w < W)
      v = __ldg(reinterpret_cast<const float4*>(x + ((static_cast<long long>(n) * H + h) * W + w) * C + 4 * l));
    st_half4(col + ((static_cast<long long>(n) * Ho + ho) * Wo + wo) * 9 * C + tap * C + 4 * l, v.x, v.y, v.z, v.w);
  }
}

__global__ void col2im3x3_kernel(const float* __restrict__ dcol, float* __restrict__ dx, int acc, int N, int H,
                                 int W, int C, int stride, int Ho, int Wo) {
  const int lanes = C >> 2;
  const long long total = static_cast<long long>(N) * H * W * lanes;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total; i += gs) {
    const int l = static_cast<int>(i % lanes);
    long long t = i / lanes;
    const int w = static_cast<int>(t % W);
    t /= W;
    const int h = static_cast<int>(t % H);
    const int n = static_cast<int>(t / H);
    float4 s = make_float4(0, 0, 0, 0);
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int hn = h + 1 - tap / 3, wn = w + 1 - tap % 3;
      if (hn < 0 || wn < 0 || (hn % stride) != 0 || (wn % stride) != 0) continue;
      const int ho = hn / stride, wo = wn / stride;
      if (ho >= Ho || wo >= Wo) continue;
      const float4 v = __ldg(reinterpret_cast<const float4*>(
          dcol + ((static_cast<long long>(n) * Ho + ho) * Wo + wo) * 9 * C + tap * C + 4 * l));
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    float* o = dx + ((static_cast<long long>(n) * H + h) * W + w) * C + 4 * l;
    if (acc) {
      const float4 old = *reinterpret_cast<const float4*>(o);
      s.x += old.x; s.y += old.y; s.z += old.z; s.w += old.w;
    }
    *reinterpret_cast<float4*>(o) = s;
  }
}

__global__ void im2col_input_kernel(const float* __restrict__ x, const float* __restrict__ inv_std,
                                    __half* __restrict__ col, int N, int Cin, int H, int W) {
  const long long total = static_cast<long long>(N) * H * W;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total; i += gs) {
    const int w = static_cast<int>(i % W);
    const long long t = i / W;
    const int h = static_cast<int>(t % H);
    const int n = static_cast<int>(t / H);
    const float sc = inv_std != nullptr ? inv_std[n] : 1.f;
    __align__(16) __half v[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) v[k] = __float2half_rn(0.f);
    for (int tap = 0; tap < 9; ++tap) {
      const int hh = h + tap / 3 - 1, ww = w + tap % 3 - 1;
      if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
      for (int c = 0; c < Cin; ++c)
        v[tap * Cin + c] = __float2half_rn(sc * x[((static_cast<long long>(n) * Cin + c) * H + hh) * W + ww]);
    }
    uint4* o = reinterpret_cast<uint4*>(col + i * 32);
    const uint4* s = reinterpret_cast<const uint4*>(v);
    o[0] = s[0]; o[1] = s[1]; o[2] = s[2]; o[3] = s[3];
  }
}

__global__ void upsample2x_f16_kernel(const float* __restrict__ x, __half* __restrict__ y, int N, int H, int W,
                                      int C) {
  const int lanes = C >> 2;
  const long long total = static_cast<long long>(N) * (2 * H) * (2 * W) * lanes;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total; i += gs) {
    const int l = static_cast<int>(i % lanes);
    long long t = i / lanes;
    const int w2 = static_cast<int>(t % (2 * W));
    t /= (2 * W);
    const int h2 = static_cast<int>(t % (2 * H));
    const int n = static_cast<int>(t / (2 * H));
    const float4 v = __ldg(reinterpret_cast<const float4*>(
        x + ((static_cast<long long>(n) * H + (h2 >> 1)) * W + (w2 >> 1)) * C + 4 * l));
    st_half4(y + ((static_cast<long long>(n) * 2 * H + h2) * 2 * W + w2) * C + 4 * l, v.x, v.y, v.z, v.w);
  }
}
__global__ void upsample2x_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int acc, int N,
                                      int H, int W, int C) {
  const int lanes = C >> 2;
  const long long total = static_cast<long long>(N) * H * W * lanes;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total; i += gs) {
    const int l = static_cast<int>(i % lanes);
    long long t = i / lanes;
    const int w = static_cast<int>(t % W);
    t /= W;
    const int h = static_cast<int>(t % H);
    const int n = static_cast<int>(t / H);
    float4 s = make_float4(0, 0, 0, 0);
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(
            dy + ((static_cast<long long>(n) * 2 * H + 2 * h + a) * 2 * W + 2 * w + b) * C + 4 * l));
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      }
    float* o = dx + ((static_cast<long long>(n) * H + h) * W + w) * C + 4 * l;
    if (acc) {
      const float4 old = *reinterpret_cast<const float4*>(o);
      s.x += old.x; s.y += old.y; s.z += old.z; s.w += old.w;
    }
    *reinterpret_cast<float4*>(o) = s;
  }
}

// TANH: model_output_scale s (diffusion.py:83-85): y = s * tanh(x / s) with the accurate tanhf, also written to keep
// (the NCHW output the backward seed reads) when keep is not null
template <bool TANH>
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ x, int ldc, float* __restrict__ y, int N, int C,
                                    int HW, float s, float* __restrict__ keep) {
  const long long total = static_cast<long long>(N) * C * HW;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total; i += gs) {
    const int p = static_cast<int>(i % HW);
    const long long t = i / HW;
    const int c = static_cast<int>(t % C);
    const int n = static_cast<int>(t / C);
    float v = x[(static_cast<long long>(n) * HW + p) * ldc + c];
    if (TANH) {
      v = s * tanhf(v / s);
      if (keep != nullptr) keep[i] = v;
    }
    y[i] = v;
  }
}
// d out / d o of y = s * tanh(o / s), from y itself: 1 - (y / s)^2
__device__ __forceinline__ float tanh_scale_grad(float y, float s) {
  const float t = y / s;
  return 1.f - t * t;
}
// TANH: the incoming gradient is multiplied by tanh_scale_grad(yk, s), yk in the layout of x, before the scale
template <bool TANH>
__global__ void nchw_to_nhwc_f16_kernel(const float* __restrict__ x, const float* __restrict__ scale,
                                        __half* __restrict__ y, int ldo, int N, int C, int HW, float s,
                                        const float* __restrict__ yk) {
  const long long total = static_cast<long long>(N) * HW * ldo;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  const float sc = scale != nullptr ? __ldg(scale) : 1.f;
  for (; i < total; i += gs) {
    const int c = static_cast<int>(i % ldo);
    const long long t = i / ldo;
    const int p = static_cast<int>(t % HW);
    const int n = static_cast<int>(t / HW);
    if (c >= C) {
      y[i] = __float2half_rn(0.f);
      continue;
    }
    const long long src = (static_cast<long long>(n) * C + c) * HW + p;
    float g = x[src];
    if (TANH) g *= tanh_scale_grad(yk[src], s);
    y[i] = __float2half_rn(sc * g);
  }
}

__global__ void __launch_bounds__(256)
sample_inv_std_kernel(const float* __restrict__ x, float* __restrict__ inv_std, long long per) {
  __shared__ float sh[32];
  const float* xr = x + static_cast<long long>(blockIdx.x) * per;
  float s = 0.f;
  for (long long i = threadIdx.x; i < per; i += blockDim.x) s += xr[i];
  const float mean = block_sum(s, sh) / static_cast<float>(per);
  float q = 0.f;
  for (long long i = threadIdx.x; i < per; i += blockDim.x) {
    const float d = xr[i] - mean;
    q += d * d;
  }
  const float var = block_sum(q, sh) / static_cast<float>(per - 1);  // unbiased, torch.std default
  if (threadIdx.x == 0) inv_std[blockIdx.x] = rsqrtf(var);
}

// ------------------------------------------------------------------ weight (un)packing
__global__ void pack_conv_w_kernel(const float* __restrict__ w, __half* __restrict__ p, int Co, int Ci, int taps) {
  const long long total = static_cast<long long>(Co) * Ci;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total; i += gs) {
    const int ci = static_cast<int>(i % Ci);
    const long long co = i / Ci;
    for (int t = 0; t < taps; ++t) p[(co * taps + t) * Ci + ci] = __float2half_rn(w[i * taps + t]);
  }
}
// W-folded weights of a 3x3 conv (see Engine::conv3x3_* in engine.cu): two horizontally adjacent pixels are treated as
// one pixel with twice the channels, so a Ci -> Co conv over (H, W) becomes a 2Ci -> 2Co conv over (H, W/2) on the SAME
// memory. Output column 2j+po reads input column 2(j+kwf-1)+pi through the original tap kw = 2(kwf-1)+pi-po+1 when
// that is in 0..2, else through a zero. p: [2Co][9][2Ci] fp16, row (po*Co+co), tap kh*3+kwf, column pi*Ci+ci.
__global__ void pack_conv_w_fold_kernel(const float* __restrict__ w, __half* __restrict__ p, int Co, int Ci) {
  const long long total = 4ll * Co * Ci * 9;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total; i += gs) {
    const int col = static_cast<int>(i % (2 * Ci));
    long long t = i / (2 * Ci);
    const int tap = static_cast<int>(t % 9);
    const int row = static_cast<int>(t / 9);
    const int pi = col / Ci, ci = col - pi * Ci, po = row / Co, co = row - po * Co;
    const int kh = tap / 3, kwf = tap - 3 * kh;
    const int kw = 2 * (kwf - 1) + pi - po + 1;
    float v = 0.f;
    if (kw >= 0 && kw <= 2) v = w[(static_cast<long long>(co) * Ci + ci) * 9 + kh * 3 + kw];
    p[i] = __float2half_rn(v);
  }
}
// g [Co][Ci][3][3] += inv_scale * (the entries of the folded gradient packed [2Co][9][2Ci] that map to each tap)
__global__ void unpack_conv_wgrad_fold_kernel(const float* __restrict__ packed, float* __restrict__ g, int Co, int Ci,
                                              const float* __restrict__ inv_scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Co * Ci * 9) return;
  const int tap = i % 9, ci = (i / 9) % Ci, co = i / (9 * Ci);
  const int kh = tap / 3, kw = tap - 3 * kh;
  float acc = 0.f;
  for (int po = 0; po < 2; ++po)
    for (int pi = 0; pi < 2; ++pi) {
      const int num = kw - 1 - pi + po;  // = 2 (kwf - 1)
      if (num & 1) continue;
      const int kwf = num / 2 + 1;
      if (kwf < 0 || kwf > 2) continue;
      acc += packed[(static_cast<long long>(po * Co + co) * 9 + kh * 3 + kwf) * (2 * Ci) + pi * Ci + ci];
    }
  const float inv = inv_scale != nullptr ? __ldg(inv_scale) : 1.f;
  g[i] += inv * acc;
}
__global__ void pack_conv_in_w_kernel(const float* __restrict__ w, __half* __restrict__ p, int Co, int Ci) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Co * 32) return;
  const int co = i / 32, k = i % 32;
  float v = 0.f;
  if (k < 9 * Ci) {
    const int tap = k / Ci, c = k % Ci;
    v = w[(static_cast<long long>(co) * Ci + c) * 9 + tap];
  }
  p[i] = __float2half_rn(v);
}
// packed [Co][taps][ci_ld] -> g [Co][Ci][taps] (+=). One CTA per (co, 256 input channels): coalesced reads per
// tap, transpose through shared memory (row stride `taps` = 9 words is odd: conflict-free), contiguous writes.
__global__ void __launch_bounds__(256)
unpack_conv_wgrad_kernel(const float* __restrict__ packed, float* __restrict__ g, int Co, int Ci, int taps,
                         int ci_ld, const float* __restrict__ inv_scale) {
  __shared__ float sm[9 * 256];
  const int co = blockIdx.x;
  const int ci0 = blockIdx.y * 256;
  const int n = min(256, Ci - ci0);
  const float inv = inv_scale != nullptr ? __ldg(inv_scale) : 1.f;
  if (static_cast<int>(threadIdx.x) < n)
    for (int t = 0; t < taps; ++t)
      sm[threadIdx.x * taps + t] = packed[(static_cast<long long>(co) * taps + t) * ci_ld + ci0 + threadIdx.x];
  __syncthreads();
  float* dst = g + (static_cast<long long>(co) * Ci + ci0) * taps;
  for (int idx = threadIdx.x; idx < n * taps; idx += 256) dst[idx] += inv * sm[idx];
}
__global__ void unpack_conv_in_wgrad_kernel(const float* __restrict__ packed, float* __restrict__ g, int Co,
                                            int Ci, const float* __restrict__ inv_scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Co * Ci * 9) return;
  const int tap = i % 9;
  const int c = (i / 9) % Ci;
  const int co = i / (9 * Ci);
  const float inv = inv_scale != nullptr ? __ldg(inv_scale) : 1.f;
  g[i] += inv * packed[co * 32 + tap * Ci + c];
}

// ------------------------------------------------------------------ gradient scale
template <bool TANH>
__global__ void __launch_bounds__(256) grad_amax_kernel(const float* __restrict__ g, long long n,
                                                        float* __restrict__ amax, float s, const float* __restrict__ yk) {
  float m = 0.f;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < n; i += gs) {
    const float v = TANH ? fabsf(g[i] * tanh_scale_grad(yk[i], s)) : fabsf(g[i]);
    if (v < INFINITY) m = fmaxf(m, v);  // skips NaN/Inf
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0 && m > 0.f)
    atomicMax(reinterpret_cast<int*>(amax), __float_as_int(m));  // non-negative floats order as ints
}
__global__ void grad_scale_finalize_kernel(const float* __restrict__ amax, float* __restrict__ scale,
                                           float* __restrict__ inv_scale) {
  const float a = amax[0];
  float s = 1.f;
  if (a > 0.f && a < INFINITY) {
    int e;
    frexpf(a, &e);  // a = m * 2^e, m in [0.5, 1)
    int k = 4 - e;
    k = max(-100, min(100, k));
    s = ldexpf(1.f, k);
  }
  scale[0] = s;
  inv_scale[0] = 1.f / s;
}

inline int grid_for(long long n, int tpb = 256, int cap = 132 * 16) {
  long long g = cdiv(n, tpb);
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

}  // namespace

// ======================================================================== launchers
// staged (bulk-copy ring) forms of the streaming kernels; MDM_GN_LEGACY=1 selects the register-fed ones
static const bool g_gn_staged = getenv("MDM_GN_LEGACY") == nullptr;
template <typename K>
static void rs_set_smem(K kernel, int bytes) {
  static std::vector<std::pair<const void*, int>> done;  // (kernel, largest size allowed so far)
  const void* key = reinterpret_cast<const void*>(kernel);
  for (auto& d : done)
    if (d.first == key) {
      if (bytes > d.second) {
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
        d.second = bytes;
      }
      return;
    }
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  done.emplace_back(key, bytes);
}
// Grid of a staged kernel: every CTA resident at once (as many per SM as their shared memory allows, at most 4) and an
// equal share of pixels each -- a partial second wave would leave most SMs idle for a whole CTA lifetime.
static int staged_chunks(int N, int HW, int pix, int smem_bytes) {
  int resident = std::min(4, std::max(1, (220 * 1024) / (smem_bytes + 6 * 1024)));
  long long want = (static_cast<long long>(resident) * 132) / N;
  const long long maxc = std::max<long long>(1, HW / (3ll * pix));  // >= 3 chunks per CTA (ring depth; prologue amortised)
  if (want > maxc) want = maxc;
  if (want < 1) want = 1;
  return static_cast<int>(want);
}
#define MDM_LAUNCH_STAGED(KERNEL, grid, smem, ...)        \
  do {                                                    \
    rs_set_smem(KERNEL, smem);                            \
    KERNEL<<<grid, TPB, smem, st>>>(__VA_ARGS__);         \
  } while (0)

void gn_stats(const Src2& x, int N, int HW, int G, float* sums, cudaStream_t st) {
  const int C = x.c0 + x.c1;
  dim3 grid(pixel_chunks(N, HW, host_ppi(C)), N);
  MDM_DISPATCH_NL(C, (gn_stats_kernel<NL><<<grid, TPB, 0, st>>>(x, HW, G, sums)));
  MDM_LAUNCHED();
}
// DROP: the kernels' dropout form, for a Dropout with p > 0 (p == 0 takes the plain instantiation)
#define MDM_DISPATCH_DROP(drop, ...)   \
  do {                                 \
    if ((drop).p > 0.f) {              \
      constexpr bool DROP = true;      \
      __VA_ARGS__;                     \
    } else {                           \
      constexpr bool DROP = false;     \
      __VA_ARGS__;                     \
    }                                  \
  } while (0)

void dropout_set_seed(unsigned long long* slot, unsigned long long seed, cudaStream_t st) {
  dropout_set_seed_kernel<<<1, 1, 0, st>>>(slot, seed);
  MDM_LAUNCHED();
}
void dropout_mask(unsigned long long seed, uint32_t stream, long long n, float p, float* out, cudaStream_t st) {
  Dropout d;
  d.p = p;
  const DropK k = drop_k(d);
  dropout_mask_kernel<<<grid_for(cdiv(n, 4), TPB, 132 * 8), TPB, 0, st>>>(seed, stream, k.thresh, k.scale, n, out);
  MDM_LAUNCHED();
}

void gn_apply(const Src2& x, int N, int HW, int G, const float* sums, const float* gamma, const float* beta,
              const float* film, int film_ld, int film_off, int silu, __half* y16, __half* raw16,
              cudaStream_t st, const Dropout& drop) {
  const int C = x.c0 + x.c1;
  const DropK dk = drop_k(drop);
  static const bool staged_apply = getenv("MDM_APPLY_LEGACY") == nullptr;
  if (g_gn_staged && staged_apply && (x.c0 % 4 == 0) && (x.c1 % 4 == 0) && (C % 8 == 0)) {
    int pix, sb;
    rs_geometry(C, 0, &pix, &sb);
    const int smem = RS_STAGES * sb;
    dim3 grid(staged_chunks(N, HW, pix, smem), N);
    MDM_DISPATCH_DROP(drop, MDM_DISPATCH_NL(C, MDM_LAUNCH_STAGED((gn_apply_staged_kernel<NL, DROP>), grid, smem, x, HW, G,
                                                                 sums, gamma, beta, film, film_ld, film_off, silu, y16,
                                                                 raw16, pix, sb, dk)));
    MDM_LAUNCHED();
    return;
  }
  dim3 grid(pixel_chunks(N, HW, host_ppi(C)), N);
  MDM_DISPATCH_DROP(drop, MDM_DISPATCH_NL(C, (gn_apply_kernel<NL, DROP><<<grid, TPB, 0, st>>>(
                                                 x, HW, G, sums, gamma, beta, film, film_ld, film_off, silu, y16, raw16, dk))));
  MDM_LAUNCHED();
}
void gn_bwd_reduce(const Src2& x, const void* dy, int dy_f16, int N, int HW, int G, const float* sums,
                   const float* gamma, const float* beta, const float* film, int film_ld, int film_off, int silu,
                   float* ab, cudaStream_t st, const Dropout& drop) {
  const int C = x.c0 + x.c1;
  const DropK dk = drop_k(drop);
  if (g_gn_staged && (x.c0 % 4 == 0) && (x.c1 % 4 == 0) && (C % 8 == 0)) {
    int pix, sb;
    rs_geometry(C, dy_f16 ? 2 : 4, &pix, &sb);
    const int smem = RS_STAGES * sb;
    dim3 grid(staged_chunks(N, HW, pix, smem), N);
    if (dy_f16)
      MDM_DISPATCH_DROP(drop, MDM_DISPATCH_NL(C, MDM_LAUNCH_STAGED((gn_bwd_reduce_staged_kernel<NL, true, DROP>), grid, smem,
                                                                   x, dy, HW, G, sums, gamma, beta, film, film_ld, film_off,
                                                                   silu, ab, pix, sb, dk)));
    else
      MDM_DISPATCH_DROP(drop, MDM_DISPATCH_NL(C, MDM_LAUNCH_STAGED((gn_bwd_reduce_staged_kernel<NL, false, DROP>), grid, smem,
                                                                   x, dy, HW, G, sums, gamma, beta, film, film_ld, film_off,
                                                                   silu, ab, pix, sb, dk)));
    MDM_LAUNCHED();
    return;
  }
  dim3 grid(pixel_chunks(N, HW, host_ppi(C)), N);
  if (dy_f16)
    MDM_DISPATCH_DROP(drop, MDM_DISPATCH_NL(C, (gn_bwd_reduce_kernel<NL, true, DROP><<<grid, TPB, 0, st>>>(
                                                   x, dy, HW, G, sums, gamma, beta, film, film_ld, film_off, silu, ab, dk))));
  else
    MDM_DISPATCH_DROP(drop, MDM_DISPATCH_NL(C, (gn_bwd_reduce_kernel<NL, false, DROP><<<grid, TPB, 0, st>>>(
                                                   x, dy, HW, G, sums, gamma, beta, film, film_ld, film_off, silu, ab, dk))));
  MDM_LAUNCHED();
}
void gn_bwd_finalize(int N, int C, int G, int HW, const float* ab, const float* gamma, const float* beta,
                     const float* film, int film_ld, int film_off, float* pg, float* dgamma, float* dbeta,
                     float* dfilm, const float* inv_scale, cudaStream_t st) {
  gn_bwd_finalize_kernel<<<N, 256, 0, st>>>(C, G, HW, ab, gamma, beta, film, film_ld, film_off, pg, dgamma,
                                            dbeta, dfilm, inv_scale);
  MDM_LAUNCHED();
}
void gn_bwd_apply(const Src2& x, const void* dy, int dy_f16, int N, int HW, int G, const float* sums,
                  const float* gamma, const float* beta, const float* film, int film_ld, int film_off, int silu,
                  const float* pg, const float* extra, const Dst2& dst, cudaStream_t st, const Dropout& drop) {
  const int C = x.c0 + x.c1;
  const DropK dk = drop_k(drop);
  if (g_gn_staged && (x.c0 % 4 == 0) && (x.c1 % 4 == 0) && (C % 8 == 0)) {
    int pix, sb;
    rs_geometry(C, dy_f16 ? 2 : 4, &pix, &sb);
    const int smem = RS_STAGES * sb;
    dim3 grid(staged_chunks(N, HW, pix, smem), N);
    if (dy_f16)
      MDM_DISPATCH_DROP(drop, MDM_DISPATCH_NL(C, MDM_LAUNCH_STAGED((gn_bwd_apply_staged_kernel<NL, true, DROP>), grid, smem,
                                                                   x, dy, HW, G, sums, gamma, beta, film, film_ld, film_off,
                                                                   silu, pg, extra, dst, pix, sb, dk)));
    else
      MDM_DISPATCH_DROP(drop, MDM_DISPATCH_NL(C, MDM_LAUNCH_STAGED((gn_bwd_apply_staged_kernel<NL, false, DROP>), grid, smem,
                                                                   x, dy, HW, G, sums, gamma, beta, film, film_ld, film_off,
                                                                   silu, pg, extra, dst, pix, sb, dk)));
    MDM_LAUNCHED();
    return;
  }
  dim3 grid(pixel_chunks(N, HW, host_ppi(C)), N);
  if (dy_f16)
    MDM_DISPATCH_DROP(drop, MDM_DISPATCH_NL(C, (gn_bwd_apply_kernel<NL, true, DROP><<<grid, TPB, 0, st>>>(
                                                   x, dy, HW, G, sums, gamma, beta, film, film_ld, film_off, silu, pg, extra,
                                                   dst, dk))));
  else
    MDM_DISPATCH_DROP(drop, MDM_DISPATCH_NL(C, (gn_bwd_apply_kernel<NL, false, DROP><<<grid, TPB, 0, st>>>(
                                                   x, dy, HW, G, sums, gamma, beta, film, film_ld, film_off, silu, pg, extra,
                                                   dst, dk))));
  MDM_LAUNCHED();
}

static dim3 colsum_grid(long long rows, int C, bool coarse) {
  const int ctiles = static_cast<int>(cdiv(C, 4 * TPB));
  const int Ct = std::min(C, 4 * TPB);
  // every CTA ends with one atomic per column: the fp16 column-sum passes are faster with few long CTAs, the
  // fp32->fp16 cast passes with many short ones.
  long long chunks = coarse ? cdiv(rows, 128ll * host_ppi(Ct)) : cdiv(rows, 2ll * host_ppi(Ct));
  const long long cap = std::max<long long>(1, (coarse ? 132 * 2 : 132 * 8) / ctiles);
  if (chunks > cap) chunks = cap;
  if (chunks < 1) chunks = 1;
  return dim3(static_cast<unsigned>(chunks), ctiles);
}
void cast_colsum(const float* in, __half* out16, long long rows, int C, float* colsum, const float* inv_scale,
                 cudaStream_t st) {
  static const bool staged_cast = getenv("MDM_CAST_LEGACY") == nullptr;
  if (g_gn_staged && staged_cast && C <= 4 * TPB && C % 8 == 0 && rows >= 4096) {
    int pix, sb;
    rs_geometry(C, 0, &pix, &sb);
    const int smem = RS_STAGES * sb;
    const long long chunks = staged_chunks(1, static_cast<int>(std::min<long long>(rows, 2147483647ll)), pix, smem);
    MDM_LAUNCH_STAGED(cast_colsum_staged_kernel, dim3(static_cast<unsigned>(chunks)), smem, in, out16, rows, C, colsum,
                      inv_scale, pix, sb);
    MDM_LAUNCHED();
    return;
  }
  cast_colsum_kernel<false><<<colsum_grid(rows, C, false), TPB, 0, st>>>(in, out16, rows, C, colsum, inv_scale);
  MDM_LAUNCHED();
}
void colsum_f16(const __half* in, long long rows, int C, float* colsum, const float* inv_scale, cudaStream_t st) {
  static const bool wide = getenv("MDM_COLSUM_LEGACY") == nullptr;
  if (wide && C % 8 == 0 && rows >= 64) {
    const int ctiles = static_cast<int>(cdiv(C, 8 * TPB));
    const int Ct = std::min(C, 8 * TPB);
    const int lanes = Ct / 8;
    const int ppi = lanes <= TPB ? TPB / lanes : 1;
    long long chunks = std::max<long long>(1, (132 * 4) / ctiles);           // ~4 CTAs per SM, all resident
    chunks = std::min<long long>(chunks, cdiv(rows, 8ll * ppi));               // at least one full trip each
    colsum_f16_wide_kernel<<<dim3(static_cast<unsigned>(chunks), ctiles), TPB, 0, st>>>(in, rows, C, colsum, inv_scale);
    MDM_LAUNCHED();
    return;
  }
  cast_colsum_kernel<true><<<colsum_grid(rows, C, true), TPB, 0, st>>>(in, nullptr, rows, C, colsum, inv_scale);
  MDM_LAUNCHED();
}
void cast_f32_to_f16(const float* in, __half* out, long long n, cudaStream_t st) {
  cast_f32_to_f16_kernel<<<grid_for(cdiv(n, 4)), 256, 0, st>>>(in, out, n);
  MDM_LAUNCHED();
}
void cast_rowscale_f16(const float* in, const float* rowscale, __half* out, long long rows, int D, cudaStream_t st) {
  cast_rowscale_f16_kernel<<<grid_for(rows * (D / 4)), 256, 0, st>>>(in, rowscale, out, rows, D);
  MDM_LAUNCHED();
}
void add_f32(float* dst, const float* a, const float* b, long long n, cudaStream_t st) {
  add_f32_kernel<<<grid_for(n), 256, 0, st>>>(dst, a, b, n);
  MDM_LAUNCHED();
}
void axpy_f32(float* dst, const float* a, float alpha, long long n, int acc, cudaStream_t st) {
  axpy_f32_kernel<<<grid_for(n), 256, 0, st>>>(dst, a, alpha, n, acc);
  MDM_LAUNCHED();
}
void scale_f32(float* dst, const float* a, const float* scale, long long n, cudaStream_t st) {
  scale_f32_kernel<<<grid_for(n), 256, 0, st>>>(dst, a, scale, n);
  MDM_LAUNCHED();
}

void softmax_rows(const float* scores, __half* P16, long long rows, int S, int ld, const float* mask,
                  long long rows_per_batch, cudaStream_t st) {
  softmax_rows_kernel<<<static_cast<unsigned>(cdiv(rows, 8)), 256, 0, st>>>(scores, P16, rows, S, ld, mask,
                                                                          rows_per_batch);
  MDM_LAUNCHED();
}
void softmax_bwd_rows(const __half* P16, const float* dP, __half* dS16, long long rows, int S, int ld, float scale,
                      cudaStream_t st) {
  softmax_bwd_rows_kernel<<<static_cast<unsigned>(cdiv(rows, 8)), 256, 0, st>>>(P16, dP, dS16, rows, S, ld, scale);
  MDM_LAUNCHED();
}

void layernorm_fwd(const float* x, const float* w, const float* b, __half* y16, float* stats, long long rows, int D,
                   cudaStream_t st) {
  layernorm_fwd_kernel<<<static_cast<unsigned>(rows), 256, 0, st>>>(x, w, b, y16, stats, D);
  MDM_LAUNCHED();
}
void layernorm_bwd(const float* x, const float* w, const float* stats, const float* dy, float* dx, int acc_dx,
                   float* dw, float* db, const float* inv_scale, long long rows, int D, cudaStream_t st) {
  layernorm_bwd_kernel<<<static_cast<unsigned>(cdiv(rows, LN_ROWS)), 256, 0, st>>>(x, w, stats, dy, dx, acc_dx, dw,
                                                                                 db, inv_scale, rows, D);
  MDM_LAUNCHED();
}

void fold_ln_weight(const float* W, const float* w, __half* out, __half* lo, long long rows, int D, cudaStream_t st) {
  fold_ln_weight_kernel<<<grid_for(rows * D), 256, 0, st>>>(W, w, out, lo, rows, D);
  MDM_LAUNCHED();
}
__global__ void f16_lo_plane_kernel(const float* __restrict__ in, __half* __restrict__ lo, long long n) {
  long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 4;
  for (; i < n; i += stride) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(in + i));
    st_half4_lo(lo + i, v.x, v.y, v.z, v.w);
  }
}
void f16_lo_plane(const float* in, __half* lo, long long n, cudaStream_t st) {
  f16_lo_plane_kernel<<<grid_for(cdiv(n, 4)), 256, 0, st>>>(in, lo, n);
  MDM_LAUNCHED();
}
void f16_residual(const float* in, float* out, long long n, cudaStream_t st) {
  f16_residual_kernel<<<grid_for(n), 256, 0, st>>>(in, out, n);
  MDM_LAUNCHED();
}
void fold_ln_bias(const float* W, const float* b, const float* bias, float* out, int rows, int D, cudaStream_t st) {
  fold_ln_bias_kernel<<<static_cast<unsigned>(cdiv(rows, 8)), 256, 0, st>>>(W, b, bias, out, rows, D);
  MDM_LAUNCHED();
}
void unfold_ln_grads(const float* dWf, const float* dbf, const float* W, const float* w, const float* b, float* dW,
                     float* dw, float* db, int rows, int D, cudaStream_t st) {
  dim3 grid(static_cast<unsigned>(cdiv(D, 256)), static_cast<unsigned>(cdiv(rows, 64)));
  unfold_ln_grads_kernel<<<grid, 256, 0, st>>>(dWf, dbf, W, w, b, dW, dw, db, rows, D);
  MDM_LAUNCHED();
}

void sinusoid_embed(const long long* times, const MicroKeys* micro, const float* freq, int B, int half,
                    long long key_stride, __half* e16, cudaStream_t st) {
  MicroKeys keys{};
  if (micro != nullptr) keys = *micro;
  const dim3 grid(static_cast<unsigned>(cdiv(static_cast<long long>(B) * half, 256)),
                  times != nullptr ? 1u : static_cast<unsigned>(keys.num));
  sinusoid_embed_kernel<<<grid, 256, 0, st>>>(times, keys, freq, B, half, key_stride, e16);
  MDM_LAUNCHED();
}
void silu_f16(const float* x, __half* y16, long long n, cudaStream_t st) {
  silu_f16_kernel<<<grid_for(n), 256, 0, st>>>(x, y16, n);
  MDM_LAUNCHED();
}
void silu_bwd(const float* x, const float* dy, float* dx, long long n, int acc, cudaStream_t st) {
  silu_bwd_kernel<<<grid_for(n), 256, 0, st>>>(x, dy, dx, n, acc);
  MDM_LAUNCHED();
}
void gelu_bwd(const __half* u16, const float* dg, __half* du16, long long n, cudaStream_t st) {
  gelu_bwd_kernel<<<grid_for(n), 256, 0, st>>>(u16, dg, du16, n);
  MDM_LAUNCHED();
}
void masked_mean(const float* x, const float* mask, float* y, __half* y16, int B, int S, int D, cudaStream_t st) {
  dim3 grid(static_cast<unsigned>(cdiv(D, 256)), B);
  masked_mean_kernel<<<grid, 256, 0, st>>>(x, mask, y, y16, S, D);
  MDM_LAUNCHED();
}
void masked_mean_bwd(const float* dy, const float* mask, float* dx, int acc, int B, int S, int D, cudaStream_t st) {
  dim3 grid(static_cast<unsigned>(cdiv(D, 256)), S, B);
  masked_mean_bwd_kernel<<<grid, 256, 0, st>>>(dy, mask, dx, acc, S, D);
  MDM_LAUNCHED();
}

void im2col3x3(const float* x, __half* col16, int N, int H, int W, int C, int stride, cudaStream_t st) {
  const int Ho = (H + 2 - 3) / stride + 1, Wo = (W + 2 - 3) / stride + 1;
  const long long total = static_cast<long long>(N) * Ho * Wo * 9 * (C / 4);
  im2col3x3_kernel<<<grid_for(total), 256, 0, st>>>(x, col16, N, H, W, C, stride, Ho, Wo);
  MDM_LAUNCHED();
}
void col2im3x3(const float* dcol, float* dx, int acc, int N, int H, int W, int C, int stride, cudaStream_t st) {
  const int Ho = (H + 2 - 3) / stride + 1, Wo = (W + 2 - 3) / stride + 1;
  const long long total = static_cast<long long>(N) * H * W * (C / 4);
  col2im3x3_kernel<<<grid_for(total), 256, 0, st>>>(dcol, dx, acc, N, H, W, C, stride, Ho, Wo);
  MDM_LAUNCHED();
}
void im2col_input(const float* x_nchw, const float* inv_std, __half* col16, int N, int Cin, int H, int W,
                  cudaStream_t st) {
  im2col_input_kernel<<<grid_for(static_cast<long long>(N) * H * W, 128), 128, 0, st>>>(x_nchw, inv_std, col16, N,
                                                                                      Cin, H, W);
  MDM_LAUNCHED();
}
void upsample2x_f16(const float* x, __half* y16, int N, int H, int W, int C, cudaStream_t st) {
  upsample2x_f16_kernel<<<grid_for(static_cast<long long>(N) * 4 * H * W * (C / 4)), 256, 0, st>>>(x, y16, N, H, W, C);
  MDM_LAUNCHED();
}
void upsample2x_bwd(const float* dy, float* dx, int acc, int N, int H, int W, int C, cudaStream_t st) {
  upsample2x_bwd_kernel<<<grid_for(static_cast<long long>(N) * H * W * (C / 4)), 256, 0, st>>>(dy, dx, acc, N, H, W, C);
  MDM_LAUNCHED();
}
void nhwc_to_nchw(const float* x, int ldc, float* y, int N, int C, int HW, cudaStream_t st, float tanh_scale,
                  float* keep) {
  const unsigned grid = grid_for(static_cast<long long>(N) * C * HW);
  if (tanh_scale != 0.f)
    nhwc_to_nchw_kernel<true><<<grid, 256, 0, st>>>(x, ldc, y, N, C, HW, tanh_scale, keep);
  else
    nhwc_to_nchw_kernel<false><<<grid, 256, 0, st>>>(x, ldc, y, N, C, HW, 0.f, nullptr);
  MDM_LAUNCHED();
}
void nchw_to_nhwc_f16(const float* x_nchw, const float* scale, __half* y16, int ldo, int N, int C, int HW,
                      cudaStream_t st, float tanh_scale, const float* y_out) {
  const unsigned grid = grid_for(static_cast<long long>(N) * HW * ldo);
  if (tanh_scale != 0.f && y_out != nullptr)
    nchw_to_nhwc_f16_kernel<true><<<grid, 256, 0, st>>>(x_nchw, scale, y16, ldo, N, C, HW, tanh_scale, y_out);
  else
    nchw_to_nhwc_f16_kernel<false><<<grid, 256, 0, st>>>(x_nchw, scale, y16, ldo, N, C, HW, 0.f, nullptr);
  MDM_LAUNCHED();
}
void sample_inv_std(const float* x, float* inv_std, int N, long long per, cudaStream_t st) {
  sample_inv_std_kernel<<<N, 256, 0, st>>>(x, inv_std, per);
  MDM_LAUNCHED();
}

void pack_conv_w(const float* w_oihw, __half* packed, int Co, int Ci, int taps, cudaStream_t st) {
  pack_conv_w_kernel<<<grid_for(static_cast<long long>(Co) * Ci), 256, 0, st>>>(w_oihw, packed, Co, Ci, taps);
  MDM_LAUNCHED();
}
void pack_conv_w_fold(const float* w_oihw, __half* packed, int Co, int Ci, cudaStream_t st) {
  pack_conv_w_fold_kernel<<<grid_for(4ll * Co * Ci * 9), 256, 0, st>>>(w_oihw, packed, Co, Ci);
  MDM_LAUNCHED();
}
void unpack_conv_wgrad_fold(const float* packed, float* g_oihw, int Co, int Ci, const float* inv_scale,
                            cudaStream_t st) {
  unpack_conv_wgrad_fold_kernel<<<static_cast<unsigned>(cdiv(static_cast<long long>(Co) * Ci * 9, 256)), 256, 0, st>>>(
      packed, g_oihw, Co, Ci, inv_scale);
  MDM_LAUNCHED();
}
void pack_conv_in_w(const float* w_oihw, __half* packed, int Co, int Ci, cudaStream_t st) {
  pack_conv_in_w_kernel<<<static_cast<unsigned>(cdiv(Co * 32, 256)), 256, 0, st>>>(w_oihw, packed, Co, Ci);
  MDM_LAUNCHED();
}
void unpack_conv_wgrad(const float* packed, float* g_oihw, int Co, int Ci, int taps, int ci_ld,
                       const float* inv_scale, cudaStream_t st) {
  if (taps > 9) throw std::runtime_error("unpack_conv_wgrad: at most 9 taps");
  unpack_conv_wgrad_kernel<<<dim3(Co, static_cast<unsigned>(cdiv(Ci, 256))), 256, 0, st>>>(packed, g_oihw, Co, Ci, taps,
                                                                                          ci_ld, inv_scale);
  MDM_LAUNCHED();
}
void unpack_conv_in_wgrad(const float* packed, float* g_oihw, int Co, int Ci, const float* inv_scale,
                          cudaStream_t st) {
  unpack_conv_in_wgrad_kernel<<<static_cast<unsigned>(cdiv(Co * Ci * 9, 256)), 256, 0, st>>>(packed, g_oihw, Co, Ci,
                                                                                           inv_scale);
  MDM_LAUNCHED();
}

void grad_amax(const float* g, long long n, float* amax_buf, cudaStream_t st, float tanh_scale, const float* y_out) {
  const unsigned grid = grid_for(n, 256, 132 * 4);
  if (tanh_scale != 0.f && y_out != nullptr)
    grad_amax_kernel<true><<<grid, 256, 0, st>>>(g, n, amax_buf, tanh_scale, y_out);
  else
    grad_amax_kernel<false><<<grid, 256, 0, st>>>(g, n, amax_buf, 0.f, nullptr);
  MDM_LAUNCHED();
}
void grad_scale_finalize(const float* amax_buf, float* scale, float* inv_scale, cudaStream_t st) {
  grad_scale_finalize_kernel<<<1, 1, 0, st>>>(amax_buf, scale, inv_scale);
  MDM_LAUNCHED();
}

}  // namespace mdm
