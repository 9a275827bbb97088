// Engine: memory pool and the GEMM / implicit-conv wrappers over the wgmma kernel.
#include "engine.cuh"

#include <algorithm>

namespace mdm {

// ------------------------------------------------------------------ Pool
static size_t round_size(size_t b) {
  if (b == 0) b = 1;
  const size_t q = b < (1u << 20) ? 512 : (1u << 16);
  return (b + q - 1) / q * q;
}
Pool::~Pool() { trim(); }
void* Pool::alloc(size_t bytes) {
  const size_t sz = round_size(bytes);
  auto it = free_.find(sz);
  void* p = nullptr;
  if (it != free_.end() && !it->second.empty()) {
    p = it->second.back();
    it->second.pop_back();
  } else {
    cudaError_t e = cudaMalloc(&p, sz);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      // drop cached blocks of other sizes and retry once
      ++epoch_;
      for (auto& kv : free_) {
        for (void* q : kv.second) {
          cudaFree(q);
          size_of_.erase(q);
          reserved_ -= kv.first;
        }
        kv.second.clear();
      }
      e = cudaMalloc(&p, sz);
      if (e != cudaSuccess)
        throw MdmFail("device out of memory in mdm_b200 pool (requested " + std::to_string(sz) + " B, reserved " +
                      std::to_string(reserved_) + " B)");
    }
    size_of_[p] = sz;
    reserved_ += sz;
  }
  live_[p] = true;
  in_use_ += sz;
  high_ = std::max(high_, in_use_);
  return p;
}
void Pool::release(void* p) {
  if (p == nullptr) return;
  auto it = live_.find(p);
  if (it == live_.end() || !it->second) return;
  it->second = false;
  const size_t sz = size_of_[p];
  in_use_ -= sz;
  free_[sz].push_back(p);
}
void Pool::reset() {
  for (auto& kv : live_) {
    if (kv.second) {
      kv.second = false;
      const size_t sz = size_of_[kv.first];
      free_[sz].push_back(kv.first);
    }
  }
  in_use_ = 0;
}
void Pool::trim() {
  ++epoch_;
  for (auto& kv : size_of_) cudaFree(kv.first);
  size_of_.clear();
  free_.clear();
  live_.clear();
  reserved_ = in_use_ = 0;
}

// ------------------------------------------------------------------ Engine helpers
float* Engine::zeros_f32(long long n) {
  float* p = alloc<float>(n);
  MDM_CUDA(cudaMemsetAsync(p, 0, static_cast<size_t>(n) * sizeof(float), st));
  return p;
}
Act* Engine::new_act(int n, int h, int w, int c, bool alloc_data) {
  acts.emplace_back();
  Act* a = &acts.back();
  a->n = n;
  a->h = h;
  a->w = w;
  a->c = c;
  if (alloc_data) a->p = alloc<float>(a->numel());
  return a;
}
float* Engine::grad_buf(Act* a, int* acc) {
  if (a->g == nullptr) a->g = alloc<float>(a->numel());
  *acc = a->ginit ? 1 : 0;
  a->ginit = true;
  return a->g;
}

cudaEvent_t Engine::next_event() {
  if (ev_next == events.size()) {
    cudaEvent_t e = nullptr;
    MDM_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    events.push_back(e);
  }
  return events[ev_next++];
}
void Engine::side_begin() {
  if (!side_enabled || !capturing) return;
  if (side == nullptr) MDM_CUDA(cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking));
  cudaEvent_t e = next_event();
  MDM_CUDA(cudaEventRecord(e, st));
  MDM_CUDA(cudaStreamWaitEvent(side, e, 0));
  main_saved = st;
  st = side;
  side_active = true;
}
void Engine::side_end() {
  if (main_saved == nullptr) return;
  st = main_saved;
  main_saved = nullptr;
}
void Engine::side_join() {
  if (main_saved != nullptr) side_end();
  if (!side_active) return;
  cudaEvent_t e = next_event();
  MDM_CUDA(cudaEventRecord(e, side));
  MDM_CUDA(cudaStreamWaitEvent(st, e, 0));
  side_active = false;
  for (void* p : deferred) cur_pool().release(p);
  deferred.clear();
}

namespace {

constexpr int kNumSMs = 132;  // H100 SXM: one GEMM CTA per SM

int round16(int n) { return (n + 15) / 16 * 16; }

// Tile width of the linear and 3x3-conv forward / data-gradient GEMMs: one tile up to 176 columns, 128-column tiles
// beyond. Measured on an H100 80GB HBM3 at 400 W on the cc12m_64x64 shapes at batch 64 (M = 8 K - 262 K rows,
// 768-3072 columns), 256-column tiles took 1.2-2.8x and 192-column tiles 1.3-2.7x as long as 128-column ones.
int pick_block_n(int N) { return N < 192 ? round16(N) : 128; }

TmapSpec spec(const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3, uint64_t s1, uint64_t s2,
              uint64_t s3, uint32_t b0, uint32_t b1, uint32_t b2, uint32_t b3) {
  TmapSpec s;
  s.ptr = ptr;
  s.dims[0] = d0; s.dims[1] = d1; s.dims[2] = d2; s.dims[3] = d3;
  s.strides[0] = 1; s.strides[1] = s1; s.strides[2] = s2; s.strides[3] = s3;
  s.box[0] = b0; s.box[1] = b1; s.box[2] = b2; s.box[3] = b3;
  return s;
}

void fill_epi(GemmParams& p, const Epi& e, long long dense_ld) {
  p.alpha = e.alpha;
  p.alpha_dev = e.alpha_dev;
  p.bias = e.bias;
  p.residual = e.residual;
  p.out_f32 = e.out_f32;
  p.out_f16 = e.out_f16;
  p.out_act_f16 = e.out_act_f16;
  p.act = e.act;
  p.gelu_grad_src = e.gelu_grad_src;
  p.ldc = e.ldc > 0 ? e.ldc : dense_ld;
}

void run(const TmapSpec& A, const TmapSpec& B, int a_mn, int b_mn, GemmParams& p, const Epi& e, long long tiles,
         cudaStream_t st, const void* b_lo) {
  p.nsplit = 1;
  p.atomic = 0;
  if (e.atomic_ok) {
    MDM_CHECK(e.bias == nullptr && e.residual == nullptr && e.out_f16 == nullptr && e.out_act_f16 == nullptr,
              "split-K epilogue can only accumulate fp32");
    p.atomic = 1;
    long long want = kNumSMs / std::max<long long>(tiles, 1);
    want = std::min<long long>(want, p.num_kblocks / 2);
    p.nsplit = static_cast<int>(std::max<long long>(want, 1));
  }
  const int rc = launch_gemm(A, B, a_mn, b_mn, p, st, b_lo, e.a_lo);
  if (rc != 0) throw MdmFail("GEMM launch failed, rc=" + std::to_string(rc));
}

}  // namespace

void Engine::gemm_nt(const __half* A, long long lda, const __half* W, long long ldw, int M, int N, int K,
                     const Epi& e) {
  GemmParams p{};
  p.kind = GEMM_PLAIN;
  p.M = M; p.N = N; p.K = K;
  const long long mt = (M + 127) / 128;
  p.block_n = pick_block_n(N);
  p.nz1 = p.nz2 = 1;
  p.num_kblocks = (K + 63) / 64;
  fill_epi(p, e, N);
  TmapSpec a = spec(A, K, M, 1, 1, lda, lda * M, lda * M, 64, 128, 1, 1);
  TmapSpec b = spec(W, K, N, 1, 1, ldw, ldw * N, ldw * N, 64, p.block_n, 1, 1);
  run(a, b, 0, 0, p, e, mt * ((N + p.block_n - 1) / p.block_n), st, b_lo(W));
}

void Engine::gemm_nn(const __half* A, long long lda, const __half* Bm, long long ldb, int M, int N, int K,
                     const Epi& e) {
  GemmParams p{};
  p.kind = GEMM_PLAIN;
  p.M = M; p.N = N; p.K = K;
  const long long mt = (M + 127) / 128;
  p.block_n = pick_block_n(N);
  p.nz1 = p.nz2 = 1;
  p.num_kblocks = (K + 63) / 64;
  fill_epi(p, e, N);
  TmapSpec a = spec(A, K, M, 1, 1, lda, lda * M, lda * M, 64, 128, 1, 1);
  TmapSpec b = spec(Bm, N, K, 1, 1, ldb, ldb * K, ldb * K, 64, 64, 1, 1);
  run(a, b, 0, 1, p, e, mt * ((N + p.block_n - 1) / p.block_n), st, b_lo(Bm));
}

void Engine::gemm_tn(const __half* At, long long lda, const __half* Bm, long long ldb, int M, int N, int K,
                     const Epi& e) {
  GemmParams p{};
  p.kind = GEMM_PLAIN;
  p.M = M; p.N = N; p.K = K;
  const long long mt = (M + 127) / 128;
  // weight gradients: long contraction, small output -> widest tile, parallelism from split-K
  p.block_n = e.atomic_ok ? (N >= 256 ? 256 : round16(N)) : pick_block_n(N);
  p.nz1 = p.nz2 = 1;
  p.num_kblocks = (K + 63) / 64;
  fill_epi(p, e, N);
  TmapSpec a = spec(At, M, K, 1, 1, lda, lda * K, lda * K, 64, 64, 1, 1);
  TmapSpec b = spec(Bm, N, K, 1, 1, ldb, ldb * K, ldb * K, 64, 64, 1, 1);
  run(a, b, 1, 1, p, e, mt * ((N + p.block_n - 1) / p.block_n), st, nullptr);
}

static void conv_geom(GemmParams& p, int N, int H, int W, int pixels_per_tile) {
  p.H = H;
  p.W = W;
  p.PW = W >= 16 ? 16 : 8;
  p.PH = pixels_per_tile / p.PW;
  p.tiles_w = (W + p.PW - 1) / p.PW;
  p.tiles_h = (H + p.PH - 1) / p.PH;
  p.nimg = N;
}

static const bool g_fold = getenv("MDM_NO_WFOLD") == nullptr;

void Engine::conv3x3_fwd(const __half* x16, int ldx, int N, int H, int W, int Cin, const __half* w16, int Cout,
                         const Epi& e, const __half* w16f, const float* bias_f) {
  if (g_fold && w16f != nullptr && fold_ok(Cin, Cout) && ldx == Cin && (W & 1) == 0 && (e.ldc == 0 || e.ldc == Cout) &&
      (e.bias == nullptr || bias_f != nullptr) && e.gelu_grad_src == nullptr) {
    Epi f = e;
    f.bias = e.bias != nullptr ? bias_f : nullptr;
    f.ldc = 0;
    conv3x3_fwd(x16, 2 * Cin, N, H, W / 2, 2 * Cin, w16f, 2 * Cout, f);
    return;
  }
  GemmParams p{};
  p.kind = GEMM_CONV;
  p.N = Cout; p.K = Cin;
  conv_geom(p, N, H, W, 128);
  const long long mt = static_cast<long long>(N) * p.tiles_h * p.tiles_w;
  p.block_n = pick_block_n(Cout);
  p.nz1 = p.nz2 = 1;
  p.taps = 9;
  p.kblocks_c = (Cin + 63) / 64;
  p.num_kblocks = 9 * p.kblocks_c;
  fill_epi(p, e, Cout);
  TmapSpec a = spec(x16, Cin, W, H, N, ldx, static_cast<uint64_t>(W) * ldx, static_cast<uint64_t>(H) * W * ldx, 64,
                    p.PW, p.PH, 1);
  TmapSpec b = spec(w16, Cin, Cout, 9, 1, 9ull * Cin, Cin, 9ull * Cin * Cout, 64, p.block_n, 1, 1);
  run(a, b, 0, 0, p, e, mt * ((Cout + p.block_n - 1) / p.block_n), st, b_lo(w16));
}

void Engine::conv3x3_dgrad(const __half* dy16, int ldy, int N, int H, int W, int Cout, const __half* w16, int Cin,
                           const Epi& e, const __half* w16f) {
  if (g_fold && w16f != nullptr && fold_ok(Cin, Cout) && ldy == Cout && (W & 1) == 0 && (e.ldc == 0 || e.ldc == Cin) &&
      e.bias == nullptr && e.gelu_grad_src == nullptr) {
    Epi f = e;
    f.ldc = 0;
    conv3x3_dgrad(dy16, 2 * Cout, N, H, W / 2, 2 * Cout, w16f, 2 * Cin, f);
    return;
  }
  GemmParams p{};
  p.kind = GEMM_CONV;
  p.N = Cin; p.K = Cout;
  conv_geom(p, N, H, W, 128);
  const long long mt = static_cast<long long>(N) * p.tiles_h * p.tiles_w;
  p.block_n = pick_block_n(Cin);
  p.nz1 = p.nz2 = 1;
  p.taps = 9;
  p.flip = 1;
  p.kblocks_c = (Cout + 63) / 64;
  p.num_kblocks = 9 * p.kblocks_c;
  fill_epi(p, e, Cin);
  TmapSpec a = spec(dy16, Cout, W, H, N, ldy, static_cast<uint64_t>(W) * ldy, static_cast<uint64_t>(H) * W * ldy, 64,
                    p.PW, p.PH, 1);
  TmapSpec b = spec(w16, Cin, Cout, 9, 1, 9ull * Cin, Cin, 9ull * Cin * Cout, 64, 64, 1, 1);
  run(a, b, 0, 1, p, e, mt * ((Cin + p.block_n - 1) / p.block_n), st, b_lo(w16));
}

bool Engine::conv3x3_wgrad(const __half* dy16, int ldy, const __half* x16, int ldx, int N, int H, int W, int Cin,
                           int Cout, float* packed_out, bool allow_fold) {
  if (g_fold && allow_fold && fold_ok(Cin, Cout) && ldy == Cout && ldx == Cin && (W & 1) == 0) {
    conv3x3_wgrad(dy16, 2 * Cout, x16, 2 * Cin, N, H, W / 2, 2 * Cin, 2 * Cout, packed_out, false);
    return true;
  }
  GemmParams p{};
  p.kind = GEMM_CONV_WGRAD;
  p.M = Cout; p.N = Cin;
  // <= 64 channels on both sides: 256-pixel stages (gemm_tc.cu, kfactor). MDM_WGRAD_KFACTOR=1 restores 64.
  static const int kf_env = getenv("MDM_WGRAD_KFACTOR") ? atoi(getenv("MDM_WGRAD_KFACTOR")) : 4;
  const int kf = (Cout <= 64 && Cin <= 64 && H >= 16 && W >= 16 && kf_env > 1) ? kf_env : 1;
  p.kfactor = kf;
  conv_geom(p, N, H, W, 64 * kf);
  const long long mt = (Cout + 127) / 128;
  p.block_n = Cin >= 256 ? 256 : round16(Cin);
  p.nz1 = 9;
  p.nz2 = 1;
  p.taps = 9;
  p.num_kblocks = N * p.tiles_h * p.tiles_w;
  Epi e;
  e.out_f32 = packed_out;
  fill_epi(p, e, 9ll * Cin);
  p.c_z1_stride = Cin;
  const long long tiles = mt * ((Cin + p.block_n - 1) / p.block_n) * 9;
  long long want = kNumSMs / std::max<long long>(tiles, 1);
  want = std::min<long long>(want, p.num_kblocks / 2);
  p.nsplit = static_cast<int>(std::max<long long>(want, 1));
  p.atomic = p.nsplit > 1 ? 1 : 0;
  if (p.atomic) MDM_CUDA(cudaMemsetAsync(packed_out, 0, sizeof(float) * 9ull * Cin * Cout, st));
  TmapSpec a = spec(dy16, Cout, W, H, N, ldy, static_cast<uint64_t>(W) * ldy, static_cast<uint64_t>(H) * W * ldy, 64,
                    p.PW, p.PH, 1);
  TmapSpec b = spec(x16, Cin, W, H, N, ldx, static_cast<uint64_t>(W) * ldx, static_cast<uint64_t>(H) * W * ldx, 64,
                    p.PW, p.PH, 1);
  const int rc = launch_gemm(a, b, 1, 1, p, st);
  if (rc != 0) throw MdmFail("conv wgrad launch failed, rc=" + std::to_string(rc));
  return false;
}

}  // namespace mdm
