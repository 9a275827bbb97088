// Host-side engine of the denoising path: device memory pool, parameter table, GEMM/conv wrappers
// and the backward tape.  The network definition itself lives in net.cu.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <deque>
#include <functional>
#include <map>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "gemm_tc.cuh"
#include "kernels.cuh"

namespace mdm {

void set_error(const char* fmt, ...);

struct MdmFail : public std::runtime_error {
  explicit MdmFail(const std::string& m) : std::runtime_error(m) {}
};
#define MDM_CHECK(cond, msg)                                                             \
  do {                                                                                   \
    if (!(cond)) throw ::mdm::MdmFail(std::string(msg) + " [" #cond "] at " __FILE__ ":" + \
                                      std::to_string(__LINE__));                         \
  } while (0)
#define MDM_CUDA(call)                                                                         \
  do {                                                                                         \
    cudaError_t e__ = (call);                                                                  \
    if (e__ != cudaSuccess)                                                                    \
      throw ::mdm::MdmFail(std::string("CUDA error: ") + cudaGetErrorString(e__) + " in " #call + \
                           " at " __FILE__ ":" + std::to_string(__LINE__));                    \
  } while (0)

// Size-class caching allocator. Blocks are handed out per step and all returned by reset();
// after the first step with a given shape no cudaMalloc happens on the hot path.
class Pool {
 public:
  ~Pool();
  void* alloc(size_t bytes);
  void release(void* p);  // early return of a temporary
  void reset();           // every live block becomes free
  void trim();            // cudaFree everything
  size_t reserved() const { return reserved_; }
  size_t high_water() const { return high_; }
  // bumped whenever memory goes back to the driver: addresses recorded in CUDA graphs are dead from then on
  unsigned long long epoch() const { return epoch_; }

 private:
  std::unordered_map<size_t, std::vector<void*>> free_;
  std::unordered_map<void*, size_t> size_of_;
  std::unordered_map<void*, bool> live_;
  size_t reserved_ = 0, in_use_ = 0, high_ = 0;
  unsigned long long epoch_ = 1;
};

// fp32 NHWC activation on the residual stream (or any fp32 node that receives gradients).
struct Act {
  float* p = nullptr;
  float* g = nullptr;  // gradient (same shape), allocated on first contribution
  bool ginit = false;
  int n = 0, h = 0, w = 0, c = 0;
  long long numel() const { return static_cast<long long>(n) * h * w * c; }
  long long rows() const { return static_cast<long long>(n) * h * w; }
};

struct Param {
  std::string name;
  std::vector<int64_t> shape;
  int64_t numel = 0;
  float* w = nullptr;  // bound fp32 master weights (owned by the caller)
  float* g = nullptr;  // bound fp32 gradient buffer (owned by the caller), may be null
  __half* w16 = nullptr;  // packed fp16 operand copy (owned by the engine), null if not a GEMM weight
  int pack = 0;           // 0 none, 1 plain cast, 2 conv [Co][taps][Ci], 3 conv_in [Co][32]
  // narrow 3x3 convs (fold_ok): W-folded weights [2Co][9][2Ci] and the bias repeated twice (engine-owned)
  __half* w16f = nullptr;
  float* bias_f = nullptr;
};

struct Epi {
  float alpha = 1.f;
  const float* alpha_dev = nullptr;
  const float* bias = nullptr;
  const float* residual = nullptr;
  float* out_f32 = nullptr;
  __half* out_f16 = nullptr;
  __half* out_act_f16 = nullptr;
  int act = 0;
  long long ldc = 0;  // 0: dense
  bool atomic_ok = false;  // out_f32 is zero-initialised (or accumulating) and split-K may be used
  const __half* gelu_grad_src = nullptr;  // result *= gelu'(src[row][col])
  // optional second fp16 plane of a K-major A operand (fp16(a - A), laid out like A): the product then also takes
  // A_lo x B, so that A enters at ~22 significant bits (data gradients that feed a GroupNorm backward)
  const __half* a_lo = nullptr;
};

struct Engine {
  cudaStream_t st = nullptr;
  Pool pool;
  // while set, alloc / rel draw from this pool instead: the text path of a split forward (net.cu) runs beside a held
  // tape and must neither reset nor hand out the blocks that tape (or a captured graph) still owns
  Pool* alt = nullptr;
  Pool& cur_pool() { return alt != nullptr ? *alt : pool; }
  // Weights are held as two fp16 planes, hi = fp16(w) and lo = fp16(w - hi), in one allocation [hi | lo]; a GEMM whose
  // B operand lies in a hi plane also multiplies the lo plane, so weights enter every product at ~22 significant bits
  // and only the activation operands are rounded to fp16. Key: hi-plane base address, value: plane size (halves).
  std::map<uintptr_t, size_t> weight_planes;
  void add_weight_planes(const __half* hi, size_t n) { weight_planes[reinterpret_cast<uintptr_t>(hi)] = n; }
  // the lo-plane address of a pointer into a registered hi plane, else nullptr
  const __half* lo_plane(const void* p) const {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    auto it = weight_planes.upper_bound(a);
    if (it == weight_planes.begin()) return nullptr;
    --it;
    if (a >= it->first + it->second * sizeof(__half)) return nullptr;
    return static_cast<const __half*>(p) + it->second;
  }
  // Plane mode of the pass being recorded or replayed (mdm_net_io.single_plane): a single-plane pass multiplies the hi
  // planes only, so its weight products get no B lo plane and its data gradients no A lo plane. A backward runs in the
  // mode of the forward whose tape it replays.
  bool single_plane = false;
  // the B lo plane a weight product multiplies: lo_plane(p), or none in a single-plane pass
  const __half* b_lo(const void* p) const { return single_plane ? nullptr : lo_plane(p); }
  bool training = false;
  std::vector<std::function<void()>> tape;
  std::deque<Act> acts;
  // device scalars for gradient scaling
  float* d_scale = nullptr;
  float* d_inv_scale = nullptr;
  float* d_amax = nullptr;
  // seed of the ResNet dropout masks (kernels.cuh Dropout): written on the caller's stream by every forward that
  // drops, read by the kernels, so a replayed graph draws fresh masks and its backward regenerates the same ones
  unsigned long long* d_drop_seed = nullptr;

  // ---- side stream for weight gradients. A weight gradient feeds nothing else in the step, so its kernels (the
  // wgrad GEMM, its memset and un-pack) can run beside the data-gradient / GroupNorm-backward chain of the same layer
  // instead of in front of it. In a captured backward this turns the linear chain of ~1.5 k nodes into a graph with
  // parallel branches (the 1024-px step is bound by per-kernel latency). MDM_SIDE_WGRAD=0 turns it off. Buffers the side work reads are released
  // through rel() (deferred to the join) and must not be overwritten by the main stream before it.
  // Only while a backward is being CAPTURED: there the fork / join events become explicit graph edges. Run eagerly
  // (first step of a signature, MDM_NO_GRAPH) everything stays on the caller's stream -- ordering a non-blocking side
  // stream against torch's legacy default stream by events did not hold up in the tests (later main-stream readers saw
  // incomplete weight gradients), and the eager path is not where the time goes.
  bool side_enabled = false;
  bool capturing = false;
  bool side_active = false;  // side work was forked since the last join
  cudaStream_t side = nullptr;
  cudaStream_t main_saved = nullptr;
  std::vector<cudaEvent_t> events;
  size_t ev_next = 0;
  std::vector<void*> deferred;  // buffers released while side work may still read them
  cudaEvent_t next_event();
  // from here on `st` is the side stream, ordered after everything enqueued on the main stream so far
  void side_begin();
  // back to the main stream (the side work keeps running)
  void side_end();
  // main stream waits for the side work; buffers released meanwhile go back to the pool
  void side_join();
  // release that is safe while side work is in flight
  void rel(void* p) {
    if (p == nullptr) return;
    if (side_active) deferred.push_back(p);
    else cur_pool().release(p);
  }

  template <typename T>
  T* alloc(long long n) {
    return static_cast<T*>(cur_pool().alloc(static_cast<size_t>(n) * sizeof(T)));
  }
  float* zeros_f32(long long n);
  Act* new_act(int n, int h, int w, int c, bool alloc_data = true);
  // returns the gradient buffer of `a` and whether the caller must accumulate (1) or overwrite (0)
  float* grad_buf(Act* a, int* acc);

  // ---- GEMM wrappers (fp16 operands)
  // C[M,N] = A[M,K] * W[N,K]^T
  void gemm_nt(const __half* A, long long lda, const __half* W, long long ldw, int M, int N, int K, const Epi& e);
  // C[M,N] = A[M,K] * Bm[K,N]      (Bm row-major, i.e. MN-major operand)
  void gemm_nn(const __half* A, long long lda, const __half* Bm, long long ldb, int M, int N, int K, const Epi& e);
  // C[M,N] = At[K,M]^T * Bm[K,N]   (both MN-major; contraction over rows)
  void gemm_tn(const __half* At, long long lda, const __half* Bm, long long ldb, int M, int N, int K, const Epi& e);
  // 3x3 / pad 1 / stride 1 conv over NHWC fp16 x (channel stride ldx), packed weights [Cout][9][Cin].
  // w16f / bias_f (optional): the layer's W-folded weights and doubled bias; when given and the tensors are dense and W
  // is even the conv runs on the folded view (2Cin -> 2Cout over W/2): TMA moves one <= 128-byte row per pixel at a
  // fixed rate, so 32-channel tensors (64-byte rows) otherwise run at half speed.
  static bool fold_ok(int Cin, int Cout) { return Cin <= 64 && Cout <= 64 && (Cin <= 32 || Cout <= 32); }
  void conv3x3_fwd(const __half* x16, int ldx, int N, int H, int W, int Cin, const __half* w16, int Cout,
                   const Epi& e, const __half* w16f = nullptr, const float* bias_f = nullptr);
  void conv3x3_dgrad(const __half* dy16, int ldy, int N, int H, int W, int Cout, const __half* w16, int Cin,
                     const Epi& e, const __half* w16f = nullptr);
  // packed_out: [Cout][9][Cin] fp32, overwritten -- or, when `folded` (same conditions), [2Cout][9][2Cin] of the
  // folded problem (to be un-folded by unpack_conv_wgrad_fold); returns whether the folded form was used
  bool conv3x3_wgrad(const __half* dy16, int ldy, const __half* x16, int ldx, int N, int H, int W, int Cin,
                     int Cout, float* packed_out, bool allow_fold = false);
};

// Fused attention (attention.cu)
void attention_forward(const __half* qkv, const __half* kv, const float* mask, int B, int T, int S, int C, int heads,
                       __half* h16, __half* oself16, float* stats, cudaStream_t st);
void attention_backward(const __half* qkv, const __half* kv, const float* mask, const __half* dO, const __half* h16,
                        const __half* oself16, const float* stats, int B, int T, int S, int C, int heads, float* Dterm,
                        float* dq32, __half* dqkv16, __half* dkv16, cudaStream_t st);

// Masked self-attention over text tokens (token_attention.cu): qkv [B*T][3D], mask [B][T] or null -> o16 [B*T][D];
// stats [B][heads][T][2] (may be null without a backward). Backward: Dterm [B][heads][T] and dq32 [B*T][D] scratch.
void token_attention_forward(const __half* qkv, const float* mask, int B, int T, int D, int heads, __half* o16,
                             float* stats, cudaStream_t st);
void token_attention_backward(const __half* qkv, const float* mask, const __half* dO, const __half* o16,
                              const float* stats, int B, int T, int D, int heads, float* Dterm, float* dq32,
                              __half* dqkv16, cudaStream_t st);

}  // namespace mdm
