// Shared device/host helpers for the sm_90a kernels of the matcher + pose hot path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define MVM_OK 0
#define MVM_ERR_INVALID 1
#define MVM_ERR_LAUNCH 2
#define MVM_ERR_WORKSPACE 3

extern unsigned long long g_mvm_launches;   // kernels launched by this library (profile.cu)

// kernel classes for the optional event profiler (mvm_profile_*)
enum MvmTag { MVM_TAG_GEMM = 0, MVM_TAG_ATTN, MVM_TAG_SINKHORN, MVM_TAG_SCORE, MVM_TAG_MATCH,
              MVM_TAG_CONF, MVM_TAG_KENC, MVM_TAG_W8PT, MVM_TAG_BA2, MVM_TAG_MVBA, MVM_TAG_MISC,
              MVM_N_TAGS };
struct MvmProfScope {
  MvmProfScope(int tag, cudaStream_t s);
  ~MvmProfScope();
  int tag_; cudaStream_t s_; int idx_;
};

#define MVM_CHECK_LAUNCH()                                                        \
  do {                                                                            \
    ++g_mvm_launches;                                                             \
    cudaError_t e__ = cudaGetLastError();                                         \
    if (e__ != cudaSuccess) {                                                     \
      fprintf(stderr, "[mvm_b200] launch failed at %s:%d: %s\n", __FILE__,        \
              __LINE__, cudaGetErrorString(e__));                                 \
      return MVM_ERR_LAUNCH;                                                      \
    }                                                                             \
  } while (0)

#define MVM_REQUIRE(cond)                                                         \
  do {                                                                            \
    if (!(cond)) {                                                                \
      fprintf(stderr, "[mvm_b200] invalid argument at %s:%d: %s\n", __FILE__,     \
              __LINE__, #cond);                                                   \
      return MVM_ERR_INVALID;                                                     \
    }                                                                             \
  } while (0)

static inline int mvm_div_up(int a, int b) { return (a + b - 1) / b; }

// ---- per-device state (profile.cu) -------------------------------------------------------
// Function attributes (opt-in shared memory, cluster size) and the SM count are PER DEVICE: a process may
// drive several GPUs (nn.DataParallel, model.to('cuda:1')) from several threads.  mvm_dev_info() describes
// the CURRENT device; mvm_once_per_device(slot, f) runs f exactly once per (device, slot) under a mutex.
#include <mutex>
struct MvmDevInfo { int dev; int n_sm; size_t max_smem; };
const MvmDevInfo& mvm_dev_info();
std::mutex& mvm_attr_mutex();
bool* mvm_attr_flag(int slot);   // flag of (current device, slot); call with mvm_attr_mutex() held
enum MvmOnceSlot { MVM_ONCE_SINKHORN_CL = 0, MVM_ONCE_SINKHORN_EXP, MVM_ONCE_SINKHORN_LOG, MVM_ONCE_ATTN_TC,
                   MVM_ONCE_ATTN_SIMT, MVM_ONCE_GEMM_TC, MVM_ONCE_GEMM_PERSIST, MVM_ONCE_GEMM_SCORE, MVM_ONCE_KENC,
                   MVM_ONCE_MVBA, MVM_ONCE_ATTN_H3, MVM_ONCE_ATTN_H3S, MVM_ONCE_ATTN_BWD, MVM_ONCE_SINKHORN_TRAIN,
                   MVM_ONCE_SP_SELECT, MVM_N_ONCE = 32 };
template <class F>
static inline void mvm_once_per_device(int slot, F&& f) {
  std::lock_guard<std::mutex> g(mvm_attr_mutex());
  bool* fl = mvm_attr_flag(slot);
  if (!*fl) { f(); *fl = true; }
}

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
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- GEMM descriptor shared by the SIMT and tensor-core paths ------------------------------
// C[M,N] = act(alpha * [A | A2][M,K] * W[N,K]^T + bias[N]) + R[M,N]
// A covers k in [0,K1), A2 covers k in [K1,K) (concat-by-K-split; A2 == nullptr -> K1 == K).
struct GemmDesc {
  const float* A;  int lda;
  const float* A2; int lda2; int K1;
  const float* W;  int ldw;
  const float* Whi; const float* Wlo;          // optional pre-split tf32 planes of W (3xTF32 mode)
  const void* Whi16; const void* Wlo16;        // optional half-precision planes of wscale * W (fp16x3 mode, persistent schedule)
  float wscale;
  const float* bias;
  const float* R;  int ldr;
  float* C;        int ldc;
  int M, N, K;
  float alpha;
  int relu;
  int batch;                                   // gridDim.z
  long long sA, sA2, sW, sR, sC;               // per-batch element strides
};

int launch_gemm_simt(const GemmDesc& g, cudaStream_t stream);
