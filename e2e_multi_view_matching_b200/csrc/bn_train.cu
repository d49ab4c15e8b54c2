// BatchNorm1d in TRAINING mode on point-major activations (the train branch of the matcher, SURVEY.md 8 a8 / f-2:
// multi_view_matcher.py:8-22 MLP = Conv1d + BatchNorm1d + ReLU; statistics over all B*T*N points of the call):
//   y = act(gamma * (x - mean_c) / sqrt(var_c + eps) + beta),  var biased for the normalisation,
//   running_mean <- (1 - momentum) running_mean + momentum mean,  running_var likewise with the UNBIASED variance
// x, y [rows, C] with row stride ld (y may be x); mean and 1/sqrt(var + eps) can be saved for the backward; only rows whose index inside their n_pad-row view slot is < n_valid count (the
// padding rows of a slot are left untouched), and only the slots s with s % slot_mod == slot_rem (the pairwise train
// path normalises every view on its own, multi_view_matcher.py:169-173 / superglue.py:131-140).  Two launches: per-channel sums in double (shifted by the first valid
// row: no cancellation), then normalise in place.
#include "../../include/mvm_b200.h"
#include "common.cuh"
#include "kernels.cuh"

namespace {

// grid (row blocks), block = C threads (<= 1024): thread c accumulates channel c over the block's rows
__global__ void bn_sums_kernel(const float* __restrict__ x, int rows, int C, int ld, int n_pad, int n_valid,
                               int slot_mod, int slot_rem, int rows_per_block, double* sums) {
  const int c = threadIdx.x;
  if (c >= C) return;
  const float shift = (float)sums[2 * C + c];   // row 0 of the buffer (always a valid row), stored by bn_shift_kernel
  const int r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  double s = 0.0, q = 0.0;
  for (int r = r0; r < r1; ++r) {
    if (r % n_pad >= n_valid || (r / n_pad) % slot_mod != slot_rem) continue;
    const double d = (double)(x[(long long)r * ld + c] - shift);
    s += d; q += d * d;
  }
  atomicAdd(sums + c, s);
  atomicAdd(sums + C + c, q);
}

__global__ void bn_apply_kernel(const float* x, float* y, int rows, int C, int ld, int n_pad, int n_valid, int slot_mod,
                                int slot_rem, float* __restrict__ save_stats,
                                const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int relu,
                                float* __restrict__ running_mean, float* __restrict__ running_var, float momentum,
                                const double* __restrict__ sums, long long count) {
  const int c = threadIdx.x;
  if (c >= C) return;
  const double sh = sums[2 * C + c];              // row 0's ORIGINAL value (block 0 rewrites row 0 below)
  const double n = (double)count;
  const double mean_s = sums[c] / n;                                    // mean of (x - shift)
  const double var = fmax(sums[C + c] / n - mean_s * mean_s, 0.0);      // biased
  const double mean = mean_s + sh;
  const double scale_d = (double)gamma[c] / sqrt(var + (double)eps);
  const float scale = (float)scale_d;
  // y = (x - mean_hi) scale + (beta - mean_lo scale): x - mean_hi is exact near the mean, so a channel whose mean is
  // large against its spread (or constant) keeps its bits; x scale + (beta - mean scale) lost ~ulp(mean scale) of them
  const float mean_hi = (float)mean;
  const float bias = (float)((double)beta[c] - (mean - (double)mean_hi) * scale_d);
  if (blockIdx.x == 0 && save_stats != nullptr) { save_stats[c] = (float)mean; save_stats[C + c] = (float)(1.0 / sqrt(var + (double)eps)); }
  if (blockIdx.x == 0 && running_mean != nullptr) {
    running_mean[c] = (float)((1.0 - momentum) * (double)running_mean[c] + momentum * mean);
    const double unbiased = n > 1.0 ? var * n / (n - 1.0) : var;
    running_var[c] = (float)((1.0 - momentum) * (double)running_var[c] + momentum * unbiased);
  }
  const int rows_per_block = (rows + gridDim.x - 1) / gridDim.x;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  for (int r = r0; r < r1; ++r) {
    if (r % n_pad >= n_valid || (r / n_pad) % slot_mod != slot_rem) continue;
    float o = fmaf(x[(long long)r * ld + c] - mean_hi, scale, bias);
    if (relu) o = fmaxf(o, 0.f);
    y[(long long)r * ld + c] = o;
  }
}

__global__ void bn_shift_kernel(const float* __restrict__ x, int C, long long first_row_off, double* __restrict__ sums) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) { sums[c] = 0.0; sums[C + c] = 0.0; sums[2 * C + c] = (double)x[first_row_off + c]; }
}

// ---- backward:  g = dy o (y > 0)  (ReLU),  xhat = (x - mean) invstd,
//   dgamma = sum g xhat,  dbeta = sum g,  dx = gamma invstd (g - dbeta / n - xhat dgamma / n)      (in place on dy)
__global__ void bn_bwd_sums_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dy,
                                   int rows, int C, int ld, int n_pad, int n_valid, int slot_mod, int slot_rem,
                                   const float* __restrict__ stats, int relu, int rows_per_block, double* sums) {
  const int c = threadIdx.x;
  if (c >= C) return;
  const float mean = stats[c], invstd = stats[C + c];
  const int r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  double sg = 0.0, sgx = 0.0;
  for (int r = r0; r < r1; ++r) {
    if (r % n_pad >= n_valid || (r / n_pad) % slot_mod != slot_rem) continue;
    const long long o = (long long)r * ld + c;
    float gq = dy[o];
    if (relu && !(y[o] > 0.f)) gq = 0.f;
    sg += (double)gq;
    sgx += (double)gq * (double)((x[o] - mean) * invstd);
  }
  atomicAdd(sums + c, sg);
  atomicAdd(sums + C + c, sgx);
}

__global__ void bn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ y, float* __restrict__ dy,
                                    int rows, int C, int ld, int n_pad, int n_valid, int slot_mod, int slot_rem,
                                    const float* __restrict__ gamma, const float* __restrict__ stats, int relu,
                                    float* __restrict__ dgamma, float* __restrict__ dbeta, int accumulate,
                                    const double* __restrict__ sums, long long count) {
  const int c = threadIdx.x;
  if (c >= C) return;
  const float mean = stats[c], invstd = stats[C + c];
  const double n = (double)count;
  const float mg = (float)(sums[c] / n), mgx = (float)(sums[C + c] / n);
  const float k = gamma[c] * invstd;
  if (blockIdx.x == 0) {
    dgamma[c] = (accumulate ? dgamma[c] : 0.f) + (float)sums[C + c];
    dbeta[c] = (accumulate ? dbeta[c] : 0.f) + (float)sums[c];
  }
  const int rows_per_block = (rows + gridDim.x - 1) / gridDim.x;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  for (int r = r0; r < r1; ++r) {
    if (r % n_pad >= n_valid || (r / n_pad) % slot_mod != slot_rem) continue;
    const long long o = (long long)r * ld + c;
    float gq = dy[o];
    if (relu && !(y[o] > 0.f)) gq = 0.f;
    const float xh = (x[o] - mean) * invstd;
    dy[o] = k * (gq - mg - xh * mgx);
  }
}

__global__ void zero_d_kernel(double* p, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = 0.0;
}

// column sums of x [rows, C] (bias gradients): per-block partials in double, one double atomic per block and channel
__global__ void colsum_kernel(const float* __restrict__ x, int rows, int C, int ld, int rows_per_block, double* sums) {
  const int c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  double s = 0.0;
  for (int r = r0; r < r1; ++r) s += (double)x[(long long)r * ld + c];
  atomicAdd(sums + c, s);
}
__global__ void colsum_final_kernel(const double* __restrict__ sums, float* __restrict__ out, int C, int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) out[c] = (accumulate ? out[c] : 0.f) + (float)sums[c];
}

__device__ __forceinline__ float tf32_rn(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
// x [R, C] (row stride ld) -> transposed copies [C, R] (row stride ldo): raw and / or the tf32 hi / lo planes the
// tensor-core GEMM takes as its W operand (hi = rn_tf32(x), lo = rn_tf32(x - hi))
__global__ void transpose_split_kernel(const float* __restrict__ x, int R, int C, int ld, float* __restrict__ raw,
                                       float* __restrict__ hi, float* __restrict__ lo, long long ldo) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < R && c < C) ? x[(long long)r * ld + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (c >= C || r >= R) continue;
    const float v = tile[threadIdx.x][i];
    const long long o = (long long)c * ldo + r;
    if (raw) raw[o] = v;
    if (hi) { const float h = tf32_rn(v); hi[o] = h; lo[o] = tf32_rn(v - h); }
  }
}

}  // namespace

extern "C" int mvm_batchnorm_train_backward(const float* x, const float* y, float* dy, int rows, int C, int ld, int n_pad,
                                            int n_valid, int slot_mod, int slot_rem, const float* gamma,
                                            const float* save_stats, int relu, float* dgamma, float* dbeta,
                                            int accumulate, double* ws /* 2 C doubles */, void* stream) {
  MVM_REQUIRE(x && dy && gamma && save_stats && dgamma && dbeta && ws && rows >= 1 && C >= 1 && C <= 1024 && ld >= C);
  MVM_REQUIRE((!relu || y) && n_pad >= 1 && n_valid >= 1 && n_valid <= n_pad && rows % n_pad == 0);
  MVM_REQUIRE(slot_mod >= 1 && slot_rem >= 0 && slot_rem < slot_mod && (rows / n_pad) % slot_mod == 0);
  cudaStream_t s = (cudaStream_t)stream;
  MvmProfScope prof__(MVM_TAG_MISC, s);
  const int threads = ((C + 31) / 32) * 32;
  const int blocks = rows < 592 ? rows : 592;
  const int rpb = (rows + blocks - 1) / blocks;
  const long long count = (long long)(rows / n_pad / slot_mod) * n_valid;
  zero_d_kernel<<<(2 * C + 255) / 256, 256, 0, s>>>(ws, 2 * C);
  MVM_CHECK_LAUNCH();
  bn_bwd_sums_kernel<<<blocks, threads, 0, s>>>(x, y, dy, rows, C, ld, n_pad, n_valid, slot_mod, slot_rem, save_stats, relu, rpb, ws);
  MVM_CHECK_LAUNCH();
  bn_bwd_apply_kernel<<<blocks, threads, 0, s>>>(x, y, dy, rows, C, ld, n_pad, n_valid, slot_mod, slot_rem, gamma, save_stats, relu,
                                                 dgamma, dbeta, accumulate, ws, count);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

extern "C" int mvm_colsum(const float* x, int rows, int C, int ld, float* out, int accumulate, double* ws /* C doubles */,
                          void* stream) {
  MVM_REQUIRE(x && out && ws && rows >= 1 && C >= 1 && ld >= C);
  cudaStream_t s = (cudaStream_t)stream;
  MvmProfScope prof__(MVM_TAG_MISC, s);
  const int blocks = rows < 296 ? rows : 296;
  const int rpb = (rows + blocks - 1) / blocks;
  zero_d_kernel<<<(C + 255) / 256, 256, 0, s>>>(ws, C);
  MVM_CHECK_LAUNCH();
  colsum_kernel<<<dim3(blocks, (C + 255) / 256), 256, 0, s>>>(x, rows, C, ld, rpb, ws);
  MVM_CHECK_LAUNCH();
  colsum_final_kernel<<<(C + 255) / 256, 256, 0, s>>>(ws, out, C, accumulate);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

extern "C" int mvm_transpose_split(const float* x, int R, int C, int ld, float* raw, float* hi, float* lo, long long ldo,
                                   void* stream) {
  MVM_REQUIRE(x && (raw || hi) && (hi == nullptr) == (lo == nullptr) && R >= 1 && C >= 1 && ld >= C && ldo >= R);
  cudaStream_t s = (cudaStream_t)stream;
  MvmProfScope prof__(MVM_TAG_MISC, s);
  transpose_split_kernel<<<dim3((C + 31) / 32, (R + 31) / 32), dim3(32, 8), 0, s>>>(x, R, C, ld, raw, hi, lo, ldo);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

extern "C" int mvm_batchnorm_train(const float* x, float* y, int rows, int C, int ld, int n_pad, int n_valid, int slot_mod,
                                   int slot_rem, const float* gamma,
                                   const float* beta, float eps, int relu, float* running_mean, float* running_var,
                                   float momentum, float* save_stats, double* ws /* 3 C doubles */, void* stream) {
  MVM_REQUIRE(x && y && gamma && beta && ws && rows >= 1 && C >= 1 && C <= 1024 && ld >= C);
  MVM_REQUIRE(n_pad >= 1 && n_valid >= 1 && n_valid <= n_pad && rows % n_pad == 0);
  MVM_REQUIRE(slot_mod >= 1 && slot_rem >= 0 && slot_rem < slot_mod && (rows / n_pad) % slot_mod == 0);
  MVM_REQUIRE((running_mean == nullptr) == (running_var == nullptr));
  cudaStream_t s = (cudaStream_t)stream;
  MvmProfScope prof__(MVM_TAG_MISC, s);
  const int threads = ((C + 31) / 32) * 32;
  const int max_blocks = 4 * mvm_dev_info().n_sm;
  const int blocks = rows < max_blocks ? rows : max_blocks;
  const int rpb = (rows + blocks - 1) / blocks;
  const long long count = (long long)(rows / n_pad / slot_mod) * n_valid;
  bn_shift_kernel<<<(C + 255) / 256, 256, 0, s>>>(x, C, (long long)slot_rem * n_pad * ld, ws);
  MVM_CHECK_LAUNCH();
  bn_sums_kernel<<<blocks, threads, 0, s>>>(x, rows, C, ld, n_pad, n_valid, slot_mod, slot_rem, rpb, ws);
  MVM_CHECK_LAUNCH();
  bn_apply_kernel<<<blocks, threads, 0, s>>>(x, y, rows, C, ld, n_pad, n_valid, slot_mod, slot_rem, save_stats, gamma, beta, eps, relu,
                                             running_mean, running_var, momentum, ws, count);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
