// Training-side consumers of the matcher output (SURVEY.md §8 a20 / f-2): the weighted negative
// log-likelihood of the ground-truth assignment on the log-coupling matrix, compute_match_loss (helpers.py:228-241),
// forward and backward.  log_p [bs, ft, ft] (ft = keypoints + 1 dustbin), gt_indices [bs, 2, ft] int64 (index of the
// partner in the other view, -1 = last = dustbin, Python negative indexing), gt_weights [bs, 2, ft]:
//   loss = ( sum_{b,i} -log_p[b, i, idx0[b,i]] w0[b,i]  +  sum_{b,j} -log_p[b, idx1[b,j], j] w1[b,j] ) / bs
#include "../../include/mvm_b200.h"
#include "common.cuh"

namespace {

__device__ __forceinline__ int wrap(long long idx, int ft) { return (int)(idx < 0 ? idx + ft : idx); }

// one CTA per batch item: partial[b] = sum of the 2 ft weighted terms (fixed order -> deterministic)
__global__ void __launch_bounds__(256) match_loss_fwd_kernel(const float* __restrict__ log_p, const long long* __restrict__ idx,
                                                             const float* __restrict__ wgt, double* __restrict__ partial,
                                                             int ft) {
  const int b = blockIdx.x;
  const float* lp = log_p + (long long)b * ft * ft;
  const long long* i0 = idx + (long long)b * 2 * ft;
  const long long* i1 = i0 + ft;
  const float* w0 = wgt + (long long)b * 2 * ft;
  const float* w1 = w0 + ft;
  double s = 0.0;
  for (int i = threadIdx.x; i < ft; i += blockDim.x) {
    s += -(double)lp[(long long)i * ft + wrap(i0[i], ft)] * (double)w0[i];
    s += -(double)lp[(long long)wrap(i1[i], ft) * ft + i] * (double)w1[i];
  }
  __shared__ double red[8];
  s = warp_sum_d(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w];
    partial[b] = t;
  }
}
__global__ void match_loss_sum_kernel(const double* __restrict__ partial, float* __restrict__ loss, int bs) {
  double t = 0.0;
  for (int b = 0; b < bs; ++b) t += partial[b];
  loss[0] = (float)(t / bs);
}
// grad_log_p must be zero-filled; every element receives at most two contributions (a mutual ground-truth match)
__global__ void match_loss_bwd_kernel(const long long* __restrict__ idx, const float* __restrict__ wgt,
                                      const float* __restrict__ grad_out, float* __restrict__ grad_log_p, int bs, int ft) {
  const long long n = (long long)bs * ft;
  const float g = grad_out[0] / (float)bs;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(e / ft), i = (int)(e % ft);
    const long long* i0 = idx + (long long)b * 2 * ft;
    const float* w0 = wgt + (long long)b * 2 * ft;
    float* gp = grad_log_p + (long long)b * ft * ft;
    atomicAdd(gp + (long long)i * ft + wrap(i0[i], ft), -w0[i] * g);
    atomicAdd(gp + (long long)wrap(i0[ft + i], ft) * ft + i, -w0[ft + i] * g);
  }
}

}  // namespace

extern "C" {

int mvm_match_loss_forward(const float* log_p, const int64_t* gt_indices, const float* gt_weights, int bs, int ft,
                           double* partial_ws, float* loss, void* stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MVM_REQUIRE(log_p && gt_indices && gt_weights && partial_ws && loss && bs >= 1 && ft >= 2);
  MvmProfScope prof__(MVM_TAG_MISC, s);
  match_loss_fwd_kernel<<<bs, 256, 0, s>>>(log_p, (const long long*)gt_indices, gt_weights, partial_ws, ft);
  MVM_CHECK_LAUNCH();
  match_loss_sum_kernel<<<1, 1, 0, s>>>(partial_ws, loss, bs);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

int mvm_match_loss_backward(const int64_t* gt_indices, const float* gt_weights, const float* grad_loss, int bs, int ft,
                            float* grad_log_p, void* stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MVM_REQUIRE(gt_indices && gt_weights && grad_loss && grad_log_p && bs >= 1 && ft >= 2);
  MvmProfScope prof__(MVM_TAG_MISC, s);
  cudaMemsetAsync(grad_log_p, 0, (size_t)bs * ft * ft * sizeof(float), s);
  match_loss_bwd_kernel<<<mvm_dev_info().n_sm * 2, 256, 0, s>>>((const long long*)gt_indices, gt_weights, grad_loss, grad_log_p, bs, ft);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

}  // extern "C"
