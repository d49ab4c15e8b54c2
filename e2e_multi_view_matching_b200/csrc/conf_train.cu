// Backward of the ConfidenceMLP in the train branch (stage 2 of training, the pose loss): the two steps that the
// generic backward kernels (GEMMs, BatchNorm, colsum) do not cover.  The reference head (multi_view_matcher.py:39-53,
// 302-306) is
//   conf = sigmoid(layers(layers_f(cat[m0, m1g]) + layers_c(add))),  layers = one Conv1d 256 -> 1,
//   m0 = mdesc_a[:, :N],  m1g = mdesc_b[b, i0[i]],  add = Z[b, i, i0[i]]
// where i0 = -1 (unmatched) indexes keypoint N-1 of mdesc_b and the dustbin column N of the couplings Z.
//
// mvm_conf_tail_backward:   sigmoid' and the 256 -> 1 layer: g_logit = g_conf c (1 - c), g_h = g_logit w_last,
//                           dW_last = sum_r g_logit_r h_r, db_last = sum_r g_logit_r.
// mvm_conf_gather_backward: the transposes of the three gathers: g_x[:, :256] -> g_md[b, a, i],
//                           g_x[:, 256:] -> g_md[b, b_slot, wrap(i0[i])], and the score-input layer (K = 1):
//                           g_add_i = sum_k g_pre_c0[i, k] w_c0[k] -> g_scores[b, i, i0[i] or N],
//                           dW_c0[k] = sum_i g_pre_c0[i, k] add_i.
// Rows are pair-major: r = (p * B + b) * N + i.  Both are deterministic: every sum runs in a fixed order (rows
// ascending within fixed 128-row chunks, chunks ascending, fp64 accumulators), there are no floating-point atomics,
// and each output element is written by exactly one thread.
#include <climits>

#include "../../include/mvm_b200.h"
#include "common.cuh"

namespace {

constexpr int kChunk = 128;      // rows per partial sum of the weight / bias reductions
constexpr int kC = 256;          // channels of the head's hidden layers

__device__ __forceinline__ double warp_sum_fixed(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// grid = chunks, block = kC: thread k owns channel k; rows of the chunk in ascending order
__global__ void __launch_bounds__(kC) conf_tail_kernel(const float* __restrict__ conf, const float* __restrict__ g_conf,
                                                       const float* __restrict__ h, const float* __restrict__ w_last,
                                                       int rows, float* __restrict__ g_h, double* __restrict__ part) {
  const int k = threadIdx.x;
  const int r0 = blockIdx.x * kChunk, r1 = min(rows, r0 + kChunk);
  const float w = w_last[k];
  double sw = 0.0, sb = 0.0;
  for (int r = r0; r < r1; ++r) {
    const float c = conf[r];
    const float gl = g_conf[r] * (c * (1.f - c));
    g_h[(long long)r * kC + k] = gl * w;
    sw += (double)gl * (double)h[(long long)r * kC + k];
    sb += (double)gl;
  }
  part[(long long)blockIdx.x * (kC + 1) + k] = sw;
  if (k == 0) part[(long long)blockIdx.x * (kC + 1) + kC] = sb;
}

// out[k] = sum over chunks (ascending) of part[chunk * stride + k], k < n
__global__ void conf_partial_sum_kernel(const double* __restrict__ part, int chunks, int stride, int n,
                                        float* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  double s = 0.0;
  for (int c = 0; c < chunks; ++c) s += part[(long long)c * stride + k];
  out[k] = (float)s;
}

struct PairSlots { int a[MVM_CONF_MAX_PAIRS]; int b[MVM_CONF_MAX_PAIRS]; };

// grid (N, T, B), block = kC: target row (b, t, j) of g_md, channel k.  Pairs ascending; for a pair whose second view
// is t, the rows i with wrap(i0[i]) == j ascending (a warp-wide ballot over 32 rows at a time: every warp scans the
// same rows, so the hits are uniform and the additions run in row order).
__global__ void __launch_bounds__(kC) conf_gather_md_kernel(const float* __restrict__ g_x, const int64_t* __restrict__ i0,
                                                            int P, int B, int N, int T, int n_pad, PairSlots slots,
                                                            float* __restrict__ g_md) {
  const int j = blockIdx.x, t = blockIdx.y, b = blockIdx.z, k = threadIdx.x, lane = threadIdx.x & 31;
  double acc = 0.0;
  bool any = false;
  for (int p = 0; p < P; ++p) {
    const long long base = (long long)(p * B + b) * N;
    if (slots.a[p] == t) {
      acc += (double)g_x[(base + j) * 2 * kC + k];
      any = true;
    }
    if (slots.b[p] == t) {
      for (int i0b = 0; i0b < N; i0b += 32) {
        const int i = i0b + lane;
        bool hit = false;
        if (i < N) {
          const long long m = i0[base + i];
          hit = (m < 0 ? N - 1 : (int)m) == j;
        }
        unsigned mask = __ballot_sync(0xffffffffu, hit);
        while (mask) {
          const int l = __ffs(mask) - 1;
          mask &= mask - 1;
          acc += (double)g_x[(base + i0b + l) * 2 * kC + kC + k];
          any = true;
        }
      }
    }
  }
  if (any) {
    float* o = g_md + ((long long)(b * T + t) * n_pad + j) * kC + k;
    *o = (float)((double)*o + acc);
  }
}

// grid = chunks, block = kC (8 warps): warp w takes the chunk's rows r = r0 + w, r0 + w + 8, ...; lane l holds the
// channels l + 32 q.  g_add_r = sum_k g_pre_c0[r, k] w_c0[k] (lane partials in q order, then the xor tree) goes to
// g_scores[p * B + b, i, col] (one thread per row: no other row writes there); the dW_c0 partials of the 8 warps are
// summed in warp order.
__global__ void __launch_bounds__(kC) conf_score_input_kernel(const float* __restrict__ g_pre_c0, const float* __restrict__ add,
                                                              const float* __restrict__ w_c0, const int64_t* __restrict__ i0,
                                                              int rows, int N, float* __restrict__ g_scores,
                                                              double* __restrict__ part) {
  __shared__ double s_part[kC / 32][kC];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = blockIdx.x * kChunk, r1 = min(rows, r0 + kChunk);
  float w[8];
  double dw[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) { w[q] = w_c0[lane + 32 * q]; dw[q] = 0.0; }
  for (int r = r0 + warp; r < r1; r += kC / 32) {
    const float* g = g_pre_c0 + (long long)r * kC;
    const double a = (double)add[r];
    double dot = 0.0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const double v = (double)g[lane + 32 * q];
      dot += v * (double)w[q];
      dw[q] += v * a;
    }
    dot = warp_sum_fixed(dot);
    if (lane == 0) {
      const long long pb = r / N;
      const int i = r - (int)(pb * N);
      const long long m = i0[r];
      float* o = g_scores + (pb * (N + 1) + i) * (long long)(N + 1) + (m < 0 ? N : (int)m);
      *o = (float)((double)*o + dot);
    }
  }
#pragma unroll
  for (int q = 0; q < 8; ++q) s_part[warp][lane + 32 * q] = dw[q];
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int ww = 0; ww < kC / 32; ++ww) s += s_part[ww][threadIdx.x];
  part[(long long)blockIdx.x * kC + threadIdx.x] = s;
}

// i0 range over every entry: integer min / max (order-independent)
__global__ void conf_i0_range_kernel(const int64_t* __restrict__ i0, long long n, long long* __restrict__ mm) {
  long long lo = LLONG_MAX, hi = LLONG_MIN;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long v = i0[e];
    lo = v < lo ? v : lo;
    hi = v > hi ? v : hi;
  }
  atomicMin(mm, lo);
  atomicMax(mm + 1, hi);
}

__global__ void conf_i0_range_init_kernel(long long* mm) { mm[0] = LLONG_MAX; mm[1] = LLONG_MIN; }

int g_conf_i0_check = 1;     // mvm_debug_set_conf_i0_check

}  // namespace

extern "C" void mvm_debug_set_conf_i0_check(int on) { g_conf_i0_check = on != 0; }

extern "C" size_t mvm_conf_backward_ws_doubles(int rows) {
  return rows < 1 ? 0 : (size_t)mvm_div_up(rows, kChunk) * (kC + 1) + 2;
}

extern "C" int mvm_conf_tail_backward(const float* conf, const float* g_conf, const float* h, const float* w_last, int rows,
                                      float* g_h, float* dw_last, float* db_last, double* ws, size_t ws_doubles,
                                      void* stream) {
  MVM_REQUIRE(conf && g_conf && h && w_last && g_h && dw_last && db_last && ws && rows >= 1);
  const int chunks = mvm_div_up(rows, kChunk);
  MVM_REQUIRE(ws_doubles >= mvm_conf_backward_ws_doubles(rows));
  cudaStream_t s = (cudaStream_t)stream;
  MvmProfScope prof__(MVM_TAG_CONF, s);
  conf_tail_kernel<<<chunks, kC, 0, s>>>(conf, g_conf, h, w_last, rows, g_h, ws);
  MVM_CHECK_LAUNCH();
  conf_partial_sum_kernel<<<1, kC, 0, s>>>(ws, chunks, kC + 1, kC, dw_last);
  MVM_CHECK_LAUNCH();
  conf_partial_sum_kernel<<<1, 32, 0, s>>>(ws + kC, chunks, kC + 1, 1, db_last);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

extern "C" int mvm_conf_gather_backward(const float* g_x, const float* g_pre_c0, const float* add, const float* w_c0,
                                        const int64_t* i0, int n_pairs, int batch, int n, int n_views, int n_pad,
                                        const int* slot_a, const int* slot_b, float* g_md, float* g_scores, float* dw_c0,
                                        double* ws, size_t ws_doubles, void* stream) {
  MVM_REQUIRE(g_x && g_pre_c0 && add && w_c0 && i0 && slot_a && slot_b && g_md && g_scores && dw_c0 && ws);
  MVM_REQUIRE(n_pairs >= 1 && n_pairs <= MVM_CONF_MAX_PAIRS && batch >= 1 && n >= 1 && n_views >= 2 &&
              n_views <= MVM_MAX_VIEWS && n_pad >= n && batch <= 65535 && n_views <= 65535);
  const long long rows_ll = (long long)n_pairs * batch * n;
  MVM_REQUIRE(rows_ll <= 0x7fffffffLL);
  const int rows = (int)rows_ll;
  MVM_REQUIRE(ws_doubles >= mvm_conf_backward_ws_doubles(rows));
  PairSlots slots;
  for (int p = 0; p < n_pairs; ++p) {
    MVM_REQUIRE(slot_a[p] >= 0 && slot_a[p] < n_views && slot_b[p] >= 0 && slot_b[p] < n_views && slot_a[p] != slot_b[p]);
    slots.a[p] = slot_a[p];
    slots.b[p] = slot_b[p];
  }
  cudaStream_t s = (cudaStream_t)stream;
  MvmProfScope prof__(MVM_TAG_CONF, s);
  // i0 must lie in [-1, n): its range is read back before the gathers launch (one 16-byte copy)
  if (g_conf_i0_check) {
    long long* mm = reinterpret_cast<long long*>(ws + (ws_doubles - 2));
    conf_i0_range_init_kernel<<<1, 1, 0, s>>>(mm);
    MVM_CHECK_LAUNCH();
    conf_i0_range_kernel<<<mvm_div_up(rows, 256) < 120 ? mvm_div_up(rows, 256) : 120, 256, 0, s>>>(i0, rows_ll, mm);
    MVM_CHECK_LAUNCH();
    long long range[2];
    if (cudaMemcpyAsync(range, mm, sizeof(range), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
        cudaStreamSynchronize(s) != cudaSuccess)
      return MVM_ERR_LAUNCH;
    MVM_REQUIRE(range[0] >= -1 && range[1] < n);
  }
  const int chunks = mvm_div_up(rows, kChunk);
  conf_gather_md_kernel<<<dim3(n, n_views, batch), kC, 0, s>>>(g_x, i0, n_pairs, batch, n, n_views, n_pad, slots, g_md);
  MVM_CHECK_LAUNCH();
  conf_score_input_kernel<<<chunks, kC, 0, s>>>(g_pre_c0, add, w_c0, i0, rows, n, g_scores, ws);
  MVM_CHECK_LAUNCH();
  conf_partial_sum_kernel<<<1, kC, 0, s>>>(ws, chunks, kC, kC, dw_c0);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
