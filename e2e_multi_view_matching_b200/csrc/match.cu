// Mutual-nearest-neighbour match extraction on the coupling matrix, reference:
// multi_view_matcher.py:288-300 (threshold 0.) and superglue.py:268-278 (threshold 0.2);
// SURVEY.md appendix A.4.  Ties resolve to the first maximal index like torch.max.
#include "common.cuh"
#include "kernels.cuh"

namespace {

struct ArgMax {
  float v;
  int i;
};
__device__ __forceinline__ ArgMax better(ArgMax a, ArgMax b) {
  // larger value wins; on ties the smaller index (first occurrence)
  if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}

// blockIdx.y = problem (pair*batch + bi); blockIdx.x covers rows (first part) then column
// chunks.  idx layout per problem: idx0[n_pad] | idx1[n_pad] ; max0 floats alias after.
__global__ void __launch_bounds__(256) rowcol_argmax_kernel(PairTable tab, int batch, int n_pad,
                                                            int row_blocks, int* __restrict__ idx_ws,
                                                            float* __restrict__ max_ws) {
  const int prob = blockIdx.y;
  const int p = prob / batch, bi = prob % batch;
  const int ld = tab.n[p] + 1;
  const int m = slot_count(tab.slot, bi, tab.n_views, tab.a[p], tab.m[p]);
  const int n = slot_count(tab.slot, bi, tab.n_views, tab.b[p], tab.n[p]);
  const float* Z = tab.scores[p] + (long long)bi * (tab.m[p] + 1) * ld;
  int* idx0 = idx_ws + (long long)prob * 2 * n_pad;
  int* idx1 = idx0 + n_pad;
  float* max0 = max_ws + (long long)prob * n_pad;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  if ((int)blockIdx.x < row_blocks) {
    const int i = blockIdx.x * 8 + warp;
    if (i >= m) return;
    const float* zr = Z + (long long)i * ld;
    ArgMax best{-INFINITY, 0x7fffffff};
    for (int j = lane; j < n; j += 32) best = better(best, ArgMax{zr[j], j});
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ArgMax other{__shfl_xor_sync(0xffffffffu, best.v, o), __shfl_xor_sync(0xffffffffu, best.i, o)};
      best = better(best, other);
    }
    // an all-NaN row never replaces the sentinel: clamp so that the index stays usable (the reference returns
    // garbage for NaN inputs; an out-of-range index here would be an illegal address in mutual_kernel / conf_gather)
    if (lane == 0) { idx0[i] = best.i == 0x7fffffff ? 0 : best.i; max0[i] = best.v; }
  } else {
    __shared__ float sv[8][32];
    __shared__ int si[8][32];
    const int j = (blockIdx.x - row_blocks) * 32 + lane;
    ArgMax best{-INFINITY, 0x7fffffff};
    if (j < n)
      for (int i = warp; i < m; i += 8) best = better(best, ArgMax{Z[(long long)i * ld + j], i});
    sv[warp][lane] = best.v; si[warp][lane] = best.i;
    __syncthreads();
    if (warp == 0 && j < n) {
      for (int w = 1; w < 8; ++w) best = better(best, ArgMax{sv[w][lane], si[w][lane]});
      idx1[j] = best.i == 0x7fffffff ? 0 : best.i;
    }
  }
}

__global__ void __launch_bounds__(256) mutual_kernel(PairTable tab, int batch, int n_pad,
                                                     float thresh, const int* __restrict__ idx_ws,
                                                     const float* __restrict__ max_ws) {
  const int prob = blockIdx.y;
  const int p = prob / batch, bi = prob % batch;
  const int mc = tab.m[p], nc = tab.n[p];      // capacities: the row strides of the outputs
  const int m = slot_count(tab.slot, bi, tab.n_views, tab.a[p], mc);
  const int n = slot_count(tab.slot, bi, tab.n_views, tab.b[p], nc);
  const int* idx0 = idx_ws + (long long)prob * 2 * n_pad;
  const int* idx1 = idx0 + n_pad;
  const float* max0 = max_ws + (long long)prob * n_pad;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  // keypoints past this tuple's counts: no match
  if (t >= m && t < mc) { tab.matches_a[p][(long long)bi * mc + t] = -1; tab.ms_a[p][(long long)bi * mc + t] = 0.f; }
  if (t >= n && t < nc) { tab.matches_b[p][(long long)bi * nc + t] = -1; tab.ms_b[p][(long long)bi * nc + t] = 0.f; }
  if (m == 0 || n == 0) {
    // one view of this tuple has no keypoints: nothing to match, and the argmax pass wrote no index of the other side
    // (the indices below would be read from an earlier call's workspace)
    if (t < m) { tab.matches_a[p][(long long)bi * mc + t] = -1; tab.ms_a[p][(long long)bi * mc + t] = 0.f; }
    if (t < n) { tab.matches_b[p][(long long)bi * nc + t] = -1; tab.ms_b[p][(long long)bi * nc + t] = 0.f; }
    return;
  }
  if (t < m) {
    const int j = idx0[t];
    const bool mutual = idx1[j] == t;
    const float ms = mutual ? expf(max0[t]) : 0.f;
    const bool valid = mutual && (ms > thresh);
    tab.matches_a[p][(long long)bi * mc + t] = valid ? (int64_t)j : (int64_t)-1;
    tab.ms_a[p][(long long)bi * mc + t] = ms;
  }
  if (t < n) {
    const int i = idx1[t];
    const bool mutual1 = idx0[i] == t;
    // mscores0[i] / valid0[i] recomputed for the partner row
    const bool mutual0_i = idx1[idx0[i]] == i;
    const float ms0_i = mutual0_i ? expf(max0[i]) : 0.f;
    const bool valid0_i = mutual0_i && (ms0_i > thresh);
    const float ms1 = mutual1 ? ms0_i : 0.f;
    const bool valid1 = mutual1 && valid0_i;
    tab.matches_b[p][(long long)bi * nc + t] = valid1 ? (int64_t)i : (int64_t)-1;
    tab.ms_b[p][(long long)bi * nc + t] = ms1;
  }
}

}  // namespace

int launch_extract_matches(const PairTable& tab, int batch, int n_pad, float thresh, int* idx_ws,
                           cudaStream_t stream) {
  MvmProfScope prof__(MVM_TAG_MATCH, stream);
  int max_m = 0, max_n = 0;
  for (int p = 0; p < tab.n_pairs; ++p) {
    max_m = tab.m[p] > max_m ? tab.m[p] : max_m;
    max_n = tab.n[p] > max_n ? tab.n[p] : max_n;
  }
  MVM_REQUIRE(max_m <= n_pad && max_n <= n_pad && max_m > 0 && max_n > 0);
  const int probs = tab.n_pairs * batch;
  float* max_ws = reinterpret_cast<float*>(idx_ws + (long long)probs * 2 * n_pad);
  const int row_blocks = mvm_div_up(max_m, 8), col_blocks = mvm_div_up(max_n, 32);
  rowcol_argmax_kernel<<<dim3(row_blocks + col_blocks, probs), 256, 0, stream>>>(
      tab, batch, n_pad, row_blocks, idx_ws, max_ws);
  MVM_CHECK_LAUNCH();
  const int mx = max_m > max_n ? max_m : max_n;
  mutual_kernel<<<dim3(mvm_div_up(mx, 256), probs), 256, 0, stream>>>(tab, batch, n_pad, thresh,
                                                                      idx_ws, max_ws);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
