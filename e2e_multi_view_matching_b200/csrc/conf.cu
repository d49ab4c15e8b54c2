// Confidence head glue kernels.  Reference: ConfidenceMLP multi_view_matcher.py:39-53 and its
// call site :302-306 -- inputs are mdesc0, mdesc1 gathered at indices0 (a -1 index wraps to the
// LAST keypoint of view b) and the OT score scores[b, i, indices0[i]] (-1 selects the dustbin
// column).  The 512->512->256 and 256->256 layers run as GEMMs; these kernels do the gather,
// the scalar->256 first layer of layers_c, and the final 256->1 + sigmoid.
#include "common.cuh"
#include "kernels.cuh"

namespace {

__global__ void __launch_bounds__(256) conf_gather_kernel(const float* __restrict__ mdesc,
                                                          PairTable tab, int batch, int n_pad,
                                                          float* __restrict__ feat,
                                                          float* __restrict__ sc) {
  const int prob = blockIdx.y;
  const int p = prob / batch, bi = prob % batch;
  const int mc = tab.m[p], nc = tab.n[p];      // capacities: the strides of matches_a and scores
  const int m = slot_count(tab.slot, bi, tab.n_views, tab.a[p], mc);
  const int n = slot_count(tab.slot, bi, tab.n_views, tab.b[p], nc);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * 8 + warp;
  if (i >= n_pad) return;
  const long long r = (long long)prob * n_pad + i;
  float4* fo = reinterpret_cast<float4*>(feat + r * 512);
  if (i >= m) {
    for (int c = lane; c < 128; c += 32) fo[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane == 0) sc[r] = 0.f;
    return;
  }
  const long long idx = tab.matches_a[p][(long long)bi * mc + i];
  // python negative index -1 -> this tuple's last keypoint (row 0 stands in when view b has none: m rows of a
  // tuple without keypoints in b are never valid matches)
  const int jb = idx < 0 ? max(n - 1, 0) : (int)idx;
  const int js = idx < 0 ? n : (int)idx;       // scores[..., -1] -> this tuple's dustbin column
  const float4* ra = reinterpret_cast<const float4*>(
      mdesc + ((long long)(bi * tab.n_views + tab.a[p]) * n_pad + i) * 256);
  const float4* rb = reinterpret_cast<const float4*>(
      mdesc + ((long long)(bi * tab.n_views + tab.b[p]) * n_pad + jb) * 256);
  for (int c = lane; c < 64; c += 32) {
    fo[c] = ra[c];
    fo[64 + c] = rb[c];
  }
  if (lane == 0)
    sc[r] = tab.scores[p][(long long)bi * (mc + 1) * (nc + 1) + (long long)i * (nc + 1) + js];
}

__global__ void conf_c0_kernel(const float* __restrict__ sc, const float* __restrict__ w,
                               const float* __restrict__ b, float* __restrict__ out,
                               long long rows) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= rows * 256) return;
  const long long r = e >> 8;
  const int c = (int)(e & 255);
  out[e] = fmaxf(fmaf(w[c], sc[r], b[c]), 0.f);
}

__global__ void __launch_bounds__(256) conf_final_kernel(const float* __restrict__ h,
                                                         const float* __restrict__ wl, float bl,
                                                         PairTable tab, int batch, int n_pad) {
  const int prob = blockIdx.y;
  const int p = prob / batch, bi = prob % batch;
  const int mc = tab.m[p], m = slot_count(tab.slot, bi, tab.n_views, tab.a[p], mc);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * 8 + warp;
  if (i >= mc) return;
  if (i >= m) {                                // past this tuple's count
    if (lane == 0) tab.conf[p][(long long)bi * mc + i] = 0.f;
    return;
  }
  const float* hr = h + ((long long)prob * n_pad + i) * 256;
  float acc = 0.f;
  for (int c = lane; c < 256; c += 32) acc = fmaf(hr[c], wl[c], acc);
  acc = warp_sum(acc);
  if (lane == 0) tab.conf[p][(long long)bi * mc + i] = 1.f / (1.f + expf(-(acc + bl)));
}

}  // namespace

int launch_conf_gather(const float* mdesc, const PairTable& tab, int batch, int n_pad, float* feat,
                       float* sc, cudaStream_t stream) {
  MvmProfScope prof__(MVM_TAG_CONF, stream);
  conf_gather_kernel<<<dim3(mvm_div_up(n_pad, 8), tab.n_pairs * batch), 256, 0, stream>>>(
      mdesc, tab, batch, n_pad, feat, sc);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

int launch_conf_c0(const float* sc, const float* w, const float* b, float* out, long long rows,
                   cudaStream_t stream) {
  MvmProfScope prof__(MVM_TAG_CONF, stream);
  const long long total = rows * 256;
  conf_c0_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(sc, w, b, out, rows);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

int launch_conf_final(const float* h, const float* wl, float bl, const PairTable& tab, int batch,
                      int n_pad, cudaStream_t stream) {
  MvmProfScope prof__(MVM_TAG_CONF, stream);
  conf_final_kernel<<<dim3(mvm_div_up(n_pad, 8), tab.n_pairs * batch), 256, 0, stream>>>(
      h, wl, bl, tab, batch, n_pad);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
