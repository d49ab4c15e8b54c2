// One launch that gathers the per-view inputs of a matcher call (the reference's `data` dict: keypoints{i} [B,n_i,2],
// scores{i} [B,n_i], descriptors{i} [B,256,n_i]; multi_view_matcher.py:229-262) into the zero-padded view-slot-major
// buffers mvm_matcher_forward reads: kpts [B,T,n_pad,2], scores [B,T,n_pad], desc [B,T,256,n_pad].  Replaces the
// 3 fills + 3 strided copies per view the Python mirror used to issue.
#include "../../include/mvm_b200.h"
#include "common.cuh"
#include "kernels.cuh"

namespace {

struct PackArgs {
  const float* kpts[MVM_MAX_VIEWS];
  const float* scores[MVM_MAX_VIEWS];
  const float* desc[MVM_MAX_VIEWS];
  int counts[MVM_MAX_VIEWS];            // widths of the source tensors
  const int* slot_counts;               // device [batch * n_views] or nullptr (every slot holds counts[t])
  int batch, n_views, n_pad;
  float* out_kpts; float* out_scores; float* out_desc;
};

// grid (258 row blocks, T, B): rows 0..255 = descriptor channels, 256 = scores, 257 = keypoints
__global__ void __launch_bounds__(256) pack_views_kernel(const __grid_constant__ PackArgs g) {
  const int r = blockIdx.x, t = blockIdx.y, b = blockIdx.z;
  const int w = g.counts[t], n_pad = g.n_pad;
  const int n = slot_count(g.slot_counts, b, g.n_views, t, w);   // rows n .. n_pad are zero, whatever the source holds
  const long long slot = (long long)b * g.n_views + t;
  if (r < 256) {
    const float* src = g.desc[t] + ((long long)b * 256 + r) * w;
    float* dst = g.out_desc + (slot * 256 + r) * n_pad;
    for (int i = threadIdx.x; i < n_pad; i += blockDim.x) dst[i] = i < n ? __ldg(src + i) : 0.f;
  } else if (r == 256) {
    const float* src = g.scores[t] + (long long)b * w;
    float* dst = g.out_scores + slot * n_pad;
    for (int i = threadIdx.x; i < n_pad; i += blockDim.x) dst[i] = i < n ? __ldg(src + i) : 0.f;
  } else {
    const float* src = g.kpts[t] + (long long)b * w * 2;
    float* dst = g.out_kpts + slot * n_pad * 2;
    for (int i = threadIdx.x; i < 2 * n_pad; i += blockDim.x) dst[i] = i < 2 * n ? __ldg(src + i) : 0.f;
  }
}

}  // namespace

extern "C" int mvm_pack_views(const float* const* kpts, const float* const* scores, const float* const* desc,
                              const int* counts, int batch, int n_views, int n_pad, float* out_kpts,
                              float* out_scores, float* out_desc, void* stream) {
  return mvm_pack_views_ragged(kpts, scores, desc, counts, nullptr, batch, n_views, n_pad, out_kpts, out_scores, out_desc,
                               stream);
}

extern "C" int mvm_pack_views_ragged(const float* const* kpts, const float* const* scores, const float* const* desc,
                                     const int* counts, const int* slot_counts, int batch, int n_views, int n_pad,
                                     float* out_kpts, float* out_scores, float* out_desc, void* stream) {
  MVM_REQUIRE(kpts && scores && desc && counts && out_kpts && out_scores && out_desc);
  MVM_REQUIRE(n_views >= 1 && n_views <= MVM_MAX_VIEWS && batch >= 1 && n_pad >= 1);
  PackArgs g;
  for (int t = 0; t < n_views; ++t) {
    MVM_REQUIRE(counts[t] >= 0 && counts[t] <= n_pad);
    MVM_REQUIRE(counts[t] == 0 || (kpts[t] && scores[t] && desc[t]));
    g.kpts[t] = kpts[t]; g.scores[t] = scores[t]; g.desc[t] = desc[t]; g.counts[t] = counts[t];
  }
  g.slot_counts = slot_counts;
  g.batch = batch; g.n_views = n_views; g.n_pad = n_pad;
  g.out_kpts = out_kpts; g.out_scores = out_scores; g.out_desc = out_desc;
  MvmProfScope prof__(MVM_TAG_MISC, (cudaStream_t)stream);
  pack_views_kernel<<<dim3(258, n_views, batch), 256, 0, (cudaStream_t)stream>>>(g);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
