// Multi-head attention with multi-view key/value segments, fp32 CUDA cores, flash-style
// (the probability tensor prob[B,4,N,M] of superglue.py:89-91 is never materialised).
// Reference semantics: attention() superglue.py:87-91, MultiHeadedAttention :94-109,
// cross source = concatenation of the other views, multi_view_matcher.py:76-78,92-95.
// This is the exact-fp32 cross-check path; the tensor-core kernels live in attention_wg.cuh.
#include "common.cuh"
#include "kernels.cuh"

namespace {

constexpr int BQ = 64, BKV = 64, HD = 64, LDS = 68;
constexpr int QKV_LD = 768;

// smem: Qt[HD][LDS] | Kt[HD][LDS] (reused as Pt[BKV][LDS]) | Vs[BKV][HD]
constexpr int SMEM_FLOATS = HD * LDS * 2 + BKV * HD;

__global__ void __launch_bounds__(256) attention_simt_kernel(const float* __restrict__ qkv,
                                                             float* __restrict__ out, int n_pad,
                                                             AttnSegs segs, int is_cross) {
  extern __shared__ float smem[];
  float* Qt = smem;
  float* Kt = smem + HD * LDS;
  float* Vs = smem + 2 * HD * LDS;

  const int q0 = blockIdx.x * BQ;
  const int h = blockIdx.y;
  const int v = blockIdx.z;
  const int T = segs.n_views;
  const int t = v % T, b = v / T;
  if (q0 >= segs.counts[t]) return;  // padded query tile: nothing to produce

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;

  // load Q tile transposed: Qt[d][q]
  {
    const float* qb = qkv + ((long long)v * n_pad + q0) * QKV_LD + h * HD;
    for (int i = tid; i < BQ * (HD / 4); i += 256) {
      const int r = i / (HD / 4), d4 = (i % (HD / 4)) * 4;
      const float4 x = *reinterpret_cast<const float4*>(qb + (long long)r * QKV_LD + d4);
      Qt[(d4 + 0) * LDS + r] = x.x; Qt[(d4 + 1) * LDS + r] = x.y;
      Qt[(d4 + 2) * LDS + r] = x.z; Qt[(d4 + 3) * LDS + r] = x.w;
    }
  }

  float m_run[4], l_run[4], o[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m_run[i] = -INFINITY; l_run[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  }
  const float scale_l2e = 0.125f * 1.4426950408889634f;  // 1/sqrt(64) * log2(e)

  for (int s = 0; s < T; ++s) {
    if (is_cross ? (s == t) : (s != t)) continue;
    const int cnt = segs.counts[s];
    const int vs = b * T + s;
    for (int k0 = 0; k0 < cnt; k0 += BKV) {
      __syncthreads();  // previous tile's P/V reads done (and Q stores visible on first pass)
      const float* kb = qkv + ((long long)vs * n_pad + k0) * QKV_LD + 256 + h * HD;
      const float* vb = kb + 256;
      for (int i = tid; i < BKV * (HD / 4); i += 256) {
        const int r = i / (HD / 4), d4 = (i % (HD / 4)) * 4;
        const float4 x = *reinterpret_cast<const float4*>(kb + (long long)r * QKV_LD + d4);
        Kt[(d4 + 0) * LDS + r] = x.x; Kt[(d4 + 1) * LDS + r] = x.y;
        Kt[(d4 + 2) * LDS + r] = x.z; Kt[(d4 + 3) * LDS + r] = x.w;
        *reinterpret_cast<float4*>(Vs + r * HD + d4) =
            *reinterpret_cast<const float4*>(vb + (long long)r * QKV_LD + d4);
      }
      __syncthreads();

      float sacc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) sacc[i][j] = 0.f;
#pragma unroll 8
      for (int d = 0; d < HD; ++d) {
        const float4 qa = *reinterpret_cast<const float4*>(Qt + d * LDS + ty * 4);
        const float4 ka = *reinterpret_cast<const float4*>(Kt + d * LDS + tx * 4);
        const float q[4] = {qa.x, qa.y, qa.z, qa.w};
        const float k[4] = {ka.x, ka.y, ka.z, ka.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) sacc[i][j] = fmaf(q[i], k[j], sacc[i][j]);
      }
      // scale, mask, online softmax
      float p[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float mx = -INFINITY;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const bool valid = (k0 + tx * 4 + j) < cnt;
          sacc[i][j] = valid ? sacc[i][j] * scale_l2e : -INFINITY;
          mx = fmaxf(mx, sacc[i][j]);
        }
#pragma unroll
        for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
        const float m_new = fmaxf(m_run[i], mx);
        const float corr = exp2f(m_run[i] - m_new);  // exp2f(-inf) = 0 on the first tile
        float rs = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          p[i][j] = exp2f(sacc[i][j] - m_new);
          rs += p[i][j];
        }
#pragma unroll
        for (int off = 8; off > 0; off >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, off);
        l_run[i] = l_run[i] * corr + rs;
        m_run[i] = m_new;
#pragma unroll
        for (int j = 0; j < 4; ++j) o[i][j] *= corr;
      }
      __syncthreads();  // all S reads of Kt done -> reuse as Pt[k][q]
      float* Pt = Kt;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) Pt[(tx * 4 + j) * LDS + ty * 4 + i] = p[i][j];
      __syncthreads();
#pragma unroll 8
      for (int k = 0; k < BKV; ++k) {
        const float4 pa = *reinterpret_cast<const float4*>(Pt + k * LDS + ty * 4);
        const float4 va = *reinterpret_cast<const float4*>(Vs + k * HD + tx * 4);
        const float pp[4] = {pa.x, pa.y, pa.z, pa.w};
        const float vv[4] = {va.x, va.y, va.z, va.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) o[i][j] = fmaf(pp[i], vv[j], o[i][j]);
      }
    }
  }

  float* ob = out + ((long long)v * n_pad + q0) * 256 + h * HD;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float inv = 1.f / l_run[i];
    float4 r = make_float4(o[i][0] * inv, o[i][1] * inv, o[i][2] * inv, o[i][3] * inv);
    *reinterpret_cast<float4*>(ob + (long long)(ty * 4 + i) * 256 + tx * 4) = r;
  }
}

}  // namespace

int launch_attention_simt(const float* qkv, float* out, int batch, int n_pad, AttnSegs segs,
                          int is_cross, cudaStream_t stream) {
  MVM_REQUIRE(n_pad % BQ == 0 && attn_segs_valid(segs, n_pad, is_cross));
  MvmProfScope prof__(MVM_TAG_ATTN, stream);
  const int smem_bytes = SMEM_FLOATS * (int)sizeof(float);
  mvm_once_per_device(MVM_ONCE_ATTN_SIMT, [&] {
    cudaFuncSetAttribute(attention_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
  });
  dim3 grid(n_pad / BQ, 4, batch * segs.n_views);
  attention_simt_kernel<<<grid, 256, smem_bytes, stream>>>(qkv, out, n_pad, segs, is_cross);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
