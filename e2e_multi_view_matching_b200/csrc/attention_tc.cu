// Multi-head attention on the tensor cores with tf32 operands (single pass, or 3xTF32 with the hi / lo planes of K and
// V^T written by the QKV GEMM epilogue); the kernel is attn_wg::attention_wg_kernel (attention_wg.cuh).
#include "attention_wg.cuh"

long long* g_attn_dbg = nullptr;   // clock64 trace buffer of mvm_debug_set_attention_timing (no kernel of this build writes it)

extern "C" void mvm_debug_set_attention_timing(long long* buf) { g_attn_dbg = buf; }

// qkv [V, n_pad, 768] (q | k | unused-v), vt [V, 256, n_pad] = V^T per head; out [V, n_pad, 256]
int launch_attention_tc(const float* qkv, const float* vt, float* out, int batch, int n_pad, AttnSegs segs,
                        int is_cross, int n_pass, cudaStream_t stream, const float* klo, const float* vtlo) {
  MVM_REQUIRE(n_pad % 64 == 0 && attn_segs_valid(segs, n_pad, is_cross));
  MvmProfScope prof__(MVM_TAG_ATTN, stream);
  const int V = batch * segs.n_views;
  const long long rows = (long long)V * n_pad;
  const CUtensorMap* tK = mvm_get_tmap_2d(qkv, rows, 768, 768, attn_wg::Cfg<1>::BKV);
  const CUtensorMap* tV = mvm_get_tmap_2d(vt, (long long)V * 256, n_pad, n_pad, attn_wg::HD);
  if (n_pass == 3) {
    MVM_REQUIRE(klo && vtlo);
    const CUtensorMap* tKlo = mvm_get_tmap_2d(klo, rows, 256, 256, attn_wg::Cfg<1>::BKV);
    const CUtensorMap* tVlo = mvm_get_tmap_2d(vtlo, (long long)V * 256, n_pad, n_pad, attn_wg::HD);
    return attn_wg::launch<3>(tK, tV, tKlo, tVlo, qkv, out, batch, n_pad, segs, is_cross, stream);
  }
  return attn_wg::launch<1>(tK, tV, tK, tV, qkv, out, batch, n_pad, segs, is_cross, stream);
}
