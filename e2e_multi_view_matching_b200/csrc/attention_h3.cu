// fp32-faithful multi-head attention with HALF-PRECISION operand planes ("fp16x3"): every product is
// A_hi.B_hi + A_hi.B_lo + A_lo.B_hi with hi = fp16(x), lo = fp16(x - hi), fp32 accumulation.  hi + lo carries 22
// mantissa bits -- the same as the tf32 hi/lo pair of attention_tc.cu -- but an f16 wgmma moves K = 16 per instruction
// where tf32 moves K = 8, so the three passes cost 1.5 tf32 passes.  (lo is an fp16 subnormal, exact to 2^-24
// absolute, once |x| < 2^-3, so a small V loses relative precision; DESIGN.md section 3 gives the measured edge.)
// The kernel is attn_wg::attention_wg_kernel<16> (attention_wg.cuh): K_hi | K_lo and V_hi | V_lo [64 keys x 64 d] fp16
// tiles by TMA from the planes the QKV GEMM epilogue writes; V is read key-major as an MN-major B operand.
#include "attention_wg.cuh"

// Kernel variant of the fp16-plane attention (mvm_debug_set_attention_h3_variant).  This build has one kernel; the
// setting is kept so that callers of the A/B hook keep working, and both values run it.
int g_attn_h3_variant = 1;
extern "C" void mvm_debug_set_attention_h3_variant(int v) { g_attn_h3_variant = v ? 1 : 0; }

// K / V planes in half precision: kh, kl, vh, vl [rows, 256] (written by the QKV GEMM epilogue)
int launch_attention_h3(const float* qkv, const __half* kh, const __half* kl, const __half* vh, const __half* vl,
                        float* out, int batch, int n_pad, AttnSegs segs, int is_cross, cudaStream_t stream) {
  MVM_REQUIRE(qkv && kh && kl && vh && vl && out);
  MVM_REQUIRE(n_pad % 64 == 0 && attn_segs_valid(segs, n_pad, is_cross));
  MvmProfScope prof__(MVM_TAG_ATTN, stream);
  const long long rows = (long long)batch * segs.n_views * n_pad;
  const CUtensorMap* tK = mvm_get_tmap_2d_f16(kh, rows, 256, 256, attn_wg::Cfg<16>::BKV);
  const CUtensorMap* tKlo = mvm_get_tmap_2d_f16(kl, rows, 256, 256, attn_wg::Cfg<16>::BKV);
  const CUtensorMap* tV = mvm_get_tmap_2d_f16(vh, rows, 256, 256, attn_wg::Cfg<16>::BKV);
  const CUtensorMap* tVlo = mvm_get_tmap_2d_f16(vl, rows, 256, 256, attn_wg::Cfg<16>::BKV);
  return attn_wg::launch<16>(tK, tV, tKlo, tVlo, qkv, out, batch, n_pad, segs, is_cross, stream);
}
