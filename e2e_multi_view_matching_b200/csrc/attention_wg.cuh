// Flash-style multi-head attention on the Hopper tensor cores (TMA + mbarrier ring + wgmma) with multi-view key/value
// segments.  Reference semantics: attention() superglue.py:87-91, MultiHeadedAttention :94-109, cross source =
// concatenation of the other views (multi_view_matcher.py:76-78,92-95).  prob[B,4,N,M] is never materialised.
//
// One CTA = 128 queries of one (view, head); keys / values stream through in tiles of BKV (128 in MODE 16, 64 in the
// tf32 modes).  384 threads:
//   warps 0-3, 4-7   two consumer warpgroups, queries [0,64) and [64,128) of the block: S = Q K^T with wgmma (A = Q
//                    fragments in registers, B = K tile in shared memory), online softmax on the accumulator registers
//                    (a row lives in the four threads of a quad), P re-packed in registers as the A operand of O += P V
//                    (B = V tile in shared memory); O stays in registers until the end
//   warps 8-11       the producer warpgroup: one lane of warp 8 issues the TMA loads of the K and V planes of every key
//                    tile into ST-deep rings
// Operand arithmetic (MODE):
//   1   single-pass TF32: K from the fused QKV projection [rows, 768], V^T [view * 256 + h * 64 + d, key] written by the
//       QKV GEMM epilogue (tf32 wgmma has no transposed B: both operands K-major)
//   3   3xTF32 (fp32-faithful): every product is A.B + A.B_lo + A_lo.B; the tf32 hi / lo planes of K and V^T are
//       written by the QKV GEMM epilogue, Q and P are split in registers
//   16  fp16x3: the same three products on half-precision hi / lo planes (hi = fp16(x), lo = fp16(x - hi): 22 bits like
//       the tf32 pair) at K = 16 per instruction; K and V planes [rows, 256] come from the QKV GEMM epilogue and V is
//       read key-major as an MN-major B operand (no transposed copy); Q is split once per CTA into hi / lo register
//       fragments, so S = Q K^T reads only K from shared memory.  128-key tiles halve the per-key cost of what each
//       tile pays once on a warpgroup's critical path (the waits, the ping-pong barriers, the rescale decision, the
//       issue); the rescale points of the online softmax and the grouping of the row sums follow the tile, so results
//       differ from 64-key tiles by reordered fp32 rounding
// Schedule (MODE 16): inside a warpgroup, S(j+1) = Q K(j+1)^T and O += P(j) V(j) are issued back to back and the
// softmax of tile j+1 runs while P(j) V(j) is on the tensor cores; across the two warpgroups, named barriers make them
// take turns issuing (FlashAttention-3 §3.1 ping-pong), so one warpgroup's MMAs cover the other's softmax.  The tf32
// modes run each tile's S, softmax and P V in order; MODE 1 showed no gain beyond run-to-run noise from the ping-pong
// alone and has not been measured with the overlap inside a warpgroup.
// For a given tile size, every schedule does the same operations on every output element in the same order.
#pragma once
#include <cuda_fp16.h>
#include "common.cuh"
#include "kernels.cuh"
#include "tc_common.cuh"

namespace attn_wg {

constexpr int BQ = 128, HD = 64;
constexpr int PRODUCER_WARP = 8;
// 384 threads (warps 8-11 are the producer warpgroup) and setmaxnreg 2 x 232 + 40 = the 504 per-thread registers of one
// SM sub-partition (one warp of each warpgroup).  ptxas budgets a wgmma kernel by whole warpgroups, so 288 threads cap
// every thread at 168 registers: too few for the Q hi / lo fragments next to the pipelined fp16x3 schedule, and the
// 3xTF32 instance spilled under that cap.
constexpr int NTHREADS = 384;
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
// named barriers (0 is __syncthreads): warpgroup w may issue its MMAs once PP_BAR + w completes
constexpr int PP_BAR = 1;

template <int MODE>
struct Cfg {
  static constexpr bool F16 = MODE == 16;
  static constexpr bool PIPE = F16;                           // pipelined + ping-pong schedule
  // keys per tile: S is one m64 x n128 wgmma per k-step in MODE 16 (the tf32 modes keep n64: their operand planes are
  // twice as wide)
  static constexpr int BKV = F16 ? 128 : 64;
  static constexpr int PL = MODE == 1 ? 1 : 2;                // operand planes per tile (hi [, lo])
  static constexpr int PLANE = 16384;                         // [128 x 64] fp16 box, or two [64 x 32] fp32 boxes
  static constexpr int TILE = PL * PLANE;
  static constexpr int ST = MODE == 1 ? 4 : 3;                // ring depth of K and of V (MODE 16: 192 KB)
  static constexpr int OFF_V = ST * TILE;
  static constexpr int OFF_BAR = 2 * ST * TILE;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
};

struct Args {
  const float* qkv;    // [V, n_pad, 768]
  float* out;          // [V, n_pad, 256]
  int n_pad;
  AttnSegs segs;
  int is_cross;
};

__device__ __forceinline__ float ex2_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// rn_tf32 of a finite value (ties away, == cvt.rna.tf32.f32) in two integer instructions
__device__ __forceinline__ float tf32_hi(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
}
__device__ __forceinline__ void split_pack(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void named_bar_sync(int id, int n) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int n) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory");
}
// A-operand registers of an issued wgmma stay live (and unchanged) until this point, after the wait that retires it
template <int N>
__device__ __forceinline__ void fence_regs(uint32_t (*a)[4]) {
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) asm volatile("" : "+r"(a[i][e])::"memory");
}

template <int MODE>
__global__ void __launch_bounds__(NTHREADS, 1)
attention_wg_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                    const __grid_constant__ CUtensorMap tmKlo, const __grid_constant__ CUtensorMap tmVlo,
                    const __grid_constant__ Args g) {
  using C_ = Cfg<MODE>;
  constexpr bool F16 = C_::F16, PIPE = C_::PIPE;
  constexpr int ST = C_::ST, PLANE = C_::PLANE, TILE = C_::TILE, BKV = C_::BKV;
  constexpr int KS = F16 ? 4 : 8;                             // K steps over d (S)
  constexpr int KP = BKV / (F16 ? 16 : 8);                    // K steps over keys (P V)
  constexpr int NSC = BKV / 2;                                // S accumulators per thread
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C_::OFF_BAR);
  uint64_t* k_full = bars;              // [ST]
  uint64_t* k_empty = bars + ST;        // [ST] (256 arrivals)
  uint64_t* v_full = bars + 2 * ST;     // [ST]
  uint64_t* v_empty = bars + 3 * ST;    // [ST] (256 arrivals)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * BQ;
  const int h = blockIdx.y;
  const int v = blockIdx.z;
  const int T = g.segs.n_views;
  const int t = v % T, b = v / T;
  if (q0 >= slot_count(g.segs.slot, b, T, t, g.segs.counts[t])) return;

  if (threadIdx.x == 0) {
    for (int i = 0; i < ST; ++i) {
      tc::mbar_init(k_full + i, 1); tc::mbar_init(k_empty + i, 256);
      tc::mbar_init(v_full + i, 1); tc::mbar_init(v_empty + i, 256);
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp >= PRODUCER_WARP) {
    // =========================== TMA producer: K(j), V(j) in key-tile order ===========================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
    if (warp == PRODUCER_WARP && lane == 0) {
      tc::prefetch_tmap(&tmK); tc::prefetch_tmap(&tmV);
      if (MODE != 1) { tc::prefetch_tmap(&tmKlo); tc::prefetch_tmap(&tmVlo); }
      int j = 0;
      for (int sg = 0; sg < T; ++sg) {
        if (g.is_cross ? (sg == t) : (sg != t)) continue;
        const int cnt = slot_count(g.segs.slot, b, T, sg, g.segs.counts[sg]);
        for (int k0 = 0; k0 < cnt; k0 += BKV, ++j) {
          const int s = j % ST;
          const uint32_t ph = ((j / ST) & 1) ^ 1;
          const int krow = (b * T + sg) * g.n_pad + k0;          // row of the tile's first key in the K / V planes
          uint8_t* sk = smem + s * TILE;
          uint8_t* sv = smem + C_::OFF_V + s * TILE;
          tc::mbar_wait(k_empty + s, ph);
          tc::mbar_arrive_expect_tx(k_full + s, TILE);
          if (F16) {
            tc::tma_load_2d(sk, &tmK, k_full + s, h * HD, krow);
            tc::tma_load_2d(sk + PLANE, &tmKlo, k_full + s, h * HD, krow);
          } else {
            tc::tma_load_2d(sk, &tmK, k_full + s, 256 + h * HD, krow);
            tc::tma_load_2d(sk + 8192, &tmK, k_full + s, 256 + h * HD + 32, krow);
            if (MODE == 3) {
              tc::tma_load_2d(sk + PLANE, &tmKlo, k_full + s, h * HD, krow);
              tc::tma_load_2d(sk + PLANE + 8192, &tmKlo, k_full + s, h * HD + 32, krow);
            }
          }
          tc::mbar_wait(v_empty + s, ph);
          tc::mbar_arrive_expect_tx(v_full + s, TILE);
          if (F16) {
            tc::tma_load_2d(sv, &tmV, v_full + s, h * HD, krow);
            tc::tma_load_2d(sv + PLANE, &tmVlo, v_full + s, h * HD, krow);
          } else {
            const int vrow = (b * T + sg) * 256 + h * HD;        // V^T rows = d, columns = keys
            tc::tma_load_2d(sv, &tmV, v_full + s, k0, vrow);
            tc::tma_load_2d(sv + 8192, &tmV, v_full + s, k0 + 32, vrow);
            if (MODE == 3) {
              tc::tma_load_2d(sv + PLANE, &tmVlo, v_full + s, k0, vrow);
              tc::tma_load_2d(sv + PLANE + 8192, &tmVlo, v_full + s, k0 + 32, vrow);
            }
          }
        }
      }
    }
    return;
  }

  // =========================== consumers ===========================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
  const int wg = warp >> 2, wq = warp & 3;
  const int gr = lane >> 2, tq = lane & 3;
  const int lrow = wg * 64 + wq * 16 + gr;                      // query rows of this thread: lrow, lrow + 8
  // Q fragments, raw fp32 (rows past the view are read but never written back; rows past the buffer read as zero).
  // MODE 16 splits them once into the hi / lo operand registers; the tf32 modes split them inside the key-tile loop.
  // When operand registers defined only before the loop are not pinned past the wait that retires their wgmma, ptxas
  // (CUDA 12.9) reuses them inside the loop body and later tiles read stale Q_lo: retire_s fences them.
  float2 qraw[KS][4];
  {
    const long long total = (long long)gridDim.z * g.n_pad;
    const long long r0 = (long long)v * g.n_pad + q0 + lrow;
    const float* q_r0 = g.qkv + r0 * 768 + h * HD;
    const float* q_r1 = q_r0 + 8 * 768;
    const bool in0 = r0 < total, in1 = r0 + 8 < total;
    const float2 z = make_float2(0.f, 0.f);
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
      if (F16) {
        const int c = 16 * kk + 2 * tq;
        qraw[kk][0] = in0 ? __ldg(reinterpret_cast<const float2*>(q_r0 + c)) : z;
        qraw[kk][1] = in1 ? __ldg(reinterpret_cast<const float2*>(q_r1 + c)) : z;
        qraw[kk][2] = in0 ? __ldg(reinterpret_cast<const float2*>(q_r0 + c + 8)) : z;
        qraw[kk][3] = in1 ? __ldg(reinterpret_cast<const float2*>(q_r1 + c + 8)) : z;
      } else {
        const int c = 8 * kk + tq;
        qraw[kk][0] = make_float2(in0 ? __ldg(q_r0 + c) : 0.f, 0.f);
        qraw[kk][1] = make_float2(in1 ? __ldg(q_r1 + c) : 0.f, 0.f);
        qraw[kk][2] = make_float2(in0 ? __ldg(q_r0 + c + 4) : 0.f, 0.f);
        qraw[kk][3] = make_float2(in1 ? __ldg(q_r1 + c + 4) : 0.f, 0.f);
      }
    }
  }
  uint32_t qhi[KS][4], qlo[KS][4];                              // the Q operand of S
  if constexpr (F16) {
    // the f16 k16 A fragment of d [16 kk, 16 kk + 16) is the pair layout qraw[kk] was loaded in
#pragma unroll
    for (int kk = 0; kk < KS; ++kk)
#pragma unroll
      for (int e = 0; e < 4; ++e) split_pack(qraw[kk][e].x, qraw[kk][e].y, qhi[kk][e], qlo[kk][e]);
  }

  // online softmax in log2 units (scores * log2(e) / sqrt(d)); row hh of this thread = lrow + 8 hh.  The reference m of
  // a row is only raised (and O, l rescaled) when the row maximum outgrows it by more than 2^8, and P is taken relative
  // to 2^-7 of it: softmax is invariant to the reference, P stays <= 2^15 (inside the fp16 range), and the fp16 lo plane
  // of a small probability stays far from the fp16 subnormals
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const float scale_l2e = 0.125f * 1.4426950408889634f;
  const int srcA = (lane & ~3) | (tq >> 1), srcB = srcA + 2;   // tf32 P fragments: owners of keys tq and tq + 4
  float sc[NSC], fo[2];                                          // fo: rescale of O by the last softmax (1: none)
  uint32_t phi[KP][4], plo[KP][4];                              // P of a softmax: the A operand of its P V

  auto prep_s = [&] {
    if constexpr (!F16) {
#pragma unroll
      for (int kk = 0; kk < KS; ++kk) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float x = qraw[kk][e].x;
          asm volatile("" : "+f"(x));                           // keeps the split inside the loop (no hoisting)
          const float hi = MODE == 3 ? tf32_hi(x) : x;
          qhi[kk][e] = __float_as_uint(hi);
          qlo[kk][e] = __float_as_uint(MODE == 3 ? tf32_hi(x - hi) : 0.f);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < NSC; ++i) sc[i] = 0.f;
    tc::fence_acc<BKV>(sc);                                     // zeroed before the wgmma fence
  };
  // ---- S = Q K^T on the K tile of ring stage st (issue only)
  auto issue_s = [&](int st, uint32_t ph) {
    tc::mbar_wait(k_full + st, ph);
    const uint32_t kb = tc::smem_u32(smem + st * TILE);
    tc::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
      if (F16) {
        const uint64_t dk = tc::make_sw128_desc(kb + kk * 32);
        tc::wgmma_f16_rs<BKV, 0>(sc, qhi[kk], dk);
        tc::wgmma_f16_rs<BKV, 0>(sc, qhi[kk], tc::make_sw128_desc(kb + PLANE + kk * 32));
        tc::wgmma_f16_rs<BKV, 0>(sc, qlo[kk], dk);
      } else {
        const uint32_t off = (kk >> 2) * 8192 + (kk & 3) * 32;
        const uint64_t dk = tc::make_sw128_desc(kb + off);
        tc::wgmma_tf32_rs<64>(sc, qhi[kk], dk);
        if (MODE == 3) {
          tc::wgmma_tf32_rs<64>(sc, qhi[kk], tc::make_sw128_desc(kb + PLANE + off));
          tc::wgmma_tf32_rs<64>(sc, qlo[kk], dk);
        }
      }
    }
    tc::wgmma_commit();
  };
  // after the wait that retired the S of ring stage st
  auto retire_s = [&](int st) {
    tc::fence_acc<BKV>(sc);
    fence_regs<KS>(qhi);
    fence_regs<KS>(qlo);
    tc::mbar_arrive(k_empty + st);
  };
  // ---- O += P V on the V tile of ring stage st (issue only)
  auto issue_pv = [&](int st, uint32_t ph) {
    tc::mbar_wait(v_full + st, ph);
    const uint32_t vb = tc::smem_u32(smem + C_::OFF_V + st * TILE);
    tc::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KP; ++kk) {
      if (F16) {
        const uint64_t dv = tc::make_sw128_desc(vb + kk * 2048);      // 16 keys x 128 B, V key-major (MN-major B)
        tc::wgmma_f16_rs<64, 1>(o, phi[kk], dv);
        tc::wgmma_f16_rs<64, 1>(o, phi[kk], tc::make_sw128_desc(vb + PLANE + kk * 2048));
        tc::wgmma_f16_rs<64, 1>(o, plo[kk], dv);
      } else {
        const uint32_t off = (kk >> 2) * 8192 + (kk & 3) * 32;
        const uint64_t dv = tc::make_sw128_desc(vb + off);
        tc::wgmma_tf32_rs<64>(o, phi[kk], dv);
        if (MODE == 3) {
          tc::wgmma_tf32_rs<64>(o, phi[kk], tc::make_sw128_desc(vb + PLANE + off));
          tc::wgmma_tf32_rs<64>(o, plo[kk], dv);
        }
      }
    }
    tc::wgmma_commit();
  };
  // after the wait that retired the P V of ring stage st
  auto retire_pv = [&](int st) {
    tc::fence_acc<64>(o);
    fence_regs<KP>(phi);
    fence_regs<KP>(plo);
    tc::mbar_arrive(v_empty + st);
  };
  // ---- online softmax of S in place (a row is spread over the four threads of a quad); sets fo, leaves O alone
  auto softmax = [&](int nvalid) {
    if (nvalid < BKV) {
#pragma unroll
      for (int i = 0; i < BKV / 8; ++i) {
        const int key = 8 * i + 2 * tq;
        if (key >= nvalid) { sc[4 * i] = -INFINITY; sc[4 * i + 2] = -INFINITY; }
        if (key + 1 >= nvalid) { sc[4 * i + 1] = -INFINITY; sc[4 * i + 3] = -INFINITY; }
      }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float mx = sc[2 * hh];
#pragma unroll
      for (int i = 0; i < BKV / 8; ++i) mx = fmaxf(mx, fmaxf(sc[4 * i + 2 * hh], sc[4 * i + 2 * hh + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      mx *= scale_l2e;
      fo[hh] = 1.f;
      if (mx > m_run[hh] + 8.f) {                               // the same decision in the four threads of the quad
        fo[hh] = ex2_ftz(m_run[hh] - mx);                       // < 2^-8
        m_run[hh] = mx;
        l_run[hh] *= fo[hh];
      }
      const float nm = 7.f - m_run[hh];
      float rs = 0.f;
#pragma unroll
      for (int i = 0; i < BKV / 8; ++i) {
        const float p0 = ex2_ftz(fmaf(sc[4 * i + 2 * hh], scale_l2e, nm));
        const float p1 = ex2_ftz(fmaf(sc[4 * i + 2 * hh + 1], scale_l2e, nm));
        sc[4 * i + 2 * hh] = p0;
        sc[4 * i + 2 * hh + 1] = p1;
        rs += p0 + p1;
      }
      l_run[hh] += rs;
    }
  };
  auto rescale_o = [&] {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      if (fo[hh] != 1.f) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o[4 * i + 2 * hh] *= fo[hh];
          o[4 * i + 2 * hh + 1] *= fo[hh];
        }
      }
    }
  };
  // ---- P as the register A operand of O += P V
  auto split_p = [&] {
#pragma unroll
    for (int kk = 0; kk < KP; ++kk) {
      if (F16) {
        // the accumulator layout of keys [16 kk, 16 kk + 16) is the k16 A fragment layout
#pragma unroll
        for (int e = 0; e < 4; ++e) split_pack(sc[8 * kk + 2 * e], sc[8 * kk + 2 * e + 1], phi[kk][e], plo[kk][e]);
      } else {
        // k8 A fragment: keys tq and tq + 4 of the step, held by quad lanes tq / 2 and 2 + tq / 2
        float a[4];
        const bool odd = tq & 1;
        const float x0 = __shfl_sync(0xffffffffu, sc[4 * kk], srcA), x1 = __shfl_sync(0xffffffffu, sc[4 * kk + 1], srcA);
        const float y0 = __shfl_sync(0xffffffffu, sc[4 * kk + 2], srcA), y1 = __shfl_sync(0xffffffffu, sc[4 * kk + 3], srcA);
        const float z0 = __shfl_sync(0xffffffffu, sc[4 * kk], srcB), z1 = __shfl_sync(0xffffffffu, sc[4 * kk + 1], srcB);
        const float w0 = __shfl_sync(0xffffffffu, sc[4 * kk + 2], srcB), w1 = __shfl_sync(0xffffffffu, sc[4 * kk + 3], srcB);
        a[0] = odd ? x1 : x0; a[1] = odd ? y1 : y0; a[2] = odd ? z1 : z0; a[3] = odd ? w1 : w0;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float hi = MODE == 3 ? tf32_hi(a[e]) : a[e];
          phi[kk][e] = __float_as_uint(hi);
          plo[kk][e] = __float_as_uint(a[e] - hi);   // the tensor core reads the top 19 bits: truncation costs 2^-21 |p|
        }
      }
    }
  };

  // Ping-pong: every stage (one per key tile, plus a last one for the final P V) is one bar.sync on the warpgroup's own
  // barrier before it issues and one bar.arrive on the other's after.  Warpgroup 1 opens with an extra arrive (warpgroup 0
  // issues first) and skips its arrive after the last stage, so both barriers end complete.  A warpgroup whose rows lie
  // past the view runs every stage all the same.
  // Stage j issues S(j) and P(j-1) V(j-1), and the softmax of tile j runs while P(j-1) V(j-1) is in flight.  That P V is
  // retired at the top of stage j+1 (then O is rescaled and P(j) split): ptxas places a wgmma wait as early as its basic
  // block allows, so a wait after the softmax in the same block would run before it; the top of the next stage lies
  // behind the loop's back edge.  The first stage has its own issue branch: a wgmma issued under a condition (j > 0)
  // that the following wait does not share makes ptxas serialise every wgmma of the kernel.
  auto finish_pv = [&](int jn) {                                // before stage jn: O += P(jn-1) V(jn-1) can be issued
    tc::wgmma_wait<0>();                                        // P(jn-2) V(jn-2)
    tc::fence_acc<64>(o);
    fence_regs<KP>(phi);
    fence_regs<KP>(plo);
    if (jn >= 2) tc::mbar_arrive(v_empty + (jn - 2) % ST);
    if (jn >= 1) {
      rescale_o();
      split_p();
    }
  };
  if (PIPE && wg == 1) named_bar_arrive(PP_BAR + 0, 256);
  int j = 0;
  for (int sg = 0; sg < T; ++sg) {
    if (g.is_cross ? (sg == t) : (sg != t)) continue;
    const int cnt = slot_count(g.segs.slot, b, T, sg, g.segs.counts[sg]);
    for (int k0 = 0; k0 < cnt; k0 += BKV, ++j) {
      const int nvalid = cnt - k0;      // keys of this tile that exist
      const int s = j % ST;
      const uint32_t ph = (j / ST) & 1;
      if constexpr (PIPE) {
        finish_pv(j);
        prep_s();
        named_bar_sync(PP_BAR + wg, 256);
        if (j == 0) {
          issue_s(s, ph);
          named_bar_arrive(PP_BAR + (wg ^ 1), 256);
          tc::wgmma_wait<0>();
        } else {
          issue_s(s, ph);
          issue_pv((j - 1) % ST, ((j - 1) / ST) & 1);
          named_bar_arrive(PP_BAR + (wg ^ 1), 256);
          tc::wgmma_wait<1>();
        }
        retire_s(s);
        softmax(nvalid);
      } else {
        prep_s();
        issue_s(s, ph);
        tc::wgmma_wait<0>();
        retire_s(s);
        softmax(nvalid);
        rescale_o();
        split_p();
        issue_pv(s, ph);
        tc::wgmma_wait<0>();
        retire_pv(s);
      }
    }
  }
  if constexpr (PIPE) {                                         // last stage: O += P V of the last tile
    finish_pv(j);
    named_bar_sync(PP_BAR + wg, 256);
    if (j > 0) issue_pv((j - 1) % ST, ((j - 1) / ST) & 1);
    if (wg == 0) named_bar_arrive(PP_BAR + 1, 256);
    tc::wgmma_wait<0>();
    if (j > 0) retire_pv((j - 1) % ST);
  }

  // ---- out = O / l
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float l = l_run[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.f / l;
    const int r = lrow + 8 * hh;
    if (q0 + r < g.n_pad) {
      float* op = g.out + ((long long)v * g.n_pad + q0 + r) * 256 + h * HD + 2 * tq;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<float2*>(op + 8 * i) = make_float2(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv);
    }
  }
}

template <int MODE>
int launch(const CUtensorMap* tK, const CUtensorMap* tV, const CUtensorMap* tKlo, const CUtensorMap* tVlo, const float* qkv,
           float* out, int batch, int n_pad, const AttnSegs& segs, int is_cross, cudaStream_t stream) {
  using C_ = Cfg<MODE>;
  if (!tK || !tV || !tKlo || !tVlo) return MVM_ERR_LAUNCH;
  mvm_once_per_device(MODE == 16 ? MVM_ONCE_ATTN_H3 : MVM_ONCE_ATTN_TC + 16 * (MODE == 3), [&] {
    cudaFuncSetAttribute(attention_wg_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, C_::SMEM_BYTES);
  });
  Args g;
  g.qkv = qkv; g.out = out; g.n_pad = n_pad; g.segs = segs; g.is_cross = is_cross;
  dim3 grid(mvm_div_up(n_pad, BQ), 4, batch * segs.n_views);
  attention_wg_kernel<MODE><<<grid, NTHREADS, C_::SMEM_BYTES, stream>>>(*tK, *tV, *tKlo, *tVlo, g);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

}  // namespace attn_wg
