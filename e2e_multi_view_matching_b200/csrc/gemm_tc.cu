// Tensor-core GEMM (sm_90a: TMA + mbarrier ring + wgmma) with fused epilogue for the 1x1 convolutions of the matcher
// (superglue.py:51-62,101-121; multi_view_matcher.py:8-53) and for its score matrices (multi_view_matcher.py:278-280):
//   C[M,N] = act(alpha * [A | A2][M,K] . W[N,K]^T + bias[N]) + R[M,N]      (fp32, both operands K-major)
//
// Operand arithmetic (template parameters NPASS, WM):
//   NPASS 1             single-pass TF32 (what torch 1.10 did by default on Ampere+)
//   NPASS 3, W_RAW      3xTF32: D += A_hi.W_hi + A_hi.W_lo + A_lo.W_hi, hi = rn_tf32(x), lo = rn_tf32(x - hi); the W tile
//                       is split into its hi / lo planes in shared memory after it lands
//   NPASS 3, W_TF32     3xTF32 with W given as its two tf32 planes (what packing.py stores next to the raw weights)
//   NPASS 3, W_F16      fp16x3: W given as fp16 hi / lo planes of wscale * W (packing.py), A split into fp16 hi / lo;
//                       the same 22-bit operands, K = 16 per instruction instead of 8
// A is split on chip in every mode: it is the register operand of wgmma, so its hi / lo planes never touch shared memory.
//
// One CTA computes 128 x BN output tiles:
//   warps 0-3, 4-7   two consumer warpgroups, tile rows [0,64) and [64,128): A fragments from the 128B-swizzled shared
//                    tile -> hi / lo in registers -> wgmma m64 x BN (B = the W planes, shared-memory descriptors), fp32
//                    accumulators in registers; then the epilogue (below).  With BN = 128 the
//                    wgmma of k-block kt are issued before the A fragments of kt + 1 are split, so the split runs under
//                    them (two fragment sets in registers, raised to 232 per thread by setmaxnreg)
//   warps 8-11       the producer warpgroup (40 registers): one lane of warp 8 issues the
//                    TMA loads of A [128 x BK] (fp32) and the W planes [BN x 128 B] into a STAGES-deep ring
// Epilogue of the persistent instances (128 columns, pre-split W planes: Cfg::STAGED): the consumers finish the tile in
// rounds of one 16 KB TMA box ([128 x 32] fp32 or [128 x 64] of one fp16 plane), written swizzled into one of two
// staging buffers after the ring, and go back to the mainloop of the next tile after the last round; lane 0 of warp 9
// (the storer) drains each round by a TMA store and, for a residual, loads the residual box of the round that will use
// that buffer next, so the residual arrives in shared memory before it is needed (in place R == C stays correct: a box
// is loaded before the same box is stored, and tiles do not overlap).  The tensor maps carry the logical M x N, so rows
// >= M and columns N .. ldc are never written.  The score matrices (rows of n + 1 floats: not 16-byte aligned), the V^T
// output of the tf32 attention, C or R with only 8-byte alignment, and the other instances keep the direct stores
// from the accumulators, with the bias / residual operands of eight column groups loaded at once.
// The tile schedule is static: with `persistent` one CTA per SM walks the tiles (the producer fills the ring for the
// next tile under the epilogue of the current one), otherwise one tile per CTA.  Both issue the same instructions per
// tile, so their results are bit-identical.
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>
#include <cuda_fp16.h>
#include "common.cuh"
#include "kernels.cuh"
#include "tc_common.cuh"

namespace {

constexpr int BM = 128;
constexpr int PRODUCER_WARP = 8;
// 384 threads (warps 8-11 are the producer warpgroup) and setmaxnreg 2 x 232 + 40 = the 504 per-thread registers of one
// SM sub-partition (one warp of each warpgroup): the second fragment set of the pipelined mainloop (128-column tiles), or
// the 128 accumulators of the in-order one (256-column tiles).  ptxas budgets a wgmma kernel by whole warpgroups, so
// 288 threads would cap every thread at 168 registers, and the 256-column instances spilled under that cap.
constexpr int NTHREADS = 384;
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
enum { W_RAW = 0, W_TF32 = 1, W_F16 = 2 };

template <int BN, int NPASS, int WM>
struct Cfg {
  static constexpr int BK = WM == W_F16 ? 64 : 32;            // one 128-byte swizzle row of W per k-block
  static constexpr int A_BYTES = BM * BK * 4;                 // raw fp32 A: one or two [128 x 32] boxes
  static constexpr int W_PLANE = BN * 128;
  static constexpr int PLANES = NPASS == 3 ? 2 : 1;
  static constexpr int STAGE_BYTES = A_BYTES + PLANES * W_PLANE;
  static constexpr int TMA_BYTES = A_BYTES + (WM == W_RAW ? 1 : PLANES) * W_PLANE;
  static constexpr int STAGES = (196608 / STAGE_BYTES) < 6 ? (196608 / STAGE_BYTES) : 6;
  // the persistent instances (128-column tiles, pre-split W planes) stage their output tiles for TMA stores in two
  // [128 rows x 128 B] buffers after the ring
  static constexpr bool STAGED = BN == 128 && NPASS == 3 && WM != W_RAW;
  static constexpr int OUT_BYTES = STAGED ? 2 * 16384 : 0;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + OUT_BYTES + 1024 /*align*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 232448, "over the sm_90 dynamic shared memory opt-in limit");
};

struct GArgs {
  const float* bias;
  const float* R; int ldr;
  float* C; int ldc;
  int M, N, K, K1;
  float alpha;
  int relu;
  // optional transposed output for columns >= vt_col0: VT[(m / n_pad), n - vt_col0, m % n_pad] (V^T of the QKV
  // projection for the tf32 attention kernel), with its tf32 lo plane in VTLO
  float* VT; int vt_col0; int n_pad;
  // tf32 planes of the attention's K operand: columns [256,512) are stored as rn_tf32 in C, the remainder in KLO [M,256]
  float* KLO; float* VTLO;
  // half-precision operand planes for attention_h3.cu (fp16x3): K hi / lo and V hi / lo, all [rows, 256] (V stays
  // key-major: the attention reads it as an MN-major B operand); when set they replace the fp32 K and V thirds of C
  __half* KH16; __half* KL16; __half* VH16; __half* VL16;
  int tiles_m, tiles_n;
  // split-K (weight-gradient GEMMs: few output tiles, a very long contraction): K is cut into `ksplit` slices, slice s
  // writes its partial product to rows [s * tiles_m * BM, ...) of C (a slab buffer that a small kernel sums afterwards,
  // in fixed order).  1 = off.
  int ksplit;
  // 1: output tiles leave through the staging buffers by TMA stores (maps in StoreMaps), all but the V^T columns
  int stage;
};

// Tensor maps of the staged epilogue: C [rows, N] fp32 (rows = M, or the split-K slabs), the residual R [M, N], and the
// output planes [M, 256]: KH16, KL16, VH16, VL16 (fp16 boxes [128 x 64]) or KLO in p[0] (fp32 boxes [128 x 32]).
struct StoreMaps {
  CUtensorMap c, r, p[4];
};

// SCORE mode: one launch computes every (pair, tuple) score matrix  scores = mdesc_a . mdesc_b^T * alpha  into the
// inner [m, n] block of the [m+1, n+1] coupling buffers.  A = descriptors of view a (raw fp32, split on chip), W = the
// tf32 planes of the descriptors of view b.
struct ScoreTab {
  int n_pairs, batch, n_views, n_pad;
  int a[MVM_MAX_PAIRS], b[MVM_MAX_PAIRS], m[MVM_MAX_PAIRS], n[MVM_MAX_PAIRS];
  float* scores[MVM_MAX_PAIRS];
  const int* slot;             // PairTable::slot (m / n are then the capacities)
};

// rn_tf32 of a finite value (ties away, == cvt.rna.tf32.f32) in two integer instructions
__device__ __forceinline__ float tf32_hi(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
}
__device__ __forceinline__ void split_pack_h(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
// shared-memory accesses of the staging buffers (the aligned dynamic-smem pointer is generic to the compiler)
__device__ __forceinline__ void sts_f2(uint32_t a, float2 v) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(v.x), "f"(v.y) : "memory");
}
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ float2 lds_f2(uint32_t a) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory");
  return v;
}
// A-fragment registers of an issued wgmma stay live (and unchanged) until this point, after the wait that retires it
__device__ __forceinline__ void fence_afrag(uint32_t (&a)[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) asm volatile("" : "+r"(a[i][e])::"memory");
}

template <int BN, int NPASS, int WM, bool SCORE>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_wg_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
               const __grid_constant__ CUtensorMap tmWhi, const __grid_constant__ CUtensorMap tmWlo,
               const __grid_constant__ GArgs g, const __grid_constant__ ScoreTab st,
               const __grid_constant__ StoreMaps sm) {
  using C_ = Cfg<BN, NPASS, WM>;
  static_assert(NPASS == 3 || WM == W_RAW, "single pass reads the raw W");
  constexpr int BK = C_::BK, STAGES = C_::STAGES, A_BYTES = C_::A_BYTES, W_PLANE = C_::W_PLANE;
  constexpr int STAGE_BYTES = C_::STAGE_BYTES;
  constexpr int KSTEPS = 4;                                   // 4 x (K = 8 tf32 | K = 16 halves) per k-block
  constexpr bool PIPE = BN == 128;                            // pipelined mainloop (see the consumers)
  constexpr bool STAGED = C_::STAGED && !SCORE;               // staged epilogue (when g.stage)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* obuf = smem + STAGES * STAGE_BYTES;                                  // [2][16 KB] output staging
  uint64_t* full = reinterpret_cast<uint64_t*>(obuf + C_::OUT_BYTES);          // [STAGES] TMA landed
  uint64_t* empty = full + STAGES;                                              // [STAGES] both warpgroups done (256)
  uint64_t* ostaged = empty + STAGES;      // [2] staging buffer written by all 256 consumer threads
  uint64_t* ofree = ostaged + 2;           // [2] staging buffer drained by its store (and holding its residual box)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nk = SCORE ? g.K / BK : g.K / BK / g.ksplit;     // k-blocks per tile (per K slice)
  const int per_prob = g.tiles_m * g.tiles_n;
  const int n_tiles = SCORE ? per_prob * st.n_pairs * st.batch : per_prob * g.ksplit;
  // tile -> output tile origin (m0, n0), the rows the A / W boxes start at, and the problem (K slice or pair x tuple)
  auto decode = [&](int tile, int& m0, int& n0, int& a_row, int& w_row, int& prob) {
    prob = tile / per_prob;
    const int r = tile % per_prob;
    m0 = (r / g.tiles_n) * BM; n0 = (r % g.tiles_n) * BN;
    if (!SCORE) {
      a_row = m0; w_row = n0;
    } else {
      const int p = prob / st.batch, bi = prob % st.batch;
      a_row = (bi * st.n_views + st.a[p]) * st.n_pad + m0;
      w_row = (bi * st.n_views + st.b[p]) * st.n_pad + n0;
    }
  };
  // How the staged epilogue writes the tile at column n0, in rounds of one 16 KB box per staging buffer (the same
  // precedence as the direct stores below): 0 = fp32 C, four [128 x 32] boxes; 1 = the fp16 K / V planes, hi and lo of
  // two [128 x 64] halves; 2 = the tf32 K planes, rn_tf32 in C and the remainder in KLO, of four [128 x 32] quarters;
  // -1 = not staged (V^T, direct stores)
  auto tile_kind = [&](int n0) {
    if (g.VT && n0 >= g.vt_col0) return -1;
    if (g.KH16 && n0 >= 256) return 1;
    if (g.KLO && n0 >= 256 && n0 < 512) return 2;
    return 0;
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      tc::mbar_init(full + s, 1);
      tc::mbar_init(empty + s, 256);
    }
    if (STAGED)
      for (int b = 0; b < 2; ++b) {
        tc::mbar_init(ostaged + b, 256);
        tc::mbar_init(ofree + b, 1);
      }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp >= PRODUCER_WARP) {
    // ================================ TMA producer ================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
    if (STAGED && g.stage && warp == PRODUCER_WARP + 1 && lane == 0) {
      // ---- storer: drains each staged round by a TMA store, then hands its buffer back for round u + 2 (loading
      // that round's residual box first, if any: a residual is only staged into a plain fp32 C)
      tc::prefetch_tmap(&sm.c);
      if (g.R) tc::prefetch_tmap(&sm.r);
      if (g.KH16)
        for (int i = 0; i < 4; ++i) tc::prefetch_tmap(&sm.p[i]);
      if (g.KLO) tc::prefetch_tmap(&sm.p[0]);
      auto hand_back = [&](uint32_t u, int tile, int q) {
        uint64_t* bar = ofree + (u & 1);
        if (!g.R) {
          tc::mbar_arrive(bar);
        } else if (tile < n_tiles) {
          int m0, n0, a_row, w_row, prob;
          decode(tile, m0, n0, a_row, w_row, prob);
          tc::mbar_arrive_expect_tx(bar, 16384);
          tc::tma_load_2d(obuf + (u & 1) * 16384, &sm.r, bar, n0 + 32 * q, m0);
        }
      };
      hand_back(0, blockIdx.x, 0);
      hand_back(1, blockIdx.x, 1);
      uint32_t u = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int m0, n0, a_row, w_row, prob;
        decode(tile, m0, n0, a_row, w_row, prob);
        const int kind = tile_kind(n0);
        if (kind < 0) continue;
        const int rounds = kind == 2 ? 8 : 4;
        for (int j = 0; j < rounds; ++j, ++u) {
          const uint8_t* buf = obuf + (u & 1) * 16384;
          tc::mbar_wait(ostaged + (u & 1), (u >> 1) & 1);
          if (kind == 0) {
            tc::tma_store_2d(&sm.c, buf, n0 + 32 * j, m0 + prob * g.tiles_m * BM);
          } else if (kind == 1) {
            const bool v = n0 >= 512;
            tc::tma_store_2d(&sm.p[(v ? 2 : 0) + (j & 1)], buf, n0 - (v ? 512 : 256) + 64 * (j >> 1), m0);
          } else {
            if (j & 1) tc::tma_store_2d(&sm.p[0], buf, n0 - 256 + 32 * (j >> 1), m0);
            else tc::tma_store_2d(&sm.c, buf, n0 + 32 * (j >> 1), m0);
          }
          tc::tma_store_commit();
          tc::tma_store_wait_read<0>();
          // with a residual every tile has 4 rounds: round u + 2 is quarter j + 2 of this tile or j - 2 of the next
          hand_back(u + 2, j < 2 ? tile : tile + gridDim.x, (j + 2) & 3);
        }
      }
      tc::tma_store_wait_all();
    }
    if (warp == PRODUCER_WARP && lane == 0) {
      tc::prefetch_tmap(&tmA); tc::prefetch_tmap(&tmA2); tc::prefetch_tmap(&tmWhi); tc::prefetch_tmap(&tmWlo);
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int m0, n0, a_row, w_row, prob;
        decode(tile, m0, n0, a_row, w_row, prob);
        for (int kt = 0; kt < nk; ++kt, ++it) {
          const int s = it % STAGES;
          tc::mbar_wait(empty + s, ((it / STAGES) & 1) ^ 1);
          tc::mbar_arrive_expect_tx(full + s, C_::TMA_BYTES);
          uint8_t* sp = smem + s * STAGE_BYTES;
          const int k = kt * BK + (SCORE ? 0 : prob * nk * BK);
          if (k < g.K1) tc::tma_load_2d(sp, &tmA, full + s, k, a_row);
          else tc::tma_load_2d(sp, &tmA2, full + s, k - g.K1, a_row);
          if (WM == W_F16) {   // second [128 x 32] fp32 box of the 64-wide k-block (K1 is a multiple of 64)
            if (k < g.K1) tc::tma_load_2d(sp + 16384, &tmA, full + s, k + 32, a_row);
            else tc::tma_load_2d(sp + 16384, &tmA2, full + s, k + 32 - g.K1, a_row);
          }
          tc::tma_load_2d(sp + A_BYTES, &tmWhi, full + s, k, w_row);
          if (WM != W_RAW) tc::tma_load_2d(sp + A_BYTES + W_PLANE, &tmWlo, full + s, k, w_row);
        }
      }
    }
    return;
  }

  // ================================ consumers ================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
  const int wg = warp >> 2, wq = warp & 3;
  const int gr = lane >> 2, tq = lane & 3;
  const int row0 = wg * 64 + wq * 16 + gr;                     // tile rows of this thread: row0, row0 + 8
  float acc[BN / 2];
  // A fragments (hi / lo) of two consecutive k-blocks: k-block kt + 1 is split into one set while the wgmma of kt,
  // which read the other, are in flight
  uint32_t ahi0[KSTEPS][4], alo0[KSTEPS][4], ahi1[KSTEPS][4], alo1[KSTEPS][4];

  // wait for ring stage `it`, split its W tile (3xTF32 on raw W) and the A fragments of this thread's rows
  auto prep = [&](uint32_t it, uint32_t (&ahi)[KSTEPS][4], uint32_t (&alo)[KSTEPS][4]) {
      const int s = it % STAGES;
      tc::mbar_wait(full + s, (it / STAGES) & 1);
      uint8_t* sp = smem + s * STAGE_BYTES;
      if (WM == W_RAW && NPASS == 3) {
        // hi = rn_tf32(w) replaces the landed tile in place, lo = rn_tf32(w - hi) goes to the second plane; both are
        // element-wise images of the tile, so the (swizzled) offsets carry over
        float4* w = reinterpret_cast<float4*>(sp + A_BYTES);
        float4* wl = reinterpret_cast<float4*>(sp + A_BYTES + W_PLANE);
#pragma unroll 4
        for (int i = threadIdx.x; i < BN * 32 / 4; i += 256) {
          const float4 x = w[i];
          float4 h;
          h.x = tc::tf32_rn(x.x); h.y = tc::tf32_rn(x.y); h.z = tc::tf32_rn(x.z); h.w = tc::tf32_rn(x.w);
          w[i] = h;
          wl[i] = make_float4(tc::tf32_rn(x.x - h.x), tc::tf32_rn(x.y - h.y), tc::tf32_rn(x.z - h.z), tc::tf32_rn(x.w - h.w));
        }
        tc::fence_proxy_async();      // generic-proxy writes -> visible to the tensor core (async proxy)
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
      // A fragments of rows row0 / row0 + 8 from the 128B-swizzled tile: 16-byte chunk c of row r sits at c ^ (r & 7)
      const uint8_t* ar = sp + row0 * 128;
#pragma unroll
      for (int kk = 0; kk < KSTEPS; ++kk) {
        if (WM == W_F16) {
          const uint8_t* ab = ar + (kk >> 1) * 16384;
          const int ch = 4 * (kk & 1) + (tq >> 1), wo = (tq & 1) * 8;
          const float2 x0 = *reinterpret_cast<const float2*>(ab + ((ch ^ gr) << 4) + wo);
          const float2 x1 = *reinterpret_cast<const float2*>(ab + 1024 + ((ch ^ gr) << 4) + wo);
          const float2 x2 = *reinterpret_cast<const float2*>(ab + (((ch + 2) ^ gr) << 4) + wo);
          const float2 x3 = *reinterpret_cast<const float2*>(ab + 1024 + (((ch + 2) ^ gr) << 4) + wo);
          split_pack_h(x0.x, x0.y, ahi[kk][0], alo[kk][0]);
          split_pack_h(x1.x, x1.y, ahi[kk][1], alo[kk][1]);
          split_pack_h(x2.x, x2.y, ahi[kk][2], alo[kk][2]);
          split_pack_h(x3.x, x3.y, ahi[kk][3], alo[kk][3]);
        } else {
          float x[4];
          x[0] = *reinterpret_cast<const float*>(ar + (((2 * kk) ^ gr) << 4) + tq * 4);
          x[1] = *reinterpret_cast<const float*>(ar + 1024 + (((2 * kk) ^ gr) << 4) + tq * 4);
          x[2] = *reinterpret_cast<const float*>(ar + (((2 * kk + 1) ^ gr) << 4) + tq * 4);
          x[3] = *reinterpret_cast<const float*>(ar + 1024 + (((2 * kk + 1) ^ gr) << 4) + tq * 4);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            if (NPASS == 3) {
              const float h = tf32_hi(x[e]);
              ahi[kk][e] = __float_as_uint(h);
              alo[kk][e] = __float_as_uint(tf32_hi(x[e] - h));
            } else {
              ahi[kk][e] = __float_as_uint(x[e]);   // the tensor core reads the top 19 bits
            }
          }
        }
      }
  };
  // issue the 4 x 3 (or 4 x 1) wgmma of ring stage `it` as one commit group
  auto issue = [&](uint32_t it, const uint32_t (&ahi)[KSTEPS][4], const uint32_t (&alo)[KSTEPS][4]) {
      const uint32_t whi = tc::smem_u32(smem + (it % STAGES) * STAGE_BYTES + A_BYTES);
      tc::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KSTEPS; ++kk) {
#pragma unroll
        for (int nh = 0; nh < BN / 128; ++nh) {
          float* d = acc + nh * 64;
          const uint32_t wb = whi + nh * 16384 + kk * 32;     // 32 bytes along K inside the 128-byte row
          if (WM == W_F16) {
            tc::wgmma_f16_rs<128, 0>(d, ahi[kk], tc::make_sw128_desc(wb));
            tc::wgmma_f16_rs<128, 0>(d, ahi[kk], tc::make_sw128_desc(wb + W_PLANE));
            tc::wgmma_f16_rs<128, 0>(d, alo[kk], tc::make_sw128_desc(wb));
          } else {
            tc::wgmma_tf32_rs<128>(d, ahi[kk], tc::make_sw128_desc(wb));
            if (NPASS == 3) {
              tc::wgmma_tf32_rs<128>(d, ahi[kk], tc::make_sw128_desc(wb + W_PLANE));
              tc::wgmma_tf32_rs<128>(d, alo[kk], tc::make_sw128_desc(wb));
            }
          }
        }
      }
      tc::wgmma_commit();
  };
  auto keep = [&](uint32_t (&ahi)[KSTEPS][4], uint32_t (&alo)[KSTEPS][4]) {
    fence_afrag(ahi);
    if (NPASS == 3) fence_afrag(alo);
  };

  // one staged round: the column groups [i0, i0 + ni) of both rows of this thread, finished in the order of the direct
  // stores (rounded products and sums, never contracted), written into staging buffer u & 1 in the TMA box's 128B
  // swizzle (16-byte chunk c of row r at c ^ (r & 7): each warp writes 8 rows x 32 B, or 8 rows x 16 B of fp16,
  // free of bank conflicts).  mode 0: fp32 pairs (+ the residual the storer loaded into the buffer); mode 1: the fp16
  // hi (plane 0) or lo (plane 1) of the pairs; mode 2: rn_tf32 (plane 0) or the tf32 remainder (plane 1).
  auto stage_round = [&](uint32_t u, int n0, int i0, int ni, int mode, int plane) {
    const uint32_t buf = tc::smem_u32(obuf + (u & 1) * 16384);
    float2 bv[8];
#pragma unroll
    for (int c = 0; c < ni; ++c) {
      const int n = n0 + 8 * (i0 + c) + 2 * tq;
      bv[c] = g.bias ? make_float2(__ldg(g.bias + n), __ldg(g.bias + n + 1)) : make_float2(0.f, 0.f);
    }
    tc::mbar_wait(ofree + (u & 1), (u >> 1) & 1);
#pragma unroll
    for (int c = 0; c < ni; ++c) {
      const int i = i0 + c;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = row0 + 8 * hh;
        float x0 = __fmul_rn(g.alpha, acc[4 * i + 2 * hh]), x1 = __fmul_rn(g.alpha, acc[4 * i + 2 * hh + 1]);
        if (g.bias) { x0 = __fadd_rn(x0, bv[c].x); x1 = __fadd_rn(x1, bv[c].y); }
        if (g.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
        if (mode == 1) {
          uint32_t hi, lo;
          split_pack_h(x0, x1, hi, lo);
          sts_u32(buf + r * 128 + ((c ^ (r & 7)) << 4) + 4 * tq, plane ? lo : hi);
        } else {
          const uint32_t p = buf + r * 128 + (((2 * c + (tq >> 1)) ^ (r & 7)) << 4) + 8 * (tq & 1);
          if (mode == 2) {
            const float h0 = tf32_hi(x0), h1 = tf32_hi(x1);
            sts_f2(p, plane ? make_float2(tf32_hi(x0 - h0), tf32_hi(x1 - h1)) : make_float2(h0, h1));
          } else {
            if (g.R) { const float2 rv = lds_f2(p); x0 = __fadd_rn(x0, rv.x); x1 = __fadd_rn(x1, rv.y); }
            sts_f2(p, make_float2(x0, x1));
          }
        }
      }
    }
    tc::fence_proxy_async();      // generic-proxy writes -> visible to the TMA store (async proxy)
    tc::mbar_arrive(ostaged + (u & 1));
  };

  uint32_t it = 0, u = 0;         // u: staged rounds so far (buffer u & 1)
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    int m0, n0, a_row, w_row, prob;
    decode(tile, m0, n0, a_row, w_row, prob);
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    // Pipelined mainloop (BN = 128), two k-blocks per trip so that each fragment set has a fixed name.  Every issue is followed by
    // wait<1> in the same branch: it retires the previous k-block (whose stage is then released and whose fragment
    // set is refilled), and the split of the next k-block runs while this one's wgmma are on the tensor cores.  The
    // wait sits before the split because the set it refills is still being read by the retiring wgmma.  The wgmma
    // sequence, and so every accumulator's sum order, is the same as issuing and retiring one k-block at a time.
    if constexpr (PIPE) {
      prep(it, ahi0, alo0);
      for (int kt = 0; kt < nk; kt += 2) {
        issue(it + kt, ahi0, alo0);
        tc::wgmma_wait<1>();
        keep(ahi1, alo1);
        if (kt > 0) tc::mbar_arrive(empty + (it + kt - 1) % STAGES);
        if (kt + 1 < nk) {
          prep(it + kt + 1, ahi1, alo1);
          issue(it + kt + 1, ahi1, alo1);
          tc::wgmma_wait<1>();
          keep(ahi0, alo0);
          tc::mbar_arrive(empty + (it + kt) % STAGES);
          if (kt + 2 < nk) prep(it + kt + 2, ahi0, alo0);
        }
      }
      tc::wgmma_wait<0>();
      tc::fence_acc<BN>(acc);
      keep(ahi0, alo0);
      keep(ahi1, alo1);
      tc::mbar_arrive(empty + (it + nk - 1) % STAGES);
    } else {                                  // 256-column tiles: 128 accumulators leave no room for a second set
      for (int kt = 0; kt < nk; ++kt) {
        prep(it + kt, ahi0, alo0);
        issue(it + kt, ahi0, alo0);
        tc::wgmma_wait<0>();
        tc::fence_acc<BN>(acc);
        keep(ahi0, alo0);
        tc::mbar_arrive(empty + (it + kt) % STAGES);
      }
    }
    it += nk;

    // ================================ epilogue ================================
    if (SCORE) {
      // rows of the coupling buffer are n+1 floats long: plain stores inside the [m, n] block
      const int p = prob / st.batch, bi = prob % st.batch;
      const int pm = st.m[p], pn = st.n[p];                     // capacities: the buffer's shape
      const int em = slot_count(st.slot, bi, st.n_views, st.a[p], pm);      // this tuple's [em, en] block
      const int en = slot_count(st.slot, bi, st.n_views, st.b[p], pn);
      float* Cp = st.scores[p] + (long long)bi * (pm + 1) * (pn + 1);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int gm = m0 + row0 + 8 * hh;
        if (gm >= em) continue;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
          const int gn = n0 + 8 * i + 2 * tq;
          if (gn < en) Cp[(long long)gm * (pn + 1) + gn] = g.alpha * acc[4 * i + 2 * hh];
          if (gn + 1 < en) Cp[(long long)gm * (pn + 1) + gn + 1] = g.alpha * acc[4 * i + 2 * hh + 1];
        }
      }
      continue;
    }
    if constexpr (STAGED) {
      const int kind = g.stage ? tile_kind(n0) : -1;
      if (kind >= 0) {
        // the storer drains each round while the next is written and, after the last, while the mainloop of the
        // next tile runs; rows >= M and columns beyond N lie outside the tensor maps and are never stored
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (kind == 1) {
            if (j < 4) stage_round(u + j, n0, 8 * (j >> 1), 8, 1, j & 1);
          } else if (kind == 2) {
            stage_round(u + j, n0, 4 * (j >> 1), 4, 2, j & 1);
          } else if (j < 4) {
            stage_round(u + j, n0, 4 * j, 4, 0, 0);
          }
        }
        u += kind == 2 ? 8 : 4;
        continue;
      }
    }
    // store the finished pair (x0, x1) of row m, columns n, n + 1 in the layout(s) the caller asked for
    auto put = [&](int m, int n, float x0, float x1) {
      if (g.VT && n >= g.vt_col0) {
        // V^T (and its tf32 lo plane) for the tf32 attention kernel
        const int slab = m / g.n_pad, ii = m % g.n_pad;
        const long long off = ((long long)slab * (g.N - g.vt_col0) + (n - g.vt_col0)) * g.n_pad + ii;
        if (g.VTLO) {
          const float h0 = tf32_hi(x0), h1 = tf32_hi(x1);
          g.VT[off] = h0; g.VT[off + g.n_pad] = h1;
          g.VTLO[off] = tf32_hi(x0 - h0); g.VTLO[off + g.n_pad] = tf32_hi(x1 - h1);
        } else {
          g.VT[off] = x0; g.VT[off + g.n_pad] = x1;
        }
      } else if (g.KH16 && n >= 256) {
        // K (columns 256..511) and V (512..767) hi / lo planes in half precision
        const bool is_v = n >= 512;
        const long long o = (long long)m * 256 + n - (is_v ? 512 : 256);
        uint32_t hi, lo;
        split_pack_h(x0, x1, hi, lo);
        *reinterpret_cast<uint32_t*>((is_v ? g.VH16 : g.KH16) + o) = hi;
        *reinterpret_cast<uint32_t*>((is_v ? g.VL16 : g.KL16) + o) = lo;
      } else if (g.KLO && n >= 256 && n < 512) {
        const float h0 = tf32_hi(x0), h1 = tf32_hi(x1);
        *reinterpret_cast<float2*>(g.C + (long long)m * g.ldc + n) = make_float2(h0, h1);
        *reinterpret_cast<float2*>(g.KLO + (long long)m * 256 + n - 256) = make_float2(tf32_hi(x0 - h0), tf32_hi(x1 - h1));
      } else {
        const long long c_row = m + (long long)prob * g.tiles_m * BM;     // split-K: slab of this K slice
        *reinterpret_cast<float2*>(g.C + c_row * g.ldc + n) = make_float2(x0, x1);
      }
    };
    if constexpr (PIPE) {
      // The bias and residual operands of ICH column groups are loaded first, all at once, so that their latencies
      // overlap instead of each standing between the stores of two elements.
      constexpr int ICH = 8;
#pragma unroll
      for (int i0 = 0; i0 < BN / 8; i0 += ICH) {
        float2 bv[ICH], rv[ICH][2];
#pragma unroll
        for (int c = 0; c < ICH; ++c) {
          const int n = n0 + 8 * (i0 + c) + 2 * tq;
          bv[c] = g.bias ? make_float2(__ldg(g.bias + n), __ldg(g.bias + n + 1)) : make_float2(0.f, 0.f);
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int m = m0 + row0 + 8 * hh;
            rv[c][hh] = g.R && m < g.M ? __ldg(reinterpret_cast<const float2*>(g.R + (long long)m * g.ldr + n))
                                       : make_float2(0.f, 0.f);
          }
        }
#pragma unroll
        for (int c = 0; c < ICH; ++c) {
          const int i = i0 + c, n = n0 + 8 * i + 2 * tq;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int m = m0 + row0 + 8 * hh;
            if (m >= g.M) continue;
            float x0 = g.alpha * acc[4 * i + 2 * hh], x1 = g.alpha * acc[4 * i + 2 * hh + 1];
            if (g.bias) { x0 += bv[c].x; x1 += bv[c].y; }
            if (g.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
            if (g.R) { x0 += rv[c][hh].x; x1 += rv[c][hh].y; }
            put(m, n, x0, x1);
          }
        }
      }
    } else {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int m = m0 + row0 + 8 * hh;
        if (m >= g.M) continue;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
          const int n = n0 + 8 * i + 2 * tq;
          float x0 = g.alpha * acc[4 * i + 2 * hh], x1 = g.alpha * acc[4 * i + 2 * hh + 1];
          if (g.bias) { x0 += __ldg(g.bias + n); x1 += __ldg(g.bias + n + 1); }
          if (g.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
          if (g.R) {
            const float2 r = __ldg(reinterpret_cast<const float2*>(g.R + (long long)m * g.ldr + n));
            x0 += r.x; x1 += r.y;
          }
          put(m, n, x0, x1);
        }
      }
    }
  }
}

template <int BN, int NPASS, int WM, bool SCORE>
int launch_wg(const CUtensorMap* tA, const CUtensorMap* tA2, const CUtensorMap* tWhi, const CUtensorMap* tWlo,
              const GArgs& g, const ScoreTab& st, long long n_tiles, bool persistent, cudaStream_t stream,
              const StoreMaps& sm) {
  using C_ = Cfg<BN, NPASS, WM>;
  if (!tA || !tA2 || !tWhi || !tWlo) return MVM_ERR_LAUNCH;
  if (n_tiles <= 0) return MVM_OK;
  // cheap and idempotent: set on every launch (per-device attribute)
  if (cudaFuncSetAttribute(gemm_wg_kernel<BN, NPASS, WM, SCORE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           C_::SMEM_BYTES) != cudaSuccess)
    return MVM_ERR_LAUNCH;
  const int n_sm = mvm_dev_info().n_sm;
  const int grid = (persistent && n_tiles > n_sm) ? n_sm : (int)n_tiles;
  gemm_wg_kernel<BN, NPASS, WM, SCORE><<<grid, NTHREADS, C_::SMEM_BYTES, stream>>>(*tA, *tA2, *tWhi, *tWlo, g, st, sm);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

StoreMaps no_store_maps() {
  StoreMaps none;
  memset(&none, 0, sizeof(none));
  return none;
}

GArgs make_args(const GemmDesc& d, float* VT, int vt_col0, int n_pad, float* KLO, float* VTLO, int bn) {
  GArgs g;
  memset(&g, 0, sizeof(g));
  g.bias = d.bias; g.R = d.R; g.ldr = d.ldr; g.C = d.C; g.ldc = d.ldc; g.M = d.M; g.N = d.N; g.K = d.K;
  g.K1 = d.K1; g.alpha = d.alpha; g.relu = d.relu; g.VT = VT; g.vt_col0 = vt_col0; g.n_pad = n_pad;
  g.KLO = KLO; g.VTLO = VTLO;
  g.tiles_m = mvm_div_up(d.M, BM); g.tiles_n = d.N / bn; g.ksplit = 1;
  return g;
}

ScoreTab no_scores() {
  ScoreTab none;
  memset(&none, 0, sizeof(none));
  return none;
}

template <int BN, int NPASS, int WM>
int launch_cfg(const GemmDesc& d, float* VT, int vt_col0, int n_pad, float* KLO, float* VTLO, bool persistent,
               cudaStream_t stream) {
  const CUtensorMap* tA = mvm_get_tmap_2d(d.A, d.M, d.K1, d.lda, BM);
  const CUtensorMap* tA2 = d.A2 ? mvm_get_tmap_2d(d.A2, d.M, d.K - d.K1, d.lda2, BM) : tA;
  const CUtensorMap* tW = mvm_get_tmap_2d(WM == W_TF32 ? d.Whi : d.W, d.N, d.K, d.ldw, BN);
  const CUtensorMap* tWlo = WM == W_TF32 ? mvm_get_tmap_2d(d.Wlo, d.N, d.K, d.ldw, BN) : tW;
  const GArgs g = make_args(d, VT, vt_col0, n_pad, KLO, VTLO, BN);
  return launch_wg<BN, NPASS, WM, false>(tA, tA2, tW, tWlo, g, no_scores(), (long long)g.tiles_m * g.tiles_n, persistent,
                                         stream, no_store_maps());
}


// hi = rn_tf32(x), lo = rn_tf32(x - hi) of a whole buffer (the W-operand planes of the score GEMM)
__global__ void split_planes_kernel(const float4* __restrict__ x, float4* __restrict__ hi, float4* __restrict__ lo,
                                    long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = x[i];
    float4 h, l;
    h.x = tf32_hi(v.x); h.y = tf32_hi(v.y); h.z = tf32_hi(v.z); h.w = tf32_hi(v.w);
    l.x = tf32_hi(v.x - h.x); l.y = tf32_hi(v.y - h.y); l.z = tf32_hi(v.z - h.z); l.w = tf32_hi(v.w - h.w);
    hi[i] = h;
    lo[i] = l;
  }
}

// C[m, n] = sum_s slabs[s][m][n] (fixed order: deterministic)
__global__ void splitk_reduce_kernel(const float4* __restrict__ slabs, float* __restrict__ C, int M, int N4, int ldc, int S) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)M * N4) return;
  const int m = (int)(i / N4), n4 = (int)(i % N4);
  float4 a = slabs[i];
  for (int s = 1; s < S; ++s) {
    const float4 b = slabs[(long long)s * M * N4 + i];
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
  }
  *reinterpret_cast<float4*>(C + (long long)m * ldc + 4 * n4) = a;
}

// ---- host: tensor-map cache -------------------------------------------------------------------
typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                             const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                             CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) return nullptr;
    fn = reinterpret_cast<EncodeFn>(p);
  }
  return fn;
}
typedef std::tuple<const void*, long long, long long, long long, long long, long long, int> TmKey;
std::map<TmKey, CUtensorMap*> g_tmaps;
std::mutex g_tmap_mu;

}  // namespace

const CUtensorMap* mvm_get_tmap_3d(const float* base, long long slabs, long long rows, long long cols,
                                   long long ld_row, long long ld_slab, int box_rows) {
  std::lock_guard<std::mutex> lk(g_tmap_mu);
  TmKey key(base, slabs, rows, cols, ld_row, ld_slab, box_rows);
  auto it = g_tmaps.find(key);
  if (it != g_tmaps.end()) return it->second;
  EncodeFn enc = get_encode();
  if (!enc) return nullptr;
  CUtensorMap* tm = new CUtensorMap;
  const int rank = slabs > 0 ? 3 : 2;
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)(slabs > 0 ? slabs : 1)};
  cuuint64_t strides[2] = {(cuuint64_t)ld_row * 4, (cuuint64_t)ld_slab * 4};
  cuuint32_t box[3] = {32, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, const_cast<float*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[mvm_b200] cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld\n", (int)r, rows, cols, ld_row);
    delete tm;
    return nullptr;
  }
  g_tmaps[key] = tm;
  return tm;
}

const CUtensorMap* mvm_get_tmap_2d(const float* base, long long rows, long long cols, long long ld, int box_rows) {
  return mvm_get_tmap_3d(base, 0, rows, cols, ld, 0, box_rows);
}

// 2-D fp16 row-major [rows, cols] with row stride ld (elements), box = [box_rows, 64 cols = 128 B], 128B swizzle
const CUtensorMap* mvm_get_tmap_2d_f16(const void* base, long long rows, long long cols, long long ld, int box_rows) {
  std::lock_guard<std::mutex> lk(g_tmap_mu);
  TmKey key(base, -16, rows, cols, ld, 0, box_rows);      // slabs = -16 marks the half-precision maps
  auto it = g_tmaps.find(key);
  if (it != g_tmaps.end()) return it->second;
  EncodeFn enc = get_encode();
  if (!enc) return nullptr;
  CUtensorMap* tm = new CUtensorMap;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[mvm_b200] cuTensorMapEncodeTiled (f16) failed (%d) rows=%lld cols=%lld ld=%lld\n", (int)r, rows, cols, ld);
    delete tm;
    return nullptr;
  }
  g_tmaps[key] = tm;
  return tm;
}


int g_gemm_bn = 256;   // output tile width of the one-tile-per-CTA schedule (128 or 256), see mvm_debug_set_gemm_tile
extern "C" void mvm_debug_set_gemm_tile(int bn) { g_gemm_bn = bn == 256 ? 256 : 128; }
int g_gemm_persist = 1;   // 1: the persistent schedule with pre-split W planes serves the 3xTF32 path (default)
extern "C" void mvm_debug_set_gemm_kernel(int persistent) { g_gemm_persist = persistent ? 1 : 0; }

// GEMM on the tensor cores.  Requirements: gemm_desc_valid(d, GEMM_TC_TF32) (kernels.cuh).  n_pass: 3 = fp32-faithful
// 3xTF32, 1 = single-pass TF32.
int mvm_default_gemm_tile() { return g_gemm_bn; }
int mvm_default_gemm_persistent() { return g_gemm_persist; }

int launch_gemm_tc(const GemmDesc& d, int n_pass, float* VT, int vt_col0, int n_pad, cudaStream_t stream,
                   float* KLO, float* VTLO, int gemm_tile, int gemm_persist) {
  if (gemm_tile < 0) gemm_tile = g_gemm_bn;            // stage-level callers: the process defaults
  if (gemm_persist < 0) gemm_persist = g_gemm_persist;
  MVM_REQUIRE(gemm_desc_valid(d, GEMM_TC_TF32));
  MVM_REQUIRE(d.W || (n_pass == 3 && d.Whi && d.Wlo));
  MVM_REQUIRE(mvm_aligned(KLO, 8));
  MvmProfScope prof__(MVM_TAG_GEMM, stream);
  if (gemm_persist && n_pass == 3 && d.Whi && d.Wlo) return launch_gemm_tc_persist(d, VT, vt_col0, n_pad, KLO, VTLO, stream);
  if (gemm_tile == 256 && d.N % 256 == 0) {
    if (n_pass == 3 && d.Whi && d.Wlo) return launch_cfg<256, 3, W_TF32>(d, VT, vt_col0, n_pad, KLO, VTLO, false, stream);
    if (n_pass == 1) return launch_cfg<256, 1, W_RAW>(d, VT, vt_col0, n_pad, nullptr, nullptr, false, stream);
  }
  if (n_pass == 3 && d.Whi && d.Wlo) return launch_cfg<128, 3, W_TF32>(d, VT, vt_col0, n_pad, KLO, VTLO, false, stream);
  if (n_pass == 3) return launch_cfg<128, 3, W_RAW>(d, VT, vt_col0, n_pad, KLO, VTLO, false, stream);
  return launch_cfg<128, 1, W_RAW>(d, VT, vt_col0, n_pad, nullptr, nullptr, false, stream);
}

// Persistent schedule, 128-column tiles, W given as its tf32 planes or (fp16x3) as half-precision planes of
// wscale * W.  Requirements: gemm_desc_valid(d, GEMM_TC_F16) for the fp16 planes, which are used when given and K, K1
// are multiples of 64; otherwise gemm_desc_valid(d, GEMM_TC_TF32) and both tf32 planes.
int launch_gemm_tc_persist(const GemmDesc& d, float* VT, int vt_col0, int n_pad, float* KLO, float* VTLO,
                           cudaStream_t stream, const HalfPlanes* hp, int ksplit, float* slabs) {
  // split-K: partial products of the K slices go to slabs [ksplit, M, N] (M a multiple of the tile height), summed by
  // launch_splitk_reduce afterwards; no bias / residual / activation / concat in that mode
  MVM_REQUIRE(ksplit >= 1 && (ksplit == 1 || (slabs && d.M % BM == 0 && d.K % (32 * ksplit) == 0 && !d.Whi16 && !d.bias && !d.R && !d.A2 &&
                                               !d.relu && !VT && !KLO && !hp)));
  const bool f16 = d.Whi16 != nullptr && d.Wlo16 != nullptr && d.K % 64 == 0 && d.K1 % 64 == 0 && d.wscale > 0.f;
  MVM_REQUIRE(f16 ? gemm_desc_valid(d, GEMM_TC_F16) : gemm_desc_valid(d, GEMM_TC_TF32) && d.Whi && d.Wlo);
  MVM_REQUIRE(mvm_aligned(KLO, 8) && mvm_aligned(slabs, 16));
  MVM_REQUIRE(!hp || (mvm_aligned(hp->kh, 4) && mvm_aligned(hp->kl, 4) && mvm_aligned(hp->vh, 4) && mvm_aligned(hp->vl, 4)));
  const CUtensorMap* tA = mvm_get_tmap_2d(d.A, d.M, d.K1, d.lda, BM);
  const CUtensorMap* tA2 = d.A2 ? mvm_get_tmap_2d(d.A2, d.M, d.K - d.K1, d.lda2, BM) : tA;
  GArgs g = make_args(d, VT, vt_col0, n_pad, KLO, VTLO, 128);
  if (ksplit > 1) { g.C = slabs; g.ldc = d.N; }
  g.ksplit = ksplit;
  if (hp) {
    g.KH16 = (__half*)hp->kh; g.KL16 = (__half*)hp->kl; g.VH16 = (__half*)hp->vh; g.VL16 = (__half*)hp->vl;
  }
  const long long n_tiles = (long long)g.tiles_m * g.tiles_n * ksplit;
  // Output tiles leave by TMA stores when every buffer they touch can be a TMA base (16-byte aligned; gemm_desc_valid
  // also accepts an 8-byte aligned C and R, which keep the direct stores), and a residual only with a plain fp32 C.
  StoreMaps sm = no_store_maps();
  const void* planes[4] = {g.KH16, g.KL16, g.VH16, g.VL16};
  bool stage = mvm_aligned(g.C, 16) && mvm_aligned(g.R, 16) && mvm_aligned(g.KLO, 16) && (!g.VT || g.vt_col0 % 128 == 0) &&
               (!g.R || (!g.KH16 && !g.KLO && !g.VT));
  for (const void* p : planes) stage = stage && mvm_aligned(p, 16);
  if (stage) {
    const CUtensorMap* c = mvm_get_tmap_2d(g.C, (long long)(ksplit - 1) * g.tiles_m * BM + g.M, g.N, g.ldc, BM);
    const CUtensorMap* r = g.R ? mvm_get_tmap_2d(g.R, g.M, g.N, g.ldr, BM) : c;
    if (!c || !r) return MVM_ERR_LAUNCH;
    sm.c = *c; sm.r = *r;
    for (int i = 0; i < 4; ++i) {
      const CUtensorMap* p = g.KH16 ? mvm_get_tmap_2d_f16(planes[i], g.M, 256, 256, BM)
                                    : g.KLO && i == 0 ? mvm_get_tmap_2d(g.KLO, g.M, 256, 256, BM) : c;
      if (!p) return MVM_ERR_LAUNCH;
      sm.p[i] = *p;
    }
    g.stage = 1;
  }
  if (f16) {
    g.alpha = d.alpha / d.wscale;
    const CUtensorMap* tWhi = mvm_get_tmap_2d_f16(d.Whi16, d.N, d.K, d.ldw, 128);
    const CUtensorMap* tWlo = mvm_get_tmap_2d_f16(d.Wlo16, d.N, d.K, d.ldw, 128);
    return launch_wg<128, 3, W_F16, false>(tA, tA2, tWhi, tWlo, g, no_scores(), n_tiles, true, stream, sm);
  }
  const CUtensorMap* tWhi = mvm_get_tmap_2d(d.Whi, d.N, d.K, d.ldw, 128);
  const CUtensorMap* tWlo = mvm_get_tmap_2d(d.Wlo, d.N, d.K, d.ldw, 128);
  return launch_wg<128, 3, W_TF32, false>(tA, tA2, tWhi, tWlo, g, no_scores(), n_tiles, true, stream, sm);
}

int launch_splitk_reduce(const float* slabs, float* C, int M, int N, int ldc, int ksplit, cudaStream_t stream) {
  MVM_REQUIRE(N % 4 == 0 && ldc % 4 == 0 && mvm_aligned(slabs, 16) && mvm_aligned(C, 16));
  const long long n = (long long)M * (N / 4);
  splitk_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(slabs), C, M, N / 4, ldc, ksplit);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

// All (pair, tuple) score matrices on the tensor cores (3xTF32).  mdesc [rows_total, 256] point-major; hi / lo:
// scratch planes of the same size (filled here).
int launch_score_gemm_tc(const float* mdesc, float* hi, float* lo, int n_pad, const PairTable& tab, int batch,
                         float alpha, cudaStream_t stream) {
  MvmProfScope prof__(MVM_TAG_SCORE, stream);
  const int n_sm = mvm_dev_info().n_sm;
  const long long rows = (long long)batch * tab.n_views * n_pad;
  split_planes_kernel<<<n_sm * 4, 256, 0, stream>>>(reinterpret_cast<const float4*>(mdesc), reinterpret_cast<float4*>(hi),
                                                    reinterpret_cast<float4*>(lo), rows * 256 / 4);
  MVM_CHECK_LAUNCH();
  const CUtensorMap* tA = mvm_get_tmap_2d(mdesc, rows, 256, 256, BM);
  const CUtensorMap* tWhi = mvm_get_tmap_2d(hi, rows, 256, 256, 128);
  const CUtensorMap* tWlo = mvm_get_tmap_2d(lo, rows, 256, 256, 128);
  ScoreTab st = no_scores();
  st.slot = tab.slot;
  st.n_pairs = tab.n_pairs; st.batch = batch; st.n_views = tab.n_views; st.n_pad = n_pad;
  int max_m = 0, max_n = 0;
  for (int p = 0; p < tab.n_pairs; ++p) {
    st.a[p] = tab.a[p]; st.b[p] = tab.b[p]; st.m[p] = tab.m[p]; st.n[p] = tab.n[p]; st.scores[p] = tab.scores[p];
    max_m = tab.m[p] > max_m ? tab.m[p] : max_m;
    max_n = tab.n[p] > max_n ? tab.n[p] : max_n;
  }
  GArgs g;
  memset(&g, 0, sizeof(g));
  g.K = 256; g.K1 = 256; g.alpha = alpha; g.ksplit = 1;
  g.tiles_m = mvm_div_up(max_m, BM); g.tiles_n = mvm_div_up(max_n, 128);
  const long long n_tiles = (long long)g.tiles_m * g.tiles_n * tab.n_pairs * batch;
  return launch_wg<128, 3, W_TF32, true>(tA, tA, tWhi, tWlo, g, st, n_tiles, true, stream, no_store_maps());
}
