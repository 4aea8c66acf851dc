// Shared pieces of the implicit-GEMM convolution kernel (conv_igemm.cu): launch parameters, shared-memory plan,
// epilogue math.
#pragma once
#include "common.cuh"
#include "tc.cuh"

namespace nslam {

constexpr int CG_EPI_WARPS = 8;                            // two warpgroups: MMA + epilogue
// Four TMA-issuing warps (one warpgroup) behind them: a single warp issues one cp.async.bulk / tensor-map load at a
// time, different warps of an SM overlap, and a 64-channel block of a 3x3 convolution is 3 boxes + 9 weight blocks.
constexpr int CG_A_WARPS = 2, CG_W_WARPS = 2;              // activation-box issuers: warps 8, 9; weight issuers: 10, 11
constexpr int CG_THREADS = 32 * (CG_EPI_WARPS + CG_A_WARPS + CG_W_WARPS);
constexpr int CG_SCR_LD = 40;                              // fp32 accumulator chunk per warpgroup: [128][32 + 8 padding]
template <int N> struct CgStages { static constexpr int value = (N >= 256) ? 3 : 4; };
constexpr int CG_TH = 8, CG_TW = 16;

struct ConvParams {
  int B, H, W;
  int tiles_h, tiles_w;
  int n_src;
  int src_cb[4];       // 64-channel blocks per source
  int cb_total;
  int KH, KW, pad;
  int N;               // output channels of this launch (multiple of 16, <= 256)
  int mode, act;
  const __half* wpacked;   // [taps*cb_total][N][64] swizzled image
  const float* bias;       // [N]
  const float* gctx;       // [B][N] or null
  const __half* net;       // [B,H,W,128] (modes 1,2,3)
  const __half* zbuf;      // [B,H,W,128] (mode 2)
  float* gsum;             // [B][128] (mode 3)
  float* stats;            // [B][N][2] per-image channel sum / sum of squares of the fp16 outputs (mode 4) or null
  int sub;                 // mode 4: 1 = store every pixel, 2 = store (and count) even rows/cols only (stride-2 conv)
  float* partials;         // modes 3 / 4 with stats: per-(tile, row quarter) column sums [B*T][4][N][1 or 2]
};

struct ConvMaps {
  CUtensorMap src[4];
  CUtensorMap out[2];
};

__device__ __forceinline__ float act_apply(float x, int act) {
  if (act == 1) return fmaxf(x, 0.f);
  if (act == 2) return 1.f / (1.f + __expf(-x));
  if (act == 3) return tanhf(x);
  return x;
}

__device__ __forceinline__ void bulk_copy_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          tc::smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(tc::smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(m),
               "r"(tc::smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

// smem: A stages | B stages | out staging [NOUT64][16384] | bias / column sums | barriers
//   plain : A stage = one 8x16-pixel tile (16 KB) per (tap, channel block), B stage = its weight block
//   HALO  : (3x3, pad 1) A stage = one COLUMN-SHIFTED copy of the tile with a 1-pixel vertical halo
//           (box {64c,16w,10h} = 20 KB, loaded once per (channel block, dx)); the three taps dy = 0,1,2 of that
//           column read it at descriptor offsets dy * 16 rows * 128 B = dy * 2048 B (swizzle-atom aligned).
//           A traffic per channel block: 3 x 20 KB instead of 9 x 16 KB.  Weight blocks have their own ring.
template <int N, bool HALO>
struct CgSmem {
  static constexpr int STAGES = CgStages<N>::value;
  static constexpr int A_STAGE = HALO ? 20480 : 16384;
  // the loops are latency-bound on the weight blocks (one 1-D bulk copy per tap and channel block, ~1.5 us
  // round trip): keep as many of them in flight as shared memory allows
  static constexpr int A_STAGES = HALO ? ((N >= 256) ? 2 : 3) : STAGES;
  static constexpr int B_STAGES = HALO ? ((N >= 256) ? 3 : (N >= 128 ? 4 : 8)) : STAGES;
  static constexpr int A = 0;
  static constexpr int B = A_STAGES * A_STAGE;
  static constexpr int OUT = B + B_STAGES * N * 128;
  static constexpr int PASSES = (N >= 256) ? 2 : 1;        // N = 256: the epilogue stages / stores 128 columns at a time
  static constexpr int NOUT64 = (N >= 64) ? (N / PASSES) / 64 : 1;    // 64-channel staging tiles
  static constexpr int BIAS = OUT + NOUT64 * 16384;
  static constexpr int SCR = BIAS + N * 4;         // bias
  static constexpr int BAR = SCR + 2 * 128 * CG_SCR_LD * 4;
  static constexpr int TOTAL = BAR + 256;
  static_assert(TOTAL + 1024 <= 227 * 1024, "shared memory plan");
};

// transpose-reduce: on entry lane l holds v[0..31] (32 columns of ITS pixel); on exit every lane
// returns the sum over the warp's 32 pixels of column `lane` (31 shuffles instead of 32 x 5)
__device__ __forceinline__ float warp_colsum32(float (&v)[32], int lane) {
#pragma unroll
  for (int off = 16, n = 32; off >= 1; off >>= 1, n >>= 1) {
    const int half = n >> 1;
    const bool up = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < half; i++) {
      const float send = up ? v[i] : v[i + half];
      const float keep = up ? v[i + half] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
  return v[0];
}

// one 32-column chunk of the epilogue: x = acc + bias (+ gctx) -> mode-specific map -> v[]
template <int MODE>
__device__ __forceinline__ void epi_chunk(const uint32_t (&r)[32], float (&v)[32], const float* __restrict__ sb,
                                          const float* __restrict__ g, int c0, int act, bool valid,
                                          const uint4 (&an)[4], const uint4 (&az)[4]) {
#pragma unroll
  for (int i = 0; i < 32; i += 4) {
    const float4 b4 = *reinterpret_cast<const float4*>(sb + c0 + i);
    float4 g4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (g) g4 = __ldg(reinterpret_cast<const float4*>(g + c0 + i));
    v[i + 0] = __uint_as_float(r[i + 0]) + b4.x + g4.x; v[i + 1] = __uint_as_float(r[i + 1]) + b4.y + g4.y;
    v[i + 2] = __uint_as_float(r[i + 2]) + b4.z + g4.z; v[i + 3] = __uint_as_float(r[i + 3]) + b4.w + g4.w;
  }
  if (MODE == 0 || MODE == 4) {
    if (act == 1) {
#pragma unroll
      for (int i = 0; i < 32; i++) v[i] = fmaxf(v[i], 0.f);
    } else if (act != 0) {
#pragma unroll
      for (int i = 0; i < 32; i++) v[i] = act_apply(v[i], act);
    }
  } else if (MODE == 1) {
    if (c0 < 128) {                       // z
#pragma unroll
      for (int i = 0; i < 32; i++) v[i] = 1.f / (1.f + __expf(-v[i]));
    } else {                              // r * net
#pragma unroll
      for (int i = 0; i < 32; i++) {
        const __half* hv = reinterpret_cast<const __half*>(&an[i >> 3]);
        v[i] = __half2float(hv[i & 7]) / (1.f + __expf(-v[i]));
      }
    }
  } else if (MODE == 2) {
#pragma unroll
    for (int i = 0; i < 32; i++) {
      const __half* hn = reinterpret_cast<const __half*>(&an[i >> 3]);
      const __half* hz = reinterpret_cast<const __half*>(&az[i >> 3]);
      const float z = __half2float(hz[i & 7]), nt = __half2float(hn[i & 7]);
      v[i] = (1.f - z) * nt + z * tanhf(v[i]);
    }
  } else {                                // MODE 3: sigmoid(acc) * net
#pragma unroll
    for (int i = 0; i < 32; i++) {
      const __half* hn = reinterpret_cast<const __half*>(&an[i >> 3]);
      v[i] = valid ? __half2float(hn[i & 7]) / (1.f + __expf(-v[i])) : 0.f;
    }
  }
}

}  // namespace nslam
