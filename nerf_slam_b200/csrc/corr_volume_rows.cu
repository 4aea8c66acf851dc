// A2 — correlation volume + pyramid with ROW-PAIR tiles (default for W in {64, 80}; bit-identical to corr_volume.cu).
//
// Same function as csrc/corr_volume.cu (reference networks/modules/corr.py:23-38,63-72).  That kernel walks the
// target image in 8x16-pixel tiles, so every source row writes its volume row in 32-byte pieces (1024 segments
// per 128x128 tile) and stalls at 32 % of the HBM peak on the store path.  Here a tile is TWO FULL TARGET ROWS
// (N = 2*W2 columns of one MMA, W2 = 80 at 640x480 -> N = 160): in the flattened [HW_src, HW_tgt] view of level 0
// a tile is a dense 128 x 160 block, i.e. 320 contiguous bytes per source row (128 segments per tile, one TMA
// store), level 1 (the 2x2 means of exactly these two rows) is 80 contiguous bytes per source row (one more TMA
// store); levels 2 and 3 are pooled in registers across 2 / 4 consecutive row pairs and written directly
// (6 % of the bytes).  The fp16 rounding chain of the reference (each level rounded, pooled from the previous
// fp16 level, summation order (h0,w0),(h0,w1),(h1,w0),(h1,w1)) is kept.
//
// Pipeline: persistent CTAs over (edge, 128-source-pixel strip, chunk of row pairs [multiple of 4]); warp 8 = TMA
// producer (A strip once per item, B = 2W2 x 128 channels per row pair, 2-stage ring), warps 0..7 = two warpgroups
// that split the columns in halves (w < W2/2 | w >= W2/2): each issues its wgmmas (M64 x N(W2/2) x K16, both target
// rows, both 64-row halves of the strip), then passes the fp32 accumulators through the B stage it has just consumed
// so that thread = source pixel, and runs the epilogue.
// Requirements: C = 128, W2 % 16 == 0, 2*W2 <= 192, H2 even.  tests/test_gpu_parity.py::test_corr_volume_rows_*.
#include "common.cuh"
#include "tc.cuh"

namespace nslam {

constexpr int CR_THREADS = 288;
constexpr int CR_STAGES = 2;      // the epilogue / store path bounds the kernel

struct CrParams {
  __half* out[4];
  const int* ii;
  const int* jj;
  const int* slots;    // output slot of edge e in the pyramid arena (NULL: e itself)
  int HW, H2, RP;      // RP = H2 / 2 row pairs
  int MT, nwork, split, rp_chunk;
};

__device__ __forceinline__ void cr_tma_store_3d(const CUtensorMap* m, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(m),
               "r"(tc::smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ float cr_h2f(__half h) { return __half2float(h); }
// 2x2 mean in the reference's order and rounding
__device__ __forceinline__ __half cr_pool(__half a, __half b, __half c, __half d) {
  return __float2half_rn((((cr_h2f(a) + cr_h2f(b)) + cr_h2f(c)) + cr_h2f(d)) * 0.25f);
}

template <int W2>
struct CrSmem {
  static constexpr int NB = 2 * W2;
  static constexpr int A = 0;                                  // 2 x 16384
  static constexpr int B = 32768;                              // STAGES x 2 x NB*128
  static constexpr int BSTAGE = 2 * NB * 128;
  // staging of levels 0 / 1, DOUBLE buffered: the TMA store of tile t reads buffer t&1 while tile t+1 is written
  static constexpr int ST0 = B + CR_STAGES * BSTAGE;           // 2 x [128][NB] halfs
  static constexpr int ST0_BYTES = 128 * NB * 2;
  static constexpr int ST1 = ST0 + 2 * ST0_BYTES;              // 2 x [128][W2/2] halfs
  static constexpr int ST1_BYTES = 128 * W2;
  static constexpr int BAR = ST1 + 2 * ST1_BYTES;
  static constexpr int TOTAL = BAR + 128;
  static_assert(TOTAL + 1024 <= 227 * 1024, "shared memory plan");
};

template <int W2>
__global__ void __launch_bounds__(CR_THREADS, 1)
corr_volume_rows_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                        const __grid_constant__ CUtensorMap tmO0, const __grid_constant__ CUtensorMap tmO1, CrParams p) {
  using SM = CrSmem<W2>;
  constexpr int NB = SM::NB, WH = W2 / 2;                      // columns per warp half and target row
  static_assert(W2 % 16 == 0 && NB <= 192, "row-pair tile");
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sm = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + SM::BAR);
  uint64_t* full_b = bars;
  uint64_t* empty_b = bars + CR_STAGES;
  uint64_t* a_full = bars + 2 * CR_STAGES;
  uint64_t* a_empty = a_full + 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tmA); tc::tma_prefetch_desc(&tmB);
    for (int s = 0; s < CR_STAGES; s++) { tc::mbar_init(&full_b[s], 1); tc::mbar_init(&empty_b[s], 8); }
    tc::mbar_init(a_full, 1); tc::mbar_init(a_empty, 8);
    tc::fence_barrier_init();
  }
  __syncthreads();

  // work item w -> (edge, strip, row-pair range)
  auto item = [&](int w, int& e, int& m0, int& rp_lo, int& rp_hi) {
    const int ws = w / p.split, ck = w % p.split;
    e = ws / p.MT; m0 = (ws % p.MT) * 128;
    rp_lo = ck * p.rp_chunk; rp_hi = min(p.RP, rp_lo + p.rp_chunk);
  };

  if (warp == 8) {
    if (lane == 0) {
      uint32_t t = 0, wi = 0;
      for (int w = blockIdx.x; w < p.nwork; w += gridDim.x, wi++) {
        int e, m0, rp_lo, rp_hi;
        item(w, e, m0, rp_lo, rp_hi);
        const int fi = p.ii[e], fj = p.jj[e];
        tc::mbar_wait(a_empty, (wi & 1) ^ 1);
        tc::mbar_arrive_expect_tx(a_full, 32768);
        tc::tma_load_3d(sm + SM::A, &tmA, a_full, 0, m0, fi);
        tc::tma_load_3d(sm + SM::A + 16384, &tmA, a_full, 64, m0, fi);
        for (int rp = rp_lo; rp < rp_hi; rp++, t++) {
          const int s = t % CR_STAGES, ph = (t / CR_STAGES) & 1;
          tc::mbar_wait(&empty_b[s], ph ^ 1);
          unsigned char* dst = sm + SM::B + s * SM::BSTAGE;
          tc::mbar_arrive_expect_tx(&full_b[s], SM::BSTAGE);
          tc::tma_load_3d(dst, &tmB, &full_b[s], 0, 2 * rp * W2, fj);
          tc::tma_load_3d(dst + NB * 128, &tmB, &full_b[s], 64, 2 * rp * W2, fj);
        }
      }
    }
  } else {
    const int hsel = warp >> 2;                  // column half = warpgroup
    const int row = threadIdx.x & 127;
    const int etid = threadIdx.x;
    const int c0 = hsel * WH;
    const int H2l = p.H2 >> 2, H3l = p.H2 >> 3;
    const uint32_t a_addr = tc::smem_u32(sm + SM::A);
    uint32_t t = 0, wi = 0;
    for (int w = blockIdx.x; w < p.nwork; w += gridDim.x, wi++) {
      int e, m0, rp_lo, rp_hi;
      item(w, e, m0, rp_lo, rp_hi);
      const int m = m0 + row;
      const bool mok = m < p.HW;
      const int eo = p.slots ? p.slots[e] : e;      // where this edge's volumes live (CorrPool slot)
      __half l1p[WH / 2], l2p[WH / 4];           // carries: level 1 of the previous (even) row pair, level 2 of the previous (even) quad
      tc::mbar_wait(a_full, wi & 1);
      for (int rp = rp_lo; rp < rp_hi; rp++, t++) {
        const int s = t % CR_STAGES, ph = (t / CR_STAGES) & 1;
        unsigned char* st0 = sm + SM::ST0 + (t & 1) * SM::ST0_BYTES + row * (NB * 2);
        unsigned char* st1 = sm + SM::ST1 + (t & 1) * SM::ST1_BYTES + row * W2;
        tc::mbar_wait(&full_b[s], ph);
        unsigned char* bst = sm + SM::B + s * SM::BSTAGE;
        const uint32_t b_addr = tc::smem_u32(bst);
        // this warpgroup's columns: target row tr, w in [c0, c0 + WH)  (B rows tr * W2 + c0 ..)
        float acc[2][2][WH / 2];
#pragma unroll
        for (int tr = 0; tr < 2; tr++)
#pragma unroll
          for (int h = 0; h < 2; h++)
#pragma unroll
            for (int i = 0; i < WH / 2; i++) acc[tr][h][i] = 0.f;
        tc::wgmma_fence();
#pragma unroll
        for (int kh = 0; kh < 2; kh++)
#pragma unroll
          for (int k = 0; k < 4; k++)
#pragma unroll
            for (int tr = 0; tr < 2; tr++) {
              const uint64_t bd = tc::desc_sw128(b_addr + kh * (NB * 128) + (tr * W2 + c0) * 128 + k * 32);
#pragma unroll
              for (int h = 0; h < 2; h++)
                tc::wgmma_f16<WH>(acc[tr][h], tc::desc_sw128(a_addr + kh * 16384 + h * 8192 + k * 32), bd, (kh | k) ? 1u : 0u);
            }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
#pragma unroll
        for (int tr = 0; tr < 2; tr++) { tc::acc_fence(acc[tr][0]); tc::acc_fence(acc[tr][1]); }
        // staging buffer t&1 is free once the store of tile t-2 has read it (at most ONE newer store group may be pending);
        // the B stage is done for both warpgroups' MMAs after this barrier and becomes the accumulator tile
        if (etid == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
        asm volatile("bar.sync 1, 256;" ::: "memory");
        float* scr = reinterpret_cast<float*>(bst) + hsel * 128 * WH;
        uint32_t ra[2][WH];
#pragma unroll
        for (int tr = 0; tr < 2; tr++) {
          if (tr) tc::named_sync(3 + hsel, 128);
          tc::acc_to_smem<WH>(scr, WH, 0, 0, acc[tr][0], row);
          tc::acc_to_smem<WH>(scr, WH, 64, 0, acc[tr][1], row);
          tc::named_sync(3 + hsel, 128);
          tc::smem_row_ld<WH>(scr, WH, row, 0, ra[tr]);
        }
        tc::fence_proxy_async();
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&empty_b[s]);          // the B stage may be refilled
        __half h0[WH], h1[WH];
#pragma unroll
        for (int tr = 0; tr < 2; tr++) {
          __half* h = tr ? h1 : h0;
#pragma unroll
          for (int i = 0; i < WH; i += 2) {
            const __half2 v = __floats2half2_rn(__uint_as_float(ra[tr][i]) * 0.0625f, __uint_as_float(ra[tr][i + 1]) * 0.0625f);
            h[i] = __low2half(v); h[i + 1] = __high2half(v);
          }
#pragma unroll
          for (int k = 0; k < WH / 8; k++)
            *reinterpret_cast<uint4*>(st0 + (tr * W2 + c0 + 8 * k) * 2) = *reinterpret_cast<const uint4*>(h + 8 * k);
        }
        // level 1: 2x2 means of the two rows of this tile
        __half l1[WH / 2];
#pragma unroll
        for (int x = 0; x < WH / 2; x++) l1[x] = cr_pool(h0[2 * x], h0[2 * x + 1], h1[2 * x], h1[2 * x + 1]);
#pragma unroll
        for (int x = 0; x < WH / 2; x += 4)
          *reinterpret_cast<uint2*>(st1 + (c0 / 2 + x) * 2) = *reinterpret_cast<const uint2*>(l1 + x);
        // level 2 (every second row pair) and level 3 (every fourth): registers -> global
        if (rp & 1) {
          __half l2[WH / 4];
#pragma unroll
          for (int y = 0; y < WH / 4; y++) l2[y] = cr_pool(l1p[2 * y], l1p[2 * y + 1], l1[2 * y], l1[2 * y + 1]);
          const int q2 = rp >> 1;
          if (mok && q2 < H2l) {
            __half* dst = p.out[2] + ((size_t)eo * p.HW + m) * ((size_t)H2l * (W2 / 4)) + (size_t)q2 * (W2 / 4) + c0 / 4;
#pragma unroll
            for (int y = 0; y < WH / 4; y += 2) *reinterpret_cast<__half2*>(dst + y) = *reinterpret_cast<const __half2*>(l2 + y);
          }
          if ((rp & 3) == 3) {
            const int q3 = rp >> 2;
            if (mok && q3 < H3l) {
              __half* dst3 = p.out[3] + ((size_t)eo * p.HW + m) * ((size_t)H3l * (W2 / 8)) + (size_t)q3 * (W2 / 8) + c0 / 8;
#pragma unroll
              for (int z = 0; z < WH / 8; z++) dst3[z] = cr_pool(l2p[2 * z], l2p[2 * z + 1], l2[2 * z], l2[2 * z + 1]);
            }
          } else {
#pragma unroll
            for (int y = 0; y < WH / 4; y++) l2p[y] = l2[y];
          }
        } else {
#pragma unroll
          for (int x = 0; x < WH / 2; x++) l1p[x] = l1[x];
        }
        // levels 0 and 1: one TMA store each, straight from the dense staging rows
        tc::fence_proxy_async();
        asm volatile("bar.sync 2, 256;" ::: "memory");
        if (etid == 0) {
          cr_tma_store_3d(&tmO0, sm + SM::ST0 + (t & 1) * SM::ST0_BYTES, 2 * rp * W2, m0, eo);
          cr_tma_store_3d(&tmO1, sm + SM::ST1 + (t & 1) * SM::ST1_BYTES, rp * (W2 / 2), m0, eo);
          asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
      }
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(a_empty);             // this warp's MMAs of the strip are complete
    }
    if (etid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

template <int W2>
static int launch_rows(const void* fmaps, int NF, int H, const int* ii, const int* jj, int E, void* const* outs,
                       cudaStream_t st, const int* slots = nullptr, int n_slots = 0) {
  using SM = CrSmem<W2>;
  const int W = W2, HW = H * W, C = 128;
  CUtensorMap tmA, tmB, tmO0, tmO1;
  {
    uint64_t dims[3] = {(uint64_t)C, (uint64_t)HW, (uint64_t)NF};
    uint64_t strides[2] = {(uint64_t)C * 2, (uint64_t)HW * C * 2};
    uint32_t boxA[3] = {64, 128, 1}, boxB[3] = {64, (uint32_t)(2 * W), 1};
    int r = tc::make_tmap_f16(&tmA, fmaps, 3, dims, strides, boxA);
    if (r) return r;
    r = tc::make_tmap_f16(&tmB, fmaps, 3, dims, strides, boxB);
    if (r) return r;
  }
  {
    const uint64_t n0 = (uint64_t)H * W, n1 = (uint64_t)(H / 2) * (W / 2);
    const uint64_t NE = slots ? (uint64_t)n_slots : (uint64_t)E;      // edges (or arena slots) along the outer dimension
    uint64_t d0[3] = {n0, (uint64_t)HW, NE}, s0[2] = {n0 * 2, (uint64_t)HW * n0 * 2};
    uint64_t d1[3] = {n1, (uint64_t)HW, NE}, s1[2] = {n1 * 2, (uint64_t)HW * n1 * 2};
    uint32_t b0[3] = {(uint32_t)(2 * W), 128, 1}, b1[3] = {(uint32_t)(W / 2), 128, 1};
    int r = tc::make_tmap_f16(&tmO0, outs[0], 3, d0, s0, b0, false, nullptr, false);
    if (r) return r;
    r = tc::make_tmap_f16(&tmO1, outs[1], 3, d1, s1, b1, false, nullptr, false);
    if (r) return r;
  }
  CrParams p;
  for (int l = 0; l < 4; l++) p.out[l] = (__half*)outs[l];
  p.ii = ii; p.jj = jj; p.slots = slots; p.HW = HW; p.H2 = H; p.RP = H / 2;
  p.MT = (HW + 127) / 128;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // chunks of row pairs (multiples of 4, so that the level-2/3 carries never cross a chunk) when E*MT < #SMs
  int split = (sms + E * p.MT - 1) / (E * p.MT);
  const int quads = (p.RP + 3) / 4;
  if (split > quads) split = quads;
  if (split < 1) split = 1;
  p.rp_chunk = ((quads + split - 1) / split) * 4;
  p.split = (p.RP + p.rp_chunk - 1) / p.rp_chunk;
  p.nwork = E * p.MT * p.split;
  const int smem = SM::TOTAL + 1024;
  if (cudaError_t e = ensure_dyn_smem<corr_volume_rows_kernel<W2>>(smem)) return (int)e;
  const int grid = p.nwork < sms ? p.nwork : sms;
  corr_volume_rows_kernel<W2><<<grid, CR_THREADS, smem, st>>>(tmA, tmB, tmO0, tmO1, p);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

}  // namespace nslam

extern "C" {

/* row-pair variant of nslam_corr_volume_build (same arguments and outputs).  Supported shapes:
 * C = 128, H even, W in {64, 80}; returns cudaErrorNotSupported otherwise (callers then use the tiled kernel). */
int nslam_corr_volume_build_rows(const void* fmaps, int NF, int H, int W, int C, const int* ii, const int* jj, int E,
                                 void* out0, void* out1, void* out2, void* out3, void* stream) {
  using namespace nslam;
  if (E == 0) return 0;
  if (C != 128 || (H & 1)) return (int)cudaErrorNotSupported;
  void* outs[4] = {out0, out1, out2, out3};
  switch (W) {
    case 80: return launch_rows<80>(fmaps, NF, H, ii, jj, E, outs, (cudaStream_t)stream);
    case 64: return launch_rows<64>(fmaps, NF, H, ii, jj, E, outs, (cudaStream_t)stream);
    default: return (int)cudaErrorNotSupported;
  }
}

/* As nslam_corr_volume_build_rows, but edge e is written into slot slots[e] of pyramid ARENAS out0..3 =
 * [n_slots,H,W,H>>l,W>>l] (CorrPool): all new edges of a keyframe in ONE launch, whatever slots they were given. */
int nslam_corr_volume_build_slots(const void* fmaps, int NF, int H, int W, int C, const int* ii, const int* jj,
                                  const int* slots, int E, int n_slots, void* out0, void* out1, void* out2, void* out3,
                                  void* stream) {
  using namespace nslam;
  if (E == 0) return 0;
  if (C != 128 || (H & 1) || slots == nullptr || n_slots <= 0) return (int)cudaErrorNotSupported;
  void* outs[4] = {out0, out1, out2, out3};
  switch (W) {
    case 80: return launch_rows<80>(fmaps, NF, H, ii, jj, E, outs, (cudaStream_t)stream, slots, n_slots);
    case 64: return launch_rows<64>(fmaps, NF, H, ii, jj, E, outs, (cudaStream_t)stream, slots, n_slots);
    default: return (int)cudaErrorNotSupported;
  }
}

}  // extern "C"
