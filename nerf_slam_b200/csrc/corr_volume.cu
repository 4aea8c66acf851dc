// A2 — all-pairs correlation volume + 4-level pyramid in ONE pass.
//
// Replaces CorrBlock.__init__/CorrBlock.corr (reference networks/modules/corr.py:23-38,63-72):
//   corr = (f1/4)^T (f2/4)  [fp16 out, fp32 accumulate]  followed by 3x F.avg_pool2d(2,2) over the
//   TARGET dims, each level rounded to fp16 and pooled from the previous fp16 level.
//
// The reference runs a cuBLAS HGEMM that writes level 0 (61 MB/edge at 640x480), then three
// pooling kernels that each re-read the previous level, and `CorrBlock.cat` re-copies the whole
// pool on every add.  The op is HBM-write bound (AI ~93 FLOP/B, SURVEY.md §8d: 63.6 MB/edge).
//
// Design: per CTA one (edge, 128-source-pixel) strip.  A (128 px x C=128, fp16) is loaded once
// by TMA; the CTA then walks the target image in 8x16-pixel tiles: TMA brings the 128x128 B tile
// (box {64c,16w,8h}, SWIZZLE_128B, OOB rows zero-filled) through a 2-stage mbarrier ring.  Two
// warpgroups take alternate tiles (one computes while the other stores): each issues 2 x 8 wgmma
// (M64 N128 K16, fp32 accumulators in registers), passes the accumulators through a 32-column fp32
// shared tile so that thread = source pixel, scales by 1/16, rounds to fp16 and
// builds pyramid levels 1..3 from the SAME registers (an 8x16 target tile contains complete
// 2x2/4x4/8x8 pooling cells; the fp16 rounding chain of the reference is reproduced), stage the
// four tiles in shared memory and write every level once: levels 0/1 with one TMA store per tile
// ({16,8,128} box straight from the staging buffer), levels 2/3 with cooperative stores.
// HBM traffic = algorithmic: features in once (L2 resident), each volume byte written once.
#include "common.cuh"
#include "tc.cuh"

namespace nslam {

constexpr int CV_STAGES = 2;
constexpr int CV_THREADS = 288;            // 2 warpgroups (MMA + epilogue), TMA warp
constexpr int CV_SCR_LD = 40;              // fp32 accumulator chunk [128][32 + 8 padding]
constexpr int CV_TH = 8, CV_TW = 16;       // target tile
constexpr int CV_L0_STRIDE = 256;          // bytes per staged row: dense [8][16] halfs = the TMA store box
constexpr int CV_L1_STRIDE = 64;           // dense [4][8]
constexpr int CV_L2_STRIDE = 16;
constexpr int CV_L3_STRIDE = 4;
constexpr int CV_STAGE_BYTES = 128 * (CV_L0_STRIDE + CV_L1_STRIDE + CV_L2_STRIDE + CV_L3_STRIDE);

struct CvSmem {
  // offsets in bytes from the 1024-aligned base
  static constexpr int A = 0;                          // 2 x 16384
  static constexpr int B = 32768;                      // STAGES x 2 x 16384
  static constexpr int ST = B + CV_STAGES * 32768;     // 2 epilogue groups x staging (L0|L1|L2|L3)
  static constexpr int L0 = 0;
  static constexpr int L1 = L0 + 128 * CV_L0_STRIDE;
  static constexpr int L2 = L1 + 128 * CV_L1_STRIDE;
  static constexpr int L3 = L2 + 128 * CV_L2_STRIDE;
  static constexpr int SCR = ST + 2 * CV_STAGE_BYTES;  // 2 warpgroups x [128][CV_SCR_LD] fp32
  static constexpr int BAR = SCR + 2 * 128 * CV_SCR_LD * 4;  // mbarriers
  static constexpr int TOTAL = BAR + 128;
  static_assert(TOTAL + 1024 <= 227 * 1024, "shared memory plan");
};

struct CvParams {
  __half* out[4];
  const int* ii;   // [E] frame index of fmap1
  const int* jj;   // [E] frame index of fmap2
  int HW, H2, W2;
  int NH, NW;      // target tiles
  int MT;          // 128-pixel source strips per edge
  int nwork;       // E * MT * split work items, walked persistently
  int split;       // target-tile chunks per (edge, strip): keeps all SMs busy when E * MT < #SMs
  int tma_l0, tma_l1;  // levels 0/1 stored by TMA (their row pitch is a multiple of 16 bytes)
};

__device__ __forceinline__ void cv_tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(m),
               "r"(tc::smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}

__device__ __forceinline__ float h2f(__half h) { return __half2float(h); }

// store one pyramid level's staged tile to global memory.
//   PX: pixels per contiguous segment (16>>l), TH: tile rows (8>>l)
template <int PX, int TH>
__device__ __forceinline__ void cv_store_level(const unsigned char* stage, int row_stride,
                                               __half* __restrict__ out, int e, int HW, int m0,
                                               int Hl, int Wl, int h0l, int w0l, int tid) {
  constexpr int SEG_BYTES = PX * 2;
  const bool vec = (Wl % PX) == 0;
  if (vec) {
    // one item = one (row, hh) segment, possibly split in 16-byte pieces
    constexpr int PIECES = SEG_BYTES >= 16 ? SEG_BYTES / 16 : 1;
    constexpr int PB = SEG_BYTES >= 16 ? 16 : SEG_BYTES;  // bytes per piece: 16, 8 or 4
    const int nitems = 128 * TH * PIECES;
    for (int id = tid; id < nitems; id += 128) {
      const int row = id / (TH * PIECES);
      const int rem = id % (TH * PIECES);
      const int hh = rem / PIECES, j = rem % PIECES;
      const int m = m0 + row, h = h0l + hh, w = w0l + j * (PB / 2);
      if (m >= HW || h >= Hl || w >= Wl) continue;
      const unsigned char* src = stage + row * row_stride + hh * SEG_BYTES + j * PB;
      __half* dst = out + (((size_t)e * HW + m) * Hl + h) * (size_t)Wl + w;
      if (PB == 16) *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
      else if (PB == 8) *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(src);
      else *reinterpret_cast<uint32_t*>(dst) = *reinterpret_cast<const uint32_t*>(src);
    }
  } else {
    const int nitems = 128 * TH * PX;
    for (int id = tid; id < nitems; id += 128) {
      const int row = id / (TH * PX);
      const int rem = id % (TH * PX);
      const int hh = rem / PX, ww = rem % PX;
      const int m = m0 + row, h = h0l + hh, w = w0l + ww;
      if (m >= HW || h >= Hl || w >= Wl) continue;
      const __half* src =
          reinterpret_cast<const __half*>(stage + row * row_stride + hh * SEG_BYTES) + ww;
      out[(((size_t)e * HW + m) * Hl + h) * (size_t)Wl + w] = *src;
    }
  }
}

// Persistent kernel: grid = min(#SMs, nwork).  Work item = (edge, 128-source-pixel strip); the
// B-tile ring and the two warpgroups run across work items without draining (global tile counter t:
// ring slot = t % STAGES, warpgroup = t & 1).
__global__ void __launch_bounds__(CV_THREADS, 1)
corr_volume_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const __grid_constant__ CUtensorMap tmO0, const __grid_constant__ CUtensorMap tmO1, CvParams p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sm = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + CvSmem::BAR);
  uint64_t* full_b = bars;                    // [STAGES]
  uint64_t* empty_b = bars + CV_STAGES;       // [STAGES]
  uint64_t* a_full = bars + 2 * CV_STAGES;    // [1]
  uint64_t* a_empty = a_full + 1;             // [1]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int NT = p.NH * p.NW;

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tmA);
    tc::tma_prefetch_desc(&tmB);
    for (int s = 0; s < CV_STAGES; s++) { tc::mbar_init(&full_b[s], 1); tc::mbar_init(&empty_b[s], 4); }
    tc::mbar_init(a_full, 1);
    tc::mbar_init(a_empty, 8);                // every warp of both warpgroups, once per strip
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      uint32_t t = 0, wi = 0;
      for (int w = blockIdx.x; w < p.nwork; w += gridDim.x, wi++) {
        const int ws = w / p.split, ck = w % p.split;
        const int e = ws / p.MT, m0 = (ws % p.MT) * 128;
        const int n_lo = ck * NT / p.split, n_hi = (ck + 1) * NT / p.split;
        const int fi = p.ii[e], fj = p.jj[e];
        tc::mbar_wait(a_empty, (wi & 1) ^ 1);          // MMAs of the previous strip are done with A
        tc::mbar_arrive_expect_tx(a_full, 32768);
        tc::tma_load_3d(sm + CvSmem::A, &tmA, a_full, 0, m0, fi);
        tc::tma_load_3d(sm + CvSmem::A + 16384, &tmA, a_full, 64, m0, fi);
        for (int n = n_lo; n < n_hi; n++, t++) {
          const int s = t % CV_STAGES, ph = (t / CV_STAGES) & 1;
          tc::mbar_wait(&empty_b[s], ph ^ 1);
          const int h0 = (n / p.NW) * CV_TH, w0 = (n % p.NW) * CV_TW;
          unsigned char* dst = sm + CvSmem::B + s * 32768;
          tc::mbar_arrive_expect_tx(&full_b[s], 32768);
          tc::tma_load_4d(dst, &tmB, &full_b[s], 0, w0, h0, fj);
          tc::tma_load_4d(dst + 16384, &tmB, &full_b[s], 64, w0, h0, fj);
        }
      }
    }
  } else {
    // ===================== 2 warpgroups: MMA + epilogue, thread <-> accumulator row =====================
    const int grp = warp >> 2;            // warpgroup g serves tiles with (t & 1) == g
    const int etid = threadIdx.x & 127;
    const int row = etid;                 // row inside the 128-row strip
    unsigned char* stg = sm + CvSmem::ST + grp * CV_STAGE_BYTES;
    unsigned char* st0 = stg + CvSmem::L0 + row * CV_L0_STRIDE;
    unsigned char* st1 = stg + CvSmem::L1 + row * CV_L1_STRIDE;
    unsigned char* st2 = stg + CvSmem::L2 + row * CV_L2_STRIDE;
    unsigned char* st3 = stg + CvSmem::L3 + row * CV_L3_STRIDE;
    float* scr = reinterpret_cast<float*>(sm + CvSmem::SCR) + grp * 128 * CV_SCR_LD;
    const uint32_t a_addr = tc::smem_u32(sm + CvSmem::A);
    uint32_t t = 0, wi = 0;
    for (int w = blockIdx.x; w < p.nwork; w += gridDim.x, wi++) {
      const int ws = w / p.split, ck = w % p.split;
      const int e = ws / p.MT, m0 = (ws % p.MT) * 128;
      const int n_lo = ck * NT / p.split, n_hi = (ck + 1) * NT / p.split;
      tc::mbar_wait(a_full, wi & 1);
      for (int n = n_lo; n < n_hi; n++, t++) {
        if ((int)(t & 1) != grp) continue;
        const int s = t % CV_STAGES, ph = (t / CV_STAGES) & 1;
        tc::mbar_wait(&full_b[s], ph);
        float acc[2][64];
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
          for (int i = 0; i < 64; i++) acc[h][i] = 0.f;
        const uint32_t b_addr = tc::smem_u32(sm + CvSmem::B + s * 32768);
        tc::wgmma_fence();
#pragma unroll
        for (int kh = 0; kh < 2; kh++) {
#pragma unroll
          for (int k = 0; k < 4; k++) {
            const uint64_t bd = tc::desc_sw128(b_addr + kh * 16384 + k * 32);
#pragma unroll
            for (int h = 0; h < 2; h++)
              tc::wgmma_f16<128>(acc[h], tc::desc_sw128(a_addr + kh * 16384 + h * 8192 + k * 32), bd, (kh | k) ? 1u : 0u);
          }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::acc_fence(acc[0]);
        tc::acc_fence(acc[1]);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&empty_b[s]);     // B stage free for the next TMA load
        // this group's staging buffers are free once its previous tile's stores have read them
        if (etid == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        if (grp == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
        else asm volatile("bar.sync 3, 128;" ::: "memory");
        __half l1[4][8];
#pragma unroll
        for (int c = 0; c < 4; c++) {
          uint32_t r[32];
          // accumulator columns 32c .. 32c+31 (target rows 2c, 2c+1 of the tile) of every strip row
          if (c > 0) tc::named_sync(5 + grp, 128);
          tc::acc_to_smem<128>(scr, CV_SCR_LD, 0, 0, acc[0], etid, 4 * c, 4 * c + 4);
          tc::acc_to_smem<128>(scr, CV_SCR_LD, 64, 0, acc[1], etid, 4 * c, 4 * c + 4);
          tc::named_sync(5 + grp, 128);
          tc::smem_row_ld<32>(scr, CV_SCR_LD, row, 0, r);
          __half h[32];
#pragma unroll
          for (int i = 0; i < 32; i++) h[i] = __float2half_rn(__uint_as_float(r[i]) * 0.0625f);
          // level 0: rows 2c, 2c+1 of the tile (16 px each)
          uint4* d0 = reinterpret_cast<uint4*>(st0 + c * 64);
          const uint4* hs = reinterpret_cast<const uint4*>(h);
          d0[0] = hs[0]; d0[1] = hs[1]; d0[2] = hs[2]; d0[3] = hs[3];
          // level 1: 2x2 means, summation order (h0,w0),(h0,w1),(h1,w0),(h1,w1) like avg_pool2d
#pragma unroll
          for (int wp = 0; wp < 8; wp++) {
            const float s = ((h2f(h[2 * wp]) + h2f(h[2 * wp + 1])) + h2f(h[16 + 2 * wp])) +
                            h2f(h[16 + 2 * wp + 1]);
            l1[c][wp] = __float2half_rn(s * 0.25f);
          }
          *reinterpret_cast<uint4*>(st1 + c * 16) = *reinterpret_cast<const uint4*>(l1[c]);
        }
        tc::named_sync(5 + grp, 128);                      // chunk tile free for the next tile of this group
        __half l2[2][4];
#pragma unroll
        for (int c2 = 0; c2 < 2; c2++) {
#pragma unroll
          for (int wq = 0; wq < 4; wq++) {
            const float s = ((h2f(l1[2 * c2][2 * wq]) + h2f(l1[2 * c2][2 * wq + 1])) +
                             h2f(l1[2 * c2 + 1][2 * wq])) + h2f(l1[2 * c2 + 1][2 * wq + 1]);
            l2[c2][wq] = __float2half_rn(s * 0.25f);
          }
        }
        *reinterpret_cast<uint4*>(st2) = *reinterpret_cast<const uint4*>(l2);
        __half l3[2];
#pragma unroll
        for (int wr = 0; wr < 2; wr++) {
          const float s = ((h2f(l2[0][2 * wr]) + h2f(l2[0][2 * wr + 1])) + h2f(l2[1][2 * wr])) +
                          h2f(l2[1][2 * wr + 1]);
          l3[wr] = __float2half_rn(s * 0.25f);
        }
        *reinterpret_cast<uint32_t*>(st3) = *reinterpret_cast<const uint32_t*>(l3);
        tc::fence_proxy_async();
        if (grp == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
        else asm volatile("bar.sync 4, 128;" ::: "memory");
        // levels 0 and 1 (94 % of the bytes): one TMA store each (the box clips partial tiles);
        // the two small levels (and odd row pitches) by cooperative stores
        const int h0 = (n / p.NW) * CV_TH, w0 = (n % p.NW) * CV_TW;
        if (etid == 0) {
          if (p.tma_l0) cv_tma_store_4d(&tmO0, stg + CvSmem::L0, w0, h0, m0, e);
          if (p.tma_l1) cv_tma_store_4d(&tmO1, stg + CvSmem::L1, w0 >> 1, h0 >> 1, m0, e);
          asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        if (!p.tma_l0)
          cv_store_level<16, 8>(stg + CvSmem::L0, CV_L0_STRIDE, p.out[0], e, p.HW, m0, p.H2, p.W2, h0,
                                w0, etid);
        if (!p.tma_l1)
          cv_store_level<8, 4>(stg + CvSmem::L1, CV_L1_STRIDE, p.out[1], e, p.HW, m0, p.H2 >> 1,
                               p.W2 >> 1, h0 >> 1, w0 >> 1, etid);
        cv_store_level<4, 2>(stg + CvSmem::L2, CV_L2_STRIDE, p.out[2], e, p.HW, m0, p.H2 >> 2,
                             p.W2 >> 2, h0 >> 2, w0 >> 2, etid);
        cv_store_level<2, 1>(stg + CvSmem::L3, CV_L3_STRIDE, p.out[3], e, p.HW, m0, p.H2 >> 3,
                             p.W2 >> 3, h0 >> 3, w0 >> 3, etid);
      }
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(a_empty);             // this warp's MMAs of the strip are complete
    }
    if (etid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

// ------------------------------------------------------------------------------------------
// Plain SIMT statement of the same op (test cross-check of the tensor-core path and the path
// for C % 64 != 0).  level 0: one thread per output element; levels 1..3 pool the previous level.
__global__ void corr_volume_simt_l0_kernel(const __half* __restrict__ fmaps, const int* ii,
                                           const int* jj, __half* __restrict__ out, int HW, int C) {
  const int e = blockIdx.z;
  const int m = blockIdx.y;
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= HW) return;
  const __half* a = fmaps + ((size_t)ii[e] * HW + m) * C;
  const __half* b = fmaps + ((size_t)jj[e] * HW + n) * C;
  float s = 0.f;
  for (int c = 0; c < C; c++) s += __half2float(a[c]) * __half2float(b[c]);
  out[((size_t)e * HW + m) * HW + n] = __float2half_rn(s * 0.0625f);
}
__global__ void corr_volume_pool_kernel(const __half* __restrict__ in, __half* __restrict__ out,
                                        size_t planes, int Hi, int Wi) {
  const int Ho = Hi >> 1, Wo = Wi >> 1;
  const size_t total = planes * Ho * Wo;
  for (size_t id = blockIdx.x * (size_t)blockDim.x + threadIdx.x; id < total;
       id += (size_t)gridDim.x * blockDim.x) {
    const size_t pl = id / (Ho * Wo);
    const int r = (int)(id % (Ho * Wo));
    const int y = r / Wo, x = r % Wo;
    const __half* s = in + pl * Hi * Wi + (size_t)(2 * y) * Wi + 2 * x;
    const float v = ((h2f(s[0]) + h2f(s[1])) + h2f(s[Wi])) + h2f(s[Wi + 1]);
    out[id] = __float2half_rn(v * 0.25f);
  }
}

}  // namespace nslam

extern "C" {

// fmaps: [NF, H, W, C] fp16 channels-last; ii/jj: [E] int32 frame indices (device);
// out[l]: [E, H, W, H>>l, W>>l] fp16, l = 0..3.
int nslam_corr_volume_build(const void* fmaps, int NF, int H, int W, int C, const int* ii,
                            const int* jj, int E, void* out0, void* out1, void* out2, void* out3,
                            void* stream) {
  using namespace nslam;
  if (E == 0) return 0;
  if (C != 128) return (int)cudaErrorInvalidValue;  // K = 128 = 2 swizzle atoms (DROID feature dim)
  const int HW = H * W;
  CUtensorMap tmA, tmB;
  {
    uint64_t dims[3] = {(uint64_t)C, (uint64_t)HW, (uint64_t)NF};
    uint64_t strides[2] = {(uint64_t)C * 2, (uint64_t)HW * C * 2};
    uint32_t box[3] = {64, 128, 1};
    int r = tc::make_tmap_f16(&tmA, fmaps, 3, dims, strides, box);
    if (r) return r;
  }
  {
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)NF};
    uint64_t strides[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)HW * C * 2};
    uint32_t box[4] = {64, CV_TW, CV_TH, 1};
    int r = tc::make_tmap_f16(&tmB, fmaps, 4, dims, strides, box);
    if (r) return r;
  }
  CvParams p;
  p.out[0] = (__half*)out0; p.out[1] = (__half*)out1; p.out[2] = (__half*)out2; p.out[3] = (__half*)out3;
  p.ii = ii; p.jj = jj; p.HW = HW; p.H2 = H; p.W2 = W;
  p.NH = (H + CV_TH - 1) / CV_TH; p.NW = (W + CV_TW - 1) / CV_TW;
  p.MT = (HW + 127) / 128;
  int dev0 = 0, sms0 = 132;
  cudaGetDevice(&dev0);
  cudaDeviceGetAttribute(&sms0, cudaDevAttrMultiProcessorCount, dev0);
  // few edges (the per-frame motion filter builds ONE volume): split the target tiles of a strip over
  // several CTAs so that E * MT * split >= #SMs (the A strip is re-loaded per chunk: 32 KB, L2-resident)
  p.split = (sms0 + E * p.MT - 1) / (E * p.MT);
  if (p.split > 8) p.split = 8;
  if (p.split > p.NH * p.NW) p.split = p.NH * p.NW;
  if (p.split < 1) p.split = 1;
  p.nwork = E * p.MT * p.split;
  // output tensor maps for levels 0/1: {W_l, H_l, HW, E}, box {16>>l, 8>>l, 128, 1}, no swizzle
  CUtensorMap tmO[2];
  int use_tma[2] = {0, 0};
  for (int l = 0; l < 2; l++) {
    const int Hl = H >> l, Wl = W >> l;
    if (Hl == 0 || Wl == 0 || (Wl * 2) % 16 != 0 || ((size_t)Hl * Wl * 2) % 16 != 0) { tmO[l] = tmA; continue; }
    uint64_t dims[4] = {(uint64_t)Wl, (uint64_t)Hl, (uint64_t)HW, (uint64_t)E};
    uint64_t strides[3] = {(uint64_t)Wl * 2, (uint64_t)Hl * Wl * 2, (uint64_t)HW * Hl * Wl * 2};
    uint32_t box[4] = {(uint32_t)(CV_TW >> l), (uint32_t)(CV_TH >> l), 128, 1};
    int r = tc::make_tmap_f16(&tmO[l], p.out[l], 4, dims, strides, box, false, nullptr, /*swizzle128=*/false);
    if (r) return r;
    use_tma[l] = 1;
  }
  p.tma_l0 = use_tma[0]; p.tma_l1 = use_tma[1];
  const int smem = CvSmem::TOTAL + 1024;
  static bool configured = false;
  if (!configured) {
    cudaError_t er = cudaFuncSetAttribute(corr_volume_tc_kernel,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (er != cudaSuccess) return (int)er;
    configured = true;
  }
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int grid = p.nwork < sms ? p.nwork : sms;
  corr_volume_tc_kernel<<<grid, CV_THREADS, smem, (cudaStream_t)stream>>>(tmA, tmB, tmO[0], tmO[1], p);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_corr_volume_build_simt(const void* fmaps, int NF, int H, int W, int C, const int* ii,
                                 const int* jj, int E, void* out0, void* out1, void* out2,
                                 void* out3, void* stream) {
  using namespace nslam;
  (void)NF;
  if (E == 0) return 0;
  const int HW = H * W;
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid((HW + 127) / 128, HW, E);
  corr_volume_simt_l0_kernel<<<grid, 128, 0, st>>>((const __half*)fmaps, ii, jj, (__half*)out0, HW, C);
  NSLAM_CHECK_LAUNCH();
  void* outs[4] = {out0, out1, out2, out3};
  int Hi = H, Wi = W;
  for (int l = 1; l < 4; l++) {
    const size_t planes = (size_t)E * HW;
    corr_volume_pool_kernel<<<1184, 256, 0, st>>>((const __half*)outs[l - 1], (__half*)outs[l],
                                                 planes, Hi, Wi);
    NSLAM_CHECK_LAUNCH();
    Hi >>= 1; Wi >>= 1;
  }
  return 0;
}

}  // extern "C"
