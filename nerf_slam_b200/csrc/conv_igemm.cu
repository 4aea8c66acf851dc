// A5/A1 — convolutions of the update operator as implicit GEMM on Hopper tensor cores (wgmma, sm_90a).
//
// Replaces the cuDNN convolutions behind UpdateModule / ConvGRU / GraphAgg
// (reference networks/droid_net.py:78-150, networks/modules/gru.py:5-32) and the
// torch.cat / sigmoid / tanh / gating elementwise kernels around them.
//
//   out[n,h,w,:] = epilogue( sum_{taps, sources} A_src[n, h+dy, w+dx, :] . W[tap, src] + bias )
//
// * activations are NHWC fp16; the concatenated conv input (hidden | context | corr | flow, 448
//   channels for the GRU) is never materialised: every 64-channel K-block is fetched by TMA from
//   the SOURCE tensor it belongs to (up to 4 tensor maps);
// * one CTA tile = 8x16 output pixels (M = 128) x N output channels (N = 16..256); for tap
//   (dy,dx) the A tile is the TMA box {64c, 16w, 8h} shifted by (dx-pad, dy-pad): out-of-image
//   rows/cols are zero-filled by TMA, which IS the convolution's zero padding;
// * weights are pre-packed on the host into the exact 128B-swizzled K-major smem image, one
//   contiguous N*128-byte block per (tap, channel-block): a 1-D bulk copy lands it wgmma-ready;
// * mbarrier rings fed by a warpgroup of TMA-issuing warps; two consumer warpgroups each own half of
//   the output columns (N >= 64) and issue wgmma (2 x M64, N/2 or N/4 per pass, K16) into fp32
//   register accumulators;
// * persistent CTAs (grid = #SMs) walk the (image, tile) list;
// * epilogue (the same two warpgroups, thread = pixel): accumulators -> 32-column fp32 shared tile ->
//   +bias (+ per-image global-context vector) -> activation / GRU gating -> fp16 ->
//   swizzled smem -> TMA store (clips partial tiles).  Kernel templated on the epilogue mode.
//
// Epilogue modes:
//   0 ACT   y = act(acc + bias [+ gctx[n]])                          act: 0 none 1 relu 2 sigmoid 3 tanh
//   1 ZR    N = 256: z = sigmoid(acc[0:128]+..), r = sigmoid(acc[128:256]+..);
//           out0 = z, out1 = r * net          (ConvGRU z,r gates, gru.py:27-29)
//   2 Q     q = tanh(acc + ..); out0 = (1 - z) * net + z * q         (gru.py:29-31)
//   3 GLO   y = sigmoid(acc + bias) * net; per-tile column sums (warp transpose-reduce, one partial per warp and
//           tile, no atomics) reduced in a fixed order into gsum[n][c] (fp32) -> glo = mean (gru.py:23-25); nothing
//           is stored
//   4 ENC   encoder layers (BasicEncoder, extractor.py): y = act(acc + bias) like mode 0, plus (a) optional
//           per-(image, channel) sum / sum of squares of the fp16 outputs for the instance norm that follows
//           and (b) optional stride-2 output: the conv is evaluated at stride 1 and only even rows/columns
//           are stored and counted (a 3x3/s2 conv reads every input pixel anyway).
// Roofline: tensor pipe; FLOPs = 2 * pixels * taps * Cin * Cout.
#include "conv_common.cuh"

namespace nslam {

template <int N, int MODE, bool HALO>
__global__ void __launch_bounds__(CG_THREADS, 1)
conv_igemm_kernel(const __grid_constant__ ConvMaps maps, ConvParams p) {
  using SM = CgSmem<N, HALO>;
  constexpr int CG_STAGES = SM::STAGES;
  constexpr int AS = SM::A_STAGES, BS = SM::B_STAGES;
  constexpr int PASSES = SM::PASSES, CPP = N / PASSES;          // columns staged per pass
  constexpr int GC = (N >= 64) ? CPP / 2 : N;                   // columns per warpgroup per pass
  constexpr int MMA_WARPS = (N >= 64) ? 8 : 4;                  // N < 64: warpgroup 0 computes every column
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sm = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + SM::BAR);
  uint64_t* full_b = bars;                       // plain: one ring; HALO: the weight-block ring
  uint64_t* empty_b = bars + BS;
  uint64_t* full_a = bars + 2 * BS;              // HALO only: the shifted-tile ring
  uint64_t* empty_a = full_a + AS;
  float* sbias = reinterpret_cast<float*>(sm + SM::BIAS);
  static_assert((4 * 4 + 4) * 8 + 8 <= 256, "barrier block");

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_img = p.tiles_h * p.tiles_w;
  const int ntiles = p.B * tiles_per_img;
  const int taps = p.KH * p.KW;
  const int nkb = taps * p.cb_total;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.n_src; s++) tc::tma_prefetch_desc(&maps.src[s]);
    for (int s = 0; s < BS; s++) { tc::mbar_init(&full_b[s], HALO ? 1 : 2); tc::mbar_init(&empty_b[s], MMA_WARPS); }
    for (int s = 0; s < AS; s++) { tc::mbar_init(&full_a[s], 1); tc::mbar_init(&empty_a[s], MMA_WARPS); }
    tc::fence_barrier_init();
  }
  for (int i = threadIdx.x; i < N; i += CG_THREADS) sbias[i] = p.bias ? p.bias[i] : 0.f;
  __syncthreads();

  // warp roles: 0..7 = two warpgroups (MMA + epilogue), 8 and 9 = activation (A) producers, 10 and 11 = weight (B) producers
  const int a_part = (warp == CG_EPI_WARPS) ? 0 : (warp == CG_EPI_WARPS + 1) ? 1 : -1;
  const int w_part = (warp >= CG_EPI_WARPS + CG_A_WARPS) ? warp - (CG_EPI_WARPS + CG_A_WARPS) : -1;
  if (a_part >= 0 || w_part >= 0) {
    // ===================== TMA producers =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    // Every producer warp walks the same sequence of load units and issues those of its own parity: an A warp the
    // activation loads with (counter % CG_A_WARPS) == a_part, a W warp the weight blocks with (counter % CG_W_WARPS) ==
    // w_part.  Whole warp in the loop, elected lane issues (uniform control flow).
    const uint32_t lead = tc::elect_one() ? 1u : 0u;
    auto src_of = [&](int g, int& sidx, int& cb) { sidx = 0; cb = g; while (cb >= p.src_cb[sidx]) { cb -= p.src_cb[sidx]; sidx++; } };
    if (HALO) {
      // unit = (channel block, dx): one shifted halo tile (A ring) + the three weight blocks of its taps dy = 0..2 (B ring)
      const int units = p.cb_total * 3;
      uint32_t ia = 0, ib = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int n = tile / tiles_per_img, tt = tile % tiles_per_img;
        const int h0 = (tt / p.tiles_w) * CG_TH, w0 = (tt % p.tiles_w) * CG_TW;
        if (a_part >= 0) {
          for (int u = 0; u < units; u++, ia++) {
            if ((int)(ia % CG_A_WARPS) != a_part) continue;
            int s, cb;
            src_of(u / 3, s, cb);
            const int sa = ia % AS, pa = (ia / AS) & 1;
            tc::mbar_wait(&empty_a[sa], pa ^ 1);
            tc::mbar_arrive_expect_tx_lead(&full_a[sa], SM::A_STAGE, lead);
            tc::tma_load_4d_lead(sm + SM::A + sa * SM::A_STAGE, &maps.src[s], &full_a[sa], cb * 64, w0 + (u % 3) - 1, h0 - 1, n, lead);
          }
        } else {
          for (int u = 0; u < units; u++) {
            const int cbg = u / 3, dx = u % 3;
            for (int dy = 0; dy < 3; dy++, ib++) {
              if ((int)(ib % CG_W_WARPS) != w_part) continue;
              const int sb = ib % BS, pb = (ib / BS) & 1;
              tc::mbar_wait(&empty_b[sb], pb ^ 1);
              tc::mbar_arrive_expect_tx_lead(&full_b[sb], N * 128, lead);
              tc::bulk_copy_g2s_lead(sm + SM::B + sb * (N * 128), p.wpacked + (size_t)((dy * 3 + dx) * p.cb_total + cbg) * N * 64,
                                     N * 128, &full_b[sb], lead);
            }
          }
        }
      }
    } else {
      // unit = (tap, channel block): one activation tile and one weight block complete on the SAME barrier (init count 2:
      // one arrive.expect_tx from the A warp, one from the W warp)
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int n = tile / tiles_per_img, tt = tile % tiles_per_img;
        const int h0 = (tt / p.tiles_w) * CG_TH, w0 = (tt % p.tiles_w) * CG_TW;
        for (int tap = 0; tap < taps; tap++) {
          const int dy = tap / p.KW - p.pad, dx = tap % p.KW - p.pad;
          int cbg = 0;
          for (int s = 0; s < p.n_src; s++) {
            for (int cb = 0; cb < p.src_cb[s]; cb++, cbg++, it++) {
              const bool mine = (a_part >= 0) ? ((int)(it % CG_A_WARPS) == a_part) : ((int)(it % CG_W_WARPS) == w_part);
              if (!mine) continue;
              const int st = it % CG_STAGES, ph = (it / CG_STAGES) & 1;
              tc::mbar_wait(&empty_b[st], ph ^ 1);
              if (a_part >= 0) {
                tc::mbar_arrive_expect_tx_lead(&full_b[st], 16384, lead);
                tc::tma_load_4d_lead(sm + SM::A + st * 16384, &maps.src[s], &full_b[st], cb * 64, w0 + dx, h0 + dy, n, lead);
              } else {
                tc::mbar_arrive_expect_tx_lead(&full_b[st], N * 128, lead);
                tc::bulk_copy_g2s_lead(sm + SM::B + st * (N * 128), p.wpacked + (size_t)(tap * p.cb_total + cbg) * N * 64,
                                       N * 128, &full_b[st], lead);
              }
            }
          }
        }
      }
    }
  } else {
    // ===================== two warpgroups: MMA, then epilogue (thread = output pixel) =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int q = warp & 3;
    const int grp = warp >> 2;
    const int row = q * 32 + lane;
    const int wtid = threadIdx.x & 127;
    const int hh = row / CG_TW, ww = row % CG_TW;
    const int etid = threadIdx.x;
    const bool works = (N >= 64) || grp == 0;
    float* scr = reinterpret_cast<float*>(sm + SM::SCR) + grp * 128 * CG_SCR_LD;
    uint32_t it = 0, ia = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      // ---- MMAs: this warpgroup's columns pass * CPP + grp * GC + [0, GC) of all 128 pixels
      float acc[PASSES][2][GC / 2];
#pragma unroll
      for (int ps = 0; ps < PASSES; ps++)
#pragma unroll
        for (int hf = 0; hf < 2; hf++)
#pragma unroll
          for (int i = 0; i < GC / 2; i++) acc[ps][hf][i] = 0.f;
      const uint32_t b_col = (uint32_t)((N >= 64) ? grp * GC : 0) * 128;
      if (works) {
        if (HALO) {
          const int units = p.cb_total * 3;
          for (int u = 0; u < units; u++, ia++) {
            const int sa = ia % AS, pa = (ia / AS) & 1;
            tc::mbar_wait(&full_a[sa], pa);
            // the tile's first row; +dy * 16 rows (2048 B) selects the tap, +64 rows (8192 B) the second half
            const uint32_t a_addr = tc::smem_u32(sm + SM::A + sa * SM::A_STAGE);
            int sbs[3];
#pragma unroll
            for (int dy = 0; dy < 3; dy++, it++) {
              const int sb = it % BS, pb = (it / BS) & 1;
              sbs[dy] = sb;
              tc::mbar_wait(&full_b[sb], pb);
              const uint32_t b_addr = tc::smem_u32(sm + SM::B + sb * (N * 128)) + b_col;
              tc::wgmma_fence();
#pragma unroll
              for (int k = 0; k < 4; k++)
#pragma unroll
                for (int ps = 0; ps < PASSES; ps++) {
                  const uint64_t bd = tc::desc_sw128(b_addr + ps * CPP * 128 + k * 32);
#pragma unroll
                  for (int hf = 0; hf < 2; hf++)
                    tc::wgmma_f16<GC>(acc[ps][hf], tc::desc_sw128(a_addr + dy * 2048 + hf * 8192 + k * 32), bd,
                                      (u | dy | k) ? 1u : 0u);
                }
              tc::wgmma_commit();
            }
            tc::wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) {
#pragma unroll
              for (int dy = 0; dy < 3; dy++) tc::mbar_arrive(&empty_b[sbs[dy]]);
              tc::mbar_arrive(&empty_a[sa]);
            }
          }
        } else {
          for (int kb = 0; kb < nkb; kb++, it++) {
            const int st = it % CG_STAGES, ph = (it / CG_STAGES) & 1;
            tc::mbar_wait(&full_b[st], ph);
            const uint32_t a_addr = tc::smem_u32(sm + SM::A + st * 16384);
            const uint32_t b_addr = tc::smem_u32(sm + SM::B + st * (N * 128)) + b_col;
            tc::wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; k++)
#pragma unroll
              for (int ps = 0; ps < PASSES; ps++) {
                const uint64_t bd = tc::desc_sw128(b_addr + ps * CPP * 128 + k * 32);
#pragma unroll
                for (int hf = 0; hf < 2; hf++)
                  tc::wgmma_f16<GC>(acc[ps][hf], tc::desc_sw128(a_addr + hf * 8192 + k * 32), bd, (kb | k) ? 1u : 0u);
              }
            tc::wgmma_commit();
            tc::wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(&empty_b[st]);
          }
        }
#pragma unroll
        for (int ps = 0; ps < PASSES; ps++) { tc::acc_fence(acc[ps][0]); tc::acc_fence(acc[ps][1]); }
      }
      const int n = tile / tiles_per_img, tt = tile % tiles_per_img;
      const int h0 = (tt / p.tiles_w) * CG_TH, w0 = (tt % p.tiles_w) * CG_TW;
      const int h = h0 + hh, w = w0 + ww;
      const bool valid = (h < p.H) && (w < p.W);
      const size_t pix = ((size_t)n * p.H + h) * p.W + w;
      // mode 4 with sub == 2: only even rows/cols are kept; they are compacted to a 4x8 staging tile
      const bool kept = (MODE != 4) || (p.sub == 1) || (((hh | ww) & 1) == 0);
      const int srow = (MODE == 4 && p.sub == 2) ? (hh >> 1) * (CG_TW / 2) + (ww >> 1) : row;
      // staging buffers free again once the previous tile's TMA stores have read them
      if (MODE != 3 && etid == 0) tma_store_wait_read();
      asm volatile("bar.sync 1, 256;" ::: "memory");
      const float* g = p.gctx ? p.gctx + (size_t)n * N : nullptr;
#pragma unroll
      for (int pass = 0; pass < PASSES; pass++) {
        if (pass > 0) {
          // the staging tiles are reused: wait until the previous pass' TMA stores have read them
          if (etid == 0) tma_store_wait_read();
          asm volatile("bar.sync 1, 256;" ::: "memory");
        }
        const int cbeg = pass * CPP + ((N >= 64) ? grp * GC : 0);
        if (works) {
#pragma unroll
          for (int c0 = cbeg; c0 < cbeg + GC; c0 += 32) {
            uint32_t r[32];
            // accumulator columns c0 .. c0+31 of this warpgroup -> row of this thread
            const int j0 = (c0 - cbeg) / 8;
            tc::named_sync(5 + grp, 128);
            tc::acc_to_smem<GC>(scr, CG_SCR_LD, 0, 0, acc[pass][0], wtid, j0, j0 + 4);
            tc::acc_to_smem<GC>(scr, CG_SCR_LD, 64, 0, acc[pass][1], wtid, j0, j0 + 4);
            tc::named_sync(5 + grp, 128);
            tc::smem_row_ld<32>(scr, CG_SCR_LD, row, 0, r);
            // operand loads of the gating modes overlap the accumulator read
            uint4 an[4] = {}, az[4] = {};
            if (MODE == 1) {
              if (c0 >= 128 && valid) {
                const uint4* np = reinterpret_cast<const uint4*>(p.net + pix * 128 + (c0 - 128));
#pragma unroll
                for (int i = 0; i < 4; i++) an[i] = np[i];
              }
            } else if (MODE == 2 || MODE == 3) {
              if (valid) {
                const uint4* np = reinterpret_cast<const uint4*>(p.net + pix * 128 + c0);
#pragma unroll
                for (int i = 0; i < 4; i++) an[i] = np[i];
                if (MODE == 2) {
                  const uint4* zp = reinterpret_cast<const uint4*>(p.zbuf + pix * 128 + c0);
#pragma unroll
                  for (int i = 0; i < 4; i++) az[i] = zp[i];
                }
              }
            }
            float v[32];
            epi_chunk<MODE>(r, v, sbias, g, c0, p.act, valid, an, az);
            if (MODE == 3) {
              const float cs = warp_colsum32(v, lane);
              p.partials[((size_t)tile * 4 + q) * N + c0 + lane] = cs;     // (tile, row quarter, column)
            } else {
              // fp16, into the staging tile of this 64-channel group (tile index within the pass)
              const int t64 = (c0 - pass * CPP) / 64;
              if (kept) {
#pragma unroll
                for (int i = 0; i < 32; i += 8) {
                  if (c0 + i >= N) break;
                  __half2 h2[4];
#pragma unroll
                  for (int j = 0; j < 4; j++) h2[j] = __floats2half2_rn(v[i + 2 * j], v[i + 2 * j + 1]);
                  if (N >= 64) {
                    // 128B-swizzled staging tile (matches the SWIZZLE_128B output tensor map)
                    unsigned char* st = sm + SM::OUT + t64 * 16384 + srow * 128;
                    const int chunk = ((c0 % 64) + i) / 8;
                    *reinterpret_cast<uint4*>(st + ((chunk ^ (srow & 7)) * 16)) = *reinterpret_cast<const uint4*>(h2);
                  } else {
                    // narrow outputs: dense rows of N halfs, un-swizzled tensor map
                    unsigned char* st = sm + SM::OUT + srow * (N * 2);
                    *reinterpret_cast<uint4*>(st + (c0 + i) * 2) = *reinterpret_cast<const uint4*>(h2);
                  }
                }
              }
              if (MODE == 4 && p.stats) {
                // statistics of what the next layer will read: the fp16-rounded values of the kept, in-image pixels
                float q2[32];
                const bool cnt = kept && valid;
#pragma unroll
                for (int i = 0; i < 32; i++) {
                  const float hv = cnt ? __half2float(__float2half_rn(v[i])) : 0.f;
                  v[i] = hv; q2[i] = hv * hv;
                }
                const float cs = warp_colsum32(v, lane), cq = warp_colsum32(q2, lane);
                if (c0 + lane < N)
                  *reinterpret_cast<float2*>(p.partials + (((size_t)tile * 4 + q) * N + c0 + lane) * 2) = make_float2(cs, cq);
              }
            }
          }
        }
        if (MODE != 3) {
          tc::fence_proxy_async();
          asm volatile("bar.sync 2, 256;" ::: "memory");
          if (etid == 0) {
            if (MODE == 1) {
              // pass 0: z (columns 0..127) -> out0 ; pass 1: r * net (columns 128..255) -> out1
              tma_store_4d(&maps.out[pass], sm + SM::OUT + 0 * 16384, 0, w0, h0, n);
              tma_store_4d(&maps.out[pass], sm + SM::OUT + 1 * 16384, 64, w0, h0, n);
            } else if (MODE == 4 && p.sub == 2) {
              for (int t = 0; t < SM::NOUT64; t++)
                tma_store_4d(&maps.out[0], sm + SM::OUT + t * 16384, pass * CPP + t * 64, w0 >> 1, h0 >> 1, n);
            } else {
              for (int t = 0; t < SM::NOUT64; t++)
                tma_store_4d(&maps.out[0], sm + SM::OUT + t * 16384, pass * CPP + t * 64, w0, h0, n);
            }
            tma_store_commit();
          }
        }
      }
    }
    if (MODE != 3 && etid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

// Per-tile partial sums -> per-image sums in a FIXED order (tiles of the image in order, row quarters in order), so
// that the result does not depend on which CTA ran which tile: partials [B][T][4][N][K] -> out[b][c][k] +=
// (out row stride `ld` columns).  Block = 32 (column, k) entries x 8 tile lanes; lane l takes tiles l, l+8, ...
__global__ void __launch_bounds__(256)
conv_partials_reduce_kernel(const float* __restrict__ partials, float* __restrict__ out, int T, int N, int K, int ld) {
  __shared__ float red[8][33];
  const int b = blockIdx.y, ck = blockIdx.x * 32 + (threadIdx.x & 31), l = threadIdx.x >> 5;
  const int NK = N * K;
  float s = 0.f;
  if (ck < NK) {
    for (int t = l; t < T; t += 8) {
      const float* pt = partials + ((size_t)b * T + t) * 4 * NK + ck;
      s += ((pt[0] + pt[NK]) + pt[2 * NK]) + pt[3 * NK];
    }
  }
  red[l][threadIdx.x & 31] = s;
  __syncthreads();
  if (l == 0 && ck < NK) {
    float v = red[0][threadIdx.x];
#pragma unroll
    for (int i = 1; i < 8; i++) v += red[i][threadIdx.x];
    out[(size_t)b * ld * K + ck] += v;
  }
}

template <int N, int MODE, bool HALO>
static int launch_conv_mh(const ConvMaps& maps, const ConvParams& p, int num_sms, cudaStream_t st) {
  const int smem = CgSmem<N, HALO>::TOTAL + 1024;
  if (cudaError_t e = ensure_dyn_smem<conv_igemm_kernel<N, MODE, HALO>>(smem)) return (int)e;
  const int ntiles = p.B * p.tiles_h * p.tiles_w;
  const int grid = ntiles < num_sms ? ntiles : num_sms;
  conv_igemm_kernel<N, MODE, HALO><<<grid, CG_THREADS, smem, st>>>(maps, p);
  NSLAM_CHECK_LAUNCH();
  return 0;
}
template <int N, int MODE>
static int launch_conv_m(const ConvMaps& maps, const ConvParams& p, bool halo, int num_sms, cudaStream_t st) {
  return halo ? launch_conv_mh<N, MODE, true>(maps, p, num_sms, st) : launch_conv_mh<N, MODE, false>(maps, p, num_sms, st);
}

// only the (N, mode) pairs the update operator uses are instantiated
static int launch_conv(int N, const ConvMaps& maps, const ConvParams& p, bool halo, int num_sms, cudaStream_t st) {
  if (p.mode == 0) {
    switch (N) {
      case 16: return launch_conv_m<16, 0>(maps, p, halo, num_sms, st);
      case 32: return launch_conv_m<32, 0>(maps, p, halo, num_sms, st);
      case 64: return launch_conv_m<64, 0>(maps, p, halo, num_sms, st);
      case 128: return launch_conv_m<128, 0>(maps, p, halo, num_sms, st);
      case 256: return launch_conv_m<256, 0>(maps, p, halo, num_sms, st);
    }
  } else if (p.mode == 1 && N == 256) {
    return launch_conv_m<256, 1>(maps, p, halo, num_sms, st);
  } else if (p.mode == 2 && N == 128) {
    return launch_conv_m<128, 2>(maps, p, halo, num_sms, st);
  } else if (p.mode == 3 && N == 128) {
    return launch_conv_mh<128, 3, false>(maps, p, num_sms, st);
  } else if (p.mode == 4) {
    switch (N) {
      case 32: return launch_conv_m<32, 4>(maps, p, halo, num_sms, st);
      case 64: return launch_conv_m<64, 4>(maps, p, halo, num_sms, st);
      case 128: return launch_conv_m<128, 4>(maps, p, halo, num_sms, st);
      case 256: return launch_conv_m<256, 4>(maps, p, halo, num_sms, st);
    }
  }
  return (int)cudaErrorInvalidValue;
}

}  // namespace nslam

extern "C" {

/* NHWC fp16 convolution (stride 1) on tensor cores.
 *   srcs[i]: [B,H,W,src_channels[i]] fp16 (channels need not be multiples of 64: the tail of the
 *            last 64-block is zero-filled by TMA; the packed weights must be zero there too)
 *   wpacked: produced by nslam_conv_pack_weights; bias [N] fp32 or NULL
 *   out0 (and out1 for mode 1): [B,H,W,out_channels] fp16; N = 16,32,64,128,256 columns per launch
 *   mode/act/gctx/net/zbuf/gsum: see the epilogue modes above. */
int nslam_conv_igemm_ex(const void* const* srcs, const int* src_channels, int n_src, int B, int H, int W,
                        int KH, int KW, int pad, int N, const void* wpacked, const float* bias, int mode,
                        int act, const float* gctx, const void* net, const void* zbuf, float* gsum,
                        void* out0, int out0_channels, void* out1, float* stats, int sub, float* partials, int num_sms,
                        void* stream) {
  using namespace nslam;
  if (n_src < 1 || n_src > 4 || B <= 0) return (int)cudaErrorInvalidValue;
  ConvMaps maps;
  ConvParams p{};
  p.B = B; p.H = H; p.W = W;
  p.tiles_h = (H + CG_TH - 1) / CG_TH; p.tiles_w = (W + CG_TW - 1) / CG_TW;
  p.n_src = n_src; p.KH = KH; p.KW = KW; p.pad = pad; p.N = N; p.mode = mode; p.act = act;
  p.wpacked = (const __half*)wpacked; p.bias = bias; p.gctx = gctx; p.net = (const __half*)net;
  p.zbuf = (const __half*)zbuf; p.gsum = gsum; p.stats = stats; p.partials = partials; p.sub = (mode == 4 && sub == 2) ? 2 : 1;
  const bool reduce = (mode == 3) || (mode == 4 && stats != nullptr);
  if (reduce && partials == nullptr) return (int)cudaErrorInvalidValue;
  if (mode == 4 && sub != 1 && sub != 2) return (int)cudaErrorInvalidValue;
  // 3x3 / pad 1: column-shifted halo tiles (see CgSmem); everything else: one tile per tap
  const bool halo = (KH == 3 && KW == 3 && pad == 1 && mode != 3);
  int cbt = 0;
  for (int s = 0; s < n_src; s++) {
    const int C = src_channels[s];
    if (C % 8 != 0) return (int)cudaErrorInvalidValue;   // TMA strides must be multiples of 16 bytes
    p.src_cb[s] = (C + 63) / 64;
    cbt += p.src_cb[s];
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
    uint32_t box[4] = {64, CG_TW, (uint32_t)(halo ? CG_TH + 2 : CG_TH), 1};
    int r = tc::make_tmap_f16(&maps.src[s], srcs[s], 4, dims, strides, box);
    if (r) return r;
  }
  p.cb_total = cbt;
  if (mode != 3) {
    void* outs[2] = {out0, out1};
    const int nout = (mode == 1) ? 2 : 1;
    for (int o = 0; o < nout; o++) {
      const int C = (mode == 1) ? 128 : out0_channels;
      const int Wo = (W + p.sub - 1) / p.sub, Ho = (H + p.sub - 1) / p.sub;     // stride-2 layers store every other pixel
      uint64_t dims[4] = {(uint64_t)C, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)B};
      uint64_t strides[3] = {(uint64_t)C * 2, (uint64_t)Wo * C * 2, (uint64_t)Ho * Wo * C * 2};
      uint32_t box[4] = {(uint32_t)(C < 64 ? C : 64), (uint32_t)(CG_TW / p.sub), (uint32_t)(CG_TH / p.sub), 1};
      int r = tc::make_tmap_f16(&maps.out[o], outs[o], 4, dims, strides, box, false, nullptr, /*swizzle128=*/N >= 64);
      if (r) return r;
    }
  }
  int r = launch_conv(N, maps, p, halo, num_sms, (cudaStream_t)stream);
  if (r || !reduce) return r;
  const int K = (mode == 3) ? 1 : 2;
  const dim3 grid((N * K + 31) / 32, B);
  conv_partials_reduce_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(partials, mode == 3 ? gsum : stats,
                                                                      p.tiles_h * p.tiles_w, N, K, mode == 3 ? 128 : N);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_conv_igemm(const void* const* srcs, const int* src_channels, int n_src, int B, int H, int W,
                     int KH, int KW, int pad, int N, const void* wpacked, const float* bias, int mode,
                     int act, const float* gctx, const void* net, const void* zbuf, float* gsum,
                     void* out0, int out0_channels, void* out1, float* partials, int num_sms, void* stream) {
  return nslam_conv_igemm_ex(srcs, src_channels, n_src, B, H, W, KH, KW, pad, N, wpacked, bias, mode, act, gctx, net, zbuf,
                             gsum, out0, out0_channels, out1, nullptr, 1, partials, num_sms, stream);
}

}  // extern "C"
