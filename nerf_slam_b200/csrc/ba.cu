// Dense bundle adjustment on one stream with zero host round-trips  (SURVEY.md §8 A7-A15).
//
// Reference pipeline (src/droid_kernels.cu): projective_transform_kernel (1 CTA / edge, 90
// accumulators + 90 serial block reductions) -> Eigen triplets on the CPU in fp64 -> accum_cuda
// x3 (CPU argsort + CSR) -> host O(P^2 deg^2) enumeration -> EEt6x6/Ev6x1 (one CTA per
// (i,j,k) triple, each re-reading 13*HW floats) -> Eigen dense -> GPU; then gtsam on the CPU.
//
// Design:
//  * work is organised by DEPTH MAP (source frame) x PIXEL TILE, grid = (T, K): everything that
//    the Schur complement needs for depth map k (C, w, Ei and every Ej row that shares k) is
//    produced by the same CTA, so E is written once and read once more (L2-hot);
//  * the 12x12 per-edge Hessian is not accumulated per pixel: only the camera-frame Gram matrix
//    G = sum w J J^T (21 unique) and g = sum w r J (6) are, and the 6x6 frame changes
//    (Ad^T of G_ij, of the body extrinsics, sign, GTSAM reorder) are applied once per edge:
//        Hii = Mi G Mi^T, Hij = Mi G Mj^T, Hjj = Mj G Mj^T, vi = Mi g, vj = Mj g
//    -> 27 instead of 90 reductions, done with warp shuffles;
//  * the Schur products for one depth map are one small SYRK X diag(Q) X^T on smem tiles;
//  * the reduced system is assembled densely on the device through a CSR of contributions
//    (deterministic order, fp64 accumulation like the reference's Eigen path), factorised by a
//    single-CTA fp64 Cholesky (n <= 168 in shared memory) and the SE3/inverse-depth updates
//    follow on the same stream.
#include "common.cuh"
#include "../../include/nslam_ba.h"

namespace nslam {

constexpr int TILE = 128;  // pixels per CTA tile (one pixel per thread); 640x480/8: 38 tiles x K maps keeps all SMs busy
constexpr int AUX = 80;    // floats per edge in edge_aux

// ------------------------------------------------------------------------------------------
// per-edge constants: relative pose, stereo flag, Mi, Mj
__global__ void ba_prep_edges_kernel(nslam_ba_graph g, const float* __restrict__ poses,
                                     const float* __restrict__ ext, float* __restrict__ aux) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= g.E) return;
  const int i = g.ii[e], j = g.jj[e];
  float t[3], q[4];
  const bool stereo = (i == j);
  if (stereo) {
    t[0] = -0.1f; t[1] = 0.f; t[2] = 0.f; q[0] = 0.f; q[1] = 0.f; q[2] = 0.f; q[3] = 1.f;
  } else {
    se3_rel(poses + 7 * i, poses + 7 * i + 3, poses + 7 * j, poses + 7 * j + 3, t, q);
  }
  float* a = aux + (size_t)e * AUX;
  a[0] = t[0]; a[1] = t[1]; a[2] = t[2]; a[3] = q[0]; a[4] = q[1]; a[5] = q[2]; a[6] = q[3];
  a[7] = stereo ? 1.f : 0.f;
  float Aij[36], Aex[36];
  se3_adjT_matrix(t, q, Aij);
  se3_adjT_matrix(ext, ext + 3, Aex);
  // Jj' = perm(-Aex Jj)       Ji' = perm(+Aex Aij Jj)      perm: [t,w] -> [w,t]
  float* Mi = a + 8;
  float* Mj = a + 44;
  for (int r = 0; r < 6; r++) {
    const int rr = (r + 3) % 6;  // output row r takes input row r+3 mod 6
    for (int c = 0; c < 6; c++) {
      float s = 0.f;
      for (int k = 0; k < 6; k++) s += Aex[rr * 6 + k] * Aij[k * 6 + c];
      Mi[r * 6 + c] = s;
      Mj[r * 6 + c] = -Aex[rr * 6 + c];
    }
  }
}

// ------------------------------------------------------------------------------------------
// A7 + A8 + depth prior (A11): grid (T, K), 256 threads, one pixel per thread.
__global__ void __launch_bounds__(TILE)
ba_linearize_kernel(nslam_ba_graph g, nslam_ba_buffers b) {
  const int k = blockIdx.y, tile = blockIdx.x;
  const int hw = b.ht * b.wd;
  const int p = tile * TILE + threadIdx.x;
  const bool act = p < hw;
  const int frame = g.kx[k];
  const int pi = frame - g.kf0;
  const bool in_window = (pi >= 0) && (pi < g.P);
  const float fx = b.intrinsics[0], fy = b.intrinsics[1], cx = b.intrinsics[2], cy = b.intrinsics[3];

  __shared__ float red[27 * (TILE / 32)];
  __shared__ float sM[AUX];

  float u = 0.f, v = 0.f, di = 0.f;
  if (act) {
    u = (float)(p % b.wd); v = (float)(p / b.wd);
    di = b.disps[(size_t)frame * hw + p];
  }
  const float X = (u - cx) / fx, Y = (v - cy) / fy;

  float C = 0.f, wacc = 0.f, Ei[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};

  const int e0 = g.src_ptr[k], e1 = g.src_ptr[k + 1];
  for (int s = e0; s < e1; s++) {
    const int e = g.src_edges[s];
    __syncthreads();
    if (threadIdx.x < AUX) sM[threadIdx.x] = b.edge_aux[(size_t)e * AUX + threadIdx.x];
    __syncthreads();
    const float* t = sM;
    const float* q = sM + 3;
    const bool stereo = sM[7] != 0.f;
    const float* Mi = sM + 8;
    const float* Mj = sM + 44;

    float acc[27];
#pragma unroll
    for (int n = 0; n < 27; n++) acc[n] = 0.f;

    if (act) {
      float Xi[4] = {X, Y, 1.0f, di}, Xj[4];
      se3_act4(t, q, Xi, Xj);
      const float x = Xj[0], y = Xj[1], Z = Xj[2], h = Xj[3];
      const bool bad = Z < NSLAM_MIN_DEPTH;
      const float d = bad ? 0.f : 1.0f / Z;
      const float d2 = d * d;
      float wu = bad ? 0.f : 0.001f * b.weights[((size_t)e * 2 + 0) * hw + p];
      float wv = bad ? 0.f : 0.001f * b.weights[((size_t)e * 2 + 1) * hw + p];
      const float ru = b.targets[((size_t)e * 2 + 0) * hw + p] - (fx * d * x + cx);
      const float rv = b.targets[((size_t)e * 2 + 1) * hw + p] - (fy * d * y + cy);
      const float Jzu = fx * (t[0] * d - t[2] * (x * d2));
      const float Jzv = fy * (t[1] * d - t[2] * (y * d2));
      C += wu * Jzu * Jzu + wv * Jzv * Jzv;
      wacc += wu * ru * Jzu + wv * rv * Jzv;
      if (stereo) { wu = 0.f; wv = 0.f; }

      float Ju[6] = {fx * (h * d), 0.f, fx * (-x * h * d2), fx * (-x * y * d2),
                     fx * (1.0f + x * x * d2), fx * (-y * d)};
      float Jv[6] = {0.f, fy * (h * d), fy * (-y * h * d2), fy * (-1.0f - y * y * d2),
                     fy * (x * y * d2), fy * (x * d)};
      int l = 0;
#pragma unroll
      for (int n = 0; n < 6; n++) {
#pragma unroll
        for (int m = 0; m <= n; m++) {
          acc[l] = wu * Ju[n] * Ju[m] + wv * Jv[n] * Jv[m];
          l++;
        }
      }
      float ec[6];
#pragma unroll
      for (int n = 0; n < 6; n++) {
        acc[21 + n] = wu * ru * Ju[n] + wv * rv * Jv[n];
        ec[n] = wu * Jzu * Ju[n] + wv * Jzv * Jv[n];
      }
      // E rows in the final (body frame, GTSAM order) coordinates
      float* Ej = b.Emat + ((size_t)(g.P + e) * 6) * hw + p;
#pragma unroll
      for (int n = 0; n < 6; n++) {
        float sj = 0.f, si = 0.f;
#pragma unroll
        for (int m = 0; m < 6; m++) {
          sj += Mj[n * 6 + m] * ec[m];
          si += Mi[n * 6 + m] * ec[m];
        }
        Ej[(size_t)n * hw] = sj;
        Ei[n] += si;
      }
    }
    // tile reduction of the 27 Gram / gradient entries: per-warp shuffle sums (27 independent chains), then 27
    // threads add the per-warp partials and write the tile's partial directly (the next iteration's barriers
    // protect `red`)
    {
      constexpr int NW = TILE / 32;
      const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
      for (int n = 0; n < 27; n++) {
        const float v = warp_sum(acc[n]);
        if (lane == 0) red[n * NW + wid] = v;
      }
      __syncthreads();
      if (threadIdx.x < 27) {
        float sred = 0.f;
#pragma unroll
        for (int w = 0; w < NW; w++) sred += red[threadIdx.x * NW + w];
        b.part[((size_t)e * b.T + tile) * 27 + threadIdx.x] = sred;
      }
    }
  }

  if (act) {
    // depth prior: alpha where a sensed inverse depth exists, eta elsewhere
    const float alpha = 0.05f;
    const float ds = b.disps_sens ? b.disps_sens[(size_t)frame * hw + p] : 0.f;
    const float m = (ds > 0.f) ? 1.f : 0.f;
    const float Ck = C + m * alpha + (1.f - m) * b.eta[(size_t)k * hw + p];
    const float wk = wacc - m * alpha * (di - ds);
    b.Q[(size_t)k * hw + p] = 1.0f / Ck;
    b.w[(size_t)k * hw + p] = wk;
    if (in_window) {
      float* Er = b.Emat + ((size_t)pi * 6) * hw + p;
#pragma unroll
      for (int n = 0; n < 6; n++) Er[(size_t)n * hw] = Ei[n];
    }
  }
}

// per-edge 6x6 blocks from the reduced Gram matrix: one warp per edge
__global__ void ba_edge_blocks_kernel(nslam_ba_graph g, nslam_ba_buffers b) {
  const int e = blockIdx.x;
  const int lane = threadIdx.x;  // 64 threads
  __shared__ float G[36], gv[6], Mi[36], Mj[36], T1[36], T2[36];
  if (lane < 27) {
    float s = 0.f;
    const float* src = b.part + (size_t)e * b.T * 27 + lane;
    for (int t = 0; t < b.T; t++) s += src[(size_t)t * 27];
    if (lane < 21) {
      // unpack lower-triangular index
      int n = 0, acc = 0;
      while (acc + n + 1 <= lane) { acc += n + 1; n++; }
      const int m = lane - acc;
      G[n * 6 + m] = s; G[m * 6 + n] = s;
    } else {
      gv[lane - 21] = s;
    }
  }
  if (lane < 36) {
    Mi[lane] = b.edge_aux[(size_t)e * AUX + 8 + lane];
    Mj[lane] = b.edge_aux[(size_t)e * AUX + 44 + lane];
  }
  __syncthreads();
  if (lane < 36) {
    const int r = lane / 6, c = lane % 6;
    float s1 = 0.f, s2 = 0.f;
    for (int k = 0; k < 6; k++) { s1 += Mi[r * 6 + k] * G[k * 6 + c]; s2 += Mj[r * 6 + k] * G[k * 6 + c]; }
    T1[lane] = s1; T2[lane] = s2;  // Mi G, Mj G
  }
  __syncthreads();
  if (lane < 36) {
    const int r = lane / 6, c = lane % 6;
    float hii = 0.f, hij = 0.f, hjj = 0.f;
    for (int k = 0; k < 6; k++) {
      hii += T1[r * 6 + k] * Mi[c * 6 + k];
      hij += T1[r * 6 + k] * Mj[c * 6 + k];
      hjj += T2[r * 6 + k] * Mj[c * 6 + k];
    }
    const size_t E36 = (size_t)g.E * 36;
    b.Hs[0 * E36 + (size_t)e * 36 + lane] = hii;
    b.Hs[1 * E36 + (size_t)e * 36 + lane] = hij;
    b.Hs[2 * E36 + (size_t)e * 36 + c * 6 + r] = hij;  // Hji = Hij^T
    b.Hs[3 * E36 + (size_t)e * 36 + lane] = hjj;
  }
  if (lane < 6) {
    float vi = 0.f, vj = 0.f;
    for (int k = 0; k < 6; k++) { vi += Mi[lane * 6 + k] * gv[k]; vj += Mj[lane * 6 + k] * gv[k]; }
    b.vs[(size_t)e * 6 + lane] = vi;
    b.vs[(size_t)g.E * 6 + (size_t)e * 6 + lane] = vj;
  }
}

// ------------------------------------------------------------------------------------------
// A9: Schur products for depth map k on one pixel tile: S_ab = sum_p Q e_a e_b^T, v_a = sum_p Q w e_a
// grid (T, K), TILE threads, dynamic smem: (6*RMAX) rows x (TILE+1) floats + 2*TILE
__global__ void __launch_bounds__(TILE)
ba_schur_kernel(nslam_ba_graph g, nslam_ba_buffers b) {
  extern __shared__ float sm[];
  const int k = blockIdx.y, tile = blockIdx.x;
  const int hw = b.ht * b.wd;
  const int r0 = g.row_ptr[k], R = g.row_ptr[k + 1] - r0;
  if (R == 0) return;
  const int LD = TILE + 1;
  float* Xs = sm;                  // [6R][LD]
  float* qs = sm + 6 * R * LD;     // [TILE]   Q
  float* qw = qs + TILE;           // [TILE]   Q*w
  const int p = tile * TILE + threadIdx.x;
  const bool act = p < hw;
  {
    const float qv = act ? b.Q[(size_t)k * hw + p] : 0.f;
    const float wv = act ? b.w[(size_t)k * hw + p] : 0.f;
    qs[threadIdx.x] = qv;
    qw[threadIdx.x] = qv * wv;
    for (int r = 0; r < R; r++) {
      const float* src = b.Emat + ((size_t)g.row_erow[r0 + r] * 6) * hw + p;
#pragma unroll
      for (int n = 0; n < 6; n++)
        Xs[(r * 6 + n) * LD + threadIdx.x] = act ? src[(size_t)n * hw] : 0.f;
    }
  }
  __syncthreads();
  const int D = 6 * R;
  const int poff = g.pair_off[k];
  // S blocks: entry (ra*R + rb)*36 + m*6 + n  <->  X row (ra*6+m), X row (rb*6+n).
  // Only the block pairs ra <= rb are computed (S_ba = S_ab^T is written from the same registers) and one
  // work item produces a whole block ROW (6 entries): 8 shared-memory loads per 6 FMAs instead of 18.
  const int npairs = R * (R + 1) / 2;
  for (int item = threadIdx.x; item < npairs * 6; item += TILE) {
    const int pr = item / 6, m = item % 6;
    int ra = 0, rem = pr;
    while (rem >= R - ra) { rem -= R - ra; ra++; }
    const int rb = ra + rem;
    const float* xa = Xs + (ra * 6 + m) * LD;
    const float* xb = Xs + (rb * 6) * LD;
    float acc6[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
    for (int t = 0; t < TILE; t++) {
      const float a = xa[t] * qs[t];
#pragma unroll
      for (int n = 0; n < 6; n++) acc6[n] = fmaf(a, xb[n * LD + t], acc6[n]);
    }
    float* dab = b.spart + ((size_t)(poff + ra * R + rb) * 36 + m * 6) * b.T + tile;
#pragma unroll
    for (int n = 0; n < 6; n++) dab[(size_t)n * b.T] = acc6[n];
    if (ra != rb) {
      float* dba = b.spart + ((size_t)(poff + rb * R + ra) * 36 + m) * b.T + tile;
#pragma unroll
      for (int n = 0; n < 6; n++) dba[(size_t)n * 6 * b.T] = acc6[n];
    }
  }
  float* vpart = b.spart + (size_t)g.NPAIR * 36 * b.T;
  for (int id = threadIdx.x; id < D; id += TILE) {
    const float* xa = Xs + id * LD;
    float s = 0.f;
#pragma unroll 8
    for (int t = 0; t < TILE; t++) s += xa[t] * qw[t];
    vpart[((size_t)r0 * 6 + id) * b.T + tile] = s;
  }
}

// sum the per-tile partials: one thread per value
__global__ void ba_schur_reduce_kernel(const float* __restrict__ spart, float* __restrict__ sblk,
                                       int nvals, int T) {
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= nvals) return;
  const float* s = spart + (size_t)id * T;
  float acc = 0.f;
  for (int t = 0; t < T; t++) acc += s[t];
  sblk[id] = acc;
}

// A10/A11: dense assembly H = A - S, v = b_A - b_S (fp64 accumulate, fp32 store)
// grid: P*P + P blocks of 36 threads
__global__ void ba_assemble_kernel(nslam_ba_graph g, nslam_ba_buffers b) {
  const int P = g.P;
  const int blk = blockIdx.x;
  const int lane = threadIdx.x;
  const float* sv = b.sblk + (size_t)g.NPAIR * 36;
  if (blk < P * P) {
    const int a = blk / P, c = blk % P;
    double s = 0.0;
    for (int q = g.hc_ptr[blk]; q < g.hc_ptr[blk + 1]; q++) {
      const int id = g.hc_idx[q];
      if (id >= 0) s += (double)b.Hs[(size_t)id * 36 + lane];
      else s -= (double)b.sblk[(size_t)(-id - 1) * 36 + lane];
    }
    const int r = lane / 6, cc = lane % 6;
    b.H[(size_t)(a * 6 + r) * (6 * P) + c * 6 + cc] = (float)s;
  } else if (lane < 6) {
    const int a = blk - P * P;
    double s = 0.0;
    for (int q = g.vc_ptr[a]; q < g.vc_ptr[a + 1]; q++) {
      const int id = g.vc_idx[q];
      if (id >= 0) s += (double)b.vs[(size_t)id * 6 + lane];
      else s -= (double)sv[(size_t)(-id - 1) * 6 + lane];
    }
    b.v[a * 6 + lane] = (float)s;
  }
}

// ------------------------------------------------------------------------------------------
// A12: single-CTA fp64 Cholesky solve.  A lives in shared memory when it fits, else in `work`.
template <bool SMEM>
__global__ void __launch_bounds__(256)
ba_solve_kernel(const float* __restrict__ Hin, const float* __restrict__ vin, int n,
                int prior_idx, const float* __restrict__ prior_err, float prior_info, float lm,
                float ep, double* __restrict__ work, float* __restrict__ dx,
                float* __restrict__ Linv, int* __restrict__ status, int* __restrict__ fail_count) {
  extern __shared__ double sA[];
  double* A = SMEM ? sA : work;
  double* y = work + (size_t)n * n;  // rhs / solution
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int id = tid; id < n * n; id += nt) {
    const int r = id / n, c = id % n;
    double a = (double)Hin[id];
    if (r == c) {
      a += (double)ep + (double)lm * a;
      if (prior_idx >= 0 && r >= prior_idx * 6 && r < prior_idx * 6 + 6) a += (double)prior_info;
    }
    A[id] = a;
  }
  for (int id = tid; id < n; id += nt) {
    double r = (double)vin[id];
    if (prior_idx >= 0 && id >= prior_idx * 6 && id < prior_idx * 6 + 6)
      r -= (double)prior_info * (double)prior_err[id - prior_idx * 6];
    y[id] = r;
  }
  __syncthreads();
  // Blocked right-looking Cholesky with the natural 6x6 pose blocks (n = 6P), lower triangle, in place:
  //   per block column: every panel thread factors the 6x6 diagonal block itself (registers; identical
  //   arithmetic in all threads -> a uniform failure test, no broadcast barrier), solves its own row of the
  //   panel against it, barrier, rank-6 trailing update with a 2-D thread mapping, barrier.
  //   P x 2 barriers instead of n x 3 and 6 FMAs per trailing element per barrier.
  __shared__ int s_fail;
  if (tid == 0) s_fail = 0;
  double* diag = y + n;                       // [n] 1 / L[j][j]
  const int tx = tid & 15, ty = tid >> 4;     // 16 x 16
  const int P = n / 6;
  __syncthreads();
  for (int jb = 0; jb < P; jb++) {
    const int j0 = 6 * jb;
    // ---- diagonal block: Ljj (lower) and the reciprocals of its diagonal, redundantly per thread
    double Lb[6][6], rd[6];
    bool bad = false;
#pragma unroll
    for (int r = 0; r < 6; r++)
#pragma unroll
      for (int c = 0; c <= r; c++) Lb[r][c] = A[(size_t)(j0 + r) * n + j0 + c];
#pragma unroll
    for (int c = 0; c < 6; c++) {
      double d = Lb[c][c];
#pragma unroll
      for (int k = 0; k < c; k++) d -= Lb[c][k] * Lb[c][k];
      if (!(d > 0.0)) bad = true;
      const double l = sqrt(d);
      rd[c] = 1.0 / l;
      Lb[c][c] = l;
#pragma unroll
      for (int r = c + 1; r < 6; r++) {
        double v = Lb[r][c];
#pragma unroll
        for (int k = 0; k < c; k++) v -= Lb[r][k] * Lb[c][k];
        Lb[r][c] = v * rd[c];
      }
    }
    if (bad) { s_fail = 1; }
    // ---- panel rows i > j0 + 5: row_i(L) = row_i(A) * Ljj^-T   (thread per row)
    for (int i = j0 + 6 + tid; i < n; i += nt) {
      double x[6];
#pragma unroll
      for (int c = 0; c < 6; c++) {
        double v = A[(size_t)i * n + j0 + c];
#pragma unroll
        for (int k = 0; k < c; k++) v -= x[k] * Lb[c][k];
        x[c] = v * rd[c];
      }
#pragma unroll
      for (int c = 0; c < 6; c++) A[(size_t)i * n + j0 + c] = x[c];
    }
    __syncthreads();                          // panel complete, diagonal block of A still unfactored in memory
    if (s_fail) break;
    {                                         // threads 0..20 write Ljj (lower) and the reciprocal diagonal
      int idx = 0;                            // (statically unrolled: Lb must stay in registers)
#pragma unroll
      for (int r = 0; r < 6; r++)
#pragma unroll
        for (int c = 0; c <= r; c++, idx++)
          if (tid == idx) {
            A[(size_t)(j0 + r) * n + j0 + c] = Lb[r][c];
            if (r == c) diag[j0 + r] = rd[r];
          }
    }
    // ---- trailing update: A[i][c] -= sum_k L[i][j0+k] L[c][j0+k],  j0+6 <= c <= i
    for (int i = j0 + 6 + ty; i < n; i += 16) {
      double li[6];
#pragma unroll
      for (int k = 0; k < 6; k++) li[k] = A[(size_t)i * n + j0 + k];
      for (int c = j0 + 6 + tx; c <= i; c += 16) {
        double acc = A[(size_t)i * n + c];
#pragma unroll
        for (int k = 0; k < 6; k++) acc -= li[k] * A[(size_t)c * n + j0 + k];
        A[(size_t)i * n + c] = acc;
      }
    }
    __syncthreads();
  }
  if (s_fail) {
    for (int id = tid; id < n; id += nt) dx[id] = 0.f;
    if (Linv) for (int id = tid; id < n * n; id += nt) Linv[id] = 0.f;
    if (tid == 0 && status) *status = 1;
    if (tid == 0 && fail_count) *fail_count += 1;     // single CTA, stream-ordered: no atomic needed
    return;
  }
  // L is now in the lower triangle of A (diagonal included); diag[] holds 1 / L[i][i].
  // blocked forward / back substitution (6x6 pose blocks): thread 0 solves the diagonal block, all threads
  // eliminate it from the remaining rows: 2 barriers per block instead of one warp-serial step per row
  for (int jb = 0; jb < P; jb++) {                       // L z = y
    const int j0 = 6 * jb;
    if (tid == 0) {
#pragma unroll
      for (int c = 0; c < 6; c++) {
        double v = y[j0 + c];
#pragma unroll
        for (int k = 0; k < c; k++) v -= A[(size_t)(j0 + c) * n + j0 + k] * y[j0 + k];
        y[j0 + c] = v * diag[j0 + c];
      }
    }
    __syncthreads();
    for (int i = j0 + 6 + tid; i < n; i += nt) {
      double acc = 0.0;
#pragma unroll
      for (int k = 0; k < 6; k++) acc += A[(size_t)i * n + j0 + k] * y[j0 + k];
      y[i] -= acc;
    }
    __syncthreads();
  }
  for (int jb = P - 1; jb >= 0; jb--) {                  // L^T x = z
    const int j0 = 6 * jb;
    if (tid == 0) {
#pragma unroll
      for (int c = 5; c >= 0; c--) {
        double v = y[j0 + c];
#pragma unroll
        for (int k = c + 1; k < 6; k++) v -= A[(size_t)(j0 + k) * n + j0 + c] * y[j0 + k];
        y[j0 + c] = v * diag[j0 + c];
      }
    }
    __syncthreads();
    for (int i = tid; i < j0; i += nt) {
      double acc = 0.0;
#pragma unroll
      for (int k = 0; k < 6; k++) acc += A[(size_t)(j0 + k) * n + i] * y[j0 + k];
      y[i] -= acc;
    }
    __syncthreads();
  }
  for (int id = tid; id < n; id += nt) dx[id] = (float)y[id];
  if (tid == 0 && status) *status = 0;
  if (Linv) {
    // column c of X = L^-1: forward substitution, one thread per column, X stored in the UPPER triangle
    // (X[i][c] at A[c*n + i], i >= c; the diagonal entry X[c][c] = 1/L[c][c] stays in diag[])
    for (int c = tid; c < n; c += nt) {
      for (int i = 0; i < c; i++) Linv[(size_t)i * n + c] = 0.f;
      const double xcc = diag[c];
      Linv[(size_t)c * n + c] = (float)xcc;
      for (int i = c + 1; i < n; i++) {
        // four independent accumulators: the fp64 dependency chain, not the loads, bounds this loop
        double s0 = -A[(size_t)i * n + c] * xcc, s1 = 0.0, s2 = 0.0, s3 = 0.0;     // k = c term
        int k = c + 1;
        for (; k + 3 < i; k += 4) {
          s0 -= A[(size_t)i * n + k] * A[(size_t)c * n + k];                      // L[i][k] * X[k][c]
          s1 -= A[(size_t)i * n + k + 1] * A[(size_t)c * n + k + 1];
          s2 -= A[(size_t)i * n + k + 2] * A[(size_t)c * n + k + 2];
          s3 -= A[(size_t)i * n + k + 3] * A[(size_t)c * n + k + 3];
        }
        for (; k < i; k++) s0 -= A[(size_t)i * n + k] * A[(size_t)c * n + k];
        const double x = ((s0 + s1) + (s2 + s3)) * diag[i];
        A[(size_t)c * n + i] = x;
        Linv[(size_t)i * n + c] = (float)x;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// gtsam-style retraction on world_T_body, in double, one thread per pose.
__device__ inline void d_rot_apply(const double* q, const double* v, double* o) {
  const double ux = 2.0 * (q[1] * v[2] - q[2] * v[1]);
  const double uy = 2.0 * (q[2] * v[0] - q[0] * v[2]);
  const double uz = 2.0 * (q[0] * v[1] - q[1] * v[0]);
  o[0] = v[0] + q[3] * ux + (q[1] * uz - q[2] * uy);
  o[1] = v[1] + q[3] * uy + (q[2] * ux - q[0] * uz);
  o[2] = v[2] + q[3] * uz + (q[0] * uy - q[1] * ux);
}
__device__ inline void d_quat_mul(const double* a, const double* b, double* o) {
  const double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  const double y = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  const double z = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  const double w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  o[0] = x; o[1] = y; o[2] = z; o[3] = w;
}
// Pose3::Expmap([omega, v]) -> (dt, dq)
__device__ inline void d_pose3_expmap(const double* xi, double* dt, double* dq) {
  const double wx = xi[0], wy = xi[1], wz = xi[2];
  const double v[3] = {xi[3], xi[4], xi[5]};
  const double th2 = wx * wx + wy * wy + wz * wz;
  const double th = sqrt(th2);
  double A, B, Cc;  // sin(th)/th, (1-cos)/th^2, (th - sin)/th^3
  double imag, real;
  if (th < 1e-10) {
    A = 1.0 - th2 / 6.0; B = 0.5 - th2 / 24.0; Cc = 1.0 / 6.0 - th2 / 120.0;
    imag = 0.5 - th2 / 48.0; real = 1.0 - th2 / 8.0;
  } else {
    A = sin(th) / th; B = (1.0 - cos(th)) / th2; Cc = (th - sin(th)) / (th2 * th);
    imag = sin(0.5 * th) / th; real = cos(0.5 * th);
  }
  (void)A;
  dq[0] = imag * wx; dq[1] = imag * wy; dq[2] = imag * wz; dq[3] = real;
  // t = V v, V = I + B [w]x + C [w]x^2
  const double wv[3] = {wy * v[2] - wz * v[1], wz * v[0] - wx * v[2], wx * v[1] - wy * v[0]};
  const double wwv[3] = {wy * wv[2] - wz * wv[1], wz * wv[0] - wx * wv[2], wx * wv[1] - wy * wv[0]};
  for (int k = 0; k < 3; k++) dt[k] = v[k] + B * wv[k] + Cc * wwv[k];
}

__global__ void ba_retract_kernel(float* __restrict__ wTb, float* __restrict__ cTw,
                                  const float* __restrict__ cTb, const float* __restrict__ dx,
                                  int kf0, int P, const int* __restrict__ guard) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  if (guard && *guard) return;      // the solve of this iteration failed: leave the state untouched
  float* T = wTb + (size_t)(kf0 + i) * 7;
  double t[3] = {T[0], T[1], T[2]}, q[4] = {T[3], T[4], T[5], T[6]};
  double xi[6];
  for (int k = 0; k < 6; k++) xi[k] = dx[i * 6 + k];
  double dt[3], dq[4], rt[3], qn[4];
  d_pose3_expmap(xi, dt, dq);
  d_rot_apply(q, dt, rt);
  d_quat_mul(q, dq, qn);
  const double nrm = 1.0 / sqrt(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3]);
  for (int k = 0; k < 4; k++) qn[k] *= nrm;
  const double tn[3] = {t[0] + rt[0], t[1] + rt[1], t[2] + rt[2]};
  T[0] = (float)tn[0]; T[1] = (float)tn[1]; T[2] = (float)tn[2];
  T[3] = (float)qn[0]; T[4] = (float)qn[1]; T[5] = (float)qn[2]; T[6] = (float)qn[3];
  // cam_T_world = cam_T_body * (world_T_body)^-1, from the fp32-rounded world_T_body like the reference
  double q32[4] = {(double)T[3], (double)T[4], (double)T[5], (double)T[6]};
  double t32[3] = {(double)T[0], (double)T[1], (double)T[2]};
  double qi[4] = {-q32[0], -q32[1], -q32[2], q32[3]};
  double ti[3], tmp[3];
  d_rot_apply(qi, t32, tmp);
  ti[0] = -tmp[0]; ti[1] = -tmp[1]; ti[2] = -tmp[2];
  double qc[4] = {cTb[3], cTb[4], cTb[5], cTb[6]}, tc[3] = {cTb[0], cTb[1], cTb[2]};
  double qo[4], to[3];
  d_quat_mul(qc, qi, qo);
  d_rot_apply(qc, ti, to);
  float* C = cTw + (size_t)(kf0 + i) * 7;
  C[0] = (float)(to[0] + tc[0]); C[1] = (float)(to[1] + tc[1]); C[2] = (float)(to[2] + tc[2]);
  C[3] = (float)qo[0]; C[4] = (float)qo[1]; C[5] = (float)qo[2]; C[6] = (float)qo[3];
}

// legacy DROID left retraction (solve_poses / ba)
__global__ void pose_retr_kernel(float* __restrict__ poses, const float* __restrict__ dx, int kf0,
                                 int kf1) {
  for (int k = kf0 + threadIdx.x; k < kf1; k += blockDim.x) {
    float* T = poses + (size_t)k * 7;
    float t[3] = {T[0], T[1], T[2]}, q[4] = {T[3], T[4], T[5], T[6]};
    float dt[3], dq[4], t1[3], q1[4];
    se3_exp(dx + (size_t)(k - kf0) * 6, dt, dq);
    quat_mul(dq, q, q1);
    rot_apply(dq, t, t1);
    T[0] = t1[0] + dt[0]; T[1] = t1[1] + dt[1]; T[2] = t1[2] + dt[2];
    T[3] = q1[0]; T[4] = q1[1]; T[5] = q1[2]; T[6] = q1[3];
  }
}

// Log(prior^-1 * x) in [omega, t] (gtsam Pose3::Logmap), single thread, double
__global__ void pose_prior_error_kernel(const float* __restrict__ x, const float* __restrict__ pr,
                                        float* __restrict__ err) {
  if (threadIdx.x != 0) return;
  double qp[4] = {-(double)pr[3], -(double)pr[4], -(double)pr[5], (double)pr[6]};  // prior^-1 rot
  double qx[4] = {x[3], x[4], x[5], x[6]};
  double q[4];
  d_quat_mul(qp, qx, q);
  double dtw[3] = {(double)x[0] - pr[0], (double)x[1] - pr[1], (double)x[2] - pr[2]}, t[3];
  d_rot_apply(qp, dtw, t);
  if (q[3] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
  const double sn = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
  double w[3];
  double th;
  if (sn < 1e-12) {
    th = 0.0; w[0] = 2.0 * q[0]; w[1] = 2.0 * q[1]; w[2] = 2.0 * q[2];
  } else {
    th = 2.0 * atan2(sn, q[3]);
    const double s = th / sn;
    w[0] = s * q[0]; w[1] = s * q[1]; w[2] = s * q[2];
  }
  // u = V^-1 t,  V^-1 = I - 1/2 [w]x + c [w]x^2,  c = (1 - (th sin th)/(2(1-cos th)))/th^2
  double c;
  if (th < 1e-5) c = 1.0 / 12.0;
  else c = (1.0 - th * sin(th) / (2.0 * (1.0 - cos(th)))) / (th * th);
  const double wt[3] = {w[1] * t[2] - w[2] * t[1], w[2] * t[0] - w[0] * t[2], w[0] * t[1] - w[1] * t[0]};
  const double wwt[3] = {w[1] * wt[2] - w[2] * wt[1], w[2] * wt[0] - w[0] * wt[2], w[0] * wt[1] - w[1] * wt[0]};
  for (int k = 0; k < 3; k++) {
    err[k] = (float)w[k];
    err[3 + k] = (float)(t[k] - 0.5 * wt[k] + c * wwt[k]);
  }
}

// ------------------------------------------------------------------------------------------
// A13: depth back-substitution, grid (T, K)
__global__ void __launch_bounds__(TILE)
ba_depth_kernel(nslam_ba_graph g, nslam_ba_buffers b, const float* __restrict__ dx,
                float clamp_min, const int* __restrict__ guard) {
  if (guard && *guard) return;      // failed solve: no depth step either (the live path's gtsam solve would raise)
  const int k = blockIdx.y;
  const int hw = b.ht * b.wd;
  const int p = blockIdx.x * TILE + threadIdx.x;
  if (p >= hw) return;
  const int r0 = g.row_ptr[k], r1 = g.row_ptr[k + 1];
  float dw = 0.f;
  for (int r = r0; r < r1; r++) {
    const int pose = g.row_pose[r];
    if (pose <= 0 || pose >= g.P) continue;  // `idx <= 0` quirk of EvT6x1_kernel (src/droid_kernels.cu:1225)
    const float* src = b.Emat + ((size_t)g.row_erow[r] * 6) * hw + p;
    float s = 0.f;
#pragma unroll
    for (int n = 0; n < 6; n++) s += src[(size_t)n * hw] * dx[pose * 6 + n];
    dw += s;
  }
  const float dz = b.Q[(size_t)k * hw + p] * (b.w[(size_t)k * hw + p] - dw);
  float* d = b.disps + (size_t)g.kx[k] * hw + p;
  float nv = *d + dz;
  if (clamp_min > 0.f) nv = fmaxf(nv, clamp_min);
  *d = nv;
}

// A14: z_cov[k][p] = Q + sum_j (Q * (x^T Linv)_j)^2 = Q + Q^2 x^T (Linv Linv^T) x, where x stacks
// the E rows of depth map k (non-zero only on the 6-blocks of the poses that see k).
// M = Linv Linv^T is formed once (n^3, tiny); the per-pixel work is then (6R)^2 FMAs instead of
// the reference's dense [K*HW, 6P] x [6P, 6P] GEMM over a zero-filled K*K*6*HW scratch tensor.
__global__ void ba_cov_M_kernel(const float* __restrict__ Linv, int n, float* __restrict__ M) {
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n * n) return;
  const int r = id / n, c = id % n;
  float s = 0.f;
  const int kmax = (r < c ? r : c);  // Linv is lower triangular
  for (int k = 0; k <= kmax; k++) s += Linv[(size_t)r * n + k] * Linv[(size_t)c * n + k];
  M[id] = s;
}

// grid (T, K), dynamic smem: R*R*36 floats (the M blocks of the pose pairs touching k)
__global__ void __launch_bounds__(TILE)
ba_cov_kernel(nslam_ba_graph g, nslam_ba_buffers b, const float* __restrict__ M,
              float* __restrict__ z_cov, float* __restrict__ depth_cov) {
  extern __shared__ float sMb[];
  const int k = blockIdx.y;
  const int hw = b.ht * b.wd;
  const int n = 6 * g.P;
  const int r0 = g.row_ptr[k], R = g.row_ptr[k + 1] - r0;
  for (int id = threadIdx.x; id < R * R * 36; id += TILE) {
    const int blk = id / 36, mn = id % 36;
    const int pa = g.row_pose[r0 + blk / R], pb = g.row_pose[r0 + blk % R];
    sMb[id] = M[(size_t)(pa * 6 + mn / 6) * n + pb * 6 + mn % 6];
  }
  __syncthreads();
  const int p = blockIdx.x * TILE + threadIdx.x;
  if (p >= hw) return;
  const float q = b.Q[(size_t)k * hw + p];
  float acc = 0.f;
  for (int ra = 0; ra < R; ra++) {
    const float* sa = b.Emat + ((size_t)g.row_erow[r0 + ra] * 6) * hw + p;
    float ea[6];
#pragma unroll
    for (int m = 0; m < 6; m++) ea[m] = sa[(size_t)m * hw];
    for (int rb = 0; rb < R; rb++) {
      const float* sb = b.Emat + ((size_t)g.row_erow[r0 + rb] * 6) * hw + p;
      const float* Mb = sMb + (ra * R + rb) * 36;
#pragma unroll
      for (int nn = 0; nn < 6; nn++) {
        const float eb = sb[(size_t)nn * hw];
        float s = 0.f;
#pragma unroll
        for (int m = 0; m < 6; m++) s += ea[m] * Mb[m * 6 + nn];
        acc += s * eb;
      }
    }
  }
  const float zc = q + q * q * acc;
  z_cov[(size_t)k * hw + p] = zc;
  if (depth_cov) {
    const float d = b.disps[(size_t)g.kx[k] * hw + p];
    const float d2 = d * d;
    depth_cov[(size_t)k * hw + p] = zc / (d2 * d2);
  }
}

__global__ void ba_pose_cov_kernel(const float* __restrict__ Linv, int P, float* __restrict__ sg) {
  const int i = blockIdx.x;
  const int r = threadIdx.x / 6, c = threadIdx.x % 6;
  const int n = 6 * P;
  float s = 0.f;
  for (int k = 0; k < n; k++) s += Linv[(size_t)k * n + i * 6 + r] * Linv[(size_t)k * n + i * 6 + c];
  sg[(size_t)i * 36 + threadIdx.x] = s;
}

}  // namespace nslam

extern "C" {

int nslam_ba_reduced_camera_matrix(const nslam_ba_graph* g, const nslam_ba_buffers* b,
                                   void* stream) {
  using namespace nslam;
  cudaStream_t st = (cudaStream_t)stream;
  if (g->P <= 0) return (int)cudaErrorInvalidValue;
  if (g->E > 0) {
    ba_prep_edges_kernel<<<(g->E + 63) / 64, 64, 0, st>>>(*g, b->poses, b->extrinsics, b->edge_aux);
    NSLAM_CHECK_LAUNCH();
  }
  dim3 grid(b->T, g->K);
  ba_linearize_kernel<<<grid, TILE, 0, st>>>(*g, *b);
  NSLAM_CHECK_LAUNCH();
  if (g->E > 0) {
    ba_edge_blocks_kernel<<<g->E, 64, 0, st>>>(*g, *b);
    NSLAM_CHECK_LAUNCH();
  }
  const size_t smem = ((size_t)6 * g->RMAX * (TILE + 1) + 2 * TILE) * sizeof(float);
  if (smem > 227 * 1024) return (int)cudaErrorInvalidValue;
  if (cudaError_t e = ensure_dyn_smem<ba_schur_kernel>(smem)) return (int)e;
  ba_schur_kernel<<<grid, TILE, smem, st>>>(*g, *b);
  NSLAM_CHECK_LAUNCH();
  const int nvals = g->NPAIR * 36 + g->NR * 6;
  if (nvals > 0) {
    ba_schur_reduce_kernel<<<(nvals + 255) / 256, 256, 0, st>>>(b->spart, b->sblk, nvals, b->T);
    NSLAM_CHECK_LAUNCH();
  }
  ba_assemble_kernel<<<g->P * g->P + g->P, 36, 0, st>>>(*g, *b);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

static int launch_solve(const float* Hin, const float* vin, int P, int prior_pose_idx,
                        const float* prior_err, float prior_info, float lm, float ep, double* work,
                        float* dx, float* Linv, int* status, int* fail_count, cudaStream_t st) {
  using namespace nslam;
  const int n = 6 * P;
  const size_t smem = (size_t)n * n * sizeof(double);
  if (smem <= 200 * 1024) {
    if (cudaError_t e = ensure_dyn_smem<ba_solve_kernel<true>>(smem > 48 * 1024 ? (size_t)200 * 1024 : smem)) return (int)e;
    ba_solve_kernel<true><<<1, 256, smem, st>>>(Hin, vin, n, prior_pose_idx, prior_err, prior_info,
                                                lm, ep, work, dx, Linv, status, fail_count);
  } else {
    ba_solve_kernel<false><<<1, 256, 0, st>>>(Hin, vin, n, prior_pose_idx, prior_err, prior_info,
                                              lm, ep, work, dx, Linv, status, fail_count);
  }
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_ba_solve(const float* Hin, const float* vin, int P, int prior_pose_idx,
                   const float* prior_err, float prior_info, float lm, float ep, double* work,
                   float* dx, float* Linv, int* status, void* stream) {
  return launch_solve(Hin, vin, P, prior_pose_idx, prior_err, prior_info, lm, ep, work, dx, Linv, status, nullptr,
                      (cudaStream_t)stream);
}

/* pixels per CTA tile of the BA kernels: callers size `part`/`spart` with T = ceil(ht*wd / tile) */
int nslam_ba_tile_pixels(void) { return nslam::TILE; }

int nslam_ba_retract(float* world_T_body, float* cam_T_world, const float* cam_T_body,
                     const float* dx, int kf0, int P, void* stream) {
  if (P <= 0) return 0;
  nslam::ba_retract_kernel<<<(P + 63) / 64, 64, 0, (cudaStream_t)stream>>>(
      world_T_body, cam_T_world, cam_T_body, dx, kf0, P, nullptr);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_pose_retr(float* poses, const float* dx, int kf0, int kf1, void* stream) {
  nslam::pose_retr_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(poses, dx, kf0, kf1);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_pose_prior_error(const float* world_T_body_k, const float* prior_pose, float* err6,
                           void* stream) {
  nslam::pose_prior_error_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(world_T_body_k, prior_pose, err6);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_ba_depth(const nslam_ba_graph* g, const nslam_ba_buffers* b, const float* dx,
                   float clamp_min, void* stream) {
  dim3 grid(b->T, g->K);
  nslam::ba_depth_kernel<<<grid, nslam::TILE, 0, (cudaStream_t)stream>>>(*g, *b, dx, clamp_min, nullptr);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_ba_cov(const nslam_ba_graph* g, const nslam_ba_buffers* b, const float* Linv,
                 float* Mscratch, float* z_cov, float* depth_cov, void* stream) {
  using namespace nslam;
  const int n = 6 * g->P;
  cudaStream_t st = (cudaStream_t)stream;
  ba_cov_M_kernel<<<(n * n + 255) / 256, 256, 0, st>>>(Linv, n, Mscratch);
  NSLAM_CHECK_LAUNCH();
  const size_t smem = (size_t)g->RMAX * g->RMAX * 36 * sizeof(float);
  if (smem > 227 * 1024) return (int)cudaErrorInvalidValue;
  if (cudaError_t e = ensure_dyn_smem<ba_cov_kernel>(smem)) return (int)e;
  dim3 grid(b->T, g->K);
  ba_cov_kernel<<<grid, TILE, smem, st>>>(*g, *b, Mscratch, z_cov, depth_cov);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

int nslam_ba_pose_cov(const float* Linv, int P, float* sigma_g, void* stream) {
  if (P <= 0) return 0;
  nslam::ba_pose_cov_kernel<<<P, 36, 0, (cudaStream_t)stream>>>(Linv, P, sigma_g);
  NSLAM_CHECK_LAUNCH();
  return 0;
}

/* Front-end fast path: `iters` complete Gauss-Newton iterations in ONE host call
 * (linearise -> Schur -> assemble -> [prior] -> fp64 Cholesky -> gtsam-style retract -> depth update).
 * b->poses must alias cam_T_world (it is refreshed by the retraction between iterations). */
int nslam_ba_gn_iterations(const nslam_ba_graph* g, const nslam_ba_buffers* b, int iters,
                           float* world_T_body, float* cam_T_world, const float* cam_T_body,
                           int prior_pose_idx, const float* prior_pose, float prior_info,
                           double* work, float* dx, float* Linv, float* prior_err, int* status,
                           float clamp_min, void* stream) {
  for (int it = 0; it < iters; it++) {
    int r = nslam_ba_reduced_camera_matrix(g, b, stream);
    if (r) return r;
    if (prior_pose_idx >= 0) {
      r = nslam_pose_prior_error(world_T_body + (size_t)(g->kf0 + prior_pose_idx) * 7, prior_pose, prior_err, stream);
      if (r) return r;
    }
    r = nslam_ba_solve(b->H, b->v, g->P, prior_pose_idx, prior_err, prior_pose_idx >= 0 ? prior_info : 0.f, 0.f, 0.f,
                       work, dx, (it == iters - 1) ? Linv : nullptr, status, stream);
    if (r) return r;
    r = nslam_ba_retract(world_T_body, cam_T_world, cam_T_body, dx, g->kf0, g->P, stream);
    if (r) return r;
    r = nslam_ba_depth(g, b, dx, clamp_min, stream);
    if (r) return r;
  }
  return 0;
}

/* The live front end's whole BA step in ONE host call (visual_frontend.py:1097-1230): `iters` Gauss-Newton iterations
 * as nslam_ba_gn_iterations, then the covariance block written straight into the keyframe arenas.  A failed
 * factorisation (status[0] = 1, status[1] += 1) leaves poses, depths and covariances of that iteration untouched —
 * the reference's gtsam solve raises there; its CUDA twin zeroes dx but still applies dz = Q w.
 * lm, ep: Levenberg damping of the pose system, diag += ep + lm*diag (0, 0 on the live path; DROID's FactorGraph
 * passes 1e-4 / 0.1, networks/factor_graph.py:251-253). */
int nslam_ba_frontend_update(const nslam_ba_graph* g, const nslam_ba_buffers* b, int iters,
                             float* world_T_body, float* cam_T_world, const float* cam_T_body,
                             int prior_pose_idx, const float* prior_pose, float prior_info,
                             float lm, float ep,
                             double* work, float* dx, float* Linv, float* prior_err, int* status,
                             float clamp_min, int cov_mode, float* Mscratch, float* idepths_cov,
                             float* depths_cov, float* pose_cov, void* stream) {
  using namespace nslam;
  cudaStream_t st = (cudaStream_t)stream;
  const bool want_cov = cov_mode >= 0;
  for (int it = 0; it < iters; it++) {
    int r = nslam_ba_reduced_camera_matrix(g, b, stream);
    if (r) return r;
    if (prior_pose_idx >= 0) {
      r = nslam_pose_prior_error(world_T_body + (size_t)(g->kf0 + prior_pose_idx) * 7, prior_pose, prior_err, stream);
      if (r) return r;
    }
    r = launch_solve(b->H, b->v, g->P, prior_pose_idx, prior_err, prior_pose_idx >= 0 ? prior_info : 0.f, lm, ep,
                     work, dx, (want_cov && it == iters - 1) ? Linv : nullptr, status, status + 1, st);
    if (r) return r;
    ba_retract_kernel<<<(g->P + 63) / 64, 64, 0, st>>>(world_T_body, cam_T_world, cam_T_body, dx, g->kf0, g->P, status);
    NSLAM_CHECK_LAUNCH();
    dim3 grid(b->T, g->K);
    ba_depth_kernel<<<grid, TILE, 0, st>>>(*g, *b, dx, clamp_min, status);
    NSLAM_CHECK_LAUNCH();
  }
  if (want_cov && iters > 0)
    return nslam_ba_cov_arena(g, b, Linv, Mscratch, cov_mode, status, idepths_cov, depths_cov, pose_cov, stream);
  return 0;
}

}  // extern "C"
