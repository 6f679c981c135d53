// Gram phase of the 32-wide update kernels (update_tile.cu: FP32 layer chain; update_umma32.cu: tensor-core layer chain): the
// weight gradients as Gram products over one tile of samples staged feature-major in shared memory,
//     dW0 = X^T D1, db0 = 1^T D1, dW1 = H1^T D2, db1 = 1^T D2, dWout = H2^T DM, dbout = 1^T DM, dlog_std = 1^T DL,
// accumulated by 128 threads: dW1 (32 x 32 outputs, the bulk) in register tiles, rows interleaved by 8 so that every
// LDS.128 of a warp is conflict-free; the small outputs spread over the four warps (see TileGram).  A 128-sample stage
// splits dW1 in two K-halves of 64 samples over the threads (4x4 tiles); a 64-sample stage (one 64-row MMA block of
// update_umma32.cu, one of those K-halves) gives every thread 8 outputs over the whole stage (4x2 tiles), so each dW1
// float32 sum covers the same samples in the same order either way.  Per-stage float32 dW1 sums are folded into float64
// register accumulators that live across the persistent tile loop; write() stores the block's float64 partial vector.
#pragma once
#include "update_common.cuh"

namespace b200rl {

// distribution constants of one pass (A <= TILE_AMAX, entries k < A in use; a register-resident local); FVP: old == new
constexpr int TILE_AMAX = 6;
struct TileDist {
  float ls_new[TILE_AMAX], inv_std[TILE_AMAX], ls_old[TILE_AMAX], inv_std_old[TILE_AMAX], Mmu[TILE_AMAX],
      var_new[TILE_AMAX], var_new2[TILE_AMAX], var_old[TILE_AMAX];
  float sum_ls_new, sum_ls_old, half_log2pi_A;
};

template <class N, int MODE>
__device__ __forceinline__ void tile_dist_init(TileDist& D, const float* log_std_params, const UpdArgs& a) {
  constexpr int A = N::A;
  static_assert(A <= TILE_AMAX, "act_dim beyond the TileDist arrays");
  D.sum_ls_new = 0.f;
  D.sum_ls_old = 0.f;
#pragma unroll
  for (int k = 0; k < A; ++k) {
    D.ls_new[k] = clamp_log_std(log_std_params[k], a.log_min_std);
    const float sd = expf(D.ls_new[k]);
    D.inv_std[k] = 1.0f / sd;
    D.var_new[k] = sd * sd;
    D.var_new2[k] = 2.0f * sd * sd + 1e-8f;
    D.Mmu[k] = 2.0f / D.var_new2[k];
    D.ls_old[k] = (MODE == MODE_FVP) ? D.ls_new[k] : a.old_log_std[k];
    const float so = expf(D.ls_old[k]);
    D.inv_std_old[k] = 1.0f / so;
    D.var_old[k] = so * so;
    D.sum_ls_new += D.ls_new[k];
    D.sum_ls_old += D.ls_old[k];
  }
  D.half_log2pi_A = 0.5f * (float)A * 1.8378770664093453f;
}

// RX..RDM: first stage row of X, H1, H2, D1, D2, DM (DL rows follow DM); LD: row pitch in floats (stage length + 4);
// TILE: samples of one stage (128, or 64 for a caller that stages one 64-row MMA block at a time).
// The accumulation is split in two parts so that a caller whose D1 rows only exist later (update_umma32.cu: D1 needs one
// more tensor-core GEMM) can run part A behind that GEMM, and may alias the D1 rows with the H2 rows (dead after part A):
//   part A  dW1 = H1^T D2 (all 128 threads: 4x4 register tiles x two K-halves, or 4x2 tiles over a 64-sample stage),
//           dWout[:, k] / db1 (A <= 3: warp k / warp 3; A <= 6: job j = column j < A or db1 at j = A, on warp j % 4,
//           slot j / 4), dbout / dlog_std row sums (threads < 2A)                   -- reads H1, H2, D2, DM, DL
//   part B  dW0[o, :] for o = warp, warp + 4, ... and db0 (warp 3)                     -- reads X, D1
// Every small output is spread over the four warps: with one warp per output group (the first layout) warp 0 carried
// dW1 + all of dW0 -- 2.7x the work of the others for obs_dim 13 -- and set the length of the phase.
// The small outputs keep float32 partial sums (pA, pT, pB) until fold_a() / fold_b(): a caller that stages a 128-sample
// tile as two 64-sample stages runs both through part_a / part_b and folds once per tile, so those sums see the samples
// in the order of one pass over the whole tile.  accumulate_a / accumulate_b: one part and its fold.
// PACKED: dW1 with float2 even / odd partial sums (two samples per ffma2()).
template <class N, int RX, int RH1, int RH2, int RD1, int RD2, int RDM, int LD, bool PACKED = false, int TILE = 128>
struct TileGram {
  static constexpr int O = N::O, H = 32, A = N::A;
  static_assert(TILE == 128 || TILE == 64, "128- or 64-sample stages");
  static constexpr int WC = TILE == 128 ? 4 : 2;  // dW1 columns per thread (4 rows each)
  static constexpr int CS = 32 / WC;              // column stride of a thread's dW1 tile
  static constexpr int OQ = (O + 3) / 4;          // obs rows per warp in part B
  static_assert(N::H1 == 32 && N::H2 == 32 && A <= 6, "32-wide layers, act_dim <= 6");
  static constexpr int NS = A <= 3 ? 1 : 2;       // part-A jobs per warp
  static constexpr int JDB = A <= 3 ? 3 : A;      // job index of db1
  double accW1[4][WC];
  double accB[OQ + 1];   // part B: dW0[warp + 4 i][lane], i < OQ; [OQ]: db0[lane] (warp 3)
  double accA, accA1;    // part A, job j = warp + 4 s (s = 0: accA, 1: accA1): dWout[lane][j] (j < A) | db1 (j == JDB)
  double accT;           // part A: dbout[tid] / dlog_std[tid - A] row sums (tid < 2A)
  float pA[NS][2], pT, pB[OQ + 1];   // float32 partial sums of accA / accA1, accT, accB since the last fold

  // this thread's dW1 tile: rows ti + 8 r, columns tj + CS c, over samples [kh * 64, kh * 64 + 64) of the stage
  __device__ __forceinline__ static void w1_tile_of(int tid, int& ti, int& tj, int& kh) {
    if constexpr (TILE == 128) {
      ti = (tid & 63) >> 3;
      tj = tid & 7;
      kh = tid >> 6;
    } else {
      ti = tid & 7;
      tj = tid >> 3;
      kh = 0;
    }
  }

  __device__ __forceinline__ void zero_partials() {
#pragma unroll
    for (int s = 0; s < NS; ++s) pA[s][0] = pA[s][1] = 0.f;
    pT = 0.f;
#pragma unroll
    for (int i = 0; i <= OQ; ++i) pB[i] = 0.f;
  }

  __device__ __forceinline__ void init() {
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < WC; ++c) accW1[r][c] = 0.0;
#pragma unroll
    for (int k = 0; k <= OQ; ++k) accB[k] = 0.0;
    accA = 0.0;
    accA1 = 0.0;
    accT = 0.0;
    zero_partials();
  }

  __device__ __forceinline__ void accumulate_a(const float* stage, int tid) {
    part_a(stage, tid);
    fold_a(tid);
  }
  __device__ __forceinline__ void accumulate_b(const float* stage, int tid) {
    part_b<LD>(stage, stage + RX * LD, tid);
    fold_b();
  }

  __device__ __forceinline__ void part_a(const float* stage, int tid) {
    int ti, tj, kh;
    w1_tile_of(tid, ti, tj, kh);
    const float* U = stage + (RH1 + ti) * LD + kh * 64;
    const float* V = stage + (RD2 + tj) * LD + kh * 64;
    if constexpr (PACKED) {
      float2 acc[4][WC];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < WC; ++c) acc[r][c] = make_float2(0.f, 0.f);
#pragma unroll 2
      for (int k = 0; k < 64; k += 4) {
        float4 u[4], v[WC];
#pragma unroll
        for (int r = 0; r < 4; ++r) u[r] = *reinterpret_cast<const float4*>(U + r * 8 * LD + k);
#pragma unroll
        for (int c = 0; c < WC; ++c) v[c] = *reinterpret_cast<const float4*>(V + c * CS * LD + k);
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < WC; ++c) gram_fma4(u[r], v[c], acc[r][c]);
      }
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < WC; ++c) accW1[r][c] += (double)(acc[r][c].x + acc[r][c].y);
    } else {
      float acc[4][WC];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < WC; ++c) acc[r][c] = 0.f;
#pragma unroll 4
      for (int k = 0; k < 64; k += 4) {
        float4 u[4], v[WC];
#pragma unroll
        for (int r = 0; r < 4; ++r) u[r] = *reinterpret_cast<const float4*>(U + r * 8 * LD + k);
#pragma unroll
        for (int c = 0; c < WC; ++c) v[c] = *reinterpret_cast<const float4*>(V + c * CS * LD + k);
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < WC; ++c) {
            acc[r][c] = fmaf(u[r].x, v[c].x, acc[r][c]);
            acc[r][c] = fmaf(u[r].y, v[c].y, acc[r][c]);
            acc[r][c] = fmaf(u[r].z, v[c].z, acc[r][c]);
            acc[r][c] = fmaf(u[r].w, v[c].w, acc[r][c]);
          }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < WC; ++c) accW1[r][c] += (double)acc[r][c];
    }
    // small outputs of part A: job j < A -> dWout[lane][j] = H2[lane] . DM[j]; job JDB -> db1[lane] = sum D2[lane]
    const int lane = tid & 31, wq = tid >> 5;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
    const int j = wq + 4 * s;
    if (j < A) {
      const float* Hh = stage + (RH2 + lane) * LD;
      const float* M = stage + (RDM + j) * LD;
      float s0 = pA[s][0], s1 = pA[s][1];
#pragma unroll 4
      for (int k = 0; k < TILE; k += 4) {
        const float4 hv = *reinterpret_cast<const float4*>(Hh + k);
        const float4 m = *reinterpret_cast<const float4*>(M + k);
        s0 = fmaf(hv.x, m.x, s0); s1 = fmaf(hv.y, m.y, s1);
        s0 = fmaf(hv.z, m.z, s0); s1 = fmaf(hv.w, m.w, s1);
      }
      pA[s][0] = s0;
      pA[s][1] = s1;
    } else if (j == JDB) {
      const float* Dr = stage + (RD2 + lane) * LD;
      float s0 = pA[s][0];
#pragma unroll 4
      for (int k = 0; k < TILE; k += 4) {
        const float4 d = *reinterpret_cast<const float4*>(Dr + k);
        s0 += (d.x + d.y) + (d.z + d.w);
      }
      pA[s][0] = s0;
    }
    }
    if (tid < 2 * A) {
      const float* Dr = stage + (RDM + tid) * LD;   // rows DM[0..A-1], DL[0..A-1] are contiguous
      float s0 = pT;
#pragma unroll 4
      for (int k = 0; k < TILE; k += 4) {
        const float4 d = *reinterpret_cast<const float4*>(Dr + k);
        s0 += (d.x + d.y) + (d.z + d.w);
      }
      pT = s0;
    }
  }

  __device__ __forceinline__ void fold_a(int tid) {
    const int wq = tid >> 5;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      const int j = wq + 4 * s;
      double& acc = s == 0 ? accA : accA1;
      if (j < A) acc += (double)(pA[s][0] + pA[s][1]);
      else if (j == JDB) acc += (double)pA[s][0];
      pA[s][0] = pA[s][1] = 0.f;
    }
    if (tid < 2 * A) accT += (double)pT;
    pT = 0.f;
  }

  // X: row 0 of the X rows (pitch XLD; X[o][k] at X + o * XLD + k, k < TILE)
  template <int XLD>
  __device__ __forceinline__ void part_b(const float* stage, const float* X, int tid) {
    const int lane = tid & 31, wq = tid >> 5;
    const float* Dr = stage + (RD1 + lane) * LD;
    float sa[OQ + 1];
#pragma unroll
    for (int i = 0; i <= OQ; ++i) sa[i] = pB[i];
#pragma unroll 4
    for (int k = 0; k < TILE; k += 4) {
      const float4 d = *reinterpret_cast<const float4*>(Dr + k);
#pragma unroll
      for (int i = 0; i < OQ; ++i) {
        const int o = wq + 4 * i;
        if (o < O) {
          const float4 xv = *reinterpret_cast<const float4*>(X + o * XLD + k);
          sa[i] = fmaf(xv.x, d.x, sa[i]); sa[i] = fmaf(xv.y, d.y, sa[i]);
          sa[i] = fmaf(xv.z, d.z, sa[i]); sa[i] = fmaf(xv.w, d.w, sa[i]);
        }
      }
      if (wq == 3) sa[OQ] += (d.x + d.y) + (d.z + d.w);
    }
#pragma unroll
    for (int i = 0; i <= OQ; ++i) pB[i] = sa[i];
  }

  __device__ __forceinline__ void fold_b() {
#pragma unroll
    for (int i = 0; i <= OQ; ++i) {
      accB[i] += (double)pB[i];
      pB[i] = 0.f;
    }
  }

  // out: this block's partial vector [P]; scr: >= 2 * 64 * 16 doubles of shared memory no thread still reads (128-sample
  // stages: the two K-halves of dW1 are combined there; unused for 64); sync: the barrier of the 128 threads
  // (__syncthreads, or a warpgroup's named barrier when a CTA holds several)
  __device__ __forceinline__ void write(double* out, double* scr, int tid) {
    write(out, scr, tid, [] { __syncthreads(); });
  }
  template <class Sync>
  __device__ __forceinline__ void write(double* out, double* scr, int tid, Sync sync) {
    int ti, tj, kh;
    w1_tile_of(tid, ti, tj, kh);
    if constexpr (TILE == 128) {
      const int w1_tile = tid & 63;
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) scr[(kh * 64 + w1_tile) * 16 + r * 4 + c] = accW1[r][c];
      sync();
      if (tid < 64) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c)
            out[N::oW1 + (ti + 8 * r) * H + (tj + 8 * c)] = scr[w1_tile * 16 + r * 4 + c] + scr[(64 + w1_tile) * 16 + r * 4 + c];
      }
    } else {
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < WC; ++c) out[N::oW1 + (ti + 8 * r) * H + (tj + CS * c)] = accW1[r][c];
    }
    const int lane = tid & 31, wq = tid >> 5;
#pragma unroll
    for (int i = 0; i < OQ; ++i) {
      const int o = wq + 4 * i;
      if (o < O) out[N::oW0 + o * H + lane] = accB[i];
    }
    if constexpr (A <= 3) {
      if (wq == 3) {
        out[N::ob0 + lane] = accB[OQ];
        out[N::ob1 + lane] = accA;
      } else if (wq < A) {
        out[N::oWo + lane * A + wq] = accA;
      }
    } else {
      if (wq == 3) out[N::ob0 + lane] = accB[OQ];
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        const int j = wq + 4 * s;
        const double acc = s == 0 ? accA : accA1;
        if (j == JDB) out[N::ob1 + lane] = acc;
        else if (j < A) out[N::oWo + lane * A + j] = acc;
      }
    }
    if (tid < 2 * A) out[N::obo + tid] = accT;   // obo.. then ols.. are contiguous in the flat layout
  }
};

}  // namespace b200rl
