// Gram phase of the 32-wide update kernels (update_tile.cu: FP32 layer chain; update_umma32.cu: tensor-core layer chain): the
// weight gradients as Gram products over one 128-sample tile staged feature-major in shared memory,
//     dW0 = X^T D1, db0 = 1^T D1, dW1 = H1^T D2, db1 = 1^T D2, dWout = H2^T DM, dbout = 1^T DM, dlog_std = 1^T DL,
// accumulated by the 128 threads of the CTA: dW1 (32 x 32 outputs, the bulk) in 4x4 register tiles, rows interleaved by 8
// so that every LDS.128 of a warp is conflict-free, split in two K-halves over the threads; the small outputs spread over
// the four warps (see TileGram).  Per-tile float32 partial products are folded into float64 register accumulators that
// live across the persistent tile loop; write() combines the K-halves through shared memory and stores the block's float64
// partial vector.
#pragma once
#include "update_common.cuh"

namespace b200rl {

// distribution constants of one pass (A <= 3); FVP: old == new
struct TileDist {
  float ls_new[3], inv_std[3], ls_old[3], inv_std_old[3], Mmu[3], var_new[3], var_new2[3], var_old[3];
  float sum_ls_new, sum_ls_old, half_log2pi_A;
};

template <class N, int MODE>
__device__ __forceinline__ void tile_dist_init(TileDist& D, const float* log_std_params, const UpdArgs& a) {
  constexpr int A = N::A;
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

// RX..RDM: first stage row of X, H1, H2, D1, D2, DM (DL rows follow DM); LD: row pitch in floats (tile + 4).
// The accumulation is split in two parts so that a caller whose D1 rows only exist later (update_umma32.cu: D1 needs one
// more tensor-core GEMM) can run part A behind that GEMM, and may alias the D1 rows with the H2 rows (dead after part A):
//   part A  dW1 = H1^T D2 (all 128 threads: 4x4 register tiles x two K-halves), dWout[:, k] / db1 (warp k / warp 3),
//           dbout / dlog_std row sums (threads < 2A)                                   -- reads H1, H2, D2, DM, DL
//   part B  dW0[o, :] for o = warp, warp + 4, ... and db0 (warp 3)                     -- reads X, D1
// Every small output is spread over the four warps: with one warp per output group (the first layout) warp 0 carried
// dW1 + all of dW0 -- 2.7x the work of the others for obs_dim 13 -- and set the length of the phase.
// PACKED: dW1 with float2 even / odd partial sums (two samples per ffma2()).
template <class N, int RX, int RH1, int RH2, int RD1, int RD2, int RDM, int LD, bool PACKED = false>
struct TileGram {
  static constexpr int O = N::O, H = 32, A = N::A, TILE = 128;
  static constexpr int OQ = (O + 3) / 4;          // obs rows per warp in part B
  static_assert(N::H1 == 32 && N::H2 == 32 && A <= 3, "32-wide layers, act_dim <= 3");
  double accW1[4][4];
  double accB[OQ + 1];   // part B: dW0[warp + 4 i][lane], i < OQ; [OQ]: db0[lane] (warp 3)
  double accA;           // part A: dWout[lane][warp] (warp < A) | db1[lane] (warp 3)
  double accT;           // part A: dbout[tid] / dlog_std[tid - A] row sums (tid < 2A)

  __device__ __forceinline__ void init() {
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) accW1[r][c] = 0.0;
#pragma unroll
    for (int k = 0; k <= OQ; ++k) accB[k] = 0.0;
    accA = 0.0;
    accT = 0.0;
  }

  __device__ __forceinline__ void accumulate_a(const float* stage, int tid) {
    const int w1_tile = tid & 63, kh = tid >> 6;
    const int ti = w1_tile >> 3, tj = w1_tile & 7;
    const float* U = stage + (RH1 + ti) * LD + kh * 64;
    const float* V = stage + (RD2 + tj) * LD + kh * 64;
    if constexpr (PACKED) {
      float2 acc[4][4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = make_float2(0.f, 0.f);
#pragma unroll 2
      for (int k = 0; k < 64; k += 4) {
        float4 u[4], v[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) u[r] = *reinterpret_cast<const float4*>(U + r * 8 * LD + k);
#pragma unroll
        for (int c = 0; c < 4; ++c) v[c] = *reinterpret_cast<const float4*>(V + c * 8 * LD + k);
        gram_4x4(u, v, acc);
      }
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) accW1[r][c] += (double)(acc[r][c].x + acc[r][c].y);
    } else {
      float acc[4][4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
#pragma unroll 4
      for (int k = 0; k < 64; k += 4) {
        float4 u[4], v[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) u[r] = *reinterpret_cast<const float4*>(U + r * 8 * LD + k);
#pragma unroll
        for (int c = 0; c < 4; ++c) v[c] = *reinterpret_cast<const float4*>(V + c * 8 * LD + k);
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            acc[r][c] = fmaf(u[r].x, v[c].x, acc[r][c]);
            acc[r][c] = fmaf(u[r].y, v[c].y, acc[r][c]);
            acc[r][c] = fmaf(u[r].z, v[c].z, acc[r][c]);
            acc[r][c] = fmaf(u[r].w, v[c].w, acc[r][c]);
          }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) accW1[r][c] += (double)acc[r][c];
    }
    // small outputs of part A: warp k < A -> dWout[lane][k] = H2[lane] . DM[k]; warp 3 -> db1[lane] = sum D2[lane]
    const int lane = tid & 31, wq = tid >> 5;
    if (wq < A) {
      const float* Hh = stage + (RH2 + lane) * LD;
      const float* M = stage + (RDM + wq) * LD;
      float s0 = 0.f, s1 = 0.f;
#pragma unroll 4
      for (int k = 0; k < TILE; k += 4) {
        const float4 hv = *reinterpret_cast<const float4*>(Hh + k);
        const float4 m = *reinterpret_cast<const float4*>(M + k);
        s0 = fmaf(hv.x, m.x, s0); s1 = fmaf(hv.y, m.y, s1);
        s0 = fmaf(hv.z, m.z, s0); s1 = fmaf(hv.w, m.w, s1);
      }
      accA += (double)(s0 + s1);
    } else if (wq == 3) {
      const float* Dr = stage + (RD2 + lane) * LD;
      float s0 = 0.f;
#pragma unroll 4
      for (int k = 0; k < TILE; k += 4) {
        const float4 d = *reinterpret_cast<const float4*>(Dr + k);
        s0 += (d.x + d.y) + (d.z + d.w);
      }
      accA += (double)s0;
    }
    if (tid < 2 * A) {
      const float* Dr = stage + (RDM + tid) * LD;   // rows DM[0..A-1], DL[0..A-1] are contiguous
      float s0 = 0.f;
#pragma unroll 4
      for (int k = 0; k < TILE; k += 4) {
        const float4 d = *reinterpret_cast<const float4*>(Dr + k);
        s0 += (d.x + d.y) + (d.z + d.w);
      }
      accT += (double)s0;
    }
  }

  __device__ __forceinline__ void accumulate_b(const float* stage, int tid) {
    const int lane = tid & 31, wq = tid >> 5;
    const float* Dr = stage + (RD1 + lane) * LD;
    float sa[OQ + 1];
#pragma unroll
    for (int i = 0; i <= OQ; ++i) sa[i] = 0.f;
#pragma unroll 4
    for (int k = 0; k < TILE; k += 4) {
      const float4 d = *reinterpret_cast<const float4*>(Dr + k);
#pragma unroll
      for (int i = 0; i < OQ; ++i) {
        const int o = wq + 4 * i;
        if (o < O) {
          const float4 xv = *reinterpret_cast<const float4*>(stage + (RX + o) * LD + k);
          sa[i] = fmaf(xv.x, d.x, sa[i]); sa[i] = fmaf(xv.y, d.y, sa[i]);
          sa[i] = fmaf(xv.z, d.z, sa[i]); sa[i] = fmaf(xv.w, d.w, sa[i]);
        }
      }
      if (wq == 3) sa[OQ] += (d.x + d.y) + (d.z + d.w);
    }
#pragma unroll
    for (int i = 0; i <= OQ; ++i) accB[i] += (double)sa[i];
  }

  // out: this block's partial vector [P]; scr: >= 2 * 64 * 16 doubles of shared memory no thread still reads
  __device__ __forceinline__ void write(double* out, double* scr, int tid) {
    const int w1_tile = tid & 63, kh = tid >> 6;
    const int ti = w1_tile >> 3, tj = w1_tile & 7;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) scr[(kh * 64 + w1_tile) * 16 + r * 4 + c] = accW1[r][c];
    __syncthreads();
    if (tid < 64) {
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c)
          out[N::oW1 + (ti + 8 * r) * H + (tj + 8 * c)] = scr[w1_tile * 16 + r * 4 + c] + scr[(64 + w1_tile) * 16 + r * 4 + c];
    }
    const int lane = tid & 31, wq = tid >> 5;
#pragma unroll
    for (int i = 0; i < OQ; ++i) {
      const int o = wq + 4 * i;
      if (o < O) out[N::oW0 + o * H + lane] = accB[i];
    }
    if (wq == 3) {
      out[N::ob0 + lane] = accB[OQ];
      out[N::ob1 + lane] = accA;
    } else if (wq < A) {
      out[N::oWo + lane * A + wq] = accA;
    }
    if (tid < 2 * A) out[N::obo + tid] = accT;   // obo.. then ols.. are contiguous in the flat layout
  }
};

}  // namespace b200rl
