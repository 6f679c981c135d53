// Surrogate gradient and Fisher-vector product for 64-wide policies with the dense layer chain on the warpgroup tensor
// cores (wgmma.mma_async .tf32: accumulators and A operands in registers, weight images in shared memory).
//
// The description below is the Fisher-vector pass (MODE_FVP).  The gradient pass (MODE_GRAD) runs the same pipeline with
// the forward chain in place of the tangent chain: B  H1pre = X W0;  C  h1 = tanh(H1pre + b0) -> A operand (and the
// activation cache);  D  H2pre = H1 W1;  E  h2 = tanh(H2pre + b1), mean, log-likelihood, surrogate / KL terms, dmu,
// dlog_std, d2;  F, G, H as below.  Its forward is float32-grade, not bit-identical to the FFMA chain of the rollout.
//
// Per 128-sample tile (one CTA of 256 threads = two warpgroups per SM, persistent over tiles; warpgroup w owns samples
// 64 w .. 64 w + 63 of the tile, each thread two of them in the accumulator fragment layout of umma_common.cuh):
//   A   load X and the cached activations H1 (written by b200rl_grad at the same theta) -> A-operand registers (hi + lo
//       words) and -> feature-major fp32 rows in shared memory for the Gram phase
//   B   MMA  T1pre = X V0          (K = obs_dim padded to 8)  and, in the same group,  T2pre = H1 V1
//   C   epilogue: T1 = (T1pre + vb0)(1 - H1^2) -> A operand
//   D   MMA  T2pre += T1 W1
//   E   epilogue: T2 = (T2pre + vb1)(1 - H2^2); mu_dot = T2 Wout + H2 Vout + vbout (CUDA cores, N = A <= 6, the four
//       threads of a row combine by shuffles); dmu = M mu_dot; D2 = (dmu Wout^T)(1 - H2^2) -> A operand + shared-memory rows
//   F   MMA  D1pre = D2 W1^T, and behind it: dWout / dbout partial sums (warp reduce-scatter of h2[j] dmu[k])
//   G   epilogue: D1 = D1pre (1 - H1^2) -> shared-memory rows
//   H   Gram products on the CUDA cores (dW1 = H1^T D2, dW0 = X^T D1, db0, db1) exactly as update_gemm.cu
// i.e. the K = 64 / K = obs_dim GEMMs of the tangent-forward / backward chain move to the tensor cores; the sample-axis
// reductions stay on the FP32 pipe (their operands would need a second, transposed set of hi/lo operand images in shared
// memory, which does not fit next to the weight images).
//
// Precision: float32-grade via the three-pass TF32 split  a b ~ a_lo b_hi + a_hi b_lo + a_hi b_hi  (hi = the word with
// its 13 low mantissa bits cleared, exactly representable in TF32; lo = x - hi, exact in float32), accumulated in float32,
// small terms first.  scripts/tf32_split_study.py: 4e-7 of the output scale, the same as the FFMA chains.
//
// Operand formats: B = [64 x K] weight image in shared memory in the canonical K-major no-swizzle layout (8 rows x 16 B
// core matrices): element (n, k) at (k%4)*4 + (n%8)*16 + (n/8)*128 + (k/4)*1024 bytes with k = u_kperm(input feature).
// TF32 operands exist only K-major, which is why every weight matrix gets its own image (W1 both as [j][i] and [i][j]).
//
// Replaces f_Hx_plain of rllab/optimizers/conjugate_gradient_optimizer.py:22-55 (PerlmutterHvp) for hidden (64,64).
#include "tile_phase_a.cuh"
#include "umma_common.cuh"

namespace b200rl {

constexpr int U_THREADS = 256, U_TILE = 128, U_LD = U_TILE + 4, U_FLUSH = 8;
constexpr int U_KX = 24;   // obs columns of the X weight image (O <= 20 padded with zeros to a multiple of 8)

template <class N, int MODE>
struct UmmaSmem {
  static constexpr int O = N::O, H = 64, A = N::A;
  static_assert(N::H1 == 64 && N::H2 == 64 && O <= U_KX, "tensor-core 64-wide kernel: (64,64) nets, obs_dim <= 24");
  static constexpr int KSX = (O + 7) / 8;                                  // k-steps of the X GEMM
  static constexpr int IMG64 = 64 * 64 * 4, IMGX = 64 * U_KX * 4;            // bytes of one [64 x K] operand image
  // weight images (hi then lo): bW1T [j][i], bV1T [j][i] (FVP only), bW1 [i][j], bV0T [j][o] (GRAD: W0^T)
  static constexpr int o_bW1T = 0, o_bV1T = o_bW1T + 2 * IMG64, o_bW1 = o_bV1T + (MODE == MODE_FVP ? 2 * IMG64 : 0),
                       o_bV0T = o_bW1 + 2 * IMG64;
  static constexpr int o_small = o_bV0T + 2 * IMGX;          // floats: Wout, Vout, vb0 | b0, vb1 | b1, vbout | bout
  static constexpr int n_small = ((2 * H * A + 2 * H + A + 3) / 4) * 4;
  static constexpr int o_stage = o_small + n_small * 4;
  static constexpr int rX = 0, rH1 = rX + O, rD1 = rH1 + H, rD2 = rD1 + H, R = rD2 + H;
  static constexpr int o_red = ((o_stage + R * U_LD * 4 + 15) / 16) * 16;     // 3 x 32 doubles: loss / KL block reduction
  static constexpr size_t bytes = (size_t)o_red + 3 * 32 * 8;
  static_assert(bytes <= 232448, "does not fit the 227 KB of shared memory");
  // dWout / dbout / dlog_std combine scratch, per warp: KG groups of 3 actions x 64 columns, then dbout, dlog_std
  static constexpr int KG = (A + 2) / 3, SCR = KG == 1 ? 200 : 192 * KG + 16, SBO = 192 * KG, SLS = SBO + (KG == 1 ? 4 : 8);
  static_assert(A <= 6, "act_dim <= 6");
  static_assert(8 * SCR * 4 <= H * U_LD * 4, "the D1 rows must hold the dWout / dbout combine scratch");
};

// element (n, k) of a K-major [64 x K] image, byte offset (k: input feature, stored at u_kperm(k))
__device__ __forceinline__ int u_boff(int n, int k) {
  const int kp = u_kperm(k);
  return (kp & 3) * 4 + (n & 7) * 16 + (n >> 3) * 128 + (kp >> 2) * 1024;
}

template <class N, int MODE>
__global__ void __launch_bounds__(U_THREADS, 1) update_umma64_kernel(UpdArgs a) {
  using SM = UmmaSmem<N, MODE>;
  constexpr int O = N::O, H = 64, A = N::A, P = N::P, LD = U_LD, KSX = SM::KSX;
  extern __shared__ __align__(1024) unsigned char smem[];
  float* small = reinterpret_cast<float*>(smem + SM::o_small);
  float* sWout = small, *sVout = small + H * A, *svb0 = small + 2 * H * A, *svb1 = svb0 + H, *svbo = svb1 + H;
  float* stage = reinterpret_cast<float*>(smem + SM::o_stage);
  double* red_scratch = reinterpret_cast<double*>(smem + SM::o_red);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, t4 = lane & 3;
  const int row0 = (warp >> 2) * 64 + (warp & 3) * 16;                       // this warp's 16 rows of the tile

  // ---- one-time setup: operand images of the weights, small parameters
  for (int e = tid; e < H * H; e += U_THREADS) {
    const int i = e / H, j = e % H;                                         // W1[i][j] (row-major in theta)
    const float w = a.params[N::oW1 + e];
    const float wh = tf32_hi(w);
    *reinterpret_cast<float*>(smem + SM::o_bW1T + u_boff(j, i)) = wh;
    *reinterpret_cast<float*>(smem + SM::o_bW1T + SM::IMG64 + u_boff(j, i)) = w - wh;
    if constexpr (MODE == MODE_FVP) {
      const float v = (float)a.xvec[N::oW1 + e];
      const float vh = tf32_hi(v);
      *reinterpret_cast<float*>(smem + SM::o_bV1T + u_boff(j, i)) = vh;
      *reinterpret_cast<float*>(smem + SM::o_bV1T + SM::IMG64 + u_boff(j, i)) = v - vh;
    }
    *reinterpret_cast<float*>(smem + SM::o_bW1 + u_boff(i, j)) = wh;
    *reinterpret_cast<float*>(smem + SM::o_bW1 + SM::IMG64 + u_boff(i, j)) = w - wh;
  }
  for (int e = tid; e < U_KX * H; e += U_THREADS) {
    const int o = e / H, j = e % H;
    float v = 0.f;
    if (o < O) v = (MODE == MODE_FVP) ? (float)a.xvec[N::oW0 + o * H + j] : a.params[N::oW0 + o * H + j];
    const float vh = tf32_hi(v);
    *reinterpret_cast<float*>(smem + SM::o_bV0T + u_boff(j, o)) = vh;
    *reinterpret_cast<float*>(smem + SM::o_bV0T + SM::IMGX + u_boff(j, o)) = v - vh;
  }
  for (int e = tid; e < H * A; e += U_THREADS) {
    sWout[e] = a.params[N::oWo + e];
    sVout[e] = (MODE == MODE_FVP) ? (float)a.xvec[N::oWo + e] : 0.f;
  }
  for (int e = tid; e < H; e += U_THREADS) {      // GRAD: the biases themselves
    svb0[e] = (MODE == MODE_FVP) ? (float)a.xvec[N::ob0 + e] : a.params[N::ob0 + e];
    svb1[e] = (MODE == MODE_FVP) ? (float)a.xvec[N::ob1 + e] : a.params[N::ob1 + e];
  }
  if (tid < A) svbo[tid] = (MODE == MODE_FVP) ? (float)a.xvec[N::obo + tid] : a.params[N::obo + tid];
  double* out = a.partial + (size_t)blockIdx.x * P;
  for (int i = tid; i < P; i += U_THREADS) out[i] = 0.0;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes of the images -> visible to wgmma
  __syncthreads();

  TileDist D;
  tile_dist_init<N, MODE>(D, a.params + N::ols, a);
  const uint64_t dW1T_hi = u_desc(u_smem_u32(smem + SM::o_bW1T), 1024, 128), dW1T_lo = u_desc(u_smem_u32(smem + SM::o_bW1T + SM::IMG64), 1024, 128);
  const uint64_t dV1T_hi = u_desc(u_smem_u32(smem + SM::o_bV1T), 1024, 128), dV1T_lo = u_desc(u_smem_u32(smem + SM::o_bV1T + SM::IMG64), 1024, 128);
  const uint64_t dW1_hi = u_desc(u_smem_u32(smem + SM::o_bW1), 1024, 128), dW1_lo = u_desc(u_smem_u32(smem + SM::o_bW1 + SM::IMG64), 1024, 128);
  const uint64_t dV0T_hi = u_desc(u_smem_u32(smem + SM::o_bV0T), 1024, 128), dV0T_lo = u_desc(u_smem_u32(smem + SM::o_bV0T + SM::IMGX), 1024, 128);

  // ---- Gram ownership (as update_gemm.cu, 256 threads: one 4x4 tile of dW1 per thread)
  const int ti = tid / 16, tj = tid % 16;
  float2 gW1[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) gW1[r][c] = make_float2(0.f, 0.f);
  // small outputs, all 256 threads: thread (j = tid % 64, quarter = tid / 64) owns dW0[o][j] for the quarter's obs rows;
  // quarter 0 also sums db0[j] (the D1 row it streams anyway), quarter 1 db1[j] (one extra row)
  constexpr int OH = (O + 3) / 4;
  const int sj = tid & 63, soh = tid >> 6;
  float2 gS[OH + 1];
#pragma unroll
  for (int k = 0; k <= OH; ++k) gS[k] = make_float2(0.f, 0.f);
  // dWout: the thread's 16 columns x 3 actions (flat c * 3 + k, c = 2 (column block) + column parity) are reduce-scattered
  // over the eight row lanes of the warp; lane keeps flat indices wo_base .. wo_base + 5 (per group g of 3 actions)
  constexpr int KG = SM::KG;
  float gWo[KG][6];
#pragma unroll
  for (int g = 0; g < KG; ++g)
#pragma unroll
    for (int r = 0; r < 6; ++r) gWo[g][r] = 0.f;
  const int wo_base = ((lane >> 4) & 1) * 24 + ((lane >> 3) & 1) * 12 + ((lane >> 2) & 1) * 6;
  float gbo[A], gls[A];               // dbout, dlog_std (GRAD): lane 0 of every warp
#pragma unroll
  for (int k = 0; k < A; ++k) { gbo[k] = 0.f; gls[k] = 0.f; }
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;   // GRAD: surrogate / KL terms, counted by the t4 == 0 thread of a row

  auto flush = [&]() {
    {
      double t[4][4];                          // loads first, then stores
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) t[r][c] = out[N::oW1 + (ti + 16 * r) * H + (tj + 16 * c)];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          out[N::oW1 + (ti + 16 * r) * H + (tj + 16 * c)] = t[r][c] + (double)(gW1[r][c].x + gW1[r][c].y);
          gW1[r][c] = make_float2(0.f, 0.f);
        }
    }
    {
      double t[OH + 1];
#pragma unroll
      for (int oo = 0; oo < OH; ++oo) {
        const int o = soh * OH + oo;
        t[oo] = o < O ? out[N::oW0 + o * H + sj] : 0.0;
      }
      t[OH] = soh == 0 ? out[N::ob0 + sj] : (soh == 1 ? out[N::ob1 + sj] : 0.0);
#pragma unroll
      for (int oo = 0; oo < OH; ++oo) {
        const int o = soh * OH + oo;
        if (o < O) out[N::oW0 + o * H + sj] = t[oo] + (double)(gS[oo].x + gS[oo].y);
      }
      if (soh == 0) out[N::ob0 + sj] = t[OH] + (double)(gS[OH].x + gS[OH].y);
      if (soh == 1) out[N::ob1 + sj] = t[OH] + (double)(gS[OH].x + gS[OH].y);
    }
#pragma unroll
    for (int k = 0; k <= OH; ++k) gS[k] = make_float2(0.f, 0.f);
    // dWout / dbout / dlog_std: the eight warps hold partial sums of the same entries -> combine through the (idle) D1
    // rows in fixed warp order.  scr[warp][SCR]: [192 g + col * 3 + k] dWout (action 3 g + k), [SBO + k] dbout,
    // [SLS + k] dlog_std
    constexpr int SCR = SM::SCR, SBO = SM::SBO, SLS = SM::SLS;
    float* scr = stage + SM::rD1 * LD;
#pragma unroll
    for (int g = 0; g < KG; ++g)
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        const int f = wo_base + r, c = f / 3, k = f % 3;
        if (3 * g + k < A) scr[warp * SCR + 192 * g + (8 * (c >> 1) + 2 * t4 + (c & 1)) * 3 + k] = gWo[g][r];
      }
    if (lane == 0)
#pragma unroll
      for (int k = 0; k < A; ++k) {
        scr[warp * SCR + SBO + k] = gbo[k];
        scr[warp * SCR + SLS + k] = gls[k];
      }
    __syncthreads();
    auto sum8 = [&](int idx) {
      return ((scr[0 * SCR + idx] + scr[1 * SCR + idx]) + (scr[2 * SCR + idx] + scr[3 * SCR + idx])) +
             ((scr[4 * SCR + idx] + scr[5 * SCR + idx]) + (scr[6 * SCR + idx] + scr[7 * SCR + idx]));
    };
    if constexpr (H * A + 2 * A <= U_THREADS) {
      if (tid < H * A) {
        const int col = tid / A, k = tid % A;
        out[N::oWo + col * A + k] += (double)sum8(col * 3 + k);
      } else if (tid < H * A + A) {
        const int k = tid - H * A;
        out[N::obo + k] += (double)sum8(SBO + k);
      } else if (is_grad_mode(MODE) && tid < H * A + 2 * A) {
        const int k = tid - H * A - A;
        out[N::ols + k] += (double)sum8(SLS + k);
      }
    } else {
      for (int e = tid; e < H * A + 2 * A; e += U_THREADS) {
        if (e < H * A) {
          const int col = e / A, k = e % A;
          out[N::oWo + col * A + k] += (double)sum8(192 * (k / 3) + col * 3 + k % 3);
        } else if (e < H * A + A) {
          const int k = e - H * A;
          out[N::obo + k] += (double)sum8(SBO + k);
        } else if (is_grad_mode(MODE)) {
          const int k = e - H * A - A;
          out[N::ols + k] += (double)sum8(SLS + k);
        }
      }
    }
#pragma unroll
    for (int g = 0; g < KG; ++g)
#pragma unroll
      for (int r = 0; r < 6; ++r) gWo[g][r] = 0.f;
#pragma unroll
    for (int k = 0; k < A; ++k) { gbo[k] = 0.f; gls[k] = 0.f; }
    __syncthreads();
  };

  const long long ntiles = n_tiles_of(a, U_TILE);
  int since_flush = 0;
  for (long long ti_ = blockIdx.x; ti_ < ntiles; ti_ += gridDim.x) {
    const long long tile = tile_at(a, ti_);
    long long sl[2];
    bool valid[2], inrange[2];
    int trow[2];                               // the thread's two rows inside the tile
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      trow[h] = row0 + u_frag_row(2 * h, lane);
      const long long s = tile * U_TILE + trow[h];
      inrange[h] = s < a.B;
      valid[h] = sample_valid(a, s);
      sl[h] = inrange[h] ? s : a.B - 1;
    }
    // ================= A: loads; X / H1 -> A operands + feature-major rows
    float accA[32], accB[32];
    {
      float xf[4 * KSX];
#pragma unroll
      for (int i = 0; i < 4 * KSX; ++i) {
        const int o = u_frag_col(i, lane), h = (i >> 1) & 1;
        float x = 0.f;
        if (o < O) {
          x = a.obs[(size_t)o * a.B + sl[h]];
          stage[(SM::rX + o) * LD + trow[h]] = x;
        }
        xf[i] = x;
      }
      uint32_t xhi[4 * KSX], xlo[4 * KSX];
      u_to_operand(xf, xhi, xlo);
      // ================= B: T1pre = X V0 ; T2pre = H1 V1
      if constexpr (MODE == MODE_FVP) {
        float h1f[32];
        const float* hc = a.h_cache;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int c = u_frag_col(i, lane), h = (i >> 1) & 1;
          h1f[i] = hc[(size_t)c * a.B + sl[h]];
          stage[(SM::rH1 + c) * LD + trow[h]] = h1f[i];
        }
        uint32_t hhi[32], hlo[32];
        u_to_operand(h1f, hhi, hlo);
        wg_fence();
        wg_split_gemm(accA, xhi, xlo, dV0T_hi, dV0T_lo, 2048, KSX, false);      // X V0
        wg_split_gemm(accB, hhi, hlo, dV1T_hi, dV1T_lo, 2048, 8, false);        // H1 V1
        wg_commit();
        wg_wait_all();
      } else {
        wg_fence();
        wg_split_gemm(accA, xhi, xlo, dV0T_hi, dV0T_lo, 2048, KSX, false);      // GRAD: X W0
        wg_commit();
      }
    }
    // GRAD: the remaining per-sample inputs, requested while the first GEMM runs
    float act[2][A], om[2][A], adv_s[2] = {0.f, 0.f};
    if constexpr (is_grad_mode(MODE)) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int k = 0; k < A; ++k) {
          act[h][k] = a.act[(size_t)k * a.B + sl[h]];
          om[h][k] = a.old_mean[(size_t)k * a.B + sl[h]];
        }
        adv_s[h] = a.adv[sl[h]];
      }
      wg_wait_all();
    }
    wg_fence_operand(accA);
    wg_fence_operand(accB);
    // ================= C: T1 = (T1pre + vb0)(1 - H1^2) -> A operand  |  GRAD: h1 = tanh(H1pre + b0)
    {
      float tf[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int c = u_frag_col(i, lane), h = (i >> 1) & 1;
        if constexpr (MODE == MODE_FVP) {
          const float h1 = stage[(SM::rH1 + c) * LD + trow[h]];
          tf[i] = (accA[i] + svb0[c]) * (1.0f - h1 * h1);
        } else {
          tf[i] = tanh_f(accA[i] + svb0[c]);
          stage[(SM::rH1 + c) * LD + trow[h]] = tf[i];
          if (a.h_cache != nullptr && inrange[h]) a.h_cache[(size_t)c * a.B + sl[h]] = tf[i];
        }
      }
      uint32_t thi[32], tlo[32];
      u_to_operand(tf, thi, tlo);
      // ================= D: T2pre += T1 W1  |  GRAD: H1 W1
      wg_fence();
      wg_split_gemm(accB, thi, tlo, dW1T_hi, dW1T_lo, 2048, 8, MODE == MODE_FVP);
      wg_commit();
    }
    float h2f[32];
    if constexpr (MODE == MODE_FVP) {               // cached h2, requested while the GEMM runs
#pragma unroll
      for (int i = 0; i < 32; ++i) h2f[i] = a.h_cache[(size_t)(H + u_frag_col(i, lane)) * a.B + sl[(i >> 1) & 1]];
    }
    wg_wait_all();
    wg_fence_operand(accB);
    // ================= E: T2, mu_dot, dmu, D2  |  GRAD: h2, mean, surrogate / KL terms, dmu, dlog_std, D2
    float dmu[2][A], dl[2][A];
    {
      float md[2][A];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int k = 0; k < A; ++k) md[h][k] = 0.f;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int c = u_frag_col(i, lane), h = (i >> 1) & 1;
        if constexpr (MODE == MODE_FVP) {
          const float t2 = (accB[i] + svb1[c]) * (1.0f - h2f[i] * h2f[i]);
#pragma unroll
          for (int k = 0; k < A; ++k) md[h][k] = fmaf(t2, sWout[c * A + k], fmaf(h2f[i], sVout[c * A + k], md[h][k]));
        } else {
          h2f[i] = tanh_f(accB[i] + svb1[c]);
          if (a.h_cache != nullptr && inrange[h]) a.h_cache[(size_t)(H + c) * a.B + sl[h]] = h2f[i];
#pragma unroll
          for (int k = 0; k < A; ++k) md[h][k] = fmaf(h2f[i], sWout[c * A + k], md[h][k]);
        }
      }
      // the four threads of a row (t4 = 0..3) hold disjoint column sets: combine
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int k = 0; k < A; ++k) {
          md[h][k] += __shfl_xor_sync(0xffffffffu, md[h][k], 1);
          md[h][k] += __shfl_xor_sync(0xffffffffu, md[h][k], 2);
        }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if constexpr (MODE == MODE_FVP) {
#pragma unroll
          for (int k = 0; k < A; ++k) {
            dmu[h][k] = valid[h] ? (svbo[k] + md[h][k]) * D.Mmu[k] : 0.f;
            dl[h][k] = 0.f;
          }
        } else {
          float z[A], dmk[A], zsq = 0.f, zsq_old = 0.f, kl = 0.f;
#pragma unroll
          for (int k = 0; k < A; ++k) {
            const float mu = svbo[k] + md[h][k];
            z[k] = (act[h][k] - mu) * D.inv_std[k];
            zsq += z[k] * z[k];
            const float zo = (act[h][k] - om[h][k]) * D.inv_std_old[k];
            zsq_old += zo * zo;
            const float dm = om[h][k] - mu;
            dmk[k] = dm;
            kl += (dm * dm + D.var_old[k] - D.var_new[k]) / D.var_new2[k] + D.ls_new[k] - D.ls_old[k];
          }
          const float logp_new = -D.sum_ls_new - 0.5f * zsq - D.half_log2pi_A;
          float w_s, term;
          if (a.loss_kind == B200RL_LOSS_TRPO) {
            const float logp_old = -D.sum_ls_old - 0.5f * zsq_old - D.half_log2pi_A;
            w_s = expf(logp_new - logp_old) * adv_s[h];
            term = -w_s;
          } else {
            w_s = adv_s[h];
            term = -logp_new * adv_s[h];
          }
          if (!valid[h]) { w_s = 0.f; term = 0.f; }
          if (t4 == 0) {
            s_loss += (double)term;
            if (valid[h]) { s_kl += (double)kl; m_kl = fmax(m_kl, (double)kl); }
          }
#pragma unroll
          for (int k = 0; k < A; ++k) {
            dmu[h][k] = -w_s * z[k] * D.inv_std[k];
            dl[h][k] = -w_s * (z[k] * z[k] - 1.0f);
            if constexpr (MODE == MODE_GRAD_KL) {
              if (valid[h]) add_kl_penalty(a.penalty, dmk[k], D.var_new[k], D.var_new2[k], D.var_old[k], dmu[h][k], dl[h][k]);
            }
          }
        }
      }
      float d2f[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int c = u_frag_col(i, lane), h = (i >> 1) & 1;
        float sacc = 0.f;
#pragma unroll
        for (int k = 0; k < A; ++k) sacc = fmaf(dmu[h][k], sWout[c * A + k], sacc);
        d2f[i] = sacc * (1.0f - h2f[i] * h2f[i]);
        stage[(SM::rD2 + c) * LD + trow[h]] = d2f[i];
      }
      uint32_t dhi[32], dlo[32];
      u_to_operand(d2f, dhi, dlo);
      // ================= F: D1pre = D2 W1^T
      wg_fence();
      wg_split_gemm(accA, dhi, dlo, dW1_hi, dW1_lo, 2048, 8, false);
      wg_commit();
    }
    // behind the GEMM: warp reduce-scatter of h2[j] * dmu[k] over the 16 rows of this warp (flat (c, k) index, 48 values:
    // 24 + 12 + 6 shuffles), once per group g of 3 actions; lane ends with the sums of flat indices wo_base .. wo_base + 5
#pragma unroll
    for (int g = 0; g < KG; ++g) {
      float dm3[2][3];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int k = 0; k < 3; ++k) dm3[h][k] = 3 * g + k < A ? dmu[h][3 * g + k] : 0.f;
      auto val = [&](int f) {
        const int c = f / 3, k = f % 3, i = 4 * (c >> 1) + (c & 1);
        return h2f[i] * dm3[0][k] + h2f[i + 2] * dm3[1][k];
      };
      float pr[24];
#pragma unroll
      for (int i = 0; i < 24; ++i) {
        const bool up = (lane >> 4) & 1;
        const float plo = val(i), phi = val(24 + i);
        pr[i] = (up ? phi : plo) + __shfl_xor_sync(0xffffffffu, up ? plo : phi, 16);
      }
#pragma unroll
      for (int i = 0; i < 12; ++i) {
        const bool up = (lane >> 3) & 1;
        pr[i] = (up ? pr[12 + i] : pr[i]) + __shfl_xor_sync(0xffffffffu, up ? pr[i] : pr[12 + i], 8);
      }
#pragma unroll
      for (int i = 0; i < 6; ++i) {
        const bool up = (lane >> 2) & 1;
        gWo[g][i] += (up ? pr[6 + i] : pr[i]) + __shfl_xor_sync(0xffffffffu, up ? pr[i] : pr[6 + i], 4);
      }
    }
    {
#pragma unroll
      for (int k = 0; k < A; ++k) {
        const float sdm = warp_sum(t4 == 0 ? dmu[0][k] + dmu[1][k] : 0.f);
        if (lane == 0) gbo[k] += sdm;
        if constexpr (is_grad_mode(MODE)) {
          const float sdl = warp_sum(t4 == 0 ? dl[0][k] + dl[1][k] : 0.f);
          if (lane == 0) gls[k] += sdl;
        }
      }
    }
    // ================= G: D1 = D1pre (1 - H1^2) -> rows
    wg_wait_all();
    wg_fence_operand(accA);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int c = u_frag_col(i, lane), h = (i >> 1) & 1;
      const float h1 = stage[(SM::rH1 + c) * LD + trow[h]];
      stage[(SM::rD1 + c) * LD + trow[h]] = accA[i] * (1.0f - h1 * h1);
    }
    __syncthreads();
    // ================= H: Gram products over the tile (FP32 pipe)
    {
      // while the FP32 pipe works on this tile, pull the next tile's rows into L2 (its loads are otherwise fully exposed)
      const long long nti = ti_ + gridDim.x;
      if (nti < ntiles) {
        const int q = warp & 3, hf = warp >> 2, j0 = hf * 32;
        const long long ns = tile_at(a, nti) * U_TILE + q * 32;      // one 128 B line per (row, warp): lane 0 fetches it
        if (lane == 0 && ns < a.B) {
          const float* hcn = a.h_cache + ns;
          if constexpr (MODE == MODE_FVP) {
#pragma unroll 8
            for (int c = 0; c < 32; ++c) {
              asm volatile("prefetch.global.L2 [%0];" ::"l"(hcn + (size_t)(j0 + c) * a.B));
              asm volatile("prefetch.global.L2 [%0];" ::"l"(hcn + (size_t)(H + j0 + c) * a.B));
            }
          }
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const int o = hf * 16 + c;
            if (o < O) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.obs + (size_t)o * a.B + ns));
          }
        }
      }
    }
    {
      const float* Ur = stage + (SM::rH1 + ti) * LD;
      const float* Vr = stage + (SM::rD2 + tj) * LD;
#pragma unroll 2
      for (int k = 0; k < U_TILE; k += 4) {
        float4 u[4], v[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) u[r] = *reinterpret_cast<const float4*>(Ur + r * 16 * LD + k);
#pragma unroll
        for (int c = 0; c < 4; ++c) v[c] = *reinterpret_cast<const float4*>(Vr + c * 16 * LD + k);
        gram_4x4(u, v, gW1);
      }
      {
        const float* Dr = stage + (SM::rD1 + sj) * LD;
        const float* D2r = stage + (SM::rD2 + sj) * LD;
#pragma unroll 2
        for (int k = 0; k < U_TILE; k += 4) {
          const float4 d = *reinterpret_cast<const float4*>(Dr + k);
#pragma unroll
          for (int oo = 0; oo < OH; ++oo) {
            const int o = soh * OH + oo;
            if (o < O) {
              const float4 xv = *reinterpret_cast<const float4*>(stage + (SM::rX + o) * LD + k);
              gram_fma4(xv, d, gS[oo]);
            }
          }
          if (soh == 0) gS[OH].x += (d.x + d.y) + (d.z + d.w);
          if (soh == 1) {
            const float4 e = *reinterpret_cast<const float4*>(D2r + k);
            gS[OH].x += (e.x + e.y) + (e.z + e.w);
          }
        }
      }
    }
    __syncthreads();
    if (++since_flush == U_FLUSH) {
      flush();
      since_flush = 0;
    }
  }
  if (since_flush > 0) flush();
  if constexpr (is_grad_mode(MODE)) {
    __syncthreads();
    double v[2] = {s_loss, s_kl};
    double mx[1] = {m_kl};
    double* sc = a.partial + (size_t)gridDim.x * P + (size_t)blockIdx.x * 3;
    block_reduce_store<2, false>(v, red_scratch, sc);
    block_reduce_store<1, true>(mx, red_scratch, sc + 2);
  }
}

template <class N, int MODE>
static int launch_umma(const UpdArgs& a, int* grid_out, cudaStream_t st) {
  using SM = UmmaSmem<N, MODE>;
  B200RL_SET_MAX_SMEM((update_umma64_kernel<N, MODE>), SM::bytes);
  long long grid = num_sms();                      // one CTA per SM (up to 220 KB of shared memory)
  const long long ntiles = host_n_tiles(a, U_TILE);
  if (grid > ntiles) grid = ntiles;
  if (grid < 1) grid = 1;
  update_umma64_kernel<N, MODE><<<(unsigned)grid, U_THREADS, SM::bytes, st>>>(a);
  B200RL_LAUNCH_CHECK("update_umma64_kernel");
  *grid_out = (int)grid;
  return 0;
}

int update_umma64_launch(int mode, int obs_dim, int act_dim, const UpdArgs& a, int* grid_out, int* P_out, int* ols_out,
                         cudaStream_t st) {
  const int h1 = 64, h2 = 64;
  B200RL_DISPATCH_NET_H(64, {
    *P_out = NetT::P;
    *ols_out = NetT::ols;
    int rc = (mode == MODE_GRAD)      ? launch_umma<NetT, MODE_GRAD>(a, grid_out, st)
             : (mode == MODE_GRAD_KL) ? launch_umma<NetT, MODE_GRAD_KL>(a, grid_out, st)
                                      : launch_umma<NetT, MODE_FVP>(a, grid_out, st);
    if (rc) return rc;
  });
  return 0;
}

}  // namespace b200rl
