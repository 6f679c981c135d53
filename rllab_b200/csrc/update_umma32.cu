// Surrogate gradient and Fisher-vector product for 32-wide policies with the dense layer chain on the warpgroup tensor
// cores (wgmma.mma_async .tf32, accumulators and A operands in registers) -- the 32-wide sibling of update_umma.cu.
//
// One CTA of 128 threads (one warpgroup) per 128-sample tile, several CTAs resident per SM (persistent over tiles).  The
// warpgroup covers the tile as two 64-row MMA blocks; each thread holds four samples of it in the accumulator fragment
// layout of umma_common.cuh.  The CUDA cores only do what is elementwise per sample (bias, tanh, the distribution math,
// (1 - h^2) factors, the hi/lo operand split) and the sample-axis Gram products (tile_gram.cuh); every dense layer is a
// 128 x 32 x K tensor-core GEMM whose A operand the previous epilogue left in registers:
//
//   GRAD   A  x -> A operand                    MMA  H1pre = X W0                  (K = obs_dim padded to 8)
//          E1 h1 = tanh(H1pre + b0)             MMA  H2pre = H1 W1
//          E2 h2 = tanh(H2pre + b1); mean, log-likelihood, surrogate / KL terms, dmu, dlog_std;
//             d2 = (dmu Wout^T)(1 - h2^2)                                          MMA  D1pre = D2 W1^T
//          E3 d1 = D1pre (1 - h1^2)             Gram products (FP32 pipe)
//   FVP    A  x, cached h1 / h2                 MMA  T1pre = X V0 ; T2pre = H1 V1
//          C  t1 = (T1pre + vb0)(1 - h1^2)                                         MMA  T2pre += T1 W1
//          E  t2 = (T2pre + vb1)(1 - h2^2); mu_dot; dmu = M mu_dot; d2             MMA  D1pre = D2 W1^T
//          G  d1 = D1pre (1 - h1^2)             Gram products
//
// Against update_tile.cu (the same passes with FFMA chains) this removes the 2 200 FMA + 550 weight LDS per sample of the
// layer chain from the issue slots and the LSU.  Precision: the three-pass TF32 split a b ~ a_lo b_hi + a_hi b_lo + a_hi
// b_hi with float32 accumulation (update_umma.cu; 4e-7 of the output scale).  The tensor-core forward is NOT
// bit-identical to the FFMA chain of the rollout / loss kernels: the (loss, KL) triple a gradient pass emits at theta_old
// is -mean(adv) and 0 to ~1e-7 instead of exactly; the forward-only mode (MODE_LOSS) runs the gradient pass's forward
// instruction for instruction, so the two agree bit for bit at equal theta.
//
// Operand formats as update_umma.cu: B = [32 x K] weight image in shared memory, K-major no-swizzle: element (n, k) at
// (k%4)*4 + (n%8)*16 + (n/8)*128 + (k/4)*512 bytes, k = u_kperm(input feature) (LBO 512, SBO 128).
//
// Replaces f_grad / f_Hx_plain of rllab/optimizers/conjugate_gradient_optimizer.py:184-215,22-55 and the gradient half of
// f_opt in rllab/optimizers/first_order_optimizer.py:62-76 for hidden (32,32).
#include "tile_gram.cuh"
#include "umma_common.cuh"

namespace b200rl {

constexpr int V_THREADS = 128, V_TILE = 128, V_LD = V_TILE + 4;
#ifndef B200RL_V_PACKED_GRAM
#define B200RL_V_PACKED_GRAM 1          // dW1 Gram with even / odd packed partial sums (tile_gram.cuh)
#endif
#ifndef B200RL_V_MAXB
#define B200RL_V_MAXB 2                 // resident CTAs per SM of the gradient / Fisher passes: at three (168 registers)
#endif                                  // the gradient pass spills

template <class N, int MODE>
struct Umma32 {
  static constexpr int O = N::O, H = 32, A = N::A;
  static_assert(N::H1 == 32 && N::H2 == 32 && O <= 24, "tensor-core 32-wide kernel: (32,32) nets, obs_dim <= 24");
  static constexpr int KX = ((O + 7) / 8) * 8;                 // obs columns of the X operand, zero padded
  static constexpr int IMG = 32 * 32 * 4, IMGX = 32 * KX * 4;   // bytes of one [32 x K] operand image
  // weight images (hi then lo).  GRAD: W0^T [j][o], W1^T [j][i], W1 [i][j].  FVP: V0^T, V1^T, W1^T, W1.
  // LOSS (forward only): W0^T, W1^T.
  static constexpr int o_bXT = 0, o_bW1T = o_bXT + 2 * IMGX, o_bW1 = o_bW1T + 2 * IMG,
                       o_bV1T = o_bW1 + (MODE == MODE_LOSS ? 0 : 2 * IMG),
                       o_img_end = o_bV1T + (MODE == MODE_FVP ? 2 * IMG : 0);
  // small parameters (floats): GRAD b0[32] b1[32] Wout[32A] bout[A];  FVP vb0[32] vb1[32] Wout[32A] Vout[32A] vbout[A]
  static constexpr int n_small = ((64 + 2 * H * A + A + 3) / 4) * 4;
  static constexpr int o_small = o_img_end, o_stage = o_small + n_small * 4;
  // stage rows; D1 reuses the H2 rows (H2 is dead once part A of the Gram phase has run, D1 only exists after it)
  // (the forward-only loss pass stages nothing)
  static constexpr int rX = 0, rH1 = rX + O, rH2 = rH1 + H, rD1 = rH2, rD2 = rH2 + H, rDM = rD2 + H, rDL = rDM + A,
                       R = (MODE == MODE_LOSS) ? 0 : rDL + A;
  static constexpr int o_red = ((o_stage + R * V_LD * 4 + 15) / 16) * 16;   // 3 x 32 doubles of reduction scratch
  static constexpr size_t bytes = (size_t)o_red + 3 * 32 * 8;
  static_assert(MODE == MODE_LOSS || 2 * 64 * 16 * 8 <= R * V_LD * 4, "stage region must hold the K-half combine scratch");
  static_assert(bytes <= 232448, "does not fit the 227 KB of shared memory");
  // resident CTAs per SM: shared memory (228 KB, 1 KB reserved per CTA), registers (64 K / 128 threads)
  static constexpr int by_smem = (int)((228 * 1024) / (bytes + 1024));
  static constexpr int cap = (MODE == MODE_LOSS) ? 3 : B200RL_V_MAXB;
  static constexpr int MINB = by_smem < cap ? (by_smem < 1 ? 1 : by_smem) : cap;
};

// element (n, k) of a K-major [32 x K] image, byte offset (k: input feature, stored at u_kperm(k))
__device__ __forceinline__ int v_boff(int n, int k) {
  const int kp = u_kperm(k);
  return (kp & 3) * 4 + (n & 7) * 16 + (n >> 3) * 128 + (kp >> 2) * 512;
}

template <class N, int MODE>
__global__ void __launch_bounds__(V_THREADS, (Umma32<N, MODE>::MINB)) update_umma32_kernel(UpdArgs a) {
  using SM = Umma32<N, MODE>;
  constexpr int O = N::O, H = 32, A = N::A, P = N::P, LD = V_LD, KX = SM::KX, KSX = KX / 8;
  extern __shared__ __align__(1024) unsigned char smem[];
  float* small = reinterpret_cast<float*>(smem + SM::o_small);
  float* sb0 = small, *sb1 = small + H, *sWout = small + 2 * H, *sVout = sWout + H * A;   // sVout: FVP only
  float* sbo = (MODE == MODE_FVP) ? sVout + H * A : sWout + H * A;
  float* stage = reinterpret_cast<float*>(smem + SM::o_stage);
  double* red_scratch = reinterpret_cast<double*>(smem + SM::o_red);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, t4 = lane & 3;

  // ---- one-time setup: operand images of the weights, small parameters
  // MODE_GRAD: the chain multiplies by theta (params); MODE_FVP: first layers by the tangent x (xvec), W1 by theta
  for (int e = tid; e < H * H; e += V_THREADS) {
    const int i = e / H, j = e % H;                                         // W1[i][j] (row-major in theta)
    const float w = a.params[N::oW1 + e];
    const float wh = tf32_hi(w);
    *reinterpret_cast<float*>(smem + SM::o_bW1T + v_boff(j, i)) = wh;
    *reinterpret_cast<float*>(smem + SM::o_bW1T + SM::IMG + v_boff(j, i)) = w - wh;
    if constexpr (MODE != MODE_LOSS) {
      *reinterpret_cast<float*>(smem + SM::o_bW1 + v_boff(i, j)) = wh;
      *reinterpret_cast<float*>(smem + SM::o_bW1 + SM::IMG + v_boff(i, j)) = w - wh;
    }
    if constexpr (MODE == MODE_FVP) {
      const float v = (float)a.xvec[N::oW1 + e];
      const float vh = tf32_hi(v);
      *reinterpret_cast<float*>(smem + SM::o_bV1T + v_boff(j, i)) = vh;
      *reinterpret_cast<float*>(smem + SM::o_bV1T + SM::IMG + v_boff(j, i)) = v - vh;
    }
  }
  for (int e = tid; e < KX * H; e += V_THREADS) {
    const int o = e / H, j = e % H;
    float v = 0.f;
    if (o < O) v = (MODE == MODE_FVP) ? (float)a.xvec[N::oW0 + o * H + j] : a.params[N::oW0 + o * H + j];
    const float vh = tf32_hi(v);
    *reinterpret_cast<float*>(smem + SM::o_bXT + v_boff(j, o)) = vh;
    *reinterpret_cast<float*>(smem + SM::o_bXT + SM::IMGX + v_boff(j, o)) = v - vh;
  }
  for (int e = tid; e < H * A; e += V_THREADS) {
    sWout[e] = a.params[N::oWo + e];
    if constexpr (MODE == MODE_FVP) sVout[e] = (float)a.xvec[N::oWo + e];
  }
  for (int e = tid; e < H; e += V_THREADS) {
    sb0[e] = (MODE == MODE_FVP) ? (float)a.xvec[N::ob0 + e] : a.params[N::ob0 + e];
    sb1[e] = (MODE == MODE_FVP) ? (float)a.xvec[N::ob1 + e] : a.params[N::ob1 + e];
  }
  if (tid < A) sbo[tid] = (MODE == MODE_FVP) ? (float)a.xvec[N::obo + tid] : a.params[N::obo + tid];
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes of the images -> visible to wgmma
  __syncthreads();

  TileDist D;
  tile_dist_init<N, MODE>(D, a.params + N::ols, a);

  const uint64_t dXT_hi = u_desc(u_smem_u32(smem + SM::o_bXT), 512, 128), dXT_lo = u_desc(u_smem_u32(smem + SM::o_bXT + SM::IMGX), 512, 128);
  const uint64_t dW1T_hi = u_desc(u_smem_u32(smem + SM::o_bW1T), 512, 128), dW1T_lo = u_desc(u_smem_u32(smem + SM::o_bW1T + SM::IMG), 512, 128);
  const uint64_t dW1_hi = u_desc(u_smem_u32(smem + SM::o_bW1), 512, 128), dW1_lo = u_desc(u_smem_u32(smem + SM::o_bW1 + SM::IMG), 512, 128);
  const uint64_t dV1T_hi = u_desc(u_smem_u32(smem + SM::o_bV1T), 512, 128), dV1T_lo = u_desc(u_smem_u32(smem + SM::o_bV1T + SM::IMG), 512, 128);

  // split GEMM of both 64-row blocks: acc[mb] (+)= f[mb] B, f[mb]: accumulator-ordered A values of KS k-steps
  auto gemm2 = [&](float (&acc)[2][16], auto& f, uint64_t b_hi, uint64_t b_lo, int KS, bool accumulate) {
    constexpr int NV = sizeof(f[0]) / sizeof(float);
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
      uint32_t hi[NV], lo[NV];
      u_to_operand(f[mb], hi, lo);
      wg_split_gemm(acc[mb], hi, lo, b_hi, b_lo, 1024, KS, accumulate);
    }
  };

  TileGram<N, SM::rX, SM::rH1, SM::rH2, SM::rD1, SM::rD2, SM::rDM, LD, B200RL_V_PACKED_GRAM != 0> gram;
  if constexpr (MODE != MODE_LOSS) gram.init();
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;

  const long long ntiles = n_tiles_of(a, V_TILE);
  for (long long ti_ = blockIdx.x; ti_ < ntiles; ti_ += gridDim.x) {
    const long long tile = tile_at(a, ti_);
    // the thread's four samples: rows trow[mb][h] of the tile
    int trow[2][2];
    long long sl[2][2];
    bool inrange[2][2], valid[2][2];
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        trow[mb][h] = mb * 64 + warp * 16 + u_frag_row(2 * h, lane);
        const long long s = tile * V_TILE + trow[mb][h];
        inrange[mb][h] = s < a.B;
        valid[mb][h] = sample_valid(a, s);
        sl[mb][h] = inrange[mb][h] ? s : a.B - 1;
      }
    float accA[2][16], accB[2][16];
    // ================= A: observations -> X operand + stage rows; FVP: cached activations, H1 -> operand
    {
      float xf[2][4 * KSX];
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int i = 0; i < 4 * KSX; ++i) {
          const int o = u_frag_col(i, lane), h = (i >> 1) & 1;
          float x = 0.f;
          if (o < O) {
            x = a.obs[(size_t)o * a.B + sl[mb][h]];
            if constexpr (MODE != MODE_LOSS) stage[(SM::rX + o) * LD + trow[mb][h]] = x;
          }
          xf[mb][i] = x;
        }
      if constexpr (MODE == MODE_FVP) {
        float h1f[2][16];
#pragma unroll
        for (int mb = 0; mb < 2; ++mb)
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int c = u_frag_col(i, lane), h = (i >> 1) & 1;
            h1f[mb][i] = a.h_cache[(size_t)c * a.B + sl[mb][h]];
            stage[(SM::rH1 + c) * LD + trow[mb][h]] = h1f[mb][i];
          }
        wg_fence();
        gemm2(accA, xf, dXT_hi, dXT_lo, KSX, false);                  // X V0
        gemm2(accB, h1f, dV1T_hi, dV1T_lo, 4, false);                 // H1 V1
        wg_commit();
      } else {
        wg_fence();
        gemm2(accA, xf, dXT_hi, dXT_lo, KSX, false);                  // X W0
        wg_commit();
      }
    }
    // GRAD / LOSS: the remaining per-sample inputs, requested while the first GEMM runs
    float act[2][2][A], om[2][2][A], adv_s[2][2];
    if constexpr (MODE != MODE_FVP) {
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int k = 0; k < A; ++k) {
            act[mb][h][k] = a.act[(size_t)k * a.B + sl[mb][h]];
            om[mb][h][k] = a.old_mean[(size_t)k * a.B + sl[mb][h]];
          }
          adv_s[mb][h] = a.adv[sl[mb][h]];
        }
    }
    wg_wait_all();
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
      wg_fence_operand(accA[mb]);
      wg_fence_operand(accB[mb]);
    }
    // ================= E1 / C: first epilogue -> operand of the second GEMM
    {
      float v[2][16];
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int c = u_frag_col(i, lane), h = (i >> 1) & 1;
          if constexpr (MODE != MODE_FVP) {
            v[mb][i] = tanh_f(accA[mb][i] + sb0[c]);
            if constexpr (MODE == MODE_GRAD) {
              stage[(SM::rH1 + c) * LD + trow[mb][h]] = v[mb][i];
              if (a.h_cache != nullptr && inrange[mb][h]) a.h_cache[(size_t)c * a.B + sl[mb][h]] = v[mb][i];
            }
          } else {
            const float h1 = stage[(SM::rH1 + c) * LD + trow[mb][h]];
            v[mb][i] = (accA[mb][i] + sb0[c]) * (1.0f - h1 * h1);                                    // t1
          }
        }
      wg_fence();
      gemm2(accB, v, dW1T_hi, dW1T_lo, 4, MODE == MODE_FVP);          // H1 W1  |  += T1 W1
      wg_commit();
    }
    float h2f[2][16];
    if constexpr (MODE == MODE_FVP) {             // cached h2, requested while the GEMM runs
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int i = 0; i < 16; ++i)
          h2f[mb][i] = a.h_cache[(size_t)(H + u_frag_col(i, lane)) * a.B + sl[mb][(i >> 1) & 1]];
    }
    wg_wait_all();
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) wg_fence_operand(accB[mb]);
    // ================= E2 / E: second epilogue -> dmu, d2
    {
      float md[2][2][A];
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int k = 0; k < A; ++k) md[mb][h][k] = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int c = u_frag_col(i, lane), h = (i >> 1) & 1;
          if constexpr (MODE != MODE_FVP) {
            h2f[mb][i] = tanh_f(accB[mb][i] + sb1[c]);
            if constexpr (MODE == MODE_GRAD) {
              stage[(SM::rH2 + c) * LD + trow[mb][h]] = h2f[mb][i];
              if (a.h_cache != nullptr && inrange[mb][h]) a.h_cache[(size_t)(H + c) * a.B + sl[mb][h]] = h2f[mb][i];
            }
#pragma unroll
            for (int k = 0; k < A; ++k) md[mb][h][k] = fmaf(h2f[mb][i], sWout[c * A + k], md[mb][h][k]);
          } else {
            stage[(SM::rH2 + c) * LD + trow[mb][h]] = h2f[mb][i];
            const float t2 = (accB[mb][i] + sb1[c]) * (1.0f - h2f[mb][i] * h2f[mb][i]);
#pragma unroll
            for (int k = 0; k < A; ++k)
              md[mb][h][k] = fmaf(t2, sWout[c * A + k], fmaf(h2f[mb][i], sVout[c * A + k], md[mb][h][k]));
          }
        }
      }
      // the four threads of a row (t4 = 0..3) hold disjoint column sets: combine
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int k = 0; k < A; ++k) {
            md[mb][h][k] += __shfl_xor_sync(0xffffffffu, md[mb][h][k], 1);
            md[mb][h][k] += __shfl_xor_sync(0xffffffffu, md[mb][h][k], 2);
          }
      float dmu[2][2][A];
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = trow[mb][h];
          if constexpr (MODE != MODE_FVP) {
            float z[A], zsq = 0.f, zsq_old = 0.f, kl = 0.f;
#pragma unroll
            for (int k = 0; k < A; ++k) {
              const float mu = sbo[k] + md[mb][h][k];
              z[k] = (act[mb][h][k] - mu) * D.inv_std[k];
              zsq += z[k] * z[k];
              const float zo = (act[mb][h][k] - om[mb][h][k]) * D.inv_std_old[k];
              zsq_old += zo * zo;
              const float dm = om[mb][h][k] - mu;
              kl += (dm * dm + D.var_old[k] - D.var_new[k]) / D.var_new2[k] + D.ls_new[k] - D.ls_old[k];
            }
            const float logp_new = -D.sum_ls_new - 0.5f * zsq - D.half_log2pi_A;
            float w_s, term;
            if (a.loss_kind == B200RL_LOSS_TRPO) {
              const float logp_old = -D.sum_ls_old - 0.5f * zsq_old - D.half_log2pi_A;
              w_s = expf(logp_new - logp_old) * adv_s[mb][h];
              term = -w_s;
            } else {
              w_s = adv_s[mb][h];
              term = -logp_new * adv_s[mb][h];
            }
            if (!valid[mb][h]) { w_s = 0.f; term = 0.f; }
            if (t4 == 0) {
              s_loss += (double)term;
              if (valid[mb][h]) { s_kl += (double)kl; m_kl = fmax(m_kl, (double)kl); }
            }
            if constexpr (MODE == MODE_GRAD) {
#pragma unroll
              for (int k = 0; k < A; ++k) {
                dmu[mb][h][k] = -w_s * z[k] * D.inv_std[k];
                if (t4 == 0) {
                  stage[(SM::rDM + k) * LD + r] = dmu[mb][h][k];
                  stage[(SM::rDL + k) * LD + r] = -w_s * (z[k] * z[k] - 1.0f);
                }
              }
            }
          } else {
#pragma unroll
            for (int k = 0; k < A; ++k) {
              dmu[mb][h][k] = valid[mb][h] ? (sbo[k] + md[mb][h][k]) * D.Mmu[k] : 0.f;
              if (t4 == 0) {
                stage[(SM::rDM + k) * LD + r] = dmu[mb][h][k];
                stage[(SM::rDL + k) * LD + r] = 0.f;
              }
            }
          }
        }
      if constexpr (MODE != MODE_LOSS) {
        float v[2][16];
#pragma unroll
        for (int mb = 0; mb < 2; ++mb)
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int c = u_frag_col(i, lane), h = (i >> 1) & 1;
            float sacc = 0.f;
#pragma unroll
            for (int k = 0; k < A; ++k) sacc = fmaf(dmu[mb][h][k], sWout[c * A + k], sacc);
            v[mb][i] = sacc * (1.0f - h2f[mb][i] * h2f[mb][i]);
            stage[(SM::rD2 + c) * LD + trow[mb][h]] = v[mb][i];
          }
        wg_fence();
        gemm2(accA, v, dW1_hi, dW1_lo, 4, false);                     // D2 W1^T
        wg_commit();
      }
    }
    if constexpr (MODE != MODE_LOSS) {
      __syncthreads();                       // stage rows of the whole tile written
      // ================= Gram part A behind the last GEMM: dW1 = H1^T D2, dWout, db1, dbout, dlog_std (tile_gram.cuh)
      gram.accumulate_a(stage, tid);
      __syncthreads();                       // every thread is done with the H2 rows: D1 may overwrite them
      wg_wait_all();
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) wg_fence_operand(accA[mb]);
      // ================= E3 / G: d1 = D1pre (1 - h1^2)
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int c = u_frag_col(i, lane), r = trow[mb][(i >> 1) & 1];
          const float h1 = stage[(SM::rH1 + c) * LD + r];
          stage[(SM::rD1 + c) * LD + r] = accA[mb][i] * (1.0f - h1 * h1);
        }
      __syncthreads();
      // ================= Gram part B: dW0 = X^T D1, db0
      gram.accumulate_b(stage, tid);
      __syncthreads();
    }
  }

  if constexpr (MODE != MODE_LOSS) {
    double* out = a.partial + (size_t)blockIdx.x * P;
    gram.write(out, reinterpret_cast<double*>(stage), tid);
  }
  if constexpr (MODE != MODE_FVP) {
    // per-block (loss, sum KL | max KL): after the [grid][P] partial vectors (GRAD) or alone (LOSS), as loss_thread_kernel
    if constexpr (MODE == MODE_GRAD) __syncthreads();
    double v[2] = {s_loss, s_kl};
    double mx[1] = {m_kl};
    double* sc = a.partial + (MODE == MODE_GRAD ? (size_t)gridDim.x * P : (size_t)0) + (size_t)blockIdx.x * 3;
    block_reduce_store<2, false>(v, red_scratch, sc);
    block_reduce_store<1, true>(mx, red_scratch, sc + 2);
  }
}

template <class N, int MODE>
static int launch_umma32(const UpdArgs& a, int* grid_out, cudaStream_t st) {
  using SM = Umma32<N, MODE>;
  B200RL_SET_MAX_SMEM((update_umma32_kernel<N, MODE>), SM::bytes);
  long long grid = (long long)num_sms() * SM::MINB;        // persistent: every CTA resident
  const long long ntiles = host_n_tiles(a, V_TILE);
  if (grid > ntiles) grid = ntiles;
  if (grid > MAX_PARTIAL_BLOCKS) grid = MAX_PARTIAL_BLOCKS;
  if (grid < 1) grid = 1;
  update_umma32_kernel<N, MODE><<<(unsigned)grid, V_THREADS, SM::bytes, st>>>(a);
  B200RL_LAUNCH_CHECK("update_umma32_kernel");
  *grid_out = (int)grid;
  return 0;
}

int update_umma32_launch(int mode, int obs_dim, int act_dim, const UpdArgs& a, int* grid_out, int* P_out, int* ols_out,
                         cudaStream_t st) {
  const int h1 = 32, h2 = 32;
  B200RL_DISPATCH_NET_H(32, {
    *P_out = NetT::P;
    *ols_out = NetT::ols;
    int rc = (mode == MODE_GRAD)   ? launch_umma32<NetT, MODE_GRAD>(a, grid_out, st)
             : (mode == MODE_LOSS) ? launch_umma32<NetT, MODE_LOSS>(a, grid_out, st)
                                   : launch_umma32<NetT, MODE_FVP>(a, grid_out, st);
    if (rc) return rc;
  });
  return 0;
}

}  // namespace b200rl
