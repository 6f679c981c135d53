// Surrogate gradient and Fisher-vector product for 32-wide policies with the dense layer chain on the warpgroup tensor
// cores (wgmma.mma_async .tf32, accumulators and A operands in registers) -- the 32-wide sibling of update_umma.cu.
//
// One persistent CTA per SM of NWG warpgroups; each warpgroup takes 128-sample tiles and covers a tile as two 64-row MMA
// blocks, each thread holding two samples of a block in the accumulator fragment layout of umma_common.cuh.  The loss and
// Fisher passes run the chain below over both blocks at once; the gradient family of act_dim 1 runs it for one block and
// then for the other (Umma32::BLK), which halves the registers and stage rows a warpgroup holds, so that four warpgroups
// fit on an SM.  The CUDA cores only do what is elementwise per sample (bias, tanh, the distribution math, (1 - h^2)
// factors, the hi/lo operand split) and the sample-axis Gram products (tile_gram.cuh); every dense layer is a
// 64 x 32 x K tensor-core GEMM per block whose A operand the previous epilogue left in registers:
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
#ifndef B200RL_V_NWG_GRAD
#define B200RL_V_NWG_GRAD 4             // warpgroups per SM of the block-at-a-time gradient pass (Umma32::BLK)
#endif

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
  // BLK: the gradient family of act_dim 1 runs the whole chain (GEMMs, epilogues, Gram) for one 64-row MMA block of the
  // tile and then for the other: half the accumulator, operand and activation registers and half the stage rows of a
  // pass over both blocks, so that more warpgroups fit on an SM.  NB: 64-row blocks per pass of the chain.
  static constexpr bool BLK = is_grad_mode(MODE) && A == 1;
  static constexpr int NB = BLK ? 1 : 2;
  // warpgroups of the one CTA per SM: registers (64 K / 128 per warpgroup) and shared memory (227 KB; the images and
  // small parameters are staged once per CTA).  BLK: B200RL_V_NWG_GRAD (DESIGN section 6).  Three (168 registers) for
  // the loss pass; two for the gradient pass of act_dim 2 / 3 (at 168 registers it spills) and for the Fisher pass
  // (240+ registers).  Every shape fits its count in shared memory.
  static constexpr int NWG = BLK ? B200RL_V_NWG_GRAD : MODE == MODE_LOSS ? 3 : 2;
  // SEP_D1: D1 has stage rows of its own (BLK at up to four warpgroups, where they fit in shared memory)
  static constexpr bool SEP_D1 = BLK && NWG <= 4;
  // stage rows of one pass (NB * 64 samples, pitch LD; LD mod 32 = 4 keeps the epilogue stores and the Gram's LDS.128
  // conflict-free).  SEP_D1: D1 has rows of its own, so that E3 runs before the Gram phase and both Gram parts run
  // behind one barrier.  Otherwise D1 reuses the H2 rows (H2 is dead once part A of the Gram phase has run, D1 only
  // exists after it).  X is read from the input ring.  The forward-only loss pass stages nothing.
  static constexpr int LD = NB * 64 + 4;
  static constexpr int rH1 = 0, rH2 = rH1 + H, rD2 = rH2 + H, rDM = rD2 + H, rDL = rDM + A,
                       rD1 = SEP_D1 ? rDL + A : rH2, R = (MODE == MODE_LOSS) ? 0 : SEP_D1 ? rD1 + H : rDL + A;
  // input ring: two slots of RR rows (pitch V_LD) -- obs[o], then (GRAD / LOSS) act[k], old_mean[k], adv -- filled by
  // cp.async one tile ahead of the warpgroup that reads them
  static constexpr int RR = O + (MODE == MODE_FVP ? 0 : 2 * A + 1), qX = 0, qAct = O, qOm = O + A, qAdv = O + 2 * A;
  // every warpgroup owns one region: stage rows, 3 x 32 doubles of reduction scratch, input ring
  static constexpr int w_red = ((R * LD * 4 + 15) / 16) * 16, w_ring = w_red + 3 * 32 * 8,
                       w_bytes = w_ring + 2 * RR * V_LD * 4;
  // distribution constants of the pass (TileDist), set up once per CTA: E2 reads them from shared memory rather than
  // holding them in registers across the tile loop
  static constexpr int o_dist = ((o_stage + 15) / 16) * 16;
  static constexpr int o_wg = ((o_dist + (int)sizeof(TileDist) + 15) / 16) * 16;
  static_assert(MODE == MODE_LOSS || BLK || 2 * 64 * 16 * 8 <= R * LD * 4, "stage region must hold the K-half combine scratch");
  static constexpr size_t bytes = (size_t)o_wg + (size_t)NWG * w_bytes;
  static_assert(bytes <= 232448, "does not fit the 227 KB of shared memory");
};

// named barrier of one warpgroup (id 0 is __syncthreads)
__device__ __forceinline__ void v_wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory"); }

// one warpgroup's fixed-order reduction of K per-thread values, stored to out[0..K) (block_reduce_store for 128 threads)
template <int K, bool IS_MAX>
__device__ __forceinline__ void v_wg_reduce_store(const double (&v)[K], double* scratch, double* out, int tid, int wg) {
  const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double s = IS_MAX ? warp_max(v[k]) : warp_sum(v[k]);
    if (lane == 0) scratch[k * 32 + warp] = s;
  }
  v_wg_sync(wg);
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double s = lane < 4 ? scratch[k * 32 + lane] : (IS_MAX ? -1.0e300 : 0.0);
      s = IS_MAX ? warp_max(s) : warp_sum(s);
      if (lane == 0) out[k] = s;
    }
  }
  v_wg_sync(wg);
}

// request the ring rows of `tile` into `slot`: thread t copies sample t of every row (clamped to the last sample of the
// batch, as the reads of a partial tile are), 4 B cp.async each (a row starts anywhere when B is not a multiple of 4)
template <class SMT>
__device__ __forceinline__ void v_ring_load(const UpdArgs& a, float* ring, int slot, long long tile, int tid) {
  long long s = tile * V_TILE + tid;
  if (s >= a.B) s = a.B - 1;
  float* dst = ring + (size_t)slot * SMT::RR * V_LD + tid;
#pragma unroll
  for (int q = 0; q < SMT::RR; ++q) {
    const float* src = q < SMT::qAct ? a.obs + (size_t)q * a.B + s
                       : q < SMT::qOm ? a.act + (size_t)(q - SMT::qAct) * a.B + s
                       : q < SMT::qAdv ? a.old_mean + (size_t)(q - SMT::qOm) * a.B + s
                                       : a.adv + s;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(u_smem_u32(dst + q * V_LD)), "l"(src) : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// element (n, k) of a K-major [32 x K] image, byte offset (k: input feature, stored at u_kperm(k))
__device__ __forceinline__ int v_boff(int n, int k) {
  const int kp = u_kperm(k);
  return (kp & 3) * 4 + (n & 7) * 16 + (n >> 3) * 128 + (kp >> 2) * 512;
}

template <class N, int MODE>
__global__ void __launch_bounds__(V_THREADS * Umma32<N, MODE>::NWG, 1) update_umma32_kernel(UpdArgs a) {
  using SM = Umma32<N, MODE>;
  constexpr int O = N::O, H = 32, A = N::A, P = N::P, RLD = V_LD, LD = SM::LD, KX = SM::KX, KSX = KX / 8, NB = SM::NB;
  extern __shared__ __align__(1024) unsigned char smem[];
  float* small = reinterpret_cast<float*>(smem + SM::o_small);
  float* sb0 = small, *sb1 = small + H, *sWout = small + 2 * H, *sVout = sWout + H * A;   // sVout: FVP only
  float* sbo = (MODE == MODE_FVP) ? sVout + H * A : sWout + H * A;
  constexpr int NWG = SM::NWG, NT = NWG * V_THREADS;
  // warpgroup wg works on its own tiles with its own stage rows and ring; tid, warp: inside the warpgroup
  const int gtid = threadIdx.x, wg = gtid >> 7, tid = gtid & (V_THREADS - 1), warp = tid >> 5, lane = tid & 31, t4 = lane & 3;
  unsigned char* wreg = smem + SM::o_wg + (size_t)wg * SM::w_bytes;
  float* stage = reinterpret_cast<float*>(wreg);
  double* red_scratch = reinterpret_cast<double*>(wreg + SM::w_red);
  float* ring = reinterpret_cast<float*>(wreg + SM::w_ring);

  // ---- one-time setup: operand images of the weights, small parameters
  // MODE_GRAD: the chain multiplies by theta (params); MODE_FVP: first layers by the tangent x (xvec), W1 by theta
  for (int e = gtid; e < H * H; e += NT) {
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
  for (int e = gtid; e < KX * H; e += NT) {
    const int o = e / H, j = e % H;
    float v = 0.f;
    if (o < O) v = (MODE == MODE_FVP) ? (float)a.xvec[N::oW0 + o * H + j] : a.params[N::oW0 + o * H + j];
    const float vh = tf32_hi(v);
    *reinterpret_cast<float*>(smem + SM::o_bXT + v_boff(j, o)) = vh;
    *reinterpret_cast<float*>(smem + SM::o_bXT + SM::IMGX + v_boff(j, o)) = v - vh;
  }
  for (int e = gtid; e < H * A; e += NT) {
    sWout[e] = a.params[N::oWo + e];
    if constexpr (MODE == MODE_FVP) sVout[e] = (float)a.xvec[N::oWo + e];
  }
  for (int e = gtid; e < H; e += NT) {
    sb0[e] = (MODE == MODE_FVP) ? (float)a.xvec[N::ob0 + e] : a.params[N::ob0 + e];
    sb1[e] = (MODE == MODE_FVP) ? (float)a.xvec[N::ob1 + e] : a.params[N::ob1 + e];
  }
  if (gtid < A) sbo[gtid] = (MODE == MODE_FVP) ? (float)a.xvec[N::obo + gtid] : a.params[N::obo + gtid];
  TileDist& D = *reinterpret_cast<TileDist*>(smem + SM::o_dist);
  if (gtid == 0) tile_dist_init<N, MODE>(D, a.params + N::ols, a);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes of the images -> visible to wgmma
  __syncthreads();

  // split GEMM of the pass's 64-row blocks: acc[mb] (+)= f[mb] B, f[mb]: accumulator-ordered A values of KS k-steps; B:
  // the hi / lo weight images at byte offsets o_img, o_img + img of shared memory.  The descriptors are rebuilt from the
  // 32-bit shared-memory base at every GEMM rather than held across the tile loop.
  const uint32_t sbase = u_smem_u32(smem);
  auto gemm = [&](auto& acc, auto& f, int o_img, int img, int KS, bool accumulate) {
    constexpr int NV = sizeof(f[0]) / sizeof(float);
    const uint64_t b_hi = u_desc(sbase + o_img, 512, 128), b_lo = u_desc(sbase + o_img + img, 512, 128);
#pragma unroll
    for (int mb = 0; mb < NB; ++mb) {
      uint32_t hi[NV], lo[NV];
      u_to_operand(f[mb], hi, lo);
      wg_split_gemm(acc[mb], hi, lo, b_hi, b_lo, 1024, KS, accumulate);
    }
  };

  // (RX = 0 is unused: part B gets the X rows of the ring)
  TileGram<N, 0, SM::rH1, SM::rH2, SM::rD1, SM::rD2, SM::rDM, LD, B200RL_V_PACKED_GRAM != 0, NB * 64> gram;
  if constexpr (MODE != MODE_LOSS) gram.init();
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;

  // tiles go to the warpgroups of the grid round-robin: warpgroup vb takes tiles vb, vb + nvb, ...
  const int ntiles = (int)n_tiles_of(a, V_TILE), nvb = gridDim.x * NWG, vb = blockIdx.x * NWG + wg;
  if (vb < ntiles) v_ring_load<SM>(a, ring, 0, tile_at(a, vb), tid);
  int slot = 0;
  for (int ti_ = vb; ti_ < ntiles; ti_ += nvb, slot ^= 1) {
    const long long tile = tile_at(a, ti_);
    // this tile's ring rows have landed (every thread waits for its own copies, the barrier publishes them), and every
    // thread is done with the other slot: the next tile's rows go there while this one computes.  The slot stays valid
    // for the whole tile (the Gram phase reads X from it).
    asm volatile("cp.async.wait_all;" ::: "memory");
    v_wg_sync(wg);
    if (ti_ + nvb < ntiles) v_ring_load<SM>(a, ring, slot ^ 1, tile_at(a, ti_ + nvb), tid);
    // one pass of the chain per NB 64-row blocks, starting at tile row b0; rs: the pass's rows of the ring slot
#pragma unroll 1
    for (int b0 = 0; b0 < V_TILE; b0 += NB * 64) {
      const float* rs = ring + (size_t)slot * SM::RR * RLD + b0;
      // the thread's 2 NB samples: rows trow[mb][h] of the pass (stage and rs columns)
      int trow[NB][2];
      long long sl[NB][2];
      bool inrange[NB][2], valid[NB][2];
#pragma unroll
      for (int mb = 0; mb < NB; ++mb)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          trow[mb][h] = mb * 64 + warp * 16 + u_frag_row(2 * h, lane);
          const long long s = tile * V_TILE + b0 + trow[mb][h];
          inrange[mb][h] = s < a.B;
          valid[mb][h] = sample_valid(a, s);
          sl[mb][h] = inrange[mb][h] ? s : a.B - 1;
        }
      float accA[NB][16], accB[NB][16];
      // ================= A: observations -> X operand; FVP: cached activations, H1 -> operand + stage rows
      {
        float xf[NB][4 * KSX];
#pragma unroll
        for (int mb = 0; mb < NB; ++mb)
#pragma unroll
          for (int i = 0; i < 4 * KSX; ++i) {
            const int o = u_frag_col(i, lane), h = (i >> 1) & 1;
            xf[mb][i] = o < O ? rs[(SM::qX + o) * RLD + trow[mb][h]] : 0.f;
          }
        if constexpr (MODE == MODE_FVP) {
          float h1f[NB][16];
#pragma unroll
          for (int mb = 0; mb < NB; ++mb)
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const int c = u_frag_col(i, lane), h = (i >> 1) & 1;
              h1f[mb][i] = a.h_cache[(size_t)c * a.B + sl[mb][h]];
              stage[(SM::rH1 + c) * LD + trow[mb][h]] = h1f[mb][i];
            }
          wg_fence();
          gemm(accA, xf, SM::o_bXT, SM::IMGX, KSX, false);                 // X V0
          gemm(accB, h1f, SM::o_bV1T, SM::IMG, 4, false);                // H1 V1
          wg_commit();
        } else {
          wg_fence();
          gemm(accA, xf, SM::o_bXT, SM::IMGX, KSX, false);                 // X W0
          wg_commit();
        }
      }
      // SEP_D1, second pass of a tile: every thread is done with the first pass's Gram phase before E1 overwrites its stage
      // rows (the first pass of the next tile is behind the barrier at the top of the tile loop)
      if (SM::SEP_D1 && b0 > 0) v_wg_sync(wg);
      wg_wait_all();
#pragma unroll
      for (int mb = 0; mb < NB; ++mb) {
        wg_fence_operand(accA[mb]);
        wg_fence_operand(accB[mb]);
      }
      // ================= E1 / C: first epilogue -> operand of the second GEMM
      {
        float v[NB][16];
#pragma unroll
        for (int mb = 0; mb < NB; ++mb)
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int c = u_frag_col(i, lane), h = (i >> 1) & 1;
            if constexpr (MODE != MODE_FVP) {
              v[mb][i] = tanh_f(accA[mb][i] + sb0[c]);
              if constexpr (is_grad_mode(MODE)) {
                stage[(SM::rH1 + c) * LD + trow[mb][h]] = v[mb][i];
                if (a.h_cache != nullptr && inrange[mb][h]) a.h_cache[(size_t)c * a.B + sl[mb][h]] = v[mb][i];
              }
            } else {
              const float h1 = stage[(SM::rH1 + c) * LD + trow[mb][h]];
              v[mb][i] = (accA[mb][i] + sb0[c]) * (1.0f - h1 * h1);                                    // t1
            }
          }
        wg_fence();
        gemm(accB, v, SM::o_bW1T, SM::IMG, 4, MODE == MODE_FVP);        // H1 W1  |  += T1 W1
        wg_commit();
      }
      float h2f[NB][16];
      if constexpr (MODE == MODE_FVP) {             // cached h2, requested while the GEMM runs
#pragma unroll
        for (int mb = 0; mb < NB; ++mb)
#pragma unroll
          for (int i = 0; i < 16; ++i)
            h2f[mb][i] = a.h_cache[(size_t)(H + u_frag_col(i, lane)) * a.B + sl[mb][(i >> 1) & 1]];
      }
      wg_wait_all();
#pragma unroll
      for (int mb = 0; mb < NB; ++mb) wg_fence_operand(accB[mb]);
      // ================= E2 / E: second epilogue -> dmu, d2
      {
        float md[NB][2][A];
#pragma unroll
        for (int mb = 0; mb < NB; ++mb) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int k = 0; k < A; ++k) md[mb][h][k] = 0.f;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int c = u_frag_col(i, lane), h = (i >> 1) & 1;
            if constexpr (MODE != MODE_FVP) {
              h2f[mb][i] = tanh_f(accB[mb][i] + sb1[c]);
              if constexpr (is_grad_mode(MODE)) {
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
        for (int mb = 0; mb < NB; ++mb)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int k = 0; k < A; ++k) {
              md[mb][h][k] += __shfl_xor_sync(0xffffffffu, md[mb][h][k], 1);
              md[mb][h][k] += __shfl_xor_sync(0xffffffffu, md[mb][h][k], 2);
            }
        float dmu[NB][2][A];
#pragma unroll
        for (int mb = 0; mb < NB; ++mb)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = trow[mb][h];
            if constexpr (MODE != MODE_FVP) {
              // the remaining per-sample inputs, from the ring (no registers held across the GEMMs)
              float act[A], om[A];
#pragma unroll
              for (int k = 0; k < A; ++k) {
                act[k] = rs[(SM::qAct + k) * RLD + r];
                om[k] = rs[(SM::qOm + k) * RLD + r];
              }
              const float adv_s = rs[SM::qAdv * RLD + r];
              // z^2 is rounded on its own (__fmul_rn): the gradient pass reuses it for dlog_std, and a product that is free
              // to contract into zsq's add would make the loss of the two modes differ in the last bit for A > 1
              float z[A], zz[A], dmk[A], zsq = 0.f, zsq_old = 0.f, kl = 0.f;
#pragma unroll
              for (int k = 0; k < A; ++k) {
                const float mu = sbo[k] + md[mb][h][k];
                z[k] = (act[k] - mu) * D.inv_std[k];
                zz[k] = __fmul_rn(z[k], z[k]);
                zsq += zz[k];
                const float zo = (act[k] - om[k]) * D.inv_std_old[k];
                zsq_old += zo * zo;
                const float dm = om[k] - mu;
                dmk[k] = dm;
                kl += (dm * dm + D.var_old[k] - D.var_new[k]) / D.var_new2[k] + D.ls_new[k] - D.ls_old[k];
              }
              const float logp_new = -D.sum_ls_new - 0.5f * zsq - D.half_log2pi_A;
              float w_s, term;
              if (a.loss_kind == B200RL_LOSS_TRPO) {
                const float logp_old = -D.sum_ls_old - 0.5f * zsq_old - D.half_log2pi_A;
                w_s = expf(logp_new - logp_old) * adv_s;
                term = -w_s;
              } else {
                w_s = adv_s;
                term = -logp_new * adv_s;
              }
              if (!valid[mb][h]) { w_s = 0.f; term = 0.f; }
              if (t4 == 0) {
                s_loss += (double)term;
                if (valid[mb][h]) { s_kl += (double)kl; m_kl = fmax(m_kl, (double)kl); }
              }
              if constexpr (is_grad_mode(MODE)) {
#pragma unroll
                for (int k = 0; k < A; ++k) {
                  dmu[mb][h][k] = -w_s * z[k] * D.inv_std[k];
                  if constexpr (MODE == MODE_GRAD_KL) {
                    float dls = -w_s * (zz[k] - 1.0f);
                    if (valid[mb][h])
                      add_kl_penalty(a.penalty, dmk[k], D.var_new[k], D.var_new2[k], D.var_old[k], dmu[mb][h][k], dls);
                    if (t4 == 0) {
                      stage[(SM::rDM + k) * LD + r] = dmu[mb][h][k];
                      stage[(SM::rDL + k) * LD + r] = dls;
                    }
                  } else if (t4 == 0) {
                    stage[(SM::rDM + k) * LD + r] = dmu[mb][h][k];
                    stage[(SM::rDL + k) * LD + r] = -w_s * (zz[k] - 1.0f);
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
          float v[NB][16];
#pragma unroll
          for (int mb = 0; mb < NB; ++mb)
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
          gemm(accA, v, SM::o_bW1, SM::IMG, 4, false);                  // D2 W1^T
          wg_commit();
        }
      }
      if constexpr (MODE != MODE_LOSS) {
        // ================= E3 / G: d1 = D1pre (1 - h1^2) (every thread reads the H1 entries it staged itself)
        auto e3 = [&] {
#pragma unroll
          for (int mb = 0; mb < NB; ++mb)
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const int c = u_frag_col(i, lane), r = trow[mb][(i >> 1) & 1];
              const float h1 = stage[(SM::rH1 + c) * LD + r];
              stage[(SM::rD1 + c) * LD + r] = accA[mb][i] * (1.0f - h1 * h1);
            }
        };
        if constexpr (SM::SEP_D1) {
          wg_wait_all();
#pragma unroll
          for (int mb = 0; mb < NB; ++mb) wg_fence_operand(accA[mb]);
          e3();
          v_wg_sync(wg);                       // stage rows of the pass written
          // ================= Gram: dW1 = H1^T D2, dWout, db1, dbout, dlog_std; dW0 = X^T D1, db0 (X: ring rows)
          gram.part_a(stage, tid);
          gram.template part_b<RLD>(stage, rs + SM::qX * RLD, tid);
        } else {
          // at three or more warpgroups per SM the last GEMM completes before the Gram phase: behind it, its A operand
          // would stay live through part A; the other warpgroups cover the wait.  At two, part A runs behind it.
          constexpr bool wait_first = NWG >= 3;
          if constexpr (wait_first) {
            wg_wait_all();
#pragma unroll
            for (int mb = 0; mb < NB; ++mb) wg_fence_operand(accA[mb]);
          }
          v_wg_sync(wg);                       // stage rows of the pass written
          // ================= Gram part A: dW1 = H1^T D2, dWout, db1, dbout, dlog_std (tile_gram.cuh)
          gram.part_a(stage, tid);
          v_wg_sync(wg);                       // every thread is done with the H2 rows: D1 may overwrite them
          if constexpr (!wait_first) {
            wg_wait_all();
#pragma unroll
            for (int mb = 0; mb < NB; ++mb) wg_fence_operand(accA[mb]);
          }
          e3();
          v_wg_sync(wg);
          // ================= Gram part B: dW0 = X^T D1, db0 (X: the ring rows of the pass)
          gram.template part_b<RLD>(stage, rs + SM::qX * RLD, tid);
          v_wg_sync(wg);
        }
      }
    }
    if constexpr (MODE != MODE_LOSS) {
      // the small outputs' float32 sums of the tile -> float64
      gram.fold_a(tid);
      gram.fold_b();
    }
  }

  if constexpr (MODE != MODE_LOSS) {
    double* out = a.partial + (size_t)vb * P;
    gram.write(out, reinterpret_cast<double*>(stage), tid, [wg] { v_wg_sync(wg); });
  }
  if constexpr (MODE != MODE_FVP) {
    // per-warpgroup (loss, sum KL | max KL): after the [nvb][P] partial vectors (GRAD) or alone (LOSS), as
    // loss_thread_kernel
    double v[2] = {s_loss, s_kl};
    double mx[1] = {m_kl};
    double* sc = a.partial + (is_grad_mode(MODE) ? (size_t)nvb * P : (size_t)0) + (size_t)vb * 3;
    v_wg_reduce_store<2, false>(v, red_scratch, sc, tid, wg);
    v_wg_reduce_store<1, true>(mx, red_scratch, sc + 2, tid, wg);
  }
}

template <class N, int MODE>
static int launch_umma32(const UpdArgs& a, int* grid_out, cudaStream_t st) {
  using SM = Umma32<N, MODE>;
  B200RL_SET_MAX_SMEM((update_umma32_kernel<N, MODE>), SM::bytes);
  long long grid = num_sms();                              // persistent: one CTA of NWG warpgroups per SM
  const long long ntiles = host_n_tiles(a, V_TILE);
  if (grid > (ntiles + SM::NWG - 1) / SM::NWG) grid = (ntiles + SM::NWG - 1) / SM::NWG;
  if (grid > MAX_PARTIAL_BLOCKS / SM::NWG) grid = MAX_PARTIAL_BLOCKS / SM::NWG;
  if (grid < 1) grid = 1;
  update_umma32_kernel<N, MODE><<<(unsigned)grid, V_THREADS * SM::NWG, SM::bytes, st>>>(a);
  B200RL_LAUNCH_CHECK("update_umma32_kernel");
  *grid_out = (int)grid * SM::NWG;                         // one partial vector (and loss triple) per warpgroup
  return 0;
}

int update_umma32_launch(int mode, int obs_dim, int act_dim, const UpdArgs& a, int* grid_out, int* P_out, int* ols_out,
                         cudaStream_t st) {
  const int h1 = 32, h2 = 32;
  B200RL_DISPATCH_NET_H(32, {
    *P_out = NetT::P;
    *ols_out = NetT::ols;
    int rc = (mode == MODE_GRAD)      ? launch_umma32<NetT, MODE_GRAD>(a, grid_out, st)
             : (mode == MODE_GRAD_KL) ? launch_umma32<NetT, MODE_GRAD_KL>(a, grid_out, st)
             : (mode == MODE_LOSS)    ? launch_umma32<NetT, MODE_LOSS>(a, grid_out, st)
                                      : launch_umma32<NetT, MODE_FVP>(a, grid_out, st);
    if (rc) return rc;
  });
  return 0;
}

}  // namespace b200rl
