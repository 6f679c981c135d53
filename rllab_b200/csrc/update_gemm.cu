// Surrogate gradient and Fisher-vector product as a chain of shared-memory tiled GEMMs over a 128-sample tile
// (32- and 64-wide policies).  Every layer of the forward / tangent-forward / backward pass is
//     OUT[rows][128 samples] = f( W^T . IN[rows][128 samples] )
// with a register tile of 8 samples x H/8 units per thread (16 FFMA2 per 3-4 LDS.128), activations staged
// feature-major in shared memory; the weight gradients are Gram products of the staged rows (4x4 register tiles).
// The even/odd-k accumulation chains reproduce the canonical summation order of the rollout kernel (mlp.cuh), so
// mean(theta_old) is bit-identical to what the rollout recorded.
//
//   S0  X                      <- obs                                   (thread = sample)
//   S1  H1 = tanh(W0^T X + b0)                                          (GEMM, K = O)
//   S2  H2 = tanh(W1^T H1 + b1)                                         (GEMM, K = H)
//       FVP: T1 = (1-H1^2)(V0^T X + vb0) ; T2 = (1-H2^2)(W1^T T1 + V1^T H1 + vb1)   (T1/T2 parked in the D1/D2 rows)
//   S3  mu / dist / dmu (GRAD)   or   mu_dot -> dmu = M mu_dot (FVP)    (thread = sample)
//   S4  D2 = (Wout DM)(1-H2^2)                                          (tile, K = A)
//   S5  D1 = (W1 D2)(1-H1^2)                                            (GEMM with W1^T staged once per block, K = H)
//   S6  dW0 += X D1^T, dW1 += H1 D2^T, dWout += H2 DM^T, biases, dlog_std   (Gram, float32 per <= 8 tiles -> float64)
//
// Replaces f_grad / f_Hx_plain of rllab/optimizers/conjugate_gradient_optimizer.py:184-215,22-55 and the gradient
// half of f_opt in rllab/optimizers/first_order_optimizer.py:62-76.
#include "tile_phase_a.cuh"

namespace b200rl {

constexpr int G_TS = 128, G_LD = G_TS + 4, G_FLUSH = 8;   // 128 or 256 threads per 128-sample tile (template NTH)

template <class N, int MODE>
struct GemmSmem {
  static constexpr int O = N::O, H = N::H1, A = N::A;
  static_assert(N::H1 == N::H2 && (N::H1 == 32 || N::H1 == 64), "32- or 64-wide layers");
  static constexpr int rX = 0, rH1 = rX + O, rH2 = rH1 + H, rD1 = rH2 + H, rD2 = rD1 + H, rDM = rD2 + H, rDL = rDM + A,
                       R = rDL + A;
  static constexpr int P4 = (N::P + 3) & ~3;
  static constexpr int o_sp = 0, o_w1t = P4, o_sv = o_w1t + H * H, o_stage = o_sv + (MODE == MODE_FVP ? P4 : 0);
  static constexpr int n_floats = o_stage + R * G_LD;
  static constexpr int scratch_off = ((n_floats * 4 + 15) / 16) * 16;
  static constexpr size_t bytes = (size_t)scratch_off + 3 * 32 * 8;
};

// acc[p][c] += IN[k][s0 + 2p .. 2p+1] * W[k][j0 + c]  for k in [0, K): even k into ae, odd k into ao.
template <int K, int H, int RJ>
__device__ __forceinline__ void gemm_acc(const float* in_rows, const float* W, int s0, int j0, float2 (&ae)[4][RJ],
                                         float2 (&ao)[4][RJ]) {
#pragma unroll 4
  for (int k = 0; k < K; ++k) {
    const float4 a0 = *reinterpret_cast<const float4*>(in_rows + k * G_LD + s0);
    const float4 a1 = *reinterpret_cast<const float4*>(in_rows + k * G_LD + s0 + 4);
    float w[RJ];
#pragma unroll
    for (int c = 0; c < RJ; c += 4) {
      const float4 wv = *reinterpret_cast<const float4*>(W + k * H + j0 + c);
      w[c] = wv.x; w[c + 1] = wv.y; w[c + 2] = wv.z; w[c + 3] = wv.w;
    }
    const float2 p0 = make_float2(a0.x, a0.y), p1 = make_float2(a0.z, a0.w), p2 = make_float2(a1.x, a1.y),
                 p3 = make_float2(a1.z, a1.w);
    if ((k & 1) == 0) {
#pragma unroll
      for (int c = 0; c < RJ; ++c) {
        const float2 ww = make_float2(w[c], w[c]);
        ae[0][c] = ffma2(p0, ww, ae[0][c]); ae[1][c] = ffma2(p1, ww, ae[1][c]);
        ae[2][c] = ffma2(p2, ww, ae[2][c]); ae[3][c] = ffma2(p3, ww, ae[3][c]);
      }
    } else {
#pragma unroll
      for (int c = 0; c < RJ; ++c) {
        const float2 ww = make_float2(w[c], w[c]);
        ao[0][c] = ffma2(p0, ww, ao[0][c]); ao[1][c] = ffma2(p1, ww, ao[1][c]);
        ao[2][c] = ffma2(p2, ww, ao[2][c]); ao[3][c] = ffma2(p3, ww, ao[3][c]);
      }
    }
  }
}

template <int RJ>
__device__ __forceinline__ void acc_init(float2 (&ae)[4][RJ], float2 (&ao)[4][RJ], const float* bias, int j0) {
#pragma unroll
  for (int c = 0; c < RJ; ++c) {
    const float b = bias ? bias[j0 + c] : 0.f;
#pragma unroll
    for (int p = 0; p < 4; ++p) { ae[p][c] = make_float2(b, b); ao[p][c] = make_float2(0.f, 0.f); }
  }
}

// tile element (sample s0 + 2p + {0,1}, unit c) = ae[p][c] + ao[p][c]; rows of the staged matrix are G_LD apart
template <int RJ>
__device__ __forceinline__ void store_tanh_tile(const float2 (&ae)[4][RJ], const float2 (&ao)[4][RJ], float* dst) {
#pragma unroll
  for (int c = 0; c < RJ; ++c) {
    float v[8];
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      v[2 * p] = tanh_f(ae[p][c].x + ao[p][c].x);
      v[2 * p + 1] = tanh_f(ae[p][c].y + ao[p][c].y);
    }
    *reinterpret_cast<float4*>(dst + c * G_LD) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(dst + c * G_LD + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
}
// activation cache <-> staged tile (RJ rows x 8 samples starting at sample index sbase; rows are B apart in the cache)
// (rows of the cache are 16-byte aligned when B % 4 == 0: two LDG.128 / STG.128 per row instead of eight scalar accesses)
template <int RJ>
__device__ __forceinline__ void load_cached_tile(const float* src, long long B, long long sbase, float* dst) {
  if ((B & 3) == 0 && sbase + 8 <= B) {
#pragma unroll
    for (int c = 0; c < RJ; ++c) {
      const float4 v0 = __ldg(reinterpret_cast<const float4*>(src + (size_t)c * B + sbase));
      const float4 v1 = __ldg(reinterpret_cast<const float4*>(src + (size_t)c * B + sbase + 4));
      *reinterpret_cast<float4*>(dst + c * G_LD) = v0;
      *reinterpret_cast<float4*>(dst + c * G_LD + 4) = v1;
    }
    return;
  }
#pragma unroll
  for (int c = 0; c < RJ; ++c) {
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const long long s = sbase + e;
      v[e] = src[(size_t)c * B + (s < B ? s : B - 1)];
    }
    *reinterpret_cast<float4*>(dst + c * G_LD) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(dst + c * G_LD + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
}
template <int RJ>
__device__ __forceinline__ void save_cached_tile(const float* src, float* dst, long long B, long long sbase) {
  if ((B & 3) == 0 && sbase + 8 <= B) {
#pragma unroll
    for (int c = 0; c < RJ; ++c) {
      *reinterpret_cast<float4*>(dst + (size_t)c * B + sbase) = *reinterpret_cast<const float4*>(src + c * G_LD);
      *reinterpret_cast<float4*>(dst + (size_t)c * B + sbase + 4) = *reinterpret_cast<const float4*>(src + c * G_LD + 4);
    }
    return;
  }
#pragma unroll
  for (int c = 0; c < RJ; ++c) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const long long s = sbase + e;
      if (s < B) dst[(size_t)c * B + s] = src[c * G_LD + e];
    }
  }
}

// dst = (ae + ao) * (1 - h^2) with h read back from this thread's own tile of the staged activation rows
template <int RJ>
__device__ __forceinline__ void store_scaled_tile(const float2 (&ae)[4][RJ], const float2 (&ao)[4][RJ],
                                                  const float* hsrc, float* dst) {
#pragma unroll
  for (int c = 0; c < RJ; ++c) {
    const float4 h0 = *reinterpret_cast<const float4*>(hsrc + c * G_LD);
    const float4 h1 = *reinterpret_cast<const float4*>(hsrc + c * G_LD + 4);
    float4 d0, d1;
    d0.x = (ae[0][c].x + ao[0][c].x) * (1.0f - h0.x * h0.x); d0.y = (ae[0][c].y + ao[0][c].y) * (1.0f - h0.y * h0.y);
    d0.z = (ae[1][c].x + ao[1][c].x) * (1.0f - h0.z * h0.z); d0.w = (ae[1][c].y + ao[1][c].y) * (1.0f - h0.w * h0.w);
    d1.x = (ae[2][c].x + ao[2][c].x) * (1.0f - h1.x * h1.x); d1.y = (ae[2][c].y + ao[2][c].y) * (1.0f - h1.y * h1.y);
    d1.z = (ae[3][c].x + ao[3][c].x) * (1.0f - h1.z * h1.z); d1.w = (ae[3][c].y + ao[3][c].y) * (1.0f - h1.w * h1.w);
    *reinterpret_cast<float4*>(dst + c * G_LD) = d0;
    *reinterpret_cast<float4*>(dst + c * G_LD + 4) = d1;
  }
}

// NTH = 128: register tile 8 samples x H/8 units; NTH = 256 (64-wide nets): 8 samples x H/16 units, two warps per
// scheduler so that shared-memory latency overlaps with the FFMA2 chains of the other warp.
template <class N, int MODE, int NTH>
__global__ void __launch_bounds__(NTH, (N::H1 == 32 ? 2 : 1)) update_gemm_kernel(UpdArgs a) {
  using SM = GemmSmem<N, MODE>;
  constexpr int G_THREADS = NTH, UG = NTH / 16;          // unit groups per 8-sample group
  constexpr int O = N::O, H = N::H1, A = N::A, P = N::P, LD = G_LD, RJ = H / UG;
  static_assert(RJ % 4 == 0 && RJ >= 4, "register tile width must be a multiple of 4 units");
  constexpr int NT1 = (H / 4) * (H / 4);                 // 4x4 Gram tiles of dW1
  constexpr int KSPLIT = (NT1 <= 64) ? 2 : 1;            // H=32: 64 tiles x 2 K-halves; H=64: 256 tiles, 2 per thread
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sf = reinterpret_cast<float*>(smem_raw);
  float* sp = sf + SM::o_sp;
  float* w1t = sf + SM::o_w1t;
  float* sv = sf + SM::o_sv;
  float* stage = sf + SM::o_stage;
  double* red_scratch = reinterpret_cast<double*>(smem_raw + SM::scratch_off);
  const int tid = threadIdx.x;

  for (int i = tid; i < P; i += G_THREADS) sp[i] = a.params[i];
  if constexpr (MODE == MODE_FVP)
    for (int i = tid; i < P; i += G_THREADS) sv[i] = (float)a.xvec[i];
  __syncthreads();
  for (int i = tid; i < H * H; i += G_THREADS) w1t[(i % H) * H + (i / H)] = sp[N::oW1 + i];   // w1t[j][i] = W1[i][j]
  double* out = a.partial + (size_t)blockIdx.x * P;
  for (int i = tid; i < P; i += G_THREADS) out[i] = 0.0;
  __syncthreads();

  TileDist D;
  D.sum_ls_new = 0.f; D.sum_ls_old = 0.f;
#pragma unroll
  for (int k = 0; k < A; ++k) {
    D.ls_new[k] = clamp_log_std(sp[N::ols + k], a.log_min_std);
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

  // GEMM tile ownership: 16 sample groups of 8 x 8 unit groups of RJ
  const int og = tid % UG, sg = tid / UG;
  const int s0 = sg * 8, j0 = og * RJ;
  // Gram ownership
  constexpr int GT = (KSPLIT == 2) ? 1 : NT1 / G_THREADS;   // 4x4 tiles per thread
  float2 gW1[GT][4][4];               // .x / .y: even- / odd-sample partial sums (packed FFMA2, see gram_fma4)
#pragma unroll
  for (int g = 0; g < GT; ++g)
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) gW1[g][r][c] = make_float2(0.f, 0.f);
  constexpr int NS = (O + 2 > A + 1) ? O + 2 : A + 1;
  float2 gS[NS];
#pragma unroll
  for (int k = 0; k < NS; ++k) gS[k] = make_float2(0.f, 0.f);
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;

  auto flush = [&]() {
    // dW1: combine K-halves through shared memory (fixed order), then float64 read-modify-write of this block's partial
    float* scr = stage;   // free between tiles (caller syncs)
    if constexpr (KSPLIT == 2) {
      const int w1_tile = tid & 63, kh = tid >> 6;
      const int ti = w1_tile >> 3, tj = w1_tile & 7;
      if (kh == 1) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) scr[w1_tile * 16 + r * 4 + c] = gW1[0][r][c].x + gW1[0][r][c].y;
      }
      __syncthreads();
      if (kh == 0) {
        // read-modify-write of this block's float64 partial: all loads first, then all stores (a chain of 16 dependent
        // global round trips otherwise -- the compiler cannot reorder the loads across the stores)
        double t[4][4];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) t[r][c] = out[N::oW1 + (ti + 8 * r) * H + (tj + 8 * c)];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c)
            out[N::oW1 + (ti + 8 * r) * H + (tj + 8 * c)] =
                t[r][c] + ((double)(gW1[0][r][c].x + gW1[0][r][c].y) + (double)scr[w1_tile * 16 + r * 4 + c]);
      }
    } else {
#pragma unroll
      for (int g = 0; g < GT; ++g) {
        const int w1_tile = tid + g * G_THREADS;
        const int ti = w1_tile / (H / 4), tj = w1_tile % (H / 4);
        double t[4][4];                        // loads first, then stores (see above)
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) t[r][c] = out[N::oW1 + (ti + (H / 4) * r) * H + (tj + (H / 4) * c)];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c)
            out[N::oW1 + (ti + (H / 4) * r) * H + (tj + (H / 4) * c)] =
                t[r][c] + (double)(gW1[g][r][c].x + gW1[g][r][c].y);
      }
    }
#pragma unroll
    for (int g = 0; g < GT; ++g)
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) gW1[g][r][c] = make_float2(0.f, 0.f);
    // small outputs
    for (int task = tid; task < 2 * H; task += G_THREADS) {
      if (task < H) {
        double t[O + 2];
#pragma unroll
        for (int o = 0; o < O; ++o) t[o] = out[N::oW0 + o * H + task];
        t[O] = out[N::ob0 + task];
        t[O + 1] = (task < 2 * A) ? out[N::obo + task] : 0.0;
#pragma unroll
        for (int o = 0; o < O; ++o) out[N::oW0 + o * H + task] = t[o] + (double)(gS[o].x + gS[o].y);
        out[N::ob0 + task] = t[O] + (double)(gS[O].x + gS[O].y);
        if (task < 2 * A) out[N::obo + task] = t[O + 1] + (double)(gS[O + 1].x + gS[O + 1].y);   // bout[A], log_std[A] contiguous
      } else {
        const int j = task - H;
        double t[A + 1];
#pragma unroll
        for (int k = 0; k < A; ++k) t[k] = out[N::oWo + j * A + k];
        t[A] = out[N::ob1 + j];
#pragma unroll
        for (int k = 0; k < A; ++k) out[N::oWo + j * A + k] = t[k] + (double)(gS[k].x + gS[k].y);
        out[N::ob1 + j] = t[A] + (double)(gS[A].x + gS[A].y);
      }
    }
#pragma unroll
    for (int k = 0; k < NS; ++k) gS[k] = make_float2(0.f, 0.f);
    __syncthreads();
  };

  const long long ntiles = n_tiles_of(a, G_TS);
  int since_flush = 0;
  for (long long ti_ = blockIdx.x; ti_ < ntiles; ti_ += gridDim.x) {
    asm volatile("" ::: "memory");
    const long long tile = tile_at(a, ti_);
    const bool own_sample = (NTH == G_TS) || tid < G_TS;      // "thread = sample" phases (S0, S3)
    const long long s = tile * G_TS + tid;
    const bool valid = own_sample && sample_valid(a, s);
    const long long sl = (s < a.B) ? s : a.B - 1;
    // ---- S0: observations
    if (own_sample) {
#pragma unroll
      for (int o = 0; o < O; ++o) stage[(SM::rX + o) * LD + tid] = a.obs[(size_t)o * a.B + sl];
    }
    __syncthreads();
    // ---- S1: H1 = tanh(W0^T X + b0)   (and, FVP, T1 = (1-H1^2)(V0^T X + vb0) -> D1 rows)
    {
      float2 ae[4][RJ], ao[4][RJ];
      if (MODE == MODE_FVP && a.h_cache != nullptr) {
        load_cached_tile<RJ>(a.h_cache + (size_t)j0 * a.B, a.B, tile * G_TS + s0, stage + (SM::rH1 + j0) * LD + s0);
      } else {
        acc_init<RJ>(ae, ao, sp + N::ob0, j0);
        gemm_acc<O, H, RJ>(stage + SM::rX * LD, sp + N::oW0, s0, j0, ae, ao);
        store_tanh_tile<RJ>(ae, ao, stage + (SM::rH1 + j0) * LD + s0);
        if (MODE == MODE_GRAD && a.h_cache != nullptr)
          save_cached_tile<RJ>(stage + (SM::rH1 + j0) * LD + s0, a.h_cache + (size_t)j0 * a.B, a.B, tile * G_TS + s0);
      }
      if constexpr (MODE == MODE_FVP) {
        acc_init<RJ>(ae, ao, sv + N::ob0, j0);
        gemm_acc<O, H, RJ>(stage + SM::rX * LD, sv + N::oW0, s0, j0, ae, ao);
        store_scaled_tile<RJ>(ae, ao, stage + (SM::rH1 + j0) * LD + s0, stage + (SM::rD1 + j0) * LD + s0);
      }
    }
    __syncthreads();
    // ---- S2: H2 = tanh(W1^T H1 + b1)   (and, FVP, T2 = (1-H2^2)(W1^T T1 + V1^T H1 + vb1) -> D2 rows)
    {
      float2 ae[4][RJ], ao[4][RJ];
      if (MODE == MODE_FVP && a.h_cache != nullptr) {
        load_cached_tile<RJ>(a.h_cache + (size_t)(H + j0) * a.B, a.B, tile * G_TS + s0, stage + (SM::rH2 + j0) * LD + s0);
      } else {
        acc_init<RJ>(ae, ao, sp + N::ob1, j0);
        gemm_acc<H, H, RJ>(stage + SM::rH1 * LD, sp + N::oW1, s0, j0, ae, ao);
        store_tanh_tile<RJ>(ae, ao, stage + (SM::rH2 + j0) * LD + s0);
        if (MODE == MODE_GRAD && a.h_cache != nullptr)
          save_cached_tile<RJ>(stage + (SM::rH2 + j0) * LD + s0, a.h_cache + (size_t)(H + j0) * a.B, a.B, tile * G_TS + s0);
      }
      if constexpr (MODE == MODE_FVP) {
        acc_init<RJ>(ae, ao, sv + N::ob1, j0);
        gemm_acc<H, H, RJ>(stage + SM::rD1 * LD, sp + N::oW1, s0, j0, ae, ao);   // T1 W1
        gemm_acc<H, H, RJ>(stage + SM::rH1 * LD, sv + N::oW1, s0, j0, ae, ao);   // H1 V1
        store_scaled_tile<RJ>(ae, ao, stage + (SM::rH2 + j0) * LD + s0, stage + (SM::rD2 + j0) * LD + s0);
      }
    }
    __syncthreads();
    // ---- S3: per-sample distribution math (thread = sample)
    if (own_sample) {
      float dmu[A];
      if constexpr (MODE == MODE_GRAD) {
        float mu[A];
#pragma unroll
        for (int k = 0; k < A; ++k) {
          float s0_ = sp[N::obo + k], s1_ = 0.f;
#pragma unroll 8
          for (int j = 0; j < H; j += 2) {
            s0_ = fmaf(stage[(SM::rH2 + j) * LD + tid], sp[N::oWo + j * A + k], s0_);
            s1_ = fmaf(stage[(SM::rH2 + j + 1) * LD + tid], sp[N::oWo + (j + 1) * A + k], s1_);
          }
          mu[k] = s0_ + s1_;
        }
        float z[A], zsq = 0.f, zsq_old = 0.f, kl = 0.f;
#pragma unroll
        for (int k = 0; k < A; ++k) {
          const float act = a.act[(size_t)k * a.B + sl];
          const float om = a.old_mean[(size_t)k * a.B + sl];
          z[k] = (act - mu[k]) * D.inv_std[k];
          zsq += z[k] * z[k];
          const float zo = (act - om) * D.inv_std_old[k];
          zsq_old += zo * zo;
          const float dm = om - mu[k];
          kl += (dm * dm + D.var_old[k] - D.var_new[k]) / D.var_new2[k] + D.ls_new[k] - D.ls_old[k];
        }
        const float adv_s = a.adv[sl];
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
        if (!valid) { w_s = 0.f; term = 0.f; }
        s_loss += (double)term;
        if (valid) { s_kl += (double)kl; m_kl = fmax(m_kl, (double)kl); }
#pragma unroll
        for (int k = 0; k < A; ++k) {
          dmu[k] = -w_s * z[k] * D.inv_std[k];
          stage[(SM::rDM + k) * LD + tid] = dmu[k];
          stage[(SM::rDL + k) * LD + tid] = -w_s * (z[k] * z[k] - 1.0f);
        }
      } else {
        float md[A];
#pragma unroll
        for (int k = 0; k < A; ++k) md[k] = sv[N::obo + k];
#pragma unroll 8
        for (int j = 0; j < H; ++j) {
          const float t2j = stage[(SM::rD2 + j) * LD + tid], h2j = stage[(SM::rH2 + j) * LD + tid];
#pragma unroll
          for (int k = 0; k < A; ++k) md[k] = fmaf(t2j, sp[N::oWo + j * A + k], fmaf(h2j, sv[N::oWo + j * A + k], md[k]));
        }
#pragma unroll
        for (int k = 0; k < A; ++k) {
          stage[(SM::rDM + k) * LD + tid] = valid ? md[k] * D.Mmu[k] : 0.f;
          stage[(SM::rDL + k) * LD + tid] = 0.f;
        }
      }
    }
    __syncthreads();
    // ---- S4: D2 = (Wout DM)(1-H2^2)   (own tile of 8 samples x RJ units)
    {
      float4 dm0[A], dm1[A];
#pragma unroll
      for (int k = 0; k < A; ++k) {
        dm0[k] = *reinterpret_cast<const float4*>(stage + (SM::rDM + k) * LD + s0);
        dm1[k] = *reinterpret_cast<const float4*>(stage + (SM::rDM + k) * LD + s0 + 4);
      }
#pragma unroll
      for (int c = 0; c < RJ; ++c) {
        const int j = j0 + c;
        float4 h0 = *reinterpret_cast<const float4*>(stage + (SM::rH2 + j) * LD + s0);
        float4 h1 = *reinterpret_cast<const float4*>(stage + (SM::rH2 + j) * LD + s0 + 4);
        float4 d0 = make_float4(0.f, 0.f, 0.f, 0.f), d1 = d0;
#pragma unroll
        for (int k = 0; k < A; ++k) {
          const float w = sp[N::oWo + j * A + k];
          d0.x = fmaf(dm0[k].x, w, d0.x); d0.y = fmaf(dm0[k].y, w, d0.y); d0.z = fmaf(dm0[k].z, w, d0.z); d0.w = fmaf(dm0[k].w, w, d0.w);
          d1.x = fmaf(dm1[k].x, w, d1.x); d1.y = fmaf(dm1[k].y, w, d1.y); d1.z = fmaf(dm1[k].z, w, d1.z); d1.w = fmaf(dm1[k].w, w, d1.w);
        }
        d0.x *= (1.0f - h0.x * h0.x); d0.y *= (1.0f - h0.y * h0.y); d0.z *= (1.0f - h0.z * h0.z); d0.w *= (1.0f - h0.w * h0.w);
        d1.x *= (1.0f - h1.x * h1.x); d1.y *= (1.0f - h1.y * h1.y); d1.z *= (1.0f - h1.z * h1.z); d1.w *= (1.0f - h1.w * h1.w);
        *reinterpret_cast<float4*>(stage + (SM::rD2 + j) * LD + s0) = d0;
        *reinterpret_cast<float4*>(stage + (SM::rD2 + j) * LD + s0 + 4) = d1;
      }
    }
    __syncthreads();
    // ---- S5: D1 = (W1 D2)(1-H1^2)
    {
      float2 ae[4][RJ], ao[4][RJ];
      acc_init<RJ>(ae, ao, nullptr, j0);
      gemm_acc<H, H, RJ>(stage + SM::rD2 * LD, w1t, s0, j0, ae, ao);
      store_scaled_tile<RJ>(ae, ao, stage + (SM::rH1 + j0) * LD + s0, stage + (SM::rD1 + j0) * LD + s0);
    }
    __syncthreads();
    // ---- S6: Gram accumulation
    {
      if constexpr (KSPLIT == 2) {
        const int w1_tile = tid & 63, kh = tid >> 6;
        const int ti = w1_tile >> 3, tj = w1_tile & 7;
        const float* U = stage + (SM::rH1 + ti) * LD + kh * 64;
        const float* V = stage + (SM::rD2 + tj) * LD + kh * 64;
#pragma unroll 4
        for (int k = 0; k < 64; k += 4) {
          float4 u[4], v[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) u[r] = *reinterpret_cast<const float4*>(U + r * 8 * LD + k);
#pragma unroll
          for (int c = 0; c < 4; ++c) v[c] = *reinterpret_cast<const float4*>(V + c * 8 * LD + k);
          gram_4x4(u, v, gW1[0]);
        }
      } else {
#pragma unroll
        for (int g = 0; g < GT; ++g) {
          const int w1_tile = tid + g * G_THREADS;
          const int ti = w1_tile / (H / 4), tj = w1_tile % (H / 4);
          const float* U = stage + (SM::rH1 + ti) * LD;
          const float* V = stage + (SM::rD2 + tj) * LD;
#pragma unroll 2
          for (int k = 0; k < G_TS; k += 4) {
            float4 u[4], v[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) u[r] = *reinterpret_cast<const float4*>(U + r * (H / 4) * LD + k);
#pragma unroll
            for (int c = 0; c < 4; ++c) v[c] = *reinterpret_cast<const float4*>(V + c * (H / 4) * LD + k);
            gram_4x4(u, v, gW1[g]);
          }
        }
      }
      // small outputs: task t < H: (dW0[:,t], db0[t], and for t < 2A: dbout / dlog_std); task H + j: (dWout[j,:], db1[j])
      for (int task = tid; task < 2 * H; task += G_THREADS) {
        if (task < H) {
          const float* Dr = stage + (SM::rD1 + task) * LD;
          const float* Er = stage + (SM::rDM + (task < 2 * A ? task : 0)) * LD;
#pragma unroll 2
          for (int k = 0; k < G_TS; k += 4) {
            const float4 d = *reinterpret_cast<const float4*>(Dr + k);
#pragma unroll
            for (int o = 0; o < O; ++o) {
              const float4 xv = *reinterpret_cast<const float4*>(stage + (SM::rX + o) * LD + k);
              gram_fma4(xv, d, gS[o]);
            }
            gS[O].x += (d.x + d.y) + (d.z + d.w);
            if (task < 2 * A) {
              const float4 e = *reinterpret_cast<const float4*>(Er + k);
              gS[O + 1].x += (e.x + e.y) + (e.z + e.w);
            }
          }
        } else {
          const int j = task - H;
          const float* Hh = stage + (SM::rH2 + j) * LD;
          const float* Dr = stage + (SM::rD2 + j) * LD;
#pragma unroll 2
          for (int k = 0; k < G_TS; k += 4) {
            const float4 hv = *reinterpret_cast<const float4*>(Hh + k);
            const float4 d = *reinterpret_cast<const float4*>(Dr + k);
#pragma unroll
            for (int q = 0; q < A; ++q) {
              const float4 m = *reinterpret_cast<const float4*>(stage + (SM::rDM + q) * LD + k);
              gram_fma4(hv, m, gS[q]);
            }
            gS[A].x += (d.x + d.y) + (d.z + d.w);
          }
        }
      }
    }
    __syncthreads();
    if (++since_flush == G_FLUSH) {
      flush();
      since_flush = 0;
    }
  }
  if (since_flush > 0) flush();
  if constexpr (MODE == MODE_GRAD) {
    double v[2] = {s_loss, s_kl};
    double mx[1] = {m_kl};
    double* sc = a.partial + (size_t)gridDim.x * P + (size_t)blockIdx.x * 3;
    block_reduce_store<2, false>(v, red_scratch, sc);
    block_reduce_store<1, true>(mx, red_scratch, sc + 2);
  }
}

template <class N, int MODE, int NTH>
static int launch_gemm_nth(const UpdArgs& a, int* grid_out, cudaStream_t st) {
  using SM = GemmSmem<N, MODE>;
  constexpr int G_THREADS = NTH;
  B200RL_SET_MAX_SMEM((update_gemm_kernel<N, MODE, NTH>), SM::bytes);
  int per_sm = (int)((227 * 1024) / (SM::bytes + 1024));
  if (per_sm < 1) per_sm = 1;
  if (per_sm > (N::H1 == 32 ? 2 : 1)) per_sm = (N::H1 == 32 ? 2 : 1);
  long long grid = (long long)num_sms() * per_sm;
  const long long ntiles = host_n_tiles(a, G_TS);
  if (grid > ntiles) grid = ntiles;
  if (grid > MAX_PARTIAL_BLOCKS) grid = MAX_PARTIAL_BLOCKS;
  if (grid < 1) grid = 1;
  update_gemm_kernel<N, MODE, NTH><<<(unsigned)grid, G_THREADS, SM::bytes, st>>>(a);
  B200RL_LAUNCH_CHECK("update_gemm_kernel");
  *grid_out = (int)grid;
  return 0;
}

// threads per tile: 128 for 32-wide nets, 256 for 64-wide nets (8 samples x 4 units per thread: no spills, two warps per
// scheduler -- Hopper FVP 4.7 -> 3.0 ms, gradient 3.2 -> 2.4 ms against the 128-thread variant, A/B measured in round 1)
template <class N, int MODE>
static int launch_gemm(const UpdArgs& a, int* grid_out, cudaStream_t st) {
  if constexpr (N::H1 == 64) return launch_gemm_nth<N, MODE, 256>(a, grid_out, st);
  else return launch_gemm_nth<N, MODE, 128>(a, grid_out, st);
}

// The shipped library reaches this FP32 formulation only for the Fisher-vector product without an activation cache (the
// tensor-core kernels serve b200rl_grad); its gradient instantiations are built for the A/B variant only
// (-DB200RL_AB_TILE32, README.md).
namespace {   // per translation unit: update_tile.cu and update_gemm.cu each have their own
#ifdef B200RL_AB_TILE32
constexpr bool kFfmaGradBuilt = true;
#else
constexpr bool kFfmaGradBuilt = false;
#endif
template <class N, bool BUILT>
struct FfmaGrad {
  static int run(const UpdArgs& a, int* grid_out, cudaStream_t st) { return launch_gemm<N, MODE_GRAD>(a, grid_out, st); }
};
template <class N>
struct FfmaGrad<N, false> {
  static int run(const UpdArgs&, int*, cudaStream_t) {
    set_error("the FP32 gradient kernels are not part of this build (the tensor-core kernels serve b200rl_grad)");
    return B200RL_EUNSUPPORTED;
  }
};
}  // namespace

int update_gemm_launch(int mode, int obs_dim, int h, int act_dim, const UpdArgs& a, int* grid_out, int* P_out,
                       int* ols_out, cudaStream_t st) {
  const int h1 = h, h2 = h;
  B200RL_DISPATCH_NET({
    *P_out = NetT::P;
    *ols_out = NetT::ols;
    int rc = (mode == MODE_GRAD) ? FfmaGrad<NetT, kFfmaGradBuilt>::run(a, grid_out, st) : launch_gemm<NetT, MODE_FVP>(a, grid_out, st);
    if (rc) return rc;
  });
  return 0;
}

}  // namespace b200rl
