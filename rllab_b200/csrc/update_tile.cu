// Surrogate gradient and Fisher-vector product for 32-wide policies: one THREAD per sample for the per-sample math
// (forward, tangent-forward, backward -- the same canonical summation order as the rollout kernel), then a
// block-cooperative accumulation of the weight gradients as small Gram products over a 128-sample tile staged in
// shared memory:
//     dW0 = X^T D1, db0 = 1^T D1, dW1 = H1^T D2, db1 = 1^T D2, dWout = H2^T DM, dbout = 1^T DM, dlog_std = 1^T DL
// dW1 (32x32 outputs, the bulk) uses 4x4 register tiles, rows interleaved by 8 so that every LDS.128 of a warp is
// conflict-free (one wavefront), split in two K-halves over the 128 threads; per-tile float32 partial products are
// folded into float64 register accumulators; per-block float64 partials are reduced in fixed order by the caller.
//
// Replaces f_grad / f_Hx_plain of rllab/optimizers/conjugate_gradient_optimizer.py:184-215,22-55 and the gradient
// half of f_opt in rllab/optimizers/first_order_optimizer.py:62-76.
#include "tile_phase_a.cuh"

namespace b200rl {

constexpr int T_THREADS = 128, T_TILE = 128, T_LD = T_TILE + 4;

template <class N, int MODE>
struct TileSmem {
  static constexpr int O = N::O, H = N::H1, A = N::A;
  static_assert(N::H1 == 32 && N::H2 == 32, "tile kernel is specialised for 32-wide layers");
  static constexpr int rX = 0, rH1 = rX + O, rH2 = rH1 + H, rD1 = rH2 + H, rD2 = rD1 + H, rDM = rD2 + H, rDL = rDM + A,
                       R = rDL + A;
  static constexpr int P4 = (N::P + 3) & ~3;
  static constexpr int o_sp = 0, o_sv = P4, o_stage = (MODE == MODE_FVP ? 2 : 1) * P4;
  static constexpr int n_floats = o_stage + R * T_LD;
  static constexpr int scratch_off = ((n_floats * 4 + 15) / 16) * 16;
  static constexpr size_t bytes = (size_t)scratch_off + 3 * 32 * 8;
  static_assert(2 * 64 * 16 * 8 <= R * T_LD * 4, "stage region must hold the K-half combine scratch");
};

// Resident CTAs per SM: 3 when three tiles fit the 228 KB of shared memory (small O, A: CartPole / Pendulum / PointEnv
// gradient -> 168 registers, 12 warps/SM: 3.88 -> 3.44 ms on cfg2, A/B measured), otherwise 2 (<= 255 registers).
template <class N, int MODE>
constexpr int tile_minblocks() { return (TileSmem<N, MODE>::bytes + 1024) * 3 <= 228 * 1024 ? 3 : 2; }

template <class N, int MODE>
__global__ void __launch_bounds__(T_THREADS, tile_minblocks<N, MODE>()) update_tile_kernel(UpdArgs a) {
  using SM = TileSmem<N, MODE>;
  constexpr int O = N::O, H = 32, A = N::A, P = N::P, LD = T_LD;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sf = reinterpret_cast<float*>(smem_raw);
  float* sp = sf + SM::o_sp;
  float* sv = sf + SM::o_sv;
  float* stage = sf + SM::o_stage;
  double* red_scratch = reinterpret_cast<double*>(smem_raw + SM::scratch_off);
  const int tid = threadIdx.x;

  for (int i = tid; i < P; i += T_THREADS) sp[i] = a.params[i];
  if constexpr (MODE == MODE_FVP)
    for (int i = tid; i < P; i += T_THREADS) sv[i] = (float)a.xvec[i];
  __syncthreads();

  TileDist D;
  tile_dist_init<N, MODE>(D, sp + N::ols, a);
  TileGram<N, SM::rX, SM::rH1, SM::rH2, SM::rD1, SM::rD2, SM::rDM, LD> gram;
  gram.init();
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;

  const long long ntiles = n_tiles_of(a, T_TILE);
  for (long long ti_ = blockIdx.x; ti_ < ntiles; ti_ += gridDim.x) {
    asm volatile("" ::: "memory");
    const long long s = tile_at(a, ti_) * T_TILE + tid;
    const bool inrange = s < a.B;
    const bool valid = sample_valid(a, s);
    // ================= phase A: per-sample forward / (tangent) / backward, staged to shared memory
    tile_phase_a<N, MODE, SM, LD>(a, sp, sv, stage, D, inrange ? s : a.B - 1, inrange, valid, tid, s_loss, s_kl, m_kl);
    __syncthreads();
    // ================= phase B: Gram accumulation over the tile (tile_gram.cuh)
    gram.accumulate_a(stage, tid);
    gram.accumulate_b(stage, tid);
    __syncthreads();
  }

  // ================= write this block's partial vector (float64)
  double* out = a.partial + (size_t)blockIdx.x * P;
  gram.write(out, reinterpret_cast<double*>(stage), tid);   // scratch [2][64][16] doubles in the (idle) stage region
  if constexpr (MODE == MODE_GRAD) {
    __syncthreads();
    double v[2] = {s_loss, s_kl};
    double mx[1] = {m_kl};
    double* sc = a.partial + (size_t)gridDim.x * P + (size_t)blockIdx.x * 3;
    block_reduce_store<2, false>(v, red_scratch, sc);
    block_reduce_store<1, true>(mx, red_scratch, sc + 2);
  }
}

template <class N, int MODE>
static int launch_tile(const UpdArgs& a, int* grid_out, cudaStream_t st) {
  using SM = TileSmem<N, MODE>;
  B200RL_SET_MAX_SMEM((update_tile_kernel<N, MODE>), SM::bytes);
  int per_sm = (int)((228 * 1024) / (SM::bytes + 1024));   // 228 KB per SM, 1 KB reserved per resident CTA
  if (per_sm < 1) per_sm = 1;
  if (per_sm > tile_minblocks<N, MODE>()) per_sm = tile_minblocks<N, MODE>();
  long long grid = (long long)num_sms() * per_sm;
  const long long ntiles = host_n_tiles(a, T_TILE);
  if (grid > ntiles) grid = ntiles;
  if (grid > MAX_PARTIAL_BLOCKS) grid = MAX_PARTIAL_BLOCKS;
  if (grid < 1) grid = 1;
  update_tile_kernel<N, MODE><<<(unsigned)grid, T_THREADS, SM::bytes, st>>>(a);
  B200RL_LAUNCH_CHECK("update_tile_kernel");
  *grid_out = (int)grid;
  return 0;
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
  static int run(const UpdArgs& a, int* grid_out, cudaStream_t st) { return launch_tile<N, MODE_GRAD>(a, grid_out, st); }
};
template <class N>
struct FfmaGrad<N, false> {
  static int run(const UpdArgs&, int*, cudaStream_t) {
    set_error("the FP32 gradient kernels are not part of this build (the tensor-core kernels serve b200rl_grad)");
    return B200RL_EUNSUPPORTED;
  }
};
}  // namespace

int update_tile_launch(int mode, int obs_dim, int act_dim, const UpdArgs& a, int* grid_out, int* P_out, int* ols_out,
                       cudaStream_t st) {
  const int h1 = 32, h2 = 32;
  B200RL_DISPATCH_NET_H(32, {
    *P_out = NetT::P;
    *ols_out = NetT::ols;
    int rc = (mode == MODE_GRAD) ? FfmaGrad<NetT, kFfmaGradBuilt>::run(a, grid_out, st) : launch_tile<NetT, MODE_FVP>(a, grid_out, st);
    if (rc) return rc;
  });
  return 0;
}

}  // namespace b200rl
