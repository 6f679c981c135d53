// Shared declarations of the policy-update kernels (update.cu: loss/KL pass + the C entry points; update_tile.cu:
// thread-per-sample + shared-memory Gram accumulation, 32-wide nets; update_gemm.cu: tiled-GEMM formulation, 64-wide nets).
#pragma once
#include "mlp.cuh"

namespace b200rl {

constexpr bool is_grad_mode(int mode) { return mode == MODE_GRAD || mode == MODE_GRAD_KL; }

struct UpdArgs {
  const float* params;
  const double* xvec;  // FVP: tangent vector (float64, P)
  float* h_cache;      // [H1+H2][B] hidden activations: written by GRAD (if non-null), read by FVP (if non-null)
  float log_min_std;
  long long B;
  const float *obs, *act, *adv, *old_mean, *old_log_std;
  int loss_kind;
  const unsigned char* flags;  // [B] or NULL: samples carrying B200RL_FLAG_MASKED contribute nothing
  const int* tile_list;        // FVP sub-sampling: indices of the 128-sample tiles to visit (device), or NULL = all tiles
  int n_list;
  double* partial;
  float penalty;               // MODE_GRAD_KL only: weight of the KL term (after the other fields: their offsets stay)
};

// The KL-penalty terms of one valid sample and action dimension k, added to the surrogate's output deltas: the exact
// derivatives of  kl_k = (dm^2 + var_old - var_new) / var_new2 + ls_new - ls_old,  dm = old_mean - mu,
// var_new2 = 2 sigma^2 + 1e-8 (diagonal_gaussian.py:14-34), with respect to mu and log_std:
//   dkl/dmu = -2 dm / var_new2,   dkl/dls = 1 - 2 sigma^2 (var_new2 + 2 num) / var_new2^2,   num = dm^2 + var_old - var_new
// Every operation is rounded on its own, so no product of these terms contracts into the surrogate's arithmetic.
__device__ __forceinline__ void add_kl_penalty(float pen, float dm, float var_new, float var_new2, float var_old,
                                               float& dmu, float& dls) {
  const float num = __fadd_rn(__fadd_rn(__fmul_rn(dm, dm), var_old), -var_new);
  const float g_mu = __fdiv_rn(__fmul_rn(-2.0f, dm), var_new2);
  const float t = __fmul_rn(__fmul_rn(2.0f, var_new), __fadd_rn(var_new2, __fmul_rn(2.0f, num)));
  const float g_ls = __fadd_rn(1.0f, -__fdiv_rn(t, __fmul_rn(var_new2, var_new2)));
  dmu = __fadd_rn(dmu, __fmul_rn(pen, g_mu));
  dls = __fadd_rn(dls, __fmul_rn(pen, g_ls));
}

// valid sample: inside the batch and not masked out by process_samples(drop_cut_paths)
__device__ __forceinline__ bool sample_valid(const UpdArgs& a, long long s) {
  return s < a.B && !(a.flags != nullptr && (a.flags[s] & B200RL_FLAG_MASKED));
}
// number of tiles a kernel iterates over and the i-th of them
__device__ __forceinline__ long long n_tiles_of(const UpdArgs& a, int tile) {
  return a.tile_list != nullptr ? (long long)a.n_list : (a.B + tile - 1) / tile;
}
__device__ __forceinline__ long long tile_at(const UpdArgs& a, long long i) {
  return a.tile_list != nullptr ? (long long)a.tile_list[i] : i;
}
inline long long host_n_tiles(const UpdArgs& a, int tile) {
  return a.tile_list != nullptr ? (long long)a.n_list : (a.B + tile - 1) / tile;
}

// 32-wide nets.  Launches the tile kernel on `a` (a.partial = workspace); returns the grid size used (blocks that
// wrote partial[block][P] (+ [grid][3] loss scalars after them in MODE_GRAD)), P and the log_std offset.
int update_tile_launch(int mode, int obs_dim, int act_dim, const UpdArgs& a, int* grid_out, int* P_out, int* ols_out,
                       cudaStream_t st);

// 32- and 64-wide nets: the tiled-GEMM formulation (update_gemm.cu); same contract as update_tile_launch.
int update_gemm_launch(int mode, int obs_dim, int h, int act_dim, const UpdArgs& a, int* grid_out, int* P_out,
                       int* ols_out, cudaStream_t st);


// 64-wide nets, gradient and (with cached activations) Fisher-vector product: dense layer chain on the tensor cores
// (update_umma.cu); same contract as update_tile_launch.
int update_umma64_launch(int mode, int obs_dim, int act_dim, const UpdArgs& a, int* grid_out, int* P_out, int* ols_out,
                         cudaStream_t st);


// 32-wide nets, gradient and (with cached activations) Fisher-vector product: dense layer chain on the tensor cores
// (update_umma32.cu); same contract as update_tile_launch.
int update_umma32_launch(int mode, int obs_dim, int act_dim, const UpdArgs& a, int* grid_out, int* P_out, int* ols_out,
                         cudaStream_t st);


}  // namespace b200rl
