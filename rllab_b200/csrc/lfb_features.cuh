// The linear feature map shared by LinearFeatureBaseline (linear_feature_baseline.py:19-23) and REPS (reps.py:207-211):
//   phi(o, t) = [clip(o, +-10), o^2, t/100, (t/100)^2, (t/100)^3, 1]      (2 O + 4 entries)
// float32 observations and the uint16 step index in, float64 features out.  process.cu (baseline predict) and reps.cu
// (Bellman error of the dual) both evaluate it through lfb_feature.
#pragma once

namespace b200rl {

// feature j of phi(ov, ts); j is a compile-time constant after unrolling, so the branches fold away and the shared
// subexpressions (the clipped observation, t/100) are computed once per sample
template <int OT>
__device__ __forceinline__ double lfb_feature(const float (&ov)[OT], unsigned short ts, int j) {
  if (j < 2 * OT) {
    const int k = j < OT ? j : j - OT;
    const double o = (double)fminf(fmaxf(ov[k], -10.0f), 10.0f);
    return j < OT ? o : o * o;
  }
  const double al = (double)ts / 100.0;
  if (j == 2 * OT) return al;
  if (j == 2 * OT + 1) return al * al;
  if (j == 2 * OT + 2) return al * al * al;
  return 1.0;
}

// phi(o, t) . w, summed in feature-pair order: (o_k w_k + o_k^2 w_{O+k}) for k = 0..O-1, then the time terms
template <int OT>
__device__ __forceinline__ double lfb_dot(const float (&ov)[OT], unsigned short ts, const double* __restrict__ w) {
  double acc = 0.0;
#pragma unroll
  for (int k = 0; k < OT; ++k) acc += lfb_feature<OT>(ov, ts, k) * w[k] + lfb_feature<OT>(ov, ts, OT + k) * w[OT + k];
  acc += lfb_feature<OT>(ov, ts, 2 * OT) * w[2 * OT] + lfb_feature<OT>(ov, ts, 2 * OT + 1) * w[2 * OT + 1] +
         lfb_feature<OT>(ov, ts, 2 * OT + 2) * w[2 * OT + 2] + w[2 * OT + 3];       // the constant feature is 1
  return acc;
}

}  // namespace b200rl
