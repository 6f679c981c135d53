// process_samples numeric core on the lane layout: LinearFeatureBaseline.predict + GAE/returns reverse scan +
// the reductions behind the tabular statistics; advantage centering; LinearFeatureBaseline.fit normal equations.
//
// Replaces: rllab/sampler/base.py:48-93,163-180 ; rllab/misc/special.py:51-59,107-111 ; rllab/algos/util.py:7-12 ;
//           rllab/baselines/linear_feature_baseline.py:19-43.
// All three kernels are HBM-streaming (16-40 B per sample); sums are float64, two-stage, fixed order.
#include "mlp.cuh"   // gram_4x4 (packed FFMA2 outer products); includes common.cuh

namespace b200rl {

constexpr int OMAX = 32;  // max obs_dim handled by the runtime-O feature code

// LinearFeatureBaseline features . w  (linear_feature_baseline.py:19-23): [clip(o,+-10), o^2, al, al^2, al^3, 1]
// OT > 0: compile-time obs_dim -- the O loads of a step are issued back to back (and, with the caller's step loop
// unrolled, hoisted across steps) instead of one load -> use chain per feature (in-order issue stalls at the first use of
// every load: the runtime-O loop exposed 8 x O serial DRAM latencies per window -- 0.55 ms on cfg2, round 2 measurement)
template <int OT>
__device__ __forceinline__ double lfb_predict(const float* __restrict__ obs, size_t plane, size_t idx, int O_rt,
                                              unsigned short ts, const double* __restrict__ w) {
  double acc = 0.0;
  const int O = OT > 0 ? OT : O_rt;
  if constexpr (OT > 0) {
    float ov[OT];
#pragma unroll
    for (int k = 0; k < OT; ++k) ov[k] = obs[k * plane + idx];
#pragma unroll
    for (int k = 0; k < OT; ++k) {
      const double o = (double)fminf(fmaxf(ov[k], -10.0f), 10.0f);
      acc += o * w[k] + (o * o) * w[OT + k];
    }
  } else {
    for (int k = 0; k < O; ++k) {
      double o = (double)fminf(fmaxf(obs[k * plane + idx], -10.0f), 10.0f);
      acc += o * w[k] + (o * o) * w[O + k];
    }
  }
  double al = (double)ts / 100.0;
  acc += al * w[2 * O] + (al * al) * w[2 * O + 1] + (al * al * al) * w[2 * O + 2] + w[2 * O + 3];
  return acc;
}

// process_samples = two streaming kernels (round 2, second design; the block-cooperative time-parallel scan of the first
// round-2 design spent its time in barriers between its load / scan / carry phases: 0.54 ms on cfg2, 13 % of HBM):
//
//   lfb_predict_kernel   elementwise over the flattened (t, n) sample index, four samples per thread with 128-bit loads:
//                        b = features(obs, tstep) . w in float64, stored as float32 `base`.  4*O + 2 B read, 4 B written per
//                        sample, no dependence between samples -> a pure HBM stream.
//   gae_scan_kernel      one thread per lane walks T backwards (the recurrences x_t = c_t + m_t x_{t+1} are sequential in
//                        t) in chunks of SC_CH steps, register double-buffered: the 4 x SC_CH loads of the next chunk
//                        (rew, base, flags, tstep -- all independent of the recurrence) are in flight while the current
//                        chunk is scanned, i.e. ~350 B per thread outstanding at any time.  11 B read + 8 B written per
//                        sample; float64 recurrences and statistics, as the reference runs them (sampler/base.py:57-66,
//                        special.py:107-111).  The deltas use the float32-rounded baseline (6e-8 relative).
//
// drop_cut != 0: a path that carries FLAG_CUT on its last sample (cut by the end of the lane buffer) is dropped, the
// way the reference's samplers only ever return whole paths (batch_polopt.py:30-34 with whole_paths=True;
// vectorized_sampler.py drops unfinished running_paths): its samples get FLAG_MASKED, adv = 0, and are excluded from
// every statistic (count, path counts, returns); downstream kernels skip masked samples.
constexpr int PRED_THREADS = 256;

template <int OT>
__device__ __forceinline__ double lfb_dot(const float (&ov)[OT > 0 ? OT : 1], unsigned short ts, const double* __restrict__ w) {
  double acc = 0.0;
#pragma unroll
  for (int k = 0; k < OT; ++k) {
    const double o = (double)fminf(fmaxf(ov[k], -10.0f), 10.0f);
    acc += o * w[k] + (o * o) * w[OT + k];
  }
  const double al = (double)ts / 100.0;
  acc += al * w[2 * OT] + (al * al) * w[2 * OT + 1] + (al * al * al) * w[2 * OT + 2] + w[2 * OT + 3];
  return acc;
}

template <int OT>
__global__ void __launch_bounds__(PRED_THREADS) lfb_predict_kernel(int O_rt, long long B, const float* __restrict__ obs,
                                                                   const unsigned short* __restrict__ tstep,
                                                                   const double* __restrict__ w,
                                                                   float* __restrict__ base) {
  __shared__ double sw[2 * OMAX + 4];
  const int O = OT > 0 ? OT : O_rt;
  for (int i = threadIdx.x; i < 2 * O + 4; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const long long stride = (long long)gridDim.x * blockDim.x, gt = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long done = 0;
  if constexpr (OT > 0) {
    if ((B & 3) == 0) {            // every obs plane is 16 B aligned: 128-bit loads, 4 samples per thread
      const long long nvec = B >> 2;
      for (long long v = gt; v < nvec; v += stride) {
        float4 o4[OT];
#pragma unroll
        for (int k = 0; k < OT; ++k) o4[k] = reinterpret_cast<const float4*>(obs + (size_t)k * B)[v];
        const ushort4 ts = reinterpret_cast<const ushort4*>(tstep)[v];
        float ov[4][OT];
#pragma unroll
        for (int k = 0; k < OT; ++k) { ov[0][k] = o4[k].x; ov[1][k] = o4[k].y; ov[2][k] = o4[k].z; ov[3][k] = o4[k].w; }
        float4 out;
        out.x = (float)lfb_dot<OT>(ov[0], ts.x, sw);
        out.y = (float)lfb_dot<OT>(ov[1], ts.y, sw);
        out.z = (float)lfb_dot<OT>(ov[2], ts.z, sw);
        out.w = (float)lfb_dot<OT>(ov[3], ts.w, sw);
        reinterpret_cast<float4*>(base)[v] = out;
      }
      done = B;
    }
  }
  for (long long i = done + gt; i < B; i += stride) base[i] = (float)lfb_predict<OT>(obs, (size_t)B, (size_t)i, O, tstep[i], sw);
}

// 14 warps of 32 lanes per SM hold cfg2's 65 536 lanes in about one wave (132 x 14 x 32 = 59 136).  The inputs of the next
// SC_AHEAD chunks of SC_CH steps are staged through a warp-private shared-memory ring with cp.async (LDGSTS, 16 B per
// lane, 22 lanes per step row: 128 B rew + 128 B base + 64 B tstep + 32 B flags), so the look-ahead (32 steps = 11 KB per
// warp, 154 KB per SM in flight) does not cost registers; the scan reads its step back with four conflict-free LDS.
// Lane counts that are not a multiple of 32 (rows not 16 B aligned) take the register double-buffered path.
constexpr int SC_CH = 8, SC_THREADS = 32, SC_BLOCKS_PER_SM = 14, SC_AHEAD = 4, SC_RING = SC_AHEAD + 1;
constexpr int SC_ROW_BYTES = 128 + 128 + 64 + 32;        // rew | base | tstep | flags of one step row of a warp

struct ScanChunk {     // one chunk of SC_CH steps of one lane, in registers (unaligned path)
  float rw[SC_CH], bs[SC_CH];
  unsigned int fl[SC_CH];          // flags | (tstep == 0) << 8
};

__device__ __forceinline__ void scan_load(ScanChunk& c, int t_hi, int N, int n, const float* __restrict__ rew,
                                          const float* __restrict__ base, const unsigned char* __restrict__ flags,
                                          const unsigned short* __restrict__ tstep) {
#pragma unroll
  for (int u = 0; u < SC_CH; ++u) {
    const int t = t_hi - u;
    if (t >= 0) {
      const size_t idx = (size_t)t * N + n;
      c.rw[u] = rew[idx];
      c.bs[u] = base[idx];
      c.fl[u] = (unsigned int)flags[idx] | (tstep[idx] == 0 ? 0x100u : 0u);
    }
  }
}

template <bool STAGED>
__global__ void __launch_bounds__(SC_THREADS, SC_BLOCKS_PER_SM)
    gae_scan_kernel(int N, int T, const float* __restrict__ rew, const float* __restrict__ base,
                    unsigned char* __restrict__ flags, const unsigned short* __restrict__ tstep, double discount,
                    double gl, int drop_cut, float* __restrict__ adv, float* __restrict__ ret,
                    double* __restrict__ partial_sum, double* __restrict__ partial_max) {
  __shared__ __align__(16) unsigned char ring[STAGED ? SC_RING * SC_CH * SC_ROW_BYTES : 16];
  const int lane = threadIdx.x;
  const int n0 = blockIdx.x * SC_THREADS;
  const int n_raw = n0 + lane;
  const bool lane_ok = n_raw < N;
  const int n = lane_ok ? n_raw : N - 1;          // out-of-range threads shadow the last lane (no stores, no statistics)
  double s[B200RL_PS_NSUM];
  double m[B200RL_PS_NMAX];
#pragma unroll
  for (int i = 0; i < B200RL_PS_NSUM; ++i) s[i] = 0.0;
#pragma unroll
  for (int i = 0; i < B200RL_PS_NMAX; ++i) m[i] = -1.0e300;
  double a_n = 0.0, r_n = 0.0, u_n = 0.0, b_n = 0.0;
  bool dropped = false;

  // one step of the reverse scan (base.py:57-66): inputs of sample (t, lane) -> adv / ret / statistics
  auto step = [&](int t, float rwf, float bsf, unsigned int f) {
    const size_t idx = (size_t)t * N + n;
    if (f & B200RL_FLAG_END) {
      a_n = 0.0; r_n = 0.0; u_n = 0.0; b_n = 0.0;
      dropped = drop_cut && (f & B200RL_FLAG_CUT);
    }
    const double r = (double)rwf, b = (double)bsf;
    a_n = (r + discount * b_n - b) + gl * a_n;          // base.py:59-61, discount_cumsum(deltas, discount*lambda)
    r_n = r + discount * r_n;                            // discount_cumsum(rewards, discount)
    u_n = r + u_n;
    b_n = b;
    if (!lane_ok) return;
    ret[idx] = (float)r_n;
    if (dropped) {
      adv[idx] = 0.f;
      flags[idx] = (unsigned char)((f & 0xFFu) | B200RL_FLAG_MASKED);
      return;
    }
    adv[idx] = (float)a_n;
    // statistics use the float64 values (as the reference does)
    s[0] += a_n; s[1] += a_n * a_n; s[2] += 1.0;
    s[7] += r_n; s[8] += r_n * r_n; s[9] += b; s[10] += b * b;
    const double res = r_n - b;
    s[11] += res; s[12] += res * res;
    m[2] = fmax(m[2], -a_n); m[3] = fmax(m[3], a_n);
    if (f & 0x100u) {  // first sample of a path
      s[3] += 1.0; s[4] += r_n; s[5] += u_n; s[6] += u_n * u_n;
      m[0] = fmax(m[0], u_n); m[1] = fmax(m[1], -u_n);
    }
  };

  if constexpr (STAGED) {
    // lane role in a step-row copy: which 16 B piece of which array this lane moves
    const unsigned char* src0;        // address of this lane's piece in row t = 0
    size_t row_stride;                // bytes between consecutive rows of that array
    int dst_off;                      // offset of the piece inside a staged row
    if (lane < 8) {
      src0 = reinterpret_cast<const unsigned char*>(rew + n0) + lane * 16; row_stride = (size_t)N * 4; dst_off = lane * 16;
    } else if (lane < 16) {
      src0 = reinterpret_cast<const unsigned char*>(base + n0) + (lane - 8) * 16; row_stride = (size_t)N * 4;
      dst_off = 128 + (lane - 8) * 16;
    } else if (lane < 20) {
      src0 = reinterpret_cast<const unsigned char*>(tstep + n0) + (lane - 16) * 16; row_stride = (size_t)N * 2;
      dst_off = 256 + (lane - 16) * 16;
    } else {
      src0 = reinterpret_cast<const unsigned char*>(flags + n0) + ((lane - 20) & 1) * 16; row_stride = (size_t)N;
      dst_off = 320 + ((lane - 20) & 1) * 16;
    }
    const bool copier = lane < 22;
    const unsigned int ring_s = (unsigned int)__cvta_generic_to_shared(ring);
    auto stage_chunk = [&](int chunk) {            // chunk c covers steps T-1 - c*SC_CH ... (reverse order), ring slot c % SC_RING
      const int t_hi = T - 1 - chunk * SC_CH;
      const unsigned int slot = ring_s + (unsigned int)((chunk % SC_RING) * SC_CH * SC_ROW_BYTES);
      if (copier) {
#pragma unroll
        for (int u = 0; u < SC_CH; ++u) {
          const int t = t_hi - u;
          if (t >= 0)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(slot + u * SC_ROW_BYTES + dst_off),
                         "l"(src0 + (size_t)t * row_stride) : "memory");
        }
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    };
    const int nchunks = (T + SC_CH - 1) / SC_CH;
#pragma unroll
    for (int c = 0; c < SC_AHEAD; ++c) stage_chunk(c);           // (empty groups past the end keep the counting uniform)
    for (int c = 0; c < nchunks; ++c) {
      stage_chunk(c + SC_AHEAD);
      asm volatile("cp.async.wait_group %0;" ::"n"(SC_AHEAD) : "memory");   // chunk c has landed
      __syncwarp();
      const unsigned char* slot = ring + (c % SC_RING) * SC_CH * SC_ROW_BYTES;
      const int t_hi = T - 1 - c * SC_CH;
#pragma unroll
      for (int u = 0; u < SC_CH; ++u) {
        const int t = t_hi - u;
        if (t < 0) break;
        const unsigned char* row = slot + u * SC_ROW_BYTES;
        const float rwf = reinterpret_cast<const float*>(row)[lane];
        const float bsf = reinterpret_cast<const float*>(row + 128)[lane];
        const unsigned int ts = reinterpret_cast<const unsigned short*>(row + 256)[lane];
        const unsigned int f = (unsigned int)row[320 + lane] | (ts == 0 ? 0x100u : 0u);
        step(t, rwf, bsf, f);
      }
      __syncwarp();                                // the slot is refilled by the next stage_chunk
    }
  } else {
    // the compiler barriers keep the loads of the NEXT chunk ahead of the scan of the current one
    auto scan = [&](const ScanChunk& c, int t_hi) {
#pragma unroll
      for (int u = 0; u < SC_CH; ++u) {
        const int t = t_hi - u;
        if (t >= 0) step(t, c.rw[u], c.bs[u], c.fl[u]);
      }
    };
    ScanChunk ca, cb;
    scan_load(ca, T - 1, N, n, rew, base, flags, tstep);
    for (int t_hi = T - 1; t_hi >= 0; t_hi -= 2 * SC_CH) {
      scan_load(cb, t_hi - SC_CH, N, n, rew, base, flags, tstep);
      asm volatile("" ::: "memory");
      scan(ca, t_hi);
      asm volatile("" ::: "memory");
      scan_load(ca, t_hi - 2 * SC_CH, N, n, rew, base, flags, tstep);
      asm volatile("" ::: "memory");
      scan(cb, t_hi - SC_CH);
      asm volatile("" ::: "memory");
    }
  }
  // the block is one warp: plain warp reductions, lane 0 stores (no shared-memory scratch: the ring owns the budget)
  static_assert(SC_THREADS == 32, "one warp per block");
#pragma unroll
  for (int i = 0; i < B200RL_PS_NSUM; ++i) {
    const double v = warp_sum(s[i]);
    if (lane == 0) partial_sum[(size_t)blockIdx.x * B200RL_PS_NSUM + i] = v;
  }
#pragma unroll
  for (int i = 0; i < B200RL_PS_NMAX; ++i) {
    const double v = warp_max(m[i]);
    if (lane == 0) partial_max[(size_t)blockIdx.x * B200RL_PS_NMAX + i] = v;
  }
}

// (adv - mean) / (std + 1e-8), then optionally (adv - min) + 1e-8   (algos/util.py:7-12)
__global__ void center_adv_kernel(float* __restrict__ adv, long long B, const unsigned char* __restrict__ flags,
                                  const double* __restrict__ sums, const double* __restrict__ maxs, int center,
                                  int positive) {
  const double cnt = sums[2];
  const double mean = sums[0] / cnt;
  double var = sums[1] / cnt - mean * mean;
  if (var < 0.0) var = 0.0;
  const double stdv = sqrt(var) + 1e-8;
  double mn = -maxs[2];
  if (center) mn = (mn - mean) / stdv;
  const long long stride = (long long)gridDim.x * blockDim.x, gt = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  auto one = [&](float a32) {
    double a = (double)a32;
    if (center) a = (a - mean) / stdv;
    if (positive) a = (a - mn) + 1e-8;
    return (float)a;
  };
  long long done = 0;
  if ((((uintptr_t)adv) & 15) == 0 && (flags == nullptr || (((uintptr_t)flags) & 3) == 0)) {
    // four samples per thread: 128-bit loads / stores (the scalar loop ran at 1.7 TB/s)
    const long long nvec = B >> 2;
    for (long long v = gt; v < nvec; v += stride) {
      float4 a4 = reinterpret_cast<float4*>(adv)[v];
      const unsigned int f4 = flags != nullptr ? reinterpret_cast<const unsigned int*>(flags)[v] : 0u;
      if (!(f4 & (unsigned)B200RL_FLAG_MASKED)) a4.x = one(a4.x);          // dropped path: adv stays 0
      if (!((f4 >> 8) & (unsigned)B200RL_FLAG_MASKED)) a4.y = one(a4.y);
      if (!((f4 >> 16) & (unsigned)B200RL_FLAG_MASKED)) a4.z = one(a4.z);
      if (!((f4 >> 24) & (unsigned)B200RL_FLAG_MASKED)) a4.w = one(a4.w);
      reinterpret_cast<float4*>(adv)[v] = a4;
    }
    done = nvec << 2;
  }
  for (long long i = done + gt; i < B; i += stride) {
    if (flags != nullptr && (flags[i] & B200RL_FLAG_MASKED)) continue;   // dropped path: adv stays 0
    adv[i] = one(adv[i]);
  }
}

// Gram matrix of f = [features(d), ret] over samples: upper triangle, float64.
// Tile = 128 samples per block iteration; features staged in shared memory [d+1][TILE+4]; thread p owns pairs
// p, p+blockDim, ...; per-tile float32 dot products, float64 accumulation across tiles.
constexpr int GRAM_TILE = 128;
constexpr int GRAM_LD = GRAM_TILE + 4;
constexpr int GRAM_THREADS = 128;
constexpr int GRAM_MAXPAIRS_PER_THREAD = 9;  // (2*20+5)*(2*20+6)/2 = 1035 pairs / 128 threads

__global__ void __launch_bounds__(GRAM_THREADS)
    lfb_gram_kernel(int O, long long B, const float* __restrict__ obs, const unsigned short* __restrict__ tstep,
                    const float* __restrict__ ret, const unsigned char* __restrict__ flags,
                    double* __restrict__ partial) {
  extern __shared__ __align__(16) float F[];  // [(d+1)][GRAM_LD]
  const int d1 = 2 * O + 5;
  const int npairs = d1 * (d1 + 1) / 2;
  double acc[GRAM_MAXPAIRS_PER_THREAD];
  int pi[GRAM_MAXPAIRS_PER_THREAD], pj[GRAM_MAXPAIRS_PER_THREAD];
#pragma unroll
  for (int q = 0; q < GRAM_MAXPAIRS_PER_THREAD; ++q) {
    acc[q] = 0.0;
    int p = threadIdx.x + q * GRAM_THREADS;
    // decode p -> (i, j), i <= j, row-major upper triangle
    int i = 0, rem = p;
    if (p < npairs) {
      while (rem >= d1 - i) { rem -= d1 - i; ++i; }
      pi[q] = i; pj[q] = i + rem;
    } else {
      pi[q] = 0; pj[q] = 0;
    }
  }
  const long long ntiles = (B + GRAM_TILE - 1) / GRAM_TILE;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long sidx = tile * GRAM_TILE + threadIdx.x;
    __syncthreads();
    if (sidx < B && !(flags != nullptr && (flags[sidx] & B200RL_FLAG_MASKED))) {
      for (int k = 0; k < O; ++k) {
        float o = fminf(fmaxf(obs[(size_t)k * B + sidx], -10.0f), 10.0f);
        F[k * GRAM_LD + threadIdx.x] = o;
        F[(O + k) * GRAM_LD + threadIdx.x] = o * o;
      }
      float al = (float)tstep[sidx] / 100.0f;
      F[(2 * O) * GRAM_LD + threadIdx.x] = al;
      F[(2 * O + 1) * GRAM_LD + threadIdx.x] = al * al;
      F[(2 * O + 2) * GRAM_LD + threadIdx.x] = al * al * al;
      F[(2 * O + 3) * GRAM_LD + threadIdx.x] = 1.0f;
      F[(2 * O + 4) * GRAM_LD + threadIdx.x] = ret[sidx];
    } else {
      for (int k = 0; k < d1; ++k) F[k * GRAM_LD + threadIdx.x] = 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < GRAM_MAXPAIRS_PER_THREAD; ++q) {
      if (threadIdx.x + q * GRAM_THREADS < npairs) {
        const float4* ra = reinterpret_cast<const float4*>(F + pi[q] * GRAM_LD);
        const float4* rb = reinterpret_cast<const float4*>(F + pj[q] * GRAM_LD);
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll 8
        for (int k = 0; k < GRAM_TILE / 4; ++k) {
          float4 a = ra[k], b = rb[k];
          s0 = fmaf(a.x, b.x, s0); s1 = fmaf(a.y, b.y, s1); s2 = fmaf(a.z, b.z, s2); s3 = fmaf(a.w, b.w, s3);
        }
        acc[q] += (double)((s0 + s1) + (s2 + s3));
      }
    }
  }
#pragma unroll
  for (int q = 0; q < GRAM_MAXPAIRS_PER_THREAD; ++q) {
    int p = threadIdx.x + q * GRAM_THREADS;
    if (p < npairs) partial[(size_t)blockIdx.x * npairs + p] = acc[q];
  }
}

// Small observation spaces (O <= 4, i.e. d+1 <= 13 features): the whole upper triangle (<= 91 products) fits in one
// thread's registers, so each thread streams its samples (coalesced across the warp), accumulates the outer products
// in float32 registers (<= ~100 samples per thread), and the block folds them once into float64 -- no shared-memory
// staging, no bank conflicts (the staged kernel above spends its time in 13 M conflicts and LSU latency).
template <int O>
__global__ void __launch_bounds__(128, 3) lfb_gram_reg_kernel(long long B, const float* __restrict__ obs,
                                                           const unsigned short* __restrict__ tstep,
                                                           const float* __restrict__ ret,
                                                           const unsigned char* __restrict__ flags,
                                                           double* __restrict__ partial) {
  constexpr int D1 = 2 * O + 5, NP = D1 * (D1 + 1) / 2;
  __shared__ double red[NP];
  float acc[NP];
#pragma unroll
  for (int p = 0; p < NP; ++p) acc[p] = 0.f;
  for (int p = threadIdx.x; p < NP; p += blockDim.x) red[p] = 0.0;
  __syncthreads();
  const long long stride = (long long)gridDim.x * blockDim.x;
  constexpr int UNR = 4;   // 4 samples' loads in flight per thread (memory-level parallelism; one is latency bound)
  // one sample's outer product into the register triangle
  auto accumulate = [&](const float (&o_raw)[O], float ts, float rt) {
    float f[D1];
#pragma unroll
    for (int k = 0; k < O; ++k) {
      const float o = fminf(fmaxf(o_raw[k], -10.0f), 10.0f);
      f[k] = o;
      f[O + k] = o * o;
    }
    const float al = ts / 100.0f;
    f[2 * O] = al; f[2 * O + 1] = al * al; f[2 * O + 2] = al * al * al; f[2 * O + 3] = 1.0f; f[2 * O + 4] = rt;
    int p = 0;
#pragma unroll
    for (int i = 0; i < D1; ++i)
#pragma unroll
      for (int j = i; j < D1; ++j) { acc[p] = fmaf(f[i], f[j], acc[p]); ++p; }
  };
  long long first_scalar = 0;
  if ((B & 3) == 0) {
    // every plane is 16 B aligned: four consecutive samples per thread with 128-bit loads, two groups in flight
    const long long nvec = B >> 2;
    constexpr int VU = 2;
    for (long long v0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; v0 < nvec; v0 += VU * stride) {
      float4 o4[VU][O], r4[VU];
      ushort4 t4[VU];
      unsigned int f4[VU];
      bool okv[VU];
#pragma unroll
      for (int u = 0; u < VU; ++u) {
        const long long v = v0 + u * stride;
        okv[u] = v < nvec;
        const long long vl = okv[u] ? v : v0;
#pragma unroll
        for (int k = 0; k < O; ++k) o4[u][k] = reinterpret_cast<const float4*>(obs + (size_t)k * B)[vl];
        t4[u] = reinterpret_cast<const ushort4*>(tstep)[vl];
        r4[u] = reinterpret_cast<const float4*>(ret)[vl];
        f4[u] = flags != nullptr ? reinterpret_cast<const unsigned int*>(flags)[vl] : 0u;
      }
#pragma unroll
      for (int u = 0; u < VU; ++u) {
        if (!okv[u]) continue;
        float ov[O];
        if (!(f4[u] & (unsigned)B200RL_FLAG_MASKED)) {
#pragma unroll
          for (int k = 0; k < O; ++k) ov[k] = o4[u][k].x;
          accumulate(ov, (float)t4[u].x, r4[u].x);
        }
        if (!((f4[u] >> 8) & (unsigned)B200RL_FLAG_MASKED)) {
#pragma unroll
          for (int k = 0; k < O; ++k) ov[k] = o4[u][k].y;
          accumulate(ov, (float)t4[u].y, r4[u].y);
        }
        if (!((f4[u] >> 16) & (unsigned)B200RL_FLAG_MASKED)) {
#pragma unroll
          for (int k = 0; k < O; ++k) ov[k] = o4[u][k].z;
          accumulate(ov, (float)t4[u].z, r4[u].z);
        }
        if (!((f4[u] >> 24) & (unsigned)B200RL_FLAG_MASKED)) {
#pragma unroll
          for (int k = 0; k < O; ++k) ov[k] = o4[u][k].w;
          accumulate(ov, (float)t4[u].w, r4[u].w);
        }
      }
    }
    first_scalar = B;
  }
  for (long long s0 = first_scalar + (long long)blockIdx.x * blockDim.x + threadIdx.x; s0 < B; s0 += UNR * stride) {
    float raw[UNR][O + 2];
    bool use[UNR];
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      const long long s = s0 + u * stride;
      const bool ok = s < B;
      const long long sl = ok ? s : s0;
      use[u] = ok && !(flags != nullptr && (flags[sl] & B200RL_FLAG_MASKED));
#pragma unroll
      for (int k = 0; k < O; ++k) raw[u][k] = obs[(size_t)k * B + sl];
      raw[u][O] = (float)tstep[sl];
      raw[u][O + 1] = ret[sl];
    }
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      if (use[u]) {
        float ov[O];
#pragma unroll
        for (int k = 0; k < O; ++k) ov[k] = raw[u][k];
        accumulate(ov, raw[u][O], raw[u][O + 1]);
      }
    }
  }
  // fold: warp shuffle in float64, then one shared-memory add per warp in fixed warp order
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
    if (warp == w) {
#pragma unroll
      for (int p = 0; p < NP; ++p) {
        const double v = warp_sum((double)acc[p]);
        if (lane == 0) red[p] += v;
      }
    }
    __syncthreads();
  }
  for (int p = threadIdx.x; p < NP; p += blockDim.x) partial[(size_t)blockIdx.x * NP + p] = red[p];
}

// Larger observation spaces (obs_dim 6 / 13 / 20: DoublePendulum, Swimmer, Hopper): the d1 x d1 Gram (d1 = 2 O + 5 <= 45)
// in 4x4 register tiles over the upper triangle, as tile_gram.cuh does for dW1: features of a 128-sample tile staged
// feature-major in shared memory, thread = (tile of the upper triangle, K-slice of the 128 samples), 8 LDS.128 per 32
// packed FFMA2, float32 inside a tile and float64 across tiles.  The pair-per-thread kernel above (kept for other
// obs_dim) re-reads two whole rows per pair: 1.25 ms per Swimmer iteration against 0.3 ms here.
template <int O>
struct GramTile {
  static constexpr int D1 = 2 * O + 5, NB = (D1 + 3) / 4, NT = NB * (NB + 1) / 2;      // 4x4 tiles of the upper triangle
  static constexpr int KS = (GRAM_THREADS / NT) < 1 ? 1 : (GRAM_THREADS / NT);           // K-slices per tile
  static constexpr int PER = ((GRAM_TILE / KS + 3) / 4) * 4;                            // samples per slice (multiple of 4)
  static constexpr int ROWS = NB * 4;
  static_assert(NT <= GRAM_THREADS, "one thread per (tile, slice)");
  static constexpr size_t tile_bytes = (size_t)ROWS * GRAM_LD * sizeof(float), scr_bytes = (size_t)KS * NT * 16 * 8;
  static constexpr size_t smem = tile_bytes > scr_bytes ? tile_bytes : scr_bytes;   // the slice-combine scratch reuses it
};

template <int O>
__global__ void __launch_bounds__(GRAM_THREADS, 3)
    lfb_gram_tile_kernel(long long B, const float* __restrict__ obs, const unsigned short* __restrict__ tstep,
                         const float* __restrict__ ret, const unsigned char* __restrict__ flags,
                         double* __restrict__ partial) {
  using G = GramTile<O>;
  constexpr int D1 = G::D1, NB = G::NB, NP = D1 * (D1 + 1) / 2, LD = GRAM_LD;
  extern __shared__ __align__(16) float F[];    // [ROWS][LD]; rows >= D1 stay zero
  const int tid = threadIdx.x;
  // this thread's tile (bi <= bj) and K-slice
  const int tix = tid % G::NT, ks = tid / G::NT;
  const bool worker = ks < G::KS;
  int bi = 0, rem = tix;
  while (rem >= NB - bi) { rem -= NB - bi; ++bi; }
  const int bj = bi + rem;
  const int k_lo = ks * G::PER, k_hi = (k_lo + G::PER < GRAM_TILE) ? k_lo + G::PER : GRAM_TILE;
  double acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
  for (int i = tid; i < G::ROWS * LD; i += GRAM_THREADS) F[i] = 0.f;
  const long long ntiles = (B + GRAM_TILE - 1) / GRAM_TILE;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long sidx = tile * GRAM_TILE + tid;
    __syncthreads();
    if (sidx < B && !(flags != nullptr && (flags[sidx] & B200RL_FLAG_MASKED))) {
      float ov[O];
#pragma unroll
      for (int k = 0; k < O; ++k) ov[k] = obs[(size_t)k * B + sidx];
      const float al = (float)tstep[sidx] / 100.0f, rt = ret[sidx];
#pragma unroll
      for (int k = 0; k < O; ++k) {
        const float o = fminf(fmaxf(ov[k], -10.0f), 10.0f);
        F[k * LD + tid] = o;
        F[(O + k) * LD + tid] = o * o;
      }
      F[(2 * O) * LD + tid] = al;
      F[(2 * O + 1) * LD + tid] = al * al;
      F[(2 * O + 2) * LD + tid] = al * al * al;
      F[(2 * O + 3) * LD + tid] = 1.0f;
      F[(2 * O + 4) * LD + tid] = rt;
    } else {
#pragma unroll
      for (int k = 0; k < D1; ++k) F[k * LD + tid] = 0.0f;
    }
    __syncthreads();
    if (worker) {
      float2 a2[4][4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) a2[r][c] = make_float2(0.f, 0.f);
      const float* U = F + (bi * 4) * LD;
      const float* V = F + (bj * 4) * LD;
#pragma unroll 2
      for (int k = k_lo; k < k_hi; k += 4) {
        float4 u[4], v[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) u[r] = *reinterpret_cast<const float4*>(U + r * LD + k);
#pragma unroll
        for (int c = 0; c < 4; ++c) v[c] = *reinterpret_cast<const float4*>(V + c * LD + k);
        gram_4x4(u, v, a2);
      }
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] += (double)(a2[r][c].x + a2[r][c].y);
    }
  }
  // combine the K-slices of a tile in fixed order through shared memory, then store the upper-triangle entries
  __syncthreads();
  double* scr = reinterpret_cast<double*>(F);     // [KS][NT][16] doubles (GramTile::smem covers it)
  if (worker) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) scr[((size_t)ks * G::NT + tix) * 16 + r * 4 + c] = acc[r][c];
  }
  __syncthreads();
  if (tid < G::NT) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int i = bi * 4 + r, j = bj * 4 + c;
        if (i <= j && j < D1) {
          double v = 0.0;
          for (int q = 0; q < G::KS; ++q) v += scr[((size_t)q * G::NT + tix) * 16 + r * 4 + c];
          partial[(size_t)blockIdx.x * NP + (i * D1 - i * (i - 1) / 2 + (j - i))] = v;
        }
      }
  }
}

template <int O>
static int launch_gram_tile(long long B, const float* obs, const unsigned short* tstep, const float* ret,
                            const unsigned char* flags, double* ws, int* grid_out, cudaStream_t st) {
  using G = GramTile<O>;
  static_assert(G::smem <= 48 * 1024, "default dynamic shared-memory limit");
  long long g = (long long)num_sms() * 3;
  const long long ntiles = (B + GRAM_TILE - 1) / GRAM_TILE;
  if (g > ntiles) g = ntiles;
  if (g > MAX_PARTIAL_BLOCKS) g = MAX_PARTIAL_BLOCKS;
  lfb_gram_tile_kernel<O><<<(unsigned)g, GRAM_THREADS, G::smem, st>>>(B, obs, tstep, ret, flags, ws);
  B200RL_LAUNCH_CHECK("lfb_gram_tile_kernel");
  *grid_out = (int)g;
  return 0;
}

__global__ void planes_to_rows_kernel(int dim, long long B, const float* __restrict__ src, double* __restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  for (int k = 0; k < dim; ++k) dst[i * dim + k] = (double)src[(size_t)k * B + i];
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_process_samples(int obs_dim, int N, int T, const float* obs, const float* rew, unsigned char* flags,
                           const unsigned short* tstep, const double* w, double discount, double gae_lambda,
                           int drop_cut_paths, float* adv, float* ret, float* base, double* sums_out, double* maxs_out,
                           double* ws, void* stream) {
  B200RL_REQUIRE(obs && rew && flags && tstep && adv && ret && base && sums_out && maxs_out && ws,
                 "process_samples: null buffer");
  B200RL_REQUIRE(N > 0 && T > 0 && obs_dim > 0 && obs_dim <= OMAX, "process_samples: bad sizes");
  const int grid = (N + SC_THREADS - 1) / SC_THREADS;          // scan: one thread per lane
  cudaStream_t st = (cudaStream_t)stream;
  double* psum = ws;
  double* pmax = ws + (size_t)grid * B200RL_PS_NSUM;
  B200RL_REQUIRE((long long)grid * (B200RL_PS_NSUM + B200RL_PS_NMAX) <= b200rl_ws_doubles(), "workspace too small");
  const long long B = (long long)N * T;
  if (w == nullptr) {                      // first iteration: the reference's baseline predicts zeros
    B200RL_CUDA_CHECK(cudaMemsetAsync(base, 0, (size_t)B * sizeof(float), st));
  } else {
    long long pg = (B / 4 + PRED_THREADS - 1) / PRED_THREADS;
    const long long cap = (long long)num_sms() * 16;
    if (pg > cap) pg = cap;
    if (pg < 1) pg = 1;
#define B200RL_PRED_LAUNCH(OT) lfb_predict_kernel<OT><<<(unsigned)pg, PRED_THREADS, 0, st>>>(obs_dim, B, obs, tstep, w, base)
    switch (obs_dim) {                 // the obs dims of the compiled envs get an unrolled, vectorised predictor
      case 2: B200RL_PRED_LAUNCH(2); break;
      case 3: B200RL_PRED_LAUNCH(3); break;
      case 4: B200RL_PRED_LAUNCH(4); break;
      case 13: B200RL_PRED_LAUNCH(13); break;
      case 20: B200RL_PRED_LAUNCH(20); break;
      default: B200RL_PRED_LAUNCH(0); break;
    }
#undef B200RL_PRED_LAUNCH
    B200RL_LAUNCH_CHECK("lfb_predict_kernel");
  }
  const bool staged = (N % 32) == 0 && (((uintptr_t)rew | (uintptr_t)base | (uintptr_t)tstep | (uintptr_t)flags) & 15) == 0;
  if (staged)
    gae_scan_kernel<true><<<grid, SC_THREADS, 0, st>>>(N, T, rew, base, flags, tstep, discount, discount * gae_lambda,
                                                       drop_cut_paths, adv, ret, psum, pmax);
  else
    gae_scan_kernel<false><<<grid, SC_THREADS, 0, st>>>(N, T, rew, base, flags, tstep, discount, discount * gae_lambda,
                                                        drop_cut_paths, adv, ret, psum, pmax);
  B200RL_LAUNCH_CHECK("gae_scan_kernel");
  int rc = launch_finalize_sum(psum, grid, B200RL_PS_NSUM, sums_out, 1.0, st);
  if (rc) return rc;
  return launch_finalize_max(pmax, grid, B200RL_PS_NMAX, maxs_out, st);
}

int b200rl_center_advantages(float* adv, long long B, const unsigned char* flags, const double* sums,
                             const double* maxs, int center, int positive, void* stream) {
  B200RL_REQUIRE(adv && sums && maxs && B > 0, "center_advantages: bad arguments");
  if (!center && !positive) return 0;
  long long blocks = (B / 4 + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  center_adv_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(adv, B, flags, sums, maxs, center,
                                                                         positive);
  B200RL_LAUNCH_CHECK("center_adv_kernel");
  return 0;
}

int b200rl_lfb_gram(int obs_dim, long long B, const float* obs, const unsigned short* tstep, const float* ret,
                    const unsigned char* flags, double* gram_out, double* ws, void* stream) {
  B200RL_REQUIRE(obs && tstep && ret && gram_out && ws && B > 0, "lfb_gram: bad arguments");
  B200RL_REQUIRE(obs_dim > 0 && obs_dim <= 20, "lfb_gram: obs_dim must be in 1..20");
  const int d1 = 2 * obs_dim + 5;
  const int npairs = d1 * (d1 + 1) / 2;
  const long long ntiles = (B + GRAM_TILE - 1) / GRAM_TILE;
  int grid = num_sms() * 4;
  if (grid > ntiles) grid = (int)ntiles;
  if (grid > MAX_PARTIAL_BLOCKS) grid = MAX_PARTIAL_BLOCKS;
  const size_t smem = (size_t)d1 * GRAM_LD * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  if (obs_dim <= 4) {
    long long g = (long long)num_sms() * 3;   // 3 resident CTAs (<= 168 registers), one wave
    const long long need = (B / 4 + 127) / 128 + 1;
    if (g > need) g = need;
    grid = (int)g;
    switch (obs_dim) {
      case 1: lfb_gram_reg_kernel<1><<<grid, 128, 0, st>>>(B, obs, tstep, ret, flags, ws); break;
      case 2: lfb_gram_reg_kernel<2><<<grid, 128, 0, st>>>(B, obs, tstep, ret, flags, ws); break;
      case 3: lfb_gram_reg_kernel<3><<<grid, 128, 0, st>>>(B, obs, tstep, ret, flags, ws); break;
      default: lfb_gram_reg_kernel<4><<<grid, 128, 0, st>>>(B, obs, tstep, ret, flags, ws); break;
    }
    B200RL_LAUNCH_CHECK("lfb_gram_reg_kernel");
    return launch_finalize_sum(ws, grid, npairs, gram_out, 1.0, st);
  }
  if (obs_dim == 6 || obs_dim == 13 || obs_dim == 20) {         // the compiled envs: register-tiled kernel
    int rc = obs_dim == 6    ? launch_gram_tile<6>(B, obs, tstep, ret, flags, ws, &grid, st)
             : obs_dim == 13 ? launch_gram_tile<13>(B, obs, tstep, ret, flags, ws, &grid, st)
                             : launch_gram_tile<20>(B, obs, tstep, ret, flags, ws, &grid, st);
    if (rc) return rc;
    return launch_finalize_sum(ws, grid, npairs, gram_out, 1.0, st);
  }
  // smem <= 45 rows x 528 B = 23.8 KB: below the default 48 KB dynamic limit, no attribute needed (and a per-kernel
  // attribute set for a small obs_dim would cap a later, larger one)
  lfb_gram_kernel<<<grid, GRAM_THREADS, smem, st>>>(obs_dim, B, obs, tstep, ret, flags, ws);
  B200RL_LAUNCH_CHECK("lfb_gram_kernel");
  return launch_finalize_sum(ws, grid, npairs, gram_out, 1.0, st);
}

int b200rl_planes_to_rows_f64(int dim, long long B, const float* src, double* dst, void* stream) {
  B200RL_REQUIRE(src && dst && dim > 0 && B > 0, "planes_to_rows: bad arguments");
  planes_to_rows_kernel<<<(unsigned)((B + 255) / 256), 256, 0, (cudaStream_t)stream>>>(dim, B, src, dst);
  B200RL_LAUNCH_CHECK("planes_to_rows_kernel");
  return 0;
}
}
