// r4_gauss.cuh -- the Gaussian policy of the continuous-action env (PPO_conti / A2C_conti) and its learner, as CUDA kernels.
//
//   policy   RLlib 1.5 default FullyConnectedNetwork, vf_share_layers off: obs(256) -> FC 256 tanh -> FC 256 tanh -> fc_out
//            2D (mean | log_std); value branch obs -> FC 256 tanh -> FC 256 tanh -> value_out 1.
//   act      StochasticSampling over DiagGaussian: a = mu + exp(log_std) * N(0,1) (mu when explore = 0).  The noise is
//            counter-based (Box-Muller on splitmix64 keyed by seed, counter + row, dim): the same seed and counter give the
//            same actions.  The env receives clip(a, -1, 1); logp is taken on the unclipped a (clip_actions: True).
//   learner  RLlib 1.5 PPO surrogate loss or A2C summed loss over the DiagGaussian, hand-derived backward, fp32.
//
// Flat parameter layout: fc_1 w[256,256] b[256] | fc_2 w[256,256] b[256] | fc_out w[256,2D] b[2D] |
//                        fc_value_1 w[256,256] b[256] | fc_value_2 w[256,256] b[256] | value_out w[256] b[1].
//
// The gradient runs in two launches per chunk of at most CH samples:
//   k_gauss_rows   one CTA per TS samples: forward of both branches, loss derivatives, backward through the activations;
//                  writes every layer's input rows X and output-gradient rows dZ (no weight gradients).
//   k_gauss_wgrad  one CTA owns one 64 x 64 tile of one dW = X^T dZ (or a bias = column sum of dZ) and walks the samples
//                  in order: every gradient element has exactly one writer and a fixed summation order, so the result is
//                  deterministic without per-CTA partial gradients.  One extra CTA sums the per-sample loss statistics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "r4_ppo.cuh"

namespace r4gauss {

constexpr int OBS = 256, H = 256, TS = 8, NT = 256, MAXD = 64;
constexpr int CH = 2048;                  // samples per gradient chunk (bounds the scratch)
constexpr int NPLANE = 9;                 // x h1 h2 g1 g2 d1 d2 e1 e2, each [CH][256]
constexpr float HALF_LOG_2PI = 0.91893853320467274f;
constexpr float HALF_LOG_2PIE = 1.41893853320467274f;

struct Layout {
  int D, p_w1, p_b1, p_w2, p_b2, p_wo, p_bo, v_w1, v_b1, v_w2, v_b2, v_wo, v_bo, n;
};
__host__ __device__ inline Layout make_layout(int D) {
  Layout L;
  L.D = D;
  L.p_w1 = 0;              L.p_b1 = L.p_w1 + OBS * H;
  L.p_w2 = L.p_b1 + H;     L.p_b2 = L.p_w2 + H * H;
  L.p_wo = L.p_b2 + H;     L.p_bo = L.p_wo + H * 2 * D;
  L.v_w1 = L.p_bo + 2 * D; L.v_b1 = L.v_w1 + OBS * H;
  L.v_w2 = L.v_b1 + H;     L.v_b2 = L.v_w2 + H * H;
  L.v_wo = L.v_b2 + H;     L.v_bo = L.v_wo + H;
  L.n = L.v_bo + 1;
  return L;
}
// scratch floats of the gradient: the planes, dout [CH][2D], dv [CH], per-sample stats [CH][5], gradient sum [n] + its
// 5 statistics (the layout r4comm::k_exchange_adam reads with G = 1), and 5 raw statistic sums
__host__ __device__ inline size_t scratch_floats(int D) {
  return (size_t)CH * (NPLANE * H + 2 * D + 1 + 5) + (size_t)make_layout(D).n + 5 + 5;
}

// out[s][j] = act(sum_k in[s][k] W[k][j] + b[j]) for the TS samples of a tile; thread j owns column j (N <= NT).
template <bool TANH>
__device__ inline void dense_tile(const float* __restrict__ W, const float* __restrict__ b, const float* in, int K, int N,
                                  float* out) {
  const int j = threadIdx.x;
  if (j < N) {
    float acc[TS];
#pragma unroll
    for (int s = 0; s < TS; ++s) acc[s] = 0.f;
#pragma unroll 4
    for (int k = 0; k < K; ++k) {
      const float w = __ldg(W + (size_t)k * N + j);
#pragma unroll
      for (int s = 0; s < TS; ++s) acc[s] = fmaf(in[s * K + k], w, acc[s]);
    }
    const float bj = __ldg(b + j);
#pragma unroll
    for (int s = 0; s < TS; ++s) out[s * N + j] = TANH ? tanhf(acc[s] + bj) : acc[s] + bj;
  }
  __syncthreads();
}

// din[s][j] = (sum_c dout[s][c] W[j][c]) (1 - a[s][j]^2) for j < 256 (the tanh layer whose output a fed W); N % 4 == 0.
__device__ inline void dense_back_tile(const float* __restrict__ W, const float* dout, int N, const float* a, float* din) {
  const int j = threadIdx.x;
  float acc[TS];
#pragma unroll
  for (int s = 0; s < TS; ++s) acc[s] = 0.f;
  const float4* w4 = reinterpret_cast<const float4*>(W + (size_t)j * N);
  for (int c4 = 0; c4 < N / 4; ++c4) {
    const float4 w = __ldg(w4 + c4);
#pragma unroll
    for (int s = 0; s < TS; ++s) {
      const float* d = dout + s * N + 4 * c4;
      acc[s] = fmaf(d[0], w.x, fmaf(d[1], w.y, fmaf(d[2], w.z, fmaf(d[3], w.w, acc[s]))));
    }
  }
#pragma unroll
  for (int s = 0; s < TS; ++s) { const float h = a[s * H + j]; din[s * H + j] = acc[s] * (1.f - h * h); }
  __syncthreads();
}

// Shared memory: x, h1, h2, g1, g2 [TS][256], o [TS][2D] (dist inputs) and the values; the gradient rows kernel adds two
// [TS][256] backward buffers and the value gradients.
constexpr size_t ACT_SMEM = (size_t)(5 * TS * H + TS * 2 * MAXD + TS) * 4;
constexpr size_t ROWS_SMEM = (size_t)(7 * TS * H + TS * 2 * MAXD + 2 * TS) * 4;

// Forward of both branches for the TS rows src[0..TS) (rows >= nvalid are zero observations).
__device__ inline void forward_rows(const Layout& L, const float* __restrict__ prm, const float* __restrict__ obs,
                                    const int64_t* src, int nvalid, float* x, float* h1, float* h2, float* g1, float* g2,
                                    float* o, float* val) {
  const int tid = threadIdx.x;
  for (int i = tid; i < TS * OBS / 4; i += NT) {
    const int s = i / (OBS / 4), k4 = i % (OBS / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (s < nvalid) v = __ldg(reinterpret_cast<const float4*>(obs + src[s] * OBS) + k4);
    reinterpret_cast<float4*>(x)[i] = v;
  }
  __syncthreads();
  dense_tile<true>(prm + L.p_w1, prm + L.p_b1, x, OBS, H, h1);
  dense_tile<true>(prm + L.p_w2, prm + L.p_b2, h1, H, H, h2);
  dense_tile<false>(prm + L.p_wo, prm + L.p_bo, h2, H, 2 * L.D, o);
  dense_tile<true>(prm + L.v_w1, prm + L.v_b1, x, OBS, H, g1);
  dense_tile<true>(prm + L.v_w2, prm + L.v_b2, g1, H, H, g2);
  {  // value = g2 . wo + bo: one warp per sample
    const int warp = tid >> 5, lane = tid & 31;
    for (int s = warp; s < TS; s += NT / 32) {
      float a = 0.f;
      for (int k = lane; k < H; k += 32) a = fmaf(g2[s * H + k], __ldg(prm + L.v_wo + k), a);
      a = r4ppo::warp_sum(a);
      if (lane == 0) val[s] = a + __ldg(prm + L.v_bo);
    }
  }
  __syncthreads();
}

__device__ __forceinline__ float gauss_noise(uint64_t seed, uint64_t counter, int64_t row, int dim) {
  const uint64_t r = r4ppo::splitmix64(seed ^ r4ppo::splitmix64(((counter + (uint64_t)row) << 6) + (uint64_t)dim));
  const float u1 = ((float)(r >> 40) + 0.5f) * (1.0f / 16777216.0f);            // (0, 1)
  const float u2 = (float)((r >> 16) & 0xFFFFFFull) * (1.0f / 16777216.0f);     // [0, 1)
  return sqrtf(-2.f * logf(u1)) * cospif(2.f * u2);
}

// ------------------------------------------------------------------------------------------------
// act: forward, sample (or mean), clip; writes the unclipped action, the env action, logp, value, dist inputs.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) k_gauss_act(Layout L, const float* __restrict__ prm, const float* __restrict__ obs, int B,
                                                  int explore, uint64_t seed, uint64_t counter, float* __restrict__ action,
                                                  float* __restrict__ env_action, float* __restrict__ logp,
                                                  float* __restrict__ value, float* __restrict__ dist_out) {
  extern __shared__ __align__(16) float sm[];
  float *x = sm, *h1 = x + TS * H, *h2 = h1 + TS * H, *g1 = h2 + TS * H, *g2 = g1 + TS * H;
  float *o = g2 + TS * H, *val = o + TS * 2 * MAXD;
  __shared__ int64_t src[TS];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, D = L.D;
  const int s0 = blockIdx.x * TS, nvalid = min(TS, B - s0);
  if (tid < TS) src[tid] = min(s0 + tid, B - 1);
  __syncthreads();
  forward_rows(L, prm, obs, src, nvalid, x, h1, h2, g1, g2, o, val);
  for (int s = warp; s < nvalid; s += NT / 32) {
    const int64_t row = s0 + s;
    float q = 0.f, sls = 0.f;
    for (int i = lane; i < D; i += 32) {
      const float mu = o[s * 2 * D + i], ls = o[s * 2 * D + D + i], sd = expf(ls);
      const float a = explore ? fmaf(sd, gauss_noise(seed, counter, row, i), mu) : mu;
      const float z = (a - mu) / sd;
      q = fmaf(z, z, q); sls += ls;
      action[row * D + i] = a;
      env_action[row * D + i] = fminf(fmaxf(a, -1.f), 1.f);
    }
    q = r4ppo::warp_sum(q); sls = r4ppo::warp_sum(sls);
    if (lane == 0) { logp[row] = -0.5f * q - sls - HALF_LOG_2PI * D; value[row] = val[s]; }
    if (dist_out)
      for (int i = lane; i < 2 * D; i += 32) dist_out[row * 2 * D + i] = o[s * 2 * D + i];
  }
}

// ------------------------------------------------------------------------------------------------
// gradient, part 1: per-sample rows.  Positions p = c0 .. c0+cn of the sample list (idx[p], or p when idx == nullptr);
// row q = p - c0 of every plane.  mode 0 = PPO (loss mean: inv_n), mode 1 = A2C (sums).
// ------------------------------------------------------------------------------------------------
struct Planes {
  float *x, *h1, *h2, *g1, *g2, *d1, *d2, *e1, *e2, *dout, *dv, *stats;
};
__host__ __device__ inline Planes make_planes(float* scratch, int D) {
  Planes P;
  float* p = scratch;
  float** pl[NPLANE] = {&P.x, &P.h1, &P.h2, &P.g1, &P.g2, &P.d1, &P.d2, &P.e1, &P.e2};
  for (int k = 0; k < NPLANE; ++k) { *pl[k] = p; p += (size_t)CH * H; }
  P.dout = p; p += (size_t)CH * 2 * D;
  P.dv = p; p += CH;
  P.stats = p;
  return P;
}

__global__ void __launch_bounds__(NT) k_gauss_rows(Layout L, r4ppo::LossHyper hp, const float* __restrict__ prm, const float* __restrict__ obs,
                                                   const float* __restrict__ action, const float* __restrict__ old_logp,
                                                   const float* __restrict__ old_dist, const float* __restrict__ old_value,
                                                   const float* __restrict__ adv, const float* __restrict__ target,
                                                   const int64_t* __restrict__ idx, int c0, int cn, Planes P) {
  extern __shared__ __align__(16) float sm[];
  float *x = sm, *h1 = x + TS * H, *h2 = h1 + TS * H, *g1 = h2 + TS * H, *g2 = g1 + TS * H, *da = g2 + TS * H, *db = da + TS * H;
  float *o = db + TS * H, *val = o + TS * 2 * MAXD, *dvs = val + TS;
  __shared__ int64_t src[TS];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, D = L.D, N2 = 2 * D;
  const int q0 = blockIdx.x * TS, nvalid = min(TS, cn - q0);
  if (tid < TS) { const int p = c0 + min(q0 + tid, cn - 1); src[tid] = idx ? idx[p] : (int64_t)p; }
  __syncthreads();
  forward_rows(L, prm, obs, src, nvalid, x, h1, h2, g1, g2, o, val);
  // ---- per-sample loss derivatives w.r.t. (mu, log_std) and the value: one warp per sample ----
  for (int s = warp; s < TS; s += NT / 32) {
    float* od = o + s * N2;
    if (s >= nvalid) {
      for (int i = lane; i < N2; i += 32) od[i] = 0.f;
      if (lane == 0) dvs[s] = 0.f;
      continue;
    }
    const int64_t r = src[s];
    float q = 0.f, sls = 0.f, kl = 0.f;
    for (int i = lane; i < D; i += 32) {
      const float mu = od[i], ls = od[D + i], z = (__ldg(action + r * D + i) - mu) / expf(ls);
      q = fmaf(z, z, q); sls += ls;
      if (old_dist) {
        const float muo = __ldg(old_dist + r * N2 + i), lso = __ldg(old_dist + r * N2 + D + i), so = expf(lso);
        const float dm = muo - mu, s2 = expf(2.f * ls);
        kl += ls - lso + (so * so + dm * dm) / (2.f * s2) - 0.5f;
      }
    }
    q = r4ppo::warp_sum(q); sls = r4ppo::warp_sum(sls); kl = r4ppo::warp_sum(kl);
    const float logp = -0.5f * q - sls - HALF_LOG_2PI * D;
    const float ent = sls + HALF_LOG_2PIE * D;
    const float advv = adv[r], tg = target[r], v = val[s];
    const r4ppo::SampleLoss sl = r4ppo::sample_loss(hp, logp, hp.mode == 0 ? old_logp[r] : 0.f, advv, tg, v,
                                                    hp.mode == 0 ? old_value[r] : 0.f, kl, ent);
    // d logp / d mu = z / sd, d logp / d ls = z^2 - 1; d ent / d ls = 1;
    // d kl / d mu = (mu - mu_o) / sd^2, d kl / d ls = 1 - (sd_o^2 + (mu_o - mu)^2) / sd^2
    for (int i = lane; i < D; i += 32) {
      const float mu = od[i], ls = od[D + i], sd = expf(ls), z = (__ldg(action + r * D + i) - mu) / sd;
      float gm = sl.ca * (z / sd), gl = sl.ca * (z * z - 1.f) - sl.cent;
      if (old_dist && sl.ckl != 0.f) {
        const float muo = __ldg(old_dist + r * N2 + i), so = expf(__ldg(old_dist + r * N2 + D + i));
        const float dm = muo - mu, s2 = expf(2.f * ls);
        gm = fmaf(sl.ckl, -dm / s2, gm);
        gl = fmaf(sl.ckl, 1.f - (so * so + dm * dm) / s2, gl);
      }
      od[i] = gm; od[D + i] = gl;
    }
    if (lane == 0) {
      dvs[s] = sl.dv;
      float* st = P.stats + (size_t)(q0 + s) * 5;
      st[0] = sl.pl; st[1] = sl.vl; st[2] = sl.kl; st[3] = sl.ent; st[4] = sl.total;
    }
  }
  __syncthreads();
  // ---- backward through the activations: policy d2 = dout W_o^T (1-h2^2), d1 = d2 W_2^T (1-h1^2) ----
  dense_back_tile(prm + L.p_wo, o, N2, h2, db);
  dense_back_tile(prm + L.p_w2, db, H, h1, da);
  // store the policy planes (x, h1, h2 inputs; d1, d2, dout gradients), then reuse da / db for the value branch
  for (int i = tid; i < nvalid * H; i += NT) {
    const size_t q = (size_t)q0 * H + i;
    P.x[q] = x[i]; P.h1[q] = h1[i]; P.h2[q] = h2[i]; P.g1[q] = g1[i]; P.g2[q] = g2[i]; P.d1[q] = da[i]; P.d2[q] = db[i];
  }
  for (int i = tid; i < nvalid * N2; i += NT) P.dout[(size_t)q0 * N2 + i] = o[i];
  if (tid < nvalid) P.dv[q0 + tid] = dvs[tid];
  __syncthreads();
  // value branch: e2 = dv w_vo (1-g2^2), e1 = e2 W_v2^T (1-g1^2)
  for (int i = tid; i < TS * H; i += NT) {
    const int s = i / H, k = i % H;
    const float g = g2[i];
    db[i] = dvs[s] * __ldg(prm + L.v_wo + k) * (1.f - g * g);
  }
  __syncthreads();
  dense_back_tile(prm + L.v_w2, db, H, g1, da);
  for (int i = tid; i < nvalid * H; i += NT) {
    const size_t q = (size_t)q0 * H + i;
    P.e1[q] = da[i]; P.e2[q] = db[i];
  }
}

// ------------------------------------------------------------------------------------------------
// gradient, part 2: weight gradients.  Job j: out[i][c] (+)= sum_q X[q][i] dZ[q][c] over the cn rows (X == nullptr: a
// bias, X = 1 and M = 1).  64 x 64 output tile per CTA, 4 x 4 per thread; first chunk stores, later chunks add.
// ------------------------------------------------------------------------------------------------
constexpr int NJOB = 12, WT = 64, WK = 32;
struct Job {
  const float* X;
  const float* Z;
  int M, N, off, tile0;
};
struct Jobs {
  Job j[NJOB];
  int ntiles;
};

__global__ void __launch_bounds__(NT) k_gauss_wgrad(Jobs jobs, int cn, int first, float* __restrict__ grad,
                                                    const float* __restrict__ stats, float* __restrict__ stat_sum,
                                                    float* __restrict__ stats_accum, float stat_scale) {
  __shared__ float xs[WK][WT];
  __shared__ float zs[WK][WT];
  const int tid = threadIdx.x;
  if ((int)blockIdx.x == jobs.ntiles) {                    // the loss statistics, summed in sample order
    if (tid < 5) {
      float a = first ? 0.f : stat_sum[tid];
      for (int q = 0; q < cn; ++q) a += stats[q * 5 + tid];
      stat_sum[tid] = a;
      if (stats_accum) stats_accum[tid] += a * stat_scale;
    }
    return;
  }
  int jb = 0;
  while (jb + 1 < NJOB && (int)blockIdx.x >= jobs.j[jb + 1].tile0) ++jb;
  const Job J = jobs.j[jb];
  const int t = blockIdx.x - J.tile0, tn = (J.N + WT - 1) / WT;
  const int i0 = (t / tn) * WT, c0 = (t % tn) * WT;
  const int ty = tid / 16, tx = tid % 16;                  // rows i0 + 4 ty .. +3, columns c0 + 4 tx .. +3
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
  for (int k0 = 0; k0 < cn; k0 += WK) {
    __syncthreads();
    for (int e = tid; e < WK * WT; e += NT) {
      const int k = e / WT, c = e % WT, q = k0 + k;
      const bool ok = q < cn;
      xs[k][c] = (ok && i0 + c < J.M) ? (J.X ? J.X[(size_t)q * J.M + i0 + c] : 1.f) : 0.f;
      zs[k][c] = (ok && c0 + c < J.N) ? J.Z[(size_t)q * J.N + c0 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < WK; ++k) {
      float xv[4], zv[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) { xv[a] = xs[k][4 * ty + a]; zv[a] = zs[k][4 * tx + a]; }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fmaf(xv[a], zv[b], acc[a][b]);
    }
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int i = i0 + 4 * ty + a;
    if (i >= J.M) continue;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int c = c0 + 4 * tx + b;
      if (c >= J.N) continue;
      float* g = grad + J.off + (size_t)i * J.N + c;
      *g = first ? acc[a][b] : *g + acc[a][b];
    }
  }
}

// The twelve jobs of one chunk, in parameter order.
inline Jobs make_jobs(const Layout& L, const Planes& P) {
  Jobs J;
  const int D2 = 2 * L.D;
  const Job list[NJOB] = {
      {P.x, P.d1, OBS, H, L.p_w1, 0},     {nullptr, P.d1, 1, H, L.p_b1, 0},
      {P.h1, P.d2, H, H, L.p_w2, 0},      {nullptr, P.d2, 1, H, L.p_b2, 0},
      {P.h2, P.dout, H, D2, L.p_wo, 0},   {nullptr, P.dout, 1, D2, L.p_bo, 0},
      {P.x, P.e1, OBS, H, L.v_w1, 0},     {nullptr, P.e1, 1, H, L.v_b1, 0},
      {P.g1, P.e2, H, H, L.v_w2, 0},      {nullptr, P.e2, 1, H, L.v_b2, 0},
      {P.g2, P.dv, H, 1, L.v_wo, 0},      {nullptr, P.dv, 1, 1, L.v_bo, 0}};
  int t = 0;
  for (int k = 0; k < NJOB; ++k) {
    J.j[k] = list[k];
    J.j[k].tile0 = t;
    t += ((list[k].M + WT - 1) / WT) * ((list[k].N + WT - 1) / WT);
  }
  J.ntiles = t;
  return J;
}

}  // namespace r4gauss
