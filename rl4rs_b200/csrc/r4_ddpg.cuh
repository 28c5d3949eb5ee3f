// r4_ddpg.cuh -- DDPG / TD3 on the continuous-action env: the deterministic actor, the device replay and the actor-critic
// learner, as fp32 CUDA kernels (no tensor cores: parity with autograd is the bar, DESIGN.md section 7).
//
//   actor    obs(256) -> 400 relu -> 300 relu -> D, squashed (high - low) sigmoid(2x) + low = tanh(x) on Box(-1, 1)
//   critic   concat(obs, a) (288) -> 400 relu -> 300 relu -> 1; TD3 adds a twin critic with its own weights
//   act      mode 0 the actor output, 1 Ornstein-Uhlenbeck noise around it (one state per policy, shared by every row),
//            2 U(-1, 1) per row and dimension (the random phase).  Counter-based draws keyed by (seed, counter + row, dim).
//   replay   a ring of transitions in caller-owned device arrays; uniform or proportional (prioritized) sampling from
//            caller-supplied uniforms; priority update where the later position of a repeated index wins.
//   learner  critic loss mean(w * (td1^2 + td2^2) / 2), actor loss -mean Q1(s, pi(s)), hand-derived backward.
//
// Flat parameter layout: actor  w1[256,400] b1[400] w2[400,300] b2[300] w3[300,D] b3[D] |
//                        critic w1[288,400] b1[400] w2[400,300] b2[300] w3[300] b3[1] | twin critic (TD3) as the critic.
// The target parameters have the same layout, so the soft update is one pass over one buffer.
//
// The gradient runs in two launches:
//   k_ddpg_rows   one CTA per TS samples: target actor (+ smoothing) and target critic(s) on s', the critic(s) on (s, a),
//                 the TD errors, Q1(s, pi(s)), and the backward rows of both losses; writes every layer's input rows X and
//                 output-gradient rows dZ to the scratch planes.
//   r4dense::k_dense_wgrad  one CTA per 64 x 64 tile of one dW = X^T dZ (or a bias), walking the samples in order:
//                 deterministic, every element has one writer.  One extra CTA sums the loss statistics.
// k_ddpg_apply then adds the l2 terms, runs both Adams (the actor's skipped on delayed steps) and the soft target update.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "r4_dense.cuh"
#include "r4_ppo.cuh"

namespace r4ddpg {

constexpr int OBS = 256, H1 = 400, H2 = 300, TS = 8, NT = 256, MAXD = 32;
constexpr int XIN = OBS + MAXD;          // row stride of the [s | a] plane

struct Net {                             // one MLP inside the flat buffer: w1 b1 w2 b2 w3 b3
  int w1, b1, w2, b2, w3, b3, K, N3, end;
};
__host__ __device__ inline Net make_net(int off, int K, int N3) {
  Net n;
  n.K = K; n.N3 = N3;
  n.w1 = off;             n.b1 = n.w1 + K * H1;
  n.w2 = n.b1 + H1;       n.b2 = n.w2 + H1 * H2;
  n.w3 = n.b2 + H2;       n.b3 = n.w3 + H2 * N3;
  n.end = n.b3 + N3;
  return n;
}
struct Layout {
  int D, twin;
  Net actor, q1, q2;
  int n;
};
__host__ __device__ inline Layout make_layout(int D, int twin) {
  Layout L;
  L.D = D; L.twin = twin;
  L.actor = make_net(0, OBS, D);
  L.q1 = make_net(L.actor.end, OBS + D, 1);
  L.q2 = make_net(L.q1.end, OBS + D, 1);
  L.n = twin ? L.q2.end : L.q1.end;
  return L;
}

// Scratch planes of the learner, n rows each.
struct Planes {
  float *x;                               // [n][XIN]   s | a (the critic input; the actor reads its first 256 columns)
  float *ch1[2], *ch2[2], *cd1[2], *cd2[2], *cd3[2];   // critic k: h1 [n][400], h2 [n][300], dZ1, dZ2, dZ3 [n]
  float *ah1, *ah2, *ad1, *ad2, *ad3;     // actor: h1, h2, dZ1, dZ2, dZ3 [n][D]
  float *td, *stats;                      // td1 [n], per-sample statistics [n][3]
  float *grad;                            // [np + 5]: the gradient, then 5 zero statistics (the r4_grad_exchange_n layout)
  float *weights;                         // [n] importance weights of the sampled batch
  int64_t* idx;                           // [n] sampled indices
};
__host__ __device__ inline size_t row_floats(int D, int twin) {
  return XIN + (size_t)(twin ? 2 : 1) * (2 * H1 + 2 * H2 + 1) + 2 * H1 + 2 * H2 + D + 1 + 3 + 1 + 2;
}
__host__ __device__ inline size_t scratch_floats(int D, int twin, int n) {
  return (size_t)n * row_floats(D, twin) + 2 * (size_t)make_layout(D, twin).n + 5 + 4;   // + the summed gradient [np]
}
__host__ __device__ inline Planes make_planes(float* s, int D, int twin, int n) {
  Planes P;
  float* p = s;
  auto take = [&](size_t k) { float* q = p; p += k; return q; };
  P.idx = reinterpret_cast<int64_t*>(take((size_t)2 * n));      // first: the scratch base is 8-byte aligned
  P.x = take((size_t)n * XIN);
  for (int k = 0; k < 2; ++k) {
    const bool on = k == 0 || twin;
    P.ch1[k] = on ? take((size_t)n * H1) : nullptr; P.ch2[k] = on ? take((size_t)n * H2) : nullptr;
    P.cd1[k] = on ? take((size_t)n * H1) : nullptr; P.cd2[k] = on ? take((size_t)n * H2) : nullptr;
    P.cd3[k] = on ? take((size_t)n) : nullptr;
  }
  P.ah1 = take((size_t)n * H1); P.ah2 = take((size_t)n * H2);
  P.ad1 = take((size_t)n * H1); P.ad2 = take((size_t)n * H2); P.ad3 = take((size_t)n * D);
  P.td = take(n); P.stats = take((size_t)n * 3); P.weights = take(n);
  P.grad = take((size_t)make_layout(D, twin).n + 5);
  return P;
}

// out[s][j] = act(sum_k in[s][k] W[k][j] + b[j]) for the TS rows of a tile (row strides ldi / ldo); ACT 0 none, 1 relu, 2 tanh.
template <int ACT>
__device__ inline void dense(const float* __restrict__ W, const float* __restrict__ b, const float* in, int ldi, int K, int N,
                             float* out, int ldo) {
  for (int j = threadIdx.x; j < N; j += NT) {
    float acc[TS];
#pragma unroll
    for (int s = 0; s < TS; ++s) acc[s] = 0.f;
#pragma unroll 4
    for (int k = 0; k < K; ++k) {
      const float w = __ldg(W + (size_t)k * N + j);
#pragma unroll
      for (int s = 0; s < TS; ++s) acc[s] = fmaf(in[s * ldi + k], w, acc[s]);
    }
    const float bj = __ldg(b + j);
#pragma unroll
    for (int s = 0; s < TS; ++s) {
      const float z = acc[s] + bj;
      out[s * ldo + j] = ACT == 1 ? fmaxf(z, 0.f) : ACT == 2 ? tanhf(z) : z;
    }
  }
  __syncthreads();
}

// din[s][k] = (sum_c dz[s][c] W[k0 + k][c]) * (a == nullptr ? 1 : [a[s][k] > 0]) for k < K (the relu layer whose output a
// fed W's rows k0 ..).
__device__ inline void dense_back(const float* __restrict__ W, int k0, const float* dz, int N, int K, const float* a, float* din,
                                  int ldo) {
  for (int k = threadIdx.x; k < K; k += NT) {
    float acc[TS];
#pragma unroll
    for (int s = 0; s < TS; ++s) acc[s] = 0.f;
    const float* wr = W + (size_t)(k0 + k) * N;
    for (int c = 0; c < N; ++c) {
      const float w = __ldg(wr + c);
#pragma unroll
      for (int s = 0; s < TS; ++s) acc[s] = fmaf(dz[s * N + c], w, acc[s]);
    }
#pragma unroll
    for (int s = 0; s < TS; ++s) din[s * ldo + k] = (a && a[s * ldo + k] <= 0.f) ? 0.f : acc[s];
  }
  __syncthreads();
}

// q[s] = h2[s] . w3 + b3, one warp per row.
__device__ inline void head(const float* __restrict__ prm, const Net& q, const float* h2, float* out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int s = warp; s < TS; s += NT / 32) {
    float a = 0.f;
    for (int k = lane; k < H2; k += 32) a = fmaf(h2[s * H2 + k], __ldg(prm + q.w3 + k), a);
    a = r4ppo::warp_sum(a);
    if (lane == 0) out[s] = a + __ldg(prm + q.b3);
  }
  __syncthreads();
}

// The actor on the TS rows of x (stride XIN) -> h1, h2 and the squashed action a[s][0..D) (stride lda).
__device__ inline void actor_fwd(const float* __restrict__ prm, const Layout& L, const float* x, float* h1, float* h2, float* a,
                                 int lda) {
  dense<1>(prm + L.actor.w1, prm + L.actor.b1, x, XIN, OBS, H1, h1, H1);
  dense<1>(prm + L.actor.w2, prm + L.actor.b2, h1, H1, H1, H2, h2, H2);
  dense<2>(prm + L.actor.w3, prm + L.actor.b3, h2, H2, H2, L.D, a, lda);
}
// A critic on the TS rows of x = [s | a] (stride XIN) -> h1, h2 and q.
__device__ inline void critic_fwd(const float* __restrict__ prm, const Net& q, int K, const float* x, float* h1, float* h2,
                                  float* out) {
  dense<1>(prm + q.w1, prm + q.b1, x, XIN, K, H1, h1, H1);
  dense<1>(prm + q.w2, prm + q.b2, h1, H1, H1, H2, h2, H2);
  head(prm, q, h2, out);
}

__device__ __forceinline__ uint64_t draw(uint64_t seed, uint64_t counter, int64_t row, int dim) {
  return r4ppo::splitmix64(seed ^ r4ppo::splitmix64(((counter + (uint64_t)row) << 6) + (uint64_t)dim));
}
__device__ __forceinline__ float uniform_pm1(uint64_t r) {            // U[-1, 1) from the top 24 bits
  return (float)(r >> 40) * (2.0f / 16777216.0f) - 1.f;
}
__device__ __forceinline__ float normal(uint64_t r) {                 // Box-Muller, as r4gauss::gauss_noise
  const float u1 = ((float)(r >> 40) + 0.5f) * (1.0f / 16777216.0f);
  const float u2 = (float)((r >> 16) & 0xFFFFFFull) * (1.0f / 16777216.0f);
  return sqrtf(-2.f * logf(u1)) * cospif(2.f * u2);
}

// ------------------------------------------------------------------------------------------------
// act.  mode 1 (OU): x' = x + theta (-x) + sigma N(0, I) with the draws (seed, counter, row 0, dim); every CTA computes the
// same x' and CTA 0 stores it in ou_out (ou_in != ou_out: the caller alternates two buffers); a = clip(mu + ns x', -1, 1)
// with ns = scale * base_scale * (high - low).  mode 2: a = U(-1, 1) from (seed, counter, row, dim).
// ------------------------------------------------------------------------------------------------
constexpr size_t ACT_SMEM = (size_t)(TS * XIN + TS * H1 + TS * H2 + TS * MAXD + MAXD) * 4;

__global__ void __launch_bounds__(NT) k_ddpg_act(Layout L, const float* __restrict__ prm, const float* __restrict__ obs, int B,
                                                 int mode, uint64_t seed, uint64_t counter, const float* __restrict__ ou_in,
                                                 float* __restrict__ ou_out, float theta, float sigma, float ns,
                                                 float* __restrict__ action) {
  extern __shared__ __align__(16) float sm[];
  float *x = sm, *h1 = x + TS * XIN, *h2 = h1 + TS * H1, *a = h2 + TS * H2, *ou = a + TS * MAXD;
  const int tid = threadIdx.x, D = L.D;
  const int s0 = blockIdx.x * TS, nvalid = min(TS, B - s0);
  if (mode == 2) {
    for (int i = tid; i < nvalid * D; i += NT) {
      const int s = i / D, d = i % D;
      action[(size_t)(s0 + s) * D + d] = uniform_pm1(draw(seed, counter, s0 + s, d));
    }
    return;
  }
  for (int i = tid; i < TS * OBS; i += NT) {
    const int s = i / OBS, k = i % OBS;
    x[s * XIN + k] = s < nvalid ? __ldg(obs + (size_t)(s0 + s) * OBS + k) : 0.f;
  }
  if (mode == 1 && tid < D) {
    const float xo = ou_in[tid];
    const float xn = xo + (theta * -xo + sigma * normal(draw(seed, counter, 0, tid)));
    ou[tid] = xn;
    if (blockIdx.x == 0) ou_out[tid] = xn;
  }
  __syncthreads();
  actor_fwd(prm, L, x, h1, h2, a, MAXD);
  for (int i = tid; i < nvalid * D; i += NT) {
    const int s = i / D, d = i % D;
    float v = a[s * MAXD + d];
    if (mode == 1) v = fminf(fmaxf(v + ns * ou[d], -1.f), 1.f);
    action[(size_t)(s0 + s) * D + d] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// replay
// ------------------------------------------------------------------------------------------------
// Row r = t * B + b of a [T, B] rollout goes to slot (pos + r) % C; new_obs is obs of row r + B, or final_obs[b] on the last
// step.  Only the last C rows are written when T * B > C (earlier ones would be overwritten in the same call).  New items get
// priority max_prio^alpha.
__global__ void k_replay_store(float* __restrict__ r_obs, float* __restrict__ r_act, float* __restrict__ r_rew,
                               float* __restrict__ r_new, uint8_t* __restrict__ r_done, float* __restrict__ r_prio,
                               const float* __restrict__ max_prio, int C, int D, int64_t pos, float alpha,
                               const float* __restrict__ obs, const float* __restrict__ final_obs,
                               const float* __restrict__ act, const float* __restrict__ rew, const uint8_t* __restrict__ done,
                               int T, int B) {
  const int64_t n = (int64_t)T * B, first = n > C ? n - C : 0;
  const int64_t r = first + blockIdx.x;
  if (r >= n) return;
  const int64_t slot = (pos + r) % C;
  const float* nx = r + B < n ? obs + (r + B) * OBS : final_obs + (r % B) * OBS;
  for (int k = threadIdx.x; k < OBS; k += blockDim.x) {
    r_obs[slot * OBS + k] = obs[r * OBS + k];
    r_new[slot * OBS + k] = nx[k];
  }
  for (int k = threadIdx.x; k < D; k += blockDim.x) r_act[slot * D + k] = act[r * D + k];
  if (threadIdx.x == 0) {
    r_rew[slot] = rew[r];
    r_done[slot] = done[r];
    if (r_prio) r_prio[slot] = powf(max_prio[0], alpha);
  }
}

// One CTA.  prio == nullptr: idx = min(floor(u * size), size - 1), weight 1.  Otherwise proportional: mass = u * total,
// idx = the first i with prefix(i) > mass (prefix sums in float64, in a fixed order), weight (p_i N)^-beta / (p_min N)^-beta.
constexpr int SNT = 1024;
__global__ void __launch_bounds__(SNT) k_replay_sample(const float* __restrict__ prio, int size, int n, float beta,
                                                       const float* __restrict__ u, int64_t* __restrict__ idx,
                                                       float* __restrict__ weights) {
  __shared__ double part[SNT + 1];
  __shared__ float pmin[SNT / 32];
  const int tid = threadIdx.x;
  if (!prio) {
    for (int i = tid; i < n; i += SNT) {
      idx[i] = min((int64_t)((double)u[i] * size), (int64_t)size - 1);
      weights[i] = 1.f;
    }
    return;
  }
  const int per = (size + SNT - 1) / SNT;
  const int lo = min(tid * per, size), hi = min(lo + per, size);
  double s = 0.0;
  float mn = 3.4e38f;
  for (int i = lo; i < hi; ++i) { s += (double)prio[i]; mn = fminf(mn, prio[i]); }
  part[tid + 1] = s;
  for (int o = 16; o > 0; o >>= 1) mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  if ((tid & 31) == 0) pmin[tid >> 5] = mn;
  __syncthreads();
  if (tid == 0) {                        // exclusive prefix of the chunk sums, in chunk order
    part[0] = 0.0;
    for (int c = 1; c <= SNT; ++c) part[c] += part[c - 1];
    float m = pmin[0];
    for (int w = 1; w < SNT / 32; ++w) m = fminf(m, pmin[w]);
    pmin[0] = m;
  }
  __syncthreads();
  const double total = part[SNT];
  const double maxw = pow((double)pmin[0] / total * size, -(double)beta);
  for (int i = tid; i < n; i += SNT) {
    const double mass = (double)u[i] * total;
    int a = 0, b = SNT - 1;              // the chunk c with part[c] <= mass < part[c + 1]
    while (a < b) {
      const int m = (a + b + 1) / 2;
      if (part[m] <= mass) a = m; else b = m - 1;
    }
    double acc = part[a];
    int j = min(a * per, size - 1);
    const int end = min(a * per + per, size);
    for (; j < end - 1; ++j) {
      acc += (double)prio[j];
      if (acc > mass) break;
    }
    idx[i] = j;
    weights[i] = (float)(pow((double)prio[j] / total * size, -(double)beta) / maxw);
  }
}

// One CTA.  prio[idx[i]] = (|td[i]| + eps)^alpha where no later position holds the same index; max_prio = max(max_prio,
// max_i |td[i]| + eps).
__global__ void __launch_bounds__(SNT) k_replay_priorities(float* __restrict__ prio, float* __restrict__ max_prio,
                                                           const int64_t* __restrict__ idx, const float* __restrict__ td,
                                                           int n, float alpha, float eps) {
  __shared__ float red[SNT / 32];
  float mx = 0.f;
  for (int i = threadIdx.x; i < n; i += SNT) {
    const int64_t k = idx[i];
    bool last = true;
    for (int j = i + 1; j < n && last; ++j) last = idx[j] != k;
    const float p = fabsf(td[i]) + eps;
    mx = fmaxf(mx, p);
    if (last) prio[k] = powf(p, alpha);
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = max_prio[0];
    for (int w = 0; w < SNT / 32; ++w) m = fmaxf(m, red[w]);
    max_prio[0] = m;
  }
}

// ------------------------------------------------------------------------------------------------
// learner, part 1: per-sample rows
// ------------------------------------------------------------------------------------------------
struct Hyper {
  float gamma, target_noise, noise_clip, inv_n;
};
struct Replay {
  const float *obs, *act, *rew, *new_obs;
  const uint8_t* done;
};
// x [TS][XIN] s|a, x2 [TS][XIN] s'|a' then s|pi(s), h1 h2 g1 g2 g3 [TS][400], small per-row values
constexpr size_t ROWS_SMEM = (size_t)(2 * TS * XIN + 5 * TS * H1 + 8 * TS) * 4;

__global__ void __launch_bounds__(NT) k_ddpg_rows(Layout L, Hyper hp, const float* __restrict__ prm, const float* __restrict__ tgt,
                                                  Replay R, const int64_t* __restrict__ idx, const float* __restrict__ weights,
                                                  const float* __restrict__ noise, int n, Planes P) {
  extern __shared__ __align__(16) float sm[];
  float *x = sm, *x2 = x + TS * XIN, *h1 = x2 + TS * XIN, *h2 = h1 + TS * H1, *g1 = h2 + TS * H1, *g2 = g1 + TS * H1;
  float *g3 = g2 + TS * H1, *qa = g3 + TS * H1, *qb = qa + TS, *y = qb + TS, *dq = y + TS;
  __shared__ int64_t src[TS];
  const int tid = threadIdx.x, D = L.D, K = OBS + D;
  const int q0 = blockIdx.x * TS, nvalid = min(TS, n - q0);
  if (tid < TS) src[tid] = idx[min(q0 + tid, n - 1)];
  __syncthreads();
  for (int i = tid; i < TS * K; i += NT) {
    const int s = i / K, k = i % K;
    const int64_t r = src[s];
    const bool ok = s < nvalid;
    x[s * XIN + k] = !ok ? 0.f : k < OBS ? __ldg(R.obs + r * OBS + k) : __ldg(R.act + r * D + k - OBS);
    x2[s * XIN + k] = !ok || k >= OBS ? 0.f : __ldg(R.new_obs + r * OBS + k);
  }
  __syncthreads();
  for (int i = tid; i < nvalid * K; i += NT) P.x[(size_t)q0 * XIN + (i / K) * XIN + i % K] = x[(i / K) * XIN + i % K];
  // ---- target: a' = clip(pi'(s') + clip(target_noise N, -c, c), -1, 1), y = r + gamma (1 - done) min_k Q'_k(s', a') ----
  actor_fwd(tgt, L, x2, h1, h2, x2 + OBS, XIN);
  if (noise) {
    for (int i = tid; i < TS * D; i += NT) {
      const int s = i / D, d = i % D;
      if (s >= nvalid) continue;
      const float e = fminf(fmaxf(hp.target_noise * noise[(size_t)(q0 + s) * D + d], -hp.noise_clip), hp.noise_clip);
      x2[s * XIN + OBS + d] = fminf(fmaxf(x2[s * XIN + OBS + d] + e, -1.f), 1.f);
    }
    __syncthreads();
  }
  critic_fwd(tgt, L.q1, K, x2, h1, h2, qa);
  if (L.twin) critic_fwd(tgt, L.q2, K, x2, h1, h2, qb);
  if (tid < TS) {
    const int64_t r = src[tid];
    const float qt = L.twin ? fminf(qa[tid], qb[tid]) : qa[tid];
    y[tid] = __ldg(R.rew + r) + hp.gamma * (1.f - (float)R.done[r]) * qt;
  }
  __syncthreads();
  // ---- critics on (s, a): td_k = Q_k - y, dQ_k = w td_k / n; backward rows g2 = dQ w3 [h2 > 0], g1 = g2 W2^T [h1 > 0] ----
  float closs = 0.f;
  for (int c = 0; c < (L.twin ? 2 : 1); ++c) {
    const Net& q = c ? L.q2 : L.q1;
    critic_fwd(prm, q, K, x, h1, h2, qa);
    if (tid < TS) {
      const float td = qa[tid] - y[tid];
      const float w = tid < nvalid ? (weights ? weights[q0 + tid] : 1.f) : 0.f;
      dq[tid] = w * td * hp.inv_n;
      closs += 0.5f * w * td * td;           // thread tid's row
      if (c == 0 && tid < nvalid) P.td[q0 + tid] = td;
    }
    __syncthreads();
    for (int i = tid; i < TS * H2; i += NT) {
      const int s = i / H2, k = i % H2;
      g2[s * H2 + k] = h2[s * H2 + k] > 0.f ? dq[s] * __ldg(prm + q.w3 + k) : 0.f;
    }
    __syncthreads();
    dense_back(prm + q.w2, 0, g2, H2, H1, h1, g1, H1);
    for (int i = tid; i < nvalid * H1; i += NT) {
      const size_t o = (size_t)q0 * H1 + i;
      P.ch1[c][o] = h1[i]; P.cd1[c][o] = g1[i];
    }
    for (int i = tid; i < nvalid * H2; i += NT) {
      const size_t o = (size_t)q0 * H2 + i;
      P.ch2[c][o] = h2[i]; P.cd2[c][o] = g2[i];
    }
    if (tid < nvalid) P.cd3[c][q0 + tid] = dq[tid];
    __syncthreads();
  }
  // ---- actor: a_pi = pi(s); actor loss -mean Q1(s, a_pi) back through critic 1 into a_pi, then through the actor ----
  for (int i = tid; i < TS * OBS; i += NT) x2[(i / OBS) * XIN + i % OBS] = x[(i / OBS) * XIN + i % OBS];
  __syncthreads();
  actor_fwd(prm, L, x2, h1, h2, x2 + OBS, XIN);
  critic_fwd(prm, L.q1, K, x2, g1, g2, qb);
  for (int i = tid; i < TS * H2; i += NT) {
    const int s = i / H2, k = i % H2;
    g2[s * H2 + k] = (s < nvalid && g2[s * H2 + k] > 0.f) ? -hp.inv_n * __ldg(prm + L.q1.w3 + k) : 0.f;
  }
  __syncthreads();
  dense_back(prm + L.q1.w2, 0, g2, H2, H1, g1, g3, H1);               // dZ1 of critic 1 on (s, a_pi)
  float* da = g1;                                                     // [TS][MAXD]: g1 is free now
  dense_back(prm + L.q1.w1, OBS, g3, H1, D, nullptr, da, MAXD);       // dQ/da = dZ1 W1[256 + i, :]^T
  for (int i = tid; i < TS * D; i += NT) {
    const int s = i / D, d = i % D;
    const float a = x2[s * XIN + OBS + d];
    da[s * MAXD + d] *= 1.f - a * a;                                  // tanh'
  }
  __syncthreads();
  // dense_back reads dz with row stride N: compact da to [TS][D] in g3
  for (int i = tid; i < TS * D; i += NT) g3[i] = da[(i / D) * MAXD + i % D];
  __syncthreads();
  dense_back(prm + L.actor.w3, 0, g3, D, H2, h2, g2, H2);
  dense_back(prm + L.actor.w2, 0, g2, H2, H1, h1, g1, H1);
  for (int i = tid; i < nvalid * H1; i += NT) {
    const size_t o = (size_t)q0 * H1 + i;
    P.ah1[o] = h1[i]; P.ad1[o] = g1[i];
  }
  for (int i = tid; i < nvalid * H2; i += NT) {
    const size_t o = (size_t)q0 * H2 + i;
    P.ah2[o] = h2[i]; P.ad2[o] = g2[i];
  }
  for (int i = tid; i < nvalid * D; i += NT) P.ad3[(size_t)q0 * D + i] = g3[i];
  if (tid < nvalid) {
    float* st = P.stats + (size_t)(q0 + tid) * 3;
    st[0] = closs; st[1] = -qb[tid]; st[2] = qb[tid];
  }
}

// The weight-gradient jobs (r4dense::k_dense_wgrad), six per net; the first layers read the [s | a] plane at its row stride
// (the actor only its s columns).
inline r4dense::Jobs make_jobs(const Layout& L, const Planes& P) {
  r4dense::Jobs J;
  int k = 0;
  auto net = [&](const Net& q, const float* X, int ldx, const float* h1, const float* h2, const float* d1, const float* d2,
                 const float* d3) {
    r4dense::layer_jobs(J, k, X, ldx, d1, q.K, H1, q.w1, q.b1);
    r4dense::layer_jobs(J, k, h1, H1, d2, H1, H2, q.w2, q.b2);
    r4dense::layer_jobs(J, k, h2, H2, d3, H2, q.N3, q.w3, q.b3);
  };
  net(L.actor, P.x, XIN, P.ah1, P.ah2, P.ad1, P.ad2, P.ad3);
  net(L.q1, P.x, XIN, P.ch1[0], P.ch2[0], P.cd1[0], P.cd2[0], P.cd3[0]);
  if (L.twin) net(L.q2, P.x, XIN, P.ch1[1], P.ch2[1], P.cd1[1], P.cd2[1], P.cd3[1]);
  r4dense::tile_jobs(J, k);
  return J;
}

// ------------------------------------------------------------------------------------------------
// apply: g = grad * grad_scale + l2 * p on the kernels (w1 w2 w3 of every net, not the biases); torch.optim.Adam per optimiser
// (the actor's with its own step count, skipped when actor_step == 0); then target = tau p + (1 - tau) target.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool is_kernel(const Net& q, int i) {
  return (i >= q.w1 && i < q.b1) || (i >= q.w2 && i < q.b2) || (i >= q.w3 && i < q.b3);
}
__global__ void k_ddpg_apply(Layout L, float* __restrict__ prm, float* __restrict__ tgt, const float* __restrict__ grad,
                             float* __restrict__ m, float* __restrict__ v, int actor_step, int critic_step, float actor_lr,
                             float critic_lr, float l2, float tau, float grad_scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L.n) return;
  const bool actor = i < L.actor.end;
  float p = prm[i];
  if (!actor || actor_step > 0) {
    const bool kern = actor ? is_kernel(L.actor, i) : i < L.q1.end ? is_kernel(L.q1, i) : is_kernel(L.q2, i);
    float g = grad[i] * grad_scale;
    if (kern && l2 != 0.f) g = fmaf(l2, p, g);
    float mi = m[i], vi = v[i];
    r4ppo::adam_update(g, p, mi, vi, actor ? actor_step : critic_step, actor ? actor_lr : critic_lr, 0.9f, 0.999f, 1e-8f);
    prm[i] = p; m[i] = mi; v[i] = vi;
  }
  tgt[i] = __fadd_rn(__fmul_rn(tau, p), __fmul_rn(1.f - tau, tgt[i]));
}

}  // namespace r4ddpg
