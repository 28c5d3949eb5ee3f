// r4_rainbow.cuh -- RAINBOW on the discrete env: the distributional dueling Q network, the n-step replay store and the
// learner (double Q, categorical projection, prioritized weights), as fp32 CUDA kernels (no tensor cores: parity with
// autograd is the bar, as for r4_ddpg.cuh).
//
//   trunk    obs(256) -> 256 tanh -> 256 tanh                       (RLlib's default FullyConnectedNetwork, no_final_linear)
//   streams  advantage 256 -> 128 relu -> A * atoms ; state score 256 -> 128 relu -> atoms
//   combine  logits[a][k] = score[k] + (adv[a][k] - mean_a adv[a][k]),  p = softmax_k,  Q(s, a) = sum_k z_k p[a][k],
//            z_k = v_min + k dz, dz = (v_max - v_min) / (atoms - 1)
//   act      argmax_a Q, or SoftQ(T = 1): a ~ softmax(Q) by inverse CDF over one counter-based uniform per row
//   learner  a* = argmax Q_online(s', .), p' = p_target(s', a*), m = the projection of r + gamma^n (1 - done) z onto the
//            support, td = -sum_k m_k log p_online(s, a)_k, loss = sum_i w_i td_i * inv_n; hand-derived backward.
//
// Flat parameter layout: w1[256,256] b1[256] w2[256,256] b2[256] | aw1[256,128] ab1[128] aw2[128,A*atoms] ab2[A*atoms] |
//                        sw1[256,128] sb1[128] sw2[128,atoms] sb2[atoms]      (12 tensors; the target has the same layout)
//
// The gradient runs in two launches: k_rainbow_rows (one CTA per TS samples: both nets on s', the projection, the online
// net on s, the loss and the backward rows, written to the scratch planes), then r4ddpg::k_ddpg_wgrad over this net's 12
// jobs (one CTA per 64 x 64 tile of dW = X^T dZ, samples walked in order: deterministic).  k_rainbow_apply clips every
// tensor's gradient to norm <= clip on its own (RLlib's minimize_and_clip), runs Adam and, when flagged, copies the
// parameters into the target.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "r4_ddpg.cuh"

namespace r4rb {

using r4ddpg::NT;
using r4ddpg::TS;
constexpr int OBS = 256, HT = 256, HQ = 128, MAXZ = 32;   // MAXZ: the most atoms
constexpr int MAXAZ = 4096, MAXA = 512;                    // A * atoms and A bounds (shared-memory planes of one tile)
static_assert(TS == NT / 32, "one warp per sample row");

struct Layout {
  int A, Z, AZ;
  int w1, b1, w2, b2, aw1, ab1, aw2, ab2, sw1, sb1, sw2, sb2, n;
};
__host__ __device__ inline Layout make_layout(int A, int Z) {
  Layout L;
  L.A = A; L.Z = Z; L.AZ = A * Z;
  L.w1 = 0;                L.b1 = L.w1 + OBS * HT;
  L.w2 = L.b1 + HT;        L.b2 = L.w2 + HT * HT;
  L.aw1 = L.b2 + HT;       L.ab1 = L.aw1 + HT * HQ;
  L.aw2 = L.ab1 + HQ;      L.ab2 = L.aw2 + HQ * L.AZ;
  L.sw1 = L.ab2 + L.AZ;    L.sb1 = L.sw1 + HT * HQ;
  L.sw2 = L.sb1 + HQ;      L.sb2 = L.sw2 + HQ * Z;
  L.n = L.sb2 + Z;
  return L;
}

// Scratch planes of the learner, n rows each (every layer's input rows X and output-gradient rows dZ).
struct Planes {
  int64_t* idx;                          // [n] sampled indices
  float *x, *h1, *h2, *ha, *hs;          // obs [n][256], trunk [n][256] x 2, stream hiddens [n][128] x 2
  float *d1, *d2, *da1, *da2, *ds1, *ds2;   // dZ of trunk 1, 2 [n][256], advantage [n][128] / [n][A*atoms], score [n][128] / [n][atoms]
  float *td, *stats, *weights;           // td [n], per-sample statistics [n][3], importance weights [n]
  float* grad;                           // [np + 5], then the rank sum [np + 5] (the r4_grad_exchange_n layout)
};
__host__ __device__ inline size_t row_floats(const Layout& L) {
  return 2 + OBS + 4 * HT + 4 * HQ + L.AZ + L.Z + 1 + 3 + 1;
}
__host__ __device__ inline size_t scratch_floats(const Layout& L, int n) {
  return (size_t)n * row_floats(L) + 2 * ((size_t)L.n + 5);
}
__host__ __device__ inline Planes make_planes(float* s, const Layout& L, int n) {
  Planes P;
  float* p = s;
  auto take = [&](size_t k) { float* q = p; p += k; return q; };
  P.idx = reinterpret_cast<int64_t*>(take((size_t)2 * n));      // first: the scratch base is 8-byte aligned
  P.x = take((size_t)n * OBS);
  P.h1 = take((size_t)n * HT); P.h2 = take((size_t)n * HT);
  P.ha = take((size_t)n * HQ); P.hs = take((size_t)n * HQ);
  P.d1 = take((size_t)n * HT); P.d2 = take((size_t)n * HT);
  P.da1 = take((size_t)n * HQ); P.da2 = take((size_t)n * L.AZ);
  P.ds1 = take((size_t)n * HQ); P.ds2 = take((size_t)n * L.Z);
  P.td = take(n); P.stats = take((size_t)n * 3); P.weights = take(n);
  P.grad = take((size_t)L.n + 5);
  return P;
}

// The forward planes of one tile of TS rows in shared memory.
struct Fwd {
  float *h1, *h2, *ha, *hs, *adv, *sc, *mean, *q;   // [TS][256] x 2, [TS][128] x 2, [TS][A*atoms], [TS][MAXZ] x 2, [TS][A]
};
__device__ __forceinline__ float logit(const Fwd& f, const Layout& L, int s, int a, int k) {
  return f.sc[s * MAXZ + k] + (f.adv[(size_t)s * L.AZ + a * L.Z + k] - f.mean[s * MAXZ + k]);
}
__device__ __forceinline__ float atom(float vmin, float dz, int k) { return __fadd_rn(vmin, __fmul_rn((float)k, dz)); }

// The network on the TS rows of x [TS][256] -> every plane of f; with want_q, Q [TS][A] as well.
__device__ inline void forward(const float* __restrict__ prm, const Layout& L, const float* x, const Fwd& f, float vmin,
                               float dz, bool want_q) {
  using r4ddpg::dense;
  dense<2>(prm + L.w1, prm + L.b1, x, OBS, OBS, HT, f.h1, HT);
  dense<2>(prm + L.w2, prm + L.b2, f.h1, HT, HT, HT, f.h2, HT);
  dense<1>(prm + L.aw1, prm + L.ab1, f.h2, HT, HT, HQ, f.ha, HQ);
  dense<1>(prm + L.sw1, prm + L.sb1, f.h2, HT, HT, HQ, f.hs, HQ);
  dense<0>(prm + L.aw2, prm + L.ab2, f.ha, HQ, HQ, L.AZ, f.adv, L.AZ);
  dense<0>(prm + L.sw2, prm + L.sb2, f.hs, HQ, HQ, L.Z, f.sc, MAXZ);
  for (int i = threadIdx.x; i < TS * L.Z; i += NT) {      // the dueling mean, summed over the actions in order
    const int s = i / L.Z, k = i % L.Z;
    float acc = 0.f;
    for (int a = 0; a < L.A; ++a) acc += f.adv[(size_t)s * L.AZ + a * L.Z + k];
    f.mean[s * MAXZ + k] = acc / (float)L.A;
  }
  __syncthreads();
  if (!want_q) return;
  for (int i = threadIdx.x; i < TS * L.A; i += NT) {
    const int s = i / L.A, a = i % L.A;
    float m = -INFINITY;
    for (int k = 0; k < L.Z; ++k) m = fmaxf(m, logit(f, L, s, a, k));
    float se = 0.f, sz = 0.f;
    for (int k = 0; k < L.Z; ++k) {
      const float e = expf(logit(f, L, s, a, k) - m);
      se += e;
      sz = fmaf(atom(vmin, dz, k), e, sz);
    }
    f.q[i] = sz / se;
  }
  __syncthreads();
}

// out[s] = the first index of the largest Q [TS][A] of row s; one warp per row.
__device__ inline void argmax_rows(const float* q, int A, int* out) {
  const int s = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float best = -INFINITY;
  int bi = A;
  for (int a = lane; a < A; a += 32) {
    const float v = q[s * A + a];
    if (v > best) { best = v; bi = a; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) out[s] = bi < A ? bi : 0;
  __syncthreads();
}

__host__ __device__ inline size_t fwd_floats(int A, int AZ) {
  return (size_t)2 * TS * HT + 2 * TS * HQ + (size_t)TS * AZ + 2 * TS * MAXZ + (size_t)TS * A;
}
__device__ inline Fwd carve(float* p, const Layout& L) {
  Fwd f;
  f.h1 = p; f.h2 = f.h1 + TS * HT; f.ha = f.h2 + TS * HT; f.hs = f.ha + TS * HQ;
  f.sc = f.hs + TS * HQ; f.mean = f.sc + TS * MAXZ; f.q = f.mean + TS * MAXZ; f.adv = f.q + TS * L.A;
  return f;
}

// ------------------------------------------------------------------------------------------------
// act: explore 0 -> argmax Q; 1 -> SoftQ, a = the first a with sum_{a' <= a} e^(Q_a' - max) > u * sum_a e^(Q_a - max),
// u = the top 24 bits of r4ddpg::draw(seed, counter, row, 0) / 2^24.  q (may be NULL) receives Q [n][A].
// ------------------------------------------------------------------------------------------------
__host__ __device__ inline size_t act_smem(int A, int AZ) { return ((size_t)TS * OBS + fwd_floats(A, AZ)) * 4; }

__global__ void __launch_bounds__(NT) k_rainbow_act(Layout L, const float* __restrict__ prm, const float* __restrict__ obs, int n,
                                                    float vmin, float dz, int explore, uint64_t seed, uint64_t counter,
                                                    int32_t* __restrict__ action, float* __restrict__ qout) {
  extern __shared__ __align__(16) float sm[];
  __shared__ int pick[TS];
  float* x = sm;
  const Fwd f = carve(x + TS * OBS, L);
  const int tid = threadIdx.x, A = L.A;
  const int s0 = blockIdx.x * TS, nvalid = min(TS, n - s0);
  for (int i = tid; i < TS * OBS; i += NT) {
    const int s = i / OBS;
    x[i] = s < nvalid ? __ldg(obs + (size_t)s0 * OBS + i) : 0.f;
  }
  __syncthreads();
  forward(prm, L, x, f, vmin, dz, true);
  if (qout)
    for (int i = tid; i < nvalid * A; i += NT) qout[(size_t)s0 * A + i] = f.q[i];
  if (!explore) {
    argmax_rows(f.q, A, pick);
  } else if ((tid & 31) == 0) {               // lane 0 of warp s walks row s in action order
    const int s = tid >> 5;
    const float* q = f.q + s * A;
    float m = q[0];
    for (int a = 1; a < A; ++a) m = fmaxf(m, q[a]);
    float se = 0.f;
    for (int a = 0; a < A; ++a) se += expf(q[a] - m);
    const float u = (float)(r4ddpg::draw(seed, counter, s0 + s, 0) >> 40) * (1.0f / 16777216.0f) * se;
    int a = 0;
    float run = 0.f;
    for (; a < A - 1; ++a) {
      run += expf(q[a] - m);
      if (u < run) break;
    }
    pick[s] = a;
  }
  __syncthreads();
  if (tid < nvalid) action[s0 + tid] = pick[tid];
}

// ------------------------------------------------------------------------------------------------
// n-step store (RLlib _adjust_nstep per episode): row r = t * B + b of a [T, B] rollout goes to slot (pos + r) % C with
// reward sum_{j < n, t + j < T} gamma^j rew[t + j] (the original rewards, accumulated in j order), and new_obs / done of
// row t' = min(t + n - 1, T - 1): new_obs = obs of row t' + 1, or final_obs[b] when t' = T - 1.  Only the last C rows are
// written when T * B > C.  New items get priority max_prio^alpha.
// ------------------------------------------------------------------------------------------------
__global__ void k_replay_store_nstep(float* __restrict__ r_obs, int32_t* __restrict__ r_act, float* __restrict__ r_rew,
                                     float* __restrict__ r_new, uint8_t* __restrict__ r_done, float* __restrict__ r_prio,
                                     const float* __restrict__ max_prio, int C, int64_t pos, float alpha, int nstep, float gamma,
                                     const float* __restrict__ obs, const float* __restrict__ final_obs,
                                     const int32_t* __restrict__ act, const float* __restrict__ rew,
                                     const uint8_t* __restrict__ done, int T, int B) {
  const int64_t n = (int64_t)T * B, first = n > C ? n - C : 0;
  const int64_t r = first + blockIdx.x;
  if (r >= n) return;
  const int64_t slot = (pos + r) % C;
  const int t = (int)(r / B), b = (int)(r % B);
  const int t2 = min(t + nstep - 1, T - 1);
  const float* nx = t2 + 1 < T ? obs + ((int64_t)(t2 + 1) * B + b) * OBS : final_obs + (int64_t)b * OBS;
  for (int k = threadIdx.x; k < OBS; k += blockDim.x) {
    r_obs[slot * OBS + k] = obs[r * OBS + k];
    r_new[slot * OBS + k] = nx[k];
  }
  if (threadIdx.x == 0) {
    float R = rew[r], gj = 1.f;
    for (int j = 1; j < nstep && t + j < T; ++j) {
      gj = __fmul_rn(gj, gamma);
      R = __fadd_rn(R, __fmul_rn(gj, rew[(int64_t)(t + j) * B + b]));
    }
    r_rew[slot] = R;
    r_act[slot] = act[r];
    r_done[slot] = done[(int64_t)t2 * B + b];
    if (r_prio) r_prio[slot] = powf(max_prio[0], alpha);
  }
}

// ------------------------------------------------------------------------------------------------
// learner, part 1: per-sample rows
// ------------------------------------------------------------------------------------------------
struct Hyper {
  float vmin, vmax, dz, gamma_n, inv_n;
};
struct Replay {
  const float* obs;
  const int32_t* act;
  const float *rew, *new_obs;
  const uint8_t* done;
};
// x, x2 [TS][256], t1, t2 [TS][256], da1, ds1 [TS][128], pt, mp, ds2 [TS][MAXZ], then the forward planes
__host__ __device__ inline size_t rows_smem(int A, int AZ) {
  return ((size_t)2 * TS * OBS + 2 * TS * HT + 2 * TS * HQ + 3 * TS * MAXZ + fwd_floats(A, AZ)) * 4;
}

__global__ void __launch_bounds__(NT) k_rainbow_rows(Layout L, Hyper hp, const float* __restrict__ prm,
                                                     const float* __restrict__ tgt, Replay R, const int64_t* __restrict__ idx,
                                                     const float* __restrict__ weights, int n, Planes P) {
  extern __shared__ __align__(16) float sm[];
  float *x = sm, *x2 = x + TS * OBS, *t1 = x2 + TS * OBS, *t2 = t1 + TS * HT, *da1 = t2 + TS * HT, *ds1 = da1 + TS * HQ;
  float *pt = ds1 + TS * HQ, *mp = pt + TS * MAXZ, *ds2 = mp + TS * MAXZ;
  const Fwd f = carve(ds2 + TS * MAXZ, L);
  __shared__ int64_t src[TS];
  __shared__ int astar[TS], taken[TS];
  const int tid = threadIdx.x, A = L.A, Z = L.Z;
  const int q0 = blockIdx.x * TS, nvalid = min(TS, n - q0);
  if (tid < TS) src[tid] = idx[min(q0 + tid, n - 1)];
  __syncthreads();
  for (int i = tid; i < TS * OBS; i += NT) {
    const int s = i / OBS, k = i % OBS;
    const bool ok = s < nvalid;
    x[i] = ok ? __ldg(R.obs + src[s] * OBS + k) : 0.f;
    x2[i] = ok ? __ldg(R.new_obs + src[s] * OBS + k) : 0.f;
  }
  __syncthreads();
  // ---- double Q: a* from the online net on s', p' from the target net on s' ----
  forward(prm, L, x2, f, hp.vmin, hp.dz, true);
  argmax_rows(f.q, A, astar);
  forward(tgt, L, x2, f, hp.vmin, hp.dz, false);
  if (tid < TS) {
    const int s = tid, a = astar[s];
    float m = -INFINITY, se = 0.f;
    for (int k = 0; k < Z; ++k) m = fmaxf(m, logit(f, L, s, a, k));
    for (int k = 0; k < Z; ++k) se += expf(logit(f, L, s, a, k) - m);
    for (int k = 0; k < Z; ++k) { pt[s * MAXZ + k] = expf(logit(f, L, s, a, k) - m) / se; mp[s * MAXZ + k] = 0.f; }
    // ---- projection of r + gamma^n (1 - done) z onto the support (RLlib QLoss, the same operation order) ----
    const int64_t r = src[s];
    const float nd = __fmul_rn(hp.gamma_n, 1.f - (float)R.done[r]), rw = R.rew[r];
    for (int j = 0; j < Z; ++j) {
      const float rt = fminf(fmaxf(__fadd_rn(rw, __fmul_rn(nd, atom(hp.vmin, hp.dz, j))), hp.vmin), hp.vmax);
      const float b = __fdiv_rn(__fsub_rn(rt, hp.vmin), hp.dz), lb = floorf(b), ub = ceilf(b);
      const float feq = ub - lb < 0.5f ? 1.f : 0.f;
      const int il = (int)lb, iu = (int)ub;             // an index off the support adds nothing (tf.one_hot)
      const float p = pt[s * MAXZ + j];
      if (il >= 0 && il < Z) mp[s * MAXZ + il] = __fadd_rn(mp[s * MAXZ + il], __fmul_rn(p, __fadd_rn(__fsub_rn(ub, b), feq)));
      if (iu >= 0 && iu < Z) mp[s * MAXZ + iu] = __fadd_rn(mp[s * MAXZ + iu], __fmul_rn(p, __fsub_rn(b, lb)));
    }
  }
  __syncthreads();
  // ---- the online net on s: td = -sum m log p(s, a), dL/dlogit = w inv_n (p sum(m) - m) ----
  forward(prm, L, x, f, hp.vmin, hp.dz, false);
  if (tid < TS) {
    const int s = tid;
    const int a = R.act[src[s]];
    taken[s] = a;
    float m = -INFINITY, se = 0.f;
    for (int k = 0; k < Z; ++k) m = fmaxf(m, logit(f, L, s, a, k));
    for (int k = 0; k < Z; ++k) se += expf(logit(f, L, s, a, k) - m);
    const float lse = m + logf(se);
    float td = 0.f, msum = 0.f, qsel = 0.f;
    for (int k = 0; k < Z; ++k) {
      const float lp = logit(f, L, s, a, k) - lse, mk = mp[s * MAXZ + k];
      td -= mk * lp;
      msum += mk;
      qsel = fmaf(atom(hp.vmin, hp.dz, k), expf(lp), qsel);
    }
    const float w = s < nvalid ? (weights ? weights[q0 + s] : 1.f) : 0.f;
    const float c = w * hp.inv_n;
    for (int k = 0; k < Z; ++k) ds2[s * Z + k] = c * (expf(logit(f, L, s, a, k) - lse) * msum - mp[s * MAXZ + k]);
    if (s < nvalid) {
      P.td[q0 + s] = td;
      float* st = P.stats + (size_t)(q0 + s) * 3;
      st[0] = w * td; st[1] = td; st[2] = qsel;
    }
  }
  __syncthreads();
  // ---- backward: the dueling mean spreads -g / A over every action; the taken action gets g on top ----
  float* da2 = f.adv;                                      // the advantage outputs are not read again
  for (int i = tid; i < TS * L.AZ; i += NT) {
    const int s = i / L.AZ, c = i % L.AZ, a = c / Z, k = c % Z;
    const float g = ds2[s * Z + k], gm = g / (float)A;
    da2[i] = a == taken[s] ? g - gm : -gm;
  }
  __syncthreads();
  r4ddpg::dense_back(prm + L.aw2, 0, da2, L.AZ, HQ, f.ha, da1, HQ);
  r4ddpg::dense_back(prm + L.sw2, 0, ds2, Z, HQ, f.hs, ds1, HQ);
  r4ddpg::dense_back(prm + L.aw1, 0, da1, HQ, HT, nullptr, t1, HT);
  r4ddpg::dense_back(prm + L.sw1, 0, ds1, HQ, HT, nullptr, t2, HT);
  for (int i = tid; i < TS * HT; i += NT) t1[i] = (t1[i] + t2[i]) * (1.f - f.h2[i] * f.h2[i]);    // tanh'
  __syncthreads();
  r4ddpg::dense_back(prm + L.w2, 0, t1, HT, HT, nullptr, t2, HT);
  for (int i = tid; i < TS * HT; i += NT) t2[i] *= 1.f - f.h1[i] * f.h1[i];
  __syncthreads();
  for (int i = tid; i < nvalid * OBS; i += NT) P.x[(size_t)q0 * OBS + i] = x[i];
  for (int i = tid; i < nvalid * HT; i += NT) {
    const size_t o = (size_t)q0 * HT + i;
    P.h1[o] = f.h1[i]; P.h2[o] = f.h2[i]; P.d1[o] = t2[i]; P.d2[o] = t1[i];
  }
  for (int i = tid; i < nvalid * HQ; i += NT) {
    const size_t o = (size_t)q0 * HQ + i;
    P.ha[o] = f.ha[i]; P.hs[o] = f.hs[i]; P.da1[o] = da1[i]; P.ds1[o] = ds1[i];
  }
  for (int i = tid; i < nvalid * L.AZ; i += NT) P.da2[(size_t)q0 * L.AZ + i] = da2[i];
  for (int i = tid; i < nvalid * Z; i += NT) P.ds2[(size_t)q0 * Z + i] = ds2[i];
}

// ------------------------------------------------------------------------------------------------
// learner, part 2: the weight gradients of the 12 tensors, as jobs of r4ddpg::k_ddpg_wgrad
// ------------------------------------------------------------------------------------------------
inline r4ddpg::Jobs make_jobs(const Layout& L, const Planes& P) {
  r4ddpg::Jobs J;
  int k = 0;
  auto layer = [&](const float* X, const float* dZ, int M, int N, int w, int b) {
    J.j[k++] = {X, dZ, M, M, N, w, 0};
    J.j[k++] = {nullptr, dZ, 1, 1, N, b, 0};
  };
  layer(P.x, P.d1, OBS, HT, L.w1, L.b1);
  layer(P.h1, P.d2, HT, HT, L.w2, L.b2);
  layer(P.h2, P.da1, HT, HQ, L.aw1, L.ab1);
  layer(P.ha, P.da2, HQ, L.AZ, L.aw2, L.ab2);
  layer(P.h2, P.ds1, HT, HQ, L.sw1, L.sb1);
  layer(P.hs, P.ds2, HQ, L.Z, L.sw2, L.sb2);
  J.njob = k;
  int t = 0;
  for (int i = 0; i < k; ++i) {
    J.j[i].tile0 = t;
    t += ((J.j[i].M + r4ddpg::WT - 1) / r4ddpg::WT) * ((J.j[i].N + r4ddpg::WT - 1) / r4ddpg::WT);
  }
  J.ntiles = t;
  return J;
}

// ------------------------------------------------------------------------------------------------
// apply: per tensor, g *= clip / ||g|| when ||g|| > clip (clip <= 0: off; the norm summed in a fixed order, the same in
// every CTA of the tensor), then torch.optim.Adam (betas 0.9 / 0.999), then target = params when copy_target.
// One CTA per chunk of ACH elements of one tensor.
// ------------------------------------------------------------------------------------------------
constexpr int NTEN = 12, ACH = 16384, ANT = 256;
struct Split {
  int start[NTEN + 1], cta0[NTEN + 1];
};
inline Split make_split(const Layout& L) {
  const int st[NTEN + 1] = {L.w1, L.b1, L.w2, L.b2, L.aw1, L.ab1, L.aw2, L.ab2, L.sw1, L.sb1, L.sw2, L.sb2, L.n};
  Split S;
  S.cta0[0] = 0;
  for (int k = 0; k <= NTEN; ++k) S.start[k] = st[k];
  for (int k = 0; k < NTEN; ++k) S.cta0[k + 1] = S.cta0[k] + (st[k + 1] - st[k] + ACH - 1) / ACH;
  return S;
}

__global__ void __launch_bounds__(ANT) k_rainbow_apply(Split S, float* __restrict__ prm, float* __restrict__ tgt,
                                                       const float* __restrict__ grad, float* __restrict__ m,
                                                       float* __restrict__ v, int step, float lr, float eps, float clip,
                                                       int copy_target) {
  __shared__ float red[ANT];
  const int tid = threadIdx.x;
  int k = 0;
  while (k + 1 < NTEN && (int)blockIdx.x >= S.cta0[k + 1]) ++k;
  const int lo = S.start[k], hi = S.start[k + 1];
  float ss = 0.f;
  for (int i = lo + tid; i < hi; i += ANT) ss = fmaf(grad[i], grad[i], ss);
  red[tid] = ss;
  __syncthreads();
  for (int o = ANT / 2; o > 0; o >>= 1) {
    if (tid < o) red[tid] += red[tid + o];
    __syncthreads();
  }
  const float norm = sqrtf(red[0]);
  const bool scale = clip > 0.f && norm > clip;
  const float f = scale ? clip / norm : 1.f;
  const int c0 = lo + ((int)blockIdx.x - S.cta0[k]) * ACH, c1 = min(c0 + ACH, hi);
  for (int i = c0 + tid; i < c1; i += ANT) {
    float g = grad[i];
    if (scale) g *= f;
    float p = prm[i], mi = m[i], vi = v[i];
    r4ppo::adam_update(g, p, mi, vi, step, lr, 0.9f, 0.999f, eps);
    prm[i] = p; m[i] = mi; v[i] = vi;
    if (copy_target) tgt[i] = p;
  }
}

}  // namespace r4rb
