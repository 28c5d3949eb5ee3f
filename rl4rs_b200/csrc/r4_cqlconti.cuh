// r4_cqlconti.cuh -- continuous-action CQL on the logged dataset: d3rlpy 0.91's CQL as script/batchrl_trainer.py:61-73 /
// 91-107 configures it for 'CQL-conti' (INTEGRATION.md section 3, not verified), as fp32 CUDA kernels.  The dense layers run
// through r4dense::k_dense_gemm (forward: bias + relu epilogue; backward: dZ W^T with the relu-derivative epilogue) and
// r4dense::k_dense_wgrad; the kernels here do the gathers, the noise, the squash / log-prob, the losses and Adam.
//
//   actor   x [K] -> 256 relu -> 256 relu -> [mu | logstd] [2D]  (d3rlpy's two heads as one [256, 2D] layer)
//           logstd clamped to [-20, 2]; u = mu + exp(logstd) eps; a = tanh(u);
//           log pi = sum_j (-eps^2 / 2 - logstd - log(2 pi) / 2 - 2 (log 2 - u - softplus(-2 u)))
//   critic  k = 0, 1: [x | a] [K + D] -> 256 relu -> 256 relu -> Q [1]; the target holds both critics
//   step    temperature, alpha, critic, actor (each with the parameters the earlier phases left), then the soft target update
//           temp   loss = -exp(log_temp) mean(log pi(eps_t) - D)
//           cons_k = w (lse_j[Q_k(s, a_j) - log pi_j ; Q_k(s, u_j) - D log 0.5] - Q_k(s, a)) - threshold, over S policy
//                    samples a_j (eps_ap / eps_cp) and S uniform samples u_j; cons = clamp(exp(log_alpha), 0, 1e6) mean_i sum_k
//           alpha  loss = -cons (policy and uniform samples of stream 1, 2)
//           critic loss = sum_k mean (Q_k(s, a) - y)^2 + cons (streams 3, 4), y = r' + gamma (1 - done) min_k Q'_k(s', tanh mu(s'))
//           actor  loss = mean(exp(log_temp) log pi(eps_pi) - min_k Q_k(s, a(eps_pi)))   (stream 5)
//
// Flat parameter layout: actor w1[K,256] b1 w2[256,256] b2 w3[256,2D] b3[2D] | critic 0 w1[K+D,256] b1 w2 b2 w3[256,1] b3[1]
// | critic 1 (same) | log_temp | log_alpha.  The target is [critic 0 | critic 1].
//
// Noise: draw(seed, counter, stream, row, sample, dim) = splitmix64(splitmix64(seed ^ splitmix64(counter << 3 | stream)) ^
// (row << 24 | sample << 12 | dim)) (sample, dim < 4096); the uniform is hi * 2 / 2^24 - 1 and the normal Box-Muller (in
// double) on (2 hi + 1) / 2^25 and bits 16..39 / 2^24, hi = the top 24 bits.  policy.cqlc_draws restates it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "r4_batchrl.cuh"
#include "r4_dense.cuh"
#include "r4_ppo.cuh"

namespace r4cqlc {

using r4dense::NT;
constexpr int H = 256;
constexpr int MAXK = r4bq::MAXK, MAXD = 512, MAXN = 4096, MAXS = 64;
constexpr int MAXACT = 1 << 20;   // rows of one predict call (the GEMM grid's y extent is rows / 64 <= 65535)
enum { ST_TEMP = 0, ST_APOL, ST_AUNI, ST_CPOL, ST_CUNI, ST_ACT, NSTREAM };
enum { PH_ALPHA = 0, PH_CRITIC, PH_ACTOR };
enum { PK_ALPHA = 0, PK_CRITIC, PK_TARGET, PK_ACTOR };
constexpr int NSTAT = 5;   // critic loss, actor loss, temperature loss, alpha loss, mean Q_0(s, a)

struct Net {
  int w1, b1, w2, b2, w3, b3, end, in, out;
};
__host__ __device__ inline Net make_net(int off, int in, int out) {
  Net m;
  m.in = in; m.out = out;
  m.w1 = off;            m.b1 = m.w1 + in * H;
  m.w2 = m.b1 + H;       m.b2 = m.w2 + H * H;
  m.w3 = m.b2 + H;       m.b3 = m.w3 + H * out;
  m.end = m.b3 + out;
  return m;
}
struct Layout {
  int K, D;
  Net actor, c[2];
  int lt, la, n, t0, ntgt;   // log_temp, log_alpha, total; the target covers params [t0, t0 + ntgt)
};
__host__ __device__ inline Layout make_layout(int K, int D) {
  Layout L;
  L.K = K; L.D = D;
  L.actor = make_net(0, K, 2 * D);
  L.c[0] = make_net(L.actor.end, K + D, 1);
  L.c[1] = make_net(L.c[0].end, K + D, 1);
  L.lt = L.c[1].end; L.la = L.lt + 1; L.n = L.la + 1;
  L.t0 = L.c[0].w1; L.ntgt = L.c[1].end - L.c[0].w1;
  return L;
}
inline bool dims_ok(int K, int D) { return K >= 1 && K <= MAXK && D >= 1 && D <= MAXD; }

// Scratch planes for minibatches of up to n rows with S samples; R = (1 + 2 S) n critic rows (data | policy | uniform).
struct CPlanes {
  float *h1, *h2, *q, *dq, *dz2, *dz1;   // [R][H], [R][H], [R], [R], [R][H], [R][H]
};
struct Planes {
  float *xs, *xn, *act, *rew, *term;     // [n][K], [n][K], [n][D], [n], [n]
  float* noise;                          // streams: [n][D], 4 x [n][S][D], [n][D]
  float *ah1, *ah2, *ao, *nh1, *nh2, *no;   // the actor on s and on s': [n][H], [n][H], [n][2D]
  float* x;                              // [R][K + D] the critic input rows
  float* lp;                             // [n S] the policy samples' log-probs (the actor phase: [n])
  CPlanes c[2];
  float* qt;                             // [2][n] the target critics on s'
  float *da, *dout, *adz2, *adz1;        // [n][D], [n][2D], [n][H], [n][H]
  float* rowv;                           // [n]
  float* grad;                           // [np]
};
__host__ __device__ inline size_t noise_off(int stream, int n, int S, int D) {
  return stream == ST_TEMP ? 0 : stream == ST_ACT ? (size_t)(1 + 4 * S) * n * D : (size_t)n * D + (size_t)(stream - 1) * n * S * D;
}
__host__ __device__ inline size_t scratch_floats(const Layout& L, int S, int n) {
  const size_t K = L.K, D = L.D, N = n, R = (size_t)(1 + 2 * S) * n;
  return N * (2 * K + D + 2) + (size_t)(2 + 4 * S) * N * D + N * (4 * H + 4 * D) + R * (K + D) + (size_t)S * N +
         2 * (4 * R * H + 2 * R) + 2 * N + N * (3 * D + 2 * H) + N + L.n;
}
__host__ __device__ inline Planes make_planes(float* s, const Layout& L, int S, int n) {
  Planes P = {};
  float* p = s;
  auto take = [&](size_t k) { float* q = p; p += k; return q; };
  const size_t K = L.K, D = L.D, N = n, R = (size_t)(1 + 2 * S) * n;
  P.xs = take(N * K); P.xn = take(N * K); P.act = take(N * D); P.rew = take(N); P.term = take(N);
  P.noise = take((size_t)(2 + 4 * S) * N * D);
  P.ah1 = take(N * H); P.ah2 = take(N * H); P.ao = take(N * 2 * D);
  P.nh1 = take(N * H); P.nh2 = take(N * H); P.no = take(N * 2 * D);
  P.x = take(R * (K + D));
  P.lp = take((size_t)S * N);
  for (int k = 0; k < 2; ++k) {
    CPlanes& c = P.c[k];
    c.h1 = take(R * H); c.h2 = take(R * H); c.q = take(R); c.dq = take(R); c.dz2 = take(R * H); c.dz1 = take(R * H);
  }
  P.qt = take(2 * N);
  P.da = take(N * D); P.dout = take(N * 2 * D); P.adz2 = take(N * H); P.adz1 = take(N * H);
  P.rowv = take(N);
  P.grad = take(L.n);
  return P;
}
// predict: the f32 observation, the actor's planes, the critic input and the two critics' planes for n rows
__host__ __device__ inline size_t act_scratch_floats(const Layout& L, int n) {
  return (size_t)n * (L.K + 2 * H + 2 * L.D + (L.K + L.D) + 2 * (2 * H + 1));
}

struct Data {
  const float* obs;          // [N][K]
  const float* act;          // [N][D]
  const float* rew;          // [N]
  const uint8_t* term;       // [N]
  const int64_t* tidx;       // [T]
};
struct Hyper {
  float gamma, tau, eps, threshold, weight, rmean, rden, lrand;   // lrand = D log 0.5 (the uniform samples' log-density)
  float lr_actor, lr_critic, lr_temp, lr_alpha;
  int S;
  uint64_t seed;
};

__host__ __device__ inline uint64_t mix(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__device__ __forceinline__ uint64_t draw(uint64_t seed, uint64_t counter, int stream, int64_t row, int sample, int dim) {
  const uint64_t base = mix(seed ^ mix((counter << 3) | (uint64_t)stream));
  return mix(base ^ (((uint64_t)row << 24) | ((uint64_t)sample << 12) | (uint64_t)dim));
}
__device__ __forceinline__ float uniform(uint64_t x) { return (float)(x >> 40) * (2.f / 16777216.f) - 1.f; }
// Box-Muller in double (u1 = (2 hi + 1) / 2^25 and u2 are exact there), rounded once to float: the float64 restatement
// rounds to the same float except where a draw sits within double roundoff of a float rounding boundary.
__device__ __forceinline__ float normal(uint64_t x) {
  const double u1 = (double)(2 * (x >> 40) + 1) * (1.0 / 33554432.0);
  const double u2 = (double)((x >> 16) & 0xFFFFFFull) * (1.0 / 16777216.0);
  return (float)(sqrt(-2.0 * log(u1)) * cospi(2.0 * u2));
}

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The squashed sample of one element: mu, the raw logstd, eps -> (a, the element's log-prob)
__device__ __forceinline__ float squash(float mu, float ls_raw, float e, float& lp) {
  const float ls = fminf(fmaxf(ls_raw, -20.f), 2.f);
  const float u = fmaf(expf(ls), e, mu);
  const float sp = fmaxf(-2.f * u, 0.f) + log1pf(expf(-fabsf(2.f * u)));   // softplus(-2 u)
  lp = -0.5f * e * e - ls - 0.91893853320467274f - 2.f * (0.69314718055994531f - u - sp);
  return tanhf(u);
}

// The minibatch rows of the transitions idx[0..n) and every noise stream of the step.
__global__ void __launch_bounds__(NT) k_cqlc_gather(Layout L, Hyper hp, Data D, const int64_t* __restrict__ idx, int n,
                                                    uint64_t counter, Planes P) {
  pdl_wait();
  const int K = L.K, A = L.D, S = hp.S;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x, t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t i = t0; i < (int64_t)n * K; i += stride) {
    const int r = (int)(i / K), k = (int)(i % K);
    const int64_t e = D.tidx[idx[r]];
    P.xs[i] = D.obs[e * K + k];
    P.xn[i] = D.obs[(e + 1) * K + k];
  }
  for (int64_t i = t0; i < (int64_t)n * A; i += stride) {
    const int r = (int)(i / A), j = (int)(i % A);
    P.act[i] = D.act[D.tidx[idx[r]] * A + j];
  }
  for (int64_t i = t0; i < n; i += stride) {
    const int64_t e1 = D.tidx[idx[i]] + 1;
    P.rew[i] = D.rew[e1];
    P.term[i] = (float)D.term[e1];
  }
  const int64_t total = (int64_t)(2 + 4 * S) * n * A;
  for (int64_t i = t0; i < total; i += stride) {
    int st, r, s = 0, j;
    const int64_t one = (int64_t)n * A, many = (int64_t)n * S * A;
    if (i < one) { st = ST_TEMP; r = (int)(i / A); j = (int)(i % A); }
    else if (i < one + 4 * many) {
      const int64_t o = i - one;
      st = ST_APOL + (int)(o / many);
      const int64_t w = o % many;
      r = (int)(w / ((int64_t)S * A)); s = (int)((w / A) % S); j = (int)(w % A);
    } else { st = ST_ACT; const int64_t o = i - one - 4 * many; r = (int)(o / A); j = (int)(o % A); }
    const uint64_t x = draw(hp.seed, counter, st, r, s, j);
    P.noise[i] = (st == ST_AUNI || st == ST_CUNI) ? uniform(x) : normal(x);
  }
}

// The critic input rows, one warp per row.  PK_ALPHA / PK_CRITIC: R = (1 + 2 S) n rows [s | a] (data), [s | a_j] (policy
// samples of stream ST_APOL / ST_CPOL, log-probs to lp), [s | u_j] (uniform samples of ST_AUNI / ST_CUNI); PK_TARGET: n rows
// [s' | tanh mu(s')]; PK_ACTOR: n rows [s | a(eps_pi)] with their log-probs.
__global__ void __launch_bounds__(NT) k_cqlc_pack(Layout L, int S, int n, int mode, Planes P) {
  pdl_wait();
  const int K = L.K, A = L.D, KD = K + A, lane = threadIdx.x & 31;
  const int rows = (mode == PK_ALPHA || mode == PK_CRITIC) ? (1 + 2 * S) * n : n;
  const int r = blockIdx.x * (NT / 32) + (threadIdx.x >> 5);
  if (r >= rows) return;
  int i = r, kind = 0, s = 0;             // kind 0: data / target / actor row, 1: policy sample, 2: uniform sample
  if (mode == PK_ALPHA || mode == PK_CRITIC) {
    if (r >= n + n * S) { kind = 2; i = (r - n - n * S) / S; s = (r - n - n * S) % S; }
    else if (r >= n) { kind = 1; i = (r - n) / S; s = (r - n) % S; }
  }
  const float* src = mode == PK_TARGET ? P.xn : P.xs;
  float* x = P.x + (size_t)r * KD;
  for (int k = lane; k < K; k += 32) x[k] = src[(size_t)i * K + k];
  const float* o = (mode == PK_TARGET ? P.no : P.ao) + (size_t)i * 2 * A;
  const int pst = mode == PK_ALPHA ? ST_APOL : ST_CPOL, ust = mode == PK_ALPHA ? ST_AUNI : ST_CUNI;
  float lp = 0.f;
  for (int j = lane; j < A; j += 32) {
    float a, l = 0.f;
    if (mode == PK_TARGET) a = tanhf(o[j]);
    else if (kind == 0 && mode != PK_ACTOR) a = P.act[(size_t)i * A + j];
    else if (kind == 2) a = P.noise[noise_off(ust, n, S, A) + ((size_t)i * S + s) * A + j];
    else {
      const float e = mode == PK_ACTOR ? P.noise[noise_off(ST_ACT, n, S, A) + (size_t)i * A + j]
                                       : P.noise[noise_off(pst, n, S, A) + ((size_t)i * S + s) * A + j];
      a = squash(o[j], o[A + j], e, l);
    }
    lp += l;
    x[K + j] = a;
  }
  lp = warp_sum(lp);
  if (lane == 0) {
    if (mode == PK_ACTOR) P.lp[i] = lp;
    else if (kind == 1) P.lp[(size_t)i * S + s] = lp;
  }
}

// One CTA: the temperature's gradient -exp(log_temp) mean(log pi(eps_t) - D) (rows summed in order), then its Adam when
// apply.  stats[2] = the loss.
__global__ void __launch_bounds__(NT) k_cqlc_temp(Layout L, Hyper hp, int n, Planes P, float* __restrict__ prm,
                                                  float* __restrict__ m, float* __restrict__ v, int step, int apply,
                                                  float* __restrict__ stats) {
  pdl_wait();
  const int A = L.D, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = warp; i < n; i += NT / 32) {
    const float* o = P.ao + (size_t)i * 2 * A;
    float lp = 0.f;
    for (int j = lane; j < A; j += 32) {
      float l;
      squash(o[j], o[A + j], P.noise[(size_t)i * A + j], l);
      lp += l;
    }
    lp = warp_sum(lp);
    if (lane == 0) P.rowv[i] = lp - (float)A;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < n; ++i) s += P.rowv[i];
    const float mean = s / (float)n, et = expf(prm[L.lt]);
    const float g = -et * mean;
    P.grad[L.lt] = g;
    if (stats) stats[2] = -et * mean;
    if (apply) {
      float p = prm[L.lt], mi = m[L.lt], vi = v[L.lt];
      r4ppo::adam_update(g, p, mi, vi, step, hp.lr_temp, 0.9f, 0.999f, hp.eps);
      prm[L.lt] = p; m[L.lt] = mi; v[L.lt] = vi;
    }
  }
}

// The conservative row terms cons_k[i] of both critics over their R rows (max-subtracted logsumexp).
__device__ inline float cons_row(const Hyper& hp, const float* q, const float* lp, int n, int i, float* lse_out) {
  const int S = hp.S;
  float mx = -INFINITY;
  for (int j = 0; j < S; ++j) {
    mx = fmaxf(mx, q[n + i * S + j] - lp[i * S + j]);
    mx = fmaxf(mx, q[n + n * S + i * S + j] - hp.lrand);
  }
  float se = 0.f;
  for (int j = 0; j < S; ++j) {
    se += expf(q[n + i * S + j] - lp[i * S + j] - mx);
    se += expf(q[n + n * S + i * S + j] - hp.lrand - mx);
  }
  const float lse = mx + logf(se);
  *lse_out = lse;
  return hp.weight * (lse - q[i]) - hp.threshold;
}

// One CTA, one thread per row (rows summed in order by thread 0).
//   PH_ALPHA   grad[la] = -exp(log_alpha) [exp(log_alpha) <= 1e6] mean_i sum_k cons_k[i]; Adam on log_alpha when apply.
//   PH_CRITIC  y, the TD and conservative terms; dq_k of every critic row; stats[0] (loss), stats[4] (mean Q_0(s, a)).
//   PH_ACTOR   min_k Q_k on the actor rows, dq_k = -1/n at the smaller critic (the first on ties); stats[1].
__global__ void __launch_bounds__(NT) k_cqlc_loss(Layout L, Hyper hp, int n, int phase, Planes P, float* __restrict__ prm,
                                                  float* __restrict__ m, float* __restrict__ v, int step, int apply,
                                                  float* __restrict__ stats) {
  pdl_wait();
  const int S = hp.S, tid = threadIdx.x;
  const float inv_n = 1.f / (float)n;
  const float ea = expf(prm[L.la]), alpha = fminf(fmaxf(ea, 0.f), 1e6f), temp = expf(prm[L.lt]);
  if (phase == PH_ACTOR) {
    for (int i = tid; i < n; i += NT) {
      const float q0 = P.c[0].q[i], q1 = P.c[1].q[i];
      const int k = q1 < q0 ? 1 : 0;
      P.c[k].dq[i] = -inv_n;
      P.c[1 - k].dq[i] = 0.f;
      P.rowv[i] = temp * P.lp[i] - fminf(q0, q1);
    }
  } else {
    for (int i = tid; i < n; i += NT) {
      float c = 0.f, td = 0.f;
      const float y = phase == PH_CRITIC
          ? (P.rew[i] - hp.rmean) / hp.rden + hp.gamma * (1.f - P.term[i]) * fminf(P.qt[i], P.qt[n + i]) : 0.f;
      for (int k = 0; k < 2; ++k) {
        const float* q = P.c[k].q;
        float lse;
        c += cons_row(hp, q, P.lp, n, i, &lse);
        if (phase == PH_CRITIC) {
          const float d = q[i] - y;
          td += d * d;
          const float cw = alpha * hp.weight * inv_n;
          float* dq = P.c[k].dq;
          dq[i] = 2.f * d * inv_n - cw;
          for (int j = 0; j < S; ++j) {
            dq[n + i * S + j] = cw * expf(q[n + i * S + j] - P.lp[i * S + j] - lse);
            dq[n + n * S + i * S + j] = cw * expf(q[n + n * S + i * S + j] - hp.lrand - lse);
          }
        }
      }
      P.rowv[i] = phase == PH_CRITIC ? td + alpha * c : c;
    }
  }
  __syncthreads();
  if (tid == 0) {
    float s = 0.f, q = 0.f;
    for (int i = 0; i < n; ++i) s += P.rowv[i];
    const float mean = s * inv_n;
    if (phase == PH_ALPHA) {
      const float g = -(ea <= 1e6f ? ea : 0.f) * mean;
      P.grad[L.la] = g;
      if (stats) stats[3] = -alpha * mean;
      if (apply) {
        float p = prm[L.la], mi = m[L.la], vi = v[L.la];
        r4ppo::adam_update(g, p, mi, vi, step, hp.lr_alpha, 0.9f, 0.999f, hp.eps);
        prm[L.la] = p; m[L.la] = mi; v[L.la] = vi;
      }
    } else if (phase == PH_CRITIC) {
      for (int i = 0; i < n; ++i) q += P.c[0].q[i];
      if (stats) { stats[0] = mean; stats[4] = q * inv_n; }
    } else if (stats) {
      stats[1] = mean;
    }
  }
}

// The actor head's gradient dout [n][2D] from da = d(-min Q / n)/da and the entropy term exp(log_temp) log pi / n.
__global__ void __launch_bounds__(NT) k_cqlc_head(Layout L, Hyper hp, int n, Planes P, const float* __restrict__ prm) {
  pdl_wait();
  const int A = L.D;
  const float c = expf(prm[L.lt]) / (float)n;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * A) return;
  const int r = (int)(i / A), j = (int)(i % A);
  const float* o = P.ao + (size_t)r * 2 * A;
  const float e = P.noise[noise_off(ST_ACT, n, hp.S, A) + i];
  const float ls_raw = o[A + j], ls = fminf(fmaxf(ls_raw, -20.f), 2.f), sd = expf(ls);
  const float a = tanhf(fmaf(sd, e, o[j]));
  const float du = P.da[i] * (1.f - a * a) + c * 2.f * a;
  P.dout[(size_t)r * 2 * A + j] = du;
  P.dout[(size_t)r * 2 * A + A + j] = (ls_raw >= -20.f && ls_raw <= 2.f) ? du * sd * e - c : 0.f;
}

// torch.optim.Adam over params [lo, lo + cnt); then, when tgt is given, the soft update tgt = tau p + (1 - tau) tgt of the
// same elements (tgt indexed from lo).
__global__ void k_cqlc_adam(int lo, int cnt, float* __restrict__ prm, const float* __restrict__ grad, float* __restrict__ m,
                            float* __restrict__ v, int step, float lr, float eps, float* __restrict__ tgt, float tau) {
  pdl_wait();
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= cnt) return;
  const int i = lo + k;
  float p = prm[i], mi = m[i], vi = v[i];
  r4ppo::adam_update(grad[i], p, mi, vi, step, lr, 0.9f, 0.999f, eps);
  prm[i] = p; m[i] = mi; v[i] = vi;
  if (tgt) tgt[k] = tau * p + (1.f - tau) * tgt[k];
}

// predict: the f32 copy of the observation (f64 or f32 in) -> x [n][K]
__global__ void k_cqlc_obs(const float* __restrict__ obs32, const double* __restrict__ obs64, int64_t total, float* __restrict__ x) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) x[i] = obs32 ? obs32[i] : (float)obs64[i];
}
// predict: action = tanh mu [n][D] (may be NULL); when xa is given, the critic rows [x | a] with a = act_in (when given)
// or tanh mu
__global__ void k_cqlc_predict(int K, int D, int n, const float* __restrict__ x, const float* __restrict__ o,
                               const float* __restrict__ act_in, float* __restrict__ act_out, float* __restrict__ xa) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int KD = K + D;
  if (i >= (int64_t)n * KD) return;
  const int r = (int)(i / KD), k = (int)(i % KD);
  if (k < K) {
    if (xa) xa[i] = x[(size_t)r * K + k];
    return;
  }
  const int j = k - K;
  const float a = tanhf(o[(size_t)r * 2 * D + j]);
  if (act_out) act_out[(size_t)r * D + j] = a;
  if (xa) xa[i] = act_in ? act_in[(size_t)r * D + j] : a;
}
// predict: q = (Q_0 + Q_1) / 2 (d3rlpy's predict_value: the ensemble mean)
__global__ void k_cqlc_qmean(int n, const float* __restrict__ q0, const float* __restrict__ q1, float* __restrict__ q) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) q[i] = 0.5f * (q0[i] + q1[i]);
}

}  // namespace r4cqlc
