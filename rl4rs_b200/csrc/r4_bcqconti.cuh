// r4_bcqconti.cuh -- continuous-action BCQ on the logged dataset: d3rlpy 0.91's BCQ as script/batchrl_trainer.py:61-73 /
// 91-107 configures it for 'BCQ-conti' (INTEGRATION.md section 3, not verified), as fp32 CUDA kernels.  The dense layers run
// through r4dense::k_dense_gemm / k_dense_wgrad (host side in r4_learn.cu, shared with r4_cqlconti.cuh); the kernels here
// build the input rows, the VAE terms, the lambda-mixed max over the sampled actions, the actor head and the argmax of predict.
//
//   encoder  [s | a] [K + D] -> 256 relu -> 256 relu -> [mu | logstd] [2 L], logstd clamped to [-20, 2]
//   decoder  [s | z] [K + L] -> 256 relu -> 256 relu -> tanh [D]
//   actor    [s | a] -> 256 relu -> 256 relu -> f [D];  pi(s, a) = clamp(a + flex tanh(f), -1, 1)
//   critic   k = 0, 1: [s | a] -> 256 relu -> 256 relu -> Q [1];  the target holds the actor and both critics
//   step     imitator, critic, actor (each with the parameters the earlier phases left), soft update of the targets
//            imitator  loss = mean (dec(s, mu + sigma eps) - a)^2 + beta mean KL(N(mu, sigma) || N(0, 1))     (stream 0)
//            critic    a_j = pi'(s', dec(s', clamp(z_j, +-0.5))) for S samples (stream 1); v_j = lam min_k Q'_k + (1 - lam)
//                      max_k Q'_k; y = r + gamma (1 - done) max_j v_j; loss = sum_k mean (Q_k(s, a) - y)^2
//            actor     loss = -mean Q_0(s, pi(s, dec(s, clamp(z, +-0.5))))                              (stream 2)
//   predict  S candidates pi(s, dec(s, clamp(z_j, +-0.5))) (stream 3, keyed by the act call's counter), argmax_j Q_0
//
// Flat parameter layout (each net w1[in,256] b1 w2[256,256] b2 w3[256,out] b3[out]): actor (K+D -> D) | critic 0 (K+D -> 1)
// | critic 1 | encoder (K+D -> 2L) | decoder (K+L -> D).  The target is [actor | critic 0 | critic 1] (the first ntgt floats).
// Noise: r4cqlc::draw with these streams; standard normal.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "r4_cqlconti.cuh"

namespace r4bcqc {

using r4cqlc::H;
using r4cqlc::Net;
using r4cqlc::NT;
constexpr int MAXK = r4cqlc::MAXK, MAXD = r4cqlc::MAXD, MAXN = r4cqlc::MAXN, MAXL = 512, MAXS = 256;
enum { ST_VAE = 0, ST_TARGET, ST_ACTOR, ST_PREDICT };
enum { PK_PLAIN = 0, PK_TANH, PK_LATENT, PK_PERTURB, PK_REPARAM };
constexpr int NSTAT = 5;   // imitator loss, critic loss, actor loss, mean Q_0(s, a), VAE reconstruction mse

struct Layout {
  int K, D, L;
  Net actor, c[2], enc, dec;
  int n, ntgt;
};
__host__ __device__ inline Layout make_layout(int K, int D, int Lat) {
  Layout L;
  L.K = K; L.D = D; L.L = Lat;
  L.actor = r4cqlc::make_net(0, K + D, D);
  L.c[0] = r4cqlc::make_net(L.actor.end, K + D, 1);
  L.c[1] = r4cqlc::make_net(L.c[0].end, K + D, 1);
  L.enc = r4cqlc::make_net(L.c[1].end, K + D, 2 * Lat);
  L.dec = r4cqlc::make_net(L.enc.end, K + Lat, D);
  L.n = L.dec.end; L.ntgt = L.c[1].end;
  return L;
}
inline bool dims_ok(int K, int D, int Lat) {
  return K >= 1 && K <= MAXK && D >= 1 && D <= MAXD && Lat >= 1 && Lat <= MAXL;
}

// Scratch for minibatches of up to n rows and S samples, R = n S.
struct Planes {
  float *xs, *xn, *act, *rew, *term;      // [n][K], [n][K], [n][D], [n], [n]
  float *eps, *zt, *za;                   // [n][L], [R][L], [n][L]
  float* x;                               // [R][K + max(D, L)] the input rows of the current forward
  float *h1, *h2;                         // [R][H] the hidden planes of the current forward
  float *o, *base, *qa, *qb;              // [R][max(D, 2L)] the current net's output, [R][D] base actions, [R], [R]
  float *eh1, *eh2, *dh1, *dh2, *eo, *ex, *dx;   // the VAE: encoder / decoder hidden [n][H], eo [n][2L], their inputs
  float *ah1, *ah2, *ax, *ao, *abase;     // the actor on its loss rows: [n][H] x2, [n][K+D], [n][D], [n][D]
  float *ch1[2], *ch2[2], *cq[2], *cx;    // the critics on the data rows (and the actor rows): [n][H] x2, [n], [n][K+D]
  float *dq[2], *dz2[2], *dz1[2];         // [n], [n][H], [n][H]
  float *dout, *ddz2, *ddz1, *dlat, *deo, *edz2, *edz1;   // decoder / encoder gradients
  float *da, *adz2, *adz1;                // actor gradients
  float* y;                               // [n]
  float* grad;                            // [np]
};
__host__ __device__ inline size_t plane_sizes(const Layout& L, int S, int n, Planes* P, float* base) {
  const size_t K = L.K, D = L.D, La = L.L, N = n, R = (size_t)n * S, W = K + (D > La ? D : La), O = D > 2 * La ? D : 2 * La;
  size_t off = 0;
  auto take = [&](float** dst, size_t k) { if (P) *dst = base + off; off += k; };
  float* dummy;
  float** d = &dummy;
#define T(f, k) take(P ? &P->f : d, (k))
  T(xs, N * K); T(xn, N * K); T(act, N * D); T(rew, N); T(term, N);
  T(eps, N * La); T(zt, R * La); T(za, N * La);
  T(x, R * W); T(h1, R * H); T(h2, R * H); T(o, R * O); T(base, R * D); T(qa, R); T(qb, R);
  T(eh1, N * H); T(eh2, N * H); T(dh1, N * H); T(dh2, N * H); T(eo, N * 2 * La); T(ex, N * (K + D)); T(dx, N * (K + La));
  T(ah1, N * H); T(ah2, N * H); T(ax, N * (K + D)); T(ao, N * D); T(abase, N * D);
  for (int k = 0; k < 2; ++k) { T(ch1[k], N * H); T(ch2[k], N * H); T(cq[k], N); T(dq[k], N); T(dz2[k], N * H); T(dz1[k], N * H); }
  T(cx, N * (K + D));
  T(dout, N * D); T(ddz2, N * H); T(ddz1, N * H); T(dlat, N * La); T(deo, N * 2 * La); T(edz2, N * H); T(edz1, N * H);
  T(da, N * D); T(adz2, N * H); T(adz1, N * H);
  T(y, N);
  T(grad, (size_t)L.n);
#undef T
  return off;
}
inline size_t scratch_floats(const Layout& L, int S, int n) { return plane_sizes(L, S, n, nullptr, nullptr); }
inline Planes make_planes(float* s, const Layout& L, int S, int n) {
  Planes P = {};
  plane_sizes(L, S, n, &P, s);
  return P;
}
// predict: x [n][K], then per candidate row (R = n S): input [R][K + max(D, L)], hidden 2 x [R][H], output, base, q [R];
// plus the critics' rows for the q output
__host__ __device__ inline size_t act_scratch_floats(const Layout& L, int S, int n) {
  const size_t R = (size_t)n * S, W = L.K + (L.D > L.L ? L.D : L.L);
  return (size_t)n * L.K + R * (W + 2 * H + 2 * (size_t)L.D + 1 + L.L) + (size_t)n * (L.K + L.D + 2 * (2 * H + 1));
}

struct Hyper {
  float gamma, tau, lam, beta, flex, eps, rmean, rden;
  float lr_actor, lr_critic, lr_imitator;
  int S;
  uint64_t seed;
};

// Draw the step's latent noise: eps [n][L] (stream 0), zt [n][S][L] (stream 1), za [n][L] (stream 2).
__global__ void __launch_bounds__(NT) k_bcqc_noise(Layout L, Hyper hp, int n, uint64_t counter, Planes P) {
  r4cqlc::pdl_wait();
  const int La = L.L, S = hp.S;
  const int64_t one = (int64_t)n * La, many = (int64_t)n * S * La, total = 2 * one + many;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int st, r, s = 0, j;
    float* dst;
    if (i < one) { st = ST_VAE; r = (int)(i / La); j = (int)(i % La); dst = P.eps + i; }
    else if (i < one + many) {
      const int64_t o = i - one;
      st = ST_TARGET; r = (int)(o / ((int64_t)S * La)); s = (int)((o / La) % S); j = (int)(o % La); dst = P.zt + o;
    } else { const int64_t o = i - one - many; st = ST_ACTOR; r = (int)(o / La); j = (int)(o % La); dst = P.za + o; }
    *dst = r4cqlc::normal(r4cqlc::draw(hp.seed, counter, st, r, s, j));
  }
}

// The gather of the minibatch rows (no noise)
__global__ void __launch_bounds__(NT) k_bcqc_gather(int K, int D, r4cqlc::Data Dt, const int64_t* __restrict__ idx, int n,
                                                    Planes P) {
  r4cqlc::pdl_wait();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x, t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t i = t0; i < (int64_t)n * K; i += stride) {
    const int r = (int)(i / K), k = (int)(i % K);
    const int64_t e = Dt.tidx[idx[r]];
    P.xs[i] = Dt.obs[e * K + k];
    P.xn[i] = Dt.obs[(e + 1) * K + k];
  }
  for (int64_t i = t0; i < (int64_t)n * D; i += stride) P.act[i] = Dt.act[Dt.tidx[idx[i / D]] * D + i % D];
  for (int64_t i = t0; i < n; i += stride) {
    const int64_t e1 = Dt.tidx[idx[i]] + 1;
    P.rew[i] = Dt.rew[e1];
    P.term[i] = (float)Dt.term[e1];
  }
}

// Input rows x[r] = [obs[r / rep] | a_r] (width K + W), one warp per row, a_r by mode from A (row stride lda) and B:
//   PK_PLAIN   A[r]                 PK_TANH     tanh(A[r]) (also stored to out[r])     PK_LATENT  clamp(A[r], -0.5, 0.5)
//   PK_PERTURB clamp(B[r] + flex tanh(A[r]), -1, 1) (also stored to out[r])            PK_REPARAM mu + exp(clamp(ls)) B[r],
//   mu = A[r][0..W), ls = A[r][W..2W)
__global__ void __launch_bounds__(NT) k_bcqc_pack(const float* __restrict__ obs, int K, int rep, const float* __restrict__ A,
                                                  int lda, const float* __restrict__ B, int W, int mode, float flex, int R,
                                                  float* __restrict__ x, float* __restrict__ out) {
  r4cqlc::pdl_wait();
  const int r = blockIdx.x * (NT / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= R) return;
  float* xr = x + (size_t)r * (K + W);
  const float* src = obs + (size_t)(r / rep) * K;
  for (int k = lane; k < K; k += 32) xr[k] = src[k];
  const float* a = A + (size_t)r * lda;
  for (int j = lane; j < W; j += 32) {
    float v;
    if (mode == PK_PLAIN) v = a[j];
    else if (mode == PK_TANH) v = tanhf(a[j]);
    else if (mode == PK_LATENT) v = fminf(fmaxf(a[j], -0.5f), 0.5f);
    else if (mode == PK_PERTURB) v = fminf(fmaxf(fmaf(flex, tanhf(a[j]), B[(size_t)r * W + j]), -1.f), 1.f);
    else v = fmaf(expf(fminf(fmaxf(a[W + j], -20.f), 2.f)), B[(size_t)r * W + j], a[j]);
    xr[K + j] = v;
    if (out && (mode == PK_TANH || mode == PK_PERTURB)) out[(size_t)r * W + j] = v;
  }
}

// One CTA: the VAE loss.  dout [n][D] = 2 (tanh(o) - a) (1 - tanh(o)^2) / (n D) (the decoder output's gradient);
// stats[0] = mse + beta KL, stats[4] = mse.  Sums: per thread in index order, then the threads in order.
__global__ void __launch_bounds__(NT) k_bcqc_vae(Layout L, Hyper hp, int n, Planes P, const float* __restrict__ o,
                                                 float* __restrict__ stats) {
  r4cqlc::pdl_wait();
  __shared__ float part[2][NT];
  const int D = L.D, La = L.L, tid = threadIdx.x;
  const float cm = 2.f / ((float)n * D);
  float se = 0.f, kl = 0.f;
  for (int i = tid; i < n * D; i += NT) {
    const float r = tanhf(o[i]), d = r - P.act[i];
    se = fmaf(d, d, se);
    P.dout[i] = cm * d * (1.f - r * r);
  }
  for (int i = tid; i < n * La; i += NT) {
    const int row = i / La, j = i % La;
    const float mu = P.eo[(size_t)row * 2 * La + j], ls = fminf(fmaxf(P.eo[(size_t)row * 2 * La + La + j], -20.f), 2.f);
    kl += -ls + 0.5f * (expf(2.f * ls) + mu * mu) - 0.5f;
  }
  part[0][tid] = se; part[1][tid] = kl;
  __syncthreads();
  if (tid == 0 && stats) {
    float a = 0.f, b = 0.f;
    for (int t = 0; t < NT; ++t) { a += part[0][t]; b += part[1][t]; }
    const float mse = a / ((float)n * D);
    stats[0] = mse + hp.beta * b / ((float)n * La);
    stats[4] = mse;
  }
}
// The encoder output's gradient deo [n][2L] from the latent's gradient dlat (through the reparameterisation) and the KL.
__global__ void __launch_bounds__(NT) k_bcqc_vae_head(Layout L, Hyper hp, int n, Planes P) {
  r4cqlc::pdl_wait();
  const int La = L.L;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * La) return;
  const int row = (int)(i / La), j = (int)(i % La);
  const float c = hp.beta / ((float)n * La);
  const float mu = P.eo[(size_t)row * 2 * La + j], lsr = P.eo[(size_t)row * 2 * La + La + j];
  const float ls = fminf(fmaxf(lsr, -20.f), 2.f), sd = expf(ls), g = P.dlat[i];
  P.deo[(size_t)row * 2 * La + j] = g + c * mu;
  P.deo[(size_t)row * 2 * La + La + j] = (lsr >= -20.f && lsr <= 2.f) ? fmaf(g, sd * P.eps[i], c * (sd * sd - 1.f)) : 0.f;
}

// One CTA, a thread per row: y = r' + gamma (1 - done) max_j (lam min_k + (1 - lam) max_k) Q'_k(s', a_j) (the first max),
// then dq_k = 2 (Q_k(s, a) - y) / n.  stats[1] = the critic loss, stats[3] = mean Q_0(s, a).
__global__ void __launch_bounds__(NT) k_bcqc_critic(Hyper hp, int n, Planes P, float* __restrict__ stats) {
  r4cqlc::pdl_wait();
  __shared__ float part[2][NT];
  const int S = hp.S, tid = threadIdx.x;
  const float inv_n = 1.f / (float)n;
  float l = 0.f, qs = 0.f;
  for (int i = tid; i < n; i += NT) {
    float best = -INFINITY;
    for (int j = 0; j < S; ++j) {
      const float a = P.qa[(size_t)i * S + j], b = P.qb[(size_t)i * S + j];
      const float v = hp.lam * fminf(a, b) + (1.f - hp.lam) * fmaxf(a, b);
      best = fmaxf(best, v);
    }
    const float y = (P.rew[i] - hp.rmean) / hp.rden + hp.gamma * (1.f - P.term[i]) * best;
    P.y[i] = y;
    for (int k = 0; k < 2; ++k) {
      const float d = P.cq[k][i] - y;
      l = fmaf(d, d, l);
      P.dq[k][i] = 2.f * d * inv_n;
    }
    qs += P.cq[0][i];
  }
  part[0][tid] = l; part[1][tid] = qs;
  __syncthreads();
  if (tid == 0 && stats) {
    float a = 0.f, b = 0.f;
    for (int t = 0; t < NT; ++t) { a += part[0][t]; b += part[1][t]; }
    stats[1] = a * inv_n;
    stats[3] = b * inv_n;
  }
}

// One CTA: the actor loss -mean Q_0(s, pi) -> stats[2]; dq_0 = -1/n on the actor rows.
__global__ void __launch_bounds__(NT) k_bcqc_actor_loss(int n, Planes P, float* __restrict__ stats) {
  r4cqlc::pdl_wait();
  __shared__ float part[NT];
  const int tid = threadIdx.x;
  float s = 0.f;
  for (int i = tid; i < n; i += NT) {
    s += P.cq[0][i];
    P.dq[0][i] = -1.f / (float)n;
  }
  part[tid] = s;
  __syncthreads();
  if (tid == 0 && stats) {
    float a = 0.f;
    for (int t = 0; t < NT; ++t) a += part[t];
    stats[2] = -a / (float)n;
  }
}
// The actor head: d f = da flex (1 - tanh(f)^2) where the clamp passes (|base + flex tanh f| <= 1), else 0 -> dout
__global__ void __launch_bounds__(NT) k_bcqc_actor_head(int D, float flex, int n, Planes P) {
  r4cqlc::pdl_wait();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * D) return;
  const float t = tanhf(P.ao[i]), v = fmaf(flex, t, P.abase[i]);
  P.dout[i] = (v >= -1.f && v <= 1.f) ? P.da[i] * flex * (1.f - t * t) : 0.f;
}

// predict: per row the candidate with the largest Q_0 (the first on ties) -> action [n][D]; one warp per row
__global__ void __launch_bounds__(NT) k_bcqc_argmax(int D, int S, int n, const float* __restrict__ q, const float* __restrict__ cand,
                                                    float* __restrict__ action) {
  const int r = blockIdx.x * (NT / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= n) return;
  int bi = 0;
  float best = q[(size_t)r * S];
  for (int j = 1; j < S; ++j) {
    const float v = q[(size_t)r * S + j];
    if (v > best) { best = v; bi = j; }
  }
  for (int j = lane; j < D; j += 32) action[(size_t)r * D + j] = cand[((size_t)r * S + bi) * D + j];
}
// predict: the step's latent draws [n][S][L] for the act call's counter (stream ST_PREDICT)
__global__ void k_bcqc_predict_noise(int La, int S, int n, uint64_t seed, uint64_t counter, float* __restrict__ z) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * S * La) return;
  const int r = (int)(i / ((int64_t)S * La)), s = (int)((i / La) % S), j = (int)(i % La);
  z[i] = r4cqlc::normal(r4cqlc::draw(seed, counter, ST_PREDICT, r, s, j));
}

}  // namespace r4bcqc
