// r4_batchrl.cuh -- batch (offline) RL on the logged dataset: the discrete BC, BCQ and CQL learners of d3rlpy 0.91 as the
// reference configures them (script/batchrl_trainer.py:34-90), as fp32 CUDA kernels (no tensor cores: parity with autograd
// is the bar, as for r4_ddpg.cuh / r4_rainbow.cuh).
//
//   masked net M (BC imitator; BCQ Q function and imitator, each its own): the reference's custom encoder with_q
//            h = relu(x W1 + b1) [256] ; e = flatten(Emb[x[:, K-10:K]]) [10 x 32] ; f = ([h | e] W2 + b2) * keep [A] ;
//            then d3rlpy's head z = f W3 + b3 [A]   (x = the d3rl observation [K]: simulator obs | 9 prev actions | step)
//   keep     location_mask[step % 9 / 3][a], 0 for the 9 prev actions, 0 for every special item when a prev action is one
//   plain net C (CQL, d3rlpy's default encoder): relu(x W1 + b1) -> relu(. W2 + b2) [256] -> z = . W3 + b3 [A]
//   BC       loss = nll(log_softmax(z), a) + beta mean(z^2)
//   BCQ      a* = argmax((Q(s') - min Q(s')) [log pi(s') - max log pi(s') > log flex]), y = r + gamma (1 - done) Q_targ(s', a*),
//            loss = huber(Q(s, a) - y) + the imitator's BC loss (its own beta)
//   CQL      a* = argmax Q(s'), y = r' + gamma (1 - done) Q_targ(s', a*) with r' = (r - mean) / den,
//            loss = huber(Q(s, a) - y) + alpha (logsumexp Q(s, .) - Q(s, a))
//   every loss is the minibatch mean; huber is d3rlpy's (delta 1).
//
// Flat parameter layout: M = w1[K,256] b1[256] emb[A,32] w2[576,A] b2[A] w3[A,A] b3[A];  C = w1[K,256] b1 w2[256,256] b2 w3[256,A] b3.
//   BC: M (imitator) ; BCQ: M (Q) | M (imitator) ; CQL: C.   The target holds the Q part only (BCQ: the first M; CQL: C).
//
// One SGD step is four launches: k_bq_rows (one CTA per TS samples: the forwards on s' and s, the loss rows and the
// backward rows, written to the scratch planes), r4dense::k_dense_wgrad over the dense layers (dW = X^T dZ, one CTA per
// 64 x 64 tile, samples walked in order), k_bq_embgrad (the embedding scatter, one thread per table element walking the
// samples and slots in order: deterministic, no atomics) and k_bq_apply (Adam, then the hard target copy when due).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "r4_ddpg.cuh"

namespace r4bq {

using r4ddpg::NT;
using r4ddpg::TS;
constexpr int H = 256, E = 32, W = 10, PW = 9, HE = H + W * E;   // W: the mask columns (9 prev actions + step)
constexpr int MAXA = 512, MAXK = 4096;
enum { BC = 0, BCQ = 1, CQL = 2 };
static_assert(TS == NT / 32, "one warp per sample row");

struct MNet {
  int w1, b1, emb, w2, b2, w3, b3, end;
};
__host__ __device__ inline MNet make_mnet(int off, int K, int A) {
  MNet m;
  m.w1 = off;              m.b1 = m.w1 + K * H;
  m.emb = m.b1 + H;        m.w2 = m.emb + A * E;
  m.b2 = m.w2 + HE * A;    m.w3 = m.b2 + A;
  m.b3 = m.w3 + A * A;     m.end = m.b3 + A;
  return m;
}
struct CNet {
  int w1, b1, w2, b2, w3, b3, end;
};
__host__ __device__ inline CNet make_cnet(int off, int K, int A) {
  CNet c;
  c.w1 = off;              c.b1 = c.w1 + K * H;
  c.w2 = c.b1 + H;         c.b2 = c.w2 + H * H;
  c.w3 = c.b2 + H;         c.b3 = c.w3 + H * A;
  c.end = c.b3 + A;
  return c;
}
struct Layout {
  int algo, K, A;
  MNet q, imi;          // BC: imi only; BCQ: both
  CNet c;               // CQL
  int n, ntgt;
};
__host__ __device__ inline Layout make_layout(int algo, int K, int A) {
  Layout L;
  L.algo = algo; L.K = K; L.A = A;
  L.q = make_mnet(0, K, A);
  L.imi = make_mnet(algo == BCQ ? L.q.end : 0, K, A);
  L.c = make_cnet(0, K, A);
  L.n = algo == BC ? L.imi.end : algo == BCQ ? L.imi.end : L.c.end;
  L.ntgt = algo == BC ? 0 : algo == BCQ ? L.q.end : L.c.end;
  return L;
}

// Scratch planes, n rows each.  mp[k]: the k-th masked net's he [n][HE], f [n][A], d1 [n][H], de [n][W*E], d2 [n][A],
// d3 [n][A]; CQL's h1, h2, c1, c2 [n][H], c3 [n][A] (dZ of the three layers).
struct MPlanes {
  float *he, *f, *d1, *de, *d2, *d3;
};
struct Planes {
  int32_t* ids;         // [n][W] the embedding ids
  float* x;             // [n][K]
  MPlanes mp[2];
  float *h1, *h2, *c1, *c2, *c3;
  float* stats;         // [n][3]
  float* grad;          // [np]
};
__host__ __device__ inline int n_mnets(int algo) { return algo == BCQ ? 2 : algo == BC ? 1 : 0; }
__host__ __device__ inline size_t scratch_floats(const Layout& L, int n) {
  const size_t m = (size_t)HE + 3 * L.A + H + W * E + 0;
  size_t r = W + L.K + 3 + (size_t)n_mnets(L.algo) * m + (L.algo == CQL ? 4 * H + L.A : 0);
  return (size_t)n * r + L.n + 4;
}
__host__ __device__ inline Planes make_planes(float* s, const Layout& L, int n) {
  Planes P = {};
  float* p = s;
  auto take = [&](size_t k) { float* q = p; p += k; return q; };
  P.ids = reinterpret_cast<int32_t*>(take((size_t)n * W));
  P.x = take((size_t)n * L.K);
  for (int k = 0; k < n_mnets(L.algo); ++k) {
    MPlanes& M = P.mp[k];
    M.he = take((size_t)n * HE); M.f = take((size_t)n * L.A);
    M.d1 = take((size_t)n * H); M.de = take((size_t)n * W * E);
    M.d2 = take((size_t)n * L.A); M.d3 = take((size_t)n * L.A);
  }
  if (L.algo == CQL) {
    P.h1 = take((size_t)n * H); P.h2 = take((size_t)n * H);
    P.c1 = take((size_t)n * H); P.c2 = take((size_t)n * H); P.c3 = take((size_t)n * L.A);
  }
  P.stats = take((size_t)n * 3);
  P.grad = take(L.n);
  return P;
}

// The dataset on the device and the masking tables.  locm [3][A] (1 = the layer allows the item), special [A] (1 = special).
struct Data {
  const float* obs;          // [N][K]
  const int32_t* act;        // [N]
  const float* rew;          // [N]
  const uint8_t* term;       // [N]
  const int64_t* tidx;       // [T] entry index of every transition (the entry t of (s_t, a_t, r_t+1, s_t+1, done_t+1))
  const uint8_t* locm;
  const uint8_t* special;
};
struct Hyper {
  float gamma, inv_n, beta, alpha, log_flex, rmean, rden;
};

__device__ __forceinline__ float warp_max(float v) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// the first index of the largest v[0..A) (every lane gets it)
__device__ __forceinline__ int warp_argmax(const float* v, int A) {
  const int lane = threadIdx.x & 31;
  float best = -INFINITY;
  int bi = A;
  for (int a = lane; a < A; a += 32)
    if (v[a] > best) { best = v[a]; bi = a; }
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  return bi < A ? bi : 0;
}
// log sum exp of v[0..A) (every lane gets it)
__device__ __forceinline__ float warp_lse(const float* v, int A) {
  const int lane = threadIdx.x & 31;
  float m = -INFINITY;
  for (int a = lane; a < A; a += 32) m = fmaxf(m, v[a]);
  m = warp_max(m);
  float se = 0.f;
  for (int a = lane; a < A; a += 32) se += expf(v[a] - m);
  return m + logf(r4ppo::warp_sum(se));
}

// The TS observation rows of row[s] (s < nvalid; zero rows after) -> x [TS][K], the embedding ids [TS][W] and keep [TS][A].
__device__ inline void load_rows(const Layout& L, const float* __restrict__ obs32, const double* __restrict__ obs64,
                                 const int64_t* row, int nvalid, const Data& D, float* x, int* ids, float* keep, int* hs) {
  const int tid = threadIdx.x, K = L.K, A = L.A;
  for (int i = tid; i < TS * K; i += NT) {
    const int s = i / K, k = i % K;
    x[i] = s >= nvalid ? 0.f : obs32 ? __ldg(obs32 + row[s] * K + k) : (float)__ldg(obs64 + row[s] * K + k);
  }
  __syncthreads();
  if (tid < TS * W) {
    const int s = tid / W, j = tid % W;
    ids[tid] = min(max((int)x[s * K + K - W + j], 0), A - 1);
  }
  __syncthreads();
  if (tid < TS) {
    int h = 0;
    for (int j = 0; j < PW; ++j) h |= D.special[ids[tid * W + j]];
    hs[tid] = h;
  }
  __syncthreads();
  for (int i = tid; i < TS * A; i += NT) {
    const int s = i / A, a = i % A;
    const int layer = (max((int)x[s * K + K - 1], 0) % PW) / 3;
    bool k = D.locm[layer * A + a] != 0;
    for (int j = 0; j < PW; ++j) k = k && ids[s * W + j] != a;
    if (hs[s] && D.special[a]) k = false;
    keep[i] = k ? 1.f : 0.f;
  }
  __syncthreads();
}

// The masked net M on x -> he [TS][HE] (h | e), f [TS][A] (masked features), z [TS][A].
__device__ inline void m_forward(const float* __restrict__ prm, const MNet& m, const Layout& L, const float* x, const int* ids,
                                 const float* keep, float* he, float* f, float* z) {
  const int K = L.K, A = L.A;
  r4ddpg::dense<1>(prm + m.w1, prm + m.b1, x, K, K, H, he, HE);
  for (int i = threadIdx.x; i < TS * W * E; i += NT) {
    const int s = i / (W * E), r = i % (W * E), j = r / E, c = r % E;
    he[s * HE + H + r] = __ldg(prm + m.emb + (size_t)ids[s * W + j] * E + c);
  }
  __syncthreads();
  r4ddpg::dense<0>(prm + m.w2, prm + m.b2, he, HE, HE, A, f, A);
  for (int i = threadIdx.x; i < TS * A; i += NT) f[i] = keep[i] != 0.f ? f[i] : 0.f;
  __syncthreads();
  r4ddpg::dense<0>(prm + m.w3, prm + m.b3, f, A, A, A, z, A);
}
// dz [TS][A] -> d2 [TS][A] (the fc2 output gradient, masked) and dhe [TS][HE] (d1 = dh [h > 0] | de).
__device__ inline void m_backward(const float* __restrict__ prm, const MNet& m, const Layout& L, const float* he, const float* keep,
                                  const float* dz, float* d2, float* dhe) {
  const int A = L.A;
  r4ddpg::dense_back(prm + m.w3, 0, dz, A, A, nullptr, d2, A);
  for (int i = threadIdx.x; i < TS * A; i += NT) d2[i] = keep[i] != 0.f ? d2[i] : 0.f;
  __syncthreads();
  r4ddpg::dense_back(prm + m.w2, 0, d2, A, H, he, dhe, HE);
  r4ddpg::dense_back(prm + m.w2, H, d2, A, W * E, nullptr, dhe + H, HE);
}
__device__ inline void c_forward(const float* __restrict__ prm, const CNet& c, const Layout& L, const float* x, float* h1, float* h2,
                                 float* z) {
  r4ddpg::dense<1>(prm + c.w1, prm + c.b1, x, L.K, L.K, H, h1, H);
  r4ddpg::dense<1>(prm + c.w2, prm + c.b2, h1, H, H, H, h2, H);
  r4ddpg::dense<0>(prm + c.w3, prm + c.b3, h2, H, H, L.A, z, L.A);
}

// x [TS][K], he and dhe [TS][HE], six [TS][max(A, H)] planes (f z dz d2 aux keep; CQL keeps [TS][H] rows in them), ids
__host__ __device__ inline int plane(int A) { return A > H ? A : H; }
__host__ __device__ inline size_t rows_smem(int K, int A) {
  return ((size_t)TS * K + 2 * TS * HE + 6 * (size_t)TS * plane(A) + TS * W) * 4;
}

// The BC loss row of warp s over logits z [A]: dz = c ((softmax - onehot(a)) + beta 2 z / A); returns (nll, mean z^2).
__device__ inline void bc_row(const float* z, float* dz, int A, int a, float beta, float c, float& nll, float& pen) {
  const int lane = threadIdx.x & 31;
  const float lse = warp_lse(z, A);
  float zz = 0.f;
  for (int j = lane; j < A; j += 32) {
    zz = fmaf(z[j], z[j], zz);
    dz[j] = c * ((expf(z[j] - lse) - (j == a ? 1.f : 0.f)) + beta * 2.f * z[j] / (float)A);
  }
  nll = lse - z[a];
  pen = r4ppo::warp_sum(zz) / (float)A;
}
__device__ __forceinline__ float huber(float td) { return fabsf(td) < 1.f ? 0.5f * td * td : fabsf(td) - 0.5f; }
__device__ __forceinline__ float huber_grad(float td) { return fabsf(td) < 1.f ? td : copysignf(1.f, td); }

template <int ALGO>
__global__ void __launch_bounds__(NT) k_bq_rows(Layout L, Hyper hp, const float* __restrict__ prm, const float* __restrict__ tgt,
                                                Data D, const int64_t* __restrict__ idx, int n, Planes P) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  extern __shared__ __align__(16) float sm[];
  const int K = L.K, A = L.A, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int AB = TS * plane(A);
  float *x = sm, *he = x + TS * K, *dhe = he + TS * HE, *f = dhe + TS * HE, *z = f + AB, *dz = z + AB;
  float *d2 = dz + AB, *aux = d2 + AB, *keep = aux + AB;
  int* ids = reinterpret_cast<int*>(keep + AB);
  __shared__ int64_t ent[TS], nxt[TS];
  __shared__ int hs[TS], taken[TS];
  __shared__ float y[TS];
  const int q0 = blockIdx.x * TS, nvalid = min(TS, n - q0);
  if (tid < TS) {
    const int64_t e = D.tidx[idx[min(q0 + tid, n - 1)]];
    ent[tid] = e; nxt[tid] = e + 1;
    taken[tid] = min(max(D.act[e], 0), A - 1);
  }
  __syncthreads();
  // ---- the target y on s' (BCQ, CQL) ----
  if (ALGO != BC) {
    load_rows(L, D.obs, nullptr, nxt, nvalid, D, x, ids, keep, hs);
    if (ALGO == BCQ) {
      m_forward(prm, L.q, L, x, ids, keep, he, f, aux);             // Q(s')
      m_forward(prm, L.imi, L, x, ids, keep, he, f, z);             // imitator logits on s'
      {
        const float* q = aux + warp * A;
        const float* lg = z + warp * A;
        const float lse = warp_lse(lg, A);
        float lpm = -INFINITY, qm = INFINITY;
        for (int a = lane; a < A; a += 32) { lpm = fmaxf(lpm, lg[a] - lse); qm = fminf(qm, q[a]); }
        lpm = warp_max(lpm); qm = warp_min(qm);
        float* fl = dz + warp * A;
        for (int a = lane; a < A; a += 32) fl[a] = (q[a] - qm) * (((lg[a] - lse) - lpm) > hp.log_flex ? 1.f : 0.f);
        __syncwarp();
        const int as = warp_argmax(fl, A);
        if (lane == 0) hs[warp] = as;
      }
      __syncthreads();
      m_forward(tgt, L.q, L, x, ids, keep, he, f, z);               // Q_targ(s')
    } else {
      c_forward(prm, L.c, L, x, he, dhe, z);
      {
        const int as = warp_argmax(z + warp * A, A);
        if (lane == 0) hs[warp] = as;
      }
      __syncthreads();
      c_forward(tgt, L.c, L, x, he, dhe, z);
    }
    if (tid < TS) {
      const int64_t e1 = nxt[tid];
      const float r = (D.rew[e1] - hp.rmean) / hp.rden;
      y[tid] = r + hp.gamma * (1.f - (float)D.term[e1]) * z[tid * A + hs[tid]];
    }
    __syncthreads();
  }
  // ---- s: the forwards, the loss rows and the backward ----
  load_rows(L, D.obs, nullptr, ent, nvalid, D, x, ids, keep, hs);
  for (int i = tid; i < nvalid * K; i += NT) P.x[(size_t)q0 * K + i] = x[i];
  for (int i = tid; i < nvalid * W; i += NT) P.ids[(size_t)q0 * W + i] = ids[i];
  const bool valid = warp < nvalid;
  const float c = valid ? hp.inv_n : 0.f;
  float st0 = 0.f, st1 = 0.f, st2 = 0.f;
  for (int net = 0; net < (ALGO == BCQ ? 2 : 1); ++net) {
    const int a = taken[warp];
    if (ALGO == CQL) {
      c_forward(prm, L.c, L, x, he, dhe, z);
      const float* q = z + warp * A;
      const float lse = warp_lse(q, A);
      const float td = q[a] - y[warp], g = huber_grad(td);
      for (int j = lane; j < A; j += 32)
        dz[warp * A + j] = c * ((j == a ? g : 0.f) + hp.alpha * (expf(q[j] - lse) - (j == a ? 1.f : 0.f)));
      st1 = huber(td); st0 = st1 + hp.alpha * (lse - q[a]); st2 = q[a];
    } else {
      const bool imi = ALGO == BC || net == 1;
      const MNet& m = imi ? L.imi : L.q;
      m_forward(prm, m, L, x, ids, keep, he, f, z);
      if (imi) {
        float nll, pen;
        bc_row(z + warp * A, dz + warp * A, A, a, hp.beta, c, nll, pen);
        const float lb = nll + hp.beta * pen;
        if (ALGO == BC) { st0 = lb; st1 = nll; st2 = pen; } else { st0 += lb; }
      } else {
        const float* q = z + warp * A;
        const float td = q[a] - y[warp], g = huber_grad(td);
        for (int j = lane; j < A; j += 32) dz[warp * A + j] = j == a ? c * g : 0.f;
        st0 = st1 = huber(td); st2 = q[a];
      }
    }
    __syncthreads();
    if (ALGO == CQL) {
      r4ddpg::dense_back(prm + L.c.w3, 0, dz, A, H, dhe, d2, H);       // dZ2 = dz W3^T [h2 > 0]   (d2: [TS][H])
      r4ddpg::dense_back(prm + L.c.w2, 0, d2, H, H, he, aux, H);        // dZ1 = dZ2 W2^T [h1 > 0]
      for (int i = tid; i < nvalid * H; i += NT) {
        const size_t o = (size_t)q0 * H + i;
        P.h1[o] = he[i]; P.h2[o] = dhe[i]; P.c1[o] = aux[i]; P.c2[o] = d2[i];
      }
      for (int i = tid; i < nvalid * A; i += NT) P.c3[(size_t)q0 * A + i] = dz[i];
    } else {
      const MNet& m = (ALGO == BC || net == 1) ? L.imi : L.q;
      m_backward(prm, m, L, he, keep, dz, d2, dhe);
      const MPlanes& M = P.mp[net];
      for (int i = tid; i < nvalid * HE; i += NT) {
        const int s = i / HE, k = i % HE;
        M.he[(size_t)q0 * HE + i] = he[i];
        if (k < H) M.d1[(size_t)(q0 + s) * H + k] = dhe[i];
        else M.de[(size_t)(q0 + s) * (W * E) + k - H] = dhe[i];
      }
      for (int i = tid; i < nvalid * A; i += NT) {
        const size_t o = (size_t)q0 * A + i;
        M.f[o] = f[i]; M.d2[o] = d2[i]; M.d3[o] = dz[i];
      }
    }
    __syncthreads();
  }
  if (lane == 0 && valid) {
    float* st = P.stats + (size_t)(q0 + warp) * 3;
    st[0] = st0; st[1] = st1; st[2] = st2;
  }
}

inline r4dense::Jobs make_jobs(const Layout& L, const Planes& P) {
  r4dense::Jobs J;
  int k = 0;
  auto layer = [&](const float* X, int ldx, const float* dZ, int M, int N, int w, int b) {
    J.j[k++] = {X, dZ, ldx, M, N, w, 0};
    J.j[k++] = {nullptr, dZ, 1, 1, N, b, 0};
  };
  auto mnet = [&](const MNet& m, const MPlanes& M) {
    layer(P.x, L.K, M.d1, L.K, H, m.w1, m.b1);
    layer(M.he, HE, M.d2, HE, L.A, m.w2, m.b2);
    layer(M.f, L.A, M.d3, L.A, L.A, m.w3, m.b3);
  };
  if (L.algo == BC) mnet(L.imi, P.mp[0]);
  if (L.algo == BCQ) { mnet(L.q, P.mp[0]); mnet(L.imi, P.mp[1]); }
  if (L.algo == CQL) {
    layer(P.x, L.K, P.c1, L.K, H, L.c.w1, L.c.b1);
    layer(P.h1, H, P.c2, H, H, L.c.w2, L.c.b2);
    layer(P.h2, H, P.c3, H, L.A, L.c.w3, L.c.b3);
  }
  r4dense::tile_jobs(J, k);
  return J;
}

// The embedding gradient: one thread per element (row r, column c) of one net's table sums de[q][j][c] over the samples q
// and slots j with ids[q][j] == r, in (q, j) order.  grid = nets x ceil(A * E / EGT).
constexpr int EGT = 256, EGCH = 2048;
__global__ void __launch_bounds__(EGT) k_bq_embgrad(Layout L, Planes P, int n, int cta_per_net) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  __shared__ int sid[EGCH];
  const int net = blockIdx.x / cta_per_net;
  const int e = (blockIdx.x % cta_per_net) * EGT + threadIdx.x;
  const int r = e / E, c = e % E;
  const MNet& m = (L.algo == BCQ && net == 1) ? L.imi : (L.algo == BCQ ? L.q : L.imi);
  const float* de = P.mp[net].de;
  float acc = 0.f;
  const int total = n * W;
  for (int b = 0; b < total; b += EGCH) {
    __syncthreads();
    for (int i = threadIdx.x; i < EGCH && b + i < total; i += EGT) sid[i] = P.ids[b + i];
    __syncthreads();
    if (r < L.A) {
      const int end = min(EGCH, total - b);
      for (int i = 0; i < end; ++i)
        if (sid[i] == r) acc += de[(size_t)(b + i) * E + c];
    }
  }
  if (r < L.A) P.grad[m.emb + e] = acc;
}

// Adam (torch.optim.Adam, betas 0.9 / 0.999), then target = params on the Q part when copy_target.
__global__ void k_bq_apply(int np, int ntgt, float* __restrict__ prm, float* __restrict__ tgt, const float* __restrict__ grad,
                           float* __restrict__ m, float* __restrict__ v, int step, float lr, float eps, int copy_target) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= np) return;
  float p = prm[i], mi = m[i], vi = v[i];
  r4ppo::adam_update(grad[i], p, mi, vi, step, lr, 0.9f, 0.999f, eps);
  prm[i] = p; m[i] = mi; v[i] = vi;
  if (copy_target && i < ntgt) tgt[i] = p;
}

// ------------------------------------------------------------------------------------------------
// act.  mode 0: the evaluation rule of rl4rs/policy/policy_model.py predict_with_mask -- action_probs (BC: the imitator's
// log-probs, BCQ / CQL: softmax(Q)), -2^15 where keep is 0, the first argmax.  mode 1: d3rlpy's predict (BC: argmax of the
// log-probs, BCQ: the imitator-filtered argmax of Q, CQL: argmax Q).  probs [n][A] (may be NULL) receives action_probs,
// values [n][A] (may be NULL) the raw net output (BC: logits, BCQ / CQL: Q).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) k_bq_act(Layout L, const float* __restrict__ prm, const float* __restrict__ obs32,
                                               const double* __restrict__ obs64, int n, Data D, int mode, float log_flex,
                                               int32_t* __restrict__ action, float* __restrict__ probs, float* __restrict__ values) {
  extern __shared__ __align__(16) float sm[];
  const int K = L.K, A = L.A, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int AB = TS * plane(A);
  float *x = sm, *he = x + TS * K, *dhe = he + TS * HE, *f = dhe + TS * HE, *z = f + AB, *pr = z + AB;
  float *aux = pr + AB, *keep = aux + AB;
  int* ids = reinterpret_cast<int*>(keep + AB);
  __shared__ int64_t row[TS];
  __shared__ int hs[TS];
  const int s0 = blockIdx.x * TS, nvalid = min(TS, n - s0);
  if (tid < TS) row[tid] = s0 + min(tid, nvalid - 1);
  __syncthreads();
  load_rows(L, obs32, obs64, row, nvalid, D, x, ids, keep, hs);
  if (L.algo == CQL) c_forward(prm, L.c, L, x, he, dhe, z);
  else m_forward(prm, L.algo == BC ? L.imi : L.q, L, x, ids, keep, he, f, z);
  {
    const float* q = z + warp * A;
    float* p = pr + warp * A;
    const float lse = warp_lse(q, A);
    for (int a = lane; a < A; a += 32) p[a] = L.algo == BC ? q[a] - lse : expf(q[a] - lse);
  }
  __syncthreads();
  for (int i = tid; i < nvalid * A; i += NT) {
    if (probs) probs[(size_t)s0 * A + i] = pr[i];
    if (values) values[(size_t)s0 * A + i] = z[i];
  }
  if (mode == 1 && L.algo == BCQ) {
    for (int i = tid; i < TS * A; i += NT) aux[i] = z[i];
    __syncthreads();
    m_forward(prm, L.imi, L, x, ids, keep, he, f, z);
    const float* q = aux + warp * A;
    const float* lg = z + warp * A;
    const float lse = warp_lse(lg, A);
    float lpm = -INFINITY, qm = INFINITY;
    for (int a = lane; a < A; a += 32) { lpm = fmaxf(lpm, lg[a] - lse); qm = fminf(qm, q[a]); }
    lpm = warp_max(lpm); qm = warp_min(qm);
    float* fl = pr + warp * A;
    for (int a = lane; a < A; a += 32) fl[a] = (q[a] - qm) * (((lg[a] - lse) - lpm) > log_flex ? 1.f : 0.f);
  } else if (mode == 0) {
    for (int i = tid; i < TS * A; i += NT)
      if (keep[i] == 0.f) pr[i] = -32768.f;
  }
  __syncthreads();
  const int a = warp_argmax(pr + warp * A, A);
  if (lane == 0 && warp < nvalid) action[s0 + warp] = a;
}
__host__ __device__ inline size_t act_smem(int K, int A) { return rows_smem(K, A); }
// the shared planes of k_bq_rows / k_bq_act (with the 1 KB of static shared memory) fit the 227 KB of an H100 SM
inline bool dims_ok(int algo, int K, int A) {
  return algo >= BC && algo <= CQL && K > W && K <= MAXK && A >= 2 && A <= MAXA && rows_smem(K, A) + 1024 <= 227 * 1024;
}

// ------------------------------------------------------------------------------------------------
// The transition list: index[t] = the t-th entry i (in order) with term[i] == 0 and i < the last terminal entry, i.e. every
// entry that has a successor in its episode (episodes end at terminal entries; entries after the last terminal are an
// unfinished episode and are dropped).  One CTA: per-thread chunk counts, a prefix over the threads, then the writes.
// ------------------------------------------------------------------------------------------------
constexpr int TRT = 1024;
__global__ void __launch_bounds__(TRT) k_bq_transitions(const uint8_t* __restrict__ term, int64_t N, int64_t* __restrict__ index,
                                                        int64_t* __restrict__ count) {
  __shared__ int64_t part[TRT + 1];
  __shared__ int64_t lastw[TRT / 32];
  const int tid = threadIdx.x;
  const int64_t per = (N + TRT - 1) / TRT, lo = min((int64_t)tid * per, N), hi = min(lo + per, N);
  int64_t last = -1;
  for (int64_t i = lo; i < hi; ++i)
    if (term[i]) last = i;
  for (int o = 16; o > 0; o >>= 1) last = max(last, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)last, o));
  if ((tid & 31) == 0) lastw[tid >> 5] = last;
  __syncthreads();
  if (tid == 0) {
    int64_t m = -1;
    for (int w = 0; w < TRT / 32; ++w) m = max(m, lastw[w]);
    lastw[0] = m;
  }
  __syncthreads();
  const int64_t lt = lastw[0];
  int64_t c = 0;
  for (int64_t i = lo; i < hi; ++i) c += (i < lt && !term[i]) ? 1 : 0;
  part[tid + 1] = c;
  __syncthreads();
  if (tid == 0) {
    part[0] = 0;
    for (int k = 1; k <= TRT; ++k) part[k] += part[k - 1];
    count[0] = part[TRT];
  }
  __syncthreads();
  int64_t o = part[tid];
  for (int64_t i = lo; i < hi; ++i)
    if (i < lt && !term[i]) index[o++] = i;
}

}  // namespace r4bq

#include "r4_cqlconti.cuh"   // continuous-action CQL, on the same dataset planes and launch family
#include "r4_bcqconti.cuh"   // continuous-action BCQ, likewise
#include "r4_ope.cuh"         // off-policy evaluation of the batch-RL and model-free policies: its own launch family
