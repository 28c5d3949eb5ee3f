// r4_dense.cuh -- the dense-layer kernels the learner families share: the tiled fp32 GEMM, the weight-gradient jobs and
// Keras / TF1 Adam.  fp32 CUDA cores (parity with float64 references is the bar), deterministic: every output element has
// one writer that sums in a fixed order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace r4dense {

constexpr int NT = 256;

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float elu(float x) { return x > 0.f ? x : expm1f(x); }

// ------------------------------------------------------------------------------------------------
// k_dense_gemm: C[z](m, n) = epilogue(alpha sum_k A[z](m, k) B[z](k, n)).  Operand X's element (i, j) of batch z sits at
// X + (z / zdiv) so + (z % zdiv) si + i s0 + j s1; a transposed row-major B is Op{B, 0, 0, 1, ldb}.  ktot > 0: split-K,
// batch z covers k in [z K, min((z + 1) K, ktot)) and A / B advance by z K along k (their batch strides are then ignored),
// C by z cso.  The epilogue, in this order:
//   v = alpha acc;  v += bias[n] (bias may be NULL);  then by epi
//     EP_LIN  v        EP_RELU  max(v, 0)     EP_SIG  sigmoid(v)     EP_ELU  elu(v)
//     EP_DSIG v y (1 - y)      EP_DELU  v (y > 0 ? 1 : y + 1)        EP_DRELU  y > 0 ? v : 0
//     (y = aux[m][n], the forward activation);
//   pre[m][n] = v (pre may be NULL);  v *= mul[m][n] (mul may be NULL);  C = accum ? C + v : v.
// aux, mul and pre have leading dimension N and serve unbatched products only.
// 64 x 64 tile, 256 threads of 4 x 4 outputs, K in 16-deep slices through shared memory, each output summed over k in order.
// AT: A is m-contiguous (s0 == 1), else k-contiguous (s1 == 1); BT: B is k-contiguous (s0 == 1), else n-contiguous
// (s1 == 1).  The layouts are template parameters so the loaders index with a known unit stride (gemm_kernel picks one).
// ------------------------------------------------------------------------------------------------
enum { EP_LIN = 0, EP_RELU, EP_SIG, EP_ELU, EP_DSIG, EP_DELU, EP_DRELU };
struct Op { const float* p; int64_t so, si, s0, s1; };
struct Gemm {
  Op A, B;
  float* C; int64_t cso, csi, cs0, cs1;
  const float* bias;
  const float* aux;
  const float* mul;
  float* pre;
  int M, N, K, zdiv;
  int64_t ktot;
  float alpha;
  int epi, accum;
};
constexpr int GT = 64, GK = 16;
// The sigmoid / ELU activations and their derivatives (y = the forward activation), called out of line: inlined at each
// of a thread's 16 outputs they made the kernel 1.6 times as long, which slowed the small, latency-bound products.
__device__ __noinline__ float activate(float v, int epi, float y) {
  if (epi == EP_SIG) return sigm(v);
  if (epi == EP_ELU) return elu(v);
  if (epi == EP_DSIG) return v * (y * (1.f - y));
  if (epi == EP_DRELU) return y > 0.f ? v : 0.f;
  return v * (y > 0.f ? 1.f : y + 1.f);
}
// At most 48 registers (5 CTAs per SM): ptxas would take 64, and fits 48 without spills.
template <bool AT, bool BT>
__global__ void __launch_bounds__(NT, 5) k_dense_gemm(Gemm g) {
  __shared__ float As[GK][GT + 4], Bs[GK][GT + 4];
  const int z = blockIdx.z, zo = z / g.zdiv, zi = z % g.zdiv;
  const int m0 = blockIdx.y * GT, n0 = blockIdx.x * GT;
  const float* A = g.A.p;
  const float* B = g.B.p;
  int K = g.K;
  if (g.ktot > 0) {
    const int64_t k0 = (int64_t)z * g.K;
    A += k0 * g.A.s1; B += k0 * g.B.s0;
    K = (int)min((int64_t)g.K, g.ktot - k0);
  } else {
    A += zo * g.A.so + zi * g.A.si; B += zo * g.B.so + zi * g.B.si;
  }
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += GK) {
    for (int e = tid; e < GT * GK; e += NT) {
      // A: e -> (m, k) with its contiguous index fastest; B likewise with (k, n)
      const int am = AT ? e % GT : e / GK, ak = AT ? e / GT : e % GK;
      const int bk = BT ? e % GK : e / GT, bn = BT ? e / GK : e % GT;
      const int gm = m0 + am, gk = k0 + ak;
      As[ak][am] = (gm < g.M && gk < K) ? (AT ? A[gm + (int64_t)gk * g.A.s1] : A[gm * g.A.s0 + gk]) : 0.f;
      const int gk2 = k0 + bk, gn = n0 + bn;
      Bs[bk][bn] = (gn < g.N && gk2 < K) ? (BT ? B[gk2 + gn * g.B.s1] : B[(int64_t)gk2 * g.B.s0 + gn]) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty + 16 * i]; b[i] = Bs[kk][tx + 16 * i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* C = g.C + (g.ktot > 0 ? (int64_t)z * g.cso : zo * g.cso + zi * g.csi);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty + 16 * i;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx + 16 * j;
      if (n >= g.N) continue;
      const size_t o = (size_t)m * g.N + n;
      float v = g.alpha * acc[i][j];
      if (g.bias) v += g.bias[n];
      if (g.epi == EP_RELU) v = fmaxf(v, 0.f);
      else if (g.epi != EP_LIN) v = activate(v, g.epi, g.epi >= EP_DSIG ? g.aux[o] : 0.f);
      if (g.pre) g.pre[o] = v;
      if (g.mul) v *= g.mul[o];
      float* c = C + m * g.cs0 + n * g.cs1;
      *c = g.accum ? *c + v : v;
    }
  }
}

// The instance of k_dense_gemm for g's operand layouts.
inline void (*gemm_kernel(const Gemm& g))(Gemm) {
  if (g.A.s1 != 1) return g.B.s1 != 1 ? k_dense_gemm<true, true> : k_dense_gemm<true, false>;
  return g.B.s1 != 1 ? k_dense_gemm<false, true> : k_dense_gemm<false, false>;
}

// ------------------------------------------------------------------------------------------------
// k_dense_wgrad: weight gradients as jobs.  Job j: out[i][c] = sum_q X[q][i] dZ[q][c] over the n rows q, X at row stride
// ldx (X == NULL: a bias, X = 1 and M = 1), stored at grad + off as [M][N], or added to it when first == 0 (a later chunk
// of rows).  One CTA owns one 64 x 64 output tile and walks the rows in order: every gradient element has one writer and a
// fixed summation order, so the result is deterministic without per-CTA partial gradients.  Launched with ntiles + 1
// CTAs, the last sums the per-row loss statistics (Stats).
// ------------------------------------------------------------------------------------------------
constexpr int NJOB = 18, WT = 64, WK = 32;
struct Job {
  const float* X;
  const float* Z;
  int ldx, M, N, off, tile0;
};
struct Jobs {
  Job j[NJOB];
  int njob, ntiles;
};
// Numbers the tiles of the first njob jobs, in job order.
inline void tile_jobs(Jobs& J, int njob) {
  J.njob = njob;
  int t = 0;
  for (int i = 0; i < njob; ++i) {
    J.j[i].tile0 = t;
    t += ((J.j[i].M + WT - 1) / WT) * ((J.j[i].N + WT - 1) / WT);
  }
  J.ntiles = t;
}
// The job of the gradient [M][N] at grad + off from X (row stride ldx; NULL: a bias, M = 1) and dZ [n][N].
inline Job grad_job(const float* X, int ldx, const float* dZ, int M, int N, int64_t off) {
  return Job{X, dZ, ldx, M, N, (int)off, 0};
}
// Appends the two jobs of one dense layer over its output gradient dZ [n][N] at k: its weight [M][N] at off w from X at
// row stride ldx, then its bias [N] at off b.
inline void layer_jobs(Jobs& J, int& k, const float* X, int ldx, const float* dZ, int M, int N, int64_t w, int64_t b) {
  J.j[k++] = grad_job(X, ldx, dZ, M, N, w);
  J.j[k++] = grad_job(nullptr, 1, dZ, 1, N, b);
}
// The statistics: column c < cols of the rows in[n][cols], summed in row order from 0, or from run[c] when run is given and
// first == 0.  run (may be NULL) keeps the sum; out (may be NULL) receives sum * scale, or with add fmaf(sum, scale, out).
struct Stats {
  const float* in;
  int cols;
  float* run;
  float* out;
  float scale;
  int add;
};

__global__ void __launch_bounds__(NT) k_dense_wgrad(Jobs jobs, int n, int first, float* __restrict__ grad, Stats st) {
  __shared__ float xs[WK][WT];
  __shared__ float zs[WK][WT];
  const int tid = threadIdx.x;
  if ((int)blockIdx.x == jobs.ntiles) {
    if (tid < st.cols) {
      float a = st.run && !first ? st.run[tid] : 0.f;
      for (int q = 0; q < n; ++q) a += st.in[q * st.cols + tid];
      if (st.run) st.run[tid] = a;
      if (st.out) st.out[tid] = st.add ? fmaf(a, st.scale, st.out[tid]) : a * st.scale;
    }
    return;
  }
  int jb = 0;
  while (jb + 1 < jobs.njob && (int)blockIdx.x >= jobs.j[jb + 1].tile0) ++jb;
  const Job J = jobs.j[jb];
  const int t = blockIdx.x - J.tile0, tn = (J.N + WT - 1) / WT;
  const int i0 = (t / tn) * WT, c0 = (t % tn) * WT;
  const int ty = tid / 16, tx = tid % 16;                  // rows i0 + 4 ty .. +3, columns c0 + 4 tx .. +3
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
  for (int k0 = 0; k0 < n; k0 += WK) {
    __syncthreads();
    for (int e = tid; e < WK * WT; e += NT) {
      const int k = e / WT, c = e % WT, q = k0 + k;
      const bool ok = q < n;
      xs[k][c] = (ok && i0 + c < J.M) ? (J.X ? J.X[(size_t)q * J.ldx + i0 + c] : 1.f) : 0.f;
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

// ------------------------------------------------------------------------------------------------
// Keras Adam (OptimizerV2 / ResourceApplyAdam; TF1's AdamOptimizer is the same update): m += (g - m)(1 - b1),
// v += (g^2 - v)(1 - b2), p -= alpha m / (sqrt(v) + eps) with alpha = lr sqrt(1 - b2^t) / (1 - b1^t).  Dense over every
// parameter (the sparse embedding apply of OptimizerV2 decays m and v on every row too).  Clears the nonzero gradient
// entries of the two embedding tables [emb_cat, emb_cat + len) and [emb_seq, emb_seq + len), so their part of grad is zero
// again for the next pass (a net without a sequence table names its category table twice; len 0: no table).
// ------------------------------------------------------------------------------------------------
__global__ void k_keras_adam(int64_t np, int64_t len, int64_t emb_cat, int64_t emb_seq, float* __restrict__ prm,
                             float* __restrict__ grad, float* __restrict__ m, float* __restrict__ v, float alpha, float b1,
                             float b2, float eps) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= np) return;
  const float g = grad[i];
  float mi = m[i], vi = v[i];
  mi += (g - mi) * (1.f - b1);
  vi += (g * g - vi) * (1.f - b2);
  prm[i] -= alpha * mi / (sqrtf(vi) + eps);
  m[i] = mi; v[i] = vi;
  const bool emb = (i >= emb_cat && i < emb_cat + len) || (i >= emb_seq && i < emb_seq + len);
  if (emb && g != 0.f) grad[i] = 0.f;
}

}  // namespace r4dense
