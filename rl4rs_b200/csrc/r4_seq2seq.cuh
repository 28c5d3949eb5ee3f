// r4_seq2seq.cuh -- the MDP checker's encoder-decoder transformer (keras-transformer 0.40's get_model): the row kernels of
// its forward and backward, the clipped masked cross-entropy, the embedding-gradient scatter and the beam-search selection.
// fp32 CUDA cores (parity with a float64 autograd reference is the bar), deterministic: every output element has one
// writer that sums in a fixed order.  The dropout draws are Exact-K's (r4ek::kept).
//
// Model, E = embed_dim, H heads of E / H, F = hidden_dim (include/rl4rs_b200.h lists the flat parameters):
//   X0 = emb[token] + trig(position)                                  k_s2s_embed
//   sub-layer  out = LN(x + dropout(f(x))), eps 1e-14                  k_s2s_ln / k_s2s_ln_bwd
//   attention  softmax(QK^T / sqrt(E / H) - 1e4 causal - 1e4 (1 - key mask)) V, projections through r4dense::k_dense_gemm
//                                                                      k_s2s_softmax / k_s2s_softmax_bwd
//   FFN        relu(x W1 + b1) W2 + b2 (the relu backward is k_dense_gemm's EP_DRELU epilogue)
//   output     softmax(h emb_dec^T + b); loss sum(mask ce) / sum(mask), ce on probabilities clipped to [1e-7, 1 - 1e-7]
//                                                                      k_s2s_count, k_s2s_out, k_s2s_lsum
//   embedding gradient   tokens grouped by value in position order     k_s2s_tok_csr, k_s2s_tok_place, k_s2s_emb_grad
//   beam search          top-k per prefix, top-beam of the products    k_s2s_topk, k_s2s_beam; k_s2s_pick
//   Adam                 k_s2s_adam (r4dense::k_keras_adam)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "r4_dense.cuh"
#include "r4_exactk.cuh"

namespace r4s2s {

// the family's Adam: keras 2.2.5's update is r4dense::k_keras_adam's (dense over every parameter)
constexpr auto k_s2s_adam = r4dense::k_keras_adam;

constexpr int MAXE = 512, MAXF = 1024, MAXBLK = 6, MAXT = 64, MINV = 4, MAXV = 65536;
constexpr int MAXBEAM = 256, MAXK = 8192;        // beam width; top-k of one call (the candidate list) at most
constexpr float MASKV = 10000.f;
constexpr float CLIP = 1e-7f;

// ---- parameter layout (floats) in the order include/rl4rs_b200.h documents ----
struct Cfg { int Vs, Vt, E, H, F, Le, Ld, same; };
struct Att { int64_t wq, bq, wk, bk, wv, bv, wo, bo; };
struct Norm { int64_t g, b; };
struct FF { int64_t w1, b1, w2, b2; };
struct EncBlk { Att sa; Norm n1; FF ff; Norm n2; };
struct DecBlk { Att sa; Norm n1; Att qa; Norm n2; FF ff; Norm n3; };
struct Layout {
  int64_t emb_enc, emb_dec;
  EncBlk enc[MAXBLK];
  DecBlk dec[MAXBLK];
  int64_t out_b, n;
};
inline Layout make_layout(const Cfg& c) {
  Layout L = {};
  int64_t o = 0;
  const int64_t E = c.E;
  auto take = [&](int64_t k) { int64_t r = o; o += k; return r; };
  auto att = [&](Att& a) {
    a.wq = take(E * E); a.bq = take(E); a.wk = take(E * E); a.bk = take(E);
    a.wv = take(E * E); a.bv = take(E); a.wo = take(E * E); a.bo = take(E);
  };
  auto norm = [&](Norm& n) { n.g = take(E); n.b = take(E); };
  auto ff = [&](FF& f) { f.w1 = take(E * c.F); f.b1 = take(c.F); f.w2 = take((int64_t)c.F * E); f.b2 = take(E); };
  L.emb_enc = take((int64_t)c.Vs * E);
  L.emb_dec = c.same ? L.emb_enc : take((int64_t)c.Vt * E);
  for (int l = 0; l < c.Le; ++l) { att(L.enc[l].sa); norm(L.enc[l].n1); ff(L.enc[l].ff); norm(L.enc[l].n2); }
  for (int l = 0; l < c.Ld; ++l) {
    DecBlk& d = L.dec[l];
    att(d.sa); norm(d.n1); att(d.qa); norm(d.n2); ff(d.ff); norm(d.n3);
  }
  L.out_b = take(c.Vt);
  L.n = o;
  return L;
}

// the dropout keep of element elem of sub-layer `layer` in call `call`: Exact-K's draw, on the stream-0 key call * 32 + layer
__device__ __forceinline__ bool keep(uint64_t seed, uint64_t call, int layer, uint64_t elem, float rate) {
  return r4ek::kept(seed, call * 32u + (uint64_t)layer, 0, elem, rate);
}

// block-wide sum / max in a fixed tree (blockDim.x a multiple of 32, at most 1024); red holds 32 floats
__device__ inline float block_sum(float v, float* red) {
  const int lane = threadIdx.x % 32, w = threadIdx.x / 32, nw = blockDim.x / 32;
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float s = 0.f;
  for (int i = 0; i < nw; ++i) s += red[i];
  return s;
}
__device__ inline float block_max(float v, float* red) {
  const int lane = threadIdx.x % 32, w = threadIdx.x / 32, nw = blockDim.x / 32;
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float s = -INFINITY;
  for (int i = 0; i < nw; ++i) s = fmaxf(s, red[i]);
  return s;
}

__device__ __forceinline__ int clamp_tok(int t, int V) { return min(max(t, 0), V - 1); }

// k_s2s_embed: X[r T + t, c] = emb[tok[r ld + t], c] + trig(t, c), trig(t, 2k) = sin(t / 10000^(2k / E)), trig(t, 2k + 1) =
// cos(the same angle).  Tokens outside [0, V) are clamped into it.
__global__ void k_s2s_embed(const int32_t* __restrict__ tok, int64_t ld, int rows, int T, const float* __restrict__ emb,
                            int V, int E, float* __restrict__ X) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)rows * T * E) return;
  const int c = (int)(e % E);
  const int64_t q = e / E;
  const int t = (int)(q % T);
  const int64_t r = q / T;
  const int v = clamp_tok(tok[r * ld + t], V);
  const float inv = 1.0f / powf(10000.0f, (float)(c - c % 2) / (float)E);
  const float ang = (float)t * inv;
  X[e] = emb[(int64_t)v * E + c] + (c % 2 == 0 ? sinf(ang) : cosf(ang));
}

// k_s2s_softmax: one warp per score row (g, h, m) of S [G, H, Mq, Tk], in place: A = softmax(s - 1e4 [causal and j > m % Tq]
// - 1e4 [tok[g kld + j] == 0]), the max subtracted first.  Tk <= 64.
__global__ void k_s2s_softmax(float* __restrict__ S, const int32_t* __restrict__ ktok, int64_t kld, int64_t rows, int H,
                              int Mq, int Tk, int Tq, int causal) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (row >= rows) return;
  const int m = (int)(row % Mq);
  const int64_t g = row / ((int64_t)H * Mq);
  const int qp = m % Tq;
  float* s = S + row * Tk;
  float v[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int j = lane + 32 * k;
    v[k] = -INFINITY;
    if (j < Tk) {
      float x = s[j];
      if (causal && j > qp) x -= MASKV;
      if (ktok[g * kld + j] == 0) x -= MASKV;
      v[k] = x;
    }
  }
  float mx = fmaxf(v[0], v[1]);
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float e[2], den = 0.f;
#pragma unroll
  for (int k = 0; k < 2; ++k) { e[k] = lane + 32 * k < Tk ? expf(v[k] - mx) : 0.f; den += e[k]; }
  for (int o = 16; o; o >>= 1) den += __shfl_xor_sync(0xffffffffu, den, o);
#pragma unroll
  for (int k = 0; k < 2; ++k)
    if (lane + 32 * k < Tk) s[lane + 32 * k] = e[k] / den;
}

// k_s2s_softmax_bwd: dS = A (dA - sum_j A dA), in place on dA; one warp per row of Tk <= 64
__global__ void k_s2s_softmax_bwd(const float* __restrict__ A, float* __restrict__ dA, int64_t rows, int Tk) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (row >= rows) return;
  float a[2], d[2], dot = 0.f;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int j = lane + 32 * k;
    a[k] = j < Tk ? A[row * Tk + j] : 0.f;
    d[k] = j < Tk ? dA[row * Tk + j] : 0.f;
    dot += a[k] * d[k];
  }
  for (int o = 16; o; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
#pragma unroll
  for (int k = 0; k < 2; ++k)
    if (lane + 32 * k < Tk) dA[row * Tk + lane + 32 * k] = a[k] * (d[k] - dot);
}

// k_s2s_ln: out = gamma xhat + beta, xhat = (z - mean) / sqrt(var + 1e-14), z = X + dropout(Y); one warp per row of E
// (E a multiple of 32, at most 512).  Stores xhat and 1 / std.
__global__ void k_s2s_ln(const float* __restrict__ X, const float* __restrict__ Y, int64_t R, int E,
                         const float* __restrict__ gamma, const float* __restrict__ beta, uint64_t seed, uint64_t call,
                         int layer, float rate, float* __restrict__ out, float* __restrict__ xh, float* __restrict__ rs) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32, nk = E / 32;
  if (r >= R) return;
  const float ks = 1.0f / (1.0f - rate);
  float z[MAXE / 32], s = 0.f;
#pragma unroll
  for (int k = 0; k < MAXE / 32; ++k) {
    if (k >= nk) break;
    const int64_t o = r * E + lane + 32 * k;
    z[k] = X[o] + (keep(seed, call, layer, (uint64_t)o, rate) ? Y[o] * ks : 0.f);
    s += z[k];
  }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / E;
  float v = 0.f;
#pragma unroll
  for (int k = 0; k < MAXE / 32; ++k) {
    if (k >= nk) break;
    z[k] -= mean;
    v += z[k] * z[k];
  }
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const float rstd = 1.0f / sqrtf(v / E + 1e-14f);
#pragma unroll
  for (int k = 0; k < MAXE / 32; ++k) {
    if (k >= nk) break;
    const int c = lane + 32 * k;
    const float x = z[k] * rstd;
    xh[r * E + c] = x;
    out[r * E + c] = x * gamma[c] + beta[c];
  }
  if (lane == 0) rs[r] = rstd;
}

// k_s2s_ln_bwd: from dOut: dZ = rstd (g - mean(g) - xhat mean(g xhat)), g = dOut gamma (the residual's gradient),
// dY = dropout'(dZ) (the sub-layer output's), gx = dOut xhat (for gamma's gradient).  dOut is left as it is.
__global__ void k_s2s_ln_bwd(const float* __restrict__ dOut, const float* __restrict__ xh, const float* __restrict__ rs,
                             int64_t R, int E, const float* __restrict__ gamma, uint64_t seed, uint64_t call, int layer,
                             float rate, float* __restrict__ dZ, float* __restrict__ dY, float* __restrict__ gx) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32, nk = E / 32;
  if (r >= R) return;
  float g[MAXE / 32], x[MAXE / 32], s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int k = 0; k < MAXE / 32; ++k) {
    if (k >= nk) break;
    const int64_t o = r * E + lane + 32 * k;
    const float dy = dOut[o];
    x[k] = xh[o];
    gx[o] = dy * x[k];
    g[k] = dy * gamma[lane + 32 * k];
    s1 += g[k]; s2 += g[k] * x[k];
  }
  for (int o = 16; o; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
  const float rstd = rs[r], ks = 1.0f / (1.0f - rate);
#pragma unroll
  for (int k = 0; k < MAXE / 32; ++k) {
    if (k >= nk) break;
    const int64_t o = r * E + lane + 32 * k;
    const float dz = rstd * (g[k] - s1 / E - x[k] * (s2 / E));
    dZ[o] = dz;
    dY[o] = keep(seed, call, layer, (uint64_t)o, rate) ? dz * ks : 0.f;
  }
}

// k_s2s_count: inv[0] = 1 / sum_q (tok[q] != 0) over the N decoder-input tokens (one CTA of 1024, fixed order)
__global__ void __launch_bounds__(1024) k_s2s_count(const int32_t* __restrict__ tok, int N, float* __restrict__ inv) {
  __shared__ float red[32];
  float c = 0.f;
  for (int q = threadIdx.x; q < N; q += blockDim.x) c += tok[q] != 0 ? 1.f : 0.f;
  const float s = block_sum(c, red);
  if (threadIdx.x == 0) inv[0] = 1.0f / s;
}

// k_s2s_out: one CTA per row of logits Z [rows, V] (bias added), in place.  y == NULL: Z = softmax(Z).  Otherwise the
// clipped cross-entropy of keras 2.2.5 (log of the clipped probabilities q, renormalised by sparse softmax
// cross-entropy; tf.clip_by_value passes the gradient on [1e-7, 1 - 1e-7], ends included): ce = log(sum q) - log q_y;
// Z = d(mask ce inv) / d(logits) with mask = (mtok != 0), inv = *inv; ce_row[q] = mask ce.  Each thread reads and writes
// only its own columns after the reductions.  Tokens y outside [0, V) are clamped into it.
__global__ void __launch_bounds__(256) k_s2s_out(float* __restrict__ Z, int V, const int32_t* __restrict__ y,
                                                 const int32_t* __restrict__ mtok, const float* __restrict__ inv,
                                                 float* __restrict__ ce_row) {
  __shared__ float red[32];
  const int64_t q = blockIdx.x;
  float* z = Z + q * V;
  const int t = y ? clamp_tok(y[q], V) : 0;
  // the target's logit, read before any thread overwrites its columns with the gradient below (no barrier separates the
  // write loop from a late warp's reads)
  const float zt = y ? z[t] : 0.f;
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < V; j += blockDim.x) mx = fmaxf(mx, z[j]);
  mx = block_max(mx, red);
  float den = 0.f;
  for (int j = threadIdx.x; j < V; j += blockDim.x) den += expf(z[j] - mx);
  den = block_sum(den, red);
  if (!y) {
    for (int j = threadIdx.x; j < V; j += blockDim.x) z[j] = expf(z[j] - mx) / den;
    return;
  }
  float sq = 0.f, a1 = 0.f;
  for (int j = threadIdx.x; j < V; j += blockDim.x) {
    const float p = expf(z[j] - mx) / den;
    const bool in = p >= CLIP && p <= 1.f - CLIP;
    sq += fminf(fmaxf(p, CLIP), 1.f - CLIP);
    a1 += in ? p : 0.f;
  }
  sq = block_sum(sq, red);
  a1 = block_sum(a1, red);
  const float pt = expf(zt - mx) / den;
  const bool int_ = pt >= CLIP && pt <= 1.f - CLIP;
  const float qt = fminf(fmaxf(pt, CLIP), 1.f - CLIP);
  const float msk = mtok[q] != 0 ? 1.f : 0.f, sc = msk * inv[0];
  // dL/dp_j = in_j (1 / S - [j == t] / q_t); dL/dz_k = p_k (dL/dp_k - sum_j p_j dL/dp_j), sum_j p_j dL/dp_j = a1 / S - in_t
  const float dot = a1 / sq - (int_ ? 1.f : 0.f);
  for (int j = threadIdx.x; j < V; j += blockDim.x) {
    const float p = expf(z[j] - mx) / den;
    const bool in = p >= CLIP && p <= 1.f - CLIP;
    const float dp = in ? (1.f / sq - (j == t ? 1.f / qt : 0.f)) : 0.f;
    z[j] = sc * p * (dp - dot);
  }
  if (threadIdx.x == 0) ce_row[q] = msk * (logf(sq) - logf(qt));
}

// k_s2s_lsum: loss[0] = inv[0] sum_q ce_row[q] (one CTA of 1024, fixed order)
__global__ void __launch_bounds__(1024) k_s2s_lsum(const float* __restrict__ ce_row, int N, const float* __restrict__ inv,
                                                   float* __restrict__ loss) {
  __shared__ float red[32];
  float c = 0.f;
  for (int q = threadIdx.x; q < N; q += blockDim.x) c += ce_row[q];
  const float s = block_sum(c, red) * inv[0];
  if (threadIdx.x == 0) loss[0] = s;
}

// ---- embedding gradient: the positions of each token value in position order, then one writer per (value, column) ----
// k_s2s_tok_csr (one CTA of 1024): cnt[v] = positions holding v, off[v] = their exclusive prefix sum.  Positions
// q = r T + t read tok[r ld + t].
__global__ void __launch_bounds__(1024) k_s2s_tok_csr(const int32_t* __restrict__ tok, int64_t ld, int rows, int T, int V,
                                                      int* __restrict__ cnt, int* __restrict__ off) {
  __shared__ int part[1024];
  for (int v = threadIdx.x; v < V; v += blockDim.x) cnt[v] = 0;
  __syncthreads();
  for (int q = threadIdx.x; q < rows * T; q += blockDim.x) atomicAdd(&cnt[clamp_tok(tok[(int64_t)(q / T) * ld + q % T], V)], 1);
  __syncthreads();
  const int per = (V + blockDim.x - 1) / blockDim.x, v0 = threadIdx.x * per;
  int s = 0;
  for (int v = v0; v < min(V, v0 + per); ++v) s += cnt[v];
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int i = 0; i < (int)blockDim.x; ++i) { const int c = part[i]; part[i] = run; run += c; }
  }
  __syncthreads();
  s = part[threadIdx.x];
  for (int v = v0; v < min(V, v0 + per); ++v) { off[v] = s; s += cnt[v]; }
}

// k_s2s_tok_place: order[off[v] + rank] = q, rank = the positions before q holding the same v (position order)
__global__ void __launch_bounds__(256) k_s2s_tok_place(const int32_t* __restrict__ tok, int64_t ld, int rows, int T, int V,
                                                       const int* __restrict__ off, int* __restrict__ order) {
  __shared__ int tile[256];
  const int N = rows * T;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int v = q < N ? clamp_tok(tok[(int64_t)(q / T) * ld + q % T], V) : -1;
  int rank = 0;
  for (int b = 0; b < (int)(blockIdx.x + 1) * (int)blockDim.x && b < N; b += blockDim.x) {
    __syncthreads();
    const int p = b + threadIdx.x;
    tile[threadIdx.x] = p < N ? clamp_tok(tok[(int64_t)(p / T) * ld + p % T], V) : -2;
    __syncthreads();
    const int lim = min((int)blockDim.x, q - b);
    for (int i = 0; i < lim; ++i) rank += tile[i] == v;
  }
  if (q < N) order[off[v] + rank] = q;
}

// k_s2s_emb_grad: dEmb[v, c] += sum over v's positions q (in order) of dX[q, c]; one thread per (v, c)
__global__ void k_s2s_emb_grad(const float* __restrict__ dX, int E, int V, const int* __restrict__ cnt,
                               const int* __restrict__ off, const int* __restrict__ order, float* __restrict__ dEmb) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)V * E) return;
  const int v = (int)(e / E), c = (int)(e % E), k = cnt[v];
  if (k == 0) return;
  const int* o = order + off[v];
  float s = 0.f;
  for (int i = 0; i < k; ++i) s += dX[(int64_t)o[i] * E + c];
  dEmb[e] += s;
}

// ---- beam search ----
// cta_topk: the k largest of N non-negative doubles key(i) (k <= N, k <= MAXK), ordered by value descending then index
// ascending (a stable sort's order), into sk / si [0, k).  A radix select on the key bits finds the k-th value, the entries
// above it and the first ones equal to it (in index order) are gathered, and a bitonic sort orders them.  P: the power of
// two >= k that sk / si hold.  blockDim.x == 256.
template <class Key>
__device__ void cta_topk(const Key& key, int N, int k, int P, unsigned long long* sk, int* si) {
  __shared__ int hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_need, s_base[2], s_wc[2][8];
  const int tid = threadIdx.x, lane = tid % 32, w = tid / 32;
  unsigned long long prefix = 0, mask = 0;
  int need = k;
  for (int pass = 7; pass >= 0; --pass) {
    hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < N; i += 256) {
      const unsigned long long b = (unsigned long long)__double_as_longlong(key(i));
      if ((b & mask) == prefix) atomicAdd(&hist[(int)((b >> (8 * pass)) & 255)], 1);
    }
    __syncthreads();
    if (tid == 0) {
      int cum = 0, bin = 255;
      for (; bin > 0; --bin) {
        if (cum + hist[bin] >= need) break;
        cum += hist[bin];
      }
      s_prefix = prefix | ((unsigned long long)bin << (8 * pass));
      s_need = need - cum;
    }
    __syncthreads();
    prefix = s_prefix; need = s_need;
    mask |= 255ull << (8 * pass);
  }
  // gather: keys above prefix, and the first `need` equal to it, by index order
  if (tid == 0) { s_base[0] = 0; s_base[1] = k - need; }
  __syncthreads();
  for (int i0 = 0; i0 < N; i0 += 256) {
    const int i = i0 + tid;
    unsigned long long b = 0;
    if (i < N) b = (unsigned long long)__double_as_longlong(key(i));
    const bool gt = i < N && b > prefix, eq = i < N && b == prefix;
    const unsigned bg = __ballot_sync(0xffffffffu, gt), be = __ballot_sync(0xffffffffu, eq);
    if (lane == 0) { s_wc[0][w] = __popc(bg); s_wc[1][w] = __popc(be); }
    __syncthreads();
    int og = s_base[0], oe = s_base[1];
    for (int x = 0; x < w; ++x) { og += s_wc[0][x]; oe += s_wc[1][x]; }
    og += __popc(bg & ((1u << lane) - 1)); oe += __popc(be & ((1u << lane) - 1));
    if (gt) { sk[og] = b; si[og] = i; }
    if (eq && oe < k) { sk[oe] = b; si[oe] = i; }
    __syncthreads();
    if (tid == 0) {
      for (int x = 0; x < 8; ++x) { s_base[0] += s_wc[0][x]; s_base[1] += s_wc[1][x]; }
    }
    __syncthreads();
  }
  for (int i = k + tid; i < P; i += 256) { sk[i] = 0; si[i] = 0x7fffffff; }
  __syncthreads();
  // bitonic sort: "a before b" when a's key is larger, or equal with the smaller index
  for (int size = 2; size <= P; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < P; i += 256) {
        const int j = i ^ stride;
        if (j > i) {
          const bool up = (i & size) == 0;
          const bool before = sk[j] > sk[i] || (sk[j] == sk[i] && si[j] < si[i]);   // j should precede i
          if (before == up) {
            const unsigned long long tk = sk[i]; sk[i] = sk[j]; sk[j] = tk;
            const int ti = si[i]; si[i] = si[j]; si[j] = ti;
          }
        }
      }
      __syncthreads();
    }
}

__host__ __device__ inline int pow2_at_least(int k) { int p = 1; while (p < k) p <<= 1; return p; }

// k_s2s_topk: one CTA per prefix row r of probabilities P [rows, V]: the k best tokens of p (times the candidate mask of
// its source row r / group when cand != NULL: cand [rows / group, C]), as (value f64, index) into val / idx [rows, k].
// Dynamic smem: P2 * 12 bytes + V / 8 bytes (the candidate bit set).
__global__ void __launch_bounds__(256) k_s2s_topk(const float* __restrict__ P, int V, const int32_t* __restrict__ cand, int C,
                                                  int group, int k, double* __restrict__ val, int32_t* __restrict__ idx) {
  extern __shared__ __align__(16) unsigned char smb[];
  const int P2 = pow2_at_least(k);
  unsigned long long* sk = reinterpret_cast<unsigned long long*>(smb);
  int* si = reinterpret_cast<int*>(sk + P2);
  unsigned* bits = reinterpret_cast<unsigned*>(si + P2);
  const int64_t r = blockIdx.x;
  const float* p = P + r * V;
  if (cand) {
    for (int i = threadIdx.x; i < (V + 31) / 32; i += 256) bits[i] = 0;
    __syncthreads();
    const int32_t* c = cand + (r / group) * C;
    for (int i = threadIdx.x; i < C; i += 256) {
      const int t = c[i];
      if (t >= 0 && t < V) atomicOr(&bits[t / 32], 1u << (t % 32));
    }
    __syncthreads();
  }
  auto key = [&](int i) -> double {
    return (!cand || (bits[i / 32] >> (i % 32)) & 1u) ? (double)p[i] : 0.0;
  };
  cta_topk(key, V, k, P2, sk, si);
  for (int i = threadIdx.x; i < k; i += 256) {
    val[r * k + i] = __longlong_as_double((long long)sk[i]);
    idx[r * k + i] = si[i];
  }
}

// k_s2s_beam: one CTA per source row b, step `pos` (the token written is path[.., pos]): the B = beam best of the beam^2
// products score[b, i] val[b beam + i, j], ties to the lower flat index i beam + j; then
// out_path[b, x, :] = path[b, i_x, :], out_path[b, x, pos] = idx[b beam + i_x, j_x], out_score[b, x] = the product.
// Paths are [n, beam, L] int32.  Dynamic smem: P2 * 12 bytes for P2 >= beam.
__global__ void __launch_bounds__(256) k_s2s_beam(const double* __restrict__ score, const double* __restrict__ val,
                                                  const int32_t* __restrict__ idx, const int32_t* __restrict__ path, int beam,
                                                  int L, int pos, int32_t* __restrict__ out_path, double* __restrict__ out_score) {
  extern __shared__ __align__(16) unsigned char smb[];
  const int P2 = pow2_at_least(beam);
  unsigned long long* sk = reinterpret_cast<unsigned long long*>(smb);
  int* si = reinterpret_cast<int*>(sk + P2);
  const int64_t b = blockIdx.x;
  const double* sc = score + b * beam;
  const double* vv = val + b * beam * beam;
  auto key = [&](int f) -> double { return sc[f / beam] * vv[f]; };
  cta_topk(key, beam * beam, beam, P2, sk, si);
  for (int e = threadIdx.x; e < beam * L; e += 256) {
    const int x = e / L, t = e % L, f = si[x], i = f / beam;
    out_path[(b * beam + x) * L + t] = t == pos ? idx[b * beam * beam + f] : path[(b * beam + i) * L + t];
  }
  for (int x = threadIdx.x; x < beam; x += 256) out_score[b * beam + x] = __longlong_as_double((long long)sk[x]);
}

// k_s2s_start: every path [n * beam, L] = START (1), then zeros
__global__ void k_s2s_start(int64_t rows, int L, int32_t* __restrict__ path) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < rows * L) path[e] = e % L == 0 ? 1 : 0;
}

// k_s2s_first: step 0 of a search: path[b, x, 1] = idx[b, x]; score[b, x] = val[b, x]
__global__ void k_s2s_first(const double* __restrict__ val, const int32_t* __restrict__ idx, int64_t rows, int L,
                            int32_t* __restrict__ path, double* __restrict__ score) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= rows) return;
  path[e * L + 1] = idx[e];
  score[e] = val[e];
}

// k_s2s_gather: the rows idx[0..n) of the token arrays e [., Ts], d and y [., Tt] into eo, do_, yo (a minibatch)
__global__ void k_s2s_gather(const int32_t* __restrict__ e, int Ts, const int32_t* __restrict__ d,
                             const int32_t* __restrict__ y, int Tt, const int64_t* __restrict__ idx, int n,
                             int32_t* __restrict__ eo, int32_t* __restrict__ do_, int32_t* __restrict__ yo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int W = Ts + 2 * Tt;
  if (i >= (int64_t)n * W) return;
  const int64_t r = i / W, src = idx[r];
  const int c = (int)(i % W);
  if (c < Ts) eo[r * Ts + c] = e[src * Ts + c];
  else if (c < Ts + Tt) do_[r * Tt + c - Ts] = d[src * Tt + c - Ts];
  else yo[r * Tt + c - Ts - Tt] = y[src * Tt + c - Ts - Tt];
}

// k_s2s_pick: out[r, i] = P[r T + i, path[r L + i + 1]] for i < T (the probability each path gives its own next token)
__global__ void k_s2s_pick(const float* __restrict__ P, int V, const int32_t* __restrict__ path, int L, int rows, int T,
                           float* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)rows * T) return;
  const int64_t r = e / T;
  const int i = (int)(e % T);
  out[e] = P[e * V + clamp_tok(path[r * L + i + 1], V)];
}

}  // namespace r4s2s
