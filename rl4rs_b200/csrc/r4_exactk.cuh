// r4_exactk.cuh -- Exact-K (nets/exact_k/model.py): the transformer-encoder / pointer-network slate generator and its
// reward critic, forward, backward and the draws they make.  fp32 CUDA cores (parity with a float64 autograd reference is
// the bar), deterministic: every output element has one writer that sums in a fixed order.
//
// Generator, for n rows of user features [256] over the candidates 0..T-1 (D = 128 = 2 * hidden_units):
//   encoder  X0 = dropout([relu(user W_u + b_u) tiled over T | emb[0..T-1] * 8]), then two blocks of
//            Y1 = LN(X + dropout(mask(softmax(mask(QK^T / sqrt(32))))) V),  Q|K|V = relu(X W_qkv + b_qkv), 4 heads of 32;
//            Y2 = LN(Y1 + relu(Y1 W_1 + b_1) W_2 + b_2)
//   decoder  nine steps of an LSTM (128), the intra-attention over its earlier outputs, one glimpse and the pointer
//            attention over the encoder outputs, the point mask, and the SAMPLE / GREEDY / TRAIN choice of the next index
// Kernels (host sequence in r4_learn.cu):
//   r4dense::k_dense_gemm  C = epilogue(alpha A B [+ C] [+ bias]) over strided, two-level batched operands; split-K
//                    partials
//   k_ek_colsum      out (+)= sum over rows of a strided plane (bias, LayerNorm and split-K reductions), rows in order
//   k_ek_input       X0 and its dropout; k_ek_rowmask the key / query masks sign(|sum_c X|)
//   k_ek_softmax     the masked attention softmax and its dropout; k_ek_softmax_bwd its backward
//   k_ek_ln / _bwd   residual add + LayerNorm (eps 1e-8) and its backward
//   k_ek_cell / _bwd the LSTM cell (gates i, j, f, o; forget bias 1)
//   k_ek_intra / _bwd, k_ek_glimpse / _bwd, k_ek_point / _bwd   the decoder attentions, one CTA per row
//   k_ek_loss_bwd    d(logits) of the policy loss; k_ek_gloss the loss; k_ek_closs the critic's summed squared error
//   k_ek_cell_bwd, k_ek_input_bwd, k_ek_relu_bwd, k_ek_emb_bwd   the element-wise backward pieces
// Adam is r4dense::k_keras_adam (TF1 AdamOptimizer and Keras Adam are the same ResourceApplyAdam update).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace r4ek {

constexpr int D = 128;             // 2 * hidden_units: encoder width, LSTM and attention size
constexpr int HU = 64;             // hidden_units
constexpr int UIN = 256;           // user feature width
constexpr int NH = 4, DH = 32;     // heads, head width
constexpr int FF = 256;            // feed-forward inner width
constexpr int VOCAB = 500;         // item embedding rows
constexpr int RES = 9;             // res_length: slate positions
constexpr int NBLK = 2;            // encoder blocks
constexpr int TMIN = 9, TMAX = 500;
constexpr int MAXN = 4096;
constexpr float NEG = -4294967295.0f;        // -2^32 + 1 (rounds to -2^32 in fp32, as in the reference graph)

// ---- parameter layouts (floats), in the order include/rl4rs_b200.h documents ----
struct Block { int64_t qkv_w, qkv_b, ln1_b, ln1_g, f1_w, f1_b, f2_w, f2_b, ln2_b, ln2_g; };
struct Att { int64_t w_q, w_dec, v, bias, w_ref; };
struct Layout {
  int64_t u_w, u_b, emb;
  Block blk[NBLK];
  int64_t lstm_w, lstm_b, c0, x0, h0;          // x0 | h0 adjacent: the first LSTM input row
  int64_t w_b, v_dec, w_bef, bias_dec;
  Att att[2];                       // 0: glimpse_0, 1: attention (the pointer)
  int64_t n;
};
__host__ __device__ inline Layout make_layout() {
  Layout L;
  int64_t o = 0;
  auto take = [&](int64_t k) { int64_t r = o; o += k; return r; };
  L.u_w = take(UIN * HU); L.u_b = take(HU); L.emb = take(VOCAB * HU);
  for (int l = 0; l < NBLK; ++l) {
    Block& b = L.blk[l];
    b.qkv_w = take(D * 3 * D); b.qkv_b = take(3 * D); b.ln1_b = take(D); b.ln1_g = take(D);
    b.f1_w = take(D * FF); b.f1_b = take(FF); b.f2_w = take(FF * D); b.f2_b = take(D); b.ln2_b = take(D); b.ln2_g = take(D);
  }
  L.lstm_w = take(2 * D * 4 * D); L.lstm_b = take(4 * D); L.c0 = take(D); L.x0 = take(D); L.h0 = take(D);
  L.w_b = take(D * D); L.v_dec = take(D); L.w_bef = take(D * D); L.bias_dec = take(D);
  for (int a = 0; a < 2; ++a) {
    Att& t = L.att[a];
    t.w_q = take(D * D); t.w_dec = take(D * D); t.v = take(D); t.bias = take(D); t.w_ref = take(D * D);
  }
  L.n = o;
  return L;
}
// critic: 256 -> 128 -> 128 -> 128 (relu) -> 1
constexpr int CH = 128;
struct CLayout { int64_t w[4], b[4], n; };
__host__ __device__ inline CLayout make_clayout() {
  CLayout L;
  const int in[4] = {UIN, CH, CH, CH}, out[4] = {CH, CH, CH, 1};
  int64_t o = 0;
  for (int i = 0; i < 4; ++i) { L.w[i] = o; o += (int64_t)in[i] * out[i]; L.b[i] = o; o += out[i]; }
  L.n = o;
  return L;
}

// ---- draws: U[0,1) from the top 24 bits of a counter-based hash keyed by (seed, call, stream, element) ----
enum Stream { ST_INPUT = 0, ST_ATT0 = 1, ST_ATT1 = 2, ST_SAMPLE = 3 };
__host__ __device__ inline uint64_t mix64(uint64_t x) {      // splitmix64's finaliser, as r4ppo::splitmix64
  x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull; return x ^ (x >> 31);
}
__host__ __device__ inline uint32_t draw24(uint64_t seed, uint64_t call, int stream, uint64_t elem) {
  return (uint32_t)(mix64(seed ^ mix64(mix64(call * 8u + (uint64_t)stream) + elem)) >> 40);
}
// dropout keep of one element: kept when U >= rate (TF's floor(keep_prob + U) == 1)
__device__ __forceinline__ bool kept(uint64_t seed, uint64_t call, int stream, uint64_t elem, float rate) {
  return rate <= 0.f || (float)draw24(seed, call, stream, elem) * (1.0f / 16777216.0f) >= rate;
}

// k_ek_colsum: out[i] (+)= scale sum_{r < R} in[r rs + (i / w) ls + i % w], rows in order, for i < N.  blockIdx.y = chunk of
// rows [y rc, (y + 1) rc); chunk y writes out + y ostride (one chunk: the final sum).
__global__ void k_ek_colsum(const float* __restrict__ in, int64_t R, int64_t rs, int w, int64_t ls, int N, int64_t rc,
                            float* __restrict__ out, int64_t ostride, float scale, int accumulate) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int64_t r0 = (int64_t)blockIdx.y * rc, r1 = min(R, r0 + rc);
  const float* p = in + (int64_t)(i / w) * ls + i % w;
  float s = 0.f;
  for (int64_t r = r0; r < r1; ++r) s += p[r * rs];
  float* o = out + (int64_t)blockIdx.y * ostride + i;
  *o = (accumulate ? *o : 0.f) + scale * s;
}

// k_ek_input: X0[b, t, c] = dropout(c < 64 ? uenc[b, c] : emb[t, c - 64] * 8), one thread per element
__global__ void k_ek_input(const float* __restrict__ uenc, const float* __restrict__ emb, int n, int T, uint64_t seed,
                           uint64_t call, float rate, float* __restrict__ X) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)n * T * D) return;
  const int c = (int)(e % D);
  const int64_t bt = e / D;
  const int t = (int)(bt % T), b = (int)(bt / T);
  float x = c < HU ? uenc[(int64_t)b * HU + c] : emb[(int64_t)t * HU + c - HU] * 8.0f;
  X[e] = kept(seed, call, ST_INPUT, (uint64_t)e, rate) ? x * (1.0f / (1.0f - rate)) : 0.f;
}

// k_ek_emb_bwd: from dX0 [n, T, D]: dU[b, c] = sum_t dX0'[b, t, c] (c < 64) with dX0' the dropout backward, and the
// embedding rows' gradient demb[t, c] = 8 sum_b dX0'[b, t, 64 + c].  One thread per output, rows in order.
__global__ void k_ek_emb_bwd(const float* __restrict__ dX, int n, int T, uint64_t seed, uint64_t call, float rate,
                             float* __restrict__ dU, float* __restrict__ demb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const float ks = 1.0f / (1.0f - rate);
  if (i < n * HU) {
    const int b = i / HU, c = i % HU;
    float s = 0.f;
    for (int t = 0; t < T; ++t) {
      const int64_t e = ((int64_t)b * T + t) * D + c;
      if (kept(seed, call, ST_INPUT, (uint64_t)e, rate)) s += dX[e] * ks;
    }
    dU[i] = s;
  } else if (i < n * HU + T * HU) {
    const int j = i - n * HU, t = j / HU, c = j % HU;
    float s = 0.f;
    for (int b = 0; b < n; ++b) {
      const int64_t e = ((int64_t)b * T + t) * D + HU + c;
      if (kept(seed, call, ST_INPUT, (uint64_t)e, rate)) s += dX[e] * ks;
    }
    demb[(int64_t)t * HU + c] = 8.0f * s;
  }
}

// k_ek_rowmask: m[r] = sign(|sum_c X[r, c]|), one warp per row of D
__global__ void k_ek_rowmask(const float* __restrict__ X, int64_t R, float* __restrict__ m) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (r >= R) return;
  float s = 0.f;
  for (int c = lane; c < D; c += 32) s += X[r * D + c];
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) m[r] = s != 0.f ? 1.f : 0.f;
}

// k_ek_softmax: one warp per score row (b, h, i) of S [n, 4, T, T]: key-masked softmax -> A; P = A * qmask[b, i] * dropout
__global__ void k_ek_softmax(const float* __restrict__ S, const float* __restrict__ mask, int n, int T, uint64_t seed,
                             uint64_t call, int stream, float rate, float* __restrict__ A, float* __restrict__ P) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (row >= (int64_t)n * NH * T) return;
  const int i = (int)(row % T);
  const int b = (int)(row / ((int64_t)NH * T));
  const float* s = S + row * T;
  const float* km = mask + (int64_t)b * T;
  float mx = -INFINITY;
  for (int j = lane; j < T; j += 32) mx = fmaxf(mx, km[j] != 0.f ? s[j] : NEG);
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float den = 0.f;
  for (int j = lane; j < T; j += 32) den += expf((km[j] != 0.f ? s[j] : NEG) - mx);
  for (int o = 16; o; o >>= 1) den += __shfl_xor_sync(0xffffffffu, den, o);
  const float qm = km[i], ks = 1.0f / (1.0f - rate);
  for (int j = lane; j < T; j += 32) {
    const float a = expf((km[j] != 0.f ? s[j] : NEG) - mx) / den;
    A[row * T + j] = a;
    P[row * T + j] = kept(seed, call, stream, (uint64_t)(row * T + j), rate) ? a * qm * ks : 0.f;
  }
}

// k_ek_softmax_bwd: dS = A (dA - sum A dA) on unmasked keys, 0 on masked ones; dA = dP * qmask * dropout.  In place on dP.
__global__ void k_ek_softmax_bwd(const float* __restrict__ A, const float* __restrict__ mask, int n, int T, uint64_t seed,
                                 uint64_t call, int stream, float rate, float* __restrict__ dP) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (row >= (int64_t)n * NH * T) return;
  const int i = (int)(row % T);
  const int b = (int)(row / ((int64_t)NH * T));
  const float* km = mask + (int64_t)b * T;
  const float sc = km[i] / (1.0f - rate);
  float dot = 0.f;
  for (int j = lane; j < T; j += 32) {
    const float da = kept(seed, call, stream, (uint64_t)(row * T + j), rate) ? dP[row * T + j] * sc : 0.f;
    dot += A[row * T + j] * da;
  }
  for (int o = 16; o; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  for (int j = lane; j < T; j += 32) {
    const float da = kept(seed, call, stream, (uint64_t)(row * T + j), rate) ? dP[row * T + j] * sc : 0.f;
    dP[row * T + j] = km[j] != 0.f ? A[row * T + j] * (da - dot) : 0.f;
  }
}

// k_ek_ln: Y = gamma xhat + beta, xhat = (Z - mean) / sqrt(var + 1e-8), Z = X + R; one warp per row of D.  Stores xhat, rstd.
__global__ void k_ek_ln(const float* __restrict__ X, const float* __restrict__ Rz, int64_t R, const float* __restrict__ beta,
                        const float* __restrict__ gamma, float* __restrict__ Y, float* __restrict__ xh, float* __restrict__ rs) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (r >= R) return;
  float z[D / 32], s = 0.f;
#pragma unroll
  for (int k = 0; k < D / 32; ++k) { z[k] = X[r * D + lane + 32 * k] + Rz[r * D + lane + 32 * k]; s += z[k]; }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / D;
  float v = 0.f;
#pragma unroll
  for (int k = 0; k < D / 32; ++k) { z[k] -= mean; v += z[k] * z[k]; }
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const float rstd = 1.0f / sqrtf(v / D + 1e-8f);
#pragma unroll
  for (int k = 0; k < D / 32; ++k) {
    const int c = lane + 32 * k;
    const float x = z[k] * rstd;
    xh[r * D + c] = x;
    Y[r * D + c] = gamma[c] * x + beta[c];
  }
  if (lane == 0) rs[r] = rstd;
}

// k_ek_ln_bwd: dZ = rstd (g - mean(g) - xhat mean(g xhat)), g = dY gamma; gx = dY xhat (for gamma's gradient).  In place on dY.
__global__ void k_ek_ln_bwd(const float* __restrict__ xh, const float* __restrict__ rs, int64_t R,
                            const float* __restrict__ gamma, float* __restrict__ dY, float* __restrict__ gx) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (r >= R) return;
  float g[D / 32], x[D / 32], s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int k = 0; k < D / 32; ++k) {
    const int c = lane + 32 * k;
    const float dy = dY[r * D + c];
    x[k] = xh[r * D + c];
    gx[r * D + c] = dy * x[k];
    g[k] = dy * gamma[c];
    s1 += g[k]; s2 += g[k] * x[k];
  }
  for (int o = 16; o; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
  const float rstd = rs[r];
#pragma unroll
  for (int k = 0; k < D / 32; ++k) dY[r * D + lane + 32 * k] = rstd * (g[k] - s1 / D - x[k] * (s2 / D));
}

// k_ek_relu_bwd: dY *= (Y > 0) over a plane of rows of width w at row stride ys / ds
__global__ void k_ek_relu_bwd(const float* __restrict__ Y, int64_t ys, float* __restrict__ dY, int64_t ds, int64_t R, int w) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= R * w) return;
  const int64_t r = e / w;
  const int c = (int)(e % w);
  if (!(Y[r * ys + c] > 0.f)) dY[r * ds + c] = 0.f;
}

// ---- decoder ----
// Per step t the scratch holds, for each row b: XH[t] = [x_t | h_{t-1}] (the LSTM input), G[t] = the activated gates
// (sig(i), tanh(j), sig(f + 1), sig(o)), C[t], H[t], the intra-attention output IN[t] and weights PI[t], HB[t] = h_t W_bef,
// QB[t] = h_t W_b, the glimpse and pointer query vectors A1[t], A2[t] (before their bias), the glimpse weights P1[t] and
// output GL[t].  logits [n, 9, T]; path [n, 9].
struct Dec {
  int n, T;
  const float* enc;                      // [n, T, D]
  const float* eref[2];                  // enc W_ref of the glimpse and the pointer, [n, T, D]
  float *XH, *G, *C, *H, *IN, *PI, *HB, *QB, *A1, *A2, *P1, *GL;
  float* logits;
  int32_t* path;
  const uint8_t* masks;                  // [4][T]: location masks of positions 0-2, 3-5, 6-8, and the special items
};
__host__ __device__ inline int64_t plane(int n, int t, int w) { return (int64_t)t * n * w; }

// the point mask of step t at candidate j, given the row's earlier choices
__device__ inline bool point_ok(const uint8_t* masks, int T, const int32_t* prev, int t, int j) {
  if (!masks[(t / 3) * T + j]) return false;
  if (t == 0) return true;
  const bool sp = masks[3 * T + j] != 0;
  for (int k = 0; k < t; ++k) {
    if (prev[k] == j) return false;
    if (sp && masks[3 * T + prev[k]]) return false;
  }
  return true;
}

// k_ek_cell: the LSTM cell of step t, one thread per (b, d); gates pre-activations in G[t] on entry.
// c = sig(f + 1) c_prev + sig(i) tanh(j); h = sig(o) tanh(c).  h goes to H[t] and XH[t + 1][:, D:].
__global__ void k_ek_cell(Dec d, int t, const float* __restrict__ c0) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= d.n * D) return;
  const int b = e / D, k = e % D;
  float* g = d.G + plane(d.n, t, 4 * D) + (int64_t)b * 4 * D;
  const float gi = 1.f / (1.f + expf(-g[k])), gj = tanhf(g[D + k]), gf = 1.f / (1.f + expf(-(g[2 * D + k] + 1.0f))),
              go = 1.f / (1.f + expf(-g[3 * D + k]));
  const float cp = t == 0 ? c0[k] : d.C[plane(d.n, t - 1, D) + e];
  const float c = gf * cp + gi * gj;
  const float h = go * tanhf(c);
  g[k] = gi; g[D + k] = gj; g[2 * D + k] = gf; g[3 * D + k] = go;
  d.C[plane(d.n, t, D) + e] = c;
  d.H[plane(d.n, t, D) + e] = h;
  if (t + 1 < RES) d.XH[plane(d.n, t + 1, 2 * D) + (int64_t)b * 2 * D + D + k] = h;
}

// k_ek_intra: the intra-attention of step t >= 2 over h_0..h_{t-1}: s_k = v_dec . tanh(HB[k] + QB[t] + bias_dec),
// IN[t] = sum_k softmax(s)_k h_k.  One CTA of 128 threads (one per d) per row.  t == 1: IN = h_0; t == 0: zeros.
__global__ void __launch_bounds__(D) k_ek_intra(Dec d, int t, const float* __restrict__ prm, Layout L) {
  const int b = blockIdx.x, k = threadIdx.x;
  __shared__ float red[D / 32][RES], p[RES];
  float* out = d.IN + plane(d.n, t, D) + (int64_t)b * D;
  if (t == 0) { out[k] = 0.f; return; }
  if (t == 1) { out[k] = d.H[(int64_t)b * D + k]; return; }
  const float q = d.QB[plane(d.n, t, D) + (int64_t)b * D + k] + prm[L.bias_dec + k], v = prm[L.v_dec + k];
  for (int j = 0; j < t; ++j) {
    float s = v * tanhf(d.HB[plane(d.n, j, D) + (int64_t)b * D + k] + q);
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (k % 32 == 0) red[k / 32][j] = s;
  }
  __syncthreads();
  if (k == 0) {
    float mx = -INFINITY, sc[RES];
    for (int j = 0; j < t; ++j) { sc[j] = red[0][j] + red[1][j] + red[2][j] + red[3][j]; mx = fmaxf(mx, sc[j]); }
    float den = 0.f;
    for (int j = 0; j < t; ++j) { sc[j] = expf(sc[j] - mx); den += sc[j]; }
    for (int j = 0; j < t; ++j) p[j] = sc[j] / den;
  }
  __syncthreads();
  float acc = 0.f;
  for (int j = 0; j < t; ++j) acc += p[j] * d.H[plane(d.n, j, D) + (int64_t)b * D + k];
  out[k] = acc;
  if (k < t) d.PI[plane(d.n, t, RES) + (int64_t)b * RES + k] = p[k];
}

// scores s_j = v . tanh(eref[b, j] + a), one warp per candidate j, 8 warps per CTA; a = query vector + bias in smem
constexpr int RNT = 256;
__device__ inline void att_scores(const float* __restrict__ eref, const float* a, const float* __restrict__ v, int T,
                                  float* s) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  float vv[D / 32], aa[D / 32];
#pragma unroll
  for (int k = 0; k < D / 32; ++k) { vv[k] = v[lane + 32 * k]; aa[k] = a[lane + 32 * k]; }
  for (int j = warp; j < T; j += RNT / 32) {
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < D / 32; ++k) acc += vv[k] * tanhf(eref[(int64_t)j * D + lane + 32 * k] + aa[k]);
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) s[j] = acc;
  }
}

// k_ek_glimpse: p = softmax_j(v . tanh(eref0[b, j] + A1 + bias)), GL = sum_j p_j enc[b, j].  One CTA per row; smem T floats.
__global__ void __launch_bounds__(RNT) k_ek_glimpse(Dec d, int t, const float* __restrict__ prm, Layout L) {
  extern __shared__ float sm[];
  __shared__ float a[D], red[2];
  const int b = blockIdx.x, tid = threadIdx.x, T = d.T;
  if (tid < D) a[tid] = d.A1[plane(d.n, t, D) + (int64_t)b * D + tid] + prm[L.att[0].bias + tid];
  __syncthreads();
  att_scores(d.eref[0] + (int64_t)b * T * D, a, prm + L.att[0].v, T, sm);
  __syncthreads();
  if (tid == 0) {
    float mx = -INFINITY, den = 0.f;
    for (int j = 0; j < T; ++j) mx = fmaxf(mx, sm[j]);
    for (int j = 0; j < T; ++j) { sm[j] = expf(sm[j] - mx); den += sm[j]; }
    red[0] = den;
  }
  __syncthreads();
  float* p1 = d.P1 + plane(d.n, t, T) + (int64_t)b * T;
  for (int j = tid; j < T; j += RNT) { sm[j] /= red[0]; p1[j] = sm[j]; }
  __syncthreads();
  if (tid < D) {
    const float* e = d.enc + (int64_t)b * T * D + tid;
    float acc = 0.f;
    for (int j = 0; j < T; ++j) acc += sm[j] * e[(int64_t)j * D];
    d.GL[plane(d.n, t, D) + (int64_t)b * D + tid] = acc;
  }
}

// k_ek_point: logits = v . tanh(eref1[b, j] + A2 + bias), masked to NEG off the point mask; then the step's choice:
// mode 0 SAMPLE (inverse CDF of softmax(logits / temperature) on one draw of (seed, call, ST_SAMPLE, 9 b + t)),
// 1 GREEDY (first argmax), 2 TRAIN (path[b, t] given, clamped into [0, T)).  Writes logits[b, t], path[b, t] and
// x_{t+1} = enc[b, path[b, t]].
__global__ void __launch_bounds__(RNT) k_ek_point(Dec d, int t, int mode, float temperature, uint64_t seed, uint64_t call,
                                                  const float* __restrict__ prm, Layout L) {
  extern __shared__ float sm[];
  __shared__ float a[D];
  __shared__ int pick;
  const int b = blockIdx.x, tid = threadIdx.x, T = d.T;
  if (tid < D) a[tid] = d.A2[plane(d.n, t, D) + (int64_t)b * D + tid] + prm[L.att[1].bias + tid];
  __syncthreads();
  att_scores(d.eref[1] + (int64_t)b * T * D, a, prm + L.att[1].v, T, sm);
  __syncthreads();
  int32_t* path = d.path + (int64_t)b * RES;
  float* lg = d.logits + ((int64_t)b * RES + t) * T;
  for (int j = tid; j < T; j += RNT) {
    if (!point_ok(d.masks, T, path, t, j)) sm[j] = NEG;
    lg[j] = sm[j];
  }
  __syncthreads();
  if (tid == 0) {
    int c = 0;
    if (mode == 2) {
      c = min(max(path[t], 0), T - 1);                     // the teacher path, clamped into the candidates
    } else if (mode == 1) {
      float mx = sm[0];
      for (int j = 1; j < T; ++j) if (sm[j] > mx) { mx = sm[j]; c = j; }
    } else {
      float mx = -INFINITY, tot = 0.f;
      for (int j = 0; j < T; ++j) mx = fmaxf(mx, sm[j] / temperature);
      for (int j = 0; j < T; ++j) tot += expf(sm[j] / temperature - mx);
      const float u = ((float)draw24(seed, call, ST_SAMPLE, (uint64_t)b * RES + t) + 0.5f) * (1.0f / 16777216.0f) * tot;
      float run = 0.f;
      c = -1;
      int last = 0;
      for (int j = 0; j < T; ++j) {
        const float e = expf(sm[j] / temperature - mx);
        if (e > 0.f) last = j;
        run += e;
        if (c < 0 && e > 0.f && run >= u) c = j;
      }
      if (c < 0) c = last;                                   // u above the rounded total: the last candidate with mass
    }
    path[t] = c;
    pick = c;
  }
  __syncthreads();
  if (t + 1 < RES && tid < D)
    d.XH[plane(d.n, t + 1, 2 * D) + (int64_t)b * 2 * D + tid] = d.enc[((int64_t)b * T + pick) * D + tid];
}

// ---- decoder backward ----
// Per row b: the gradient planes dA (d of the query vector incl. bias) and the per-row sums of v's and bias's gradient,
// accumulated over the steps in the row's own slot (one writer), reduced over rows afterwards.
struct DecBack {
  float* dlog;            // [n, T] the step's d(logits)
  float* deref[2];        // [n, T, D] accumulated over steps
  float* denc;            // [n, T, D] accumulated (glimpse sums and next-input gathers)
  float *dA1, *dA2;       // [n, D] of the current step
  float* dGL;             // [n, D]
  float* dIN;             // [n, D]
  float* dH;              // [n, D] total dh_t
  float* dC;              // [n, D] dc_t (carried to t - 1)
  float* dHB;             // [9][n, D]: d(h_k W_bef) accumulated from later steps
  float* dQB;             // [n, D]
  float* dG;              // [9][n, 4D] gate pre-activation gradients
  float* dXH;             // [n, 2D]
  float* rv;              // per-row sums [n][RV_N][D] of v's and bias's gradients
};
enum { RV_V0 = 0, RV_B0, RV_V1, RV_B1, RV_VDEC, RV_BDEC, RV_N };

// k_ek_loss_bwd: d(logits) of step t for the policy loss mean_b(sum_t CE(logits[b, t], path[b, t]) reward[b]):
// (softmax - onehot) reward[b] / n on the point mask, 0 off it.  loss_rows[b] += CE (for the reported loss).
__global__ void __launch_bounds__(RNT) k_ek_loss_bwd(Dec d, DecBack g, int t, const float* __restrict__ reward,
                                                     float* __restrict__ ce) {
  const int b = blockIdx.x, tid = threadIdx.x, T = d.T;
  __shared__ float red[2];
  const float* lg = d.logits + ((int64_t)b * RES + t) * T;
  if (tid == 0) {
    float mx = -INFINITY, den = 0.f;
    for (int j = 0; j < T; ++j) mx = fmaxf(mx, lg[j]);
    for (int j = 0; j < T; ++j) den += expf(lg[j] - mx);
    red[0] = mx; red[1] = den;
    const float l = logf(den) + mx - lg[d.path[(int64_t)b * RES + t]];
    ce[b] = (t == RES - 1 ? 0.f : ce[b]) + l;
  }
  __syncthreads();
  const float sc = reward[b] / (float)d.n;
  const int tgt = d.path[(int64_t)b * RES + t];
  for (int j = tid; j < T; j += RNT) {
    const bool ok = point_ok(d.masks, T, d.path + (int64_t)b * RES, t, j);
    const float p = expf(lg[j] - red[0]) / red[1];
    g.dlog[(int64_t)b * T + j] = ok ? (p - (j == tgt ? 1.f : 0.f)) * sc : 0.f;
  }
}

// the backward of s_j = v . tanh(eref[j] + a) for given ds_j (in smem): deref[j] += ds_j v (1 - th^2); da = sum_j ...;
// rv_v += sum_j ds_j th.  Warp per j; the per-warp partials of da / rv_v are summed over warps in order.
__device__ inline void att_scores_bwd(const float* __restrict__ eref, float* __restrict__ deref, const float* a,
                                      const float* __restrict__ v, int T, const float* ds, float* da_out, float* dv_row,
                                      float* dbias_row, float (*part)[2][D]) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  float vv[D / 32], aa[D / 32], pa[D / 32] = {}, pv[D / 32] = {};
#pragma unroll
  for (int k = 0; k < D / 32; ++k) { vv[k] = v[lane + 32 * k]; aa[k] = a[lane + 32 * k]; }
  for (int j = warp; j < T; j += RNT / 32) {
    const float s = ds[j];
    if (s == 0.f) continue;
#pragma unroll
    for (int k = 0; k < D / 32; ++k) {
      const int64_t o = (int64_t)j * D + lane + 32 * k;
      const float th = tanhf(eref[o] + aa[k]);
      const float du = s * vv[k] * (1.f - th * th);
      deref[o] += du;
      pa[k] += du;
      pv[k] += s * th;
    }
  }
#pragma unroll
  for (int k = 0; k < D / 32; ++k) { part[warp][0][lane + 32 * k] = pa[k]; part[warp][1][lane + 32 * k] = pv[k]; }
  __syncthreads();
  if (threadIdx.x < D) {
    float sa = 0.f, sv = 0.f;
    for (int w = 0; w < RNT / 32; ++w) { sa += part[w][0][threadIdx.x]; sv += part[w][1][threadIdx.x]; }
    da_out[threadIdx.x] = sa;
    dv_row[threadIdx.x] += sv;
    dbias_row[threadIdx.x] += sa;
  }
  __syncthreads();
}

// k_ek_point_bwd: the pointer attention's backward at step t: dA2 (query-vector gradient), deref1 += ..., per-row v1 / bias1.
__global__ void __launch_bounds__(RNT) k_ek_point_bwd(Dec d, DecBack g, int t, const float* __restrict__ prm, Layout L) {
  extern __shared__ float sm[];
  __shared__ float a[D];
  __shared__ float part[RNT / 32][2][D];
  const int b = blockIdx.x, tid = threadIdx.x, T = d.T;
  if (tid < D) a[tid] = d.A2[plane(d.n, t, D) + (int64_t)b * D + tid] + prm[L.att[1].bias + tid];
  for (int j = tid; j < T; j += RNT) sm[j] = g.dlog[(int64_t)b * T + j];
  __syncthreads();
  float* rv = g.rv + (int64_t)b * RV_N * D;
  att_scores_bwd(d.eref[1] + (int64_t)b * T * D, g.deref[1] + (int64_t)b * T * D, a, prm + L.att[1].v, T, sm,
                 g.dA2 + (int64_t)b * D, rv + RV_V1 * D, rv + RV_B1 * D, part);
}

// k_ek_glimpse_bwd: given dGL (from dA2 W_q2^T): dp_j = dGL . enc[b, j], denc[b, j] += p_j dGL, ds = p (dp - p . dp), then
// the score backward into deref0, dA1 and the per-row v0 / bias0 sums.
__global__ void __launch_bounds__(RNT) k_ek_glimpse_bwd(Dec d, DecBack g, int t, const float* __restrict__ prm, Layout L) {
  extern __shared__ float sm[];
  __shared__ float a[D], dgl[D], red[RNT / 32];
  __shared__ float part[RNT / 32][2][D];
  const int b = blockIdx.x, tid = threadIdx.x, T = d.T, warp = tid / 32, lane = tid % 32;
  if (tid < D) {
    a[tid] = d.A1[plane(d.n, t, D) + (int64_t)b * D + tid] + prm[L.att[0].bias + tid];
    dgl[tid] = g.dGL[(int64_t)b * D + tid];
  }
  __syncthreads();
  const float* p1 = d.P1 + plane(d.n, t, T) + (int64_t)b * T;
  const float* e = d.enc + (int64_t)b * T * D;
  float* de = g.denc + (int64_t)b * T * D;
  float pd = 0.f;
  for (int j = warp; j < T; j += RNT / 32) {
    float s = 0.f;
    const float p = p1[j];
#pragma unroll
    for (int k = 0; k < D / 32; ++k) {
      const int c = lane + 32 * k;
      s += dgl[c] * e[(int64_t)j * D + c];
      de[(int64_t)j * D + c] += p * dgl[c];
    }
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) sm[j] = s;
    pd += p * s;
  }
  if (lane == 0) red[warp] = pd;
  __syncthreads();
  float dot = 0.f;
  for (int w = 0; w < RNT / 32; ++w) dot += red[w];
  for (int j = tid; j < T; j += RNT) sm[j] = p1[j] * (sm[j] - dot);
  __syncthreads();
  float* rv = g.rv + (int64_t)b * RV_N * D;
  att_scores_bwd(d.eref[0] + (int64_t)b * T * D, g.deref[0] + (int64_t)b * T * D, a, prm + L.att[0].v, T, sm,
                 g.dA1 + (int64_t)b * D, rv + RV_V0 * D, rv + RV_B0 * D, part);
}

// k_ek_intra_bwd: given dIN of step t: t == 1 -> dH[0] gets dIN (through dHB's slot 0 side plane dH0); t >= 2 -> the
// softmax-attention backward: dh_k += p_k dIN, dHB[k] += du_k, dQB = sum_k du_k, per-row v_dec / bias_dec sums.
// dHs [9][n, D] collects the direct dh_k contributions of later steps.
__global__ void __launch_bounds__(D) k_ek_intra_bwd(Dec d, DecBack g, int t, float* __restrict__ dHs,
                                                    const float* __restrict__ prm, Layout L) {
  const int b = blockIdx.x, k = threadIdx.x;
  __shared__ float red[D / 32][RES], ds[RES];
  const float din = g.dIN[(int64_t)b * D + k];
  float* rv = g.rv + (int64_t)b * RV_N * D;
  if (t == 0) return;
  if (t == 1) { dHs[(int64_t)b * D + k] += din; return; }
  const float* pi = d.PI + plane(d.n, t, RES) + (int64_t)b * RES;
  for (int j = 0; j < t; ++j) {
    float s = din * d.H[plane(d.n, j, D) + (int64_t)b * D + k];
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (k % 32 == 0) red[k / 32][j] = s;
    dHs[plane(d.n, j, D) + (int64_t)b * D + k] += pi[j] * din;
  }
  __syncthreads();
  if (k == 0) {
    float dp[RES], dot = 0.f;
    for (int j = 0; j < t; ++j) { dp[j] = red[0][j] + red[1][j] + red[2][j] + red[3][j]; dot += pi[j] * dp[j]; }
    for (int j = 0; j < t; ++j) ds[j] = pi[j] * (dp[j] - dot);
  }
  __syncthreads();
  const float q = d.QB[plane(d.n, t, D) + (int64_t)b * D + k] + prm[L.bias_dec + k], v = prm[L.v_dec + k];
  float dq = 0.f, dv = 0.f;
  for (int j = 0; j < t; ++j) {
    const float th = tanhf(d.HB[plane(d.n, j, D) + (int64_t)b * D + k] + q);
    const float du = ds[j] * v * (1.f - th * th);
    g.dHB[plane(d.n, j, D) + (int64_t)b * D + k] += du;
    dq += du;
    dv += ds[j] * th;
  }
  g.dQB[(int64_t)b * D + k] = dq;
  rv[RV_VDEC * D + k] += dv;
  rv[RV_BDEC * D + k] += dq;
}

// k_ek_cell_bwd: dh = dH (step t's terms) + dXH[t + 1][:, D:] (as the next step's h_prev), dc from step t + 1 -> the gate
// pre-activation gradients dG[t] and dc_{t-1} into dC (at t == 0: the initial c's per-row gradient).
__global__ void k_ek_cell_bwd(Dec d, DecBack g, int t, const float* __restrict__ c0, const float* __restrict__ dxh_next) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= d.n * D) return;
  const int b = e / D, k = e % D;
  const float* ga = d.G + plane(d.n, t, 4 * D) + (int64_t)b * 4 * D;
  const float gi = ga[k], gj = ga[D + k], gf = ga[2 * D + k], go = ga[3 * D + k];
  const float c = d.C[plane(d.n, t, D) + e], tc = tanhf(c);
  const float cp = t == 0 ? c0[k] : d.C[plane(d.n, t - 1, D) + e];
  const float dh = g.dH[e] + (dxh_next ? dxh_next[(int64_t)b * 2 * D + D + k] : 0.f);
  const float dc = (t == RES - 1 ? 0.f : g.dC[e]) + dh * go * (1.f - tc * tc);
  float* dg = g.dG + plane(d.n, t, 4 * D) + (int64_t)b * 4 * D;
  dg[k] = dc * gj * gi * (1.f - gi);
  dg[D + k] = dc * gi * (1.f - gj * gj);
  dg[2 * D + k] = dc * cp * gf * (1.f - gf);
  dg[3 * D + k] = dh * tc * go * (1.f - go);
  g.dC[e] = dc * gf;
}

// k_ek_input_bwd: dXH[t] = [dx_t | dh_{t-1}], t >= 1 -> dx_t into denc[b, path[b, t - 1]] (x_t is that encoder output)
__global__ void k_ek_input_bwd(Dec d, DecBack g, int t) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= d.n * D) return;
  const int b = e / D, k = e % D;
  g.denc[((int64_t)b * d.T + d.path[(int64_t)b * RES + t - 1]) * D + k] += g.dXH[(int64_t)b * 2 * D + k];
}

// ---- critic ----
// k_ek_closs: pred = Z[:, 0]; loss = sum_b (target - pred)^2 (one CTA, rows in order); dZ = -2 (target - pred)
__global__ void k_ek_closs(const float* __restrict__ Z, const float* __restrict__ target, int n, float* __restrict__ pred,
                           float* __restrict__ dZ, float* __restrict__ loss) {
  __shared__ float part[256];
  float s = 0.f;
  for (int b = threadIdx.x; b < n; b += 256) {
    const float p = Z[b];
    if (pred) pred[b] = p;
    if (target) {
      const float r = target[b] - p;
      s += r * r;
      dZ[b] = -2.f * r;
    }
  }
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0 && loss && target) {
    float t = 0.f;
    for (int i = 0; i < 256; ++i) t += part[i];
    *loss = t;
  }
}

// k_ek_gloss: loss = scale sum_b ce[b] reward[b] (one thread, rows in order)
__global__ void k_ek_gloss(const float* __restrict__ ce, const float* __restrict__ reward, int n, float scale,
                           float* __restrict__ loss) {
  float s = 0.f;
  for (int b = 0; b < n; ++b) s += ce[b] * reward[b];
  *loss = s * scale;
}

}  // namespace r4ek

// The MDP checker's seq2seq transformer draws its dropout with r4ek::kept.
#include "r4_seq2seq.cuh"
