// r4_simtrain.cuh -- training the DIEN user simulator (nets/dien.py:8-45 in training mode) on item samples: the forward
// with saved activations, the hand-derived backward (two BPTT recurrences per sequence and the DIN attention), the weight
// and embedding gradients, and Keras's Adam.  fp32 CUDA cores throughout (no tensor cores: parity with a float64 autograd
// reference is the bar), deterministic (every gradient element has one writer that sums in a fixed order).
//
// One gradient pass over n samples is a fixed sequence of launches over scratch planes of n rows (per sample) or
// R = 64 n rows (per sample and time step):
//   k_st_gather      per sample: the sample's cat / dense / seq features from the per-record store, the dropout keep scales,
//                    the category self-attention (softmax(E E^T) E, mean over the 21 slots | flatten E), the query q (mean of
//                    emb_seq over the last 10 cat ids) and the emb_seq rows of both sequences
//   k_st_gemm        C = epilogue(A B [+ bias]) for every batched dense product (towers, input projections, attention MLP,
//                    head, and their transposed products in the backward)
//   k_st_gru_fwd     GRU-1 (hidden 128) and the AUGRU (hidden 256) over 64 steps, 8 samples per CTA, the hidden state in
//                    shared memory and the recurrent weights streamed from L2; stores h_{t-1}, r, u, c~ and r h_{t-1}
//   k_st_gru_bwd     the same recurrences in reverse (BPTT), dh kept in shared memory; writes the pre-activation gradients
//                    of the gates and the candidate, and the AUGRU's d(score)
//   k_st_attin(_bwd) the DIN attention input [q, k, q - k, q k] and its backward (dq summed over t, dk into dH)
//   k_st_loss        softmax output, Keras binary_crossentropy on one_hot(label, 2) with the clip, dlogits, the batch
//                    statistics and the AUC histograms (one CTA, samples summed in order)
//   k_st_loss_slate  the slate-label heads (nets/dien_slate.py, dien_slate_multiclass.py): 9 sigmoid columns against the
//                    page's clicks, or a 22-way softmax against the click pattern's class; same one-CTA ordered sums
//   k_st_cat_bwd     the category self-attention backward
//   r4ddpg::k_ddpg_wgrad  every dW = X^T dZ and bias, one CTA per 64 x 64 tile walking the rows in order
//   k_st_embkeys + a stable CUB radix sort + k_st_embsum   the two embedding tables' gradients: (table, id) keys of every
//                    (sample, slot) sorted stably, each run summed in order into the dense gradient buffer
//   k_st_apply       Keras Adam over every parameter; clears the embedding gradient rows the step wrote
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/device/device_radix_sort.cuh>

#include "r4_ddpg.cuh"

namespace r4st {

constexpr int E = 128;           // emb_size
constexpr int NC = 21;           // category_feature_num
constexpr int ND = 432;          // dense_feature_num
constexpr int U = 128;           // hidden_units (dense tower)
constexpr int T = 64;            // maxlen
constexpr int HA = 2 * E;        // AUGRU hidden size
constexpr int A1 = 64, A2 = 16;  // attention MLP
constexpr int OBS = 256;
constexpr int FEAT = 2 * HA + U + E + NC * E;   // 3456: [augru0 | augru1 | dense tower | cat attention | flatten]
constexpr int F_DENSE = 2 * HA, F_CATT = F_DENSE + U, F_FLAT = F_CATT + E;
constexpr int NSLOT = NC + 2 * T + 10;          // embedding slots per sample: 21 emb_cat, 128 + 10 emb_seq
constexpr int MAXN = 4096;                      // samples per pass
constexpr int MAXH = 4000000;                   // category_hash_size
constexpr int NTH = 256;

// ---- the heads: the item head of nets/dien.py and the two slate-label heads ----
// A head sets the width C of simulator_reward ([OBS, C] + [C]) and whether a sample is (record idx / 9, item idx % 9) or the
// record idx itself (the slate samples of data_preprocess.py tfrecord_slate: cat slot 20 and dense 392..431 are padding).
enum { HEAD_ITEM = 0, HEAD_SLATE = 1, HEAD_SLATE_MULTICLASS = 2, NHEAD = 3 };
constexpr int NS = 9;            // slate columns: one per exposed item
constexpr int NMC = 22;          // click-pattern classes: sum_j y_j [1, 2, 4, 1, 2, 4, 1, 2, 4]_j in 0..21
__host__ __device__ constexpr int head_classes(int head) { return head == HEAD_SLATE ? NS : head == HEAD_SLATE_MULTICLASS ? NMC : 2; }

// ---- the flat parameter layout: tf_checkpoint.dien_layer_plan order ----
struct Seq {
  int64_t gwg, gbg, gwc, gbc;                 // GRU-1: wg [2E, 2E], bg [2E], wc [2E, E], bc [E]
  int64_t aw1, ab1, aw2, ab2, ak, ab;         // attention: w1 [4E, 64], b1, w2 [64, 16], b2, k [16, 1], b [1]
  int64_t uwg, ubg, uwc, ubc;                 // AUGRU: wg [3E, 4E], bg [4E], wc [3E, 2E], bc [2E]
};
struct Layout {
  int64_t H;
  int64_t emb_cat, dw1, db1, dw2, db2, emb_seq;
  Seq s[2];
  int64_t ow, ob, rw, rb, n;
};
__host__ __device__ inline Layout make_layout(int64_t H, int C = 2) {
  Layout L;
  int64_t o = 0;
  auto take = [&](int64_t k) { int64_t r = o; o += k; return r; };
  L.H = H;
  L.emb_cat = take(H * E);
  L.dw1 = take((int64_t)ND * U); L.db1 = take(U);
  L.dw2 = take((int64_t)U * U);  L.db2 = take(U);
  L.emb_seq = take(H * E);
  for (int i = 0; i < 2; ++i) {
    Seq& s = L.s[i];
    s.gwg = take(2 * E * 2 * E); s.gbg = take(2 * E); s.gwc = take(2 * E * E); s.gbc = take(E);
    s.aw1 = take(4 * E * A1); s.ab1 = take(A1); s.aw2 = take(A1 * A2); s.ab2 = take(A2); s.ak = take(A2); s.ab = take(1);
    s.uwg = take(3 * E * 4 * E); s.ubg = take(4 * E); s.uwc = take(3 * E * 2 * E); s.ubc = take(2 * E);
  }
  L.ow = take((int64_t)FEAT * OBS); L.ob = take(OBS);
  L.rw = take(OBS * C); L.rb = take(C);
  L.n = o;
  return L;
}

// ---- the per-record sample store (ItemSamples): item sample i is (record i / 9, exposed item i % 9), slate sample i is
// record i ----
struct Data {
  const int32_t* ucat;     // [N][10] portrait ids
  const float* udense;     // [N][32] portrait dense
  const int32_t* seqid;    // [N] sequence_id
  const int32_t* items;    // [N][9] exposed items
  const uint8_t* label;    // [N][9] user_feedback
  const float* ifeat;      // [N][360] the record's item features
  const int32_t* seq;      // [N][2][64] pre-padded user_seqfeature | earlier pages' items
};

// ---- scratch planes ----
struct SeqPlanes {                       // R = 64 n rows each
  float *X, *XG1, *XC1, *H1, *Hp1, *G1, *C1, *RH1;       // GRU-1 (XG1 / XC1 hold dG1 / dC1 in the backward)
  float *Ain, *At1, *At2, *S;                            // attention input, MLP activations, raw score
  float *XG2, *XC2, *Hp2, *G2, *C2, *RH2;                // AUGRU (XG2 / XC2 hold dG2 / dC2 in the backward)
  float *dS, *dH1, *dA2, *dA1, *dAin, *dX, *dq;          // dq [n][E]
};
struct Planes {
  int32_t* cat;                          // [n][21]
  float *dense, *keep /* [2][n][U] keep scales */, *T1, *T1d, *T2, *allf, *P, *q, *O, *Z, *dZ, *dO, *dAllf, *dT1, *dT2, *dEcat, *dqs, *stats;
  SeqPlanes sp[2];
  uint32_t *keys, *keys2;                // [n * NSLOT]
  int32_t *vals, *vals2;
  void* cub_tmp;
  size_t cub_bytes;
  size_t bytes;                          // the end of the radix sort's reserve: the scratch size the layout needs
};
__host__ inline size_t cub_reserve(int n) { return ((size_t)4 << 20) + (size_t)16 * n * NSLOT; }

// The planes are cut from the scratch in this order, each rounded up to 256 bytes, and the radix sort's reserve follows.
// With base = nullptr only the offsets are formed: scratch_bytes is the end of the same cuts, so the size a caller
// allocates and the layout a launch uses cannot disagree.  C is the head's width: the logits Z and dZ are [n][C].
__host__ inline Planes make_planes(void* base, int n, int C = 2) {
  Planes P;
  const uintptr_t b = reinterpret_cast<uintptr_t>(base);
  size_t o = 0;
  auto take = [&](size_t floats) { float* q = reinterpret_cast<float*>(b + o); o += ((floats * 4 + 255) / 256) * 256; return q; };
  const size_t R = (size_t)n * T;
  P.cat = reinterpret_cast<int32_t*>(take((size_t)n * NC));
  P.dense = take((size_t)n * ND); P.keep = take((size_t)n * 2 * U);
  P.T1 = take((size_t)n * U); P.T1d = take((size_t)n * U); P.T2 = take((size_t)n * U);
  P.allf = take((size_t)n * FEAT); P.P = take((size_t)n * NC * NC); P.q = take((size_t)n * E);
  P.O = take((size_t)n * OBS); P.Z = take((size_t)n * C); P.dZ = take((size_t)n * C); P.dO = take((size_t)n * OBS);
  P.dAllf = take((size_t)n * FEAT); P.dT1 = take((size_t)n * U); P.dT2 = take((size_t)n * U);
  P.dEcat = take((size_t)n * NC * E); P.dqs = take((size_t)n * E); P.stats = take((size_t)n * 2);
  for (int i = 0; i < 2; ++i) {
    SeqPlanes& s = P.sp[i];
    s.X = take(R * E); s.XG1 = take(R * 2 * E); s.XC1 = take(R * E); s.H1 = take(R * E); s.Hp1 = take(R * E);
    s.G1 = take(R * 2 * E); s.C1 = take(R * E); s.RH1 = take(R * E);
    s.Ain = take(R * 4 * E); s.At1 = take(R * A1); s.At2 = take(R * A2); s.S = take(R);
    s.XG2 = take(R * 4 * E); s.XC2 = take(R * 2 * E); s.Hp2 = take(R * HA); s.G2 = take(R * 2 * HA); s.C2 = take(R * HA);
    s.RH2 = take(R * HA);
    s.dS = take(R); s.dH1 = take(R * E); s.dA2 = take(R * A2); s.dA1 = take(R * A1); s.dAin = take(R * 4 * E);
    s.dX = take(R * E); s.dq = take((size_t)n * E);
  }
  P.keys = reinterpret_cast<uint32_t*>(take((size_t)n * NSLOT)); P.keys2 = reinterpret_cast<uint32_t*>(take((size_t)n * NSLOT));
  P.vals = reinterpret_cast<int32_t*>(take((size_t)n * NSLOT)); P.vals2 = reinterpret_cast<int32_t*>(take((size_t)n * NSLOT));
  P.cub_tmp = reinterpret_cast<void*>(b + o);
  P.cub_bytes = cub_reserve(n);
  P.bytes = o + P.cub_bytes;
  return P;
}
__host__ inline size_t scratch_bytes(int n, int C = 2) { return make_planes(nullptr, n, C).bytes; }

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float elu(float x) { return x > 0.f ? x : expm1f(x); }
__device__ __forceinline__ int clampid(int id, int64_t H) { return id < 0 ? 0 : (id >= H ? (int)(H - 1) : id); }

// the dropout draw of (seed, counter, sample, unit): U[0, 1) from the top 24 bits of a counter-based hash
__device__ __forceinline__ float drop_u(uint64_t seed, uint64_t counter, int s, int unit) {
  const uint64_t r = r4ppo::splitmix64(seed ^ r4ppo::splitmix64(r4ppo::splitmix64(counter) + (uint64_t)s * 256u + (uint64_t)unit));
  return (float)(r >> 40) * (1.0f / 16777216.0f);
}

// ------------------------------------------------------------------------------------------------
// k_st_gather: one CTA (128 threads) per sample s of the batch (sample index idx[s]).  slate: the sample is record idx[s],
// its cat slot 20 the pad id 0 and its dense features 392..431 zero (pad_sequences post-padding of tfrecord_slate's rows).
// keep: keep_in != NULL -> keep_in[s][256] (u8, 1 = kept); else the draw of (seed, counter, s, unit) >= rate.  The keep
// scale is 1 / (1 - rate) (inverted dropout); rate 0 keeps every unit at scale 1.  keep_out (may be NULL) receives the bits.
// ------------------------------------------------------------------------------------------------
struct GatherArgs {
  Layout L;
  Data D;
  const int64_t* idx;
  int n;
  uint64_t seed, counter;
  float rate;
  const uint8_t* keep_in;
  uint8_t* keep_out;
  int slate;
};
__global__ void __launch_bounds__(E) k_st_gather(GatherArgs g, const float* __restrict__ prm, Planes P) {
  __shared__ float Es[NC][E + 1];
  __shared__ float Ps[NC][NC];
  __shared__ int ids[NC];
  __shared__ float w[NC];
  const int s = blockIdx.x, c = threadIdx.x;
  const int64_t smp = g.idx[s], rec = g.slate ? smp : smp / 9;
  const int j = g.slate ? -1 : (int)(smp % 9);
  const Data& D = g.D;
  const Layout& L = g.L;
  if (c < NC) {
    int id = c < 10 ? D.ucat[rec * 10 + c] : c == 10 ? D.seqid[rec] : c < 20 ? D.items[rec * 9 + c - 11] : j < 0 ? 0 : D.items[rec * 9 + j];
    id = clampid(id, L.H);
    ids[c] = id;
    P.cat[(size_t)s * NC + c] = id;
  }
  for (int k = c; k < ND; k += E) {
    const float v = k < 32 ? D.udense[rec * 32 + k] : k < 392 ? D.ifeat[rec * 360 + k - 32] : j < 0 ? 0.f : D.ifeat[rec * 360 + j * 40 + k - 392];
    P.dense[(size_t)s * ND + k] = v;
  }
  for (int u = c; u < 2 * U; u += E) {
    bool kept;
    if (g.keep_in) kept = g.keep_in[(size_t)s * 2 * U + u] != 0;
    else kept = g.rate <= 0.f || drop_u(g.seed, g.counter, s, u) >= g.rate;
    if (g.keep_out) g.keep_out[(size_t)s * 2 * U + u] = kept ? 1 : 0;
    P.keep[((size_t)(u / U) * g.n + s) * U + u % U] = kept ? 1.f / (1.f - g.rate) : 0.f;   // [layer][n][U]
  }
  __syncthreads();
  float* allf = P.allf + (size_t)s * FEAT;
  for (int r = 0; r < NC; ++r) {
    const float v = __ldg(prm + L.emb_cat + (int64_t)ids[r] * E + c);
    Es[r][c] = v;
    allf[F_FLAT + r * E + c] = v;
  }
  __syncthreads();
  for (int p = c; p < NC * NC; p += E) {
    const int a = p / NC, b = p % NC;
    float acc = 0.f;
    for (int k = 0; k < E; ++k) acc = fmaf(Es[a][k], Es[b][k], acc);
    Ps[a][b] = acc;
  }
  __syncthreads();
  if (c < NC) {
    float m = -INFINITY;
    for (int b = 0; b < NC; ++b) m = fmaxf(m, Ps[c][b]);
    float z = 0.f;
    for (int b = 0; b < NC; ++b) { const float e = expf(Ps[c][b] - m); Ps[c][b] = e; z += e; }
    for (int b = 0; b < NC; ++b) Ps[c][b] /= z;
  }
  __syncthreads();
  if (c < NC) {
    float a = 0.f;
    for (int r = 0; r < NC; ++r) a += Ps[r][c];
    w[c] = a;
  }
  for (int p = c; p < NC * NC; p += E) P.P[(size_t)s * NC * NC + p] = Ps[p / NC][p % NC];
  __syncthreads();
  {
    float a = 0.f;
    for (int b = 0; b < NC; ++b) a = fmaf(w[b], Es[b][c], a);
    allf[F_CATT + c] = a / (float)NC;
    float q = 0.f;
    for (int r = NC - 10; r < NC; ++r) q += __ldg(prm + L.emb_seq + (int64_t)ids[r] * E + c);
    P.q[(size_t)s * E + c] = q / 10.f;
  }
  for (int i = 0; i < 2; ++i)
    for (int t = 0; t < T; ++t) {
      const int id = clampid(D.seq[(rec * 2 + i) * T + t], L.H);
      P.sp[i].X[((size_t)s * T + t) * E + c] = __ldg(prm + L.emb_seq + (int64_t)id * E + c);
    }
}

// ------------------------------------------------------------------------------------------------
// k_st_gemm: C[M][N] (ldc) = epi(sum_k A[m][k] B[k][n] (+ bias[n])), B = W[k][n] (ldb) or, TB, W[n][k] (ldb).
//   EP_LIN   v = acc + bias         EP_SIG  v = sigmoid(acc + bias)     EP_ELU  v = elu(acc + bias)
//   EP_DSIG  v = acc y (1 - y)      EP_DELU v = acc (y > 0 ? 1 : y + 1)   (y = aux[m][n], ld N: the forward activation)
// then pre (may be NULL, ld N) receives v, v *= mul[m][n] (may be NULL, ld N), and C = v or C += v (accum).
// 64 x 64 tiles, 16-deep k-slices, 4 x 4 outputs per thread, each output summed over k in order.
// ------------------------------------------------------------------------------------------------
enum { EP_LIN = 0, EP_SIG = 1, EP_ELU = 2, EP_DSIG = 3, EP_DELU = 4 };
struct Gemm {
  const float* A; int lda;
  const float* B; int ldb;
  const float* bias;
  float* C; int ldc;
  int M, N, K, epi, accum;
  const float* aux;
  const float* mul;
  float* pre;
};
constexpr int GT = 64, GK = 16;
template <bool TB>
__global__ void __launch_bounds__(NTH) k_st_gemm(Gemm g) {
  __shared__ float as[GK][GT + 4];
  __shared__ float bs[GK][GT + 4];
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  const int m0 = blockIdx.y * GT, n0 = blockIdx.x * GT;
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
  for (int k0 = 0; k0 < g.K; k0 += GK) {
    for (int e = tid; e < GK * GT; e += NTH) {
      const int r = e / GK, k = e % GK;           // A: rows m0 + r, k contiguous
      const int m = m0 + r, kk = k0 + k;
      as[k][r] = (m < g.M && kk < g.K) ? g.A[(size_t)m * g.lda + kk] : 0.f;
    }
    for (int e = tid; e < GK * GT; e += NTH) {
      int k, c;
      if (TB) { c = e / GK; k = e % GK; } else { k = e / GT; c = e % GT; }
      const int nn = n0 + c, kk = k0 + k;
      float v = 0.f;
      if (nn < g.N && kk < g.K) v = TB ? g.B[(size_t)nn * g.ldb + kk] : g.B[(size_t)kk * g.ldb + nn];
      bs[k][c] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GK; ++k) {
      float av[4], bv[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) { av[a] = as[k][ty + 16 * a]; bv[a] = bs[k][tx + 16 * a]; }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fmaf(av[a], bv[b], acc[a][b]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int m = m0 + ty + 16 * a;
    if (m >= g.M) continue;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int n = n0 + tx + 16 * b;
      if (n >= g.N) continue;
      const size_t o = (size_t)m * g.N + n;
      float v = acc[a][b];
      if (g.epi <= EP_ELU) {
        if (g.bias) v += g.bias[n];
        v = g.epi == EP_SIG ? sigm(v) : g.epi == EP_ELU ? elu(v) : v;
      } else {
        const float y = g.aux[o];
        v = g.epi == EP_DSIG ? v * (y * (1.f - y)) : v * (y > 0.f ? 1.f : y + 1.f);
      }
      if (g.pre) g.pre[o] = v;
      if (g.mul) v *= g.mul[o];
      float* cp = g.C + (size_t)m * g.ldc + n;
      *cp = g.accum ? *cp + v : v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// The recurrences.  HD = hidden size (GRU-1: E, AUGRU: 2E), input size E; wg [(E + HD)][2 HD] = [x rows | h rows],
// wc [(E + HD)][HD].  XG = x wg_x + bg and XC = x wc_x + bc come precomputed ([R][2 HD], [R][HD]).
//   g = sigmoid(XG_t + h wg_h), r = g[:HD], u = g[HD:], c = tanh(XC_t + (r h) wc_h),
//   u' = u (GRU-1) or (1 - score_t) u (AUGRU), h' = u' h + (1 - u') c.
// SB samples per CTA; h, r h and g in shared memory; the weights are read from global memory (L2-resident).
// ------------------------------------------------------------------------------------------------
constexpr int SB = 8;
template <int HD>
struct RecArgs {
  const float* wg_h; const float* wc_h;
  const float* XG; const float* XC; const float* S;     // S: scores [R] (AUGRU) or NULL
  float *Hp, *G, *C, *RH, *H;                           // H [R][HD] (GRU-1) or NULL
  float* hT; int ldT;                                   // final state (AUGRU: the allf columns) or NULL
  int n;
};
template <int HD>
__global__ void __launch_bounds__(NTH) k_st_gru_fwd(RecArgs<HD> a) {
  __shared__ float h[SB][HD];
  __shared__ float rh[SB][HD];
  __shared__ float gs[SB][2 * HD];
  const int tid = threadIdx.x, s0 = blockIdx.x * SB;
  const int nv = min(SB, a.n - s0);
  for (int i = tid; i < SB * HD; i += NTH) h[i / HD][i % HD] = 0.f;
  __syncthreads();
  for (int t = 0; t < T; ++t) {
    for (int j = tid; j < 2 * HD; j += NTH) {
      float acc[SB];
#pragma unroll
      for (int s = 0; s < SB; ++s) acc[s] = 0.f;
#pragma unroll 4
      for (int k = 0; k < HD; ++k) {
        const float w = __ldg(a.wg_h + (size_t)k * 2 * HD + j);
#pragma unroll
        for (int s = 0; s < SB; ++s) acc[s] = fmaf(h[s][k], w, acc[s]);
      }
#pragma unroll
      for (int s = 0; s < SB; ++s) {
        if (s >= nv) { gs[s][j] = 0.f; continue; }
        const size_t row = (size_t)(s0 + s) * T + t;
        const float v = sigm(a.XG[row * 2 * HD + j] + acc[s]);
        gs[s][j] = v;
        a.G[row * 2 * HD + j] = v;
      }
    }
    __syncthreads();
    for (int i = tid; i < SB * HD; i += NTH) {
      const int s = i / HD, k = i % HD;
      const float v = gs[s][k] * h[s][k];
      rh[s][k] = v;
      if (s < nv) {
        const size_t row = (size_t)(s0 + s) * T + t;
        a.RH[row * HD + k] = v;
        a.Hp[row * HD + k] = h[s][k];
      }
    }
    __syncthreads();
    for (int j = tid; j < HD; j += NTH) {
      float acc[SB];
#pragma unroll
      for (int s = 0; s < SB; ++s) acc[s] = 0.f;
#pragma unroll 4
      for (int k = 0; k < HD; ++k) {
        const float w = __ldg(a.wc_h + (size_t)k * HD + j);
#pragma unroll
        for (int s = 0; s < SB; ++s) acc[s] = fmaf(rh[s][k], w, acc[s]);
      }
#pragma unroll
      for (int s = 0; s < SB; ++s) {
        if (s >= nv) continue;
        const size_t row = (size_t)(s0 + s) * T + t;
        const float c = tanhf(a.XC[row * HD + j] + acc[s]);
        float u = gs[s][HD + j];
        if (a.S) u = (1.f - a.S[row]) * u;
        const float hn = u * h[s][j] + (1.f - u) * c;
        a.C[row * HD + j] = c;
        if (a.H) a.H[row * HD + j] = hn;
        h[s][j] = hn;                                    // only this thread reads h[s][j] in this phase
      }
    }
    __syncthreads();
  }
  if (a.hT)
    for (int i = tid; i < nv * HD; i += NTH) a.hT[(size_t)(s0 + i / HD) * a.ldT + i % HD] = h[i / HD][i % HD];
}

// BPTT of k_st_gru_fwd.  dh starts at dT (ld ldT; NULL: 0) and takes dext[row] (may be NULL) at every step; writes
// dG [R][2 HD] = d(gate pre-activations), dC [R][HD] = d(candidate pre-activation) and, AUGRU, dS [R] = d(score).
template <int HD>
struct RecBack {
  const float* wg_h; const float* wc_h;
  const float *Hp, *G, *C, *S, *dext, *dT;
  int ldT;
  float *dG, *dC, *dS;
  int n;
};
template <int HD>
__global__ void __launch_bounds__(NTH) k_st_gru_bwd(RecBack<HD> a) {
  __shared__ float dh[SB][HD];
  __shared__ float dgp[SB][2 * HD];
  __shared__ float dcp[SB][HD];
  __shared__ float red[SB][HD];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, s0 = blockIdx.x * SB;
  const int nv = min(SB, a.n - s0);
  for (int i = tid; i < SB * HD; i += NTH) {
    const int s = i / HD, k = i % HD;
    dh[s][k] = (a.dT && s < nv) ? a.dT[(size_t)(s0 + s) * a.ldT + k] : 0.f;
  }
  __syncthreads();
  for (int t = T - 1; t >= 0; --t) {
    // the cell output: dh -> d(u'), d(c), the carried dh u'
    for (int i = tid; i < SB * HD; i += NTH) {
      const int s = i / HD, k = i % HD;
      if (s >= nv) { dcp[s][k] = 0.f; dgp[s][HD + k] = 0.f; red[s][k] = 0.f; continue; }
      const size_t row = (size_t)(s0 + s) * T + t;
      float d = dh[s][k];
      if (a.dext) d += a.dext[row * HD + k];
      const float hp = a.Hp[row * HD + k], u = a.G[row * 2 * HD + HD + k], c = a.C[row * HD + k];
      const float sc = a.S ? a.S[row] : 0.f;
      const float up = a.S ? (1.f - sc) * u : u;
      const float dup = d * (hp - c);
      const float dc = d * (1.f - up) * (1.f - c * c);
      const float du = a.S ? dup * (1.f - sc) : dup;
      dcp[s][k] = dc;
      dgp[s][HD + k] = du * u * (1.f - u);
      red[s][k] = -dup * u;
      dh[s][k] = d * up;
      a.dC[row * HD + k] = dc;
    }
    __syncthreads();
    if (a.S && warp < SB && warp < nv) {                 // d(score) = -sum_k du'_k u_k, lanes then a fixed shuffle tree
      float v = 0.f;
      for (int k = lane; k < HD; k += 32) v += red[warp][k];
      v = r4ppo::warp_sum(v);
      if (lane == 0) a.dS[(size_t)(s0 + warp) * T + t] = v;
    }
    // d(r h) = dc~ wc_h^T: one warp per row k of wc_h
    for (int k = warp; k < HD; k += NTH / 32) {
      float p[SB];
#pragma unroll
      for (int s = 0; s < SB; ++s) p[s] = 0.f;
      for (int j = lane; j < HD; j += 32) {
        const float w = __ldg(a.wc_h + (size_t)k * HD + j);
#pragma unroll
        for (int s = 0; s < SB; ++s) p[s] = fmaf(dcp[s][j], w, p[s]);
      }
#pragma unroll
      for (int s = 0; s < SB; ++s) p[s] = r4ppo::warp_sum(p[s]);
      if (lane < SB && lane < nv) {
        float drh = 0.f;
#pragma unroll
        for (int s = 0; s < SB; ++s) if (s == lane) drh = p[s];
        const int s = lane;
        const size_t row = (size_t)(s0 + s) * T + t;
        const float hp = a.Hp[row * HD + k], r = a.G[row * 2 * HD + k];
        dgp[s][k] = drh * hp * r * (1.f - r);
        dh[s][k] += drh * r;
      } else if (lane < SB) {
        dgp[lane][k] = 0.f;
      }
    }
    __syncthreads();
    for (int i = tid; i < nv * 2 * HD; i += NTH) {
      const int s = i / (2 * HD), j = i % (2 * HD);
      a.dG[((size_t)(s0 + s) * T + t) * 2 * HD + j] = dgp[s][j];
    }
    // dh += d(gates) wg_h^T
    for (int k = warp; k < HD; k += NTH / 32) {
      float p[SB];
#pragma unroll
      for (int s = 0; s < SB; ++s) p[s] = 0.f;
      for (int j = lane; j < 2 * HD; j += 32) {
        const float w = __ldg(a.wg_h + (size_t)k * 2 * HD + j);
#pragma unroll
        for (int s = 0; s < SB; ++s) p[s] = fmaf(dgp[s][j], w, p[s]);
      }
#pragma unroll
      for (int s = 0; s < SB; ++s) p[s] = r4ppo::warp_sum(p[s]);
      if (lane < SB) {
        float v = 0.f;
#pragma unroll
        for (int s = 0; s < SB; ++s) if (s == lane) v = p[s];
        dh[lane][k] += v;
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// The DIN attention input Ain[row] = [q, k, q - k, q k] (k = H1[row]) and its backward: dH1[row] += dk, dq = sum over t.
// ------------------------------------------------------------------------------------------------
__global__ void k_st_attin(const float* __restrict__ q, const float* __restrict__ H1, float* __restrict__ Ain, int n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n * T * E) return;
  const size_t row = i / E;
  const int c = (int)(i % E);
  const float qv = q[(row / T) * E + c], kv = H1[i];
  float* o = Ain + row * 4 * E;
  o[c] = qv; o[E + c] = kv; o[2 * E + c] = qv - kv; o[3 * E + c] = qv * kv;
}
__global__ void __launch_bounds__(E) k_st_attin_bwd(const float* __restrict__ q, const float* __restrict__ H1,
                                                    const float* __restrict__ dAin, float* __restrict__ dH1, float* __restrict__ dq) {
  const int s = blockIdx.x, c = threadIdx.x;
  const float qv = q[(size_t)s * E + c];
  float acc = 0.f;
  for (int t = 0; t < T; ++t) {
    const size_t row = (size_t)s * T + t;
    const float* d = dAin + row * 4 * E;
    const float kv = H1[row * E + c];
    acc += d[c] + d[2 * E + c] + d[3 * E + c] * kv;
    dH1[row * E + c] += d[E + c] - d[2 * E + c] + d[3 * E + c] * qv;
  }
  dq[(size_t)s * E + c] = acc;
}

// ------------------------------------------------------------------------------------------------
// k_st_loss (one CTA): p = softmax(z); Keras binary_crossentropy against one_hot(label, 2) with p clipped to [eps, 1 - eps]
// (zero gradient where clipped), the mean over both columns and the batch; dz = p (dp - p . dp).  stats (may be NULL)
// receives {mean loss, mean binary accuracy}.  acc (may be NULL) f64[3 + 2 * 201] accumulates {loss sum, accuracy sum, count,
// positives histogram, negatives histogram} where bin b counts the predictions above exactly b of Keras's 200 AUC thresholds.
// probs (may be NULL) receives p.
// ------------------------------------------------------------------------------------------------
constexpr int NBIN = 201, NACC = 3 + 2 * NBIN;
constexpr float CLIP = 1e-7f;
__device__ inline int auc_bin(float p) {
  int b = 1;                                               // -1e-7 < p always; 1 + 1e-7 > p always
  int k = max(1, min(198, (int)(p * 199.f)));
  while (k > 1 && p <= (float)((double)k / 199.0)) --k;
  while (k <= 198 && p > (float)((double)k / 199.0)) ++k;   // k = the first threshold index with p <= t_k
  b += k - 1;
  return b;
}
__global__ void __launch_bounds__(NTH) k_st_loss(Data D, const int64_t* __restrict__ idx, int n, const float* __restrict__ Z,
                                                 float* __restrict__ dZ, float* __restrict__ srow, float* __restrict__ stats,
                                                 double* __restrict__ acc, float* __restrict__ probs) {
  __shared__ unsigned int hist[2][NBIN];
  const int tid = threadIdx.x;
  for (int i = tid; i < 2 * NBIN; i += NTH) hist[i / NBIN][i % NBIN] = 0u;
  __syncthreads();
  const float inv = 1.f / (2.f * (float)n);
  for (int s = tid; s < n; s += NTH) {
    const int64_t smp = idx[s];
    const int y = D.label[(smp / 9) * 9 + smp % 9] != 0 ? 1 : 0;
    const float z0 = Z[2 * s], z1 = Z[2 * s + 1], m = fmaxf(z0, z1);
    const float e0 = expf(z0 - m), e1 = expf(z1 - m), den = e0 + e1;
    const float p[2] = {e0 / den, e1 / den};
    // 1 - p[c] is p[1 - c]: taken from its own exponential, so a confident row keeps its relative precision
    float loss = 0.f, dp[2], hit = 0.f;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float yc = (c == y) ? 1.f : 0.f;
      const float q = p[1 - c];
      const bool clipped = p[c] < CLIP || q < CLIP;
      const float pc = fminf(fmaxf(p[c], CLIP), 1.f - CLIP), qc = fminf(fmaxf(q, CLIP), 1.f - CLIP);
      loss += -(yc * logf(pc) + (1.f - yc) * logf(qc));
      dp[c] = clipped ? 0.f : (c == y ? -q : p[c]) / (p[c] * q) * inv;
      hit += ((p[c] > 0.5f ? 1.f : 0.f) == yc) ? 1.f : 0.f;
      if (acc) atomicAdd(&hist[yc != 0.f ? 0 : 1][auc_bin(p[c])], 1u);
    }
    // the softmax backward p (dp - p . dp) of two columns: dz0 = p0 p1 (dp0 - dp1) = -dz1
    const float dz0 = p[0] * p[1] * (dp[0] - dp[1]);
    if (dZ) { dZ[2 * s] = dz0; dZ[2 * s + 1] = -dz0; }
    if (probs) { probs[2 * s] = p[0]; probs[2 * s + 1] = p[1]; }
    srow[2 * s] = 0.5f * loss;
    srow[2 * s + 1] = 0.5f * hit;
  }
  __syncthreads();
  if (tid == 0) {
    double l = 0.0, h = 0.0;
    for (int s = 0; s < n; ++s) { l += srow[2 * s]; h += srow[2 * s + 1]; }
    if (stats) { stats[0] = (float)(l / n); stats[1] = (float)(h / n); }
    if (acc) { acc[0] += l; acc[1] += h; acc[2] += n; }
  }
  if (acc)
    for (int i = tid; i < 2 * NBIN; i += NTH) acc[3 + i] += (double)hist[i / NBIN][i % NBIN];
}

// ------------------------------------------------------------------------------------------------
// k_st_loss_slate<C> (one CTA), sample s = record idx[s] with the page's clicks y[9]; Keras takes the logits path for a
// Sigmoid / Softmax output (no clip, INTEGRATION.md section 8).
//   C = 9:  p = sigmoid(z), loss = mean over the 9 columns and the batch of max(z, 0) - z y + log(1 + exp(-|z|)),
//           dz = (p - y) / (9 n).  acc (may be NULL) f64[NACC_SLATE] accumulates {loss sum, binary accuracy sum, samples,
//           positives[201], negatives[201] (the k_st_loss histograms over all 9 columns), TP, FP, FN at p > 0.5}.
//   C = 22: class = sum_j y_j [1, 2, 4, 1, 2, 4, 1, 2, 4]_j, p = softmax(z), loss = mean of logsumexp(z) - z_class,
//           dz = (p - one_hot(class)) / n.  acc f64[NACC_MC] accumulates {loss sum, hits, samples}: a hit is the first
//           argmax of p (tf.argmax) at the class.
// stats (may be NULL) f32[2] = {mean loss, mean binary accuracy | categorical accuracy}; probs (may be NULL) [n][C].
// ------------------------------------------------------------------------------------------------
constexpr int NACC_SLATE = NACC + 3, NACC_MC = 3;
template <int C>
__global__ void __launch_bounds__(NTH) k_st_loss_slate(Data D, const int64_t* __restrict__ idx, int n, const float* __restrict__ Z,
                                                       float* __restrict__ dZ, float* __restrict__ srow, float* __restrict__ stats,
                                                       double* __restrict__ acc, float* __restrict__ probs) {
  __shared__ unsigned int hist[2][NBIN];
  __shared__ unsigned int cnt[3];
  const int tid = threadIdx.x;
  for (int i = tid; i < 2 * NBIN; i += NTH) hist[i / NBIN][i % NBIN] = 0u;
  if (tid < 3) cnt[tid] = 0u;
  __syncthreads();
  const float inv = 1.f / ((float)n * (C == NS ? (float)NS : 1.f));
  for (int s = tid; s < n; s += NTH) {
    const uint8_t* y = D.label + idx[s] * 9;
    const float* z = Z + (size_t)s * C;
    if constexpr (C == NS) {
      float loss = 0.f, hit = 0.f;
#pragma unroll
      for (int j = 0; j < NS; ++j) {
        const bool yj = y[j] != 0;
        const float zj = z[j], e = expf(-fabsf(zj));
        const float p = zj >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
        loss += fmaxf(zj, 0.f) - (yj ? zj : 0.f) + log1pf(e);
        if (dZ) dZ[(size_t)s * C + j] = (p - (yj ? 1.f : 0.f)) * inv;
        if (probs) probs[(size_t)s * C + j] = p;
        const bool pos = p > 0.5f;
        hit += pos == yj ? 1.f : 0.f;
        if (acc) {
          atomicAdd(&hist[yj ? 0 : 1][auc_bin(p)], 1u);
          if (pos || yj) atomicAdd(&cnt[pos ? (yj ? 0 : 1) : 2], 1u);
        }
      }
      srow[2 * s] = loss / (float)NS;
      srow[2 * s + 1] = hit / (float)NS;
    } else {
      int cls = 0;
#pragma unroll
      for (int j = 0; j < NS; ++j) cls += y[j] != 0 ? 1 << (j % 3) : 0;
      float m = -INFINITY;
#pragma unroll
      for (int k = 0; k < C; ++k) m = fmaxf(m, z[k]);
      float e[C], den = 0.f;
#pragma unroll
      for (int k = 0; k < C; ++k) { e[k] = expf(z[k] - m); den += e[k]; }
      int am = 0;
      float best = -1.f;
#pragma unroll
      for (int k = 0; k < C; ++k) {
        const float p = e[k] / den;
        if (p > best) { best = p; am = k; }
        if (dZ) dZ[(size_t)s * C + k] = (p - (k == cls ? 1.f : 0.f)) * inv;
        if (probs) probs[(size_t)s * C + k] = p;
      }
      srow[2 * s] = m + logf(den) - z[cls];
      srow[2 * s + 1] = am == cls ? 1.f : 0.f;
    }
  }
  __syncthreads();
  if (tid == 0) {
    double l = 0.0, h = 0.0;
    for (int s = 0; s < n; ++s) { l += srow[2 * s]; h += srow[2 * s + 1]; }
    if (stats) { stats[0] = (float)(l / n); stats[1] = (float)(h / n); }
    if (acc) { acc[0] += l; acc[1] += h; acc[2] += n; }
  }
  if (acc && C == NS) {
    for (int i = tid; i < 2 * NBIN; i += NTH) acc[3 + i] += (double)hist[i / NBIN][i % NBIN];
    if (tid < 3) acc[NACC + tid] += (double)cnt[tid];
  }
}

// ------------------------------------------------------------------------------------------------
// k_st_cat_bwd: one CTA (128 threads) per sample.  c1 = (1/21) sum_i sum_j P_ij E_j; dE_j = d(flatten)_j
//   + (w_j / 21) dc1 + sum_i dS_ij E_i + sum_i dS_ji E_i   with w_j = sum_i P_ij, a_j = (dc1 . E_j) / 21,
//   dS_ij = P_ij (a_j - sum_k P_ik a_k).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(E) k_st_cat_bwd(const float* __restrict__ allf, const float* __restrict__ Pm,
                                                  const float* __restrict__ dAllf, float* __restrict__ dEcat) {
  __shared__ float Es[NC][E + 1];
  __shared__ float Ps[NC][NC], dS[NC][NC];
  __shared__ float av[NC], wv[NC], dc1[E];
  const int s = blockIdx.x, c = threadIdx.x, warp = c >> 5, lane = c & 31;
  const float* f = allf + (size_t)s * FEAT;
  const float* df = dAllf + (size_t)s * FEAT;
  for (int r = 0; r < NC; ++r) Es[r][c] = f[F_FLAT + r * E + c];
  for (int p = c; p < NC * NC; p += E) Ps[p / NC][p % NC] = Pm[(size_t)s * NC * NC + p];
  dc1[c] = df[F_CATT + c];
  __syncthreads();
  for (int j = warp; j < NC; j += E / 32) {
    float v = 0.f;
    for (int k = lane; k < E; k += 32) v = fmaf(dc1[k], Es[j][k], v);
    v = r4ppo::warp_sum(v);
    if (lane == 0) av[j] = v / (float)NC;
  }
  if (c < NC) {
    float w = 0.f;
    for (int i = 0; i < NC; ++i) w += Ps[i][c];
    wv[c] = w;
  }
  __syncthreads();
  if (c < NC) {
    float pa = 0.f;
    for (int k = 0; k < NC; ++k) pa = fmaf(Ps[c][k], av[k], pa);
    for (int j = 0; j < NC; ++j) dS[c][j] = Ps[c][j] * (av[j] - pa);
  }
  __syncthreads();
  for (int j = 0; j < NC; ++j) {
    float g = df[F_FLAT + j * E + c] + wv[j] * dc1[c] / (float)NC;
    for (int i = 0; i < NC; ++i) g = fmaf(dS[j][i] + dS[i][j], Es[i][c], g);
    dEcat[((size_t)s * NC + j) * E + c] = g;
  }
}

// q = mean of 10 emb_seq rows: every slot's row gradient is (dq0 + dq1) / 10
__global__ void k_st_dq(const float* __restrict__ dq0, const float* __restrict__ dq1, float* __restrict__ dqs, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n * E) dqs[i] = (dq0[i] + dq1[i]) / 10.f;
}

// ------------------------------------------------------------------------------------------------
// The embedding gradients.  Entry e = s * NSLOT + k of sample s: k < 21 the emb_cat slot k (source row dEcat[s][k]);
// 21 <= k < 149 emb_seq for sequence (k - 21) / 64, step (k - 21) % 64 (source dX); k >= 149 emb_seq of cat slot 11 + (k - 149)
// (the query, source dqs[s]).  key = table * H + id; a stable radix sort keeps equal keys in (s, k) order.  slate: the
// sequences are record idx[s]'s, and the pad id 0 of cat slot 20 (in the query too) keys row 0 like any other id.
// ------------------------------------------------------------------------------------------------
__global__ void k_st_embkeys(Layout L, Data D, const int64_t* __restrict__ idx, int n, int slate, const int32_t* __restrict__ cat,
                             uint32_t* __restrict__ keys, int32_t* __restrict__ vals) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n * NSLOT) return;
  const int s = e / NSLOT, k = e % NSLOT;
  uint32_t key;
  if (k < NC) {
    key = (uint32_t)cat[s * NC + k];
  } else if (k < NC + 2 * T) {
    const int i = (k - NC) / T, t = (k - NC) % T;
    const int64_t rec = slate ? idx[s] : idx[s] / 9;
    key = (uint32_t)(L.H + clampid(D.seq[(rec * 2 + i) * T + t], L.H));
  } else {
    key = (uint32_t)(L.H + cat[s * NC + NC - 10 + (k - NC - 2 * T)]);
  }
  keys[e] = key;
  vals[e] = e;
}
constexpr int EST = 512, ESG = EST / E;        // 4 row groups x 128 columns
__global__ void __launch_bounds__(EST) k_st_embsum(Layout L, const uint32_t* __restrict__ keys, const int32_t* __restrict__ vals,
                                                   int total, const float* __restrict__ dEcat, const float* __restrict__ dX0,
                                                   const float* __restrict__ dX1, const float* __restrict__ dqs,
                                                   float* __restrict__ grad) {
  __shared__ float part[ESG][E];
  const int i0 = blockIdx.x;
  const uint32_t key = keys[i0];
  if (i0 > 0 && keys[i0 - 1] == key) return;           // one CTA per run: the one at its first entry
  const int c = threadIdx.x % E, grp = threadIdx.x / E;
  float acc = 0.f;
  for (int i = i0 + grp; i < total && keys[i] == key; i += ESG) {
    const int e = vals[i], s = e / NSLOT, k = e % NSLOT;
    const float* src;
    if (k < NC) src = dEcat + ((size_t)s * NC + k) * E;
    else if (k < NC + 2 * T) src = ((k - NC) / T ? dX1 : dX0) + ((size_t)s * T + (k - NC) % T) * E;
    else src = dqs + (size_t)s * E;
    acc += src[c];
  }
  part[grp][c] = acc;
  __syncthreads();
  if (grp == 0) {
    float v = part[0][c];
    for (int g = 1; g < ESG; ++g) v += part[g][c];
    const int64_t base = key < (uint32_t)L.H ? L.emb_cat + (int64_t)key * E : L.emb_seq + (int64_t)(key - L.H) * E;
    grad[base + c] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// Keras Adam (OptimizerV2 / ResourceApplyAdam): m += (g - m)(1 - b1), v += (g^2 - v)(1 - b2),
// p -= alpha m / (sqrt(v) + eps) with alpha = lr sqrt(1 - b2^t) / (1 - b1^t).  Dense over every parameter (the sparse
// embedding apply of OptimizerV2 decays m and v on every row too).  Clears the nonzero embedding gradient entries, so the
// embedding part of grad is zero again for the next r4_simtrain_grad.
// ------------------------------------------------------------------------------------------------
__global__ void k_st_apply(Layout L, float* __restrict__ prm, float* __restrict__ grad, float* __restrict__ m,
                           float* __restrict__ v, float alpha, float b1, float b2, float eps) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L.n) return;
  const float g = grad[i];
  float mi = m[i], vi = v[i];
  mi += (g - mi) * (1.f - b1);
  vi += (g * g - vi) * (1.f - b2);
  prm[i] -= alpha * mi / (sqrtf(vi) + eps);
  m[i] = mi; v[i] = vi;
  const bool emb = (i >= L.emb_cat && i < L.emb_cat + L.H * E) || (i >= L.emb_seq && i < L.emb_seq + L.H * E);
  if (emb && g != 0.f) grad[i] = 0.f;
}

}  // namespace r4st
