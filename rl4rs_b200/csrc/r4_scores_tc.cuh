// r4_scores_tc.cuh -- K8 on the tensor cores: DIN local-activation scores (deepctr AttentionSequencePoolingLayer
// (att_hidden_units=(64,16), return_score=True, weight_normalization=False); nets/utils.py:114-115,121-122).
//
//   q      = mean_j E_s[cat[-10:]]                                     (query, per feature row)
//   z1_t   = sigmoid(q (Wq+Wd) + b1 + k_t (Wk-Wd) + (q * k_t) Wp)       k_t = GRU-1 output t (cached H)
//   z2_t   = sigmoid(z1_t W2 + b2);   score_t = z2_t . kv + b           (raw, unbounded)
//
// The only GEMM-shaped term, (q*k_t) Wp, is a [64 keys x 128] x [128 x 64] product per (row, sequence); the second
// layer is a [64 keys x 64] x [64 x 16] product.  Both run on wgmma (k_scores_tc2 below).
#pragma once
#include "r4_augru_tc.cuh"
#include "r4_gemm_tc.cuh"

namespace r4tc {

constexpr int S_K = 128, S_N = 64, S_KEYS = 64, AH2_N = 16;
constexpr int S_B_SPLIT = S_N * S_K * 2;           // 16 KB per split
constexpr int S_B_BYTES = 3 * S_B_SPLIT;           // 48 KB, resident
constexpr int S_SBO = (S_K / 8) * 128;             // 2048: 8-row groups (B: the weight image)
// cached key half k_t (Wk - Wd): Kp [n_cached][16 column quads][64 keys][4] (r4_gemm_tc.cuh: kq_index)

// host: Wp [128 k][64 n] fp32 -> 3 splits of [64 n x 128 k] K-major core matrices
inline void build_scores_image(const float* Wp, uint8_t* img) {
  for (int sp = 0; sp < 3; ++sp)
    for (int n = 0; n < S_N; ++n)
      for (int k = 0; k < S_K; ++k) {
        float w = Wp[(size_t)k * S_N + n];
        uint16_t hi = host_bf16_bits(w);
        float r1 = w - host_bf16_val(hi);
        uint16_t mid = host_bf16_bits(r1);
        uint16_t lo = host_bf16_bits(r1 - host_bf16_val(mid));
        uint16_t v = sp == 0 ? hi : (sp == 1 ? mid : lo);
        memcpy(img + (size_t)sp * S_B_SPLIT + (n / 8) * S_SBO + (k / 8) * LBO + (n % 8) * 16 + (k % 8) * 2, &v, 2);
      }
}

struct ScoreTcSeq {
  const float* qa;       // [R, 64]  q (Wq+Wd) + b1, from k_query
  const float* H;        // [n_cached, 64, 128]
  const float* Kp;       // [n_cached, 64, 64]   k_t (Wk - Wd)
  const uint8_t* WpImg;  // S_B_BYTES
  const float* Wqd;      // [128, 64]
  const float* b1;       // [64]
  const float* W2;       // [64, 16]
  const float* b2;       // [16]
  const float* kv;       // [16]
  float bk;
  float* scoresT;        // [ceil(R/128), 64, 128]
  int shared;
};
struct ScoreTcParams {
  ScoreTcSeq s[2];
  const float* q;        // [R, 128]  mean of the 10 slate embeddings, from k_query
  int R, row0, div;
};

// q = reduce_mean(E_s[cat[-10:]]) and qa_i = q (Wq_i + Wd_i) + b1_i for both sequences (nets/utils.py:114-115 and
// the query half of :121-122).  8 rows per CTA, 128 threads.  Keeping this out of k_scores_tc takes two dependent
// HBM round trips (category ids -> embedding rows) and a 128-long serial FMA chain off its per-tile critical path.
__global__ void __launch_bounds__(128) k_query(int R, const int32_t* __restrict__ cat, const float* __restrict__ emb_seq,
                                               const float* __restrict__ Wqd0, const float* __restrict__ b10,
                                               const float* __restrict__ Wqd1, const float* __restrict__ b11,
                                               float* __restrict__ q_out, float* __restrict__ qa0, float* __restrict__ qa1) {
  __shared__ float q_s[8][S_K];
  const int tid = threadIdx.x, r0 = blockIdx.x * 8;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int r = min(r0 + i, R - 1);
    const int32_t* crow = cat + (size_t)r * 21;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 10; ++j) acc += __ldg(emb_seq + (size_t)crow[11 + j] * S_K + tid);
    acc = acc / 10.0f;
    q_s[i][tid] = acc;
    if (r0 + i < R) q_out[(size_t)(r0 + i) * S_K + tid] = acc;
  }
  __syncthreads();
  const int sq = tid >> 6, j = tid & 63;
  const float* W = sq ? Wqd1 : Wqd0;
  float acc[8];
  const float b = __ldg((sq ? b11 : b10) + j);
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = b;
  // 16 weight loads in flight per thread (with 4 the 128-long loop was 32 exposed L2 round trips; the kernel sits between
  // k_assemble and k_scores_tc on the critical path of every pass)
  for (int k0 = 0; k0 < S_K; k0 += 16) {
    float w[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) w[u] = __ldg(W + (k0 + u) * S_N + j);
#pragma unroll
    for (int u = 0; u < 16; ++u)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(q_s[i][k0 + u], w[u], acc[i]);
  }
  float* o = sq ? qa1 : qa0;
#pragma unroll
  for (int i = 0; i < 8; ++i) if (r0 + i < R) o[(size_t)(r0 + i) * S_N + j] = acc[i];
}

constexpr int S_W2_SPLIT = AH2_N * S_N * 2;        // 2 KB per split: [16 n x 64 k] K-major core matrices
constexpr int S_W2_BYTES = 3 * S_W2_SPLIT;         // 6 KB, resident behind the Wp image
constexpr int S_W2_SBO = (S_N / 8) * 128;          // 1024: 8-row groups of the W2 image
constexpr int S_IMG_BYTES = S_B_BYTES + S_W2_BYTES;    // what build_scores_image2 writes and the loader warp copies

// host: Wp image followed by W2 [64 k][16 n] fp32 -> 3 splits of [16 n x 64 k] K-major core matrices
inline void build_scores_image2(const float* Wp, const float* W2, uint8_t* img) {
  build_scores_image(Wp, img);
  uint8_t* w2 = img + S_B_BYTES;
  for (int sp = 0; sp < 3; ++sp)
    for (int n = 0; n < AH2_N; ++n)
      for (int k = 0; k < S_N; ++k) {
        float w = W2[(size_t)k * AH2_N + n];
        uint16_t hi = host_bf16_bits(w);
        float r1 = w - host_bf16_val(hi);
        uint16_t mid = host_bf16_bits(r1);
        uint16_t lo = host_bf16_bits(r1 - host_bf16_val(mid));
        uint16_t v = sp == 0 ? hi : (sp == 1 ? mid : lo);
        memcpy(w2 + (size_t)sp * S_W2_SPLIT + (n / 8) * S_W2_SBO + (k / 8) * LBO + (n % 8) * 16 + (k % 8) * 2, &v, 2);
      }
}

// How many of `ctas` CTAs walk sequence 0 (the rest walk sequence 1).  A sequence whose cached rows are SHARED by all feature
// rows (Slate's constant second sequence) streams nothing from HBM and its tiles finish sooner : it gets the
// smaller share, `shared_pct` per cent of an even split's.
__host__ __device__ inline int scores_grid_split(int ctas, int ntiles, int shared0, int shared1, int shared_pct) {
  if (ctas < 2) return ctas;
  int n0 = ctas / 2;
  if (shared0 != shared1) {
    const int small = max(1, (ctas / 2) * shared_pct / 100);
    n0 = shared1 ? ctas - small : small;
  }
  (void)ntiles;
  return n0;
}

// One warpgroup per CTA, two CTAs per SM.  CTAs [0, n0) walk the feature rows of sequence 0, the rest those of
// sequence 1 (scores_grid_split); a tile is one feature row = its 64 keys = the wgmma M.  Per tile: A = q*H as bf16 hi/lo
// in shared memory; layer 1 [64 x 128] x Wp[128 x 64] as 5 wgmmas per K16 (A 2-way x Wp 3-way split: lo*mid, hi*lo, lo*hi,
// hi*mid, hi*hi); z1 = sigmoid(layer 1 + q(Wq+Wd) + b1 + k_t(Wk-Wd)) stays in the accumulator registers, which ARE the
// register A-operand fragments of layer 2 [64 x 64] x W2[64 x 16] (same split, 5 wgmmas per K16); the 16 -> 1 tail is a
// dot product over the four threads that hold a key's 16 units.
constexpr int S2_THREADS = 128;
constexpr int S2_A_SPLIT = S_KEYS * S_K * 2;            // 16 KB
constexpr int S2_SMEM_BYTES = 2 * S2_A_SPLIT + S_IMG_BYTES;
__global__ void __launch_bounds__(S2_THREADS, 2) k_scores_tc2(ScoreTcParams p, int n0) {
  const int sq = (int)blockIdx.x >= n0 ? 1 : 0;
  const int bx = (int)blockIdx.x - (sq ? n0 : 0), nbx = sq ? (int)gridDim.x - n0 : n0;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sA = smem;                           // hi, lo
  uint8_t* sB = smem + 2 * S2_A_SPLIT;          // Wp hi/mid/lo, then W2 hi/mid/lo
  __shared__ uint64_t bar_w;
  __shared__ float b2_s[AH2_N], kv_s[AH2_N];
  const ScoreTcSeq& S = p.s[sq];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
  if (tid == 0) {
    mbar_init(&bar_w, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(&bar_w, S_IMG_BYTES);
    bulk_g2s(sB, S.WpImg, S_IMG_BYTES, &bar_w);
  }
  if (tid < AH2_N) { b2_s[tid] = __ldg(S.b2 + tid); kv_s[tid] = __ldg(S.kv + tid); }
  __syncthreads();
  mbar_wait(&bar_w, 0);
  const uint32_t a0 = smem_u32(sA), b0 = smem_u32(sB), w0 = b0 + S_B_BYTES;
  constexpr int A_SBO = (S_K / 8) * LBO;                 // 2048
  const int pkey = tid >> 1, pk0 = (tid & 1) * 64;      // producer role: key row, first of 64 K values
  for (int r = bx; r < p.R; r += nbx) {
    const size_t ci = S.shared ? 0 : (size_t)((p.row0 + r) / p.div);
    // ---- A = q * H_t (bf16 hi / lo) ----
    const float* hrow = S.H + (ci * S_KEYS + pkey) * S_K + pk0;
    const float* qrow = p.q + (size_t)r * S_K + pk0;
    __syncthreads();                                     // the previous tile's wgmmas have read A
#pragma unroll
    for (int k8 = 0; k8 < 8; ++k8) {
      float v[8];
      const float4 h0 = __ldg(reinterpret_cast<const float4*>(hrow + k8 * 8)), h1 = __ldg(reinterpret_cast<const float4*>(hrow + k8 * 8 + 4));
      const float4 q0 = __ldg(reinterpret_cast<const float4*>(qrow + k8 * 8)), q1 = __ldg(reinterpret_cast<const float4*>(qrow + k8 * 8 + 4));
      v[0] = h0.x * q0.x; v[1] = h0.y * q0.y; v[2] = h0.z * q0.z; v[3] = h0.w * q0.w;
      v[4] = h1.x * q1.x; v[5] = h1.y * q1.y; v[6] = h1.z * q1.z; v[7] = h1.w * q1.w;
      uint4 hi, lo;
      split8(v, hi, lo);
      const uint32_t off = (uint32_t)(pkey / 8) * A_SBO + (uint32_t)(pk0 / 8 + k8) * LBO + (uint32_t)(pkey % 8) * 16;
      *reinterpret_cast<uint4*>(sA + off) = hi;
      *reinterpret_cast<uint4*>(sA + S2_A_SPLIT + off) = lo;
    }
    proxy_fence();
    __syncthreads();
    // ---- layer 1 ----
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < S_K / 16; ++j) {
      const uint32_t ko = j * 2 * LBO;
      const uint64_t ah = make_desc(a0 + ko, LBO, A_SBO), al = make_desc(a0 + S2_A_SPLIT + ko, LBO, A_SBO);
      const uint64_t bh = make_desc(b0 + ko, LBO, S_SBO), bm = make_desc(b0 + S_B_SPLIT + ko, LBO, S_SBO);
      const uint64_t bl = make_desc(b0 + 2 * S_B_SPLIT + ko, LBO, S_SBO);
      wgmma_m64n64k16(acc, al, bm);
      wgmma_m64n64k16(acc, ah, bl);
      wgmma_m64n64k16(acc, al, bh);
      wgmma_m64n64k16(acc, ah, bm);
      wgmma_m64n64k16(acc, ah, bh);
    }
    wgmma_commit();
    // the epilogue's own inputs load while the wgmmas run
    float2 qa[8], kp[2][8];
    const int key0 = warp * 16 + g;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int col = jj * 8 + 2 * tq;
      qa[jj] = __ldg(reinterpret_cast<const float2*>(S.qa + (size_t)r * S_N + col));
#pragma unroll
      for (int h = 0; h < 2; ++h)
        kp[h][jj] = __ldg(reinterpret_cast<const float2*>(S.Kp + kq_index(ci, S_N / 4, col / 4, S_KEYS, key0 + 8 * h) + (col & 3)));
    }
    wgmma_wait<0>();
    // ---- z1 -> layer-2 A fragments (k slice ks: registers 8 ks .. 8 ks + 7 of the accumulator) ----
    uint32_t zh[4][4], zl[4][4];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = jj * 4 + 2 * h;
        const float z0 = fast_sigmoid(acc[i] + qa[jj].x + kp[h][jj].x), z1 = fast_sigmoid(acc[i + 1] + qa[jj].y + kp[h][jj].y);
        split2(z0, z1, zh[jj >> 1][(jj & 1) * 2 + h], zl[jj >> 1][(jj & 1) * 2 + h]);
      }
    float acc2[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc2[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < S_N / 16; ++ks) {
      const uint32_t ko = ks * 2 * LBO;
      const uint64_t wh = make_desc(w0 + ko, LBO, S_W2_SBO), wm = make_desc(w0 + S_W2_SPLIT + ko, LBO, S_W2_SBO);
      const uint64_t wl = make_desc(w0 + 2 * S_W2_SPLIT + ko, LBO, S_W2_SBO);
      wgmma_m64n16k16_rs(acc2, zl[ks], wm);
      wgmma_m64n16k16_rs(acc2, zh[ks], wl);
      wgmma_m64n16k16_rs(acc2, zl[ks], wh);
      wgmma_m64n16k16_rs(acc2, zh[ks], wm);
      wgmma_m64n16k16_rs(acc2, zh[ks], wh);
    }
    wgmma_commit();
    wgmma_wait<0>();
    // ---- tail: score = sigmoid(z2 + b2) . kv + bk ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float sc = 0.f;
#pragma unroll
      for (int jn = 0; jn < 2; ++jn)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = jn * 8 + 2 * tq + e;
          sc = fmaf(fast_sigmoid(acc2[jn * 4 + 2 * h + e] + b2_s[col]), kv_s[col], sc);
        }
      sc += __shfl_xor_sync(0xffffffffu, sc, 1);
      sc += __shfl_xor_sync(0xffffffffu, sc, 2);
      if (tq == 0) S.scoresT[((size_t)(r >> 7) * S_KEYS + key0 + 8 * h) * 128 + (r & 127)] = sc + S.bk;
    }
  }
}

}  // namespace r4tc
