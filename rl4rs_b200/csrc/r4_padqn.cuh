// r4_padqn.cuh -- parametric-action DQN on the discrete env: a state-action Q network scored over every (row, item) pair.
//
//   input    x = [obs(s) (256) | e(a) (D)], e(a) the fixed item vector (row a of the env's action_emb)
//   net      Dense 256 tanh -> Dense 256 tanh -> Dense 1                 (RLlib's default fcnet over the concatenation)
//   mask     Qm(s, a) = Q(s, a) where the action mask is set, float32.min where it is not (MyMaskActionsModel's
//            Q + max(log mask, float32.min), as a select)
//   act      the first argmax of Qm, or SoftQ(T = 1) by inverse CDF over one counter-based uniform per row (RAINBOW's rule)
//   learner  a* = argmax Qm_online(s', .), y = r + gamma (1 - done) Qm_target(s', a*), td = Q(s, a) - y,
//            loss = sum_i w_i huber(td_i) inv_n (delta 1); hand-derived backward.
//
// Flat parameter layout: w1[256+D, 256] b1[256] w2[256,256] b2[256] w3[256,1] b3[1]   (6 tensors; the target the same)
//
// The first layer splits exactly: x w1 + b1 = S[s] + P[a] with S = obs w1[:256] + b1 (per row, k_dense_gemm) and
// P = E w1[256:] (per item, once per parameter version).  The pair scorer k_padqn_pairs forms h1 = tanh(S[s] + P[a]) of a
// tile of 128 pairs in shared memory as the wgmma A operand (split three ways into bf16, as k_gemm_tc splits its
// operands), multiplies it by a pre-tiled bf16 hi/mid/lo image of w2 over the six products whose magnitude exceeds 2^-24
// of the result, and reduces tanh(. + b2) . w3 + b3 in registers: the [n A, 256] hidden planes never reach memory.
// The image and P live in a per-net cache that k_padqn_refresh rebuilds after every parameter change.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <float.h>
#include <stdint.h>

#include "r4_augru_tc.cuh"
#include "r4_ddpg.cuh"
#include "r4_dense.cuh"

namespace r4pa {

using r4ddpg::NT;
using r4ddpg::TS;
constexpr int OBS = 256, H = 256, MAXA = 512, MAXD = 512;
constexpr int MAXN = 65535 * 64;    // rows: k_dense_gemm's 64-row tiles of S on gridDim.y

struct Layout {
  int A, D, K;                      // K = 256 + D: the first layer's input width
  int w1, b1, w2, b2, w3, b3, n;
};
__host__ __device__ inline Layout make_layout(int A, int D) {
  Layout L;
  L.A = A; L.D = D; L.K = OBS + D;
  L.w1 = 0;               L.b1 = L.w1 + L.K * H;
  L.w2 = L.b1 + H;        L.b2 = L.w2 + H * H;
  L.w3 = L.b2 + H;        L.b3 = L.w3 + H;
  L.n = L.b3 + 1;
  return L;
}

// ---- the per-net cache: the w2 image (r4tc::build_gemm_image's layout at K = N = 256, one 256-wide n-tile), then P [A][256]
constexpr int BK = 32, KBN = H / BK, SPLIT = 3;
constexpr size_t IMG_BYTES = (size_t)KBN * SPLIT * H * BK * 2;      // 384 KB
__host__ __device__ inline size_t cache_bytes(int A) { return IMG_BYTES + (size_t)A * H * 4; }
__host__ __device__ inline const float* cache_p(const uint8_t* c) { return reinterpret_cast<const float*>(c + IMG_BYTES); }

// Blocks [0, IMG_CTAS) write the image (one thread per (K block, column, k) element, its three splits); block IMG_CTAS + a
// writes P[a][:] = sum_d E[a][d] w1[256 + d][:] (d in order).  cache2 (may be NULL) receives the same bytes.
constexpr int IMG_CTAS = KBN * H * BK / 256;
__global__ void __launch_bounds__(256) k_padqn_refresh(Layout L, const float* __restrict__ prm, const float* __restrict__ emb,
                                                        uint8_t* __restrict__ cache, uint8_t* __restrict__ cache2) {
  const int tid = threadIdx.x;
  if ((int)blockIdx.x < IMG_CTAS) {
    const int e = blockIdx.x * 256 + tid, kb = e / (H * BK), r = e % (H * BK), n = r / BK, kk = r % BK;
    const float w = __ldg(prm + L.w2 + (size_t)(kb * BK + kk) * H + n);
    const __nv_bfloat16 hi = __float2bfloat16_rn(w);
    const float r1 = w - __bfloat162float(hi);
    const __nv_bfloat16 mid = __float2bfloat16_rn(r1);
    const __nv_bfloat16 lo = __float2bfloat16_rn(r1 - __bfloat162float(mid));
    const __nv_bfloat16 v[3] = {hi, mid, lo};
    const size_t in = (size_t)(n / 8) * (BK / 8 * 128) + (kk / 8) * r4tc::LBO + (n % 8) * 16 + (kk % 8) * 2;
#pragma unroll
    for (int sp = 0; sp < SPLIT; ++sp) {
      const size_t o = ((size_t)kb * SPLIT + sp) * H * BK * 2 + in;
      *reinterpret_cast<__nv_bfloat16*>(cache + o) = v[sp];
      if (cache2) *reinterpret_cast<__nv_bfloat16*>(cache2 + o) = v[sp];
    }
    return;
  }
  const int a = blockIdx.x - IMG_CTAS;
  const float* e = emb + (size_t)a * L.D;
  const float* w = prm + L.w1 + (size_t)OBS * H + tid;
  float acc = 0.f;
  for (int d = 0; d < L.D; ++d) acc = fmaf(__ldg(e + d), __ldg(w + (size_t)d * H), acc);
  const size_t o = IMG_BYTES / 4 + (size_t)a * H + tid;
  reinterpret_cast<float*>(cache)[o] = acc;
  if (cache2) reinterpret_cast<float*>(cache2)[o] = acc;
}

// ------------------------------------------------------------------------------------------------
// The pair scorer: Qm[p] for the flat pairs p = s A + a < n A, in tiles of 128 consecutive pairs (persistent CTAs).  Two
// warpgroups, each the wgmma issuer of 64 of the tile's rows over the 4 64-column chunks of the 256 outputs.  Per K block of
// 32: every thread forms 8 consecutive h1 values of two pairs (tanhf of S + P, fp32) and writes their hi / mid / lo core
// matrices; one thread streams the w2 image's stage by bulk copy; the wgmmas of K block i run while K block i + 1 is formed.
// Epilogue in registers: each thread holds 2 rows x 64 columns; tanh(acc + b2) . w3 summed in a fixed order, then over the
// four lanes of the row by shuffles (deterministic), + b3, then the mask select.
// ------------------------------------------------------------------------------------------------
constexpr int PM = 128, PTHREADS = 256;
constexpr int A_STAGE = PM * BK * 2;                            // 8 KB per split
constexpr int B_STAGE = H * BK * 2;                             // 16 KB per split
constexpr int STAGE_BYTES = SPLIT * (A_STAGE + B_STAGE);        // 72 KB
constexpr int PAIRS_SMEM = 2 * STAGE_BYTES;                     // 144 KB
constexpr int SBO = (BK / 8) * 128;

__global__ void __launch_bounds__(PTHREADS, 1) k_padqn_pairs(const float* __restrict__ S, const uint8_t* __restrict__ cache,
                                                             const float* __restrict__ prm, Layout L, const uint8_t* __restrict__ mask,
                                                             int n, float* __restrict__ qm) {
  using namespace r4tc;
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ uint64_t bar[2];
  __shared__ float b2s[H], w3s[H];
  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, tq = lane & 3;
  const int A = L.A;
  const int64_t npairs = (int64_t)n * A;
  const int ntiles = (int)((npairs + PM - 1) / PM);
  const float* P = cache_p(cache);
  b2s[tid] = __ldg(prm + L.b2 + tid);
  w3s[tid] = __ldg(prm + L.w3 + tid);
  const float b3 = __ldg(prm + L.b3);
  if (tid == 0) {
    mbar_init(&bar[0], 1); mbar_init(&bar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int kc = tid & 3, r8 = tid >> 2;               // this thread forms rows r8 and 64 + r8, k = kb 32 + kc 8 .. + 8
  int it = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t p0 = (int64_t)tile * PM;
    const float *srow[2], *prow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t p = min(p0 + h * 64 + r8, npairs - 1);
      srow[h] = S + (p / A) * H + kc * 8;
      prow[h] = P + (p % A) * H + kc * 8;
    }
    float acc[4][32];
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;
    for (int kb = 0; kb < KBN; ++kb, ++it) {
      const int s = it & 1;
      uint8_t* sa = smem + s * STAGE_BYTES;
      float v[2][8];
#pragma unroll
      for (int h = 0; h < 2; ++h) {                  // loads first: they overlap the wgmmas of the previous K block
        const float4 a0 = __ldg(reinterpret_cast<const float4*>(srow[h] + kb * BK));
        const float4 a1 = __ldg(reinterpret_cast<const float4*>(srow[h] + kb * BK + 4));
        const float4 c0 = __ldg(reinterpret_cast<const float4*>(prow[h] + kb * BK));
        const float4 c1 = __ldg(reinterpret_cast<const float4*>(prow[h] + kb * BK + 4));
        v[h][0] = a0.x + c0.x; v[h][1] = a0.y + c0.y; v[h][2] = a0.z + c0.z; v[h][3] = a0.w + c0.w;
        v[h][4] = a1.x + c1.x; v[h][5] = a1.y + c1.y; v[h][6] = a1.z + c1.z; v[h][7] = a1.w + c1.w;
      }
      wgmma_wait<1>();                // this warpgroup's wgmmas of K block it - 2 (the last reader of stage s) are done
      __syncthreads();                // ... and the other warpgroup's
      if (tid == 0) {
        mbar_expect_tx(&bar[s], SPLIT * B_STAGE);
#pragma unroll
        for (int sp = 0; sp < SPLIT; ++sp)
          bulk_g2s(sa + SPLIT * A_STAGE + sp * B_STAGE, cache + ((size_t)kb * SPLIT + sp) * B_STAGE, B_STAGE, &bar[s]);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = h * 64 + r8;
        float x[8], r1[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = tanhf(v[h][j]);
        uint4 hi, mid;
        split8(x, hi, mid);                               // hi and bf16(x - hi)
        const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&hi);
        const __nv_bfloat162* m2 = reinterpret_cast<const __nv_bfloat162*>(&mid);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          r1[2 * j] = (x[2 * j] - __bfloat162float(h2[j].x)) - __bfloat162float(m2[j].x);
          r1[2 * j + 1] = (x[2 * j + 1] - __bfloat162float(h2[j].y)) - __bfloat162float(m2[j].y);
        }
        uint32_t l[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          __nv_bfloat162 ll = __floats2bfloat162_rn(r1[2 * j], r1[2 * j + 1]);
          l[j] = *reinterpret_cast<uint32_t*>(&ll);
        }
        const uint32_t off = (uint32_t)(row / 8) * SBO + (uint32_t)kc * LBO + (uint32_t)(row % 8) * 16;
        *reinterpret_cast<uint4*>(sa + off) = hi;
        *reinterpret_cast<uint4*>(sa + A_STAGE + off) = mid;
        *reinterpret_cast<uint4*>(sa + 2 * A_STAGE + off) = make_uint4(l[0], l[1], l[2], l[3]);
      }
      proxy_fence();
      __syncthreads();                // the whole A stage is written
      mbar_wait(&bar[s], (uint32_t)((it >> 1) & 1));
      wgmma_fence();
      const uint32_t a0 = smem_u32(sa) + (uint32_t)wg * 8 * SBO, b0 = smem_u32(sa + SPLIT * A_STAGE);
#pragma unroll
      for (int j = 0; j < BK / 16; ++j) {
        uint64_t a[3];
#pragma unroll
        for (int sp = 0; sp < 3; ++sp) a[sp] = make_desc(a0 + sp * A_STAGE + j * 2 * LBO, LBO, SBO);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          uint64_t b[3];
#pragma unroll
          for (int sp = 0; sp < 3; ++sp) b[sp] = make_desc(b0 + sp * B_STAGE + c * 8 * SBO + j * 2 * LBO, LBO, SBO);
          // smallest products first so they are not absorbed by a large partial sum
          wgmma_m64n64k16(acc[c], a[1], b[1]);   // mid*mid
          wgmma_m64n64k16(acc[c], a[0], b[2]);   // hi*lo
          wgmma_m64n64k16(acc[c], a[2], b[0]);   // lo*hi
          wgmma_m64n64k16(acc[c], a[0], b[1]);   // hi*mid
          wgmma_m64n64k16(acc[c], a[1], b[0]);   // mid*hi
          wgmma_m64n64k16(acc[c], a[0], b[0]);   // hi*hi
        }
      }
      wgmma_commit();
    }
    wgmma_wait<0>();
    // register i of chunk c: row 16 wq + g + 8 ((i / 2) % 2), column 64 c + 8 (i / 4) + 2 tq + i % 2
    float part[2] = {0.f, 0.f};
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int col = c * 64 + (i >> 2) * 8 + 2 * tq + (i & 1);
        part[(i >> 1) & 1] = fmaf(tanhf(acc[c][i] + b2s[col]), w3s[col], part[(i >> 1) & 1]);
      }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      part[h] += __shfl_xor_sync(0xffffffffu, part[h], 1);
      part[h] += __shfl_xor_sync(0xffffffffu, part[h], 2);
    }
    if (tq < 2) {
      const int64_t p = p0 + wg * 64 + wq * 16 + g + 8 * tq;
      if (p < npairs) qm[p] = mask[p] ? part[tq] + b3 : -FLT_MAX;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// act: one warp per row of Qm [n][A].  explore 0 -> the first argmax; 1 -> SoftQ, a = the first a with
// sum_{a' <= a} e^(Qm_a' - max) > u sum_a e^(Qm_a - max), u = the top 24 bits of r4ddpg::draw(seed, counter, row, 0) / 2^24
// (k_rainbow_act's rule; lane 0 walks the row in action order).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int first_argmax(const float* q, int A) {
  const int lane = threadIdx.x & 31;
  float best = -INFINITY;
  int bi = A;
  for (int a = lane; a < A; a += 32) {
    const float v = q[a];
    if (v > best) { best = v; bi = a; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  return bi < A ? bi : 0;
}

__global__ void __launch_bounds__(NT) k_padqn_act(const float* __restrict__ qm, int n, int A, int explore, uint64_t seed,
                                                  uint64_t counter, int32_t* __restrict__ action) {
  const int row = blockIdx.x * (NT / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= n) return;
  const float* q = qm + (size_t)row * A;
  if (!explore) {
    const int a = first_argmax(q, A);
    if (lane == 0) action[row] = a;
    return;
  }
  if (lane) return;
  float m = q[0];
  for (int a = 1; a < A; ++a) m = fmaxf(m, q[a]);
  float se = 0.f;
  for (int a = 0; a < A; ++a) se += expf(q[a] - m);
  const float u = (float)(r4ddpg::draw(seed, counter, row, 0) >> 40) * (1.0f / 16777216.0f) * se;
  int a = 0;
  float run = 0.f;
  for (; a < A - 1; ++a) {
    run += expf(q[a] - m);
    if (u < run) break;
  }
  action[row] = a;
}

// ------------------------------------------------------------------------------------------------
// store (1-step): row r = t B + b of a [T, B] rollout goes to slot (pos + r) % C; new_obs and the next-state mask are row
// r + B's, or final_obs[b] / final_mask[b] at t = T - 1.  Only the last C rows are written when T B > C.  New items get
// priority max_prio^alpha.
// ------------------------------------------------------------------------------------------------
struct Ring {
  float* obs;
  int32_t* act;
  float *rew, *new_obs;
  uint8_t *done, *next_mask;
};
__global__ void k_padqn_store(Ring R, float* __restrict__ r_prio, const float* __restrict__ max_prio, int C, int A, int64_t pos,
                              float alpha, const float* __restrict__ obs, const float* __restrict__ final_obs,
                              const uint8_t* __restrict__ mask, const uint8_t* __restrict__ final_mask,
                              const int32_t* __restrict__ act, const float* __restrict__ rew, const uint8_t* __restrict__ done,
                              int T, int B) {
  const int64_t n = (int64_t)T * B, first = n > C ? n - C : 0;
  const int64_t r = first + blockIdx.x;
  if (r >= n) return;
  const int64_t slot = (pos + r) % C;
  const int t = (int)(r / B), b = (int)(r % B);
  const bool last = t == T - 1;
  const float* nx = last ? final_obs + (int64_t)b * OBS : obs + (r + B) * OBS;
  const uint8_t* nm = last ? final_mask + (int64_t)b * A : mask + (r + B) * A;
  for (int k = threadIdx.x; k < OBS; k += blockDim.x) {
    R.obs[slot * OBS + k] = obs[r * OBS + k];
    R.new_obs[slot * OBS + k] = nx[k];
  }
  for (int k = threadIdx.x; k < A; k += blockDim.x) R.next_mask[slot * A + k] = nm[k];
  if (threadIdx.x == 0) {
    R.rew[slot] = rew[r];
    R.act[slot] = act[r];
    R.done[slot] = done[r];
    if (r_prio) r_prio[slot] = powf(max_prio[0], alpha);
  }
}

// ------------------------------------------------------------------------------------------------
// learner scratch planes, n rows each
// ------------------------------------------------------------------------------------------------
struct Planes {
  int64_t* idx;                    // [n] sampled indices
  float *weights, *x2, *s_on, *s_tg, *q_on, *q_tg;   // weights [n]; s' rows [n][256]; S of both nets [n][256]; Qm(s') [n][A] x 2
  uint8_t* m2;                     // next-state masks [n][A]
  float *x, *h1, *h2, *d1, *d2, *dq;                 // [s | e(a)] [n][256+D], hiddens and their dZ [n][256], dQ [n]
  float *td, *stats;               // td [n], per-sample statistics [n][3]
  float* grad;                     // [np]
};
// Every plane starts on a 16-byte boundary (the pair scorer reads S rows as float4), whatever n is.  With s == NULL only
// the size is computed: -> the floats the planes take.
__host__ __device__ inline size_t carve(float* s, const Layout& L, int n, Planes* P) {
  size_t off = 0;
  auto take = [&](size_t k) { float* q = s ? s + off : nullptr; off += (k + 3) & ~(size_t)3; return q; };
  const size_t N = (size_t)n;
  P->idx = reinterpret_cast<int64_t*>(take(2 * N));  // first: the scratch base is 8-byte aligned
  P->weights = take(N);
  P->x2 = take(N * H); P->s_on = take(N * H); P->s_tg = take(N * H);
  P->q_on = take(N * L.A); P->q_tg = take(N * L.A);
  P->m2 = reinterpret_cast<uint8_t*>(take((N * L.A + 3) / 4));
  P->x = take(N * L.K);
  P->h1 = take(N * H); P->h2 = take(N * H); P->d1 = take(N * H); P->d2 = take(N * H);
  P->dq = take(N); P->td = take(N); P->stats = take(3 * N);
  P->grad = take(L.n);
  return off;
}
__host__ __device__ inline size_t scratch_floats(const Layout& L, int n) {
  Planes P;
  return carve(nullptr, L, n, &P);
}
__host__ __device__ inline Planes make_planes(float* s, const Layout& L, int n) {
  Planes P;
  carve(s, L, n, &P);
  return P;
}

// x2[i] = new_obs[idx[i]], m2[i] = next_mask[idx[i]]: one CTA per sample
__global__ void k_padqn_gather(const float* __restrict__ r_new_obs, const uint8_t* __restrict__ r_next_mask, int A,
                               const int64_t* __restrict__ idx, float* __restrict__ x2, uint8_t* __restrict__ m2) {
  const int i = blockIdx.x;
  const int64_t r = idx[i];
  for (int k = threadIdx.x; k < OBS; k += blockDim.x) x2[(size_t)i * OBS + k] = __ldg(r_new_obs + r * OBS + k);
  for (int k = threadIdx.x; k < A; k += blockDim.x) m2[(size_t)i * A + k] = r_next_mask[r * A + k];
}

struct Replay {
  const float* obs;
  const int32_t* act;
  const float* rew;
  const uint8_t* done;
};
// x [TS][256+D], h1, h2, t1, t2 [TS][256]
__host__ __device__ inline size_t rows_smem(const Layout& L) { return ((size_t)TS * L.K + 4 * TS * H) * 4; }

// The taken pairs, TS samples per CTA: a* and y from the pair scorer's Qm planes, the online net on [s | e(a)] in fp32 FMAs,
// td, the Huber loss and its backward rows, written to the planes k_dense_wgrad reads.
__global__ void __launch_bounds__(NT) k_padqn_rows(Layout L, const float* __restrict__ prm, const float* __restrict__ emb,
                                                   Replay R, float gamma, float inv_n, const int64_t* __restrict__ idx,
                                                   const float* __restrict__ weights, int n, Planes P) {
  extern __shared__ __align__(16) float sm[];
  float *x = sm, *h1 = x + TS * L.K, *h2 = h1 + TS * H, *t1 = h2 + TS * H, *t2 = t1 + TS * H;
  __shared__ int64_t src[TS];
  __shared__ int taken[TS];
  __shared__ float ys[TS], dqs[TS];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, A = L.A;
  const int q0 = blockIdx.x * TS, nvalid = min(TS, n - q0);
  if (tid < TS) {
    src[tid] = idx[min(q0 + tid, n - 1)];
    taken[tid] = R.act[src[tid]];
  }
  __syncthreads();
  // ---- double Q: a* = the first argmax of the online Qm(s', .), y = r + gamma (1 - done) Qm_target(s', a*) ----
  {
    const int s = warp, q = min(q0 + s, n - 1);
    const int astar = first_argmax(P.q_on + (size_t)q * A, A);
    if (lane == 0) {
      const float nd = __fmul_rn(gamma, 1.f - (float)R.done[src[s]]);
      ys[s] = __fadd_rn(R.rew[src[s]], __fmul_rn(nd, P.q_tg[(size_t)q * A + astar]));
    }
  }
  for (int i = tid; i < TS * L.K; i += NT) {
    const int s = i / L.K, k = i % L.K;
    x[i] = k < OBS ? __ldg(R.obs + src[s] * OBS + k) : __ldg(emb + (size_t)taken[s] * L.D + (k - OBS));
  }
  __syncthreads();
  r4ddpg::dense<2>(prm + L.w1, prm + L.b1, x, L.K, L.K, H, h1, H);
  r4ddpg::dense<2>(prm + L.w2, prm + L.b2, h1, H, H, H, h2, H);
  {
    const int s = warp;
    float a = 0.f;
    for (int k = lane; k < H; k += 32) a = fmaf(h2[s * H + k], __ldg(prm + L.w3 + k), a);
    a = r4ppo::warp_sum(a);
    if (lane == 0) {
      const float q = a + __ldg(prm + L.b3), td = q - ys[s];
      const float w = s < nvalid ? (weights ? weights[q0 + s] : 1.f) : 0.f;
      const float at = fabsf(td), hub = at <= 1.f ? 0.5f * td * td : at - 0.5f;
      dqs[s] = w * fminf(fmaxf(td, -1.f), 1.f) * inv_n;
      if (s < nvalid) {
        P.td[q0 + s] = td;
        P.dq[q0 + s] = dqs[s];
        float* st = P.stats + (size_t)(q0 + s) * 3;
        st[0] = w * hub; st[1] = td; st[2] = q;
      }
    }
  }
  __syncthreads();
  // ---- backward: dZ2 = dQ w3 (1 - h2^2), dZ1 = (dZ2 w2^T) (1 - h1^2) ----
  for (int i = tid; i < TS * H; i += NT) t2[i] = dqs[i / H] * __ldg(prm + L.w3 + i % H) * (1.f - h2[i] * h2[i]);
  __syncthreads();
  r4ddpg::dense_back(prm + L.w2, 0, t2, H, H, nullptr, t1, H);
  for (int i = tid; i < TS * H; i += NT) t1[i] *= 1.f - h1[i] * h1[i];
  __syncthreads();
  for (int i = tid; i < nvalid * L.K; i += NT) P.x[(size_t)q0 * L.K + i] = x[i];
  for (int i = tid; i < nvalid * H; i += NT) {
    const size_t o = (size_t)q0 * H + i;
    P.h1[o] = h1[i]; P.h2[o] = h2[i]; P.d1[o] = t1[i]; P.d2[o] = t2[i];
  }
}

// The weight gradients of the 6 tensors, as jobs of r4dense::k_dense_wgrad
inline r4dense::Jobs make_jobs(const Layout& L, const Planes& P) {
  r4dense::Jobs J;
  int k = 0;
  r4dense::layer_jobs(J, k, P.x, L.K, P.d1, L.K, H, L.w1, L.b1);
  r4dense::layer_jobs(J, k, P.h1, H, P.d2, H, H, L.w2, L.b2);
  r4dense::layer_jobs(J, k, P.h2, H, P.dq, H, 1, L.w3, L.b3);
  r4dense::tile_jobs(J, k);
  return J;
}

}  // namespace r4pa
