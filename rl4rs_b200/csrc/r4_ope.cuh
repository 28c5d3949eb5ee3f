// r4_ope.cuh -- off-policy evaluation (script/offline_evaluation.py's `ope` stage): the row kernels of the logged-policy
// (behaviour) net and the per-step gather of the propensities, values and rewards.  The behaviour net is nets/dnn.py's
// graph at 50 dense features; its dense products are r4dense::k_dense_gemm, launched by r4_learn.cu.  fp32 with f64 sums,
// deterministic: every output has one writer and every sum a fixed order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "r4_dense.cuh"

namespace r4ope {

constexpr int E = 128;          // the category embedding width (emb_size)
constexpr int NCAT = 21;        // category_feature_num of behavior_model.py:12
constexpr int NDENSE = 50;      // dense_feature_num of behavior_model.py:13
constexpr int NHEAD = 11;       // user_protrait[:10] + [sequence_id]
constexpr int NITEMF = 5;       // the first 5 of each item's features
constexpr int CAT_LD = 256;     // the concat row [mean embedding 128 | dense tower 128]
constexpr int NT = 256;

// Column of the behaviour block [B, C - 1] (column c - 1 holds y[c] renormalised over its slice) that action_probs
// reads for `layer` (behavior_model.py:47-58): layer 1 -> y[1:40], 2 -> y[40:148], any other -> y[148:], each index
// clipped as the reference clips it.
__host__ __device__ inline int block_col(int layer, int a) {
  if (layer == 1) return min(max(a - 1, 0), 38);
  if (layer == 2) return 39 + min(max(a - 40, 0), 107);
  return 147 + min(max(a - 148, 0), 233);
}

// One CTA per row b: the page's category ids (head[b][0..10], items[b][page K ..][0..K-1], post-padded with 0 to 21) ->
// the mean of their embedding rows into cat[b][0..127]; the page's dense row (feat[b][page 5K ..][0..5K-1], post-padded
// with 0 to 50) -> dense[b][0..49].  Ids outside [0, H) are clamped into the table.
__global__ void __launch_bounds__(E) k_ope_inputs(int B, int K, int P, int page, int H, const int32_t* __restrict__ head,
                                                  const int32_t* __restrict__ items, const float* __restrict__ feat,
                                                  const float* __restrict__ emb, float* __restrict__ cat,
                                                  float* __restrict__ dense) {
  const int b = blockIdx.x, e = threadIdx.x;
  if (b >= B) return;
  __shared__ int ids[NCAT];
  if (e < NCAT) {
    int v = 0;
    if (e < NHEAD) v = head[(int64_t)b * NHEAD + e];
    else if (e - NHEAD < K) v = items[(int64_t)b * P * K + (int64_t)page * K + (e - NHEAD)];
    ids[e] = min(max(v, 0), H - 1);
  }
  if (e < NDENSE) {
    const int nd = NITEMF * K;
    dense[(int64_t)b * NDENSE + e] = e < nd ? feat[(int64_t)b * P * nd + (int64_t)page * nd + e] : 0.f;
  }
  __syncthreads();
  float s = 0.f;
  for (int j = 0; j < NCAT; ++j) s += emb[(int64_t)ids[j] * E + e];
  cat[(int64_t)b * CAT_LD + e] = s / (float)NCAT;
}

// Sum of v over the CTA's NT threads in a fixed tree order (every thread gets the result).
__device__ __forceinline__ double block_sum(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int w = NT / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

__device__ __forceinline__ float block_max(float v, float* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int w = NT / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + w]);
    __syncthreads();
  }
  const float r = red[0];
  __syncthreads();
  return r;
}

// One CTA per row b: y = softmax(z[b]) over C classes (exp in f32, the sum in f64), then the three slices y[1:40],
// y[40:148], y[148:C] each divided by its own f64 sum -> out[b][c - 1] for c in 1..C-1.
__global__ void __launch_bounds__(NT) k_ope_softmax(int B, int C, const float* __restrict__ z, float* __restrict__ out) {
  __shared__ double red[NT];
  __shared__ float redf[NT];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (b >= B) return;
  const float* zr = z + (int64_t)b * C;
  float* o = out + (int64_t)b * (C - 1);
  float m = -INFINITY;
  for (int c = tid; c < C; c += NT) m = fmaxf(m, zr[c]);
  m = block_max(m, redf);
  double s = 0.0;
  for (int c = tid; c < C; c += NT) s += (double)expf(zr[c] - m);
  s = block_sum(s, red);
  double s1 = 0.0, s2 = 0.0, s3 = 0.0;
  for (int c = 1 + tid; c < C; c += NT) {
    const float y = (float)((double)expf(zr[c] - m) / s);
    o[c - 1] = y;
    if (c < 40) s1 += (double)y;
    else if (c < 148) s2 += (double)y;
    else s3 += (double)y;
  }
  s1 = block_sum(s1, red);
  s2 = block_sum(s2, red);
  s3 = block_sum(s3, red);
  for (int c = 1 + tid; c < C; c += NT) o[c - 1] = (float)((double)o[c - 1] / (c < 40 ? s1 : (c < 148 ? s2 : s3)));
}

// The per-step gather, one warp per row b, column t of the [T, B] buffers:
//   pol[t][b]  = the policy's probability of the offline action off[b]: probs[b][off] (logits == 0), or the softmax of
//                the logits row at off (exp in f32 after the row max, the sum in f64);
//   beh[t][b]  = block[b][block_col(layer, off[b])], the behaviour probability of the offline action;
//   val[t][b]  = values[b][own[b]] (per_action), or values[b];
//   rew[t][b]  = reward[b];  offr[t][b] = off_reward[b].
// A device-side action outside [0, A) gives NaN in the columns that index with it.
__global__ void __launch_bounds__(NT) k_ope_step(int t, int B, int A, int C, int layer, const float* __restrict__ probs,
                                                 int logits, const int32_t* __restrict__ off,
                                                 const float* __restrict__ block, const int32_t* __restrict__ own,
                                                 const float* __restrict__ values, int per_action,
                                                 const double* __restrict__ reward, const double* __restrict__ off_reward,
                                                 float* __restrict__ pol, float* __restrict__ beh, float* __restrict__ val,
                                                 double* __restrict__ rew, double* __restrict__ offr) {
  const int lane = threadIdx.x & 31, b = blockIdx.x * (NT / 32) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int64_t o = (int64_t)t * B + b;
  const int a = off[b];
  const bool ok = a >= 0 && a < A;
  const float* row = probs + (int64_t)b * A;
  float p;
  if (!logits) {
    p = ok ? row[a] : NAN;
  } else {
    float m = -INFINITY;
    for (int c = lane; c < A; c += 32) m = fmaxf(m, row[c]);
    for (int w = 16; w > 0; w >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, w));
    double s = 0.0;
    for (int c = lane; c < A; c += 32) s += (double)expf(row[c] - m);
    for (int w = 16; w > 0; w >>= 1) s += __shfl_xor_sync(0xffffffffu, s, w);
    p = ok ? (float)((double)expf(row[a] - m) / s) : NAN;
  }
  if (lane != 0) return;
  pol[o] = p;
  beh[o] = ok ? block[(int64_t)b * (C - 1) + block_col(layer, a)] : NAN;
  if (per_action) {
    const int g = own[b];
    val[o] = (g >= 0 && g < A) ? values[(int64_t)b * A + g] : NAN;
  } else {
    val[o] = values[b];
  }
  rew[o] = reward[b];
  offr[o] = off_reward[b];
}

}  // namespace r4ope
