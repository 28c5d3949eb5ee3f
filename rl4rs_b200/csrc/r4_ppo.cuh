// r4_ppo.cuh -- K12: the policy the reference trains on this env and its learner, as CUDA kernels.
//
//   policy   MyMaskActionsModel (rl4rs/nets/rllib/rllib_mask_model.py:41-62): obs(256) -> FC 64 tanh ->
//            A logits + max(log(mask), float32.min); value head on the shared 64-d hidden.
//   act      SoftQ(T=1) exploration = sample from softmax(masked logits); argmax when explore = 0
//            (modelfree_train.py:398-402,412-414).
//   learner  RLlib 1.5 PPO surrogate loss (clip, clipped value loss, KL penalty, entropy) or A3C/A2C
//            summed loss, hand-derived backward, deterministic gradient reduction, Adam.
//
// Flat parameter layout (one buffer => ONE gradient all-reduce): w1[256,64] b1[64] w2[64,A] b2[A] wv[64] bv[1].
// The network is tiny (34 973 parameters at A = 284): the kernels are latency-bound, so the design goal is
// few launches (2 per SGD step) and determinism (per-CTA partial gradients summed in fixed order).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace r4ppo {

constexpr int OBS = 256, HID = 64, TS = 4;       // TS = samples per CTA tile (small: the kernels are latency-bound,
                                                 // so a 256-sample minibatch should spread over 64 SMs, not 16)
constexpr int SPG = TS / 4;                      // samples per thread group in the first layer
constexpr int NT = 256;
constexpr float FLOAT_MIN = -3.402823466e+38f;

struct Layout {
  int A, o_w1, o_b1, o_w2, o_b2, o_wv, o_bv, n;
};
__host__ __device__ inline Layout make_layout(int A) {
  Layout L;
  L.A = A; L.o_w1 = 0; L.o_b1 = OBS * HID; L.o_w2 = L.o_b1 + HID; L.o_b2 = L.o_w2 + HID * A;
  L.o_wv = L.o_b2 + A; L.o_bv = L.o_wv + HID; L.n = L.o_bv + 1;
  return L;
}

__device__ __forceinline__ float warp_max(float v) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull; return x ^ (x >> 31);
}

// Forward of one tile of TS samples (rows given by src index): fills h_s[TS][HID], lg_s[TS][A]
// (masked logits), val_s[TS].  obs_s[TS][OBS] is loaded here.  All 256 threads participate.
template <bool WS>   // WS: w1p / w2p point to shared-memory copies of the two weight matrices
__device__ __forceinline__ float ldw(const float* p) { return WS ? *p : __ldg(p); }

template <bool WS>
__device__ inline void forward_tile(const Layout& L, const float* __restrict__ prm, const float* w1p, const float* w2p,
                                    const float* __restrict__ obs, const uint8_t* __restrict__ mask, const int64_t* src,
                                    int nvalid, float* obs_s, float* h_s, float* lg_s, float* val_s) {
  const int tid = threadIdx.x;
  for (int i = tid; i < TS * OBS / 4; i += NT) {
    int s = i / (OBS / 4), k4 = i % (OBS / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (s < nvalid) v = __ldg(reinterpret_cast<const float4*>(obs + src[s] * OBS) + k4);
    reinterpret_cast<float4*>(obs_s)[i] = v;
  }
  __syncthreads();
  {  // h = tanh(obs W1 + b1): thread (j = tid%64, g = tid/64) -> samples SPG*g .. SPG*g+SPG-1
    const int j = tid & 63, g = tid >> 6;
    float acc[SPG];
#pragma unroll
    for (int i = 0; i < SPG; ++i) acc[i] = 0.f;
    const float* w = w1p + j;
#pragma unroll 8
    for (int k = 0; k < OBS; ++k) {
      float wk = ldw<WS>(w + k * HID);
#pragma unroll
      for (int i = 0; i < SPG; ++i) acc[i] = fmaf(obs_s[(SPG * g + i) * OBS + k], wk, acc[i]);
    }
    float b = __ldg(prm + L.o_b1 + j);
#pragma unroll
    for (int i = 0; i < SPG; ++i) h_s[(SPG * g + i) * HID + j] = tanhf(acc[i] + b);
  }
  __syncthreads();
  for (int col = tid; col < L.A; col += NT) {  // logits = h W2 + b2 + clamp(log(mask))
    float acc[TS];
#pragma unroll
    for (int s = 0; s < TS; ++s) acc[s] = 0.f;
    const float* w = w2p + col;
#pragma unroll 4
    for (int k = 0; k < HID; ++k) {
      float wk = ldw<WS>(w + (size_t)k * L.A);
#pragma unroll
      for (int s = 0; s < TS; ++s) acc[s] = fmaf(h_s[s * HID + k], wk, acc[s]);
    }
    float b = __ldg(prm + L.o_b2 + col);
#pragma unroll
    for (int s = 0; s < TS; ++s) {
      float m = (s < nvalid && mask[src[s] * L.A + col]) ? 0.f : FLOAT_MIN;   // log(1) = 0 / log(0) clamped
      lg_s[s * L.A + col] = acc[s] + b + m;
    }
  }
  if (tid < TS) {
    float v = __ldg(prm + L.o_bv);
    for (int k = 0; k < HID; ++k) v = fmaf(h_s[tid * HID + k], __ldg(prm + L.o_wv + k), v);
    val_s[tid] = v;
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// act: forward + sample / argmax; writes action, logp(action), value and the masked logits.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) k_policy_act(Layout L, const float* __restrict__ prm, const float* __restrict__ obs,
                                                   const uint8_t* __restrict__ mask, int B, int explore, uint64_t seed,
                                                   uint64_t counter, int32_t* __restrict__ action, float* __restrict__ logp,
                                                   float* __restrict__ value, float* __restrict__ logits_out) {
  extern __shared__ __align__(16) float sm[];
  float* obs_s = sm; float* h_s = obs_s + TS * OBS; float* lg_s = h_s + TS * HID; float* val_s = lg_s + TS * L.A;
  __shared__ int64_t src[TS];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int s0 = blockIdx.x * TS;
  const int nvalid = min(TS, B - s0);
  if (tid < TS) src[tid] = min(s0 + tid, B - 1);
  __syncthreads();
  forward_tile<false>(L, prm, prm + L.o_w1, prm + L.o_w2, obs, mask, src, nvalid, obs_s, h_s, lg_s, val_s);
  for (int s = warp; s < nvalid; s += NT / 32) {
    const float* lg = lg_s + s * L.A;
    float m = -INFINITY;
    for (int c = lane; c < L.A; c += 32) m = fmaxf(m, lg[c]);
    m = warp_max(m);
    float se = 0.f;
    for (int c = lane; c < L.A; c += 32) se += expf(lg[c] - m);
    se = warp_sum(se);
    const float lse = m + logf(se);
    int a = 0;
    if (explore) {
      // inverse CDF over the A probabilities with one counter-based uniform per row
      uint64_t r = splitmix64(seed ^ splitmix64(counter + (uint64_t)(s0 + s)));
      float u = (float)((r >> 40) + 0.5) * (1.0f / 16777216.0f) * se;      // in (0, sum)
      float run = 0.f; int found = -1;
      for (int c0 = 0; c0 < L.A && found < 0; c0 += 32) {
        int c = c0 + lane;
        float e = c < L.A ? expf(lg[c] - m) : 0.f;
        float incl = e;                                                   // inclusive scan in the warp
        for (int o = 1; o < 32; o <<= 1) { float t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        bool hit = (run + incl >= u) && e > 0.f;
        unsigned bal = __ballot_sync(0xffffffffu, hit);
        if (bal) found = c0 + __ffs(bal) - 1;
        run += __shfl_sync(0xffffffffu, incl, 31);
      }
      if (found < 0) {                                                     // rounding at the tail: last allowed id
        for (int c = L.A - 1; c >= 0; --c) if (lg[c] > -1e30f) { found = c; break; }
        if (found < 0) found = 0;
      }
      a = found;
    } else {
      float bv = -INFINITY; int bi = 0x7fffffff;
      for (int c = lane; c < L.A; c += 32) if (lg[c] > bv) { bv = lg[c]; bi = c; }
      for (int o = 16; o > 0; o >>= 1) {
        float v2 = __shfl_xor_sync(0xffffffffu, bv, o); int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
        if (v2 > bv || (v2 == bv && i2 < bi)) { bv = v2; bi = i2; }
      }
      a = bi;
    }
    if (lane == 0) {
      action[s0 + s] = a;
      logp[s0 + s] = lg[a] - lse;
      value[s0 + s] = val_s[s];
    }
    if (logits_out)
      for (int c = lane; c < L.A; c += 32) logits_out[(size_t)(s0 + s) * L.A + c] = lg[c];
  }
}

// ------------------------------------------------------------------------------------------------
// learner gradient.  mode 0 = PPO (mean over the n_samples of this call), mode 1 = A2C (sums).
// Samples are idx[0..n) into the rollout arrays (idx == nullptr: 0..n-1).  CTA c accumulates the
// gradient of its tiles in shared memory (each parameter element is owned by one thread) and writes it to
// partial[c, :]; r4 sums partials in fixed order (k_grad_reduce / k_adam) -> bitwise reproducible.
// ------------------------------------------------------------------------------------------------
struct LossHyper {
  int mode;
  float clip, vf_clip, vf_coeff, kl_coeff, ent_coeff, inv_n;
};

// The per-sample scalars of the loss, for both policies' gradient kernels (k_policy_grad, r4gauss::k_gauss_rows): from the
// sample's logp of the taken action, value, KL and entropy, the loss derivatives d/dlogp = ca, d/dkl = ckl,
// d/dentropy = -cent, d/dvalue = dv, and the statistics pl, vl, kl, ent, total.  old_logp and old_value are used in mode 0 only.
struct SampleLoss {
  float ca, ckl, cent, dv, pl, vl, kl, ent, total;
};
__device__ __forceinline__ SampleLoss sample_loss(const LossHyper& hp, float logp, float old_logp, float adv, float target,
                                                  float value, float old_value, float kl, float ent) {
  SampleLoss o;
  const float v = value, tg = target;
  o.ckl = 0.f; o.cent = hp.ent_coeff; o.kl = kl; o.ent = ent;
  if (hp.mode == 0) {
    const float ratio = expf(logp - old_logp);
    const float lo = 1.f - hp.clip, hi = 1.f + hp.clip;
    const float t1 = adv * ratio, t2 = adv * fminf(fmaxf(ratio, lo), hi);
    const float g2 = (ratio >= lo && ratio <= hi) ? adv : 0.f;
    const float g = t1 < t2 ? adv : (t2 < t1 ? g2 : 0.5f * (adv + g2));     // torch.min ties split evenly
    o.ca = -g * ratio * hp.inv_n;
    o.ckl = hp.kl_coeff * hp.inv_n;
    o.cent *= hp.inv_n;
    const float vo = old_value, d = v - vo;
    const float dcl = fminf(fmaxf(d, -hp.vf_clip), hp.vf_clip), vcl = vo + dcl;
    const float vf1 = (v - tg) * (v - tg), vf2 = (vcl - tg) * (vcl - tg);
    const float gv1 = 2.f * (v - tg), gv2 = (fabsf(d) <= hp.vf_clip) ? 2.f * (vcl - tg) : 0.f;
    const float gv = vf1 > vf2 ? gv1 : (vf2 > vf1 ? gv2 : 0.5f * (gv1 + gv2));
    o.dv = hp.vf_coeff * gv * hp.inv_n;
    o.pl = -fminf(t1, t2); o.vl = fmaxf(vf1, vf2);
  } else {
    o.ca = -adv;
    o.dv = hp.vf_coeff * (v - tg);
    o.pl = -logp * adv; o.vl = 0.5f * (v - tg) * (v - tg);
  }
  o.total = hp.mode == 0 ? (o.pl + hp.kl_coeff * kl + hp.vf_coeff * o.vl - hp.ent_coeff * ent)
                         : (o.pl + hp.vf_coeff * o.vl - hp.ent_coeff * ent);
  return o;
}

// SINGLE = true: the grid has exactly one tile per CTA (a PPO minibatch): no shared-memory gradient accumulator;
// instead both weight matrices are staged in shared memory once (136 KB) so every inner loop reads shared memory, and
// each gradient element is stored straight to this CTA's partial row by its owner thread.
template <bool SINGLE>
__global__ void __launch_bounds__(NT) k_policy_grad(Layout L, LossHyper hp, const float* __restrict__ prm,
                                                    const float* __restrict__ obs, const uint8_t* __restrict__ mask,
                                                    const int64_t* __restrict__ action, const float* __restrict__ old_logp,
                                                    const float* __restrict__ old_logits, const float* __restrict__ old_value,
                                                    const float* __restrict__ adv, const float* __restrict__ target,
                                                    const int64_t* __restrict__ idx, int n, float* __restrict__ partial,
                                                    float* __restrict__ stat_partial /*[grid,5]*/) {
  extern __shared__ __align__(16) float sm[];
  // Programmatic dependent launch (r4_ppo_epoch launches its 288 kernels per epoch with
  // cudaLaunchAttributeProgrammaticStreamSerialization): let the next kernel of the chain be scheduled while this one runs, and
  // do not touch global memory before the previous one (the optimiser step that wrote `prm` and read `partial`) has completed.
  // Both are no-ops for a plain launch.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  float* g_s = sm;                              // !SINGLE: [L.n] gradient accumulator; SINGLE: w1 | w2 copies
  const int head = SINGLE ? (OBS * HID + ((HID * L.A + 3) & ~3)) : ((L.n + 3) & ~3);
  float* obs_s = g_s + head;
  float* h_s = obs_s + TS * OBS;
  float* lg_s = h_s + TS * HID;                 // logits -> logp_all -> dlogits
  float* val_s = lg_s + TS * L.A;
  float* dpre_s = val_s + TS;                   // [TS][HID]
  float* dv_s = dpre_s + TS * HID;              // [TS]
  __shared__ int64_t src[TS];
  __shared__ float stat_s[5];
  __shared__ float stat_t[TS][5];               // per-sample terms of this tile, summed in sample order (deterministic)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float* gout = partial + (size_t)blockIdx.x * L.n;
  const float* w1p = prm + L.o_w1;
  const float* w2p = prm + L.o_w2;
  __shared__ uint64_t wbar;
  if (SINGLE) {
    // Both weight matrices (64 KB + 71 KB) come in through the bulk-copy engine: ONE thread issues two cp.async.bulk and
    // everybody waits on the mbarrier right before the first use.  (ncu, round 2: the per-thread ld -> st.shared copy
    // loop this replaces was 38 % of the kernel's 36 us -- 71 dependent L2 round trips per thread.)
    float* w2s = g_s + OBS * HID;
    if (tid == 0) {
      const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&wbar);
      const uint32_t b1 = OBS * HID * 4, b2 = (uint32_t)(HID * L.A * 4);
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(mb) : "memory");
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mb), "r"(b1 + b2) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   :: "r"((uint32_t)__cvta_generic_to_shared(g_s)), "l"(prm + L.o_w1), "r"(b1), "r"(mb) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   :: "r"((uint32_t)__cvta_generic_to_shared(w2s)), "l"(prm + L.o_w2), "r"(b2), "r"(mb) : "memory");
    }
    w1p = g_s; w2p = w2s;
  } else {
    for (int i = tid; i < L.n; i += NT) g_s[i] = 0.f;
  }
  if (tid < 5) stat_s[tid] = 0.f;
  const int ntiles = (n + TS - 1) / TS;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int s0 = tile * TS;
    const int nvalid = min(TS, n - s0);
    __syncthreads();
    if (tid < TS) { int i = min(s0 + tid, n - 1); src[tid] = idx ? idx[i] : (int64_t)i; }
    __syncthreads();
    if (SINGLE) {                                  // the weights have landed (the barrier was initialised before the __syncthreads)
      const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&wbar);
      asm volatile("{\n\t.reg .pred p;\n\tPG_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t@p bra PG_DONE;\n\tbra PG_WAIT;\n\tPG_DONE:\n\t}\n"
                   :: "r"(mb) : "memory");
    }
    forward_tile<SINGLE>(L, prm, w1p, w2p, obs, mask, src, nvalid, obs_s, h_s, lg_s, val_s);
    // ---- per-sample loss derivatives: one warp per sample ----
    for (int s = warp; s < TS; s += NT / 32) {
      float* lg = lg_s + s * L.A;
      if (s >= nvalid) {
        for (int c = lane; c < L.A; c += 32) lg[c] = 0.f;
        if (lane == 0) { dv_s[s] = 0.f; for (int k = 0; k < 5; ++k) stat_t[s][k] = 0.f; }
        continue;
      }
      const int64_t r = src[s];
      float m = -INFINITY, mo = -INFINITY;
      const float* ol = old_logits + r * L.A;
      for (int c = lane; c < L.A; c += 32) { m = fmaxf(m, lg[c]); mo = fmaxf(mo, __ldg(ol + c)); }
      m = warp_max(m); mo = warp_max(mo);
      float se = 0.f, so = 0.f;
      for (int c = lane; c < L.A; c += 32) { se += expf(lg[c] - m); so += expf(__ldg(ol + c) - mo); }
      se = warp_sum(se); so = warp_sum(so);
      const float lse = m + logf(se), lso = mo + logf(so);
      const int a = (int)action[r];
      const float logp = lg[a] - lse;
      const float advv = adv[r], tg = target[r], v = val_s[s];
      float kl = 0.f, ent = 0.f;
      for (int c = lane; c < L.A; c += 32) {
        float lp = lg[c] - lse, lpo = __ldg(ol + c) - lso;
        float p = expf(lp), po = expf(lpo);
        if (po > 0.f) kl += po * (lpo - lp);
        if (p > 0.f) ent -= p * lp;
      }
      kl = warp_sum(kl); ent = warp_sum(ent);
      const SampleLoss o = sample_loss(hp, logp, hp.mode == 0 ? old_logp[r] : 0.f, advv, tg, v,
                                       hp.mode == 0 ? old_value[r] : 0.f, kl, ent);
      // dlogits_j = ca (delta_ja - p_j) + ckl (p_j - p_old_j) + cent p_j (logp_j + H)
      for (int c = lane; c < L.A; c += 32) {
        float lp = lg[c] - lse, p = expf(lp), po = expf(__ldg(ol + c) - lso);
        float dz = o.ca * ((c == a ? 1.f : 0.f) - p) + o.ckl * (p - po);
        if (o.cent != 0.f && p > 0.f) dz += o.cent * p * (lp + ent);
        lg[c] = dz;
      }
      if (lane == 0) {
        dv_s[s] = o.dv;
        stat_t[s][0] = o.pl; stat_t[s][1] = o.vl; stat_t[s][2] = o.kl; stat_t[s][3] = o.ent; stat_t[s][4] = o.total;
      }
    }
    __syncthreads();
    if (tid < 5) { float a = stat_s[tid]; for (int k = 0; k < TS; ++k) a += stat_t[k][tid]; stat_s[tid] = a; }
    // ---- backward ----
    for (int col = tid; col < L.A; col += NT) {          // dW2[k][col], db2[col]
      float d[TS];
      float sb = 0.f;
#pragma unroll
      for (int s = 0; s < TS; ++s) { d[s] = lg_s[s * L.A + col]; sb += d[s]; }
      if (SINGLE) gout[L.o_b2 + col] = sb; else g_s[L.o_b2 + col] += sb;
      for (int k = 0; k < HID; ++k) {
        float acc = 0.f;
#pragma unroll
        for (int s = 0; s < TS; ++s) acc = fmaf(h_s[s * HID + k], d[s], acc);
        if (SINGLE) gout[L.o_w2 + k * L.A + col] = acc; else g_s[L.o_w2 + k * L.A + col] += acc;
      }
    }
    // dh[s][k] = sum_col dlog[s][col] W2[k][col] + dv[s] wv[k];  dpre = dh (1 - h^2): warp per (s, k-range)
    for (int p = warp; p < TS * HID / 8; p += NT / 32) {  // 8 k's per pass
      const int s = p / (HID / 8), k0 = (p % (HID / 8)) * 8;
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
      for (int c = lane; c < L.A; c += 32) {
        float dz = lg_s[s * L.A + c];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(dz, ldw<SINGLE>(w2p + (size_t)(k0 + i) * L.A + c), acc[i]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = warp_sum(acc[i]);
      if (lane < 8) {
        float a = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) if (lane == i) a = acc[i];
        const int k = k0 + lane;
        float hv = h_s[s * HID + k];
        dpre_s[s * HID + k] = (a + dv_s[s] * __ldg(prm + L.o_wv + k)) * (1.f - hv * hv);
      }
    }
    __syncthreads();
    {  // dW1[i][k] (+ b1, wv, bv): thread (k = tid%64, ig = tid/64 -> 64 inputs)
      const int k = tid & 63, ig = tid >> 6;
      float dp[TS];
#pragma unroll
      for (int s = 0; s < TS; ++s) dp[s] = dpre_s[s * HID + k];
      for (int i = ig * 64; i < ig * 64 + 64; ++i) {
        float acc = 0.f;
#pragma unroll
        for (int s = 0; s < TS; ++s) acc = fmaf(obs_s[s * OBS + i], dp[s], acc);
        if (SINGLE) gout[L.o_w1 + i * HID + k] = acc; else g_s[L.o_w1 + i * HID + k] += acc;
      }
      if (ig == 0) {
        float sb = 0.f, sw = 0.f;
#pragma unroll
        for (int s = 0; s < TS; ++s) { sb += dp[s]; sw = fmaf(h_s[s * HID + k], dv_s[s], sw); }
        if (SINGLE) { gout[L.o_b1 + k] = sb; gout[L.o_wv + k] = sw; } else { g_s[L.o_b1 + k] += sb; g_s[L.o_wv + k] += sw; }
      }
      if (tid == 0) {
        float sv = 0.f;
#pragma unroll
        for (int s = 0; s < TS; ++s) sv += dv_s[s];
        if (SINGLE) gout[L.o_bv] = sv; else g_s[L.o_bv] += sv;
      }
    }
  }
  __syncthreads();
  if (!SINGLE) for (int i = tid; i < L.n; i += NT) gout[i] = g_s[i];
  if (tid < 5) stat_partial[blockIdx.x * 5 + tid] = stat_s[tid];
}

// flat[i] = sum_c partial[c][i]  (fixed order); stats_accum[j] += sum_c stat_partial[c][j] * stat_scale
__global__ void k_grad_reduce(int n, int G, const float* __restrict__ partial, float* __restrict__ flat,
                              const float* __restrict__ stat_partial, float* __restrict__ stats_accum, float stat_scale) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    float s = 0.f;
    for (int c = 0; c < G; ++c) s += partial[(size_t)c * n + i];
    flat[i] = s;
  }
  if (blockIdx.x == 0 && threadIdx.x < 5 && stats_accum) {
    float s = 0.f;
    for (int c = 0; c < G; ++c) s += stat_partial[c * 5 + threadIdx.x];
    stats_accum[threadIdx.x] += s * stat_scale;
  }
}

// torch.optim.Adam (no weight decay, no amsgrad) on one parameter; shared by k_adam and k_reduce_adam so that the
// fused and the two-kernel paths round identically.
__device__ __forceinline__ void adam_update(float g, float& p, float& mi_io, float& vi_io, int step, float lr, float b1,
                                            float b2, float eps) {
  float mi = b1 * mi_io + (1.f - b1) * g;
  float vi = b2 * vi_io + (1.f - b2) * g * g;
  mi_io = mi; vi_io = vi;
  float bc1 = 1.f - powf(b1, (float)step), bc2 = 1.f - powf(b2, (float)step);
  float denom = sqrtf(vi) / sqrtf(bc2) + eps;
  p -= (lr / bc1) * (mi / denom);
}

// Adam with optional global-norm clipping (clip <= 0: off).
// grad_scale multiplies the gradient first (1/world after a SUM all-reduce).  step is the 1-based count.
__global__ void k_adam(int n, float* __restrict__ prm, const float* __restrict__ grad, float* __restrict__ m,
                       float* __restrict__ v, int step, float lr, float b1, float b2, float eps, float grad_scale,
                       const float* __restrict__ gnorm_sq /*[1] or null*/, float clip) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float g = grad[i] * grad_scale;
  if (gnorm_sq && clip > 0.f) {
    float gn = sqrtf(gnorm_sq[0]) * grad_scale;
    float c = clip / (gn + 1e-6f);                       // torch clip_grad_norm_
    if (c < 1.f) g *= c;
  }
  float p = prm[i], mi = m[i], vi = v[i];
  adam_update(g, p, mi, vi, step, lr, b1, b2, eps);
  prm[i] = p; m[i] = mi; v[i] = vi;
}

// k_grad_reduce + k_adam (no clipping, grad_scale 1) in one launch: the single-GPU PPO epoch has nothing between them.
__global__ void k_reduce_adam(int n, int G, const float* __restrict__ partial, float* __restrict__ flat,
                              const float* __restrict__ stat_partial, float* __restrict__ stats_accum, float stat_scale,
                              float* __restrict__ prm, float* __restrict__ m, float* __restrict__ v, int step, float lr,
                              float b1, float b2, float eps) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // see k_policy_grad
  asm volatile("griddepcontrol.wait;" ::: "memory");
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    // fixed order c = 0, 1, ... (bitwise reproducible), 16 loads in flight: with the plain loop the 64 partials of a PPO
    // minibatch were 64 L2 round trips taken four at a time
    float s = 0.f;
    int c = 0;
    for (; c + 16 <= G; c += 16) {
      float v[16];
#pragma unroll
      for (int u = 0; u < 16; ++u) v[u] = partial[(size_t)(c + u) * n + i];
#pragma unroll
      for (int u = 0; u < 16; ++u) s += v[u];
    }
    for (; c < G; ++c) s += partial[(size_t)c * n + i];
    flat[i] = s;
    float g = s * 1.0f;
    float p = prm[i], mi = m[i], vi = v[i];
    adam_update(g, p, mi, vi, step, lr, b1, b2, eps);
    prm[i] = p; m[i] = mi; v[i] = vi;
  }
  if (blockIdx.x == 0 && threadIdx.x < 5 && stats_accum) {
    float s = 0.f;
    for (int c = 0; c < G; ++c) s += stat_partial[c * 5 + threadIdx.x];
    stats_accum[threadIdx.x] += s * stat_scale;
  }
}

// GAE over complete episodes (RLlib compute_advantages with a zero bootstrap value): one thread = one env row, the same
// recursion in the same order as the torch loop it replaces (45 tiny launches per iteration at T = 9):
//     delta_t = r_t + gamma v_{t+1} - v_t ;  adv_t = delta_t + gamma lambda adv_{t+1} ;  target_t = adv_t + v_t
__global__ void k_gae(int T, int B, const float* __restrict__ reward, const float* __restrict__ value, float gamma, float gamma_lam,
                      float* __restrict__ adv, float* __restrict__ target) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float last = 0.f, nv = 0.f;
  for (int t = T - 1; t >= 0; --t) {
    const float v = value[(size_t)t * B + b];
    const float delta = __fadd_rn(__fadd_rn(reward[(size_t)t * B + b], __fmul_rn(gamma, nv)), -v);
    last = __fadd_rn(delta, __fmul_rn(gamma_lam, last));
    adv[(size_t)t * B + b] = last;
    target[(size_t)t * B + b] = __fadd_rn(last, v);
    nv = v;
  }
}

__global__ void k_sumsq(int n, const float* __restrict__ x, float* __restrict__ out) {
  __shared__ float red[32];
  float s = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) s += x[i] * x[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    s = warp_sum(s);
    if (threadIdx.x == 0) atomicAdd(out, s);
  }
}

}  // namespace r4ppo
