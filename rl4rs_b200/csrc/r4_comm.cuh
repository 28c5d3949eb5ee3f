// r4_comm.cuh -- the policy-gradient exchange of the data-parallel learner as ONE kernel over NVLink peer memory:
// local reduction of the per-CTA partial gradients, all-to-all push into every rank's inbox, flag hand-shake, fixed-order
// sum and the Adam update -- no NCCL call, no host round trip between the SGD steps of an epoch (SURVEY.md section 8e:
// "fuse behind the last backward kernel rather than bucket").  The reference has no counterpart (Ray object store).
//
// Memory (per rank, one cudaMalloc exported with cudaIpcGetMemHandle, opened by every peer):
//     inbox  f32 [2 parities][world][n]      rank s writes its reduced gradient into slot [parity][s] of EVERY rank
//     flags  u32 [2 parities][world][nblk]   ... and then, per 256-parameter block, the sequence number of the step
// One thread owns one parameter: it sums the partials, stores the value into the `world` inboxes (coalesced 128-byte
// remote stores), the block fences (system scope) and publishes its flag to every rank; then it waits for the `world`
// flags of ITS block on its own device, sums the inbox slots in rank order (identical on every rank, so the replicas
// stay bit-identical) and applies Adam.  Blocks are independent: no grid-wide barrier.  Two parities suffice: a rank
// can only reach step s+2 after it has seen every peer's flag of step s+1, which a peer publishes only after it has
// finished reading the inbox of step s.
#pragma once
#include "r4_ppo.cuh"

namespace r4comm {

constexpr int MAX_WORLD = 16;
constexpr int BLK = 256;

struct Peers {
  float* inbox[MAX_WORLD];        // peer r's inbox base (device pointers valid on THIS device)
  uint32_t* flags[MAX_WORLD];
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ float ld_relaxed_sys(const float* p) {
  float v; asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory"); return v;
}

// do_adam = 1: parameters updated in place (PPO epoch);  0: the summed gradient is written to `flat` (A2C: global-norm
// clipping needs the whole gradient first).  `seq` = 1-based global step count of this communicator.
__global__ void __launch_bounds__(BLK) k_exchange_adam(int n, int G, const float* __restrict__ partial, float* __restrict__ flat,
                                                       const float* __restrict__ stat_partial, float* __restrict__ stats_accum,
                                                       float stat_scale, Peers peers, int rank, int world, uint32_t seq,
                                                       int do_adam, float* __restrict__ prm, float* __restrict__ m,
                                                       float* __restrict__ v, int step, float lr, float b1, float b2, float eps) {
  const int i = blockIdx.x * BLK + threadIdx.x;
  const int nblk = gridDim.x;
  const uint32_t parity = seq & 1u;
  float s = 0.f;
  if (i < n) {
    for (int c = 0; c < G; ++c) s += partial[(size_t)c * n + i];
    const size_t slot = ((size_t)parity * world + rank) * n + i;
    for (int r = 0; r < world; ++r) peers.inbox[r][slot] = s;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x < world)
    st_release_sys(peers.flags[threadIdx.x] + ((size_t)parity * world + rank) * nblk + blockIdx.x, seq);
  if (threadIdx.x < world) {
    const uint32_t* f = peers.flags[rank] + ((size_t)parity * world + threadIdx.x) * nblk + blockIdx.x;
    while ((int32_t)(ld_acquire_sys(f) - seq) < 0) { }
  }
  __syncthreads();
  if (i < n) {
    float g = 0.f;
    const float* in = peers.inbox[rank] + (size_t)parity * world * n + i;
    for (int r = 0; r < world; ++r) g += ld_relaxed_sys(in + (size_t)r * n);
    if (flat) flat[i] = g;
    if (do_adam) {
      float p = prm[i], mi = m[i], vi = v[i];
      r4ppo::adam_update(g, p, mi, vi, step, lr, b1, b2, eps);
      prm[i] = p; m[i] = mi; v[i] = vi;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < 5 && stats_accum) {
    float a = 0.f;
    for (int c = 0; c < G; ++c) a += stat_partial[c * 5 + threadIdx.x];
    stats_accum[threadIdx.x] = fmaf(a, stat_scale, stats_accum[threadIdx.x]);   // one rounding, as k_dense_wgrad's Stats
  }
}

}  // namespace r4comm
