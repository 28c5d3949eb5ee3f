// r4_learn.cu -- host side of the learner entry points of include/rl4rs_b200.h: PPO / A2C, the peer-memory gradient
// exchange, the Gaussian policy, DDPG / TD3, RAINBOW, batch RL and the simulator trainer.  Stateless: every call enqueues
// its kernels on the caller's stream through r4h::launch, which counts them (r4_learner_launch_count).  See DESIGN.md.
#include "../../include/rl4rs_b200.h"
#include "r4_host.h"
#include "r4_ppo.cuh"
#include "r4_comm.cuh"
#include "r4_gauss.cuh"
#include "r4_ddpg.cuh"
#include "r4_rainbow.cuh"
#include "r4_batchrl.cuh"
#include "r4_simtrain.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

using namespace r4h;

// Dynamic shared memory starts at one offset for every kernel of a module, aligned for the module's most-aligned
// extern __shared__ array.  The env module's tensor-core kernels align theirs to 1024 bytes; the learner kernels were
// tuned at that alignment, and at 16 bytes k_policy_grad (whose weights arrive by bulk copy) runs about 6 % slower on an
// H100.  This never-launched kernel keeps a 1024-byte-aligned array in use, so the learner module keeps the alignment.
extern __shared__ __align__(1024) uint8_t r4_learn_smem_align[];
__global__ void r4_learn_smem_align_anchor() { r4_learn_smem_align[threadIdx.x] = 0; }

struct r4_comm {
  int rank = 0, world = 1, n = 0, nblk = 0, device = 0;
  void* base = nullptr;
  size_t inbox_bytes = 0, bytes = 0;
  r4comm::Peers peers{};
  std::vector<void*> opened;
  uint32_t seq = 0;
  bool ready = false;
};

extern "C" {

int64_t r4_learner_launch_count(void) {
  int64_t n = 0;
  for (const auto& c : g_launches) n += c.load(std::memory_order_relaxed);
  return n;
}

// ---- K12: policy / learner kernels (stateless) ---------------------------------------------------
int r4_policy_num_params(int action_size) { return (action_size < 2 || action_size > 512) ? -1 : r4ppo::make_layout(action_size).n; }

int r4_policy_act(const float* params, const float* obs, const uint8_t* mask, int n, int action_size, int explore,
                  uint64_t seed, uint64_t counter, int32_t* action, float* logp, float* value, float* logits,
                  void* stream) {
  if (!params || !obs || !mask || !action || !logp || !value || n < 1 || action_size < 2 || action_size > 512)
    return fail(R4_ERR_ARG, "r4_policy_act: bad argument");
  r4ppo::Layout L = r4ppo::make_layout(action_size);
  size_t smem = (size_t)(r4ppo::TS * r4ppo::OBS + r4ppo::TS * r4ppo::HID + r4ppo::TS * action_size + r4ppo::TS) * 4;
  return launch(FAM_ONLINE, "k_policy_act", r4ppo::k_policy_act, (n + r4ppo::TS - 1) / r4ppo::TS, r4ppo::NT, smem, S(stream),
                false, L, params, obs, mask, n, explore, seed, counter, action, logp, value, logits);
}

static int policy_grad_impl(int mode, const float* params, const float* obs, const uint8_t* mask, const int64_t* action,
                            const float* old_logp, const float* old_logits, const float* old_value, const float* adv,
                            const float* target, const int64_t* idx, int n, int action_size, float clip, float vf_clip,
                            float vf_coeff, float kl_coeff, float ent_coeff, float inv_n, float* scratch, int G,
                            float* flat_grad, float* stats_accum, float stat_scale, void* stream, bool reduce, bool pdl = false) {
  if (!params || !obs || !mask || !action || !old_logits || !adv || !target || !scratch || !flat_grad || n < 1 ||
      G < 1 || action_size < 2 || action_size > 512 || (mode == 0 && (!old_logp || !old_value)))
    return fail(R4_ERR_ARG, "r4_policy_grad: bad argument");
  r4ppo::Layout L = r4ppo::make_layout(action_size);
  r4ppo::LossHyper hp{mode, clip, vf_clip, vf_coeff, kl_coeff, ent_coeff, inv_n};
  const bool single = ((n + r4ppo::TS - 1) / r4ppo::TS) == G;      // one tile per CTA (PPO minibatch)
  const size_t head = single ? (size_t)(r4ppo::OBS * r4ppo::HID + ((r4ppo::HID * action_size + 3) & ~3)) : (size_t)((L.n + 3) & ~3);
  size_t smem = (head + r4ppo::TS * r4ppo::OBS + 2 * r4ppo::TS * r4ppo::HID + r4ppo::TS * action_size + 2 * r4ppo::TS) * 4;
  if (smem > 226 * 1024) return fail(R4_ERR_ARG, "r4_policy_grad: action_size too large for the shared-memory layout");
  float* partial = scratch;
  float* stat_partial = scratch + (size_t)G * L.n;
  auto grad = [&](auto kernel, bool chained) {
    return launch(FAM_ONLINE, "k_policy_grad", kernel, G, r4ppo::NT, smem, S(stream), chained, L, hp, params, obs, mask, action,
                  old_logp, old_logits, old_value, adv, target, idx, n, partial, stat_partial);
  };
  // programmatic dependent launch only for the one-tile-per-CTA form of the fused epoch (r4_ppo_epoch)
  if (int rc = single ? grad(r4ppo::k_policy_grad<true>, pdl) : grad(r4ppo::k_policy_grad<false>, false)) return rc;
  if (!reduce) return R4_OK;       // the caller folds the reduction into its optimiser kernel (r4_ppo_epoch)
  return launch(FAM_ONLINE, "k_grad_reduce", r4ppo::k_grad_reduce, (L.n + 255) / 256, 256, 0, S(stream), false, L.n, G, partial,
                flat_grad, stat_partial, stats_accum, stat_scale);
}

int r4_policy_grad(int mode, const float* params, const float* obs, const uint8_t* mask, const int64_t* action,
                   const float* old_logp, const float* old_logits, const float* old_value, const float* adv,
                   const float* target, const int64_t* idx, int n, int action_size, float clip, float vf_clip,
                   float vf_coeff, float kl_coeff, float ent_coeff, float inv_n, float* scratch, int G,
                   float* flat_grad, float* stats_accum, float stat_scale, void* stream) {
  return policy_grad_impl(mode, params, obs, mask, action, old_logp, old_logits, old_value, adv, target, idx, n, action_size,
                          clip, vf_clip, vf_coeff, kl_coeff, ent_coeff, inv_n, scratch, G, flat_grad, stats_accum, stat_scale,
                          stream, true);
}

int r4_gae(const float* reward, const float* value, int T, int B, float gamma, float gamma_lambda, float* adv, float* target, void* stream) {
  if (!reward || !value || !adv || !target || T < 1 || B < 1) return fail(R4_ERR_ARG, "r4_gae: bad argument");
  return launch(FAM_ONLINE, "k_gae", r4ppo::k_gae, (B + 255) / 256, 256, 0, S(stream), false, T, B, reward, value, gamma,
                gamma_lambda, adv, target);
}

int r4_adam_step(float* params, const float* grad, float* m, float* v, int n, int step, float lr, float beta1,
                 float beta2, float eps, float grad_scale, float clip, float* norm_scratch, void* stream) {
  if (!params || !grad || !m || !v || n < 1 || step < 1 || (clip > 0.f && !norm_scratch))
    return fail(R4_ERR_ARG, "r4_adam_step: bad argument");
  if (clip > 0.f) {
    cudaMemsetAsync(norm_scratch, 0, 4, S(stream));
    if (int rc = launch(FAM_ONLINE, "k_sumsq", r4ppo::k_sumsq, 32, 256, 0, S(stream), false, n, grad, norm_scratch)) return rc;
  }
  return launch(FAM_ONLINE, "k_adam", r4ppo::k_adam, (n + 255) / 256, 256, 0, S(stream), false, n, params, grad, m, v, step, lr,
                beta1, beta2, eps, grad_scale, clip > 0.f ? norm_scratch : nullptr, clip);
}

int r4_ppo_epoch(float* params, const float* obs, const uint8_t* mask, const int64_t* action, const float* old_logp,
                 const float* old_logits, const float* old_value, const float* adv, const float* target,
                 const int64_t* perm, int n, int mb, int action_size, float clip, float vf_clip, float vf_coeff,
                 float kl_coeff, float ent_coeff, float* scratch, float* flat_grad, float* stats_accum, float* m,
                 float* v, int step0, float lr, float beta1, float beta2, float eps, float grad_clip,
                 float* norm_scratch, void* stream) {
  if (!perm || n < 1 || mb < 1 || mb > n || step0 < 0) return fail(R4_ERR_ARG, "r4_ppo_epoch: bad argument");
  const int G = std::max(1, std::min((mb + r4ppo::TS - 1) / r4ppo::TS, sm_count()));
  const int np = r4ppo::make_layout(action_size).n;
  int steps = 0;
  const bool fused = !(grad_clip > 0.f);      // global-norm clipping needs the reduced gradient first
  if (!params || !m || !v || !flat_grad || !scratch) return fail(R4_ERR_ARG, "r4_ppo_epoch: bad argument");
  for (int s = 0; s + mb <= n; s += mb, ++steps) {
    // programmatic dependent launch for the grad / optimiser chain of the fused epoch
    int rc = policy_grad_impl(0, params, obs, mask, action, old_logp, old_logits, old_value, adv, target, perm + s, mb,
                              action_size, clip, vf_clip, vf_coeff, kl_coeff, ent_coeff, 1.0f / mb, scratch, G, flat_grad,
                              stats_accum, 1.0f / mb, stream, !fused, fused);
    if (rc) return rc;
    if (fused)
      rc = launch(FAM_ONLINE, "k_reduce_adam", r4ppo::k_reduce_adam, (np + 255) / 256, 256, 0, S(stream), true, np, G, scratch,
                  flat_grad, scratch + (size_t)G * np, stats_accum, 1.0f / mb, params, m, v, step0 + steps + 1, lr, beta1, beta2,
                  eps);
    else
      rc = r4_adam_step(params, flat_grad, m, v, np, step0 + steps + 1, lr, beta1, beta2, eps, 1.0f, grad_clip, norm_scratch, stream);
    if (rc) return rc;
  }
  return steps;
}

// ---- data-parallel learner: peer-memory gradient exchange (r4_comm.cuh) -------------------------------------
int r4_comm_create(int rank, int world, int n_params, r4_comm** out) {
  if (!out || world < 1 || world > r4comm::MAX_WORLD || rank < 0 || rank >= world || n_params < 1)
    return fail(R4_ERR_ARG, "r4_comm_create: bad argument (world <= 16)");
  *out = nullptr;
  r4_comm* c = new r4_comm();
  c->rank = rank; c->world = world; c->n = n_params; c->nblk = (n_params + r4comm::BLK - 1) / r4comm::BLK;
  cudaGetDevice(&c->device);
  c->inbox_bytes = (((size_t)2 * world * n_params * 4) + 255) & ~(size_t)255;
  c->bytes = c->inbox_bytes + (size_t)2 * world * c->nblk * 4;
  cudaError_t st = cudaMalloc(&c->base, c->bytes);
  if (st == cudaSuccess) st = cudaMemset(c->base, 0, c->bytes);
  if (st == cudaSuccess) st = cudaDeviceSynchronize();
  if (st != cudaSuccess) { if (c->base) cudaFree(c->base); delete c; return fail(R4_ERR_CUDA, std::string("r4_comm_create: ") + cudaGetErrorString(st)); }
  c->peers.inbox[rank] = reinterpret_cast<float*>(c->base);
  c->peers.flags[rank] = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(c->base) + c->inbox_bytes);
  c->ready = world == 1;
  *out = c;
  return R4_OK;
}

int r4_comm_handle(r4_comm* c, void* handle_out_64) {
  if (!c || !handle_out_64) return fail(R4_ERR_ARG, "r4_comm_handle: null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  cudaIpcMemHandle_t h;
  cudaError_t st = cudaIpcGetMemHandle(&h, c->base);
  if (st != cudaSuccess) return fail(R4_ERR_CUDA, std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(st));
  memcpy(handle_out_64, &h, 64);
  return R4_OK;
}

int r4_comm_open(r4_comm* c, const void* handles, int n_handles) {
  if (!c || !handles || n_handles != c->world) return fail(R4_ERR_ARG, "r4_comm_open: need one handle per rank");
  cudaSetDevice(c->device);
  for (int r = 0; r < c->world; ++r) {
    if (r == c->rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, reinterpret_cast<const uint8_t*>(handles) + (size_t)r * 64, 64);
    void* p = nullptr;
    cudaError_t st = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (st != cudaSuccess) {
      cudaGetLastError();
      return fail(R4_ERR_CUDA, std::string("cudaIpcOpenMemHandle(rank ") + std::to_string(r) + "): " + cudaGetErrorString(st));
    }
    c->opened.push_back(p);
    c->peers.inbox[r] = reinterpret_cast<float*>(p);
    c->peers.flags[r] = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(p) + c->inbox_bytes);
  }
  c->ready = true;
  return R4_OK;
}

void r4_comm_destroy(r4_comm* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  for (void* p : c->opened) cudaIpcCloseMemHandle(p);
  if (c->base) cudaFree(c->base);
  delete c;
}

int r4_policy_grad_partial(int mode, const float* params, const float* obs, const uint8_t* mask, const int64_t* action,
                           const float* old_logp, const float* old_logits, const float* old_value, const float* adv,
                           const float* target, const int64_t* idx, int n, int action_size, float clip, float vf_clip,
                           float vf_coeff, float kl_coeff, float ent_coeff, float inv_n, float* scratch, int G,
                           void* stream) {
  return policy_grad_impl(mode, params, obs, mask, action, old_logp, old_logits, old_value, adv, target, idx, n, action_size,
                          clip, vf_clip, vf_coeff, kl_coeff, ent_coeff, inv_n, scratch, G, scratch /*unused*/, nullptr, 0.f,
                          stream, false);
}

static int exchange_launch(r4_comm* c, const float* scratch, int G, int np, float* flat, float* stats_accum, float stat_scale,
                           int do_adam, float* params, float* m, float* v, int step, float lr, float b1, float b2, float eps,
                           void* stream) {
  if (!c->ready) return fail(R4_ERR_STATE, "r4_comm: open the peers' handles first (r4_comm_open)");
  if (np != c->n) return fail(R4_ERR_ARG, "r4_comm: parameter count differs from the communicator's");
  ++c->seq;
  return launch(FAM_ONLINE, "k_exchange_adam", r4comm::k_exchange_adam, c->nblk, r4comm::BLK, 0, S(stream), false, np, G, scratch,
                flat, scratch + (size_t)G * np, stats_accum, stat_scale, c->peers, c->rank, c->world, c->seq, do_adam, params, m,
                v, step, lr, b1, b2, eps);
}

int r4_grad_exchange(r4_comm* c, const float* scratch, int G, int action_size, float* flat_grad, float* stats_accum,
                     float stat_scale, void* stream) {
  return r4_grad_exchange_n(c, scratch, G, r4ppo::make_layout(action_size).n, flat_grad, stats_accum, stat_scale, stream);
}

int r4_ppo_epoch_dist(r4_comm* c, float* params, const float* obs, const uint8_t* mask, const int64_t* action,
                      const float* old_logp, const float* old_logits, const float* old_value, const float* adv,
                      const float* target, const int64_t* perm, int n, int mb, int action_size, float clip,
                      float vf_clip, float vf_coeff, float kl_coeff, float ent_coeff, float* scratch, float* flat_grad,
                      float* stats_accum, float* m, float* v, int step0, float lr, float beta1, float beta2, float eps,
                      void* stream) {
  if (!c || !params || !perm || !m || !v || !scratch || n < 1 || mb < 1 || mb > n || step0 < 0)
    return fail(R4_ERR_ARG, "r4_ppo_epoch_dist: bad argument");
  const int G = std::max(1, std::min((mb + r4ppo::TS - 1) / r4ppo::TS, sm_count()));
  const int np = r4ppo::make_layout(action_size).n;
  const float inv = 1.0f / ((float)mb * (float)c->world);
  int steps = 0;
  for (int s = 0; s + mb <= n; s += mb, ++steps) {
    int rc = policy_grad_impl(0, params, obs, mask, action, old_logp, old_logits, old_value, adv, target, perm + s, mb,
                              action_size, clip, vf_clip, vf_coeff, kl_coeff, ent_coeff, inv, scratch, G, scratch, nullptr, 0.f,
                              stream, false);
    if (rc) return rc;
    // statistics stay per-rank means over this rank's mb samples (the trainer averages them over the ranks)
    rc = exchange_launch(c, scratch, G, np, flat_grad, stats_accum, 1.0f / (float)mb, 1, params, m, v, step0 + steps + 1, lr, beta1, beta2,
                         eps, stream);
    if (rc) return rc;
  }
  return steps;
}

int r4_grad_exchange_n(r4_comm* c, const float* partial, int G, int n_params, float* flat_grad, float* stats_accum,
                       float stat_scale, void* stream) {
  if (!c || !partial || !flat_grad || G < 1 || n_params < 1) return fail(R4_ERR_ARG, "r4_grad_exchange_n: bad argument");
  return exchange_launch(c, partial, G, n_params, flat_grad, stats_accum, stat_scale, 0, nullptr, nullptr, nullptr, 0, 0.f, 0.f, 0.f,
                         0.f, stream);
}

// ---- Gaussian policy of the continuous-action env (r4_gauss.cuh) -------------------------------------------
static bool gauss_dim_ok(int D) { return D >= 2 && D <= r4gauss::MAXD && D % 2 == 0; }

int r4_gauss_num_params(int action_dim) { return gauss_dim_ok(action_dim) ? r4gauss::make_layout(action_dim).n : -1; }

int64_t r4_gauss_scratch_size(int action_dim) {
  return gauss_dim_ok(action_dim) ? (int64_t)r4gauss::scratch_floats(action_dim) : -1;
}

int r4_gauss_act(const float* params, const float* obs, int n, int action_dim, int explore, uint64_t seed, uint64_t counter,
                 float* action, float* env_action, float* logp, float* value, float* dist_inputs, void* stream) {
  if (!params || !obs || !action || !env_action || !logp || !value || n < 1 || !gauss_dim_ok(action_dim))
    return fail(R4_ERR_ARG, "r4_gauss_act: bad argument (action_dim even, 2..64)");
  return launch(FAM_ONLINE, "k_gauss_act", r4gauss::k_gauss_act, (n + r4gauss::TS - 1) / r4gauss::TS, r4gauss::NT,
                r4gauss::ACT_SMEM, S(stream), false, r4gauss::make_layout(action_dim), params, obs, n, explore, seed, counter,
                action, env_action, logp, value, dist_inputs);
}

// grad_out[np] = the gradient over samples idx[0..n) (chunks of CH, accumulated in order); stat_sum[5] = the raw statistic
// sums; stats_accum (may be NULL) += stat_sum * stat_scale.
static int gauss_grad_impl(int mode, const float* params, const float* obs, const float* action, const float* old_logp,
                           const float* old_dist, const float* old_value, const float* adv, const float* target,
                           const int64_t* idx, int n, int D, float clip, float vf_clip, float vf_coeff, float kl_coeff,
                           float ent_coeff, float inv_n, float* scratch, float* grad_out, float* stat_sum, float* stats_accum,
                           float stat_scale, void* stream) {
  if (!params || !obs || !action || !adv || !target || !scratch || !grad_out || n < 1 || !gauss_dim_ok(D) ||
      (mode == 0 && (!old_logp || !old_value || !old_dist)) || (mode != 0 && mode != 1))
    return fail(R4_ERR_ARG, "r4_gauss_grad: bad argument");
  const r4gauss::Layout L = r4gauss::make_layout(D);
  const r4ppo::LossHyper hp{mode, clip, vf_clip, vf_coeff, kl_coeff, ent_coeff, inv_n};
  const r4gauss::Planes P = r4gauss::make_planes(scratch, D);
  const r4gauss::Jobs J = r4gauss::make_jobs(L, P);
  for (int c0 = 0; c0 < n; c0 += r4gauss::CH) {
    const int cn = std::min(r4gauss::CH, n - c0);
    const bool last = c0 + cn >= n;
    int rc = launch(FAM_ONLINE, "k_gauss_rows", r4gauss::k_gauss_rows, (cn + r4gauss::TS - 1) / r4gauss::TS, r4gauss::NT,
                    r4gauss::ROWS_SMEM, S(stream), false, L, hp, params, obs, action, old_logp, old_dist, old_value, adv, target,
                    idx, c0, cn, P);
    if (!rc)
      rc = launch(FAM_ONLINE, "k_gauss_wgrad", r4gauss::k_gauss_wgrad, J.ntiles + 1, r4gauss::NT, 0, S(stream), false, J, cn,
                  c0 == 0, grad_out, P.stats, stat_sum, last ? stats_accum : nullptr, stat_scale);
    if (rc) return rc;
  }
  return R4_OK;
}

static float* gauss_gsum(float* scratch, int D) {           // [np] gradient + [5] statistics, then [5] raw statistics
  return scratch + (size_t)r4gauss::CH * (r4gauss::NPLANE * r4gauss::H + 2 * D + 1 + 5);
}

int r4_gauss_grad(int mode, const float* params, const float* obs, const float* action, const float* old_logp,
                  const float* old_dist, const float* old_value, const float* adv, const float* target, const int64_t* idx,
                  int n, int action_dim, float clip, float vf_clip, float vf_coeff, float kl_coeff, float ent_coeff,
                  float inv_n, float* scratch, float* flat_grad, float* stats_accum, float stat_scale, void* stream) {
  if (!scratch || !gauss_dim_ok(action_dim)) return fail(R4_ERR_ARG, "r4_gauss_grad: bad argument");
  float* raw = gauss_gsum(scratch, action_dim) + r4gauss::make_layout(action_dim).n + 5;
  return gauss_grad_impl(mode, params, obs, action, old_logp, old_dist, old_value, adv, target, idx, n, action_dim, clip, vf_clip,
                         vf_coeff, kl_coeff, ent_coeff, inv_n, scratch, flat_grad, raw, stats_accum, stat_scale, stream);
}

int r4_gauss_ppo_epoch(float* params, const float* obs, const float* action, const float* old_logp, const float* old_dist,
                       const float* old_value, const float* adv, const float* target, const int64_t* perm, int n, int mb,
                       int action_dim, float clip, float vf_clip, float vf_coeff, float kl_coeff, float ent_coeff,
                       float* scratch, float* flat_grad, float* stats_accum, float* m, float* v, int step0, float lr,
                       float beta1, float beta2, float eps, float grad_clip, float* norm_scratch, void* stream) {
  if (!perm || !params || !m || !v || !flat_grad || !scratch || n < 1 || mb < 1 || mb > n || step0 < 0 || !gauss_dim_ok(action_dim))
    return fail(R4_ERR_ARG, "r4_gauss_ppo_epoch: bad argument");
  const int np = r4gauss::make_layout(action_dim).n;
  int steps = 0;
  for (int s = 0; s + mb <= n; s += mb, ++steps) {
    int rc = r4_gauss_grad(0, params, obs, action, old_logp, old_dist, old_value, adv, target, perm + s, mb, action_dim, clip, vf_clip,
                           vf_coeff, kl_coeff, ent_coeff, 1.0f / mb, scratch, flat_grad, stats_accum, 1.0f / mb, stream);
    if (rc) return rc;
    rc = r4_adam_step(params, flat_grad, m, v, np, step0 + steps + 1, lr, beta1, beta2, eps, 1.0f, grad_clip, norm_scratch, stream);
    if (rc) return rc;
  }
  return steps;
}

int r4_gauss_ppo_epoch_dist(r4_comm* c, float* params, const float* obs, const float* action, const float* old_logp,
                            const float* old_dist, const float* old_value, const float* adv, const float* target,
                            const int64_t* perm, int n, int mb, int action_dim, float clip, float vf_clip, float vf_coeff,
                            float kl_coeff, float ent_coeff, float* scratch, float* flat_grad, float* stats_accum, float* m,
                            float* v, int step0, float lr, float beta1, float beta2, float eps, void* stream) {
  if (!c || !params || !perm || !m || !v || !scratch || n < 1 || mb < 1 || mb > n || step0 < 0 || !gauss_dim_ok(action_dim))
    return fail(R4_ERR_ARG, "r4_gauss_ppo_epoch_dist: bad argument");
  const int np = r4gauss::make_layout(action_dim).n;
  const float inv = 1.0f / ((float)mb * (float)c->world);
  float* gsum = gauss_gsum(scratch, action_dim);
  int steps = 0;
  for (int s = 0; s + mb <= n; s += mb, ++steps) {
    int rc = gauss_grad_impl(0, params, obs, action, old_logp, old_dist, old_value, adv, target, perm + s, mb, action_dim, clip,
                             vf_clip, vf_coeff, kl_coeff, ent_coeff, inv, scratch, gsum, gsum + np, nullptr, 0.f, stream);
    if (rc) return rc;
    // one "partial" (G = 1): the exchange sums it over the ranks in rank order and applies Adam; statistics stay per-rank means
    rc = exchange_launch(c, gsum, 1, np, flat_grad, stats_accum, 1.0f / (float)mb, 1, params, m, v, step0 + steps + 1, lr, beta1,
                         beta2, eps, stream);
    if (rc) return rc;
  }
  return steps;
}

// ---- IMPALA: forward at the stored actions, V-trace, the fused learner step (r4_ppo.cuh, r4_gauss.cuh) ----------------------------
static bool vtrace_args_ok(int T, int B, float gamma, float rho_bar, float rho_pg_bar, int drop_last) {
  return T >= (drop_last ? 2 : 1) && T <= r4ppo::MAXT && B >= 1 && (int64_t)T * B <= 0x7fffffff && gamma >= 0.f &&
         gamma <= 1.f && rho_bar > 0.f && rho_pg_bar > 0.f && std::isfinite(rho_bar) && std::isfinite(rho_pg_bar);
}

static size_t policy_eval_smem(int A) {
  return (size_t)(r4ppo::TS * r4ppo::OBS + r4ppo::TS * r4ppo::HID + r4ppo::TS * A + r4ppo::TS) * 4;
}

int r4_policy_eval(const float* params, const float* obs, const uint8_t* mask, const int64_t* action, int n, int action_size,
                   float* logp, float* value, void* stream) {
  if (!params || !obs || !mask || !action || !logp || !value || n < 1 || action_size < 2 || action_size > 512)
    return fail(R4_ERR_ARG, "r4_policy_eval: bad argument");
  return launch(FAM_ONLINE, "k_policy_eval", r4ppo::k_policy_eval, (n + r4ppo::TS - 1) / r4ppo::TS, r4ppo::NT,
                policy_eval_smem(action_size), S(stream), false, r4ppo::make_layout(action_size), params, obs, mask, action, n,
                logp, value);
}

int r4_gauss_eval(const float* params, const float* obs, const float* action, int n, int action_dim, float* logp, float* value,
                  void* stream) {
  if (!params || !obs || !action || !logp || !value || n < 1 || !gauss_dim_ok(action_dim))
    return fail(R4_ERR_ARG, "r4_gauss_eval: bad argument (action_dim even, 2..64)");
  return launch(FAM_ONLINE, "k_gauss_eval", r4gauss::k_gauss_eval, (n + r4gauss::TS - 1) / r4gauss::TS, r4gauss::NT,
                r4gauss::ACT_SMEM, S(stream), false, r4gauss::make_layout(action_dim), params, obs, action, n, logp, value);
}

int r4_vtrace(const float* behaviour_logp, const float* target_logp, const float* value, const float* reward, int T, int B,
              float gamma, float rho_bar, float rho_pg_bar, int drop_last, float* vs, float* pg_adv, void* stream) {
  if (!behaviour_logp || !target_logp || !value || !reward || !vs || !pg_adv ||
      !vtrace_args_ok(T, B, gamma, rho_bar, rho_pg_bar, drop_last))
    return fail(R4_ERR_ARG, "r4_vtrace: bad argument (T 1..81, 2..81 with drop_last, gamma in [0, 1], thresholds > 0)");
  return launch(FAM_ONLINE, "k_vtrace", r4ppo::k_vtrace, (B + 255) / 256, 256, 0, S(stream), false, T, B, behaviour_logp,
                target_logp, value, reward, gamma, rho_bar, rho_pg_bar, (int)(drop_last != 0), vs, pg_adv);
}

// The tail of both fused IMPALA steps: (the exchange of this rank's partials over peer memory,) the global-norm clip in a
// fixed order and Adam.
static int impala_tail(r4_comm* comm, const float* partial, int G, int np, float* params, float* flat_grad, float* stats_accum,
                       float* m, float* v, int step, float lr, float b1, float b2, float eps, float grad_clip,
                       float* norm_scratch, cudaStream_t st) {
  int rc = R4_OK;
  if (comm && (rc = exchange_launch(comm, partial, G, np, flat_grad, stats_accum, 1.f, 0, nullptr, nullptr, nullptr, 0, 0.f, 0.f,
                                    0.f, 0.f, st)))
    return rc;
  if (grad_clip > 0.f &&
      (rc = launch(FAM_ONLINE, "k_sumsq_one", r4ppo::k_sumsq_one, 1, r4ppo::SQT, 0, st, false, np, flat_grad, norm_scratch)))
    return rc;
  return launch(FAM_ONLINE, "k_adam", r4ppo::k_adam, (np + 255) / 256, 256, 0, st, false, np, params, flat_grad, m, v, step, lr,
                b1, b2, eps, 1.f, grad_clip > 0.f ? norm_scratch : nullptr, grad_clip);
}

static bool impala_comm_ok(r4_comm* comm, int np) { return !comm || (comm->ready && comm->n == np); }

int r4_impala_step(r4_comm* comm, float* params, const float* obs, const uint8_t* mask, const int64_t* action,
                   const float* behaviour_logp, const float* logits, const float* reward, int T, int B, int action_size,
                   float gamma, float rho_bar, float rho_pg_bar, int drop_last, float vf_coeff, float ent_coeff, float* logp,
                   float* value, float* vs, float* pg_adv, float* scratch, float* flat_grad, float* stats_accum, float* m,
                   float* v, int step, float lr, float beta1, float beta2, float eps, float grad_clip, float* norm_scratch,
                   void* stream) {
  if (!params || !obs || !mask || !action || !behaviour_logp || !logits || !reward || !logp || !value || !vs || !pg_adv ||
      !scratch || !flat_grad || !m || !v || step < 1 || (grad_clip > 0.f && !norm_scratch) || action_size < 2 ||
      action_size > 512 || !vtrace_args_ok(T, B, gamma, rho_bar, rho_pg_bar, drop_last) ||
      !impala_comm_ok(comm, r4ppo::make_layout(action_size).n))
    return fail(R4_ERR_ARG, "r4_impala_step: bad argument");
  const int n = T * B, nk = (drop_last ? T - 1 : T) * B;          // the kept rows are the first T - 1 (or T) time steps
  const int np = r4ppo::make_layout(action_size).n;
  const int G = std::max(1, std::min((nk + r4ppo::TS - 1) / r4ppo::TS, sm_count()));
  cudaStream_t st = S(stream);
  int rc = r4_policy_eval(params, obs, mask, action, n, action_size, logp, value, stream);
  if (!rc) rc = r4_vtrace(behaviour_logp, logp, value, reward, T, B, gamma, rho_bar, rho_pg_bar, drop_last, vs, pg_adv, stream);
  // A2C mode: -sum logp pg_adv + vf_coeff * 0.5 sum (V - vs)^2 - ent_coeff * sum H over the kept rows
  if (!rc) rc = policy_grad_impl(1, params, obs, mask, action, nullptr, logits, nullptr, pg_adv, vs, nullptr, nk, action_size, 0.f,
                                 0.f, vf_coeff, 0.f, ent_coeff, 1.f, scratch, G, flat_grad, stats_accum, 1.f, stream, !comm);
  if (rc) return rc;
  return impala_tail(comm, scratch, G, np, params, flat_grad, stats_accum, m, v, step, lr, beta1, beta2, eps, grad_clip,
                     norm_scratch, st);
}

int r4_gauss_impala_step(r4_comm* comm, float* params, const float* obs, const float* action, const float* behaviour_logp,
                         const float* reward, int T, int B, int action_dim, float gamma, float rho_bar, float rho_pg_bar,
                         int drop_last, float vf_coeff, float ent_coeff, float* logp, float* value, float* vs, float* pg_adv,
                         float* scratch, float* flat_grad, float* stats_accum, float* m, float* v, int step, float lr,
                         float beta1, float beta2, float eps, float grad_clip, float* norm_scratch, void* stream) {
  if (!params || !obs || !action || !behaviour_logp || !reward || !logp || !value || !vs || !pg_adv || !scratch || !flat_grad ||
      !m || !v || step < 1 || (grad_clip > 0.f && !norm_scratch) || !gauss_dim_ok(action_dim) ||
      !vtrace_args_ok(T, B, gamma, rho_bar, rho_pg_bar, drop_last) ||
      !impala_comm_ok(comm, r4gauss::make_layout(action_dim).n))
    return fail(R4_ERR_ARG, "r4_gauss_impala_step: bad argument");
  const int n = T * B, nk = (drop_last ? T - 1 : T) * B;
  const int np = r4gauss::make_layout(action_dim).n;
  float* gsum = gauss_gsum(scratch, action_dim);
  cudaStream_t st = S(stream);
  int rc = r4_gauss_eval(params, obs, action, n, action_dim, logp, value, stream);
  if (!rc) rc = r4_vtrace(behaviour_logp, logp, value, reward, T, B, gamma, rho_bar, rho_pg_bar, drop_last, vs, pg_adv, stream);
  if (!rc) {
    if (comm)      // one partial (G = 1): the gradient and its statistics, summed over the ranks by the exchange
      rc = gauss_grad_impl(1, params, obs, action, nullptr, nullptr, nullptr, pg_adv, vs, nullptr, nk, action_dim, 0.f, 0.f,
                           vf_coeff, 0.f, ent_coeff, 1.f, scratch, gsum, gsum + np, nullptr, 0.f, stream);
    else
      rc = gauss_grad_impl(1, params, obs, action, nullptr, nullptr, nullptr, pg_adv, vs, nullptr, nk, action_dim, 0.f, 0.f,
                           vf_coeff, 0.f, ent_coeff, 1.f, scratch, flat_grad, gsum + np + 5, stats_accum, 1.f, stream);
  }
  if (rc) return rc;
  return impala_tail(comm, gsum, 1, np, params, flat_grad, stats_accum, m, v, step, lr, beta1, beta2, eps, grad_clip,
                     norm_scratch, st);
}

// ---- DDPG / TD3 (r4_ddpg.cuh) ---------------------------------------------------------------------------------
static bool ddpg_dim_ok(int D) { return D >= 2 && D <= r4ddpg::MAXD; }

int r4_ddpg_num_params(int action_dim, int twin) { return ddpg_dim_ok(action_dim) ? r4ddpg::make_layout(action_dim, twin != 0).n : -1; }

int64_t r4_ddpg_scratch_size(int action_dim, int twin, int n) {
  return (!ddpg_dim_ok(action_dim) || n < 1) ? -1 : (int64_t)r4ddpg::scratch_floats(action_dim, twin != 0, n);
}

int r4_ddpg_act(const float* params, const float* obs, int n, int action_dim, int mode, uint64_t seed, uint64_t counter,
                const float* ou_in, float* ou_out, float ou_theta, float ou_sigma, float noise_scale, float* action,
                void* stream) {
  if (!params || !obs || !action || n < 1 || !ddpg_dim_ok(action_dim) || mode < 0 || mode > 2 ||
      (mode == 1 && (!ou_in || !ou_out || ou_in == ou_out)))
    return fail(R4_ERR_ARG, "r4_ddpg_act: bad argument (action_dim 2..32, mode 0..2, OU needs two state buffers)");
  return launch(FAM_ONLINE, "k_ddpg_act", r4ddpg::k_ddpg_act, (n + r4ddpg::TS - 1) / r4ddpg::TS, r4ddpg::NT, r4ddpg::ACT_SMEM,
                S(stream), false, r4ddpg::make_layout(action_dim, 0), params, obs, n, mode, seed, counter, ou_in, ou_out, ou_theta,
                ou_sigma, noise_scale, action);
}

int r4_replay_store(float* r_obs, float* r_action, float* r_reward, float* r_new_obs, uint8_t* r_done, float* r_prio,
                    const float* max_prio, int capacity, int action_dim, int64_t pos, float alpha, const float* obs,
                    const float* final_obs, const float* action, const float* reward, const uint8_t* done, int T, int B,
                    void* stream) {
  if (!r_obs || !r_action || !r_reward || !r_new_obs || !r_done || (r_prio && !max_prio) || capacity < 1 || pos < 0 ||
      !ddpg_dim_ok(action_dim) || !obs || !final_obs || !action || !reward || !done || T < 1 || B < 1)
    return fail(R4_ERR_ARG, "r4_replay_store: bad argument");
  const int64_t rows = std::min<int64_t>((int64_t)T * B, capacity);
  return launch(FAM_ONLINE, "k_replay_store", r4ddpg::k_replay_store, (unsigned)rows, 64, 0, S(stream), false, r_obs, r_action,
                r_reward, r_new_obs, r_done, r_prio, max_prio, capacity, action_dim, pos, alpha, obs, final_obs, action, reward,
                done, T, B);
}

int r4_replay_sample(const float* prio, int size, int n, float beta, const float* u, int64_t* idx, float* weights, void* stream) {
  if (size < 1 || n < 1 || !u || !idx || !weights) return fail(R4_ERR_ARG, "r4_replay_sample: bad argument");
  return launch(FAM_ONLINE, "k_replay_sample", r4ddpg::k_replay_sample, 1, r4ddpg::SNT, 0, S(stream), false, prio, size, n, beta,
                u, idx, weights);
}

int r4_replay_update_priorities(float* prio, float* max_prio, const int64_t* idx, const float* td, int n, float alpha,
                                float eps, void* stream) {
  if (!prio || !max_prio || !idx || !td || n < 1) return fail(R4_ERR_ARG, "r4_replay_update_priorities: bad argument");
  return launch(FAM_ONLINE, "k_replay_priorities", r4ddpg::k_replay_priorities, 1, r4ddpg::SNT, 0, S(stream), false, prio,
                max_prio, idx, td, n, alpha, eps);
}

int r4_ddpg_grad(const float* params, const float* target, int action_dim, int twin, const float* r_obs, const float* r_action,
                 const float* r_reward, const float* r_new_obs, const uint8_t* r_done, const int64_t* idx, const float* weights,
                 const float* smooth_noise, int n, float gamma, float target_noise, float noise_clip, float inv_n,
                 float* scratch, float* grad, float* td, float* stats, void* stream) {
  if (!params || !target || !ddpg_dim_ok(action_dim) || !r_obs || !r_action || !r_reward || !r_new_obs || !r_done || !idx ||
      n < 1 || !scratch || !grad)
    return fail(R4_ERR_ARG, "r4_ddpg_grad: bad argument");
  const r4ddpg::Layout L = r4ddpg::make_layout(action_dim, twin != 0);
  r4ddpg::Planes P = r4ddpg::make_planes(scratch, action_dim, twin != 0, n);
  if (td) P.td = td;
  const r4ddpg::Jobs J = r4ddpg::make_jobs(L, P);
  const r4ddpg::Replay R{r_obs, r_action, r_reward, r_new_obs, r_done};
  const r4ddpg::Hyper hp{gamma, target_noise, noise_clip, inv_n};
  if (int rc = launch(FAM_ONLINE, "k_ddpg_rows", r4ddpg::k_ddpg_rows, (n + r4ddpg::TS - 1) / r4ddpg::TS, r4ddpg::NT,
                      r4ddpg::ROWS_SMEM, S(stream), false, L, hp, params, target, R, idx, weights, smooth_noise, n, P))
    return rc;
  return launch(FAM_ONLINE, "k_ddpg_wgrad", r4ddpg::k_ddpg_wgrad, J.ntiles + 1, r4ddpg::NT, 0, S(stream), false, J, n, grad,
                P.stats, stats, inv_n);
}

int r4_ddpg_apply(float* params, float* target, const float* grad, float* m, float* v, int action_dim, int twin, int actor_step,
                  int critic_step, float actor_lr, float critic_lr, float l2_reg, float tau, float grad_scale, void* stream) {
  if (!params || !target || !grad || !m || !v || !ddpg_dim_ok(action_dim) || actor_step < 0 || critic_step < 1)
    return fail(R4_ERR_ARG, "r4_ddpg_apply: bad argument");
  const r4ddpg::Layout L = r4ddpg::make_layout(action_dim, twin != 0);
  return launch(FAM_ONLINE, "k_ddpg_apply", r4ddpg::k_ddpg_apply, (L.n + 255) / 256, 256, 0, S(stream), false, L, params, target,
                grad, m, v, actor_step, critic_step, actor_lr, critic_lr, l2_reg, tau, grad_scale);
}

int r4_ddpg_train_step(r4_comm* comm, float* params, float* target, float* m, float* v, int action_dim, int twin,
                       const float* r_obs, const float* r_action, const float* r_reward, const float* r_new_obs,
                       const uint8_t* r_done, float* r_prio, float* max_prio, int size, int n, const float* u,
                       const float* smooth_noise, float beta, float alpha, float prio_eps, float gamma, float target_noise,
                       float noise_clip, int actor_step, int critic_step, float actor_lr, float critic_lr, float l2_reg,
                       float tau, float* scratch, float* stats, void* stream) {
  if (!scratch || !ddpg_dim_ok(action_dim) || n < 1 || (r_prio && !max_prio))
    return fail(R4_ERR_ARG, "r4_ddpg_train_step: bad argument");
  const int np = r4ddpg::make_layout(action_dim, twin != 0).n;
  const r4ddpg::Planes P = r4ddpg::make_planes(scratch, action_dim, twin != 0, n);
  const int world = comm ? comm->world : 1;
  int rc = r4_replay_sample(r_prio, size, n, beta, u, P.idx, P.weights, stream);
  if (rc) return rc;
  rc = r4_ddpg_grad(params, target, action_dim, twin, r_obs, r_action, r_reward, r_new_obs, r_done, P.idx,
                    r_prio ? P.weights : nullptr, smooth_noise, n, gamma, target_noise, noise_clip, 1.0f / ((float)n * world),
                    scratch, P.grad, nullptr, stats, stream);
  if (rc) return rc;
  const float* g = P.grad;
  if (comm) {        // one partial (G = 1) per rank, summed in rank order into the scratch's second gradient
    float* sum = P.grad + np + 5;
    if ((rc = exchange_launch(comm, P.grad, 1, np, sum, nullptr, 0.f, 0, nullptr, nullptr, nullptr, 0, 0.f, 0.f, 0.f, 0.f, stream)))
      return rc;
    g = sum;
  }
  rc = r4_ddpg_apply(params, target, g, m, v, action_dim, twin, actor_step, critic_step, actor_lr, critic_lr, l2_reg, tau, 1.0f,
                     stream);
  if (rc || !r_prio) return rc;
  return r4_replay_update_priorities(r_prio, max_prio, P.idx, P.td, n, alpha, prio_eps, stream);
}

// ---- RAINBOW (r4_rainbow.cuh) ---------------------------------------------------------------------------------
static bool rainbow_dims_ok(int A, int Z) {
  return A >= 2 && A <= r4rb::MAXA && Z >= 2 && Z <= r4rb::MAXZ && A * Z <= r4rb::MAXAZ;
}

int r4_rainbow_num_params(int num_actions, int num_atoms) {
  return rainbow_dims_ok(num_actions, num_atoms) ? r4rb::make_layout(num_actions, num_atoms).n : -1;
}

int64_t r4_rainbow_scratch_size(int num_actions, int num_atoms, int n) {
  if (!rainbow_dims_ok(num_actions, num_atoms) || n < 1) return -1;
  return (int64_t)r4rb::scratch_floats(r4rb::make_layout(num_actions, num_atoms), n);
}

int r4_rainbow_act(const float* params, const float* obs, int n, int num_actions, int num_atoms, float v_min, float v_max,
                   int explore, uint64_t seed, uint64_t counter, int32_t* action, float* q, void* stream) {
  if (!params || !obs || !action || n < 1 || !rainbow_dims_ok(num_actions, num_atoms) || !(v_max > v_min))
    return fail(R4_ERR_ARG, "r4_rainbow_act: bad argument (actions 2..512, atoms 2..32, actions x atoms <= 4096)");
  const r4rb::Layout L = r4rb::make_layout(num_actions, num_atoms);
  return launch(FAM_ONLINE, "k_rainbow_act", r4rb::k_rainbow_act, (n + r4rb::TS - 1) / r4rb::TS, r4rb::NT,
                r4rb::act_smem(L.A, L.AZ), S(stream), false, L, params, obs, n, v_min,
                (v_max - v_min) / (float)(num_atoms - 1), explore != 0, seed, counter, action, q);
}

int r4_replay_store_nstep(float* r_obs, int32_t* r_action, float* r_reward, float* r_new_obs, uint8_t* r_done, float* r_prio,
                          const float* max_prio, int capacity, int64_t pos, float alpha, int n_step, float gamma,
                          const float* obs, const float* final_obs, const int32_t* action, const float* reward,
                          const uint8_t* done, int T, int B, void* stream) {
  if (!r_obs || !r_action || !r_reward || !r_new_obs || !r_done || (r_prio && !max_prio) || capacity < 1 || pos < 0 ||
      n_step < 1 || !obs || !final_obs || !action || !reward || !done || T < 1 || B < 1)
    return fail(R4_ERR_ARG, "r4_replay_store_nstep: bad argument");
  const int64_t rows = std::min<int64_t>((int64_t)T * B, capacity);
  return launch(FAM_ONLINE, "k_replay_store_nstep", r4rb::k_replay_store_nstep, (unsigned)rows, 64, 0, S(stream), false, r_obs,
                r_action, r_reward, r_new_obs, r_done, r_prio, max_prio, capacity, pos, alpha, n_step, gamma, obs, final_obs,
                action, reward, done, T, B);
}

int r4_rainbow_grad(const float* params, const float* target, int num_actions, int num_atoms, float v_min, float v_max,
                    const float* r_obs, const int32_t* r_action, const float* r_reward, const float* r_new_obs,
                    const uint8_t* r_done, const int64_t* idx, const float* weights, int n, float gamma_n, float inv_n,
                    float* scratch, float* grad, float* td, float* stats, void* stream) {
  if (!params || !target || !rainbow_dims_ok(num_actions, num_atoms) || !(v_max > v_min) || !r_obs || !r_action ||
      !r_reward || !r_new_obs || !r_done || !idx || n < 1 || !scratch || !grad)
    return fail(R4_ERR_ARG, "r4_rainbow_grad: bad argument");
  const r4rb::Layout L = r4rb::make_layout(num_actions, num_atoms);
  r4rb::Planes P = r4rb::make_planes(scratch, L, n);
  if (td) P.td = td;
  const r4ddpg::Jobs J = r4rb::make_jobs(L, P);
  const r4rb::Replay R{r_obs, r_action, r_reward, r_new_obs, r_done};
  const r4rb::Hyper hp{v_min, v_max, (v_max - v_min) / (float)(num_atoms - 1), gamma_n, inv_n};
  if (int rc = launch(FAM_ONLINE, "k_rainbow_rows", r4rb::k_rainbow_rows, (n + r4rb::TS - 1) / r4rb::TS, r4rb::NT,
                      r4rb::rows_smem(L.A, L.AZ), S(stream), false, L, hp, params, target, R, idx, weights, n, P))
    return rc;
  return launch(FAM_ONLINE, "k_ddpg_wgrad", r4ddpg::k_ddpg_wgrad, J.ntiles + 1, r4ddpg::NT, 0, S(stream), false, J, n, grad,
                P.stats, stats, inv_n);
}

int r4_rainbow_apply(float* params, float* target, const float* grad, float* m, float* v, int num_actions, int num_atoms,
                     int step, float lr, float adam_eps, float grad_clip, int copy_target, void* stream) {
  if (!params || !target || !grad || !m || !v || !rainbow_dims_ok(num_actions, num_atoms) || step < 1)
    return fail(R4_ERR_ARG, "r4_rainbow_apply: bad argument");
  const r4rb::Split Sp = r4rb::make_split(r4rb::make_layout(num_actions, num_atoms));
  return launch(FAM_ONLINE, "k_rainbow_apply", r4rb::k_rainbow_apply, Sp.cta0[r4rb::NTEN], r4rb::ANT, 0, S(stream), false, Sp,
                params, target, grad, m, v, step, lr, adam_eps, grad_clip, copy_target != 0);
}

int r4_rainbow_train_step(r4_comm* comm, float* params, float* target, float* m, float* v, int num_actions, int num_atoms,
                          float v_min, float v_max, const float* r_obs, const int32_t* r_action, const float* r_reward,
                          const float* r_new_obs, const uint8_t* r_done, float* r_prio, float* max_prio, int size, int n,
                          const float* u, float beta, float alpha, float prio_eps, float gamma_n, int step, float lr,
                          float adam_eps, float grad_clip, int copy_target, float* scratch, float* stats, void* stream) {
  if (!scratch || !rainbow_dims_ok(num_actions, num_atoms) || n < 1 || (r_prio && !max_prio))
    return fail(R4_ERR_ARG, "r4_rainbow_train_step: bad argument");
  const r4rb::Layout L = r4rb::make_layout(num_actions, num_atoms);
  const r4rb::Planes P = r4rb::make_planes(scratch, L, n);
  const int world = comm ? comm->world : 1;
  int rc = r4_replay_sample(r_prio, size, n, beta, u, P.idx, P.weights, stream);
  if (rc) return rc;
  rc = r4_rainbow_grad(params, target, num_actions, num_atoms, v_min, v_max, r_obs, r_action, r_reward, r_new_obs, r_done,
                       P.idx, r_prio ? P.weights : nullptr, n, gamma_n, 1.0f / ((float)n * world), scratch, P.grad, nullptr,
                       stats, stream);
  if (rc) return rc;
  const float* g = P.grad;
  if (comm) {        // one partial (G = 1) per rank, summed in rank order into the scratch's second gradient
    float* sum = P.grad + L.n + 5;
    if ((rc = exchange_launch(comm, P.grad, 1, L.n, sum, nullptr, 0.f, 0, nullptr, nullptr, nullptr, 0, 0.f, 0.f, 0.f, 0.f, stream)))
      return rc;
    g = sum;
  }
  rc = r4_rainbow_apply(params, target, g, m, v, num_actions, num_atoms, step, lr, adam_eps, grad_clip, copy_target, stream);
  if (rc || !r_prio) return rc;
  return r4_replay_update_priorities(r_prio, max_prio, P.idx, P.td, n, alpha, prio_eps, stream);
}

// ---- batch RL: discrete BC / BCQ / CQL (r4_batchrl.cuh) -----------------------------------------------------------
int64_t r4_batchrl_launch_count(void) { return g_launches[FAM_BATCHRL].load(std::memory_order_relaxed); }

int r4_batchrl_num_params(int algo, int obs_dim, int action_size) {
  return r4bq::dims_ok(algo, obs_dim, action_size) ? r4bq::make_layout(algo, obs_dim, action_size).n : -1;
}

int r4_batchrl_target_size(int algo, int obs_dim, int action_size) {
  return r4bq::dims_ok(algo, obs_dim, action_size) ? r4bq::make_layout(algo, obs_dim, action_size).ntgt : -1;
}

int64_t r4_batchrl_scratch_size(int algo, int obs_dim, int action_size, int n) {
  if (!r4bq::dims_ok(algo, obs_dim, action_size) || n < 1) return -1;
  return (int64_t)r4bq::scratch_floats(r4bq::make_layout(algo, obs_dim, action_size), n);
}

int r4_batchrl_transitions(const uint8_t* terminal, int64_t N, int64_t* index, int64_t* count, void* stream) {
  if (!terminal || N < 1 || !index || !count) return fail(R4_ERR_ARG, "r4_batchrl_transitions: bad argument");
  return launch(FAM_BATCHRL, "k_bq_transitions", r4bq::k_bq_transitions, 1, r4bq::TRT, 0, S(stream), false, terminal, N, index,
                count);
}

static r4bq::Data bq_data(const r4_batchrl_data* d) {
  return r4bq::Data{d->obs, d->action, d->reward, d->terminal, d->transitions, d->location_mask, d->special};
}

// the kernels of one SGD step; pdl: launch the chain with programmatic dependent launch (r4_batchrl_epoch)
static int bq_grad(int algo, int K, int A, const float* params, const float* target, const r4_batchrl_data* data,
                   const r4_batchrl_hyper* h, const int64_t* idx, int n, float* scratch, float* grad, float* stats,
                   cudaStream_t st, bool pdl) {
  decltype(&r4bq::k_bq_rows<r4bq::BC>) const rows[3] = {r4bq::k_bq_rows<r4bq::BC>, r4bq::k_bq_rows<r4bq::BCQ>,
                                                        r4bq::k_bq_rows<r4bq::CQL>};
  r4bq::Layout L = r4bq::make_layout(algo, K, A);
  r4bq::Planes P = r4bq::make_planes(scratch, L, n);
  P.grad = grad;
  const r4bq::Hyper hp{h->gamma, 1.0f / (float)n, h->beta, h->alpha, h->log_flex, h->reward_mean, h->reward_den};
  int rc = launch(FAM_BATCHRL, "k_bq_rows", rows[algo], (n + r4bq::TS - 1) / r4bq::TS, r4bq::NT, r4bq::rows_smem(K, A), st, pdl,
                  L, hp, params, target, bq_data(data), idx, n, P);
  if (rc) return rc;
  const r4ddpg::Jobs J = r4bq::make_jobs(L, P);
  if ((rc = launch(FAM_BATCHRL, "k_ddpg_wgrad", r4ddpg::k_ddpg_wgrad, J.ntiles + 1, r4ddpg::NT, 0, st, false, J, n, grad, P.stats,
                   stats, 1.0f / (float)n)))
    return rc;
  const int nets = r4bq::n_mnets(algo);
  if (!nets) return R4_OK;
  const int per = (A * r4bq::E + r4bq::EGT - 1) / r4bq::EGT;
  return launch(FAM_BATCHRL, "k_bq_embgrad", r4bq::k_bq_embgrad, nets * per, r4bq::EGT, 0, st, pdl, L, P, n, per);
}

static int bq_apply(int algo, int K, int A, float* params, float* target, const float* grad, float* m, float* v, int step,
                    float lr, float eps, int copy, cudaStream_t st, bool pdl) {
  const r4bq::Layout L = r4bq::make_layout(algo, K, A);
  return launch(FAM_BATCHRL, "k_bq_apply", r4bq::k_bq_apply, (L.n + 255) / 256, 256, 0, st, pdl, L.n, L.ntgt, params, target,
                grad, m, v, step, lr, eps, copy);
}

static bool bq_data_ok(const r4_batchrl_data* d) {
  return d && d->obs && d->action && d->reward && d->terminal && d->transitions && d->location_mask && d->special;
}

int r4_batchrl_grad(int algo, int obs_dim, int action_size, const float* params, const float* target,
                    const r4_batchrl_data* data, const r4_batchrl_hyper* hp, const int64_t* idx, int n, float* scratch,
                    float* grad, float* stats, void* stream) {
  if (!r4bq::dims_ok(algo, obs_dim, action_size) || !params || (algo != r4bq::BC && !target) || !bq_data_ok(data) || !hp ||
      !idx || n < 1 || !scratch || !grad)
    return fail(R4_ERR_ARG, "r4_batchrl_grad: bad argument (algo 0..2, obs_dim 11..4096, action_size 2..512, shared planes <= 226 KB)");
  return bq_grad(algo, obs_dim, action_size, params, target, data, hp, idx, n, scratch, grad, stats, S(stream), false);
}

int r4_batchrl_apply(int algo, int obs_dim, int action_size, float* params, float* target, const float* grad, float* m,
                     float* v, int step, float lr, float adam_eps, int copy_target, void* stream) {
  if (!r4bq::dims_ok(algo, obs_dim, action_size) || !params || !grad || !m || !v || step < 1 || (copy_target && algo != r4bq::BC && !target))
    return fail(R4_ERR_ARG, "r4_batchrl_apply: bad argument");
  return bq_apply(algo, obs_dim, action_size, params, target, grad, m, v, step, lr, adam_eps, copy_target, S(stream), false);
}

int r4_batchrl_epoch(int algo, int obs_dim, int action_size, float* params, float* target, float* m, float* v,
                     const r4_batchrl_data* data, const r4_batchrl_hyper* hp, const int64_t* perm, int64_t n_perm, int mb,
                     int step0, float lr, float adam_eps, int target_interval, float* scratch, float* stats, void* stream) {
  if (!r4bq::dims_ok(algo, obs_dim, action_size) || !params || (algo != r4bq::BC && !target) || !m || !v || !bq_data_ok(data) ||
      !hp || !perm || n_perm < 1 || mb < 1 || step0 < 0 || !scratch)
    return fail(R4_ERR_ARG, "r4_batchrl_epoch: bad argument");
  const int64_t steps = n_perm / mb;
  if (steps > (int64_t)0x7fffffff - step0) return fail(R4_ERR_ARG, "r4_batchrl_epoch: too many steps");
  const r4bq::Layout L = r4bq::make_layout(algo, obs_dim, action_size);
  float* grad = r4bq::make_planes(scratch, L, mb).grad;
  cudaStream_t st = S(stream);
  for (int64_t k = 0; k < steps; ++k) {
    const int step = step0 + (int)k + 1;
    const int copy = L.ntgt > 0 && target_interval > 0 && (step - 1) % target_interval == 0;
    int rc = bq_grad(algo, obs_dim, action_size, params, target, data, hp, perm + k * mb, mb, scratch, grad,
                     stats ? stats + 3 * k : nullptr, st, true);
    if (rc) return rc;
    if ((rc = bq_apply(algo, obs_dim, action_size, params, target, grad, m, v, step, lr, adam_eps, copy, st, true))) return rc;
  }
  return (int)steps;
}

int r4_batchrl_act(int algo, int obs_dim, int action_size, const float* params, const void* obs, int obs_f64, int n,
                   const r4_batchrl_data* data, int mode, float log_flex, int32_t* action, float* probs, float* values,
                   void* stream) {
  if (!r4bq::dims_ok(algo, obs_dim, action_size) || !params || !obs || n < 1 || !data || !data->location_mask ||
      !data->special || mode < 0 || mode > 1 || !action)
    return fail(R4_ERR_ARG, "r4_batchrl_act: bad argument");
  const r4bq::Layout L = r4bq::make_layout(algo, obs_dim, action_size);
  r4bq::Data D{};
  D.locm = data->location_mask; D.special = data->special;
  return launch(FAM_BATCHRL, "k_bq_act", r4bq::k_bq_act, (n + r4bq::TS - 1) / r4bq::TS, r4bq::NT,
                r4bq::act_smem(obs_dim, action_size), S(stream), false, L, params, obs_f64 ? nullptr : (const float*)obs,
                obs_f64 ? (const double*)obs : nullptr, n, D, mode, log_flex, action, probs, values);
}

}  // extern "C"

// ---- training the DIEN simulator (r4_simtrain.cuh) -------------------------------------------------------------------
// kernels launched by the r4_simtrain_* entry points in this process (the radix sort counted once)
int64_t r4_simtrain_launch_count(void) { return g_launches[FAM_SIMTRAIN].load(std::memory_order_relaxed); }

static bool st_hash_ok(int H) { return H >= 1 && H <= r4st::MAXH; }
static bool st_head_ok(int head) { return head >= 0 && head < r4st::NHEAD; }

int64_t r4_simtrain_head_num_params(int head, int hash_size) {
  return st_head_ok(head) && st_hash_ok(hash_size) ? r4st::make_layout(hash_size, r4st::head_classes(head)).n : -1;
}
int64_t r4_simtrain_head_scratch_size(int head, int n) {
  return (!st_head_ok(head) || n < 1 || n > r4st::MAXN) ? -1 : (int64_t)r4st::scratch_bytes(n, r4st::head_classes(head));
}
int64_t r4_simtrain_num_params(int hash_size) { return r4_simtrain_head_num_params(R4_SIMHEAD_ITEM, hash_size); }
int64_t r4_simtrain_scratch_size(int n) { return r4_simtrain_head_scratch_size(R4_SIMHEAD_ITEM, n); }

template <typename... P, typename... A>
static int st_launch(const char* name, void (*kernel)(P...), dim3 grid, int threads, cudaStream_t st, A&&... args) {
  return launch(FAM_SIMTRAIN, name, kernel, grid, threads, 0, st, false, std::forward<A>(args)...);
}

static r4st::Data st_data(const r4_simtrain_data* d) {
  return r4st::Data{d->user_cat, d->user_dense, d->sequence_id, d->items, d->feedback, d->item_feature, d->seq};
}
static bool st_data_ok(const r4_simtrain_data* d) {
  return d && d->user_cat && d->user_dense && d->sequence_id && d->items && d->feedback && d->item_feature && d->seq;
}

static int st_gemm(bool tb, const float* A, int lda, const float* B, int ldb, const float* bias, float* C, int ldc, int M, int N,
                   int K, int epi, cudaStream_t st, const float* aux = nullptr, const float* mul = nullptr, float* pre = nullptr,
                   int accum = 0) {
  const r4st::Gemm g{A, lda, B, ldb, bias, C, ldc, M, N, K, epi, accum, aux, mul, pre};
  const dim3 grid((N + r4st::GT - 1) / r4st::GT, (M + r4st::GT - 1) / r4st::GT);
  return st_launch("k_st_gemm", tb ? r4st::k_st_gemm<true> : r4st::k_st_gemm<false>, grid, r4st::NTH, st, g);
}

// The forward with saved activations: gather, towers, both sequences (GRU-1, attention, AUGRU), the head and the loss.
static int st_forward(int head, const r4st::Layout& L, const float* prm, const r4st::Data& D, const int64_t* idx, int n,
                      uint64_t seed, uint64_t counter, float rate, const uint8_t* keep_in, uint8_t* keep_out, const r4st::Planes& P,
                      bool with_grad, float* stats, double* acc, float* probs, cudaStream_t st) {
  using namespace r4st;
  const int R = n * T, C = head_classes(head);
  const GatherArgs ga{L, D, idx, n, seed, counter, rate, keep_in, keep_out, head != HEAD_ITEM};
  int rc;
  if ((rc = st_launch("k_st_gather", k_st_gather, n, E, st, ga, prm, P))) return rc;
  const float* keep0 = P.keep;
  const float* keep1 = P.keep + (size_t)n * U;
  if ((rc = st_gemm(false, P.dense, ND, prm + L.dw1, U, prm + L.db1, P.T1d, U, n, U, ND, EP_ELU, st, nullptr, keep0, P.T1))) return rc;
  if ((rc = st_gemm(false, P.T1d, U, prm + L.dw2, U, prm + L.db2, P.allf + F_DENSE, FEAT, n, U, U, EP_ELU, st, nullptr, keep1, P.T2)))
    return rc;
  for (int i = 0; i < 2; ++i) {
    const Seq& w = L.s[i];
    const SeqPlanes& s = P.sp[i];
    if ((rc = st_gemm(false, s.X, E, prm + w.gwg, 2 * E, prm + w.gbg, s.XG1, 2 * E, R, 2 * E, E, EP_LIN, st))) return rc;
    if ((rc = st_gemm(false, s.X, E, prm + w.gwc, E, prm + w.gbc, s.XC1, E, R, E, E, EP_LIN, st))) return rc;
    const RecArgs<E> g1{prm + w.gwg + E * 2 * E, prm + w.gwc + E * E, s.XG1, s.XC1, nullptr, s.Hp1, s.G1, s.C1, s.RH1, s.H1, nullptr, 0, n};
    if ((rc = st_launch("k_st_gru_fwd<128>", k_st_gru_fwd<E>, (n + SB - 1) / SB, NTH, st, g1))) return rc;
    if ((rc = st_launch("k_st_attin", k_st_attin, (unsigned)(((size_t)R * E + 255) / 256), 256, st, P.q, s.H1, s.Ain, n))) return rc;
    if ((rc = st_gemm(false, s.Ain, 4 * E, prm + w.aw1, A1, prm + w.ab1, s.At1, A1, R, A1, 4 * E, EP_SIG, st))) return rc;
    if ((rc = st_gemm(false, s.At1, A1, prm + w.aw2, A2, prm + w.ab2, s.At2, A2, R, A2, A1, EP_SIG, st))) return rc;
    if ((rc = st_gemm(false, s.At2, A2, prm + w.ak, 1, prm + w.ab, s.S, 1, R, 1, A2, EP_LIN, st))) return rc;
    if ((rc = st_gemm(false, s.H1, E, prm + w.uwg, 4 * E, prm + w.ubg, s.XG2, 4 * E, R, 4 * E, E, EP_LIN, st))) return rc;
    if ((rc = st_gemm(false, s.H1, E, prm + w.uwc, 2 * E, prm + w.ubc, s.XC2, 2 * E, R, 2 * E, E, EP_LIN, st))) return rc;
    const RecArgs<HA> g2{prm + w.uwg + E * 4 * E, prm + w.uwc + E * 2 * E, s.XG2, s.XC2, s.S, s.Hp2, s.G2, s.C2, s.RH2, nullptr,
                         P.allf + i * HA, FEAT, n};
    if ((rc = st_launch("k_st_gru_fwd<256>", k_st_gru_fwd<HA>, (n + SB - 1) / SB, NTH, st, g2))) return rc;
  }
  if ((rc = st_gemm(false, P.allf, FEAT, prm + L.ow, OBS, prm + L.ob, P.O, OBS, n, OBS, FEAT, EP_ELU, st))) return rc;
  if ((rc = st_gemm(false, P.O, OBS, prm + L.rw, C, prm + L.rb, P.Z, C, n, C, OBS, EP_LIN, st))) return rc;
  float* dZ = with_grad ? P.dZ : nullptr;
  if (head == HEAD_SLATE)
    return st_launch("k_st_loss_slate<9>", k_st_loss_slate<NS>, 1, NTH, st, D, idx, n, P.Z, dZ, P.stats, stats, acc, probs);
  if (head == HEAD_SLATE_MULTICLASS)
    return st_launch("k_st_loss_slate<22>", k_st_loss_slate<NMC>, 1, NTH, st, D, idx, n, P.Z, dZ, P.stats, stats, acc, probs);
  return st_launch("k_st_loss", k_st_loss, 1, NTH, st, D, idx, n, P.Z, dZ, P.stats, stats, acc, probs);
}

static r4ddpg::Job st_job(const float* X, int ldx, const float* Z, int M, int N, int64_t off) {
  return r4ddpg::Job{X, Z, ldx, M, N, (int)off, 0};
}
static int st_wgrad(r4ddpg::Jobs J, int njob, int rows, float* grad, cudaStream_t st) {
  J.njob = njob;
  int t = 0;
  for (int i = 0; i < njob; ++i) {
    J.j[i].tile0 = t;
    t += ((J.j[i].M + r4ddpg::WT - 1) / r4ddpg::WT) * ((J.j[i].N + r4ddpg::WT - 1) / r4ddpg::WT);
  }
  J.ntiles = t;
  return st_launch("k_ddpg_wgrad", r4ddpg::k_ddpg_wgrad, t, r4ddpg::NT, st, J, rows, grad, nullptr, nullptr, 0.f);
}

static int st_backward(int head, const r4st::Layout& L, const float* prm, const r4st::Data& D, const int64_t* idx, int n,
                       const r4st::Planes& P, float* grad, cudaStream_t st) {
  using namespace r4st;
  const int R = n * T, C = head_classes(head);
  int rc;
  // head: dO = dZ rew_w^T elu'(O); dAllf = dO obs_w^T; the dense tower's columns again with its activation and dropout
  if ((rc = st_gemm(true, P.dZ, C, prm + L.rw, C, nullptr, P.dO, OBS, n, OBS, C, EP_DELU, st, P.O))) return rc;
  if ((rc = st_gemm(true, P.dO, OBS, prm + L.ow, OBS, nullptr, P.dAllf, FEAT, n, FEAT, OBS, EP_LIN, st))) return rc;
  if ((rc = st_gemm(true, P.dO, OBS, prm + L.ow + (int64_t)F_DENSE * OBS, OBS, nullptr, P.dT2, U, n, U, OBS, EP_DELU, st, P.T2,
                    P.keep + (size_t)n * U)))
    return rc;
  if ((rc = st_gemm(true, P.dT2, U, prm + L.dw2, U, nullptr, P.dT1, U, n, U, U, EP_DELU, st, P.T1, P.keep))) return rc;
  if ((rc = st_launch("k_st_cat_bwd", k_st_cat_bwd, n, E, st, P.allf, P.P, P.dAllf, P.dEcat))) return rc;
  for (int i = 0; i < 2; ++i) {
    const Seq& w = L.s[i];
    const SeqPlanes& s = P.sp[i];
    const RecBack<HA> b2{prm + w.uwg + E * 4 * E, prm + w.uwc + E * 2 * E, s.Hp2, s.G2, s.C2, s.S, nullptr, P.dAllf + i * HA, FEAT,
                         s.XG2, s.XC2, s.dS, n};
    if ((rc = st_launch("k_st_gru_bwd<256>", k_st_gru_bwd<HA>, (n + SB - 1) / SB, NTH, st, b2))) return rc;
    if ((rc = st_gemm(true, s.XG2, 4 * E, prm + w.uwg, 4 * E, nullptr, s.dH1, E, R, E, 4 * E, EP_LIN, st))) return rc;
    if ((rc = st_gemm(true, s.XC2, 2 * E, prm + w.uwc, 2 * E, nullptr, s.dH1, E, R, E, 2 * E, EP_LIN, st, nullptr, nullptr,
                      nullptr, 1)))
      return rc;
    if ((rc = st_gemm(true, s.dS, 1, prm + w.ak, 1, nullptr, s.dA2, A2, R, A2, 1, EP_DSIG, st, s.At2))) return rc;
    if ((rc = st_gemm(true, s.dA2, A2, prm + w.aw2, A2, nullptr, s.dA1, A1, R, A1, A2, EP_DSIG, st, s.At1))) return rc;
    if ((rc = st_gemm(true, s.dA1, A1, prm + w.aw1, A1, nullptr, s.dAin, 4 * E, R, 4 * E, A1, EP_LIN, st))) return rc;
    if ((rc = st_launch("k_st_attin_bwd", k_st_attin_bwd, n, E, st, P.q, s.H1, s.dAin, s.dH1, s.dq))) return rc;
    const RecBack<E> b1{prm + w.gwg + E * 2 * E, prm + w.gwc + E * E, s.Hp1, s.G1, s.C1, nullptr, s.dH1, nullptr, 0, s.XG1, s.XC1,
                        nullptr, n};
    if ((rc = st_launch("k_st_gru_bwd<128>", k_st_gru_bwd<E>, (n + SB - 1) / SB, NTH, st, b1))) return rc;
    if ((rc = st_gemm(true, s.XG1, 2 * E, prm + w.gwg, 2 * E, nullptr, s.dX, E, R, E, 2 * E, EP_LIN, st))) return rc;
    if ((rc = st_gemm(true, s.XC1, E, prm + w.gwc, E, nullptr, s.dX, E, R, E, E, EP_LIN, st, nullptr, nullptr, nullptr, 1)))
      return rc;
  }
  // dense weight gradients: one launch over the n-row jobs, one per sequence over its 64 n-row jobs
  r4ddpg::Jobs J;
  int k = 0;
  J.j[k++] = st_job(P.dense, ND, P.dT1, ND, U, L.dw1);  J.j[k++] = st_job(nullptr, 1, P.dT1, 1, U, L.db1);
  J.j[k++] = st_job(P.T1d, U, P.dT2, U, U, L.dw2);      J.j[k++] = st_job(nullptr, 1, P.dT2, 1, U, L.db2);
  J.j[k++] = st_job(P.allf, FEAT, P.dO, FEAT, OBS, L.ow); J.j[k++] = st_job(nullptr, 1, P.dO, 1, OBS, L.ob);
  J.j[k++] = st_job(P.O, OBS, P.dZ, OBS, C, L.rw);      J.j[k++] = st_job(nullptr, 1, P.dZ, 1, C, L.rb);
  if ((rc = st_wgrad(J, k, n, grad, st))) return rc;
  for (int i = 0; i < 2; ++i) {
    const Seq& w = L.s[i];
    const SeqPlanes& s = P.sp[i];
    k = 0;
    J.j[k++] = st_job(s.X, E, s.XG1, E, 2 * E, w.gwg);   J.j[k++] = st_job(s.Hp1, E, s.XG1, E, 2 * E, w.gwg + E * 2 * E);
    J.j[k++] = st_job(nullptr, 1, s.XG1, 1, 2 * E, w.gbg);
    J.j[k++] = st_job(s.X, E, s.XC1, E, E, w.gwc);       J.j[k++] = st_job(s.RH1, E, s.XC1, E, E, w.gwc + E * E);
    J.j[k++] = st_job(nullptr, 1, s.XC1, 1, E, w.gbc);
    J.j[k++] = st_job(s.Ain, 4 * E, s.dA1, 4 * E, A1, w.aw1); J.j[k++] = st_job(nullptr, 1, s.dA1, 1, A1, w.ab1);
    J.j[k++] = st_job(s.At1, A1, s.dA2, A1, A2, w.aw2);  J.j[k++] = st_job(nullptr, 1, s.dA2, 1, A2, w.ab2);
    J.j[k++] = st_job(s.At2, A2, s.dS, A2, 1, w.ak);     J.j[k++] = st_job(nullptr, 1, s.dS, 1, 1, w.ab);
    J.j[k++] = st_job(s.H1, E, s.XG2, E, 4 * E, w.uwg);  J.j[k++] = st_job(s.Hp2, HA, s.XG2, HA, 4 * E, w.uwg + E * 4 * E);
    J.j[k++] = st_job(nullptr, 1, s.XG2, 1, 4 * E, w.ubg);
    J.j[k++] = st_job(s.H1, E, s.XC2, E, 2 * E, w.uwc);  J.j[k++] = st_job(s.RH2, HA, s.XC2, HA, 2 * E, w.uwc + E * 2 * E);
    J.j[k++] = st_job(nullptr, 1, s.XC2, 1, 2 * E, w.ubc);
    if ((rc = st_wgrad(J, k, R, grad, st))) return rc;
  }
  // embedding gradients: keys, a stable radix sort by (table, id), one ordered sum per run
  const int total = n * NSLOT;
  if ((rc = st_launch("k_st_dq", k_st_dq, (n * E + 255) / 256, 256, st, P.sp[0].dq, P.sp[1].dq, P.dqs, n))) return rc;
  if ((rc = st_launch("k_st_embkeys", k_st_embkeys, (total + 255) / 256, 256, st, L, D, idx, n, (int)(head != HEAD_ITEM), P.cat, P.keys,
                       P.vals))) return rc;
  int bits = 1;
  while (bits < 32 && ((uint64_t)1 << bits) < (uint64_t)(2 * L.H)) ++bits;
  cub::DoubleBuffer<uint32_t> kb(P.keys, P.keys2);
  cub::DoubleBuffer<int32_t> vb(P.vals, P.vals2);
  size_t need = 0;
  if (cub::DeviceRadixSort::SortPairs(nullptr, need, kb, vb, total, 0, bits, st) != cudaSuccess || need > P.cub_bytes)
    return fail(R4_ERR_NOMEM, "r4_simtrain: radix sort temporary storage exceeds the scratch reserve");
  size_t have = P.cub_bytes;
  if (cub::DeviceRadixSort::SortPairs(P.cub_tmp, have, kb, vb, total, 0, bits, st) != cudaSuccess)
    return fail(R4_ERR_CUDA, std::string("cub::DeviceRadixSort: ") + cudaGetErrorString(cudaGetLastError()));
  count_launch(FAM_SIMTRAIN);      // the sort's own launches count as one
  return st_launch("k_st_embsum", k_st_embsum, total, EST, st, L, kb.Current(), vb.Current(), total, P.dEcat, P.sp[0].dX,
                   P.sp[1].dX, P.dqs, grad);
}

static int st_apply(int head, int H, float* params, float* grad, float* m, float* v, int step, float lr, float b1, float b2,
                    float eps, cudaStream_t st) {
  const r4st::Layout L = r4st::make_layout(H, r4st::head_classes(head));
  const double alpha = (double)lr * std::sqrt(1.0 - std::pow((double)b2, step)) / (1.0 - std::pow((double)b1, step));
  return st_launch("k_st_apply", r4st::k_st_apply, (unsigned)((L.n + 255) / 256), 256, st, L, params, grad, m, v, (float)alpha,
                   b1, b2, eps);
}

int r4_simtrain_head_grad(int head, int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx, int n,
                          uint64_t seed, uint64_t counter, float drop_rate, const uint8_t* keep_in, uint8_t* keep_out,
                          void* scratch, float* grad, float* stats, double* acc, void* stream) {
  if (!st_head_ok(head) || !st_hash_ok(hash_size) || !params || !st_data_ok(data) || !idx || n < 1 || n > r4st::MAXN ||
      !(drop_rate >= 0.f) || !(drop_rate < 1.f) || !scratch || !grad)
    return fail(R4_ERR_ARG, "r4_simtrain_grad: bad argument (head 0..2, hash_size 1..4000000, n 1..4096, drop_rate in [0, 1))");
  const int C = r4st::head_classes(head);
  const r4st::Layout L = r4st::make_layout(hash_size, C);
  const r4st::Planes P = r4st::make_planes(scratch, n, C);
  const r4st::Data D = st_data(data);
  cudaStream_t st = S(stream);
  int rc = st_forward(head, L, params, D, idx, n, seed, counter, drop_rate, keep_in, keep_out, P, true, stats, acc, nullptr, st);
  return rc ? rc : st_backward(head, L, params, D, idx, n, P, grad, st);
}

int r4_simtrain_head_apply(int head, int hash_size, float* params, float* grad, float* m, float* v, int step, float lr,
                           float beta1, float beta2, float eps, void* stream) {
  if (!st_head_ok(head) || !st_hash_ok(hash_size) || !params || !grad || !m || !v || step < 1)
    return fail(R4_ERR_ARG, "r4_simtrain_apply: bad argument");
  return st_apply(head, hash_size, params, grad, m, v, step, lr, beta1, beta2, eps, S(stream));
}

int r4_simtrain_head_step(int head, int hash_size, float* params, float* grad, float* m, float* v, const r4_simtrain_data* data,
                          const int64_t* idx, int n, uint64_t seed, uint64_t counter, float drop_rate, int step, float lr,
                          float beta1, float beta2, float eps, void* scratch, float* stats, double* acc, void* stream) {
  if (!m || !v || step < 1) return fail(R4_ERR_ARG, "r4_simtrain_step: bad argument");
  int rc = r4_simtrain_head_grad(head, hash_size, params, data, idx, n, seed, counter, drop_rate, nullptr, nullptr, scratch, grad,
                                 stats, acc, stream);
  return rc ? rc : st_apply(head, hash_size, params, grad, m, v, step, lr, beta1, beta2, eps, S(stream));
}

int r4_simtrain_head_eval(int head, int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx, int n,
                          void* scratch, float* probs, double* acc, void* stream) {
  if (!st_head_ok(head) || !st_hash_ok(hash_size) || !params || !st_data_ok(data) || !idx || n < 1 || n > r4st::MAXN || !scratch)
    return fail(R4_ERR_ARG, "r4_simtrain_eval: bad argument");
  const int C = r4st::head_classes(head);
  const r4st::Layout L = r4st::make_layout(hash_size, C);
  const r4st::Planes P = r4st::make_planes(scratch, n, C);
  return st_forward(head, L, params, st_data(data), idx, n, 0, 0, 0.f, nullptr, nullptr, P, false, nullptr, acc, probs, S(stream));
}

// the item head's entry points
int r4_simtrain_grad(int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx, int n, uint64_t seed,
                     uint64_t counter, float drop_rate, const uint8_t* keep_in, uint8_t* keep_out, void* scratch, float* grad,
                     float* stats, double* acc, void* stream) {
  return r4_simtrain_head_grad(R4_SIMHEAD_ITEM, hash_size, params, data, idx, n, seed, counter, drop_rate, keep_in, keep_out,
                               scratch, grad, stats, acc, stream);
}

int r4_simtrain_apply(int hash_size, float* params, float* grad, float* m, float* v, int step, float lr, float beta1, float beta2,
                      float eps, void* stream) {
  return r4_simtrain_head_apply(R4_SIMHEAD_ITEM, hash_size, params, grad, m, v, step, lr, beta1, beta2, eps, stream);
}

int r4_simtrain_step(int hash_size, float* params, float* grad, float* m, float* v, const r4_simtrain_data* data,
                     const int64_t* idx, int n, uint64_t seed, uint64_t counter, float drop_rate, int step, float lr, float beta1,
                     float beta2, float eps, void* scratch, float* stats, double* acc, void* stream) {
  return r4_simtrain_head_step(R4_SIMHEAD_ITEM, hash_size, params, grad, m, v, data, idx, n, seed, counter, drop_rate, step, lr,
                               beta1, beta2, eps, scratch, stats, acc, stream);
}

int r4_simtrain_eval(int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx, int n, void* scratch,
                     float* probs, double* acc, void* stream) {
  return r4_simtrain_head_eval(R4_SIMHEAD_ITEM, hash_size, params, data, idx, n, scratch, probs, acc, stream);
}
