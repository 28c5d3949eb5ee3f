// r4_learn.cu -- host side of the learner entry points of include/rl4rs_b200.h: PPO / A2C, the peer-memory gradient
// exchange, the Gaussian policy, DDPG / TD3, RAINBOW, PA-DQN, batch RL and the simulator trainer.  Stateless: every call enqueues
// its kernels on the caller's stream through r4h::launch, which counts them (r4_learner_launch_count).  See DESIGN.md.
#include "../../include/rl4rs_b200.h"
#include "r4_host.h"
#include "r4_ppo.cuh"
#include "r4_comm.cuh"
#include "r4_gauss.cuh"
#include "r4_ddpg.cuh"
#include "r4_rainbow.cuh"
#include "r4_batchrl.cuh"
#include "r4_cqlconti.cuh"
#include "r4_bcqconti.cuh"
#include "r4_simtrain.cuh"
#include "r4_dense.cuh"
#include "r4_exactk.cuh"
#include "r4_seq2seq.cuh"
#include "r4_ope.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <initializer_list>
#include <string>
#include <vector>

using namespace r4h;
using namespace r4dense;

// Dynamic shared memory starts at one offset for every kernel of a module, aligned for the module's most-aligned
// extern __shared__ array.  The env module's tensor-core kernels align theirs to 1024 bytes; the learner kernels were
// tuned at that alignment, and at 16 bytes k_policy_grad (whose weights arrive by bulk copy) runs about 6 % slower on an
// H100.  This never-launched kernel keeps a 1024-byte-aligned array in use, so the learner module keeps the alignment.
extern __shared__ __align__(1024) uint8_t r4_learn_smem_align[];
__global__ void r4_learn_smem_align_anchor() { r4_learn_smem_align[threadIdx.x] = 0; }

// ---- the shared dense kernels (r4_dense.cuh): every family launches k_dense_gemm and k_dense_wgrad through these -----------
namespace {
unsigned blocks(int64_t n, int per) { return (unsigned)((n + per - 1) / per); }

// a [rows, cols] row-major matrix at leading dimension ld as a GEMM operand, or its transpose
Op rm(const float* p, int64_t ld) { return Op{p, 0, 0, ld, 1}; }
Op tr(const float* p, int64_t ld) { return Op{p, 0, 0, 1, ld}; }

// k_dense_gemm over the 64 x 64 tiles of C in z batches
int dense_gemm(Family fam, cudaStream_t st, const Gemm& g, unsigned z) {
  return launch(fam, "k_dense_gemm", gemm_kernel(g), dim3(blocks(g.N, GT), blocks(g.M, GT), z), NT, 0, st, false, g);
}

// C[M, N] (ldc) (+ C when accum) = epi(A B + bias), aux the forward activation of a derivative epilogue; pre and mul as
// k_dense_gemm's epilogue
int dense_mm(Family fam, cudaStream_t st, Op A, Op B, float* C, int64_t ldc, int M, int N, int K, const float* bias = nullptr,
             int accum = 0, int epi = EP_LIN, const float* aux = nullptr, const float* mul = nullptr, float* pre = nullptr) {
  return dense_gemm(fam, st, Gemm{A, B, C, 0, 0, ldc, 1, bias, aux, mul, pre, M, N, K, 1, 0, 1.f, epi, accum}, 1);
}

// Per (group, head) products C = alpha A B, batch z = g H + h, element (m, n) of C at C + g cso + h csi + m cs0 + n.
// ktot > 0: split-K instead, G partials (H = 1) of K rows each out of ktot, partial g at C + g cso.
int dense_bmm(Family fam, cudaStream_t st, Op A, Op B, float* C, int64_t cso, int64_t csi, int64_t cs0, int M, int N, int K,
              int64_t G, int H, float alpha, int64_t ktot = 0) {
  const Gemm g{A, B, C, cso, csi, cs0, 1, nullptr, nullptr, nullptr, nullptr, M, N, K, H, ktot, alpha, EP_LIN, 0};
  return dense_gemm(fam, st, g, (unsigned)(G * H));
}

// k_dense_wgrad over the tiled jobs J on n rows (first: store the gradients, else add them), with its ntiles + 1 CTAs:
// the last sums the statistics s, and returns at once without them.
int dense_wgrad(Family fam, cudaStream_t st, const Jobs& J, int64_t n, int first, float* grad, const Stats& s = Stats{}) {
  return launch(fam, "k_dense_wgrad", k_dense_wgrad, J.ntiles + 1, NT, 0, st, false, J, (int)n, first, grad, s);
}
}  // namespace

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
  // the norm in one CTA and a fixed order, so that two clipped steps from the same state are bit-identical
  if (clip > 0.f)
    if (int rc = launch(FAM_ONLINE, "k_sumsq_one", r4ppo::k_sumsq_one, 1, r4ppo::SQT, 0, S(stream), false, n, grad, norm_scratch))
      return rc;
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

// The communicator check every entry point that takes one makes first, before it launches or writes anything: a
// communicator whose peers are not mapped yet (r4_comm_open; world 1 is ready at creation) is R4_ERR_STATE, one created
// for another parameter count R4_ERR_ARG.  NULL passes: the single-GPU form of the entry points that allow it.
static int comm_check(const r4_comm* c, int np, const char* who) {
  if (!c) return R4_OK;
  if (!c->ready) return fail(R4_ERR_STATE, std::string(who) + ": open the peers' handles first (r4_comm_open)");
  if (np != c->n) return fail(R4_ERR_ARG, std::string(who) + ": parameter count differs from the communicator's");
  return R4_OK;
}

// The exchange kernel.  Its callers have checked the communicator up front (comm_check); the same check here is the
// backstop in front of k_exchange_adam, which stores through and spins on the peers' pointers (null until r4_comm_open).
// Either way a refused call never reaches the ++seq.
static int exchange_launch(r4_comm* c, const float* scratch, int G, int np, float* flat, float* stats_accum, float stat_scale,
                           int do_adam, float* params, float* m, float* v, int step, float lr, float b1, float b2, float eps,
                           void* stream) {
  if (int rc = comm_check(c, np, "r4_comm")) return rc;
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
  if (!c || !params || !perm || !m || !v || !scratch || n < 1 || mb < 1 || mb > n || step0 < 0 || action_size < 2 ||
      action_size > 512)
    return fail(R4_ERR_ARG, "r4_ppo_epoch_dist: bad argument");
  const int np = r4ppo::make_layout(action_size).n;
  if (int rc = comm_check(c, np, "r4_ppo_epoch_dist")) return rc;
  const int G = std::max(1, std::min((mb + r4ppo::TS - 1) / r4ppo::TS, sm_count()));
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
  if (int rc = comm_check(c, n_params, "r4_grad_exchange_n")) return rc;
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
  const Jobs J = r4gauss::make_jobs(L, P);
  for (int c0 = 0; c0 < n; c0 += r4gauss::CH) {
    const int cn = std::min(r4gauss::CH, n - c0);
    const bool last = c0 + cn >= n;
    int rc = launch(FAM_ONLINE, "k_gauss_rows", r4gauss::k_gauss_rows, (cn + r4gauss::TS - 1) / r4gauss::TS, r4gauss::NT,
                    r4gauss::ROWS_SMEM, S(stream), false, L, hp, params, obs, action, old_logp, old_dist, old_value, adv, target,
                    idx, c0, cn, P);
    if (!rc)
      rc = dense_wgrad(FAM_ONLINE, S(stream), J, cn, c0 == 0, grad_out,
                       Stats{P.stats, 5, stat_sum, last ? stats_accum : nullptr, stat_scale, 1});
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
  if (int rc = comm_check(c, np, "r4_gauss_ppo_epoch_dist")) return rc;
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

int r4_impala_step(r4_comm* comm, float* params, const float* obs, const uint8_t* mask, const int64_t* action,
                   const float* behaviour_logp, const float* logits, const float* reward, int T, int B, int action_size,
                   float gamma, float rho_bar, float rho_pg_bar, int drop_last, float vf_coeff, float ent_coeff, float* logp,
                   float* value, float* vs, float* pg_adv, float* scratch, float* flat_grad, float* stats_accum, float* m,
                   float* v, int step, float lr, float beta1, float beta2, float eps, float grad_clip, float* norm_scratch,
                   void* stream) {
  if (!params || !obs || !mask || !action || !behaviour_logp || !logits || !reward || !logp || !value || !vs || !pg_adv ||
      !scratch || !flat_grad || !m || !v || step < 1 || (grad_clip > 0.f && !norm_scratch) || action_size < 2 ||
      action_size > 512 || !vtrace_args_ok(T, B, gamma, rho_bar, rho_pg_bar, drop_last))
    return fail(R4_ERR_ARG, "r4_impala_step: bad argument");
  const int np = r4ppo::make_layout(action_size).n;
  if (int rc = comm_check(comm, np, "r4_impala_step")) return rc;
  const int n = T * B, nk = (drop_last ? T - 1 : T) * B;          // the kept rows are the first T - 1 (or T) time steps
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
      !vtrace_args_ok(T, B, gamma, rho_bar, rho_pg_bar, drop_last))
    return fail(R4_ERR_ARG, "r4_gauss_impala_step: bad argument");
  const int np = r4gauss::make_layout(action_dim).n;
  if (int rc = comm_check(comm, np, "r4_gauss_impala_step")) return rc;
  const int n = T * B, nk = (drop_last ? T - 1 : T) * B;
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
  const Jobs J = r4ddpg::make_jobs(L, P);
  const r4ddpg::Replay R{r_obs, r_action, r_reward, r_new_obs, r_done};
  const r4ddpg::Hyper hp{gamma, target_noise, noise_clip, inv_n};
  if (int rc = launch(FAM_ONLINE, "k_ddpg_rows", r4ddpg::k_ddpg_rows, (n + r4ddpg::TS - 1) / r4ddpg::TS, r4ddpg::NT,
                      r4ddpg::ROWS_SMEM, S(stream), false, L, hp, params, target, R, idx, weights, smooth_noise, n, P))
    return rc;
  return dense_wgrad(FAM_ONLINE, S(stream), J, n, 1, grad, Stats{P.stats, 3, nullptr, stats, inv_n, 0});
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
  if (int rc = comm_check(comm, np, "r4_ddpg_train_step")) return rc;
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
  const Jobs J = r4rb::make_jobs(L, P);
  const r4rb::Replay R{r_obs, r_action, r_reward, r_new_obs, r_done};
  const r4rb::Hyper hp{v_min, v_max, (v_max - v_min) / (float)(num_atoms - 1), gamma_n, inv_n};
  if (int rc = launch(FAM_ONLINE, "k_rainbow_rows", r4rb::k_rainbow_rows, (n + r4rb::TS - 1) / r4rb::TS, r4rb::NT,
                      r4rb::rows_smem(L.A, L.AZ), S(stream), false, L, hp, params, target, R, idx, weights, n, P))
    return rc;
  return dense_wgrad(FAM_ONLINE, S(stream), J, n, 1, grad, Stats{P.stats, 3, nullptr, stats, inv_n, 0});
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
  if (int rc = comm_check(comm, L.n, "r4_rainbow_train_step")) return rc;
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

// ---- PA-DQN (r4_padqn.cuh) ----------------------------------------------------------------------------------
static bool padqn_dims_ok(int A, int D) { return A >= 2 && A <= r4pa::MAXA && D >= 1 && D <= r4pa::MAXD; }
// n rows: k_dense_gemm puts the 64-row tiles of S = obs w1[:256] + b1 on gridDim.y (at most 65535), and the flat pair
// index of the scorer's tiles stays an int (implied by the first bound at every A <= 512; kept as a guard)
static bool padqn_rows_ok(int A, int n) {
  return n >= 1 && n <= r4pa::MAXN && (int64_t)n * A <= (int64_t)0x7fffffff - r4pa::PM;
}
// the scratch and the caches are read by float4 loads and bulk copies
static bool a16(const void* p) { return ((uintptr_t)p & 15) == 0; }

int r4_padqn_num_params(int num_actions, int emb_dim) {
  return padqn_dims_ok(num_actions, emb_dim) ? r4pa::make_layout(num_actions, emb_dim).n : -1;
}

int64_t r4_padqn_scratch_size(int num_actions, int emb_dim, int n) {
  if (!padqn_dims_ok(num_actions, emb_dim) || !padqn_rows_ok(num_actions, n)) return -1;
  return (int64_t)r4pa::scratch_floats(r4pa::make_layout(num_actions, emb_dim), n);
}

int64_t r4_padqn_cache_size(int num_actions) {
  return num_actions >= 2 && num_actions <= r4pa::MAXA ? (int64_t)r4pa::cache_bytes(num_actions) : -1;
}

int r4_padqn_refresh(const float* params, const float* emb, int num_actions, int emb_dim, uint8_t* cache, uint8_t* cache2,
                     void* stream) {
  if (!params || !emb || !cache || cache == cache2 || !a16(cache) || !a16(cache2) || !padqn_dims_ok(num_actions, emb_dim))
    return fail(R4_ERR_ARG, "r4_padqn_refresh: bad argument");
  return launch(FAM_ONLINE, "k_padqn_refresh", r4pa::k_padqn_refresh, r4pa::IMG_CTAS + num_actions, 256, 0, S(stream), false,
                r4pa::make_layout(num_actions, emb_dim), params, emb, cache, cache2);
}

// Qm [n][A] of the rows S [n][256] against the cache's items: the pair scorer, one persistent CTA per SM at most
static int padqn_pairs(const r4pa::Layout& L, const float* params, const uint8_t* cache, const float* s, const uint8_t* mask,
                       int n, float* qm, cudaStream_t st) {
  const int64_t tiles = ((int64_t)n * L.A + r4pa::PM - 1) / r4pa::PM;
  return launch(FAM_ONLINE, "k_padqn_pairs", r4pa::k_padqn_pairs, (unsigned)std::min<int64_t>(tiles, sm_count()),
                r4pa::PTHREADS, r4pa::PAIRS_SMEM, st, false, s, cache, params, L, mask, n, qm);
}

int r4_padqn_act(const float* params, const uint8_t* cache, const float* obs, const uint8_t* mask, int n, int num_actions,
                 int emb_dim, int explore, uint64_t seed, uint64_t counter, int32_t* action, float* q, float* scratch,
                 void* stream) {
  if (!params || !cache || !obs || !mask || !action || !scratch || !a16(cache) || !a16(scratch) ||
      !padqn_dims_ok(num_actions, emb_dim) || !padqn_rows_ok(num_actions, n))
    return fail(R4_ERR_ARG, "r4_padqn_act: bad argument (actions 2..512, emb_dim 1..512, n 1..4194240)");
  const r4pa::Layout L = r4pa::make_layout(num_actions, emb_dim);
  const r4pa::Planes P = r4pa::make_planes(scratch, L, n);
  float* qm = q ? q : P.q_on;
  cudaStream_t st = S(stream);
  int rc = dense_mm(FAM_ONLINE, st, rm(obs, r4pa::OBS), rm(params + L.w1, r4pa::H), P.s_on, r4pa::H, n, r4pa::H, r4pa::OBS,
                    params + L.b1);
  if (!rc) rc = padqn_pairs(L, params, cache, P.s_on, mask, n, qm, st);
  if (rc) return rc;
  return launch(FAM_ONLINE, "k_padqn_act", r4pa::k_padqn_act, blocks(n, r4pa::NT / 32), r4pa::NT, 0, st, false, qm, n,
                num_actions, explore != 0, seed, counter, action);
}

int r4_padqn_store(float* r_obs, int32_t* r_action, float* r_reward, float* r_new_obs, uint8_t* r_done, uint8_t* r_next_mask,
                   float* r_prio, const float* max_prio, int capacity, int num_actions, int64_t pos, float alpha,
                   const float* obs, const float* final_obs, const uint8_t* mask, const uint8_t* final_mask,
                   const int32_t* action, const float* reward, const uint8_t* done, int T, int B, void* stream) {
  if (!r_obs || !r_action || !r_reward || !r_new_obs || !r_done || !r_next_mask || (r_prio && !max_prio) || capacity < 1 ||
      pos < 0 || num_actions < 2 || num_actions > r4pa::MAXA || !obs || !final_obs || !mask || !final_mask || !action ||
      !reward || !done || T < 1 || B < 1)
    return fail(R4_ERR_ARG, "r4_padqn_store: bad argument");
  const int64_t rows = std::min<int64_t>((int64_t)T * B, capacity);
  const r4pa::Ring R{r_obs, r_action, r_reward, r_new_obs, r_done, r_next_mask};
  return launch(FAM_ONLINE, "k_padqn_store", r4pa::k_padqn_store, (unsigned)rows, 64, 0, S(stream), false, R, r_prio, max_prio,
                capacity, num_actions, pos, alpha, obs, final_obs, mask, final_mask, action, reward, done, T, B);
}

int r4_padqn_grad(const float* params, const float* target, const uint8_t* cache, const uint8_t* target_cache, const float* emb,
                  int num_actions, int emb_dim, const float* r_obs, const int32_t* r_action, const float* r_reward,
                  const float* r_new_obs, const uint8_t* r_done, const uint8_t* r_next_mask, const int64_t* idx,
                  const float* weights, int n, float gamma, float inv_n, float* scratch, float* grad, float* td, float* stats,
                  void* stream) {
  if (!params || !target || !cache || !target_cache || !emb || !padqn_dims_ok(num_actions, emb_dim) || !r_obs || !r_action ||
      !r_reward || !r_new_obs || !r_done || !r_next_mask || !idx || !padqn_rows_ok(num_actions, n) || !scratch || !grad ||
      !a16(scratch) || !a16(cache) || !a16(target_cache))
    return fail(R4_ERR_ARG, "r4_padqn_grad: bad argument");
  const r4pa::Layout L = r4pa::make_layout(num_actions, emb_dim);
  r4pa::Planes P = r4pa::make_planes(scratch, L, n);
  if (td) P.td = td;
  cudaStream_t st = S(stream);
  using r4pa::H;
  using r4pa::OBS;
  int rc = launch(FAM_ONLINE, "k_padqn_gather", r4pa::k_padqn_gather, n, 128, 0, st, false, r_new_obs, r_next_mask, num_actions,
                  idx, P.x2, P.m2);
  if (!rc) rc = dense_mm(FAM_ONLINE, st, rm(P.x2, OBS), rm(params + L.w1, H), P.s_on, H, n, H, OBS, params + L.b1);
  if (!rc) rc = dense_mm(FAM_ONLINE, st, rm(P.x2, OBS), rm(target + L.w1, H), P.s_tg, H, n, H, OBS, target + L.b1);
  if (!rc) rc = padqn_pairs(L, params, cache, P.s_on, P.m2, n, P.q_on, st);
  if (!rc) rc = padqn_pairs(L, target, target_cache, P.s_tg, P.m2, n, P.q_tg, st);
  if (!rc) rc = launch(FAM_ONLINE, "k_padqn_rows", r4pa::k_padqn_rows, blocks(n, r4pa::TS), r4pa::NT, r4pa::rows_smem(L), st,
                       false, L, params, emb, r4pa::Replay{r_obs, r_action, r_reward, r_done}, gamma, inv_n, idx, weights, n, P);
  if (rc) return rc;
  return dense_wgrad(FAM_ONLINE, st, r4pa::make_jobs(L, P), n, 1, grad, Stats{P.stats, 3, nullptr, stats, inv_n, 0});
}

int r4_padqn_apply(float* params, float* target, const float* grad, float* m, float* v, const float* emb, int num_actions,
                   int emb_dim, uint8_t* cache, uint8_t* target_cache, int step, float lr, float adam_eps, float grad_clip,
                   int copy_target, void* stream) {
  if (!params || !target || !grad || !m || !v || !emb || !cache || !target_cache || cache == target_cache || !a16(cache) ||
      !a16(target_cache) || !padqn_dims_ok(num_actions, emb_dim) || step < 1)
    return fail(R4_ERR_ARG, "r4_padqn_apply: bad argument");
  const r4pa::Layout L = r4pa::make_layout(num_actions, emb_dim);
  // k_rainbow_apply over PA-DQN's 6 tensors; the split's other 6 entries are empty and own no CTA
  r4rb::Split Sp;
  const int st6[7] = {L.w1, L.b1, L.w2, L.b2, L.w3, L.b3, L.n};
  Sp.cta0[0] = 0;
  for (int k = 0; k <= r4rb::NTEN; ++k) Sp.start[k] = k < 7 ? st6[k] : L.n;
  for (int k = 0; k < r4rb::NTEN; ++k) Sp.cta0[k + 1] = Sp.cta0[k] + (Sp.start[k + 1] - Sp.start[k] + r4rb::ACH - 1) / r4rb::ACH;
  int rc = launch(FAM_ONLINE, "k_rainbow_apply", r4rb::k_rainbow_apply, Sp.cta0[r4rb::NTEN], r4rb::ANT, 0, S(stream), false, Sp,
                  params, target, grad, m, v, step, lr, adam_eps, grad_clip, copy_target != 0);
  if (rc) return rc;
  return r4_padqn_refresh(params, emb, num_actions, emb_dim, cache, copy_target ? target_cache : nullptr, stream);
}

int r4_padqn_train_step(float* params, float* target, float* m, float* v, const float* emb, uint8_t* cache,
                        uint8_t* target_cache, int num_actions, int emb_dim, const float* r_obs, const int32_t* r_action,
                        const float* r_reward, const float* r_new_obs, const uint8_t* r_done, const uint8_t* r_next_mask,
                        float* r_prio, float* max_prio, int size, int n, const float* u, float beta, float alpha,
                        float prio_eps, float gamma, int step, float lr, float adam_eps, float grad_clip, int copy_target,
                        float* scratch, float* stats, void* stream) {
  if (!scratch || !padqn_dims_ok(num_actions, emb_dim) || !padqn_rows_ok(num_actions, n) || (r_prio && !max_prio) ||
      size < 1 || !u || step < 1 || !params || !target || !m || !v || !emb || !cache || !target_cache || cache == target_cache ||
      !r_obs || !r_action || !r_reward || !r_new_obs || !r_done || !r_next_mask || !a16(scratch) || !a16(cache) ||
      !a16(target_cache))
    return fail(R4_ERR_ARG, "r4_padqn_train_step: bad argument");
  const r4pa::Planes P = r4pa::make_planes(scratch, r4pa::make_layout(num_actions, emb_dim), n);
  int rc = r4_replay_sample(r_prio, size, n, beta, u, P.idx, P.weights, stream);
  if (rc) return rc;
  rc = r4_padqn_grad(params, target, cache, target_cache, emb, num_actions, emb_dim, r_obs, r_action, r_reward, r_new_obs,
                     r_done, r_next_mask, P.idx, r_prio ? P.weights : nullptr, n, gamma, 1.0f / (float)n, scratch, P.grad,
                     nullptr, stats, stream);
  if (rc) return rc;
  rc = r4_padqn_apply(params, target, P.grad, m, v, emb, num_actions, emb_dim, cache, target_cache, step, lr, adam_eps,
                      grad_clip, copy_target, stream);
  if (rc || !r_prio) return rc;
  return r4_replay_update_priorities(r_prio, max_prio, P.idx, P.td, n, alpha, prio_eps, stream);
}

}  // extern "C"

// ---- batch RL: discrete BC / BCQ / CQL (r4_batchrl.cuh) -----------------------------------------------------------
namespace {
// The epoch of every batch-RL family: n_perm / mb SGD steps, step k (1-based step0 + k + 1) on the rows perm[k mb, (k + 1)
// mb) with its statistics at stats + nstat k.  -> the number of steps.
template <typename Step>
int batchrl_epoch(const char* fn, const int64_t* perm, int64_t n_perm, int mb, int step0, float* stats, int nstat,
                  Step&& sgd_step) {
  const int64_t steps = n_perm / mb;
  if (steps > (int64_t)0x7fffffff - step0) return fail(R4_ERR_ARG, std::string(fn) + ": too many steps");
  for (int64_t k = 0; k < steps; ++k) {
    const int rc = sgd_step(perm + k * mb, step0 + (int)k + 1, stats ? stats + nstat * k : nullptr);
    if (rc) return rc;
  }
  return (int)steps;
}

// the dataset planes of both continuous families (r4_cqlc_data) as their kernels take them; false when one is missing
bool conti_data(const r4_cqlc_data* d, r4cqlc::Data* out) {
  if (!d || !d->obs || !d->action || !d->reward || !d->terminal || !d->transitions) return false;
  *out = r4cqlc::Data{d->obs, d->action, d->reward, d->terminal, d->transitions};
  return true;
}
}  // namespace

extern "C" {

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
  const Jobs J = r4bq::make_jobs(L, P);
  if ((rc = dense_wgrad(FAM_BATCHRL, st, J, n, 1, grad, Stats{P.stats, 3, nullptr, stats, 1.0f / (float)n, 0}))) return rc;
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
  const r4bq::Layout L = r4bq::make_layout(algo, obs_dim, action_size);
  float* grad = r4bq::make_planes(scratch, L, mb).grad;
  cudaStream_t st = S(stream);
  return batchrl_epoch("r4_batchrl_epoch", perm, n_perm, mb, step0, stats, 3, [&](const int64_t* idx, int step, float* sk) {
    const int copy = L.ntgt > 0 && target_interval > 0 && (step - 1) % target_interval == 0;
    const int rc = bq_grad(algo, obs_dim, action_size, params, target, data, hp, idx, mb, scratch, grad, sk, st, true);
    return rc ? rc : bq_apply(algo, obs_dim, action_size, params, target, grad, m, v, step, lr, adam_eps, copy, st, true);
  });
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

// ---- batch RL: continuous-action CQL (r4_cqlconti.cuh), counted with the discrete learners ------------------------
namespace {
using r4cqlc::H;

// the relu MLP of net m on rows x [M][m.in] -> h1, h2 [M][H], out [M][m.out]
int cq_forward(cudaStream_t st, const float* prm, const r4cqlc::Net& m, const float* x, int M, float* h1, float* h2,
               float* out) {
  int rc;
  if ((rc = dense_mm(FAM_BATCHRL, st, rm(x, m.in), rm(prm + m.w1, H), h1, H, M, H, m.in, prm + m.b1, 0, EP_RELU))) return rc;
  if ((rc = dense_mm(FAM_BATCHRL, st, rm(h1, H), rm(prm + m.w2, H), h2, H, M, H, H, prm + m.b2, 0, EP_RELU))) return rc;
  return dense_mm(FAM_BATCHRL, st, rm(h2, H), rm(prm + m.w3, m.out), out, m.out, M, m.out, H, prm + m.b3);
}
// dout [M][m.out] -> dz2 = dout W3^T [h2 > 0], dz1 = dz2 W2^T [h1 > 0]
int cq_backward(cudaStream_t st, const float* prm, const r4cqlc::Net& m, const float* dout, int M, const float* h1,
                const float* h2, float* dz2, float* dz1) {
  int rc;
  if ((rc = dense_mm(FAM_BATCHRL, st, rm(dout, m.out), tr(prm + m.w3, m.out), dz2, H, M, H, m.out, nullptr, 0, EP_DRELU, h2)))
    return rc;
  return dense_mm(FAM_BATCHRL, st, rm(dz2, H), tr(prm + m.w2, H), dz1, H, M, H, H, nullptr, 0, EP_DRELU, h1);
}
// the six weight-gradient jobs of net m over rows x, h1, h2 and their output gradients dz1, dz2, dout
void cq_jobs(Jobs& J, int& k, const r4cqlc::Net& m, const float* x, const float* h1, const float* h2, const float* dz1,
             const float* dz2, const float* dout) {
  layer_jobs(J, k, x, m.in, dz1, m.in, H, m.w1, m.b1);
  layer_jobs(J, k, h1, H, dz2, H, H, m.w2, m.b2);
  layer_jobs(J, k, h2, H, dout, H, m.out, m.w3, m.b3);
}
template <typename... P, typename... A>
int cq_launch(const char* name, void (*kernel)(P...), unsigned grid, cudaStream_t st, bool pdl, A&&... args) {
  return launch(FAM_BATCHRL, name, kernel, grid, r4cqlc::NT, 0, st, pdl, std::forward<A>(args)...);
}

// One SGD step at 1-based step `step` (the noise counter): temperature, alpha, critic, actor.  apply: each phase's Adam
// (the critic's with the soft target update) runs before the next phase; else the phases' gradients at the given
// parameters go to P.grad and nothing is updated.  pdl: the r4cqlc kernels of the chain wait on griddepcontrol.
int cq_step(const r4cqlc::Layout& L, const r4cqlc::Hyper& hp, float* prm, float* tgt, float* m, float* v,
            const r4cqlc::Data& D, const int64_t* idx, int n, int step, int apply, const r4cqlc::Planes& P, float* stats,
            cudaStream_t st, bool pdl) {
  using namespace r4cqlc;
  const int S = hp.S, R = (1 + 2 * S) * n;
  const int ap = apply ? step : 1;
  int rc;
  if ((rc = cq_launch("k_cqlc_gather", k_cqlc_gather, 2 * sm_count(), st, pdl, L, hp, D, idx, n, (uint64_t)step, P))) return rc;
  if ((rc = cq_forward(st, prm, L.actor, P.xs, n, P.ah1, P.ah2, P.ao))) return rc;
  if ((rc = cq_launch("k_cqlc_temp", k_cqlc_temp, 1, st, pdl, L, hp, n, P, prm, m, v, ap, apply, stats))) return rc;
  // alpha
  if ((rc = cq_launch("k_cqlc_pack", k_cqlc_pack, blocks(R, NT / 32), st, pdl, L, S, n, (int)PK_ALPHA, P))) return rc;
  for (int k = 0; k < 2; ++k)
    if ((rc = cq_forward(st, prm, L.c[k], P.x, R, P.c[k].h1, P.c[k].h2, P.c[k].q))) return rc;
  if ((rc = cq_launch("k_cqlc_loss", k_cqlc_loss, 1, st, pdl, L, hp, n, (int)PH_ALPHA, P, prm, m, v, ap, apply, stats))) return rc;
  // critic: the target on s', then the critic rows
  if ((rc = cq_forward(st, prm, L.actor, P.xn, n, P.nh1, P.nh2, P.no))) return rc;
  if ((rc = cq_launch("k_cqlc_pack", k_cqlc_pack, blocks(n, NT / 32), st, pdl, L, S, n, (int)PK_TARGET, P))) return rc;
  for (int k = 0; k < 2; ++k)
    if ((rc = cq_forward(st, tgt, r4cqlc::make_net(L.c[k].w1 - L.t0, L.c[k].in, L.c[k].out), P.x, n, P.c[k].h1, P.c[k].h2,
                         P.qt + (size_t)k * n)))
      return rc;
  if ((rc = cq_launch("k_cqlc_pack", k_cqlc_pack, blocks(R, NT / 32), st, pdl, L, S, n, (int)PK_CRITIC, P))) return rc;
  for (int k = 0; k < 2; ++k)
    if ((rc = cq_forward(st, prm, L.c[k], P.x, R, P.c[k].h1, P.c[k].h2, P.c[k].q))) return rc;
  if ((rc = cq_launch("k_cqlc_loss", k_cqlc_loss, 1, st, pdl, L, hp, n, (int)PH_CRITIC, P, prm, m, v, ap, apply, stats))) return rc;
  Jobs J;
  int nj = 0;
  for (int k = 0; k < 2; ++k) {
    const CPlanes& c = P.c[k];
    if ((rc = cq_backward(st, prm, L.c[k], c.dq, R, c.h1, c.h2, c.dz2, c.dz1))) return rc;
    cq_jobs(J, nj, L.c[k], P.x, c.h1, c.h2, c.dz1, c.dz2, c.dq);
  }
  tile_jobs(J, nj);
  if ((rc = dense_wgrad(FAM_BATCHRL, st, J, R, 1, P.grad))) return rc;
  if (apply && (rc = cq_launch("k_cqlc_adam", k_cqlc_adam, blocks(L.ntgt, NT), st, pdl, L.t0, L.ntgt, prm,
                               (const float*)P.grad, m, v, step, hp.lr_critic, hp.eps, tgt, hp.tau)))
    return rc;
  // actor: d(-min_k Q_k)/da through the critics, then the squashed head and the actor's layers
  if ((rc = cq_launch("k_cqlc_pack", k_cqlc_pack, blocks(n, NT / 32), st, pdl, L, S, n, (int)PK_ACTOR, P))) return rc;
  for (int k = 0; k < 2; ++k)
    if ((rc = cq_forward(st, prm, L.c[k], P.x, n, P.c[k].h1, P.c[k].h2, P.c[k].q))) return rc;
  if ((rc = cq_launch("k_cqlc_loss", k_cqlc_loss, 1, st, pdl, L, hp, n, (int)PH_ACTOR, P, prm, m, v, ap, apply, stats))) return rc;
  for (int k = 0; k < 2; ++k) {
    const CPlanes& c = P.c[k];
    if ((rc = cq_backward(st, prm, L.c[k], c.dq, n, c.h1, c.h2, c.dz2, c.dz1))) return rc;
    if ((rc = dense_mm(FAM_BATCHRL, st, rm(c.dz1, H), tr(prm + L.c[k].w1 + (size_t)L.K * H, H), P.da, L.D, n, L.D, H, nullptr,
                       k)))
      return rc;
  }
  if ((rc = cq_launch("k_cqlc_head", k_cqlc_head, blocks((int64_t)n * L.D, NT), st, pdl, L, hp, n, P, (const float*)prm)))
    return rc;
  if ((rc = cq_backward(st, prm, L.actor, P.dout, n, P.ah1, P.ah2, P.adz2, P.adz1))) return rc;
  nj = 0;
  cq_jobs(J, nj, L.actor, P.xs, P.ah1, P.ah2, P.adz1, P.adz2, P.dout);
  tile_jobs(J, nj);
  if ((rc = dense_wgrad(FAM_BATCHRL, st, J, n, 1, P.grad))) return rc;
  if (apply && (rc = cq_launch("k_cqlc_adam", k_cqlc_adam, blocks(L.actor.end, NT), st, pdl, 0, L.actor.end, prm,
                               (const float*)P.grad, m, v, step, hp.lr_actor, hp.eps, (float*)nullptr, 0.f)))
    return rc;
  return R4_OK;
}

r4cqlc::Hyper cq_hyper(const r4_cqlc_hyper* h, int D) {
  return r4cqlc::Hyper{h->gamma, h->tau, h->adam_eps, h->alpha_threshold, h->conservative_weight, h->reward_mean,
                       h->reward_den, (float)((double)D * std::log(0.5)), h->lr_actor, h->lr_critic, h->lr_temp,
                       h->lr_alpha, h->n_action_samples, h->seed};
}
// the arguments r4_cqlc_grad and r4_cqlc_epoch share, and the dataset planes into *out
bool cq_args_ok(int K, int D, const r4_cqlc_data* d, const r4_cqlc_hyper* h, int n, r4cqlc::Data* out) {
  return r4cqlc::dims_ok(K, D) && conti_data(d, out) && h && h->n_action_samples >= 1 && h->n_action_samples <= r4cqlc::MAXS &&
         n >= 1 && n <= r4cqlc::MAXN;
}
}  // namespace

extern "C" {

int r4_cqlc_num_params(int obs_dim, int action_dim) {
  return r4cqlc::dims_ok(obs_dim, action_dim) ? r4cqlc::make_layout(obs_dim, action_dim).n : -1;
}

int r4_cqlc_target_size(int obs_dim, int action_dim) {
  return r4cqlc::dims_ok(obs_dim, action_dim) ? r4cqlc::make_layout(obs_dim, action_dim).ntgt : -1;
}

int64_t r4_cqlc_scratch_size(int obs_dim, int action_dim, int n_action_samples, int n) {
  if (!r4cqlc::dims_ok(obs_dim, action_dim) || n_action_samples < 1 || n_action_samples > r4cqlc::MAXS || n < 1 ||
      n > r4cqlc::MAXN)
    return -1;
  return (int64_t)r4cqlc::scratch_floats(r4cqlc::make_layout(obs_dim, action_dim), n_action_samples, n);
}

int64_t r4_cqlc_act_scratch_size(int obs_dim, int action_dim, int n) {
  if (!r4cqlc::dims_ok(obs_dim, action_dim) || n < 1 || n > r4cqlc::MAXACT) return -1;
  return (int64_t)r4cqlc::act_scratch_floats(r4cqlc::make_layout(obs_dim, action_dim), n);
}

int r4_cqlc_grad(int obs_dim, int action_dim, const float* params, const float* target, const r4_cqlc_data* data,
                 const r4_cqlc_hyper* hp, const int64_t* idx, int n, int step, float* scratch, float* grad, float* stats,
                 void* stream) {
  r4cqlc::Data D;
  if (!cq_args_ok(obs_dim, action_dim, data, hp, n, &D) || !params || !target || !idx || step < 1 || !scratch || !grad)
    return fail(R4_ERR_ARG, "r4_cqlc_grad: bad argument (obs_dim 1..4096, action_dim 1..512, n 1..4096, samples 1..64)");
  const r4cqlc::Layout L = r4cqlc::make_layout(obs_dim, action_dim);
  r4cqlc::Planes P = r4cqlc::make_planes(scratch, L, hp->n_action_samples, n);
  P.grad = grad;
  return cq_step(L, cq_hyper(hp, action_dim), const_cast<float*>(params), const_cast<float*>(target), nullptr, nullptr, D,
                 idx, n, step, 0, P, stats, S(stream), false);
}

int r4_cqlc_epoch(int obs_dim, int action_dim, float* params, float* target, float* m, float* v, const r4_cqlc_data* data,
                  const r4_cqlc_hyper* hp, const int64_t* perm, int64_t n_perm, int mb, int step0, float* scratch,
                  float* stats, void* stream) {
  r4cqlc::Data D;
  if (!cq_args_ok(obs_dim, action_dim, data, hp, mb, &D) || !params || !target || !m || !v || !perm || n_perm < 1 ||
      step0 < 0 || !scratch)
    return fail(R4_ERR_ARG, "r4_cqlc_epoch: bad argument");
  const r4cqlc::Layout L = r4cqlc::make_layout(obs_dim, action_dim);
  const r4cqlc::Planes P = r4cqlc::make_planes(scratch, L, hp->n_action_samples, mb);
  const r4cqlc::Hyper h = cq_hyper(hp, action_dim);
  return batchrl_epoch("r4_cqlc_epoch", perm, n_perm, mb, step0, stats, r4cqlc::NSTAT,
                       [&](const int64_t* idx, int step, float* sk) {
                         return cq_step(L, h, params, target, m, v, D, idx, mb, step, 1, P, sk, S(stream), true);
                       });
}

int r4_cqlc_act(int obs_dim, int action_dim, const float* params, const void* obs, int obs_f64, int n,
                const float* action_in, float* action, float* q, float* scratch, void* stream) {
  if (!r4cqlc::dims_ok(obs_dim, action_dim) || !params || !obs || n < 1 || n > r4cqlc::MAXACT || !scratch || (!action && !q))
    return fail(R4_ERR_ARG, "r4_cqlc_act: bad argument");
  using namespace r4cqlc;
  const Layout L = make_layout(obs_dim, action_dim);
  const int K = obs_dim, D = action_dim;
  cudaStream_t st = S(stream);
  float* p = scratch;
  float *x = p, *h1 = x + (size_t)n * K, *h2 = h1 + (size_t)n * H, *o = h2 + (size_t)n * H, *xa = o + (size_t)n * 2 * D;
  float* ch = xa + (size_t)n * (K + D);          // per critic: h1, h2 [n][H], q [n]
  const int64_t total = (int64_t)n * K;
  int rc;
  if ((rc = cq_launch("k_cqlc_obs", k_cqlc_obs, blocks(total, NT), st, false, obs_f64 ? nullptr : (const float*)obs,
                      obs_f64 ? (const double*)obs : nullptr, total, x)))
    return rc;
  if ((rc = cq_forward(st, params, L.actor, x, n, h1, h2, o))) return rc;
  if ((rc = cq_launch("k_cqlc_predict", k_cqlc_predict, blocks((int64_t)n * (K + D), NT), st, false, K, D, n,
                      (const float*)x, (const float*)o, action_in, action, q ? xa : nullptr)))
    return rc;
  if (!q) return R4_OK;
  float* qk[2];
  for (int k = 0; k < 2; ++k) {
    float* c = ch + (size_t)k * n * (2 * H + 1);
    qk[k] = c + (size_t)n * 2 * H;
    if ((rc = cq_forward(st, params, L.c[k], xa, n, c, c + (size_t)n * H, qk[k]))) return rc;
  }
  return cq_launch("k_cqlc_qmean", k_cqlc_qmean, blocks(n, NT), st, false, n, (const float*)qk[0], (const float*)qk[1], q);
}

}  // extern "C"

// ---- training the simulators (r4_simtrain.cuh): DIEN, the dnn / widedeep / lstm backbones and adversarial_slate --------
// kernels launched by the r4_simtrain_* entry points in this process (the radix sort counted once)
int64_t r4_simtrain_launch_count(void) { return g_launches[FAM_SIMTRAIN].load(std::memory_order_relaxed); }

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

// The pieces every net shares.  Lay / Pl are a net's layout and planes (Layout / Planes for DIEN, NLayout / NPlanes for the
// others), which name the dense tower's weights and planes alike.
// The dense tower with dropout: T1d = ELU(dense dw1 + db1) keep0 (T1 before the keep), out (ld ldo) = ELU(T1d dw2 + db2) keep1.
template <class Lay, class Pl>
static int st_tower(const Lay& L, const float* prm, const Pl& P, int n, float* out, int ldo, cudaStream_t st) {
  using namespace r4st;
  const int rc = dense_mm(FAM_SIMTRAIN, st, rm(P.dense, ND), rm(prm + L.dw1, U), P.T1d, U, n, U, ND, prm + L.db1, 0, EP_ELU,
                          nullptr, P.keep, P.T1);
  return rc ? rc : dense_mm(FAM_SIMTRAIN, st, rm(P.T1d, U), rm(prm + L.dw2, U), out, ldo, n, U, U, prm + L.db2, 0, EP_ELU,
                            nullptr, P.keep + (size_t)n * U, P.T2);
}
// Its backward from the layer above: dT2 = (dtop W^T) elu'(T2) keep1, with W the rows of that layer's weight (ld wide) the
// tower feeds, then dT1 = (dT2 dw2^T) elu'(T1) keep0.
template <class Lay, class Pl>
static int st_tower_bwd(const Lay& L, const float* prm, const Pl& P, int n, const float* dtop, const float* W, int ld, cudaStream_t st) {
  using namespace r4st;
  const int rc = dense_mm(FAM_SIMTRAIN, st, rm(dtop, ld), tr(W, ld), P.dT2, U, n, U, ld, nullptr, 0, EP_DELU, P.T2,
                          P.keep + (size_t)n * U);
  return rc ? rc : dense_mm(FAM_SIMTRAIN, st, rm(P.dT2, U), tr(prm + L.dw2, U), P.dT1, U, n, U, U, nullptr, 0, EP_DELU, P.T1,
                            P.keep);
}

// the tower's four weight-gradient jobs, the first of a net's n-row jobs; returns the job count
template <class Lay, class Pl>
static int st_tower_jobs(Jobs& J, const Lay& L, const Pl& P) {
  using namespace r4st;
  int k = 0;
  layer_jobs(J, k, P.dense, ND, P.dT1, ND, U, L.dw1, L.db1);
  layer_jobs(J, k, P.T1d, U, P.dT2, U, U, L.dw2, L.db2);
  return k;
}

// The head's loss: logits Z [n][C] -> dZ (may be NULL), the per-sample rows srow, stats, acc and probs.
static int st_loss(int head, const r4st::Data& D, const int64_t* idx, int n, const float* Z, float* dZ, float* srow, float* stats,
                   double* acc, float* probs, cudaStream_t st) {
  using namespace r4st;
  if (head == HEAD_ADV) return st_launch("k_st_loss_adv", k_st_loss_adv, 1, NTH, st, D, idx, n, Z, dZ, srow, stats, acc, probs);
  if (head == HEAD_SLATE)
    return st_launch("k_st_loss_slate<9>", k_st_loss_slate<NS>, 1, NTH, st, D, idx, n, Z, dZ, srow, stats, acc, probs);
  if (head == HEAD_SLATE_MULTICLASS)
    return st_launch("k_st_loss_slate<22>", k_st_loss_slate<NMC>, 1, NTH, st, D, idx, n, Z, dZ, srow, stats, acc, probs);
  return st_launch("k_st_loss", k_st_loss, 1, NTH, st, D, idx, n, Z, dZ, srow, stats, acc, probs);
}

// The embedding gradients: keys of every (sample, slot), a stable radix sort by (table, id), one ordered sum per run.
template <int NQ>
static int st_embgrad(const r4st::Slots& sl, const r4st::Data& D, const int64_t* idx, int n, int slate, const int32_t* cat,
                      const r4st::SortPlanes& sb, const float* dEcat, const float* dX0, const float* dX1, const float* dqs,
                      float* grad, cudaStream_t st) {
  const int total = n * r4st::slot_count<NQ>(sl);
  int rc;
  if ((rc = st_launch("k_st_embkeys", r4st::k_st_embkeys<NQ>, (total + 255) / 256, 256, st, sl, D, idx, n, slate, cat, sb.keys, sb.vals)))
    return rc;
  int bits = 1;
  while (bits < 32 && ((uint64_t)1 << bits) < (uint64_t)(2 * sl.H)) ++bits;
  cub::DoubleBuffer<uint32_t> kb(sb.keys, sb.keys2);
  cub::DoubleBuffer<int32_t> vb(sb.vals, sb.vals2);
  size_t need = 0;
  if (cub::DeviceRadixSort::SortPairs(nullptr, need, kb, vb, total, 0, bits, st) != cudaSuccess || need > sb.cub_bytes)
    return fail(R4_ERR_NOMEM, "r4_simtrain: radix sort temporary storage exceeds the scratch reserve");
  size_t have = sb.cub_bytes;
  if (cub::DeviceRadixSort::SortPairs(sb.cub_tmp, have, kb, vb, total, 0, bits, st) != cudaSuccess)
    return fail(R4_ERR_CUDA, std::string("cub::DeviceRadixSort: ") + cudaGetErrorString(cudaGetLastError()));
  count_launch(FAM_SIMTRAIN);      // the sort's own launches count as one
  return st_launch("k_st_embsum", r4st::k_st_embsum<NQ>, total, r4st::EST, st, sl, kb.Current(), vb.Current(), total, dEcat, dX0, dX1,
                   dqs, grad);
}

// DIEN's forward with saved activations: gather, towers, both sequences (GRU-1, attention, AUGRU), the head and the loss.
static int st_forward(int head, const r4st::Layout& L, const float* prm, const r4st::Data& D, const int64_t* idx, int n,
                      uint64_t seed, uint64_t counter, float rate, const uint8_t* keep_in, uint8_t* keep_out, const r4st::Planes& P,
                      bool with_grad, float* stats, double* acc, float* probs, cudaStream_t st) {
  using namespace r4st;
  const int R = n * T, C = head_classes(head);
  const GatherArgs ga{L.H, D, idx, n, seed, counter, rate, keep_in, keep_out, head != HEAD_ITEM};
  int rc;
  if ((rc = st_launch("k_st_gather", k_st_gather, n, E, st, ga, L.emb_cat, L.emb_seq, prm, P))) return rc;
  if ((rc = st_tower(L, prm, P, n, P.allf + F_DENSE, FEAT, st))) return rc;
  for (int i = 0; i < 2; ++i) {
    const Seq& w = L.s[i];
    const SeqPlanes& s = P.sp[i];
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.X, E), rm(prm + w.gwg, 2 * E), s.XG1, 2 * E, R, 2 * E, E, prm + w.gbg))) return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.X, E), rm(prm + w.gwc, E), s.XC1, E, R, E, E, prm + w.gbc))) return rc;
    const RecArgs<E> g1{prm + w.gwg + E * 2 * E, prm + w.gwc + E * E, s.XG1, s.XC1, nullptr, s.Hp1, s.G1, s.C1, s.RH1, s.H1, nullptr, 0, n};
    if ((rc = st_launch("k_st_gru_fwd<128>", k_st_gru_fwd<E>, (n + SB - 1) / SB, NTH, st, g1))) return rc;
    if ((rc = st_launch("k_st_attin", k_st_attin, (unsigned)(((size_t)R * E + 255) / 256), 256, st, P.q, s.H1, s.Ain, n))) return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.Ain, 4 * E), rm(prm + w.aw1, A1), s.At1, A1, R, A1, 4 * E, prm + w.ab1, 0, EP_SIG)))
      return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.At1, A1), rm(prm + w.aw2, A2), s.At2, A2, R, A2, A1, prm + w.ab2, 0, EP_SIG)))
      return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.At2, A2), rm(prm + w.ak, 1), s.S, 1, R, 1, A2, prm + w.ab))) return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.H1, E), rm(prm + w.uwg, 4 * E), s.XG2, 4 * E, R, 4 * E, E, prm + w.ubg))) return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.H1, E), rm(prm + w.uwc, 2 * E), s.XC2, 2 * E, R, 2 * E, E, prm + w.ubc))) return rc;
    const RecArgs<HA> g2{prm + w.uwg + E * 4 * E, prm + w.uwc + E * 2 * E, s.XG2, s.XC2, s.S, s.Hp2, s.G2, s.C2, s.RH2, nullptr,
                         P.allf + i * HA, FEAT, n};
    if ((rc = st_launch("k_st_gru_fwd<256>", k_st_gru_fwd<HA>, (n + SB - 1) / SB, NTH, st, g2))) return rc;
  }
  if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.allf, FEAT), rm(prm + L.ow, OBS), P.O, OBS, n, OBS, FEAT, prm + L.ob, 0, EP_ELU)))
    return rc;
  if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.O, OBS), rm(prm + L.rw, C), P.Z, C, n, C, OBS, prm + L.rb))) return rc;
  return st_loss(head, D, idx, n, P.Z, with_grad ? P.dZ : nullptr, P.stats, stats, acc, probs, st);
}

static int st_backward(int head, const r4st::Layout& L, const float* prm, const r4st::Data& D, const int64_t* idx, int n,
                       const r4st::Planes& P, float* grad, cudaStream_t st) {
  using namespace r4st;
  const int R = n * T, C = head_classes(head);
  int rc;
  // head: dO = dZ rew_w^T elu'(O); dAllf = dO obs_w^T; the dense tower's columns again with its activation and dropout
  if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.dZ, C), tr(prm + L.rw, C), P.dO, OBS, n, OBS, C, nullptr, 0, EP_DELU, P.O)))
    return rc;
  if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.dO, OBS), tr(prm + L.ow, OBS), P.dAllf, FEAT, n, FEAT, OBS))) return rc;
  if ((rc = st_tower_bwd(L, prm, P, n, P.dO, prm + L.ow + (int64_t)F_DENSE * OBS, OBS, st))) return rc;
  if ((rc = st_launch("k_st_cat_bwd", k_st_cat_bwd, n, E, st, P.allf, P.P, P.dAllf, P.dEcat))) return rc;
  for (int i = 0; i < 2; ++i) {
    const Seq& w = L.s[i];
    const SeqPlanes& s = P.sp[i];
    const RecBack<HA> b2{prm + w.uwg + E * 4 * E, prm + w.uwc + E * 2 * E, s.Hp2, s.G2, s.C2, s.S, nullptr, P.dAllf + i * HA, FEAT,
                         s.XG2, s.XC2, s.dS, n};
    if ((rc = st_launch("k_st_gru_bwd<256>", k_st_gru_bwd<HA>, (n + SB - 1) / SB, NTH, st, b2))) return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.XG2, 4 * E), tr(prm + w.uwg, 4 * E), s.dH1, E, R, E, 4 * E))) return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.XC2, 2 * E), tr(prm + w.uwc, 2 * E), s.dH1, E, R, E, 2 * E, nullptr, 1))) return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.dS, 1), tr(prm + w.ak, 1), s.dA2, A2, R, A2, 1, nullptr, 0, EP_DSIG, s.At2)))
      return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.dA2, A2), tr(prm + w.aw2, A2), s.dA1, A1, R, A1, A2, nullptr, 0, EP_DSIG, s.At1)))
      return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.dA1, A1), tr(prm + w.aw1, A1), s.dAin, 4 * E, R, 4 * E, A1))) return rc;
    if ((rc = st_launch("k_st_attin_bwd", k_st_attin_bwd, n, E, st, P.q, s.H1, s.dAin, s.dH1, s.dq))) return rc;
    const RecBack<E> b1{prm + w.gwg + E * 2 * E, prm + w.gwc + E * E, s.Hp1, s.G1, s.C1, nullptr, s.dH1, nullptr, 0, s.XG1, s.XC1,
                        nullptr, n};
    if ((rc = st_launch("k_st_gru_bwd<128>", k_st_gru_bwd<E>, (n + SB - 1) / SB, NTH, st, b1))) return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.XG1, 2 * E), tr(prm + w.gwg, 2 * E), s.dX, E, R, E, 2 * E))) return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(s.XC1, E), tr(prm + w.gwc, E), s.dX, E, R, E, E, nullptr, 1))) return rc;
  }
  // dense weight gradients: one launch over the n-row jobs, one per sequence over its 64 n-row jobs
  Jobs J;
  int k = st_tower_jobs(J, L, P);
  layer_jobs(J, k, P.allf, FEAT, P.dO, FEAT, OBS, L.ow, L.ob);
  layer_jobs(J, k, P.O, OBS, P.dZ, OBS, C, L.rw, L.rb);
  tile_jobs(J, k);
  if ((rc = dense_wgrad(FAM_SIMTRAIN, st, J, n, 1, grad))) return rc;
  for (int i = 0; i < 2; ++i) {
    const Seq& w = L.s[i];
    const SeqPlanes& s = P.sp[i];
    k = 0;
    // a GRU kernel's input rows and its recurrent rows are two jobs, the second with the bias
    J.j[k++] = grad_job(s.X, E, s.XG1, E, 2 * E, w.gwg);
    layer_jobs(J, k, s.Hp1, E, s.XG1, E, 2 * E, w.gwg + E * 2 * E, w.gbg);
    J.j[k++] = grad_job(s.X, E, s.XC1, E, E, w.gwc);
    layer_jobs(J, k, s.RH1, E, s.XC1, E, E, w.gwc + E * E, w.gbc);
    layer_jobs(J, k, s.Ain, 4 * E, s.dA1, 4 * E, A1, w.aw1, w.ab1);
    layer_jobs(J, k, s.At1, A1, s.dA2, A1, A2, w.aw2, w.ab2);
    layer_jobs(J, k, s.At2, A2, s.dS, A2, 1, w.ak, w.ab);
    J.j[k++] = grad_job(s.H1, E, s.XG2, E, 4 * E, w.uwg);
    layer_jobs(J, k, s.Hp2, HA, s.XG2, HA, 4 * E, w.uwg + E * 4 * E, w.ubg);
    J.j[k++] = grad_job(s.H1, E, s.XC2, E, 2 * E, w.uwc);
    layer_jobs(J, k, s.RH2, HA, s.XC2, HA, 2 * E, w.uwc + E * 2 * E, w.ubc);
    tile_jobs(J, k);
    if ((rc = dense_wgrad(FAM_SIMTRAIN, st, J, R, 1, grad))) return rc;
  }
  // embedding gradients: the 21 cat slots, both sequences and the query's 10 emb_seq slots (dqs)
  if ((rc = st_launch("k_st_dq", k_st_dq, (n * E + 255) / 256, 256, st, P.sp[0].dq, P.sp[1].dq, P.dqs, n))) return rc;
  const Slots sl{L.H, L.emb_cat, L.emb_seq, NC, 2 * T};
  return st_embgrad<10>(sl, D, idx, n, head != HEAD_ITEM, P.cat, P.sort, P.dEcat, P.sp[0].dX, P.sp[1].dX, P.dqs, grad, st);
}

// A backbone's forward with saved activations: the embedding front, the dense tower, lstm's three GRUs, the net's dense
// layers, the head and the loss.
static int sn_forward(int head, const r4st::NLayout& L, const float* prm, const r4st::Data& D, const int64_t* idx, int n,
                      uint64_t seed, uint64_t counter, float rate, const uint8_t* keep_in, uint8_t* keep_out,
                      const r4st::NPlanes& P, bool with_grad, float* stats, double* acc, float* probs, cudaStream_t st) {
  using namespace r4st;
  const GatherArgs ga{L.H, D, idx, n, seed, counter, rate, keep_in, keep_out, head != HEAD_ITEM};
  Front f{};
  f.ncp = L.ncp;
  if (L.net == NET_DNN) { f.cpool = P.A; f.ldc = L.FA; }
  if (L.net == NET_ADV) { f.cpool = P.A + 2 * E + U; f.ldc = L.FA; }
  if (L.net == NET_WIDEDEEP) { f.flat = P.O + OBS + U; f.ldf = L.FO; }
  if (L.net == NET_LSTM) { f.flat = P.A + 4 * U; f.ldf = L.FA; f.xc = P.g[0].X; f.xs0 = P.g[1].X; f.xs1 = P.g[2].X; }
  if (L.net == NET_WIDEDEEP || L.net == NET_ADV) { f.spool = P.A; f.lds = L.FA; }
  int rc;
  if ((rc = st_launch("k_st_front", k_st_front, n, E, st, ga, L.emb_cat, L.emb_seq, prm, P.cat, P.dense, P.keep, f))) return rc;
  float* tower = L.A_tower >= 0 ? P.A + L.A_tower : P.O + L.O_tower;
  const int ldt = L.A_tower >= 0 ? L.FA : L.FO;
  if ((rc = st_tower(L, prm, P, n, tower, ldt, st))) return rc;
  if (L.net == NET_LSTM) {
    const int col[3] = {3 * U, 0, U};             // the category GRU's state after the tower; the sequence GRUs first
    for (int i = 0; i < 3; ++i) {
      const GruPlanes& g = P.g[i];
      const int nt = i ? T : NC, R = n * nt;
      if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(g.X, E), rm(prm + L.g[i].k, NG3), g.XG, NG3, R, NG3, E, prm + L.g[i].b))) return rc;
      const KGru a{prm + L.g[i].rk, g.XG, g.Hp, g.A, g.HH, g.RH, P.A + col[i], L.FA, n, nt};
      if ((rc = st_launch("k_st_kgru_fwd", k_st_kgru_fwd, (n + SB - 1) / SB, NTH, st, a))) return rc;
    }
  }
  if (L.net == NET_DNN) {
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.A, L.FA), rm(prm + L.fcw, OBS), P.F, OBS, n, OBS, L.FA, prm + L.fcb, 0, EP_ELU)))
      return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.F, OBS), rm(prm + L.ow, OBS), P.O, OBS, n, OBS, OBS, prm + L.ob, 0, EP_ELU)))
      return rc;
  } else if (L.net == NET_WIDEDEEP) {             // O[:, :256], its activations kept apart in F for the backward
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.A, L.FA), rm(prm + L.fcw, OBS), P.O, L.FO, n, OBS, L.FA, prm + L.fcb, 0, EP_ELU,
                       nullptr, nullptr, P.F)))
      return rc;
  } else if (L.net == NET_LSTM) {
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.A, L.FA), rm(prm + L.ow, OBS), P.O, OBS, n, OBS, L.FA, prm + L.ob, 0, EP_ELU)))
      return rc;
  }
  const float* hin = L.FO ? P.O : P.A;
  if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(hin, L.FH), rm(prm + L.rw, L.C), P.Z, L.C, n, L.C, L.FH, prm + L.rb))) return rc;
  return st_loss(head, D, idx, n, P.Z, with_grad ? P.dZ : nullptr, P.srow, stats, acc, probs, st);
}

static int sn_backward(int head, const r4st::NLayout& L, const float* prm, const r4st::Data& D, const int64_t* idx, int n,
                       const r4st::NPlanes& P, float* grad, cudaStream_t st) {
  using namespace r4st;
  const int C = L.C;
  int rc;
  // the head and dense layers down to dA (the front's and GRUs' columns) and dT2 (the tower's output, with its activation
  // and dropout); Wt(w, r0) is the weight w from its row r0 on, read transposed
  auto Wt = [&](int64_t w, int r0, int ld) { return prm + w + (int64_t)r0 * ld; };
  int tower_r0 = 0, tower_ld = 0;
  const float* dtop = nullptr;
  if (L.net == NET_DNN) {
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.dZ, C), tr(Wt(L.rw, 0, C), C), P.dO, OBS, n, OBS, C, nullptr, 0, EP_DELU, P.O)))
      return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.dO, OBS), tr(Wt(L.ow, 0, OBS), OBS), P.dF, OBS, n, OBS, OBS, nullptr, 0, EP_DELU,
                       P.F)))
      return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.dF, OBS), tr(Wt(L.fcw, 0, OBS), OBS), P.dA, L.FA, n, E, OBS))) return rc;
    dtop = P.dF; tower_r0 = E; tower_ld = OBS;
  } else if (L.net == NET_WIDEDEEP) {
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.dZ, C), tr(Wt(L.rw, 0, C), C), P.dF, OBS, n, OBS, C, nullptr, 0, EP_DELU, P.F)))
      return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.dZ, C), tr(Wt(L.rw, OBS + U, C), C), P.dO + OBS + U, L.FO, n, NC * E, C)))
      return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.dF, OBS), tr(Wt(L.fcw, 0, OBS), OBS), P.dA, L.FA, n, L.FA, OBS))) return rc;
    dtop = P.dZ; tower_r0 = OBS; tower_ld = C;
  } else if (L.net == NET_LSTM) {
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.dZ, C), tr(Wt(L.rw, 0, C), C), P.dO, OBS, n, OBS, C, nullptr, 0, EP_DELU, P.O)))
      return rc;
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.dO, OBS), tr(Wt(L.ow, 0, OBS), OBS), P.dA, L.FA, n, L.FA, OBS))) return rc;
    dtop = P.dO; tower_r0 = L.A_tower; tower_ld = OBS;
  } else {
    if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(P.dZ, C), tr(Wt(L.rw, 0, C), C), P.dA, L.FA, n, L.FA, C))) return rc;
    dtop = P.dZ; tower_r0 = L.A_tower; tower_ld = C;
  }
  const int64_t tw = L.net == NET_DNN ? L.fcw : L.net == NET_LSTM ? L.ow : L.rw;
  if ((rc = st_tower_bwd(L, prm, P, n, dtop, Wt(tw, tower_r0, tower_ld), tower_ld, st))) return rc;
  // the embedding front: pools and Flatten; lstm's GRUs (BPTT) and their input gradients
  FrontBack fb{};
  fb.ncp = L.ncp;
  if (L.net == NET_DNN) { fb.dcpool = P.dA; fb.ldc = L.FA; }
  if (L.net == NET_ADV) { fb.dcpool = P.dA + 2 * E + U; fb.ldc = L.FA; }
  if (L.net == NET_WIDEDEEP) { fb.dflat = P.dO + OBS + U; fb.ldf = L.FO; }
  if (L.net == NET_LSTM) { fb.dflat = P.dA + 4 * U; fb.ldf = L.FA; }
  if (L.net == NET_WIDEDEEP || L.net == NET_ADV) { fb.dspool = P.dA; fb.lds = L.FA; }
  if ((rc = st_launch("k_st_front_bwd", k_st_front_bwd, n, E, st, fb, P.dEcat, P.dX[0], P.dX[1]))) return rc;
  if (L.net == NET_LSTM) {
    const int col[3] = {3 * U, 0, U};
    for (int i = 0; i < 3; ++i) {
      const GruPlanes& g = P.g[i];
      const int nt = i ? T : NC, R = n * nt;
      const KGruBack b{prm + L.g[i].rk, g.Hp, g.A, g.HH, P.dA + col[i], L.FA, g.dZR, g.dHH, n, nt};
      if ((rc = st_launch("k_st_kgru_bwd", k_st_kgru_bwd, (n + SB - 1) / SB, NTH, st, b))) return rc;
      float* dX = i ? P.dX[i - 1] : P.dEcat;      // the category GRU's input gradient adds to the Flatten one
      if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(g.dZR, 2 * U), tr(prm + L.g[i].k, NG3), dX, E, R, E, 2 * U, nullptr, i ? 0 : 1)))
        return rc;
      if ((rc = dense_mm(FAM_SIMTRAIN, st, rm(g.dHH, U), tr(prm + L.g[i].k + 2 * U, NG3), dX, E, R, E, U, nullptr, 1))) return rc;
    }
  }
  // dense weight gradients over the n-row jobs
  Jobs J;
  int k = st_tower_jobs(J, L, P);
  if (L.net == NET_DNN) {
    layer_jobs(J, k, P.A, L.FA, P.dF, L.FA, OBS, L.fcw, L.fcb);
    layer_jobs(J, k, P.F, OBS, P.dO, OBS, OBS, L.ow, L.ob);
  } else if (L.net == NET_WIDEDEEP) {
    layer_jobs(J, k, P.A, L.FA, P.dF, L.FA, OBS, L.fcw, L.fcb);
  } else if (L.net == NET_LSTM) {
    layer_jobs(J, k, P.A, L.FA, P.dO, L.FA, OBS, L.ow, L.ob);
  }
  const float* hin = L.FO ? P.O : P.A;
  layer_jobs(J, k, hin, L.FH, P.dZ, L.FH, C, L.rw, L.rb);
  tile_jobs(J, k);
  if ((rc = dense_wgrad(FAM_SIMTRAIN, st, J, n, 1, grad))) return rc;
  if (L.net == NET_LSTM) {
    // each GRU's [z | r] and h column blocks into gtmp, the category GRU's (21 n rows) then both sequence GRUs' (64 n rows)
    auto gru_jobs = [&](int i, int& kk) {
      const GruPlanes& g = P.g[i];
      const int64_t zr = (int64_t)i * GROWS * NG3, hc = zr + (int64_t)GROWS * 2 * U;
      J.j[kk++] = grad_job(g.X, E, g.dZR, E, 2 * U, zr);
      layer_jobs(J, kk, g.Hp, U, g.dZR, U, 2 * U, zr + (int64_t)E * 2 * U, zr + (int64_t)(E + U) * 2 * U);
      J.j[kk++] = grad_job(g.X, E, g.dHH, E, U, hc);
      layer_jobs(J, kk, g.RH, U, g.dHH, U, U, hc + (int64_t)E * U, hc + (int64_t)(E + U) * U);
    };
    k = 0;
    gru_jobs(0, k);
    tile_jobs(J, k);
    if ((rc = dense_wgrad(FAM_SIMTRAIN, st, J, n * NC, 1, P.gtmp))) return rc;
    k = 0;
    gru_jobs(1, k);
    gru_jobs(2, k);
    tile_jobs(J, k);
    if ((rc = dense_wgrad(FAM_SIMTRAIN, st, J, n * T, 1, P.gtmp))) return rc;
    if ((rc = st_launch("k_st_kgru_merge", k_st_kgru_merge, (3 * GROWS * NG3 + 255) / 256, 256, st, (const float*)P.gtmp, grad,
                        L.g[0].k, L.g[1].k, L.g[2].k)))
      return rc;
  }
  // embedding gradients: the net's pooled / Flattened cat slots and, but for dnn, both sequences
  const Slots sl{L.H, L.emb_cat, L.emb_seq, L.ncp, L.nseq};
  return st_embgrad<0>(sl, D, idx, n, head != HEAD_ITEM, P.cat, P.sort, P.dEcat, P.dX[0], P.dX[1], nullptr, grad, st);
}

// One pass of (net, head) over n samples: the forward with saved activations, then, with grad, the backward into grad.
static int st_pass(int net, int head, int H, const float* prm, const r4_simtrain_data* data, const int64_t* idx, int n,
                   uint64_t seed, uint64_t counter, float rate, const uint8_t* keep_in, uint8_t* keep_out, void* scratch,
                   float* grad, float* stats, double* acc, float* probs, cudaStream_t st) {
  using namespace r4st;
  const int C = head_classes(head);
  const Data D = st_data(data);
  int rc;
  if (net == NET_DIEN) {
    const Layout L = make_layout(H, C);
    const Planes P = make_planes(scratch, n, C);
    rc = st_forward(head, L, prm, D, idx, n, seed, counter, rate, keep_in, keep_out, P, grad != nullptr, stats, acc, probs, st);
    return rc || !grad ? rc : st_backward(head, L, prm, D, idx, n, P, grad, st);
  }
  const NLayout L = make_nlayout(net, H, C);
  const NPlanes P = make_nplanes(scratch, L, n);
  rc = sn_forward(head, L, prm, D, idx, n, seed, counter, rate, keep_in, keep_out, P, grad != nullptr, stats, acc, probs, st);
  return rc || !grad ? rc : sn_backward(head, L, prm, D, idx, n, P, grad, st);
}

// Keras Adam over every parameter of (net, head), clearing the embedding tables' gradient rows.
static int st_apply(int net, int head, int H, float* params, float* grad, float* m, float* v, int step, float lr, float b1, float b2,
                    float eps, cudaStream_t st) {
  using namespace r4st;
  const int C = head_classes(head);
  int64_t np, emb_cat, emb_seq;
  if (net == NET_DIEN) {
    const Layout L = make_layout(H, C);
    np = L.n; emb_cat = L.emb_cat; emb_seq = L.emb_seq;
  } else {
    const NLayout L = make_nlayout(net, H, C);
    np = L.n; emb_cat = L.emb_cat; emb_seq = L.emb_seq >= 0 ? L.emb_seq : L.emb_cat;
  }
  const double alpha = (double)lr * std::sqrt(1.0 - std::pow((double)b2, step)) / (1.0 - std::pow((double)b1, step));
  return st_launch("k_keras_adam", k_keras_adam, (unsigned)((np + 255) / 256), 256, st, np, (int64_t)H * E, emb_cat, emb_seq, params,
                   grad, m, v, (float)alpha, b1, b2, eps);
}

// The one argument check of every entry point: the (net, head) pair, the hash size, n, the drop rate, the Adam step and the
// pointers.  An entry point passes a valid value for what it does not take.
static bool st_args_ok(int net, int head, int H, int n, float rate, int step, std::initializer_list<const void*> ptrs) {
  using namespace r4st;
  for (const void* p : ptrs)
    if (!p) return false;
  const bool pair = net == NET_ADV ? head == HEAD_ADV : net >= 0 && net < NET_ADV && head >= 0 && head < HEAD_ADV;
  return pair && H >= 1 && H <= MAXH && n >= 1 && n <= MAXN && rate >= 0.f && rate < 1.f && step >= 1;
}
static int st_reject(const char* fn) {
  return fail(R4_ERR_ARG, std::string(fn) + ": bad argument (nets 0..3 take heads 0..2, net 4 head 3; hash_size 1..4000000, "
                                            "n 1..4096, drop_rate in [0, 1), step >= 1, no NULL pointer)");
}

int64_t r4_simtrain_net_num_params(int net, int head, int hash_size) {
  if (!st_args_ok(net, head, hash_size, 1, 0.f, 1, {})) return -1;
  const int C = r4st::head_classes(head);
  return net == r4st::NET_DIEN ? r4st::make_layout(hash_size, C).n : r4st::make_nlayout(net, hash_size, C).n;
}
int64_t r4_simtrain_net_scratch_size(int net, int head, int n) {
  if (!st_args_ok(net, head, 1, n, 0.f, 1, {})) return -1;
  const int C = r4st::head_classes(head);
  return (int64_t)(net == r4st::NET_DIEN ? r4st::scratch_bytes(n, C) : r4st::make_nplanes(nullptr, r4st::make_nlayout(net, 1, C), n).bytes);
}

int r4_simtrain_net_grad(int net, int head, int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx,
                         int n, uint64_t seed, uint64_t counter, float drop_rate, const uint8_t* keep_in, uint8_t* keep_out,
                         void* scratch, float* grad, float* stats, double* acc, void* stream) {
  if (!st_args_ok(net, head, hash_size, n, drop_rate, 1, {params, idx, scratch, grad}) || !st_data_ok(data))
    return st_reject("r4_simtrain_net_grad");
  return st_pass(net, head, hash_size, params, data, idx, n, seed, counter, drop_rate, keep_in, keep_out, scratch, grad, stats, acc,
                 nullptr, S(stream));
}

int r4_simtrain_net_apply(int net, int head, int hash_size, float* params, float* grad, float* m, float* v, int step, float lr,
                          float beta1, float beta2, float eps, void* stream) {
  if (!st_args_ok(net, head, hash_size, 1, 0.f, step, {params, grad, m, v})) return st_reject("r4_simtrain_net_apply");
  return st_apply(net, head, hash_size, params, grad, m, v, step, lr, beta1, beta2, eps, S(stream));
}

int r4_simtrain_net_step(int net, int head, int hash_size, float* params, float* grad, float* m, float* v,
                         const r4_simtrain_data* data, const int64_t* idx, int n, uint64_t seed, uint64_t counter, float drop_rate,
                         int step, float lr, float beta1, float beta2, float eps, void* scratch, float* stats, double* acc,
                         void* stream) {
  if (!st_args_ok(net, head, hash_size, n, drop_rate, step, {params, grad, m, v, idx, scratch}) || !st_data_ok(data))
    return st_reject("r4_simtrain_net_step");
  const int rc = st_pass(net, head, hash_size, params, data, idx, n, seed, counter, drop_rate, nullptr, nullptr, scratch, grad, stats,
                         acc, nullptr, S(stream));
  return rc ? rc : st_apply(net, head, hash_size, params, grad, m, v, step, lr, beta1, beta2, eps, S(stream));
}

int r4_simtrain_net_eval(int net, int head, int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx,
                         int n, void* scratch, float* probs, double* acc, void* stream) {
  if (!st_args_ok(net, head, hash_size, n, 0.f, 1, {params, idx, scratch}) || !st_data_ok(data))
    return st_reject("r4_simtrain_net_eval");
  return st_pass(net, head, hash_size, params, data, idx, n, 0, 0, 0.f, nullptr, nullptr, scratch, nullptr, nullptr, acc, probs,
                 S(stream));
}

// DIEN's heads: net 0
int64_t r4_simtrain_head_num_params(int head, int hash_size) { return r4_simtrain_net_num_params(R4_SIM_DIEN, head, hash_size); }
int64_t r4_simtrain_head_scratch_size(int head, int n) { return r4_simtrain_net_scratch_size(R4_SIM_DIEN, head, n); }

int r4_simtrain_head_grad(int head, int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx, int n,
                          uint64_t seed, uint64_t counter, float drop_rate, const uint8_t* keep_in, uint8_t* keep_out,
                          void* scratch, float* grad, float* stats, double* acc, void* stream) {
  return r4_simtrain_net_grad(R4_SIM_DIEN, head, hash_size, params, data, idx, n, seed, counter, drop_rate, keep_in, keep_out,
                              scratch, grad, stats, acc, stream);
}

int r4_simtrain_head_apply(int head, int hash_size, float* params, float* grad, float* m, float* v, int step, float lr,
                           float beta1, float beta2, float eps, void* stream) {
  return r4_simtrain_net_apply(R4_SIM_DIEN, head, hash_size, params, grad, m, v, step, lr, beta1, beta2, eps, stream);
}

int r4_simtrain_head_step(int head, int hash_size, float* params, float* grad, float* m, float* v, const r4_simtrain_data* data,
                          const int64_t* idx, int n, uint64_t seed, uint64_t counter, float drop_rate, int step, float lr,
                          float beta1, float beta2, float eps, void* scratch, float* stats, double* acc, void* stream) {
  return r4_simtrain_net_step(R4_SIM_DIEN, head, hash_size, params, grad, m, v, data, idx, n, seed, counter, drop_rate, step, lr,
                              beta1, beta2, eps, scratch, stats, acc, stream);
}

int r4_simtrain_head_eval(int head, int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx, int n,
                          void* scratch, float* probs, double* acc, void* stream) {
  return r4_simtrain_net_eval(R4_SIM_DIEN, head, hash_size, params, data, idx, n, scratch, probs, acc, stream);
}

// DIEN's item head: net 0, head 0
int64_t r4_simtrain_num_params(int hash_size) { return r4_simtrain_head_num_params(R4_SIMHEAD_ITEM, hash_size); }
int64_t r4_simtrain_scratch_size(int n) { return r4_simtrain_head_scratch_size(R4_SIMHEAD_ITEM, n); }

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

// ---- Exact-K (r4_exactk.cuh): the pointer-network generator and its reward critic ----------------------------------------
int64_t r4_exactk_launch_count(void) { return g_launches[FAM_EXACTK].load(std::memory_order_relaxed); }

namespace {

template <typename... P, typename... A>
int ek_launch(const char* name, void (*kernel)(P...), dim3 grid, int threads, size_t smem, cudaStream_t st, A&&... args) {
  return launch(FAM_EXACTK, name, kernel, grid, threads, smem, st, false, std::forward<A>(args)...);
}

constexpr int EK_SPLITS = 128;                 // split-K partials of a weight gradient at most
constexpr int64_t EK_KC = 1024;                // rows per split-K partial at least

// out[N] (+)= sum over R rows (stride rs) of in[r, (i / w) ls + i % w]: chunks of rows into partials, then their sum
// (two launches at every size, so a pass launches the same number of kernels for every n)
int ek_colsum(cudaStream_t st, const float* in, int64_t R, int64_t rs, int w, int64_t ls, int N, float* out, int accumulate,
              float* part, float scale = 1.f) {
  const int64_t S = std::max<int64_t>(1, std::min<int64_t>(EK_SPLITS, (R + EK_KC - 1) / EK_KC));
  const int64_t rc = (R + S - 1) / S;
  if (int rc2 = ek_launch("k_ek_colsum", r4ek::k_ek_colsum, dim3(blocks(N, 128), (unsigned)S), 128, 0, st, in, R, rs, w, ls, N,
                          rc, part, (int64_t)N, 1.f, 0))
    return rc2;
  return ek_launch("k_ek_colsum", r4ek::k_ek_colsum, dim3(blocks(N, 128), 1), 128, 0, st, (const float*)part, S, (int64_t)N, N,
                   (int64_t)0, N, S, out, (int64_t)0, scale, accumulate);
}

// dW[K, N] += X^T dY over R rows (X at ldx, dY at ldy): split-K partials, then their sum in order
int ek_wgrad(cudaStream_t st, const float* X, int64_t ldx, const float* dY, int64_t ldy, int64_t R, int K, int N, float* dW,
             float* part) {
  const int64_t S = std::min<int64_t>(EK_SPLITS, (R + EK_KC - 1) / EK_KC);
  const int64_t kc = (R + S - 1) / S;
  if (int rc = dense_bmm(FAM_EXACTK, st, tr(X, ldx), rm(dY, ldy), part, (int64_t)K * N, 0, N, K, N, (int)kc, S, 1, 1.f, R))
    return rc;
  return ek_launch("k_ek_colsum", r4ek::k_ek_colsum, dim3(blocks((int64_t)K * N, 128), 1), 128, 0, st, (const float*)part, S,
                   (int64_t)K * N, K * N, (int64_t)0, K * N, S, dW, (int64_t)0, 1.f, 1);
}

// a linear layer's gradients: dW += X^T dY, db += colsum dY
int ek_lin_grad(cudaStream_t st, const float* X, int64_t ldx, const float* dY, int64_t ldy, int64_t R, int K, int N, float* dW,
                float* db, float* part) {
  if (int rc = ek_wgrad(st, X, ldx, dY, ldy, R, K, N, dW, part)) return rc;
  return ek_colsum(st, dY, R, ldy, N, 0, N, db, 1, part);
}

// Scratch planes of the generator for n rows over T candidates (offsets in floats; path in int32 slots)
struct EkPlanes {
  int64_t uenc, X0, m[2], QKV[2], A[2], P[2], O[2], Y1[2], xh1[2], rs1[2], F1[2], Y2[2], xh2[2], rs2[2], eref[2];
  int64_t XH, G, C, H, IN, PI, HB, QB, A1, A2, P1, GL, logits, path, ce;
  int64_t dlog, deref[2], denc, dA1, dA2, dGL, dIN, dHs, dC, dHB, dQB, dG, dXH, rv;
  int64_t dY, dZ, dF1, dQKV, dP, gx, dU, part, n;
};
EkPlanes ek_planes(int64_t n, int64_t T) {
  using namespace r4ek;
  EkPlanes p;
  int64_t o = 0;
  auto take = [&](int64_t k) { int64_t r = o; o += (k + 63) / 64 * 64; return r; };
  const int64_t nT = n * T, S4 = n * NH * T * T;
  p.uenc = take(n * HU); p.X0 = take(nT * D);
  for (int l = 0; l < NBLK; ++l) {
    p.m[l] = take(nT); p.QKV[l] = take(nT * 3 * D); p.A[l] = take(S4); p.P[l] = take(S4); p.O[l] = take(nT * D);
    p.Y1[l] = take(nT * D); p.xh1[l] = take(nT * D); p.rs1[l] = take(nT); p.F1[l] = take(nT * FF); p.Y2[l] = take(nT * D);
    p.xh2[l] = take(nT * D); p.rs2[l] = take(nT);
  }
  p.eref[0] = take(nT * D); p.eref[1] = take(nT * D);
  p.XH = take(RES * n * 2 * D); p.G = take(RES * n * 4 * D); p.C = take(RES * n * D); p.H = take(RES * n * D);
  p.IN = take(RES * n * D); p.PI = take(RES * n * RES); p.HB = take(RES * n * D); p.QB = take(RES * n * D);
  p.A1 = take(RES * n * D); p.A2 = take(RES * n * D); p.P1 = take(RES * nT); p.GL = take(RES * n * D);
  p.logits = take(n * RES * T); p.path = take(n * RES); p.ce = take(n);
  p.dlog = take(nT); p.deref[0] = take(nT * D); p.deref[1] = take(nT * D); p.denc = take(nT * D);
  p.dA1 = take(RES * n * D); p.dA2 = take(RES * n * D); p.dGL = take(n * D); p.dIN = take(n * D); p.dHs = take(RES * n * D);
  p.dC = take(n * D); p.dHB = take(RES * n * D); p.dQB = take(RES * n * D); p.dG = take(RES * n * 4 * D);
  p.dXH = take(RES * n * 2 * D); p.rv = take(n * RV_N * D);
  p.dY = take(nT * D); p.dZ = take(nT * D); p.dF1 = take(nT * FF); p.dQKV = take(nT * 3 * D); p.dP = take(S4);
  p.gx = take(nT * D); p.dU = take(n * HU);
  p.part = take((int64_t)EK_SPLITS * 2 * D * 4 * D);
  p.n = o;
  return p;
}

bool ek_shape_ok(int n, int T) {
  return n >= 1 && n <= r4ek::MAXN && T >= r4ek::TMIN && T <= r4ek::TMAX && (int64_t)n * T * T <= r4ek::MAXNTT;
}

struct EkRun {
  const float* prm;
  r4ek::Layout L;
  int n, T;
  uint64_t seed, call;
  float rate;
  float* s;
  EkPlanes p;
  cudaStream_t st;
  float* f(int64_t off) const { return s + off; }
};

// the encoder forward: enc = Y2 of block 1; eref[a] = enc W_ref[a]
int ek_encoder(const EkRun& r, const float* user) {
  using namespace r4ek;
  const int n = r.n, T = r.T;
  const int64_t nT = (int64_t)n * T;
  const float* prm = r.prm;
  const Layout& L = r.L;
  cudaStream_t st = r.st;
  int rc;
  if ((rc = dense_mm(FAM_EXACTK, st, rm(user, UIN), rm(prm + L.u_w, HU), r.f(r.p.uenc), HU, n, HU, UIN, prm + L.u_b, 0, EP_RELU)))
    return rc;
  if ((rc = ek_launch("k_ek_input", k_ek_input, blocks(nT * D, 256), 256, 0, st, (const float*)r.f(r.p.uenc), prm + L.emb, n,
                      T, r.seed, r.call, r.rate, r.f(r.p.X0))))
    return rc;
  const float inv = 1.0f / sqrtf((float)DH);
  for (int l = 0; l < NBLK; ++l) {
    const Block& B = L.blk[l];
    const float* X = l == 0 ? r.f(r.p.X0) : r.f(r.p.Y2[0]);
    float* QKV = r.f(r.p.QKV[l]);
    float* S = r.f(r.p.dP);
    if ((rc = ek_launch("k_ek_rowmask", k_ek_rowmask, blocks(nT * 32, 256), 256, 0, st, X, nT, r.f(r.p.m[l])))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(X, D), rm(prm + B.qkv_w, 3 * D), QKV, 3 * D, (int)nT, 3 * D, D, prm + B.qkv_b, 0,
                       EP_RELU)))
      return rc;
    if ((rc = dense_bmm(FAM_EXACTK, st, Op{QKV, T * 3 * D, DH, 3 * D, 1}, Op{QKV + D, T * 3 * D, DH, 1, 3 * D}, S,
                        (int64_t)NH * T * T, (int64_t)T * T, T, T, T, DH, n, NH, inv)))
      return rc;
    if ((rc = ek_launch("k_ek_softmax", k_ek_softmax, blocks((int64_t)n * NH * T * 32, 256), 256, 0, st, (const float*)S,
                        (const float*)r.f(r.p.m[l]), n, T, r.seed, r.call, l == 0 ? ST_ATT0 : ST_ATT1, r.rate, r.f(r.p.A[l]),
                        r.f(r.p.P[l]))))
      return rc;
    if ((rc = dense_bmm(FAM_EXACTK, st, Op{r.f(r.p.P[l]), (int64_t)NH * T * T, (int64_t)T * T, T, 1},
                        Op{QKV + 2 * D, T * 3 * D, DH, 3 * D, 1}, r.f(r.p.O[l]), (int64_t)T * D, DH, D, T, DH, T, n, NH, 1.f)))
      return rc;
    if ((rc = ek_launch("k_ek_ln", k_ek_ln, blocks(nT * 32, 256), 256, 0, st, (const float*)r.f(r.p.O[l]), X, nT,
                        prm + B.ln1_b, prm + B.ln1_g, r.f(r.p.Y1[l]), r.f(r.p.xh1[l]), r.f(r.p.rs1[l]))))
      return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(r.f(r.p.Y1[l]), D), rm(prm + B.f1_w, FF), r.f(r.p.F1[l]), FF, (int)nT, FF, D,
                       prm + B.f1_b, 0, EP_RELU)))
      return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(r.f(r.p.F1[l]), FF), rm(prm + B.f2_w, D), r.f(r.p.dY), D, (int)nT, D, FF,
                       prm + B.f2_b)))
      return rc;
    if ((rc = ek_launch("k_ek_ln", k_ek_ln, blocks(nT * 32, 256), 256, 0, st, (const float*)r.f(r.p.dY),
                        (const float*)r.f(r.p.Y1[l]), nT, prm + B.ln2_b, prm + B.ln2_g, r.f(r.p.Y2[l]), r.f(r.p.xh2[l]),
                        r.f(r.p.rs2[l]))))
      return rc;
  }
  for (int a = 0; a < 2; ++a)
    if ((rc = dense_mm(FAM_EXACTK, st, rm(r.f(r.p.Y2[1]), D), rm(prm + L.att[a].w_ref, D), r.f(r.p.eref[a]), D, (int)nT, D, D)))
      return rc;
  return R4_OK;
}

r4ek::Dec ek_dec(const EkRun& r, const uint8_t* masks, int32_t* path, float* logits) {
  r4ek::Dec d;
  d.n = r.n; d.T = r.T;
  d.enc = r.f(r.p.Y2[1]);
  d.eref[0] = r.f(r.p.eref[0]); d.eref[1] = r.f(r.p.eref[1]);
  d.XH = r.f(r.p.XH); d.G = r.f(r.p.G); d.C = r.f(r.p.C); d.H = r.f(r.p.H); d.IN = r.f(r.p.IN); d.PI = r.f(r.p.PI);
  d.HB = r.f(r.p.HB); d.QB = r.f(r.p.QB); d.A1 = r.f(r.p.A1); d.A2 = r.f(r.p.A2); d.P1 = r.f(r.p.P1); d.GL = r.f(r.p.GL);
  d.logits = logits; d.path = path; d.masks = masks;
  return d;
}

// the nine decode steps (mode 0 SAMPLE, 1 GREEDY, 2 TRAIN on the path already in d.path)
int ek_decoder(const EkRun& r, const r4ek::Dec& d, int mode, float temperature) {
  using namespace r4ek;
  const int n = r.n, T = r.T;
  const float* prm = r.prm;
  const Layout& L = r.L;
  cudaStream_t st = r.st;
  const size_t smT = (size_t)T * sizeof(float);
  int rc;
  // XH[0] = [first input | initial h] in every row: a K = 0 product with that row as its bias
  if ((rc = dense_mm(FAM_EXACTK, st, Op{nullptr, 0, 0, 0, 0}, Op{prm + L.x0, 0, 0, 0, 1}, d.XH, 2 * D, n, 2 * D, 0, prm + L.x0)))
    return rc;
  for (int t = 0; t < RES; ++t) {
    float* H = d.H + plane(n, t, D);
    float* IN = d.IN + plane(n, t, D);
    if ((rc = dense_mm(FAM_EXACTK, st, rm(d.XH + plane(n, t, 2 * D), 2 * D), rm(prm + L.lstm_w, 4 * D), d.G + plane(n, t, 4 * D),
                       4 * D, n, 4 * D, 2 * D, prm + L.lstm_b)))
      return rc;
    if ((rc = ek_launch("k_ek_cell", k_ek_cell, blocks((int64_t)n * D, 256), 256, 0, st, d, t, prm + L.c0))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(H, D), rm(prm + L.w_bef, D), d.HB + plane(n, t, D), D, n, D, D))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(H, D), rm(prm + L.w_b, D), d.QB + plane(n, t, D), D, n, D, D))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(H, D), rm(prm + L.att[0].w_q, D), d.A1 + plane(n, t, D), D, n, D, D))) return rc;
    if ((rc = ek_launch("k_ek_intra", k_ek_intra, n, D, 0, st, d, t, prm, L))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(IN, D), rm(prm + L.att[0].w_dec, D), d.A1 + plane(n, t, D), D, n, D, D, nullptr, 1)))
      return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(IN, D), rm(prm + L.att[1].w_dec, D), d.A2 + plane(n, t, D), D, n, D, D))) return rc;
    if ((rc = ek_launch("k_ek_glimpse", k_ek_glimpse, n, RNT, smT, st, d, t, prm, L))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(d.GL + plane(n, t, D), D), rm(prm + L.att[1].w_q, D), d.A2 + plane(n, t, D), D, n, D,
                       D, nullptr, 1)))
      return rc;
    if ((rc = ek_launch("k_ek_point", k_ek_point, n, RNT, smT, st, d, t, mode, temperature, r.seed, r.call, prm, L))) return rc;
  }
  return R4_OK;
}

// the backward of the policy loss mean_b(sum_t CE(logits[b, t], path[b, t]) reward[b]) into grad (zeroed here)
int ek_backward(const EkRun& r, const r4ek::Dec& d, const float* user, const float* reward, float* grad, float* loss) {
  using namespace r4ek;
  const int n = r.n, T = r.T;
  const int64_t nT = (int64_t)n * T;
  const float* prm = r.prm;
  const Layout& L = r.L;
  cudaStream_t st = r.st;
  const size_t smT = (size_t)T * sizeof(float);
  float* part = r.f(r.p.part);
  int rc;
  cudaError_t ce = cudaSuccess;
  auto zero = [&](int64_t off, int64_t k) { if (ce == cudaSuccess) ce = cudaMemsetAsync(r.f(off), 0, k * sizeof(float), st); };
  if (cudaMemsetAsync(grad, 0, L.n * sizeof(float), st) != cudaSuccess) return fail(R4_ERR_CUDA, "r4_exactk_grad: memset");
  zero(r.p.deref[0], nT * D); zero(r.p.deref[1], nT * D); zero(r.p.denc, nT * D); zero(r.p.dHs, RES * n * D);
  zero(r.p.dHB, RES * n * D); zero(r.p.dQB, RES * n * D); zero(r.p.rv, n * RV_N * D);
  if (ce != cudaSuccess) return fail(R4_ERR_CUDA, "r4_exactk_grad: memset");
  DecBack g;
  g.dlog = r.f(r.p.dlog); g.deref[0] = r.f(r.p.deref[0]); g.deref[1] = r.f(r.p.deref[1]); g.denc = r.f(r.p.denc);
  g.dGL = r.f(r.p.dGL); g.dIN = r.f(r.p.dIN); g.dC = r.f(r.p.dC); g.dHB = r.f(r.p.dHB); g.rv = r.f(r.p.rv);
  float* ceb = r.f(r.p.ce);
  for (int t = RES - 1; t >= 0; --t) {
    g.dA1 = r.f(r.p.dA1) + plane(n, t, D); g.dA2 = r.f(r.p.dA2) + plane(n, t, D);
    g.dH = r.f(r.p.dHs) + plane(n, t, D); g.dQB = r.f(r.p.dQB) + plane(n, t, D);
    g.dG = r.f(r.p.dG); g.dXH = r.f(r.p.dXH) + plane(n, t, 2 * D);
    float* dHt = g.dH;
    if ((rc = ek_launch("k_ek_loss_bwd", k_ek_loss_bwd, n, RNT, 0, st, d, g, t, reward, ceb))) return rc;
    if ((rc = ek_launch("k_ek_point_bwd", k_ek_point_bwd, n, RNT, smT, st, d, g, t, prm, L))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(g.dA2, D), tr(prm + L.att[1].w_q, D), g.dGL, D, n, D, D))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(g.dA2, D), tr(prm + L.att[1].w_dec, D), g.dIN, D, n, D, D))) return rc;
    if ((rc = ek_launch("k_ek_glimpse_bwd", k_ek_glimpse_bwd, n, RNT, smT, st, d, g, t, prm, L))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(g.dA1, D), tr(prm + L.att[0].w_dec, D), g.dIN, D, n, D, D, nullptr, 1))) return rc;
    if ((rc = ek_launch("k_ek_intra_bwd", k_ek_intra_bwd, n, D, 0, st, d, g, t, r.f(r.p.dHs), prm, L))) return rc;
    // dh_t: the later steps' direct terms (in dHs[t]) + the glimpse query + the intra-attention query and keys
    if ((rc = dense_mm(FAM_EXACTK, st, rm(g.dA1, D), tr(prm + L.att[0].w_q, D), dHt, D, n, D, D, nullptr, 1))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(g.dQB, D), tr(prm + L.w_b, D), dHt, D, n, D, D, nullptr, 1))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(r.f(r.p.dHB) + plane(n, t, D), D), tr(prm + L.w_bef, D), dHt, D, n, D, D, nullptr, 1)))
      return rc;
    if ((rc = ek_launch("k_ek_cell_bwd", k_ek_cell_bwd, blocks((int64_t)n * D, 256), 256, 0, st, d, g, t, prm + L.c0,
                        t + 1 < RES ? (const float*)(r.f(r.p.dXH) + plane(n, t + 1, 2 * D)) : (const float*)nullptr)))
      return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(g.dG + plane(n, t, 4 * D), 4 * D), tr(prm + L.lstm_w, 4 * D), g.dXH, 2 * D, n, 2 * D,
                       4 * D)))
      return rc;
    if (t > 0 && (rc = ek_launch("k_ek_input_bwd", k_ek_input_bwd, blocks((int64_t)n * D, 256), 256, 0, st, d, g, t))) return rc;
  }
  if (loss && (rc = ek_launch("k_ek_gloss", k_ek_gloss, 1, 1, 0, st, (const float*)ceb, reward, n, 1.0f / n, loss))) return rc;
  // decoder weights: stacked over the nine steps
  const int64_t R9 = (int64_t)RES * n;
  float* dgr = grad;
  if ((rc = ek_lin_grad(st, r.f(r.p.XH), 2 * D, r.f(r.p.dG), 4 * D, R9, 2 * D, 4 * D, dgr + L.lstm_w, dgr + L.lstm_b, part)))
    return rc;
  if ((rc = ek_colsum(st, r.f(r.p.dC), n, D, D, 0, D, dgr + L.c0, 1, part))) return rc;
  if ((rc = ek_colsum(st, r.f(r.p.dXH), n, 2 * D, D, 0, D, dgr + L.x0, 1, part))) return rc;
  if ((rc = ek_colsum(st, r.f(r.p.dXH) + D, n, 2 * D, D, 0, D, dgr + L.h0, 1, part))) return rc;
  if ((rc = ek_wgrad(st, r.f(r.p.H), D, r.f(r.p.dHB), D, R9, D, D, dgr + L.w_bef, part))) return rc;
  if ((rc = ek_wgrad(st, r.f(r.p.H), D, r.f(r.p.dQB), D, R9, D, D, dgr + L.w_b, part))) return rc;
  if ((rc = ek_wgrad(st, r.f(r.p.H), D, r.f(r.p.dA1), D, R9, D, D, dgr + L.att[0].w_q, part))) return rc;
  if ((rc = ek_wgrad(st, r.f(r.p.IN), D, r.f(r.p.dA1), D, R9, D, D, dgr + L.att[0].w_dec, part))) return rc;
  if ((rc = ek_wgrad(st, r.f(r.p.GL), D, r.f(r.p.dA2), D, R9, D, D, dgr + L.att[1].w_q, part))) return rc;
  if ((rc = ek_wgrad(st, r.f(r.p.IN), D, r.f(r.p.dA2), D, R9, D, D, dgr + L.att[1].w_dec, part))) return rc;
  const int64_t rvo[RV_N] = {L.att[0].v, L.att[0].bias, L.att[1].v, L.att[1].bias, L.v_dec, L.bias_dec};
  for (int k = 0; k < RV_N; ++k)
    if ((rc = ek_colsum(st, r.f(r.p.rv) + k * D, n, RV_N * D, D, 0, D, dgr + rvo[k], 1, part))) return rc;
  // the encoder outputs: the W_ref projections, then the blocks in reverse
  const float* enc = r.f(r.p.Y2[1]);
  float* dY = r.f(r.p.denc);
  for (int a = 0; a < 2; ++a) {
    if ((rc = ek_wgrad(st, enc, D, r.f(r.p.deref[a]), D, nT, D, D, dgr + L.att[a].w_ref, part))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(r.f(r.p.deref[a]), D), tr(prm + L.att[a].w_ref, D), dY, D, (int)nT, D, D, nullptr, 1)))
      return rc;
  }
  const float inv = 1.0f / sqrtf((float)DH);
  for (int l = NBLK - 1; l >= 0; --l) {
    const Block& B = L.blk[l];
    const float* X = l == 0 ? r.f(r.p.X0) : r.f(r.p.Y2[0]);
    const float* QKV = r.f(r.p.QKV[l]);
    float* gx = r.f(r.p.gx);
    float* dZ = r.f(r.p.dZ);
    float* dF1 = r.f(r.p.dF1);
    float* dQKV = r.f(r.p.dQKV);
    float* dP = r.f(r.p.dP);
    // Y2 = LN(F1 W2 + b2 + Y1): beta's gradient from dY, then dY (in place) -> d(sum)
    if ((rc = ek_colsum(st, dY, nT, D, D, 0, D, dgr + B.ln2_b, 1, part))) return rc;
    if ((rc = ek_launch("k_ek_ln_bwd", k_ek_ln_bwd, blocks(nT * 32, 256), 256, 0, st, (const float*)r.f(r.p.xh2[l]),
                        (const float*)r.f(r.p.rs2[l]), nT, prm + B.ln2_g, dY, gx)))
      return rc;
    if ((rc = ek_colsum(st, gx, nT, D, D, 0, D, dgr + B.ln2_g, 1, part))) return rc;
    if ((rc = ek_lin_grad(st, r.f(r.p.F1[l]), FF, dY, D, nT, FF, D, dgr + B.f2_w, dgr + B.f2_b, part))) return rc;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(dY, D), tr(prm + B.f2_w, D), dF1, FF, (int)nT, FF, D))) return rc;
    if ((rc = ek_launch("k_ek_relu_bwd", k_ek_relu_bwd, blocks(nT * FF, 256), 256, 0, st, (const float*)r.f(r.p.F1[l]),
                        (int64_t)FF, dF1, (int64_t)FF, nT, FF)))
      return rc;
    if ((rc = ek_lin_grad(st, r.f(r.p.Y1[l]), D, dF1, FF, nT, D, FF, dgr + B.f1_w, dgr + B.f1_b, part))) return rc;
    // dY1
    if ((rc = dense_mm(FAM_EXACTK, st, rm(dF1, FF), tr(prm + B.f1_w, FF), dY, D, (int)nT, D, FF, nullptr, 1))) return rc;
    // Y1 = LN(O + X)
    if ((rc = ek_colsum(st, dY, nT, D, D, 0, D, dgr + B.ln1_b, 1, part))) return rc;
    if ((rc = ek_launch("k_ek_ln_bwd", k_ek_ln_bwd, blocks(nT * 32, 256), 256, 0, st, (const float*)r.f(r.p.xh1[l]),
                        (const float*)r.f(r.p.rs1[l]), nT, prm + B.ln1_g, dY, gx)))
      return rc;
    if ((rc = ek_colsum(st, gx, nT, D, D, 0, D, dgr + B.ln1_g, 1, part))) return rc;
    // O_h = P V_h: dP = dO_h V_h^T, dV_h = P^T dO_h
    if ((rc = dense_bmm(FAM_EXACTK, st, Op{dY, (int64_t)T * D, DH, D, 1}, Op{QKV + 2 * D, (int64_t)T * 3 * D, DH, 1, 3 * D}, dP,
                        (int64_t)NH * T * T, (int64_t)T * T, T, T, T, DH, n, NH, 1.f)))
      return rc;
    if ((rc = dense_bmm(FAM_EXACTK, st, Op{r.f(r.p.P[l]), (int64_t)NH * T * T, (int64_t)T * T, 1, T},
                        Op{dY, (int64_t)T * D, DH, D, 1}, dQKV + 2 * D, (int64_t)T * 3 * D, DH, 3 * D, T, DH, T, n, NH, 1.f)))
      return rc;
    if ((rc = ek_launch("k_ek_softmax_bwd", k_ek_softmax_bwd, blocks((int64_t)n * NH * T * 32, 256), 256, 0, st,
                        (const float*)r.f(r.p.A[l]), (const float*)r.f(r.p.m[l]), n, T, r.seed, r.call,
                        l == 0 ? ST_ATT0 : ST_ATT1, r.rate, dP)))
      return rc;
    // S = Q K^T / sqrt(32): dQ_h = dS K_h / sqrt(32), dK_h = dS^T Q_h / sqrt(32)
    if ((rc = dense_bmm(FAM_EXACTK, st, Op{dP, (int64_t)NH * T * T, (int64_t)T * T, T, 1},
                        Op{QKV + D, (int64_t)T * 3 * D, DH, 3 * D, 1}, dQKV, (int64_t)T * 3 * D, DH, 3 * D, T, DH, T, n, NH,
                        inv)))
      return rc;
    if ((rc = dense_bmm(FAM_EXACTK, st, Op{dP, (int64_t)NH * T * T, (int64_t)T * T, 1, T},
                        Op{QKV, (int64_t)T * 3 * D, DH, 3 * D, 1}, dQKV + D, (int64_t)T * 3 * D, DH, 3 * D, T, DH, T, n, NH,
                        inv)))
      return rc;
    if ((rc = ek_launch("k_ek_relu_bwd", k_ek_relu_bwd, blocks(nT * 3 * D, 256), 256, 0, st, QKV, (int64_t)3 * D, dQKV,
                        (int64_t)3 * D, nT, 3 * D)))
      return rc;
    if ((rc = ek_lin_grad(st, X, D, dQKV, 3 * D, nT, D, 3 * D, dgr + B.qkv_w, dgr + B.qkv_b, part))) return rc;
    // dX = d(sum) (the residual) + dQKV W_qkv^T: the block input's gradient, kept in dY
    if ((rc = dense_mm(FAM_EXACTK, st, rm(dQKV, 3 * D), tr(prm + B.qkv_w, 3 * D), dY, D, (int)nT, D, 3 * D, nullptr, 1)))
      return rc;
  }
  // X0 = dropout([relu(user W_u + b_u) | emb * 8])
  float* dU = r.f(r.p.dU);
  if ((rc = ek_launch("k_ek_emb_bwd", k_ek_emb_bwd, blocks((int64_t)(n + T) * HU, 128), 128, 0, st, (const float*)dY, n, T,
                      r.seed, r.call, r.rate, dU, dgr + L.emb)))
    return rc;
  if ((rc = ek_launch("k_ek_relu_bwd", k_ek_relu_bwd, blocks((int64_t)n * HU, 256), 256, 0, st, (const float*)r.f(r.p.uenc),
                      (int64_t)HU, dU, (int64_t)HU, (int64_t)n, HU)))
    return rc;
  return ek_lin_grad(st, user, UIN, dU, HU, n, UIN, HU, dgr + L.u_w, dgr + L.u_b, part);
}

struct CPlanes { int64_t Z[4], dZ[4], part, n; };
CPlanes ek_cplanes(int64_t n) {
  CPlanes p;
  int64_t o = 0;
  auto take = [&](int64_t k) { int64_t r = o; o += (k + 63) / 64 * 64; return r; };
  for (int i = 0; i < 4; ++i) { p.Z[i] = take(n * r4ek::CH); p.dZ[i] = take(n * r4ek::CH); }
  p.part = take((int64_t)EK_SPLITS * r4ek::UIN * r4ek::CH);
  p.n = o;
  return p;
}

}  // namespace

int64_t r4_exactk_num_params(int net) {
  return net == R4_EXACTK_GENERATOR ? r4ek::make_layout().n : net == R4_EXACTK_CRITIC ? r4ek::make_clayout().n : -1;
}

int64_t r4_exactk_scratch_size(int net, int n, int seq_length) {
  if (n < 1 || n > r4ek::MAXN) return -1;
  if (net == R4_EXACTK_CRITIC) return ek_cplanes(n).n * (int64_t)sizeof(float);
  if (net != R4_EXACTK_GENERATOR || !ek_shape_ok(n, seq_length)) return -1;
  return ek_planes(n, seq_length).n * (int64_t)sizeof(float);
}

static int ek_run(const float* params, int n, int T, uint64_t seed, uint64_t call, float dropout, void* scratch, void* stream,
                  EkRun* r) {
  if (!params || !scratch || !ek_shape_ok(n, T) || !(dropout >= 0.f && dropout < 1.f)) return fail(R4_ERR_ARG, "bad argument");
  r->prm = params; r->L = r4ek::make_layout(); r->n = n; r->T = T; r->seed = seed; r->call = call; r->rate = dropout;
  r->s = static_cast<float*>(scratch); r->p = ek_planes(n, T); r->st = S(stream);
  return R4_OK;
}

int r4_exactk_decode(const float* params, const float* user, int n, int seq_length, const uint8_t* masks, int mode,
                     float temperature, uint64_t seed, uint64_t call, float dropout, int32_t* path, float* logits, void* scratch,
                     void* stream) {
  EkRun r;
  if (int rc = ek_run(params, n, seq_length, seed, call, dropout, scratch, stream, &r)) return rc;
  if (!user || !masks || !path || mode < R4_EXACTK_SAMPLE || mode > R4_EXACTK_TRAIN || !(temperature > 0.f))
    return fail(R4_ERR_ARG, "bad argument");
  if (int rc = ek_encoder(r, user)) return rc;
  return ek_decoder(r, ek_dec(r, masks, path, logits ? logits : r.f(r.p.logits)), mode, temperature);
}

int r4_exactk_grad(const float* params, const float* user, int n, int seq_length, const uint8_t* masks, const int32_t* target,
                   const float* reward, uint64_t seed, uint64_t call, float dropout, float* grad, float* loss, void* scratch,
                   void* stream) {
  EkRun r;
  if (int rc = ek_run(params, n, seq_length, seed, call, dropout, scratch, stream, &r)) return rc;
  if (!user || !masks || !target || !reward || !grad) return fail(R4_ERR_ARG, "bad argument");
  int32_t* path = reinterpret_cast<int32_t*>(r.f(r.p.path));
  if (cudaMemcpyAsync(path, target, (size_t)n * r4ek::RES * sizeof(int32_t), cudaMemcpyDeviceToDevice, r.st) != cudaSuccess)
    return fail(R4_ERR_CUDA, "r4_exactk_grad: copy");
  if (int rc = ek_encoder(r, user)) return rc;
  const r4ek::Dec d = ek_dec(r, masks, path, r.f(r.p.logits));
  if (int rc = ek_decoder(r, d, R4_EXACTK_TRAIN, 1.f)) return rc;
  return ek_backward(r, d, user, reward, grad, loss);
}

int r4_exactk_critic(const float* params, const float* user, int n, const float* target, float* pred, float* grad, float* loss,
                     void* scratch, void* stream) {
  using namespace r4ek;
  if (!params || !user || !scratch || n < 1 || n > MAXN || (target && !grad)) return fail(R4_ERR_ARG, "bad argument");
  const CLayout L = make_clayout();
  const CPlanes p = ek_cplanes(n);
  float* s = static_cast<float*>(scratch);
  cudaStream_t st = S(stream);
  const int in[4] = {UIN, CH, CH, CH}, out[4] = {CH, CH, CH, 1};
  int rc;
  const float* X = user;
  for (int i = 0; i < 4; ++i) {
    if ((rc = dense_mm(FAM_EXACTK, st, rm(X, in[i]), rm(params + L.w[i], out[i]), s + p.Z[i], out[i], n, out[i], in[i],
                       params + L.b[i], 0, i < 3 ? EP_RELU : EP_LIN)))
      return rc;
    X = s + p.Z[i];
  }
  if ((rc = ek_launch("k_ek_closs", k_ek_closs, 1, 256, 0, st, (const float*)(s + p.Z[3]), target, n, pred, s + p.dZ[3], loss)))
    return rc;
  if (!target) return R4_OK;
  if (cudaMemsetAsync(grad, 0, L.n * sizeof(float), st) != cudaSuccess) return fail(R4_ERR_CUDA, "r4_exactk_critic: memset");
  for (int i = 3; i >= 0; --i) {
    const float* Xi = i == 0 ? user : s + p.Z[i - 1];
    if ((rc = ek_lin_grad(st, Xi, in[i], s + p.dZ[i], out[i], n, in[i], out[i], grad + L.w[i], grad + L.b[i], s + p.part)))
      return rc;
    if (i == 0) break;
    if ((rc = dense_mm(FAM_EXACTK, st, rm(s + p.dZ[i], out[i]), tr(params + L.w[i], out[i]), s + p.dZ[i - 1], CH, n, CH, out[i])))
      return rc;
    if ((rc = ek_launch("k_ek_relu_bwd", k_ek_relu_bwd, blocks((int64_t)n * CH, 256), 256, 0, st, (const float*)(s + p.Z[i - 1]),
                        (int64_t)CH, s + p.dZ[i - 1], (int64_t)CH, (int64_t)n, CH)))
      return rc;
  }
  return R4_OK;
}

int r4_exactk_adam(int net, float* params, float* grad, float* m, float* v, int step, float lr, float beta1, float beta2,
                   float eps, void* stream) {
  const int64_t np = r4_exactk_num_params(net);
  if (np < 0 || !params || !grad || !m || !v || step < 1) return fail(R4_ERR_ARG, "bad argument");
  const float alpha = lr * sqrtf(1.f - powf(beta2, (float)step)) / (1.f - powf(beta1, (float)step));
  return ek_launch("k_keras_adam", k_keras_adam, blocks(np, 256), 256, 0, S(stream), np, (int64_t)0, np, np, params, grad, m,
                   v, alpha, beta1, beta2, eps);
}

// ---- batch RL: continuous-action BCQ (r4_bcqconti.cuh), counted with the discrete learners ------------------------
namespace {

int bc_pack(cudaStream_t st, bool pdl, const float* obs, int K, int rep, const float* A, int lda, const float* B, int W,
            int mode, float flex, int R, float* x, float* out) {
  return cq_launch("k_bcqc_pack", r4bcqc::k_bcqc_pack, blocks(R, NT / 32), st, pdl, obs, K, rep, A, lda, B, W, mode, flex, R,
                   x, out);
}

// One SGD step at 1-based step `step`: imitator, critic, actor (each phase's Adam before the next when apply; the
// critic's and the actor's Adam with the soft update of their targets), else every group's gradient at the given
// parameters into P.grad.
int bc_step(const r4bcqc::Layout& L, const r4bcqc::Hyper& hp, float* prm, float* tgt, float* m, float* v,
            const r4cqlc::Data& Dt, const int64_t* idx, int n, int step, int apply, const r4bcqc::Planes& P, float* stats,
            cudaStream_t st, bool pdl) {
  using namespace r4bcqc;
  const int K = L.K, D = L.D, La = L.L, S = hp.S, R = n * S;
  int rc;
  if ((rc = cq_launch("k_bcqc_gather", k_bcqc_gather, 2 * sm_count(), st, pdl, K, D, Dt, idx, n, P))) return rc;
  if ((rc = cq_launch("k_bcqc_noise", k_bcqc_noise, 2 * sm_count(), st, pdl, L, hp, n, (uint64_t)step, P))) return rc;
  // imitator: the conditional VAE
  if ((rc = bc_pack(st, pdl, P.xs, K, 1, P.act, D, nullptr, D, PK_PLAIN, 0.f, n, P.ex, nullptr))) return rc;
  if ((rc = cq_forward(st, prm, L.enc, P.ex, n, P.eh1, P.eh2, P.eo))) return rc;
  if ((rc = bc_pack(st, pdl, P.xs, K, 1, P.eo, 2 * La, P.eps, La, PK_REPARAM, 0.f, n, P.dx, nullptr))) return rc;
  if ((rc = cq_forward(st, prm, L.dec, P.dx, n, P.dh1, P.dh2, P.o))) return rc;
  if ((rc = cq_launch("k_bcqc_vae", k_bcqc_vae, 1, st, pdl, L, hp, n, P, (const float*)P.o, stats))) return rc;
  if ((rc = cq_backward(st, prm, L.dec, P.dout, n, P.dh1, P.dh2, P.ddz2, P.ddz1))) return rc;
  if ((rc = dense_mm(FAM_BATCHRL, st, rm(P.ddz1, H), tr(prm + L.dec.w1 + (size_t)K * H, H), P.dlat, La, n, La, H))) return rc;
  if ((rc = cq_launch("k_bcqc_vae_head", k_bcqc_vae_head, blocks((int64_t)n * La, NT), st, pdl, L, hp, n, P))) return rc;
  if ((rc = cq_backward(st, prm, L.enc, P.deo, n, P.eh1, P.eh2, P.edz2, P.edz1))) return rc;
  Jobs J;
  int nj = 0;
  cq_jobs(J, nj, L.dec, P.dx, P.dh1, P.dh2, P.ddz1, P.ddz2, P.dout);
  cq_jobs(J, nj, L.enc, P.ex, P.eh1, P.eh2, P.edz1, P.edz2, P.deo);
  tile_jobs(J, nj);
  if ((rc = dense_wgrad(FAM_BATCHRL, st, J, n, 1, P.grad))) return rc;
  if (apply && (rc = cq_launch("k_cqlc_adam", r4cqlc::k_cqlc_adam, blocks(L.dec.end - L.enc.w1, NT), st, pdl, L.enc.w1,
                               L.dec.end - L.enc.w1, prm, (const float*)P.grad, m, v, step, hp.lr_imitator, hp.eps,
                               (float*)nullptr, 0.f)))
    return rc;
  // critic: the target over S decoded, perturbed actions per s'
  if ((rc = bc_pack(st, pdl, P.xn, K, S, P.zt, La, nullptr, La, PK_LATENT, 0.f, R, P.x, nullptr))) return rc;
  if ((rc = cq_forward(st, prm, L.dec, P.x, R, P.h1, P.h2, P.o))) return rc;
  if ((rc = bc_pack(st, pdl, P.xn, K, S, P.o, D, nullptr, D, PK_TANH, 0.f, R, P.x, P.base))) return rc;
  if ((rc = cq_forward(st, tgt, L.actor, P.x, R, P.h1, P.h2, P.o))) return rc;
  if ((rc = bc_pack(st, pdl, P.xn, K, S, P.o, D, P.base, D, PK_PERTURB, hp.flex, R, P.x, nullptr))) return rc;
  for (int k = 0; k < 2; ++k)
    if ((rc = cq_forward(st, tgt, L.c[k], P.x, R, P.h1, P.h2, k ? P.qb : P.qa))) return rc;
  if ((rc = bc_pack(st, pdl, P.xs, K, 1, P.act, D, nullptr, D, PK_PLAIN, 0.f, n, P.cx, nullptr))) return rc;
  for (int k = 0; k < 2; ++k)
    if ((rc = cq_forward(st, prm, L.c[k], P.cx, n, P.ch1[k], P.ch2[k], P.cq[k]))) return rc;
  if ((rc = cq_launch("k_bcqc_critic", k_bcqc_critic, 1, st, pdl, hp, n, P, stats))) return rc;
  nj = 0;
  for (int k = 0; k < 2; ++k) {
    if ((rc = cq_backward(st, prm, L.c[k], P.dq[k], n, P.ch1[k], P.ch2[k], P.dz2[k], P.dz1[k]))) return rc;
    cq_jobs(J, nj, L.c[k], P.cx, P.ch1[k], P.ch2[k], P.dz1[k], P.dz2[k], P.dq[k]);
  }
  tile_jobs(J, nj);
  if ((rc = dense_wgrad(FAM_BATCHRL, st, J, n, 1, P.grad))) return rc;
  const int c0 = L.c[0].w1, nc = L.c[1].end - c0;
  if (apply && (rc = cq_launch("k_cqlc_adam", r4cqlc::k_cqlc_adam, blocks(nc, NT), st, pdl, c0, nc, prm,
                               (const float*)P.grad, m, v, step, hp.lr_critic, hp.eps, tgt + c0, hp.tau)))
    return rc;
  // actor: -Q_0(s, pi(s, dec(s, clamp(z))))
  if ((rc = bc_pack(st, pdl, P.xs, K, 1, P.za, La, nullptr, La, PK_LATENT, 0.f, n, P.x, nullptr))) return rc;
  if ((rc = cq_forward(st, prm, L.dec, P.x, n, P.h1, P.h2, P.o))) return rc;
  if ((rc = bc_pack(st, pdl, P.xs, K, 1, P.o, D, nullptr, D, PK_TANH, 0.f, n, P.ax, P.abase))) return rc;
  if ((rc = cq_forward(st, prm, L.actor, P.ax, n, P.ah1, P.ah2, P.ao))) return rc;
  if ((rc = bc_pack(st, pdl, P.xs, K, 1, P.ao, D, P.abase, D, PK_PERTURB, hp.flex, n, P.cx, nullptr))) return rc;
  if ((rc = cq_forward(st, prm, L.c[0], P.cx, n, P.ch1[0], P.ch2[0], P.cq[0]))) return rc;
  if ((rc = cq_launch("k_bcqc_actor_loss", k_bcqc_actor_loss, 1, st, pdl, n, P, stats))) return rc;
  if ((rc = cq_backward(st, prm, L.c[0], P.dq[0], n, P.ch1[0], P.ch2[0], P.dz2[0], P.dz1[0]))) return rc;
  if ((rc = dense_mm(FAM_BATCHRL, st, rm(P.dz1[0], H), tr(prm + L.c[0].w1 + (size_t)K * H, H), P.da, D, n, D, H))) return rc;
  if ((rc = cq_launch("k_bcqc_actor_head", k_bcqc_actor_head, blocks((int64_t)n * D, NT), st, pdl, D, hp.flex, n, P)))
    return rc;
  if ((rc = cq_backward(st, prm, L.actor, P.dout, n, P.ah1, P.ah2, P.adz2, P.adz1))) return rc;
  nj = 0;
  cq_jobs(J, nj, L.actor, P.ax, P.ah1, P.ah2, P.adz1, P.adz2, P.dout);
  tile_jobs(J, nj);
  if ((rc = dense_wgrad(FAM_BATCHRL, st, J, n, 1, P.grad))) return rc;
  if (apply && (rc = cq_launch("k_cqlc_adam", r4cqlc::k_cqlc_adam, blocks(L.actor.end, NT), st, pdl, 0, L.actor.end, prm,
                               (const float*)P.grad, m, v, step, hp.lr_actor, hp.eps, tgt, hp.tau)))
    return rc;
  return R4_OK;
}

r4bcqc::Hyper bc_hyper(const r4_bcqc_hyper* h) {
  return r4bcqc::Hyper{h->gamma, h->tau, h->lam, h->beta, h->action_flexibility, h->adam_eps, h->reward_mean, h->reward_den,
                       h->lr_actor, h->lr_critic, h->lr_imitator, h->n_action_samples, h->seed};
}
// the arguments r4_bcqc_grad and r4_bcqc_epoch share, and the dataset planes into *out
bool bc_args_ok(int K, int D, const r4_cqlc_data* d, const r4_bcqc_hyper* h, int n, r4cqlc::Data* out) {
  return h && r4bcqc::dims_ok(K, D, h->latent_size) && conti_data(d, out) && h->n_action_samples >= 1 &&
         h->n_action_samples <= r4bcqc::MAXS && n >= 1 && n <= r4bcqc::MAXN;
}
}  // namespace

extern "C" {

int r4_bcqc_num_params(int obs_dim, int action_dim, int latent_size) {
  return r4bcqc::dims_ok(obs_dim, action_dim, latent_size) ? r4bcqc::make_layout(obs_dim, action_dim, latent_size).n : -1;
}

int r4_bcqc_target_size(int obs_dim, int action_dim, int latent_size) {
  return r4bcqc::dims_ok(obs_dim, action_dim, latent_size) ? r4bcqc::make_layout(obs_dim, action_dim, latent_size).ntgt : -1;
}

int64_t r4_bcqc_scratch_size(int obs_dim, int action_dim, int latent_size, int n_action_samples, int n) {
  if (!r4bcqc::dims_ok(obs_dim, action_dim, latent_size) || n_action_samples < 1 || n_action_samples > r4bcqc::MAXS ||
      n < 1 || n > r4bcqc::MAXN)
    return -1;
  return (int64_t)r4bcqc::scratch_floats(r4bcqc::make_layout(obs_dim, action_dim, latent_size), n_action_samples, n);
}

int64_t r4_bcqc_act_scratch_size(int obs_dim, int action_dim, int latent_size, int n_action_samples, int n) {
  if (!r4bcqc::dims_ok(obs_dim, action_dim, latent_size) || n_action_samples < 1 || n_action_samples > r4bcqc::MAXS ||
      n < 1 || (int64_t)n * n_action_samples > r4cqlc::MAXACT)
    return -1;
  return (int64_t)r4bcqc::act_scratch_floats(r4bcqc::make_layout(obs_dim, action_dim, latent_size), n_action_samples, n);
}

int r4_bcqc_grad(int obs_dim, int action_dim, const float* params, const float* target, const r4_cqlc_data* data,
                 const r4_bcqc_hyper* hp, const int64_t* idx, int n, int step, float* scratch, float* grad, float* stats,
                 void* stream) {
  r4cqlc::Data D;
  if (!bc_args_ok(obs_dim, action_dim, data, hp, n, &D) || !params || !target || !idx || step < 1 || !scratch || !grad)
    return fail(R4_ERR_ARG, "r4_bcqc_grad: bad argument (obs_dim 1..4096, action_dim 1..512, latent 1..512, n 1..4096, "
                            "samples 1..256)");
  const r4bcqc::Layout L = r4bcqc::make_layout(obs_dim, action_dim, hp->latent_size);
  r4bcqc::Planes P = r4bcqc::make_planes(scratch, L, hp->n_action_samples, n);
  P.grad = grad;
  return bc_step(L, bc_hyper(hp), const_cast<float*>(params), const_cast<float*>(target), nullptr, nullptr, D, idx, n, step,
                 0, P, stats, S(stream), false);
}

int r4_bcqc_epoch(int obs_dim, int action_dim, float* params, float* target, float* m, float* v, const r4_cqlc_data* data,
                  const r4_bcqc_hyper* hp, const int64_t* perm, int64_t n_perm, int mb, int step0, float* scratch,
                  float* stats, void* stream) {
  r4cqlc::Data D;
  if (!bc_args_ok(obs_dim, action_dim, data, hp, mb, &D) || !params || !target || !m || !v || !perm || n_perm < 1 ||
      step0 < 0 || !scratch)
    return fail(R4_ERR_ARG, "r4_bcqc_epoch: bad argument");
  const r4bcqc::Layout L = r4bcqc::make_layout(obs_dim, action_dim, hp->latent_size);
  const r4bcqc::Planes P = r4bcqc::make_planes(scratch, L, hp->n_action_samples, mb);
  const r4bcqc::Hyper h = bc_hyper(hp);
  return batchrl_epoch("r4_bcqc_epoch", perm, n_perm, mb, step0, stats, r4bcqc::NSTAT,
                       [&](const int64_t* idx, int step, float* sk) {
                         return bc_step(L, h, params, target, m, v, D, idx, mb, step, 1, P, sk, S(stream), true);
                       });
}

int r4_bcqc_act(int obs_dim, int action_dim, const float* params, const void* obs, int obs_f64, int n,
                const r4_bcqc_hyper* hp, uint64_t counter, const float* action_in, float* action, float* q, float* scratch,
                void* stream) {
  if (!hp || !r4bcqc::dims_ok(obs_dim, action_dim, hp->latent_size) || hp->n_action_samples < 1 ||
      hp->n_action_samples > r4bcqc::MAXS || !params || !obs || n < 1 ||
      (int64_t)n * hp->n_action_samples > r4cqlc::MAXACT || !scratch || (!action && !(q && action_in)))
    return fail(R4_ERR_ARG, "r4_bcqc_act: bad argument");
  using namespace r4bcqc;
  const Layout L = make_layout(obs_dim, action_dim, hp->latent_size);
  const int K = obs_dim, D = action_dim, La = hp->latent_size, NS = hp->n_action_samples, R = n * NS;
  const int W = D > La ? D : La;
  cudaStream_t st = r4h::S(stream);
  float *x = scratch, *xin = x + (size_t)n * K, *h1 = xin + (size_t)R * (K + W), *h2 = h1 + (size_t)R * H;
  float *o = h2 + (size_t)R * H, *base = o + (size_t)R * D, *cq = base + (size_t)R * D, *z = cq + R;
  float *xa = z + (size_t)R * La, *ch = xa + (size_t)n * (K + D);
  const int64_t total = (int64_t)n * K;
  int rc;
  if ((rc = cq_launch("k_cqlc_obs", r4cqlc::k_cqlc_obs, blocks(total, NT), st, false,
                      obs_f64 ? nullptr : (const float*)obs, obs_f64 ? (const double*)obs : nullptr, total, x)))
    return rc;
  if (action) {
    if ((rc = cq_launch("k_bcqc_predict_noise", k_bcqc_predict_noise, blocks((int64_t)R * La, NT), st, false, La, NS, n,
                        hp->seed, counter, z)))
      return rc;
    if ((rc = bc_pack(st, false, x, K, NS, z, La, nullptr, La, PK_LATENT, 0.f, R, xin, nullptr))) return rc;
    if ((rc = cq_forward(st, params, L.dec, xin, R, h1, h2, o))) return rc;
    if ((rc = bc_pack(st, false, x, K, NS, o, D, nullptr, D, PK_TANH, 0.f, R, xin, base))) return rc;
    if ((rc = cq_forward(st, params, L.actor, xin, R, h1, h2, o))) return rc;
    if ((rc = bc_pack(st, false, x, K, NS, o, D, base, D, PK_PERTURB, hp->action_flexibility, R, xin, base))) return rc;
    if ((rc = cq_forward(st, params, L.c[0], xin, R, h1, h2, cq))) return rc;
    if ((rc = cq_launch("k_bcqc_argmax", k_bcqc_argmax, blocks(n, NT / 32), st, false, D, NS, n, (const float*)cq,
                        (const float*)base, action)))
      return rc;
  }
  if (!q) return R4_OK;
  if ((rc = bc_pack(st, false, x, K, 1, action_in ? action_in : action, D, nullptr, D, PK_PLAIN, 0.f, n, xa, nullptr)))
    return rc;
  float* qk[2];
  for (int k = 0; k < 2; ++k) {
    float* c = ch + (size_t)k * n * (2 * H + 1);
    qk[k] = c + (size_t)n * 2 * H;
    if ((rc = cq_forward(st, params, L.c[k], xa, n, c, c + (size_t)n * H, qk[k]))) return rc;
  }
  return cq_launch("k_cqlc_qmean", r4cqlc::k_cqlc_qmean, blocks(n, NT), st, false, n, (const float*)qk[0],
                   (const float*)qk[1], q);
}

}  // extern "C"

// ---- the MDP checker's seq2seq transformer (r4_seq2seq.cuh) ---------------------------------------------------------------
namespace {
using namespace r4s2s;

template <typename... P, typename... A>
int s2_launch(const char* name, void (*kernel)(P...), dim3 grid, int threads, size_t smem, cudaStream_t st, A&&... args) {
  return launch(FAM_SEQ2SEQ, name, kernel, grid, threads, smem, st, false, std::forward<A>(args)...);
}

bool s2_cfg_ok(const r4_s2s_config* c) {
  if (!c) return false;
  const bool v = c->src_tokens >= MINV && c->src_tokens <= MAXV && c->tgt_tokens >= MINV && c->tgt_tokens <= MAXV;
  return v && (!c->use_same_embed || c->src_tokens == c->tgt_tokens) && c->embed_dim >= 32 && c->embed_dim <= MAXE &&
         c->embed_dim % 32 == 0 && c->head_num >= 1 && c->embed_dim % c->head_num == 0 && c->hidden_dim >= 32 &&
         c->hidden_dim <= MAXF && c->hidden_dim % 32 == 0 && c->encoder_num >= 1 && c->encoder_num <= MAXBLK &&
         c->decoder_num >= 1 && c->decoder_num <= MAXBLK;
}
Cfg s2_cfg(const r4_s2s_config* c) {
  return Cfg{c->src_tokens, c->tgt_tokens, c->embed_dim, c->head_num, c->hidden_dim, c->encoder_num, c->decoder_num,
             c->use_same_embed ? 1 : 0};
}

// The activations of one sub-layer: attention Q, K, V, the concatenated heads O, the softmax A; FeedForward relu(x W1 + b1)
// in q; the sub-layer output y, the LayerNorm output, its normalised input and 1 / std.
struct SubP { int64_t q, k, v, o, a, y, out, xh, rs; };
// Scratch planes (floats) of one call over n source rows of Ts and R decoder prefixes per row of Tt positions; logits of
// `lrows` rows; the backward's planes when train; a search's paths and scores for `beam`, and its candidate list of k.
struct Plan {
  int64_t xe, xd;
  SubP enc[MAXBLK][2], dec[MAXBLK][3];
  int64_t logits, ce, inv;
  int64_t g[2], dy, gx, dq, dk, dv, dO, dA, dF, denc, cnt, off, order;
  int64_t et, dt, yt;                              // a minibatch's tokens (epoch)
  int64_t path[2], score[2], val, idx, cval, cand;  // search; cval / cand: the candidate list
  int64_t n;
};
Plan s2_plan(const Cfg& c, int64_t n, int64_t Ts, int64_t Tt, int64_t R, int64_t lrows, bool train, int64_t beam, int64_t k) {
  Plan p = {};
  int64_t o = 0;
  auto take = [&](int64_t x) { int64_t r = o; o += (x + 63) / 64 * 64; return r; };
  const int64_t E = c.E, F = c.F, Ne = n * Ts, Nd = n * R * Tt, H = c.H;
  auto sub = [&](SubP& s, int64_t rows, int64_t kvrows, int64_t att, bool ffn) {
    s.q = take(rows * (ffn ? F : E));
    if (!ffn) { s.k = take(kvrows * E); s.v = take(kvrows * E); s.o = take(rows * E); s.a = take(att); }
    s.y = take(rows * E); s.out = take(rows * E); s.xh = take(rows * E); s.rs = take(rows);
  };
  p.xe = take(Ne * E);
  for (int l = 0; l < c.Le; ++l) { sub(p.enc[l][0], Ne, Ne, n * H * Ts * Ts, false); sub(p.enc[l][1], Ne, 0, 0, true); }
  p.xd = take(Nd * E);
  for (int l = 0; l < c.Ld; ++l) {
    sub(p.dec[l][0], Nd, Nd, n * R * H * Tt * Tt, false);
    sub(p.dec[l][1], Nd, Ne, n * H * R * Tt * Ts, false);
    sub(p.dec[l][2], Nd, 0, 0, true);
  }
  p.logits = take(lrows * c.Vt);
  if (train) {
    const int64_t rows = std::max(Ne, Nd);
    p.ce = take(Nd); p.inv = take(1);
    p.g[0] = take(rows * E); p.g[1] = take(rows * E); p.dy = take(rows * E); p.gx = take(rows * E);
    p.dq = take(rows * E); p.dk = take(rows * E); p.dv = take(rows * E); p.dO = take(rows * E);
    p.dA = take(std::max(n * H * Ts * Ts, std::max(n * R * H * Tt * Tt, n * H * R * Tt * Ts)));
    p.dF = take(rows * F); p.denc = take(Ne * E);
    p.cnt = take(std::max(c.Vs, c.Vt)); p.off = take(std::max(c.Vs, c.Vt)); p.order = take(rows);
    p.et = take(Ne); p.dt = take(Nd); p.yt = take(Nd);
  }
  if (beam > 0) {
    const int64_t L = Tt + 1;
    p.path[0] = take(n * beam * L); p.path[1] = take(n * beam * L);
    p.score[0] = take(2 * n * beam); p.score[1] = take(2 * n * beam);
    p.val = take(2 * n * beam * beam); p.idx = take(n * beam * beam);
  }
  if (k > 0) { p.cval = take(2 * n * k); p.cand = take(n * k); }
  p.n = o;
  return p;
}

struct S2Run {
  const float* prm;
  Cfg c;
  Layout L;
  Plan p;
  float* s;
  cudaStream_t st;
  int n, Ts;
  const int32_t* etok;
  uint64_t seed, call;
  float rate;
  float* f(int64_t o) const { return s + o; }
  template <class T> T* as(int64_t o) const { return reinterpret_cast<T*>(s + o); }
};

// One attention sub-layer: out = LN(xq + dropout(MHA(xq, xkv))).  Groups g of Mq queries attend over Tk keys each
// (the query rows of group g are g Mq .., its key rows g Tk ..); key j of group g is masked when ktok[g kld + j] == 0,
// and, when causal, when j > m % Tq.  kv: compute K and V (else they are already in P).
int s2_att(const S2Run& r, const Att& W, const Norm& Nw, const SubP& P, const float* xq, int64_t Nq, const float* xkv,
           int64_t Nk, int64_t G, int Mq, int Tk, int Tq, int causal, const int32_t* ktok, int64_t kld, bool kv, int layer) {
  const int E = r.c.E, H = r.c.H, dh = E / H;
  const float* w = r.prm;
  cudaStream_t st = r.st;
  float *Q = r.f(P.q), *K = r.f(P.k), *V = r.f(P.v), *O = r.f(P.o), *A = r.f(P.a), *Y = r.f(P.y);
  int rc;
  if ((rc = dense_mm(FAM_SEQ2SEQ, st, rm(xq, E), rm(w + W.wq, E), Q, E, Nq, E, E, w + W.bq))) return rc;
  if (kv) {
    if ((rc = dense_mm(FAM_SEQ2SEQ, st, rm(xkv, E), rm(w + W.wk, E), K, E, Nk, E, E, w + W.bk))) return rc;
    if ((rc = dense_mm(FAM_SEQ2SEQ, st, rm(xkv, E), rm(w + W.wv, E), V, E, Nk, E, E, w + W.bv))) return rc;
  }
  const int64_t cso = (int64_t)H * Mq * Tk, csi = (int64_t)Mq * Tk;
  if ((rc = dense_bmm(FAM_SEQ2SEQ, st, Op{Q, (int64_t)Mq * E, dh, E, 1}, Op{K, (int64_t)Tk * E, dh, 1, E}, A, cso, csi, Tk, Mq,
                      Tk, dh, G, H, 1.0f / sqrtf((float)dh))))
    return rc;
  const int64_t rows = G * H * Mq;
  if ((rc = s2_launch("k_s2s_softmax", k_s2s_softmax, blocks(rows * 32, 256), 256, 0, st, A, ktok, kld, rows, H, Mq, Tk,
                      Tq, causal)))
    return rc;
  if ((rc = dense_bmm(FAM_SEQ2SEQ, st, Op{A, cso, csi, Tk, 1}, Op{V, (int64_t)Tk * E, dh, E, 1}, O, (int64_t)Mq * E, dh, E, Mq,
                      dh, Tk, G, H, 1.f)))
    return rc;
  if ((rc = dense_mm(FAM_SEQ2SEQ, st, rm(O, E), rm(w + W.wo, E), Y, E, Nq, E, E, w + W.bo))) return rc;
  return s2_launch("k_s2s_ln", k_s2s_ln, blocks(Nq * 32, 256), 256, 0, st, xq, (const float*)Y, Nq, E, w + Nw.g, w + Nw.b,
                   r.seed, r.call, layer, r.rate, r.f(P.out), r.f(P.xh), r.f(P.rs));
}

int s2_ffn(const S2Run& r, const FF& W, const Norm& Nw, const SubP& P, const float* x, int64_t N, int layer) {
  const int E = r.c.E, F = r.c.F;
  const float* w = r.prm;
  int rc;
  if ((rc = dense_mm(FAM_SEQ2SEQ, r.st, rm(x, E), rm(w + W.w1, F), r.f(P.q), F, N, F, E, w + W.b1, 0, EP_RELU))) return rc;
  if ((rc = dense_mm(FAM_SEQ2SEQ, r.st, rm(r.f(P.q), F), rm(w + W.w2, E), r.f(P.y), E, N, E, F, w + W.b2))) return rc;
  return s2_launch("k_s2s_ln", k_s2s_ln, blocks(N * 32, 256), 256, 0, r.st, x, (const float*)r.f(P.y), N, E, w + Nw.g,
                   w + Nw.b, r.seed, r.call, layer, r.rate, r.f(P.out), r.f(P.xh), r.f(P.rs));
}

const float* s2_enc_out(const S2Run& r) { return r.f(r.p.enc[r.c.Le - 1][1].out); }
const float* s2_dec_out(const S2Run& r) { return r.f(r.p.dec[r.c.Ld - 1][2].out); }

int s2_encoder(const S2Run& r) {
  const int64_t Ne = (int64_t)r.n * r.Ts;
  int rc;
  if ((rc = s2_launch("k_s2s_embed", k_s2s_embed, blocks(Ne * r.c.E, 256), 256, 0, r.st, r.etok, (int64_t)r.Ts, r.n, r.Ts,
                      r.prm + r.L.emb_enc, r.c.Vs, r.c.E, r.f(r.p.xe))))
    return rc;
  const float* x = r.f(r.p.xe);
  for (int l = 0; l < r.c.Le; ++l) {
    const EncBlk& B = r.L.enc[l];
    if ((rc = s2_att(r, B.sa, B.n1, r.p.enc[l][0], x, Ne, x, Ne, r.n, r.Ts, r.Ts, r.Ts, 0, r.etok, r.Ts, true, 2 * l)))
      return rc;
    if ((rc = s2_ffn(r, B.ff, B.n2, r.p.enc[l][1], r.f(r.p.enc[l][0].out), Ne, 2 * l + 1))) return rc;
    x = r.f(r.p.enc[l][1].out);
  }
  return R4_OK;
}

// the cross-attention K / V of every decoder block from the encoder output (once per source row)
int s2_cross_kv(const S2Run& r) {
  const int E = r.c.E;
  const int64_t Ne = (int64_t)r.n * r.Ts;
  int rc;
  for (int l = 0; l < r.c.Ld; ++l) {
    const Att& W = r.L.dec[l].qa;
    if ((rc = dense_mm(FAM_SEQ2SEQ, r.st, rm(s2_enc_out(r), E), rm(r.prm + W.wk, E), r.f(r.p.dec[l][1].k), E, Ne, E, E,
                       r.prm + W.bk)))
      return rc;
    if ((rc = dense_mm(FAM_SEQ2SEQ, r.st, rm(s2_enc_out(r), E), rm(r.prm + W.wv, E), r.f(r.p.dec[l][1].v), E, Ne, E, E,
                       r.prm + W.bv)))
      return rc;
  }
  return R4_OK;
}

// the decoder over R prefixes per source row, each of Tt tokens at dtok + (row R + i) dld; kv: compute the cross K / V
int s2_decoder(const S2Run& r, const int32_t* dtok, int64_t dld, int R, int Tt, bool kv) {
  const int64_t P = (int64_t)r.n * R, Nd = P * Tt, Ne = (int64_t)r.n * r.Ts;
  int rc;
  if ((rc = s2_launch("k_s2s_embed", k_s2s_embed, blocks(Nd * r.c.E, 256), 256, 0, r.st, dtok, dld, (int)P, Tt,
                      r.prm + r.L.emb_dec, r.c.Vt, r.c.E, r.f(r.p.xd))))
    return rc;
  const float* x = r.f(r.p.xd);
  const int base = 2 * r.c.Le;
  for (int l = 0; l < r.c.Ld; ++l) {
    const DecBlk& B = r.L.dec[l];
    if ((rc = s2_att(r, B.sa, B.n1, r.p.dec[l][0], x, Nd, x, Nd, P, Tt, Tt, Tt, 1, dtok, dld, true, base + 3 * l))) return rc;
    if ((rc = s2_att(r, B.qa, B.n2, r.p.dec[l][1], r.f(r.p.dec[l][0].out), Nd, s2_enc_out(r), Ne, r.n, R * Tt, r.Ts, R * Tt, 0,
                     r.etok, r.Ts, kv, base + 3 * l + 1)))
      return rc;
    if ((rc = s2_ffn(r, B.ff, B.n3, r.p.dec[l][2], r.f(r.p.dec[l][1].out), Nd, base + 3 * l + 2))) return rc;
    x = r.f(r.p.dec[l][2].out);
  }
  return R4_OK;
}

// logits [rows, Vt] = h emb_dec^T + b for rows at row stride ld of the decoder output, from position `pos0`
int s2_logits(const S2Run& r, int64_t rows, int64_t ld, int pos0, float* out) {
  const int E = r.c.E;
  return dense_mm(FAM_SEQ2SEQ, r.st, Op{s2_dec_out(r) + (int64_t)pos0 * E, 0, 0, ld, 1}, tr(r.prm + r.L.emb_dec, E), out, r.c.Vt,
                  rows, r.c.Vt, E, r.prm + r.L.out_b);
}

// ---- backward ----
// LN backward of a sub-layer from dOut: gz <- the residual's gradient, dy <- the sub-layer output's; gx for gamma
int s2_ln_bwd(const S2Run& r, const Norm& Nw, const SubP& P, const float* dOut, int64_t N, int layer, float* gz) {
  return s2_launch("k_s2s_ln_bwd", k_s2s_ln_bwd, blocks(N * 32, 256), 256, 0, r.st, dOut, (const float*)r.f(P.xh),
                   (const float*)r.f(P.rs), N, r.c.E, r.prm + Nw.g, r.seed, r.call, layer, r.rate, gz, r.f(r.p.dy),
                   r.f(r.p.gx));
}

// FeedForward sub-layer backward: gz <- d(x) (x the sub-layer input) from dOut; weight gradients into grad
int s2_ffn_bwd(const S2Run& r, const FF& W, const Norm& Nw, const SubP& P, const float* x, int64_t N, int layer,
               const float* dOut, float* gz, float* grad) {
  const int E = r.c.E, F = r.c.F;
  const float* w = r.prm;
  int rc;
  if ((rc = s2_ln_bwd(r, Nw, P, dOut, N, layer, gz))) return rc;
  float *dy = r.f(r.p.dy), *dF = r.f(r.p.dF);
  if ((rc = dense_mm(FAM_SEQ2SEQ, r.st, rm(dy, E), tr(w + W.w2, E), dF, F, N, F, E, nullptr, 0, EP_DRELU, r.f(P.q)))) return rc;
  if ((rc = dense_mm(FAM_SEQ2SEQ, r.st, rm(dF, F), tr(w + W.w1, F), gz, E, N, E, F, nullptr, 1))) return rc;
  Jobs J;
  J.j[0] = grad_job(nullptr, 1, r.f(r.p.gx), 1, E, Nw.g);
  J.j[1] = grad_job(nullptr, 1, dOut, 1, E, Nw.b);
  int k = 2;
  layer_jobs(J, k, r.f(P.q), F, dy, F, E, W.w2, W.b2);
  layer_jobs(J, k, x, E, dF, E, F, W.w1, W.b1);
  tile_jobs(J, k);
  return dense_wgrad(FAM_SEQ2SEQ, r.st, J, N, 0, grad);
}

// attention sub-layer backward (the forward's arguments): gz <- d(xq); d(xkv) added into gkv (== gz for self-attention).
// Self-attention's key / value weight gradients share the query side's wgrad launch; cross-attention's, over the encoder
// rows, take a second one.
int s2_att_bwd(const S2Run& r, const Att& W, const Norm& Nw, const SubP& P, const float* xq, int64_t Nq, const float* xkv,
               int64_t Nk, int64_t G, int Mq, int Tk, bool self, int layer, const float* dOut, float* gz, float* gkv,
               float* grad) {
  const int E = r.c.E, H = r.c.H, dh = E / H;
  const float* w = r.prm;
  cudaStream_t st = r.st;
  int rc;
  if ((rc = s2_ln_bwd(r, Nw, P, dOut, Nq, layer, gz))) return rc;
  float *dy = r.f(r.p.dy), *dO = r.f(r.p.dO), *dA = r.f(r.p.dA), *dq = r.f(r.p.dq), *dk = r.f(r.p.dk), *dv = r.f(r.p.dv);
  const float *Q = r.f(P.q), *K = r.f(P.k), *V = r.f(P.v), *A = r.f(P.a);
  const int64_t cso = (int64_t)H * Mq * Tk, csi = (int64_t)Mq * Tk;
  const float alpha = 1.0f / sqrtf((float)dh);
  if ((rc = dense_mm(FAM_SEQ2SEQ, st, rm(dy, E), tr(w + W.wo, E), dO, E, Nq, E, E))) return rc;
  // dA = dO_h V_h^T; dV_h = A^T dO_h
  if ((rc = dense_bmm(FAM_SEQ2SEQ, st, Op{dO, (int64_t)Mq * E, dh, E, 1}, Op{V, (int64_t)Tk * E, dh, 1, E}, dA, cso, csi, Tk, Mq,
                      Tk, dh, G, H, 1.f)))
    return rc;
  if ((rc = dense_bmm(FAM_SEQ2SEQ, st, Op{A, cso, csi, 1, Tk}, Op{dO, (int64_t)Mq * E, dh, E, 1}, dv, (int64_t)Tk * E, dh, E, Tk,
                      dh, Mq, G, H, 1.f)))
    return rc;
  const int64_t rows = G * H * Mq;
  if ((rc = s2_launch("k_s2s_softmax_bwd", k_s2s_softmax_bwd, blocks(rows * 32, 256), 256, 0, st, A, dA, rows, Tk))) return rc;
  // dQ_h = alpha dS K_h; dK_h = alpha dS^T Q_h
  if ((rc = dense_bmm(FAM_SEQ2SEQ, st, Op{dA, cso, csi, Tk, 1}, Op{K, (int64_t)Tk * E, dh, E, 1}, dq, (int64_t)Mq * E, dh, E, Mq,
                      dh, Tk, G, H, alpha)))
    return rc;
  if ((rc = dense_bmm(FAM_SEQ2SEQ, st, Op{dA, cso, csi, 1, Tk}, Op{Q, (int64_t)Mq * E, dh, E, 1}, dk, (int64_t)Tk * E, dh, E, Tk,
                      dh, Mq, G, H, alpha)))
    return rc;
  if ((rc = dense_mm(FAM_SEQ2SEQ, st, rm(dq, E), tr(w + W.wq, E), gz, E, Nq, E, E, nullptr, 1))) return rc;
  if ((rc = dense_mm(FAM_SEQ2SEQ, st, rm(dk, E), tr(w + W.wk, E), gkv, E, Nk, E, E, nullptr, 1))) return rc;
  if ((rc = dense_mm(FAM_SEQ2SEQ, st, rm(dv, E), tr(w + W.wv, E), gkv, E, Nk, E, E, nullptr, 1))) return rc;
  Jobs J;
  J.j[0] = grad_job(nullptr, 1, r.f(r.p.gx), 1, E, Nw.g);
  J.j[1] = grad_job(nullptr, 1, dOut, 1, E, Nw.b);
  int nj = 2;
  layer_jobs(J, nj, r.f(P.o), E, dy, E, E, W.wo, W.bo);
  layer_jobs(J, nj, xq, E, dq, E, E, W.wq, W.bq);
  if (self) {
    layer_jobs(J, nj, xkv, E, dk, E, E, W.wk, W.bk);
    layer_jobs(J, nj, xkv, E, dv, E, E, W.wv, W.bv);
  }
  tile_jobs(J, nj);
  if ((rc = dense_wgrad(FAM_SEQ2SEQ, st, J, Nq, 0, grad))) return rc;
  if (self) return R4_OK;
  Jobs K2;
  nj = 0;
  layer_jobs(K2, nj, xkv, E, dk, E, E, W.wk, W.bk);
  layer_jobs(K2, nj, xkv, E, dv, E, E, W.wv, W.bv);
  tile_jobs(K2, nj);
  return dense_wgrad(FAM_SEQ2SEQ, st, K2, Nk, 0, grad);
}

// emb[tok] += dX over the positions of tok [rows, T] (contiguous)
int s2_emb_bwd(const S2Run& r, const int32_t* tok, int rows, int T, int V, const float* dX, float* demb) {
  int *cnt = r.as<int>(r.p.cnt), *off = r.as<int>(r.p.off), *order = r.as<int>(r.p.order);
  int rc;
  if ((rc = s2_launch("k_s2s_tok_csr", k_s2s_tok_csr, 1, 1024, 0, r.st, tok, (int64_t)T, rows, T, V, cnt, off))) return rc;
  if ((rc = s2_launch("k_s2s_tok_place", k_s2s_tok_place, blocks((int64_t)rows * T, 256), 256, 0, r.st, tok, (int64_t)T,
                      rows, T, V, (const int*)off, order)))
    return rc;
  return s2_launch("k_s2s_emb_grad", k_s2s_emb_grad, blocks((int64_t)V * r.c.E, 256), 256, 0, r.st, dX, r.c.E, V,
                   (const int*)cnt, (const int*)off, (const int*)order, demb);
}

// forward, loss and backward of one minibatch (tokens contiguous); grad overwritten
int s2_train(const S2Run& r, const int32_t* dtok, const int32_t* ytok, int Tt, float* grad, float* loss) {
  const int E = r.c.E, V = r.c.Vt, n = r.n;
  const int64_t Nd = (int64_t)n * Tt, Ne = (int64_t)n * r.Ts;
  const Layout& L = r.L;
  int rc;
  if (cudaMemsetAsync(grad, 0, L.n * sizeof(float), r.st) != cudaSuccess ||
      cudaMemsetAsync(r.f(r.p.denc), 0, Ne * E * sizeof(float), r.st) != cudaSuccess)
    return fail(R4_ERR_CUDA, "r4_s2s_grad: memset");
  if ((rc = s2_encoder(r))) return rc;
  if ((rc = s2_decoder(r, dtok, Tt, 1, Tt, true))) return rc;
  float* Z = r.f(r.p.logits);
  if ((rc = s2_logits(r, Nd, E, 0, Z))) return rc;
  if ((rc = s2_launch("k_s2s_count", k_s2s_count, 1, 1024, 0, r.st, dtok, (int)Nd, r.f(r.p.inv)))) return rc;
  if ((rc = s2_launch("k_s2s_out", k_s2s_out, (unsigned)Nd, 256, 0, r.st, Z, V, ytok, dtok, (const float*)r.f(r.p.inv),
                      r.f(r.p.ce))))
    return rc;
  if (loss && (rc = s2_launch("k_s2s_lsum", k_s2s_lsum, 1, 1024, 0, r.st, (const float*)r.f(r.p.ce), (int)Nd,
                              (const float*)r.f(r.p.inv), loss)))
    return rc;
  // output: dH = dZ emb_dec; emb_dec += dZ^T H; b += colsum dZ
  float* g[2] = {r.f(r.p.g[0]), r.f(r.p.g[1])};
  if ((rc = dense_mm(FAM_SEQ2SEQ, r.st, rm(Z, V), rm(r.prm + L.emb_dec, E), g[0], E, Nd, E, V))) return rc;
  Jobs J;
  J.j[0] = grad_job(Z, V, s2_dec_out(r), V, E, L.emb_dec);
  J.j[1] = grad_job(nullptr, 1, Z, 1, V, L.out_b);
  tile_jobs(J, 2);
  if ((rc = dense_wgrad(FAM_SEQ2SEQ, r.st, J, Nd, 0, grad))) return rc;
  int a = 0;
  const int base = 2 * r.c.Le;
  float* denc = r.f(r.p.denc);
  for (int l = r.c.Ld - 1; l >= 0; --l) {
    const DecBlk& B = L.dec[l];
    const Plan& p = r.p;
    const float* xin = l == 0 ? r.f(p.xd) : r.f(p.dec[l - 1][2].out);
    if ((rc = s2_ffn_bwd(r, B.ff, B.n3, p.dec[l][2], r.f(p.dec[l][1].out), Nd, base + 3 * l + 2, g[a], g[1 - a], grad)))
      return rc;
    a = 1 - a;
    if ((rc = s2_att_bwd(r, B.qa, B.n2, p.dec[l][1], r.f(p.dec[l][0].out), Nd, s2_enc_out(r), Ne, n, Tt, r.Ts, false,
                         base + 3 * l + 1, g[a], g[1 - a], denc, grad)))
      return rc;
    a = 1 - a;
    if ((rc = s2_att_bwd(r, B.sa, B.n1, p.dec[l][0], xin, Nd, xin, Nd, n, Tt, Tt, true, base + 3 * l, g[a], g[1 - a],
                         g[1 - a], grad)))
      return rc;
    a = 1 - a;
  }
  if ((rc = s2_emb_bwd(r, dtok, n, Tt, V, g[a], grad + L.emb_dec))) return rc;
  const float* cur = denc;
  for (int l = r.c.Le - 1; l >= 0; --l) {
    const EncBlk& B = L.enc[l];
    const Plan& p = r.p;
    const float* xin = l == 0 ? r.f(p.xe) : r.f(p.enc[l - 1][1].out);
    if ((rc = s2_ffn_bwd(r, B.ff, B.n2, p.enc[l][1], r.f(p.enc[l][0].out), Ne, 2 * l + 1, cur, g[a], grad))) return rc;
    if ((rc = s2_att_bwd(r, B.sa, B.n1, p.enc[l][0], xin, Ne, xin, Ne, n, r.Ts, r.Ts, true, 2 * l, g[a], g[1 - a], g[1 - a],
                         grad)))
      return rc;
    cur = g[1 - a];
  }
  return s2_emb_bwd(r, r.etok, n, r.Ts, r.c.Vs, cur, grad + L.emb_enc);
}

bool s2_len_ok(int T) { return T >= 1 && T <= MAXT; }

int s2_init(S2Run* r, const r4_s2s_config* cfg, const float* params, const int32_t* enc, int n, int Ts, void* scratch,
            void* stream) {
  if (!s2_cfg_ok(cfg) || !params || !enc || !scratch || n < 1 || !s2_len_ok(Ts) || (int64_t)n * cfg->head_num > 65535)
    return fail(R4_ERR_ARG, "bad argument");
  r->prm = params; r->c = s2_cfg(cfg); r->L = make_layout(r->c); r->s = static_cast<float*>(scratch); r->st = S(stream);
  r->n = n; r->Ts = Ts; r->etok = enc; r->seed = 0; r->call = 0; r->rate = 0.f;
  return R4_OK;
}

int s2_adam(const Cfg& c, float* params, const float* grad, float* m, float* v, int step, float lr, float b1, float b2,
            float eps, cudaStream_t st) {
  const int64_t np = make_layout(c).n;
  const float alpha = lr * sqrtf(1.f - powf(b2, (float)step)) / (1.f - powf(b1, (float)step));
  return s2_launch("k_s2s_adam", k_s2s_adam, blocks(np, 256), 256, 0, st, np, (int64_t)0, np, np, params,
                   const_cast<float*>(grad), m, v, alpha, b1, b2, eps);
}

// the top-k step after the decoder ran over n R prefixes of Tt tokens: probabilities of the last position, then top-k
int s2_topk(const S2Run& r, int64_t P, int Tt, const int32_t* cand, int C, int group, int k, double* val, int32_t* idx) {
  float* Z = r.f(r.p.logits);
  const int V = r.c.Vt;
  int rc;
  if ((rc = s2_logits(r, P, (int64_t)Tt * r.c.E, Tt - 1, Z))) return rc;
  if ((rc = s2_launch("k_s2s_out", k_s2s_out, (unsigned)P, 256, 0, r.st, Z, V, (const int32_t*)nullptr,
                      (const int32_t*)nullptr, (const float*)nullptr, (float*)nullptr)))
    return rc;
  const int P2 = pow2_at_least(k);
  const size_t smem = (size_t)P2 * 12 + (cand ? (size_t)(V + 31) / 32 * 4 : 0);
  return s2_launch("k_s2s_topk", k_s2s_topk, (unsigned)P, 256, smem, r.st, (const float*)Z, V, cand, C, group, k, val, idx);
}

}  // namespace

extern "C" {

int64_t r4_s2s_launch_count(void) { return g_launches[FAM_SEQ2SEQ].load(std::memory_order_relaxed); }

int64_t r4_s2s_num_params(const r4_s2s_config* cfg) { return s2_cfg_ok(cfg) ? make_layout(s2_cfg(cfg)).n : -1; }

int64_t r4_s2s_scratch_size(const r4_s2s_config* cfg, int mode, int n, int src_len, int tgt_len, int beam, int k) {
  if (!s2_cfg_ok(cfg) || n < 1 || !s2_len_ok(src_len) || !s2_len_ok(tgt_len) || beam < 1 || beam > MAXBEAM) return -1;
  if ((int64_t)n * beam * cfg->head_num > 65535) return -1;
  const Cfg c = s2_cfg(cfg);
  Plan p;
  if (mode == R4_S2S_TRAIN) p = s2_plan(c, n, src_len, tgt_len, 1, (int64_t)n * tgt_len, true, 0, 0);
  else if (mode == R4_S2S_PREDICT) p = s2_plan(c, n, src_len, tgt_len, beam, (int64_t)n * beam * tgt_len, false, 0, 0);
  else if (mode == R4_S2S_SEARCH) {
    if (tgt_len >= MAXT || k < 0 || k > MAXK) return -1;
    p = s2_plan(c, n, src_len, tgt_len, beam, (int64_t)n * beam, false, beam, k);
  } else if (mode == R4_S2S_STEP) {
    if (k < 1 || k > MAXK) return -1;
    p = s2_plan(c, n, src_len, tgt_len, 1, n, false, 0, 0);
  } else {
    return -1;
  }
  return p.n * (int64_t)sizeof(float);
}

int r4_s2s_relu_offsets(const r4_s2s_config* cfg, int n, int src_len, int tgt_len, int64_t* offsets) {
  // the shapes r4_s2s_grad accepts, the grid's z extent n * heads included: offsets of a plan no training call can run
  // would describe nothing
  if (!s2_cfg_ok(cfg) || !offsets || n < 1 || !s2_len_ok(src_len) || !s2_len_ok(tgt_len) ||
      (int64_t)n * cfg->head_num > 65535)
    return fail(R4_ERR_ARG, "bad argument");
  const Cfg c = s2_cfg(cfg);
  const Plan p = s2_plan(c, n, src_len, tgt_len, 1, (int64_t)n * tgt_len, true, 0, 0);
  int k = 0;
  for (int l = 0; l < c.Le; ++l) offsets[k++] = p.enc[l][1].q * (int64_t)sizeof(float);
  for (int l = 0; l < c.Ld; ++l) offsets[k++] = p.dec[l][2].q * (int64_t)sizeof(float);
  return k;
}

int r4_s2s_grad(const r4_s2s_config* cfg, const float* params, const int32_t* enc, const int32_t* dec, const int32_t* target,
                int n, int src_len, int tgt_len, uint64_t seed, uint64_t call, float dropout, float* grad, float* loss,
                void* scratch, void* stream) {
  S2Run r;
  if (int rc = s2_init(&r, cfg, params, enc, n, src_len, scratch, stream)) return rc;
  if (!dec || !target || !grad || !s2_len_ok(tgt_len) || !(dropout >= 0.f && dropout < 1.f))
    return fail(R4_ERR_ARG, "bad argument");
  r.seed = seed; r.call = call; r.rate = dropout;
  r.p = s2_plan(r.c, n, src_len, tgt_len, 1, (int64_t)n * tgt_len, true, 0, 0);
  return s2_train(r, dec, target, tgt_len, grad, loss);
}

int r4_s2s_apply(const r4_s2s_config* cfg, float* params, const float* grad, float* m, float* v, int step, float lr,
                 float beta1, float beta2, float eps, void* stream) {
  if (!s2_cfg_ok(cfg) || !params || !grad || !m || !v || step < 1) return fail(R4_ERR_ARG, "bad argument");
  return s2_adam(s2_cfg(cfg), params, grad, m, v, step, lr, beta1, beta2, eps, S(stream));
}

int r4_s2s_epoch(const r4_s2s_config* cfg, float* params, float* grad, float* m, float* v, const int32_t* enc,
                 const int32_t* dec, const int32_t* target, int64_t N, int src_len, int tgt_len, const int64_t* perm,
                 int64_t n_perm, int batch, int step0, uint64_t seed, uint64_t call0, float dropout, float lr, float beta1,
                 float beta2, float eps, float* losses, void* scratch, void* stream) {
  S2Run r;
  if (int rc = s2_init(&r, cfg, params, enc, batch, src_len, scratch, stream)) return rc;
  if (!grad || !m || !v || !dec || !target || !perm || !losses || N < 1 || n_perm < 1 || step0 < 0 || !s2_len_ok(tgt_len) ||
      !(dropout >= 0.f && dropout < 1.f))
    return fail(R4_ERR_ARG, "bad argument");
  const int64_t steps = (n_perm + batch - 1) / batch;
  const Plan full = s2_plan(r.c, batch, src_len, tgt_len, 1, (int64_t)batch * tgt_len, true, 0, 0);
  int32_t *et = r.as<int32_t>(full.et), *dt = r.as<int32_t>(full.dt), *yt = r.as<int32_t>(full.yt);
  r.seed = seed; r.rate = dropout;
  for (int64_t k = 0; k < steps; ++k) {
    const int nb = (int)std::min<int64_t>(batch, n_perm - k * batch);
    const int W = src_len + 2 * tgt_len;
    if (int rc = s2_launch("k_s2s_gather", k_s2s_gather, blocks((int64_t)nb * W, 256), 256, 0, r.st, enc, src_len, dec,
                           target, tgt_len, perm + k * batch, nb, et, dt, yt))
      return rc;
    // the minibatch's planes: the plan of nb rows, its token planes at the full batch's offsets (past every other plane)
    r.n = nb; r.etok = et; r.call = call0 + (uint64_t)k;
    r.p = s2_plan(r.c, nb, src_len, tgt_len, 1, (int64_t)nb * tgt_len, true, 0, 0);
    if (int rc = s2_train(r, dt, yt, tgt_len, grad, losses + k)) return rc;
    if (int rc = s2_adam(r.c, params, grad, m, v, step0 + (int)k + 1, lr, beta1, beta2, eps, r.st)) return rc;
  }
  return R4_OK;
}

int r4_s2s_predict(const r4_s2s_config* cfg, const float* params, const int32_t* enc, const int32_t* dec, int n, int src_len,
                   int tgt_len, float* probs, void* scratch, void* stream) {
  S2Run r;
  if (int rc = s2_init(&r, cfg, params, enc, n, src_len, scratch, stream)) return rc;
  if (!dec || !probs || !s2_len_ok(tgt_len)) return fail(R4_ERR_ARG, "bad argument");
  r.p = s2_plan(r.c, n, src_len, tgt_len, 1, 0, false, 0, 0);
  int rc;
  if ((rc = s2_encoder(r)) || (rc = s2_decoder(r, dec, tgt_len, 1, tgt_len, true))) return rc;
  const int64_t rows = (int64_t)n * tgt_len;
  if ((rc = s2_logits(r, rows, r.c.E, 0, probs))) return rc;
  return s2_launch("k_s2s_out", k_s2s_out, (unsigned)rows, 256, 0, r.st, probs, r.c.Vt, (const int32_t*)nullptr,
                   (const int32_t*)nullptr, (const float*)nullptr, (float*)nullptr);
}

int r4_s2s_decode_step(const r4_s2s_config* cfg, const float* params, const int32_t* enc, int n, int src_len,
                       const int32_t* dec, int tgt_len, const int32_t* cand, int n_cand, int k, double* val, int32_t* idx,
                       void* scratch, void* stream) {
  S2Run r;
  if (int rc = s2_init(&r, cfg, params, enc, n, src_len, scratch, stream)) return rc;
  if (!dec || !val || !idx || !s2_len_ok(tgt_len) || k < 1 || k > MAXK || k >= cfg->tgt_tokens ||
      (cand && (n_cand < 1 || n_cand > MAXK)))
    return fail(R4_ERR_ARG, "bad argument");
  r.p = s2_plan(r.c, n, src_len, tgt_len, 1, n, false, 0, 0);
  int rc;
  if ((rc = s2_encoder(r)) || (rc = s2_decoder(r, dec, tgt_len, 1, tgt_len, true))) return rc;
  return s2_topk(r, n, tgt_len, cand, n_cand, 1, k, val, idx);
}

int r4_s2s_beam_search(const r4_s2s_config* cfg, const float* params, const int32_t* enc, int n, int src_len, int beam,
                       int target_len, int n_cand, int32_t* path, double* score, void* scratch, void* stream) {
  S2Run r;
  if (int rc = s2_init(&r, cfg, params, enc, n, src_len, scratch, stream)) return rc;
  if (!path || !score || beam < 1 || beam > MAXBEAM || beam >= cfg->tgt_tokens || target_len < 1 || target_len >= MAXT ||
      n_cand < 0 || n_cand > MAXK || n_cand >= cfg->tgt_tokens || (int64_t)n * beam * cfg->head_num > 65535)
    return fail(R4_ERR_ARG, "bad argument");
  r.p = s2_plan(r.c, n, src_len, target_len, beam, (int64_t)n * beam, false, beam, n_cand);
  const int L = target_len + 1;
  const int64_t P = (int64_t)n * beam;
  int32_t* pa[2] = {r.as<int32_t>(r.p.path[0]), r.as<int32_t>(r.p.path[1])};
  double* sa[2] = {r.as<double>(r.p.score[0]), r.as<double>(r.p.score[1])};
  double* val = r.as<double>(r.p.val);
  int32_t* idx = r.as<int32_t>(r.p.idx);
  int32_t* cand = n_cand > 0 ? r.as<int32_t>(r.p.cand) : nullptr;
  int rc;
  if ((rc = s2_launch("k_s2s_start", k_s2s_start, blocks(P * L, 256), 256, 0, r.st, P, L, pa[0]))) return rc;
  if ((rc = s2_encoder(r)) || (rc = s2_cross_kv(r))) return rc;
  // step 1: the n START prefixes (row b's beam 0), top beam; the candidates are the top n_cand of the same probabilities
  if ((rc = s2_decoder(r, pa[0], (int64_t)beam * L, 1, 1, false))) return rc;
  if ((rc = s2_topk(r, n, 1, nullptr, 0, 1, beam, val, idx))) return rc;
  if ((rc = s2_launch("k_s2s_first", k_s2s_first, blocks(P, 256), 256, 0, r.st, (const double*)val, (const int32_t*)idx, P,
                      L, pa[0], sa[0])))
    return rc;
  if (cand) {
    const size_t smem = (size_t)pow2_at_least(n_cand) * 12;
    if ((rc = s2_launch("k_s2s_topk", k_s2s_topk, (unsigned)n, 256, smem, r.st, (const float*)r.f(r.p.logits), r.c.Vt,
                        (const int32_t*)nullptr, 0, 1, n_cand, r.as<double>(r.p.cval), cand)))
      return rc;
  }
  int cur = 0;
  const size_t bsm = (size_t)pow2_at_least(beam) * 12;
  for (int i = 1; i < target_len; ++i) {
    if ((rc = s2_decoder(r, pa[cur], L, beam, i + 1, false))) return rc;
    if ((rc = s2_topk(r, P, i + 1, cand, n_cand, beam, beam, val, idx))) return rc;
    if ((rc = s2_launch("k_s2s_beam", k_s2s_beam, (unsigned)n, 256, bsm, r.st, (const double*)sa[cur], (const double*)val,
                        (const int32_t*)idx, (const int32_t*)pa[cur], beam, L, i + 1, pa[1 - cur], sa[1 - cur])))
      return rc;
    cur = 1 - cur;
  }
  if (cudaMemcpyAsync(path, pa[cur], P * L * sizeof(int32_t), cudaMemcpyDeviceToDevice, r.st) != cudaSuccess ||
      cudaMemcpyAsync(score, sa[cur], P * sizeof(double), cudaMemcpyDeviceToDevice, r.st) != cudaSuccess)
    return fail(R4_ERR_CUDA, "r4_s2s_beam_search: copy");
  return R4_OK;
}

int r4_s2s_score(const r4_s2s_config* cfg, const float* params, const int32_t* enc, int n, int src_len, const int32_t* path,
                 int beam, int target_len, float* prob, void* scratch, void* stream) {
  S2Run r;
  if (int rc = s2_init(&r, cfg, params, enc, n, src_len, scratch, stream)) return rc;
  if (!path || !prob || beam < 1 || beam > MAXBEAM || !s2_len_ok(target_len) || (int64_t)n * beam * cfg->head_num > 65535)
    return fail(R4_ERR_ARG, "bad argument");
  const int64_t P = (int64_t)n * beam, rows = P * target_len;
  r.p = s2_plan(r.c, n, src_len, target_len, beam, rows, false, 0, 0);
  int rc;
  if ((rc = s2_encoder(r)) || (rc = s2_decoder(r, path, target_len + 1, beam, target_len, true))) return rc;
  float* Z = r.f(r.p.logits);
  if ((rc = s2_logits(r, rows, r.c.E, 0, Z))) return rc;
  if ((rc = s2_launch("k_s2s_out", k_s2s_out, (unsigned)rows, 256, 0, r.st, Z, r.c.Vt, (const int32_t*)nullptr,
                      (const int32_t*)nullptr, (const float*)nullptr, (float*)nullptr)))
    return rc;
  return s2_launch("k_s2s_pick", k_s2s_pick, blocks(rows, 256), 256, 0, r.st, (const float*)Z, r.c.Vt, path,
                   target_len + 1, (int)P, target_len, prob);
}

}  // extern "C"

// ---- off-policy evaluation (r4_ope.cuh) ------------------------------------------------------------------------------------
namespace {
using namespace r4ope;

template <typename... P, typename... A>
int ope_launch(const char* name, void (*kernel)(P...), dim3 grid, int threads, cudaStream_t st, A&&... args) {
  return launch(FAM_OPE, name, kernel, grid, threads, 0, st, false, std::forward<A>(args)...);
}

constexpr int OPE_MAX_B = 1 << 21, OPE_MAX_C = 1 << 16, OPE_MAX_H = 1 << 24, OPE_MAX_A = 1 << 16;
constexpr int OPE_U = 128, OPE_F = 256;        // the dense tower's width, the two 256-unit layers

bool ope_c_ok(int C) { return C >= 149 && C <= OPE_MAX_C; }

// Float offsets of the behaviour net's flat parameters, in the order include/rl4rs_b200.h documents.
struct OpeLayout { int64_t emb, w1, b1, w2, b2, fc_w, fc_b, obs_w, obs_b, rew_w, rew_b, n; };
OpeLayout ope_layout(int H, int C) {
  OpeLayout L;
  int64_t o = 0;
  auto take = [&](int64_t k) { const int64_t r = o; o += k; return r; };
  L.emb = take((int64_t)H * E);
  L.w1 = take((int64_t)NDENSE * OPE_U); L.b1 = take(OPE_U);
  L.w2 = take((int64_t)OPE_U * OPE_U); L.b2 = take(OPE_U);
  L.fc_w = take((int64_t)CAT_LD * OPE_F); L.fc_b = take(OPE_F);
  L.obs_w = take((int64_t)OPE_F * OPE_F); L.obs_b = take(OPE_F);
  L.rew_w = take((int64_t)OPE_F * C); L.rew_b = take(C);
  L.n = o;
  return L;
}
}  // namespace

extern "C" {

int64_t r4_ope_num_params(int H, int C) {
  if (H < 1 || H > OPE_MAX_H || !ope_c_ok(C)) return -1;
  return ope_layout(H, C).n;
}

int64_t r4_ope_behavior_scratch_size(int B, int C) {
  if (B < 1 || B > OPE_MAX_B || !ope_c_ok(C)) return -1;
  return (int64_t)B * (NDENSE + OPE_U + CAT_LD + 2 * OPE_F + C);
}

int r4_ope_behavior(int B, int H, int C, int K, int P, int page, const float* params, const int32_t* head,
                    const int32_t* items, const float* feat, float* out, float* scratch, void* stream) {
  if (B < 1 || B > OPE_MAX_B || H < 1 || H > OPE_MAX_H || !ope_c_ok(C) || K < 1 || K > NCAT - NHEAD || P < 1 ||
      page < 0 || page >= P || !params || !head || !items || !feat || !out || !scratch)
    return fail(R4_ERR_ARG, "r4_ope_behavior: bad argument");
  const OpeLayout L = ope_layout(H, C);
  const cudaStream_t st = S(stream);
  float* dense = scratch;
  float* h1 = dense + (size_t)B * NDENSE;
  float* cat = h1 + (size_t)B * OPE_U;
  float* a = cat + (size_t)B * CAT_LD;
  float* o = a + (size_t)B * OPE_F;
  float* z = o + (size_t)B * OPE_F;
  const float* p = params;
  int rc;
  if ((rc = ope_launch("k_ope_inputs", k_ope_inputs, dim3(B), E, st, B, K, P, page, H, head, items, feat, p + L.emb, cat,
                       dense)) ||
      (rc = dense_mm(FAM_OPE, st, rm(dense, NDENSE), rm(p + L.w1, OPE_U), h1, OPE_U, B, OPE_U, NDENSE, p + L.b1, 0, EP_ELU)) ||
      (rc = dense_mm(FAM_OPE, st, rm(h1, OPE_U), rm(p + L.w2, OPE_U), cat + E, CAT_LD, B, OPE_U, OPE_U, p + L.b2, 0, EP_ELU)) ||
      (rc = dense_mm(FAM_OPE, st, rm(cat, CAT_LD), rm(p + L.fc_w, OPE_F), a, OPE_F, B, OPE_F, CAT_LD, p + L.fc_b, 0, EP_ELU)) ||
      (rc = dense_mm(FAM_OPE, st, rm(a, OPE_F), rm(p + L.obs_w, OPE_F), o, OPE_F, B, OPE_F, OPE_F, p + L.obs_b, 0, EP_ELU)) ||
      (rc = dense_mm(FAM_OPE, st, rm(o, OPE_F), rm(p + L.rew_w, C), z, C, B, C, OPE_F, p + L.rew_b)))
    return rc;
  return ope_launch("k_ope_softmax", k_ope_softmax, dim3(B), r4ope::NT, st, B, C, (const float*)z, out);
}

int r4_ope_step(int t, int T, int B, int A, int C, int layer, const float* probs, int logits, const int32_t* off,
                const float* block, const int32_t* own, const float* values, int per_action, const double* reward,
                const double* off_reward, float* pol, float* beh, float* val, double* rew, double* offr, void* stream) {
  if (T < 1 || t < 0 || t >= T || B < 1 || B > OPE_MAX_B || A < 2 || A > OPE_MAX_A || !ope_c_ok(C) || C < A ||
      layer < 1 || (logits != 0 && logits != 1) || (per_action != 0 && per_action != 1) || !probs || !off || !block ||
      (per_action && !own) || !values || !reward || !off_reward || !pol || !beh || !val || !rew || !offr)
    return fail(R4_ERR_ARG, "r4_ope_step: bad argument");
  constexpr int rows = r4ope::NT / 32;
  return ope_launch("k_ope_step", k_ope_step, dim3((B + rows - 1) / rows), r4ope::NT, S(stream), t, B, A, C, layer, probs,
                    logits, off, block, own, values, per_action, reward, off_reward, pol, beh, val, rew, offr);
}

int64_t r4_ope_launch_count(void) { return g_launches[FAM_OPE].load(std::memory_order_relaxed); }

}  // extern "C"
