// r4_host.h -- host pieces shared by r4_capi.cu (the env) and r4_learn.cu (the learners): the process-wide error message,
// per-device SM counts, and the one launcher every learner kernel goes through.  Plain CUDA runtime, no kernels.
#pragma once
#include "../../include/rl4rs_b200.h"

#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <utility>

namespace r4h {

// The message r4_last_error(NULL) returns: the last failure of a call that has no env handle, from either file.
inline std::string& last_error() {
  static std::string s;
  return s;
}

inline int fail(int code, const std::string& msg) {
  last_error() = msg;
  return code;
}

inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// SMs of the current device (132 on an H100 SXM), queried once per device
inline int sm_count() {
  static std::mutex mu;
  static std::map<int, int> sms;
  int d = 0;
  cudaGetDevice(&d);
  std::lock_guard<std::mutex> lock(mu);
  auto it = sms.find(d);
  if (it == sms.end()) {
    int v = 132;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d);
    it = sms.emplace(d, v).first;
  }
  return it->second;
}

// Learner families, each with its own launch counter (r4_batchrl_launch_count, r4_simtrain_launch_count,
// r4_exactk_launch_count, r4_s2s_launch_count, r4_ope_launch_count); the online learners (PPO / A2C, Gaussian, DDPG / TD3, RAINBOW and the
// peer-memory exchange) share one.
enum Family { FAM_ONLINE, FAM_BATCHRL, FAM_SIMTRAIN, FAM_EXACTK, FAM_SEQ2SEQ, FAM_OPE, FAM_COUNT };

inline std::atomic<int64_t> g_launches[FAM_COUNT];

inline void count_launch(Family f) { g_launches[f].fetch_add(1, std::memory_order_relaxed); }

// Raise fn's dynamic shared-memory limit on the current device to smem when smem is above the 48 KB default and above the
// value last set for fn there.  cudaFuncSetAttribute applies per device, so the record is kept per (kernel, device).
inline cudaError_t smem_optin(const void* fn, size_t smem) {
  if (smem <= 48 * 1024) return cudaSuccess;
  int d = 0;
  cudaError_t st = cudaGetDevice(&d);
  if (st != cudaSuccess) return st;
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> set;
  std::lock_guard<std::mutex> lock(mu);
  size_t& cur = set[{fn, d}];
  if (smem <= cur) return cudaSuccess;
  st = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (st == cudaSuccess) cur = smem;
  return st;
}

// Launch one learner kernel and count it against its family.  pdl: programmatic dependent launch, for chains whose
// kernels wait on griddepcontrol.  Returns R4_OK, or R4_ERR_CUDA with "<name>: <cuda error>".
template <typename... P, typename... A>
int launch(Family fam, const char* name, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
           bool pdl, A&&... args) {
  cudaError_t st = smem_optin((const void*)kernel, smem);
  if (st != cudaSuccess) {
    cudaGetLastError();
    return fail(R4_ERR_CUDA, std::string("cudaFuncSetAttribute(") + name + "): " + cudaGetErrorString(st));
  }
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t lc = {};
  lc.gridDim = grid;
  lc.blockDim = block;
  lc.dynamicSmemBytes = smem;
  lc.stream = stream;
  lc.attrs = at;
  lc.numAttrs = pdl ? 1 : 0;
  count_launch(fam);
  st = cudaLaunchKernelEx(&lc, kernel, std::forward<A>(args)...);
  const cudaError_t last = cudaGetLastError();   // also reports (and clears) an earlier asynchronous error
  if (st == cudaSuccess) st = last;
  return st == cudaSuccess ? R4_OK : fail(R4_ERR_CUDA, std::string(name) + ": " + cudaGetErrorString(st));
}

}  // namespace r4h
