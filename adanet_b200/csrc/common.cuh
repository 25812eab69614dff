// Shared helpers for the adanet_b200 CUDA library (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/adanet_b200.h"

namespace adn {

extern thread_local char g_err[512];
extern std::atomic<long long> g_launches;

int fail(int code, const char* fmt, ...);

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Every kernel launch in the library goes through this so that
// adn_query(ADN_Q_LAUNCH_COUNT) is an honest count of OUR kernels.
#define ADN_COUNT_LAUNCH() (::adn::g_launches.fetch_add(1, std::memory_order_relaxed))

#define ADN_CHECK_LAUNCH(what)                                                         \
  do {                                                                                 \
    ADN_COUNT_LAUNCH();                                                                \
    cudaError_t e__ = cudaGetLastError();                                              \
    if (e__ != cudaSuccess) return ::adn::fail(ADN_ERR_CUDA, "%s: launch failed: %s",  \
                                               what, cudaGetErrorString(e__));         \
  } while (0)

#define ADN_CUDA(call)                                                                 \
  do {                                                                                 \
    cudaError_t e__ = (call);                                                          \
    if (e__ != cudaSuccess) return ::adn::fail(ADN_ERR_CUDA, "%s failed: %s", #call,   \
                                               cudaGetErrorString(e__));               \
  } while (0)

int sm_count();

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline int64_t align_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }

// dense path selection (dense_api.cu)
int dense_path();

}  // namespace adn
