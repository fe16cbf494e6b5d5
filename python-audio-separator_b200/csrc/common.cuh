// Shared helpers for libb200sep (sm_90a).  Error plumbing, launch accounting, small device utilities.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/b200sep.h"

namespace b200sep {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define B2_CHECK_ARG(cond, ...)            \
  do {                                     \
    if (!(cond)) {                         \
      ::b200sep::set_error(__VA_ARGS__);   \
      return B200SEP_ERR_ARG;              \
    }                                      \
  } while (0)

#define B2_CUDA(call)                                                                              \
  do {                                                                                             \
    cudaError_t e__ = (call);                                                                      \
    if (e__ != cudaSuccess) {                                                                      \
      ::b200sep::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
      (void)cudaGetLastError(); /* a failed launch API call also latches the error: do not let the NEXT launch check report it */ \
      return B200SEP_ERR_CUDA;                                                                     \
    }                                                                                              \
  } while (0)

// call after a kernel launch
#define B2_LAUNCHED()                                                                          \
  do {                                                                                         \
    ::b200sep::count_launch();                                                                 \
    cudaError_t e__ = cudaGetLastError();                                                      \
    if (e__ != cudaSuccess) {                                                                  \
      ::b200sep::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
      return B200SEP_ERR_CUDA;                                                                 \
    }                                                                                          \
  } while (0)

static inline int cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

constexpr int kNumSMs = 132;  // H100 SXM

}  // namespace b200sep
