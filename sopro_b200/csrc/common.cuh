// Host-side helpers every unit of the library shares: the error message behind sopro_last_error(), the check of a CUDA
// runtime call, and the row lengths of a ragged-batch launch.
#pragma once

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>

#include "../../include/sopro_b200.h"

namespace mimi {
void set_error(const char* msg);  // the library's per-thread error message (ar_engine.cu)
}

// formats the message sopro_last_error() returns on this thread, and returns `code`
inline int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  mimi::set_error(buf);
  return code;
}

#define CK(call)                                                                                      \
  do {                                                                                                \
    cudaError_t e__ = (call);                                                                         \
    if (e__ != cudaSuccess)                                                                           \
      return fail(SOPRO_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

// the valid samples of each row of one launch: passed by value, so the lengths travel as a kernel parameter
template <int N>
struct RowLens {
  long long v[N];
};
