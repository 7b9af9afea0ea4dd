// Host-side helpers every unit of the library shares: the error message behind sopro_last_error(), the check of a CUDA
// runtime call, the device check of every create, and the checks and row lengths of a ragged batch.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdint>
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

// makes `device` current for a unit that runs on it (`what` names the unit): SOPRO_ERR_UNSUPPORTED without a CUDA
// device or on one that is not sm_90 (the library is built for sm_90a only), SOPRO_ERR_INVALID for a device out of range
inline int open_device(int device, const char* what) {
  int ndev = 0;
  const cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev <= 0)
    return fail(SOPRO_ERR_UNSUPPORTED, "no CUDA device (%s); %s has no CPU fallback",
                ce == cudaSuccess ? "device count 0" : cudaGetErrorString(ce), what);
  if (device < 0 || device >= ndev) return fail(SOPRO_ERR_INVALID, "device %d out of range [0,%d)", device, ndev);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9)
    return fail(SOPRO_ERR_UNSUPPORTED, "device %d is sm_%d%d; this build targets sm_90a only", device, prop.major, prop.minor);
  CK(cudaSetDevice(device));
  return SOPRO_OK;
}

// A ragged batch: row b is x + b * x_stride with lens[b] valid samples (x_stride each when lens is null).  Checks B,
// x_stride <= max_len (the unit's length bound), every lens[b] in [0, x_stride], and x when a row is non-empty; the
// longest row's length -> *most.
inline int check_rows(const float* x, int B, long long x_stride, const int64_t* lens, long long max_len, long long* most) {
  if (B < 1 || x_stride < 0 || x_stride > max_len)
    return fail(SOPRO_ERR_INVALID, "bad batch geometry (B=%d, x_stride=%lld)", B, x_stride);
  *most = 0;
  for (int b = 0; b < B; ++b) {
    const long long len = lens ? lens[b] : x_stride;
    if (len < 0 || len > x_stride) return fail(SOPRO_ERR_INVALID, "lens[%d] = %lld not in [0, x_stride = %lld]", b, len, x_stride);
    *most = std::max(*most, len);
  }
  if (!x && *most > 0) return fail(SOPRO_ERR_INVALID, "null argument");
  return SOPRO_OK;
}

// the output rows of a ragged batch: y when any row has outputs, and room for the longest row's `most` between rows
inline int check_out_rows(const float* y, int B, long long y_stride, long long most) {
  if (!y && most > 0) return fail(SOPRO_ERR_INVALID, "null argument");
  if (B > 1 && y_stride < most) return fail(SOPRO_ERR_INVALID, "y_stride %lld < the longest row's %lld outputs", y_stride, most);
  return SOPRO_OK;
}

// the valid samples of each row of one launch: passed by value, so the lengths travel as a kernel parameter
template <int N>
struct RowLens {
  long long v[N];
};

// rows [b0, b0 + rows) of a ragged batch, rows <= N
template <int N>
RowLens<N> row_lens(const int64_t* lens, long long x_stride, int b0, int rows) {
  RowLens<N> L{};
  for (int i = 0; i < rows; ++i) L.v[i] = lens ? lens[b0 + i] : x_stride;
  return L;
}
