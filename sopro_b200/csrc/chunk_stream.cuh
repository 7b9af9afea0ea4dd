// What every streaming output stage shares.  The contract (include/sopro_b200.h): one utterance pushed in chunks of at
// most max_chunk samples; once finished, a push or a finish is SOPRO_ERR_STATE until a reset; an oversized push is
// refused with nothing launched and the state unchanged.  Here are the state behind that contract, its preconditions, and the
// carried tail: the input samples that a later push or the finish still reads.  A stage keeps only its geometry (what a
// push makes ready, where its tail starts), its launches and its own state.
#pragma once

#include "common.cuh"

namespace chunk {

// where the input sample at logical index k comes from: [0, split) from a (a[k - a_base]), [split, limit) from b
// (b[k - split]), zero elsewhere -- the one-shot path has a single source, a stream its carried tail and the new chunk
struct Src {
  const float* a;
  const float* b;
  long long a_base, split, limit;
};

__device__ __forceinline__ float src_at(const Src& s, long long k) {
  if (k < 0 || k >= s.limit) return 0.0f;
  return k < s.split ? s.a[k - s.a_base] : s.b[k - s.split];
}

// An utterance's input samples [base, seen), carried on the device from one push to the next in buf[cur].  The pair
// is a ping-pong: a push reads the old tail while the new one is copied into the other buffer.  A base below 0 holds
// nothing there (the samples before the utterance are zero and never read).
struct Tail {
  int device = 0;  // the device the buffers live on
  float* buf[2] = {nullptr, nullptr};
  int cur = 0;
  long long base = 0, seen = 0;

  // two buffers of cap samples on the current device
  cudaError_t alloc(size_t cap) {
    cudaError_t e = cudaGetDevice(&device);
    for (int i = 0; i < 2 && e == cudaSuccess; ++i) e = cudaMalloc(&buf[i], cap * sizeof(float));
    return e;
  }
  // frees the buffers, and leaves their device current
  void release() {
    cudaSetDevice(device);
    cudaFree(buf[0]);
    cudaFree(buf[1]);
  }
  void restart(long long b) {
    cur = 0;
    base = b;
    seen = 0;
  }
  const float* data() const { return buf[cur]; }
  long long held() const { return seen - base; }
  // the tail, then the chunk x [n]
  Src src(const float* x, long long n) const { return Src{buf[cur], x, base, seen, seen + n}; }
  // after a push of x [n]: the tail becomes [new_base, seen + n) in the other buffer, from what is left of the old
  // tail and then from the chunk
  int keep(long long new_base, const float* x, long long n, cudaStream_t st) {
    const long long end = seen + n;
    float* dst = buf[cur ^ 1];
    long long k = new_base;
    if (k < seen) {
      CK(cudaMemcpyAsync(dst, buf[cur] + (k - base), (size_t)(seen - k) * sizeof(float), cudaMemcpyDeviceToDevice, st));
      k = seen;
    }
    if (end > k) CK(cudaMemcpyAsync(dst + (k - new_base), x + (k - seen), (size_t)(end - k) * sizeof(float), cudaMemcpyDeviceToDevice, st));
    cur ^= 1;
    base = new_base;
    seen = end;
    return SOPRO_OK;
  }
};

// The state of every streaming stage; a stage's state derives from it.  A stage with device buffers of its own hides
// alloc_own / free_own.
struct ChunkStream {
  long long max_chunk = 0;
  const char* unset = nullptr;  // what the first reset supplies ("speed", "key") until it has run; null after
  bool finished = false;
  Tail tail;  // its device is the state's

  cudaError_t alloc_own() { return cudaSuccess; }
  void free_own() {}
  // a new utterance whose tail starts at `base`
  void restart(long long base) {
    unset = nullptr;
    finished = false;
    tail.restart(base);
  }
};

// before a create touches the device: somewhere to put the state (cleared), and max_chunk in range
template <class S>
int check_create(long long max_chunk, S** out) {
  if (!out) return fail(SOPRO_ERR_INVALID, "null argument");
  *out = nullptr;
  if (max_chunk < 1 || max_chunk > (1LL << 32)) return fail(SOPRO_ERR_INVALID, "max_chunk must be in [1, 2^32]");
  return SOPRO_OK;
}

// frees s and everything it allocated, on its device
template <class S>
int destroy(S* s) {
  if (!s) return SOPRO_OK;
  s->tail.release();
  s->free_own();
  delete s;
  return SOPRO_OK;
}

// s on the current device: its tail of cap samples, then its own buffers; a failed allocation destroys s
template <class S>
int create(S* s, long long max_chunk, size_t cap, const char* what, S** out) {
  s->max_chunk = max_chunk;
  cudaError_t e = s->tail.alloc(cap);
  if (e == cudaSuccess) e = s->alloc_own();
  if (e != cudaSuccess) {
    destroy(s);
    return fail(SOPRO_ERR_CUDA, "%s stream state: %s", what, cudaGetErrorString(e));
  }
  *out = s;
  return SOPRO_OK;
}

// stream_ready's precondition: -1 is returned otherwise
inline bool can_run(const ChunkStream* s, long long n_more) { return s && n_more >= 0 && !s->finished && !s->unset; }

// a push of n samples, preconditions 1-4 in order: a handle, reset since created, not finished, n in [0, max_chunk]
inline int check_push(const ChunkStream* s, long long n) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null argument");
  if (s->unset) return fail(SOPRO_ERR_STATE, "push before reset: set the %s first", s->unset);
  if (s->finished) return fail(SOPRO_ERR_STATE, "push after finish: reset the stream first");
  if (n < 0 || n > s->max_chunk) return fail(SOPRO_ERR_INVALID, "push of %lld samples: must be in [0, max_chunk = %lld]", n, s->max_chunk);
  return SOPRO_OK;
}

// finish, preconditions 1-3
inline int check_finish(const ChunkStream* s) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null argument");
  if (s->unset) return fail(SOPRO_ERR_STATE, "finish before reset: set the %s first", s->unset);
  if (s->finished) return fail(SOPRO_ERR_STATE, "finish after finish: reset the stream first");
  return SOPRO_OK;
}

// precondition 5: the pushed samples, and y when the call writes outputs
inline int check_io(const float* x, long long n, const float* y, long long outputs) {
  if ((n > 0 && !x) || (outputs > 0 && !y)) return fail(SOPRO_ERR_INVALID, "null argument");
  return SOPRO_OK;
}

}  // namespace chunk
