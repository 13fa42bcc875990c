// Shared host-side helpers for libscannet_b200.so: thread-local error text, CUDA status checks, scoped owners of CUDA
// resources.
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

#include "../../include/scannet_b200.h"

namespace scn {

std::string& last_error_ref();
int fail(int code, const char* fmt, ...);

}  // namespace scn

#ifdef __CUDACC__
#include <cuda_runtime.h>

#include <memory>
#include <utility>

#define SCN_CUDA_TRY(expr)                                                                   \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess)                                                                   \
      return scn::fail(SCN_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                       __FILE__, __LINE__);                                                  \
  } while (0)

namespace scn {

// cudaMalloc with scope lifetime.  alloc() frees the old block first, and a zero-byte request still gets a block; a failed
// alloc() leaves the buffer empty and clears the error.
struct DBuf {
  void* p = nullptr;
  DBuf() = default;
  DBuf(const DBuf&) = delete;
  DBuf& operator=(const DBuf&) = delete;
  ~DBuf() { reset(); }
  template <typename T> T* as() const { return (T*)p; }
  void reset() { if (p) cudaFree(p); p = nullptr; }
  bool alloc(size_t bytes) { reset(); if (cudaMalloc(&p, bytes ? bytes : 4) == cudaSuccess) return true; p = nullptr; cudaGetLastError(); return false; }
  void swap(DBuf& o) { std::swap(p, o.p); }
};
#define SCN_ALLOC(buf, bytes) do { if (!(buf).alloc(bytes)) return scn::fail(SCN_ERR_CUDA, "cudaMalloc(%zu) failed (%s:%d)", (size_t)(bytes), __FILE__, __LINE__); } while (0)

// Host-side owners: std::unique_ptr with the matching release call.  A malloc'd result is handed to the caller with release().
template <auto fn> struct Release { template <class P> void operator()(P p) const { fn(p); } };
template <class T> using PinnedPtr = std::unique_ptr<T[], Release<cudaFreeHost>>;
template <class T> using MallocPtr = std::unique_ptr<T[], Release<free>>;
using EventPtr = std::unique_ptr<CUevent_st, Release<cudaEventDestroy>>;
using StreamPtr = std::unique_ptr<CUstream_st, Release<cudaStreamDestroy>>;

// create(owner, ...) makes the resource and hands it to the owner; it returns the CUDA status
template <class T> cudaError_t create(PinnedPtr<T>& p, size_t bytes) {
  void* x = nullptr; const cudaError_t e = cudaHostAlloc(&x, bytes, cudaHostAllocDefault); p.reset(e ? nullptr : (T*)x); return e;
}
inline cudaError_t create(EventPtr& ev, unsigned flags = cudaEventDefault) {
  cudaEvent_t x = nullptr; const cudaError_t e = cudaEventCreateWithFlags(&x, flags); ev.reset(e ? nullptr : x); return e;
}
inline cudaError_t create(StreamPtr& st, EventPtr* ev, int n_ev) {              // a non-blocking stream and its timing events
  cudaStream_t x = nullptr; cudaError_t e = cudaStreamCreateWithFlags(&x, cudaStreamNonBlocking); st.reset(e ? nullptr : x);
  for (int i = 0; i < n_ev && !e; ++i) e = create(ev[i]);
  return e;
}

inline unsigned grid_for(size_t n) { return (unsigned)((n + 255) / 256); }

}  // namespace scn
#endif
