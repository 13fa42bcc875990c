// Shared host-side helpers for libscannet_b200.so: thread-local error text, CUDA status checks, scoped owners of CUDA
// resources and of the C-ABI handles, and the .sens frame helpers the scene drivers share.
#pragma once
#include <chrono>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/scannet_b200.h"

namespace scn {

std::string& last_error_ref();
int fail(int code, const char* fmt, ...);

inline double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// Host-side owners: std::unique_ptr with the matching release call.  A malloc'd result is handed to the caller with release();
// the arrays the library hands out are released with MallocPtr, as scn_free is free.
template <auto fn> struct Release { template <class P> void operator()(P p) const { fn(p); } };
template <class T> using MallocPtr = std::unique_ptr<T[], Release<free>>;
template <class T> using PinnedPtr = std::unique_ptr<T[], Release<scn_host_free>>;
template <class T> using DevicePtr = std::unique_ptr<T[], Release<scn_device_free>>;
using SensPtr = std::unique_ptr<scn_sens, Release<scn_sens_close>>;
using FreespacePtr = std::unique_ptr<scn_freespace, Release<scn_freespace_destroy>>;
using HandleStreamPtr = std::unique_ptr<void, Release<scn_stream_destroy>>;        // a scn_stream_create stream
inline int create(HandleStreamPtr& st) { void* x = nullptr; const int rc = scn_stream_create(&x); st.reset(x); return rc; }

// .sens helpers of the scene drivers (sens.cpp, inflate.cu)
struct PosedFrames { std::vector<uint64_t> frames; std::vector<float> poses; };     // poses: 16 floats per frame
// The frames of [f0, f1) that have a pose, with their poses (a frame without one is never decoded: sensorData.h:382).
int posed_frames(const scn_sens* s, uint64_t f0, uint64_t f1, PosedFrames& out);
// Decodes the colour of `frame` into `scratch` (color_width x color_height RGB8) and registers it to the depth image:
// out[p] = scratch[lut[p]], black where lut[p] < 0, for the n_px depth pixels.
// Colour pixel for every depth pixel (row-major, -1 = outside the colour image): K_c * K_d^-1 * (x, y, 1), nearest
// (sensorData.h:1577-1586 with identity extrinsics).
void build_color_lut(const scn_sens_info_t& in, std::vector<int32_t>& lut);
int sens_color_to_depth(const scn_sens* s, uint64_t frame, const int32_t* lut, size_t n_px, uint8_t* scratch, uint8_t* out);
// The depth of frames[0..n) into device memory, frame after frame (u16, row-major): zlib streams through the GPU inflate, raw
// frames uploaded.  Returns when the frames are on the device.
int sens_depth_to_device(const scn_sens* s, const uint64_t* frames, uint32_t n, uint16_t* d_out, void* stream);
// scn_fuse_scene on a stream that is already open, with the poses it holds in memory (fuse.cpp); label names it in errors
int fuse_sens(const scn_sens* s, const char* label, const char* out_ply, const scn_tsdf_params* params, int device, scn_fuse_report_t* report);

}  // namespace scn

#ifdef __CUDACC__
#include <cuda_runtime.h>

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
