// libb200tts.so -- host-side plumbing shared by the C-ABI translation units (include/b200tts.h): status codes and error text,
// RAII device / pinned buffers, device switching, weight-tensor lookup and packing.  No kernels.
#pragma once
#include "../../include/b200tts.h"

#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"

namespace b200tts {

// The text b200tts_last_error returns: set by every entry point that fails, per calling thread (defined in api.cu).
extern thread_local std::string g_err;

#define API_BEGIN try {
#define API_END                                       \
  }                                                   \
  catch (const ::b200tts::Error& e) {                 \
    ::b200tts::g_err = e.what();                      \
    return e.code;                                    \
  }                                                   \
  catch (const std::bad_alloc&) {                     \
    ::b200tts::g_err = "host allocation failed";      \
    return B200TTS_ENOMEM;                            \
  }                                                   \
  catch (const std::exception& e) {                   \
    ::b200tts::g_err = e.what();                      \
    return B200TTS_EINVAL;                            \
  }                                                   \
  return B200TTS_OK;

#define REQUIRE(cond, code, msg)                                 \
  do {                                                           \
    if (!(cond)) throw ::b200tts::Error((code), std::string(msg)); \
  } while (0)

// Device memory that grows on demand and is freed with its owner.  release() frees it early.
struct DeviceBuf {
  void* p = nullptr;
  size_t bytes = 0;
  DeviceBuf() = default;
  DeviceBuf(const DeviceBuf&) = delete;
  DeviceBuf& operator=(const DeviceBuf&) = delete;
  ~DeviceBuf() { release(); }
  void ensure(size_t n) {
    if (n <= bytes) return;
    if (p) B200_CUDA(cudaFree(p));
    p = nullptr;
    bytes = 0;
    cudaError_t e = cudaMalloc(&p, n);
    if (e != cudaSuccess) {
      p = nullptr;
      throw Error(B200TTS_ENOMEM, std::string("cudaMalloc(") + std::to_string(n) + "): " + cudaGetErrorString(e));
    }
    bytes = n;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

// Page-locked host memory, same ownership as DeviceBuf.
struct HostPinned {
  void* p = nullptr;
  size_t bytes = 0;
  HostPinned() = default;
  HostPinned(const HostPinned&) = delete;
  HostPinned& operator=(const HostPinned&) = delete;
  ~HostPinned() { release(); }
  void ensure(size_t n) {
    if (n <= bytes) return;
    if (p) cudaFreeHost(p);
    p = nullptr;
    bytes = 0;
    cudaError_t e = cudaMallocHost(&p, n);
    if (e != cudaSuccess) {
      p = nullptr;
      throw Error(B200TTS_ENOMEM, std::string("cudaMallocHost: ") + cudaGetErrorString(e));
    }
    bytes = n;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    bytes = 0;
  }
};

// Makes `dev` current for the guard's lifetime.  The throwing form is for entry points that return a status; the non-throwing
// one (nothrow = true) is for the *_destroy functions, which free a context's memory on the device it was allocated on.
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev, bool nothrow = false) {
    if (nothrow) {
      if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
      cudaSetDevice(dev);
      return;
    }
    B200_CUDA(cudaGetDevice(&prev));
    if (prev != dev) B200_CUDA(cudaSetDevice(dev));
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// The device argument of a *_create names an existing CUDA device.
inline void check_device(int device) {
  int ndev = 0;
  B200_CUDA(cudaGetDeviceCount(&ndev));
  REQUIRE(device >= 0 && device < ndev, B200TTS_EINVAL, "no such CUDA device");
}

using TensorMap = std::map<std::string, const b200tts_tensor*>;

inline const b200tts_tensor* need(const TensorMap& m, const std::string& name, std::initializer_list<int64_t> shape) {
  auto it = m.find(name);
  if (it == m.end()) throw Error(B200TTS_EMISSING, "missing weight tensor '" + name + "'");
  const b200tts_tensor* t = it->second;
  size_t nd = shape.size();
  bool ok = (size_t)t->ndim == nd && t->data != nullptr;
  size_t i = 0;
  for (int64_t s : shape) {
    if (ok && t->shape[i] != s) ok = false;
    ++i;
  }
  if (!ok) {
    std::string got = "[";
    for (int k = 0; k < t->ndim && k < 4; ++k) got += (k ? "," : "") + std::to_string(t->shape[k]);
    got += "]";
    std::string want = "[";
    i = 0;
    for (int64_t s : shape) want += (i++ ? "," : "") + std::to_string(s);
    want += "]";
    throw Error(B200TTS_ESHAPE, "weight '" + name + "' has shape " + got + ", expected " + want);
  }
  return t;
}

// Host-side staging of one packed fp32 blob; every sub-array starts 16-byte aligned.
struct Packer {
  std::vector<float> h;
  size_t add(size_t n) {
    size_t off = (h.size() + 3) & ~size_t(3);
    h.resize(off + n, 0.f);
    return off;
  }
  // appends weight tensor `name`, which must have `shape`, as it is; returns its offset
  size_t copy(const TensorMap& tm, const std::string& name, std::initializer_list<int64_t> shape) {
    const b200tts_tensor* t = need(tm, name, shape);
    size_t n = 1;
    for (int64_t s : shape) n *= (size_t)s;
    size_t off = add(n);
    std::memcpy(&h[off], t->data, n * sizeof(float));
    return off;
  }
};

inline int round4(int x) { return (x + 3) & ~3; }

// push_init_kernel (wavernn_push.cuh, compiled in wavernn.cu): fills `nvec` words of a flag-in-data exchange buffer with the
// sentinel, clears `nbest` winner words and the error flag if `error` is not null.  The Tacotron grid decoder arms its exchange
// buffers with it too.
void launch_push_init(uint32_t* vec, size_t nvec, unsigned long long* best, size_t nbest, int* error, int grid, cudaStream_t st);

}  // namespace b200tts
