// libb200tts.so -- library-wide C entry points: ABI version, last error, device count, and the fp32 peak probe.
#include <algorithm>

#include "api.h"

namespace b200tts {
thread_local std::string g_err;
}  // namespace b200tts

using namespace b200tts;

extern "C" int b200tts_abi_version(void) { return B200TTS_ABI_VERSION; }
extern "C" const char* b200tts_last_error(void) { return g_err.c_str(); }
extern "C" int b200tts_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    g_err = std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e);
    cudaGetLastError();
    return B200TTS_ECUDA;
  }
  return n;
}

// Register-only packed-fp32 FMA loop on every SM: the measured fp32 CUDA-core ceiling bench.py quotes the FLOP form against.
__global__ void fp32_peak_kernel(float* out, int iters) {
  float2 a[8], x = make_float2(1.0001f + threadIdx.x * 1e-7f, 0.9999f), y = make_float2(1e-3f, -1e-3f);
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = make_float2((float)i, (float)(i + 1));
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = fma2_rn(a[i], x, y);
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += a[i].x + a[i].y;
  if (s == 123.456f) out[0] = s;
}
extern "C" int b200tts_debug_fp32_peak(int device, double* tflops) {
  API_BEGIN
  REQUIRE(tflops, B200TTS_EINVAL, "null argument");
  DeviceGuard dg(device);
  int sms = 0;
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  float* d = nullptr;
  B200_CUDA(cudaMalloc(&d, 16));
  cudaEvent_t e0, e1;
  B200_CUDA(cudaEventCreate(&e0));
  B200_CUDA(cudaEventCreate(&e1));
  const int iters = 20000, threads = 512, blocks = sms * 2;
  fp32_peak_kernel<<<blocks, threads>>>(d, 2000);       // warm-up
  double best = 0.0;
  for (int rep = 0; rep < 3; ++rep) {
    B200_CUDA(cudaEventRecord(e0));
    fp32_peak_kernel<<<blocks, threads>>>(d, iters);
    B200_CUDA(cudaEventRecord(e1));
    B200_CUDA(cudaEventSynchronize(e1));
    float ms = 0.f;
    B200_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    const double flop = 2.0 * 2.0 * 32.0 * (double)iters * blocks * threads;   // 32 FFMA2 per iteration, 2 FMAs each
    best = std::max(best, flop / (ms * 1e-3) / 1e12);
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(d);
  *tflops = best;
  API_END
}
