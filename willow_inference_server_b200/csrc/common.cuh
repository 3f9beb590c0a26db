// Shared host/device helpers for libwisb200.so
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <stdexcept>
#include <string>

namespace wisb {

constexpr int T_ENC = 1500;      // encoder positions per 30-s window
constexpr int T_ENC_PAD = 1536;  // rows per window in every encoder activation (12 x 128)
constexpr int N_FRAMES = 3000;
constexpr int N_SAMPLES = 480000;
constexpr int HEAD_DIM = 64;
constexpr int H1_ROWS = 2 * T_ENC_PAD;  // conv1 output rows per window: 1 zero row + 3000 frames + zero tail

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define WISB_CUDA(expr)                                                                                   \
  do {                                                                                                    \
    cudaError_t _e = (expr);                                                                              \
    if (_e != cudaSuccess)                                                                                \
      throw ::wisb::Error(2, std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " (" + __FILE__ + \
                                 ":" + std::to_string(__LINE__) + ")");                                   \
  } while (0)

#define WISB_REQUIRE(cond, msg)                       \
  do {                                                \
    if (!(cond)) throw ::wisb::Error(1, std::string(msg)); \
  } while (0)

// Function attributes (dynamic shared memory size ...) belong to a device's context: a process that drives several GPUs
// (ctranslate2-style device_index=[0..N-1] replicas, main.py:295,346) must set them once PER DEVICE.
// `done` is a per-call-site bit mask of devices already configured (a benign race sets an attribute twice).
template <typename F>
inline void once_per_device(std::atomic<unsigned long long>& done, F&& f) {
  int dev = 0;
  WISB_CUDA(cudaGetDevice(&dev));
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(done.load(std::memory_order_acquire) & bit)) {
    f();
    done.fetch_or(bit, std::memory_order_release);
  }
}

inline int cdiv(int a, int b) { return (a + b - 1) / b; }
inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline int round_up(int a, int b) { return cdiv(a, b) * b; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// exact (erf) GELU, as torch.nn.functional.gelu default / [HF] ACT2FN["gelu"]
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

}  // namespace wisb
