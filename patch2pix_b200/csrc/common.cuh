// Shared helpers for the patch2pix_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>

namespace p2p {

// ---- error plumbing (no exceptions cross the C ABI) -------------------------------------------
void set_last_error(const std::string& msg);

#define P2P_CUDA_OK(expr)                                                                      \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      ::p2p::set_last_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " at " +      \
                            __FILE__ + ":" + std::to_string(__LINE__));                        \
      return -2;                                                                               \
    }                                                                                          \
  } while (0)

#define P2P_REQUIRE(cond, msg)                                                                 \
  do {                                                                                         \
    if (!(cond)) {                                                                             \
      ::p2p::set_last_error(std::string("invalid argument: ") + (msg) + " [" #cond "]");       \
      return -1;                                                                               \
    }                                                                                          \
  } while (0)

extern long long g_launch_count;  // kernels enqueued by this library (bench.py's gpu_launches)
#define P2P_LAUNCH_OK()                \
  do {                                 \
    ++::p2p::g_launch_count;           \
    P2P_CUDA_OK(cudaGetLastError());   \
  } while (0)

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) only when this kernel on this device has not been granted at least
// `bytes` yet (the attribute is sticky; setting it on every launch costs a driver call per kernel per pair).
int ensure_dyn_smem(const void* kernel, int bytes);
#define P2P_ENSURE_SMEM(kern, bytes)                                            \
  do {                                                                          \
    int _rc = ::p2p::ensure_dyn_smem(reinterpret_cast<const void*>(kern), (int)(bytes)); \
    if (_rc) return _rc;                                                        \
  } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ---- device helpers -----------------------------------------------------------------------------
// Order-preserving float <-> uint32 map so that atomicMax works on signed floats.
__device__ __forceinline__ unsigned int f2ord(float f) {
  unsigned int b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned int u) {
  unsigned int b = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
  return __uint_as_float(b);
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Bump allocator over one scratch block: each take is padded and 256-byte aligned.
struct Carve {
  char* p;
  template <typename T>
  T* take(size_t n) {
    T* r = (T*)p;
    p += align_up(n * sizeof(T) + 16, 256);
    return r;
  }
};

// Grow-only device scratch arena owned by a handle.  Growth is a (synchronising)
// cudaMalloc; after the first pair of a given shape the arena is stable.
struct Arena {
  char* base = nullptr;
  size_t cap = 0;
  size_t off = 0;
  int reserve(size_t bytes);  // ensure capacity (may free + malloc); resets offset
  void reset() { off = 0; }
  void* take(size_t bytes) {
    size_t o = align_up(off, 1024);
    if (o + bytes > cap) return nullptr;
    off = o + bytes;
    return base + o;
  }
  void release();
};

}  // namespace p2p
