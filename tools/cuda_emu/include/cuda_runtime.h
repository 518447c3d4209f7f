// TEST TOOLING — NOT PRODUCT CODE. A tiny CUDA-on-CPU shim that lets the *unmodified* kernel and host sources of
// khronos_b200/csrc be compiled with g++ into libkhronos_b200_emu.so (tools/cuda_emu/build_emu.py), so that the kernels'
// logic can be checked against the oracle in a container without a GPU. It shadows <cuda_runtime.h> for that build
// only. Semantics: one OS thread; every CUDA thread of a block is a fiber (ucontext); fibers yield at warp / block
// synchronising intrinsics and are resumed when all active lanes (threads) have arrived; blocks run one after the
// other, so atomics are plain read-modify-writes and `__shared__` is a function-local static. Nothing about timing,
// memory spaces, races or sm_90a code generation is modelled. The product never loads this library.
#pragma once
#define __CUDACC__ 1
#define KB_CUDA_EMU 1

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <functional>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __grid_constant__
#define __shared__ static

struct uint3 { unsigned x, y, z; };
struct dim3 {
  unsigned x = 1, y = 1, z = 1;
  dim3() = default;
  dim3(unsigned x_, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
  dim3(int x_, int y_ = 1, int z_ = 1) : x(static_cast<unsigned>(x_)), y(static_cast<unsigned>(y_)), z(static_cast<unsigned>(z_)) {}
  dim3(size_t x_) : x(static_cast<unsigned>(x_)) {}
};
struct float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct int3 { int x, y, z; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct uchar3 { unsigned char x, y, z; };
struct alignas(4) uchar4 { unsigned char x, y, z, w; };
inline float2 make_float2(float x, float y) { return {x, y}; }
inline float4 make_float4(float x, float y, float z, float w) { return {x, y, z, w}; }
inline int3 make_int3(int x, int y, int z) { return {x, y, z}; }
inline uchar3 make_uchar3(unsigned char x, unsigned char y, unsigned char z) { return {x, y, z}; }
inline uchar4 make_uchar4(unsigned char x, unsigned char y, unsigned char z, unsigned char w) { return {x, y, z, w}; }

extern uint3 threadIdx, blockIdx;
extern dim3 blockDim, gridDim;

// ---- runtime API (device memory == host memory) ----------------------------------------------------------------
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1 };
typedef struct emuStream* cudaStream_t;
typedef struct emuEvent* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
struct cudaDeviceProp { int multiProcessorCount; char name[64]; };

inline cudaError_t cudaGetDeviceCount(int* n) { *n = 8; return cudaSuccess; }  // any rank of a multi-process dry run
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) { p->multiProcessorCount = 2; std::strcpy(p->name, "cuda_emu"); return cudaSuccess; }
template <typename T> cudaError_t cudaMalloc(T** p, size_t n) { *p = static_cast<T*>(std::malloc(n ? n : 1)); return *p ? cudaSuccess : cudaErrorInvalidValue; }
inline cudaError_t cudaFree(void* p) { std::free(p); return cudaSuccess; }
template <typename T> cudaError_t cudaMallocHost(T** p, size_t n) { *p = static_cast<T*>(std::malloc(n ? n : 1)); return cudaSuccess; }
inline cudaError_t cudaFreeHost(void* p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaMemset(void* p, int v, size_t n) { std::memset(p, v, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t = nullptr) { std::memset(p, v, n); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = reinterpret_cast<cudaStream_t>(std::malloc(8)); return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { std::free(s); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = reinterpret_cast<cudaEvent_t>(std::malloc(8)); return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { std::free(e); return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
template <typename F> cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) { *n = 1; return cudaSuccess; }

// ---- device-side built-ins ---------------------------------------------------------------------------------------
inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
inline long long min(long long a, long long b) { return a < b ? a : b; }
inline long long max(long long a, long long b) { return a > b ? a : b; }
template <typename T> inline T __ldg(const T* p) { return *p; }
inline int __ffs(unsigned v) { return __builtin_ffs(static_cast<int>(v)); }
inline int __ffs(int v) { return __builtin_ffs(v); }
inline int __popc(unsigned v) { return __builtin_popcount(v); }

template <typename T> inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
inline int atomicSub(int* p, int v) { int o = *p; *p = o - v; return o; }
template <typename T> inline T atomicExch(T* p, T v) { T o = *p; *p = v; return o; }
template <typename T> inline T atomicOr(T* p, T v) { T o = *p; *p = o | v; return o; }
template <typename T> inline T atomicCAS(T* p, T c, T v) { T o = *p; if (o == c) *p = v; return o; }
template <typename T> inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }

namespace emu {
void launch_(std::function<void()> body, dim3 grid, dim3 block, size_t smem = 0, cudaStream_t s = nullptr);
void* dyn_smem();
unsigned long long warp_exchange(unsigned long long v, int src_lane, int mode, int arg);  // see emu_runtime.cpp
int block_reduce(int v, int mode);
void block_barrier();
unsigned active_mask();
template <typename T> inline unsigned long long pack(T v) { unsigned long long r = 0; std::memcpy(&r, &v, sizeof(T)); return r; }
template <typename T> inline T unpack(unsigned long long r) { T v; std::memcpy(&v, &r, sizeof(T)); return v; }
enum { kShfl = 0, kShflXor = 1, kShflUp = 2, kBallot = 3, kAny = 4 };
}  // namespace emu

inline void __syncthreads() { emu::block_barrier(); }
inline int __syncthreads_and(int v) { return emu::block_reduce(v, 0); }
inline int __syncthreads_or(int v) { return emu::block_reduce(v, 1); }
inline unsigned __activemask() { return emu::active_mask(); }
template <typename T> inline T __shfl_sync(unsigned, T v, int src) { return emu::unpack<T>(emu::warp_exchange(emu::pack(v), src, emu::kShfl, 0)); }
template <typename T> inline T __shfl_xor_sync(unsigned, T v, int m) { return emu::unpack<T>(emu::warp_exchange(emu::pack(v), 0, emu::kShflXor, m)); }
template <typename T> inline T __shfl_up_sync(unsigned, T v, unsigned d) { return emu::unpack<T>(emu::warp_exchange(emu::pack(v), 0, emu::kShflUp, static_cast<int>(d))); }
inline unsigned __ballot_sync(unsigned, int pred) { return static_cast<unsigned>(emu::warp_exchange(pred ? 1ull : 0ull, 0, emu::kBallot, 0)); }
inline int __any_sync(unsigned, int pred) { return static_cast<int>(emu::warp_exchange(pred ? 1ull : 0ull, 0, emu::kAny, 0)); }
