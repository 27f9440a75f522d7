// Shared helpers for libcotb200 (sm_90a).  Host-side error plumbing + device-side element traits.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include <type_traits>

#include "../../include/cotb200.h"

namespace cotb200 {

// ---------------------------------------------------------------- host: errors + launch accounting
void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return (int)e;
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

// Optional per-launch timing (cotb200_prof_enable): CUDA events recorded on the launch stream around each kernel.
// Disabled by default (zero overhead beyond one relaxed atomic load); never enable under graph capture.
struct ProfScope {
  const char* name; cudaStream_t st; cudaEvent_t e0; bool on; double bytes;
  ProfScope(const char* n, cudaStream_t s, double algorithmic_bytes = 0.0);
  ~ProfScope();
};
// `bytes` = ALGORITHMIC bytes of the launch (DESIGN.md section 4): what the kernel must move, not what it happened to.
#define COTB200_PROF(name) cotb200::ProfScope _prof_scope(name, st)
#define COTB200_PROF_B(name, bytes) cotb200::ProfScope _prof_scope(name, st, (double)(bytes))

// Per-device memo slots: a process may drive several GPUs (the reference memoises its kernels per device too,
// cupy_layers/utils.py:14), so nothing that depends on the device is cached in a plain static.
inline int cur_dev_slot() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev & 63;
}
struct PerDevFlag {
  bool v[64] = {};
  bool& get() { return v[cur_dev_slot()]; }
};
inline int num_sms() {
  static int sms[64] = {};
  int& s = sms[cur_dev_slot()];
  if (!s) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&s, cudaDevAttrMultiProcessorCount, dev);
    if (s <= 0) s = 132;
  }
  return s;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ---------------------------------------------------------------- device: element traits
template <typename T> struct Elem;
template <> struct Elem<float> {
  using Acc = float;
  __device__ __forceinline__ static float ld(const float* p) { return __ldg(p); }
  __device__ __forceinline__ static float from(float a) { return a; }
};
template <> struct Elem<double> {
  using Acc = double;
  __device__ __forceinline__ static double ld(const double* p) { return __ldg(p); }
  __device__ __forceinline__ static double from(double a) { return a; }
};
template <> struct Elem<__nv_bfloat16> {
  using Acc = float;
  __device__ __forceinline__ static float ld(const __nv_bfloat16* p) {
    return __bfloat162float(__ldg(p));
  }
  __device__ __forceinline__ static __nv_bfloat16 from(float a) { return __float2bfloat16_rn(a); }
};
template <> struct Elem<__half> {
  using Acc = float;
  __device__ __forceinline__ static float ld(const __half* p) { return __half2float(__ldg(p)); }
  __device__ __forceinline__ static __half from(float a) { return __float2half_rn(a); }
};

// A VEC-wide packet of T moved with one load/store instruction (VEC*sizeof(T) <= 16 bytes).
template <typename T, int VEC> struct alignas(sizeof(T) * VEC) Pack { T v[VEC]; };

template <typename T, int VEC>
__device__ __forceinline__ Pack<T, VEC> ld_pack(const T* p) {
  Pack<T, VEC> r;
  constexpr int B = sizeof(T) * VEC;
  if constexpr (B == 16) {
    uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
    r = *reinterpret_cast<Pack<T, VEC>*>(&u);
  } else if constexpr (B == 8) {
    uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
    r = *reinterpret_cast<Pack<T, VEC>*>(&u);
  } else if constexpr (B == 4) {
    unsigned u = __ldg(reinterpret_cast<const unsigned*>(p));
    r = *reinterpret_cast<Pack<T, VEC>*>(&u);
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) r.v[i] = __ldg(p + i);
  }
  return r;
}

template <typename T, int VEC>
__device__ __forceinline__ void st_pack(T* p, const Pack<T, VEC>& r) {
  constexpr int B = sizeof(T) * VEC;
  if constexpr (B == 16) {
    *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(&r);
  } else if constexpr (B == 8) {
    *reinterpret_cast<uint2*>(p) = *reinterpret_cast<const uint2*>(&r);
  } else if constexpr (B == 4) {
    *reinterpret_cast<unsigned*>(p) = *reinterpret_cast<const unsigned*>(&r);
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) p[i] = r.v[i];
  }
}

template <typename T> __device__ __forceinline__ typename Elem<T>::Acc to_acc(T v);
template <> __device__ __forceinline__ float to_acc<float>(float v) { return v; }
template <> __device__ __forceinline__ double to_acc<double>(double v) { return v; }
template <> __device__ __forceinline__ float to_acc<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_acc<__half>(__half v) { return __half2float(v); }

// d = a*b + c with 16-bit a, b widened to fp32 and one fp32 FMA.  The product of two bf16 (or two fp16) values is exact in
// fp32, so this is the single-rounding a*b + c.  (sm_90 has no mixed-precision fma.f32.bf16.)
template <typename T> __device__ __forceinline__ float mfma(T a, T b, float c);
template <> __device__ __forceinline__ float mfma<float>(float a, float b, float c) { return fmaf(a, b, c); }
template <> __device__ __forceinline__ float mfma<__nv_bfloat16>(__nv_bfloat16 a, __nv_bfloat16 b, float c) {
  return fmaf(__bfloat162float(a), __bfloat162float(b), c);
}
template <> __device__ __forceinline__ float mfma<__half>(__half a, __half b, float c) {
  return fmaf(__half2float(a), __half2float(b), c);
}
template <typename T> __device__ __forceinline__ T one_of();
template <> __device__ __forceinline__ float one_of<float>() { return 1.f; }
template <> __device__ __forceinline__ __nv_bfloat16 one_of<__nv_bfloat16>() { return __ushort_as_bfloat16((unsigned short)0x3F80); }
template <> __device__ __forceinline__ __half one_of<__half>() { return __ushort_as_half((unsigned short)0x3C00); }

// ---------------------------------------------------------------- deterministic cross-CTA sums
// Floating-point atomics add the partial sums of the CTAs in the order the CTAs happen to finish, so such a sum changes from run
// to run in its last bits, and a training run amplifies that into different weights.  Instead every CTA of a group stores its
// partials to its own row of a scratch area and the LAST CTA of the group to arrive (ticket counters) adds the rows in row order.
// The scratch of a launch is stream-ordered: DetScratch allocates it with cudaMallocAsync and zeroes its tickets with
// cudaMemsetAsync on the launch's stream, and frees it with cudaFreeAsync on that stream after the launch (under graph capture
// these become the graph's own allocation / memset / free nodes).  Launches on different streams never share scratch.
struct DetArena { float* scr; unsigned* tick; };
static constexpr int DET_TICKETS_PER_GROUP = 64;   // one reduction = 1 final ticket + up to 63 first-level tickets

struct DetScratch {
  DetArena a{nullptr, nullptr};
  void* base = nullptr;
  cudaStream_t st = nullptr;
  // `floats` of scratch and `groups` independent reductions' tickets, on stream s
  int alloc(size_t floats, int groups, cudaStream_t s) {
    st = s;
    const size_t tick_bytes = ((size_t)groups * DET_TICKETS_PER_GROUP * sizeof(unsigned) + 255) & ~(size_t)255;
    cudaError_t e = cudaMallocAsync(&base, tick_bytes + floats * sizeof(float), st);
    if (e == cudaSuccess && tick_bytes) e = cudaMemsetAsync(base, 0, tick_bytes, st);
    if (e != cudaSuccess) { set_error("reduction scratch (%zu floats): %s", floats, cudaGetErrorString(e)); return (int)e; }
    a.tick = (unsigned*)base;
    a.scr = (float*)((char*)base + tick_bytes);
    return 0;
  }
  ~DetScratch() { if (base) cudaFreeAsync(base, st); }
};

// Two levels keep the serial tail short: the rows are added in fixed blocks of `fan` rows by the last CTA of each block, the
// block totals by the last block.  Everything about the order is a function of nslots only.
__host__ __device__ __forceinline__ int det_fan(int nslots) {
  const int f = (nslots + DET_TICKETS_PER_GROUP - 2) / (DET_TICKETS_PER_GROUP - 1);
  return f < 16 ? 16 : f;
}
__host__ __device__ __forceinline__ int det_blocks(int nslots) { return (nslots + det_fan(nslots) - 1) / det_fan(nslots); }
// floats of scratch one reduction of nslots rows of n values uses (its rows + the block totals)
__host__ __device__ __forceinline__ size_t det_floats(int nslots, int n) { return (size_t)(nslots + det_blocks(nslots)) * n; }

template <bool NAMED>
__device__ __forceinline__ void det_bar(int nthr) {
  if constexpr (NAMED) asm volatile("bar.sync 1, %0;" ::"r"(nthr) : "memory");
  else __syncthreads();
}

// Adds rows [j0, j1) of scr (row pitch n) in row order, element k: four independent chains j = j0 + 4i + q added as ((0+1)+(2+3)).
__device__ __forceinline__ float det_sum_rows(const float* scr, int n, int j0, int j1, int k) {
  float t[4] = {0.f, 0.f, 0.f, 0.f};
  int j = j0;
  for (; j + 3 < j1; j += 4) {
#pragma unroll
    for (int q = 0; q < 4; ++q) t[q] += __ldcg(scr + (size_t)(j + q) * n + k);
  }
  for (int q = 0; j < j1; ++j, ++q) t[q] += __ldcg(scr + (size_t)j * n + k);
  return (t[0] + t[1]) + (t[2] + t[3]);
}

// scr: the reduction's det_floats(nslots, n) area, rows [0, nslots) = one per CTA; ticket: its DET_TICKETS_PER_GROUP counters,
// zeroed by DetScratch.  Every participating thread (tid < nthr; NAMED: barrier 1 instead of __syncthreads) calls this after
// the CTA stored its own row `slot`.  add(k, total) runs in exactly one CTA with the run-to-run identical total of element k.
template <bool NAMED = false, class F>
__device__ __forceinline__ void det_finish(float* scr, int n, int slot, int nslots, unsigned* ticket, int tid, int nthr, F add) {
  __shared__ unsigned s_det_last;
  const int fan = det_fan(nslots), nblk = det_blocks(nslots), blk = slot / fan;
  const int j0 = blk * fan, j1 = min(nslots, j0 + fan);
  float* btot = scr + (size_t)nslots * n;
  __threadfence();
  det_bar<NAMED>(nthr);
  if (tid == 0) s_det_last = atomicAdd(ticket + 1 + blk, 1u) == (unsigned)(j1 - j0 - 1) ? 1u : 0u;
  det_bar<NAMED>(nthr);
  if (!s_det_last) return;
  __threadfence();
  for (int k = tid; k < n; k += nthr) btot[(size_t)blk * n + k] = det_sum_rows(scr, n, j0, j1, k);
  __threadfence();
  det_bar<NAMED>(nthr);
  if (tid == 0) s_det_last = atomicAdd(ticket, 1u) == (unsigned)(nblk - 1) ? 1u : 0u;
  det_bar<NAMED>(nthr);
  if (!s_det_last) return;
  __threadfence();
  for (int k = tid; k < n; k += nthr) add(k, det_sum_rows(btot, n, 0, nblk, k));
}

// dtype dispatch on the host
#define COTB200_DISPATCH_DTYPE(dtype, ...)                                   \
  switch (dtype) {                                                           \
    case COTB200_F32:  { using T = float;          __VA_ARGS__; } break;     \
    case COTB200_F64:  { using T = double;         __VA_ARGS__; } break;     \
    case COTB200_BF16: { using T = __nv_bfloat16;  __VA_ARGS__; } break;     \
    case COTB200_F16:  { using T = __half;         __VA_ARGS__; } break;     \
    default: cotb200::set_error("unknown dtype %d", (int)(dtype)); return COTB200_EDTYPE; \
  }

}  // namespace cotb200
