// Shared device/host helpers for the vil_attn kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include "../../include/vil_attn.h"

namespace vil {

// Geometry + mode of one call, passed by value to every kernel.
// Mirrors the quantities of Long2DSCSelfAttention.forward (longformer2d.py:107-149):
// padx/pady (:138), mx/my (:139-140), the chunk offsets visited for `mode`
// (slidingchunk_2d.py:15-24, 37-79).
struct Geo {
  int B, H, D;
  int nx, ny, w, g, exact, mode;
  int padx, pady, mx, my;
  int Nloc, N, w2;
  int npc;              // 64-row pieces per chunk = ceil(w2 / 64)
  int noffs;            // number of chunk offsets visited
  int offR[9], offC[9]; // (chunk-row, chunk-col) offsets, reference column order
  int has_bias;
  float scale;
};

// backward workspace layout (floats): [delta (B*H*Nloc)] [delta_g (B*H*g)]
inline long long ws_off_delta_g(const Geo& g) { return ((long long)g.B * g.H * g.Nloc + 63) & ~63LL; }
inline long long ws_floats(const Geo& g) { return ws_off_delta_g(g) + (((long long)g.B * g.H * g.g + 63) & ~63LL); }

struct T4 {             // device view (B,H,T,D), unit stride on D
  char* p;
  long long sb, sh, st;
};

template <typename T> struct ElemTraits;
template <> struct ElemTraits<float> {
  static __device__ __forceinline__ float to_f(float x) { return x; }
  static __device__ __forceinline__ float from_f(float x) { return x; }
};
template <> struct ElemTraits<__nv_bfloat16> {
  static __device__ __forceinline__ float to_f(__nv_bfloat16 x) { return __bfloat162float(x); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float x) { return __float2bfloat16_rn(x); }
};
template <> struct ElemTraits<__half> {
  static __device__ __forceinline__ float to_f(__half x) { return __half2float(x); }
  static __device__ __forceinline__ __half from_f(float x) { return __float2half_rn(x); }
};

template <typename T>
__device__ __forceinline__ const T* row_ptr(const T4& t, int b, int h, long long tok) {
  return reinterpret_cast<const T*>(t.p) + (long long)b * t.sb + (long long)h * t.sh + tok * t.st;
}
template <typename T>
__device__ __forceinline__ T* row_ptr_w(const T4& t, int b, int h, long long tok) {
  return reinterpret_cast<T*>(t.p) + (long long)b * t.sb + (long long)h * t.sh + tok * t.st;
}

// Load `CNT` consecutive elements of a row starting at column c0 into fp32 registers;
// columns >= D read as zero.  Vectorised (16-byte) when the row segment is aligned and full.
template <typename T, int CNT>
__device__ __forceinline__ void load_seg(const T* __restrict__ row, int c0, int D, float (&r)[CNT]) {
  constexpr int PER16 = 16 / (int)sizeof(T);
  if constexpr (CNT % PER16 == 0) {
    if (c0 + CNT <= D && ((reinterpret_cast<uintptr_t>(row + c0)) & 15) == 0) {
#pragma unroll
      for (int v = 0; v < CNT / PER16; ++v) {
        int4 raw = __ldg(reinterpret_cast<const int4*>(row + c0) + v);
        const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
        for (int u = 0; u < PER16; ++u) r[v * PER16 + u] = ElemTraits<T>::to_f(e[u]);
      }
      return;
    }
  }
#pragma unroll
  for (int c = 0; c < CNT; ++c) r[c] = (c0 + c < D) ? ElemTraits<T>::to_f(row[c0 + c]) : 0.f;
}

template <typename T, int CNT>
__device__ __forceinline__ void store_seg(T* __restrict__ row, int c0, int D, const float (&r)[CNT]) {
  constexpr int PER16 = 16 / (int)sizeof(T);
  if constexpr (CNT % PER16 == 0) {
    if (c0 + CNT <= D && ((reinterpret_cast<uintptr_t>(row + c0)) & 15) == 0) {
#pragma unroll
      for (int v = 0; v < CNT / PER16; ++v) {
        int4 raw;
        T* e = reinterpret_cast<T*>(&raw);
#pragma unroll
        for (int u = 0; u < PER16; ++u) e[u] = ElemTraits<T>::from_f(r[v * PER16 + u]);
        reinterpret_cast<int4*>(row + c0)[v] = raw;
      }
      return;
    }
  }
#pragma unroll
  for (int c = 0; c < CNT; ++c)
    if (c0 + c < D) row[c0 + c] = ElemTraits<T>::from_f(r[c]);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace vil
