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
  // attention dropout (VilAttnParams::dropout_*): a column is kept iff its Philox word >= drop_thresh, and kept
  // probabilities are scaled by drop_scale = 1 / (1 - p).  Read only by the DROP instantiations of the kernels.
  float drop_p, drop_scale;
  uint32_t drop_thresh;
  uint32_t seed_lo, seed_hi, drop_off;
  // with the bias table: backward pass 1 runs nslice * H * mx * my * npc CTAs, CTA slice s taking the images
  // s, s + nslice, ...; a function of the geometry and the SM count only, so the table partials do not grow with B
  int nslice;
  // dilation (VIL_FLAG_DILATED): 1, or d > 1 for a call run by the DIL instantiations of the local kernels (SubGrid below).
  // The field fills the struct's tail padding, so the kernel parameters after it keep their offsets.
  int d;
};

// Per-image grids (vil_attn_fwd_sized_sm100 / _bwd_sized_sm100): image b's grid of ih x iw tokens, its image_hw entry
// clamped to [1, nx] x [1, ny] so that a bad entry cannot address past the padded grid; without sizes (image_hw == NULL)
// the whole nx x ny grid.
__device__ __forceinline__ void image_extent(const Geo& g, const int* __restrict__ image_hw, int b, int& ih, int& iw) {
  ih = g.nx; iw = g.ny;
  if (image_hw != nullptr) {
    ih = min(max(image_hw[2 * b], 1), g.nx);
    iw = min(max(image_hw[2 * b + 1], 1), g.ny);
  }
}
// local token t (row t / ny, column t % ny of the padded grid) lies on an ih x iw image
__device__ __forceinline__ bool on_image(const Geo& g, int ih, int iw, long long t) { return t / g.ny < ih && t % g.ny < iw; }

// Dilated calls (d > 1) run the operator on each of the d^2 residue sub-grids of the image: residue (a, b) holds the local
// tokens (a + d r, b + d c).  mx / my then count the chunks of a virtual grid of d mx0 x d my0 chunks (mx0 x my0: the chunk
// grid of the largest sub-grid, residue (0, 0)); virtual chunk (R', C') is chunk (R' / d, C' / d) of residue
// (R' % d, C' % d).  Every grid, CTA count and workspace size derived from mx / my thereby covers the d^2 sub-grids, and a
// CTA whose chunk lies outside its (smaller) sub-grid exits.  SubGrid is the geometry a CTA's masks use: its sub-grid's
// tokens, padding and chunk counts, and its residue; undilated, Geo's own.
// The same instantiations (DIL) run calls with per-image grids, dilated or not (d = 1): the sub-grids are then those of
// image b's ih x iw crop (image_extent), while token addresses keep the padded grid's row stride geo.ny (VIL_SUB_*).
template <bool DIL> struct SubGrid;
template <> struct SubGrid<true> {
  int nx_, ny_, padx_, pady_, mx_, my_;
  int r0_, c0_;         // residue (a, b)
  // the residue's sub-grid of image b (image_extent); r0_, c0_ set
  __device__ __forceinline__ void fit(const Geo& g, const int* __restrict__ image_hw, int b) {
    int ih, iw;
    image_extent(g, image_hw, b, ih, iw);
    nx_ = (ih - r0_ + g.d - 1) / g.d;
    ny_ = (iw - c0_ + g.d - 1) / g.d;
    padx_ = (g.w - nx_ % g.w) % g.w;
    pady_ = (g.w - ny_ % g.w) % g.w;
    mx_ = (nx_ + padx_) / g.w;
    my_ = (ny_ + pady_) / g.w;
  }
  __device__ __forceinline__ int nx() const { return nx_; }
  __device__ __forceinline__ int ny() const { return ny_; }
  __device__ __forceinline__ int padx() const { return padx_; }
  __device__ __forceinline__ int pady() const { return pady_; }
  __device__ __forceinline__ int mx() const { return mx_; }
  __device__ __forceinline__ int my() const { return my_; }
  __device__ __forceinline__ int r0() const { return r0_; }
  __device__ __forceinline__ int c0() const { return c0_; }
};
// undilated: Geo's own fields.  The kernels read them through VIL_SG / VIL_SUB_* below, which compile to the direct reads
// of Geo the undilated kernels have always made.
template <> struct SubGrid<false> {
  const Geo& g;
  __device__ __forceinline__ int nx() const { return g.nx; }
  __device__ __forceinline__ int ny() const { return g.ny; }
  __device__ __forceinline__ int padx() const { return g.padx; }
  __device__ __forceinline__ int pady() const { return g.pady; }
  __device__ __forceinline__ int mx() const { return g.mx; }
  __device__ __forceinline__ int my() const { return g.my; }
  __device__ __forceinline__ int r0() const { return 0; }
  __device__ __forceinline__ int c0() const { return 0; }
};

// The CTA's sub-grid in image b; R, C: in the virtual chunk position, out the chunk position in the sub-grid
template <bool DIL>
__device__ __forceinline__ SubGrid<DIL> sub_grid(const Geo& g, int& R, int& C, const int* __restrict__ image_hw, int b) {
  if constexpr (DIL) {
    SubGrid<true> s;
    s.r0_ = R % g.d; R /= g.d;
    s.c0_ = C % g.d; C /= g.d;
    s.fit(g, image_hw, b);
    return s;
  } else {
    return SubGrid<false>{g};
  }
}
// Field f (nx, ny, padx, pady, mx, my) of the sub-grid sg of a kernel or helper with template flag DIL and Geo `geo`.
// Undilated it is geo.f read where it is used, so that those instantiations compile to the code they had before dilation
// (read through SubGrid<false>, the same values compile to differently scheduled code).
#define VIL_SG(f) (DIL ? sg.f() : geo.f)

// a CTA of a dilated or sized call whose chunk lies outside its sub-grid (never one of the plain instantiations)
template <bool DIL>
__device__ __forceinline__ bool off_sub_grid(const SubGrid<DIL>& s, int R, int C) {
  if constexpr (DIL) return R >= s.mx() || C >= s.my();
  else return false;
}

// The one mapping from a sub-grid position (r, c) to the image (tokens (a + d r, b + d c)), in a kernel or helper with
// template flag DIL, Geo `geo` and sub-grid `sg`: the local token (row of q, o, lse, delta, dq), the same as a 32-bit value
// (dropout rows), and the key token (row of k, v, dk, dv, after the g global tokens).  Macros for the reason VIL_SG is
// one: undilated they are the expressions the kernels had before dilation.
#define VIL_SUB_TOK(r, c) \
  (DIL ? (long long)(sg.r0() + geo.d * (r)) * geo.ny + (sg.c0() + geo.d * (c)) : (long long)(r) * geo.ny + (c))
#define VIL_SUB_ROW(r, c) (DIL ? (sg.r0() + geo.d * (r)) * geo.ny + (sg.c0() + geo.d * (c)) : (r) * geo.ny + (c))
#define VIL_SUB_KEY(r, c) \
  (DIL ? geo.g + (long long)(sg.r0() + geo.d * (r)) * geo.ny + (sg.c0() + geo.d * (c)) : geo.g + (long long)(r) * geo.ny + (c))

// backward workspace layout (floats), each part 64-float aligned:
//   [delta (B*H*Nloc)] [delta_g (B*H*g)]
//   with the bias table only: [table partials (nslice*H*mx*my*npc, (4w-1)^2): one row per pass-1 CTA (dilated: of the
//                              virtual chunk grid, a CTA off its sub-grid leaving a row of zeros)]
//                             [global-bias partials: d_g2l[1] (B,H,g) | d_g2l[0] (B,H,g) | d_g2g (B,H,g,g)]
inline long long ws_align(long long n) { return (n + 63) & ~63LL; }
inline long long ws_off_delta_g(const Geo& g) { return ws_align((long long)g.B * g.H * g.Nloc); }
inline int table_entries(const Geo& g) { return (4 * g.w - 1) * (4 * g.w - 1); }
inline long long tab_ctas(const Geo& g) { return (long long)g.nslice * g.H * g.mx * g.my * g.npc; }
inline long long ws_off_tab(const Geo& g) { return ws_off_delta_g(g) + ws_align((long long)g.B * g.H * g.g); }
inline long long ws_off_glob(const Geo& g) { return ws_off_tab(g) + (g.has_bias ? ws_align(tab_ctas(g) * table_entries(g)) : 0); }
inline long long ws_floats(const Geo& g) {
  return ws_off_glob(g) + (g.has_bias && g.g > 0 ? ws_align((long long)g.B * g.H * g.g * (2 + g.g)) : 0);
}

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

// ---------------------------------------------------------------- attention dropout (include/vil_attn.h, "Attention dropout")
// Philox4x32-10 (Salmon et al., SC'11; the Random123 constants) of counter (c0, c1, c2, drop_off) under key (seed_lo, seed_hi)
__device__ __forceinline__ uint4 philox(const Geo& g, uint32_t c0, uint32_t c1, uint32_t c2) {
  uint32_t x0 = c0, x1 = c1, x2 = c2, x3 = g.drop_off, k0 = g.seed_lo, k1 = g.seed_hi;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * x0, hi0 = __umulhi(0xD2511F53u, x0);
    const uint32_t lo1 = 0xCD9E8D57u * x2, hi1 = __umulhi(0xCD9E8D57u, x2);
    x0 = hi1 ^ x1 ^ k0; x1 = lo1; x2 = hi0 ^ x3 ^ k1; x3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(x0, x1, x2, x3);
}
__device__ __forceinline__ uint32_t philox_word(const uint4& x, uint32_t w) {
  return w == 0 ? x.x : w == 1 ? x.y : w == 2 ? x.z : x.w;
}
// Keep bit of one element: row / col are the reference's coordinates, sid = 2 (b H + h) + stream (0: local query rows
// over the columns of attn1, 1: global query rows over the N keys of attn0)
__device__ __forceinline__ bool drop_keep(const Geo& g, uint32_t row, uint32_t col, uint32_t sid) {
  return philox_word(philox(g, col >> 2, row, sid), col & 3) >= g.drop_thresh;
}
// Keep bits of the adjacent columns col, col + 1 of one row: one Philox call unless col is the last word of its counter
__device__ __forceinline__ void drop_keep2(const Geo& g, uint32_t row, uint32_t col, uint32_t sid, bool& k0, bool& k1) {
  const uint4 x = philox(g, col >> 2, row, sid);
  const uint32_t w = col & 3;
  k0 = philox_word(x, w) >= g.drop_thresh;
  const uint32_t u1 = w == 3 ? philox(g, (col >> 2) + 1, row, sid).x : philox_word(x, w + 1);
  k1 = u1 >= g.drop_thresh;
}

// ---------------------------------------------------------------- bias-table gradient in a fixed order (backward pass 1)
// tile[i * ld + j] holds dS of query slot i of query piece qp and key slot j of key piece kp of the chunk at offset
// (dR, dC); masked pairs, rows past the chunk and empty slots hold 0.  The pair (query qr, qc; key kr, kc) adds to entry
// (qr - kr - dR w + 2w - 1) (4w - 1) + (qc - kc - dC w + 2w - 1).  The pairs of one entry have one (u, v) = (qr - kr,
// qc - kc), so its queries form a rectangle, clipped to the two pieces' slot ranges row by row.  The (2w - 1)^2 windows
// (u, v) are dealt out to the `nthreads` threads of the CTA; each adds its pairs in ascending query-slot order and then
// adds that sum to acc[entry], which no other thread touches until the next barrier.  Every CTA thereby sums in one fixed
// order, whatever the number of threads that share the windows.
__device__ __forceinline__ void table_grad_piece(const float* tile, int ld, float* acc, const Geo& geo, int dR, int dC,
                                                 int qp, int kp, int nthreads) {
  const int w = geo.w, tw = 4 * w - 1, ww = 2 * w - 1;
  const int q0 = qp * 64, k0 = kp * 64;
  for (int x = threadIdx.x; x < ww * ww; x += nthreads) {
    const int u = x / ww - (w - 1), v = x % ww - (w - 1);
    const int c_lo = max(0, v), c_hi = min(w - 1, w - 1 + v);
    float sum = 0.f;
    bool any = false;
    for (int qr = max(0, u); qr <= min(w - 1, w - 1 + u); ++qr) {
      const int kr = qr - u;
      // query slot qr w + qc in [q0, q0 + 64), key slot kr w + qc - v in [k0, k0 + 64)
      const int lo = max(c_lo, max(q0 - qr * w, k0 - kr * w + v));
      const int hi = min(c_hi, min(q0 + 63 - qr * w, k0 + 63 - kr * w + v));
      const int base = (qr * w - q0) * ld + (kr * w - v - k0);
      for (int qc = lo; qc <= hi; ++qc) sum += tile[base + qc * (ld + 1)];
      any |= lo <= hi;
    }
    if (any) acc[(u - dR * w + 2 * w - 1) * tw + (v - dC * w + 2 * w - 1)] += sum;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace vil
