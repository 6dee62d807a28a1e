// Tensor-core (wgmma) kernel family of the Vision-Longformer attention, bf16 / fp16 operands, fp32 accumulation.
//
// Same decomposition and masking rules as the SIMT family (vil_simt.cuh), with every product on the tensor cores:
// a CTA is one warpgroup (128 threads) owning a 64-row tile; it walks 64-column pieces (the global keys, then the
// visited chunks piece by piece).  Per piece the operands are staged into shared memory as 8x8 core matrices and
//   forward          S = Q K^T (SS), online softmax in registers, O += P V (RS: P stays in registers)
//   backward pass 1  S = Q K^T, dP = dO V^T (SS), dS = P (dP - delta), dQ += dS K (RS)         (query-stationary)
//   backward pass 2  S^T = K Q^T, dP^T = V dO^T (SS), dV += P^T dO, dK += dS^T Q (RS)           (key-stationary)
// The global query rows and the global key columns of the backward are served by the shared SIMT global-token kernels.
//
// Accumulator fragment of m64nNk16 (fp32): thread t of warp wp holds, for register i, row 16 wp + (t / 4) + 8 ((i / 2) % 2)
// and column 8 (i / 4) + 2 (t % 4) + (i % 2).  The A fragment of a k16 slice is the same layout over 16 columns, so an
// accumulator tile converts to the A operand of the next product without leaving registers.
#pragma once
#include "vil_common.cuh"
#include "vil_sm90.cuh"

namespace vil {
namespace wg {

constexpr int kThreads = 128;

struct Cta { int b, h, R, C, piece; };

__device__ __forceinline__ Cta decode(const Geo& g, int bid) {
  Cta c;
  c.piece = bid % g.npc; bid /= g.npc;
  c.C = bid % g.my; bid /= g.my;
  c.R = bid % g.mx; bid /= g.mx;
  c.h = bid % g.H;
  c.b = bid / g.H;
  return c;
}

__device__ __forceinline__ int acc_row(int i) { return ((threadIdx.x >> 5) << 4) + ((threadIdx.x & 31) >> 2) + (((i >> 1) & 1) << 3); }
__device__ __forceinline__ int acc_col(int i) { return ((i >> 2) << 3) + ((threadIdx.x & 3) << 1) + (i & 1); }

// half a row (HD/2 values of tile row `row`) -> (64 x HD) core-matrix tile; optionally also into the transposed (HD x 64) tile
template <typename T, int HD>
__device__ __forceinline__ void stage_half_row(T* tile, T* tile_t, const float (&x)[HD / 2], int row, int half) {
  constexpr int HH = HD / 2;
#pragma unroll
  for (int g8 = 0; g8 < HH / 8; ++g8) {
    uint4 u;
    u.x = sm90::pack2<T>(x[g8 * 8 + 0], x[g8 * 8 + 1]);
    u.y = sm90::pack2<T>(x[g8 * 8 + 2], x[g8 * 8 + 3]);
    u.z = sm90::pack2<T>(x[g8 * 8 + 4], x[g8 * 8 + 5]);
    u.w = sm90::pack2<T>(x[g8 * 8 + 6], x[g8 * 8 + 7]);
    *reinterpret_cast<uint4*>(tile + sm90::core_off(row, half * HH + g8 * 8, HD)) = u;
  }
  if (tile_t != nullptr) {
#pragma unroll
    for (int i = 0; i < HH; ++i) tile_t[sm90::core_off(half * HH + i, row, 64)] = ElemTraits<T>::from_f(x[i]);
  }
}

// A operand of the k16 slice kk from a 64-column accumulator tile
template <typename T>
__device__ __forceinline__ void to_a_frag(const float (&s)[32], int kk, uint32_t (&a)[4]) {
  a[0] = sm90::pack2<T>(s[8 * kk + 0], s[8 * kk + 1]);
  a[1] = sm90::pack2<T>(s[8 * kk + 2], s[8 * kk + 3]);
  a[2] = sm90::pack2<T>(s[8 * kk + 4], s[8 * kk + 5]);
  a[3] = sm90::pack2<T>(s[8 * kk + 6], s[8 * kk + 7]);
}

// acc (64 x HD) rows -> global rows (only the first D columns)
template <typename TO, int HD>
__device__ __forceinline__ void store_rows(const float (&acc)[HD / 2], int e, TO* row, int D, float mul) {
  const int c0 = (threadIdx.x & 3) << 1;
#pragma unroll
  for (int j = 0; j < HD / 8; ++j) {
    const int col = 8 * j + c0;
    if (col < D) row[col] = ElemTraits<TO>::from_f(acc[4 * j + 2 * e] * mul);
    if (col + 1 < D) row[col + 1] = ElemTraits<TO>::from_f(acc[4 * j + 2 * e + 1] * mul);
  }
}

// One piece of <= 64 keys visible from query chunk (R, C): which tokens, which flags (0 none, 1 local, 2 global) and the
// (row, column) of every key relative to the query chunk's origin -- the rules of simt_fwd_local.
struct KeyPieces {
  int ngp, n;
  __device__ KeyPieces(const Geo& g) : ngp((g.g + 63) / 64), n((g.g + 63) / 64 + g.noffs * g.npc) {}
};
// returns false when the piece lies outside the image (CTA-uniform skip)
__device__ __forceinline__ bool key_piece(const Geo& geo, int R, int C, int pi, int ngp, int slot, long long& tok, int& flag,
                                          int& vr, int& vc) {
  tok = -1; flag = 0; vr = 0; vc = 0;
  const int w = geo.w;
  if (pi < ngp) {
    const int t = pi * 64 + slot;
    if (t < geo.g) { flag = 2; vr = t; tok = t; }
    return true;
  }
  const int oi = (pi - ngp) / geo.npc, kp = (pi - ngp) % geo.npc;
  const int dR = geo.offR[oi], dC = geo.offC[oi];
  int KR = R + dR, KC = C + dC;
  if (geo.exact == -1) { KR = (KR + geo.mx) % geo.mx; KC = (KC + geo.my) % geo.my; }
  else if (KR < 0 || KR >= geo.mx || KC < 0 || KC >= geo.my) return false;
  const int lk = kp * 64 + slot;
  if (lk < geo.w2) {
    const int kr = lk / w, kc = lk % w;
    const int ar = KR * w + kr, ac = KC * w + kc;
    const bool real = (ar < geo.nx) && (ac < geo.ny);
    if (geo.exact == -1)
      flag = !(((R + dR == geo.mx - 1) && (kr >= w - geo.padx)) || ((C + dC == geo.my - 1) && (kc >= w - geo.pady)));
    else
      flag = real;
    if (flag && real) tok = geo.g + (long long)ar * geo.ny + ac;   // phantom padding keys keep K = V = 0
    vr = dR * w + kr; vc = dC * w + kc;
  }
  return true;
}

// additive bias of (query row qr, qc) against key j; false when the pair is masked
__device__ __forceinline__ bool pair_bias(const Geo& geo, int f, int kvr, int kvc, int qr, int qc, int h, const float* tab,
                                          const float* __restrict__ g2l, float& bias, int& bidx) {
  bias = 0.f; bidx = -1;
  if (f == 2) {
    if (geo.has_bias) bias = g2l[((long long)geo.H + h) * geo.g + kvr];
    return true;
  }
  const int w = geo.w, dr = qr - kvr, dc = qc - kvc;
  if (geo.exact == 1 && (abs(dr) > w || abs(dc) > w)) return false;
  if (geo.has_bias) { bidx = (dr + 2 * w - 1) * (4 * w - 1) + dc + 2 * w - 1; bias = tab[bidx]; }
  return true;
}

template <int HD> struct FwdSmem {
  static constexpr size_t tiles = 3 * 64 * HD * 2;
  static size_t total(int tabn) { return (tiles + (size_t)tabn * 4 + 64 * 5 + 15) & ~size_t(15); }
};
template <int HD> struct DqSmem {
  static constexpr size_t tiles = 5 * 64 * HD * 2;
  static size_t total(int tabn) { return (tiles + (size_t)tabn * 4 + 64 * 5 + 15) & ~size_t(15); }
};
template <int HD> struct DkvSmem {
  static constexpr size_t tiles = 6 * 64 * HD * 2;
  static size_t total(int tabn) { return (tiles + (size_t)tabn * 4 + 64 * 13 + 15) & ~size_t(15); }
};

// ----------------------------------------------------------------------------------------------
// forward, local queries
// ----------------------------------------------------------------------------------------------
template <typename T, int HD, typename TO>
__global__ void __launch_bounds__(kThreads)
wg_fwd_local(Geo geo, T4 q, T4 k, T4 v, T4 o, float* __restrict__ lse, const float* __restrict__ table,
             const float* __restrict__ g2l) {
  constexpr int HH = HD / 2;
  using W64 = sm90::Wg<T, 64>;
  using WHD = sm90::Wg<T, HD>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* Qs = reinterpret_cast<T*>(smem_raw);
  T* Ks = Qs + 64 * HD;
  T* Vt = Ks + 64 * HD;
  float* tab = reinterpret_cast<float*>(Vt + 64 * HD);
  const int tw = 4 * geo.w - 1;
  const int tabn = geo.has_bias ? tw * tw : 0;
  short* kvr = reinterpret_cast<short*>(tab + tabn);
  short* kvc = kvr + 64;
  unsigned char* kfl = reinterpret_cast<unsigned char*>(kvc + 64);

  const Cta cid = decode(geo, blockIdx.x);
  const int b = cid.b, h = cid.h, R = cid.R, C = cid.C;
  const int tid = threadIdx.x, slot = tid >> 1, half = tid & 1;
  const int w = geo.w, D = geo.D;
  for (int i = tid; i < tabn; i += kThreads) tab[i] = table[(long long)i * geo.H + h];
  {
    const int l = cid.piece * 64 + slot;
    const int r = R * w + l / w, c = C * w + l % w;
    float x[HH];
#pragma unroll
    for (int i = 0; i < HH; ++i) x[i] = 0.f;
    if (l < geo.w2 && r < geo.nx && c < geo.ny) load_seg<T, HH>(row_ptr<T>(q, b, h, (long long)r * geo.ny + c), half * HH, D, x);
    stage_half_row<T, HD>(Qs, nullptr, x, slot, half);
  }
  int qr[2], qc[2];
  bool qok[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int l = cid.piece * 64 + acc_row(2 * e);
    qr[e] = l / w; qc[e] = l % w;
    qok[e] = (l < geo.w2) && (R * w + qr[e] < geo.nx) && (C * w + qc[e] < geo.ny);
  }
  float m[2] = {-INFINITY, -INFINITY}, lsum[2] = {0.f, 0.f};
  float oacc[HH];
#pragma unroll
  for (int i = 0; i < HH; ++i) oacc[i] = 0.f;

  const KeyPieces kp(geo);
  for (int pi = 0; pi < kp.n; ++pi) {
    long long tok; int flag, vr, vc;
    if (!key_piece(geo, R, C, pi, kp.ngp, slot, tok, flag, vr, vc)) continue;   // CTA-uniform
    __syncthreads();
    {
      float kk[HH], vv[HH];
#pragma unroll
      for (int i = 0; i < HH; ++i) { kk[i] = 0.f; vv[i] = 0.f; }
      if (tok >= 0) {
        load_seg<T, HH>(row_ptr<T>(k, b, h, tok), half * HH, D, kk);
        load_seg<T, HH>(row_ptr<T>(v, b, h, tok), half * HH, D, vv);
      }
      stage_half_row<T, HD>(Ks, nullptr, kk, slot, half);
#pragma unroll
      for (int i = 0; i < HH; ++i) Vt[sm90::core_off(half * HH + i, slot, 64)] = ElemTraits<T>::from_f(vv[i]);
      if (half == 0) { kvr[slot] = (short)vr; kvc[slot] = (short)vc; kfl[slot] = (unsigned char)flag; }
    }
    sm90::fence_proxy_async();
    __syncthreads();
    float s[32];
    sm90::wg_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) W64::ss(s, sm90::desc(Qs, HD, kk), sm90::desc(Ks, HD, kk), kk > 0);
    sm90::wg_commit();
    sm90::wg_wait0();
    sm90::reg_fence(s);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int e = (i >> 1) & 1, j = acc_col(i), f = kfl[j];
      float val = -INFINITY, bias;
      int bidx;
      if (f && qok[e] && pair_bias(geo, f, kvr[j], kvc[j], qr[e], qc[e], h, tab, g2l, bias, bidx)) val = fmaf(geo.scale, s[i], bias);
      s[i] = val;
      mx[e] = fmaxf(mx[e], val);
    }
    float corr[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 1));
      mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 2));
      const float mn = fmaxf(m[e], mx[e]);
      corr[e] = (mn == -INFINITY) ? 1.f : __expf(m[e] - mn);
      m[e] = mn;
      lsum[e] *= corr[e];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int e = (i >> 1) & 1;
      const float p = (m[e] == -INFINITY) ? 0.f : __expf(s[i] - m[e]);
      s[i] = p;
      lsum[e] += p;
    }
#pragma unroll
    for (int i = 0; i < HH; ++i) oacc[i] *= corr[(i >> 1) & 1];
    uint32_t a[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) to_a_frag<T>(s, kk, a[kk]);
    sm90::wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) WHD::rs(oacc, a[kk], sm90::desc(Vt, 64, kk), 1);
    sm90::wg_commit();
    sm90::wg_wait0();
    sm90::reg_fence(oacc);
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    lsum[e] += __shfl_xor_sync(0xffffffffu, lsum[e], 1);
    lsum[e] += __shfl_xor_sync(0xffffffffu, lsum[e], 2);
    if (!qok[e]) continue;
    const long long tokq = (long long)(R * w + qr[e]) * geo.ny + (C * w + qc[e]);
    store_rows<TO, HD>(oacc, e, row_ptr_w<TO>(o, b, h, tokq), D, lsum[e] > 0.f ? 1.f / lsum[e] : 0.f);
    if ((tid & 3) == 0) lse[((long long)b * geo.H + h) * geo.Nloc + tokq] = m[e] + logf(lsum[e]);
  }
}

// ----------------------------------------------------------------------------------------------
// backward pass 1 (query-stationary): dq and the local-bias-table gradient
// ----------------------------------------------------------------------------------------------
template <typename T, int HD, typename TO>
__global__ void __launch_bounds__(kThreads)
wg_bwd_dq(Geo geo, T4 q, T4 k, T4 v, T4 d_o, T4 dq, const float* __restrict__ lse, const float* __restrict__ delta,
          const float* __restrict__ table, const float* __restrict__ g2l, float* __restrict__ d_table) {
  constexpr int HH = HD / 2;
  using W64 = sm90::Wg<T, 64>;
  using WHD = sm90::Wg<T, HD>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* Qs = reinterpret_cast<T*>(smem_raw);
  T* Gs = Qs + 64 * HD;
  T* Ks = Gs + 64 * HD;
  T* Vs = Ks + 64 * HD;
  T* Kt = Vs + 64 * HD;
  float* tab = reinterpret_cast<float*>(Kt + 64 * HD);
  const int tw = 4 * geo.w - 1;
  const int tabn = geo.has_bias ? tw * tw : 0;
  short* kvr = reinterpret_cast<short*>(tab + tabn);
  short* kvc = kvr + 64;
  unsigned char* kfl = reinterpret_cast<unsigned char*>(kvc + 64);

  const Cta cid = decode(geo, blockIdx.x);
  const int b = cid.b, h = cid.h, R = cid.R, C = cid.C;
  const int tid = threadIdx.x, slot = tid >> 1, half = tid & 1;
  const int w = geo.w, D = geo.D;
  const long long bh = (long long)b * geo.H + h;
  for (int i = tid; i < tabn; i += kThreads) tab[i] = table[(long long)i * geo.H + h];
  {
    const int l = cid.piece * 64 + slot;
    const int r = R * w + l / w, c = C * w + l % w;
    float x[HH], y[HH];
#pragma unroll
    for (int i = 0; i < HH; ++i) { x[i] = 0.f; y[i] = 0.f; }
    if (l < geo.w2 && r < geo.nx && c < geo.ny) {
      load_seg<T, HH>(row_ptr<T>(q, b, h, (long long)r * geo.ny + c), half * HH, D, x);
      load_seg<T, HH>(row_ptr<T>(d_o, b, h, (long long)r * geo.ny + c), half * HH, D, y);
    }
    stage_half_row<T, HD>(Qs, nullptr, x, slot, half);
    stage_half_row<T, HD>(Gs, nullptr, y, slot, half);
  }
  int qr[2], qc[2];
  bool qok[2];
  float lse_r[2], del_r[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int l = cid.piece * 64 + acc_row(2 * e);
    qr[e] = l / w; qc[e] = l % w;
    qok[e] = (l < geo.w2) && (R * w + qr[e] < geo.nx) && (C * w + qc[e] < geo.ny);
    lse_r[e] = INFINITY; del_r[e] = 0.f;
    if (qok[e]) {
      const long long tokq = (long long)(R * w + qr[e]) * geo.ny + (C * w + qc[e]);
      lse_r[e] = lse[bh * geo.Nloc + tokq];
      del_r[e] = delta[bh * geo.Nloc + tokq];
    }
  }
  float dqacc[HH];
#pragma unroll
  for (int i = 0; i < HH; ++i) dqacc[i] = 0.f;

  const KeyPieces kp(geo);
  for (int pi = 0; pi < kp.n; ++pi) {
    long long tok; int flag, vr, vc;
    if (!key_piece(geo, R, C, pi, kp.ngp, slot, tok, flag, vr, vc)) continue;
    __syncthreads();
    {
      float kk[HH], vv[HH];
#pragma unroll
      for (int i = 0; i < HH; ++i) { kk[i] = 0.f; vv[i] = 0.f; }
      if (tok >= 0) {
        load_seg<T, HH>(row_ptr<T>(k, b, h, tok), half * HH, D, kk);
        load_seg<T, HH>(row_ptr<T>(v, b, h, tok), half * HH, D, vv);
      }
      stage_half_row<T, HD>(Ks, Kt, kk, slot, half);
      stage_half_row<T, HD>(Vs, nullptr, vv, slot, half);
      if (half == 0) { kvr[slot] = (short)vr; kvc[slot] = (short)vc; kfl[slot] = (unsigned char)flag; }
    }
    sm90::fence_proxy_async();
    __syncthreads();
    float s[32], dp[32];
    sm90::wg_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) W64::ss(s, sm90::desc(Qs, HD, kk), sm90::desc(Ks, HD, kk), kk > 0);
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) W64::ss(dp, sm90::desc(Gs, HD, kk), sm90::desc(Vs, HD, kk), kk > 0);
    sm90::wg_commit();
    sm90::wg_wait0();
    sm90::reg_fence(s);
    sm90::reg_fence(dp);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int e = (i >> 1) & 1, j = acc_col(i), f = kfl[j];
      float ds = 0.f, bias;
      int bidx;
      if (f && qok[e] && pair_bias(geo, f, kvr[j], kvc[j], qr[e], qc[e], h, tab, g2l, bias, bidx)) {
        const float p = __expf(fmaf(geo.scale, s[i], bias) - lse_r[e]);
        ds = p * (dp[i] - del_r[e]);
        if (bidx >= 0 && d_table != nullptr) atomicAdd(d_table + (long long)bidx * geo.H + h, ds);
      }
      s[i] = ds;
    }
    uint32_t a[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) to_a_frag<T>(s, kk, a[kk]);
    sm90::wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) WHD::rs(dqacc, a[kk], sm90::desc(Kt, 64, kk), 1);
    sm90::wg_commit();
    sm90::wg_wait0();
    sm90::reg_fence(dqacc);
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    if (!qok[e]) continue;
    const long long tokq = (long long)(R * w + qr[e]) * geo.ny + (C * w + qc[e]);
    store_rows<TO, HD>(dqacc, e, row_ptr_w<TO>(dq, b, h, tokq), D, geo.scale);
  }
}

// ----------------------------------------------------------------------------------------------
// backward pass 2 (key-stationary): dk, dv of the LOCAL key rows.  CTA = one 64-key piece of one key chunk; it walks the
// query chunks that visit it (the symmetric image of the offset list), 64 queries at a time.
// ----------------------------------------------------------------------------------------------
template <typename T, int HD, typename TO>
__global__ void __launch_bounds__(kThreads)
wg_bwd_dkv(Geo geo, T4 q, T4 k, T4 v, T4 d_o, T4 dk, T4 dv, const float* __restrict__ lse, const float* __restrict__ delta,
           const float* __restrict__ table) {
  constexpr int HH = HD / 2;
  using W64 = sm90::Wg<T, 64>;
  using WHD = sm90::Wg<T, HD>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* Ks = reinterpret_cast<T*>(smem_raw);
  T* Vs = Ks + 64 * HD;
  T* Qs = Vs + 64 * HD;
  T* Gs = Qs + 64 * HD;
  T* Qt = Gs + 64 * HD;
  T* Gt = Qt + 64 * HD;
  float* tab = reinterpret_cast<float*>(Gt + 64 * HD);
  const int tw = 4 * geo.w - 1;
  const int tabn = geo.has_bias ? tw * tw : 0;
  float* lse_s = tab + tabn;
  float* del_s = lse_s + 64;
  short* qrs = reinterpret_cast<short*>(del_s + 64);
  short* qcs = qrs + 64;
  unsigned char* qfl = reinterpret_cast<unsigned char*>(qcs + 64);

  const Cta cid = decode(geo, blockIdx.x);
  const int b = cid.b, h = cid.h, KR = cid.R, KC = cid.C;
  const int tid = threadIdx.x, slot = tid >> 1, half = tid & 1;
  const int w = geo.w, D = geo.D;
  const long long bh = (long long)b * geo.H + h;
  for (int i = tid; i < tabn; i += kThreads) tab[i] = table[(long long)i * geo.H + h];
  {
    const int lk = cid.piece * 64 + slot;
    const int ar = KR * w + lk / w, ac = KC * w + lk % w;
    float x[HH], y[HH];
#pragma unroll
    for (int i = 0; i < HH; ++i) { x[i] = 0.f; y[i] = 0.f; }
    if (lk < geo.w2 && ar < geo.nx && ac < geo.ny) {
      const long long tokk = geo.g + (long long)ar * geo.ny + ac;
      load_seg<T, HH>(row_ptr<T>(k, b, h, tokk), half * HH, D, x);
      load_seg<T, HH>(row_ptr<T>(v, b, h, tokk), half * HH, D, y);
    }
    stage_half_row<T, HD>(Ks, nullptr, x, slot, half);
    stage_half_row<T, HD>(Vs, nullptr, y, slot, half);
  }
  int kr[2], kc[2];
  bool kreal[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int lk = cid.piece * 64 + acc_row(2 * e);
    kr[e] = lk / w; kc[e] = lk % w;
    kreal[e] = (lk < geo.w2) && (KR * w + kr[e] < geo.nx) && (KC * w + kc[e] < geo.ny);
  }
  float dkacc[HH], dvacc[HH];
#pragma unroll
  for (int i = 0; i < HH; ++i) { dkacc[i] = 0.f; dvacc[i] = 0.f; }

  for (int oi = 0; oi < geo.noffs; ++oi) {
    const int dR = geo.offR[oi], dC = geo.offC[oi];
    int QR = KR - dR, QC = KC - dC;
    if (geo.exact == -1) { QR = (QR + geo.mx) % geo.mx; QC = (QC + geo.my) % geo.my; }
    else if (QR < 0 || QR >= geo.mx || QC < 0 || QC >= geo.my) continue;
    bool kvis[2];
    int vr[2], vc[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      kvis[e] = kreal[e];
      if (geo.exact == -1)
        kvis[e] = kreal[e] && !(((QR + dR == geo.mx - 1) && (kr[e] >= w - geo.padx)) ||
                                ((QC + dC == geo.my - 1) && (kc[e] >= w - geo.pady)));
      vr[e] = dR * w + kr[e]; vc[e] = dC * w + kc[e];
    }
    for (int qp = 0; qp < geo.npc; ++qp) {
      __syncthreads();
      {
        const int l = qp * 64 + slot;
        const int qrr = l / w, qcc = l % w;
        const int r = QR * w + qrr, c = QC * w + qcc;
        const bool qv = (l < geo.w2) && (r < geo.nx) && (c < geo.ny);
        float x[HH], y[HH];
#pragma unroll
        for (int i = 0; i < HH; ++i) { x[i] = 0.f; y[i] = 0.f; }
        if (qv) {
          const long long tq = (long long)r * geo.ny + c;
          load_seg<T, HH>(row_ptr<T>(q, b, h, tq), half * HH, D, x);
          load_seg<T, HH>(row_ptr<T>(d_o, b, h, tq), half * HH, D, y);
          if (half == 0) { lse_s[slot] = lse[bh * geo.Nloc + tq]; del_s[slot] = delta[bh * geo.Nloc + tq]; }
        }
        stage_half_row<T, HD>(Qs, Qt, x, slot, half);
        stage_half_row<T, HD>(Gs, Gt, y, slot, half);
        if (half == 0) { qrs[slot] = (short)qrr; qcs[slot] = (short)qcc; qfl[slot] = (unsigned char)qv; }
      }
      sm90::fence_proxy_async();
      __syncthreads();
      float s[32], dp[32];
      sm90::wg_fence();
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) W64::ss(s, sm90::desc(Ks, HD, kk), sm90::desc(Qs, HD, kk), kk > 0);
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) W64::ss(dp, sm90::desc(Vs, HD, kk), sm90::desc(Gs, HD, kk), kk > 0);
      sm90::wg_commit();
      sm90::wg_wait0();
      sm90::reg_fence(s);
      sm90::reg_fence(dp);
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int e = (i >> 1) & 1, j = acc_col(i);
        float p = 0.f, ds = 0.f;
        if (qfl[j] && kvis[e]) {
          const int dr = qrs[j] - vr[e], dc = qcs[j] - vc[e];
          if (!(geo.exact == 1 && (abs(dr) > w || abs(dc) > w))) {
            const float bias = geo.has_bias ? tab[(dr + 2 * w - 1) * tw + dc + 2 * w - 1] : 0.f;
            p = __expf(fmaf(geo.scale, s[i], bias) - lse_s[j]);
            ds = p * (dp[i] - del_s[j]);
          }
        }
        s[i] = p;
        dp[i] = ds;
      }
      uint32_t ap[4][4], ad[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) { to_a_frag<T>(s, kk, ap[kk]); to_a_frag<T>(dp, kk, ad[kk]); }
      sm90::wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) WHD::rs(dvacc, ap[kk], sm90::desc(Gt, 64, kk), 1);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) WHD::rs(dkacc, ad[kk], sm90::desc(Qt, 64, kk), 1);
      sm90::wg_commit();
      sm90::wg_wait0();
      sm90::reg_fence(dvacc);
      sm90::reg_fence(dkacc);
    }
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    if (!kreal[e]) continue;
    const long long tokk = geo.g + (long long)(KR * w + kr[e]) * geo.ny + (KC * w + kc[e]);
    store_rows<TO, HD>(dkacc, e, row_ptr_w<TO>(dk, b, h, tokk), D, geo.scale);
    store_rows<TO, HD>(dvacc, e, row_ptr_w<TO>(dv, b, h, tokk), D, 1.f);
  }
}

}  // namespace wg
}  // namespace vil
