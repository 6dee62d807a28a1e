// Tensor-core (wgmma) kernel family of the Vision-Longformer attention, bf16 / fp16 operands, fp32 accumulation.
//
// Same decomposition and masking rules as the SIMT family (vil_simt.cuh), with every product on the tensor cores:
// a CTA is one warpgroup (128 threads) owning a 64-row tile; it walks 64-column pieces (the global keys, then the
// visited chunks piece by piece).  Per piece the operands are staged into shared memory as 8x8 core matrices, with the
// mask / bias terms of every column, and
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

// Attention dropout of a key piece (forward, pass 1): x[i] *= mul where the element is kept, else 0.  row[e] = the local
// token of the thread's row e, cbase = the attn1 column of the piece's slot 0 (the slots of a piece are consecutive
// columns), sid = 2 (b H + h).
// The keep bits are drawn in a rolled loop: unrolled, the 16 Philox calls cost the forward spills.
__device__ __forceinline__ void drop_key_piece(float (&x)[32], const Geo& geo, const uint32_t (&row)[2], int cbase, uint32_t sid,
                                               float mul) {
  uint32_t keep = 0;
#pragma unroll 1
  for (int i = 0; i < 32; i += 2) {
    bool k0, k1;
    drop_keep2(geo, (i & 2) ? row[1] : row[0], (uint32_t)(cbase + acc_col(i)), sid, k0, k1);
    keep |= ((uint32_t)k0 | ((uint32_t)k1 << 1)) << i;
  }
#pragma unroll
  for (int i = 0; i < 32; ++i) x[i] = (keep >> i) & 1u ? x[i] * mul : 0.f;
}

// local token of the thread's two tile rows (past the image: any value, those rows are dropped)
__device__ __forceinline__ void drop_rows(const Geo& geo, int R, int C, int piece, uint32_t (&row)[2]) {
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int l = piece * 64 + acc_row(2 * e);
    row[e] = (uint32_t)((R * geo.w + l / geo.w) * geo.ny + C * geo.w + l % geo.w);
  }
}

// The walk.  A CTA lists the chunks it visits once, in shared memory: chunks outside the image are dropped (wrapped when
// exact == -1), the rest kept in offset order.  The forward and pass 1 take ceil(g / 64) pieces of global keys, then npc
// pieces per visited chunk; pass 2 takes npc query pieces per chunk that visits its keys.  Each chunk starts a piece of
// its own: the grouping of keys into pieces fixes the order of the fp32 sums of O, dQ, dK and dV and the running max that
// P is rounded against, and with it the bits of every result.
struct Visit {
  int r, c;     // the visited chunk
  int dR, dC;   // its offset (key chunk = query chunk + offset)
  int cut;      // exact == -1: bit 0 / 1 = the query chunk + offset is the last chunk row / column (its padded keys are cut)
  int oi;       // the offset's index in Geo::offR / offC (the reference's block order; dropout columns)
};

// sgn = +1: the key chunks seen by query chunk (R, C); sgn = -1: the query chunks that see key chunk (R, C)
__device__ __forceinline__ int visit_list(const Geo& geo, int R, int C, int sgn, Visit* vl) {
  int n = 0;
  for (int oi = 0; oi < geo.noffs; ++oi) {
    const int dR = geo.offR[oi], dC = geo.offC[oi];
    int r = R + sgn * dR, c = C + sgn * dC;
    if (geo.exact == -1) { r = (r + geo.mx) % geo.mx; c = (c + geo.my) % geo.my; }
    else if (r < 0 || r >= geo.mx || c < 0 || c >= geo.my) continue;
    const int qR = sgn > 0 ? R : r, qC = sgn > 0 ? C : c;
    if (threadIdx.x == 0) vl[n] = Visit{r, c, dR, dC, (qR + dR == geo.mx - 1) | ((qC + dC == geo.my - 1) << 1), oi};
    ++n;
  }
  return n;
}

// attn1 column of slot 0 of key piece pi (ngp pieces of global keys, then npc per visited chunk)
__device__ __forceinline__ int drop_col_base(const Geo& geo, const Visit* vl, int ngp, int pi) {
  if (pi < ngp) return pi * 64;
  const int vi = (pi - ngp) / geo.npc;
  return geo.g + vl[vi].oi * geo.w2 + (pi - ngp - vi * geo.npc) * 64;
}

// Key lk (< w^2) of visited chunk v: the token (-1: a zero row), whether the column takes part at all (the pad-cut rule
// folded in), and the key's (row, column) relative to the query chunk's origin -- the rules of simt_fwd_local.
__device__ __forceinline__ void chunk_key(const Geo& geo, const Visit& v, int lk, long long& tok, bool& ok, int& vr, int& vc) {
  const int w = geo.w, kr = lk / w, kc = lk - kr * w;
  const int ar = v.r * w + kr, ac = v.c * w + kc;
  const bool real = (ar < geo.nx) && (ac < geo.ny);
  if (geo.exact == -1)
    ok = !(((v.cut & 1) && (kr >= w - geo.padx)) || ((v.cut & 2) && (kc >= w - geo.pady)));
  else
    ok = real;
  tok = (ok && real) ? geo.g + (long long)ar * geo.ny + ac : -1;   // phantom padding keys keep K = V = 0
  vr = v.dR * w + kr; vc = v.dC * w + kc;
}

// Column slot of key piece pi (ngp pieces of global keys, then npc per visited chunk): gk = the global key (-1 for a
// local one or an empty slot), then as chunk_key.  Global keys sit at (0, 0), which every query of the chunk sees under
// the exact window.
__device__ __forceinline__ void key_slot(const Geo& geo, const Visit* vl, int ngp, int pi, int slot, int& gk, long long& tok,
                                         bool& ok, int& vr, int& vc) {
  gk = -1; tok = -1; ok = false; vr = 0; vc = 0;
  if (pi < ngp) {
    const int t = pi * 64 + slot;
    if (t < geo.g) { gk = t; tok = t; ok = true; }
    return;
  }
  const int vi = (pi - ngp) / geo.npc, lk = (pi - ngp - vi * geo.npc) * 64 + slot;
  if (lk < geo.w2) chunk_key(geo, vl[vi], lk, tok, ok, vr, vc);
}

// Per-column metadata of a staged key piece, written once per round.  The score of (query row, key column j) is
// scale * s + bias[j] (+ tab[row base - tix[j]] with the bias table), -inf where bias[j] = -inf or the exact window
// |qr - kr[j]|, |qc - kc[j]| <= w fails.
struct KeyCols {
  float* bias;   // 0, the global key's g2l bias, or -inf for a masked column
  int* tix;      // bias-table offset of the key: kr * (4w - 1) + kc
  short* kr;
  short* kc;
};
// query row of the 64-row tile: chunk-relative position (0 for rows past the chunk, which are computed and dropped)
struct QRows {
  int qr[2], qc[2];
  bool ok[2];
};

__device__ __forceinline__ QRows query_rows(const Geo& geo, int R, int C, int piece) {
  QRows q;
  const int w = geo.w;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int l = piece * 64 + acc_row(2 * e);
    const bool in = l < geo.w2;
    q.qr[e] = in ? l / w : 0; q.qc[e] = in ? l % w : 0;
    q.ok[e] = in && (R * w + q.qr[e] < geo.nx) && (C * w + q.qc[e] < geo.ny);
  }
  return q;
}

__device__ __forceinline__ void stage_key_cols(const Geo& geo, const KeyCols& kc, int h, const float* __restrict__ g2l, int gk,
                                               bool ok, int vr, int vc) {
  const int slot = threadIdx.x >> 1;
  float bias = ok ? 0.f : -INFINITY;
  if (gk >= 0 && geo.has_bias) bias = g2l[((long long)geo.H + h) * geo.g + gk];
  kc.bias[slot] = bias;
  kc.tix[slot] = vr * (4 * geo.w - 1) + vc;
  kc.kr[slot] = (short)vr;
  kc.kc[slot] = (short)vc;
}

// bias-table offset of the query rows (dr = dc = 0 at the table's centre): the entry of a pair is tb - KeyCols::tix
__device__ __forceinline__ void row_tix(const Geo& geo, const QRows& q, int (&tb)[2]) {
  const int w = geo.w, tw = 4 * w - 1;
  tb[0] = (q.qr[0] + 2 * w - 1) * tw + q.qc[0] + 2 * w - 1;
  tb[1] = (q.qr[1] + 2 * w - 1) * tw + q.qc[1] + 2 * w - 1;
}

// Masked, biased score of accumulator element s (row e of the thread, key column j); bidx = the bias-table entry it used
// (-1 for a global key or without the table).  gl = g - 64 * piece: columns j < gl are global keys.
template <bool RPE, bool WIN>
__device__ __forceinline__ float key_score(const Geo& geo, const KeyCols& kc, const float* tab, const QRows& q, const int (&tb)[2],
                                           int e, int j, int gl, float s, int& bidx) {
  float bias = kc.bias[j];
  bidx = -1;
  if (RPE && j >= gl) { bidx = tb[e] - kc.tix[j]; bias += tab[bidx]; }
  if (WIN && (abs(q.qr[e] - kc.kr[j]) > geo.w || abs(q.qc[e] - kc.kc[j]) > geo.w)) return -INFINITY;
  return fmaf(geo.scale, s, bias);
}

// Score epilogue: which of the four per-element forms a CTA runs, chosen once from the call's configuration
__device__ __forceinline__ int key_epilogue(const Geo& geo) { return (geo.has_bias ? 2 : 0) | (geo.exact == 1 ? 1 : 0); }

// forward: scores of one piece and their row maxima
template <bool RPE, bool WIN>
__device__ __forceinline__ void fwd_scores(float (&s)[32], float (&mx)[2], const Geo& geo, const KeyCols& kc, const float* tab,
                                           const QRows& q, int gl) {
  int tb[2] = {0, 0};
  if (RPE) row_tix(geo, q, tb);
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int e = (i >> 1) & 1;
    int bidx;
    s[i] = key_score<RPE, WIN>(geo, kc, tab, q, tb, e, acc_col(i), gl, s[i], bidx);
    mx[e] = fmaxf(mx[e], s[i]);
  }
}

// pass 1: dS = P (dP - delta) of one piece into s, and the bias-table gradient when d_table is set.  Rows past the chunk
// carry lse = +inf, so their P is 0.
template <bool RPE, bool WIN>
__device__ __forceinline__ void dq_scores(float (&s)[32], const float (&dp)[32], const Geo& geo, const KeyCols& kc,
                                          const float* tab, const QRows& q, int gl, const float (&lse_r)[2],
                                          const float (&del_r)[2], float* __restrict__ d_table, int h) {
  int tb[2] = {0, 0};
  if (RPE) row_tix(geo, q, tb);
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int e = (i >> 1) & 1;
    int bidx;
    const float val = key_score<RPE, WIN>(geo, kc, tab, q, tb, e, acc_col(i), gl, s[i], bidx);
    const float ds = __expf(val - lse_r[e]) * (dp[i] - del_r[e]);
    if (RPE && d_table != nullptr && bidx >= 0 && q.ok[e] && val != -INFINITY)
      atomicAdd(d_table + (long long)bidx * geo.H + h, ds);
    s[i] = ds;
  }
}

constexpr size_t kKeyMeta = 64 * (4 + 4 + 2 + 2) + 9 * sizeof(Visit);
constexpr size_t kQueryMeta = 64 * (4 + 4 + 4 + 2 + 2 + 1) + 9 * sizeof(Visit);

__device__ __forceinline__ KeyCols key_cols(float* base, Visit*& vl) {
  KeyCols kc;
  kc.bias = base;
  kc.tix = reinterpret_cast<int*>(kc.bias + 64);
  vl = reinterpret_cast<Visit*>(kc.tix + 64);
  kc.kr = reinterpret_cast<short*>(vl + 9);
  kc.kc = kc.kr + 64;
  return kc;
}

template <int HD> struct FwdSmem {
  static constexpr size_t tiles = 3 * 64 * HD * 2;
  static size_t total(int tabn) { return (tiles + (size_t)tabn * 4 + kKeyMeta + 15) & ~size_t(15); }
};
template <int HD> struct DqSmem {
  static constexpr size_t tiles = 5 * 64 * HD * 2;
  static size_t total(int tabn) { return (tiles + (size_t)tabn * 4 + kKeyMeta + 15) & ~size_t(15); }
};
template <int HD> struct DkvSmem {
  static constexpr size_t tiles = 6 * 64 * HD * 2;
  static size_t total(int tabn, bool drop = false) {
    return (tiles + (size_t)tabn * 4 + kQueryMeta + (drop ? 64 * sizeof(int) : 0) + 15) & ~size_t(15);
  }
};

// ----------------------------------------------------------------------------------------------
// forward, local queries
// ----------------------------------------------------------------------------------------------
// held to 5 / 3 CTAs per SM (HD <= 32 / 64): left alone, ptxas spends registers on hoisting the column loads and drops one
template <typename T, int HD, typename TO, bool DROP = false>
__global__ void __launch_bounds__(kThreads, HD <= 32 ? 5 : 3)
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
  const int tabn = geo.has_bias ? (4 * geo.w - 1) * (4 * geo.w - 1) : 0;
  Visit* vl;
  const KeyCols kcol = key_cols(tab + tabn, vl);

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
  float m[2] = {-INFINITY, -INFINITY}, lsum[2] = {0.f, 0.f};
  float oacc[HH];
#pragma unroll
  for (int i = 0; i < HH; ++i) oacc[i] = 0.f;

  const int ngp = (geo.g + 63) / 64, npieces = ngp + visit_list(geo, R, C, 1, vl) * geo.npc;
  const int epi = key_epilogue(geo);
  for (int pi = 0; pi < npieces; ++pi) {
    __syncthreads();
    {
      int gk, vr, vc;
      long long tok;
      bool ok;
      key_slot(geo, vl, ngp, pi, slot, gk, tok, ok, vr, vc);
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
      if (half == 0) stage_key_cols(geo, kcol, h, g2l, gk, ok, vr, vc);
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
    const int gl = geo.g - pi * 64;
    // the row coordinates are derived where they are used: kept live across the loop, they cost the HD 32 forward a spill
    switch (epi) {   // CTA-uniform
      case 0: fwd_scores<false, false>(s, mx, geo, kcol, tab, query_rows(geo, R, C, cid.piece), gl); break;
      case 1: fwd_scores<false, true>(s, mx, geo, kcol, tab, query_rows(geo, R, C, cid.piece), gl); break;
      case 2: fwd_scores<true, false>(s, mx, geo, kcol, tab, query_rows(geo, R, C, cid.piece), gl); break;
      default: fwd_scores<true, true>(s, mx, geo, kcol, tab, query_rows(geo, R, C, cid.piece), gl); break;
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
    if constexpr (DROP) {    // lsum keeps the undropped P; P V takes P * keep, 1 / (1 - p) is applied by the final store
      uint32_t drow[2];
      drop_rows(geo, R, C, cid.piece, drow);
      drop_key_piece(s, geo, drow, drop_col_base(geo, vl, ngp, pi), 2u * (uint32_t)(b * geo.H + h), 1.f);
    }
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
  const QRows qrow = query_rows(geo, R, C, cid.piece);
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    lsum[e] += __shfl_xor_sync(0xffffffffu, lsum[e], 1);
    lsum[e] += __shfl_xor_sync(0xffffffffu, lsum[e], 2);
    if (!qrow.ok[e]) continue;
    const long long tokq = (long long)(R * w + qrow.qr[e]) * geo.ny + (C * w + qrow.qc[e]);
    const float inv = lsum[e] > 0.f ? 1.f / lsum[e] : 0.f;
    store_rows<TO, HD>(oacc, e, row_ptr_w<TO>(o, b, h, tokq), D, DROP ? inv * geo.drop_scale : inv);
    if ((tid & 3) == 0) lse[((long long)b * geo.H + h) * geo.Nloc + tokq] = m[e] + logf(lsum[e]);
  }
}

// ----------------------------------------------------------------------------------------------
// backward pass 1 (query-stationary): dq and the local-bias-table gradient
// ----------------------------------------------------------------------------------------------
template <typename T, int HD, typename TO, bool DROP = false>
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
  const int tabn = geo.has_bias ? (4 * geo.w - 1) * (4 * geo.w - 1) : 0;
  Visit* vl;
  const KeyCols kcol = key_cols(tab + tabn, vl);

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
  const QRows qrow = query_rows(geo, R, C, cid.piece);
  float lse_r[2], del_r[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    lse_r[e] = INFINITY; del_r[e] = 0.f;
    if (qrow.ok[e]) {
      const long long tokq = (long long)(R * w + qrow.qr[e]) * geo.ny + (C * w + qrow.qc[e]);
      lse_r[e] = lse[bh * geo.Nloc + tokq];
      del_r[e] = delta[bh * geo.Nloc + tokq];
    }
  }
  float dqacc[HH];
#pragma unroll
  for (int i = 0; i < HH; ++i) dqacc[i] = 0.f;

  const int ngp = (geo.g + 63) / 64, npieces = ngp + visit_list(geo, R, C, 1, vl) * geo.npc;
  const int epi = key_epilogue(geo);
  for (int pi = 0; pi < npieces; ++pi) {
    __syncthreads();
    {
      int gk, vr, vc;
      long long tok;
      bool ok;
      key_slot(geo, vl, ngp, pi, slot, gk, tok, ok, vr, vc);
      float kk[HH], vv[HH];
#pragma unroll
      for (int i = 0; i < HH; ++i) { kk[i] = 0.f; vv[i] = 0.f; }
      if (tok >= 0) {
        load_seg<T, HH>(row_ptr<T>(k, b, h, tok), half * HH, D, kk);
        load_seg<T, HH>(row_ptr<T>(v, b, h, tok), half * HH, D, vv);
      }
      stage_half_row<T, HD>(Ks, Kt, kk, slot, half);
      stage_half_row<T, HD>(Vs, nullptr, vv, slot, half);
      if (half == 0) stage_key_cols(geo, kcol, h, g2l, gk, ok, vr, vc);
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
    const int gl = geo.g - pi * 64;
    if constexpr (DROP) {    // dS = P (dP keep / (1 - p) - delta)
      uint32_t drow[2];
      drop_rows(geo, R, C, cid.piece, drow);
      drop_key_piece(dp, geo, drow, drop_col_base(geo, vl, ngp, pi), 2u * (uint32_t)(b * geo.H + h), geo.drop_scale);
    }
    switch (epi) {   // CTA-uniform
      case 0: dq_scores<false, false>(s, dp, geo, kcol, tab, qrow, gl, lse_r, del_r, d_table, h); break;
      case 1: dq_scores<false, true>(s, dp, geo, kcol, tab, qrow, gl, lse_r, del_r, d_table, h); break;
      case 2: dq_scores<true, false>(s, dp, geo, kcol, tab, qrow, gl, lse_r, del_r, d_table, h); break;
      default: dq_scores<true, true>(s, dp, geo, kcol, tab, qrow, gl, lse_r, del_r, d_table, h); break;
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
    if (!qrow.ok[e]) continue;
    const long long tokq = (long long)(R * w + qrow.qr[e]) * geo.ny + (C * w + qrow.qc[e]);
    store_rows<TO, HD>(dqacc, e, row_ptr_w<TO>(dq, b, h, tokq), D, geo.scale);
  }
}

// ----------------------------------------------------------------------------------------------
// backward pass 2 (key-stationary): dk, dv of the LOCAL key rows.  CTA = one 64-key piece of one key chunk; it walks the
// query chunks that visit it (the symmetric image of the offset list), 64 queries at a time.
// ----------------------------------------------------------------------------------------------

// Per-column metadata of a staged query piece.  With (qr, qc) = the query's position minus offset * w, the pair with key
// row (kr, kc) of the key chunk has dr = qr - kr, dc = qc - kc.
struct QueryCols {
  float* lse;            // +inf for a column without a real query, so that its P is 0
  float* del;
  int* tix;              // bias-table offset: qr * (4w - 1) + qc
  short* qr;
  short* qc;
  unsigned char* cut;    // Visit::cut of the query's chunk
  int* tok;              // DROP only: the query's local token (the dropout row)
};
// key row of the 64-row tile (0 for rows past the chunk, which are computed and dropped)
struct KRows {
  int kr[2], kc[2], tb[2];   // tb: bias entry of the pair = tix[j] - tb
  int cut[2];                // exact == -1: bit 0 / 1 = the key lies in the padded rows / columns of its chunk
  bool real[2];
};

__device__ __forceinline__ QueryCols query_cols(float* base, Visit*& vl) {
  QueryCols qc;
  qc.lse = base;
  qc.del = qc.lse + 64;
  qc.tix = reinterpret_cast<int*>(qc.del + 64);
  vl = reinterpret_cast<Visit*>(qc.tix + 64);
  qc.qr = reinterpret_cast<short*>(vl + 9);
  qc.qc = qc.qr + 64;
  qc.cut = reinterpret_cast<unsigned char*>(qc.qc + 64);
  qc.tok = reinterpret_cast<int*>(qc.cut + 64);
  return qc;
}

// Pass 2's per-element forms: RPE adds the bias table, MASK 1 is the exact window (exact == 1), MASK 2 the pad cut of
// exact == -1
__device__ __forceinline__ int query_epilogue(const Geo& geo) {
  return (geo.has_bias ? 3 : 0) + (geo.exact == 1 ? 1 : geo.exact == -1 ? 2 : 0);
}

// P^T into s and dS^T into dp for one query piece
template <bool RPE, int MASK>
__device__ __forceinline__ void dkv_probs(float (&s)[32], float (&dp)[32], const Geo& geo, const QueryCols& qc, const float* tab,
                                          const KRows& kr) {
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int e = (i >> 1) & 1, j = acc_col(i);
    float x = fmaf(geo.scale, s[i], RPE ? tab[qc.tix[j] - kr.tb[e]] : 0.f) - qc.lse[j];
    if (MASK == 1 && (abs(qc.qr[j] - kr.kr[e]) > geo.w || abs(qc.qc[j] - kr.kc[e]) > geo.w)) x = -INFINITY;
    if (MASK == 2 && (qc.cut[j] & kr.cut[e])) x = -INFINITY;
    const float p = __expf(x);
    s[i] = p;
    dp[i] = p * (dp[i] - qc.del[j]);
  }
}

template <typename T, int HD, typename TO, bool DROP = false>
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
  Visit* vl;
  const QueryCols qcol = query_cols(tab + tabn, vl);

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
  KRows krow;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int lk = cid.piece * 64 + acc_row(2 * e);
    const bool in = lk < geo.w2;
    krow.kr[e] = in ? lk / w : 0; krow.kc[e] = in ? lk % w : 0;
    krow.real[e] = in && (KR * w + krow.kr[e] < geo.nx) && (KC * w + krow.kc[e] < geo.ny);
    krow.tb[e] = krow.kr[e] * tw + krow.kc[e] - (2 * w - 1) * (tw + 1);
    krow.cut[e] = (krow.kr[e] >= w - geo.padx) | ((krow.kc[e] >= w - geo.pady) << 1);
  }
  float dkacc[HH], dvacc[HH];
#pragma unroll
  for (int i = 0; i < HH; ++i) { dkacc[i] = 0.f; dvacc[i] = 0.f; }

  const int npieces = visit_list(geo, KR, KC, -1, vl) * geo.npc;
  const int epi = query_epilogue(geo);
  for (int qp = 0; qp < npieces; ++qp) {
    __syncthreads();
    {
      const int vi = qp / geo.npc, l = (qp - vi * geo.npc) * 64 + slot;
      bool qv = false;
      long long tq = 0;
      int qa = 0, qb = 0, cut = 0;
      if (l < geo.w2) {
        const int qrr = l / w, qcc = l - qrr * w;
        const Visit vq = vl[vi];
        const int r = vq.r * w + qrr, c = vq.c * w + qcc;
        qv = (r < geo.nx) && (c < geo.ny);
        tq = (long long)r * geo.ny + c;
        qa = qrr - vq.dR * w; qb = qcc - vq.dC * w; cut = vq.cut;
      }
      float x[HH], y[HH];
#pragma unroll
      for (int i = 0; i < HH; ++i) { x[i] = 0.f; y[i] = 0.f; }
      if (qv) {
        load_seg<T, HH>(row_ptr<T>(q, b, h, tq), half * HH, D, x);
        load_seg<T, HH>(row_ptr<T>(d_o, b, h, tq), half * HH, D, y);
      }
      stage_half_row<T, HD>(Qs, Qt, x, slot, half);
      stage_half_row<T, HD>(Gs, Gt, y, slot, half);
      if (half == 0) {
        qcol.lse[slot] = qv ? lse[bh * geo.Nloc + tq] : INFINITY;
        qcol.del[slot] = qv ? delta[bh * geo.Nloc + tq] : 0.f;
        qcol.tix[slot] = qa * tw + qb;
        qcol.qr[slot] = (short)qa; qcol.qc[slot] = (short)qb;
        qcol.cut[slot] = (unsigned char)cut;
        if (DROP) qcol.tok[slot] = (int)tq;
      }
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
    uint32_t keep = 0;       // dropout: bit i = element i is kept
    if constexpr (DROP) {    // dS = P (dP keep / (1 - p) - delta); the A operand of dV is P keep / (1 - p)
      const int vi = qp / geo.npc;
      const uint32_t c0 = (uint32_t)(geo.g + vl[vi].oi * geo.w2 + cid.piece * 64), sid = 2u * (uint32_t)(b * geo.H + h);
#pragma unroll 1
      for (int i = 0; i < 32; ++i)
        keep |= (uint32_t)drop_keep(geo, (uint32_t)qcol.tok[acc_col(i)], c0 + (uint32_t)acc_row(i), sid) << i;
#pragma unroll
      for (int i = 0; i < 32; ++i) dp[i] = (keep >> i) & 1u ? dp[i] * geo.drop_scale : 0.f;
    }
    switch (epi) {   // CTA-uniform
      case 0: dkv_probs<false, 0>(s, dp, geo, qcol, tab, krow); break;
      case 1: dkv_probs<false, 1>(s, dp, geo, qcol, tab, krow); break;
      case 2: dkv_probs<false, 2>(s, dp, geo, qcol, tab, krow); break;
      case 3: dkv_probs<true, 0>(s, dp, geo, qcol, tab, krow); break;
      case 4: dkv_probs<true, 1>(s, dp, geo, qcol, tab, krow); break;
      default: dkv_probs<true, 2>(s, dp, geo, qcol, tab, krow); break;
    }
    if constexpr (DROP) {
#pragma unroll
      for (int i = 0; i < 32; ++i) s[i] = (keep >> i) & 1u ? s[i] * geo.drop_scale : 0.f;
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
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    if (!krow.real[e]) continue;
    const long long tokk = geo.g + (long long)(KR * w + krow.kr[e]) * geo.ny + (KC * w + krow.kc[e]);
    store_rows<TO, HD>(dkacc, e, row_ptr_w<TO>(dk, b, h, tokk), D, geo.scale);
    store_rows<TO, HD>(dvacc, e, row_ptr_w<TO>(dv, b, h, tokk), D, 1.f);
  }
}

}  // namespace wg
}  // namespace vil
