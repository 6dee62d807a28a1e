// Tensor-core (wgmma) kernel family of the Vision-Longformer attention, bf16 / fp16 operands, fp32 accumulation; fp32
// operands run as split bf16 pairs (T = float, below).
//
// Same decomposition and masking rules as the SIMT family (vil_simt.cuh), with every product on the tensor cores:
// a CTA is one warpgroup (128 threads) owning a 64-row tile; it walks 64-column pieces (the global keys, then the
// visited chunks piece by piece).  Per piece the operands are copied (cp.async, a few pieces ahead) into shared memory as
// 8x8 core matrices in their natural (token, d) layout, with the mask / bias terms of every column, and
//   forward          S = Q K^T (SS), online softmax in registers, O += P V (RS: P stays in registers)
//   backward pass 1  S = Q K^T, dP = dO V^T (SS), dS = P (dP - delta), dQ += dS K (RS)         (query-stationary)
//   backward pass 2  S^T = K Q^T, dP^T = V dO^T (SS), dV += P^T dO, dK += dS^T Q (RS)           (key-stationary)
// The global query rows and the global key columns of the backward are served by the shared SIMT global-token kernels.
//
// Accumulator fragment of m64nNk16 (fp32): thread t of warp wp holds, for register i, row 16 wp + (t / 4) + 8 ((i / 2) % 2)
// and column 8 (i / 4) + 2 (t % 4) + (i % 2).  The A fragment of a k16 slice is the same layout over 16 columns, so an
// accumulator tile converts to the A operand of the next product without leaving registers.  The B operand of an RS
// product (V, K, dO, Q: consumed along the token axis) is the same (token, d) tile an SS product reads K-major, read
// MN-major.
#pragma once
#include <type_traits>
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

// Ring of operand stages: piece pi is staged into stage pi % kStages<HD> while the pieces before it are multiplied, so the
// copies of kStages<HD> - 1 pieces are in flight behind the MMAs of a round.  3 stages up to HD 64; at HD 128 a stage is
// two 16 KB tiles and 2 stages keep two CTAs on an SM (3 would leave one, DESIGN.md section 3).
template <int HD> constexpr int kStages = HD <= 64 ? 3 : 2;

// fp32 operands as split bf16 pairs (VIL_FLAG_F32_SPLIT): with T = float every product A B runs as
// A_hi B_hi + A_hi B_lo + A_lo B_hi, hi = bf16(x), lo = bf16(x - hi), all three into the same fp32 accumulators.  A
// (64 x HD) fp32 tile holds the hi tile in its first half and the lo tile in its second, each in the core-matrix layout
// of a bf16 tile.  Such a tile has the bytes of a bf16 tile of head width 2 HD (kTileHD), and takes that tile's ring
// depth and CTAs per SM.
template <typename T> constexpr bool kSplit = std::is_same<T, float>::value;
template <typename T> using Op = std::conditional_t<kSplit<T>, __nv_bfloat16, T>;   // element type of the products
template <typename T, int HD> constexpr int kTileHD = kSplit<T> ? 2 * HD : HD;
template <typename T, int HD> constexpr int kRing = kStages<kTileHD<T, HD>>;

// The thread's row segment of a (64 x HD) tile: row `row`, columns [half HD / 2, (half + 1) HD / 2), copied 16 bytes at a
// time from row `tok` of the (b, h) slice `base` (row stride st) straight into the core-matrix layout.  tok < 0 (a phantom
// row) and 8-column groups at or past D are zero-filled without a read: padding keys / queries keep K = V = 0, which the
// masks rely on (a NaN in a masked column would survive the fmaf with -inf).  Needs D % 8 == 0 and 16-byte aligned rows.
// A split fp32 tile takes the 8 values of a core-matrix row as two 16-byte copies: the first four into the bytes of
// their hi row, the last four into those of their lo row, where split_row converts them in place.
template <typename T, int HD>
__device__ __forceinline__ void stage_row(T* tile, const T* base, long long st, long long tok, int row, int half, int D) {
  constexpr int HH = HD / 2;
  const T* src = base + (tok < 0 ? 0 : tok * st);
#pragma unroll
  for (int g8 = 0; g8 < HH / 8; ++g8) {
    const int c = half * HH + g8 * 8;
    const bool in = tok >= 0 && c < D;
    if constexpr (kSplit<T>) {
      __nv_bfloat16* hi = reinterpret_cast<__nv_bfloat16*>(tile) + sm90::core_off(row, c, HD);
      sm90::cp_async16(hi, in ? src + c : base, in ? 16 : 0);
      sm90::cp_async16(hi + 64 * HD, in ? src + c + 4 : base, in ? 16 : 0);
    } else {
      sm90::cp_async16(tile + sm90::core_off(row, c, HD), in ? src + c : base, in ? 16 : 0);
    }
  }
}

// hi = bf16(x), lo = bf16(x - hi) of two values, packed as an A fragment register (x - hi is exact in fp32)
__device__ __forceinline__ void split2(float x, float y, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = sm90::pack2<__nv_bfloat16>(x - __low2float(h), y - __high2float(h));
}

// Converts in place the row segment stage_row copied into a split fp32 tile (run by the thread that copied it, after its
// copies have landed: it reads and writes only those bytes).  Zero-filled phantom rows and columns give hi = lo = 0.
template <int HD>
__device__ __forceinline__ void split_row(float* tile, int row, int half) {
  constexpr int HH = HD / 2;
#pragma unroll
  for (int g8 = 0; g8 < HH / 8; ++g8) {
    __nv_bfloat16* hp = reinterpret_cast<__nv_bfloat16*>(tile) + sm90::core_off(row, half * HH + g8 * 8, HD);
    uint4* hi = reinterpret_cast<uint4*>(hp);
    uint4* lo = reinterpret_cast<uint4*>(hp + 64 * HD);
    const float4 x = *reinterpret_cast<const float4*>(hi), y = *reinterpret_cast<const float4*>(lo);
    uint4 h, l;
    split2(x.x, x.y, h.x, l.x);
    split2(x.z, x.w, h.y, l.y);
    split2(y.x, y.y, h.z, l.z);
    split2(y.z, y.w, h.w, l.w);
    *hi = h;
    *lo = l;
  }
}

// The two products the split adds to an SS product over HD: A_hi B_lo + A_lo B_hi (A, B: split fp32 tiles)
template <int HD>
__device__ __forceinline__ void split_ss(float (&d)[32], const float* A, const float* B) {
  using W64 = sm90::Wg<__nv_bfloat16, 64>;
  const __nv_bfloat16* a = reinterpret_cast<const __nv_bfloat16*>(A);
  const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(B);
#pragma unroll
  for (int kk = 0; kk < HD / 16; ++kk) W64::ss(d, sm90::desc(a, HD, kk), sm90::desc(b + 64 * HD, HD, kk), 1);
#pragma unroll
  for (int kk = 0; kk < HD / 16; ++kk) W64::ss(d, sm90::desc(a + 64 * HD, HD, kk), sm90::desc(b, HD, kk), 1);
}

// The two products the split adds to an RS product over the 64 columns of a piece: A_hi B_lo + A_lo B_hi (A: the hi /
// lo fragments of an accumulator tile, B: a split fp32 tile read MN-major)
template <int HD>
__device__ __forceinline__ void split_rs(float (&d)[HD / 2], const uint32_t (&hi)[4][4], const uint32_t (&lo)[4][4], const float* B) {
  using WHD = sm90::Wg<__nv_bfloat16, HD>;
  const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(B);
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) WHD::rs(d, hi[kk], sm90::desc_mn(b + 64 * HD, HD, kk), 1);
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) WHD::rs(d, lo[kk], sm90::desc_mn(b, HD, kk), 1);
}

// A operand of the k16 slice kk from a 64-column accumulator tile
template <typename T>
__device__ __forceinline__ void to_a_frag(const float (&s)[32], int kk, uint32_t (&a)[4]) {
  a[0] = sm90::pack2<T>(s[8 * kk + 0], s[8 * kk + 1]);
  a[1] = sm90::pack2<T>(s[8 * kk + 2], s[8 * kk + 3]);
  a[2] = sm90::pack2<T>(s[8 * kk + 4], s[8 * kk + 5]);
  a[3] = sm90::pack2<T>(s[8 * kk + 6], s[8 * kk + 7]);
}

// A operands of all four k16 slices of a 64-column accumulator tile; split: also the lo fragments
template <typename T>
__device__ __forceinline__ void to_a_frags(const float (&s)[32], uint32_t (&a)[4][4], uint32_t (&lo)[4][4]) {
  if constexpr (kSplit<T>) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int j = 0; j < 4; ++j) split2(s[8 * kk + 2 * j], s[8 * kk + 2 * j + 1], a[kk][j], lo[kk][j]);
  } else {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) to_a_frag<T>(s, kk, a[kk]);
  }
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
template <bool DIL>
__device__ __forceinline__ void drop_rows(const Geo& geo, const SubGrid<DIL>& sg, int R, int C, int piece, uint32_t (&row)[2]) {
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int l = piece * 64 + acc_row(2 * e);
    row[e] = DIL ? (uint32_t)VIL_SUB_ROW(R * geo.w + l / geo.w, C * geo.w + l % geo.w)
                 : (uint32_t)((R * geo.w + l / geo.w) * geo.ny + C * geo.w + l % geo.w);
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

// sgn = +1: the key chunks seen by query chunk (R, C); sgn = -1: the query chunks that see key chunk (R, C).  Chunks of the
// CTA's sub-grid sg.
template <bool DIL>
__device__ __forceinline__ int visit_list(const Geo& geo, const SubGrid<DIL>& sg, int R, int C, int sgn, Visit* vl) {
  int n = 0;
  for (int oi = 0; oi < geo.noffs; ++oi) {
    const int dR = geo.offR[oi], dC = geo.offC[oi];
    int r = R + sgn * dR, c = C + sgn * dC;
    if (geo.exact == -1) { r = (r + VIL_SG(mx)) % VIL_SG(mx); c = (c + VIL_SG(my)) % VIL_SG(my); }
    else if (r < 0 || r >= VIL_SG(mx) || c < 0 || c >= VIL_SG(my)) continue;
    const int qR = sgn > 0 ? R : r, qC = sgn > 0 ? C : c;
    if (threadIdx.x == 0) vl[n] = Visit{r, c, dR, dC, (qR + dR == VIL_SG(mx) - 1) | ((qC + dC == VIL_SG(my) - 1) << 1), oi};
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

// The thread's slot in the next chunk piece to stage: slot `slot` of piece pj of visited chunk vi is the chunk's position
// pj * 64 + slot = (kr, kc) (kr >= w: an empty slot).  One piece further is 64 positions further, so walking the pieces in
// order needs no division.
struct SlotWalk {
  int vi, pj, kr, kc;
  int r0, c0, dr, dc;   // slot / w, slot % w, 64 / w, 64 % w
  __device__ __forceinline__ SlotWalk(const Geo& geo, int slot)
      : vi(0), pj(0), r0(slot / geo.w), c0(slot % geo.w), dr(64 / geo.w), dc(64 % geo.w) { kr = r0; kc = c0; }
  __device__ __forceinline__ void next(const Geo& geo) {
    if (++pj == geo.npc) { pj = 0; ++vi; kr = r0; kc = c0; return; }
    kr += dr; kc += dc;
    if (kc >= geo.w) { kc -= geo.w; ++kr; }
  }
};

// SlotWalk holding only the position: the start and the step are recomputed (two divisions per piece) rather than kept
// in registers across the loop.  Pass 2 at HD 128 uses it: its 128 accumulator registers leave none to spare.
struct SlotWalkLean {
  int vi, pj, kr, kc;
  __device__ __forceinline__ SlotWalkLean(const Geo& geo, int slot) : vi(0), pj(0), kr(slot / geo.w), kc(slot % geo.w) {}
  __device__ __forceinline__ void next(const Geo& geo) {
    const int slot = threadIdx.x >> 1;
    if (++pj == geo.npc) { pj = 0; ++vi; kr = slot / geo.w; kc = slot % geo.w; return; }
    kr += 64 / geo.w; kc += 64 % geo.w;
    if (kc >= geo.w) { kc -= geo.w; ++kr; }
  }
};

// Key (kr, kc) (kr < w) of visited chunk v: the token (-1: a zero row), whether the column takes part at all (the pad-cut
// rule folded in), and the key's (row, column) relative to the query chunk's origin -- the rules of simt_fwd_local.
template <bool DIL>
__device__ __forceinline__ void chunk_key(const Geo& geo, const SubGrid<DIL>& sg, const Visit& v, int kr, int kc, long long& tok, bool& ok,
                                          int& vr, int& vc) {
  const int w = geo.w;
  const int ar = v.r * w + kr, ac = v.c * w + kc;
  const bool real = (ar < VIL_SG(nx)) && (ac < VIL_SG(ny));
  if (geo.exact == -1)
    ok = !(((v.cut & 1) && (kr >= w - VIL_SG(padx))) || ((v.cut & 2) && (kc >= w - VIL_SG(pady))));
  else
    ok = real;
  tok = (ok && real) ? VIL_SUB_KEY(ar, ac) : -1;   // phantom padding keys keep K = V = 0
  vr = v.dR * w + kr; vc = v.dC * w + kc;
}

// Column slot of key piece pi (ngp pieces of global keys, then npc per visited chunk, taken in order: the chunk pieces
// advance `wk`): gk = the global key (-1 for a local one or an empty slot), then as chunk_key.  Global keys sit at (0, 0),
// which every query of the chunk sees under the exact window.
template <bool DIL>
__device__ __forceinline__ void key_slot(const Geo& geo, const SubGrid<DIL>& sg, const Visit* vl, int ngp, int pi, int slot, SlotWalk& wk,
                                         int& gk, long long& tok, bool& ok, int& vr, int& vc) {
  gk = -1; tok = -1; ok = false; vr = 0; vc = 0;
  if (pi < ngp) {
    const int t = pi * 64 + slot;
    if (t < geo.g) { gk = t; tok = t; ok = true; }
    return;
  }
  if (wk.kr < geo.w) chunk_key<DIL>(geo, sg, vl[wk.vi], wk.kr, wk.kc, tok, ok, vr, vc);
  wk.next(geo);
}

// Per-column metadata of a staged key piece, written when the piece is issued.  The score of (query row, key column j) is
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

template <bool DIL>
__device__ __forceinline__ QRows query_rows(const Geo& geo, const SubGrid<DIL>& sg, int R, int C, int piece) {
  QRows q;
  const int w = geo.w;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int l = piece * 64 + acc_row(2 * e);
    const bool in = l < geo.w2;
    q.qr[e] = in ? l / w : 0; q.qc[e] = in ? l % w : 0;
    q.ok[e] = in && (R * w + q.qr[e] < VIL_SG(nx)) && (C * w + q.qc[e] < VIL_SG(ny));
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

// pass 1: dS = P (dP - delta) of one piece into s.  Rows past the chunk carry lse = +inf, so their P is 0.  With the bias
// table (RPE) the dS that enter its gradient also go to the fp32 tile dst (row stride kDsLd); every other element of the
// tile gets 0.
constexpr int kDsLd = 72;   // a row of 64 + 8: the float2 stores of a warp's 8 rows x 4 column pairs fall in distinct banks
constexpr size_t kDsTile = 64 * kDsLd * sizeof(float);

template <bool RPE, bool WIN>
__device__ __forceinline__ void dq_scores(float (&s)[32], const float (&dp)[32], const Geo& geo, const KeyCols& kc,
                                          const float* tab, const QRows& q, int gl, const float (&lse_r)[2],
                                          const float (&del_r)[2], float* __restrict__ dst) {
  int tb[2] = {0, 0};
  if (RPE) row_tix(geo, q, tb);
  float prev = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int e = (i >> 1) & 1;
    int bidx;
    const float val = key_score<RPE, WIN>(geo, kc, tab, q, tb, e, acc_col(i), gl, s[i], bidx);
    const float ds = __expf(val - lse_r[e]) * (dp[i] - del_r[e]);
    if (RPE) {
      const float t = (bidx >= 0 && q.ok[e] && val != -INFINITY) ? ds : 0.f;
      if (i & 1) *reinterpret_cast<float2*>(dst + acc_row(i) * kDsLd + acc_col(i - 1)) = make_float2(prev, t);
      prev = t;
    }
    s[i] = ds;
  }
}

// Shared memory of a CTA: the stationary tiles, kRing<T, HD> stages of two streamed tiles each, as many sets of per-column
// metadata, the visit list and the bias table.
constexpr size_t kKeyCols = 64 * (4 + 4 + 2 + 2);
constexpr size_t kQueryCols = 64 * (4 + 4 + 4 + 2 + 2 + 1);
constexpr size_t kVisits = 9 * sizeof(Visit);
// pass 2 with dropout also stages each query column's token
__host__ __device__ constexpr size_t query_cols_bytes(bool drop) { return kQueryCols + (drop ? 64 * sizeof(int) : 0); }

__device__ __forceinline__ KeyCols key_cols(unsigned char* meta, int stage) {
  KeyCols kc;
  kc.bias = reinterpret_cast<float*>(meta + stage * kKeyCols);
  kc.tix = reinterpret_cast<int*>(kc.bias + 64);
  kc.kr = reinterpret_cast<short*>(kc.tix + 64);
  kc.kc = kc.kr + 64;
  return kc;
}

template <typename T, int HD> struct FwdSmem {     // Q; K, V per stage
  static constexpr size_t tiles = (1 + 2 * kRing<T, HD>) * 64 * HD * sizeof(T);
  static size_t total(int tabn) { return (tiles + kRing<T, HD> * kKeyCols + kVisits + (size_t)tabn * 4 + 15) & ~size_t(15); }
};
template <typename T, int HD> struct DqSmem {      // Q, dO; K, V per stage; with the bias table, the dS tile after the table
  static constexpr size_t tiles = (2 + 2 * kRing<T, HD>) * 64 * HD * sizeof(T);
  static size_t total(int tabn, bool tab = false) {
    return ((tiles + kRing<T, HD> * kKeyCols + kVisits + (size_t)tabn * 4 + 15) & ~size_t(15)) + (tab ? kDsTile : 0);
  }
};
template <typename T, int HD> struct DkvSmem {     // K, V; Q, dO per stage; the key rows' chunk positions
  static constexpr size_t tiles = (2 + 2 * kRing<T, HD>) * 64 * HD * sizeof(T);
  static size_t total(int tabn, bool drop = false) {
    return (tiles + kRing<T, HD> * query_cols_bytes(drop) + kVisits + 64 * sizeof(int) + (size_t)tabn * 4 + 15) & ~size_t(15);
  }
};

// Stages key piece pi (K and V rows, the column metadata) into ring stage pi % kRing<T, HD> and commits it as one cp.async
// group; past the last piece it commits an empty group, so that every round waits on the same group count.
template <typename T, int HD, bool DIL>
__device__ __forceinline__ void issue_key_piece(const Geo& geo, const SubGrid<DIL>& sg, int pi, int npieces, int ngp, const Visit* vl, SlotWalk& wk,
                                                T* ring, unsigned char* meta, const T* kb, long long kst, const T* vb,
                                                long long vst, int h, const float* __restrict__ g2l) {
  if (pi < npieces) {
    const int slot = threadIdx.x >> 1, half = threadIdx.x & 1, st = pi % kRing<T, HD>;
    int gk, vr, vc;
    long long tok;
    bool ok;
    key_slot<DIL>(geo, sg, vl, ngp, pi, slot, wk, gk, tok, ok, vr, vc);
    T* Ks = ring + st * 2 * 64 * HD;
    stage_row<T, HD>(Ks, kb, kst, tok, slot, half, geo.D);
    stage_row<T, HD>(Ks + 64 * HD, vb, vst, tok, slot, half, geo.D);
    if (half == 0) stage_key_cols(geo, key_cols(meta, st), h, g2l, gk, ok, vr, vc);
  }
  sm90::cp_async_commit();
}

// Top of round pi: piece pi has landed in every thread's copies, is visible to the async proxy, and every thread is done
// with round pi - 1, whose stage the next issue refills.  Split fp32 tiles: before the barrier each thread converts the
// rows it copied, those of the piece's two tiles at `piece` and in round 0 those of the n0 stationary tiles at `fixed`.
template <typename T, int HD>
__device__ __forceinline__ void ring_wait(T* piece, T* fixed, int n0) {
  sm90::cp_async_wait<kRing<T, HD> - 2>();
  if constexpr (kSplit<T>) {
    const int slot = threadIdx.x >> 1, half = threadIdx.x & 1;
    split_row<HD>(piece, slot, half);
    split_row<HD>(piece + 64 * HD, slot, half);
    for (int i = 0; i < n0; ++i) split_row<HD>(fixed + i * 64 * HD, slot, half);
  }
  sm90::fence_proxy_async();
  __syncthreads();
}

// ----------------------------------------------------------------------------------------------
// forward, local queries
// ----------------------------------------------------------------------------------------------
// held to 5 / 3 CTAs per SM (HD <= 32 / 64): left alone, ptxas spends registers on hoisting the column loads and drops one.
// HD 128: 2, what the 2-stage ring fits (the O accumulator alone is 64 registers).  Split fp32 tiles: 4 / 3 / 2 (HD 16 /
// 32 / 64); at 5 the HD 16 kernel, with its lo fragments, spills.  DIL at HD 16: 4; at 5 it spills 24 bytes once the
// sub-grid comes from a per-image size read from memory, which ptxas cannot rematerialise from the kernel parameters.
template <typename T, int HD, typename TO, bool DROP = false, bool DIL = false>
__global__ void __launch_bounds__(kThreads, kSplit<T> ? (HD <= 16 ? 4 : HD <= 32 ? 3 : 2)
                                                      : HD <= 16 && DIL ? 4 : HD <= 32 ? 5 : HD <= 64 ? 3 : 2)
wg_fwd_local(Geo geo, T4 q, T4 k, T4 v, T4 o, float* __restrict__ lse, const float* __restrict__ table,
             const float* __restrict__ g2l, const int* __restrict__ image_hw) {
  constexpr int HH = HD / 2, TILE = 64 * HD;
  using W64 = sm90::Wg<Op<T>, 64>;
  using WHD = sm90::Wg<Op<T>, HD>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* Qs = reinterpret_cast<T*>(smem_raw);
  T* ring = Qs + TILE;                                            // stage s: K at ring + 2 s TILE, V after it
  unsigned char* meta = reinterpret_cast<unsigned char*>(ring + 2 * kRing<T, HD> * TILE);
  Visit* vl = reinterpret_cast<Visit*>(meta + kRing<T, HD> * kKeyCols);
  float* tab = reinterpret_cast<float*>(vl + 9);
  const int tabn = geo.has_bias ? (4 * geo.w - 1) * (4 * geo.w - 1) : 0;

  const Cta cid = decode(geo, blockIdx.x);
  const int b = cid.b, h = cid.h;
  int R = cid.R, C = cid.C;
  const int tid = threadIdx.x, slot = tid >> 1, half = tid & 1;
  const int w = geo.w, D = geo.D;
  for (int i = tid; i < tabn; i += kThreads) tab[i] = table[(long long)i * geo.H + h];
  const auto sg = sub_grid<DIL>(geo, R, C, image_hw, b);
  if (off_sub_grid<DIL>(sg, R, C)) return;
  {
    const int l = cid.piece * 64 + slot;
    const int r = R * w + l / w, c = C * w + l % w;
    const bool real = l < geo.w2 && r < VIL_SG(nx) && c < VIL_SG(ny);
    stage_row<T, HD>(Qs, row_ptr<T>(q, b, h, 0), q.st, real ? VIL_SUB_TOK(r, c) : -1, slot, half, D);
  }
  float m[2] = {-INFINITY, -INFINITY}, lsum[2] = {0.f, 0.f};
  float oacc[HH];
#pragma unroll
  for (int i = 0; i < HH; ++i) oacc[i] = 0.f;

  const int ngp = (geo.g + 63) / 64, npieces = ngp + visit_list(geo, sg, R, C, 1, vl) * geo.npc;
  const int epi = key_epilogue(geo);
  const T* kb = row_ptr<T>(k, b, h, 0);
  const T* vb = row_ptr<T>(v, b, h, 0);
  SlotWalk wk(geo, slot);
  __syncthreads();                                                // the visit list
#pragma unroll
  for (int p = 0; p < kRing<T, HD> - 1; ++p)                       // the first group also carries Q
    issue_key_piece<T, HD, DIL>(geo, sg, p, npieces, ngp, vl, wk, ring, meta, kb, k.st, vb, v.st, h, g2l);
  for (int pi = 0; pi < npieces; ++pi) {
    ring_wait<T, HD>(ring + pi % kRing<T, HD> * 2 * TILE, Qs, pi == 0 ? 1 : 0);
    issue_key_piece<T, HD, DIL>(geo, sg, pi + kRing<T, HD> - 1, npieces, ngp, vl, wk, ring, meta, kb, k.st, vb, v.st, h, g2l);
    const int st = pi % kRing<T, HD>;
    const T* Ks = ring + st * 2 * TILE;
    const T* Vs = Ks + TILE;
    const KeyCols kcol = key_cols(meta, st);
    float s[32];
    sm90::wg_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) W64::ss(s, sm90::desc(Qs, HD, kk), sm90::desc(Ks, HD, kk), kk > 0);
    if constexpr (kSplit<T>) split_ss<HD>(s, Qs, Ks);
    sm90::wg_commit();
    sm90::wg_wait0();
    sm90::reg_fence(s);
    float mx[2] = {-INFINITY, -INFINITY};
    const int gl = geo.g - pi * 64;
    // the row coordinates are derived where they are used: kept live across the loop, they cost the HD 32 forward a spill
    switch (epi) {   // CTA-uniform
      case 0: fwd_scores<false, false>(s, mx, geo, kcol, tab, query_rows(geo, sg, R, C, cid.piece), gl); break;
      case 1: fwd_scores<false, true>(s, mx, geo, kcol, tab, query_rows(geo, sg, R, C, cid.piece), gl); break;
      case 2: fwd_scores<true, false>(s, mx, geo, kcol, tab, query_rows(geo, sg, R, C, cid.piece), gl); break;
      default: fwd_scores<true, true>(s, mx, geo, kcol, tab, query_rows(geo, sg, R, C, cid.piece), gl); break;
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
      drop_rows<DIL>(geo, sg, R, C, cid.piece, drow);
      drop_key_piece(s, geo, drow, drop_col_base(geo, vl, ngp, pi), 2u * (uint32_t)(b * geo.H + h), 1.f);
    }
    uint32_t a[4][4], al[4][4];
    to_a_frags<T>(s, a, al);
    sm90::wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) WHD::rs(oacc, a[kk], sm90::desc_mn(Vs, HD, kk), 1);
    if constexpr (kSplit<T>) split_rs<HD>(oacc, a, al, Vs);
    sm90::wg_commit();
    sm90::wg_wait0();
    sm90::reg_fence(oacc);
  }
  const QRows qrow = query_rows(geo, sg, R, C, cid.piece);
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    lsum[e] += __shfl_xor_sync(0xffffffffu, lsum[e], 1);
    lsum[e] += __shfl_xor_sync(0xffffffffu, lsum[e], 2);
    if (!qrow.ok[e]) continue;
    const long long tokq = VIL_SUB_TOK(R * w + qrow.qr[e], C * w + qrow.qc[e]);
    const float inv = lsum[e] > 0.f ? 1.f / lsum[e] : 0.f;
    store_rows<TO, HD>(oacc, e, row_ptr_w<TO>(o, b, h, tokq), D, DROP ? inv * geo.drop_scale : inv);
    if ((tid & 3) == 0) lse[((long long)b * geo.H + h) * geo.Nloc + tokq] = m[e] + logf(lsum[e]);
  }
}

// ----------------------------------------------------------------------------------------------
// backward pass 1 (query-stationary): dq and the local-bias-table gradient
// ----------------------------------------------------------------------------------------------
// TAB (the call has the bias table): the CTA is slice cid.b of the images and runs images cid.b, cid.b + nslice, ...;
// after each chunk piece's dQ product its dS tile is added, in a fixed order, to the CTA's row of table partials tpart
// (vil_common.cuh: table_grad_piece).  Without TAB, one image per CTA and none of that code.
// HD 128 is held to 2 CTAs per SM, what the 2-stage ring fits; below it ptxas is left alone, except for DIL at HD <= 32:
// its sub-grid, read from memory for per-image sizes, cannot be rematerialised from the kernel parameters, and left alone
// ptxas gives up a CTA per SM for it.  Held to the CTAs per SM the kernels had before per-image sizes, where that does
// not spill: 3 with dropout, 4 without (split fp32 tiles; bf16 / fp16 at HD 32 with the table and HD 16 without).
// bf16 / fp16 at HD 32 without the table stays at 3 (at 4 it spills 4 bytes), at HD 16 with the table at the 3 it had.
template <typename T, int HD, typename TO, bool DROP = false, bool TAB = false, bool DIL = false>
__global__ void __launch_bounds__(kThreads, kTileHD<T, HD> <= 64
                                                ? (DIL && HD <= 32 ? (DROP ? 3 : kSplit<T> || HD == (TAB ? 32 : 16) ? 4 : 0) : 0)
                                                : 2)
wg_bwd_dq(Geo geo, T4 q, T4 k, T4 v, T4 d_o, T4 dq, const float* __restrict__ lse, const float* __restrict__ delta,
          const float* __restrict__ table, const float* __restrict__ g2l, float* __restrict__ tpart,
          const int* __restrict__ image_hw) {
  constexpr int HH = HD / 2, TILE = 64 * HD;
  using W64 = sm90::Wg<Op<T>, 64>;
  using WHD = sm90::Wg<Op<T>, HD>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* Qs = reinterpret_cast<T*>(smem_raw);
  T* Gs = Qs + TILE;
  T* ring = Gs + TILE;                                            // stage s: K at ring + 2 s TILE, V after it
  unsigned char* meta = reinterpret_cast<unsigned char*>(ring + 2 * kRing<T, HD> * TILE);
  Visit* vl = reinterpret_cast<Visit*>(meta + kRing<T, HD> * kKeyCols);
  float* tab = reinterpret_cast<float*>(vl + 9);
  const int tabn = TAB ? (4 * geo.w - 1) * (4 * geo.w - 1) : 0;
  float* dst = nullptr;                                           // TAB: the dS tile, 16-byte aligned after the table
  float* acc = nullptr;                                           // TAB: the CTA's row of table partials

  const Cta cid = decode(geo, blockIdx.x);
  const int h = cid.h;
  int R = cid.R, C = cid.C;
  const int tid = threadIdx.x, slot = tid >> 1, half = tid & 1;
  const int w = geo.w, D = geo.D;
  for (int i = tid; i < tabn; i += kThreads) tab[i] = table[(long long)i * geo.H + h];
  if constexpr (TAB) {
    dst = reinterpret_cast<float*>(smem_raw + ((reinterpret_cast<unsigned char*>(tab + tabn) - smem_raw + 15) & ~15));
    acc = tpart + (long long)blockIdx.x * tabn;
    for (int i = tid; i < tabn; i += kThreads) acc[i] = 0.f;
  }
  auto sg = sub_grid<DIL>(geo, R, C, image_hw, cid.b);
  // after zeroing its row of table partials; TAB: per image below, since the sub-grid depends on the image's size
  if (!TAB && off_sub_grid<DIL>(sg, R, C)) return;
  const int nimg = TAB ? (geo.B - cid.b + geo.nslice - 1) / geo.nslice : 1;
  for (int it = 0; it < nimg; ++it) {
  const int b = cid.b + it * geo.nslice;
  const long long bh = (long long)b * geo.H + h;
  if constexpr (TAB && DIL) {                                     // CTA-uniform: skip an image the chunk lies outside of
    if (it > 0 && image_hw != nullptr) sg.fit(geo, image_hw, b);  // (dilated without sizes: the same sub-grid)
    if (off_sub_grid<DIL>(sg, R, C)) continue;
  }
  if (TAB && it > 0) __syncthreads();                             // the previous image is done with Qs, Gs, vl and the tile
  {
    const int l = cid.piece * 64 + slot;
    const int r = R * w + l / w, c = C * w + l % w;
    const long long tokq = (l < geo.w2 && r < VIL_SG(nx) && c < VIL_SG(ny)) ? VIL_SUB_TOK(r, c) : -1;
    stage_row<T, HD>(Qs, row_ptr<T>(q, b, h, 0), q.st, tokq, slot, half, D);
    stage_row<T, HD>(Gs, row_ptr<T>(d_o, b, h, 0), d_o.st, tokq, slot, half, D);
  }
  const QRows qrow = query_rows(geo, sg, R, C, cid.piece);
  float lse_r[2], del_r[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    lse_r[e] = INFINITY; del_r[e] = 0.f;
    if (qrow.ok[e]) {
      const long long tokq = VIL_SUB_TOK(R * w + qrow.qr[e], C * w + qrow.qc[e]);
      lse_r[e] = lse[bh * geo.Nloc + tokq];
      del_r[e] = delta[bh * geo.Nloc + tokq];
    }
  }
  float dqacc[HH];
#pragma unroll
  for (int i = 0; i < HH; ++i) dqacc[i] = 0.f;

  const int ngp = (geo.g + 63) / 64, npieces = ngp + visit_list(geo, sg, R, C, 1, vl) * geo.npc;
  const T* kb = row_ptr<T>(k, b, h, 0);
  const T* vb = row_ptr<T>(v, b, h, 0);
  SlotWalk wk(geo, slot);
  __syncthreads();                                                // the visit list
#pragma unroll
  for (int p = 0; p < kRing<T, HD> - 1; ++p)                       // the first group also carries Q and dO
    issue_key_piece<T, HD, DIL>(geo, sg, p, npieces, ngp, vl, wk, ring, meta, kb, k.st, vb, v.st, h, g2l);
  for (int pi = 0; pi < npieces; ++pi) {
    ring_wait<T, HD>(ring + pi % kRing<T, HD> * 2 * TILE, Qs, pi == 0 ? 2 : 0);
    issue_key_piece<T, HD, DIL>(geo, sg, pi + kRing<T, HD> - 1, npieces, ngp, vl, wk, ring, meta, kb, k.st, vb, v.st, h, g2l);
    const int st = pi % kRing<T, HD>;
    const T* Ks = ring + st * 2 * TILE;
    const T* Vs = Ks + TILE;
    const KeyCols kcol = key_cols(meta, st);
    float s[32], dp[32];
    sm90::wg_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) W64::ss(s, sm90::desc(Qs, HD, kk), sm90::desc(Ks, HD, kk), kk > 0);
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) W64::ss(dp, sm90::desc(Gs, HD, kk), sm90::desc(Vs, HD, kk), kk > 0);
    if constexpr (kSplit<T>) {
      split_ss<HD>(s, Qs, Ks);
      split_ss<HD>(dp, Gs, Vs);
    }
    sm90::wg_commit();
    sm90::wg_wait0();
    sm90::reg_fence(s);
    sm90::reg_fence(dp);
    const int gl = geo.g - pi * 64;
    if constexpr (DROP) {    // dS = P (dP keep / (1 - p) - delta)
      uint32_t drow[2];
      drop_rows<DIL>(geo, sg, R, C, cid.piece, drow);
      drop_key_piece(dp, geo, drow, drop_col_base(geo, vl, ngp, pi), 2u * (uint32_t)(b * geo.H + h), geo.drop_scale);
    }
    // CTA-uniform: the bias-table forms run only in the TAB instantiation
    if (geo.exact == 1) dq_scores<TAB, true>(s, dp, geo, kcol, tab, qrow, gl, lse_r, del_r, dst);
    else dq_scores<TAB, false>(s, dp, geo, kcol, tab, qrow, gl, lse_r, del_r, dst);
    uint32_t a[4][4], al[4][4];
    to_a_frags<T>(s, a, al);
    sm90::wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) WHD::rs(dqacc, a[kk], sm90::desc_mn(Ks, HD, kk), 1);
    if constexpr (kSplit<T>) split_rs<HD>(dqacc, a, al, Ks);
    sm90::wg_commit();
    sm90::wg_wait0();
    sm90::reg_fence(dqacc);
    if constexpr (TAB) {
      if (pi >= ngp) {       // a chunk piece (CTA-uniform); the tile is rewritten only after the next round's barrier
        __syncthreads();     // every thread's dS is in the tile
        const int c = pi - ngp, vi = c / geo.npc;
        table_grad_piece(dst, kDsLd, acc, geo, vl[vi].dR, vl[vi].dC, cid.piece, c - vi * geo.npc, kThreads);
      }
    }
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    if (!qrow.ok[e]) continue;
    const long long tokq = VIL_SUB_TOK(R * w + qrow.qr[e], C * w + qrow.qc[e]);
    store_rows<TO, HD>(dqacc, e, row_ptr_w<TO>(dq, b, h, tokq), D, geo.scale);
  }
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

// Chunk position of tile row `row` of key piece `piece`, packed as kr | kc << 8 | (row lies in the chunk) << 16 (w <= 48);
// rows past the chunk read (0, 0).  Written once per CTA into shared memory, so that the loop runs no division.
__device__ __forceinline__ int key_pos(const Geo& geo, int piece, int row) {
  const int lk = piece * 64 + row;
  return lk < geo.w2 ? (lk / geo.w) | ((lk % geo.w) << 8) | (1 << 16) : 0;
}

// The thread's two key rows, from the positions key_pos wrote to kpos[64]
template <bool DIL>
__device__ __forceinline__ KRows key_rows(const Geo& geo, const SubGrid<DIL>& sg, int KR, int KC, const int* kpos) {
  KRows k;
  const int w = geo.w, tw = 4 * w - 1;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int pos = kpos[acc_row(2 * e)];
    const bool in = pos >> 16;
    k.kr[e] = pos & 0xff; k.kc[e] = (pos >> 8) & 0xff;
    k.real[e] = in && (KR * w + k.kr[e] < VIL_SG(nx)) && (KC * w + k.kc[e] < VIL_SG(ny));
    k.tb[e] = k.kr[e] * tw + k.kc[e] - (2 * w - 1) * (tw + 1);
    k.cut[e] = (k.kr[e] >= w - VIL_SG(padx)) | ((k.kc[e] >= w - VIL_SG(pady)) << 1);
  }
  return k;
}

// the metadata of ring stage `stage`; `bytes` = query_cols_bytes(DROP) per stage
__device__ __forceinline__ QueryCols query_cols(unsigned char* meta, int stage, int bytes) {
  QueryCols qc;
  qc.lse = reinterpret_cast<float*>(meta + stage * bytes);
  qc.del = qc.lse + 64;
  qc.tix = reinterpret_cast<int*>(qc.del + 64);
  qc.qr = reinterpret_cast<short*>(qc.tix + 64);
  qc.qc = qc.qr + 64;
  qc.cut = reinterpret_cast<unsigned char*>(qc.qc + 64);
  qc.tok = reinterpret_cast<int*>(qc.cut + 64);
  return qc;
}

// Stages query piece qp (Q and dO rows, the column metadata with lse and delta) into ring stage qp % kRing<T, HD> and commits it
// as one cp.async group (an empty one past the last piece).  The walk runs over the chunks of vl, npc pieces each.
template <typename T, int HD, bool DROP, bool DIL, typename Walk>
__device__ __forceinline__ void issue_query_piece(const Geo& geo, const SubGrid<DIL>& sg, int qp, int npieces, const Visit* vl, Walk& wk, T* ring,
                                                  unsigned char* meta, const T* qb, long long qst, const T* gb, long long gst,
                                                  const float* __restrict__ lse, const float* __restrict__ delta) {
  if (qp < npieces) {
    const int slot = threadIdx.x >> 1, half = threadIdx.x & 1, st = qp % kRing<T, HD>, w = geo.w;
    bool qv = false;
    long long tq = 0;
    int qa = 0, qb2 = 0, cut = 0;
    if (wk.kr < w) {
      const Visit vq = vl[wk.vi];
      const int r = vq.r * w + wk.kr, c = vq.c * w + wk.kc;
      qv = (r < VIL_SG(nx)) && (c < VIL_SG(ny));
      tq = VIL_SUB_TOK(r, c);
      qa = wk.kr - vq.dR * w; qb2 = wk.kc - vq.dC * w; cut = vq.cut;
    }
    wk.next(geo);
    T* Qs = ring + st * 2 * 64 * HD;
    stage_row<T, HD>(Qs, qb, qst, qv ? tq : -1, slot, half, geo.D);
    stage_row<T, HD>(Qs + 64 * HD, gb, gst, qv ? tq : -1, slot, half, geo.D);
    if (half == 0) {
      const QueryCols qcol = query_cols(meta, st, (int)query_cols_bytes(DROP));
      if (qv) {
        sm90::cp_async4(qcol.lse + slot, lse + tq);
        sm90::cp_async4(qcol.del + slot, delta + tq);
      } else {
        qcol.lse[slot] = INFINITY;
        qcol.del[slot] = 0.f;
      }
      const int tw = 4 * w - 1;
      qcol.tix[slot] = qa * tw + qb2;
      qcol.qr[slot] = (short)qa; qcol.qc[slot] = (short)qb2;
      qcol.cut[slot] = (unsigned char)cut;
      if (DROP) qcol.tok[slot] = (int)tq;
    }
  }
  sm90::cp_async_commit();
}

// Pass 2's per-element forms: RPE adds the bias table, MASK 1 is the exact window (exact == 1), MASK 2 the pad cut of
// exact == -1
__device__ __forceinline__ int query_epilogue(const Geo& geo) {
  return (geo.has_bias ? 3 : 0) + (geo.exact == 1 ? 1 : geo.exact == -1 ? 2 : 0);
}

// Dropout bits of query piece qp in pass 2: bit i = element i of the thread's fragment is kept
__device__ __forceinline__ uint32_t query_piece_keep(const Geo& geo, const Visit* vl, const QueryCols& qc, int qp, int piece,
                                                     int b, int h) {
  const int vi = qp / geo.npc;
  const uint32_t c0 = (uint32_t)(geo.g + vl[vi].oi * geo.w2 + piece * 64), sid = 2u * (uint32_t)(b * geo.H + h);
  uint32_t keep = 0;
#pragma unroll 1
  for (int i = 0; i < 32; ++i)
    keep |= (uint32_t)drop_keep(geo, (uint32_t)qc.tok[acc_col(i)], c0 + (uint32_t)acc_row(i), sid) << i;
  return keep;
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

// held to 4 / 3 CTAs per SM (HD <= 32 / 64) without dropout, 3 / 2 with it: left alone, ptxas takes more registers and
// fits one less.  HD 128: 2 with or without dropout, what the 2-stage ring fits.  Split fp32 tiles: 3 / 2 / 2 (HD 16 / 32
// / 64): the hi and lo fragments of P and dS are 64 registers, and at one CTA more the HD 16 and HD 32 kernels spill.
template <typename T, int HD, typename TO, bool DROP = false, bool DIL = false>
__global__ void __launch_bounds__(kThreads, kSplit<T> ? (HD <= 16 ? 3 : 2) : HD > 64 ? 2 : (HD <= 32 ? 4 : 3) - (DROP ? 1 : 0))
wg_bwd_dkv(Geo geo, T4 q, T4 k, T4 v, T4 d_o, T4 dk, T4 dv, const float* __restrict__ lse, const float* __restrict__ delta,
           const float* __restrict__ table, const int* __restrict__ image_hw) {
  constexpr int HH = HD / 2, TILE = 64 * HD;
  using W64 = sm90::Wg<Op<T>, 64>;
  using WHD = sm90::Wg<Op<T>, HD>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* Ks = reinterpret_cast<T*>(smem_raw);
  T* Vs = Ks + TILE;
  T* ring = Vs + TILE;                                            // stage s: Q at ring + 2 s TILE, dO after it
  unsigned char* meta = reinterpret_cast<unsigned char*>(ring + 2 * kRing<T, HD> * TILE);
  const int cols = (int)query_cols_bytes(DROP);
  Visit* vl = reinterpret_cast<Visit*>(meta + kRing<T, HD> * cols);
  int* kpos = reinterpret_cast<int*>(vl + 9);
  float* tab = reinterpret_cast<float*>(kpos + 64);
  const int tw = 4 * geo.w - 1;
  const int tabn = geo.has_bias ? tw * tw : 0;

  const Cta cid = decode(geo, blockIdx.x);
  const int b = cid.b, h = cid.h;
  int KR = cid.R, KC = cid.C;
  const int tid = threadIdx.x, slot = tid >> 1, half = tid & 1;
  const int w = geo.w, D = geo.D;
  const long long bh = (long long)b * geo.H + h;
  for (int i = tid; i < tabn; i += kThreads) tab[i] = table[(long long)i * geo.H + h];
  const auto sg = sub_grid<DIL>(geo, KR, KC, image_hw, b);
  if (off_sub_grid<DIL>(sg, KR, KC)) return;
  {
    const int lk = cid.piece * 64 + slot;
    const int ar = KR * w + lk / w, ac = KC * w + lk % w;
    const long long tokk = (lk < geo.w2 && ar < VIL_SG(nx) && ac < VIL_SG(ny)) ? VIL_SUB_KEY(ar, ac) : -1;
    stage_row<T, HD>(Ks, row_ptr<T>(k, b, h, 0), k.st, tokk, slot, half, D);
    stage_row<T, HD>(Vs, row_ptr<T>(v, b, h, 0), v.st, tokk, slot, half, D);
    if (half == 0) kpos[slot] = key_pos(geo, cid.piece, slot);
  }
  float dkacc[HH], dvacc[HH];
#pragma unroll
  for (int i = 0; i < HH; ++i) { dkacc[i] = 0.f; dvacc[i] = 0.f; }

  const int npieces = visit_list(geo, sg, KR, KC, -1, vl) * geo.npc;
  const int epi = query_epilogue(geo);
  std::conditional_t<(HD > 64), SlotWalkLean, SlotWalk> wk(geo, slot);
  // the (b, h) slices of q, dO, lse and delta are recomputed at each issue: kept live across the loop, they cost the
  // dropout kernel at HD 32 a spill
  __syncthreads();                                                // the visit list, kpos
#pragma unroll
  for (int p = 0; p < kRing<T, HD> - 1; ++p)                       // the first group also carries K and V
    issue_query_piece<T, HD, DROP, DIL>(geo, sg, p, npieces, vl, wk, ring, meta, row_ptr<T>(q, b, h, 0), q.st,
                                   row_ptr<T>(d_o, b, h, 0), d_o.st, lse + bh * geo.Nloc, delta + bh * geo.Nloc);
  for (int qp = 0; qp < npieces; ++qp) {
    ring_wait<T, HD>(ring + qp % kRing<T, HD> * 2 * TILE, Ks, qp == 0 ? 2 : 0);
    issue_query_piece<T, HD, DROP, DIL>(geo, sg, qp + kRing<T, HD> - 1, npieces, vl, wk, ring, meta, row_ptr<T>(q, b, h, 0), q.st,
                                   row_ptr<T>(d_o, b, h, 0), d_o.st, lse + bh * geo.Nloc, delta + bh * geo.Nloc);
    const int st = qp % kRing<T, HD>;
    const T* Qs = ring + st * 2 * TILE;
    const T* Gs = Qs + TILE;
    const QueryCols qcol = query_cols(meta, st, cols);
    // dropout: bit i = element i is kept.  Up to HD 64 drawn before the products: the draws need neither, and with s and
    // dp not yet live the Philox rounds fit 3 CTAs per SM without spilling (HD <= 32).  At HD 128 drawn after them: held
    // across the products, the bits and the walk cost the kernel a spill.
    uint32_t keep = 0;
    if constexpr (DROP && HD <= 64) keep = query_piece_keep(geo, vl, qcol, qp, cid.piece, b, h);
    float s[32], dp[32];
    sm90::wg_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) W64::ss(s, sm90::desc(Ks, HD, kk), sm90::desc(Qs, HD, kk), kk > 0);
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) W64::ss(dp, sm90::desc(Vs, HD, kk), sm90::desc(Gs, HD, kk), kk > 0);
    if constexpr (kSplit<T>) {
      split_ss<HD>(s, Ks, Qs);
      split_ss<HD>(dp, Vs, Gs);
    }
    sm90::wg_commit();
    sm90::wg_wait0();
    sm90::reg_fence(s);
    sm90::reg_fence(dp);
    if constexpr (DROP && HD > 64) keep = query_piece_keep(geo, vl, qcol, qp, cid.piece, b, h);
    if constexpr (DROP) {    // dS = P (dP keep / (1 - p) - delta); the A operand of dV is P keep / (1 - p)
#pragma unroll
      for (int i = 0; i < 32; ++i) dp[i] = (keep >> i) & 1u ? dp[i] * geo.drop_scale : 0.f;
    }
    // the key rows are read from kpos where they are used: kept live across the loop, they cost the HD 32 kernel a spill
    switch (epi) {   // CTA-uniform
      case 0: dkv_probs<false, 0>(s, dp, geo, qcol, tab, key_rows(geo, sg, KR, KC, kpos)); break;
      case 1: dkv_probs<false, 1>(s, dp, geo, qcol, tab, key_rows(geo, sg, KR, KC, kpos)); break;
      case 2: dkv_probs<false, 2>(s, dp, geo, qcol, tab, key_rows(geo, sg, KR, KC, kpos)); break;
      case 3: dkv_probs<true, 0>(s, dp, geo, qcol, tab, key_rows(geo, sg, KR, KC, kpos)); break;
      case 4: dkv_probs<true, 1>(s, dp, geo, qcol, tab, key_rows(geo, sg, KR, KC, kpos)); break;
      default: dkv_probs<true, 2>(s, dp, geo, qcol, tab, key_rows(geo, sg, KR, KC, kpos)); break;
    }
    if constexpr (DROP) {
#pragma unroll
      for (int i = 0; i < 32; ++i) s[i] = (keep >> i) & 1u ? s[i] * geo.drop_scale : 0.f;
    }
    uint32_t ap[4][4], ad[4][4];
    if constexpr (kSplit<T>) {
      uint32_t apl[4][4], adl[4][4];
      to_a_frags<T>(s, ap, apl);
      to_a_frags<T>(dp, ad, adl);
      sm90::wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) WHD::rs(dvacc, ap[kk], sm90::desc_mn(Gs, HD, kk), 1);
      split_rs<HD>(dvacc, ap, apl, Gs);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) WHD::rs(dkacc, ad[kk], sm90::desc_mn(Qs, HD, kk), 1);
      split_rs<HD>(dkacc, ad, adl, Qs);
    } else {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) { to_a_frag<T>(s, kk, ap[kk]); to_a_frag<T>(dp, kk, ad[kk]); }
      sm90::wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) WHD::rs(dvacc, ap[kk], sm90::desc_mn(Gs, HD, kk), 1);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) WHD::rs(dkacc, ad[kk], sm90::desc_mn(Qs, HD, kk), 1);
    }
    sm90::wg_commit();
    sm90::wg_wait0();
    sm90::reg_fence(dvacc);
    sm90::reg_fence(dkacc);
  }
  const KRows krow = key_rows(geo, sg, KR, KC, kpos);
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    if (!krow.real[e]) continue;
    const long long tokk = VIL_SUB_KEY(KR * w + krow.kr[e], KC * w + krow.kc[e]);
    store_rows<TO, HD>(dkacc, e, row_ptr_w<TO>(dk, b, h, tokk), D, geo.scale);
    store_rows<TO, HD>(dvacc, e, row_ptr_w<TO>(dv, b, h, tokk), D, 1.f);
  }
}

}  // namespace wg
}  // namespace vil
