// SIMT (CUDA-core, fp32 accumulate) kernel family of the Vision-Longformer attention.
//
// Covers EVERY configuration of the reference operator (any w, exact in {0,1,-1},
// mode in {-1,0,1..8}, any nglo, fp32 / bf16 / fp16 I/O) at D <= 128, with one limit: backward
// and dropout at 64 < D <= 128 are fp32 only (the local kernels at four lanes per row); bf16 / fp16
// SIMT training stops at D = 64.  It is (a) the fp32 parity build (1e-5 vs the fp64 oracle),
// (b) the path for configurations the wgmma family does not cover, and (c) the home of
// the small global-token kernels that both families share (every D <= 128: bf16 / fp16
// training at 64 < D <= 128 runs on the wgmma family and these kernels).
//
// Math restated from the reference (closed forms verified in oracle/vil_oracle.py):
//   local query i=(r_i,c_i) in chunk (R,C); for every visited chunk offset (dR,dC)
//   (slidingchunk_2d.py:37-79) and key (kr,kc) of chunk (R+dR, C+dC):
//     allowed   <- mask rules of slidingchunk_2d.py:249-318 (zero / exact / cyclic)
//     bias      <- table[(dr + 2w-1)*(4w-1) + (dc + 2w-1), h],  dr = qr-(dR*w+kr), dc likewise
//                  (longformer2d.py:68-100, 159-178)
//   joint softmax over [global keys | allowed local keys] (longformer2d.py:183-185),
//   o = P.[v_g | v_loc] (:194-200).  Backward: dS = P o (dP - delta) (SlidingChunk2D.backward
//   + softmax autograd, slidingchunk_2d.py:234-246).
#pragma once
#include "vil_common.cuh"

namespace vil {

// ----------------------------------------------------------------------------------------------
// Local-query kernels: CTA = one 64-slot piece of one chunk of one (b,h), L lanes per row.  Lane `part` = tid & (L-1) of
// slot tid >> (L/2) owns the HP = HD/L consecutive channels [part HP, part HP + HP) of its row; a dot product is its
// HP-term FMA chain plus log2(L) xor-shuffle steps, and lane 0 of a slot writes the per-row values (lse, delta, the dS
// tile, the staged key / query metadata).  L = 2, except for fp32 training at 64 < D <= 128: at HD 128 two lanes would
// hold 64 floats per row tensor (192 in pass 1, 256 in pass 2) and spill, so those kernels run L = 4.  The grids, the
// workspace and the fixed order of the table gradient do not depend on L.  The lane decode is a shift and a mask (tid is
// signed: tid / L, tid % L compile to different code), and the shuffle steps and the key-piece staging of the forward
// and pass 1 are written out in each kernel: moved into __forceinline__ helpers (group_sum<L> included), they compile
// to differently scheduled SASS.
// ----------------------------------------------------------------------------------------------
// fp32 smem tile row: L parts of HP floats.  L = 2: the halves are 4 floats apart, so the two threads of a (row, half)
// pair hit different banks.  L = 4: the quarters sit at a stride of HP + 1, so the four lanes of a row hit four banks and
// the 8 rows a warp stages hit all 32 (the row stride HD + 4 is 4 banks); with the HD + 8 row, pass 1 with the table at
// HD 128 and w = 48 would need 232 528 bytes, 80 over the limit, and with HD + 4 it needs 230 480.
template <int HD, int L> struct Tile {
  static constexpr int HP = HD / L;
  static constexpr int HS = L == 2 ? HD + 8 : HD + 4;
  static __device__ __forceinline__ int off(int part) { return part * (HP + (L == 2 ? 4 : 1)); }
};

struct ChunkId { int b, h, R, C, piece; };

__device__ __forceinline__ ChunkId decode_block(const Geo& g, int bid) {
  ChunkId c;
  c.piece = bid % g.npc; bid /= g.npc;
  c.C = bid % g.my; bid /= g.my;
  c.R = bid % g.mx; bid /= g.mx;
  c.h = bid % g.H;
  c.b = bid / g.H;
  return c;
}

// ----------------------------------------------------------------------------------------------
// forward, local queries
// ----------------------------------------------------------------------------------------------
template <typename T, int HD, int L, bool DROP, bool DIL = false>
__global__ void __launch_bounds__(64 * L, L == 4 ? 1 : 0)
simt_fwd_local(Geo geo, T4 q, T4 k, T4 v, T4 o, float* __restrict__ lse,
               const float* __restrict__ table, const float* __restrict__ g2l, const int* __restrict__ image_hw) {
  using TL = Tile<HD, L>;
  constexpr int HP = TL::HP, HS = TL::HS;
  extern __shared__ float smem[];
  float* Ks = smem;
  float* Vs = Ks + 64 * HS;
  float* tab = Vs + 64 * HS;
  const int tw = 4 * geo.w - 1;
  const int tabn = geo.has_bias ? tw * tw : 0;
  short* kvr = reinterpret_cast<short*>(tab + tabn);
  short* kvc = kvr + 64;
  unsigned char* kfl = reinterpret_cast<unsigned char*>(kvc + 64);

  const ChunkId cid = decode_block(geo, blockIdx.x);
  const int b = cid.b, h = cid.h;
  int R = cid.R, C = cid.C;
  const int tid = threadIdx.x, slot = tid >> (L / 2), part = tid & (L - 1);
  const int w = geo.w, D = geo.D;

  for (int i = tid; i < tabn; i += 64 * L) tab[i] = table[(long long)i * geo.H + h];
  const auto sg = sub_grid<DIL>(geo, R, C, image_hw, b);
  if (off_sub_grid<DIL>(sg, R, C)) return;

  const int l = cid.piece * 64 + slot;
  const int qr = l / w, qc = l % w;
  const int r = R * w + qr, c = C * w + qc;
  const bool qvalid = (l < geo.w2) && (r < VIL_SG(nx)) && (c < VIL_SG(ny));

  float qh[HP], oh[HP];
#pragma unroll
  for (int i = 0; i < HP; ++i) { qh[i] = 0.f; oh[i] = 0.f; }
  if (qvalid) load_seg<T, HP>(row_ptr<T>(q, b, h, VIL_SUB_TOK(r, c)), part * HP, D, qh);
  float m = -INFINITY, lsum = 0.f;
  const uint32_t drow = (uint32_t)VIL_SUB_ROW(r, c), dsid = 2u * (uint32_t)(b * geo.H + h);   // dropout: row, stream 0

  const int ngp = (geo.g + 63) / 64;
  const int npieces = ngp + geo.noffs * geo.npc;
  for (int pi = 0; pi < npieces; ++pi) {
    const bool isg = pi < ngp;
    int dR = 0, dC = 0, KR = 0, KC = 0, kp = 0;
    int cbase = pi * 64;                  // dropout: attn1 column of the piece's slot 0
    if (!isg) {
      const int oi = (pi - ngp) / geo.npc;
      kp = (pi - ngp) % geo.npc;
      if (DROP) cbase = geo.g + oi * geo.w2 + kp * 64;
      dR = geo.offR[oi]; dC = geo.offC[oi];
      KR = R + dR; KC = C + dC;
      if (geo.exact == -1) { KR = (KR + VIL_SG(mx)) % VIL_SG(mx); KC = (KC + VIL_SG(my)) % VIL_SG(my); }
      else if (KR < 0 || KR >= VIL_SG(mx) || KC < 0 || KC >= VIL_SG(my)) continue;   // CTA-uniform
    }
    __syncthreads();
    {   // stage one piece of <=64 keys: lane `part` of a slot loads its HP channels of a row of K and V
      float kk[HP], vv[HP];
#pragma unroll
      for (int i = 0; i < HP; ++i) { kk[i] = 0.f; vv[i] = 0.f; }
      int flag = 0, vr = 0, vc = 0; long long tok = -1;
      if (isg) {
        const int t = pi * 64 + slot;
        if (t < geo.g) { flag = 2; vr = t; tok = t; }
      } else {
        const int lk = kp * 64 + slot;
        if (lk < geo.w2) {
          const int kr = lk / w, kc = lk % w;
          const int ar = KR * w + kr, ac = KC * w + kc;
          const bool real = (ar < VIL_SG(nx)) && (ac < VIL_SG(ny));
          if (geo.exact == -1)
            flag = !(((R + dR == VIL_SG(mx) - 1) && (kr >= w - VIL_SG(padx))) ||
                     ((C + dC == VIL_SG(my) - 1) && (kc >= w - VIL_SG(pady))));
          else
            flag = real;
          if (flag && real) tok = VIL_SUB_KEY(ar, ac);   // phantom padding keys keep K=V=0
          vr = dR * w + kr; vc = dC * w + kc;
        }
      }
      if (tok >= 0) {
        load_seg<T, HP>(row_ptr<T>(k, b, h, tok), part * HP, D, kk);
        load_seg<T, HP>(row_ptr<T>(v, b, h, tok), part * HP, D, vv);
      }
      float* kd = Ks + slot * HS + TL::off(part);
      float* vd = Vs + slot * HS + TL::off(part);
#pragma unroll
      for (int i = 0; i < HP; ++i) { kd[i] = kk[i]; vd[i] = vv[i]; }
      if (part == 0) { kvr[slot] = (short)vr; kvc[slot] = (short)vc; kfl[slot] = (unsigned char)flag; }
    }
    __syncthreads();
    for (int j = 0; j < 64; ++j) {
      const int f = kfl[j];
      if (!f) continue;                                   // warp-uniform
      const float* kd = Ks + j * HS + TL::off(part);
      float sp = 0.f;
#pragma unroll
      for (int i = 0; i < HP; ++i) sp = fmaf(qh[i], kd[i], sp);
      sp += __shfl_xor_sync(0xffffffffu, sp, 1);           // over the L lanes of the row
      if constexpr (L == 4) sp += __shfl_xor_sync(0xffffffffu, sp, 2);
      float bias = 0.f; bool ok = qvalid;
      if (f == 2) {
        if (geo.has_bias) bias = g2l[((long long)geo.H + h) * geo.g + kvr[j]];
      } else {
        const int dr = qr - kvr[j], dc = qc - kvc[j];
        if (geo.exact == 1 && (abs(dr) > w || abs(dc) > w)) ok = false;
        if (geo.has_bias && ok) bias = tab[(dr + 2 * w - 1) * tw + dc + 2 * w - 1];
      }
      if (ok) {
        const float s = fmaf(geo.scale, sp, bias);
        const float* vd = Vs + j * HS + TL::off(part);
        // dropout: lsum sums the undropped P; O sums P * keep, scaled by 1 / (1 - p) at the end
        const float km = DROP ? (drop_keep(geo, drow, (uint32_t)(cbase + j), dsid) ? 1.f : 0.f) : 1.f;
        if (s > m) {
          const float corr = __expf(m - s);
          lsum = lsum * corr + 1.f;
#pragma unroll
          for (int i = 0; i < HP; ++i) oh[i] = fmaf(oh[i], corr, km * vd[i]);
          m = s;
        } else {
          const float p = __expf(s - m);
          lsum += p;
#pragma unroll
          for (int i = 0; i < HP; ++i) oh[i] = fmaf(p * km, vd[i], oh[i]);
        }
      }
    }
  }
  if (qvalid) {
    const float inv = (lsum > 0.f ? 1.f / lsum : 0.f) * (DROP ? geo.drop_scale : 1.f);
#pragma unroll
    for (int i = 0; i < HP; ++i) oh[i] *= inv;
    const long long tokq = VIL_SUB_TOK(r, c);
    store_seg<T, HP>(row_ptr_w<T>(o, b, h, tokq), part * HP, D, oh);
    if (part == 0) lse[((long long)b * geo.H + h) * geo.Nloc + tokq] = m + logf(lsum);
  }
}

// ----------------------------------------------------------------------------------------------
// Global-token kernels: sub-warp ROW GROUPS.  LPR = HD/8 lanes share one token row, lane `sub` owns the 8 channels
// [8 sub, 8 sub + 8) (one 16-byte load for bf16 / fp16), so a warp streams 32/LPR rows per iteration with fully
// coalesced accesses and ~40 registers per thread.  (The first version gave every thread a whole row: HD-long
// register arrays, 1 CTA per SM, 0.5 ms per layer for a few hundred MB of traffic.)
// ----------------------------------------------------------------------------------------------
template <int LPR>
__device__ __forceinline__ float group_sum(float v) {          // over the LPR lanes of one row group
#pragma unroll
  for (int o = 1; o < LPR; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <int LPR>
__device__ __forceinline__ float rows_sum(float v) {           // over the 32/LPR row groups of a warp (same `sub`)
#pragma unroll
  for (int o = LPR; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float dot8(const float (&a)[8], const float (&b)[8]) {
  float s0 = a[0] * b[0], s1 = a[1] * b[1];
#pragma unroll
  for (int i = 2; i < 8; i += 2) { s0 = fmaf(a[i], b[i], s0); s1 = fmaf(a[i + 1], b[i + 1], s1); }
  return s0 + s1;
}

// ----------------------------------------------------------------------------------------------
// forward, global query rows: dense attention of the nglo global queries over all N keys
// (longformer2d.py:210-227).  CTA = one (b, h, a); 8 warps x (32/LPR) rows per iteration.
// SIZED (per-image grids): only the global keys and the keys on image b's grid take part; the others are never loaded
// (a masked score alone would still let a NaN through 0 * v).
// ----------------------------------------------------------------------------------------------
template <typename T, int HD, typename TO = T, bool DROP = false, bool SIZED = false>   // TO: element type of the OUTPUT
__global__ void __launch_bounds__(256)
simt_fwd_global(Geo geo, T4 qg, T4 kg, T4 vg, T4 og, float* __restrict__ lse_g, const float* __restrict__ g2l,
                const float* __restrict__ g2g, const int* __restrict__ image_hw) {
  constexpr int LPR = HD / 8, RPW = 32 / LPR, ROWS = 8 * RPW;
  __shared__ float red_m[8], red_l[8];
  __shared__ float red_o[8][HD];
  const int a = blockIdx.x % geo.g;
  const int h = (blockIdx.x / geo.g) % geo.H;
  const int b = blockIdx.x / (geo.g * geo.H);
  const int tid = threadIdx.x, D = geo.D, lane = tid & 31, warp = tid >> 5, sub = lane % LPR, rw = lane / LPR;
  const int row0 = 0, row1 = geo.N;
  float q8[8];
  load_seg<T, 8>(row_ptr<T>(qg, b, h, a), 8 * sub, D, q8);
  float m = -INFINITY, lsum = 0.f, oacc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) oacc[i] = 0.f;
  const float bl = geo.has_bias ? g2l[(long long)h * geo.g + a] : 0.f;       // g2l[0][h][a]
  int ih = 0, iw = 0;
  if constexpr (SIZED) image_extent(geo, image_hw, b, ih, iw);
  for (int base = row0 + warp * RPW; base < row1; base += ROWS) {
    const int j = base + rw;
    bool valid = j < row1;
    const int jc = valid ? j : row1 - 1;
    float kk[8], vv[8];
    if (SIZED && !(jc < geo.g || on_image(geo, ih, iw, jc - geo.g))) {
      valid = false;
#pragma unroll
      for (int i = 0; i < 8; ++i) { kk[i] = 0.f; vv[i] = 0.f; }
    } else {
      load_seg<T, 8>(row_ptr<T>(kg, b, h, jc), 8 * sub, D, kk);
      load_seg<T, 8>(row_ptr<T>(vg, b, h, jc), 8 * sub, D, vv);
    }
    const float sp = group_sum<LPR>(dot8(q8, kk));
    float bias = bl;
    if (geo.has_bias && jc < geo.g) bias = g2g[((long long)h * geo.g + a) * geo.g + jc];
    const float sc = valid ? fmaf(geo.scale, sp, bias) : -INFINITY;
    const float mn = fmaxf(m, sc);
    if (mn > -INFINITY) {                        // branch-free online softmax step of this row group
      const float corr = __expf(m - mn), p = __expf(sc - mn);
      lsum = fmaf(lsum, corr, p);
      float pk = p;                              // dropout: O sums P * keep, lsum the undropped P
      if constexpr (DROP) {
        if (!drop_keep(geo, (uint32_t)a, (uint32_t)j, 2u * (uint32_t)(b * geo.H + h) + 1u)) pk = 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) oacc[i] = fmaf(oacc[i], corr, pk * vv[i]);
      m = mn;
    }
  }
  // merge the row groups of the warp, then the 8 warps (fixed order: deterministic)
  float mw = m;
#pragma unroll
  for (int o = LPR; o < 32; o <<= 1) mw = fmaxf(mw, __shfl_xor_sync(0xffffffffu, mw, o));
  const float scw = (m == -INFINITY) ? 0.f : __expf(m - mw);
  const float lw = rows_sum<LPR>(lsum * scw);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float x = rows_sum<LPR>(oacc[i] * scw);
    if (rw == 0) red_o[warp][8 * sub + i] = x;
  }
  if (lane == 0) { red_m[warp] = mw; red_l[warp] = lw; }
  __syncthreads();
  if (tid < HD) {
    float M = -INFINITY;
    for (int x = 0; x < 8; ++x) M = fmaxf(M, red_m[x]);
    float L = 0.f, O = 0.f;
    for (int x = 0; x < 8; ++x) {
      const float s2 = (red_m[x] == -INFINITY) ? 0.f : __expf(red_m[x] - M);
      L += red_l[x] * s2; O += red_o[x][tid] * s2;
    }
    if (tid < D) row_ptr_w<TO>(og, b, h, a)[tid] = ElemTraits<TO>::from_f(DROP ? O / L * geo.drop_scale : O / L);
    if (tid == 0) lse_g[((long long)b * geo.H + h) * geo.g + a] = M + logf(L);
  }
}

// ----------------------------------------------------------------------------------------------
// backward prologue: delta_i = sum_c dO_ic * O_ic for local rows (into delta) and global rows (delta_g)
// ----------------------------------------------------------------------------------------------
template <typename T, typename TO = T>               // TO: element type of o / og (fp32 in the parity build)
__global__ void simt_bwd_delta(Geo geo, T4 o, T4 d_o, T4 og, T4 d_og,
                               float* __restrict__ delta, float* __restrict__ delta_g) {
  const long long rows_loc = (long long)geo.B * geo.H * geo.Nloc;
  const long long rows = rows_loc + (long long)geo.B * geo.H * geo.g;
  const long long idx = (long long)blockIdx.x * (blockDim.x >> 2) + (threadIdx.x >> 2);  // 4 threads per row
  const int sub = threadIdx.x & 3;
  float acc = 0.f;
  if (idx < rows) {
    const TO* po;
    const T* pd;
    if (idx < rows_loc) {
      const long long t = idx % geo.Nloc; const long long bh = idx / geo.Nloc;
      po = row_ptr<TO>(o, (int)(bh / geo.H), (int)(bh % geo.H), t);
      pd = row_ptr<T>(d_o, (int)(bh / geo.H), (int)(bh % geo.H), t);
    } else {
      const long long e = idx - rows_loc;
      const long long t = e % geo.g; const long long bh = e / geo.g;
      po = row_ptr<TO>(og, (int)(bh / geo.H), (int)(bh % geo.H), t);
      pd = row_ptr<T>(d_og, (int)(bh / geo.H), (int)(bh % geo.H), t);
    }
    for (int cc = sub; cc < geo.D; cc += 4)
      acc = fmaf(ElemTraits<TO>::to_f(po[cc]), ElemTraits<T>::to_f(pd[cc]), acc);
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  if (idx < rows && sub == 0) {
    if (idx < rows_loc) delta[idx] = acc; else delta_g[idx - rows_loc] = acc;
  }
}

// ----------------------------------------------------------------------------------------------
// backward pass 1 (query-stationary): dq, and with the bias table (TAB) its gradient.  Same tiling as simt_fwd_local.
// TAB: as wg_bwd_dq, the CTA is slice cid.b of the images and runs images cid.b, cid.b + nslice, ...; the dS of each
// chunk piece go to a tile and are added in a fixed order to the CTA's row of table partials tpart (table_grad_piece).
// ----------------------------------------------------------------------------------------------
constexpr int kSimtDsLd = 65;   // dS tile row stride: the 16 query slots of a warp write one column in distinct banks
inline size_t simt_ds_tile_bytes() { return 64 * kSimtDsLd * sizeof(float); }

template <typename T, int HD, int L, bool DROP, bool TAB, bool DIL = false>
__global__ void __launch_bounds__(64 * L, L == 4 ? 1 : (TAB && HD <= 8 ? 4 : 0))
simt_bwd_dq(Geo geo, T4 q, T4 k, T4 v, T4 d_o, T4 dq, const float* __restrict__ lse,
            const float* __restrict__ delta, const float* __restrict__ table,
            const float* __restrict__ g2l, float* __restrict__ tpart, const int* __restrict__ image_hw) {
  using TL = Tile<HD, L>;
  constexpr int HP = TL::HP, HS = TL::HS;
  extern __shared__ float smem[];
  float* Ks = smem;
  float* Vs = Ks + 64 * HS;
  float* tab = Vs + 64 * HS;
  const int tw = 4 * geo.w - 1;
  const int tabn = geo.has_bias ? tw * tw : 0;
  short* kvr = reinterpret_cast<short*>(tab + tabn);
  short* kvc = kvr + 64;
  unsigned char* kfl = reinterpret_cast<unsigned char*>(kvc + 64);
  float* dst = nullptr;                                   // TAB: the dS tile, 16-byte aligned after kfl
  float* acc = nullptr;                                   // TAB: the CTA's row of table partials

  const ChunkId cid = decode_block(geo, blockIdx.x);
  const int h = cid.h;
  int R = cid.R, C = cid.C;
  const int tid = threadIdx.x, slot = tid >> (L / 2), part = tid & (L - 1);
  const int w = geo.w, D = geo.D;
  for (int i = tid; i < tabn; i += 64 * L) tab[i] = table[(long long)i * geo.H + h];
  if constexpr (TAB) {
    dst = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(smem) +
                                   ((reinterpret_cast<unsigned char*>(kfl + 64) - reinterpret_cast<unsigned char*>(smem) + 15) & ~15));
    acc = tpart + (long long)blockIdx.x * tabn;
    for (int i = tid; i < tabn; i += 64 * L) acc[i] = 0.f;
  }
  auto sg = sub_grid<DIL>(geo, R, C, image_hw, cid.b);
  // after zeroing its row of table partials; TAB: per image below, since the sub-grid depends on the image's size
  if (!TAB && off_sub_grid<DIL>(sg, R, C)) return;

  const int l = cid.piece * 64 + slot;
  const int qr = l / w, qc = l % w;
  const int r = R * w + qr, c = C * w + qc;
  bool qvalid = (l < geo.w2) && (r < VIL_SG(nx)) && (c < VIL_SG(ny));
  const long long tokq = VIL_SUB_TOK(r, c);

  const int nimg = TAB ? (geo.B - cid.b + geo.nslice - 1) / geo.nslice : 1;
  for (int it = 0; it < nimg; ++it) {
  const int b = cid.b + it * geo.nslice;
  if constexpr (TAB && DIL) {          // CTA-uniform: skip an image the chunk lies outside of; the query row's validity
    if (it > 0 && image_hw != nullptr) {   // (hoisted above for one image per CTA) follows the image's sub-grid
      sg.fit(geo, image_hw, b);
      qvalid = (l < geo.w2) && (r < sg.nx()) && (c < sg.ny());
    }
    if (off_sub_grid<DIL>(sg, R, C)) continue;
  }
  float qh[HP], doh[HP], dqh[HP];
#pragma unroll
  for (int i = 0; i < HP; ++i) { qh[i] = 0.f; doh[i] = 0.f; dqh[i] = 0.f; }
  float lse_i = INFINITY, del_i = 0.f;
  if (qvalid) {
    load_seg<T, HP>(row_ptr<T>(q, b, h, tokq), part * HP, D, qh);
    load_seg<T, HP>(row_ptr<T>(d_o, b, h, tokq), part * HP, D, doh);
    lse_i = lse[((long long)b * geo.H + h) * geo.Nloc + tokq];
    del_i = delta[((long long)b * geo.H + h) * geo.Nloc + tokq];
  }
  const uint32_t drow = (uint32_t)tokq, dsid = 2u * (uint32_t)(b * geo.H + h);   // dropout: row, stream 0

  const int ngp = (geo.g + 63) / 64;
  const int npieces = ngp + geo.noffs * geo.npc;
  for (int pi = 0; pi < npieces; ++pi) {
    const bool isg = pi < ngp;
    int dR = 0, dC = 0, KR = 0, KC = 0, kp = 0;
    int cbase = pi * 64;                  // dropout: attn1 column of the piece's slot 0
    if (!isg) {
      const int oi = (pi - ngp) / geo.npc;
      kp = (pi - ngp) % geo.npc;
      if (DROP) cbase = geo.g + oi * geo.w2 + kp * 64;
      dR = geo.offR[oi]; dC = geo.offC[oi];
      KR = R + dR; KC = C + dC;
      if (geo.exact == -1) { KR = (KR + VIL_SG(mx)) % VIL_SG(mx); KC = (KC + VIL_SG(my)) % VIL_SG(my); }
      else if (KR < 0 || KR >= VIL_SG(mx) || KC < 0 || KC >= VIL_SG(my)) continue;   // CTA-uniform
    }
    __syncthreads();
    {
      float kk[HP], vv[HP];
#pragma unroll
      for (int i = 0; i < HP; ++i) { kk[i] = 0.f; vv[i] = 0.f; }
      int flag = 0, vr = 0, vc = 0; long long tok = -1;
      if (isg) {
        const int t = pi * 64 + slot;
        if (t < geo.g) { flag = 2; vr = t; tok = t; }
      } else {
        const int lk = kp * 64 + slot;
        if (lk < geo.w2) {
          const int kr = lk / w, kc = lk % w;
          const int ar = KR * w + kr, ac = KC * w + kc;
          const bool real = (ar < VIL_SG(nx)) && (ac < VIL_SG(ny));
          if (geo.exact == -1)
            flag = !(((R + dR == VIL_SG(mx) - 1) && (kr >= w - VIL_SG(padx))) ||
                     ((C + dC == VIL_SG(my) - 1) && (kc >= w - VIL_SG(pady))));
          else
            flag = real;
          if (flag && real) tok = VIL_SUB_KEY(ar, ac);   // phantom padding keys keep K=V=0
          vr = dR * w + kr; vc = dC * w + kc;
        }
      }
      if (tok >= 0) {
        load_seg<T, HP>(row_ptr<T>(k, b, h, tok), part * HP, D, kk);
        load_seg<T, HP>(row_ptr<T>(v, b, h, tok), part * HP, D, vv);
      }
      float* kd = Ks + slot * HS + TL::off(part);
      float* vd = Vs + slot * HS + TL::off(part);
#pragma unroll
      for (int i = 0; i < HP; ++i) { kd[i] = kk[i]; vd[i] = vv[i]; }
      if (part == 0) { kvr[slot] = (short)vr; kvc[slot] = (short)vc; kfl[slot] = (unsigned char)flag; }
    }
    __syncthreads();
    for (int j = 0; j < 64; ++j) {
      const int f = kfl[j];
      if (!f) {
        if (TAB && part == 0) dst[slot * kSimtDsLd + j] = 0.f;
        continue;
      }
      float km = 1.f;                                    // dropout: keep / (1 - p) of the column
      if constexpr (DROP) km = drop_keep(geo, drow, (uint32_t)(cbase + j), dsid) ? geo.drop_scale : 0.f;
      const float* kd = Ks + j * HS + TL::off(part);
      const float* vd = Vs + j * HS + TL::off(part);
      float sp = 0.f, dpp = 0.f;
#pragma unroll
      for (int i = 0; i < HP; ++i) { sp = fmaf(qh[i], kd[i], sp); dpp = fmaf(doh[i], vd[i], dpp); }
      sp += __shfl_xor_sync(0xffffffffu, sp, 1);           // over the L lanes of the row
      if constexpr (L == 4) sp += __shfl_xor_sync(0xffffffffu, sp, 2);
      dpp += __shfl_xor_sync(0xffffffffu, dpp, 1);
      if constexpr (L == 4) dpp += __shfl_xor_sync(0xffffffffu, dpp, 2);
      float bias = 0.f; bool ok = qvalid; int bidx = -1;
      if (f == 2) {
        if (geo.has_bias) bias = g2l[((long long)geo.H + h) * geo.g + kvr[j]];
      } else {
        const int dr = qr - kvr[j], dc = qc - kvc[j];
        if (geo.exact == 1 && (abs(dr) > w || abs(dc) > w)) ok = false;
        if (geo.has_bias && ok) { bidx = (dr + 2 * w - 1) * tw + dc + 2 * w - 1; bias = tab[bidx]; }
      }
      float tg = 0.f;                                    // TAB: this row's term of the table gradient
      if (ok) {
        const float p = __expf(fmaf(geo.scale, sp, bias) - lse_i);
        if constexpr (DROP) dpp *= km;
        const float ds = p * (dpp - del_i);
#pragma unroll
        for (int i = 0; i < HP; ++i) dqh[i] = fmaf(ds, kd[i], dqh[i]);
        if (bidx >= 0) tg = ds;
      }
      if (TAB && part == 0) dst[slot * kSimtDsLd + j] = tg;
    }
    if constexpr (TAB) {
      if (!isg) {            // CTA-uniform; the next piece writes the tile only after its two barriers
        __syncthreads();     // every query's dS is in the tile
        table_grad_piece(dst, kSimtDsLd, acc, geo, dR, dC, cid.piece, kp, 64 * L);
      }
    }
  }
  if (qvalid) {
#pragma unroll
    for (int i = 0; i < HP; ++i) dqh[i] *= geo.scale;
    store_seg<T, HP>(row_ptr_w<T>(dq, b, h, tokq), part * HP, D, dqh);
  }
  }
}

// ----------------------------------------------------------------------------------------------
// backward pass 2 (key-stationary): dk, dv of the LOCAL key rows.  CTA = one 64-key piece of one
// key chunk; it walks the query chunks that visit it (the symmetric image of the offset list).
// ----------------------------------------------------------------------------------------------
template <typename T, int HD, int L, bool DROP, bool DIL = false>
__global__ void __launch_bounds__(64 * L, L == 4 ? 1 : 0)
simt_bwd_dkv(Geo geo, T4 q, T4 k, T4 v, T4 d_o, T4 dk, T4 dv, const float* __restrict__ lse,
             const float* __restrict__ delta, const float* __restrict__ table, const int* __restrict__ image_hw) {
  using TL = Tile<HD, L>;
  constexpr int HP = TL::HP, HS = TL::HS;
  extern __shared__ float smem[];
  float* Qs = smem;
  float* Gs = Qs + 64 * HS;
  float* tab = Gs + 64 * HS;
  const int tw = 4 * geo.w - 1;
  const int tabn = geo.has_bias ? tw * tw : 0;
  float* lse_s = tab + tabn;
  float* del_s = lse_s + 64;
  short* qrs = reinterpret_cast<short*>(del_s + 64);
  short* qcs = qrs + 64;
  unsigned char* qfl = reinterpret_cast<unsigned char*>(qcs + 64);
  int* qtok = reinterpret_cast<int*>(qfl + 64);            // DROP only: the query token of each staged column

  const ChunkId cid = decode_block(geo, blockIdx.x);
  const int b = cid.b, h = cid.h;
  int KR = cid.R, KC = cid.C;
  const int tid = threadIdx.x, slot = tid >> (L / 2), part = tid & (L - 1);
  const int w = geo.w, D = geo.D;
  for (int i = tid; i < tabn; i += 64 * L) tab[i] = table[(long long)i * geo.H + h];
  const auto sg = sub_grid<DIL>(geo, KR, KC, image_hw, b);
  if (off_sub_grid<DIL>(sg, KR, KC)) return;

  const int lk = cid.piece * 64 + slot;
  const int kr = lk / w, kc = lk % w;
  const int ar = KR * w + kr, ac = KC * w + kc;
  const bool kreal = (lk < geo.w2) && (ar < VIL_SG(nx)) && (ac < VIL_SG(ny));
  const long long tokk = VIL_SUB_KEY(ar, ac);

  float kh[HP], vh[HP], dkh[HP], dvh[HP];
#pragma unroll
  for (int i = 0; i < HP; ++i) { kh[i] = 0.f; vh[i] = 0.f; dkh[i] = 0.f; dvh[i] = 0.f; }
  if (kreal) {
    load_seg<T, HP>(row_ptr<T>(k, b, h, tokk), part * HP, D, kh);
    load_seg<T, HP>(row_ptr<T>(v, b, h, tokk), part * HP, D, vh);
  }

  for (int oi = 0; oi < geo.noffs; ++oi) {
    const int dR = geo.offR[oi], dC = geo.offC[oi];
    int QR = KR - dR, QC = KC - dC;
    if (geo.exact == -1) { QR = (QR + VIL_SG(mx)) % VIL_SG(mx); QC = (QC + VIL_SG(my)) % VIL_SG(my); }
    else if (QR < 0 || QR >= VIL_SG(mx) || QC < 0 || QC >= VIL_SG(my)) continue;
    // is this key visible from query chunk (QR,QC) through offset (dR,dC)?
    bool kvis = kreal;
    if (geo.exact == -1)
      kvis = kreal && !(((QR + dR == VIL_SG(mx) - 1) && (kr >= w - VIL_SG(padx))) ||
                        ((QC + dC == VIL_SG(my) - 1) && (kc >= w - VIL_SG(pady))));
    const int vr = dR * w + kr, vc = dC * w + kc;
    for (int qp = 0; qp < geo.npc; ++qp) {
      __syncthreads();
      {
        float qq[HP], gg[HP];
#pragma unroll
        for (int i = 0; i < HP; ++i) { qq[i] = 0.f; gg[i] = 0.f; }
        const int l = qp * 64 + slot;
        const int qr = l / w, qc = l % w;
        const int r = QR * w + qr, c = QC * w + qc;
        const bool qv = (l < geo.w2) && (r < VIL_SG(nx)) && (c < VIL_SG(ny));
        if (qv) {
          const long long tq = VIL_SUB_TOK(r, c);
          load_seg<T, HP>(row_ptr<T>(q, b, h, tq), part * HP, D, qq);
          load_seg<T, HP>(row_ptr<T>(d_o, b, h, tq), part * HP, D, gg);
          if (part == 0) {
            lse_s[slot] = lse[((long long)b * geo.H + h) * geo.Nloc + tq];
            del_s[slot] = delta[((long long)b * geo.H + h) * geo.Nloc + tq];
          }
        }
        float* qd = Qs + slot * HS + TL::off(part);
        float* gd = Gs + slot * HS + TL::off(part);
#pragma unroll
        for (int i = 0; i < HP; ++i) { qd[i] = qq[i]; gd[i] = gg[i]; }
        if (part == 0) { qrs[slot] = (short)qr; qcs[slot] = (short)qc; qfl[slot] = (unsigned char)qv; }
        if (DROP && part == 0) qtok[slot] = VIL_SUB_ROW(r, c);
      }
      __syncthreads();
      for (int i2 = 0; i2 < 64; ++i2) {
        if (!qfl[i2]) continue;                              // warp-uniform
        const float* qd = Qs + i2 * HS + TL::off(part);
        const float* gd = Gs + i2 * HS + TL::off(part);
        float sp = 0.f, dpp = 0.f;
#pragma unroll
        for (int i = 0; i < HP; ++i) { sp = fmaf(kh[i], qd[i], sp); dpp = fmaf(vh[i], gd[i], dpp); }
        sp += __shfl_xor_sync(0xffffffffu, sp, 1);           // over the L lanes of the row
        if constexpr (L == 4) sp += __shfl_xor_sync(0xffffffffu, sp, 2);
        dpp += __shfl_xor_sync(0xffffffffu, dpp, 1);
        if constexpr (L == 4) dpp += __shfl_xor_sync(0xffffffffu, dpp, 2);
        const int dr = qrs[i2] - vr, dc = qcs[i2] - vc;
        bool ok = kvis;
        if (geo.exact == 1 && (abs(dr) > w || abs(dc) > w)) ok = false;
        if (ok) {
          const float bias = geo.has_bias ? tab[(dr + 2 * w - 1) * tw + dc + 2 * w - 1] : 0.f;
          float p = __expf(fmaf(geo.scale, sp, bias) - lse_s[i2]);
          if constexpr (DROP) {            // dS = P (dP keep / (1 - p) - delta), dV += P keep / (1 - p) dO
            const float km = drop_keep(geo, (uint32_t)qtok[i2], (uint32_t)(geo.g + oi * geo.w2 + lk), 2u * (uint32_t)(b * geo.H + h))
                                 ? geo.drop_scale : 0.f;
            const float ds = p * (dpp * km - del_s[i2]);
            p *= km;
#pragma unroll
            for (int i = 0; i < HP; ++i) { dkh[i] = fmaf(ds, qd[i], dkh[i]); dvh[i] = fmaf(p, gd[i], dvh[i]); }
          } else {
            const float ds = p * (dpp - del_s[i2]);
#pragma unroll
            for (int i = 0; i < HP; ++i) { dkh[i] = fmaf(ds, qd[i], dkh[i]); dvh[i] = fmaf(p, gd[i], dvh[i]); }
          }
        }
      }
    }
  }
  if (kreal) {
#pragma unroll
    for (int i = 0; i < HP; ++i) dkh[i] *= geo.scale;
    store_seg<T, HP>(row_ptr_w<T>(dk, b, h, tokk), part * HP, D, dkh);
    store_seg<T, HP>(row_ptr_w<T>(dv, b, h, tokk), part * HP, D, dvh);
  }
}

// block-wide sum of a per-thread value (256 threads), result valid in thread 0
__device__ __forceinline__ float block_sum_256(float v, float* red /*[8]*/) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  if (threadIdx.x == 0) for (int i = 0; i < 8; ++i) t += red[i];
  return t;
}

// ----------------------------------------------------------------------------------------------
// backward, global KEY columns seen by the local queries: dk[t], dv[t] for t < nglo and, with the bias table, this
// image's term of d_g2l[1][h][t] into pcol[b][h][t] (summed over the images by simt_bwd_bias_reduce).
// CTA = one (b, h, t); row groups stride over the local queries.  SIZED (per-image grids): only the queries on image b's
// grid; the others, whose d_o, lse and delta are arbitrary, are never loaded.
// ----------------------------------------------------------------------------------------------
template <typename T, int HD, typename TO = T, bool DROP = false, bool SIZED = false>
__global__ void __launch_bounds__(256)
simt_bwd_gcol(Geo geo, T4 q, T4 k, T4 v, T4 d_o, T4 dk, T4 dv, const float* __restrict__ lse,
              const float* __restrict__ delta, const float* __restrict__ g2l, float* __restrict__ pcol,
              const int* __restrict__ image_hw) {
  constexpr int LPR = HD / 8, RPW = 32 / LPR, ROWS = 8 * RPW;
  __shared__ float red[8];
  __shared__ float accs[8][2][HD];
  const int t = blockIdx.x % geo.g;
  const int h = (blockIdx.x / geo.g) % geo.H;
  const int b = blockIdx.x / (geo.g * geo.H);
  const int tid = threadIdx.x, D = geo.D, lane = tid & 31, warp = tid >> 5, sub = lane % LPR, rw = lane / LPR;
  const int row0 = 0, row1 = geo.Nloc;
  float k8[8], v8[8];
  load_seg<T, 8>(row_ptr<T>(k, b, h, t), 8 * sub, D, k8);
  load_seg<T, 8>(row_ptr<T>(v, b, h, t), 8 * sub, D, v8);
  const float bias = geo.has_bias ? g2l[((long long)geo.H + h) * geo.g + t] : 0.f;
  float adk[8], adv[8], adb = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) { adk[i] = 0.f; adv[i] = 0.f; }
  const long long base_l = ((long long)b * geo.H + h) * geo.Nloc;
  int ih = 0, iw = 0;
  if constexpr (SIZED) image_extent(geo, image_hw, b, ih, iw);
  for (int base = row0 + warp * RPW; base < row1; base += ROWS) {
    const int i2 = base + rw;
    bool valid = i2 < row1;
    const int ic = valid ? i2 : row1 - 1;
    float qq[8], gg[8], ls, dl;
    if (SIZED && !on_image(geo, ih, iw, ic)) {
      valid = false; ls = 0.f; dl = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) { qq[i] = 0.f; gg[i] = 0.f; }
    } else {
      load_seg<T, 8>(row_ptr<T>(q, b, h, ic), 8 * sub, D, qq);
      load_seg<T, 8>(row_ptr<T>(d_o, b, h, ic), 8 * sub, D, gg);
      ls = lse[base_l + ic]; dl = delta[base_l + ic];
    }
    const float sp = group_sum<LPR>(dot8(qq, k8)), dpp = group_sum<LPR>(dot8(gg, v8));
    float p = valid ? __expf(fmaf(geo.scale, sp, bias) - ls) : 0.f;
    float dpk = dpp;
    if constexpr (DROP) {                          // dS = P (dP keep / (1 - p) - delta), dV += P keep / (1 - p) dO
      const float km = drop_keep(geo, (uint32_t)ic, (uint32_t)t, 2u * (uint32_t)(b * geo.H + h)) ? geo.drop_scale : 0.f;
      dpk = dpp * km;
      const float ds = p * (dpk - dl);
      if (sub == 0) adb += ds;
      p *= km;
#pragma unroll
      for (int i = 0; i < 8; ++i) { adk[i] = fmaf(ds, qq[i], adk[i]); adv[i] = fmaf(p, gg[i], adv[i]); }
    } else {
      const float ds = p * (dpk - dl);
      if (sub == 0) adb += ds;
#pragma unroll
      for (int i = 0; i < 8; ++i) { adk[i] = fmaf(ds, qq[i], adk[i]); adv[i] = fmaf(p, gg[i], adv[i]); }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float x = rows_sum<LPR>(adk[i]), y = rows_sum<LPR>(adv[i]);
    if (rw == 0) { accs[warp][0][8 * sub + i] = x; accs[warp][1][8 * sub + i] = y; }
  }
  const float tb = block_sum_256(adb, red);
  __syncthreads();
  if (tid < D) {
    float x = 0.f, y = 0.f;
    for (int w2 = 0; w2 < 8; ++w2) { x += accs[w2][0][tid]; y += accs[w2][1][tid]; }
    row_ptr_w<TO>(dk, b, h, t)[tid] = ElemTraits<TO>::from_f(x * geo.scale);
    row_ptr_w<TO>(dv, b, h, t)[tid] = ElemTraits<TO>::from_f(y);
  }
  if (tid == 0 && geo.has_bias) pcol[((long long)b * geo.H + h) * geo.g + t] = tb;
}

// ----------------------------------------------------------------------------------------------
// backward, global QUERY rows: dqg, contributions to dkg / dvg over all N keys, and with the bias table this image's
// terms of d_g2g into pgg[b][h][a][j] and of d_g2l[0] into prow[b][h][a] (summed over the images by simt_bwd_bias_reduce).
// CTA = one (b, h); row groups stride over the keys.  `accumulate` != 0: add into dkg/dvg (they alias dk/dv,
// already written by the dK/dV pass and simt_bwd_gcol earlier on the same stream); else overwrite.
// SIZED (per-image grids): as simt_fwd_global, the keys off image b's grid are never loaded and get P = 0.
// ----------------------------------------------------------------------------------------------
template <typename T, int HD, typename TO = T, bool DROP = false, bool SIZED = false>
__global__ void __launch_bounds__(256, SIZED ? 2 : 0)   // SIZED: at ptxas's own choice of 80 registers it spills
simt_bwd_grow(Geo geo, T4 qg, T4 kg, T4 vg, T4 d_og, T4 dqg, T4 dkg, T4 dvg,
              const float* __restrict__ lse_g, const float* __restrict__ delta_g,
              const float* __restrict__ g2l, const float* __restrict__ g2g,
              float* __restrict__ prow, float* __restrict__ pgg, int accumulate, int rmw_rows,
              const int* __restrict__ image_hw) {
  // rmw_rows: keys [0, rmw_rows) get their dkg / dvg rows updated here
  constexpr int LPR = HD / 8, RPW = 32 / LPR, ROWS = 8 * RPW;
  __shared__ float red[8];
  __shared__ float accs[8][HD];
  const int h = blockIdx.x % geo.H;
  const int b = blockIdx.x / geo.H;
  const int tid = threadIdx.x, D = geo.D, lane = tid & 31, warp = tid >> 5, sub = lane % LPR, rw = lane / LPR;
  const int row0 = 0, row1 = geo.N;
  int ih = 0, iw = 0;
  if constexpr (SIZED) image_extent(geo, image_hw, b, ih, iw);
  for (int a = 0; a < geo.g; ++a) {
    float q8[8], g8[8];
    load_seg<T, 8>(row_ptr<T>(qg, b, h, a), 8 * sub, D, q8);
    load_seg<T, 8>(row_ptr<T>(d_og, b, h, a), 8 * sub, D, g8);
    const float lg = lse_g[((long long)b * geo.H + h) * geo.g + a];
    const float dg = delta_g[((long long)b * geo.H + h) * geo.g + a];
    const float bl = geo.has_bias ? g2l[(long long)h * geo.g + a] : 0.f;
    const bool add = accumulate || a > 0;
    float adq[8], adb = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) adq[i] = 0.f;
    for (int base = row0 + warp * RPW; base < row1; base += ROWS) {
      const int j = base + rw;
      const bool valid = j < row1;
      const int jc = valid ? j : row1 - 1;
      float kk[8], vv[8], ok_[8], ov_[8];
      const bool live = !SIZED || jc < geo.g || on_image(geo, ih, iw, jc - geo.g);
      if (SIZED && !live) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { kk[i] = 0.f; vv[i] = 0.f; }
      } else {
        load_seg<T, 8>(row_ptr<T>(kg, b, h, jc), 8 * sub, D, kk);
        load_seg<T, 8>(row_ptr<T>(vg, b, h, jc), 8 * sub, D, vv);
      }
      const bool rmw = base < rmw_rows;                 // warp-uniform up to the last partial row batch
      if (add && rmw) {
        load_seg<TO, 8>(row_ptr<TO>(dkg, b, h, jc), 8 * sub, D, ok_);
        load_seg<TO, 8>(row_ptr<TO>(dvg, b, h, jc), 8 * sub, D, ov_);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) { ok_[i] = 0.f; ov_[i] = 0.f; }
      }
      const float sp = group_sum<LPR>(dot8(q8, kk)), dpp = group_sum<LPR>(dot8(g8, vv));
      float bias = bl;
      if (geo.has_bias && jc < geo.g) bias = g2g[((long long)h * geo.g + a) * geo.g + jc];
      const float p = valid && live ? __expf(fmaf(geo.scale, sp, bias) - lg) : 0.f;
      float km = 1.f;                              // dropout: dS = P (dP keep / (1 - p) - delta), dV += P keep / (1 - p) dO
      if constexpr (DROP) km = drop_keep(geo, (uint32_t)a, (uint32_t)jc, 2u * (uint32_t)(b * geo.H + h) + 1u) ? geo.drop_scale : 0.f;
      const float ds = DROP ? p * (dpp * km - dg) : p * (dpp - dg);
      const float pv = DROP ? p * km : p;
      if (geo.has_bias && valid && sub == 0) {   // each j < g is one row group's, once per a
        if (j < geo.g) pgg[(((long long)b * geo.H + h) * geo.g + a) * geo.g + j] = ds;
        else adb += ds;
      }
      const float dss = ds * geo.scale;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        adq[i] = fmaf(ds, kk[i], adq[i]);
        ok_[i] = fmaf(dss, q8[i], ok_[i]);        // dkg_j += scale * ds * qg_a
        ov_[i] = fmaf(pv, g8[i], ov_[i]);         // dvg_j += p * dOg_a
      }
      if (valid && j < rmw_rows && 8 * sub < D) {
        store_seg<TO, 8>(row_ptr_w<TO>(dkg, b, h, j), 8 * sub, D, ok_);
        store_seg<TO, 8>(row_ptr_w<TO>(dvg, b, h, j), 8 * sub, D, ov_);
      }
    }
    __syncthreads();                               // accs / red of the previous global query have been consumed
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float x = rows_sum<LPR>(adq[i]);
      if (rw == 0) accs[warp][8 * sub + i] = x;
    }
    const float tb = block_sum_256(adb, red);
    __syncthreads();
    if (tid < D) {
      float x = 0.f;
      for (int w2 = 0; w2 < 8; ++w2) x += accs[w2][tid];
      row_ptr_w<TO>(dqg, b, h, a)[tid] = ElemTraits<TO>::from_f(x * geo.scale);
    }
    if (tid == 0 && geo.has_bias) prow[((long long)b * geo.H + h) * geo.g + a] = tb;
  }
}

// ----------------------------------------------------------------------------------------------
// backward, bias gradients: every partial summed in a fixed order and added into the caller's tensors.  Thread x < ntab:
// d_bias_table entry e of head h (x = h tabn + e) over the pass-1 CTAs of h, slice by slice; then (x - ntab < nglob) the
// global-bias entries over the images.  ntab / nglob are 0 when the kernel that writes those partials did not run.
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
simt_bwd_bias_reduce(Geo geo, const float* __restrict__ tpart, const float* __restrict__ gpart, float* __restrict__ d_table,
                     float* __restrict__ d_g2l, float* __restrict__ d_g2g, int ntab, int nglob) {
  long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int H = geo.H;
  float sum = 0.f;
  if (x < ntab) {
    const int tabn = ntab / H, h = (int)(x / tabn), e = (int)(x % tabn);
    const long long m = (long long)geo.mx * geo.my * geo.npc;   // pass-1 CTAs of one (slice, head)
    for (int s = 0; s < geo.nslice; ++s) {
      const float* p = tpart + ((long long)s * H + h) * m * tabn + e;
#pragma unroll 4
      for (long long c = 0; c < m; ++c) sum += p[c * tabn];
    }
    d_table[(long long)e * H + h] += sum;
    return;
  }
  x -= ntab;
  if (x >= nglob) return;
  const long long hg = (long long)H * geo.g, bhg = (long long)geo.B * hg;
  if (x < 2 * hg) {          // d_g2l[1] (simt_bwd_gcol), then d_g2l[0] (simt_bwd_grow); x % hg = h g + t
    const int part = x < hg ? 0 : 1;
    const long long i = x - part * hg;
    const float* p = gpart + part * bhg + i;
    for (int b = 0; b < geo.B; ++b) sum += p[b * hg];
    if (d_g2l != nullptr) d_g2l[(part == 0 ? hg : 0) + i] += sum;
  } else {                   // d_g2g: i = (h g + a) g + j
    const long long i = x - 2 * hg;
    const float* p = gpart + 2 * bhg + i;
    for (int b = 0; b < geo.B; ++b) sum += p[b * hg * geo.g];
    if (d_g2g != nullptr) d_g2g[i] += sum;
  }
}

// ----------------------------------------------------------------------------------------------
// Sized calls (per-image grids): exact zeros in the rows of the local tokens off image b's grid, which no other kernel
// writes -- row t + off[i] of each of the n outputs rows[i] -- and lse = -inf there (an empty softmax) when lse is
// given.  One warp per local row; E: an unsigned integer of the element's size (zero bits are 0 in fp32, bf16 and fp16).
// ----------------------------------------------------------------------------------------------
struct OffImageRows {
  T4 rows[5];
  int off[5];
  int n;
  float* lse;
};
template <typename E>
__global__ void __launch_bounds__(256)
simt_zero_off_image(Geo geo, OffImageRows z, const int* __restrict__ image_hw) {
  const long long nrows = (long long)geo.B * geo.H * geo.Nloc;
  const long long stride = (long long)gridDim.x * (blockDim.x >> 5);
  const int lane = threadIdx.x & 31;
  for (long long x = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); x < nrows; x += stride) {
    const long long t = x % geo.Nloc, bh = x / geo.Nloc;
    const int b = (int)(bh / geo.H), h = (int)(bh % geo.H);
    int ih, iw;
    image_extent(geo, image_hw, b, ih, iw);
    if (on_image(geo, ih, iw, t)) continue;                  // warp-uniform
    for (int i = 0; i < z.n; ++i)
      for (int c = lane; c < geo.D; c += 32) row_ptr_w<E>(z.rows[i], b, h, t + z.off[i])[c] = E(0);
    if (z.lse != nullptr && lane == 0) z.lse[x] = -INFINITY;
  }
}

// ---------------------------------------------------------------- host launchers (both kernel families)
// image_hw != NULL (a sized call) runs the SIZED instantiations
template <typename T, int HD, typename TO = T>
inline void launch_global_fwd_kernels(const Geo& g, T4 qg, T4 kg, T4 vg, T4 og, float* lse_g, const float* g2l,
                                      const float* g2g, const int* image_hw, cudaStream_t s) {
  const auto kernel = g.drop_p > 0.f ? (image_hw ? simt_fwd_global<T, HD, TO, true, true> : simt_fwd_global<T, HD, TO, true>)
                                     : (image_hw ? simt_fwd_global<T, HD, TO, false, true> : simt_fwd_global<T, HD, TO>);
  kernel<<<g.B * g.H * g.g, 256, 0, s>>>(g, qg, kg, vg, og, lse_g, g2l, g2g, image_hw);
}
template <typename T, int HD, typename TO = T>
inline void launch_global_bwd_kernels(const Geo& g, T4 q, T4 k, T4 v, T4 d_o, T4 dk, T4 dv, T4 qg, T4 kg, T4 vg, T4 d_og,
                                      T4 dqg, T4 dkg, T4 dvg, const float* lse, const float* delta, const float* lse_g,
                                      const float* delta_g, const float* g2l, const float* g2g, float* gpart,
                                      int accumulate, int rmw_rows, const int* image_hw, cudaStream_t s) {
  // gpart: the global-bias partials (vil_common.cuh, ws_off_glob), read only with the bias table
  const long long bhg = (long long)g.B * g.H * g.g;
  float* pcol = gpart;
  float* prow = gpart ? gpart + bhg : nullptr;
  float* pgg = gpart ? gpart + 2 * bhg : nullptr;
  const bool drop = g.drop_p > 0.f;
  const auto gcol = drop ? (image_hw ? simt_bwd_gcol<T, HD, TO, true, true> : simt_bwd_gcol<T, HD, TO, true>)
                         : (image_hw ? simt_bwd_gcol<T, HD, TO, false, true> : simt_bwd_gcol<T, HD, TO>);
  const auto grow = drop ? (image_hw ? simt_bwd_grow<T, HD, TO, true, true> : simt_bwd_grow<T, HD, TO, true>)
                         : (image_hw ? simt_bwd_grow<T, HD, TO, false, true> : simt_bwd_grow<T, HD, TO>);
  gcol<<<g.B * g.H * g.g, 256, 0, s>>>(g, q, k, v, d_o, dk, dv, lse, delta, g2l, pcol, image_hw);
  grow<<<g.B * g.H, 256, 0, s>>>(g, qg, kg, vg, d_og, dqg, dkg, dvg, lse_g, delta_g, g2l, g2g, prow, pgg, accumulate, rmw_rows,
                                 image_hw);
}

}  // namespace vil
