// Translation unit of the SIMT (CUDA-core) kernel family + the global-token / delta kernels both families share.
#include <algorithm>
#include <cstdio>
#include <type_traits>
#include "vil_host.cuh"
#include "vil_simt.cuh"

namespace vil {
namespace {

int head_bucket(int D) { return D <= 8 ? 8 : D <= 16 ? 16 : D <= 32 ? 32 : D <= 64 ? 64 : 128; }

// HS: floats per tile row (Tile<HD, L>::HS)
size_t simt_tile_smem(const Geo& g, int HS, bool dkv) {
  const int tw = 4 * g.w - 1;
  size_t bytes = (size_t)(2 * 64 * HS + (g.has_bias ? tw * tw : 0)) * sizeof(float);
  if (dkv) bytes += 2 * 64 * sizeof(float);
  bytes += 64 * 2 * sizeof(short) + 64;
  if (dkv && g.drop_p > 0.f) bytes += 64 * sizeof(int);          // the query token of each column (dropout rows)
  return (bytes + 15) & ~size_t(15);
}

template <typename K>
int set_smem(K kernel, size_t bytes) {
  if (bytes > 48 * 1024) {
    if (bytes > 227 * 1024) return shared_fail(VIL_E_UNSUPPORTED, "configuration needs more than 227 KB of shared memory");
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return shared_fail(VIL_E_CUDA, cudaGetErrorString(e));
  }
  return VIL_OK;
}

inline float* ws_delta(const VilAttnParams* p) { return static_cast<float*>(p->workspace); }
inline float* ws_delta_g(const VilAttnParams* p, const Geo& g) { return static_cast<float*>(p->workspace) + ws_off_delta_g(g); }

// ------------------------------------------------------------------ shared global-token kernels
// a dilated (g.d > 1) or sized call runs the DIL instantiations over the residue sub-grids of each image
// (vil_common.cuh, SubGrid)
inline bool sub_grids(const Geo& g, const int* image_hw) { return g.d > 1 || image_hw != nullptr; }

template <typename T, int HD, typename TO>
int global_fwd_t(const VilAttnParams* p, const Geo& g, cudaStream_t s, const int* hw) {
  launch_global_fwd_kernels<T, HD, TO>(g, t4(p->qg), t4(p->kg), t4(p->vg), t4(p->og), p->lse_g, p->g2l, p->g2g, hw, s);
  count_launch();
  return launch_check("simt_fwd_global");
}

template <typename T, typename TO>
int delta_t(const VilAttnParams* p, const Geo& g, cudaStream_t s) {
  const long long rows = (long long)g.B * g.H * (g.Nloc + g.g);
  simt_bwd_delta<T, TO><<<(unsigned)((rows + 63) / 64), 256, 0, s>>>(g, t4(p->o), t4(p->d_o), t4(p->og), t4(p->d_og),
                                                                      ws_delta(p), ws_delta_g(p, g));
  count_launch();
  return launch_check("simt_bwd_delta");
}

template <typename T, int HD, typename TO>
int global_bwd_t(const VilAttnParams* p, const Geo& g, cudaStream_t s, int rmw_rows, const int* hw) {
  const bool shared = (p->kg.ptr == p->k.ptr) && (p->vg.ptr == p->v.ptr);
  launch_global_bwd_kernels<T, HD, TO>(g, t4(p->q), t4(p->k), t4(p->v), t4(p->d_o), t4(p->dk), t4(p->dv), t4(p->qg), t4(p->kg),
                                       t4(p->vg), t4(p->d_og), t4(p->dqg), t4(shared ? p->dk : p->dkg),
                                       t4(shared ? p->dv : p->dvg), p->lse, ws_delta(p), p->lse_g, ws_delta_g(p, g), p->g2l,
                                       p->g2g, g.has_bias ? ws_at(p, ws_off_glob(g)) : nullptr, shared ? 1 : 0, rmw_rows, hw, s);
  count_launch();
  count_launch();
  return launch_check("simt_bwd_gcol / simt_bwd_grow");
}

// dispatch on (element type, output type, head-dim bucket); F: functor template with operator()<T, HD, TO>()
#define VIL_SIMT_HD(T, TO, CALL)                                   \
  switch (head_bucket(g.D)) {                                      \
    case 8:   return CALL(T, 8, TO);                               \
    case 16:  return CALL(T, 16, TO);                              \
    case 32:  return CALL(T, 32, TO);                              \
    case 64:  return CALL(T, 64, TO);                              \
    default:  return CALL(T, 128, TO);                             \
  }
#define VIL_SIMT_TYPES(HDM, CALL)                                                                   \
  if (p->dtype == VIL_F32) { HDM(float, float, CALL) }                                         \
  if (p->dtype == VIL_BF16) {                                                                  \
    if (out_f32(p)) { HDM(__nv_bfloat16, float, CALL) }                                        \
    HDM(__nv_bfloat16, __nv_bfloat16, CALL)                                                    \
  }                                                                                            \
  if (out_f32(p)) { HDM(__half, float, CALL) }                                                 \
  HDM(__half, __half, CALL)

// ------------------------------------------------------------------ SIMT family proper
// L: lanes per row of the local-query kernels (vil_simt.cuh).  fp32 backward and dropout at 64 < D <= 128 run four (two
// would spill); the forward without dropout runs two at every head dim.  bf16 / fp16 train at those head dims on the
// wgmma family.
template <typename T, int HD, bool DROP>
int simt_forward(const VilAttnParams* p, const Geo& g, cudaStream_t s, const int* hw) {
  if constexpr (DROP && HD > 64 && !std::is_same<T, float>::value) {   // the bf16 / fp16 backward stops at 64 as well
    return shared_fail(VIL_E_UNSUPPORTED, "attention dropout supports head dim <= 64");
  } else {
  constexpr int L = DROP && std::is_same<T, float>::value && HD > 64 ? 4 : 2;
  const auto kernel = sub_grids(g, hw) ? simt_fwd_local<T, HD, L, DROP, true> : simt_fwd_local<T, HD, L, DROP>;
  const size_t sm = simt_tile_smem(g, Tile<HD, L>::HS, false);
  int rc = set_smem(kernel, sm);
  if (rc) return rc;
  const long long blocks = (long long)g.B * g.H * g.mx * g.my * g.npc;
  if (!(p->skip_mask & 2)) {
    kernel<<<(unsigned)blocks, 64 * L, sm, s>>>(g, t4(p->q), t4(p->k), t4(p->v), t4(p->o), p->lse, p->bias_table, p->g2l, hw);
    count_launch();
  }
  if (g.g > 0 && !(p->skip_mask & 1)) {
    if ((rc = global_fwd_t<T, HD, T>(p, g, s, hw))) return rc;
  }
  return launch_check("simt forward");
  }
}

// backward pass 1; TAB (the bias table): nslice image slices per (head, chunk, piece), table partials into the workspace
template <typename T, int HD, int L, bool DROP, bool TAB>
int simt_dq_pass(const VilAttnParams* p, const Geo& g, cudaStream_t s, const int* hw) {
  const auto kernel = sub_grids(g, hw) ? simt_bwd_dq<T, HD, L, DROP, TAB, true> : simt_bwd_dq<T, HD, L, DROP, TAB>;
  const size_t sm = simt_tile_smem(g, Tile<HD, L>::HS, false) + (TAB ? simt_ds_tile_bytes() : 0);
  int rc = set_smem(kernel, sm);
  if (rc) return rc;
  const long long ctas = TAB ? tab_ctas(g) : (long long)g.B * g.H * g.mx * g.my * g.npc;
  kernel<<<(unsigned)ctas, 64 * L, sm, s>>>(g, t4(p->q), t4(p->k), t4(p->v), t4(p->d_o), t4(p->dq), p->lse, ws_delta(p),
                                            p->bias_table, p->g2l, TAB ? ws_at(p, ws_off_tab(g)) : nullptr, hw);
  count_launch();
  return VIL_OK;
}

template <typename T, int HD, bool DROP>
int simt_backward(const VilAttnParams* p, const Geo& g, cudaStream_t s, const int* hw) {
  if constexpr (HD > 64 && !std::is_same<T, float>::value) {
    return shared_fail(VIL_E_UNSUPPORTED,
                       "the SIMT backward supports head dim <= 64; 64 < D <= 128 is trained by the wgmma family "
                       "(bf16 / fp16 with 16-byte-aligned rows)");
  } else {
    constexpr int L = std::is_same<T, float>::value && HD > 64 ? 4 : 2;
    int rc = (p->skip_mask & 8) ? VIL_OK : delta_t<T, T>(p, g, s);
    if (rc) return rc;
    const auto dkv = sub_grids(g, hw) ? simt_bwd_dkv<T, HD, L, DROP, true> : simt_bwd_dkv<T, HD, L, DROP>;
    const size_t sm2 = simt_tile_smem(g, Tile<HD, L>::HS, true);
    if ((rc = set_smem(dkv, sm2))) return rc;
    const long long blocks = (long long)g.B * g.H * g.mx * g.my * g.npc;
    if (!(p->skip_mask & 2)) {
      if ((rc = g.has_bias ? simt_dq_pass<T, HD, L, DROP, true>(p, g, s, hw) : simt_dq_pass<T, HD, L, DROP, false>(p, g, s, hw)))
        return rc;
    }
    if (!(p->skip_mask & 4)) {
      dkv<<<(unsigned)blocks, 64 * L, sm2, s>>>(g, t4(p->q), t4(p->k), t4(p->v), t4(p->d_o), t4(p->dk), t4(p->dv), p->lse,
                                                ws_delta(p), p->bias_table, hw);
      count_launch();
    }
    if (g.g > 0 && !(p->skip_mask & 1)) {
      if ((rc = global_bwd_t<T, HD, T>(p, g, s, g.N, hw))) return rc;
    }
    if ((rc = launch_check("simt backward"))) return rc;
    return simt_bias_reduce(p, g, s);
  }
}

template <typename T, bool DROP>
int simt_dispatch_hd(const VilAttnParams* p, const Geo& g, cudaStream_t s, bool bwd, const int* hw) {
  switch (head_bucket(g.D)) {
    case 8:   return bwd ? simt_backward<T, 8, DROP>(p, g, s, hw) : simt_forward<T, 8, DROP>(p, g, s, hw);
    case 16:  return bwd ? simt_backward<T, 16, DROP>(p, g, s, hw) : simt_forward<T, 16, DROP>(p, g, s, hw);
    case 32:  return bwd ? simt_backward<T, 32, DROP>(p, g, s, hw) : simt_forward<T, 32, DROP>(p, g, s, hw);
    case 64:  return bwd ? simt_backward<T, 64, DROP>(p, g, s, hw) : simt_forward<T, 64, DROP>(p, g, s, hw);
    default:  return bwd ? simt_backward<T, 128, DROP>(p, g, s, hw) : simt_forward<T, 128, DROP>(p, g, s, hw);
  }
}

template <typename T>
int simt_dispatch(const VilAttnParams* p, const Geo& g, cudaStream_t s, bool bwd, const int* hw) {
  return g.drop_p > 0.f ? simt_dispatch_hd<T, true>(p, g, s, bwd, hw) : simt_dispatch_hd<T, false>(p, g, s, bwd, hw);
}

}  // namespace

int simt_run(const VilAttnParams* p, const Geo& g, cudaStream_t s, bool bwd, const int* image_hw) {
  if (out_f32(p) && p->dtype != VIL_F32)
    return shared_fail(VIL_E_UNSUPPORTED, "VIL_FLAG_F32_OUT (parity build) is implemented by the wgmma family only");
  switch (p->dtype) {
    case VIL_F32:  return simt_dispatch<float>(p, g, s, bwd, image_hw);
    case VIL_BF16: return simt_dispatch<__nv_bfloat16>(p, g, s, bwd, image_hw);
    default:       return simt_dispatch<__half>(p, g, s, bwd, image_hw);
  }
}

int simt_global_fwd(const VilAttnParams* p, const Geo& g, cudaStream_t s, const int* image_hw) {
#define CALL_GF(T, HD, TO) global_fwd_t<T, HD, TO>(p, g, s, image_hw)
  VIL_SIMT_TYPES(VIL_SIMT_HD, CALL_GF)
#undef CALL_GF
}

int simt_delta(const VilAttnParams* p, const Geo& g, cudaStream_t s) {
  if (p->dtype == VIL_F32) return delta_t<float, float>(p, g, s);
  if (p->dtype == VIL_BF16) return out_f32(p) ? delta_t<__nv_bfloat16, float>(p, g, s) : delta_t<__nv_bfloat16, __nv_bfloat16>(p, g, s);
  return out_f32(p) ? delta_t<__half, float>(p, g, s) : delta_t<__half, __half>(p, g, s);
}

int simt_bias_reduce(const VilAttnParams* p, const Geo& g, cudaStream_t s) {
  if (!g.has_bias) return VIL_OK;
  // only the partials of kernels that ran (skip_mask) are summed
  const long long ntab = (p->skip_mask & 2) ? 0 : (long long)table_entries(g) * g.H;
  const long long nglob = (g.g == 0 || (p->skip_mask & 1)) ? 0 : (long long)g.H * g.g * (2 + g.g);
  if (ntab + nglob == 0) return VIL_OK;
  simt_bwd_bias_reduce<<<(unsigned)((ntab + nglob + 255) / 256), 256, 0, s>>>(
      g, ws_at(p, ws_off_tab(g)), ws_at(p, ws_off_glob(g)), p->d_bias_table, p->d_g2l, p->d_g2g, (int)ntab, (int)nglob);
  count_launch();
  return launch_check("simt_bwd_bias_reduce");
}

int simt_global_bwd(const VilAttnParams* p, const Geo& g, cudaStream_t s, int rmw_rows, const int* image_hw) {
#define CALL_GB(T, HD, TO) global_bwd_t<T, HD, TO>(p, g, s, rmw_rows, image_hw)
  VIL_SIMT_TYPES(VIL_SIMT_HD, CALL_GB)
#undef CALL_GB
}

int simt_zero_off_image(const VilAttnParams* p, const Geo& g, cudaStream_t s, bool bwd, const int* image_hw) {
  OffImageRows z{};
  if (!bwd) {
    z.rows[0] = t4(p->o);
    z.n = 1;
    z.lse = p->lse;
  } else {
    const VilTensor4* out[5] = {&p->dq, &p->dk, &p->dv, &p->dkg, &p->dvg};
    const bool shared = (p->kg.ptr == p->k.ptr) && (p->vg.ptr == p->v.ptr);
    z.n = g.g > 0 && !shared ? 5 : 3;                 // separate global keys: dkg / dvg have local rows too
    for (int i = 0; i < z.n; ++i) { z.rows[i] = t4(*out[i]); z.off[i] = i == 0 ? 0 : g.g; }
  }
  const bool wide = p->dtype == VIL_F32 || out_f32(p);   // the outputs' element size: 4 or 2 bytes
  const long long rows = (long long)g.B * g.H * g.Nloc;
  const unsigned ctas = (unsigned)std::min<long long>((rows + 7) / 8, 132LL * 16);
  if (wide) simt_zero_off_image<uint32_t><<<ctas, 256, 0, s>>>(g, z, image_hw);
  else simt_zero_off_image<uint16_t><<<ctas, 256, 0, s>>>(g, z, image_hw);
  count_launch();
  return launch_check("simt_zero_off_image");
}

}  // namespace vil
