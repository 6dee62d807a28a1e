// TU: C-ABI entry points of the residual / LayerNorm / bias epilogue kernels (vil_epilogue.cuh; include/vil_attn.h).
// Host side only: validation, grid sizing (multiples of the 132 SMs of an H100 SXM), launches on the caller's stream.  No allocation.
#include <cstdio>
#include <cstdlib>
#include "vil_host.cuh"
#include "vil_epilogue.cuh"

namespace {

using namespace vil;

constexpr int kSMs = 132;

int efail(int code, const char* msg) { return shared_fail(code, msg); }

// ---------------------------------------------------------------------------------------------------------- addnorm
inline int an_bwd_grid(long long rows) {
  long long g = rows / (epi::kWarps * 32);          // >= 32 rows per warp: the per-CTA partial rows stay <= 1/32 of the stream
  if (g < kSMs * 2) g = kSMs * 2;
  if (g > kSMs * 12) g = kSMs * 12;
  return (int)g;
}

int an_check(const VilAddNormParams* p, bool bwd) {
  if (p == nullptr) return efail(VIL_E_BADARG, "params is NULL");
  if (p->struct_bytes != (int32_t)sizeof(VilAddNormParams)) return efail(VIL_E_BADARG, "VilAddNormParams size mismatch");
  if (p->C <= 0 || p->C > 1024 || p->C % 4 != 0) return efail(VIL_E_UNSUPPORTED, "addnorm supports C % 4 == 0, C <= 1024");
  if (p->rows < 0) return efail(VIL_E_BADARG, "rows must be >= 0");
  if (p->b_dtype < 0 || p->b_dtype > 2 || p->y_dtype < 0 || p->y_dtype > 2) return efail(VIL_E_BADARG, "bad dtype");
  if (p->rows == 0) return VIL_OK;                  // empty stream: nothing is read or launched (empty tensors have NULL data)
  if (p->br != nullptr && p->b_dtype != p->y_dtype && p->b_dtype != VIL_F32 && p->y_dtype != VIL_F32)
    return efail(VIL_E_UNSUPPORTED, "addnorm: br and y must share their low-precision type");
  // 128-bit accesses to the fp32 rows and gamma, 64-bit ones to the low-precision rows: one rule for every pointer of the call
  // (checked before the NULL checks, so that a refused call never depends on which other tensors were given)
  const uintptr_t al = !bwd
      ? ((uintptr_t)p->x | (uintptr_t)p->br | (uintptr_t)p->bias | (uintptr_t)p->rowscale | (uintptr_t)p->gamma |
         (uintptr_t)p->beta | (uintptr_t)p->xo | (uintptr_t)p->y | (uintptr_t)p->mean | (uintptr_t)p->rstd)
      : ((uintptr_t)p->x | (uintptr_t)p->gamma | (uintptr_t)p->beta | (uintptr_t)p->rowscale | (uintptr_t)p->mean |
         (uintptr_t)p->rstd | (uintptr_t)p->dy | (uintptr_t)p->gres | (uintptr_t)p->dx | (uintptr_t)p->dbr |
         (uintptr_t)p->dgamma | (uintptr_t)p->dbeta | (uintptr_t)p->dbias | (uintptr_t)p->workspace);
  if (al & 15) return efail(VIL_E_BADARG, "addnorm: tensors must be 16-byte aligned");
  if (!p->x || !p->gamma || !p->beta || !p->mean || !p->rstd) return efail(VIL_E_BADARG, "addnorm: NULL tensor");
  if (p->rowscale != nullptr && p->rows_per_sample <= 0) return efail(VIL_E_BADARG, "addnorm: rows_per_sample must be positive");
  if (!bwd) {
    if (!p->y || (p->br != nullptr && !p->xo)) return efail(VIL_E_BADARG, "addnorm: NULL output");
  } else {
    if (!p->dy || !p->dx || !p->dgamma || !p->dbeta) return efail(VIL_E_BADARG, "addnorm backward: NULL tensor");
    if (!p->workspace || p->workspace_bytes < vil_addnorm_workspace_bytes(p))
      return efail(VIL_E_WORKSPACE, "addnorm workspace too small");
  }
  return VIL_OK;
}

epi::AddNormArgs an_args(const VilAddNormParams* p) {
  epi::AddNormArgs a;
  a.x = p->x; a.br = p->br; a.bias = p->bias; a.rowscale = p->rowscale; a.gamma = p->gamma; a.beta = p->beta;
  a.xo = p->xo; a.y = p->y; a.mean = p->mean; a.rstd = p->rstd;
  a.dy = p->dy; a.gres = p->gres; a.dx = p->dx; a.dbr = p->dbr; a.partial = static_cast<float*>(p->workspace);
  a.rows = p->rows; a.rows_per_sample = p->rows_per_sample > 0 ? p->rows_per_sample : 1; a.C = p->C; a.eps = p->eps;
  return a;
}

template <typename TB, typename TY, int L, int NVL>
int an_launch(const VilAddNormParams* p, cudaStream_t s, bool bwd) {
  if (p->rows == 0) return VIL_OK;
  const epi::AddNormArgs a = an_args(p);
  constexpr int RPW = 32 / L;                      // rows per warp
  const long long wrows = (p->rows + RPW - 1) / RPW;
  if (!bwd) {
    long long ctas = (wrows + epi::kWarps - 1) / epi::kWarps;
    if (ctas > kSMs * 16) ctas = kSMs * 16;
    epi::addnorm_fwd<TB, TY, L, NVL><<<(unsigned)ctas, epi::kAnThreads, 0, s>>>(a);
    count_launch();
  } else {
    const int grid = an_bwd_grid(p->rows);
    epi::addnorm_bwd<TB, TY, L, NVL><<<grid, epi::kAnThreads, 0, s>>>(a);
    count_launch();
    epi::colsum_reduce<<<(3 * p->C + 31) / 32, 256, 0, s>>>(a.partial, grid, 3, p->C, p->dgamma, p->dbeta,
                                                             p->dbr != nullptr ? p->dbias : nullptr);
    count_launch();
  }
  return launch_check("addnorm");
}

// lanes per row / vectors per lane: 3 vectors (48 B of fp32) per lane up to 384 channels, then 32 lanes with more vectors
template <typename TB, typename TY>
int an_dispatch_c(const VilAddNormParams* p, cudaStream_t s, bool bwd) {
  const int C = p->C;
  if (C <= 48) return an_launch<TB, TY, 4, 3>(p, s, bwd);
  if (C <= 96) return an_launch<TB, TY, 8, 3>(p, s, bwd);
  if (C <= 192) return an_launch<TB, TY, 16, 3>(p, s, bwd);
  if (C <= 384) return an_launch<TB, TY, 32, 3>(p, s, bwd);
  if (C <= 512) return an_launch<TB, TY, 32, 4>(p, s, bwd);
  if (C <= 768) return an_launch<TB, TY, 32, 6>(p, s, bwd);
  return an_launch<TB, TY, 32, 8>(p, s, bwd);
}

int an_run(const VilAddNormParams* p, void* stream, bool bwd) {
  int rc = an_check(p, bwd);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // instantiated pairs: (br, y) both T, or y fp32 with br T (norms whose output stays in the fp32 stream), or all fp32
  const int bt = p->br != nullptr || p->dbr != nullptr ? p->b_dtype : p->y_dtype;
  if (p->y_dtype == VIL_F32) {
    if (bt == VIL_BF16) return an_dispatch_c<__nv_bfloat16, float>(p, s, bwd);
    if (bt == VIL_F16) return an_dispatch_c<__half, float>(p, s, bwd);
    return an_dispatch_c<float, float>(p, s, bwd);
  }
  if (p->y_dtype == VIL_BF16)
    return bt == VIL_F32 ? an_dispatch_c<float, __nv_bfloat16>(p, s, bwd) : an_dispatch_c<__nv_bfloat16, __nv_bfloat16>(p, s, bwd);
  return bt == VIL_F32 ? an_dispatch_c<float, __half>(p, s, bwd) : an_dispatch_c<__half, __half>(p, s, bwd);
}

// ---------------------------------------------------------------------------------------------------------- bias + act
struct BaPlan { int gs, ncs; long long rows_per_slab; int nrs; };

BaPlan ba_plan(const VilBiasActParams* p) {
  const int n = p->dtype == VIL_F32 ? 4 : 8;
  const int G = p->C / n;
  BaPlan b;
  b.ncs = (G + epi::kThreads - 1) / epi::kThreads;
  b.gs = (G + b.ncs - 1) / b.ncs;
  const int rpi = epi::kThreads / b.gs;
  long long want = (kSMs * 8) / b.ncs;                      // row slabs: ~8 CTAs per SM in total
  long long per = (p->rows + want - 1) / want;
  if (per < 4LL * rpi) per = 4LL * rpi;                     // at least a few iterations per thread
  b.rows_per_slab = per;
  b.nrs = (int)((p->rows + per - 1) / per);
  if (b.nrs < 1) b.nrs = 1;
  return b;
}

int ba_check(const VilBiasActParams* p, bool bwd) {
  if (p == nullptr) return efail(VIL_E_BADARG, "params is NULL");
  if (p->struct_bytes != (int32_t)sizeof(VilBiasActParams)) return efail(VIL_E_BADARG, "VilBiasActParams size mismatch");
  if (p->dtype < 0 || p->dtype > 2) return efail(VIL_E_BADARG, "bad dtype");
  const int n = p->dtype == VIL_F32 ? 4 : 8;
  if (p->C <= 0 || p->C % n != 0) return efail(VIL_E_UNSUPPORTED, "bias_act: a row must be a whole number of 16-byte vectors");
  if (p->rows < 0) return efail(VIL_E_BADARG, "rows must be >= 0");
  if (p->act != VIL_ACT_NONE && p->act != VIL_ACT_GELU) return efail(VIL_E_BADARG, "bias_act: unknown activation");
  if (p->rows == 0 && !(bwd && !p->dbias)) return VIL_OK;       // empty stream (d_bias is zero-filled by the launcher)
  if (!bwd) {
    if (!p->z || !p->a) return efail(VIL_E_BADARG, "bias_act: NULL tensor");
  } else {
    if (!p->da || !p->dbias) return efail(VIL_E_BADARG, "bias_act backward: NULL tensor");
    if (p->act != VIL_ACT_NONE && (!p->z || !p->dz)) return efail(VIL_E_BADARG, "bias_act backward: z / dz needed for the activation");
    if (!p->workspace || p->workspace_bytes < vil_bias_act_workspace_bytes(p))
      return efail(VIL_E_WORKSPACE, "bias_act workspace too small");
  }
  const uintptr_t al = (uintptr_t)p->z | (uintptr_t)p->a | (uintptr_t)p->da | (uintptr_t)p->dz | (uintptr_t)p->bias;
  if (al & 15) return efail(VIL_E_BADARG, "bias_act: tensors must be 16-byte aligned");
  return VIL_OK;
}

template <typename T>
int ba_launch(const VilBiasActParams* p, cudaStream_t s, bool bwd) {
  if (p->rows == 0) {
    if (bwd) cudaMemsetAsync(p->dbias, 0, (size_t)p->C * 4, s);
    return VIL_OK;
  }
  constexpr int N = epi::Vec16<T>::N;
  const T* z = static_cast<const T*>(p->z);
  if (!bwd) {
    const long long nvec = p->rows * (p->C / N);
    long long ctas = (nvec + epi::kThreads * 4 - 1) / (epi::kThreads * 4);      // 4 vectors per thread and iteration
    if (ctas > kSMs * 8) ctas = kSMs * 8;
    if (p->act == VIL_ACT_GELU) epi::bias_act_fwd<T, 1><<<(unsigned)ctas, epi::kThreads, 0, s>>>(z, p->bias, static_cast<T*>(p->a), nvec, p->C);
    else                        epi::bias_act_fwd<T, 0><<<(unsigned)ctas, epi::kThreads, 0, s>>>(z, p->bias, static_cast<T*>(p->a), nvec, p->C);
    count_launch();
  } else {
    const BaPlan b = ba_plan(p);
    float* partial = static_cast<float*>(p->workspace);
    dim3 grid(b.ncs, b.nrs);
    if (p->act == VIL_ACT_GELU)
      epi::bias_act_bwd<T, 1><<<grid, epi::kThreads, 0, s>>>(z, p->bias, static_cast<const T*>(p->da), static_cast<T*>(p->dz), partial,
                                                             p->rows, p->C, b.gs, b.rows_per_slab);
    else
      epi::bias_act_bwd<T, 0><<<grid, epi::kThreads, 0, s>>>(z, p->bias, static_cast<const T*>(p->da), static_cast<T*>(p->dz), partial,
                                                             p->rows, p->C, b.gs, b.rows_per_slab);
    count_launch();
    epi::colsum_reduce<<<(p->C + 31) / 32, 256, 0, s>>>(partial, b.nrs, 1, p->C, p->dbias, nullptr, nullptr);
    count_launch();
  }
  return launch_check("bias_act");
}

int ba_run(const VilBiasActParams* p, void* stream, bool bwd) {
  int rc = ba_check(p, bwd);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (p->dtype == VIL_F32) return ba_launch<float>(p, s, bwd);
  if (p->dtype == VIL_BF16) return ba_launch<__nv_bfloat16>(p, s, bwd);
  return ba_launch<__half>(p, s, bwd);
}

}  // namespace

extern "C" {

int64_t vil_addnorm_workspace_bytes(const VilAddNormParams* p) {
  if (p == nullptr || p->C <= 0) return VIL_E_BADARG;
  return (int64_t)an_bwd_grid(p->rows) * 3 * p->C * 4 + 256;
}
int vil_addnorm_fwd_sm100(const VilAddNormParams* p, void* stream) { return an_run(p, stream, false); }
int vil_addnorm_bwd_sm100(const VilAddNormParams* p, void* stream) { return an_run(p, stream, true); }

int64_t vil_bias_act_workspace_bytes(const VilBiasActParams* p) {
  if (p == nullptr || p->C <= 0 || p->dtype < 0 || p->dtype > 2 || p->C % (p->dtype == VIL_F32 ? 4 : 8) != 0) return VIL_E_BADARG;
  const BaPlan b = ba_plan(p);
  return (int64_t)b.nrs * p->C * 4 + 256;
}
int vil_bias_act_fwd_sm100(const VilBiasActParams* p, void* stream) { return ba_run(p, stream, false); }
int vil_bias_act_bwd_sm100(const VilBiasActParams* p, void* stream) { return ba_run(p, stream, true); }

}  // extern "C"
