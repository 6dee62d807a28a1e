// C-ABI entry points of libvil_attn.so (see include/vil_attn.h).
// Host-side only: argument validation (mirroring the reference's asserts / ValueErrors,
// longformer2d.py:22,45-46,111 and slidingchunk_2d.py:331-343), geometry set-up, kernel
// family selection and launches on the caller's stream.  No allocation, no host sync.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "vil_host.cuh"
#include "vil_layernorm.cuh"

namespace {

constexpr int kSMs = 132;                       // H100 SXM

thread_local char g_err[512] = "";
thread_local const char* g_last_impl = "none";
thread_local const char* g_last_kernel = "";
std::atomic<long long> g_launches{0};

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

#define VIL_CUDA_OK(expr)                                                                  \
  do {                                                                                     \
    cudaError_t e__ = (expr);                                                              \
    if (e__ != cudaSuccess) return fail(VIL_E_CUDA, "%s: %s", #expr, cudaGetErrorString(e__)); \
  } while (0)

#define VIL_LAUNCHED() g_launches.fetch_add(1, std::memory_order_relaxed)

int make_geo(const VilAttnParams* p, vil::Geo* g) {
  if (p == nullptr) return fail(VIL_E_BADARG, "params is NULL");
  if (p->struct_bytes != (int32_t)sizeof(VilAttnParams))
    return fail(VIL_E_BADARG, "VilAttnParams size mismatch: caller %d, library %d (ABI drift)", p->struct_bytes,
                (int)sizeof(VilAttnParams));
  if (p->dtype != VIL_F32 && p->dtype != VIL_BF16 && p->dtype != VIL_F16)
    return fail(VIL_E_BADARG, "dtype must be VIL_F32, VIL_BF16 or VIL_F16");
  if (p->B <= 0 || p->H <= 0 || p->D <= 0 || p->nx <= 0 || p->ny <= 0 || p->w <= 0 || p->nglo < 0)
    return fail(VIL_E_BADARG, "B, H, D, nx, ny, w must be positive and nglo non-negative");
  // mask_invalid_locations: "longsc exact should be in [0,1,-1]!" (slidingchunk_2d.py:343)
  if (p->exact != 0 && p->exact != 1 && p->exact != -1)
    return fail(VIL_E_BADARG, "longsc exact should be in [0,1,-1]!");
  if (p->mode < -1 || p->mode > 8) return fail(VIL_E_BADARG, "mode must be in [-1, 8]");
  if (p->flags & ~(VIL_FLAG_F32_OUT | VIL_FLAG_UNFUSED | VIL_FLAG_F32_SPLIT | VIL_FLAG_DILATED))
    return fail(VIL_E_BADARG, "unknown bits in flags");
  const int d = (p->flags & VIL_FLAG_DILATED) ? p->dilation : 1;
  if (d < 1) return fail(VIL_E_BADARG, "dilation must be >= 1 with VIL_FLAG_DILATED (got %d)", p->dilation);
  if ((p->flags & VIL_FLAG_F32_OUT) && p->dtype == VIL_F32)
    return fail(VIL_E_BADARG, "VIL_FLAG_F32_OUT is the parity build of the bf16 / fp16 kernels; dtype is already fp32");
  if ((p->flags & VIL_FLAG_F32_SPLIT) && p->dtype != VIL_F32)
    return fail(VIL_E_BADARG, "VIL_FLAG_F32_SPLIT applies to fp32 operands only (dtype must be VIL_F32)");
  // the exact mask has 9*w^2 columns only: exact=1 with mode != 0 raises in the reference (:331-343)
  if (p->exact == 1 && p->mode != 0)
    return fail(VIL_E_BADARG, "exact sliding window (exact=1) only supports mode=0");
  if (p->D > 128) return fail(VIL_E_UNSUPPORTED, "head dim %d > 128 is not supported", p->D);
  if (p->w > 48) return fail(VIL_E_UNSUPPORTED, "window %d > 48 is not supported", p->w);
  if ((long long)p->nx * p->ny + p->nglo > 0x7fffffffLL / 4) return fail(VIL_E_UNSUPPORTED, "too many tokens");
  memset(g, 0, sizeof(*g));
  g->B = p->B; g->H = p->H; g->D = p->D;
  g->nx = p->nx; g->ny = p->ny; g->w = p->w; g->g = p->nglo; g->exact = p->exact; g->mode = p->mode;
  g->padx = (p->w - p->nx % p->w) % p->w;
  g->pady = (p->w - p->ny % p->w) % p->w;
  g->mx = (p->nx + g->padx) / p->w;
  g->my = (p->ny + g->pady) / p->w;
  g->d = d;
  if (d > 1) {   // the virtual chunk grid of the d^2 residue sub-grids (vil_common.cuh, SubGrid): d x the largest one's
    const int nx0 = (p->nx + d - 1) / d, ny0 = (p->ny + d - 1) / d;
    g->mx = d * ((nx0 + p->w - 1) / p->w);
    g->my = d * ((ny0 + p->w - 1) / p->w);
  }
  g->Nloc = p->nx * p->ny;
  g->N = g->Nloc + p->nglo;
  g->w2 = p->w * p->w;
  g->npc = (g->w2 + 63) / 64;
  static const int o9[9][2] = {{-1, -1}, {-1, 0}, {-1, 1}, {0, -1}, {0, 0}, {0, 1}, {1, -1}, {1, 0}, {1, 1}};
  static const int om[9][2] = {{0, 0}, {-1, -1}, {-1, 0}, {-1, 1}, {0, -1}, {0, 1}, {1, -1}, {1, 0}, {1, 1}};
  if (p->mode == 0) {
    g->noffs = 9;
    for (int i = 0; i < 9; ++i) { g->offR[i] = o9[i][0]; g->offC[i] = o9[i][1]; }
  } else if (p->mode == -1) {
    g->noffs = 1;
  } else {
    g->noffs = 2;
    g->offR[1] = om[p->mode][0]; g->offC[1] = om[p->mode][1];
  }
  g->has_bias = p->bias_table != nullptr;
  g->scale = p->scale;
  // pass-1 image slices with the bias table: about 8 CTAs per SM in all, several waves at the 2-4 CTAs per SM that the
  // pass-1 kernels fit, and never more slices than images
  const long long per_slice = (long long)p->H * g->mx * g->my * g->npc;
  g->nslice = (int)std::min<long long>(p->B, (8LL * kSMs + per_slice - 1) / per_slice);
  if (g->has_bias && p->nglo > 0 && (p->g2l == nullptr || p->g2g == nullptr))
    return fail(VIL_E_BADARG, "bias_table given but g2l / g2g missing while nglo > 0");
  // the reference creates the three bias parameters together (rpe, longformer2d.py:68-100): every kernel family keys them on
  // the table, so g2l / g2g without a table would be applied by some kernels and ignored by others
  if (!g->has_bias && (p->g2l != nullptr || p->g2g != nullptr))
    return fail(VIL_E_BADARG, "g2l / g2g given without bias_table (rpe parameters come together)");
  if (!(p->dropout_p >= 0.f && p->dropout_p < 1.f))   // also rejects NaN
    return fail(VIL_E_BADARG, "dropout_p must be in [0, 1) (got %g)", (double)p->dropout_p);
  g->drop_p = p->dropout_p;
  g->drop_scale = 1.0f / (1.0f - p->dropout_p);
  const double t = std::floor((double)p->dropout_p * 4294967296.0);
  g->drop_thresh = t >= 4294967295.0 ? 0xffffffffu : (uint32_t)t;
  g->seed_lo = (uint32_t)(p->dropout_seed & 0xffffffffu);
  g->seed_hi = (uint32_t)(p->dropout_seed >> 32);
  g->drop_off = (uint32_t)p->dropout_offset;
  return VIL_OK;
}

int check_tensor(const VilTensor4& t, const char* name) {
  if (t.ptr == nullptr) return fail(VIL_E_BADARG, "tensor %s is NULL", name);
  return VIL_OK;
}

int check_common(const VilAttnParams* p, const vil::Geo& g, bool bwd) {
  int rc;
  if ((rc = check_tensor(p->q, "q")) || (rc = check_tensor(p->k, "k")) || (rc = check_tensor(p->v, "v")) ||
      (rc = check_tensor(p->o, "o")))
    return rc;
  if (p->lse == nullptr) return fail(VIL_E_BADARG, "lse is NULL");
  if (g.g > 0) {
    if ((rc = check_tensor(p->qg, "qg")) || (rc = check_tensor(p->kg, "kg")) || (rc = check_tensor(p->vg, "vg")) ||
        (rc = check_tensor(p->og, "og")))
      return rc;
    if (p->lse_g == nullptr) return fail(VIL_E_BADARG, "lse_g is NULL");
  }
  if (bwd) {
    if ((rc = check_tensor(p->d_o, "d_o")) || (rc = check_tensor(p->dq, "dq")) || (rc = check_tensor(p->dk, "dk")) ||
        (rc = check_tensor(p->dv, "dv")))
      return rc;
    if (g.g > 0) {
      if ((rc = check_tensor(p->d_og, "d_og")) || (rc = check_tensor(p->dqg, "dqg"))) return rc;
      const bool shared = (p->kg.ptr == p->k.ptr) && (p->vg.ptr == p->v.ptr);
      if (!shared && ((rc = check_tensor(p->dkg, "dkg")) || (rc = check_tensor(p->dvg, "dvg")))) return rc;
    }
    const long long need = vil_attn_workspace_bytes(p, 1);
    if (p->workspace == nullptr || p->workspace_bytes < need)
      return fail(VIL_E_WORKSPACE, "workspace too small: need %lld bytes, got %lld", need,
                  (long long)p->workspace_bytes);
    if (g.has_bias && p->d_bias_table == nullptr) return fail(VIL_E_BADARG, "bias_table given but d_bias_table is NULL");
  }
  return VIL_OK;
}

// image_hw: the per-image grids of a sized call (device memory), NULL for the unsized entry points
int run(const VilAttnParams* p, void* stream, bool bwd, const int32_t* image_hw) {
  vil::Geo g;
  int rc = make_geo(p, &g);
  if (rc) return rc;
  if ((rc = check_common(p, g, bwd))) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int tc_ok = vil::tc_supported(p, g, bwd);
  int impl = p->impl;
  if (impl == VIL_IMPL_AUTO) impl = tc_ok ? VIL_IMPL_WGMMA : VIL_IMPL_SIMT;
  const char* name;
  if (impl == VIL_IMPL_WGMMA) {
    if (!tc_ok) return fail(VIL_E_UNSUPPORTED, "the wgmma family does not cover this configuration: %s", vil::tc_why_not(p, g, bwd));
    rc = bwd ? vil::tc_backward(p, g, s, image_hw) : vil::tc_forward(p, g, s, image_hw);
    name = "wgmma";
  } else {
    if (impl != VIL_IMPL_SIMT) return fail(VIL_E_BADARG, "impl must be VIL_IMPL_AUTO, _SIMT or _TCGEN05");
    rc = vil::simt_run(p, g, s, bwd, image_hw);
    name = "simt";
  }
  // the rows of off-image tokens, which the kernels above leave alone, get their zeros (and lse its -inf)
  if (rc == VIL_OK && image_hw != nullptr) rc = vil::simt_zero_off_image(p, g, s, bwd, image_hw);
  if (rc == VIL_OK) g_last_impl = name;
  return rc;
}

}  // namespace

namespace vil {
// hooks used by the wgmma family (vil_wgmma.cu) for the kernels it shares with the SIMT family
int shared_fail(int code, const char* msg) { return fail(code, "%s", msg); }
void count_launch() { VIL_LAUNCHED(); }
void note_kernel(const char* name) { g_last_kernel = name; }
}  // namespace vil

namespace {

// backward grid: enough warps to cover HBM latency (up to 8 CTAs x 8 warps per SM), fewer for short streams so the
// per-warp partial d_gamma / d_beta rows stay small next to the activations
inline int ln_bwd_grid(long long rows) {
  long long g = rows / (vil::ln::kWarpsPerCta * 16);
  if (g < kSMs) g = kSMs;
  if (g > kSMs * 8) g = kSMs * 8;
  return (int)g;
}

int ln_check(const VilLayerNormParams* p, bool bwd) {
  if (p == nullptr) return fail(VIL_E_BADARG, "params is NULL");
  if (p->struct_bytes != (int32_t)sizeof(VilLayerNormParams)) return fail(VIL_E_BADARG, "VilLayerNormParams size mismatch");
  if (p->C <= 0 || p->C > 1024) return fail(VIL_E_UNSUPPORTED, "LayerNorm supports 1 <= C <= 1024 (got %d)", p->C);
  if (p->rows < 0) return fail(VIL_E_BADARG, "rows must be >= 0");
  const bool same = p->x_dtype == p->y_dtype;
  const bool mixed = p->x_dtype == VIL_F32 && (p->y_dtype == VIL_BF16 || p->y_dtype == VIL_F16);
  // low-precision in -> fp32 out: the patch-embedding norm under autocast (bf16 Conv2d output -> fp32 residual stream)
  const bool widen = (p->x_dtype == VIL_BF16 || p->x_dtype == VIL_F16) && p->y_dtype == VIL_F32;
  if (!(same || mixed || widen) || p->x_dtype < 0 || p->x_dtype > 2) return fail(VIL_E_UNSUPPORTED, "unsupported LayerNorm dtype pair");
  if (!p->x || !p->gamma || !p->beta || !p->mean || !p->rstd) return fail(VIL_E_BADARG, "LayerNorm: NULL tensor");
  if (!bwd && !p->y) return fail(VIL_E_BADARG, "LayerNorm: y is NULL");
  if (bwd) {
    if (!p->dy || !p->dx || !p->dgamma || !p->dbeta) return fail(VIL_E_BADARG, "LayerNorm backward: NULL tensor");
    if (!p->workspace || p->workspace_bytes < vil_layernorm_workspace_bytes(p))
      return fail(VIL_E_WORKSPACE, "LayerNorm workspace too small");
  }
  return VIL_OK;
}

template <typename TX, typename TY, int NPL>
int ln_launch(const VilLayerNormParams* p, cudaStream_t s, bool bwd) {
  if (p->rows == 0) return VIL_OK;
  if (!bwd) {
    long long ctas = (p->rows + vil::ln::kWarpsPerCta - 1) / vil::ln::kWarpsPerCta;
    if (ctas > kSMs * 8) ctas = kSMs * 8;
    vil::ln::layernorm_fwd<TX, TY, NPL><<<(unsigned)ctas, vil::ln::kWarpsPerCta * 32, 0, s>>>(
        static_cast<const TX*>(p->x), p->gamma, p->beta, static_cast<TY*>(p->y), p->mean, p->rstd, p->rows, p->C, p->eps);
    VIL_LAUNCHED();
  } else {
    float* partial = static_cast<float*>(p->workspace);
    const int grid = ln_bwd_grid(p->rows);
    vil::ln::layernorm_bwd<TX, TY, NPL><<<grid, vil::ln::kWarpsPerCta * 32, 0, s>>>(
        static_cast<const TY*>(p->dy), static_cast<const TX*>(p->x), p->gamma, p->mean, p->rstd, static_cast<TX*>(p->dx),
        partial, p->rows, p->C);
    VIL_LAUNCHED();
    vil::ln::layernorm_bwd_reduce<<<(2 * p->C + 31) / 32, 256, 0, s>>>(partial, p->dgamma, p->dbeta, grid, p->C);
    VIL_LAUNCHED();
  }
  VIL_CUDA_OK(cudaGetLastError());
  return VIL_OK;
}

template <typename TX, typename TY>
int ln_dispatch_c(const VilLayerNormParams* p, cudaStream_t s, bool bwd) {
  const int npl = (p->C + 31) / 32;
  if (npl <= 3) return ln_launch<TX, TY, 3>(p, s, bwd);
  if (npl <= 6) return ln_launch<TX, TY, 6>(p, s, bwd);
  if (npl <= 12) return ln_launch<TX, TY, 12>(p, s, bwd);
  if (npl <= 24) return ln_launch<TX, TY, 24>(p, s, bwd);
  return ln_launch<TX, TY, 32>(p, s, bwd);
}

int ln_run(const VilLayerNormParams* p, void* stream, bool bwd) {
  int rc = ln_check(p, bwd);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (p->x_dtype == VIL_F32) {
    if (p->y_dtype == VIL_F32) return ln_dispatch_c<float, float>(p, s, bwd);
    if (p->y_dtype == VIL_BF16) return ln_dispatch_c<float, __nv_bfloat16>(p, s, bwd);
    return ln_dispatch_c<float, __half>(p, s, bwd);
  }
  if (p->x_dtype == VIL_BF16)
    return p->y_dtype == VIL_F32 ? ln_dispatch_c<__nv_bfloat16, float>(p, s, bwd) : ln_dispatch_c<__nv_bfloat16, __nv_bfloat16>(p, s, bwd);
  return p->y_dtype == VIL_F32 ? ln_dispatch_c<__half, float>(p, s, bwd) : ln_dispatch_c<__half, __half>(p, s, bwd);
}

}  // namespace

extern "C" {

int64_t vil_layernorm_workspace_bytes(const VilLayerNormParams* p) {
  if (p == nullptr || p->C <= 0) return VIL_E_BADARG;
  return (int64_t)ln_bwd_grid(p->rows) * 2 * p->C * 4 + 256;
}
int vil_layernorm_fwd_sm100(const VilLayerNormParams* p, void* stream) { return ln_run(p, stream, false); }
int vil_layernorm_bwd_sm100(const VilLayerNormParams* p, void* stream) { return ln_run(p, stream, true); }

#ifdef VIL_TRACE
// debug builds only: device buffer of 8 x 1024 (tag, clock) pairs filled by CTA 0 (tools/trace_timeline.py)
int vil_attn_debug_set_trace(void* dev_ptr) {
  long long* p = static_cast<long long*>(dev_ptr);
  return (int)cudaMemcpyToSymbol(g_vil_trace, &p, sizeof(p));
}
#endif

int vil_attn_abi_version(void) { return VIL_ATTN_ABI_VERSION; }
const char* vil_attn_last_error(void) { return g_err; }
int64_t vil_attn_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
const char* vil_attn_last_impl(void) { return g_last_impl; }
const char* vil_attn_last_kernel(void) { return g_last_kernel; }

int64_t vil_attn_workspace_bytes(const VilAttnParams* p, int backward) {
  vil::Geo g;
  int rc = make_geo(p, &g);
  if (rc) return rc;
  long long bytes = 256;
  if (backward) bytes += vil::ws_floats(g) * 4;
  return bytes;
}

int vil_attn_wgmma_supported(const VilAttnParams* p) {
  vil::Geo g;
  int rc = make_geo(p, &g);
  if (rc) return rc;
  return vil::tc_supported(p, g, false) ? 1 : 0;
}

int vil_attn_fwd_sm100(const VilAttnParams* p, void* stream) { return run(p, stream, false, nullptr); }
int vil_attn_bwd_sm100(const VilAttnParams* p, void* stream) { return run(p, stream, true, nullptr); }

int vil_attn_fwd_sized_sm100(const VilAttnParams* p, const int32_t* image_hw, void* stream) {
  if (image_hw == nullptr) return fail(VIL_E_BADARG, "image_hw is NULL (the sized entry points need the per-image grids)");
  return run(p, stream, false, image_hw);
}
int vil_attn_bwd_sized_sm100(const VilAttnParams* p, const int32_t* image_hw, void* stream) {
  if (image_hw == nullptr) return fail(VIL_E_BADARG, "image_hw is NULL (the sized entry points need the per-image grids)");
  return run(p, stream, true, image_hw);
}

}  // extern "C"
