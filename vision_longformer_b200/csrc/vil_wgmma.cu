// TU: coverage test and launches of the tensor-core (wgmma) kernel family (vil_wgmma.cuh).  The global query rows, the
// global key columns of the backward and delta = rowsum(dO * O) come from the shared SIMT kernels (vil_simt.cu).
#include <cstdio>
#include "vil_host.cuh"
#include "vil_wgmma.cuh"

namespace vil {
namespace {

int head_tile(int D) { return D <= 16 ? 16 : D <= 32 ? 32 : D <= 64 ? 64 : 128; }
int table_floats(const Geo& g) { return g.has_bias ? (4 * g.w - 1) * (4 * g.w - 1) : 0; }

template <typename K>
int set_smem(K kernel, size_t bytes) {
  if (bytes > 227 * 1024) return shared_fail(VIL_E_UNSUPPORTED, "configuration needs more than 227 KB of shared memory");
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) return shared_fail(VIL_E_CUDA, cudaGetErrorString(e));
  return VIL_OK;
}

// The kernels stage operand rows with 16-byte cp.async copies: every row of the view must start 16-byte aligned.
// e: bytes per element
bool rows_aligned16(const VilTensor4& t, long long e) {
  return reinterpret_cast<uintptr_t>(t.ptr) % 16 == 0 && (t.sb * e) % 16 == 0 && (t.sh * e) % 16 == 0 && (t.st * e) % 16 == 0;
}

// Shared memory of the call's kernels at head tile HD beside its bias table.  Every call checks all three kernels, so that
// a forward runs on this family only if its backward can as well.  Up to HD 64 everything fits up to the largest window
// (w = 48); at HD 128, and for split fp32 tiles at HD 64, the bias table fits up to w = 42, limited by pass 1 with its dS
// tile (DESIGN.md section 3).
template <typename T, int HD>
const char* smem_why_not(const Geo& g) {
  constexpr size_t cap = 227 * 1024;
  const int tabn = table_floats(g);
  if (wg::FwdSmem<T, HD>::total(tabn) > cap || wg::DkvSmem<T, HD>::total(tabn, g.drop_p > 0.f) > cap)
    return "bias table does not fit in shared memory";
  if (g.has_bias && wg::DqSmem<T, HD>::total(tabn, true) > cap)
    return "bias table and the dS tile of its gradient do not fit in shared memory";
  return nullptr;
}

template <typename T>
const char* smem_why_not_hd(const Geo& g) {
  switch (head_tile(g.D)) {
    case 16: return smem_why_not<T, 16>(g);
    case 32: return smem_why_not<T, 32>(g);
    case 64: return smem_why_not<T, 64>(g);
    default: return smem_why_not<T, 128>(g);
  }
}

const char* why_not(const VilAttnParams* p, const Geo& g, bool bwd) {
  const bool split = split_f32(p);
  if (p->dtype == VIL_F32 && !split) return "dtype is fp32 (wgmma operands are bf16 / fp16)";
  // split fp32 P / dS fragments next to the 128-column accumulators of pass 2 would spill
  if (split && g.D > 64) return "head dim > 64 with VIL_FLAG_F32_SPLIT (the split kernels have head tiles 16, 32 and 64)";
  const long long e = split ? 4 : 2;
  if (g.D % 8 != 0 || !rows_aligned16(p->q, e) || !rows_aligned16(p->k, e) || !rows_aligned16(p->v, e) ||
      (bwd && !rows_aligned16(p->d_o, e)))
    return "q / k / v / d_o rows are not 16-byte aligned (D % 8 != 0, or a pointer or b / h / t stride off 16 bytes)";
  return split ? smem_why_not_hd<float>(g) : smem_why_not_hd<__nv_bfloat16>(g);
}

long long blocks(const Geo& g) { return (long long)g.B * g.H * g.mx * g.my * g.npc; }

// a dilated (g.d > 1) or sized call runs the DIL instantiations over the residue sub-grids of each image
// (vil_common.cuh, SubGrid)
inline bool sub_grids(const Geo& g, const int* image_hw) { return g.d > 1 || image_hw != nullptr; }

template <typename T, int HD, typename TO, bool DROP>
int forward_t(const VilAttnParams* p, const Geo& g, cudaStream_t s, const int* image_hw) {
  int rc;
  if (!(p->skip_mask & 2)) {
    const size_t sm = wg::FwdSmem<T, HD>::total(table_floats(g));
    const auto kernel = sub_grids(g, image_hw) ? wg::wg_fwd_local<T, HD, TO, DROP, true> : wg::wg_fwd_local<T, HD, TO, DROP>;
    if ((rc = set_smem(kernel, sm))) return rc;
    kernel<<<(unsigned)blocks(g), wg::kThreads, sm, s>>>(g, t4(p->q), t4(p->k), t4(p->v), t4(p->o), p->lse, p->bias_table, p->g2l,
                                                         image_hw);
    count_launch();
    if ((rc = launch_check("wgmma_fwd_local"))) return rc;
  }
  if (g.g > 0 && !(p->skip_mask & 1)) return simt_global_fwd(p, g, s, image_hw);
  return VIL_OK;
}

// backward pass 1; TAB (the bias table): nslice image slices per (head, chunk, piece), table partials into the workspace
template <typename T, int HD, typename TO, bool DROP, bool TAB>
int dq_pass(const VilAttnParams* p, const Geo& g, cudaStream_t s, const int* image_hw) {
  int rc;
  const size_t sm = wg::DqSmem<T, HD>::total(table_floats(g), TAB);
  const auto kernel = sub_grids(g, image_hw) ? wg::wg_bwd_dq<T, HD, TO, DROP, TAB, true> : wg::wg_bwd_dq<T, HD, TO, DROP, TAB>;
  if ((rc = set_smem(kernel, sm))) return rc;
  const long long ctas = TAB ? tab_ctas(g) : blocks(g);
  kernel<<<(unsigned)ctas, wg::kThreads, sm, s>>>(
      g, t4(p->q), t4(p->k), t4(p->v), t4(p->d_o), t4(p->dq), p->lse, ws_at(p, 0), p->bias_table, p->g2l,
      TAB ? ws_at(p, ws_off_tab(g)) : nullptr, image_hw);
  count_launch();
  return launch_check("wgmma_bwd_dq");
}

template <typename T, int HD, typename TO, bool DROP>
int backward_t(const VilAttnParams* p, const Geo& g, cudaStream_t s, const int* image_hw) {
  int rc;
  if (!(p->skip_mask & 8) && (rc = simt_delta(p, g, s))) return rc;
  float* delta = static_cast<float*>(p->workspace);
  const int tabn = table_floats(g);
  if (!(p->skip_mask & 2)) {
    if ((rc = g.has_bias ? dq_pass<T, HD, TO, DROP, true>(p, g, s, image_hw) : dq_pass<T, HD, TO, DROP, false>(p, g, s, image_hw)))
      return rc;
  }
  if (!(p->skip_mask & 4)) {
    const size_t sm = wg::DkvSmem<T, HD>::total(tabn, DROP);
    const auto kernel = sub_grids(g, image_hw) ? wg::wg_bwd_dkv<T, HD, TO, DROP, true> : wg::wg_bwd_dkv<T, HD, TO, DROP>;
    if ((rc = set_smem(kernel, sm))) return rc;
    kernel<<<(unsigned)blocks(g), wg::kThreads, sm, s>>>(g, t4(p->q), t4(p->k), t4(p->v), t4(p->d_o), t4(p->dk), t4(p->dv), p->lse,
                                                         delta, p->bias_table, image_hw);
    count_launch();
    if ((rc = launch_check("wgmma_bwd_dkv"))) return rc;
  }
  if (g.g > 0 && !(p->skip_mask & 1) && (rc = simt_global_bwd(p, g, s, g.N, image_hw))) return rc;
  return simt_bias_reduce(p, g, s);
}

template <typename T, typename TO, bool DROP>
int dispatch_hd_drop(const VilAttnParams* p, const Geo& g, cudaStream_t s, bool bwd, const int* hw) {
  switch (head_tile(g.D)) {
    case 16: return bwd ? backward_t<T, 16, TO, DROP>(p, g, s, hw) : forward_t<T, 16, TO, DROP>(p, g, s, hw);
    case 32: return bwd ? backward_t<T, 32, TO, DROP>(p, g, s, hw) : forward_t<T, 32, TO, DROP>(p, g, s, hw);
    case 64: return bwd ? backward_t<T, 64, TO, DROP>(p, g, s, hw) : forward_t<T, 64, TO, DROP>(p, g, s, hw);
    default:
      if constexpr (wg::kSplit<T>) return shared_fail(VIL_E_UNSUPPORTED, "split fp32 kernels stop at head dim 64");
      else return bwd ? backward_t<T, 128, TO, DROP>(p, g, s, hw) : forward_t<T, 128, TO, DROP>(p, g, s, hw);
  }
}

template <typename T, typename TO>
int dispatch_hd(const VilAttnParams* p, const Geo& g, cudaStream_t s, bool bwd, const int* hw) {
  return g.drop_p > 0.f ? dispatch_hd_drop<T, TO, true>(p, g, s, bwd, hw) : dispatch_hd_drop<T, TO, false>(p, g, s, bwd, hw);
}

int run(const VilAttnParams* p, const Geo& g, cudaStream_t s, bool bwd, const int* hw) {
  if (p->dtype == VIL_F32) {   // why_not admits fp32 only with VIL_FLAG_F32_SPLIT
    note_kernel(bwd ? "wgmma_f32split_bwd" : "wgmma_f32split_fwd");
    return dispatch_hd<float, float>(p, g, s, bwd, hw);
  }
  note_kernel(bwd ? "wgmma_bwd" : "wgmma_fwd");
  if (p->dtype == VIL_BF16)
    return out_f32(p) ? dispatch_hd<__nv_bfloat16, float>(p, g, s, bwd, hw)
                      : dispatch_hd<__nv_bfloat16, __nv_bfloat16>(p, g, s, bwd, hw);
  return out_f32(p) ? dispatch_hd<__half, float>(p, g, s, bwd, hw) : dispatch_hd<__half, __half>(p, g, s, bwd, hw);
}

}  // namespace

const char* tc_why_not(const VilAttnParams* p, const Geo& g, bool bwd) {
  const char* w = why_not(p, g, bwd);
  return w ? w : "supported";
}
int tc_supported(const VilAttnParams* p, const Geo& g, bool bwd) { return why_not(p, g, bwd) == nullptr; }
int tc_forward(const VilAttnParams* p, const Geo& g, cudaStream_t s, const int* image_hw) { return run(p, g, s, false, image_hw); }
int tc_backward(const VilAttnParams* p, const Geo& g, cudaStream_t s, const int* image_hw) { return run(p, g, s, true, image_hw); }

}  // namespace vil
