// Host-side glue shared by the translation units of libvil_attn.so.  The library is compiled as several TUs
// (one per kernel family / pass, built in parallel by __graft_entry__.build()); every kernel lives entirely in one
// TU, so no relocatable device code is needed.
#pragma once
#include <cuda_runtime.h>
#include "vil_common.cuh"

namespace vil {

// vil_attn_api.cu
int shared_fail(int code, const char* msg);     // records the thread-local error message, returns `code`
void count_launch();                            // vil_attn_launch_count()
void note_kernel(const char* name);             // vil_attn_last_kernel(): static string naming the main kernel variant

inline int launch_check(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return VIL_OK;
  char msg[192];
  snprintf(msg, sizeof(msg), "%s: %s", what, cudaGetErrorString(e));
  return shared_fail(VIL_E_CUDA, msg);
}

inline T4 t4(const VilTensor4& t) { T4 r; r.p = static_cast<char*>(t.ptr); r.sb = t.sb; r.sh = t.sh; r.st = t.st; return r; }

// flags of VilAttnParams
inline bool out_f32(const VilAttnParams* p) { return (p->flags & VIL_FLAG_F32_OUT) != 0; }
inline bool split_f32(const VilAttnParams* p) { return (p->flags & VIL_FLAG_F32_SPLIT) != 0; }

// the backward workspace at float offset `off` (vil_common.cuh: ws_off_*)
inline float* ws_at(const VilAttnParams* p, long long off) { return static_cast<float*>(p->workspace) + off; }

// ---- vil_simt.cu: the CUDA-core family and the small global-token kernels both families share
int simt_run(const VilAttnParams* p, const Geo& g, cudaStream_t s, bool bwd);
int simt_global_fwd(const VilAttnParams* p, const Geo& g, cudaStream_t s);                 // og, lse_g
int simt_delta(const VilAttnParams* p, const Geo& g, cudaStream_t s);                      // delta, delta_g -> workspace
// global key columns + global query rows; rmw_rows: keys whose dk / dv rows simt_bwd_grow still updates
int simt_global_bwd(const VilAttnParams* p, const Geo& g, cudaStream_t s, int rmw_rows);
// with the bias table: sums the partials pass 1 and the global-token kernels left in the workspace, in a fixed order, into
// d_bias_table, d_g2l, d_g2g (one launch; none without the table)
int simt_bias_reduce(const VilAttnParams* p, const Geo& g, cudaStream_t s);

// ---- vil_wgmma.cu: the tensor-core (wgmma) family
const char* tc_why_not(const VilAttnParams* p, const Geo& g, bool bwd);
int tc_supported(const VilAttnParams* p, const Geo& g, bool bwd);
int tc_forward(const VilAttnParams* p, const Geo& g, cudaStream_t s);
int tc_backward(const VilAttnParams* p, const Geo& g, cudaStream_t s);

}  // namespace vil
