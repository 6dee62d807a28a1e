/*
 * vil_attn.h -- C ABI of the H100 (sm_90a) Vision-Longformer attention library
 *               (libvil_attn.so).  Entry-point names keep the _sm100 suffix of their first target.
 *
 * This is the drop-in boundary for ONE hot path of microsoft/vision-longformer:
 * the "2-D sliding-chunk local + global-token" attention that
 * MODEL.VIT.MSVIT.ATTN_TYPE='longformerhand' selects.  It replaces, as one fused
 * operator, everything between the q/kv Linears and the output projection of
 *
 *   Long2DSCSelfAttention.forward        src/models/layers/longformer2d.py:126-202, 210-226
 *   SlidingChunk2D.forward / .backward   src/models/layers/slidingchunk_2d.py:202-246
 *   slidingchunk_qk / _av / _agrad       src/models/layers/slidingchunk_2d.py:26-200
 *   mask_invalid_locations (+3 builders) src/models/layers/slidingchunk_2d.py:249-357
 *   relative-position-bias gather        src/models/layers/longformer2d.py:159-178, 216-222
 *
 * The reference has no native code and therefore no FFI of its own; the seam the
 * authors used for their (unshipped) CUDA plug-in is the `attn_type` string in
 * AttnBlock (src/models/msvit.py:263-268).  A maintainer binds this library with
 * ctypes from a torch.autograd.Function (see INTEGRATION.md); nothing in the
 * signatures below is a torch / C++ type.
 *
 * Conventions
 * -----------
 *  - All pointers are DEVICE pointers owned by the caller.  The library never
 *    allocates, frees or retains them, never synchronises the host, and launches
 *    only on the stream passed in.  It is stateless and re-entrant.
 *  - A VilTensor4 is a logical (B, H, T, D) view with unit stride on D and
 *    arbitrary element strides on B, H, T - so q can be read straight out of the
 *    `query` Linear output ((B, Nloc, H*D): sh = D, st = H*D) and k / v straight
 *    out of the fused `kv` Linear output ((B, N, 2, H, D): st = 2*H*D) without the
 *    transposes / .contiguous() copies of longformer2d.py:126-149.
 *  - Token order: T index t of k / v / kg / vg: rows [0, nglo) are the global
 *    tokens, row nglo + r*ny + c is the local token at image row r, column c
 *    (r < nx, c < ny).  q / o / d_o / dq hold the nx*ny local rows only,
 *    qg / og / d_og / dqg the nglo global rows only.
 *  - S = scale * (q . k) + bias ; the softmax of a local query is JOINT over
 *    [nglo global keys | the local keys its mask allows] (longformer2d.py:183-185).
 *  - Return value: 0 on success, negative VIL_E_* otherwise; vil_attn_last_error()
 *    then returns a thread-local human-readable message.
 */
#ifndef VIL_ATTN_H_
#define VIL_ATTN_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VIL_ATTN_ABI_VERSION 3

/* element type of q/k/v/o and their gradients (arithmetic is always fp32-accumulated) */
enum { VIL_F32 = 0, VIL_BF16 = 1, VIL_F16 = 2 };

/* kernel family selection */
enum {
  VIL_IMPL_AUTO    = 0, /* wgmma path when the configuration is covered, else SIMT; fp32 takes the wgmma path only
                           with VIL_FLAG_F32_SPLIT */
  VIL_IMPL_SIMT    = 1, /* CUDA-core fp32 path: every (w, exact, mode, nglo) incl. fp32 I/O; forward D <= 128;
                           backward and dropout D <= 128 in fp32, D <= 64 in bf16 / fp16.  Ignores VIL_FLAG_F32_SPLIT */
  VIL_IMPL_WGMMA   = 2  /* wgmma tensor-core path (bf16/fp16, D <= 128 with D % 8 == 0 and 16-byte-aligned rows; with
                           the bias table w <= 42 when D > 64; fp32 with VIL_FLAG_F32_SPLIT, below): error if the
                           configuration is not covered */
};

/* VilAttnParams.flags */
enum {
  /* PARITY BUILD (tests only, SURVEY.md section 8(c) protocol step 1): q/k/v/d_o stay bf16/fp16 but every OUTPUT tensor
     (o, og, dq, dk, dv, dqg, dkg, dvg) is fp32 - VilTensor4 strides then count fp32 elements.  It isolates the
     kernels' internal error (bf16 P / dS operands, fp32 accumulation) from the rounding of the stored result.
     wgmma family only. */
  VIL_FLAG_F32_OUT = 1,
  /* accepted for ABI compatibility: every family runs one pipeline, so it changes nothing */
  VIL_FLAG_UNFUSED = 2,
  /* fp32 operands may run on the wgmma tensor cores as split bf16 products (torch's
     set_float32_matmul_precision("high") / ("medium")): each fp32 x is hi = bf16(x) plus lo = bf16(x - hi), and each
     product A B is A_hi B_hi + A_hi B_lo + A_lo B_hi in fp32 accumulators (about 16 significant bits per term, against
     the SIMT family's full fp32).  dtype must be VIL_F32 (else VIL_E_BADARG).  Covered: D <= 64 with D % 8 == 0 and
     16-byte-aligned fp32 rows; with the bias table w <= 42 when D > 32.  VIL_IMPL_AUTO runs the split wgmma kernels where
     they cover the call and the SIMT family elsewhere; VIL_IMPL_WGMMA fails where they do not; VIL_IMPL_SIMT ignores the
     flag.  The backward must be given the flag of its forward.  The bit leaves VilAttnParams as it was, so the ABI version
     stays 3: a library that predates the flag refuses it as an unknown bit (VIL_E_BADARG) rather than misreading it. */
  VIL_FLAG_F32_SPLIT = 4
};

/* error codes */
enum {
  VIL_OK = 0,
  VIL_E_BADARG = -1,      /* invalid / inconsistent argument (mirrors the reference's asserts / ValueError) */
  VIL_E_UNSUPPORTED = -2, /* valid in the reference but not covered by this build (message says what) */
  VIL_E_CUDA = -3,        /* a CUDA runtime / driver call failed (message carries cudaGetErrorString) */
  VIL_E_WORKSPACE = -4    /* workspace too small: see vil_attn_workspace_bytes */
};

typedef struct VilTensor4 {
  void*   ptr;        /* device pointer to element (0,0,0,0) */
  int64_t sb, sh, st; /* element strides of B, H, T; stride of D is 1 */
} VilTensor4;

typedef struct VilAttnParams {
  int32_t struct_bytes; /* = sizeof(VilAttnParams); guards against ABI drift */
  int32_t dtype;        /* VIL_F32 / VIL_BF16 / VIL_F16 */
  int32_t impl;         /* VIL_IMPL_* */
  int32_t B, H, D;      /* batch, heads, head dim (reference: B, num_heads, head_dim) */
  int32_t nx, ny;       /* local token grid: rows, cols  (forward(x, nx, ny), longformer2d.py:106) */
  int32_t w;            /* chunk / one-sided window size (attention_window, msvit.py:459 field `f`) */
  int32_t nglo;         /* number of global tokens (msvit.py field `g`) */
  int32_t exact;        /* SW_EXACT: 0 sliding-chunk (default), 1 exact (2w+1)^2 window, -1 cyclic chunks */
  int32_t mode;         /* 0 all 9 chunks, -1 own chunk only, 1..8 own + one neighbour (slidingchunk_2d.py:15-24) */
  float   scale;        /* qk_scale or head_dim**-0.5 (longformer2d.py:19), applied to q.k inside the kernel */
  int32_t skip_mask;    /* profiling aid, normally 0: bit0 skip the global-token kernels, bit1 skip the local
                           forward / dq pass, bit2 skip the dk/dv pass, bit3 skip the delta prologue */
  int32_t flags;        /* VIL_FLAG_* bit set, normally 0 */

  /* ---- forward ---- */
  VilTensor4 q;         /* (B,H,nx*ny,D) local queries, UNscaled */
  VilTensor4 k, v;      /* (B,H,nglo+nx*ny,D) */
  VilTensor4 qg;        /* (B,H,nglo,D) global queries (query_global output); ignored if nglo == 0 */
  VilTensor4 kg, vg;    /* (B,H,N,D) keys / values the global queries see (kv_global output);
                           alias k / v when the weights are shared (sharew, longformer2d.py:28-36) */
  VilTensor4 o;         /* out: (B,H,nx*ny,D) */
  VilTensor4 og;        /* out: (B,H,nglo,D) */
  float* lse;           /* out: (B,H,nx*ny) natural-log sum-exp of each local row; contiguous */
  float* lse_g;         /* out: (B,H,nglo) */
  const float* bias_table; /* local_relative_position_bias_table ((4w-1)^2, H) fp32 or NULL (rpe off) */
  const float* g2l;        /* g2l_relative_position_bias (2,H,nglo) fp32; NULL iff bias_table is NULL (rpe creates all
                              three, longformer2d.py:68-100; g2l / g2g without a table -> VIL_E_BADARG) */
  const float* g2g;        /* g2g_relative_position_bias (H,nglo,nglo) fp32 or NULL */

  /* ---- backward (vil_attn_bwd_sm100 only; forward fields above must be filled as in forward,
          with o / og / lse / lse_g holding the forward results) ---- */
  VilTensor4 d_o, d_og;    /* in : gradients of o, og */
  VilTensor4 dq, dk, dv;   /* out: gradients of q, k, v (every row is written) */
  VilTensor4 dqg;          /* out: gradient of qg */
  VilTensor4 dkg, dvg;     /* out: gradients of kg, vg.  If kg.ptr == k.ptr and vg.ptr == v.ptr
                                   (shared weights) the global-query contributions are accumulated
                                   into dk / dv and these two are ignored. */
  float* d_bias_table;     /* fp32 ((4w-1)^2, H), ACCUMULATED INTO (caller zero-fills), or NULL */
  float* d_g2l;            /* fp32 (2,H,nglo), accumulated into, or NULL */
  float* d_g2g;            /* fp32 (H,nglo,nglo), accumulated into, or NULL */

  void*   workspace;       /* device scratch, >= vil_attn_workspace_bytes(), 256-byte aligned.  The backward keeps
                              delta = rowsum(dO * O) of the local and global rows there and, when bias_table != NULL,
                              the partial sums of the three bias gradients (a bounded set for the table: it does not
                              grow with B; per image for g2l / g2g) */
  int64_t workspace_bytes;

  /* ---- attention dropout (nn.Dropout on the softmax probabilities, longformer2d.py:186, 224); ABI v3 ----
     0 <= dropout_p < 1 (else VIL_E_BADARG); 0 runs exactly the kernels without dropout.  The backward must be given the
     forward's p, seed and offset: the mask is recomputed, never stored.  Mask of one element:
       stream 0, local query rows: row = local token i in [0, nx*ny); col = the column of the reference's attn1:
                 t for global key t < nglo, nglo + oi*w*w + lk for key lk of the chunk at offset index oi (oi indexes the
                 reference's block order: 9 blocks for mode 0, [own, neighbour] for mode > 0, own only for mode -1)
       stream 1, global query rows: row = a in [0, nglo); col = key token j in [0, N)
       x = Philox4x32-10(key = (seed & 0xffffffff, seed >> 32),
                         counter = (col >> 2, row, 2*(b*H + h) + stream, (uint32_t)dropout_offset)),  u = x[col & 3]
       kept iff u >= min(floor(p * 2^32), 2^32 - 1) (computed in double); kept probabilities are scaled by 1.0f/(1.0f - p).
     A (query, key) pair the reference visits through two offsets is two columns with two draws.  lse / lse_g stay the
     undropped softmax's. */
  float    dropout_p;
  uint32_t reserved2;
  uint64_t dropout_seed;
  uint64_t dropout_offset;
} VilAttnParams;

/* ABI / diagnostics */
int         vil_attn_abi_version(void);
const char* vil_attn_last_error(void);
/* number of kernel launches this library has issued since it was loaded (all threads) */
int64_t     vil_attn_launch_count(void);
/* name of the kernel family the last successful fwd / bwd call on this thread used ("simt" / "wgmma") */
const char* vil_attn_last_impl(void);
/* name of the main kernel the last wgmma forward / backward launch on this thread used ("wgmma_fwd", "wgmma_bwd";
   "wgmma_f32split_fwd", "wgmma_f32split_bwd" for the split fp32 kernels; "" when the family does not report one) - lets
   tests assert which variant ran */
const char* vil_attn_last_kernel(void);

/* scratch size needed by the forward (backward == 0) or backward (backward != 0) call; < 0 on error */
int64_t vil_attn_workspace_bytes(const VilAttnParams* p, int backward);

/* returns 1 if the wgmma family covers this configuration (the split fp32 kernels when flags has VIL_FLAG_F32_SPLIT),
   0 if only the SIMT family does, < 0 on error */
int vil_attn_wgmma_supported(const VilAttnParams* p);

/* fused forward: o, og, lse, lse_g.  `stream` is a cudaStream_t. */
int vil_attn_fwd_sm100(const VilAttnParams* p, void* stream);

/* fused backward: dq, dk, dv, dqg, (dkg, dvg), d_bias_table, d_g2l, d_g2g.
   Deterministic: for a given build and GPU model, identical inputs give bitwise-identical outputs, including the three
   bias gradients, however the launches and CTAs are scheduled.  No output is summed with atomics: the bias gradients
   are reduced from workspace partials in a fixed order (which order is an implementation detail, not part of the ABI)
   and then added into d_bias_table / d_g2l / d_g2g. */
int vil_attn_bwd_sm100(const VilAttnParams* p, void* stream);

/*
 * LayerNorm over the last dimension of a contiguous (rows, C) token stream - SURVEY.md section 8 (f) row 4, the
 * `norm` in front of the attention / MLP of AttnBlock and MlpBlock (src/models/msvit.py:256, 313-316, 327, 337-339).
 * fp32 statistics; x may be fp32 (the residual stream under autocast) while y is bf16/fp16, which replaces
 * autocast's "fp32 LayerNorm + cast in front of the Linear" pair by one pass.  C <= 1024.
 */
typedef struct VilLayerNormParams {
  int32_t struct_bytes;    /* = sizeof(VilLayerNormParams) */
  int32_t x_dtype;         /* VIL_F32 / VIL_BF16 / VIL_F16: element type of x and dx */
  int32_t y_dtype;         /* element type of y and dy: x_dtype; for x_dtype == VIL_F32 also BF16 / F16 (fp32 residual ->
                              low-precision Linear input); for x_dtype BF16 / F16 also VIL_F32 (patch-embedding norm under
                              autocast: low-precision Conv2d output -> fp32 residual stream) */
  int32_t C;               /* normalized_shape (channels) */
  int64_t rows;            /* number of token rows */
  float   eps;
  int32_t reserved;
  const void*  x;          /* (rows, C) */
  const float* gamma;      /* (C) fp32 weight */
  const float* beta;       /* (C) fp32 bias */
  void*        y;          /* fwd out: (rows, C) */
  float*       mean;       /* fwd out / bwd in: (rows) */
  float*       rstd;       /* fwd out / bwd in: (rows) */
  const void*  dy;         /* bwd in : (rows, C), y_dtype */
  void*        dx;         /* bwd out: (rows, C), x_dtype */
  float*       dgamma;     /* bwd out: (C) fp32 (overwritten) */
  float*       dbeta;      /* bwd out: (C) fp32 (overwritten) */
  void*        workspace;  /* bwd scratch >= vil_layernorm_workspace_bytes() */
  int64_t      workspace_bytes;
} VilLayerNormParams;

int64_t vil_layernorm_workspace_bytes(const VilLayerNormParams* p);
int vil_layernorm_fwd_sm100(const VilLayerNormParams* p, void* stream);
int vil_layernorm_bwd_sm100(const VilLayerNormParams* p, void* stream);

/*
 * Residual / LayerNorm / bias epilogues between the GEMMs of a block - SURVEY.md section 8 (f) row 4 ("LayerNorm -> q/kv
 * Linear and proj -> residual epilogues"), the element-wise chain of AttnBlock.forward / MlpBlock.forward
 * (src/models/msvit.py:313-316, 337-339):   x = x + drop_path(branch(norm(x))).
 *
 * vil_addnorm_fwd_sm100:  xo = x + rowscale[row / rows_per_sample] * (br + bias);   y = LayerNorm(xo) * gamma + beta
 *                         (br == NULL: xo is not written, y = LayerNorm(x): the first norm of a stage)
 * vil_addnorm_bwd_sm100:  dx = gres + LayerNorm'(dy)  (x = the residual stream the norm saw, i.e. the forward's xo);
 *                         dbr = rowscale * dx;  dgamma, dbeta, dbias = column sums (deterministic two-stage reduction)
 * The residual stream (x, xo, gres, dx) is fp32; br / dbr carry b_dtype, y / dy carry y_dtype.  C % 4 == 0, C <= 1024.
 * Contiguous tensors; every non-NULL pointer of a call must be 16-byte aligned (the kernels make 128-bit accesses to the
 * fp32 rows and gamma, 64-bit ones to the bf16 / fp16 rows), else VIL_E_BADARG.  Caching-allocator tensors always are;
 * a contiguous view that starts mid-allocation may not be.
 */
typedef struct VilAddNormParams {
  int32_t struct_bytes;    /* = sizeof(VilAddNormParams) */
  int32_t b_dtype;         /* element type of br / dbr */
  int32_t y_dtype;         /* element type of y / dy */
  int32_t C;
  int64_t rows;
  int64_t rows_per_sample; /* rows that share one rowscale entry (tokens per image); ignored when rowscale is NULL */
  float   eps;
  int32_t reserved;
  const float* x;          /* (rows, C) fp32 */
  const void*  br;         /* (rows, C) b_dtype, or NULL */
  const float* bias;       /* (C) fp32 bias added to br (the bias of the Linear that produced it), or NULL */
  const float* rowscale;   /* (rows / rows_per_sample) fp32 DropPath scale per sample (0 or 1 / keep), or NULL */
  const float* gamma;      /* (C) fp32 */
  const float* beta;       /* (C) fp32 */
  float*       xo;         /* fwd out: (rows, C) fp32; ignored when br is NULL */
  void*        y;          /* fwd out: (rows, C) y_dtype */
  float*       mean;       /* fwd out / bwd in: (rows) */
  float*       rstd;       /* fwd out / bwd in: (rows) */
  const void*  dy;         /* bwd in : (rows, C) y_dtype */
  const float* gres;       /* bwd in : (rows, C) fp32 gradient reaching xo from the rest of the residual stream, or NULL */
  float*       dx;         /* bwd out: (rows, C) fp32 */
  void*        dbr;        /* bwd out: (rows, C) b_dtype, or NULL (no branch) */
  float*       dgamma;     /* bwd out: (C) fp32, overwritten */
  float*       dbeta;      /* bwd out: (C) fp32, overwritten */
  float*       dbias;      /* bwd out: (C) fp32, overwritten; or NULL */
  void*        workspace;  /* bwd scratch >= vil_addnorm_workspace_bytes() */
  int64_t      workspace_bytes;
} VilAddNormParams;

int64_t vil_addnorm_workspace_bytes(const VilAddNormParams* p);
int vil_addnorm_fwd_sm100(const VilAddNormParams* p, void* stream);
int vil_addnorm_bwd_sm100(const VilAddNormParams* p, void* stream);

/*
 * Bias + activation around a GEMM whose bias is kept out of the GEMM so that its gradient falls out of the pass that
 * already reads the tensor (Mlp.fc1 + GELU, src/models/msvit.py:15-33; and the plain column sum that is the bias
 * gradient of the q / kv / qkv Linears, longformer2d.py:24-26):
 * vil_bias_act_fwd_sm100:  a = act(z + bias)
 * vil_bias_act_bwd_sm100:  dz = da * act'(z + bias);  dbias = column sums of dz   (dz == NULL with VIL_ACT_NONE: dbias =
 *                          column sums of da, nothing else is written)
 * Contiguous (rows, C), 16-byte aligned, C * sizeof(element) % 16 == 0.
 */
enum { VIL_ACT_NONE = 0, VIL_ACT_GELU = 1 };   /* GELU: exact (erf) form, nn.GELU() */
typedef struct VilBiasActParams {
  int32_t struct_bytes;    /* = sizeof(VilBiasActParams) */
  int32_t dtype;           /* element type of z, a, da, dz */
  int32_t C;
  int32_t act;             /* VIL_ACT_* */
  int64_t rows;
  const void*  z;          /* (rows, C) pre-bias GEMM output (fwd in, bwd in when act != NONE) */
  const float* bias;       /* (C) fp32 or NULL */
  void*        a;          /* fwd out */
  const void*  da;         /* bwd in */
  void*        dz;         /* bwd out, or NULL */
  float*       dbias;      /* bwd out: (C) fp32, overwritten */
  void*        workspace;  /* bwd scratch >= vil_bias_act_workspace_bytes() */
  int64_t      workspace_bytes;
} VilBiasActParams;

int64_t vil_bias_act_workspace_bytes(const VilBiasActParams* p);
int vil_bias_act_fwd_sm100(const VilBiasActParams* p, void* stream);
int vil_bias_act_bwd_sm100(const VilBiasActParams* p, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VIL_ATTN_H_ */
