"""Fused LayerNorm for the token streams around the attention kernel (SURVEY.md section 8 (f) row 4).

`B200LayerNorm` is an `nn.LayerNorm` subclass (same parameters / state_dict keys: `weight`, `bias`) whose forward
runs `vil_layernorm_fwd_sm100` and whose backward runs `vil_layernorm_bwd_sm100` (include/vil_attn.h).  Under
`torch.autocast` an fp32 input (the residual stream) produces a bf16/fp16 output directly - numerically the same
as autocast's fp32 `layer_norm` followed by the cast in front of the next Linear, in one HBM pass instead of two.
CPU tensors fall through to `nn.LayerNorm` (this op is not on the no-CPU-fallback attention path; the harness
is also used on CPU with the oracle attention for the reference arm).
"""
from __future__ import annotations

import ctypes

import torch
from torch import nn

from . import _lib

_DT = {torch.float32: _lib.VIL_F32, torch.bfloat16: _lib.VIL_BF16, torch.float16: _lib.VIL_F16}


def _vec_params(x2, y_dtype, C, eps):
    """fp32 stream with C % 4 == 0: the 128-bit vectorised kernels shared with the residual epilogue (vil_addnorm_*, br = NULL)."""
    p = _lib.VilAddNormParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilAddNormParams)
    p.b_dtype, p.y_dtype, p.C, p.rows, p.rows_per_sample, p.eps = _DT[y_dtype], _DT[y_dtype], C, x2.shape[0], 1, float(eps)
    return p


def _params(x2, y_dtype, C, eps):
    p = _lib.VilLayerNormParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilLayerNormParams)
    p.x_dtype, p.y_dtype, p.C, p.rows, p.eps = _DT[x2.dtype], _DT[y_dtype], C, x2.shape[0], float(eps)
    return p


class _FusedLayerNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps, out_dtype):
        C = x.shape[-1]
        x2 = _lib.aligned(x.reshape(-1, C).contiguous())
        w32, b32 = _lib.aligned(weight.detach().float().contiguous()), _lib.aligned(bias.detach().float().contiguous())
        y = torch.empty(x2.shape, dtype=out_dtype, device=x.device)
        mean = torch.empty(x2.shape[0], dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        vec = x2.dtype == torch.float32 and C % 4 == 0
        p = _vec_params(x2, out_dtype, C, eps) if vec else _params(x2, out_dtype, C, eps)
        p.x, p.gamma, p.beta, p.y, p.mean, p.rstd = x2.data_ptr(), w32.data_ptr(), b32.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr()
        lib = _lib.load()
        with torch.cuda.device(x.device):
            rc = (lib.vil_addnorm_fwd_sm100 if vec else lib.vil_layernorm_fwd_sm100)(
                ctypes.byref(p), ctypes.c_void_p(torch.cuda.current_stream(x.device).cuda_stream))
        _lib.raise_for(rc)
        ctx.save_for_backward(x2, w32, b32, mean, rstd)
        ctx.meta = (x.shape, C, eps, out_dtype, weight.dtype, bias.dtype, vec)
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        x2, w32, b32, mean, rstd = ctx.saved_tensors
        shape, C, eps, out_dtype, wdt, bdt, vec = ctx.meta
        dy2 = dy.reshape(-1, C)
        if dy2.dtype != out_dtype:
            dy2 = dy2.to(out_dtype)
        dy2 = _lib.aligned(dy2.contiguous())
        dx = torch.empty_like(x2)
        # rows == 0: the library returns without launching, so the parameter gradients must already be zero
        alloc = torch.zeros if x2.shape[0] == 0 else torch.empty
        dg = alloc(C, dtype=torch.float32, device=x2.device)
        db = alloc(C, dtype=torch.float32, device=x2.device)
        p = _vec_params(x2, out_dtype, C, eps) if vec else _params(x2, out_dtype, C, eps)
        lib = _lib.load()
        need = int((lib.vil_addnorm_workspace_bytes if vec else lib.vil_layernorm_workspace_bytes)(ctypes.byref(p)))
        ws = torch.empty(need, dtype=torch.uint8, device=x2.device)
        p.x, p.gamma, p.beta, p.mean, p.rstd = x2.data_ptr(), w32.data_ptr(), b32.data_ptr(), mean.data_ptr(), rstd.data_ptr()
        p.dy, p.dx, p.dgamma, p.dbeta = dy2.data_ptr(), dx.data_ptr(), dg.data_ptr(), db.data_ptr()
        p.workspace, p.workspace_bytes = ws.data_ptr(), need
        with torch.cuda.device(x2.device):
            rc = (lib.vil_addnorm_bwd_sm100 if vec else lib.vil_layernorm_bwd_sm100)(
                ctypes.byref(p), ctypes.c_void_p(torch.cuda.current_stream(x2.device).cuda_stream))
        _lib.raise_for(rc)
        return dx.view(shape), dg.to(wdt), db.to(bdt), None, None


class B200LayerNorm(nn.LayerNorm):
    """Drop-in `nn.LayerNorm` (last-dim, affine) backed by the sm_90a kernels.  `keep_dtype=True` marks a norm whose
    output joins the fp32 residual stream (the patch-embedding norm): an fp32 input stays fp32 even under autocast,
    and a bf16/fp16 input under autocast (the Conv2d output) is normalised into an fp32 result by the low-precision-in ->
    fp32-out kernel variant - the dtype `nn.LayerNorm` gives the reference there (autocast runs layer_norm in fp32), in
    one HBM pass instead of cast + norm."""

    def __init__(self, normalized_shape, eps=1e-5, keep_dtype=False, **kw):
        super().__init__(normalized_shape, eps=eps, **kw)
        self.keep_dtype = keep_dtype

    def forward(self, x):
        if (not x.is_cuda) or len(self.normalized_shape) != 1 or self.weight is None or self.bias is None \
                or x.dtype not in _DT or x.shape[-1] > 1024:
            return super().forward(x)
        out_dtype = x.dtype
        if torch.is_autocast_enabled("cuda"):
            if self.keep_dtype and x.dtype != torch.float32:
                out_dtype = torch.float32          # autocast: low-precision in -> fp32 out (residual stream), one pass
            if not self.keep_dtype and x.dtype == torch.float32:
                out_dtype = torch.get_autocast_dtype("cuda")
        return _FusedLayerNorm.apply(x, self.weight, self.bias, self.eps, out_dtype)
