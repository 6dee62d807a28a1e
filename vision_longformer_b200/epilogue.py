"""Residual / LayerNorm / bias epilogues between the GEMMs of a block (SURVEY.md section 8 (f) row 4; the element-wise chain of
`AttnBlock.forward` / `MlpBlock.forward`, src/models/msvit.py:313-316, 337-339).

    add_norm(x, br, bias, rowscale, norm)  ->  (xo, y)      xo = x + rowscale * (br + bias),  y = norm(xo)
    bias_gelu(z, bias)                     ->  a            a = GELU(z + bias)
    linear_colsum_bias(x, weight, bias)    ->  y            F.linear whose bias gradient is one column-sum kernel

Each is one HBM pass forward and one backward (`vil_addnorm_*`, `vil_bias_act_*`, include/vil_attn.h); the bias gradients of
the Linears fall out of passes that read the tensor anyway (deterministic two-stage column sums, no atomics).  These are CUDA
ops: callers check `applies(...)` and keep the stock PyTorch composition on CPU tensors (the harness also runs on CPU with the
oracle attention for the reference arm).
"""
from __future__ import annotations

import ctypes
import math

import torch
import torch.nn.functional as F

from . import _lib

_DT = {torch.float32: _lib.VIL_F32, torch.bfloat16: _lib.VIL_BF16, torch.float16: _lib.VIL_F16}
_aligned = _lib.aligned


def _stream(t):
    return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _ptr(t):
    return None if t is None else t.data_ptr()


def addnorm_applies(x, br, C) -> bool:
    """fp32 residual stream on CUDA, channel count the kernels take, branch in a supported dtype."""
    return (x.is_cuda and x.dtype == torch.float32 and C % 4 == 0 and C <= 1024
            and (br is None or (br.dtype in _DT and br.shape == x.shape)))


def addnorm_raw_forward(x2, br2, bias32, rowscale32, gamma32, beta32, xo, y, mean, rstd, eps, rows_per_sample=1):
    """`vil_addnorm_fwd_sm100` on preallocated contiguous (rows, C) tensors (fp32 x / xo, gamma, beta, bias, rowscale)."""
    p = _lib.VilAddNormParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilAddNormParams)
    p.b_dtype = _DT[br2.dtype] if br2 is not None else _DT[y.dtype]
    p.y_dtype, p.C, p.rows, p.rows_per_sample, p.eps = _DT[y.dtype], x2.shape[1], x2.shape[0], rows_per_sample, float(eps)
    p.x, p.br, p.bias, p.rowscale, p.gamma, p.beta = x2.data_ptr(), _ptr(br2), _ptr(bias32), _ptr(rowscale32), gamma32.data_ptr(), beta32.data_ptr()
    p.xo, p.y, p.mean, p.rstd = _ptr(xo), y.data_ptr(), mean.data_ptr(), rstd.data_ptr()
    with torch.cuda.device(x2.device):
        _lib.raise_for(_lib.load().vil_addnorm_fwd_sm100(ctypes.byref(p), _stream(x2)))


def addnorm_workspace(rows, C, device):
    p = _lib.VilAddNormParams()
    p.struct_bytes, p.C, p.rows = ctypes.sizeof(_lib.VilAddNormParams), C, rows
    return torch.empty(int(_lib.load().vil_addnorm_workspace_bytes(ctypes.byref(p))), dtype=torch.uint8, device=device)


def addnorm_raw_backward(xo, gamma32, mean, rstd, rowscale32, dy, gres, dx, dbr, dgamma, dbeta, dbias, ws, eps, rows_per_sample=1):
    """`vil_addnorm_bwd_sm100`: dx = gres + LayerNorm'(dy), dbr = rowscale * dx, column sums -> dgamma / dbeta / dbias."""
    p = _lib.VilAddNormParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilAddNormParams)
    p.b_dtype = _DT[dbr.dtype] if dbr is not None else _DT[dy.dtype]
    p.y_dtype, p.C, p.rows, p.rows_per_sample, p.eps = _DT[dy.dtype], xo.shape[1], xo.shape[0], rows_per_sample, float(eps)
    p.x, p.gamma, p.beta, p.mean, p.rstd, p.rowscale = xo.data_ptr(), gamma32.data_ptr(), gamma32.data_ptr(), mean.data_ptr(), rstd.data_ptr(), _ptr(rowscale32)
    p.dy, p.gres, p.dx, p.dbr = dy.data_ptr(), _ptr(gres), dx.data_ptr(), _ptr(dbr)
    p.dgamma, p.dbeta, p.dbias = dgamma.data_ptr(), dbeta.data_ptr(), _ptr(dbias)
    p.workspace, p.workspace_bytes = ws.data_ptr(), ws.numel()
    with torch.cuda.device(xo.device):
        _lib.raise_for(_lib.load().vil_addnorm_bwd_sm100(ctypes.byref(p), _stream(xo)))


class _AddNorm(torch.autograd.Function):
    """(x, br, bias, rowscale, gamma, beta) -> (xo, y).  x / xo: fp32 residual stream; br: branch output before its bias."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, x, br, bias, rowscale, gamma, beta, eps, out_dtype, rows_per_sample):
        C = x.shape[-1]
        x2 = _aligned(x.reshape(-1, C).contiguous())
        br2 = _aligned(br.reshape(-1, C).contiguous())
        g32, b32 = _aligned(gamma.detach().float().contiguous()), _aligned(beta.detach().float().contiguous())
        bias32 = None if bias is None else _aligned(bias.detach().float().contiguous())
        rs32 = None if rowscale is None else _aligned(rowscale.detach().float().contiguous())
        rows = x2.shape[0]
        xo = torch.empty_like(x2)
        y = torch.empty((rows, C), dtype=out_dtype, device=x.device)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        addnorm_raw_forward(x2, br2, bias32, rs32, g32, b32, xo, y, mean, rstd, eps, rows_per_sample)
        ctx.save_for_backward(xo, g32, mean, rstd, rs32)
        ctx.meta = (x.shape, C, eps, out_dtype, br.dtype, rows_per_sample, gamma.dtype, beta.dtype,
                    None if bias is None else bias.dtype)
        return xo.view(x.shape), y.view(x.shape)

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, g_xo, g_y):
        xo, g32, mean, rstd, rs32 = ctx.saved_tensors
        shape, C, eps, out_dtype, br_dtype, rps, gdt, bdt, biasdt = ctx.meta
        rows = xo.shape[0]
        dev = xo.device
        if g_y is None:
            g_y = torch.zeros((rows, C), dtype=out_dtype, device=dev)
        dy = g_y.reshape(-1, C)
        dy = _aligned((dy if dy.dtype == out_dtype else dy.to(out_dtype)).contiguous())
        gres = None
        if g_xo is not None:
            gres = g_xo.reshape(-1, C)
            gres = _aligned((gres if gres.dtype == torch.float32 else gres.float()).contiguous())
        dx = torch.empty_like(xo)
        dbr = torch.empty((rows, C), dtype=br_dtype, device=dev)
        alloc = torch.zeros if rows == 0 else torch.empty
        dg, db, dbias = (alloc(C, dtype=torch.float32, device=dev) for _ in range(3))
        addnorm_raw_backward(xo, g32, mean, rstd, rs32, dy, gres, dx, dbr, dg, db, dbias, addnorm_workspace(rows, C, dev), eps, rps)
        return (dx.view(shape), dbr.view(shape), None if biasdt is None else dbias.to(biasdt), None,
                dg.to(gdt), db.to(bdt), None, None, None)


def add_norm(x, br, bias, rowscale, norm, out_dtype=None):
    """xo = x + rowscale[sample] * (br + bias);  y = norm(xo).  `norm`: an affine last-dim nn.LayerNorm.  x: (B, ..., C) fp32;
    rowscale: (B) with one entry per sample x[b], or None."""
    if out_dtype is None:
        out_dtype = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else x.dtype
    if rowscale is not None and (x.dim() < 2 or rowscale.numel() != x.shape[0]):
        raise ValueError(f"add_norm: rowscale has {rowscale.numel()} entries for a stream of shape {tuple(x.shape)}; "
                         "it needs one per sample (x.shape[0])")
    rps = math.prod(x.shape[1:-1])                         # rows of one sample: every dim between the batch and the channels
    return _AddNorm.apply(x, br, bias, rowscale, norm.weight, norm.bias, norm.eps, out_dtype, rps)


def _ba_params(t2, C, act):
    p = _lib.VilBiasActParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilBiasActParams)
    p.dtype, p.C, p.act, p.rows = _DT[t2.dtype], C, act, t2.shape[0]
    return p


def bias_act_applies(z) -> bool:
    return z.is_cuda and z.dtype in _DT and (z.shape[-1] * z.element_size()) % 16 == 0


def bias_act_workspace(like2, act=_lib.VIL_ACT_NONE):
    p = _ba_params(like2, like2.shape[1], act)
    return torch.empty(int(_lib.load().vil_bias_act_workspace_bytes(ctypes.byref(p))), dtype=torch.uint8, device=like2.device)


def bias_act_raw_forward(z2, bias32, a, act=_lib.VIL_ACT_GELU):
    """`vil_bias_act_fwd_sm100`: a = act(z2 + bias) on contiguous (rows, C) tensors."""
    p = _ba_params(z2, z2.shape[1], act)
    p.z, p.bias, p.a = z2.data_ptr(), _ptr(bias32), a.data_ptr()
    with torch.cuda.device(z2.device):
        _lib.raise_for(_lib.load().vil_bias_act_fwd_sm100(ctypes.byref(p), _stream(z2)))


def bias_act_raw_backward(da2, z2, bias32, dz, dbias, ws, act=_lib.VIL_ACT_NONE):
    """`vil_bias_act_bwd_sm100`: dz = da2 * act'(z2 + bias) (dz None with act NONE: nothing written), dbias = column sums."""
    p = _ba_params(da2, da2.shape[1], act)
    p.z, p.bias, p.da, p.dz, p.dbias = _ptr(z2), _ptr(bias32), da2.data_ptr(), _ptr(dz), dbias.data_ptr()
    p.workspace, p.workspace_bytes = ws.data_ptr(), ws.numel()
    with torch.cuda.device(da2.device):
        _lib.raise_for(_lib.load().vil_bias_act_bwd_sm100(ctypes.byref(p), _stream(da2)))


def _colsum(dy2, z2=None, bias32=None, act=_lib.VIL_ACT_NONE):
    """d_bias (fp32, (C)) = column sums of dy2 * act'(z2 + bias); returns (dz or None, d_bias)."""
    dbias = torch.empty(dy2.shape[1], dtype=torch.float32, device=dy2.device)
    dz = torch.empty_like(dy2) if act != _lib.VIL_ACT_NONE else None
    bias_act_raw_backward(dy2, z2, bias32, dz, dbias, bias_act_workspace(dy2, act), act)
    return dz, dbias


class _BiasGelu(torch.autograd.Function):
    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, z, bias):
        C = z.shape[-1]
        z2 = _aligned(z.reshape(-1, C).contiguous())
        b32 = _aligned(bias.detach().float().contiguous())
        a = torch.empty_like(z2)
        bias_act_raw_forward(z2, b32, a, _lib.VIL_ACT_GELU)
        ctx.save_for_backward(z2, b32)
        ctx.meta = (z.shape, bias.dtype)
        return a.view(z.shape)

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, da):
        z2, b32 = ctx.saved_tensors
        shape, bdt = ctx.meta
        da2 = da.reshape(-1, z2.shape[1])
        da2 = _aligned((da2 if da2.dtype == z2.dtype else da2.to(z2.dtype)).contiguous())
        dz, dbias = _colsum(da2, z2, b32, _lib.VIL_ACT_GELU)
        return dz.view(shape), dbias.to(bdt)


def bias_gelu(z, bias):
    """GELU(z + bias) (exact erf form, nn.GELU()); the bias gradient is produced by the backward pass over z."""
    return _BiasGelu.apply(z, bias)


class _LinearColsumBias(torch.autograd.Function):
    """y = x W^T + b with stock GEMMs; d_b by one column-sum kernel instead of ATen's generic reduction."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, x, weight, bias):
        ctx.save_for_backward(x, weight)
        ctx.bdt = bias.dtype
        return F.linear(x, weight, bias)

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        Cout, Cin = weight.shape
        dy2 = _aligned(dy.reshape(-1, Cout).contiguous())
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = (dy2 @ weight).view(x.shape)
        if ctx.needs_input_grad[1]:
            dw = dy2.t() @ x.reshape(-1, Cin)
        _, dbias = _colsum(dy2)
        return dx, dw, dbias.to(ctx.bdt)


def linear_colsum_bias(x, weight, bias):
    """`F.linear(x, weight, bias)` (autocast-aware) whose bias gradient is computed by `vil_bias_act_bwd_sm100`."""
    if bias is None or not (x.is_cuda and torch.is_grad_enabled() and bias.requires_grad):
        return F.linear(x, weight, bias)
    if torch.is_autocast_enabled("cuda"):
        dt = torch.get_autocast_dtype("cuda")
        x, weight, bias = x.to(dt), weight.to(dt), bias.to(dt)
    if x.dtype not in _DT or weight.dtype != x.dtype or (weight.shape[0] * x.element_size()) % 16 != 0:
        return F.linear(x, weight, bias)
    return _LinearColsumBias.apply(x, weight, bias)
