"""The fused Vision-Longformer attention operator (Python side of the C ABI).

`vil_attention_raw_forward/backward` take strided (B, H, T, D) views and call
`vil_attn_fwd_sm100` / `vil_attn_bwd_sm100` (include/vil_attn.h) on the current
CUDA stream.  `vil_attention` is the autograd-aware entry the module uses; it
consumes the outputs of the `query` / `kv` Linears *in place* (no transposes or
.contiguous() copies, cf. longformer2d.py:126-149) and writes the attention
output directly in (B, N, H*D) layout for `proj` (cf. :201-203).

fp32 calls follow torch's fp32 matmul precision: when `torch.backends.cuda.matmul.fp32_precision` is "tf32" (after
`torch.set_float32_matmul_precision("high")` or `("medium")`), `impl="auto"` and `impl="wgmma"` run fp32 on the wgmma
tensor cores as split bf16 products (VIL_FLAG_F32_SPLIT, include/vil_attn.h); otherwise, and with `impl="simt"`, fp32
runs on the SIMT family in full fp32.  The choice is made in the forward and reused by its backward.

The backward is deterministic: identical inputs give bitwise-identical gradients on a given build and GPU model,
including those of the relative-position-bias parameters (summed in a fixed order, no atomics), so it needs no special
handling under torch.use_deterministic_algorithms(True).  The workspace is sized by vil_attn_workspace_bytes, which
includes the bias-gradient partials when the table is given.

Replaces: longformer2d.py:126-202 + :210-226 and everything in
slidingchunk_2d.py they call.
"""
from __future__ import annotations

import ctypes
import operator
from typing import Optional

import torch

from . import _lib
from ._lib import VilAttnParams, VilTensor4

_DTYPES = {torch.float32: _lib.VIL_F32, torch.bfloat16: _lib.VIL_BF16, torch.float16: _lib.VIL_F16}
_IMPLS = {"auto": _lib.VIL_IMPL_AUTO, "simt": _lib.VIL_IMPL_SIMT, "wgmma": _lib.VIL_IMPL_WGMMA}


def _require_cuda(t: torch.Tensor, name: str):
    if not t.is_cuda:
        raise RuntimeError(
            f"vil_attention: `{name}` is on {t.device}; this operator only runs on a CUDA (sm_90a) device - "
            "there is no CPU fallback")


def _t4(t: Optional[torch.Tensor]) -> VilTensor4:
    if t is None:
        return VilTensor4(None, 0, 0, 0)
    assert t.dim() == 4 and (t.stride(3) == 1 or t.shape[3] == 1), "expected a (B,H,T,D) view with unit stride on D"
    return VilTensor4(t.data_ptr(), t.stride(0), t.stride(1), t.stride(2))


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _f32c(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    if t is None:
        return None
    return t.detach().to(torch.float32).contiguous()


def _base_params(q, k, nx, ny, w, nglo, exact, mode, scale, impl, skip_mask=0, flags=0, dropout_p=0.0, dropout_seed=0,
                 dropout_offset=0, dilation=1) -> VilAttnParams:
    if exact not in (0, 1, -1):
        raise ValueError("longsc exact should be in [0,1,-1]!")          # slidingchunk_2d.py:343
    if int(dilation) != dilation or dilation < 1:
        raise ValueError(f"dilation must be an integer >= 1 (got {dilation})")
    if exact == 1 and mode != 0:
        raise ValueError("exact sliding window (exact=1) only supports mode=0")
    if q.dtype not in _DTYPES:
        raise TypeError(f"unsupported dtype {q.dtype}")
    p = VilAttnParams()
    p.struct_bytes = ctypes.sizeof(VilAttnParams)
    p.dtype = _DTYPES[q.dtype]
    p.impl = _IMPLS[impl]
    p.B, p.H, p.D = q.shape[0], q.shape[1], q.shape[3]
    p.nx, p.ny, p.w, p.nglo, p.exact, p.mode = nx, ny, w, nglo, exact, mode
    p.scale = float(scale)
    p.skip_mask = int(skip_mask)
    p.flags = int(flags)
    if dilation > 1:                             # d = 1 leaves the flag clear: the undilated operator, bit for bit
        p.flags |= _lib.VIL_FLAG_DILATED
        p.dilation = int(dilation)
    p.dropout_p = float(dropout_p)
    p.dropout_seed, p.dropout_offset = int(dropout_seed), int(dropout_offset)
    return p


def image_sizes_host(image_sizes, B: int, nx: int, ny: int) -> Optional[torch.Tensor]:
    """Validate per-image token grids on the host: `image_sizes` is a sequence of B (h, w) pairs or a CPU integer tensor
    of shape (B, 2), with 1 <= h <= nx and 1 <= w <= ny.  Returns them as a CPU int32 (B, 2) tensor, or None when
    `image_sizes` is None or every image fills the nx x ny grid (the unsized operator, bit for bit)."""
    if image_sizes is None:
        return None
    if isinstance(image_sizes, torch.Tensor):
        if image_sizes.device.type != "cpu":
            raise TypeError(f"image_sizes is on {image_sizes.device}: pass host data (a sequence of (h, w) or a CPU tensor); "
                            "the sizes are validated on the host, which a device tensor would need a synchronise for")
        if image_sizes.is_floating_point() or image_sizes.is_complex() or image_sizes.dtype == torch.bool:
            raise TypeError(f"image_sizes must hold integers (got {image_sizes.dtype})")
        t = image_sizes.to(torch.int64)
    else:
        try:
            t = torch.tensor([[operator.index(v) for v in hw] for hw in image_sizes], dtype=torch.int64)
        except TypeError as e:
            raise TypeError(f"image_sizes must be a sequence of (h, w) integer pairs: {e}") from None
    if tuple(t.shape) != (B, 2):
        raise ValueError(f"image_sizes must have shape ({B}, 2), one (h, w) per image (got {tuple(t.shape)})")
    bad = (t[:, 0] < 1) | (t[:, 0] > nx) | (t[:, 1] < 1) | (t[:, 1] > ny)
    if bool(bad.any()):
        b = int(bad.nonzero()[0, 0])
        raise ValueError(f"image_sizes[{b}] = ({int(t[b, 0])}, {int(t[b, 1])}) is outside [1, {nx}] x [1, {ny}]")
    if bool((t[:, 0] == nx).all()) and bool((t[:, 1] == ny).all()):
        return None
    return t.to(torch.int32)


def image_sizes_device(image_sizes, B: int, nx: int, ny: int, device) -> Optional[torch.Tensor]:
    """`image_sizes_host`, uploaded to `device` without a host synchronise (pinned memory, non-blocking copy)."""
    t = image_sizes_host(image_sizes, B, nx, ny)
    if t is None:
        return None
    return t.pin_memory().to(device, non_blocking=True)


def _call(fn_plain, fn_sized, p: VilAttnParams, image_hw: Optional[torch.Tensor], device):
    """One library call on `device`'s current stream: the sized entry point when per-image grids are given."""
    with torch.cuda.device(device):            # launch on the tensors' device and on ITS current stream
        stream = ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        if image_hw is None:
            return fn_plain(ctypes.byref(p), stream)
        return fn_sized(ctypes.byref(p), ctypes.c_void_p(image_hw.data_ptr()), stream)


def _split_flag(x: torch.Tensor, impl: str) -> int:
    """VIL_FLAG_F32_SPLIT for an fp32 call that may use the tensor cores: torch's fp32 matmul precision allows TF32 or
    split-bf16 products.  `fp32_precision` is read rather than get_float32_matmul_precision() or matmul.allow_tf32,
    which raise once the legacy and the new precision APIs have been mixed."""
    if x.dtype != torch.float32 or impl == "simt":
        return 0
    return _lib.VIL_FLAG_F32_SPLIT if torch.backends.cuda.matmul.fp32_precision == "tf32" else 0


def _dropout_state(device: torch.device, dropout_p: float):
    """(seed, offset) of one dropout forward, drawn from the default CUDA generator of `device` the way torch's own
    Philox-based kernels draw theirs: the generator's seed and its current offset, which is then advanced.  Host-side
    generator state only (no host-device synchronisation); `torch.manual_seed` reproduces it.  The kernels take the
    offset in units of 4 (one Philox counter word)."""
    if dropout_p <= 0.0:
        return 0, 0
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("vil_attention: attention dropout cannot be captured in a CUDA graph (the mask's seed and offset "
                           "are drawn on the host at each call)")
    idx = device.index if device.index is not None else torch.cuda.current_device()
    gen = torch.cuda.default_generators[idx]
    seed, offset = gen.initial_seed(), gen.get_offset()
    gen.set_offset(offset + 4)
    return seed, offset // 4


def _workspace(p: VilAttnParams, backward: bool, device) -> torch.Tensor:
    lib = _lib.load()
    need = lib.vil_attn_workspace_bytes(ctypes.byref(p), 1 if backward else 0)
    if need < 0:
        _lib.raise_for(int(need))
    ws = torch.empty(int(need), dtype=torch.uint8, device=device)
    p.workspace, p.workspace_bytes = ws.data_ptr(), int(need)
    return ws


def vil_attention_raw_forward(q, k, v, qg, kg, vg, table, g2l, g2g, o, og, *, nx, ny, w, exact=0, mode=0,
                              scale=1.0, impl="auto", skip_mask=0, flags=0, dropout_p=0.0, dropout_seed=0, dropout_offset=0,
                              dilation=1, image_sizes=None, _image_hw=None):
    """q:(B,H,Nloc,D) k,v:(B,H,N,D) qg:(B,H,g,D) kg,vg:(B,H,N,D) views; o/og preallocated output views.
    `flags`: VIL_FLAG_* of include/vil_attn.h (F32_OUT = 1: o / og are fp32 tensors - the parity build; F32_SPLIT = 4:
    fp32 operands on the wgmma tensor cores as split bf16 products).
    `dropout_p` > 0: attention dropout with the mask of (dropout_seed, dropout_offset) (include/vil_attn.h); the
    backward must be given the same three values.
    `dilation` d > 1: dilated sliding-chunk attention (VIL_FLAG_DILATED, include/vil_attn.h): each local query attends
    within its residue sub-grid of image positions (a + d r', b + d c'); the backward must be given the same d.
    `image_sizes`: per-image token grids of a padded batch, host data of B (h, w) (see `vil_attention`); the backward
    must be given the same sizes.
    Returns (lse (B,H,Nloc) fp32, lse_g (B,H,g) fp32 or None)."""
    _require_cuda(q, "q")
    B, H, Nloc, D = q.shape
    g = k.shape[2] - Nloc
    assert Nloc == nx * ny, "Global dimension does not match!"           # longformer2d.py:111
    hw = _image_hw if _image_hw is not None else image_sizes_device(image_sizes, B, nx, ny, q.device)
    p = _base_params(q, k, nx, ny, w, g, exact, mode, scale, impl, skip_mask, flags, dropout_p, dropout_seed, dropout_offset,
                     dilation)
    lse = torch.empty(B, H, Nloc, dtype=torch.float32, device=q.device)
    lse_g = torch.empty(B, H, g, dtype=torch.float32, device=q.device) if g > 0 else None
    p.q, p.k, p.v, p.o = _t4(q), _t4(k), _t4(v), _t4(o)
    if g > 0:
        p.qg, p.kg, p.vg, p.og = _t4(qg), _t4(kg), _t4(vg), _t4(og)
    p.lse, p.lse_g = _ptr(lse), _ptr(lse_g)
    p.bias_table, p.g2l, p.g2g = _ptr(table), _ptr(g2l), _ptr(g2g)
    ws = _workspace(p, False, q.device)
    lib = _lib.load()
    _lib.raise_for(_call(lib.vil_attn_fwd_sm100, lib.vil_attn_fwd_sized_sm100, p, hw, q.device))
    del ws
    return lse, lse_g


def vil_attention_raw_backward(q, k, v, qg, kg, vg, table, g2l, g2g, o, og, lse, lse_g, d_o, d_og,
                               dq, dk, dv, dqg, dkg, dvg, d_table, d_g2l, d_g2g, *, nx, ny, w, exact=0, mode=0,
                               scale=1.0, impl="auto", skip_mask=0, flags=0, dropout_p=0.0, dropout_seed=0, dropout_offset=0,
                               dilation=1, image_sizes=None, _image_hw=None):
    _require_cuda(q, "q")
    Nloc = q.shape[2]
    g = k.shape[2] - Nloc
    hw = _image_hw if _image_hw is not None else image_sizes_device(image_sizes, q.shape[0], nx, ny, q.device)
    p = _base_params(q, k, nx, ny, w, g, exact, mode, scale, impl, skip_mask, flags, dropout_p, dropout_seed, dropout_offset,
                     dilation)
    p.q, p.k, p.v, p.o = _t4(q), _t4(k), _t4(v), _t4(o)
    p.d_o, p.dq, p.dk, p.dv = _t4(d_o), _t4(dq), _t4(dk), _t4(dv)
    if g > 0:
        p.qg, p.kg, p.vg, p.og = _t4(qg), _t4(kg), _t4(vg), _t4(og)
        p.d_og, p.dqg, p.dkg, p.dvg = _t4(d_og), _t4(dqg), _t4(dkg), _t4(dvg)
    p.lse, p.lse_g = _ptr(lse), _ptr(lse_g)
    p.bias_table, p.g2l, p.g2g = _ptr(table), _ptr(g2l), _ptr(g2g)
    p.d_bias_table, p.d_g2l, p.d_g2g = _ptr(d_table), _ptr(d_g2l), _ptr(d_g2g)
    ws = _workspace(p, True, q.device)
    lib = _lib.load()
    _lib.raise_for(_call(lib.vil_attn_bwd_sm100, lib.vil_attn_bwd_sized_sm100, p, hw, q.device))
    del ws


def _heads(t: torch.Tensor, H: int, which: int = 0, parts: int = 1) -> torch.Tensor:
    """(B, T, parts*H*D) Linear output -> (B, H, T, D) strided view of part `which` (no copy)."""
    B, T, C = t.shape
    D = C // (parts * H)
    return t.view(B, T, parts, H, D)[:, :, which].permute(0, 2, 1, 3)


class _VilAttention(torch.autograd.Function):
    # AMP contract (SURVEY.md section 8(b)): custom_fwd records the autocast state and runs the op with autocast off,
    # custom_bwd replays that state in backward.  The cast of the activations to the autocast dtype happens in
    # `vil_attention` (not via cast_inputs, which would also round the fp32 bias tables to bf16).
    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, q_all, kv, qg_all, kvg, table, g2l, g2g, H, nx, ny, w, nglo, exact, mode, scale, impl, dropout_p, dilation,
                image_sizes):
        _require_cuda(q_all, "q")
        B = q_all.shape[0]
        C = q_all.shape[2]
        N = kv.shape[1]
        g = nglo
        Nloc = nx * ny
        assert g + Nloc == N, "Global dimension does not match!"
        q_all = q_all if q_all.stride(2) == 1 else q_all.contiguous()
        kv = kv if kv.stride(2) == 1 else kv.contiguous()
        k, v = _heads(kv, H, 0, 2), _heads(kv, H, 1, 2)
        shared = qg_all is None
        if g > 0:
            if shared:                       # sharew: rows [0,g) of q_all are the global queries
                q = _heads(q_all, H)[:, :, g:]
                qg = _heads(q_all, H)[:, :, :g]
                kg, vg = k, v
            else:
                qg_all = qg_all if qg_all.stride(2) == 1 else qg_all.contiguous()
                kvg = kvg if kvg.stride(2) == 1 else kvg.contiguous()
                q, qg = _heads(q_all, H), _heads(qg_all, H)
                kg, vg = _heads(kvg, H, 0, 2), _heads(kvg, H, 1, 2)
        else:
            q, qg, kg, vg = _heads(q_all, H), None, None, None
        tab32, g2l32, g2g32 = _f32c(table), _f32c(g2l) if g > 0 else None, _f32c(g2g) if g > 0 else None
        out = torch.empty(B, N, C, dtype=q_all.dtype, device=q_all.device)
        o = _heads(out, H)[:, :, g:]
        og = _heads(out, H)[:, :, :g] if g > 0 else None
        hw = image_sizes_device(image_sizes, B, nx, ny, q_all.device)   # kept on the device for the backward
        seed, offset = _dropout_state(q_all.device, dropout_p)
        flags = _split_flag(q_all, impl)
        lse, lse_g = vil_attention_raw_forward(q, k, v, qg, kg, vg, tab32, g2l32, g2g32, o, og, nx=nx, ny=ny, w=w,
                                               exact=exact, mode=mode, scale=scale, impl=impl, flags=flags,
                                               dropout_p=dropout_p, dropout_seed=seed, dropout_offset=offset,
                                               dilation=dilation, _image_hw=hw)
        ctx.save_for_backward(q_all, kv, qg_all, kvg, table, g2l, g2g, out, lse, lse_g)
        ctx.cfg = (H, nx, ny, w, g, exact, mode, scale, impl, shared, flags, dilation)
        ctx.hw = hw
        ctx.drop = (dropout_p, seed, offset)
        return out

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, d_out):
        q_all, kv, qg_all, kvg, table, g2l, g2g, out, lse, lse_g = ctx.saved_tensors
        H, nx, ny, w, g, exact, mode, scale, impl, shared, flags, dilation = ctx.cfg
        dropout_p, seed, offset = ctx.drop
        d_out = d_out.contiguous()
        k, v = _heads(kv, H, 0, 2), _heads(kv, H, 1, 2)
        dq_all = torch.empty_like(q_all, memory_format=torch.contiguous_format)
        dkv = torch.empty_like(kv, memory_format=torch.contiguous_format)
        dk, dv = _heads(dkv, H, 0, 2), _heads(dkv, H, 1, 2)
        dqg_all = dkvg = None
        if g > 0:
            if shared:
                q, qg = _heads(q_all, H)[:, :, g:], _heads(q_all, H)[:, :, :g]
                dq, dqg = _heads(dq_all, H)[:, :, g:], _heads(dq_all, H)[:, :, :g]
                kg, vg, dkg, dvg = k, v, dk, dv
            else:
                q, qg = _heads(q_all, H), _heads(qg_all, H)
                dqg_all = torch.empty_like(qg_all, memory_format=torch.contiguous_format)
                dkvg = torch.empty_like(kvg, memory_format=torch.contiguous_format)
                dq, dqg = _heads(dq_all, H), _heads(dqg_all, H)
                kg, vg = _heads(kvg, H, 0, 2), _heads(kvg, H, 1, 2)
                dkg, dvg = _heads(dkvg, H, 0, 2), _heads(dkvg, H, 1, 2)
            o, og = _heads(out, H)[:, :, g:], _heads(out, H)[:, :, :g]
            d_o, d_og = _heads(d_out, H)[:, :, g:], _heads(d_out, H)[:, :, :g]
        else:
            q, qg, kg, vg, dq, dqg, dkg, dvg = _heads(q_all, H), None, None, None, _heads(dq_all, H), None, None, None
            o, og, d_o, d_og = _heads(out, H), None, _heads(d_out, H), None
        tab32 = _f32c(table)
        g2l32, g2g32 = (_f32c(g2l), _f32c(g2g)) if g > 0 else (None, None)
        d_tab = torch.zeros_like(tab32) if tab32 is not None else None
        d_g2l = torch.zeros_like(g2l32) if g2l32 is not None else None
        d_g2g = torch.zeros_like(g2g32) if g2g32 is not None else None
        vil_attention_raw_backward(q, k, v, qg, kg, vg, tab32, g2l32, g2g32, o, og, lse, lse_g, d_o, d_og,
                                   dq, dk, dv, dqg, dkg, dvg, d_tab, d_g2l, d_g2g, nx=nx, ny=ny, w=w, exact=exact,
                                   mode=mode, scale=scale, impl=impl, flags=flags, dropout_p=dropout_p,
                                   dropout_seed=seed, dropout_offset=offset, dilation=dilation, _image_hw=ctx.hw)
        cast = lambda d, ref: None if d is None else d.to(ref.dtype)
        return (dq_all, dkv, dqg_all, dkvg, cast(d_tab, table) if table is not None else None,
                cast(d_g2l, g2l) if g2l is not None else None, cast(d_g2g, g2g) if g2g is not None else None,
                None, None, None, None, None, None, None, None, None, None, None, None)


def vil_attention(q_all, kv, qg_all=None, kvg=None, table=None, g2l=None, g2g=None, *, num_heads, nx, ny, w,
                  nglo, exact=0, mode=0, scale=1.0, impl="auto", dropout_p=0.0, dilation=1, image_sizes=None):
    """Fused local+global Vision-Longformer attention.

    shared weights (sharew):   q_all (B, nglo+nx*ny, C) = query(x);          kv (B, N, 2C) = kv(x)
    separate global weights:   q_all (B, nx*ny, C)      = query(x[:, nglo:]); qg_all (B, nglo, C) = query_global(x[:, :nglo]);
                               kvg (B, N, 2C) = kv_global(x)
    returns (B, N, C): rows [0,nglo) = global-token outputs, the rest = local outputs, head-merged.

    Under `torch.autocast('cuda')` the activations are cast to the autocast dtype first (the reference's
    `@autocast()`-decorated SlidingChunk2D does the same, slidingchunk_2d.py:203,235), so an fp32 caller gets the
    tensor-core path and bf16/fp16 outputs; the bias tables stay fp32.

    `dropout_p` in [0, 1): attention dropout on the probabilities (the reference's `attn_drop`, longformer2d.py:186, 224).
    Each call draws a fresh mask from the device's default CUDA generator; the backward reuses it.

    `dilation` d >= 1: dilated sliding-chunk attention.  The local tokens fall into d^2 residue sub-grids (image rows and
    columns congruent mod d); each local query attends to the global tokens and, with the same w / exact / mode / bias
    table, to the keys of its own sub-grid, so its window reaches w * d image positions.  Global queries are unchanged.
    d = 1 is the undilated operator, bit for bit.

    `image_sizes`: per-image token grids of a padded batch (detection batches of images of different sizes).  Host data:
    a sequence of B (h, w) pairs or a CPU integer tensor of shape (B, 2), 1 <= h <= nx, 1 <= w <= ny; image b's real
    tokens are its top-left h x w of the nx x ny grid, in the padded layout.  Each real token gets exactly what the call
    on image b alone, cropped to h x w, gives it (local and global queries, all gradients); the output rows of the
    off-image local tokens are zeros and their gradients are zeros, and the contents of q / kv at those tokens never
    reach any output.  Validated on the host (ValueError / TypeError) and uploaded without a host synchronise; with every
    image at (nx, ny) this is the call without sizes.  Composes with dilation (the crop's residue sub-grids) and dropout.
    """
    if q_all.is_cuda and torch.is_autocast_enabled("cuda"):
        dt = torch.get_autocast_dtype("cuda")
        cast = lambda t: t if (t is None or t.dtype == dt) else t.to(dt)
        q_all, kv, qg_all, kvg = cast(q_all), cast(kv), cast(qg_all), cast(kvg)
    return _VilAttention.apply(q_all, kv, qg_all, kvg, table, g2l, g2g, num_heads, nx, ny, w, nglo, exact, mode,
                               float(scale), impl, float(dropout_p), int(dilation), image_sizes)


class _VilAttentionPacked(torch.autograd.Function):
    """Same operator on the output of ONE fused `qkv` Linear ((B, N, 3*H*D), token 0..nglo-1 = global tokens): the dense
    attention of a wx x wy (+nglo) stage is the single-chunk case of the sliding-chunk operator (w = wx = wy, one chunk,
    every local query sees every local key) - SURVEY.md section 8(f) row 2, reference `Attention` (msvit.py:37-120).
    q / k / v are strided views of `qkv`; the backward writes dq | dk | dv straight into one (B, N, 3*H*D) buffer."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, qkv, table, g2l, g2g, H, nx, ny, w, nglo, scale, dropout_p):
        _require_cuda(qkv, "qkv")
        B, N, C3 = qkv.shape
        C, g = C3 // 3, nglo
        assert g + nx * ny == N, "Global dimension does not match!"
        qkv = qkv if qkv.stride(2) == 1 else qkv.contiguous()
        q_all, kv = qkv[:, :, :C], qkv[:, :, C:]
        k, v = _heads(kv, H, 0, 2), _heads(kv, H, 1, 2)
        q = _heads(q_all, H)[:, :, g:]
        qg = _heads(q_all, H)[:, :, :g] if g > 0 else None
        tab32, g2l32, g2g32 = _f32c(table), _f32c(g2l) if g > 0 else None, _f32c(g2g) if g > 0 else None
        out = torch.empty(B, N, C, dtype=qkv.dtype, device=qkv.device)
        o = _heads(out, H)[:, :, g:]
        og = _heads(out, H)[:, :, :g] if g > 0 else None
        seed, offset = _dropout_state(qkv.device, dropout_p)
        flags = _split_flag(qkv, "auto")
        lse, lse_g = vil_attention_raw_forward(q, k, v, qg, k if g > 0 else None, v if g > 0 else None, tab32, g2l32, g2g32, o, og,
                                               nx=nx, ny=ny, w=w, exact=0, mode=0, scale=scale, flags=flags,
                                               dropout_p=dropout_p, dropout_seed=seed, dropout_offset=offset)
        ctx.save_for_backward(qkv, table, g2l, g2g, out, lse, lse_g)
        ctx.cfg = (H, nx, ny, w, g, scale, flags)
        ctx.drop = (dropout_p, seed, offset)
        return out

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, d_out):
        qkv, table, g2l, g2g, out, lse, lse_g = ctx.saved_tensors
        H, nx, ny, w, g, scale, flags = ctx.cfg
        dropout_p, seed, offset = ctx.drop
        B, N, C3 = qkv.shape
        C = C3 // 3
        d_out = d_out.contiguous()
        d_qkv = torch.empty(B, N, C3, dtype=qkv.dtype, device=qkv.device)
        q_all, kv, dq_all, dkv = qkv[:, :, :C], qkv[:, :, C:], d_qkv[:, :, :C], d_qkv[:, :, C:]
        k, v, dk, dv = _heads(kv, H, 0, 2), _heads(kv, H, 1, 2), _heads(dkv, H, 0, 2), _heads(dkv, H, 1, 2)
        hq, hdq, ho, hdo = _heads(q_all, H), _heads(dq_all, H), _heads(out, H), _heads(d_out, H)
        gsl = lambda t: (t[:, :, g:], t[:, :, :g] if g > 0 else None)
        (q, qg), (dq, dqg), (o, og), (d_o, d_og) = gsl(hq), gsl(hdq), gsl(ho), gsl(hdo)
        tab32 = _f32c(table)
        g2l32, g2g32 = (_f32c(g2l), _f32c(g2g)) if g > 0 else (None, None)
        d_tab = torch.zeros_like(tab32) if tab32 is not None else None
        d_g2l = torch.zeros_like(g2l32) if g2l32 is not None else None
        d_g2g = torch.zeros_like(g2g32) if g2g32 is not None else None
        kg, vg, dkg, dvg = (k, v, dk, dv) if g > 0 else (None, None, None, None)
        vil_attention_raw_backward(q, k, v, qg, kg, vg, tab32, g2l32, g2g32, o, og, lse, lse_g, d_o, d_og, dq, dk, dv, dqg, dkg, dvg,
                                   d_tab, d_g2l, d_g2g, nx=nx, ny=ny, w=w, exact=0, mode=0, scale=scale, flags=flags,
                                   dropout_p=dropout_p, dropout_seed=seed, dropout_offset=offset)
        cast = lambda d, ref: None if (d is None or ref is None) else d.to(ref.dtype)
        return d_qkv, cast(d_tab, table), cast(d_g2l, g2l), cast(d_g2g, g2g), None, None, None, None, None, None, None


def vil_dense_attention(qkv, table=None, g2l=None, g2g=None, *, num_heads, nx, ny, nglo, scale, dropout_p=0.0):
    """Dense attention over nglo + nx*ny tokens (nx == ny == w in {7, 14}: one chunk) with the operator's kernels.
    `table` must already be in the ((4w-1)^2, H) layout of the sliding-chunk operator (see msvit.DenseAttention).
    `dropout_p`: attention dropout as in `vil_attention`; the mask is the sliding-chunk operator's at mode 0, where the one
    chunk is the centre block (offset index 4) of attn1."""
    assert nx == ny, "single-chunk dense attention needs a square token grid"
    if qkv.is_cuda and torch.is_autocast_enabled("cuda"):
        qkv = qkv.to(torch.get_autocast_dtype("cuda"))
    return _VilAttentionPacked.apply(qkv, table, g2l, g2g, num_heads, nx, ny, nx, nglo, float(scale), float(dropout_p))
