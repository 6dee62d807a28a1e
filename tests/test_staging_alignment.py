"""The wgmma family copies operand rows into shared memory with 16-byte cp.async: it serves a call only when D % 8 == 0
and every q / k / v (and, in the backward, d_o) row starts on a 16-byte boundary.  Other calls go to the SIMT family.
The CPU test checks the selection of the forward through vil_attn_wgmma_supported (no pointer is dereferenced); the GPU
tests run calls that take the SIMT family, for both passes or for the backward alone, against the oracle."""
import ctypes

import pytest
import torch

import __graft_entry__ as ge
from vision_longformer_b200 import _lib


def _params(D=32, ptr=1 << 20, st=None, **kw):
    p = _lib.VilAttnParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilAttnParams)
    p.dtype, p.impl = _lib.VIL_BF16, _lib.VIL_IMPL_AUTO
    p.B, p.H, p.D, p.nx, p.ny, p.w, p.nglo, p.exact, p.mode = 2, 3, D, 56, 56, 7, 1, 0, 0
    p.scale = D ** -0.5
    C = 3 * D
    for name in ("q", "k", "v"):
        t = getattr(p, name)
        t.ptr, t.sb, t.sh, t.st = ptr, 3137 * C, D, C if st is None else st
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def test_wgmma_needs_16_byte_aligned_rows():
    ge.build()
    lib = _lib.load()
    ok = lambda **kw: lib.vil_attn_wgmma_supported(ctypes.byref(_params(**kw)))
    for D in (16, 32, 48, 64):                        # every production layout: Linear outputs, strides in whole rows
        assert ok(D=D) == 1, D
    assert ok(D=20) == 0                              # D % 8 != 0
    assert ok(ptr=(1 << 20) + 2) == 0                 # storage offset of one element
    assert ok(st=100) == 0                            # 200-byte token stride


@pytest.mark.gpu
def test_unaligned_call_takes_simt_and_matches_oracle():
    from tests.test_gpu_parity import TOL, check_against, kernel_run, make_inputs, oracle_run
    case = (1, 2, 20, 14, 14, 1, 7, 0, 0, True)       # D = 20: rows of 40 bytes
    B, H, D, nx, ny, g, w, exact, mode, rpe = case
    dtype = torch.bfloat16
    t = make_inputs(B, H, D, nx, ny, g, w, rpe)
    ref = oracle_run(t, nx, ny, w, exact, mode, D ** -0.5, dtype)
    out, fam_f, fam_b = kernel_run(t, nx, ny, w, exact, mode, D ** -0.5, dtype, "auto")
    assert (fam_f, fam_b) == ("simt", "simt")
    tf, tb = TOL[dtype]
    check_against(out, ref, g, rpe, tf, tb, 5e-2, "unaligned_call_takes_simt", case, "bf16/contig")


@pytest.mark.gpu
def test_unaligned_d_o_sends_only_the_backward_to_simt():
    """q, k, v aligned and dO a view at an odd storage offset: the forward runs on wgmma, the backward on SIMT, and the
    mixed pair matches the oracle."""
    from tests.test_gpu_parity import TOL, check_against, make_inputs, oracle_run
    from vision_longformer_b200 import vil_attention_raw_backward, vil_attention_raw_forward
    case = (1, 2, 32, 14, 14, 1, 7, 0, 0, True)
    B, H, D, nx, ny, g, w, exact, mode, rpe = case
    dtype, dev = torch.bfloat16, "cuda"
    t = make_inputs(B, H, D, nx, ny, g, w, rpe)
    ref = oracle_run(t, nx, ny, w, exact, mode, D ** -0.5, dtype)
    cuda = lambda x: x.to(dev, dtype).contiguous()
    q, k, v, qg, gog = cuda(t["q"]), cuda(t["k"]), cuda(t["v"]), cuda(t["qg"]), cuda(t["gog"])
    buf = torch.empty(t["go"].numel() + 1, device=dev, dtype=dtype)
    go = buf[1:].view(t["go"].shape)                  # rows start 2 bytes past a 16-byte boundary
    go.copy_(t["go"])
    assert go.data_ptr() % 16 != 0
    f32 = lambda x: x.to(dev, torch.float32).contiguous()
    table, g2l, g2g = f32(t["table"]), f32(t["g2l"]), f32(t["g2g"])
    o, og = torch.empty_like(q), torch.empty_like(qg)
    dq, dk, dv, dqg = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v), torch.empty_like(qg)
    dt, dgl, dgg = torch.zeros_like(table), torch.zeros_like(g2l), torch.zeros_like(g2g)
    kw = dict(nx=nx, ny=ny, w=w, exact=exact, mode=mode, scale=D ** -0.5, impl="auto")
    lse, lse_g = vil_attention_raw_forward(q, k, v, qg, k, v, table, g2l, g2g, o, og, **kw)
    fam_f = _lib.last_impl()
    vil_attention_raw_backward(q, k, v, qg, k, v, table, g2l, g2g, o, og, lse, lse_g, go, gog, dq, dk, dv, dqg, dk, dv,
                               dt, dgl, dgg, **kw)
    torch.cuda.synchronize()
    assert (fam_f, _lib.last_impl()) == ("wgmma", "simt")
    out = dict(o=o, og=og, lse=lse, lse_g=lse_g, dq=dq, dk=dk, dv=dv, dqg=dqg, dtable=dt, dg2l=dgl, dg2g=dgg)
    tf, tb = TOL[dtype]
    check_against(out, ref, g, rpe, tf, tb, 5e-2, "unaligned_d_o_backward_takes_simt", case, "bf16/contig")
