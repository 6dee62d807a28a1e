"""Attention dropout (`attn_drop` > 0) of the fused sliding-chunk attention.

The mask is a pure function of the reference's coordinates (include/vil_attn.h, "attention dropout"): a numpy
restatement of it here builds the keep tensors of the reference's attn1 / attn0, and an fp64 chunked reference (the
reference's own per-column algorithm, as oracle/vil_oracle.py::chunked_attention, with the probabilities multiplied by
those tensors as `self.attn_drop` does at longformer2d.py:186, 224) is compared with both kernel families.

CPU tests: the Philox restatement (Random123 known-answer vectors), the keep rate, the ABI's argument checks.
GPU tests: oracle parity with the exact mask, agreement of the two families, the generator contract, p = 0 is the
path without dropout, and module-level training.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import vil_oracle as vo
from tests.util import record, relerr
from vision_longformer_b200 import _lib, vil_attention_raw_backward, vil_attention_raw_forward

DEV = "cuda"
gpu = pytest.mark.gpu

# --------------------------------------------------------------------------- numpy restatement of the mask
_M0, _M1, _W0, _W1, _U32 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85, 0xFFFFFFFF


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint32 arrays (broadcast): returns the four output words."""
    c = [np.asarray(x, dtype=np.uint64) & _U32 for x in (c0, c1, c2, c3)]
    c0, c1, c2, c3 = np.broadcast_arrays(*c)
    k0, k1 = np.uint64(k0 & _U32), np.uint64(k1 & _U32)
    for _ in range(10):
        p0, p1 = np.uint64(_M0) * c0, np.uint64(_M1) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & np.uint64(_U32), (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & np.uint64(_U32)
        k0, k1 = (k0 + np.uint64(_W0)) & np.uint64(_U32), (k1 + np.uint64(_W1)) & np.uint64(_U32)
    return c0, c1, c2, c3


def threshold(p):
    return min(math.floor(p * 2.0 ** 32), 2 ** 32 - 1)


def keep_bits(row, col, sid, seed, offset, p):
    """The kernels' keep decision for elements (row, col) of stream id sid = 2 (b H + h) + stream."""
    row, col, sid = np.broadcast_arrays(np.asarray(row, np.int64), np.asarray(col, np.int64), np.asarray(sid, np.int64))
    x = philox4x32_10(col >> 2, row, sid, offset & _U32, seed & _U32, seed >> 32)
    u = np.choose(col & 3, x)
    return u >= np.uint64(threshold(p))


def keep_tensors(seed, offset, p, B, H, nx, ny, w, g, mode):
    """m / (1 - p) in the layouts of the reference's attn1 (B*H, mx, my, w2, g + n*w2) and attn0 (B*H, g, N)."""
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    w2, n = w * w, len(vo.mode_offsets(mode))
    sc = np.float32(1.0) / (np.float32(1.0) - np.float32(p))
    R, C, l = np.meshgrid(np.arange(mx), np.arange(my), np.arange(w2), indexing="ij")
    qr, qc = R * w + l // w, C * w + l % w
    row = np.where((qr < nx) & (qc < ny), qr * ny + qc, 0)                          # padded rows are cropped anyway
    col = np.arange(g + n * w2)
    bh = np.arange(B * H)
    k1 = keep_bits(row[None, ..., None], col[None, None, None, None, :], 2 * bh[:, None, None, None, None], seed, offset, p)
    keep = torch.from_numpy(k1.astype(np.float64) * float(sc))
    keep_g = None
    if g:
        N = g + nx * ny
        k0 = keep_bits(np.arange(g)[None, :, None], np.arange(N)[None, None, :], 2 * bh[:, None, None] + 1, seed, offset, p)
        keep_g = torch.from_numpy(k0.astype(np.float64) * float(sc))
    return keep, keep_g


def chunked_dropout_reference(q, k, v, qg, kg, vg, table, g2l, g2g, keep, keep_g, *, nx, ny, w, exact, mode, scale):
    """The reference's per-column algorithm (longformer2d.py:126-227, as oracle.vil_oracle.chunked_attention) with
    attn1 / attn0 multiplied by keep / keep_g after the softmax (longformer2d.py:186, 224).  Differentiable."""
    B, H, Nloc, D = q.shape
    N = k.shape[2]
    g = N - Nloc
    w2 = w * w
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    offs = vo.mode_offsets(mode)

    def to_chunks(t):
        img = t.reshape(B * H, nx, ny, D).permute(0, 3, 1, 2)
        if padx or pady:
            img = torch.nn.functional.pad(img, (0, pady, 0, padx))
        return img.reshape(B * H, D, mx, w, my, w).permute(0, 1, 2, 4, 3, 5).reshape(B * H, D, mx, my, w2)

    qc, kc, vc = to_chunks(q * scale), to_chunks(k[:, :, g:]), to_chunks(v[:, :, g:])
    s = vo._ChunkProduct.scores(qc, kc, offs)
    if table is not None:
        rpi = vo.relative_position_index(w)
        pos = {o: i for i, o in enumerate(vo.OFFSETS9)}
        rpi = torch.cat([rpi[:, pos[o] * w2:(pos[o] + 1) * w2] for o in offs], dim=-1)
        bias = table[rpi.reshape(-1)].reshape(w2, len(offs) * w2, H).permute(2, 0, 1)
        s = s + bias[None].expand(B, -1, -1, -1).reshape(B * H, 1, 1, w2, -1)
    s = s.masked_fill(vo.chunk_mask(nx, ny, w, exact, mode), float("-inf"))
    if g:
        s_glo = torch.einsum("bcmnl,btc->bmnlt", qc, k[:, :, :g].reshape(B * H, g, D))
        if g2l is not None:
            s_glo = s_glo + g2l[1][None].expand(B, -1, -1).reshape(B * H, 1, 1, 1, g)
        s = torch.cat([s_glo, s], dim=-1)
    p = s.softmax(dim=-1) * keep
    ctx = vo._ChunkProduct.context(p[..., g:], vc, offs)
    if g:
        ctx = ctx + torch.einsum("bmnlt,btc->bcmnl", p[..., :g], v[:, :, :g].reshape(B * H, g, D))
    ctx = ctx.reshape(B * H, D, mx, my, w, w).permute(0, 2, 4, 3, 5, 1).reshape(B * H, mx * w, my * w, D)
    o = ctx[:, :nx, :ny].reshape(B, H, Nloc, D)
    if not g:
        return o, None
    sg = torch.einsum("bhad,bhjd->bhaj", qg * scale, kg)
    if g2g is not None:
        sg = sg + torch.cat([g2g, g2l[0][:, :, None].expand(H, g, Nloc)], dim=-1)[None]
    pg = sg.softmax(dim=-1) * keep_g.reshape(B, H, g, N)
    return o, torch.einsum("bhaj,bhjd->bhad", pg, vg)


# --------------------------------------------------------------------------- CPU tests
def test_philox_known_answer_vectors():
    """Random123's kat_vectors for philox4x32_10"""
    def kat(ctr, key):
        return [int(np.asarray(x)) for x in philox4x32_10(*ctr, *key)]
    assert kat((0, 0, 0, 0), (0, 0)) == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    assert kat((_U32,) * 4, (_U32, _U32)) == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    assert kat((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0)) == \
        [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_rate(p):
    n = 10 ** 6
    idx = np.arange(n)
    kept = keep_bits(idx // 1000, idx % 1000, 6, seed=0x1234567890ab, offset=17, p=p).mean()
    assert abs(kept - (1 - p)) < 5 * math.sqrt(p * (1 - p) / n), kept


def _params(**kw):
    p = _lib.VilAttnParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilAttnParams)
    p.dtype, p.impl = _lib.VIL_BF16, _lib.VIL_IMPL_AUTO
    p.B, p.H, p.D, p.nx, p.ny, p.w, p.nglo, p.exact, p.mode = 2, 3, 32, 56, 56, 7, 1, 0, 0
    p.scale = 32 ** -0.5
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def test_abi_validates_dropout_p():
    import __graft_entry__ as ge
    ge.build()
    lib = _lib.load()
    assert lib.vil_attn_abi_version() == 3 == _lib.ABI_VERSION
    for bad in (-0.1, 1.0, 1.5, float("nan")):
        assert lib.vil_attn_workspace_bytes(ctypes.byref(_params(dropout_p=bad)), 0) == _lib.VIL_E_BADARG, bad
        assert "dropout_p" in _lib.last_error()
    for good in (0.0, 0.1, 0.999):
        assert lib.vil_attn_workspace_bytes(ctypes.byref(_params(dropout_p=good)), 1) > 0
    # the wgmma family covers the same configurations with and without dropout
    for dt in (_lib.VIL_BF16, _lib.VIL_F32):
        assert lib.vil_attn_wgmma_supported(ctypes.byref(_params(dtype=dt, dropout_p=0.3))) == \
            lib.vil_attn_wgmma_supported(ctypes.byref(_params(dtype=dt)))


# --------------------------------------------------------------------------- GPU: op parity with the exact mask
def make_inputs(B, H, D, nx, ny, g, w, rpe, sep, seed=300):
    gen = torch.Generator().manual_seed(seed)
    N = g + nx * ny
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    t = dict(q=r(B, H, nx * ny, D), k=r(B, H, N, D), v=r(B, H, N, D), qg=r(B, H, g, D),
             table=0.5 * r((4 * w - 1) ** 2, H) if rpe else None,
             g2l=0.5 * r(2, H, g) if (rpe and g) else None, g2g=0.5 * r(H, g, g) if (rpe and g) else None,
             go=r(B, H, nx * ny, D), gog=r(B, H, g, D))
    t["kg"], t["vg"] = (r(B, H, N, D), r(B, H, N, D)) if sep else (t["k"], t["v"])
    return t


def reference_run(t, cfg, dtype, keep, keep_g):
    nx, ny, w, exact, mode, scale = cfg
    sep = t["kg"] is not t["k"]
    rd = lambda x: None if x is None else x.to(dtype).double().requires_grad_(True)
    q, k, v, qg = rd(t["q"]), rd(t["k"]), rd(t["v"]), rd(t["qg"])
    kg, vg = (rd(t["kg"]), rd(t["vg"])) if sep else (k, v)
    table, g2l, g2g = [None if t[n] is None else t[n].float().double().requires_grad_(True) for n in ("table", "g2l", "g2g")]
    g = k.shape[2] - q.shape[2]
    o, og = chunked_dropout_reference(q, k, v, qg, kg, vg, table, g2l, g2g, keep, keep_g, nx=nx, ny=ny, w=w, exact=exact,
                                      mode=mode, scale=scale)
    loss = (o * t["go"].to(dtype).double()).sum() + ((og * t["gog"].to(dtype).double()).sum() if g else 0)
    names = ["q", "k", "v"] + (["qg"] + (["kg", "vg"] if sep else []) if g else []) + \
        [n for n in ("table", "g2l", "g2g") if t[n] is not None]
    ins = dict(q=q, k=k, v=v, qg=qg, kg=kg, vg=vg, table=table, g2l=g2l, g2g=g2g)
    grads = torch.autograd.grad(loss, [ins[n] for n in names])
    return dict(o=o, og=og, **{"d" + n: gr for n, gr in zip(names, grads)})


def kernel_run(t, cfg, dtype, impl, drop, f32out=False):
    """one forward + backward through the C ABI with dropout (p, seed, offset); contiguous (B, H, T, D) tensors"""
    nx, ny, w, exact, mode, scale = cfg
    p, seed, offset = drop
    sep = t["kg"] is not t["k"]
    B, H, Nloc, D = t["q"].shape
    g = t["k"].shape[2] - Nloc
    odt = torch.float32 if f32out else dtype
    dev = lambda x: x.to(DEV, dtype).contiguous()
    f32 = lambda x: None if x is None else x.to(DEV, torch.float32).contiguous()
    q, k, v, go = dev(t["q"]), dev(t["k"]), dev(t["v"]), dev(t["go"])
    qg, gog = (dev(t["qg"]), dev(t["gog"])) if g else (None, None)
    kg, vg = ((dev(t["kg"]), dev(t["vg"])) if sep else (k, v)) if g else (None, None)
    table, g2l, g2g = f32(t["table"]), f32(t["g2l"]), f32(t["g2g"])
    o = torch.empty_like(q, dtype=odt)
    og = torch.empty_like(qg, dtype=odt) if g else None
    kw = dict(nx=nx, ny=ny, w=w, exact=exact, mode=mode, scale=scale, impl=impl,
              flags=_lib.VIL_FLAG_F32_OUT if f32out else 0, dropout_p=p, dropout_seed=seed, dropout_offset=offset)
    lse, lse_g = vil_attention_raw_forward(q, k, v, qg, kg, vg, table, g2l, g2g, o, og, **kw)
    fam = _lib.last_impl()
    e = lambda x: None if x is None else torch.empty_like(x, dtype=odt)
    dq, dk, dv, dqg = e(q), e(k), e(v), e(qg)
    dkg, dvg = ((e(kg), e(vg)) if sep else (dk, dv)) if g else (None, None)
    z = lambda x: None if x is None else torch.zeros_like(x)
    dt, dgl, dgg = z(table), z(g2l), z(g2g)
    vil_attention_raw_backward(q, k, v, qg, kg, vg, table, g2l, g2g, o, og, lse, lse_g, go, gog, dq, dk, dv, dqg, dkg, dvg,
                               dt, dgl, dgg, **kw)
    torch.cuda.synchronize()
    assert _lib.last_impl() == fam
    out = dict(o=o, og=og, dq=dq, dk=dk, dv=dv, dqg=dqg, dtable=dt, dg2l=dgl, dg2g=dgg)
    if g and sep:
        out.update(dkg=dkg, dvg=dvg)
    return out, fam


DROP_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, rpe, separate global weights, p
    (2, 2, 32, 14, 14, 1, 7, 0, 0, True, False, 0.1),
    (1, 2, 64, 15, 13, 2, 7, 0, 0, False, True, 0.5),     # padding, D = 64, separate global weights
    (1, 2, 32, 16, 24, 0, 8, 0, 0, True, False, 0.1),     # w = 8, no global tokens
    (1, 2, 32, 14, 15, 1, 7, 1, 0, True, True, 0.5),      # exact window
    (1, 2, 32, 10, 9, 2, 4, -1, 0, True, False, 0.1),     # cyclic chunks with padding
    (1, 2, 32, 8, 5, 1, 4, -1, 0, False, True, 0.5),      # mx = my = 2: two offsets reach the same chunk (per-column draws)
    (1, 2, 32, 15, 13, 1, 7, 0, 3, True, False, 0.5),     # random-shift mode 3
    (1, 2, 64, 15, 13, 2, 7, 0, -1, False, False, 0.1),   # own chunk only
]
CASE_ID = lambda c: "B%d_H%d_D%d_%dx%d_g%d_w%d_e%d_m%d_%s_%s_p%g" % (c[:9] + ("rpe" if c[9] else "nob", "sep" if c[10] else "shared", c[11]))
# family, dtype, VIL_FLAG_F32_OUT, forward bar, backward bar, bias-gradient bar
VARIANTS = {
    "simt_fp32": ("simt", torch.float32, False, 1e-5, 2e-5, 1e-4),
    "wgmma_fp16_f32out": ("wgmma", torch.float16, True, 1e-3, 1e-3, 1e-2),
    "wgmma_bf16_f32out": ("wgmma", torch.bfloat16, True, 2e-3, 2e-3, 5e-2),
    "wgmma_bf16": ("wgmma", torch.bfloat16, False, 4e-3, 8e-3, 5e-2),
}
SEED, OFFSET = 0x5eed0000cafe, 1234


@gpu
@pytest.mark.parametrize("case", DROP_CASES, ids=CASE_ID)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_dropout_matches_reference_with_the_exact_mask(case, variant):
    B, H, D, nx, ny, g, w, exact, mode, rpe, sep, p = case
    impl, dtype, f32out, tf, tb, tbias = VARIANTS[variant]
    t = make_inputs(B, H, D, nx, ny, g, w, rpe, sep)
    cfg = (nx, ny, w, exact, mode, D ** -0.5)
    keep, keep_g = keep_tensors(SEED, OFFSET, p, B, H, nx, ny, w, g, mode)
    ref = reference_run(t, cfg, dtype, keep, keep_g)
    out, fam = kernel_run(t, cfg, dtype, impl, (p, SEED, OFFSET), f32out)
    assert fam == impl
    names = ["o", "dq", "dk", "dv"] + (["og", "dqg"] + (["dkg", "dvg"] if sep else []) if g else []) + \
        (["dtable"] + (["dg2l", "dg2g"] if g else []) if rpe else [])
    errs = {n: relerr(out[n], ref[n]) for n in names}
    record("dropout_matches_reference", CASE_ID(case) + "/" + variant, **errs)
    for n, e in errs.items():
        bar = tf if n in ("o", "og") else tbias if n in ("dtable", "dg2l", "dg2g") else tb
        assert e < bar, (n, errs)


@gpu
def test_mask_differs_from_a_shifted_mask():
    """the kernels' mask is the restated one, not merely some mask: the same run against a reference given the mask of
    another offset is off by O(1)"""
    case = DROP_CASES[0]
    B, H, D, nx, ny, g, w, exact, mode, rpe, sep, p = case
    t = make_inputs(B, H, D, nx, ny, g, w, rpe, sep)
    cfg = (nx, ny, w, exact, mode, D ** -0.5)
    out, _ = kernel_run(t, cfg, torch.float32, "simt", (p, SEED, OFFSET))
    keep, keep_g = keep_tensors(SEED, OFFSET + 1, p, B, H, nx, ny, w, g, mode)
    ref = reference_run(t, cfg, torch.float32, keep, keep_g)
    assert relerr(out["o"], ref["o"]) > 0.05


@gpu
@pytest.mark.parametrize("case", [DROP_CASES[0], DROP_CASES[1], DROP_CASES[5]], ids=CASE_ID)
def test_both_families_draw_the_same_mask(case):
    B, H, D, nx, ny, g, w, exact, mode, rpe, sep, p = case
    t = make_inputs(B, H, D, nx, ny, g, w, rpe, sep, seed=301)
    t = {n: (None if x is None else x.to(torch.bfloat16).double()) if n not in ("table", "g2l", "g2g") else x for n, x in t.items()}
    if not sep:
        t["kg"], t["vg"] = t["k"], t["v"]
    cfg = (nx, ny, w, exact, mode, D ** -0.5)
    a, fa = kernel_run(t, cfg, torch.float32, "simt", (p, 99, 7))
    b, fb = kernel_run(t, cfg, torch.bfloat16, "wgmma", (p, 99, 7), f32out=True)
    assert (fa, fb) == ("simt", "wgmma")
    errs = {n: relerr(b[n], a[n]) for n in a if a[n] is not None}
    record("dropout_families_agree", CASE_ID(case), **errs)
    for n, e in errs.items():      # the bf16 bars: 4e-3 forward, 8e-3 backward
        assert e < (5e-2 if n in ("dtable", "dg2l", "dg2g") else 4e-3 if n in ("o", "og") else 8e-3), (n, errs)


# --------------------------------------------------------------------------- GPU: the generator contract and p = 0
def _module(attn_drop, **kw):
    from vision_longformer_b200 import B200Long2DSCSelfAttention
    torch.manual_seed(5)
    return B200Long2DSCSelfAttention(96, num_heads=3, qkv_bias=True, attn_drop=attn_drop, w=7, nglo=1, sharew=True, **kw).to(DEV)


def _fwd_bwd(mod, x, gy, nx=14, ny=14):
    xx = x.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = mod(xx, nx, ny)
    (y.float() * gy).sum().backward()
    return y.detach(), xx.grad


@gpu
def test_generator_contract():
    mod = _module(0.1).train()
    x = torch.randn(2, 1 + 14 * 14, 96, device=DEV)
    gy = torch.randn_like(x)
    torch.manual_seed(11)
    y1, g1 = _fwd_bwd(mod, x, gy)
    torch.manual_seed(11)
    y2, g2 = _fwd_bwd(mod, x, gy)
    assert torch.equal(y1, y2) and torch.equal(g1, g2)          # manual_seed reproduces the mask
    y3, _ = _fwd_bwd(mod, x, gy)
    assert not torch.equal(y1, y3)                              # a second call draws a new one
    # the backward uses its forward's mask, whatever ran in between
    torch.manual_seed(11)
    xx = x.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = mod(xx, 14, 14)
        mod(x, 14, 14)
    (y.float() * gy).sum().backward()
    assert torch.equal(y.detach(), y1) and torch.equal(xx.grad, g1)


@gpu
def test_no_host_sync_with_dropout():
    mod = _module(0.1).train()
    x = torch.randn(2, 1 + 14 * 14, 96, device=DEV, requires_grad=True)
    gy = torch.randn_like(x)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = mod(x, 14, 14)
        (y.float() * gy).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


@gpu
def test_p0_is_the_path_without_dropout():
    from tests import test_gpu_parity as tp
    case = DROP_CASES[0]                        # shared global weights, as test_gpu_parity's runner
    B, H, D, nx, ny, g, w, exact, mode, rpe, sep, _ = case
    t = make_inputs(B, H, D, nx, ny, g, w, rpe, sep)
    cfg = (nx, ny, w, exact, mode, D ** -0.5)
    for impl, dtype in (("simt", torch.float32), ("wgmma", torch.bfloat16)):
        a, _ = kernel_run(t, cfg, dtype, impl, (0.0, SEED, OFFSET))
        b, _, _ = tp.kernel_run(t, nx, ny, w, exact, mode, D ** -0.5, dtype, impl)     # no dropout arguments at all
        for n in ("o", "og", "dq", "dk", "dv", "dqg"):
            assert torch.equal(a[n], b[n]), (impl, n)
        for n in ("dtable", "dg2l", "dg2g"):    # accumulated with atomics: equal up to the order of the fp32 additions
            assert relerr(a[n], b[n]) < 1e-5, (impl, n)
    # eval() with attn_drop > 0 is bitwise the module without dropout
    x = torch.randn(2, 1 + 14 * 14, 96, device=DEV)
    gy = torch.randn_like(x)
    ya, ga = _fwd_bwd(_module(0.1).eval(), x, gy)
    yb, gb = _fwd_bwd(_module(0.0).eval(), x, gy)
    assert torch.equal(ya, yb) and torch.equal(ga, gb)
    # and dropout adds no launch to the operator: 2 forward + 5 backward
    from vision_longformer_b200 import vil_attention
    q = torch.randn(2, 1 + 14 * 14, 96, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    kv = torch.randn(2, 1 + 14 * 14, 192, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    before = _lib.launch_count()
    y = vil_attention(q, kv, num_heads=3, nx=14, ny=14, w=7, nglo=1, scale=32 ** -0.5, dropout_p=0.1)
    y.float().sum().backward()
    torch.cuda.synchronize()
    assert _lib.launch_count() - before == 7


@gpu
def test_p0_op_call_is_bitwise_the_default_call():
    from vision_longformer_b200 import vil_attention
    torch.manual_seed(3)
    B, nx, ny, H, D = 2, 14, 14, 3, 32
    q = torch.randn(B, 1 + nx * ny, H * D, device=DEV, dtype=torch.bfloat16)
    kv = torch.randn(B, 1 + nx * ny, 2 * H * D, device=DEV, dtype=torch.bfloat16)
    kw = dict(num_heads=H, nx=nx, ny=ny, w=7, nglo=1, scale=D ** -0.5)
    assert torch.equal(vil_attention(q, kv, **kw), vil_attention(q, kv, dropout_p=0.0, **kw))


@gpu
def test_dropout_one_leaves_only_the_projection_bias():
    mod = _module(1.0).train()
    x = torch.randn(2, 1 + 14 * 14, 96, device=DEV, requires_grad=True)
    y = mod(x, 14, 14)
    assert torch.equal(y, mod.proj.bias.detach().expand_as(y))
    y.sum().backward()
    assert mod.proj.bias.grad is not None and mod.query.weight.grad is None


# --------------------------------------------------------------------------- GPU: module level
@gpu
def test_module_trains_with_dropout_at_vil_small_stage1():
    from vision_longformer_b200 import B200Long2DSCSelfAttention
    torch.manual_seed(6)
    mod = B200Long2DSCSelfAttention(96, num_heads=3, qkv_bias=True, attn_drop=0.1, w=7, nglo=1, sharew=True).to(DEV).train()
    x = torch.randn(4, 1 + 56 * 56, 96, device=DEV, requires_grad=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = mod(x, 56, 56)
    y.float().square().mean().backward()
    assert _lib.last_impl() == "wgmma"
    assert torch.isfinite(y.float()).all() and torch.isfinite(x.grad).all()
    for n, p_ in mod.named_parameters():
        assert p_.grad is not None and torch.isfinite(p_.grad).all(), n


@gpu
def test_vil_small_trains_with_attn_drop_rate():
    from vision_longformer_b200 import build_vil

    def grads_of(rate, steps):
        torch.manual_seed(7)
        net = build_vil("vil_small", attn_drop_rate=rate, num_classes=10).to(DEV).train()
        opt = torch.optim.SGD(net.parameters(), lr=1e-3, momentum=0.9)
        x = torch.randn(4, 3, 224, 224, device=DEV)
        lab = torch.randint(0, 10, (4,), device=DEV)
        losses, has = [], {}
        for _ in range(steps):
            opt.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = torch.nn.functional.cross_entropy(net(x).float(), lab)
            loss.backward()
            has = {n: p.grad for n, p in net.named_parameters() if p.grad is not None}
            opt.step()
            losses.append(loss.item())
        return losses, has

    _, base = grads_of(0.0, 1)
    losses, got = grads_of(0.1, 3)
    assert all(math.isfinite(l) for l in losses), losses
    for n in base:
        assert n in got and torch.isfinite(got[n]).all(), n


@gpu
def test_dense_attention_vil_with_dropout_matches_the_masked_reference():
    """DenseAttention(impl="vil") is the single-chunk case of the operator (mode 0, the chunk is block 4 of attn1)"""
    from vision_longformer_b200.msvit import DenseAttention
    torch.manual_seed(8)
    dim, H, w, g, p = 64, 2, 7, 1, 0.1
    mod = DenseAttention(dim, num_heads=H, qkv_bias=True, attn_drop=p, wx=w, wy=w, nglo=g, impl="vil").to(DEV).train()
    x = torch.randn(2, g + w * w, dim, device=DEV)
    gy = torch.randn_like(x)
    xm = x.clone().requires_grad_(True)
    gen = torch.cuda.default_generators[torch.device(DEV).index or 0]
    torch.manual_seed(9)
    seed, offset = gen.initial_seed(), gen.get_offset() // 4
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = mod(xm)
    (y.float() * gy).sum().backward()
    assert gen.get_offset() // 4 == offset + 1
    # reference: the same module in fp64 with the chunked per-column algorithm and the restated mask
    B, N, C, D = 2, g + w * w, dim, dim // H
    W = {n: p_.detach().double().cpu().requires_grad_(True) for n, p_ in mod.named_parameters()}
    xr = x.double().cpu().requires_grad_(True)
    qkv = torch.nn.functional.linear(xr, W["qkv.weight"], W["qkv.bias"]).view(B, N, 3, H, D).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    keep, keep_g = keep_tensors(seed, offset, p, B, H, w, w, w, g, 0)
    o, og = chunked_dropout_reference(q[:, :, g:], k, v, q[:, :, :g], k, v, None, None, None, keep, keep_g, nx=w, ny=w, w=w,
                                      exact=0, mode=0, scale=mod.scale)
    out = torch.cat([og, o], dim=2).transpose(1, 2).reshape(B, N, C)
    yr = torch.nn.functional.linear(out, W["proj.weight"], W["proj.bias"])
    (yr * gy.double().cpu()).sum().backward()
    errs = dict(y=relerr(y, yr), dx=relerr(xm.grad, xr.grad), dqkv_w=relerr(mod.qkv.weight.grad, W["qkv.weight"].grad))
    record("dense_attention_vil_dropout", "w7_g1", **errs)
    assert errs["y"] < 3e-2 and errs["dx"] < 6e-2 and errs["dqkv_w"] < 6e-2, errs
