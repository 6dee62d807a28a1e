"""Dilated sliding-chunk attention (VIL_FLAG_DILATED), the parts that need no GPU: the dilated oracle against the
undilated one and against an image-wide fp64 restatement of the dilated mask, and the host-side validation of the flag
and its word."""
import ctypes

import pytest
import torch

import __graft_entry__ as ge
from oracle.vil_oracle import dense_attention
from tests.dilated_oracle import dilated_attention, dilated_bruteforce, residues
from vision_longformer_b200 import _lib

EXACT_MODES = [(1, 0)] + [(e, m) for e in (0, -1) for m in (-1, 0, 1, 2, 3, 4, 5, 6, 7, 8)]


def _inputs(nx, ny, w, g, H=2, D=5, rpe=True, seed=0):
    gen = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    N = g + nx * ny
    q, k, v = r(1, H, nx * ny, D), r(1, H, N, D), r(1, H, N, D)
    qg, kg, vg = (r(1, H, g, D), r(1, H, N, D), r(1, H, N, D)) if g else (None, None, None)
    table = r((4 * w - 1) ** 2, H) if rpe else None
    g2l = r(2, H, g) if rpe and g else None
    g2g = r(H, g, g) if rpe and g else None
    return q, k, v, qg, kg, vg, table, g2l, g2g


def test_residues_tile_the_image():
    for nx, ny, d in ((13, 10, 3), (2, 9, 3), (8, 8, 2), (1, 1, 4)):
        idx = torch.cat([r[4] for r in residues(nx, ny, d)])
        assert sorted(idx.tolist()) == list(range(nx * ny))
        for a, b, na, nb, _ in residues(nx, ny, d):
            assert (na, nb) == (-(-(nx - a) // d), -(-(ny - b) // d))


@pytest.mark.parametrize("exact,mode", [(1, 0), (0, 0), (0, -1), (0, 3), (-1, 0), (-1, 6)])
def test_d1_is_the_oracle_bitwise(exact, mode):
    x = _inputs(9, 11, 4, 1)
    kw = dict(nx=9, ny=11, w=4, exact=exact, mode=mode, scale=0.4)
    for a, b in zip(dilated_attention(*x, d=1, **kw), dense_attention(*x, **kw)):
        assert torch.equal(a, b)


@pytest.mark.parametrize("exact,mode", EXACT_MODES)
@pytest.mark.parametrize("nx,ny,w,d,g,rpe", [
    (13, 10, 3, 3, 1, True),      # residues of 5x4, 5x3, 4x4, 4x3 tokens: different padding and chunk grids
    (12, 9, 2, 2, 2, True),
    (11, 7, 4, 2, 0, True),
    (2, 9, 2, 3, 1, False),       # d > nx: a residue row class is empty
    (10, 10, 1, 3, 1, True),      # w = 1: one-token chunks
])
def test_dilated_oracle_matches_the_bruteforce_mask(exact, mode, nx, ny, w, d, g, rpe):
    q, k, v, qg, kg, vg, table, g2l, g2g = _inputs(nx, ny, w, g, rpe=rpe, seed=nx * 100 + ny)
    kw = dict(nx=nx, ny=ny, w=w, exact=exact, mode=mode, scale=0.37)
    o, og, lse, lse_g = dilated_attention(q, k, v, qg, kg, vg, table, g2l, g2g, d=d, **kw)
    ob, lseb = dilated_bruteforce(q, k, v, table, g2l, d=d, **kw)
    assert (o - ob).abs().max() < 1e-12 and (lse - lseb).abs().max() < 1e-12
    if g:
        o1, og1, _, lse_g1 = dense_attention(q, k, v, qg, kg, vg, table, g2l, g2g, **kw)
        assert torch.equal(og, og1) and torch.equal(lse_g, lse_g1)


def test_exact_window_reaches_w_times_d():
    """exact = 1 at d = 2: a query sees the key 2w positions away on its own rows and columns, and nothing off its residue"""
    nx = ny = 12
    w, d = 2, 2
    q, k, v, *_ = _inputs(nx, ny, w, 0, H=1, D=3, rpe=False)
    kw = dict(nx=nx, ny=ny, w=w, exact=1, mode=0, scale=1.0, d=d)
    i = 5 * ny + 5
    for j, seen in ((1 * ny + 1, True), (9 * ny + 9, True), (5 * ny + 6, False), (10 * ny + 5, False)):
        v2 = v.clone()
        v2[0, 0, j] += 1.0
        o, _ = dilated_bruteforce(q, k, v, None, None, **kw)
        o2, _ = dilated_bruteforce(q, k, v2, None, None, **kw)
        assert bool((o2[0, 0, i] != o[0, 0, i]).any()) == seen, j


# ---------------------------------------------------------------- host-side ABI
DIL = 16


@pytest.fixture(scope="module")
def lib():
    ge.build()
    return _lib.load()


def _params(flags=0, dilation=0, rpe=False, **kw):
    p = _lib.VilAttnParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilAttnParams)
    p.dtype, p.impl, p.flags, p.dilation = _lib.VIL_BF16, _lib.VIL_IMPL_AUTO, flags, dilation
    p.B, p.H, p.D, p.nx, p.ny, p.w, p.nglo, p.exact, p.mode = 2, 3, 32, 56, 56, 7, 1, 0, 0
    p.scale = 32 ** -0.5
    for name, st in (("q", 96), ("k", 192), ("v", 192), ("d_o", 96)):
        t = getattr(p, name)
        t.ptr, t.sb, t.sh, t.st = 1 << 20, 3137 * st, 32, st
    if rpe:
        p.bias_table, p.g2l, p.g2g = 1 << 21, 1 << 22, 1 << 23
    for key, val in kw.items():
        setattr(p, key, val)
    return p


def test_flag_and_word_leave_the_struct_as_it_was(lib):
    assert lib.vil_attn_abi_version() == 3 == _lib.ABI_VERSION
    assert _lib.VIL_FLAG_DILATED == DIL
    assert DIL & (_lib.VIL_FLAG_F32_OUT | _lib.VIL_FLAG_UNFUSED | _lib.VIL_FLAG_F32_SPLIT) == 0
    # the word is the former padding after dropout_p: same offset, same size, same struct
    assert _lib.VilAttnParams.dilation.offset == _lib.VilAttnParams.dropout_p.offset + 4
    assert _lib.VilAttnParams.dropout_seed.offset == _lib.VilAttnParams.dilation.offset + 4
    assert ctypes.sizeof(_lib.VilAttnParams) == 680


def test_flag_needs_a_positive_dilation(lib):
    for d in (0, -1, -7):
        assert lib.vil_attn_wgmma_supported(ctypes.byref(_params(flags=DIL, dilation=d))) == _lib.VIL_E_BADARG
        assert "dilation" in _lib.last_error()
        assert lib.vil_attn_workspace_bytes(ctypes.byref(_params(flags=DIL, dilation=d)), 1) == _lib.VIL_E_BADARG
    assert lib.vil_attn_wgmma_supported(ctypes.byref(_params(flags=DIL, dilation=1))) == 1
    assert lib.vil_attn_wgmma_supported(ctypes.byref(_params(flags=DIL | 32, dilation=2))) == _lib.VIL_E_BADARG
    assert "unknown bits" in _lib.last_error()


def test_word_is_ignored_without_the_flag(lib):
    for d in (-5, 0, 3):
        for rpe in (False, True):
            for bwd in (0, 1):
                assert lib.vil_attn_workspace_bytes(ctypes.byref(_params(dilation=d, rpe=rpe)), bwd) == \
                    lib.vil_attn_workspace_bytes(ctypes.byref(_params(rpe=rpe)), bwd)
        assert lib.vil_attn_wgmma_supported(ctypes.byref(_params(dilation=d))) == 1


def test_coverage_is_the_same_dilated(lib):
    for D in (8, 12, 32, 64, 128):
        for dt in (_lib.VIL_BF16, _lib.VIL_F32):
            for w in (7, 42, 48):
                base = lib.vil_attn_wgmma_supported(ctypes.byref(_params(D=D, dtype=dt, w=w, rpe=True)))
                for d in (1, 2, 3):
                    assert lib.vil_attn_wgmma_supported(ctypes.byref(_params(D=D, dtype=dt, w=w, rpe=True, flags=DIL,
                                                                             dilation=d))) == base


def _tab_rows(nx, ny, w, d, B=2, H=3):
    """pass-1 CTAs with the bias table (one row of table partials each): the d^2 residues over the largest sub-grid's
    chunk grid, in nslice image slices"""
    cdiv = lambda a, b: -(-a // b)
    mx, my = d * cdiv(cdiv(nx, d), w), d * cdiv(cdiv(ny, d), w)
    npc = cdiv(w * w, 64)
    per = H * mx * my * npc
    nslice = min(B, cdiv(8 * 132, per))
    return nslice * per


def test_workspace_counts_the_residue_table_rows(lib):
    w, tabn = 7, (4 * 7 - 1) ** 2
    base = lib.vil_attn_workspace_bytes(ctypes.byref(_params(rpe=True)), 1)
    for d in (2, 3, 5):
        ws = lib.vil_attn_workspace_bytes(ctypes.byref(_params(rpe=True, flags=DIL, dilation=d)), 1)
        extra = (_tab_rows(56, 56, w, d) - _tab_rows(56, 56, w, 1)) * tabn * 4
        assert abs(ws - base - extra) <= 2 * 64 * 4, (d, ws, base, extra)     # up to the 64-float alignment of parts
        # without the table the workspace does not depend on d
        assert lib.vil_attn_workspace_bytes(ctypes.byref(_params(flags=DIL, dilation=d)), 1) == \
            lib.vil_attn_workspace_bytes(ctypes.byref(_params()), 1)


def test_python_sets_the_flag_only_above_one():
    from vision_longformer_b200 import ops
    q = torch.empty(1, 1, 4, 8)
    for d, flags, word in ((1, 0, 0), (2, DIL, 2), (5, DIL, 5)):
        p = ops._base_params(q, q, 2, 2, 1, 0, 0, 0, 1.0, "auto", dilation=d)
        assert (p.flags, p.dilation) == (flags, word)
    for bad in (0, -1, 1.5):
        with pytest.raises(ValueError):
            ops._base_params(q, q, 2, 2, 1, 0, 0, 0, 1.0, "auto", dilation=bad)


def test_module_accepts_dilation():
    from vision_longformer_b200 import B200Long2DSCSelfAttention
    from vision_longformer_b200.msvit import MsViT
    m = B200Long2DSCSelfAttention(32, num_heads=2, w=4, d=3, rpe=True)
    assert m.attention_dilation == 3
    # the state_dict does not depend on d
    assert {k: v.shape for k, v in m.state_dict().items()} == \
        {k: v.shape for k, v in B200Long2DSCSelfAttention(32, num_heads=2, w=4, d=1, rpe=True).state_dict().items()}
    for bad in (0, -2, 1.5):
        with pytest.raises(ValueError):
            B200Long2DSCSelfAttention(32, num_heads=2, w=4, d=bad)
    # two longformer stages and a dense (s0) one, which has no dilation
    model = MsViT("l1,h2,d16,n1,s1,g1,p4,f4,a0_l2,h2,d32,n2,s1,g1,p2,f4_l3,h2,d32,n1,s0,g1,p2,f7", img_size=32,
                  num_classes=7, d=2)
    longformer = [mod for mod in model.modules() if isinstance(mod, B200Long2DSCSelfAttention)]
    assert len(longformer) == 3 and all(mod.attention_dilation == 2 for mod in longformer)
    assert not any(isinstance(mod, B200Long2DSCSelfAttention) for mod in model.layer3.modules())
