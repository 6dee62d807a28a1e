"""Per-image token grids in a padded batch (vil_attn_fwd_sized_sm100 / _bwd_sized_sm100), the parts that need no GPU:
the cropping fp64 oracle against an independent brute-force mask over the padded grid, the host-side validation of the
sizes, and the sized entry points' refusals before any launch."""
import ctypes

import pytest
import torch

import __graft_entry__ as ge
from oracle.vil_oracle import dense_attention
from tests.sized_oracle import image_index, sized_attention, sized_bruteforce, sized_global_bruteforce
from vision_longformer_b200 import _lib, ops

EXACT_MODES = [(1, 0)] + [(e, m) for e in (0, -1) for m in (-1, 0, 1, 2, 3, 4, 5, 6, 7, 8)]


def _inputs(B, nx, ny, w, g, H=2, D=5, rpe=True, seed=0):
    gen = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    N = g + nx * ny
    q, k, v = r(B, H, nx * ny, D), r(B, H, N, D), r(B, H, N, D)
    qg, kg, vg = (r(B, H, g, D), r(B, H, N, D), r(B, H, N, D)) if g else (None, None, None)
    table = r((4 * w - 1) ** 2, H) if rpe else None
    g2l = r(2, H, g) if rpe and g else None
    g2g = r(H, g, g) if rpe and g else None
    return q, k, v, qg, kg, vg, table, g2l, g2g


@pytest.mark.parametrize("exact,mode", EXACT_MODES)
@pytest.mark.parametrize("nx,ny,w,d,g,rpe,sizes", [
    (11, 9, 3, 1, 1, True, [(11, 9), (7, 5), (1, 9), (11, 1)]),     # full, ragged, 1 x n, n x 1
    (10, 13, 4, 1, 2, True, [(5, 13), (10, 6)]),                    # sizes that are not multiples of w
    (9, 8, 2, 1, 0, False, [(1, 1), (9, 3)]),
    (13, 10, 3, 3, 1, True, [(13, 10), (8, 7), (2, 10)]),           # dilation: the crop's residue sub-grids
    (12, 9, 2, 2, 1, True, [(1, 9), (12, 1), (7, 4)]),
])
def test_sized_oracle_matches_the_bruteforce_mask(exact, mode, nx, ny, w, d, g, rpe, sizes):
    B = len(sizes)
    q, k, v, qg, kg, vg, table, g2l, g2g = _inputs(B, nx, ny, w, g, rpe=rpe, seed=nx * 100 + ny + d)
    kw = dict(nx=nx, ny=ny, w=w, exact=exact, mode=mode, scale=0.37)
    o, og, lse, lse_g = sized_attention(q, k, v, qg, kg, vg, table, g2l, g2g, sizes=sizes, d=d, **kw)
    ob, lseb = sized_bruteforce(q, k, v, table, g2l, sizes=sizes, d=d, **kw)
    assert (o - ob).abs().max() < 1e-12
    on = torch.isfinite(lseb)
    assert torch.equal(on, torch.isfinite(lse)) and (lse[on] - lseb[on]).abs().max() < 1e-12
    for b, (h, wb) in enumerate(sizes):               # the real rows are exactly the on-image tokens
        assert on[b, 0].nonzero().flatten().tolist() == image_index(nx, ny, h, wb).tolist()
    if g:
        ogb, lgb = sized_global_bruteforce(qg, kg, vg, g2l, g2g, nx=nx, ny=ny, sizes=sizes, scale=0.37)
        assert (og - ogb).abs().max() < 1e-12 and (lse_g - lgb).abs().max() < 1e-12


@pytest.mark.parametrize("exact,mode", [(1, 0), (0, 0), (-1, 0), (-1, 5)])
def test_full_sizes_are_the_unsized_oracle(exact, mode):
    x = _inputs(2, 9, 11, 4, 1)
    kw = dict(nx=9, ny=11, w=4, exact=exact, mode=mode, scale=0.4)
    for a, b in zip(sized_attention(*x, sizes=[(9, 11)] * 2, **kw), dense_attention(*x, **kw)):
        assert torch.allclose(a, b, rtol=0, atol=1e-13)


def test_padding_values_do_not_reach_the_oracle():
    nx, ny, sizes = 8, 7, [(5, 3), (8, 7)]
    x = list(_inputs(2, nx, ny, 3, 1))
    ref = sized_attention(*x, nx=nx, ny=ny, w=3, sizes=sizes, exact=-1, scale=0.5)
    off = torch.ones(nx * ny, dtype=torch.bool)
    off[image_index(nx, ny, 5, 3)] = False
    for i in (0, 1, 2, 4, 5):                          # q, k, v, kg, vg at the off-image tokens of image 0
        t = x[i].clone()
        t[0, :, off.nonzero().flatten() + (0 if i == 0 else 1)] = float("nan")    # k / v rows: after the global token
        x2 = list(x)
        x2[i] = t
        for a, b in zip(sized_attention(*x2, nx=nx, ny=ny, w=3, sizes=sizes, exact=-1, scale=0.5), ref):
            assert torch.equal(a, b)


# ---------------------------------------------------------------- host-side validation (ops)
def test_host_validation_accepts_sequences_and_cpu_tensors():
    want = torch.tensor([[3, 4], [5, 1]], dtype=torch.int32)
    for sizes in ([(3, 4), (5, 1)], ((3, 4), [5, 1]), torch.tensor([[3, 4], [5, 1]]),
                  torch.tensor([[3, 4], [5, 1]], dtype=torch.int16)):
        t = ops.image_sizes_host(sizes, 2, 5, 6)
        assert t.dtype == torch.int32 and torch.equal(t, want)
    assert ops.image_sizes_host(None, 2, 5, 6) is None
    # every image full: the unsized call
    assert ops.image_sizes_host([(5, 6), (5, 6)], 2, 5, 6) is None


@pytest.mark.parametrize("sizes,msg", [
    ([(3, 4)], "shape"),
    ([(3, 4), (5, 1), (2, 2)], "shape"),
    ([(3, 4, 1), (5, 1, 1)], "shape"),
    ([(0, 4), (5, 1)], r"image_sizes\[0\] = \(0, 4\) is outside \[1, 5\] x \[1, 6\]"),
    ([(3, 4), (6, 1)], r"image_sizes\[1\]"),
    ([(3, 7), (5, 1)], r"image_sizes\[0\]"),
    ([(3, -1), (5, 1)], r"image_sizes\[0\]"),
])
def test_host_validation_refuses_bad_shapes_and_ranges(sizes, msg):
    with pytest.raises(ValueError, match=msg):
        ops.image_sizes_host(sizes, 2, 5, 6)


def test_host_validation_refuses_non_integers_and_device_tensors():
    for bad in ([(3.0, 4), (5, 1)], torch.tensor([[3.0, 4.0], [5.0, 1.0]]), torch.ones(2, 2, dtype=torch.bool)):
        with pytest.raises(TypeError, match="integer"):
            ops.image_sizes_host(bad, 2, 5, 6)
    with pytest.raises(TypeError, match="host data"):
        ops.image_sizes_host(torch.ones(2, 2, dtype=torch.int32, device="meta"), 2, 5, 6)


# ---------------------------------------------------------------- the sized entry points
@pytest.fixture(scope="module")
def lib():
    ge.build()
    return _lib.load()


def _params(**kw):
    p = _lib.VilAttnParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilAttnParams)
    p.dtype, p.impl = _lib.VIL_BF16, _lib.VIL_IMPL_AUTO
    p.B, p.H, p.D, p.nx, p.ny, p.w, p.nglo, p.exact, p.mode = 2, 3, 32, 56, 56, 7, 1, 0, 0
    p.scale = 32 ** -0.5
    for name, st in (("q", 96), ("k", 192), ("v", 192), ("d_o", 96)):
        t = getattr(p, name)
        t.ptr, t.sb, t.sh, t.st = 1 << 20, 3137 * st, 32, st
    for key, val in kw.items():
        setattr(p, key, val)
    return p


def test_abi_is_unchanged(lib):
    assert lib.vil_attn_abi_version() == 3 == _lib.ABI_VERSION
    assert ctypes.sizeof(_lib.VilAttnParams) == 680
    assert (_lib.VIL_FLAG_F32_OUT, _lib.VIL_FLAG_UNFUSED, _lib.VIL_FLAG_F32_SPLIT, _lib.VIL_FLAG_DILATED) == (1, 2, 4, 16)
    for sym in ("vil_attn_fwd_sized_sm100", "vil_attn_bwd_sized_sm100"):
        assert sym in _lib.EXPORTS and hasattr(lib, sym)


def test_sized_entry_points_refuse_before_any_launch(lib):
    hw = ctypes.c_void_p(1 << 24)                         # never dereferenced: every call below fails on the host
    before = _lib.launch_count()
    for fn in (lib.vil_attn_fwd_sized_sm100, lib.vil_attn_bwd_sized_sm100):
        assert fn(ctypes.byref(_params()), None, None) == _lib.VIL_E_BADARG
        assert "image_hw is NULL" in _lib.last_error()
        assert fn(None, hw, None) == _lib.VIL_E_BADARG
        assert fn(ctypes.byref(_params(exact=2)), hw, None) == _lib.VIL_E_BADARG
        assert "exact" in _lib.last_error()
        assert fn(ctypes.byref(_params(flags=32)), hw, None) == _lib.VIL_E_BADARG
        assert "unknown bits" in _lib.last_error()
        assert fn(ctypes.byref(_params(flags=_lib.VIL_FLAG_DILATED, dilation=0)), hw, None) == _lib.VIL_E_BADARG
        p = _params()
        p.q.ptr = None
        assert fn(ctypes.byref(p), hw, None) == _lib.VIL_E_BADARG
        assert "tensor q is NULL" in _lib.last_error()
    # the backward's workspace check comes first too
    assert lib.vil_attn_bwd_sized_sm100(ctypes.byref(_params(o=_lib.VilTensor4(1 << 20, 0, 0, 0), lse=1 << 20,
                                                             dq=_lib.VilTensor4(1 << 20, 0, 0, 0),
                                                             dk=_lib.VilTensor4(1 << 20, 0, 0, 0),
                                                             dv=_lib.VilTensor4(1 << 20, 0, 0, 0),
                                                             nglo=0)), hw, None) == _lib.VIL_E_WORKSPACE
    assert _lib.launch_count() == before


def test_module_signature_takes_image_sizes():
    import inspect
    from vision_longformer_b200 import B200Long2DSCSelfAttention
    from vision_longformer_b200.msvit import DenseAttention
    sig = inspect.signature(B200Long2DSCSelfAttention.forward)
    assert list(sig.parameters)[1:] == ["x", "nx", "ny", "defer_proj_bias", "image_sizes"]
    assert sig.parameters["image_sizes"].default is None
    assert "image_sizes" in inspect.signature(ops.vil_attention).parameters
    # the dense single-chunk path has no sizes
    assert "image_sizes" not in inspect.signature(ops.vil_dense_attention).parameters
    assert "image_sizes" not in inspect.signature(DenseAttention.forward).parameters
