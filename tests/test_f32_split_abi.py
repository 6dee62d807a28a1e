"""fp32 attention on the wgmma tensor cores as split bf16 products (VIL_FLAG_F32_SPLIT), the parts that need no GPU:
the flag's validation, the ABI version, which calls the split kernels cover (vil_attn_wgmma_supported), and when `ops`
sets the flag from torch's fp32 matmul precision.  tests/test_gpu_f32_split.py runs the kernels."""
import ctypes

import pytest
import torch

import __graft_entry__ as ge
from vision_longformer_b200 import _lib, ops

SPLIT = 4


def _params(D=32, dtype=_lib.VIL_F32, flags=SPLIT, ptr=1 << 20, **kw):
    """ViL-Small stage 1 (56 x 56 tokens, w = 7, one global token) in the q / kv Linear-output layouts of fp32 rows"""
    p = _lib.VilAttnParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilAttnParams)
    p.dtype, p.impl, p.flags = dtype, _lib.VIL_IMPL_AUTO, flags
    p.B, p.H, p.D, p.nx, p.ny, p.w, p.nglo, p.exact, p.mode = 2, 3, D, 56, 56, 7, 1, 0, 0
    p.scale = D ** -0.5
    C = 3 * D
    for name, st in (("q", C), ("k", 2 * C), ("v", 2 * C)):
        t = getattr(p, name)
        t.ptr, t.sb, t.sh, t.st = ptr, 3137 * st, D, st
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.fixture(scope="module")
def lib():
    ge.build()
    return _lib.load()


def test_flag_is_a_new_bit_of_an_unchanged_abi(lib):
    """the flag adds a bit to `flags` and nothing to VilAttnParams: the version stays 3, and any other unknown bit is
    still refused"""
    assert lib.vil_attn_abi_version() == 3 == _lib.ABI_VERSION
    assert _lib.VIL_FLAG_F32_SPLIT == SPLIT
    assert SPLIT & (_lib.VIL_FLAG_F32_OUT | _lib.VIL_FLAG_UNFUSED) == 0
    assert lib.vil_attn_wgmma_supported(ctypes.byref(_params(flags=SPLIT | 8))) == _lib.VIL_E_BADARG
    assert "unknown bits" in _lib.last_error()


def test_split_coverage_is_the_same_with_dropout(lib):
    for D in (16, 32, 64, 128):
        assert lib.vil_attn_wgmma_supported(ctypes.byref(_params(D=D, dropout_p=0.3))) == \
            lib.vil_attn_wgmma_supported(ctypes.byref(_params(D=D)))


@pytest.mark.parametrize("dtype", [_lib.VIL_BF16, _lib.VIL_F16])
def test_flag_is_rejected_with_bf16_and_fp16(lib, dtype):
    p = _params(dtype=dtype)
    assert lib.vil_attn_wgmma_supported(ctypes.byref(p)) == _lib.VIL_E_BADARG
    assert "VIL_FLAG_F32_SPLIT" in _lib.last_error()
    assert lib.vil_attn_workspace_bytes(ctypes.byref(p), 1) == _lib.VIL_E_BADARG
    assert lib.vil_attn_fwd_sm100(ctypes.byref(p), None) == _lib.VIL_E_BADARG
    assert lib.vil_attn_bwd_sm100(ctypes.byref(p), None) == _lib.VIL_E_BADARG


def test_split_kernels_cover_vil_small(lib):
    ok = lambda **kw: lib.vil_attn_wgmma_supported(ctypes.byref(_params(**kw)))
    for D in (16, 24, 32, 48, 64):                      # ViL's head dims are 32, 48 and 64
        assert ok(D=D) == 1, D
        assert ok(D=D, flags=0) == 0, D                 # without the flag fp32 stays on the SIMT family
    assert ok(D=32, w=12, exact=1) == 1 and ok(D=64, mode=-1) == 1 and ok(D=32, exact=-1) == 1


def test_split_kernels_leave_the_rest_to_simt(lib):
    ok = lambda **kw: lib.vil_attn_wgmma_supported(ctypes.byref(_params(**kw)))
    assert ok(D=128) == 0 and ok(D=72) == 0             # the split kernels stop at the 64 head tile
    assert "head dim > 64" in _reason(lib, D=128)
    assert ok(D=36) == 0                                # D % 8 != 0
    assert ok(D=32, ptr=(1 << 20) + 8) == 0             # fp32 rows 8 bytes off a 16-byte boundary
    q = _params(D=32)
    q.q.st = 3 * 32 + 2                                 # a row stride of 392 bytes
    assert lib.vil_attn_wgmma_supported(ctypes.byref(q)) == 0
    # the same offsets in bf16 elements keep bf16 rows aligned: the check counts fp32 bytes
    assert lib.vil_attn_wgmma_supported(ctypes.byref(_params(D=32, dtype=_lib.VIL_BF16, flags=0, ptr=(1 << 20) + 16))) == 1


def _reason(lib, **kw):
    """the message of a forward forced onto the wgmma family (it fails before any launch)"""
    p = _params(impl=_lib.VIL_IMPL_WGMMA, **kw)
    for name in ("o", "qg", "kg", "vg", "og"):
        setattr(p, name, getattr(p, "k"))
    p.lse = p.lse_g = 1 << 20
    assert lib.vil_attn_fwd_sm100(ctypes.byref(p), None) == _lib.VIL_E_UNSUPPORTED
    return _lib.last_error()


# shared memory of the split kernels (vil_wgmma.cuh: FwdSmem / DqSmem / DkvSmem with T = float): a (64 x HD) fp32 tile
# is 64 HD 4 bytes, and the ring holds 3 stages at HD <= 32 and 2 at HD 64
CAP = 227 * 1024
KEYCOLS, QUERYCOLS, VISITS, DSTILE = 64 * 12, 64 * 17, 9 * 24, 64 * 72 * 4


def _stages(HD):
    return 3 if HD <= 32 else 2


def _fits(HD, w, drop=False):
    tabn = (4 * w - 1) ** 2
    al = lambda n: (n + 15) & ~15
    tile, S = 64 * HD * 4, _stages(HD)
    fwd = al((1 + 2 * S) * tile + S * KEYCOLS + VISITS + 4 * tabn)
    dq = al((2 + 2 * S) * tile + S * KEYCOLS + VISITS + 4 * tabn) + DSTILE
    dkv = al((2 + 2 * S) * tile + S * (QUERYCOLS + (256 if drop else 0)) + VISITS + 256 + 4 * tabn)
    return max(fwd, dq, dkv) <= CAP


def _w_limit(HD):
    return max(w for w in range(1, 49) if _fits(HD, w) and _fits(HD, w, True))


def test_bias_table_limit_of_the_split_kernels(lib):
    """computed from the shared memory of the three kernels: pass 1 with its dS tile is the limit at HD 64 (w = 42);
    the 16 and 32 tiles fit every window up to 48"""
    assert (_w_limit(16), _w_limit(32), _w_limit(64)) == (48, 48, 42)
    ok = lambda D, w, tab=256: lib.vil_attn_wgmma_supported(ctypes.byref(_params(D=D, w=w, bias_table=tab, g2l=tab, g2g=tab)))
    assert ok(64, 42) == 1 and ok(64, 43) == 0 and ok(48, 43) == 0 and ok(64, 48) == 0
    assert ok(32, 48) == 1 and ok(16, 48) == 1
    assert ok(64, 48, tab=None) == 1                    # without the table every window fits


# --------------------------------------------------------------------------- ops: the flag from torch's precision
@pytest.fixture
def precision():
    before = torch.backends.cuda.matmul.fp32_precision
    yield
    torch.backends.cuda.matmul.fp32_precision = before


@pytest.mark.parametrize("setting,split", [("high", True), ("medium", True), ("highest", False)])
def test_ops_sets_the_flag_from_the_matmul_precision(precision, setting, split):
    x = torch.zeros(2, 3)
    torch.set_float32_matmul_precision(setting)
    assert torch.backends.cuda.matmul.fp32_precision == ("tf32" if split else "ieee")
    for impl in ("auto", "wgmma"):
        assert ops._split_flag(x, impl) == (SPLIT if split else 0)
    assert ops._split_flag(x, "simt") == 0
    for dt in (torch.bfloat16, torch.float16):           # autocast has cast the activations before the flag is decided
        assert ops._split_flag(x.to(dt), "auto") == 0


def test_ops_default_precision_keeps_fp32_on_simt(precision):
    torch.backends.cuda.matmul.fp32_precision = "none"
    assert ops._split_flag(torch.zeros(1), "auto") == 0


def test_ops_reads_the_precision_after_the_apis_were_mixed(precision):
    x = torch.zeros(1)
    torch.set_float32_matmul_precision("high")
    torch.backends.cuda.matmul.allow_tf32 = False        # the legacy API after the new one
    with pytest.raises(RuntimeError):
        torch.get_float32_matmul_precision()
    assert ops._split_flag(x, "auto") == 0
    torch.backends.cuda.matmul.allow_tf32 = True
    assert torch.backends.cuda.matmul.fp32_precision == "tf32"
    assert ops._split_flag(x, "auto") == SPLIT
