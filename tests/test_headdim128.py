"""Head dims 64 < D <= 128 (D % 8 == 0) on the wgmma family: a 128-wide head tile in the forward and both backward passes,
and the global-token backward kernels at HD 128.

CPU tests: which calls the family takes (vil_attn_wgmma_supported), the bias-table limit of the 128 tile, the workspace.
GPU tests: parity with the fp64 oracle through the C ABI (contiguous and production layouts, every mask and mode), the
fp32-output parity build, dropout against the exact-mask restatement, repeatability, the table-fit fallback, and module-
level training (B200Long2DSCSelfAttention, DenseAttention(impl="vil"), a small MsViT).
"""
import ctypes
import math

import pytest
import torch

import __graft_entry__ as ge
from tests.test_gpu_dropout import VARIANTS as DROP_VARIANTS
from tests.test_gpu_dropout import kernel_run as drop_kernel_run
from tests.test_gpu_dropout import keep_tensors, reference_run
from tests.test_gpu_dropout import make_inputs as drop_inputs
from tests.test_gpu_parity import CASE_ID, DT_NAME, TOL, check_against, kernel_run, make_inputs, oracle_run
from tests.util import record, relerr
from vision_longformer_b200 import _lib, vil_attention_raw_backward, vil_attention_raw_forward

DEV = "cuda"
gpu = pytest.mark.gpu


# --------------------------------------------------------------------------- CPU: family selection
def _params(D=128, dtype=None, ptr=1 << 20, **kw):
    p = _lib.VilAttnParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilAttnParams)
    p.dtype = _lib.VIL_BF16 if dtype is None else dtype
    p.impl = _lib.VIL_IMPL_AUTO
    p.B, p.H, p.D, p.nx, p.ny, p.w, p.nglo, p.exact, p.mode = 2, 2, D, 56, 56, 7, 1, 0, 0
    p.scale = D ** -0.5
    C = 2 * D                                    # the q / kv Linear-output layouts: rows of whole heads
    for name in ("q", "k", "v"):
        t = getattr(p, name)
        t.ptr, t.sb, t.sh, t.st = ptr, 3137 * C, D, C
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _lib_built():
    ge.build()
    return _lib.load()


def test_wgmma_takes_head_dims_up_to_128():
    lib = _lib_built()
    ok = lambda **kw: lib.vil_attn_wgmma_supported(ctypes.byref(_params(**kw)))
    for D in (72, 80, 96, 112, 128):
        for dt in (_lib.VIL_BF16, _lib.VIL_F16):
            assert ok(D=D, dtype=dt) == 1, (D, dt)
    assert ok(D=128, dtype=_lib.VIL_F32) == 0           # fp32 stays on the SIMT family
    assert ok(D=100) == 0                               # D % 8 != 0
    assert ok(D=96, ptr=(1 << 20) + 2) == 0             # rows off 16 bytes
    assert ok(D=136) == _lib.VIL_E_UNSUPPORTED          # head dims above 128 are not supported at all
    assert "136" in _lib.last_error()


def test_bias_table_limit_of_the_128_tile():
    """pass 1 with the table and its dS tile fits beside the 2-stage 128 tiles up to w = 42; the 64 tiles fit every w"""
    lib = _lib_built()
    # the size checks never dereference the tables: any non-NULL address selects the call with the bias table
    ok = lambda tab=256, **kw: lib.vil_attn_wgmma_supported(ctypes.byref(_params(bias_table=tab, g2l=tab, g2g=tab, **kw)))
    assert ok(D=128, w=42) == 1
    assert ok(D=128, w=43) == 0 and ok(D=128, w=48) == 0
    assert ok(D=72, w=43) == 0                          # every 64 < D <= 128 runs the 128 tile
    assert ok(D=64, w=43) == 1 and ok(D=64, w=48) == 1
    assert ok(D=128, w=48, tab=None) == 1               # without the table every window fits


def test_workspace_does_not_depend_on_the_head_dim():
    lib = _lib_built()
    for tab in (None, 256):
        sizes = {D: lib.vil_attn_workspace_bytes(ctypes.byref(_params(D=D, bias_table=tab, g2l=tab, g2g=tab)), 1)
                 for D in (32, 64, 72, 128)}
        assert len(set(sizes.values())) == 1 and min(sizes.values()) > 0, sizes


# --------------------------------------------------------------------------- GPU: op parity vs the fp64 oracle
CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, rpe  -- all must be served by the wgmma family
    (1, 1, 128, 56, 56, 1, 7, 0, 0, False),    # ViL-like stage 1 grid
    (1, 2, 96, 28, 28, 1, 7, 0, 0, True),      # rpe (the bias-table variant of pass 1)
    (1, 1, 72, 19, 17, 2, 7, 0, 0, True),      # padding in both directions, 2 global tokens, D = 72 (zero-filled to 128)
    (1, 2, 128, 18, 15, 1, 6, 1, 0, True),     # exact window
    (1, 2, 128, 8, 5, 1, 4, -1, 0, False),     # cyclic chunks on a 2 x 2 chunk grid: chunks visited twice
    (1, 2, 72, 23, 33, 1, 7, 0, -1, True),     # own chunk only
    (1, 2, 128, 23, 33, 2, 7, 0, 3, False),    # random-shift mode 3
    (1, 2, 96, 22, 20, 1, 7, 0, 8, True),      # random-shift mode 8
    (1, 2, 128, 24, 24, 1, 12, 0, 0, True),    # w = 12: three pieces per chunk
    (1, 2, 96, 12, 12, 0, 6, 0, 0, True),      # no global tokens
    (1, 2, 128, 12, 12, 8, 6, 0, 0, True),     # g = 8
]


@gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_ID)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("layout", ["contig", "linear"])
def test_headdim128_matches_oracle(case, dtype, layout):
    B, H, D, nx, ny, g, w, exact, mode, rpe = case
    t = make_inputs(B, H, D, nx, ny, g, w, rpe, seed=304)
    scale = D ** -0.5
    ref = oracle_run(t, nx, ny, w, exact, mode, scale, dtype, key=("hd128",) + case)
    out, fam_f, fam_b = kernel_run(t, nx, ny, w, exact, mode, scale, dtype, "auto", layout=layout)
    assert (fam_f, fam_b) == ("wgmma", "wgmma")
    tf, tb = TOL[dtype]
    tbias = {torch.float16: 1e-2, torch.bfloat16: 5e-2}[dtype]
    check_against(out, ref, g, rpe, tf, tb, tbias, "headdim128_matches_oracle", case, DT_NAME[dtype] + "/" + layout)
    if layout == "linear":                      # every row of the strided outputs has been written
        for n in ("o", "dq", "dk", "dv"):
            assert torch.isfinite(out[n].float()).all(), n


@gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_headdim128_separate_global_weights(dtype):
    """kg / vg not k / v: the global query rows read their own key and value tensors (the global-token kernels at HD 128)"""
    case = (1, 2, 128, 15, 13, 2, 7, 0, 0, True, True, 0.0)
    B, H, D, nx, ny, g, w, exact, mode, rpe, sep, p = case
    t = drop_inputs(B, H, D, nx, ny, g, w, rpe, sep, seed=305)
    cfg = (nx, ny, w, exact, mode, D ** -0.5)
    keep, keep_g = keep_tensors(0, 0, p, B, H, nx, ny, w, g, mode)
    ref = reference_run(t, cfg, dtype, keep, keep_g)
    out, fam = drop_kernel_run(t, cfg, dtype, "wgmma", (p, 0, 0))
    assert fam == "wgmma"
    tf, tb = TOL[dtype]
    tbias = {torch.float16: 1e-2, torch.bfloat16: 5e-2}[dtype]
    errs = {n: relerr(out[n], ref[n]) for n in ("o", "og", "dq", "dk", "dv", "dqg", "dkg", "dvg", "dtable", "dg2l", "dg2g")}
    record("headdim128_separate_global_weights", DT_NAME[dtype], **errs)
    for n, e in errs.items():
        assert e < (tf if n in ("o", "og") else tbias if n in ("dtable", "dg2l", "dg2g") else tb), (n, errs)


@gpu
@pytest.mark.parametrize("case", [CASES[0], CASES[1], CASES[6]], ids=CASE_ID)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_headdim128_fp32_out_parity(case, dtype):
    """VIL_FLAG_F32_OUT at D = 128: 1e-3 (fp16) / 2e-3 (bf16) forward and backward, as at D <= 64"""
    B, H, D, nx, ny, g, w, exact, mode, rpe = case
    t = make_inputs(B, H, D, nx, ny, g, w, rpe, seed=306)
    scale = D ** -0.5
    ref = oracle_run(t, nx, ny, w, exact, mode, scale, dtype, key=("hd128_f32out",) + case)
    out, fam_f, fam_b = kernel_run(t, nx, ny, w, exact, mode, scale, dtype, "auto", f32out=True)
    assert (fam_f, fam_b) == ("wgmma", "wgmma")
    bar = 1e-3 if dtype == torch.float16 else 2e-3
    check_against(out, ref, g, rpe, bar, bar, 2e-2, "headdim128_fp32_out_parity", case, DT_NAME[dtype] + "/fp32out")


# --------------------------------------------------------------------------- GPU: dropout and repeatability
DROP_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, rpe, separate global weights, p
    (1, 2, 128, 14, 14, 1, 7, 0, 0, True, False, 0.1),
    (1, 2, 128, 8, 5, 1, 4, -1, 0, False, True, 0.1),     # 2 x 2 chunk grid: two offsets reach the same chunk
    (1, 2, 96, 15, 13, 2, 7, 1, 0, True, False, 0.1),     # exact window, padding
]
DROP_ID = lambda c: "B%d_H%d_D%d_%dx%d_g%d_w%d_e%d_m%d_%s_%s_p%g" % (c[:9] + ("rpe" if c[9] else "nob", "sep" if c[10] else "shared", c[11]))
SEED, OFFSET = 0x5eed0000d128, 99


@gpu
@pytest.mark.parametrize("case", DROP_CASES, ids=DROP_ID)
@pytest.mark.parametrize("variant", ["wgmma_bf16", "wgmma_bf16_f32out", "wgmma_fp16_f32out"])
def test_headdim128_dropout_matches_the_exact_mask(case, variant):
    B, H, D, nx, ny, g, w, exact, mode, rpe, sep, p = case
    impl, dtype, f32out, tf, tb, tbias = DROP_VARIANTS[variant]
    t = drop_inputs(B, H, D, nx, ny, g, w, rpe, sep)
    cfg = (nx, ny, w, exact, mode, D ** -0.5)
    keep, keep_g = keep_tensors(SEED, OFFSET, p, B, H, nx, ny, w, g, mode)
    ref = reference_run(t, cfg, dtype, keep, keep_g)
    out, fam = drop_kernel_run(t, cfg, dtype, impl, (p, SEED, OFFSET), f32out)
    assert fam == "wgmma"
    names = ["o", "dq", "dk", "dv"] + (["og", "dqg"] + (["dkg", "dvg"] if sep else []) if g else []) + \
        (["dtable"] + (["dg2l", "dg2g"] if g else []) if rpe else [])
    errs = {n: relerr(out[n], ref[n]) for n in names}
    record("headdim128_dropout", DROP_ID(case) + "/" + variant, **errs)
    for n, e in errs.items():
        assert e < (tf if n in ("o", "og") else tbias if n in ("dtable", "dg2l", "dg2g") else tb), (n, errs)


@gpu
def test_headdim128_p0_is_the_path_without_dropout():
    B, H, D, nx, ny, g, w, exact, mode, rpe, sep, _ = DROP_CASES[0]
    t = drop_inputs(B, H, D, nx, ny, g, w, rpe, sep)
    a, fam = drop_kernel_run(t, (nx, ny, w, exact, mode, D ** -0.5), torch.bfloat16, "auto", (0.0, SEED, OFFSET))
    b, fam_f, fam_b = kernel_run(t, nx, ny, w, exact, mode, D ** -0.5, torch.bfloat16, "auto")
    assert fam == fam_f == fam_b == "wgmma"
    for n in ("o", "og", "dq", "dk", "dv", "dqg", "dtable", "dg2l", "dg2g"):
        assert torch.equal(a[n], b[n]), n


@gpu
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_headdim128_backward_repeats_bitwise(p):
    case = (2, 2, 128, 15, 13, 3, 7, 0, 0, True, True)
    B, H, D, nx, ny, g, w, exact, mode, rpe, sep = case
    t = drop_inputs(B, H, D, nx, ny, g, w, rpe, sep, seed=310)
    cfg = (nx, ny, w, exact, mode, D ** -0.5)
    a, fa = drop_kernel_run(t, cfg, torch.bfloat16, "auto", (p, SEED, OFFSET))
    b, fb = drop_kernel_run(t, cfg, torch.bfloat16, "auto", (p, SEED, OFFSET))
    assert fa == fb == "wgmma" and a["dtable"] is not None
    for n in a:
        if a[n] is not None:
            assert torch.equal(a[n], b[n]), n


@gpu
def test_table_that_does_not_fit_beside_the_128_tile_falls_back_to_simt():
    """rpe at w = 43: the table fits beside the 64 tiles but not beside pass 1's 128 tiles and its dS tile.  The forward
    runs on SIMT; the SIMT backward stops at D = 64 and says which family trains this head dim.  No launch fails."""
    B, H, D, nx, ny, g, w = 1, 1, 128, 43, 43, 1, 43
    t = make_inputs(B, H, D, nx, ny, g, w, True, seed=307)
    cuda = lambda x: x.to(DEV, torch.bfloat16).contiguous()
    f32 = lambda x: x.to(DEV, torch.float32).contiguous()
    q, k, v, qg, go, gog = cuda(t["q"]), cuda(t["k"]), cuda(t["v"]), cuda(t["qg"]), cuda(t["go"]), cuda(t["gog"])
    table, g2l, g2g = f32(t["table"]), f32(t["g2l"]), f32(t["g2g"])
    o, og = torch.empty_like(q), torch.empty_like(qg)
    kw = dict(nx=nx, ny=ny, w=w, exact=0, mode=0, scale=D ** -0.5)
    lse, lse_g = vil_attention_raw_forward(q, k, v, qg, k, v, table, g2l, g2g, o, og, **kw)
    torch.cuda.synchronize()
    assert _lib.last_impl() == "simt"
    assert torch.isfinite(o.float()).all()
    dq, dk, dv, dqg = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v), torch.empty_like(qg)
    z = torch.zeros_like
    with pytest.raises(NotImplementedError, match="64 < D <= 128 is trained by the wgmma family"):
        vil_attention_raw_backward(q, k, v, qg, k, v, table, g2l, g2g, o, og, lse, lse_g, go, gog, dq, dk, dv, dqg, dk, dv,
                                   z(table), z(g2l), z(g2g), **kw)
    torch.cuda.synchronize()


# --------------------------------------------------------------------------- GPU: modules
@gpu
def test_module_at_head_dim_128_matches_the_reference():
    from oracle.vil_oracle import OracleLong2DSCSelfAttention
    from vision_longformer_b200 import B200Long2DSCSelfAttention
    torch.manual_seed(12)
    kw = dict(dim=256, num_heads=2, rpe=True)
    nx = ny = 28
    ref = OracleLong2DSCSelfAttention(**kw).double().eval()
    for n, p_ in ref.named_parameters():                    # biases large enough to matter
        if "relative_position" in n:
            torch.nn.init.normal_(p_, std=0.3)
    x = torch.randn(2, 1 + nx * ny, 256, dtype=torch.float64, requires_grad=True)
    gy = torch.randn(2, 1 + nx * ny, 256, dtype=torch.float64)
    y_ref = ref(x, nx, ny)
    (y_ref * gy).sum().backward()
    mod = B200Long2DSCSelfAttention(**kw).to(DEV).eval()
    mod.load_state_dict({k_: v_.float() for k_, v_ in ref.state_dict().items()})
    xg = x.detach().float().to(DEV).requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = mod(xg, nx, ny)
    assert _lib.last_impl() == "wgmma"
    (y.float() * gy.float().to(DEV)).sum().backward()
    torch.cuda.synchronize()
    assert _lib.last_impl() == "wgmma"
    e_y, e_dx = relerr(y, y_ref), relerr(xg.grad, x.grad)
    record("headdim128_module", "dim256_h2_rpe_28x28", y=e_y, dx=e_dx)
    assert e_y < 3e-2 and e_dx < 6e-2, (e_y, e_dx)


@gpu
@pytest.mark.parametrize("w", [7, 14])
@pytest.mark.parametrize("rpe", [True, False], ids=["rpe", "nob"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_dense_attention_vil_at_head_dim_128(w, rpe, dtype):
    from vision_longformer_b200.msvit import DenseAttention
    dim, H, g = 256, 2, 1
    torch.manual_seed(13)
    ref = DenseAttention(dim, num_heads=H, qkv_bias=True, rpe=rpe, wx=w, wy=w, nglo=g, impl="sdpa").to(DEV)
    if rpe:
        for p_ in (ref.local_relative_position_bias_table, ref.g2l_relative_position_bias, ref.g2g_relative_position_bias):
            torch.nn.init.normal_(p_, std=0.3)
    mod = DenseAttention(dim, num_heads=H, qkv_bias=True, rpe=rpe, wx=w, wy=w, nglo=g, impl="vil").to(DEV)
    mod.load_state_dict(ref.state_dict())
    mod = mod.to(dtype)
    x = torch.randn(3, g + w * w, dim, device=DEV)
    gy = torch.randn_like(x)
    xr = x.clone().requires_grad_(True)
    yr = ref(xr)
    (yr * gy).sum().backward()
    xm = x.to(dtype).requires_grad_(True)
    ym = mod(xm)
    assert _lib.last_impl() == "wgmma"
    (ym * gy.to(dtype)).sum().backward()
    torch.cuda.synchronize()
    assert _lib.last_impl() == "wgmma"
    errs = dict(y=relerr(ym, yr), dx=relerr(xm.grad, xr.grad), dqkv_w=relerr(mod.qkv.weight.grad, ref.qkv.weight.grad))
    if rpe:
        errs["dtable"] = relerr(mod.local_relative_position_bias_table.grad, ref.local_relative_position_bias_table.grad)
    record("headdim128_dense_attention", "w%d_%s/%s" % (w, "rpe" if rpe else "nob", DT_NAME[dtype]), **errs)
    tol = 3e-2 if dtype == torch.bfloat16 else 6e-3
    assert errs["y"] < tol and errs["dx"] < 2 * tol and errs["dqkv_w"] < 2 * tol, errs
    if rpe:
        assert errs["dtable"] < 0.1, errs


@gpu
def test_msvit_with_head_dim_128_trains():
    from vision_longformer_b200 import B200Long2DSCSelfAttention, build_vil
    from vision_longformer_b200.msvit import DenseAttention
    torch.manual_seed(14)
    arch = "l1,h1,d128,n1,s1,g1,p4,f7_l2,h2,d256,n1,s1,g1,p2,f7_l3,h2,d256,n1,s0,g1,p2,f7"
    net = build_vil(arch, img_size=112, num_classes=10, dense_impl="vil").to(DEV).train()
    fams = []
    hooks = [m.register_forward_hook(lambda *_: fams.append(_lib.last_impl())) for m in net.modules()
             if isinstance(m, (B200Long2DSCSelfAttention, DenseAttention))]
    opt = torch.optim.AdamW(net.parameters(), lr=1e-3)
    x = torch.randn(4, 3, 112, 112, device=DEV)
    lab = torch.randint(0, 10, (4,), device=DEV)
    losses = []
    for _ in range(3):
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(net(x).float(), lab)
        loss.backward()
        assert _lib.last_impl() == "wgmma"
        for n, p_ in net.named_parameters():
            assert p_.grad is not None and torch.isfinite(p_.grad).all(), n
        opt.step()
        losses.append(loss.item())
    for h in hooks:
        h.remove()
    assert len(fams) == 3 * 3 and set(fams) == {"wgmma"}, fams
    assert all(math.isfinite(v) for v in losses), losses
