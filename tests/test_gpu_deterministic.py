"""The attention backward is deterministic: identical inputs give bitwise-identical outputs, including the three
relative-position-bias gradients (d_bias_table, d_g2l, d_g2g).

Those three are summed in a fixed order: backward pass 1 adds each chunk piece's dS to per-CTA table partials, the
global-token kernels write per-image partials, and one reduce kernel sums them into the caller's tensors.

CPU tests: the workspace layout (the table partials do not grow with the batch; without the table the size is unchanged).
GPU tests: two backward calls agree bit for bit over both kernel families, every mask, mode, window and dropout setting;
the bias gradients match the fp64 reference; the table adds one launch; module forward / backward and AdamW steps repeat
bit for bit under torch.use_deterministic_algorithms(True).
"""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

from tests.test_gpu_dropout import kernel_run, keep_tensors, make_inputs, reference_run
from tests.util import record, relerr
from vision_longformer_b200 import _lib

DEV = "cuda"
gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# --------------------------------------------------------------------------- CPU: workspace layout
def _params(**kw):
    p = _lib.VilAttnParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilAttnParams)
    p.dtype, p.impl = _lib.VIL_BF16, _lib.VIL_IMPL_AUTO
    p.B, p.H, p.D, p.nx, p.ny, p.w, p.nglo, p.exact, p.mode = 256, 3, 32, 56, 56, 7, 1, 0, 0
    p.scale = 32 ** -0.5
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _ws(**kw):
    import __graft_entry__ as ge
    ge.build()
    return _lib.load().vil_attn_workspace_bytes(ctypes.byref(_params(**kw)), 1)


align64 = lambda n: (n + 63) // 64 * 64


def test_table_partials_do_not_grow_with_the_batch():
    # the size query never dereferences the table: any non-NULL address selects the layout with the bias table
    a, b = _ws(B=1024, nglo=0, bias_table=256), _ws(B=2048, nglo=0, bias_table=256)
    assert b - a == 4 * (align64(2048 * 3 * 56 * 56) - align64(1024 * 3 * 56 * 56))
    assert a > _ws(B=1024, nglo=0)                 # the table partials are there


@pytest.mark.parametrize("B,H,nx,ny,g", [(256, 3, 56, 56, 1), (7, 2, 15, 13, 3), (1, 6, 28, 28, 0)])
def test_workspace_without_the_table_is_unchanged(B, H, nx, ny, g):
    assert _ws(B=B, H=H, nx=nx, ny=ny, nglo=g) == 256 + 4 * (align64(B * H * nx * ny) + align64(B * H * g))


# --------------------------------------------------------------------------- GPU: repeatability and parity
CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, separate global weights, p      (all with the bias table)
    (2, 2, 32, 15, 13, 1, 7, 0, 0, False, 0.0),     # padding in both directions
    (2, 2, 32, 15, 13, 3, 7, 1, 0, True, 0.1),      # exact window, 3 global tokens, separate kg / vg, dropout
    (2, 2, 32, 10, 9, 1, 4, -1, 0, False, 0.0),     # cyclic chunks with padding, w = 4
    (1, 2, 32, 8, 5, 1, 4, -1, 0, True, 0.1),       # 2 x 2 chunk grid: one chunk reached through two offsets
    (2, 2, 64, 26, 25, 1, 12, 0, 3, True, 0.0),     # w = 12: three pieces per chunk, random-shift mode 3
    (2, 2, 32, 26, 37, 0, 12, 0, -1, False, 0.1),   # own chunk only, no global tokens
    (2, 3, 16, 21, 22, 3, 7, 0, 0, False, 0.0),     # D = 16
]
CASE_ID = lambda c: "B%d_H%d_D%d_%dx%d_g%d_w%d_e%d_m%d_%s_p%g" % (c[:9] + ("sep" if c[9] else "shared", c[10]))
VARIANTS = {"wgmma_bf16": ("wgmma", torch.bfloat16), "wgmma_fp16": ("wgmma", torch.float16), "simt_fp32": ("simt", torch.float32)}
TBIAS = {torch.float32: 1e-4, torch.float16: 1e-2, torch.bfloat16: 5e-2}   # test_gpu_parity's bars for the bias gradients
SEED, OFFSET = 0x5eed0000beef, 77


def _run(case, impl, dtype, seed=310):
    B, H, D, nx, ny, g, w, exact, mode, sep, p = case
    t = make_inputs(B, H, D, nx, ny, g, w, True, sep, seed=seed)
    cfg = (nx, ny, w, exact, mode, D ** -0.5)
    out, fam = kernel_run(t, cfg, dtype, impl, (p, SEED, OFFSET))
    assert fam == impl
    return t, cfg, out


def _assert_bitwise(a, b):
    for n in a:
        if a[n] is not None:
            assert torch.equal(a[n], b[n]), n


@gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_ID)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_backward_repeats_bitwise(case, variant):
    impl, dtype = VARIANTS[variant]
    _, _, a = _run(case, impl, dtype)
    _, _, b = _run(case, impl, dtype)
    assert a["dtable"] is not None and (case[5] == 0 or a["dg2l"] is not None)
    _assert_bitwise(a, b)


@gpu
def test_backward_repeats_bitwise_at_vil_small_stage1():
    """many CTAs and images per table entry: the shape at which the old atomics differed run to run"""
    case = (8, 3, 32, 56, 56, 1, 7, 0, 0, False, 0.0)
    _, _, a = _run(case, "wgmma", torch.bfloat16, seed=311)
    _, _, b = _run(case, "wgmma", torch.bfloat16, seed=311)
    _assert_bitwise(a, b)


@gpu
@pytest.mark.parametrize("case", [CASES[0], CASES[1], CASES[3], CASES[4], CASES[6]], ids=CASE_ID)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_bias_gradients_match_reference(case, variant):
    impl, dtype = VARIANTS[variant]
    B, H, D, nx, ny, g, w, exact, mode, sep, p = case
    t, cfg, out = _run(case, impl, dtype)
    keep, keep_g = keep_tensors(SEED, OFFSET, p, B, H, nx, ny, w, g, mode)
    ref = reference_run(t, cfg, dtype, keep, keep_g)
    names = ["dtable"] + (["dg2l", "dg2g"] if g else [])
    errs = {n: relerr(out[n], ref[n]) for n in names}
    record("deterministic_bias_gradients", CASE_ID(case) + "/" + variant, **errs)
    for n, e in errs.items():
        assert e < TBIAS[dtype], (n, errs)


@gpu
def test_the_table_adds_one_launch():
    from tests import test_gpu_parity as tp
    counts = {}
    for rpe in (False, True):
        t = tp.make_inputs(2, 3, 32, 14, 14, 1, 7, rpe)
        before = _lib.launch_count()
        tp.kernel_run(t, 14, 14, 7, 0, 0, 32 ** -0.5, torch.bfloat16, "auto")
        counts[rpe] = _lib.launch_count() - before
    assert counts == {False: 7, True: 8}, counts


# --------------------------------------------------------------------------- GPU: modules under deterministic mode
_MODULE_SCRIPT = r"""
import random
import torch
torch.use_deterministic_algorithms(True)
from vision_longformer_b200 import B200Long2DSCSelfAttention, build_vil
from vision_longformer_b200.msvit import DenseAttention

def module_run(make, shape, call):
    torch.manual_seed(0)
    random.seed(0)
    mod = make().cuda().train()
    x = torch.randn(*shape, device="cuda", requires_grad=True)
    gy = torch.randn(*shape, device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = call(mod, x)
    (y.float() * gy).sum().backward()
    return [y.detach(), x.grad] + [p.grad for p in mod.parameters()]

cases = {
    "B200Long2DSCSelfAttention": (lambda: B200Long2DSCSelfAttention(96, num_heads=3, qkv_bias=True, w=7, nglo=1, sharew=True,
                                                                    rpe=True, mode=1), (2, 1 + 28 * 28, 96),
                                  lambda m, x: m(x, 28, 28)),
    "DenseAttention": (lambda: DenseAttention(64, num_heads=2, qkv_bias=True, rpe=True, wx=7, wy=7, nglo=1, impl="vil"),
                       (2, 1 + 49, 64), lambda m, x: m(x)),
}
for name, (make, shape, call) in cases.items():
    a, b = module_run(make, shape, call), module_run(make, shape, call)
    assert len(a) > 3 and all(u is not None and torch.equal(u, v) for u, v in zip(a, b)), name

ARCH = "l1,h1,d32,n1,s1,g1,p4,f7,a0_l2,h2,d64,n1,s1,g1,p2,f7,a0_l3,h2,d64,n1,s0,g1,p2,f7,a0_l4,h2,d64,n1,s0,g0,p2,f7,a0"

def train_run():
    torch.manual_seed(1)
    random.seed(1)
    net = build_vil(ARCH, num_classes=10, dense_impl="vil").cuda().train()
    opt = torch.optim.AdamW(net.parameters(), lr=1e-3)
    x = torch.randn(2, 3, 224, 224, device="cuda")
    lab = torch.randint(0, 10, (2,), device="cuda")
    for _ in range(2):
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(net(x).float(), lab)
        loss.backward()
        opt.step()
    return [p.detach().clone() for p in net.parameters()]

a, b = train_run(), train_run()
assert all(torch.equal(u, v) for u, v in zip(a, b))
print("DETERMINISTIC OK")
"""


@gpu
def test_modules_and_training_repeat_under_deterministic_algorithms():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", PYTHONPATH=ROOT)
    res = subprocess.run([sys.executable, "-c", _MODULE_SCRIPT], cwd=ROOT, env=env, capture_output=True, text=True,
                         timeout=900)
    assert res.returncode == 0 and "DETERMINISTIC OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]
