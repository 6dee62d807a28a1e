"""fp32 attention on the wgmma tensor cores as split bf16 products (VIL_FLAG_F32_SPLIT) against the fp64 oracles.

Each fp32 operand x is hi = bf16(x) plus lo = bf16(x - hi), and each product A B is A_hi B_hi + A_hi B_lo + A_lo B_hi:
every term keeps about 16 significant bits where the SIMT family keeps 24.  The measurements are those of
test_gpu_attention_rows (rows, chunks, lse), test_gpu_bias_entries (the bias gradients entry by entry) and
test_gpu_dropout (the exact mask), run on the split kernels under the variant name "wgmma_f32split"; then repeatability,
the image slices of pass 1, the routing of fp32 calls by torch's matmul precision, and the module against its fp64
oracle.

The bars were measured on an H100 SXM (700 W power limit): each is about 3x the worst value seen over this file
(DESIGN.md section 4).
"""
import pytest
import torch

from oracle.vil_oracle import OracleLong2DSCSelfAttention
from tests import test_gpu_attention_rows as tar
from tests import test_gpu_bias_entries as tbe
from tests import test_gpu_dropout as tdrop
from tests import test_gpu_parity as tpar
from tests.test_gpu_batch_slices import nslice_of_the_library
from tests.util import record, relerr
from vision_longformer_b200 import B200Long2DSCSelfAttention, _lib

gpu = pytest.mark.gpu
F32 = torch.float32
V = "wgmma_f32split"
DEV = "cuda"

# Worst values measured with randn inputs, dropout included (rows forward / backward, chunks forward / backward):
# 2.2e-5 / 6.0e-5, 1.1e-5 / 2.0e-5; lse 8.0e-6; bias gradients (whole tensor) 7.6e-6.
BARS = dict(row=(7e-5, 1e-4), chunk=(3.5e-5, 6e-5), lse=2.5e-5)
BIAS_BAR = 2.5e-5
# one dS enters a bias entry with eps_o ||dO|| ||o||: delta from the stored fp32 o, and the split P operand (2^-16);
# worst err / T_e measured over the file 2.5e-6
EPS_O = 2.0 ** -24 + 2.0 ** -16
KAPPA = 7.5e-6
# the floors of a saturated softmax scale with the error of the products: 2^-17 per split term against fp32's 2^-24
FLOOR_SCALE = 2.0 ** 7
# A score s carries an absolute error of about 2^-16 |s| (the lo x lo term the split leaves out, against fp32's 2^-24 |s|),
# and P = exp(s - lse) that error relative.  Where scores exceed 16 (the peaked cases reach 500), SCORE_ROUNDINGS of it
# are allowed on top of the bars, as test_gpu_attention_rows allows 16 fp32 roundings; nothing for ordinary scores.
SCORE_ROUNDINGS = 8.0
# the module under "high", TF32 Linears included: worst 3.5e-3 (the g2l gradient), 4.8e-4 for dx
MODULE_BAR = 1e-2


def run_split(t, cfg, variant=V, drop=(0.0, 0, 0), layout="contig"):
    nx, ny, w, exact, mode, scale = cfg
    out, fam_f, fam_b = tpar.kernel_run(t, nx, ny, w, exact, mode, scale, F32, "wgmma", layout=layout,
                                        flags=_lib.VIL_FLAG_F32_SPLIT, drop=drop)
    assert (fam_f, fam_b) == ("wgmma", "wgmma"), (fam_f, fam_b)
    assert _lib.last_kernel() == "wgmma_f32split_bwd"
    return out


def _check_split(check):
    def run(test, tag, out, ref, case, variant, **kw):
        top = float(ref["lse"].abs().max()) if ref.get("lse") is not None else 0.0
        big = SCORE_ROUNDINGS * 2.0 ** -16 * top if top > 16 else 0.0
        tar.BARS[V] = dict(row=tuple(x + big for x in BARS["row"]), chunk=tuple(x + big for x in BARS["chunk"]),
                           lse=BARS["lse"] + big)
        return check(test, tag, out, ref, case, variant, **kw)
    return run


@pytest.fixture(autouse=True)
def split_variant(monkeypatch):
    """the helpers of the row and bias-entry files, taught the split variant for the duration of one test"""
    monkeypatch.setitem(tar.VARIANTS, V, ("wgmma", F32, False, "contig"))
    monkeypatch.setitem(tar.BARS, V, BARS)
    monkeypatch.setattr(tar, "check", _check_split(tar.check))
    monkeypatch.setitem(tar.BIAS_BARS, V, BIAS_BAR)
    monkeypatch.setitem(tbe.VARIANTS, V, ("wgmma", F32, False, "contig"))
    monkeypatch.setitem(tbe.EPS_O, V, EPS_O)
    monkeypatch.setitem(tbe.KAPPA, V, KAPPA)
    floors = tar.peak_floors
    monkeypatch.setattr(tar, "peak_floors", lambda *a: {k: x * FLOOR_SCALE for k, x in floors(*a).items()})


def cases_upto_64(cases):
    """the split kernels' head tiles stop at 64; the 56 x 56 oracle is left to the bf16 variants, as in the row file"""
    return [c for c in cases if c[2] <= 64 and c[3] * c[4] <= 2000]


ids = lambda cases: [tar.CASE_ID(c) for c in cases]

# --------------------------------------------------------------------------- rows and chunks
ROW_CASES = cases_upto_64(tar.GEOMETRY_CASES)
GLOBAL_CASES = cases_upto_64(tar.MANY_GLOBAL_CASES)
MASKED_CASES = cases_upto_64(tar.MASKED_CASES)


@gpu
@pytest.mark.parametrize("case", ROW_CASES, ids=ids(ROW_CASES))
def test_rows_random_inputs(case):
    t = tar.make_inputs(case, seed=310)
    cfg = tar.cfg_of(case)
    ref = tar.oracle(t, cfg, F32, ("geo",) + case)
    tar.check("f32split_rows_random_inputs", "randn", run_split(t, cfg), ref, case, V)


@gpu
@pytest.mark.parametrize("case", GLOBAL_CASES, ids=ids(GLOBAL_CASES))
def test_rows_more_than_64_global_tokens(case):
    t = tar.make_inputs(case, seed=340, sep=case[10])
    cfg = tar.cfg_of(case)
    ref = tar.oracle(t, cfg, F32, ("glob",) + case)
    tar.check("f32split_rows_more_than_64_global_tokens", "randn", run_split(t, cfg), ref, case, V)


@gpu
@pytest.mark.parametrize("case", MASKED_CASES, ids=ids(MASKED_CASES))
def test_rows_masked_leading_pieces(case):
    t = tar.make_inputs(case, seed=330)
    cfg = tar.cfg_of(case)
    ref = tar.oracle(t, cfg, F32, ("masked",) + case)
    tar.check("f32split_rows_masked_leading_pieces", "randn", run_split(t, cfg), ref, case, V)


# o against the hot key's v row once every other probability is below e^-100: the split v carries 2^-17 of each element
HOT_O_BAR = 2.0 ** -15


def check_peaked(test, case, t, tag, L, hot=None):
    """test_gpu_attention_rows.check_peaked with the split's bars for o and lse against the hot key (L >= 100)"""
    cfg = tar.cfg_of(case)
    ref = tar.oracle(t, cfg, F32, (test, tag) + case)
    out = run_split(t, cfg)
    tar.check(test, tag, out, ref, case, V, floors=tar.peak_floors(t, cfg, V, case[5]), bias=False)
    if hot is not None and L >= 100:
        sh, logp = tar.realized_gap(ref["lse"], t, case, F32, hot)
        assert float(logp.min()) > -1e-9, float(logp.min())
        val, idx = tar.worst(tar.row_errors(out["o"], t["v"].to(F32).double()[:, :, hot]))
        lerr = float((out["lse"].double().cpu() - sh).abs().max())
        record(test, tar.CASE_ID(case) + "/" + tag + "/" + V, o_vs_hot_v=val, lse_vs_hot_score=lerr)
        assert val < HOT_O_BAR, (val, tar.where_local(idx, case[3], case[4], case[6]))
        assert lerr < BARS["lse"] + SCORE_ROUNDINGS * 2.0 ** -16 * float(sh.abs().max()), lerr


def _peak_params():
    return [pytest.param(*p.values[:3], id=p.id.rsplit("-", 1)[0]) for p in tar._peak_params() if p.values[3] == "simt_fp32"]


@gpu
@pytest.mark.parametrize("case,target,L", _peak_params())
def test_rows_peaked_through_q_and_k(case, target, L):
    tag = "%s_L%d" % ("_".join(str(x) for x in target), L)
    t, hot = tar.peak_through_qk(tar.make_inputs(case, seed=320), case, F32, L, target)
    check_peaked("f32split_rows_peaked_through_q_and_k", case, t, tag, L, hot)


@gpu
@pytest.mark.parametrize("L", tar.GAPS)
@pytest.mark.parametrize("what", tar.TABLE_PEAKS, ids=lambda x: "_".join(str(y) for y in x))
def test_rows_peaked_through_the_bias(what, L):
    t = tar.peak_through_table(tar.make_inputs(tar.PK_TABLE, seed=321), tar.PK_TABLE, L, what)
    check_peaked("f32split_rows_peaked_through_the_bias", tar.PK_TABLE, t, "%s_L%d" % ("_".join(str(x) for x in what), L), L)


@gpu
@pytest.mark.parametrize("case", tar.MASKED_CASES[:2], ids=ids(tar.MASKED_CASES[:2]))
@pytest.mark.parametrize("L", [40, 100])
def test_rows_masked_leading_pieces_then_the_maximum_in_the_last_chunk(case, L):
    t, hot = tar.peak_through_qk(tar.make_inputs(case, seed=331), case, F32, L, ("off", 1, 1, "same"))
    check_peaked("f32split_rows_masked_leading_pieces_then_the_maximum_in_the_last_chunk", case, t, "off_1_1_L%d" % L, L, hot)


# --------------------------------------------------------------------------- dropout
DROP_CASES = [(1, 2, 32, 15, 13, 2, 7, 0, 0, True), (1, 2, 32, 14, 14, 65, 7, 0, 0, True, False),
              (1, 2, 64, 15, 13, 2, 7, 0, -1, False), (1, 2, 16, 10, 9, 2, 4, -1, 0, True)]


@gpu
@pytest.mark.parametrize("case", DROP_CASES, ids=ids(DROP_CASES))
def test_rows_dropout_with_the_exact_mask(case):
    t = tar.make_inputs(case, seed=311)
    ref = tar.dropout_reference(t, case, F32)
    tar.check("f32split_rows_dropout", "p0.1", run_split(t, tar.cfg_of(case), drop=tar.DROP), ref, case, V)


@gpu
def test_dropout_p0_is_the_call_without_dropout():
    case = DROP_CASES[0]
    t = tar.make_inputs(case, seed=312)
    a = run_split(t, tar.cfg_of(case), drop=(0.0, tar.DROP[1], tar.DROP[2]))
    b = run_split(t, tar.cfg_of(case))
    for n, x in a.items():
        if x is not None:
            assert torch.equal(x, b[n]), n


# --------------------------------------------------------------------------- bias gradients entry by entry
BIAS_CASES = [c for c in tbe.RANDOM_CASES + tbe.MANY_GLOBAL_CASES if 8 < c[2] <= 64]


@gpu
@pytest.mark.parametrize("case", BIAS_CASES, ids=[tbe.CASE_ID(c) for c in BIAS_CASES])
def test_bias_entries_random_inputs(case):
    t = tar.make_inputs(tbe.full(case), seed=410, sep=tbe.full(case)[10])
    terms = tbe.terms_of(("rand",) + case, t, case, F32)
    tbe.hold_entries("f32split_bias_entries_random_inputs", "randn", run_split(t, tar.cfg_of(tbe.full(case))), terms, case, V)


BIAS_DROP_CASES = [c for c in tbe.DROP_CASES if c[2] <= 64][:4]


@gpu
@pytest.mark.parametrize("case", BIAS_DROP_CASES, ids=[tbe.CASE_ID(c) for c in BIAS_DROP_CASES])
def test_bias_entries_dropout(case):
    B, H, D, nx, ny, g, w, exact, mode, sep, p = case
    t = tar.make_inputs(tbe.full(case), seed=411, sep=sep)
    keep, keep_g = tdrop.keep_tensors(tbe.SEED, tbe.OFFSET, p, B, H, nx, ny, w, g, mode)
    terms = tbe.terms_of(("drop",) + case, t, case, F32, keep, keep_g)
    out = run_split(t, tar.cfg_of(tbe.full(case)), drop=(p, tbe.SEED, tbe.OFFSET))
    tbe.hold_entries("f32split_bias_entries_dropout", "p%g" % p, out, terms, case, V)


# --------------------------------------------------------------------------- repeatability and image slices
SLICE_CASE = (11, 64, 16, 8, 5, 1, 4, -1, 0, True)


@gpu
def test_repeatable_and_each_image_of_a_sliced_batch_is_a_one_image_call():
    """B = 11 images over fewer pass-1 slices: every image's outputs are bitwise those of a call with that image alone"""
    case = SLICE_CASE
    assert nslice_of_the_library(case) < case[0]
    t = tar.make_inputs(case, seed=420)
    cfg = tar.cfg_of(case)
    a, b = run_split(t, cfg), run_split(t, cfg)
    for n, x in a.items():
        if x is not None:
            assert torch.equal(x, b[n]), n
    for i in (0, 4, 5, 10):
        one = {n: (x[i:i + 1] if n in ("q", "k", "v", "qg", "go", "gog") else x) for n, x in t.items()}
        one["kg"], one["vg"] = one["k"], one["v"]                          # shared global weights, as in t
        o1 = run_split(one, cfg)
        for n in ("o", "og", "lse", "lse_g", "dq", "dk", "dv", "dqg"):
            assert torch.equal(a[n][i:i + 1], o1[n]), (i, n)


# --------------------------------------------------------------------------- routing through ops and the module
KW = dict(dim=96, num_heads=3, qkv_bias=True, w=7, nglo=1, exact=0, rpe=True, sharew=True)


@pytest.fixture
def precision():
    before = torch.backends.cuda.matmul.fp32_precision
    yield
    torch.backends.cuda.matmul.fp32_precision = before


def _module(impl="auto", **kw):
    mod = B200Long2DSCSelfAttention(**dict(KW, **kw)).to(DEV)
    mod.impl = impl
    return mod


def _module_run(mod, x, gy):
    """output, input gradient, and the family / main kernel of the forward and of the backward.  The library reports
    them per thread, and autograd runs the backward on a thread of its own: a hook on x reads them there."""
    x = x.detach().clone().requires_grad_(True)
    seen = []
    x.register_hook(lambda g: seen.append((_lib.last_impl(), _lib.last_kernel())))
    y = mod(x, 14, 14)
    fwd = (_lib.last_impl(), _lib.last_kernel())
    (y * gy).sum().backward()
    torch.cuda.synchronize()
    return y, x.grad, fwd, seen[0]


@gpu
def test_default_precision_runs_simt_bitwise(precision):
    torch.backends.cuda.matmul.fp32_precision = "none"
    torch.manual_seed(0)
    mods = {impl: _module(impl) for impl in ("auto", "simt")}
    mods["simt"].load_state_dict(mods["auto"].state_dict())
    x = torch.randn(2, 1 + 196, 96, device=DEV)
    gy = torch.randn_like(x)
    ya, ga, fa, ba = _module_run(mods["auto"], x, gy)
    ys, gs, _, _ = _module_run(mods["simt"], x, gy)
    assert (fa[0], ba[0]) == ("simt", "simt")
    assert torch.equal(ya, ys) and torch.equal(ga, gs)


@gpu
def test_high_precision_routes_d32_to_split_and_d128_to_simt(precision):
    torch.set_float32_matmul_precision("high")
    torch.manual_seed(0)
    x = torch.randn(2, 1 + 196, 96, device=DEV)
    gy = torch.randn_like(x)
    _, _, fwd, bwd = _module_run(_module(), x, gy)
    assert (fwd, bwd) == (("wgmma", "wgmma_f32split_fwd"), ("wgmma", "wgmma_f32split_bwd"))
    _, _, fwd, bwd = _module_run(_module("simt"), x, gy)                 # impl="simt" keeps forcing SIMT
    assert (fwd[0], bwd[0]) == ("simt", "simt")
    x = torch.randn(2, 1 + 196, 256, device=DEV)                         # D = 128
    _, _, fwd, bwd = _module_run(_module(dim=256, num_heads=2), x, torch.randn_like(x))
    assert (fwd[0], bwd[0]) == ("simt", "simt")


@gpu
def test_backward_keeps_the_forwards_choice(precision):
    torch.set_float32_matmul_precision("high")
    torch.manual_seed(0)
    mod = _module()
    x = torch.randn(2, 197, 96, device=DEV, requires_grad=True)
    seen = []
    x.register_hook(lambda g: seen.append((_lib.last_impl(), _lib.last_kernel())))
    y = mod(x, 14, 14)
    torch.set_float32_matmul_precision("highest")
    y.sum().backward()
    torch.cuda.synchronize()
    assert seen == [("wgmma", "wgmma_f32split_bwd")]


@gpu
def test_module_fp32_under_high_precision_matches_the_fp64_oracle(precision):
    """as a user runs it: under "high" the module's q / kv / proj Linears run TF32 as well, so the bar is TF32's"""
    torch.set_float32_matmul_precision("high")
    torch.manual_seed(0)
    ref = OracleLong2DSCSelfAttention(**KW).double()
    with torch.no_grad():                     # a bias table and global biases of the size training gives them
        for n, p in ref.named_parameters():
            if "relative_position" in n:
                p.normal_(0.0, 0.5)
    x = torch.randn(2, 197, 96, dtype=torch.float64, requires_grad=True)
    y_ref = ref(x, 14, 14)
    gy = torch.randn_like(y_ref)
    (y_ref * gy).sum().backward()
    mod = _module()
    mod.load_state_dict(ref.state_dict())
    xg = x.detach().float().to(DEV).requires_grad_(True)
    y = mod(xg, 14, 14)
    (y * gy.float().to(DEV)).sum().backward()
    torch.cuda.synchronize()
    assert _lib.last_kernel() == "wgmma_f32split_fwd"
    errs = dict(y=relerr(y, y_ref), dx=relerr(xg.grad, x.grad))
    gref = dict(ref.named_parameters())
    for n, p in mod.named_parameters():
        errs["d" + n] = relerr(p.grad, gref[n].grad)
    record("f32split_module_vs_fp64_oracle", "rpe_w7_g1", **errs)
    bad = {n: e for n, e in errs.items() if not e < MODULE_BAR}
    assert not bad, bad
