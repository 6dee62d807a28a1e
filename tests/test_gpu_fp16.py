"""The fp16 paths and the gradients under GradScaler's loss scales.

The reference trains under fp16 autocast with a GradScaler, so that is where a reference training run lands on this port.
This file holds what the precisions the other files were built around (bf16, fp32) leave open:

* row by row (the measurements of test_gpu_attention_rows, and the bias gradients entry by entry of
  test_gpu_bias_entries), the outputs the router can pick that no row test held: the wgmma kernels with fp16 outputs,
  contiguous and in the production layout, and the SIMT kernels in fp16 and bf16 (the family `impl="auto"` falls back to
  for D % 8 != 0, misaligned views and outside the wgmma coverage);
* loss scales dO 2^s: bitwise equivariance where the outputs have fp32's exponent range; in fp16, the gradients (÷ 2^s)
  at the row bars over the scales that stay in range, and an overflow that always comes out non-finite, never as a
  clamped finite value (GradScaler's only signal);
* a non-finite dO entry reaches the gradients and the bias-table gradients of the attention, and a non-finite dy reaches
  the gradients of the LayerNorm, addnorm and bias epilogue kernels;
* the harness trained under fp16 autocast with torch.amp.GradScaler: the fused residual path against the stock
  composition and against fp32, and the scaler's skip / step decisions.

Floors for fp16 outputs (`store_eps`, `peak_floors` below): delta is formed from the stored o, eps_o = 2^-11; a stored
gradient row that the global-query backward adds one term into per global query pays 2^-12 sqrt(g) rms (the fp16
counterpart of the bf16 2^-9 of test_gpu_attention_rows); and a stored fp16 value below 2^-14 is subnormal, so every
gradient row takes a floor of 2^-24 sqrt(D) for its store.  The SIMT kernels do their arithmetic in fp32: only their
stored outputs round.

The bars were measured on an H100 SXM (700 W power limit), each about 2.5x the worst value seen over this file
(DESIGN.md section 4).
"""
import ctypes
import math

import pytest
import torch

import __graft_entry__ as ge
from oracle import vil_oracle as vo
from tests import test_gpu_attention_rows as tar
from tests import test_gpu_bias_entries as tbe
from tests import test_gpu_dropout as tdrop
from tests import test_gpu_epilogue_rounds as tep
from tests import test_gpu_f32_split as tsplit
from tests import test_gpu_parity as tpar
from tests import test_staging_alignment as tsa
from tests.util import record, relerr
from vision_longformer_b200 import _lib, epilogue, ops
from vision_longformer_b200.msvit import DropPath, build_vil

gpu = pytest.mark.gpu
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
DEV = "cuda"
FP16_MAX = 65504.0

# family, dtype, VIL_FLAG_F32_OUT, layout (test_gpu_attention_rows.VARIANTS)
VARIANTS = {
    "wgmma_fp16": ("wgmma", F16, False, "contig"),
    "wgmma_fp16_linear": ("wgmma", F16, False, "linear"),
    "simt_fp16": ("simt", F16, False, "contig"),
    "simt_bf16": ("simt", BF16, False, "contig"),
}
# Rows forward / backward, chunks forward / backward, lse absolute.  Worst values measured (rows, chunks): see DESIGN.md
# section 4.
# Worst values measured (rows forward / backward, chunks forward / backward; backward rows of the global keys at g >= 4
# apart, which take the allowance for the global-query roundings on top): wgmma fp16 (both layouts) 5.0e-4 / 1.7e-3,
# 3.1e-4 / 5.3e-4; SIMT fp16 3.6e-4 / 1.6e-3, 2.6e-4 / 5.9e-4; SIMT bf16 2.9e-3 / 6.5e-3, 2.0e-3 / 3.8e-3; lse 2.3e-6.
# The worst backward rows are dq rows of the mode-8 case in both fp16 families alike: delta formed from the stored fp16 o.
BARS = {
    "wgmma_fp16": dict(row=(1.25e-3, 4e-3), chunk=(8e-4, 1.3e-3), lse=5e-6),
    "simt_fp16": dict(row=(1e-3, 4e-3), chunk=(6.5e-4, 1.5e-3), lse=6e-6),
    "simt_bf16": dict(row=(7.5e-3, 1.6e-2), chunk=(5e-3, 1e-2), lse=6e-6),
}
BARS["wgmma_fp16_linear"] = BARS["wgmma_fp16"]
# the bias gradients over the whole tensor, and entry by entry (test_gpu_bias_entries: err <= kappa T_e; eps_o is the
# roundoff of the o that delta is formed from: the stored type, plus the fp16 P operand in the wgmma family).  Worst
# measured over the tensor: wgmma fp16 5.2e-4, SIMT fp16 5.2e-4, SIMT bf16 6.7e-3; err / T_e: wgmma fp16 in the
# production layout 6.9e-5, SIMT fp16 6.9e-5, SIMT bf16 7.7e-4 (sparse entries of the dropout cases)
BIAS_BARS = {"wgmma_fp16": 1.5e-3, "wgmma_fp16_linear": 1.5e-3, "simt_fp16": 1.5e-3, "simt_bf16": 2e-2}
EPS_O = {"wgmma_fp16_linear": 2.0 ** -10, "simt_fp16": tbe.U32 + 2.0 ** -11, "simt_bf16": tbe.U32 + 2.0 ** -8}
KAPPA = {"wgmma_fp16_linear": 2e-4, "simt_fp16": 2e-4, "simt_bf16": 2e-3}
PEAK_VARIANTS = ["wgmma_fp16", "simt_fp16", "simt_bf16"]


def fp16_out(variant):
    impl, dtype, f32out, layout = tar.VARIANTS[variant]
    return dtype == F16 and not f32out


def _store_eps(orig):
    def store_eps(variant):
        return (2.0 ** -11, 2.0 ** -12) if fp16_out(variant) else orig(variant)
    return store_eps


def _peak_floors(orig):
    """the row file's floors, plus the store of a gradient row in fp16's subnormal range: 2^-24 sqrt(D) per row"""
    def peak_floors(t, cfg, variant, g):
        f = orig(t, cfg, variant, g)
        if fp16_out(variant):
            store = 2.0 ** -24 * t["q"].shape[-1] ** 0.5
            f = {n: x + store for n, x in f.items()}
            for n in ("dq", "dk", "dv", "dqg", "dkg", "dvg"):
                f.setdefault(n, store)
        return f
    return peak_floors


@pytest.fixture(autouse=True)
def fp16_variants(monkeypatch):
    """the helpers of the row and bias-entry files, taught the variants of this file for the duration of one test"""
    for n, v in VARIANTS.items():
        monkeypatch.setitem(tar.VARIANTS, n, v)
        monkeypatch.setitem(tar.BARS, n, BARS[n])
        monkeypatch.setitem(tar.BIAS_BARS, n, BIAS_BARS[n])
        monkeypatch.setitem(tbe.VARIANTS, n, v)
    for n in EPS_O:
        monkeypatch.setitem(tbe.EPS_O, n, EPS_O[n])
        monkeypatch.setitem(tbe.KAPPA, n, KAPPA[n])
    monkeypatch.setattr(tar, "store_eps", _store_eps(tar.store_eps))
    monkeypatch.setattr(tar, "peak_floors", _peak_floors(tar.peak_floors))


def variants_for(case, names=None):
    """the SIMT backward refuses bf16 / fp16 above D = 64; the 56 x 56 oracle is run for bf16 only"""
    out = []
    for n in names or VARIANTS:
        if VARIANTS[n][0] == "simt" and case[2] > 64:
            continue
        if case[3] * case[4] > 2000 and VARIANTS[n][1] != BF16:
            continue
        out.append(n)
    return out


def expand(cases, names=None):
    return [pytest.param(c, n, id=tar.CASE_ID(c) + "-" + n) for c in cases for n in variants_for(c, names)]


# --------------------------------------------------------------------------- (1) row by row
@gpu
@pytest.mark.parametrize("case,variant", expand(tar.GEOMETRY_CASES))
def test_rows_random_inputs(case, variant):
    t = tar.make_inputs(case, seed=310)
    cfg = tar.cfg_of(case)
    ref = tar.oracle(t, cfg, VARIANTS[variant][1], ("geo",) + case)
    tar.check("fp16_rows_random_inputs", "randn", tar.run_kernels(t, cfg, variant), ref, case, variant)


@gpu
@pytest.mark.parametrize("case,variant", expand(tar.MASKED_CASES))
def test_rows_masked_leading_pieces(case, variant):
    t = tar.make_inputs(case, seed=330)
    cfg = tar.cfg_of(case)
    ref = tar.oracle(t, cfg, VARIANTS[variant][1], ("masked",) + case)
    tar.check("fp16_rows_masked_leading_pieces", "randn", tar.run_kernels(t, cfg, variant), ref, case, variant)


@gpu
@pytest.mark.parametrize("case,variant", expand(tar.MANY_GLOBAL_CASES))
def test_rows_more_than_64_global_tokens(case, variant):
    t = tar.make_inputs(case, seed=340, sep=case[10])
    cfg = tar.cfg_of(case)
    ref = tar.oracle(t, cfg, VARIANTS[variant][1], ("glob",) + case)
    tar.check("fp16_rows_more_than_64_global_tokens", "randn", tar.run_kernels(t, cfg, variant), ref, case, variant)


DROP_CASES = [(1, 2, 32, 15, 13, 2, 7, 0, 0, True), (1, 2, 32, 14, 14, 65, 7, 0, 0, True, False)]


@gpu
@pytest.mark.parametrize("case,variant", expand(DROP_CASES))
def test_rows_dropout(case, variant):
    t = tar.make_inputs(case, seed=311)
    ref = tar.dropout_reference(t, case, VARIANTS[variant][1])
    tar.check("fp16_rows_dropout", "p0.1", tar.run_kernels(t, tar.cfg_of(case), variant, drop=tar.DROP), ref, case, variant)


def _peak_params():
    return [pytest.param(*p.values[:3], v, id=p.id.rsplit("-", 1)[0] + "-" + v)
            for p in tar._peak_params() if p.values[3] == "simt_fp32" for v in PEAK_VARIANTS]


@gpu
@pytest.mark.parametrize("case,target,L,variant", _peak_params())
def test_rows_peaked_through_q_and_k(case, target, L, variant):
    tag = "%s_L%d" % ("_".join(str(x) for x in target), L)
    t, hot = tar.peak_through_qk(tar.make_inputs(case, seed=320), case, VARIANTS[variant][1], L, target)
    tar.check_peaked("fp16_rows_peaked_through_q_and_k", case, variant, t, tag, L, hot)


@gpu
@pytest.mark.parametrize("variant", PEAK_VARIANTS)
@pytest.mark.parametrize("L", tar.GAPS)
@pytest.mark.parametrize("what", tar.TABLE_PEAKS, ids=lambda x: "_".join(str(y) for y in x))
def test_rows_peaked_through_the_bias(what, L, variant):
    t = tar.peak_through_table(tar.make_inputs(tar.PK_TABLE, seed=321), tar.PK_TABLE, L, what)
    tar.check_peaked("fp16_rows_peaked_through_the_bias", tar.PK_TABLE, variant, t,
                     "%s_L%d" % ("_".join(str(x) for x in what), L), L)


@gpu
@pytest.mark.parametrize("variant", PEAK_VARIANTS)
@pytest.mark.parametrize("shift", [60, -60])
def test_rows_common_shift_of_all_scores(shift, variant):
    """test_gpu_attention_rows' common shift: o must not move, lse moves by the row's shift.  The gradients are recorded,
    not held: delta from an o stored in fp16 / bf16 leaves eps_o |dS| c of the common component c u of every k_j in dq"""
    case = (1, 2, 32, 21, 21, 2, 7, 0, 0, False)
    D = case[2]
    t = tar.make_inputs(case, seed=322)
    u = torch.nn.functional.normalize(t["q"].mean(dim=2, keepdim=True), dim=-1)
    t["q"] = t["q"] - (t["q"] * u).sum(-1, keepdim=True) * u + (2 + 0.3 * (t["q"] * u).sum(-1, keepdim=True)) * u
    t["k"] = t["k"] + shift / (2 * D ** -0.5) * u
    t["kg"] = t["k"]
    tar.check_peaked("fp16_rows_common_shift_of_all_scores", case, variant, t, "shift%d" % shift, abs(shift) * 2,
                     floors=False, backward=False)


@gpu
@pytest.mark.parametrize("case,variant", expand(tar.MASKED_CASES[:2], PEAK_VARIANTS))
@pytest.mark.parametrize("L", [40, 100])
def test_rows_masked_leading_pieces_then_the_maximum_in_the_last_chunk(case, variant, L):
    t, hot = tar.peak_through_qk(tar.make_inputs(case, seed=331), case, VARIANTS[variant][1], L, ("off", 1, 1, "same"))
    tar.check_peaked("fp16_rows_masked_leading_pieces_then_the_maximum_in_the_last_chunk", case, variant, t,
                     "off_1_1_L%d" % L, L, hot)


# --------------------------------------------------------------------------- routing to SIMT through impl="auto"
ROUTE_CASE = (1, 2, 20, 15, 13, 2, 7, 0, 0, True)          # D = 20: rows of 40 bytes


@gpu
@pytest.mark.parametrize("dtype", [F16, BF16], ids=["fp16", "bf16"])
def test_auto_takes_simt_for_a_head_dim_off_8(dtype):
    case = ROUTE_CASE
    t = tar.make_inputs(case, seed=350)
    cfg = tar.cfg_of(case)
    out, fam_f, fam_b = tpar.kernel_run(t, *cfg, dtype, "auto")
    assert (fam_f, fam_b) == ("simt", "simt")
    variant = "simt_fp16" if dtype == F16 else "simt_bf16"
    tar.check("fp16_auto_simt_head_dim_20", "randn", out, tar.oracle(t, cfg, dtype, ("route",) + case), case, variant)


def misaligned_run(t, cfg, dtype):
    """forward + backward through the C ABI with impl="auto", every input a contiguous view that starts one element past
    a 16-byte boundary"""
    nx, ny, w, exact, mode, scale = cfg

    def off(x):
        buf = torch.empty(x.numel() + 1, device=DEV, dtype=dtype)
        v = buf[1:].view(x.shape)
        v.copy_(x)
        assert v.data_ptr() % 16 != 0
        return v

    q, k, v, qg, go, gog = (off(t[n]) for n in ("q", "k", "v", "qg", "go", "gog"))
    f32 = lambda x: x.to(DEV, F32).contiguous()
    table, g2l, g2g = f32(t["table"]), f32(t["g2l"]), f32(t["g2g"])
    o, og = torch.empty_like(q), torch.empty_like(qg)
    dq, dk, dv, dqg = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v), torch.empty_like(qg)
    dt, dgl, dgg = torch.zeros_like(table), torch.zeros_like(g2l), torch.zeros_like(g2g)
    kw = dict(nx=nx, ny=ny, w=w, exact=exact, mode=mode, scale=scale, impl="auto")
    lse, lse_g = ops.vil_attention_raw_forward(q, k, v, qg, k, v, table, g2l, g2g, o, og, **kw)
    fam_f = _lib.last_impl()
    ops.vil_attention_raw_backward(q, k, v, qg, k, v, table, g2l, g2g, o, og, lse, lse_g, go, gog, dq, dk, dv, dqg, dk, dv,
                                   dt, dgl, dgg, **kw)
    torch.cuda.synchronize()
    return dict(o=o, og=og, lse=lse, lse_g=lse_g, dq=dq, dk=dk, dv=dv, dqg=dqg, dtable=dt, dg2l=dgl, dg2g=dgg), fam_f, _lib.last_impl()


@gpu
def test_auto_takes_simt_for_misaligned_fp16_views():
    case = (1, 2, 32, 15, 13, 2, 7, 0, 0, True)
    t = tar.make_inputs(case, seed=351)
    cfg = tar.cfg_of(case)
    out, fam_f, fam_b = misaligned_run(t, cfg, F16)
    assert (fam_f, fam_b) == ("simt", "simt")
    tar.check("fp16_auto_simt_misaligned", "randn", out, tar.oracle(t, cfg, F16, ("misaligned",) + case), case, "simt_fp16")


# --------------------------------------------------------------------------- the bias gradients entry by entry
BIAS_CASES = [c for c in tbe.RANDOM_CASES + tbe.MANY_GLOBAL_CASES if c[3] * c[4] <= 2000]
BIAS_NAMES = ["wgmma_fp16_linear", "simt_fp16", "simt_bf16"]


def bias_expand(cases):
    return [pytest.param(c, v, id=tbe.CASE_ID(c) + "-" + v) for c in cases for v in BIAS_NAMES
            if not (VARIANTS[v][0] == "simt" and c[2] > 64)]


@gpu
@pytest.mark.parametrize("case,variant", bias_expand(BIAS_CASES))
def test_bias_entries_random_inputs(case, variant):
    t = tar.make_inputs(tbe.full(case), seed=410, sep=tbe.full(case)[10])
    terms = tbe.terms_of(("rand",) + case, t, case, VARIANTS[variant][1])
    tbe.hold_entries("fp16_bias_entries_random_inputs", "randn", tbe.run_variant(t, case, variant), terms, case, variant)


@gpu
@pytest.mark.parametrize("case,variant", bias_expand([c for c in tbe.DROP_CASES if c[2] <= 64]))
def test_bias_entries_dropout(case, variant):
    B, H, D, nx, ny, g, w, exact, mode, sep, p = case
    t = tar.make_inputs(tbe.full(case), seed=411, sep=sep)
    keep, keep_g = tdrop.keep_tensors(tbe.SEED, tbe.OFFSET, p, B, H, nx, ny, w, g, mode)
    terms = tbe.terms_of(("drop",) + case, t, case, VARIANTS[variant][1], keep, keep_g)
    out = tbe.run_variant(t, case, variant, drop=(p, tbe.SEED, tbe.OFFSET))
    tbe.hold_entries("fp16_bias_entries_dropout", "p%g" % p, out, terms, case, variant)


# --------------------------------------------------------------------------- (2) loss scales
SCALE_CASE = (1, 2, 32, 15, 13, 2, 7, 0, 0, True)           # the table, two global tokens, padding in both directions
FWD = ("o", "og", "lse", "lse_g")
OUTS = ("dq", "dk", "dv", "dqg", "dkg", "dvg")
GRADS = ("dq", "dk", "dv", "dqg", "dtable", "dg2l", "dg2g")
SPLIT = tsplit.V
NODROP = (0.0, 0, 0)


def run(t, cfg, variant, drop=NODROP):
    if variant == SPLIT:
        return tsplit.run_split(t, cfg, drop=drop)
    return tar.run_kernels(t, cfg, variant, drop=drop)


def scaled(t, s, dtype):
    """(t for the kernel, t for the reference) with dO 2^s: the kernel sees dO 2^s rounded to dtype, the reference that
    same value / 2^s (exact in fp64), so that the gradients / 2^s are compared on the dO the kernel saw"""
    rk = lambda x: (x * 2.0 ** s).to(dtype).double()
    tk = dict(t, go=rk(t["go"]), gog=rk(t["gog"]))
    return tk, dict(t, go=tk["go"] / 2.0 ** s, gog=tk["gog"] / 2.0 ** s)


def unscaled(out, s):
    return {n: (x if (x is None or n in FWD) else x.double() / 2.0 ** s) for n, x in out.items()}


def max_ds(t, cfg, dtype):
    """max |dS| = max |P (dP - delta)| of the fp64 dense restatement (vo.dense_attention) on the inputs rounded to dtype,
    over the local rows and the global rows"""
    nx, ny, w, exact, mode, scale = cfg
    rd = lambda x: x.to(dtype).double()
    b32 = lambda n: None if t[n] is None else t[n].float().double()
    q, k, v, go = rd(t["q"]), rd(t["k"]), rd(t["v"]), rd(t["go"])
    table, g2l, g2g = b32("table"), b32("g2l"), b32("g2g")
    g, H = k.shape[2] - q.shape[2], q.shape[1]
    E = vo.visit_weights(nx, ny, w, exact, mode, table, H, dtype=torch.float64)
    s = scale * torch.einsum("bhid,bhjd->bhij", q, vo._pad_keys(k[:, :, g:], nx, ny, w))
    s = s + torch.where(E > 0, torch.log(E.clamp_min(1e-300)), torch.full_like(E, float("-inf")))[None]
    vv = vo._pad_keys(v[:, :, g:], nx, ny, w)
    if g:
        sg = scale * torch.einsum("bhid,bhtd->bhit", q, k[:, :, :g])
        s = torch.cat([sg + (g2l[1][None, :, None, :] if g2l is not None else 0), s], dim=-1)
        vv = torch.cat([v[:, :, :g], vv], dim=2)

    def ds(s, vv, go):
        p = torch.softmax(s, dim=-1)
        o = p @ vv
        return float((p * (go @ vv.transpose(-1, -2) - (go * o).sum(-1, keepdim=True))).abs().max())

    top = ds(s, vv, go)
    if g:
        qg, gog, kg, vg = rd(t["qg"]), rd(t["gog"]), rd(t["kg"]), rd(t["vg"])
        sgl = scale * qg @ kg.transpose(-1, -2)
        if g2g is not None:
            sgl = sgl + torch.cat([g2g, g2l[0][:, :, None].expand(H, g, q.shape[2])], dim=-1)[None]
        top = max(top, ds(sgl, vg, gog))
    return top


def reference_tops(t, cfg, dtype, key):
    """the largest magnitudes at s = 0: the reference's dS, dq, dk, dv, dqg, and the dO the kernel reads"""
    ref = tar.oracle(t, cfg, dtype, key)
    tops = {n: float(ref[n].abs().max()) for n in OUTS if n in ref}
    tops["ds"] = max_ds(t, cfg, dtype)
    tops["do"] = max(float(t[n].to(dtype).abs().max()) for n in ("go", "gog"))
    return ref, tops


def scale_inputs(seed, kind="ds_first"):
    """SCALE_CASE inputs whose gradients leave fp16's range before the scaled dO does.
    "ds_first": v 16 times randn, so that dS, dq and dk grow 16-fold (o and dv do not); dS leaves the range first.
    "dv_first": every query of a chunk dominated (gap 12 through q k) by the first key of its chunk, and dO randn + 2:
    dv of those keys sums 49 dO rows of the same sign, while dS, dq and dk stay small (a saturated softmax).  Separate
    global weights, so that the local dv rows are the wgmma kernels' stores alone (with shared weights the global-query
    pass adds into them and stores them again)."""
    if kind == "ds_first":
        t = tar.make_inputs(SCALE_CASE, seed=seed)
        t["v"] = t["v"] * 16
        t["vg"] = t["v"]
        return t
    t = tar.make_inputs(SCALE_CASE, seed=seed, sep=True)
    kg, vg = t["kg"], t["vg"]
    t, _ = tar.peak_through_qk(t, SCALE_CASE, F16, 12, ("off", 0, 0, "first"))
    return dict(t, kg=kg, vg=vg, go=t["go"] + 2, gog=t["gog"] + 2)


def flush_floors(t, cfg, variant, g):
    """`peak_floors` without its delta term (no saturated softmax here): the flush of P and dS below the operand type
    and the store of a row in fp16's subnormal range"""
    orig = tar.store_eps
    tar.store_eps = lambda v: (0.0, orig(v)[1])
    try:
        return tar.peak_floors(t, cfg, variant, g)
    finally:
        tar.store_eps = orig


EQUI_VARIANTS = ["wgmma_bf16", "wgmma_bf16_linear", SPLIT, "simt_fp32", "simt_bf16"]


@gpu
@pytest.mark.parametrize("drop", [NODROP, tar.DROP], ids=["p0", "p0.1"])
@pytest.mark.parametrize("variant", EQUI_VARIANTS)
def test_gradients_are_bitwise_equivariant_under_power_of_two_loss_scales(variant, drop):
    """outputs with fp32's exponent range: scaling dO by 2^s commutes with every rounding, so every gradient is bitwise
    2^s times the s = 0 one, and the forward does not move.  Dropout's 1 / (1 - p) is one more constant factor."""
    case = SCALE_CASE
    t = tar.make_inputs(case, seed=510)
    cfg = tar.cfg_of(case)
    base = run(t, cfg, variant, drop)
    for s in range(-20, 21):
        if s == 0:
            continue
        out = run(dict(t, go=t["go"] * 2.0 ** s, gog=t["gog"] * 2.0 ** s), cfg, variant, drop)
        for n in FWD:
            assert torch.equal(out[n], base[n]), (s, n)
        for n in GRADS:
            if base[n] is not None:
                want = base[n] * 2.0 ** s
                assert torch.equal(out[n], want), (s, n, float((out[n].double() - want.double()).abs().max()))


FP16_VARIANTS = ["wgmma_fp16", "wgmma_fp16_linear", "simt_fp16"]


def largest_scale_in_range(tops):
    """the largest s at which every scaled reference dS, dq, dk, dv and dqg stays under 65504 / 2"""
    return int(math.floor(math.log2(FP16_MAX / 2 / max(tops.values()))))


@gpu
@pytest.mark.parametrize("variant", FP16_VARIANTS)
def test_fp16_gradients_follow_the_loss_scale_in_range(variant):
    """From s = -10 (dO 2^-10: a twentieth of its entries subnormal in fp16) up to the largest s in range, the gradients
    / 2^s meet the row bars plus the flush floors of `peak_floors` recomputed for the scaled dO; at that s everything is
    finite"""
    case = SCALE_CASE
    t = scale_inputs(511)
    cfg = tar.cfg_of(case)
    _, tops = reference_tops(t, cfg, F16, ("scale", "ds_first", 0) + case)
    smax = largest_scale_in_range(tops)
    assert smax >= 8, tops
    for s in range(-10, smax + 1):
        tk, tr = scaled(t, s, F16)
        ref = tar.oracle(tr, cfg, F16, ("scale", "ds_first", s) + case)
        out = run(tk, cfg, variant)
        floors = {n: x / 2.0 ** s for n, x in flush_floors(tk, cfg, variant, case[5]).items()}
        tar.check("fp16_loss_scales_in_range", "s%+d" % s, unscaled(out, s), ref, case, variant, floors=floors)
        if s == smax:
            for n, x in out.items():
                assert x is None or bool(torch.isfinite(x).all()), (s, n)
    record("fp16_loss_scales_in_range", tar.CASE_ID(case) + "/" + variant, largest_scale_in_range=smax, **tops)


@gpu
@pytest.mark.parametrize("kind", ["ds_first", "dv_first"])
@pytest.mark.parametrize("variant", FP16_VARIANTS)
def test_fp16_overflow_comes_out_non_finite(variant, kind):
    """Past the largest s in range: an output whose scaled reference exceeds fp16's range (65520 rounds to inf) contains
    a non-finite value, and an output that is finite is right (÷ 2^s, at the whole-tensor backward bar), never a clamped
    65504.  A non-finite output whose reference is in range needs an overflow of dS, which the wgmma kernels round to
    fp16 for the tensor cores (the reference's own fp16 einsums have the same limit; the SIMT kernels keep dS in fp32),
    or of the scaled dO itself.  Under the saturated softmax of "dv_first" dq and dk are cancellations (held row by row
    with floors elsewhere), so there only dv is held for its value."""
    case = SCALE_CASE
    t = scale_inputs(511, kind)
    held = ("dq", "dk", "dv", "dqg") if kind == "ds_first" else ("dv",)
    cfg = tar.cfg_of(case)
    _, tops = reference_tops(t, cfg, F16, ("scale", kind, 0) + case)
    smax = largest_scale_in_range(tops)
    first, reached, fails = None, False, []
    bar = BARS[variant]["row"][1]
    for s in range(smax, smax + 6):
        tk, tr = scaled(t, s, F16)
        ref = tar.oracle(tr, cfg, F16, ("scale", kind, s) + case)
        out = run(tk, cfg, variant)
        outs = [n for n in OUTS if n in ref]
        bad = {n for n in outs if not bool(torch.isfinite(out[n]).all())}
        bias_bad = {n for n in ("dtable", "dg2l", "dg2g") if not bool(torch.isfinite(out[n]).all())}
        over = {n for n in outs if tops[n] * 2.0 ** s > 65520 * 1.01}
        near = {n for n in outs if tops[n] * 2.0 ** s > FP16_MAX * 0.99}
        ds_over = tops["ds"] * 2.0 ** s > FP16_MAX * 0.99
        do_over = tops["do"] * 2.0 ** s > FP16_MAX
        reached = reached or bool(over)
        if first is None and (bad or bias_bad):
            first = s
            record("fp16_overflow", tar.CASE_ID(case) + "/" + kind + "/" + variant, first_non_finite_scale=s,
                   first_non_finite_outputs=len(bad), non_finite_bias_gradients=len(bias_bad),
                   ds_over=float(ds_over), do_over=float(do_over), reference_outputs_over=len(near))
        if s == smax and (bad or bias_bad):
            fails.append("s = %d (in range): non-finite %s" % (s, sorted(bad | bias_bad)))
        if over - bad:
            fails.append("s = %d: %s exceed fp16's range in the reference and came out finite" % (s, sorted(over - bad)))
        if (bad - near) and not ((VARIANTS[variant][0] == "wgmma" and ds_over) or do_over):
            fails.append("s = %d: %s non-finite with the reference in range and no dS overflow" % (s, sorted(bad - near)))
        for n in held:
            if n not in bad and n not in near:
                e = relerr(out[n].double() / 2.0 ** s, ref[n])
                if not e < bar:
                    fails.append("s = %d: %s finite but wrong, %.3e (bar %.1e)" % (s, n, e, bar))
    assert not fails, "\n".join(fails)
    # an output left the range in the reference, and a non-finite value came before the scaled dO itself overflowed
    assert reached and first is not None and tops["do"] * 2.0 ** first < FP16_MAX, (first, smax, tops)


NF_VARIANTS = ["simt_fp32", SPLIT, "wgmma_fp16_f32out", "wgmma_bf16", "wgmma_bf16_linear", "wgmma_fp16",
               "wgmma_fp16_linear", "simt_fp16", "simt_bf16"]


@gpu
@pytest.mark.parametrize("where", ["local", "global"])
@pytest.mark.parametrize("value", [float("inf"), float("nan")], ids=["inf", "nan"])
@pytest.mark.parametrize("rpe", [True, False], ids=["table", "no_table"])
@pytest.mark.parametrize("variant", NF_VARIANTS)
def test_non_finite_d_o_reaches_the_gradients(variant, rpe, value, where):
    """One entry of one dO row +inf or NaN: the dq row of that query is non-finite, so are the bias gradients the row
    feeds (a local row: the table and g2l; a global row: g2g and g2l), and the forward is bit for bit the clean one.
    Nothing is said about the other rows: a masked P = 0 times an infinite delta is NaN in the kernels where the
    reference's masked fill zeroes it, and the step is skipped either way."""
    case = SCALE_CASE[:9] + (rpe,)
    t = tar.make_inputs(case, seed=520)
    cfg = tar.cfg_of(case)
    clean = run(t, cfg, variant)
    key, row = ("go", 100) if where == "local" else ("gog", 1)
    x = t[key].clone()
    x[0, 1, row, 3] = value
    out = run(dict(t, **{key: x}), cfg, variant)
    for n in FWD:
        assert torch.equal(out[n], clean[n]), n
    dq = out["dq" if where == "local" else "dqg"][0, 1, row]
    assert not bool(torch.isfinite(dq).all()), dq
    if rpe:
        for n in (("dtable", "dg2l") if where == "local" else ("dg2g", "dg2l")):
            assert not bool(torch.isfinite(out[n]).all()), n
    record("fp16_non_finite_d_o", "%s/%s/%s/%s" % (variant, "table" if rpe else "no_table", value, where),
           **{"non_finite_" + n: float((~torch.isfinite(out[n])).sum()) for n in GRADS if out[n] is not None})


def _hold_non_finite(name, x, rows=None, cols=None):
    """x non-finite exactly in the given rows (every one of them) or columns (every one of them)"""
    bad = ~torch.isfinite(x.float())
    if rows is not None:
        per = bad.reshape(x.shape[0], -1).any(dim=1)
        assert bool(per[rows].all()) and int(per.sum()) == len(rows), (name, per.nonzero().flatten().tolist()[:8])
    else:
        per = bad.reshape(-1, x.shape[-1]).any(dim=0)
        assert bool(per[cols].all()) and int(per.sum()) == len(cols), (name, per.nonzero().flatten().tolist()[:8])


EP_ROWS, EP_BAD = 3001, (1777, 41)


@gpu
@pytest.mark.parametrize("value", [float("inf"), float("nan")], ids=["inf", "nan"])
@pytest.mark.parametrize("xdt,ydt,C", [(F16, F16, 96), (BF16, BF16, 96), (F32, F16, 97), (F16, F32, 96), (F32, F16, 96),
                                       (F32, BF16, 96)],
                         ids=["layernorm_f16", "layernorm_bf16", "layernorm_f32_f16_scalar", "layernorm_f16_f32",
                              "addnorm_vec_f32_f16", "addnorm_vec_f32_bf16"])
def test_layernorm_backward_passes_a_non_finite_dy(xdt, ydt, C, value):
    """B200LayerNorm: the vil_layernorm_* kernels (bf16 / fp16 input, or fp32 with C % 4 != 0) and the vectorised
    vil_addnorm_* route (fp32 input, C % 4 == 0).  One dy entry non-finite: that dx row, and the dgamma and dbeta
    columns of that entry, through the fixed-order reduce of the per-CTA partials; nothing else."""
    gen = torch.Generator(device=DEV).manual_seed(60)
    ln, amp = tep._ln_module(C, xdt, ydt, gen)
    x = (torch.randn(EP_ROWS, C, device=DEV, generator=gen) * 2 + 0.5).to(xdt).requires_grad_(True)
    y = tep._ln_run(ln, amp, x)
    assert y.dtype == ydt
    dy = torch.randn(EP_ROWS, C, device=DEV, generator=gen).to(ydt)
    dy[EP_BAD] = value
    dx, dg, db = torch.autograd.grad(y, (x, ln.weight, ln.bias), dy)
    _hold_non_finite("dx", dx, rows=[EP_BAD[0]])
    _hold_non_finite("dgamma", dg, cols=[EP_BAD[1]])
    _hold_non_finite("dbeta", db, cols=[EP_BAD[1]])


@gpu
@pytest.mark.parametrize("value", [float("inf"), float("nan")], ids=["inf", "nan"])
@pytest.mark.parametrize("dt", [F16, BF16], ids=["f16", "bf16"])
def test_addnorm_backward_passes_a_non_finite_dy(dt, value):
    """epilogue.addnorm_raw_backward with bf16 / fp16 dy and dbr: the dx and dbr rows of the entry, the dgamma and dbeta
    columns of the entry, and every column of dbias (the column sums of dbr, whose row is non-finite throughout)"""
    gen = torch.Generator(device=DEV).manual_seed(61)
    rnd = lambda *s: torch.randn(*s, device=DEV, generator=gen)
    C = 96
    x, br, bias = rnd(EP_ROWS, C) * 2 + 0.5, rnd(EP_ROWS, C).to(dt), 0.3 * rnd(C)
    gamma, beta = 1 + 0.3 * rnd(C), 0.3 * rnd(C)
    xo, y = torch.empty_like(x), torch.empty(EP_ROWS, C, device=DEV, dtype=dt)
    mean, rstd = torch.empty(EP_ROWS, device=DEV), torch.empty(EP_ROWS, device=DEV)
    epilogue.addnorm_raw_forward(x, br, bias, None, gamma, beta, xo, y, mean, rstd, tep.EPS)
    dy, gres = rnd(EP_ROWS, C).to(dt), rnd(EP_ROWS, C)
    dy[EP_BAD] = value
    dx, dbr = torch.empty_like(x), torch.empty_like(br)
    dg, db, dbias = (torch.empty(C, device=DEV) for _ in range(3))
    epilogue.addnorm_raw_backward(xo, gamma, mean, rstd, None, dy, gres, dx, dbr, dg, db, dbias,
                                  epilogue.addnorm_workspace(EP_ROWS, C, DEV), tep.EPS)
    torch.cuda.synchronize()
    for n, v in (("dx", dx), ("dbr", dbr)):
        _hold_non_finite(n, v, rows=[EP_BAD[0]])
    for n, v in (("dgamma", dg), ("dbeta", db)):
        _hold_non_finite(n, v, cols=[EP_BAD[1]])
    _hold_non_finite("dbias", dbias, cols=list(range(C)))


@gpu
@pytest.mark.parametrize("value", [float("inf"), float("nan")], ids=["inf", "nan"])
@pytest.mark.parametrize("act", ["gelu", "none"])
@pytest.mark.parametrize("dt", [F16, BF16], ids=["f16", "bf16"])
def test_bias_act_backward_passes_a_non_finite_da(dt, act, value):
    """epilogue.bias_act_raw_backward: dz = da GELU'(z + bias) non-finite at the entry alone, and the dbias column of
    the entry"""
    gen = torch.Generator(device=DEV).manual_seed(62)
    C = 384
    code = _lib.VIL_ACT_GELU if act == "gelu" else _lib.VIL_ACT_NONE
    z = (2 * torch.randn(EP_ROWS, C, device=DEV, generator=gen)).to(dt)
    bias = 0.5 * torch.randn(C, device=DEV, generator=gen)
    da = torch.randn(EP_ROWS, C, device=DEV, generator=gen).to(dt)
    da[EP_BAD] = value
    dz = torch.empty_like(z) if act == "gelu" else None
    dbias = torch.empty(C, device=DEV)
    epilogue.bias_act_raw_backward(da, z, bias, dz, dbias, epilogue.bias_act_workspace(da, code), code)
    torch.cuda.synchronize()
    if dz is not None:
        bad = ~torch.isfinite(dz.float())
        assert bool(bad[EP_BAD]) and int(bad.sum()) == 1
    _hold_non_finite("dbias", dbias, cols=[EP_BAD[1]])


# --------------------------------------------------------------------------- (3) the harness under fp16 autocast
ARCH = "l1,h2,d64,n2,s1,g1,p4,f7_l2,h2,d128,n2,s0,g1,p2,f7_l3,h4,d256,n1,s0,g0,p2,f7"
# Worst over logits, input gradient and every parameter gradient, measured on an H100 SXM (700 W): fused against stock
# 6.0e-4, fp16 against fp32 1.0e-3, the update of the first step taken 1.7e-3 (both nets took it at 2^13)
MODEL_BAR = 1.5e-3          # fused against stock, both under fp16 autocast
MODEL_F32_BAR = 2.5e-3      # fused under fp16 autocast against fused in fp32 (SIMT attention)
STEP_BAR = 4e-3             # the parameter update of the first step taken, fused against stock


@pytest.fixture
def nets(monkeypatch):
    """test_fused_residual_matches_stock_in_fp32's pair: the 112-px arch, fused_residual=True and the stock composition
    with the same weights, every DropPath module returning fixed, distinct per-sample scales in the same order"""
    before = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    torch.manual_seed(0)
    kw = dict(img_size=112, num_classes=50, drop_path_rate=0.2)
    a = build_vil(ARCH, fused_residual=True, **kw).to(DEV).train()
    b = build_vil(ARCH, fused_residual=False, **kw).to(DEV).train()
    b.load_state_dict(a.state_dict())
    calls = [0]
    base = torch.tensor([0.0, 0.8, 1.25, 1.6], device=DEV)

    def fixed_scale(self, batch, device):
        if self.drop_prob == 0. or not self.training:
            return None
        calls[0] += 1
        return base.roll(calls[0])[:batch].clone()

    monkeypatch.setattr(DropPath, "sample_scale", fixed_scale)
    gen = torch.Generator(device=DEV).manual_seed(7)
    x = torch.randn(4, 3, 112, 112, device=DEV, generator=gen)
    gy = torch.randn(4, 50, device=DEV, generator=gen)
    yield a, b, x, gy, calls
    torch.backends.cuda.matmul.fp32_precision = before


def _forward_backward(net, x, gy, calls, scaler=None, amp=True):
    calls[0] = 0
    xg = x.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=F16, enabled=amp):
        y = net(xg)
    loss = (y.float() * gy).sum()
    (scaler.scale(loss) if scaler is not None else loss).backward()
    return y.float(), xg.grad


def _opt(net):
    return torch.optim.SGD(net.parameters(), lr=0.01)


@gpu
def test_harness_under_fp16_autocast_matches_stock_and_fp32(nets):
    """logits, input gradient and every parameter gradient after scaler.unscale_: the fused net against the stock
    composition under fp16 autocast, and against the fused net in fp32 without autocast (attention on SIMT)"""
    a, b, x, gy, calls = nets
    res = {}
    for name, net in (("fused", a), ("stock", b)):
        scaler, opt = torch.amp.GradScaler("cuda", init_scale=2.0 ** 10), _opt(net)
        opt.zero_grad(set_to_none=True)
        y, dx = _forward_backward(net, x, gy, calls, scaler)
        scaler.unscale_(opt)
        res[name] = (y, dx / 2.0 ** 10, {k: p.grad.clone() for k, p in net.named_parameters() if p.grad is not None})
        assert all(bool(torch.isfinite(g).all()) for g in res[name][2].values()), name
    a.zero_grad(set_to_none=True)
    y32, dx32 = _forward_backward(a, x, gy, calls, amp=False)
    assert _lib.last_impl() == "simt"
    res["fp32"] = (y32, dx32, {k: p.grad.clone() for k, p in a.named_parameters() if p.grad is not None})

    def errs(u, v):
        e = {"logits": relerr(u[0], v[0]), "dx": relerr(u[1], v[1])}
        e.update({k: relerr(g, v[2][k]) for k, g in u[2].items() if v[2][k].numel() > 0 and v[2][k].abs().max() > 0})
        return e

    assert res["fused"][2].keys() == res["stock"][2].keys() == res["fp32"][2].keys()
    e16, e32 = errs(res["fused"], res["stock"]), errs(res["fused"], res["fp32"])
    w16, w32 = max(e16.items(), key=lambda kv: kv[1]), max(e32.items(), key=lambda kv: kv[1])
    record("fp16_harness_fused_vs_stock", ARCH, logits=e16["logits"], dx=e16["dx"], worst_param=max(e16.values()))
    record("fp16_harness_fp16_vs_fp32", ARCH, logits=e32["logits"], dx=e32["dx"], worst_param=max(e32.values()))
    assert w16[1] < MODEL_BAR, w16
    assert w32[1] < MODEL_F32_BAR, w32


def _step(net, opt, scaler, x, gy, calls):
    """one training step; True when it was taken (the scale did not halve)"""
    opt.zero_grad(set_to_none=True)
    _forward_backward(net, x, gy, calls, scaler)
    before = scaler.get_scale()
    scaler.step(opt)
    scaler.update()
    return scaler.get_scale() >= before


@gpu
def test_grad_scaler_decisions_of_fused_and_stock(nets):
    """init_scale 2^40: the first step is skipped in both nets, the scale halves and no parameter bit moves.  Stepping on
    from there, both nets take their first step within one halving of each other, and the updates of that step agree.
    init_scale 2^10: the first step is taken."""
    a, b, x, gy, calls = nets
    p0 = {k: p.detach().clone() for k, p in a.named_parameters()}
    taken, updates = {}, {}
    for name, net in (("fused", a), ("stock", b)):
        opt, scaler = _opt(net), torch.amp.GradScaler("cuda", init_scale=2.0 ** 40)
        assert not _step(net, opt, scaler, x, gy, calls), name
        assert scaler.get_scale() == 2.0 ** 39
        for k, p in net.named_parameters():
            assert torch.equal(p, p0[k]), (name, k)
        for _ in range(40):
            scale = scaler.get_scale()
            if _step(net, opt, scaler, x, gy, calls):
                taken[name] = scale
                break
        assert name in taken, name
        updates[name] = {k: (p.detach() - p0[k]) for k, p in net.named_parameters()}
    assert abs(math.log2(taken["fused"]) - math.log2(taken["stock"])) <= 1, taken
    errs = {k: relerr(u, updates["stock"][k]) for k, u in updates["fused"].items()
            if updates["stock"][k].numel() > 0 and updates["stock"][k].abs().max() > 0}
    worst = max(errs.items(), key=lambda kv: kv[1])
    record("fp16_grad_scaler", ARCH, fused_first_scale=math.log2(taken["fused"]), stock_first_scale=math.log2(taken["stock"]),
           worst_update=worst[1])
    assert worst[1] < STEP_BAR, worst
    opt, scaler = _opt(a), torch.amp.GradScaler("cuda", init_scale=2.0 ** 10)
    assert _step(a, opt, scaler, x, gy, calls)


# --------------------------------------------------------------------------- (4) CPU: routing completeness, floors
def test_every_path_the_router_reaches_has_row_bars(monkeypatch):
    """CPU.  The (family, dtype, output type) combinations a call can reach, from the library's coverage test
    (vil_attn_wgmma_supported), the fp32 split rule of ops._split_flag and `impl`; each has a row variant with bars in
    test_gpu_attention_rows, test_gpu_f32_split or this file, so a new path cannot slip past the row checks."""
    ge.build()
    lib = _lib.load()
    codes = {F32: _lib.VIL_F32, F16: _lib.VIL_F16, BF16: _lib.VIL_BF16}
    reach = set()
    for dtype, code in codes.items():
        x = torch.empty(0, dtype=dtype)
        for prec in ("ieee", "tf32"):
            monkeypatch.setattr(torch.backends.cuda.matmul, "fp32_precision", prec)
            for impl in ("auto", "wgmma", "simt"):
                for f32out in (0, _lib.VIL_FLAG_F32_OUT):          # the parity build asks for fp32 outputs
                    flags = ops._split_flag(x, impl) | f32out
                    out = F32 if (f32out or dtype == F32) else dtype
                    for D in (32, 20):                              # D % 8 != 0: the wgmma family declines
                        p = tsa._params(D=D, dtype=code, flags=flags, impl=ops._IMPLS[impl])
                        wg = lib.vil_attn_wgmma_supported(ctypes.byref(p)) == 1
                        if impl != "simt" and wg:
                            reach.add(("wgmma", dtype, out, bool(flags & _lib.VIL_FLAG_F32_SPLIT)))
                        elif impl != "wgmma" and not f32out:        # SIMT refuses VIL_FLAG_F32_OUT
                            reach.add(("simt", dtype, dtype, False))
    variants = {(impl, dt, F32 if (f32o or dt == F32) else dt, False): n for n, (impl, dt, f32o, _) in
                list(tar.VARIANTS.items()) + list(VARIANTS.items())}
    variants[("wgmma", F32, F32, True)] = SPLIT
    bars = dict(tar.BARS, **BARS, **{SPLIT: tsplit.BARS})
    assert ("wgmma", F32, F32, False) not in reach                  # fp32 reaches wgmma only as split products
    assert {("wgmma", F16, F16, False), ("simt", F16, F16, False), ("simt", BF16, BF16, False)} <= reach
    missing = [c for c in reach if c not in variants or not all(k in bars[variants[c]] for k in ("row", "chunk", "lse"))]
    assert not missing, missing
    assert len(reach) == 8, sorted(map(str, reach))


def _dense_local(t, cfg, dtype, o_round=None):
    """fp64 dq of the local rows of vo.dense_attention (no global tokens), with delta formed from o rounded to o_round"""
    nx, ny, w, exact, mode, scale = cfg
    rd = lambda x: x.to(dtype).double()
    q, k, v, go = rd(t["q"]), rd(t["k"]), rd(t["v"]), rd(t["go"])
    E = vo.visit_weights(nx, ny, w, exact, mode, None, q.shape[1], dtype=torch.float64)
    kp, vp = vo._pad_keys(k, nx, ny, w), vo._pad_keys(v, nx, ny, w)
    s = scale * q @ kp.transpose(-1, -2) + torch.where(E > 0, torch.log(E.clamp_min(1e-300)), torch.full_like(E, float("-inf")))
    p = torch.softmax(s, dim=-1)
    o = p @ vp
    if o_round is not None:
        o = o.to(o_round).double()
    ds = p * (go @ vp.transpose(-1, -2) - (go * o).sum(-1, keepdim=True))
    return scale * ds @ kp


@pytest.mark.parametrize("variant", ["wgmma_fp16", "simt_fp16", "simt_bf16"])
def test_delta_floor_covers_the_stored_o_directly(variant):
    """CPU.  Under a peaked softmax (gap 12 through q k) the dq of delta formed from o rounded to the stored type,
    against the exact one, row by row in fp64: within one dq floor of `peak_floors` (its eps_o term).  The floor bounds
    |dO . (o_stored - o)| by eps_o ||dO|| ||o|| and ||o|| by max ||v||: the worst row measures about 1 % of it."""
    case = (1, 2, 16, 12, 12, 0, 4, 0, 0, False)
    dtype = VARIANTS[variant][1]
    t, _ = tar.peak_through_qk(tar.make_inputs(case, seed=530), case, dtype, 12, ("off", 0, 0, "same"))
    cfg = tar.cfg_of(case)
    exact = _dense_local(t, cfg, dtype)
    stored = _dense_local(t, cfg, dtype, o_round=dtype)
    floor = tar.peak_floors(t, cfg, variant, 0)["dq"]
    ratio = (stored - exact).norm(dim=-1) / floor
    record("fp16_floor_model", variant, delta_over_floor=float(ratio.max()))
    assert 0.0 < float(ratio.max()) <= 1.0


@pytest.mark.parametrize("g", [16, 65, 130])
@pytest.mark.parametrize("dtype", [F16, BF16], ids=["fp16", "bf16"])
def test_global_query_roundings_stay_under_their_allowance(dtype, g):
    """CPU.  A stored gradient row of a shared-weight global key collects one term per global query, rounded to the
    output type after each: simulated in fp64 for 4096 rows of D = 32, the worst row is within the allowance of the row
    check (3 out_eps sqrt(g), out_eps = 2^-12 in fp16, 2^-9 in bf16) and its rms is of the size out_eps sqrt(g)."""
    out_eps = 2.0 ** -12 if dtype == F16 else 2.0 ** -9
    gen = torch.Generator().manual_seed(531)
    terms = torch.randn(4096, g + 1, 32, generator=gen, dtype=torch.float64)
    acc = terms[:, 0].to(dtype).double()                      # the local part, stored first
    for a in range(1, g + 1):
        acc = (acc + terms[:, a]).to(dtype).double()
    exact = terms.sum(dim=1)
    e = (acc - exact).norm(dim=-1) / exact.norm(dim=-1)
    record("fp16_floor_model", "g%d_%s" % (g, dtype), worst=float(e.max()) / (out_eps * g ** 0.5),
           rms=float(e.pow(2).mean().sqrt()) / (out_eps * g ** 0.5))
    assert float(e.max()) < 3 * out_eps * g ** 0.5
    assert 0.2 < float(e.pow(2).mean().sqrt()) / (out_eps * g ** 0.5) < 1.5
