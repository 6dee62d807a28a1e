"""The attention kernels over the geometry domain the C ABI accepts, row by row.

The other attention files hold hand-picked geometries.  Tallied over their case lists, part of what `make_geo` accepts
(vil_attn_api.cu) is held by one whole-tensor norm at most, and part of it never runs:

* shift modes 1, 2, 4, 5, 6 and 7 on the SIMT family (fp32 training without TF32, and the fp16 / bf16 backward at
  D % 8 != 0 or on misaligned rows).  `mode > 0` draws one of them on every training forward, each sends its neighbour's
  pairs to its own quadrant of the (4w-1)^2 bias table and gives the neighbour its own dropout columns (oi w^2);
* cyclic chunks (exact = -1) with any mode but 0: the wrap of the neighbour and the pad cut, the rule that decides from
  the unwrapped offset whether the phantom zero keys of a padded chunk join the softmax (`Visit::cut` / `chunk_key` in
  vil_wgmma.cuh, the same rule in vil_simt.cuh), on a 1 x 1 chunk grid as well, where every offset lands on the query's
  own chunk;
* grids smaller than the window (nx < w or ny < w), one token wide, a single token: one padded chunk holds every key;
* windows 1, 2 and 3: `SlotWalk` steps 64 / w rows and 64 % w columns per piece, and the 3 x 3 to 11 x 11 bias table is
  nearly all edge;
* head dims below 8 (the SIMT HD 8 tile) and 12 (HD 16 with D % 8 != 0).

Each case is held at the bars of the file whose machinery it reuses, with no bar of its own:
  (a) every (exact, mode) pair the ABI accepts on a 4 x 3 chunk grid with padding, on every variant the router reaches,
      and cyclic chunks at every mode on 2 x 2 and 1 x 1 grids: test_gpu_attention_rows' rows, chunks and lse;
  (b) degenerate grids and windows at exact 0, 1 and -1, with and without global tokens, and head dims 4, 8 and 12;
  (c) the bias gradients entry by entry (test_gpu_bias_entries) at every mode and on the cyclic small grids;
  (d) dropout with the exact mask (test_gpu_dropout's keep tensors) at every mode and on a 1 x 1 cyclic grid;
  (e) the module's random-shift training path: B200Long2DSCSelfAttention(mode=1) with each draw pinned, against its
      fp64 oracle, at the module bars of test_gpu_parity;
  (f) CPU guards: the lattice is the ABI's, the wgmma cases are the wgmma family's, and no other file had these cases.
The variants of test_gpu_fp16 (SIMT fp16 / bf16, wgmma fp16) and test_gpu_f32_split (split fp32) come with their
fixtures, imported below.
"""
import ctypes
import random

import pytest
import torch

import __graft_entry__ as ge
from oracle import vil_oracle as vo
from oracle.vil_oracle import OracleLong2DSCSelfAttention
from tests import test_gpu_attention_rows as tar
from tests import test_gpu_batch_slices as tbs
from tests import test_gpu_bias_entries as tbe
from tests import test_gpu_deterministic as tdet
from tests import test_gpu_dropout as tdrop
from tests import test_gpu_f32_split as tsplit
from tests import test_gpu_fp16 as tfp16
from tests import test_gpu_parity as tpar
from tests import test_headdim128 as thd
from tests import test_simt_headdim128 as tshd
from tests import test_staging_alignment as tsa
from tests.test_gpu_f32_split import split_variant  # noqa: F401  (autouse: the split variant in the shared helpers)
from tests.test_gpu_fp16 import fp16_variants  # noqa: F401  (autouse: the fp16 / bf16 variants and their bars)
from tests.util import record, relerr
from vision_longformer_b200 import B200Long2DSCSelfAttention, _lib

gpu = pytest.mark.gpu
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
DEV = "cuda"
SPLIT = tsplit.V

# name: (family, dtype, VIL_FLAG_F32_OUT); known here at collection time, before the fixtures register the variants
VARIANTS = {n: v[:3] for n, v in list(tar.VARIANTS.items()) + list(tfp16.VARIANTS.items())}
VARIANTS[SPLIT] = ("wgmma", F32, False)
ALL = ["simt_fp32", "simt_bf16", "simt_fp16", "wgmma_bf16", "wgmma_bf16_linear", "wgmma_fp16", "wgmma_fp16_f32out",
       "wgmma_bf16_f32out", SPLIT]
NODROP = (0.0, 0, 0)


def run(t, cfg, variant, drop=NODROP):
    """one forward + backward through the C ABI on the family the variant names (asserted by the runners)"""
    return tfp16.run(t, cfg, variant, drop)


def expand(cases, names):
    """(case, variant) pairs; a wgmma variant only where D % 8 == 0 (the family declines the rest)"""
    return [pytest.param(c, n, id=tar.CASE_ID(c) + "-" + n) for c in cases for n in names
            if VARIANTS[n][0] == "simt" or c[2] % 8 == 0]


def stored_o_oracle(t, cfg, dtype, key):
    """test_gpu_attention_rows.oracle with delta = rowsum(dO * o) formed from o rounded to `dtype`, as the kernels form
    it from the o they stored (and the reference's own autograd in that dtype).  Its dS is P (dP - delta - c) with
    c = dO . (o_stored - o), which is the gradient of  sum dO . o - sum c lse  at fixed c.  The difference from the
    exact gradient is -scale c k_bar in a dq row (k_bar = sum_j P_ij k_j): with few keys, or a softmax that leaves dq
    small against ||dO|| ||o|| ||k_bar||, it is a large part of the row.  Four rows of this file exceed the bf16 row bar
    against the exact reference; this term predicts their errors, 1.9e-2, 7.3e-2, 4.5e-2 and 3.3e-2 (dqg), and the bf16
    outputs measured 1.9e-2 / 2.0e-2 (SIMT / wgmma), 7.2e-2, 4.5e-2 / 3.9e-2 and 3.3e-2 on an H100 SXM (700 W).
    This is the operator's contract, not one kernel's choice: the backward is a separate call that is given o in its
    stored type (include/vil_attn.h: delta = rowsum(dO * O) of the O passed in) and has no other o to form delta from."""
    if (key, dtype) in tar._REFS:
        return tar._REFS[(key, dtype)]
    rd = lambda x: x.to(dtype).double().requires_grad_(True)
    q, k, v, qg = rd(t["q"]), rd(t["k"]), rd(t["v"]), rd(t["qg"])
    g = k.shape[2] - q.shape[2]
    table, g2l, g2g = [None if t[n] is None else t[n].float().double().requires_grad_(True) for n in ("table", "g2l", "g2g")]
    o, og, lse, lse_g = tar._dense(q, k, v, qg if g else None, k, v, table, g2l, g2g, cfg)
    go, gog = t["go"].to(dtype).double(), t["gog"].to(dtype).double()
    c = (go * (o.detach().to(dtype).double() - o.detach())).sum(-1)
    loss = (o * go).sum() - (c * lse).sum()
    if g:
        cg = (gog * (og.detach().to(dtype).double() - og.detach())).sum(-1)
        loss = loss + (og * gog).sum() - (cg * lse_g).sum()
    ins = dict(q=q, k=k, v=v, **(dict(qg=qg) if g else {}))
    ins.update({n: x for n, x in (("table", table), ("g2l", g2l), ("g2g", g2g)) if x is not None})
    grads = torch.autograd.grad(loss, list(ins.values()))
    ref = dict(o=o.detach(), og=None if og is None else og.detach(), lse=lse.detach(),
               lse_g=None if lse_g is None else lse_g.detach(), **{"d" + n: x for n, x in zip(ins, grads)})
    tar._REFS[(key, dtype)] = ref
    return ref


# test_gpu_attention_rows.peak_floors as that file defines it, taken before any fixture replaces it: the split variant's
# fixture scales the floors of every variant by its FLOOR_SCALE, which belongs to the split variant alone (`floors_of`)
PEAK_FLOORS = tar.peak_floors


def floors_of(t, cfg, variant, g):
    """the saturated-softmax floors each variant takes in its home file: test_gpu_attention_rows' (with test_gpu_fp16's
    store floor for fp16 outputs), and those times FLOOR_SCALE for the split products of test_gpu_f32_split"""
    f = tfp16._peak_floors(PEAK_FLOORS)(t, cfg, variant, g)
    if variant == SPLIT:
        f = {n: x * tsplit.FLOOR_SCALE for n, x in f.items()}
    return f


def repeated_visits(case):
    """k: the most times one row visits one key (cyclic chunks on grids of one or two chunk rows or columns, where
    several offsets wrap onto the same chunk; 1 elsewhere)"""
    B, H, D, nx, ny, g, w, exact, mode = case[:9]
    return int(vo.visit_weights(nx, ny, w, exact, mode, None, 1).max())


def fewest_keys(case):
    """the fewest keys any local row's softmax takes (global keys included; a key of two visits counts once)"""
    B, H, D, nx, ny, g, w, exact, mode = case[:9]
    return g + int((vo.visit_weights(nx, ny, w, exact, mode, None, 1)[0] > 0).sum(dim=-1).min())


def rows_case(test, case, variant, seed, monkeypatch, entries=False):
    """test_gpu_attention_rows' measurements of one case on one variant, with four rules of that file's error model
    made explicit for the corners here:
    * an o stored in bf16 / fp16 is the o of delta (`stored_o_oracle`);
    * a row whose softmax takes at most 3 keys is a cancellation (sum_j dS_ij = 0 over 1 to 3 terms, exactly 0 for one
      key): the floors of a saturated softmax, `peak_floors`;
    * at w = 1 a chunk is one token: its block is held at the row bar;
    * a row that visits a key k times (`repeated_visits`) sums k identical copies of that key's terms, each with the
      same rounding: over n distinct keys the error of the sum grows as k sqrt(n) roundings, where n k independent terms
      give sqrt(k n).  The bars of the variants with fp32 outputs, whose per-term roundings (fp32 sums, the bf16 / fp16
      P operand, the split products) are what they measure, are taken sqrt(k) times; a stored bf16 / fp16 output adds one
      rounding per element, which is not repeated.  (Measured on an H100 SXM before this rule: 1.42 times the SIMT fp32
      chunk bar in dq of the 1 x 40 grid at w = 7 without global tokens, where k = 3.)
    entries: the bias gradients entry by entry (test_gpu_bias_entries) rather than by a whole-tensor norm, for the small
    grids whose d_g2l (2 H g entries) or table (9 entries at w = 1) make that norm one entry's error; by the norm where
    the entry bar would exceed the case's error ceiling (D = 4).
    The oracle of a case is kept for the variants that follow it and dropped after."""
    key = (test,) + case
    for k in [k for k in tar._REFS if k[0][0].startswith("lattice") and k[0][:len(key)] != key]:
        del tar._REFS[k]
    t = tar.make_inputs(case, seed=seed)
    cfg = tar.cfg_of(case)
    dtype = VARIANTS[variant][1]
    stored = tar.store_eps(variant)[0] > 2.0 ** -24
    ref = stored_o_oracle(t, cfg, dtype, key + ("stored",)) if stored else tar.oracle(t, cfg, dtype, key)
    B, H, D, nx, ny, g, w, exact, mode, rpe = case[:10]
    floors = floors_of(t, cfg, variant, g) if fewest_keys(case) <= 3 else None
    bars = dict(tsplit.BARS if variant == SPLIT else tar.BARS[variant])     # the split's check reads tsplit.BARS
    if w == 1:
        bars["chunk"] = bars["row"]
    k = repeated_visits(case)
    if k > 1 and not stored:
        r = k ** 0.5
        bars = dict(row=tuple(r * x for x in bars["row"]), chunk=tuple(r * x for x in bars["chunk"]), lse=r * bars["lse"])
    if variant == SPLIT:
        monkeypatch.setattr(tsplit, "BARS", bars)
    else:
        monkeypatch.setitem(tar.BARS, variant, bars)
    terms = tbe.terms_of((test,) + case, t, case[:9], dtype) if entries and rpe else None
    if terms is not None:      # the entry bar must stay under the case's error ceiling (not so at D = 4)
        nmax = max(float(terms[n][2].max()) for n in tbe.NAMES if n in terms)
        if tbe.bar_of(variant, terms["smax"]) > tbe.ceiling(variant, D, terms["smax"], nmax):
            terms = None
    out = run(t, cfg, variant)
    tar.check(test, "randn", out, ref, case, variant, floors=floors, bias=terms is None)
    if terms is not None:
        tbe.hold_entries(test, "randn", out, terms, case[:9], variant, whole=False)


# --------------------------------------------------------------------------- (a) the (exact, mode) lattice
def accepted_pairs():
    """every (exact, mode) for which the library's argument checks pass (make_geo), over a range wider than the rules"""
    ge.build()
    lib = _lib.load()
    return {(e, m) for e in range(-3, 4) for m in range(-3, 11)
            if lib.vil_attn_workspace_bytes(ctypes.byref(tsa._params(exact=e, mode=m)), 0) > 0}


# 4 x 3 chunks, 5 padding rows and 2 padding columns: the centre chunks see every neighbour, the edge chunks lose some
# (exact = 0) or wrap (exact = -1) onto a padded chunk; the bias table with the odd modes
LATTICE_PAIRS = [(e, m) for e in (0, -1) for m in range(-1, 9)] + [(1, 0)]
LATTICE = [(2, 2, 32, 23, 19, 2, 7, e, m, m % 2 == 1 or e == 1) for e, m in LATTICE_PAIRS]
# cyclic chunks at every mode on a 2 x 2 grid (two offsets reach one chunk) and on one padded chunk (all of them do)
CYCLIC_SMALL = [(1, 2, 16, nx, ny, 1, 4, -1, m, m % 2 == 1) for nx, ny in ((8, 5), (3, 3)) for m in range(-1, 9)]
CYCLIC_VARIANTS = ["simt_fp32", "wgmma_bf16_f32out", SPLIT]


@gpu
@pytest.mark.parametrize("case,variant", expand(LATTICE, ALL))
def test_rows_every_exact_and_mode(case, variant, monkeypatch):
    rows_case("lattice_rows", case, variant, seed=610, monkeypatch=monkeypatch)


@gpu
@pytest.mark.parametrize("case,variant", expand(CYCLIC_SMALL, CYCLIC_VARIANTS))
def test_rows_cyclic_chunks_on_small_grids(case, variant, monkeypatch):
    rows_case("lattice_cyclic_small_grids", case, variant, seed=611, monkeypatch=monkeypatch)


# --------------------------------------------------------------------------- (b) degenerate grids and windows
DEGENERATE_GRIDS = [
    # nx, ny, w
    (5, 3, 7), (6, 6, 7),            # smaller than the window: one padded chunk
    (1, 40, 7), (40, 1, 7),          # one token wide
    (1, 1, 7),                       # a single token
    (9, 30, 12),                     # three pieces per chunk, 9 real rows: the pieces below the image are skipped
    (7, 6, 1), (5, 7, 2), (8, 8, 3), (7, 10, 3),   # windows below 4
]
DEGENERATE = [(1, 2, 32, nx, ny, g, w, e, 0, g > 0) for nx, ny, w in DEGENERATE_GRIDS for e in (0, 1, -1) for g in (0, 2)]
# a random-shift draw on each grid, every mode once, with the wrap on half of them
DEGENERATE_MODES = [(1, 2, 32, nx, ny, 1, w, e, m, True) for (nx, ny, w), e, m in zip(
    DEGENERATE_GRIDS, (0, -1, -1, 0, -1, -1, 0, -1, 0, -1), (1, 4, 2, 5, 8, 6, 3, 7, 8, 1))]
# head dims below 16 no other file runs: D = 4 (the SIMT HD 8 tile) and D = 12 (HD 16, D % 8 != 0: SIMT only), D = 8
SMALL_HEADS = [
    (1, 2, 4, 5, 3, 1, 7, 0, 0, True), (1, 2, 4, 8, 8, 0, 3, -1, 4, True), (1, 2, 4, 23, 19, 2, 7, 0, 0, True),
    (1, 2, 12, 7, 10, 2, 3, 1, 0, True), (1, 2, 12, 1, 40, 1, 7, -1, 0, False), (1, 2, 12, 23, 19, 2, 7, -1, 6, True),
    (1, 2, 8, 5, 7, 1, 2, 1, 0, True), (1, 2, 8, 9, 30, 2, 12, -1, 0, True), (1, 2, 8, 23, 19, 2, 7, 0, 2, True),
]
DEGENERATE_VARIANTS = ["simt_fp32", "simt_bf16", "wgmma_bf16_f32out", "wgmma_fp16", SPLIT]


@gpu
@pytest.mark.parametrize("case,variant", expand(DEGENERATE + DEGENERATE_MODES, DEGENERATE_VARIANTS))
def test_rows_degenerate_grids_and_windows(case, variant, monkeypatch):
    rows_case("lattice_degenerate", case, variant, seed=612, monkeypatch=monkeypatch, entries=True)


@gpu
@pytest.mark.parametrize("case,variant", expand(SMALL_HEADS, ["simt_fp32", "simt_bf16", "simt_fp16",
                                                              "wgmma_bf16_f32out", "wgmma_bf16", SPLIT]))
def test_rows_small_head_dims(case, variant, monkeypatch):
    rows_case("lattice_small_head_dims", case, variant, seed=613, monkeypatch=monkeypatch, entries=True)


# --------------------------------------------------------------------------- (c) the bias gradients entry by entry
BIAS_CASES = (
    # B, H, D, nx, ny, g, w, exact, mode
    [(1, 2, 32, 23, 19, 2, 7, 0, m) for m in range(1, 9)] +
    [(1, 2, 32, 3, 3, 1, 4, -1, m) for m in range(-1, 9)] +                    # one padded chunk, cyclic
    [(1, 2, 32, 8, 5, 1, 4, -1, m) for m in (-1, 1, 3, 6, 8)] +                # 2 x 2 chunks, cyclic
    [(1, 2, 32, nx, ny, 1, w, e, 0) for nx, ny, w in ((7, 6, 1), (5, 7, 2), (8, 8, 3)) for e in (0, 1, -1)] +
    [(1, 2, 32, 7, 6, 1, 1, -1, 3), (1, 2, 32, 8, 8, 2, 3, 0, 6), (1, 2, 32, 5, 7, 0, 2, -1, 7)]
)
BIAS_VARIANTS = ["simt_fp32", "wgmma_bf16_f32out", "simt_bf16"]


@pytest.mark.parametrize("case", BIAS_CASES, ids=tbe.CASE_ID)
def test_restatement_matches_the_dense_oracle(case):
    """CPU: test_gpu_bias_entries' per-entry restatement against autograd of the dense oracle on each new geometry"""
    t = tar.make_inputs(tbe.full(case), seed=620)
    terms = tbe.bias_grad_terms(t, case, F32)
    tbe._pin(terms, tbe._autograd_bias(t, case, F32, vo.dense_attention))
    assert float(tbe.table_npairs(case).sum()) == float(vo.visit_weights(*case[3:5], case[6], case[7], case[8], None, 1).sum())


@gpu
@pytest.mark.parametrize("case,variant", [pytest.param(c, v, id=tbe.CASE_ID(c) + "-" + v)
                                          for c in BIAS_CASES for v in BIAS_VARIANTS])
def test_bias_entries(case, variant):
    t = tar.make_inputs(tbe.full(case), seed=621)
    terms = tbe.terms_of(("lattice",) + case, t, case, VARIANTS[variant][1])
    out = run(t, tar.cfg_of(tbe.full(case)), variant)
    tbe.hold_entries("lattice_bias_entries", "randn", out, terms, case, variant)


# --------------------------------------------------------------------------- (d) dropout with the exact mask
DROP_CASES = [(1, 2, 32, 23, 19, 2, 7, 0, m, m % 2 == 1) for m in range(1, 9)] + \
    [(1, 2, 16, 3, 3, 1, 4, -1, m, True) for m in (1, 5, 8)]   # one chunk: its own chunk is two columns with two draws
DROP_VARIANTS = ["simt_fp32", "wgmma_bf16_f32out", SPLIT]


@gpu
@pytest.mark.parametrize("case,variant", expand(DROP_CASES, DROP_VARIANTS))
def test_rows_dropout_with_the_exact_mask(case, variant):
    t = tar.make_inputs(case, seed=630)
    ref = tar.dropout_reference(t, case, VARIANTS[variant][1])
    tar.check("lattice_rows_dropout", "p0.1", run(t, tar.cfg_of(case), variant, drop=tar.DROP), ref, case, variant)


# --------------------------------------------------------------------------- (e) the module's random-shift path
MODULE_KW = dict(dim=32, num_heads=2, qkv_bias=True, w=4, nglo=1, rpe=True, sharew=True, mode=1)
MODULE_NX, MODULE_NY = 10, 9          # 3 x 3 chunks with padding: every neighbour exists for the centre chunk
# test_gpu_parity: the module against the golden vectors in fp32 (y, dx, parameter gradients), in low precision (y, dx)
# and the weight / bias-table gradients of the dense attention on the operator kernels in bf16
MODULE_BARS = {"fp32": dict(y=1e-5, dx=2e-5, param=5e-5, bias=5e-5), "bf16": dict(y=3e-2, dx=6e-2, param=6e-2, bias=0.1)}


@pytest.fixture
def ieee_matmul():
    """fp32 matmuls without TF32: fp32 attention on the SIMT family, fp32 Linears in full precision"""
    before = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    yield
    torch.backends.cuda.matmul.fp32_precision = before


@gpu
@pytest.mark.parametrize("pick", range(1, 9))
@pytest.mark.parametrize("exact", [0, -1])
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_module_random_shift_training(prec, exact, pick, monkeypatch, ieee_matmul):
    """B200Long2DSCSelfAttention(mode=1) in train(): the draw random.randrange(1, 9) pinned to `pick`, as
    oracle/make_golden.py pins the reference's; output and every parameter gradient against the fp64 oracle run at that
    mode, in fp32 (SIMT) and under bf16 autocast (wgmma)"""
    torch.manual_seed(640 + pick)
    ref = OracleLong2DSCSelfAttention(exact=exact, **MODULE_KW).double().train()
    with torch.no_grad():
        for n, p in ref.named_parameters():
            if "relative_position" in n:
                p.normal_(0.0, 0.5)
    x = torch.randn(2, 1 + MODULE_NX * MODULE_NY, MODULE_KW["dim"], dtype=torch.float64, requires_grad=True)
    y_ref = ref(x, MODULE_NX, MODULE_NY, mode_override=pick)
    gy = torch.randn_like(y_ref)
    (y_ref * gy).sum().backward()
    mod = B200Long2DSCSelfAttention(exact=exact, **MODULE_KW).to(DEV)
    mod.load_state_dict(ref.state_dict())
    mod.train()
    draws = []
    monkeypatch.setattr(random, "randrange", lambda *a: draws.append(a) or pick)
    xg = x.detach().float().to(DEV).requires_grad_(True)
    with torch.autocast("cuda", dtype=BF16, enabled=prec == "bf16"):
        y = mod(xg, MODULE_NX, MODULE_NY)
    fam = _lib.last_impl()
    (y.float() * gy.float().to(DEV)).sum().backward()
    torch.cuda.synchronize()
    assert draws == [(1, 9)], draws
    assert fam == ("simt" if prec == "fp32" else "wgmma"), fam
    bars = MODULE_BARS[prec]
    errs = dict(y=relerr(y, y_ref), dx=relerr(xg.grad, x.grad))
    gref = dict(ref.named_parameters())
    for n, p in mod.named_parameters():
        errs["d" + n] = relerr(p.grad, gref[n].grad)
    record("lattice_module_random_shift", "e%d_pick%d/%s" % (exact, pick, prec), **errs)
    bar = lambda n: bars[n] if n in ("y", "dx") else bars["bias" if "relative_position" in n else "param"]
    bad = {n: e for n, e in errs.items() if not e < bar(n)}
    assert not bad, bad


# --------------------------------------------------------------------------- (f) CPU guards
def params_of(case, variant):
    """the C ABI's parameters of one case and variant, as the runners pass them (contiguous rows of D elements; the
    coverage query never dereferences a pointer)"""
    B, H, D, nx, ny, g, w, exact, mode, rpe = case[:10]
    fam, dtype, f32out = VARIANTS[variant]
    code = {F32: _lib.VIL_F32, F16: _lib.VIL_F16, BF16: _lib.VIL_BF16}[dtype]
    flags = (_lib.VIL_FLAG_F32_OUT if f32out else 0) | (_lib.VIL_FLAG_F32_SPLIT if variant == SPLIT else 0)
    tab = 256 if rpe else None
    p = tsa._params(D=D, st=D, dtype=code, flags=flags, B=B, H=H, nx=nx, ny=ny, w=w, nglo=g, exact=exact, mode=mode,
                    bias_table=tab, g2l=tab if g else None, g2g=tab if g else None)
    for name in ("q", "k", "v"):
        getattr(p, name).sh = (g + nx * ny) * D
    return p


GPU_ROW_PARAMS = (expand(LATTICE, ALL) + expand(CYCLIC_SMALL, CYCLIC_VARIANTS) +
                  expand(DEGENERATE + DEGENERATE_MODES, DEGENERATE_VARIANTS) +
                  expand(SMALL_HEADS, ["simt_fp32", "simt_bf16", "simt_fp16", "wgmma_bf16_f32out", "wgmma_bf16", SPLIT]) +
                  expand(DROP_CASES, DROP_VARIANTS))


def test_lattice_is_every_pair_the_abi_accepts():
    """the (exact, mode) pairs of (a) are the ones make_geo accepts, enumerated from the library's own checks, and each
    runs on every variant the router reaches (test_gpu_fp16's routing test lists the same eight paths, plus split fp32)"""
    acc = accepted_pairs()
    assert acc == set(LATTICE_PAIRS) and len(acc) == 21, sorted(acc)
    ran = {}
    for p in expand(LATTICE, ALL):
        case, variant = p.values
        ran.setdefault((case[7], case[8]), set()).add(variant)
    assert set(ran) == acc
    assert all(v == set(ALL) for v in ran.values())
    assert set(ALL) == set(VARIANTS) - {"wgmma_fp16_linear"}
    for nx, ny in ((8, 5), (3, 3)):
        assert {c[8] for c in CYCLIC_SMALL if c[3:5] == (nx, ny)} == {m for e, m in acc if e == -1}
        assert vo.geometry(nx, ny, 4)[2:] == ((2, 2) if nx == 8 else (1, 1))


def test_lattice_geometry_has_interior_and_edge_chunks():
    B, H, D, nx, ny, g, w = LATTICE[0][:7]
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    assert mx >= 3 and my >= 3 and padx > 0 and pady > 0


def test_wgmma_cases_run_where_the_family_covers_them():
    """Through vil_attn_wgmma_supported (no kernel launched): every case a wgmma variant runs is covered by that family,
    so the runners' family assertion holds for the reason the case names; the SIMT variants run with impl="simt", and
    the head dims off 8 are the cases impl="auto" sends to SIMT"""
    ge.build()
    lib = _lib.load()
    for p in GPU_ROW_PARAMS + [pytest.param(c, v) for c in BIAS_CASES for v in BIAS_VARIANTS]:
        case, variant = p.values
        case = tbe.full(case) if len(case) == 9 else case
        ok = lib.vil_attn_wgmma_supported(ctypes.byref(params_of(case, variant)))
        if VARIANTS[variant][0] == "wgmma":
            assert ok == 1, (case, variant, _lib.last_error())
        else:
            assert tar.VARIANTS[variant][0] == "simt"             # the runners pass impl="simt"
            if case[2] % 8:
                assert ok == 0, (case, variant)
    assert {c[2] for c in SMALL_HEADS} == {4, 8, 12}


def other_cases():
    """(cases that run on the SIMT family, every case) of the other attention files' case lists: op level, rows, bias
    entries, dropout, batch slices, determinism, head dim 128, fp16 and split fp32"""
    simt = (tpar.OP_CASES + tar.GEOMETRY_CASES + tar.MASKED_CASES + tar.MANY_GLOBAL_CASES +
            [tar.PK_MODE0, tar.PK_W12, tar.PK_MODE3, tar.PK_CYCLIC, tar.PK_GLOBAL, tar.PK_GLOBAL2, tar.PK_TABLE] +
            tbe.ALL_CASES + tbe.PIN_CASES + tbe.CONTRACT_CASES + tdrop.DROP_CASES + tfp16.DROP_CASES +
            [tfp16.ROUTE_CASE, tfp16.SCALE_CASE] + tsplit.DROP_CASES + [tsplit.SLICE_CASE] + tbs.CASES +
            [tbs.S1_B13, tbs.S1_B64] + tdet.CASES + tshd.ROW_CASES + [tshd.PK_QK, tshd.PK_TABLE] + tshd.ENTRY_CASES +
            tshd.LARGE_CASES + tshd.DROP_CASES)
    wgmma = tpar.TC_CASES + tpar.MODE_CASES + tpar.TC_BIG_CASES + tpar.F32OUT_CASES + thd.CASES + thd.DROP_CASES
    return simt, simt + wgmma


def test_no_other_case_list_has_these_geometries():
    """The gap this file closes.  Before it, no case list of the attention files ran the SIMT family at modes 1, 2, 4,
    5, 6 or 7, cyclic chunks with a mode other than 0, a grid narrower than its window, a window below 4 or a head dim
    below 8 (the golden module vectors run two pinned draws, modes 3 and 6, end to end at one norm).  Each is here."""
    simt, every = other_cases()
    assert len(every) > 150
    rare = {1, 2, 4, 5, 6, 7}
    assert not [c for c in simt if c[8] in rare]
    assert not [c for c in every if c[7] == -1 and c[8] != 0]
    assert not [c for c in every if c[3] < c[6] or c[4] < c[6]]
    assert not [c for c in every if c[6] < 4]
    assert not [c for c in every if c[2] < 8]
    mine = [p.values for p in GPU_ROW_PARAMS]
    assert {c[8] for c, v in mine if VARIANTS[v][0] == "simt"} >= rare
    assert {c[8] for c, v in mine if c[7] == -1} == set(range(-1, 9))
    assert any(c[3] < c[6] and c[4] < c[6] for c, v in mine) and any(min(c[3], c[4]) == 1 for c, v in mine)
    assert {c[6] for c, v in mine} >= {1, 2, 3}
    assert {c[2] for c, v in mine if VARIANTS[v][0] == "simt"} >= {4, 12}
    assert {c[2] for c, v in mine if VARIANTS[v][0] == "wgmma"} >= {8}


def test_bias_cases_cover_every_mode_and_the_small_windows():
    modes = {c[8] for c in BIAS_CASES}
    assert modes == set(range(-1, 9))
    assert {c[8] for c in BIAS_CASES if c[7] == -1 and c[3:5] == (3, 3)} == set(range(-1, 9))
    assert {c[6] for c in BIAS_CASES} >= {1, 2, 3}
    for case in BIAS_CASES:       # the entry bars stay under their error ceilings here as well
        nmax = max(float(case[0] * tbe.table_npairs(case).max()), float(case[0] * case[3] * case[4]) if case[5] else 0.0)
        for v in ("simt_fp32", "wgmma_bf16_f32out"):
            assert tbe.bar_of(v, 0.0) <= tbe.ceiling(v, case[2], 0.0, nmax), (case, v)


def test_dropout_cases_cover_every_mode_and_a_one_chunk_cyclic_grid():
    assert {c[8] for c in DROP_CASES} == set(range(1, 9))
    one = [c for c in DROP_CASES if c[7] == -1 and vo.geometry(c[3], c[4], c[6])[2:] == (1, 1)]
    assert one and all(c[8] > 0 for c in one)
    # there, both offsets of a mode are the query's own chunk: two columns of attn1 with two draws per pair
    c = one[0]
    keep, _ = tdrop.keep_tensors(tar.DROP[1], tar.DROP[2], tar.DROP[0], c[0], c[1], c[3], c[4], c[6], c[5], c[8])
    w2 = c[6] ** 2
    assert keep.shape[-1] == c[5] + 2 * w2
    assert not torch.equal(keep[..., c[5]:c[5] + w2], keep[..., c[5] + w2:])


def test_floors_are_the_home_files():
    """the few-key floors: test_gpu_attention_rows' peak_floors for every variant but the split one, which alone takes
    test_gpu_f32_split's FLOOR_SCALE (the split fixture active here scales the floors of every variant)"""
    case = (1, 2, 32, 1, 1, 2, 7, 0, 0, True)
    t = tar.make_inputs(case, seed=612)
    cfg = tar.cfg_of(case)
    home = PEAK_FLOORS(t, cfg, "simt_fp32", 2)
    for v in ("simt_fp32", "simt_bf16", "wgmma_bf16", "wgmma_bf16_f32out"):
        want = PEAK_FLOORS(t, cfg, v, 2)
        got = floors_of(t, cfg, v, 2)
        assert got.keys() == want.keys() and all(torch.equal(torch.as_tensor(got[n]), torch.as_tensor(want[n])) for n in want), v
    split = floors_of(t, cfg, SPLIT, 2)
    assert all(torch.equal(torch.as_tensor(split[n]), torch.as_tensor(home[n] * tsplit.FLOOR_SCALE)) for n in home)
    fp16, pf = floors_of(t, cfg, "wgmma_fp16", 2), PEAK_FLOORS(t, cfg, "wgmma_fp16", 2)     # plus the fp16 store floor
    assert all(bool((torch.as_tensor(fp16[n]) > torch.as_tensor(pf[n])).all()) for n in pf)


def test_repeated_visits_of_the_cases():
    """k = 1 off the cyclic small grids; 3 on one-chunk-row grids, 4 on 2 x 2 and 9 on 1 x 1 grids"""
    assert {repeated_visits(c) for c in LATTICE} == {1}
    assert repeated_visits((1, 2, 32, 1, 40, 0, 7, -1, 0, False)) == 3
    assert repeated_visits((1, 2, 32, 9, 30, 0, 12, -1, 0, False)) == 3
    assert repeated_visits((1, 2, 16, 8, 5, 1, 4, -1, 0, False)) == 4
    assert repeated_visits((1, 2, 16, 3, 3, 1, 4, -1, 0, False)) == 9
    assert repeated_visits((1, 2, 16, 3, 3, 1, 4, -1, 8, False)) == 2
    assert repeated_visits((1, 2, 32, 1, 40, 0, 7, 0, 0, False)) == 1
