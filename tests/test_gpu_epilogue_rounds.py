"""The residual / LayerNorm / bias epilogue kernels (vil_addnorm_*, vil_layernorm_*, vil_bias_act_*) past their first
grid-stride round, at every instantiation and on the lane-masking edges of every dispatch bucket, against fp64 references
computed on the device.

The forward launchers cap their grids (addnorm: 2112 CTAs x 4 warps x 32 / L rows; LayerNorm: 1056 CTAs x 8 rows; bias_act:
1056 CTAs x 1024 vectors), so on a long stream every warp carries state from one round to the next: the DropPath sample
of its row (`sq` / `srem`), the column group of its vector (`cg`), the dead rows of a short last round.  The CPU tests
restate the launch geometry, check it against the library's workspace queries and assert that the GPU cases below reach
those rounds; they also check that misaligned pointers are refused before anything is launched.

Bars: the whole-tensor norm ratios of tests/test_gpu_epilogue.py, plus localized ones, so that an error confined to one
round, one sample or one column slab is not diluted by the rest of the tensor: the worst row (the worst sample where a
rowscale is involved), the worst column of a column sum normalised by that column's sum of |terms|, and for bf16 / fp16
outputs the worst element in ulps of the output type (plus a small absolute floor for values next to 0)."""
import ctypes
import math
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

import __graft_entry__ as ge
from tests.util import record, relerr
from vision_longformer_b200 import B200LayerNorm, _lib, epilogue
from vision_longformer_b200.msvit import DropPath, build_vil

DEV = "cuda"
EPS = 1e-6
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
NAME = {F32: "f32", BF16: "bf16", F16: "f16"}
TINY = 1e-300

# ------------------------------------------------------------------------------------------------ launch geometry (restated)
SMS = 132                                   # grids are sized in multiples of the 132 SMs of an H100 SXM
AN_WARPS, LN_WARPS, BA_THREADS = 4, 8, 256


def cdiv(a, b):
    return -(-a // b)


def an_lanes(C):
    """addnorm: (L lanes per row, NVL 16-byte vectors per lane) of the instantiation that serves C channels."""
    for cmax, L, nvl in ((48, 4, 3), (96, 8, 3), (192, 16, 3), (384, 32, 3), (512, 32, 4), (768, 32, 6), (1024, 32, 8)):
        if C <= cmax:
            return L, nvl
    raise ValueError(C)


def an_rpw(C):
    return 32 // an_lanes(C)[0]


def an_fwd_grid(rows, C):
    return min(cdiv(cdiv(rows, an_rpw(C)), AN_WARPS), SMS * 16)


def an_fwd_round(rows, C):
    """rows one grid-stride round of addnorm_fwd covers"""
    return an_fwd_grid(rows, C) * AN_WARPS * an_rpw(C)


def an_bwd_grid(rows):
    return min(max(rows // (AN_WARPS * 32), SMS * 2), SMS * 12)


def ln_npl(C):
    """LayerNorm (scalar path): the NPL bucket (channels per lane) of the instantiation that serves C channels."""
    npl = cdiv(C, 32)
    return next(b for b in (3, 6, 12, 24, 32) if npl <= b)


def ln_fwd_grid(rows):
    return min(cdiv(rows, LN_WARPS), SMS * 8)


def ln_bwd_grid(rows):
    return min(max(rows // (LN_WARPS * 16), SMS), SMS * 8)


def ba_n(dtype):
    return 4 if dtype == F32 else 8                     # elements per 16-byte vector


def ba_fwd_grid(rows, C, dtype):
    return min(cdiv(rows * (C // ba_n(dtype)), BA_THREADS * 4), SMS * 8)


def ba_fwd_rounds(rows, C, dtype):
    return cdiv(rows * (C // ba_n(dtype)), ba_fwd_grid(rows, C, dtype) * BA_THREADS * 4)


def ba_plan(rows, C, dtype):
    """bias_act backward: column slabs ncs of gs 16-byte groups, rpi row lanes per CTA, nrs row slabs of `per` rows."""
    G = C // ba_n(dtype)
    ncs = cdiv(G, BA_THREADS)
    gs = cdiv(G, ncs)
    rpi = BA_THREADS // gs
    per = max(cdiv(rows, (SMS * 8) // ncs), 4 * rpi)
    return SimpleNamespace(G=G, ncs=ncs, gs=gs, rpi=rpi, per=per, nrs=max(cdiv(rows, per), 1))


# ------------------------------------------------------------------------------------------------ cases
AN_PAIRS = [(F32, F32), (BF16, BF16), (F16, F16), (BF16, F32), (F16, F32), (F32, BF16), (F32, F16)]   # (br / dbr, y / dy)
AN_BUCKET_C = [44, 52, 100, 196, 388, 516, 772]          # one C just past each dispatch boundary, per (L, NVL)
AN_SWEEP_C = [4, 44, 48, 52, 92, 96, 100, 188, 192, 196, 380, 384, 388, 508, 512, 516, 764, 768, 772, 1020, 1024]
# which optional operands a case passes: branch, bias, DropPath rowscale, residual-stream gradient, branch gradient
AN_OPTS = {"full": ("br", "bias", "scale", "gres", "dbr"), "nobias": ("br", "scale", "gres", "dbr"),
           "noscale_nogres": ("br", "bias", "dbr"), "nodbr": ("br", "bias", "scale", "gres"), "norm_only": ("gres",)}
RPS_KINDS = ["1", "3", "rpw-1", "517", "3137", "round-1", "round+1", "gt_rows"]


def _rps(kind, rows, C):
    return {"1": 1, "3": 3, "rpw-1": max(an_rpw(C) - 1, 1), "517": 517, "3137": 3137,
            "round-1": an_fwd_round(rows, C) - 1, "round+1": an_fwd_round(rows, C) + 1, "gt_rows": rows + 5}[kind]


def _an_cases():
    cases = []
    # three forward rounds (two full ones and a 3-row tail) at every (L, NVL) x dtype pair, every operand present
    for i, (pair, C) in enumerate((p, c) for p in AN_PAIRS for c in AN_BUCKET_C):
        rows = 2 * (SMS * 16 * AN_WARPS * an_rpw(C)) + 3
        kind = RPS_KINDS[i % len(RPS_KINDS)]
        cases.append(SimpleNamespace(pair=pair, C=C, rows=rows, rps=_rps(kind, rows, C), rps_kind=kind, opts="full"))
    # the C sweep over every bucket edge: small streams, every operand combination in turn
    names = list(AN_OPTS)
    for i, (pair, C) in enumerate((p, c) for p in AN_PAIRS for c in AN_SWEEP_C):
        rows = 997 + 8 * (i % 3)
        kind = ("1", "3", "517", "gt_rows")[i % 4]
        cases.append(SimpleNamespace(pair=pair, C=C, rows=rows, rps=_rps(kind, rows, C), rps_kind=kind, opts=names[i % len(names)]))
    return cases


AN_CASES = _an_cases()


def _an_id(c):
    return f"{NAME[c.pair[0]]}-{NAME[c.pair[1]]}-C{c.C}-r{c.rows}-rps{c.rps_kind}-{c.opts}"


def _an_kernel_pairs(c):
    """(TB, TY) instantiations the forward and the backward of a case run (vil_epilogue.cu an_run)."""
    opts = AN_OPTS[c.opts]
    tb, ty = c.pair
    return ((tb if "br" in opts else ty, ty), (tb if "dbr" in opts else ty, ty))


LN_PAIRS = [(F32, F32), (F32, BF16), (F32, F16), (BF16, BF16), (F16, F16), (BF16, F32), (F16, F32)]   # (x, y)
LN_SWEEP_C = [1, 33, 96, 97, 98, 192, 193, 384, 385, 768, 769, 1023, 1024]
LN_BUCKET_C = [33, 97, 193, 385, 769]                    # one per NPL bucket; C % 4 != 0: fp32 input takes the scalar path


def _ln_cases():
    cases = [SimpleNamespace(xdt=xdt, ydt=ydt, C=C, rows=2 * SMS * 8 * LN_WARPS + 5) for xdt, ydt in LN_PAIRS for C in LN_BUCKET_C]
    cases += [SimpleNamespace(xdt=xdt, ydt=ydt, C=C, rows=301) for xdt, ydt in LN_PAIRS for C in LN_SWEEP_C]
    return cases


LN_CASES = _ln_cases()


def _ln_vec(c):
    """fp32 input with C % 4 == 0 runs the vectorised addnorm kernels (br = NULL), everything else vil_layernorm_*"""
    return c.xdt == F32 and c.C % 4 == 0


def _ba_cases():
    cases = []
    for dt in (F32, BF16, F16):
        for act in ("gelu", "none"):
            C = 1028 if dt == F32 else 2056                  # 257 column groups: two slabs, the second one short
            cases.append(SimpleNamespace(dt=dt, act=act, C=C, rows=9000))
            for C in ((4, 8, 200, 1028, 2056, 3072) if dt == F32 else (8, 200, 2056, 3072)):
                cases.append(SimpleNamespace(dt=dt, act=act, C=C, rows=3001))
    return cases


BA_CASES = _ba_cases()

# ------------------------------------------------------------------------------------------------ CPU: geometry and coverage


@pytest.fixture(scope="module")
def lib():
    ge.build()
    return _lib.load()


def _an_params(rows, C):
    p = _lib.VilAddNormParams()
    p.struct_bytes, p.C, p.rows = ctypes.sizeof(_lib.VilAddNormParams), C, rows
    return p


def test_backward_grids_match_their_documented_formulas(lib):
    """The backward grids, read back from the workspace queries (one partial row of 3 / 2 / 1 x C floats per CTA or row
    slab, plus 256 bytes), equal the formulas the round counts below are computed with."""
    for rows in (1, 997, 33791, 33792, 50000, 202751, 202752, 270339, 10 ** 6):
        for C in (4, 96, 772, 1024):
            ws = lib.vil_addnorm_workspace_bytes(ctypes.byref(_an_params(rows, C)))
            assert (ws - 256) % (12 * C) == 0 and (ws - 256) // (12 * C) == an_bwd_grid(rows), (rows, C)
            p = _lib.VilLayerNormParams()
            p.struct_bytes, p.C, p.rows = ctypes.sizeof(_lib.VilLayerNormParams), C, rows
            ws = lib.vil_layernorm_workspace_bytes(ctypes.byref(p))
            assert (ws - 256) % (8 * C) == 0 and (ws - 256) // (8 * C) == ln_bwd_grid(rows), (rows, C)
    for c in BA_CASES + [SimpleNamespace(dt=BF16, C=384, rows=r) for r in (1, 100, 5000, 10 ** 6)]:
        p = _lib.VilBiasActParams()
        p.struct_bytes, p.dtype, p.C, p.act, p.rows = ctypes.sizeof(_lib.VilBiasActParams), epilogue._DT[c.dt], c.C, 0, c.rows
        ws = lib.vil_bias_act_workspace_bytes(ctypes.byref(p))
        assert (ws - 256) % (4 * c.C) == 0 and (ws - 256) // (4 * c.C) == ba_plan(c.rows, c.C, c.dt).nrs, (c.dt, c.C, c.rows)


def test_cases_reach_every_round_bucket_and_dtype_pair():
    """Taken together, the GPU cases run >= 3 grid-stride rounds of every kernel at every (L, NVL) / NPL bucket and dtype
    pair, end on short last rounds, and sweep every dispatch edge.  Re-sizing a grid so that a case drops back to one
    round fails here."""
    buckets = {an_lanes(C) for C in range(4, 1025, 4)}
    assert len(buckets) == 7 and {an_lanes(C) for C in AN_BUCKET_C} == buckets
    multi_fwd, multi_bwd, short_round, short_rpw, swept = set(), set(), False, False, set()
    for c in AN_CASES:
        fwd_pair, bwd_pair = _an_kernel_pairs(c)
        swept.add((an_lanes(c.C), fwd_pair, c.C))
        rnd = an_fwd_round(c.rows, c.C)
        if cdiv(c.rows, rnd) >= 3:
            multi_fwd.add((an_lanes(c.C), fwd_pair))
            short_round |= c.rows % rnd != 0
            short_rpw |= c.rows % an_rpw(c.C) != 0
        if cdiv(c.rows, an_bwd_grid(c.rows) * AN_WARPS * an_rpw(c.C)) >= 3:
            multi_bwd.add((an_lanes(c.C), bwd_pair))
    every = {(b, p) for b in buckets for p in AN_PAIRS}
    assert multi_fwd == every and multi_bwd == every
    assert short_round and short_rpw
    assert {C for _, _, C in swept} == set(AN_SWEEP_C) and {(b, p) for b, p, _ in swept} == every
    assert {k for c in AN_CASES if "scale" in AN_OPTS[c.opts] for k in [c.rps_kind]} == set(RPS_KINDS)
    assert all(set(AN_OPTS[c.opts]) >= {"br", "scale"} for c in AN_CASES if c.rps_kind in ("round-1", "round+1"))

    ln_multi = {(ln_npl(c.C), c.xdt, c.ydt) for c in LN_CASES if not _ln_vec(c)
                and cdiv(c.rows, ln_fwd_grid(c.rows) * LN_WARPS) >= 3 and cdiv(c.rows, ln_bwd_grid(c.rows) * LN_WARPS) >= 3
                and c.rows % (ln_fwd_grid(c.rows) * LN_WARPS) != 0}
    assert ln_multi == {(b, x, y) for b in (3, 6, 12, 24, 32) for x, y in LN_PAIRS}
    edges = {96, 97, 192, 193, 384, 385, 768, 769, 1024}
    assert all(any(c.C == C and c.xdt == x and c.ydt == y for c in LN_CASES) for C in edges for x, y in LN_PAIRS)
    assert {c.C for c in LN_CASES if c.xdt == F32 and not _ln_vec(c)} >= {1, 33, 97, 98, 1023}

    for dt in (F32, BF16, F16):
        for act in ("gelu", "none"):
            mine = [c for c in BA_CASES if c.dt == dt and c.act == act]
            assert any(ba_fwd_rounds(c.rows, c.C, dt) >= 3 and (c.rows * (c.C // ba_n(dt))) % (SMS * 8 * BA_THREADS * 4) != 0
                       for c in mine)
            # more than one column slab with a short last one, on a stream with >= 3 row slabs of >= 3 rows per row lane
            assert any((lambda b: b.ncs > 1 and b.G % b.gs != 0 and b.nrs >= 3 and cdiv(b.per, b.rpi) >= 3)(ba_plan(c.rows, c.C, dt))
                       for c in mine)
            # a row slab reduced over several row lanes (the CTA reduction of bias_act_bwd)
            assert any(ba_plan(c.rows, c.C, dt).rpi >= 2 for c in mine)
            # the column group of a vector moves between outer iterations of bias_act_fwd (4 x stride mod G != 0)
            assert any(ba_fwd_rounds(c.rows, c.C, dt) >= 3
                       and (4 * ba_fwd_grid(c.rows, c.C, dt) * BA_THREADS) % (c.C // ba_n(dt)) != 0 for c in mine)
    assert {c.C for c in BA_CASES if c.dt == F32} >= {4, 1028} and {c.C for c in BA_CASES} >= {8, 200, 2056, 3072}


FAKE = 1 << 20                     # a 16-byte-aligned address that is never dereferenced: every call below is refused


def test_misaligned_pointers_are_refused_before_any_launch(lib):
    """addnorm: any non-NULL pointer off a 16-byte boundary is refused with VIL_E_BADARG, before the NULL-tensor and
    workspace checks.  `mean` (forward) / `workspace` (backward) stay NULL, so even a library without the alignment check
    stops at those checks and never launches on the fake pointers."""
    n0 = _lib.launch_count()
    fwd = ("x", "br", "bias", "rowscale", "gamma", "beta", "xo", "y", "rstd")
    bwd = ("x", "gamma", "beta", "rowscale", "mean", "rstd", "dy", "gres", "dx", "dbr", "dgamma", "dbeta", "dbias")
    for names, fn, held_back in ((fwd, lib.vil_addnorm_fwd_sm100, "mean"), (bwd, lib.vil_addnorm_bwd_sm100, "workspace")):
        for bad in (None,) + names:
            p = _an_params(1000, 96)
            p.b_dtype, p.y_dtype, p.rows_per_sample, p.eps = _lib.VIL_BF16, _lib.VIL_BF16, 10, 1e-6
            for k in names:
                setattr(p, k, FAKE + (4 if k == bad else 0))
            p.workspace_bytes = 1 << 30
            rc = fn(ctypes.byref(p), None)
            if bad is None:                                    # all aligned: stops at the NULL mean / workspace
                assert rc in (_lib.VIL_E_BADARG, _lib.VIL_E_WORKSPACE) and "aligned" not in _lib.last_error(), held_back
            else:
                assert rc == _lib.VIL_E_BADARG and "aligned" in _lib.last_error(), (held_back, bad, _lib.last_error())
    assert _lib.launch_count() == n0


def test_add_norm_rowscale_must_have_one_entry_per_sample(monkeypatch):
    """`add_norm` indexes rowscale by x[b]: rows_per_sample is the product of the dims between batch and channels (4-D
    streams included), and a rowscale of any other length than x.shape[0] is refused before anything runs."""
    seen = []
    monkeypatch.setattr(epilogue._AddNorm, "apply", lambda *a: seen.append(a[-1]))
    ln = torch.nn.LayerNorm(8)
    for shape, rps in (((2, 5, 8), 5), ((2, 3, 4, 8), 12), ((6, 8), 1), ((2, 1, 7, 3, 8), 21)):
        x = torch.zeros(shape)
        epilogue.add_norm(x, x, None, torch.ones(shape[0]), ln, out_dtype=torch.float32)
        assert seen.pop() == rps, shape
    with pytest.raises(ValueError, match="rowscale"):
        epilogue.add_norm(torch.zeros(2, 3, 4, 8), torch.zeros(2, 3, 4, 8), None, torch.ones(6), ln, out_dtype=torch.float32)
    with pytest.raises(ValueError, match="rowscale"):
        epilogue.add_norm(torch.zeros(8), torch.zeros(8), None, torch.ones(1), ln, out_dtype=torch.float32)


# ------------------------------------------------------------------------------------------------ GPU: error measures
# Whole-tensor bars as in tests/test_gpu_epilogue.py.  The localized ones are set from the worst value measured over every
# case of this file on an H100 SXM (700 W), given in brackets.
WHOLE = {F32: 1e-6, F16: 6e-4, BF16: 4e-3}
WHOLE_BWD = {F32: 2e-6, F16: 6e-4, BF16: 4e-3}
ROW_F32 = 1e-5                    # worst row / sample of an fp32 output, norm-relative [2.3e-6: dx of a 4-channel row]
COL = 5e-7                        # worst column sum, |error| / sum over the column of |terms| [5.5e-8]
ULP = 0.6                         # worst bf16 / fp16 element, in ulps of its fp64 value (+ FLOOR) [0.4999: correctly rounded]
FLOOR = 1e-5                      # absolute: fp32 rounding of O(1) terms that cancel next to 0
STAT = 3e-6                       # mean (in units of the row's standard deviation) and rstd (relative) [6.8e-7]


class Err:
    """One output against its fp64 reference, accumulated over row chunks: whole-tensor norm ratio, worst row, worst sample
    (`groups`: the sample of each row) and, for a bf16 / fp16 output, the worst element in ulps.  `scale`: a row's norm is
    taken as at least scale x sqrt(C), for outputs whose accuracy is absolute rather than relative (the erf approximation
    of GELU: a row of pre-activations far below 0 has values of 1e-5 and errors of 1e-7)."""

    def __init__(self, ngroups=0, scale=0.0):
        self.d2 = self.n2 = self.row = self.ulps = 0.0
        self.scale2 = scale * scale
        self.grouped = False
        self.gd2 = torch.zeros(ngroups, dtype=torch.float64, device=DEV)
        self.gn2 = torch.zeros(ngroups, dtype=torch.float64, device=DEV)

    @torch.no_grad()
    def add(self, got, ref, groups=None):
        diff = got.double() - ref
        d2, n2 = diff.square().sum(-1), ref.square().sum(-1)
        self.d2 += d2.sum().item()
        self.n2 += n2.sum().item()
        self.row = max(self.row, (d2.sqrt() / (n2 + self.scale2 * ref.shape[-1]).sqrt().clamp_min(TINY)).max().item())
        if groups is not None:
            self.grouped = True
            self.gd2.index_add_(0, groups, d2)
            self.gn2.index_add_(0, groups, n2)
        if got.dtype in (BF16, F16):
            _, e = torch.frexp(ref)                            # |ref| in [2^(e-1), 2^e): ulp = 2^(e - significand bits)
            ulp = torch.ldexp(torch.ones_like(ref), e - (8 if got.dtype == BF16 else 11))
            if got.dtype == F16:
                ulp = ulp.clamp_min(2.0 ** -24)                # subnormal spacing
            self.ulps = max(self.ulps, (diff.abs() / (ulp + FLOOR)).max().item())
        return self

    @property
    def whole(self):
        return math.sqrt(self.d2) / max(math.sqrt(self.n2), TINY)

    @property
    def sample(self):
        return (self.gd2.sqrt() / self.gn2.sqrt().clamp_min(TINY)).max().item() if self.grouped else self.row

    def check(self, name, dtype, bwd=False, log=None):
        """whole-tensor bar; worst row / sample for fp32 outputs, worst element in ulps for bf16 / fp16 ones"""
        if log is not None:
            log[name] = self.whole
            log[name + "_row"] = self.row
            log[name + "_sample"] = self.sample
            if dtype != F32:
                log[name + "_ulps"] = self.ulps
        assert self.whole < (WHOLE_BWD if bwd else WHOLE)[dtype], (name, self.whole)
        if dtype == F32:
            assert max(self.row, self.sample) < ROW_F32, (name, self.row, self.sample)
        else:
            assert self.ulps <= ULP, (name, self.ulps)


class ColErr:
    """A column sum against its fp64 reference, normalised per column by the sum of |terms| (cancellation-aware)."""

    def __init__(self, C):
        self.ref = torch.zeros(C, dtype=torch.float64, device=DEV)
        self.abs = torch.zeros(C, dtype=torch.float64, device=DEV)

    @torch.no_grad()
    def add(self, terms):
        self.ref += terms.sum(0)
        self.abs += terms.abs().sum(0)

    def check(self, name, got, log=None):
        e = ((got.double() - self.ref).abs() / self.abs.clamp_min(TINY)).max().item()
        w = relerr(got, self.ref)
        if log is not None:
            log[name] = w
            log[name + "_col"] = e
        assert w < 1e-5 and e < COL, (name, w, e)


def _chunks(rows, C, budget=1 << 22):
    step = max(1, budget // max(C, 1))
    return [(r0, min(rows, r0 + step)) for r0 in range(0, rows, step)]


def _distinct_scales(n, gen):
    """n distinct DropPath-like factors in [0.5, 1.5) with one dropped sample (0) when there is more than one"""
    s = 0.5 + torch.randperm(n, device=DEV, generator=gen).float() / n
    if n > 1:
        s[n // 2] = 0.0
    return s


def _ln_ref_rows(xo, g, b, dy, gres):
    """fp64 LayerNorm of the rows of xo and its backward for dy (+ gres): (y, mean, rstd, xhat, dx)"""
    mu = xo.mean(1, keepdim=True)
    xc = xo - mu
    rs = (xc.square().mean(1, keepdim=True) + EPS).rsqrt()
    xh = xc * rs
    gy = dy * g
    dx = rs * (gy - gy.mean(1, keepdim=True) - xh * (gy * xh).mean(1, keepdim=True))
    if gres is not None:
        dx = dx + gres
    return xh * g + b, mu.squeeze(1), rs.squeeze(1), xh, dx


def _stat_errs(mean, rstd, mu_r, rs_r):
    return ((mean.double() - mu_r).abs() * rs_r).max().item(), (rstd.double() / rs_r - 1).abs().max().item()


# ------------------------------------------------------------------------------------------------ GPU: addnorm, raw ABI
@pytest.mark.gpu
@pytest.mark.parametrize("c", AN_CASES, ids=_an_id)
def test_addnorm_rounds_match_fp64(c):
    TB, TY = c.pair
    opts = AN_OPTS[c.opts]
    rows, C, rps = c.rows, c.C, c.rps
    gen = torch.Generator(device=DEV).manual_seed(rows * 1031 + C)
    rnd = lambda *s: torch.randn(*s, device=DEV, generator=gen)
    x = rnd(rows, C) * 2 + 0.5
    br = rnd(rows, C).to(TB) if "br" in opts else None
    bias = 0.3 * rnd(C) if "bias" in opts else None
    gamma, beta = 1 + 0.3 * rnd(C), 0.3 * rnd(C)
    nsamp = cdiv(rows, rps)
    scale = _distinct_scales(nsamp, gen) if "scale" in opts else None
    dy = rnd(rows, C).to(TY)
    gres = rnd(rows, C) if "gres" in opts else None
    xo = torch.empty_like(x) if br is not None else None
    y = torch.empty(rows, C, dtype=TY, device=DEV)
    mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    n0 = _lib.launch_count()
    epilogue.addnorm_raw_forward(x, br, bias, scale, gamma, beta, xo, y, mean, rstd, EPS, rps)
    assert _lib.launch_count() == n0 + 1
    dx = torch.empty_like(x)
    dbr = torch.empty(rows, C, dtype=TB, device=DEV) if "dbr" in opts else None
    dg, db = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    dbias = torch.empty(C, device=DEV) if dbr is not None else None
    ws = epilogue.addnorm_workspace(rows, C, DEV)
    xs = xo if xo is not None else x
    epilogue.addnorm_raw_backward(xs, gamma, mean, rstd, scale, dy, gres, dx, dbr, dg, db, dbias, ws, EPS, rps)

    sample = torch.arange(rows, device=DEV) // rps
    s_rows = scale.double()[sample] if scale is not None else None
    grp = sample if scale is not None else None
    errs = {k: Err(nsamp) for k in ("xo", "y", "dx", "dbr")}
    cols = {k: ColErr(C) for k in ("dgamma", "dbeta", "dbias")}
    stat = [0.0, 0.0]
    g64, b64 = gamma.double(), beta.double()
    for r0, r1 in _chunks(rows, C):
        xo_r = x[r0:r1].double()
        if br is not None:
            t = br[r0:r1].double() + (bias.double() if bias is not None else 0.0)
            xo_r = xo_r + (t * s_rows[r0:r1, None] if s_rows is not None else t)
            errs["xo"].add(xo[r0:r1], xo_r, grp[r0:r1] if grp is not None else None)
        d = dy[r0:r1].double()
        y_r, mu_r, rs_r, xh, dx_r = _ln_ref_rows(xo_r, g64, b64, d, gres[r0:r1].double() if gres is not None else None)
        del xo_r
        errs["y"].add(y[r0:r1], y_r)
        e_mu, e_rs = _stat_errs(mean[r0:r1], rstd[r0:r1], mu_r, rs_r)
        stat = [max(stat[0], e_mu), max(stat[1], e_rs)]
        cols["dgamma"].add(d * xh)
        cols["dbeta"].add(d)
        del y_r, xh
        errs["dx"].add(dx[r0:r1], dx_r)
        if dbr is not None:
            dbr_r = dx_r * s_rows[r0:r1, None] if s_rows is not None else dx_r
            errs["dbr"].add(dbr[r0:r1], dbr_r, grp[r0:r1] if grp is not None else None)
            cols["dbias"].add(dbr_r)
    log = {}
    if br is not None:
        errs["xo"].check("xo", F32, log=log)
    errs["y"].check("y", TY, log=log)
    errs["dx"].check("dx", F32, bwd=True, log=log)
    if dbr is not None:
        errs["dbr"].check("dbr", TB, bwd=True, log=log)
        cols["dbias"].check("dbias", dbias, log=log)
    cols["dgamma"].check("dgamma", dg, log=log)
    cols["dbeta"].check("dbeta", db, log=log)
    log["mean"], log["rstd"] = stat
    record("addnorm_rounds", _an_id(c), **log)
    assert stat[0] < STAT and stat[1] < STAT, stat
    if scale is not None and dbr is not None and nsamp > 1:     # the dropped sample gets exactly no branch gradient
        assert torch.all(dbr[sample == nsamp // 2] == 0)
    # no atomics: a second backward gives the same bits
    if c.rows > 10000:
        dx2, dg2, db2 = torch.empty_like(dx), torch.empty_like(dg), torch.empty_like(db)
        dbr2 = torch.empty_like(dbr) if dbr is not None else None
        dbias2 = torch.empty_like(dbias) if dbias is not None else None
        epilogue.addnorm_raw_backward(xs, gamma, mean, rstd, scale, dy, gres, dx2, dbr2, dg2, db2, dbias2, ws, EPS, rps)
        assert torch.equal(dx, dx2) and torch.equal(dg, dg2) and torch.equal(db, db2)
        assert dbr is None or (torch.equal(dbr, dbr2) and torch.equal(dbias, dbias2))


# ------------------------------------------------------------------------------------------------ GPU: LayerNorm module
def _ln_id(c):
    return f"{NAME[c.xdt]}-{NAME[c.ydt]}-C{c.C}-r{c.rows}"


def _ln_module(C, xdt, ydt, gen):
    """B200LayerNorm whose forward emits ydt from an xdt input: fp32 -> bf16 / fp16 under autocast, bf16 / fp16 -> fp32 with
    keep_dtype under autocast, and no autocast for the same-dtype pairs."""
    ln = B200LayerNorm(C, eps=EPS, keep_dtype=xdt != F32 and ydt == F32).to(DEV)
    with torch.no_grad():
        ln.weight.copy_(1 + 0.3 * torch.randn(C, device=DEV, generator=gen))
        ln.bias.copy_(0.3 * torch.randn(C, device=DEV, generator=gen))
    amp = None if xdt == ydt else (ydt if xdt == F32 else xdt)
    return ln, amp


def _ln_run(ln, amp, x):
    with torch.autocast("cuda", dtype=amp or BF16, enabled=amp is not None):
        return ln(x)


@pytest.mark.gpu
@pytest.mark.parametrize("c", LN_CASES, ids=_ln_id)
def test_layernorm_module_rounds_match_fp64(c):
    gen = torch.Generator(device=DEV).manual_seed(c.rows * 7 + c.C)
    ln, amp = _ln_module(c.C, c.xdt, c.ydt, gen)
    x = (torch.randn(c.rows, c.C, device=DEV, generator=gen) * 2 + 0.5).to(c.xdt).requires_grad_(True)
    n0 = _lib.launch_count()
    y = _ln_run(ln, amp, x)
    assert _lib.launch_count() == n0 + 1 and y.dtype == c.ydt
    gy = torch.randn(c.rows, c.C, device=DEV, generator=gen).to(c.ydt)
    dx, dg, db = torch.autograd.grad(y, (x, ln.weight, ln.bias), gy, retain_graph=True)
    dx2, dg2, db2 = torch.autograd.grad(y, (x, ln.weight, ln.bias), gy)
    assert torch.equal(dx, dx2) and torch.equal(dg, dg2) and torch.equal(db, db2)      # no atomics
    ey, edx = Err(), Err()
    cg, cb = ColErr(c.C), ColErr(c.C)
    g64, b64 = ln.weight.detach().double(), ln.bias.detach().double()
    for r0, r1 in _chunks(c.rows, c.C):
        d = gy[r0:r1].double()
        y_r, _, _, xh, dx_r = _ln_ref_rows(x[r0:r1].detach().double(), g64, b64, d, None)
        ey.add(y[r0:r1], y_r)
        edx.add(dx[r0:r1], dx_r)
        cg.add(d * xh)
        cb.add(d)
    log = {}
    ey.check("y", c.ydt, log=log)
    edx.check("dx", c.xdt, bwd=True, log=log)
    cg.check("dgamma", dg, log=log)
    cb.check("dbeta", db, log=log)
    record("layernorm_rounds", _ln_id(c), **log)


# ------------------------------------------------------------------------------------------------ GPU: bias + activation
def _ba_id(c):
    return f"{NAME[c.dt]}-{c.act}-C{c.C}-r{c.rows}"


def _gelu_grad64(u):
    return 0.5 * (1 + torch.erf(u * 0.5 ** 0.5)) + u * torch.exp(-0.5 * u * u) * (2 * math.pi) ** -0.5


def _gelu_check(z2, bias, a2, da2, dz2, dbias, log, prefix=""):
    """a = GELU(z + bias) and dz = da GELU'(z + bias) elementwise against fp64; d_bias against the fp64 column sum of dz AS
    STORED.  That is the kernel's documented semantics (the sum autograd would take over the tensor the next GEMM sees), and
    it makes the bar a pure check of the reduction: the fp64 dz rounded to bf16 differs from the kernel's fp32 dz rounded to
    bf16 by one ulp wherever the two straddle a rounding boundary, which alone moved column sums by 1e-5 of their |terms|."""
    C = z2.shape[1]
    ea, edz, col = Err(scale=1.0), Err(scale=1.0), ColErr(C)
    for r0, r1 in _chunks(z2.shape[0], C):
        u = z2[r0:r1].detach().double() + bias.detach().double()
        ea.add(a2[r0:r1], F.gelu(u))
        edz.add(dz2[r0:r1], da2[r0:r1].double() * _gelu_grad64(u))
        col.add(dz2[r0:r1].double())
    ea.check(prefix + "a", a2.dtype, log=log)
    edz.check(prefix + "dz", dz2.dtype, bwd=True, log=log)
    col.check(prefix + "dbias", dbias, log=log)


@pytest.mark.gpu
@pytest.mark.parametrize("c", BA_CASES, ids=_ba_id)
def test_bias_act_rounds_match_fp64(c):
    gen = torch.Generator(device=DEV).manual_seed(c.rows * 13 + c.C)
    act = _lib.VIL_ACT_GELU if c.act == "gelu" else _lib.VIL_ACT_NONE
    z = (2 * torch.randn(c.rows, c.C, device=DEV, generator=gen)).to(c.dt)
    bias = 0.5 * torch.randn(c.C, device=DEV, generator=gen)
    da = torch.randn(c.rows, c.C, device=DEV, generator=gen).to(c.dt)
    a = torch.empty_like(z)
    n0 = _lib.launch_count()
    epilogue.bias_act_raw_forward(z, bias, a, act)
    assert _lib.launch_count() == n0 + 1
    dz = torch.empty_like(z) if act == _lib.VIL_ACT_GELU else None       # act none: the plain column sum of da
    dbias = torch.empty(c.C, device=DEV)
    ws = epilogue.bias_act_workspace(da, act)
    epilogue.bias_act_raw_backward(da, z, bias, dz, dbias, ws, act)
    dz2 = torch.empty_like(dz) if dz is not None else None
    dbias2 = torch.empty_like(dbias)
    epilogue.bias_act_raw_backward(da, z, bias, dz2, dbias2, ws, act)
    assert torch.equal(dbias, dbias2) and (dz is None or torch.equal(dz, dz2))        # no atomics
    ea, edz, col = Err(scale=1.0), Err(scale=1.0), ColErr(c.C)
    b64 = bias.double()
    for r0, r1 in _chunks(c.rows, c.C):
        u = z[r0:r1].double() + b64
        ea.add(a[r0:r1], F.gelu(u) if act == _lib.VIL_ACT_GELU else u)
        d = da[r0:r1].double()
        if dz is not None:
            edz.add(dz[r0:r1], d * _gelu_grad64(u))
            d = dz[r0:r1].double()           # d_bias: the column sum of dz as stored (see _gelu_check)
        col.add(d)
    log = {}
    ea.check("a", c.dt, log=log)
    if dz is not None:
        edz.check("dz", c.dt, bwd=True, log=log)
    col.check("dbias", dbias, log=log)
    record("bias_act_rounds", _ba_id(c), **log)


# ------------------------------------------------------------------------------------------------ GPU: production shape
def _addnorm_autograd_check(x, br, bias, scale, ln, out_dtype, g_xo, g_y, name, launches=1):
    """epilogue.add_norm forward + backward on a (B, ..., C) stream against fp64, chunk by chunk over the samples"""
    n0 = _lib.launch_count()
    xo, y = epilogue.add_norm(x, br, bias, scale, ln, out_dtype=out_dtype)
    assert _lib.launch_count() == n0 + launches
    dx, dbr, dbias, dg, db = torch.autograd.grad((xo, y), (x, br, bias, ln.weight, ln.bias), (g_xo, g_y))
    B, C = x.shape[0], x.shape[-1]
    rows = x.numel() // C
    rps = rows // B
    x2, br2, xo2, y2 = (t.detach().reshape(rows, C) for t in (x, br, xo, y))
    gx2, gy2, dx2, dbr2 = (t.reshape(rows, C) for t in (g_xo, g_y, dx, dbr))
    s_rows = scale.double().repeat_interleave(rps)
    grp = torch.arange(rows, device=DEV) // rps
    errs = {k: Err(B) for k in ("xo", "y", "dx", "dbr")}
    cols = {k: ColErr(C) for k in ("dgamma", "dbeta", "dbias")}
    g64, b64 = ln.weight.detach().double(), ln.bias.detach().double()
    for r0, r1 in _chunks(rows, C):
        t = (br2[r0:r1].double() + bias.detach().double()) * s_rows[r0:r1, None]
        xo_r = x2[r0:r1].detach().double() + t
        d = gy2[r0:r1].double()
        y_r, _, _, xh, dx_r = _ln_ref_rows(xo_r, g64, b64, d, gx2[r0:r1].double())
        errs["xo"].add(xo2[r0:r1], xo_r, grp[r0:r1])
        errs["y"].add(y2[r0:r1], y_r, grp[r0:r1])
        errs["dx"].add(dx2[r0:r1], dx_r, grp[r0:r1])
        dbr_r = dx_r * s_rows[r0:r1, None]
        errs["dbr"].add(dbr2[r0:r1], dbr_r, grp[r0:r1])
        cols["dgamma"].add(d * xh)
        cols["dbeta"].add(d)
        cols["dbias"].add(dbr_r)
    log = {}
    errs["xo"].check("xo", F32, log=log)
    errs["y"].check("y", out_dtype, log=log)
    errs["dx"].check("dx", F32, bwd=True, log=log)
    errs["dbr"].check("dbr", br.dtype, bwd=True, log=log)
    for k, got in (("dgamma", dg), ("dbeta", db), ("dbias", dbias)):
        cols[k].check(k, got, log=log)
    record("addnorm_autograd", name, **log)
    assert torch.all(dbr[scale == 0] == 0)


@pytest.mark.gpu
def test_production_stage1_b64():
    """ViL-Small stage 1 at B = 64 (56 x 56 + 1 tokens, C = 96: six forward rounds of addnorm) through add_norm, bias_gelu
    and linear_colsum_bias, with a distinct DropPath scale per sample (one 0), checked sample by sample."""
    B, N, C = 64, 3137, 96
    gen = torch.Generator(device=DEV).manual_seed(64)
    rnd = lambda *s: torch.randn(*s, device=DEV, generator=gen)
    ln, _ = _ln_module(C, F32, F32, gen)
    x = (rnd(B, N, C) * 2 + 0.5).requires_grad_(True)
    br = rnd(B, N, C).to(BF16).requires_grad_(True)
    bias = (0.3 * rnd(C)).requires_grad_(True)
    scale = _distinct_scales(B, gen)
    assert cdiv(B * N, an_fwd_round(B * N, C)) == 6
    _addnorm_autograd_check(x, br, bias, scale, ln, BF16, rnd(B, N, C), rnd(B, N, C).to(BF16), "vil_small_s1_b64")
    del x, br

    z = (2 * rnd(B, N, C)).to(BF16).requires_grad_(True)
    bias = (0.5 * rnd(C)).requires_grad_(True)
    n0 = _lib.launch_count()
    a = epilogue.bias_gelu(z, bias)
    assert _lib.launch_count() == n0 + 1
    da = rnd(B, N, C).to(BF16)
    dz, dbias = torch.autograd.grad(a, (z, bias), da)
    log = {}
    _gelu_check(z.reshape(-1, C), bias, a.reshape(-1, C), da.reshape(-1, C), dz.reshape(-1, C), dbias, log)
    record("bias_gelu_autograd", "vil_small_s1_b64", **log)
    del z, a, dz

    lin = torch.nn.Linear(C, C).to(DEV)              # fp32: the bias gradient is the kernel's sum, not a bf16 rounding of it
    y = epilogue.linear_colsum_bias(rnd(B, N, C), lin.weight, lin.bias)
    gy = rnd(B, N, C)
    (dbias,) = torch.autograd.grad(y, (lin.bias,), gy)
    col = ColErr(C)
    for r0, r1 in _chunks(B * N, C):
        col.add(gy.reshape(-1, C)[r0:r1].double())
    log = {}
    col.check("dbias", dbias, log=log)
    record("linear_colsum_bias", "vil_small_s1_b64", **log)


# ------------------------------------------------------------------------------------------------ GPU: the two fixes
def _misaligned(shape, dtype, gen, scale=1.0, shift=0.0):
    """a contiguous view of `shape` that starts one element past a 16-byte boundary"""
    n = math.prod(shape)
    buf = (torch.randn(n + 1, device=DEV, generator=gen) * scale + shift).to(dtype)
    t = buf[1:].view(shape)
    assert t.is_contiguous() and t.data_ptr() % 16 != 0
    return t


@pytest.mark.gpu
def test_misaligned_views_take_one_launch_and_match_fp64():
    """Contiguous views that start mid-allocation (inputs, gradients, and parameters that are views into a flat buffer)
    through B200LayerNorm, add_norm, bias_gelu and linear_colsum_bias: each op copies what is misaligned and still runs
    one kernel forward."""
    gen = torch.Generator(device=DEV).manual_seed(5)
    B, N, C = 3, 1001, 100
    # B200LayerNorm, the vectorised fp32 path, with its weight and bias views into one flat parameter buffer
    ln = B200LayerNorm(C, eps=EPS).to(DEV)
    flat = torch.randn(2 * C + 1, device=DEV, generator=gen) * 0.3
    flat[1:C + 1] += 1.0
    ln.weight, ln.bias = torch.nn.Parameter(flat[1:C + 1]), torch.nn.Parameter(flat[C + 1:])
    assert ln.weight.data_ptr() % 16 != 0 and ln.bias.data_ptr() % 16 != 0
    x = _misaligned((B, N, C), F32, gen, 2.0, 0.5).requires_grad_(True)
    gy = _misaligned((B, N, C), F32, gen)
    n0 = _lib.launch_count()
    y = ln(x)
    assert _lib.launch_count() == n0 + 1
    dx, dg, db = torch.autograd.grad(y, (x, ln.weight, ln.bias), gy)
    y_r, _, _, xh, dx_r = _ln_ref_rows(x.detach().double().reshape(-1, C), ln.weight.detach().double(), ln.bias.detach().double(),
                                       gy.double().reshape(-1, C), None)
    log = {}
    Err().add(y.reshape(-1, C), y_r).check("ln_y", F32, log=log)
    Err().add(dx.reshape(-1, C), dx_r).check("ln_dx", F32, bwd=True, log=log)
    for name, got, terms in (("ln_dgamma", dg, gy.double().reshape(-1, C) * xh), ("ln_dbeta", db, gy.double().reshape(-1, C))):
        col = ColErr(C)
        col.add(terms)
        col.check(name, got, log=log)

    # add_norm: stream, branch, bias, rowscale and both incoming gradients misaligned
    x = _misaligned((B, N, C), F32, gen, 2.0, 0.5).requires_grad_(True)
    br = _misaligned((B, N, C), BF16, gen).requires_grad_(True)
    bias = _misaligned((C,), F32, gen, 0.3).requires_grad_(True)
    scale = torch.zeros(B + 1, device=DEV)[1:]
    scale.copy_(torch.tensor([1.3, 0.0, 0.7], device=DEV))
    _addnorm_autograd_check(x, br, bias, scale, ln, BF16, _misaligned((B, N, C), F32, gen), _misaligned((B, N, C), BF16, gen),
                            "misaligned")

    # bias_gelu and linear_colsum_bias: bf16 rows one element (2 bytes) off
    z = _misaligned((B, N, 384), BF16, gen, 2.0).requires_grad_(True)
    bias = _misaligned((384,), F32, gen, 0.5).requires_grad_(True)
    n0 = _lib.launch_count()
    a = epilogue.bias_gelu(z, bias)
    assert _lib.launch_count() == n0 + 1
    da = _misaligned((B, N, 384), BF16, gen)
    dz, dbias = torch.autograd.grad(a, (z, bias), da)
    _gelu_check(z.reshape(-1, 384), bias, a.reshape(-1, 384), da.reshape(-1, 384), dz.reshape(-1, 384), dbias, log, "gelu_")
    lin = torch.nn.Linear(C, 384).to(DEV)
    y = epilogue.linear_colsum_bias(torch.randn(B, N, C, device=DEV, generator=gen), lin.weight, lin.bias)
    gy = _misaligned((B, N, 384), F32, gen)
    (dbias,) = torch.autograd.grad(y, (lin.bias,), gy)
    col = ColErr(384)
    col.add(gy.double().reshape(-1, 384))
    col.check("linear_dbias", dbias, log=log)
    record("misaligned", "views", **log)


@pytest.mark.gpu
def test_add_norm_4d_stream_with_distinct_scales():
    """A (B, H, W, C) stream: every sample's H x W rows take that sample's DropPath scale."""
    gen = torch.Generator(device=DEV).manual_seed(4)
    B, H, W, C = 5, 23, 31, 192
    rnd = lambda *s: torch.randn(*s, device=DEV, generator=gen)
    ln, _ = _ln_module(C, F32, F32, gen)
    x = (rnd(B, H, W, C) * 2 + 0.5).requires_grad_(True)
    br = rnd(B, H, W, C).to(BF16).requires_grad_(True)
    bias = (0.3 * rnd(C)).requires_grad_(True)
    scale = torch.tensor([0.6, 1.4, 0.0, 1.1, 0.9], device=DEV)
    _addnorm_autograd_check(x, br, bias, scale, ln, BF16, rnd(B, H, W, C), rnd(B, H, W, C).to(BF16), "4d")
    with pytest.raises(ValueError, match="rowscale"):
        epilogue.add_norm(x, br, bias, torch.ones(B * H, device=DEV), ln, out_dtype=BF16)


# ------------------------------------------------------------------------------------------------ GPU: model level, fp32
MODEL_BAR = 2.5e-4                # H100 SXM: logits 7.7e-6, input gradient 3.8e-5, worst parameter gradient 7.0e-5


@pytest.mark.gpu
def test_fused_residual_matches_stock_in_fp32(monkeypatch):
    """fused_residual=True against the stock composition in fp32 (no autocast), train mode, with every DropPath module of
    both nets returning the same fixed, distinct per-sample scales in the same order (one sample dropped per module): logits,
    input gradient and every parameter gradient agree to fp32 rounding, which the bf16 comparison in
    tests/test_gpu_epilogue.py (bars of 8e-2) cannot resolve."""
    arch = "l1,h2,d64,n2,s1,g1,p4,f7_l2,h2,d128,n2,s0,g1,p2,f7_l3,h4,d256,n1,s0,g0,p2,f7"
    torch.manual_seed(0)
    kw = dict(img_size=112, num_classes=50, drop_path_rate=0.2)
    a = build_vil(arch, fused_residual=True, **kw).to(DEV).train()
    b = build_vil(arch, fused_residual=False, **kw).to(DEV).train()
    b.load_state_dict(a.state_dict())
    calls = [0]
    base = torch.tensor([0.0, 0.8, 1.25, 1.6], device=DEV)

    def fixed_scale(self, batch, device):
        if self.drop_prob == 0. or not self.training:
            return None
        calls[0] += 1
        return base.roll(calls[0])[:batch].clone()

    monkeypatch.setattr(DropPath, "sample_scale", fixed_scale)
    x = torch.randn(4, 3, 112, 112, device=DEV)
    gy = torch.randn(4, 50, device=DEV)
    outs = []
    for net in (a, b):
        calls[0] = 0
        xg = x.clone().requires_grad_(True)
        n0 = _lib.launch_count()
        y = net(xg)
        (y * gy).sum().backward()
        outs.append((y, xg.grad, {k: p.grad for k, p in net.named_parameters()}, _lib.launch_count() - n0, calls[0]))
    (ya, dxa, ga, la, ca), (yb, dxb, gb, lb, cb) = outs
    assert ca == cb > 0 and la > lb
    assert all((ga[k] is None) == (gb[k] is None) for k in ga)
    errs = {"logits": relerr(ya, yb), "dx": relerr(dxa, dxb)}
    errs.update({k: relerr(ga[k], gb[k]) for k in ga if gb[k] is not None and gb[k].numel() > 0 and gb[k].abs().max() > 0})
    worst = max(errs.items(), key=lambda kv: kv[1])
    record("fused_residual_fp32", arch, logits=errs["logits"], dx=errs["dx"], worst_param=max(errs.values()))
    assert worst[1] < MODEL_BAR, worst
