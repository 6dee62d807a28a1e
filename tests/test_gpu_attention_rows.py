"""The attention kernels row by row.

The other parity files draw q, k, v from randn and hold one norm per tensor.  That leaves three gaps, closed here:

* the softmax of randn inputs is diffuse: the running maximum hardly moves between pieces, nothing underflows, and no row
  ever starts with a piece in which every column is masked (the `-inf` guards of the online softmax);
* a norm over the whole tensor dilutes an error that sits in one row, one chunk or one piece;
* no other test has more than 16 global tokens, so a second 64-key piece of global keys never runs.

Metrics (all against the fp64 dense oracle on the inputs rounded to the kernel's dtype, through the C ABI):
  query-row and key-row tensors   max over (image, head, row) of ||x - ref|| / (||ref|| + floor) over D, global rows apart
                                  from local ones; the failure message names the row's chunk, 64-row piece and edge state
  per chunk                       max over (image, head, chunk) of the norm-relative error of the chunk's block
  lse, lse_g                      max absolute error, finite everywhere
  bias gradients                  whole-tensor norm at the bars of test_gpu_parity; tests/test_gpu_bias_entries.py holds
                                  them entry by entry
The floor is 0 except under a saturated softmax (`peak_floors`).  Every maximum is recorded (tests.util.record).

The bars were measured on an H100 SXM (700 W power limit): each is at most about 3x the worst value seen over this file
and at most 4x the whole-tensor bar of the variant (DESIGN.md section 4).
"""
import pytest
import torch

from oracle import vil_oracle as vo
from tests import test_gpu_dropout as tdrop
from tests import test_gpu_parity as tpar
from tests import test_headdim128 as thd
from tests.util import record, relerr

gpu = pytest.mark.gpu
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16

# family, dtype, VIL_FLAG_F32_OUT (fp32 outputs: the kernel without the rounding of its stores), layout
VARIANTS = {
    "simt_fp32": ("simt", F32, False, "contig"),
    "wgmma_fp16_f32out": ("wgmma", F16, True, "contig"),
    "wgmma_bf16_f32out": ("wgmma", BF16, True, "contig"),
    "wgmma_bf16": ("wgmma", BF16, False, "contig"),
    "wgmma_bf16_linear": ("wgmma", BF16, False, "linear"),
}
# Localized bars: (forward, backward) for the worst row and the worst chunk, lse absolute.  Whole-tensor bars of the same
# variants (test_gpu_parity): 1e-5 / 2e-5, 1e-3 / 1e-3, 2e-3 / 2e-3, 4e-3 / 8e-3.
# Worst values measured with randn inputs (rows forward / backward, chunks forward / backward): SIMT fp32 2.3e-6 / 2.3e-6,
# 9.6e-7 / 1.0e-6; fp16 with fp32 outputs 3.8e-4 / 5.7e-4, 2.3e-4 / 3.6e-4; bf16 with fp32 outputs 3.2e-3 / 5.6e-3,
# 1.9e-3 / 2.5e-3; bf16 production 4.1e-3 / 7.0e-3, 2.6e-3 / 4.4e-3; lse 2.1e-6, lse_g 6.6e-7.
BARS = {
    "simt_fp32": dict(row=(6e-6, 6e-6), chunk=(2.5e-6, 2.5e-6), lse=5e-6),
    "wgmma_fp16_f32out": dict(row=(1e-3, 1.5e-3), chunk=(6e-4, 9e-4), lse=5e-6),
    "wgmma_bf16_f32out": dict(row=(8e-3, 8e-3), chunk=(4.5e-3, 6e-3), lse=5e-6),
    "wgmma_bf16": dict(row=(1e-2, 1.6e-2), chunk=(6.5e-3, 1.1e-2), lse=5e-6),
}
# A floor enters as  ||err|| <= bar ||ref|| + FLOOR_ROUNDINGS floor: the floor is one rounding of the named quantity, and a
# handful of them meet in a row (measured: up to 1.4 floors in dq under a saturated softmax).
FLOOR_ROUNDINGS = 16.0
BARS["wgmma_bf16_linear"] = BARS["wgmma_bf16"]
BIAS_BARS = {"simt_fp32": 1e-4, "wgmma_fp16_f32out": 1e-2, "wgmma_bf16_f32out": 5e-2, "wgmma_bf16": 5e-2,
             "wgmma_bf16_linear": 5e-2}

CASE_ID = lambda c: "B%d_H%d_D%d_%dx%d_g%d_w%d_e%d_m%d_%s" % (c[:9] + ("rpe" if c[9] else "nob",)) + \
    ("_sep" if len(c) > 10 and c[10] else "")


# --------------------------------------------------------------------------- inputs and the oracle
def make_inputs(case, seed, sep=False):
    B, H, D, nx, ny, g, w, exact, mode, rpe = case[:10]
    gen = torch.Generator().manual_seed(seed)
    N = g + nx * ny
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    t = dict(q=r(B, H, nx * ny, D), k=r(B, H, N, D), v=r(B, H, N, D), qg=r(B, H, g, D),
             table=0.5 * r((4 * w - 1) ** 2, H) if rpe else None,
             g2l=0.5 * r(2, H, g) if (rpe and g) else None, g2g=0.5 * r(H, g, g) if (rpe and g) else None,
             go=r(B, H, nx * ny, D), gog=r(B, H, g, D))
    t["kg"], t["vg"] = (r(B, H, N, D), r(B, H, N, D)) if (sep and g) else (t["k"], t["v"])
    return t


def cfg_of(case):
    B, H, D, nx, ny, g, w, exact, mode, rpe = case[:10]
    return nx, ny, w, exact, mode, D ** -0.5


_VISITS, _REFS = {}, {}


def _dense(q, k, v, qg, kg, vg, table, g2l, g2g, cfg):
    """vo.dense_attention; without the table the visit weights depend on the geometry alone and are built once"""
    nx, ny, w, exact, mode, scale = cfg
    kw = dict(nx=nx, ny=ny, w=w, exact=exact, mode=mode, scale=scale)
    if table is not None:
        return vo.dense_attention(q, k, v, qg, kg, vg, table, g2l, g2g, **kw)
    key = (nx, ny, w, exact, mode, q.shape[1])
    if key not in _VISITS:
        _VISITS[key] = vo.visit_weights(nx, ny, w, exact, mode, None, q.shape[1])
    orig = vo.visit_weights
    vo.visit_weights = lambda *a, **k_: _VISITS[key]
    try:
        return vo.dense_attention(q, k, v, qg, kg, vg, None, None, None, **kw)
    finally:
        vo.visit_weights = orig


def oracle(t, cfg, dtype, key):
    """fp64 dense oracle, forward and gradients, on the values the kernel sees (inputs rounded to `dtype`)"""
    if (key, dtype) in _REFS:
        return _REFS[(key, dtype)]
    rd = lambda x: x.to(dtype).double().requires_grad_(True)
    q, k, v, qg = rd(t["q"]), rd(t["k"]), rd(t["v"]), rd(t["qg"])
    g = k.shape[2] - q.shape[2]
    sep = g > 0 and t["kg"] is not t["k"]
    kg, vg = (rd(t["kg"]), rd(t["vg"])) if sep else (k, v)
    table, g2l, g2g = [None if t[n] is None else t[n].float().double().requires_grad_(True) for n in ("table", "g2l", "g2g")]
    o, og, lse, lse_g = _dense(q, k, v, qg if g else None, kg, vg, table, g2l, g2g, cfg)
    loss = (o * t["go"].to(dtype).double()).sum() + ((og * t["gog"].to(dtype).double()).sum() if g else 0)
    ins = dict(q=q, k=k, v=v)
    if g:
        ins["qg"] = qg
        if sep:
            ins.update(kg=kg, vg=vg)
    ins.update({n: x for n, x in (("table", table), ("g2l", g2l), ("g2g", g2g)) if x is not None})
    grads = torch.autograd.grad(loss, list(ins.values()))
    ref = dict(o=o.detach(), og=None if og is None else og.detach(), lse=lse.detach(),
               lse_g=None if lse_g is None else lse_g.detach(), **{"d" + n: x for n, x in zip(ins, grads)})
    _REFS[(key, dtype)] = ref
    return ref


def run_kernels(t, cfg, variant, drop=(0.0, 0, 0)):
    impl, dtype, f32out, layout = VARIANTS[variant]
    nx, ny, w, exact, mode, scale = cfg
    out, fam_f, fam_b = tpar.kernel_run(t, nx, ny, w, exact, mode, scale, dtype, impl, layout=layout, f32out=f32out, drop=drop)
    assert fam_f == impl and fam_b == impl, (fam_f, fam_b)             # no other family behind the name
    return out


# --------------------------------------------------------------------------- localized metrics
def row_errors(x, ref, floor=0.0):
    """(B, H, T): ||x - ref||_2 / (||ref||_2 + floor) over D of every row; floor is a number or broadcasts to (B, H, T)"""
    x, ref = x.detach().double().cpu(), ref.detach().double().cpu()
    return (x - ref).norm(dim=-1) / (ref.norm(dim=-1) + floor).clamp_min(1e-300)


def chunk_errors(x, ref, nx, ny, w, floor=0.0):
    """(B, H, mx, my): norm-relative error of each chunk's block of a local-row tensor (B, H, nx * ny, D); the floor of a
    block is the norm of its rows' floors"""
    padx, pady, mx, my = vo.geometry(nx, ny, w)

    def blocks(a):
        B, H, _, D = a.shape
        img = torch.nn.functional.pad(a.reshape(B, H, nx, ny, D), (0, 0, 0, pady, 0, padx))
        return img.reshape(B, H, mx, w, my, w, D).pow(2).sum(dim=(3, 5, 6)).sqrt()

    x, ref = x.detach().double().cpu(), ref.detach().double().cpu()
    fl = blocks((torch.zeros(ref.shape[:3], dtype=torch.float64) + floor)[..., None])
    return blocks(x - ref) / (blocks(ref) + fl).clamp_min(1e-300)


def worst(e):
    """(max, index tuple) of an error tensor; NaN counts as the worst"""
    e = torch.where(torch.isnan(e), torch.full_like(e, float("inf")), e)
    i = int(e.argmax())
    idx = []
    for n in reversed(e.shape):
        idx.append(i % n)
        i //= n
    return float(e.flatten()[int(e.argmax())]), tuple(reversed(idx))


def where_local(idx, nx, ny, w):
    """where local token idx = (b, h, t) lies, in the terms the kernels are written in"""
    b, h, t = idx
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    r, c = divmod(t, ny)
    R, C = r // w, c // w
    piece = ((r % w) * w + c % w) // 64
    edge = R in (0, mx - 1) or C in (0, my - 1)
    padded = (R == mx - 1 and padx > 0) or (C == my - 1 and pady > 0)
    return "image %d head %d token (%d, %d) chunk (%d, %d) of %d x %d, piece %d of %d%s%s" % (
        b, h, r, c, R, C, mx, my, piece, (w * w + 63) // 64, ", edge chunk" if edge else "", ", padded chunk" if padded else "")


def where_chunk(idx, nx, ny, w):
    b, h, R, C = idx
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    return "image %d head %d chunk (%d, %d) of %d x %d%s" % (
        b, h, R, C, mx, my, ", padded" if (R == mx - 1 and padx) or (C == my - 1 and pady) else "")


def peak_floors(t, cfg, variant, g):
    """Floors for the gradients under a saturated softmax, where a reference row is tiny by construction.

    dS = P (dP - delta) for the dominant key is a cancellation: P -> 1 and dP - delta -> 0, with dP = dO . v and
    delta = dO . o of size ||dO|| ||v||.  delta is computed from the STORED o, and dP in fp32, so dS carries an absolute
    error of eps ||dO|| ||v|| with eps = the machine epsilon of the type o is stored in (bf16 in the production build, fp32
    under VIL_FLAG_F32_OUT and in the SIMT family) whatever the size of the exact dS.  It enters
      dq_i  = scale sum_j dS_ij k_j    as  eps scale ||dO_i|| max||v|| max||k||                 (one dominant key per row)
      dk_j  = scale sum_i dS_ij q_i    as  eps scale max||dO|| max||v|| max||q|| sqrt(n)       n = queries that see key j:
                                           at most 9 w^2 for a local key, all of them for a global key
    and the same with (qg, kg, vg, dOg) for the global rows (n = g).  dv = P^T dO has no cancellation; its floor is the
    flush to zero of a P below the smallest number of its type (`tiny`: fp32 in the exponential, fp16 as the tensor-core
    operand), times max||dO|| over the seeing queries; the same flush of dS adds tiny scale max||q|| (||k||) to dk (dq).
    """
    impl, dtype, f32out, layout = VARIANTS[variant]
    nx, ny, w, exact, mode, scale = cfg
    eps = 2.0 ** -8 if (dtype == BF16 and not f32out) else 2.0 ** -24
    tiny = 2.0 ** -24 if dtype == F16 else 2.0 ** -126      # P and dS below it are flushed to zero as tensor-core operands
    rn = lambda x: x.to(dtype).double().norm(dim=-1)
    nloc = nx * ny
    nsee = min(9 * w * w, nloc)
    go, v, k, q = rn(t["go"]), rn(t["v"]), rn(t["k"]), rn(t["q"])
    f = dict(dq=eps * scale * go * v.max() * k.max() + tiny * scale * float(k.max()) * nsee ** 0.5)
    dk = torch.full(k.shape, float(eps * scale * go.max() * v.max() * q.max() + tiny * scale * q.max()), dtype=torch.float64)
    dk[:, :, g:] *= nsee ** 0.5
    dk[:, :, :g] *= nloc ** 0.5
    f["dk"] = dk
    f["dv"] = tiny * float(go.max()) * nloc ** 0.5
    if g:
        gog, vg, kg, qg = rn(t["gog"]), rn(t["vg"]), rn(t["kg"]), rn(t["qg"])
        f["dqg"] = eps * scale * gog * vg.max() * kg.max()
        fg = float(eps * scale * gog.max() * vg.max() * qg.max()) * g ** 0.5
        if t["kg"] is t["k"]:
            f["dk"] = f["dk"] + fg
        else:
            f["dkg"] = fg
        f["dvg"] = 2.0 ** -126 * float(gog.max()) * g
    return f


def check(test, tag, out, ref, case, variant, floors=None, bias=True, backward=True):
    """measure, record and assert every output of one run; backward=False records the gradients without holding them"""
    nx, ny, w = case[3], case[4], case[6]
    g = case[5]
    bars = BARS[variant]
    floors = floors or {}
    vals, fails = {}, []

    def hold(name, val, bar, loc):
        vals[name] = val
        if name[0] == "d" and not backward:
            return
        if not val < bar:
            fails.append("%s = %.3e (bar %.1e) at %s" % (name, val, bar, loc))

    def rows(name, x, r, bar, lo=0, hi=None, local=True, fl=0.0):
        hi = x.shape[2] if hi is None else hi
        if torch.is_tensor(fl) and fl.dim() == 3:
            fl = fl[:, :, lo:hi]
        val, idx = worst(row_errors(x[:, :, lo:hi], r[:, :, lo:hi], fl * (FLOOR_ROUNDINGS / bar)))
        loc = where_local(idx, nx, ny, w) if local else "image %d head %d global row %d" % idx
        hold(name, val, bar, loc)

    def chunks(name, x, r, bar, fl=0.0):
        if torch.is_tensor(fl) and fl.dim() == 3:
            fl = fl[:, :, g:] if fl.shape[2] > nx * ny else fl
        val, idx = worst(chunk_errors(x, r, nx, ny, w, fl * (FLOOR_ROUNDINGS / bar)))
        hold(name, val, bar, where_chunk(idx, nx, ny, w))

    # Scores far above 16 (the peaked cases reach 500): P = exp(s - lse) of an fp32 s carries |s| 2^-24 per rounding of s,
    # relative, in every output; 16 of them are allowed on top of the bars, nothing for ordinary scores.
    top = float(ref["lse"].abs().max()) if ref.get("lse") is not None else 0.0
    big = 16 * 2.0 ** -24 * top if top > 16 else 0.0
    rf, rb = (x + big for x in bars["row"])
    cf, cb = (x + big for x in bars["chunk"])
    # The global-query backward adds each global query's term into the stored dkg / dvg rows (dk / dv with shared global
    # weights): g successive roundings to the output type, 2^-9 sqrt(g) rms in bf16 (measured: 2.8e-3 sqrt(g) in the worst
    # row at g = 16, 64, 65, 130).  DESIGN.md section 3 has it as a known loss of the bf16 / fp16 outputs at large g.
    out_eps = 2.0 ** -9 if (VARIANTS[variant][1] == BF16 and not VARIANTS[variant][2]) else 0.0
    many = 3 * out_eps * g ** 0.5 if g >= 4 else 0.0
    shared = "dkg" not in ref
    rows("o.row", out["o"], ref["o"], rf)
    chunks("o.chunk", out["o"], ref["o"], cf)
    rows("dq.row", out["dq"], ref["dq"], rb, fl=floors.get("dq", 0.0))
    chunks("dq.chunk", out["dq"], ref["dq"], cb, floors.get("dq", 0.0))
    for n in ("dk", "dv"):
        fl, more = floors.get(n, 0.0), (many if shared else 0.0)
        rows(n + ".row", out[n], ref[n], rb + more, lo=g, fl=fl)
        chunks(n + ".chunk", out[n][:, :, g:], ref[n][:, :, g:], cb + more, fl)
        if g:
            rows(n + ".grow", out[n], ref[n], rb + more, hi=g, local=False, fl=fl)
    if g:
        rows("og.row", out["og"], ref["og"], rf, local=False)
        rows("dqg.row", out["dqg"], ref["dqg"], rb, local=False, fl=floors.get("dqg", 0.0))
        for n in ("dkg", "dvg"):
            if n in ref:
                fl = floors.get(n, 0.0)
                rows(n + ".row", out[n], ref[n], rb + many, lo=g, fl=fl)
                rows(n + ".grow", out[n], ref[n], rb + many, hi=g, local=False, fl=fl)
    for n in ("lse", "lse_g"):
        if ref.get(n) is not None:
            x = out[n].detach().double().cpu()
            if not torch.isfinite(x).all():
                fails.append(n + " is not finite")
            val, idx = worst((x - ref[n]).abs())
            loc = where_local(idx, nx, ny, w) if n == "lse" else "image %d head %d global row %d" % idx
            # lse is an fp32 number: beyond the bar, 8 roundings of its own size (it reaches 500 in the peaked cases)
            hold(n + ".abs", val, max(bars["lse"], 8 * 2.0 ** -24 * float(ref[n].abs().max())), loc)
    for n in ("o", "dq", "dk", "dv"):
        if not torch.isfinite(out[n].float()).all():
            fails.append(n + " is not finite")
    for n in ("dtable", "dg2l", "dg2g"):
        if n in ref:
            vals[n] = relerr(out[n], ref[n])
            if bias and not vals[n] < BIAS_BARS[variant]:
                fails.append("%s = %.3e (bar %.1e)" % (n, vals[n], BIAS_BARS[variant]))
    record(test, CASE_ID(case) + "/" + tag + "/" + variant, **vals)
    assert not fails, "\n".join(fails)


def variants_for(case, names=None):
    """the SIMT backward stops at D = 64; the 56 x 56 oracle is run for one dtype"""
    out = []
    for n in names or VARIANTS:
        if n == "simt_fp32" and case[2] > 64:
            continue
        if case[3] * case[4] > 2000 and VARIANTS[n][1] != BF16:
            continue
        out.append(n)
    return out


def expand(cases, names=None):
    return [pytest.param(c, n, id=CASE_ID(c) + "-" + n) for c in cases for n in variants_for(c, names)]


# --------------------------------------------------------------------------- (b) random inputs, localized bars
GEOMETRY_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, rpe
    (1, 3, 32, 56, 56, 1, 7, 0, 0, False),     # ViL-Small stage 1
    (2, 3, 64, 28, 28, 1, 7, 0, 0, False),     # ViL-Small stage 2
    (1, 2, 32, 15, 22, 1, 7, 0, 0, True),      # last chunk row and last chunk column hold one real row / column
    (1, 3, 32, 14, 7, 2, 7, 0, 0, False),      # one chunk column
    (2, 2, 64, 7, 7, 16, 7, 0, 0, True),       # a single chunk, 16 global tokens
    (1, 2, 32, 24, 40, 1, 8, 0, 0, True),      # w = 8: every piece has 64 real slots
    (1, 2, 32, 36, 25, 1, 12, 1, 0, True),     # w = 12 (short last piece), exact window with the table, padding
    (1, 2, 64, 31, 45, 1, 15, 1, 0, False),    # w = 15, exact window without the table
    (1, 2, 32, 26, 37, 2, 12, 0, 0, False),    # w = 12, padding in both directions
    (1, 1, 32, 35, 40, 1, 31, 0, 0, False),    # w = 31: the last chunk row holds 4 real rows, pieces below are skipped
    (1, 2, 16, 10, 9, 2, 4, -1, 0, True),      # cyclic chunks, 3 x 3 grid with padding, D = 16
    (1, 2, 16, 8, 5, 1, 4, -1, 0, False),      # cyclic chunks, 2 x 2 grid: chunks visited twice
    (1, 2, 32, 23, 33, 0, 7, 0, -1, False),    # own chunk only, no global tokens
    (1, 2, 32, 23, 33, 1, 7, 0, 3, True),      # random-shift modes
    (1, 2, 32, 23, 33, 1, 7, 0, 8, False),
    (1, 1, 48, 19, 17, 2, 7, 0, 0, True),      # D = 48 (zero-filled to 64)
    (1, 1, 72, 15, 13, 1, 7, 0, 0, False),     # D = 72 (zero-filled to 128)
    (1, 2, 128, 26, 24, 1, 12, 0, 0, True),    # D = 128, three pieces per chunk
]


@gpu
@pytest.mark.parametrize("case,variant", expand(GEOMETRY_CASES))
def test_rows_random_inputs(case, variant):
    t = make_inputs(case, seed=310)
    cfg = cfg_of(case)
    ref = oracle(t, cfg, VARIANTS[variant][1], ("geo",) + case)
    check("rows_random_inputs", "randn", run_kernels(t, cfg, variant), ref, case, variant)


DROP = (0.1, 0x5eed0000cafe, 1234)


def dropout_reference(t, case, dtype):
    """test_gpu_dropout's chunked fp64 reference with the exact keep mask of the call"""
    B, H, D, nx, ny, g, w, exact, mode, rpe = case[:10]
    keep, keep_g = tdrop.keep_tensors(DROP[1], DROP[2], DROP[0], B, H, nx, ny, w, g, mode)
    ref = tdrop.reference_run(t, cfg_of(case), dtype, keep, keep_g)
    return {n: (None if x is None else x.detach()) for n, x in ref.items()}


@gpu
@pytest.mark.parametrize("case,variant", expand([(1, 2, 32, 15, 13, 2, 7, 0, 0, True)], ["simt_fp32", "wgmma_bf16_f32out"]))
def test_rows_dropout(case, variant):
    t = make_inputs(case, seed=311)
    ref = dropout_reference(t, case, VARIANTS[variant][1])
    check("rows_dropout", "p0.1", run_kernels(t, cfg_of(case), variant, drop=DROP), ref, case, variant)


# --------------------------------------------------------------------------- (c) peaked and late-maximum scores
def hot_keys(case, target):
    """(Nloc,) the key each query gets as its dominant one, as an index into the call's N keys.
    target = ("glob", t): global key t for every row.
    target = ("off", dR, dC, slot): the key of the chunk at offset (dR, dC) from the query's chunk (wrapped when
    exact == -1), at the query's own position in the chunk (slot "same"), the chunk's first (slot "first": piece 0) or
    last position (slot "last": the short last piece); where that key is outside the image or masked for the query (read
    off the oracle's visit weights), the query's own position."""
    B, H, D, nx, ny, g, w, exact, mode, rpe = case[:10]
    nloc = nx * ny
    if target[0] == "glob":
        return torch.full((nloc,), target[1], dtype=torch.long)
    _, dR, dC, slot = target
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    PY = my * w
    vis = vo.visit_weights(nx, ny, w, exact, mode, None, 1)[0] > 0            # (Nloc, padded keys)
    i = torch.arange(nloc)
    r, c = i // ny, i % ny
    KR, KC = r // w + dR, c // w + dC
    if exact == -1:
        KR, KC = KR % mx, KC % my
    kr, kc = {"same": (r % w, c % w), "first": (0 * r, 0 * c), "last": (0 * r + w - 1, 0 * c + w - 1)}[slot]
    ar, ac = KR * w + kr, KC * w + kc
    ok = (KR >= 0) & (KR < mx) & (KC >= 0) & (KC < my) & (ar < nx) & (ac < ny)
    ok = ok & vis[i, (ar * PY + ac).clamp(0, vis.shape[1] - 1)]
    return g + torch.where(ok, ar * ny + ac, i)


def peak_through_qk(t, case, dtype, L, target):
    """k rows scaled to a common norm sqrt(D), then q_i += beta_i k_hot(i) / ||k_hot(i)|| with beta_i the smallest value
    for which the hot score exceeds every other visible score of the row by at least L (scores are linear in beta_i, and
    with equal norms the hot key gains the most).  Computed on the rounded k; the rounding of q moves the gap by O(L eps)."""
    B, H, D, nx, ny, g, w, exact, mode, rpe = case[:10]
    nx, ny, w, exact, mode, scale = cfg_of(case)
    t = dict(t)
    t["k"] = t["k"] / t["k"].norm(dim=-1, keepdim=True) * D ** 0.5
    t["kg"] = t["k"]
    k = t["k"].to(dtype).double()
    hot = hot_keys(case, target)                                              # (Nloc,)
    vis = vo.visit_weights(nx, ny, w, exact, mode, None, 1)[0] > 0            # (Nloc, P)
    kp = vo._pad_keys(k[:, :, g:], nx, ny, w)
    keys = torch.cat([k[:, :, :g], kp], dim=2)                                # global keys, then the padded grid
    seen = torch.cat([torch.ones(nx * ny, g, dtype=torch.bool), vis], dim=1)
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    hl = hot - g
    hot_col = torch.where(hot < g, hot, g + (hl // ny) * (my * w) + hl % ny)  # the hot key's column in `keys`
    kh = k[:, :, hot]                                                          # (B, H, Nloc, D)
    u = kh / kh.norm(dim=-1, keepdim=True)
    s0 = scale * torch.einsum("bhid,bhjd->bhij", t["q"].to(dtype).double(), keys)
    cj = scale * torch.einsum("bhid,bhjd->bhij", u, keys)                      # d score / d beta
    ii = torch.arange(nx * ny)
    s0h, ch = s0[:, :, ii, hot_col], cj[:, :, ii, hot_col]
    need = (L - (s0h[..., None] - s0)) / (ch[..., None] - cj).clamp_min(1e-9)
    other = seen[None, None].clone().expand_as(need).clone()
    other[:, :, ii, hot_col] = False
    beta = torch.where(other, need, torch.zeros_like(need)).amax(dim=-1).clamp_min(0.0)
    t["q"] = t["q"].to(dtype).double() + beta[..., None] * u
    return t, hot


def realized_gap(ref_lse, t, case, dtype, hot):
    """min over rows of -log(1 - P_hot) ~ the gap the oracle saw, via lse: hot score - lse = log P_hot"""
    B, H, D, nx, ny, g, w, exact, mode, rpe = case[:10]
    q, k = t["q"].to(dtype).double(), t["k"].to(dtype).double()
    sh = D ** -0.5 * (q * k[:, :, hot]).sum(-1)
    return sh, (sh - ref_lse)                                                  # hot score, log P_hot (<= 0)


def check_peaked(test, case, variant, t, tag, L, hot=None, floors=True, bias=False, backward=True):
    cfg = cfg_of(case)
    dtype = VARIANTS[variant][1]
    ref = oracle(t, cfg, dtype, (test, tag) + case)
    out = run_kernels(t, cfg, variant)
    g = case[5]
    check(test, tag, out, ref, case, variant, floors=peak_floors(t, cfg, variant, g) if floors else None, bias=bias,
          backward=backward)
    if hot is not None and L >= 100:
        # every other probability is below e^-L: o is the hot key's v row to the rounding of the output, lse the hot score
        sh, logp = realized_gap(ref["lse"], t, case, dtype, hot)
        assert float(logp.min()) > -1e-9, float(logp.min())
        vh = t["v"].to(dtype).double()[:, :, hot]
        f32 = VARIANTS[variant][2] or dtype == F32
        val, idx = worst(row_errors(out["o"], vh))
        record(test, CASE_ID(case) + "/" + tag + "/" + variant, o_vs_hot_v=val,
               lse_vs_hot_score=float((out["lse"].double().cpu() - sh).abs().max()))
        assert val < (1e-6 if f32 else 2.0 ** -8), (val, where_local(idx, case[3], case[4], case[6]))
        assert float((out["lse"].double().cpu() - sh).abs().max()) < max(1e-4, 8 * 2.0 ** -24 * float(sh.abs().max()))


PEAK_VARIANTS = ["simt_fp32", "wgmma_fp16_f32out", "wgmma_bf16_f32out", "wgmma_bf16"]
GAPS = [12, 40, 100]
PK_MODE0 = (1, 2, 32, 21, 21, 1, 7, 0, 0, False)        # 3 x 3 chunks: the centre chunk sees all nine offsets
PK_W12 = (1, 2, 32, 36, 36, 1, 12, 0, 0, False)         # 3 x 3 chunks of three pieces (64, 64, 16 keys)
PK_MODE3 = (1, 2, 32, 21, 21, 1, 7, 0, 3, False)        # the own chunk and the one above right
PK_CYCLIC = (1, 2, 16, 10, 9, 1, 4, -1, 0, False)       # 3 x 3 cyclic chunks with padding: edge chunks wrap
PK_GLOBAL = (1, 2, 32, 21, 21, 2, 7, 0, 0, False)
PK_GLOBAL2 = (1, 2, 32, 14, 14, 70, 7, 0, 0, False)     # the hot key in the second piece of global keys


def _peak_params():
    ps = []
    add = lambda name, case, target: ps.extend(
        pytest.param(case, target, L, v, id="%s-L%d-%s" % (name, L, v)) for L in GAPS for v in variants_for(case, PEAK_VARIANTS))
    for dR, dC in vo.OFFSETS9:
        add("mode0_off(%d,%d)" % (dR, dC), PK_MODE0, ("off", dR, dC, "same"))
    for dR, dC in ((-1, -1), (0, 0), (1, 1)):
        for slot in ("first", "last"):
            add("w12_off(%d,%d)_%s_piece" % (dR, dC, slot), PK_W12, ("off", dR, dC, slot))
    for dR, dC in vo.mode_offsets(3):
        add("mode3_off(%d,%d)" % (dR, dC), PK_MODE3, ("off", dR, dC, "same"))
    for dR, dC in ((-1, -1), (-1, 1), (0, 1), (1, 0), (1, 1)):
        add("cyclic_wrapped_off(%d,%d)" % (dR, dC), PK_CYCLIC, ("off", dR, dC, "same"))
    add("global_key_1_of_2", PK_GLOBAL, ("glob", 1))
    add("global_key_69_of_70", PK_GLOBAL2, ("glob", 69))
    return ps


@gpu
@pytest.mark.parametrize("case,target,L,variant", _peak_params())
def test_rows_peaked_through_q_and_k(case, target, L, variant):
    """one dominant key per row, placed in every offset of the walk, in the first and the last piece of a multi-piece
    chunk and among the global keys: the row maximum arrives first, last, or rises over several pieces"""
    tag = "%s_L%d" % ("_".join(str(x) for x in target), L)
    t, hot = peak_through_qk(make_inputs(case, seed=320), case, VARIANTS[variant][1], L, target)
    check_peaked("rows_peaked_through_q_and_k", case, variant, t, tag, L, hot)


PK_TABLE = (1, 2, 32, 21, 21, 2, 7, 0, 0, True)


def peak_through_table(t, case, L, what):
    """what = ("entry", dr, dc): the table entry of relative displacement (query - key) = (dr, dc) set to +L;
    ("band",): every entry with |dr| > 3 or |dc| > 3 set to -L (a soft mask);
    ("l2g", t, s): g2l[1][:, t] = s L (global key t hot / dead for every local row);
    ("g2l", a, s): g2l[0][:, a] = s L (every local key of global row a);  ("g2g", a, t, s): g2g[:, a, t] = s L"""
    w = case[6]
    t = dict(t)
    tw = 4 * w - 1
    for n in ("table", "g2l", "g2g"):
        t[n] = t[n].clone()
    if what[0] == "entry":
        t["table"][(what[1] + 2 * w - 1) * tw + what[2] + 2 * w - 1] = L
    elif what[0] == "band":
        d = torch.arange(tw) - (2 * w - 1)
        far = (d.abs()[:, None] > 3) | (d.abs()[None, :] > 3)
        t["table"][far.reshape(-1)] = -L
    elif what[0] == "l2g":
        t["g2l"][1, :, what[1]] = what[2] * L
    elif what[0] == "g2l":
        t["g2l"][0, :, what[1]] = what[2] * L
    else:
        t["g2g"][:, what[1], what[2]] = what[3] * L
    return t


TABLE_PEAKS = [("entry", 0, 0), ("entry", 7, 7), ("entry", -7, 7), ("entry", 3, -10), ("band",), ("l2g", 1, 1), ("l2g", 0, -1),
               ("g2l", 1, 1), ("g2g", 0, 1, 1), ("g2g", 1, 1, -1)]


@gpu
@pytest.mark.parametrize("variant", PEAK_VARIANTS)
@pytest.mark.parametrize("L", GAPS)
@pytest.mark.parametrize("what", TABLE_PEAKS, ids=lambda x: "_".join(str(y) for y in x))
def test_rows_peaked_through_the_bias(what, L, variant):
    t = peak_through_table(make_inputs(PK_TABLE, seed=321), PK_TABLE, L, what)
    check_peaked("rows_peaked_through_the_bias", PK_TABLE, variant, t, "%s_L%d" % ("_".join(str(x) for x in what), L), L)


@gpu
@pytest.mark.parametrize("variant", PEAK_VARIANTS)
@pytest.mark.parametrize("shift", [60, -60])
def test_rows_common_shift_of_all_scores(shift, variant):
    """every q of a head has a component 2 along one unit vector u, and k += c u: all scores of a row move together (by
    about `shift`, between a third and twice that from row to row).  o must not move, lse moves by the row's shift.
    The gradients are held on the SIMT family only: dq = scale sum_j dS_j k_j with sum_j dS_j = 0 cancels the common
    component c u of every k_j, and a dS rounded to bf16 / fp16 for the tensor cores leaves eps |dS| c of it behind."""
    case = (1, 2, 32, 21, 21, 2, 7, 0, 0, False)
    B, H, D = case[:3]
    t = make_inputs(case, seed=322)
    u = torch.nn.functional.normalize(t["q"].mean(dim=2, keepdim=True), dim=-1)
    t["q"] = t["q"] - (t["q"] * u).sum(-1, keepdim=True) * u + (2 + 0.3 * (t["q"] * u).sum(-1, keepdim=True)) * u
    t["k"] = t["k"] + shift / (2 * D ** -0.5) * u
    t["kg"] = t["k"]
    check_peaked("rows_common_shift_of_all_scores", case, variant, t, "shift%d" % shift, abs(shift) * 2, floors=False,
                 backward=variant == "simt_fp32")


# --------------------------------------------------------------------------- (d) fully masked leading pieces
MASKED_CASES = [
    # g = 0 and the exact window at w^2 > 64: no global piece in front, and the first 64 keys of the chunk row above are
    # further than w from every query of the lower part of a chunk
    (1, 2, 32, 34, 30, 0, 12, 1, 0, False),    # 3 x 3 chunks, padding in both directions
    (1, 2, 64, 40, 43, 0, 15, 1, 0, False),    # w = 15
    (1, 2, 32, 30, 34, 0, 12, 1, 0, True),     # with the bias table
    (1, 1, 128, 34, 30, 0, 12, 1, 0, False),   # D = 128
]


def masked_pieces(nx, ny, w, exact, mode):
    """From the reference's mask (vo.chunk_mask, columns in the reference's block order) and nothing else:
    empty[oi][p] (mx, my, w2) = real query rows for which every column of 64-key piece p of the chunk at offset oi is
    masked although that chunk lies in the image;  lead (mx, my, w2) = the index oi of the offset whose piece 0 is the
    first piece of a chunk in the image in that order and is wholly masked for the row, else -1."""
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    w2, offs = w * w, vo.mode_offsets(mode)
    mask = vo.chunk_mask(nx, ny, w, exact, mode)[0].expand(mx, my, w2, len(offs) * w2)
    l = torch.arange(w2)
    R, C = torch.arange(mx)[:, None, None], torch.arange(my)[None, :, None]
    real = ((R * w + l // w) < nx) & ((C * w + l % w) < ny)                    # (mx, my, w2)
    empty, lead, seen_first = [], torch.full((mx, my, w2), -1), torch.zeros(mx, my, 1, dtype=torch.bool)
    for oi, (dR, dC) in enumerate(offs):
        inside = (R + dR >= 0) & (R + dR < mx) & (C + dC >= 0) & (C + dC < my) if exact != -1 else torch.ones(mx, my, 1, dtype=torch.bool)
        per_piece = []
        for p in range((w2 + 63) // 64):
            cols = mask[..., oi * w2 + p * 64: oi * w2 + min(p * 64 + 64, w2)].all(dim=-1)
            per_piece.append(cols & real & inside)
        empty.append(per_piece)
        first_here = inside & ~seen_first
        lead = torch.where(first_here & per_piece[0], torch.full_like(lead, oi), lead)
        seen_first = seen_first | inside
    return empty, lead


@pytest.mark.parametrize("case", MASKED_CASES, ids=CASE_ID)
def test_masked_cases_have_rows_whose_leading_piece_is_wholly_masked(case):
    """CPU.  In the reference's block order the chunks of the row above come first.  (-1, -1) is the first offset inside
    the image for an interior chunk and (-1, 0) for a chunk of the first chunk column; for both the case has rows whose
    walk STARTS with a wholly masked piece: the running maximum is still -inf after it.  No other offset can lead with one:
    (-1, 1) is never the first inside the image, and a 64-key piece of (0, -1) spans the query's own rows and all w columns
    beside its chunk.  Every offset of the row above and, after the own chunk, of the row below has wholly masked pieces
    somewhere in the walk (the far rows of those chunks)."""
    nx, ny, w, exact, mode = case[3], case[4], case[6], case[7], case[8]
    empty, lead = masked_pieces(nx, ny, w, exact, mode)
    offs = vo.mode_offsets(mode)
    assert sorted(set(lead[lead >= 0].tolist())) == [offs.index((-1, -1)), offs.index((-1, 0))]
    for oi, (dR, dC) in enumerate(offs):
        if dR != 0:
            assert any(int(e.sum()) > 0 for e in empty[oi]), offs[oi]
    # the peaked variant below puts the row maximum behind them: rows with an empty leading piece see the chunk at (1, 1)
    hot = hot_keys(case, ("off", 1, 1, "same")).reshape(nx, ny)
    i = torch.arange(nx * ny).reshape(nx, ny)
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    lead_img = lead.reshape(mx, my, w, w).permute(0, 2, 1, 3).reshape(mx * w, my * w)[:nx, :ny]
    assert int(((hot != i) & (lead_img >= 0)).sum()) > 0


def test_no_other_case_without_global_tokens_has_such_a_row():
    """CPU: the gap this file closes.  With g >= 1 the walk starts with the global keys, which no row has masked; the
    g = 0 cases of the other attention files have no row with a wholly masked leading piece."""
    others = tpar.OP_CASES + tpar.TC_CASES + tpar.MODE_CASES + tpar.TC_BIG_CASES + tpar.F32OUT_CASES + thd.CASES + \
        [c[:10] for c in tdrop.DROP_CASES + thd.DROP_CASES]
    g0 = [c for c in others if c[5] == 0]
    assert len(g0) >= 4
    for c in g0:
        _, lead = masked_pieces(c[3], c[4], c[6], c[7], c[8])
        assert int((lead >= 0).sum()) == 0, c


@gpu
@pytest.mark.parametrize("case,variant", expand(MASKED_CASES))
def test_rows_masked_leading_pieces(case, variant):
    t = make_inputs(case, seed=330)
    cfg = cfg_of(case)
    ref = oracle(t, cfg, VARIANTS[variant][1], ("masked",) + case)
    check("rows_masked_leading_pieces", "randn", run_kernels(t, cfg, variant), ref, case, variant)


@gpu
@pytest.mark.parametrize("case,variant", expand(MASKED_CASES[:2], PEAK_VARIANTS))
@pytest.mark.parametrize("L", [40, 100])
def test_rows_masked_leading_pieces_then_the_maximum_in_the_last_chunk(case, variant, L):
    """the dominant key in the chunk at offset (1, 1), the last of the walk, behind the empty pieces"""
    t, hot = peak_through_qk(make_inputs(case, seed=331), case, VARIANTS[variant][1], L, ("off", 1, 1, "same"))
    check_peaked("rows_masked_leading_pieces_then_the_maximum_in_the_last_chunk", case, variant, t, "off_1_1_L%d" % L, L, hot)


# --------------------------------------------------------------------------- (e) more than 64 global tokens
MANY_GLOBAL_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, rpe, separate global weights
    (1, 2, 32, 14, 14, 64, 7, 0, 0, True, False),     # one full piece of global keys
    (1, 2, 32, 14, 14, 65, 7, 0, 0, False, True),     # the second piece holds one key
    (1, 2, 32, 14, 14, 65, 7, 0, 0, True, False),
    (1, 2, 32, 24, 24, 130, 12, 0, 0, True, True),    # three pieces, w = 12
    (1, 1, 64, 14, 14, 130, 7, 1, 0, False, False),   # exact window: global keys sit inside every row's window
]


@gpu
@pytest.mark.parametrize("case,variant", expand(MANY_GLOBAL_CASES))
def test_rows_more_than_64_global_tokens(case, variant):
    t = make_inputs(case, seed=340, sep=case[10])
    cfg = cfg_of(case)
    ref = oracle(t, cfg, VARIANTS[variant][1], ("glob",) + case)
    check("rows_more_than_64_global_tokens", "randn", run_kernels(t, cfg, variant), ref, case, variant)


@gpu
@pytest.mark.parametrize("case,variant", expand([(1, 2, 32, 14, 14, 65, 7, 0, 0, True, False)], ["simt_fp32", "wgmma_bf16_f32out"]))
def test_rows_more_than_64_global_tokens_dropout(case, variant):
    """the attn1 column of global key t is t: the second piece starts at column 64"""
    t = make_inputs(case, seed=341)
    ref = dropout_reference(t, case, VARIANTS[variant][1])
    check("rows_more_than_64_global_tokens_dropout", "p0.1", run_kernels(t, cfg_of(case), variant, drop=DROP), ref, case, variant)
