"""GPU parity tests (`pytest -m gpu`).  Everything goes through the C ABI
(libvil_attn.so via ctypes) and is compared with
  * the golden vectors generated from the unmodified reference (tests/golden/attn_*.pt), and
  * the CPU oracle (oracle/vil_oracle.py) on seeded inputs,
plus size-independent properties at the BASELINE shapes.

Tolerances (norm-relative, ||x - ref||_F / ||ref||_F, documented in DESIGN.md):
  fp32 I/O            : 1e-5 forward / 2e-5 backward  (BASELINE north_star 1e-5)
  fp16 I/O            : 1e-3 forward / 2e-3 backward  (north_star 1e-3)
  fp16 in, fp32 OUT   : 1e-3 forward AND backward     (north_star 1e-3; SURVEY.md section 8(c) protocol step 1: the
                        parity build VIL_FLAG_F32_OUT isolates the kernel-internal error - P / dS tensor-core operands,
                        fp32 accumulation - from the rounding of the stored result; `test_tcgen05_fp32_out_parity`)
  bf16 in, fp32 OUT   : 2e-3 forward AND backward     -- the quantisation of the P / dS operand to bf16 (8-bit mantissa,
                        rms 2^-9/sqrt(3) * O(1)) that any kernel feeding a bf16 tensor-core operand carries; wgmma takes
                        both operands in one element type, so P / dS have V's / K's type.  1e-3 is met in fp16.
  bf16 I/O            : 4e-3 forward / 8e-3 backward  -- the bf16 OUTPUT rounding alone is 1.65e-3 (BASELINE.md
                        section 5) and the reference module itself sits at 3.3e-3 / 6.8e-3 in bf16 (protocol step 2:
                        required <= the reference's own bf16 error; the measured values are logged beside the floor)
Every measured error is recorded (tests/util.py::record; written out when VIL_ERRORS_JSON names a file).
The test names keep the `tcgen05` of the tensor-core family they were written for; that family is the wgmma one now.
"""
import pytest
import torch

from oracle import vil_oracle as vo
from tests.util import attn_cases, load_attn, load_golden, load_state, record, relerr
from vision_longformer_b200 import (B200Long2DSCSelfAttention, MsViT, _lib, build_vil, vil_attention,
                                    vil_attention_raw_backward, vil_attention_raw_forward)

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {torch.float32: (1e-5, 2e-5), torch.float16: (1e-3, 2e-3), torch.bfloat16: (4e-3, 8e-3)}


# --------------------------------------------------------------------------- golden module parity
@pytest.mark.parametrize("name", attn_cases())
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_module_matches_reference_golden_fp32(name, impl):
    gold = load_attn(name)
    mod = B200Long2DSCSelfAttention(**gold["kwargs"]).to(DEV)
    load_state(mod, gold["state_dict"])
    mod.impl = impl
    pick = gold["picked_mode"]
    mod.train(pick is not None)
    if pick is not None:
        mod._pick_mode = lambda: pick
    x = gold["x"].to(DEV).requires_grad_(True)
    y = mod(x, gold["nx"], gold["ny"])
    (y * gold["gy"].to(DEV)).sum().backward()
    assert relerr(y, gold["y"]) < 1e-5
    assert relerr(x.grad, gold["dx"]) < 2e-5
    grads = {n: p.grad for n, p in mod.named_parameters()}
    for n, gref in gold["param_grads"].items():
        assert grads[n] is not None, n
        assert relerr(grads[n], gref) < 5e-5, n


@pytest.mark.parametrize("name", ["w7_g1_exact0_rpe", "w7_g1_exact1_rpe", "w8_g1_exact0_d32", "w7_g1_exact0_d64_28",
                                  "w4_g2_exact0_norpe_nosharew"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_module_matches_reference_golden_lowp(name, dtype):
    gold = load_attn(name)
    mod = B200Long2DSCSelfAttention(**gold["kwargs"]).to(DEV)
    load_state(mod, gold["state_dict"])
    mod = mod.to(dtype).eval()
    x = gold["x"].to(DEV, dtype).requires_grad_(True)
    y = mod(x, gold["nx"], gold["ny"])
    (y * gold["gy"].to(DEV, dtype)).sum().backward()
    # the Linears run in low precision here as well, so this is a loose end-to-end check
    assert relerr(y, gold["y"]) < 3e-2
    assert relerr(x.grad, gold["dx"]) < 6e-2


# --------------------------------------------------------------------------- op-level parity vs oracle
def make_inputs(B, H, D, nx, ny, g, w, rpe, seed=300, dtype=torch.float64):
    gen = torch.Generator().manual_seed(seed)       # the reference tests' seed
    N = g + nx * ny
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    t = dict(q=r(B, H, nx * ny, D), k=r(B, H, N, D), v=r(B, H, N, D), qg=r(B, H, max(g, 1), D)[:, :, :g],
             table=0.5 * r((4 * w - 1) ** 2, H) if rpe else None,
             g2l=0.5 * r(2, H, g) if (rpe and g) else None, g2g=0.5 * r(H, g, g) if (rpe and g) else None,
             go=r(B, H, nx * ny, D), gog=r(B, H, max(g, 1), D)[:, :, :g])
    return t


_ORACLE_CACHE = {}


def oracle_run(t, nx, ny, w, exact, mode, scale, dtype, key=None):
    """fp64 oracle on the values the kernel actually sees (inputs rounded to `dtype`)."""
    if key is not None and (key, dtype) in _ORACLE_CACHE:
        return _ORACLE_CACHE[(key, dtype)]
    out = _oracle_run(t, nx, ny, w, exact, mode, scale, dtype)
    if key is not None:
        _ORACLE_CACHE[(key, dtype)] = out
    return out


def _oracle_run(t, nx, ny, w, exact, mode, scale, dtype):
    rd = lambda x: None if x is None else x.to(dtype).double().requires_grad_(True)
    q, k, v, qg = rd(t["q"]), rd(t["k"]), rd(t["v"]), rd(t["qg"])
    table, g2l, g2g = [None if t[n] is None else t[n].float().double().requires_grad_(True) for n in ("table", "g2l", "g2g")]
    g = k.shape[2] - q.shape[2]
    o, og, lse, lse_g = vo.dense_attention(q, k, v, qg if g else None, k, v, table, g2l, g2g, nx=nx, ny=ny, w=w,
                                           exact=exact, mode=mode, scale=scale)
    go, gog = t["go"].to(dtype).double(), t["gog"].to(dtype).double()
    loss = (o * go).sum() + ((og * gog).sum() if g else 0)
    ins = [x for x in (q, k, v, qg if g else None, table, g2l, g2g) if x is not None]
    grads = torch.autograd.grad(loss, ins)
    names = [n for n, x in zip(("q", "k", "v", "qg", "table", "g2l", "g2g"), (q, k, v, qg if g else None, table, g2l, g2g)) if x is not None]
    return dict(o=o, og=og, lse=lse, lse_g=lse_g, **{"d" + n: gr for n, gr in zip(names, grads)})


def _heads(t, H, which=0, parts=1):
    B, T, C = t.shape
    return t.view(B, T, parts, H, C // (parts * H))[:, :, which].permute(0, 2, 1, 3)


def kernel_run(t, nx, ny, w, exact, mode, scale, dtype, impl, layout="contig", f32out=False, flags=0, drop=(0.0, 0, 0)):
    """One forward + backward through the C ABI.
    layout = "contig": contiguous (B,H,T,D) tensors;  "linear": the PRODUCTION layout - q / k / v are strided views of
    the `query` / `kv` Linear outputs ((B,N,H*D) with the global rows first, (B,N,2*H*D)), the output is head-merged
    (B,N,H*D), gradients are written into dq_all / dkv buffers of the same layouts (ops._heads; what bench.py and every
    module call runs).  f32out: VIL_FLAG_F32_OUT parity build (bf16/fp16 inputs, fp32 outputs).
    Separate global weights when t["kg"] / t["vg"] are not t["k"] / t["v"] (test_gpu_dropout.make_inputs): in the
    linear layout they are views of a `kv_global` output, and their gradients come back as dkg / dvg.
    drop = (p, seed, offset): attention dropout."""
    B, H, Nloc, D = t["q"].shape
    N = t["k"].shape[2]
    g = N - Nloc
    sep = g > 0 and t.get("kg") is not None and t["kg"] is not t["k"]
    odt = torch.float32 if f32out else dtype
    f32 = lambda x: None if x is None else x.to(DEV, torch.float32).contiguous()
    table, g2l, g2g = f32(t["table"]), f32(t["g2l"]), f32(t["g2g"])
    if f32out:
        flags |= _lib.VIL_FLAG_F32_OUT
    if layout == "contig":
        dev = lambda x: None if x is None else x.to(DEV, dtype).contiguous()
        q, k, v, qg = dev(t["q"]), dev(t["k"]), dev(t["v"]), dev(t["qg"])
        go, gog = dev(t["go"]), dev(t["gog"])
        o, og = torch.empty_like(q, dtype=odt), (torch.empty_like(qg, dtype=odt) if g else None)
        dq, dk, dv = torch.empty_like(q, dtype=odt), torch.empty_like(k, dtype=odt), torch.empty_like(v, dtype=odt)
        dqg = torch.empty_like(qg, dtype=odt) if g else None
        kg, vg, dkg, dvg = k, v, dk, dv
        if sep:
            kg, vg = dev(t["kg"]), dev(t["vg"])
            dkg, dvg = torch.empty_like(kg, dtype=odt), torch.empty_like(vg, dtype=odt)
    else:
        C = H * D
        q_all = torch.empty(B, N, C, device=DEV, dtype=dtype)
        kv = torch.empty(B, N, 2 * C, device=DEV, dtype=dtype)
        d_out = torch.empty(B, N, C, device=DEV, dtype=dtype)
        out = torch.full((B, N, C), float("nan"), device=DEV, dtype=odt)
        dq_all = torch.full((B, N, C), float("nan"), device=DEV, dtype=odt)
        dkv = torch.full((B, N, 2 * C), float("nan"), device=DEV, dtype=odt)
        q, qg = _heads(q_all, H)[:, :, g:], _heads(q_all, H)[:, :, :g]
        k, v = _heads(kv, H, 0, 2), _heads(kv, H, 1, 2)
        go, gog = _heads(d_out, H)[:, :, g:], _heads(d_out, H)[:, :, :g]
        q.copy_(t["q"]); k.copy_(t["k"]); v.copy_(t["v"]); go.copy_(t["go"])
        if g:
            qg.copy_(t["qg"]); gog.copy_(t["gog"])
        o, og = _heads(out, H)[:, :, g:], (_heads(out, H)[:, :, :g] if g else None)
        dq, dqg = _heads(dq_all, H)[:, :, g:], (_heads(dq_all, H)[:, :, :g] if g else None)
        dk, dv = _heads(dkv, H, 0, 2), _heads(dkv, H, 1, 2)
        kg, vg, dkg, dvg = k, v, dk, dv
        if sep:
            kvg = torch.empty(B, N, 2 * C, device=DEV, dtype=dtype)
            dkvg = torch.full((B, N, 2 * C), float("nan"), device=DEV, dtype=odt)
            kg, vg = _heads(kvg, H, 0, 2), _heads(kvg, H, 1, 2)
            kg.copy_(t["kg"]); vg.copy_(t["vg"])
            dkg, dvg = _heads(dkvg, H, 0, 2), _heads(dkvg, H, 1, 2)
    kw = dict(nx=nx, ny=ny, w=w, exact=exact, mode=mode, scale=scale, impl=impl, flags=flags,
              dropout_p=drop[0], dropout_seed=drop[1], dropout_offset=drop[2])
    lse, lse_g = vil_attention_raw_forward(q, k, v, qg if g else None, kg if g else None, vg if g else None, table, g2l,
                                           g2g, o, og, **kw)
    fam_f = _lib.last_impl()
    zl = lambda x: None if x is None else torch.zeros_like(x)
    dt, dgl, dgg = zl(table), zl(g2l), zl(g2g)
    vil_attention_raw_backward(q, k, v, qg if g else None, kg if g else None, vg if g else None, table, g2l, g2g, o, og,
                               lse, lse_g, go, gog if g else None, dq, dk, dv, dqg,
                               dkg if g else None, dvg if g else None, dt, dgl, dgg, **kw)
    torch.cuda.synchronize()
    out_d = dict(o=o, og=og, lse=lse, lse_g=lse_g, dq=dq, dk=dk, dv=dv, dqg=dqg, dtable=dt, dg2l=dgl, dg2g=dgg)
    if sep:
        out_d.update(dkg=dkg, dvg=dvg)
    return out_d, fam_f, _lib.last_impl()


CASE_ID = lambda c: "B%d_H%d_D%d_%dx%d_g%d_w%d_e%d_m%d_%s" % (c[:9] + ("rpe" if c[9] else "nob",))


def check_against(out, ref, g, rpe, tf, tb, tbias, test, case, tag):
    """assert + record every output of one run"""
    errs = dict(o=relerr(out["o"], ref["o"]), lse=relerr(out["lse"], ref["lse"]))
    for n in ("dq", "dk", "dv"):
        errs[n] = relerr(out[n], ref[n])
    if g:
        errs["og"] = relerr(out["og"], ref["og"])
        errs["dqg"] = relerr(out["dqg"], ref["dqg"])
    if rpe:
        errs["dtable"] = relerr(out["dtable"], ref["dtable"])
        if g:
            errs["dg2l"] = relerr(out["dg2l"], ref["dg2l"])
            errs["dg2g"] = relerr(out["dg2g"], ref["dg2g"])
    record(test, CASE_ID(case) + "/" + tag, **errs)
    assert errs["o"] < tf, errs
    assert errs["lse"] < 1e-4, errs
    for n in ("dq", "dk", "dv"):
        assert errs[n] < tb, (n, errs)
    if g:
        assert errs["og"] < tf and errs["dqg"] < tb, errs
    if rpe:
        assert errs["dtable"] < tbias, errs
        if g:
            assert errs["dg2l"] < tbias and errs["dg2g"] < tbias, errs


OP_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, rpe
    (2, 3, 32, 14, 14, 1, 7, 0, 0, True),
    (2, 3, 32, 14, 14, 1, 7, 0, 0, False),
    (1, 2, 64, 21, 14, 1, 7, 0, 0, True),
    (2, 2, 32, 16, 24, 1, 8, 0, 0, False),
    (1, 3, 32, 19, 17, 1, 7, 0, 0, True),      # padding in both directions
    (1, 2, 32, 14, 14, 1, 7, 1, 0, True),      # exact window
    (1, 2, 64, 15, 13, 2, 7, 1, 0, False),
    (1, 2, 32, 15, 13, 2, 7, 0, 3, True),      # random-shift modes
    (1, 2, 32, 15, 13, 1, 7, 0, 8, False),
    (1, 2, 32, 15, 13, 1, 7, 0, -1, True),
    (1, 2, 16, 10, 9, 3, 4, -1, 0, True),      # cyclic chunks + padding quirk
    (1, 2, 16, 8, 5, 1, 4, -1, 0, False),      # mx, my <= 2: chunks visited twice
    (1, 1, 48, 14, 14, 1, 7, 0, 0, True),      # ViL-Tiny stage-1 head dim
    (1, 2, 32, 24, 24, 1, 12, 0, 0, True),     # w^2 > 64: multi-piece chunks
    (1, 2, 32, 30, 17, 1, 15, 1, 0, False),
    (1, 2, 32, 12, 12, 0, 6, 0, 0, True),      # no global tokens
    (1, 2, 32, 12, 12, 8, 6, 0, 0, True),      # g = 8
]


@pytest.mark.parametrize("case", OP_CASES, ids=CASE_ID)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_op_matches_oracle(case, dtype, impl):
    B, H, D, nx, ny, g, w, exact, mode, rpe = case
    t = make_inputs(B, H, D, nx, ny, g, w, rpe)
    scale = D ** -0.5
    ref = oracle_run(t, nx, ny, w, exact, mode, scale, dtype, key=case)
    out, fam_f, fam_b = kernel_run(t, nx, ny, w, exact, mode, scale, dtype, impl)
    tf, tb = TOL[dtype]
    # bias gradients are sums of dS over thousands of (query, key) pairs with heavy cancellation; in low
    # precision they inherit the rounding of the STORED o (delta = dO.o uses the bf16/fp16 output, exactly as
    # the reference's autograd does), hence the looser bound there.
    tbias = {torch.float32: 1e-4, torch.float16: 1e-2, torch.bfloat16: 5e-2}[dtype]
    check_against(out, ref, g, rpe, tf, tb, tbias, "op_matches_oracle", case, "%s/%s/%s+%s" % (
        {torch.float32: "fp32", torch.bfloat16: "bf16", torch.float16: "fp16"}[dtype], impl, fam_f, fam_b))


TC_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, rpe  -- all must be served by the tensor-core (wgmma) family
    (2, 3, 32, 56, 56, 1, 7, 0, 0, False),     # ViL-Small stage 1 (rpe off, published arch)
    (2, 3, 64, 28, 28, 1, 7, 0, 0, False),     # ViL-Small stage 2
    (2, 3, 32, 28, 28, 1, 7, 0, 0, True),
    (1, 2, 64, 21, 35, 1, 7, 0, 0, True),      # odd number of chunk columns (slot B missing in the last pair)
    (1, 1, 48, 19, 17, 2, 7, 0, 0, True),      # D=48 (padded to 64 by TMA), padding rows/cols, 2 global tokens
    (1, 2, 32, 24, 40, 1, 8, 0, 0, True),      # w=8: full 64-row slots
    (1, 2, 64, 18, 15, 1, 6, 1, 0, True),      # w=6, exact window, padding
    (1, 2, 32, 20, 22, 1, 7, 1, 0, False),     # exact window without rpe (mask-only table)
    (1, 2, 32, 22, 20, 1, 7, 0, 5, True),      # random-shift mode
    (1, 2, 32, 22, 20, 0, 7, 0, -1, False),    # own chunk only, no global tokens
    (1, 2, 16, 15, 29, 16, 7, 0, 0, True),     # D=16 (padded to 32), 16 global tokens
    (1, 3, 32, 14, 7, 1, 7, 0, 0, False),      # one chunk column only (no slot B anywhere), 2 chunk rows
    (2, 2, 64, 7, 7, 8, 7, 0, 0, False),       # a single chunk, 8 global tokens
    (1, 3, 32, 64, 64, 1, 8, 0, 0, False),     # w = 8 without rpe (Medium-Deep-384 stage-1 window on a smaller grid)
]
# every random-shift mode (slidingchunk_2d.py:15-24) and the own-chunk mode, with padding, odd chunk-column count
MODE_CASES = [(1, 2, 32, 23, 33, 1, 7, 0, m, bool(m % 2)) for m in (-1, 1, 2, 3, 4, 5, 6, 7, 8)]
DT_NAME = {torch.float32: "fp32", torch.bfloat16: "bf16", torch.float16: "fp16"}


@pytest.mark.parametrize("case", TC_CASES + MODE_CASES, ids=CASE_ID)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("layout", ["contig", "linear"])
def test_tcgen05_matches_oracle(case, dtype, layout):
    """forward + backward on the tensor-core family, contiguous AND production (strided Linear-output) layouts, at the
    kernel tolerance of the dtype"""
    B, H, D, nx, ny, g, w, exact, mode, rpe = case
    t = make_inputs(B, H, D, nx, ny, g, w, rpe, seed=301)
    scale = D ** -0.5
    ref = oracle_run(t, nx, ny, w, exact, mode, scale, dtype, key=("tc",) + case)
    out, fam_f, fam_b = kernel_run(t, nx, ny, w, exact, mode, scale, dtype, "auto", layout=layout)
    assert fam_f == "wgmma", fam_f            # no silent fallback
    assert fam_b == "wgmma", fam_b            # incl. the bias-table-gradient variant of the dQ pass
    tf, tb = TOL[dtype]
    tbias = {torch.float16: 1e-2, torch.bfloat16: 5e-2}[dtype]
    check_against(out, ref, g, rpe, tf, tb, tbias, "tcgen05_matches_oracle", case, DT_NAME[dtype] + "/" + layout)
    if layout == "linear":                      # every row of the gradient buffers has been written
        for n in ("o", "dq", "dk", "dv"):
            assert torch.isfinite(out[n].float()).all(), n


@pytest.mark.parametrize("case", [TC_CASES[0], TC_CASES[1], TC_CASES[2], TC_CASES[4], TC_CASES[7], TC_CASES[8]], ids=CASE_ID)
def test_tcgen05_unfused_pipeline_matches_oracle(case):
    """VIL_FLAG_UNFUSED is accepted by every family and must not change the result or add launches."""
    B, H, D, nx, ny, g, w, exact, mode, rpe = case
    dtype = torch.bfloat16
    t = make_inputs(B, H, D, nx, ny, g, w, rpe, seed=301)
    scale = D ** -0.5
    ref = oracle_run(t, nx, ny, w, exact, mode, scale, dtype, key=("tc",) + case)
    before = _lib.launch_count()
    out, fam_f, fam_b = kernel_run(t, nx, ny, w, exact, mode, scale, dtype, "auto", layout="linear", flags=_lib.VIL_FLAG_UNFUSED)
    n_unfused = _lib.launch_count() - before
    assert fam_f == "wgmma" and fam_b == "wgmma"
    tf, tb = TOL[dtype]
    check_against(out, ref, g, rpe, tf, tb, 5e-2, "tcgen05_unfused_pipeline_matches_oracle", case, "bf16/linear")
    before = _lib.launch_count()
    kernel_run(t, nx, ny, w, exact, mode, scale, dtype, "auto", layout="linear")
    n_fused = _lib.launch_count() - before
    record("launches_fwd_plus_bwd", CASE_ID(case), fused=n_fused, unfused=n_unfused)
    assert n_fused <= n_unfused


TC_BIG_CASES = [
    # chunk sizes > 8: chunks of more than 64 tokens are walked in 64-token pieces
    (1, 2, 32, 24, 24, 1, 12, 0, 0, True),     # Medium-Deep-384 stage-2 window
    (1, 2, 32, 26, 37, 2, 12, 0, 3, True),     # padding, 2 global tokens, random-shift mode
    (1, 2, 64, 30, 17, 1, 15, 1, 0, False),    # exact window (mask-only table), short last piece
    (1, 1, 48, 15, 15, 1, 15, 0, 0, True),     # single chunk
    (1, 1, 32, 62, 40, 1, 31, 0, 0, False),    # w = 31: 16 pieces per chunk, padding
    (2, 2, 32, 36, 25, 1, 12, 0, 0, False),    # 3 x 3 chunks, padding
    (1, 2, 64, 31, 45, 2, 15, 0, 6, False),    # random-shift mode, D = 64
    (1, 3, 64, 48, 48, 1, 12, 0, 0, False),    # Medium-Deep-384 stage 2 as published (48x48 tokens, w = 12, D = 64)
    # heavy zero padding of the last chunk row (config-5 sweep: 27 / 29 of 31 rows): pieces below the image are skipped
    (1, 1, 32, 35, 40, 1, 31, 0, 0, False),    # 2 chunk rows, the second holds 4 real rows: 2 of its 16 pieces exist
    (1, 2, 64, 33, 20, 1, 15, 0, 0, False),    # 3 chunk rows, the last holds 3 real rows: 1 of its 4 pieces exists
    (1, 1, 32, 35, 62, 2, 31, 0, 7, False),    # same with the random-shift neighbour below
]


@pytest.mark.parametrize("case", TC_BIG_CASES, ids=CASE_ID)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("layout", ["contig", "linear"])
def test_tcgen05_big_window_matches_oracle(case, dtype, layout):
    B, H, D, nx, ny, g, w, exact, mode, rpe = case
    t = make_inputs(B, H, D, nx, ny, g, w, rpe, seed=302)
    scale = D ** -0.5
    ref = oracle_run(t, nx, ny, w, exact, mode, scale, dtype, key=("tcbig",) + case)
    out, fam_f, fam_b = kernel_run(t, nx, ny, w, exact, mode, scale, dtype, "auto", layout=layout)
    assert fam_f == "wgmma" and fam_b == "wgmma", (fam_f, fam_b)     # incl. the bias-table gradient
    tf, tb = TOL[dtype]
    tbias = {torch.float16: 1e-2, torch.bfloat16: 5e-2}[dtype]
    check_against(out, ref, g, rpe, tf, tb, tbias, "tcgen05_big_window_matches_oracle", case, DT_NAME[dtype] + "/" + layout)


# --------------------------------------------------------------------------- the 1e-3 bar: fp32-output parity build
F32OUT_CASES = [
    (2, 3, 32, 56, 56, 1, 7, 0, 0, False),     # ViL-Small stage 1 (BASELINE config 2 shape S1, batch reduced)
    (2, 3, 64, 28, 28, 1, 7, 0, 0, False),     # ViL-Small stage 2 (S2)
    (1, 3, 32, 56, 56, 1, 7, 1, 0, False),     # S1 with the exact (2w+1)^2 window
    (1, 3, 32, 28, 28, 1, 7, 0, 0, True),      # rpe on (bias-gradient variant of pass 1)
    (1, 3, 32, 64, 64, 1, 8, 0, 0, False),     # Medium-Deep-384 stage-1 window (w = 8)
    (1, 3, 64, 48, 48, 1, 12, 0, 0, False),    # Medium-Deep-384 stage 2 (48x48 tokens, w = 12)
    (1, 2, 32, 23, 33, 2, 7, 0, 3, False),     # random-shift mode, padding, 2 global tokens
]


@pytest.mark.parametrize("case", F32OUT_CASES, ids=CASE_ID)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("layout", ["contig", "linear"])
def test_tcgen05_fp32_out_parity(case, dtype, layout):
    """north_star bar on the tensor-core kernels: bf16/fp16-valued inputs, fp32 outputs (VIL_FLAG_F32_OUT), fp64 oracle on the
    same values.  fp16: 1e-3 forward AND backward.  bf16: 2e-3 - the bf16 quantisation of the P / dS tensor-core operand
    (see the module docstring); the measured values are recorded.  The production (bf16/fp16-output) run of the same case
    is recorded beside it with the output-rounding floor (1.65e-3 for bf16, BASELINE.md section 5)."""
    B, H, D, nx, ny, g, w, exact, mode, rpe = case
    t = make_inputs(B, H, D, nx, ny, g, w, rpe, seed=303)
    scale = D ** -0.5
    ref = oracle_run(t, nx, ny, w, exact, mode, scale, dtype, key=("f32out",) + case)
    out, fam_f, fam_b = kernel_run(t, nx, ny, w, exact, mode, scale, dtype, "auto", layout=layout, f32out=True)
    assert fam_f == "wgmma" and fam_b == "wgmma", (fam_f, fam_b)
    for n in ("o", "dq", "dk", "dv"):
        assert out[n].dtype == torch.float32
    bar = 1e-3 if dtype == torch.float16 else 2e-3
    check_against(out, ref, g, rpe, bar, bar, 2e-2, "tcgen05_fp32_out_parity", case, DT_NAME[dtype] + "/" + layout + "/fp32out")
    if layout == "contig":
        prod, _, _ = kernel_run(t, nx, ny, w, exact, mode, scale, dtype, "auto", layout=layout)
        record("tcgen05_fp32_out_parity", CASE_ID(case) + "/" + DT_NAME[dtype] + "/production_out",
               o=relerr(prod["o"], ref["o"]), dq=relerr(prod["dq"], ref["dq"]), dk=relerr(prod["dk"], ref["dk"]),
               dv=relerr(prod["dv"], ref["dv"]),
               rounding_floor_of_the_output_dtype=relerr(ref["o"].to(dtype), ref["o"]))


def test_autograd_function_on_strided_linear_outputs():
    """q / kv consumed in place from the Linear layouts, output produced head-merged; separate global weights."""
    torch.manual_seed(5)
    B, H, D, nx, ny, g, w = 2, 3, 32, 15, 14, 2, 7
    C, N = H * D, g + nx * ny
    mk = lambda *s: torch.randn(*s, dtype=torch.float64)
    q_all, qg_all, kv, kvg = mk(B, nx * ny, C), mk(B, g, C), mk(B, N, 2 * C), mk(B, N, 2 * C)
    table, g2l, g2g = 0.3 * mk((4 * w - 1) ** 2, H), 0.3 * mk(2, H, g), 0.3 * mk(H, g, g)
    gy = mk(B, N, C)
    ins64 = [x.clone().requires_grad_(True) for x in (q_all, kv, qg_all, kvg, table, g2l, g2g)]
    hd = lambda t, i=0, p=1: t.view(B, t.shape[1], p, H, D)[:, :, i].permute(0, 2, 1, 3)
    o, og, _, _ = vo.dense_attention(hd(ins64[0]), hd(ins64[1], 0, 2), hd(ins64[1], 1, 2), hd(ins64[2]),
                                     hd(ins64[3], 0, 2), hd(ins64[3], 1, 2), ins64[4], ins64[5], ins64[6],
                                     nx=nx, ny=ny, w=w, exact=0, mode=0, scale=D ** -0.5)
    y_ref = torch.cat([og.transpose(1, 2).reshape(B, g, C), o.transpose(1, 2).reshape(B, nx * ny, C)], dim=1)
    g_ref = torch.autograd.grad((y_ref * gy).sum(), ins64)
    ins = [x.to(DEV, torch.float32).requires_grad_(True) for x in (q_all, kv, qg_all, kvg, table, g2l, g2g)]
    y = vil_attention(ins[0], ins[1], ins[2], ins[3], ins[4], ins[5], ins[6], num_heads=H, nx=nx, ny=ny, w=w, nglo=g,
                      exact=0, mode=0, scale=D ** -0.5)
    grads = torch.autograd.grad((y * gy.to(DEV, torch.float32)).sum(), ins)
    assert relerr(y, y_ref) < 1e-5
    for a, b in zip(grads, g_ref):
        assert relerr(a, b) < 3e-5


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_autograd_function_separate_global_weights_on_tcgen05(dtype):
    """sharew=False in low precision: the global queries see their own kv_global tensors (global-token kernels next to
    the tensor-core local kernels)."""
    torch.manual_seed(6)
    B, H, D, nx, ny, g, w = 2, 3, 32, 21, 14, 2, 7
    C, N = H * D, g + nx * ny
    mk = lambda *s: torch.randn(*s, dtype=torch.float64)
    rd = lambda t: t.to(dtype).double()
    q_all, qg_all, kv, kvg = rd(mk(B, nx * ny, C)), rd(mk(B, g, C)), rd(mk(B, N, 2 * C)), rd(mk(B, N, 2 * C))
    gy = rd(mk(B, N, C))
    ins64 = [x.clone().requires_grad_(True) for x in (q_all, kv, qg_all, kvg)]
    hd = lambda t, i=0, p=1: t.view(B, t.shape[1], p, H, D)[:, :, i].permute(0, 2, 1, 3)
    o, og, _, _ = vo.dense_attention(hd(ins64[0]), hd(ins64[1], 0, 2), hd(ins64[1], 1, 2), hd(ins64[2]),
                                     hd(ins64[3], 0, 2), hd(ins64[3], 1, 2), None, None, None,
                                     nx=nx, ny=ny, w=w, exact=0, mode=0, scale=D ** -0.5)
    y_ref = torch.cat([og.transpose(1, 2).reshape(B, g, C), o.transpose(1, 2).reshape(B, nx * ny, C)], dim=1)
    g_ref = torch.autograd.grad((y_ref * gy).sum(), ins64)
    ins = [x.to(DEV, dtype).requires_grad_(True) for x in (q_all, kv, qg_all, kvg)]
    y = vil_attention(ins[0], ins[1], ins[2], ins[3], None, None, None, num_heads=H, nx=nx, ny=ny, w=w, nglo=g,
                      exact=0, mode=0, scale=D ** -0.5)
    assert _lib.last_impl() == "wgmma"
    grads = torch.autograd.grad((y * gy.to(DEV, dtype)).sum(), ins)
    assert _lib.last_impl() == "wgmma"
    tf, tb = TOL[dtype]
    errs = dict(y=relerr(y, y_ref), **{n: relerr(a, b) for n, a, b in zip(("dq", "dkv", "dqg", "dkvg"), grads, g_ref)})
    record("autograd_function_separate_global_weights_on_tcgen05", DT_NAME[dtype], **errs)
    assert errs["y"] < tf and all(errs[n] < tb for n in ("dq", "dkv", "dqg", "dkvg")), errs


# --------------------------------------------------------------------------- error behaviour
def test_errors_mirror_reference():
    q = torch.randn(1, 2, 49, 32, device=DEV)
    k = torch.randn(1, 2, 50, 32, device=DEV)
    o, og = torch.empty_like(q), torch.empty(1, 2, 1, 32, device=DEV)
    with pytest.raises(ValueError, match="exact"):
        vil_attention_raw_forward(q, k, k, k[:, :, :1], k, k, None, None, None, o, og, nx=7, ny=7, w=7, exact=2)
    with pytest.raises(ValueError):
        vil_attention_raw_forward(q, k, k, k[:, :, :1], k, k, None, None, None, o, og, nx=7, ny=7, w=7, exact=1, mode=2)
    with pytest.raises(AssertionError, match="Global dimension"):
        vil_attention_raw_forward(q, k, k, k[:, :, :1], k, k, None, None, None, o, og, nx=6, ny=7, w=7)
    with pytest.raises(RuntimeError, match="no CPU"):
        vil_attention_raw_forward(q.cpu(), k.cpu(), k.cpu(), None, None, None, None, None, None, o.cpu(), None,
                                  nx=7, ny=7, w=7)


# --------------------------------------------------------------------------- properties at BASELINE shapes
@pytest.mark.parametrize("shape", [(8, 3, 32, 56, 56), (8, 3, 64, 28, 28)], ids=["S1", "S2"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_full_size_properties(shape, dtype):
    """ViL-Small stage-1 / stage-2 shapes (BASELINE config 2; batch reduced to 8, the kernel is batch-independent):
    (1) rows of P sum to one: V = 1 -> O = 1;  (2) linearity in V;  (3) batch independence;
    (4) dV column sums equal dO column sums (sum_j dV_j = sum_i dO_i because P rows sum to 1);
    (5) the two kernel families agree where both apply."""
    B, H, D, nx, ny = shape
    w, g = 7, 1
    N = g + nx * ny
    gen = torch.Generator(device=DEV).manual_seed(300)
    r = lambda *s: torch.randn(*s, generator=gen, device=DEV, dtype=torch.float32).to(dtype)
    q, k, v1, v2 = r(B, H, nx * ny, D), r(B, H, N, D), r(B, H, N, D), r(B, H, N, D)
    qg = r(B, H, g, D)
    kw = dict(nx=nx, ny=ny, w=w, exact=0, mode=0, scale=D ** -0.5)

    def fwd(qq, kk, vv, qgg, impl="auto"):
        o, og = torch.empty_like(qq), torch.empty_like(qgg)
        lse, lse_g = vil_attention_raw_forward(qq, kk, vv, qgg, kk, vv, None, None, None, o, og, impl=impl, **kw)
        return o, og, lse, lse_g

    ones = torch.ones_like(v1)
    o1, og1, _, _ = fwd(q, k, ones, qg)
    tol = 1e-5 if dtype == torch.float32 else 8e-3
    assert (o1.float() - 1).abs().max() < tol and (og1.float() - 1).abs().max() < tol
    oa, _, lse_a, _ = fwd(q, k, v1, qg)
    ob, _, _, _ = fwd(q, k, v2, qg)
    oc, _, _, _ = fwd(q, k, (v1.float() + v2.float()).to(dtype), qg)
    assert relerr(oc, oa.float() + ob.float()) < (2e-5 if dtype == torch.float32 else 1e-2)
    o_half, _, lse_h, _ = fwd(q[:2], k[:2], v1[:2], qg[:2])
    assert torch.equal(o_half, oa[:2]) and torch.equal(lse_h, lse_a[:2])
    o_s, _, lse_s, _ = fwd(q, k, v1, qg, impl="simt")
    assert relerr(oa, o_s) < (1e-5 if dtype == torch.float32 else 6e-3)
    assert relerr(lse_a, lse_s) < 1e-3

    go, gog = r(B, H, nx * ny, D), r(B, H, g, D)
    o, og, lse, lse_g = fwd(q, k, v1, qg)
    dq, dk, dv, dqg = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v1), torch.empty_like(qg)
    vil_attention_raw_backward(q, k, v1, qg, k, v1, None, None, None, o, og, lse, lse_g, go, gog, dq, dk, dv, dqg,
                               dk, dv, None, None, None, **kw)
    lhs = dv.float().sum(dim=2)
    rhs = go.float().sum(dim=2) + gog.float().sum(dim=2)
    assert relerr(lhs, rhs) < (2e-5 if dtype == torch.float32 else 2e-2)
    # dK columns: sum_j dk_j . anything is not conserved, but sum over keys of dS is zero per query row:
    # check via dq . q  +  ... skipped; gradient parity is covered by test_op_matches_oracle.


# --------------------------------------------------------------------------- MsViT end to end
@pytest.mark.parametrize("name", ["tiny_rpe", "tiny_ape"])
def test_msvit_end_to_end_fp32(name):
    gold = load_golden(f"msvit_{name}.pt")
    net = MsViT(**gold["kwargs"]).to(DEV).eval()
    load_state(net, gold["state_dict"])
    x = gold["x"].to(DEV).requires_grad_(True)
    with torch.backends.cudnn.flags(allow_tf32=False):
        y = net(x)
        (y * gold["gy"].to(DEV).float()).sum().backward()
    assert relerr(y, gold["y"]) < 2e-5
    assert relerr(x.grad, gold["dx"]) < 1e-4


def test_msvit_vil_small_bf16_on_tcgen05():
    """ViL-Small 224 (the BASELINE config 3 network) under bf16 autocast: every longformer stage must run on the tensor-core
    family (production strided layouts, fused LayerNorm), logits and input gradient against the same network in fp32
    on the CPU with the oracle attention plugged in."""
    from oracle.vil_oracle import OracleLong2DSCSelfAttention
    torch.manual_seed(0)
    kw = dict(img_size=224, num_classes=100, drop_path_rate=0.0)
    ref = build_vil("vil_small", attn_cls=OracleLong2DSCSelfAttention, fused_norm=False, **kw).eval()
    net = build_vil("vil_small", **kw).to(DEV).eval()
    net.load_state_dict(ref.state_dict())
    x = torch.randn(2, 3, 224, 224)
    gy = torch.randn(2, 100)
    xr = x.clone().requires_grad_(True)
    yr = ref(xr)
    (yr * gy).sum().backward()
    fams = []
    hooks = [m.register_forward_hook(lambda *_: fams.append(_lib.last_impl())) for m in net.modules()
             if isinstance(m, B200Long2DSCSelfAttention)]
    xg = x.to(DEV).requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = net(xg)
    (y.float() * gy.to(DEV)).sum().backward()
    torch.cuda.synchronize()
    for h in hooks:
        h.remove()
    assert fams == ["wgmma"] * 3, fams                      # 1 stage-1 + 2 stage-2 longformer layers
    assert _lib.last_impl() == "wgmma"                      # ... and their backward
    e_y, e_dx = relerr(y, yr), relerr(xg.grad, xr.grad)
    record("msvit_vil_small_bf16_on_tcgen05", "vil_small_224_B2", logits=e_y, dx=e_dx)
    assert y.dtype == torch.bfloat16 or y.dtype == torch.float32
    assert e_y < 3e-2 and e_dx < 8e-2, (e_y, e_dx)            # a 12-layer bf16 network against fp32


def test_reset_vil_mode_switches_the_kernel_mode():
    """VIL_MODE_SWITCH (run_experiment.py:223-230 -> MsViT.reset_vil_mode, msvit.py:532-541): mode > 0 draws one of the 8
    neighbour chunks per forward in training and is 0 in eval; flipping it back to 0 restores the 9-chunk attention."""
    torch.manual_seed(1)
    net = build_vil("l1,h2,d64,n1,s1,g1,p4,f7_l2,h2,d64,n1,s0,g1,p2,f7_l3,h2,d64,n1,s0,g0,p2,f7", img_size=112,
                    num_classes=10, drop_path_rate=0.0, mode=0).to(DEV)
    attn = net.layer1[1].attn
    x = torch.randn(2, 3, 112, 112, device=DEV)
    net.eval()
    y0 = net(x)
    net.reset_vil_mode(1)
    assert attn.mode == 1
    assert torch.equal(net(x), y0)                            # eval: always mode 0 whatever self.mode is
    net.train()
    picked = []
    orig = attn._pick_mode
    attn._pick_mode = lambda: picked.append(orig()) or picked[-1]
    y1 = net(x)
    assert picked and 1 <= picked[0] <= 8 and not torch.allclose(y1, y0)
    net.reset_vil_mode(-1)
    assert attn.mode == -1 and attn._pick_mode() == -1
    net.reset_vil_mode(0)
    attn._pick_mode = orig
    net.eval()
    assert torch.equal(net(x), y0)


def test_only_glo_branch_matches_dense_restatement():
    """ONLY_GLOBAL ablation (longformer2d.py:130-132,189-192): local queries attend to the global tokens only."""
    torch.manual_seed(2)
    B, nx, ny, g, H, D = 2, 9, 8, 4, 2, 16
    C = H * D
    mod = B200Long2DSCSelfAttention(C, num_heads=H, qkv_bias=True, w=4, nglo=g, only_glo=True, sharew=False, rpe=True).to(DEV)
    x = torch.randn(B, g + nx * ny, C, device=DEV)
    y = mod(x, nx, ny)
    with torch.no_grad():
        hd = lambda t: t.reshape(B, -1, H, D).transpose(1, 2)
        q = hd(mod.query(x[:, g:])) * mod.scale
        k, v = [hd(t) for t in mod.kv(x).chunk(2, dim=-1)]
        x1 = mod.proj(((q @ k[:, :, :g].transpose(-1, -2)).softmax(-1) @ v[:, :, :g]).transpose(1, 2).reshape(B, nx * ny, C))
        qg = hd(mod.query_global(x[:, :g])) * mod.scale
        kg, vg = [hd(t) for t in mod.kv_global(x).chunk(2, dim=-1)]
        a0 = qg @ kg.transpose(-1, -2)
        a0 = a0 + torch.cat([mod.g2g_relative_position_bias,
                             mod.g2l_relative_position_bias[0].unsqueeze(-1).expand(-1, -1, nx * ny)], dim=-1)
        x0 = mod.proj_global((a0.softmax(-1) @ vg).transpose(1, 2).reshape(B, g, C))
    assert relerr(y, torch.cat([x0, x1], dim=1)) < 1e-5


def test_autocast_contract_fp32_caller_gets_tcgen05():
    """SURVEY.md section 8(b) AMP row: under autocast an fp32 caller is cast to the autocast dtype (tensor-core path, bf16
    output); the fused patch-embedding norm keeps the residual stream in fp32 like nn.LayerNorm does."""
    torch.manual_seed(3)
    B, H, D, nx, ny, g = 2, 3, 32, 14, 14, 1
    C, N = H * D, g + nx * ny
    q_all, kv = torch.randn(B, N, C, device=DEV, requires_grad=True), torch.randn(B, N, 2 * C, device=DEV, requires_grad=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = vil_attention(q_all, kv, num_heads=H, nx=nx, ny=ny, w=7, nglo=g, scale=D ** -0.5)
    assert y.dtype == torch.bfloat16 and _lib.last_impl() == "wgmma"
    y.float().sum().backward()
    assert q_all.grad.dtype == torch.float32 and kv.grad.dtype == torch.float32 and _lib.last_impl() == "wgmma"
    y32 = vil_attention(q_all.detach(), kv.detach(), num_heads=H, nx=nx, ny=ny, w=7, nglo=g, scale=D ** -0.5)
    assert y32.dtype == torch.float32 and _lib.last_impl() == "simt" and relerr(y, y32) < 1e-2
    for fused in (True, False):
        net = build_vil("vil_tiny", img_size=224, num_classes=10, fused_norm=fused).to(DEV).eval()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            xs, _, _ = net.layer1[0]((torch.randn(2, 3, 224, 224, device=DEV), None, None))
        assert xs.dtype == torch.float32, fused


@pytest.mark.parametrize("cfg", [(384, 6, 14, 1, True), (384, 6, 14, 1, False), (768, 12, 7, 0, False), (192, 3, 14, 2, True),
                                 (128, 4, 7, 1, True)], ids=lambda c: "dim%d_h%d_w%d_g%d_%s" % (c[:4] + ("rpe" if c[4] else "nob",)))
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_dense_attention_on_the_operator_kernels(cfg, dtype):
    """SURVEY.md section 8(f) row 2: the dense attention of the 14x14 / 7x7 stages (reference `Attention`, msvit.py:37-120,
    Swin-style bias + g2l / g2g) served by the sliding-chunk kernels as their single-chunk case, against the same module
    in fp32 through stock SDPA with the materialised (H,N,N) bias."""
    from vision_longformer_b200.msvit import DenseAttention
    dim, H, w, g, rpe = cfg
    torch.manual_seed(4)
    ref = DenseAttention(dim, num_heads=H, qkv_bias=True, rpe=rpe, wx=w, wy=w, nglo=g, impl="sdpa").to(DEV)
    if rpe:
        for p_ in (ref.local_relative_position_bias_table, *( [ref.g2l_relative_position_bias, ref.g2g_relative_position_bias] if g else [])):
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
    before = _lib.launch_count()
    ym = mod(xm)
    (ym * gy.to(dtype)).sum().backward()
    torch.cuda.synchronize()
    assert _lib.launch_count() > before and _lib.last_impl() in ("wgmma", "simt")
    errs = dict(y=relerr(ym, yr), dx=relerr(xm.grad, xr.grad), dqkv_w=relerr(mod.qkv.weight.grad, ref.qkv.weight.grad))
    if rpe:
        errs["dtable"] = relerr(mod.local_relative_position_bias_table.grad, ref.local_relative_position_bias_table.grad)
        if g:
            errs["dg2l"] = relerr(mod.g2l_relative_position_bias.grad, ref.g2l_relative_position_bias.grad)
            errs["dg2g"] = relerr(mod.g2g_relative_position_bias.grad, ref.g2g_relative_position_bias.grad)
    record("dense_attention_on_the_operator_kernels", "dim%d_h%d_w%d_g%d_%s/%s" % (cfg[:4] + ("rpe" if rpe else "nob", DT_NAME[dtype])), **errs)
    tol = 3e-2 if dtype == torch.bfloat16 else 6e-3            # the Linears run in low precision too
    assert errs["y"] < tol and errs["dx"] < 2 * tol and errs["dqkv_w"] < 2 * tol, errs
    for n in ("dtable", "dg2l", "dg2g"):
        if n in errs:
            assert errs[n] < 0.1, (n, errs)


def test_gpu_launch_counter_and_family():
    before = _lib.launch_count()
    t = make_inputs(1, 2, 32, 14, 14, 1, 7, False)
    kernel_run(t, 14, 14, 7, 0, 0, 32 ** -0.5, torch.bfloat16, "auto")
    # forward = local kernel + global query rows; backward = delta, pass 1, pass 2, global key columns, global query rows
    assert _lib.launch_count() - before == 7
    assert _lib.last_impl() in ("simt", "wgmma")
