"""Dilated sliding-chunk attention (VIL_FLAG_DILATED) on the GPU, both kernel families, fp32 / split fp32 / bf16 / fp16.

A dilated call is the undilated operator run on each of the d^2 residue sub-grids of the image, with the global tokens
shared (include/vil_attn.h).  So:
- the local rows of o, lse and dq, and the local-key rows of dk / dv, are bitwise those of d^2 ordinary calls on the
  gathered sub-grid tensors (a local key is seen only by the queries of its residue, and the walk is the same);
- the global rows (og, lse_g, dqg) and the gradients of g2l[0] and g2g are bitwise those of the d = 1 call;
- the global-key rows of dk / dv and the gradients of the table and of g2l[1] are sums over the residues, equal to the
  sum of the sub-grid calls' up to fp32 reordering;
- everything agrees with the fp64 dilated oracle (tests/dilated_oracle.py) at the bars of the undilated operator.
All calls use the production layouts (q / kv Linear outputs viewed per head, outputs written head-merged).
"""
import numpy as np
import pytest
import torch

from tests import test_gpu_dropout as tdrop
from tests.dilated_oracle import dilated_attention, residues
from tests.util import relerr
from vision_longformer_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
SPLIT = _lib.VIL_FLAG_F32_SPLIT

# name: (dtype, impl, flags, bar of the whole-tensor relative error against the fp64 oracle)
VARIANTS = {
    "simt_f32": (torch.float32, "simt", 0, 2e-5),
    "wgmma_f32split": (torch.float32, "wgmma", SPLIT, 3e-4),
    "wgmma_bf16": (torch.bfloat16, "wgmma", 0, 3e-2),
    "wgmma_f16": (torch.float16, "wgmma", 0, 5e-3),
    "simt_bf16": (torch.bfloat16, "simt", 0, 3e-2),
    "simt_f16": (torch.float16, "simt", 0, 5e-3),
}
# relative error of a sum reordered across residues, for outputs stored in the variant's type
REORDER = {torch.float32: 2e-5, torch.bfloat16: 1.6e-2, torch.float16: 2e-3}

EXACT_MODES = [(1, 0)] + [(e, m) for e in (0, -1) for m in (-1, 0, 1, 2, 3, 4, 5, 6, 7, 8)]
# (nx, ny, w, d, g, rpe, sep, exact, mode)
CASES = [(13, 10, 3, 3, i % 3, i % 4 != 3, i % 2 == 1, e, m) for i, (e, m) in enumerate(EXACT_MODES)] + [
    (16, 16, 4, 2, 0, False, False, 0, 0),
    (9, 11, 4, 2, 2, True, True, -1, 3),
    (2, 9, 2, 3, 1, True, False, 0, 0),        # d > nx: empty residues
    (14, 14, 7, 2, 1, True, False, 1, 0),      # each 7 x 7 sub-grid is one chunk
    (28, 28, 7, 2, 1, True, True, 0, 0),       # ViL stage-3-like sub-grids of 14 x 14
    (20, 17, 5, 3, 1, True, False, -1, 0),
]
CID = lambda c: "%dx%d_w%d_d%d_g%d_%s_%s_e%d_m%d" % (c[0], c[1], c[2], c[3], c[4], "rpe" if c[5] else "norpe",
                                                      "sep" if c[6] else "shared", c[7], c[8])


def make(case, B=2, H=2, D=16, seed=0):
    """fp32 leaf tensors in the Linear-output layouts: q_all (B, [g +] Nloc, H D), kv (B, N, 2 H D), and with separate
    global weights qg_all (B, g, H D), kvg (B, N, 2 H D); the bias parameters; the output gradient (B, N, H D)"""
    nx, ny, w, d, g, rpe, sep, exact, mode = case
    gen = torch.Generator().manual_seed(seed + 7 * nx + ny + 131 * g)
    r = lambda *s: torch.randn(*s, generator=gen)
    N, C = g + nx * ny, H * D
    t = dict(q_all=r(B, N if (g and not sep) else nx * ny, C), kv=r(B, N, 2 * C), dout=r(B, N, C))
    if g and sep:
        t.update(qg_all=r(B, g, C), kvg=r(B, N, 2 * C))
    if rpe:
        t["table"] = 0.5 * r((4 * w - 1) ** 2, H)
        if g:
            t["g2l"], t["g2g"] = 0.5 * r(2, H, g), 0.5 * r(H, g, g)
    t["H"], t["D"] = H, D
    return t


def views(t, case, dtype):
    """(B, H, T, D) views of the call: q, k, v, qg, kg, vg and the gradient views of d_out"""
    nx, ny, w, d, g, rpe, sep, exact, mode = case
    H = t["H"]
    cv = lambda x: x.to(DEV, dtype)
    kv = cv(t["kv"])
    k, v = ops._heads(kv, H, 0, 2), ops._heads(kv, H, 1, 2)
    qa = ops._heads(cv(t["q_all"]), H)
    if g and not sep:
        q, qg, kg, vg = qa[:, :, g:], qa[:, :, :g], k, v
    elif g:
        kvg = cv(t["kvg"])
        q, qg, kg, vg = qa, ops._heads(cv(t["qg_all"]), H), ops._heads(kvg, H, 0, 2), ops._heads(kvg, H, 1, 2)
    else:
        q, qg, kg, vg = qa, None, None, None
    dout = ops._heads(cv(t["dout"]), H)
    return q, k, v, qg, kg, vg, dout[:, :, g:], (dout[:, :, :g] if g else None)


def run(q, k, v, qg, kg, vg, d_o, d_og, t, case, variant, d, drop=(0.0, 0, 0)):
    """forward + backward through the raw ABI; outputs in the production head-merged layout"""
    nx, ny, w, _, g, rpe, sep, exact, mode = case
    dtype, impl, flags, _ = VARIANTS[variant]
    B, H, Nloc, D = q.shape
    N = k.shape[2]
    shared = g > 0 and kg.data_ptr() == k.data_ptr()
    tab = t["table"].to(DEV) if rpe else None
    g2l = t["g2l"].to(DEV) if (rpe and g) else None
    g2g = t["g2g"].to(DEV) if (rpe and g) else None
    out = torch.empty(B, N, H * D, dtype=dtype, device=DEV)
    o = ops._heads(out, H)[:, :, g:]
    og = ops._heads(out, H)[:, :, :g] if g else None
    kw = dict(nx=nx, ny=ny, w=w, exact=exact, mode=mode, scale=D ** -0.5, impl=impl, flags=flags, dilation=d,
              dropout_p=drop[0], dropout_seed=drop[1], dropout_offset=drop[2])
    lse, lse_g = ops.vil_attention_raw_forward(q, k, v, qg, kg, vg, tab, g2l, g2g, o, og, **kw)
    fam = _lib.last_impl()
    dq = ops._heads(torch.empty(B, Nloc, H * D, dtype=dtype, device=DEV), H)
    dkv = torch.empty(B, N, 2 * H * D, dtype=dtype, device=DEV)
    dk, dv = ops._heads(dkv, H, 0, 2), ops._heads(dkv, H, 1, 2)
    dqg = dkg = dvg = None
    if g:
        dqg = torch.empty(B, H, g, D, dtype=dtype, device=DEV)
        if shared:
            dkg, dvg = dk, dv
        else:
            dkvg = torch.empty(B, N, 2 * H * D, dtype=dtype, device=DEV)
            dkg, dvg = ops._heads(dkvg, H, 0, 2), ops._heads(dkvg, H, 1, 2)
    d_tab = torch.zeros_like(tab) if rpe else None
    d_g2l = torch.zeros_like(g2l) if g2l is not None else None
    d_g2g = torch.zeros_like(g2g) if g2g is not None else None
    ops.vil_attention_raw_backward(q, k, v, qg, kg, vg, tab, g2l, g2g, o, og, lse, lse_g, d_o, d_og, dq, dk, dv, dqg, dkg,
                                   dvg, d_tab, d_g2l, d_g2g, **kw)
    assert (fam, _lib.last_impl()) == (impl, impl)
    return dict(o=o, og=og, lse=lse, lse_g=lse_g, dq=dq, dk=dk, dv=dv, dqg=dqg, dkg=dkg if not shared else None,
                dvg=dvg if not shared else None, d_tab=d_tab, d_g2l=d_g2l, d_g2g=d_g2g)


def sub_inputs(views_, g, idx, separate):
    """the gathered tensors of one residue: its local queries and keys after the same global tokens.  `separate`: the
    global queries get their own (equal-valued) keys, so that the local-key gradients hold the local queries' terms only"""
    q, k, v, qg, kg, vg, d_o, d_og = views_
    cat = lambda x: torch.cat([x[:, :, :g], x[:, :, g + idx]], dim=2)
    ks, vs = cat(k), cat(v)
    if g:
        shared = kg.data_ptr() == k.data_ptr()
        kgs, vgs = (ks.clone(), vs.clone()) if (shared and separate) else ((ks, vs) if shared else (cat(kg), cat(vg)))
    else:
        kgs = vgs = None
    return q[:, :, idx].contiguous(), ks, vs, qg, kgs, vgs, d_o[:, :, idx].contiguous(), d_og


def same(a, b, what):
    assert a.shape == b.shape, what
    assert torch.equal(a, b), (what, float((a.float() - b.float()).abs().max()))


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("case", CASES, ids=CID)
def test_dilated_call_is_the_sub_grid_calls(case, variant):
    nx, ny, w, d, g, rpe, sep, exact, mode = case
    dtype = VARIANTS[variant][0]
    t = make(case)
    vw = views(t, case, dtype)
    dil = run(*vw, t, case, variant, d)
    und = run(*vw, t, case, variant, 1)
    # global rows: the d = 1 call's, bit for bit
    if g:
        for key in ("og", "lse_g", "dqg", "d_g2g"):
            if dil[key] is not None:
                same(dil[key], und[key], key)
        if rpe:
            same(dil["d_g2l"][0], und["d_g2l"][0], "d_g2l[0]")
    sums = {}
    for a, b, na, nb, idx in residues(nx, ny, d):
        idx = idx.to(DEV)
        # with shared weights the global queries' terms of the local-key gradients go to dkg of the sub call
        sub = run(*sub_inputs(vw, g, idx, separate=True), t, (na, nb) + case[2:], variant, 1)
        same(dil["o"][:, :, idx], sub["o"], "o")
        same(dil["lse"][:, :, idx], sub["lse"], "lse")
        same(dil["dq"][:, :, idx], sub["dq"], "dq")
        if sep or g == 0:
            same(dil["dk"][:, :, g + idx], sub["dk"][:, :, g:], "dk")
            same(dil["dv"][:, :, g + idx], sub["dv"][:, :, g:], "dv")
        for key, x in (("dk", sub["dk"][:, :, :g] if g else None), ("dv", sub["dv"][:, :, :g] if g else None),
                       ("d_tab", sub["d_tab"]), ("d_g2l1", sub["d_g2l"][1] if sub["d_g2l"] is not None else None)):
            if x is not None:
                sums[key] = sums.get(key, 0) + x.double()
    for key, x in (("dk", dil["dk"][:, :, :g]), ("dv", dil["dv"][:, :, :g]), ("d_tab", dil["d_tab"]),
                   ("d_g2l1", dil["d_g2l"][1] if dil["d_g2l"] is not None else None)):
        if x is None or key not in sums:
            continue
        if key in ("dk", "dv") and not (sep or g == 0):
            continue                             # shared weights: plus the global queries' terms (oracle test below)
        bar = REORDER[dtype] if key in ("dk", "dv") else REORDER[torch.float32]
        assert relerr(x.double(), sums[key]) < bar, (key, relerr(x.double(), sums[key]))


def oracle(t, case):
    """fp64 dilated oracle: outputs and the gradients of dout . out"""
    nx, ny, w, d, g, rpe, sep, exact, mode = case
    H, D = t["H"], t["D"]
    leaf = {k: t[k].double().requires_grad_(True) for k in ("q_all", "kv", "qg_all", "kvg", "table", "g2l", "g2g") if k in t}
    kv = leaf["kv"]
    k, v = ops._heads(kv, H, 0, 2), ops._heads(kv, H, 1, 2)
    qa = ops._heads(leaf["q_all"], H)
    if g and not sep:
        q, qg, kg, vg = qa[:, :, g:], qa[:, :, :g], k, v
    elif g:
        q, qg = qa, ops._heads(leaf["qg_all"], H)
        kg, vg = ops._heads(leaf["kvg"], H, 0, 2), ops._heads(leaf["kvg"], H, 1, 2)
    else:
        q, qg, kg, vg = qa, None, None, None
    o, og, lse, lse_g = dilated_attention(q, k, v, qg, kg, vg, leaf.get("table"), leaf.get("g2l"), leaf.get("g2g"), nx=nx,
                                          ny=ny, w=w, exact=exact, mode=mode, scale=D ** -0.5, d=d)
    dout = ops._heads(t["dout"].double(), H)
    loss = (o * dout[:, :, g:]).sum() + ((og * dout[:, :, :g]).sum() if g else 0)
    loss.backward()
    return o.detach(), og, {k: x.grad for k, x in leaf.items()}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("case", CASES[::3] + CASES[-6:], ids=CID)
def test_dilated_module_op_matches_the_oracle(case, variant):
    """ops.vil_attention(dilation=d) forward and backward, every leaf gradient, against the fp64 oracle"""
    nx, ny, w, d, g, rpe, sep, exact, mode = case
    dtype, impl, flags, bar = VARIANTS[variant]
    t = make(case, seed=5)
    leaf = {k: (t[k].to(DEV, dtype) if k in ("q_all", "kv", "qg_all", "kvg") else t[k].to(DEV)).requires_grad_(True)
            for k in ("q_all", "kv", "qg_all", "kvg", "table", "g2l", "g2g") if k in t}
    prec = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32" if flags & SPLIT else "ieee"
    try:
        out = ops.vil_attention(leaf["q_all"], leaf["kv"], leaf.get("qg_all"), leaf.get("kvg"), leaf.get("table"),
                                leaf.get("g2l"), leaf.get("g2g"), num_heads=t["H"], nx=nx, ny=ny, w=w, nglo=g,
                                exact=exact, mode=mode, scale=t["D"] ** -0.5, impl=impl, dilation=d)
        out.backward(t["dout"].to(DEV, dtype))
    finally:
        torch.backends.cuda.matmul.fp32_precision = prec
    assert _lib.last_impl() == impl
    o_ref, og_ref, grads = oracle(t, case)
    H = t["H"]
    o = ops._heads(out.detach().double().cpu(), H)
    assert relerr(o[:, :, g:], o_ref) < bar
    if g:
        assert relerr(o[:, :, :g], og_ref) < bar
    for key, ref in grads.items():
        err = relerr(leaf[key].grad.double().cpu(), ref)
        assert err < bar, (key, err)


def _keep_sub(seed, offset, p, B, H, nx, ny, w, g, mode, d, a, b, na, nb):
    """keep / (1 - p) of one residue's attn1 in the reference layout: the rows are the queries' image-grid tokens"""
    from oracle import vil_oracle as vo
    padx, pady, mx, my = vo.geometry(na, nb, w)
    w2, n = w * w, len(vo.mode_offsets(mode))
    sc = np.float32(1.0) / (np.float32(1.0) - np.float32(p))
    R, C, l = np.meshgrid(np.arange(mx), np.arange(my), np.arange(w2), indexing="ij")
    qr, qc = R * w + l // w, C * w + l % w
    row = np.where((qr < na) & (qc < nb), (a + d * qr) * ny + (b + d * qc), 0)
    col = np.arange(g + n * w2)
    bh = np.arange(B * H)
    k1 = tdrop.keep_bits(row[None, ..., None], col[None, None, None, None, :], 2 * bh[:, None, None, None, None], seed,
                         offset, p)
    return torch.from_numpy(k1.astype(np.float64) * float(sc))


@pytest.mark.parametrize("variant", ["simt_f32", "wgmma_f32split", "wgmma_bf16", "simt_bf16"])
@pytest.mark.parametrize("case", [CASES[1], CASES[7], CASES[15], CASES[-1]], ids=CID)
def test_dropout_matches_the_mask_restatement(case, variant):
    """the local rows with dropout against the reference algorithm on each sub-grid with the exact mask: row = the query's
    image-grid token, col = its column of the sub-grid's attn1"""
    nx, ny, w, d, g, rpe, sep, exact, mode = case
    dtype, impl, flags, bar = VARIANTS[variant]
    p, seed, offset = 0.3, 1234567, 17
    t = make(case, seed=9)
    vw = views(t, case, dtype)
    res = run(*vw, t, case, variant, d, drop=(p, seed, offset))
    B, H = vw[0].shape[:2]
    q64, k64, v64 = (x.double().cpu() for x in vw[:3])
    qg64 = vw[3].double().cpu() if g else None
    d_o = vw[6].double().cpu()
    tab = t["table"].double() if rpe else None
    g2l = t["g2l"].double() if (rpe and g) else None
    g2g = t["g2g"].double() if (rpe and g) else None
    for a, b, na, nb, idx in residues(nx, ny, d):
        keep = _keep_sub(seed, offset, p, B, H, nx, ny, w, g, mode, d, a, b, na, nb)
        qs = q64[:, :, idx].clone().requires_grad_(True)
        ks = torch.cat([k64[:, :, :g], k64[:, :, g + idx]], dim=2).requires_grad_(True)
        vs = torch.cat([v64[:, :, :g], v64[:, :, g + idx]], dim=2).requires_grad_(True)
        # the global rows of the sub-grid call are not compared: any keys and an all-ones mask serve them
        keep_g = torch.ones(B * H, g, g + len(idx), dtype=torch.float64) if g else None
        o, _ = tdrop.chunked_dropout_reference(qs, ks, vs, qg64, ks.detach() if g else None, vs.detach() if g else None,
                                               tab, g2l, g2g, keep, keep_g, nx=na, ny=nb, w=w, exact=exact, mode=mode,
                                               scale=t["D"] ** -0.5)
        (o * d_o[:, :, idx]).sum().backward()
        assert relerr(res["o"][:, :, idx].double().cpu(), o.detach()) < bar
        assert relerr(res["dq"][:, :, idx].double().cpu(), qs.grad) < bar
        if sep or g == 0:
            assert relerr(res["dk"][:, :, g + idx].double().cpu(), ks.grad[:, :, g:]) < bar
            assert relerr(res["dv"][:, :, g + idx].double().cpu(), vs.grad[:, :, g:]) < bar


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_deterministic_and_workspace_independent(variant):
    case = (20, 17, 5, 3, 1, True, False, -1, 0)
    t = make(case, seed=3)
    vw = views(t, case, VARIANTS[variant][0])
    first = run(*vw, t, case, variant, 3)
    junk = torch.full((64 << 20,), float("nan"), device=DEV)      # the next workspaces are carved from dirty memory
    del junk
    second = run(*vw, t, case, variant, 3)
    for key, x in first.items():
        if x is not None:
            same(x, second[key], key)


def test_d1_is_the_undilated_call_bitwise():
    """dilation=1 leaves the flag clear: the call is the default one"""
    case = (13, 10, 3, 1, 1, True, False, 0, 0)
    t = make(case)
    for variant in ("simt_f32", "wgmma_bf16"):
        vw = views(t, case, VARIANTS[variant][0])
        a = run(*vw, t, case, variant, 1)
        b = run(*vw, t, case, variant, 1)
        for key, x in a.items():
            if x is not None:
                same(x, b[key], key)


# ---------------------------------------------------------------- module level
def _oracle_module(ref, x, nx, ny, d):
    """OracleLong2DSCSelfAttention.forward with the dilated oracle in place of the attention core"""
    B, N, C = x.shape
    g, H, M = ref.Nglo, ref.num_heads, ref.head_dim
    q = ref.query(x[:, g:]).reshape(B, nx * ny, H, M).transpose(1, 2)
    kv = ref.kv(x).reshape(B, N, 2, H, M).permute(2, 0, 3, 1, 4)
    qg = ref.query_global(x[:, :g]).reshape(B, g, H, M).transpose(1, 2)
    kvg = ref.kv_global(x).reshape(B, N, 2, H, M).permute(2, 0, 3, 1, 4)
    o, og, _, _ = dilated_attention(q, kv[0], kv[1], qg, kvg[0], kvg[1], ref.local_relative_position_bias_table,
                                    ref.g2l_relative_position_bias, ref.g2g_relative_position_bias, nx=nx, ny=ny,
                                    w=ref.attention_window, exact=ref.exact, mode=0, scale=ref.scale, d=d)
    return torch.cat([ref.proj_global(og.transpose(1, 2).reshape(B, g, C)),
                      ref.proj(o.transpose(1, 2).reshape(B, nx * ny, C))], dim=1)


@pytest.mark.parametrize("exact", [0, 1, -1])
def test_module_with_dilation_matches_the_oracle(exact):
    from oracle.vil_oracle import OracleLong2DSCSelfAttention
    from vision_longformer_b200 import B200Long2DSCSelfAttention
    torch.manual_seed(0)
    kw = dict(dim=96, num_heads=3, qkv_bias=True, w=7, nglo=1, exact=exact, rpe=True, sharew=True)
    nx = ny = 28
    ref = OracleLong2DSCSelfAttention(**kw).double().eval()
    x = torch.randn(2, 1 + nx * ny, 96, dtype=torch.float64, requires_grad=True)
    y_ref = _oracle_module(ref, x, nx, ny, 2)
    gy = torch.randn_like(y_ref)
    (y_ref * gy).sum().backward()
    for dtype, tol in ((torch.float32, 2e-5), (torch.bfloat16, 2e-2)):
        mod = B200Long2DSCSelfAttention(d=2, **kw).to(DEV).eval()
        mod.load_state_dict(ref.state_dict())
        mod = mod.to(dtype)
        xg = x.detach().to(DEV, dtype).requires_grad_(True)
        y = mod(xg, nx, ny)
        (y * gy.to(DEV, dtype)).sum().backward()
        assert relerr(y.double().cpu(), y_ref) < tol
        assert relerr(xg.grad.double().cpu(), x.grad) < tol
        for name, prm in mod.named_parameters():
            assert relerr(prm.grad.double().cpu(), dict(ref.named_parameters())[name].grad) < tol, name


def test_vil_tiny_trains_with_dilation_under_autocast():
    from vision_longformer_b200 import B200Long2DSCSelfAttention
    from vision_longformer_b200.msvit import build_vil
    torch.manual_seed(0)
    net = build_vil("vil_tiny", img_size=224, num_classes=10, d=2).to(DEV).train()
    attn = [m for m in net.modules() if isinstance(m, B200Long2DSCSelfAttention)]
    assert attn and all(m.attention_dilation == 2 for m in attn)
    opt = torch.optim.SGD(net.parameters(), lr=0.01)
    x = torch.randn(4, 3, 224, 224, device=DEV)
    y = torch.randint(0, 10, (4,), device=DEV)
    losses = []
    for _ in range(3):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(net(x), y)
        opt.zero_grad()
        loss.backward()
        assert all(p.grad is None or bool(torch.isfinite(p.grad).all()) for p in net.parameters())
        opt.step()
        losses.append(loss.item())
    assert np.isfinite(losses).all() and len(set(losses)) == 3
