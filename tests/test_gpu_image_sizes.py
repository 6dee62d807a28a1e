"""Per-image token grids in a padded batch (vil_attn_fwd_sized_sm100 / _bwd_sized_sm100) on the GPU, both kernel
families, fp32 / split fp32 / bf16 / fp16.

A sized call gives every real token of image b what the unsized call on image b alone, cropped to its h_b x w_b grid,
gives it (include/vil_attn.h).  So:
- the local rows of o, lse and dq are bitwise those of a B = 1 call on the contiguous crop, and so are the local-key rows
  of dk / dv when no global query feeds them (g = 0 or separate global weights);
- the global rows, the global-key gradients and the three bias gradients agree with the crop calls up to fp32 reordering;
- the off-image rows of o, dq, dk, dv are exact zeros and lse is -inf there, whatever the inputs hold at those tokens and
  whatever the outputs and the workspace held before;
- everything agrees with the fp64 cropping oracle (tests/sized_oracle.py) at the bars of the unsized operator.
All calls use the production layouts (q / kv Linear outputs viewed per head, outputs written head-merged).
"""
import numpy as np
import pytest
import torch

from tests import test_gpu_dropout as tdrop
from tests.sized_oracle import image_index, sized_attention
from tests.test_gpu_dilation import REORDER, SPLIT, VARIANTS, _keep_sub, same
from tests.util import relerr
from vision_longformer_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (nx, ny, w, d, g, rpe, sep, exact, mode, sizes): full images, 1 x n, n x 1 and sizes that are not multiples of w
CASES = [
    (13, 11, 4, 1, 1, True, False, 0, 0, [(13, 11), (7, 5), (1, 11), (13, 1)]),
    (13, 11, 4, 1, 2, True, True, -1, 0, [(9, 6), (13, 11), (1, 1), (5, 11)]),
    (12, 10, 3, 1, 0, False, False, 1, 0, [(12, 2), (4, 10), (12, 10)]),
    (12, 10, 3, 1, 1, False, True, 0, -1, [(6, 7), (12, 1)]),
    (11, 14, 5, 1, 2, True, False, -1, 3, [(11, 9), (3, 14)]),
    (10, 9, 3, 1, 1, True, True, 0, 6, [(1, 9), (10, 4)]),
    (13, 10, 3, 2, 1, True, True, 0, 0, [(13, 10), (8, 7), (2, 10)]),      # with dilation: the crop's residues
    (12, 12, 3, 3, 1, True, False, -1, 0, [(7, 12), (12, 5)]),
    (12, 9, 2, 2, 0, True, False, 1, 0, [(1, 9), (12, 1), (7, 4)]),
]
CID = lambda c: "%dx%d_w%d_d%d_g%d_%s_%s_e%d_m%d_%s" % (c[0], c[1], c[2], c[3], c[4], "rpe" if c[5] else "norpe",
                                                         "sep" if c[6] else "shared", c[7], c[8],
                                                         "-".join("%dx%d" % s for s in c[9]))


def make(case, H=2, D=16, seed=0):
    """fp32 leaf tensors in the Linear-output layouts (as tests/test_gpu_dilation.make), B = the number of sizes"""
    nx, ny, w, d, g, rpe, sep, exact, mode, sizes = case
    B = len(sizes)
    gen = torch.Generator().manual_seed(seed + 7 * nx + ny + 131 * g + 17 * B)
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


def off_image(case):
    """(B, nx * ny) bool: the off-image local tokens"""
    nx, ny, sizes = case[0], case[1], case[9]
    off = torch.ones(len(sizes), nx * ny, dtype=torch.bool)
    for b, (h, wb) in enumerate(sizes):
        off[b, image_index(nx, ny, h, wb)] = False
    return off


def poison(t, case):
    """the leaf tensors with NaN / +-inf at every off-image token (q, kv, kvg and the output gradient)"""
    g, sep = case[4], case[6]
    off = off_image(case)
    t = dict(t)
    vals = torch.tensor([float("nan"), float("inf"), -float("inf")])
    for key in ("q_all", "kv", "dout", "kvg"):
        if key not in t:
            continue
        x = t[key].clone()
        lead = 0 if (key == "q_all" and (sep or g == 0)) else g
        for b in range(x.shape[0]):
            rows = lead + off[b].nonzero().flatten()
            x[b, rows] = vals[torch.arange(len(rows) * x.shape[2]) % 3].reshape(len(rows), x.shape[2])
        t[key] = x
    return t


def views(t, case, dtype):
    nx, ny, w, d, g, rpe, sep, exact, mode, sizes = case
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


def run(q, k, v, qg, kg, vg, d_o, d_og, t, geo, variant, sizes=None, hw=None, fill=None, drop=(0.0, 0, 0)):
    """forward + backward through the raw ABI; geo = (nx, ny, w, d, g, rpe, exact, mode).  `hw`: a device (B, 2) int32
    tensor passed straight to the sized entry points; `fill`: prefill every output (and the workspaces) with this value"""
    nx, ny, w, d, g, rpe, exact, mode = geo
    dtype, impl, flags, _ = VARIANTS[variant]
    B, H, Nloc, D = q.shape
    N = k.shape[2]
    shared = g > 0 and kg.data_ptr() == k.data_ptr()
    new = (lambda *s: torch.full(s, fill, dtype=dtype, device=DEV)) if fill is not None else \
        (lambda *s: torch.empty(*s, dtype=dtype, device=DEV))
    tab = t["table"].to(DEV) if rpe else None
    g2l = t["g2l"].to(DEV) if (rpe and g) else None
    g2g = t["g2g"].to(DEV) if (rpe and g) else None
    out = new(B, N, H * D)
    o = ops._heads(out, H)[:, :, g:]
    og = ops._heads(out, H)[:, :, :g] if g else None
    kw = dict(nx=nx, ny=ny, w=w, exact=exact, mode=mode, scale=D ** -0.5, impl=impl, flags=flags, dilation=d,
              dropout_p=drop[0], dropout_seed=drop[1], dropout_offset=drop[2], image_sizes=sizes, _image_hw=hw)
    if fill is not None:
        junk = torch.full((32 << 20,), fill, device=DEV)      # the workspaces are carved from this memory
        del junk
    lse, lse_g = ops.vil_attention_raw_forward(q, k, v, qg, kg, vg, tab, g2l, g2g, o, og, **kw)
    fam = _lib.last_impl()
    dq = ops._heads(new(B, Nloc, H * D), H)
    dkv = new(B, N, 2 * H * D)
    dk, dv = ops._heads(dkv, H, 0, 2), ops._heads(dkv, H, 1, 2)
    dqg = dkg = dvg = None
    if g:
        dqg = new(B, H, g, D)
        if shared:
            dkg, dvg = dk, dv
        else:
            dkvg = new(B, N, 2 * H * D)
            dkg, dvg = ops._heads(dkvg, H, 0, 2), ops._heads(dkvg, H, 1, 2)
    d_tab = torch.zeros_like(tab) if rpe else None
    d_g2l = torch.zeros_like(g2l) if g2l is not None else None
    d_g2g = torch.zeros_like(g2g) if g2g is not None else None
    if fill is not None:
        junk = torch.full((32 << 20,), fill, device=DEV)
        del junk
    ops.vil_attention_raw_backward(q, k, v, qg, kg, vg, tab, g2l, g2g, o, og, lse, lse_g, d_o, d_og, dq, dk, dv, dqg, dkg,
                                   dvg, d_tab, d_g2l, d_g2g, **kw)
    assert (fam, _lib.last_impl()) == (impl, impl)
    return dict(o=o, og=og, lse=lse, lse_g=lse_g, dq=dq, dk=dk, dv=dv, dqg=dqg, dkg=dkg if not shared else None,
                dvg=dvg if not shared else None, d_tab=d_tab, d_g2l=d_g2l, d_g2g=d_g2g)


def geo_of(case):
    nx, ny, w, d, g, rpe, sep, exact, mode, sizes = case
    return nx, ny, w, d, g, rpe, exact, mode


def crop_inputs(vw, g, b, idx):
    """image b's contiguous crop: its local queries, and its keys after the same global tokens"""
    q, k, v, qg, kg, vg, d_o, d_og = vw
    cat = lambda x: torch.cat([x[b:b + 1, :, :g], x[b:b + 1, :, g + idx]], dim=2)
    ks, vs = cat(k), cat(v)
    if g:
        shared = kg.data_ptr() == k.data_ptr()
        kgs, vgs = (ks, vs) if shared else (cat(kg), cat(vg))
    else:
        kgs = vgs = None
    sl = lambda x: x[b:b + 1].contiguous() if x is not None else None
    return q[b:b + 1, :, idx].contiguous(), ks, vs, sl(qg), kgs, vgs, d_o[b:b + 1, :, idx].contiguous(), sl(d_og)


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("case", CASES, ids=CID)
def test_sized_call_is_the_crop_calls(case, variant):
    nx, ny, w, d, g, rpe, sep, exact, mode, sizes = case
    dtype = VARIANTS[variant][0]
    t = make(case)
    vw = views(t, case, dtype)
    res = run(*vw, t, geo_of(case), variant, sizes=sizes)
    sums = {}
    f32 = REORDER[torch.float32]
    for b, (h, wb) in enumerate(sizes):
        idx = image_index(nx, ny, h, wb).to(DEV)
        sub = run(*crop_inputs(vw, g, b, idx), t, (h, wb, w, d, g, rpe, exact, mode), variant)
        same(res["o"][b:b + 1, :, idx], sub["o"], "o")
        same(res["lse"][b:b + 1, :, idx], sub["lse"], "lse")
        same(res["dq"][b:b + 1, :, idx], sub["dq"], "dq")
        if sep or g == 0:
            same(res["dk"][b:b + 1, :, g + idx], sub["dk"][:, :, g:], "dk")
            same(res["dv"][b:b + 1, :, g + idx], sub["dv"][:, :, g:], "dv")
        else:
            assert relerr(res["dk"][b:b + 1, :, g + idx], sub["dk"][:, :, g:]) < REORDER[dtype]
            assert relerr(res["dv"][b:b + 1, :, g + idx], sub["dv"][:, :, g:]) < REORDER[dtype]
        if g:
            for key in ("og", "dqg"):
                assert relerr(res[key][b:b + 1], sub[key]) < REORDER[dtype], key
            assert relerr(res["lse_g"][b:b + 1], sub["lse_g"]) < f32
            for key in ("dk", "dv"):                  # the global keys' rows
                assert relerr(res[key][b:b + 1, :, :g], sub[key][:, :, :g]) < REORDER[dtype], key
            if sep:                                  # separate global keys: [global | the image's local keys]
                for key in ("dkg", "dvg"):
                    assert relerr(res[key][b:b + 1, :, :g], sub[key][:, :, :g]) < REORDER[dtype], key
                    assert relerr(res[key][b:b + 1, :, g + idx], sub[key][:, :, g:]) < REORDER[dtype], key
        for key in ("d_tab", "d_g2l", "d_g2g"):
            if sub[key] is not None:
                sums[key] = sums.get(key, 0) + sub[key].double()
    for key, x in sums.items():
        assert relerr(res[key].double(), x) < f32, (key, relerr(res[key].double(), x))


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("case", CASES[:2] + CASES[4:5] + CASES[6:7], ids=CID)
def test_full_sizes_are_the_unsized_call_bitwise(case, variant):
    """the sized entry points with every image full are the unsized ones, on every output"""
    dtype = VARIANTS[variant][0]
    t = make(case, seed=1)
    vw = views(t, case, dtype)
    B = len(case[9])
    full = torch.tensor([[case[0], case[1]]] * B, dtype=torch.int32, device=DEV)
    a = run(*vw, t, geo_of(case), variant, hw=full)
    b = run(*vw, t, geo_of(case), variant)
    for key, x in a.items():
        if x is not None:
            same(x, b[key], key)


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("case", CASES, ids=CID)
def test_padding_never_leaks(case, variant):
    """NaN / +-inf at every off-image input token, NaN in every output and workspace beforehand: the real tokens' outputs
    are unchanged bit for bit, and the off-image rows are exact zeros (lse -inf)"""
    nx, ny, w, d, g, rpe, sep, exact, mode, sizes = case
    dtype = VARIANTS[variant][0]
    t = make(case, seed=2)
    clean = run(*views(t, case, dtype), t, geo_of(case), variant, sizes=sizes)
    dirty = run(*views(poison(t, case), case, dtype), t, geo_of(case), variant, sizes=sizes, fill=float("nan"))
    off = off_image(case).to(DEV)
    for key, x in clean.items():
        if x is None:
            continue
        y = dirty[key]
        if key in ("o", "dq", "lse"):
            on_rows = ~off
            same(x[on_rows[:, None].expand(x.shape[:3])], y[on_rows[:, None].expand(x.shape[:3])], key)
            offv = y[off[:, None].expand(y.shape[:3])]
            if key == "lse":
                assert bool((offv == -float("inf")).all()), key
            else:
                assert bool((offv == 0).all()), key
        elif key in ("dk", "dv", "dkg", "dvg"):
            keys_off = torch.cat([torch.zeros_like(off[:, :g]), off], dim=1)
            same(x[~keys_off[:, None].expand(x.shape[:3])], y[~keys_off[:, None].expand(x.shape[:3])], key)
            assert bool((y[keys_off[:, None].expand(y.shape[:3])] == 0).all()), key
        else:
            same(x, y, key)


def oracle(t, case):
    """fp64 cropping oracle: outputs and the gradients of dout . out"""
    nx, ny, w, d, g, rpe, sep, exact, mode, sizes = case
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
    o, og, lse, lse_g = sized_attention(q, k, v, qg, kg, vg, leaf.get("table"), leaf.get("g2l"), leaf.get("g2g"), nx=nx,
                                        ny=ny, w=w, sizes=sizes, exact=exact, mode=mode, scale=D ** -0.5, d=d)
    dout = ops._heads(t["dout"].double(), H)
    loss = (o * dout[:, :, g:]).sum() + ((og * dout[:, :, :g]).sum() if g else 0)
    loss.backward()
    return o.detach(), og, {k: x.grad for k, x in leaf.items()}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("case", CASES, ids=CID)
def test_op_matches_the_oracle(case, variant):
    """ops.vil_attention(image_sizes=...) forward and backward, every leaf gradient, against the fp64 oracle"""
    nx, ny, w, d, g, rpe, sep, exact, mode, sizes = case
    dtype, impl, flags, bar = VARIANTS[variant]
    t = make(case, seed=5)
    leaf = {k: (t[k].to(DEV, dtype) if k in ("q_all", "kv", "qg_all", "kvg") else t[k].to(DEV)).requires_grad_(True)
            for k in ("q_all", "kv", "qg_all", "kvg", "table", "g2l", "g2g") if k in t}
    prec = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32" if flags & SPLIT else "ieee"
    try:
        out = ops.vil_attention(leaf["q_all"], leaf["kv"], leaf.get("qg_all"), leaf.get("kvg"), leaf.get("table"),
                                leaf.get("g2l"), leaf.get("g2g"), num_heads=t["H"], nx=nx, ny=ny, w=w, nglo=g,
                                exact=exact, mode=mode, scale=t["D"] ** -0.5, impl=impl, dilation=d,
                                image_sizes=torch.tensor(sizes))
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


@pytest.mark.parametrize("variant", ["simt_f32", "wgmma_f32split", "wgmma_bf16", "simt_bf16"])
@pytest.mark.parametrize("case", [CASES[0], CASES[3], CASES[5], CASES[6]], ids=CID)
def test_dropout_matches_the_mask_restatement(case, variant):
    """the local rows with dropout against the reference algorithm on each crop with the exact mask: row = the query's
    padded-grid token, col = its column of the crop's attn1 (for d > 1, of its residue of the crop)"""
    from tests.dilated_oracle import residues
    nx, ny, w, d, g, rpe, sep, exact, mode, sizes = case
    dtype, impl, flags, bar = VARIANTS[variant]
    p, seed, offset = 0.3, 1234567, 17
    t = make(case, seed=9)
    vw = views(t, case, dtype)
    res = run(*vw, t, geo_of(case), variant, sizes=sizes, drop=(p, seed, offset))
    B, H = vw[0].shape[:2]
    q64, k64, v64 = (x.double().cpu() for x in vw[:3])
    qg64 = vw[3].double().cpu() if g else None
    d_o = vw[6].double().cpu()
    tab = t["table"].double() if rpe else None
    g2l = t["g2l"].double() if (rpe and g) else None
    g2g = t["g2g"].double() if (rpe and g) else None
    for bi, (h, wb) in enumerate(sizes):
        for a, b, na, nb, ridx in residues(h, wb, d):
            # crop-local token r * wb + c -> padded-grid token r * ny + c
            idx = (ridx // wb) * ny + ridx % wb
            keep = _keep_sub(seed, offset, p, B, H, nx, ny, w, g, mode, d, a, b, na, nb)[bi * H:(bi + 1) * H]
            qs = q64[bi:bi + 1, :, idx].clone().requires_grad_(True)
            ks = torch.cat([k64[bi:bi + 1, :, :g], k64[bi:bi + 1, :, g + idx]], dim=2).requires_grad_(True)
            vs = torch.cat([v64[bi:bi + 1, :, :g], v64[bi:bi + 1, :, g + idx]], dim=2).requires_grad_(True)
            keep_g = torch.ones(H, g, g + len(idx), dtype=torch.float64) if g else None
            o, _ = tdrop.chunked_dropout_reference(qs, ks, vs, qg64[bi:bi + 1] if g else None, ks.detach() if g else None,
                                                   vs.detach() if g else None, tab, g2l, g2g, keep, keep_g, nx=na, ny=nb,
                                                   w=w, exact=exact, mode=mode, scale=t["D"] ** -0.5)
            (o * d_o[bi:bi + 1, :, idx]).sum().backward()
            assert relerr(res["o"][bi:bi + 1, :, idx].double().cpu(), o.detach()) < bar
            assert relerr(res["dq"][bi:bi + 1, :, idx].double().cpu(), qs.grad) < bar
            if sep or g == 0:
                assert relerr(res["dk"][bi:bi + 1, :, g + idx].double().cpu(), ks.grad[:, :, g:]) < bar
                assert relerr(res["dv"][bi:bi + 1, :, g + idx].double().cpu(), vs.grad[:, :, g:]) < bar


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_deterministic_with_a_dirty_workspace(variant):
    case = CASES[1]
    t = make(case, seed=3)
    vw = views(t, case, VARIANTS[variant][0])
    first = run(*vw, t, geo_of(case), variant, sizes=case[9])
    second = run(*vw, t, geo_of(case), variant, sizes=case[9], fill=float("nan"))
    for key, x in first.items():
        if x is not None:
            same(x, second[key], key)


@pytest.mark.parametrize("variant", ["wgmma_bf16", "simt_f32"])
def test_pass1_slices_serving_several_images(variant):
    """with the bias table, a pass-1 CTA serves several images (B > nslice): its sub-grid follows each image"""
    sizes = [(56, 56), (20, 33), (1, 56), (56, 1), (7, 7), (49, 50), (3, 40), (56, 12), (30, 30), (13, 56), (8, 2), (41, 55)]
    case = (56, 56, 7, 1, 1, True, True, 0, 0, sizes)
    dtype = VARIANTS[variant][0]
    t = make(case, seed=4)
    vw = views(t, case, dtype)
    res = run(*vw, t, geo_of(case), variant, sizes=sizes)
    tab = 0
    for b, (h, wb) in enumerate(sizes):
        idx = image_index(56, 56, h, wb).to(DEV)
        sub = run(*crop_inputs(vw, 1, b, idx), t, (h, wb, 7, 1, 1, True, 0, 0), variant)
        same(res["dq"][b:b + 1, :, idx], sub["dq"], "dq")
        tab = tab + sub["d_tab"].double()
    assert relerr(res["d_tab"].double(), tab) < REORDER[torch.float32]


# ---------------------------------------------------------------- module level
def _module_crop_reference(mod, x, nx, ny, sizes):
    """the module on each cropped image alone (B = 1, no sizes), scattered back; off-image rows: proj of a zero output"""
    B, N, C = x.shape
    g = mod.Nglo
    y = mod.proj(torch.zeros(B, N, C, dtype=x.dtype, device=x.device))
    for b, (h, wb) in enumerate(sizes):
        idx = image_index(nx, ny, h, wb).to(x.device)
        xb = torch.cat([x[b:b + 1, :g], x[b:b + 1, g + idx]], dim=1)
        yb = mod(xb, h, wb)
        y[b, :g] = yb[0, :g]
        y[b, g + idx] = yb[0, g:]
    return y


@pytest.mark.parametrize("only_glo", [False, True])
@pytest.mark.parametrize("sharew", [True, False])
def test_module_matches_the_crop_reference(only_glo, sharew):
    """B200Long2DSCSelfAttention(image_sizes=...) in fp32 on the GPU (SIMT family) against itself on each crop, forward
    and every gradient; NaN at the off-image input tokens does not reach them"""
    from vision_longformer_b200 import B200Long2DSCSelfAttention
    torch.manual_seed(0)
    nx, ny, sizes = 21, 17, [(21, 17), (9, 12), (1, 17), (21, 2)]
    mod = B200Long2DSCSelfAttention(48, num_heads=3, qkv_bias=True, w=7, nglo=1, exact=-1, rpe=True, sharew=sharew,
                                    only_glo=only_glo).to(DEV).eval()
    x = torch.randn(len(sizes), 1 + nx * ny, 48, device=DEV)
    gy = torch.randn_like(x)
    off = off_image((nx, ny, 7, 1, 1, True, False, 0, 0, sizes)).to(DEV)
    xr = x.clone().requires_grad_(True)
    y = mod(xr, nx, ny, image_sizes=sizes)
    (y * gy).sum().backward()
    grads = {n: p.grad.clone() for n, p in mod.named_parameters() if p.grad is not None}   # only_glo: no local table
    mod.zero_grad()
    xc = x.clone().requires_grad_(True)
    yc = _module_crop_reference(mod, xc, nx, ny, sizes)
    (yc * gy).sum().backward()
    assert relerr(y, yc) < 2e-5
    keys_on = ~torch.cat([torch.zeros_like(off[:, :1]), off], 1)
    assert relerr(xr.grad[keys_on], xc.grad[keys_on]) < 2e-5
    for n, p in mod.named_parameters():
        assert (p.grad is None) == (n not in grads), n
        if p.grad is not None:
            assert relerr(grads[n], p.grad) < 2e-5, n
    # NaN at the off-image tokens: same outputs at every row
    xn = torch.where(keys_on[..., None], x, float("nan"))
    assert relerr(mod(xn, nx, ny, image_sizes=sizes), y.detach()) < 1e-6


def test_module_trains_with_sizes_under_autocast():
    from vision_longformer_b200 import B200Long2DSCSelfAttention
    torch.manual_seed(0)
    nx, ny = 28, 40
    layers = torch.nn.ModuleList(B200Long2DSCSelfAttention(96, num_heads=3, qkv_bias=True, w=7, nglo=1, rpe=True,
                                                           sharew=True, mode=1, attn_drop=0.1) for _ in range(2)).to(DEV)
    layers.train()
    opt = torch.optim.SGD(layers.parameters(), lr=0.05)
    x = torch.randn(4, 1 + nx * ny, 96, device=DEV)
    sizes = [(28, 40), (20, 31), (9, 40), (28, 13)]
    losses = []
    for _ in range(3):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            h = x
            for m in layers:
                h = h + m(h, nx, ny, image_sizes=sizes)
            loss = h.float().pow(2).mean()
        opt.zero_grad()
        loss.backward()
        assert all(bool(torch.isfinite(p.grad).all()) for p in layers.parameters())
        opt.step()
        losses.append(loss.item())
    assert np.isfinite(losses).all() and len(set(losses)) == 3
