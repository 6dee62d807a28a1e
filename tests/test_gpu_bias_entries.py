"""The relative-position-bias gradients entry by entry: d_bias_table, d_g2l and d_g2g.

The other parity files hold these three by one norm over the whole tensor.  The central table entries collect thousands
of (query, key) pairs per image and dominate that norm; the entries at the edge of the table collect a handful.  A clip
off by one row or column in the table scatter, or a pair sent to its neighbour entry, changes a few sparse entries by
100 % and stays far under a whole-tensor bar.  Here every entry is held on its own.

Reference (CPU, fp64, `bias_grad_terms`): the chunked layout of oracle.vil_oracle.chunked_attention on the inputs rounded
to the kernel's dtype, looped over the offsets so that memory stays linear in the image (w = 48 needs it).  It forms P,
dP = dO.v, delta = rowsum(dO * o) and dS = P (dP m - delta), m = keep / (1 - p) with dropout and 1 without, and scatters
for every entry e
  ref[e]     sum of dS over the visible pairs that index e
  scale[e]   T_e = sum of P ||dO_i|| (m ||v_j|| + ||o_i||) over the same pairs (|dS| <= that term by term)
  npairs[e]  the number of visible pairs.
A pair that two wrapped offsets reach (exact = -1 on a 2 x 2 chunk grid) is two columns of attn1: two entries and, with
dropout, two draws.  The CPU tests pin `ref` to the autograd gradients of the dense oracle, of the chunked oracle and of
test_gpu_dropout's chunked dropout reference to 1e-12 T_e.

Metric (GPU, through the C ABI): err[e] = |out[e] - ref[e]| <= bar T_e + floor_e, and out[e] == 0.0 exactly where
npairs[e] == 0 (structural zeros).  floor_e = npairs[e] 2^-126 max||dO|| (max m max||v|| + max||o||) is the flush of a P
below fp32's smallest normal.  Every maximum of err / T_e is recorded (tests.util.record) with its entry.

Contract tests: the three gradients are ACCUMULATED into (include/vil_attn.h), so a pre-filled X must come back as X plus
the clean result bit for bit; and a workspace full of 0xFF bytes (NaN as fp32) must change no output bit.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import vil_oracle as vo
from tests import test_gpu_attention_rows as tar
from tests import test_gpu_dropout as tdrop
from tests import test_gpu_parity as tpar
from tests.test_gpu_batch_slices import nslice_of_the_library
from tests.test_gpu_deterministic import _params
from tests.util import record, relerr

gpu = pytest.mark.gpu
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
U32 = 2.0 ** -24
NAMES = ("dtable", "dg2l", "dg2g")

# test_gpu_attention_rows' variants and the fp16 production build
VARIANTS = dict(tar.VARIANTS, wgmma_fp16=("wgmma", F16, False, "contig"))

# --------------------------------------------------------------------------- bars
# One dS enters an entry with an error of at most
#   eps_o ||dO|| ||o||                        delta = rowsum(dO * o) from the STORED o.  eps_o = the unit roundoff of its
#                                             type (2^-8 bf16, 2^-11 fp16, 2^-24 fp32) plus, in the wgmma family, that of
#                                             the P operand the forward multiplied V with (P is rounded to the input type
#                                             for the tensor cores, so the fp32 o of VIL_FLAG_F32_OUT carries it as well)
#   + (2 D + 2 smax + 8) 2^-24 ||dO|| (m ||v|| + ||o||)
#                                             the fp32 dot products dP and s (D roundings each), P = __expf(s - lse) with
#                                             smax = max |s| + |lse| (the relative error of P grows with its argument)
# and the fp32 sum of the entry's npairs terms adds at most (npairs - 1) 2^-24 T_e.  With |dS| <= P ||dO|| (m ||v|| + ||o||)
# that gives err[e] <= ceiling T_e, ceiling = eps_o + (2 D + 2 smax + 8 + max npairs) 2^-24 (`ceiling`).
# The bars are about 3x the worst err / T_e measured on an H100 SXM (700 W power limit) over this file, plus 2 smax 2^-24
# for the peaked cases; each is asserted below the ceiling of every case it holds.
EPS_O = {"simt_fp32": U32, "wgmma_fp16_f32out": U32 + 2.0 ** -11, "wgmma_bf16_f32out": U32 + 2.0 ** -8,
         "wgmma_bf16": 2.0 ** -7, "wgmma_bf16_linear": 2.0 ** -7, "wgmma_fp16": 2.0 ** -10}
# worst err / T_e measured over the file: SIMT fp32 1.5e-6 (g2g under a peaked g2g bias, 6.2e-7 in the table); fp16 with
# fp32 outputs 3.4e-5; bf16 with fp32 outputs 2.9e-4; bf16 production 7.3e-4 (both layouts); fp16 production 6.9e-5.  All
# in sparse entries (1 to 44 pairs) of the dropout and cyclic 2 x 2 cases.
KAPPA = {"simt_fp32": 4e-6, "wgmma_fp16_f32out": 1e-4, "wgmma_bf16_f32out": 9e-4, "wgmma_bf16": 2.2e-3,
         "wgmma_bf16_linear": 2.2e-3, "wgmma_fp16": 2e-4}


def ceiling(variant, D, smax, nmax):
    return EPS_O[variant] + (2 * D + 2 * smax + 8 + nmax) * U32


def bar_of(variant, smax):
    return KAPPA[variant] + 2 * smax * U32


CASE_ID = lambda c: "B%d_H%d_D%d_%dx%d_g%d_w%d_e%d_m%d" % tuple(c[:9]) + ("_sep" if len(c) > 9 and c[9] else "")


def full(case):
    """test_gpu_attention_rows' case layout: (..., rpe = True, separate global weights)"""
    return tuple(case[:9]) + (True, bool(len(case) > 9 and case[9]))


# --------------------------------------------------------------------------- the per-entry fp64 restatement
def _chunks(x, nx, ny, w):
    """(B, H, nx ny, D) -> (B H, mx, my, w2, D), zero-padded (the layout of vo.chunked_attention, channels last)"""
    B, H, _, D = x.shape
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    img = F.pad(x.reshape(B * H, nx, ny, D), (0, 0, 0, pady, 0, padx))
    return img.reshape(B * H, mx, w, my, w, D).permute(0, 1, 3, 2, 4, 5).reshape(B * H, mx, my, w * w, D)


def _roll(x, dR, dC):
    """bring chunk (m + dR, n + dC) to (m, n), cyclic (vo._roll_chunks)"""
    return x if dR == 0 and dC == 0 else torch.roll(x, shifts=(-dR, -dC), dims=(1, 2))


def offset_blocks(case):
    """per visited offset (dR, dC): the (w2, w2) table index of its block (vo.relative_position_index in the reference's
    block order) and the visible pairs (mx, my, w2, w2) from vo.chunk_mask and the real query rows"""
    B, H, D, nx, ny, g, w, exact, mode = case[:9]
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    w2 = w * w
    rpi = vo.relative_position_index(w)
    mask = vo.chunk_mask(nx, ny, w, exact, mode)[0]
    l = torch.arange(w2)
    R, C = torch.arange(mx)[:, None, None], torch.arange(my)[None, :, None]
    real = ((R * w + l // w) < nx) & ((C * w + l % w) < ny)                      # (mx, my, w2) real query rows
    out = []
    for oi, (dR, dC) in enumerate(vo.mode_offsets(mode)):
        pos = vo.OFFSETS9.index((dR, dC))
        vis = (~mask[..., oi * w2:(oi + 1) * w2]).expand(mx, my, w2, w2) & real[..., None]
        out.append(((dR, dC), rpi[:, pos * w2:(pos + 1) * w2], vis))
    return out, real


def table_npairs(case):
    """(4w-1)^2: visible pairs per image and head that index each table entry (the geometry alone)"""
    w = case[6]
    n = torch.zeros((4 * w - 1) ** 2, dtype=torch.float64)
    blocks, _ = offset_blocks(case)
    for _, idx, vis in blocks:
        n.index_add_(0, idx.reshape(-1), vis.sum(dim=(0, 1)).reshape(-1).double())
    return n


def _rounded(t, dtype):
    r = {n: None if t[n] is None else t[n].to(dtype).double() for n in ("q", "k", "v", "qg", "kg", "vg", "go", "gog")}
    r.update({n: None if t[n] is None else t[n].float().double() for n in ("table", "g2l", "g2g")})
    return r


def bias_grad_terms(t, case, dtype, keep=None, keep_g=None):
    """{name: (ref, T, npairs)} for dtable ((4w-1)^2, H), dg2l (2, H, g) and dg2g (H, g, g), plus "smax" (max |s| + max
    |lse| over the visible pairs) and the norms that make the floor.  keep / keep_g: test_gpu_dropout.keep_tensors."""
    B, H, D, nx, ny, g, w, exact, mode = case[:9]
    scale = D ** -0.5
    r = _rounded(t, dtype)
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    w2, tw, BH = w * w, 4 * w - 1, B * H
    blocks, real = offset_blocks(case)
    qc = _chunks(r["q"], nx, ny, w) * scale
    kc, vc = _chunks(r["k"][:, :, g:], nx, ny, w), _chunks(r["v"][:, :, g:], nx, ny, w)
    doc = _chunks(r["go"], nx, ny, w)
    heads = lambda x: x.reshape(1, H, *x.shape[1:]).expand(B, *x.shape).reshape(BH, *x.shape[1:])   # (H, ...) -> (BH, ...)
    bias = [heads(r["table"][idx.reshape(-1)].reshape(w2, w2, H).permute(2, 0, 1))[:, None, None] for _, idx, _ in blocks]
    ninf = torch.tensor(float("-inf"), dtype=torch.float64)

    def scores(oi):
        (dR, dC), _, vis = blocks[oi]
        s = torch.einsum("bmnld,bmntd->bmnlt", qc, _roll(kc, dR, dC)) + bias[oi]
        return torch.where(vis, s, ninf), vis

    def kcols(oi):                   # dropout factors of block oi (columns g + oi w2 ...)
        return 1.0 if keep is None else keep[..., g + oi * w2:g + (oi + 1) * w2]

    if g:
        kgl, vgl = r["k"][:, :, :g].reshape(BH, 1, 1, g, D), r["v"][:, :, :g].reshape(BH, 1, 1, g, D)
        s_glo = torch.einsum("bmnld,bmntd->bmnlt", qc, kgl.expand(BH, mx, my, g, D)) + \
            heads(r["g2l"][1])[:, None, None, None, :]
        s_glo = torch.where(real[None, ..., None], s_glo, ninf)
    # pass 1: lse over the global keys and every block; pass 2: o; pass 3: dS and the scatter
    lse = torch.logsumexp(s_glo, dim=-1) if g else torch.full((BH, mx, my, w2), float("-inf"), dtype=torch.float64)
    smax = float(s_glo[torch.isfinite(s_glo)].abs().max()) if g else 0.0
    for oi in range(len(blocks)):
        s, vis = scores(oi)
        lse = torch.logaddexp(lse, torch.logsumexp(s, dim=-1))
        if vis.any():
            smax = max(smax, float(s[vis.expand_as(s)].abs().max()))
    lse = torch.where(torch.isfinite(lse), lse, torch.zeros_like(lse))
    smax += float(lse.abs().max())
    prob = lambda s: torch.exp(s - lse[..., None])
    o = torch.zeros_like(qc)
    if g:
        pg_loc = prob(s_glo)
        o = o + torch.einsum("bmnlt,bmntd->bmnld", pg_loc * (1.0 if keep is None else keep[..., :g]), vgl.expand(BH, mx, my, g, D))
    for oi, ((dR, dC), _, _) in enumerate(blocks):
        o = o + torch.einsum("bmnlt,bmntd->bmnld", prob(scores(oi)[0]) * kcols(oi), _roll(vc, dR, dC))
    delta = (doc * o).sum(-1)
    ndo, no, nv = doc.norm(dim=-1), o.norm(dim=-1), vc.norm(dim=-1)
    out = {}
    tab = [torch.zeros(H, tw * tw, dtype=torch.float64) for _ in range(2)]
    npairs = torch.zeros(tw * tw, dtype=torch.float64)
    for oi, ((dR, dC), idx, vis) in enumerate(blocks):
        p = prob(scores(oi)[0])
        m = kcols(oi)
        dp = torch.einsum("bmnld,bmntd->bmnlt", doc, _roll(vc, dR, dC))
        ds = p * (dp * m - delta[..., None])
        T = p * ndo[..., None] * (m * _roll(nv, dR, dC)[..., None, :] + no[..., None])
        for acc, x in zip(tab, (ds, T)):
            acc.index_add_(1, idx.reshape(-1), x.reshape(B, H, -1, w2 * w2).sum(dim=(0, 2)))
        npairs.index_add_(0, idx.reshape(-1), vis.sum(dim=(0, 1)).reshape(-1).double())
    out["dtable"] = (tab[0].t().contiguous(), tab[1].t().contiguous(), (B * npairs)[:, None].expand(-1, H).contiguous())
    norms = dict(dO=float(ndo.max()), o=float(no.max()), v=float(nv.max()))
    mmax = 1.0 if keep is None else float(keep.max())
    if g:
        # local rows x global keys: g2l[1]
        m = 1.0 if keep is None else keep[..., :g]
        dp = torch.einsum("bmnld,bmntd->bmnlt", doc, vgl.expand(BH, mx, my, g, D))
        ds1 = (pg_loc * (dp * m - delta[..., None])).reshape(B, H, -1, g).sum(dim=(0, 2))
        T1 = (pg_loc * ndo[..., None] * (m * vgl.norm(dim=-1).unsqueeze(-2) + no[..., None])).reshape(B, H, -1, g).sum(dim=(0, 2))
        # global rows over all N keys: g2g (t < g) and g2l[0] (the local keys)
        qg, kg, vg, gog = r["qg"], r["kg"], r["vg"], r["gog"]
        sg = scale * torch.einsum("bhad,bhjd->bhaj", qg, kg) + \
            torch.cat([r["g2g"], r["g2l"][0][:, :, None].expand(H, g, nx * ny)], dim=-1)[None]
        lse_g = torch.logsumexp(sg, dim=-1)
        smax = max(smax, float(sg.abs().max()) + float(lse_g.abs().max()))
        pg = torch.exp(sg - lse_g[..., None])
        mg = 1.0 if keep_g is None else keep_g.reshape(B, H, g, -1)
        og = torch.einsum("bhaj,bhjd->bhad", pg * mg, vg)
        dsg = pg * (torch.einsum("bhad,bhjd->bhaj", gog, vg) * mg - (gog * og).sum(-1)[..., None])
        Tg = pg * gog.norm(dim=-1)[..., None] * (mg * vg.norm(dim=-1)[:, :, None, :] + og.norm(dim=-1)[..., None])
        ds0, T0 = dsg[..., g:].sum(dim=(0, 3)), Tg[..., g:].sum(dim=(0, 3))
        nl = float(B * nx * ny)
        out["dg2l"] = (torch.stack([ds0, ds1]), torch.stack([T0, T1]), torch.full((2, H, g), nl, dtype=torch.float64))
        out["dg2g"] = (dsg[..., :g].sum(0), Tg[..., :g].sum(0), torch.full((H, g, g), float(B), dtype=torch.float64))
        norms = dict(dO=max(norms["dO"], float(gog.norm(dim=-1).max())), o=max(norms["o"], float(og.norm(dim=-1).max())),
                     v=max(norms["v"], float(vg.norm(dim=-1).max()), float(r["v"].norm(dim=-1).max())))
        if keep_g is not None:
            mmax = max(mmax, float(keep_g.max()))
    out["smax"] = smax
    out["floor_unit"] = 2.0 ** -126 * norms["dO"] * (mmax * norms["v"] + norms["o"])
    return out


# --------------------------------------------------------------------------- holding the entries
def where_entry(name, idx, case):
    """an entry in the terms of the kernels: table displacement and the offsets whose windows reach it, or (part, h, t)"""
    w, mode = case[6], case[8]
    if name == "dtable":
        e, h = idx
        tw = 4 * w - 1
        dr, dc = e // tw - (2 * w - 1), e % tw - (2 * w - 1)
        reach = [(dR, dC) for dR, dC in vo.mode_offsets(mode) if abs(dr + dR * w) <= w - 1 and abs(dc + dC * w) <= w - 1]
        return "table entry %d head %d, displacement (dr, dc) = (%d, %d), window (u, v) = (dr + dR w, dc + dC w) of offsets %s" % (
            e, h, dr, dc, reach)
    if name == "dg2l":
        return "g2l[%d] head %d global token %d (%s)" % (idx + ("global rows x local keys" if idx[0] == 0 else "local rows x global keys",))
    return "g2g head %d global row %d global key %d" % idx


def _argmax(x):
    i = int(torch.where(torch.isnan(x), torch.full_like(x, float("inf")), x).argmax())
    return tuple(int(j) for j in torch.unravel_index(torch.tensor(i), x.shape))


def hold_entries(test, tag, out, terms, case, variant, whole=True):
    """every entry of the three gradients: exact zeros where no pair indexes it, err <= bar T_e + floor_e elsewhere"""
    D = case[2]
    smax = terms["smax"]
    bar = bar_of(variant, smax)
    nmax = max(float(terms[n][2].max()) for n in NAMES if n in terms)
    assert bar <= ceiling(variant, D, smax, nmax), (variant, bar, ceiling(variant, D, smax, nmax))
    vals, fails = {"smax": smax, "bar": bar}, []
    for name in NAMES:
        if name not in terms:
            continue
        ref, T, n = terms[name]
        x = out[name].detach().double().cpu()
        assert x.shape == ref.shape, (name, x.shape, ref.shape)
        zero = n == 0
        if zero.any():
            nz = zero & (x != 0)
            vals[name + ".structural_zeros"] = int(zero.sum())
            if nz.any():
                i = _argmax(nz.double())
                fails.append("%s: %d structural zeros are not 0.0, e.g. %.3e at %s (npairs 0)" % (
                    name, int(nz.sum()), float(x[i]), where_entry(name, i, case)))
        err = (x - ref).abs()
        floor = n * terms["floor_unit"]
        ratio = torch.where(zero, torch.zeros_like(err), (err - floor).clamp_min(0) / T.clamp_min(1e-300))
        ratio = torch.where(torch.isfinite(x), ratio, torch.full_like(ratio, float("inf")))
        i = _argmax(ratio)
        vals[name + ".err_over_T"] = float(ratio[i])
        vals[name + ".worst_npairs"] = float(n[i])
        vals[name + ".worst_entry"] = float(i[0])
        sparse = (n > 0) & (n <= 4 * case[0])
        if sparse.any():
            vals[name + ".sparse_err_over_T"] = float(ratio[sparse].max())
        if not float(ratio[i]) <= bar:
            fails.append("%s: err / T = %.3e (bar %.2e) at %s, npairs %d, out %.9e, ref %.9e, T %.3e" % (
                name, float(ratio[i]), bar, where_entry(name, i, case), int(n[i]), float(x[i]), float(ref[i]), float(T[i])))
        if whole:            # the whole-tensor bar of the other files, on this reference
            vals[name + ".relerr"] = relerr(x, ref)
            if not vals[name + ".relerr"] < tar.BIAS_BARS.get(variant, 1e-2):
                fails.append("%s: whole-tensor %.3e" % (name, vals[name + ".relerr"]))
    record(test, CASE_ID(case) + "/" + tag + "/" + variant, **vals)
    assert not fails, "\n".join(fails)


def run_variant(t, case, variant, drop=(0.0, 0, 0)):
    impl, dtype, f32out, layout = VARIANTS[variant]
    B, H, D, nx, ny, g, w, exact, mode = case[:9]
    out, fam_f, fam_b = tpar.kernel_run(t, nx, ny, w, exact, mode, D ** -0.5, dtype, impl, layout=layout, f32out=f32out,
                                        drop=drop)
    assert (fam_f, fam_b) == (impl, impl), (fam_f, fam_b)          # the family the variant names ran
    return out


def variants_for(case, names=None):
    """the SIMT backward stops at D = 64"""
    return [n for n in (names or VARIANTS) if not (VARIANTS[n][0] == "simt" and case[2] > 64)]


def expand(cases, names=None):
    return [pytest.param(c, v, id=CASE_ID(c) + "-" + v) for c in cases for v in variants_for(c, names)]


# --------------------------------------------------------------------------- cases
RANDOM_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode
    (2, 3, 32, 56, 56, 1, 7, 0, 0),         # ViL-Small stage 1
    (1, 2, 32, 15, 22, 1, 7, 0, 0),         # one real row and one real column in the last chunks
    (1, 2, 32, 14, 14, 1, 7, 1, 0),         # exact window
    (1, 2, 32, 23, 33, 2, 7, 0, 3),         # mode 3
    (1, 2, 32, 23, 33, 1, 7, 0, -1),        # own chunk only
    (1, 2, 16, 10, 9, 3, 4, -1, 0),         # cyclic chunks, 3 x 3 with padding
    (1, 2, 16, 8, 5, 1, 4, -1, 0),          # cyclic chunks, 2 x 2: chunks visited twice
    (1, 2, 32, 24, 24, 1, 12, 0, 0),        # w = 12, pieces ending mid-row
    (1, 2, 32, 30, 34, 0, 12, 1, 0),        # g = 0, exact window: wholly masked leading pieces
    (1, 1, 8, 19, 17, 2, 7, 0, 0),          # D = 8 (the SIMT HD-8 bucket)
    (1, 2, 48, 19, 17, 2, 7, 0, 0),         # D = 48
    (1, 2, 128, 26, 24, 1, 12, 0, 0),       # D = 128
]
MANY_GLOBAL_CASES = [
    (1, 2, 32, 14, 14, 64, 7, 0, 0, False),
    (1, 2, 32, 14, 14, 65, 7, 0, 0, True),
    (1, 2, 32, 24, 24, 130, 12, 0, 0, True),
]
DROP_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, separate global weights, p
    (1, 2, 32, 14, 15, 2, 7, 1, 0, False, 0.1),
    (1, 2, 32, 14, 15, 2, 7, 1, 0, True, 0.5),
    (1, 2, 16, 8, 5, 1, 4, -1, 0, False, 0.1),
    (1, 2, 16, 8, 5, 1, 4, -1, 0, False, 0.5),
    (1, 2, 128, 15, 13, 1, 7, 0, 0, False, 0.1),
    (1, 2, 128, 15, 13, 1, 7, 0, 0, True, 0.5),
]
SLICE_CASES = [(11, 64, 16, 8, 5, 1, 4, -1, 0)]
S1_B13 = (13, 3, 32, 56, 56, 1, 7, 0, 0)
LARGE_CASES = [
    # w, what it reaches
    (1, 1, 32, 40, 35, 1, 16, 0, 0),        # 16: four full pieces
    (1, 1, 32, 45, 41, 1, 20, 1, 0),        # 20: exact window, a 16-slot last piece
    (1, 1, 64, 62, 40, 1, 31, 0, 0),        # 31: 16 pieces, 15 129 entries
    (1, 1, 128, 50, 47, 1, 42, 0, 0),       # 42: the HD 128 pass-1 limit (wgmma only)
    (1, 1, 64, 60, 53, 1, 48, 0, 0),        # 48: the largest table, 32 bytes under the pass-1 limit at HD <= 64
    (1, 1, 32, 60, 53, 2, 48, 0, 3),        # 48, mode 3
    (1, 1, 32, 50, 50, 0, 48, -1, 0),       # 48, cyclic chunks on a 2 x 2 grid
]
SEED, OFFSET = 0x5eed0000b1a5, 4321
ALL_CASES = RANDOM_CASES + MANY_GLOBAL_CASES + [c[:10] for c in DROP_CASES] + SLICE_CASES + [S1_B13] + LARGE_CASES


def structural_zero_claims(case):
    """(4w-1)^2 bool: entries that no pair can index by the geometry of the walk alone"""
    B, H, D, nx, ny, g, w, exact, mode = case[:9]
    tw = 4 * w - 1
    d = torch.arange(tw) - (2 * w - 1)
    dr, dc = d[:, None].expand(tw, tw), d[None, :].expand(tw, tw)
    reach = torch.zeros(tw, tw, dtype=torch.bool)
    for dR, dC in vo.mode_offsets(mode):
        reach |= ((dr + dR * w).abs() <= w - 1) & ((dc + dC * w).abs() <= w - 1)
    zero = ~reach
    if exact == 1:
        zero |= (dr.abs() > w) | (dc.abs() > w)
    padx, pady, mx, my = vo.geometry(nx, ny, w)
    if exact != -1:
        zero |= dr.abs() >= nx       # no two real tokens that far apart
        zero |= dc.abs() >= ny
        if mx == 1:
            zero |= dr.abs() >= w
        if my == 1:
            zero |= dc.abs() >= w
    return zero.reshape(-1)


# --------------------------------------------------------------------------- CPU: the restatement pinned to autograd
PIN_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, separate global weights
    (2, 2, 8, 9, 11, 1, 4, 0, 0, False),     # padding in both directions
    (1, 2, 8, 11, 9, 3, 4, 1, 0, True),      # exact window, g = 3, separate global weights
    (1, 2, 8, 10, 9, 0, 4, -1, 0, False),    # cyclic 3 x 3, g = 0
    (1, 2, 8, 8, 5, 1, 4, -1, 0, False),     # cyclic 2 x 2: two offsets reach one chunk
    (1, 1, 8, 10, 13, 3, 4, 0, -1, True),    # own chunk only
    (1, 2, 8, 11, 10, 1, 4, 0, 3, False),    # mode 3
    (1, 2, 8, 11, 10, 3, 4, 0, 8, True),     # mode 8
    (1, 1, 8, 12, 12, 1, 4, 1, 0, False),    # exact window, no padding
]


def _autograd_bias(t, case, dtype, fn, **extra):
    B, H, D, nx, ny, g, w, exact, mode = case[:9]
    r = _rounded(t, dtype)
    leaves = {n: r[n].clone().requires_grad_(True) for n in ("table", "g2l", "g2g") if r[n] is not None}
    sep = t["kg"] is not t["k"]
    kg, vg = (r["kg"], r["vg"]) if sep else (r["k"], r["v"])
    res = fn(r["q"], r["k"], r["v"], r["qg"] if g else None, kg, vg, leaves.get("table"), leaves.get("g2l"), leaves.get("g2g"),
             nx=nx, ny=ny, w=w, exact=exact, mode=mode, scale=D ** -0.5, **extra)
    o, og = res[0], res[1]
    loss = (o * r["go"]).sum() + ((og * r["gog"]).sum() if g else 0)
    grads = torch.autograd.grad(loss, list(leaves.values()))
    return {"d" + n: x for n, x in zip(leaves, grads)}


def _pin(terms, auto):
    for name, x in auto.items():
        ref, T, n = terms[name]
        err = (ref - x).abs()
        assert bool((err <= 1e-12 * T).all()), (name, float((err / T.clamp_min(1e-300)).max()))
        assert bool((ref[n == 0] == 0).all()) and bool((x[n == 0] == 0).all()), name


@pytest.mark.parametrize("case", PIN_CASES, ids=CASE_ID)
def test_restatement_matches_the_dense_oracle(case):
    t = tar.make_inputs(full(case), seed=400, sep=case[9])
    terms = bias_grad_terms(t, case, F32)
    _pin(terms, _autograd_bias(t, case, F32, vo.dense_attention))
    assert case[5] == 0 or ("dg2l" in terms and "dg2g" in terms)


@pytest.mark.parametrize("case", [c for c in PIN_CASES if c[7] == -1], ids=CASE_ID)
def test_restatement_matches_the_chunked_oracle_on_cyclic_grids(case):
    t = tar.make_inputs(full(case), seed=401, sep=case[9])
    _pin(bias_grad_terms(t, case, BF16), _autograd_bias(t, case, BF16, vo.chunked_attention))


@pytest.mark.parametrize("case", [PIN_CASES[1], PIN_CASES[3], PIN_CASES[5]], ids=CASE_ID)
def test_restatement_matches_the_dropout_reference(case):
    B, H, D, nx, ny, g, w, exact, mode = case[:9]
    t = tar.make_inputs(full(case), seed=402, sep=case[9])
    keep, keep_g = tdrop.keep_tensors(SEED, OFFSET, 0.1, B, H, nx, ny, w, g, mode)
    terms = bias_grad_terms(t, case, F16, keep, keep_g)
    auto = _autograd_bias(t, case, F16, tdrop.chunked_dropout_reference, keep=keep, keep_g=keep_g)
    _pin(terms, auto)
    # the mask matters: the reference without it is off by O(1) in the table
    assert relerr(bias_grad_terms(t, case, F16)["dtable"][0], auto["dtable"]) > 1e-2


def test_restatement_counts_the_visits_of_the_dense_oracle():
    """sum over the table of npairs = the visits of vo.visit_weights (two per pair that two wrapped offsets reach)"""
    for case in PIN_CASES + RANDOM_CASES[1:8]:
        B, H, D, nx, ny, g, w, exact, mode = case[:9]
        E = vo.visit_weights(nx, ny, w, exact, mode, None, 1)
        assert float(table_npairs(case).sum()) == float(E.sum()), case


def claims_sparse(case):
    """mode 0 without the exact window on a grid of at most about 7 x 7 chunks: the corner entries of the table collect
    one pair per chunk pair, and the chunk pairs of the far offsets are few (an 8 x 8 grid has 49 of them)"""
    return case[7] != 1 and case[8] == 0 and case[3] * case[4] < 3000


@pytest.mark.parametrize("case", ALL_CASES, ids=CASE_ID)
def test_cases_have_structural_zeros_and_sparse_entries(case):
    """the zeros the geometry implies (entries no offset's window reaches, |dr| or |dc| > w under exact = 1, the rows or
    columns an image does not span) are zeros of npairs; the cases that claim sparse entries have entries of 1 to 4
    pairs per image"""
    n = table_npairs(case)
    claim = structural_zero_claims(case)
    assert bool((n[claim] == 0).all())
    if case[7] == 1 or case[8] in (-1, 3):
        assert int(claim.sum()) > 0
    if claims_sparse(case):
        assert int(((n > 0) & (n <= 4)).sum()) > 0, float(n[n > 0].min())


def test_most_cases_claim_sparse_entries():
    assert sum(claims_sparse(c) for c in ALL_CASES) >= len(ALL_CASES) // 2


@pytest.mark.parametrize("case", ALL_CASES + [tar.PK_TABLE[:9]], ids=CASE_ID)
def test_bars_stay_under_the_ceiling(case):
    """bar <= ceiling for every variant a case runs (the 2 smax 2^-24 of the bar is in the ceiling as well)"""
    B, D, g = case[0], case[2], case[5]
    nmax = max(float(B * table_npairs(case).max()), float(B * case[3] * case[4]) if g else 0.0)
    for v in variants_for(case):
        assert bar_of(v, 0.0) <= ceiling(v, D, 0.0, nmax), (v, KAPPA[v], ceiling(v, D, 0.0, nmax))


def test_batch_cases_run_several_images_per_pass1_cta():
    for case in SLICE_CASES + [S1_B13]:
        assert nslice_of_the_library(case) < case[0], case


# --------------------------------------------------------------------------- CPU: shared memory of the large windows
CAP = 227 * 1024
K_KEY_COLS, K_QUERY_COLS, K_VISITS, K_DS_TILE = 64 * 12, 64 * 17, 9 * 24, 64 * 72 * 4     # vil_wgmma.cuh
stages = lambda HD: 3 if HD <= 64 else 2
up16 = lambda n: (n + 15) & ~15
head_tile = lambda D: 16 if D <= 16 else 32 if D <= 32 else 64 if D <= 64 else 128


def fwd_smem(HD, tabn):
    return up16((1 + 2 * stages(HD)) * 64 * HD * 2 + stages(HD) * K_KEY_COLS + K_VISITS + 4 * tabn)


def dq_smem(HD, tabn):
    return up16((2 + 2 * stages(HD)) * 64 * HD * 2 + stages(HD) * K_KEY_COLS + K_VISITS + 4 * tabn) + K_DS_TILE


def dkv_smem(HD, tabn, drop=False):
    return up16((2 + 2 * stages(HD)) * 64 * HD * 2 + stages(HD) * (K_QUERY_COLS + (256 if drop else 0)) + K_VISITS + 256 + 4 * tabn)


@pytest.mark.parametrize("D,w,fits", [(64, 48, True), (32, 48, True), (128, 42, True), (128, 43, False), (64, 31, True),
                                      (32, 20, True), (32, 16, True)])
def test_large_window_shared_memory_matches_the_library(D, w, fits):
    import __graft_entry__ as ge
    ge.build()
    from vision_longformer_b200 import _lib
    HD, tabn = head_tile(D), (4 * w - 1) ** 2
    room = {"fwd": CAP - fwd_smem(HD, tabn), "dq": CAP - dq_smem(HD, tabn), "dkv": CAP - dkv_smem(HD, tabn),
            "dkv_dropout": CAP - dkv_smem(HD, tabn, True)}
    print("D %d (tile %d) w %d: bytes to spare %s" % (D, HD, w, room))
    assert (min(room.values()) >= 0) == fits, room
    lib = _lib.load()
    p = _params(B=1, H=1, D=D, nx=2 * w, ny=2 * w, w=w, nglo=1, bias_table=256, g2l=256, g2g=256)
    assert lib.vil_attn_wgmma_supported(ctypes.byref(p)) == (1 if fits else 0)
    if (D, w) == (64, 48):
        assert room["dq"] == 32                  # 232 416 of 232 448 bytes
    if (D, w) == (128, 42):
        assert dq_smem(128, tabn) == 230048


# --------------------------------------------------------------------------- GPU: per-entry parity
_TERMS = {}


def terms_of(key, t, case, dtype, keep=None, keep_g=None):
    if (key, dtype) not in _TERMS:
        if any(k[0] != key for k in _TERMS):
            _TERMS.clear()
        _TERMS[(key, dtype)] = bias_grad_terms(t, case, dtype, keep, keep_g)
    return _TERMS[(key, dtype)]


@gpu
@pytest.mark.parametrize("case,variant", expand(RANDOM_CASES + MANY_GLOBAL_CASES))
def test_entries_random_inputs(case, variant):
    t = tar.make_inputs(full(case), seed=410, sep=full(case)[10])
    terms = terms_of(("rand",) + case, t, case, VARIANTS[variant][1])
    hold_entries("bias_entries_random_inputs", "randn", run_variant(t, case, variant), terms, case, variant)


@gpu
@pytest.mark.parametrize("case,variant", expand(DROP_CASES))
def test_entries_dropout(case, variant):
    B, H, D, nx, ny, g, w, exact, mode, sep, p = case
    t = tar.make_inputs(full(case), seed=411, sep=sep)
    keep, keep_g = tdrop.keep_tensors(SEED, OFFSET, p, B, H, nx, ny, w, g, mode)
    terms = terms_of(("drop",) + case, t, case, VARIANTS[variant][1], keep, keep_g)
    out = run_variant(t, case, variant, drop=(p, SEED, OFFSET))
    hold_entries("bias_entries_dropout", "p%g" % p, out, terms, case, variant)


@gpu
@pytest.mark.parametrize("case,variant", expand(SLICE_CASES) + expand([S1_B13], ["wgmma_bf16_linear"]))
def test_entries_several_images_per_pass1_cta(case, variant):
    assert nslice_of_the_library(case) < case[0]
    t = tar.make_inputs(full(case), seed=412)
    terms = terms_of(("slices",) + case, t, case, VARIANTS[variant][1])
    hold_entries("bias_entries_several_images_per_cta", "randn", run_variant(t, case, variant), terms, case, variant)


@gpu
@pytest.mark.parametrize("variant", tar.PEAK_VARIANTS)
@pytest.mark.parametrize("L", tar.GAPS)
@pytest.mark.parametrize("what", tar.TABLE_PEAKS, ids=lambda x: "_".join(str(y) for y in x))
def test_entries_peaked_through_the_bias(what, L, variant):
    """test_gpu_attention_rows' peaked bias cases, the bias gradients held per entry: under a saturated softmax the dS of
    the dominant key is a cancellation of terms of size T_e, and the floor covers the flushed P under a -L band"""
    case = tar.PK_TABLE[:9]
    t = tar.peak_through_table(tar.make_inputs(tar.PK_TABLE, seed=321), tar.PK_TABLE, L, what)
    terms = bias_grad_terms(t, case, VARIANTS[variant][1])
    hold_entries("bias_entries_peaked_through_the_bias", "%s_L%d" % ("_".join(str(x) for x in what), L),
                 run_variant(t, case, variant), terms, case, variant, whole=False)


@gpu
@pytest.mark.parametrize("case,variant", expand(LARGE_CASES))
def test_entries_large_windows(case, variant, monkeypatch):
    """w = 16 ... 48 with the table: o, dq, dk, dv and lse row by row at test_gpu_attention_rows' bars, the bias
    gradients per entry"""
    fc = full(case)
    t = tar.make_inputs(fc, seed=413)
    dtype = VARIANTS[variant][1]
    out = run_variant(t, case, variant)
    ref = tar.oracle(t, tar.cfg_of(fc), dtype, ("large",) + case)
    if variant == "simt_fp32" and case[7] == -1:
        # exact = -1 on a 2 x 2 grid at w = 48: nine offsets reach four chunks, 20 736 columns per row, the longest fp32
        # sums of any case (9x a w = 48 chunk; 1.3x the worst row of tar's w = 31).  Its row bars, set at w <= 31, are
        # taken 1.5 times (measured on an H100: o row 6.0e-6, lse 5.8e-6)
        b = tar.BARS[variant]
        monkeypatch.setitem(tar.BARS, variant, dict(row=tuple(1.5 * x for x in b["row"]),
                                                    chunk=tuple(1.5 * x for x in b["chunk"]), lse=1.5 * b["lse"]))
    tar.check("bias_entries_large_windows", "randn", out, ref, fc, variant if variant in tar.BARS else "wgmma_bf16", bias=False)
    hold_entries("bias_entries_large_windows", "randn", out, terms_of(("large",) + case, t, case, dtype), case, variant)


# --------------------------------------------------------------------------- GPU: the contract
CONTRACT_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, separate global weights, p
    (1, 2, 32, 15, 13, 2, 7, 1, 0, True, 0.1),      # exact window, separate global weights, dropout
    (1, 2, 32, 15, 13, 2, 7, 0, 0, False, 0.0),
    (11, 64, 16, 8, 5, 1, 4, -1, 0, False, 0.0),    # B > nslice
    (11, 64, 16, 8, 5, 1, 4, -1, 0, False, 0.5),
]


@gpu
@pytest.mark.parametrize("impl", ["simt", "wgmma"])
@pytest.mark.parametrize("case", [c for c in CONTRACT_CASES if c[10] > 0 or c[0] > 1], ids=lambda c: CASE_ID(c) + "_p%g" % c[10])
def test_bias_gradients_are_accumulated_into(case, impl, monkeypatch):
    """d_bias_table, d_g2l and d_g2g pre-filled with X come back as X + the clean result, bit for bit: the kernel adds
    one fp32 sum into each element"""
    B, H, D, nx, ny, g, w, exact, mode, sep, p = case
    dtype = F32 if impl == "simt" else BF16
    t = tar.make_inputs(full(case), seed=420, sep=sep)
    run = lambda: tpar.kernel_run(t, nx, ny, w, exact, mode, D ** -0.5, dtype, impl, drop=(p, SEED, OFFSET))
    clean, fam_f, fam_b = run()
    assert (fam_f, fam_b) == (impl, impl)
    gen = torch.Generator().manual_seed(421)
    X = {n: torch.randn(clean[n].shape, generator=gen).to(clean[n].device) * float(clean[n].abs().max())
         for n in NAMES}
    orig = tpar.vil_attention_raw_backward

    def prefilled(*a, **kw):
        a = list(a)
        for i, n in zip((21, 22, 23), NAMES):
            a[i].copy_(X[n])
        return orig(*a, **kw)

    monkeypatch.setattr(tpar, "vil_attention_raw_backward", prefilled)
    acc, _, _ = run()
    for n in NAMES:
        assert torch.equal(acc[n], X[n] + clean[n]), (n, float((acc[n] - X[n] - clean[n]).abs().max()))


@gpu
@pytest.mark.parametrize("rpe", [True, False], ids=["table", "no_table"])
@pytest.mark.parametrize("impl", ["simt", "wgmma"])
@pytest.mark.parametrize("case", CONTRACT_CASES, ids=lambda c: CASE_ID(c) + "_p%g" % c[10])
def test_dirty_workspace_changes_no_output_bit(case, impl, rpe, monkeypatch):
    """the workspace filled with 0xFF bytes (NaN as fp32) before every call: forward and backward outputs bit-identical
    to a run whose workspace was zero-filled"""
    from vision_longformer_b200 import ops
    B, H, D, nx, ny, g, w, exact, mode, sep, p = case
    dtype = F32 if impl == "simt" else BF16
    t = tar.make_inputs(tuple(case[:9]) + (rpe, sep), seed=422, sep=sep)
    orig = ops._workspace
    outs = []
    for byte in (0x00, 0xFF):
        def filled(*a, _b=byte, **kw):
            ws = orig(*a, **kw)
            ws.fill_(_b)
            return ws
        monkeypatch.setattr(ops, "_workspace", filled)
        out, fam_f, fam_b = tpar.kernel_run(t, nx, ny, w, exact, mode, D ** -0.5, dtype, impl, drop=(p, SEED, OFFSET))
        assert (fam_f, fam_b) == (impl, impl)
        outs.append(out)
    if rpe:
        assert outs[0]["dtable"] is not None
    for n, x in outs[0].items():
        if x is not None:
            assert torch.equal(x, outs[1][n]), n
