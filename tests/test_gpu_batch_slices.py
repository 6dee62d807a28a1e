"""Backward pass 1 with the relative-position bias table at batch sizes where one CTA serves several images.

With the table, pass 1 launches nslice * H * mx * my * npc CTAs, nslice = min(B, ceil(8 * 132 / (H * mx * my * npc))),
and CTA slice s runs images s, s + nslice, ... one after another (vil_common.cuh, Geo::nslice).  Per image it restages
Q and dO, reloads lse and delta, rebuilds the visit list and writes dQ, while it keeps adding into one row of table
partials; simt_bwd_bias_reduce then sums the rows slice by slice.  Every case here has nslice < B, so a mistake that
only shows from the second image of a slice on (the first image's lse / delta, partials zeroed per image, dQ written to
the first image's rows, a missing barrier between images) shows in dQ or the bias gradients.

CPU tests: nslice, read back from the workspace size, is the formula above, and the cases run several images per CTA.
GPU tests: parity with the fp64 references over the whole tensor and image by image (an error confined to some images is
diluted by about sqrt(B) in a whole-tensor norm); image b of a B-image call is bitwise a one-image call on image b, and
the batched bias gradients are the sum of the one-image ones; ViL-Small stage 1 at B = 13 against the chunked oracle.
"""
import pytest
import torch

from oracle import vil_oracle as vo
from tests import test_gpu_dropout as dp
from tests import test_gpu_parity as tp
from tests.test_gpu_deterministic import CASE_ID, _ws, align64
from tests.util import record, relerr

gpu = pytest.mark.gpu

# all with the bias table; (per_slice, nslice, most images per CTA) in the comments
CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, separate global weights, p
    (11, 32, 16, 14, 14, 1, 7, 0, 0, False, 0.0),      # (128, 9, 2) HD 16 tile
    (10, 16, 32, 21, 19, 3, 7, 1, 0, True, 0.1),       # (144, 8, 2) exact window, padding, 3 global tokens, dropout
    (11, 64, 16, 8, 5, 1, 4, -1, 0, False, 0.0),       # (256, 5, 3) cyclic chunks on a 2 x 2 grid, a slice of 3 images
    (13, 8, 64, 24, 26, 1, 12, 0, 3, False, 0.0),      # (144, 8, 2) 3 pieces per chunk, random-shift mode
    (19, 16, 128, 14, 14, 1, 7, 0, 0, False, 0.1),     # (64, 17, 2) HD 128 tile (2-stage ring), dropout
    (12, 32, 32, 12, 12, 0, 6, 0, 0, False, 0.0),      # (128, 9, 2) no global tokens (no global-bias partials)
]
S1_B13 = (13, 3, 32, 56, 56, 1, 7, 0, 0, False, 0.0)   # ViL-Small stage 1: (192, 6, 3), slice 0 runs images 0, 6, 12
S1_B64 = (64, 3, 32, 56, 56, 1, 7, 0, 0, False, 0.0)   # (192, 6, 11)
SEED, OFFSET = 0x5eed0000f00d, 91


# --------------------------------------------------------------------------- CPU: every case reaches the multi-image path
def per_slice(case):
    B, H, D, nx, ny, g, w = case[:7]
    _, _, mx, my = vo.geometry(nx, ny, w)
    return H * mx * my * -(-w * w // 64)


def nslice_of_the_library(case):
    """nslice from the workspace size: the table adds 4 align64(nslice per_slice (4w-1)^2) bytes of partials, and with
    global tokens 4 align64(B H g (2 + g)) of global-bias partials"""
    B, H, D, nx, ny, g, w, exact, mode = case[:9]
    kw = dict(B=B, H=H, D=D, nx=nx, ny=ny, nglo=g, w=w, exact=exact, mode=mode, scale=D ** -0.5)
    rpe = dict(bias_table=256, g2l=256, g2g=256) if g else dict(bias_table=256)    # never dereferenced
    grown = _ws(**kw, **rpe) - _ws(**kw)
    if g:
        grown -= 4 * align64(B * H * g * (2 + g))
    fits = [n for n in range(1, B + 1) if 4 * align64(n * per_slice(case) * (4 * w - 1) ** 2) == grown]
    assert len(fits) == 1, (grown, fits)
    return fits[0]


@pytest.mark.parametrize("case", CASES + [S1_B13, S1_B64], ids=CASE_ID)
def test_pass1_ctas_run_several_images(case):
    B = case[0]
    ns = nslice_of_the_library(case)
    assert ns == min(B, -(-8 * 132 // per_slice(case)))
    assert ns < B


def test_the_oracle_cases_reach_three_images_per_cta_and_a_short_last_round():
    ns = {c: nslice_of_the_library(c) for c in CASES}
    assert any(-(-c[0] // ns[c]) >= 3 for c in CASES), ns
    assert any(c[0] % ns[c] for c in CASES), ns


# --------------------------------------------------------------------------- GPU: fp64 parity, whole tensor and per image
# family, dtype, VIL_FLAG_F32_OUT, forward / backward / bias-gradient bars (test_gpu_dropout's), layout
VARIANTS = {n: v + ("contig",) for n, v in dp.VARIANTS.items()}
VARIANTS["wgmma_bf16_linear"] = dp.VARIANTS["wgmma_bf16"] + ("linear",)
PARITY = [(c, v) for c in CASES for v in VARIANTS if not (VARIANTS[v][0] == "simt" and c[2] > 64)]   # case-major
_REF = {}


def _rounded(t, dtype):
    """the inputs as the kernel sees them (the bias parameters in fp32), in fp64; all but dO are autograd leaves"""
    rd = lambda n, x: (x.float() if n in ("table", "g2l", "g2g") else x.to(dtype)).double().requires_grad_(n[:2] != "go")
    return {n: None if x is None else rd(n, x) for n, x in t.items()}


def dense_lse(r, case):
    """lse of the dense fp64 oracle, image by image (its memory grows with the square of the image)"""
    B, H, D, nx, ny, g, w, exact, mode = case[:9]
    kw = dict(nx=nx, ny=ny, w=w, exact=exact, mode=mode, scale=D ** -0.5)
    im = lambda n, b: r[n][b:b + 1] if g or n in ("q", "k", "v") else None
    with torch.no_grad():
        return torch.cat([vo.dense_attention(im("q", b), im("k", b), im("v", b), im("qg", b), im("kg", b), im("vg", b),
                                             r["table"], r["g2l"], r["g2g"], **kw)[2] for b in range(B)])


def reference(case, t, dtype):
    """fp64 reference on the inputs rounded to `dtype`: the dense oracle, or with dropout / separate global weights the
    chunked reference with the restated mask.  Kept for the variants of the current case only."""
    if (case, dtype) not in _REF:
        if any(k[0] != case for k in _REF):
            _REF.clear()
        B, H, D, nx, ny, g, w, exact, mode, sep, p = case
        cfg = (nx, ny, w, exact, mode, D ** -0.5)
        if p == 0 and not sep:
            ref = tp.oracle_run(t, *cfg, dtype)
        else:
            if (case, "keep") not in _REF:
                _REF[(case, "keep")] = dp.keep_tensors(SEED, OFFSET, p, B, H, nx, ny, w, g, mode)
            ref = dp.reference_run(t, cfg, dtype, *_REF[(case, "keep")])
            ref["lse"] = dense_lse(_rounded(t, dtype), case)
        _REF[(case, dtype)] = {n: None if x is None else x.detach() for n, x in ref.items()}
    return _REF[(case, dtype)]


def check(out, ref, case, variant, bars, test):
    """test_gpu_parity's bars (forward tf, lse 1e-4, backward tb, bias gradients tbias) over the whole tensor, and image
    by image for everything but the bias gradients, which are sums over the images"""
    B = case[0]
    tf, tb, tbias = bars
    names = [n for n in ("o", "lse", "dq", "dk", "dv", "og", "dqg", "dkg", "dvg") if ref.get(n) is not None]
    bias = [n for n in ("dtable", "dg2l", "dg2g") if ref.get(n) is not None]
    bar = lambda n: tf if n in ("o", "og") else 1e-4 if n == "lse" else tbias if n in bias else tb
    errs = {n: relerr(out[n], ref[n]) for n in names + bias}
    errs.update({"%s[%d]" % (n, b): relerr(out[n][b], ref[n][b]) for n in names for b in range(B)})
    record(test, CASE_ID(case) + "/" + variant, **errs)
    bad = {k: e for k, e in errs.items() if not e < bar(k.split("[")[0])}
    assert not bad, bad


@gpu
@pytest.mark.parametrize("case,variant", PARITY, ids=[CASE_ID(c) + "-" + v for c, v in PARITY])
def test_matches_reference_image_by_image(case, variant):
    impl, dtype, f32out, tf, tb, tbias, layout = VARIANTS[variant]
    B, H, D, nx, ny, g, w, exact, mode, sep, p = case
    t = dp.make_inputs(B, H, D, nx, ny, g, w, True, sep, seed=320)
    out, fam_f, fam_b = tp.kernel_run(t, nx, ny, w, exact, mode, D ** -0.5, dtype, impl, layout=layout, f32out=f32out,
                                      drop=(p, SEED, OFFSET))
    assert (fam_f, fam_b) == (impl, impl)
    check(out, reference(case, t, dtype), case, variant, (tf, tb, tbias), "batch_slices_matches_reference")


@gpu
def test_vil_small_stage1_matches_the_chunked_oracle_image_by_image():
    """B = 13, nslice 6: slice 0 runs images 0, 6 and 12.  The dense oracle would need tens of GB here; the chunked one
    (pinned to the reference goldens by test_oracle) has linear memory.  It forms no lse; the forward runs one image per
    CTA whatever B, test_gpu_parity checks its lse at this image size, and the B = 64 test below each image's."""
    case = S1_B13
    B, H, D, nx, ny, g, w, exact, mode, sep, p = case
    t = dp.make_inputs(B, H, D, nx, ny, g, w, True, sep, seed=340)
    out, fam_f, fam_b = tp.kernel_run(t, nx, ny, w, exact, mode, D ** -0.5, torch.bfloat16, "wgmma", layout="linear")
    assert (fam_f, fam_b) == ("wgmma", "wgmma")
    r = _rounded(t, torch.bfloat16)
    kw = dict(nx=nx, ny=ny, w=w, exact=exact, mode=mode, scale=D ** -0.5)
    o, og = vo.chunked_attention(r["q"], r["k"], r["v"], r["qg"], r["k"], r["v"], r["table"], r["g2l"], r["g2g"], **kw)
    loss = (o * r["go"]).sum() + (og * r["gog"]).sum()
    names = ("q", "k", "v", "qg", "table", "g2l", "g2g")
    grads = torch.autograd.grad(loss, [r[n] for n in names])
    ref = dict(o=o.detach(), og=og.detach(), **{"d" + n: x for n, x in zip(names, grads)})
    check(out, ref, case, "wgmma_bf16_linear", VARIANTS["wgmma_bf16_linear"][3:6], "batch_slices_vil_small_stage1")


# --------------------------------------------------------------------------- GPU: batch invariance, bit for bit
def _image(t, b):
    one = {n: x if x is None or n in ("table", "g2l", "g2g") else x[b:b + 1] for n, x in t.items()}
    if t["kg"] is t["k"]:
        one["kg"], one["vg"] = one["k"], one["v"]
    return one


def batch_invariance(case, impl, dtype, layout, test):
    """Pass 1 resets its dQ accumulator per image, and everything else is per image as well: image b of the batched
    call equals a one-image call (nslice 1) bit for bit.  The bias gradients are sums over the images; their fp32
    partials are added in another order, so they agree with the fp64 sum of the one-image results to rounding."""
    B, H, D, nx, ny, g, w, exact, mode, sep, p = case
    t = dp.make_inputs(B, H, D, nx, ny, g, w, True, sep, seed=330)
    run = lambda x: tp.kernel_run(x, nx, ny, w, exact, mode, D ** -0.5, dtype, impl, layout=layout)
    full, fam_f, fam_b = run(t)
    assert (fam_f, fam_b) == (impl, impl)
    bias = [n for n in ("dtable", "dg2l", "dg2g") if full[n] is not None]
    sums = {n: torch.zeros(full[n].shape, dtype=torch.float64) for n in bias}
    for b in range(B):
        one, _, _ = run(_image(t, b))
        for n, x in one.items():
            if n in sums:
                sums[n] += x.double().cpu()
            elif x is not None:
                assert torch.equal(full[n][b:b + 1], x), (b, n)
    errs = {n: relerr(full[n], sums[n]) for n in bias}
    record(test, CASE_ID(case) + "/%s_%s" % (impl, layout), **errs)
    assert all(e < 1e-4 for e in errs.values()), errs     # measured on an H100: at most 3.8e-7 (B = 64)


INVARIANCE = [(c[:10] + (0.0,), impl, layout) for c in CASES for impl in ("wgmma", "simt") for layout in ("contig", "linear")
              if not (impl == "simt" and c[2] > 64)]


@gpu
@pytest.mark.parametrize("case,impl,layout", INVARIANCE, ids=["%s-%s-%s" % (CASE_ID(c), i, l) for c, i, l in INVARIANCE])
def test_each_image_is_bitwise_a_one_image_call(case, impl, layout):
    batch_invariance(case, impl, torch.bfloat16 if impl == "wgmma" else torch.float32, layout, "batch_slices_invariance")


@gpu
def test_each_image_is_bitwise_a_one_image_call_at_vil_small_stage1():
    """B = 64: every pass-1 CTA runs 10 or 11 images"""
    batch_invariance(S1_B64, "wgmma", torch.bfloat16, "linear", "batch_slices_invariance")
