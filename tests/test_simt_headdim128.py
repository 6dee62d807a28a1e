"""fp32 training at head dims 64 < D <= 128 on the SIMT family: the local kernels at four lanes per row (vil_simt.cuh,
L = 4, Tile<128, 4>).

The fp32 backward at D > 64 and the fp32 dropout forward at D > 64 run simt_bwd_dq<float, 128, 4, DROP, TAB> /
simt_bwd_dkv<float, 128, 4, DROP> / simt_fwd_local<float, 128, 4, true>; the forward without dropout stays on the
two-lane kernel.  Everything is held with the machinery of the other files, at their SIMT fp32 bars:
  rows and chunks of every output against the fp64 dense oracle     test_gpu_attention_rows (check, oracle)
  the bias gradients entry by entry                                  test_gpu_bias_entries (hold_entries)
  dropout against the exact-mask restatement                         test_gpu_dropout (reference_run)
plus the contracts of the backward (repeatability, images of a batch, accumulation into the bias gradients, a dirty
workspace) and module-level training.  The variant lists of those files leave SIMT out at D > 64; the cases here are
this file's own.

CPU tests: the B > nslice case runs several images per pass-1 CTA, the masked case has wholly masked leading pieces, and
the pass-1 shared memory at w = 48 fits beside the table with the four-quarter tile row.
"""
import math

import pytest
import torch

from tests import test_gpu_attention_rows as tar
from tests import test_gpu_bias_entries as tbe
from tests import test_gpu_dropout as tdrop
from tests import test_gpu_parity as tpar
from tests.test_gpu_batch_slices import nslice_of_the_library
from tests.util import record, relerr
from vision_longformer_b200 import _lib

DEV = "cuda"
gpu = pytest.mark.gpu
F32 = torch.float32
VARIANT = "simt_fp32"

# --------------------------------------------------------------------------- cases
ROW_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, rpe
    (1, 1, 128, 56, 56, 1, 7, 0, 0, False),    # ViL-like stage-1 grid
    (1, 2, 96, 28, 28, 1, 7, 0, 0, True),      # the bias table
    (1, 1, 72, 19, 17, 2, 7, 0, 0, True),      # padding in both directions, D = 72
    (1, 2, 100, 18, 15, 1, 6, 1, 0, True),     # exact window, D % 8 != 0 (no wgmma kernel takes it)
    (1, 2, 128, 8, 5, 1, 4, -1, 0, False),     # cyclic chunks on a 2 x 2 grid: chunks visited twice
    (1, 2, 128, 23, 33, 1, 7, 0, -1, True),    # own chunk only
    (1, 2, 128, 23, 33, 2, 7, 0, 3, False),    # random-shift mode 3
    (1, 2, 128, 24, 24, 1, 12, 0, 0, True),    # w = 12: three pieces per chunk
    (1, 2, 128, 12, 12, 0, 6, 0, 0, True),     # no global tokens
    (1, 1, 128, 12, 12, 65, 6, 0, 0, True),    # a second piece of global keys
    tar.MASKED_CASES[3],                       # g = 0, exact window, w = 12: wholly masked leading pieces
]
PK_QK = (1, 2, 128, 21, 21, 1, 7, 0, 0, False)
PK_TABLE = (1, 2, 128, 21, 21, 2, 7, 0, 0, True)

ENTRY_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode
    (2, 2, 128, 28, 28, 1, 7, 0, 0),           # ViL-like, random inputs
    (1, 2, 128, 8, 5, 1, 4, -1, 0),            # cyclic 2 x 2
    (1, 2, 96, 24, 24, 1, 12, 0, 0),           # w = 12
]
LARGE_CASES = [
    (1, 1, 128, 50, 47, 1, 43, 0, 0),          # w = 43: past the wgmma HD 128 table limit
    (1, 1, 128, 60, 53, 1, 48, 0, 0),          # w = 48: 230 480 of 232 448 bytes in pass 1
]
S1_B13 = (13, 3, 128, 56, 56, 1, 7, 0, 0)      # nslice = 6: slice 0 runs images 0, 6, 12

DROP_CASES = [
    # B, H, D, nx, ny, g, w, exact, mode, rpe, separate global weights, p
    (1, 2, 128, 15, 13, 2, 7, 0, 0, True, True, 0.1),
    (1, 2, 128, 15, 13, 2, 7, 0, 0, True, True, 0.5),
    (1, 2, 96, 8, 5, 1, 4, -1, 0, True, False, 0.5),       # two offsets reach one chunk: two draws per pair
]
SEED, OFFSET = 0x5eed0000d128, 77


def simt_run(t, case, layout="contig", drop=(0.0, 0, 0)):
    """one forward + backward through the C ABI in fp32; both directions must have run the SIMT family"""
    nx, ny, w, exact, mode, scale = tar.cfg_of(case)
    if layout == "contig":
        return tar.run_kernels(t, tar.cfg_of(case), VARIANT, drop)
    out, fam_f, fam_b = tpar.kernel_run(t, nx, ny, w, exact, mode, scale, F32, "simt", layout=layout, drop=drop)
    assert (fam_f, fam_b) == ("simt", "simt")
    return out


# --------------------------------------------------------------------------- CPU
def test_batch_case_runs_several_images_per_pass1_cta():
    assert nslice_of_the_library(S1_B13) == 6 < S1_B13[0]


def test_masked_case_has_wholly_masked_leading_pieces():
    c = tar.MASKED_CASES[3]
    assert c[2] == 128
    _, lead = tar.masked_pieces(c[3], c[4], c[6], c[7], c[8])
    assert int((lead >= 0).sum()) > 0


def test_pass1_tile_fits_the_largest_table():
    """pass 1 with the table at w = 48: tiles + table + metadata, rounded to 16 bytes, + the dS tile.  Rows of HD + 8
    floats (the two-lane tile) would be 80 bytes over the 227 KB limit; the four-quarter row of HD + 4 floats fits"""
    up16 = lambda n: (n + 15) & ~15
    tabn = (4 * 48 - 1) ** 2
    pass1 = lambda hs: up16(4 * (2 * 64 * hs + tabn) + 64 * 2 * 2 + 64) + 64 * 65 * 4
    assert pass1(128 + 8) == 232528 > 227 * 1024
    assert pass1(128 + 4) == 230480 <= 227 * 1024


# --------------------------------------------------------------------------- GPU: rows and chunks
@gpu
@pytest.mark.parametrize("layout", ["contig", "linear"])
@pytest.mark.parametrize("case", ROW_CASES, ids=tar.CASE_ID)
def test_rows_against_the_dense_oracle(case, layout):
    t = tar.make_inputs(case, seed=350)
    ref = tar.oracle(t, tar.cfg_of(case), F32, ("simt128",) + case)
    out = simt_run(t, case, layout)
    assert _lib.last_impl() == "simt"
    tar.check("simt_headdim128_rows", "randn_" + layout, out, ref, case, VARIANT)


@gpu
@pytest.mark.parametrize("L", [40, 100])
def test_rows_peaked_through_q_and_k(L):
    t, hot = tar.peak_through_qk(tar.make_inputs(PK_QK, seed=351), PK_QK, F32, L, ("off", 1, 1, "same"))
    tar.check_peaked("simt_headdim128_peaked_qk", PK_QK, VARIANT, t, "off_1_1_L%d" % L, L, hot)


@gpu
@pytest.mark.parametrize("what", [("entry", 7, 7), ("band",), ("l2g", 1, 1)], ids=lambda x: "_".join(str(y) for y in x))
def test_rows_peaked_through_the_bias(what):
    L = 100
    t = tar.peak_through_table(tar.make_inputs(PK_TABLE, seed=352), PK_TABLE, L, what)
    tar.check_peaked("simt_headdim128_peaked_bias", PK_TABLE, VARIANT, t, "%s_L%d" % ("_".join(str(x) for x in what), L), L)


# --------------------------------------------------------------------------- GPU: bias gradients entry by entry
@gpu
@pytest.mark.parametrize("case", ENTRY_CASES + [S1_B13], ids=tbe.CASE_ID)
def test_bias_entries(case):
    t = tar.make_inputs(tbe.full(case), seed=360)
    out = tbe.run_variant(t, case, VARIANT)
    assert _lib.last_impl() == "simt"
    tbe.hold_entries("simt_headdim128_entries", "randn", out, tbe.bias_grad_terms(t, case, F32), case, VARIANT)


@gpu
@pytest.mark.parametrize("case", LARGE_CASES, ids=tbe.CASE_ID)
def test_bias_entries_large_windows(case):
    """the table at w = 43 and 48 beside the HD 128 tiles: rows at the SIMT bars, the bias gradients per entry"""
    fc = tbe.full(case)
    t = tar.make_inputs(fc, seed=361)
    out = tbe.run_variant(t, case, VARIANT)
    assert _lib.last_impl() == "simt"
    tar.check("simt_headdim128_large_windows", "randn", out, tar.oracle(t, tar.cfg_of(fc), F32, ("simt128_large",) + case),
              fc, VARIANT, bias=False)
    tbe.hold_entries("simt_headdim128_large_windows", "randn", out, tbe.bias_grad_terms(t, case, F32), case, VARIANT)


# --------------------------------------------------------------------------- GPU: dropout
DROP_ID = lambda c: tdrop.CASE_ID(c)


@gpu
@pytest.mark.parametrize("case", DROP_CASES, ids=DROP_ID)
def test_dropout_matches_the_exact_mask(case):
    B, H, D, nx, ny, g, w, exact, mode, rpe, sep, p = case
    _, _, _, tf, tb, tbias = tdrop.VARIANTS[VARIANT]
    t = tdrop.make_inputs(B, H, D, nx, ny, g, w, rpe, sep, seed=370)
    cfg = (nx, ny, w, exact, mode, D ** -0.5)
    keep, keep_g = tdrop.keep_tensors(SEED, OFFSET, p, B, H, nx, ny, w, g, mode)
    ref = tdrop.reference_run(t, cfg, F32, keep, keep_g)
    out, fam = tdrop.kernel_run(t, cfg, F32, "simt", (p, SEED, OFFSET))
    assert fam == "simt" and _lib.last_impl() == "simt"
    names = ["o", "dq", "dk", "dv"] + (["og", "dqg"] + (["dkg", "dvg"] if sep else []) if g else []) + \
        (["dtable"] + (["dg2l", "dg2g"] if g else []) if rpe else [])
    errs = {n: relerr(out[n], ref[n]) for n in names}
    record("simt_headdim128_dropout", DROP_ID(case), **errs)
    for n, e in errs.items():
        assert e < (tf if n in ("o", "og") else tbias if n in ("dtable", "dg2l", "dg2g") else tb), (n, errs)


@gpu
def test_p0_is_the_call_without_dropout():
    B, H, D, nx, ny, g, w, exact, mode, rpe, sep, _ = DROP_CASES[0]
    t = tdrop.make_inputs(B, H, D, nx, ny, g, w, rpe, sep, seed=371)
    cfg = (nx, ny, w, exact, mode, D ** -0.5)
    a, fam = tdrop.kernel_run(t, cfg, F32, "simt", (0.0, SEED, OFFSET))
    b, _ = tdrop.kernel_run(t, cfg, F32, "simt", (0.0, 0, 0))
    c, fam_f, fam_b = tpar.kernel_run(t, nx, ny, w, exact, mode, D ** -0.5, F32, "simt")
    assert fam == fam_f == fam_b == "simt"
    for n in a:
        if a[n] is not None:
            assert torch.equal(a[n], b[n]) and torch.equal(a[n], c[n]), n


# --------------------------------------------------------------------------- GPU: contracts of the backward
REPEAT_CASE = (2, 2, 128, 15, 13, 3, 7, 0, 0, True, True)


@gpu
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_backward_repeats_bitwise(p):
    B, H, D, nx, ny, g, w, exact, mode, rpe, sep = REPEAT_CASE
    t = tdrop.make_inputs(B, H, D, nx, ny, g, w, rpe, sep, seed=372)
    cfg = (nx, ny, w, exact, mode, D ** -0.5)
    a, fa = tdrop.kernel_run(t, cfg, F32, "simt", (p, SEED, OFFSET))
    b, fb = tdrop.kernel_run(t, cfg, F32, "simt", (p, SEED, OFFSET))
    assert fa == fb == "simt" and a["dtable"] is not None
    for n in a:
        if a[n] is not None:
            assert torch.equal(a[n], b[n]), n


def _image(t, b):
    """the inputs of image b alone (the global-weight tensors stay the local ones when they were)"""
    one = dict(t)
    for n in ("q", "k", "v", "qg", "go", "gog"):
        one[n] = t[n][b:b + 1]
    one["kg"], one["vg"] = (one["k"], one["v"]) if t["kg"] is t["k"] else (t["kg"][b:b + 1], t["vg"][b:b + 1])
    return one


@gpu
def test_every_image_of_a_batch_is_a_one_image_call():
    """B = 13 > nslice = 6: pass-1 CTAs of slice s run images s, s + 6, s + 12.  Every per-image output of the batched
    call is bitwise the one-image call's (the bias gradients sum over the images and are held in test_bias_entries)"""
    case = tbe.full(S1_B13)
    t = tar.make_inputs(case, seed=373)
    full = simt_run(t, case)
    for b in range(S1_B13[0]):
        one = simt_run(_image(t, b), (1,) + case[1:])
        for n in ("o", "lse", "dq", "dk", "dv", "og", "lse_g", "dqg"):
            assert torch.equal(full[n][b:b + 1], one[n]), (b, n)


@gpu
def test_bias_gradients_are_accumulated_into(monkeypatch):
    """d_bias_table, d_g2l and d_g2g pre-filled with X come back as X + the clean result, bit for bit"""
    B, H, D, nx, ny, g, w, exact, mode, sep, p = (2, 2, 128, 15, 13, 2, 7, 1, 0, True, 0.1)
    t = tar.make_inputs((B, H, D, nx, ny, g, w, exact, mode, True), seed=374, sep=sep)
    run = lambda: tpar.kernel_run(t, nx, ny, w, exact, mode, D ** -0.5, F32, "simt", drop=(p, SEED, OFFSET))
    clean, fam_f, fam_b = run()
    assert (fam_f, fam_b) == ("simt", "simt")
    gen = torch.Generator().manual_seed(375)
    X = {n: torch.randn(clean[n].shape, generator=gen).to(clean[n].device) * float(clean[n].abs().max())
         for n in tbe.NAMES}
    orig = tpar.vil_attention_raw_backward

    def prefilled(*a, **kw):
        a = list(a)
        for i, n in zip((21, 22, 23), tbe.NAMES):
            a[i].copy_(X[n])
        return orig(*a, **kw)

    monkeypatch.setattr(tpar, "vil_attention_raw_backward", prefilled)
    acc, _, _ = run()
    for n in tbe.NAMES:
        assert torch.equal(acc[n], X[n] + clean[n]), (n, float((acc[n] - X[n] - clean[n]).abs().max()))


@gpu
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_dirty_workspace_changes_no_output_bit(p, monkeypatch):
    from vision_longformer_b200 import ops
    B, H, D, nx, ny, g, w, exact, mode, sep = (13, 3, 128, 14, 14, 1, 7, 0, 0, False)
    t = tar.make_inputs((B, H, D, nx, ny, g, w, exact, mode, True), seed=376, sep=sep)
    orig = ops._workspace
    outs = []
    for byte in (0x00, 0xFF):
        def filled(*a, _b=byte, **kw):
            ws = orig(*a, **kw)
            ws.fill_(_b)
            return ws
        monkeypatch.setattr(ops, "_workspace", filled)
        out, fam_f, fam_b = tpar.kernel_run(t, nx, ny, w, exact, mode, D ** -0.5, F32, "simt", drop=(p, SEED, OFFSET))
        assert (fam_f, fam_b) == ("simt", "simt")
        outs.append(out)
    assert outs[0]["dtable"] is not None
    for n, x in outs[0].items():
        if x is not None:
            assert torch.equal(x, outs[1][n]), n


# --------------------------------------------------------------------------- GPU: modules
def _module_pair(**kw):
    from oracle.vil_oracle import OracleLong2DSCSelfAttention
    from vision_longformer_b200 import B200Long2DSCSelfAttention
    torch.manual_seed(15)
    ref = OracleLong2DSCSelfAttention(dim=256, num_heads=2, rpe=True).double().eval()
    for n, p_ in ref.named_parameters():                    # biases large enough to matter
        if "relative_position" in n:
            torch.nn.init.normal_(p_, std=0.3)
    mod = B200Long2DSCSelfAttention(dim=256, num_heads=2, rpe=True, **kw).to(DEV)
    mod.load_state_dict({k_: v_.float() for k_, v_ in ref.state_dict().items()})
    return ref, mod


@gpu
def test_module_in_fp32_matches_the_reference():
    ref, mod = _module_pair()
    mod.eval()
    nx = ny = 28
    x = torch.randn(2, 1 + nx * ny, 256, dtype=torch.float64, requires_grad=True)
    gy = torch.randn(2, 1 + nx * ny, 256, dtype=torch.float64)
    y_ref = ref(x, nx, ny)
    (y_ref * gy).sum().backward()
    xg = x.detach().float().to(DEV).requires_grad_(True)
    y = mod(xg, nx, ny)
    assert y.dtype == F32 and _lib.last_impl() == "simt"
    (y * gy.float().to(DEV)).sum().backward()
    torch.cuda.synchronize()
    assert _lib.last_impl() == "simt"
    errs = dict(y=relerr(y, y_ref), dx=relerr(xg.grad, x.grad))
    grads = dict(ref.named_parameters())
    for n, p_ in mod.named_parameters():
        errs["d" + n] = relerr(p_.grad, grads[n].grad)
    record("simt_headdim128_module", "dim256_h2_rpe_28x28", **errs)
    assert errs["y"] < 2e-5 and errs["dx"] < 4e-5, errs
    assert all(e < 1e-4 for e in errs.values()), errs


@gpu
def test_module_trains_in_fp32_with_attention_dropout():
    _, mod = _module_pair(attn_drop=0.1)
    mod.train()
    nx = ny = 28
    x = torch.randn(2, 1 + nx * ny, 256, device=DEV, requires_grad=True)
    y = mod(x, nx, ny)
    assert _lib.last_impl() == "simt"
    loss = (y * torch.randn_like(y)).sum()
    loss.backward()
    torch.cuda.synchronize()
    assert _lib.last_impl() == "simt" and math.isfinite(loss.item())
    assert torch.isfinite(x.grad).all()
    for n, p_ in mod.named_parameters():
        assert p_.grad is not None and torch.isfinite(p_.grad).all(), n
