"""Dilated (VIL_FLAG_DILATED) and sized (per-image token grids) attention across every kernel instantiation they launch.

A dilated or sized call runs the `DIL` instantiations of the local forward, pass 1 and pass 2 in both families, and a
sized call with global tokens the `SIZED` instantiations of simt_fwd_global / simt_bwd_grow / simt_bwd_gcol.  Those are
templated over the operand and output types, the head tile (wgmma: head_tile) or bucket (SIMT: head_bucket), the lanes
per row (SIMT: L), dropout and the bias table (pass 1: TAB).  tests/test_gpu_dilation.py and
tests/test_gpu_image_sizes.py hold them at head dim 16; this file carries the same checks to every instantiation:

- the bitwise identities: local o / lse / dq and the unshared local-key dk / dv of a call are those of ordinary calls
  (non-`DIL` kernels, same head dim) on each image's residue sub-grids; the global rows of a dilated call are those of
  the d = 1 call; a sized call with every image full is the unsized call; sums reordered across residues or images
  agree within fp32 reordering;
- the fp64 oracles (tests/dilated_oracle.py, tests/sized_oracle.py) on inputs that are exact in the operand type, at
  the bars the unsized operator has for the variant in its own files;
- NaN / inf at off-image inputs and NaN in every output and workspace change no real output;
- dropout against the exact-mask restatement; repeatability with a dirty workspace.

The case list covers the instantiations rather than their product.  The CPU guards below enumerate, from a mirror of
the dispatch rules pinned to the head-dim switches of vil_wgmma.cu and vil_simt.cu, every instantiation a dilated or
sized call can reach, and fail naming any that no case reaches.
"""
import ctypes
import math
import os
import re
from typing import NamedTuple, Optional

import pytest
import torch

from tests import test_gpu_dropout as tdrop
from tests.dilated_oracle import dilated_attention, residues
from tests.sized_oracle import image_index, sized_attention
from tests.test_gpu_dilation import EXACT_MODES, REORDER, _keep_sub, same
from tests.test_gpu_image_sizes import off_image, poison
from tests.util import record, relerr
from vision_longformer_b200 import _lib, ops

DEV = "cuda"
gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "vision_longformer_b200", "csrc")
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
SPLIT, F32OUT = _lib.VIL_FLAG_F32_SPLIT, _lib.VIL_FLAG_F32_OUT
TNAME = {F32: "f32", BF16: "bf16", F16: "f16"}

# name: (operand dtype, family, flags, output dtype, bars (o, gradients, bias gradients) against the fp64 oracle).  The
# bars are those of the unsized operator: test_gpu_parity.TOL and its bias bars (fp32 / bf16 / fp16, either family),
# test_gpu_f32_split (split fp32), test_headdim128.test_headdim128_fp32_out_parity (fp32 outputs).
VARIANTS = {
    "simt_f32": (F32, "simt", 0, F32, (1e-5, 2e-5, 1e-4)),
    "simt_bf16": (BF16, "simt", 0, BF16, (4e-3, 8e-3, 5e-2)),
    "simt_f16": (F16, "simt", 0, F16, (1e-3, 2e-3, 1e-2)),
    "wgmma_f32split": (F32, "wgmma", SPLIT, F32, (7e-5, 1e-4, 2.5e-5)),
    "wgmma_bf16": (BF16, "wgmma", 0, BF16, (4e-3, 8e-3, 5e-2)),
    "wgmma_f16": (F16, "wgmma", 0, F16, (1e-3, 2e-3, 1e-2)),
    "wgmma_bf16_f32out": (BF16, "wgmma", F32OUT, F32, (2e-3, 2e-3, 2e-2)),
    "wgmma_f16_f32out": (F16, "wgmma", F32OUT, F32, (1e-3, 1e-3, 2e-2)),
}
LSE_BAR = 1e-4
P_DROP, SEED, OFFSET = 0.3, 0x5eed00051ced, 23


class Case(NamedTuple):
    variant: str
    D: int
    nx: int
    ny: int
    w: int
    d: int
    g: int
    rpe: bool
    sep: bool                       # separate global weights (qg / kvg of their own)
    exact: int
    mode: int
    sizes: Optional[tuple]          # B (h, w) per-image grids, or None (an unsized call)
    p: float = 0.0                  # attention dropout
    B: int = 2                      # images of an unsized call
    H: int = 2


def nimg(c):
    return len(c.sizes) if c.sizes else c.B


def cid(c):
    sz = "-".join("%dx%d" % s for s in c.sizes) if c.sizes else "nosizes"
    return "%s_D%d_%dx%d_w%d_d%d_g%d%s_%s_e%d_m%d_%s%s%s" % (
        c.variant, c.D, c.nx, c.ny, c.w, c.d, c.g, "sep" if c.sep else "", "rpe" if c.rpe else "norpe", c.exact, c.mode,
        sz, "_p%g" % c.p if c.p else "", "_H%d" % c.H if c.H != 2 else "")


# --------------------------------------------------------------------------- the mirror of the dispatch rules
def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _function(src, name):
    """the text of the first definition of function `name` (up to its closing brace at column 0)"""
    m = re.search(r"\n[^\n]*\b%s\([^;{]*\)\s*\{" % re.escape(name), src)
    assert m, name
    end = src.index("\n}\n", m.end())
    return src[m.start():end]


def _ladder(src, name):
    """`int name(int D) { return D <= a ? a : D <= b ? b : ... : z; }` -> [a, b, ..., z]"""
    m = re.search(r"int %s\(int D\) \{ return ((?:D <= \d+ \? \d+ : )+)(\d+); \}" % name, src)
    assert m, name
    steps = re.findall(r"D <= (\d+) \? (\d+)", m.group(1))
    assert all(a == b for a, b in steps), steps
    return [int(a) for a, _ in steps] + [int(m.group(2))]


def _switch(src, fn, on):
    """case labels of `switch (on)` in function fn, the default standing for the largest value of the ladder"""
    body = _function(src, fn)
    i = body.index("switch (%s)" % on)
    block = body[i:body.index("\n  }", i)]
    return [int(x) for x in re.findall(r"case (\d+):", block)], "default:" in block


def _one(pattern, text):
    found = re.findall(pattern, text)
    assert len(found) == 1, (pattern, found)
    return int(found[0])


class Rules:
    """What vil_wgmma.cu / vil_simt.cu dispatch a call to, with every number read from the source"""

    def __init__(self):
        wg, sm = _src("vil_wgmma.cu"), _src("vil_simt.cu")
        self.wg_tiles = _ladder(wg, "head_tile")
        self.simt_buckets = _ladder(sm, "head_bucket")
        why = _function(wg, "why_not")
        self.split_max = _one(r"split && g\.D > (\d+)", why)
        self.wg_align = _one(r"g\.D % (\d+) != 0", why)
        fwd, bwd = _function(sm, "simt_forward"), _function(sm, "simt_backward")
        self.simt_drop_fwd_max = _one(r"if constexpr \(DROP && HD > (\d+) && !std::is_same<T, float>::value\)", fwd)
        self.simt_fwd_l4 = _one(r"constexpr int L = DROP && std::is_same<T, float>::value && HD > (\d+) \? 4 : 2;", fwd)
        self.simt_bwd_max = _one(r"if constexpr \(HD > (\d+) && !std::is_same<T, float>::value\)", bwd)
        self.simt_bwd_l4 = _one(r"constexpr int L = std::is_same<T, float>::value && HD > (\d+) \? 4 : 2;", bwd)
        self.switches = dict(
            wg_dispatch=(_switch(wg, "dispatch_hd_drop", "head_tile(g.D)"), self.wg_tiles),
            wg_smem=(_switch(wg, "smem_why_not_hd", "head_tile(g.D)"), self.wg_tiles),
            simt_local=(_switch(sm, "simt_dispatch_hd", "head_bucket(g.D)"), self.simt_buckets),
        )
        m = re.search(r"#define VIL_SIMT_HD\(T, TO, CALL\)(.*?)\n\n", sm, re.S)
        self.switches["simt_global"] = (([int(x) for x in re.findall(r"case (\d+):", m.group(1))],
                                         "default:" in m.group(1)), self.simt_buckets)

    @staticmethod
    def pick(ladder, D):
        return next(x for x in ladder if D <= x)

    def tile(self, D):
        return self.pick(self.wg_tiles, D)

    def bucket(self, D):
        return self.pick(self.simt_buckets, D)

    def trains(self, family, T, D):
        """False where the backward is refused: the SIMT family's bf16 / fp16 backward above its limit"""
        return not (family == "simt" and T != "f32" and self.bucket(D) > self.simt_bwd_max)

    def launches(self, family, T, TO, D, drop, rpe, sub, glob, train):
        """(family, kernel, T, TO, tile, L, DROP, TAB) of the DIL / SIZED kernels of one call.  sub: a dilated or sized
        call (the DIL local kernels); glob: a sized call with global tokens (the SIZED global kernels)"""
        out = set()
        if sub and family == "wgmma":
            hd = self.tile(D)
            out.add(("wgmma", "fwd", T, TO, hd, None, drop, None))
            if train:
                out |= {("wgmma", "dq", T, TO, hd, None, drop, rpe), ("wgmma", "dkv", T, TO, hd, None, drop, None)}
        elif sub:
            hd = self.bucket(D)
            lf = 4 if (drop and T == "f32" and hd > self.simt_fwd_l4) else 2
            lb = 4 if (T == "f32" and hd > self.simt_bwd_l4) else 2
            out.add(("simt", "fwd", T, TO, hd, lf, drop, None))
            if train:
                out |= {("simt", "dq", T, TO, hd, lb, drop, rpe), ("simt", "dkv", T, TO, hd, lb, drop, None)}
        if glob:                                      # both families launch the global kernels at head_bucket
            hd = self.bucket(D)
            out.add(("global", "fwd", T, TO, hd, None, drop, None))
            if train:
                out |= {("global", "gcol", T, TO, hd, None, drop, None), ("global", "grow", T, TO, hd, None, drop, None)}
        return out

    def refused(self, family, T, D, drop):
        return family == "simt" and T != "f32" and drop and self.bucket(D) > self.simt_drop_fwd_max

    def reachable(self):
        """every DIL / SIZED instantiation some dilated or sized call launches"""
        calls = []                                    # (family, T, TO, D)
        for T in ("f32", "bf16", "f16"):
            calls += [("simt", T, T, D) for D in range(1, self.simt_buckets[-1] + 1)]
        for T, TO in (("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f16", "f32"), ("f32", "f32")):
            top = self.split_max if T == "f32" else self.wg_tiles[-1]
            calls += [("wgmma", T, TO, D) for D in range(self.wg_align, top + 1, self.wg_align)]
        out = set()
        for fam, T, TO, D in calls:
            for drop in (False, True):
                if self.refused(fam, T, D, drop):
                    continue
                for rpe in (False, True):
                    out |= self.launches(fam, T, TO, D, drop, rpe, True, True, self.trains(fam, T, D))
        return out

    def of_case(self, c):
        dtype, fam, flags, odt, _ = VARIANTS[c.variant]
        T, TO = TNAME[dtype], TNAME[odt]
        return self.launches(fam, T, TO, c.D, c.p > 0, c.rpe, c.d > 1 or c.sizes is not None,
                             c.sizes is not None and c.g > 0, self.trains(fam, T, c.D))


RULES = Rules()


def trains(c):
    dtype, fam = VARIANTS[c.variant][:2]
    return RULES.trains(fam, TNAME[dtype], c.D)


# --------------------------------------------------------------------------- the cases
def _group(variant, Da, Db, gi, train=True):
    """The cases of one (family, T, TO, head tile): dilation only, sizes only and both; g = 0, shared and separate global
    weights; with and without the bias table; with and without dropout.  Da / Db: two head dims of the tile (a partial
    one first), which with global tokens also reach two SIMT buckets where the tile spans them (wgmma 16: 8 and 16)."""
    em = lambda k: EXACT_MODES[(5 * gi + k) % len(EXACT_MODES)]
    out = [
        Case(variant, Da, 13, 11, 3, 2, 0, True, False, *em(0), None),
        Case(variant, Da, 11, 13, 4, 1, 1, False, False, *em(1), ((11, 9), (6, 13), (1, 13))),
        Case(variant, Db, 12, 12, 3, 3, 2, True, True, *em(2), ((12, 10), (7, 12))),
    ]
    if train:
        out += [Case(variant, Da, 10, 11, 4, 2, 1, True, False, *em(3), ((10, 11), (9, 5)), p=P_DROP),
                Case(variant, Db, 13, 10, 3, 1, 1, False, True, *em(4), ((9, 7), (13, 2)), p=P_DROP)]
    return out


_DIMS = {  # head tile / bucket -> (a partial head dim, the full one)
    "wgmma": {16: (8, 16), 32: (24, 32), 64: (40, 64), 128: (96, 128)},
    "simt": {8: (4, 8), 16: (12, 16), 32: (24, 32), 64: (40, 64), 128: (96, 128)},
}


def _matrix():
    cases = []
    for variant, (dtype, fam, flags, odt, _) in VARIANTS.items():
        for hd, (Da, Db) in _DIMS[fam].items():
            if flags & SPLIT and hd > RULES.split_max:
                continue
            if variant == "wgmma_f16" and hd == 128:
                Da = 120
            cases += _group(variant, Da, Db, len(cases) // 5, train=RULES.trains(fam, TNAME[dtype], Db))
    return cases


MATRIX = _matrix()
# w^2 > 64: chunks of npc = 2, 3, 4 pieces.  Sizes that are not multiples of w, crops narrower than w, and sub-grids that
# are one partial chunk (e.g. 13 x 5 at d = 2: residues of 7 x 3 and 6 x 2).
MULTI = [
    Case("wgmma_bf16", 32, 25, 22, 9, 2, 1, True, False, 0, 0, ((25, 22), (19, 13), (13, 5))),
    Case("wgmma_f16", 64, 31, 28, 12, 3, 2, True, True, -1, 0, ((31, 28), (17, 25), (10, 7))),
    Case("wgmma_bf16_f32out", 128, 33, 20, 15, 1, 1, False, False, 1, 0, ((33, 20), (14, 19), (11, 13))),
    Case("wgmma_f32split", 64, 24, 26, 12, 2, 0, True, False, 0, 0, None),
    Case("wgmma_f16_f32out", 32, 34, 31, 15, 2, 1, True, True, 0, 3, ((34, 31), (29, 9))),
    Case("simt_f32", 128, 25, 22, 9, 2, 1, True, False, 0, 0, ((25, 22), (19, 13), (13, 5))),
    Case("simt_f32", 32, 33, 20, 15, 3, 2, True, True, -1, 0, ((33, 20), (14, 19))),
    Case("simt_bf16", 64, 31, 28, 12, 1, 1, False, False, 1, 0, ((31, 28), (17, 25), (10, 7))),
    Case("simt_f16", 16, 20, 19, 9, 2, 1, True, True, 0, 3, None),
    Case("simt_f32", 96, 26, 25, 12, 2, 1, True, False, 0, 0, ((26, 25), (15, 11)), p=P_DROP),
    Case("wgmma_bf16", 64, 22, 20, 9, 2, 1, True, True, -1, 0, ((22, 20), (13, 5)), p=P_DROP),
    Case("wgmma_bf16_f32out", 128, 25, 26, 12, 3, 0, True, False, 0, 0, None, p=P_DROP),
]
# ViL-Small stage 1 (56 x 56, w = 7, 3 heads of 32, one global token, the table) as a detection backbone runs it: 8 padded
# images of mixed sizes, dilation 2; more images than pass-1 slices.  Its stage-2-like sibling: 28 x 28, 6 heads of 64.
PRODUCTION = [
    Case("wgmma_bf16", 32, 56, 56, 7, 2, 1, True, False, 0, 0,
         ((56, 56), (48, 40), (31, 56), (56, 17), (20, 25), (56, 56), (9, 3), (44, 51)), H=3),
    Case("wgmma_f16", 64, 28, 28, 7, 2, 1, True, False, 0, 0,
         ((28, 28), (21, 14), (28, 9), (5, 28), (17, 23), (28, 28), (11, 2), (26, 27)), H=6),
]
ALL = MATRIX + MULTI + PRODUCTION
PLAIN = [c for c in ALL if not c.p]
SIZED = [c for c in ALL if c.sizes]
DROPPED = [c for c in ALL if c.p]
# the oracle of the 56 x 56 case is a dense fp64 softmax over 3136 keys per image; its identities hold it instead
ORACLE = [c for c in PLAIN if c is not PRODUCTION[0]]
ids = lambda cases: [cid(c) for c in cases]


# --------------------------------------------------------------------------- inputs and the raw runner
def make(c, seed=0):
    """fp32 leaf tensors in the Linear-output layouts (tests/test_gpu_dilation.make), exact in the operand type, so that
    the fp64 oracle on them is the oracle on what the kernels read"""
    dtype = VARIANTS[c.variant][0]
    gen = torch.Generator().manual_seed(seed + 7 * c.nx + c.ny + 131 * c.g + 17 * c.D + 3 * c.d)
    r = lambda *s: torch.randn(*s, generator=gen).to(dtype).float()
    B, N, C = nimg(c), c.g + c.nx * c.ny, c.H * c.D
    t = dict(q_all=r(B, N if (c.g and not c.sep) else c.nx * c.ny, C), kv=r(B, N, 2 * C), dout=r(B, N, C))
    if c.g and c.sep:
        t.update(qg_all=r(B, c.g, C), kvg=r(B, N, 2 * C))
    if c.rpe:
        t["table"] = 0.5 * torch.randn((4 * c.w - 1) ** 2, c.H, generator=gen)
        if c.g:
            t["g2l"], t["g2g"] = 0.5 * torch.randn(2, c.H, c.g, generator=gen), 0.5 * torch.randn(c.H, c.g, c.g, generator=gen)
    t["H"], t["D"] = c.H, c.D
    return t


def views(t, c, dev=DEV, dtype=None):
    """(B, H, T, D) views of the call: q, k, v, qg, kg, vg and the two views of d_out"""
    dtype = dtype or VARIANTS[c.variant][0]
    H, g = c.H, c.g
    cv = lambda x: x.to(dev, dtype)
    kv = cv(t["kv"])
    k, v = ops._heads(kv, H, 0, 2), ops._heads(kv, H, 1, 2)
    qa = ops._heads(cv(t["q_all"]), H)
    if g and not c.sep:
        q, qg, kg, vg = qa[:, :, g:], qa[:, :, :g], k, v
    elif g:
        kvg = cv(t["kvg"])
        q, qg, kg, vg = qa, ops._heads(cv(t["qg_all"]), H), ops._heads(kvg, H, 0, 2), ops._heads(kvg, H, 1, 2)
    else:
        q, qg, kg, vg = qa, None, None, None
    dout = ops._heads(cv(t["dout"]), H)
    return q, k, v, qg, kg, vg, dout[:, :, g:], (dout[:, :, :g] if g else None)


def geo(c, d=None):
    return c.nx, c.ny, c.w, c.d if d is None else d, c.g, c.rpe, c.exact, c.mode


def drop_of(c):
    return (c.p, SEED, OFFSET) if c.p else (0.0, 0, 0)


def run(q, k, v, qg, kg, vg, d_o, d_og, t, geo_, variant, sizes=None, hw=None, fill=None, drop=(0.0, 0, 0), bwd=True):
    """forward (+ backward) through the raw ABI, outputs in the variant's output type and the production head-merged
    layout (tests/test_gpu_image_sizes.run with fp32 outputs).  `hw`: a device (B, 2) int32 tensor for the sized entry
    points; `fill`: prefill every output and the workspaces with this value"""
    nx, ny, w, d, g, rpe, exact, mode = geo_
    dtype, impl, flags, odt, _ = VARIANTS[variant]
    B, H, Nloc, D = q.shape
    N = k.shape[2]
    shared = g > 0 and kg.data_ptr() == k.data_ptr()
    new = (lambda *s: torch.full(s, fill, dtype=odt, device=DEV)) if fill is not None else \
        (lambda *s: torch.empty(*s, dtype=odt, device=DEV))
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
    assert _lib.last_impl() == impl
    res = dict(o=o, og=og, lse=lse, lse_g=lse_g)
    if not bwd:
        return res
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
    assert _lib.last_impl() == impl
    res.update(dq=dq, dk=dk, dv=dv, dqg=dqg, dkg=dkg if not shared else None, dvg=dvg if not shared else None,
               d_tab=d_tab, d_g2l=d_g2l, d_g2g=d_g2g)
    return res


def images(c):
    """(batch slice, h, w): the whole batch of an unsized call, each image of a sized one"""
    if c.sizes is None:
        return [(slice(0, c.B), c.nx, c.ny)]
    return [(slice(b, b + 1), h, wb) for b, (h, wb) in enumerate(c.sizes)]


def part_inputs(vw, g, bs, idx):
    """images bs restricted to the local tokens idx, after the same global tokens.  Shared global weights get equal-valued
    keys of their own, so that the local-key gradients hold the local queries' terms only"""
    q, k, v, qg, kg, vg, d_o, d_og = vw
    cat = lambda x: torch.cat([x[bs, :, :g], x[bs, :, g + idx]], dim=2)
    ks, vs = cat(k), cat(v)
    if g:
        shared = kg.data_ptr() == k.data_ptr()
        kgs, vgs = (ks.clone(), vs.clone()) if shared else (cat(kg), cat(vg))
    else:
        kgs = vgs = None
    sl = lambda x: x[bs].contiguous() if x is not None else None
    return q[bs, :, idx].contiguous(), ks, vs, sl(qg), kgs, vgs, d_o[bs, :, idx].contiguous(), sl(d_og)


# --------------------------------------------------------------------------- GPU: bitwise identities
@gpu
@pytest.mark.parametrize("case", PLAIN, ids=ids(PLAIN))
def test_call_is_the_sub_grid_calls(case):
    """local rows bitwise those of the ordinary calls on each image's residue sub-grids; global rows of a dilated call
    bitwise the d = 1 call's; a sized call with every image full bitwise the unsized call"""
    c = case
    bwd = trains(c)
    odt = VARIANTS[c.variant][3]
    t = make(c)
    vw = views(t, c)
    res = run(*vw, t, geo(c), c.variant, sizes=c.sizes, bwd=bwd)
    if c.d > 1 and c.g:
        und = run(*vw, t, geo(c, 1), c.variant, sizes=c.sizes, bwd=bwd)
        for key in ("og", "lse_g", "dqg", "dkg", "dvg", "d_g2g"):
            if res.get(key) is not None:
                same(res[key], und[key], key)
        if c.rpe and bwd:
            same(res["d_g2l"][0], und["d_g2l"][0], "d_g2l[0]")
    sums = {}

    def add(key, x, bs=None):
        if bs is None:
            sums[key] = sums.get(key, 0) + x.double()
        else:
            sums.setdefault(key, torch.zeros_like(res[key][:, :, :c.g], dtype=torch.float64))[bs] += x.double()

    for bs, h, wb in images(c):
        crop = c.sizes is not None and c.d == 1              # the sub-grid is the image's crop, global rows included
        for a, b, na, nb, ridx in residues(h, wb, c.d):
            idx = ((ridx // wb) * c.ny + ridx % wb).to(DEV)
            sub = run(*part_inputs(vw, c.g, bs, idx), t, (na, nb) + geo(c, 1)[2:], c.variant, bwd=bwd)
            for key in ("o", "lse") + (("dq",) if bwd else ()):
                same(res[key][bs, :, idx], sub[key], key)
            if crop and c.g:
                assert relerr(res["og"][bs], sub["og"]) < REORDER[odt]
                assert relerr(res["lse_g"][bs], sub["lse_g"]) < REORDER[F32]
                if bwd:
                    assert relerr(res["dqg"][bs], sub["dqg"]) < REORDER[odt]
            if not bwd:
                continue
            if c.sep or c.g == 0:
                same(res["dk"][bs, :, c.g + idx], sub["dk"][:, :, c.g:], "dk")
                same(res["dv"][bs, :, c.g + idx], sub["dv"][:, :, c.g:], "dv")
                if c.g:
                    add("dk", sub["dk"][:, :, :c.g], bs)
                    add("dv", sub["dv"][:, :, :c.g], bs)
            if c.rpe:
                add("d_tab", sub["d_tab"])
                if c.g:
                    add("d_g2l1", sub["d_g2l"][1])
                    if crop:
                        add("d_g2l0", sub["d_g2l"][0])
                        add("d_g2g", sub["d_g2g"])
    got = lambda key: res[key][:, :, :c.g] if key in ("dk", "dv") else \
        res["d_g2l"][int(key[-1])] if key.startswith("d_g2l") else res[key]
    for key, x in sums.items():
        bar = REORDER[odt] if key in ("dk", "dv") else REORDER[F32]
        assert relerr(got(key).double(), x) < bar, (key, relerr(got(key).double(), x))
    if c.sizes:
        full = torch.tensor([[c.nx, c.ny]] * nimg(c), dtype=torch.int32, device=DEV)
        a = run(*vw, t, geo(c), c.variant, hw=full, bwd=bwd)
        b = run(*vw, t, geo(c), c.variant, bwd=bwd)
        for key, x in a.items():
            if x is not None:
                same(x, b[key], key)


# --------------------------------------------------------------------------- GPU: the fp64 oracle
def oracle(t, c):
    """fp64 dilated / sized oracle: outputs, lse and the gradients of dout . out, per leaf and per view"""
    g, H = c.g, c.H
    leaf = {k: t[k].double().requires_grad_(True) for k in ("q_all", "kv", "qg_all", "kvg", "table", "g2l", "g2g") if k in t}
    q, k, v, qg, kg, vg, _, _ = views(dict(leaf, dout=t["dout"]), c, dev="cpu", dtype=torch.float64)
    kw = dict(nx=c.nx, ny=c.ny, w=c.w, exact=c.exact, mode=c.mode, scale=c.D ** -0.5, d=c.d)
    args = (q, k, v, qg, kg, vg, leaf.get("table"), leaf.get("g2l"), leaf.get("g2g"))
    o, og, lse, lse_g = sized_attention(*args, sizes=c.sizes, **kw) if c.sizes else dilated_attention(*args, **kw)
    dout = ops._heads(t["dout"].double(), H)
    loss = (o * dout[:, :, g:]).sum() + ((og * dout[:, :, :g]).sum() if g else 0)
    loss.backward()
    grads = {key: x.grad for key, x in leaf.items()}
    qa = ops._heads(grads["q_all"], H)
    per_view = dict(o=o.detach(), lse=lse.detach(), dk=ops._heads(grads["kv"], H, 0, 2), dv=ops._heads(grads["kv"], H, 1, 2),
                    d_tab=grads.get("table"), d_g2l=grads.get("g2l"), d_g2g=grads.get("g2g"))
    if g and not c.sep:
        per_view.update(og=og.detach(), lse_g=lse_g.detach(), dq=qa[:, :, g:], dqg=qa[:, :, :g])
    elif g:
        per_view.update(og=og.detach(), lse_g=lse_g.detach(), dq=qa, dqg=ops._heads(grads["qg_all"], H),
                        dkg=ops._heads(grads["kvg"], H, 0, 2), dvg=ops._heads(grads["kvg"], H, 1, 2))
    else:
        per_view["dq"] = qa
    return grads, per_view


def _bar(key, bars):
    tf, tb, tbias = bars
    return tf if key in ("o", "og", "out") else LSE_BAR if key in ("lse", "lse_g") else \
        tbias if key in ("d_tab", "d_g2l", "d_g2g", "table", "g2l", "g2g") else tb


@gpu
@pytest.mark.parametrize("case", ORACLE, ids=ids(ORACLE))
def test_matches_the_fp64_oracle(case):
    """Through ops.vil_attention(dilation=, image_sizes=): the output and every leaf gradient.  The fp32-output variants
    (which ops.vil_attention does not build) and the forward-only SIMT variants through the raw runner: every output"""
    c = case
    dtype, impl, flags, odt, bars = VARIANTS[c.variant]
    t = make(c, seed=5)
    grads, ref = oracle(t, c)
    errs = {}
    if flags & F32OUT or not trains(c):
        res = run(*views(t, c), t, geo(c), c.variant, sizes=c.sizes, bwd=trains(c))
        for key, x in res.items():
            if x is None:
                continue
            r = ref[key]
            if key == "lse":                               # -inf at the off-image rows of a sized call
                real = torch.isfinite(r)
                assert bool((x.cpu()[~real] == -math.inf).all())
                x, r = x.cpu()[real], r[real]
            errs[key] = relerr(x, r)
    else:
        leaf = {k: (t[k].to(DEV, dtype) if k in ("q_all", "kv", "qg_all", "kvg") else t[k].to(DEV)).requires_grad_(True)
                for k in ("q_all", "kv", "qg_all", "kvg", "table", "g2l", "g2g") if k in t}
        prec = torch.backends.cuda.matmul.fp32_precision
        torch.backends.cuda.matmul.fp32_precision = "tf32" if flags & SPLIT else "ieee"
        try:
            out = ops.vil_attention(leaf["q_all"], leaf["kv"], leaf.get("qg_all"), leaf.get("kvg"), leaf.get("table"),
                                    leaf.get("g2l"), leaf.get("g2g"), num_heads=c.H, nx=c.nx, ny=c.ny, w=c.w, nglo=c.g,
                                    exact=c.exact, mode=c.mode, scale=c.D ** -0.5, impl=impl, dilation=c.d,
                                    image_sizes=torch.tensor(c.sizes) if c.sizes else None)
            assert _lib.last_impl() == impl
            out.backward(t["dout"].to(DEV, dtype))
        finally:
            torch.backends.cuda.matmul.fp32_precision = prec
        assert _lib.last_impl() == impl
        o = ops._heads(out.detach().double().cpu(), c.H)
        errs["o"] = relerr(o[:, :, c.g:], ref["o"])
        if c.g:
            errs["og"] = relerr(o[:, :, :c.g], ref["og"])
        for key, x in grads.items():
            errs[key] = relerr(leaf[key].grad, x)
    record("subgrid_matrix_oracle", cid(c), **errs)
    bad = {key: e for key, e in errs.items() if not e < _bar(key, bars)}
    assert not bad, (bad, errs)


# --------------------------------------------------------------------------- GPU: padding, dropout, repeatability
@gpu
@pytest.mark.parametrize("case", SIZED, ids=ids(SIZED))
def test_padding_never_leaks(case):
    """NaN / +-inf at every off-image input token, NaN in every output and workspace beforehand: the real tokens' outputs
    are unchanged bit for bit, and the off-image rows are exact zeros (lse -inf), in 2- and 4-byte outputs alike"""
    c = case
    legacy = (c.nx, c.ny, c.w, c.d, c.g, c.rpe, c.sep, c.exact, c.mode, c.sizes)
    t = make(c, seed=2)
    kw = dict(sizes=c.sizes, drop=drop_of(c), bwd=trains(c))
    clean = run(*views(t, c), t, geo(c), c.variant, **kw)
    dirty = run(*views(poison(t, legacy), c), t, geo(c), c.variant, fill=float("nan"), **kw)
    off = off_image(legacy).to(DEV)
    for key, x in clean.items():
        if x is None:
            continue
        y = dirty[key]
        if key in ("o", "dq", "lse"):
            on_rows = ~off[:, None].expand(x.shape[:3])
            same(x[on_rows], y[on_rows], key)
            offv = y[~on_rows]
            assert bool((offv == (-math.inf if key == "lse" else 0)).all()), key
        elif key in ("dk", "dv", "dkg", "dvg"):
            keys_off = torch.cat([torch.zeros_like(off[:, :c.g]), off], dim=1)[:, None].expand(x.shape[:3])
            same(x[~keys_off], y[~keys_off], key)
            assert bool((y[keys_off] == 0).all()), key
        else:
            same(x, y, key)


@gpu
@pytest.mark.parametrize("case", DROPPED, ids=ids(DROPPED))
def test_dropout_matches_the_mask_restatement(case):
    """the local rows with dropout against the reference algorithm on each image's residue sub-grids with the exact mask:
    row = the query's padded-grid token, col = its column of the sub-grid's attn1 (tests/test_gpu_dilation.py)"""
    c = case
    dtype, impl, flags, odt, (tf, tb, _) = VARIANTS[c.variant]
    t = make(c, seed=9)
    vw = views(t, c)
    res = run(*vw, t, geo(c), c.variant, sizes=c.sizes, drop=drop_of(c))
    g, H, B = c.g, c.H, nimg(c)
    q64, k64, v64 = (x.double().cpu() for x in vw[:3])
    qg64 = vw[3].double().cpu() if g else None
    d_o = vw[6].double().cpu()
    tab = t["table"].double() if c.rpe else None
    g2l = t["g2l"].double() if (c.rpe and g) else None
    g2g = t["g2g"].double() if (c.rpe and g) else None
    # the reference is assembled over every image and residue and compared as whole tensors (off-image rows zero on both
    # sides), the metric of the bars
    ref = {key: torch.zeros(res[key].shape, dtype=torch.float64) for key in ("o", "dq", "dk", "dv")}
    for bi in range(B):
        h, wb = c.sizes[bi] if c.sizes else (c.nx, c.ny)
        for a, b, na, nb, ridx in residues(h, wb, c.d):
            idx = (ridx // wb) * c.ny + ridx % wb
            keep = _keep_sub(SEED, OFFSET, c.p, B, H, c.nx, c.ny, c.w, g, c.mode, c.d, a, b, na, nb)[bi * H:(bi + 1) * H]
            qs = q64[bi:bi + 1, :, idx].clone().requires_grad_(True)
            ks = torch.cat([k64[bi:bi + 1, :, :g], k64[bi:bi + 1, :, g + idx]], dim=2).requires_grad_(True)
            vs = torch.cat([v64[bi:bi + 1, :, :g], v64[bi:bi + 1, :, g + idx]], dim=2).requires_grad_(True)
            keep_g = torch.ones(H, g, g + len(idx), dtype=torch.float64) if g else None
            o, _ = tdrop.chunked_dropout_reference(qs, ks, vs, qg64[bi:bi + 1] if g else None, ks.detach() if g else None,
                                                   vs.detach() if g else None, tab, g2l, g2g, keep, keep_g, nx=na, ny=nb,
                                                   w=c.w, exact=c.exact, mode=c.mode, scale=c.D ** -0.5)
            (o * d_o[bi:bi + 1, :, idx]).sum().backward()
            ref["o"][bi, :, idx], ref["dq"][bi, :, idx] = o.detach()[0], qs.grad[0]
            ref["dk"][bi, :, g + idx], ref["dv"][bi, :, g + idx] = ks.grad[0, :, g:], vs.grad[0, :, g:]
    errs = dict(o=relerr(res["o"], ref["o"]), dq=relerr(res["dq"], ref["dq"]))
    if c.sep or g == 0:                      # shared weights: the local keys' rows also hold the global queries' terms
        errs.update(dk=relerr(res["dk"][:, :, g:], ref["dk"][:, :, g:]), dv=relerr(res["dv"][:, :, g:], ref["dv"][:, :, g:]))
    record("subgrid_matrix_dropout", cid(c), **errs)
    bad = {key: e for key, e in errs.items() if not e < (tf if key == "o" else tb)}
    assert not bad, (bad, errs)


DETERMINISM = [c for c in MATRIX if c.D == 128 and c.p and c.variant in ("wgmma_bf16", "simt_f32")][:2] + PRODUCTION


@gpu
@pytest.mark.parametrize("case", DETERMINISM, ids=ids(DETERMINISM))
def test_backward_repeats_bitwise_with_a_dirty_workspace(case):
    c = case
    t = make(c, seed=3)
    vw = views(t, c)
    first = run(*vw, t, geo(c), c.variant, sizes=c.sizes, drop=drop_of(c))
    second = run(*vw, t, geo(c), c.variant, sizes=c.sizes, drop=drop_of(c), fill=float("nan"))
    for key, x in first.items():
        if x is not None:
            same(x, second[key], key)


@gpu
def test_split_fp32_above_its_head_tiles_falls_back_to_simt():
    """fp32 under TF32 matmuls at D = 96, dilated and sized: the wgmma family declines it (split tiles stop at 64) and
    ops.vil_attention runs the SIMT family, at its fp32 bars"""
    c = Case("simt_f32", 96, 12, 11, 4, 2, 1, True, False, 0, 0, ((12, 11), (7, 6)))
    t = make(c, seed=6)
    leaf = {k: t[k].to(DEV).requires_grad_(True) for k in ("q_all", "kv", "table", "g2l", "g2g")}
    prec = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    try:
        out = ops.vil_attention(leaf["q_all"], leaf["kv"], None, None, leaf["table"], leaf["g2l"], leaf["g2g"],
                                num_heads=c.H, nx=c.nx, ny=c.ny, w=c.w, nglo=c.g, scale=c.D ** -0.5, dilation=c.d,
                                image_sizes=c.sizes)
        assert _lib.last_impl() == "simt"
        out.backward(t["dout"].to(DEV))
        assert _lib.last_impl() == "simt"
    finally:
        torch.backends.cuda.matmul.fp32_precision = prec
    grads, ref = oracle(t, c)
    o = ops._heads(out.detach().double().cpu(), c.H)
    assert relerr(o[:, :, c.g:], ref["o"]) < 1e-5 and relerr(o[:, :, :c.g], ref["og"]) < 1e-5
    for key, x in grads.items():
        assert relerr(leaf[key].grad, x) < _bar(key, VARIANTS["simt_f32"][4]), key


# --------------------------------------------------------------------------- CPU: the guards
def test_mirror_reads_the_head_dim_switches():
    """every head-dim switch of the two families takes exactly the tiles / buckets of its ladder (the default standing
    for the largest), so the mirror's tiles are the dispatch's"""
    assert RULES.wg_tiles[-1] == RULES.simt_buckets[-1] == 128
    for name, ((labels, default), ladder) in RULES.switches.items():
        assert default and sorted(labels + [ladder[-1]]) == ladder, (name, labels, ladder)
    assert RULES.split_max in RULES.wg_tiles and RULES.wg_align == 8


def test_every_dil_and_sized_instantiation_is_covered():
    """every DIL / SIZED kernel instantiation a dilated or sized call can launch is launched by some case"""
    reach = RULES.reachable()
    covered = set().union(*(RULES.of_case(c) for c in ALL))
    missing = sorted(reach - covered, key=str)
    assert not missing, "no case launches:\n" + "\n".join(map(str, missing))
    assert covered <= reach, sorted(covered - reach, key=str)
    # wgmma: (T, TO) x tiles (split without 128) x DROP x (forward, pass 1 with / without the table, pass 2)
    assert sum(1 for x in reach if x[0] == "wgmma") == (4 * len(RULES.wg_tiles) + 3) * 2 * 4


def test_each_tile_sees_every_feature():
    """each (family, T, TO, head tile): with and without the table and dropout; g = 0, shared and separate global
    weights; dilation only, sizes only and both"""
    groups = {}
    for c in ALL:
        dtype, fam, _, odt, _ = VARIANTS[c.variant]
        hd = RULES.tile(c.D) if fam == "wgmma" else RULES.bucket(c.D)
        groups.setdefault((fam, dtype, odt, hd), []).append(c)
    for key, cs in groups.items():
        kinds = {"dil" if c.sizes is None else "sizes" if c.d == 1 else "both" for c in cs}
        globs = {"g0" if c.g == 0 else "sep" if c.sep else "shared" for c in cs}
        assert kinds == {"dil", "sizes", "both"} and globs == {"g0", "sep", "shared"}, (key, kinds, globs)
        assert {c.rpe for c in cs} == {False, True}, key
        assert {c.p > 0 for c in cs} == ({False, True} if trains(cs[0]) else {False}), key


def test_multi_piece_chunks_are_covered():
    """npc = ceil(w^2 / 64) >= 2 under DIL on each family: w = 9, 12 and 15, at least two head tiles, d = 1, 2 and 3,
    sizes that are not multiples of w, crops narrower than w and sub-grids of a single partial chunk"""
    for fam in ("wgmma", "simt"):
        cs = [c for c in ALL if VARIANTS[c.variant][1] == fam and (c.w * c.w + 63) // 64 >= 2 and (c.d > 1 or c.sizes)]
        hd = RULES.tile if fam == "wgmma" else RULES.bucket
        assert {c.w for c in cs} >= {9, 12, 15} and len({hd(c.D) for c in cs}) >= 2, fam
        assert {c.d for c in cs} >= {1, 2, 3} and any(c.p for c in cs), fam
        sized = [c for c in cs if c.sizes]
        assert any(h % c.w and wb % c.w for c in sized for h, wb in c.sizes), fam
        assert any(min(h, wb) < c.w for c in sized for h, wb in c.sizes), fam
        assert any(0 < na < c.w and 0 < nb < c.w for c in sized for h, wb in c.sizes
                   for _, _, na, nb, _ in residues(h, wb, c.d)), fam


def test_cases_are_well_formed():
    for c in ALL:
        dtype, fam = VARIANTS[c.variant][:2]
        assert not RULES.refused(fam, TNAME[dtype], c.D, c.p > 0), cid(c)
        if fam == "wgmma":
            assert c.D % RULES.wg_align == 0, cid(c)
        assert c.exact in (0, 1, -1) and (c.exact != 1 or c.mode == 0), cid(c)
        if c.sizes:
            assert all(1 <= h <= c.nx and 1 <= wb <= c.ny for h, wb in c.sizes), cid(c)
            assert any((h, wb) != (c.nx, c.ny) for h, wb in c.sizes), cid(c)   # else the unsized call
    assert len(set(ids(ALL))) == len(ALL)


def _nslice(c):
    """vil_attn_api.cu make_geo: pass-1 image slices of a call with the bias table (132 SMs)"""
    n0, m0 = -(-c.nx // c.d), -(-c.ny // c.d)
    mx, my = c.d * -(-n0 // c.w), c.d * -(-m0 // c.w)
    per_slice = c.H * mx * my * ((c.w * c.w + 63) // 64)
    return min(nimg(c), -(-8 * 132 // per_slice))


def test_production_case_runs_several_images_per_pass1_cta():
    c = PRODUCTION[0]
    assert (c.nx, c.ny, c.w, c.H, c.D, c.g, c.rpe, c.d) == (56, 56, 7, 3, 32, 1, True, 2)
    assert nimg(c) == 8 > _nslice(c)
    assert len(set(c.sizes)) > 2


# --------------------------------------------------------------------------- CPU: refusals before any launch
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    return _lib.load()


def _params(D, dtype, bwd, impl=None, **kw):
    """a SIMT call on 2 images of 28 x 28 at head dim D in the Linear-output layouts; never dereferenced"""
    p = _lib.VilAttnParams()
    p.struct_bytes = ctypes.sizeof(_lib.VilAttnParams)
    p.dtype, p.impl = dtype, _lib.VIL_IMPL_SIMT if impl is None else impl
    p.B, p.H, p.D, p.nx, p.ny, p.w, p.nglo, p.exact, p.mode = 2, 2, D, 28, 28, 7, 0, 0, 0
    p.scale = D ** -0.5
    names = ("q", "k", "v", "o") + (("d_o", "dq", "dk", "dv") if bwd else ())
    for name in names:
        x = getattr(p, name)
        x.ptr, x.sb, x.sh, x.st = 1 << 20, 784 * 2 * 2 * D, D, 2 * 2 * D
    p.lse = 1 << 20
    for key, val in kw.items():
        setattr(p, key, val)
    if bwd:
        need = _lib.load().vil_attn_workspace_bytes(ctypes.byref(p), 1)
        assert need > 0
        p.workspace, p.workspace_bytes = 1 << 24, need
    return p


@pytest.mark.parametrize("dtype", [_lib.VIL_BF16, _lib.VIL_F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("how", ["dilated", "sized", "both"])
def test_simt_lowp_refusals_under_dilation_and_sizes(lib, dtype, how):
    """the bf16 / fp16 SIMT backward above head dim 64, and their forward with dropout there, are refused with
    VIL_E_UNSUPPORTED before any launch, dilated or sized"""
    dil = dict(flags=_lib.VIL_FLAG_DILATED, dilation=2) if how != "sized" else {}
    before = _lib.launch_count()
    for D in (72, 96, 128):
        assert _call(lib, how, True, _params(D, dtype, True, **dil)) == _lib.VIL_E_UNSUPPORTED
        assert "64 < D <= 128 is trained by the wgmma family" in _lib.last_error()
        assert _call(lib, how, False, _params(D, dtype, False, dropout_p=0.1, **dil)) == _lib.VIL_E_UNSUPPORTED
        assert "dropout supports head dim <= 64" in _lib.last_error()
        # the same calls at head dim 64 pass every host check: their refusal is the head dim's
        assert RULES.bucket(D) > RULES.simt_bwd_max == RULES.simt_drop_fwd_max == 64
    assert _lib.launch_count() == before


def _call(lib, how, bwd, p):
    """the plain entry point for a dilated call, the sized one (grids never dereferenced) otherwise"""
    if how == "dilated":
        return (lib.vil_attn_bwd_sm100 if bwd else lib.vil_attn_fwd_sm100)(ctypes.byref(p), None)
    fn = lib.vil_attn_bwd_sized_sm100 if bwd else lib.vil_attn_fwd_sized_sm100
    return fn(ctypes.byref(p), ctypes.c_void_p(1 << 24), None)


@pytest.mark.parametrize("how", ["dilated", "sized"])
def test_split_fp32_above_64_is_declined_by_wgmma(lib, how):
    """split fp32 at D > 64 is not a wgmma call (vil_attn_wgmma_supported), dilated or sized; forcing the family is
    refused before any launch, and the automatic choice is the SIMT family (test_split_fp32_above_its_head_tiles_...)"""
    dil = dict(flags=_lib.VIL_FLAG_F32_SPLIT | _lib.VIL_FLAG_DILATED, dilation=3) if how == "dilated" else \
        dict(flags=_lib.VIL_FLAG_F32_SPLIT)
    before = _lib.launch_count()
    for D in (64, 72, 128):
        p = _params(D, _lib.VIL_F32, False, impl=_lib.VIL_IMPL_AUTO, **dil)
        assert lib.vil_attn_wgmma_supported(ctypes.byref(p)) == (1 if D <= RULES.split_max else 0), D
    for bwd in (False, True):
        rc = _call(lib, how, bwd, _params(96, _lib.VIL_F32, bwd, impl=_lib.VIL_IMPL_WGMMA, **dil))
        assert rc == _lib.VIL_E_UNSUPPORTED and "head dim > 64" in _lib.last_error(), (bwd, _lib.last_error())
    assert _lib.launch_count() == before
