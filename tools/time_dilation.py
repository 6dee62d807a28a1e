"""Dilated sliding-chunk attention (VIL_FLAG_DILATED): the forward, backward pass 1 and pass 2 at dilation d = 1, 2 and 3,
at the ViL-Small stage 1 (56x56 tokens, 3 heads of 32) and stage 2 (28x28, 3 heads of 64) shapes, w = 7, one global token,
the bias table on, bf16 on the wgmma family and fp32 on the SIMT family, 256 images, through the C ABI.  CUDA events
after warm-up, the configurations alternated and the medians reported, with the card's name and power limit read in the
same run.  Beside each time: the chunks the d^2 sub-grids have against d = 1 (every chunk costs a CTA per piece, padded
or not).  Writes time_dilation.json to the output directory.   usage: python tools/time_dilation.py --out DIR"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.time_headdim import card, median, timed  # noqa: E402
from vision_longformer_b200 import _lib, vil_attention_raw_backward, vil_attention_raw_forward  # noqa: E402

SHAPES = {"S1": dict(H=3, D=32, nx=56, ny=56), "S2": dict(H=3, D=64, nx=28, ny=28)}
FAMILIES = {"wgmma_bf16": (torch.bfloat16, "wgmma"), "simt_f32": (torch.float32, "simt")}
DILATIONS = (1, 2, 3)


def chunks(nx, ny, w, d):
    """chunks of the d^2 residue sub-grids (real ones, without the CTAs of the virtual grid that exit at once)"""
    cdiv = lambda a, b: -(-a // b)
    return sum(cdiv(cdiv(nx - a, d), w) * cdiv(cdiv(ny - b, d), w) for a in range(d) for b in range(d))


def setup(dev, H, D, nx, ny, dtype, impl, d, B=256, w=7, g=1):
    N = g + nx * ny
    gen = torch.Generator(device=dev).manual_seed(300)
    mk = lambda *s: torch.randn(*s, generator=gen, device=dev, dtype=torch.float32).to(dtype)
    q, k, v, qg, go, gog = mk(B, H, nx * ny, D), mk(B, H, N, D), mk(B, H, N, D), mk(B, H, g, D), mk(B, H, nx * ny, D), mk(B, H, g, D)
    tab = 0.02 * torch.randn((4 * w - 1) ** 2, H, generator=gen, device=dev)
    g2l, g2g = 0.02 * torch.randn(2, H, g, generator=gen, device=dev), 0.02 * torch.randn(H, g, g, generator=gen, device=dev)
    dtab, dg2l, dg2g = torch.zeros_like(tab), torch.zeros_like(g2l), torch.zeros_like(g2g)
    o, og = torch.empty_like(q), torch.empty_like(qg)
    dq, dk, dv, dqg = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v), torch.empty_like(qg)
    kw = dict(nx=nx, ny=ny, w=w, exact=0, mode=0, scale=D ** -0.5, impl=impl, dilation=d)
    lse, lse_g = vil_attention_raw_forward(q, k, v, qg, k, v, tab, g2l, g2g, o, og, **kw)
    vil_attention_raw_backward(q, k, v, qg, k, v, tab, g2l, g2g, o, og, lse, lse_g, go, gog, dq, dk, dv, dqg, dk, dv,
                               dtab, dg2l, dg2g, **kw)
    fam = _lib.last_impl()
    # skip_mask: bit0 global-token kernels, bit1 local forward / pass 1, bit2 pass 2, bit3 delta; pass 1 includes the
    # bias-table reduction it feeds
    fwd = lambda: vil_attention_raw_forward(q, k, v, qg, k, v, tab, g2l, g2g, o, og, skip_mask=1, **kw)
    bwd = lambda sk: vil_attention_raw_backward(q, k, v, qg, k, v, tab, g2l, g2g, o, og, lse, lse_g, go, gog, dq, dk, dv, dqg,
                                                dk, dv, dtab, dg2l, dg2g, skip_mask=sk, **kw)
    return fam, {"fwd": fwd, "pass1": lambda: bwd(1 | 4 | 8), "pass2": lambda: bwd(1 | 2 | 8)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--images", type=int, default=256)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_dilation needs a CUDA device")
    dev = torch.device("cuda")
    B = a.images
    res = {"card": card(), "what": "w=7 g=1 rpe, %d images; dilation 1 / 2 / 3" % B}
    for fname, (dtype, impl) in FAMILIES.items():
        runs = {}
        for sname, shp in SHAPES.items():
            for d in DILATIONS:
                res[f"{sname}_d{d}_chunks_over_d1"] = round(chunks(shp["nx"], shp["ny"], 7, d) / chunks(shp["nx"], shp["ny"], 7, 1), 3)
                fam, fns = setup(dev, B=B, dtype=dtype, impl=impl, d=d, **shp)
                assert fam == impl, (fam, impl)
                for ph, fn in fns.items():
                    runs[f"{fname}_{sname}_{ph}_d{d}"] = fn
        times = {name: [] for name in runs}
        for fn in runs.values():                            # warm-up
            timed(fn, 3)
        for _ in range(a.rounds):                           # alternate the configurations
            for name, fn in runs.items():
                times[name] += timed(fn, a.reps)
        for name, ts in times.items():
            res[name + "_ms"] = round(median(ts), 4)
        for sname in SHAPES:
            for ph in ("fwd", "pass1", "pass2"):
                for d in DILATIONS[1:]:
                    res[f"{fname}_{sname}_{ph}_d{d}_over_d1"] = round(
                        res[f"{fname}_{sname}_{ph}_d{d}_ms"] / res[f"{fname}_{sname}_{ph}_d1_ms"], 3)
        del runs, times
        torch.cuda.empty_cache()
    res["card_after"] = card()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "time_dilation.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
