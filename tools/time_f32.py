"""fp32 attention, SIMT against the split-bf16 wgmma kernels (VIL_FLAG_F32_SPLIT): the forward, backward pass 1 and pass 2
at the ViL-Small stage 1 (56x56 tokens, 3 heads of 32) and stage 2 (28x28, 3 heads of 64) shapes, w = 7, one global token,
256 images, through the C ABI.  CUDA events after warm-up, the configurations alternated and the medians reported, with
the card's name and power limit read in the same run; beside the times, the norm-relative difference of the two families'
o, dq, dk and dv.  Writes time_f32.json to the output directory.   usage: python tools/time_f32.py --out DIR"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.time_headdim import card, median, timed  # noqa: E402
from vision_longformer_b200 import _lib, vil_attention_raw_backward, vil_attention_raw_forward  # noqa: E402

SHAPES = {"S1": dict(H=3, D=32, nx=56, ny=56), "S2": dict(H=3, D=64, nx=28, ny=28)}


def setup(dev, H, D, nx, ny, impl, flags, B=256, w=7, g=1):
    N = g + nx * ny
    gen = torch.Generator(device=dev).manual_seed(300)
    mk = lambda *s: torch.randn(*s, generator=gen, device=dev, dtype=torch.float32)
    q, k, v, qg, go, gog = mk(B, H, nx * ny, D), mk(B, H, N, D), mk(B, H, N, D), mk(B, H, g, D), mk(B, H, nx * ny, D), mk(B, H, g, D)
    o, og = torch.empty_like(q), torch.empty_like(qg)
    dq, dk, dv, dqg = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v), torch.empty_like(qg)
    kw = dict(nx=nx, ny=ny, w=w, exact=0, mode=0, scale=D ** -0.5, impl=impl, flags=flags)
    lse, lse_g = vil_attention_raw_forward(q, k, v, qg, k, v, None, None, None, o, og, **kw)
    vil_attention_raw_backward(q, k, v, qg, k, v, None, None, None, o, og, lse, lse_g, go, gog, dq, dk, dv, dqg, dk, dv,
                               None, None, None, **kw)
    fam = (_lib.last_impl(), _lib.last_kernel())
    outs = {"o": o.clone(), "dq": dq.clone(), "dk": dk.clone(), "dv": dv.clone()}
    # skip_mask: bit0 global-token kernels, bit1 local forward / pass 1, bit2 pass 2, bit3 delta
    fwd = lambda: vil_attention_raw_forward(q, k, v, qg, k, v, None, None, None, o, og, skip_mask=1, **kw)
    bwd = lambda sk: vil_attention_raw_backward(q, k, v, qg, k, v, None, None, None, o, og, lse, lse_g, go, gog, dq, dk, dv, dqg,
                                                dk, dv, None, None, None, skip_mask=sk, **kw)
    return fam, outs, {"fwd": fwd, "pass1": lambda: bwd(1 | 4 | 8), "pass2": lambda: bwd(1 | 2 | 8)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--images", type=int, default=256)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_f32 needs a CUDA device")
    dev = torch.device("cuda")
    B = a.images
    res = {"card": card(), "what": "fp32, w=7 g=1, %d images; SIMT vs split-bf16 wgmma (VIL_FLAG_F32_SPLIT)" % B}
    runs = {}
    for sname, shp in SHAPES.items():
        outs = {}
        for fname, impl, flags in (("simt", "simt", 0), ("split", "wgmma", _lib.VIL_FLAG_F32_SPLIT)):
            fam, outs[fname], fns = setup(dev, B=B, impl=impl, flags=flags, **shp)
            res[f"{sname}_{fname}_family"] = "/".join(fam)
            for ph, fn in fns.items():
                runs[f"{sname}_{ph}_{fname}"] = fn
        for n in ("o", "dq", "dk", "dv"):
            x, r = outs["split"][n].double(), outs["simt"][n].double()
            res[f"{sname}_{n}_split_vs_simt_relerr"] = float((x - r).norm() / r.norm())
        del outs
    times = {name: [] for name in runs}
    for fn in runs.values():                            # warm-up
        timed(fn, 3)
    for _ in range(a.rounds):                           # alternate the configurations
        for name, fn in runs.items():
            times[name] += timed(fn, a.reps)
    for name, ts in times.items():
        res[name + "_ms"] = round(median(ts), 4)
    faster = True
    for sname in SHAPES:
        for ph in ("fwd", "pass1", "pass2"):
            sp = res[f"{sname}_{ph}_simt_ms"] / res[f"{sname}_{ph}_split_ms"]
            res[f"{sname}_{ph}_simt_over_split"] = round(sp, 2)
            faster &= sp > 1.0
    res["split_faster_everywhere"] = faster
    res["card_after"] = card()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "time_f32.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
