"""Per-image token grids in a padded batch (vil_attn_fwd_sized_sm100 / _bwd_sized_sm100): the forward, backward pass 1
and pass 2 on a detection-style batch of 8 images padded to 200 x 336 tokens (ViL-Small stage 1: 3 heads of 32) and to
100 x 168 (stage 2: 3 heads of 64), with seeded sizes whose long side spans 200-336 (stage 2: half of it, rounded up).
w = 7, one global token, the bias table on, bf16 on the wgmma family and fp32 on the SIMT family, through the C ABI.

Four ways to run the same batch, the configurations alternated, CUDA events after warm-up, medians reported, with the
card's name and power limit read in the same run:
  padded     no sizes: every padding token attends and is attended to (the call without image_sizes)
  sized      with the sizes (includes the one launch that writes the off-image rows)
  per_image  one B = 1 call per cropped image (the crops made beforehand, not timed)
  full_dil   every image full, through the sized entry point: the DIL instantiations at d = 1 where `padded` runs the plain
             ones.  The op never takes this path (full sizes call the unsized entry point); it prices the per-CTA
             sub-grid of the DIL instantiations plus the extra zero-fill launch (which finds no off-image row).
Writes time_image_sizes.json to the output directory.   usage: python tools/time_image_sizes.py --out DIR"""
import argparse
import json
import os
import random
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.time_headdim import card, median, timed  # noqa: E402
from vision_longformer_b200 import _lib, vil_attention_raw_backward, vil_attention_raw_forward  # noqa: E402

SHAPES = {"S1": dict(H=3, D=32, nx=200, ny=336, div=1), "S2": dict(H=3, D=64, nx=100, ny=168, div=2)}
FAMILIES = {"wgmma_bf16": (torch.bfloat16, "wgmma"), "simt_f32": (torch.float32, "simt")}


def batch_sizes(n=8, seed=0):
    """seeded (h, w) of n detection-style images padded to 200 x 336: the long side spans 200-336, portrait ones fit"""
    rnd = random.Random(seed)
    out = []
    for _ in range(n):
        long_side = rnd.randint(200, 336)
        short = rnd.randint(120, 200)
        out.append((short, long_side))
    return out


def setup(dev, H, D, nx, ny, div, dtype, impl, how, w=7, g=1):
    sizes = [(-(-h // div), -(-wb // div)) for h, wb in batch_sizes()]
    B = len(sizes)
    N = g + nx * ny
    gen = torch.Generator(device=dev).manual_seed(300)
    mk = lambda *s: torch.randn(*s, generator=gen, device=dev, dtype=torch.float32).to(dtype)
    q, k, v, qg, go, gog = mk(B, H, nx * ny, D), mk(B, H, N, D), mk(B, H, N, D), mk(B, H, g, D), mk(B, H, nx * ny, D), mk(B, H, g, D)
    tab = 0.02 * torch.randn((4 * w - 1) ** 2, H, generator=gen, device=dev)
    g2l, g2g = 0.02 * torch.randn(2, H, g, generator=gen, device=dev), 0.02 * torch.randn(H, g, g, generator=gen, device=dev)

    def calls(q, k, v, qg, go, gog, nx, ny, **extra):
        o, og = torch.empty_like(q), torch.empty_like(qg)
        dq, dk, dv, dqg = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v), torch.empty_like(qg)
        dtab, dg2l, dg2g = torch.zeros_like(tab), torch.zeros_like(g2l), torch.zeros_like(g2g)
        kw = dict(nx=nx, ny=ny, w=w, exact=0, mode=0, scale=D ** -0.5, impl=impl, **extra)
        lse, lse_g = vil_attention_raw_forward(q, k, v, qg, k, v, tab, g2l, g2g, o, og, **kw)
        # skip_mask: bit0 global-token kernels, bit1 local forward / pass 1, bit2 pass 2, bit3 delta
        fwd = lambda: vil_attention_raw_forward(q, k, v, qg, k, v, tab, g2l, g2g, o, og, skip_mask=1, **kw)
        bwd = lambda sk: vil_attention_raw_backward(q, k, v, qg, k, v, tab, g2l, g2g, o, og, lse, lse_g, go, gog, dq, dk, dv,
                                                    dqg, dk, dv, dtab, dg2l, dg2g, skip_mask=sk, **kw)
        return [fwd, lambda: bwd(1 | 4 | 8), lambda: bwd(1 | 2 | 8)]

    if how == "padded":
        fns = calls(q, k, v, qg, go, gog, nx, ny)
    elif how == "sized":
        fns = calls(q, k, v, qg, go, gog, nx, ny, image_sizes=sizes)
    elif how == "full_dil":
        fns = calls(q, k, v, qg, go, gog, nx, ny, _image_hw=torch.tensor([[nx, ny]] * B, dtype=torch.int32, device=dev))
    else:
        per = []
        for b, (h, wb) in enumerate(sizes):
            idx = (torch.arange(h, device=dev)[:, None] * ny + torch.arange(wb, device=dev)[None, :]).reshape(-1)
            crop = lambda t: torch.cat([t[b:b + 1, :, :g], t[b:b + 1, :, g + idx]], dim=2).contiguous()
            per.append(calls(q[b:b + 1, :, idx].contiguous(), crop(k), crop(v), qg[b:b + 1].contiguous(),
                             go[b:b + 1, :, idx].contiguous(), gog[b:b + 1].contiguous(), h, wb))
        fns = [lambda i=i: [p[i]() for p in per] for i in range(3)]
    fam = _lib.last_impl()
    real = sum(h * wb for h, wb in sizes) / (B * nx * ny)
    return fam, dict(zip(("fwd", "pass1", "pass2"), fns)), real


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_image_sizes needs a CUDA device")
    dev = torch.device("cuda")
    res = {"card": card(), "what": "w=7 g=1 rpe, 8 images padded to 200x336 (S1) / 100x168 (S2)",
           "sizes_S1": batch_sizes()}
    hows = ("padded", "sized", "per_image", "full_dil")
    for fname, (dtype, impl) in FAMILIES.items():
        runs = {}
        for sname, shp in SHAPES.items():
            for how in hows:
                fam, fns, real = setup(dev, dtype=dtype, impl=impl, how=how, **shp)
                assert fam == impl, (fam, impl)
                res[f"{sname}_real_token_fraction"] = round(real, 3)
                for ph, fn in fns.items():
                    runs[f"{fname}_{sname}_{ph}_{how}"] = fn
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
                for how in hows[1:]:
                    res[f"{fname}_{sname}_{ph}_{how}_over_padded"] = round(
                        res[f"{fname}_{sname}_{ph}_{how}_ms"] / res[f"{fname}_{sname}_{ph}_padded_ms"], 3)
        del runs, times
        torch.cuda.empty_cache()
    res["card_after"] = card()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "time_image_sizes.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
