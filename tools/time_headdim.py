"""What a 128-wide head tile costs: the attention operator's forward, backward pass 1 and pass 2 at head dim 64 and 128 on a
ViL-like grid (56x56 tokens, w = 7, one global token, 256 images, bf16, through the C ABI).  The two head dims keep
H * D = 128 (H = 2 at D = 64, H = 1 at D = 128), so both rows are the same channels per image.  Beside them the SIMT
forward at D = 128 (impl="simt"), the path such a call took before the wgmma family had a 128 tile.  CUDA events after
warm-up, the configurations alternated and the medians reported, with the card's name and power limit read in the same
run.   usage: python tools/time_headdim.py"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vision_longformer_b200 import _lib, vil_attention_raw_backward, vil_attention_raw_forward  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit": None}


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return ts


def median(ts):
    ts = sorted(ts)
    return ts[len(ts) // 2]


def setup(dev, H, D, B=256, nx=56, ny=56, w=7, g=1):
    N = g + nx * ny
    gen = torch.Generator(device=dev).manual_seed(300)
    mk = lambda *s: torch.randn(*s, generator=gen, device=dev, dtype=torch.float32).to(torch.bfloat16)
    q, k, v, qg, go, gog = mk(B, H, nx * ny, D), mk(B, H, N, D), mk(B, H, N, D), mk(B, H, g, D), mk(B, H, nx * ny, D), mk(B, H, g, D)
    o, og = torch.empty_like(q), torch.empty_like(qg)
    dq, dk, dv, dqg = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v), torch.empty_like(qg)
    kw = dict(nx=nx, ny=ny, w=w, exact=0, mode=0, scale=D ** -0.5)
    lse, lse_g = vil_attention_raw_forward(q, k, v, qg, k, v, None, None, None, o, og, **kw)
    fam = _lib.last_impl()
    # skip_mask: bit0 global-token kernels, bit1 local forward / pass 1, bit2 pass 2, bit3 delta
    fwd = lambda impl="auto": vil_attention_raw_forward(q, k, v, qg, k, v, None, None, None, o, og, skip_mask=1, impl=impl, **kw)
    bwd = lambda sk: vil_attention_raw_backward(q, k, v, qg, k, v, None, None, None, o, og, lse, lse_g, go, gog, dq, dk, dv, dqg,
                                                dk, dv, None, None, None, skip_mask=sk, **kw)
    return fam, {"fwd": fwd, "pass1": lambda: bwd(1 | 4 | 8), "pass2": lambda: bwd(1 | 2 | 8)}


def main(rounds=4, reps=10, B=256):
    dev = torch.device("cuda")
    out = {"card": card(), "grid": "56x56 w=7 g=1, %d images, bf16, H*D = 128" % B}
    runs, keep = {}, []
    for H, D in ((2, 64), (1, 128)):
        fam, fns = setup(dev, H, D, B)
        out[f"D{D}_family"] = fam
        for ph, fn in fns.items():
            runs[f"D{D}_{ph}"] = fn
        keep.append(fns)
    runs["D128_fwd_simt"] = lambda f=keep[1]["fwd"]: f("simt")
    times = {name: [] for name in runs}
    for fn in runs.values():                            # warm-up
        timed(fn, 3)
    for _ in range(rounds):                             # alternate the configurations
        for name, fn in runs.items():
            times[name] += timed(fn, reps)
    for name, ts in times.items():
        ms = median(ts)
        out[name + "_ms"] = round(ms, 4)
        out[name + "_us_per_image"] = round(1e3 * ms / B, 3)
    out["D128_fwd_simt_over_wgmma"] = round(out["D128_fwd_simt_ms"] / out["D128_fwd_ms"], 2)
    for ph in ("fwd", "pass1", "pass2"):
        out[f"{ph}_D128_over_D64"] = round(out[f"D128_{ph}_ms"] / out[f"D64_{ph}_ms"], 3)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
