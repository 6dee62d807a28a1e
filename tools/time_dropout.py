"""What attention dropout costs: the attention operator's forward and backward at p = 0 and p = 0.1 (ViL-Small stage-1 and
stage-2 shapes, 256 images, bf16, through the C ABI) and ViL-Small training img/s at attn_drop_rate 0 and 0.1 (256 images
per step, bf16 autocast, AdamW).  CUDA events after warm-up; the two settings are alternated and the medians reported,
with the card's name and power limit read in the same run.   usage: python tools/time_dropout.py [--no-train]"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vision_longformer_b200 import build_vil, vil_attention_raw_backward, vil_attention_raw_forward  # noqa: E402


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


def operator(dev, rounds=4, reps=10):
    res = {}
    for tag, (H, M, nx, ny) in {"S1": (3, 32, 56, 56), "S2": (3, 64, 28, 28)}.items():
        B, w, g = 256, 7, 1
        N = g + nx * ny
        gen = torch.Generator(device=dev).manual_seed(300)
        mk = lambda *s: torch.randn(*s, generator=gen, device=dev, dtype=torch.float32).to(torch.bfloat16)
        q, k, v, qg, go, gog = mk(B, H, nx * ny, M), mk(B, H, N, M), mk(B, H, N, M), mk(B, H, g, M), mk(B, H, nx * ny, M), mk(B, H, g, M)
        o, og = torch.empty_like(q), torch.empty_like(qg)
        dq, dk, dv, dqg = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v), torch.empty_like(qg)
        kw = dict(nx=nx, ny=ny, w=w, exact=0, mode=0, scale=M ** -0.5)
        st = {}
        for p in (0.0, 0.1):
            d = dict(dropout_p=p, dropout_seed=1234, dropout_offset=0)
            lse, lse_g = vil_attention_raw_forward(q, k, v, qg, k, v, None, None, None, o, og, **kw, **d)
            bwd = lambda sk, d=d, lse=lse, lse_g=lse_g: vil_attention_raw_backward(
                q, k, v, qg, k, v, None, None, None, o, og, lse, lse_g, go, gog, dq, dk, dv, dqg, dk, dv, None, None, None,
                skip_mask=sk, **kw, **d)
            fwd = lambda sk, d=d: vil_attention_raw_forward(q, k, v, qg, k, v, None, None, None, o, og, skip_mask=sk, **kw, **d)
            # whole calls, and each kernel alone (skip_mask: bit0 global-token kernels, bit1 local forward / pass 1,
            # bit2 pass 2, bit3 delta)
            st[p] = dict(fwd=lambda f=fwd: f(0), bwd=lambda b=bwd: b(0), fwd_local=lambda f=fwd: f(1),
                         fwd_global=lambda f=fwd: f(2), bwd_pass1=lambda b=bwd: b(1 | 4 | 8),
                         bwd_pass2=lambda b=bwd: b(1 | 2 | 8), bwd_global=lambda b=bwd: b(2 | 4 | 8))
        phases = list(st[0.0])
        times = {(p, ph): [] for p in st for ph in phases}
        for p in st:                                    # warm-up
            for ph in phases:
                timed(st[p][ph], 3)
        for _ in range(rounds):                         # alternate the two settings
            for p in st:
                for ph in phases:
                    times[(p, ph)] += timed(st[p][ph], reps)
        for (p, ph), ts in times.items():
            res[f"{tag}_{ph}_p{p}_ms"] = round(median(ts), 4)
        for ph in phases:
            res[f"{tag}_{ph}_ratio"] = round(res[f"{tag}_{ph}_p0.1_ms"] / res[f"{tag}_{ph}_p0.0_ms"], 3)
        del q, k, v, qg, go, gog, o, og, dq, dk, dv, dqg
        torch.cuda.empty_cache()
    return res


def training(dev, B=256, rounds=2, steps=8, warmup=3):
    res = {}
    x = torch.randn(B, 3, 224, 224, device=dev)
    y = torch.randint(0, 1000, (B,), device=dev)
    runs = {}
    for rate in (0.0, 0.1):
        torch.manual_seed(1234)
        net = build_vil("vil_small", attn_drop_rate=rate).to(dev).train()
        opt = torch.optim.AdamW(net.parameters(), lr=5e-4, weight_decay=0.05, fused=True)

        def step(net=net, opt=opt):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = torch.nn.functional.cross_entropy(net(x), y)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()

        for _ in range(warmup):
            step()
        runs[rate] = step
    ips = {rate: [] for rate in runs}
    for _ in range(rounds):
        for rate, step in runs.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            ips[rate].append(B * steps / (e0.elapsed_time(e1) * 1e-3))
    for rate, v in ips.items():
        res[f"train_img_s_attn_drop{rate}"] = [round(x, 1) for x in v]
    return res


def main():
    dev = torch.device("cuda")
    out = {"card": card()}
    out.update(operator(dev))
    if "--no-train" not in sys.argv:
        out.update(training(dev))
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
