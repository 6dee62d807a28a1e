"""fp64 CPU restatements of per-image token grids in a padded batch (vil_attn_fwd_sized_sm100, include/vil_attn.h), for
the tests.

Image b of a batch padded to nx x ny tokens has its own grid of h_b x w_b tokens at the top left: padded-grid local token
r * ny + c is real iff r < h_b and c < w_b.

* `sized_attention` crops each image out of the padded tensors, runs `oracle.vil_oracle.dense_attention` (or
  `tests.dilated_oracle.dilated_attention` for d > 1) on the crop with the global tokens, and scatters the rows back:
  zeros at off-image rows of o, -inf at off-image rows of lse.
* `sized_bruteforce` never crops: it lists, for every real local query of the padded grid, the keys the sliding-chunk
  rules give it (chunk offsets of `mode`, the crop's chunk grid, its cyclic wrap and pad cut, its residue sub-grid under
  dilation), as padded-grid key tokens, phantom zero keys or global keys, and runs one dense softmax per query.
"""
from __future__ import annotations

import math

import torch

from oracle.vil_oracle import dense_attention, mode_offsets
from tests.dilated_oracle import dilated_attention


def image_index(nx: int, ny: int, h: int, w: int) -> torch.Tensor:
    """padded-grid local tokens of an h x w image, row-major over the crop"""
    return (torch.arange(h)[:, None] * ny + torch.arange(w)[None, :]).reshape(-1)


def sized_attention(q, k, v, qg, kg, vg, table, g2l, g2g, *, nx, ny, w, sizes, exact=0, mode=0, scale=1.0, d=1):
    """(o, og, lse, lse_g) of a sized call: dense_attention's signature plus `sizes`, B (h, w) pairs"""
    B, H, Nloc, D = q.shape
    g = k.shape[2] - Nloc
    o = torch.zeros_like(q)
    lse = torch.full(q.shape[:3], -math.inf, dtype=q.dtype)
    og = torch.zeros_like(qg) if g else None
    lse_g = torch.zeros(B, H, g, dtype=q.dtype) if g else None
    for b, (h, wb) in enumerate(sizes):
        idx = image_index(nx, ny, h, wb)
        crop = lambda t: torch.cat([t[b:b + 1, :, :g], t[b:b + 1, :, g + idx]], dim=2)
        ob, ogb, lb, lgb = dilated_attention(q[b:b + 1, :, idx], crop(k), crop(v), qg[b:b + 1] if g else None,
                                             crop(kg) if g else None, crop(vg) if g else None, table, g2l, g2g,
                                             nx=h, ny=wb, w=w, exact=exact, mode=mode, scale=scale, d=d)
        o[b, :, idx] = ob[0]
        lse[b, :, idx] = lb[0]
        if g:
            og[b], lse_g[b] = ogb[0], lgb[0]
    return o, og, lse, lse_g


def _query_columns(nx, ny, h, wb, w, exact, mode, d):
    """{padded local query token: [(key, du, dv)]}: key = padded key token (>= 0, local), -1 for a phantom zero key; (du, dv)
    the bias-table offset of the pair (query minus key position, chunk-relative, in sub-grid units)"""
    cols = {}
    for r in range(h):
        for c in range(wb):
            a, bb = r % d, c % d
            sn, sm = -(-(h - a) // d), -(-(wb - bb) // d)          # the residue's sub-grid of the crop
            mx, my = -(-sn // w), -(-sm // w)
            padx, pady = mx * w - sn, my * w - sm
            rr, cc = r // d, c // d                                  # sub-grid position
            R, C, qr, qc = rr // w, cc // w, rr % w, cc % w
            lst = []
            if exact == 1:
                for kr in range(sn):
                    for kc in range(sm):
                        if abs(rr - kr) <= w and abs(cc - kc) <= w:
                            lst.append(((a + d * kr) * ny + bb + d * kc, rr - kr, cc - kc))
            else:
                for dR, dC in mode_offsets(mode):
                    KR, KC = R + dR, C + dC
                    if exact == 0 and not (0 <= KR < mx and 0 <= KC < my):
                        continue
                    cut_r, cut_c = KR == mx - 1, KC == my - 1          # before the wrap
                    KR, KC = KR % mx, KC % my
                    for kr in range(w):
                        for kc in range(w):
                            ar, ac = KR * w + kr, KC * w + kc
                            real = ar < sn and ac < sm
                            if exact == 0:
                                take = real
                            else:
                                take = not ((cut_r and kr >= w - padx) or (cut_c and kc >= w - pady))
                            if take:
                                key = (a + d * ar) * ny + bb + d * ac if real else -1
                                lst.append((key, qr - (dR * w + kr), qc - (dC * w + kc)))
            cols[r * ny + c] = lst
    return cols


def sized_bruteforce(q, k, v, table, g2l, *, nx, ny, w, sizes, exact=0, mode=0, scale=1.0, d=1):
    """(o, lse) of the local query rows, zeros / -inf off the images (see the module docstring)"""
    B, H, Nloc, D = q.shape
    g = k.shape[2] - Nloc
    dt = torch.float64
    o = torch.zeros(B, H, Nloc, D, dtype=dt)
    lse = torch.full((B, H, Nloc), -math.inf, dtype=dt)
    tw = 4 * w - 1
    for b, (h, wb) in enumerate(sizes):
        for i, lst in _query_columns(nx, ny, h, wb, w, exact, mode, d).items():
            keys = torch.tensor([e[0] for e in lst], dtype=torch.long)
            real = keys >= 0
            kk = torch.zeros(H, len(lst), D, dtype=dt)
            vv = torch.zeros(H, len(lst), D, dtype=dt)
            kk[:, real] = k[b, :, g + keys[real]].to(dt)
            vv[:, real] = v[b, :, g + keys[real]].to(dt)
            s = scale * torch.einsum("hd,hjd->hj", q[b, :, i].to(dt), kk)
            if table is not None:
                ent = torch.tensor([(du + 2 * w - 1) * tw + dv + 2 * w - 1 for _, du, dv in lst], dtype=torch.long)
                s = s + table.to(dt)[ent].T
            if g:
                sg = scale * torch.einsum("hd,htd->ht", q[b, :, i].to(dt), k[b, :, :g].to(dt))
                if g2l is not None:
                    sg = sg + g2l[1].to(dt)
                s = torch.cat([sg, s], dim=1)
                vv = torch.cat([v[b, :, :g].to(dt), vv], dim=1)
            lse[b, :, i] = torch.logsumexp(s, dim=1)
            o[b, :, i] = torch.einsum("hj,hjd->hd", torch.softmax(s, dim=1), vv)
    return o, lse


def sized_global_bruteforce(qg, kg, vg, g2l, g2g, *, nx, ny, sizes, scale=1.0):
    """(og, lse_g) of the global query rows: a masked dense softmax over the padded grid's N keys"""
    B, H, g, D = qg.shape
    dt = torch.float64
    s = scale * torch.einsum("bhad,bhjd->bhaj", qg.to(dt), kg.to(dt))
    if g2l is not None:
        s = s + torch.cat([g2g.to(dt), g2l[0].to(dt)[..., None].expand(H, g, nx * ny)], dim=-1)[None]
    on = torch.zeros(B, nx * ny, dtype=torch.bool)
    for b, (h, wb) in enumerate(sizes):
        on[b, image_index(nx, ny, h, wb)] = True
    keep = torch.cat([torch.ones(B, g, dtype=torch.bool), on], dim=1)[:, None, None, :]
    s = s.masked_fill(~keep, -math.inf)
    vz = torch.where(keep[:, :, 0, :, None], vg.to(dt), 0.)
    return torch.einsum("bhaj,bhjd->bhad", torch.softmax(s, dim=-1), vz), torch.logsumexp(s, dim=-1)
