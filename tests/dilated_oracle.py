"""fp64 CPU restatements of dilated sliding-chunk attention (VIL_FLAG_DILATED, include/vil_attn.h), for the tests.

Dilation d splits the nx x ny local tokens into d^2 residue sub-grids: residue (a, b) holds image positions
(a + d r', b + d c'), a sub-grid of ceil((nx - a) / d) x ceil((ny - b) / d) tokens.  A local query attends to the global
tokens and, exactly as the undilated operator on its own sub-grid, to the keys of its sub-grid; global queries attend to
all N tokens as at d = 1.

* `dilated_attention` gathers each sub-grid, runs `oracle.vil_oracle.dense_attention` on it with the shared global
  tokens, and scatters the local rows back; the global rows come from the d = 1 call.
* `dilated_bruteforce` builds one (query, key) weight matrix over the whole image instead: the exact window
  |dr|, |dc| <= w d with dr = dc = 0 (mod d) written out for exact = 1, and for exact 0 / -1 the oracle's visit weights
  (the reference's mask builders) evaluated in sub-grid coordinates, every sub-grid's padding keys as columns of their
  own.  One dense joint softmax then gives o and lse.
"""
from __future__ import annotations

import math

import torch

from oracle.vil_oracle import dense_attention, visit_weights, _pad_keys


def residues(nx: int, ny: int, d: int):
    """(a, b, nx_a, ny_b, local token indices (row-major over the sub-grid)) of every non-empty residue sub-grid"""
    out = []
    for a in range(d):
        for b in range(d):
            if a >= nx or b >= ny:
                continue
            rows = torch.arange(a, nx, d)
            cols = torch.arange(b, ny, d)
            idx = (rows[:, None] * ny + cols[None, :]).reshape(-1)
            out.append((a, b, len(rows), len(cols), idx))
    return out


def dilated_attention(q, k, v, qg, kg, vg, table, g2l, g2g, *, nx, ny, w, exact=0, mode=0, scale=1.0, d=1):
    """Same signature and results as dense_attention, with dilation d"""
    o1, og, lse1, lse_g = dense_attention(q, k, v, qg, kg, vg, table, g2l, g2g, nx=nx, ny=ny, w=w, exact=exact,
                                          mode=mode, scale=scale)
    if d == 1:
        return o1, og, lse1, lse_g
    B, H, Nloc, D = q.shape
    g = k.shape[2] - Nloc
    o = torch.zeros_like(o1)
    lse = torch.zeros_like(lse1)
    for a, b, na, nb, idx in residues(nx, ny, d):
        ks = torch.cat([k[:, :, :g], k[:, :, g + idx]], dim=2)
        vs = torch.cat([v[:, :, :g], v[:, :, g + idx]], dim=2)
        # the global rows of the sub-grid call are not used: give it the sub-grid's own tokens as global keys
        kgs = torch.cat([kg[:, :, :g], kg[:, :, g + idx]], dim=2) if g > 0 else None
        vgs = torch.cat([vg[:, :, :g], vg[:, :, g + idx]], dim=2) if g > 0 else None
        os_, _, ls, _ = dense_attention(q[:, :, idx], ks, vs, qg, kgs, vgs, table, g2l, g2g, nx=na, ny=nb, w=w,
                                        exact=exact, mode=mode, scale=scale)
        o[:, :, idx] = os_
        lse[:, :, idx] = ls
    return o, og, lse, lse_g


def dilated_bruteforce(q, k, v, table, g2l, *, nx, ny, w, exact=0, mode=0, scale=1.0, d=1):
    """(o, lse) of the local query rows from one image-wide weight matrix (see the module docstring)"""
    B, H, Nloc, D = q.shape
    g = k.shape[2] - Nloc
    dt = torch.float64
    q, k, v = q.to(dt), k.to(dt), v.to(dt)
    tab = table.to(dt) if table is not None else None
    if exact == 1:
        r = torch.arange(Nloc) // ny
        c = torch.arange(Nloc) % ny
        dr = r[:, None] - r[None, :]
        dc = c[:, None] - c[None, :]
        ok = (dr % d == 0) & (dc % d == 0) & (dr.abs() <= w * d) & (dc.abs() <= w * d)
        logw = torch.where(ok, torch.zeros((), dtype=dt), torch.full((), -math.inf, dtype=dt)).expand(H, Nloc, Nloc)
        if tab is not None:                      # offsets in sub-grid units
            u = torch.where(ok, dr // d, 0) + 2 * w - 1
            t = torch.where(ok, dc // d, 0) + 2 * w - 1
            logw = logw + tab[(u * (4 * w - 1) + t).reshape(-1)].reshape(Nloc, Nloc, H).permute(2, 0, 1)
        kl, vl = k[:, :, g:], v[:, :, g:]
    else:
        blocks, kls, vls = [], [], []
        for a, b, na, nb, idx in residues(nx, ny, d):
            E = visit_weights(na, nb, w, exact, mode, tab, H, dtype=dt)            # (H, na*nb, padded sub-grid keys)
            full = torch.zeros(H, Nloc, E.shape[-1], dtype=dt)
            full[:, idx] = E
            blocks.append(full)
            kls.append(_pad_keys(k[:, :, g + idx], na, nb, w))
            vls.append(_pad_keys(v[:, :, g + idx], na, nb, w))
        Ew = torch.cat(blocks, dim=-1)
        logw = torch.where(Ew > 0, torch.log(Ew.clamp_min(1e-300)), torch.full_like(Ew, -math.inf))
        kl, vl = torch.cat(kls, dim=2), torch.cat(vls, dim=2)
    s = scale * torch.einsum("bhid,bhjd->bhij", q, kl) + logw[None]
    if g > 0:
        sgl = scale * torch.einsum("bhid,bhtd->bhit", q, k[:, :, :g])
        if g2l is not None:
            sgl = sgl + g2l[1].to(dt)[None, :, None, :]
        s = torch.cat([sgl, s], dim=-1)
    lse = torch.logsumexp(s, dim=-1)
    p = torch.exp(s - lse[..., None])
    o = torch.einsum("bhij,bhjd->bhid", p[..., g:], vl)
    if g > 0:
        o = o + torch.einsum("bhit,bhtd->bhid", p[..., :g], v[:, :, :g])
    return o, lse
