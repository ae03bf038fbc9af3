"""A float64 restatement of the shadow-map lookup (DESIGN.md §7.15) that takes every discrete decision exactly as the
CUDA kernels take it, so that continuous random depths, receivers on rendered surfaces and large maps can be compared
at the 1e-4 bar with no tie exclusions.

`lookups` and `_depth_steps` restate the kernels' fp32 decisions in numpy:
  - the clip coordinates come from the kernels' FMA chain h_c = fma(p2, M[2,c], fma(p1, M[1,c], fma(p0, M[0,c],
    M[3,c]))); a product of two fp32 values is exact in float64, so each fma is one float64 add, bit for bit;
  - x/w, X, Yd, floor and the fractions in float64, the fractions then rounded to fp32;
  - zb = f32(f32(z) - bias), d = f32(zb - depth), and step = d > 0 for softness 0.
`reference` evaluates the value and its gradients in float64 torch autograd with those decisions fixed: the fp32
fractions and, for softness > 0, the fp32 d in the sigmoid (each as a float64 value with its float64 derivative), and
the derivatives with respect to the fractions formed as the kernels form them.
`deterministic_map_gradient` restates the deterministic backward's map gradient for softness 0 bit for bit: each
texel's float64 sum, in the documented order, of the default kernel's fp32 terms, rounded once to fp32."""
import math

import numpy as np
import torch

f32 = np.float32


def _flat(positions, matrix, smap):
    """fp32-rounded float64 arrays: positions [B, N, 3], matrices [nm, 4, 4], maps [nm, SH, SW, 2] (nm = B per item,
    1 shared), and the leading shape."""
    p = np.asarray(positions, np.float32).astype(np.float64)
    M = np.asarray(matrix, np.float32).astype(np.float64)
    m = np.asarray(smap, np.float32).astype(np.float64)
    lead, N = p.shape[:-2], p.shape[-2]
    B = math.prod(lead)
    per_item = M.ndim > 2
    nm = B if per_item else 1
    return p.reshape(B, N, 3), M.reshape(nm, 4, 4), m.reshape((nm,) + m.shape[-3:]), lead


def lookups(p, M, SH, SW):
    """The kernels' per-point decisions for p [B, N, 3] and M [nm, 4, 4] (float64 holding fp32 values): a dict of
    valid [B, N]; r0, c0 (int64, 0 where invalid); fr, fc (fp32, 0 where invalid); h [B, N, 4] (fp32)."""
    Mr = M[:, None]   # [nm, 1, 4, 4], broadcast over the points
    with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
        h = p[..., 2:3] * Mr[..., 2, :] + (p[..., 1:2] * Mr[..., 1, :] + (p[..., 0:1] * Mr[..., 0, :] + Mr[..., 3, :]))
        valid = np.isfinite(h).all(-1) & (h[..., 3] > 0)
        xn, yn = h[..., 0] / h[..., 3], h[..., 1] / h[..., 3]
        X, Yd = (xn + 1.0) * (0.5 * SW), (1.0 - yn) * (0.5 * SH)
        valid &= (X >= 0) & (X < SW) & (Yd >= 0) & (Yd < SH)
    u, v = np.where(valid, X - 0.5, 0.), np.where(valid, Yd - 0.5, 0.)
    cf, rf = np.floor(u), np.floor(v)
    return dict(valid=valid, c0=cf.astype(np.int64), r0=rf.astype(np.int64), fc=(u - cf).astype(np.float32),
                fr=(v - rf).astype(np.float32), h=h.astype(np.float32))


def _tap(look, R, i, k, SH, SW):
    """The clamped row and column of tap (i, k) of every point."""
    return np.clip(look['r0'] - R + i, 0, SH - 1), np.clip(look['c0'] - R + k, 0, SW - 1)


def _item_maps(B, nm):
    return np.arange(B)[:, None] if nm > 1 else np.zeros((B, 1), np.int64)


def _depth_steps(look, m, R, i, k, bias):
    """d = f32(f32(f32(z) - bias) - depth) of tap (i, k) (0 where invalid) and the texel index into m [nm, SH, SW]."""
    nm, SH, SW = m.shape[:3]
    B = look['valid'].shape[0]
    r, c = _tap(look, R, i, k, SH, SW)
    mi = _item_maps(B, nm)
    depth = m[mi, r, c, 1].astype(np.float32)
    with np.errstate(invalid='ignore', over='ignore'):
        zb = look['h'][..., 2] - f32(bias)
        d = (zb - depth).astype(np.float32)
    return np.where(look['valid'], d, f32(0)), (mi, r, c)


def tap_weight(R, i, f):
    return 1. - f if i == 0 else (f if i == 2 * R + 1 else torch.ones_like(f))


def reference(positions, matrix, smap, R, softness, bias, grad_out=None, want=(True, True, True), device='cpu'):
    """The visibility [*, N, 1] and, with grad_out [*, N, 1], the gradients (positions, light matrix, map) of the wanted
    inputs (None for the others), as float64 numpy arrays in the inputs' shapes.  positions [*, N, 3] with matrix
    [*, 4, 4] and smap [*, SH, SW, 2] (per item) or [4, 4] and [SH, SW, 2] (shared); any float arrays, rounded to fp32
    first.  `device` is where the float64 evaluation runs."""
    p, M, m, lead = _flat(positions, matrix, smap)
    B, N = p.shape[:2]
    nm, SH, SW = m.shape[:3]
    look = lookups(p, M, SH, SW)
    dev = torch.device(device)

    def t(x, dtype=torch.float64):
        return torch.as_tensor(np.ascontiguousarray(x)).to(device=dev, dtype=dtype)

    tp, tM, tm = (t(x).requires_grad_(w) for x, w in zip((p, M, m), want))
    valid = t(look['valid'], torch.bool)
    ps = torch.where(valid[..., None], tp, 0.)
    h = torch.matmul(torch.cat([ps, torch.ones_like(ps[..., :1])], -1), tM)
    h = torch.where(valid[..., None], h, t(np.array([0., 0., 0., 1.])))
    x, y, z, w = h.unbind(-1)
    fc = (x / w + 1.) * (0.5 * SW) - 0.5 - t(look['c0'])
    fr = (1. - y / w) * (0.5 * SH) - 0.5 - t(look['r0'])
    fc = fc + (t(look['fc']) - fc).detach()   # the kernels' fp32 fraction, with its float64 derivative
    fr = fr + (t(look['fr']) - fr).detach()
    flat = tm.reshape(nm, SH * SW, 2)
    T = 2 * R + 2
    s = [[None] * T for _ in range(T)]
    for i in range(T):
        for k in range(T):
            d32, (mi, r, c) = _depth_steps(look, m, R, i, k, bias)
            tap = flat[t(mi, torch.long), t(r * SW + c, torch.long)]
            if softness > 0:
                d = z - tap[..., 1] - bias
                d = d + (t(d32) - d).detach()
                step = torch.sigmoid(d / softness)
            else:
                step = t(d32 > 0)
            s[i][k] = 1. - tap[..., 0] * step
    # V = sum_i a_i sum_k b_k s_ik is bilinear in the 1-D weights: its fraction derivatives are written out as the
    # kernels form them, row_last - row_0 and sum_i a_i (s_i,last - s_i,0), so that they cancel exactly where the
    # clamped taps repeat one texel (a one-row or one-column map), as the kernels' do
    a = [tap_weight(R, i, fr.detach()) for i in range(T)]
    b = [tap_weight(R, k, fc.detach()) for k in range(T)]
    rows = [sum(b[k] * s[i][k] for k in range(T)) for i in range(T)]
    vis = sum(a[i] * rows[i] for i in range(T))
    d_fr = rows[T - 1] - rows[0]
    d_fc = sum(a[i] * (s[i][T - 1] - s[i][0]) for i in range(T))
    vis = vis + (fr - fr.detach()) * d_fr.detach() + (fc - fc.detach()) * d_fc.detach()
    vis = torch.where(valid, vis / (2 * R + 1) ** 2, 1.)
    out = vis.detach().cpu().numpy().reshape(lead + (N, 1))
    if grad_out is None:
        return out
    (vis * t(np.asarray(grad_out, np.float32).reshape(B, N))).sum().backward()
    shapes = (np.shape(positions), np.shape(matrix), np.shape(smap))
    grads = tuple(x.grad.cpu().numpy().reshape(s) if w else None for x, w, s in zip((tp, tM, tm), want, shapes))
    return out, grads


def sequential_sums(segment, values):
    """Per segment of `segment` (sorted, non-decreasing), the float64 sum from +0.0 of its `values` in their order,
    one addition at a time (np.sum is pairwise); returns (segment ids, sums)."""
    starts = np.flatnonzero(np.r_[True, segment[1:] != segment[:-1]])
    lens = np.diff(np.r_[starts, len(segment)])
    acc = np.zeros(len(starts))
    long_runs = lens > 1024
    for s in np.flatnonzero(long_runs):   # np.cumsum adds one value at a time
        acc[s] = np.cumsum(values[starts[s]:starts[s] + lens[s]])[-1]
    short = np.flatnonzero(~long_runs)
    for j in range(int(lens[short].max()) if short.size else 0):
        sel = short[lens[short] > j]
        acc[sel] = acc[sel] + values[starts[sel] + j]
    return segment[starts], acc


def deterministic_map_gradient(positions, matrix, smap, R, bias, grad_out):
    """The map gradient of dirt_shadow_backward_deterministic at softness 0, bit for bit: per texel, the float64 sum
    from +0.0 of the fp32 terms g/K * -(w step) in the order tap row i, base row r0, tap column k, base column c0,
    point id b N + n, rounded once to fp32 (DESIGN.md §7.15).  The depth channel is 0.  Shapes as `reference`."""
    p, M, m, _ = _flat(positions, matrix, smap)
    B, N = p.shape[:2]
    nm, SH, SW = m.shape[:3]
    look = lookups(p, M, SH, SW)
    inv_k = f32(1) / f32((2 * R + 1) ** 2)
    gk = (np.asarray(grad_out, np.float32).reshape(B, N) * inv_k).astype(np.float32)
    ids = np.arange(B * N).reshape(B, N)
    ok = look['valid']
    fr, fc = look['fr'], look['fc']
    keys, terms = [], []
    T = 2 * R + 2
    for i in range(T):
        wr = f32(1) - fr if i == 0 else (fr if i == T - 1 else np.ones_like(fr))
        for k in range(T):
            wc = f32(1) - fc if k == 0 else (fc if k == T - 1 else np.ones_like(fc))
            d32, (mi, r, c) = _depth_steps(look, m, R, i, k, bias)
            st = (d32 > 0).astype(np.float32)
            term = (gk * -((wr * wc).astype(np.float32) * st)).astype(np.float32)
            texel = (np.broadcast_to(mi, (B, N)) * SH + r) * SW + c
            keys.append(np.stack([texel[ok], np.full(ok.sum(), i), look['r0'][ok], np.full(ok.sum(), k),
                                  look['c0'][ok], ids[ok]]))
            terms.append(term[ok])
    keys, terms = np.concatenate(keys, 1), np.concatenate(terms)
    order = np.lexsort(keys[::-1])
    texels, sums = sequential_sums(keys[0][order], terms[order].astype(np.float64))
    out = np.zeros((nm * SH * SW, 2), np.float32)
    out[texels, 0] = sums.astype(np.float32)
    return out.reshape(np.shape(smap))


def sort_passes(B, per_item, SH, SW):
    """The radix-sort passes of the deterministic backward: one per 8 bits of its key count (sort.cuh)."""
    keys = (B if per_item else 1) * (SH + 1) * (SW + 1)
    return (int(keys).bit_length() + 7) // 8
