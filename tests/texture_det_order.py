"""The deterministic texture gradient (dirt_texture_sample_backward_deterministic, DESIGN.md §7.5) restated in numpy:
the terms, their order per texel and the summation tree, float64 adds in the kernels' order, so that the result is
bit-identical to the kernels'."""
import numpy as np

CHUNK = 4096   # terms per chunk
LANES = 32     # lanes of the lattice inside a chunk


def taps(indices, TB, TH, TW, N, mode):
    """taps_of per lookup: (valid, texture tb, r0, c0, r1, c1, fr, fc), in fp32 arithmetic."""
    ir = np.ascontiguousarray(indices[:, 0], np.float32)
    ic = np.ascontiguousarray(indices[:, 1], np.float32)
    valid = np.isfinite(ir) & np.isfinite(ic)
    ir = np.where(valid, ir, np.float32(0))
    ic = np.where(valid, ic, np.float32(0))
    g = np.arange(ir.shape[0], dtype=np.int64)
    tb = g // N if TB > 1 else np.zeros_like(g)
    if mode == 'nearest':
        r0 = np.clip(np.trunc(ir).astype(np.int64), 0, TH - 1)
        c0 = np.clip(np.trunc(ic).astype(np.int64), 0, TW - 1)
        fr = fc = np.zeros_like(ir)
        r1, c1 = r0, c0
    else:
        flr, flc = np.floor(ir), np.floor(ic)
        fr, fc = ir - flr, ic - flc                     # fp32 subtractions
        r0 = np.mod(flr.astype(np.int64), TH)           # sign of the divisor
        c0 = np.mod(flc.astype(np.int64), TW)
        r1, c1 = (r0 + 1) % TH, (c0 + 1) % TW
    z = np.zeros_like(r0)
    return (valid, tb, np.where(valid, r0, z), np.where(valid, c0, z), np.where(valid, r1, z), np.where(valid, c1, z),
            fr, fc)


def ordered_terms(indices, grad_out, TB, TH, TW, N, mode):
    """(texel, terms [n, C] float64) of every term, sorted into the kernels' order: by texel, then corner 00, 01, 10, 11,
    then ascending lookup id."""
    valid, tb, r0, c0, r1, c1, fr, fc = taps(indices, TB, TH, TW, N, mode)
    one = np.float32(1)
    texel, corner, ids, terms = [], [], [], []
    gout = np.asarray(grad_out, np.float32)
    for k in range(4 if mode == 'bilinear' else 1):
        w = (fc if k & 1 else one - fc) * (fr if k & 2 else one - fr)   # fp32 product
        r, c = (r1 if k & 2 else r0), (c1 if k & 1 else c0)
        sel = np.nonzero(valid)[0]
        t = np.where((w[sel] != 0)[:, None], (gout[sel] * w[sel, None]).astype(np.float64), 0.0)
        texel.append(tb[sel] * TH * TW + r[sel] * TW + c[sel])
        corner.append(np.full(sel.shape, k))
        ids.append(sel)
        terms.append(t)
    texel, corner, ids, terms = (np.concatenate(a) for a in (texel, corner, ids, terms))
    order = np.lexsort((ids, corner, texel))
    return texel[order], terms[order]


def tree_sum(texel, terms, K):
    """The per-texel sums of terms [n, C] already in order (texel ascending): chunks of CHUNK terms, lane t of LANES sums
    terms t, t + LANES, ... of its chunk from +0.0, an xor butterfly over the lanes, the chunk sums added in chunk order
    from +0.0, one rounding to fp32.  Returns [K, C] float32."""
    C = terms.shape[1]
    out = np.zeros((K, C), np.float64)
    n = texel.shape[0]
    if n == 0:
        return out.astype(np.float32)
    new_run = np.r_[True, texel[1:] != texel[:-1]]
    run_start = np.maximum.accumulate(np.where(new_run, np.arange(n), 0))
    i = np.arange(n) - run_start
    q, row, lane = i // CHUNK, (i % CHUNK) // LANES, i % LANES
    new_pair = new_run | np.r_[True, q[1:] != q[:-1]]
    pair = np.cumsum(new_pair) - 1
    acc = np.zeros((pair[-1] + 1, LANES, C), np.float64)
    by_row = np.argsort(row, kind='stable')
    bounds = np.searchsorted(row[by_row], np.arange(row.max() + 2))
    for r in range(row.max() + 1):
        s = by_row[bounds[r]:bounds[r + 1]]          # one term per (pair, lane) in a row
        acc[pair[s], lane[s]] = acc[pair[s], lane[s]] + terms[s]
    perm = np.arange(LANES)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, perm ^ o]
    partial = acc[:, 0]
    first = np.nonzero(new_pair)[0]
    pair_texel, pair_q = texel[first], q[first]
    for c in range(pair_q.max() + 1):
        s = pair_q == c
        out[pair_texel[s]] = out[pair_texel[s]] + partial[s]
    return out.astype(np.float32)


def grad_texture(texture_shape, indices, grad_out, mode='bilinear'):
    """texture_shape (TB, TH, TW, C), indices [B, N, 2], grad_out [B, N, C] (numpy) -> grad_texture [TB, TH, TW, C]."""
    TB, TH, TW, C = texture_shape
    B, N = indices.shape[0], indices.shape[1]
    texel, terms = ordered_terms(indices.reshape(B * N, 2), grad_out.reshape(B * N, C), TB, TH, TW, N, mode)
    return tree_sum(texel, terms, TB * TH * TW).reshape(TB, TH, TW, C)
