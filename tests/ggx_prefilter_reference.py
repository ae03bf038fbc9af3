"""Rows and columns of tests/cubemap_ggx_restatement.py's GGX prefilter at any S: the dense `weights` matrix is
[6 S_k^2, 6 S_s^2] float64, which stops at S = 64, while these slices cost one pass over a level per row or column.

    rows(k, S, idx)       output texels idx of level k against every texel of source level s = min(k, s*)
    columns(k, S, jdx)    source texels jdx of level s against every output texel of level k (the pairs are the same:
                          the fp32 cosine is symmetric in its two directions)
    adjoint_rows(...)     the prefilter's adjoint at source texels, on given level gradients and normalisers

Support and weights are the restatement's: pair (r, l) is in the sum iff the fp32 cosine c = pair_cos(r, l) has c > 0
and c >= c_k, and w = D(c) c Omega_l in float64 from that fp32 c.  The support is decided first by the float64 cosine of
the fp32 directions (products exact, two roundings), which differs from the fp32 one by a few 1e-8; only pairs whose
float64 cosine lies within BAND of 0 or of c_k are decided by the exact fp32 cosine.  For speed, each row scans only the
8 x 8 texel blocks that a float64 bounding-cone test (exact, with margin 2 BAND) cannot rule out; nothing is culled that
could be in the support, and nothing here shares the kernels' fp32 cones.

Texels are flat indices f * S_k^2 + r * S_k + c of a level's [6, S_k, S_k] faces."""
import math

import numpy as np
import scipy.sparse
import torch

import cubemap_ggx_restatement as ibl

BAND = 1e-4   # the float64 cosine decides pairs farther than this from 0 and from c_k


def level_source(k, S):
    """(s, alpha2 float64, c_k fp32) of output level k >= 1."""
    alpha2, _, ck = ibl.lobe(k, ibl.level_count(S))
    return min(k, ibl.source_cap(S)), alpha2, ck


def decide(c64, ck):
    """The float64 pre-decision: (in_support, undecided) masks; the exact fp32 cosine settles the undecided pairs."""
    ck = float(ck)
    undecided = (np.abs(c64) < BAND) | (np.abs(c64 - ck) < BAND)
    return ~undecided & (c64 > 0) & (c64 >= ck), undecided


_BLOCKS = {}


def _blocks(Sb):
    """The texels of a level of Sb per edge in 8 x 8 blocks: (texel order by block, block starts, axes [nb, 3], half-angles
    [nb]) in float64, each half-angle the largest angle from the axis to one of the block's texel directions."""
    if Sb not in _BLOCKS:
        d = ibl.texel_table(Sb)[0].reshape(-1, 3).astype(np.float64)
        x = np.arange(d.shape[0])
        nb = (Sb + 7) // 8
        bid = ((x // (Sb * Sb)) * nb + x // Sb % Sb // 8) * nb + x % Sb // 8
        order = np.argsort(bid, kind='stable')
        starts = np.searchsorted(bid[order], np.arange(6 * nb * nb + 1))
        axis = np.add.reduceat(d[order], starts[:-1])
        axis /= np.linalg.norm(axis, axis=-1, keepdims=True)
        cos = np.minimum.reduceat((d[order] * np.repeat(axis, np.diff(starts), 0)).sum(-1), starts[:-1])
        _BLOCKS[Sb] = (order, starts, axis, np.arccos(np.clip(cos, -1, 1)) + 1e-9)
    return _BLOCKS[Sb]


def _support(a, b, Sb, ck):
    """Directions a [n, 3] against b, the texel table of a level of Sb per edge, fp32: (indptr, indices, fp32 c) of each
    row's support, indices sorted.  Only the blocks of b that can hold a pair with float64 cosine at least
    max(c_k, 0) - 2 BAND are scanned (the angle from the row to the block's axis, less the block's half-angle, is a
    lower bound of the angle to any of its texels)."""
    b = b.reshape(-1, 3)
    order, starts, axis, theta = _blocks(Sb)
    reach = np.arccos(max(float(ck), 0.0) - 2 * BAND)
    indptr, indices, cos = [0], [], []
    for i in range(a.shape[0]):
        r64 = a[i].astype(np.float64)
        near = np.arccos(np.clip(axis @ r64, -1, 1)) - theta <= reach
        cand = np.sort(np.concatenate([order[s:e] for s, e in zip(starts[:-1][near], starts[1:][near])]))
        sure, undecided = decide(b[cand].astype(np.float64) @ r64, ck)
        cand, sure = cand[sure | undecided], sure[sure | undecided]
        c = ibl.pair_cos(a[i][None], b[cand])[0]
        keep = sure | ((c > 0) & (c >= ck))
        indices.append(cand[keep])
        cos.append(c[keep])
        indptr.append(indptr[-1] + int(keep.sum()))
    return np.asarray(indptr), np.concatenate(indices), np.concatenate(cos)


def _w(c, alpha2, omega):
    """D(c) c Omega in float64 of the fp32 cosine c, as cubemap_ggx_restatement._weights writes it."""
    c = c.astype(np.float64)
    kk = alpha2 + (1.0 - c) * (1.0 - alpha2) / 2.0
    return alpha2 / (math.pi * kk * kk) * c * omega


def rows(k, S, idx):
    """Output texels idx of level k: (w, W) with w scipy.sparse.csr_matrix [len(idx), 6 S_s^2] float64 whose stored
    entries are exactly the support, and W [len(idx)] the row sums."""
    s, alpha2, ck = level_source(k, S)
    rd, _ = ibl.texel_table(S >> k)
    ld, lw = ibl.texel_table(S >> s)
    lw = lw.reshape(-1).astype(np.float64)
    indptr, indices, c = _support(rd.reshape(-1, 3)[np.asarray(idx)], ld, S >> s, ck)
    w = scipy.sparse.csr_matrix((_w(c, alpha2, lw[indices]), indices, indptr), shape=(len(idx), lw.size))
    return w, np.asarray(w.sum(1)).reshape(-1)


def columns(k, S, jdx):
    """Source texels jdx of level s = min(k, s*) against the output texels of level k: the transposed slice of the
    same pairs, scipy.sparse.csr_matrix [len(jdx), 6 S_k^2] float64, w = D(c) c Omega_j."""
    s, alpha2, ck = level_source(k, S)
    rd, _ = ibl.texel_table(S >> k)
    ld, lw = ibl.texel_table(S >> s)
    jdx = np.asarray(jdx)
    indptr, indices, c = _support(ld.reshape(-1, 3)[jdx], rd, S >> k, ck)
    omega = np.repeat(lw.reshape(-1)[jdx].astype(np.float64), np.diff(indptr))
    return scipy.sparse.csr_matrix((_w(c, alpha2, omega), indices, indptr), shape=(len(jdx), rd[..., 0].size))


def adjoint_rows(S, s, jdx, grads, W):
    """The prefilter's adjoint at texels jdx of source level s >= 1: Omega_j sum_k sum_r D_k(c) c g_k(r) / W_k(r) over
    the output levels k >= 1 with min(k, s*) = s.  grads[k] [6 S_k^2, C] and W[k] [6 S_k^2] (the GPU's own
    normalisers, as the adjoint kernel reads them), float64 -> [len(jdx), C]."""
    out = None
    for k in range(1, ibl.level_count(S)):
        if level_source(k, S)[0] != s:
            continue
        term = columns(k, S, jdx) @ (np.asarray(grads[k], np.float64) / np.asarray(W[k], np.float64)[:, None])
        out = term if out is None else out + term
    return out


_CENTRES = {}


def _edge_centres(Sk):
    """Per texel index i of an Sk-texel edge, an fp32 x in the face plane with (((x / 1 + 1) * 0.5) * Sk - 0.5) + 1 =
    i + 1 in fp32, each operation rounded as cubemap_restatement's lookup rounds it: among the 32 fp32 values on each
    side of (2i + 1) / Sk - 1, the nearest.  At a power-of-two Sk that value itself is exact.  At other Sk, near
    x = -1 the values (x + 1) / 2 are spaced more coarsely than s must be placed for s * Sk to round to i + 0.5, so
    some low indices have none (NaN): 2 of 15, 3 of 30, 8 of 60, 18 of 120, 40 of 240."""
    if Sk not in _CENTRES:
        i = np.arange(Sk)
        x0 = ((2.0 * i + 1.0) / Sk - 1.0).astype(np.float32)
        found = np.full(Sk, np.nan, np.float32)
        for sign in (1, -1):
            x = x0.copy()
            for step in range(32):
                t = torch.from_numpy(x)
                p = (((t / torch.ones_like(t) + 1.) * 0.5) * Sk - 0.5) + 1.
                hit = np.isnan(found) & (p.numpy() == i + 1)
                found[hit] = x[hit]
                x = np.nextafter(x, np.float32(sign * np.inf))
        _CENTRES[Sk] = found
    return _CENTRES[Sk]


def has_exact_centre(k, S, texels):
    """bool [n]: whether exact_centre_directions has a direction for each of level k's flat texel indices."""
    Sk = S >> k
    texels = np.asarray(texels)
    ok = ~np.isnan(_edge_centres(Sk))
    return ok[texels // Sk % Sk] & ok[texels % Sk]


def exact_centre_directions(k, S, texels):
    """fp32 directions [n, 3] whose padded (row, col) at level k (S_k = S >> k) under cubemap_restatement.face_coords
    are exactly texel (f, r, c)'s (r + 1, c + 1): a bilinear lookup there reads that texel with weight 1 and its
    neighbours with weight 0.  texels: flat indices of level k; NaN rows where has_exact_centre is False."""
    Sk = S >> k
    texels = np.asarray(texels)
    f, r, c = texels // (Sk * Sk), texels // Sk % Sk, texels % Sk
    x = _edge_centres(Sk)
    out = np.zeros((texels.size, 3), np.float32)
    for face in range(6):
        m = f == face
        out[m] = np.stack([np.asarray(v, np.float32) * np.ones(m.sum(), np.float32)
                           for v in ibl._face_point(face, x[c[m]], x[r[m]])], -1)
    return out
