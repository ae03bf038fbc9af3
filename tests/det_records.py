"""A numpy restatement of the rasteriser's deterministic backward pass (csrc/deterministic.cu, DESIGN.md section 7.4),
term by term, and a reader for the scratch it leaves behind.

From the visibility of a scene (face ids and G-buffer, bit-identical between the oracle and the GPU), its vertices,
pixels and grad_pixels, `restate` forms, per channel group:
    codes       the one-byte dilation code of every pixel (include/dirt_b200.h): bits 0-1 none / own face / first /
                second neighbour, bit 2 the preferred step runs along the row; on interior pixels only (an edge pixel with
                a face is 1)
    records     the fp32 (dL/dx, dL/dy) of every pixel with a code, (+0, +0) elsewhere
    terms       the nine fp32 position terms a coded pixel gives its receiving face and the 3*N0 colour terms a covered
                pixel gives its own face, as sweep_face forms them
The fp32 operation order is the SASS of deterministic.cu (nvcc contracts by default; `cuobjdump -sass` of the sm_90a
build): Scharr sums as grad_pixel.cuh::scharr_comp; dL/dx = fma(gp2, sx2, fma(gp1, sx1, fma(gp0, sx0, +0))), the same
for dL/dy; clip_x = fma(b2, x2, fma(b1, x1, fma(b0, x0, +0))), the same for clip_y; inv_w = 1/w correctly rounded;
dxv_dxc = (W/2) inv_w; dxv_dwc = -((clip_x dxv_dxc) inv_w); ax = r.x b_k; the terms ax dxv_dxc, ay dyv_dyc and
fma(ay, dyv_dwc, ax dxv_dwc); colour terms gp b_k.

`face_partials` and `vertex_sums` then restate the documented float64 summation order: thread t of T (32 for a box of
at most DET_WARP_BOX pixels, else 256) sums the pixels t, t + T, ... of the face's box in raster order; the xor butterfly
joins the lanes of a warp (and, for a CTA, warps 0..7 in order); position partials add up over the groups in group order;
each vertex row sums the partials of its corners in ascending corner id k*F + f, then over the items in order (shared
geometry), and rounds once to fp32.

`term_sums` gives, per output entry, the float64 sum S of its restated terms, the sum of their magnitudes, a magnitude
bound m of the intermediate products each term is made of and the term count n: `bound` turns them into the per-element
fp32 bound of any summation order, gamma_n sum|t| + TERM_SLACK_ULPS u sum m (u = 2^-24).  The slack covers a term formed
in another fp32 operation order than the restatement's (the default tile path's fast reciprocal and factoring, or the
oracle's float64 terms); m is the sum of the magnitudes of the products behind the term, since dL/dx, clip_x and the w
term are sums that can cancel."""
import numpy as np

from cubemap_ggx_restatement import fmaf

DIL_NONE, DIL_OWN, DIL_FIRST, DIL_SECOND, DIL_ALONG_ROW = 0, 1, 2, 3, 4
SHARED_GEOMETRY, SKIP_POSITION, SKIP_COLOUR = 1, 2, 4
DET_WARP_BOX = 2048   # deterministic.cu: larger boxes are swept by one CTA
CTA_THREADS = 256
U = 2.0 ** -24
TERM_SLACK_ULPS = 32


def groups_of(C, groups=None):
    from oracle.oracle import default_groups
    return list(groups) if groups is not None else default_groups(C)


# ---- per-pixel arithmetic ---------------------------------------------------------------------------------------------

def _scharr_comp(a, b, c, d, e, f):
    return fmaf(((a + b) - c) - d, np.float32(0.09375), (e - f) * np.float32(0.3125))


def scharr(pixels, c0, n):
    """sx, sy [B,H,W,3] of the group [c0, c0+n) as grad_pixel.cuh::scharr_global forms them (clamped taps; a 1-wide
    group's components 1 and 2 are the next two pixels in flat order over the whole batch, 0 past its end)."""
    B, H, W, C = pixels.shape
    flat = pixels.reshape(-1, C)
    total = B * H * W
    b, r, c = np.arange(B)[:, None, None], np.arange(H)[None, :, None], np.arange(W)[None, None, :]

    def at(dr, dc):
        lin = (b * H + np.clip(r + dr, 0, H - 1)) * W + np.clip(c + dc, 0, W - 1)
        if n == 3:
            return [flat[lin, c0 + i] for i in range(3)]
        out = []
        for i in range(3):
            j = lin + i
            out.append(np.where(j < total, flat[np.minimum(j, total - 1), c0], np.float32(0)))
        return out

    a_mm, a_mp, a_pm, a_pp = at(1, -1), at(-1, -1), at(1, 1), at(-1, 1)
    a_m0, a_p0, a_0m, a_0p = at(0, -1), at(0, 1), at(1, 0), at(-1, 0)
    sx = np.stack([_scharr_comp(a_mm[i], a_mp[i], a_pm[i], a_pp[i], a_m0[i], a_p0[i]) for i in range(3)], -1)
    sy = np.stack([_scharr_comp(a_mm[i], a_pm[i], a_mp[i], a_pp[i], a_0m[i], a_0p[i]) for i in range(3)], -1)
    return sx, sy


def _l1(s):
    return (np.abs(s[..., 0]) + np.abs(s[..., 1])) + np.abs(s[..., 2])


def restate(vertices, faces, pixels, grad_pixels, ids, gbuf, groups=None, flags=0):
    """-> list with one dict per channel group: c0, n, codes uint8 [B,H,W], rec float32 [B,H,W,2] and the terms:
    pos_p, pos_f (pixel linear index and receiving face b*F + f), pos_t float32 [n,3 corners,3] (x, y, w terms),
    pos_m float64 [n,3,3] (their magnitude bounds); col_p, col_f, col_t float32 [n,3,n0] (the own face's colour terms)."""
    vertices, faces = np.asarray(vertices, np.float32), np.asarray(faces, np.int32)
    pixels, grad_pixels = np.asarray(pixels, np.float32), np.asarray(grad_pixels, np.float32)
    B, H, W, C = pixels.shape
    F = faces.shape[1]
    want_pos, want_col = not flags & SKIP_POSITION, not flags & SKIP_COLOUR
    bb = np.broadcast_to(np.arange(B)[:, None, None], ids.shape)
    rr = np.broadcast_to(np.arange(H)[None, :, None], ids.shape)
    cc = np.broadcast_to(np.arange(W)[None, None, :], ids.shape)
    covered = ids >= 0
    tri = faces[bb, np.maximum(ids, 0)]                              # vertex triple of the own face
    g_w = np.where(covered, gbuf[..., 3], np.float32(np.inf))
    interior = (cc > 0) & (rr > 0) & (cc < W - 1) & (rr < H - 1)
    out = []
    c0 = 0
    with np.errstate(all='ignore'):
        for n in groups_of(C, groups):
            g = dict(c0=c0, n=n)
            gp = grad_pixels[..., c0:c0 + n]
            if want_col:
                p = np.flatnonzero(covered)
                bary = gbuf.reshape(-1, 4)[p, :3]
                g['col_p'], g['col_f'] = p, (bb.ravel()[p] * F + ids.ravel()[p]).astype(np.int64)
                g['col_t'] = bary[:, :, None] * gp.reshape(-1, n)[p][:, None, :]
            else:
                g['col_p'] = g['col_f'] = np.zeros(0, np.int64)
                g['col_t'] = np.zeros((0, 3, n), np.float32)
            codes = np.zeros(ids.shape, np.uint8)
            rec = np.zeros(ids.shape + (2,), np.float32)
            g['pos_p'] = g['pos_f'] = np.zeros(0, np.int64)
            g['pos_t'], g['pos_m'] = np.zeros((0, 3, 3), np.float32), np.zeros((0, 3, 3))
            if want_pos:
                sx, sy = scharr(pixels, c0, n)
                along = _l1(sx) > _l1(sy)
                dx = np.where(along, 1, 0)
                dy = 1 - dx
                odd = ((cc + rr) & 1) == 1
                dx, dy = np.where(odd, -dx, dx), np.where(odd, -dy, dy)
                f = np.where(covered, ids, -1)
                nr, nc = rr.copy(), cc.copy()
                code = np.where(interior & along, DIL_OWN | DIL_ALONG_ROW, DIL_OWN)
                done = ~interior
                for attempt, sgn in ((0, 1), (1, -1)):
                    tc = np.clip(cc + sgn * dx, 0, W - 1)
                    tr = np.clip(rr - sgn * dy, 0, H - 1)
                    fn = ids[bb, tr, tc]
                    differs = ~covered | (faces[bb, np.maximum(fn, 0)] != tri).any(-1)
                    take = ~done & (fn >= 0) & differs & (g_w > gbuf[bb, tr, tc, 3])
                    f, nr, nc = np.where(take, fn, f), np.where(take, tr, nr), np.where(take, tc, nc)
                    code = np.where(take, code + 1 + attempt, code)
                    done |= take
                has = f >= 0
                codes = np.where(has, code, 0).astype(np.uint8)
                dLdx, dLdy = np.zeros(ids.shape, np.float32), np.zeros(ids.shape, np.float32)
                for ch in range(n):
                    dLdx = fmaf(gp[..., ch], sx[..., ch], dLdx)
                    dLdy = fmaf(gp[..., ch], sy[..., ch], dLdy)
                rec = np.where(has[..., None], np.stack([dLdx, dLdy], -1), np.float32(0))
                P = (np.abs(gp.astype(np.float64)) * np.abs(sx[..., :n])).sum(-1)
                Q = (np.abs(gp.astype(np.float64)) * np.abs(sy[..., :n])).sum(-1)
                p = np.flatnonzero(has)
                b_p, f_p = bb.ravel()[p], f.ravel()[p]
                src = (b_p * H + nr.ravel()[p]) * W + nc.ravel()[p]      # the fragment's source pixel
                G = gbuf.reshape(-1, 4)[src]
                bary, w = G[:, :3], G[:, 3]
                xy = vertices[b_p[:, None], faces[b_p, f_p], :2]          # [n, 3 corners, 2]
                zero = np.zeros(len(p), np.float32)
                clip_x = fmaf(bary[:, 2], xy[:, 2, 0], fmaf(bary[:, 1], xy[:, 1, 0], fmaf(bary[:, 0], xy[:, 0, 0], zero)))
                clip_y = fmaf(bary[:, 2], xy[:, 2, 1], fmaf(bary[:, 1], xy[:, 1, 1], fmaf(bary[:, 0], xy[:, 0, 1], zero)))
                inv_w = np.float32(1) / w
                half_w, half_h = np.float32(0.5) * np.float32(W), np.float32(0.5) * np.float32(H)
                dxv_dxc, dyv_dyc = half_w * inv_w, half_h * inv_w
                dxv_dwc, dyv_dwc = -((clip_x * dxv_dxc) * inv_w), -((clip_y * dyv_dyc) * inv_w)
                r = rec.reshape(-1, 2)[p]
                ax, ay = r[:, :1] * bary, r[:, 1:] * bary                 # [n, 3 corners]
                t = np.stack([ax * dxv_dxc[:, None], ay * dyv_dyc[:, None],
                              fmaf(ay, dyv_dwc[:, None], ax * dxv_dwc[:, None])], -1)
                ab, iw = np.abs(bary.astype(np.float64)), np.abs(inv_w.astype(np.float64))
                cx = (np.abs(bary.astype(np.float64)) * np.abs(xy[..., 0])).sum(-1)
                cy = (np.abs(bary.astype(np.float64)) * np.abs(xy[..., 1])).sum(-1)
                Pp, Qp = P.ravel()[p], Q.ravel()[p]
                mx, my = Pp * float(half_w) * iw, Qp * float(half_h) * iw
                mw = mx * cx * iw + my * cy * iw
                g['pos_p'], g['pos_f'] = p, (b_p * F + f_p).astype(np.int64)
                g['pos_t'], g['pos_m'] = t, np.stack([ab * mx[:, None], ab * my[:, None], ab * mw[:, None]], -1)
            g['codes'], g['rec'] = codes, rec
            out.append(g)
            c0 += n
    return out


# ---- the deterministic summation order -----------------------------------------------------------------------------------

def _segment_sums(seg, order, vals):
    """Sums of the rows of vals [n, K] (float64) per segment id, each a sequential float64 sum from +0 in ascending
    `order`.  -> (segment ids, sums [segments, K])."""
    if len(seg) == 0:
        return np.zeros(0, np.int64), np.zeros((0, vals.shape[1]))
    idx = np.lexsort((order, seg))
    seg, vals = seg[idx], vals[idx]
    ids, starts, counts = np.unique(seg, return_index=True, return_counts=True)
    by_len = np.argsort(-counts, kind='stable')
    st, ct = starts[by_len], counts[by_len]
    acc = np.zeros((len(ids), vals.shape[1]))
    for j in range(int(ct[0])):
        live = int(np.searchsorted(-ct, -j, side='left'))   # the segments longer than j, a prefix
        acc[:live] += vals[st[:live] + j]
    sums = np.empty_like(acc)
    sums[by_len] = acc
    return ids, sums


def _butterfly(x):
    """xor butterfly over the last axis (32 lanes): lane 0's result."""
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        x = x + x[..., lanes ^ o]
    return x[..., 0]


def boxes(group, shape, F, flags=0):
    """[B*F, 4] uint32 {min col, min row, ~max col, ~max row} of the faces named by the group's pixels (all ones:
    none), as the record pass grows them."""
    B, H, W = shape
    lo = np.full((B * F, 2), np.iinfo(np.int64).max)
    hi = np.full((B * F, 2), -1)
    for p, f in ((group['col_p'], group['col_f']), (group['pos_p'], group['pos_f'])):
        pix = p % (H * W)
        rc = np.stack([pix % W, pix // W], -1)
        np.minimum.at(lo, f, rc)
        np.maximum.at(hi, f, rc)
    out = np.full((B * F, 4), 0xffffffff, np.uint32)
    used = hi[:, 0] >= 0
    out[used, :2] = lo[used]
    out[used, 2:] = ~hi[used].astype(np.uint32)
    return out


def face_partials(groups, shape, F, C):
    """The per-face float64 partials [B*F, 3, 3 + C] of the deterministic path, in its summation order."""
    B, H, W = shape
    part = np.zeros((B * F, 3, 3 + C))
    for g in groups:
        n = g['n']
        box = boxes(g, shape, F).astype(np.int64)
        used = box[:, 0] != 0xffffffff
        bw = np.where(used, (~box[:, 2] & 0xffffffff) - box[:, 0] + 1, 0)
        bh = np.where(used, (~box[:, 3] & 0xffffffff) - box[:, 1] + 1, 0)
        large = bw * bh > DET_WARP_BOX
        K = 9 + 3 * n
        rows = []
        for p, f, vals, first in ((g['pos_p'], g['pos_f'], g['pos_t'].reshape(-1, 9), 0),
                                  (g['col_p'], g['col_f'], g['col_t'].reshape(-1, 3 * n), 9)):
            v = np.zeros((len(p), K))
            v[:, first:first + vals.shape[1]] = vals
            pix = p % (H * W)
            i = (pix // W - box[f, 1]) * bw[f] + (pix % W - box[f, 0])
            rows.append((f, i, v))
        f = np.concatenate([r[0] for r in rows])
        i = np.concatenate([r[1] for r in rows])
        v = np.concatenate([r[2] for r in rows])
        for cta in (False, True):
            sel = large[f] == cta
            T = CTA_THREADS if cta else 32
            seg, sums = _segment_sums(f[sel] * T + i[sel] % T, i[sel] // T, v[sel])
            faces_u, inv = np.unique(seg // T, return_inverse=True)
            lanes = np.zeros((len(faces_u), T, K))
            lanes[inv, seg % T] = sums
            if cta:   # each warp's butterfly, then warps 0..7 in order
                warps = _butterfly(lanes.reshape(-1, 8, 32, K).transpose(0, 1, 3, 2))
                tot = warps[:, 0]
                for w in range(1, 8):
                    tot = tot + warps[:, w]
            else:
                tot = _butterfly(lanes.transpose(0, 2, 1))
            part[faces_u, :, :3] = part[faces_u, :, :3] + tot[:, :9].reshape(-1, 3, 3)
            part[faces_u, :, 3 + g['c0']:3 + g['c0'] + n] = tot[:, 9:].reshape(-1, 3, n)
    return part


def _corners(faces, V):
    """(row b*V + v, item b, corner id k*F + f, face b*F + f, k) of every corner naming a vertex in range."""
    B, F, _ = faces.shape
    b, f, k = np.meshgrid(np.arange(B), np.arange(F), np.arange(3), indexing='ij')
    v = faces[b, f, k]
    ok = (v >= 0) & (v < V)
    return (b * V + v)[ok], b[ok], (k * F + f)[ok], (b * F + f)[ok], k[ok]


def vertex_sums(part, faces, V, C, shared=False):
    """grad_vertices [rows, 4] and grad_vertex_colors [rows, C] from the partials, rows = B*V (V when shared)."""
    faces = np.asarray(faces, np.int32)
    B = faces.shape[0]
    row, b, corner, gf, k = _corners(faces, V)
    if shared:
        row = row - b * V
    nrows = V if shared else B * V
    seg, sums = _segment_sums(row, b * 3 * faces.shape[1] + corner, part[gf, k])
    s = np.zeros((nrows, 3 + C))
    s[seg] = sums
    s = s.astype(np.float32)
    gv = np.zeros((nrows, 4), np.float32)
    gv[:, [0, 1, 3]] = s[:, :3]
    return gv, s[:, 3:]


def grad_background(ids, grad_pixels):
    return np.where((ids >= 0)[..., None], np.float32(0), grad_pixels).astype(np.float32)


# ---- per-element bound of any summation order -------------------------------------------------------------------------

def term_sums(groups, faces, V, C, shared=False):
    """Per output entry of grad_vertices [rows, 4] and grad_vertex_colors [rows, C]: (S, sum|t|, sum m, n), each an
    array of that shape (S, sum|t| and sum m in float64)."""
    faces = np.asarray(faces, np.int32)
    B, F, _ = faces.shape
    nrows = V if shared else B * V

    def rows_of(gf, k):
        b, f = gf // F, gf % F
        v = faces[b, f, k]
        ok = (v >= 0) & (v < V)   # a visible face names vertices in range
        assert ok.all()
        return v if shared else b * V + v

    out = {}
    for name, width in (('gv', 4), ('gc', C)):
        out[name] = [np.zeros((nrows, width)) for _ in range(3)] + [np.zeros((nrows, width), np.int64)]
    for g in groups:
        for key, tk, mk in (('gv', 'pos_t', 'pos_m'), ('gc', 'col_t', None)):
            t = g[tk].astype(np.float64)
            m = np.abs(t) if mk is None else g[mk]
            cols = [0, 1, 3] if key == 'gv' else list(range(g['c0'], g['c0'] + g['n']))
            f = g['pos_f'] if key == 'gv' else g['col_f']
            for k in range(3):
                r = rows_of(f, np.full(len(f), k))
                for j, col in enumerate(cols):
                    S, A, M, N = out[key]
                    S[:, col] += np.bincount(r, t[:, k, j], nrows)
                    A[:, col] += np.bincount(r, np.abs(t[:, k, j]), nrows)
                    M[:, col] += np.bincount(r, m[:, k, j], nrows)
                    N[:, col] += np.bincount(r, None, nrows)
    return out['gv'], out['gc']


def bound(A, M, N):
    n = N.astype(np.float64)
    return n * U / (1 - n * U) * A + TERM_SLACK_ULPS * U * M


def bound_ratio(got, sums):
    """Worst |got - S| / bound over the entries, and the index of the first entry past its bound (None if none).
    An entry without terms must be exactly 0."""
    S, A, M, N = sums
    got = np.asarray(got, np.float64)
    err = np.abs(got - S)
    lim = bound(A, M, N)
    with np.errstate(all='ignore'):
        ratio = np.where(lim > 0, err / lim, np.where(err > 0, np.inf, 0.0))
    bad = np.argwhere(~(ratio <= 1.0))
    return (float(ratio.max()) if ratio.size else 0.0), (tuple(bad[0]) if len(bad) else None)


# ---- the scratch --------------------------------------------------------------------------------------------------------

SCRATCH_BLOCKS = ('codes', 'rec', 'boxes', 'large', 'large_count', 'partial', 'offsets', 'counts', 'inc', 'unsorted')


def scratch_layout(B, H, W, C, V, F):
    """carve_det_scratch restated: {block: (offset, bytes)} and 'bytes', every block 256-byte aligned."""
    px, bf, bv = B * H * W, B * F, B * V
    sizes = dict(codes=px * C, rec=px * 8, boxes=bf * 16, large=bf * 4, large_count=4, partial=bf * 3 * (3 + C) * 8,
                 offsets=(bv + 1) * 4, counts=bv * 4, inc=bf * 12, unsorted=bf * 12)
    lay, off = {}, 0
    for name in SCRATCH_BLOCKS:
        lay[name] = (off, sizes[name])
        off += (sizes[name] + 255) // 256 * 256
    lay['bytes'] = off if B > 0 else 0
    return lay


def read_scratch(buf, B, H, W, C, V, F):
    """numpy views of a scratch buffer (uint8) after a call."""
    lay = scratch_layout(B, H, W, C, V, F)
    buf = np.asarray(buf, np.uint8)

    def view(name, dtype, shape):
        o, n = lay[name]
        return buf[o:o + n].view(dtype).reshape(shape)

    return dict(codes=view('codes', np.uint8, (C, B, H, W)), rec=view('rec', np.float32, (B, H, W, 2)),
                boxes=view('boxes', np.uint32, (B * F, 4)), large=view('large', np.int32, (B * F,)),
                large_count=int(view('large_count', np.int32, (1,))[0]),
                partial=view('partial', np.float64, (B * F, 3, 3 + C)))


def large_faces(group, shape, F):
    """The faces whose box the CTA pass sweeps."""
    box = boxes(group, shape, F).astype(np.int64)
    used = box[:, 0] != 0xffffffff
    area = ((~box[:, 2] & 0xffffffff) - box[:, 0] + 1) * ((~box[:, 3] & 0xffffffff) - box[:, 1] + 1)
    return np.flatnonzero(used & (area > DET_WARP_BOX))
