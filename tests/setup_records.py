"""The triangle-setup kernel's output, read straight out of a workspace and checked against the contract it must meet.

CPU only (numpy and the CPU oracle, no torch.cuda).  `layout` restates carve_workspace (dirt_b200/csrc/common.cuh) and
`read_workspace` returns numpy views of a workspace's bytes.  `expected` builds, from the oracle's per-face setup records
(oracle/dirt_oracle.c dirt_oracle_setup), what setup.cu must write for (vertices, faces, H, W): the GPU kind of every
face, its TriCov, TriInterp, TriXY and TriShade records and the tiles it is binned to.  `check` compares a workspace
with that and returns the first mismatch as a message naming the image, face or tile, the field, the expected and the
actual value (None when everything holds).  Bins and lists are filled in atomic order, so they are compared as sets.

tests/test_setup_records_host.py shows that the checker rejects each way a workspace can be wrong; tests/
test_gpu_setup_records.py runs it on what the kernels wrote.
"""
import ctypes

import numpy as np

TILE_W, TILE_H = 16, 8          # common.cuh: forward raster / binning tile
SMALL_TILE_LIMIT = 16           # common.cuh: faces whose box spans more tiles go to the image's large list
BIN_CAP = 128                   # common.cuh: references a tile's bin holds
OVF_ROW_CAP = 1024              # common.cuh: entries of one row of tiles' overflow list
SHADE_MAX_CHANNELS = 4          # common.cuh shade_records_ok
SHADE_MAX_EXTENT = 65536
KIND_CULLED, KIND_SMALL, KIND_HARD, KIND_LARGE = 0, 1, 2, 3
KIND_NAMES = {KIND_CULLED: 'culled', KIND_SMALL: 'small', KIND_HARD: 'hard', KIND_LARGE: 'large'}

# ---- record layouts (common.cuh) ----------------------------------------------------------------------------------------


def _struct(fields):
    names, formats, offsets, off = [], [], [], 0
    for name, *fmt in fields:
        dt = np.dtype(tuple(fmt) if len(fmt) > 1 else fmt[0])
        names.append(name)
        formats.append(dt)
        offsets.append(off)
        off += dt.itemsize
    return names, formats, offsets


def _dtype(fields, itemsize):
    names, formats, offsets = _struct(fields)
    return np.dtype(dict(names=names, formats=formats, offsets=offsets, itemsize=itemsize))


_EDGES = [('A0', '<i4'), ('B0', '<i4'), ('A1', '<i4'), ('B1', '<i4'), ('A2', '<i4'), ('B2', '<i4')]
# TriCov, the two layouts of its union: KIND_SMALL (q relative to the box corner, int32) and KIND_LARGE / KIND_HARD
# (absolute int64 q).  `kind` sits at byte 60 in both.
COV_SMALL = _dtype(_EDGES + [('q0r', '<i4'), ('q1r', '<i4'), ('q2r', '<i4'), ('zA', '<f4'), ('zB', '<f4'), ('zC', '<f4'),
                             ('cref', '<i4'), ('rref', '<i4'), ('pad', '<i4'), ('kind', '<u4')], 64)
COV_LARGE = _dtype(_EDGES + [('zA', '<f4'), ('zB', '<f4'), ('q0', '<i8'), ('q1', '<i8'), ('q2', '<i8'), ('zC', '<f4'),
                             ('kind', '<u4')], 64)
ITP = _dtype([(n, '<f4') for n in ('q0A', 'q0B', 'q0C', 'q1A', 'q1B', 'q1C', 'sA', 'sB', 'sC')] +
             [(n, '<i4') for n in ('v0', 'v1', 'v2', 'cref', 'rref', 'pad0', 'pad1')], 64)
XY = _dtype([(n, '<f4') for n in ('x0', 'y0', 'x1', 'y1', 'x2', 'y2', 'pad0', 'pad1')], 32)
SHADE = _dtype([('sA', '<f4'), ('sB', '<f4'), ('sC', '<f4'), ('ref', '<u4'), ('n', '<f4', (4, 3))], 64)
HEADER = _dtype([('tag', '<u8'), ('error', '<i4'), ('pad', '<i4')], 16)
ITP_PLANES = ('q0A', 'q0B', 'q0C', 'q1A', 'q1B', 'q1C', 'sA', 'sB', 'sC')
XY_FIELDS = ('x0', 'y0', 'x1', 'y1', 'x2', 'y2')

BLOCKS = ('cov', 'itp', 'xy', 'shade', 'tile_count', 'tile_flags', 'face_in_large', 'large_count', 'ovf_count', 'header',
          'large_list', 'bins', 'ovf', 'gc_pad', 'face_ids')


def tiles_of(H, W):
    """(tiles_x, tiles_y) of the 16x8 binning tiles of an H x W frame."""
    return -(-W // TILE_W), -(-H // TILE_H)


def layout(B, H, W, C, V, F):
    """carve_workspace: {block: (byte offset, bytes)}, plus 'bytes_min' (what dirt_workspace_bytes_min asks for: every
    block before face_ids, and 256 bytes of slack) and 'bytes' (dirt_workspace_bytes: all blocks and the slack).  Blocks
    follow each other in BLOCKS order, each at a 256-byte aligned offset."""
    tx, ty = tiles_of(H, W)
    BF, BT, rows = B * F, B * tx * ty, B * ty
    size = dict(cov=BF * 64, itp=BF * 64, xy=BF * 32, shade=BF * 64, tile_count=BT * 4, tile_flags=BT, face_in_large=BF,
                large_count=B * 4, ovf_count=rows * 4, header=256, large_list=BF * 4, bins=BT * BIN_CAP * 4,
                ovf=rows * OVF_ROW_CAP * 8, gc_pad=B * V * 16 if C == 3 else 0, face_ids=B * H * W * 4)
    out, off = {}, 0
    for name in BLOCKS:
        out[name] = (off, size[name])
        off = -(-(off + size[name]) // 256) * 256
    out['bytes_min'] = out['face_ids'][0] + 256
    out['bytes'] = off + 256
    return out


def read_workspace(ws, B, H, W, C, V, F):
    """Numpy views of a workspace's bytes (a uint8 array of at least dirt_workspace_bytes_min), per image:
    cov_small / cov_large [B, F] (the two TriCov layouts), itp [B, F], xy [B, F], shade [B, F], tile_count [B, T],
    tile_flags [B, T], face_in_large [B, F], large_count [B], ovf_count [B, tiles_y], header [1] (tag, error),
    large_list [B, F], bins [B, T, 128], ovf [B * tiles_y, 1024, 2] ((tile, face) pairs)."""
    ws = np.asarray(ws)
    assert ws.dtype == np.uint8 and ws.ndim == 1
    lay = layout(B, H, W, C, V, F)
    assert ws.size >= lay['bytes_min'] - 256, 'workspace of %d bytes, the layout needs %d' % (ws.size, lay['bytes_min'] - 256)
    tx, ty = tiles_of(H, W)
    T = tx * ty

    def block(name, dtype, shape):
        off, n = lay[name]
        return ws[off:off + n].view(dtype).reshape(shape)

    return dict(cov_small=block('cov', COV_SMALL, (B, F)), cov_large=block('cov', COV_LARGE, (B, F)),
                itp=block('itp', ITP, (B, F)), xy=block('xy', XY, (B, F)), shade=block('shade', SHADE, (B, F)),
                tile_count=block('tile_count', '<i4', (B, T)), tile_flags=block('tile_flags', np.uint8, (B, T)),
                face_in_large=block('face_in_large', np.uint8, (B, F)), large_count=block('large_count', '<i4', (B,)),
                ovf_count=block('ovf_count', '<i4', (B, ty)), header=block('header', HEADER, (16,))[:1],
                large_list=block('large_list', '<i4', (B, F)), bins=block('bins', '<i4', (B, T, BIN_CAP)),
                ovf=block('ovf', '<i4', (B * ty, OVF_ROW_CAP, 2)))


def workspace_tag(vertices_ptr, faces_ptr, B, H, W, V, F):
    """common.cuh workspace_tag: FNV-1a over the bytes of the seven 64-bit words (pointers, then sizes); never 0."""
    h = 1469598103934665603
    for word in (vertices_ptr, faces_ptr, B, H, W, V, F):
        for k in range(8):
            h ^= (int(word) >> (8 * k)) & 0xff
            h = (h * 1099511628211) & 0xffffffffffffffff
    return h or 1


# ---- what the oracle says -----------------------------------------------------------------------------------------------

# oracle/dirt_oracle.c TriExport, as a numpy record (checked against oracle.TriExport's ctypes layout)
EXPORT = np.dtype([('A', '<i4', 3), ('B', '<i4', 3), ('q', '<i8', 3), ('z', '<f4', 3), ('q0', '<f4', 3), ('q1', '<f4', 3),
                   ('s', '<f4', 3), ('cref', '<i4'), ('rref', '<i4'), ('kind', '<i4'), ('bbox', '<i4', 4)], align=True)


def oracle_records(vertices, faces, H, W):
    """The oracle's setup records of every image: a structured [B, F] array of EXPORT (bbox = cmin, rmin, cmax, rmax)."""
    from oracle import oracle
    ct = oracle.TriExport
    assert EXPORT.itemsize == ctypes.sizeof(ct)
    assert all(EXPORT.fields[n][1] == getattr(ct, n).offset for n in EXPORT.names)
    vertices = np.ascontiguousarray(vertices, np.float32)
    faces = np.ascontiguousarray(faces, np.int32)
    B, V, _ = vertices.shape
    F = faces.shape[1]
    out = np.zeros((B, max(F, 1)), EXPORT)[:, :F]
    fn = oracle.lib().dirt_oracle_setup
    for b in range(B):
        if F:
            fn(vertices[b].ctypes.data_as(ctypes.c_void_p), faces[b].ctypes.data_as(ctypes.c_void_p),
               out[b].ctypes.data_as(ctypes.c_void_p), H, W, V, F)
    return out


def planes_double(p, H, W):
    """common.cuh exact::planes_double restated in numpy float64 (every operation IEEE-rounded, none fused):
    p [N, 3, 4] float32 clip vertices -> gq [N, 3, 3] (the planes of q_k), gs [N, 3] (the plane of 1/w)."""
    x, y, w = (p[..., j].astype(np.float64) for j in (0, 1, 3))
    x0, x1, x2 = x[:, 0], x[:, 1], x[:, 2]
    y0, y1, y2 = y[:, 0], y[:, 1], y[:, 2]
    w0, w1, w2 = w[:, 0], w[:, 1], w[:, 2]
    c = np.stack([np.stack([y1 * w2 - y2 * w1, y2 * w0 - y0 * w2, y0 * w1 - y1 * w0], 1),
                  np.stack([w1 * x2 - w2 * x1, w2 * x0 - w0 * x2, w0 * x1 - w1 * x0], 1),
                  np.stack([x1 * y2 - x2 * y1, x2 * y0 - x0 * y2, x0 * y1 - x1 * y0], 1)], 1)
    with np.errstate(all='ignore'):
        det = (x0 * c[:, 0, 0] + y0 * c[:, 1, 0]) + w0 * c[:, 2, 0]
        inv = c * (1.0 / det)[:, None, None]
    two_over_W, two_over_H, inv_W, inv_H = 2.0 / W, 2.0 / H, 1.0 / W, 1.0 / H

    def to_pixel(a, b, cc):
        return np.stack([a * two_over_W, -(b * two_over_H), (a * (inv_W - 1.0) + b * (1.0 - inv_H)) + cc], -1)

    gq = np.stack([to_pixel(inv[:, 0, k], inv[:, 1, k], inv[:, 2, k]) for k in range(3)], 1)
    gs = to_pixel(*[(inv[:, r, 0] + inv[:, r, 1]) + inv[:, r, 2] for r in range(3)])
    return gq, gs


def snapped(p, H, W):
    """S1-S2 of setup.cu: the window position of each vertex in 1/256 px, int64 [N, 3] x and y (float32 arithmetic in
    the kernel's order, round half to even)."""
    with np.errstate(all='ignore'):
        xn = p[..., 0] / p[..., 3]
        yn = p[..., 1] / p[..., 3]
        X = (xn + np.float32(1.0)) * np.float32(0.5 * W)
        Y = (np.float32(1.0) - yn) * np.float32(0.5 * H)
        fx, fy = np.rint(X * np.float32(256.0)), np.rint(Y * np.float32(256.0))
    # outside the guard band (hard faces) the value is not used
    return (np.clip(np.nan_to_num(fx), -2.0 ** 40, 2.0 ** 40).astype(np.int64),
            np.clip(np.nan_to_num(fy), -2.0 ** 40, 2.0 ** 40).astype(np.int64))


def gpu_kind(rec, H, W):
    """The kind setup.cu gives each face, from the oracle's kind (0 culled, 1 normal, 2 hard).  A normal face is
    KIND_SMALL when its box spans at most SMALL_TILE_LIMIT 16x8 tiles and its edge functions fit the raster loop's
    int32 arithmetic: |A|, |B| < 2^18 and |q + A*cmin + B*rmin| < 2^29 for each edge (setup.cu:261-273); otherwise
    KIND_LARGE."""
    kind = np.full(rec.shape, KIND_CULLED, np.uint32)
    kind[rec['kind'] == 2] = KIND_HARD
    normal = rec['kind'] == 1
    cmin, rmin, cmax, rmax = (rec['bbox'][..., j].astype(np.int64) for j in range(4))
    n_tiles = (cmax // TILE_W - cmin // TILE_W + 1) * (rmax // TILE_H - rmin // TILE_H + 1)
    A, Bc = rec['A'].astype(np.int64), rec['B'].astype(np.int64)
    qr = rec['q'] + A * cmin[..., None] + Bc * rmin[..., None]
    fits = (np.maximum(np.abs(A), np.abs(Bc)).max(-1) < 2 ** 18) & (np.abs(qr) < 2 ** 29).all(-1)
    small = normal & (n_tiles <= SMALL_TILE_LIMIT) & fits
    kind[small] = KIND_SMALL
    kind[normal & ~small] = KIND_LARGE
    return kind


def expected(vertices, faces, vertex_colors, H, W):
    """What setup.cu must write for (vertices [B,V,4], faces [B,F,3]) on an H x W frame: a dict with the oracle's records
    ('rec'), the GPU kind of each face ('kind' [B,F]), the exact TriCov / TriInterp / TriXY bytes ('cov', 'itp', 'xy':
    structured [B,F] arrays), and, when `vertex_colors` [B,V,C] is given, the TriShade record: its exact fields
    ('shade': sA, sB and ref) and the float64 values its fp32 fields approximate ('shade_sC', 'shade_n' [B,F,4,3]) with
    the sums of the magnitudes of their terms ('shade_sC_terms', 'shade_n_terms')."""
    vertices = np.ascontiguousarray(vertices, np.float32)
    faces = np.ascontiguousarray(faces, np.int32)
    B, V = vertices.shape[:2]
    F = faces.shape[1]
    rec = oracle_records(vertices, faces, H, W)
    kind = gpu_kind(rec, H, W)
    live = kind != KIND_CULLED
    small = kind == KIND_SMALL
    cmin, rmin = rec['bbox'][..., 0], rec['bbox'][..., 1]

    # TriCov.  Culled: edge functions that reject every pixel (A = B = 0, q = -1), z = 0 (setup.cu:82-93).  Hard: A = B = 0
    # and q = -1 as well (hard faces are tested from their vertices, not from these fields), the z plane.
    cl = np.zeros((B, F), COV_LARGE)
    for k in range(3):
        cl['A%d' % k] = np.where(kind == KIND_LARGE, rec['A'][..., k], 0)
        cl['B%d' % k] = np.where(kind == KIND_LARGE, rec['B'][..., k], 0)
        cl['q%d' % k] = np.where(kind == KIND_LARGE, rec['q'][..., k], -1)
    for j, n in enumerate(('zA', 'zB', 'zC')):
        cl[n] = np.where(live, rec['z'][..., j], np.float32(0))
    cl['kind'] = kind
    cov = cl.view(np.uint8).reshape(B, F, 64).copy()
    cs = np.zeros((B, F), COV_SMALL)
    for k in range(3):
        cs['A%d' % k], cs['B%d' % k] = rec['A'][..., k], rec['B'][..., k]
        cs['q%dr' % k] = rec['q'][..., k] + rec['A'][..., k].astype(np.int64) * cmin + rec['B'][..., k].astype(np.int64) * rmin
    for j, n in enumerate(('zA', 'zB', 'zC')):
        cs[n] = rec['z'][..., j]
    cs['cref'], cs['rref'], cs['kind'] = cmin, rmin, KIND_SMALL
    cov[small] = cs.view(np.uint8).reshape(B, F, 64)[small]
    cov = cov.reshape(-1).view(COV_LARGE).reshape(B, F)

    # TriInterp: the oracle's planes, vertex ids and reference pixel; a culled face has sC = 1 and zeros elsewhere
    itp = np.zeros((B, F), ITP)
    for j in range(3):
        itp['q0' + 'ABC'[j]] = rec['q0'][..., j]
        itp['q1' + 'ABC'[j]] = rec['q1'][..., j]
        itp['s' + 'ABC'[j]] = rec['s'][..., j]
        itp['v%d' % j] = np.where(live, faces[..., j], 0)
    itp['cref'], itp['rref'] = rec['cref'], rec['rref']
    itp[~live] = np.zeros(1, ITP)[0]
    itp['sC'][~live] = 1.0

    # TriXY: the clip x and y of the three vertices; zeros for a culled face
    xy = np.zeros((B, F), XY)
    safe = np.clip(faces, 0, max(V - 1, 0))
    if V:
        p = np.take_along_axis(vertices, safe.reshape(B, F * 3, 1), 1).reshape(B, F, 3, 4)
    else:
        p = np.zeros((B, F, 3, 4), np.float32)
    for k in range(3):
        xy['x%d' % k] = np.where(live, p[..., k, 0], np.float32(0))
        xy['y%d' % k] = np.where(live, p[..., k, 1], np.float32(0))
    out = dict(rec=rec, kind=kind, cov=cov, itp=itp, xy=xy)
    if vertex_colors is not None:
        C = np.shape(vertex_colors)[-1]
        col = np.zeros((B * F, 3, C), np.float32)
        if V:
            col = np.take_along_axis(np.asarray(vertex_colors, np.float32), safe.reshape(B, F * 3, 1), 1).reshape(B * F, 3, C)
        out.update(_expected_shade(p.reshape(B * F, 3, 4), rec.reshape(-1), kind.reshape(-1), itp.reshape(-1), col, H, W,
                                   (B, F)))
    return out


def _expected_shade(p, rec, kind, itp, col, H, W, shape):
    """TriShade (setup.cu:234-258).  The record is re-based to the pixel under the face's vertex of largest clip w (the
    first of equals): for a normal face its snapped window position, clamped to the box; for a hard face the
    interpolation record's reference pixel.  sA and sB are TriInterp's; sC and the N_c planes are float64 sums rounded to
    fp32 once, whose operation order the kernel leaves to the compiler (contracted or not), so they are compared with
    the float64 value at the accuracy of one fp32 rounding of a float64 sum."""
    N = p.shape[0]
    far = np.zeros(N, np.int64)
    for k in (1, 2):
        far = np.where(p[:, k, 3] > p[np.arange(N), far, 3], k, far)
    fx, fy = snapped(p, H, W)
    cmin, rmin, cmax, rmax = (rec['bbox'][:, j].astype(np.int64) for j in range(4))
    fcol = np.clip(fx[np.arange(N), far] >> 8, cmin, cmax)
    frow = np.clip(fy[np.arange(N), far] >> 8, rmin, rmax)
    hard = kind == KIND_HARD
    fcol = np.where(hard, rec['cref'], fcol)
    frow = np.where(hard, rec['rref'], frow)
    live = kind != KIND_CULLED
    fcol, frow = np.where(live, fcol, 0), np.where(live, frow, 0)
    with np.errstate(all='ignore'):
        gq, gs = planes_double(p, H, W)
    fc, fr = fcol.astype(np.float64), frow.astype(np.float64)
    shade = np.zeros(N, SHADE)
    shade['sA'], shade['sB'] = itp['sA'], itp['sB']
    shade['ref'] = (fcol.astype(np.uint32) | (frow.astype(np.uint32) << 16))
    C = col.shape[-1]
    c = np.zeros((N, 3, 4))
    c[..., :min(C, 4)] = col[..., :4]
    with np.errstate(all='ignore'):
        sC = (gs[:, 0] * fc + gs[:, 1] * fr) + gs[:, 2]
        sC_terms = np.abs(gs[:, 0] * fc) + np.abs(gs[:, 1] * fr) + np.abs(gs[:, 2])
        d0, d1, c2 = c[:, 0] - c[:, 2], c[:, 1] - c[:, 2], c[:, 2]                     # [N, 4]
        t = [gq[:, 0, j, None] * d0 + gq[:, 1, j, None] * d1 + gs[:, j, None] * c2 for j in range(3)]
        m = [np.abs(gq[:, 0, j, None] * d0) + np.abs(gq[:, 1, j, None] * d1) + np.abs(gs[:, j, None] * c2) for j in range(3)]
        n = np.stack([t[0], t[1], (t[0] * fc[:, None] + t[1] * fr[:, None]) + t[2]], -1)
        n_terms = np.stack([m[0], m[1], m[0] * fc[:, None] + m[1] * fr[:, None] + m[2]], -1)
    return dict(shade=shade.reshape(shape), shade_sC=sC.reshape(shape), shade_sC_terms=sC_terms.reshape(shape),
                shade_n=n.reshape(shape + (4, 3)), shade_n_terms=n_terms.reshape(shape + (4, 3)))


def shade_error(actual, exact, terms):
    """|fp32 actual - float64 exact| as a multiple of what one fp32 rounding of a float64 sum may be off by:
    2^-24 |exact| (the rounding to fp32) + 2^-48 * (sum of the magnitudes of its terms) (the float64 sum, in any order,
    fused or not)."""
    allowed = 2.0 ** -24 * np.abs(exact) + 2.0 ** -48 * terms + 1e-45
    return np.abs(np.asarray(actual, np.float64) - exact) / allowed


def binned_tiles(kind, rec, H, W):
    """Every (image, tile, face) reference the small faces put in bins: int64 keys (b*T + t)*F + f, ascending."""
    B, F = kind.shape
    tx_n, ty_n = tiles_of(H, W)
    T = tx_n * ty_n
    b, f = np.nonzero(kind == KIND_SMALL)
    box = rec['bbox'][b, f].astype(np.int64)
    tx0, ty0 = box[:, 0] // TILE_W, box[:, 1] // TILE_H
    sx, sy = box[:, 2] // TILE_W - tx0 + 1, box[:, 3] // TILE_H - ty0 + 1
    n = sx * sy
    face = np.repeat(np.arange(len(f)), n)
    k = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
    t = (ty0[face] + k // sx[face]) * tx_n + tx0[face] + k % sx[face]
    return np.sort((b[face].astype(np.int64) * T + t) * F + f[face])


def tile_flags_of(face_ids, H, W):
    """tile_flags as the raster kernel must leave them: 1 on every 16x8 tile within one tile (3x3) of a tile that shows a
    face, from face ids [B,H,W]."""
    B = face_ids.shape[0]
    tx, ty = tiles_of(H, W)
    shows = np.zeros((B, ty * TILE_H, tx * TILE_W), bool)
    shows[:, :H, :W] = face_ids >= 0
    shows = shows.reshape(B, ty, TILE_H, tx, TILE_W).any((2, 4))
    pad = np.zeros((B, ty + 2, tx + 2), bool)
    pad[:, 1:-1, 1:-1] = shows
    flags = np.zeros((B, ty, tx), bool)
    for dy in range(3):
        for dx in range(3):
            flags |= pad[:, dy:dy + ty, dx:dx + tx]
    return flags.reshape(B, -1).astype(np.uint8)


# ---- the checker -----------------------------------------------------------------------------------------------------


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype.itemsize == 4 else np.uint64)


def _first(mask):
    idx = np.argwhere(mask)
    return tuple(int(i) for i in idx[0]) if len(idx) else None


def _fmt(v):
    if isinstance(v, (np.floating, float)):
        return '%r (0x%08x)' % (float(v), int(np.float32(v).view(np.uint32)))
    return repr(v.item() if hasattr(v, 'item') else v)


def check_records(view, exp, images, shade=False, stats=None):
    """The TriCov, TriInterp and TriXY records (and TriShade with `shade`) of `images` against `exp`; first mismatch or None."""
    kind = exp['kind']
    small = kind == KIND_SMALL
    label = lambda b, f: 'image %d face %d (%s)' % (images[b], f, KIND_NAMES[int(kind[b, f])])
    got_small, got_large = view['cov_small'][images], view['cov_large'][images]
    got_kind = got_small['kind']
    bad = got_kind != kind
    if bad.any():
        b, f = _first(bad)
        return '%s: TriCov.kind expected %d (%s), got %d' % (label(b, f), kind[b, f], KIND_NAMES[int(kind[b, f])], got_kind[b, f])
    want_small = np.ascontiguousarray(exp['cov']).view(COV_SMALL)
    for name in COV_SMALL.names:
        if name == 'kind':
            continue
        g, w = _bits(got_small[name]), _bits(want_small[name])
        bad = small & (g != w)
        if bad.any():
            b, f = _first(bad)
            return '%s: TriCov.%s expected %s, got %s' % (label(b, f), name, _fmt(want_small[name][b, f]),
                                                          _fmt(got_small[name][b, f]))
    for name in COV_LARGE.names:
        if name == 'kind':
            continue
        g, w = _bits(got_large[name]), _bits(exp['cov'][name])
        bad = ~small & (g != w)
        if bad.any():
            b, f = _first(bad)
            return '%s: TriCov.%s expected %s, got %s' % (label(b, f), name, _fmt(exp['cov'][name][b, f]),
                                                          _fmt(got_large[name][b, f]))
    for rec, dtype, got in (('TriInterp', ITP, view['itp'][images]), ('TriXY', XY, view['xy'][images])):
        want = exp['itp'] if rec == 'TriInterp' else exp['xy']
        for name in dtype.names:
            bad = _bits(got[name]) != _bits(want[name])
            if bad.any():
                b, f = _first(bad)
                return '%s: %s.%s expected %s, got %s' % (label(b, f), rec, name, _fmt(want[name][b, f]),
                                                          _fmt(got[name][b, f]))
    if shade:
        got = view['shade'][images]
        live = kind != KIND_CULLED   # a culled face has no shading record
        for name in ('sA', 'sB', 'ref'):
            bad = live & (_bits(got[name]) != _bits(exp['shade'][name]))
            if bad.any():
                b, f = _first(bad)
                return '%s: TriShade.%s expected %s, got %s' % (label(b, f), name, _fmt(exp['shade'][name][b, f]),
                                                                _fmt(got[name][b, f]))
        r_sC = np.where(live, shade_error(got['sC'], exp['shade_sC'], exp['shade_sC_terms']), 0.0)
        r_n = np.where(live[..., None, None], shade_error(got['n'], exp['shade_n'], exp['shade_n_terms']), 0.0)
        if stats is not None:
            stats['shade_ratio'] = max(stats.get('shade_ratio', 0.0), float(r_sC.max(initial=0)), float(r_n.max(initial=0)))
        if (r_sC > 1).any():
            b, f = _first(r_sC > 1)
            return '%s: TriShade.sC expected %r (float64), got %s: %.1fx one fp32 rounding' % (
                label(b, f), exp['shade_sC'][b, f], _fmt(got['sC'][b, f]), r_sC[b, f])
        if (r_n > 1).any():
            b, f, c, j = _first(r_n > 1)
            return '%s: TriShade.n[%d][%d] expected %r (float64), got %s: %.1fx one fp32 rounding' % (
                label(b, f), c, j, exp['shade_n'][b, f, c, j], _fmt(got['n'][b, f, c, j]), r_n[b, f, c, j])
    return None


def check_lists(view, exp, images, H, W, stats=None):
    """tile_count, the bins, the row overflow lists, face_in_large and the large list of `images`; first mismatch or None."""
    kind, rec = exp['kind'], exp['rec']
    nb, F = kind.shape
    tx, ty = tiles_of(H, W)
    T = tx * ty
    count = view['tile_count'][images].astype(np.int64)
    want = binned_tiles(kind, rec, H, W)
    want_count = np.bincount(want // F, minlength=nb * T).reshape(nb, T)
    bad = count != want_count
    if bad.any():
        b, t = _first(bad)
        return 'image %d tile %d: tile_count expected %d (small faces whose box touches the tile), got %d' % (
            images[b], t, want_count[b, t], count[b, t])
    ovf_count = view['ovf_count'][images].astype(np.int64)
    want_ovf = np.maximum(want_count - BIN_CAP, 0).reshape(nb, ty, tx).sum(-1)
    bad = ovf_count != want_ovf
    if bad.any():
        b, r = _first(bad)
        return 'image %d tile row %d: ovf_count expected %d (references past full bins), got %d' % (
            images[b], r, want_ovf[b, r], ovf_count[b, r])

    # the references actually stored: bins[:min(count, 128)] and the first min(ovf_count, 1024) row-list entries
    bins = view['bins'][images].astype(np.int64)
    held = np.arange(BIN_CAP)[None, None, :] < np.minimum(count, BIN_CAP)[..., None]
    bt = np.broadcast_to((np.arange(nb)[:, None] * T + np.arange(T)[None, :])[..., None], bins.shape)
    f_bin, bt_bin = bins[held], bt[held]
    rows = np.asarray(images)[:, None] * ty + np.arange(ty)[None, :]
    ovf = view['ovf'][rows.reshape(-1)].reshape(nb, ty, OVF_ROW_CAP, 2).astype(np.int64)
    held = np.arange(OVF_ROW_CAP)[None, None, :] < np.minimum(ovf_count, OVF_ROW_CAP)[..., None]
    t_ovf, f_ovf = ovf[..., 0][held], ovf[..., 1][held]
    b_ovf, r_ovf = np.nonzero(held)[:2]
    bad = (t_ovf < 0) | (t_ovf >= T) | (t_ovf // max(tx, 1) != r_ovf)
    if bad.any():
        i = int(np.argmax(bad))
        return 'image %d tile row %d: row-list entry names tile %d, which is not in the row' % (images[b_ovf[i]], r_ovf[i], t_ovf[i])
    faces = np.concatenate([f_bin, f_ovf])
    where = np.concatenate([bt_bin, b_ovf * T + t_ovf])
    bad = (faces < 0) | (faces >= F)
    if bad.any():
        i = int(np.argmax(bad))
        return 'image %d tile %d: reference to face %d, not a face index' % (images[where[i] // T], where[i] % T, faces[i])
    got = np.sort(where * F + faces)
    dup = got[1:] == got[:-1]
    if dup.any():
        key = got[1:][dup][0]
        return 'image %d tile %d: duplicated reference to face %d' % (images[key // F // T], key // F % T, key % F)
    extra = got[~np.isin(got, want, assume_unique=True)]
    if extra.size:
        key = extra[0]
        b, t, f = key // F // T, key // F % T, key % F
        what = 'whose box does not touch the tile' if kind[b, f] == KIND_SMALL else 'of kind %s' % KIND_NAMES[int(kind[b, f])]
        return 'image %d tile %d: reference to face %d %s (box %s)' % (images[b], t, f, what, list(rec['bbox'][b, f]))
    missing = want[~np.isin(want, got, assume_unique=True)]
    # a reference neither in its bin nor in its row's list must have gone to the large list, which happens only when the
    # row's list was full
    mb, mt, mf = missing // F // T, missing // F % T, missing % F
    lc = view['large_count'][images].astype(np.int64)
    in_large = np.zeros((nb, F), bool)
    for b in range(nb):
        lst = view['large_list'][images[b], :int(np.clip(lc[b], 0, F))]
        in_large[b, lst[(lst >= 0) & (lst < F)]] = True
    bad = (ovf_count[mb, mt // max(tx, 1)] <= OVF_ROW_CAP) | ~in_large[mb, mf]
    if bad.any():
        i = int(np.argmax(bad))
        return 'image %d tile %d: dropped reference to face %d (in neither the bin, the row list nor the large list)' % (
            images[mb[i]], mt[i], mf[i])
    spilled = np.zeros((nb, F), bool)
    spilled[mb, mf] = True
    fil = view['face_in_large'][images]
    bad = (fil != 0) != spilled
    if bad.any():
        b, f = _first(bad)
        return 'image %d face %d: face_in_large expected %d, got %d' % (images[b], f, spilled[b, f], fil[b, f])
    bad = (fil != 0) & (fil != 1)
    if bad.any():
        b, f = _first(bad)
        return 'image %d face %d: face_in_large expected 1, got %d' % (images[b], f, fil[b, f])

    # the large list: the large and hard faces, and each spilled small face, exactly once
    want_large = (kind == KIND_LARGE) | (kind == KIND_HARD) | spilled
    for b in range(nb):
        n = want_large[b].sum()
        if lc[b] != n:
            if 0 <= lc[b] <= F:
                lst = view['large_list'][images[b], :lc[b]]
                wrong = [int(f) for f in lst if not (0 <= f < F and want_large[b, f])]
                if wrong:
                    f = wrong[0]
                    what = 'not a face index' if not 0 <= f < F else 'a %s face that was not spilled' % KIND_NAMES[int(kind[b, f])]
                    return 'image %d: large list holds face %d, %s' % (images[b], f, what)
            return 'image %d: large_count expected %d, got %d' % (images[b], n, lc[b])
        lst = np.sort(view['large_list'][images[b], :n].astype(np.int64))
        if (lst[1:] == lst[:-1]).any():
            return 'image %d: large list holds face %d twice' % (images[b], lst[1:][lst[1:] == lst[:-1]][0])
        want_b = np.nonzero(want_large[b])[0]
        if not np.array_equal(lst, want_b):
            f = int(np.setdiff1d(lst, want_b)[0])
            what = 'not a face index' if not 0 <= f < F else 'a %s face that was not spilled' % KIND_NAMES[int(kind[b, f])]
            return 'image %d: large list holds face %d, %s' % (images[b], f, what)
    if stats is not None:
        stats['bins_past_cap'] = stats.get('bins_past_cap', 0) + int((count > BIN_CAP).sum())
        stats['rows_in_list'] = stats.get('rows_in_list', 0) + int((ovf_count > 0).sum())
        stats['rows_past_cap'] = stats.get('rows_past_cap', 0) + int((ovf_count > OVF_ROW_CAP).sum())
        stats['tiles_spilled_to_large'] = stats.get('tiles_spilled_to_large', 0) + int(len(np.unique(missing // F)))
        stats['faces_spilled_to_large'] = stats.get('faces_spilled_to_large', 0) + int(spilled.sum())
    return None


def check(ws, vertices, faces, H, W, C, vertex_colors=None, face_ids=None, lists=True, shade=None, images=None,
          tag=None, exp=None, stats=None):
    """The setup output in workspace bytes `ws` (uint8 numpy array) of a call on (vertices [B,V,4], faces [B,F,3]) and an
    H x W frame of C channels, for `images` (default: all).  Checks the records; with `lists` tile_count, bins, row lists,
    face_in_large and the large list (a call that binned); with `shade` (default: C <= 4 and the frame within the
    shading record's 16-bit reference pixel, when `vertex_colors` is given) the TriShade records; with `face_ids`
    [B,H,W] tile_flags (a call that ran the raster kernel); with `tag` the header.  `exp` is expected()'s result for
    these images, if already built.  Counts of kinds and list levels go into `stats`.  Returns the first mismatch as a
    message, or None."""
    B, V = np.shape(vertices)[:2]
    F = np.shape(faces)[1]
    images = np.arange(B) if images is None else np.asarray(images)
    view = read_workspace(ws, B, H, W, C, V, F)
    if shade is None:
        shade = vertex_colors is not None and C <= SHADE_MAX_CHANNELS and H <= SHADE_MAX_EXTENT and W <= SHADE_MAX_EXTENT
    if exp is None:
        exp = expected(np.asarray(vertices)[images], np.asarray(faces)[images],
                       None if not shade else np.asarray(vertex_colors)[images], H, W)
    if tag is not None:
        hdr = view['header']
        if int(hdr['tag'][0]) != tag:
            return 'header: tag expected 0x%016x (workspace_tag of this call), got 0x%016x' % (tag, int(hdr['tag'][0]))
        if int(hdr['error'][0]) != 0:
            return 'header: error expected 0, got %d' % int(hdr['error'][0])
    if stats is not None:
        for k, name in KIND_NAMES.items():
            stats[name] = stats.get(name, 0) + int((exp['kind'] == k).sum())
    msg = check_records(view, exp, images, shade=shade, stats=stats)
    if msg is None and lists:
        msg = check_lists(view, exp, images, H, W, stats=stats)
    if msg is None and face_ids is not None:
        want = tile_flags_of(np.asarray(face_ids)[images], H, W)
        got = view['tile_flags'][images]
        bad = got != want
        if bad.any():
            b, t = _first(bad)
            what = 'missing tile flag' if want[b, t] else 'extra tile flag'
            return 'image %d tile %d: %s: tile_flags expected %d, got %d' % (images[b], t, what, want[b, t], got[b, t])
    return msg


def perfect_workspace(vertices, faces, vertex_colors, H, W, C, face_ids=None, tag=0, seed=0):
    """Workspace bytes that hold exactly what `check` asks of a forward call: the expected records, each small face in
    the bins of the tiles its box touches (in a shuffled order, spilling to the row lists and the large list as
    setup.cu does), tile_flags from `face_ids`, and the header's tag.  For testing the checker."""
    vertices, faces = np.asarray(vertices, np.float32), np.asarray(faces, np.int32)
    B, V = vertices.shape[:2]
    F = faces.shape[1]
    lay = layout(B, H, W, C, V, F)
    ws = np.zeros(lay['bytes'], np.uint8)
    view = read_workspace(ws, B, H, W, C, V, F)
    exp = expected(vertices, faces, vertex_colors, H, W)
    view['cov_large'][:] = exp['cov']
    view['itp'][:] = exp['itp']
    view['xy'][:] = exp['xy']
    if 'shade' in exp:
        sh = exp['shade'].copy()
        sh['sC'] = exp['shade_sC']
        sh['n'] = exp['shade_n']
        view['shade'][:] = sh
    tx, ty = tiles_of(H, W)
    T = tx * ty
    keys = binned_tiles(exp['kind'], exp['rec'], H, W)
    keys = keys[np.random.default_rng(seed).permutation(len(keys))]   # atomic order
    large = [list(np.nonzero((exp['kind'][b] == KIND_LARGE) | (exp['kind'][b] == KIND_HARD))[0]) for b in range(B)]
    for key in keys:
        b, t, f = int(key // F // T), int(key // F % T), int(key % F)
        pos = view['tile_count'][b, t]
        view['tile_count'][b, t] += 1
        if pos < BIN_CAP:
            view['bins'][b, t, pos] = f
            continue
        row = b * ty + t // tx
        q = view['ovf_count'][b, t // tx]
        view['ovf_count'][b, t // tx] += 1
        if q < OVF_ROW_CAP:
            view['ovf'][row, q] = (t, f)
        elif not view['face_in_large'][b, f]:
            view['face_in_large'][b, f] = 1
            large[b].append(f)
    for b in range(B):
        order = np.random.default_rng(seed + b).permutation(len(large[b]))
        view['large_list'][b, :len(large[b])] = np.asarray(large[b], np.int64)[order]
        view['large_count'][b] = len(large[b])
    if face_ids is not None:
        view['tile_flags'][:] = tile_flags_of(face_ids, H, W)
    view['header']['tag'] = tag
    return ws
