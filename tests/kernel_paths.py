"""Scenes that drive the CUDA kernels down their rarely taken code paths, and numpy restatements of the rules by which
the kernels pick those paths.

CPU only (numpy and the CPU oracle, no torch.cuda).  The predicates work from the oracle's face ids and sizes and restate
the dispatch of dirt_b200/csrc/backward.cu and raster.cu; each docstring names the lines it mirrors.
tests/test_kernel_paths.py shows on the CPU that every scene of tests/test_gpu_paths.py reaches the path it is there
for; tests/test_gpu_paths.py runs the same scenes on the GPU against the oracle.
"""
import numpy as np

BWD_TILE = 8            # backward.cu TILE: one warp per 8x8 tile
HALO_COLS = 12          # backward.cu HALO_COLS
SLOTS_C4 = 24           # DIRT_BWD_SLOTS_C4: face-table slots of the fused C = 4 launch
SLOTS_C3 = 32           # DIRT_BWD_SLOTS_C3: slots of every launch of one 3- or 1-wide group
SHADE_MAX_CHANNELS = 4  # common.cuh: shading records exist for C <= 4 ...
SHADE_MAX_EXTENT = 65536  # ... and frames up to 65536 x 65536 (16-bit reference pixel)
RASTER_TILE_W, RASTER_TILE_H = 16, 8
SMALL_TILE_LIMIT = 16   # common.cuh: faces whose bounding box spans more tiles go to the image's large list
BIN_CAP = 128           # common.cuh: references a tile's bin holds before the row's overflow list takes the rest
GRID_Z_LIMIT = 65535    # images per launch along gridDim.z


# ---- scene generators --------------------------------------------------------------------------------------------------

def clip_vertices(px, py, z_ndc, w, H, W):
    """Clip-space vertices [n,4] float32 of points in pixel coordinates (x to the right, y down, pixel (col, row) has its
    centre at (col + 0.5, row + 0.5)) at NDC depth z_ndc and clip w."""
    px, py = np.asarray(px, np.float64), np.asarray(py, np.float64)
    x = px / W * 2.0 - 1.0
    y = 1.0 - py / H * 2.0
    w = np.broadcast_to(np.asarray(w, np.float64), x.shape)
    z = np.broadcast_to(np.asarray(z_ndc, np.float64), x.shape)
    return np.stack([x * w, y * w, z * w, w], axis=-1).astype(np.float32)


def _batch(images, H, W, channels, rng):
    """Stack per-image (vertices [V,4], faces [F,3]) into a scene with random background and vertex colours."""
    verts = np.stack([v for v, _ in images]).astype(np.float32)
    faces = np.stack([f for _, f in images]).astype(np.int32)
    B, V = verts.shape[:2]
    return dict(background=rng.uniform(size=(B, H, W, channels)).astype(np.float32), vertices=verts,
                vertex_colors=rng.uniform(-1.0, 1.0, size=(B, V, channels)).astype(np.float32), faces=faces)


def fan(H, W, centres, n, channels, batch=1, radius=9.0, seed=0):
    """`n` thin wedges around each of `centres` (pixel coordinates), random z and w per vertex, random colours.  All
    wedges meet at the centre, so the backward tile holding it sees up to n distinct faces in its face table; a fan on
    a frame corner shows a quarter of its wedges, one on an edge half.  `n` may be one count for every centre or one
    per centre.  Image b of a batch turns its wedges by a different angle and draws other depths; odd images put every
    vertex at w = 1, so that neighbouring faces tie exactly in clip_w."""
    rng = np.random.default_rng(seed)
    counts = [n] * len(centres) if np.isscalar(n) else list(n)
    images = []
    for b in range(batch):
        pts, faces = [], []
        for (cx, cy), k in zip(centres, counts):
            base = len(pts)
            pts.append((cx, cy))
            a = 2.0 * np.pi * np.arange(k) / k + 0.01 + 0.37 * b / k
            pts += list(zip(cx + radius * np.cos(a), cy + radius * np.sin(a)))
            faces += [(base, base + 1 + i, base + 1 + (i + 1) % k) for i in range(k)]
        p = np.array(pts)
        z, w = rng.uniform(-0.5, 0.5, len(p)), rng.uniform(0.8, 1.2, len(p))
        if b % 2 == 1:
            w[:] = 1.0   # clip_w exactly 1 everywhere: the dilation's strict "nearer" test meets exact ties
        v = clip_vertices(p[:, 0], p[:, 1], z, w, H, W)
        images.append((v, np.array(faces)))
    return _batch(images, H, W, channels, rng)


def full_coverage_mesh(batch, H, W, channels, cell=3.0, seed=0):
    """A jittered grid of `cell`-pixel quads, two triangles each, that covers the whole frame and a margin around it.
    Every face has its own three vertices with random colours and depths, so colour and depth jump across every edge
    and the Scharr sums are non-zero everywhere, the frame border and the last pixel of each image included.  Each image
    of a batch has its own jitter."""
    rng = np.random.default_rng(seed)
    xs = np.arange(-cell, W + 2 * cell, cell)
    ys = np.arange(-cell, H + 2 * cell, cell)
    nx, ny = len(xs), len(ys)
    images = []
    for _ in range(batch):
        gx = xs[None, :] + rng.uniform(-0.3, 0.3, (ny, nx)) * cell
        gy = ys[:, None] + rng.uniform(-0.3, 0.3, (ny, nx)) * cell
        idx = np.arange(ny * nx).reshape(ny, nx)
        a, b_, c, d = idx[:-1, :-1].ravel(), idx[:-1, 1:].ravel(), idx[1:, :-1].ravel(), idx[1:, 1:].ravel()
        tris = np.concatenate([np.stack([a, b_, c], 1), np.stack([b_, d, c], 1)])
        corner = tris.ravel()
        v = clip_vertices(gx.ravel()[corner], gy.ravel()[corner], rng.uniform(-0.8, 0.8, corner.size),
                          rng.uniform(0.7, 1.4, corner.size), H, W)
        images.append((v, np.arange(corner.size).reshape(-1, 3)))
    return _batch(images, H, W, channels, rng)


def tie_depth(key=1 << 18):
    """NDC depth whose window depth (z + 1) / 2 lies half-way between depth keys `key` and `key + 1` (a key is the
    window depth in units of 2^-23, common.cuh exact::depth_key), so that rounding errors in a face's depth plane cannot
    change its key.  Exact in float32, and so is z * w for w a power of two."""
    return (2.0 * key + 1.0) / 2.0 ** 23 - 1.0


def coplanar_tie_scene(channels=3, batch=1, seed=0):
    """Faces at one constant depth (tie_depth, clip w a power of two) on 128 x 96 frames, so that every covered pixel
    is a tie of depth keys that the face index alone decides (the lowest index wins).  They come from all three lists of the raster pass:
      - face LARGE_FACE: a triangle over most of the frame, more than SMALL_TILE_LIMIT tiles: the large list;
      - 24 "cover" triangles of about 34 x 18 px, each spanning at most 16 tiles (bins), 12 with lower and 12 with
        higher index than the large face, which is consumed after them;
      - 150 small triangles inside the raster tile of rows 48-55 and columns 48-63, half with lower and half with
        higher index: that tile's bin holds 128 references and the rest sits in its row's overflow list.  They cover
        the tile, so the tile's farthest covered key is the tie key before the large face comes.
    A second image (batch=2) mirrors the layout left to right and swaps the order of the small faces."""
    H, W = 96, 128
    rng = np.random.default_rng(seed)
    z = tie_depth()
    images = []
    for b in range(batch):
        lo_cover, hi_cover, lo_small, hi_small = [], [], [], []
        for i in range(24):
            cx, cy = 14 + (i % 6) * 20 + rng.uniform(-3, 3), 10 + (i // 6) * 24 + rng.uniform(-3, 3)
            tri = [(cx - 17, cy - 9), (cx + 17, cy - 8), (cx - 1, cy + 9)]
            (lo_cover if i % 2 == 0 else hi_cover).append(tri)
        for i in range(150):
            cx, cy = rng.uniform(53, 59), rng.uniform(51, 52.5)
            tri = [(cx - 4, cy - 2.5), (cx + 4, cy - 2), (cx + rng.uniform(-2, 2), cy + 2.5)]
            (lo_small if i % 2 == 0 else hi_small).append(tri)
        if b % 2 == 1:
            lo_small, hi_small = hi_small[::-1], lo_small[::-1]
        large = [(8.0, 6.0), (121.0, 20.0), (40.0, 92.0)]
        polys = lo_small[:40] + lo_cover + lo_small[40:] + [large] + hi_cover + hi_small
        p = np.array(polys, np.float64).reshape(-1, 2)
        if b % 2 == 1:
            p[:, 0] = W - p[:, 0]
        v = clip_vertices(p[:, 0], p[:, 1], z, rng.choice([0.5, 1.0, 2.0], len(p)), H, W)
        images.append((v, np.arange(len(p)).reshape(-1, 3)))
    return _batch(images, H, W, channels, rng)


LARGE_FACE = 87   # index of the large face in coplanar_tie_scene: after 40 + 12 + 35 lower-index faces


def bin_overflow_scene(batch=1, n=1200, second=300):
    """`n` random faces of about 13 x 7 px stacked in the middle of a 96 x 64 frame, C = 3, so that the raster pass's
    three list levels all fill: the busiest tile takes about 1040 references against bins of BIN_CAP, the busiest row
    of tiles about 1580 past its bins against row lists of 1024 entries, and the rest goes to the image's large list.
    With batch=2 the second image keeps its first `second` faces (the rest degenerate): bins and row lists only, with
    the busiest row 185 entries past its bins."""
    rng = np.random.default_rng(12)
    W, H = 96, 64
    tri = rng.uniform(-0.28, 0.28, size=(n, 3, 2)) + np.array([0.1, -0.05])
    z = rng.uniform(-0.8, 0.8, size=(n, 3, 1))
    verts = np.concatenate([tri, z, np.ones((n, 3, 1))], axis=2).reshape(1, n * 3, 4).astype(np.float32)
    s = dict(background=rng.uniform(size=(1, H, W, 3)).astype(np.float32), vertices=verts,
             vertex_colors=rng.uniform(size=(1, n * 3, 3)).astype(np.float32),
             faces=np.arange(n * 3, dtype=np.int32).reshape(1, n, 3))
    if batch == 2:
        s = {k: np.concatenate([v, v], axis=0) for k, v in s.items()}
        s['faces'][1, second:] = 0
    return s


def coverage_masks(vertices, faces, H, W):
    """bool [F,H,W]: the pixels each face of one image covers when drawn alone (the oracle's coverage rule, with no
    depth test involved)."""
    from oracle import oracle
    F = faces.shape[0]
    ids = oracle.visibility(np.broadcast_to(vertices, (F,) + vertices.shape), faces[:, None, :], H, W)[0]
    return ids >= 0


def two_faces_per_image(batch, H, W, channels, seed=0):
    """`batch` images, each with its own two random triangles (any index or stride mistake between images shows up as
    a wrong image).  The triangles are well shaped (corners about 120 degrees apart around their centre, clip w within
    a factor of two): among 65544 images of unconstrained random triangles, slivers put the oracle's own fp32
    interpolation 4x past the 1e-4 bar from fp64 truth, which would hide what this scene is for.  Vectorised for batches past the grid's 65535 images."""
    rng = np.random.default_rng(seed)
    n = min(W, H)
    centre = rng.uniform(-0.2 * n, 1.2 * n, (batch, 2, 1, 2))
    angle = rng.uniform(0, 2 * np.pi, (batch, 2, 1)) + np.array([0.0, 2.0, 4.0]) * np.pi / 3 + \
        rng.uniform(-0.4, 0.4, (batch, 2, 3))
    radius = rng.uniform(0.5 * n, 1.2 * n, (batch, 2, 3))
    px = (centre[..., 0] + radius * np.cos(angle)).reshape(batch, 6)
    py = (centre[..., 1] + radius * np.sin(angle)).reshape(batch, 6)
    v = clip_vertices(px, py, rng.uniform(-0.9, 0.9, (batch, 6)), rng.uniform(0.7, 1.4, (batch, 6)), H, W)
    faces = np.broadcast_to(np.arange(6, dtype=np.int32).reshape(2, 3), (batch, 2, 3)).copy()
    return dict(background=rng.uniform(size=(batch, H, W, channels)).astype(np.float32), vertices=v,
                vertex_colors=rng.uniform(-1.0, 1.0, size=(batch, 6, channels)).astype(np.float32), faces=faces)


def edge_strip(H, W, channels, seed=0):
    """Random triangles in the last 16 columns (W >> H) or rows (H >> W) of a W x H frame, where the 16-bit reference
    pixel of a face's shading record is at its largest, plus one across the whole short side there."""
    rng = np.random.default_rng(seed)
    long_ = max(W, H)
    n = 12
    a = rng.uniform(long_ - 16.5, long_ + 0.5, (n, 3))
    b = rng.uniform(-2.0, min(W, H) + 2.0, (n, 3))
    a = np.concatenate([a, [[long_ - 15.2, long_ - 0.3, long_ - 0.5]]])
    b = np.concatenate([b, [[-1.0, 3.0, min(W, H) + 1.0]]])
    px, py = (a, b) if W > H else (b, a)
    v = clip_vertices(px.ravel(), py.ravel(), rng.uniform(-0.9, 0.9, px.size), rng.uniform(0.5, 2.0, px.size), H, W)
    return _batch([(v, np.arange(px.size).reshape(-1, 3))], H, W, channels, rng)


def big_triangle(H, W, w, channels, seed=0, span=0.95):
    """One triangle over most of the frame whose vertices have clip w = `w` (three values): perspective interpolation
    across it is as uneven as max(w) / min(w)."""
    rng = np.random.default_rng(seed)
    ndc = np.array([[-span, -span], [span, -span * 0.9], [-span * 0.8, span]])
    w = np.asarray(w, np.float64)
    z = np.array([0.0, 0.1, -0.1])
    verts = np.concatenate([ndc * w[:, None], (z * w)[:, None], w[:, None]], 1).astype(np.float32)
    return dict(background=rng.uniform(size=(1, H, W, channels)).astype(np.float32), vertices=verts[None],
                vertex_colors=rng.uniform(0.0, 1.0, (1, 3, channels)).astype(np.float32),
                faces=np.array([[[0, 1, 2]]], np.int32))


def fp64_pixels(vertices, vertex_colors, faces, ids):
    """Perspective-correct interpolation in float64 at the centres of the pixels `ids` [H,W] marks as covered, from one
    image's vertices [V,4], vertex_colors [V,C] and faces [F,3]: solve M^T lam = (x_ndc, y_ndc, 1) with M the rows
    (x, y, w) of the face's vertices, normalise lam to sum 1 and interpolate.  Uncovered pixels are NaN."""
    H, W = ids.shape
    out = np.full((H, W, vertex_colors.shape[-1]), np.nan)
    rows, cols = np.nonzero(ids >= 0)
    xn = (cols + 0.5) / W * 2.0 - 1.0
    yn = 1.0 - (rows + 0.5) / H * 2.0
    fid = ids[rows, cols]
    for f in np.unique(fid):
        sel = fid == f
        v = vertices[faces[f]].astype(np.float64)
        lam = np.linalg.solve(v[:, [0, 1, 3]].T, np.stack([xn[sel], yn[sel], np.ones(int(sel.sum()))]))
        lam /= lam.sum(0, keepdims=True)
        out[rows[sel], cols[sel]] = lam.T @ vertex_colors[faces[f]].astype(np.float64)
    return out


# ---- predicates: which path a call takes -------------------------------------------------------------------------------

def _tile_cells(ids):
    """[B, tiles_y, tiles_x, 96]: the face ids of each backward tile's 64 pixels and its 32-pixel ring (corners excluded),
    -1 outside the frame."""
    B, H, W = ids.shape
    ty, tx = -(-H // BWD_TILE), -(-W // BWD_TILE)
    pad = np.full((B, ty * BWD_TILE + 2, tx * BWD_TILE + 2), -1, np.int64)
    pad[:, 1:H + 1, 1:W + 1] = ids
    cells = [pad[:, r:r + ty * BWD_TILE:BWD_TILE, c:c + tx * BWD_TILE:BWD_TILE]
             for r in range(BWD_TILE + 2) for c in range(BWD_TILE + 2)
             if not (r in (0, BWD_TILE + 1) and c in (0, BWD_TILE + 1))]
    return np.stack(cells, axis=-1)


def tile_distinct_faces(ids):
    """Distinct faces each backward tile puts into its face table, [B, ceil(H/8), ceil(W/8)] from face ids [B,H,W].

    backward.cu:664-666 inserts the ids of the lane's two pixels (id0, id1) and of one ring cell (idr) with slot_of();
    the ring cells are ring_r / ring_c of :571-572, i.e. the 10 x 10 halo without its four corners.  Ids outside the
    frame are -1 (the cp.async staging writes -1 there, :603; TMA staging only serves tiles whose halo is inside the
    frame, :575-576) and take no slot.  A tile with more distinct faces than slots overflows (:668) and runs
    tile_generic."""
    s = np.sort(_tile_cells(ids), axis=-1)
    new = np.ones(s.shape, bool)
    new[..., 1:] = s[..., 1:] != s[..., :-1]
    return ((s >= 0) & new).sum(-1)


def tile_inner(H, W):
    """[tiles_y, tiles_x] `inner` of backward.cu:575: the tile's whole staged halo (12 columns, 10 rows) lies inside the
    frame.  Only such tiles are staged by TMA (:576); the rest, the frame-border tiles, by per-lane cp.async."""
    trow0 = np.arange(-(-H // BWD_TILE))[:, None] * BWD_TILE
    tcol0 = np.arange(-(-W // BWD_TILE))[None, :] * BWD_TILE
    return (tcol0 >= 1) & (trow0 >= 1) & (tcol0 + HALO_COLS - 2 <= W - 1) & (trow0 + BWD_TILE <= H - 1)


def staged_taps(W, width):
    """[tiles_x] `staged_taps` of backward.cu:713 for a launch on a group of `width` channels (4: the fused pair): the
    Scharr taps of the whole tile come from the staged halo.  REACH (:492) is the columns right of a pixel that its taps
    read: 1 for a 3-wide group, 3 when a 1-wide group reads the next two pixels in flat order.  Tiles without it read
    their taps from global memory (scharr_global)."""
    reach = 1 if width == 3 else 3
    tcol0 = np.arange(-(-W // BWD_TILE)) * BWD_TILE
    return tcol0 + BWD_TILE - 1 + reach <= W - 1


def backward_launches(C, groups=None, aligned16=True):
    """The launches of launch_backward (backward.cu:1027-1057) as a list of (kernel width, face-table slots): one fused
    launch for C = 4 grouped {3,1} with 16-byte aligned pixels / grad_pixels / grad_background / grad_vertex_colors,
    otherwise one per channel group."""
    groups = list(groups) if groups else default_groups(C)
    if C == 4 and groups == [3, 1] and aligned16:
        return [(4, SLOTS_C4)]
    return [(g, SLOTS_C3) for g in groups]


def uses_tma(C, W, groups=None, aligned16=True):
    """backward.cu:1036: halos staged by TMA (for the `inner` tiles) iff the call is one launch over whole pixels --
    C = 1, C = 3, or the fused C = 4 -- with W % 4 == 0 and 16-byte aligned pixels and face ids."""
    launches = backward_launches(C, groups, aligned16)
    return len(launches) == 1 and launches[0][0] == C and C in (1, 3, 4) and W % 4 == 0 and aligned16


def raster_instantiation(C, H, W, align=16):
    """(MODE, CT, REC) of the raster_kernel a forward call takes (raster.cu:472-488), `align` being the largest power of
    two that divides the addresses of background, pixels and vertex_colors."""
    rec = C <= SHADE_MAX_CHANNELS and W <= SHADE_MAX_EXTENT and H <= SHADE_MAX_EXTENT   # common.cuh shade_records_ok
    if C == 4 and align % 16 == 0 and rec:
        return (0, 4, True)
    if C == 3 and W % 2 == 0 and align % 8 == 0 and rec:
        return (0, 3, True)
    return (0, 0, rec)


def default_groups(C):
    """The reference's greedy split of C channels into groups of 3, then 1 (api.cu make_groups)."""
    if C in (1, 3):
        return [C]
    out, begin = [], 0
    while begin < C:
        out.append(3 if begin + 3 <= C else 1)
        begin += out[-1]
    return out


def raster_lists(setup_records, H, W):
    """Per face of one image, from oracle.setup_records: 'small' (binned to every raster tile its bounding box touches,
    setup.cu:184), 'large' (the image's large list) or None (culled), and the tiles it is binned to."""
    tiles_x = -(-W // RASTER_TILE_W)
    out = []
    for r in setup_records:
        if r['kind'] == 0:
            out.append((None, []))
            continue
        cmin, rmin, cmax, rmax = r['bbox']
        tx0, tx1, ty0, ty1 = cmin // RASTER_TILE_W, cmax // RASTER_TILE_W, rmin // RASTER_TILE_H, rmax // RASTER_TILE_H
        if r['kind'] == 1 and (tx1 - tx0 + 1) * (ty1 - ty0 + 1) <= SMALL_TILE_LIMIT:
            out.append(('small', [ty * tiles_x + tx for ty in range(ty0, ty1 + 1) for tx in range(tx0, tx1 + 1)]))
        else:
            out.append(('large', []))
    return out


# ---- the scenes of tests/test_gpu_paths.py -----------------------------------------------------------------------------

# face-table overflow matrix: (channels, channel groups) x frame width; W % 4 == 0 lets the one-launch calls stage by TMA
OVERFLOW_CHANNELS = [(1, None), (3, None), (4, None), (4, [1, 3]), (7, None)]
OVERFLOW_WIDTHS = [64, 62]


def overflow_scene(channels, W, seed=0):
    """Two 48 x W images with four fans each: 48 wedges at (20, 20) (an interior tile), 192 on the top-left corner, 112
    on the right edge and 40 near the bottom border -- tiles with more distinct faces than either table size."""
    return fan(48, W, [(20.0, 20.0), (0.3, 0.4), (W - 0.3, 30.0), (44.0, 42.0)], [48, 192, 112, 40], channels, batch=2,
               seed=seed)


def full_table_scene(channels, W, seed=1):
    """Two 48 x W images with fans of 24 and 32 wedges: tiles whose face table is exactly full (every slot taken, the
    hash probe wraps round) for both table sizes, and no tile over either."""
    return fan(48, W, [(20.0, 20.0), (44.0, 28.0)], [24, 32], channels, batch=2, seed=seed)


# flat-order reads of 1-wide groups: (channels, groups) x W = 8k + 0..7, three 16-row images covered edge to edge
FLAT_ORDER_CHANNELS = [(1, None), (4, None), (3, [1, 1, 1]), (4, [1, 3])]
FLAT_ORDER_WIDTHS = list(range(32, 40))
FLAT_ORDER_H = 16


def flat_order_scene(channels, W, seed=0):
    return full_coverage_mesh(3, FLAT_ORDER_H, W, channels, seed=seed)


GRID_LIMIT_BATCH = GRID_Z_LIMIT + 9


def grid_limit_scene():
    """65544 images of 8 x 8, two faces each, C = 4: past the grid's z limit in both kernels."""
    return two_faces_per_image(GRID_LIMIT_BATCH, 8, 8, 4, seed=3)


# shading-record limit: W x 8 and 8 x H frames with W, H at and one past SHADE_MAX_EXTENT
RECORD_LIMIT_FRAMES = [(8, 65536), (8, 65537), (65536, 8), (65537, 8)]   # (H, W)
RECORD_LIMIT_CHANNELS = [1, 3, 4]

# pixels against fp64 truth: clip w of the three vertices of big_triangle
FP64_W = {'1': (1.0, 1.0, 1.0), '1e2': (0.1, 1.0, 10.0), '1e4': (0.01, 1.0, 100.0)}
FP64_W_LOGGED = {'1e6': (0.001, 1.0, 1000.0)}   # measured and reported, not asserted
FP64_SIZES = [512, 2048]
FP64_CHANNELS = [2, 3, 4, 5]
# (H, W, channels, byte offset of background / pixels / colours): every raster_kernel instantiation
FP64_EXTRA = [(512, 512, 3, 4), (512, 512, 4, 4), (8, 65536, 4, 0), (8, 65537, 2, 0), (8, 65537, 3, 0), (8, 65537, 4, 0)]
