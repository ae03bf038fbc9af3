"""Inputs on which the fast (atomic and reduced) gradient paths must return the exact sum of their terms.

If every term of an output element is a multiple of 2^-m and the sum of their magnitudes times 2^m is below 2^24, then
every partial sum, in any order and any grouping, is a multiple of 2^-m below 2^(24-m) in magnitude: an fp32 value.  fp32
addition of such values is exact and associative, so a kernel that adds each term exactly once returns the float64 sum,
bit for bit, whatever order its atomics or reductions take.  A lost, duplicated or misrouted term then shows as a
difference of at least 2^-m in one element, however many terms that element has.

The builders below put every input of a family on a dyadic grid, so that the fp32 evaluation takes exactly the intended
fractions and weights.  `check_exact` proves the condition for every output element of a scene from the float64 terms,
which come from the existing restatements of each operation: examples/textured.py for the texture lookup,
lighting._diffuse_directional for the directional diffuse model, and oracle.visibility's face ids and G-buffer for the
rasteriser (they match the kernel bit for bit under the visibility specification, DESIGN.md section 2.1).
tests/test_exact_sums_host.py checks each scene on the CPU; tests/test_gpu_exact_sums.py compares the kernels with `==`.

Everything here is torch or numpy on any device; nothing needs a GPU."""
import math

import numpy as np
import torch

F64 = torch.float64


# ---- the exactness condition ---------------------------------------------------------------------------------------

def check_exact(terms, index, size, m):
    """terms: float64 [T], the terms of every output element; index: int64 [T], the output element each one goes to;
    size: the number of output elements.  Asserts that every term is a multiple of 2^-m and that sum |t| * 2^m < 2^24 for
    every element.  Returns (the float64 sums, the number of nonzero terms per element)."""
    return check_exact_chunks([(terms, index)], size, m)


def check_exact_chunks(chunks, size, m, device=None):
    """check_exact over the (terms, index) pairs that `chunks` yields, so that a scene's terms need not all be held at
    once."""
    mag = sums = counts = None
    for terms, index in chunks:
        terms = terms.to(F64).reshape(-1)
        index = index.reshape(-1).to(torch.int64)
        if mag is None:
            dev = terms.device if device is None else device
            mag = torch.zeros(size, dtype=F64, device=dev)
            sums = torch.zeros(size, dtype=F64, device=dev)
            counts = torch.zeros(size, dtype=torch.int64, device=dev)
        scaled = terms * 2.0 ** m
        bad = scaled != torch.round(scaled)
        assert not bad.any(), 'a term is not a multiple of 2^-%d: %r' % (m, float(terms[bad][0]))
        index = index.to(mag.device)
        mag.index_add_(0, index, terms.abs().to(mag.device))
        sums.index_add_(0, index, terms.to(mag.device))
        counts.index_add_(0, index, (terms != 0).to(torch.int64).to(mag.device))
    worst = float(mag.max()) * 2.0 ** m if size else 0.0
    assert worst < 2.0 ** 24, 'sum |t| * 2^%d reaches %.0f, not below 2^24' % (m, worst)
    return sums, counts


def check_exact_sums(sums, magnitudes, m):
    """The condition where a restatement gives only each element's sum and, from autograd with |grad_out| (every weight
    of these scenes is >= 0), its sum of magnitudes: asserts that both are multiples of 2^-m and sum |t| * 2^m < 2^24.
    That the terms themselves are multiples of 2^-m is the scene's own claim (its fractions and weights are dyadic),
    which tests/test_exact_sums_host.py checks lookup by lookup."""
    for name, t in (('sum', sums), ('magnitude', magnitudes)):
        scaled = t.to(F64) * 2.0 ** m
        assert (scaled == torch.round(scaled)).all(), 'a %s is not a multiple of 2^-%d' % (name, m)
    worst = float(magnitudes.max()) * 2.0 ** m if magnitudes.numel() else 0.0
    assert worst < 2.0 ** 24, 'sum |t| * 2^%d reaches %.0f, not below 2^24' % (m, worst)


def first_difference(got, want, counts=None):
    """'' if got == want elementwise (as float64, so -0 == +0), else a description of the first differing element."""
    g = got.detach().to(F64).reshape(-1).cpu()
    w = want.detach().to(F64).reshape(-1).cpu()
    assert g.shape == w.shape, (tuple(got.shape), tuple(want.shape))
    diff = (g != w).nonzero()
    if not diff.numel():
        return ''
    i = int(diff[0])
    where = np.unravel_index(i, tuple(want.shape))
    n = '' if counts is None else ', %d terms' % int(counts.reshape(-1)[i])
    return '%d of %d elements differ; first at %s: got %r, want %r%s' % (diff.numel(), g.numel(), tuple(int(x) for x in where),
                                                                      float(g[i]), float(w[i]), n)


def _gen(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def dyadic(shape, values, seed, device='cpu'):
    """A float32 tensor of `shape` whose elements are drawn uniformly from `values` (each one exact in fp32)."""
    v = torch.tensor(values, dtype=torch.float32, device=device)
    return v[torch.randint(0, len(values), tuple(shape), generator=_gen(seed, device), device=device)]


# ---- B. texture lookup, bilinear and nearest (examples/textured.py:sample_texture) -----------------------------------

TEXELS = [k / 4 for k in range(16)]              # texel values: multiples of 1/4 in [0, 4)
GRADS = [-1.0, -0.5, 0.0, 0.5, 1.0]              # grad_out values: multiples of 1/2
QUARTERS = [0.0, 0.25, 0.5, 0.75]                # index fractions
TEXTURE_M = 5   # grad_texture: grad_out (2^-1) * two factors 1 - f or f (2^-2 each); grad_indices: grad_out (2^-1) *
                # a texel difference (2^-2) * 1 - f or f (2^-2)


def texture_indices(H, W, n, seed, device='cpu'):
    """n (row, col) indices: an integer in [-3H, 3H) x [-3W, 3W) plus a fraction in {0, 1/4, 1/2, 3/4} per axis."""
    g = _gen(seed, device)
    whole = torch.stack([torch.randint(-3 * H, 3 * H, (n,), generator=g, device=device),
                         torch.randint(-3 * W, 3 * W, (n,), generator=g, device=device)], -1).to(torch.float32)
    return whole + dyadic((n, 2), QUARTERS, seed + 1, device)


def texture_scene(TB, H, W, C, B, N, seed, device='cpu'):
    """texture [TB, H, W, C] (TB = 1: shared by the B items), indices [B, N, 2], grad_out [B, N, C]."""
    return (dyadic((TB, H, W, C), TEXELS, seed, device),
            texture_indices(H, W, B * N, seed + 2, device).reshape(B, N, 2),
            dyadic((B, N, C), GRADS, seed + 3, device))


def _taps(indices, H, W, mode):
    """Per lookup: rows, cols [.., 4] of the four corners (00, 01, 10, 11) and their weights [.., 4], from the
    restatement's fp32 floor and fraction; nearest puts weight 1 on corner 00 and 0 elsewhere.  Non-finite lookups get
    weight 0."""
    ok = torch.isfinite(indices).all(-1)
    ix = torch.where(ok[..., None], indices, torch.zeros_like(indices))
    if mode == 'nearest':
        idx = ix.long()
        r = idx[..., 0].clamp(0, H - 1)[..., None].expand(*idx.shape[:-1], 4)
        c = idx[..., 1].clamp(0, W - 1)[..., None].expand(*idx.shape[:-1], 4)
        w = torch.zeros(idx.shape[:-1] + (4,), dtype=F64, device=indices.device)
        w[..., 0] = 1.0
        return r, c, w * ok[..., None]
    floor = ix.floor()
    frac = (ix - floor).to(F64)                  # the restatement's fp32 fraction
    r0, c0 = floor[..., 0].long() % H, floor[..., 1].long() % W
    r1, c1 = (r0 + 1) % H, (c0 + 1) % W
    fr, fc = frac[..., 0], frac[..., 1]
    r = torch.stack([r0, r0, r1, r1], -1)
    c = torch.stack([c0, c1, c0, c1], -1)
    w = torch.stack([(1 - fc) * (1 - fr), fc * (1 - fr), (1 - fc) * fr, fc * fr], -1)
    return r, c, w * ok[..., None]


def texture_terms(texture_shape, indices, grad_out, mode):
    """The terms grad_out[g, ch] * w_k(g) of grad_texture [TB, H, W, C] -> (terms, index, size)."""
    TB, H, W, C = texture_shape
    B, N = indices.shape[:2]
    r, c, w = _taps(indices, H, W, mode)                                       # [B, N, 4]
    tb = (torch.arange(B, device=indices.device) if TB > 1 else torch.zeros(B, dtype=torch.long, device=indices.device))
    texel = (tb[:, None, None] * H + r) * W + c                                 # [B, N, 4]
    terms = grad_out.to(F64)[:, :, None, :] * w[..., None]                      # [B, N, 4, C]
    index = texel[..., None] * C + torch.arange(C, device=indices.device)
    return terms.reshape(-1), index.reshape(-1), TB * H * W * C


def texture_index_terms(texture, indices, grad_out, mode):
    """The terms of grad_indices [B, N, 2]: per channel go * (t01 - t00) * (1 - fr), go * (t11 - t10) * fr to the column
    and go * (t10 - t00) * (1 - fc), go * (t11 - t01) * fc to the row.  Nearest has none (all zero).
    -> (terms, index, size)."""
    TB, H, W, C = texture.shape
    B, N = indices.shape[:2]
    dev = indices.device
    if mode == 'nearest':
        return torch.zeros(1, dtype=F64, device=dev), torch.zeros(1, dtype=torch.long, device=dev), B * N * 2
    r, c, _ = _taps(indices, H, W, mode)
    ok = torch.isfinite(indices).all(-1)
    frac = torch.where(ok[..., None], indices - indices.floor(), torch.zeros_like(indices)).to(F64)
    fr, fc = frac[..., 0:1], frac[..., 1:2]
    tex = texture.to(F64)
    tb = torch.arange(B, device=dev) if TB > 1 else torch.zeros(B, dtype=torch.long, device=dev)
    t = tex[tb[:, None, None], r, c]                                            # [B, N, 4, C]
    go = grad_out.to(F64) * ok[..., None]
    col = torch.stack([go * (t[:, :, 1] - t[:, :, 0]) * (1 - fr), go * (t[:, :, 3] - t[:, :, 2]) * fr], -1)
    row = torch.stack([go * (t[:, :, 2] - t[:, :, 0]) * (1 - fc), go * (t[:, :, 3] - t[:, :, 1]) * fc], -1)
    g = torch.arange(B * N, device=dev).reshape(B, N, 1, 1)
    terms = torch.cat([row, col], -1)                                           # [B, N, C, 4]: row, row, col, col
    index = (g * 2 + torch.tensor([0, 0, 1, 1], device=dev)).expand(B, N, C, 4)
    return terms.reshape(-1), index.reshape(-1), B * N * 2


def texture_expected(texture, indices, grad_out, mode, chunk=None):
    """(grad_texture, its term counts, grad_indices, its term counts), exact, after proving the condition.  With
    `chunk`, the terms are formed `chunk` lookups at a time and the sums kept on the CPU."""
    B, N = indices.shape[:2]
    step = N if chunk is None else chunk
    cpu = None if chunk is None else 'cpu'
    parts = lambda: ((indices[:, s:s + step], grad_out[:, s:s + step], s) for s in range(0, N, step))
    gt, nt = check_exact_chunks(((t, i) for t, i, _ in (texture_terms(tuple(texture.shape), ix, go, mode)
                                                       for ix, go, _ in parts())), texture.numel(), TEXTURE_M, cpu)
    offset = lambda i, s, n: (i // (2 * n)) * 2 * N + s * 2 + i % (2 * n)   # an index of a slice [B, n, 2] into [B, N, 2]
    gi, ni = check_exact_chunks(((t, offset(i, s, ix.shape[1])) for (t, i, _), ix, s in
                                 ((texture_index_terms(texture, ix, go, mode), ix, s) for ix, go, s in parts())),
                                B * N * 2, TEXTURE_M, cpu)
    return gt.reshape(texture.shape), nt.reshape(texture.shape), gi.reshape(indices.shape), ni.reshape(indices.shape)


# Warp patterns of the texture backward pass's aggregation (common.cuh agg_plan / agg_sum).  For each corner of a
# bilinear lookup the lanes of a warp that hit the same texel with a nonzero weight form a group.  agg_plan has each
# leader pull its members one by one when (largest group - 1) <= 5 * (groups of two or more), and otherwise runs one
# butterfly over the warp per group.  A pattern lists its group sizes; 'x' is an invalid (NaN) lane and 'z' a lane whose
# fractions are 0 (three of its four corner weights are zero).  Lanes not listed are singletons.
WARP_PATTERNS = {
    'one32': [32],
    'six': [6],                    # 5 <= 5: pull
    'seven': [7],                  # 6 > 5: butterfly
    'six_pair': [6, 2],
    'seven_pair': [7, 2],
    'eleven_pair': [11, 2],        # 10 <= 10: pull
    'twelve_pair': [12, 2],        # 11 > 10: butterfly, two leaders
    'halves': [16, 16],            # butterfly, two leaders
    'pairs': [2] * 16,
    'mixed': [2, 3, 'x', 'x', 'z', 'z', 'z', 'x'],
}


def agg_pull(sizes):
    """agg_plan's rule for a warp whose groups have `sizes` (singletons included): None when no group has two lanes (no
    aggregation), True for pull, False for one butterfly per group."""
    groups = sum(1 for s in sizes if s > 1)
    if not groups:
        return None
    return max(sizes) - 1 <= 5 * groups


def warp_pattern_indices(pattern, warps, H, W, seed, device='cpu'):
    """Indices [warps * 32, 2] into an H x W texture (H, W >= 8, H * W >= 128) in which every warp has the group
    structure of WARP_PATTERNS[pattern], its lanes shuffled.  Members of a group share the base texel and take
    fractions in {1/4, 1/2, 3/4} (nonzero weights on all four corners); groups sit on distinct bases two texels apart
    in both axes, so no corner of one group meets a corner of another.  Each warp places its groups at other bases."""
    spec = WARP_PATTERNS[pattern]
    rng = np.random.default_rng(seed)
    slots = [(2 * i, 2 * j) for i in range(H // 2 - 1) for j in range(W // 2 - 1)]
    assert len(slots) >= 32
    out = np.empty((warps, 32, 2), np.float32)
    for w in range(warps):
        kinds = []
        for s in spec:
            kinds += [s] * s if isinstance(s, int) else [s]
        kinds += [1] * (32 - len(kinds))
        bases = rng.permutation(len(slots))
        lanes, g = [], 0
        k = 0
        while k < len(kinds):
            s = kinds[k]
            r, c = slots[bases[g]]
            g += 1
            if s == 'x':
                lanes.append((np.nan, np.nan))
                k += 1
            elif s == 'z':
                lanes.append((r, c))
                k += 1
            else:
                for _ in range(s):
                    fr, fc = rng.choice([0.25, 0.5, 0.75], 2)
                    lanes.append((r + fr, c + fc))
                k += s
        out[w] = np.asarray(lanes, np.float32)[rng.permutation(32)]
    return torch.from_numpy(out.reshape(warps * 32, 2)).to(device)


def warp_sides(indices, H, W):
    """agg_pull of every (warp, corner) of bilinear lookups [warps * 32, 2] into an H x W texture, from the texel keys
    and nonzero weights as texel_grad_level forms them -> list per warp of the four corners' sides."""
    r, c, w = _taps(indices, H, W, 'bilinear')
    key = (r * W + c).cpu().numpy().reshape(-1, 32, 4)
    on = (w != 0).cpu().numpy().reshape(-1, 32, 4)
    sides = []
    for wk in range(key.shape[0]):
        per = []
        for k in range(4):
            live = key[wk, on[wk, :, k], k]
            sizes = list(np.unique(live, return_counts=True)[1]) + [1] * int((~on[wk, :, k]).sum())
            per.append(agg_pull(sizes))
        sides.append(per)
    return sides


# ---- F. diffuse_directional (lighting._diffuse_directional) --------------------------------------------------------

NORMAL_VALUES = [-1.0, -0.5, 0.0, 0.5, 1.0]
LIGHT_VALUES = [-0.75, -0.5, -0.25, 0.25, 0.5, 0.75]
COLOUR_VALUES = [0.25, 0.5, 0.75, 1.0]
POINT_GRADS = [-1.0, 0.0, 1.0]
DIFFUSE_M = 5   # light direction: grad_out (1) * light colour (2^-2) * colour (2^-2) * normal (2^-1); light colour:
                # grad_out (1) * |cos| (normal 2^-1 * light 2^-2) * colour (2^-2)


def diffuse_scene(lead, V, C, per_item, seed, device='cpu', sparse=1):
    """Inputs of diffuse_directional on dyadic grids: normals [*, V, 3], colours [*, V, C], light direction and colour
    ([*, 3], [*, C] per item, else [3], [C]), and grad_out [*, V, C] of which all but one in `sparse` points are zero
    (to keep a shared parameter's sum over millions of points inside the condition)."""
    lead = tuple(lead)
    x = dict(n=dyadic(lead + (V, 3), NORMAL_VALUES, seed, device),
             k=dyadic(lead + (V, C), COLOUR_VALUES, seed + 1, device),
             L=dyadic((lead if per_item else ()) + (3,), LIGHT_VALUES, seed + 2, device),
             lc=dyadic((lead if per_item else ()) + (C,), COLOUR_VALUES, seed + 3, device))
    g = dyadic(lead + (V, C), POINT_GRADS, seed + 4, device)
    if sparse > 1:
        keep = torch.randint(0, sparse, lead + (V, 1), generator=_gen(seed + 5, device), device=device) == 0
        g = g * keep
    return x, g


def diffuse_terms(x, g, double_sided=True):
    """Per point, the terms of the light direction's gradient, -(gc * n_i) with gc = sum_c g_c l_c k_c * d|cos|/dcos,
    and of the light colour's, g_c * |cos| * k_c, as autograd of the restatement forms them -> {'L': (terms, index, size),
    'lc': (terms, index, size)}, each index over the flattened parameter ([*, 3] / [*, C] per item, else [3] / [C])."""
    n, k, L, lc = (x[key].to(F64) for key in ('n', 'k', 'L', 'lc'))
    g = g.to(F64)
    lead = n.shape[:-2]
    per_item = L.dim() > 1
    cos = (n * -L[..., None, :]).sum(-1, keepdim=True)                           # [*, V, 1]
    if double_sided:
        f, dcos = cos.abs(), torch.sign(cos)
    else:
        f, dcos = cos.clamp(min=0), (cos > 0).to(F64)
    lcb = lc[..., None, :] if lc.dim() > 1 else lc
    gc = (g * lcb * k).sum(-1, keepdim=True) * dcos                               # [*, V, 1]
    tL = -(gc * n)                                                                # [*, V, 3]
    tlc = g * f * k                                                               # [*, V, C]
    B = math.prod(lead)
    V, C = n.shape[-2], k.shape[-1]
    out = {}
    for name, t, width in (('L', tL, 3), ('lc', tlc, C)):
        t = t.reshape(B, V, width)
        col = torch.arange(width, device=t.device)
        item = torch.arange(B, device=t.device)[:, None, None] if per_item else torch.zeros(1, 1, 1, dtype=torch.long,
                                                                                             device=t.device)
        index = (item * width + col).expand(B, V, width)
        out[name] = (t.reshape(-1), index.reshape(-1), (B if per_item else 1) * width)
    return out


def diffuse_expected(x, g, double_sided=True, items=None):
    """{'L': (sums, counts), 'lc': (sums, counts)} shaped like the parameters, after proving the condition.  With
    `items`, the terms are formed that many leading items at a time (leading shape [B] only)."""
    B = x['n'].shape[0]
    step = B if items is None else items
    per_item = x['L'].dim() > 1
    out = {}
    for name in ('L', 'lc'):
        def chunks():
            for s in range(0, B, step):
                part = {k: (v[s:s + step] if (k in ('n', 'k') or per_item) else v) for k, v in x.items()}
                t, i, _ = diffuse_terms(part, g[s:s + step], double_sided)[name]
                yield t, (i + s * x[name].shape[-1]) if per_item else i
        sums, counts = check_exact_chunks(chunks(), x[name].numel(), DIFFUSE_M)
        out[name] = (sums.reshape(x[name].shape), counts.reshape(x[name].shape))
    return out


# ---- A. rasteriser, grad_vertex_colors (oracle.visibility, assemble_grads' undilated colour terms) ---------------------

RASTER_GRADS = [-1.0, 0.0, 1.0]


def _clip(px, py, H, W, z=0.5):
    """Clip-space (x, y, z, 1) of pixel coordinates (col, row from the top-left corner), exact for power-of-two W, H."""
    px, py = np.asarray(px, np.float64), np.asarray(py, np.float64)
    return np.stack([2 * px / W - 1, 1 - 2 * py / H, np.full_like(px, z), np.ones_like(px)], -1).astype(np.float32)


def _right_triangles(squares, leg, H, W, flip):
    """Every square (col, row) of side `leg` split into two right triangles with their own vertices, along the
    diagonal from top-left to bottom-right (flip: the other one) -> vertices [6 * squares, 4], faces [2 * squares, 3]."""
    px, py = [], []
    for (c, r) in squares:
        a, b, cc, d = (c, r), (c + leg, r), (c, r + leg), (c + leg, r + leg)
        tris = [(a, b, d), (a, d, cc)] if flip else [(a, b, cc), (b, d, cc)]
        for t in tris:
            for (x, y) in t:
                px.append(x)
                py.append(y)
    verts = _clip(px, py, H, W)
    faces = np.arange(len(px), dtype=np.int32).reshape(-1, 3)
    return verts, faces


def raster_scene(kind, C, B, seed):
    """A rasteriser scene whose pixel centres all take dyadic barycentrics, with grad_pixels in {-1, 0, 1}:
    'large': a 512 x 512 frame of four 256-pixel squares, eight right triangles of about 32 640 pixels each;
    'tiny': a 64 x 64 frame tiled by 2-pixel squares, 2048 right triangles, so that every backward tile and its ring see
    about 50 faces, more than either face table holds (tile_generic).
    Image b splits its squares along the other diagonal when b is odd.  -> (scene dict as oracle.forward takes it,
    grad_pixels [B, H, W, C] float32, m)."""
    if kind == 'large':
        H = W = 512
        leg = 256
        squares = [(0, 0), (256, 0), (0, 256), (256, 256)]
    elif kind == 'tiny':
        H = W = 64
        leg = 2
        squares = [(c, r) for r in range(0, 64, 2) for c in range(0, 64, 2)]
    else:
        raise ValueError(kind)
    vs, fs = zip(*[_right_triangles(squares, leg, H, W, b % 2 == 1) for b in range(B)])
    rng = np.random.default_rng(seed)
    s = dict(background=rng.integers(0, 4, (B, H, W, C)).astype(np.float32) / 4,
             vertices=np.stack(vs), vertex_colors=rng.integers(0, 4, (B, len(vs[0]), C)).astype(np.float32) / 4,
             faces=np.stack(fs))
    gp = np.asarray(RASTER_GRADS, np.float32)[rng.integers(0, len(RASTER_GRADS), (B, H, W, C))]
    m = int(math.log2(leg)) + 1     # pixel centres at (k + 1/2) / leg
    return s, gp, m


def raster_colour_terms(vertices, faces, grad_pixels, ids, gbuf, shared):
    """The terms grad_pixels[b, y, x, ch] * bary_k of every covered pixel, to vertex k of its face (assemble_grads'
    colour splat with the undilated barycentrics) -> (terms, index, size) over grad_vertex_colors [B, V, C], or [V, C]
    summed over the batch when `shared`."""
    B, H, W, C = grad_pixels.shape
    V = vertices.shape[1]
    b, y, x = np.nonzero(ids >= 0)
    f = ids[b, y, x]
    vid = faces[b, f]                                                  # [P, 3]
    bary = gbuf[b, y, x, :3].astype(np.float64)                        # [P, 3]
    gp = grad_pixels[b, y, x].astype(np.float64)                       # [P, C]
    terms = bary[:, :, None] * gp[:, None, :]                          # [P, 3, C]
    row = vid if shared else b[:, None] * V + vid
    index = row[:, :, None] * C + np.arange(C)
    size = (1 if shared else B) * V * C
    return torch.from_numpy(terms.reshape(-1)), torch.from_numpy(index.reshape(-1).astype(np.int64)), size


def raster_expected(s, gp, m, oracle, shared=False):
    """(grad_vertex_colors, term counts) of scene s, exact, after proving the condition; also the face ids and G-buffer."""
    B, H, W, C = gp.shape
    ids, gbuf = oracle.visibility(s['vertices'], s['faces'], H, W)
    sums, counts = check_exact(*raster_colour_terms(s['vertices'], s['faces'], gp, ids, gbuf, shared), m)
    shape = ((1 if shared else B), s['vertices'].shape[1], C)
    return sums.reshape(shape[1:] if shared else shape), counts.reshape(shape[1:] if shared else shape), ids, gbuf


# ---- C. trilinear texture lookup at power-of-two footprints (tests/texture_mip_restatement.py) ------------------------

MIP_M = 13   # level l <= 2: grad_out (2^-1) * bilinear weights at level l (2^-(4 + 2l)) * the pyramid's 1/4 per level (4^-l)


def trilinear_scene(TB, H, W, C, B, N, seed, levels=(0, 1, 2), device='cpu'):
    """texture [TB, H, W, C] (H, W powers of two), indices with quarter fractions, derivatives (2^l, 0, 0, 0) for l
    drawn from `levels` -- a footprint of exactly 2^l texels, so lambda = l and the lookup reads level l alone -- and
    grad_out on a 1/2 grid."""
    tex, idx, gout = texture_scene(TB, H, W, C, B, N, seed, device)
    l = torch.tensor(levels, dtype=torch.float32, device=device)[
        torch.randint(0, len(levels), (B, N), generator=_gen(seed + 5, device), device=device)]
    der = torch.zeros(B, N, 4, device=device)
    der[..., 0] = torch.exp2(l)
    return tex, idx, der, gout


def restatement_grads(restate, table, coords, grad_out, extra=()):
    """float64 autograd of `restate(table, coords, *extra)` weighted by grad_out and by |grad_out| -> (grad of the
    table, grad of the coordinates, the table's sum of term magnitudes)."""
    t = table.detach().double().requires_grad_(True)
    c = coords.detach().double().requires_grad_(True)
    ex = [e.detach().double() for e in extra]
    (restate(t, c, *ex) * grad_out.double()).sum().backward()
    ta = table.detach().double().requires_grad_(True)
    (restate(ta, coords.detach().double(), *ex) * grad_out.double().abs()).sum().backward()
    return t.grad, c.grad, ta.grad


def trilinear_expected(tex, idx, der, gout):
    """(grad_texture, grad_indices) from float64 autograd of the restatement, after check_exact_sums."""
    import texture_mip_restatement as mip
    if tex.shape[0] > 1:
        gt, gi, mag = restatement_grads(mip.sample, tex, idx, gout, (der,))
    else:              # a shared texture: every item's lookups as one list
        gt, gi, mag = restatement_grads(lambda t, i, d: mip.sample(t[0], i, d), tex, idx.reshape(-1, 2),
                                        gout.reshape(-1, gout.shape[-1]), (der.reshape(-1, 4),))
        gi = gi.reshape(idx.shape)
    check_exact_sums(gt, mag, MIP_M)
    return gt, gi


# ---- D. cube-map lookup (tests/cubemap_restatement.py, tests/cubemap_mip_restatement.py) -----------------------------

CUBE_S = 8
CUBE_GRADS = [-3.0, -1.5, 0.0, 1.5, 3.0]   # multiples of 3: the border corners' average of three has an exact adjoint
CUBE_M = 15  # grad_out / 3 (2^-1) * bilinear weights at level k <= 2 (2^-(4 + 2k)) * the blend (2^-2) * 4^-k


def cube_directions(n, seed, device='cpu'):
    """n directions with major axis exactly +-1 and minor axes on a 1/16 grid in (-1, 1): with S = 8, every padded
    coordinate s S + 1/2 is a multiple of 1/4 at level 0 (1/8, 1/16 at levels 1, 2), and lookups reach the border
    texels, the faces' edges and their corners."""
    g = _gen(seed, device)
    axis = torch.randint(0, 3, (n,), generator=g, device=device)
    sign = torch.randint(0, 2, (n,), generator=g, device=device).to(torch.float32) * 2 - 1
    minor = torch.randint(-15, 16, (n, 3), generator=g, device=device).to(torch.float32) / 16
    d = minor.clone()
    d[torch.arange(n, device=device), axis] = sign
    return d


def cube_scene(B, C, N, per_item, seed, device='cpu'):
    """cube map [6, S, S, C] (or [B, 6, S, S, C]) on a 1/4 grid, directions [B, N, 3], lod [B, N] on a 1/4 grid in
    [0, 2], grad_out [B, N, C] in CUBE_GRADS."""
    cube = dyadic(((B,) if per_item else ()) + (6, CUBE_S, CUBE_S, C), TEXELS, seed, device)
    d = cube_directions(B * N, seed + 1, device).reshape(B, N, 3)
    lod = dyadic((B, N), [k / 4 for k in range(9)], seed + 2, device)
    return cube, d, lod, dyadic((B, N, C), CUBE_GRADS, seed + 3, device)


def cube_expected(cube, d, lod, gout, mode):
    """grad of the cube map from float64 autograd of the restatement, after check_exact_sums."""
    import cubemap_mip_restatement as cmm
    import cubemap_restatement as cm
    per_item = cube.dim() == 5
    if not per_item:   # a shared map: every item's lookups as one list
        d, lod, gout = d.reshape(-1, 3), lod.reshape(-1), gout.reshape(-1, gout.shape[-1])
    if mode == 'trilinear':
        restate, extra = cmm.sample, (lod,)
    else:
        restate, extra = (lambda c, x: cm.sample(c, x, mode)), ()
    gc, _, mag = restatement_grads(restate, cube, d, gout, extra)
    check_exact_sums(gc, mag, CUBE_M)
    return gc


# ---- E. shadow map, the map gradient at R = 0 and softness 0 (tests/shadow_reference.py) ------------------------------

SHADOW_M = 5   # grad_out (2^-1) * the two tap weights (2^-2 each)


def shadow_scene(B, N, per_item, S, seed, X=None, Y=None):
    """shadow_reference's dyadic inputs on an S x S map (S a power of two): identity light matrices, points whose map
    coordinates X, Y (in texels) lie on a 1/4 grid, so that every tap fraction is 0, 1/4, 1/2 or 3/4; depths on a 1/16
    grid; grad_out on a 1/2 grid.  X, Y [B, N] choose the points (default: over the map)."""
    g = np.random.default_rng(seed)
    if X is None:
        X = g.integers(0, 4 * S, (B, N)) / 4.
        Y = g.integers(0, 4 * S, (B, N)) / 4.
    p = np.stack([X / (S / 2) - 1, 1 - Y / (S / 2), g.integers(-8, 8, (B, N)) / 16. + 1 / 32.], -1)
    nm = B if per_item else 1
    smap = np.stack([g.uniform(size=(nm, S, S)) < 0.6, g.integers(-8, 8, (nm, S, S)) / 16.], -1)
    M = np.tile(np.eye(4), (nm, 1, 1))
    if not per_item:
        M, smap = M[0], smap[0]
    gout = np.asarray(GRADS)[g.integers(0, len(GRADS), (B, N, 1))]
    return [np.asarray(x, np.float32) for x in (p, M, smap, gout)]


SHADOW_CASES = ['map16', 'small_map', 'one_texel', 'corners']


def shadow_case(name, per_item):
    """The dyadic shadow scenes: points over a 16 x 16 map, 2^18 points on a 4 x 4 map, 20 000 per item
    sharing one base texel, and piles within half a texel of a 16 x 16 map's corners and edges."""
    g = np.random.default_rng(90)
    B = 2
    if name == 'map16':
        return shadow_scene(B, 5000, per_item, 16, 91)
    if name == 'small_map':
        X, Y = np.meshgrid(np.arange(512) % 16 / 4., np.arange(512) // 32 / 4.)
        return shadow_scene(1, X.size, per_item, 4, 92, X.reshape(1, -1), Y.reshape(1, -1))
    if name == 'one_texel':
        X = g.integers(0, 4, (B, 20000)) / 4. + 3.5
        Y = g.integers(0, 4, (B, 20000)) / 4. + 4.5
        return shadow_scene(B, 20000, per_item, 8, 93, X, Y)
    edge = lambda: np.where(g.uniform(size=(B, 6000)) < 0.5, g.integers(0, 2, (B, 6000)) / 4.,
                            16 - g.integers(1, 3, (B, 6000)) / 4.)
    return shadow_scene(B, 6000, per_item, 16, 94, edge(), edge())


def shadow_map_terms(p, M, smap, R, bias, gout):
    """The terms of the map gradient's occupancy channel, g / K * -(w step) per tap (K = (2R + 1)^2, fp32 as the kernels
    form them: shadow_reference.deterministic_map_gradient's terms at softness 0) -> (terms, index, size) over the
    flattened map [nm, SH, SW, 2] (the depth channel takes none)."""
    import shadow_reference as sr
    P, Mf, m, _ = sr._flat(p, M, smap)
    B, N = P.shape[:2]
    nm, SH, SW = m.shape[:3]
    look = sr.lookups(P, Mf, SH, SW)
    f32 = np.float32
    gk = (np.asarray(gout, f32).reshape(B, N) * (f32(1) / f32((2 * R + 1) ** 2))).astype(f32)
    ok, fr, fc, T = look['valid'], look['fr'], look['fc'], 2 * R + 2
    terms, index = [], []
    for i in range(T):
        wr = f32(1) - fr if i == 0 else (fr if i == T - 1 else np.ones_like(fr))
        for k in range(T):
            wc = f32(1) - fc if k == 0 else (fc if k == T - 1 else np.ones_like(fc))
            d32, (mi, r, c) = sr._depth_steps(look, m, R, i, k, bias)
            term = (gk * -((wr * wc).astype(f32) * (d32 > 0).astype(f32))).astype(f32)
            texel = (np.broadcast_to(mi, (B, N)) * SH + r) * SW + c
            terms.append(term[ok])
            index.append(texel[ok] * 2)
    return (torch.from_numpy(np.concatenate(terms).astype(np.float64)), torch.from_numpy(np.concatenate(index)),
            nm * SH * SW * 2)


def shadow_expected(p, M, smap, R, bias, gout):
    sums, counts = check_exact(*shadow_map_terms(p, M, smap, R, bias, gout), SHADOW_M)
    return sums.reshape(np.shape(smap)), counts.reshape(np.shape(smap))
