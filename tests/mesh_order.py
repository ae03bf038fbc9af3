"""A numpy restatement of the mesh kernels of csrc/normals.cu in float32, operation by operation (DESIGN.md §7.3,
§7.14, §7.16), and of the corner adjacency they share with the deterministic rasteriser backward pass.

Every operation of those kernels is an explicitly rounded intrinsic (__fadd_rn, __fmul_rn, __fmaf_rn, __fdiv_rn,
__fsqrt_rn), so numpy's float32 arithmetic with `cubemap_ggx_restatement.fmaf` for the fused multiply-adds gives the
same bits, provided every expression is formed in the kernel's order:
    dot3(a, b)        fma(a.z, b.z, fma(a.y, b.y, a.x b.x))
    normalise(x)      x / (sqrt(dot3(x, x)) + 1e-12f)
    normalise_grad    nr = sqrt(dot3(x, x)), d = nr + 1e-12f, k = nr == 0 ? 0 : -(dot3(g, x) / (d d)) / nr,
                      fma(x, k, g / d)
and every row sum in the row's fixed order (`row_sum`).  The adjacency is the CSR the kernels build: row b*V + v holds
the ids b*3F + k*F + f of the corners k of faces f of table b that name v, in ascending order; a face with an index
outside [0, V) is left out.

Arrays: positions P float32 [B, V, 3], faces int [F, 3] shared by the batch.  Per-corner terms are formed for every
position j of the adjacency's `inc` as arrays [n, B, ...] and summed into rows [V, B, ...]."""
import numpy as np

from cubemap_ggx_restatement import fmaf

LONG_ROW = 32          # NORMALS_LONG_ROW: longer rows are summed by the whole warp
EPS = np.float32(1e-12)
F0 = np.float32(0)
AVERAGE, PRE_SPLIT = 0, 1
UNIFORM, COTANGENT = 0, 1


# ---- the adjacency --------------------------------------------------------------------------------------------------

def adjacency(faces, V, items=1, face_stride=0):
    """(offsets int64 [items*V + 1], inc int64 [corners]) of `items` face tables of F faces each, table b starting
    b*face_stride ints into the flat faces (0: one table for every item).  faces: [F, 3] or [items, F, 3]."""
    faces = np.asarray(faces, np.int64)
    F = faces.shape[-2] if faces.ndim >= 2 else 0
    flat = faces.reshape(-1)
    rows, ids = [], []
    for b in range(items):
        t = flat[b * face_stride:b * face_stride + 3 * F].reshape(F, 3)
        ok = ((t >= 0) & (t < V)).all(1)
        f = np.flatnonzero(ok)
        for k in range(3):
            rows.append(b * V + t[f, k])
            ids.append(b * 3 * F + k * F + f)
    rows = np.concatenate(rows) if rows else np.zeros(0, np.int64)
    ids = np.concatenate(ids) if ids else np.zeros(0, np.int64)
    order = np.argsort(rows * (3 * F * items + 1) + ids, kind='stable')
    offsets = np.zeros(items * V + 1, np.int64)
    offsets[1:] = np.cumsum(np.bincount(rows, minlength=items * V))
    return offsets, ids[order]


# ---- the row sums ---------------------------------------------------------------------------------------------------

def row_sum(offsets, terms, long_row=LONG_ROW):
    """Sums [rows, ...] float32 of the terms [n, ...] (one per position of inc) over each row [offsets[r], offsets[r+1]).
    A row of up to `long_row` terms is summed left to right from +0; a longer one as 32 lane partials (lane l sums the
    terms l, l + 32, ... from +0) joined by the xor butterfly 16, 8, 4, 2, 1 (every lane ends with the same bits, since
    fp32 addition is commutative).  long_row=None sums every row left to right."""
    offsets = np.asarray(offsets, np.int64)
    terms = np.asarray(terms, np.float32)
    lo, n = offsets[:-1], np.diff(offsets)
    out = np.zeros((len(lo),) + terms.shape[1:], np.float32)
    tree = n > long_row if long_row is not None else np.zeros(len(n), bool)
    for r in np.flatnonzero((n > LONG_ROW) & ~tree):   # long rows left to right: ufunc.accumulate is sequential
        zero = np.zeros((1,) + terms.shape[1:], np.float32)
        out[r] = np.add.accumulate(np.concatenate([zero, terms[lo[r]:lo[r] + n[r]]]), axis=0)[-1]
    seq = np.flatnonzero((n > 0) & (n <= LONG_ROW) & ~tree)
    ns = n[seq]
    for j in range(int(ns.max()) if len(seq) else 0):
        live = seq[ns > j]
        out[live] = out[live] + terms[lo[live] + j]
    tall = np.flatnonzero(tree)
    if len(tall):
        lane = np.arange(32)
        acc = np.zeros((len(tall), 32) + terms.shape[1:], np.float32)
        nt = n[tall]
        for m in range(int(-(-nt.max() // 32))):
            r, l = np.nonzero(lane[None, :] + 32 * m < nt[:, None])
            acc[r, l] = acc[r, l] + terms[lo[tall][r] + l + 32 * m]
        for o in (16, 8, 4, 2, 1):
            acc = acc + acc[:, lane ^ o]
        out[tall] = acc[:, 0]
    return out


# ---- fp32 vector arithmetic in the kernels' order ---------------------------------------------------------------------

def dot3(a, b):
    return fmaf(a[..., 2], b[..., 2], fmaf(a[..., 1], b[..., 1], a[..., 0] * b[..., 0]))


def cross3(a, b):
    """torch.linalg.cross: (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0)"""
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def normalise(x):
    d = np.sqrt(dot3(x, x)) + EPS
    return x / d[..., None]


def normalise_grad(x, g):
    """torch autograd's gradient of normalise at x for the output gradient g (none through the norm of 0)."""
    nr = np.sqrt(dot3(x, x))
    d = nr + EPS
    gd = -(dot3(g, x) / (d * d))
    k = np.where(nr == 0, F0, gd / np.where(nr == 0, np.float32(1), nr))
    return fmaf(x, k[..., None], g / d[..., None])


def _negsum(a, b):
    return -(a + b)


# ---- the corners of the adjacency ------------------------------------------------------------------------------------

class Corners:
    """Per position j of inc (items = 1): i = inc[j], corner k = i // F of face f = i % F, its vertex triple tri."""

    def __init__(self, faces, V):
        self.faces = np.asarray(faces, np.int64).reshape(-1, 3)
        self.F, self.V = len(self.faces), V
        self.offsets, self.inc = adjacency(self.faces, V)
        F = max(self.F, 1)
        self.k, self.f = self.inc // F, self.inc % F
        self.tri = self.faces[self.f]
        self.count = np.diff(self.offsets)

    def edges(self, Pt):
        """e1 = p1 - p0, e2 = p2 - p0 [n, B, 3] of each position's face, from positions Pt [V, B, 3]."""
        p0 = Pt[self.tri[:, 0]]
        return Pt[self.tri[:, 1]] - p0, Pt[self.tri[:, 2]] - p0

    def pick(self, g0, g1, g2):
        """corner k's value of each position: g1 (k = 1), g2 (k = 2), -(g1 + g2) (k = 0)"""
        k = self.k.reshape((-1,) + (1,) * (g1.ndim - 1))
        return np.where(k == 1, g1, np.where(k == 2, g2, g0))


def _t(a):
    """[B, V, ...] <-> [V, B, ...]"""
    return np.ascontiguousarray(np.swapaxes(np.asarray(a, np.float32), 0, 1))


# ---- vertex normals (DESIGN.md §7.3) ----------------------------------------------------------------------------------

def face_unit(c, Pt):
    """FaceUnit: u_f of each position's face [n, B, 3]"""
    e1, e2 = c.edges(Pt)
    return normalise(cross3(e1, e2))


def normals_forward(P, faces, mode=AVERAGE):
    P = np.asarray(P, np.float32)
    c, Pt = Corners(faces, P.shape[1]), _t(P)
    if mode == AVERAGE:
        return _t(normalise(row_sum(c.offsets, face_unit(c, Pt))))
    out = np.zeros(Pt.shape, np.float32)
    used = np.flatnonzero(c.count > 0)
    last = c.offsets[used + 1] - 1
    out[used] = face_unit(c, Pt)[last]
    return _t(out)


def normals_sum_grad(c, Pt, Gt):
    """normals_sum_grad_kernel: gs = normalise_grad(s_v, grad_v) [V, B, 3]"""
    return normalise_grad(row_sum(c.offsets, face_unit(c, Pt)), Gt)


def corner_grad(c, Pt, Gt, mode, gs=None):
    """CornerGrad<MODE>: each position's corner gradient [n, B, 3].  Gt is grad_normals [V, B, 3]; gs the average
    mode's sum gradient."""
    e1, e2 = c.edges(Pt)
    gu = np.zeros(e1.shape, np.float32)
    for j in range(3):
        v = c.tri[:, j]
        if mode == AVERAGE:
            gu = gu + gs[v]
        else:
            last = c.inc[c.offsets[v + 1] - 1] == j * c.F + c.f
            gu = np.where(last[:, None, None], gu + Gt[v], gu)
    gn = normalise_grad(cross3(e1, e2), gu)
    g1, g2 = cross3(e2, gn), cross3(gn, e1)
    return c.pick(_negsum(g1, g2), g1, g2)


def normals_backward(P, faces, grad, mode=AVERAGE):
    """grad_vertices [B, V, 3] for grad_normals [B, V, 3]"""
    P = np.asarray(P, np.float32)
    c, Pt, Gt = Corners(faces, P.shape[1]), _t(P), _t(grad)
    if c.F == 0:
        return np.zeros(P.shape, np.float32)
    gs = normals_sum_grad(c, Pt, Gt) if mode == AVERAGE else None
    return _t(row_sum(c.offsets, corner_grad(c, Pt, Gt, mode, gs)))


# ---- vertex tangents (DESIGN.md §7.14) --------------------------------------------------------------------------------

class UvFace:
    """uv_face of each position: edges, uv differences, the sign s of the uv area (0 for 0 and NaN)."""

    def __init__(self, c, Pt, Ut):
        self.e1, self.e2 = c.edges(Pt)
        u0, v0 = Ut[c.tri[:, 0], ..., 0], Ut[c.tri[:, 0], ..., 1]
        self.du1, self.dv1 = Ut[c.tri[:, 1], ..., 0] - u0, Ut[c.tri[:, 1], ..., 1] - v0
        self.du2, self.dv2 = Ut[c.tri[:, 2], ..., 0] - u0, Ut[c.tri[:, 2], ..., 1] - v0
        r = self.du1 * self.dv2 - self.du2 * self.dv1
        self.s = np.where(r > 0, np.float32(1), np.where(r < 0, np.float32(-1), F0)).astype(np.float32)

    def face_u(self):
        """s (e1 dv2 - e2 dv1)"""
        s, dv1, dv2 = self.s[..., None], self.dv1[..., None], self.dv2[..., None]
        return s * (self.e1 * dv2 - self.e2 * dv1)

    def face_v(self):
        """s (e2 du1 - e1 du2)"""
        s, du1, du2 = self.s[..., None], self.du1[..., None], self.du2[..., None]
        return s * (self.e2 * du1 - self.e1 * du2)


def _uv_rows(U, B):
    U = np.asarray(U, np.float32)
    return _t(np.broadcast_to(U, (B,) + U.shape[-2:]) if U.ndim == 2 else U)


def gram(N, t):
    """n = unit(normal), d = n . t, x = t - d n"""
    n = normalise(N)
    d = dot3(n, t)
    return n, d, t - n * d[..., None]


def tangents_forward(P, U, N, faces):
    """[B, V, 4]; U [V, 2] (shared) or [B, V, 2], N [B, V, 3]"""
    P = np.asarray(P, np.float32)
    B = P.shape[0]
    c, Pt = Corners(faces, P.shape[1]), _t(P)
    u = UvFace(c, Pt, _uv_rows(U, B))
    s = row_sum(c.offsets, np.concatenate([normalise(u.face_u()), normalise(u.face_v())], -1))
    n, _, x = gram(_t(N), s[..., :3])
    T = normalise(x)
    w = np.where(dot3(cross3(n, T), s[..., 3:]) < 0, np.float32(-1), np.float32(1))
    return _t(np.concatenate([T, w[..., None]], -1))


def tangent_corner_grad(c, u, gt):
    """TangentCornerGrad: each position's (grad position [n, B, 3], grad v [n, B])"""
    g = np.zeros(u.e1.shape, np.float32)
    for j in range(3):
        g = g + gt[c.tri[:, j]]
    gy = normalise_grad(u.face_u(), g) * u.s[..., None]
    g1, g2 = gy * u.dv2[..., None], gy * (-u.dv1)[..., None]
    gdv2, gdv1 = dot3(gy, u.e1), -dot3(gy, u.e2)
    return c.pick(_negsum(g1, g2), g1, g2), c.pick(_negsum(gdv1, gdv2), gdv1, gdv2)


def tangents_backward(P, U, N, faces, grad, vertices=True, uvs=True, normals=True):
    """(grad_vertices [B, V, 3], grad_uvs [B, V, 2], grad_normals [B, V, 3]) for grad_tangents [B, V, 4], per item
    (shared uvs too); None for an output not asked for."""
    P = np.asarray(P, np.float32)
    B, V = P.shape[:2]
    c, Pt, Nt = Corners(faces, V), _t(P), _t(N)
    if c.F == 0:
        return tuple(np.zeros((B, V, w), np.float32) if want else None
                     for w, want in ((3, vertices), (2, uvs), (3, normals)))
    u = UvFace(c, Pt, _uv_rows(U, B))
    t = row_sum(c.offsets, normalise(u.face_u()))
    n, d, x = gram(Nt, t)
    gx = normalise_grad(x, _t(grad)[..., :3])
    gxn = dot3(gx, n)[..., None]
    out = [None, None, None]
    if normals:
        out[2] = _t(normalise_grad(Nt, gx * (-d)[..., None] - t * gxn))
    if vertices or uvs:
        gp, gv = tangent_corner_grad(c, u, gx - n * gxn)
        s = row_sum(c.offsets, np.concatenate([gp, gv[..., None]], -1))
        if vertices:
            out[0] = _t(s[..., :3])
        if uvs:
            out[1] = _t(np.stack([np.zeros_like(s[..., 3]), s[..., 3]], -1))
    return tuple(out)


# ---- the mesh Laplacian (DESIGN.md §7.16) -----------------------------------------------------------------------------

class Wedge:
    """Each position's corner rotated to q0: v = (f[k], f[k+1], f[k+2]) and its edges; with the cotangents."""

    def __init__(self, c, Pt):
        k = c.k
        self.v = np.stack([c.tri[np.arange(len(k)), (k + j) % 3] for j in range(3)], 1) if len(k) else \
            np.zeros((0, 3), np.int64)
        q0, q1, q2 = (Pt[self.v[:, j]] for j in range(3))
        self.e01, self.e02, self.e12 = q1 - q0, q2 - q0, q2 - q1
        self.n = cross3(self.e01, self.e02)
        self.nn = np.sqrt(dot3(self.n, self.n))
        self.den = self.nn + EPS
        self.c0 = dot3(self.e01, self.e02) / self.den
        self.c1 = -(dot3(self.e12, self.e01) / self.den)
        self.c2 = dot3(self.e02, self.e12) / self.den


def laplacian_terms(w, mode):
    """LaplacianTerm: (S, D) [n, B, 4] of each position's corner"""
    if mode == UNIFORM:
        s = w.e01 + w.e02
        return np.concatenate([s, np.full(s.shape[:-1] + (1,), 2, np.float32)], -1)
    s = w.e01 * w.c2[..., None] + w.e02 * w.c1[..., None]
    return np.concatenate([s, (w.nn / np.float32(3))[..., None]], -1)


def laplacian_forward(P, faces, mode):
    P = np.asarray(P, np.float32)
    c, Pt = Corners(faces, P.shape[1]), _t(P)
    if c.F == 0:
        return np.zeros(P.shape, np.float32)
    s = row_sum(c.offsets, laplacian_terms(Wedge(c, Pt), mode))
    return _t(s[..., :3] / (s[..., 3:] + EPS))


def uniform_den(c):
    """D_u + 1e-12 of every vertex, from the length of its row"""
    return np.float32(2) * c.count.astype(np.float32) + EPS


def uniform_neighbour_grad(c, Gt):
    """UniformNeighbourGrad: g_u / (D_u + 1e-12) summed over the corners j != k of each position's face"""
    den = uniform_den(c)
    g = np.zeros((len(c.k),) + Gt.shape[1:], np.float32)
    for j in range(3):
        u = c.tri[:, j]
        g = np.where((c.k == j)[:, None, None], g, g + Gt[u] / den[u][:, None, None])
    return g


def laplacian_sum_grad(c, Pt, Gt):
    """laplacian_sum_grad_kernel: (g_S, g_D) [V, B, 4]"""
    s = row_sum(c.offsets, laplacian_terms(Wedge(c, Pt), COTANGENT))
    d = s[..., 3] + EPS
    gD = -(dot3(Gt, s[..., :3]) / (d * d))
    return np.concatenate([Gt / d[..., None], gD[..., None]], -1)


def cotangent_corner_grad(c, Pt, gs):
    """CotangentCornerGrad: each position's gradient [n, B, 3] from (g_S, g_D) [V, B, 4]"""
    w = Wedge(c, Pt)
    g0, g1, g2 = (gs[w.v[:, j]] for j in range(3))
    s0, s1, s2 = g0[..., :3], g1[..., :3], g2[..., :3]
    gd = (g0[..., 3] + g1[..., 3]) + g2[..., 3]
    w0, w1, w2 = dot3(s1 - s2, w.e12), -dot3(s2 - s0, w.e02), dot3(s0 - s1, w.e01)
    wc = fmaf(w2, w.c2, fmaf(w1, w.c1, w0 * w.c0))
    gnn = gd / np.float32(3) - wc / w.den
    k = np.where(w.nn == 0, F0, gnn / np.where(w.nn == 0, np.float32(1), w.nn))
    gn = w.n * k[..., None]
    g = (w.e01 + w.e02) * (-(w0 / w.den))[..., None] + w.e12 * ((w1 - w2) / w.den)[..., None]
    g = g + ((s2 - s0) * w.c1[..., None] - (s0 - s1) * w.c2[..., None])
    return g + cross3(gn, w.e12)


def laplacian_backward(P, faces, grad, mode):
    """grad_vertices [B, V, 3] for grad_out [B, V, 3]"""
    P = np.asarray(P, np.float32)
    c, Pt, Gt = Corners(faces, P.shape[1]), _t(P), _t(grad)
    if c.F == 0:
        return np.zeros(P.shape, np.float32)
    if mode == UNIFORM:
        s = row_sum(c.offsets, uniform_neighbour_grad(c, Gt))
        D = np.float32(2) * c.count.astype(np.float32)
        gs = Gt / (D + EPS)[:, None, None]
        return _t(s - gs * D[:, None, None])
    return _t(row_sum(c.offsets, cotangent_corner_grad(c, Pt, laplacian_sum_grad(c, Pt, Gt))))


# ---- edge lengths and normal consistency (DESIGN.md §7.17) ------------------------------------------------------------
#
# One value per face edge, [B, F, 3]: edge k of face f runs from v_k to v_{k+1 mod 3}.  The face passes are one thread
# per (item, face); the vertex passes are the row sums above.

LENGTH, CONSISTENCY = 0, 1


class Partners:
    """for_each_partner of every edge (f, k) of every valid face with v_k != v_{k+1}: the other valid faces g that name
    both ends, each once, in the kernel's order.  It scans the shorter of the two rows (the smaller vertex id's when they
    are equally long) in row order and takes each face at its first corner naming that row's vertex.  Arrays per edge:
    f, k, x = v_k, y = v_{k+1}, count; per partner, in order: edge (its index), slot (its place in the edge's order)
    and g."""

    def __init__(self, c):
        F, faces = c.F, c.faces
        ok = ((faces >= 0) & (faces < c.V)).all(1) if F else np.zeros(0, bool)
        self.valid = ok
        f, k = np.nonzero(np.repeat(ok[:, None], 3, 1))
        x, y = faces[f, k], faces[f, (k + 1) % 3]
        keep = x != y
        self.f, self.k, self.x, self.y = f[keep], k[keep], x[keep], y[keep]
        n = c.count
        lx, ly = n[self.x], n[self.y]
        by_x = (lx < ly) | ((lx == ly) & (self.x < self.y))
        r, o = np.where(by_x, self.x, self.y), np.where(by_x, self.y, self.x)
        length = n[r]
        edge = np.repeat(np.arange(len(r)), length)
        j = c.offsets[r][edge] + np.arange(len(edge)) - np.repeat(np.cumsum(length) - length, length)
        i = c.inc[j]
        kk, g = i // max(F, 1), i % max(F, 1)
        w = faces[g]
        first = ~(((kk > 0) & (w[:, 0] == r[edge])) | ((kk > 1) & (w[:, 1] == r[edge])))
        named = (w == o[edge, None]).any(1)
        take = (g != self.f[edge]) & first & named
        self.edge, self.g = edge[take], g[take]
        self.count = np.bincount(self.edge, minlength=len(r))
        start = np.cumsum(self.count) - self.count
        self.slot = np.arange(len(self.edge)) - start[self.edge]

    def ordered_sum(self, terms, zero):
        """[edges, ...] float32: the sum per edge of terms [partners, ...] in partner order, from `zero`."""
        s = np.broadcast_to(zero, (len(self.f),) + zero.shape).copy()
        for m in range(int(self.slot.max()) + 1 if len(self.slot) else 0):
            at = self.slot == m
            s[self.edge[at]] = s[self.edge[at]] + terms[at]
        return s


def face_units(faces, Pt):
    """unit_of: u_g [F, B, 3] of every face from its own corners (only the valid faces' are used)"""
    f = np.clip(np.asarray(faces, np.int64).reshape(-1, 3), 0, max(len(Pt) - 1, 0))
    p0 = Pt[f[:, 0]]
    return normalise(cross3(Pt[f[:, 1]] - p0, Pt[f[:, 2]] - p0))


def edge_terms_forward(P, faces, mode):
    """edge_terms_forward_kernel: [B, F, 3]; 0 for a face with an invalid index"""
    P = np.asarray(P, np.float32)
    c, Pt = Corners(faces, P.shape[1]), _t(P)
    out = np.zeros((c.F, P.shape[0], 3), np.float32)
    if c.F == 0 or c.V == 0:
        return _t(out)
    ok = ((c.faces >= 0) & (c.faces < c.V)).all(1)
    if mode == LENGTH:
        f = np.flatnonzero(ok)
        for k in range(3):
            d = Pt[c.faces[f, (k + 1) % 3]] - Pt[c.faces[f, k]]
            out[f, :, k] = np.sqrt(dot3(d, d))
        return _t(out)
    p = Partners(c)
    u = face_units(c.faces, Pt)
    s = p.ordered_sum(u[p.g], np.zeros(u.shape[1:], np.float32))
    e = np.flatnonzero(p.count > 0)
    uf = u[p.f[e]]
    out[p.f[e], :, p.k[e]] = np.float32(1) - dot3(uf, s[e]) / p.count[e].astype(np.float32)[:, None]
    return _t(out)


def edge_length_corner_grad(c, Pt, Gt):
    """EdgeLengthCornerGrad: each position's gradient [n, B, 3] for grad_out Gt [F, B, 3]"""
    w = Wedge(c, Pt)
    l1, l2 = np.sqrt(dot3(w.e01, w.e01)), np.sqrt(dot3(w.e02, w.e02))
    G1, G2 = Gt[c.f, :, c.k], Gt[c.f, :, (c.k + 2) % 3]
    k1 = np.where(l1 == 0, F0, G1 / np.where(l1 == 0, np.float32(1), l1))
    k2 = np.where(l2 == 0, F0, G2 / np.where(l2 == 0, np.float32(1), l2))
    return -(w.e01 * k1[..., None] + w.e02 * k2[..., None])


def pair_grad(faces, Gt, g, x, y):
    """pair_grad: [n, B] the sum of grad_out over the edges of faces g that join x and y, in edge order from +0"""
    w = faces[g]
    s = np.zeros((len(g),) + Gt.shape[1:-1], np.float32)
    for k in range(3):
        a, b = w[:, k], w[:, (k + 1) % 3]
        s = np.where((((a == x) & (b == y)) | ((a == y) & (b == x)))[:, None], s + Gt[g, :, k], s)
    return s


def same_pair(v, j, k):
    """whether edges j and k [n] of faces v [n, 3] join the same unordered pair"""
    n = np.arange(len(v))
    a, b, c, d = v[:, j], v[:, (j + 1) % 3], v[n, k], v[n, (k + 1) % 3]
    return ((a == c) & (b == d)) | ((a == d) & (b == c))


def consistency_face_grad(c, Pt, Gt):
    """consistency_face_grad_kernel: dL/dn_f [F, B, 3] of every valid face (0 for the others) for grad_out Gt
    [F, B, 3].  Each distinct unordered pair of f's edges, in edge order, adds -(G_f sum du + sum G_g du) / |P| to
    dL/du_f and G_f + (sum G_g) / |P| to beta, du = u_g - u_f."""
    p = Partners(c)
    u = face_units(c.faces, Pt)
    B = Pt.shape[1]
    zero3, zero = np.zeros((B, 3), np.float32), np.zeros(B, np.float32)
    du = u[p.g] - u[p.f[p.edge]]
    G = pair_grad(c.faces, Gt, p.g, p.x[p.edge], p.y[p.edge])
    s = p.ordered_sum(du, zero3)
    sg = p.ordered_sum(du * G[..., None], zero3)
    gsum = p.ordered_sum(G, zero)
    n = np.maximum(p.count, 1).astype(np.float32)[:, None]
    Gf = pair_grad(c.faces, Gt, p.f, p.x, p.y)
    dgu = (s * Gf[..., None] + sg) / n[..., None]
    dbeta = Gf + gsum / n
    v = c.faces[p.f]
    counted = (p.count > 0) & ~((p.k > 0) & same_pair(v, 0, p.k)) & ~((p.k > 1) & same_pair(v, 1, p.k))
    gu, beta = np.zeros((c.F, B, 3), np.float32), np.zeros((c.F, B), np.float32)
    for k in range(3):   # f's edges in order; at most one per (f, k)
        e = np.flatnonzero(counted & (p.k == k))
        gu[p.f[e]] = gu[p.f[e]] - dgu[e]
        beta[p.f[e]] = beta[p.f[e]] + dbeta[e]
    f = c.faces.clip(0, max(c.V - 1, 0))
    p0 = Pt[f[:, 0]]
    nf = cross3(Pt[f[:, 1]] - p0, Pt[f[:, 2]] - p0)
    d = np.sqrt(dot3(nf, nf)) + EPS
    k = (beta * np.float32(1e-12)) / ((d * d) * d)
    out = normalise_grad(nf, gu) - nf * k[..., None]
    return np.where(p.valid[:, None, None], out, F0)


def consistency_corner_grad(c, Pt, gs):
    """ConsistencyCornerGrad: each position's gradient [n, B, 3] through n = e1 x e2 from dL/dn_f gs [F, B, 3]"""
    e1, e2 = c.edges(Pt)
    gn = gs[c.f]
    g1, g2 = cross3(e2, gn), cross3(gn, e1)
    return c.pick(_negsum(g1, g2), g1, g2)


def edge_terms_backward(P, faces, grad, mode):
    """grad_vertices [B, V, 3] for grad_out [B, F, 3]"""
    P = np.asarray(P, np.float32)
    c, Pt, Gt = Corners(faces, P.shape[1]), _t(P), _t(grad)
    if c.F == 0:
        return np.zeros(P.shape, np.float32)
    if mode == LENGTH:
        return _t(row_sum(c.offsets, edge_length_corner_grad(c, Pt, Gt)))
    return _t(row_sum(c.offsets, consistency_corner_grad(c, Pt, consistency_face_grad(c, Pt, Gt))))


# ---- bit-for-bit comparison -------------------------------------------------------------------------------------------

def first_difference(got, want):
    """None if the float32 arrays are equal bit for bit (any NaN matching any NaN), else a message naming the first
    differing entry and how many differ."""
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    if got.shape != want.shape:
        return 'shape %s, restated %s' % (got.shape, want.shape)
    nan = np.isnan(got) & np.isnan(want)
    bad = np.argwhere((got.view(np.int32) != want.view(np.int32)) & ~nan)
    if bad.size == 0:
        return None
    i = tuple(bad[0])
    return '%d of %d entries differ, first at %s: %r, restated %r' % (len(bad), got.size, list(i), got[i], want[i])


# ---- meshes -------------------------------------------------------------------------------------------------------------
#
# Each returns float32 positions [V, 3] and int32 faces [F, 3].

def icosphere():
    from dirt_b200 import scenes
    v, f = scenes.icosphere(3)
    r = np.random.default_rng(1)
    return (v * (1. + 0.2 * r.standard_normal((v.shape[0], 1)))).astype(np.float32), f


def uv_sphere(columns=224, rows=112):
    """cfg5's sphere by default: poles of valence 224, rows the whole warp sums"""
    from dirt_b200 import scenes
    return scenes.uv_sphere(columns, rows, displacement=0.1)


def fan(n=100000):
    """n faces around vertex 0, the rim turning by the golden angle and rising slowly"""
    i = np.arange(n + 1)
    t = i * (np.pi * (3. - np.sqrt(5.)))
    rim = np.stack([np.cos(t), np.sin(t), -0.3 + 0.6 * i / n], axis=1)
    v = np.concatenate([np.zeros((1, 3)), rim]).astype(np.float32)
    f = np.stack([np.zeros(n), np.arange(1, n + 1), np.arange(2, n + 2)], axis=1).astype(np.int32)
    return v, f


def grid(n=24):
    """An open, gently curved n x n grid: boundary vertices of valence 2 to 4, interior of valence 6."""
    y, x = np.meshgrid(np.linspace(-1, 1, n), np.linspace(-1, 1, n), indexing='ij')
    z = 0.3 * np.sin(2. * x) * np.cos(1.5 * y)
    v = np.stack([x.ravel(), y.ravel(), z.ravel()], axis=1)
    v[:, :2] += 0.01 * np.random.default_rng(2).standard_normal((n * n, 2))
    q = (np.arange(n - 1)[:, None] * n + np.arange(n - 1)[None, :]).ravel()
    f = np.concatenate([np.stack([q, q + 1, q + n + 1], 1), np.stack([q, q + n + 1, q + n], 1)])
    return v.astype(np.float32), f.astype(np.int32)


def odd():
    """An icosphere with unused vertices between the used ones and faces that name one vertex twice."""
    v, f = icosphere()
    r = np.random.default_rng(2)
    V = v.shape[0]
    spread = np.concatenate([v, r.standard_normal((V // 2, 3)).astype(np.float32)])
    perm = r.permutation(spread.shape[0])
    inverse = np.argsort(perm)
    v2, f2 = spread[perm], inverse[f].astype(np.int32)
    repeated = np.array([[f2[i, 0], f2[i, 0], f2[i + 1, 1]] for i in range(0, 60, 3)], np.int32)
    return v2, np.concatenate([f2, repeated])


def degenerate():
    """A noisy grid with, inside it: faces naming a vertex twice (in each position) and three times, collinear and
    zero-area faces (coincident corners), a face with its reversed copy, duplicated faces, non-manifold edges of 3, 4
    and 5 faces, an isolated vertex and vertices named only by faces with an invalid index."""
    v, f = grid(12)
    V = len(v)
    r = np.random.default_rng(3)
    v = v + 0.05 * r.standard_normal(v.shape).astype(np.float32)
    line = np.array([[2., 2., 0.], [2.5, 2., 0.], [3., 2., 0.], [3., 2., 0.]], np.float32)    # collinear, coincident
    wing = (np.array([[0., 0., 1.], [0., 1., 1.], [1., 0., 1.], [0.5, 0.5, 2.], [-0.5, 0.5, 1.5]])
            + 0.1 * r.standard_normal((5, 3))).astype(np.float32)                                 # edge fins
    spare = r.standard_normal((3, 3)).astype(np.float32)        # V+9: isolated; V+10, V+11: named by invalid faces
    v = np.concatenate([v, line, wing, spare])
    L, W = V, V + 4
    extra = [[13, 13, 27], [14, 40, 14], [41, 15, 15], [16, 16, 16], [17, 17, 17],
             [L, L + 1, L + 2], [L + 2, L + 3, 50], [L + 3, L + 2, 51], [L, L + 1, L + 1],
             [60, 61, 73], [60, 73, 61], [80, 81, 93], [80, 81, 93], [80, 81, 93],
             [W, W + 1, W + 2], [W + 1, W, W + 3], [W, W + 1, W + 4], [W + 1, W, 100], [W, W + 1, 101],
             [V + 10, V + 11, -1], [V + 11, V + 10 + 3, 5]]
    return v, np.concatenate([f, np.array(extra)]).astype(np.int32)


def folded():
    """A strip folded back onto itself: the fold's vertices sum face normals that nearly cancel."""
    n = 16
    x = np.linspace(-1., 1., n)
    y = np.linspace(0., 1., 5)
    xx, yy = np.meshgrid(x, y, indexing='ij')
    fold = np.where(xx > 0, -xx + 1e-3 * xx, xx)
    z = np.where(xx > 0, 1e-4 + 1e-3 * xx, 0.)
    v = np.stack([fold.ravel(), yy.ravel(), z.ravel()], 1)
    v += 1e-5 * np.random.default_rng(4).standard_normal(v.shape)
    q = (np.arange(n - 1)[:, None] * 5 + np.arange(4)[None, :]).ravel()
    f = np.concatenate([np.stack([q, q + 5, q + 6], 1), np.stack([q, q + 6, q + 1], 1)])
    return v.astype(np.float32), f.astype(np.int32)


def slivers():
    """Cotangent slivers: near-flat triangles with one corner of nearly 180 degrees, some of them exactly flat."""
    r = np.random.default_rng(5)
    m = 40
    a = r.standard_normal((m, 3))
    b = a + r.standard_normal((m, 3))
    t = r.uniform(0.2, 0.8, (m, 1))
    c = a + t * (b - a) + np.where(np.arange(m)[:, None] % 4 == 0, 0., 1e-3) * r.standard_normal((m, 3))
    v = np.stack([a, b, c], 1).reshape(-1, 3)
    i = np.arange(m)[:, None] * 3
    f = np.concatenate([i + [0, 1, 2], (i + [2, 1, 5])[:-1] % (3 * m)])
    return v.astype(np.float32), f.astype(np.int32)


def hubs(V, centres, valence, seed=6):
    """V vertices at random positions and, around each centre vertex c with valence[c] faces, a fan whose rim walks
    the other vertices in a random order: rows of exactly the given lengths for the centres (and long rows on the
    rims too)."""
    r = np.random.default_rng(seed)
    v = r.standard_normal((V, 3)).astype(np.float32)
    f = []
    others = np.setdiff1d(np.arange(V), centres)
    for c in centres:
        rim = r.choice(others, valence[c] + 1, replace=len(others) < valence[c] + 1)
        for j in range(valence[c]):
            a, b = rim[j], rim[j + 1]
            if a == b:
                b = others[(np.searchsorted(others, a) + 1) % len(others)]
            f.append([c, a, b] if j % 2 else [b, c, a])
    return v, np.array(f, np.int32)


def rows_32_33():
    """Vertex 3 names exactly 32 corners, vertex 7 exactly 33: either side of NORMALS_LONG_ROW."""
    return hubs(200, [3, 7], {3: 32, 7: 33})


def full_warp():
    """Vertices 0..31, one warp, all with rows of 33 to 64 corners."""
    return hubs(400, list(range(32)), {c: 33 + c for c in range(32)})


def straddle():
    """V = 45: with B = 3, the warps over the rows b*V + v straddle the items, with long rows on either side of each
    boundary, and the last warp (rows 128..134) is partly empty with long rows in it."""
    centres = [0, 1, 5, 18, 31, 32, 33, 40, 44]
    return hubs(45, centres, {c: 33 + 3 * j for j, c in enumerate(centres)})


def seamed_sphere(columns=224, rows=112):
    """A uv sphere whose seam column is split, with its spherical uvs: float32 positions [V, 3], uvs [V, 2] and int32
    faces [F, 3] (poles of valence `columns`)."""
    u = np.arange(columns + 1) / columns
    v = np.arange(rows + 1) / rows
    uu, vv = np.meshgrid(u, v)
    phi, theta = 2 * np.pi * uu, np.pi * vv
    p = np.stack([np.sin(theta) * np.sin(phi), np.cos(theta), np.sin(theta) * np.cos(phi)], -1).reshape(-1, 3)
    uv = np.stack([uu, vv], -1).reshape(-1, 2)
    i = np.arange(rows)[:, None] * (columns + 1) + np.arange(columns)[None, :]
    a, b, c, d = i, i + 1, i + columns + 1, i + columns + 2
    f = np.concatenate([np.stack([a, c, b], -1)[1:], np.stack([b, c, d], -1)[:-1]]).reshape(-1, 3)
    return p.astype(np.float32), uv.astype(np.float32), f.astype(np.int32)


def uv_for(v):
    """uvs from the positions (a planar projection), float32"""
    return (0.5 + 0.4 * v[:, :2] + 0.1 * v[:, 2:] * v[:, :1]).astype(np.float32)


def tangent_cases():
    """A grid with uvs, whose faces include: zero uv area with collinear uvs and with identical uvs, mirrored uvs, and
    a face tangent parallel to its vertex's normal; returns (positions, uvs, faces, normals) with one zero normal."""
    v, f = grid(10)
    uv = uv_for(v)
    mirrored = np.arange(0, len(f), 7)
    f[mirrored] = f[mirrored][:, [0, 2, 1]]      # reversed winding, same uvs: s flips
    uv[[11, 12, 13]] = uv[11] + np.array([[0., 0.], [0.1, 0.05], [0.2, 0.1]], np.float32)    # collinear uvs
    uv[[30, 31]] = uv[29]                                                                     # identical uvs
    f = np.concatenate([f, [[11, 12, 13], [29, 30, 31]]]).astype(np.int32)
    from dirt_b200 import lighting
    import torch
    n = lighting._vertex_normals(torch.tensor(v[None].astype(np.float64)), torch.tensor(f)).numpy()[0]
    n = n + 0.05 * np.random.default_rng(7).standard_normal(n.shape)
    n[5] = 0.                                           # a zero normal input
    n = n.astype(np.float32)
    # vertex 45's normal along its first face's tangent: T = unit(t - (n . t) n) is then (nearly) 0
    c = Corners(f, len(v))
    u = UvFace(c, _t(v[None]), _t(uv[None]))
    j = c.offsets[45]
    n[45] = normalise(u.face_u())[j, 0]
    return v, uv, f, n
