"""The seamless cube-map lookup of sample_cubemap (DESIGN.md §7.10) restated in torch.  It is the specification: in
float32 on the GPU the CUDA forward equals `sample` bit for bit, and the gradients are torch autograd's of `sample`.

Every fp32 step below is one IEEE-rounded torch operation, in the order written:
    face      the component of largest magnitude, ties to x over y over z (exact comparisons of |x|, |y|, |z|), the
              face + or - by its sign; faces +X, -X, +Y, -Y, +Z, -Z are 0 .. 5
    sc, tc    the OpenGL table (FACE_AXES), ma = |major component|
    s, t      (sc / ma + 1) * 0.5, (tc / ma + 1) * 0.5
    bilinear  pr = (t * S - 0.5) + 1, pc = (s * S - 0.5) + 1 on the padded face (S + 2 square); r0 = floor(pr),
              fr = pr - r0 (likewise c0, fc) and examples/textured.py's blend of padded texels (r0, c0) .. (r0+1, c0+1):
              t00*(1-fc)*(1-fr) + t01*fc*(1-fr) + t10*(1-fc)*fr + t11*fc*fr
    nearest   the face texel (clamp(floor(t * S), 0, S-1), clamp(floor(s * S), 0, S-1))
A zero or non-finite direction returns 0 and passes no gradient.

The padded faces (`atlas`): texel (i, j), 0 <= i, j < S + 2, of face f is face texel (i - 1, j - 1) inside; a border
texel with one coordinate outside 1 .. S is the texel of the adjacent face that holds the projection of the direction
through its centre (`border_table`, float64); a border corner is ((own corner texel + row-neighbour border texel) +
column-neighbour border texel) / 3 in fp32."""
import numpy as np
import torch

# face -> (major axis, (sc axis, sign), (tc axis, sign))
FACE_AXES = [(0, (2, -1), (1, -1)), (0, (2, 1), (1, -1)), (1, (0, 1), (2, 1)),
             (1, (0, 1), (2, -1)), (2, (0, 1), (1, -1)), (2, (0, -1), (1, -1))]


def _face_np(d):
    a = np.abs(d)
    if a[0] >= a[1] and a[0] >= a[2]:
        return 0 if d[0] > 0 else 1
    if a[1] >= a[2]:
        return 2 if d[1] > 0 else 3
    return 4 if d[2] > 0 else 5


def _direction_of(f, sc, tc):
    """The point (sc, tc) of face f's plane (|major| = 1) as a direction, float64."""
    a, (js, ss), (jt, st) = FACE_AXES[f]
    d = np.zeros(3)
    d[a] = 1.0 if f % 2 == 0 else -1.0
    d[js] = ss * sc
    d[jt] = st * tc
    return d


def border_source(f, i, j, S):
    """(face, row, col) of the cube texel that border texel (i, j) of face f's padded face copies (exactly one of i, j
    outside 1 .. S): the texel holding the projection of the direction through the border texel's centre."""
    d = _direction_of(f, 2.0 * (j - 0.5) / S - 1.0, 2.0 * (i - 0.5) / S - 1.0)
    g = _face_np(d)
    a, (js, ss), (jt, st) = FACE_AXES[g]
    ma = abs(d[a])
    s, t = (ss * d[js] / ma + 1.0) * 0.5, (st * d[jt] / ma + 1.0) * 0.5
    return g, min(max(int(np.floor(t * S)), 0), S - 1), min(max(int(np.floor(s * S)), 0), S - 1)


_TABLES = {}


def border_table(S):
    """int64 [3, 6, S+2, S+2] flat cube-texel indices (f*S*S + r*S + c) read by each padded texel, and bool [6, S+2, S+2]
    marking the corners, which average all three (own corner texel, row-neighbour, column-neighbour); every other
    padded texel copies index 0."""
    if S not in _TABLES:
        P = S + 2
        src = np.zeros((3, 6, P, P), np.int64)
        corner = np.zeros((6, P, P), bool)
        flat = lambda g, r, c: (g * S + r) * S + c
        src[:, :, 1:P - 1, 1:P - 1] = np.arange(6 * S * S).reshape(6, S, S)
        ring = [(i, j) for i in range(P) for j in range(P) if i in (0, P - 1) or j in (0, P - 1)]
        for f in range(6):
            for i, j in ring:
                if (i in (0, P - 1)) != (j in (0, P - 1)):
                    src[:, f, i, j] = flat(*border_source(f, i, j, S))
                else:
                    ii, jj = (1 if i == 0 else S), (1 if j == 0 else S)
                    src[:, f, i, j] = [flat(f, ii - 1, jj - 1), flat(*border_source(f, i, jj, S)),
                                       flat(*border_source(f, ii, j, S))]
                    corner[f, i, j] = True
        _TABLES[S] = (src, corner)
    return _TABLES[S]


def atlas(cubemap):
    """[6, S, S, C] -> the padded faces [6, S+2, S+2, C]."""
    S = cubemap.shape[-2]
    src, corner = border_table(S)
    flat = cubemap.reshape(6 * S * S, cubemap.shape[-1])
    dev = cubemap.device
    t0, t1, t2 = (flat[torch.as_tensor(src[k], device=dev)] for k in range(3))
    # a tensor divisor: torch divides by a Python scalar as a multiplication by its reciprocal, rounded differently
    three = torch.full_like(t0, 3.)
    return torch.where(torch.as_tensor(corner, device=dev)[..., None], ((t0 + t1) + t2) / three, t0)


def face_coords(directions):
    """directions [..., 3] -> (face int64 [...], s, t [...], valid bool [...]); s and t carry gradients to the
    directions through the selected face only.  Invalid lookups get face 0 and s = t = 0.5."""
    valid = torch.isfinite(directions).all(-1) & (directions != 0).any(-1)
    d = torch.where(valid[..., None], directions, torch.ones_like(directions))
    x, y, z = d.unbind(-1)
    ax, ay, az = x.abs(), y.abs(), z.abs()
    use_x = (ax >= ay) & (ax >= az)
    use_y = ~use_x & (ay >= az)
    face = torch.where(use_x, torch.where(x > 0, 0, 1), torch.where(use_y, torch.where(y > 0, 2, 3),
                                                                      torch.where(z > 0, 4, 5)))
    sc = torch.stack([-z, z, x, x, x, -x], -1).gather(-1, face[..., None])[..., 0]
    tc = torch.stack([-y, -y, z, -z, -y, -y], -1).gather(-1, face[..., None])[..., 0]
    ma = torch.stack([ax, ax, ay, ay, az, az], -1).gather(-1, face[..., None])[..., 0]
    s = (sc / ma + 1.) * 0.5
    t = (tc / ma + 1.) * 0.5
    return face, s, t, valid


def sample_padded(padded, face, s, t, valid, mode='bilinear'):
    """padded [6, S+2, S+2, C], face / s / t / valid [...] -> [..., C]."""
    S = padded.shape[-2] - 2
    P = S + 2
    flat = padded.reshape(6 * P * P, padded.shape[-1])
    if mode == 'nearest':
        r = (t.detach() * S).floor().clamp(0, S - 1).long() + 1
        c = (s.detach() * S).floor().clamp(0, S - 1).long() + 1
        out = flat[(face * P + r) * P + c]
    elif mode == 'bilinear':
        pr = (t * S - 0.5) + 1.
        pc = (s * S - 0.5) + 1.
        fl_r, fl_c = pr.detach().floor(), pc.detach().floor()
        fr, fc = (pr - fl_r)[..., None], (pc - fl_c)[..., None]
        r0, c0 = fl_r.long(), fl_c.long()
        at = lambda r, c: flat[(face * P + r) * P + c]
        out = (at(r0, c0) * (1. - fc) * (1. - fr) + at(r0, c0 + 1) * fc * (1. - fr) +
               at(r0 + 1, c0) * (1. - fc) * fr + at(r0 + 1, c0 + 1) * fc * fr)
    else:
        raise NotImplementedError(mode)
    return torch.where(valid[..., None], out, torch.zeros_like(out))


def sample(cubemap, directions, mode='bilinear'):
    """cubemap [6, S, S, C] with directions [..., 3], or [B, 6, S, S, C] with directions [B, ..., 3] -> [..., C]."""
    if cubemap.dim() == 5:
        return torch.stack([sample(cubemap[b], directions[b], mode) for b in range(cubemap.shape[0])])
    face, s, t, valid = face_coords(directions)
    return sample_padded(atlas(cubemap), face, s, t, valid, mode)
