"""The equirectangular-to-cube-map conversion of latlong_to_cubemap (DESIGN.md §7.13) restated in torch.  It is the
specification: in float32 on the GPU the CUDA forward equals `to_cubemap` bit for bit, and the gradient to the panorama
is torch autograd's of `to_cubemap`.

Every fp32 step below is one IEEE-rounded torch operation, in the kernel's order.  Constants are rounded to fp32 once:
INV_2PI = fp32(1 / (2 pi)) = 0.15915494 and INV_PI = fp32(1 / pi) = 0.31830987.  Every divisor is a tensor, since torch
divides by a Python scalar as a multiplication by its reciprocal, which rounds differently.
    n         samples(H, W, S) = max(1, ceil(max(W, 2H) / (pi S))), in float64
    sc, tc    (2 (c n + j) + 1) / (S n) - 1 and (2 (r n + i) + 1) / (S n) - 1: an exact fp32 integer over the exact fp32
              S n, then - 1, for sample (i, j) of cube texel (f, r, c)
    x, y, z   cubemap_restatement.FACE_AXES with |major| = 1, not normalised; negations keep signed zeros
    phi       atan2(x, -z);  theta = atan2(sqrt(x * x + z * z), y)
    u, v      phi * INV_2PI + 0.5, theta * INV_PI
    pc, pr    u * W - 0.5, (v * H - 0.5) + 1
    taps      r0 = floor(pr), fr = pr - r0, c0 = floor(pc), fc = pc - c0; rows r0, r0 + 1 of the panorama padded by a
              copy of row 0 above and of row H-1 below (panorama rows clamp(r0 - 1), clamp(r0)), columns c0, c0 + 1
              modulo W
    bilinear  t00*(1-fc)*(1-fr) + t01*fc*(1-fr) + t10*(1-fc)*fr + t11*fc*fr
    mean      the n^2 samples added to 0 in row-major order (i, then j), then divided by n^2
Only the panorama gets a gradient: the sample positions are constants."""
import math

import torch

from cubemap_restatement import FACE_AXES

INV_2PI = 0.5 / math.pi   # rounded to the coordinate dtype where used
INV_PI = 1.0 / math.pi


def samples(H, W, S):
    """n, the sub-samples per cube-texel edge."""
    return max(1, math.ceil(max(W, 2 * H) / (math.pi * S)))


def _full(like, value):
    return torch.full_like(like, value)


def sample_directions(S, n, i, j, dtype=torch.float32, device=None):
    """Sample (i, j) of every cube texel as (x, y, z), each [6, S, S] of `dtype`."""
    r = torch.arange(S, device=device)
    tnum = (2 * (r * n + i) + 1).to(dtype)
    snum = (2 * (r * n + j) + 1).to(dtype)
    tc = (tnum / _full(tnum, float(S * n)) - 1.)[:, None].expand(S, S)
    sc = (snum / _full(snum, float(S * n)) - 1.)[None, :].expand(S, S)
    xyz = []
    for f in range(6):
        a, (js, ss), (jt, st) = FACE_AXES[f]
        comp = [None] * 3
        comp[a] = torch.full((S, S), 1. if f % 2 == 0 else -1., dtype=dtype, device=device)
        comp[js] = sc if ss > 0 else -sc
        comp[jt] = tc if st > 0 else -tc
        xyz.append(comp)
    return tuple(torch.stack([d[k] for d in xyz]) for k in range(3))


def coordinates(x, y, z, H, W):
    """Directions -> padded (row, col) of the panorama, pr and pc, in the directions' dtype."""
    phi = torch.atan2(x, -z)
    theta = torch.atan2(torch.sqrt(x * x + z * z), y)
    u = phi * _full(phi, INV_2PI) + 0.5
    v = theta * _full(theta, INV_PI)
    pc = u * _full(u, float(W)) - 0.5
    pr = (v * _full(v, float(H)) - 0.5) + 1.
    return pr, pc


def taps(pr, pc, H, W):
    """(rows ra, rb, columns c0, c1 as int64; fractions fr, fc) of the bilinear lookups at padded (pr, pc)."""
    fl_r, fl_c = pr.floor(), pc.floor()
    r0, c0 = fl_r.long(), torch.remainder(fl_c.long(), W)
    return ((r0 - 1).clamp(0, H - 1), r0.clamp(0, H - 1), c0, torch.remainder(c0 + 1, W), pr - fl_r, pc - fl_c)


def bilinear(panorama, ra, rb, c0, c1, fr, fc):
    """panorama [H, W, C] read at the taps [...] -> [..., C], fr and fc cast to the panorama's dtype."""
    W = panorama.shape[1]
    flat = panorama.reshape(-1, panorama.shape[-1])
    at = lambda r, c: flat[r * W + c]
    fr, fc = fr.to(panorama.dtype)[..., None], fc.to(panorama.dtype)[..., None]
    return (at(ra, c0) * (1. - fc) * (1. - fr) + at(ra, c1) * fc * (1. - fr) +
            at(rb, c0) * (1. - fc) * fr + at(rb, c1) * fc * fr)


def to_cubemap(panorama, S, coord_dtype=torch.float32):
    """panorama [H, W, C] -> [6, S, S, C], or [B, H, W, C] -> [B, 6, S, S, C], in the panorama's dtype.  The sample
    coordinates are computed in coord_dtype on the panorama's device: float32 is the kernel's arithmetic (a float64
    panorama then gives the float64 evaluation at the float32 coordinates); float64 is the conversion in float64."""
    if panorama.dim() == 4:
        return torch.stack([to_cubemap(p, S, coord_dtype) for p in panorama])
    H, W, _ = panorama.shape
    n = samples(H, W, S)
    acc = None
    for i in range(n):
        for j in range(n):
            x, y, z = sample_directions(S, n, i, j, coord_dtype, panorama.device)
            s = bilinear(panorama, *taps(*coordinates(x, y, z, H, W), H, W))
            acc = (torch.zeros_like(s) if acc is None else acc) + s
    return acc / _full(acc, float(n * n))
