"""The mipmapped (trilinear) cube-map lookup of sample_cubemap(..., mode='trilinear', lod=...) (DESIGN.md §7.11)
restated in torch.  It is the specification: in float32 on the GPU the CUDA forward equals `sample` bit for bit, and the
gradients are torch autograd's of `sample`.

    levels    level 0 is the cube map [6, S, S, C]; levels 1 .. L-1 are each face's box pyramid
              (texture_mip_restatement.pyramid), L = level_count(S, S), S >> k texels per edge at level k
    b_k       level k read with cubemap_restatement's bilinear rule on its own padded faces: atlas(level k), at
              ((t * S_k - 0.5) + 1, (s * S_k - 0.5) + 1), S_k = S >> k
    lod       lambda = lod, NaN -> 0, clamped to [0, L-1]; l = floor(lambda), f = lambda - l
    out       (1-f) * b_l + f * b_{l+1}, rounded in that order; b_l alone (level l+1 not read) where f == 0
    d/d lod   sum_c grad_out_c * (b_{m+1,c} - b_{m,c}), m = min(l, L-2); 0 where lod < 0, lod > L-1, lod is NaN,
              L = 1 or the direction is invalid
A zero or non-finite direction returns 0 and passes no gradient."""
import torch

import cubemap_restatement as cm
import texture_mip_restatement as tm


def level_count(S):
    return tm.level_count(S, S)


def pyramid(cubemap):
    """[6, S, S, C] -> the levels 0 .. L-1, each [6, S >> k, S >> k, C]."""
    return tm.pyramid(cubemap)


def lod_split(lod, L):
    """(lambda, l, f), no gradient: lambda = lod with NaN -> 0, clamped to [0, L-1]; l = floor(lambda), f = lambda - l."""
    x = lod.detach()
    lam = torch.where(torch.isnan(x), torch.zeros_like(x), x).clamp(0., float(L - 1))
    l = lam.floor()
    return lam, l, lam - l


class _LodGrad(torch.autograd.Function):
    """The identity on `out`, with d out / d lod = slope (per channel): the lod's gradient alone, so that the forward
    value is not touched by a term such as 0 * b."""

    @staticmethod
    def forward(ctx, out, lod, slope):
        ctx.save_for_backward(slope)
        ctx.lod_dtype = lod.dtype
        return out.clone()

    @staticmethod
    def backward(ctx, grad):
        slope, = ctx.saved_tensors
        return grad, (grad * slope).sum(-1).to(ctx.lod_dtype), None


def blend(reads, lod, valid):
    """reads: b_0 .. b_{L-1} [..., C]; lod, valid [...] -> [..., C]."""
    L = len(reads)
    lam, l, f = lod_split(lod, L)
    l, f = l[..., None], f[..., None].to(reads[0].dtype)
    lo, hi = reads[0], reads[min(1, L - 1)]
    for k in range(1, L):
        lo = torch.where(l == k, reads[k], lo)
        hi = torch.where(l + 1 == k, reads[k], hi) if k > 1 else hi
    out = torch.where(f == 0, lo, (1. - f) * lo + f * hi)
    if not lod.requires_grad:
        return out
    # d out / d lod: the difference of levels m + 1 and m, m = min(l, L-2), where lod lies in [0, L-1]
    with torch.no_grad():
        m = l.clamp(max=max(L - 2, 0))
        b0, b1 = reads[0], reads[min(1, L - 1)]
        for k in range(1, L):
            b0 = torch.where(m == k, reads[k], b0)
            b1 = torch.where(m + 1 == k, reads[k], b1) if k > 1 else b1
        x = lod.detach()
        live = valid & ~torch.isnan(x) & (x >= 0) & (x <= L - 1) & (L > 1)
        slope = torch.where(live[..., None], b1 - b0, torch.zeros_like(b0))
    return _LodGrad.apply(out, lod, slope)


def sample(cubemap, directions, lod, coords_of=None):
    """cubemap [6, S, S, C] with directions [..., 3] and lod [...], or [B, 6, S, S, C] with [B, ..., 3] and [B, ...]
    -> [..., C].  `coords_of(directions, k, S_k)` replaces cubemap_restatement.face_coords at level k (the float64
    gradient checks move s and t onto each level's float32 lookup)."""
    if cubemap.dim() == 5:
        return torch.stack([sample(cubemap[b], directions[b], lod[b], coords_of) for b in range(cubemap.shape[0])])
    levels = pyramid(cubemap)
    reads = []
    for k, level in enumerate(levels):
        face, s, t, valid = (coords_of or (lambda d, k, S: cm.face_coords(d)))(directions, k, level.shape[-2])
        reads.append(cm.sample_padded(cm.atlas(level), face, s, t, valid, 'bilinear'))
    valid = cm.face_coords(directions)[3]
    return blend(reads, lod, valid)


def level_lookup(cubemap, directions, k):
    """b_k alone: level k of the pyramid read with the bilinear rule on its padded faces."""
    face, s, t, valid = cm.face_coords(directions)
    return cm.sample_padded(cm.atlas(pyramid(cubemap)[k]), face, s, t, valid, 'bilinear')
