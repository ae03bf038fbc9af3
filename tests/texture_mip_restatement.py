"""The mipmapped (trilinear) lookup of sample_texture(mode='trilinear') (DESIGN.md §7.6) restated in torch: the pyramid,
the index mapping, the level of detail, the blend, and the rule of index_derivatives.  Each level's lookup is
examples/textured.py:sample_texture, the bilinear restatement; in float32 on the GPU the pyramid, and every lookup whose
fraction of level is 0, are bit-identical to the kernels'."""
import importlib.util
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _example():
    spec = importlib.util.spec_from_file_location('textured_example', os.path.join(ROOT, 'examples', 'textured.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_ex = _example()


def level_count(H, W):
    """Level k+1 exists while level k has both dimensions even (a 1x1 level has none)."""
    L = 1
    while H % 2 == 0 and W % 2 == 0:
        H, W, L = H // 2, W // 2, L + 1
    return L


def pyramid(texture):
    """[..., H, W, C] -> the levels 0 .. L-1, each the 2x2 box mean of the one before, rounded as written."""
    levels = [texture]
    while len(levels) < level_count(texture.shape[-3], texture.shape[-2]):
        t = levels[-1]
        levels.append(((t[..., 0::2, 0::2, :] + t[..., 0::2, 1::2, :]) + (t[..., 1::2, 0::2, :] + t[..., 1::2, 1::2, :])) * 0.25)
    return levels


def level_index(indices, k):
    """Level k >= 1 is read at (index + 0.5) * 2^-k - 0.5, rounded in that order; level 0 at the index itself."""
    return indices if k == 0 else (indices + 0.5) * 2.0 ** -k - 0.5


def lod(derivatives, L):
    """(l, f) [..., 1]: rho^2 = max(d0^2 + d1^2, d2^2 + d3^2), lambda = 0.5 log2(rho^2), NaN -> 0, clamped to [0, L-1],
    l = floor(lambda), f = lambda - l.  No gradient."""
    d = derivatives.detach()
    rho2 = torch.maximum(d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1], d[..., 2] * d[..., 2] + d[..., 3] * d[..., 3])
    lam = 0.5 * torch.log2(rho2)
    lam = torch.where(torch.isnan(lam), torch.zeros_like(lam), lam).clamp(0., float(L - 1))
    l = lam.floor()
    return l[..., None], (lam - l)[..., None]


def sample(texture, indices, derivatives, lod_of=None, index_of=None):
    """texture [H, W, C] or [B, H, W, C] (then indices [B, ..., 2]), indices [..., 2], derivatives [..., 4] -> [..., C]:
    (1-f) * bilinear_l + f * bilinear_{l+1}, and bilinear_l alone where f == 0; 0 for a non-finite index.
    `lod_of(derivatives, L)` and `index_of(indices, k)` replace `lod` and `level_index` (the float64 comparisons pass
    the float32 values, so that both pick the same levels and texels)."""
    if texture.dim() == 4:
        return torch.stack([sample(texture[b], indices[b], derivatives[b], lod_of, index_of) for b in range(texture.shape[0])])
    levels = pyramid(texture)
    L = len(levels)
    l, f = (lod_of or lod)(derivatives, L)
    valid = torch.isfinite(indices).all(-1, keepdim=True)
    safe = torch.where(valid, indices, torch.zeros_like(indices))
    reads = [_ex.sample_texture(levels[k], (index_of or level_index)(safe, k)) for k in range(L)]
    lo, hi = reads[0], reads[min(1, L - 1)]
    for k in range(1, L):
        lo = torch.where(l == k, reads[k], lo)
        hi = torch.where(l + 1 == k, reads[k], hi) if k > 1 else hi
    f = f.to(lo.dtype)
    out = torch.where(f == 0, lo, (1. - f) * lo + f * hi)
    return torch.where(valid, out, torch.zeros_like(out))


def index_derivatives(indices, texture_shape):
    """index_derivatives' rule, pixel by pixel in numpy float64: [..., H, W, 2] -> [..., H, W, 4]."""
    a = np.asarray(indices, np.float64)
    S = np.array([float(texture_shape[0]), float(texture_shape[1])])
    out = np.zeros(a.shape[:-1] + (4,))

    def wrapped(d):
        return np.mod(d + S / 2, S) - S / 2

    def pick(fwd, bwd):
        if fwd is None or bwd is None:
            return fwd if bwd is None else bwd
        mf, mb = (fwd * fwd).sum(), (bwd * bwd).sum()
        mf, mb = (mf if np.isfinite(mf) else np.inf), (mb if np.isfinite(mb) else np.inf)
        return fwd if mf <= mb else bwd

    H, W = a.shape[-3], a.shape[-2]
    for lead in np.ndindex(*a.shape[:-3]):
        img = a[lead]
        for i in range(H):
            for j in range(W):
                fx = wrapped(img[i, j + 1] - img[i, j]) if j + 1 < W else None
                bx = wrapped(img[i, j] - img[i, j - 1]) if j > 0 else None
                fy = wrapped(img[i + 1, j] - img[i, j]) if i + 1 < H else None
                by = wrapped(img[i, j] - img[i - 1, j]) if i > 0 else None
                dx = pick(fx, bx) if W > 1 else np.zeros(2)
                dy = pick(fy, by) if H > 1 else np.zeros(2)
                out[lead + (i, j)] = np.concatenate([dx, dy])
    return out
