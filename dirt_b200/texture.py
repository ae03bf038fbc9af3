"""Texture lookup with gradients to the texels and to the texture coordinates.

The lookup of the reference's textured sample (samples/textured.py:15-60) as a CUDA op: `uvs_to_pixel_indices` maps
uv coordinates to fractional texel indices (plain torch, any device), `sample_texture` reads the texture there
(dirt_texture_sample / dirt_texture_sample_backward of include/dirt_b200.h).  The values are those of the torch
restatement in examples/textured.py, bit for bit; see DESIGN.md §7.1.  `mode='trilinear'` reads a mip pyramid of the
texture at a level of detail taken from screen-space index derivatives (`index_derivatives` makes them from an index
image); see DESIGN.md §7.6.  `latlong_to_cubemap` converts an equirectangular panorama to the cube map that
`sample_cubemap` reads (DESIGN.md §7.13).
"""
import ctypes
import math

import torch
from torch.autograd.function import once_differentiable

from . import _lib
from .rasterise_ops import _as, _pick_device, _ptr, _require_cuda, _stream_ptr

_MODES = {'bilinear': _lib.TEXTURE_BILINEAR, 'nearest': _lib.TEXTURE_NEAREST}


def uvs_to_pixel_indices(uvs, texture_shape, mode='repeat'):
    """uv coordinates [..., 2] -> fractional (row, column) texel indices [..., 2]; u = 0, v = 0 is the TOP-left texel
    corner (as in samples/textured.py:15-27, unlike OpenGL).  `mode`: 'repeat' wraps uv into [0, 1), 'clamp' clamps it
    to [0, 1]."""
    uvs = uvs.flip(-1)   # (u, v) = (x, y) -> (row, column)
    shape = torch.as_tensor(texture_shape, dtype=uvs.dtype, device=uvs.device)
    if mode == 'repeat':
        return uvs % 1. * shape
    if mode == 'clamp':
        return uvs.clamp(0., 1.) * shape
    raise NotImplementedError(mode)


def _backward(device, want_table, entry, size, op, too_large):
    """Runs a lookup's backward entry point, `entry(deterministic, scratch, scratch_bytes, stream)`, on `device`, with
    the scratch of `size(deterministic)` bytes it asks for.  The deterministic (sorted) path is taken when the gradient
    of the texture or cube map is wanted under torch.use_deterministic_algorithms(True); the gradients of the lookup
    coordinates alone are per lookup and already reproducible.  `too_large` names the shapes a deterministic call
    refuses with ERR_BAD_SHAPE, for the RuntimeError that then names the flag."""
    deterministic = bool(want_table and torch.are_deterministic_algorithms_enabled())
    scratch_bytes = int(size(deterministic))
    scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=device) if scratch_bytes else None
    with torch.cuda.device(device):
        rc = entry(deterministic, _ptr(scratch), scratch_bytes, _stream_ptr(device))
    if deterministic and rc == _lib.ERR_BAD_SHAPE:
        # the shapes passed the forward call: what fails are the sorted path's 32-bit limits
        raise RuntimeError(too_large + ', but torch.use_deterministic_algorithms(True) is set')
    _lib.check(rc, op)


class _SampleTexture(torch.autograd.Function):
    """dirt_texture_sample, or for mode 'trilinear' dirt_texture_mip_build then dirt_texture_sample_trilinear, with the
    gradient.  texture [TB, TH, TW, C], indices [B, N, 2], derivatives [B, N, 4] ('trilinear' only), contiguous fp32
    CUDA.  The trilinear pyramid is built per call and kept for the backward pass."""

    @staticmethod
    def forward(ctx, texture, indices, mode, out_shape, derivatives=None):
        TB, TH, TW, C = texture.shape
        B, N = indices.shape[0], indices.shape[1]
        L = _lib.lib()
        out = torch.empty(out_shape, dtype=torch.float32, device=indices.device)
        pyramid = None
        with torch.cuda.device(indices.device):
            stream = _stream_ptr(indices.device)
            if mode == 'trilinear':
                pyramid_floats = int(L.dirt_texture_mip_pyramid_bytes(TB, TH, TW, C)) // 4
                if pyramid_floats:
                    pyramid = torch.empty(pyramid_floats, dtype=torch.float32, device=indices.device)
                rc = L.dirt_texture_mip_build(_ptr(texture), _ptr(pyramid), TB, TH, TW, C, stream)
                _lib.check(rc, 'SampleTextureMipBuild')
                rc = L.dirt_texture_sample_trilinear(_ptr(texture), _ptr(pyramid), _ptr(indices), _ptr(derivatives),
                                                     _ptr(out), TB, TH, TW, C, B, N, stream)
            else:
                rc = L.dirt_texture_sample(_ptr(texture), _ptr(indices), _ptr(out), TB, TH, TW, C, B, N, mode, stream)
        _lib.check(rc, 'SampleTexture')
        ctx.save_for_backward(texture, indices, pyramid, derivatives)
        ctx.mode = mode
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        want_texture, want_indices = ctx.needs_input_grad[:2]
        if not (want_texture or want_indices):
            return None, None, None, None, None
        texture, indices, pyramid, derivatives = ctx.saved_tensors
        TB, TH, TW, C = texture.shape
        B, N = indices.shape[0], indices.shape[1]
        L = _lib.lib()
        grad_out = grad_out.contiguous().to(torch.float32)
        grad_texture = torch.empty_like(texture) if want_texture else None
        grad_indices = torch.empty_like(indices) if want_indices else None
        if ctx.mode == 'trilinear':
            ptrs = [_ptr(t) for t in (texture, pyramid, indices, derivatives, grad_out, grad_texture, grad_indices)]
            dims = (TB, TH, TW, C, B, N)
            entry = lambda det, scratch, nbytes, stream: L.dirt_texture_sample_trilinear_backward(
                *ptrs, *dims, int(det), scratch, nbytes, stream)
            size = lambda det: L.dirt_texture_sample_trilinear_backward_bytes(*dims, int(det))
        else:
            # bilinear and nearest: the default entry point takes no scratch, the deterministic one has its own
            ptrs = [_ptr(t) for t in (texture, indices, grad_out, grad_texture, grad_indices)]
            dims = (TB, TH, TW, C, B, N, ctx.mode)
            entry = lambda det, scratch, nbytes, stream: (
                L.dirt_texture_sample_backward_deterministic(*ptrs, *dims, scratch, nbytes, stream) if det
                else L.dirt_texture_sample_backward(*ptrs, *dims, stream))
            size = lambda det: L.dirt_texture_sample_backward_deterministic_bytes(*dims) if det else 0
        _backward(indices.device, want_texture, entry, size, 'SampleTextureGrad',
                  'sample_texture backward: the texture gradient has no deterministic implementation for %d lookups '
                  'into %d x %d x %d texels (it needs fewer than 2^31 of each)' % (B * N, TB, TH, TW))
        return grad_texture, grad_indices, None, None, None


def _wrapped_difference(d, sizes):
    """d [..., 2] reduced modulo (TH, TW) into [-S/2, S/2): a difference across a `repeat` seam is not a jump."""
    half = sizes * 0.5
    return torch.remainder(d + half, sizes) - half


def index_derivatives(indices, texture_shape):
    """Screen-space derivatives of an index image, for `sample_texture(..., mode='trilinear')`.

    Args:
        indices: float tensor [..., H, W, 2] of (row, column) texel indices, one per pixel (for example
            `uvs_to_pixel_indices` of a G-buffer's uv channels); x runs along W, y along H
        texture_shape: (TH, TW), the texture's level-0 size

    Returns:
        tensor [..., H, W, 4] = (d row / dx, d col / dx, d row / dy, d col / dy) in texels per pixel, with no gradient.
        On each screen axis it takes the forward and the backward neighbour difference, reduces each modulo the texture
        size into [-S/2, S/2), and keeps the one of smaller (row, col) magnitude, the forward one on a tie (a non-finite
        difference counts as infinitely large), so a silhouette or a uv seam on one side does not inflate it.  At the
        image border it takes the only neighbour there is; an axis of length 1 gives 0.
    """
    with torch.no_grad():
        sizes = torch.as_tensor([float(texture_shape[0]), float(texture_shape[1])], dtype=indices.dtype,
                                device=indices.device)

        def along(dim):
            n = indices.shape[dim]
            if n < 2:
                return torch.zeros_like(indices)
            diff = _wrapped_difference(indices.narrow(dim, 1, n - 1) - indices.narrow(dim, 0, n - 1), sizes)
            edge = diff.narrow(dim, 0, 1)
            fwd = torch.cat([diff, diff.narrow(dim, n - 2, 1)], dim)    # the last pixel: its backward difference
            bwd = torch.cat([edge, diff], dim)                          # the first pixel: its forward difference
            mf, mb = (fwd * fwd).sum(-1, keepdim=True), (bwd * bwd).sum(-1, keepdim=True)
            inf = torch.full_like(mf, float('inf'))
            mf, mb = torch.where(torch.isfinite(mf), mf, inf), torch.where(torch.isfinite(mb), mb, inf)
            return torch.where(mf <= mb, fwd, bwd)

        return torch.cat([along(indices.dim() - 2), along(indices.dim() - 3)], -1)


def _batched(table, coords, item_dims, per_item_error):
    """The lookups of sample_texture and sample_cubemap as one batch.  A table of `item_dims` dimensions is shared by
    every lookup; one with a leading batch axis holds one table per batch item, and the coordinates then lead with the
    same axis (else ValueError(per_item_error)).  Returns the table [TB, ...] and the coordinates [B, N, K], both
    contiguous, B, N and the lookup's output shape coords.shape[:-1] + (C,)."""
    per_item = table.dim() == item_dims + 1
    if per_item and (coords.dim() < 2 or coords.shape[0] != table.shape[0]):
        raise ValueError(per_item_error)
    B = int(coords.shape[0]) if per_item else 1
    N = math.prod(int(n) for n in coords.shape[(1 if per_item else 0):-1])
    return ((table if per_item else table[None]).contiguous(), coords.reshape(B, N, coords.shape[-1]).contiguous(), B, N,
            tuple(coords.shape[:-1]) + (int(table.shape[-1]),))


def sample_texture(texture, indices, mode='bilinear', derivatives=None):
    """Reads `texture` at fractional (row, column) texel indices, with gradients to the texture and to the indices.

    Args:
        texture: float32 tensor [H, W, C], shared by every lookup, or [B, H, W, C], one texture per batch item
        indices: float32 tensor [..., 2] for a shared texture, [B, ..., 2] for per-item textures; (0, 0) is the
            top-left corner of the top-left texel (`uvs_to_pixel_indices` makes them from uv coordinates)
        mode: 'bilinear' (the four texels around the index, wrapping around the texture edge), 'nearest' (the texel
            the truncated index names, clamped to the texture; no gradient to the indices) or 'trilinear' (bilinear
            lookups of the two mip levels around the level of detail the derivatives give, blended; DESIGN.md §7.6)
        derivatives: 'trilinear' only, and required there: float32 tensor indices.shape[:-1] + (4,) of
            (d row / dx, d col / dx, d row / dy, d col / dy) in texels per pixel (`index_derivatives` makes them).
            They choose the level of detail, lambda = log2 of the longer screen axis's footprint, clamped to the
            pyramid; they get no gradient (lambda is treated as a constant, as 'nearest' treats its index).
            Where the footprint is at most one texel, 'trilinear' returns exactly what 'bilinear' returns.

    Returns:
        float32 tensor indices.shape[:-1] + (C,), equal bit for bit to the torch restatement in examples/textured.py
        ('bilinear', 'nearest').  A lookup with a non-finite index returns 0 in every channel and passes no gradient back.

    Needs CUDA tensors (there is no CPU kernel); anything else array-like is moved to the current CUDA device.
    """
    if mode not in _MODES and mode != 'trilinear':
        raise ValueError("sample_texture: mode must be 'bilinear', 'nearest' or 'trilinear', not %r" % (mode,))
    if mode == 'trilinear' and derivatives is None:
        raise ValueError("sample_texture: mode 'trilinear' needs derivatives, shaped indices.shape[:-1] + (4,)")
    if mode != 'trilinear' and derivatives is not None:
        raise ValueError("sample_texture: derivatives are only used by mode 'trilinear', not by %r" % (mode,))
    device = _pick_device(texture, indices)
    texture = _as(texture, torch.float32, device)
    indices = _as(indices, torch.float32, device)
    if texture.dim() not in (3, 4):
        raise ValueError('SampleTexture expects texture to be 3D or 4D, and texture.shape == [height, width, channels] '
                         'or [None, height, width, channels]')
    if texture.shape[-3] <= 0 or texture.shape[-2] <= 0 or texture.shape[-1] <= 0:
        raise ValueError('SampleTexture expects a texture with positive height, width and channels')
    if indices.dim() < 1 or indices.shape[-1] != 2:
        raise ValueError('SampleTexture expects indices.shape[-1] == 2')
    tex, flat, B, N, out_shape = _batched(
        texture, indices, 3, 'SampleTexture expects indices of per-item textures to be at least 2D, and indices.shape[0] '
        '== texture.shape[0]')
    if mode == 'trilinear':
        derivatives = _as(derivatives, torch.float32, device)
        if tuple(derivatives.shape) != tuple(indices.shape[:-1]) + (4,):
            raise ValueError('SampleTexture expects derivatives.shape == indices.shape[:-1] + (4,), got %s for indices %s'
                             % (tuple(derivatives.shape), tuple(indices.shape)))
        _require_cuda(texture, indices, derivatives)
        return _SampleTexture.apply(tex, flat, mode, out_shape, derivatives.detach().reshape(B, N, 4).contiguous())
    _require_cuda(texture, indices)
    return _SampleTexture.apply(tex, flat, _MODES[mode], out_shape)


# per sample_cubemap mode: the atlas size query, the lookup, the backward scratch size query, the backward pass and the
# op's name in errors
_CUBEMAP_ENTRIES = {
    'bilinear': ('dirt_cubemap_atlas_bytes', 'dirt_cubemap_sample', 'dirt_cubemap_sample_backward_bytes',
                 'dirt_cubemap_sample_backward', 'SampleCubemap'),
    'trilinear': ('dirt_cubemap_mip_atlas_bytes', 'dirt_cubemap_sample_trilinear',
                  'dirt_cubemap_sample_trilinear_backward_bytes', 'dirt_cubemap_sample_trilinear_backward',
                  'SampleCubemapTrilinear'),
    'ggx': ('dirt_cubemap_ggx_atlas_bytes', 'dirt_cubemap_sample_ggx', 'dirt_cubemap_sample_ggx_backward_bytes',
            'dirt_cubemap_sample_ggx_backward', 'SampleCubemapGGX'),
}
_CUBEMAP_ENTRIES['nearest'] = _CUBEMAP_ENTRIES['bilinear']


class _SampleCubemap(torch.autograd.Function):
    """dirt_cubemap_sample / dirt_cubemap_sample_backward, or for mode 'trilinear' and 'ggx' the
    dirt_cubemap_sample_trilinear and dirt_cubemap_sample_ggx pairs.  cubemap [TB, 6, S, S, C], directions [B, N, 3],
    lod [B, N] ('trilinear' and 'ggx' only, else None), contiguous fp32 CUDA.  The atlas of padded faces ('trilinear':
    every level's; 'ggx': also the prefiltered levels, their normalisers and the texel table) is built per call and kept
    for the backward pass in place of the cube map."""

    @staticmethod
    def forward(ctx, cubemap, directions, lod, mode, out_shape):
        TB, _, S, _, C = cubemap.shape
        B, N = directions.shape[0], directions.shape[1]
        L = _lib.lib()
        atlas_bytes, sample, _, _, op = _CUBEMAP_ENTRIES[mode]
        out = torch.empty(out_shape, dtype=torch.float32, device=directions.device)
        atlas = torch.empty(int(getattr(L, atlas_bytes)(TB, S, C)) // 4, dtype=torch.float32, device=directions.device)
        # bilinear and nearest take the mode, trilinear and ggx the level of detail
        lod_arg, mode_arg = ((), (_MODES[mode],)) if lod is None else ((_ptr(lod),), ())
        with torch.cuda.device(directions.device):
            rc = getattr(L, sample)(_ptr(cubemap), _ptr(directions), *lod_arg, _ptr(atlas), _ptr(out), TB, S, C, B, N,
                                    *mode_arg, _stream_ptr(directions.device))
        _lib.check(rc, op)
        ctx.save_for_backward(atlas, directions, lod)
        ctx.mode, ctx.shape = mode, (TB, S, C)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        want_cubemap, want_directions, want_lod = ctx.needs_input_grad[:3]
        if not (want_cubemap or want_directions or want_lod):
            return None, None, None, None, None
        atlas, directions, lod = ctx.saved_tensors
        TB, S, C = ctx.shape
        B, N = directions.shape[0], directions.shape[1]
        L = _lib.lib()
        _, _, size, entry, op = _CUBEMAP_ENTRIES[ctx.mode]
        grad_out = grad_out.contiguous().to(torch.float32)
        dev = directions.device
        grad_cubemap = torch.empty((TB, 6, S, S, C), dtype=torch.float32, device=dev) if want_cubemap else None
        grad_directions = torch.empty_like(directions) if want_directions else None
        grad_lod = torch.empty_like(lod) if want_lod else None
        # bilinear and nearest take the mode, trilinear and ggx the level of detail and its gradient
        if lod is None:
            ptrs = [_ptr(t) for t in (atlas, directions, grad_out, grad_cubemap, grad_directions)]
            dims = (TB, S, C, B, N, _MODES[ctx.mode])
        else:
            ptrs = [_ptr(t) for t in (atlas, directions, lod, grad_out, grad_cubemap, grad_directions, grad_lod)]
            dims = (TB, S, C, B, N)
        _backward(dev, want_cubemap,
                  lambda det, scratch, nbytes, stream: getattr(L, entry)(*ptrs, *dims, int(det), scratch, nbytes, stream),
                  lambda det: getattr(L, size)(*dims, int(det)), op + 'Grad',
                  'sample_cubemap backward: the cube-map gradient has no deterministic implementation for %d lookups '
                  'into %d x 6 x %d x %d texels (it needs fewer than 2^31 lookups and padded texels per face)'
                  % (B * N, TB, S, S))
        return grad_cubemap, grad_directions, grad_lod, None, None


def sample_cubemap(cubemap, directions, mode='bilinear', lod=None, roughness=None):
    """Reads a cube map in the given directions, seamlessly across its edges and corners, with gradients to the texels
    and to the directions.

    Args:
        cubemap: float32 tensor [6, S, S, C], shared by every lookup, or [B, 6, S, S, C], one cube map per batch item.
            Faces +X, -X, +Y, -Y, +Z, -Z, each oriented as in OpenGL: face texel (0, 0) is at the face's (s, t) =
            (0, 0) corner, rows running along t
        directions: float32 tensor [..., 3] for a shared cube map, [B, ..., 3] for per-item cube maps; any length
        mode: 'bilinear' (the four texels around the lookup; near an edge or a corner they come from the adjacent faces,
            so there is no seam), 'nearest' (the texel the lookup falls in; no gradient to the directions) or
            'trilinear' (bilinear lookups of the two levels of the cube map's box pyramid around `lod`, blended;
            DESIGN.md §7.11)
        lod: 'trilinear' only, and required there: the level of detail in levels, 0 the finest and
            log2(S) the 1 x 1 level of an S = 2^n map (an odd S has level 0 alone).  A float, or a float32 tensor
            broadcastable to directions.shape[:-1]; it gets a gradient (the difference of the two levels' values,
            0 where it is clamped to the pyramid or NaN).  lod <= 0 returns exactly what 'bilinear' returns, and an
            integer lod = k the bilinear lookup of level k.  A typical use maps a roughness to a level.
        roughness: 'ggx' only, and required there: the GGX roughness of a split-sum environment lookup (DESIGN.md
            §7.12).  'ggx' is 'trilinear' with lod = roughness * (L-1) on the levels of the cube map prefiltered with
            the GGX lobe of roughness k / (L-1) (level 0 the map itself); a float or a float32 tensor broadcastable
            to directions.shape[:-1], with a gradient (L-1 times lod's).  roughness <= 0 returns exactly what
            'bilinear' returns.  Needs an even S (L >= 2); the prefiltered levels are rebuilt on every call.

    Returns:
        float32 tensor directions.shape[:-1] + (C,), equal bit for bit to the torch restatement in
        tests/cubemap_restatement.py (DESIGN.md §7.10; 'trilinear': tests/cubemap_mip_restatement.py; 'ggx': the
        same level blend of the prefiltered levels, which tests/cubemap_ggx_restatement.py defines).  A zero or non-finite direction returns 0 in every channel and
        passes no gradient back.  Under torch.use_deterministic_algorithms(True) the cube-map gradient is
        bit-reproducible.

    Needs CUDA tensors (there is no CPU kernel); anything else array-like is moved to the current CUDA device.
    """
    if mode not in _MODES and mode not in ('trilinear', 'ggx'):
        raise ValueError("sample_cubemap: mode must be 'bilinear', 'nearest', 'trilinear' or 'ggx', not %r" % (mode,))
    if mode == 'trilinear' and lod is None:
        raise ValueError("sample_cubemap: mode 'trilinear' needs lod, a float or a tensor broadcastable to "
                         "directions.shape[:-1]")
    if mode != 'trilinear' and lod is not None:
        raise ValueError("sample_cubemap: lod is only used by mode 'trilinear', not by %r" % (mode,))
    if mode == 'ggx' and roughness is None:
        raise ValueError("sample_cubemap: mode 'ggx' needs roughness, a float or a tensor broadcastable to "
                         "directions.shape[:-1]")
    if mode != 'ggx' and roughness is not None:
        raise ValueError("sample_cubemap: roughness is only used by mode 'ggx', not by %r" % (mode,))
    device = _pick_device(cubemap, directions)
    cubemap = _as(cubemap, torch.float32, device)
    directions = _as(directions, torch.float32, device)
    if cubemap.dim() not in (4, 5) or cubemap.shape[-4] != 6 or cubemap.shape[-3] != cubemap.shape[-2]:
        raise ValueError('SampleCubemap expects cubemap.shape == [6, size, size, channels] or '
                         '[None, 6, size, size, channels]')
    if cubemap.shape[-2] <= 0 or cubemap.shape[-1] <= 0:
        raise ValueError('SampleCubemap expects a cube map with positive size and channels')
    if directions.dim() < 1 or directions.shape[-1] != 3:
        raise ValueError('SampleCubemap expects directions.shape[-1] == 3')
    cube, flat, B, N, out_shape = _batched(
        cubemap, directions, 4, 'SampleCubemap expects directions of per-item cube maps to be at least 2D, and '
        'directions.shape[0] == cubemap.shape[0]')
    if mode == 'ggx':
        S = int(cubemap.shape[-2])
        if S % 2:
            raise ValueError("sample_cubemap: mode 'ggx' needs an even cube-map size (a mip chain of at least two "
                             "levels), got %d; with one level the roughness would be ignored" % S)
        # lod = roughness * (L-1) in torch, so that autograd carries lod's gradient to the roughness
        lod = _as(roughness, torch.float32, device) * float(_mip_level_count(S) - 1)
    if mode in ('trilinear', 'ggx'):
        lod = _as(lod, torch.float32, device)
        try:
            # broadcast before the autograd Function, so that autograd sums the gradient of a broadcast lod
            lod = lod.expand(directions.shape[:-1])
        except RuntimeError:
            raise ValueError('SampleCubemap expects lod broadcastable to directions.shape[:-1] = %s, got %s'
                             % (tuple(directions.shape[:-1]), tuple(lod.shape)))
        _require_cuda(cubemap, directions, lod)
        lod = lod.reshape(B, N).contiguous()
    else:
        _require_cuda(cubemap, directions)
    return _SampleCubemap.apply(cube, flat, lod, mode, out_shape)


def _mip_level_count(S):
    """Levels of an S x S face's box pyramid: one more per halving while the edge is even."""
    L = 1
    while S > 0 and S % 2 == 0:
        S //= 2
        L += 1
    return L


class _LatlongToCubemap(torch.autograd.Function):
    """dirt_latlong_to_cubemap / dirt_latlong_to_cubemap_backward.  panorama [TB, H, W, C] contiguous fp32 CUDA.  The
    operator depends on the shapes alone, so the backward pass keeps nothing but them."""

    @staticmethod
    def forward(ctx, panorama, size):
        TB, H, W, C = panorama.shape
        L = _lib.lib()
        out = torch.empty((TB, 6, size, size, C), dtype=torch.float32, device=panorama.device)
        with torch.cuda.device(panorama.device):
            rc = L.dirt_latlong_to_cubemap(_ptr(panorama), _ptr(out), TB, H, W, size, C, _stream_ptr(panorama.device))
        _lib.check(rc, 'LatlongToCubemap')
        ctx.shape = (TB, H, W, size, C)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        if not ctx.needs_input_grad[0]:
            return None, None
        TB, H, W, S, C = ctx.shape
        grad_out = grad_out.contiguous().to(torch.float32)
        grad_panorama = torch.empty((TB, H, W, C), dtype=torch.float32, device=grad_out.device)
        with torch.cuda.device(grad_out.device):
            rc = _lib.lib().dirt_latlong_to_cubemap_backward(_ptr(grad_out), _ptr(grad_panorama), TB, H, W, S, C,
                                                             _stream_ptr(grad_out.device))
        _lib.check(rc, 'LatlongToCubemapGrad')
        return grad_panorama, None


def latlong_to_cubemap(panorama, size):
    """Converts an equirectangular (latitude-longitude) panorama to a cube map, with the gradient to the panorama.

    Args:
        panorama: float32 tensor [H, W, C], or [B, H, W, C] for one panorama per batch item; any H, W >= 1.  Row 0 is
            the zenith (+Y); texel (r, c) is centred at theta = (r + 1/2) pi / H from +Y and longitude
            phi = (c + 1/2) 2 pi / W - pi, in direction (sin theta sin phi, cos theta, -sin theta cos phi): the centre
            column faces -Z and, seen from inside, columns run towards +X (`latlong_directions` gives these directions)
        size: S, the cube map's texels per face edge

    Returns:
        float32 tensor [6, S, S, C] or [B, 6, S, S, C] for `sample_cubemap` and `lighting.cubemap_spherical_harmonics`.
        Each cube texel is the mean of n x n bilinear lookups of the panorama at its sub-sample directions,
        n = max(1, ceil(max(W, 2H) / (pi S))), at least one sample per panorama texel at the centre of a side face.
        Columns wrap around; rows do not (a lookup near a pole blends the pole row with itself).  Equal bit for bit
        to the torch restatement in tests/latlong_restatement.py (DESIGN.md §7.13).  The gradient is a gather with no
        atomics, so it is bit-reproducible with or without torch.use_deterministic_algorithms(True).

    Needs CUDA tensors (there is no CPU kernel); anything else array-like is moved to the current CUDA device.
    """
    device = _pick_device(panorama)
    panorama = _as(panorama, torch.float32, device)
    if panorama.dim() not in (3, 4):
        raise ValueError('LatlongToCubemap expects panorama.shape == [height, width, channels] or '
                         '[None, height, width, channels]')
    if panorama.shape[-3] <= 0 or panorama.shape[-2] <= 0 or panorama.shape[-1] <= 0:
        raise ValueError('LatlongToCubemap expects a panorama with positive height, width and channels')
    if isinstance(size, bool) or int(size) != size or size <= 0:
        raise ValueError('LatlongToCubemap expects a positive integer size, got %r' % (size,))
    _require_cuda(panorama)
    per_item = panorama.dim() == 4
    out = _LatlongToCubemap.apply((panorama if per_item else panorama[None]).contiguous(), int(size))
    return out if per_item else out[0]


def latlong_directions(height, width, device=None):
    """The unit directions of an equirectangular panorama's texel centres, float32 [height, width, 3], in the
    convention of `latlong_to_cubemap` (computed in float64, rounded once).  `sample_cubemap(cubemap,
    latlong_directions(H, W))` turns a cube map back into a panorama, for example to view or export a fitted one."""
    if int(height) != height or int(width) != width or height <= 0 or width <= 0:
        raise ValueError('latlong_directions expects a positive integer height and width, got %r, %r' % (height, width))
    theta = (torch.arange(int(height), dtype=torch.float64, device=device) + 0.5) * (math.pi / height)
    phi = (torch.arange(int(width), dtype=torch.float64, device=device) + 0.5) * (2 * math.pi / width) - math.pi
    st, ct = torch.sin(theta)[:, None], torch.cos(theta)[:, None]
    sp, cp = torch.sin(phi)[None, :], torch.cos(phi)[None, :]
    return torch.stack([st * sp, ct.expand(-1, int(width)), -st * cp], -1).to(torch.float32)
