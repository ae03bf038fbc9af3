"""Texture lookup with gradients to the texels and to the texture coordinates.

The lookup of the reference's textured sample (samples/textured.py:15-60) as a CUDA op: `uvs_to_pixel_indices` maps
uv coordinates to fractional texel indices (plain torch, any device), `sample_texture` reads the texture there
(dirt_texture_sample / dirt_texture_sample_backward of include/dirt_b200.h).  The values are those of the torch
restatement in examples/textured.py, bit for bit; see DESIGN.md §7.1.  `mode='trilinear'` reads a mip pyramid of the
texture at a level of detail taken from screen-space index derivatives (`index_derivatives` makes them from an index
image); see DESIGN.md §7.6.
"""
import ctypes

import torch
from torch.autograd.function import once_differentiable

from . import _lib
from .rasterise_ops import _as_f32, _pick_device, _ptr, _require_cuda, _stream_ptr

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


class _SampleTexture(torch.autograd.Function):
    """dirt_texture_sample with its gradient.  texture [TB, TH, TW, C], indices [B, N, 2], contiguous fp32 CUDA."""

    @staticmethod
    def forward(ctx, texture, indices, mode, out_shape):
        TB, TH, TW, C = texture.shape
        B, N = indices.shape[0], indices.shape[1]
        out = torch.empty(out_shape, dtype=torch.float32, device=indices.device)
        with torch.cuda.device(indices.device):
            rc = _lib.lib().dirt_texture_sample(_ptr(texture), _ptr(indices), _ptr(out), TB, TH, TW, C, B, N, mode,
                                                _stream_ptr(indices.device))
        _lib.check(rc, 'SampleTexture')
        ctx.save_for_backward(texture, indices)
        ctx.mode = mode
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        want_texture, want_indices = ctx.needs_input_grad[:2]
        if not (want_texture or want_indices):
            return None, None, None, None
        texture, indices = ctx.saved_tensors
        TB, TH, TW, C = texture.shape
        B, N = indices.shape[0], indices.shape[1]
        grad_out = grad_out.contiguous().to(torch.float32)
        grad_texture = torch.empty_like(texture) if want_texture else None
        grad_indices = torch.empty_like(indices) if want_indices else None
        # grad_indices alone is per lookup and already reproducible; grad_texture needs the sorted path
        deterministic = want_texture and torch.are_deterministic_algorithms_enabled()
        with torch.cuda.device(indices.device):
            if deterministic:
                L = _lib.lib()
                scratch_bytes = max(int(L.dirt_texture_sample_backward_deterministic_bytes(TB, TH, TW, C, B, N, ctx.mode)), 256)
                scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=indices.device)
                rc = L.dirt_texture_sample_backward_deterministic(
                    _ptr(texture), _ptr(indices), _ptr(grad_out), _ptr(grad_texture), _ptr(grad_indices), TB, TH, TW, C, B, N,
                    ctx.mode, _ptr(scratch), scratch_bytes, _stream_ptr(indices.device))
                if rc == _lib.ERR_BAD_SHAPE:
                    # the shapes passed the forward call: what fails are the sorted path's 32-bit limits
                    raise RuntimeError(
                        'sample_texture backward: the texture gradient has no deterministic implementation for %d lookups '
                        'into %d x %d x %d texels (it needs fewer than 2^31 of each), but '
                        'torch.use_deterministic_algorithms(True) is set' % (B * N, TB, TH, TW))
            else:
                rc = _lib.lib().dirt_texture_sample_backward(_ptr(texture), _ptr(indices), _ptr(grad_out),
                                                             _ptr(grad_texture), _ptr(grad_indices), TB, TH, TW, C, B, N,
                                                             ctx.mode, _stream_ptr(indices.device))
        _lib.check(rc, 'SampleTextureGrad')
        return grad_texture, grad_indices, None, None


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


class _SampleTextureTrilinear(torch.autograd.Function):
    """dirt_texture_sample_trilinear with its gradient.  texture [TB, TH, TW, C], indices [B, N, 2], derivatives
    [B, N, 4], contiguous fp32 CUDA.  The pyramid is built per call and kept for the backward pass."""

    @staticmethod
    def forward(ctx, texture, indices, derivatives, out_shape):
        TB, TH, TW, C = texture.shape
        B, N = indices.shape[0], indices.shape[1]
        L = _lib.lib()
        out = torch.empty(out_shape, dtype=torch.float32, device=indices.device)
        pyramid_floats = int(L.dirt_texture_mip_pyramid_bytes(TB, TH, TW, C)) // 4
        pyramid = torch.empty(pyramid_floats, dtype=torch.float32, device=indices.device) if pyramid_floats else None
        with torch.cuda.device(indices.device):
            stream = _stream_ptr(indices.device)
            rc = L.dirt_texture_mip_build(_ptr(texture), _ptr(pyramid), TB, TH, TW, C, stream)
            _lib.check(rc, 'SampleTextureMipBuild')
            rc = L.dirt_texture_sample_trilinear(_ptr(texture), _ptr(pyramid), _ptr(indices), _ptr(derivatives), _ptr(out),
                                                 TB, TH, TW, C, B, N, stream)
        _lib.check(rc, 'SampleTextureTrilinear')
        ctx.save_for_backward(texture, pyramid, indices, derivatives)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        want_texture, want_indices = ctx.needs_input_grad[:2]
        if not (want_texture or want_indices):
            return None, None, None, None
        texture, pyramid, indices, derivatives = ctx.saved_tensors
        TB, TH, TW, C = texture.shape
        B, N = indices.shape[0], indices.shape[1]
        L = _lib.lib()
        grad_out = grad_out.contiguous().to(torch.float32)
        grad_texture = torch.empty_like(texture) if want_texture else None
        grad_indices = torch.empty_like(indices) if want_indices else None
        deterministic = int(bool(want_texture and torch.are_deterministic_algorithms_enabled()))
        scratch_bytes = int(L.dirt_texture_sample_trilinear_backward_bytes(TB, TH, TW, C, B, N, deterministic))
        scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=indices.device) if scratch_bytes else None
        with torch.cuda.device(indices.device):
            rc = L.dirt_texture_sample_trilinear_backward(
                _ptr(texture), _ptr(pyramid), _ptr(indices), _ptr(derivatives), _ptr(grad_out), _ptr(grad_texture),
                _ptr(grad_indices), TB, TH, TW, C, B, N, deterministic, _ptr(scratch), scratch_bytes,
                _stream_ptr(indices.device))
        if deterministic and rc == _lib.ERR_BAD_SHAPE:
            # the shapes passed the forward call: what fails are the sorted path's 32-bit limits
            raise RuntimeError(
                'sample_texture backward: the texture gradient has no deterministic implementation for %d lookups '
                'into %d x %d x %d texels (it needs fewer than 2^31 of each), but '
                'torch.use_deterministic_algorithms(True) is set' % (B * N, TB, TH, TW))
        _lib.check(rc, 'SampleTextureTrilinearGrad')
        return grad_texture, grad_indices, None, None


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
    texture = _as_f32(texture, device)
    indices = _as_f32(indices, device)
    if texture.dim() not in (3, 4):
        raise ValueError('SampleTexture expects texture to be 3D or 4D, and texture.shape == [height, width, channels] '
                         'or [None, height, width, channels]')
    if texture.shape[-3] <= 0 or texture.shape[-2] <= 0 or texture.shape[-1] <= 0:
        raise ValueError('SampleTexture expects a texture with positive height, width and channels')
    if indices.dim() < 1 or indices.shape[-1] != 2:
        raise ValueError('SampleTexture expects indices.shape[-1] == 2')
    per_item = texture.dim() == 4
    if per_item and (indices.dim() < 2 or indices.shape[0] != texture.shape[0]):
        raise ValueError('SampleTexture expects indices of per-item textures to be at least 2D, and indices.shape[0] == '
                         'texture.shape[0]')
    if mode == 'trilinear':
        derivatives = _as_f32(derivatives, device)
        if tuple(derivatives.shape) != tuple(indices.shape[:-1]) + (4,):
            raise ValueError('SampleTexture expects derivatives.shape == indices.shape[:-1] + (4,), got %s for indices %s'
                             % (tuple(derivatives.shape), tuple(indices.shape)))
        _require_cuda(texture, indices, derivatives)
    else:
        _require_cuda(texture, indices)
    out_shape = tuple(indices.shape[:-1]) + (int(texture.shape[-1]),)
    B = int(indices.shape[0]) if per_item else 1
    N = 1
    for n in indices.shape[(1 if per_item else 0):-1]:
        N *= int(n)
    flat = indices.reshape(B, N, 2).contiguous()
    tex = (texture if per_item else texture[None]).contiguous()
    if mode == 'trilinear':
        return _SampleTextureTrilinear.apply(tex, flat, derivatives.detach().reshape(B, N, 4).contiguous(), out_shape)
    return _SampleTexture.apply(tex, flat, _MODES[mode], out_shape)
