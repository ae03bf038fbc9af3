"""Homogeneous transform matrices for row vectors (torch); mirrors the API of dirt/matrices.py.

Matrices RIGHT-multiply the vectors they transform (`vertices @ matrix`), i.e. they are indexed
[..., in, out], exactly as in the reference (dirt/matrices.py:1-9).
"""
import torch


def _t(x, like=None):
    if isinstance(x, torch.Tensor):
        return x if x.is_floating_point() else x.to(torch.float32)
    return torch.as_tensor(x, dtype=torch.float32, device=None if like is None else like.device)


def pad_3x3_to_4x4(matrix, name=None):
    """[*,3,3] -> [*,4,4] with a unit w row/column (dirt/matrices.py:156-180)."""
    matrix = _t(matrix)
    out = torch.zeros(matrix.shape[:-2] + (4, 4), dtype=matrix.dtype, device=matrix.device)
    out[..., :3, :3] = matrix
    out[..., 3, 3] = 1.
    return out


def rodrigues(vectors, name=None, three_by_three=False):
    """Angle-axis vectors [*,3] -> rotation matrices [*,4,4] (or [*,3,3]) (dirt/matrices.py:15-61)."""
    vectors = _t(vectors) + 1.e-12  # keeps the derivative finite at zero, as the reference does
    angle = torch.linalg.norm(vectors, dim=-1, keepdim=True)
    axis = vectors / angle
    angle = angle[..., 0]
    x, y, z = axis[..., 0], axis[..., 1], axis[..., 2]
    zero = torch.zeros_like(x)
    # K indexed [*, in, out] for row vectors
    K = torch.stack([torch.stack([zero, -z, y], dim=-1),
                     torch.stack([z, zero, -x], dim=-1),
                     torch.stack([-y, x, zero], dim=-1)], dim=-2)
    c = torch.cos(angle)[..., None, None]
    s = torch.sin(angle)[..., None, None]
    eye = torch.eye(3, dtype=vectors.dtype, device=vectors.device)
    result = c * eye + (1 - c) * axis[..., :, None] * axis[..., None, :] + s * K
    return result if three_by_three else pad_3x3_to_4x4(result)


def translation(x, name=None):
    """Displacements [*,3] -> translation matrices [*,4,4] (dirt/matrices.py:64-88)."""
    x = _t(x)
    out = torch.eye(4, dtype=x.dtype, device=x.device).expand(x.shape[:-1] + (4, 4)).clone()
    out[..., 3, :3] = x
    return out


def scale(x, name=None):
    """Scale factors [*,3] -> scaling matrices [*,4,4] (dirt/matrices.py:91-107)."""
    x = _t(x)
    return torch.diag_embed(torch.cat([x, torch.ones_like(x[..., :1])], dim=-1))


def perspective_projection(near, far, right, aspect, name=None):
    """OpenGL-convention perspective matrices [A1..An,4,4]; camera looks along -z in view space
    (dirt/matrices.py:110-153).  `aspect` is height / width."""
    near, far, right, aspect = torch.broadcast_tensors(_t(near), _t(far), _t(right), _t(aspect))
    top = right * aspect
    out = torch.zeros(near.shape + (4, 4), dtype=near.dtype, device=near.device)
    out[..., 0, 0] = near / right
    out[..., 1, 1] = near / top
    out[..., 2, 2] = -(far + near) / (far - near)
    out[..., 3, 2] = -2. * far * near / (far - near)
    out[..., 2, 3] = -1.
    return out


def orthographic_projection(left, right, bottom, top, near, far, name=None):
    """OpenGL-convention orthographic matrices [A1..An,4,4] (glOrtho), in the [in, out] layout of
    `perspective_projection`: view-space x in [left, right], y in [bottom, top] and z in [-near, -far] map to clip x, y,
    z in [-1, 1], with w = 1.  The view looks along -z; a directional light's shadow map uses one."""
    left, right, bottom, top, near, far = torch.broadcast_tensors(_t(left), _t(right), _t(bottom), _t(top), _t(near),
                                                                  _t(far))
    out = torch.zeros(near.shape + (4, 4), dtype=near.dtype, device=near.device)
    out[..., 0, 0] = 2. / (right - left)
    out[..., 1, 1] = 2. / (top - bottom)
    out[..., 2, 2] = -2. / (far - near)
    out[..., 3, 0] = -(right + left) / (right - left)
    out[..., 3, 1] = -(top + bottom) / (top - bottom)
    out[..., 3, 2] = -(far + near) / (far - near)
    out[..., 3, 3] = 1.
    return out


def compose(*matrices):
    """Product of the given matrices, the first applied first (dirt/matrices.py:183-207)."""
    if len(matrices) == 0:
        return torch.eye(4)
    result = _t(matrices[0])
    for m in matrices[1:]:
        result = torch.matmul(result, _t(m, result).to(result.device))
    return result
