"""Mesh terms for fitting shapes: the mesh Laplacian, a smoothness term on the vertices.

`laplacian` runs CUDA kernels (dirt_laplacian_forward / _backward of include/dirt_b200.h) when its vertices are float32
on a CUDA device in the shapes `lighting.normals_route` accepts, and its torch restatement `_vertex_laplacian`
otherwise; see DESIGN.md §7.16.  The kernels share the vertex normals' adjacency and per-vertex passes, and their
autograd node is the normals' (`lighting._MeshFunction`).
"""
from functools import partial

import torch

from . import _lib
from .lighting import _MeshOp, _mesh, _normals_route, _point_rows, _prepare, _stride, _ptr, _unflat_points

MODES = {'uniform': _lib.LAPLACIAN_UNIFORM, 'cotangent': _lib.LAPLACIAN_COTANGENT}


def _vertex_laplacian(vertices, faces, mode='uniform'):
    """The torch restatement of `laplacian`: its CPU implementation and its specification.  Keeps the dtype of its
    inputs (the tests evaluate it in float64)."""
    _check_mode(mode)
    vertices, faces = _prepare(vertices, faces)
    p = vertices[..., :3]
    corners = p[..., faces, :]   # [*, F, 3, 3]
    if mode == 'cotangent':
        n = torch.linalg.cross(corners[..., 1, :] - corners[..., 0, :], corners[..., 2, :] - corners[..., 0, :], dim=-1)
        area = torch.linalg.vector_norm(n, dim=-1)   # twice the face's area
        cot = [((corners[..., (j + 1) % 3, :] - corners[..., j, :]) * (corners[..., (j + 2) % 3, :] - corners[..., j, :]))
               .sum(-1, keepdim=True) / (area[..., None] + 1.e-12) for j in range(3)]
    S = torch.zeros(corners.shape[:-3] + p.shape[-2:], dtype=corners.dtype, device=corners.device)
    D = torch.zeros(S.shape[:-1], dtype=S.dtype, device=S.device)
    for k in range(3):
        a, b = (k + 1) % 3, (k + 2) % 3
        to_a, to_b = corners[..., a, :] - corners[..., k, :], corners[..., b, :] - corners[..., k, :]
        if mode == 'cotangent':
            s, d = cot[b] * to_a + cot[a] * to_b, area / 3.
        else:
            s, d = to_a + to_b, torch.full(corners.shape[:-2], 2., dtype=S.dtype, device=S.device)
        S = S.index_add(-2, faces[:, k], s)
        D = D.index_add(-1, faces[:, k], d)
    return S / (D[..., None] + 1.e-12)


def _check_mode(mode):
    if mode not in MODES:
        raise ValueError("laplacian: mode must be 'uniform' or 'cotangent', not %r" % (mode,))


def _laplacian_inputs(mode, route, faces, rows):
    """The input arguments of dirt_laplacian_forward / _backward, in their order."""
    return [MODES[mode], _ptr(rows), _stride(rows, 3), _ptr(faces)]


def _restate_laplacian(mode, route, faces, rows):
    return _vertex_laplacian(_unflat_points(rows, route), faces, mode)


_LAPLACIAN = {mode: _MeshOp('Laplacian', 'dirt_laplacian_forward', 'dirt_laplacian_backward',
                            'dirt_laplacian_workspace_bytes', partial(_laplacian_inputs, mode), 3, (3,),
                            partial(_restate_laplacian, mode))
              for mode in MODES}


def laplacian(vertices, faces, mode='uniform', name=None):
    """The mesh Laplacian of each vertex: vertices [*, V, 3|4] (a w column is ignored), faces [F, 3] -> [*, V, 3].

    For corner k of a face that names v, with a = k+1 mod 3 and b = k+2 mod 3, sums over every corner that names v
        uniform:    S_v = sum (p_a - p_v) + (p_b - p_v),          D_v = sum 2
        cotangent:  S_v = sum c_b (p_a - p_v) + c_a (p_b - p_v),  D_v = sum |n_f| / 3
    with n_f = (p1 - p0) x (p2 - p0) and c_j = ((p_{j+1} - p_j) . (p_{j+2} - p_j)) / (|n_f| + 1e-12) the cotangent at
    corner j, and returns S_v / (D_v + 1e-12); a vertex that no face names gets 0.

    The uniform mode is, on a closed manifold mesh, the mean of p_u - p_v over the distinct neighbours u of v; on a
    boundary, boundary edges weigh half.  The cotangent mode is the discrete mean-curvature normal (barycentric areas),
    about -(2/r) n on a sphere of radius r.  As a fitting term, mean |laplacian|^2 keeps a mesh from folding and
    spiking where the image gradient is zero or noisy.  Gradients are torch autograd's of these expressions, through the
    cotangents and the areas; a zero-area face gives the 1e12-scale values the formula implies.

    On CUDA in the shapes `lighting.normals_route` accepts, deterministic kernels compute it (a face with an index
    outside [0, V) is then left out); any other call runs the torch restatement `_vertex_laplacian` (DESIGN.md §7.16)."""
    _check_mode(mode)
    route = _normals_route(vertices, faces)
    if route is None:
        return _vertex_laplacian(vertices, faces, mode)
    return _mesh(_LAPLACIAN[mode], route, faces, _point_rows(vertices[..., :3], 3))
