"""Mesh terms for fitting shapes: the mesh Laplacian, a smoothness term on the vertices, and the edge lengths and
normal consistency of every face edge.

`laplacian` runs CUDA kernels (dirt_laplacian_forward / _backward of include/dirt_b200.h) when its vertices are float32
on a CUDA device in the shapes `lighting.normals_route` accepts, and its torch restatement `_vertex_laplacian`
otherwise; see DESIGN.md §7.16.  `edge_lengths` and `normal_consistency` are routed the same way, between
dirt_edge_terms_forward / _backward and `_edge_lengths` / `_normal_consistency`; see DESIGN.md §7.17.  The kernels
share the vertex normals' adjacency and per-vertex passes, and their autograd node is the normals'
(`lighting._MeshFunction`).
"""
from functools import partial

import torch

from . import _lib
from .lighting import _MeshOp, _face_normals, _mesh, _normals_route, _prepare, _restate_rows, _routed, _rows_inputs

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


_LAPLACIAN = {mode: _MeshOp('Laplacian', 'dirt_laplacian_forward', 'dirt_laplacian_backward',
                            'dirt_laplacian_workspace_bytes', partial(_rows_inputs, MODES[mode]), 3, (3,),
                            partial(_restate_rows, partial(_vertex_laplacian, mode=mode)))
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
    return _routed(_LAPLACIAN[mode], partial(_vertex_laplacian, mode=mode), vertices, faces, _normals_route, _mesh)


# ---- edge lengths and normal consistency (DESIGN.md §7.17) -------------------------------------------------------------

def _edge_lengths(vertices, faces):
    """The torch restatement of `edge_lengths`: its CPU implementation and its specification.  Keeps the dtype of its
    inputs (the tests evaluate it in float64)."""
    vertices, faces = _prepare(vertices, faces)
    corners = vertices[..., :3][..., faces, :]   # [*, F, 3, 3]
    return torch.linalg.vector_norm(corners[..., [1, 2, 0], :] - corners, dim=-1)


def _normal_consistency(vertices, faces):
    """The torch restatement of `normal_consistency`: its CPU implementation and its specification.  Keeps the dtype
    of its inputs (the tests evaluate it in float64).  The half-edges are grouped by their unordered pair of vertices;
    S sums u over the distinct faces of each pair and c counts them, so that the partners of face f sum to S - u_f."""
    vertices, faces = _prepare(vertices, faces)
    u = _face_normals(vertices[..., :3], faces)   # [*, F, 3]
    F, V = faces.shape[0], vertices.shape[-2]
    a, b = faces, faces[:, [1, 2, 0]]
    key = torch.minimum(a, b) * V + torch.maximum(a, b)                                 # [F, 3]
    face = torch.arange(F, device=faces.device)[:, None].expand(F, 3)
    pairs, half_edge = torch.unique(torch.stack([key.reshape(-1), face.reshape(-1)], 1), dim=0, return_inverse=True)
    keys, pair_key = torch.unique(pairs[:, 0], return_inverse=True)                   # each (pair, face) once
    count = torch.zeros(keys.shape[0], dtype=u.dtype, device=u.device).index_add(
        0, pair_key, torch.ones(pairs.shape[0], dtype=u.dtype, device=u.device))
    S = torch.zeros(u.shape[:-2] + (keys.shape[0], 3), dtype=u.dtype, device=u.device).index_add(
        -2, pair_key, u[..., pairs[:, 1], :])
    k = pair_key[half_edge].reshape(F, 3)
    c = count[k]
    partners = (S[..., k, :] - u[..., None, :]) / (c - 1.).clamp(min=1.)[..., None]   # [*, F, 3, 3]
    value = 1. - (u[..., None, :] * partners).sum(-1)
    return torch.where((c > 1.) & (a != b), value, torch.zeros_like(value))


EDGE_MODES = {'edge_lengths': _lib.EDGE_LENGTH, 'normal_consistency': _lib.NORMAL_CONSISTENCY}


_EDGE_LENGTHS = _MeshOp('EdgeLengths', 'dirt_edge_terms_forward', 'dirt_edge_terms_backward',
                        'dirt_edge_terms_workspace_bytes', partial(_rows_inputs, _lib.EDGE_LENGTH), 3, (3,),
                        partial(_restate_rows, _edge_lengths), rows='F')
_NORMAL_CONSISTENCY = _EDGE_LENGTHS._replace(name='NormalConsistency',
                                             inputs=partial(_rows_inputs, _lib.NORMAL_CONSISTENCY),
                                             restate=partial(_restate_rows, _normal_consistency))


def edge_lengths(vertices, faces, name=None):
    """The length of every face edge: vertices [*, V, 3|4] (a w column is ignored), faces [F, 3] -> [*, F, 3].

    Entry k of face f = (v0, v1, v2) is its edge k, from v_k to v_{k+1 mod 3}: |p_{k+1} - p_k|.  An interior edge of a
    manifold mesh appears twice, once from each face.  As a fitting term, for example the variance of the lengths or
    their mean squared offset from the starting lengths, it keeps triangles from collapsing or stretching while the
    mesh deforms.  Gradients are torch autograd's of `torch.linalg.vector_norm`; a zero-length edge passes none.

    On CUDA in the shapes `lighting.normals_route` accepts, deterministic kernels compute it (a face with an index
    outside [0, V) then gets 0 and receives no gradient); any other call runs the torch restatement `_edge_lengths`
    (DESIGN.md §7.17)."""
    return _routed(_EDGE_LENGTHS, _edge_lengths, vertices, faces, _normals_route, _mesh)


def normal_consistency(vertices, faces, name=None):
    """How far each face edge folds: vertices [*, V, 3|4] (a w column is ignored), faces [F, 3] -> [*, F, 3].

    With u_f = n_f / (|n_f| + 1e-12) and n_f = (p1 - p0) x (p2 - p0), entry k of face f, for its edge from a = v_k to
    b = v_{k+1 mod 3}, is
        1 - u_f . (sum of u_g over P) / |P|
    where P holds the faces other than f that name both a and b, each once (also when it names a or b twice); it is 0
    when P is empty (a boundary edge) or a == b.  A flat edge gives 0, a right angle 1 and an edge between a face and
    a reversed neighbour about 2; on a non-manifold edge it averages over all the other faces, and a duplicated face is
    a partner of its copy.  An interior edge of a manifold mesh appears twice, with equal values.  As a fitting term,
    its mean penalises the folds between adjacent faces that a Laplacian does not see directly.  Gradients are torch
    autograd's of this expression; a zero-area face (u_f = 0, value 1) gives the 1e12-scale values the normals' formula
    implies.

    On CUDA in the shapes `lighting.normals_route` accepts, deterministic kernels compute it (a face with an index
    outside [0, V) then gets 0, receives no gradient and is nobody's partner); any other call runs the torch
    restatement `_normal_consistency` (DESIGN.md §7.17)."""
    return _routed(_NORMAL_CONSISTENCY, _normal_consistency, vertices, faces, _normals_route, _mesh)
