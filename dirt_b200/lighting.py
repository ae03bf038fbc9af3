"""Mesh normals and simple reflectance models; mirrors the API of dirt/lighting.py.

`vertex_normals` and `vertex_normals_pre_split` run CUDA kernels (dirt_normals_forward / _backward of
include/dirt_b200.h) when their vertices are float32 on a CUDA device in the shapes `normals_route` accepts, and their
torch restatements (`_vertex_normals`, `_vertex_normals_pre_split`) otherwise; see DESIGN.md §7.3.  The three
reflectance models run CUDA kernels (dirt_lighting_forward / _backward) when their inputs are on one CUDA device in the
shapes `cuda_route` accepts, and their torch restatements (`_diffuse_directional`, `_specular_directional`,
`_diffuse_point`) otherwise; see DESIGN.md §7.2.  `diffuse_spherical_harmonics` (order-2 SH environment lighting) is
routed the same way, between dirt_sh_lighting_forward / _backward and `_diffuse_spherical_harmonics`; see DESIGN.md
§7.8.  So are `specular_ggx_directional` and `specular_ggx_point` (GGX microfacet specular), between
dirt_ggx_lighting_forward / _backward and `_specular_ggx`; see DESIGN.md §7.9.  `ggx_environment_brdf` and
`specular_ggx_environment` (split-sum GGX environment lighting, DESIGN.md §7.12) are torch code around a CUDA table and
the CUDA cube-map lookup; `cubemap_spherical_harmonics` projects a cube map onto order-2 SH with CUDA kernels.  `split_vertices_by_face` is torch code.
`vertex_tangents` and `perturb_normals` (tangent-space normal mapping, DESIGN.md §7.14) run CUDA kernels
(dirt_tangents_* and dirt_normal_map_*) in the shapes `tangents_route` and `cuda_route` accept, and their torch
restatements (`_vertex_tangents`, `_perturb_normals`) otherwise.
`shadow_map` rasterises a light-view map of (occupancy, depth) with `rasterise_batch`, and `shadow_visibility` looks it
up with percentage-closer filtering: CUDA kernels (dirt_shadow_forward / _backward) in the shapes `shadow_route`
accepts, its torch restatement `_shadow_visibility` otherwise; see DESIGN.md §7.15.
"""
import math
from collections import namedtuple
from functools import partial

import torch

from . import _lib


def _prepare(vertices, faces):
    vertices = vertices if isinstance(vertices, torch.Tensor) else torch.as_tensor(vertices, dtype=torch.float32)
    faces = faces if isinstance(faces, torch.Tensor) else torch.as_tensor(faces)
    return vertices, faces.to(device=vertices.device, dtype=torch.long)


def _face_normals(vertices, faces):
    corners = vertices[..., faces, :]  # [*, F, 3, 3]
    n = torch.linalg.cross(corners[..., 1, :] - corners[..., 0, :], corners[..., 2, :] - corners[..., 0, :], dim=-1)
    return n / (torch.linalg.norm(n, dim=-1, keepdim=True) + 1.e-12)


def _vertex_normals(vertices, faces):
    """The torch restatement of `vertex_normals`: its CPU implementation and its specification."""
    vertices, faces = _prepare(vertices, faces)
    vertices = vertices[..., :3]
    normals_by_face = _face_normals(vertices, faces)  # [*, F, 3]
    summed = torch.zeros_like(vertices)
    for corner in range(3):
        summed = summed.index_add(-2, faces[:, corner], normals_by_face)
    return summed / (torch.linalg.norm(summed, dim=-1, keepdim=True) + 1.e-12)


def _vertex_normals_pre_split(vertices, faces):
    """The torch restatement of `vertex_normals_pre_split`: its CPU implementation and its specification."""
    vertices, faces = _prepare(vertices, faces)
    vertices = vertices[..., :3]
    normals_by_face = _face_normals(vertices, faces)
    out = torch.zeros_like(vertices)
    for corner in range(3):
        out = out.index_copy(-2, faces[:, corner], normals_by_face)
    return out


def vertex_normals(vertices, faces, name=None):
    """Per-vertex normals: normalised sum of the unit normals of the faces using each vertex
    (dirt/lighting.py:34-93).  vertices [*,V,3|4], faces [F,3] -> [*,V,3].  On CUDA in the shapes `normals_route`
    accepts, kernels compute it (a face with an index outside [0, V) is then left out); any other call runs the torch
    restatement."""
    route = _normals_route(vertices, faces)
    if route is None:
        return _vertex_normals(vertices, faces)
    return _mesh(_NORMALS, route, faces, _point_rows(vertices[..., :3], 3))


def vertex_normals_pre_split(vertices, faces, name=None, static=False):
    """As `vertex_normals` for meshes where every vertex belongs to exactly one face
    (dirt/lighting.py:101-133): each vertex takes the unit normal of its face (of its last face corner, corner-major,
    when there are several).  Routed as `vertex_normals`."""
    route = _normals_route(vertices, faces)
    if route is None:
        return _vertex_normals_pre_split(vertices, faces)
    return _mesh(_NORMALS_PRE_SPLIT, route, faces, _point_rows(vertices[..., :3], 3))


def split_vertices_by_face(vertices, faces, name=None):
    """Duplicates vertices so that each is used by one face: returns (new_vertices [*,3F,D], new_faces [F,3])
    (dirt/lighting.py:136-179)."""
    vertices, faces = _prepare(vertices, faces)
    new_vertices = vertices[..., faces.reshape(-1), :]
    new_faces = torch.arange(faces.shape[0] * 3, device=vertices.device, dtype=torch.int32).reshape(-1, 3)
    return new_vertices, new_faces


def _cosine_term(cosines, double_sided):
    return cosines.abs() if double_sided else cosines.clamp(min=0.)


def _diffuse_directional(vertex_normals, vertex_colors, light_direction, light_color, double_sided=True):
    """The torch restatement of `diffuse_directional`: its CPU implementation and its specification.
    Takes tensors of one dtype and device, and keeps that dtype (the tests evaluate it in float64)."""
    cosines = torch.matmul(vertex_normals, -light_direction[..., None])  # [*, V, 1]
    return light_color[..., None, :] * vertex_colors * _cosine_term(cosines, double_sided)


def _specular_directional(vertex_positions, vertex_normals, vertex_reflectivities, light_direction, light_color,
                          camera_position, shininess, double_sided=True):
    """The torch restatement of `specular_directional`: its CPU implementation and its specification.
    Takes tensors of one dtype and device, and keeps that dtype (the tests evaluate it in float64)."""
    to_light = -light_direction
    # (the reference adds `-to_light` of shape [*,3] to a [*,V,3] tensor, which only broadcasts without batch dimensions,
    # dirt/lighting.py:272; the vertex axis is inserted here so that batches work as its docstring promises)
    reflected = -to_light[..., None, :] + 2. * torch.matmul(vertex_normals, to_light[..., None]) * vertex_normals
    to_camera = camera_position[..., None, :] - vertex_positions
    # the reference adds its epsilon after the division (dirt/lighting.py:279); kept for parity
    cosines = ((to_camera / torch.linalg.norm(to_camera, dim=-1, keepdim=True) + 1.e-12) * reflected).sum(-1, keepdim=True)
    return light_color[..., None, :] * vertex_reflectivities * torch.pow(_cosine_term(cosines, double_sided),
                                                                         shininess[..., None, None])


def _diffuse_point(vertex_positions, vertex_normals, vertex_colors, light_position, light_color, double_sided=True):
    """The torch restatement of `diffuse_point`: its CPU implementation and its specification.
    Takes tensors of one dtype and device, and keeps that dtype (the tests evaluate it in float64)."""
    relative = vertex_positions - light_position[..., None, :]
    incident = relative / (torch.linalg.norm(relative, dim=-1, keepdim=True) + 1.e-12)
    cosines = (vertex_normals * incident).sum(-1)
    return light_color[..., None, :] * vertex_colors * _cosine_term(cosines, double_sided)[..., None]


def _unit(x):
    return x / (torch.linalg.norm(x, dim=-1, keepdim=True) + 1.e-12)


GGX_MIN_ROUGHNESS = 0.045


def _specular_ggx(vertex_positions, vertex_normals, vertex_roughness, vertex_specular, light, light_color,
                  camera_position, point_light, double_sided):
    """The torch restatement of `specular_ggx_directional` (point_light False, `light` a direction) and
    `specular_ggx_point` (`light` a position): their CPU implementation and their specification.  Takes tensors of one
    dtype and device, and keeps that dtype (the tests evaluate it in float64).

    The output is pi * light_color * F * D * Vis * NdotL where NdotL > 0 and NdotV > 0, else 0.  The factor pi makes
    `diffuse_directional(albedo) + specular_ggx_directional(...)` the usual diffuse-plus-GGX model under one light
    intensity: `diffuse_directional` returns albedo * I * cos, which is Lambert's radiance albedo / pi * I * cos times pi.
    Inside the `where`, the points it masks take safe values, so that their gradients are exactly 0 and not NaN."""
    n = _unit(vertex_normals)
    v = _unit(camera_position[..., None, :] - vertex_positions)
    l = _unit(light[..., None, :] - vertex_positions) if point_light else _unit(-light[..., None, :])
    if double_sided:   # turned to face the camera; no flip at exactly 0
        n = torch.where((n * v).sum(-1, keepdim=True) < 0, -n, n)
    n_dot_l = (n * l).sum(-1, keepdim=True)
    n_dot_v = (n * v).sum(-1, keepdim=True)
    h = _unit(l + v)
    n_dot_h = (n * h).sum(-1, keepdim=True)
    v_dot_h = (v * h).sum(-1, keepdim=True)
    lit = (n_dot_l > 0) & (n_dot_v > 0)
    n_dot_l, n_dot_v = torch.where(lit, n_dot_l, 1.), torch.where(lit, n_dot_v, 1.)
    a = vertex_roughness.clamp(min=GGX_MIN_ROUGHNESS)
    alpha2 = (a * a).square()
    # k = NdotH^2 (alpha2 - 1) + 1 for unit n and h, in a form that does not cancel for small alpha2
    k = torch.where(lit, alpha2 * n_dot_h.square() + torch.linalg.cross(n, h, dim=-1).square().sum(-1, keepdim=True), 1.)
    D = alpha2 / (math.pi * k * k)
    vis = 0.5 / (n_dot_l * torch.sqrt(n_dot_v.square() * (1 - alpha2) + alpha2) +
                 n_dot_v * torch.sqrt(n_dot_l.square() * (1 - alpha2) + alpha2))
    m = 1 - v_dot_h
    fresnel = vertex_specular + (1 - vertex_specular) * (m * m).square() * m
    return torch.where(lit, math.pi * light_color[..., None, :] * fresnel * D * vis * n_dot_l, 0.)


def _sh_basis(n):
    """The real order-2 spherical harmonics without the Condon-Shortley phase at n [..., 3], used as given (not
    normalised): [..., 9], index k = l^2 + l + m."""
    x, y, z = n.unbind(-1)
    return torch.stack([torch.full_like(x, 0.28209479177387814),
                        0.4886025119029199 * y, 0.4886025119029199 * z, 0.4886025119029199 * x,
                        1.0925484305920792 * x * y, 1.0925484305920792 * y * z, 0.31539156525252005 * (3 * z * z - 1),
                        1.0925484305920792 * x * z, 0.5462742152960396 * (x * x - y * y)], dim=-1)


def _diffuse_spherical_harmonics(vertex_normals, vertex_colors, coefficients):
    """The torch restatement of `diffuse_spherical_harmonics`: its CPU implementation and its specification.
    Takes tensors of one dtype and device, and keeps that dtype (the tests evaluate it in float64).

    coefficients are the SH coefficients L_lm of the incident radiance; the result is Lambertian reflected radiance,
    albedo * sum_k w_l(k) L_k Y_k(n), with the clamped cosine's band weights A_l / pi = 1, 2/3, 1/4."""
    w = torch.tensor([1., 2 / 3, 2 / 3, 2 / 3, 0.25, 0.25, 0.25, 0.25, 0.25], dtype=coefficients.dtype,
                     device=coefficients.device)
    irradiance = torch.matmul(_sh_basis(vertex_normals), w[:, None] * coefficients)   # [*, V, C]
    return vertex_colors * irradiance


# ---- the CUDA path --------------------------------------------------------------------------------------------------

Route = namedtuple('Route', 'lead B V C per_item')


def cuda_route(point_shapes, item_shapes, devices, point_widths=None):
    """Whether a reflectance call runs the CUDA kernels, decided from shapes and devices alone.

    point_shapes: the shapes of the per-point tensors, colours (or reflectivities) last: [*, V, 3], ..., [*, V, C].
    item_shapes: (shape, width) of each per-item tensor, width 3 (a direction or position), 'C' (the light colour), 0
        (the shininess, a scalar per item) or a tuple of those (the tail (9, 'C') of SH coefficients); each must have
        leading shape exactly `*` (one value per item) or none (shared by all points).
    devices: the devices of all the tensors; they must be one CUDA device.
    point_widths: the last dimension each per-point tensor must have, an int or 'C'; by default 3 for every one but the
        last, which is C (the GGX model's roughness is 1 wide).

    Returns a Route (lead = `*`, B = its product, V, C, per_item flags in the order of item_shapes) or None."""
    devices = list(devices)
    if not devices or any(d.type != 'cuda' for d in devices) or any(d != devices[0] for d in devices):
        return None
    first = tuple(point_shapes[0])
    if len(first) < 2:
        return None
    lead, V, C = first[:-2], first[-2], tuple(point_shapes[-1])[-1] if len(point_shapes[-1]) else 0
    if C < 1:
        return None
    if point_widths is None:
        point_widths = [3] * (len(point_shapes) - 1) + ['C']
    for shape, width in zip(point_shapes, point_widths):
        shape = tuple(shape)
        if len(shape) != len(first) or shape[:-1] != first[:-1] or shape[-1] != (C if width == 'C' else width):
            return None
    per_item = []
    for shape, width in item_shapes:
        if isinstance(width, tuple):
            tail = tuple(C if w == 'C' else w for w in width)
        else:
            width = C if width == 'C' else width
            tail = (width,) if width else ()
        shape = tuple(shape)
        if shape == tail:
            per_item.append(False)
        elif shape == lead + tail:
            per_item.append(True)
        else:
            return None
    B = math.prod(lead)
    if B >= 1 << 31:
        return None
    return Route(lead, B, V, C, tuple(per_item))


def _route(points, items, point_widths=None):
    tensors = list(points) + [t for t, _ in items]
    return cuda_route([t.shape for t in points], [(t.shape, w) for t, w in items], [t.device for t in tensors],
                      point_widths)


def _rows(t, k):
    """A per-point tensor [*, V, k] as [rows, k] with unit stride along k: a view when one exists (for example the
    normals of a G-buffer, gbuffer[..., 7:].reshape(-1, 3)), else a contiguous copy."""
    try:
        r = t.view(-1, k)
    except RuntimeError:
        return t.reshape(-1, k).contiguous()
    return r if k == 1 or r.stride(1) == 1 else r.contiguous()


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _point_stride(t):
    """The row stride of per-point rows in the fused per-point ops' arguments: 0 for one row or an input not read."""
    return t.stride(0) if t is not None and t.shape[0] > 1 else 0


def _flat_item(t, route, per_item):
    """A per-item input [*, ...] as contiguous [B, ...]; a shared one contiguous as it is."""
    return (t.reshape((route.B,) + t.shape[len(route.lead):]) if per_item else t).contiguous()


def _unflat_points(t, route):
    """Per-point rows [rows, k] as [*, V, k]."""
    return t.reshape(route.lead + (route.V, t.shape[-1]))


def _unflat_item(t, route, per_item):
    """A per-item input [B, ...] as [*, ...]; a shared one as it is."""
    return t.reshape(route.lead + t.shape[1:]) if per_item else t


def _stream(device):
    return torch.cuda.current_stream(device).cuda_stream


def _bvc(route):
    return route.B, route.V, route.C


# A fused per-point op: reflectance, GGX, spherical harmonics or normal mapping.
#   name: the op's name in errors (its backward's is name + 'Grad');
#   forward, backward: its entry points in the library;
#   inputs(*flags, route, *inputs): their input arguments, in their order;
#   sizes(route): their size arguments;
#   restate(*flags, route, *inputs): the torch restatement on the op's own inputs, in the output's shape;
#   first_param: the index of the first per-item parameter.  The gradients of these parameters need a partials
#     workspace of workspace_bytes(*sizes(route)) bytes, where workspace_bytes is an entry point; both are None for an
#     op without such parameters, whose backward then takes no workspace.
#   deterministic: for an op whose backward uses float atomics, (entry point, scratch_bytes) of its deterministic
#     backward, which takes the backward's arguments plus (scratch, scratch bytes) before the sizes and runs under
#     torch.use_deterministic_algorithms(True); scratch_bytes(lib, route, want, *inputs) gives the bytes, 0 for none.
_PointOp = namedtuple('_PointOp', 'name forward backward inputs sizes restate first_param workspace_bytes deterministic',
                      defaults=(None, None, None))


class _PointFunction(torch.autograd.Function):
    """The forward entry point of a _PointOp with its gradient.  flags are the op's non-tensor arguments (the model or
    point_light, then double_sided; none for the SH lighting and the normal map).  Per-point inputs are [rows, k] with
    unit stride along k; per-item inputs contiguous [B, ...] or shared.  The node keeps only its inputs: the backward
    kernel recomputes the forward from them."""

    @staticmethod
    def forward(ctx, op, flags, route, *inputs):
        dev = inputs[0].device
        out = torch.empty(route.lead + (route.V, route.C), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            rc = getattr(_lib.lib(), op.forward)(*op.inputs(*flags, route, *inputs), _ptr(out), *op.sizes(route),
                                                 _stream(dev))
        _lib.check(rc, op.name)
        ctx.save_for_backward(*inputs)
        ctx.op, ctx.flags, ctx.route = op, flags, route
        return out

    @staticmethod
    def backward(ctx, grad_out):
        op, flags, route = ctx.op, ctx.flags, ctx.route
        want = ctx.needs_input_grad[3:]
        if not any(want):
            return (None,) * (3 + len(want))
        inputs = ctx.saved_tensors
        if torch.is_grad_enabled():
            # create_graph=True: differentiable gradients through the restatement
            out = op.restate(*flags, route, *inputs)
            wanted = [t for t, w in zip(inputs, want) if w]
            grads = iter(torch.autograd.grad(out, wanted, grad_out, create_graph=True))
            return (None,) * 3 + tuple(next(grads) if w else None for w in want)
        dev = inputs[0].device
        grads = [torch.empty(t.shape, dtype=torch.float32, device=dev) if w else None for t, w in zip(inputs, want)]
        lib = _lib.lib()
        workspace_args = ()
        if op.workspace_bytes is not None:
            ws_bytes = int(getattr(lib, op.workspace_bytes)(*op.sizes(route))) if any(want[op.first_param:]) else 0
            workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if ws_bytes else None
            workspace_args = (_ptr(workspace), ws_bytes)
        entry, scratch_args = op.backward, ()
        if op.deterministic is not None and torch.are_deterministic_algorithms_enabled():
            entry, scratch_bytes = op.deterministic
            sc_bytes = int(scratch_bytes(lib, route, want, *inputs))
            scratch = torch.empty(sc_bytes, dtype=torch.uint8, device=dev) if sc_bytes else None
            scratch_args = (_ptr(scratch), sc_bytes)
        grad_out = grad_out.to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            rc = getattr(lib, entry)(*op.inputs(*flags, route, *inputs), _ptr(grad_out), *[_ptr(g) for g in grads],
                                     *workspace_args, *scratch_args, *op.sizes(route), _stream(dev))
        _lib.check(rc, op.name + 'Grad')
        return (None,) * 3 + tuple(grads)


def _restate(model, double_sided, route, normals, positions, colors, light, light_color, camera, shininess):
    """The restatement on the op's own inputs (flattened per-point rows, per-item rows): its value has the op's output
    shape, and autograd through it gives differentiable gradients (double backward)."""
    p_light, p_color, *p_rest = route.per_item
    n, k = _unflat_points(normals, route), _unflat_points(colors, route)
    L, lc = _unflat_item(light, route, p_light), _unflat_item(light_color, route, p_color)
    if model == _lib.LIGHT_DIFFUSE_DIRECTIONAL:
        return _diffuse_directional(n, k, L, lc, double_sided)
    if model == _lib.LIGHT_DIFFUSE_POINT:
        return _diffuse_point(_unflat_points(positions, route), n, k, L, lc, double_sided)
    return _specular_directional(_unflat_points(positions, route), n, k, L, lc, _unflat_item(camera, route, p_rest[0]),
                                 _unflat_item(shininess, route, p_rest[1]), double_sided)


def _inputs(model, double_sided, route, normals, positions, colors, light, light_color, camera, shininess):
    """The input arguments of dirt_lighting_forward / _backward, in their order."""
    per_item = list(route.per_item) + [False] * (4 - len(route.per_item))
    return [model, int(bool(double_sided)), _ptr(normals), _point_stride(normals), _ptr(positions),
            _point_stride(positions), _ptr(colors), _point_stride(colors), _ptr(light), int(per_item[0]),
            _ptr(light_color), int(per_item[1]), _ptr(camera), int(per_item[2]), _ptr(shininess), int(per_item[3])]


_REFLECTANCE = {model: _PointOp(name, 'dirt_lighting_forward', 'dirt_lighting_backward', _inputs, _bvc, _restate,
                                first_param=3, workspace_bytes='dirt_lighting_workspace_bytes')
                for model, name in ((_lib.LIGHT_DIFFUSE_DIRECTIONAL, 'DiffuseDirectional'),
                                    (_lib.LIGHT_SPECULAR_DIRECTIONAL, 'SpecularDirectional'),
                                    (_lib.LIGHT_DIFFUSE_POINT, 'DiffusePoint'))}


def _reflectance(model, double_sided, route, normals, colors, light, light_color, positions=None, camera=None,
                 shininess=None):
    """The CUDA path of a call that `cuda_route` accepted."""
    flags = list(route.per_item) + [False] * (4 - len(route.per_item))
    items = [_flat_item(t, route, per_item) if t is not None else None
             for t, per_item in zip((light, light_color, camera, shininess), flags)]
    return _PointFunction.apply(_REFLECTANCE[model], (model, double_sided), route, _rows(normals, 3),
                                _rows(positions, 3) if positions is not None else None, _rows(colors, route.C), *items)


def diffuse_directional(vertex_normals, vertex_colors, light_direction, light_color, double_sided=True, name=None):
    """Lambertian reflectance under one directional light (dirt/lighting.py:182-225).

    vertex_normals [*, V, 3], vertex_colors [*, V, C], light_direction [*, 3] or [3], light_color [*, C] or [C]
    -> [*, V, C].  On CUDA in these shapes a fused kernel computes it; any other call runs the torch restatement."""
    vertex_normals = torch.as_tensor(vertex_normals, dtype=torch.float32)
    dev = vertex_normals.device
    vertex_colors = torch.as_tensor(vertex_colors, dtype=torch.float32, device=dev)
    light_direction = torch.as_tensor(light_direction, dtype=torch.float32, device=dev)
    light_color = torch.as_tensor(light_color, dtype=torch.float32, device=dev)
    route = _route([vertex_normals, vertex_colors], [(light_direction, 3), (light_color, 'C')])
    if route is None:
        return _diffuse_directional(vertex_normals, vertex_colors, light_direction, light_color, double_sided)
    return _reflectance(_lib.LIGHT_DIFFUSE_DIRECTIONAL, double_sided, route, vertex_normals, vertex_colors,
                        light_direction, light_color)


def specular_directional(vertex_positions, vertex_normals, vertex_reflectivities, light_direction, light_color,
                         camera_position, shininess, double_sided=True, name=None):
    """Phong reflectance under one directional light (dirt/lighting.py:228-288).

    vertex_positions, vertex_normals [*, V, 3], vertex_reflectivities [*, V, C], light_direction and camera_position
    [*, 3] or [3], light_color [*, C] or [C], shininess [*] or [] -> [*, V, C].  On CUDA in these shapes a fused kernel
    computes it; any other call runs the torch restatement."""
    vertex_positions = torch.as_tensor(vertex_positions, dtype=torch.float32)
    dev = vertex_positions.device
    vertex_normals = torch.as_tensor(vertex_normals, dtype=torch.float32, device=dev)
    vertex_reflectivities = torch.as_tensor(vertex_reflectivities, dtype=torch.float32, device=dev)
    light_direction = torch.as_tensor(light_direction, dtype=torch.float32, device=dev)
    light_color = torch.as_tensor(light_color, dtype=torch.float32, device=dev)
    camera_position = torch.as_tensor(camera_position, dtype=torch.float32, device=dev)
    shininess = torch.as_tensor(shininess, dtype=torch.float32, device=dev)
    route = _route([vertex_positions, vertex_normals, vertex_reflectivities],
                   [(light_direction, 3), (light_color, 'C'), (camera_position, 3), (shininess, 0)])
    if route is None:
        return _specular_directional(vertex_positions, vertex_normals, vertex_reflectivities, light_direction,
                                     light_color, camera_position, shininess, double_sided)
    return _reflectance(_lib.LIGHT_SPECULAR_DIRECTIONAL, double_sided, route, vertex_normals, vertex_reflectivities,
                        light_direction, light_color, vertex_positions, camera_position, shininess)


def diffuse_point(vertex_positions, vertex_normals, vertex_colors, light_position, light_color, double_sided=True, name=None):
    """Lambertian reflectance under one point light (dirt/lighting.py:291-343).

    vertex_positions, vertex_normals [*, V, 3], vertex_colors [*, V, C], light_position [*, 3] or [3], light_color
    [*, C] or [C] -> [*, V, C].  On CUDA in these shapes a fused kernel computes it; any other call runs the torch
    restatement."""
    vertex_positions = torch.as_tensor(vertex_positions, dtype=torch.float32)
    dev = vertex_positions.device
    vertex_normals = torch.as_tensor(vertex_normals, dtype=torch.float32, device=dev)
    vertex_colors = torch.as_tensor(vertex_colors, dtype=torch.float32, device=dev)
    light_position = torch.as_tensor(light_position, dtype=torch.float32, device=dev)
    light_color = torch.as_tensor(light_color, dtype=torch.float32, device=dev)
    route = _route([vertex_positions, vertex_normals, vertex_colors], [(light_position, 3), (light_color, 'C')])
    if route is None:
        return _diffuse_point(vertex_positions, vertex_normals, vertex_colors, light_position, light_color, double_sided)
    return _reflectance(_lib.LIGHT_DIFFUSE_POINT, double_sided, route, vertex_normals, vertex_colors, light_position,
                        light_color, vertex_positions)


# ---- the CUDA path of the GGX specular model -------------------------------------------------------------------------

def _ggx_inputs(point_light, double_sided, route, normals, positions, roughness, specular, light, light_color, camera):
    """The input arguments of dirt_ggx_lighting_forward / _backward, in their order."""
    return [int(bool(point_light)), int(bool(double_sided)), _ptr(normals), _point_stride(normals), _ptr(positions),
            _point_stride(positions), _ptr(roughness), _point_stride(roughness), _ptr(specular), _point_stride(specular),
            _ptr(light), int(route.per_item[0]), _ptr(light_color), int(route.per_item[1]), _ptr(camera),
            int(route.per_item[2])]


def _restate_ggx(point_light, double_sided, route, normals, positions, roughness, specular, light, light_color, camera):
    """The restatement on the op's own inputs (flattened per-point rows, per-item rows)."""
    points = [_unflat_points(t, route) for t in (positions, normals, roughness, specular)]
    items = [_unflat_item(t, route, per_item) for t, per_item in zip((light, light_color, camera), route.per_item)]
    return _specular_ggx(*points, *items, point_light, double_sided)


_GGX = _PointOp('SpecularGGX', 'dirt_ggx_lighting_forward', 'dirt_ggx_lighting_backward', _ggx_inputs, _bvc,
                _restate_ggx, first_param=4, workspace_bytes='dirt_lighting_workspace_bytes')


def _specular_ggx_call(point_light, vertex_positions, vertex_normals, vertex_roughness, vertex_specular, light,
                       light_color, camera_position, double_sided):
    vertex_positions = torch.as_tensor(vertex_positions, dtype=torch.float32)
    dev = vertex_positions.device
    f = lambda t: torch.as_tensor(t, dtype=torch.float32, device=dev)
    vertex_normals, vertex_roughness, vertex_specular = f(vertex_normals), f(vertex_roughness), f(vertex_specular)
    light, light_color, camera_position = f(light), f(light_color), f(camera_position)
    route = _route([vertex_positions, vertex_normals, vertex_roughness, vertex_specular],
                   [(light, 3), (light_color, 'C'), (camera_position, 3)], [3, 3, 1, 'C'])
    if route is None:
        return _specular_ggx(vertex_positions, vertex_normals, vertex_roughness, vertex_specular, light, light_color,
                             camera_position, point_light, double_sided)
    items = [_flat_item(t, route, per_item) for t, per_item in zip((light, light_color, camera_position), route.per_item)]
    return _PointFunction.apply(_GGX, (point_light, double_sided), route, _rows(vertex_normals, 3),
                                _rows(vertex_positions, 3), _rows(vertex_roughness, 1), _rows(vertex_specular, route.C),
                                *items)


def specular_ggx_directional(vertex_positions, vertex_normals, vertex_roughness, vertex_specular, light_direction,
                             light_color, camera_position, double_sided=False, name=None):
    """GGX microfacet specular reflectance (Cook-Torrance: Trowbridge-Reitz distribution, height-correlated Smith
    visibility, Schlick Fresnel) under one directional light travelling along `light_direction`.

    vertex_positions, vertex_normals [*, V, 3], vertex_roughness [*, V, 1] (perceptual roughness a, clamped below at
    0.045; the distribution uses a^4), vertex_specular [*, V, C] (F0), light_direction and camera_position [*, 3] or
    [3], light_color [*, C] or [C] -> [*, V, C]: pi * light_color * F * D * Vis * (n . l) where n . l > 0 and n . v > 0,
    else 0.  With the factor pi, `diffuse_directional(albedo) + specular_ggx_directional(...)` is the usual
    diffuse-plus-GGX model under one light intensity.  double_sided turns normals facing away from the camera towards
    it.  On CUDA in these shapes fused kernels compute it, with reproducible parameter gradients; any other call runs
    the torch restatement `_specular_ggx`."""
    return _specular_ggx_call(False, vertex_positions, vertex_normals, vertex_roughness, vertex_specular,
                              light_direction, light_color, camera_position, double_sided)


def specular_ggx_point(vertex_positions, vertex_normals, vertex_roughness, vertex_specular, light_position, light_color,
                       camera_position, double_sided=False, name=None):
    """As `specular_ggx_directional`, under one point light at `light_position`: l = normalize(light_position - p)
    points from the surface towards the light (unlike `diffuse_point`'s incident direction), and, like
    `diffuse_point`, there is no distance falloff."""
    return _specular_ggx_call(True, vertex_positions, vertex_normals, vertex_roughness, vertex_specular,
                              light_position, light_color, camera_position, double_sided)


# ---- split-sum GGX image-based lighting (DESIGN.md §7.12) ----------------------------------------------------------

GGX_BRDF_TABLE_SIZE = 128
_BRDF_TABLES = {}


def _ggx_brdf_table(device):
    """The split-sum table [N, N, 2] of dirt_ggx_brdf_table on `device`, built once per device."""
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device())
    if key not in _BRDF_TABLES:
        N = GGX_BRDF_TABLE_SIZE
        table = torch.empty((N, N, 2), dtype=torch.float32, device=device)
        with torch.cuda.device(device):
            rc = _lib.lib().dirt_ggx_brdf_table(table.data_ptr(), N, torch.cuda.current_stream(device).cuda_stream)
        _lib.check(rc, 'GGXBRDFTable')
        _BRDF_TABLES[key] = table
    return _BRDF_TABLES[key]


def ggx_environment_brdf(n_dot_v, roughness):
    """The split-sum GGX BRDF (A, B): the integrals over light directions of (1 - F_c) D Vis (n.l) and F_c D Vis (n.l),
    F_c = (1 - v.h)^5, with `specular_ggx_directional`'s D and Vis (roughness clamped below at 0.045).  Under a uniform
    environment of radiance E, E * (F0 * A + B) is `specular_ggx_directional / pi` integrated over light directions.

    n_dot_v, roughness: float32 CUDA tensors (or floats), broadcastable together -> [..., 2].  A bilinear read of a
    128 x 128 table (nodes at (i + 0.5) / 128 on both axes, clamped to the outer nodes), differentiable in both
    arguments; the table comes from a CUDA kernel and is kept once per device."""
    device = next((t.device for t in (n_dot_v, roughness) if isinstance(t, torch.Tensor)), None)
    if device is None or device.type != 'cuda':
        device = torch.device('cuda')
    n_dot_v = torch.as_tensor(n_dot_v, dtype=torch.float32, device=device)
    roughness = torch.as_tensor(roughness, dtype=torch.float32, device=device)
    n_dot_v, roughness = torch.broadcast_tensors(n_dot_v, roughness)
    table = _ggx_brdf_table(device)
    N = table.shape[0]

    def split(u):
        x = (u * N - 0.5).clamp(0., N - 1.)
        i0 = x.detach().floor().clamp(max=N - 2).long()
        return i0, (x - i0)[..., None]

    i0, fx = split(n_dot_v)
    j0, fy = split(roughness)
    return ((table[i0, j0] * (1. - fy) + table[i0, j0 + 1] * fy) * (1. - fx) +
            (table[i0 + 1, j0] * (1. - fy) + table[i0 + 1, j0 + 1] * fy) * fx)


class _CubemapSH(torch.autograd.Function):
    """dirt_cubemap_sh_project / _backward: cubemap [TB, 6, S, S, C] contiguous fp32 CUDA -> [TB, 9, C]."""

    @staticmethod
    def forward(ctx, cubemap):
        TB, _, S, _, C = cubemap.shape
        L = _lib.lib()
        out = torch.empty((TB, 9, C), dtype=torch.float32, device=cubemap.device)
        nbytes = int(L.dirt_cubemap_sh_project_bytes(TB, S, C))
        scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=cubemap.device)
        with torch.cuda.device(cubemap.device):
            rc = L.dirt_cubemap_sh_project(cubemap.data_ptr(), out.data_ptr(), scratch.data_ptr(), nbytes, TB, S, C,
                                           torch.cuda.current_stream(cubemap.device).cuda_stream)
        _lib.check(rc, 'CubemapSH')
        ctx.shape = (TB, S, C)
        return out

    @staticmethod
    def backward(ctx, grad):
        TB, S, C = ctx.shape
        L = _lib.lib()
        grad = grad.contiguous().to(torch.float32)
        out = torch.empty((TB, 6, S, S, C), dtype=torch.float32, device=grad.device)
        nbytes = int(L.dirt_cubemap_sh_project_bytes(TB, S, C))
        scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=grad.device)
        with torch.cuda.device(grad.device):
            rc = L.dirt_cubemap_sh_project_backward(grad.data_ptr(), out.data_ptr(), scratch.data_ptr(), nbytes, TB, S, C,
                                                    torch.cuda.current_stream(grad.device).cuda_stream)
        _lib.check(rc, 'CubemapSHGrad')
        return out


def cubemap_spherical_harmonics(cubemap):
    """The order-2 SH coefficients of the radiance in a cube map: L_k = sum_j L(l_j) Y_k(l_j) Omega_j over its texels,
    with the texel directions and solid angles of the split-sum prefilter (DESIGN.md §7.12) and the basis of
    `diffuse_spherical_harmonics`, which takes the result as it stands, so that diffuse and specular lighting come from
    one map.

    cubemap: float32 CUDA tensor [6, S, S, C] or [B, 6, S, S, C] -> [9, C] or [B, 9, C].  A CUDA reduction in a fixed
    order (float64 partial sums), so bit-reproducible; the gradient to the cube map is elementwise."""
    if not isinstance(cubemap, torch.Tensor) or cubemap.device.type != 'cuda':
        raise RuntimeError('cubemap_spherical_harmonics needs a CUDA tensor (there is no CPU kernel)')
    if cubemap.dim() not in (4, 5) or cubemap.shape[-4] != 6 or cubemap.shape[-3] != cubemap.shape[-2] or \
            cubemap.shape[-2] <= 0 or cubemap.shape[-1] <= 0:
        raise ValueError('cubemap_spherical_harmonics expects cubemap.shape == [6, S, S, C] or [B, 6, S, S, C]')
    per_item = cubemap.dim() == 5
    cube = (cubemap if per_item else cubemap[None]).to(torch.float32).contiguous()
    out = _CubemapSH.apply(cube)
    return out if per_item else out[0]


def specular_ggx_environment(vertex_positions, vertex_normals, vertex_roughness, vertex_specular, cubemap,
                             camera_position, double_sided=True, name=None):
    """GGX specular reflection of an environment cube map, by the split-sum approximation: the cube map prefiltered
    with the GGX lobe (`sample_cubemap(..., mode='ggx')`) read in the mirror direction, times F0 * A + B of
    `ggx_environment_brdf`.  In radiance units, like `diffuse_spherical_harmonics`.

    vertex_positions, vertex_normals [*, V, 3], vertex_roughness [*, V, 1], vertex_specular [*, V, C] (F0), cubemap
    [6, S, S, C] (shared) or [B, 6, S, S, C] (one per item, with * = B), camera_position [*, 3] or [3] -> [*, V, C].
    As in `specular_ggx_directional`, v runs towards the camera, double_sided turns normals facing away from it towards
    it, and the result is 0 where n . v <= 0.  Composed in torch from the CUDA lookup and table."""
    from .texture import sample_cubemap
    n = _unit(vertex_normals)
    v = _unit(camera_position[..., None, :] - vertex_positions)
    if double_sided:
        n = torch.where((n * v).sum(-1, keepdim=True) < 0, -n, n)
    n_dot_v = (n * v).sum(-1, keepdim=True)
    lit = n_dot_v > 0
    reflected = 2. * n_dot_v * n - v
    roughness = vertex_roughness[..., 0]
    radiance = sample_cubemap(cubemap, reflected, mode='ggx', roughness=roughness)
    ab = ggx_environment_brdf(n_dot_v[..., 0].clamp(0., 1.), roughness)
    return torch.where(lit, radiance * (vertex_specular * ab[..., :1] + ab[..., 1:]), 0.)


# ---- the CUDA path of the spherical-harmonics lighting --------------------------------------------------------------

def _sh_inputs(route, normals, albedo, coefficients):
    """The input arguments of dirt_sh_lighting_forward / _backward, in their order."""
    return [_ptr(normals), _point_stride(normals), _ptr(albedo), _point_stride(albedo), _ptr(coefficients),
            int(route.per_item[0])]


def _restate_sh(route, normals, albedo, coefficients):
    """The restatement on the op's own inputs (flattened per-point rows, per-item coefficients)."""
    return _diffuse_spherical_harmonics(_unflat_points(normals, route), _unflat_points(albedo, route),
                                        _unflat_item(coefficients, route, route.per_item[0]))


_SH = _PointOp('DiffuseSphericalHarmonics', 'dirt_sh_lighting_forward', 'dirt_sh_lighting_backward', _sh_inputs, _bvc,
               _restate_sh, first_param=2, workspace_bytes='dirt_sh_lighting_workspace_bytes')


def diffuse_spherical_harmonics(vertex_normals, vertex_colors, coefficients, name=None):
    """Lambertian reflectance under an environment given as order-2 spherical harmonics (Ramamoorthi & Hanrahan 2001).

    vertex_normals [*, V, 3] (used as given, not normalised), vertex_colors [*, V, C] (the albedo), coefficients
    [*, 9, C] (one set per item) or [9, C] (shared): the SH coefficients L_lm of the incident radiance, k = l^2 + l + m,
    real basis without the Condon-Shortley phase -> [*, V, C] reflected radiance,
    albedo * sum_k w_l(k) L_k Y_k(n) with w = (1, 2/3, 1/4).  A uniform environment of radiance 1 is
    L = (2 sqrt(pi), 0, ..., 0) and returns the albedo.  On CUDA in these shapes a fused kernel computes it, with a
    bit-reproducible coefficient gradient; any other call runs the torch restatement."""
    vertex_normals = torch.as_tensor(vertex_normals, dtype=torch.float32)
    dev = vertex_normals.device
    vertex_colors = torch.as_tensor(vertex_colors, dtype=torch.float32, device=dev)
    coefficients = torch.as_tensor(coefficients, dtype=torch.float32, device=dev)
    route = _route([vertex_normals, vertex_colors], [(coefficients, (9, 'C'))])
    if route is None:
        return _diffuse_spherical_harmonics(vertex_normals, vertex_colors, coefficients)
    return _PointFunction.apply(_SH, (), route, _rows(vertex_normals, 3), _rows(vertex_colors, route.C),
                                _flat_item(coefficients, route, route.per_item[0]))


# ---- the CUDA path of the normals and of every mesh op -------------------------------------------------------------

NormalsRoute = namedtuple('NormalsRoute', 'lead B V F')


def normals_route(vertex_shape, vertex_dtype, vertex_device, face_shape, face_dtype):
    """Whether a normals call runs the CUDA kernels, decided from shapes, dtypes and devices alone: float32 vertices
    [*, V, 3] or [*, V, 4] on a CUDA device, with prod(*) < 2^31 and V < 2^31, and int32 or int64 faces [F, 3] on any
    device, with 3F < 2^31.  Returns a NormalsRoute (lead = `*`, B = its product, V, F) or None."""
    vertex_shape, face_shape = tuple(vertex_shape), tuple(face_shape)
    if vertex_device.type != 'cuda' or vertex_dtype != torch.float32 or face_dtype not in (torch.int32, torch.int64):
        return None
    if len(vertex_shape) < 2 or vertex_shape[-1] not in (3, 4) or len(face_shape) != 2 or face_shape[1] != 3:
        return None
    lead, V, F = vertex_shape[:-2], vertex_shape[-2], face_shape[0]
    B = math.prod(lead)
    if B >= 1 << 31 or V >= 1 << 31 or 3 * F >= 1 << 31:
        return None
    return NormalsRoute(lead, B, V, F)


def _normals_route(vertices, faces):
    if not isinstance(vertices, torch.Tensor):
        return None
    faces = faces if isinstance(faces, torch.Tensor) else torch.as_tensor(faces)
    return normals_route(vertices.shape, vertices.dtype, vertices.device, faces.shape, faces.dtype)


def _point_rows(t, k):
    """`_rows`, with a row stride of at least k (the C ABI's requirement for these rows)."""
    r = _rows(t, k)
    return r.contiguous() if r.shape[0] > 1 and r.stride(0) < k else r


def _stride(rows, k):
    return rows.stride(0) if rows.shape[0] > 1 else k


# A mesh op: vertex normals (either mode), vertex tangents, the Laplacian or an edge term.  Its forward builds a
# corner-adjacency workspace of workspace_bytes(B, V, F) bytes, where workspace_bytes is an entry point, and its
# backward reads that adjacency.
#   name: the op's name in errors (its backward's is name + 'Grad');
#   forward, backward: its entry points in the library;
#   inputs(route, faces, *inputs): their input arguments, in their order;
#   width: the width of the output rows; input_widths: the width of each input's gradient rows, B*V of them;
#   restate(route, faces, *inputs): the torch restatement on the op's own inputs and the faces the kernels use, in the
#     output's shape;
#   finish(route, grads): turns the backward's gradient rows into the inputs' gradients; None where they are the same;
#   rows: 'V' for one output row per (item, vertex), 'F' for one per (item, face).
_MeshOp = namedtuple('_MeshOp', 'name forward backward workspace_bytes inputs width input_widths restate finish rows',
                     defaults=(None, 'V'))


class _MeshFunction(torch.autograd.Function):
    """The forward entry point of a _MeshOp with its gradient.  faces: int32 [F, 3] on the inputs' device; inputs: the
    op's per-vertex rows, [B*V, k] ([V, k] for shared uvs) with unit stride along k and a row stride of at least k.  The
    node keeps its inputs and the forward's workspace, whose adjacency the backward kernels read."""

    @staticmethod
    def forward(ctx, op, route, faces, *inputs):
        dev = inputs[0].device
        lib = _lib.lib()
        out = torch.empty((route.B * getattr(route, op.rows), op.width), dtype=torch.float32, device=dev)
        ws_bytes = int(getattr(lib, op.workspace_bytes)(route.B, route.V, route.F))
        workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if ws_bytes else None
        with torch.cuda.device(dev):
            rc = getattr(lib, op.forward)(*op.inputs(route, faces, *inputs), _ptr(out), _ptr(workspace), ws_bytes,
                                          route.B, route.V, route.F, _stream(dev))
        _lib.check(rc, op.name)
        ctx.save_for_backward(faces, *inputs)
        ctx.op, ctx.route, ctx.workspace, ctx.ws_bytes = op, route, workspace, ws_bytes
        return out

    @staticmethod
    def backward(ctx, grad_out):
        op, route = ctx.op, ctx.route
        want = ctx.needs_input_grad[3:]
        if not any(want):
            return (None,) * (3 + len(want))
        faces, *inputs = ctx.saved_tensors
        if torch.is_grad_enabled():
            # create_graph=True: differentiable gradients through the restatement, on the faces the kernels used; a
            # per-face output has the rows of the faces left out back as zeros
            valid = ((faces >= 0) & (faces < route.V)).all(1)
            out = op.restate(route, faces[valid], *inputs)
            if op.rows == 'F':
                out = out.new_zeros(route.lead + (route.F, op.width)).index_copy(-2, valid.nonzero()[:, 0], out)
            wanted = [t for t, w in zip(inputs, want) if w]
            grads = iter(torch.autograd.grad(out, wanted, grad_out.reshape(out.shape), create_graph=True))
            return (None,) * 3 + tuple(next(grads) if w else None for w in want)
        dev = inputs[0].device
        grads = [torch.empty((route.B * route.V, k), dtype=torch.float32, device=dev) if w else None
                 for k, w in zip(op.input_widths, want)]
        grad_out = grad_out.to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            rc = getattr(_lib.lib(), op.backward)(*op.inputs(route, faces, *inputs), _ptr(grad_out),
                                                  *[_ptr(g) for g in grads], _ptr(ctx.workspace), ctx.ws_bytes,
                                                  route.B, route.V, route.F, _stream(dev))
        _lib.check(rc, op.name + 'Grad')
        return (None,) * 3 + tuple(op.finish(route, grads) if op.finish else grads)


def _mesh(op, route, faces, *inputs):
    """The CUDA path of a mesh op's call that its route accepted, on its per-vertex rows (`_point_rows`)."""
    faces = torch.as_tensor(faces).to(device=inputs[0].device)
    if faces.dtype == torch.int64:
        faces = faces.clamp(-1, (1 << 31) - 1)   # above int32: >= V, so left out like any other invalid index
    out = _MeshFunction.apply(op, route, faces.to(torch.int32).contiguous(), *inputs)
    return out.reshape(route.lead + (getattr(route, op.rows), op.width))


def _normals_inputs(mode, route, faces, rows):
    """The input arguments of dirt_normals_forward / _backward, in their order."""
    return [mode, _ptr(rows), _stride(rows, 3), _ptr(faces)]


def _restate_normals(restate, route, faces, rows):
    return restate(_unflat_points(rows, route), faces)


_NORMALS = _MeshOp('VertexNormals', 'dirt_normals_forward', 'dirt_normals_backward', 'dirt_normals_workspace_bytes',
                   partial(_normals_inputs, _lib.NORMALS_AVERAGE), 3, (3,), partial(_restate_normals, _vertex_normals))
_NORMALS_PRE_SPLIT = _NORMALS._replace(name='VertexNormalsPreSplit',
                                       inputs=partial(_normals_inputs, _lib.NORMALS_PRE_SPLIT),
                                       restate=partial(_restate_normals, _vertex_normals_pre_split))


# ---- tangent-space normal mapping (DESIGN.md §7.14) -------------------------------------------------------------------

def _vertex_tangents(vertices, uvs, faces, vertex_normals):
    """The torch restatement of `vertex_tangents`: its CPU implementation and its specification.  Keeps the dtype of its
    inputs (the tests evaluate it in float64)."""
    vertices, faces = _prepare(vertices, faces)
    p = vertices[..., :3]
    uvs = uvs if isinstance(uvs, torch.Tensor) else torch.as_tensor(uvs, dtype=p.dtype, device=p.device)
    n = vertex_normals if isinstance(vertex_normals, torch.Tensor) else torch.as_tensor(vertex_normals, dtype=p.dtype,
                                                                                        device=p.device)
    corners, tex = p[..., faces, :], uvs[..., faces, :]   # [*, F, 3, 3], [*, F, 3, 2]
    e1, e2 = corners[..., 1, :] - corners[..., 0, :], corners[..., 2, :] - corners[..., 0, :]
    d1, d2 = tex[..., 1, :] - tex[..., 0, :], tex[..., 2, :] - tex[..., 0, :]
    du1, dv1, du2, dv2 = d1[..., :1], d1[..., 1:], d2[..., :1], d2[..., 1:]
    s = torch.sign(du1 * dv2 - du2 * dv1)
    t_f = _unit(s * (e1 * dv2 - e2 * dv1))   # the unit dp/du direction of each face
    b_f = _unit(s * (e2 * du1 - e1 * du2))   # the unit dp/dv direction
    t_v = b_v = torch.zeros(t_f.shape[:-2] + p.shape[-2:], dtype=t_f.dtype, device=t_f.device)
    for corner in range(3):
        t_v = t_v.index_add(-2, faces[:, corner], t_f)
    for corner in range(3):
        b_v = b_v.index_add(-2, faces[:, corner], b_f)
    n = _unit(n)
    T = _unit(t_v - (n * t_v).sum(-1, keepdim=True) * n)
    w = 1. - 2. * ((torch.linalg.cross(n, T, dim=-1) * b_v).sum(-1, keepdim=True) < 0).to(T.dtype)
    return torch.cat([T, w], -1)


def _perturb_normals(normals, tangents, tangent_space_normals):
    """The torch restatement of `perturb_normals`: its CPU implementation and its specification.  Keeps the dtype of its
    inputs (the tests evaluate it in float64)."""
    n = _unit(normals)
    t = tangents[..., :3]
    T = _unit(t - (n * t).sum(-1, keepdim=True) * n)
    s = 1. - 2. * (tangents[..., 3:] < 0).to(T.dtype)
    m = tangent_space_normals
    return _unit(m[..., :1] * T + m[..., 1:2] * (s * torch.linalg.cross(n, T, dim=-1)) + m[..., 2:] * n)


TangentsRoute = namedtuple('TangentsRoute', 'lead B V F uv_per_item')


def tangents_route(vertex, uv, normal, face_shape, face_dtype):
    """Whether a `vertex_tangents` call runs the CUDA kernels, decided from shapes, dtypes and devices alone.  vertex,
    uv and normal are (shape, dtype, device) of the vertices, uvs and vertex normals.  The vertices and faces must be
    as `normals_route` accepts them; the uvs float32 [V, 2] (shared) or [*, V, 2] and the normals float32 [*, V, 3],
    both on the vertices' device.  Returns a TangentsRoute (lead = `*`, B, V, F, uv_per_item) or None."""
    r = normals_route(vertex[0], vertex[1], vertex[2], face_shape, face_dtype)
    if r is None:
        return None
    for shape, dtype, device in (uv, normal):
        if dtype != torch.float32 or device != vertex[2]:
            return None
    if tuple(normal[0]) != r.lead + (r.V, 3):
        return None
    if tuple(uv[0]) == (r.V, 2):
        per_item = False
    elif tuple(uv[0]) == r.lead + (r.V, 2):
        per_item = True
    else:
        return None
    return TangentsRoute(r.lead, r.B, r.V, r.F, per_item)


def _tangents_route(vertices, uvs, vertex_normals, faces):
    if not all(isinstance(t, torch.Tensor) for t in (vertices, uvs, vertex_normals)):
        return None
    faces = faces if isinstance(faces, torch.Tensor) else torch.as_tensor(faces)
    meta = lambda t: (t.shape, t.dtype, t.device)
    return tangents_route(meta(vertices), meta(uvs), meta(vertex_normals), faces.shape, faces.dtype)


def _tangent_inputs(route, faces, rows, uvs, normals):
    """The input arguments of dirt_tangents_forward / _backward, in their order."""
    uv_stride = _stride(uvs, 2)
    return [_ptr(rows), _stride(rows, 3), _ptr(uvs), uv_stride, route.V * uv_stride if route.uv_per_item else 0,
            _ptr(normals), _stride(normals, 3), _ptr(faces)]


def _restate_tangents(route, faces, rows, uvs, normals):
    return _vertex_tangents(_unflat_points(rows, route), _unflat_points(uvs, route) if route.uv_per_item else uvs,
                            faces, _unflat_points(normals, route))


def _sum_shared_uvs(route, grads):
    """Shared uvs: their gradient rows [B*V, 2] as [V, 2], by one fixed-order sum over the items."""
    g_rows, g_uvs, g_normals = grads
    if g_uvs is not None and not route.uv_per_item:
        g_uvs = g_uvs.reshape(route.B, route.V, 2).sum(0)
    return g_rows, g_uvs, g_normals


_TANGENTS = _MeshOp('VertexTangents', 'dirt_tangents_forward', 'dirt_tangents_backward',
                    'dirt_tangents_workspace_bytes', _tangent_inputs, 4, (3, 2, 3), _restate_tangents, _sum_shared_uvs)


def vertex_tangents(vertices, uvs, faces, vertex_normals, name=None):
    """Per-vertex tangent frames for tangent-space normal mapping.

    vertices [*, V, 3|4] (a w column is ignored), uvs [V, 2] (shared by the batch) or [*, V, 2], faces [F, 3] int32 or
    int64, vertex_normals [*, V, 3] (for example `vertex_normals(vertices, faces)`) -> [*, V, 4]: a unit tangent T
    orthogonal to the vertex normal, along the sum over the vertex's face corners of each face's unit dp/du direction,
    and a handedness w = +-1, so that the bitangent w (n x T) points along +v.  Faces with degenerate uvs add nothing,
    a vertex no face names gets (0, 0, 0, 1), and mirrored uvs give w = -1.  Gradients reach the positions, the v
    coordinates of the uvs (u enters only through the sign of the uv area) and the normals; none passes through w.
    On CUDA in the shapes `tangents_route` accepts, deterministic kernels compute it (a face with an index outside
    [0, V) is then left out); any other call runs the torch restatement `_vertex_tangents` (DESIGN.md §7.14)."""
    route = _tangents_route(vertices, uvs, vertex_normals, faces)
    if route is None:
        return _vertex_tangents(vertices, uvs, faces, vertex_normals)
    return _mesh(_TANGENTS, route, faces, _point_rows(vertices[..., :3], 3), _point_rows(uvs, 2),
                 _point_rows(vertex_normals, 3))


def _normal_map_inputs(route, normals, tangents, samples):
    """The input arguments of dirt_normal_map_forward / _backward, in their order."""
    return [_ptr(normals), _point_stride(normals), _ptr(tangents), _point_stride(tangents), _ptr(samples),
            _point_stride(samples)]


def _restate_normal_map(route, normals, tangents, samples):
    """The restatement on the op's own inputs (flattened per-point rows)."""
    return _perturb_normals(*[_unflat_points(t, route) for t in (normals, tangents, samples)])


# its entry points take no channel count: the output rows are 3 wide
_NORMAL_MAP = _PointOp('PerturbNormals', 'dirt_normal_map_forward', 'dirt_normal_map_backward', _normal_map_inputs,
                       lambda route: (route.B, route.V), _restate_normal_map)


def perturb_normals(normals, tangents, tangent_space_normals, name=None):
    """Tangent-space normal mapping: the normals rotated by a normal map's samples in the frame (n, T, s (n x T)).

    normals [*, N, 3] (interpolated, so not unit length), tangents [*, N, 4] (the interpolated output of
    `vertex_tangents`), tangent_space_normals [*, N, 3] (already decoded to [-1, 1], e.g. 2 * sample_texture(...) - 1;
    the decoding and the green-channel convention are the caller's) -> [*, N, 3]:
    unit(m.x T + m.y s (n x T) + m.z n) with n = unit(normals), T = unit(t - (n . t) n), s = -1 if t.w < 0 else +1.
    A point with a zero normal (a background pixel) gives 0.  Gradients reach the normals, the tangents' xyz and the
    samples.  On CUDA in these shapes a fused kernel computes it, reading G-buffer channel slices in place; any other
    call runs the torch restatement `_perturb_normals` (DESIGN.md §7.14)."""
    normals = torch.as_tensor(normals, dtype=torch.float32)
    dev = normals.device
    tangents = torch.as_tensor(tangents, dtype=torch.float32, device=dev)
    tangent_space_normals = torch.as_tensor(tangent_space_normals, dtype=torch.float32, device=dev)
    route = _route([normals, tangents, tangent_space_normals], [], [3, 4, 3])
    if route is None:
        return _perturb_normals(normals, tangents, tangent_space_normals)
    return _PointFunction.apply(_NORMAL_MAP, (), route, _rows(normals, 3), _rows(tangents, 4),
                                _rows(tangent_space_normals, 3))


# ---- shadow mapping (DESIGN.md §7.15) --------------------------------------------------------------------------------

SHADOW_MAX_RADIUS = 3


def shadow_map(vertices, faces, light_matrix, height, width):
    """A shadow map: the mesh rasterised from the light, [*, height, width, 2] = (occupancy, depth) per texel.

    vertices [*, V, 3|4] world positions (a w column is ignored), faces [F, 3] or [*, F, 3], light_matrix [*, 4, 4] or
    [4, 4] world -> light clip (row vectors, as in `matrices`, e.g. a view matrix composed with
    `orthographic_projection` for a directional light).  One `rasterise_batch` call over a zero background, with clip
    vertices (p, 1) @ light_matrix and vertex colours (1, clip z): occupancy is exactly 1 on covered texels and 0
    elsewhere, and depth is the interpolated clip z (0 where nothing is covered), exact for orthographic and perspective
    lights alike because clip z is affine in the light's view space.  Gradients reach `vertices` and `light_matrix`
    through the rasteriser's backward pass; the occupancy channel's carries the occluders' gradient (DESIGN.md §7.15).
    This is the map format `shadow_visibility` reads.  Needs CUDA, as `rasterise_batch` does."""
    from .rasterise_ops import rasterise_batch
    vertices = torch.as_tensor(vertices, dtype=torch.float32)
    dev = vertices.device
    light_matrix = torch.as_tensor(light_matrix, dtype=torch.float32, device=dev)
    faces = torch.as_tensor(faces, device=dev)
    lead, V, F = vertices.shape[:-2], vertices.shape[-2], faces.shape[-2]
    B = math.prod(lead)
    p = vertices[..., :3]
    clip = torch.matmul(torch.cat([p, torch.ones_like(p[..., :1])], -1), light_matrix)   # [*, V, 4]
    colors = torch.stack([torch.ones_like(clip[..., 2]), clip[..., 2]], -1)
    faces = faces.expand(lead + (F, 3)) if faces.dim() == 2 else faces
    background = torch.zeros((B, height, width, 2), dtype=torch.float32, device=dev)
    out = rasterise_batch(background, clip.reshape(B, V, 4), colors.reshape(B, V, 2), faces.reshape(B, F, 3))
    return out.reshape(lead + (height, width, 2))


def _shadow_visibility(positions, light_matrix, shadow_map, radius=1, softness=0., bias=0.):
    """The torch restatement of `shadow_visibility`: its CPU implementation and its specification.  Keeps the dtype of
    its inputs (the tests evaluate it in float64).  Points that are not looked up take safe values inside the `where`s,
    so that their gradients are exactly 0 and not NaN."""
    p = positions
    SH, SW = shadow_map.shape[-3], shadow_map.shape[-2]
    ones = torch.ones_like(p[..., :1])
    with torch.no_grad():
        h0 = torch.matmul(torch.cat([p, ones], -1), light_matrix)
        ok = torch.isfinite(h0).all(-1) & (h0[..., 3] > 0)
    p = torch.where(ok[..., None], p, 0.)
    h = torch.matmul(torch.cat([p, ones], -1), light_matrix)
    h = torch.where(ok[..., None], h, torch.tensor([0., 0., 0., 1.], dtype=h.dtype, device=h.device))
    x, y, z, w = h.unbind(-1)
    X = (x / w + 1.) * (0.5 * SW)
    Yd = (1. - y / w) * (0.5 * SH)
    valid = ok & (X >= 0) & (X < SW) & (Yd >= 0) & (Yd < SH)
    u, v = torch.where(valid, X, 0.5) - 0.5, torch.where(valid, Yd, 0.5) - 0.5
    c0, r0 = u.detach().floor(), v.detach().floor()
    fc, fr = u - c0, v - r0
    flat = shadow_map.reshape(shadow_map.shape[:-3] + (SH * SW, 2))

    def texel(r, c):
        idx = (r * SW + c).long()
        if flat.dim() == 2:
            return flat[idx]
        return torch.gather(flat, -2, idx[..., None].expand(idx.shape + (2,)))

    def weight(i, f):
        return 1. - f if i == 0 else (f if i == 2 * radius + 1 else torch.ones_like(f))

    vis = torch.zeros_like(fc)
    for i in range(2 * radius + 2):
        r = (r0 - radius + i).clamp(0, SH - 1)
        for k in range(2 * radius + 2):
            t = texel(r, (c0 - radius + k).clamp(0, SW - 1))
            d = z - t[..., 1] - bias
            step = torch.sigmoid(d / softness) if softness > 0 else (d > 0).to(d.dtype)
            vis = vis + weight(i, fr) * weight(k, fc) * (1. - t[..., 0] * step)
    vis = vis / (2 * radius + 1) ** 2
    return torch.where(valid, vis, 1.)[..., None]


def shadow_route(position_shape, matrix_shape, map_shape, devices):
    """Whether a `shadow_visibility` call runs the CUDA kernels, decided from shapes and devices alone: positions
    [*, N, 3], and light_matrix [*, 4, 4] with shadow_map [*, SH, SW, 2] (one per item) or [4, 4] with [SH, SW, 2]
    (shared), all on one CUDA device.  Returns a Route (C = 1, the output's width; per_item = (matrix, map)) or None."""
    map_shape = tuple(map_shape)
    if len(map_shape) < 3 or map_shape[-1] != 2:
        return None
    route = cuda_route([position_shape], [(matrix_shape, (4, 4)), (map_shape, map_shape[-3:])], devices, [3])
    if route is None or route.per_item[0] != route.per_item[1]:
        return None
    return route._replace(C=1)


def _shadow_inputs(radius, softness, bias, route, positions, light_matrix, shadow_map):
    """The input arguments of dirt_shadow_forward / _backward, in their order."""
    return [_ptr(positions), _point_stride(positions), _ptr(light_matrix), _ptr(shadow_map), int(route.per_item[0]),
            shadow_map.shape[-3], shadow_map.shape[-2], radius, softness, bias]


def _restate_shadow(radius, softness, bias, route, positions, light_matrix, shadow_map):
    """The restatement on the op's own inputs (flattened per-point rows, per-item matrix and map)."""
    return _shadow_visibility(_unflat_points(positions, route), _unflat_item(light_matrix, route, route.per_item[0]),
                              _unflat_item(shadow_map, route, route.per_item[1]), radius, softness, bias)


def _shadow_scratch_bytes(lib, route, want, positions, light_matrix, shadow_map):
    """The deterministic backward's scratch: needed only for the map gradient."""
    if not want[2]:
        return 0
    return lib.dirt_shadow_backward_deterministic_bytes(route.B, route.V, int(route.per_item[0]), shadow_map.shape[-3],
                                                        shadow_map.shape[-2])


_SHADOW = _PointOp('ShadowVisibility', 'dirt_shadow_forward', 'dirt_shadow_backward', _shadow_inputs,
                   lambda route: (route.B, route.V), _restate_shadow, first_param=1,
                   workspace_bytes='dirt_shadow_workspace_bytes',
                   deterministic=('dirt_shadow_backward_deterministic', _shadow_scratch_bytes))


def shadow_visibility(positions, light_matrix, shadow_map, radius=1, softness=0., bias=0., name=None):
    """The fraction of a light that reaches each point past the occluders of a shadow map, by percentage-closer
    filtering.

    positions [*, N, 3] world points; light_matrix [*, 4, 4] with shadow_map [*, SH, SW, 2] (one per item), or [4, 4]
    with [SH, SW, 2] (shared): the matrix and the `shadow_map` output it was rendered with -> visibility [*, N, 1] in
    [0, 1].  With (x, y, z, w) = (p, 1) @ light_matrix, the point falls at X = (x/w + 1) SW/2, Yd = (1 - y/w) SH/2 (the
    texel the rasteriser covers there); the (2R+2)^2 texels around it, clamped into the map, each give
    s = 1 - occupancy * step((z - depth - bias) / softness), and V is their box-of-bilinear average with 1-D weights
    (1 - f, 1, ..., 1, f) / (2R+1) (radius R = 0: bilinear).  step is the logistic sigmoid for softness > 0 and the
    Heaviside step (step(0) = 0) for softness = 0.  A point behind the light (w <= 0), with a non-finite coordinate or
    outside the map is lit: V = 1, with no gradient.  Gradients reach the positions, the light matrix and both channels
    of the map (none through the step for softness = 0; the occupancy gradient is what carries the occluders'
    gradient); softness and bias are plain floats without gradient.

    radius in 0..3, softness >= 0, bias >= 0.  On CUDA in the shapes `shadow_route` accepts fused kernels compute it,
    reading G-buffer channel slices in place, with a bit-reproducible light-matrix gradient.  The map gradient is summed
    with float atomics, or, under torch.use_deterministic_algorithms(True), by a sort of the points by texel and
    fixed-order float64 sums, bit-reproducible.  Any other call runs the torch restatement `_shadow_visibility`
    (DESIGN.md §7.15)."""
    radius, softness, bias = int(radius), float(softness), float(bias)
    if not 0 <= radius <= SHADOW_MAX_RADIUS:
        raise ValueError('shadow_visibility: radius must be in 0..%d, got %d' % (SHADOW_MAX_RADIUS, radius))
    if not (softness >= 0 and bias >= 0 and math.isfinite(softness) and math.isfinite(bias)):
        raise ValueError('shadow_visibility: softness and bias must be finite and >= 0')
    positions = torch.as_tensor(positions, dtype=torch.float32)
    dev = positions.device
    light_matrix = torch.as_tensor(light_matrix, dtype=torch.float32, device=dev)
    shadow_map = torch.as_tensor(shadow_map, dtype=torch.float32, device=dev)
    route = shadow_route(positions.shape, light_matrix.shape, shadow_map.shape,
                         [t.device for t in (positions, light_matrix, shadow_map)])
    if route is None:
        return _shadow_visibility(positions, light_matrix, shadow_map, radius, softness, bias)
    flat_map = _flat_item(shadow_map, route, route.per_item[1])
    if flat_map.data_ptr() % 8:
        flat_map = flat_map.clone()   # the kernels read float2 texels
    return _PointFunction.apply(_SHADOW, (radius, softness, bias), route, _rows(positions, 3),
                                _flat_item(light_matrix, route, route.per_item[0]), flat_map)
