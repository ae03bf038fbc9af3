"""`rasterise` / `rasterise_batch` and their deferred-shading variants on the H100-native library.

Host-side mirror of the reference's dirt/rasterise_ops.py: same function names, argument order,
defaults and error behaviour, with `torch.Tensor` in place of `tf.Tensor` and a
`torch.autograd.Function` in place of `@ops.RegisterGradient('Rasterise')` (rasterise_ops.py:111-129).

Differences that a caller can observe:
* any channel count is rendered in ONE fused pass; the reference's greedy 3/1 channel grouping
  (rasterise_ops.py:86-108) only survives as the `channel_groups` argument of the backward kernel,
  where it changes the result (each group takes its own filter / dilation decision);
* tensors must live on a CUDA device (the reference registers a GPU kernel only,
  csrc/rasterise_egl.cpp:410); there is no CPU fallback.
"""
import ctypes
import operator

import torch

from . import _lib


def default_channel_groups(channels):
    """The reference's split of `channels` into op calls: one group if channels is 1 or 3, else greedily
    groups of 3 while at least 3 remain, then groups of 1 (dirt/rasterise_ops.py:80-108).  The library makes the same
    split (make_groups, csrc/api.cu) for a backward call given no groups, as the autograd nodes here are."""
    if channels <= 0:
        raise ValueError('channels must be positive')
    if channels == 1 or channels == 3:
        return [channels]
    groups, begin = [], 0
    while begin < channels:
        width = 3 if begin + 3 <= channels else 1
        groups.append(width)
        begin += width
    return groups


def _stream_ptr(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _workspace(B, H, W, C, V, F, device, face_id_scratch=False):
    """A workspace for one call -> (tensor, its size).  Without `face_id_scratch` it is the smaller size that serves every
    call whose caller holds the face ids (dirt_workspace_bytes_min: no B*H*W*4-byte block for deriving them), which is every
    call this module makes except a backward call without `face_ids`."""
    size = _lib.lib().dirt_workspace_bytes if face_id_scratch else _lib.lib().dirt_workspace_bytes_min
    # the allocation also covers a 3-channel call on the same geometry (its workspace carries padded gradient rows behind
    # the blocks that are laid out independently of C): deferred shading hands the G-buffer pass's workspace to the backward
    # call on the shaded, usually 3-channel, image
    alloc = max(int(size(B, H, W, C, V, F)), int(size(B, H, W, 3, V, F)), 256)
    return torch.empty(alloc, dtype=torch.uint8, device=device), alloc


def _require_cuda(*tensors):
    for t in tensors:
        if not t.is_cuda:
            raise RuntimeError(
                'dirt_b200: rasterise needs CUDA tensors (the Rasterise op has no CPU kernel); got a tensor on %s'
                % t.device)


def _check_shapes(op, background, vertices, vertex_colors, faces, height, width, channels):
    # same conditions and wording as csrc/rasterise_egl.cpp:301-316
    if background.dim() != 4 or background.shape[1] != height or background.shape[2] != width or \
            background.shape[3] != channels:
        raise ValueError('%s expects background_tensor to be 4D, and bgcolor.shape == [None, height, width, channels]' % op)
    if vertices.dim() != 3 or vertices.shape[2] != 4:
        raise ValueError('%s expects vertices to be 3D, and vertices.shape[2] == 4' % op)
    if vertex_colors.dim() != 3 or vertex_colors.shape[1] != vertices.shape[1] or vertex_colors.shape[2] != channels:
        raise ValueError('%s expects vertex_colors to be 3D, and vertex_colors.shape == [None, vertices.shape[1], channels]' % op)
    if faces.dim() != 3 or faces.shape[2] != 3:
        raise ValueError('%s expects faces to be 3D, and faces.shape[2] == 3' % op)
    B = vertices.shape[0]
    if background.shape[0] != B or vertex_colors.shape[0] != B or faces.shape[0] != B:
        raise ValueError('%s expects all arguments to have same leading (batch) dimension' % op)


def rasterise_forward_raw(background, vertices, vertex_colors, faces, want_face_ids=True, return_workspace=False):
    """One call of dirt_rasterise_forward on contiguous CUDA tensors. Returns (pixels, face_ids or None)
    [, workspace tensor holding the per-face setup records, reusable by rasterise_backward_raw]."""
    B, H, W, C = background.shape
    V, F = vertices.shape[1], faces.shape[1]
    pixels = torch.empty_like(background)
    face_ids = torch.empty((B, H, W), dtype=torch.int32, device=background.device) if want_face_ids else None
    ws, nbytes = _workspace(B, H, W, C, V, F, background.device)
    with torch.cuda.device(background.device):
        rc = _lib.lib().dirt_rasterise_forward(_ptr(background), _ptr(vertices), _ptr(vertex_colors), _ptr(faces),
                                               _ptr(pixels), _ptr(face_ids), B, H, W, C, V, F, _ptr(ws), nbytes,
                                               _stream_ptr(background.device))
    _lib.check(rc, 'Rasterise')
    if return_workspace:
        ws._dirt_setup_of = _geometry_identity(vertices, faces, H, W)
        return pixels, face_ids, ws
    return pixels, face_ids


def _geometry_identity(vertices, faces, H, W):
    """What the setup records in a workspace were computed from: the tensors' storage AND their version counters
    (an in-place update of the vertices makes the records stale; the C ABI's own tag cannot see that)."""
    return (vertices.data_ptr(), vertices._version, tuple(vertices.shape), faces.data_ptr(), faces._version, tuple(faces.shape), H, W)


def _holds_setup(workspace, vertices, faces, B, H, W, C, V, F):
    """Whether the setup records in `workspace` (a forward call's, or None) can be reused by a call on these tensors: it
    is big enough for the call and still describes exactly these tensors (storage, version counters, sizes)."""
    return (workspace is not None and workspace.numel() >= int(_lib.lib().dirt_workspace_bytes_min(B, H, W, C, V, F)) and
            getattr(workspace, '_dirt_setup_of', None) == _geometry_identity(vertices, faces, H, W))


def rasterise_backward_raw(vertices, faces, pixels, grad_pixels, face_ids=None, channel_groups=None, setup_workspace=None,
                           shared_geometry=False, want_position=True, want_colour=True, deterministic=None):
    """One call of dirt_rasterise_backward (the RasteriseGrad op, csrc/rasterise_grad_egl.cpp:33-53).
    `setup_workspace`: the workspace tensor of the forward call on the same (vertices, faces); its setup records are
    reused only if it still describes exactly these tensors (storage, version counters, sizes), otherwise they are
    recomputed.  `shared_geometry`: accumulate the vertex gradients over the batch (DIRT_BWD_SHARED_GEOMETRY):
    grad_vertices [V,4] and grad_vertex_colors [V,C] instead of [B,V,.].  want_position / want_colour = False skip
    the position terms (grad_vertices comes back zero) / the colour terms (grad_vertex_colors zero, grad_background None).
    `pixels` and `grad_pixels` are made contiguous float32 here.
    `deterministic`: run dirt_rasterise_backward_deterministic, whose outputs are bit-reproducible (float64 sums in a
    fixed order, no float atomics); None follows torch.are_deterministic_algorithms_enabled().  Its scratch is allocated
    per call.
    Returns (grad_background, grad_vertices, grad_vertex_colors)."""
    B, H, W, C = pixels.shape
    V, F = vertices.shape[1], faces.shape[1]
    # wording of csrc/rasterise_grad_egl.cpp:349-377
    if vertices.dim() != 3 or vertices.shape[2] != 4:
        raise ValueError('RasteriseGrad expects vertices to be 3D, and vertices.shape[2] == 4')
    if faces.dim() != 3 or faces.shape[2] != 3:
        raise ValueError('RasteriseGrad expects faces to be 3D, and faces.shape[2] == 3')
    if grad_pixels.shape != pixels.shape:
        raise ValueError('RasteriseGrad expects grad_pixels to be 4D, and grad_pixels.shape == [None, height, width, channels]')
    if faces.shape[0] != B or vertices.shape[0] != B:
        raise ValueError('RasteriseGrad expects all arguments to have same leading (batch) dimension')
    pixels, grad_pixels = pixels.contiguous().to(torch.float32), grad_pixels.contiguous().to(torch.float32)
    device = pixels.device
    grad_background = torch.empty_like(pixels) if want_colour else None
    lead = () if shared_geometry else (B,)
    grad_vertices = torch.empty(lead + (V, 4), dtype=torch.float32, device=device)
    grad_vertex_colors = torch.empty(lead + (V, C), dtype=torch.float32, device=device)
    if channel_groups is None:
        groups_ptr, n_groups = None, 0
    else:
        groups_arr = (ctypes.c_int * len(channel_groups))(*[int(g) for g in channel_groups])
        groups_ptr, n_groups = groups_arr, len(channel_groups)
    reuse = int(face_ids is not None and _holds_setup(setup_workspace, vertices, faces, B, H, W, C, V, F))
    ws = setup_workspace if reuse else _workspace(B, H, W, C, V, F, device, face_id_scratch=face_ids is None)[0]
    nbytes = int(ws.numel())
    flags = ((_lib.BWD_SHARED_GEOMETRY if shared_geometry else 0) | (0 if want_position else _lib.BWD_SKIP_POSITION) |
             (0 if want_colour else _lib.BWD_SKIP_COLOUR))
    if deterministic is None:
        deterministic = torch.are_deterministic_algorithms_enabled()
    with torch.cuda.device(device):
        if deterministic:
            scratch_bytes = max(int(_lib.lib().dirt_rasterise_backward_deterministic_bytes(B, H, W, C, V, F)), 256)
            scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=device)
            rc = _lib.lib().dirt_rasterise_backward_deterministic(
                _ptr(vertices), _ptr(faces), _ptr(pixels), _ptr(grad_pixels), _ptr(face_ids),
                _ptr(grad_background), _ptr(grad_vertices), _ptr(grad_vertex_colors),
                B, H, W, C, V, F, groups_ptr, n_groups, reuse, flags, _ptr(ws), nbytes, _ptr(scratch), scratch_bytes,
                _stream_ptr(device))
        else:
            rc = _lib.lib().dirt_rasterise_backward_ex(
                _ptr(vertices), _ptr(faces), _ptr(pixels), _ptr(grad_pixels), _ptr(face_ids),
                _ptr(grad_background), _ptr(grad_vertices), _ptr(grad_vertex_colors),
                B, H, W, C, V, F, groups_ptr, n_groups, reuse, flags, _ptr(ws), nbytes, _stream_ptr(device))
    _lib.check(rc, 'RasteriseGrad')
    return grad_background, grad_vertices, grad_vertex_colors


def rasterise_derivatives_raw(vertices, faces, attributes, face_ids, first_channel, channel_count, setup_workspace=None):
    """One call of dirt_rasterise_derivatives on contiguous CUDA tensors: the screen-space derivatives of attribute channels
    [first_channel, first_channel + channel_count) at the pixels `face_ids` [B,H,W] shows, [B, H, W, 2, channel_count]
    (index 0 of the `2` axis d/dx along W, index 1 d/dy down the rows; 0 on the background; DESIGN.md §7.7).
    `setup_workspace`: the workspace of the forward call that produced `face_ids`, reused under the rule of
    rasterise_backward_raw.  The result has no gradient."""
    B, H, W = face_ids.shape
    V, F, C = vertices.shape[1], faces.shape[1], attributes.shape[2]
    device = face_ids.device
    reuse = int(_holds_setup(setup_workspace, vertices, faces, B, H, W, C, V, F))
    ws = setup_workspace if reuse else _workspace(B, H, W, C, V, F, device)[0]
    out = torch.empty((B, H, W, 2, channel_count), dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        rc = _lib.lib().dirt_rasterise_derivatives(_ptr(vertices), _ptr(faces), _ptr(attributes), _ptr(face_ids), _ptr(out),
                                                   B, H, W, C, V, F, first_channel, channel_count, reuse, _ptr(ws),
                                                   int(ws.numel()), _stream_ptr(device))
    _lib.check(rc, 'RasteriseDerivatives')
    return out


def workspace_status(workspace, B, H, W, C, V, F):
    """dirt_workspace_status: waits for the stream; raises if a backward call was handed a workspace that did not hold
    the setup records it was promised (csrc/api.cu)."""
    nbytes = int(workspace.numel())
    with torch.cuda.device(workspace.device):
        rc = _lib.lib().dirt_workspace_status(_ptr(workspace), nbytes, B, H, W, C, V, F, _stream_ptr(workspace.device))
    _lib.check(rc, 'RasteriseGrad')


def rasterise_visibility_raw(vertices, faces, height, width, want_gbuffer=True):
    """dirt_rasterise_visibility: (face_ids int32 [B,H,W], gbuffer float32 [B,H,W,4] or None)."""
    B, V, F = vertices.shape[0], vertices.shape[1], faces.shape[1]
    device = vertices.device
    face_ids = torch.empty((B, height, width), dtype=torch.int32, device=device)
    gbuffer = torch.empty((B, height, width, 4), dtype=torch.float32, device=device) if want_gbuffer else None
    ws, nbytes = _workspace(B, height, width, 1, V, F, device)
    with torch.cuda.device(device):
        rc = _lib.lib().dirt_rasterise_visibility(_ptr(vertices), _ptr(faces), _ptr(face_ids), _ptr(gbuffer), B, height,
                                                  width, V, F, _ptr(ws), nbytes, _stream_ptr(device))
    _lib.check(rc, 'RasteriseVisibility')
    return face_ids, gbuffer


class _Rasterise(torch.autograd.Function):
    """The Rasterise op with its registered gradient (dirt/rasterise_ops.py:111-129)."""

    @staticmethod
    def forward(ctx, background, vertices, vertex_colors, faces):
        pixels, face_ids, ws = rasterise_forward_raw(background, vertices, vertex_colors, faces, want_face_ids=True,
                                                     return_workspace=True)
        ctx.save_for_backward(vertices, faces, pixels, face_ids)
        ctx.setup_workspace = ws   # per-face setup records of this (vertices, faces): backward reuses them
        ctx.mark_non_differentiable(face_ids)
        return pixels, face_ids

    @staticmethod
    def backward(ctx, grad_pixels, _grad_face_ids):
        want_background, want_vertices, want_colours = ctx.needs_input_grad[:3]
        if not (want_background or want_vertices or want_colours):
            return None, None, None, None
        vertices, faces, pixels, face_ids = ctx.saved_tensors
        # channel_groups=None: the library's own split of the channels, the reference's greedy 3/1 grouping
        grad_background, grad_vertices, grad_vertex_colors = rasterise_backward_raw(
            vertices, faces, pixels, grad_pixels, face_ids, None, ctx.setup_workspace,
            want_position=want_vertices, want_colour=want_background or want_colours)
        return (grad_background if want_background else None, grad_vertices if want_vertices else None,
                grad_vertex_colors if want_colours else None, None)  # None: wrt faces


def _as(x, dtype, device=None):
    t = torch.as_tensor(x, dtype=dtype) if not isinstance(x, torch.Tensor) else x.to(dtype)
    if device is not None and t.device != device:
        t = t.to(device)
    return t


def _pick_device(*xs):
    # the device of the first CUDA tensor; host inputs (lists, numpy, CPU tensors) go to the current CUDA device,
    # as TensorFlow would place the GPU-only op there.  None (-> an error downstream) when there is no GPU.
    for x in xs:
        if isinstance(x, torch.Tensor) and x.is_cuda:
            return x.device
    if torch.cuda.is_available():
        return torch.device('cuda', torch.cuda.current_device())
    return None


def _inputs(background, vertices, vertex_colors, faces, single, check):
    """The four inputs of one rasterise call as contiguous float32 tensors (faces int32) on one CUDA device, with a leading
    batch axis added when `single`.  Once the background is known to be 4-D, `check(background, vertices, vertex_colors,
    faces)` makes the caller's shape checks; its result is returned after the four tensors.  The inputs must be on a CUDA
    device only after that, so a malformed call raises its shape error on a machine without a GPU too."""
    device = _pick_device(background, vertices, vertex_colors, faces)
    inputs = [_as(x, torch.float32, device) for x in (background, vertices, vertex_colors)] + [_as(faces, torch.int32, device)]
    if single:
        inputs = [t[None] for t in inputs]
    if inputs[0].dim() != 4:
        raise ValueError('Rasterise expects background_tensor to be 4D, and bgcolor.shape == [None, height, width, channels]')
    checked = check(*inputs)
    _require_cuda(*inputs)
    return [t.contiguous() for t in inputs] + [checked]


def _rasterise(background, vertices, vertex_colors, faces, height, width, channels, single):
    def check(background, vertices, vertex_colors, faces):
        h = int(background.shape[1]) if height is None else height
        w = int(background.shape[2]) if width is None else width
        c = int(background.shape[3]) if channels is None else channels
        if not (c > 0):
            raise ValueError('channels must be positive')  # `assert channels > 0`, rasterise_ops.py:87
        if not (w > 0 and h > 0):
            raise ValueError('width and height must be positive')  # csrc/hwc.h:28
        _check_shapes('Rasterise', background, vertices, vertex_colors, faces, h, w, c)

    background, vertices, vertex_colors, faces, _ = _inputs(background, vertices, vertex_colors, faces, single, check)
    pixels, _ = _Rasterise.apply(background, vertices, vertex_colors, faces)
    return pixels[0] if single else pixels


def rasterise(background, vertices, vertex_colors, faces, height=None, width=None, channels=None, name=None):
    """Rasterises the given `vertices` and `faces` over `background` (dirt/rasterise_ops.py:13-48).

    Args:
        background: float32 tensor [height, width, channels], the image to render over
        vertices: float32 tensor [vertex count, 4] of clip-space vertex positions
        vertex_colors: float32 tensor [vertex count, channels]; interpolated perspective-correctly
        faces: int32 tensor [face count, 3] of vertex indices
        height, width, channels: optional ints; default to the shape of `background`
        name: accepted for signature compatibility, ignored

    Returns:
        float32 tensor [height, width, channels]
    """
    return _rasterise(background, vertices, vertex_colors, faces, height, width, channels, single=True)


def rasterise_batch(background, vertices, vertex_colors, faces, height=None, width=None, channels=None, name=None):
    """Rasterises a batch of meshes with the same numbers of vertices and faces (dirt/rasterise_ops.py:51-108).

    As `rasterise`, with a leading batch dimension on every argument.
    """
    return _rasterise(background, vertices, vertex_colors, faces, height, width, channels, single=False)


class _SetupHolder(object):
    """Carries the forward call's workspace (per-face setup records, tile coverage flags) from the G-buffer node to the
    vertex-gradient node of one deferred call without making it an autograd input."""

    def __init__(self, workspace):
        self.workspace = workspace


class _RasteriseAttributes(torch.autograd.Function):
    """G-buffer pass of deferred shading: gradients flow to attributes and background only
    (the second RasteriseGrad call of dirt/rasterise_ops.py:233-237)."""

    @staticmethod
    def forward(ctx, background, vertices, attributes, faces, holder):
        gbuffer, face_ids, ws = rasterise_forward_raw(background, vertices, attributes, faces, want_face_ids=True,
                                                      return_workspace=True)
        holder.workspace = ws
        ctx.holder = holder
        ctx.save_for_backward(vertices, faces, gbuffer, face_ids)
        ctx.mark_non_differentiable(face_ids)
        return gbuffer, face_ids

    @staticmethod
    def backward(ctx, d_loss_by_gbuffer, _unused):
        if not (ctx.needs_input_grad[0] or ctx.needs_input_grad[2]):
            return None, None, None, None, None
        vertices, faces, gbuffer, face_ids = ctx.saved_tensors
        # the vertex gradient of THIS call (filtering the G-buffer) is the one the reference discards (:233-237)
        grad_background, _, grad_attributes = rasterise_backward_raw(vertices, faces, gbuffer, d_loss_by_gbuffer, face_ids,
                                                                     None, ctx.holder.workspace, want_position=False)
        return grad_background, None, grad_attributes, None, None


class _InjectVertexGradient(torch.autograd.Function):
    """Identity on the shaded pixels whose backward adds the vertex gradient obtained by filtering the
    SHADED image (the first RasteriseGrad call of dirt/rasterise_ops.py:206-210)."""

    @staticmethod
    def forward(ctx, pixels, vertices, faces, face_ids, holder):
        ctx.holder = holder
        ctx.save_for_backward(pixels.detach(), vertices, faces, face_ids)
        return pixels.view_as(pixels)

    @staticmethod
    def backward(ctx, d_loss_by_pixels):
        if not ctx.needs_input_grad[1]:
            return d_loss_by_pixels, None, None, None, None
        pixels, vertices, faces, face_ids = ctx.saved_tensors
        _, d_loss_by_vertices, _ = rasterise_backward_raw(vertices, faces, pixels, d_loss_by_pixels, face_ids, None,
                                                          ctx.holder.workspace, want_colour=False)
        return d_loss_by_pixels, d_loss_by_vertices, None, None, None


def _channel_run(derivative_channels, channels):
    """(first, count) of `derivative_channels`, which must be one ascending contiguous run of channel indices in
    [0, channels), such as range(1, 3)."""
    try:
        run = [operator.index(c) for c in derivative_channels]
    except TypeError:
        run = None
    if not run or run != list(range(run[0], run[0] + len(run))) or run[0] < 0 or run[-1] >= channels:
        raise ValueError('derivative_channels must be one ascending run of consecutive attribute channels in [0, %d), '
                         'such as range(1, 3); got %r' % (channels, derivative_channels))
    return run[0], len(run)


def _rasterise_deferred_internal(background, vertices, attributes, faces, shader_fn, shader_additional_inputs, single,
                                 derivative_channels=None):
    # dirt/rasterise_ops.py:180-257.  The reference wraps everything in one tf.custom_gradient; here the same
    # three gradient paths are expressed as two autograd nodes around an ordinary call of shader_fn, so tensors
    # and parameters that shader_fn uses receive their gradients from plain autograd.
    def check(background, vertices, attributes, faces):
        _check_shapes('Rasterise', background, vertices, attributes, faces, int(background.shape[1]),
                      int(background.shape[2]), int(background.shape[3]))
        if derivative_channels is not None:
            return _channel_run(derivative_channels, int(attributes.shape[2]))

    background, vertices, attributes, faces, run = _inputs(background, vertices, attributes, faces, single, check)
    holder = _SetupHolder(None)
    gbuffer, face_ids = _RasteriseAttributes.apply(background, vertices, attributes, faces, holder)
    extra = {}
    if run is not None:
        with torch.no_grad():
            derivatives = rasterise_derivatives_raw(vertices, faces, attributes, face_ids, *run, holder.workspace)
        extra['gbuffer_derivatives'] = derivatives[0] if single else derivatives
    if single:
        pixels = shader_fn(gbuffer[0], *shader_additional_inputs, **extra)[None]
    else:
        pixels = shader_fn(gbuffer, *shader_additional_inputs, **extra)
    if pixels.dim() != 4 or pixels.shape[:3] != gbuffer.shape[:3]:
        raise ValueError('shader_fn must return pixels of shape [height, width, channels] per image')
    pixels = _InjectVertexGradient.apply(pixels.to(torch.float32), vertices, faces, face_ids, holder)
    return pixels[0] if single else pixels


def rasterise_deferred(background_attributes, vertices, vertex_attributes, faces, shader_fn, shader_additional_inputs=[], name=None,
                       derivative_channels=None):
    """Rasterises a G-buffer of vertex attributes and shades it with `shader_fn` (dirt/rasterise_ops.py:260-310).

    Equivalent to `shader_fn(rasterise(background_attributes, vertices, vertex_attributes, faces), *shader_additional_inputs)`
    in the forward direction; the gradient w.r.t. `vertices` is computed from the SHADED pixels, the gradients
    w.r.t. attributes / background from the G-buffer through `shader_fn`.

    `derivative_channels`: optional, one ascending run of consecutive attribute channels, such as range(1, 3).  Then
    `shader_fn` is called as `shader_fn(gbuffer, *shader_additional_inputs, gbuffer_derivatives=d)`, with d float32
    [H, W, 2, K] (K channels) the screen-space derivatives of those G-buffer channels at each pixel centre: d[..., 0, k]
    along x (the columns, to the right), d[..., 1, k] along y (the rows, downwards), in attribute units per pixel,
    exactly those of the perspective-correct interpolant of the face the pixel shows (no neighbour differences, so no
    error at silhouettes or uv seams); 0 on the background.  They carry no gradient (DESIGN.md §7.7).  For uv
    channels u, u + 1 read with `uvs_to_pixel_indices(..., mode='repeat')` from a TH x TW texture, the derivatives
    `sample_texture(..., mode='trilinear')` takes are
        (d[..., :, u:u+2].flip(-1) * torch.tensor([TH, TW], device=d.device)).flatten(-2)
    = (d row / dx, d col / dx, d row / dy, d col / dy).  Without it nothing else is computed or passed.
    """
    return _rasterise_deferred_internal(background_attributes, vertices, vertex_attributes, faces, shader_fn,
                                        list(shader_additional_inputs), True, derivative_channels)


def rasterise_batch_deferred(background_attributes, vertices, vertex_attributes, faces, shader_fn, shader_additional_inputs=[], name=None,
                             derivative_channels=None):
    """Batched `rasterise_deferred` (dirt/rasterise_ops.py:313-333).  With `derivative_channels`, `gbuffer_derivatives`
    is [B, H, W, 2, K]."""
    return _rasterise_deferred_internal(background_attributes, vertices, vertex_attributes, faces, shader_fn,
                                        list(shader_additional_inputs), False, derivative_channels)
