"""GPU: screen-space derivatives of G-buffer attributes (dirt_rasterise_derivatives, `derivative_channels` of the deferred
entry points; DESIGN.md §7.7).

On covered pixels the kernel is held with conftest.rel_close (1e-4) to the float64 evaluation of its formula on its own
fp32 planes, always, and to the float64 specification `fp64_derivatives` of tests/test_gbuffer_derivatives_host.py
(checked there against central differences) where the fp32 planes allow it: clip w spreads 1 and 10^2.  Spreads of
10^4 and 10^6 and faces behind the eye are logged (DESIGN.md §7.7).  Background pixels must be exactly +0.  The worst
ratios go into the end-of-run summary under names starting with 'derivatives:'.  Also:
affine faces, bit-identical outputs and gradients of the deferred path with and without the derivatives, repeats,
CUDA graph replay, item independence, a batch past the grid's 65535 images, the stale-workspace report, and the
textured cube with a trilinear lookup fed by the analytic derivatives."""
import numpy as np
import pytest
import torch

import kernel_paths as kp
from conftest import rel_close
from test_gbuffer_derivatives_host import fp64_derivatives
from test_gpu_paths import _cuda, _offset, _p, _stream, abi_forward

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)


@pytest.fixture(autouse=True)
def _needs_the_library(cuda_lib):
    return cuda_lib


def abi_derivatives(L, vertices, faces, attributes, face_ids, first, count, workspace=None, holds_setup=True, out=None):
    """dirt_rasterise_derivatives of library `L` -> [B, H, W, 2, count]; `workspace` with holds_setup is the forward's."""
    B, H, W = face_ids.shape
    V, F, C = vertices.shape[1], faces.shape[1], attributes.shape[2]
    if workspace is None:
        workspace = torch.empty(int(L.dirt_workspace_bytes_min(B, H, W, C, V, F)), dtype=torch.uint8, device=DEV)
        holds_setup = False
    if out is None:
        out = torch.full((B, H, W, 2, count), float('nan'), device=DEV)
    rc = L.dirt_rasterise_derivatives(_p(vertices), _p(faces), _p(attributes), _p(face_ids), _p(out), B, H, W, C, V, F,
                                      first, count, int(holds_setup), _p(workspace), workspace.numel(), _stream())
    assert rc == 0, L.dirt_error_string(rc)
    return out


def _render(L, s):
    """Forward call of scene `s` (its vertex colours are the attributes) -> (CUDA tensors, face ids, workspace)."""
    t = _cuda(s)
    B, H, W, C = s['background'].shape
    pixels = torch.empty_like(t['background'])
    ids = torch.empty((B, H, W), dtype=torch.int32, device=DEV)
    ws = abi_forward(L, t['background'], t['vertices'], t['vertex_colors'], t['faces'], pixels, ids)
    return t, ids, ws


# channel ranges (C, first, count) that take every instantiation: one channel (float2 store), two and four with and
# without vector attribute loads, and the scalar loop (three, five)
RANGES = [(8, 0, 4), (8, 4, 4), (8, 2, 2), (8, 1, 1), (5, 0, 1), (5, 1, 2), (5, 1, 4), (5, 0, 3), (5, 0, 5)]


def _from_the_planes(ws, gbuffer, ids, attributes, faces):
    """float64 [B, H, W, 2, C]: the formula of DESIGN.md §7.7 evaluated exactly on the G-buffer's own fp32 values
    (b0, b1, 1/S) and the fp32 plane coefficients of the face records in the forward call's workspace (the TriInterp
    block follows the TriCov block, 256-byte aligned; common.cuh carve_workspace).  What separates the kernel from this
    is its own fp32 arithmetic; what separates this from fp64 truth is the fp32 planes."""
    B, H, W = ids.shape
    F = faces.shape[1]
    off = -(-B * F * 64 // 256) * 256
    rec = ws[off:off + B * F * 64].view(torch.float32).reshape(B, F, 16).double().cpu().numpy()
    g, idn = gbuffer.double().cpu().numpy(), ids.cpu().numpy()
    out = np.zeros((B, H, W, 2, attributes.shape[-1]))
    for b in range(B):
        cov = idn[b] >= 0
        f = idn[b][cov]
        r, gb = rec[b][f], g[b][cov]
        a = attributes[b].astype(np.float64)[faces[b][f]]                        # [n, 3, C]
        d0, d1 = a[:, 0] - a[:, 2], a[:, 1] - a[:, 2]
        for axis, (q0, q1, sg) in enumerate(((0, 3, 6), (1, 4, 7))):              # (q0A, q1A, sA), (q0B, q1B, sB)
            db0 = (r[:, q0] - gb[:, 0] * r[:, sg]) * gb[:, 3]
            db1 = (r[:, q1] - gb[:, 1] * r[:, sg]) * gb[:, 3]
            out[b][cov, axis] = d0 * db0[:, None] + d1 * db1[:, None]
    return out


def _check_against_fp64(L, s, ranges, label, assert_fp64=True):
    """The kernel against _from_the_planes (always asserted) and against fp64 truth (asserted when `assert_fp64`,
    else logged: the fp32 planes' gap, DESIGN.md §7.7).  Returns the worst ratio to fp64 truth."""
    from dirt_b200 import rasterise_ops
    t, ids, ws = _render(L, s)
    B, H, W, C = s['background'].shape
    ids_v, gbuffer = rasterise_ops.rasterise_visibility_raw(t['vertices'], t['faces'], H, W)
    assert torch.equal(ids_v, ids)
    planes = _from_the_planes(ws, gbuffer, ids, s['vertex_colors'], s['faces'])
    got = {r: abi_derivatives(L, t['vertices'], t['faces'], t['vertex_colors'], ids, *r, ws).cpu().numpy() for r in ranges}
    ids_g = ids.cpu().numpy()
    worst = 0.0
    for b in range(B):
        cov = ids_g[b] >= 0
        assert cov.any()
        truth = fp64_derivatives(s['vertices'][b], s['vertex_colors'][b], s['faces'][b], ids_g[b])[cov]
        for first, count in ranges:
            mine = got[first, count][b]
            where = '%s: channels [%d, %d) of item %d' % (label, first, first + count, b)
            assert (mine[~cov] == 0).all() and not np.signbit(mine[~cov]).any(), where + ': background not +0'
            ok, ratio = rel_close(mine[cov], planes[b][cov][..., first:first + count], name='derivatives: vs its planes')
            assert ok, '%s off by %.2fx the tolerance from its own planes' % (where, ratio)
            name = 'derivatives: vs fp64' + ('' if assert_fp64 else ', %s (not asserted)' % label)
            ok, ratio = rel_close(mine[cov], truth[..., first:first + count], name=name)
            worst = max(worst, ratio)
            assert ok or not assert_fp64, '%s off by %.2fx the tolerance from fp64 truth' % (where, ratio)
    print('%s: worst ratio to fp64 truth %.3f' % (label, worst))
    return worst


# clip w spreads whose fp64 comparison is asserted; at 10^4 the fp32 planes themselves are past the bar (DESIGN.md §7.7)
FP64_ASSERTED = ('1', '1e2')


@pytest.mark.parametrize('size', kp.FP64_SIZES)
@pytest.mark.parametrize('ratio', sorted(kp.FP64_W))
def test_big_triangle_against_fp64_truth(cuda_lib, size, ratio):
    for C in (8, 5):
        s = kp.big_triangle(size, size, kp.FP64_W[ratio], C, seed=C)
        _check_against_fp64(cuda_lib, s, [(f, k) for c, f, k in RANGES if c == C],
                            'big triangle %d^2 w ratio %s C=%d' % (size, ratio, C), assert_fp64=ratio in FP64_ASSERTED)


def test_big_triangle_extreme_w_is_logged(cuda_lib):
    # a w ratio of 10^6 across one face, as for the forward pixels: measured, reported, not asserted
    for ratio, w in kp.FP64_W_LOGGED.items():
        _check_against_fp64(cuda_lib, kp.big_triangle(512, 512, w, 5), [(0, 5)], 'w ratio %s' % ratio, assert_fp64=False)


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_soup_behind_the_camera_against_fp64_truth(cuda_lib, seed):
    from dirt_b200 import scenes
    s = scenes.random_soup(batch=3, width=96, height=64, n_faces=60, channels=8, seed=seed, behind_camera=True)
    # faces with a vertex behind the eye: S crosses zero on screen and the planes keep pixel (0, 0) (DESIGN.md §2), so
    # their fp64 comparison is logged
    _check_against_fp64(cuda_lib, s, [(3, 4), (5, 2), (1, 1), (2, 5), (4, 4)], 'soup behind the camera seed %d' % seed,
                        assert_fp64=False)


def test_affine_faces_have_constant_derivatives_equal_to_the_closed_form(cuda_lib):
    s = kp.full_coverage_mesh(2, 48, 64, 3, cell=7.0, seed=4)
    v = s['vertices'].astype(np.float64)
    s['vertices'] = np.concatenate([v[..., :3] / v[..., 3:], np.ones_like(v[..., 3:])], -1).astype(np.float32)
    t, ids, ws = _render(cuda_lib, s)
    got = abi_derivatives(cuda_lib, t['vertices'], t['faces'], t['vertex_colors'], ids, 0, 3, ws).cpu().numpy()
    ids_g = ids.cpu().numpy()
    B, H, W = ids_g.shape
    faces_seen = 0
    for b in range(B):
        for f in np.unique(ids_g[b][ids_g[b] >= 0]):
            vf = s['vertices'][b][s['faces'][b][f]].astype(np.float64)
            p = np.stack([(vf[:, 0] + 1) * 0.5 * W, (1 - vf[:, 1]) * 0.5 * H], -1)   # pixel coordinates, y down
            a = s['vertex_colors'][b][s['faces'][b][f]].astype(np.float64)
            grad = np.linalg.solve(np.stack([p[1] - p[0], p[2] - p[0]]), np.stack([a[1] - a[0], a[2] - a[0]]))
            d = got[b][ids_g[b] == f]                                                     # [n, 2, 3]
            assert np.abs(d - d[:1]).max() <= 4e-7 * max(np.abs(d).max(), 1e-30), (b, f)  # a few ulps apart
            ok, ratio = rel_close(d, np.broadcast_to(grad, d.shape), name='derivatives: affine closed form')
            assert ok, (b, f, ratio)
            faces_seen += 1
    assert faces_seen > 100


def _deferred_run(s, derivative_channels):
    """rasterise_batch_deferred of scene `s` under torch.use_deterministic_algorithms(True) -> (pixels, G-buffer as the
    shader saw it, derivatives or None, gradients of background, vertices, attributes and the shader input)."""
    import dirt_b200 as dirt
    t = {k: torch.from_numpy(v).to(DEV) for k, v in s.items()}
    for k in ('background', 'vertices', 'vertex_colors'):
        t[k].requires_grad_(True)
    weight = torch.linspace(0.5, 1.5, s['background'].shape[-1], device=DEV).requires_grad_(True)
    seen = {}

    def shader(gbuffer, w, **kw):
        seen['gbuffer'] = gbuffer.detach().clone()
        seen['derivatives'] = kw.get('gbuffer_derivatives')
        return torch.sin(gbuffer * w)

    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        pixels = dirt.rasterise_batch_deferred(t['background'], t['vertices'], t['vertex_colors'], t['faces'], shader, [weight],
                                               derivative_channels=derivative_channels)
        gout = torch.from_numpy(np.random.default_rng(9).standard_normal(tuple(pixels.shape)).astype(np.float32)).to(DEV)
        (pixels * gout).sum().backward()
    finally:
        torch.use_deterministic_algorithms(before)
    grads = [t['background'].grad, t['vertices'].grad, t['vertex_colors'].grad, weight.grad]
    return pixels.detach(), seen['gbuffer'], seen['derivatives'], grads


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def test_deferred_outputs_and_gradients_do_not_change(cuda_lib):
    from dirt_b200 import scenes
    s = scenes.config3(batch=3, width=128, height=96, level=2, background='uniform')
    px0, gb0, d0, g0 = _deferred_run(s, None)
    px1, gb1, d1, g1 = _deferred_run(s, range(1, 4))
    assert d0 is None and d1.shape == (3, 96, 128, 2, 3)
    assert _bits_equal(px0, px1) and _bits_equal(gb0, gb1)
    for name, a, b in zip(['background', 'vertices', 'attributes', 'shader input'], g0, g1):
        assert a is not None and _bits_equal(a, b), name


def test_single_image_and_batch_entry_points_agree(cuda_lib):
    import dirt_b200 as dirt
    from dirt_b200 import scenes
    s = scenes.config3(batch=2, width=96, height=80, level=2)
    t = {k: torch.from_numpy(v).to(DEV) for k, v in s.items()}
    got = {}

    def shader(key):
        def fn(gbuffer, gbuffer_derivatives):
            got[key] = gbuffer_derivatives
            return gbuffer
        return fn

    dirt.rasterise_batch_deferred(t['background'], t['vertices'], t['vertex_colors'], t['faces'], shader('batch'),
                                  derivative_channels=[1, 2])
    for b in range(2):
        dirt.rasterise_deferred(t['background'][b], t['vertices'][b], t['vertex_colors'][b], t['faces'][b], shader(b),
                                derivative_channels=range(1, 3))
        assert got[b].shape == (80, 96, 2, 2) and not got[b].requires_grad
        assert _bits_equal(got[b], got['batch'][b])
    # the functional route: the same values as the C ABI on the forward call's own workspace
    rt, ids, ws = _render(cuda_lib, s)
    want = abi_derivatives(cuda_lib, rt['vertices'], rt['faces'], rt['vertex_colors'], ids, 1, 2, ws)
    assert _bits_equal(got['batch'], want)


def test_repeats_graph_replay_alignment_and_item_independence(cuda_lib):
    L = cuda_lib
    from dirt_b200 import scenes
    s = scenes.random_soup(batch=4, width=80, height=56, n_faces=50, channels=6, seed=5, behind_camera=True)
    t, ids, ws = _render(L, s)
    args = (t['vertices'], t['faces'], t['vertex_colors'], ids)
    for first, count in ((0, 1), (2, 2), (1, 4), (1, 3)):
        first_call = abi_derivatives(L, *args, first, count, ws)
        assert _bits_equal(first_call, abi_derivatives(L, *args, first, count, ws))
        assert _bits_equal(first_call, abi_derivatives(L, *args, first, count))          # records recomputed
        unaligned = _offset(torch.full_like(first_call, float('nan')))                  # the scalar path
        assert _bits_equal(first_call, abi_derivatives(L, *args, first, count, ws, out=unaligned))
        for b in range(4):
            alone = abi_derivatives(L, t['vertices'][b:b + 1], t['faces'][b:b + 1], t['vertex_colors'][b:b + 1],
                                    ids[b:b + 1], first, count)
            assert _bits_equal(alone[0], first_call[b]), (first, count, b)
    # CUDA graph replay
    out = torch.full((4, 56, 80, 2, 2), float('nan'), device=DEV)
    want = abi_derivatives(L, *args, 2, 2, ws)
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        abi_derivatives(L, *args, 2, 2, ws, out=out)
    torch.cuda.current_stream(DEV).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        abi_derivatives(L, *args, 2, 2, ws, out=out)
    for _ in range(2):
        out.fill_(float('nan'))
        graph.replay()
        torch.cuda.synchronize()
        assert _bits_equal(out, want)


def test_batch_past_the_grid_limit(cuda_lib):
    s = kp.grid_limit_scene()
    t, ids, ws = _render(cuda_lib, s)
    got = abi_derivatives(cuda_lib, t['vertices'], t['faces'], t['vertex_colors'], ids, 0, 4, ws)
    ids_g = ids.cpu().numpy()
    B = ids_g.shape[0]
    assert B == kp.GRID_LIMIT_BATCH
    picks = [0, 1, kp.GRID_Z_LIMIT - 1, kp.GRID_Z_LIMIT, B - 1]
    for b in picks:
        cov = ids_g[b] >= 0
        truth = fp64_derivatives(s['vertices'][b], s['vertex_colors'][b], s['faces'][b], ids_g[b])
        mine = got[b].cpu().numpy()
        assert (mine[~cov] == 0).all()
        if cov.any():
            ok, ratio = rel_close(mine[cov], truth[cov], name='derivatives: grid-limit batch vs fp64')
            assert ok, (b, ratio)
        alone = abi_derivatives(cuda_lib, t['vertices'][b:b + 1], t['faces'][b:b + 1], t['vertex_colors'][b:b + 1],
                                ids[b:b + 1], 0, 4)
        assert _bits_equal(alone[0], got[b]), b


def test_a_workspace_of_other_geometry_is_reported(cuda_lib):
    from dirt_b200 import _lib, rasterise_ops
    L = cuda_lib
    s = kp.two_faces_per_image(2, 32, 32, 3, seed=1)
    t, ids, ws = _render(L, s)
    other = t['vertices'].clone()    # same sizes, other storage: another tag
    out = abi_derivatives(L, other, t['faces'], t['vertex_colors'], ids, 0, 3, ws, holds_setup=True)
    B, H, W, C = s['background'].shape
    rc = L.dirt_workspace_status(_p(ws), ws.numel(), B, H, W, C, other.shape[1], t['faces'].shape[1], _stream())
    assert rc == _lib.ERR_STALE_WORKSPACE
    assert torch.isnan(out).all()
    with pytest.raises(RuntimeError, match='workspace_holds_setup'):
        rasterise_ops.workspace_status(ws, B, H, W, C, other.shape[1], t['faces'].shape[1])
    # the right geometry on a fresh forward workspace: no error
    t, ids, ws = _render(L, s)
    abi_derivatives(L, t['vertices'], t['faces'], t['vertex_colors'], ids, 0, 3, ws, holds_setup=True)
    assert L.dirt_workspace_status(_p(ws), ws.numel(), B, H, W, C, t['vertices'].shape[1], t['faces'].shape[1], _stream()) == 0


def _textured_cube_analytic(ex, texture_size=256):
    """tests/test_gpu_texture.py's textured cube, shaded with a trilinear lookup whose derivatives come from the
    G-buffer's uv channels through `derivative_channels`."""
    import dirt_b200 as dirt
    from dirt_b200 import lighting, matrices
    gen = lambda seed: torch.Generator(device=DEV).manual_seed(seed)
    vertices, uvs, faces = ex.build_cube()
    vertices_object = torch.tensor(vertices, dtype=torch.float32, device=DEV)
    uvs = torch.tensor(uvs, dtype=torch.float32, device=DEV)
    faces = torch.tensor(faces, dtype=torch.int32, device=DEV)
    texture = ex.checker_texture(size=texture_size, device=DEV)
    texture = (texture + 0.1 * torch.rand(texture.shape, generator=gen(26), device=DEV)).requires_grad_(True)
    light_direction = torch.tensor([1., 0., 0.], device=DEV, requires_grad=True)
    vertices_object = torch.cat([vertices_object, torch.ones_like(vertices_object[:, -1:])], dim=1).requires_grad_(True)
    vertices_world = vertices_object @ matrices.rodrigues([0., 0.6, 0.]).to(DEV)
    normals_world = lighting.vertex_normals(vertices_world, faces)
    view = matrices.compose(matrices.translation([0., -2., -3.2]), matrices.rodrigues([-0.5, 0., 0.])).to(DEV)
    proj = matrices.perspective_projection(near=0.1, far=20., right=0.1, aspect=120. / 160.).to(DEV)
    attributes = torch.cat([torch.ones_like(uvs[:, :1]), uvs, normals_world], dim=1)
    TH, TW = texture.shape[:2]

    def shader(gbuffer, texture, light_direction, gbuffer_derivatives):
        # channels 1, 2 are (u, v): the recipe of rasterise_deferred's docstring
        d = (gbuffer_derivatives.flip(-1) * torch.tensor([TH, TW], dtype=torch.float32, device=DEV)).flatten(-2)
        sample = lambda tex, idx: dirt.sample_texture(tex, idx, mode='trilinear', derivatives=d)
        return ex.shader_fn(gbuffer, texture, light_direction, sample=sample)

    pixels = dirt.rasterise_deferred(torch.zeros([120, 160, 6], device=DEV), vertices_world @ view @ proj, attributes, faces,
                                     shader, [texture, light_direction], derivative_channels=range(1, 3))
    weights = torch.rand(pixels.shape, generator=gen(27), device=DEV)
    (pixels * weights).sum().backward()
    return pixels.detach(), vertices_object.grad, texture.grad, light_direction.grad


def test_textured_cube_with_analytic_derivatives():
    import dirt_b200 as dirt
    from test_gpu_texture import _textured_cube
    from test_gpu_texture_mip import ex
    px_bi, *grads_bi = _textured_cube(ex, dirt.sample_texture, texture_size=256)
    px_tri, *grads_tri = _textured_cube_analytic(ex, texture_size=256)
    assert torch.isfinite(px_tri).all()
    for g in grads_tri:
        assert g is not None and torch.isfinite(g).all()
    touched_bi = int((grads_bi[1].abs().sum(-1) > 0).sum())
    touched_tri = int((grads_tri[1].abs().sum(-1) > 0).sum())
    assert touched_tri > touched_bi, (touched_tri, touched_bi)
