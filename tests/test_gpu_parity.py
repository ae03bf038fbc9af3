"""GPU: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.

Bar (BASELINE.json north_star / SURVEY 8c): face/pixel indexing bit-exact; float pixels and gradients
within 1e-4 relative (rel_close in conftest.py: |a-b| <= 1e-4 * max(|a|, |b|, 1e-2 * max|oracle|)).
"""
import os

import numpy as np
import pytest

from conftest import rel_close
from dirt_b200 import scenes

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')


def _cuda(s):
    import torch
    return {k: torch.from_numpy(v).cuda() for k, v in s.items()}


def _forward(s):
    from dirt_b200 import rasterise_ops as ops
    t = _cuda(s)
    pixels, ids = ops.rasterise_forward_raw(t['background'], t['vertices'], t['vertex_colors'], t['faces'])
    return pixels.cpu().numpy(), ids.cpu().numpy()


def _backward(s, pixels, grad_pixels, with_ids=None, groups=None):
    import torch
    from dirt_b200 import rasterise_ops as ops
    t = _cuda(s)
    ids = None if with_ids is None else torch.from_numpy(with_ids).cuda()
    gb, gv, gc = ops.rasterise_backward_raw(t['vertices'], t['faces'], torch.from_numpy(pixels).cuda(),
                                            torch.from_numpy(grad_pixels).cuda(), ids, groups)
    return gb.cpu().numpy(), gv.cpu().numpy(), gc.cpu().numpy()


def _check_scene(oracle, s, seed=0, groups=None, label=''):
    H, W = s['background'].shape[1:3]
    pixels_o, ids_o = oracle.forward(**s, return_face_ids=True)
    pixels_g, ids_g = _forward(s)
    np.testing.assert_array_equal(ids_g, ids_o, err_msg=label + ': face ids differ')
    ok, ratio = rel_close(pixels_g, pixels_o, name='pixels vs oracle')
    assert ok, '%s: pixels off by %.2fx the tolerance' % (label, ratio)
    gp = np.random.default_rng(seed).standard_normal(pixels_o.shape).astype(np.float32)
    gb_o, gv_o, gc_o = oracle.backward(s['vertices'], s['faces'], pixels_o, gp, groups)
    for ids_arg in (ids_g, None):   # cached visibility, and re-derived inside the call
        gb_g, gv_g, gc_g = _backward(s, pixels_o, gp, ids_arg, groups)
        np.testing.assert_array_equal(gb_g, gb_o, err_msg=label + ': grad_background differs')
        for name, a, b in (('grad_vertices', gv_g, gv_o), ('grad_vertex_colors', gc_g, gc_o)):
            ok, ratio = rel_close(a, b, name=name + ' vs oracle')
            assert ok, '%s: %s off by %.2fx the tolerance' % (label, name, ratio)
        assert (gv_g[..., 2] == 0).all()
    return pixels_g, ids_g


def test_square_golden_exact(cuda_lib):
    # BASELINE cfg1: tests/square_test.py, exact equality of all 16384 pixels
    pixels, ids = _forward(scenes.square_scene())
    np.testing.assert_array_equal(pixels[0, :, :, 0], np.load(os.path.join(GOLDEN, 'square_test_expected.npy')))


def test_public_api_square(cuda_lib):
    import dirt_b200 as dirt
    s = scenes.square_scene()
    pixels = dirt.rasterise(s['background'][0], s['vertices'][0], s['vertex_colors'][0], s['faces'][0],
                            height=128, width=128, channels=1)
    assert pixels.is_cuda and tuple(pixels.shape) == (128, 128, 1)
    np.testing.assert_array_equal(pixels[:, :, 0].cpu().numpy(), np.load(os.path.join(GOLDEN, 'square_test_expected.npy')))


@pytest.mark.parametrize('name,kwargs', [
    ('square_scene', dict(width=64, height=48, centre_x=20, centre_y=30, size=12)),
    ('cylinder_scene', dict()),
    ('cylinder_scene', dict(batch=2, seed=3)),
    ('bent_square_scene', dict(channels=3)),
    ('bent_square_scene', dict(channels=1)),
    ('bent_square_scene', dict(channels=4)),
    ('bent_square_scene', dict(channels=7)),
    ('bent_square_scene', dict(channels=2, width=37, height=29)),
    ('cube_scene', dict(width=160, height=120)),
    ('config2', dict()),
])
def test_reference_scenes(cuda_lib, oracle, name, kwargs):
    _check_scene(oracle, getattr(scenes, name)(**kwargs), label=name)


@pytest.mark.parametrize('seed', [0, 1, 2])
@pytest.mark.parametrize('channels', [1, 3, 4, 5])
def test_random_soup(cuda_lib, oracle, seed, channels):
    s = scenes.random_soup(batch=2, width=61, height=45, n_faces=70, channels=channels, seed=seed)
    _check_scene(oracle, s, seed=seed, label='soup')


@pytest.mark.parametrize('seed', [0, 1])
def test_behind_camera_and_guard_band(cuda_lib, oracle, seed):
    s = scenes.random_soup(batch=2, width=64, height=48, n_faces=40, channels=3, seed=10 + seed, behind_camera=True)
    _check_scene(oracle, s, seed=seed, label='behind-camera soup')
    # push some vertices far outside the guard band (>32768 px)
    s['vertices'][:, ::7, 0] *= 4000.0
    _check_scene(oracle, s, seed=seed, label='guard-band soup')


def test_reduced_configs(cuda_lib, oracle):
    _check_scene(oracle, scenes.config3(batch=3, width=160, height=128, level=3, background='uniform'), label='cfg3-small')
    _check_scene(oracle, scenes.config4(batch=2, width=128, height=128, level=3), label='cfg4-small')
    _check_scene(oracle, scenes.config5(batch=1, width=256, height=256, n_long=96, n_lat=48), label='cfg5-small')


def test_large_faces_and_many_faces_per_tile(cuda_lib, oracle):
    # faces larger than the per-tile binning limit (large list) mixed with > 32 small faces in one tile (chunking)
    rng = np.random.default_rng(4)
    s = scenes.random_soup(batch=1, width=96, height=80, n_faces=30, channels=3, seed=7)
    n = 200
    tiny_xy = rng.uniform(-0.12, 0.12, size=(n * 3, 2))
    tiny = np.concatenate([tiny_xy, rng.uniform(-0.9, 0.9, size=(n * 3, 1)), np.ones((n * 3, 1))], axis=1).astype(np.float32)
    V0 = s['vertices'].shape[1]
    s['vertices'] = np.concatenate([s['vertices'], tiny[None]], axis=1)
    s['vertex_colors'] = np.concatenate([s['vertex_colors'], rng.uniform(size=(1, n * 3, 3)).astype(np.float32)], axis=1)
    s['faces'] = np.concatenate([s['faces'], (V0 + np.arange(n * 3, dtype=np.int32)).reshape(1, n, 3)], axis=1)
    _check_scene(oracle, s, label='large+dense')


def test_edge_cases(cuda_lib, oracle):
    s = scenes.square_scene(32, 32, 16, 16, 8)
    # no faces at all: output is the background, gradients flow to the background only
    empty = dict(s, faces=np.zeros((1, 0, 3), np.int32))
    _check_scene(oracle, empty, label='no faces')
    # degenerate, out-of-range and NaN faces are ignored, not faulted on
    bad = dict(s)
    bad['faces'] = np.concatenate([s['faces'], np.array([[[0, 0, 1], [0, 1, 99], [-1, 1, 2]]], np.int32)], axis=1)
    _check_scene(oracle, bad, label='bad faces')
    nan = dict(s)
    nan['vertices'] = np.concatenate([s['vertices'], np.full((1, 1, 4), np.nan, np.float32)], axis=1)
    nan['vertex_colors'] = np.concatenate([s['vertex_colors'], np.ones((1, 1, 1), np.float32)], axis=1)
    nan['faces'] = np.concatenate([s['faces'], np.array([[[0, 1, 4]]], np.int32)], axis=1)
    _check_scene(oracle, nan, label='nan vertex')
    # frame sizes that are not multiples of the 8x8 tile, and a 1x1 frame
    _check_scene(oracle, scenes.random_soup(batch=1, width=13, height=7, n_faces=12, channels=3, seed=1), label='13x7')
    _check_scene(oracle, scenes.random_soup(batch=1, width=1, height=1, n_faces=5, channels=1, seed=2), label='1x1')


def test_visibility_gbuffer_matches_oracle(cuda_lib, oracle):
    import torch
    from dirt_b200 import rasterise_ops as ops
    s = scenes.random_soup(batch=2, width=64, height=48, n_faces=50, channels=3, seed=21, behind_camera=True)
    ids_o, gbuf_o = oracle.visibility(s['vertices'], s['faces'], 48, 64)
    t = _cuda(s)
    ids_g, gbuf_g = ops.rasterise_visibility_raw(t['vertices'], t['faces'], 48, 64)
    np.testing.assert_array_equal(ids_g.cpu().numpy(), ids_o)
    # the G-buffer arithmetic is fully specified (DESIGN.md, rule G): bit-identical, not merely close
    np.testing.assert_array_equal(gbuf_g.cpu().numpy(), gbuf_o)


def test_autograd_through_public_api(cuda_lib, oracle):
    import torch
    import dirt_b200 as dirt
    s = scenes.bent_square_scene(channels=4)
    t = _cuda(s)
    for k in ('background', 'vertices', 'vertex_colors'):
        t[k].requires_grad_(True)
    pixels = dirt.rasterise_batch(t['background'], t['vertices'], t['vertex_colors'], t['faces'])
    gp = torch.from_numpy(np.random.default_rng(0).standard_normal(tuple(pixels.shape)).astype(np.float32)).cuda()
    (pixels * gp).sum().backward()
    pixels_o = oracle.forward(**s)
    gb_o, gv_o, gc_o = oracle.backward(s['vertices'], s['faces'], pixels_o, gp.cpu().numpy())
    assert rel_close(pixels.detach().cpu().numpy(), pixels_o)[0]
    np.testing.assert_array_equal(t['background'].grad.cpu().numpy(), gb_o)
    assert rel_close(t['vertices'].grad.cpu().numpy(), gv_o)[0]
    assert rel_close(t['vertex_colors'].grad.cpu().numpy(), gc_o)[0]


def test_deferred_matches_reference_recipe(cuda_lib, oracle):
    # rasterise_deferred: vertex gradient from the SHADED pixels, attribute/background gradients through shader_fn
    # (dirt/rasterise_ops.py:180-257); compared with the same recipe evaluated with the oracle + torch autograd on CPU
    import torch
    import dirt_b200 as dirt
    s = scenes.bent_square_scene(channels=7, seed=5)
    t = _cuda(s)
    for k in ('background', 'vertices', 'vertex_colors'):
        t[k].requires_grad_(True)
    light = torch.tensor([0.3, 0.5, 0.8], device='cuda', requires_grad=True)

    def shader_fn(gbuffer, light):
        return gbuffer[..., :3] * (gbuffer[..., 3:6] * light).sum(-1, keepdim=True).abs() + 0.1 * gbuffer[..., 6:]

    pixels = dirt.rasterise_batch_deferred(t['background'], t['vertices'], t['vertex_colors'], t['faces'], shader_fn, [light])
    gp = torch.from_numpy(np.random.default_rng(0).standard_normal(tuple(pixels.shape)).astype(np.float32)).cuda()
    (pixels * gp).sum().backward()

    gbuf_o = torch.from_numpy(oracle.forward(**s)).requires_grad_(True)
    light_o = light.detach().cpu().requires_grad_(True)
    pix_o = shader_fn(gbuf_o, light_o)
    assert rel_close(pixels.detach().cpu().numpy(), pix_o.detach().numpy())[0]
    d_gbuf, d_light = torch.autograd.grad(pix_o, [gbuf_o, light_o], gp.cpu())
    _, gv_o, _ = oracle.backward(s['vertices'], s['faces'], pix_o.detach().numpy(), gp.cpu().numpy())
    gb_o, _, gc_o = oracle.backward(s['vertices'], s['faces'], gbuf_o.detach().numpy(), d_gbuf.numpy())
    assert rel_close(t['vertices'].grad.cpu().numpy(), gv_o)[0]
    assert rel_close(t['vertex_colors'].grad.cpu().numpy(), gc_o)[0]
    assert rel_close(t['background'].grad.cpu().numpy(), gb_o)[0]
    assert rel_close(light.grad.cpu().numpy(), d_light.numpy(), rel=1e-3)[0]


def test_host_entry_point_matches_oracle(cuda_lib, oracle):
    # dirt_b200.host.HostRasteriser: pinned host tensors in and out, chunked copy/compute pipeline
    import torch
    from dirt_b200.host import HostRasteriser
    s = scenes.config3(batch=5, width=96, height=64, level=2, background='uniform')
    B, H, W, C = s['background'].shape
    V, F = s['vertices'].shape[1], s['faces'].shape[1]
    gp = np.random.default_rng(3).standard_normal((B, H, W, C)).astype(np.float32)
    runner = HostRasteriser(B, H, W, C, V, F, chunks=3)
    pin = lambda a: torch.from_numpy(a).pin_memory()
    out = runner.step(pin(s['background']), pin(s['vertices']), pin(s['vertex_colors']), pin(s['faces']), pin(gp))
    runner.synchronize()
    pixels_o = oracle.forward(**s)
    gb_o, gv_o, gc_o = oracle.backward(s['vertices'], s['faces'], pixels_o, gp)
    assert rel_close(out['pixels'].numpy(), pixels_o)[0]
    np.testing.assert_array_equal(out['grad_background'].numpy(), gb_o)
    assert rel_close(out['grad_vertices'].numpy(), gv_o)[0]
    assert rel_close(out['grad_vertex_colors'].numpy(), gc_o)[0]


@pytest.mark.parametrize('channels,groups', [(3, [1, 1, 1]), (4, [1, 3]), (4, [1, 1, 1, 1]), (6, [3, 3])])
def test_custom_channel_groups(cuda_lib, oracle, channels, groups):
    # any grouping into widths 1 and 3 is a valid RasteriseGrad call sequence (dirt/rasterise_ops.py:132-177);
    # non-default groupings take the generic backward kernel
    s = scenes.bent_square_scene(40, 32, channels=channels, seed=3)
    pixels_o = oracle.forward(**s)
    gp = np.random.default_rng(1).standard_normal(pixels_o.shape).astype(np.float32)
    gb_o, gv_o, gc_o = oracle.backward(s['vertices'], s['faces'], pixels_o, gp, groups)
    gb_g, gv_g, gc_g = _backward(s, pixels_o, gp, None, groups)
    np.testing.assert_array_equal(gb_g, gb_o)
    assert rel_close(gv_g, gv_o)[0] and rel_close(gc_g, gc_o)[0]
    with pytest.raises(ValueError):
        _backward(s, pixels_o, gp, None, [2] * (channels // 2))


def test_backward_reusing_the_forward_workspace(cuda_lib, oracle):
    # workspace_holds_setup = 1: setup records and tile coverage flags of the forward call are reused
    import torch
    from dirt_b200 import rasterise_ops as ops
    s = scenes.config3(batch=3, width=160, height=96, level=2, background='uniform')
    t = _cuda(s)
    pixels, ids, ws = ops.rasterise_forward_raw(t['background'], t['vertices'], t['vertex_colors'], t['faces'], True, True)
    gp = torch.from_numpy(np.random.default_rng(5).standard_normal(tuple(pixels.shape)).astype(np.float32)).cuda()
    reused = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, gp, ids, None, ws)
    fresh = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, gp, ids, None, None)
    gb_o, gv_o, gc_o = oracle.backward(s['vertices'], s['faces'], pixels.cpu().numpy(), gp.cpu().numpy())
    for got in (reused, fresh):
        np.testing.assert_array_equal(got[0].cpu().numpy(), gb_o)
        assert rel_close(got[1].cpu().numpy(), gv_o)[0] and rel_close(got[2].cpu().numpy(), gc_o)[0]


def test_kernel_timer_hooks(cuda_lib):
    import torch
    from dirt_b200 import rasterise_ops as ops
    s = scenes.config3(batch=1, width=64, height=64, level=1)
    t = _cuda(s)
    assert cuda_lib.dirt_kernel_timer_enable(1) == 0
    ops.rasterise_forward_raw(t['background'], t['vertices'], t['vertex_colors'], t['faces'])
    ms = float(cuda_lib.dirt_kernel_timer_elapsed_ms())
    assert 0.0 < ms < 1000.0
    assert cuda_lib.dirt_kernel_timer_enable(0) == 0
    assert cuda_lib.dirt_kernel_timer_enable(7) != 0
    assert cuda_lib.dirt_last_launch_count() >= 0


def test_full_size_properties(cuda_lib):
    # BASELINE cfg3 at its full frame size (reduced batch): size-independent properties of the CUDA path
    import torch
    from dirt_b200 import rasterise_ops as ops
    s = scenes.config3(batch=4, width=512, height=512, background='uniform')
    t = _cuda(s)
    pixels, ids = ops.rasterise_forward_raw(t['background'], t['vertices'], t['vertex_colors'], t['faces'])
    cov = ids >= 0
    assert 0.40 < float(cov.float().mean()) < 0.48
    # uncovered pixels are the background, bit for bit; covered pixels of the mask channel are exactly 1 (all vertices have 1)
    assert torch.equal(pixels[~cov], t['background'][~cov])
    assert torch.equal(pixels[..., 0][cov], torch.ones_like(pixels[..., 0][cov]))
    # the normal channels of a unit sphere stay unit length up to interpolation across small faces
    n = pixels[..., 1:][cov].norm(dim=-1)
    assert float(n.min()) > 0.99 and float(n.max()) < 1.0 + 1e-5
    # linearity of the backward pass in grad_pixels; grad_background + coverage partition grad_pixels
    g1 = torch.randn_like(pixels); g2 = torch.randn_like(pixels)
    b1 = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, g1, ids)
    b2 = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, g2, ids)
    b12 = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, g1 + 2 * g2, ids)
    for k in (1, 2):
        ref = b1[k] + 2 * b2[k]
        assert float((b12[k] - ref).abs().max()) <= 2e-4 * float(ref.abs().max())
    assert torch.equal(b1[0][~cov], g1[~cov]) and float(b1[0][cov].abs().max()) == 0.0
    assert float(b1[1][..., 2].abs().max()) == 0.0


# ---- round 2: accumulation over the batch, partial gradients, workspace validation, full sizes -------------------

def test_shared_geometry_accumulates_over_the_batch(cuda_lib, oracle):
    # DIRT_BWD_SHARED_GEOMETRY: [V,4] / [V,C] outputs equal the per-item gradients summed over the batch (SURVEY 8e)
    import torch
    from dirt_b200 import rasterise_ops as ops
    for s in (scenes.config3(batch=5, width=160, height=128, level=3, background='uniform'),
              scenes.config4(batch=4, width=128, height=96, level=2)):
        t = _cuda(s)
        pixels, ids, ws = ops.rasterise_forward_raw(t['background'], t['vertices'], t['vertex_colors'], t['faces'], True, True)
        gp = torch.from_numpy(np.random.default_rng(9).standard_normal(tuple(pixels.shape)).astype(np.float32)).cuda()
        gb, gv, gc = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, gp, ids, None, ws, shared_geometry=True)
        assert tuple(gv.shape) == tuple(s['vertices'].shape[1:]) and tuple(gc.shape) == tuple(s['vertex_colors'].shape[1:])
        gb_o, gv_o, gc_o = oracle.backward(s['vertices'], s['faces'], pixels.cpu().numpy(), gp.cpu().numpy())
        np.testing.assert_array_equal(gb.cpu().numpy(), gb_o)
        for name, got, want in (('grad_vertices', gv, gv_o.astype(np.float64).sum(0)), ('grad_vertex_colors', gc, gc_o.astype(np.float64).sum(0))):
            ok, ratio = rel_close(got.cpu().numpy(), want)
            assert ok, 'shared %s off by %.2fx the tolerance' % (name, ratio)


@pytest.mark.parametrize('channels', [1, 3, 4, 7])
def test_partial_gradients(cuda_lib, oracle, channels):
    # DIRT_BWD_SKIP_POSITION / DIRT_BWD_SKIP_COLOUR: each half equals the corresponding outputs of the full call
    import torch
    from dirt_b200 import rasterise_ops as ops
    s = scenes.random_soup(batch=2, width=61, height=45, n_faces=70, channels=channels, seed=4)
    t = _cuda(s)
    pixels, ids = ops.rasterise_forward_raw(t['background'], t['vertices'], t['vertex_colors'], t['faces'])
    gp = torch.from_numpy(np.random.default_rng(2).standard_normal(tuple(pixels.shape)).astype(np.float32)).cuda()
    gb_o, gv_o, gc_o = oracle.backward(s['vertices'], s['faces'], pixels.cpu().numpy(), gp.cpu().numpy())
    gb, gv, gc = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, gp, ids, want_position=False)
    np.testing.assert_array_equal(gb.cpu().numpy(), gb_o)
    assert rel_close(gc.cpu().numpy(), gc_o)[0] and float(gv.abs().max()) == 0.0
    gb, gv, gc = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, gp, ids, want_colour=False)
    assert gb is None and float(gc.abs().max()) == 0.0
    ok, ratio = rel_close(gv.cpu().numpy(), gv_o)
    assert ok, 'position-only grad_vertices off by %.2fx the tolerance' % ratio


def test_stale_workspace_is_detected(cuda_lib, oracle):
    # workspace_holds_setup is a checked promise: a workspace filled for OTHER geometry raises the device-side flag
    # and poisons grad_vertices; the Python layer never makes the promise for a workspace that does not match
    import ctypes
    import torch
    from dirt_b200 import rasterise_ops as ops, _lib
    s = scenes.config3(batch=2, width=96, height=64, level=2, background='uniform')
    t = _cuda(s)
    other = {k: v.clone() for k, v in t.items()}
    other['vertices'][..., 0] += 0.05
    pixels, ids, ws = ops.rasterise_forward_raw(t['background'], t['vertices'], t['vertex_colors'], t['faces'], True, True)
    _, _, ws_other = ops.rasterise_forward_raw(other['background'], other['vertices'], other['vertex_colors'], other['faces'], True, True)
    gp = torch.randn_like(pixels)
    B, H, W, C = pixels.shape
    V, F = t['vertices'].shape[1], t['faces'].shape[1]
    want = oracle.backward(s['vertices'], s['faces'], pixels.cpu().numpy(), gp.cpu().numpy())
    # (a) Python layer: the foreign workspace is not reused, the result is right
    got = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, gp, ids, None, ws_other)
    assert rel_close(got[1].cpu().numpy(), want[1])[0]
    ops.workspace_status(ws_other, B, H, W, C, V, F)   # no flag raised
    # an in-place update of the vertices invalidates the matching workspace as well (version counter)
    t['vertices'].add_(0.0)
    got = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, gp, ids, None, ws)
    assert rel_close(got[1].cpu().numpy(), want[1])[0]
    # (b) C ABI: make the false promise directly
    L = _lib.lib()
    gb = torch.empty_like(pixels); gv = torch.empty((B, V, 4), device='cuda'); gc = torch.empty((B, V, C), device='cuda')
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    nbytes = int(L.dirt_workspace_bytes(B, H, W, C, V, F))
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = L.dirt_rasterise_backward(p(t['vertices']), p(t['faces']), p(pixels), p(gp), p(ids), p(gb), p(gv), p(gc),
                                   B, H, W, C, V, F, None, 0, 1, p(ws_other), nbytes, stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert bool(torch.isnan(gv.flatten()[0]))
    with pytest.raises(RuntimeError):
        ops.workspace_status(ws_other, B, H, W, C, V, F)
    # the matching workspace passes
    rc = L.dirt_rasterise_backward(p(t['vertices']), p(t['faces']), p(pixels), p(gp), p(ids), p(gb), p(gv), p(gc),
                                   B, H, W, C, V, F, None, 0, 1, p(ws), nbytes, stream)
    assert rc == 0
    ops.workspace_status(ws, B, H, W, C, V, F)
    assert rel_close(gv.cpu().numpy(), want[1])[0]


@pytest.mark.parametrize('name,kwargs', [
    ('config3', dict(batch=2, width=512, height=512, background='uniform')),       # the benched workload's frame and mesh
    ('config4', dict(batch=2, width=512, height=512)),
    ('config5', dict(batch=1, width=1024, height=1024)),                           # 49 728 faces, pole slivers
    ('cube_scene', dict(width=640, height=480)),                                   # samples/simple.py: 12 large faces
])
def test_full_size_configs_match_oracle(cuda_lib, oracle, name, kwargs):
    _check_scene(oracle, getattr(scenes, name)(**kwargs), label=name + '-full')


def test_direct_and_deferred_agree_for_a_linear_shader(cuda_lib):
    # tests/deferred_grad_test.py:168-219 renders direct (Gouraud) and deferred gradients side by side.  For a shader that
    # is LINEAR in the attributes the two recipes are the same function, so pixels and every gradient must agree:
    # vertices (filtering the shaded image), attributes / background (through shader_fn) and the shader's own inputs.
    import torch
    import dirt_b200 as dirt
    s = scenes.bent_square_scene(48, 40, channels=6, seed=2)
    t = _cuda(s)
    gp = torch.from_numpy(np.random.default_rng(4).standard_normal((48 * 40 * 3,)).astype(np.float32)).cuda().reshape(1, 40, 48, 3)

    def run(deferred):
        leaves = {k: t[k].clone().requires_grad_(True) for k in ('background', 'vertices', 'vertex_colors')}
        gain = torch.tensor([0.7, 1.3, 0.4], device='cuda', requires_grad=True)
        shade = lambda a, k: a[..., :3] * k + 0.5 * a[..., 3:6]
        if deferred:
            pixels = dirt.rasterise_batch_deferred(leaves['background'], leaves['vertices'], leaves['vertex_colors'], t['faces'],
                                                   shade, [gain])
        else:
            pixels = dirt.rasterise_batch(shade(leaves['background'], gain), leaves['vertices'], shade(leaves['vertex_colors'], gain),
                                          t['faces'])
        (pixels * gp).sum().backward()
        return pixels.detach(), [leaves[k].grad for k in ('background', 'vertices', 'vertex_colors')] + [gain.grad]

    pix_a, grads_a = run(False)
    pix_b, grads_b = run(True)
    assert rel_close(pix_b.cpu().numpy(), pix_a.cpu().numpy())[0]
    for name, a, b in zip(('background', 'vertices', 'attributes', 'gain'), grads_a, grads_b):
        ok, ratio = rel_close(b.cpu().numpy(), a.cpu().numpy(), rel=2e-4)
        assert ok, 'deferred vs direct: grad %s off by %.2fx the tolerance' % (name, ratio)


def test_pixel_jacobians_of_the_cylinder(cuda_lib, oracle):
    # tests/rasterise_tests.py:108-131 evaluates d pixel / d (translation, rotation, background, colour) one pixel at a
    # time.  Same recipe through the public API, compared with the oracle chained through the same torch transform.
    import torch
    import dirt_b200 as dirt
    s = scenes.cylinder_scene()
    H, W = s['background'].shape[1:3]
    base = torch.from_numpy(s['vertices'][0]).cuda()

    def clip_vertices(translation):
        # a clip-space shift stands in for the scene's translation parameter: x, y scale with w like a view-space shift does
        return base + torch.stack([translation[0] * base[:, 3], translation[1] * base[:, 3], translation[2] * 0 * base[:, 3],
                                   torch.zeros_like(base[:, 3])], dim=1)

    pixels_o = oracle.forward(**s)
    rng = np.random.default_rng(0)
    ids = oracle.visibility(s['vertices'], s['faces'], H, W)[0][0]
    edge = np.argwhere((ids >= 0) & ((np.roll(ids, 1, 1) < 0) | (np.roll(ids, -1, 0) < 0)))
    picks = [tuple(edge[i]) for i in rng.choice(len(edge), size=6, replace=False)] + [(H // 2, W // 2), (2, 3)]
    for (y, x) in picks:
        for c in (0, 2):
            translation = torch.zeros(3, device='cuda', requires_grad=True)
            bg = torch.from_numpy(s['background'][0]).cuda().requires_grad_(True)
            col = torch.from_numpy(s['vertex_colors'][0]).cuda().requires_grad_(True)
            pixels = dirt.rasterise(bg, clip_vertices(translation), col, torch.from_numpy(s['faces'][0]).cuda())
            pixels[y, x, c].backward()
            indicator = np.zeros_like(pixels_o); indicator[0, y, x, c] = 1.0
            gb_o, gv_o, gc_o = oracle.backward(s['vertices'], s['faces'], pixels_o, indicator)
            t_cpu = torch.zeros(3, requires_grad=True)
            b_cpu = base.cpu()
            v_cpu = b_cpu + torch.stack([t_cpu[0] * b_cpu[:, 3], t_cpu[1] * b_cpu[:, 3], t_cpu[2] * 0 * b_cpu[:, 3], torch.zeros_like(b_cpu[:, 3])], dim=1)
            (v_cpu * torch.from_numpy(gv_o[0])).sum().backward()
            np.testing.assert_allclose(translation.grad.cpu().numpy(), t_cpu.grad.numpy(), rtol=1e-4, atol=1e-6 * float(np.abs(gv_o).max() + 1))
            np.testing.assert_array_equal(bg.grad.cpu().numpy(), gb_o[0])
            assert rel_close(col.grad.cpu().numpy(), gc_o[0])[0]


def test_bin_overflow_paths(cuda_lib, oracle):
    # one-pass binning: a tile's bin holds 128 references; the rest goes to the overflow list of the tile's row of tiles
    # (1024 entries per row and image), and when that is full too to the image's large list.  1200 stacked faces reach
    # all three levels (tests/test_setup_records_host.py counts them on the CPU, tests/test_gpu_setup_records.py in
    # the workspace).
    import kernel_paths as kp
    _check_scene(oracle, kp.bin_overflow_scene(), label='bin overflow')
    # two images with different loads: the lists are per image (image 1: bins and row lists only)
    _check_scene(oracle, kp.bin_overflow_scene(batch=2), label='bin overflow, two images')
