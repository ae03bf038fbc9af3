"""CPU: every scene of tests/test_gpu_launch_limits.py takes the capped grid-stride loop it is there for past its first
round, ending on a partial round: the variant's scenes at the caps of the small-grid build, the product's at the shipped
caps.  A scene that stopped crossing its boundary (a changed size, cap or launch rule) fails here instead of silently
testing one round on the GPU."""
import os
import re

import numpy as np
import pytest

import launch_limits as ll
import kernel_paths as kp
import texture_det_order as order

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _read(name):
    with open(os.path.join(ROOT, 'dirt_b200', 'csrc', name)) as f:
        return f.read()


def test_shipped_caps_are_the_sources_defaults():
    """SHIPPED restates each `#define DIRT_..._` default of the sources, and the variant overrides every one of them."""
    found = {}
    for name in ('texture.cu', 'lighting.cu', 'normals.cu', 'deterministic.cu', 'derivatives.cu'):
        for key, value in re.findall(r'#ifndef (DIRT_\w+)\n#define \1 (.+)\n#endif', _read(name)):
            found[key] = eval(value.replace('ll', ''))   # literals such as (1ll << 20) or 0x7fffffffll
    assert found == ll.SHIPPED
    assert set(ll.SMALL) == set(ll.SHIPPED)
    assert all(ll.SMALL[k] < ll.SHIPPED[k] for k in ll.SMALL)


def test_restated_helpers():
    assert ll.rounds(10, 3) == 4 and ll.crosses(10, 3) and not ll.crosses(9, 3) and not ll.crosses(3, 3)
    assert ll.sort_passes(255) == 1 and ll.sort_passes(256) == 2 and ll.sort_passes((1 << 24) - 1) == 3
    assert ll.sort_passes(1 << 24) == 4
    assert ll.tex_blocks(1 << 24, ll.SHIPPED) == 1 << 16 and ll.tex_blocks((1 << 24) + 1, ll.SHIPPED) == 1 << 16
    assert ll.generic_step(1000, 5, ll.SMALL) == (102, 2)                    # 512 elements = 102 lookups + 2 channels
    assert ll.chunk_slots([4096, 4097, 9000]) == 2 + 3


# ---- (a) the small-grid variant --------------------------------------------------------------------------------------

@pytest.mark.parametrize('C', ll.VAR_TEX_CHANNELS)
def test_variant_texture_lookups_loop(C):
    total = ll.VAR_TEX_LOOKUPS + 78
    assert ll.crosses(*ll.tex_forward(total, C, ll.SMALL))
    assert ll.crosses(total, ll.tex_blocks(total, ll.SMALL) * ll.TEX_THREADS)           # the backward kernel
    if C in (5, 6, 7):
        assert ll.generic_step(total, C, ll.SMALL)[1] != 0                              # the step wraps the channel
    H, W = ll.VAR_TEX_SHAPE
    assert ll.crosses(*ll.segment_bounds(H * W, ll.SMALL)) and ll.crosses(*ll.gather(H * W, ll.SMALL))


@pytest.mark.parametrize('C', ll.VAR_DET_LONG_CHANNELS)
def test_variant_deterministic_chunks_loop(C):
    TH, TW = ll.VAR_DET_LONG
    idx = ll.det_long_indices()
    terms = np.bincount(order.ordered_terms(idx, np.zeros((len(idx), 1), np.float32), 1, TH, TW, len(idx), 'bilinear')[0],
                        minlength=TH * TW)
    assert (terms > ll.DET_CHUNK).all()
    slots = ll.chunk_slots(terms)
    assert ll.crosses(*ll.chunk(len(idx), 'bilinear', slots, ll.SMALL))
    assert ll.crosses(*ll.finish(len(idx), 'bilinear', TH * TW, C, ll.SMALL))
    assert ll.crosses(*ll.gather(TH * TW, ll.SMALL))


def test_variant_pyramid_and_trilinear_loop():
    TB, TH, TW = ll.VAR_MIP_SHAPE
    for C in (1, 3, 5):
        assert ll.crosses(*ll.mip_build(TB, TH, TW, C, 1, ll.SMALL)), C
        assert ll.crosses(*ll.mip_collapse(TB, TH, TW, C, ll.SMALL)), C
        total = TB * (ll.VAR_TEX_LOOKUPS + 78)
        assert ll.crosses(total, ll.tex_blocks(total, ll.SMALL) * ll.TEX_THREADS)
        for k in range(2):   # the deterministic path's passes of levels 0 and 1
            n = TB * (TH >> k) * (TW >> k)
            assert ll.crosses(*ll.segment_bounds(n, ll.SMALL)) and ll.crosses(*ll.gather(n, ll.SMALL)), k


@pytest.mark.parametrize('C', ll.VAR_LIGHT_CHANNELS)
@pytest.mark.parametrize('model', sorted(ll.LIGHT_MODELS))
def test_variant_lighting_items_and_reduction_loop(model, C):
    assert ll.crosses(*ll.point_grid(ll.VAR_LIGHT_B, ll.SMALL))
    assert ll.crosses(*ll.reduce_grid(ll.VAR_LIGHT_B * ll.param_columns(model, C), ll.SMALL))
    assert ll.VAR_LIGHT_V % 32 != 0 and ll.VAR_LIGHT_V > ll.LIGHT_THREADS


@pytest.mark.parametrize('mesh', ['icosphere', 'fan'])
def test_variant_normals_loop(mesh):
    v, f = ll.normals_meshes()[mesh]
    for name, (work, stride) in ll.normals_loops(ll.VAR_NORMALS_ITEMS, len(v), len(f), ll.SMALL).items():
        assert ll.crosses(work, stride), (mesh, name, work, stride)
    if mesh == 'fan':
        assert np.bincount(f.reshape(-1))[0] > 32   # a row longer than NORMALS_LONG_ROW


def _det_scenes():
    from dirt_b200 import scenes
    yield 'fans', kp.overflow_scene(3, ll.VAR_OVERFLOW_W)
    yield 'soup', scenes.random_soup(channels=3, **ll.VAR_SOUP)


def test_variant_deterministic_rasteriser_loops():
    for tag, s in _det_scenes():
        B, H, W, _ = s['background'].shape
        V, F = s['vertices'].shape[1], s['faces'].shape[1]
        for name, (work, stride) in ll.det_raster_loops(B, H, W, V, F, ll.SMALL).items():
            assert ll.crosses(work, stride), (tag, name, work, stride)


def test_variant_derivatives_loop():
    s = ll.VAR_DERIV_SOUP
    assert ll.crosses(*ll.derivatives_loop(s['batch'], s['height'], s['width'], ll.SMALL))


# ---- (b) the product at its shipped caps -----------------------------------------------------------------------------

@pytest.mark.parametrize('C', [3, 4])
def test_product_texture_lookups_loop(C):
    assert ll.crosses(*ll.tex_forward(ll.TEX_LOOKUPS, C, ll.SHIPPED))
    assert ll.TEX_LOOKUPS % 32 != 0                  # the last round ends inside a warp


@pytest.mark.parametrize('C', ll.GENERIC_CHANNELS)
def test_product_generic_forward_loops_and_wraps(C):
    n = ll.generic_lookups(C)
    work, stride = ll.tex_forward(n, C, ll.SHIPPED)
    assert work == n * C and ll.crosses(work, stride) and work < 2 * stride
    assert ll.generic_step(n, C, ll.SHIPPED)[1] != 0


def test_product_pyramid_loops():
    TB, TH, TW, C = ll.MIP_LARGE
    assert ll.crosses(*ll.mip_build(TB, TH, TW, C, 1, ll.SHIPPED))
    assert ll.crosses(*ll.mip_collapse(TB, TH, TW, C, ll.SHIPPED))


def test_product_deterministic_texture_loops():
    (H, W), n = ll.DET_SCAN
    assert ll.sort_tiles(n) == 260 and ll.scan_rounds(n) == 2
    (H, W), n = ll.DET_PASSES
    assert ll.sort_passes(H * W) == 4
    assert ll.crosses(*ll.segment_bounds(H * W, ll.SHIPPED)) and ll.crosses(*ll.gather(H * W, ll.SHIPPED))
    (H, W), n = ll.DET_SLOTS
    # a 2 x 2 texture: every lookup's four corners land on the four texels, n terms each
    slots = ll.chunk_slots([n] * (H * W))
    assert slots > 65536
    assert ll.crosses(*ll.chunk(n, 'bilinear', slots, ll.SHIPPED))


@pytest.mark.parametrize('model', sorted(ll.LIGHT_MODELS))
def test_product_lighting_items_and_reduction_loop(model):
    assert ll.crosses(*ll.point_grid(ll.LIGHT_B, ll.SHIPPED))
    assert ll.rounds(*ll.point_grid(ll.LIGHT_B, ll.SHIPPED)) == 3
    assert ll.crosses(*ll.reduce_grid(ll.LIGHT_B * ll.param_columns(model, ll.LIGHT_MODELS[model]), ll.SHIPPED))
    assert ll.LIGHT_V % 32 == 1
    cap = ll.SHIPPED['DIRT_LIGHT_MAX_ITEMS_PER_GRID']
    assert {cap - 1, cap, cap + 1, 2 * cap, ll.LIGHT_B - 1} <= set(ll.LIGHT_ITEMS)
