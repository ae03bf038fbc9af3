"""GPU: the atomic and reduced gradient paths on exactly summable inputs (tests/exact_sums.py), compared with `==`.

Every term of these scenes is a multiple of 2^-m and every output element's terms have sum |t| * 2^m < 2^24, so any
order of fp32 additions is exact: the kernels must return the float64 sum of the terms, bit for bit, and two runs must
agree bit for bit.  A lost, duplicated or misrouted term shows however many terms share its element, which the 1e-4
relative bar of the other suites cannot promise for sums of 10^4 to 10^6 terms.  Each test proves the condition for its
own inputs (exact_sums.check_exact) before it compares; a failure names the first differing element and its term count.

Covered: the rasteriser's grad_vertex_colors (default path, per-face reduction and tile_generic, per item and
SHARED_GEOMETRY, C = 1, 3 and 4, the deterministic path and the four-slot build); sample_texture's bilinear and nearest
default backward (grad_texture and grad_indices, C = 1, 2, 3, 4, 5, 8, shared and per-item textures, 4-byte aligned
buffers, contention, a round past 2^24 lookups, warp patterns on both sides of agg_plan's pull / butterfly rule); and
diffuse_directional's light direction and colour gradients, whose reduction kernel all the point models share; the
trilinear texture at power-of-two footprints; sample_cubemap bilinear, nearest and trilinear, default and
deterministic; and the shadow map's default map gradient at R = 0.  The small-grid build runs the texture, trilinear,
lighting and deterministic rasteriser cases again."""
import ctypes

import numpy as np
import pytest
import torch

import exact_sums as es
import variant_builds
from test_gpu_deterministic import det_call
from test_gpu_launch_limits import _through
from test_gpu_paths import abi_backward, abi_forward
from test_gpu_shadow_edges import _gpu as shadow_call

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)


@pytest.fixture(scope='module')
def small(cuda_lib, tmp_path_factory):
    return variant_builds.small_grid_library(tmp_path_factory)


@pytest.fixture(scope='module')
def four_slot(cuda_lib, tmp_path_factory):
    return variant_builds.four_slot_library(tmp_path_factory)


def _same(got, want, counts, what):
    msg = es.first_difference(got, want, counts)
    assert not msg, '%s: %s' % (what, msg)


def _bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ---- B. sample_texture, bilinear and nearest, default backward ------------------------------------------------------

def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


def _tex_backward(L, tex, idx, gout, mode, offset=0):
    """dirt_texture_sample_backward of library L -> (grad_texture, grad_indices).  offset > 0 places every buffer that
    many floats past a 256-byte boundary (4-byte aligned only: the scalar loads and REDs)."""
    TB, H, W, C = tex.shape
    B, N = idx.shape[:2]

    def place(t, copy=True):   # outputs start as NaN, so that an element the call does not write shows
        buf = torch.full((t.numel() + 8,), float('nan'), device=DEV)
        v = buf[offset:offset + t.numel()]
        if copy:
            v.copy_(t.reshape(-1))
        return v

    tx, ix, go = place(tex), place(idx), place(gout)
    gt, gi = place(tex, False), place(idx, False)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    rc = L.dirt_texture_sample_backward(p(tx), p(ix), p(go), p(gt), p(gi), TB, H, W, C, B, N,
                                        1 if mode == 'nearest' else 0, _stream())
    assert rc == 0, L.dirt_error_string(rc)
    return gt.reshape(tex.shape).clone(), gi.reshape(idx.shape).clone()


def _check_texture(L, tex, idx, gout, mode, what, offset=0, chunk=None):
    gt_want, nt, gi_want, ni = es.texture_expected(tex, idx, gout, mode, chunk)
    gt, gi = _tex_backward(L, tex, idx, gout, mode, offset)
    _same(gt, gt_want, nt, what + ' grad_texture')
    _same(gi, gi_want, ni, what + ' grad_indices')
    gt2, gi2 = _tex_backward(L, tex, idx, gout, mode, offset)
    assert _bits(gt2, gt) and _bits(gi2, gi), what + ': a second run differs'


@pytest.mark.parametrize('per_item', [False, True])
@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [1, 2, 3, 4, 5, 8])
def test_texture_channels(cuda_lib, C, mode, per_item):
    """Every channel path: v4 (C = 4), v2 (C = 2), scalar REDs (1, 3) and the any-C loop (5, 8)."""
    tex, idx, gout = es.texture_scene(3 if per_item else 1, 37, 29, C, 3, 20000, 100 + C, DEV)
    _check_texture(cuda_lib, tex, idx, gout, mode, 'C=%d %s per_item=%s' % (C, mode, per_item))


@pytest.mark.parametrize('C', [1, 2, 3, 4, 5])
def test_texture_four_byte_aligned(cuda_lib, C):
    tex, idx, gout = es.texture_scene(1, 19, 13, C, 1, 3001, 110 + C, DEV)
    _check_texture(cuda_lib, tex, idx, gout, 'bilinear', '4-byte aligned C=%d' % C, offset=1)


def test_texture_through_the_public_call(cuda_lib):
    import dirt_b200 as dirt
    tex, idx, gout = es.texture_scene(1, 37, 29, 4, 2, 5000, 120, DEV)
    gt_want, nt, gi_want, ni = es.texture_expected(tex, idx, gout, 'bilinear')
    t, i = tex[0].clone().requires_grad_(True), idx.clone().requires_grad_(True)
    (dirt.sample_texture(t, i) * gout).sum().backward()
    _same(t.grad, gt_want[0], nt[0], 'sample_texture grad_texture')
    _same(i.grad, gi_want, ni, 'sample_texture grad_indices')


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [1, 2, 4, 6])
def test_texture_contention(cuda_lib, C, mode):
    """2^20 lookups into a 2 x 2 texture: about 2^20 terms per texel (bilinear), every warp's lanes in four groups."""
    tex, idx, gout = es.texture_scene(1, 2, 2, C, 1, 1 << 20, 130 + C, DEV)
    _check_texture(cuda_lib, tex, idx, gout, mode, '2x2 contention C=%d %s' % (C, mode))


def test_texture_past_two_to_the_24_lookups(cuda_lib):
    """2^24 + 4099 lookups: one grid-stride round past the product's 2^16 CTAs of 256 lookups."""
    tex, idx, gout = es.texture_scene(1, 61, 67, 2, 1, (1 << 24) + 4099, 140, DEV)
    _check_texture(cuda_lib, tex, idx, gout, 'bilinear', '2^24 + 4099 lookups', chunk=1 << 22)


@pytest.mark.parametrize('C', [1, 2, 3, 4, 5])
@pytest.mark.parametrize('pattern', sorted(es.WARP_PATTERNS))
def test_texture_warp_patterns(cuda_lib, pattern, C):
    """Warps whose lanes form the pattern's groups on every corner (tests/test_exact_sums_host.py shows which side of
    agg_plan's rule each pattern takes), 997 warps plus a partial one."""
    H, W = 24, 40
    idx = es.warp_pattern_indices(pattern, 998, H, W, 150)[:-19].to(DEV)[None]
    tex = es.dyadic((1, H, W, C), es.TEXELS, 151, DEV)
    gout = es.dyadic((1, idx.shape[1], C), es.GRADS, 152, DEV)
    _check_texture(cuda_lib, tex, idx, gout, 'bilinear', 'pattern %s C=%d' % (pattern, C))


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [1, 2, 3, 4, 5])
def test_texture_small_grid(small, C, mode):
    """The small-grid build: two texture CTAs, so every lookup after the first 512 comes in a later round."""
    tex, idx, gout = es.texture_scene(2, 37, 29, C, 2, 3001, 160 + C, DEV)
    _check_texture(small, tex, idx, gout, mode, 'small grid C=%d %s' % (C, mode))
    for pattern in ('seven', 'twelve_pair', 'pairs'):
        pidx = es.warp_pattern_indices(pattern, 40, 24, 40, 161)[:-5].to(DEV)[None]
        ptex = es.dyadic((1, 24, 40, C), es.TEXELS, 162, DEV)
        pgout = es.dyadic((1, pidx.shape[1], C), es.GRADS, 163, DEV)
        _check_texture(small, ptex, pidx, pgout, 'bilinear', 'small grid pattern %s C=%d' % (pattern, C))


# ---- F. diffuse_directional ------------------------------------------------------------------------------------------

def _diffuse(L, x, g):
    """diffuse_directional through library L -> {key: grad} of (out * g).sum() for every input."""
    from dirt_b200 import lighting
    leaves = {k: v.clone().requires_grad_(True) for k, v in x.items()}
    with _through(L):
        out = lighting.diffuse_directional(leaves['n'], leaves['k'], leaves['L'], leaves['lc'])
        (out * g).sum().backward()
    return {k: v.grad for k, v in leaves.items()}


def _check_diffuse(L, x, g, what):
    from dirt_b200 import lighting
    want = es.diffuse_expected(x, g)
    got = _diffuse(L, x, g)
    for k in ('L', 'lc'):
        _same(got[k], want[k][0], want[k][1], '%s grad %s' % (what, k))
    # the per-point gradients are single products and sums of a few channels: exact too
    leaves = {k: v.double().requires_grad_(True) for k, v in x.items()}
    (lighting._diffuse_directional(leaves['n'], leaves['k'], leaves['L'], leaves['lc']) * g.double()).sum().backward()
    for k in ('n', 'k'):
        _same(got[k], leaves[k].grad, None, '%s grad %s' % (what, k))
    again = _diffuse(L, x, g)
    assert all(_bits(again[k], got[k]) for k in got), what + ': a second run differs'


@pytest.mark.parametrize('per_item', [False, True])
def test_diffuse_cfg3_size(cuda_lib, per_item):
    """64 x 512^2 points: 2^16 partial rows per shared parameter, 2^10 per item."""
    x, g = es.diffuse_scene((64,), 512 * 512, 3, per_item, 200, DEV, sparse=1 if per_item else 64)
    _check_diffuse(cuda_lib, x, g, 'cfg3 per_item=%s' % per_item)


@pytest.mark.parametrize('lib', ['cuda_lib', 'small'])
@pytest.mark.parametrize('per_item', [False, True])
@pytest.mark.parametrize('C', [1, 3, 4])
def test_diffuse_partial_chunks(request, lib, C, per_item):
    """V = 1000 and 257: the last CTA of each item holds 232 and 1 points."""
    L = request.getfixturevalue(lib)
    for V in (1000, 257):
        x, g = es.diffuse_scene((5, 3), V, C, per_item, 210 + V + C, DEV)
        _check_diffuse(L, x, g, '%s V=%d C=%d per_item=%s' % (lib, V, C, per_item))


@pytest.mark.parametrize('per_item', [False, True])
def test_diffuse_past_the_item_grid(cuda_lib, per_item):
    """131 077 items of 33 points: items past two rounds of gridDim.y, and per-item totals past 2^20 reduction CTAs."""
    x, g = es.diffuse_scene((131077,), 33, 3, per_item, 220, DEV, sparse=1 if per_item else 8)
    _check_diffuse(cuda_lib, x, g, '131077 items per_item=%s' % per_item)


# ---- A. rasteriser, grad_vertex_colors ---------------------------------------------------------------------------------

def _raster(L, s, gp, deterministic=False, shared=False):
    """grad_vertex_colors of scene s through library L (the deterministic call through the package's routing)."""
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in s.items()}
    B, H, W, C = gp.shape
    V = s['vertices'].shape[1]
    pixels = torch.empty_like(t['background'])
    ids = torch.empty((B, H, W), dtype=torch.int32, device=DEV)
    abi_forward(L, t['background'], t['vertices'], t['vertex_colors'], t['faces'], pixels, ids)
    g = torch.from_numpy(gp).to(DEV)
    flags = 1 if shared else 0
    if deterministic:
        with _through(L):
            return det_call(t, pixels, g, ids, flags=flags)[2], ids
    lead = () if shared else (B,)
    gb, gv = torch.empty_like(pixels), torch.empty(lead + (V, 4), device=DEV)
    gc = torch.full(lead + (V, C), float('nan'), device=DEV)
    abi_backward(L, t['vertices'], t['faces'], pixels, g, ids, gb, gv, gc, flags=flags)
    return gc, ids


@pytest.mark.parametrize('lib', ['cuda_lib', 'four_slot'])
@pytest.mark.parametrize('shared', [False, True])
@pytest.mark.parametrize('kind', ['large', 'tiny'])
@pytest.mark.parametrize('C', [1, 3, 4])
def test_raster_vertex_colours(request, oracle, lib, kind, C, shared):
    """'large': eight faces of about 32 640 pixels (per-face reduction); 'tiny': 2048 faces, every tile past its face
    table (tile_generic).  The four-slot build sends nearly every tile of both through tile_generic."""
    L = request.getfixturevalue(lib)
    s, gp, m = es.raster_scene(kind, C, 2, 300 + C)
    want, counts, ids_o, _ = es.raster_expected(s, gp, m, oracle, shared=shared)
    gc, ids = _raster(L, s, gp, shared=shared)
    assert (ids.cpu().numpy() == ids_o).all()
    what = '%s %s C=%d shared=%s' % (lib, kind, C, shared)
    _same(gc, want, counts, what)
    assert _bits(_raster(L, s, gp, shared=shared)[0], gc), what + ': a second run differs'


@pytest.mark.parametrize('lib', ['cuda_lib', 'small'])
@pytest.mark.parametrize('shared', [False, True])
@pytest.mark.parametrize('kind', ['large', 'tiny'])
@pytest.mark.parametrize('C', [1, 3, 4])
def test_raster_vertex_colours_deterministic(request, oracle, lib, kind, C, shared):
    L = request.getfixturevalue(lib)
    s, gp, m = es.raster_scene(kind, C, 2, 300 + C)
    want, counts, _, _ = es.raster_expected(s, gp, m, oracle, shared=shared)
    gc, _ = _raster(L, s, gp, deterministic=True, shared=shared)
    _same(gc, want, counts, 'deterministic %s %s C=%d shared=%s' % (lib, kind, C, shared))


# ---- C. trilinear texture at power-of-two footprints ------------------------------------------------------------------

def _trilinear(L, tex, idx, der, gout):
    import dirt_b200 as dirt
    t = (tex if tex.shape[0] > 1 else tex[0]).clone().requires_grad_(True)
    i = idx.clone().requires_grad_(True)
    with _through(L):
        (dirt.sample_texture(t, i, mode='trilinear', derivatives=der) * gout).sum().backward()
    return t.grad.reshape(tex.shape), i.grad


@pytest.mark.parametrize('lib', ['cuda_lib', 'small'])
@pytest.mark.parametrize('per_item', [False, True])
@pytest.mark.parametrize('C', [1, 2, 3, 4, 5])
def test_trilinear_one_level_per_lookup(request, lib, C, per_item):
    """Footprints of 1, 2 and 4 texels: each lookup scatters to level 0, 1 or 2 alone (per-level keys), and the pyramid
    adjoint (mip_collapse) carries levels 1 and 2 down to the texture with its 1/4 per level.  Blended levels are
    covered by the cube map's trilinear lookups below: here lambda comes from log2f and its fraction is not chosen."""
    L = request.getfixturevalue(lib)
    tex, idx, der, gout = es.trilinear_scene(3 if per_item else 1, 64, 32, C, 3, 7001, 400 + C, device=DEV)
    gt_want, gi_want = es.trilinear_expected(tex, idx, der, gout)
    gt, gi = _trilinear(L, tex, idx, der, gout)
    what = '%s trilinear C=%d per_item=%s' % (lib, C, per_item)
    _same(gt, gt_want, None, what + ' grad_texture')
    _same(gi, gi_want, None, what + ' grad_indices')
    gt2, gi2 = _trilinear(L, tex, idx, der, gout)
    assert _bits(gt2, gt) and _bits(gi2, gi), what + ': a second run differs'


# ---- D. cube maps ------------------------------------------------------------------------------------------------------

def _cube(cube, d, lod, gout, mode, deterministic):
    import dirt_b200 as dirt
    c = cube.clone().requires_grad_(True)
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        out = dirt.sample_cubemap(c, d, mode, lod=lod if mode == 'trilinear' else None)
        (out * gout).sum().backward()
    finally:
        torch.use_deterministic_algorithms(before)
    return c.grad


@pytest.mark.parametrize('deterministic', [False, True])
@pytest.mark.parametrize('per_item,N', [(False, 3000), (True, 3000), (True, 100)])
@pytest.mark.parametrize('mode', ['bilinear', 'nearest', 'trilinear'])
@pytest.mark.parametrize('C', [1, 3, 4])
def test_cube_map(cuda_lib, C, mode, per_item, N, deterministic):
    """Lookups across edges and corners (the border texels' adjoint, with its /3 at the corners), trilinear at lods on a
    1/4 grid (exact blend weights); a shared map and per-item maps of 3000 lookups, whose CTAs share one map and take
    the shared-memory accumulation of the coarse levels and its flush, and per-item maps of 100 lookups, whose CTAs
    straddle items and take the global path."""
    cube, d, lod, gout = es.cube_scene(3, C, N, per_item, 500 + C, DEV)
    want = es.cube_expected(cube, d, lod, gout, mode)
    got = _cube(cube, d, lod, gout, mode, deterministic)
    what = 'cube %s C=%d per_item=%s N=%d deterministic=%s' % (mode, C, per_item, N, deterministic)
    _same(got, want, None, what)
    assert _bits(_cube(cube, d, lod, gout, mode, deterministic), got), what + ': a second run differs'


# ---- E. shadow map, default map gradient -------------------------------------------------------------------------------

@pytest.mark.parametrize('per_item', [False, True])
@pytest.mark.parametrize('name', es.SHADOW_CASES)
def test_shadow_map_gradient(cuda_lib, name, per_item):
    """R = 0 and softness 0, the dyadic cases of test_gpu_shadow_edges.py on power-of-two maps: whole warps on one texel
    of a 4 x 4 map, 20 000 points per item sharing one base texel, and piles on a map's corners and edges."""
    p, M, smap, gout = es.shadow_case(name, per_item)
    want, counts = es.shadow_expected(p, M, smap, 0, 0.01, gout)
    got = shadow_call(p, M, smap, 0, 0., gout, (False, False, True))[3]
    _same(torch.from_numpy(got), want, counts, 'shadow %s per_item=%s' % (name, per_item))
    again = shadow_call(p, M, smap, 0, 0., gout, (False, False, True))[3]
    assert np.array_equal(again.view(np.int32), got.view(np.int32)), name
