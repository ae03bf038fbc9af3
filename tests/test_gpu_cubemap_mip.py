"""GPU: dirt_b200.sample_cubemap(..., mode='trilinear', lod=...) against the torch restatement of
tests/cubemap_mip_restatement.py.

Forward values are compared bit for bit with the float32 restatement on the same device; gradients against torch
autograd of the restatement in float64, with conftest.rel_close (1e-4 relative), evaluated at each level's float32
lookup as tests/test_gpu_cubemap.py does for one level."""
import ctypes
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

import cubemap_mip_restatement as cmm
import cubemap_mip_variants
import cubemap_restatement as cm
import variant_builds
from conftest import rel_close
from test_gpu_cubemap import _bits_equal, _cubemap, _directions, _gen

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device('cuda', 0)

SIZES = [1, 2, 3, 6, 64]   # L = 1, 2, 1, 2, 7


def _lods(n, L, seed):
    """n levels of detail uniform in [-2, L+2], then the integers -1 .. L, +-inf and NaN, repeated to n."""
    g = _gen(seed)
    lod = torch.rand(n, generator=g, device=DEV) * (L + 4) - 2
    special = torch.tensor([float(k) for k in range(-1, L + 1)] + [math.inf, -math.inf, math.nan, -0.0, 0.5],
                           device=DEV)
    idx = torch.randperm(n, generator=g, device=DEV)[:n // 4]
    lod[idx] = special[torch.arange(idx.numel(), device=DEV) % special.numel()]
    return lod


@pytest.mark.parametrize('C', [1, 2, 3, 4, 5, 8])
def test_forward_is_bit_identical_to_the_restatement(cuda_lib, C):
    import dirt_b200 as dirt
    for k, S in enumerate(SIZES):
        L = cmm.level_count(S)
        cube = _cubemap(S, C, k)
        d = _directions(5000, 100 + k, S)
        lod = _lods(d.shape[0], L, 150 + k)
        assert _bits_equal(dirt.sample_cubemap(cube, d, 'trilinear', lod=lod), cmm.sample(cube, d, lod)), (S, C)
        cubes = _cubemap(S, C, 10 + k, batch=3)
        d = torch.stack([_directions(1000, 200 + k + b, S) for b in range(3)])
        lod = _lods(d.shape[0] * d.shape[1], L, 250 + k).reshape(d.shape[:-1])
        assert _bits_equal(dirt.sample_cubemap(cubes, d, 'trilinear', lod=lod), cmm.sample(cubes, d, lod)), (S, C, 'items')


def test_lod_at_or_below_zero_is_bilinear_and_integers_are_levels(cuda_lib):
    import dirt_b200 as dirt
    for k, S in enumerate(SIZES):
        cube, d = _cubemap(S, 3, 30 + k), _directions(4000, 40 + k, S)
        bil = dirt.sample_cubemap(cube, d, 'bilinear')
        for lod in (0., -0., -1.5, -math.inf, math.nan):
            assert _bits_equal(dirt.sample_cubemap(cube, d, 'trilinear', lod=lod), bil), (S, lod)
        for level in range(cmm.level_count(S)):
            assert _bits_equal(dirt.sample_cubemap(cube, d, 'trilinear', lod=float(level)),
                               cmm.level_lookup(cube, d, level)), (S, level)


def _coords_of(x32):
    """coords_of for cubemap_mip_restatement.sample in float64: s and t moved onto level k's float32 padded (row, col),
    with the float64 derivative (tests/test_gpu_cubemap.py's _reference_coords, per level)."""
    def coords(x64, k, S):
        face, s, t, valid = cm.face_coords(x64)
        _, s32, t32, _ = cm.face_coords(x32)
        s_val = (((s32 * S - 0.5) + 1.).double() - 0.5) / S
        t_val = (((t32 * S - 0.5) + 1.).double() - 0.5) / S
        return face, s + (s_val - s).detach(), t + (t_val - t).detach(), valid
    return coords


def _off_boundaries(d, S):
    """Lookups whose float32 padded coordinates are off texel boundaries at every level: there the bilinear derivative
    jumps, and the float64 evaluation may take the other side."""
    with torch.no_grad():
        _, s32, t32, _ = cm.face_coords(d.float())
        ok = torch.ones_like(s32, dtype=torch.bool)
        for k in range(cmm.level_count(S)):
            Sk = S >> k
            pr, pc = (t32 * Sk - 0.5) + 1., (s32 * Sk - 0.5) + 1.
            ok &= (pr != pr.floor()) & (pc != pc.floor())
    return ok


def _reference_grads(cube, d, lod, grad_out):
    c = cube.detach().double().requires_grad_(True)
    x = d.detach().double().requires_grad_(True)
    lo = lod.detach().double().requires_grad_(True)

    def run(c, x, lo, x32):
        if c.dim() == 5:
            return torch.stack([run(c[b], x[b], lo[b], x32[b]) for b in range(c.shape[0])])
        return cmm.sample(c, x, lo, _coords_of(x32))

    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(False)
    try:
        (run(c, x, lo, d.detach().float()) * grad_out.double()).sum().backward()
    finally:
        torch.use_deterministic_algorithms(before)
    return c.grad, (x.grad if x.grad is not None else torch.zeros_like(x)), lo.grad


def _close(actual, expected, name):
    a, b = actual.cpu().numpy(), expected.cpu().numpy()
    if b.size and np.abs(b).max() < 1e-12:
        return bool(np.abs(a).max() < 1e-12), 0.0
    return rel_close(a, b, name=name)


def _check_grads(cube, d, lod, seed, tag, label='cubemap mip'):
    import dirt_b200 as dirt
    grad_out = torch.randn(d.shape[:-1] + (cube.shape[-1],), generator=_gen(seed), device=DEV)
    same = _off_boundaries(d, cube.shape[-2])
    assert float(same.float().mean()) > 0.9, tag
    grad_out = grad_out * same[..., None]
    c = cube.detach().clone().requires_grad_(True)
    x = d.detach().clone().requires_grad_(True)
    lo = lod.detach().clone().requires_grad_(True)
    (dirt.sample_cubemap(c, x, 'trilinear', lod=lo) * grad_out).sum().backward()
    ref_c, ref_x, ref_l = _reference_grads(cube, d, lod, grad_out)
    for name, got, want in (('grad_cubemap', c.grad, ref_c), ('grad_directions', x.grad, ref_x), ('grad_lod', lo.grad, ref_l)):
        ok, ratio = _close(got, want, label + ' ' + name)
        assert ok, (tag, name, ratio)
    return c.grad, x.grad, lo.grad


@pytest.mark.parametrize('C', [1, 3, 4, 5])
def test_backward_matches_autograd_of_the_restatement(cuda_lib, C):
    for k, S in enumerate(SIZES):
        L = cmm.level_count(S)
        d = _directions(5000, 300 + k, S)
        _check_grads(_cubemap(S, C, 20 + k), d, _lods(d.shape[0], L, 350 + k), 400 + k, (S, C))
        d = torch.stack([_directions(3000, 500 + k + b, S) for b in range(2)])
        _check_grads(_cubemap(S, C, 30 + k, batch=2), d, _lods(d.shape[0] * d.shape[1], L, 550 + k).reshape(d.shape[:-1]),
                     600 + k, (S, C, 'per item'))


@pytest.fixture
def deterministic():
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(before)


@pytest.mark.parametrize('C', [1, 3, 4, 5])
def test_deterministic_gradient(cuda_lib, deterministic, C):
    """Within the bar of float64 autograd, bit-identical on a repeat, and with per-item maps an item alone gives the
    same bits as inside the batch."""
    import dirt_b200 as dirt
    for k, S in enumerate([1, 6, 64]):
        L = cmm.level_count(S)
        cube, d = _cubemap(S, C, 50 + k), _directions(20000, 51 + k, S)
        lod = _lods(d.shape[0], L, 70 + k)
        g1 = _check_grads(cube, d, lod, 52 + k, (S, C, 'det'), label='cubemap mip deterministic')
        g2 = _check_grads(cube, d, lod, 52 + k, (S, C, 'det'), label='cubemap mip deterministic')
        assert all(_bits_equal(a, b) for a, b in zip(g1, g2))
    cubes = _cubemap(16, C, 58, batch=3)
    d = torch.stack([_directions(3000, 59 + b, 16) for b in range(3)])
    lod = _lods(3 * d.shape[1], 5, 61).reshape(3, -1)
    gout = torch.randn(3, d.shape[1], C, generator=_gen(60), device=DEV)

    def grad(c, x, lo, g):
        c = c.clone().requires_grad_(True)
        (dirt.sample_cubemap(c, x, 'trilinear', lod=lo) * g).sum().backward()
        return c.grad

    whole = grad(cubes, d, lod, gout)
    for b in range(3):
        assert _bits_equal(grad(cubes[b:b + 1], d[b:b + 1], lod[b:b + 1], gout[b:b + 1])[0], whole[b]), b


def _abi(L, fn, *args):
    return getattr(L, fn)(*[ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else
                            (ctypes.c_void_p(0) if a is None else a) for a in args],
                          ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))


def _run_abi(L, cube, d, lod, gout, det):
    """out, grad_cubemap, grad_directions, grad_lod of one library build, through the C ABI (shared map)."""
    S, C, N = cube.shape[-2], cube.shape[-1], d.shape[0]
    atlas = torch.empty(int(L.dirt_cubemap_mip_atlas_bytes(1, S, C)) // 4, device=DEV)
    out = torch.empty(N, C, device=DEV)
    assert _abi(L, 'dirt_cubemap_sample_trilinear', cube, d, lod, atlas, out, 1, S, C, 1, N) == 0
    nbytes = int(L.dirt_cubemap_sample_trilinear_backward_bytes(1, S, C, 1, N, det))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    gc, gd, gl = torch.empty_like(cube), torch.empty_like(d), torch.empty_like(lod)
    assert _abi(L, 'dirt_cubemap_sample_trilinear_backward', atlas, d, lod, gout, gc, gd, gl, 1, S, C, 1, N, det, scratch,
                ctypes.c_size_t(nbytes)) == 0
    torch.cuda.synchronize()
    return out, gc, gd, gl


def test_coarse_levels_with_and_without_shared_memory(cuda_lib, tmp_path_factory):
    """2^22 lookups on the top two levels of a 6 x 64^2 map, the case the shared-memory accumulation serves: the product
    build, the build without it and the deterministic path agree."""
    S, C = 64, 3
    L = cmm.level_count(S)
    cube = _cubemap(S, C, 80)
    d = torch.randn(1 << 22, 3, generator=_gen(81), device=DEV)
    lod = torch.rand(1 << 22, generator=_gen(82), device=DEV) + (L - 2)
    # positive, so that the ~10^5 terms per coarse texel do not cancel and fp32 sums stay within the bar
    gout = torch.rand(1 << 22, C, generator=_gen(83), device=DEV) + 0.5
    product = _run_abi(cuda_lib, cube, d, lod, gout, 0)
    plain = _run_abi(cubemap_mip_variants.no_smem_library(tmp_path_factory), cube, d, lod, gout, 0)
    det = _run_abi(cuda_lib, cube, d, lod, gout, 1)
    assert _bits_equal(product[0], plain[0]) and _bits_equal(product[0], det[0])
    for other in (plain, det):
        assert _bits_equal(product[2], other[2]) and _bits_equal(product[3], other[3])
        ok, ratio = rel_close(product[1].cpu().numpy(), other[1].cpu().numpy(), name='cubemap mip coarse levels')
        assert ok, ratio


def test_small_grid_variant(cuda_lib, tmp_path_factory):
    """The small-grid build runs every loop for many rounds: the same forward bits and deterministic gradient."""
    small = variant_builds.small_grid_library(tmp_path_factory)
    S, C = 16, 3
    cube = _cubemap(S, C, 90)
    d = _directions(7000, 91, S)
    lod = _lods(d.shape[0], cmm.level_count(S), 92)
    gout = torch.randn(d.shape[0], C, generator=_gen(93), device=DEV)
    a, b = _run_abi(cuda_lib, cube, d, lod, gout, 1), _run_abi(small, cube, d, lod, gout, 1)
    assert all(_bits_equal(x, y) for x, y in zip(a, b))
    assert _bits_equal(a[0], cmm.sample(cube, d, lod))


def test_no_lookups_and_broadcast_lod(cuda_lib):
    import dirt_b200 as dirt
    cube = torch.rand(6, 4, 4, 3, device=DEV, requires_grad=True)
    d = torch.zeros(0, 3, device=DEV, requires_grad=True)
    out = dirt.sample_cubemap(cube, d, 'trilinear', lod=1.)
    assert out.shape == (0, 3)
    out.sum().backward()
    assert cube.grad is not None and not cube.grad.any()
    # one lod per item of per-item maps, broadcast over the item's lookups: its gradient is the sum over them
    cubes = _cubemap(8, 2, 95, batch=2)
    d = torch.randn(2, 10, 50, 3, generator=_gen(96), device=DEV)
    lod = torch.tensor([0.7, 2.3], device=DEV, requires_grad=True)
    out = dirt.sample_cubemap(cubes, d, 'trilinear', lod=lod[:, None, None])
    gout = torch.randn(out.shape, generator=_gen(97), device=DEV)
    (out * gout).sum().backward()
    full = lod.detach()[:, None, None].expand(2, 10, 50).clone().requires_grad_(True)
    (dirt.sample_cubemap(cubes, d, 'trilinear', lod=full) * gout).sum().backward()
    assert torch.allclose(lod.grad, full.grad.sum((1, 2)), rtol=1e-5, atol=1e-5)


# ---- through the deferred rasteriser ---------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def glossy(cuda_lib):
    spec = importlib.util.spec_from_file_location('glossy_example', os.path.join(ROOT, 'examples', 'glossy.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_glossy_through_rasterise_batch_deferred(glossy):
    import dirt_b200 as dirt
    B = 2
    cube = glossy.env.procedural_cubemap(32, device=DEV).expand(B, -1, -1, -1, -1).contiguous().requires_grad_(True)
    roughness = torch.tensor([0.3, 0.7], device=DEV, requires_grad=True)
    pixels = glossy.render(cube, roughness, dirt.rasterise_batch_deferred, dirt.sample_cubemap, batch=B, width=160,
                           height=120, device=DEV)
    (pixels * torch.rand(pixels.shape, generator=_gen(98), device=DEV)).sum().backward()
    assert torch.isfinite(pixels).all() and torch.isfinite(cube.grad).all() and torch.isfinite(roughness.grad).all()
    assert bool((roughness.grad != 0).all())
    ref = glossy.render(cube.detach(), roughness.detach(), dirt.rasterise_batch_deferred,
                        lambda c, x, mode, lod=None: (
                            cmm.sample(c, x, torch.as_tensor(lod, dtype=torch.float32, device=DEV).expand(x.shape[:-1]))
                            if mode == 'trilinear' else cm.sample(c, x, mode)),
                        batch=B, width=160, height=120, device=DEV)
    assert _bits_equal(pixels.detach(), ref)


def test_fitting_the_roughness_through_the_rasteriser(glossy):
    """Per-item roughness (so lod) fitted with Adam from a wrong start: at least 10x closer to the truth at the end."""
    import dirt_b200 as dirt
    B = 2
    cube = glossy.env.procedural_cubemap(32, device=DEV).expand(B, -1, -1, -1, -1).contiguous()
    truth, start = torch.tensor([0.35, 0.6], device=DEV), torch.tensor([0.8, 0.15], device=DEV)
    path = glossy.fit_roughness(cube, truth, start, dirt.rasterise_batch_deferred, dirt.sample_cubemap)
    before, after = (start - truth).abs(), (path[-1] - truth).abs()
    print('roughness fit: |error| %s -> %s' % (before.tolist(), after.tolist()))
    assert bool((after * 10 <= before).all()), path[::15].tolist()
