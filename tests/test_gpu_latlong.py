"""GPU: lat-long panoramas to cube maps (DESIGN.md §7.13) against tests/latlong_restatement.py.

The forward is compared bit for bit with the restatement evaluated in float32 on the GPU; the panorama gradient with
float64 autograd of the restatement at the float32 sample coordinates; the gather's pairs by the dot-product identity
and per element over many shapes."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import rel_close
import cubemap_ggx_restatement as ibl
import latlong_restatement as ll
from test_gpu_cubemap import _bits_equal, _directions, _gen
from test_gpu_cubemap_mip import _coords_of, _off_boundaries
import variant_builds

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)

# (H, W, S): H = 1, W = 1, S = 1, odd S n (a sample on each face's centre: the poles, with signed zeros),
# magnification, strong minification (n = 21) and aspects other than 2:1
SHAPES = [(1, 1, 1), (1, 5, 3), (3, 1, 4), (16, 32, 64), (512, 1024, 16), (33, 50, 9), (20, 36, 7), (9, 30, 5),
          (64, 64, 12)]


def _panorama(H, W, C, seed, batch=None):
    shape = (H, W, C) if batch is None else (batch, H, W, C)
    return torch.rand(shape, generator=_gen(seed), device=DEV) * 2 - 0.5


def _close(actual, expected, name):
    a, b = actual.detach().cpu().numpy(), expected.detach().cpu().numpy()
    if b.size and np.abs(b).max() < 1e-12:
        return bool(np.abs(a).max() < 1e-12), 0.0
    return rel_close(a, b, name=name)


def test_odd_shapes_sample_the_poles():
    for H, W, S in SHAPES:
        if H == 33:
            assert (S * ll.samples(H, W, S)) % 2 == 1
    assert ll.samples(512, 1024, 16) == 21


@pytest.mark.parametrize('C', [1, 2, 3, 4, 5, 8])
def test_forward_is_the_restatement_bit_for_bit(cuda_lib, C):
    import dirt_b200 as dirt
    for k, (H, W, S) in enumerate(SHAPES):
        pan = _panorama(H, W, C, 10 * k + C)
        assert _bits_equal(dirt.latlong_to_cubemap(pan, S), ll.to_cubemap(pan, S)), (H, W, S, C)
        pans = _panorama(H, W, C, 10 * k + C + 100, batch=2)
        assert _bits_equal(dirt.latlong_to_cubemap(pans, S), ll.to_cubemap(pans, S)), (H, W, S, C, 'items')
    if C in (2, 4):
        # rows 4 bytes off their vector alignment: the scalar path
        H, W, S = 20, 36, 7
        buf = _panorama(H * W * C + 1, 1, 1, 300 + C).reshape(-1)
        pan = buf[1:].reshape(H, W, C)
        assert pan.data_ptr() % 8 == 4
        assert _bits_equal(dirt.latlong_to_cubemap(pan, S), ll.to_cubemap(pan, S)), C


def _gpu_grad(pan, S, g):
    import dirt_b200 as dirt
    p = pan.detach().clone().requires_grad_(True)
    (gp,) = torch.autograd.grad((dirt.latlong_to_cubemap(p, S) * g).sum(), p)
    return gp


def _reference_grad(pan, S, g):
    """float64 autograd of the restatement at the float32 sample coordinates (computed on the GPU)."""
    p = pan.detach().double().requires_grad_(True)
    (gp,) = torch.autograd.grad((ll.to_cubemap(p, S) * g.double()).sum(), p)
    return gp


@pytest.mark.parametrize('C', [1, 3, 5])
def test_gradient_matches_float64_autograd(cuda_lib, C):
    worst = 0.
    for k, (H, W, S) in enumerate(SHAPES):
        for batch in (None, 2):
            pan = _panorama(H, W, C, 20 * k + C, batch)
            g = torch.randn(((batch,) if batch else ()) + (6, S, S, C), generator=_gen(20 * k + C + 1), device=DEV)
            ok, ratio = _close(_gpu_grad(pan, S, g), _reference_grad(pan, S, g), 'latlong grad_panorama')
            worst = max(worst, ratio)
            assert ok, (H, W, S, C, batch, ratio)
    print('latlong grad_panorama: worst error / tolerance %.3f' % worst)


def _dot_shapes():
    rng = np.random.default_rng(7)
    shapes = [(1, 1, 1), (1, 1, 6), (2, 2, 9), (1, 64, 8), (64, 1, 8), (2, 3, 1), (5, 7, 2), (17, 300, 4),
              (100, 37, 11), (128, 256, 32), (256, 512, 8), (7, 1000, 5), (1000, 7, 5)]
    for _ in range(24):
        H, W = int(rng.integers(1, 200)), int(rng.integers(1, 400))
        shapes.append((H, W, int(rng.integers(1, 40))))
    return shapes


def test_gather_pairs_by_the_dot_product_identity(cuda_lib):
    """<A p, g> = <p, A^T g> in float64 accumulation, and A^T g per element against autograd of the restatement: a
    pair the candidate boxes missed or counted twice shows in both."""
    import dirt_b200 as dirt
    worst_dot, worst_el = 0., 0.
    for k, (H, W, S) in enumerate(_dot_shapes()):
        pan = _panorama(H, W, 2, 400 + k)
        g = torch.randn(6, S, S, 2, generator=_gen(500 + k), device=DEV)
        out = dirt.latlong_to_cubemap(pan, S)
        gp = _gpu_grad(pan, S, g)
        lhs, rhs = (out.double() * g.double()).sum(), (pan.double() * gp.double()).sum()
        scale = float((out.double() * g.double()).abs().sum())
        worst_dot = max(worst_dot, abs(float(lhs - rhs)) / scale)
        assert abs(float(lhs - rhs)) <= 1e-5 * scale, (H, W, S, float(lhs), float(rhs))
        ok, ratio = _close(gp, _reference_grad(pan, S, g), 'latlong grad_panorama (dot shapes)')
        worst_el = max(worst_el, ratio)
        assert ok, (H, W, S, ratio)
    print('latlong dot-product identity: worst |lhs - rhs| / sum |terms| %.2e; worst element ratio %.3f'
          % (worst_dot, worst_el))


def test_backward_is_reproducible(cuda_lib):
    H, W, S, C = 96, 160, 24, 3
    pan = _panorama(H, W, C, 600)
    g = torch.randn(6, S, S, C, generator=_gen(601), device=DEV)
    a, b = _gpu_grad(pan, S, g), _gpu_grad(pan, S, g)
    assert _bits_equal(a, b)
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        c = _gpu_grad(pan, S, g)
    finally:
        torch.use_deterministic_algorithms(before)
    assert _bits_equal(a, c)
    # a shared panorama gives the bits of one item of a batch, forward and backward
    import dirt_b200 as dirt
    pans = torch.stack([_panorama(H, W, C, 602), pan, _panorama(H, W, C, 603)])
    gs = torch.stack([torch.randn(6, S, S, C, generator=_gen(604), device=DEV), g,
                      torch.randn(6, S, S, C, generator=_gen(605), device=DEV)])
    assert _bits_equal(dirt.latlong_to_cubemap(pans, S)[1], dirt.latlong_to_cubemap(pan, S))
    assert _bits_equal(_gpu_grad(pans, S, gs)[1], a)


def _run_abi(L, pans, S, g):
    from dirt_b200 import _lib
    TB, H, W, C = pans.shape
    out = torch.empty(TB, 6, S, S, C, device=DEV)
    gp = torch.empty_like(pans)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    stream = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    with torch.cuda.device(DEV):
        _lib.check(L.dirt_latlong_to_cubemap(p(pans), p(out), TB, H, W, S, C, stream), 'forward')
        _lib.check(L.dirt_latlong_to_cubemap_backward(p(g), p(gp), TB, H, W, S, C, stream), 'backward')
    torch.cuda.synchronize()
    return out, gp


def test_small_grid_variant(cuda_lib, tmp_path_factory):
    """A build whose conversion kernels run on 3 CTAs and 2 items per grid: the same bits as the product build."""
    small = variant_builds._variant(tmp_path_factory, 'latlong_small_grid',
                                    {'DIRT_LATLONG_MAX_BLOCKS': 3, 'DIRT_LATLONG_MAX_ITEMS': 2})
    for (H, W, S, C, B) in ((40, 72, 11, 3, 5), (33, 50, 9, 5, 3), (16, 32, 20, 4, 1)):
        pans = _panorama(H, W, C, 700 + C, batch=B).contiguous()
        g = torch.randn(B, 6, S, S, C, generator=_gen(701 + C), device=DEV)
        a, b = _run_abi(cuda_lib, pans, S, g), _run_abi(small, pans, S, g)
        assert _bits_equal(a[0], b[0]) and _bits_equal(a[1], b[1]), (H, W, S, C, B)
        assert small.dirt_last_launch_count() == (C + 3) // 4


def test_sh_panorama_round_trip(cuda_lib):
    """The order-2 SH coefficients of a panorama built from them come back through the conversion and
    cubemap_spherical_harmonics: the orientation end to end."""
    import dirt_b200 as dirt
    from dirt_b200 import lighting
    H, W, S = 128, 256, 64
    coeffs = torch.rand(9, 3, generator=_gen(800), device=DEV) * 2 - 1
    d = dirt.latlong_directions(H, W, device=DEV).double()
    pan = (lighting._sh_basis(d) @ coeffs.double()).float()
    got = lighting.cubemap_spherical_harmonics(dirt.latlong_to_cubemap(pan, S))
    err = float((got - coeffs).abs().max())
    print('latlong SH round trip 128 x 256 -> 64: worst coefficient error %.2e' % err)
    assert err < 1e-3


def test_a_bright_texel_lands_where_its_direction_points(cuda_lib):
    import dirt_b200 as dirt
    H, W, S = 32, 64, 32
    d = dirt.latlong_directions(H, W, device=DEV)
    for r, c in ((10, 20), (16, 47), (5, 0), (25, 63)):
        pan = torch.zeros(H, W, 1, device=DEV)
        pan[r, c] = 1.
        back = dirt.sample_cubemap(dirt.latlong_to_cubemap(pan, S), d)[..., 0]
        assert int(back.argmax()) == r * W + c, (r, c, divmod(int(back.argmax()), W))


def test_composition_with_ggx_and_sh(cuda_lib):
    """Gradients through latlong_to_cubemap -> sample_cubemap('ggx') and -> cubemap_spherical_harmonics are finite
    and match the composed float64 restatements."""
    import dirt_b200 as dirt
    from dirt_b200 import lighting
    H, W, S, C = 24, 48, 16, 3
    pan = _panorama(H, W, C, 900)
    d = _directions(1500, 901, S)
    r = torch.rand(d.shape[0], generator=_gen(902), device=DEV)
    gout = torch.randn(d.shape[0], C, generator=_gen(903), device=DEV) * _off_boundaries(d, S)[:, None]
    gsh = torch.randn(9, C, generator=_gen(904), device=DEV)

    p = pan.detach().clone().requires_grad_(True)
    cube = dirt.latlong_to_cubemap(p, S)
    loss = (dirt.sample_cubemap(cube, d, 'ggx', roughness=r) * gout).sum() + \
        (lighting.cubemap_spherical_harmonics(cube) * gsh).sum()
    (got,) = torch.autograd.grad(loss, p)
    assert bool(torch.isfinite(got).all())

    q = pan.detach().double().requires_grad_(True)
    cube64 = ll.to_cubemap(q, S).cpu()
    x32 = d.detach().float().cpu()
    ref = (ibl.sample(cube64, d.detach().double().cpu(), r.detach().double().cpu(), _coords_of(x32)) *
           gout.double().cpu()).sum() + (ibl.sh_project(cube64) * gsh.double().cpu()).sum()
    (want,) = torch.autograd.grad(ref, q)
    ok, ratio = _close(got, want, 'latlong -> ggx / SH grad_panorama')
    assert ok, ratio
