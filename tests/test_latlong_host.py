"""CPU: the lat-long to cube-map conversion's restatement (tests/latlong_restatement.py) -- orientation, seams and
poles, the sample count, the SH round trip -- and the C ABI's and latlong_to_cubemap's argument errors."""
import ctypes
import math

import numpy as np
import pytest
import torch

import cubemap_ggx_restatement as ibl
import latlong_restatement as ll


def _directions(H, W):
    from dirt_b200 import texture
    return texture.latlong_directions(H, W).double()


def _convert(pan, S):
    """The conversion in float64, coordinates included."""
    return ll.to_cubemap(pan, S, coord_dtype=torch.float64)


def test_latlong_directions_follow_the_convention():
    H, W = 8, 16
    d = _directions(H, W)
    assert torch.allclose(d.norm(dim=-1), torch.ones(H, W, dtype=torch.float64), atol=1e-7)
    # row 0 next to +Y, row H-1 next to -Y
    assert bool((d[0, :, 1] > 0.98).all()) and bool((d[-1, :, 1] < -0.98).all())
    # the centre columns straddle -Z; column index increases towards +X
    eq = d[H // 2]
    assert float(eq[W // 2, 2]) < -0.9 and float(eq[W // 2 - 1, 2]) < -0.9
    assert float(eq[W // 2, 0]) > 0 > float(eq[W // 2 - 1, 0])
    assert float(eq[3 * W // 4, 0]) > 0.9 and float(eq[W // 4, 0]) < -0.9
    # the seam phi = +-pi faces +Z
    assert float(eq[0, 2]) > 0.9 and float(eq[-1, 2]) > 0.9


def _face_centre(cube, f):
    S = cube.shape[1]
    return cube[f, S // 2 - 1:S // 2 + 1, S // 2 - 1:S // 2 + 1].mean()


def test_rows_and_columns_land_on_the_right_faces():
    H, W, S = 16, 33, 8
    # rows 0 and 1 hold the zenith: +Y's centre reads only them, -Y does not read them
    pan = torch.zeros(H, W, 1, dtype=torch.float64)
    pan[:2] = 1.
    cube = _convert(pan, S)
    assert abs(float(_face_centre(cube, 2)) - 1.) < 1e-12 and float(cube[3].abs().max()) == 0.
    # the centre column (phi = 0, W odd) is -Z's centre column
    pan = torch.zeros(H, W, 1, dtype=torch.float64)
    pan[:, W // 2] = 1.
    cube = _convert(pan, S)
    assert float(cube[5, S // 2, S // 2 - 1:S // 2 + 1].min()) > 0.25 and float(cube[4].abs().max()) == 0.
    # phi = pi / 2 is +X and -pi / 2 is -X: to the right of -Z and to its left
    for c, f in ((3 * W // 4, 0), (W // 4, 1)):
        pan = torch.zeros(H, W, 1, dtype=torch.float64)
        pan[:, c] = 1.
        cube = _convert(pan, S)
        assert float(_face_centre(cube, f)) > 0.2 and float(cube[1 - f].abs().max()) == 0., (c, f)
    # +X is to the right of -Z seen from inside: on -Z's face (sc = -x) the right-hand column is the one nearer +X
    pan = torch.zeros(H, W, 1, dtype=torch.float64)
    pan[:, W // 2 + 2:W // 2 + 5] = 1.
    cube = _convert(pan, S)
    assert float(cube[5, :, 0].sum()) > 0 and float(cube[5, :, -1].sum()) == 0.


@pytest.mark.parametrize('H, W, S', [(16, 32, 8), (32, 64, 16), (24, 40, 12)])
def test_a_smooth_panorama_has_no_seam_or_pole_jump(H, W, S):
    """A panorama of a smooth function of the direction converts to that function, within the interpolation error,
    on every face: across the phi = +-pi seam (face +Z) and at the poles (faces +-Y) as well."""
    a = torch.tensor([0.3, 0.8, -0.5], dtype=torch.float64)
    f = lambda d: 1. + d @ a + 0.5 * d[..., 0] * d[..., 2]
    cube = _convert(f(_directions(H, W))[..., None], S)
    x, y, z = ll.sample_directions(S, 1, 0, 0, torch.float64)
    d = torch.stack([x, y, z], -1)
    d = d / d.norm(dim=-1, keepdim=True)
    err = (cube[..., 0] - f(d)).abs()
    bound = 3.0 * (math.pi / H) ** 2 + 2.0 * (2 * math.pi / W) / S   # interpolation, and the texel's own extent
    assert float(err.max()) < bound, (float(err.max()), bound)
    # the seam: +Z's centre column pairs straddle phi = +-pi
    assert float((cube[4, :, S // 2 - 1] - cube[4, :, S // 2]).abs().max()) < 4 * (2 * math.pi / S)


def test_sh_round_trip():
    """A panorama of order-2 SH radiance, converted and projected through the texel solid angles of DESIGN.md §7.12,
    gives back its coefficients (float64 throughout)."""
    from dirt_b200 import lighting
    H, W, S = 128, 256, 64
    coeffs = torch.from_numpy(np.random.default_rng(3).uniform(-1., 1., (9, 2)))
    pan = lighting._sh_basis(_directions(H, W)) @ coeffs
    got = ibl.sh_project(_convert(pan, S))
    assert float((got - coeffs).abs().max()) < 1e-3, float((got - coeffs).abs().max())


def test_float32_restatement_is_close_to_float64():
    H, W, S = 20, 36, 6
    pan = torch.from_numpy(np.random.default_rng(4).random((H, W, 2)))
    a = ll.to_cubemap(pan.float(), S)
    b = _convert(pan, S)
    assert a.dtype == torch.float32 and float((a.double() - b).abs().max()) < 1e-5


def test_gradient_is_the_adjoint():
    """Autograd of the restatement is linear in the panorama, and the dot-product identity holds."""
    H, W, S = 6, 10, 3
    rng = np.random.default_rng(5)
    p = torch.from_numpy(rng.random((H, W, 2))).requires_grad_(True)
    g = torch.from_numpy(rng.standard_normal((6, S, S, 2)))
    out = ll.to_cubemap(p, S)
    (gp,) = torch.autograd.grad((out * g).sum(), p)
    assert abs(float((out * g).sum().detach() - (p * gp).sum().detach())) < 1e-12


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_sample_count_is_the_formula(L):
    for H in (1, 2, 3, 7, 16, 100, 512, 1024, 2048, 8192):
        for W in (1, 2, 5, 16, 33, 1024, 2048, 4096, 16384):
            for S in (1, 2, 3, 16, 64, 256, 512, 1024, 4096):
                assert L.dirt_latlong_samples(H, W, S) == ll.samples(H, W, S), (H, W, S)
    assert ll.samples(1024, 2048, 512) == 2 and ll.samples(1024, 2048, 256) == 3
    assert ll.samples(8192, 16384, 1024) == 6 and ll.samples(512, 1024, 16) == 21
    assert ll.samples(1, 1, 1) == 1 and ll.samples(16, 32, 64) == 1
    assert L.dirt_latlong_samples(0, 4, 4) == 0 and L.dirt_latlong_samples(4, 0, 4) == 0
    assert L.dirt_latlong_samples(4, 4, 0) == 0


def _p(x):
    return ctypes.c_void_p(x)


def test_latlong_abi_rejects_bad_shapes(L):
    from dirt_b200 import _lib
    buf = _p(4096)   # never dereferenced: every call below fails validation first
    for call in (L.dirt_latlong_to_cubemap, L.dirt_latlong_to_cubemap_backward):
        bad = lambda TB, H, W, S, C: call(buf, buf, TB, H, W, S, C, None)
        assert bad(-1, 4, 8, 4, 3) == _lib.ERR_BAD_SHAPE              # TB < 0
        assert bad(1, 0, 8, 4, 3) == _lib.ERR_BAD_SHAPE               # H = 0
        assert bad(1, 4, 0, 4, 3) == _lib.ERR_BAD_SHAPE               # W = 0
        assert bad(1, 4, 8, 0, 3) == _lib.ERR_BAD_SHAPE               # S = 0
        assert bad(1, 4, 8, 4, 0) == _lib.ERR_BAD_SHAPE               # C = 0
        assert bad(1, 4, 8, (1 << 14) + 1, 3) == _lib.ERR_BAD_SHAPE   # S past 2^14
        assert bad(1, (1 << 20) + 1, 8, 4096, 3) == _lib.ERR_BAD_SHAPE  # H past 2^20
        assert bad(1, 8, (1 << 20) + 1, 4096, 3) == _lib.ERR_BAD_SHAPE  # W past 2^20
        assert bad(1, 8192, 16384, 1, 3) == _lib.ERR_BAD_SHAPE        # n = 5216 past 4096
        assert bad(1 << 30, 1 << 16, 1 << 16, 4096, 8) == _lib.ERR_BAD_SHAPE   # panorama elements past 2^62
        assert L.dirt_last_launch_count() == 0


def test_latlong_abi_with_no_items_launches_nothing(L):
    null = _p(0)
    assert L.dirt_latlong_to_cubemap(null, null, 0, 4, 8, 4, 3, None) == 0
    assert L.dirt_latlong_to_cubemap_backward(null, null, 0, 4, 8, 4, 3, None) == 0
    assert L.dirt_last_launch_count() == 0


def test_latlong_abi_rejects_null_and_misaligned_pointers(L):
    from dirt_b200 import _lib
    null, ok, odd = _p(0), _p(4096), _p(4098)
    for call in (L.dirt_latlong_to_cubemap, L.dirt_latlong_to_cubemap_backward):
        for k in range(2):
            args = [ok, ok]
            args[k] = null
            assert call(*args, 1, 4, 8, 4, 3, None) == _lib.ERR_NULL_POINTER, k
            args[k] = odd
            assert call(*args, 1, 4, 8, 4, 3, None) == _lib.ERR_MISALIGNED, k
        assert L.dirt_last_launch_count() == 0


def test_latlong_to_cubemap_argument_errors():
    import dirt_b200 as dirt
    pan = torch.zeros(4, 8, 3)
    with pytest.raises(ValueError, match=r'\[height, width, channels\]'):
        dirt.latlong_to_cubemap(torch.zeros(8, 3), 4)
    with pytest.raises(ValueError, match=r'\[height, width, channels\]'):
        dirt.latlong_to_cubemap(torch.zeros(1, 2, 4, 8, 3), 4)
    with pytest.raises(ValueError, match='positive'):
        dirt.latlong_to_cubemap(torch.zeros(0, 8, 3), 4)
    with pytest.raises(ValueError, match='positive'):
        dirt.latlong_to_cubemap(torch.zeros(4, 8, 0), 4)
    for size in (0, -2, 2.5):
        with pytest.raises(ValueError, match='size'):
            dirt.latlong_to_cubemap(pan, size)
    with pytest.raises(ValueError, match='height and width'):
        dirt.latlong_directions(0, 8)
    if not torch.cuda.is_available():
        # no CPU kernel: CPU tensors are an error, never a fallback
        with pytest.raises(RuntimeError, match='CUDA'):
            dirt.latlong_to_cubemap(pan, 4)
