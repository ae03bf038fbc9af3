"""CPU: the mipmapped cube-map lookup's restatement (tests/cubemap_mip_restatement.py) in float64 -- its pyramid, its
level of detail and seams at every level, its gradients -- and the C ABI's and sample_cubemap's argument errors."""
import ctypes
import itertools
import math

import numpy as np
import pytest
import torch

import cubemap_mip_restatement as cmm
import cubemap_restatement as cm
import texture_mip_restatement as tm


def _cube(S, C=3, seed=0):
    return torch.from_numpy(np.random.default_rng(seed).random((6, S, S, C)))


def _dirs(n, seed):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal((n, 3)))


def test_pyramid_is_the_texture_pyramid_of_the_faces():
    for S in (1, 3, 8, 12):
        cube = _cube(S, 2, seed=S).float()
        got, want = cmm.pyramid(cube), tm.pyramid(cube)
        assert len(got) == cmm.level_count(S) == tm.level_count(S, S)
        for a, b in zip(got, want):
            assert a.shape[:1] == (6,) and torch.equal(a, b)
        # each face's pyramid alone gives the same levels
        for f in range(6):
            for a, b in zip(got, tm.pyramid(cube[f])):
                assert torch.equal(a[f], b)


@pytest.mark.parametrize('S', [1, 2, 3, 8])
def test_lod_at_or_below_zero_nan_and_one_level_are_bilinear(S):
    cube, d = _cube(S, 3, seed=S), _dirs(600, S)
    bil = cm.sample(cube, d)
    for lod in (0., -0., -0.7, -math.inf, math.nan):
        assert torch.equal(cmm.sample(cube, d, torch.full((600,), lod, dtype=torch.float64)), bil), lod
    if cmm.level_count(S) == 1:
        for lod in (0.5, 3., math.inf):
            assert torch.equal(cmm.sample(cube, d, torch.full((600,), lod, dtype=torch.float64)), bil), lod


def test_integer_lod_is_the_level_lookup():
    S = 16
    cube, d = _cube(S, 2, seed=3), _dirs(800, 4)
    for k in range(cmm.level_count(S)):
        assert torch.equal(cmm.sample(cube, d, torch.full((800,), float(k), dtype=torch.float64)),
                           cmm.level_lookup(cube, d, k))
    # past the top: the 1 x 1 level
    top = cmm.level_lookup(cube, d, cmm.level_count(S) - 1)
    assert torch.equal(cmm.sample(cube, d, torch.full((800,), 99., dtype=torch.float64)), top)
    assert torch.equal(cmm.sample(cube, d, torch.full((800,), math.inf, dtype=torch.float64)), top)


def test_fraction_blends_the_two_levels():
    S = 8
    cube, d = _cube(S, 2, seed=5), _dirs(300, 6)
    b1, b2 = cmm.level_lookup(cube, d, 1), cmm.level_lookup(cube, d, 2)
    out = cmm.sample(cube, d, torch.full((300,), 1.25, dtype=torch.float64))
    assert torch.equal(out, 0.75 * b1 + 0.25 * b2)


def _edge_points():
    pts = []
    for a, b in itertools.combinations(range(3), 2):
        c = 3 - a - b
        for sa, sb in itertools.product((-1., 1.), repeat=2):
            p, n = np.zeros(3), np.zeros(3)
            p[a], p[b], p[c] = sa, sb, 0.37
            n[a], n[b] = sa, -sb
            pts.append((p, n))
    return pts


@pytest.mark.parametrize('S', [2, 4, 6, 8])
def test_every_level_is_continuous_across_edges_and_corners(S):
    cube = _cube(S, 2, seed=S)
    delta = 1e-9
    bound = 10 * delta * S * 4 * float(cube.abs().max())
    for k in range(cmm.level_count(S)):
        lod = lambda n: torch.full((n,), float(k), dtype=torch.float64)
        for p, n in _edge_points():
            pair = torch.from_numpy(np.stack([p + delta * n, p - delta * n]))
            f = cm.face_coords(pair)[0]
            assert int(f[0]) != int(f[1])
            out = cmm.sample(cube, pair, lod(2))
            assert float((out[0] - out[1]).abs().max()) <= bound, (k, p, n)
        rng = np.random.default_rng(S + k)
        for corner in itertools.product((-1., 1.), repeat=3):
            pts = torch.from_numpy(np.array(corner) + delta * rng.standard_normal((24, 3)))
            assert len(set(int(f) for f in cm.face_coords(pts)[0])) == 3
            out = cmm.sample(cube, pts, lod(24))
            assert float((out - out[:1]).abs().max()) <= bound, (k, corner)


def test_constant_map_is_constant_at_every_lod():
    for S in (1, 2, 6, 16):
        cube = torch.full((6, S, S, 2), 0.7, dtype=torch.float64)
        d = _dirs(1000, S)
        lod = torch.from_numpy(np.random.default_rng(S).uniform(-2, cmm.level_count(S) + 2, 1000))
        assert float((cmm.sample(cube, d, lod) - 0.7).abs().max()) <= 1e-15, S


def test_grad_lod_is_the_stated_formula_and_the_central_difference():
    S, C, n = 16, 3, 400
    L = cmm.level_count(S)
    cube, d = _cube(S, C, seed=7), _dirs(n, 8)
    rng = np.random.default_rng(9)
    lod = torch.from_numpy(rng.uniform(-1.5, L + 0.5, n))
    lod[:8] = torch.tensor([0., 1., float(L - 1), -0.5, L - 0.5, math.nan, math.inf, 2.])
    g = torch.from_numpy(rng.standard_normal((n, C)))
    x = lod.clone().requires_grad_(True)
    (cmm.sample(cube, d, x) * g).sum().backward()
    reads = [cmm.level_lookup(cube, d, k) for k in range(L)]
    want = torch.zeros(n, dtype=torch.float64)
    for i in range(n):
        v = float(lod[i])
        if math.isnan(v) or v < 0 or v > L - 1:
            continue
        m = min(int(math.floor(v)), L - 2)
        want[i] = float((g[i] * (reads[m + 1][i] - reads[m][i])).sum())
    assert torch.equal(x.grad, want)
    # float64 central differences at non-integer lambda inside the pyramid
    inside = (lod > 0.01) & (lod < L - 1.01) & ((lod - lod.floor()) > 0.01) & ((lod - lod.floor()) < 0.99)
    h = 1e-6
    fd = ((cmm.sample(cube, d, lod + h) - cmm.sample(cube, d, lod - h)) * g).sum(-1) / (2 * h)
    assert torch.allclose(x.grad[inside], fd[inside], rtol=1e-6, atol=1e-8)
    # the forward value is untouched by the lod's gradient path
    assert torch.equal(cmm.sample(cube, d, x), cmm.sample(cube, d, lod))


def test_grad_lod_is_zero_for_one_level_and_invalid_directions():
    cube = _cube(3, 2, seed=10)
    d = torch.tensor([[0., 0., 0.], [math.nan, 1., 0.], [0.3, 0.2, 1.]], dtype=torch.float64)
    x = torch.full((3,), 0.5, dtype=torch.float64, requires_grad=True)
    cmm.sample(cube, d, x).sum().backward()
    assert not x.grad.any()   # S = 3: one level
    cube = _cube(4, 2, seed=11)
    x = torch.full((3,), 0.5, dtype=torch.float64, requires_grad=True)
    cmm.sample(cube, d, x).sum().backward()
    assert not x.grad[:2].any() and bool(x.grad[2] != 0)


def test_grad_directions_and_cubemap_match_finite_differences():
    """float64 gradcheck away from texel boundaries: through both levels, their borders and the pyramid."""
    S = 4
    cube = _cube(S, 2, seed=12).requires_grad_(True)
    d = _dirs(30, 13)
    lod = torch.from_numpy(np.random.default_rng(14).uniform(0.1, 1.9, 30))
    lod[lod.sub(lod.floor()) < 0.05] += 0.1
    assert torch.autograd.gradcheck(lambda c, x: cmm.sample(c, x, lod), (cube, d.requires_grad_(True)))


def test_invalid_directions_give_zero():
    cube = _cube(4, 2) + 1.
    d = torch.tensor([[0., 0., 0.], [math.inf, 0., 1.], [0.3, -0.2, 0.9]], dtype=torch.float64)
    out = cmm.sample(cube, d, torch.tensor([0.5, 1.5, 1.5], dtype=torch.float64))
    assert not out[:2].any() and bool((out[2] != 0).all())


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _p(x):
    return ctypes.c_void_p(x)


def test_abi_rejects_bad_shapes(L):
    from dirt_b200 import _lib
    buf = _p(4096)
    fwd = lambda TB, S, C, B, N: L.dirt_cubemap_sample_trilinear(buf, buf, buf, buf, buf, TB, S, C, B, N, None)
    bwd = lambda TB, S, C, B, N: L.dirt_cubemap_sample_trilinear_backward(buf, buf, buf, buf, buf, buf, buf, TB, S, C, B,
                                                                          N, 0, buf, 1 << 40, None)
    for call in (fwd, bwd):
        assert call(1, 0, 3, 1, 8) == _lib.ERR_BAD_SHAPE
        assert call(1, (1 << 14) + 1, 3, 1, 8) == _lib.ERR_BAD_SHAPE
        assert call(1, 4, 0, 1, 8) == _lib.ERR_BAD_SHAPE
        assert call(1, 4, 3, -1, 8) == _lib.ERR_BAD_SHAPE
        assert call(1, 4, 3, 1, -1) == _lib.ERR_BAD_SHAPE
        assert call(2, 4, 3, 3, 8) == _lib.ERR_BAD_SHAPE
        assert call(1, 4, 3, 1 << 30, 1 << 40) == _lib.ERR_BAD_SHAPE
        assert L.dirt_last_launch_count() == 0
    det = lambda B, N: L.dirt_cubemap_sample_trilinear_backward(buf, buf, buf, buf, buf, buf, buf, 1, 4, 3, B, N, 1, buf,
                                                                1 << 40, None)
    assert det(1, 1 << 31) == _lib.ERR_BAD_SHAPE
    nbytes = L.dirt_cubemap_sample_trilinear_backward_bytes
    assert nbytes(1, 4, 3, 1, 1 << 31, 1) == 0 and nbytes(1, 4, 3, 1, 1 << 31, 0) > 0
    assert nbytes(1, 0, 3, 1, 8, 0) == 0 and nbytes(1, 4, 3, 1, 0, 0) == 0
    atlas = L.dirt_cubemap_mip_atlas_bytes
    assert atlas(1, 0, 3) == 0 and atlas(-1, 4, 3) == 0
    # S = 4: levels of 4, 2, 1 texels per edge, padded to 6, 4, 3
    assert atlas(2, 4, 3) == 4 * 6 * 2 * (36 + 16 + 9) * 3
    assert atlas(1, 5, 1) == L.dirt_cubemap_atlas_bytes(1, 5, 1)


def test_abi_with_no_lookups_launches_nothing(L):
    null = _p(0)
    assert L.dirt_cubemap_sample_trilinear(null, null, null, null, null, 1, 4, 3, 0, 8, None) == 0
    assert L.dirt_cubemap_sample_trilinear(null, null, null, null, null, 1, 4, 3, 2, 0, None) == 0
    assert L.dirt_cubemap_sample_trilinear_backward(null, null, null, null, null, null, null, 1, 4, 3, 0, 8, 1, null, 0,
                                                    None) == 0
    assert L.dirt_last_launch_count() == 0


def test_abi_rejects_null_and_misaligned_pointers(L):
    from dirt_b200 import _lib
    null, ok, odd = _p(0), _p(4096), _p(4098)
    fwd = L.dirt_cubemap_sample_trilinear
    for k in range(5):
        args = [ok] * 5
        args[k] = null
        assert fwd(*args, 1, 4, 3, 1, 8, None) == _lib.ERR_NULL_POINTER, k
        args[k] = odd
        assert fwd(*args, 1, 4, 3, 1, 8, None) == _lib.ERR_MISALIGNED, k
    bwd = L.dirt_cubemap_sample_trilinear_backward
    need = int(L.dirt_cubemap_sample_trilinear_backward_bytes(1, 4, 3, 1, 8, 0))
    assert need > 0
    for k in (1, 2, 3):   # directions, lod, grad_out
        args = [ok] * 7
        args[k] = null
        assert bwd(*args, 1, 4, 3, 1, 8, 0, ok, need, None) == _lib.ERR_NULL_POINTER, k
    # grad_directions or grad_lod read the atlas
    assert bwd(null, ok, ok, ok, ok, ok, null, 1, 4, 3, 1, 8, 0, ok, need, None) == _lib.ERR_NULL_POINTER
    assert bwd(null, ok, ok, ok, ok, null, ok, 1, 4, 3, 1, 8, 0, ok, need, None) == _lib.ERR_NULL_POINTER
    assert bwd(ok, ok, ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 0, null, need, None) == _lib.ERR_NULL_POINTER
    assert bwd(ok, ok, ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 0, _p(4096 + 128), need, None) == _lib.ERR_MISALIGNED
    assert bwd(ok, ok, ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 0, ok, need - 1, None) == _lib.ERR_WORKSPACE_TOO_SMALL
    det_need = int(L.dirt_cubemap_sample_trilinear_backward_bytes(1, 4, 3, 1, 8, 1))
    assert det_need > need
    assert bwd(ok, ok, ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 1, ok, det_need - 1, None) == _lib.ERR_WORKSPACE_TOO_SMALL
    for k in range(7):
        args = [ok] * 7
        args[k] = odd
        assert bwd(*args, 1, 4, 3, 1, 8, 0, ok, need, None) == _lib.ERR_MISALIGNED, k
    assert L.dirt_last_launch_count() == 0


def test_every_declared_symbol_is_exported(L):
    from dirt_b200 import _lib
    for name in ('dirt_cubemap_mip_atlas_bytes', 'dirt_cubemap_sample_trilinear',
                 'dirt_cubemap_sample_trilinear_backward_bytes', 'dirt_cubemap_sample_trilinear_backward'):
        assert name in _lib.EXPORTED_SYMBOLS
        assert getattr(L, name).restype is not None


def test_sample_cubemap_lod_argument_errors():
    import dirt_b200 as dirt
    cube = torch.zeros(6, 4, 4, 3)
    with pytest.raises(ValueError, match='needs lod'):
        dirt.sample_cubemap(cube, torch.zeros(7, 3), mode='trilinear')
    for mode in ('bilinear', 'nearest'):
        with pytest.raises(ValueError, match='only used by'):
            dirt.sample_cubemap(cube, torch.zeros(7, 3), mode=mode, lod=1.)
    with pytest.raises(ValueError, match='mode'):
        dirt.sample_cubemap(cube, torch.zeros(7, 3), mode='anisotropic', lod=1.)
    with pytest.raises(ValueError, match='broadcastable'):
        dirt.sample_cubemap(cube, torch.zeros(7, 3), mode='trilinear', lod=torch.zeros(5))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match='CUDA'):
            dirt.sample_cubemap(cube, torch.zeros(7, 3), mode='trilinear', lod=torch.zeros(7))
