"""CPU: the mipmapped lookup's torch restatement (levels, level counts), index_derivatives' rule, sample_texture's
argument errors, and the C ABI's size functions and argument checks, none of which launches anything."""
import ctypes

import numpy as np
import pytest
import torch

import texture_mip_restatement as mip


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_restatement_levels_are_the_two_by_two_means():
    tex = torch.rand(2, 8, 12, 3, generator=torch.Generator().manual_seed(0))
    levels = mip.pyramid(tex)
    assert [tuple(t.shape) for t in levels] == [(2, 8, 12, 3), (2, 4, 6, 3), (2, 2, 3, 3)]
    for k in (1, 2):
        prev = levels[k - 1].double()
        want = prev.reshape(2, prev.shape[1] // 2, 2, prev.shape[2] // 2, 2, 3).mean(dim=(2, 4))
        assert torch.allclose(levels[k].double(), want, rtol=0, atol=1e-6)
    t = levels[0]
    i, j = 3, 5
    assert levels[1][1, i, j, 2] == ((t[1, 2 * i, 2 * j, 2] + t[1, 2 * i, 2 * j + 1, 2]) +
                                     (t[1, 2 * i + 1, 2 * j, 2] + t[1, 2 * i + 1, 2 * j + 1, 2])) * 0.25


@pytest.mark.parametrize('shape, levels', [((1, 1), 1), ((2, 1), 1), ((6, 10), 2), ((640, 480), 6), ((1024, 512), 10),
                                           ((256, 256), 9), ((5, 7), 1)])
def test_level_count(L, shape, levels):
    assert mip.level_count(*shape) == levels
    assert L.dirt_texture_mip_levels(*shape) == levels
    last = mip.pyramid(torch.zeros(shape + (1,)))[-1]
    assert last.shape[:2] == {(1024, 512): (2, 1), (640, 480): (20, 15)}.get(shape, last.shape[:2])


def _helper(idx, shape):
    from dirt_b200 import index_derivatives
    got = index_derivatives(torch.as_tensor(idx, dtype=torch.float32), shape)
    np.testing.assert_allclose(got.numpy(), mip.index_derivatives(idx, shape), rtol=1e-6, atol=1e-5)
    return got.numpy()


def test_index_derivatives_of_a_linear_ramp_are_constant():
    ys, xs = np.meshgrid(np.arange(6.), np.arange(9.), indexing='ij')
    idx = np.stack([10 + 0.5 * xs + 2.0 * ys, 20 + 3.0 * xs - 1.0 * ys], -1)
    d = _helper(idx, (256, 256))
    assert np.allclose(d, [0.5, 3.0, 2.0, -1.0])


def test_index_derivatives_remove_repeat_seams():
    # a column index that wraps from 62 to 1 on a 64-wide texture: a step of +3, not -61
    idx = np.zeros((1, 8, 2))
    idx[0, :, 1] = (50 + 3 * np.arange(8)) % 64
    d = _helper(idx, (64, 64))
    assert np.allclose(d[0, :, 1], 3.0) and np.allclose(d[0, :, 0], 0.0)


def test_index_derivatives_pick_the_continuous_side_of_a_step():
    idx = np.zeros((1, 8, 2))
    idx[0, :, 1] = np.where(np.arange(8) < 4, np.arange(8) * 1.0, 40 + np.arange(8) * 1.0)
    d = _helper(idx, (128, 128))
    assert np.allclose(d[0, :, 1], 1.0)   # at pixels 3 and 4 the other side is the 41-texel step


def test_index_derivatives_at_borders_and_on_length_one_axes():
    idx = np.zeros((3, 1, 2))
    idx[:, 0, 0] = [0., 1., 3.]
    d = _helper(idx, (32, 32))
    assert np.allclose(d[..., :2], 0.0)                  # W = 1: no x derivative
    assert np.allclose(d[:, 0, 2], [1., 1., 2.])          # one-sided at the top and bottom rows, the smaller in between
    assert np.allclose(_helper(np.ones((1, 1, 2)), (8, 8)), 0.0)


def test_sample_texture_argument_errors():
    import dirt_b200 as dirt
    tex, idx = torch.zeros(8, 8, 3), torch.zeros(5, 2)
    with pytest.raises(ValueError, match='needs derivatives'):
        dirt.sample_texture(tex, idx, mode='trilinear')
    with pytest.raises(ValueError, match="only used by mode 'trilinear'"):
        dirt.sample_texture(tex, idx, derivatives=torch.zeros(5, 4))
    with pytest.raises(ValueError, match="only used by mode 'trilinear'"):
        dirt.sample_texture(tex, idx, mode='nearest', derivatives=torch.zeros(5, 4))
    if torch.cuda.is_available():
        return
    with pytest.raises(ValueError, match=r'derivatives.shape == indices.shape\[:-1\] \+ \(4,\)'):
        dirt.sample_texture(tex, idx, mode='trilinear', derivatives=torch.zeros(5, 2))
    with pytest.raises(ValueError, match='mode'):
        dirt.sample_texture(tex, idx, mode='cubic')


def _p(x):
    return ctypes.c_void_p(x)


def test_size_functions_are_pure_functions_of_the_shapes(L):
    pb = L.dirt_texture_mip_pyramid_bytes
    assert pb(1, 1024, 1024, 3) == 4 * 3 * sum((1024 >> k) ** 2 for k in range(1, 11))
    assert pb(2, 8, 4, 5) == 2 * pb(1, 8, 4, 5) == 2 * 4 * 5 * (4 * 2 + 2 * 1)
    assert pb(1, 5, 8, 3) == 0 and pb(1, 0, 8, 3) == 0 and pb(1, 8, 8, 0) == 0
    bb = L.dirt_texture_sample_trilinear_backward_bytes
    assert bb(1, 64, 64, 3, 2, 100, 0) == bb(1, 64, 64, 3, 7, 10000, 0) >= pb(1, 64, 64, 3)   # default: the pyramid's grads
    assert bb(1, 63, 64, 3, 2, 100, 0) == 0                                                   # one level: none
    a, b = bb(1, 64, 64, 3, 2, 100, 1), bb(1, 64, 64, 3, 2, 200, 1)
    assert 0 < a < b and a == bb(1, 64, 64, 3, 2, 100, 1)
    assert bb(1, 64, 64, 3, 0, 100, 1) == 0 and bb(1, 64, 64, 3, 1, 1 << 31, 1) == 0


def _bwd(L, TB=1, TH=8, TW=8, C=3, B=2, N=100, det=0, scratch=4096, scratch_bytes=1 << 30, **ptrs):
    p = dict(texture=4096, pyramid=4096, indices=4096, derivatives=4096, grad_out=4096, grad_texture=4096,
             grad_indices=4096)
    p.update(ptrs)
    return L.dirt_texture_sample_trilinear_backward(
        _p(p['texture']), _p(p['pyramid']), _p(p['indices']), _p(p['derivatives']), _p(p['grad_out']),
        _p(p['grad_texture']), _p(p['grad_indices']), TB, TH, TW, C, B, N, det, _p(scratch), scratch_bytes, None)


def test_argument_checks_return_their_codes_before_launching(L):
    from dirt_b200 import _lib
    cases = [
        (dict(TH=0), _lib.ERR_BAD_SHAPE), (dict(C=0), _lib.ERR_BAD_SHAPE), (dict(B=-1), _lib.ERR_BAD_SHAPE),
        (dict(TB=2, B=3), _lib.ERR_BAD_SHAPE), (dict(det=1, B=1, N=1 << 31), _lib.ERR_BAD_SHAPE),
        (dict(indices=0), _lib.ERR_NULL_POINTER), (dict(derivatives=0), _lib.ERR_NULL_POINTER),
        (dict(grad_out=0), _lib.ERR_NULL_POINTER), (dict(texture=0), _lib.ERR_NULL_POINTER),
        (dict(pyramid=0), _lib.ERR_NULL_POINTER), (dict(scratch=0), _lib.ERR_NULL_POINTER),
        (dict(det=1, scratch=0), _lib.ERR_NULL_POINTER),
        (dict(texture=4098), _lib.ERR_MISALIGNED), (dict(pyramid=4098), _lib.ERR_MISALIGNED),
        (dict(derivatives=4098), _lib.ERR_MISALIGNED), (dict(grad_texture=4098), _lib.ERR_MISALIGNED),
        (dict(scratch=4224), _lib.ERR_MISALIGNED),
        (dict(scratch_bytes=L.dirt_texture_sample_trilinear_backward_bytes(1, 8, 8, 3, 2, 100, 0) - 1),
         _lib.ERR_WORKSPACE_TOO_SMALL),
        (dict(det=1, scratch_bytes=L.dirt_texture_sample_trilinear_backward_bytes(1, 8, 8, 3, 2, 100, 1) - 1),
         _lib.ERR_WORKSPACE_TOO_SMALL),
    ]
    for kw, rc in cases:
        assert _bwd(L, **kw) == rc, kw
        assert L.dirt_last_launch_count() == 0
    # one level: no pyramid and no scratch needed
    assert _bwd(L, TH=7, pyramid=0, scratch=0, grad_indices=0, grad_texture=0, B=0) == 0
    # the forward and build entries
    fwd = L.dirt_texture_sample_trilinear
    assert fwd(_p(4096), _p(4096), _p(4096), _p(4096), _p(4096), 1, 8, 8, 0, 1, 10, None) == _lib.ERR_BAD_SHAPE
    assert fwd(_p(4096), _p(0), _p(4096), _p(4096), _p(4096), 1, 8, 8, 3, 1, 10, None) == _lib.ERR_NULL_POINTER
    assert fwd(_p(4096), _p(4096), _p(4096), _p(0), _p(4096), 1, 8, 8, 3, 1, 10, None) == _lib.ERR_NULL_POINTER
    assert fwd(_p(4096), _p(4096), _p(4098), _p(4096), _p(4096), 1, 8, 8, 3, 1, 10, None) == _lib.ERR_MISALIGNED
    assert fwd(_p(0), _p(0), _p(0), _p(0), _p(0), 1, 8, 8, 3, 0, 10, None) == 0
    build = L.dirt_texture_mip_build
    assert build(_p(4096), _p(4096), 1, 0, 8, 3, None) == _lib.ERR_BAD_SHAPE
    assert build(_p(4096), _p(0), 1, 8, 8, 3, None) == _lib.ERR_NULL_POINTER
    assert build(_p(4096), _p(4098), 1, 8, 8, 3, None) == _lib.ERR_MISALIGNED
    assert build(_p(0), _p(0), 1, 7, 8, 3, None) == 0      # one level: nothing to build
    assert L.dirt_last_launch_count() == 0
