"""CPU: the texture lookup's C ABI and Python layer reject bad arguments before anything is launched."""
import ctypes

import pytest
import torch


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _p(x):
    return ctypes.c_void_p(x)


def test_texture_abi_rejects_bad_shapes(L):
    from dirt_b200 import _lib
    buf = _p(4096)   # never dereferenced: every call below fails validation first
    fwd = lambda TB, TH, TW, C, B, N, mode=0: L.dirt_texture_sample(buf, buf, buf, TB, TH, TW, C, B, N, mode, None)
    bwd = lambda TB, TH, TW, C, B, N, mode=0: L.dirt_texture_sample_backward(buf, buf, buf, buf, buf, TB, TH, TW, C, B, N,
                                                                             mode, None)
    for call in (fwd, bwd):
        assert call(1, 0, 4, 3, 1, 8) == _lib.ERR_BAD_SHAPE          # TH = 0
        assert call(1, 4, 0, 3, 1, 8) == _lib.ERR_BAD_SHAPE          # TW = 0
        assert call(1, 4, 4, 0, 1, 8) == _lib.ERR_BAD_SHAPE          # C = 0
        assert call(1, 4, 4, 3, -1, 8) == _lib.ERR_BAD_SHAPE         # B < 0
        assert call(1, 4, 4, 3, 1, -1) == _lib.ERR_BAD_SHAPE         # N < 0
        assert call(2, 4, 4, 3, 3, 8) == _lib.ERR_BAD_SHAPE          # TB neither 1 nor B
        assert call(1, 4, 4, 3, 1, 8, mode=2) == _lib.ERR_BAD_SHAPE  # unknown mode
        assert call(1, 1 << 30, 1 << 30, 8, 1, 8) == _lib.ERR_BAD_SHAPE   # texel offsets past 2^62
        assert call(1, 4, 4, 3, 1 << 30, 1 << 40) == _lib.ERR_BAD_SHAPE   # lookup offsets past 2^62
        assert L.dirt_last_launch_count() == 0


def test_texture_abi_with_no_lookups_launches_nothing(L):
    null = _p(0)
    assert L.dirt_texture_sample(null, null, null, 1, 4, 4, 3, 0, 8, 0, None) == 0
    assert L.dirt_texture_sample(null, null, null, 1, 4, 4, 3, 2, 0, 1, None) == 0
    assert L.dirt_texture_sample(null, null, null, 0, 4, 4, 3, 0, 8, 0, None) == 0   # per-item textures of an empty batch
    assert L.dirt_texture_sample_backward(null, null, null, null, null, 1, 4, 4, 3, 0, 8, 0, None) == 0
    assert L.dirt_last_launch_count() == 0


def test_texture_abi_rejects_null_and_misaligned_pointers(L):
    from dirt_b200 import _lib
    null, ok, odd = _p(0), _p(4096), _p(4098)
    assert L.dirt_texture_sample(null, ok, ok, 1, 4, 4, 3, 1, 8, 0, None) == _lib.ERR_NULL_POINTER
    assert L.dirt_texture_sample(ok, null, ok, 1, 4, 4, 3, 1, 8, 0, None) == _lib.ERR_NULL_POINTER
    assert L.dirt_texture_sample(ok, ok, null, 1, 4, 4, 3, 1, 8, 0, None) == _lib.ERR_NULL_POINTER
    assert L.dirt_texture_sample(odd, ok, ok, 1, 4, 4, 3, 1, 8, 0, None) == _lib.ERR_MISALIGNED
    assert L.dirt_texture_sample(ok, odd, ok, 1, 4, 4, 3, 1, 8, 0, None) == _lib.ERR_MISALIGNED
    assert L.dirt_texture_sample(ok, ok, odd, 1, 4, 4, 3, 1, 8, 0, None) == _lib.ERR_MISALIGNED
    bwd = L.dirt_texture_sample_backward
    assert bwd(ok, null, ok, ok, ok, 1, 4, 4, 3, 1, 8, 0, None) == _lib.ERR_NULL_POINTER       # indices
    assert bwd(ok, ok, null, ok, ok, 1, 4, 4, 3, 1, 8, 0, None) == _lib.ERR_NULL_POINTER       # grad_out
    assert bwd(null, ok, ok, ok, ok, 1, 4, 4, 3, 1, 8, 0, None) == _lib.ERR_NULL_POINTER       # bilinear grad_indices reads the texture
    for k in range(5):
        args = [ok] * 5
        args[k] = odd
        assert bwd(*args, 1, 4, 4, 3, 1, 8, 0, None) == _lib.ERR_MISALIGNED, k
    assert L.dirt_last_launch_count() == 0


def test_sample_texture_argument_errors():
    import dirt_b200 as dirt
    tex = torch.zeros(4, 5, 3)
    with pytest.raises(ValueError, match='mode'):
        dirt.sample_texture(tex, torch.zeros(7, 2), mode='cubic')
    with pytest.raises(ValueError, match='3D or 4D'):
        dirt.sample_texture(torch.zeros(5, 3), torch.zeros(7, 2))
    with pytest.raises(ValueError, match='positive'):
        dirt.sample_texture(torch.zeros(0, 5, 3), torch.zeros(7, 2))
    with pytest.raises(ValueError, match=r'shape\[-1\] == 2'):
        dirt.sample_texture(tex, torch.zeros(7, 3))
    with pytest.raises(ValueError, match=r'shape\[0\] == texture.shape\[0\]'):
        dirt.sample_texture(tex[None].expand(2, 4, 5, 3), torch.zeros(3, 7, 2))
    with pytest.raises(ValueError, match='at least 2D'):
        dirt.sample_texture(tex[None], torch.zeros(2))
    if not torch.cuda.is_available():
        # no CPU kernel: CPU tensors are an error, never a fallback
        with pytest.raises(RuntimeError, match='CUDA'):
            dirt.sample_texture(tex, torch.zeros(7, 2))


def test_uvs_to_pixel_indices_is_the_examples():
    import dirt_b200 as dirt
    uv = torch.tensor([[0., 0.], [1., 1.], [-0.25, 1.5], [0.3, 0.7]])
    got = dirt.uvs_to_pixel_indices(uv, (4, 8))
    assert torch.equal(got, torch.stack([uv[:, 1] % 1. * 4, uv[:, 0] % 1. * 8], -1))
    got = dirt.uvs_to_pixel_indices(uv, (4, 8), mode='clamp')
    assert torch.equal(got, torch.stack([uv[:, 1].clamp(0, 1) * 4, uv[:, 0].clamp(0, 1) * 8], -1))
    with pytest.raises(NotImplementedError):
        dirt.uvs_to_pixel_indices(uv, (4, 8), mode='mirror')
