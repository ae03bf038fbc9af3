"""GPU: the deterministic texture backward pass (dirt_texture_sample_backward_deterministic) against the numpy
restatement of its order and tree (tests/texture_det_order.py) bit for bit, against torch autograd of
examples/textured.py in float64 at test_gpu_texture.py's bar, and its reproducibility, eagerly, under CUDA graph replay
and through the public API under torch.use_deterministic_algorithms."""
import ctypes

import numpy as np
import pytest
import torch

import texture_det_order as order
from test_gpu_texture import DEV, SHAPES, _bits_equal, _close, _gen, _indices, _reference_grads, _textured_cube, _uv_indices, ex  # noqa: F401

pytestmark = pytest.mark.gpu

_MODES = {'bilinear': 0, 'nearest': 1}


def det_call(tex, idx, gout, mode='bilinear', want_indices=True, fill=None):
    """One raw call on tex [TB, TH, TW, C], idx [B, N, 2], gout [B, N, C] -> (grad_texture, grad_indices, scratch)."""
    from dirt_b200 import _lib
    L = _lib.lib()
    TB, TH, TW, C = tex.shape
    B, N = idx.shape[0], idx.shape[1]
    nbytes = max(int(L.dirt_texture_sample_backward_deterministic_bytes(TB, TH, TW, C, B, N, _MODES[mode])), 256)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    if fill is not None:
        scratch.fill_(fill)
    gt = torch.empty_like(tex)
    gi = torch.empty_like(idx) if want_indices else None
    p = lambda t: ctypes.c_void_p(t.data_ptr() if t is not None else 0)
    rc = L.dirt_texture_sample_backward_deterministic(p(tex), p(idx), p(gout), p(gt), p(gi), TB, TH, TW, C, B, N,
                                                      _MODES[mode], p(scratch), nbytes,
                                                      ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    assert rc == 0, rc
    return gt, gi, scratch


def default_call(tex, idx, gout, mode='bilinear'):
    from dirt_b200 import _lib
    L = _lib.lib()
    TB, TH, TW, C = tex.shape
    B, N = idx.shape[0], idx.shape[1]
    gt, gi = torch.empty_like(tex), torch.empty_like(idx)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    assert L.dirt_texture_sample_backward(p(tex), p(idx), p(gout), p(gt), p(gi), TB, TH, TW, C, B, N, _MODES[mode],
                                          ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)) == 0
    return gt, gi


def _check(ex, tex, idx, gout, mode, tag):
    """tex [TB, TH, TW, C] (TB = 1: shared), idx [B, N, 2], gout [B, N, C]: bit for bit against the restatement, at the
    bar against autograd in float64, grad_indices bit for bit against the default entry."""
    gt, gi, _ = det_call(tex, idx, gout, mode)
    want = order.grad_texture(tuple(tex.shape), idx.cpu().numpy(), gout.cpu().numpy(), mode)
    got = gt.cpu().numpy()
    assert np.array_equal(got.view(np.int32), want.view(np.int32)), (tag, int((got != want).sum()))
    if tex.shape[0] == 1:
        ref_t, _ = _reference_grads(ex, tex[0], idx.reshape(-1, 2), gout.reshape(-1, tex.shape[-1]), mode)
        ok, ratio = _close(gt[0], ref_t, 'deterministic grad_texture')
        assert ok, (tag, ratio)
    else:
        for b in range(tex.shape[0]):
            ref_t, _ = _reference_grads(ex, tex[b], idx[b], gout[b], mode)
            ok, ratio = _close(gt[b], ref_t, 'deterministic grad_texture')
            assert ok, (tag, b, ratio)
    assert _bits_equal(gi, default_call(tex, idx, gout, mode)[1]), tag
    return gt


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [1, 2, 3, 4, 5, 8])
def test_matches_the_restated_order_bit_for_bit(ex, mode, C):
    for k, (H, W) in enumerate(SHAPES):
        tex = torch.rand(1, H, W, C, generator=_gen(k), device=DEV)
        for idx in (_indices(H, W, 5000, 400 + k), _uv_indices(H, W, 'repeat', 600 + k)):
            idx = idx[None].contiguous()
            gout = torch.randn(idx.shape[:-1] + (C,), generator=_gen(500 + k), device=DEV)
            _check(ex, tex, idx, gout, mode, (H, W, C, mode))


@pytest.mark.parametrize('C', [1, 3, 4, 6])
def test_contention(ex, C):
    from dirt_b200 import uvs_to_pixel_indices
    # 2^20 lookups into a 2x2 texture: 2^20 terms per texel, 256 chunks
    tex = torch.rand(1, 2, 2, C, generator=_gen(4), device=DEV)
    idx = (torch.rand(1, 1 << 20, 2, generator=_gen(5), device=DEV) * 6 - 3)
    gout = torch.rand(1, 1 << 20, C, generator=_gen(6), device=DEV) + 0.5
    _check(ex, tex, idx, gout, 'bilinear', ('2x2', C))
    _check(ex, tex, idx, gout, 'nearest', ('2x2 nearest', C))
    # a 16^2 texture over 512^2: about 4096 terms per texel, on both sides of the chunk length
    tex = torch.rand(1, 16, 16, C, generator=_gen(8), device=DEV)
    ys, xs = torch.meshgrid(torch.arange(512, device=DEV), torch.arange(512, device=DEV), indexing='ij')
    uv = torch.stack([(xs + 0.5) / 512, (ys + 0.5) / 512], -1)
    idx = uvs_to_pixel_indices(uv, (16, 16)).reshape(1, -1, 2).contiguous()
    gout = torch.rand(1, idx.shape[1], C, generator=_gen(9), device=DEV) + 0.5
    _check(ex, tex, idx, gout, 'bilinear', ('16^2 over 512^2', C))
    # minified: 1024^2 random
    tex = torch.rand(1, 1024, 1024, C, generator=_gen(10), device=DEV)
    idx = torch.rand(1, 1 << 18, 2, generator=_gen(11), device=DEV) * 1024
    gout = torch.randn(1, 1 << 18, C, generator=_gen(12), device=DEV)
    _check(ex, tex, idx, gout, 'bilinear', ('1024^2 random', C))


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
def test_every_lookup_on_one_texel(ex, mode):
    # 3 * 2^18 lookups based at one texel: 192 chunks on each texel it reaches
    n = 3 << 18
    tex = torch.rand(1, 64, 48, 3, generator=_gen(31), device=DEV)
    idx = torch.tensor([17.25, 30.5], device=DEV).expand(1, n, 2).contiguous()
    gout = torch.rand(1, n, 3, generator=_gen(32), device=DEV) + 0.5
    gt = _check(ex, tex, idx, gout, mode, ('one texel', mode))
    assert int((gt != 0).any(-1).sum()) == (4 if mode == 'bilinear' else 1)


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [3, 4, 5])
def test_per_item_textures_and_item_independence(ex, mode, C):
    B, H, W = 3, 17, 23
    tex = torch.rand(B, H, W, C, generator=_gen(13), device=DEV)
    idx = torch.stack([_indices(H, W, 1000, 14 + b) for b in range(B)]).contiguous()
    gout = torch.randn(idx.shape[:-1] + (C,), generator=_gen(15), device=DEV)
    gt = _check(ex, tex, idx, gout, mode, ('per item', C, mode))
    for b in range(B):
        alone, gi, _ = det_call(tex[b:b + 1].contiguous(), idx[b:b + 1].contiguous(), gout[b:b + 1].contiguous(), mode)
        assert _bits_equal(alone[0], gt[b]), b
    # a shared texture under a batch of indices: one sum over every item in id order
    shared = tex[:1].contiguous()
    _check(ex, shared, idx, gout, mode, ('shared, batched', C, mode))


def test_repeats_scratch_contents_and_graph_replay():
    tex = torch.rand(1, 64, 48, 4, generator=_gen(28), device=DEV)
    idx = _indices(64, 48, 100000, 29)[None].contiguous()
    gout = torch.randn(idx.shape[:-1] + (4,), generator=_gen(30), device=DEV)
    gt, gi, _ = det_call(tex, idx, gout)
    for fill in (None, 0xFF, 0):
        gt2, gi2, _ = det_call(tex, idx, gout, fill=fill)
        assert _bits_equal(gt, gt2) and _bits_equal(gi, gi2), fill
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        det_call(tex, idx, gout)
    torch.cuda.current_stream(DEV).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_t, out_i, scratch = det_call(tex, idx, gout)
    for _ in range(2):
        scratch.fill_(0xFF)
        out_t.fill_(float('nan'))
        graph.replay()
        torch.cuda.synchronize()
        assert _bits_equal(out_t, gt) and _bits_equal(out_i, gi)


@pytest.fixture
def deterministic_algorithms():
    before = torch.are_deterministic_algorithms_enabled()
    yield
    torch.use_deterministic_algorithms(before)


def _kernels(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_public_api_follows_torch_deterministic_algorithms(cuda_lib, deterministic_algorithms):
    import dirt_b200 as dirt
    tex = torch.rand(37, 29, 3, generator=_gen(40), device=DEV)
    idx = _indices(37, 29, 20000, 41)
    gout = torch.randn(idx.shape[0], 3, generator=_gen(42), device=DEV)

    def run():
        t, i = tex.clone().requires_grad_(True), idx.clone().requires_grad_(True)
        (dirt.sample_texture(t, i) * gout).sum().backward()
        return t.grad, i.grad

    torch.use_deterministic_algorithms(True)
    names = _kernels(run)
    assert any('tex_det_gather_kernel' in n for n in names)
    gt, gi = run()
    raw_t, raw_i, _ = det_call(tex[None].contiguous(), idx[None].contiguous(), gout[None].contiguous())
    assert _bits_equal(gt, raw_t[0]) and _bits_equal(gi, raw_i[0])
    torch.use_deterministic_algorithms(False)
    names = _kernels(run)
    assert not any('tex_det' in n or 'tex_sort' in n for n in names)
    assert any('texture_backward_kernel' in n for n in names)


def test_textured_cube_is_reproducible_under_the_flag(ex, deterministic_algorithms):
    import dirt_b200 as dirt
    torch.use_deterministic_algorithms(True)
    first = _textured_cube(ex, dirt.sample_texture)
    second = _textured_cube(ex, dirt.sample_texture)
    assert _bits_equal(first[0], second[0])
    for name, a, b in zip(['vertices', 'texture', 'light'], first[1:], second[1:]):
        assert a is not None and _bits_equal(a, b), name
    assert first[2].abs().sum() > 0
