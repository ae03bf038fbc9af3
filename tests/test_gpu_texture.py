"""GPU: dirt_b200.sample_texture against the torch restatement of examples/textured.py on the same device.

Forward values are compared bit for bit; gradients against torch autograd of the restatement evaluated in float64,
with conftest.rel_close (1e-4 relative)."""
import ctypes
import functools
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

from conftest import rel_close

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device('cuda', 0)


@pytest.fixture(scope='module')
def ex(cuda_lib):
    spec = importlib.util.spec_from_file_location('textured_example', os.path.join(ROOT, 'examples', 'textured.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _indices(H, W, n, seed):
    """n random (row, col) indices in [-3H, 3H] x [-3W, 3W], then the edge values: exact integers, H-1 / H / -1,
    +-1e9, and values just below 0 whose fraction rounds to 1."""
    g = _gen(seed)
    rnd = (torch.rand(n, 2, generator=g, device=DEV) * 6 - 3) * torch.tensor([H, W], device=DEV, dtype=torch.float32)
    ints = torch.randint(-2 * max(H, W), 2 * max(H, W) + 1, (64, 2), generator=g, device=DEV).to(torch.float32)
    edge = [[H - 1, W - 1], [H, W], [-1, -1], [0, 0], [H - 1, W], [H, -1], [-1, W - 1], [1e9, -1e9], [-1e9, 1e9],
            [1e9, 0.5], [-1e-8, -1e-8], [-1e-8, W - 0.5], [H - 1e-4, 0.25], [3 * H + 0.5, -3 * W - 0.5]]
    return torch.cat([rnd, ints, torch.tensor(edge, dtype=torch.float32, device=DEV)])


def _uv_indices(H, W, mode, seed):
    from dirt_b200 import uvs_to_pixel_indices
    g = _gen(seed)
    uv = torch.rand(2000, 2, generator=g, device=DEV) * 4 - 1.5
    exact = torch.tensor([[0., 0.], [1., 1.], [0., 1.], [1., 0.], [-1., 2.], [2., -1.], [0.5, 0.5]], device=DEV)
    return uvs_to_pixel_indices(torch.cat([uv, exact]), (H, W), mode=mode)


SHAPES = [(1, 1), (1, 7), (9, 1), (5, 7), (13, 11), (256, 256), (1024, 1024)]


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [1, 2, 3, 4, 5, 8])
def test_forward_is_bit_identical_to_the_restatement(ex, mode, C):
    import dirt_b200 as dirt
    for k, (H, W) in enumerate(SHAPES):
        tex = torch.rand(H, W, C, generator=_gen(k), device=DEV) * 2 - 0.5
        for idx in (_indices(H, W, 5000, 100 + k), _uv_indices(H, W, 'repeat', 200 + k), _uv_indices(H, W, 'clamp', 300 + k)):
            got = dirt.sample_texture(tex, idx, mode=mode)
            want = ex.sample_texture(tex, idx, mode=mode)
            assert _bits_equal(got, want), (H, W, C, mode, int((got != want).sum()))


def _reference_grads(ex, tex, idx, grad_out, mode):
    """torch autograd of the restatement, in float64."""
    t = tex.detach().double().requires_grad_(True)
    i = idx.detach().double().requires_grad_(mode == 'bilinear')
    (ex.sample_texture(t, i, mode=mode) * grad_out.double()).sum().backward()
    return t.grad, (i.grad if i.grad is not None else torch.zeros_like(i))


def _close(actual, expected, name):
    """rel_close; a gradient that is zero everywhere (a 1x1 texture has no index gradient: its four texels are one)
    must come back as zeros up to the float64 reference's own rounding."""
    a, b = actual.cpu().numpy(), expected.cpu().numpy()
    if b.size and np.abs(b).max() < 1e-12:
        return bool(np.abs(a).max() < 1e-12), 0.0
    return rel_close(a, b, name=name)


def _check_grads(ex, tex, idx, mode, seed, tag, want=(True, True), label='texture', positive=False):
    """`positive`: grad_out in [0.5, 1.5) (a mean-like loss).  Where 10^5-10^6 lookups share a texel, a random-sign
    grad_out sums to far less than its terms, and the fp32 accumulation's rounding (of any summation order, torch's
    included) is then measured against that small sum instead of against the terms."""
    import dirt_b200 as dirt
    shape = idx.shape[:-1] + (tex.shape[-1],)
    grad_out = (torch.rand(shape, generator=_gen(seed), device=DEV) + 0.5 if positive else
                torch.randn(shape, generator=_gen(seed), device=DEV))
    t = tex.detach().clone().requires_grad_(want[0])
    i = idx.detach().clone().requires_grad_(want[1])
    (dirt.sample_texture(t, i, mode=mode) * grad_out).sum().backward()
    ref_t, ref_i = _reference_grads(ex, tex, idx, grad_out, mode)
    if want[0]:
        ok, ratio = _close(t.grad, ref_t, label + ' grad_texture')
        assert ok, (tag, 'grad_texture', ratio)
    else:
        assert t.grad is None
    if want[1]:
        ok, ratio = _close(i.grad, ref_i, label + ' grad_indices')
        assert ok, (tag, 'grad_indices', ratio)
        if mode == 'nearest':
            assert not i.grad.any()
    else:
        assert i.grad is None


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [1, 2, 3, 4, 5, 8])
def test_backward_matches_autograd_of_the_restatement(ex, mode, C):
    for k, (H, W) in enumerate(SHAPES):
        tex = torch.rand(H, W, C, generator=_gen(k), device=DEV)
        _check_grads(ex, tex, _indices(H, W, 5000, 400 + k), mode, 500 + k, (H, W, C))
        _check_grads(ex, tex, _uv_indices(H, W, 'repeat', 600 + k), mode, 700 + k, (H, W, C, 'uv'))


@pytest.mark.parametrize('want', [(True, False), (False, True), (True, True)])
@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
def test_backward_for_every_needs_input_grad(ex, want, mode):
    tex = torch.rand(37, 29, 3, generator=_gen(1), device=DEV)
    _check_grads(ex, tex, _indices(37, 29, 20000, 2), mode, 3, want, want)


@pytest.mark.parametrize('C', [1, 3, 4, 6])
def test_backward_under_contention(ex, C):
    from dirt_b200 import uvs_to_pixel_indices
    # ~10^6 lookups into a 2x2 texture: every warp's lanes share four texels
    tex = torch.rand(2, 2, C, generator=_gen(4), device=DEV)
    idx = torch.rand(1 << 20, 2, generator=_gen(5), device=DEV) * 6 - 3
    _check_grads(ex, tex, idx, 'bilinear', 6, ('2x2', C), label='contention', positive=True)
    _check_grads(ex, tex, idx, 'nearest', 7, ('2x2 nearest', C), label='contention', positive=True)
    # a 16^2 texture stretched over a 512^2 image: runs of 32 neighbouring lookups per texel
    tex = torch.rand(16, 16, C, generator=_gen(8), device=DEV)
    ys, xs = torch.meshgrid(torch.arange(512, device=DEV), torch.arange(512, device=DEV), indexing='ij')
    uv = torch.stack([(xs + 0.5) / 512, (ys + 0.5) / 512], -1)
    _check_grads(ex, tex, uvs_to_pixel_indices(uv, (16, 16)), 'bilinear', 9, ('16^2 over 512^2', C), label='contention',
                 positive=True)
    # minified: a 1024^2 texture under random lookups (few lanes share a texel), random-sign grad_out
    tex = torch.rand(1024, 1024, C, generator=_gen(10), device=DEV)
    idx = torch.rand(1 << 18, 2, generator=_gen(11), device=DEV) * 1024
    _check_grads(ex, tex, idx, 'bilinear', 12, ('1024^2 random', C))


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [3, 4, 5])
def test_per_item_textures(ex, mode, C):
    import dirt_b200 as dirt
    B, H, W = 3, 17, 23
    tex = torch.rand(B, H, W, C, generator=_gen(13), device=DEV)
    idx = torch.stack([_indices(H, W, 1000, 14 + b) for b in range(B)]).reshape(B, 2, -1, 2)
    got = dirt.sample_texture(tex, idx, mode=mode)
    want = torch.stack([ex.sample_texture(tex[b], idx[b], mode=mode) for b in range(B)])
    assert got.shape == (B, 2, idx.shape[2], C) and _bits_equal(got, want)
    grad_out = torch.randn(got.shape, generator=_gen(15), device=DEV)
    t = tex.clone().requires_grad_(True)
    i = idx.clone().requires_grad_(True)
    (dirt.sample_texture(t, i, mode=mode) * grad_out).sum().backward()
    for b in range(B):
        ref_t, ref_i = _reference_grads(ex, tex[b], idx[b], grad_out[b], mode)
        assert _close(t.grad[b], ref_t, 'texture grad_texture')[0], b
        assert _close(i.grad[b], ref_i, 'texture grad_indices')[0], b


def test_shared_texture_under_batched_indices(ex):
    import dirt_b200 as dirt
    tex = torch.rand(31, 19, 3, generator=_gen(16), device=DEV)
    idx = _indices(31, 19, 4 * 6 * 7 - 78, 17).reshape(4, 6, 7, 2)
    assert _bits_equal(dirt.sample_texture(tex, idx), ex.sample_texture(tex, idx))
    _check_grads(ex, tex, idx, 'bilinear', 18, 'batched indices')


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
def test_non_finite_indices_give_zero_and_no_gradient(ex, mode):
    import dirt_b200 as dirt
    tex = (torch.rand(8, 8, 4, generator=_gen(19), device=DEV) + 1.).requires_grad_(True)
    bad = [math.nan, math.inf, -math.inf]
    idx = torch.tensor([[b, 3.5] for b in bad] + [[3.5, b] for b in bad] + [[math.nan, math.inf], [2.25, 3.75]],
                       device=DEV).requires_grad_(True)
    out = dirt.sample_texture(tex, idx, mode=mode)
    assert not out[:-1].any() and torch.isfinite(out).all()
    assert _bits_equal(out[-1], ex.sample_texture(tex.detach(), idx.detach()[-1:], mode=mode)[0])
    out[:-1].sum().backward()
    assert not tex.grad.any() and not idx.grad.any()


def _abi_call(L, fn, *args):
    return getattr(L, fn)(*[ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else
                            (ctypes.c_void_p(0) if a is None else a) for a in args],
                          ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))


@pytest.mark.parametrize('C', [1, 2, 3, 4, 5])
def test_four_byte_aligned_buffers_take_the_scalar_paths(cuda_lib, C):
    L = cuda_lib
    H, W, N = 19, 13, 3000
    tex = torch.rand(H, W, C, generator=_gen(20), device=DEV)
    idx = _indices(H, W, N - 78, 21)
    gout = torch.randn(N, C, generator=_gen(22), device=DEV)

    def run(offset):
        def place(t):   # t's values in a buffer that starts `offset` floats past a 256-byte boundary
            buf = torch.zeros(t.numel() + 8, device=DEV)
            buf[offset:offset + t.numel()] = t.reshape(-1)
            return buf[offset:offset + t.numel()]
        tx, ix, go = place(tex), place(idx), place(gout)
        out, gt, gi = place(torch.zeros(N * C, device=DEV)), place(torch.zeros(H * W * C, device=DEV)), place(torch.zeros(N * 2, device=DEV))
        assert _abi_call(L, 'dirt_texture_sample', tx, ix, out, 1, H, W, C, 1, N, 0) == 0
        assert L.dirt_last_launch_count() == 1
        assert _abi_call(L, 'dirt_texture_sample_backward', tx, ix, go, gt, gi, 1, H, W, C, 1, N, 0) == 0
        assert L.dirt_last_launch_count() == 1
        return out.clone(), gt.clone(), gi.clone()

    aligned, unaligned = run(0), run(1)
    assert _bits_equal(aligned[0], unaligned[0]) and _bits_equal(aligned[2], unaligned[2])
    assert rel_close(unaligned[1].cpu().numpy(), aligned[1].cpu().numpy())[0]


def test_non_contiguous_inputs(ex):
    import dirt_b200 as dirt
    big = torch.rand(40, 30, 6, generator=_gen(23), device=DEV)
    tex = big.transpose(0, 1)[:, ::2, 1:4]                      # [30, 20, 3], strided
    idx = _indices(30, 20, 4000 - 78, 24).reshape(100, 40, 2).transpose(0, 1)[:, ::3]
    assert not tex.is_contiguous() and not idx.is_contiguous()
    assert _bits_equal(dirt.sample_texture(tex, idx), ex.sample_texture(tex, idx))
    _check_grads(ex, tex, idx, 'bilinear', 25, 'non-contiguous')


def test_no_lookups():
    import dirt_b200 as dirt
    tex = torch.rand(5, 6, 3, device=DEV, requires_grad=True)
    idx = torch.zeros(0, 2, device=DEV, requires_grad=True)
    out = dirt.sample_texture(tex, idx)
    assert out.shape == (0, 3)
    out.sum().backward()
    assert tex.grad is not None and not tex.grad.any() and idx.grad.shape == (0, 2)
    # per-item textures with B = 0, and with N = 0 lookups per item
    assert dirt.sample_texture(torch.rand(0, 5, 6, 3, device=DEV), torch.zeros(0, 4, 2, device=DEV)).shape == (0, 4, 3)
    t = torch.rand(2, 5, 6, 3, device=DEV, requires_grad=True)
    out = dirt.sample_texture(t, torch.zeros(2, 0, 2, device=DEV))
    assert out.shape == (2, 0, 3)
    out.sum().backward()
    assert not t.grad.any()


def _textured_cube(ex, sample, texture_size=64):
    import dirt_b200 as dirt
    from dirt_b200 import lighting, matrices
    vertices, uvs, faces = ex.build_cube()
    vertices_object = torch.tensor(vertices, dtype=torch.float32, device=DEV)
    uvs = torch.tensor(uvs, dtype=torch.float32, device=DEV)
    faces = torch.tensor(faces, dtype=torch.int32, device=DEV)
    texture = ex.checker_texture(size=texture_size, device=DEV)
    texture = (texture + 0.1 * torch.rand(texture.shape, generator=_gen(26), device=DEV)).requires_grad_(True)
    light_direction = torch.tensor([1., 0., 0.], device=DEV, requires_grad=True)
    vertices_object = torch.cat([vertices_object, torch.ones_like(vertices_object[:, -1:])], dim=1).requires_grad_(True)
    vertices_world = vertices_object @ matrices.rodrigues([0., 0.6, 0.]).to(DEV)
    normals_world = lighting.vertex_normals(vertices_world, faces)
    view = matrices.compose(matrices.translation([0., -2., -3.2]), matrices.rodrigues([-0.5, 0., 0.])).to(DEV)
    proj = matrices.perspective_projection(near=0.1, far=20., right=0.1, aspect=120. / 160.).to(DEV)
    attributes = torch.cat([torch.ones_like(uvs[:, :1]), uvs, normals_world], dim=1)
    pixels = dirt.rasterise_deferred(torch.zeros([120, 160, 6], device=DEV), vertices_world @ view @ proj, attributes, faces,
                                     functools.partial(ex.shader_fn, sample=sample), [texture, light_direction])
    weights = torch.rand(pixels.shape, generator=_gen(27), device=DEV)
    (pixels * weights).sum().backward()
    return pixels.detach(), vertices_object.grad, texture.grad, light_direction.grad


def test_textured_cube_through_rasterise_deferred(ex):
    import dirt_b200 as dirt
    px_cuda, *grads_cuda = _textured_cube(ex, dirt.sample_texture)
    px_torch, *grads_torch = _textured_cube(ex, ex.sample_texture)
    assert _bits_equal(px_cuda, px_torch)
    assert float((px_cuda != torch.tensor([0., 0., 0.3], device=DEV)).any(-1).float().mean()) > 0.1   # the cube is in view
    for name, a, b in zip(['vertices', 'texture', 'light'], grads_cuda, grads_torch):
        ok, ratio = rel_close(a.cpu().numpy(), b.cpu().numpy(), name='textured cube grad_' + name)
        assert ok, (name, ratio)


def test_cuda_graph_capture_and_replay():
    import dirt_b200 as dirt
    tex = torch.rand(64, 48, 4, generator=_gen(28), device=DEV).requires_grad_(True)
    idx = _indices(64, 48, 100000, 29).requires_grad_(True)
    gout = torch.randn(idx.shape[0], 4, generator=_gen(30), device=DEV)

    def step():
        tex.grad, idx.grad = None, None
        out = dirt.sample_texture(tex, idx)
        (out * gout).sum().backward()
        return out

    eager = step().detach().clone()
    eager_gt, eager_gi = tex.grad.clone(), idx.grad.clone()
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        step()   # warm-up on the capture stream
    torch.cuda.current_stream(DEV).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert _bits_equal(out, eager) and _bits_equal(idx.grad, eager_gi)
        assert rel_close(tex.grad.cpu().numpy(), eager_gt.cpu().numpy())[0]
