"""GPU: sample_texture(mode='trilinear') against the torch restatement in tests/texture_mip_restatement.py.

The pyramid, every lookup whose footprint is at most one texel and every lookup at an exact power-of-two footprint are
compared bit for bit; the general lookup and both gradients against torch autograd of the restatement in float64, with
conftest.rel_close (1e-4 relative).  The deterministic backward pass is checked for bit-identical repeats, CUDA graph
replay and item independence."""
import ctypes
import math

import pytest
import torch

import texture_mip_restatement as mip
from conftest import rel_close
from test_gpu_texture import _indices, _textured_cube, _uv_indices

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
ex = mip._ex


@pytest.fixture(autouse=True)
def _needs_the_library(cuda_lib):
    return cuda_lib


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def _pyramid(L, tex):
    """dirt_texture_mip_build of tex [TB, TH, TW, C] -> the flat pyramid (None for one level)."""
    TB, TH, TW, C = tex.shape
    n = L.dirt_texture_mip_pyramid_bytes(TB, TH, TW, C) // 4
    pyr = torch.full((n,), float('nan'), device=DEV) if n else None
    assert L.dirt_texture_mip_build(_p(tex), _p(pyr), TB, TH, TW, C, _stream()) == 0
    assert L.dirt_last_launch_count() == mip.level_count(TH, TW) - 1
    return pyr


@pytest.mark.parametrize('C', [1, 2, 3, 4, 5, 8])
def test_pyramid_is_bit_identical_to_the_restatement(cuda_lib, C):
    for k, (TH, TW) in enumerate([(1, 1), (2, 1), (6, 10), (640, 480), (1024, 512), (256, 256)]):
        for TB in (1, 3):
            tex = torch.rand(TB, TH, TW, C, generator=_gen(k), device=DEV) * 2 - 0.5
            pyr = _pyramid(cuda_lib, tex)
            want = [t.reshape(-1) for t in mip.pyramid(tex)[1:]]
            if not want:
                assert pyr is None
                continue
            assert _bits_equal(pyr, torch.cat(want)), (TB, TH, TW, C)


SHAPES = [(1, 1), (1, 7), (5, 7), (2, 2), (6, 10), (64, 48), (256, 256), (1024, 1024)]


def _index_sets(H, W, seed):
    return (_indices(H, W, 3000, seed), _uv_indices(H, W, 'repeat', seed + 1), _uv_indices(H, W, 'clamp', seed + 2))


@pytest.mark.parametrize('C', [1, 3, 4, 5])
def test_footprints_of_at_most_one_texel_are_the_bilinear_lookup(C):
    import dirt_b200 as dirt
    for k, (H, W) in enumerate(SHAPES):
        tex = torch.rand(H, W, C, generator=_gen(k), device=DEV)
        for idx in _index_sets(H, W, 100 + 10 * k):
            n = idx.shape[0]
            small = (torch.rand(n, 4, generator=_gen(k + 50), device=DEV) * 1.4 - 0.7)       # rho^2 < 1
            small[: n // 8] = 0.
            small[n // 8: n // 4, 1] = float('nan')
            small[n // 4: n // 4 + 16] = torch.tensor([1., 0., 0., 1.], device=DEV)          # rho = 1 exactly
            want = dirt.sample_texture(tex, idx, mode='bilinear')
            got = dirt.sample_texture(tex, idx, mode='trilinear', derivatives=small)
            assert _bits_equal(got, want), (H, W, C, int((got != want).sum()))


@pytest.mark.parametrize('C', [1, 3, 4, 5])
def test_power_of_two_footprints_read_one_level_exactly(C):
    import dirt_b200 as dirt
    for k, (H, W) in enumerate(SHAPES):
        tex = torch.rand(H, W, C, generator=_gen(k), device=DEV)
        levels = mip.pyramid(tex)
        for idx in _index_sets(H, W, 200 + 10 * k):
            for l in range(len(levels)):
                rho = float(2 ** l)
                der = torch.tensor([0., rho, rho / 2, 0.], device=DEV).expand(idx.shape[0], 4)
                got = dirt.sample_texture(tex, idx, mode='trilinear', derivatives=der)
                want = ex.sample_texture(levels[l], mip.level_index(idx, l))
                assert _bits_equal(got, want), (H, W, C, l)


def _random_derivatives(n, L, seed):
    """lambda uniform in [-2, L+2] along a random direction, the other axis shorter; then +-inf and NaN entries."""
    g = _gen(seed)
    lam = torch.rand(n, generator=g, device=DEV) * (L + 4) - 2
    ang = torch.rand(n, generator=g, device=DEV) * 2 * math.pi
    rho = 2.0 ** lam
    short = rho * torch.rand(n, generator=g, device=DEV)
    der = torch.stack([rho * torch.cos(ang), rho * torch.sin(ang), -short * torch.sin(ang), short * torch.cos(ang)], -1)
    swap = torch.rand(n, generator=g, device=DEV) < 0.5
    der = torch.where(swap[:, None], der[:, [2, 3, 0, 1]], der)
    der[:8, 0] = float('inf')
    der[8:16, 3] = -float('inf')
    der[16:24, 2] = float('nan')
    return der.contiguous()


def _reference(tex, idx, der, grad_out):
    """forward and torch autograd of the restatement in float64, at the levels and level texels the float32 lookup
    picks (lambda from the float32 derivatives; each level's index mapped in float32, its gradient 2^-k)."""
    t = tex.detach().double().requires_grad_(True)
    i = idx.detach().double().requires_grad_(True)

    def index_of(safe, k):
        if k == 0:
            return safe
        exact = safe * 2.0 ** -k
        return exact + (mip.level_index(safe.detach().float(), k).double() - exact.detach())

    out = mip.sample(t, i, der, index_of=index_of)
    (out * grad_out.double()).sum().backward()
    return out.detach(), t.grad, i.grad


def _check(tex, idx, der, seed, tag, deterministic=False):
    import dirt_b200 as dirt
    grad_out = torch.randn(idx.shape[:-1] + (tex.shape[-1],), generator=_gen(seed), device=DEV)
    t, i = tex.clone().requires_grad_(True), idx.clone().requires_grad_(True)
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        out = dirt.sample_texture(t, i, mode='trilinear', derivatives=der)
        (out * grad_out).sum().backward()
    finally:
        torch.use_deterministic_algorithms(before)
    ref_out, ref_t, ref_i = _reference(tex, idx, der, grad_out)
    label = 'trilinear det' if deterministic else 'trilinear'
    for name, a, b in (('out', out.detach(), ref_out), ('grad_texture', t.grad, ref_t), ('grad_indices', i.grad, ref_i)):
        ok, ratio = rel_close(a.cpu().numpy(), b.cpu().numpy(), name=label + ' ' + name)
        assert ok, (tag, name, ratio)
    return t.grad, i.grad


@pytest.mark.parametrize('deterministic', [False, True])
@pytest.mark.parametrize('C', [1, 2, 3, 4, 5])
def test_random_footprints_match_autograd_of_the_restatement(C, deterministic):
    for k, (H, W) in enumerate([(5, 7), (2, 2), (6, 10), (64, 48), (256, 256), (1024, 1024)]):
        tex = torch.rand(H, W, C, generator=_gen(k), device=DEV)
        L = mip.level_count(H, W)
        for j, idx in enumerate(_index_sets(H, W, 300 + 10 * k)):
            bad = idx.clone()
            bad[-40:-30, 0] = float('nan')
            bad[-30:-20, 1] = float('inf')
            der = _random_derivatives(idx.shape[0], L, 400 + 10 * k + j)
            _check(tex, bad, der, 500 + k, (H, W, C, j), deterministic)


def test_per_item_textures_and_batched_indices():
    B, H, W, C = 3, 32, 24, 3
    tex = torch.rand(B, H, W, C, generator=_gen(60), device=DEV)
    idx = torch.stack([_indices(H, W, 1000 - 78, 61 + b) for b in range(B)]).reshape(B, 2, -1, 2)
    der = _random_derivatives(idx[..., 0].numel(), mip.level_count(H, W), 62).reshape(idx.shape[:-1] + (4,))
    _check(tex, idx, der, 63, 'per-item')
    _check(tex[0], idx, der, 64, 'shared, batched')


def _det_grad(tex, idx, der, gout, deterministic=True):
    import dirt_b200 as dirt
    t = tex.clone().requires_grad_(True)
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        (dirt.sample_texture(t, idx, mode='trilinear', derivatives=der) * gout).sum().backward()
    finally:
        torch.use_deterministic_algorithms(before)
    return t.grad


def test_deterministic_backward_repeats_and_item_independence():
    B, H, W, C = 4, 64, 32, 3
    tex = torch.rand(B, H, W, C, generator=_gen(70), device=DEV)
    n = 20000
    idx = torch.stack([_indices(H, W, n - 78, 71 + b) for b in range(B)])
    der = _random_derivatives(B * idx.shape[1], mip.level_count(H, W), 75).reshape(B, -1, 4)
    gout = torch.randn(B, idx.shape[1], C, generator=_gen(76), device=DEV)
    first = _det_grad(tex, idx, der, gout)
    assert _bits_equal(first, _det_grad(tex, idx, der, gout))
    for b in range(B):
        alone = _det_grad(tex[b:b + 1], idx[b:b + 1], der[b:b + 1], gout[b:b + 1])
        assert _bits_equal(alone[0], first[b]), b
    shared = tex[0]
    one = _det_grad(shared, idx, der, gout)
    assert _bits_equal(one, _det_grad(shared, idx, der, gout))


def test_deterministic_backward_under_graph_replay(cuda_lib):
    L = cuda_lib
    TB, H, W, C, N = 1, 128, 64, 4, 100000
    tex = torch.rand(TB, H, W, C, generator=_gen(80), device=DEV)
    idx = _indices(H, W, N - 78, 81)[None].contiguous()
    der = _random_derivatives(N, mip.level_count(H, W), 82)[None].contiguous()
    gout = torch.randn(1, N, C, generator=_gen(83), device=DEV)
    pyr = _pyramid(L, tex)
    nbytes = L.dirt_texture_sample_trilinear_backward_bytes(TB, H, W, C, 1, N, 1)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    gt, gi = torch.empty_like(tex), torch.empty_like(idx)

    def call():
        return L.dirt_texture_sample_trilinear_backward(_p(tex), _p(pyr), _p(idx), _p(der), _p(gout), _p(gt), _p(gi), TB, H,
                                                        W, C, 1, N, 1, _p(scratch), nbytes, _stream())

    assert call() == 0
    want_t, want_i = gt.clone(), gi.clone()
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        assert call() == 0
    torch.cuda.current_stream(DEV).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        assert call() == 0
    for _ in range(2):
        scratch.fill_(0xFF)
        gt.fill_(float('nan'))
        graph.replay()
        torch.cuda.synchronize()
        assert _bits_equal(gt, want_t) and _bits_equal(gi, want_i)


def test_textured_cube_with_index_derivatives():
    import dirt_b200 as dirt

    def trilinear(texture, indices):
        return dirt.sample_texture(texture, indices, mode='trilinear',
                                   derivatives=dirt.index_derivatives(indices, texture.shape[:2]))

    px_bi, *grads_bi = _textured_cube(ex, dirt.sample_texture, texture_size=256)
    px_tri, *grads_tri = _textured_cube(ex, trilinear, texture_size=256)
    for g in grads_tri:
        assert g is not None and torch.isfinite(g).all()
    touched_bi = int((grads_bi[1].abs().sum(-1) > 0).sum())
    touched_tri = int((grads_tri[1].abs().sum(-1) > 0).sum())
    # the top and bottom faces tile the 256^2 checker twice over a few dozen pixels: bilinear reaches a sparse subset
    assert touched_tri > touched_bi, (touched_tri, touched_bi)
