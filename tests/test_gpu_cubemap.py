"""GPU: dirt_b200.sample_cubemap against the torch restatement of tests/cubemap_restatement.py.

Forward values are compared bit for bit with the float32 restatement on the same device; gradients against torch
autograd of the restatement in float64, with conftest.rel_close (1e-4 relative)."""
import ctypes
import importlib.util
import itertools
import math
import os

import numpy as np
import pytest
import torch

import cubemap_restatement as cm
from conftest import rel_close

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device('cuda', 0)


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _directions(n, seed, S=4):
    """n random directions (normal, so uniform on the sphere, at random lengths), then the special ones: face centres,
    points on and beside the 12 edges and 8 corners, exact ties, texel edges of an S-texel face, zero and non-finite."""
    g = _gen(seed)
    rnd = torch.randn(n, 3, generator=g, device=DEV) * torch.rand(n, 1, generator=g, device=DEV).add(0.01) * 10
    special = [[1., 0., 0.], [0., -2., 0.], [0., 0., 3.], [1., 1., 1.], [-1., 1., -1.], [1., -1., 0.], [0., 1., 1.],
               [2., 2., 0.5], [-0.5, 3., -3.], [1., 1e-7, 1e-7], [1., -1e-7, 1e-7]]
    for a, b in itertools.combinations(range(3), 2):
        for sa, sb, t in itertools.product((-1., 1.), (-1., 1.), (0., 0.3, -0.99)):
            for e in (0., 1e-6, -1e-6):
                v = [0., 0., 0.]
                v[a], v[b], v[3 - a - b] = sa, sb * (1 + e), t
                special.append(v)
    for corner in itertools.product((-1., 1.), repeat=3):
        special.append(list(corner))
        special.append([corner[0], corner[1] * (1 - 1e-6), corner[2] * (1 + 1e-6)])
    for k in range(S + 1):   # texel edges and centres along one face's axis
        special += [[1., 0.3, 2. * k / S - 1.], [1., 0.3, 2. * (k + 0.5) / S - 1.]]
    special += [[0., 0., 0.], [-0., 0., 0.], [math.nan, 1., 0.], [math.inf, 0., 0.], [1., -math.inf, 2.]]
    return torch.cat([rnd, torch.tensor(special, device=DEV)])


def _cubemap(S, C, seed, batch=None):
    shape = (6, S, S, C) if batch is None else (batch, 6, S, S, C)
    return torch.rand(shape, generator=_gen(seed), device=DEV) * 2 - 0.5


SIZES = [1, 2, 3, 64]


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [1, 2, 3, 4, 5, 8])
def test_forward_is_bit_identical_to_the_restatement(cuda_lib, mode, C):
    import dirt_b200 as dirt
    for k, S in enumerate(SIZES):
        cube = _cubemap(S, C, k)
        d = _directions(5000, 100 + k, S)
        assert _bits_equal(dirt.sample_cubemap(cube, d, mode), cm.sample(cube, d, mode)), (S, C, mode)
        cubes = _cubemap(S, C, 10 + k, batch=3)
        d = torch.stack([_directions(1000, 200 + k + b, S) for b in range(3)])
        assert _bits_equal(dirt.sample_cubemap(cubes, d, mode), cm.sample(cubes, d, mode)), (S, C, mode, 'per item')


def _reference_coords(x64, x32, S, mode):
    """(face, s, t, valid) of the float64 restatement, with s and t moved onto the float32 evaluation's lookup: the
    float32 padded (row, col) of a bilinear lookup, the float32 (t, s) of a nearest one, each with the float64 derivative
    (as texture_mip_restatement's float64 comparisons pass the float32 indices).  The fp32 rounding of the coordinates,
    about S * 2^-24 texels, is the forward's specification, not an error of the gradients."""
    face, s, t, valid = cm.face_coords(x64)
    _, s32, t32, _ = cm.face_coords(x32)
    if mode == 'bilinear':
        s_val = (((s32 * S - 0.5) + 1.).double() - 0.5) / S
        t_val = (((t32 * S - 0.5) + 1.).double() - 0.5) / S
    else:
        s_val, t_val = s32.double(), t32.double()
    return face, s + (s_val - s).detach(), t + (t_val - t).detach(), valid


def _reference_grads(cube, d, grad_out, mode):
    """torch autograd of the restatement in float64 at the float32 lookup (_reference_coords); its gathers' adjoints are
    scatter-adds, so it runs outside the deterministic mode of the op under test."""
    c = cube.detach().double().requires_grad_(True)
    x = d.detach().double().requires_grad_(True)
    S = cube.shape[-2]

    def run(c, x, x32):
        if c.dim() == 5:
            return torch.stack([run(c[b], x[b], x32[b]) for b in range(c.shape[0])])
        return cm.sample_padded(cm.atlas(c), *_reference_coords(x, x32, S, mode), mode)

    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(False)
    try:
        (run(c, x, d.detach().float()) * grad_out.double()).sum().backward()
    finally:
        torch.use_deterministic_algorithms(before)
    return c.grad, (x.grad if x.grad is not None else torch.zeros_like(x))


def _close(actual, expected, name):
    a, b = actual.cpu().numpy(), expected.cpu().numpy()
    if b.size and np.abs(b).max() < 1e-12:
        return bool(np.abs(a).max() < 1e-12), 0.0
    return rel_close(a, b, name=name)


def _same_taps(d, S, mode):
    """Lookups that the float32 evaluation and _reference_coords place on the same texels, off a texel boundary.  On a
    boundary (such as the texel-edge cases of _directions) the nearest texel, and the bilinear derivative along the
    boundary's normal, jump, and the two may take different sides: such lookups are compared with a zero grad_out."""
    x32 = d.detach().float()
    with torch.no_grad():
        face, s, t, valid = _reference_coords(x32.double(), x32, S, mode)
        _, s32, t32, _ = cm.face_coords(x32)
    if mode == 'nearest':
        return ((t32 * S).floor() == (t * S).floor()) & ((s32 * S).floor() == (s * S).floor())
    pr32, pc32 = (t32 * S - 0.5) + 1., (s32 * S - 0.5) + 1.
    pr, pc = (t * S - 0.5) + 1., (s * S - 0.5) + 1.
    return ((pr32.floor() == pr.floor()) & (pc32.floor() == pc.floor()) & (pr32 != pr32.floor()) &
            (pc32 != pc32.floor()))


def _check_grads(cube, d, mode, seed, tag, want=(True, True), label='cubemap', positive=False):
    import dirt_b200 as dirt
    shape = d.shape[:-1] + (cube.shape[-1],)
    grad_out = (torch.rand(shape, generator=_gen(seed), device=DEV) + 0.5 if positive else
                torch.randn(shape, generator=_gen(seed), device=DEV))
    same = _same_taps(d, cube.shape[-2], mode)
    assert float(same.float().mean()) > 0.9, tag   # the special directions of _directions sit on boundaries
    grad_out = grad_out * same[..., None]
    c = cube.detach().clone().requires_grad_(want[0])
    x = d.detach().clone().requires_grad_(want[1])
    (dirt.sample_cubemap(c, x, mode) * grad_out).sum().backward()
    ref_c, ref_x = _reference_grads(cube, d, grad_out, mode)
    if want[0]:
        ok, ratio = _close(c.grad, ref_c, label + ' grad_cubemap')
        assert ok, (tag, 'grad_cubemap', ratio)
    else:
        assert c.grad is None
    if want[1]:
        if mode == 'nearest':
            assert not x.grad.any()
        else:
            ok, ratio = _close(x.grad, ref_x, label + ' grad_directions')
            assert ok, (tag, 'grad_directions', ratio)
    else:
        assert x.grad is None
    return c.grad, x.grad


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [1, 3, 4, 5])
def test_backward_matches_autograd_of_the_restatement(cuda_lib, mode, C):
    for k, S in enumerate(SIZES):
        _check_grads(_cubemap(S, C, 20 + k), _directions(5000, 300 + k, S), mode, 400 + k, (S, C))
        d = torch.stack([_directions(800, 500 + k + b, S) for b in range(2)])
        _check_grads(_cubemap(S, C, 30 + k, batch=2), d, mode, 600 + k, (S, C, 'per item'))


@pytest.mark.parametrize('want', [(True, False), (False, True), (True, True)])
@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
def test_backward_for_every_needs_input_grad(cuda_lib, want, mode):
    _check_grads(_cubemap(5, 3, 40), _directions(20000, 41, 5), mode, 42, want, want)


def _corner_directions(n, seed):
    """n lookups within a few texels of the (+1, +1, +1) corner of a 16-texel cube map: three faces, shared texels."""
    return torch.tensor([1., 1., 1.], device=DEV) + 0.1 * torch.randn(n, 3, generator=_gen(seed), device=DEV)


@pytest.mark.parametrize('C', [1, 3, 4, 6])
def test_backward_under_contention(cuda_lib, C):
    cube = _cubemap(16, C, 43)
    d = _corner_directions(1 << 20, 44)
    _check_grads(cube, d, 'bilinear', 45, ('corner', C), label='cubemap contention', positive=True)
    _check_grads(cube, d, 'nearest', 46, ('corner nearest', C), label='cubemap contention', positive=True)


@pytest.fixture
def deterministic():
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(before)


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [1, 3, 4, 5])
def test_deterministic_gradient(cuda_lib, deterministic, mode, C):
    """Within the bar of float64 autograd, bit-identical on a repeat, and with per-item maps an item alone gives the
    same bits as inside the batch."""
    import dirt_b200 as dirt
    for k, S in enumerate([1, 3, 64]):
        cube, d = _cubemap(S, C, 50 + k), _directions(20000, 51 + k, S)
        g1 = _check_grads(cube, d, mode, 52 + k, (S, C, 'det'), label='cubemap deterministic')
        g2 = _check_grads(cube, d, mode, 52 + k, (S, C, 'det'), label='cubemap deterministic')
        assert _bits_equal(g1[0], g2[0]) and _bits_equal(g1[1], g2[1])
    cube = _cubemap(16, C, 55)
    _check_grads(cube, _corner_directions(1 << 18, 56), mode, 57, ('det corner', C), label='cubemap deterministic',
                 positive=True)
    cubes = _cubemap(8, C, 58, batch=3)
    d = torch.stack([_directions(3000, 59 + b, 8) for b in range(3)])
    gout = torch.randn(3, d.shape[1], C, generator=_gen(60), device=DEV)

    def grad(c, x, g):
        c = c.clone().requires_grad_(True)
        (dirt.sample_cubemap(c, x, mode) * g).sum().backward()
        return c.grad

    whole = grad(cubes, d, gout)
    for b in range(3):
        assert _bits_equal(grad(cubes[b:b + 1], d[b:b + 1], gout[b:b + 1])[0], whole[b]), b


def test_deterministic_gradient_under_graph_replay(cuda_lib, deterministic):
    import dirt_b200 as dirt
    cube = _cubemap(32, 3, 61).requires_grad_(True)
    d = _directions(100000, 62, 32).requires_grad_(True)
    gout = torch.randn(d.shape[0], 3, generator=_gen(63), device=DEV)

    def step():
        cube.grad, d.grad = None, None
        out = dirt.sample_cubemap(cube, d)
        (out * gout).sum().backward()
        return out

    eager = step().detach().clone()
    eager_gc, eager_gd = cube.grad.clone(), d.grad.clone()
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream(DEV).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert _bits_equal(out, eager) and _bits_equal(d.grad, eager_gd) and _bits_equal(cube.grad, eager_gc)


def _abi(L, fn, *args):
    return getattr(L, fn)(*[ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else
                            (ctypes.c_void_p(0) if a is None else a) for a in args],
                          ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))


@pytest.mark.parametrize('C', [1, 2, 3, 4, 5])
def test_four_byte_aligned_buffers_take_the_scalar_paths(cuda_lib, C):
    L = cuda_lib
    S, N = 7, 3000
    cube = _cubemap(S, C, 64)
    d = _directions(N - 135, 65, S)
    N = d.shape[0]
    gout = torch.randn(N, C, generator=_gen(66), device=DEV)
    atlas_floats = int(L.dirt_cubemap_atlas_bytes(1, S, C)) // 4

    def run(offset, det):
        def place(t):
            buf = torch.zeros(t.numel() + 8, device=DEV)
            buf[offset:offset + t.numel()] = t.reshape(-1)
            return buf[offset:offset + t.numel()]
        cx, dx, go = place(cube), place(d), place(gout)
        atlas, out = place(torch.zeros(atlas_floats, device=DEV)), place(torch.zeros(N * C, device=DEV))
        gc, gd = place(torch.zeros(cube.numel(), device=DEV)), place(torch.zeros(N * 3, device=DEV))
        nbytes = int(L.dirt_cubemap_sample_backward_bytes(1, S, C, 1, N, 0, det))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        assert _abi(L, 'dirt_cubemap_sample', cx, dx, atlas, out, 1, S, C, 1, N, 0) == 0
        assert L.dirt_last_launch_count() == 2
        assert _abi(L, 'dirt_cubemap_sample_backward', atlas, dx, go, gc, gd, 1, S, C, 1, N, 0, det, scratch,
                    ctypes.c_size_t(nbytes)) == 0
        return out.clone(), gc.clone(), gd.clone()

    for det in (0, 1):
        aligned, unaligned = run(0, det), run(1, det)
        assert _bits_equal(aligned[0], unaligned[0]) and _bits_equal(aligned[2], unaligned[2])
        if det:
            assert _bits_equal(aligned[1], unaligned[1])
        else:
            assert rel_close(unaligned[1].cpu().numpy(), aligned[1].cpu().numpy())[0]
    assert _bits_equal(aligned[0].reshape(N, C), cm.sample(cube, d))


def test_non_contiguous_inputs(cuda_lib):
    import dirt_b200 as dirt
    big = torch.rand(6, 12, 12, 6, generator=_gen(67), device=DEV)
    cube = big[:, :, :, 1:4]                                        # [6, 12, 12, 3], strided
    d = _directions(3000, 68, 12)
    d = torch.cat([d, d], -1)[:, 1:4]                              # strided rows
    assert not cube.is_contiguous() and not d.is_contiguous()
    assert _bits_equal(dirt.sample_cubemap(cube, d), cm.sample(cube, d))
    _check_grads(cube, d, 'bilinear', 69, 'non-contiguous')


def test_no_lookups(cuda_lib):
    import dirt_b200 as dirt
    cube = torch.rand(6, 4, 4, 3, device=DEV, requires_grad=True)
    d = torch.zeros(0, 3, device=DEV, requires_grad=True)
    out = dirt.sample_cubemap(cube, d)
    assert out.shape == (0, 3)
    out.sum().backward()
    assert cube.grad is not None and not cube.grad.any() and d.grad.shape == (0, 3)
    assert dirt.sample_cubemap(torch.rand(0, 6, 4, 4, 3, device=DEV), torch.zeros(0, 5, 3, device=DEV)).shape == (0, 5, 3)


def test_lookups_past_the_grid_cap_run_a_second_round(cuda_lib):
    """2^24 + 4099 lookups: past the 2^16 CTAs x 256 threads of one round of the forward and backward loops."""
    import dirt_b200 as dirt
    n = (1 << 24) + 4099
    cube = _cubemap(8, 1, 70)
    d = torch.randn(n, 3, generator=_gen(71), device=DEV)
    x = d.clone().requires_grad_(True)
    out = dirt.sample_cubemap(cube, x)
    assert _bits_equal(out, cm.sample(cube, d))
    gout = torch.randn(n, 1, generator=_gen(72), device=DEV)
    (out * gout).sum().backward()
    tail = d[-4099:].clone().requires_grad_(True)
    (dirt.sample_cubemap(cube, tail) * gout[-4099:]).sum().backward()
    assert _bits_equal(x.grad[-4099:], tail.grad)


# ---- through the deferred rasteriser ---------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def env(cuda_lib):
    spec = importlib.util.spec_from_file_location('environment_example', os.path.join(ROOT, 'examples', 'environment.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_environment_through_rasterise_batch_deferred(env):
    """A batch of mirror-and-diffuse spheres over a cube-map background: pixels and gradients finite, the sphere and
    the background in view, and the cube-map gradient reaching both the background's and the reflection's texels."""
    import dirt_b200 as dirt
    B = 2
    cube = env.procedural_cubemap(32, device=DEV).expand(B, -1, -1, -1, -1).contiguous().requires_grad_(True)
    pixels = env.render(cube, dirt.rasterise_batch_deferred, dirt.sample_cubemap, batch=B, width=160, height=120,
                        device=DEV)
    weights = torch.rand(pixels.shape, generator=_gen(73), device=DEV)
    (pixels * weights).sum().backward()
    assert torch.isfinite(pixels).all() and torch.isfinite(cube.grad).all()
    assert int((cube.grad.abs().sum(-1) > 0).sum()) > 0.2 * cube.grad[..., 0].numel()
    # the same image with the float32 restatement as the lookup
    ref = env.render(cube.detach(), dirt.rasterise_batch_deferred, cm.sample, batch=B, width=160, height=120, device=DEV)
    assert _bits_equal(pixels.detach(), ref)


FIT_STEPS = 100


def test_fitting_a_cube_map_through_the_rasteriser(env):
    """Per-item cube maps fitted with Adam from a constant grey to images rendered with known ones; the masked loss
    (background and sphere) must fall at least 10x."""
    import dirt_b200 as dirt
    B, S = 2, 16
    truth = torch.stack([env.procedural_cubemap(S, device=DEV), env.procedural_cubemap(S, device=DEV).flip(-1)])
    with torch.no_grad():
        target = env.render(truth, dirt.rasterise_batch_deferred, dirt.sample_cubemap, batch=B, width=128, height=96,
                            device=DEV)
    cube = torch.full((B, 6, S, S, 3), 0.5, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([cube], lr=0.05)
    losses = []
    for _ in range(FIT_STEPS):
        opt.zero_grad()
        pixels = env.render(cube, dirt.rasterise_batch_deferred, dirt.sample_cubemap, batch=B, width=128, height=96,
                            device=DEV)
        loss = ((pixels - target) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    ratio = losses[0] / losses[-1]
    print('cube-map fit: loss %.3e -> %.3e (ratio %.1f) after %d steps' % (losses[0], losses[-1], ratio, FIT_STEPS))
    assert ratio > 10., losses[::10]
