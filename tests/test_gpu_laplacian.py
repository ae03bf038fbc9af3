"""GPU: the mesh Laplacian's CUDA path (`mesh.laplacian`) against its torch restatement (`mesh._vertex_laplacian`).

Forward values and gradients against float64 autograd of the restatement, with conftest.rel_close (1e-4), in both
modes, on a noisy icosphere, on cfg5's uv-sphere (poles of valence 224: the whole-warp row path) and on an open grid
with a boundary."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

import variant_builds
from conftest import rel_close

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device('cuda', 0)
MODES = ['uniform', 'cotangent']


@pytest.fixture(scope='module')
def mesh(cuda_lib):
    from dirt_b200 import mesh
    return mesh


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _icosphere():
    from dirt_b200 import scenes
    v, f = scenes.icosphere(3)
    r = np.random.default_rng(1)
    return (v * (1. + 0.2 * r.standard_normal((v.shape[0], 1)))).astype(np.float32), f


def _uv_sphere():
    from dirt_b200 import scenes
    return scenes.uv_sphere(224, 112, displacement=0.1)


def _grid(n=24):
    """An open, gently curved n x n grid: boundary vertices of valence 2 to 4, interior of valence 6."""
    y, x = np.meshgrid(np.linspace(-1, 1, n), np.linspace(-1, 1, n), indexing='ij')
    z = 0.3 * np.sin(2. * x) * np.cos(1.5 * y)
    v = np.stack([x.ravel(), y.ravel(), z.ravel()], axis=1)
    v[:, :2] += 0.01 * np.random.default_rng(2).standard_normal((n * n, 2))
    q = (np.arange(n - 1)[:, None] * n + np.arange(n - 1)[None, :]).ravel()
    f = np.concatenate([np.stack([q, q + 1, q + n + 1], 1), np.stack([q, q + n + 1, q + n], 1)])
    return v.astype(np.float32), f.astype(np.int32)


MESHES = {'icosphere': _icosphere, 'uv_sphere': _uv_sphere, 'grid': _grid}


def _batch(v, lead, w, seed):
    """[*lead, V, 3 | 4] on the device: the mesh scaled and shifted per item, w = 1 + noise."""
    g = np.random.default_rng(seed)
    n = int(np.prod(lead)) if lead else 1
    items = v[None] * (1. + 0.1 * g.random((n, 1, 1))) + 0.1 * g.standard_normal((n, 1, 3))
    if w:
        items = np.concatenate([items, 1. + g.random(items.shape[:-1] + (1,))], axis=-1)
    return torch.tensor(items, dtype=torch.float32, device=DEV).reshape(lead + items.shape[1:])


def _check(got, want, name):
    assert got.shape == want.shape, (got.shape, want.shape)
    ok, ratio = rel_close(np.asarray(got, np.float64), np.asarray(want, np.float64), name=name)
    assert ok, (name, ratio)


def _grads(fn, x, faces, grad_out, mode):
    leaf = x.detach().clone().requires_grad_(True)
    (fn(leaf, faces, mode) * grad_out).sum().backward()
    return leaf.grad


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('lead', [(), (2,), (2, 3)], ids=['lead0', 'lead1', 'lead2'])
@pytest.mark.parametrize('name', sorted(MESHES))
def test_forward_matches_float64(mesh, name, lead, mode):
    v, f = MESHES[name]()
    faces = torch.tensor(f, device=DEV)
    for w in (False, True):
        x = _batch(v, lead, w, len(lead) + 3 * w)
        got = mesh.laplacian(x, faces, mode)
        assert got.dtype == torch.float32 and got.shape == lead + (v.shape[0], 3)
        _check(got.cpu(), mesh._vertex_laplacian(x.double().cpu(), f, mode), 'laplacian %s fwd vs fp64' % mode)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('name', sorted(MESHES))
def test_gradients_match_float64_autograd(mesh, name, mode):
    v, f = MESHES[name]()
    faces = torch.tensor(f, device=DEV)
    for lead, w in (((), False), ((3,), True)):
        x = _batch(v, lead, w, 7)
        grad_out = torch.randn(lead + (v.shape[0], 3), generator=_gen(8), device=DEV)
        got = _grads(mesh.laplacian, x, faces, grad_out, mode)
        want = _grads(mesh._vertex_laplacian, x.double().cpu(), torch.tensor(f), grad_out.double().cpu(), mode)
        if w:
            assert not got[..., 3].any()
        _check(got.cpu(), want, 'laplacian %s grad vs fp64' % mode)


@pytest.mark.parametrize('mode', MODES)
def test_double_backward(mesh, mode):
    v, f = _icosphere()
    faces = torch.tensor(f, device=DEV)
    x = _batch(v, (2,), True, 10)
    grad_out = torch.randn(2, v.shape[0], 3, generator=_gen(11), device=DEV)
    results = []
    for fn, xx, ff, g in ((mesh.laplacian, x, faces, grad_out),
                          (mesh._vertex_laplacian, x.double().cpu(), torch.tensor(f), grad_out.double().cpu())):
        leaf = xx.detach().clone().requires_grad_(True)
        first, = torch.autograd.grad((fn(leaf, ff, mode) * g).sum(), leaf, create_graph=True)
        # the uniform mode is linear, so its first gradient does not depend on the vertices: the leaf's own term keeps
        # the second backward defined
        (first.square().sum() + leaf.square().sum()).backward()
        results.append((first.detach().cpu(), leaf.grad.cpu()))
    for a, b in zip(*results):
        _check(a, b, 'laplacian %s double backward' % mode)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('dtype', [torch.int32, torch.int64])
def test_invalid_faces_are_left_out(mesh, dtype, mode):
    v, f = _icosphere()
    V = v.shape[0]
    bad = f.astype(np.int64).copy()
    rows = np.arange(5, len(f), 37)
    values = [-1, V, V + 5, -7] + ([(1 << 32) + 3, (1 << 32) + V - 1, -(1 << 32) + 2, (1 << 31)] if dtype == torch.int64 else [])
    for j, r in enumerate(rows):
        bad[r, j % 3] = values[j % len(values)]
    keep = torch.tensor(f[np.setdiff1d(np.arange(len(f)), rows)])
    x = _batch(v, (2,), True, 13)
    grad_out = torch.randn(2, V, 3, generator=_gen(14), device=DEV)
    for faces in (torch.tensor(bad, dtype=dtype, device=DEV), torch.tensor(bad, dtype=dtype)):
        _check(mesh.laplacian(x, faces, mode).cpu(), mesh._vertex_laplacian(x.double().cpu(), keep, mode),
               'laplacian invalid faces fwd')
        _check(_grads(mesh.laplacian, x, faces, grad_out, mode).cpu(),
               _grads(mesh._vertex_laplacian, x.double().cpu(), keep, grad_out.double().cpu(), mode),
               'laplacian invalid faces grad')


@pytest.mark.parametrize('mode', MODES)
def test_empty_inputs(mesh, mode):
    from dirt_b200 import scenes
    _, f = scenes.cube()
    for lead, V, faces in (((2,), 8, np.zeros((0, 3), np.int32)), ((2,), 0, np.zeros((0, 3), np.int32)),
                           ((2,), 0, f), ((0,), 8, f), ((), 8, np.zeros((0, 3), np.int64))):
        x = torch.rand(lead + (V, 4), generator=_gen(15), device=DEV).requires_grad_(True)
        out = mesh.laplacian(x, torch.tensor(faces, device=DEV), mode)
        assert out.shape == lead + (V, 3) and not out.any()
        out.sum().backward()
        assert x.grad.shape == x.shape and not x.grad.any()


@pytest.mark.parametrize('mode', MODES)
def test_a_batch_of_70000_items(mesh, mode):
    from dirt_b200 import scenes
    v, f = scenes.cube()
    x = _batch(v, (70000,), False, 16)
    faces = torch.tensor(f, device=DEV)
    _check(mesh.laplacian(x, faces, mode).cpu(), mesh._vertex_laplacian(x.double(), faces, mode).cpu(),
           'laplacian %s fwd vs fp64' % mode)
    grad_out = torch.randn(x.shape, generator=_gen(17), device=DEV)
    _check(_grads(mesh.laplacian, x, faces, grad_out, mode).cpu(),
           _grads(mesh._vertex_laplacian, x.double(), faces, grad_out.double(), mode).cpu(),
           'laplacian %s grad vs fp64' % mode)


@pytest.mark.parametrize('mode', MODES)
def test_repeated_calls_are_bit_identical(mesh, mode):
    v, f = _uv_sphere()
    faces = torch.tensor(f, device=DEV)
    x = _batch(v, (8,), True, 18)
    grad_out = torch.randn(x.shape[:-1] + (3,), generator=_gen(19), device=DEV)
    runs = []
    for _ in range(3):
        leaf = x.detach().clone().requires_grad_(True)
        out = mesh.laplacian(leaf, faces, mode)
        (out * grad_out).sum().backward()
        runs.append((out.detach(), leaf.grad))
    for out, grad in runs[1:]:
        assert torch.equal(out.view(torch.int32), runs[0][0].view(torch.int32))
        assert torch.equal(grad.view(torch.int32), runs[0][1].view(torch.int32))


@pytest.mark.parametrize('mode', MODES)
def test_cuda_graph_capture_and_replay(mesh, mode):
    v, f = _uv_sphere()
    faces = torch.tensor(f, device=DEV)
    x = _batch(v, (4,), True, 20).requires_grad_(True)
    grad_out = torch.randn(4, v.shape[0], 3, generator=_gen(21), device=DEV)

    def step():
        x.grad = None
        out = mesh.laplacian(x, faces, mode)
        (out * grad_out).sum().backward()
        return out

    eager = step().detach().clone()
    eager_grad = x.grad.clone()
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
        assert torch.equal(out, eager)
        assert torch.equal(x.grad, eager_grad)


@pytest.mark.parametrize('mode', MODES)
def test_no_gradient_wanted_builds_no_node(mesh, cuda_lib, mode):
    v, f = _icosphere()
    x = torch.tensor(v, device=DEV)
    faces = torch.tensor(f, device=DEV)
    out = mesh.laplacian(x, faces, mode)
    assert out.grad_fn is None and not out.requires_grad
    assert cuda_lib.dirt_last_launch_count() == 5      # the adjacency's four kernels and the vertex pass
    k = torch.ones(3, device=DEV, requires_grad=True)
    (mesh.laplacian(x, faces, mode) * k).sum().backward()
    assert cuda_lib.dirt_last_launch_count() == 5 and k.grad is not None


# ---- the C ABI's alignment rule and the grid-stride rounds --------------------------------------------------------------

def _abi_calls(lib, mode, x, faces, grad_out, shift):
    """dirt_laplacian_forward then _backward on buffers that start `shift` floats into their allocations (the workspace
    4 * shift bytes in): (out, grad_vertices) as contiguous copies."""
    B, V, F = x.shape[0], x.shape[1], faces.shape[0]
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    stream = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)

    def shifted(t):
        buf = torch.full((t.numel() + shift,), float('nan'), device=DEV)
        buf[shift:] = t.reshape(-1)
        return buf[shift:]

    rows, g = shifted(x), shifted(grad_out)
    out, grad = shifted(torch.zeros(B * V * 3, device=DEV)), shifted(torch.zeros(B * V * 3, device=DEV))
    ws_bytes = int(lib.dirt_laplacian_workspace_bytes(B, V, F))
    ws = torch.empty(ws_bytes + 4 * shift, dtype=torch.uint8, device=DEV)[4 * shift:]
    assert lib.dirt_laplacian_forward(mesh_mode(mode), p(rows), 3, p(faces), p(out), p(ws), ws_bytes, B, V, F,
                                      stream) == 0
    assert lib.dirt_laplacian_backward(mesh_mode(mode), p(rows), 3, p(faces), p(g), p(grad), p(ws), ws_bytes, B, V, F,
                                       stream) == 0
    torch.cuda.synchronize()
    return out.clone(), grad.clone()


def mesh_mode(mode):
    from dirt_b200 import mesh
    return mesh.MODES[mode]


@pytest.mark.parametrize('mode', MODES)
def test_buffers_aligned_to_4_bytes_only(cuda_lib, mesh, mode):
    """The C ABI asks for 4-byte alignment: every buffer, the workspace included, at 4 bytes past a 16-byte boundary
    gives the results of aligned buffers, bit for bit."""
    v, f = _icosphere()
    x = _batch(v, (3,), False, 30)
    faces = torch.tensor(f, device=DEV)
    grad_out = torch.randn(x.shape, generator=_gen(31), device=DEV)
    aligned = _abi_calls(cuda_lib, mode, x, faces, grad_out, 0)
    for shift in (1, 3):
        got = _abi_calls(cuda_lib, mode, x, faces, grad_out, shift)
        for a, b in zip(got, aligned):
            assert not torch.isnan(b).any() and torch.equal(a, b), shift
    _check(aligned[0].reshape(x.shape).cpu(), mesh._vertex_laplacian(x.double().cpu(), f, mode),
           'laplacian %s fwd vs fp64' % mode)


@pytest.fixture(scope='module')
def small(cuda_lib, tmp_path_factory):
    return variant_builds.small_grid_library(tmp_path_factory)


def _fan(n=5000):
    """n faces around vertex 0: one row far longer than a warp's share, summed by the whole warp."""
    i = np.arange(n + 1)
    t = i * (np.pi * (3. - np.sqrt(5.)))
    rim = np.stack([np.cos(t), np.sin(t), -0.3 + 0.6 * i / n], axis=1)
    v = np.concatenate([np.zeros((1, 3)), rim]).astype(np.float32)
    f = np.stack([np.zeros(n), np.arange(1, n + 1), np.arange(2, n + 2)], axis=1).astype(np.int32)
    return v, f


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('name', ['icosphere', 'fan'])
def test_grid_stride_rounds_past_the_block_cap(cuda_lib, small, mesh, name, mode):
    """The small-grid build caps every normals.cu launch at DIRT_NORMALS_MAX_BLOCKS = 3 CTAs, so each vertex pass and
    adjacency kernel runs many grid-stride rounds, the last one partial.  Outputs and gradients must equal the product
    library's bit for bit, with the buffers the package allocates starting as NaN so that a skipped round shows."""
    from dirt_b200 import _lib
    v, f = _icosphere() if name == 'icosphere' else _fan()
    x = _batch(v, (5,), True, 32)
    faces = torch.tensor(f, device=DEV)
    grad_out = torch.randn(x.shape[:-1] + (3,), generator=_gen(33), device=DEV)
    empty = torch.empty
    runs = []
    for lib in (cuda_lib, small):
        leaf = x.detach().clone().requires_grad_(True)
        with pytest.MonkeyPatch.context() as m:
            m.setattr(_lib, 'lib', lambda lib=lib: lib)
            m.setattr(torch, 'empty', lambda *a, **k: empty(*a, **k).fill_(float('nan')) if
                      k.get('dtype', torch.float32).is_floating_point else empty(*a, **k))
            out = mesh.laplacian(leaf, faces, mode)
            (out * grad_out).sum().backward()
            torch.cuda.synchronize()
        runs.append((out.detach(), leaf.grad))
    n_rows = x.shape[0] * x.shape[1]
    assert n_rows > 3 * 256 * 4, 'several rounds of 3 CTAs of NORMALS_THREADS'
    for got, want in zip(runs[1], runs[0]):
        assert not torch.isnan(want).any() and torch.equal(got, want)


def test_the_regularised_fit_improves_the_held_out_silhouettes(cuda_lib):
    spec = importlib.util.spec_from_file_location('silhouette_example', os.path.join(ROOT, 'examples', 'silhouette.py'))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    r = ex.fit(10., 60, device=DEV, verbose=False)
    assert r['held_out_iou_end'] > r['held_out_iou_start'] + 0.1, r
