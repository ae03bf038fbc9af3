"""GPU: the vertex normals' CUDA path against their torch restatement (`_vertex_normals`, `_vertex_normals_pre_split` of
dirt_b200/lighting.py).

Forward values against the restatement in float64 and in float32 on the same device, gradients against float64
autograd of the restatement, both with conftest.rel_close (1e-4).  Pre-split normals of meshes that are not split
(where the restatement's index_copy leaves repeated indices undefined) are compared against a loop in which the last
face corner of each vertex wins."""
import functools
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import rel_close

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device('cuda', 0)


@pytest.fixture(scope='module')
def lighting(cuda_lib):
    from dirt_b200 import lighting
    return lighting


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ---- meshes -----------------------------------------------------------------------------------------------------------

def _icosphere():
    from dirt_b200 import scenes
    v, f = scenes.icosphere(3)
    r = np.random.default_rng(1)
    return (v * (1. + 0.2 * r.standard_normal((v.shape[0], 1)))).astype(np.float32), f


def _uv_sphere():
    from dirt_b200 import scenes
    return scenes.uv_sphere(224, 112, displacement=0.1)   # cfg5: poles of valence 224


def _cube():
    from dirt_b200 import scenes
    return scenes.cube()


def _split_cube():
    v, f = _cube()
    return v[f.reshape(-1)], np.arange(f.size, dtype=np.int32).reshape(-1, 3)


def _fan(n=100000):
    """n faces around vertex 0.  The rim turns by the golden angle from one vertex to the next and rises slowly, so that
    every face has a wide corner at the centre and neighbouring faces face the same way."""
    i = np.arange(n + 1)
    t = i * (np.pi * (3. - np.sqrt(5.)))
    rim = np.stack([np.cos(t), np.sin(t), -0.3 + 0.6 * i / n], axis=1)
    v = np.concatenate([np.zeros((1, 3)), rim]).astype(np.float32)
    f = np.stack([np.zeros(n), np.arange(1, n + 1), np.arange(2, n + 2)], axis=1).astype(np.int32)
    return v, f


def _odd(repeated_faces=True):
    """An icosphere with unused vertices between the used ones and faces that name one vertex twice."""
    v, f = _icosphere()
    r = np.random.default_rng(2)
    V = v.shape[0]
    spread = np.concatenate([v, r.standard_normal((V // 2, 3)).astype(np.float32)])
    perm = r.permutation(spread.shape[0])
    inverse = np.argsort(perm)
    v2, f2 = spread[perm], inverse[f].astype(np.int32)
    repeated = np.array([[f2[i, 0], f2[i, 0], f2[i + 1, 1]] for i in range(0, 60, 3)], np.int32)
    return v2, np.concatenate([f2, repeated]) if repeated_faces else f2


MESHES = {'icosphere': _icosphere, 'uv_sphere': _uv_sphere, 'cube': _cube, 'split_cube': _split_cube, 'fan': _fan,
          'odd': _odd}
SPLIT = {'split_cube'}


def _batch(v, lead, w, seed, strided=False):
    """[*lead, V, 3 | 4] on the device: the mesh scaled and shifted per item, w = 1 + noise; strided: every other item of
    a batch twice as long."""
    g = np.random.default_rng(seed)
    n = int(np.prod(lead)) if lead else 1
    items = v[None] * (1. + 0.1 * g.random((2 * n, 1, 1))) + 0.1 * g.standard_normal((2 * n, 1, 3))
    if w:
        items = np.concatenate([items, 1. + g.random(items.shape[:-1] + (1,))], axis=-1)
    t = torch.tensor(items, dtype=torch.float32, device=DEV)
    t = t[::2] if strided else t[:n]
    return t.reshape(lead + t.shape[1:])


def _last_wins(v, f, dtype=np.float64):
    """Pre-split normals with the face corners taken corner-major, then by face: the last one naming a vertex wins."""
    v = v[..., :3].astype(dtype)
    F = len(f)
    last = np.full(v.shape[-2], -1)
    for k in range(3):
        np.maximum.at(last, f[:, k], k * F + np.arange(F))
    n = np.cross(v[..., f[:, 1], :] - v[..., f[:, 0], :], v[..., f[:, 2], :] - v[..., f[:, 0], :])
    u = n / (np.linalg.norm(n, axis=-1, keepdims=True) + 1e-12)
    out = np.zeros(v.shape[:-1] + (3,))
    used = last >= 0
    out[..., used, :] = u[..., last[used] % F, :]
    return out


def _check(got, want, name):
    assert got.shape == want.shape, (got.shape, want.shape)
    ok, ratio = rel_close(np.asarray(got, np.float64), np.asarray(want, np.float64), name=name)
    assert ok, (name, ratio)


# ---- forward ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('lead', [(), (2,), (2, 2)], ids=['lead0', 'lead1', 'lead2'])
@pytest.mark.parametrize('mesh', sorted(MESHES))
def test_forward_matches_the_restatement(lighting, mesh, lead):
    v, f = MESHES[mesh]()
    faces = torch.tensor(f, device=DEV)
    for w in (False, True):
        for strided in (False, True):
            x = _batch(v, lead, w, len(lead) + 3 * w, strided)
            tag = '%s lead %d w %d strided %d' % (mesh, len(lead), w, strided)
            got = lighting.vertex_normals(x, faces)
            assert got.dtype == torch.float32 and got.shape == lead + (v.shape[0], 3)
            _check(got.cpu(), lighting._vertex_normals(x.double().cpu(), f), 'normals fwd vs fp64')
            _check(got.cpu(), lighting._vertex_normals(x, faces).cpu(), 'normals fwd vs fp32')
            got = lighting.vertex_normals_pre_split(x, faces.long())
            if mesh in SPLIT:
                _check(got.cpu(), lighting._vertex_normals_pre_split(x.double().cpu(), f), 'pre-split fwd vs fp64')
                _check(got.cpu(), lighting._vertex_normals_pre_split(x, faces).cpu(), 'pre-split fwd vs fp32')
            else:
                # one face's normal, not a sum: the uv-sphere's pole faces have a 1.6 degree corner, where a float32
                # cross product keeps about 2e-6 of the normal, so against float64 the bar is 2e-4 there
                rel = 2e-4 if mesh == 'uv_sphere' else 1e-4
                ok, ratio = rel_close(got.cpu().numpy(), _last_wins(x.cpu().numpy(), f), rel=rel,
                                      name='pre-split fwd vs last-wins loop')
                assert ok, (tag, ratio)
                _check(got.cpu(), _last_wins(x.cpu().numpy(), f, np.float32), 'pre-split fwd vs fp32 last-wins loop')
            assert np.isfinite(got.cpu().numpy()).all(), tag


# ---- gradients ------------------------------------------------------------------------------------------------------------

def _grads(fn, x, faces, grad_out):
    leaf = x.detach().clone().requires_grad_(True)
    (fn(leaf, faces) * grad_out).sum().backward()
    return leaf.grad


@pytest.mark.parametrize('w', [False, True])
@pytest.mark.parametrize('mesh', sorted(MESHES))
def test_gradients_match_autograd_of_the_restatement(lighting, mesh, w):
    # A face naming a vertex twice passes gradients of 1e12 and more to its corners (see test_kinks_match_float64_autograd),
    # which cancel in the sum of a vertex that also has ordinary faces: no float32 evaluation keeps the rest of that sum.
    v, f = _odd(repeated_faces=False) if mesh == 'odd' else MESHES[mesh]()
    faces = torch.tensor(f, device=DEV)
    for lead in ((), (3,)):
        x = _batch(v, lead, w, 7)
        grad_out = torch.randn(lead + (v.shape[0], 3), generator=_gen(8), device=DEV)
        pairs = [(lighting.vertex_normals, lighting._vertex_normals, 'normals')]
        if mesh in SPLIT:
            # elsewhere index_copy's gradient differs: it passes a repeated index's gradient to every copy
            pairs.append((lighting.vertex_normals_pre_split, lighting._vertex_normals_pre_split, 'pre-split'))
        for op, ref, name in pairs:
            got = _grads(op, x, faces, grad_out)
            want = _grads(ref, x.double().cpu(), torch.tensor(f), grad_out.double().cpu())
            if w:
                assert torch.equal(got[..., 3], torch.zeros_like(got[..., 3]))
            _check(got.cpu(), want, '%s grad vs fp64' % name)


def test_pre_split_gradient_reaches_every_vertex_of_a_face(lighting):
    """A face that names one vertex twice: that vertex takes the normal of the later corner, but the positions of all
    three vertices reach the normal (the restatement's index_copy calls each overwrite whole rows)."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 1]], np.float32)
    f = np.array([[0, 1, 2], [1, 3, 4], [2, 2, 3]], np.int32)
    x = torch.tensor(v, device=DEV)
    grad_out = torch.randn(5, 3, generator=_gen(9), device=DEV)
    got = _grads(lighting.vertex_normals_pre_split, x, torch.tensor(f, device=DEV), grad_out)
    want = _grads(lighting._vertex_normals_pre_split, x.double().cpu(), torch.tensor(f), grad_out.double().cpu())
    _check(got.cpu(), want, 'pre-split grad vs fp64')
    _check(lighting.vertex_normals_pre_split(x, torch.tensor(f, device=DEV)).cpu(), _last_wins(v, f),
           'pre-split fwd vs last-wins loop')


def test_no_gradient_wanted_builds_no_node(lighting, cuda_lib):
    v, f = _icosphere()
    x = torch.tensor(v, device=DEV)
    out = lighting.vertex_normals(x, torch.tensor(f, device=DEV))
    assert out.grad_fn is None and not out.requires_grad
    assert cuda_lib.dirt_last_launch_count() == 5      # the adjacency's four kernels and the vertex pass
    # a graph in which another input wants a gradient does not reach the normals' backward kernels
    k = torch.ones(3, device=DEV, requires_grad=True)
    (lighting.vertex_normals(x, torch.tensor(f, device=DEV)) * k).sum().backward()
    assert cuda_lib.dirt_last_launch_count() == 5 and k.grad is not None


def test_double_backward(lighting):
    v, f = _icosphere()
    faces = torch.tensor(f, device=DEV)
    x = _batch(v, (2,), True, 10)
    grad_out = torch.randn(2, v.shape[0], 3, generator=_gen(11), device=DEV)
    results = []
    for fn in (lighting.vertex_normals, lighting._vertex_normals):
        leaf = x.detach().clone().requires_grad_(True)
        first, = torch.autograd.grad((fn(leaf, faces) * grad_out).sum(), leaf, create_graph=True)
        first.square().sum().backward()
        results.append((first.detach(), leaf.grad))
    for a, b in zip(*results):
        _check(a.cpu(), b.cpu(), 'normals double backward')


# ---- kinks ------------------------------------------------------------------------------------------------------------------

def test_kinks_match_float64_autograd(lighting):
    """Integer coordinates, so that float32 and float64 see the same zeros: a collinear face and a face naming a vertex
    twice (normal 0, so the gradients pass 1e12 at each division: 1e24 through both), and a face with its reversed copy
    (their normals cancel: output 0, gradient 0)."""
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0],          # collinear
                  [3, 1, 0], [4, 2, 1],                     # (3, 3, 4)
                  [0, 5, 0], [1, 5, 2], [0, 6, 3]], np.float32)   # (5, 6, 7) and (5, 7, 6)
    f = np.array([[0, 1, 2], [3, 3, 4], [5, 6, 7], [5, 7, 6]], np.int32)
    g = np.random.default_rng(12).integers(-3, 4, (8, 3))
    g[7] = g[6]   # the two faces then add up the gradients of their corners to the same value, whatever the order
    grad_out = torch.tensor(g, dtype=torch.float32, device=DEV)
    x = torch.tensor(v, device=DEV)
    # pre-split: the two degenerate faces only (the reversed pair names vertex 5 twice in one corner column)
    for op, ref, faces in ((lighting.vertex_normals, lighting._vertex_normals, f),
                           (lighting.vertex_normals_pre_split, lighting._vertex_normals_pre_split, f[:2])):
        out = op(x, torch.tensor(faces, device=DEV))
        assert not out.any()
        assert not ref(x.double().cpu(), torch.tensor(faces)).any()
        got = _grads(op, x, torch.tensor(faces, device=DEV), grad_out).cpu().numpy()
        want = _grads(ref, x.double().cpu(), torch.tensor(faces), grad_out.double().cpu()).numpy()
        assert np.abs(want[:5]).max() > (1e23 if op is lighting.vertex_normals else 1e11)
        assert not want[5:].any() and not got[5:].any()
        # each face's vertices against the largest gradient among them, so that the 1e24s do not swamp the rest
        for rows in (slice(0, 3), slice(3, 5)):
            _check(got[rows], want[rows], 'normals kink grad')


# ---- invalid faces and empty inputs ---------------------------------------------------------------------------------------

@pytest.mark.parametrize('dtype', [torch.int32, torch.int64])
def test_invalid_faces_are_left_out(lighting, dtype):
    v, f = _icosphere()
    V = v.shape[0]
    bad = f.astype(np.int64).copy()
    rows = np.arange(5, len(f), 37)
    values = [-1, V, V + 5, -7] + ([(1 << 32) + 3, (1 << 32) + V - 1, -(1 << 32) + 2, (1 << 31)] if dtype == torch.int64 else [])
    for j, r in enumerate(rows):
        bad[r, j % 3] = values[j % len(values)]
    keep = np.setdiff1d(np.arange(len(f)), rows)
    x = _batch(v, (2,), True, 13)
    faces = torch.tensor(bad, dtype=dtype, device=DEV)
    grad_out = torch.randn(2, V, 3, generator=_gen(14), device=DEV)
    for op, ref in ((lighting.vertex_normals, lighting._vertex_normals),
                    (lighting.vertex_normals_pre_split, lighting._vertex_normals_pre_split)):
        want_faces = torch.tensor(f[keep])
        got = op(x, faces)
        if op is lighting.vertex_normals:
            _check(got.cpu(), ref(x.double().cpu(), want_faces), 'normals invalid faces fwd')
            _check(_grads(op, x, faces, grad_out).cpu(), _grads(ref, x.double().cpu(), want_faces, grad_out.double().cpu()),
                   'normals invalid faces grad')
        else:
            _check(got.cpu(), _last_wins(x.cpu().numpy(), f[keep]), 'pre-split invalid faces fwd')
    # faces on the CPU go to the vertices' device as before
    _check(lighting.vertex_normals(x, torch.tensor(bad, dtype=dtype)).cpu(),
           lighting._vertex_normals(x.double().cpu(), torch.tensor(f[keep])), 'normals invalid faces fwd')


def test_empty_inputs(lighting):
    v, f = _cube()
    for op in (lighting.vertex_normals, lighting.vertex_normals_pre_split):
        for lead, V, faces in (((2,), 8, np.zeros((0, 3), np.int32)), ((2,), 0, np.zeros((0, 3), np.int32)),
                               ((2,), 0, f), ((0,), 8, f), ((), 8, np.zeros((0, 3), np.int64))):
            x = torch.rand(lead + (V, 4), generator=_gen(15), device=DEV).requires_grad_(True)
            out = op(x, torch.tensor(faces, device=DEV))
            assert out.shape == lead + (V, 3) and not out.any()
            out.sum().backward()
            assert x.grad.shape == x.shape and not x.grad.any()


def test_more_items_than_a_grid_dimension(lighting):
    v, f = _cube()
    x = _batch(v, (70000,), False, 16)
    faces = torch.tensor(f, device=DEV)
    got = lighting.vertex_normals(x, faces)
    _check(got.cpu(), lighting._vertex_normals(x.double(), faces).cpu(), 'normals fwd vs fp64')
    grad_out = torch.randn(x.shape, generator=_gen(17), device=DEV)
    _check(_grads(lighting.vertex_normals, x, faces, grad_out).cpu(),
           _grads(lighting._vertex_normals, x.double(), faces, grad_out.double()).cpu(), 'normals grad vs fp64')


# ---- determinism ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('mesh', ['uv_sphere', 'fan'])
def test_repeated_calls_are_bit_identical(lighting, mesh):
    v, f = MESHES[mesh]()
    faces = torch.tensor(f, device=DEV)
    x = _batch(v, (8,) if mesh == 'uv_sphere' else (), True, 18)
    grad_out = torch.randn(x.shape[:-1] + (3,), generator=_gen(19), device=DEV)
    for op in (lighting.vertex_normals, lighting.vertex_normals_pre_split):
        runs = []
        for _ in range(3):
            leaf = x.detach().clone().requires_grad_(True)
            out = op(leaf, faces)
            (out * grad_out).sum().backward()
            runs.append((out.detach(), leaf.grad))
        for out, grad in runs[1:]:
            assert torch.equal(out.view(torch.int32), runs[0][0].view(torch.int32))
            assert torch.equal(grad.view(torch.int32), runs[0][1].view(torch.int32))


@pytest.mark.parametrize('pre_split', [False, True])
def test_cuda_graph_capture_and_replay(lighting, pre_split):
    op = lighting.vertex_normals_pre_split if pre_split else lighting.vertex_normals
    v, f = _uv_sphere()
    faces = torch.tensor(f, device=DEV)
    x = _batch(v, (4,), True, 20).requires_grad_(True)
    grad_out = torch.randn(4, v.shape[0], 3, generator=_gen(21), device=DEV)

    def step():
        x.grad = None
        out = op(x, faces)
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


# ---- end to end ---------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def ex(cuda_lib):
    spec = importlib.util.spec_from_file_location('textured_example', os.path.join(ROOT, 'examples', 'textured.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _textured_cube(ex, normals):
    import dirt_b200 as dirt
    from dirt_b200 import matrices
    vertices, uvs, faces = ex.build_cube()
    uvs = torch.tensor(uvs, dtype=torch.float32, device=DEV)
    faces = torch.tensor(faces, dtype=torch.int32, device=DEV)
    texture = ex.checker_texture(size=64, device=DEV)
    texture = texture + 0.1 * torch.rand(texture.shape, generator=_gen(26), device=DEV)
    light_direction = torch.tensor([1., 0., 0.], device=DEV)
    vertices_object = torch.tensor(vertices, dtype=torch.float32, device=DEV)
    vertices_object = torch.cat([vertices_object, torch.ones_like(vertices_object[:, -1:])], dim=1).requires_grad_(True)
    vertices_world = vertices_object @ matrices.rodrigues([0., 0.6, 0.]).to(DEV)
    view = matrices.compose(matrices.translation([0., -2., -3.2]), matrices.rodrigues([-0.5, 0., 0.])).to(DEV)
    proj = matrices.perspective_projection(near=0.1, far=20., right=0.1, aspect=120. / 160.).to(DEV)
    attributes = torch.cat([torch.ones_like(uvs[:, :1]), uvs, normals(vertices_world, faces)], dim=1)
    pixels = dirt.rasterise_deferred(torch.zeros([120, 160, 6], device=DEV), vertices_world @ view @ proj, attributes, faces,
                                     functools.partial(ex.shader_fn, sample=dirt.sample_texture), [texture, light_direction])
    weights = torch.rand(pixels.shape, generator=_gen(27), device=DEV)
    (pixels * weights).sum().backward()
    return pixels.detach(), vertices_object.grad


def test_textured_cube_through_rasterise_deferred(ex, lighting):
    px_cuda, gv_cuda = _textured_cube(ex, lighting.vertex_normals)
    px_torch, gv_torch = _textured_cube(ex, lighting._vertex_normals)
    assert float((px_cuda != torch.tensor([0., 0., 0.3], device=DEV)).any(-1).float().mean()) > 0.1   # the cube is in view
    _check(px_cuda.cpu(), px_torch.cpu(), 'normals textured cube pixels')
    _check(gv_cuda.cpu(), gv_torch.cpu(), 'normals textured cube grad_vertices')
