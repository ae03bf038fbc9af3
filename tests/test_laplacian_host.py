"""CPU: the mesh Laplacian's torch restatement (`_vertex_laplacian` of dirt_b200/mesh.py) has the properties its
docstring states, its C ABI rejects bad arguments before anything is launched, its workspace size is a function of the
sizes alone, its routing is the normals', and CPU calls run the restatement unchanged."""
import ctypes

import numpy as np
import pytest
import torch

UNI, COT = 0, 1
CUDA = torch.device('cuda', 0)
CPU = torch.device('cpu')


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _icosphere(level, dtype=torch.float64):
    from dirt_b200 import scenes
    v, f = scenes.icosphere(level)
    v = torch.tensor(v, dtype=torch.float64)
    return (v / v.norm(dim=-1, keepdim=True)).to(dtype), torch.tensor(f)


def _grid(n=6, jitter=0.):
    """An n x n flat grid in z = 0, every square split along the same diagonal."""
    y, x = np.meshgrid(np.arange(n), np.arange(n), indexing='ij')
    v = np.stack([x.ravel(), y.ravel(), np.zeros(n * n)], axis=1).astype(np.float64)
    if jitter:
        v[:, :2] += jitter * np.random.default_rng(0).standard_normal((n * n, 2))
    q = (np.arange(n - 1)[:, None] * n + np.arange(n - 1)[None, :]).ravel()
    f = np.concatenate([np.stack([q, q + 1, q + n + 1], 1), np.stack([q, q + n + 1, q + n], 1)])
    interior = np.array([i * n + j for i in range(1, n - 1) for j in range(1, n - 1)])
    return torch.tensor(v), torch.tensor(f), interior


# ---- the restatement ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('mode', ['uniform', 'cotangent'])
def test_translation_invariance(mode):
    from dirt_b200.mesh import _vertex_laplacian
    v, f = _icosphere(2)
    v = v * (1. + 0.2 * torch.tensor(np.random.default_rng(1).standard_normal((v.shape[0], 1))))
    moved = v + torch.tensor([0.3, -1.7, 2.5], dtype=torch.float64)
    assert torch.allclose(_vertex_laplacian(moved, f, mode), _vertex_laplacian(v, f, mode), atol=1e-12, rtol=1e-9)


@pytest.mark.parametrize('mode', ['uniform', 'cotangent'])
def test_zero_at_interior_vertices_of_a_flat_grid(mode):
    from dirt_b200.mesh import _vertex_laplacian
    v, f, interior = _grid()
    out = _vertex_laplacian(v, f, mode)
    assert out[interior].abs().max() < 1e-12
    assert out[0].abs().max() > 0.1     # a corner of the grid has no neighbours on two sides
    assert not out[:, 2].any()
    if mode == 'cotangent':   # linear precision: any flat triangulation
        v, f, interior = _grid(jitter=0.15)
        assert _vertex_laplacian(v, f, mode)[interior].abs().max() < 1e-12


@pytest.mark.parametrize('level', [1, 2, 3])
def test_uniform_is_the_distinct_neighbour_mean_on_a_closed_mesh(level):
    from dirt_b200.mesh import _vertex_laplacian
    v, f = _icosphere(level)
    v = v * (1. + 0.2 * torch.tensor(np.random.default_rng(level).standard_normal((v.shape[0], 1))))
    neighbours = [set() for _ in range(v.shape[0])]
    for a, b, c in f.tolist():
        neighbours[a] |= {b, c}
        neighbours[b] |= {a, c}
        neighbours[c] |= {a, b}
    want = torch.stack([v[sorted(n)].mean(0) - v[i] for i, n in enumerate(neighbours)])
    assert torch.allclose(_vertex_laplacian(v, f, 'uniform'), want, atol=1e-13, rtol=0)


def test_uniform_weighs_boundary_edges_half():
    from dirt_b200.mesh import _vertex_laplacian
    v, f, _ = _grid(3)
    # vertex 1 on the bottom edge: faces (0, 1, 4), (1, 2, 5), (1, 5, 4); boundary edges to 0 and 2 count once
    p = v.numpy()
    want = ((p[0] - p[1]) + (p[2] - p[1]) + 2 * (p[4] - p[1]) + 2 * (p[5] - p[1])) / 6.
    assert np.allclose(_vertex_laplacian(v, f, 'uniform')[1].numpy(), want, atol=1e-14)


def test_cotangent_approaches_the_mean_curvature_normal():
    from dirt_b200.mesh import _vertex_laplacian
    errors = []
    for level in (2, 3, 4):
        for r in (0.5, 2.):
            v, f = _icosphere(level)
            n = v.clone()
            out = _vertex_laplacian(r * v, f, 'cotangent')
            err = ((out + (2. / r) * n).norm(dim=-1) / (2. / r)).mean().item()
            if r == 2.:
                errors.append(err)
    assert errors[0] > errors[1] > errors[2]
    assert errors[2] <= 0.005, errors


def test_an_unnamed_vertex_gets_zero():
    from dirt_b200.mesh import _vertex_laplacian
    v, f = _icosphere(1)
    v = torch.cat([v, torch.ones(1, 3, dtype=v.dtype)])
    for mode in ('uniform', 'cotangent'):
        out = _vertex_laplacian(v, f, mode)
        assert not out[-1].any() and out[:-1].abs().min(-1).values.max() > 0


@pytest.mark.parametrize('mode', ['uniform', 'cotangent'])
def test_gradcheck(mode):
    from dirt_b200.mesh import _vertex_laplacian
    v, f = _icosphere(1)
    g = np.random.default_rng(3)
    v = (v * (1. + 0.2 * torch.tensor(g.standard_normal((v.shape[0], 1))))).requires_grad_(True)
    w = torch.cat([v.detach(), torch.ones(v.shape[0], 1, dtype=v.dtype)], -1).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda x: _vertex_laplacian(x, f, mode), (v,))
    assert torch.autograd.gradgradcheck(lambda x: _vertex_laplacian(x, f, mode), (v,))
    assert torch.autograd.gradcheck(lambda x: _vertex_laplacian(x, f, mode), (w,))


# ---- the C ABI ----------------------------------------------------------------------------------------------------------

def _p(x):
    return ctypes.c_void_p(x)


def _fwd(L, mode=UNI, B=2, V=8, F=4, stride=3, vertices=4096, faces=4096, out=4096, ws=4096, ws_bytes=1 << 20):
    return L.dirt_laplacian_forward(mode, _p(vertices), stride, _p(faces), _p(out), _p(ws), ws_bytes, B, V, F, None)


def _bwd(L, mode=UNI, B=2, V=8, F=4, stride=3, vertices=4096, faces=4096, grad=4096, out=4096, ws=4096,
         ws_bytes=1 << 20):
    return L.dirt_laplacian_backward(mode, _p(vertices), stride, _p(faces), _p(grad), _p(out), _p(ws), ws_bytes, B, V,
                                     F, None)


def test_laplacian_abi_rejects_bad_shapes(L):
    from dirt_b200 import _lib
    for call in (_fwd, _bwd):
        for kw in (dict(mode=2), dict(mode=-1), dict(B=-1), dict(V=-1), dict(F=-1), dict(stride=2), dict(stride=-4),
                   dict(V=1 << 31), dict(F=(1 << 31) // 3 + 1), dict(B=1 << 30, V=1 << 30, stride=1 << 20)):
            for mode in (UNI, COT):
                args = dict(dict(mode=mode), **kw)
                assert call(L, **args) == _lib.ERR_BAD_SHAPE, args
                assert L.dirt_last_launch_count() == 0
    assert L.dirt_laplacian_workspace_bytes(1, (1 << 31) - 1, 1) > 0
    assert L.dirt_laplacian_workspace_bytes(1, 3, ((1 << 31) - 1) // 3) > 0


def test_laplacian_abi_rejects_null_and_misaligned_pointers(L):
    from dirt_b200 import _lib
    for mode in (UNI, COT):
        for call in (_fwd, _bwd):
            for name in ('vertices', 'faces', 'out', 'ws'):
                assert call(L, mode, **{name: 0}) == _lib.ERR_NULL_POINTER, name
                assert call(L, mode, **{name: 4098}) == _lib.ERR_MISALIGNED, name
            assert call(L, mode, ws_bytes=L.dirt_laplacian_workspace_bytes(2, 8, 4) - 1) == _lib.ERR_WORKSPACE_TOO_SMALL
            # the normals' workspace is too small: the Laplacian's gradient scratch is 4 floats per row, not 3
            assert call(L, mode, B=64, V=1000, F=10, ws_bytes=L.dirt_normals_workspace_bytes(64, 1000, 10)) == \
                _lib.ERR_WORKSPACE_TOO_SMALL
        assert _bwd(L, mode, grad=0) == _lib.ERR_NULL_POINTER
        assert _bwd(L, mode, grad=4098) == _lib.ERR_MISALIGNED
    assert L.dirt_last_launch_count() == 0


def test_laplacian_abi_with_nothing_to_do_launches_nothing(L):
    for B, V in ((0, 8), (3, 0), (0, 0)):
        for mode in (UNI, COT):
            assert _fwd(L, mode, B=B, V=V, vertices=0, faces=0, out=0, ws=0, ws_bytes=0) == 0
            assert L.dirt_last_launch_count() == 0
            assert _bwd(L, mode, B=B, V=V, vertices=0, faces=0, grad=0, out=0, ws=0, ws_bytes=0) == 0
            assert L.dirt_last_launch_count() == 0


def _expected_workspace(B, V, F):
    up = lambda n: (n + 255) // 256 * 256
    if B == 0 or V == 0 or F == 0:
        return 0
    return up(4 * (V + 1)) + up(4 * 3 * F) + up(max(up(4 * V) + 4 * 3 * F, 4 * 4 * B * V))


def test_laplacian_workspace_is_a_pure_function_of_the_shapes(L):
    W = L.dirt_laplacian_workspace_bytes
    for B, V, F in ((0, 10, 5), (2, 0, 5), (2, 10, 0), (1, 1, 1), (2, 100, 50), (64, 2562, 5120), (64, 24866, 49728),
                    (1, 1000, 100000), (3, 7, 11), (1, 523266, 1046528)):
        assert W(B, V, F) == _expected_workspace(B, V, F), (B, V, F)
        assert W(B, V, F) == W(B, V, F)
        assert W(B, V, F) >= L.dirt_normals_workspace_bytes(B, V, F)
    assert W(-1, 10, 5) == 0 and W(1, 1 << 31, 5) == 0 and W(1, 10, -1) == 0


# ---- routing ------------------------------------------------------------------------------------------------------------

def test_laplacian_route_is_the_normals_route():
    """Accepted calls go to the mode's _MeshOp with [B*V, 3] rows (a w column dropped); the routing decision is
    lighting.normals_route, whose refusals are listed in test_normals_host.py."""
    from dirt_b200 import mesh
    from dirt_b200.lighting import normals_route
    f32, i32, i64 = torch.float32, torch.int32, torch.int64
    r = normals_route((2, 3, 7, 4), f32, CUDA, (4, 3), i64)
    assert (r.lead, r.B, r.V, r.F) == ((2, 3), 6, 7, 4)
    assert normals_route((7, 3), f32, CUDA, (0, 3), i32).F == 0
    for args in (((10, 3), f32, CPU, (4, 3), i32), ((10, 3), torch.float64, CUDA, (4, 3), i32),
                 ((10, 5), f32, CUDA, (4, 3), i32), ((10, 3), f32, CUDA, (2, 4, 3), i32),
                 ((10, 3), f32, CUDA, (4, 3), torch.int16)):
        assert normals_route(*args) is None, args
    seen = []
    real_route, real_mesh = mesh._normals_route, mesh._mesh
    try:
        mesh._normals_route = lambda v, f: normals_route(v.shape, v.dtype, CUDA, torch.as_tensor(f).shape,
                                                         torch.as_tensor(f).dtype)
        mesh._mesh = lambda op, route, faces, rows: seen.append((op, route, rows.shape, rows.stride()))
        v, f = _icosphere(1, torch.float32)
        x = torch.cat([v, torch.ones(v.shape[0], 1)], -1).expand(2, 3, -1, -1)
        for mode in ('uniform', 'cotangent'):
            mesh.laplacian(x, f, mode)
            op, route, shape, stride = seen.pop()
            assert op is mesh._LAPLACIAN[mode] and route.lead == (2, 3) and shape == (6 * v.shape[0], 3)
            assert stride[1] == 1 and stride[0] >= 3
        assert mesh._LAPLACIAN['uniform'].inputs(route, f, torch.zeros(6, 3))[0] == UNI
        assert mesh._LAPLACIAN['cotangent'].inputs(route, f, torch.zeros(6, 3))[0] == COT
        mesh.laplacian(x.double(), f)                          # float64: the restatement
        assert not seen
    finally:
        mesh._normals_route, mesh._mesh = real_route, real_mesh


# ---- CPU calls ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('mode', ['uniform', 'cotangent'])
@pytest.mark.parametrize('w', [False, True])
def test_cpu_calls_return_the_restatement(mode, w):
    import dirt_b200
    from dirt_b200.mesh import _vertex_laplacian
    v, f = _icosphere(2, torch.float32)
    for lead in ((), (2,), (2, 3)):
        n = int(np.prod(lead)) if lead else 1
        x = v * (1. + 0.3 * torch.rand((n, v.shape[0], 1), generator=torch.Generator().manual_seed(len(lead))))
        x = x.reshape(lead + v.shape)
        if w:
            x = torch.cat([x, torch.ones(x.shape[:-1] + (1,))], -1)
        want = _vertex_laplacian(x, f, mode)
        assert want.shape == lead + (v.shape[0], 3)
        assert torch.equal(dirt_b200.mesh.laplacian(x, f, mode), want)
        assert torch.equal(dirt_b200.mesh.laplacian(x, f.int(), mode), want)
    got = dirt_b200.mesh.laplacian(v.double(), f, mode)
    assert got.dtype == torch.float64 and torch.equal(got, _vertex_laplacian(v.double(), f, mode))
    got = dirt_b200.mesh.laplacian(v.numpy(), f.numpy().tolist(), mode)
    assert got.dtype == torch.float32 and torch.equal(got, _vertex_laplacian(v, f, mode))
    a, b = v.clone().requires_grad_(True), v.clone().requires_grad_(True)
    dirt_b200.mesh.laplacian(a, f, mode).square().sum().backward()
    _vertex_laplacian(b, f, mode).square().sum().backward()
    assert torch.equal(a.grad, b.grad)


def test_cpu_calls_keep_their_errors():
    from dirt_b200 import mesh
    v, f = _icosphere(1, torch.float32)
    bad = f.clone()
    bad[3, 1] = v.shape[0]
    for mode in ('uniform', 'cotangent'):
        with pytest.raises(IndexError):
            mesh.laplacian(v, bad, mode)
    for bad_mode in ('mean', 'cot', None):
        with pytest.raises(ValueError, match='mode'):
            mesh.laplacian(v, f, bad_mode)
        with pytest.raises(ValueError, match='mode'):
            mesh._vertex_laplacian(v, f, bad_mode)
