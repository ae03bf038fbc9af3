"""CPU: the edge terms' torch restatements (`_edge_lengths` and `_normal_consistency` of dirt_b200/mesh.py) have the
properties their docstrings state, their C ABI rejects bad arguments before anything is launched, its workspace size
is a function of the sizes alone, their routing is the normals', and CPU calls run the restatements unchanged."""
import ctypes
import math

import numpy as np
import pytest
import torch

LEN, CONS = 0, 1
CUDA = torch.device('cuda', 0)
CPU = torch.device('cpu')
OPS = ['edge_lengths', 'normal_consistency']


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _icosphere(level, dtype=torch.float64, noise=0.):
    from dirt_b200 import scenes
    v, f = scenes.icosphere(level)
    v = torch.tensor(v, dtype=torch.float64)
    v = v / v.norm(dim=-1, keepdim=True)
    if noise:
        v = v * (1. + noise * torch.tensor(np.random.default_rng(level).standard_normal((v.shape[0], 1))))
    return v.to(dtype), torch.tensor(f)


def _grid(n=6):
    """An n x n flat grid in z = 0 with jittered vertices, every square split along the same diagonal."""
    y, x = np.meshgrid(np.arange(n), np.arange(n), indexing='ij')
    v = np.stack([x.ravel(), y.ravel(), np.zeros(n * n)], axis=1).astype(np.float64)
    v[:, :2] += 0.15 * np.random.default_rng(0).standard_normal((n * n, 2))
    q = (np.arange(n - 1)[:, None] * n + np.arange(n - 1)[None, :]).ravel()
    f = np.concatenate([np.stack([q, q + 1, q + n + 1], 1), np.stack([q, q + n + 1, q + n], 1)])
    return torch.tensor(v), torch.tensor(f)


def _unit(n):
    return n / (np.linalg.norm(n) + 1e-12)


def _face_unit(v, face):
    p = v.numpy()[list(face)]
    return _unit(np.cross(p[1] - p[0], p[2] - p[0]))


def _rotation(seed):
    q, _ = np.linalg.qr(np.random.default_rng(seed).standard_normal((3, 3)))
    return torch.tensor(q * np.sign(np.linalg.det(q)))


# ---- the restatements ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('op', OPS)
def test_translation_and_rotation_invariance(op):
    from dirt_b200 import mesh
    fn = getattr(mesh, '_' + op)
    v, f = _icosphere(2, noise=0.2)
    want = fn(v, f)
    moved = v @ _rotation(4).T + torch.tensor([0.3, -1.7, 2.5], dtype=torch.float64)
    assert torch.allclose(fn(moved, f), want, atol=1e-12, rtol=1e-9)


def test_zero_on_a_flat_grid():
    """Every interior entry is flat and every boundary entry has no partner: 0 throughout."""
    from dirt_b200.mesh import _normal_consistency
    v, f = _grid()
    out = _normal_consistency(v, f)
    assert out.shape == (f.shape[0], 3) and out.abs().max() < 1e-10   # 2e-12 / |n_f| from the 1e-12 in u_f
    bent = v.clone()
    bent[14, 2] = 0.5     # one interior vertex lifted: the entries around it are no longer 0
    assert _normal_consistency(bent, f).abs().max() > 1e-3


def test_cube():
    """0 across each quad's diagonal, 1 across the cube's 12 edges; the z = -1 quad is wound inward, which a reversed
    pair of faces does not change."""
    from dirt_b200 import scenes
    from dirt_b200.mesh import _normal_consistency, _edge_lengths
    v, f = scenes.cube()
    v, f = torch.tensor(v, dtype=torch.float64), torch.tensor(f)
    out, lengths = _normal_consistency(v, f), _edge_lengths(v, f)
    diagonal = lengths > 2.5
    assert int(diagonal.sum()) == 12 and bool((diagonal.sum(1) == 1).all())
    assert out[diagonal].abs().max() < 1e-12
    assert (out[~diagonal] - 1.).abs().max() < 1e-12


@pytest.mark.parametrize('level', [1, 2, 3])
def test_both_entries_of_every_edge_are_equal_on_a_closed_mesh(level):
    from dirt_b200.mesh import _normal_consistency
    v, f = _icosphere(level, noise=0.2)
    out = _normal_consistency(v, f)
    seen = {}
    for face, (a, b, c) in enumerate(f.tolist()):
        for k, (x, y) in enumerate(((a, b), (b, c), (c, a))):
            seen.setdefault((min(x, y), max(x, y)), []).append(out[face, k].item())
    assert len(seen) == 3 * f.shape[0] // 2 and all(len(s) == 2 for s in seen.values())
    assert max(abs(s[0] - s[1]) for s in seen.values()) < 1e-15
    assert min(s[0] for s in seen.values()) > 0.


def test_a_reversed_face_gives_about_2_on_its_edges():
    from dirt_b200.mesh import _normal_consistency
    v, f = _icosphere(2)
    f = f.clone()
    f[7] = f[7, [0, 2, 1]]
    out = _normal_consistency(v, f)
    assert (out[7] > 1.9).all() and (out[7] < 2.).all()
    assert out.max() == out[7].max()


def _check_explicit(v, f, want):
    from dirt_b200.mesh import _normal_consistency
    got = _normal_consistency(v, torch.tensor(f))
    assert np.allclose(got.numpy(), np.array(want), atol=1e-12), (got, want)


def test_a_non_manifold_edge_averages_over_all_its_other_faces():
    v = torch.tensor([[0., 0., 0.], [1., 0., 0.], [0.3, 1., 0.], [0.4, -0.5, 0.8], [0.6, 0.2, -0.9]],
                     dtype=torch.float64)
    f = [[0, 1, 2], [1, 0, 3], [0, 1, 4]]   # three faces on the edge {0, 1}
    u = [_face_unit(v, face) for face in f]
    want = np.zeros((3, 3))
    for i, k in ((0, 0), (1, 0), (2, 0)):
        others = [u[j] for j in range(3) if j != i]
        want[i, k] = 1. - u[i] @ (others[0] + others[1]) / 2.
    _check_explicit(v, f, want)


def test_a_duplicated_face_is_a_partner_of_its_copy():
    v = torch.tensor([[0., 0., 0.], [1., 0., 0.], [0.3, 1., 0.], [0.5, -1., 0.6]], dtype=torch.float64)
    f = [[0, 1, 2], [0, 1, 2], [1, 0, 3]]
    u = [_face_unit(v, face) for face in f]
    want = np.zeros((3, 3))
    want[0, 0] = 1. - u[0] @ (u[1] + u[2]) / 2.
    want[1, 0] = 1. - u[1] @ (u[0] + u[2]) / 2.
    want[2, 0] = 1. - u[2] @ (u[0] + u[1]) / 2.
    want[0, 1:] = want[1, 1:] = 1. - u[0] @ u[1]    # edges {1, 2} and {2, 0}: the copy alone
    _check_explicit(v, f, want)


def test_a_face_naming_a_vertex_twice_counts_once():
    """(0, 0, 1) has zero area (u = 0) and two edges on {0, 1}; it is one partner of the faces on that edge, and its
    edge (0, 0) is 0."""
    v = torch.tensor([[0., 0., 0.], [1., 0., 0.], [0.3, 1., 0.], [0.5, -1., 0.6]], dtype=torch.float64)
    f = [[0, 1, 2], [1, 0, 3], [0, 0, 1]]
    u = [_face_unit(v, face) for face in f]
    assert not u[2].any()
    want = np.zeros((3, 3))
    want[0, 0] = 1. - u[0] @ u[1] / 2.
    want[1, 0] = 1. - u[1] @ u[0] / 2.
    want[2, 1] = want[2, 2] = 1.
    _check_explicit(v, f, want)


def test_a_zero_area_face_has_value_1():
    v = torch.tensor([[0., 0., 0.], [1., 0., 0.], [0.3, 1., 0.], [0.5, 0., 0.]], dtype=torch.float64)
    f = [[0, 1, 2], [1, 0, 3]]     # face 1 is collinear
    u = _face_unit(v, f[0])
    _check_explicit(v, f, [[1., 0., 0.], [1., 0., 0.]])
    assert np.linalg.norm(u) > 0.99


def test_edge_lengths_against_numpy():
    from dirt_b200.mesh import _edge_lengths
    v, f = _icosphere(2, noise=0.3)
    p, ff = v.numpy(), f.numpy()
    want = np.stack([np.linalg.norm(p[ff[:, (k + 1) % 3]] - p[ff[:, k]], axis=1) for k in range(3)], 1)
    assert np.allclose(_edge_lengths(v, f).numpy(), want, rtol=1e-14, atol=0)
    w = torch.cat([v, torch.rand(v.shape[0], 1, dtype=v.dtype)], -1)
    assert torch.equal(_edge_lengths(w, f), _edge_lengths(v, f))


def test_a_zero_length_edge_passes_no_gradient():
    from dirt_b200.mesh import _edge_lengths
    v = torch.tensor([[0., 0., 0.], [1., 0., 0.], [0.3, 1., 0.]], dtype=torch.float64, requires_grad=True)
    out = _edge_lengths(v, torch.tensor([[0, 0, 1]]))
    assert out[0, 0] == 0.
    out[0, 0].backward()
    assert not v.grad.any()


@pytest.mark.parametrize('op', OPS)
def test_gradcheck(op):
    from dirt_b200 import mesh
    fn = getattr(mesh, '_' + op)
    v, f = _icosphere(1, noise=0.2)
    v = v.requires_grad_(True)
    w = torch.cat([v.detach(), torch.ones(v.shape[0], 1, dtype=v.dtype)], -1).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda x: fn(x, f), (v,))
    assert torch.autograd.gradgradcheck(lambda x: fn(x, f), (v,))
    assert torch.autograd.gradcheck(lambda x: fn(x, f), (w,))
    # an open mesh with a boundary, a non-manifold edge and a duplicated face
    g, gf = _grid(4)
    g = (g + 0.1 * torch.tensor(np.random.default_rng(5).standard_normal(g.shape))).requires_grad_(True)
    gf = torch.cat([gf, gf[:1], torch.tensor([[0, 1, 15]])])
    assert torch.autograd.gradcheck(lambda x: fn(x, gf), (g,))


# ---- the C ABI ----------------------------------------------------------------------------------------------------------

def _p(x):
    return ctypes.c_void_p(x)


def _fwd(L, mode=LEN, B=2, V=8, F=4, stride=3, vertices=4096, faces=4096, out=4096, ws=4096, ws_bytes=1 << 20):
    return L.dirt_edge_terms_forward(mode, _p(vertices), stride, _p(faces), _p(out), _p(ws), ws_bytes, B, V, F, None)


def _bwd(L, mode=LEN, B=2, V=8, F=4, stride=3, vertices=4096, faces=4096, grad=4096, out=4096, ws=4096,
         ws_bytes=1 << 20):
    return L.dirt_edge_terms_backward(mode, _p(vertices), stride, _p(faces), _p(grad), _p(out), _p(ws), ws_bytes, B, V,
                                      F, None)


def test_edge_terms_abi_rejects_bad_shapes(L):
    from dirt_b200 import _lib
    for call in (_fwd, _bwd):
        for kw in (dict(mode=2), dict(mode=-1), dict(B=-1), dict(V=-1), dict(F=-1), dict(stride=2), dict(stride=-4),
                   dict(V=1 << 31), dict(F=(1 << 31) // 3 + 1), dict(B=1 << 30, V=1 << 30, stride=1 << 20)):
            for mode in (LEN, CONS):
                args = dict(dict(mode=mode), **kw)
                assert call(L, **args) == _lib.ERR_BAD_SHAPE, args
                assert L.dirt_last_launch_count() == 0
    assert L.dirt_edge_terms_workspace_bytes(1, (1 << 31) - 1, 1) > 0
    assert L.dirt_edge_terms_workspace_bytes(1, 3, ((1 << 31) - 1) // 3) > 0


def test_edge_terms_abi_rejects_null_and_misaligned_pointers(L):
    from dirt_b200 import _lib
    for mode in (LEN, CONS):
        for call in (_fwd, _bwd):
            for name in ('vertices', 'faces', 'out', 'ws'):
                assert call(L, mode, **{name: 0}) == _lib.ERR_NULL_POINTER, name
                assert L.dirt_last_launch_count() == 0
                assert call(L, mode, **{name: 4098}) == _lib.ERR_MISALIGNED, name
                assert L.dirt_last_launch_count() == 0
            assert call(L, mode, ws_bytes=L.dirt_edge_terms_workspace_bytes(2, 8, 4) - 1) == \
                _lib.ERR_WORKSPACE_TOO_SMALL
            # the Laplacian's workspace is too small when there are more faces than vertices: the consistency
            # backward's scratch is 3 floats per (item, face)
            assert call(L, mode, B=64, V=10, F=1000, ws_bytes=L.dirt_laplacian_workspace_bytes(64, 10, 1000)) == \
                _lib.ERR_WORKSPACE_TOO_SMALL
            assert L.dirt_last_launch_count() == 0
        assert _bwd(L, mode, grad=0) == _lib.ERR_NULL_POINTER
        assert _bwd(L, mode, grad=4098) == _lib.ERR_MISALIGNED
        # V = 0 with faces: the forward only zeroes out, so out alone is checked
        assert _fwd(L, mode, V=0, vertices=0, faces=0, ws=0, ws_bytes=0, out=0) == _lib.ERR_NULL_POINTER
        assert _fwd(L, mode, V=0, vertices=0, faces=0, ws=0, ws_bytes=0, out=4098) == _lib.ERR_MISALIGNED
    assert L.dirt_last_launch_count() == 0


def test_edge_terms_abi_with_nothing_to_do_launches_nothing(L):
    from dirt_b200 import _lib
    for B, V, F in ((0, 8, 4), (3, 8, 0), (0, 0, 0), (0, 8, 0), (0, 0, 4)):
        for mode in (LEN, CONS):
            assert _fwd(L, mode, B=B, V=V, F=F, vertices=0, faces=0, out=0, ws=0, ws_bytes=0) == 0
            assert L.dirt_last_launch_count() == 0
    for B, V, F in ((0, 8, 4), (3, 0, 4), (0, 0, 0), (0, 8, 0), (3, 0, 0)):
        for mode in (LEN, CONS):   # no vertex rows: the backward has nothing to write
            assert _bwd(L, mode, B=B, V=V, F=F, vertices=0, faces=0, grad=0, out=0, ws=0, ws_bytes=0) == 0
            assert L.dirt_last_launch_count() == 0
    for mode in (LEN, CONS):   # no faces: the backward only zeroes grad_vertices, so it alone is checked
        assert _bwd(L, mode, B=3, V=8, F=0, vertices=0, faces=0, grad=0, out=0, ws=0, ws_bytes=0) == \
            _lib.ERR_NULL_POINTER
        assert _bwd(L, mode, B=3, V=8, F=0, vertices=0, faces=0, grad=0, out=4098, ws=0, ws_bytes=0) == \
            _lib.ERR_MISALIGNED
        assert L.dirt_last_launch_count() == 0


def _expected_workspace(B, V, F):
    up = lambda n: (n + 255) // 256 * 256
    if B == 0 or V == 0 or F == 0:
        return 0
    return up(4 * (V + 1)) + up(4 * 3 * F) + up(max(up(4 * V) + 4 * 3 * F, 4 * 3 * B * F))


def test_edge_terms_workspace_is_a_pure_function_of_the_shapes(L):
    W = L.dirt_edge_terms_workspace_bytes
    for B, V, F in ((0, 10, 5), (2, 0, 5), (2, 10, 0), (1, 1, 1), (2, 100, 50), (64, 2562, 5120), (64, 24866, 49728),
                    (1, 1000, 100000), (3, 7, 11), (1, 523266, 1046528), (70000, 8, 12)):
        assert W(B, V, F) == _expected_workspace(B, V, F), (B, V, F)
        assert W(B, V, F) == W(B, V, F)
    assert W(-1, 10, 5) == 0 and W(1, 1 << 31, 5) == 0 and W(1, 10, -1) == 0


# ---- routing ------------------------------------------------------------------------------------------------------------

def test_edge_terms_route_is_the_normals_route():
    """Accepted calls go to the op's _MeshOp with [B*V, 3] rows (a w column dropped) and per-face output rows; the
    routing decision is lighting.normals_route, whose refusals are listed in test_normals_host.py."""
    from dirt_b200 import mesh
    from dirt_b200.lighting import normals_route
    seen = []
    real_route, real_mesh = mesh._normals_route, mesh._mesh
    try:
        mesh._normals_route = lambda v, f: normals_route(v.shape, v.dtype, CUDA, torch.as_tensor(f).shape,
                                                         torch.as_tensor(f).dtype)
        mesh._mesh = lambda op, route, faces, rows: seen.append((op, route, rows.shape, rows.stride()))
        v, f = _icosphere(1, torch.float32)
        x = torch.cat([v, torch.ones(v.shape[0], 1)], -1).expand(2, 3, -1, -1)
        for name, op in (('edge_lengths', mesh._EDGE_LENGTHS), ('normal_consistency', mesh._NORMAL_CONSISTENCY)):
            getattr(mesh, name)(x, f)
            got, route, shape, stride = seen.pop()
            assert got is op and route.lead == (2, 3) and route.F == f.shape[0] and shape == (6 * v.shape[0], 3)
            assert stride[1] == 1 and stride[0] >= 3
            assert op.rows == 'F' and op.width == 3 and op.input_widths == (3,)
            assert op.inputs(route, f, torch.zeros(6, 3))[0] == mesh.EDGE_MODES[name]
            getattr(mesh, name)(x.double(), f)                        # float64: the restatement
            assert not seen
    finally:
        mesh._normals_route, mesh._mesh = real_route, real_mesh
    assert mesh.EDGE_MODES == {'edge_lengths': LEN, 'normal_consistency': CONS}
    assert {op.rows for op in (mesh._LAPLACIAN['uniform'], mesh._LAPLACIAN['cotangent'])} == {'V'}


# ---- CPU calls ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('op', OPS)
@pytest.mark.parametrize('w', [False, True])
def test_cpu_calls_return_the_restatement(op, w):
    import dirt_b200
    public, restate = getattr(dirt_b200.mesh, op), getattr(dirt_b200.mesh, '_' + op)
    v, f = _icosphere(2, torch.float32)
    for lead in ((), (2,), (2, 3)):
        n = math.prod(lead)
        x = v * (1. + 0.3 * torch.rand((n, v.shape[0], 1), generator=torch.Generator().manual_seed(len(lead))))
        x = x.reshape(lead + v.shape)
        if w:
            x = torch.cat([x, torch.ones(x.shape[:-1] + (1,))], -1)
        want = restate(x, f)
        assert want.shape == lead + (f.shape[0], 3)
        assert torch.equal(public(x, f), want)
        assert torch.equal(public(x, f.int()), want)
    got = public(v.double(), f)
    assert got.dtype == torch.float64 and torch.equal(got, restate(v.double(), f))
    got = public(v.numpy(), f.numpy().tolist())
    assert got.dtype == torch.float32 and torch.equal(got, restate(v, f))
    a, b = v.clone().requires_grad_(True), v.clone().requires_grad_(True)
    public(a, f).square().sum().backward()
    restate(b, f).square().sum().backward()
    assert torch.equal(a.grad, b.grad)


def test_cpu_calls_keep_their_errors():
    from dirt_b200 import mesh
    v, f = _icosphere(1, torch.float32)
    bad = f.clone()
    bad[3, 1] = v.shape[0]
    for op in OPS:
        with pytest.raises(IndexError):
            getattr(mesh, op)(v, bad)
