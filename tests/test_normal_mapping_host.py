"""CPU: the vertex tangents' and the normal mapping's C ABI reject bad arguments before anything is launched, the
tangents' workspace size is a function of the sizes alone, the routing decisions accept exactly the shapes the kernels
take, CPU calls run the torch restatements, and the restatements have the properties DESIGN.md §7.14 states."""
import ctypes

import numpy as np
import pytest
import torch

CUDA = torch.device('cuda', 0)
CPU = torch.device('cpu')
F32, F64, I32, I64 = torch.float32, torch.float64, torch.int32, torch.int64


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _p(x):
    return ctypes.c_void_p(x)


def _tfwd(L, B=2, V=8, F=4, vs=3, us=2, uis=16, ns=3, vertices=4096, uvs=4096, normals=4096, faces=4096, out=4096,
          ws=4096, ws_bytes=1 << 20):
    return L.dirt_tangents_forward(_p(vertices), vs, _p(uvs), us, uis, _p(normals), ns, _p(faces), _p(out), _p(ws),
                                   ws_bytes, B, V, F, None)


def _tbwd(L, B=2, V=8, F=4, vs=3, us=2, uis=16, ns=3, vertices=4096, uvs=4096, normals=4096, faces=4096, grad=4096,
          gv=4096, gu=4096, gn=4096, ws=4096, ws_bytes=1 << 20):
    return L.dirt_tangents_backward(_p(vertices), vs, _p(uvs), us, uis, _p(normals), ns, _p(faces), _p(grad), _p(gv),
                                    _p(gu), _p(gn), _p(ws), ws_bytes, B, V, F, None)


def _mfwd(L, B=2, V=8, sn=3, st=4, sm=3, normals=4096, tangents=4096, samples=4096, out=4096):
    return L.dirt_normal_map_forward(_p(normals), sn, _p(tangents), st, _p(samples), sm, _p(out), B, V, None)


def _mbwd(L, B=2, V=8, sn=3, st=4, sm=3, normals=4096, tangents=4096, samples=4096, grad=4096, gn=4096, gt=4096,
          gm=4096):
    return L.dirt_normal_map_backward(_p(normals), sn, _p(tangents), st, _p(samples), sm, _p(grad), _p(gn), _p(gt),
                                      _p(gm), B, V, None)


# ---- the C ABI ------------------------------------------------------------------------------------------------------

def test_tangents_abi_rejects_bad_shapes(L):
    from dirt_b200 import _lib
    for call in (_tfwd, _tbwd):
        for kw in (dict(B=-1), dict(V=-1), dict(F=-1), dict(vs=2), dict(us=1), dict(us=-2), dict(uis=-1), dict(ns=2),
                   dict(V=1 << 31), dict(F=(1 << 31) // 3 + 1), dict(B=1 << 30, V=1 << 30, vs=1 << 20)):
            assert call(L, **kw) == _lib.ERR_BAD_SHAPE, kw
            assert L.dirt_last_launch_count() == 0


def test_tangents_abi_rejects_null_and_misaligned_pointers(L):
    from dirt_b200 import _lib
    for call in (_tfwd, _tbwd):
        for name in ('vertices', 'uvs', 'normals', 'faces', 'ws'):
            assert call(L, **{name: 0}) == _lib.ERR_NULL_POINTER, name
            assert call(L, **{name: 4098}) == _lib.ERR_MISALIGNED, name
        assert call(L, ws_bytes=L.dirt_tangents_workspace_bytes(2, 8, 4) - 1) == _lib.ERR_WORKSPACE_TOO_SMALL
    assert _tfwd(L, out=0) == _lib.ERR_NULL_POINTER
    assert _tfwd(L, out=4098) == _lib.ERR_MISALIGNED
    assert _tbwd(L, grad=0) == _lib.ERR_NULL_POINTER
    assert _tbwd(L, grad=4098) == _lib.ERR_MISALIGNED
    for name in ('gv', 'gu', 'gn'):
        assert _tbwd(L, **{name: 4098}) == _lib.ERR_MISALIGNED, name
    assert L.dirt_last_launch_count() == 0


def test_tangents_abi_with_nothing_to_do_launches_nothing(L):
    for B, V in ((0, 8), (3, 0), (0, 0)):
        assert _tfwd(L, B=B, V=V, vertices=0, uvs=0, normals=0, faces=0, out=0, ws=0, ws_bytes=0) == 0
        assert L.dirt_last_launch_count() == 0
        assert _tbwd(L, B=B, V=V, vertices=0, uvs=0, normals=0, faces=0, grad=0, gv=0, gu=0, gn=0, ws=0,
                     ws_bytes=0) == 0
        assert L.dirt_last_launch_count() == 0
    # no gradient wanted: nothing is read, nothing is launched
    assert _tbwd(L, vertices=0, uvs=0, normals=0, faces=0, grad=0, gv=0, gu=0, gn=0, ws=0, ws_bytes=0) == 0
    assert L.dirt_last_launch_count() == 0


def test_tangents_workspace_is_the_normals_workspace(L):
    up = lambda n: (n + 255) // 256 * 256
    for B, V, F in ((0, 10, 5), (2, 0, 5), (2, 10, 0), (1, 1, 1), (2, 100, 50), (64, 25088, 49728),
                    (1, 525312, 1046528), (3, 7, 11)):
        want = 0 if B == 0 or V == 0 or F == 0 else \
            up(4 * (V + 1)) + up(4 * 3 * F) + up(max(up(4 * V) + 4 * 3 * F, 4 * 3 * B * V))
        assert L.dirt_tangents_workspace_bytes(B, V, F) == want == L.dirt_normals_workspace_bytes(B, V, F), (B, V, F)
    assert L.dirt_tangents_workspace_bytes(-1, 10, 5) == 0 and L.dirt_tangents_workspace_bytes(1, 1 << 31, 5) == 0


def test_normal_map_abi_rejects_bad_arguments(L):
    from dirt_b200 import _lib
    for call in (_mfwd, _mbwd):
        for kw in (dict(B=-1), dict(V=-1), dict(sn=-3), dict(st=-4), dict(sm=-1), dict(B=1 << 30, V=1 << 30, st=1 << 20)):
            assert call(L, **kw) == _lib.ERR_BAD_SHAPE, kw
        for name in ('normals', 'tangents', 'samples'):
            assert call(L, **{name: 0}) == _lib.ERR_NULL_POINTER, name
            assert call(L, **{name: 4098}) == _lib.ERR_MISALIGNED, name
        assert L.dirt_last_launch_count() == 0
    assert _mfwd(L, out=0) == _lib.ERR_NULL_POINTER and _mfwd(L, out=4098) == _lib.ERR_MISALIGNED
    assert _mbwd(L, grad=0) == _lib.ERR_NULL_POINTER and _mbwd(L, grad=4098) == _lib.ERR_MISALIGNED
    for name in ('gn', 'gt', 'gm'):
        assert _mbwd(L, **{name: 4098}) == _lib.ERR_MISALIGNED, name
    # nothing to do
    assert _mfwd(L, B=0, normals=0, tangents=0, samples=0, out=0) == 0
    assert _mfwd(L, V=0, normals=0, tangents=0, samples=0, out=0) == 0
    assert _mbwd(L, normals=0, tangents=0, samples=0, grad=0, gn=0, gt=0, gm=0) == 0
    assert L.dirt_last_launch_count() == 0


# ---- routing --------------------------------------------------------------------------------------------------------

def test_tangents_route_accepts_the_plain_shapes():
    from dirt_b200.lighting import tangents_route
    r = tangents_route(((2562, 3), F32, CUDA), ((2562, 2), F32, CUDA), ((2562, 3), F32, CUDA), (5120, 3), I32)
    assert (r.lead, r.B, r.V, r.F, r.uv_per_item) == ((), 1, 2562, 5120, False)
    r = tangents_route(((64, 100, 4), F32, CUDA), ((100, 2), F32, CUDA), ((64, 100, 3), F32, CUDA), (50, 3), I64)
    assert (r.lead, r.B, r.V, r.F, r.uv_per_item) == ((64,), 64, 100, 50, False)
    r = tangents_route(((2, 3, 7, 3), F32, CUDA), ((2, 3, 7, 2), F32, CUDA), ((2, 3, 7, 3), F32, CUDA), (4, 3), I32)
    assert (r.lead, r.B, r.V, r.F, r.uv_per_item) == ((2, 3), 6, 7, 4, True)
    assert tangents_route(((0, 7, 3), F32, CUDA), ((7, 2), F32, CUDA), ((0, 7, 3), F32, CUDA), (4, 3), I32).B == 0
    assert tangents_route(((7, 3), F32, CUDA), ((7, 2), F32, CUDA), ((7, 3), F32, CUDA), (0, 3), I32).F == 0


def test_tangents_route_refuses_everything_else():
    from dirt_b200.lighting import tangents_route
    v, uv, n, f = ((10, 3), F32, CUDA), ((10, 2), F32, CUDA), ((10, 3), F32, CUDA), (4, 3)
    assert tangents_route(v, uv, n, f, I32) is not None
    assert tangents_route(((10, 3), F32, CPU), ((10, 2), F32, CPU), ((10, 3), F32, CPU), f, I32) is None   # CPU
    assert tangents_route(((10, 3), F64, CUDA), uv, n, f, I32) is None                  # dtypes
    assert tangents_route(v, ((10, 2), F64, CUDA), n, f, I32) is None
    assert tangents_route(v, uv, ((10, 3), torch.float16, CUDA), f, I32) is None
    assert tangents_route(v, uv, n, f, torch.int16) is None
    other = torch.device('cuda', 1)
    assert tangents_route(v, ((10, 2), F32, other), n, f, I32) is None                  # devices
    assert tangents_route(v, uv, ((10, 3), F32, CPU), f, I32) is None
    assert tangents_route(v, ((10, 3), F32, CUDA), n, f, I32) is None                   # uv width
    assert tangents_route(v, ((9, 2), F32, CUDA), n, f, I32) is None                    # uv count
    assert tangents_route(v, ((2, 10, 2), F32, CUDA), n, f, I32) is None                # uv batch without vertex batch
    assert tangents_route(((2, 10, 3), F32, CUDA), ((3, 10, 2), F32, CUDA), ((2, 10, 3), F32, CUDA), f, I32) is None
    assert tangents_route(((2, 10, 3), F32, CUDA), uv, n, f, I32) is None               # normals without the batch
    assert tangents_route(v, uv, ((10, 4), F32, CUDA), f, I32) is None                  # normal width
    assert tangents_route(v, uv, n, (4, 4), I32) is None                                # quads
    assert tangents_route(((10, 2), F32, CUDA), uv, n, f, I32) is None                  # 2-column vertices


def test_perturb_route_is_the_lighting_route():
    from dirt_b200.lighting import cuda_route
    ok = lambda shapes: cuda_route(shapes, [], [CUDA] * 3, [3, 4, 3])
    r = ok([(64, 512, 512, 3), (64, 512, 512, 4), (64, 512, 512, 3)])
    assert (r.lead, r.B, r.V) == ((64, 512), 64 * 512, 512)
    assert ok([(5, 3), (5, 4), (5, 3)]).B == 1
    assert ok([(5, 3), (5, 4), (5, 2)]) is None
    assert ok([(5, 3), (5, 3), (5, 3)]) is None
    assert ok([(2, 5, 3), (5, 4), (2, 5, 3)]) is None
    assert cuda_route([(5, 3), (5, 4), (5, 3)], [], [CUDA, CPU, CUDA], [3, 4, 3]) is None


# ---- CPU calls and the restatements -----------------------------------------------------------------------------------

def _sphere(lead=(), seed=0, w=False):
    """A uv sphere with a seam column: `scenes.uv_sphere`'s positions with their longitude and latitude as uvs."""
    from dirt_b200 import scenes
    v, f = scenes.uv_sphere(16, 8)
    v = v.astype(np.float64)
    uv = np.stack([np.arctan2(v[:, 0], v[:, 2]) / (2 * np.pi) + 0.5, np.arccos(np.clip(v[:, 1], -1, 1)) / np.pi], -1)
    r = np.random.default_rng(seed)
    x = v[None] * (1. + 0.1 * r.standard_normal((int(np.prod(lead)) if lead else 1, v.shape[0], 1)))
    x = x.reshape(lead + v.shape)
    if w:
        x = np.concatenate([x, np.ones(x.shape[:-1] + (1,))], -1)
    return torch.from_numpy(x), torch.from_numpy(uv), torch.from_numpy(f)


@pytest.mark.parametrize('dtype', [F32, F64])
def test_cpu_calls_return_the_restatements(dtype):
    from dirt_b200 import lighting
    for lead, w in (((), False), ((2,), True), ((2, 3), False)):
        x, uv, f = _sphere(lead, len(lead), w)
        x, uv = x.to(dtype), uv.to(dtype)
        n = lighting._vertex_normals(x, f)
        got = lighting.vertex_tangents(x, uv, f, n)
        assert got.dtype == dtype and got.shape == lead + (x.shape[-2], 4)
        assert torch.equal(got, lighting._vertex_tangents(x, uv, f, n))
        assert torch.equal(lighting.vertex_tangents(x, uv, f.long(), n), got)
        m = torch.nn.functional.normalize(torch.randn(n.shape, dtype=dtype), dim=-1)
        assert torch.equal(lighting.perturb_normals(n, got, m),
                           lighting._perturb_normals(n.float(), got.float(), m.float()))
    # gradients as before
    x, uv, f = _sphere((2,), 5)
    a, b = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    n = lighting._vertex_normals(x, f)
    lighting.vertex_tangents(a, uv, f, n).square().sum().backward()
    lighting._vertex_tangents(b, uv, f, n).square().sum().backward()
    assert torch.equal(a.grad, b.grad)


def test_cpu_calls_keep_their_errors():
    from dirt_b200 import lighting
    x, uv, f = _sphere()
    bad = f.clone()
    bad[3, 1] = x.shape[0]
    with pytest.raises(IndexError):
        lighting.vertex_tangents(x, uv, bad, lighting._vertex_normals(x, f))


def test_tangents_are_unit_and_orthogonal_to_the_normals():
    from dirt_b200 import lighting
    x, uv, f = _sphere((3,), 7)
    n = lighting._vertex_normals(x, f)
    t = lighting._vertex_tangents(x, uv, f, n)
    T, w = t[..., :3], t[..., 3]
    assert torch.allclose(T.norm(dim=-1), torch.ones(()).double(), atol=1e-12)
    assert (n * T).sum(-1).abs().max() < 1e-9
    assert set(w.unique().tolist()) <= {-1., 1.}


def _quad():
    v = torch.tensor([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], dtype=F64)
    return v, v[:, :2].clone(), torch.tensor([[0, 1, 2], [0, 2, 3]])


def test_unit_quad_and_mirrored_uvs():
    from dirt_b200 import lighting
    v, uv, f = _quad()
    n = lighting._vertex_normals(v, f)
    t = lighting._vertex_tangents(v, uv, f, n)
    assert torch.allclose(t, torch.tensor([1., 0., 0., 1.], dtype=F64).expand(4, 4))
    mirrored = uv.clone()
    mirrored[:, 0] = 1. - mirrored[:, 0]
    t = lighting._vertex_tangents(v, mirrored, f, n)
    assert torch.allclose(t, torch.tensor([-1., 0., 0., -1.], dtype=F64).expand(4, 4))
    # the bitangent w (n x T) points along +v in both cases: here +y
    b = t[..., 3:] * torch.linalg.cross(n, t[..., :3], dim=-1)
    assert torch.allclose(b, torch.tensor([0., 1., 0.], dtype=F64).expand(4, 3))


def test_degenerate_uv_faces_add_nothing():
    from dirt_b200 import lighting
    v, uv, f = _quad()
    # a third face over the same corners with all three uvs on one line: r = 0
    v = torch.cat([v, torch.tensor([[0.3, 0.2, 0.1]], dtype=F64)])
    uv = torch.cat([uv, torch.tensor([[0.5, 0.5]], dtype=F64)])
    uv_line = uv.clone()
    uv_line[4] = torch.tensor([2., 2.], dtype=F64)           # on the line through uv0 and uv2
    f2 = torch.cat([f, torch.tensor([[0, 2, 4]])])
    n = lighting._vertex_normals(v, f)
    with_face = lighting._vertex_tangents(v, uv_line, f2, n)
    assert torch.equal(with_face[:4], lighting._vertex_tangents(v[:4], uv[:4], f, n[:4]))
    assert torch.equal(with_face[4], torch.tensor([0., 0., 0., 1.], dtype=F64))   # named by no valid face


def test_a_seam_gives_each_side_its_own_frame():
    """Two quads sharing an edge in space but not in uv: the seam vertices are split, and the side whose u runs the
    other way gets its own, mirrored frame, while the positions along the seam agree."""
    from dirt_b200 import lighting
    v = torch.tensor([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0],             # left quad
                      [1, 0, 0], [2, 0, 0], [2, 1, 0], [1, 1, 0]], dtype=F64)  # right quad: seam copies 4, 7 of 1, 2
    uv = torch.tensor([[0, 0], [1, 0], [1, 1], [0, 1], [1, 0], [0, 0], [0, 1], [1, 1]], dtype=F64)   # mirrored in u
    f = torch.tensor([[0, 1, 2], [0, 2, 3], [4, 5, 6], [4, 6, 7]])
    n = lighting._vertex_normals(v, f)
    t = lighting._vertex_tangents(v, uv, f, n)
    assert torch.allclose(t[:4], torch.tensor([1., 0., 0., 1.], dtype=F64).expand(4, 4))
    assert torch.allclose(t[4:], torch.tensor([-1., 0., 0., -1.], dtype=F64).expand(4, 4))
    assert torch.equal(v[1], v[4]) and not torch.equal(t[1], t[4])


def test_tangent_uv_gradient_reaches_v_only():
    from dirt_b200 import lighting
    x, uv, f = _sphere((), 3)
    uv = (uv + 0.05 * torch.randn(uv.shape, dtype=F64, generator=torch.Generator().manual_seed(0))).requires_grad_(True)
    n = lighting._vertex_normals(x, f)
    (lighting._vertex_tangents(x, uv, f, n) * torch.randn(x.shape[:-1] + (4,), dtype=F64)).sum().backward()
    assert not uv.grad[:, 0].any() and uv.grad[:, 1].any()


def test_perturb_with_the_unperturbed_sample_returns_the_normal():
    from dirt_b200 import lighting
    g = torch.Generator().manual_seed(1)
    n = torch.randn(5, 64, 3, dtype=F64, generator=g) * 3.
    t = torch.cat([torch.randn(5, 64, 3, dtype=F64, generator=g), torch.randn(5, 64, 1, dtype=F64, generator=g)], -1)
    m = torch.tensor([0., 0., 1.], dtype=F64).expand(5, 64, 3)
    assert torch.allclose(lighting._perturb_normals(n, t, m), torch.nn.functional.normalize(n, dim=-1), atol=1e-12)
    # background pixels: 0
    assert not lighting._perturb_normals(torch.zeros(4, 3, dtype=F64), torch.zeros(4, 4, dtype=F64),
                                         torch.rand(4, 3, dtype=F64)).any()
    # m = (1, 0, 0) gives T, m = (0, 1, 0) the bitangent s (n x T)
    out = lighting._perturb_normals(n, t, torch.tensor([0., 1., 0.], dtype=F64).expand(5, 64, 3))
    nn = torch.nn.functional.normalize(n, dim=-1)
    T = torch.nn.functional.normalize(t[..., :3] - (nn * t[..., :3]).sum(-1, keepdim=True) * nn, dim=-1)
    s = torch.where(t[..., 3:] < 0, -1., 1.).to(F64)
    assert torch.allclose(out, s * torch.linalg.cross(nn, T, dim=-1), atol=1e-10)
