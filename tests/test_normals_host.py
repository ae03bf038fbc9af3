"""CPU: the vertex normals' C ABI rejects bad arguments before anything is launched, its workspace size is a function of
the sizes alone, the routing decision accepts exactly the shapes the kernels take, and CPU calls run the torch
restatement unchanged."""
import ctypes

import numpy as np
import pytest
import torch

AVG, PRE = 0, 1
CUDA = torch.device('cuda', 0)
CPU = torch.device('cpu')


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _p(x):
    return ctypes.c_void_p(x)


def _fwd(L, mode=AVG, B=2, V=8, F=4, stride=3, vertices=4096, faces=4096, out=4096, ws=4096, ws_bytes=1 << 20):
    return L.dirt_normals_forward(mode, _p(vertices), stride, _p(faces), _p(out), _p(ws), ws_bytes, B, V, F, None)


def _bwd(L, mode=AVG, B=2, V=8, F=4, stride=3, vertices=4096, faces=4096, grad=4096, out=4096, ws=4096,
         ws_bytes=1 << 20):
    return L.dirt_normals_backward(mode, _p(vertices), stride, _p(faces), _p(grad), _p(out), _p(ws), ws_bytes, B, V, F,
                                   None)


def test_normals_abi_rejects_bad_shapes(L):
    from dirt_b200 import _lib
    for call in (_fwd, _bwd):
        for kw in (dict(mode=2), dict(mode=-1), dict(B=-1), dict(V=-1), dict(F=-1), dict(stride=2), dict(stride=-4),
                   dict(V=1 << 31), dict(F=(1 << 31) // 3 + 1), dict(B=1 << 30, V=1 << 30, stride=1 << 20)):
            assert call(L, **kw) == _lib.ERR_BAD_SHAPE, kw
            assert L.dirt_last_launch_count() == 0
    # the largest accepted sizes
    assert L.dirt_normals_workspace_bytes(1, (1 << 31) - 1, 1) > 0
    assert L.dirt_normals_workspace_bytes(1, 3, ((1 << 31) - 1) // 3) > 0


def test_normals_abi_rejects_null_and_misaligned_pointers(L):
    from dirt_b200 import _lib
    for call in (_fwd, _bwd):
        for name in ('vertices', 'faces', 'out', 'ws'):
            assert call(L, **{name: 0}) == _lib.ERR_NULL_POINTER, name
            assert call(L, **{name: 4098}) == _lib.ERR_MISALIGNED, name
        assert call(L, ws_bytes=L.dirt_normals_workspace_bytes(2, 8, 4) - 1) == _lib.ERR_WORKSPACE_TOO_SMALL
    assert _bwd(L, grad=0) == _lib.ERR_NULL_POINTER
    assert _bwd(L, grad=4098) == _lib.ERR_MISALIGNED
    assert L.dirt_last_launch_count() == 0


def test_normals_abi_with_nothing_to_do_launches_nothing(L):
    for B, V in ((0, 8), (3, 0), (0, 0)):
        for mode in (AVG, PRE):
            assert _fwd(L, mode, B=B, V=V, vertices=0, faces=0, out=0, ws=0, ws_bytes=0) == 0
            assert L.dirt_last_launch_count() == 0
            assert _bwd(L, mode, B=B, V=V, vertices=0, faces=0, grad=0, out=0, ws=0, ws_bytes=0) == 0
            assert L.dirt_last_launch_count() == 0


def _expected_workspace(B, V, F):
    up = lambda n: (n + 255) // 256 * 256
    if B == 0 or V == 0 or F == 0:
        return 0
    return up(4 * (V + 1)) + up(4 * 3 * F) + up(max(up(4 * V) + 4 * 3 * F, 4 * 3 * B * V))


def test_normals_workspace_is_a_pure_function_of_the_shapes(L):
    W = L.dirt_normals_workspace_bytes
    for B, V, F in ((0, 10, 5), (2, 0, 5), (2, 10, 0), (1, 1, 1), (2, 100, 50), (64, 2562, 5120), (64, 24866, 49728),
                    (1, 1000, 100000), (3, 7, 11)):
        assert W(B, V, F) == _expected_workspace(B, V, F), (B, V, F)
        assert W(B, V, F) == W(B, V, F)
    assert W(-1, 10, 5) == 0 and W(1, 1 << 31, 5) == 0


def test_normals_route_accepts_the_plain_shapes():
    from dirt_b200.lighting import normals_route
    f32, i32, i64 = torch.float32, torch.int32, torch.int64
    r = normals_route((2562, 3), f32, CUDA, (5120, 3), i32)
    assert r is not None and (r.lead, r.B, r.V, r.F) == ((), 1, 2562, 5120)
    r = normals_route((64, 2562, 4), f32, CUDA, (5120, 3), i64)
    assert (r.lead, r.B, r.V, r.F) == ((64,), 64, 2562, 5120)
    r = normals_route((2, 3, 7, 3), f32, CUDA, (4, 3), i32)
    assert (r.lead, r.B, r.V, r.F) == ((2, 3), 6, 7, 4)
    assert normals_route((0, 7, 3), f32, CUDA, (4, 3), i32).B == 0
    assert normals_route((2, 0, 3), f32, CUDA, (0, 3), i64).V == 0
    assert normals_route((7, 3), f32, CUDA, (0, 3), i32).F == 0
    assert normals_route((7, 3), f32, torch.device('cuda', 1), (4, 3), i32) is not None
    assert normals_route(((1 << 31) - 1, 3), f32, CUDA, (((1 << 31) - 1) // 3, 3), i32) is not None


def test_normals_route_refuses_everything_else():
    from dirt_b200.lighting import normals_route
    f32, i32 = torch.float32, torch.int32
    assert normals_route((10, 3), f32, CPU, (4, 3), i32) is None                      # CPU
    assert normals_route((10, 3), torch.float64, CUDA, (4, 3), i32) is None           # float64
    assert normals_route((10, 3), torch.float16, CUDA, (4, 3), i32) is None
    assert normals_route((10, 3), f32, CUDA, (4, 3), torch.int16) is None             # face dtype
    assert normals_route((10, 3), f32, CUDA, (4, 3), torch.float32) is None
    assert normals_route((3,), f32, CUDA, (4, 3), i32) is None                        # no vertex axis
    assert normals_route((10, 2), f32, CUDA, (4, 3), i32) is None                     # 2 or 5 columns
    assert normals_route((10, 5), f32, CUDA, (4, 3), i32) is None
    assert normals_route((10, 3), f32, CUDA, (2, 4, 3), i32) is None                  # per-item faces
    assert normals_route((10, 3), f32, CUDA, (4, 4), i32) is None                     # quads
    assert normals_route((10, 3), f32, CUDA, (12,), i32) is None
    assert normals_route((1 << 31, 3), f32, CUDA, (4, 3), i32) is None                # V >= 2^31
    assert normals_route((10, 3), f32, CUDA, ((1 << 31) // 3 + 1, 3), i32) is None    # 3F >= 2^31
    assert normals_route((1 << 16, 1 << 15, 1, 3), f32, CUDA, (4, 3), i32) is None   # prod(*) >= 2^31


def _mesh(seed, lead=(), w=False):
    from dirt_b200 import scenes
    v, f = scenes.icosphere(2)
    r = np.random.default_rng(seed)
    v = v[None] * (1. + 0.3 * r.standard_normal((int(np.prod(lead)) if lead else 1, v.shape[0], 1)))
    v = v.reshape(lead + v.shape[1:]).astype(np.float32)
    if w:
        v = np.concatenate([v, np.ones(v.shape[:-1] + (1,), np.float32)], axis=-1)
    return torch.from_numpy(v), torch.from_numpy(f)


@pytest.mark.parametrize('w', [False, True])
def test_cpu_calls_return_the_restatement(w):
    from dirt_b200 import lighting
    for lead in ((), (2,), (2, 3)):
        v, f = _mesh(len(lead), lead, w)
        assert torch.equal(lighting.vertex_normals(v, f), lighting._vertex_normals(v, f))
        assert torch.equal(lighting.vertex_normals(v, f.long()), lighting._vertex_normals(v, f))
        sv, sf = lighting.split_vertices_by_face(v, f)
        assert torch.equal(lighting.vertex_normals_pre_split(sv, sf), lighting._vertex_normals_pre_split(sv, sf))
        assert torch.equal(lighting.vertex_normals_pre_split(sv, sf, static=True), lighting._vertex_normals_pre_split(sv, sf))
    # float64 stays float64, and array-likes are converted as before
    v, f = _mesh(5)
    got = lighting.vertex_normals(v.double(), f)
    assert got.dtype == torch.float64 and torch.equal(got, lighting._vertex_normals(v.double(), f))
    got = lighting.vertex_normals(v.numpy(), f.numpy().tolist())
    assert got.dtype == torch.float32 and torch.equal(got, lighting._vertex_normals(v, f))
    # gradients as before
    a, b = v.clone().requires_grad_(True), v.clone().requires_grad_(True)
    lighting.vertex_normals(a, f).square().sum().backward()
    lighting._vertex_normals(b, f).square().sum().backward()
    assert torch.equal(a.grad, b.grad)


def test_cpu_calls_keep_their_errors():
    from dirt_b200 import lighting
    v, f = _mesh(6)
    bad = f.clone()
    bad[3, 1] = v.shape[0]
    with pytest.raises(IndexError):
        lighting.vertex_normals(v, bad)
    with pytest.raises(IndexError):
        lighting.vertex_normals_pre_split(v, bad)
