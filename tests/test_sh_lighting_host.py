"""CPU: the spherical-harmonics lighting's restatement pins its convention (orthonormal basis, the uniform environment,
the 9-term clamped cosine), its C ABI rejects bad arguments before anything is launched, the routing decision accepts
exactly the plain shapes, and CPU calls run the restatement unchanged."""
import ctypes
import math

import numpy as np
import pytest
import torch

CUDA = torch.device('cuda', 0)


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _p(x):
    return ctypes.c_void_p(x)


def _sphere_rule():
    """Directions and weights of a product rule exact for polynomials of degree <= 15 on the sphere: 8-point
    Gauss-Legendre in cos(theta) times 16 uniform angles in phi."""
    t, wt = np.polynomial.legendre.leggauss(8)
    phi = np.arange(16) * (2 * math.pi / 16)
    T, P = np.meshgrid(t, phi, indexing='ij')
    s = np.sqrt(1 - T * T)
    dirs = np.stack([s * np.cos(P), s * np.sin(P), T], -1).reshape(-1, 3)
    weights = (wt[:, None] * np.full(16, 2 * math.pi / 16)[None]).reshape(-1)
    return torch.from_numpy(dirs), torch.from_numpy(weights)


def test_the_basis_is_orthonormal():
    from dirt_b200.lighting import _sh_basis
    dirs, weights = _sphere_rule()
    Y = _sh_basis(dirs)                                    # [N, 9] float64
    gram = (Y * weights[:, None]).T @ Y
    np.testing.assert_allclose(gram.numpy(), np.eye(9), rtol=0, atol=1e-12)


def _unit(g, shape):
    return torch.nn.functional.normalize(torch.randn(shape, generator=g, dtype=torch.float64), dim=-1)


def test_a_uniform_environment_returns_the_albedo():
    from dirt_b200.lighting import _diffuse_spherical_harmonics
    g = torch.Generator().manual_seed(0)
    for C in (1, 3, 4):
        n, albedo = _unit(g, (2, 50, 3)), torch.rand(2, 50, C, generator=g, dtype=torch.float64)
        L = torch.zeros(9, C, dtype=torch.float64)
        L[0] = 2 * math.sqrt(math.pi)
        np.testing.assert_allclose(_diffuse_spherical_harmonics(n, albedo, L).numpy(), albedo.numpy(), rtol=0, atol=1e-12)
        # per item, with a different radiance per item and channel
        scale = torch.rand(2, 1, C, generator=g, dtype=torch.float64) + 0.5
        Lb = L[None] * scale
        np.testing.assert_allclose(_diffuse_spherical_harmonics(n, albedo, Lb).numpy(), (albedo * scale).numpy(),
                                   rtol=0, atol=1e-12)


def test_a_projected_directional_light_gives_the_nine_term_clamped_cosine():
    from dirt_b200.lighting import _diffuse_spherical_harmonics, _sh_basis
    g = torch.Generator().manual_seed(1)
    for C in (1, 3):
        d = _unit(g, (3,))
        intensity = torch.rand(C, generator=g, dtype=torch.float64) + 0.5
        L = math.pi * _sh_basis(-d)[:, None] * intensity[None]          # [9, C]
        n, albedo = _unit(g, (200, 3)), torch.rand(200, C, generator=g, dtype=torch.float64)
        c = (n @ -d)[:, None]
        want = albedo * intensity * (0.25 + c / 2 + 5 * (3 * c * c - 1) / 32)
        np.testing.assert_allclose(_diffuse_spherical_harmonics(n, albedo, L).numpy(), want.numpy(), rtol=0, atol=1e-12)
    # it approximates max(c, 0), the single-sided diffuse model, to within 3/32 of the light's intensity (the
    # error at c = 0, where 1/4 - 5/32 remains)
    from dirt_b200.lighting import _diffuse_directional
    d = torch.tensor([0., 0., -1.], dtype=torch.float64)
    n = _unit(g, (2000, 3))
    ones = torch.ones(2000, 1, dtype=torch.float64)
    sh = _diffuse_spherical_harmonics(n, ones, math.pi * _sh_basis(-d)[:, None])
    exact = _diffuse_directional(n, ones, d, torch.ones(1, dtype=torch.float64), double_sided=False)
    assert float((sh - exact).abs().max()) <= 3 / 32 + 1e-12


def _fwd(L, B=1, V=8, C=3, strides=(3, 3), ptrs=None, out=None, per_item=0):
    ok = _p(4096)
    n, k, c = ptrs if ptrs is not None else [ok] * 3
    return L.dirt_sh_lighting_forward(n, strides[0], k, strides[1], c, per_item, ok if out is None else out, B, V, C, None)


def _bwd(L, B=1, V=8, C=3, strides=(3, 3), ptrs=None, grad_out=None, grads=None, ws=None, ws_bytes=1 << 20, per_item=1):
    ok = _p(4096)
    n, k, c = ptrs if ptrs is not None else [ok] * 3
    grads = grads if grads is not None else [ok] * 3
    return L.dirt_sh_lighting_backward(n, strides[0], k, strides[1], c, per_item, ok if grad_out is None else grad_out,
                                       *grads, ok if ws is None else ws, ws_bytes, B, V, C, None)


def test_sh_abi_rejects_bad_shapes(L):
    from dirt_b200 import _lib
    for call in (_fwd, _bwd):
        assert call(L, B=-1) == _lib.ERR_BAD_SHAPE
        assert call(L, V=-1) == _lib.ERR_BAD_SHAPE
        assert call(L, C=0) == _lib.ERR_BAD_SHAPE
        assert call(L, C=(1 << 26) + 1) == _lib.ERR_BAD_SHAPE            # 9*C must stay an int
        assert call(L, strides=(-3, 3)) == _lib.ERR_BAD_SHAPE
        assert call(L, strides=(3, -1)) == _lib.ERR_BAD_SHAPE
        assert call(L, B=1 << 30, V=1 << 40) == _lib.ERR_BAD_SHAPE      # element offsets past 2^62
        assert call(L, V=1 << 50, C=1) == _lib.ERR_BAD_SHAPE           # more chunks than the grid holds
        assert L.dirt_last_launch_count() == 0


def test_sh_workspace_is_a_pure_function_of_the_shapes(L):
    W = L.dirt_sh_lighting_workspace_bytes
    assert W(0, 100, 3) == 0 and W(4, 0, 3) == 0 and W(4, 100, 0) == 0
    assert W(1, 1, 3) == 4 * 27
    assert W(64, 512 * 512, 3) == 4 * 64 * 128 * 27          # 2048 points per partial row
    assert W(2, 2049, 5) == 4 * 2 * 2 * 45
    assert W(3, 1000, 4) == W(3, 1000, 4)


def test_sh_abi_with_no_points_launches_nothing(L):
    null = _p(0)
    for B, V in ((0, 8), (3, 0)):
        for per_item in (0, 1):
            assert _fwd(L, B=B, V=V, ptrs=[null] * 3, out=null, per_item=per_item) == 0
            assert L.dirt_last_launch_count() == 0
            assert _bwd(L, B=B, V=V, ptrs=[null] * 3, grad_out=null, grads=[null] * 3, ws=null, ws_bytes=0,
                        per_item=per_item) == 0
            assert L.dirt_last_launch_count() == 0


def test_sh_abi_rejects_null_and_misaligned_pointers(L):
    from dirt_b200 import _lib
    null, ok, odd = _p(0), _p(4096), _p(4098)
    for k in range(3):
        ptrs = [ok] * 3
        ptrs[k] = null
        assert _fwd(L, ptrs=ptrs) == _lib.ERR_NULL_POINTER, k
        assert _bwd(L, ptrs=ptrs) == _lib.ERR_NULL_POINTER, k
        ptrs[k] = odd
        assert _fwd(L, ptrs=ptrs) == _lib.ERR_MISALIGNED, k
        assert _bwd(L, ptrs=ptrs) == _lib.ERR_MISALIGNED, k
    assert _fwd(L, out=null) == _lib.ERR_NULL_POINTER
    assert _fwd(L, out=odd) == _lib.ERR_MISALIGNED
    assert _bwd(L, grad_out=null) == _lib.ERR_NULL_POINTER
    assert _bwd(L, grad_out=odd) == _lib.ERR_MISALIGNED
    for k in range(3):
        grads = [ok] * 3
        grads[k] = odd
        assert _bwd(L, grads=grads) == _lib.ERR_MISALIGNED, k
    assert _bwd(L, ws=null) == _lib.ERR_NULL_POINTER
    assert _bwd(L, ws=odd) == _lib.ERR_MISALIGNED
    need = L.dirt_sh_lighting_workspace_bytes(1, 8, 3)
    assert _bwd(L, ws_bytes=need - 1) == _lib.ERR_WORKSPACE_TOO_SMALL
    # the workspace is needed only for the coefficient gradient
    assert _bwd(L, grads=[null, null, null], ws=null, ws_bytes=0) == 0
    assert L.dirt_last_launch_count() == 0


def test_sh_route_accepts_the_plain_shapes():
    from dirt_b200.lighting import cuda_route
    dev = [CUDA] * 3
    SH = (9, 'C')
    r = cuda_route([(1000, 3), (1000, 5)], [((9, 5), SH)], dev)
    assert r is not None and (r.lead, r.B, r.V, r.C, r.per_item) == ((), 1, 1000, 5, (False,))
    r = cuda_route([(4, 100, 3), (4, 100, 2)], [((4, 9, 2), SH)], dev)
    assert (r.lead, r.B, r.V, r.C, r.per_item) == ((4,), 4, 100, 2, (True,))
    r = cuda_route([(4, 100, 3), (4, 100, 2)], [((9, 2), SH)], dev)
    assert r.per_item == (False,)
    r = cuda_route([(2, 3, 7, 3), (2, 3, 7, 1)], [((2, 3, 9, 1), SH)], dev)
    assert (r.lead, r.B, r.V, r.C, r.per_item) == ((2, 3), 6, 7, 1, (True,))
    assert cuda_route([(0, 7, 3), (0, 7, 3)], [((0, 9, 3), SH)], dev).B == 0
    assert cuda_route([(2, 0, 3), (2, 0, 3)], [((9, 3), SH)], dev).V == 0


def test_sh_route_refuses_everything_else():
    from dirt_b200.lighting import cuda_route
    dev = [CUDA] * 3
    SH = (9, 'C')
    assert cuda_route([(100, 3), (100, 3)], [((9, 3), SH)], [torch.device('cpu')] * 3) is None   # CPU
    assert cuda_route([(100, 3), (100, 3)], [((9, 3), SH)], [CUDA, CUDA, torch.device('cuda', 1)]) is None
    assert cuda_route([(100, 3), (100, 3)], [((8, 3), SH)], dev) is None                 # not 9 coefficients
    assert cuda_route([(100, 3), (100, 3)], [((9, 4), SH)], dev) is None                 # channels differ
    assert cuda_route([(100, 3), (100, 3)], [((9, 1), SH)], dev) is None                 # a broadcast channel axis
    assert cuda_route([(100, 3), (100, 3)], [((3, 9), SH)], dev) is None                 # transposed
    assert cuda_route([(100, 3), (100, 3)], [((1, 9, 3), SH)], dev) is None              # [1, 9, C] without batch
    assert cuda_route([(2, 100, 3), (2, 100, 3)], [((1, 9, 3), SH)], dev) is None        # a broadcast item axis
    assert cuda_route([(2, 100, 3), (2, 100, 3)], [((3, 9, 3), SH)], dev) is None
    assert cuda_route([(2, 100, 3), (2, 100, 3)], [((27,), SH)], dev) is None            # flattened
    assert cuda_route([(2, 100, 3), (100, 3)], [((9, 3), SH)], dev) is None              # albedo broadcast
    assert cuda_route([(100, 4), (100, 3)], [((9, 3), SH)], dev) is None                 # normals not 3 wide


def _inputs(seed, lead=(2,), V=9, C=3, per_item=True):
    g = torch.Generator().manual_seed(seed)
    return (torch.nn.functional.normalize(torch.randn(lead + (V, 3), generator=g), dim=-1),
            torch.rand(lead + (V, C), generator=g),
            torch.randn((lead if per_item else ()) + (9, C), generator=g))


def test_cpu_calls_return_the_restatement():
    from dirt_b200 import lighting
    for lead, C, per_item in (((2,), 3, True), ((2,), 3, False), ((), 5, False), ((2, 3), 1, True), ((2, 3), 2, False)):
        n, albedo, L = _inputs(len(lead) + C, lead, C=C, per_item=per_item)
        got = lighting.diffuse_spherical_harmonics(n, albedo, L)
        assert got.dtype == torch.float32 and got.shape == lead + (n.shape[-2], C)
        assert torch.equal(got, lighting._diffuse_spherical_harmonics(n, albedo, L))
    # broadcasting the CUDA path does not take is still the restatement's
    n, albedo, L = _inputs(3, (2,), C=3, per_item=False)
    assert torch.equal(lighting.diffuse_spherical_harmonics(n, albedo, L[None]),
                       lighting._diffuse_spherical_harmonics(n, albedo, L[None]))
    # array-likes and float64 are converted to float32, as the other models do
    n, albedo, L = _inputs(7, (), V=4, per_item=False)
    got = lighting.diffuse_spherical_harmonics(n.double().numpy(), albedo.tolist(), L.double())
    assert got.dtype == torch.float32
    np.testing.assert_array_equal(got.numpy(), lighting._diffuse_spherical_harmonics(n, albedo, L).numpy())


def test_cpu_calls_keep_their_errors():
    from dirt_b200 import lighting
    with pytest.raises(RuntimeError):
        lighting.diffuse_spherical_harmonics(torch.zeros(5, 3), torch.zeros(5, 3), torch.zeros(8, 3))
    with pytest.raises(RuntimeError):
        lighting.diffuse_spherical_harmonics(torch.zeros(5, 3), torch.zeros(5, 3), torch.zeros(9, 4))
    with pytest.raises(ValueError):   # the restatement unpacks the normals' three components
        lighting.diffuse_spherical_harmonics(torch.zeros(5, 4), torch.zeros(5, 3), torch.zeros(9, 3))
