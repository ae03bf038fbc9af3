"""CPU: the GGX specular model's restatement pins its convention in float64 (the closed form at normal incidence, the
distribution's normalisation, reciprocity, energy, the masks and the clamp), its C ABI rejects bad arguments before
anything is launched, the routing decision accepts exactly the plain shapes, and CPU calls run the restatement
unchanged."""
import ctypes
import math

import numpy as np
import pytest
import torch

CUDA = torch.device('cuda', 0)
F64 = torch.float64


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _p(x):
    return ctypes.c_void_p(x)


def _t(x):
    return torch.tensor(x, dtype=F64)


def _ggx(p, n, r, F0, light, lc, cam, point_light=False, double_sided=False):
    from dirt_b200.lighting import _specular_ggx
    return _specular_ggx(p, n, r, F0, light, lc, cam, point_light, double_sided)


def _hemisphere(n_cos, n_phi):
    """Midpoints of an n_cos x n_phi grid in (cos theta, phi) over the upper hemisphere about z, and the solid angle of
    each cell."""
    c = (torch.arange(n_cos, dtype=F64) + 0.5) / n_cos
    phi = (torch.arange(n_phi, dtype=F64) + 0.5) * (2 * math.pi / n_phi)
    C, P = torch.meshgrid(c, phi, indexing='ij')
    s = torch.sqrt(1 - C * C)
    dirs = torch.stack([s * torch.cos(P), s * torch.sin(P), C], -1).reshape(-1, 3)
    return dirs, 2 * math.pi / (n_cos * n_phi)


# ---- the restatement ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize('point_light', [False, True])
def test_closed_form_at_normal_incidence(point_light):
    """n = l = v: h = n, every cosine is 1, F = F0, D = 1 / (pi a^4), Vis = 1/4, so out = I F0 / (4 a^4).  The vectors
    are long, so that unit()'s 1e-12 moves n, l and v by less than 1e-14; on h = unit(l + v), |l + v| = 2, it leaves
    n . h = 2 / (2 + 1e-12), and D goes as (n . h)^-4, a factor 1 + 2e-12 that the expected value includes."""
    a = _t([0.045, 0.1, 0.3, 0.5, 0.8, 1.0, 1.5])[:, None]
    V = a.shape[0]
    p = _t([[0.3, -0.2, 1.0]]).expand(V, 3)
    n = _t([[0., 0., 250.]]).expand(V, 3)                      # not unit: normalised by the model
    F0 = _t([[0.04, 0.5, 1.0]]).expand(V, 3)
    I = _t([2.0, 1.0, 0.25])
    cam = _t([0.3, -0.2, 701.0])
    light = _t([0.3, -0.2, 401.0]) if point_light else _t([0., 0., -300.])
    got = _ggx(p, n, a, F0, light, I, cam, point_light)
    want = I * F0 / (4 * a ** 4) / (2 / (2 + 1e-12)) ** 4
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-12, atol=0)


def _retro_D(c, a):
    """D(n . h = c) read from the restatement: with l = v = h, out = pi I F0 D Vis c and Vis = 1 / (4 c G),
    G = sqrt(c^2 (1 - a^4) + a^4)."""
    s = torch.sqrt(1 - c * c)
    d = torch.stack([s, torch.zeros_like(s), c], -1)           # l = v = d, n = z: one point per item
    V = d.shape[0]
    out = _ggx(torch.zeros(V, 1, 3, dtype=F64), _t([[[0., 0., 1.]]]).expand(V, 1, 3),
               torch.full((V, 1, 1), a, dtype=F64), torch.ones(V, 1, 1, dtype=F64), -d, _t([1.]), d * 5, False)[:, 0]
    A = a ** 4
    vis = 1 / (4 * c * torch.sqrt(c * c * (1 - A) + A))
    return out[:, 0] / (math.pi * vis * c)


def test_the_distribution_is_normalised():
    """integral of D(h) (n . h) over the hemisphere = 1, by a 4000-point midpoint rule in cos theta (D is isotropic, so
    the phi integral is 2 pi; that it does not depend on phi is checked separately)."""
    c = (torch.arange(4000, dtype=F64) + 0.5) / 4000
    for a, tol in ((0.3, 5e-4), (0.5, 1e-4), (0.7, 1e-4), (1.0, 1e-4)):
        D = _retro_D(c, a)
        integral = float((D * c).sum() * (2 * math.pi / 4000))
        assert abs(integral - 1) < tol, (a, integral)
        A = a ** 4
        # the textbook D (up to unit()'s 1e-12, which moves it by a few 1e-12 here)
        np.testing.assert_allclose(D.numpy(), (A / (math.pi * (c * c * (A - 1) + 1) ** 2)).numpy(), rtol=1e-10)
    # isotropy: the same c at other azimuths
    dirs, _ = _hemisphere(40, 16)
    V = dirs.shape[0]
    out = _ggx(torch.zeros(V, 1, 3, dtype=F64), _t([[[0., 0., 1.]]]).expand(V, 1, 3),
               torch.full((V, 1, 1), 0.4, dtype=F64), torch.ones(V, 1, 1, dtype=F64), -dirs, _t([1.]),
               dirs * 5).reshape(40, 16)
    np.testing.assert_allclose(out.numpy(), out[:, :1].expand(40, 16).numpy(), rtol=1e-12)


def test_reciprocity():
    """out / (n . l) is the BRDF times pi I: symmetric under swapping l and v, for both light kinds.  The light and the
    camera are 1000 units away, so that unit()'s 1e-12, which breaks the symmetry for unequal lengths, stays below
    1e-14."""
    g = torch.Generator().manual_seed(0)
    V = 500
    n = torch.nn.functional.normalize(torch.randn(V, 3, generator=g, dtype=F64), dim=-1)

    def towards(n):   # a unit direction in n's hemisphere
        d = torch.nn.functional.normalize(torch.randn(V, 3, generator=g, dtype=F64), dim=-1)
        return torch.where((d * n).sum(-1, keepdim=True) < 0, -d, d)

    l, v = towards(n), towards(n)
    p = torch.randn(V, 3, generator=g, dtype=F64)
    r = torch.rand(V, 1, generator=g, dtype=F64) * 0.9 + 0.1
    F0 = torch.rand(V, 2, generator=g, dtype=F64)
    lc = _t([1.5, 0.5])
    for point_light in (False, True):
        def brdf(l, v):   # one point per item, with its own light and camera
            out = _ggx(p[:, None], n[:, None], r[:, None], F0[:, None], (p + 1000 * l) if point_light else -1000 * l,
                       lc, p + 1000 * v, point_light)[:, 0]
            return out / (n * l).sum(-1, keepdim=True)
        np.testing.assert_allclose(brdf(l, v).numpy(), brdf(v, l).numpy(), rtol=1e-12, atol=0)


def test_directional_albedo_is_at_most_one():
    """With F0 = 1 the reflected energy, the integral of out / (pi I) over the light's hemisphere, is at most 1 (the
    quadrature's error aside) for every roughness and view angle; single-scattering GGX loses energy as the roughness
    grows, so it is well below 1 for rough surfaces at grazing view."""
    dirs, dw = _hemisphere(800, 128)
    N = dirs.shape[0]   # one light direction per item, one point per item
    n = _t([[[0., 0., 1.]]]).expand(N, 1, 3)
    for a in (0.2, 0.4, 0.6, 0.8, 1.0):
        for cv in (0.1, 0.3, 0.6, 1.0):
            v = _t([math.sqrt(1 - cv * cv), 0., cv])
            out = _ggx(torch.zeros(N, 1, 3, dtype=F64), n, torch.full((N, 1, 1), a, dtype=F64),
                       torch.ones(N, 1, 1, dtype=F64), -dirs, _t([1.]), v * 4)
            albedo = float(out.sum() * dw / math.pi)
            assert 0 < albedo <= 1 + 2e-3, (a, cv, albedo)
            if a == 0.2 and cv == 1.0:
                assert albedo > 0.9, albedo


def _grads(p, n, r, F0, light, lc, cam, point_light, double_sided):
    leaves = [t.clone().requires_grad_(True) for t in (p, n, r, F0, light, lc, cam)]
    out = _ggx(*leaves, point_light, double_sided)
    out.sum().backward()
    return out.detach(), [t.grad for t in leaves]


@pytest.mark.parametrize('double_sided', [False, True])
@pytest.mark.parametrize('point_light', [False, True])
def test_unlit_points_give_exactly_zero_and_no_gradient(point_light, double_sided):
    """n . l <= 0 or n . v <= 0, including exactly 0 and the degenerate l = -v (h = 0), give 0 and zero gradients."""
    n = _t([[0., 0., 1.]] * 5)
    p = torch.zeros(5, 3, dtype=F64)
    l_dirs = _t([[1., 0., 0.], [0.6, 0., -0.8], [0., 0.6, 0.8], [0., 0., 1.], [0.6, 0., 0.8]])
    v_dirs = _t([[0., 0.6, 0.8], [0., 0.6, 0.8], [1., 0., 0.], [0.6, 0., 0.8], [-0.6, 0., -0.8]])
    # rows: n.l = 0; n.l < 0; n.v = 0; lit (control); l = -v with n.v < 0 (seen from behind: lit only double-sided
    # after the flip, where n.l < 0)
    for i in range(5):
        light = (p[i] + 2 * l_dirs[i]) if point_light else -l_dirs[i]
        out, grads = _grads(p[i:i + 1], n[i:i + 1], _t([[0.3]]), _t([[0.5, 0.2]]), light, _t([1., 2.]),
                            p[i] + 3 * v_dirs[i], point_light, double_sided)
        if i == 3:
            assert (out > 0).all() and all(g.abs().sum() > 0 for g in grads[:4])
            continue
        assert torch.equal(out, torch.zeros_like(out)), i
        for g in grads:
            assert g is not None and torch.equal(g, torch.zeros_like(g)), i


def test_double_sided_turns_the_normal_to_the_camera():
    g = torch.Generator().manual_seed(1)
    V = 200
    n = torch.randn(V, 3, generator=g, dtype=F64)
    p = torch.randn(V, 3, generator=g, dtype=F64)
    r = torch.rand(V, 1, generator=g, dtype=F64)
    F0 = torch.rand(V, 3, generator=g, dtype=F64)
    cam, lc = _t([0.5, 1., 6.]), _t([1., 0.5, 2.])
    for point_light, light in ((False, _t([0.3, -0.5, -0.8])), (True, _t([2., 3., 4.]))):
        v = cam - p
        behind = (n * v).sum(-1, keepdim=True) < 0
        mirrored = torch.where(behind, -n, n)
        ds = _ggx(p, n, r, F0, light, lc, cam, point_light, True)
        np.testing.assert_array_equal(ds.numpy(), _ggx(p, mirrored, r, F0, light, lc, cam, point_light, False).numpy())
        assert behind.any() and (ds[behind[:, 0]] > 0).any()
        # without double_sided a point seen from behind is dark
        assert (_ggx(p, n, r, F0, light, lc, cam, point_light, False)[behind[:, 0]] == 0).all()


def test_roughness_clamp_gradient():
    """Below 0.045 the roughness gets no gradient and the output is that at 0.045; at exactly 0.045 it gets the
    gradient of the unclamped expression."""
    from dirt_b200 import lighting
    p, n = torch.zeros(1, 3, dtype=F64), _t([[0.1, 0.05, 1.]])
    args = (_t([[0.5]]), _t([0., 0., -1.]), _t([1.]), _t([0.02, 0.01, 4.]))

    def run(r):
        out, grads = _grads(p, n, _t([[r]]), *args[:1], *args[1:], False, False)
        return out, grads[2]

    out_clamped, g_below = run(0.03)
    assert torch.equal(g_below, torch.zeros_like(g_below))
    out_at, g_at = run(0.045)
    assert torch.equal(out_clamped, out_at)
    assert float(g_at.abs()) > 0
    try:
        lighting.GGX_MIN_ROUGHNESS = 0.01
        _, g_free = run(0.045)
    finally:
        lighting.GGX_MIN_ROUGHNESS = 0.045
    assert torch.equal(g_at, g_free)


def test_the_k_form_equals_the_textbook_one():
    """k = A (n . h)^2 + |n x h|^2 is NdotH^2 (A - 1) + 1 for unit n and h (Lagrange's identity)."""
    g = torch.Generator().manual_seed(2)
    n = torch.nn.functional.normalize(torch.randn(1000, 3, generator=g, dtype=F64), dim=-1)
    h = torch.nn.functional.normalize(torch.randn(1000, 3, generator=g, dtype=F64), dim=-1)
    A = torch.rand(1000, generator=g, dtype=F64) ** 4
    c = (n * h).sum(-1)
    k = A * c * c + torch.linalg.cross(n, h, dim=-1).square().sum(-1)
    np.testing.assert_allclose(k.numpy(), (c * c * (A - 1) + 1).numpy(), rtol=0, atol=1e-12)


# ---- the C ABI ----------------------------------------------------------------------------------------------------

def _fwd(L, point=0, B=1, V=8, C=3, strides=(3, 3, 1, 3), ptrs=None, out=None):
    ok = _p(4096)
    n, p, r, k, l, lc, cam = ptrs if ptrs is not None else [ok] * 7
    sn, sp, sr, sk = strides
    return L.dirt_ggx_lighting_forward(point, 1, n, sn, p, sp, r, sr, k, sk, l, 0, lc, 0, cam, 0,
                                       ok if out is None else out, B, V, C, None)


def _bwd(L, point=0, B=1, V=8, C=3, strides=(3, 3, 1, 3), ptrs=None, grad_out=None, grads=None, ws=None,
         ws_bytes=1 << 20):
    ok = _p(4096)
    n, p, r, k, l, lc, cam = ptrs if ptrs is not None else [ok] * 7
    sn, sp, sr, sk = strides
    grads = grads if grads is not None else [ok] * 7
    return L.dirt_ggx_lighting_backward(point, 0, n, sn, p, sp, r, sr, k, sk, l, 1, lc, 0, cam, 1,
                                        ok if grad_out is None else grad_out, *grads, ok if ws is None else ws,
                                        ws_bytes, B, V, C, None)


def test_ggx_abi_rejects_bad_shapes(L):
    from dirt_b200 import _lib
    for call in (_fwd, _bwd):
        for point in (0, 1):
            assert call(L, point, B=-1) == _lib.ERR_BAD_SHAPE
            assert call(L, point, V=-1) == _lib.ERR_BAD_SHAPE
            assert call(L, point, C=0) == _lib.ERR_BAD_SHAPE
            for k in range(4):
                strides = [3, 3, 1, 3]
                strides[k] = -1
                assert call(L, point, strides=tuple(strides)) == _lib.ERR_BAD_SHAPE, k
            assert call(L, point, B=1 << 30, V=1 << 40) == _lib.ERR_BAD_SHAPE      # element offsets past 2^62
            assert call(L, point, V=1 << 50, C=1) == _lib.ERR_BAD_SHAPE           # more chunks than the grid holds
            assert L.dirt_last_launch_count() == 0


def test_ggx_abi_with_no_points_launches_nothing(L):
    null = _p(0)
    for B, V in ((0, 8), (3, 0)):
        for point in (0, 1):
            assert _fwd(L, point, B=B, V=V, ptrs=[null] * 7, out=null) == 0
            assert L.dirt_last_launch_count() == 0
            assert _bwd(L, point, B=B, V=V, ptrs=[null] * 7, grad_out=null, grads=[null] * 7, ws=null, ws_bytes=0) == 0
            assert L.dirt_last_launch_count() == 0


def test_ggx_abi_rejects_null_and_misaligned_pointers(L):
    from dirt_b200 import _lib
    null, ok, odd = _p(0), _p(4096), _p(4098)
    for point in (0, 1):
        for k in range(7):   # every input is read
            ptrs = [ok] * 7
            ptrs[k] = null
            assert _fwd(L, point, ptrs=ptrs) == _lib.ERR_NULL_POINTER, (point, k)
            assert _bwd(L, point, ptrs=ptrs) == _lib.ERR_NULL_POINTER, (point, k)
            ptrs[k] = odd
            assert _fwd(L, point, ptrs=ptrs) == _lib.ERR_MISALIGNED, (point, k)
            assert _bwd(L, point, ptrs=ptrs) == _lib.ERR_MISALIGNED, (point, k)
        assert _fwd(L, point, out=null) == _lib.ERR_NULL_POINTER
        assert _fwd(L, point, out=odd) == _lib.ERR_MISALIGNED
        assert _bwd(L, point, grad_out=null) == _lib.ERR_NULL_POINTER
        assert _bwd(L, point, grad_out=odd) == _lib.ERR_MISALIGNED
        for k in range(7):
            grads = [ok] * 7
            grads[k] = odd
            assert _bwd(L, point, grads=grads) == _lib.ERR_MISALIGNED, (point, k)
        assert _bwd(L, point, ws=null) == _lib.ERR_NULL_POINTER
        assert _bwd(L, point, ws=odd) == _lib.ERR_MISALIGNED
        # the workspace of the other lighting models, whose partial row (7 + C) holds light, light colour and camera
        need = L.dirt_lighting_workspace_bytes(1, 8, 3)
        assert _bwd(L, point, ws_bytes=need - 1) == _lib.ERR_WORKSPACE_TOO_SMALL
        # no gradient wanted: nothing is needed, nothing is launched
        assert _bwd(L, point, grads=[null] * 7, ws=null, ws_bytes=0) == 0
        assert L.dirt_last_launch_count() == 0


# ---- routing and the CPU path ---------------------------------------------------------------------------------------

GGX_WIDTHS = [3, 3, 1, 'C']


def test_ggx_route_accepts_the_plain_shapes():
    from dirt_b200.lighting import cuda_route
    dev = [CUDA] * 7
    items = lambda lead, C, per: [(lead + (3,) if per[0] else (3,), 3), (lead + (C,) if per[1] else (C,), 'C'),
                                  (lead + (3,) if per[2] else (3,), 3)]
    r = cuda_route([(1000, 3), (1000, 3), (1000, 1), (1000, 5)], items((), 5, (0, 0, 0)), dev, GGX_WIDTHS)
    assert r is not None and (r.lead, r.B, r.V, r.C, r.per_item) == ((), 1, 1000, 5, (False, False, False))
    r = cuda_route([(4, 100, 3), (4, 100, 3), (4, 100, 1), (4, 100, 2)], items((4,), 2, (1, 0, 1)), dev, GGX_WIDTHS)
    assert (r.B, r.V, r.C, r.per_item) == (4, 100, 2, (True, False, True))
    r = cuda_route([(2, 3, 7, 3), (2, 3, 7, 3), (2, 3, 7, 1), (2, 3, 7, 1)], items((2, 3), 1, (0, 1, 0)), dev,
                   GGX_WIDTHS)
    assert (r.lead, r.B, r.V, r.C, r.per_item) == ((2, 3), 6, 7, 1, (False, True, False))
    # the default widths are unchanged: three 3-wide tensors, colours last
    assert cuda_route([(100, 3), (100, 3), (100, 3), (100, 2)], items((), 2, (0, 0, 0)), dev) is not None
    assert cuda_route([(100, 3), (100, 3), (100, 1), (100, 2)], items((), 2, (0, 0, 0)), dev) is None


def test_ggx_route_refuses_everything_else():
    from dirt_b200.lighting import cuda_route
    dev = [CUDA] * 7
    ok_items = [((3,), 3), ((3,), 'C'), ((3,), 3)]
    shapes = [(100, 3), (100, 3), (100, 1), (100, 3)]
    assert cuda_route(shapes, ok_items, dev, GGX_WIDTHS) is not None
    assert cuda_route(shapes, ok_items, [torch.device('cpu')] * 7, GGX_WIDTHS) is None
    assert cuda_route([(100, 3), (100, 3), (100, 3), (100, 3)], ok_items, dev, GGX_WIDTHS) is None   # roughness 3 wide
    assert cuda_route([(100, 3), (100, 3), (100,), (100, 3)], ok_items, dev, GGX_WIDTHS) is None     # roughness [V]
    assert cuda_route([(100, 3), (100, 3), (1, 1), (100, 3)], ok_items, dev, GGX_WIDTHS) is None     # broadcast
    assert cuda_route([(2, 100, 3), (2, 100, 3), (100, 1), (2, 100, 3)], ok_items, dev, GGX_WIDTHS) is None
    assert cuda_route(shapes, [((3,), 3), ((3,), 'C'), ((1, 3), 3)], dev, GGX_WIDTHS) is None       # camera [1, 3]


def _inputs(seed, lead=(2,), V=9, C=3):
    g = torch.Generator().manual_seed(seed)
    return dict(pos=torch.randn(lead + (V, 3), generator=g), nrm=torch.randn(lead + (V, 3), generator=g),
                rough=torch.rand(lead + (V, 1), generator=g), spec=torch.rand(lead + (V, C), generator=g),
                ldir=torch.nn.functional.normalize(torch.randn(lead + (3,), generator=g), dim=-1),
                lpos=torch.randn(lead + (3,), generator=g) * 3, lcol=torch.rand(lead + (C,), generator=g),
                cam=torch.randn(lead + (3,), generator=g) * 4)


@pytest.mark.parametrize('double_sided', [True, False])
def test_cpu_calls_return_the_restatement(double_sided):
    from dirt_b200 import lighting
    for lead, C in (((2,), 3), ((), 5), ((2, 3), 1)):
        x = _inputs(len(lead) + C, lead, C=C)
        for fn, light, point in ((lighting.specular_ggx_directional, 'ldir', False),
                                 (lighting.specular_ggx_point, 'lpos', True)):
            got = fn(x['pos'], x['nrm'], x['rough'], x['spec'], x[light], x['lcol'], x['cam'], double_sided)
            want = lighting._specular_ggx(x['pos'], x['nrm'], x['rough'], x['spec'], x[light], x['lcol'], x['cam'],
                                          point, double_sided)
            assert got.dtype == torch.float32 and got.shape == lead + (x['pos'].shape[-2], C)
            assert torch.equal(got, want)
    # array-likes and float64 are converted to float32, as the other models do
    x = _inputs(7, (), V=4)
    got = lighting.specular_ggx_directional(x['pos'].double().numpy(), x['nrm'].tolist(), x['rough'], x['spec'],
                                            [0., 0., -1.], [1., 1., 1.], x['cam'])
    assert got.dtype == torch.float32
    np.testing.assert_array_equal(got.numpy(), lighting._specular_ggx(
        x['pos'], x['nrm'], x['rough'], x['spec'], torch.tensor([0., 0., -1.]), torch.ones(3), x['cam'], False,
        False).numpy())
