"""CPU: shadow mapping (DESIGN.md §7.15) -- the C ABI's rejections, the routing, the restatement's properties, a map
rasterised by the CPU oracle read back at its own texels, and the gradient that reaches an occluder through the map's
occupancy channel, against central differences."""
import ctypes

import numpy as np
import pytest
import torch

from dirt_b200 import _lib, lighting, matrices
from oracle import oracle


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build
    build.build()
    return _lib.lib()


# ---- the C ABI, before any launch -----------------------------------------------------------------------------------

P = 1 << 12   # a non-NULL, 8-byte aligned address; every call below returns before it would be read


def _fwd(L, pos=P, M=P, smap=P, per_item=0, SH=8, SW=8, R=1, soft=0., bias=0., out=P, B=1, V=10, stride=3):
    return L.dirt_shadow_forward(pos, stride, M, smap, per_item, SH, SW, R, soft, bias, out, B, V, None)


def _bwd(L, pos=P, M=P, smap=P, gout=P, gp=None, gM=None, gmap=None, ws=None, ws_bytes=0, R=1, soft=0., B=1, V=10):
    return L.dirt_shadow_backward(pos, 3, M, smap, 0, 8, 8, R, soft, 0., gout, gp, gM, gmap, ws, ws_bytes, B, V, None)


def test_abi_rejects_bad_parameters(L):
    for R in (-1, 4):
        assert _fwd(L, R=R) == _lib.ERR_BAD_SHAPE
        assert _bwd(L, R=R, gp=P) == _lib.ERR_BAD_SHAPE
    for soft, bias in ((-1e-3, 0.), (0., -1e-3), (float('nan'), 0.), (float('inf'), 0.), (0., float('inf'))):
        assert _fwd(L, soft=soft, bias=bias) == _lib.ERR_BAD_SHAPE
    assert _fwd(L, SH=0) == _lib.ERR_BAD_SHAPE and _fwd(L, SW=-1) == _lib.ERR_BAD_SHAPE
    assert _fwd(L, B=-1) == _lib.ERR_BAD_SHAPE and _fwd(L, V=-1) == _lib.ERR_BAD_SHAPE
    assert _fwd(L, stride=-3) == _lib.ERR_BAD_SHAPE
    assert _fwd(L, B=1 << 30, V=1 << 40) == _lib.ERR_BAD_SHAPE


def test_abi_rejects_null_and_misaligned_pointers(L):
    for k in ('pos', 'M', 'smap', 'out'):
        assert _fwd(L, **{k: None}) == _lib.ERR_NULL_POINTER
    assert _fwd(L, pos=P + 2) == _lib.ERR_MISALIGNED
    assert _fwd(L, smap=P + 4) == _lib.ERR_MISALIGNED   # float2 texels
    # nothing to do: no pointer is read
    assert _fwd(L, pos=None, M=None, smap=None, out=None, V=0) == 0
    assert _bwd(L, pos=None, M=None, smap=None, gout=None, V=0) == 0
    assert _bwd(L, pos=None, gp=P) == _lib.ERR_NULL_POINTER
    assert _bwd(L, gout=None, gp=P) == _lib.ERR_NULL_POINTER
    assert _bwd(L, gmap=P + 4) == _lib.ERR_MISALIGNED
    assert _bwd(L, gp=P + 2) == _lib.ERR_MISALIGNED
    # the light-matrix gradient needs its partials workspace
    need = L.dirt_shadow_workspace_bytes(1, 10)
    assert need == 4 * 16
    assert _bwd(L, gM=P) == _lib.ERR_NULL_POINTER
    assert _bwd(L, gM=P, ws=P, ws_bytes=need - 1) == _lib.ERR_WORKSPACE_TOO_SMALL
    assert L.dirt_shadow_workspace_bytes(64, 512 * 512) == 4 * 64 * 1024 * 16
    assert L.dirt_shadow_workspace_bytes(0, 5) == 0 and L.dirt_shadow_workspace_bytes(3, 0) == 0


# ---- routing and argument checks ------------------------------------------------------------------------------------

def test_routing():
    cuda, cpu = torch.device('cuda', 0), torch.device('cpu')
    r = lighting.shadow_route((2, 5, 7, 3), (2, 5, 4, 4), (2, 5, 16, 32, 2), [cuda] * 3)
    assert r.lead == (2, 5) and r.B == 10 and r.V == 7 and r.C == 1 and r.per_item == (True, True)
    r = lighting.shadow_route((3, 7, 3), (4, 4), (16, 32, 2), [cuda] * 3)
    assert r.B == 3 and r.per_item == (False, False)
    assert lighting.shadow_route((3, 7, 3), (4, 4), (3, 16, 32, 2), [cuda] * 3) is None   # shared matrix, per-item map
    assert lighting.shadow_route((3, 7, 3), (3, 4, 4), (16, 32, 2), [cuda] * 3) is None
    assert lighting.shadow_route((3, 7, 3), (4, 4), (16, 32, 3), [cuda] * 3) is None
    assert lighting.shadow_route((3, 7, 4), (4, 4), (16, 32, 2), [cuda] * 3) is None
    assert lighting.shadow_route((3, 7, 3), (4, 4), (16, 32, 2), [cuda, cuda, cpu]) is None
    assert lighting.shadow_route((3, 7, 3), (4, 4), (16, 32, 2), [cpu] * 3) is None


def test_cpu_call_runs_the_restatement_and_checks_its_arguments():
    g = torch.Generator().manual_seed(0)
    p = torch.rand((2, 9, 3), generator=g) * 2 - 1
    smap = torch.rand((2, 6, 5, 2), generator=g)
    M = torch.eye(4).expand(2, 4, 4)
    out = lighting.shadow_visibility(p, M, smap, radius=2, softness=0.1, bias=0.01)
    assert torch.equal(out, lighting._shadow_visibility(p, M, smap, 2, 0.1, 0.01)) and out.shape == (2, 9, 1)
    for kw in ({'radius': 4}, {'radius': -1}, {'softness': -1.}, {'bias': -0.5}, {'softness': float('nan')}):
        with pytest.raises(ValueError):
            lighting.shadow_visibility(p, M, smap, **kw)


# ---- the restatement's properties -----------------------------------------------------------------------------------

def _points(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((n, 3), generator=g, dtype=torch.float64) * 1.8 - 0.9)


@pytest.mark.parametrize('R', [0, 1, 3])
@pytest.mark.parametrize('softness', [0., 0.05])
def test_empty_map_lights_everything(R, softness):
    smap = torch.zeros((7, 9, 2), dtype=torch.float64)
    smap[..., 1] = torch.rand((7, 9), dtype=torch.float64)   # depth without occupancy casts nothing
    vis = lighting._shadow_visibility(_points(200, 1), torch.eye(4, dtype=torch.float64), smap, R, softness)
    assert torch.allclose(vis, torch.ones_like(vis), rtol=0, atol=1e-14)   # (1 - f) + f rounds


def test_radius_zero_is_a_bilinear_blend_of_texel_steps():
    SH, SW = 6, 10
    g = torch.Generator().manual_seed(2)
    smap = torch.stack([(torch.rand((SH, SW), generator=g) > 0.5).double(),
                        torch.rand((SH, SW), generator=g, dtype=torch.float64) - 0.5], -1)
    p = _points(300, 3)
    for softness, bias in ((0., 0.), (0.1, 0.02)):
        vis = lighting._shadow_visibility(p, torch.eye(4, dtype=torch.float64), smap, 0, softness, bias)[:, 0]
        X, Yd = (p[:, 0] + 1) * SW / 2, (1 - p[:, 1]) * SH / 2
        u, v = X - 0.5, Yd - 0.5
        c0, r0 = u.floor(), v.floor()
        fc, fr = u - c0, v - r0
        want = torch.zeros_like(fc)
        for dr, wr in ((0, 1 - fr), (1, fr)):
            for dc, wc in ((0, 1 - fc), (1, fc)):
                t = smap[(r0 + dr).clamp(0, SH - 1).long(), (c0 + dc).clamp(0, SW - 1).long()]
                d = p[:, 2] - t[:, 1] - bias
                step = torch.sigmoid(d / softness) if softness else (d > 0).double()
                want = want + wr * wc * (1 - t[:, 0] * step)
        assert torch.allclose(vis, want, rtol=0, atol=1e-12)


def test_points_outside_the_map_or_behind_the_light_are_lit():
    smap = torch.ones((4, 4, 2), dtype=torch.float64)
    smap[..., 1] = -1.                               # an occluder in front of every point
    p = torch.tensor([[0.1, 0.2, 0.5], [1.5, 0., 0.5], [0., -1.01, 0.5], [-1., 0., 0.5], [0., 1., 0.5],
                      [float('nan'), 0., 0.5], [0., 0., float('inf')], [0.2, 0.1, 0.5]], dtype=torch.float64,
                     requires_grad=True)
    M = torch.eye(4, dtype=torch.float64)
    M[2, 3] = 1.                                     # w = 1 + z ...
    M[3, 3] = 0.5                                    # ... - 0.5: the last point, with z = 0.5, has w = 1
    M = M.requires_grad_()
    vis = lighting._shadow_visibility(p, M, smap, 1, 0.1)[:, 0]
    # X = (x/w + 1) * 2 = 0 at x/w = -1 is inside; x/w = +1 gives X = 4 = SW, outside; y/w = +1 gives Yd = 0, inside
    assert vis[1] == 1 and vis[2] == 1 and vis[5] == 1 and vis[6] == 1
    assert vis[0] < 0.01 and vis[3] < 0.01 and vis[4] < 0.01 and vis[7] < 0.01
    behind = torch.tensor([[0., 0., -0.5], [0., 0., -0.6]], dtype=torch.float64, requires_grad=True)   # w = 0, w < 0
    vb = lighting._shadow_visibility(behind, M, smap, 1, 0.1)
    assert torch.equal(vb, torch.ones_like(vb))
    (vis.sum() + vb.sum()).backward()
    assert torch.isfinite(p.grad).all() and torch.isfinite(M.grad).all()
    for k in (1, 2, 5, 6):
        assert (p.grad[k] == 0).all()
    assert (behind.grad == 0).all()


# ---- maps from the CPU oracle ---------------------------------------------------------------------------------------

S = 64


def _quad(a, b=0.0, half=0.3, z=0.0):
    v = np.array([[a - half, b - half, z, 1], [a + half, b - half, z, 1], [a + half, b + half, z, 1],
                  [a - half, b + half, z, 1]], np.float32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int32)


def _render(v, f):
    """The map `shadow_map` makes with an identity light matrix: clip vertices v, colours (1, clip z)."""
    cols = np.stack([np.ones(len(v), np.float32), v[:, 2]], 1)
    return oracle.forward(np.zeros((1, S, S, 2), np.float32), v[None], cols[None], f[None])


def test_points_on_an_occluder_read_their_own_texels():
    v, f = _quad(0.1, -0.05, half=0.4, z=0.)
    v[:, 2] = [0.1, 0.3, 0.2, 0.0]                   # a tilted quad: depth varies over it
    smap = _render(v, f)[0].astype(np.float64)
    occ, depth = smap[..., 0], smap[..., 1]
    assert set(np.unique(occ)) == {0., 1.}
    r, c = np.meshgrid(np.arange(S), np.arange(S), indexing='ij')
    x, y = (c + 0.5) / (S / 2) - 1, 1 - (r + 0.5) / (S / 2)   # texel centres: fc = fr = 0, all weight on the texel
    m = torch.from_numpy(smap)
    M = torch.eye(4, dtype=torch.float64)
    for dz, lit_if_covered in ((1e-4, 0.), (-1e-4, 1.)):
        p = torch.from_numpy(np.stack([x, y, depth + dz], -1).reshape(-1, 3))
        vis = lighting._shadow_visibility(p, M, m, 0, 0., 0.)[:, 0].numpy().reshape(S, S)
        assert (vis[occ == 1] == lit_if_covered).all() and (vis[occ == 0] == 1.).all()
    # softness > 0 reads the depth itself: 1 - sigmoid((z - depth) / s) at the texel
    p = torch.from_numpy(np.stack([x, y, np.full_like(x, 0.15)], -1).reshape(-1, 3))
    vis = lighting._shadow_visibility(p, M, m, 0, 0.05, 0.)[:, 0].numpy().reshape(S, S)
    want = 1 - occ / (1 + np.exp(-(0.15 - depth) / 0.05))
    assert np.allclose(vis, want, rtol=0, atol=1e-12)


def test_occluder_gradient_matches_central_differences():
    """The gradient of a weighted shadow sum with respect to an occluder's x translation, through the restatement and
    the rasteriser's backward pass on the map, against central differences over one and two texels."""
    R, softness, bias = 1, 0.01, 0.005
    g = torch.linspace(-0.95, 0.95, 200, dtype=torch.float64)
    yy, xx = torch.meshgrid(g, g, indexing='ij')
    pts = torch.stack([xx.flatten(), yy.flatten(), torch.full_like(xx.flatten(), 0.5)], 1)
    weight = torch.exp(-((pts[:, 0] - 0.25) ** 2 + pts[:, 1] ** 2) / 0.1)
    M = torch.eye(4, dtype=torch.float64)

    def loss(a):
        v, f = _quad(a)
        px = _render(v, f)
        sm = torch.tensor(px[0], dtype=torch.float64, requires_grad=True)
        value = (lighting._shadow_visibility(pts, M, sm, R, softness, bias)[:, 0] * weight).sum()
        return value, sm, v, f, px

    for a in (0.0, 0.1, 0.137):
        value, sm, v, f, px = loss(a)
        value.backward()
        _, gv, _ = oracle.backward(v[None], f[None], px, sm.grad.numpy().astype(np.float32)[None])
        analytic = float(gv[0, :, 0].sum())
        assert analytic < 0
        for h in (2. / S, 4. / S):   # one and two texels of the map over [-1, 1]
            fd = (loss(a + h)[0].item() - loss(a - h)[0].item()) / (2 * h)
            assert abs(analytic - fd) <= 0.05 * abs(fd), (a, h, analytic, fd)
