"""GPU: shadow-map visibility (DESIGN.md §7.15) -- the CUDA kernels against float64 autograd of the torch restatement,
the reproducibility of the light-matrix gradient, the small-grid build, and the whole pipeline (shadow_map, then
shadow_visibility) against the CPU oracle, occluder gradient included."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import rel_close
from dirt_b200 import _lib, lighting

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device('cuda')
SH, SW = 24, 40


@pytest.fixture(autouse=True)
def _library(cuda_lib):
    """Skips without a CUDA device; builds the library if it is stale."""
    return cuda_lib


def _case(B, N, per_item, seed, bias=0.01, special=True):
    """Points, light matrices and maps whose lookups keep X, Yd and z - z_j - bias away from fp32 ties: fractions
    at least 0.01 from 0 and 1, map depths on a grid of 0.1 and point depths 0.05 off it.  With `special`, each item
    also has points near and on the map's edges (clamped taps), outside it, behind the light (w <= 0) and non-finite."""
    g = np.random.default_rng(seed)
    nm = B if per_item else 1
    M = np.tile(np.eye(4), (nm, 1, 1))
    M[:, :3, :3] += g.uniform(-0.1, 0.1, (nm, 3, 3))
    M[:, 3, :3] += g.uniform(-0.1, 0.1, (nm, 3))
    M[:, 2, 3] = g.choice([-1., 1.], nm) * g.uniform(0.02, 0.05, nm)   # w = 1 + a small multiple of z: a mild perspective
    Minv = np.linalg.inv(M)
    # choose clip-space lookups, then map them back to world points
    # X and Yd themselves (the lookups' fractions are those of X - 0.5 and Yd - 0.5)
    r = g.integers(0, SH - 1, (B, N)) + 0.5 + g.uniform(0.01, 0.99, (B, N))
    c = g.integers(0, SW - 1, (B, N)) + 0.5 + g.uniform(0.01, 0.99, (B, N))
    if special:
        r[:, :6] = [0.2, SH - 0.3, 0.6, SH - 0.9, 3.5 + 0.37, 0.05]
        c[:, :6] = [0.3, SW - 0.2, SW - 0.7, 0.4, 0.05, 5.43]
    z = g.integers(-5, 6, (B, N)) * 0.1 + 0.05 + bias
    w = g.uniform(0.8, 1.2, (B, N))
    xn, yn = c / (SW / 2) - 1, 1 - r / (SH / 2)
    h = np.stack([xn * w, yn * w, z, w], -1)
    p = np.einsum('bnk,bkj->bnj', h, Minv if per_item else np.broadcast_to(Minv, (B, 4, 4)))
    p = p[..., :3] / p[..., 3:]
    if special and N >= 12:
        p[:, 6] = [50., 0., 0.]                       # outside the map
        p[:, 7] = [0., -50., 0.]
        p[:, 8, 2] = np.nan
        p[:, 9, 0] = np.inf
    occ = (g.uniform(size=(nm, SH, SW)) < 0.6).astype(np.float64)
    depth = g.integers(-6, 7, (nm, SH, SW)) * 0.1
    smap = np.stack([occ, depth], -1)
    if not per_item:
        M, smap = M[0], smap[0]
    return p, M, smap


def _behind(p, M, per_item):
    """Replace points 10 and 11 of each item by points with w = 0 and w < 0 (the matrices have M[2, 3] != 0)."""
    Ms = M if per_item else np.broadcast_to(M, (p.shape[0], 4, 4))
    for b in range(p.shape[0]):
        # w = p . M[:3, 3] + M[3, 3]: move along z from a point until w = 0 and w = -0.5
        m = Ms[b]
        for k, target in ((10, 0.), (11, -0.5)):
            q = np.array([0.1, 0.2, 0.])
            q[2] = (target - m[3, 3] - q[:2] @ m[:2, 3]) / m[2, 3]
            p[b, k] = q
    return p


def _run(p, M, smap, R, softness, bias, gout, positions_view=None):
    """(vis, grads) of the CUDA path and of float64 autograd of the restatement, on the same fp32-rounded inputs."""
    p, M, smap = [np.asarray(x, np.float32).astype(np.float64) for x in (p, M, smap)]
    t64 = [torch.tensor(x, dtype=torch.float64, requires_grad=True) for x in (p, M, smap)]
    v64 = lighting._shadow_visibility(*t64, R, softness, bias)
    (v64 * torch.tensor(gout, dtype=torch.float64)).sum().backward()
    pos = torch.tensor(p, dtype=torch.float32, device=DEV)
    if positions_view is not None:
        pos = positions_view(pos)
    pos.requires_grad_(True)
    tM = torch.tensor(M, dtype=torch.float32, device=DEV, requires_grad=True)
    tm = torch.tensor(smap, dtype=torch.float32, device=DEV, requires_grad=True)
    v = lighting.shadow_visibility(pos, tM, tm, R, softness, bias)
    (v * torch.tensor(gout, dtype=torch.float32, device=DEV)).sum().backward()
    got = [v, pos.grad, tM.grad, tm.grad]
    want = [v64, t64[0].grad, t64[1].grad, t64[2].grad]
    return [x.detach().cpu().numpy() for x in got], [x.detach().numpy() for x in want]


def _check(got, want, names=('visibility', 'grad_positions', 'grad_light_matrix', 'grad_shadow_map')):
    for g, w, name in zip(got, want, names):
        w = np.nan_to_num(w)
        ok, worst = rel_close(g, w, name='shadow ' + name)
        assert ok, (name, worst)


@pytest.mark.parametrize('R', [0, 1, 2, 3])
@pytest.mark.parametrize('softness', [0., 0.05])
@pytest.mark.parametrize('per_item', [True, False])
def test_against_float64_restatement(R, softness, per_item):
    B, N, bias = 3, 700, 0.01
    p, M, smap = _case(B, N, per_item, seed=R * 10 + int(softness > 0) * 2 + per_item, bias=bias)
    p = _behind(p, M, per_item)
    gout = np.random.default_rng(7).standard_normal((B, N, 1))
    got, want = _run(p, M, smap, R, softness, bias, gout)
    assert np.isfinite(got[1]).all() and (got[0][:, 6:12] == 1).all()
    _check(got, want)


def test_gbuffer_views():
    """Positions read as a channel slice of a G-buffer, in place."""
    B, N = 2, 500
    p, M, smap = _case(B, N, True, seed=3)
    gout = np.random.default_rng(8).standard_normal((B, N, 1))

    def view(pos):
        gbuffer = torch.zeros((B, N, 9), dtype=torch.float32, device=DEV)
        gbuffer[..., 4:7] = pos
        return gbuffer[..., 4:7]

    got, want = _run(p, M, smap, 1, 0.05, 0.01, gout, view)
    _check(got, want)


def test_empty_batches():
    for B, N in ((0, 5), (2, 0)):
        p = torch.zeros((B, N, 3), device=DEV, requires_grad=True)
        M = torch.eye(4, device=DEV).expand(B, 4, 4).clone().requires_grad_(True)
        m = torch.rand((B, 4, 4, 2), device=DEV, requires_grad=True)
        v = lighting.shadow_visibility(p, M, m)
        assert v.shape == (B, N, 1)
        v.sum().backward()
        assert (M.grad == 0).all() and (m.grad == 0).all() and p.grad.shape == p.shape


def test_many_items():
    """70 000 items: more than one grid's worth of items (gridDim.y)."""
    B, N = 70000, 12
    p, M, smap = _case(B, N, True, seed=5)
    gout = np.random.default_rng(9).standard_normal((B, N, 1))
    got, want = _run(p, M, smap, 0, 0.05, 0.01, gout)
    _check(got, want)


def test_light_matrix_gradient_is_reproducible():
    B, N = 4, 20000
    for per_item in (True, False):
        p, M, smap = _case(B, N, per_item, seed=11, special=False)
        pos = torch.tensor(p, dtype=torch.float32, device=DEV)
        tm = torch.tensor(smap, dtype=torch.float32, device=DEV)
        gout = torch.randn((B, N, 1), device=DEV)
        grads = []
        for _ in range(2):
            tM = torch.tensor(M, dtype=torch.float32, device=DEV, requires_grad=True)
            pp = pos.clone().requires_grad_(True)
            (lighting.shadow_visibility(pp, tM, tm, 1, 0.05, 0.01) * gout).sum().backward()
            grads.append((tM.grad.clone(), pp.grad.clone()))
        assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])


def test_map_at_an_odd_float_offset():
    """A map view that is 4- but not 8-byte aligned is read through a copy: same values and gradients."""
    p, M, smap = _case(2, 300, True, seed=70)
    pos = torch.tensor(p, dtype=torch.float32, device=DEV)
    tM = torch.tensor(M, dtype=torch.float32, device=DEV)
    buf = torch.zeros(smap.size + 1, device=DEV)
    odd = buf[1:].view(smap.shape)
    odd.copy_(torch.tensor(smap))
    assert odd.data_ptr() % 8 == 4
    odd.requires_grad_(True)
    aligned = odd.detach().clone().requires_grad_(True)
    gout = torch.randn((2, 300, 1), device=DEV)
    outs = []
    for m in (odd, aligned):
        v = lighting.shadow_visibility(pos, tM, m, 1, 0.05, 0.01)
        (v * gout).sum().backward()
        outs.append(v)
    assert torch.equal(outs[0], outs[1])
    ok, worst = rel_close(odd.grad.cpu().numpy(), aligned.grad.cpu().numpy())
    assert ok, worst


def _grads(p, M, smap, R, softness, gout, deterministic):
    pos = torch.tensor(p, dtype=torch.float32, device=DEV, requires_grad=True)
    tM = torch.tensor(M, dtype=torch.float32, device=DEV, requires_grad=True)
    tm = torch.tensor(smap, dtype=torch.float32, device=DEV, requires_grad=True)
    torch.use_deterministic_algorithms(deterministic)
    try:
        (lighting.shadow_visibility(pos, tM, tm, R, softness, 0.01) * gout).sum().backward()
    finally:
        torch.use_deterministic_algorithms(False)
    return pos.grad, tM.grad, tm.grad


@pytest.mark.parametrize('R', [0, 1, 3])
@pytest.mark.parametrize('softness', [0., 0.05])
@pytest.mark.parametrize('per_item', [True, False])
def test_deterministic_backward(R, softness, per_item):
    """Under torch.use_deterministic_algorithms(True): the map gradient meets float64 autograd and is bit-identical
    across calls; the position and matrix gradients are the default path's, bit for bit."""
    B, N = 3, 2000
    p, M, smap = _case(B, N, per_item, seed=40 + R * 4 + per_item * 2 + int(softness > 0))
    p = _behind(p, M, per_item)
    gout = torch.tensor(np.random.default_rng(3).standard_normal((B, N, 1)), dtype=torch.float32, device=DEV)
    det = _grads(p, M, smap, R, softness, gout, True)
    again = _grads(p, M, smap, R, softness, gout, True)
    default = _grads(p, M, smap, R, softness, gout, False)
    assert all(torch.equal(x, y) for x, y in zip(det, again))
    assert torch.equal(det[0], default[0]) and torch.equal(det[1], default[1])
    _, want = _run(p, M, smap, R, softness, 0.01, gout.cpu().numpy())
    ok, worst = rel_close(det[2].cpu().numpy(), np.nan_to_num(want[3]), name='shadow deterministic grad_shadow_map')
    assert ok, worst


def _det_abi(L, p, M, smap, per_item, R, softness, gout, out):
    """dirt_shadow_backward_deterministic on preallocated buffers, map gradient only, into out."""
    B, N = p.shape[:2]
    sb = int(L.dirt_shadow_backward_deterministic_bytes(B, N, int(per_item), smap.shape[-3], smap.shape[-2]))
    scratch = torch.empty(sb, dtype=torch.uint8, device=DEV)

    def call():
        assert L.dirt_shadow_backward_deterministic(
            p.data_ptr(), 3, M.data_ptr(), smap.data_ptr(), int(per_item), smap.shape[-3], smap.shape[-2], R, softness,
            0.01, gout.data_ptr(), None, None, out.data_ptr(), None, 0, scratch.data_ptr(), sb, B, N,
            torch.cuda.current_stream().cuda_stream) == 0
    return call


def test_deterministic_backward_under_graph_replay():
    B, N = 2, 5000
    p, M, smap = _case(B, N, True, seed=50)
    t = [torch.tensor(x, dtype=torch.float32, device=DEV).contiguous() for x in (p, M, smap)]
    gout = torch.randn((B * N,), device=DEV)
    L = _lib.lib()
    eager = torch.empty_like(t[2])
    _det_abi(L, *t, True, 1, 0.05, gout, eager)()
    replayed = torch.full_like(t[2], float('nan'))
    call = _det_abi(L, *t, True, 1, 0.05, gout, replayed)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()   # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call()
    for _ in range(2):
        replayed.fill_(float('nan'))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(replayed, eager)


def test_deterministic_backward_equals_the_order_restated():
    """Identity light matrix and dyadic points (every fp32 step exact), softness 0: each texel's gradient is the float64
    sum, in the documented order, of the fp32 terms, rounded once."""
    R, S_H, S_W, B, N = 1, 8, 16, 2, 1500   # power-of-two sizes: X = (x + 1) * S_W / 2 is exact
    g = np.random.default_rng(60)
    X = g.integers(0, S_W * 64, (B, N)) / 64. + 1 / 128.
    Yd = g.integers(0, S_H * 64, (B, N)) / 64. + 1 / 128.
    z = g.integers(-8, 8, (B, N)) / 16. + 1 / 32.
    p = np.stack([X / (S_W / 2) - 1, 1 - Yd / (S_H / 2), z], -1).astype(np.float32)
    smap = np.stack([(g.uniform(size=(B, S_H, S_W)) < 0.6), g.integers(-8, 8, (B, S_H, S_W)) / 16.], -1).astype(np.float32)
    M = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    gout = (g.integers(-64, 64, (B, N)) / 32.).astype(np.float32)
    L = _lib.lib()
    t = [torch.tensor(x, device=DEV).contiguous() for x in (p, M, smap)]
    got = torch.empty_like(t[2])
    _det_abi(L, *t, True, R, 0., torch.tensor(gout, device=DEV), got)()
    torch.cuda.synchronize()

    T, inv_k = 2 * R + 2, np.float32(1) / np.float32((2 * R + 1) ** 2)
    terms = {}   # texel -> list of (order, occupancy term)
    f32 = np.float32
    for b in range(B):
        for n in range(N):
            u, v = X[b, n] - 0.5, Yd[b, n] - 0.5
            c0, r0 = int(np.floor(u)), int(np.floor(v))
            fc, fr = f32(u - c0), f32(v - r0)
            gk = f32(gout[b, n] * inv_k)
            zb = f32(f32(z[b, n]) - f32(0.01))
            for i in range(T):
                wr = f32(1) - fr if i == 0 else (fr if i == T - 1 else f32(1))
                r = min(max(r0 - R + i, 0), S_H - 1)
                for k in range(T):
                    wc = f32(1) - fc if k == 0 else (fc if k == T - 1 else f32(1))
                    c = min(max(c0 - R + k, 0), S_W - 1)
                    st = f32(1) if f32(zb - smap[b, r, c, 1]) > 0 else f32(0)
                    term = f32(gk * -f32(f32(wr * wc) * st))
                    terms.setdefault((b, r, c), []).append(((i, r0, k, c0, b * N + n), term))
    want = np.zeros((B, S_H, S_W, 2), np.float32)
    for x, seq in terms.items():
        acc = 0.0
        for _, term in sorted(seq, key=lambda e: e[0]):
            acc = acc + float(term)
        want[x + (0,)] = np.float32(acc)
    assert np.array_equal(got.cpu().numpy(), want)


def _abi_call(L, p, M, smap, per_item, R, softness, bias, gout):
    """Forward and backward through the library L directly: (out, grad_positions, grad_light_matrix)."""
    B, N = p.shape[:2]
    out = torch.empty((B * N,), device=DEV)
    gp = torch.empty((B * N, 3), device=DEV)
    gM = torch.empty(M.shape, device=DEV)
    ws = torch.empty(int(L.dirt_shadow_workspace_bytes(B, N)), dtype=torch.uint8, device=DEV)
    s = torch.cuda.current_stream().cuda_stream
    args = (p.data_ptr(), 3, M.data_ptr(), smap.data_ptr(), int(per_item), smap.shape[-3], smap.shape[-2], R, softness,
            bias)
    assert L.dirt_shadow_forward(*args, out.data_ptr(), B, N, s) == 0
    assert L.dirt_shadow_backward(*args, gout.data_ptr(), gp.data_ptr(), gM.data_ptr(), None, ws.data_ptr(),
                                  ws.numel(), B, N, s) == 0
    torch.cuda.synchronize()
    return out, gp, gM


def test_small_grid_build_is_bit_identical(tmp_path_factory):
    from variant_builds import small_grid_library
    small = small_grid_library(tmp_path_factory)
    B, N = 7, 3000
    for per_item in (True, False):
        p, M, smap = _case(B, N, per_item, seed=13)
        t = [torch.tensor(x, dtype=torch.float32, device=DEV).contiguous() for x in (p, M, smap)]
        gout = torch.randn((B * N,), device=DEV)
        a = _abi_call(_lib.lib(), *t, per_item, 1, 0.05, 0.01, gout)
        b = _abi_call(small, *t, per_item, 1, 0.05, 0.01, gout)
        for x, y in zip(a, b):
            assert torch.equal(x, y)


def test_pipeline_against_the_oracle():
    """shadow_map + shadow_visibility on the GPU against the oracle's map, the restatement and the oracle's backward
    pass on the map gradient: the map, the visibility and the occluder's vertex gradient."""
    from oracle import oracle
    S = 64
    half, a = 0.3, 0.1
    v = np.array([[a - half, -half, 0., 1], [a + half, -half, 0., 1], [a + half, half, 0., 1], [a - half, half, 0., 1]],
                 np.float32)
    v[:, 2] = [0.0, 0.1, 0.05, -0.05]
    f = np.array([[0, 1, 2], [0, 2, 3]], np.int32)
    cols = np.stack([np.ones(4, np.float32), v[:, 2]], 1)
    px = oracle.forward(np.zeros((1, S, S, 2), np.float32), v[None], cols[None], f[None])
    g = np.linspace(-0.95, 0.95, 150)
    yy, xx = np.meshgrid(g, g, indexing='ij')
    pts = np.stack([xx.ravel(), yy.ravel(), np.full(xx.size, 0.5)], 1)
    weight = np.exp(-((pts[:, 0] - 0.25) ** 2 + pts[:, 1] ** 2) / 0.1)

    verts = torch.tensor(v[:, :3], device=DEV, requires_grad=True)
    smap = lighting.shadow_map(verts, torch.tensor(f, device=DEV), torch.eye(4, device=DEV), S, S)
    got_map = smap.detach().cpu().numpy()
    assert np.array_equal(got_map[..., 0], px[0, ..., 0])
    ok, worst = rel_close(got_map[..., 1], px[0, ..., 1], name='shadow pipeline map depth')
    assert ok, worst
    vis = lighting.shadow_visibility(torch.tensor(pts, dtype=torch.float32, device=DEV), torch.eye(4, device=DEV), smap,
                                     1, 0.01, 0.005)
    (vis[:, 0] * torch.tensor(weight, dtype=torch.float32, device=DEV)).sum().backward()

    sm = torch.tensor(px[0], dtype=torch.float64, requires_grad=True)
    v64 = lighting._shadow_visibility(torch.tensor(pts), torch.eye(4, dtype=torch.float64), sm, 1, 0.01, 0.005)
    (v64[:, 0] * torch.tensor(weight)).sum().backward()
    ok, worst = rel_close(vis.detach().cpu().numpy(), v64.detach().numpy(), name='shadow pipeline visibility')
    assert ok, worst
    _, gv, _ = oracle.backward(v[None], f[None], px, sm.grad.numpy().astype(np.float32)[None])
    # the vertex gradient passes through the map gradient's float atomics and the rasteriser's fp32 backward pass
    ok, worst = rel_close(verts.grad.cpu().numpy(), gv[0, :, :3], rel=1e-3, name='shadow pipeline occluder gradient')
    assert ok, worst
    assert float(verts.grad[:, 0].sum()) < 0


def test_example_runs():
    spec = importlib.util.spec_from_file_location('shadow_example', os.path.join(ROOT, 'examples', 'shadow.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    err_a, err_b = mod.main(steps=3)
    assert np.isfinite(err_a) and np.isfinite(err_b)
