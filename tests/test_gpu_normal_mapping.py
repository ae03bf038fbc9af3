"""GPU: the vertex tangents' and the normal mapping's CUDA paths against their torch restatements (`_vertex_tangents`,
`_perturb_normals` of dirt_b200/lighting.py).

Forward values against the restatement in float64, gradients against float64 autograd of the restatement, both with
conftest.rel_close (1e-4).  The handedness w is a step: it is compared exactly except where |(n x T) . b_v| is within
rounding of 0."""
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


def _check(got, want, name):
    ok, ratio = rel_close(got.detach().double().cpu().numpy(), want.detach().double().cpu().numpy(), name=name)
    assert ok, '%s: worst error / tolerance %.3f' % (name, ratio)


# ---- meshes -----------------------------------------------------------------------------------------------------------

def seamed_sphere(columns, rows):
    """A uv sphere whose seam column is split: columns + 1 vertices per ring, the last a copy of the first with u = 1,
    so each side of the seam has its own uvs.  Returns float32 positions [V, 3], uvs [V, 2] and int32 faces [F, 3]."""
    u = np.arange(columns + 1) / columns
    v = np.arange(rows + 1) / rows
    uu, vv = np.meshgrid(u, v)
    phi, theta = 2 * np.pi * uu, np.pi * vv
    p = np.stack([np.sin(theta) * np.sin(phi), np.cos(theta), np.sin(theta) * np.cos(phi)], -1).reshape(-1, 3)
    uv = np.stack([uu, vv], -1).reshape(-1, 2)
    i = np.arange(rows)[:, None] * (columns + 1) + np.arange(columns)[None, :]
    a, b, c, d = i, i + 1, i + columns + 1, i + columns + 2
    f = np.concatenate([np.stack([a, c, b], -1)[1:], np.stack([b, c, d], -1)[:-1]]).reshape(-1, 3)
    return p.astype(np.float32), uv.astype(np.float32), f.astype(np.int32)


def _fan(n=120):
    """n faces around vertex 0, uvs from the positions: a row longer than 32 corners for the centre."""
    a = np.arange(n + 1) * 2.399963
    rim = np.stack([np.cos(a), np.sin(a), 0.01 * np.arange(n + 1)], -1)
    p = np.concatenate([np.zeros((1, 3)), rim]).astype(np.float32)
    uv = (0.5 + 0.4 * p[:, :2]).astype(np.float32)
    f = np.stack([np.zeros(n), np.arange(1, n + 1), np.arange(2, n + 2)], -1).astype(np.int32)
    f[-1, 2] = 1
    return p, uv, f


MESHES = {'sphere': lambda: seamed_sphere(24, 12), 'fan': _fan}


def _inputs(lighting, mesh, lead=(), uv_per_item=False, seed=0, w=False):
    p, uv, f = MESHES[mesh]() if isinstance(mesh, str) else mesh
    g = _gen(seed)
    B = int(np.prod(lead)) if lead else 1
    x = torch.tensor(p, device=DEV)[None] * (1 + 0.1 * torch.randn((B, p.shape[0], 1), generator=g, device=DEV))
    x = x.reshape(lead + p.shape)
    if w:
        x = torch.cat([x, torch.ones(x.shape[:-1] + (1,), device=DEV)], -1)
    uvs = torch.tensor(uv, device=DEV)
    if uv_per_item:
        uvs = (uvs[None] + 0.02 * torch.randn((B,) + uv.shape, generator=g, device=DEV)).reshape(lead + uv.shape)
    faces = torch.tensor(f, device=DEV)
    n = lighting.vertex_normals(x, faces).detach()
    n = n + 0.05 * torch.randn(n.shape, generator=g, device=DEV)   # not unit, not exactly the face normals
    return x, uvs, faces, n


def _compare_forward(lighting, got, x, uvs, faces, n, name):
    want = lighting._vertex_tangents(x.double(), uvs.double(), faces.long(), n.double())
    _check(got[..., :3], want[..., :3], name + ' T')
    # w: exact except where the handedness test is within rounding of 0
    nn = torch.nn.functional.normalize(n.double(), dim=-1)
    p, uv = x.double()[..., :3], uvs.double()
    b_v = torch.zeros(want.shape[:-1] + (3,), dtype=torch.float64, device=DEV)
    corners, tex = p[..., faces.long(), :], uv[..., faces.long(), :]
    e1, e2 = corners[..., 1, :] - corners[..., 0, :], corners[..., 2, :] - corners[..., 0, :]
    d1, d2 = tex[..., 1, :] - tex[..., 0, :], tex[..., 2, :] - tex[..., 0, :]
    s = torch.sign(d1[..., :1] * d2[..., 1:] - d2[..., :1] * d1[..., 1:])
    b_f = torch.nn.functional.normalize(s * (e2 * d1[..., :1] - e1 * d2[..., :1]), dim=-1, eps=1e-300)
    for k in range(3):
        b_v = b_v.index_add(-2, faces[:, k].long(), b_f.expand(want.shape[:-2] + b_f.shape[-2:]))
    h = (torch.linalg.cross(nn, want[..., :3], dim=-1) * b_v).sum(-1)
    sure = h.abs() > 1e-4 * (b_v.norm(dim=-1) + 1e-30)
    assert torch.equal(got[..., 3][sure].double(), want[..., 3][sure]), name + ' w'


@pytest.mark.parametrize('mesh', ['sphere', 'fan'])
@pytest.mark.parametrize('lead,uv_per_item,w', [((), False, False), ((3,), False, True), ((2, 2), True, False)])
def test_tangents_forward_matches_the_restatement(lighting, mesh, lead, uv_per_item, w):
    x, uvs, faces, n = _inputs(lighting, mesh, lead, uv_per_item, 1, w)
    got = lighting.vertex_tangents(x, uvs, faces, n)
    assert got.shape == lead + (x.shape[-2], 4) and got.dtype == torch.float32
    _compare_forward(lighting, got, x, uvs, faces, n, 'tangents fwd vs fp64')


def _grads(fn, inputs, wanted, grad_out):
    leaves = [t.detach().clone().requires_grad_(i in wanted) for i, t in enumerate(inputs)]
    out = fn(*leaves)
    (out * grad_out).sum().backward()
    return [leaves[i].grad for i in wanted]


def _tangents_fn(lighting, faces, restate=False):
    if restate:
        return lambda x, uv, n: lighting._vertex_tangents(x, uv, faces.long(), n)
    return lambda x, uv, n: lighting.vertex_tangents(x, uv, faces, n)


@pytest.mark.parametrize('mesh', ['sphere', 'fan'])
@pytest.mark.parametrize('lead,uv_per_item,w', [((), False, False), ((4,), False, True), ((2, 3), True, False)])
def test_tangents_gradients_match_autograd_of_the_restatement(lighting, mesh, lead, uv_per_item, w):
    x, uvs, faces, n = _inputs(lighting, mesh, lead, uv_per_item, 2, w)
    grad_out = torch.randn(x.shape[:-1] + (4,), generator=_gen(3), device=DEV)
    got = _grads(_tangents_fn(lighting, faces), (x, uvs, n), (0, 1, 2), grad_out)
    want = _grads(_tangents_fn(lighting, faces, True), (x.double(), uvs.double(), n.double()), (0, 1, 2),
                  grad_out.double())
    for g, e, name in zip(got, want, ('vertices', 'uvs', 'normals')):
        assert g.shape == e.shape
        _check(g, e, 'tangents grad %s vs fp64' % name)
    if w:
        assert not got[0][..., 3].any()
    assert not got[1][..., 0].any()
    # each gradient alone equals its value in the full call
    for i in range(3):
        alone = _grads(_tangents_fn(lighting, faces), (x, uvs, n), (i,), grad_out)[0]
        assert torch.equal(alone, got[i])


def test_tangents_invalid_int64_and_duplicated_faces(lighting):
    p, uv, f = seamed_sphere(12, 6)
    V = p.shape[0]
    bad = np.array([[0, 1, V], [-1, 2, 3], [4, V + 5, 6], [7, 8, V]], np.int64)
    dup = np.array([[5, 5, 6], [9, 10, 9]], np.int64)
    faces64 = torch.tensor(np.concatenate([f.astype(np.int64), bad, dup, [[0, 1, (1 << 33)]]]), device=DEV)
    valid = torch.tensor(np.concatenate([f.astype(np.int64), dup]), device=DEV)
    x, uvs, _, n = _inputs(lighting, (p, uv, f), (2,), False, 4)
    got = lighting.vertex_tangents(x, uvs, faces64, n)
    _compare_forward(lighting, got, x, uvs, valid, n, 'tangents fwd invalid faces')
    grad_out = torch.randn(x.shape[:-1] + (4,), generator=_gen(5), device=DEV)
    g = _grads(lambda a, b, c: lighting.vertex_tangents(a, b, faces64, c), (x, uvs, n), (0, 1, 2), grad_out)
    e = _grads(lambda a, b, c: lighting._vertex_tangents(a, b, valid, c), (x.double(), uvs.double(), n.double()),
               (0, 1, 2), grad_out.double())
    for a, b, name in zip(g, e, ('vertices', 'uvs', 'normals')):
        _check(a, b, 'tangents grad %s invalid faces' % name)


def test_tangents_empty_inputs(lighting):
    p, uv, f = seamed_sphere(6, 3)
    V = p.shape[0]
    for lead, nv, faces in (((2,), V, np.zeros((0, 3), np.int32)), ((2,), 0, np.zeros((0, 3), np.int32)),
                            ((0,), V, f), ((), V, np.zeros((0, 3), np.int64))):
        x = torch.rand(lead + (nv, 3), generator=_gen(6), device=DEV).requires_grad_(True)
        uvs = torch.rand((nv, 2), generator=_gen(7), device=DEV).requires_grad_(True)
        n = torch.rand(lead + (nv, 3), generator=_gen(8), device=DEV).requires_grad_(True)
        out = lighting.vertex_tangents(x, uvs, torch.tensor(faces, device=DEV), n)
        assert out.shape == lead + (nv, 4)
        assert not out[..., :3].any() and (out[..., 3] == 1).all()
        out.sum().backward()
        for t in (x, uvs, n):
            assert t.grad.shape == t.shape and not t.grad.any()


def test_tangents_more_items_than_a_grid_dimension(lighting):
    p, uv, f = seamed_sphere(4, 3)
    x, uvs, faces, n = _inputs(lighting, (p, uv, f), (70000,), True, 9)
    got = lighting.vertex_tangents(x, uvs, faces, n)
    _compare_forward(lighting, got, x, uvs, faces, n, 'tangents fwd 70000 items')
    grad_out = torch.randn(got.shape, generator=_gen(10), device=DEV)
    g = _grads(_tangents_fn(lighting, faces), (x, uvs, n), (0, 1, 2), grad_out)
    e = _grads(_tangents_fn(lighting, faces, True), (x.double(), uvs.double(), n.double()), (0, 1, 2), grad_out.double())
    for a, b, name in zip(g, e, ('vertices', 'uvs', 'normals')):
        _check(a, b, 'tangents grad %s 70000 items' % name)


def test_tangents_double_backward(lighting):
    x, uvs, faces, n = _inputs(lighting, 'sphere', (2,), False, 11)
    weights = torch.randn(x.shape[:-1] + (4,), generator=_gen(30), device=DEV)   # |T| = 1: out.square() would not do
    x = x.clone().requires_grad_(True)
    out = lighting.vertex_tangents(x, uvs, faces, n)
    g, = torch.autograd.grad((out * weights).square().sum(), x, create_graph=True)
    gg, = torch.autograd.grad(g.square().sum(), x)
    xd = x.detach().double().requires_grad_(True)
    outd = lighting._vertex_tangents(xd, uvs.double(), faces.long(), n.double())
    gd, = torch.autograd.grad((outd * weights.double()).square().sum(), xd, create_graph=True)
    ggd, = torch.autograd.grad(gd.square().sum(), xd)
    _check(g, gd, 'tangents grad under create_graph')
    ok, ratio = rel_close(gg.double().cpu().numpy(), ggd.cpu().numpy(), rel=1e-3)
    assert ok, ratio


# ---- perturb_normals --------------------------------------------------------------------------------------------------

def _points(shape, seed, background=False):
    """Random points with tangents like interpolated ones: mostly orthogonal to the normal (Gram-Schmidt of a tangent
    nearly along the normal is ill-conditioned in any precision).  With `background`, the first three of each row are
    background pixels, with zero normals and tangents (their normal gradient is ~1e12, as torch's, so they are left out
    of gradient comparisons)."""
    g = _gen(seed)
    n = torch.randn(shape + (3,), generator=g, device=DEV) * 2
    across = torch.nn.functional.normalize(torch.linalg.cross(n, torch.randn(shape + (3,), generator=g, device=DEV)),
                                           dim=-1)
    size = 0.5 + torch.rand(shape + (1,), generator=g, device=DEV)
    along = 0.5 * torch.randn(shape + (1,), generator=g, device=DEV)
    t = torch.cat([size * across + along * torch.nn.functional.normalize(n, dim=-1),
                   torch.randn(shape + (1,), generator=g, device=DEV)], -1)
    m = torch.nn.functional.normalize(torch.randn(shape + (3,), generator=g, device=DEV) + torch.tensor(
        [0., 0., 2.], device=DEV), dim=-1)
    if background:
        n[..., :3, :] = 0.
        t[..., :3, :] = 0.
    return n, t, m


def _perturb_grads(fn, inputs, grad_out):
    leaves = [t.detach().clone().requires_grad_(True) for t in inputs]
    (fn(*leaves) * grad_out).sum().backward()
    return [l.grad for l in leaves]


@pytest.mark.parametrize('shape', [(1000,), (3, 777), (2, 3, 257)])
def test_perturb_matches_the_restatement(lighting, shape):
    n, t, m = _points(shape, 12, background=True)
    got = lighting.perturb_normals(n, t, m)
    assert not got[..., :3, :].any()
    _check(got, lighting._perturb_normals(n.double(), t.double(), m.double()), 'perturb fwd vs fp64')
    n, t, m = _points(shape, 12)
    got = lighting.perturb_normals(n, t, m)
    grad_out = torch.randn(got.shape, generator=_gen(13), device=DEV)
    g = _perturb_grads(lighting.perturb_normals, (n, t, m), grad_out)
    e = _perturb_grads(lighting._perturb_normals, (n.double(), t.double(), m.double()), grad_out.double())
    for a, b, name in zip(g, e, ('normals', 'tangents', 'samples')):
        _check(a, b, 'perturb grad %s vs fp64' % name)
    assert not g[1][..., 3].any()


def test_perturb_on_gbuffer_views_reads_in_place(lighting):
    B, H, W = 2, 33, 47
    gbuffer = torch.randn(B, H, W, 14, generator=_gen(14), device=DEV).requires_grad_(True)
    m = torch.nn.functional.normalize(torch.randn(B, H, W, 3, generator=_gen(15), device=DEV), dim=-1)
    assert lighting._rows(gbuffer[..., 4:7], 3).data_ptr() == gbuffer[..., 4:7].data_ptr()
    assert lighting._rows(gbuffer[..., 7:11], 4).data_ptr() == gbuffer[..., 7:11].data_ptr()
    got = lighting.perturb_normals(gbuffer[..., 4:7], gbuffer[..., 7:11], m)
    contiguous = lighting.perturb_normals(gbuffer[..., 4:7].contiguous(), gbuffer[..., 7:11].contiguous(), m)
    assert torch.equal(got, contiguous)
    want = lighting._perturb_normals(gbuffer[..., 4:7].double(), gbuffer[..., 7:11].double(), m.double())
    _check(got, want, 'perturb fwd gbuffer views')
    grad_out = torch.randn(got.shape, generator=_gen(16), device=DEV)
    (got * grad_out).sum().backward()
    gd = gbuffer.detach().double().requires_grad_(True)
    (lighting._perturb_normals(gd[..., 4:7], gd[..., 7:11], m.double()) * grad_out.double()).sum().backward()
    _check(gbuffer.grad, gd.grad, 'perturb grad gbuffer views')


def test_perturb_empty_and_many_items(lighting):
    for shape in ((0, 5), (4, 0)):
        n, t, m = (torch.zeros(shape + (k,), device=DEV, requires_grad=True) for k in (3, 4, 3))
        out = lighting.perturb_normals(n, t, m)
        assert out.shape == shape + (3,)
        out.sum().backward()
        assert n.grad.shape == n.shape
    n, t, m = _points((70000, 5), 17, background=True)
    got = lighting.perturb_normals(n, t, m)
    _check(got, lighting._perturb_normals(n.double(), t.double(), m.double()), 'perturb fwd 70000 items')


def test_perturb_double_backward(lighting):
    n, t, m = _points((2, 300), 18)
    leaves = [a.clone().requires_grad_(True) for a in (n, t, m)]
    out = lighting.perturb_normals(*leaves)
    weights = torch.randn(out.shape, generator=_gen(31), device=DEV)   # |out| = 1: out.square() alone would not do
    g = torch.autograd.grad((out * weights).square().sum(), leaves, create_graph=True)
    gg = torch.autograd.grad(sum(x.square().sum() for x in g), leaves)
    dl = [a.double().requires_grad_(True) for a in (n, t, m)]
    outd = lighting._perturb_normals(*dl)
    gd = torch.autograd.grad((outd * weights.double()).square().sum(), dl, create_graph=True)
    ggd = torch.autograd.grad(sum(x.square().sum() for x in gd), dl)
    for a, b in zip(g, gd):
        _check(a, b, 'perturb grad under create_graph')
    for a, b in zip(gg, ggd):
        ok, ratio = rel_close(a.double().cpu().numpy(), b.cpu().numpy(), rel=1e-3)
        assert ok, ratio


# ---- determinism ------------------------------------------------------------------------------------------------------

def test_repeated_calls_are_bit_identical(lighting):
    x, uvs, faces, n = _inputs(lighting, _fan(400), (8,), False, 19)
    grad_out = torch.randn(x.shape[:-1] + (4,), generator=_gen(20), device=DEV)
    pn, pt, pm = _points((8, 5000), 21, background=True)
    pg = torch.randn(pn.shape, generator=_gen(22), device=DEV)
    runs = []
    for _ in range(3):
        g = _grads(_tangents_fn(lighting, faces), (x, uvs, n), (0, 1, 2), grad_out)
        q = _perturb_grads(lighting.perturb_normals, (pn, pt, pm), pg)
        runs.append([lighting.vertex_tangents(x, uvs, faces, n), lighting.perturb_normals(pn, pt, pm)] + g + q)
    for run in runs[1:]:
        for a, b in zip(run, runs[0]):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_cuda_graph_capture_and_replay(lighting):
    x, uvs, faces, n = _inputs(lighting, 'sphere', (4,), False, 23)
    x, uvs, n = (t.clone().requires_grad_(True) for t in (x, uvs, n))
    grad_out = torch.randn(4, x.shape[1], 3, generator=_gen(24), device=DEV)
    m = torch.nn.functional.normalize(torch.randn(4, x.shape[1], 3, generator=_gen(25), device=DEV), dim=-1)

    def step():
        for t in (x, uvs, n):
            t.grad = None
        out = lighting.perturb_normals(n, lighting.vertex_tangents(x, uvs, faces, n), m)
        (out * grad_out).sum().backward()
        return out

    eager = step().detach().clone()
    eager_grads = [t.grad.clone() for t in (x, uvs, n)]
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
        for t, e in zip((x, uvs, n), eager_grads):
            assert torch.equal(t.grad, e)


def test_small_grid_build_is_bit_identical(lighting, tmp_path_factory):
    """The build with every grid cap lowered (tests/variant_builds.py) runs many rounds of each grid-stride loop, the
    last one partial, and more items than its gridDim.y; its results equal the product's bit for bit."""
    import ctypes
    from variant_builds import small_grid_library
    from dirt_b200 import _lib
    small = small_grid_library(tmp_path_factory)
    x, uvs, faces, n = _inputs(lighting, _fan(300), (7,), True, 26)
    pn, pt, pm = _points((7, 3001), 27)
    grad4 = torch.randn(x.shape[:-1] + (4,), generator=_gen(28), device=DEV)
    grad3 = torch.randn(pn.shape, generator=_gen(29), device=DEV)
    rows = x.reshape(-1, 3)
    uvr, nr = uvs.reshape(-1, 2), n.reshape(-1, 3)
    B, V, F = 7, x.shape[1], faces.shape[0]
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    stream = torch.cuda.current_stream(DEV).cuda_stream
    results = []
    for lib in (_lib.lib(), small):
        ws_bytes = lib.dirt_tangents_workspace_bytes(B, V, F)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
        out = torch.empty(B * V, 4, device=DEV)
        tin = [P(rows), 3, P(uvr), 2, 2 * V, P(nr), 3, P(faces)]
        assert lib.dirt_tangents_forward(*tin, P(out), P(ws), ws_bytes, B, V, F, stream) == 0
        gv, gu, gn = torch.empty(B * V, 3, device=DEV), torch.empty(B * V, 2, device=DEV), torch.empty(B * V, 3, device=DEV)
        assert lib.dirt_tangents_backward(*tin, P(grad4), P(gv), P(gu), P(gn), P(ws), ws_bytes, B, V, F, stream) == 0
        mout = torch.empty(pn.shape, device=DEV)
        min_ = [P(pn), 3, P(pt), 4, P(pm), 3]
        assert lib.dirt_normal_map_forward(*min_, P(mout), 7, 3001, stream) == 0
        qn, qt, qm = (torch.empty(7 * 3001, k, device=DEV) for k in (3, 4, 3))
        assert lib.dirt_normal_map_backward(*min_, P(grad3), P(qn), P(qt), P(qm), 7, 3001, stream) == 0
        torch.cuda.synchronize()
        results.append([out, gv, gu, gn, mout, qn, qt, qm])
    for a, b in zip(*results):
        assert torch.equal(a, b)
    got = lighting.vertex_tangents(x, uvs, faces, n).reshape(-1, 4)
    assert torch.equal(got, results[0][0])


# ---- end to end -------------------------------------------------------------------------------------------------------

def test_normalmap_example_reduces_its_loss(cuda_lib):
    spec = importlib.util.spec_from_file_location('normalmap_example', os.path.join(ROOT, 'examples', 'normalmap.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    before, after = mod.main(steps=60, size=96, verbose=False)
    assert after < 0.25 * before, (before, after)
