"""CPU: tests/mesh_order.py, the float32 restatement of the mesh kernels, anchored to the torch restatements it restates.

On well-conditioned meshes its outputs and gradients agree with lighting._vertex_normals, _vertex_normals_pre_split,
_vertex_tangents and mesh._vertex_laplacian (float64, and float64 autograd) within conftest.rel_close, so a bit-exact
GPU test against it cannot inherit a kernel's mistake.  On integer-coordinate kinks it has the float64 zeros and signs.
Its adjacency equals an independent construction, and every fixture with long rows tells the warp's lane tree from a
left-to-right sum, so that a bit-exact match shows which row path ran."""
import numpy as np
import pytest
import torch

import mesh_order as mo
from conftest import rel_close

MESHES = {'icosphere': mo.icosphere, 'grid': mo.grid, 'uv_sphere': mo.uv_sphere, 'fan': lambda: mo.fan(3000)}


def _check(got, want, name, rel=1e-4, atol=0.):
    """rel_close, with entries within atol of float64 counted as equal"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    ok, ratio = rel_close(np.where(np.abs(got - want) <= atol, want, got), want, rel=rel)
    assert ok, '%s: worst error / tolerance %.3f' % (name, ratio)


def _batch(v, B, seed):
    g = np.random.default_rng(seed)
    return (v[None] * (1. + 0.1 * g.random((B, 1, 1))) + 0.1 * g.standard_normal((B, 1, 3))).astype(np.float32)


def _autograd(fn, inputs, wrt, grad_out):
    leaves = [torch.tensor(np.asarray(x, np.float64), requires_grad=i in wrt) for i, x in enumerate(inputs)]
    out = fn(*leaves)
    out.backward(torch.tensor(np.asarray(grad_out, np.float64)))
    return out.detach().numpy(), [leaves[i].grad.numpy() for i in wrt]


@pytest.mark.parametrize('name', sorted(MESHES))
def test_normals_agree_with_the_torch_restatement(name):
    from dirt_b200 import lighting
    v, f = MESHES[name]()
    P = _batch(v, 2, 1)
    g = np.random.default_rng(2).standard_normal(P.shape).astype(np.float32)
    want, (gw,) = _autograd(lambda x: lighting._vertex_normals(x, torch.tensor(f)), [P], [0], g)
    _check(mo.normals_forward(P, f), want, 'normals')
    _check(mo.normals_backward(P, f, g), gw, 'normals grad')
    # pre-split: against the restatement on the split mesh, where index_copy is defined
    Ps, fs = P[:, f.reshape(-1)], np.arange(f.size, dtype=np.int32).reshape(-1, 3)
    gs = np.random.default_rng(3).standard_normal(Ps.shape).astype(np.float32)
    want, (gw,) = _autograd(lambda x: lighting._vertex_normals_pre_split(x, torch.tensor(fs)), [Ps], [0], gs)
    # one face's normal, not a sum: the uv-sphere's pole faces have a 1.6 degree corner, where a float32 cross product
    # keeps about 2e-6 of the normal (test_gpu_normals.py uses the same bar there)
    _check(mo.normals_forward(Ps, fs, mo.PRE_SPLIT), want, 'pre-split', 2e-4 if name == 'uv_sphere' else 1e-4)
    _check(mo.normals_backward(Ps, fs, gs, mo.PRE_SPLIT), gw, 'pre-split grad')


@pytest.mark.parametrize('name', sorted(MESHES))
def test_tangents_agree_with_the_torch_restatement(name):
    """Planar uvs, and the uv-sphere's own spherical uvs (its seam split), where planar ones would fold."""
    from dirt_b200 import lighting
    if name == 'uv_sphere':
        v, uv, f = mo.seamed_sphere(48, 24)   # poles of valence 48: long rows (at 224 the pole tangents lose 1e-4)
        P = _batch(v, 2, 4)
        U = np.stack([uv, uv])
    else:
        v, f = MESHES[name]()
        P = _batch(v, 2, 4)
        U = np.stack([mo.uv_for(p) for p in P])
    r = np.random.default_rng(5)
    N = (mo.normals_forward(P, f) + 0.05 * r.standard_normal(P.shape)).astype(np.float32)
    g = r.standard_normal(P.shape[:-1] + (4,)).astype(np.float32)
    fn = lambda x, u, n: lighting._vertex_tangents(x, u, torch.tensor(f), n)
    want, (gp, gu, gn) = _autograd(fn, [P, U, N], [0, 1, 2], g)
    got = mo.tangents_forward(P, U, N, f)
    _check(got[..., :3], want[..., :3], 'tangents')
    assert np.array_equal(got[..., 3], want[..., 3])
    bp, bu, bn = mo.tangents_backward(P, U, N, f, g)
    _check(bp, gp, 'tangents grad vertices')
    _check(bu, gu, 'tangents grad uvs')
    _check(bn, gn, 'tangents grad normals')


@pytest.mark.parametrize('mode', ['uniform', 'cotangent'])
@pytest.mark.parametrize('name', sorted(MESHES))
def test_laplacian_agrees_with_the_torch_restatement(name, mode):
    from dirt_b200 import mesh
    v, f = MESHES[name]()
    P = _batch(v, 2, 6)
    g = np.random.default_rng(7).standard_normal(P.shape).astype(np.float32)
    want, (gw,) = _autograd(lambda x: mesh._vertex_laplacian(x, torch.tensor(f), mode), [P], [0], g)
    m = mo.UNIFORM if mode == 'uniform' else mo.COTANGENT
    _check(mo.laplacian_forward(P, f, m), want, 'laplacian')
    _check(mo.laplacian_backward(P, f, g, m), gw, 'laplacian grad')


@pytest.mark.parametrize('mode', ['edge_lengths', 'normal_consistency'])
@pytest.mark.parametrize('name', sorted(MESHES))
def test_edge_terms_agree_with_the_torch_restatement(name, mode):
    from dirt_b200 import mesh
    v, f = MESHES[name]()
    P = _batch(v, 2, 10)
    g = np.random.default_rng(11).standard_normal(P.shape[:1] + f.shape).astype(np.float32)
    want, (gw,) = _autograd(lambda x: getattr(mesh, '_' + mode)(x, torch.tensor(f)), [P], [0], g)
    m = mo.LENGTH if mode == 'edge_lengths' else mo.CONSISTENCY
    # values within 1e-6 of float64 count as equal, as in test_gpu_edge_terms.py: 1 - u_f . mean(u_g) cancels
    _check(mo.edge_terms_forward(P, f, m), want, mode, atol=1e-6)
    # the uv-sphere's pole vertices sum the consistency terms of 224 sliver faces that nearly cancel (DESIGN.md §7.17)
    _check(mo.edge_terms_backward(P, f, g, m), gw, mode + ' grad',
           5e-4 if (name, m) == ('uv_sphere', mo.CONSISTENCY) else 1e-4)


def _signs_and_zeros(got, want, zeros=True):
    """equal zeros, and equal signs wherever float64 is clear of 0"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert not zeros or np.array_equal(got == 0, want == 0)
    clear = np.abs(want) > 1e-6 * np.abs(want).max()
    assert np.array_equal(np.sign(got[clear]), np.sign(want[clear]))


def test_kinks_have_the_float64_zeros_and_signs():
    """Integer coordinates: a collinear face, a face naming a vertex twice (gradients of 1e24 through both divisions
    by 1e-12) and a face with its reversed copy (normal 0, gradient 0), and the Laplacian's zero-area faces."""
    from dirt_b200 import lighting, mesh
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [3, 1, 0], [4, 2, 1], [0, 5, 0], [1, 5, 2], [0, 6, 3]], np.float32)
    f = np.array([[0, 1, 2], [3, 3, 4], [5, 6, 7], [5, 7, 6]], np.int32)
    g = np.random.default_rng(12).integers(-3, 4, (1, 8, 3)).astype(np.float32)
    g[0, 7] = g[0, 6]
    P = v[None]
    want, (gw,) = _autograd(lambda x: lighting._vertex_normals(x, torch.tensor(f)), [P], [0], g)
    _signs_and_zeros(mo.normals_forward(P, f), want)
    _signs_and_zeros(mo.normals_backward(P, f, g), gw)
    assert np.abs(gw).max() > 1e23
    for mode, m in (('uniform', mo.UNIFORM), ('cotangent', mo.COTANGENT)):
        want, (gw,) = _autograd(lambda x: mesh._vertex_laplacian(x, torch.tensor(f), mode), [P], [0], g)
        _signs_and_zeros(mo.laplacian_forward(P, f, m), want)
        # the cotangent gradient of a zero-area face is a sum of 1e24-scale terms that cancel: its rounding residues
        # differ between float32 and float64, so there only the entries clear of them are compared
        _signs_and_zeros(mo.laplacian_backward(P, f, g, m), gw, zeros=m == mo.UNIFORM)


def test_adjacency_agrees_with_a_lexsort():
    r = np.random.default_rng(8)
    for V, F, items, stride in ((50, 300, 1, 0), (31, 64, 3, 0), (20, 40, 4, 120), (1, 5, 2, 15)):
        faces = r.integers(-2, V + 2, (max(items if stride else 1, 1), F, 3))
        offsets, inc = mo.adjacency(faces if stride else faces[0], V, items, stride)
        rows, ids = [], []
        for b in range(items):
            t = faces[b if stride else 0]
            for f in range(F):
                if ((t[f] >= 0) & (t[f] < V)).all():
                    for k in range(3):
                        rows.append(b * V + t[f, k])
                        ids.append(b * 3 * F + k * F + f)
        rows, ids = np.array(rows, np.int64), np.array(ids, np.int64)
        order = np.lexsort((ids, rows))
        assert np.array_equal(inc, ids[order])
        assert np.array_equal(offsets, np.searchsorted(rows[order], np.arange(items * V + 1)))


LONG_ROW_FIXTURES = {'uv_sphere': mo.uv_sphere, 'fan': mo.fan, 'rows_32_33': mo.rows_32_33,
                     'full_warp': mo.full_warp, 'straddle': mo.straddle}


@pytest.mark.parametrize('name', sorted(LONG_ROW_FIXTURES))
def test_long_row_fixtures_tell_the_row_paths_apart(name):
    """The long rows' lane tree gives other bits than a left-to-right sum on some rows, for the normals' face terms
    and the Laplacian's corner terms, and summing the rows of exactly 32 by the tree would too: so a bit-exact match
    shows that each row took its path."""
    v, f = LONG_ROW_FIXTURES[name]()
    P = _batch(v, 3, 9)
    c = mo.Corners(f, len(v))
    assert (c.count > mo.LONG_ROW).any()
    Pt = mo._t(P)
    for terms in (mo.face_unit(c, Pt), mo.laplacian_terms(mo.Wedge(c, Pt), mo.COTANGENT)):
        tree = mo.row_sum(c.offsets, terms)
        flat = mo.row_sum(c.offsets, terms, long_row=None)
        long_rows = c.count > mo.LONG_ROW
        assert (tree[long_rows].view(np.int32) != flat[long_rows].view(np.int32)).any(), name
        assert np.array_equal(tree[~long_rows], flat[~long_rows])
        if (c.count == mo.LONG_ROW).any():
            early = mo.row_sum(c.offsets, terms, long_row=mo.LONG_ROW - 1)
            rows = c.count == mo.LONG_ROW
            assert (early[rows].view(np.int32) != tree[rows].view(np.int32)).any(), name


def test_tangent_fixture_reaches_its_cases():
    """tangent_cases has faces with s = 0 (zero uv area, collinear and identical uvs), faces of both signs, a vertex
    whose normal lies along one of its face tangents and a zero normal."""
    v, uv, f, n = mo.tangent_cases()
    c = mo.Corners(f, len(v))
    u = mo.UvFace(c, mo._t(v[None]), mo._t(uv[None]))
    assert (u.s == 0).sum() >= 2 and (u.s > 0).any() and (u.s < 0).any()
    assert not n[5].any()
    t = mo.normalise(u.face_u())[c.offsets[45]:c.offsets[46], 0]
    assert np.abs(mo.dot3(mo.normalise(n[45]), t[0]) - 1) < 1e-6
