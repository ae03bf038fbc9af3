"""CPU: the cube-map lookup's restatement (tests/cubemap_restatement.py) in float64 -- face orientation, seams, the
border table, the nearest and invalid-direction rules -- and the C ABI's and sample_cubemap's argument errors."""
import ctypes
import itertools
import math

import numpy as np
import pytest
import torch

import cubemap_restatement as cm


def _cube(S, C=3, seed=0):
    return torch.from_numpy(np.random.default_rng(seed).random((6, S, S, C)))


def _d(*v):
    return torch.tensor(v, dtype=torch.float64)


def test_each_face_is_oriented_as_the_table():
    S = 8
    cube = torch.arange(6 * S * S, dtype=torch.float64).reshape(6, S, S, 1)
    axis = lambda f: _d(*[(1. if f % 2 == 0 else -1.) if k == f // 2 else 0. for k in range(3)])
    eps = 1e-3
    for f in range(6):
        a, (js, ss), (jt, st) = cm.FACE_AXES[f]
        # the face's centre: s = t = 0.5, the four centre texels in equal parts
        face, s, t, valid = cm.face_coords(axis(f) * 2.5)
        assert int(face) == f and float(s) == 0.5 and float(t) == 0.5 and bool(valid)
        want = cube[f, S // 2 - 1:S // 2 + 1, S // 2 - 1:S // 2 + 1, 0].mean()
        assert torch.allclose(cm.sample(cube, axis(f))[0], want)
        # towards sc = tc = -1 lies texel (0, 0); towards sc = +1, tc = -1 texel (0, S-1)
        for sc, tc, texel in ((-1, -1, (0, 0)), (1, -1, (0, S - 1)), (-1, 1, (S - 1, 0)), (1, 1, (S - 1, S - 1))):
            d = axis(f).clone()
            d[js] = ss * sc * (1 - eps)
            d[jt] = st * tc * (1 - eps)
            assert float(cm.sample(cube, d, 'nearest')[0]) == float(cube[f, texel[0], texel[1], 0]), (f, sc, tc)
    # +X: sc = -z, tc = -y, so (1, e, e) lies towards row 0, column 0
    face, s, t, _ = cm.face_coords(_d(1., 1e-3, 1e-3))
    assert int(face) == 0 and float(s) < 0.5 and float(t) < 0.5


def test_ties_go_to_x_over_y_over_z():
    assert int(cm.face_coords(_d(1., 1., 1.))[0]) == 0
    assert int(cm.face_coords(_d(-1., 1., -1.))[0]) == 1
    assert int(cm.face_coords(_d(0.5, -1., 1.))[0]) == 3
    assert int(cm.face_coords(_d(0., 0., -2.))[0]) == 5


def test_directions_are_scale_invariant():
    cube = _cube(5)
    d = torch.from_numpy(np.random.default_rng(1).standard_normal((500, 3)))
    base = cm.sample(cube, d)
    for k in (1e-20, 0.3, 7.0, 1e20):
        assert torch.allclose(cm.sample(cube, d * k), base, rtol=1e-12, atol=1e-12)
    for k in (0.25, 8.0):   # in float32 too: a power of two changes no rounding
        assert torch.equal(cm.sample(cube.float(), (d * k).float()), cm.sample(cube.float(), d.float()))


def test_constant_cube_map_is_constant_everywhere():
    for S in (1, 2, 3, 6):
        cube = torch.full((6, S, S, 2), 0.7, dtype=torch.float64)
        d = torch.from_numpy(np.random.default_rng(S).standard_normal((2000, 3)))
        corners = torch.tensor(list(itertools.product((-1., 1.), repeat=3)), dtype=torch.float64)
        edges = torch.tensor([[1., 1., 0.3], [-1., 0.2, 1.], [0.7, -1., -1.], [1., -1., 0.]], dtype=torch.float64)
        for mode in ('bilinear', 'nearest'):
            out = cm.sample(cube, torch.cat([d, corners, edges]), mode)
            assert float((out - 0.7).abs().max()) <= 1e-15, (S, mode)


def _edge_points():
    """(point, across) for the 12 edges: a point on the edge and a vector crossing it."""
    pts = []
    for a, b in itertools.combinations(range(3), 2):
        c = 3 - a - b
        for sa, sb in itertools.product((-1., 1.), repeat=2):
            p, n = np.zeros(3), np.zeros(3)
            p[a], p[b], p[c] = sa, sb, 0.37
            n[a], n[b] = sa, -sb
            pts.append((p, n))
    return pts


@pytest.mark.parametrize('S', [1, 2, 3, 7])
def test_continuity_across_all_edges_and_corners(S):
    cube = _cube(S, 2, seed=S)
    delta = 1e-9
    bound = 10 * delta * S * 4 * float(cube.abs().max())
    for p, n in _edge_points():
        pair = torch.from_numpy(np.stack([p + delta * n, p - delta * n]))
        f = cm.face_coords(pair)[0]
        assert int(f[0]) != int(f[1])   # the two lookups are on different faces
        out = cm.sample(cube, pair)
        assert float((out[0] - out[1]).abs().max()) <= bound, (p, n)
    rng = np.random.default_rng(S)
    for corner in itertools.product((-1., 1.), repeat=3):
        pts = np.array(corner) + delta * rng.standard_normal((24, 3))
        out = cm.sample(cube, torch.from_numpy(pts))
        assert len(set(int(f) for f in cm.face_coords(torch.from_numpy(pts))[0])) == 3
        assert float((out - out[:1]).abs().max()) <= bound, corner


@pytest.mark.parametrize('S', [1, 2, 3, 4, 9])
def test_border_table_copies_every_edge_texel_once_per_adjacent_border(S):
    src, corner = cm.border_table(S)
    P = S + 2
    copies = {}
    for f in range(6):
        for i in range(P):
            for j in range(P):
                out_i, out_j = i in (0, P - 1), j in (0, P - 1)
                if out_i != out_j:
                    g = int(src[0, f, i, j]) // (S * S)
                    assert g != f and g // 2 != f // 2   # an adjacent face, not this one or the opposite one
                    copies.setdefault(int(src[0, f, i, j]), []).append(f)
                elif out_i and out_j:
                    assert corner[f, i, j]
                    own = int(src[0, f, i, j])
                    # the three texels of one cube corner: one per face, all different
                    assert len({int(src[k, f, i, j]) // (S * S) for k in range(3)}) == 3 and own // (S * S) == f
    for f in range(6):
        for r in range(S):
            for c in range(S):
                edges = (r == 0) + (r == S - 1) + (c == 0) + (c == S - 1)
                got = copies.get((f * S + r) * S + c, [])
                # one copy per edge the texel lies on, each on a different adjacent face
                assert len(got) == edges and len(set(got)) == edges, (f, r, c, got)


def test_border_copies_are_mutual():
    """If border texel (i, j) of face f copies texel X of face g, then the border texel of g beside X on f's side
    copies the texel of f beside (i, j)."""
    S = 5
    P = S + 2
    for f in range(6):
        for i in range(P):
            for j in range(P):
                if (i in (0, P - 1)) == (j in (0, P - 1)):
                    continue
                g, r, c = cm.border_source(f, i, j, S)
                inner = (f, min(max(i, 1), S) - 1, min(max(j, 1), S) - 1)
                back = [cm.border_source(g, qi, qj, S) for qi, qj in
                        ((0, c + 1), (P - 1, c + 1), (r + 1, 0), (r + 1, P - 1)) if (qi in (0, P - 1)) != (qj in (0, P - 1))
                        and (qi == 0 and r == 0 or qi == P - 1 and r == S - 1 or qj == 0 and c == 0 or qj == P - 1 and c == S - 1)]
                assert inner in back, (f, i, j, (g, r, c), back)


def test_nearest_rule():
    S = 6
    cube = _cube(S, 2, seed=3)
    d = torch.from_numpy(np.random.default_rng(4).standard_normal((3000, 3)))
    out = cm.sample(cube, d, 'nearest')
    face, s, t, _ = cm.face_coords(d)
    r = (t * S).floor().clamp(0, S - 1).long()
    c = (s * S).floor().clamp(0, S - 1).long()
    assert torch.equal(out, cube[face, r, c])


def test_bilinear_is_the_texture_rule_on_the_padded_face():
    """Inside a face, away from the border, the lookup is sample_texture's at (t S - 0.5, s S - 0.5)."""
    import texture_mip_restatement as tm
    S = 8
    cube = _cube(S, 3, seed=5)
    d = torch.from_numpy(np.random.default_rng(6).standard_normal((4000, 3)))
    face, s, t, _ = cm.face_coords(d)
    inside = ((t * S - 0.5) >= 0) & ((t * S - 0.5) < S - 1) & ((s * S - 0.5) >= 0) & ((s * S - 0.5) < S - 1)
    out = cm.sample(cube, d)
    for f in range(6):
        m = inside & (face == f)
        want = tm._ex.sample_texture(cube[f], torch.stack([t[m] * S - 0.5, s[m] * S - 0.5], -1))
        assert torch.allclose(out[m], want, rtol=1e-12, atol=1e-12)


def test_invalid_directions_give_zero_and_no_gradient():
    cube = (_cube(3, 2) + 1.).requires_grad_(True)
    d = torch.tensor([[0., 0., 0.], [-0., 0., -0.], [math.inf, 0., 1.], [1., math.nan, 0.], [-math.inf, -math.inf, 2.],
                      [0.3, -0.2, 0.9]], dtype=torch.float64, requires_grad=True)
    for mode in ('bilinear', 'nearest'):
        out = cm.sample(cube, d, mode)
        assert not out[:-1].any() and bool((out[-1] != 0).all())
        cube.grad, d.grad = None, None
        out[:-1].sum().backward()
        assert not cube.grad.any() and (d.grad is None or not d.grad.any())


def test_gradients_of_the_restatement_are_its_adjoint():
    """float64 gradcheck of the restatement itself: through the border's copies and corners, and to the directions."""
    cube = _cube(2, 2, seed=7).requires_grad_(True)
    d = torch.from_numpy(np.random.default_rng(8).standard_normal((40, 3))).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda c, x: cm.sample(c, x), (cube, d))


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _p(x):
    return ctypes.c_void_p(x)


def test_cubemap_abi_rejects_bad_shapes(L):
    from dirt_b200 import _lib
    buf = _p(4096)   # never dereferenced: every call below fails validation first
    fwd = lambda TB, S, C, B, N, mode=0: L.dirt_cubemap_sample(buf, buf, buf, buf, TB, S, C, B, N, mode, None)
    bwd = lambda TB, S, C, B, N, mode=0: L.dirt_cubemap_sample_backward(buf, buf, buf, buf, buf, TB, S, C, B, N, mode, 0,
                                                                        buf, 1 << 40, None)
    for call in (fwd, bwd):
        assert call(1, 0, 3, 1, 8) == _lib.ERR_BAD_SHAPE              # S = 0
        assert call(1, (1 << 14) + 1, 3, 1, 8) == _lib.ERR_BAD_SHAPE  # S past 2^14
        assert call(1, 4, 0, 1, 8) == _lib.ERR_BAD_SHAPE              # C = 0
        assert call(1, 4, 3, -1, 8) == _lib.ERR_BAD_SHAPE             # B < 0
        assert call(1, 4, 3, 1, -1) == _lib.ERR_BAD_SHAPE             # N < 0
        assert call(2, 4, 3, 3, 8) == _lib.ERR_BAD_SHAPE              # TB neither 1 nor B
        assert call(1, 4, 3, 1, 8, mode=2) == _lib.ERR_BAD_SHAPE      # unknown mode
        assert call(1, 4, 3, 1 << 30, 1 << 40) == _lib.ERR_BAD_SHAPE  # lookup offsets past 2^62
        assert L.dirt_last_launch_count() == 0
    # the sorted path's 32-bit limits, only under the deterministic flag and only for grad_cubemap
    det = lambda gc, B, N: L.dirt_cubemap_sample_backward(buf, buf, buf, gc, buf, 1, 4, 3, B, N, 0, 1, buf, 1 << 40, None)
    assert det(buf, 1, 1 << 31) == _lib.ERR_BAD_SHAPE
    assert L.dirt_cubemap_sample_backward_bytes(1, 4, 3, 1, 1 << 31, 0, 1) == 0
    assert L.dirt_cubemap_sample_backward_bytes(1, 4, 3, 1, 1 << 31, 0, 0) > 0
    assert L.dirt_cubemap_atlas_bytes(1, 0, 3) == 0 and L.dirt_cubemap_atlas_bytes(2, 4, 3) == 4 * 6 * 2 * 36 * 3


def test_cubemap_abi_with_no_lookups_launches_nothing(L):
    null = _p(0)
    assert L.dirt_cubemap_sample(null, null, null, null, 1, 4, 3, 0, 8, 0, None) == 0
    assert L.dirt_cubemap_sample(null, null, null, null, 1, 4, 3, 2, 0, 1, None) == 0
    assert L.dirt_cubemap_sample(null, null, null, null, 0, 4, 3, 0, 8, 0, None) == 0   # per-item maps, empty batch
    assert L.dirt_cubemap_sample_backward(null, null, null, null, null, 1, 4, 3, 0, 8, 0, 1, null, 0, None) == 0
    assert L.dirt_cubemap_sample_backward_bytes(1, 4, 3, 0, 8, 0, 0) == 0
    assert L.dirt_last_launch_count() == 0


def test_cubemap_abi_rejects_null_and_misaligned_pointers(L):
    from dirt_b200 import _lib
    null, ok, odd = _p(0), _p(4096), _p(4098)
    fwd = L.dirt_cubemap_sample
    for k in range(4):
        args = [ok] * 4
        args[k] = null
        assert fwd(*args, 1, 4, 3, 1, 8, 0, None) == _lib.ERR_NULL_POINTER, k
        args[k] = odd
        assert fwd(*args, 1, 4, 3, 1, 8, 0, None) == _lib.ERR_MISALIGNED, k
    bwd = L.dirt_cubemap_sample_backward
    need = int(L.dirt_cubemap_sample_backward_bytes(1, 4, 3, 1, 8, 0, 0))
    assert need > 0
    assert bwd(ok, null, ok, ok, ok, 1, 4, 3, 1, 8, 0, 0, ok, need, None) == _lib.ERR_NULL_POINTER    # directions
    assert bwd(ok, ok, null, ok, ok, 1, 4, 3, 1, 8, 0, 0, ok, need, None) == _lib.ERR_NULL_POINTER    # grad_out
    assert bwd(null, ok, ok, ok, ok, 1, 4, 3, 1, 8, 0, 0, ok, need, None) == _lib.ERR_NULL_POINTER    # bilinear grad_directions reads the atlas
    assert bwd(ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 0, 0, null, need, None) == _lib.ERR_NULL_POINTER    # scratch
    assert bwd(ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 0, 0, _p(4096 + 128), need, None) == _lib.ERR_MISALIGNED
    assert bwd(ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 0, 0, ok, need - 1, None) == _lib.ERR_WORKSPACE_TOO_SMALL
    det_need = int(L.dirt_cubemap_sample_backward_bytes(1, 4, 3, 1, 8, 0, 1))
    assert det_need > need
    assert bwd(ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 0, 1, ok, det_need - 1, None) == _lib.ERR_WORKSPACE_TOO_SMALL
    for k in range(5):
        args = [ok] * 5
        args[k] = odd
        assert bwd(*args, 1, 4, 3, 1, 8, 0, 0, ok, need, None) == _lib.ERR_MISALIGNED, k
    assert L.dirt_last_launch_count() == 0


def test_sample_cubemap_argument_errors():
    import dirt_b200 as dirt
    cube = torch.zeros(6, 4, 4, 3)
    with pytest.raises(ValueError, match='mode'):
        dirt.sample_cubemap(cube, torch.zeros(7, 3), mode='trilinear')
    with pytest.raises(ValueError, match=r'\[6, size, size, channels\]'):
        dirt.sample_cubemap(torch.zeros(4, 4, 3), torch.zeros(7, 3))
    with pytest.raises(ValueError, match=r'\[6, size, size, channels\]'):
        dirt.sample_cubemap(torch.zeros(5, 4, 4, 3), torch.zeros(7, 3))
    with pytest.raises(ValueError, match=r'\[6, size, size, channels\]'):
        dirt.sample_cubemap(torch.zeros(6, 4, 5, 3), torch.zeros(7, 3))
    with pytest.raises(ValueError, match='positive'):
        dirt.sample_cubemap(torch.zeros(6, 0, 0, 3), torch.zeros(7, 3))
    with pytest.raises(ValueError, match=r'shape\[-1\] == 3'):
        dirt.sample_cubemap(cube, torch.zeros(7, 2))
    with pytest.raises(ValueError, match=r'shape\[0\] == cubemap.shape\[0\]'):
        dirt.sample_cubemap(cube[None].expand(2, 6, 4, 4, 3), torch.zeros(3, 7, 3))
    with pytest.raises(ValueError, match='at least 2D'):
        dirt.sample_cubemap(cube[None], torch.zeros(3))
    if not torch.cuda.is_available():
        # no CPU kernel: CPU tensors are an error, never a fallback
        with pytest.raises(RuntimeError, match='CUDA'):
            dirt.sample_cubemap(cube, torch.zeros(7, 3))
