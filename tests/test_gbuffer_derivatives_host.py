"""CPU: the float64 specification of the G-buffer derivatives (DESIGN.md §7.7) against central differences of the fp64
interpolation, the argument errors of `derivative_channels`, and the C ABI's argument checks, none of which launches
anything.  `fp64_derivatives` is the truth tests/test_gpu_gbuffer_derivatives.py holds the CUDA kernel to."""
import ctypes

import numpy as np
import pytest
import torch

import kernel_paths as kp
from conftest import rel_close


def fp64_derivatives(vertices, attributes, faces, ids):
    """[H, W, 2, C] float64: d a / dcol and d a / drow at the centres of the pixels `ids` [H,W] marks as covered, a the
    perspective-correct interpolant of one image's attributes [V,C] over the face the pixel shows (vertices [V,4], faces
    [F,3]).  As kernel_paths.fp64_pixels: with M the rows (x, y, w) of the face, lam = M^-T (X, Y, 1) is linear in NDC
    and beta = lam / sum(lam); beta is differentiated analytically, then d X / d col = 2 / W and d Y / d row = -2 / H.
    Uncovered pixels are NaN."""
    H, W = ids.shape
    out = np.full((H, W, 2, attributes.shape[-1]), np.nan)
    rows, cols = np.nonzero(ids >= 0)
    xn = (cols + 0.5) / W * 2.0 - 1.0
    yn = 1.0 - (rows + 0.5) / H * 2.0
    fid = ids[rows, cols]
    for f in np.unique(fid):
        sel = fid == f
        A = np.linalg.inv(vertices[faces[f]].astype(np.float64)[:, [0, 1, 3]].T)   # lam = A @ (X, Y, 1)
        lam = A @ np.stack([xn[sel], yn[sel], np.ones(int(sel.sum()))])          # [3, n]
        s = lam.sum(0)
        a = attributes[faces[f]].astype(np.float64)                               # [3, C]
        for axis, scale in ((0, 2.0 / W), (1, -2.0 / H)):
            dlam = A[:, axis][:, None]                                            # d lam / d X (or Y), constant
            dbeta = (dlam * s - lam * dlam.sum()) / s ** 2                       # [3, n]
            out[rows[sel], cols[sel], axis] = (dbeta.T @ a) * scale
    return out


def _inside(vertices, faces, H, W):
    """Face ids [H,W] of a scene of one face: 0 where the pixel centre lies inside it in float64, else -1."""
    ids = np.zeros((H, W), np.int64)
    beta = kp.fp64_pixels(vertices, np.eye(3)[np.arange(vertices.shape[0]) % 3], faces, ids)
    return np.where((beta >= 0).all(-1), 0, -1)


def _shifted(vertices, dx, dy):
    """The scene moved by (dx, dy) in NDC: its interpolant at a point is the original's at the point minus (dx, dy)."""
    v = vertices.astype(np.float64).copy()
    v[:, 0] += dx * v[:, 3]
    v[:, 1] += dy * v[:, 3]
    return v


def _central_differences(vertices, attributes, faces, ids, h=1e-7):
    # h in NDC: small enough for the curvature near a vertex of clip w 10^-3 and large enough for fp64 rounding
    H, W = ids.shape
    cx = (kp.fp64_pixels(_shifted(vertices, -h, 0), attributes, faces, ids) -
          kp.fp64_pixels(_shifted(vertices, h, 0), attributes, faces, ids)) / (2 * h) * (2.0 / W)
    cy = (kp.fp64_pixels(_shifted(vertices, 0, -h), attributes, faces, ids) -
          kp.fp64_pixels(_shifted(vertices, 0, h), attributes, faces, ids)) / (2 * h) * (-2.0 / H)
    return np.stack([cx, cy], -2)


@pytest.mark.parametrize('ratio', sorted(kp.FP64_W) + sorted(kp.FP64_W_LOGGED))
def test_fp64_derivatives_match_central_differences_on_the_big_triangle(ratio):
    w = {**kp.FP64_W, **kp.FP64_W_LOGGED}[ratio]
    s = kp.big_triangle(48, 64, w, 3)
    v, a, f = s['vertices'][0], s['vertex_colors'][0], s['faces'][0]
    ids = _inside(v, f, 48, 64)
    assert (ids >= 0).mean() > 0.3
    got = fp64_derivatives(v, a, f, ids)
    want = _central_differences(v, a, f, ids)
    cov = ids >= 0
    assert np.isnan(got[~cov]).all()
    ok, worst = rel_close(got[cov], want[cov], rel=1e-6)
    assert ok, worst


def test_fp64_derivatives_match_central_differences_on_a_soup_behind_the_camera(oracle):
    from dirt_b200 import scenes
    s = scenes.random_soup(batch=2, width=40, height=30, n_faces=20, channels=4, seed=3, behind_camera=True)
    ids = oracle.visibility(s['vertices'], s['faces'], 30, 40)[0]
    assert (ids >= 0).mean() > 0.3
    for b in range(2):
        v, a, f = s['vertices'][b], s['vertex_colors'][b], s['faces'][b]
        got = fp64_derivatives(v, a, f, ids[b])
        want = _central_differences(v, a, f, ids[b])
        cov = ids[b] >= 0
        ok, worst = rel_close(got[cov], want[cov], rel=1e-6)
        assert ok, (b, worst)


def test_fp64_derivatives_of_an_affine_face_are_its_screen_space_gradient():
    # w = 1: a is affine in pixel coordinates, a = a0 + (a1 - a0) * t1 + (a2 - a0) * t2 over the screen triangle
    H, W = 20, 30
    p = np.array([[3.0, 2.0], [27.0, 5.0], [8.0, 18.0]])
    v = kp.clip_vertices(p[:, 0], p[:, 1], 0.0, 1.0, H, W)
    a = np.array([[0.0, 1.0], [2.0, -1.0], [5.0, 0.5]])
    ids = np.zeros((H, W), np.int64)
    got = fp64_derivatives(v, a, np.array([[0, 1, 2]]), ids)
    grad = np.linalg.solve(np.stack([p[1] - p[0], p[2] - p[0]]), np.stack([a[1] - a[0], a[2] - a[0]]))   # [2 (x, y), C]
    assert np.allclose(got, grad[None, None], rtol=1e-6, atol=1e-9)   # the clip vertices are float32


@pytest.mark.parametrize('channels', [[], [2, 1], [0, 2], [3], [-1, 0], 'ab', [0.5], range(2, 2), 7])
def test_malformed_derivative_channels_raise_before_the_cuda_check(channels):
    import dirt_b200 as dirt
    bg, v, a, f = torch.zeros(4, 5, 3), torch.zeros(2, 4), torch.zeros(2, 3), torch.zeros(1, 3, dtype=torch.int32)
    with pytest.raises(ValueError, match='derivative_channels'):
        dirt.rasterise_deferred(bg, v, a, f, lambda g, **kw: g, derivative_channels=channels)
    with pytest.raises(ValueError, match='derivative_channels'):
        dirt.rasterise_batch_deferred(bg[None], v[None], a[None], f[None], lambda g, **kw: g, derivative_channels=channels)


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _p(x):
    return ctypes.c_void_p(x)


def _call(L, B=2, H=8, W=8, C=4, V=6, F=2, first=1, count=2, holds=1, ws_bytes=None, **ptrs):
    p = dict(vertices=4096, faces=4096, attributes=4096, face_ids=4096, derivatives=4096, workspace=4096)
    p.update(ptrs)
    if ws_bytes is None:
        ws_bytes = L.dirt_workspace_bytes_min(B, H, W, C, V, F) if B >= 0 and H > 0 and W > 0 and C > 0 else 0
    return L.dirt_rasterise_derivatives(_p(p['vertices']), _p(p['faces']), _p(p['attributes']), _p(p['face_ids']),
                                        _p(p['derivatives']), B, H, W, C, V, F, first, count, holds, _p(p['workspace']),
                                        ws_bytes, None)


def test_argument_checks_return_their_codes_before_launching(L):
    from dirt_b200 import _lib
    cases = [
        (dict(H=0), _lib.ERR_BAD_SHAPE), (dict(C=0), _lib.ERR_BAD_SHAPE), (dict(B=-1), _lib.ERR_BAD_SHAPE),
        (dict(first=-1), _lib.ERR_BAD_SHAPE), (dict(count=0), _lib.ERR_BAD_SHAPE), (dict(first=4, count=1), _lib.ERR_BAD_SHAPE),
        (dict(first=3, count=2), _lib.ERR_BAD_SHAPE), (dict(first=0, count=5), _lib.ERR_BAD_SHAPE),
        (dict(B=0, first=4), _lib.ERR_BAD_SHAPE),
        (dict(face_ids=0), _lib.ERR_NULL_POINTER), (dict(derivatives=0), _lib.ERR_NULL_POINTER),
        (dict(vertices=0), _lib.ERR_NULL_POINTER), (dict(attributes=0), _lib.ERR_NULL_POINTER),
        (dict(faces=0), _lib.ERR_NULL_POINTER), (dict(workspace=0), _lib.ERR_NULL_POINTER),
        (dict(vertices=4104), _lib.ERR_MISALIGNED), (dict(attributes=4098), _lib.ERR_MISALIGNED),
        (dict(faces=4098), _lib.ERR_MISALIGNED), (dict(face_ids=4098), _lib.ERR_MISALIGNED),
        (dict(derivatives=4098), _lib.ERR_MISALIGNED), (dict(workspace=4224), _lib.ERR_MISALIGNED),
        (dict(ws_bytes=L.dirt_workspace_bytes_min(2, 8, 8, 4, 6, 2) - 1), _lib.ERR_WORKSPACE_TOO_SMALL),
    ]
    for kw, rc in cases:
        assert _call(L, **kw) == rc, kw
        assert L.dirt_last_launch_count() == 0
    # shape errors come first, then null pointers, alignment and the workspace size
    assert _call(L, count=0, face_ids=0, vertices=4104) == _lib.ERR_BAD_SHAPE
    assert _call(L, face_ids=0, vertices=4104, ws_bytes=1) == _lib.ERR_NULL_POINTER
    assert _call(L, vertices=4104, ws_bytes=1) == _lib.ERR_MISALIGNED
    # B = 0: nothing to do, nothing needed
    assert _call(L, B=0, vertices=0, faces=0, attributes=0, face_ids=0, derivatives=0, workspace=0) == 0
    assert L.dirt_last_launch_count() == 0

