"""CPU: the decision-taking float64 reference of the shadow-map lookup (tests/shadow_reference.py) -- away from fp32
ties it is the float64 restatement `lighting._shadow_visibility`, on test_gpu_shadow.py's tie-free inputs it takes the
float64 decisions, and its deterministic-order part is the summation order test_gpu_shadow.py restates."""
import numpy as np
import pytest
import torch

import shadow_reference as sr
from dirt_b200 import lighting
from test_gpu_shadow import SH, SW, _behind, _case


def _restated(p, M, smap, R, softness, bias, gout):
    t = [torch.tensor(np.asarray(x, np.float32), dtype=torch.float64, requires_grad=True) for x in (p, M, smap)]
    v = lighting._shadow_visibility(*t, R, softness, bias)
    (v * torch.tensor(np.asarray(gout, np.float32), dtype=torch.float64)).sum().backward()
    return v.detach().numpy(), [np.nan_to_num(x.grad.numpy()) for x in t]


def _assert_near(got, want, rtol, what):
    scale = max(np.abs(want).max(), 1e-30)
    assert np.allclose(got, want, rtol=rtol, atol=rtol * scale), (what, np.abs(got - want).max(), scale)


@pytest.mark.parametrize('R', [0, 1, 2, 3])
@pytest.mark.parametrize('softness', [0., 0.05])
@pytest.mark.parametrize('per_item', [True, False])
def test_equals_the_restatement_away_from_ties(R, softness, per_item):
    """Continuous random inputs, keeping the points whose fractions are 1e-5 from 0 and 1 and whose depth differences
    are 1e-4 from 0 at every tap: the fp32 decisions are then the float64 ones, and only the fractions' and d's fp32
    rounding (a few 1e-8) separates the two."""
    g = np.random.default_rng(100 + 10 * R + 2 * per_item + int(softness > 0))
    B, N, sh, sw = 3, 600, 9, 13
    nm = B if per_item else 1
    M = np.tile(np.eye(4), (nm, 1, 1))
    M[:, :3, :3] += g.uniform(-0.2, 0.2, (nm, 3, 3))
    M[:, 2, 3] = g.uniform(0.05, 0.2, nm)
    p = g.uniform(-1.1, 1.1, (B, N, 3))
    smap = np.stack([g.uniform(size=(nm, sh, sw)) < 0.6, g.uniform(-1.2, 1.2, (nm, sh, sw))], -1)
    if not per_item:
        M, smap = M[0], smap[0]
    p, M, smap = (np.asarray(x, np.float32) for x in (p, M, smap))
    pp, MM, mm, _ = sr._flat(p, M, smap)
    look = sr.lookups(pp, MM, sh, sw)
    keep = look['valid'] & (np.minimum(look['fr'], 1 - look['fr']) > 1e-5) & \
        (np.minimum(look['fc'], 1 - look['fc']) > 1e-5)
    for i in range(2 * R + 2):
        for k in range(2 * R + 2):
            d, _ = sr._depth_steps(look, mm, R, i, k, 0.01)
            keep &= np.abs(d) > 1e-4
    n = keep.sum(1).min()
    assert n >= 100
    p = np.stack([p[b][keep[b]][:n] for b in range(B)])
    gout = g.standard_normal((B, n, 1))
    vis, grads = sr.reference(p, M, smap, R, softness, 0.01, gout)
    v64, g64 = _restated(p, M, smap, R, softness, 0.01, gout)
    _assert_near(vis, v64, 1e-6, 'visibility')
    for a, b, name in zip(grads, g64, ('positions', 'matrix', 'map')):
        _assert_near(a, b, 1e-5, name)


@pytest.mark.parametrize('R', [0, 1, 3])
@pytest.mark.parametrize('per_item', [True, False])
def test_takes_the_float64_decisions_on_the_tie_free_cases(R, per_item):
    """On test_gpu_shadow.py's _case inputs: validity, base texels and every tap's step are those of float64."""
    B, N, bias = 3, 700, 0.01
    p, M, smap = _case(B, N, per_item, seed=R * 10 + 2 + per_item, bias=bias)
    p = _behind(p, M, per_item)
    pp, MM, mm, _ = sr._flat(p, M, smap)
    look = sr.lookups(pp, MM, SH, SW)
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
        h = np.einsum('bnk,bkj->bnj', np.concatenate([pp, np.ones_like(pp[..., :1])], -1),
                      np.broadcast_to(MM, (B, 4, 4)))
        ok = np.isfinite(h).all(-1) & (h[..., 3] > 0)
        X, Yd = (h[..., 0] / h[..., 3] + 1) * SW / 2, (1 - h[..., 1] / h[..., 3]) * SH / 2
        ok &= (X >= 0) & (X < SW) & (Yd >= 0) & (Yd < SH)
    assert np.array_equal(look['valid'], ok) and (~ok).sum() == 6 * B
    assert np.array_equal(look['c0'][ok], np.floor(X[ok] - 0.5)) and np.array_equal(look['r0'][ok], np.floor(Yd[ok] - 0.5))
    for i in range(2 * R + 2):
        for k in range(2 * R + 2):
            d32, (mi, r, c) = sr._depth_steps(look, mm, R, i, k, bias)
            d64 = h[..., 2] - mm[mi, r, c, 1] - bias
            assert np.array_equal((d32 > 0)[ok], (d64 > 0)[ok])


def _order_restated(X, Yd, z, smap, gout, R, S_H, S_W):
    """test_gpu_shadow.py's restatement of the deterministic summation order (identity matrix, per-item maps)."""
    B, N = X.shape
    T, inv_k = 2 * R + 2, np.float32(1) / np.float32((2 * R + 1) ** 2)
    terms = {}
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
    return want


@pytest.mark.parametrize('R', [0, 1, 3])
@pytest.mark.parametrize('S_H, S_W', [(8, 16), (1, 4), (4, 2)])
def test_deterministic_order_reproduces_the_restated_order(R, S_H, S_W):
    B, N = 2, 400
    g = np.random.default_rng(60 + R)
    X = g.integers(0, S_W * 64, (B, N)) / 64. + 1 / 128.
    Yd = g.integers(0, S_H * 64, (B, N)) / 64. + 1 / 128.
    z = g.integers(-8, 8, (B, N)) / 16. + 1 / 32.
    p = np.stack([X / (S_W / 2) - 1, 1 - Yd / (S_H / 2), z], -1).astype(np.float32)
    smap = np.stack([(g.uniform(size=(B, S_H, S_W)) < 0.6), g.integers(-8, 8, (B, S_H, S_W)) / 16.], -1)
    smap = smap.astype(np.float32)
    gout = (g.integers(-64, 64, (B, N)) / 32.).astype(np.float32)
    M = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    got = sr.deterministic_map_gradient(p, M, smap, R, 0.01, gout)
    assert np.array_equal(got, _order_restated(X, Yd, z, smap, gout, R, S_H, S_W))


def test_sequential_sums_add_one_value_at_a_time():
    g = np.random.default_rng(5)
    seg = np.sort(np.r_[g.integers(0, 50, 3000), np.full(5000, 60)])
    vals = g.standard_normal(seg.size) * 10. ** g.integers(-8, 8, seg.size)
    ids, sums = sr.sequential_sums(seg, vals)
    assert np.array_equal(ids, np.unique(seg))
    for s, got in zip(ids, sums):
        acc = 0.0
        for v in vals[seg == s]:
            acc += v
        assert got == acc


def test_sort_passes():
    assert sr.sort_passes(3, False, 7, 1) == 1 and sr.sort_passes(3, True, 1, 1) == 1
    assert sr.sort_passes(3, True, 24, 40) == 2 and sr.sort_passes(2, True, 256, 256) == 3
    assert sr.sort_passes(1, False, 4096, 4096) == 4 and sr.sort_passes(17, True, 1024, 1024) == 4


@pytest.mark.parametrize('shape', [(1, 1), (1, 7), (7, 1)])
def test_fraction_derivatives_cancel_where_taps_repeat_a_texel(shape):
    """On a one-row or one-column map every tap of a row (column) reads one texel: the derivative with respect to the
    column (row) fraction is exactly 0, as the kernels form it, not a float64 rounding residue."""
    SH, SW = shape
    g = np.random.default_rng(sum(shape))
    p = np.asarray(np.c_[g.uniform(-1, 1, (500, 2)), g.uniform(-0.5, 0.5, 500)], np.float32)[None]
    smap = np.asarray(np.stack([g.uniform(size=(SH, SW)) < 0.6, g.uniform(-0.5, 0.5, (SH, SW))], -1), np.float32)
    for R in (1, 3):
        _, (gp, _, _) = sr.reference(p, np.eye(4, dtype=np.float32), smap, R, 0., 0.01, np.ones((1, 500, 1)))
        if SW == 1:
            assert (gp[..., 0] == 0).all()
        if SH == 1:
            assert (gp[..., 1] == 0).all()
