"""CPU: the scenes of tests/exact_sums.py meet the exactness condition, land where they claim, and their expected sums
are the restatements' and the oracle's own gradients.  tests/test_gpu_exact_sums.py compares the kernels with them."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import exact_sums as es

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def ex():
    spec = importlib.util.spec_from_file_location('textured_example', os.path.join(ROOT, 'examples', 'textured.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _autograd_texture(ex, tex, idx, gout, mode):
    """float64 autograd of the restatement per item: (grad_texture [TB, H, W, C], grad_indices [B, N, 2])."""
    TB = tex.shape[0]
    gts, gis = torch.zeros(tex.shape, dtype=torch.float64), []
    for b in range(idx.shape[0]):
        t = tex[b if TB > 1 else 0].double().requires_grad_(True)
        i = idx[b].double().requires_grad_(mode == 'bilinear')
        (ex.sample_texture(t, i, mode=mode) * gout[b].double()).sum().backward()
        gts[b if TB > 1 else 0] += t.grad
        gis.append(i.grad if i.grad is not None else torch.zeros_like(i))
    return gts, torch.stack(gis)


def test_check_exact_refuses_what_it_should():
    ok = torch.tensor([0.25, -0.5, 1.0], dtype=torch.float64)
    sums, counts = es.check_exact(ok, torch.tensor([0, 0, 1]), 3, 2)
    assert sums.tolist() == [-0.25, 1.0, 0.0] and counts.tolist() == [2, 1, 0]
    with pytest.raises(AssertionError, match='multiple'):
        es.check_exact(torch.tensor([0.125], dtype=torch.float64), torch.tensor([0]), 1, 2)
    with pytest.raises(AssertionError, match='2\\^24'):
        es.check_exact(torch.full((5,), 2.0 ** 21, dtype=torch.float64), torch.zeros(5, dtype=torch.long), 1, 1)


@pytest.mark.parametrize('per_item', [False, True])
@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [1, 2, 3, 4, 5, 8])
def test_texture_scene_is_exact_and_matches_the_restatement(ex, C, mode, per_item):
    tex, idx, gout = es.texture_scene(3 if per_item else 1, 19, 13, C, 3, 3000, 10 + C)
    frac = idx - idx.floor()
    assert ((frac == 0) | (frac == 0.25) | (frac == 0.5) | (frac == 0.75)).all()
    gt, nt, gi, ni = es.texture_expected(tex, idx, gout, mode)
    rt, ri = _autograd_texture(ex, tex, idx, gout, mode)
    assert not es.first_difference(gt, rt, nt)
    assert not es.first_difference(gi, ri, ni)
    assert int(nt.max()) > 20


@pytest.mark.parametrize('C', [1, 4])
def test_texture_contention_scene_is_exact(ex, C):
    """The 2 x 2 texture under 2^20 lookups: about 2^20 terms per texel, and still inside the condition."""
    tex, idx, gout = es.texture_scene(1, 2, 2, C, 1, 1 << 20, 40 + C)
    gt, nt, _, _ = es.texture_expected(tex, idx, gout, 'bilinear')
    assert int(nt.min()) > 500000
    rt, _ = _autograd_texture(ex, tex, idx, gout, 'bilinear')
    assert not es.first_difference(gt, rt, nt)


def test_agg_rule_restated():
    assert es.agg_pull([1] * 32) is None
    assert es.agg_pull([32]) is False
    assert es.agg_pull([6] + [1] * 26) is True and es.agg_pull([7] + [1] * 25) is False
    assert es.agg_pull([11, 2] + [1] * 19) is True and es.agg_pull([12, 2] + [1] * 18) is False
    assert es.agg_pull([2] * 16) is True and es.agg_pull([16, 16]) is False


def _intended(pattern):
    sizes = [s for s in es.WARP_PATTERNS[pattern] if isinstance(s, int)]
    return es.agg_pull(sizes + [1] * (32 - sum(sizes)))


@pytest.mark.parametrize('pattern', sorted(es.WARP_PATTERNS))
def test_warp_patterns_fall_on_the_intended_side(ex, pattern):
    """Every corner of every warp forms exactly the pattern's groups, so it takes the side agg_plan's rule gives the
    pattern; the straddling pairs (six / seven, eleven_pair / twelve_pair) sit on either side."""
    H, W = 16, 20
    idx = es.warp_pattern_indices(pattern, 24, H, W, 7)
    want = _intended(pattern)
    assert all(side == want for per in es.warp_sides(idx, H, W) for side in per)
    # and the scene is exact, as the restatement sees it
    tex = es.dyadic((1, H, W, 3), es.TEXELS, 8)
    gout = es.dyadic((1, idx.shape[0], 3), es.GRADS, 9)
    gt, nt, gi, ni = es.texture_expected(tex, idx[None], gout, 'bilinear')
    # the restatement has no rule for a NaN index (the kernel reads nothing there): give it the finite lookups alone
    ok = torch.isfinite(idx).all(-1)
    rt, ri = _autograd_texture(ex, tex, idx[None, ok], gout[:, ok], 'bilinear')
    assert not es.first_difference(gt, rt, nt) and not es.first_difference(gi[:, ok], ri, ni[:, ok])
    assert not gi[:, ~ok].any()


def test_straddling_patterns_take_both_sides():
    assert [_intended(p) for p in ('six', 'seven', 'eleven_pair', 'twelve_pair')] == [True, False, True, False]
    assert _intended('mixed') is True and _intended('one32') is False and _intended('halves') is False


def _autograd_diffuse(x, g):
    from dirt_b200 import lighting
    leaves = {k: v.double().requires_grad_(True) for k, v in x.items()}
    (lighting._diffuse_directional(leaves['n'], leaves['k'], leaves['L'], leaves['lc']) * g.double()).sum().backward()
    return {k: v.grad for k, v in leaves.items()}


@pytest.mark.parametrize('per_item', [False, True])
@pytest.mark.parametrize('lead,V,C', [((4,), 1000, 3), ((2, 3), 333, 1), ((5,), 257, 4)])
def test_diffuse_scene_is_exact_and_matches_the_restatement(lead, V, C, per_item):
    x, g = es.diffuse_scene(lead, V, C, per_item, 20 + C)
    want = es.diffuse_expected(x, g)
    got = _autograd_diffuse(x, g)
    for k in ('L', 'lc'):
        assert not es.first_difference(got[k], want[k][0], want[k][1]), k


@pytest.mark.parametrize('per_item', [False, True])
def test_diffuse_cfg3_sized_scene_is_exact(per_item):
    """The GPU test's 64 x 512^2 scene itself, its terms formed eight items at a time."""
    x, g = es.diffuse_scene((64,), 512 * 512, 3, per_item, 200, sparse=1 if per_item else 64)
    want = es.diffuse_expected(x, g, items=8)
    assert int(want['L'][1].sum()) > (1 << 17)


def test_chunked_sums_equal_whole_ones():
    tex, idx, gout = es.texture_scene(2, 19, 13, 3, 2, 3000, 60)
    whole = es.texture_expected(tex, idx, gout, 'bilinear')
    for a, b in zip(whole, es.texture_expected(tex, idx, gout, 'bilinear', chunk=700)):
        assert torch.equal(a.double(), b.double())
    x, g = es.diffuse_scene((6,), 300, 3, True, 61)
    assert all(torch.equal(es.diffuse_expected(x, g)[k][0], es.diffuse_expected(x, g, items=4)[k][0]) for k in ('L', 'lc'))


@pytest.mark.parametrize('kind', ['large', 'tiny'])
@pytest.mark.parametrize('C', [1, 3, 4])
def test_raster_scene_is_exact_and_matches_the_oracle(oracle, kind, C):
    s, gp, m = es.raster_scene(kind, C, 2, 50 + C)
    B, H, W, _ = gp.shape
    want, counts, ids, gbuf = es.raster_expected(s, gp, m, oracle)
    covered = ids >= 0
    bary = gbuf[..., :3][covered].astype(np.float64) * 2.0 ** m
    assert (bary == np.round(bary)).all() and (gbuf[..., 3][covered] == 1).all()
    if kind == 'large':
        assert covered.all()
        assert np.bincount(ids[0].reshape(-1)).min() >= 10000
    else:
        # every 8 x 8 backward tile with its one-pixel ring sees more faces than either face table's 24 / 32 slots
        for ty in range(0, H, 8):
            for tx in range(0, W, 8):
                ring = ids[0, max(ty - 1, 0):ty + 9, max(tx - 1, 0):tx + 9]
                assert len(np.unique(ring)) > 32 or (ty in (0, H - 8) or tx in (0, W - 8))
    pixels = oracle.forward(**s)
    _, _, gc = oracle.backward(s['vertices'], s['faces'], pixels, gp)
    assert not es.first_difference(torch.from_numpy(gc), want, counts)
    shared, shared_counts, _, _ = es.raster_expected(s, gp, m, oracle, shared=True)
    assert not es.first_difference(torch.from_numpy(gc.astype(np.float64).sum(0)), shared, shared_counts)


def _multiples(x, m):
    y = np.asarray(x, np.float64) * 2.0 ** m
    return bool((y == np.round(y)).all())


@pytest.mark.parametrize('per_item', [False, True])
def test_trilinear_scene_reads_one_level_at_dyadic_fractions(per_item):
    """Footprints of 2^l texels give lambda = l exactly (no blend); level l's index (i + 1/2) 2^-l - 1/2 has a fraction
    on a 2^-(2+l) grid; the restatement's sums then meet the condition."""
    import texture_mip_restatement as mip
    tex, idx, der, gout = es.trilinear_scene(3 if per_item else 1, 64, 32, 3, 3, 3000, 70)
    l, f = mip.lod(der, mip.level_count(64, 32))
    assert (f == 0).all() and set(l.unique().tolist()) == {0., 1., 2.}
    for k in range(3):
        sel = (l[..., 0] == k)
        li = mip.level_index(idx[sel], k)
        assert _multiples((li - li.floor()).numpy(), 2 + k)
    es.trilinear_expected(tex, idx, der, gout)


@pytest.mark.parametrize('mode', ['bilinear', 'nearest', 'trilinear'])
@pytest.mark.parametrize('per_item', [False, True])
def test_cube_scene_has_dyadic_padded_coordinates(mode, per_item):
    """Every lookup's padded coordinate s (S >> k) + 1/2 is on a 2^-(2+k) grid at levels 0..2, the lods on a 1/4 grid,
    some lookups reach the border and corner texels, and the restatement's sums meet the condition."""
    import cubemap_restatement as cm
    cube, d, lod, gout = es.cube_scene(2, 3, 4000, per_item, 80)
    _, s, t, valid = cm.face_coords(d)
    assert valid.all()
    for k in range(3):
        for u in (s, t):
            assert _multiples((u * (es.CUBE_S >> k) + 0.5).numpy(), 2 + k)
    assert _multiples(lod.numpy(), 2) and float(lod.max()) <= 2
    p = s * es.CUBE_S + 0.5
    assert bool((p < 1).any()) and bool((p > es.CUBE_S).any())
    es.cube_expected(cube, d, lod, gout, mode)


@pytest.mark.parametrize('per_item', [False, True])
@pytest.mark.parametrize('name', es.SHADOW_CASES)
def test_shadow_scene_is_exact_at_radius_zero(name, per_item):
    import shadow_reference as sr
    p, M, smap, gout = es.shadow_case(name, per_item)
    P, Mf, m, _ = sr._flat(p, M, smap)
    look = sr.lookups(P, Mf, m.shape[1], m.shape[2])
    assert look['valid'].all() and _multiples(look['fr'], 2) and _multiples(look['fc'], 2)
    want, counts = es.shadow_expected(p, M, smap, 0, 0.01, gout)
    ref = sr.reference(p, M, smap, 0, 0., 0.01, gout, (False, False, True))[1][2]
    assert not es.first_difference(torch.as_tensor(np.asarray(ref)), want, counts)


def test_shadow_radius_one_cannot_be_summed_exactly():
    """Past R = 0 every term carries 1 / (2R + 1)^2 rounded to fp32 (24 significant bits for 1/9), times a dyadic
    weight: no grid 2^-m with m small enough for the condition holds them, so R >= 1 stays under the 1e-4 bar."""
    p, M, smap, gout = es.shadow_case('map16', False)
    terms, index, size = es.shadow_map_terms(p, M, smap, 1, 0.01, gout)
    with pytest.raises(AssertionError):
        es.check_exact(terms, index, size, 24)
