"""CPU: the split-sum GGX restatement (tests/cubemap_ggx_restatement.py) -- its texel table, prefilter, support and
BRDF table -- and the argument errors of sample_cubemap(..., 'ggx') and of the new C ABI entries."""
import ctypes
import math

import numpy as np
import pytest
import torch

import cubemap_ggx_restatement as ibl
import cubemap_mip_restatement as cmm


def _cube(S, C=3, seed=0):
    return torch.from_numpy(np.random.default_rng(seed).random((6, S, S, C)))


@pytest.mark.parametrize('S', [1, 2, 3, 8, 64])
def test_solid_angles_sum_to_the_sphere(S):
    dirs, omega = ibl.texel_table(S)
    assert abs(omega.astype(np.float64).sum() - 4 * math.pi) < 4 * math.pi * 1e-6
    assert np.all(omega > 0)
    assert np.abs(np.linalg.norm(dirs.astype(np.float64), axis=-1) - 1).max() < 1e-6


def test_fmaf_is_the_correctly_rounded_fused_multiply_add():
    rng = np.random.default_rng(0)
    a, b, c = (rng.standard_normal(20000).astype(np.float32) for _ in range(3))
    got = ibl.fmaf(a, b, c)
    exact = [float(np.float64(x) * np.float64(y)) for x, y in zip(a, b)]   # exact products
    from fractions import Fraction
    for k in range(0, 20000, 97):
        want = Fraction(exact[k]) + Fraction(float(c[k]))
        lo = np.float32(float(want))
        # got is the nearest fp32 to the exact value
        cand = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cand, key=lambda x: abs(Fraction(float(x)) - want))
        assert got[k] == best, k
    # a float64 tie that the remainder settles: 1 + 2^-24 + 2^-60 rounds up in one step
    x = np.float32(1 + 2 ** -12)
    assert ibl.fmaf(x, x, np.float32(-2 ** -24)) == np.float32(1 + 2 ** -11)


@pytest.mark.parametrize('S', [2, 8, 16, 32])
def test_constant_map_prefilters_to_itself_and_level_zero_is_the_map(S):
    cube = torch.full((6, S, S, 2), 0.7, dtype=torch.float64)
    cube[..., 1] = -3.
    levels = ibl.prefiltered_levels(cube)
    assert len(levels) == ibl.level_count(S)
    assert levels[0] is cube
    for k, P in enumerate(levels[1:], 1):
        assert P.shape == (6, S >> k, S >> k, 2)
        assert torch.allclose(P, cube[:, :S >> k, :S >> k], rtol=0, atol=1e-12), k


def test_source_levels_and_lobes():
    assert [ibl.source_cap(S) for S in (2, 8, 16, 32, 64, 1024)] == [0, 0, 0, 1, 2, 6]
    L = ibl.level_count(64)
    for k in range(1, L):
        a2, a2f, ck = ibl.lobe(k, L)
        assert a2f == np.float32(a2) and 0 <= ck < 1
        # the cut keeps D >= 1e-3 of the peak: D(c_k) / D(1) = 1e-3 where c_k > 0
        if ck > 0:
            kk = a2 + (1 - float(ck)) * (1 - a2) / 2
            assert abs((a2 * a2) / (kk * kk) - 1e-3) < 1e-6
    assert ibl.lobe(L - 1, L)[2] == 0   # roughness 1: the whole hemisphere


@pytest.mark.parametrize('S', [4, 16])
def test_support_is_symmetric(S):
    dirs, _ = ibl.texel_table(S)
    d = dirs.reshape(-1, 3)
    L = ibl.level_count(S)
    for k in range(1, L):
        ck = ibl.lobe(k, L)[2]
        c, keep = ibl.support(d, d, ck)
        assert np.array_equal(c, c.T) and np.array_equal(keep, keep.T)
        assert keep.diagonal().all()


def test_lobe_mass_left_out_is_small():
    """The share of each level's full-hemisphere weight that the c_k cut leaves out, at S = 64 (reported in DESIGN)."""
    S = 64
    L = ibl.level_count(S)
    worst = 0.
    for k in range(1, L):
        s = min(k, ibl.source_cap(S))
        a2 = ibl.lobe(k, L)[0]
        rd, _ = ibl.texel_table(S >> k)
        ld, lw = ibl.texel_table(S >> s)
        c = ibl.pair_cos(rd.reshape(-1, 3)[::7], ld.reshape(-1, 3)).astype(np.float64)
        kk = a2 + (1 - c) * (1 - a2) / 2
        w = np.where(c > 0, a2 / (math.pi * kk * kk) * c * lw.reshape(-1), 0.)
        cut = np.where(c >= ibl.lobe(k, L)[2], w, 0.)
        worst = max(worst, float((1 - cut.sum(1) / w.sum(1)).max()))
    print('worst lobe mass left out: %.3g' % worst)
    assert worst < 0.03   # GGX has a long tail: 2.6% at S = 64


def _dense_split_sum(n_dot_v, roughness, nt=2000, nphi=3000):
    """F0 * A + B for F0 = 0 and 1 by a dense midpoint quadrature over light directions of lighting._specular_ggx / pi."""
    from dirt_b200 import lighting
    th = (torch.arange(nt, dtype=torch.float64) + 0.5) * (math.pi / 2 / nt)
    ph = (torch.arange(nphi, dtype=torch.float64) + 0.5) * (2 * math.pi / nphi)
    T, P = torch.meshgrid(th, ph, indexing='ij')
    l = torch.stack([T.sin() * P.cos(), T.sin() * P.sin(), T.cos()], -1).reshape(-1, 1, 3)
    dw = (T.sin() * (math.pi / 2 / nt) * (2 * math.pi / nphi)).reshape(-1)
    n = l.new_tensor([0., 0., 1.]).expand_as(l)
    v = l.new_tensor([math.sqrt(1 - n_dot_v ** 2), 0., n_dot_v])
    out = []
    for f0 in (0., 1.):
        spec = lighting._specular_ggx(torch.zeros_like(l), n, l.new_full((l.shape[0], 1, 1), roughness),
                                      l.new_full((l.shape[0], 1, 1), f0), -l[:, 0], l.new_ones(l.shape[0], 1),
                                      v.expand(l.shape[0], 3), False, False)
        out.append(float((spec.reshape(-1) / math.pi * dw).sum()))
    return out   # [B, A + B]


def test_brdf_table_matches_the_integral_of_specular_ggx():
    N = ibl.BRDF_N
    worst = 0.
    for i in (6, 60, 127):
        for j in (25, 127):
            nv, r = (i + 0.5) / N, (j + 0.5) / N
            A, B = ibl.brdf_node(nv, r)
            b, ab = _dense_split_sum(nv, r)
            worst = max(worst, abs(B - b), abs(A + B - ab))
    print('worst |restatement - dense quadrature|: %.3g' % worst)
    assert worst < 1e-3


def test_sample_cubemap_ggx_argument_errors():
    import dirt_b200 as dirt
    cube = torch.zeros(6, 4, 4, 3)
    with pytest.raises(ValueError, match='needs roughness'):
        dirt.sample_cubemap(cube, torch.zeros(7, 3), mode='ggx')
    with pytest.raises(ValueError, match='only used by'):
        dirt.sample_cubemap(cube, torch.zeros(7, 3), mode='ggx', lod=1., roughness=0.5)
    for mode in ('bilinear', 'nearest', 'trilinear'):
        with pytest.raises(ValueError, match='only used by'):
            dirt.sample_cubemap(cube, torch.zeros(7, 3), mode=mode, lod=1. if mode == 'trilinear' else None,
                                roughness=0.5)
    with pytest.raises(ValueError, match='even'):
        dirt.sample_cubemap(torch.zeros(6, 5, 5, 3), torch.zeros(7, 3), mode='ggx', roughness=0.5)
    with pytest.raises(ValueError, match='broadcastable'):
        dirt.sample_cubemap(cube, torch.zeros(7, 3), mode='ggx', roughness=torch.zeros(5))


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _p(x):
    return ctypes.c_void_p(x)


def test_abi_rejects_bad_shapes_and_launches_nothing(L):
    from dirt_b200 import _lib
    buf = _p(4096)
    fwd = lambda TB, S, C, B, N: L.dirt_cubemap_sample_ggx(buf, buf, buf, buf, buf, TB, S, C, B, N, None)
    bwd = lambda TB, S, C, B, N: L.dirt_cubemap_sample_ggx_backward(buf, buf, buf, buf, buf, buf, buf, TB, S, C, B, N, 0,
                                                                    buf, 1 << 40, None)
    for call in (fwd, bwd):
        assert call(1, 0, 3, 1, 8) == _lib.ERR_BAD_SHAPE
        assert call(1, (1 << 14) + 1, 3, 1, 8) == _lib.ERR_BAD_SHAPE
        assert call(1, 4, 0, 1, 8) == _lib.ERR_BAD_SHAPE
        assert call(2, 4, 3, 3, 8) == _lib.ERR_BAD_SHAPE
        assert L.dirt_last_launch_count() == 0
    assert L.dirt_cubemap_ggx_prefilter(buf, buf, 1, 0, 3, None) == _lib.ERR_BAD_SHAPE
    assert L.dirt_cubemap_ggx_prefilter(buf, buf, -1, 4, 3, None) == _lib.ERR_BAD_SHAPE
    assert L.dirt_ggx_brdf_table(buf, -1, None) == _lib.ERR_BAD_SHAPE
    assert L.dirt_ggx_brdf_table(buf, 5000, None) == _lib.ERR_BAD_SHAPE
    assert L.dirt_last_launch_count() == 0
    null = _p(0)
    assert L.dirt_cubemap_sample_ggx(null, null, null, null, null, 1, 4, 3, 0, 8, None) == 0
    assert L.dirt_cubemap_sample_ggx_backward(null, null, null, null, null, null, null, 1, 4, 3, 0, 8, 1, null, 0,
                                              None) == 0
    assert L.dirt_cubemap_ggx_prefilter(null, null, 0, 4, 3, None) == 0
    assert L.dirt_ggx_brdf_table(null, 0, None) == 0
    assert L.dirt_last_launch_count() == 0


def test_abi_sizes_are_functions_of_the_shapes(L):
    nbytes = L.dirt_cubemap_ggx_atlas_bytes
    assert nbytes(1, 0, 3) == 0 and nbytes(-1, 4, 3) == 0
    for TB, S, C in ((1, 4, 3), (2, 8, 1), (3, 16, 5)):
        lv = ibl.level_count(S)
        mip = int(L.dirt_cubemap_mip_atlas_bytes(TB, S, C)) // 4
        pyr = sum((S >> k) ** 2 for k in range(1, lv))
        levels, weights = 6 * TB * pyr * C, 6 * pyr
        table = 4 * 6 * sum((S >> k) ** 2 for k in range(lv))
        cones = 4 * 6 * sum(((S >> k) + 15) // 16 * (((S >> k) + 15) // 16) for k in range(lv))
        assert nbytes(TB, S, C) == 4 * ((mip + levels + weights + 3) // 4 * 4 + table + cones), (TB, S, C)
    b = L.dirt_cubemap_sample_ggx_backward_bytes
    assert b(1, 4, 3, 1, 8, 0) > int(L.dirt_cubemap_sample_trilinear_backward_bytes(1, 4, 3, 1, 8, 0))
    assert b(1, 4, 3, 1, 0, 0) == 0 and b(1, 4, 3, 1, 1 << 31, 1) == 0


def test_abi_rejects_null_and_misaligned_pointers(L):
    from dirt_b200 import _lib
    null, ok, odd, odd8 = _p(0), _p(4096), _p(4098), _p(4104)
    fwd = L.dirt_cubemap_sample_ggx
    for k in range(5):
        args = [ok] * 5
        args[k] = null
        assert fwd(*args, 1, 4, 3, 1, 8, None) == _lib.ERR_NULL_POINTER, k
        args[k] = odd
        assert fwd(*args, 1, 4, 3, 1, 8, None) == _lib.ERR_MISALIGNED, k
    # the atlas holds float4 rows
    assert fwd(ok, ok, ok, odd8, ok, 1, 4, 3, 1, 8, None) == _lib.ERR_MISALIGNED
    assert L.dirt_cubemap_ggx_prefilter(null, ok, 1, 4, 3, None) == _lib.ERR_NULL_POINTER
    assert L.dirt_cubemap_ggx_prefilter(ok, null, 1, 4, 3, None) == _lib.ERR_NULL_POINTER
    assert L.dirt_cubemap_ggx_prefilter(ok, odd8, 1, 4, 3, None) == _lib.ERR_MISALIGNED
    assert L.dirt_cubemap_ggx_prefilter(odd, ok, 1, 4, 3, None) == _lib.ERR_MISALIGNED
    assert L.dirt_ggx_brdf_table(null, 8, None) == _lib.ERR_NULL_POINTER
    assert L.dirt_ggx_brdf_table(odd, 8, None) == _lib.ERR_MISALIGNED
    bwd = L.dirt_cubemap_sample_ggx_backward
    need = int(L.dirt_cubemap_sample_ggx_backward_bytes(1, 4, 3, 1, 8, 0))
    for k in (1, 2, 3):   # directions, lod, grad_out
        args = [ok] * 7
        args[k] = null
        assert bwd(*args, 1, 4, 3, 1, 8, 0, ok, need, None) == _lib.ERR_NULL_POINTER, k
    # every gradient reads the atlas (grad_cubemap its normalisers and texel table)
    assert bwd(null, ok, ok, ok, ok, null, null, 1, 4, 3, 1, 8, 0, ok, need, None) == _lib.ERR_NULL_POINTER
    assert bwd(ok, ok, ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 0, null, need, None) == _lib.ERR_NULL_POINTER
    assert bwd(ok, ok, ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 0, _p(4096 + 128), need, None) == _lib.ERR_MISALIGNED
    assert bwd(ok, ok, ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 0, ok, need - 1, None) == _lib.ERR_WORKSPACE_TOO_SMALL
    det_need = int(L.dirt_cubemap_sample_ggx_backward_bytes(1, 4, 3, 1, 8, 1))
    assert bwd(ok, ok, ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 1, ok, det_need - 1, None) == _lib.ERR_WORKSPACE_TOO_SMALL
    assert bwd(odd8, ok, ok, ok, ok, ok, ok, 1, 4, 3, 1, 8, 0, ok, need, None) == _lib.ERR_MISALIGNED
    for k in range(1, 7):
        args = [ok] * 7
        args[k] = odd
        assert bwd(*args, 1, 4, 3, 1, 8, 0, ok, need, None) == _lib.ERR_MISALIGNED, k
    assert L.dirt_last_launch_count() == 0


def test_every_new_symbol_is_exported(L):
    from dirt_b200 import _lib
    for name in ('dirt_cubemap_ggx_atlas_bytes', 'dirt_cubemap_ggx_prefilter', 'dirt_cubemap_sample_ggx',
                 'dirt_cubemap_sample_ggx_backward_bytes', 'dirt_cubemap_sample_ggx_backward', 'dirt_ggx_brdf_table'):
        assert name in _lib.EXPORTED_SYMBOLS
        assert getattr(L, name).restype is not None


def test_sh_projection_approaches_known_coefficients():
    """A map whose radiance is sum_k c_k Y_k at the texel centres projects back towards c as S grows."""
    from dirt_b200 import lighting
    c = torch.from_numpy(np.random.default_rng(3).standard_normal((9, 2)))
    errors = []
    for S in (4, 16, 64):
        dirs, _ = ibl.texel_table(S)
        cube = (lighting._sh_basis(torch.from_numpy(dirs.astype(np.float64))) @ c).reshape(6, S, S, 2)
        errors.append(float((ibl.sh_project(cube) - c).abs().max()))
    print('max |projection - coefficients| at S = 4, 16, 64:', errors)
    assert errors[0] > errors[1] > errors[2] and errors[2] < 1e-3


def test_sh_projection_abi_errors(L):
    from dirt_b200 import _lib
    null, ok, odd = _p(0), _p(4096), _p(4098)
    need = int(L.dirt_cubemap_sh_project_bytes(1, 8, 3))
    assert need > 0 and L.dirt_cubemap_sh_project_bytes(1, 0, 3) == 0 and L.dirt_cubemap_sh_project_bytes(0, 8, 3) == 0
    for fn in (L.dirt_cubemap_sh_project, L.dirt_cubemap_sh_project_backward):
        assert fn(ok, ok, ok, need, 1, 0, 3, None) == _lib.ERR_BAD_SHAPE
        assert fn(ok, ok, ok, need, 1, 8, 0, None) == _lib.ERR_BAD_SHAPE
        assert fn(null, null, null, 0, 0, 8, 3, None) == 0
        for k in range(3):
            args = [ok] * 3
            args[k] = null
            assert fn(*args, need, 1, 8, 3, None) == _lib.ERR_NULL_POINTER, k
        assert fn(odd, ok, ok, need, 1, 8, 3, None) == _lib.ERR_MISALIGNED
        assert fn(ok, ok, _p(4096 + 128), need, 1, 8, 3, None) == _lib.ERR_MISALIGNED
        assert fn(ok, ok, ok, need - 1, 1, 8, 3, None) == _lib.ERR_WORKSPACE_TOO_SMALL
        assert L.dirt_last_launch_count() == 0
    for name in ('dirt_cubemap_sh_project_bytes', 'dirt_cubemap_sh_project', 'dirt_cubemap_sh_project_backward'):
        assert name in _lib.EXPORTED_SYMBOLS
